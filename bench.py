#!/usr/bin/env python
"""bench.py — throughput of the DALL-E data-parallel training step (the north-star hot path) on N H100s.

    python bench.py --gpus 1 --steps 10 --warmup 3              # N=1
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
           bench.py --gpus N --steps K --warmup W                # N>1, one rank per GPU over NCCL
    python bench.py --impl reference ...                         # the CPU restatement of the reference on host cores
    python bench.py --gpus 1 --steps 10 --dump-outputs DIR       # also write the last timed step's results as .npy

Workload (config.workload): configs/dalle_example_b200.json = BASELINE.json configs[1]: n_embd 512, 6 layers, 4 heads,
sequence 256 text + 1024 image tokens (dataset.image_size 256 through the 3-stage vae_example tokenizer), bf16,
32 sequences per GPU (weak scaling: global batch = 32 * N).  A "step" = VAE-encode the images to token ids, assemble
text|image tokens, forward, backward, bucketed gradient all-reduce, clip-by-global-norm + Adam.

One JSON line on rank 0:
  value        whole-job tokens/s with the step's inputs (images, captions) already resident in HBM
  e2e          same through the public API (dalle_model_fn's train_op) with PINNED HOST inputs: the H2D copy of
               the images / captions and a D2H read of the loss are inside the timed region, every step
  roofline     the dominant kernel (wgmma GEMM, all launches of a step): algorithmic 2*M*N*K FLOPs / CUDA-event
               time of those launches, against MEASURED_PEAKS.json's sustained bf16 figure (else the H100 SXM data
               sheet's dense bf16 rate, which a power-limited card does not reach)

--dump-outputs DIR writes, after the timed steps of the headline workload, what its last timed step returned to the
caller: the loss, the token ids it trained on (VAE codes of the images after the caption) and a fixed, seeded sample of
the updated fp32 parameters (with their flat indices).  Inputs and initial weights are seeded, so two builds run with
the same arguments can be compared output for output.  Every sum over CTAs in the DALL-E step is added in a fixed order
(no float atomics), so a build writes bit-identical outputs on every run.
  cpu_baseline the oracle (CPU port of the reference math, "reference-faithful" variant: one-hot embedding / CE,
               materialised attention) timed on the box's host cores on a bounded sample of the same workload
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PER_GPU_BATCH = 32
METRIC = "tokens_per_sec"
UNIT = "tokens/s"


WORKLOADS = {
    # name: (config file, sequences per GPU, d, layers, vocab)
    "dalle_example": ("dalle_example_b200.json", 32, 512, 6, 50771),
    "dalle_coco": ("dalle_coco_b200.json", 16, 1024, 24, 50258 + 8192 + 1),
    # BASELINE.json configs[4] width (d = 4096, 32 heads) at 40 layers = 8.5 B parameters, so that bf16 weights + fp32
    # gradients + 1/8 of the optimiser state + activations fit an 80 GB GPU; optimiser state sharded over the
    # data-parallel ranks (needs >= 2 GPUs, sized for 8), per-block recompute, synthetic inputs, throughput only
    "dalle_12b": ("dalle_12b_b200.json", 4, 4096, 40, 50258 + 8192 + 1),
}


def per_gpu_batch_for(workload, n_gpus, scaling):
    """weak: the per-GPU batch is fixed (32 sequences for dalle_example) and the global batch grows with N;
    strong: the GLOBAL batch is fixed at the weak per-GPU figure (the config's own train_batch_size: 32 -> 4 / GPU at
    N = 8, SURVEY.md §7 "hard parts") and each GPU's share shrinks."""
    per_gpu = WORKLOADS[workload][1]
    if scaling == "strong":
        if per_gpu % n_gpus:
            raise SystemExit(f"strong scaling: global batch {per_gpu} is not divisible by {n_gpus} GPUs")
        return per_gpu // n_gpus
    return per_gpu


N_LAYERS_OVERRIDE = None   # --n-layers: smoke runs of a big workload with fewer layers (shown in config.workload)


def load_params(n_gpus, workload="dalle_example", scaling="weak"):
    from dalle_mtf_b200.utils import fetch_model_params
    cfg = WORKLOADS[workload][0]
    per_gpu = per_gpu_batch_for(workload, n_gpus, scaling)
    p = fetch_model_params(os.path.join(ROOT, "configs", cfg))
    p["vae_params"] = fetch_model_params(os.path.join(ROOT, "configs", p["vae_model"] + ".json"))
    p["train_batch_size"] = per_gpu * n_gpus
    p["mesh_shape"] = f"data:{n_gpus}"
    p["vae_random_init"] = True        # no pretrained VAE checkpoint in a throughput run (random-init weights)
    p["padding_id"] = 50257
    p["model_path"] = None
    if N_LAYERS_OVERRIDE:
        p["n_layers"] = int(N_LAYERS_OVERRIDE)
    return p


def csrc_hash():
    """sha256 over the CUDA sources the .so is built from: ties a bench line or an output dump to the build it came from."""
    import glob
    import hashlib
    h = hashlib.sha256()
    for f in sorted(glob.glob(os.path.join(ROOT, "dalle_mtf_b200", "csrc", "*.cu*"))):
        h.update(os.path.basename(f).encode())
        h.update(open(f, "rb").read())
    return h.hexdigest()[:16]


def vae_train_flops_per_image(convblocks, size, K, C=3):
    """Algorithmic FLOPs of one discrete-VAE training step per image (SURVEY.md §8d: fwd + bwd = 3 x fwd; transposed
    convolutions counted at k^2/s^2 = 4 taps per output pixel): vae_example 4.03 GFLOP, vae_coco (K=8192) 1 221.6."""
    f, cin, r = 0, C, size
    for stack, ch in convblocks:
        r //= 2
        f += 2 * r * r * 16 * cin * ch + (stack - 1) * 2 * (2 * r * r * 9 * ch * ch)
        cin = ch
    f += 2 * (2 * r * r * cin * K)
    for stack, ch in reversed(convblocks):
        r *= 2
        f += 2 * r * r * 4 * cin * ch + (stack - 1) * 2 * (2 * r * r * 9 * ch * ch)
        cin = ch
    f += 2 * r * r * cin * C
    return 3 * f


def cpu_vae_step_rate(p, steps=3, warmup=1):
    """BASELINE.json configs[0] is literally "on reference CPU mesh-tensorflow": the oracle's VAE training step
    (src/vae_tf/models.py:165-184 + tf Adam, src/model_fns_tf.py:58-66) timed on the host cores, full batch."""
    from oracle import optim as OO
    from oracle import vae as OV
    cores = usable_cores()
    torch.set_num_threads(cores)
    cb, K, size, B = p["convblocks"], p["num_tokens"], p["dataset"]["image_size"], p["train_batch_size"]
    g = torch.Generator().manual_seed(1234)
    params = OV.init_params(cb, K, seed=0)
    m = {k: torch.zeros_like(v) for k, v in params.items()}
    v = {k: torch.zeros_like(v_) for k, v_ in params.items()}
    hw = size // (2 ** len(cb))
    times = []
    for it in range(warmup + steps):
        img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
        u = torch.rand(B, hw, hw, K, generator=g).clamp_(1e-9, 1.0)
        t0 = time.perf_counter()
        _, _, _, grads = OV.loss_and_grads(params, img, u, cb, 1.0, bool(p.get("train_gumbel_hard", True)),
                                           bf16=False)
        for k in params:
            params[k], m[k], v[k] = OO.adam_tf_step(params[k], m[k], v[k], grads[k], p["lr"], it + 1)
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
    mean = sum(times) / len(times)
    return {"value": B / mean, "unit": "imgs/s", "cores": cores, "kind": "port", "ms_per_step": mean * 1e3,
            "sample": f"{steps} full steps of batch {B} ({size}x{size}), fp32, fwd+bwd+Adam"}


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        return d.get("bf16_tflops_sustained", 989.0), d.get("hbm_gbs", 3350.0), "measured"
    return 989.0, 3350.0, "H100 SXM data sheet"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.samples = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.idx)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append((time.time(), line.strip()))

    def mark(self):
        return time.time()

    def stop(self, t0=None, t1=None):
        """Summarise the samples taken inside [t0, t1] (the timed region); if the region was shorter than the sampling
        period, fall back to every sample taken under load (warm-up included)."""
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        inside = [s for ts, s in self.samples if t0 is not None and t0 <= ts <= t1]
        window = "timed region" if inside else "warm-up + timed region"
        sm, mx, reasons = [], None, set()
        for s in (inside or [s for _, s in self.samples]):
            f = [x.strip() for x in s.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm), "window": window}


def usable_cores():
    """Host cores this process may actually use: scheduler affinity, capped by the cgroup CPU quota if there is one
    (os.cpu_count() reports the whole machine inside a container and oversubscribing it is far slower)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(int(txt[0]) / int(txt[1]))))
            else:
                q = int(txt[0])
                per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                if q > 0:
                    n = min(n, max(1, q // per))
        except Exception:
            pass
    return max(1, n)


def cpu_reference_step_rate(steps, warmup, seqs, label):
    """Times the oracle's reference-faithful fp32 training step (fwd + bwd + clip + Adam) on the host cores.
    Returns tokens/s.  This is the ONLY place bench.py executes oracle/ (as the CPU baseline, never as product)."""
    from oracle import dalle as O
    from oracle import optim as OO
    cores = usable_cores()
    torch.set_num_threads(cores)
    cfg = O.DalleConfig(512, 6, 4, 50258, 512, 256, 1024)
    params = O.init_params(cfg, 0)
    m = {k: torch.zeros_like(v) for k, v in params.items()}
    v = {k: torch.zeros_like(v_) for k, v_ in params.items()}
    g = torch.Generator().manual_seed(1234)
    hp = {"lr": 1e-3, "train_steps": 100000}
    times = []
    for it in range(warmup + steps):
        tokens = torch.randint(0, cfg.total_tokens - 1, (seqs, cfg.seq_len), generator=g)
        t0 = time.perf_counter()
        leaves = {k: p.clone().requires_grad_(True) for k, p in params.items()}
        loss, _, _ = O.forward(leaves, tokens, cfg, bf16=False, faithful=True)
        loss.backward()
        grads = {k: p.grad for k, p in leaves.items()}
        params, m, v, _, _ = OO.dalle_train_step(params, m, v, grads, 3000 + it, hp)
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
    mean = sum(times) / len(times)
    return seqs * cfg.seq_len / mean, mean * 1e3, cores, f"{label}: {seqs} sequences x 1280 tokens per step, fp32, " \
        f"fwd+bwd+clip+Adam, reference-faithful graph (one-hot embedding/CE, materialised [S,S] attention)"


def vae_example_rate(dp, device, steps=20, warmup=5, config="vae_example", per_gpu_batch=None, cpu_baseline=False):
    """Second half of BASELINE.json's metric: discrete-VAE training images/s through vae_model_fn's train_op.
    Default: configs/vae_example.json (CIFAR-10-shaped 32x32 inputs, 3-stage VAE, batch 32, fp32, hard Gumbel)."""
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    p = fetch_model_params(os.path.join(ROOT, "configs", config + ".json"))
    p["_dp"] = dp
    p["model_path"] = None
    if per_gpu_batch:
        p["train_batch_size"] = per_gpu_batch * dp.world
    it = iter(vae_input_fn(p))
    batches = [next(it)[0].to(device) for _ in range(4)]
    spec = vae_model_fn(batches[0], batches[0], TRAIN, p)
    for i in range(warmup):
        spec.train_op(batches[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        spec.train_op(batches[i % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    peak_tf, _, peak_kind = measured_peaks()
    f_img = vae_train_flops_per_image(p["convblocks"], p["dataset"]["image_size"], p["num_tokens"])
    imgs_s = p["train_batch_size"] * 1000.0 / ms
    achieved = imgs_s / dp.world * f_img / 1e12
    line = {"metric": "vae_imgs_per_sec", "value": imgs_s, "unit": "imgs/s", "ms_per_step": ms, "n_gpus": dp.world,
            "roofline": {"kernel": "whole step (convolutions + codebook matmuls are the tensor-bound part)",
                         "bound": "tensor", "achieved": achieved, "peak": peak_tf, "unit": "TFLOP/s",
                         "frac": achieved / peak_tf, "peak_kind": f"bf16_tflops_sustained ({peak_kind})",
                         "flops_per_image": f_img, "traffic": None},
            "config": f"{config}: {p['dataset']['image_size']}^2x3, convblocks {p['convblocks']}, K={p['num_tokens']}, "
                      f"global batch {p['train_batch_size']}, {'bf16' if p.get('use_bf16') else 'fp32'} activations, "
                      f"{'hard' if p.get('train_gumbel_hard') else 'soft'} Gumbel; fwd+bwd+Adam",
            "loss": float(spec.loss_sum.item()) * spec.loss_scale}
    if cpu_baseline and dp.rank == 0:
        line["cpu_baseline"] = cpu_vae_step_rate(p)
    del spec
    torch.cuda.empty_cache()
    return line


def measure_dalle(args, dp, device, workload, steps, warmup, full):
    """One DALL-E workload: `value` (device-resident inputs), `e2e` (pinned host inputs through train_op), GEMM and
    attention rooflines from CUDA events around every launch.  full=True adds the VAE line and the CPU baselines."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    from dalle_mtf_b200.input_fns import dalle_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn
    params = load_params(args.gpus, workload, args.scaling)
    params["_dp"] = dp
    cfg_file, _, d_model, n_layers, vocab = WORKLOADS[workload]
    n_layers = params["n_layers"]
    per_gpu_batch = per_gpu_batch_for(workload, args.gpus, args.scaling)
    it = iter(dalle_input_fn(params))
    host_batches = [next(it) for _ in range(4)]                 # pinned host memory
    dev_batches = [(f.to(device), l.to(device)) for f, l in host_batches]   # 4 x 25 MB of images: rotated every step
    spec = dalle_model_fn(host_batches[0][0], host_batches[0][1], TRAIN, params)
    spec.global_step = 3000   # past the linear warm-up so the update is not a no-op (lr(0) = 0)
    tokens_per_step = spec.tokens_per_step
    sampler = ClockSampler(dp.local_rank)

    def timed(batches, steps, read_loss):
        dp.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            f, l = batches[i % len(batches)]
            loss = spec.train_op(f, l)
            if read_loss:
                _ = float(loss.item())          # D2H read of the step's result, every step
        e1.record()
        torch.cuda.synchronize(); dp.barrier()
        return dp.max_over_ranks(e0.elapsed_time(e1))

    # ---- device-resident inputs: `value`
    sampler.start()                      # nvidia-smi needs a moment to start: launch it before the warm-up
    timed(dev_batches, warmup, False)
    ops.GEMM_PROFILE, ops.ATTN_PROFILE = [], []
    n0 = L.launch_count()
    t_begin = sampler.mark()
    ms_total = timed(dev_batches, steps, False)
    t_end = sampler.mark()
    if full and args.dump_outputs and dp.rank == 0:
        dump_outputs(args.dump_outputs, spec)
    launches = L.launch_count() - n0
    prof, ops.GEMM_PROFILE = ops.GEMM_PROFILE, None
    aprof, ops.ATTN_PROFILE = ops.ATTN_PROFILE, None
    attn = {}
    for kind in ("fwd", "bwd"):
        ms_k = sum(a.elapsed_time(b) for a, b, _, k in aprof if k == kind)
        fl_k = sum(f for _, _, f, k in aprof if k == kind)
        n_k = sum(1 for *_, k in aprof if k == kind)
        if ms_k > 0:
            attn[kind] = {"tflops": fl_k / (ms_k * 1e-3) / 1e12, "us_per_launch": 1e3 * ms_k / n_k,
                          "launches_per_step": n_k / steps, "share_of_step": ms_k / ms_total}
    ms_per_step = ms_total / steps
    value = tokens_per_step * 1000.0 / ms_per_step
    gemm_ms = sum(a.elapsed_time(b) for a, b, _, _ in prof)
    gemm_flops = sum(f for _, _, f, _ in prof)
    if os.environ.get("DB200_BENCH_VERBOSE") and dp.rank == 0:
        agg = {}
        for a, b, f, tag in prof:
            e = agg.setdefault(tag, [0, 0.0, 0.0])
            e[0] += 1; e[1] += a.elapsed_time(b); e[2] += f
        for tag, (n, ms, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            print(f"  gemm M={tag[0]:6d} N={tag[1]:6d} K={tag[2]:6d} mode={tag[3]} a_mn={tag[4]} b_mn={tag[5]}: n/step={n / steps:5.1f} "
                  f"ms/step={ms / steps:7.3f} {fl / ms / 1e9:7.1f} TFLOP/s", file=sys.stderr)
    peak_tf, _, peak_kind = measured_peaks()
    achieved_tf = gemm_flops / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else 0.0
    loss_now = float(spec.loss_sum.item()) * spec.loss_scale

    # ---- host inputs through the public API: `e2e`
    timed(host_batches, 2, True)
    ms_e2e = timed(host_batches, steps, True) / steps
    clocks = sampler.stop(t_begin, t_end)
    vae_line = None
    if full and workload == "dalle_example":   # second half of the metric: VAE imgs/s (BASELINE configs[0]) at N GPUs
        vae_line = vae_example_rate(dp, device, cpu_baseline=(args.gpus == 1 and not args.no_cpu_baseline))
    f0, l0 = host_batches[0]
    h2d = f0.numel() * f0.element_size() + l0.numel() * l0.element_size()

    line = None
    if dp.rank == 0:
        d, Lyr, S, V = d_model, n_layers, 1280, vocab
        f_tok = 3 * (Lyr * (24 * d * d + 2 * S * d) + 2 * d * V)     # BASELINE.md §4 training FLOPs per token
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": steps,
            "warmup": warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": args.scaling,
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": (f"{cfg_file[:-5]}: n_embd={d} n_layers={Lyr} n_heads={params['n_heads']} "
                                    f"seq=256+1024 (image_size 256 -> {params['vae_model']} tokenizer -> 1024 image "
                                    f"tokens), V={V}" + (", recompute_grad" if params.get("recompute_grad") else "")),
                       "global_batch": per_gpu_batch * args.gpus, "per_gpu_batch": per_gpu_batch, "seq_len": S,
                       "parallelism": f"dp{args.gpus}", "step": "vae-encode + fwd + bwd + allreduce + clip + adam",
                       "l2": "inputs rotate over 4 batches; each step streams several GB of activations (>> 50 MB L2)"},
            "tokens_per_sec_per_gpu": value / args.gpus,
            "model_flops_fraction": (value / args.gpus) * f_tok / (peak_tf * 1e12),
            "loss": loss_now,
            "e2e": {"value": tokens_per_step * 1000.0 / ms_e2e, "unit": UNIT, "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4},
            "gpu_launches": int(launches),
            "csrc_hash": csrc_hash(),
            "clocks": clocks,
            "roofline": {"kernel": "gemm_tc_kernel (wgmma, all launches of the step)", "bound": "tensor",
                         "achieved": achieved_tf, "peak": peak_tf, "unit": "TFLOP/s", "frac": achieved_tf / peak_tf,
                         "peak_kind": f"bf16_tflops_sustained ({peak_kind})",
                         "traffic": None,
                         "launches_per_step": len(prof) / steps, "share_of_step": gemm_ms / ms_total,
                         "flops_per_launch": gemm_flops / max(len(prof), 1)},
            # second roofline: the causal attention kernels (wgmma), causal-algorithmic FLOPs
            # (forward 4 S^2 dh B H / 2, backward 2.5 x) / CUDA-event time of their launches
            "roofline_attention": {k: dict(v, frac=v["tflops"] / peak_tf, peak=peak_tf, unit="TFLOP/s", bound="tensor")
                                   for k, v in attn.items()},
        }
        if vae_line is not None:
            line["vae"] = vae_line
        if full and args.gpus == 1 and not args.no_cpu_baseline and workload == "dalle_example":
            v, ms, cores, sample = cpu_reference_step_rate(2, 1, 2, "bounded sample")
            line["cpu_baseline"] = {"value": v, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
                                    "ms_per_step": ms}
    del spec
    torch.cuda.empty_cache()
    return line


DUMP_PARAM_SAMPLE = 1 << 21   # 8 MiB of fp32 values + 16 MiB of float64 indices


def dump_outputs(out_dir, spec):
    """What the timed train_op computed in its last step, as float32 / float64 .npy files (see the module doc)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    eng = spec.engine
    torch.cuda.synchronize()
    loss = float(spec.loss_sum.item()) * spec.loss_scale
    np.save(os.path.join(out_dir, "loss.npy"), np.array([loss], dtype=np.float64))
    tokens = getattr(eng, "_tokens", None)     # the (last micro-batch's) tokens of the step's forward
    if tokens is not None:
        np.save(os.path.join(out_dir, "tokens.npy"), tokens.detach().cpu().numpy().astype(np.float64))
    master = eng.master[:eng.n_params_padded] if eng.zero is None else eng.master
    n = master.numel()
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, n, (min(DUMP_PARAM_SAMPLE, n),), generator=g).sort().values
    vals = master[idx.to(master.device)].float().cpu().numpy()
    np.save(os.path.join(out_dir, "params_sample.npy"), vals.astype(np.float32))
    np.save(os.path.join(out_dir, "params_sample_index.npy"), idx.numpy().astype(np.float64))


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    seqs = 2
    args.steps = min(args.steps, 3)      # bounded: the whole run must end within a few minutes
    value, ms, cores, sample = cpu_reference_step_rate(args.steps, min(args.warmup, 1), seqs, "bounded sample")
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": min(args.warmup, 1), "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "dalle_example_b200 (n_embd=512 n_layers=6 n_heads=4 seq=256+1024)", "cpu_sample": sample},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "note": "mesh-tensorflow/TF 2.4 cannot be installed here (Python 3.12, no network): the oracle port of the "
                "reference math stands in for the reference's CPU path",
    }
    print(json.dumps(line), flush=True)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", type=str, default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--workload", type=str, default="dalle_example", choices=sorted(WORKLOADS),
                    help="dalle_example = BASELINE.json configs[1] (the default, the headline workload); "
                         "dalle_coco = configs[3] shape (n_embd 1024, 24 layers, 16 heads, 16 sequences per GPU)")
    ap.add_argument("--scaling", type=str, default="weak", choices=["weak", "strong"],
                    help="weak: 32 sequences per GPU (global batch 32 N); strong: global batch fixed at 32 (32 / N per GPU)")
    ap.add_argument("--n-layers", type=int, default=0,
                    help="override the workload's layer count (smoke runs only; the line's config names the override)")
    ap.add_argument("--no-extra", action="store_true", help="skip the bounded dalle_coco / vae_coco side measurements")
    ap.add_argument("--vae-example", action="store_true",
                    help="measure only configs/vae_example.json (BASELINE configs[0]: 32x32, fp32, batch 32)")
    ap.add_argument("--dump-outputs", type=str, default=None, metavar="DIR",
                    help="after the timed steps, write the last timed step's loss, token ids and a seeded sample of "
                         "the updated parameters to DIR/<name>.npy")
    ap.add_argument("--vae-coco", action="store_true",
                    help="measure configs/vae_coco_b200.json (256x256, K=8192, bf16, 16 images per GPU) instead")
    args = ap.parse_args()
    if args.n_layers:
        global N_LAYERS_OVERRIDE
        N_LAYERS_OVERRIDE = args.n_layers
    if args.impl == "reference":
        return run_reference(args)
    args.warmup = max(args.warmup, 3)

    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops
    from dalle_mtf_b200.dist import DataParallel
    from dalle_mtf_b200.input_fns import dalle_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn

    dp = DataParallel().init()
    if dp.world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={dp.world}: launch with torch.distributed.run")
    L.require_device()
    device = torch.device("cuda", torch.cuda.current_device())
    if args.vae_coco or args.vae_example:
        if args.vae_coco:
            line = vae_example_rate(dp, device, steps=args.steps, warmup=args.warmup, config="vae_coco_b200",
                                    per_gpu_batch=16)
        else:
            line = vae_example_rate(dp, device, steps=args.steps, warmup=args.warmup)
        line.update({"n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup})
        if dp.rank == 0:
            print(json.dumps(line), flush=True)
        dp.shutdown()
        return 0
    line = measure_dalle(args, dp, device, args.workload, args.steps, args.warmup, full=True)
    if line is not None and args.gpus == 1 and args.workload == "dalle_example" and not args.no_extra:
        # BASELINE.json's other single-GPU-measurable configurations, bounded, measured in the same run
        extra = {}
        try:
            extra["dalle_coco_b200"] = measure_dalle(args, dp, device, "dalle_coco", 5, 3, full=False)
            extra["vae_coco_b200"] = vae_example_rate(dp, device, steps=5, warmup=3, config="vae_coco_b200",
                                                      per_gpu_batch=16)
        except Exception as e:  # noqa: BLE001 — the headline line must survive a failure of the side measurements
            extra["error"] = f"{type(e).__name__}: {e}"
        line["extra"] = extra
    if dp.rank == 0 and line is not None:
        print(json.dumps(line), flush=True)
    dp.barrier()
    dp.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
