"""Cost of convolutional attention layers on one GPU.  Prints JSON lines, each with the GPU name, its power limit and
SM clocks, read in the same run:

  * attention kernels at the dalle_example shape (B 32, H 4, dh 128, S 1280 = 256 text + a 32 x 32 image grid):
    forward and backward (delta pre-pass + dQ + dK/dV) device time per launch and TFLOP/s of the pairs each computes
    (4 dh B H per pair and product; ops.attn_pairs / attn_pairs_axial / attn_pairs_conv, causal: S^2 / 2, the count
    bench.py uses), for global, row, and conv at kernel 5 and 11.  Each variant is 20 launches captured in a CUDA graph
    and timed with CUDA events around its replay; 3 rounds, variants alternated within each round;
  * the training step in tokens/s of configs/dalle_example_conv_b200.json ([axial_row, axial_col] x 2, axial_row,
    conv) against bench.py's headline dalle_example_b200, measured as bench.py measures `value`, alternated over
    --rounds rounds in one process;
  * generate_graphed images/s at the dalle_example shape (random-init weights, 32 captions, temperature 1) for all
    layers global against the conv config's layers, alternated over 3 rounds.

    python tools/bench_conv_attention.py --steps 10 --warmup 3 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

bench.WORKLOADS.setdefault("dalle_example_conv",
                           ("dalle_example_conv_b200.json",) + bench.WORKLOADS["dalle_example"][1:])
B, H, DH, TL, W = 32, 4, 128, 256, 32
S = TL + W * W
# name -> ops keyword arguments of the attention launch
VARIANTS = {"global": {}, "axial_row": {"axial": (TL, W, 0)}, "conv_k5": {"conv": (TL, W, 5)},
            "conv_k11": {"conv": (TL, W, 11)}}
LAUNCHES, ROUNDS = 20, 3
MIXED = ["axial_row", "axial_col"] * 2 + ["axial_row", "conv"]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock_max, clock = (q.stdout.strip().split(", ") + ["?"] * 4)[:4] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock_max, "sm_clock_now": clock}


def graph_of(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def kernels(info):
    from dalle_mtf_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, S, 3, H, DH, device="cuda", generator=gen)
    qkv[:, :, :2] *= 1.3 * DH ** -0.25
    qkv = qkv.to(torch.bfloat16)
    dout = torch.randn(B, S, H, DH, device="cuda", generator=gen).to(torch.bfloat16)
    out = torch.empty(B, S, H, DH, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, H, S, device="cuda")
    delta = torch.empty(B, H, S, device="cuda")
    dq = torch.zeros(1, device="cuda")
    dqkv = torch.empty_like(qkv)
    graphs = {}
    for name, kw in VARIANTS.items():
        graphs[(name, "fwd")] = graph_of(lambda kw=kw: ops.attn_fwd(qkv, out, lse, B, S, H, DH, 1.0, **kw))
        ops.attn_fwd(qkv, out, lse, B, S, H, DH, 1.0, **kw)
        graphs[(name, "bwd")] = graph_of(
            lambda kw=kw: ops.attn_bwd(qkv, out, dout, lse, dq, delta, dqkv, B, S, H, DH, 1.0, **kw))
    us = {k: [] for k in graphs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for k, g in graphs.items():
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            us[k].append(e0.elapsed_time(e1) * 1000.0 / LAUNCHES)
    for (name, kind), t in us.items():
        kw = VARIANTS[name]
        pairs = ops.attn_pairs_axial(S, *kw["axial"]) if "axial" in kw else \
            ops.attn_pairs_conv(S, *kw["conv"]) if "conv" in kw else ops.attn_pairs(S)
        flops = 4.0 * pairs * DH * B * H * (1.0 if kind == "fwd" else 2.5)
        print(json.dumps({"metric": "attention_us_per_launch", "kind": kind, "layer": name,
                          "shape": {"B": B, "H": H, "dh": DH, "S": S, "text_len": TL, "grid_w": W}, "pairs": pairs,
                          "rounds_us": [round(v, 1) for v in t], "min_us": round(min(t), 1),
                          "band_tflops_at_min": round(flops / (min(t) * 1e-6) / 1e12, 1), **info}), flush=True)


def step(info, a):
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    args = argparse.Namespace(gpus=1, scaling="weak", dump_outputs=None, no_cpu_baseline=True)
    runs = {"dalle_example": [], "dalle_example_conv": []}
    for _ in range(a.rounds):
        for w in runs:
            line = bench.measure_dalle(args, dp, device, w, a.steps, max(a.warmup, 3), full=False)
            runs[w].append({k: line[k] for k in ("value", "ms_per_step", "loss", "clocks")})
    base = [r["ms_per_step"] for r in runs["dalle_example"]]
    cv = [r["ms_per_step"] for r in runs["dalle_example_conv"]]
    print(json.dumps({"metric": "tokens_per_sec", "unit": "tokens/s", "steps": a.steps, "runs": runs,
                      "conv_step_time_ratio": (sum(cv) / len(cv)) / (sum(base) / len(base)), **info}), flush=True)
    dp.shutdown()


def generation(info):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.sampling import DalleSampler
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (32, 256), generator=g).to(torch.int32).cuda()
    samplers = {}
    for name, types in (("global", None), ("dalle_example_conv", MIXED)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, attention_types=types)
        eng.init_params(0)
        samplers[name] = DalleSampler(eng)
        samplers[name].generate_graphed(text, temperature=1.0)      # capture + warm-up
    torch.cuda.synchronize()
    ms = {k: [] for k in samplers}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for k, s in samplers.items():
            e0.record()
            s.generate_graphed(text, temperature=1.0)
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    for k, t in ms.items():
        print(json.dumps({"metric": "generated_images_per_sec", "path": "generate_graphed", "layers": k, "images": 32,
                          "rounds": [round(32 * 1000.0 / v, 2) for v in t], "ms_per_call": [round(v, 1) for v in t],
                          **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from dalle_mtf_b200 import lib as L
    L.require_device()
    info = gpu_info()
    kernels(info)
    generation(info)
    step(info, a)
    return 0


if __name__ == "__main__":
    sys.exit(main())
