"""Prompt prefill and image completion at the dalle_example_b200 shape (d=512, L=6, H=4, 256 text + 1024 image
positions, random-init weights, batch 32), on one GPU.  Prints JSON lines:

  * agreement at this size, before any timing: relative Frobenius error of DalleEngine.prefill's position-P logits
    against the full forward pass (eng.logits) on the same tokens, and of its K/V caches against the caches the
    teacher-forced per-position step (the captured prompt graph of generate_graphed) writes, per layer;
  * the prompt phase of a text-only prompt: 255 replays of the captured per-position prompt graph (what
    generate_graphed runs) against one prefill at P = 256, CUDA events around each;
  * images/s of generate_graphed (text only), complete (text only), complete with a 512-token image prefix and
    complete with 8 prompts x samples_per_prompt=4 (32 rows each), with noise at temperature 1.

Variants are alternated within each of ROUNDS rounds; every figure lists all rounds.  Every line carries the GPU name
and its power limit, read in the same run."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402

ROUNDS, BATCH, PREFIX = 3, 32, 512


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock = (q.stdout.strip().split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def relfro(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    L.require_device()
    info = gpu_info()
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    tv, iv, TL, S = eng.text_vocab_size, eng.image_vocab_size, eng.text_seq_len, eng.S
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (BATCH, TL), generator=g).to(torch.int32).cuda()
    image = torch.randint(0, iv, (BATCH, eng.image_seq_len), generator=g).to(torch.int32).cuda()
    tokens = torch.cat([text, image + tv], 1)

    # ---- agreement: prefill vs the full forward pass and vs the teacher-forced caches
    tf = DalleSampler(eng)
    tf._alloc(BATCH)
    tf._capture(BATCH, False, 1.0, None)
    kc = [torch.zeros_like(c) for c in tf.kc]
    vc = [torch.zeros_like(c) for c in tf.vc]
    for P in (TL, TL + PREFIX):
        tf.tokens.copy_(tokens)
        tf.pos_dev.zero_()
        for _ in range(P):
            tf.g_prompt.replay()
        logits = eng.prefill(tokens[:, :P].contiguous(), kc, vc)[:, :eng.V].clone()
        full = eng.logits(tokens)[:, P - 1]
        torch.cuda.synchronize()
        print(json.dumps({"metric": "prefill_agreement", "P": P, "batch": BATCH,
                          "logits_relfro_vs_full_forward": relfro(logits, full),
                          "k_relfro_vs_teacher_forced": [relfro(a[:, :P], b[:, :P]) for a, b in zip(kc, tf.kc)],
                          "v_relfro_vs_teacher_forced": [relfro(a[:, :P], b[:, :P]) for a, b in zip(vc, tf.vc)],
                          "layer0_kv_bit_identical": bool(torch.equal(kc[0][:, :P], tf.kc[0][:, :P]) and
                                                          torch.equal(vc[0][:, :P], tf.vc[0][:, :P])),
                          **info}))
    eng._bufs = eng._buf_key = None          # the training buffers of eng.logits are not needed from here on
    torch.cuda.empty_cache()

    # ---- prompt phase: 255 prompt-graph replays vs one prefill at P = 256
    def replays():
        tf.pos_dev.zero_()
        for _ in range(TL - 1):
            tf.g_prompt.replay()

    def prefill():
        return eng.prefill(text, kc, vc)

    replays(); prefill()
    torch.cuda.synchronize()
    ms = {"prompt_graph_replays": [], "prefill": []}
    for _ in range(ROUNDS):
        ms["prompt_graph_replays"].append(timed(replays)[0])
        ms["prefill"].append(timed(prefill)[0])
    flops = 2.0 * BATCH * TL * eng.L * 12 * eng.d ** 2          # the block GEMMs (24 d^2 per token and layer)
    for name, t in ms.items():
        print(json.dumps({"metric": "prompt_phase_ms", "path": name, "P": TL, "batch": BATCH,
                          "rounds": [round(v, 3) for v in t], "min": round(min(t), 3),
                          **({"block_gemm_tflops_per_s": round(flops / (min(t) * 1e-3) / 1e12, 1)}
                             if name == "prefill" else {}), **info}))

    # ---- images/s: one sampler per variant, so every timed call replays already captured graphs
    prefix = image[:, :PREFIX].contiguous()
    variants = {
        "generate_graphed (text)": lambda s: s.generate_graphed(text, temperature=1.0),
        "complete (text)": lambda s: s.complete(text, temperature=1.0),
        f"complete (text + {PREFIX} image tokens)": lambda s: s.complete(text, prefix, temperature=1.0),
        "complete (8 prompts x 4 samples)": lambda s: s.complete(text[:8].contiguous(), samples_per_prompt=4,
                                                                 temperature=1.0),
    }
    samplers = {name: DalleSampler(eng) for name in variants}
    for name, fn in variants.items():
        fn(samplers[name])
    torch.cuda.synchronize()
    ms = {name: [] for name in variants}
    for _ in range(ROUNDS):
        for name, fn in variants.items():
            t, out = timed(lambda: fn(samplers[name]))
            assert out.shape == (BATCH, S)
            ms[name].append(t)
    for name, t in ms.items():
        print(json.dumps({"metric": "generated_images_per_sec", "variant": name, "rows": BATCH,
                          "rounds": [round(BATCH * 1000.0 / v, 3) for v in t],
                          "ms_per_call": [round(v, 1) for v in t], **info}))


if __name__ == "__main__":
    main()
