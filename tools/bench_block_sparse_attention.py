"""Cost of block-sparse attention layers on one GPU.  Prints JSON lines, each with the GPU name, its power limit and
SM clocks, read in the same run:

  * attention kernels at the dalle_example shape (B 32, H 4, dh 128, S 1280 = 256 text + 1024 image tokens, b 16,
    local window 4): forward and backward (delta pre-pass + dQ + dK/dV) device time per launch and TFLOP/s of the
    pairs each computes (4 dh B H per pair and product; ops.attn_pairs_block_sparse, causal: S^2 / 2, the count
    bench.py uses), for global and block-sparse at R = 0, 5 and 20 random blocks.  Each variant is 20 launches
    captured in a CUDA graph and timed with CUDA events around its replay; 3 rounds, variants alternated;
  * attn_decode per launch at the same shape (32 rows, positions 300, 700 and 1279), global against block-sparse;
  * the training step in tokens/s of configs/dalle_example_b200.json with {"attention_types": [[["block_sparse",
    "global"], 3]]} against that config all-global, measured as bench.py measures `value`, alternated over --rounds
    rounds in one process;
  * generate_graphed images/s at the dalle_example shape (random-init weights, 32 captions, temperature 1) for all
    layers global against [block_sparse, global] x 3, alternated over 3 rounds.

    python tools/bench_block_sparse_attention.py --steps 10 --warmup 3 --rounds 3
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tools.bench_conv_attention import gpu_info, graph_of, LAUNCHES, ROUNDS  # noqa: E402

B, H, DH, TL, IL = 32, 4, 128, 256, 1024
S = TL + IL
MIXED = ["block_sparse", "global"] * 3
WORKLOAD = "dalle_example_block_sparse"
bench.WORKLOADS.setdefault(WORKLOAD, bench.WORKLOADS["dalle_example"])
_load_params = bench.load_params


def _load_with_block_sparse(n_gpus, workload="dalle_example", scaling="weak"):
    """bench.load_params, with dalle_example's layers made [block_sparse, global] x 3 for WORKLOAD."""
    p = _load_params(n_gpus, "dalle_example" if workload == WORKLOAD else workload, scaling)
    if workload == WORKLOAD:
        p["attention_types"] = [[["block_sparse", "global"], 3]]
    return p


bench.load_params = _load_with_block_sparse


def masks(ops):
    from dalle_mtf_b200.dalle_engine import block_sparse_layout
    return {f"block_sparse_R{R}": ops.BlockSparse(block_sparse_layout(S, TL, 16, 4, R, 0, 0), 16, S)
            for R in (0, 5, 20)}


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
    variants = {"global": {}, **{k: {"block_sparse": m} for k, m in masks(ops).items()}}
    graphs = {}
    for name, kw in variants.items():
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
        kw = variants[name]
        pairs = kw["block_sparse"].pairs(S) if kw else ops.attn_pairs(S)
        flops = 4.0 * pairs * DH * B * H * (1.0 if kind == "fwd" else 2.5)
        print(json.dumps({"metric": "attention_us_per_launch", "kind": kind, "layer": name,
                          "shape": {"B": B, "H": H, "dh": DH, "S": S, "text_len": TL, "block": 16}, "pairs": pairs,
                          "rounds_us": [round(v, 1) for v in t], "min_us": round(min(t), 1),
                          "pair_tflops_at_min": round(flops / (min(t) * 1e-6) / 1e12, 1), **info}), flush=True)


def decode(info):
    from dalle_mtf_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(1)
    kc = torch.randn(B, S, H, DH, device="cuda", generator=gen).to(torch.bfloat16)
    vc = torch.randn(B, S, H, DH, device="cuda", generator=gen).to(torch.bfloat16)
    step = torch.randn(B, 3, H, DH, device="cuda", generator=gen).to(torch.bfloat16)
    out = torch.empty(B, H, DH, dtype=torch.bfloat16, device="cuda")
    variants = {"global": {}, "block_sparse_R20": {"block_sparse": masks(ops)["block_sparse_R20"]}}
    for pos in (300, 700, S - 1):
        graphs = {k: graph_of(lambda kw=kw: ops.attn_decode(step, kc, vc, out, pos, 1.0, **kw))
                  for k, kw in variants.items()}
        us = {k: [] for k in graphs}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(ROUNDS):
            for k, g in graphs.items():
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                us[k].append(e0.elapsed_time(e1) * 1000.0 / LAUNCHES)
        for k, t in us.items():
            print(json.dumps({"metric": "attn_decode_us_per_launch", "layer": k, "pos": pos, "rows": B,
                              "rounds_us": [round(v, 2) for v in t], "min_us": round(min(t), 2), **info}), flush=True)


def step(info, a):
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    args = argparse.Namespace(gpus=1, scaling="weak", dump_outputs=None, no_cpu_baseline=True)
    runs = {"dalle_example": [], WORKLOAD: []}
    for _ in range(a.rounds):
        for w in runs:
            line = bench.measure_dalle(args, dp, device, w, a.steps, max(a.warmup, 3), full=False)
            runs[w].append({k: line[k] for k in ("value", "ms_per_step", "loss", "clocks")})
    base = [r["ms_per_step"] for r in runs["dalle_example"]]
    bs = [r["ms_per_step"] for r in runs[WORKLOAD]]
    print(json.dumps({"metric": "tokens_per_sec", "unit": "tokens/s", "steps": a.steps, "runs": runs,
                      "block_sparse_step_time_ratio": (sum(bs) / len(bs)) / (sum(base) / len(base)), **info}),
          flush=True)
    dp.shutdown()


def generation(info):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.sampling import DalleSampler
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (32, TL), generator=g).to(torch.int32).cuda()
    samplers = {}
    for name, types in (("global", None), ("block_sparse_global_x3", MIXED)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, IL, attention_types=types)
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
    decode(info)
    generation(info)
    step(info, a)
    return 0


if __name__ == "__main__":
    sys.exit(main())
