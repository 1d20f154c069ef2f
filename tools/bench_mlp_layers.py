"""Cost of gMLP token-mixing layers ("mlp" in attention_types) on one GPU.  Prints JSON lines:

  * per-launch device time of the three causal mixing products (sgu_mix_fwd, sgu_mix_dgrad, sgu_mix_wgrad) at
    dalle_example (B = 32, S = 1 280, 2d = 1 024) and at the dalle_coco width (B = 8, S = 1 280, 2d = 2 048), with the
    TFLOP/s of the triangle each computes (2 B C x the S (S + 1) / 2 lower-triangle entries): CUDA events around
    LAUNCHES launches, ROUNDS rounds;
  * sgu_decode per launch at the last position of dalle_example (32 rows, S = 1 280, 2d = 1 024);
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1 024 image positions, B = 32: forward, backward and
    the Adam step) with attention_types [[["axial_row", "axial_col", "mlp"], 2]] against all-global layers, alternated
    over ROUNDS rounds of STEPS steps;
  * generate_graphed images/s of the same pair (B = 8, greedy), alternated.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402
from tools.bench_gelu import gpu_info, timed  # noqa: E402

LAUNCHES, ROUNDS, STEPS, GEN_B = 20, 5, 3, 8
TL, W = 256, 32
SHAPES = {"dalle_example": (32, 1280, 1024), "dalle_coco": (8, 1280, 2048)}
MIXED = ["axial_row", "axial_col", "mlp"] * 2


def kernel_rows(info):
    for name, (B, S, C) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        bf = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
        w = torch.tril(torch.randn(S, S, device="cuda", generator=g) * S ** -0.5).to(torch.bfloat16)
        gn, res, h, mixed, dm, dgn = (bf(B * S, C) for _ in range(6))
        c = torch.ones(S, device="cuda")
        dw = torch.zeros(S, S, device="cuda")
        flop = 2.0 * B * C * S * (S + 1) / 2
        variants = {"sgu_mix_fwd": lambda: ops.sgu_mix_fwd(w, gn, res, c, h, mixed, B, S),
                    "sgu_mix_dgrad": lambda: ops.sgu_mix_dgrad(w, dm, dgn, B, S),
                    "sgu_mix_wgrad": lambda: ops.sgu_mix_wgrad(dm, gn, dw, B, S)}
        for fn in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, fn in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            print(json.dumps({"bench": "sgu_mix_launch", "shape": name, "kernel": k, "B": B, "S": S, "C": C,
                              "us_per_launch_min": 1e3 * min(v), "TFLOPs_triangle": flop / min(v) / 1e9,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del gn, res, h, mixed, dm, dgn, dw
        torch.cuda.empty_cache()
    rows, S, C = 32, 1280, 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    w = torch.tril(torch.randn(S, S, device="cuda", generator=g) * S ** -0.5).to(torch.bfloat16)
    cache = torch.randn(rows, S, C, device="cuda", generator=g).to(torch.bfloat16)
    gn, res, h = (torch.randn(rows, C, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3))
    c = torch.ones(S, device="cuda")
    fn = lambda: ops.sgu_decode(gn, res, w, c, cache, h, S - 1)  # noqa: E731
    timed(fn, 3)
    v = [timed(fn, 50) for _ in range(ROUNDS)]
    print(json.dumps({"bench": "sgu_decode_launch", "rows": rows, "S": S, "C": C, "pos": S - 1,
                      "us_per_launch_min": 1e3 * min(v), "cache_TBps": rows * S * C * 2 / min(v) / 1e9,
                      "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)


def _engine(types):
    return DalleEngine(512, 6, 4, 50258, 512, TL, W * W, attention_types=types)


def step_rows(info):
    B, IL = 32, W * W
    engines = {"global": _engine(None), "axial_axial_mlp": _engine(MIXED)}
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, 50258 + 512, (B, TL + IL), device="cuda", generator=g, dtype=torch.int32)
    T = tokens.numel()

    def step(eng):
        eng.zero_grads()
        eng.forward(tokens, step=None)
        eng.backward(1.0 / T)
        eng.optimizer_step(1e-4)

    for eng in engines.values():
        eng.init_params(seed=0)
        for _ in range(2):
            step(eng)
    ms = {k: [] for k in engines}
    for _ in range(ROUNDS):
        for k, eng in engines.items():
            ms[k].append(timed(lambda: step(eng), STEPS))
    for k, v in ms.items():
        print(json.dumps({"bench": "dalle_example_step", "layers": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k, types in (("global", None), ("axial_axial_mlp", MIXED)):
        eng = _engine(types)
        eng.init_params(seed=0)
        samplers[k] = DalleSampler(eng)
    text = torch.randint(0, 50257, (GEN_B, TL), dtype=torch.int32, device="cuda")
    for s in samplers.values():
        s.generate_graphed(text, temperature=0.0)            # capture
    rates = {k: [] for k in samplers}
    for _ in range(3):
        for k, s in samplers.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s.generate_graphed(text, temperature=0.0)
            torch.cuda.synchronize()
            rates[k].append(GEN_B / (time.perf_counter() - t0))
    for k, v in rates.items():
        print(json.dumps({"bench": "generate_graphed", "layers": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
