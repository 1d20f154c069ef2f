"""Cost of the sandwich LayerNorm (sandwich_norm) on one GPU.  Prints JSON lines:

  * per-launch device time and TB/s of layernorm_residual_fwd against layernorm_fwd at dalle_example (T = 40 960 rows,
    d = 512), the dalle_coco width (T = 10 240, d = 1 024) and the 12B width (T = 5 120, d = 4 096), and of the
    layernorm_bwd each branch adds (no residual gradient, fused bias column sums), with and without residual dropout:
    CUDA events around LAUNCHES launches, ROUNDS rounds, the kernels alternated.  Bytes: layernorm_fwd reads and writes
    T x d bf16 and writes 2 T fp32; the residual variant also reads x (T x d bf16); layernorm_bwd reads dy and x and
    writes dx (and dxm with dropout), T x d bf16 each, and reads 2 T fp32;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) without and with the key, alternated over ROUNDS rounds of STEPS
    steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) without and with the key, alternated.

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

LAUNCHES, ROUNDS, STEPS, GEN_B = 50, 5, 5, 8
TL, W = 256, 32
SHAPES = {"dalle_example": (40960, 512), "dalle_coco": (10240, 1024), "12B": (5120, 4096)}


def kernel_rows(info):
    for name, (T, d) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        bf = lambda: torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
        o, x, dy, y, dx, dxm = bf(), bf(), bf(), bf(), bf(), bf()
        gam, bet = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
        mean, rstd = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
        dg, db, dsum = (torch.zeros(d, device="cuda") for _ in range(3))
        site = L.make_dropout(0.1, 0, 1, L.dropout_site_mlp_out(0), 0)
        tb = T * d * 2
        variants = {
            "layernorm_fwd": (lambda: ops.layernorm_fwd(o, gam, bet, y, mean, rstd), 2 * tb + 8 * T),
            "layernorm_residual_fwd": (lambda: ops.layernorm_residual_fwd(o, x, gam, bet, y, mean, rstd),
                                       3 * tb + 8 * T),
            "layernorm_bwd_branch": (lambda: ops.layernorm_bwd(dy, o, gam, mean, rstd, None, dx, dg, db, dxsum=dsum),
                                     3 * tb + 8 * T),
            "layernorm_bwd_branch_dropout": (lambda: ops.layernorm_bwd(dy, o, gam, mean, rstd, None, dx, dg, db,
                                                                       dxsum=dsum, dxm=dxm, dropout=site),
                                             4 * tb + 8 * T),
        }
        for fn, _ in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, (fn, _) in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            print(json.dumps({"bench": "sandwich_launch", "shape": name, "kernel": k, "rows": T, "d": d,
                              "us_per_launch_min": 1e3 * min(v), "TBps": variants[k][1] / min(v) / 1e9,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del o, x, dy, y, dx, dxm
        torch.cuda.empty_cache()


def step_rows(info):
    B, IL = 32, W * W
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, IL, sandwich_norm=on) for k, on in (("off", False),
                                                                                           ("on", True))}
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
        print(json.dumps({"bench": "dalle_example_step", "sandwich_norm": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "on_over_off_min": min(ms["on"]) / min(ms["off"]), **info}),
          flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k, on in (("off", False), ("on", True)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, sandwich_norm=on)
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
        print(json.dumps({"bench": "generate_graphed", "sandwich_norm": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
