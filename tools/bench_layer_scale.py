"""Cost of LayerScale (layer_scale) and the stable option on one GPU.  Prints JSON lines:

  * per-launch device time and TB/s of layer_scale_residual_fwd, layernorm_scale_residual_fwd (against
    layernorm_residual_fwd), layer_scale_bwd (plain, with residual dropout and with db, and the sandwich form),
    layernorm_divmax_fwd / _bwd (against layernorm_fwd / _bwd, the backward with the fused column sum and residual
    dropout the final LayerNorm runs) and embed_bwd with and without alpha at dalle_example (T = 40 960 rows, d = 512),
    the dalle_coco width (T = 10 240, d = 1 024) and the 12B width (T = 5 120, d = 4 096): CUDA events around LAUNCHES
    launches, ROUNDS rounds, the kernels alternated.  Bytes: layer_scale_residual_fwd reads o and x and writes y,
    T x d bf16 each; the LayerNorm forwards read x and write y (and x_res read) and 2 T fp32 (3 T with m);
    layer_scale_bwd reads dy and v and writes dv, T x d bf16 each (the sandwich form also reads 2 T fp32); the
    LayerNorm backwards read dy and x and write dx and dxm; embed_bwd reads dx (its scatter's traffic is not counted);
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) with neither key, layer_scale, stable and both, alternated over
    ROUNDS rounds of STEPS steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) with neither key and with both, alternated.

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
STEP_KEYS = {"off": {}, "layer_scale": {"layer_scale": True}, "stable": {"stable": True},
             "both": {"layer_scale": True, "stable": True}}


def kernel_rows(info):
    for name, (T, d) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        bf = lambda: torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
        o, x, dy, y, dv, dxm = bf(), bf(), bf(), bf(), bf(), bf()
        gam, bet = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
        s = torch.full((d,), 0.1, device="cuda")
        mean, rstd = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
        ds, db, dg, dsum = (torch.zeros(d, device="cuda") for _ in range(4))
        m = torch.empty(T, device="cuda")
        ids = torch.randint(0, 50771, (T // 1280, 1280), device="cuda", generator=g, dtype=torch.int32)
        dwte, dwpe = torch.zeros(50771, d, device="cuda"), torch.zeros(1280, d, device="cuda")
        site = L.make_dropout(0.1, 0, 1, L.dropout_site_mlp_out(0), 0)
        ops.layernorm_fwd(o, gam, bet, y, mean, rstd)
        tb = T * d * 2
        variants = {
            "layer_scale_residual_fwd": (lambda: ops.layer_scale_residual_fwd(o, x, s, y), 3 * tb),
            "layernorm_residual_fwd": (lambda: ops.layernorm_residual_fwd(o, x, gam, bet, y, mean, rstd),
                                       3 * tb + 8 * T),
            "layernorm_scale_residual_fwd": (lambda: ops.layernorm_scale_residual_fwd(o, x, gam, bet, s, y, mean,
                                                                                      rstd), 3 * tb + 8 * T),
            "layer_scale_bwd": (lambda: ops.layer_scale_bwd(dy, o, s, dv, ds), 3 * tb),
            "layer_scale_bwd_db_dropout": (lambda: ops.layer_scale_bwd(dy, o, s, dv, ds, db=db, dropout=site), 3 * tb),
            "layer_scale_bwd_sandwich": (lambda: ops.layer_scale_bwd(dy, o, s, dv, ds, norm=(gam, bet, mean, rstd)),
                                         3 * tb + 8 * T),
            "layernorm_fwd": (lambda: ops.layernorm_fwd(o, gam, bet, y, mean, rstd), 2 * tb + 8 * T),
            "layernorm_divmax_fwd": (lambda: ops.layernorm_divmax_fwd(o, gam, bet, y, mean, rstd, m), 2 * tb + 12 * T),
            "layernorm_bwd_final": (lambda: ops.layernorm_bwd(dy, o, gam, mean, rstd, None, dv, dg, db, dxsum=dsum,
                                                              dxm=dxm, dropout=site), 4 * tb + 8 * T),
            "layernorm_divmax_bwd_final": (lambda: ops.layernorm_divmax_bwd(dy, o, gam, mean, rstd, m, None, dv, dg, db,
                                                                            dxsum=dsum, dxm=dxm, dropout=site),
                                           4 * tb + 12 * T),
            "embed_bwd": (lambda: ops.embed_bwd(ids, dy.view(-1, 1280, d), dwte, dwpe), tb),
            "embed_bwd_scaled": (lambda: ops.embed_bwd(ids, dy.view(-1, 1280, d), dwte, dwpe, alpha=0.1), tb),
        }
        for fn, _ in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, (fn, _) in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            print(json.dumps({"bench": "layer_scale_launch", "shape": name, "kernel": k, "rows": T, "d": d,
                              "us_per_launch_min": 1e3 * min(v), "TBps": variants[k][1] / min(v) / 1e9,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del o, x, dy, y, dv, dxm, dwte
        torch.cuda.empty_cache()


def step_rows(info):
    B, IL = 32, W * W
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, IL, **kw) for k, kw in STEP_KEYS.items()}
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
        print(json.dumps({"bench": "dalle_example_step", "keys": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v],
                          "over_off_min": min(v) / min(ms["off"]), **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k, kw in (("off", {}), ("both", {"layer_scale": True, "stable": True})):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, **kw)
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
        print(json.dumps({"bench": "generate_graphed", "keys": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
