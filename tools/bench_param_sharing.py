"""Cost of parameter sharing (share_input_output_emb, shared_attn_ids, shared_ff_ids) on one GPU.  Prints JSON lines:

  * per-launch device time and TFLOP/s of the five vocabulary products, tied (B = wte [Vpad, d], K-major; wgrad
    dlogits^T hf into G(wte); dgrad dlogits wte) against untied (B = wout [d, Vpad], MN-major): CE_STATS, CE_GRAD,
    the weighted CE_GRAD, the wgrad and the dgrad, at dalle_example (T = 40 960, d = 512), the dalle_coco width
    (T = 10 240, d = 1 024) and the 12B width (T = 5 120, d = 4 096) with V = 50 771, plus the logits mask's text and
    image windows (CE_STATS) at dalle_example; CUDA events around LAUNCHES launches, ROUNDS rounds, tied and untied
    alternated;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step on fixed tokens) with neither key, tied, {"shared_attn_ids": [0], "shared_ff_ids": [0]} and both,
    alternated over ROUNDS rounds of STEPS steps, with each model's parameter count;
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

LAUNCHES, ROUNDS, STEPS, GEN_B = 20, 5, 5, 8
TL, W, TV, IV = 256, 32, 50258, 512
V = TV + IV + 1
VPAD = (V + 63) // 64 * 64
SHAPES = {"dalle_example": (40960, 512), "dalle_coco": (10240, 1024), "12B": (5120, 4096)}
STEP_KEYS = {"off": {}, "tied": {"share_input_output_emb": True},
             "shared": {"shared_attn_ids": [0], "shared_ff_ids": [0]},
             "both": {"share_input_output_emb": True, "shared_attn_ids": [0], "shared_ff_ids": [0]}}


def _products(T, d, g, c0=0, N=VPAD, n_valid=V):
    """{(product, tied): (fn, flops)} of the vocabulary products over columns [c0, c0 + N)."""
    h = (torch.randn(T, d, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    wout = (torch.randn(d, VPAD, device="cuda", generator=g) * d ** -0.5).to(torch.bfloat16)
    wte = wout.t().contiguous()
    labels = torch.randint(0, n_valid, (T,), device="cuda", generator=g, dtype=torch.int32)
    bias = torch.zeros(N, device="cuda")
    nt = ops.ce_tiles(N)
    pm, ps, ll = torch.empty(nt, T, device="cuda"), torch.empty(nt, T, device="cuda"), torch.empty(T, device="cuda")
    lse, rows = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
    acc = torch.zeros(1, device="cuda")
    dl = torch.empty(T, N, device="cuda", dtype=torch.bfloat16)
    dx = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    gw, gt = torch.zeros(d, VPAD, device="cuda"), torch.zeros(VPAD, d, device="cuda")
    cs = torch.zeros(N, device="cuda")
    cew = L.make_ce_weights(1280, TL - 1, 1e-6, 7e-6, 1e-4)
    B = {True: (wte[c0:c0 + N], False), False: (wout[:, c0:c0 + N], True)}
    ops.gemm(h, wout[:, c0:c0 + N], None, T, N, d, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS, bias=bias,
             labels=labels, part_max=pm, part_sum=ps, label_logit=ll, n_valid=n_valid)
    ops.ce_finish(pm, ps, ll, lse, rows, acc)
    f = 2.0 * T * N * d
    out = {}
    for tied in (False, True):
        b, b_mn = B[tied]
        out[("ce_stats", tied)] = (lambda b=b, b_mn=b_mn: ops.gemm(
            h, b, None, T, N, d, a_mn=False, b_mn=b_mn, mode=L.EPI_CE_STATS, bias=bias, labels=labels, part_max=pm,
            part_sum=ps, label_logit=ll, n_valid=n_valid), f)
        if N != VPAD:
            continue
        out[("ce_grad", tied)] = (lambda b=b, b_mn=b_mn: ops.gemm(
            h, b, dl, T, N, d, a_mn=False, b_mn=b_mn, mode=L.EPI_CE_GRAD, alpha=1e-6, bias=bias, labels=labels,
            lse=lse, n_valid=n_valid, colsum=cs), f)
        out[("ce_grad_weighted", tied)] = (lambda b=b, b_mn=b_mn: ops.gemm(
            h, b, dl, T, N, d, a_mn=False, b_mn=b_mn, mode=L.EPI_CE_GRAD, bias=bias, labels=labels, lse=lse,
            n_valid=n_valid, colsum=cs, ce_weights=cew), f)
        out[("wgrad", tied)] = ((lambda: ops.linear_wgrad(dl, h, gt)) if tied else
                                (lambda: ops.linear_wgrad(h, dl, gw)), f)
        out[("dgrad", tied)] = ((lambda b=b: ops.linear_fwd(dl, b, dx)) if tied else
                                (lambda b=b: ops.linear_dgrad(dl, b, dx)), f)
    return out


def kernel_rows(info):
    cases = [(name, T, d, 0, VPAD, V) for name, (T, d) in SHAPES.items()]
    c0 = TV // 8 * 8   # the logits mask's windows at dalle_example: text [0, TV), image [c0, V)
    cases += [("dalle_example_mask_text", 40960 * 255 // 1280, 512, 0, (TV + 7) // 8 * 8, TV),
              ("dalle_example_mask_image", 40960 * 1025 // 1280, 512, c0, (V - c0 + 7) // 8 * 8, V - c0)]
    for name, T, d, c, N, nv in cases:
        g = torch.Generator(device="cuda").manual_seed(0)
        prods = _products(T, d, g, c, N, nv)
        for fn, _ in prods.values():
            timed(fn, 2)
        ms = {k: [] for k in prods}
        for _ in range(ROUNDS):
            for k, (fn, _) in prods.items():
                ms[k].append(timed(fn, LAUNCHES))
        for (prod, tied), v in ms.items():
            print(json.dumps({"bench": "vocab_launch", "shape": name, "product": prod, "tied": tied, "M": T, "N": N,
                              "d": d, "us_per_launch_min": 1e3 * min(v),
                              "TFLOPs": prods[(prod, tied)][1] / min(v) / 1e9,
                              "tied_over_untied": min(v) / min(ms[(prod, False)]),
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del prods
        torch.cuda.empty_cache()


def step_rows(info):
    B, IL = 32, W * W
    engines = {k: DalleEngine(512, 6, 4, TV, IV, TL, IL, **kw) for k, kw in STEP_KEYS.items()}
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, TV + IV, (B, TL + IL), device="cuda", generator=g, dtype=torch.int32)
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
        print(json.dumps({"bench": "dalle_example_step", "keys": k, "B": B, "n_params": engines[k].n_params(),
                          "ms_per_step_min": min(v), "ms_per_step_rounds": [round(x, 3) for x in v],
                          "over_off_min": min(v) / min(ms["off"]), **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k in ("off", "both"):
        eng = DalleEngine(512, 6, 4, TV, IV, TL, W * W, **STEP_KEYS[k])
        eng.init_params(seed=0)
        samplers[k] = DalleSampler(eng)
    text = torch.randint(0, TV - 1, (GEN_B, TL), dtype=torch.int32, device="cuda")
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
