"""Cost of the modality logits mask (logits_mask), on one GPU.  Prints JSON lines:

  * per-launch device time and TFLOP/s of the four vocabulary products (CE_STATS, CE_GRAD with the fused bias
    gradient, the wout wgrad and the dgrad into the final LayerNorm), plain over [T, Vpad] against the masked text
    block ([B (TL - 1)] rows over round_up(image_offset, 8) columns) and image block ([B (IL + 1)] rows over
    round_up(V - c0, 8) columns from c0 = floor8(image_offset)), at the dalle_example shape (d 512, V 50 771, B 32) and
    at the dalle_coco width (d 1 024, 8 192 image codes, B 16).  FLOPs are 2 M N K of the columns each launch computes.
    CUDA events around LAUNCHES launches, ROUNDS rounds, plain and masked alternated;
  * per-launch device time and GB/s (bytes read + written) of the row partition and the two scatters;
  * the dalle_example_b200 step (B 32: forward, backward and the Adam step on fixed tokens) with and without the key,
    alternated over ROUNDS rounds of STEPS steps.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from tools.bench_loss_weights import gpu_info, timed  # noqa: E402

LAUNCHES, ROUNDS, STEPS = 10, 5, 5
SHAPES = {"dalle_example": dict(d=512, tv=50258, iv=512, TL=256, IL=1024, B=32),
          "dalle_coco_width": dict(d=1024, tv=50258, iv=8192, TL=256, IL=1024, B=16)}


def _products(h, W, bias, labels, M, N, d, n_valid, colsum, dw):
    """The four vocabulary products of one block: name -> (launch, flops)."""
    nt = ops.ce_tiles(N)
    pm, ps = torch.empty(nt, M, device="cuda"), torch.empty(nt, M, device="cuda")
    ll, lse, lr = (torch.empty(M, device="cuda") for _ in range(3))
    stats = lambda: ops.gemm(h, W, None, M, N, d, b_mn=True, mode=L.EPI_CE_STATS, bias=bias,  # noqa: E731
                             labels=labels, part_max=pm, part_sum=ps, label_logit=ll, n_valid=n_valid)
    stats()
    ops.ce_finish(pm, ps, ll, lse, lr, torch.zeros(1, device="cuda"))
    dl = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    dx = torch.empty(M, d, dtype=torch.bfloat16, device="cuda")
    f = 2.0 * M * N * d
    return {
        "ce_stats": (stats, f),
        "ce_grad": (lambda: ops.gemm(h, W, dl, M, N, d, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / M, bias=bias,
                                     labels=labels, lse=lse, n_valid=n_valid, colsum=colsum), f),
        "wgrad": (lambda: ops.linear_wgrad(h, dl, dw), f),
        "dgrad": (lambda: ops.linear_dgrad(dl, W, dx), f),
    }


def product_rows(info, name, d, tv, iv, TL, IL, B):
    S, T = TL + IL, B * (TL + IL)
    io = tv
    V = io + iv + 1
    Vpad = (V + 63) // 64 * 64
    c0 = io // 8 * 8
    nt, ni = B * (TL - 1), B * (S - TL + 1)
    Nt, Ni = (io + 7) // 8 * 8, (V - c0 + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(0)
    hf = torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)
    W = (torch.randn(d, Vpad, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    bias = torch.zeros(Vpad, device="cuda")
    pos = torch.arange(S, device="cuda").repeat(B)
    labels = torch.where(pos < TL - 1, torch.randint(0, io, (T,), device="cuda", generator=g),
                         torch.randint(io, V, (T,), device="cuda", generator=g)).to(torch.int32)
    gw, gb = torch.zeros(d, Vpad, device="cuda"), torch.zeros(Vpad, device="cuda")
    h_t, h_i = torch.empty(nt, d, dtype=torch.bfloat16, device="cuda"), torch.empty(ni, d, dtype=torch.bfloat16,
                                                                                   device="cuda")
    l_t, l_i = torch.empty(nt, dtype=torch.int32, device="cuda"), torch.empty(ni, dtype=torch.int32, device="cuda")
    b_i = torch.empty(Ni, device="cuda")
    part = lambda: ops.logits_mask_partition(hf, labels, bias, h_t, h_i, l_t, l_i, b_i, B, S, TL - 1, c0, io,  # noqa
                                             V)
    part()
    variants = {
        "plain": _products(hf, W, bias, labels, T, Vpad, d, V, gb, gw),
        "text_block": _products(h_t, W[:, :Nt], bias, l_t, nt, Nt, d, io, gb[:Nt], gw[:, :Nt]),
        "image_block": _products(h_i, W[:, c0:c0 + Ni], b_i, l_i, ni, Ni, d, V - c0, gb[c0:c0 + Ni],
                                 gw[:, c0:c0 + Ni]),
    }
    for prods in variants.values():
        for fn, _ in prods.values():
            timed(fn, 2)
    ms = {(v, p): [] for v in variants for p in variants[v]}
    for _ in range(ROUNDS):
        for v, prods in variants.items():
            for p, (fn, _) in prods.items():
                ms[(v, p)].append(timed(fn, LAUNCHES))
    total = {v: 0.0 for v in variants}
    for (v, p), x in ms.items():
        f = variants[v][p][1]
        total[v] += min(x)
        print(json.dumps({"bench": "vocab_product", "shape": name, "variant": v, "product": p, "ms_per_launch_min":
                          round(min(x), 4), "tflops": round(f / min(x) / 1e9, 1), "tflop": round(f / 1e12, 3),
                          "ms_rounds": [round(y, 4) for y in x], **info}), flush=True)
    masked = total["text_block"] + total["image_block"]
    print(json.dumps({"bench": "vocab_product", "shape": name, "plain_ms_four_products": round(total["plain"], 3),
                      "masked_ms_four_products": round(masked, 3),
                      "masked_over_plain": round(masked / total["plain"], 4),
                      **info}), flush=True)
    # partition and scatters: bytes read + written
    dx = torch.empty(T, d, dtype=torch.bfloat16, device="cuda")
    lr, lr_t, lr_i = torch.empty(T, device="cuda"), torch.empty(nt, device="cuda"), torch.empty(ni, device="cuda")
    kernels = {
        "partition": (part, 2 * T * d * 2 + 2 * T * 4 + Ni * 8),
        "scatter_dx": (lambda: ops.logits_mask_scatter(B, S, TL - 1, dx_text=h_t, dx_image=h_i, dx=dx),
                       2 * T * d * 2),
        "scatter_loss_rows": (lambda: ops.logits_mask_scatter(B, S, TL - 1, loss_text=lr_t, loss_image=lr_i,
                                                              loss_rows=lr), 2 * T * 4),
    }
    for k, (fn, nbytes) in kernels.items():
        timed(fn, 3)
        x = [timed(fn, 50) for _ in range(ROUNDS)]
        print(json.dumps({"bench": "row_kernel", "shape": name, "kernel": k, "d": d, "rows": T,
                          "us_per_launch_min": round(min(x) * 1e3, 2), "gb_per_s": round(nbytes / min(x) / 1e6, 1),
                          **info}), flush=True)


def step_rows(info):
    B, TL, IL = 32, 256, 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.cat([torch.randint(0, 50258, (B, TL), device="cuda", generator=g, dtype=torch.int32),
                        torch.randint(50258, 50258 + 512, (B, IL), device="cuda", generator=g, dtype=torch.int32)], 1)
    T = tokens.numel()
    engines = {"plain": DalleEngine(512, 6, 4, 50258, 512, TL, IL),
               "logits_mask": DalleEngine(512, 6, 4, 50258, 512, TL, IL, logits_mask=True)}

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
        print(json.dumps({"bench": "dalle_example_step", "variant": k, "B": B, "ms_per_step_min": round(min(v), 3),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step",
                      "masked_over_plain_min": round(min(ms["logits_mask"]) / min(ms["plain"]), 4), **info}),
          flush=True)


def main():
    L.require_device()
    info = gpu_info()
    for name, shp in SHAPES.items():
        product_rows(info, name, **shp)
        torch.cuda.empty_cache()
    step_rows(info)


if __name__ == "__main__":
    main()
