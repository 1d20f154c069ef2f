"""Cost of the discrete VAE's logit-Laplace reconstruction loss (reconstruction_loss: "logit_laplace"), on one GPU.
Prints JSON lines:

  * per-launch device time of the fused loss kernel (db200_logit_laplace_fwd_bwd, with its fixed-order finish) against
    the MSE kernel (db200_mse_fwd_bwd) at 16 x 256^2 x 3 subpixels (vae_coco at 16 images per GPU): CUDA events around
    LAUNCHES launches, ROUNDS rounds, the variants alternated; with the bytes each must move and the rate that implies;
  * the decoder's final 1x1 conv at that shape (128 bf16 input channels) with 3 outputs (MSE) against 6 (mu | ln b):
    forward, dgrad and wgrad per launch, alternated the same way;
  * the configs/vae_coco_b200.json training step (256 px, K = 8 192, bf16, 16 images per GPU) through vae_model_fn's
    train_op, without the key and with reconstruction_loss "logit_laplace", alternated over ROUNDS rounds of STEPS steps.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_vae_kl import gpu_info, timed  # noqa: E402
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402

LAUNCHES, ROUNDS, STEPS = 50, 5, 10
B, HW, C, CIN = 16, 256, 3, 128
N_PIX = B * HW * HW


def alternate(variants):
    """{name: launch} -> {name: [ms per launch of each round]}, the variants alternated within every round."""
    for fn in variants.values():
        timed(fn, 3)
    ms = {k: [] for k in variants}
    for _ in range(ROUNDS):
        for k, fn in variants.items():
            ms[k].append(timed(fn, LAUNCHES))
    return ms


def loss_rows(info):
    g = torch.Generator(device="cuda").manual_seed(0)
    n = N_PIX * C
    stats = torch.randn(N_PIX, 2 * C, device="cuda", generator=g)
    x = torch.rand(N_PIX, C, device="cuda", generator=g) * 2 - 1
    dstats, xhat = torch.empty_like(stats), torch.empty_like(x)
    pred, dpred = torch.randn(N_PIX, C, device="cuda", generator=g), torch.empty_like(x)
    acc = torch.zeros(2, device="cuda")
    variants = {   # name -> (launch, bytes moved by the fp32 tensors)
        "mse": (lambda: ops.mse_fwd_bwd(pred, x, dpred, acc[:1], 1.0 / n), 3 * n * 4),
        "logit_laplace": (lambda: ops.logit_laplace(stats, x, dstats, xhat, acc[:1], acc[1:], N_PIX, C, 1.0 / n),
                          6 * n * 4),
    }
    ms = alternate({k: v[0] for k, v in variants.items()})
    for k, v in ms.items():
        nbytes = variants[k][1]
        print(json.dumps({"bench": "vae_recon_loss_launch", "variant": k, "subpixels": n, "ms_per_launch_min": min(v),
                          "ms_per_launch_rounds": [round(t, 4) for t in v], "bytes": nbytes,
                          "GB_per_s_at_min": nbytes / (min(v) * 1e-3) / 1e9, **info}), flush=True)


def conv_rows(info):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(B, HW, HW, CIN, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    dx = torch.empty_like(x)
    variants = {}
    for cout in (C, 2 * C):
        d = ops.conv_desc(B, HW, HW, CIN, cout, 1, 1, 1, act_f32=False)
        w = torch.randn(1, 1, CIN, cout, device="cuda", generator=g) * 0.1
        bias, gw, gb = torch.zeros(cout, device="cuda"), torch.zeros_like(w), torch.zeros(cout, device="cuda")
        y = torch.empty(B, HW, HW, cout, device="cuda", dtype=torch.bfloat16)
        dy = (torch.randn(B, HW, HW, cout, device="cuda", generator=g) * 1e-3).to(torch.bfloat16)
        variants[f"fwd_cout{cout}"] = lambda d=d, w=w, bias=bias, y=y: ops.conv2d_fwd(d, x, w, bias, None, y)
        variants[f"dgrad_cout{cout}"] = lambda d=d, w=w, dy=dy: ops.conv2d_dgrad(d, dy, w, None, None, dx)
        variants[f"wgrad_cout{cout}"] = lambda d=d, dy=dy, gw=gw, gb=gb: ops.conv2d_wgrad(d, x, dy, gw, gb)
    ms = alternate(variants)
    for k, v in ms.items():
        print(json.dumps({"bench": "vae_final_conv_launch", "variant": k, "shape": [B, HW, HW, CIN],
                          "ms_per_launch_min": min(v), "ms_per_launch_rounds": [round(t, 4) for t in v], **info}),
              flush=True)


def step_rows(info):
    from dalle_mtf_b200.dist import DataParallel
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    dp = DataParallel().init()
    specs, batches = {}, None
    for name, extra in (("mse", {}), ("logit_laplace", {"reconstruction_loss": "logit_laplace"})):
        p = fetch_model_params(os.path.join(ROOT, "configs", "vae_coco_b200.json"))
        p.update(extra)
        p["_dp"], p["model_path"], p["train_batch_size"] = dp, None, B
        if batches is None:
            it = iter(vae_input_fn(p))
            batches = [next(it)[0].to("cuda") for _ in range(2)]
            if hasattr(it, "close"):
                it.close()
        specs[name] = vae_model_fn(batches[0], batches[0], TRAIN, p)
    for spec in specs.values():
        for i in range(3):
            spec.train_op(batches[i % 2])
    ms = {k: [] for k in specs}
    for _ in range(ROUNDS):
        for k, spec in specs.items():
            ms[k].append(timed(lambda: spec.train_op(batches[0]), STEPS))
    for k, v in ms.items():
        print(json.dumps({"bench": "vae_coco_step", "variant": k, "images_per_gpu": B, "ms_per_step_min": min(v),
                          "imgs_per_s_at_min": B * 1000.0 / min(v), "ms_per_step_rounds": [round(t, 3) for t in v],
                          **info}), flush=True)
    print(json.dumps({"bench": "vae_coco_step", "logit_laplace_over_mse_min": min(ms["logit_laplace"]) / min(ms["mse"]),
                      **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    loss_rows(info)
    conv_rows(info)
    step_rows(info)


if __name__ == "__main__":
    main()
