"""Cost of the DALL-E paper's discrete-VAE network (architecture "dalle_paper") on one GPU.

Prints the card name and power limit, then
  * the per-launch device time of each K11p kernel at the paper geometry with 8 images (256^2, n_hid 256), with the
    bytes it must move and, for the 7x7 conv, its FLOPs;
  * the training step of configs/vae_paper_b200.json's network at 8 images per GPU: ms / step, images / s and the conv
    TFLOP/s over the step (forward + both gradients of every conv and projection, counted from shapes);
  * the encode time of 32 images by the paper encoder against vae_coco_b200's network.
Times are CUDA-event medians after warm-up.  Usage: python tools/bench_vae_paper.py [--images 8] [--steps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def conv_flops(eng, B):
    """2 * MACs of one forward of every conv and projection of a PaperVaeEngine at batch B (backward: 2x that)."""
    f = 2 * B * eng.H * eng.W * 49 * eng.C * eng.base_width
    for pre, n_in, n_out, ks, res, _ in eng.enc + eng.dec:
        h = n_out // 4
        chans = (n_in, h, h, h, n_out)
        f += sum(2 * B * res * res * ks[j] ** 2 * chans[j] * chans[j + 1] for j in range(4))
        if n_in != n_out:
            f += 2 * B * res * res * n_in * n_out
    rows = B * eng.hw * eng.hw
    f += 2 * rows * eng.n_hid * eng.K + 2 * rows * eng.K * eng.n_init
    f += 2 * B * eng.H * eng.W * eng.dec_out_cin * eng.out_C
    return f


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args(argv)
    from dalle_mtf_b200 import ops
    from dalle_mtf_b200.vae_engine import VaeEngine
    from dalle_mtf_b200.vae_paper_engine import PaperVaeEngine
    torch.cuda.set_device(0)
    res = {"card": card()}
    B, S, dev = args.images, 256, "cuda"
    bf = torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)
    img = torch.rand(B, S, S, 3, generator=g, device=dev) * 2 - 1
    # ---- kernels
    k = {}
    w7 = torch.randn(7, 7, 3, 256, device=dev) * 0.05
    b7 = torch.zeros(256, device=dev)
    x0 = torch.empty(B, S, S, 256, dtype=bf, device=dev)
    t = timed(lambda: ops.conv7x7_in_fwd(img, w7, b7, x0))
    fl = 2 * B * S * S * 147 * 256
    k["conv7x7_in_fwd"] = dict(ms=t, GBps=(img.numel() * 4 + x0.numel() * 2) / t / 1e6, TFLOPs=fl / t / 1e9)
    dw = torch.zeros_like(w7)
    db = torch.zeros_like(b7)
    t = timed(lambda: ops.conv7x7_in_wgrad(img, x0, dw, db))
    k["conv7x7_in_wgrad"] = dict(ms=t, GBps=(img.numel() * 4 + x0.numel() * 2) / t / 1e6, TFLOPs=fl / t / 1e9)
    y = torch.empty(B, S // 2, S // 2, 256, dtype=bf, device=dev)
    t = timed(lambda: ops.maxpool2x2_fwd(x0, y))
    k["maxpool2x2_fwd"] = dict(ms=t, GBps=(x0.numel() + y.numel()) * 2 / t / 1e6)
    dx = torch.empty_like(x0)
    t = timed(lambda: ops.maxpool2x2_bwd(x0, y, dx))
    k["maxpool2x2_bwd"] = dict(ms=t, GBps=(2 * x0.numel() + y.numel()) * 2 / t / 1e6)
    lo = torch.empty(B, S // 2, S // 2, 512, dtype=bf, device=dev).normal_()
    up = torch.empty(B, S, S, 512, dtype=bf, device=dev)
    t = timed(lambda: ops.upsample2x_fwd(lo, up))
    k["upsample2x_fwd"] = dict(ms=t, GBps=(lo.numel() + up.numel()) * 2 / t / 1e6)
    t = timed(lambda: ops.upsample2x_bwd(up, lo))
    k["upsample2x_bwd"] = dict(ms=t, GBps=(lo.numel() + up.numel()) * 2 / t / 1e6)
    r = torch.empty_like(x0).normal_()
    out, a = torch.empty_like(x0), torch.empty_like(x0)
    t = timed(lambda: ops.residual_gain(r, 1 / 64, id=x0, y=out, relu_y=a))
    k["residual_gain (id, y, relu_y)"] = dict(ms=t, GBps=4 * x0.numel() * 2 / t / 1e6)
    res["kernels_256px_8img"] = k
    del x0, dx, y, lo, up, r, out, a
    # ---- training step of vae_paper_b200's network
    eng = PaperVaeEngine(8192, S, use_bf16=True, kl=True, reconstruction_loss="logit_laplace")
    eng.init_params(0)
    u = torch.rand(B * eng.hw * eng.hw, 8192, generator=g, device=dev).clamp_(1e-9, 1.0)

    def step():
        eng.zero_grads()
        eng.forward(img, u, 1.0, False, kl_weight=0.034375)
        eng.backward()
        eng.optimizer_step(1e-4, 1)

    t = timed(step, reps=args.steps)
    fl = 3 * conv_flops(eng, B)
    res["vae_paper_step"] = dict(images=B, ms=t, images_per_s=B * 1000 / t, conv_TFLOPs=fl / t / 1e9,
                                 tflop_per_step=fl / 1e12)
    # ---- encode 32 images: paper encoder against vae_coco_b200's
    img32 = torch.rand(32, S, S, 3, generator=g, device=dev) * 2 - 1
    t_paper = timed(lambda: eng.encode_tokens(img32), reps=args.steps)
    del eng
    torch.cuda.empty_cache()
    cfg = json.load(open(os.path.join(ROOT, "configs", "vae_coco_b200.json")))
    coco = VaeEngine(cfg["num_tokens"], S, cfg["convblocks"], use_bf16=True)
    coco.init_params(0)
    t_coco = timed(lambda: coco.encode_tokens(img32), reps=args.steps)
    res["encode_32_images_ms"] = dict(dalle_paper=t_paper, vae_coco_b200=t_coco)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
