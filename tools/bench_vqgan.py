"""Cost of the VQGAN tokenizer (architecture "vqgan") on one GPU, at the vqgan_imagenet_f16_16384 geometry
(--geometry f16, the default) or taming's Gumbel vqgan_gumbel_f8 (--geometry gumbel_f8: 8192 codes, a 32 x 32 grid).

Prints, as JSON lines that name the card, its power limit and SM clock:
  * encode (images -> codes) and decode (codes -> images) images/s at B = 16 and 32, this project's kernels alternated
    with the same network in PyTorch bf16 (oracle/vqgan.py's functions on channels_last tensors, cuDNN) over 3 rounds;
  * per-kernel device time of one encode and one decode at B = 16 (CUDA events around each ops call): GroupNorm
    statistics and apply with the bytes they must move (TB/s), the attention (us) and the summed convolution time with
    its TFLOP/s, FLOPs counted from shapes here;
  * gumbel_f8 only: the S = 1024, C = 512 attention kernel alone at B = 16 and 32, with its TFLOP/s (4 S^2 C per
    image: the score and the weighted-sum products);
  * the tokenizer's share of a dalle_coco_b200-width training step (n_embd 1024, 24 layers, 16 heads, 16 images per
    GPU, image_vocab_size the tokenizer's codes) that tokenizes with it (vae_random_init).
Usage: python tools/bench_vqgan.py [--geometry f16|gumbel_f8] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dalle_mtf_b200 import ops                        # noqa: E402
from oracle import vqgan as O                         # noqa: E402
from oracle import vqgan_gumbel as OG                 # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, power, sm, sm_max = [s.strip() for s in out[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def conv_flops(c):
    return 2.0 * c.N * c.Ho * c.Wo * c.Cout * c.Cin * c.KH * c.KW


def per_kernel(eng, img, ids):
    """Device time per kernel class of one encode + one decode (CUDA events around every wrapped ops call)."""
    rec = []
    wrapped = {}
    for name in ("groupnorm_stats", "groupnorm_apply", "attn_noncausal", "attn_noncausal_long", "conv2d_fwd",
                 "conv2d_fwd_tc", "gemm"):
        fn = getattr(ops, name)

        def w(*a, _fn=fn, _name=name, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = _fn(*a, **k)
            e1.record()
            rec.append((_name, e0, e1, a))
            return out
        wrapped[name] = fn
        setattr(ops, name, w)
    try:
        eng.encode_tokens(img)
        eng.decode_tokens(ids)
        torch.cuda.synchronize()
    finally:
        for k, v in wrapped.items():
            setattr(ops, k, v)
    agg = {}
    for name, e0, e1, a in rec:
        ms = e0.elapsed_time(e1)
        if name.startswith("groupnorm"):
            x = a[0]
            key = f"{name} res={x.shape[1]} C={x.shape[-1]}"
            nbytes = x.numel() * 2 * (1 if name == "groupnorm_stats" else 2)
            d = agg.setdefault(key, {"ms": 0.0, "bytes": 0, "n": 0})
            d["bytes"] += nbytes
        elif name.startswith("attn_noncausal"):
            key = f"attn S={a[3]} C={a[4]}"
            d = agg.setdefault(key, {"ms": 0.0, "n": 0})
        elif name.startswith("conv2d"):
            key = "conv (all)"
            d = agg.setdefault(key, {"ms": 0.0, "flops": 0.0, "n": 0})
            d["flops"] += conv_flops(a[0])
        else:
            key = "gemm (1x1 convs, code scores)"
            d = agg.setdefault(key, {"ms": 0.0, "flops": 0.0, "n": 0})
            d["flops"] += 2.0 * a[3] * a[4] * a[5]
        d["ms"] += ms
        d["n"] += 1
    for key, d in agg.items():
        if "bytes" in d:
            d["TB/s"] = d["bytes"] / (d["ms"] * 1e-3) / 1e12
        if "flops" in d:
            d["TFLOP/s"] = d["flops"] / (d["ms"] * 1e-3) / 1e12
        if key.startswith("attn"):
            d["us_per_launch"] = 1e3 * d["ms"] / d["n"]
    return agg


def attn_kernel(info, S=1024, C=512, reps=50):
    """The long-sequence attention kernel alone (CUDA events over `reps` launches)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (16, 32):
        qkv = torch.randn(B, S, 3 * C, generator=g, device="cuda").to(torch.bfloat16)
        out = torch.empty(B, S, C, dtype=torch.bfloat16, device="cuda")
        ms = timed(lambda: ops.attn_noncausal_long(qkv, out, B, S, C, C ** -0.5), reps=reps, warm=5)
        print(json.dumps({**info, "what": "attn_noncausal_long kernel", "B": B, "S": S, "C": C,
                          "us": round(1e3 * ms, 1), "TFLOP/s": round(4.0 * B * S * S * C / (ms * 1e-3) / 1e12, 1)}))


GEOMETRIES = {"f16": (O.GEOMETRY_F16, "vae_vqgan_f16_16384_b200"),
              "gumbel_f8": (OG.GEOMETRY_GUMBEL_F8, "vae_vqgan_gumbel_f8_8192_b200")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geometry", choices=sorted(GEOMETRIES), default="f16")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    from dalle_mtf_b200.vqgan_engine import VqganEngine, import_taming_state_dict
    geo, vae_cfg = GEOMETRIES[args.geometry]
    info["geometry"] = args.geometry
    if args.geometry == "gumbel_f8":
        attn_kernel(info)
    Q = OG if OG.is_gumbel(geo) else O          # the oracle of the geometry's quantiser
    sd = Q.random_state_dict(geo, 0)
    eng = VqganEngine(geo["num_tokens"], geo["resolution"], geo["ch"], geo["ch_mult"], geo["num_res_blocks"],
                      geo["attn_resolutions"], geo["z_channels"], geo["embed_dim"],
                      quantizer=geo.get("quantizer", "vq"))
    eng.load_params(import_taming_state_dict(sd, geo))
    sd16 = O.to(sd, torch.bfloat16, "cuda")
    sdq = {k: v.float() for k, v in sd16.items() if k.startswith("quantize.")}   # the code search in f32
    torch.backends.cudnn.benchmark = True
    g = torch.Generator(device="cuda").manual_seed(0)
    n_codes = eng.image_seq_len
    res = {}
    for rnd in range(args.rounds):
        for B in (16, 32):
            img = torch.rand(B, 256, 256, 3, generator=g, device="cuda") * 2 - 1
            ids = torch.randint(0, geo["num_tokens"], (B, n_codes), generator=g, device="cuda", dtype=torch.int32)
            img_cl = img.to(torch.bfloat16)
            if OG.is_gumbel(geo):
                ref_z = lambda: OG.codes(sdq, O.encode_z(sd16, geo, img_cl).float())
            else:
                ref_z = lambda: O.nearest_codes(O.encode_z(sd16, geo, img_cl).float().reshape(-1, geo["embed_dim"]),
                                                sdq["quantize.embedding.weight"])
            with torch.no_grad():
                for name, fn in (("ours encode", lambda: eng.encode_tokens(img)),
                                 ("pytorch encode", ref_z),
                                 ("ours decode", lambda: eng.decode_tokens(ids)),
                                 ("pytorch decode", lambda: Q.decode(sd16, geo, ids.long()))):
                    ms = timed(fn)
                    res.setdefault((name, B), []).append(B / (ms * 1e-3))
    for (name, B), v in res.items():
        print(json.dumps({**info, "what": f"{name} images/s", "B": B, "rounds": [round(x, 1) for x in v],
                          "best": round(max(v), 1)}))
    img = torch.rand(16, 256, 256, 3, generator=g, device="cuda") * 2 - 1
    ids = torch.randint(0, geo["num_tokens"], (16, n_codes), generator=g, device="cuda", dtype=torch.int32)
    per_kernel(eng, img, ids)
    for key, d in per_kernel(eng, img, ids).items():
        print(json.dumps({**info, "what": "per-kernel, one encode + one decode at B=16", "kernel": key,
                          **{k: (round(v, 4) if isinstance(v, float) else v) for k, v in d.items()}}))
    del eng
    torch.cuda.empty_cache()
    share(info, vae_cfg, geo["num_tokens"])


def share(info, vae_cfg, vocab):
    """The tokenizer's share of a dalle_coco_b200-width step that tokenizes with the VQGAN (random weights)."""
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    p = defaultdict(lambda: None, fetch_model_params("dalle_coco_b200"))
    p.update({"vae_model": vae_cfg, "image_vocab_size": vocab, "mesh_shape": "data:1",
              "train_batch_size": 16, "vae_random_init": True, "model_path": None})
    p["vae_params"] = fetch_model_params(vae_cfg)
    g = torch.Generator().manual_seed(0)
    img = torch.rand(16, 256, 256, 3, generator=g) * 2 - 1
    cap = torch.randint(0, 50000, (16, p["text_seq_len"]), generator=g, dtype=torch.int32)
    spec = dalle_model_fn(img, cap, TRAIN, p)
    vae = spec.extra["vae"]
    imgd = img.cuda()
    step = timed(lambda: spec.train_op(img, cap), reps=5, warm=2)
    tok = timed(lambda: vae.encode_tokens(imgd), reps=5, warm=2)
    print(json.dumps({**info, "what": "dalle_coco_b200-width step (B=16 per GPU, 24 layers, d=1024) with the VQGAN",
                      "step_ms": round(step, 2), "tokenize_ms": round(tok, 2), "share": round(tok / step, 4)}))


if __name__ == "__main__":
    main()
