"""Cost of the discrete VAE's KL term (kl_loss_weight), on one GPU.  Prints JSON lines:

  * per-launch device time, at rows = 16 384 latent rows (vae_coco at 16 images per GPU) and K = 8 192 codes, of the KL
    statistics pass (db200_vae_kl_stats, with its fixed-order finish), of the straight-through backward with the KL
    gradient (db200_gumbel_softmax_bwd_kl) and of the plain backward (db200_gumbel_softmax_bwd): CUDA events around
    LAUNCHES launches, ROUNDS rounds, the variants alternated; with the bytes each must move and the rate that implies;
  * the configs/vae_coco_b200.json training step (256 px, K = 8 192, bf16, 16 images per GPU) through vae_model_fn's
    train_op, without the key and with kl_loss_weight, alternated over ROUNDS rounds of STEPS steps.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402

LAUNCHES, ROUNDS, STEPS = 50, 5, 10
ROWS, K = 16384, 8192


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock_max, clock = (q.stdout.strip().split(", ") + ["?"] * 4)[:4] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock_max, "sm_clock_now": clock}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_rows(info):
    g = torch.Generator(device="cuda").manual_seed(0)
    logits = torch.randn(ROWS, K, device="cuda", generator=g) * 2
    y = torch.softmax(torch.randn(ROWS, K, device="cuda", generator=g), -1)
    dy = torch.randn(ROWS, K, device="cuda", generator=g) * 1e-3
    dl = torch.empty(ROWS, K, device="cuda")
    lse, ent = torch.empty(ROWS, device="cuda"), torch.empty(ROWS, device="cuda")
    hist = torch.zeros(K, dtype=torch.int32, device="cuda")
    acc = torch.zeros(1, device="cuda")
    mat = ROWS * K * 4
    variants = {   # name -> (launch, bytes moved: reads + writes of the [rows, K] fp32 tensors)
        "kl_stats": (lambda: ops.vae_kl_stats(logits, lse, ent, hist, acc, ROWS, K, 1.0 / ROWS), mat),
        "gumbel_bwd_plain": (lambda: ops.gumbel_softmax_bwd(y, dy, dl, ROWS, K, 0.7), 3 * mat),
        "gumbel_bwd_kl": (lambda: ops.gumbel_softmax_bwd_kl(y, dy, logits, lse, ent, dl, ROWS, K, 0.7, 0.1 / ROWS),
                          4 * mat),
    }
    for fn, _ in variants.values():
        timed(fn, 3)
    ms = {k: [] for k in variants}
    for _ in range(ROUNDS):
        for k, (fn, _) in variants.items():
            ms[k].append(timed(fn, LAUNCHES))
    for k, v in ms.items():
        nbytes = variants[k][1]
        print(json.dumps({"bench": "vae_kl_launch", "variant": k, "rows": ROWS, "K": K, "ms_per_launch_min": min(v),
                          "ms_per_launch_rounds": [round(x, 4) for x in v], "bytes": nbytes,
                          "GB_per_s_at_min": nbytes / (min(v) * 1e-3) / 1e9, **info}), flush=True)
    print(json.dumps({"bench": "vae_kl_launch",
                      "kl_added_ms_min": min(ms["kl_stats"]) + min(ms["gumbel_bwd_kl"]) - min(ms["gumbel_bwd_plain"]),
                      **info}), flush=True)


def step_rows(info):
    from dalle_mtf_b200.dist import DataParallel
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    dp = DataParallel().init()
    specs, batches = {}, None
    for name, extra in (("plain", {}), ("kl", {"kl_loss_weight": 1e-3})):
        p = fetch_model_params(os.path.join(ROOT, "configs", "vae_coco_b200.json"))
        p.update(extra)
        p["_dp"], p["model_path"], p["train_batch_size"] = dp, None, 16
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
        print(json.dumps({"bench": "vae_coco_step", "variant": k, "images_per_gpu": 16, "ms_per_step_min": min(v),
                          "imgs_per_s_at_min": 16 * 1000.0 / min(v), "ms_per_step_rounds": [round(x, 3) for x in v],
                          **info}), flush=True)
    print(json.dumps({"bench": "vae_coco_step", "kl_over_plain_min": min(ms["kl"]) / min(ms["plain"]), **info}),
          flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)


if __name__ == "__main__":
    main()
