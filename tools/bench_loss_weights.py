"""Cost of the weighted cross-entropy (text_loss_weight / image_loss_weight / z_loss), on one GPU.  Prints JSON lines:

  * per-launch device time of the vocabulary product's CE_GRAD epilogue, plain (alpha = 1 / T) against weighted
    (weights 1 : 7, z_loss 1e-4), at T = 40 960 rows, V = 50 771 (Vpad 50 816), d = 512, with the fused bias-gradient
    column sums as the engine runs it: CUDA events around LAUNCHES launches, ROUNDS rounds, the two alternated;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens), the weighted configuration's loss (1 : 7, z_loss 1e-4) against the
    plain one, alternated over ROUNDS rounds of STEPS steps.  The VAE tokenizer and the caption assembly (with or
    without caption dropout) are the same kernels in both and are not part of it.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine, loss_coefficients  # noqa: E402

LAUNCHES, ROUNDS, STEPS = 20, 5, 5
WEIGHTS, Z = (1.0, 7.0), 1e-4


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
    T, d, V, S, TL = 40960, 512, 50771, 1280, 256
    Vpad = (V + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)
    W = torch.zeros(d, Vpad, device="cuda")
    W[:, :V] = torch.randn(d, V, device="cuda", generator=g) * 0.02
    W = W.to(torch.bfloat16)
    bias = torch.zeros(Vpad, device="cuda")
    labels = torch.randint(0, V, (T,), device="cuda", generator=g, dtype=torch.int32)
    nt = ops.ce_tiles(Vpad)
    pm, ps = torch.empty(nt, T, device="cuda"), torch.empty(nt, T, device="cuda")
    ll, lse, lr = (torch.empty(T, device="cuda") for _ in range(3))
    ops.gemm(h, W, None, T, Vpad, d, b_mn=True, mode=L.EPI_CE_STATS, bias=bias, labels=labels, part_max=pm,
             part_sum=ps, label_logit=ll, n_valid=V)
    ops.ce_finish(pm, ps, ll, lse, lr, torch.zeros(1, device="cuda"))
    dl = torch.empty(T, Vpad, dtype=torch.bfloat16, device="cuda")
    cs = torch.zeros(Vpad, device="cuda")
    cew = L.make_ce_weights(S, TL - 1, *loss_coefficients(WEIGHTS, TL, S - TL, T // S), Z)
    variants = {
        "plain": lambda: ops.gemm(h, W, dl, T, Vpad, d, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / T, bias=bias,
                                  labels=labels, lse=lse, n_valid=V, colsum=cs),
        "weighted": lambda: ops.gemm(h, W, dl, T, Vpad, d, b_mn=True, mode=L.EPI_CE_GRAD, bias=bias, labels=labels,
                                     lse=lse, n_valid=V, colsum=cs, ce_weights=cew),
    }
    for fn in variants.values():
        timed(fn, 3)
    ms = {k: [] for k in variants}
    for _ in range(ROUNDS):
        for k, fn in variants.items():
            ms[k].append(timed(fn, LAUNCHES))
    for k, v in ms.items():
        print(json.dumps({"bench": "ce_grad_launch", "variant": k, "T": T, "V": V, "d": d, "ms_per_launch_min": min(v),
                          "ms_per_launch_rounds": [round(x, 4) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "ce_grad_launch", "weighted_over_plain_min": min(ms["weighted"]) / min(ms["plain"]),
                      **info}), flush=True)


def step_rows(info):
    B, TL, IL = 32, 256, 1024
    engines = {"plain": DalleEngine(512, 6, 4, 50258, 512, TL, IL),
               "weighted": DalleEngine(512, 6, 4, 50258, 512, TL, IL, loss_weights=WEIGHTS, z_loss=Z)}
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, 50258 + 512, (B, TL + IL), device="cuda", generator=g, dtype=torch.int32)
    T = tokens.numel()

    def step(eng):
        eng.zero_grads()
        eng.forward(tokens, step=None)
        eng.backward(1.0 if eng.weighted_loss else 1.0 / T)
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
        print(json.dumps({"bench": "dalle_example_step", "variant": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "weighted_over_plain_min": min(ms["weighted"]) / min(ms["plain"]),
                      **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)


if __name__ == "__main__":
    main()
