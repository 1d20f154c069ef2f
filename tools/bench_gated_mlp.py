"""Cost of the gated MLP (gated_mlp, GEGLU / ReGLU) against the ungated GELU MLP, on one GPU.  Prints JSON lines:

  * per-launch device time of the MLP's W1 forward: the GLU store (h [M, 4d] and z [M, 8d]) of each gate against the
    GELU store at N = 4d (h and z [M, 4d]) and against a plain bias STORE at N = 8d (the same product without the
    gate); and of its dgrad: the GLU backward (dz [M, 8d]) of each gate against GELU_BWD (dz [M, 4d]), all with the
    fused bias-gradient column sums.  At dalle_example (M = 40 960, d = 512), the dalle_coco width (M = 10 240,
    d = 1 024) and the 12B width (M = 5 120, d = 4 096): CUDA events around LAUNCHES launches, ROUNDS rounds, the
    variants alternated;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) with GEGLU against the ungated GELU MLP, alternated over ROUNDS
    rounds of STEPS steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) both ways, alternated.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402

LAUNCHES, ROUNDS, STEPS, GEN_B = 20, 5, 5, 8
SHAPES = {"dalle_example": (40960, 512), "dalle_coco": (10240, 1024), "12B": (5120, 4096)}


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
    for name, (M, d) in SHAPES.items():
        N = 4 * d
        g = torch.Generator(device="cuda").manual_seed(0)
        bf = lambda *shape: torch.empty(*shape, dtype=torch.bfloat16, device="cuda")   # noqa: E731
        x = torch.randn(M, d, device="cuda", generator=g).to(torch.bfloat16)
        w1 = (torch.randn(d, 2 * N, device="cuda", generator=g) * d ** -0.5).to(torch.bfloat16)
        w2 = (torch.randn(N, d, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        b1 = torch.zeros(2 * N, device="cuda")
        dy = (torch.randn(M, d, device="cuda", generator=g) * 0.01).to(torch.bfloat16)
        h, z4, dh, h8, z8, dz8 = bf(M, N), bf(M, N), bf(M, N), bf(M, 2 * N), bf(M, 2 * N), bf(M, 2 * N)
        cs = torch.zeros(2 * N, device="cuda")
        w1g = w1[:, :N].contiguous()
        ops.linear_fwd(x, w1g, h, bias=b1[:N], gelu=True, z_out=z4)
        ops.linear_fwd(x, w1, h, bias=b1, glu="gelu", z_out=z8)
        variants = {
            "fwd_gelu_store_z_4d": lambda: ops.linear_fwd(x, w1g, h, bias=b1[:N], gelu=True, z_out=z4),
            "fwd_store_8d": lambda: ops.linear_fwd(x, w1, h8, bias=b1),
            "fwd_reglu_store_z": lambda: ops.linear_fwd(x, w1, h, bias=b1, glu="relu", z_out=z8),
            "fwd_geglu_store_z": lambda: ops.linear_fwd(x, w1, h, bias=b1, glu="gelu", z_out=z8),
            "dgrad_gelu_bwd_4d": lambda: ops.linear_dgrad(dy, w2, dh, gelu_grad_of=z4, colsum=cs[:N]),
            "dgrad_reglu_bwd": lambda: ops.linear_dgrad(dy, w2, dz8, glu_grad_of=z8, glu="relu", colsum=cs),
            "dgrad_geglu_bwd": lambda: ops.linear_dgrad(dy, w2, dz8, glu_grad_of=z8, glu="gelu", colsum=cs),
        }
        wide = ("fwd_store_8d", "fwd_reglu_store_z", "fwd_geglu_store_z")    # the products with 8d columns
        flops = {k: 2.0 * M * (2 * N if k in wide else N) * d for k in variants}
        for fn in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, fn in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            print(json.dumps({"bench": "mlp_launch", "shape": name, "variant": k, "M": M, "d": d,
                              "ms_per_launch_min": min(v), "tflops": flops[k] / min(v) / 1e9,
                              "ms_per_launch_rounds": [round(x, 4) for x in v], **info}), flush=True)
        best = {k: min(v) for k, v in ms.items()}
        print(json.dumps({"bench": "mlp_launch", "shape": name,
                          "fwd_geglu_over_gelu_4d": best["fwd_geglu_store_z"] / best["fwd_gelu_store_z_4d"],
                          "fwd_geglu_over_store_8d": best["fwd_geglu_store_z"] / best["fwd_store_8d"],
                          "fwd_reglu_over_store_8d": best["fwd_reglu_store_z"] / best["fwd_store_8d"],
                          "dgrad_geglu_over_gelu_bwd": best["dgrad_geglu_bwd"] / best["dgrad_gelu_bwd_4d"],
                          "dgrad_reglu_over_gelu_bwd": best["dgrad_reglu_bwd"] / best["dgrad_gelu_bwd_4d"],
                          **info}), flush=True)
        del x, w1, w1g, w2, dy, h, z4, dh, h8, z8, dz8
        torch.cuda.empty_cache()


MODELS = {"gelu": dict(activation="gelu"), "geglu": dict(activation="gelu", gated_mlp=True)}


def step_rows(info):
    B, TL, IL = 32, 256, 1024
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, IL, **kw) for k, kw in MODELS.items()}
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
        print(json.dumps({"bench": "dalle_example_step", "mlp": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "geglu_over_gelu_min": min(ms["geglu"]) / min(ms["gelu"]),
                      **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    TL, IL = 256, 1024
    samplers = {}
    for k, kw in MODELS.items():
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, IL, **kw)
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
        print(json.dumps({"bench": "generate_graphed", "mlp": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
