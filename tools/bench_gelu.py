"""Cost of the GELU MLP (activation_function "gelu") against the ReLU one, on one GPU.  Prints JSON lines:

  * per-launch device time of the MLP's W1 forward, the ReLU STORE epilogue against the GELU store that also writes z,
    and of its dgrad, RELU_BWD against the GELU backward (both with the fused bias-gradient column sums), at
    dalle_example (M = 40 960, 512 -> 2 048), the dalle_coco width (M = 10 240, 1 024 -> 4 096) and the 12B width
    (M = 5 120, 4 096 -> 16 384): CUDA events around LAUNCHES launches, ROUNDS rounds, the variants alternated;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) with each activation, alternated over ROUNDS rounds of STEPS steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) with each activation, alternated.

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
        x = torch.randn(M, d, device="cuda", generator=g).to(torch.bfloat16)
        w1 = (torch.randn(d, N, device="cuda", generator=g) * d ** -0.5).to(torch.bfloat16)
        w2 = (torch.randn(N, d, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        b1 = torch.zeros(N, device="cuda")
        dy = (torch.randn(M, d, device="cuda", generator=g) * 0.01).to(torch.bfloat16)
        h, z, dh = (torch.empty(M, N, dtype=torch.bfloat16, device="cuda") for _ in range(3))
        cs = torch.zeros(N, device="cuda")
        ops.linear_fwd(x, w1, h, bias=b1, gelu=True, z_out=z)
        variants = {
            "fwd_relu_store": lambda: ops.linear_fwd(x, w1, h, bias=b1, relu=True),
            "fwd_gelu_store_z": lambda: ops.linear_fwd(x, w1, h, bias=b1, gelu=True, z_out=z),
            "dgrad_relu_bwd": lambda: ops.linear_dgrad(dy, w2, dh, relu_mask_of=h, colsum=cs),
            "dgrad_gelu_bwd": lambda: ops.linear_dgrad(dy, w2, dh, gelu_grad_of=z, colsum=cs),
        }
        for fn in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, fn in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            print(json.dumps({"bench": "mlp_launch", "shape": name, "variant": k, "M": M, "K": d, "N": N,
                              "ms_per_launch_min": min(v), "tflops": 2.0 * M * N * d / min(v) / 1e9,
                              "ms_per_launch_rounds": [round(x, 4) for x in v], **info}), flush=True)
        print(json.dumps({"bench": "mlp_launch", "shape": name,
                          "fwd_gelu_over_relu_min": min(ms["fwd_gelu_store_z"]) / min(ms["fwd_relu_store"]),
                          "dgrad_gelu_over_relu_min": min(ms["dgrad_gelu_bwd"]) / min(ms["dgrad_relu_bwd"]),
                          **info}), flush=True)
        del x, w1, w2, dy, h, z, dh
        torch.cuda.empty_cache()


def step_rows(info):
    B, TL, IL = 32, 256, 1024
    engines = {a: DalleEngine(512, 6, 4, 50258, 512, TL, IL, activation=a) for a in ("relu", "gelu")}
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
        print(json.dumps({"bench": "dalle_example_step", "activation": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "gelu_over_relu_min": min(ms["gelu"]) / min(ms["relu"]),
                      **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    TL, IL = 256, 1024
    samplers = {}
    for a in ("relu", "gelu"):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, IL, activation=a)
        eng.init_params(seed=0)
        samplers[a] = DalleSampler(eng)
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
        print(json.dumps({"bench": "generate_graphed", "activation": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
