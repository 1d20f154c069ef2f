"""Cost of the token shift (shift_tokens) on one GPU.  Prints JSON lines:

  * per-launch device time and GB/s of shift_tokens_fwd and shift_tokens_bwd at dalle_example (T = 40 960 rows,
    d = 512), the dalle_coco width (T = 10 240, d = 1 024) and the 12B width (T = 5 120, d = 4 096), and of
    shift_tokens_decode / shift_tokens_decode_dev at 32 rows of each width (cache [32, 1280, d/2]): CUDA events around
    LAUNCHES launches, ROUNDS rounds, the kernels alternated.  Bytes: fwd / bwd read and write rows x d x 2 B; a
    decode step reads d and writes d/2 + d bf16 per row and reads d/2 from the cache;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) without and with the shift, alternated over ROUNDS rounds of STEPS
    steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) without and with the shift, alternated.

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

LAUNCHES, ROUNDS, STEPS, GEN_B, DEC_B = 50, 5, 5, 8, 32
TL, W = 256, 32
S = TL + W * W
SHAPES = {"dalle_example": (40960, 512), "dalle_coco": (10240, 1024), "12B": (5120, 4096)}


def kernel_rows(info):
    for name, (T, d) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        y = torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)
        out = torch.empty_like(y)
        step = torch.randn(DEC_B, d, device="cuda", generator=g).to(torch.bfloat16)
        cache = torch.zeros(DEC_B, S, d // 2, dtype=torch.bfloat16, device="cuda")
        pos_dev = torch.full((1,), S - 1, dtype=torch.int32, device="cuda")
        variants = {
            "shift_tokens_fwd": (lambda: ops.shift_tokens_fwd(y, out, S, TL, W), 2 * T * d * 2),
            "shift_tokens_bwd": (lambda: ops.shift_tokens_bwd(y, out, S, TL, W), 2 * T * d * 2),
            "shift_tokens_decode": (lambda: ops.shift_tokens_decode(step, cache, S - 1, TL, W), DEC_B * 3 * d * 2),
            "shift_tokens_decode_dev": (lambda: ops.shift_tokens_decode_dev(step, cache, pos_dev, TL, W),
                                        DEC_B * 3 * d * 2),
        }
        for fn, _ in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, (fn, _) in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            rows = DEC_B if "decode" in k else T
            print(json.dumps({"bench": "shift_launch", "shape": name, "kernel": k, "rows": rows, "d": d,
                              "us_per_launch_min": 1e3 * min(v), "GBps": variants[k][1] / min(v) / 1e6,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del y, out, step, cache
        torch.cuda.empty_cache()


def step_rows(info):
    B, IL = 32, W * W
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, IL, shift_tokens=on) for k, on in (("off", False),
                                                                                          ("on", True))}
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
        print(json.dumps({"bench": "dalle_example_step", "shift_tokens": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "on_over_off_min": min(ms["on"]) / min(ms["off"]), **info}),
          flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k, on in (("off", False), ("on", True)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, shift_tokens=on)
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
        print(json.dumps({"bench": "generate_graphed", "shift_tokens": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
