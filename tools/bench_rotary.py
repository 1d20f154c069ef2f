"""Cost of rotary position embeddings (rotary_dim) on one GPU.  Prints JSON lines:

  * per-launch device time and GB/s of rope_fwd and rope_bwd at dalle_example (T = 40 960 rows, H = 4, dh = 128),
    the dalle_coco width (T = 10 240, H = 16, dh = 64) and the 12B width (T = 5 120, H = 32, dh = 128), each with
    r = head_dim, and of rope_decode / rope_decode_dev at 8 rows of each width: CUDA events around LAUNCHES launches,
    ROUNDS rounds, the kernels alternated.  Bytes are the q and k dims the kernel reads and writes (2 x rows x 2H x r x
    2 B) plus the table rows it reads;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) without rotary and with rotary_dim 128 and 32, alternated over ROUNDS
    rounds of STEPS steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) without and with rotary_dim 128, alternated.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine, rope_table  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402
from tools.bench_gelu import gpu_info, timed  # noqa: E402

LAUNCHES, ROUNDS, STEPS, GEN_B, S = 50, 5, 5, 8, 1280
SHAPES = {"dalle_example": (40960, 4, 128), "dalle_coco": (10240, 16, 64), "12B": (5120, 32, 128)}


def kernel_rows(info):
    for name, (T, H, dh) in SHAPES.items():
        r = dh
        table = rope_table(S, r, 10000.0).cuda()
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(T, 3 * H * dh, device="cuda", generator=g).to(torch.bfloat16)
        step = torch.randn(GEN_B, 3 * H * dh, device="cuda", generator=g).to(torch.bfloat16)
        pos_dev = torch.full((1,), S - 1, dtype=torch.int32, device="cuda")
        variants = {
            "rope_fwd": (lambda: ops.rope_fwd(qkv, table, S, H, dh, r), T),
            "rope_bwd": (lambda: ops.rope_bwd(qkv, table, S, H, dh, r), T),
            "rope_decode": (lambda: ops.rope_decode(step, table, S - 1, H, dh, r), GEN_B),
            "rope_decode_dev": (lambda: ops.rope_decode_dev(step, table, pos_dev, H, dh, r), GEN_B),
        }
        for fn, _ in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, (fn, _) in variants.items():
                ms[k].append(timed(fn, LAUNCHES))
        for k, v in ms.items():
            rows = variants[k][1]
            nbytes = 2 * rows * 2 * H * r * 2 + min(rows, S) * r * 4
            print(json.dumps({"bench": "rope_launch", "shape": name, "kernel": k, "rows": rows, "H": H, "dh": dh,
                              "r": r, "us_per_launch_min": 1e3 * min(v), "GBps": nbytes / min(v) / 1e6,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del qkv, step
        torch.cuda.empty_cache()


def step_rows(info):
    B, TL, IL = 32, 256, 1024
    variants = {"off": None, "r128": 128, "r32": 32}
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, IL, rotary_dim=r) for k, r in variants.items()}
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
        print(json.dumps({"bench": "dalle_example_step", "rotary": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "r128_over_off_min": min(ms["r128"]) / min(ms["off"]),
                      "r32_over_off_min": min(ms["r32"]) / min(ms["off"]), **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    TL, IL = 256, 1024
    samplers = {}
    for k, r in (("off", None), ("r128", 128)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, IL, rotary_dim=r)
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
        print(json.dumps({"bench": "generate_graphed", "rotary": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
