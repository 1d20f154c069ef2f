"""Cost of the DALL-E paper's input embedding (row / column image positions, per-position padding), on one GPU.
Prints JSON lines:

  * per-launch device time and achieved GB/s of db200_pos_compose and db200_pos_fold at the dalle_example (d = 512),
    dalle_coco (d = 1024) and 12B (d = 4096) widths, 256 text + 32 x 32 image positions: LAUNCHES launches captured
    in one CUDA graph and timed with CUDA events around its replay (host launch overhead is not counted), ROUNDS
    rounds, the two alternated.  The bytes are what each kernel must move: compose reads wpe, image_row, image_col
    (bf16) and writes the [S, d] bf16 table; fold reads the fp32 [S, d] gradient once and reads and writes the three
    fp32 gradients;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) with both keys (image_position_embedding "row_col",
    per_position_padding) against without, alternated over ROUNDS rounds of STEPS steps;
  * generate_graphed images/s at that shape, 32 captions, temperature 1, both ways, alternated over 3 rounds.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402

LAUNCHES, ROUNDS, STEPS, GEN_ROUNDS = 200, 5, 5, 3
TL, W = 256, 32
SHAPES = {"dalle_example": 512, "dalle_coco": 1024, "12B": 4096}
KEYS = dict(image_position_embedding="row_col", per_position_padding=True)


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


def graph_of(fn):
    """A warmed-up CUDA graph of LAUNCHES calls of fn."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def kernel_rows(info):
    S = TL + W * W
    for shape, d in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(d)
        wpe, row, col = (torch.randn(n, d, generator=g, device="cuda").to(torch.bfloat16) for n in (TL, W, W))
        table = torch.empty(S, d, dtype=torch.bfloat16, device="cuda")
        dpos = torch.randn(S, d, generator=g, device="cuda")
        dw, dr, dc = (torch.zeros(n, d, device="cuda") for n in (TL, W, W))
        variants = {"pos_compose": (lambda: ops.pos_compose(wpe, row, col, table), 2 * (TL + 2 * W + S) * d),
                    "pos_fold": (lambda: ops.pos_fold(dpos, dw, dr, dc), 4 * (S + 2 * (TL + 2 * W)) * d)}
        graphs = {k: graph_of(fn) for k, (fn, _) in variants.items()}
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, g in graphs.items():
                ms[k].append(timed(g.replay, 1) / LAUNCHES)
        for k, v in ms.items():
            nbytes = variants[k][1]
            print(json.dumps({"bench": "kernel", "kernel": k, "shape": shape, "d": d, "S": S, "bytes": nbytes,
                              "us_per_launch_min": round(min(v) * 1000, 3),
                              "us_per_launch_rounds": [round(x * 1000, 3) for x in v],
                              "GB_per_s_at_min": round(nbytes / (min(v) * 1e-3) / 1e9, 1), **info}), flush=True)


def step_rows(info):
    B, IL = 32, W * W
    engines = {"reference_input": DalleEngine(512, 6, 4, 50258, 512, TL, IL),
               "paper_input": DalleEngine(512, 6, 4, 50258, 512, TL, IL, **KEYS)}
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
        print(json.dumps({"bench": "dalle_example_step", "variant": k, "B": B, "ms_per_step_min": round(min(v), 3),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step",
                      "paper_over_reference_min": round(min(ms["paper_input"]) / min(ms["reference_input"]), 4),
                      **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation(info):
    R = 32
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (R, TL), generator=g).to(torch.int32).cuda()
    text[:, 40:] = 50257                                       # padded captions
    samplers = {}
    for k, kw in (("reference_input", {}), ("paper_input", KEYS)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, **kw)
        eng.init_params(0)
        samplers[k] = DalleSampler(eng, padding_id=50257)
    for s in samplers.values():                                # capture + warm-up
        s.generate_graphed(text, temperature=1.0)
    torch.cuda.synchronize()
    ms = {k: [] for k in samplers}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(GEN_ROUNDS):
        for k, s in samplers.items():
            e0.record()
            s.generate_graphed(text, temperature=1.0)
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    for k, t in ms.items():
        print(json.dumps({"bench": "generate_graphed", "variant": k, "images": R,
                          "images_per_sec_rounds": [round(R * 1000.0 / v, 3) for v in t],
                          "images_per_sec_max": round(R * 1000.0 / min(t), 3), **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    step_rows(info)
    generation(info)


if __name__ == "__main__":
    main()
