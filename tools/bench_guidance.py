"""Cost of classifier-free guidance in generation, on one GPU.  Prints JSON lines:

  * per-launch device time of db200_sample_rows_guided against db200_sample_rows and db200_sample_rows_filtered at
    32 pairs (the guided kernel reads 2 x 32 logit rows, the others 32), n in {512, 8192, 32768} ids, with no filter,
    top_k=64 and top_p=0.9, guidance_scale=3 on rows whose guided mix is as wide as the plain kernels' rows: 1000
    launches captured in one CUDA graph and timed with CUDA events around its replay, so host launch overhead is not
    counted; 3 rounds, the variants alternated within each round;
  * images/s of generate_graphed and complete (text-only prompt) at the dalle_example_b200 shape (d=512, L=6, H=4,
    256 text + 1024 image positions, random-init weights, temperature 1): R = 32 with guidance_scale=3 against
    unguided R = 32 and R = 64, alternated over 3 rounds (one sampler per variant, so every timed call replays already
    captured graphs).  Guided R = 32 runs 64 rows through the decoder, like unguided R = 64, but returns 32 images.

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

LAUNCHES, ROUNDS, PAIRS, SCALE = 1000, 3, 32, 3.0
FILTERS = {"none": (0, 1.0), "top_k=64": (64, 1.0), "top_p=0.9": (0, 0.9)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock_max, clock = (q.stdout.strip().split(", ") + ["?"] * 4)[:4] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock_max, "sm_clock_now": clock}


def graph_of(fn):
    """A warmed-up CUDA graph of LAUNCHES calls of fn."""
    fn()                                       # eager warm-up: function attributes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def kernel_rows(info):
    gen = torch.Generator(device="cuda").manual_seed(0)
    # the guided mix u + s (c - u) of two independent N(0, sigma^2) rows has standard deviation
    # sigma * sqrt((1 - s)^2 + s^2): the guided kernel's rows are scaled down by that factor so that it filters
    # distributions as wide as the plain kernels' (the cost of top-p depends on how many ids the nucleus keeps)
    widen = ((1.0 - SCALE) ** 2 + SCALE ** 2) ** 0.5
    for n in (512, 8192, 32768):
        cond = torch.randn(PAIRS, n, device="cuda", generator=gen) * 3
        logits = torch.randn(2 * PAIRS, n, device="cuda", generator=gen) * (3 / widen)
        u = torch.empty(PAIRS, n, device="cuda").uniform_(1e-9, 1.0, generator=gen)
        idx = torch.empty(PAIRS, dtype=torch.int32, device="cuda")
        tok = torch.empty(2 * PAIRS, 1, dtype=torch.int32, device="cuda")
        variants = {}
        for name, (k, p) in FILTERS.items():
            if name == "none":
                variants[("sample_rows", name)] = lambda: ops.sample_rows(cond, u, idx, 0, n, 1.0)
            else:
                variants[("sample_rows_filtered", name)] = \
                    lambda k=k, p=p: ops.sample_rows_filtered(cond, u, idx, 0, n, 1.0, k, p)
            variants[("sample_rows_guided", name)] = \
                lambda k=k, p=p: ops.sample_rows_guided(logits, u, tok, 0, n, 1.0, SCALE, k, p)
        graphs = {key: graph_of(fn) for key, fn in variants.items()}
        us = {key: [] for key in variants}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(ROUNDS):
            for key, g in graphs.items():
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                us[key].append(e0.elapsed_time(e1) * 1000.0 / LAUNCHES)
        for (kernel, flt), t in us.items():
            print(json.dumps({"metric": "us_per_launch", "kernel": kernel, "pairs_or_rows": PAIRS, "n": n,
                              "filter": flt, "rounds": [round(v, 3) for v in t], "min": round(min(t), 3), **info}))
        del graphs


def generation(info):
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (2 * PAIRS, 256), generator=g).to(torch.int32).cuda()
    t32, t64 = text[:PAIRS].contiguous(), text
    variants = {
        ("generate_graphed", "unguided", 32): lambda s: s.generate_graphed(t32, temperature=1.0),
        ("generate_graphed", "unguided", 64): lambda s: s.generate_graphed(t64, temperature=1.0),
        ("generate_graphed", f"guidance_scale={SCALE:g}", 32):
            lambda s: s.generate_graphed(t32, temperature=1.0, guidance_scale=SCALE),
        ("complete", "unguided", 32): lambda s: s.complete(t32, temperature=1.0),
        ("complete", "unguided", 64): lambda s: s.complete(t64, temperature=1.0),
        ("complete", f"guidance_scale={SCALE:g}", 32): lambda s: s.complete(t32, temperature=1.0, guidance_scale=SCALE),
    }
    samplers = {key: DalleSampler(eng) for key in variants}
    for key, fn in variants.items():            # capture + warm-up
        fn(samplers[key])
    torch.cuda.synchronize()
    ms = {key: [] for key in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for key, fn in variants.items():
            e0.record()
            out = fn(samplers[key])
            e1.record()
            torch.cuda.synchronize()
            ms[key].append(e0.elapsed_time(e1))
            assert out.shape == (key[2], eng.S)
    info = {**info, **{k + "_after_run": v for k, v in gpu_info().items() if k == "sm_clock_now"}}
    for (path, variant, rows), t in ms.items():
        decoder_rows = 2 * rows if variant != "unguided" else rows
        print(json.dumps({"metric": "generated_images_per_sec", "path": path, "variant": variant, "images": rows,
                          "decoder_rows": decoder_rows, "rounds": [round(rows * 1000.0 / v, 3) for v in t],
                          "ms_per_call": [round(v, 1) for v in t], **info}))


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    generation(info)


if __name__ == "__main__":
    main()
