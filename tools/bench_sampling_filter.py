"""Cost of top-k / nucleus filtering in generation, on one GPU.  Prints JSON lines:

  * per-launch device time of db200_sample_rows against db200_sample_rows_filtered at rows = 32 (one generation
    batch), n in {512, 8192, 32768} ids, (top_k, top_p) in {(64, 1), (0, 0.9), (64, 0.9)}: 1000 launches captured in
    one CUDA graph and timed with CUDA events around its replay, so host launch overhead is not counted; 3 rounds,
    the variants alternated within each round;
  * generate_graphed images/s at the dalle_example_b200 shape (d=512, L=6, H=4, 256 text + 1024 image positions,
    random-init weights, batch 32) with no filter, top_k=64 and top_p=0.9, alternated over 3 rounds (one sampler per
    variant, so every timed call replays already captured graphs).

Every line carries the GPU name and its power limit."""
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

LAUNCHES, ROUNDS = 1000, 3


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock = (q.stdout.strip().split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def time_graph(fn):
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


def kernel_rows(info, rows=32):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for n in (512, 8192, 32768):
        logits = torch.randn(rows, n, device="cuda", generator=gen) * 3
        u = torch.empty(rows, n, device="cuda").uniform_(1e-9, 1.0, generator=gen)
        idx = torch.empty(rows, dtype=torch.int32, device="cuda")
        variants = {("sample_rows", 0, 1.0): lambda: ops.sample_rows(logits, u, idx, 0, n, 1.0)}
        for k, p in ((64, 1.0), (0, 0.9), (64, 0.9)):
            variants[("sample_rows_filtered", k, p)] = \
                lambda k=k, p=p: ops.sample_rows_filtered(logits, u, idx, 0, n, 1.0, k, p)
        graphs = {key: time_graph(fn) for key, fn in variants.items()}
        us = {key: [] for key in variants}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(ROUNDS):
            for key, g in graphs.items():
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                us[key].append(e0.elapsed_time(e1) * 1000.0 / LAUNCHES)
        for (kernel, k, p), t in us.items():
            print(json.dumps({"metric": "us_per_launch", "kernel": kernel, "rows": rows, "n": n, "top_k": k,
                              "top_p": p, "rounds": [round(v, 3) for v in t], "min": round(min(t), 3), **info}))
        del graphs


def generation(info, batch=32):
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (batch, 256), generator=g).to(torch.int32).cuda()
    variants = {"none": {}, "top_k=64": {"top_k": 64}, "top_p=0.9": {"top_p": 0.9}}
    samplers = {name: DalleSampler(eng) for name in variants}
    for name, kw in variants.items():           # capture + warm-up
        samplers[name].generate_graphed(text, temperature=1.0, **kw)
    torch.cuda.synchronize()
    ms = {name: [] for name in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for name, kw in variants.items():
            e0.record()
            out = samplers[name].generate_graphed(text, temperature=1.0, **kw)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1))
            assert out.shape == (batch, eng.S)
    for name, t in ms.items():
        print(json.dumps({"metric": "generated_images_per_sec", "filter": name, "batch": batch,
                          "mode": "cuda-graph replay", "rounds": [round(batch * 1000.0 / v, 3) for v in t],
                          "ms_per_position": [round(v / (eng.S - 1), 4) for v in t], **info}))


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    generation(info)


if __name__ == "__main__":
    main()
