"""Cost of DALLE-pytorch's rotary embedding (rotary_emb) on one GPU.  Prints JSON lines:

  * per-launch device time and GB/s of rope_emb_fwd and rope_emb_bwd at dalle_example (T = 40 960 rows, H = 4,
    dh = 128), the dalle_coco width (T = 10 240, H = 16, dh = 64) and the 12B width (T = 5 120, H = 32, dh = 128): CUDA
    events around LAUNCHES launches, ROUNDS rounds, the kernels alternated; and of rope_emb_decode /
    rope_emb_decode_dev at 8 rows of each width, timed as the replay of a CUDA graph of LAUNCHES launches, so that the
    Python wrapper's host time is not in the figure.  Bytes are the rotated q, k and v dims the kernel reads and writes
    (2 x rows x 3H x 2 pairs x 2 B) plus the table rows it reads;
  * embed_bwd at dalle_example (B = 32, d = 512) as a rotary_emb engine runs it (the zero position table's gradient
    into a scratch), per call, and split by kernel with torch.profiler in a run of its own: embed_bwd_wpe_kernel is the
    position-gradient work a no-position instantiation would save, the other kernels the wte gradient;
  * the dalle_example_b200 step (d = 512, L = 6, H = 4, 256 text + 1024 image positions, B = 32: forward, backward and
    the Adam step of the engine on fixed tokens) without and with rotary_emb, alternated over ROUNDS rounds of STEPS
    steps;
  * generate_graphed images/s of a dalle_example model (B = 8, greedy) without and with rotary_emb, alternated.

Every line carries the GPU name, its power limit and SM clocks, read in the same run."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine, rotary_emb_table  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402
from tools.bench_gelu import gpu_info, timed  # noqa: E402

LAUNCHES, ROUNDS, STEPS, GEN_B, TL, W = 50, 5, 5, 8, 256, 32
S = TL + W * W
SHAPES = {"dalle_example": (40960, 4, 128), "dalle_coco": (10240, 16, 64), "12B": (5120, 32, 128)}


def kernel_rows(info):
    for name, (T, H, dh) in SHAPES.items():
        table = rotary_emb_table(TL, W, dh).cuda()
        n = table.shape[2]
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(T, 3 * H * dh, device="cuda", generator=g).to(torch.bfloat16)
        step = torch.randn(GEN_B, 3 * H * dh, device="cuda", generator=g).to(torch.bfloat16)
        pos_dev = torch.full((1,), S - 1, dtype=torch.int32, device="cuda")
        variants = {
            "rope_emb_fwd": (lambda: ops.rope_emb_fwd(qkv, table, S, H, dh), T),
            "rope_emb_bwd": (lambda: ops.rope_emb_bwd(qkv, table, S, H, dh), T),
            "rope_emb_decode": (lambda: ops.rope_emb_decode(step, table, S - 1, H, dh), GEN_B),
            "rope_emb_decode_dev": (lambda: ops.rope_emb_decode_dev(step, table, pos_dev, H, dh), GEN_B),
        }
        for k in ("rope_emb_decode", "rope_emb_decode_dev"):   # LAUNCHES launches in one graph, replayed
            fn = variants[k][0]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                fn()
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(LAUNCHES):
                    fn()
            variants[k] = ((lambda gr: lambda: gr.replay())(graph), GEN_B)
        for fn, _ in variants.values():
            timed(fn, 3)
        ms = {k: [] for k in variants}
        for _ in range(ROUNDS):
            for k, (fn, _) in variants.items():
                t = timed(fn, LAUNCHES if k.endswith(("fwd", "bwd")) else 1)
                ms[k].append(t if k.endswith(("fwd", "bwd")) else t / LAUNCHES)
        for k, v in ms.items():
            rows = variants[k][1]
            nbytes = 2 * rows * 3 * H * 2 * n * 2 + min(rows, S) * 2 * n * 4
            print(json.dumps({"bench": "rope_emb_launch", "shape": name, "kernel": k, "rows": rows, "H": H, "dh": dh,
                              "pairs": n, "us_per_launch_min": 1e3 * min(v), "GBps": nbytes / min(v) / 1e6,
                              "us_per_launch_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
        del qkv, step
        torch.cuda.empty_cache()


def embed_rows(info):
    """embed_bwd as a rotary_emb engine runs it (position gradient into a scratch) at dalle_example."""
    B, d, V = 32, 512, 50258 + 512 + 1
    g = torch.Generator(device="cuda").manual_seed(2)
    ids = torch.randint(0, V, (B, S), device="cuda", generator=g, dtype=torch.int32)
    dx = torch.randn(B, S, d, device="cuda", generator=g).to(torch.bfloat16)
    dwte = torch.zeros(V, d, device="cuda")
    dpos = torch.zeros(S, d, device="cuda")
    fn = lambda: ops.embed_bwd(ids, dx, dwte, dpos)   # noqa: E731
    timed(fn, 3)
    v = [timed(fn, LAUNCHES) for _ in range(ROUNDS)]
    print(json.dumps({"bench": "embed_bwd", "B": B, "S": S, "d": d, "us_per_call_min": 1e3 * min(v),
                      "us_per_call_rounds": [round(1e3 * x, 2) for x in v], **info}), flush=True)
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(LAUNCHES):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():   # the project's kernels (namespace db200), by device time
        if "db200" in e.key and e.self_device_time_total > 0:
            per[e.key] = per.get(e.key, 0.0) + e.self_device_time_total / LAUNCHES
    wpe = sum(t for k, t in per.items() if "embed_bwd_wpe" in k)
    print(json.dumps({"bench": "embed_bwd_kernels", "us_per_call_position_gradient": wpe,
                      "us_per_call_other_kernels": sum(per.values()) - wpe,
                      "kernels_us_per_call": {k[:80]: round(t, 2) for k, t in per.items()}, **info}), flush=True)


def step_rows(info):
    B = 32
    variants = {"off": None, "rotary_emb": True}
    engines = {k: DalleEngine(512, 6, 4, 50258, 512, TL, W * W, rotary_emb=r) for k, r in variants.items()}
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, 50258 + 512, (B, S), device="cuda", generator=g, dtype=torch.int32)
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
        print(json.dumps({"bench": "dalle_example_step", "variant": k, "B": B, "ms_per_step_min": min(v),
                          "ms_per_step_rounds": [round(x, 3) for x in v], **info}), flush=True)
    print(json.dumps({"bench": "dalle_example_step", "rotary_emb_over_off_min": min(ms["rotary_emb"]) / min(ms["off"]),
                      **info}), flush=True)
    del engines
    torch.cuda.empty_cache()


def generation_rows(info):
    samplers = {}
    for k, r in (("off", None), ("rotary_emb", True)):
        eng = DalleEngine(512, 6, 4, 50258, 512, TL, W * W, rotary_emb=r)
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
        print(json.dumps({"bench": "generate_graphed", "variant": k, "B": GEN_B, "images_per_s_max": max(v),
                          "images_per_s_rounds": [round(x, 3) for x in v], **info}), flush=True)


def main():
    L.require_device()
    info = gpu_info()
    kernel_rows(info)
    embed_rows(info)
    step_rows(info)
    generation_rows(info)


if __name__ == "__main__":
    main()
