"""Generation throughput of the K/V-cache decoder (N4) on one GPU: dalle_example_b200 shape (d=512, L=6, H=4,
256 text + 1024 image positions), random-init weights, batch 32.  Prints one JSON line."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402


def main(batch=32):
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    smp = DalleSampler(eng)
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 50257, (batch, 256), generator=g).to(torch.int32).cuda()
    smp.generate(text[:, :], temperature=1.0)                      # warm-up (allocations, first launches)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = smp.generate(text, temperature=1.0)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    # CUDA-graph replay of the per-position step (device-side position)
    smp.generate_graphed(text, temperature=1.0)                    # capture + warm-up
    torch.cuda.synchronize()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e2.record()
    out_g = smp.generate_graphed(text, temperature=1.0)
    e3.record()
    torch.cuda.synchronize()
    ms_g = e2.elapsed_time(e3)
    assert out_g.shape == (batch, eng.S)
    print(json.dumps({"metric": "generated_images_per_sec", "value": batch * 1000.0 / ms_g, "batch": batch,
                      "mode": "cuda-graph replay", "positions": eng.S - 1, "ms_total": ms_g,
                      "ms_per_position": ms_g / (eng.S - 1), "image_tokens_per_sec": batch * 1024 * 1000.0 / ms_g}))
    print(json.dumps({"metric": "generated_images_per_sec", "value": batch * 1000.0 / ms, "batch": batch, "mode": "eager",
                      "positions": eng.S - 1, "ms_total": ms, "ms_per_position": ms / (eng.S - 1),
                      "image_tokens_per_sec": batch * 1024 * 1000.0 / ms,
                      "gpu_launches": int(L.launch_count() - n0),
                      "note": "prompt positions are teacher-forced through the same per-position step"}))
    assert out.shape == (batch, eng.S)


if __name__ == "__main__":
    main()
