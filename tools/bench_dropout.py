"""Cost of dropout in the DALL-E training step on one GPU: bench.py's headline workload (dalle_example_b200) against
the same workload with embed_dropout = attention_dropout = residual_dropout = 0.1
(configs/dalle_example_dropout_b200.json), measured the way bench.py measures `value` and alternated `--rounds` times
in one process so that both see the same card and clocks.  Prints one JSON line.

    python tools/bench_dropout.py --steps 10 --warmup 3 --rounds 2
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

# the headline workload's shape with the dropout config file
bench.WORKLOADS.setdefault("dalle_example_dropout",
                           ("dalle_example_dropout_b200.json",) + bench.WORKLOADS["dalle_example"][1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    L.require_device()
    device = torch.device("cuda", torch.cuda.current_device())
    args = argparse.Namespace(gpus=1, scaling="weak", dump_outputs=None, no_cpu_baseline=True)
    runs = {"dalle_example": [], "dalle_example_dropout": []}
    for _ in range(a.rounds):
        for w in runs:
            line = bench.measure_dalle(args, dp, device, w, a.steps, max(a.warmup, 3), full=False)
            runs[w].append({k: line[k] for k in ("value", "ms_per_step", "loss", "clocks")})
    name = torch.cuda.get_device_name()
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception:  # noqa: BLE001 — the measurement stands without the power limit; it is reported as unknown
        power = None
    base = [r["ms_per_step"] for r in runs["dalle_example"]]
    drop = [r["ms_per_step"] for r in runs["dalle_example_dropout"]]
    print(json.dumps({"metric": "tokens_per_sec", "unit": "tokens/s", "gpu": name, "power_limit": power,
                      "steps": a.steps, "runs": runs,
                      "dropout_step_time_ratio": (sum(drop) / len(drop)) / (sum(base) / len(base))}), flush=True)
    dp.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
