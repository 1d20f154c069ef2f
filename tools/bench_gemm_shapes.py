"""Per-shape device time of every GEMM product of the dalle_example training step, on one GPU.  Prints JSON lines.

The products (shape, operand majors, epilogue and its inputs) are recorded from a one-layer DalleEngine at d = 512
(forward, backward and logits() on one sequence) and replayed on fresh operands with the benchmark's 32 x 1280 =
40 960 token rows: CUDA events around LAUNCHES launches after a warm-up, ROUNDS rounds.

  --lib NAME=PATH (repeatable)  time several builds of the library in one process, alternated inside every round,
                                e.g. the parent commit's build against this tree's
                                (`make -C dalle_mtf_b200/csrc LIB=../libdalle_b200_ab.so BUILD=build_ab` in a checkout
                                of the parent).  Without it the tree's own library is timed alone.
  --sweep                       also the MLP's W1 forward (STORE, bias + ReLU, M x 4K x K) at K = 512, 1024, 2048 and
                                4096 with M K = 40 960 x 512: the contraction lengths around the rule that picks the
                                ping-pong kernel (K <= 1024).  A build with -DDB200_PP_MAX_KB=<k-blocks> moves the rule.
                                And the MLP's W2 forward shape (STORE, bias, M x 512 x 2048) at M = 64 t SMs rows,
                                t = 1 .. 5 tiles of 128 x 256 per SM: the counts around the rule that picks the wide
                                kernel (t >= 2).  A build with -DDB200_WIDE_MIN_TILES=<t> moves the rule.

For every build a line also names the GEMM kernel the product ran on (read from one profiled launch) and the operand
bytes its tile shape moves from L2 into shared memory: every 128 x BN output tile loads (128 + BN) K bf16 values
(BN = 256 on gemm_wide_kernel, 128 otherwise), divided by the kernel time.  Split-K products load the same total.

Every line carries the GPU's name, its power limit and SM clocks, read in the same run.  Fails without a GPU."""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402

T_REC, T = 1280, 40960
MODES = {L.EPI_STORE: "STORE", L.EPI_ATOMIC: "ATOMIC", L.EPI_RELU_BWD: "RELU_BWD", L.EPI_CE_STATS: "CE_STATS",
         L.EPI_CE_GRAD: "CE_GRAD"}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    name, power, clock_max, clock = (q.stdout.strip().split(", ") + ["?"] * 4)[:4] if q.returncode == 0 else \
        (torch.cuda.get_device_name(), "not read", "not read", "not read")
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock_max, "sm_clock_now": clock}


def sm_clock_now():
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader",
                        f"--id={torch.cuda.current_device()}"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       text=True)
    return q.stdout.strip() if q.returncode == 0 else "not read"


def load_libs(specs):
    """name -> loaded library; the tree's own build when no --lib is given."""
    if not specs:
        return {"tree": L.load()}
    libs = {}
    for spec in specs:
        name, path = spec.split("=", 1)
        L._lib, L.LIB_PATH = None, os.path.abspath(path)
        libs[name] = L.load()
        if L.MISSING_SYMBOLS:
            raise SystemExit(f"{path} lacks {L.MISSING_SYMBOLS}")
    return libs


def record_products():
    """Distinct ops.gemm calls of one step of a one-layer d = 512 engine: (M, N, K, keyword summary)."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(512, 1, 4, 50258, 512, 256, 1024)
    eng.init_params(seed=1)
    seen, orig = {}, ops.gemm

    def rec(a, b, out, M, N, K, **kw):
        key = (M, N, K, bool(kw.get("a_mn")), bool(kw.get("b_mn")), int(kw.get("mode", 0)),
               out is not None and out.dtype == torch.float32, kw.get("bias") is not None, bool(kw.get("relu")),
               kw.get("residual") is not None, kw.get("aux") is not None, int(kw.get("split_k", 1)),
               int(kw.get("n_valid", 0)), kw.get("colsum") is not None)
        seen.setdefault(key, None)
        return orig(a, b, out, M, N, K, **kw)

    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, 50258 + 512, (1, T_REC), device="cuda", generator=g, dtype=torch.int32)
    ops.gemm = rec
    try:
        eng.zero_grads()
        eng.forward(tokens, step=None)
        eng.backward(1.0 / T_REC)
        eng.logits(tokens)
        torch.cuda.synchronize()
    finally:
        ops.gemm = orig
    del eng
    torch.cuda.empty_cache()
    return list(seen)


def make_call(key):
    """Fresh operands of one recorded product at T token rows and a closure that launches it; its display name."""
    M, N, K, a_mn, b_mn, mode, f32, has_bias, relu, has_res, has_aux, split_k, n_valid, has_colsum = key
    M, K = (T if M == T_REC else M), (T if K == T_REC else K)
    g = torch.Generator(device="cuda").manual_seed(M + N + K)

    def randn(*shape, scale=1.0, dtype=torch.bfloat16):
        return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)

    a = randn(*((K, M) if a_mn else (M, K)))
    b = randn(*((K, N) if b_mn else (N, K)), scale=K ** -0.5)
    kw = dict(a_mn=a_mn, b_mn=b_mn, mode=mode, relu=relu, split_k=split_k)
    if has_bias:
        kw["bias"] = randn(N, scale=0.1, dtype=torch.float32)
    if has_res:
        kw["residual"] = randn(M, N)
    if has_aux:
        kw["aux"] = randn(M, N)
    if has_colsum:
        kw["colsum"] = torch.zeros(N, device="cuda")
    out = None
    if mode != L.EPI_CE_STATS:
        out = torch.zeros(M, N, dtype=torch.float32 if (f32 or mode == L.EPI_ATOMIC) else torch.bfloat16,
                          device="cuda")
    if mode in (L.EPI_CE_STATS, L.EPI_CE_GRAD):
        kw["labels"] = torch.randint(0, n_valid, (M,), device="cuda", generator=g, dtype=torch.int32)
        kw["n_valid"] = n_valid
    if mode == L.EPI_CE_STATS:
        nt = ops.ce_tiles(N)
        kw.update(part_max=torch.empty(nt, M, device="cuda"), part_sum=torch.empty(nt, M, device="cuda"),
                  label_logit=torch.zeros(M, device="cuda"))
    if mode == L.EPI_CE_GRAD:
        kw.update(lse=torch.full((M,), 11.0, device="cuda"), alpha=1.0 / M)
    name = f"{MODES[mode]} {M}x{N}x{K} aT={int(a_mn)} bT={int(b_mn)}" + "".join(
        f" {f}" for f, on in (("bias", has_bias), ("relu", relu), ("res", has_res), ("colsum", has_colsum),
                              ("f32", f32 and mode == L.EPI_STORE)) if on)
    return name, (M, N, K), lambda: ops.gemm(a, b, out, M, N, K, **kw)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def gemm_kernel(fn):
    """Name of the GEMM kernel one launch of fn runs (its split-K or column-sum reductions aside)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {m.group(0) for e in prof.events() if e.device_type == DeviceType.CUDA
             for m in [re.search(r"gemm_(tc|pp|wide)_kernel", e.name)] if m}
    if len(names) != 1:
        raise SystemExit(f"expected one GEMM kernel per launch, saw {sorted(names) or 'none'}")
    return names.pop()


def l2_operand_bytes(M, N, K, kernel):
    """Bytes the product's 128 x BN tiles load from L2 into shared memory: (128 + BN) K bf16 values per tile."""
    bn = 256 if kernel == "gemm_wide_kernel" else 128
    tiles = -(-M // 128) * -(-N // bn)
    return bn, tiles * (128 + bn) * K * 2


def bench(name, shape, fn, libs, launches, rounds, info, family):
    M, N, K = shape
    kernels = {}
    for k, lib in libs.items():
        L._lib = lib
        timed(fn, 3)
        kernels[k] = gemm_kernel(fn)
    ms = {k: [] for k in libs}
    clocks = []
    for _ in range(rounds):
        for k, lib in libs.items():
            L._lib = lib
            ms[k].append(timed(fn, launches))
        clocks.append(sm_clock_now())
    row = {"bench": family, "product": name, "M": M, "N": N, "K": K, "launches": launches,
           "sm_clock_after_rounds": clocks, **info}
    for k, v in ms.items():
        bn, l2_bytes = l2_operand_bytes(M, N, K, kernels[k])
        row[k] = {"ms_min": round(min(v), 4), "tflops": round(2.0 * M * N * K / min(v) / 1e9, 1),
                  "ms_rounds": [round(x, 4) for x in v], "kernel": kernels[k], "tile": f"128x{bn}",
                  "l2_operand_gb": round(l2_bytes / 1e9, 2), "l2_operand_tbps": round(l2_bytes / min(v) / 1e9, 2)}
    names = list(libs)
    if len(names) > 1:
        base = names[0]
        for k in names[1:]:
            row[f"{base}_over_{k}_min"] = round(min(ms[base]) / min(ms[k]), 3)
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    args = ap.parse_args()
    if args.launches < 50 or args.rounds < 1:
        raise SystemExit("at least 50 launches per round and one round")
    libs = load_libs(args.lib)
    L.require_device()
    info = gpu_info()
    L._lib = next(iter(libs.values()))
    for key in record_products():
        name, shape, fn = make_call(key)
        bench(name, shape, fn, libs, args.launches, args.rounds, info, "dalle_example_product")
        del fn
        torch.cuda.empty_cache()
    if args.sweep:
        for K in (512, 1024, 2048, 4096):
            key = (T * 512 // K, 4 * K, K, False, True, L.EPI_STORE, False, True, True, False, False, 1, 0, False)
            name, shape, fn = make_call(key)
            bench(name, shape, fn, libs, args.launches, args.rounds, info, "w1_forward_by_K")
            del fn
            torch.cuda.empty_cache()
        sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        for t in (1, 2, 3, 4, 5):
            key = (64 * t * sms, 512, 2048, False, True, L.EPI_STORE, False, True, False, False, False, 1, 0, False)
            name, shape, fn = make_call(key)
            bench(name, shape, fn, libs, args.launches, args.rounds, info, "w2_forward_by_wide_tiles_per_sm")
            del fn
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
