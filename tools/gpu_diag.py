"""GPU diagnostics: runs every kernel family against CPU fp32 torch math and prints error statistics WITHOUT
stopping at the first failure (one GPU session should tell as much as possible).  Not part of the test-suite;
tests/ hold the real parity tests.  Usage: python tools/gpu_diag.py [gemm|rowops|optim|attn|all] ...
"""
import os
import sys
import time
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402

DEV = "cuda"
RESULTS = []


def report(name, got, ref, tol):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    diff = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    rel = diff.max().item() / denom
    ok = bool(rel <= tol) and bool(torch.isfinite(got).all())
    RESULTS.append((name, ok, rel))
    print(f"[{'OK ' if ok else 'BAD'}] {name}: max|diff|={diff.max().item():.4e} max|ref|={denom:.4e} rel={rel:.3e} tol={tol}",
          flush=True)
    if not ok and got.dim() == 2:
        bad = diff > tol * denom
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        print(f"      bad elems={int(bad.sum())}/{bad.numel()} bad rows: n={len(rows)} first={rows[:8].tolist()} "
              f"last={rows[-4:].tolist()} | bad cols: n={len(cols)} first={cols[:8].tolist()} last={cols[-4:].tolist()}")
        print("      got[0,:8]=", got[0, :8].tolist())
        print("      ref[0,:8]=", ref[0, :8].tolist())
    return ok


def guarded(fn):
    def w(*a, **k):
        try:
            fn(*a, **k)
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            traceback.print_exc()
            RESULTS.append((fn.__name__ + str(a), False, float("nan")))
            print(f"[EXC] {fn.__name__}{a}: {e}", flush=True)
    return w


def bf(x):
    return x.to(torch.bfloat16)


@guarded
def gemm_case(M, N, K, a_mn, b_mn, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = bf(torch.randn(M, K, generator=g))
    B = bf(torch.randn(K, N, generator=g))
    ref = A.float() @ B.float()
    a_dev = (A.t().contiguous() if a_mn else A).to(DEV)          # [K,M] or [M,K]
    b_dev = (B if b_mn else B.t().contiguous()).to(DEV)          # [K,N] or [N,K]
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(a_dev, b_dev, out, M, N, K, a_mn=a_mn, b_mn=b_mn)
    torch.cuda.synchronize()
    report(f"gemm M={M} N={N} K={K} a_mn={int(a_mn)} b_mn={int(b_mn)}", out, ref, 1e-2)


@guarded
def gemm_epilogues():
    g = torch.Generator().manual_seed(1)
    M, N, K = 384, 512, 256
    A = bf(torch.randn(M, K, generator=g)); W = bf(torch.randn(K, N, generator=g) * 0.1)
    bias = torch.randn(N, generator=g); res = bf(torch.randn(M, N, generator=g))
    a, w = A.to(DEV), W.to(DEV)
    # bias + relu + residual, bf16 out
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.linear_fwd(a, w, out, bias=bias.to(DEV), relu=True, residual=res.to(DEV))
    ref = torch.relu(A.float() @ W.float() + bias) + res.float()
    report("gemm epi bias+relu+residual", out, ref, 1e-2)
    # fp32 out with alpha
    out32 = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, w, out32, M, N, K, a_mn=False, b_mn=True, alpha=0.5, bias=bias.to(DEV))
    report("gemm epi f32 out alpha", out32, 0.5 * (A.float() @ W.float()) + bias, 1e-5)
    # dgrad with relu mask
    DY = bf(torch.randn(M, N, generator=g)); H = bf(torch.randn(M, K, generator=g))
    dx = torch.empty(M, K, dtype=torch.bfloat16, device=DEV)
    ops.linear_dgrad(DY.to(DEV), w, dx, relu_mask_of=H.to(DEV))
    ref = (DY.float() @ W.float().t()) * (H.float() > 0)
    report("gemm epi relu_bwd (dgrad)", dx, ref, 1e-2)
    # wgrad split-K atomic accumulate
    T = 4096
    X = bf(torch.randn(T, K, generator=g)); DY2 = bf(torch.randn(T, N, generator=g))
    dw = torch.ones(K, N, dtype=torch.float32, device=DEV)
    ops.linear_wgrad(X.to(DEV), DY2.to(DEV), dw)
    ref = 1.0 + X.float().t() @ DY2.float()
    report("gemm epi atomic split-K (wgrad)", dw, ref, 1e-4)


@guarded
def gemm_ce():
    g = torch.Generator().manual_seed(2)
    T, d, V = 300, 128, 1000
    Vpad = 1024
    X = bf(torch.randn(T, d, generator=g)); W = torch.zeros(d, Vpad)
    W[:, :V] = torch.randn(d, V, generator=g) * 0.2
    W = bf(W)
    bias = torch.randn(V, generator=g) * 0.1
    labels = torch.randint(0, V, (T,), generator=g, dtype=torch.int32)
    logits = X.float() @ W.float()[:, :V] + bias
    lse_ref = torch.logsumexp(logits, -1)
    loss_ref = lse_ref - logits[torch.arange(T), labels.long()]
    nt = ops.ce_tiles(Vpad)
    pm = torch.empty(nt, T, device=DEV); ps = torch.empty(nt, T, device=DEV)
    ll = torch.zeros(T, device=DEV); lse = torch.empty(T, device=DEV); lr = torch.empty(T, device=DEV)
    lsum = torch.zeros(1, device=DEV)
    x, w, b, lab = X.to(DEV), W.to(DEV), bias.to(DEV), labels.to(DEV)
    ops.gemm(x, w, None, T, Vpad, d, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS, bias=b, labels=lab, part_max=pm,
             part_sum=ps, label_logit=ll, n_valid=V)
    ops.ce_finish(pm, ps, ll, lse, lr, lsum)
    report("ce lse", lse, lse_ref, 1e-4)
    report("ce loss rows", lr, loss_ref, 1e-3)
    report("ce loss sum", lsum, loss_ref.sum().reshape(1), 1e-4)
    dl = torch.full((T, Vpad), 7.0, dtype=torch.bfloat16, device=DEV)
    ops.gemm(x, w, dl, T, Vpad, d, a_mn=False, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / T, bias=b, labels=lab,
             lse=lse, n_valid=V)
    p = torch.softmax(logits, -1)
    p[torch.arange(T), labels.long()] -= 1
    ref = torch.zeros(T, Vpad); ref[:, :V] = p / T
    report("ce grad", dl, ref, 1e-2)


@guarded
def rowops_cases():
    g = torch.Generator().manual_seed(3)
    B, S, d, V = 3, 37, 512, 1001
    ids = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32)
    wte = bf(torch.randn(V, d, generator=g) * 0.02); wpe = bf(torch.randn(S, d, generator=g) * 0.01)
    out = torch.empty(B, S, d, dtype=torch.bfloat16, device=DEV)
    ops.embed_fwd(ids.to(DEV), wte.to(DEV), wpe.to(DEV), out)
    ref = wte.float()[ids.long()] + wpe.float()[None]
    report("embed fwd", out.reshape(B * S, d), ref.reshape(B * S, d), 1e-2)
    dx = bf(torch.randn(B, S, d, generator=g))
    dwte = torch.zeros(V, d, device=DEV); dwpe = torch.zeros(S, d, device=DEV)
    ops.embed_bwd(ids.to(DEV), dx.to(DEV), dwte, dwpe)
    ref_wte = torch.zeros(V, d).index_add_(0, ids.long().flatten(), dx.float().reshape(-1, d))
    report("embed bwd dwte", dwte, ref_wte, 1e-5)
    report("embed bwd dwpe", dwpe, dx.float().sum(0), 1e-5)
    # layernorm
    for dd in (512, 1024):
        rows = 203
        x = bf(torch.randn(rows, dd, generator=g) * 2 + 0.5)
        gg = torch.randn(dd, generator=g); bb = torch.randn(dd, generator=g)
        y = torch.empty(rows, dd, dtype=torch.bfloat16, device=DEV)
        mean = torch.empty(rows, device=DEV); rstd = torch.empty(rows, device=DEV)
        ops.layernorm_fwd(x.to(DEV), gg.to(DEV), bb.to(DEV), y, mean, rstd)
        xf = x.float().requires_grad_(True)
        gp = gg.clone().requires_grad_(True); bp = bb.clone().requires_grad_(True)
        yref = torch.nn.functional.layer_norm(xf, (dd,), gp, bp, 1e-5)
        report(f"layernorm fwd d={dd}", y, yref, 1e-2)
        dy = bf(torch.randn(rows, dd, generator=g)); dres = bf(torch.randn(rows, dd, generator=g))
        yref.backward(dy.float())
        dxo = torch.empty(rows, dd, dtype=torch.bfloat16, device=DEV)
        dg = torch.zeros(dd, device=DEV); db = torch.zeros(dd, device=DEV)
        ops.layernorm_bwd(dy.to(DEV), x.to(DEV), gg.to(DEV), mean, rstd, dres.to(DEV), dxo, dg, db)
        report(f"layernorm bwd dx d={dd}", dxo, xf.grad + dres.float(), 1e-2)
        report(f"layernorm bwd dg d={dd}", dg, gp.grad, 1e-4)
        report(f"layernorm bwd db d={dd}", db, bp.grad, 1e-4)
    # colsum
    x = bf(torch.randn(1000, 520, generator=g))
    o = torch.zeros(520, device=DEV)
    ops.colsum(x.to(DEV), o)
    report("colsum", o, x.float().sum(0), 1e-5)


@guarded
def optim_cases():
    g = torch.Generator().manual_seed(4)
    n = 100003
    p = torch.randn(n, generator=g); m = torch.randn(n, generator=g) * 0.1; v = torch.rand(n, generator=g) * 0.01
    gr = torch.randn(n, generator=g)
    acc = torch.zeros(1, device=DEV)
    ops.sqnorm(gr.to(DEV), acc)
    report("sqnorm", acc, (gr.double() ** 2).sum().float().reshape(1), 1e-5)
    # mtf-style adam with clipping
    pd, md, vd = p.to(DEV), m.to(DEV), v.to(DEV)
    p16 = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ops.adam_step(pd, md, vd, gr.to(DEV), p16, lr=1e-3, eps=1e-6, gnorm_sq=acc, clip=1.0)
    gn = gr.norm()
    gs = gr * (1.0 / max(gn.item(), 1.0))
    m2 = 0.9 * m + 0.1 * gs; v2 = 0.999 * v + 0.001 * gs * gs
    p2 = p - 1e-3 * m2 / (v2.sqrt() + 1e-6)
    report("adam(mtf) p", pd, p2, 1e-6); report("adam(mtf) m", md, m2, 1e-6); report("adam(mtf) v", vd, v2, 1e-6)
    report("adam(mtf) p_bf16", p16, p2, 1e-2)
    # tf-style adam with bias correction
    pd, md, vd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ops.adam_step(pd, md, vd, gr.to(DEV), None, lr=1e-3, eps=1e-8, bias_correction=True, step=1)
    opt_p = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([opt_p], lr=1e-3, eps=1e-8)
    opt_p.grad = gr.clone(); opt.step()
    report("adam(tf) p step1", pd, opt_p.detach(), 1e-5)


@guarded
def gemm_perf():
    for (M, N, K, a_mn, b_mn, mode) in [(40960, 512, 512, 0, 1, "fwd"), (40960, 2048, 512, 0, 1, "fwd"),
                                        (40960, 512, 2048, 0, 1, "fwd"), (40960, 1536, 512, 0, 1, "fwd"),
                                        (8192, 8192, 8192, 0, 0, "nt"), (40960, 512, 2048, 0, 0, "dgrad"),
                                        (512, 2048, 40960, 1, 1, "wgrad")]:
        a = torch.randn((K, M) if a_mn else (M, K), device=DEV).to(torch.bfloat16)
        b = torch.randn((K, N) if b_mn else (N, K), device=DEV).to(torch.bfloat16)
        if mode == "wgrad":
            out = torch.zeros(M, N, dtype=torch.float32, device=DEV)
            run = lambda: ops.gemm(a, b, out, M, N, K, a_mn=True, b_mn=True, mode=L.EPI_ATOMIC, split_k=0)
        else:
            out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
            run = lambda: ops.gemm(a, b, out, M, N, K, a_mn=bool(a_mn), b_mn=bool(b_mn))
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        print(f"[PERF] gemm {mode} M={M} N={N} K={K}: {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s", flush=True)


def main():
    which = sys.argv[1:] or ["all"]
    L.require_device()
    print("device:", torch.cuda.get_device_name(0), "lib version", L.load().db200_version(), flush=True)
    t0 = time.time()
    if "gemm" in which or "all" in which:
        gemm_case(128, 256, 64, False, False)
        gemm_case(128, 256, 64, False, True)
        gemm_case(128, 256, 64, True, False)
        gemm_case(128, 256, 64, True, True)
        for a_mn in (False, True):
            for b_mn in (False, True):
                gemm_case(256, 512, 512, a_mn, b_mn, seed=5)
        gemm_case(200, 264, 200, False, True, seed=6)
        gemm_case(200, 264, 200, True, True, seed=6)
        gemm_case(200, 264, 200, False, False, seed=6)
        gemm_case(1000, 128, 328, False, True, seed=7)     # BN=128 path
        gemm_case(2048, 1536, 512, False, True, seed=8)    # multi-wave persistent
        for a_mn in (False, True):           # large M: more tiles than SMs
            for b_mn in (False, True):
                gemm_case(19976, 520, 264, a_mn, b_mn, seed=9)
        gemm_case(40960, 512, 512, False, True, seed=10)
        gemm_epilogues()
        gemm_ce()
    if "rowops" in which or "all" in which:
        rowops_cases()
    if "optim" in which or "all" in which:
        optim_cases()
    if "attn" in which or "all" in which:
        try:
            from tools import gpu_diag_attn
            gpu_diag_attn.run(report, guarded)
        except ImportError:
            print("attn diag not present yet")
    if "perf" in which or "all" in which:
        gemm_perf()
    nbad = sum(1 for r in RESULTS if not r[1])
    print(f"SUMMARY: {len(RESULTS) - nbad} ok, {nbad} bad, {time.time() - t0:.1f}s")
    for name, ok, rel in RESULTS:
        if not ok:
            print("  BAD:", name, rel)
    return 1 if nbad else 0


if __name__ == "__main__":
    sys.exit(main())
