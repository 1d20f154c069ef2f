"""GPU parity tests of every kernel family, through the C ABI (ctypes), against CPU fp32 math / the oracle.

Tolerances (stated per test): integer / index outputs bit-exact; fp32 kernels 1e-5 relative; bf16-activation kernels
are compared with fp32 math on the SAME bf16-rounded inputs, so the only error is the output rounding
(2^-8 = 3.9e-3 relative) plus accumulation order -> max-norm-relative 1e-2.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def relmax(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-30)).item()


def bf(x):
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 512), (200, 264, 200), (1000, 128, 328), (2048, 1536, 512),
                                   (1, 8, 8), (129, 8, 72),
                                   (2504, 2056, 200)])  # ragged in M and N, more tiles than SMs
@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
def test_gemm_all_operand_layouts(ops, M, N, K, a_mn, b_mn):
    g = torch.Generator().manual_seed(M + N + K)
    A, B = bf(torch.randn(M, K, generator=g)), bf(torch.randn(K, N, generator=g))
    ref = A.float() @ B.float()

    def pitched(x):  # rows padded to a 16-byte pitch (what TMA needs): the GEMM reads the view through its row stride
        rows, cols = x.shape
        buf = torch.zeros(rows, (cols + 7) // 8 * 8, dtype=x.dtype)
        buf[:, :cols] = x
        return buf.to(DEV)[:, :cols]

    a = pitched(A.t()) if a_mn else A.to(DEV)
    b = pitched(B) if b_mn else B.t().contiguous().to(DEV)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn)
    assert relmax(out, ref) < 1e-2


def test_gemm_epilogues(ops):
    from dalle_mtf_b200 import lib as L
    g = torch.Generator().manual_seed(1)
    M, N, K = 384, 512, 256
    A, W = bf(torch.randn(M, K, generator=g)), bf(torch.randn(K, N, generator=g) * 0.1)
    bias, res = torch.randn(N, generator=g), bf(torch.randn(M, N, generator=g))
    a, w = A.to(DEV), W.to(DEV)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.linear_fwd(a, w, out, bias=bias.to(DEV), relu=True, residual=res.to(DEV))
    assert relmax(out, torch.relu(A.float() @ W.float() + bias) + res.float()) < 1e-2
    out32 = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, w, out32, M, N, K, a_mn=False, b_mn=True, alpha=0.5, bias=bias.to(DEV))
    assert relmax(out32, 0.5 * (A.float() @ W.float()) + bias) < 1e-5       # fp32 output: accumulate-order only
    DY, H = bf(torch.randn(M, N, generator=g)), bf(torch.randn(M, K, generator=g))
    dx = torch.empty(M, K, dtype=torch.bfloat16, device=DEV)
    ops.linear_dgrad(DY.to(DEV), w, dx, relu_mask_of=H.to(DEV))
    assert relmax(dx, (DY.float() @ W.float().t()) * (H.float() > 0)) < 1e-2
    cs = torch.zeros(K, device=DEV)
    dx2 = torch.empty_like(dx)
    ops.linear_dgrad(DY.to(DEV), w, dx2, relu_mask_of=H.to(DEV), colsum=cs)     # fused bias gradient
    assert torch.equal(dx2, dx) and relmax(cs, dx.float().sum(0)) < 1e-5
    T = 4096
    X, DY2 = bf(torch.randn(T, K, generator=g)), bf(torch.randn(T, N, generator=g))
    dw = torch.ones(K, N, dtype=torch.float32, device=DEV)
    ops.linear_wgrad(X.to(DEV), DY2.to(DEV), dw)                               # split-K + vector red.add, accumulates
    assert relmax(dw, 1.0 + X.float().t() @ DY2.float()) < 1e-4
    assert L.EPI_ATOMIC == 1


def test_gemm_epilogues_on_a_large_ragged_shape(ops):
    """Same epilogues on a ragged shape with more tiles than SMs (persistent CTAs take several tiles), including rows /
    columns that end inside a tile."""
    from dalle_mtf_b200 import lib as L
    g = torch.Generator().manual_seed(11)
    M, N, K = 2600, 2056, 136                      # 21 x 17 tiles of 128 x 128; the last rows end mid-tile
    A, W = bf(torch.randn(M, K, generator=g)), bf(torch.randn(K, N, generator=g) * 0.1)
    bias, res = torch.randn(N, generator=g), bf(torch.randn(M, N, generator=g))
    a, w = A.to(DEV), W.to(DEV)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.linear_fwd(a, w, out, bias=bias.to(DEV), relu=True, residual=res.to(DEV))
    assert relmax(out, torch.relu(A.float() @ W.float() + bias) + res.float()) < 1e-2
    out32 = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, w, out32, M, N, K, a_mn=False, b_mn=True, alpha=0.5, bias=bias.to(DEV))
    assert relmax(out32, 0.5 * (A.float() @ W.float()) + bias) < 1e-5
    # ReLU-masked dgrad with the fused bias gradient: dx[M, N] = (dy[M, K2] @ W2^T) * (h > 0)
    K2 = 264
    DY, W2, H = bf(torch.randn(M, K2, generator=g)), bf(torch.randn(N, K2, generator=g) * 0.1), bf(torch.randn(M, N, generator=g))
    dx = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    cs = torch.zeros(N, device=DEV)
    ops.linear_dgrad(DY.to(DEV), W2.to(DEV), dx, relu_mask_of=H.to(DEV), colsum=cs)
    assert relmax(dx, (DY.float() @ W2.float().t()) * (H.float() > 0)) < 1e-2
    assert relmax(cs, dx.float().sum(0)) < 1e-5
    # cross-entropy statistics and gradient over 21 x 16 tiles
    T, d, V, Vpad = 2600, 128, 2000, 2048
    X = bf(torch.randn(T, d, generator=g))
    Wv = torch.zeros(d, Vpad); Wv[:, :V] = torch.randn(d, V, generator=g) * 0.2; Wv = bf(Wv)
    bv = torch.randn(V, generator=g) * 0.1
    labels = torch.randint(0, V, (T,), generator=g, dtype=torch.int32)
    logits = X.float() @ Wv.float()[:, :V] + bv
    lse_ref = torch.logsumexp(logits, -1)
    nt = ops.ce_tiles(Vpad)
    pm, ps = torch.empty(nt, T, device=DEV), torch.empty(nt, T, device=DEV)
    ll, lse, lr, lsum = torch.zeros(T, device=DEV), torch.empty(T, device=DEV), torch.empty(T, device=DEV), torch.zeros(1, device=DEV)
    x, wv, lab = X.to(DEV), Wv.to(DEV), labels.to(DEV)
    bpad = torch.zeros(Vpad, device=DEV); bpad[:V] = bv.to(DEV)
    ops.gemm(x, wv, None, T, Vpad, d, b_mn=True, mode=L.EPI_CE_STATS, bias=bpad, labels=lab, part_max=pm, part_sum=ps,
             label_logit=ll, n_valid=V)
    ops.ce_finish(pm, ps, ll, lse, lr, lsum)
    assert relmax(lse, lse_ref) < 1e-4
    assert relmax(lr, lse_ref - logits[torch.arange(T), labels.long()]) < 1e-3
    dl = torch.full((T, Vpad), 7.0, dtype=torch.bfloat16, device=DEV)
    cs2 = torch.zeros(Vpad, device=DEV)
    ops.gemm(x, wv, dl, T, Vpad, d, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / T, bias=bpad, labels=lab, lse=lse,
             n_valid=V, colsum=cs2)
    p = torch.softmax(logits, -1); p[torch.arange(T), labels.long()] -= 1
    ref = torch.zeros(T, Vpad); ref[:, :V] = p / T
    assert relmax(dl, ref) < 1e-2 and (dl[:, V:] == 0).all()
    assert relmax(cs2, dl.float().sum(0)) < 1e-4


def test_gemm_is_linear_at_full_size(ops):
    """Size-independent properties at the bench shape (40960 x 2048 x 512):
    (i) D(2A) == 2 D(A) bit-exactly (power-of-two scaling commutes with every rounding);
    (ii) D(A, W) == D(A[:, :256], W[:256]) + D(A[:, 256:], W[256:]) up to fp32 accumulation order."""
    M, N, K = 40960, 2048, 512
    g = torch.Generator(device=DEV).manual_seed(0)
    a = bf(torch.randn(M, K, generator=g, device=DEV))
    w = bf(torch.randn(K, N, generator=g, device=DEV) * 0.05)
    o1, o2, o3, o4 = (torch.empty(M, N, dtype=torch.float32, device=DEV) for _ in range(4))
    ops.gemm(a, w, o1, M, N, K, b_mn=True)
    ops.gemm(bf(a.float() * 2), w, o2, M, N, K, b_mn=True)
    assert torch.equal(o2, o1 * 2)
    ops.gemm(a[:, :256], w[:256], o3, M, N, 256, b_mn=True)
    ops.gemm(a[:, 256:], w[256:], o4, M, N, 256, b_mn=True)
    assert relmax(o3 + o4, o1) < 1e-5


def test_cross_entropy_epilogues(ops):
    from dalle_mtf_b200 import lib as L
    g = torch.Generator().manual_seed(2)
    T, d, V, Vpad = 300, 128, 1000, 1024
    X = bf(torch.randn(T, d, generator=g))
    W = torch.zeros(d, Vpad); W[:, :V] = torch.randn(d, V, generator=g) * 0.2; W = bf(W)
    bias = torch.randn(V, generator=g) * 0.1
    labels = torch.randint(0, V, (T,), generator=g, dtype=torch.int32)
    logits = X.float() @ W.float()[:, :V] + bias
    lse_ref = torch.logsumexp(logits, -1)
    loss_ref = lse_ref - logits[torch.arange(T), labels.long()]
    nt = ops.ce_tiles(Vpad)
    pm, ps = torch.empty(nt, T, device=DEV), torch.empty(nt, T, device=DEV)
    ll, lse, lr, lsum = torch.zeros(T, device=DEV), torch.empty(T, device=DEV), torch.empty(T, device=DEV), torch.zeros(1, device=DEV)
    x, w, lab = X.to(DEV), W.to(DEV), labels.to(DEV)
    bpad = torch.zeros(Vpad, device=DEV); bpad[:V] = bias.to(DEV)
    ops.gemm(x, w, None, T, Vpad, d, b_mn=True, mode=L.EPI_CE_STATS, bias=bpad, labels=lab, part_max=pm, part_sum=ps,
             label_logit=ll, n_valid=V)
    ops.ce_finish(pm, ps, ll, lse, lr, lsum)
    assert relmax(lse, lse_ref) < 1e-4 and relmax(lr, loss_ref) < 1e-3        # ex2.approx: ~2 ulp per exp
    assert relmax(lsum, loss_ref.sum().reshape(1)) < 1e-4
    dl = torch.full((T, Vpad), 7.0, dtype=torch.bfloat16, device=DEV)
    ops.gemm(x, w, dl, T, Vpad, d, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / T, bias=bpad, labels=lab, lse=lse, n_valid=V)
    p = torch.softmax(logits, -1); p[torch.arange(T), labels.long()] -= 1
    ref = torch.zeros(T, Vpad); ref[:, :V] = p / T
    assert relmax(dl, ref) < 1e-2
    assert (dl[:, V:] == 0).all()                                              # padded vocabulary columns stay exactly zero
    # fused bias gradient: column sums of the bf16 values actually written
    cs = torch.zeros(Vpad, device=DEV)
    dl2 = torch.empty_like(dl)
    ops.gemm(x, w, dl2, T, Vpad, d, b_mn=True, mode=L.EPI_CE_GRAD, alpha=1.0 / T, bias=bpad, labels=lab, lse=lse, n_valid=V,
             colsum=cs)
    assert torch.equal(dl2, dl) and relmax(cs, dl.float().sum(0)) < 1e-5


def test_c_abi_reports_errors_instead_of_crashing(ops):
    from dalle_mtf_b200 import lib as L
    a = torch.zeros(16, 12, dtype=torch.bfloat16, device=DEV)                  # row pitch 24 B: not TMA-legal
    with pytest.raises(L.DB200Error, match="multiples of 8"):
        ops.gemm(a, a, torch.zeros(16, 16, dtype=torch.bfloat16, device=DEV), 16, 16, 12)
    with pytest.raises(L.DB200Error, match="head_dim"):
        ops.attn_fwd(torch.zeros(1, 8, 3, 1, 32, dtype=torch.bfloat16, device=DEV),
                     torch.zeros(1, 8, 1, 32, dtype=torch.bfloat16, device=DEV), torch.zeros(1, 1, 8, device=DEV), 1, 8, 1, 32)
    with pytest.raises(L.DB200Error):
        ops.layernorm_fwd(torch.zeros(4, 100, dtype=torch.bfloat16, device=DEV), torch.zeros(100, device=DEV),
                          torch.zeros(100, device=DEV), torch.zeros(4, 100, dtype=torch.bfloat16, device=DEV),
                          torch.zeros(4, device=DEV), torch.zeros(4, device=DEV))
    with pytest.raises(L.DB200Error, match="expected dtype"):
        ops.sqnorm(torch.zeros(8, dtype=torch.bfloat16, device=DEV), torch.zeros(1, device=DEV))


# ------------------------------------------------------------------------------------------------------- row ops
def test_embedding_fwd_bwd_and_label_shift(ops):
    g = torch.Generator().manual_seed(3)
    B, S, d, V = 3, 37, 512, 1001
    ids = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32)
    wte, wpe = bf(torch.randn(V, d, generator=g) * 0.02), bf(torch.randn(S, d, generator=g) * 0.01)
    out = torch.empty(B, S, d, dtype=torch.bfloat16, device=DEV)
    ops.embed_fwd(ids.to(DEV), wte.to(DEV), wpe.to(DEV), out)
    assert relmax(out, wte.float()[ids.long()] + wpe.float()[None]) < 1e-2
    dx = bf(torch.randn(B, S, d, generator=g))
    dwte, dwpe = torch.zeros(V, d, device=DEV), torch.zeros(S, d, device=DEV)
    ops.embed_bwd(ids.to(DEV), dx.to(DEV), dwte, dwpe)
    ref = torch.zeros(V, d).index_add_(0, ids.long().flatten(), dx.float().reshape(-1, d))
    assert relmax(dwte, ref) < 1e-5 and relmax(dwpe, dx.float().sum(0)) < 1e-5
    labels = torch.empty(B, S, dtype=torch.int32, device=DEV)
    ops.shift_labels(ids.to(DEV), labels, V - 1)
    exp = torch.cat([ids[:, 1:], torch.full((B, 1), V - 1, dtype=torch.int32)], 1)
    assert torch.equal(labels.cpu(), exp)                                      # integer work: bit-exact
    text = torch.randint(0, 50, (B, 5), generator=g, dtype=torch.int32)
    img = torch.randint(0, 16, (B, 4), generator=g, dtype=torch.int32)
    toks = torch.empty(B, 9, dtype=torch.int32, device=DEV)
    ops.assemble_tokens(text.to(DEV), img.to(DEV), toks, 50)
    assert torch.equal(toks.cpu(), torch.cat([text, img + 50], 1))


@pytest.mark.parametrize("d", [256, 512, 768, 1024, 2048, 4096])   # 4096: the wide kernel (12 B width)
def test_layernorm_fwd_bwd(ops, d):
    g = torch.Generator().manual_seed(d)
    rows = 203
    x = bf(torch.randn(rows, d, generator=g) * 2 + 0.5)
    gg, bb = torch.randn(d, generator=g), torch.randn(d, generator=g)
    y = torch.empty(rows, d, dtype=torch.bfloat16, device=DEV)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    ops.layernorm_fwd(x.to(DEV), gg.to(DEV), bb.to(DEV), y, mean, rstd)
    xf = x.float().requires_grad_(True); gp = gg.clone().requires_grad_(True); bp = bb.clone().requires_grad_(True)
    yref = torch.nn.functional.layer_norm(xf, (d,), gp, bp, 1e-5)
    assert relmax(y, yref) < 1e-2
    dy, dres = bf(torch.randn(rows, d, generator=g)), bf(torch.randn(rows, d, generator=g))
    yref.backward(dy.float())
    dx = torch.empty(rows, d, dtype=torch.bfloat16, device=DEV)
    dg, db = torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    ops.layernorm_bwd(dy.to(DEV), x.to(DEV), gg.to(DEV), mean, rstd, dres.to(DEV), dx, dg, db)
    assert relmax(dx, xf.grad + dres.float()) < 1e-2
    assert relmax(dg, gp.grad) < 1e-4 and relmax(db, bp.grad) < 1e-4
    dx2, dxs = torch.empty_like(dx), torch.zeros(d, device=DEV)
    ops.layernorm_bwd(dy.to(DEV), x.to(DEV), gg.to(DEV), mean, rstd, dres.to(DEV), dx2, torch.zeros(d, device=DEV),
                      torch.zeros(d, device=DEV), dxsum=dxs)                    # fused column sums of dx
    assert torch.equal(dx2, dx) and relmax(dxs, dx.float().sum(0)) < 1e-5
    # the entry point without dxsum: the same kernels, so the same bits
    from dalle_mtf_b200 import lib as L
    dyd, xd, gd, dresd = dy.to(DEV), x.to(DEV), gg.to(DEV), dres.to(DEV)
    dx3, dg3, db3 = torch.empty_like(dx), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    ws = L.workspace(L.load().db200_layernorm_bwd_workspace_bytes(rows, d))
    L.check(L.load().db200_layernorm_bwd(L.stream_ptr(), dyd.data_ptr(), xd.data_ptr(), gd.data_ptr(), mean.data_ptr(),
                                         rstd.data_ptr(), dresd.data_ptr(), dx3.data_ptr(), dg3.data_ptr(),
                                         db3.data_ptr(), rows, d, L.ptr(ws), ws.numel() if ws is not None else 0),
            "db200_layernorm_bwd")
    assert torch.equal(dx3, dx) and torch.equal(dg3, dg) and torch.equal(db3, db)


def test_colsum_and_casts(ops):
    g = torch.Generator().manual_seed(5)
    x = bf(torch.randn(1000, 520, generator=g))
    o = torch.zeros(520, device=DEV)
    ops.colsum(x.to(DEV), o)
    assert relmax(o, x.float().sum(0)) < 1e-5
    f = torch.randn(100003, generator=g)
    b16 = torch.empty(100003, dtype=torch.bfloat16, device=DEV)
    ops.cast_f32_to_bf16(f.to(DEV), b16)
    assert torch.equal(b16.cpu(), f.to(torch.bfloat16))                         # round-to-nearest-even: bit-exact
    back = torch.empty(100003, device=DEV)
    ops.cast_bf16_to_f32(b16, back)
    assert torch.equal(back.cpu(), f.to(torch.bfloat16).float())


# ------------------------------------------------------------------------------------------------------- optimiser
def test_sqnorm_and_adam_variants(ops):
    from oracle import optim as OO
    g = torch.Generator().manual_seed(4)
    n = 100003
    p, m, v = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1, torch.rand(n, generator=g) * 0.01
    gr = torch.randn(n, generator=g)
    acc = torch.zeros(1, device=DEV)
    ops.sqnorm(gr.to(DEV), acc)
    assert relmax(acc, (gr.double() ** 2).sum().float().reshape(1)) < 1e-5
    pd, md, vd = p.to(DEV), m.to(DEV), v.to(DEV)
    p16 = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ops.adam_step(pd, md, vd, gr.to(DEV), p16, lr=1e-3, eps=1e-6, gnorm_sq=acc, clip=1.0)   # mtf Adam + global-norm clip
    clipped, _ = OO.clip_by_global_norm({"g": gr}, 1.0)
    p2, m2, v2 = OO.adam_mtf_step(p, m, v, clipped["g"], 1e-3)
    assert relmax(pd, p2) < 1e-6 and relmax(md, m2) < 1e-6 and relmax(vd, v2) < 1e-6
    assert torch.equal(p16.cpu(), pd.cpu().to(torch.bfloat16))                  # shadow = rounded updated parameter
    pd, md, vd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ops.adam_step(pd, md, vd, gr.to(DEV), None, lr=1e-3, eps=1e-8, bias_correction=True, step=1, grad_scale=0.5)
    p3, _, _ = OO.adam_tf_step(p, torch.zeros(n), torch.zeros(n), gr * 0.5, 1e-3, 1)
    assert relmax(pd, p3) < 1e-6


# ------------------------------------------------------------------------------------------------------- attention
def _ref_attn(qkv, scale):
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    s = torch.einsum("bihe,bjhe->bhij", q, k) * scale
    S = q.shape[1]
    s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool), 1), float("-inf"))
    return torch.einsum("bhij,bjhe->bihe", torch.softmax(s, -1), v), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,S,H,dh,scale,mag", [(1, 128, 1, 128, 1.0, 0.3), (1, 128, 1, 64, 1.0, 0.4),
                                                (2, 256, 2, 128, 1.0, 0.3), (1, 300, 3, 64, 0.125, 1.0),
                                                (1, 333, 2, 128, 0.0884, 1.0), (1, 1, 1, 64, 1.0, 1.0),
                                                (2, 1280, 4, 128, 1.0, 0.25), (1, 640, 2, 128, 1.0, 1.2),
                                                (1, 520, 3, 64, 1.0, 1.5), (1, 129, 1, 128, 1.0, 0.5),
                                                (2, 1280, 3, 64, 0.125, 1.0),
                                                # more work items than SMs: several items per persistent CTA
                                                (8, 1280, 5, 128, 1.0, 0.25), (6, 1280, 8, 64, 0.125, 1.0),
                                                (5, 640, 8, 128, 1.0, 1.2)])
def test_causal_attention_fwd_bwd(ops, B, S, H, dh, scale, mag):
    g = torch.Generator().manual_seed(S + dh)
    qkv = bf(torch.randn(B, S, 3, H, dh, generator=g) * mag)
    dout = bf(torch.randn(B, S, H, dh, generator=g))
    qf = qkv.float().requires_grad_(True)
    o_ref, lse_ref = _ref_attn(qf, scale)
    o_ref.backward(dout.float())
    qd, dd = qkv.to(DEV), dout.to(DEV)
    out = torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, H, S, device=DEV)
    ops.attn_fwd(qd, out, lse, B, S, H, dh, scale)
    assert relmax(out, o_ref) < 1e-2 and relmax(lse, lse_ref) < 1e-3
    dqkv = torch.zeros_like(qd)
    ops.attn_bwd(qd, out, dd, lse, torch.zeros(1, device=DEV), torch.zeros(B, H, S, device=DEV), dqkv, B, S, H, dh, scale)
    for i in range(3):   # P and dS are rounded to bf16 before the second products -> 2e-2
        ref = qf.grad[:, :, i]
        if ref.abs().max() == 0:   # S = 1: one key, P = 1, dq = dk = 0 exactly; the kernels give dP - delta with O rounded
            assert dqkv[:, :, i].float().abs().max().item() < 1e-4     # to bf16 inside delta: ~1e-6, not 0
        else:
            assert relmax(dqkv[:, :, i], ref) < 2e-2


def test_attention_is_causal_at_full_size(ops):
    """Property at the bench shape: changing keys/values at positions > t must not change outputs at positions <= t."""
    B, S, H, dh = 2, 1280, 4, 128
    g = torch.Generator(device=DEV).manual_seed(0)
    qkv = bf(torch.randn(B, S, 3, H, dh, generator=g, device=DEV) * 0.3)
    o1, o2 = (torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    lse = torch.zeros(B, H, S, device=DEV)
    ops.attn_fwd(qkv, o1, lse, B, S, H, dh, 1.0)
    q2 = qkv.clone()
    q2[:, 700:, 1:] = bf(torch.randn(B, S - 700, 2, H, dh, generator=g, device=DEV))
    ops.attn_fwd(q2, o2, lse, B, S, H, dh, 1.0)
    assert torch.equal(o1[:, :700], o2[:, :700]) and not torch.equal(o1[:, 700:], o2[:, 700:])
