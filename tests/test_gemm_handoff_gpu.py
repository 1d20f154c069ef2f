"""The GEMM hands each accumulator tile from its MMA warpgroups to a separate epilogue warpgroup through one
single-buffered shared-memory tile.  These cases make that hand-off as tight as it gets: K = 64 (or one k-block per
split) makes every tile's mainloop a single k-block, so the MMA warpgroups are back at the accumulator tile as soon as
the epilogue releases it, and the shapes give each persistent CTA (one per SM) about ten tiles.  A missing or
misplaced wait shows up as values from the wrong tile.  Tolerances as in test_kernels_gpu.py.
"""
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


@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("b_mn", [False, True])
def test_gemm_single_k_block_many_tiles_per_cta(ops, a_mn, b_mn):
    M, N, K = 40960, 512, 64                       # 320 x 4 tiles
    g = torch.Generator().manual_seed(5)
    A, B = bf(torch.randn(M, K, generator=g)), bf(torch.randn(K, N, generator=g))
    ref = A.float() @ B.float()
    a = A.t().contiguous().to(DEV) if a_mn else A.to(DEV)
    b = B.to(DEV) if b_mn else B.t().contiguous().to(DEV)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn)
    assert relmax(out, ref) < 1e-2
    out32 = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, b, out32, M, N, K, a_mn=a_mn, b_mn=b_mn)
    assert relmax(out32, ref) < 1e-5


def test_gemm_epilogues_single_k_block_on_a_large_ragged_shape(ops):
    """Every epilogue at K = 64 on 79 x 17 tiles whose last rows and columns end inside a tile."""
    from dalle_mtf_b200 import lib as L
    g = torch.Generator().manual_seed(12)
    M, N, K = 10056, 2056, 64
    A, W = bf(torch.randn(M, K, generator=g)), bf(torch.randn(K, N, generator=g) * 0.1)
    bias, res = torch.randn(N, generator=g), bf(torch.randn(M, N, generator=g))
    a, w = A.to(DEV), W.to(DEV)
    prod = A.float() @ W.float()
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.linear_fwd(a, w, out, bias=bias.to(DEV), relu=True, residual=res.to(DEV))
    assert relmax(out, torch.relu(prod + bias) + res.float()) < 1e-2
    out32 = torch.empty(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, w, out32, M, N, K, a_mn=False, b_mn=True, alpha=0.5, bias=bias.to(DEV))
    assert relmax(out32, 0.5 * prod + bias) < 1e-5
    # red.add into D, and split-K slices with one k-block per split
    acc = torch.ones(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(a, w, acc, M, N, K, a_mn=False, b_mn=True, mode=L.EPI_ATOMIC, alpha=0.5)
    assert relmax(acc, 1.0 + 0.5 * prod) < 1e-5
    A2, W2s = bf(torch.randn(M, 128, generator=g)), bf(torch.randn(128, N, generator=g) * 0.1)
    acc2 = torch.ones(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(A2.to(DEV), W2s.to(DEV), acc2, M, N, 128, a_mn=False, b_mn=True, mode=L.EPI_ATOMIC, split_k=2)
    assert relmax(acc2, 1.0 + A2.float() @ W2s.float()) < 1e-5
    # ReLU-masked dgrad with the fused bias gradient: dx[M, N] = (dy[M, K] @ W2^T) * (h > 0)
    DY, W2, H = bf(torch.randn(M, K, generator=g)), bf(torch.randn(N, K, generator=g) * 0.1), bf(torch.randn(M, N, generator=g))
    dx = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    cs = torch.zeros(N, device=DEV)
    ops.linear_dgrad(DY.to(DEV), W2.to(DEV), dx, relu_mask_of=H.to(DEV), colsum=cs)
    assert relmax(dx, (DY.float() @ W2.float().t()) * (H.float() > 0)) < 1e-2
    assert relmax(cs, dx.float().sum(0)) < 1e-5
    # cross-entropy statistics and gradient over 79 x 16 tiles
    T, d, V, Vpad = M, K, 2000, 2048
    X = bf(torch.randn(T, d, generator=g))
    Wv = torch.zeros(d, Vpad); Wv[:, :V] = torch.randn(d, V, generator=g) * 0.3; Wv = bf(Wv)
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
