"""gMLP token-mixing layers on the GPU: the three causal mixing products (db200_sgu_mix_fwd / _dgrad / _wgrad), the SGU
backward kernels and the decoding step against float64 at the engine's, the prefill's and the decoder's shapes; the
engine against oracle/dalle_gmlp.py on mixed models (loss, logits, every gradient), with the oracle's mutants failing
the same bounds, at one and at three mixing tiles, and bit-exact causality; reproducibility, the causal invariant through
Adam with weight decay and through ZeRO-1, the sharded initialisation, in-process data-parallel ranks, decoding,
prefill, guidance and checkpoints."""
import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, relfro

pytestmark = pytest.mark.gpu
BF16, F32, I32, F64 = torch.bfloat16, torch.float32, torch.int32, torch.float64


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _rand(shape, seed, scale=1.0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _causal_w(n, seed, pitch=None):
    """A bf16 [pitch, pitch] weight whose top-left lower triangle is random (row i ~ N(0, 1 / (i + 1))), zero above."""
    pitch = pitch or n
    rows = torch.arange(pitch, device=DEV, dtype=F32)[:, None] + 1
    return torch.tril(_rand((pitch, pitch), seed, dtype=F32) / rows.sqrt()).to(BF16)


def _close(got, want, tol, what=""):
    e = relfro(got, want)
    assert e < tol, (what, e)


# ------------------------------------------------------------------------------------------------ mixing products
# (B, n, C): dalle_example (S 1280, 2d 1024) at part of its batch, the dalle_coco width (2d 2048), partial last m-tiles
# (n = 192, 320), one-tile sequences and the prefill's lengths (fwd only: any n)
SHAPES = [(8, 1280, 1024), (2, 256, 2048), (3, 192, 512), (2, 320, 1024), (4, 64, 512), (1, 128, 4096)]
PREFILL = [(2, 1, 1024), (3, 70, 512), (2, 200, 1024), (1, 1279, 1024)]


def _fwd64(w, gn, res, c, B, n):
    C = gn.shape[1]
    m = torch.einsum("ij,bjc->bic", torch.tril(w[:n, :n].double()), gn.double().view(B, n, C)) + \
        c[:n].double()[None, :, None]
    return m.reshape(B * n, C), (m.reshape(B * n, C) * res.double())


@pytest.mark.parametrize("B,n,C", SHAPES + PREFILL, ids=[f"{b}x{n}x{c}" for b, n, c in SHAPES + PREFILL])
def test_mix_fwd_matches_float64(ops, B, n, C):
    S = max(n, 64 * ((n + 63) // 64))
    w = _causal_w(n, 1, pitch=S)                              # the prefill reads the top-left n x n block
    gn, u = _rand((B * n, C), 2), _rand((B * n, 2 * C), 3)
    res = u[:, :C]                                            # the first half of proj_in's output, pitch 2C
    c = _rand((S,), 4, 0.3, F32) + 1
    h, mixed = torch.empty(B * n, C, dtype=BF16, device=DEV), torch.empty(B * n, C, dtype=BF16, device=DEV)
    ops.sgu_mix_fwd(w, gn, res, c, h, mixed, B, n)
    m64, h64 = _fwd64(w, gn, res, c, B, n)
    _close(mixed, m64, 5e-3, "mixed")
    _close(h, h64, 5e-3, "h")
    h2 = torch.empty_like(h)
    ops.sgu_mix_fwd(w, gn, res, c, h2, None, B, n)           # without the mixed output: the same h
    assert torch.equal(h, h2)


@pytest.mark.parametrize("B,n,C", SHAPES, ids=[f"{b}x{n}x{c}" for b, n, c in SHAPES])
def test_mix_dgrad_and_wgrad_match_float64(ops, B, n, C):
    w = _causal_w(n, 5)
    dm, gn = _rand((B * n, C), 6), _rand((B * n, C), 7)
    dgn = torch.empty(B * n, C, dtype=BF16, device=DEV)
    ops.sgu_mix_dgrad(w, dm, dgn, B, n)
    want = torch.einsum("ij,bic->bjc", w.double(), dm.double().view(B, n, C)).reshape(B * n, C)
    _close(dgn, want, 5e-3, "dgn")
    dw0 = _rand((n, n), 8, 1.0, F32)                          # accumulates into what is there
    dw = dw0.clone()
    ops.sgu_mix_wgrad(dm, gn, dw, B, n)
    full = torch.einsum("bic,bjc->ij", dm.double().view(B, n, C), gn.double().view(B, n, C))
    low = torch.tril(torch.ones(n, n, dtype=torch.bool, device=DEV))
    _close((dw.double() - dw0.double())[low], full[low], 1e-4, "dW")
    assert torch.equal(dw[~low], dw0[~low])                    # the strict upper triangle is never written
    z = torch.zeros(n, n, dtype=F32, device=DEV)
    ops.sgu_mix_wgrad(dm, gn, z, B, n)
    assert not z.triu(1).any()                                 # ... so a zero gradient stays exactly zero there
    z2 = torch.zeros_like(z)
    ops.sgu_mix_wgrad(dm, gn, z2, B, n)
    assert torch.equal(z, z2)                                  # fixed order: bit-reproducible


@pytest.mark.parametrize("B,n,C", [(2, 256, 512), (3, 320, 1024), (2, 70, 512), (2, 200, 512)])
def test_forward_k_range_ends_with_the_diagonal_tile(ops, B, n, C):
    """A weight that is non-zero everywhere above its diagonal: the forward product of the 128-row tile of row i reads
    the columns j < min(128 (i // 128 + 1), n) (the triangle is an invariant the engine keeps, not a mask applied at
    use), so the entries inside the diagonal tile count and every entry past it is ignored."""
    pitch = 64 * ((n + 63) // 64)                             # a prefill's length: the block of a longer weight
    w = _causal_w(pitch, 9).float() + torch.triu(torch.ones(pitch, pitch, device=DEV), 1) * 0.5
    i = torch.arange(n, device=DEV)[:, None]
    j = torch.arange(n, device=DEV)[None, :]
    read = j < torch.clamp(128 * (i // 128 + 1), max=n)
    w = w.to(BF16)
    gn, res = _rand((B * n, C), 10), _rand((B * n, C), 11)
    c = torch.ones(n, device=DEV)
    h = torch.empty(B * n, C, dtype=BF16, device=DEV)
    ops.sgu_mix_fwd(w, gn, res, c, h, None, B, n)
    wn = w[:n, :n].double()
    want = torch.einsum("ij,bjc->bic", torch.where(read, wn, 0.0), gn.double().view(B, n, C)) + 1
    _close(h, (want.reshape(B * n, C) * res.double()), 5e-3, "tile-bounded K range")
    over = torch.einsum("ij,bjc->bic", wn, gn.double().view(B, n, C)) + 1
    if not bool(read.all()):   # reading past the diagonal tile would be far outside the bound
        assert relfro(h, over.reshape(B * n, C) * res.double()) > 0.1


def test_argument_checks(ops):
    from dalle_mtf_b200 import lib as L
    w = _causal_w(128, 1)
    gn = _rand((256, 512), 2)
    with pytest.raises(L.DB200Error):
        ops.sgu_mix_dgrad(w, gn[:, :96].contiguous(), torch.empty(256, 96, dtype=BF16, device=DEV), 2, 128)  # C % 64
    with pytest.raises(L.DB200Error):
        ops.sgu_mix_wgrad(gn[:200], gn[:200], torch.zeros(100, 100, device=DEV), 2, 100)                      # n % 64
    with pytest.raises(L.DB200Error):
        ops.sgu_decode(gn[:2], gn[:2], w, torch.ones(128, device=DEV), torch.zeros(2, 128, 512, dtype=BF16,
                                                                                     device=DEV),
                       torch.empty(2, 512, dtype=BF16, device=DEV), 128)                                        # pos


# ------------------------------------------------------------------------------------------------ SGU backward
@pytest.mark.parametrize("B,n,C", [(32, 1280, 1024), (4, 256, 2048), (3, 192, 512)])
def test_sgu_bwd_and_gate_bwd_match_float64(ops, B, n, C):
    from oracle.dalle_gelu import gelu_grad
    T = B * n
    dh, mixed = _rand((T, C), 1), _rand((T, C), 2)
    u, z = _rand((T, 2 * C), 3), _rand((T, 2 * C), 4)
    dmixed = torch.empty(T, C, dtype=BF16, device=DEV)
    du = torch.zeros(T, 2 * C, dtype=BF16, device=DEV)
    dc0 = _rand((n,), 5, 1.0, F32)
    dc = dc0.clone()
    ops.sgu_bwd(dh, mixed, u[:, :C], z[:, :C], dmixed, du[:, :C], dc, B, n)
    dm64 = dh.double() * u[:, :C].double()
    assert (dmixed.double() - dm64).abs().max() <= (dm64.abs() * 2 ** -8).max()
    dres64 = dh.double() * mixed.double() * gelu_grad(z[:, :C].double())
    _close(du[:, :C], dres64, 5e-3, "du_res")
    dc64 = dmixed.double().view(B, n, C).sum((0, 2))
    _close(dc.double() - dc0.double(), dc64, 1e-5, "dc")
    dc2 = dc0.clone()
    ops.sgu_bwd(dh, mixed, u[:, :C], z[:, :C], dmixed, du[:, :C], dc2, B, n)
    assert torch.equal(dc, dc2)
    dgate = _rand((T, C), 6)
    ops.sgu_gate_bwd(dgate, z[:, C:], du[:, C:])
    _close(du[:, C:], dgate.double() * gelu_grad(z[:, C:].double()), 5e-3, "du_gate")


# ------------------------------------------------------------------------------------------------ decoding kernels
@pytest.mark.parametrize("rows,S,C", [(32, 1280, 1024), (64, 1280, 1024), (8, 320, 2048), (3, 64, 512)])
def test_sgu_decode_and_cache_fill_match_float64(ops, rows, S, C):
    w = _causal_w(S, 1)
    c = _rand((S,), 2, 0.3, F32) + 1
    cache = _rand((rows, S, C), 3)
    pos_dev = torch.zeros(1, dtype=I32, device=DEV)
    for pos in sorted({0, 1, 63, 64, S // 2, S - 1} & set(range(S))):
        gn, res = _rand((rows, C), 10 + pos), _rand((rows, 2 * C), 20 + pos)[:, :C]
        h = torch.empty(rows, C, dtype=BF16, device=DEV)
        ops.sgu_decode(gn, res, w, c, cache, h, pos)
        assert torch.equal(cache[:, pos], gn)
        m = torch.einsum("j,rjc->rc", w[pos, :pos + 1].double(), cache[:, :pos + 1].double()) + c[pos].double()
        _close(h, m * res.double(), 5e-3, pos)
        h2 = torch.empty_like(h)
        pos_dev.fill_(pos)
        ops.sgu_decode_dev(gn, res, w, c, cache, h2, pos_dev)
        assert torch.equal(h, h2)
    before = cache.clone()
    pos_dev.fill_(S)                                           # outside [0, S): nothing changes
    ops.sgu_decode_dev(gn, res, w, c, cache, h2, pos_dev)
    assert torch.equal(cache, before)
    B, P, rep = 2, min(37, S - 1), 3
    src = _rand((B * P, C), 5)
    fill = torch.zeros(B * rep, S, C, dtype=BF16, device=DEV)
    ops.sgu_cache_fill(src, fill, P, rep)
    for b in range(B):
        for r in range(rep):
            assert torch.equal(fill[b * rep + r, :P], src[b * P:(b + 1) * P])
    assert not fill[:, P:].any()


# ------------------------------------------------------------------------------------------------ engine vs oracle
TYPE_SETS = {"global_mlp": ("global", "mlp"), "axial_mlp": ("axial_row", "axial_col", "mlp")}
# S = 64 text + 256 image positions: three 128-row mixing tiles, the last one partial
LONG = dict(TL=64, W=16)
VARIANTS = {"plain": {}, "sandwich": {"sandwich_norm": True}, "shift": {"shift_tokens": True},
            "geglu_rotary": {"gated_mlp": True, "activation": "gelu", "rotary_dim": 32},
            "dropout": {"dropout": (0.1, 0.1, 0.2)}, "recompute": {"recompute_grad": True}}


def _gmlp_model(types, seed=3, d=256, H=2, TL=28, W=10):
    from oracle import dalle as O, dalle_gmlp as OM, dalle_local as OL
    cfg = OL.LocalConfig(d, len(types), H, 300, 64, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    tokens = O.assemble_tokens(torch.randint(0, 299, (2, TL), generator=g),
                               torch.randint(0, 64, (2, W * W), generator=g), 300)
    return cfg, params, tokens


def _oracle_kw(cfg, variant):
    from oracle import dalle_gmlp as OM  # noqa: F401
    import axial_oracle as AX
    kw = {"bf16": True, "layers": AX}
    if variant.get("sandwich_norm"):
        kw["sandwich_norm"] = True
    if variant.get("shift_tokens"):
        kw["shift_tokens"] = True
    if variant.get("gated_mlp"):
        kw.update(gated=True, activation="gelu", rotary=(variant["rotary_dim"], 10000.0))
    return kw


def _with_variant_params(cfg, params, variant):
    from oracle import dalle_glu as OGL, dalle_sandwich as OSW
    if variant.get("sandwich_norm"):
        params = OSW.init_params(params, cfg, 11)
    if variant.get("gated_mlp"):
        params = OGL.init_params(params, cfg, 12)
    return params


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("types", list(TYPE_SETS))
def test_engine_matches_the_oracle(types, variant):
    import axial_oracle as AX
    from oracle import dalle_gmlp as OM
    v = VARIANTS[variant]
    cfg, params, tokens = _gmlp_model(TYPE_SETS[types])
    cfg = AX.AxialConfig(**{**cfg.__dict__})
    params = _with_variant_params(cfg, params, v)
    kw = _oracle_kw(cfg, v)
    dropout = None
    if "dropout" in v:
        dropout = (v["dropout"], 7, 3, 0)
    loss_ref, rows_ref, logits_ref, grads_ref = OM.loss_and_grads(params, tokens, cfg, dropout=dropout, **kw)
    grads32 = OM.loss_and_grads(params, tokens, cfg, dropout=dropout, **{**kw, "bf16": False})[3]
    eng = _engine(cfg, attention_types=list(cfg.attention_types), dropout_seed=7, **v)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    eng.zero_grads()
    T = tok.numel()
    acc = eng.forward(tok, step=3 if dropout else None)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    assert abs(loss - loss_ref.item()) / loss_ref.item() < 2e-3, (loss, loss_ref.item())
    grads = eng.export_params(eng.grads)
    # every gradient no further from the fp32 oracle than 1.25 x the oracle's own bf16 policy + 1e-2
    excess = max((relfro(grads[k], grads32[k]) - 1.25 * relfro(grads_ref[k], grads32[k]) - 1e-2, k)
                 for k in grads32 if grads32[k].norm() > 0)
    print(f"[gmlp {types}/{variant}] loss {loss:.6f} oracle {loss_ref.item():.6f}; worst excess {excess}")
    assert excess[0] <= 0, excess
    for k in grads:
        if k.endswith("gmlp/sgu/weight"):
            assert not grads[k].triu(1).any(), k
    if not dropout:
        _close(eng.logits(tok), logits_ref, 1e-2, "logits")
    if variant == "plain":   # each mutant fails the bounds the engine passes
        for m in OM.MUTATIONS:
            # "unmasked" computes what the oracle computes on every weight the engine can hold (the upper triangle is
            # kept at exactly 0; test_engine_is_causal_bit_for_bit_over_several_mixing_tiles checks causality itself),
            # and "erf_gelu" moves u by at most 4.7e-4, 3 % of a bf16 ulp there (test_mlp_layers_cpu.py: it differs)
            if m in ("unmasked", "erf_gelu"):
                continue
            lm, _, _, gm = OM.loss_and_grads(params, tokens, cfg, gmlp_mutate=m, **kw)
            gm32 = OM.loss_and_grads(params, tokens, cfg, gmlp_mutate=m, **{**kw, "bf16": False})[3]
            wm = max(relfro(grads[k], gm32[k]) - 1.25 * relfro(gm[k], gm32[k]) - 1e-2 for k in gm32
                     if gm32[k].norm() > 0)
            assert abs(loss - lm.item()) / lm.item() >= 2e-3 or wm > 0, m


@pytest.mark.parametrize("types", list(TYPE_SETS))
def test_engine_matches_the_oracle_over_several_mixing_tiles(types):
    """S = 320 (three m-tiles of the mixing products, tiles on and beside the diagonal, a partial last tile): loss and
    every gradient within the bf16-policy bound of the fp32 oracle."""
    import axial_oracle as AX
    from oracle import dalle_gmlp as OM
    cfg, params, tokens = _gmlp_model(TYPE_SETS[types], **LONG)
    cfg = AX.AxialConfig(**{**cfg.__dict__})
    kw = _oracle_kw(cfg, {})
    loss_ref, _, logits_ref, grads_ref = OM.loss_and_grads(params, tokens, cfg, **kw)
    grads32 = OM.loss_and_grads(params, tokens, cfg, **{**kw, "bf16": False})[3]
    eng = _engine(cfg, attention_types=list(cfg.attention_types))
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    eng.zero_grads()
    T = tok.numel()
    loss = eng.forward(tok).item() / T
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    assert abs(loss - loss_ref.item()) / loss_ref.item() < 2e-3, (loss, loss_ref.item())
    grads = eng.export_params(eng.grads)
    excess = max((relfro(grads[k], grads32[k]) - 1.25 * relfro(grads_ref[k], grads32[k]) - 1e-2, k)
                 for k in grads32 if grads32[k].norm() > 0)
    print(f"[gmlp S=320 {types}] loss {loss:.6f} oracle {loss_ref.item():.6f}; worst excess {excess}")
    assert excess[0] <= 0, excess
    _close(eng.logits(tok), logits_ref, 1e-2, "logits")


def test_engine_is_causal_bit_for_bit_over_several_mixing_tiles():
    """Changing token j leaves the engine's logits at every position before j bit-identical (S = 320, gMLP layers
    only besides the embedding and head)."""
    cfg, params, tokens = _gmlp_model(("mlp", "mlp"), **LONG)
    eng = _engine(cfg, attention_types=list(cfg.attention_types))
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    base = eng.logits(tok).clone()
    for j in (1, 127, 128, 200, 256, 319):
        t2 = tok.clone()
        t2[:, j] = (t2[:, j] + 1) % 300
        got = eng.logits(t2)
        assert torch.equal(got[:, :j], base[:, :j]), j
        assert not torch.equal(got[:, j:], base[:, j:]), j


def test_two_steps_are_bit_identical_and_adam_keeps_the_triangle_zero():
    cfg, params, tokens = _gmlp_model(("global", "mlp", "mlp"))
    tok = tokens.to(I32).to(DEV)
    eng = _engine(cfg, attention_types=list(cfg.attention_types), dropout=(0.1, 0.0, 0.1))
    eng.load_params(params)
    eng.zero_grads(); eng.forward(tok, step=1); eng.backward(1e-2)
    g1 = eng.grads.clone()
    eng.zero_grads(); eng.forward(tok, step=1); eng.backward(1e-2)
    assert torch.equal(g1, eng.grads)
    for step in range(4):
        eng.zero_grads(); eng.forward(tok, step=step); eng.backward(1e-2)
        eng.optimizer_step(1e-2, weight_decay=0.1)
    torch.cuda.synchronize()
    out = eng.export_params()
    for i in (1, 2):
        w = out[f"layer_{i}/gmlp/sgu/weight"]
        assert not w.triu(1).any()
        assert not torch.equal(w, params[f"layer_{i}/gmlp/sgu/weight"])   # the lower triangle trained


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_initialisation_equals_the_replicated_one_and_keeps_the_triangle(world):
    """init_params of ZeRO-1 ranks (_init_params_sharded, one tensor at a time) draws the same random stream as the
    replicated init_params: every rank's bf16 parameters are the replicated ones rounded to bf16, bit for bit; the
    mixing weight starts lower triangular within U(-1e-3/S, 1e-3/S) and c_sgu = 1."""
    from test_zero1_gpu import Loopback
    cfg, _, _ = _gmlp_model(("mlp", "global", "mlp"))
    types = list(cfg.attention_types)
    eng = _engine(cfg, attention_types=types)
    eng.init_params(seed=3)
    grp = Loopback(world)
    grp.engines = ranks = [_engine(cfg, attention_types=types, zero=grp.member(r)) for r in range(world)]
    for e in ranks:
        e.init_params(seed=3)
    torch.cuda.synchronize()
    p = eng.export_params()
    for r, e in enumerate(ranks):
        ex = e.export_params()
        for k, v in p.items():
            assert torch.equal(ex[k], v.to(BF16).float()), (r, k)
    S = cfg.seq_len
    for i in (0, 2):
        w = p[f"layer_{i}/gmlp/sgu/weight"]
        assert not w.triu(1).any() and w.abs().max() <= 1e-3 / S and w.tril().abs().max() > 0
        assert torch.equal(p[f"layer_{i}/gmlp/sgu/bias"], torch.ones(S))


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion (bit for bit, every bucket all-reduced once per step) on a model with
    gMLP layers and every feature of that test: S = 48 text + 16 image positions."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, text_seq_len=48, attention_types=[[["global", "mlp", "axial_row", "mlp"], 1]])
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    assert _seq_len(p) == 64
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


@pytest.mark.parametrize("world", [2, 3])
def test_zero1_step_equals_the_replicated_step_bitwise_and_keeps_the_triangle(ops, world):
    """test_zero1_gpu.py's emulation: W ranks with sharded optimiser state (the gMLP vectors gm_bin, sgu_g / sgu_b,
    sgu_c and gm_bout in the fp32 vector table) give the replicated step's gradients and parameters bit for bit, and
    the mixing weights' strict upper triangles stay exactly 0 through the sharded Adam steps."""
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tokens = _gmlp_model(("global", "mlp", "axial_col", "mlp"), seed=11)
    types = list(cfg.attention_types)
    params = {k: v.to(BF16).float() for k, v in params.items()}
    tok = tokens.to(I32).to(DEV)
    grp = Loopback(world)
    grp.engines = ranks = [_engine(cfg, attention_types=types, zero=grp.member(r)) for r in range(world)]
    twin = _engine(cfg, attention_types=types)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    # the replicated optimiser state, stepped by the Adam kernel on the full buffer (test_zero1_gpu.py's emulation)
    P = twin.master[:n].clone()
    M, V = torch.zeros_like(P), torch.zeros_like(P)
    gn = torch.zeros(1, dtype=F32, device=DEV)
    for step in range(3):
        # the twin reads its vector parameters as the ZeRO engine's fp32 table does: rebuilt from the bf16 copy
        _twin_from(twin, P, ranks[0])
        assert_same_bits(twin.shadow[:n], ranks[0].shadow[:n], f"step {step}: twin bf16 parameters")
        g_ref = _step(twin, tok, 1e-2)
        for r, e in enumerate(ranks):
            assert_same_bits(_step(e, tok, 1e-2), g_ref, f"ZeRO-1 rank {r} step {step} gradients")
        for e in ranks:
            e.optimizer_step(1e-3, clip=1.0)
        gn.zero_()
        ops.sqnorm(g_ref[:n], gn)
        ops.adam_step(P, M, V, g_ref[:n], twin.shadow[:n], 1e-3, 0.9, 0.999, 1e-6, 0.0, gn, 1.0, 1.0, False, 0)
        for r, e in enumerate(ranks):
            lo, hi = e.shard
            assert_same_bits(e.master[:hi - lo], P[lo:hi], f"ZeRO-1 rank {r} step {step} fp32 slice")
            assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} step {step} parameters")
    twin.master[:n].copy_(P)
    ex = ranks[0].export_params()
    for k, v in twin.export_params().items():
        assert torch.equal(ex[k], v.to(BF16).float()), k
    for i in (1, 3):
        w = ex[f"layer_{i}/gmlp/sgu/weight"]
        assert not w.triu(1).any()
        assert not torch.equal(w, params[f"layer_{i}/gmlp/sgu/weight"])   # the lower triangle trained


def test_checkpoint_round_trip_resume_and_refusals():
    from dalle_mtf_b200 import lib as L
    cfg, params, tokens = _gmlp_model(("axial_row", "mlp"))
    tok = tokens.to(I32).to(DEV)
    a = _engine(cfg, attention_types=list(cfg.attention_types))
    a.load_params(params)
    for s in range(2):
        _step(a, tok, 1e-2); a.optimizer_step(1e-3)
    saved = {n: a.export_params(src) for n, src in (("p", None), ("m", a.adam_m), ("v", a.adam_v))}
    _step(a, tok, 1e-2); a.optimizer_step(1e-3)
    b = _engine(cfg, attention_types=list(cfg.attention_types))
    b.load_params(saved["p"])
    b.load_flat(b.adam_m, saved["m"]); b.load_flat(b.adam_v, saved["v"])
    _step(b, tok, 1e-2)
    b.optimizer_step(1e-3)
    torch.cuda.synchronize()
    assert torch.equal(a.master, b.master)                     # the resumed step equals the uninterrupted one
    with pytest.raises(L.DB200Error, match="layer_1/gmlp"):
        _engine(cfg, attention_types=["axial_row", "global"]).load_params(saved["p"])
    bad = dict(saved["p"])
    bad["layer_1/gmlp/sgu/weight"] = bad["layer_1/gmlp/sgu/weight"].clone()
    bad["layer_1/gmlp/sgu/weight"][0, 5] = 1.0
    with pytest.raises(L.DB200Error, match="upper triangle"):
        b.load_params(bad)


# ------------------------------------------------------------------------------------------------ decoding
def test_decoding_follows_the_full_forward_and_the_prefill():
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward
    types = ("axial_row", "mlp", "axial_col", "mlp")
    cfg, params, _ = _gmlp_model(types, seed=5)
    for k in params:
        if "wte" in k or "linear_out" in k:
            params[k] = params[k] * 4
    ts, W = cfg.text_seq_len, 10
    S = ts + W * W
    eng = _engine(cfg, attention_types=list(types))
    eng.load_params(params)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, 299, (3, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    out, step_logits = smp.generate(text, 0.0, return_logits=True)
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), out)
    greedy_agrees_with_full_forward(eng, out, ts)
    full = eng.logits(out)
    e = relfro(torch.stack(step_logits, 1), full[:, :S - 1])
    assert e < 2e-2, e
    smp.generate(text, 0.0)
    eager = [c.clone() for c in smp.kc]
    for P in (ts, ts + W + 3, S - 1):
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [None if c is None else torch.zeros_like(c) for c in smp.vc]
        logits = eng.prefill(out[:, :P].contiguous(), kc, vc).clone()
        for i in range(len(kc)):
            ei = relfro(kc[i][:, :P], eager[i][:, :P])
            assert ei < 2e-2, (P, i, ei)
        ep = relfro(logits[:, :eng.V], step_logits[P - 1])
        print(f"[gmlp] decode vs full {e:.2e}, prefill P={P} vs decoding {ep:.2e}")
        assert ep < 2e-2, ep
    done = smp.complete(text, out[:, ts:ts + W + 3].contiguous() - eng.image_offset, temperature=0)
    greedy_agrees_with_full_forward(eng, done, ts + W + 3)
    torch.manual_seed(0)
    guided = smp.complete(text[:2], out[:2, ts:ts + W + 3].contiguous() - eng.image_offset, samples_per_prompt=2,
                          guidance_scale=3.0, top_k=16, top_p=0.9)
    assert guided.shape == (4, S)
    gg = smp.generate_graphed(text[:2], temperature=0.0, guidance_scale=2.0)
    ge = smp.generate(text[:2], 0.0, guidance_scale=2.0)
    assert torch.equal(gg, ge)
