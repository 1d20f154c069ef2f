"""DALLE-pytorch's rotary embedding (rotary_emb) on the GPU: the four rope_emb kernels bit for bit against the float32
torch evaluation of their expression (include/dalle_b200.h) at the engine's widths, their adjoint in float64 and their
argument checks; the engine against oracle/dalle_rotary_emb.py (loss, loss rows, every gradient, one Adam update),
with each oracle mutant failing the same bounds; reproducibility, in-process micro-batches, ZeRO-1; greedy decoding,
graph replay, the k and v caches and the prefill; checkpoints through the model functions and generate_dalle.py.
Without the key the engine launches exactly what it launched before."""
import math
import os

import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
TAG = "rotary_emb"


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _table(TL, W, dh):
    from dalle_mtf_b200.dalle_engine import rotary_emb_table
    return rotary_emb_table(TL, W, dh).to(DEV)


def torch_rope_emb(qkv, table, H, dh, S=None, pos=None, inv=False):
    """The kernels' expression in float32 torch, one rounded operation at a time: a copy of qkv (bf16 [rows, 3*H*dh])
    with the interleaved pairs of every q, k and v head rotated, row t at position t mod S (or every row at pos)."""
    rows, n = qkv.shape[0], table.shape[2]
    x = qkv.view(rows, 3, H, dh).float()
    p = torch.arange(rows, device=qkv.device) % S if pos is None else torch.full((rows,), pos, device=qkv.device)
    c, s = table[p, 0][:, None, None, :], table[p, 1][:, None, None, :]
    a, b = x[..., 0:2 * n:2], x[..., 1:2 * n:2]
    ac, bs, bc, as_ = a * c, b * s, b * c, a * s
    ao, bo = (ac + bs, bc - as_) if inv else (ac - bs, bc + as_)
    out = qkv.clone().view(rows, 3, H, dh)
    out[..., 0:2 * n:2] = ao.to(BF16)
    out[..., 1:2 * n:2] = bo.to(BF16)
    return out.view(rows, 3 * H * dh)


def _qkv(rows, H, dh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(rows, 3 * H * dh, generator=g, device=DEV) * 2).to(BF16)


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------ kernels
# (name, rows, TL, W, H, dh): dalle_example (B 32, S 1280, d 512), the dalle_coco width (d 1024, 16 heads of 64), the
# 12B width (d 4096, 32 heads of 128) on slabs of rows, and a row count that is not a multiple of S
KERNEL_SHAPES = [("dalle_example", 40960, 256, 32, 4, 128), ("dalle_coco", 2560, 256, 32, 16, 64),
                 ("12B", 2560, 128, 32, 32, 128), ("partial", 1000, 24, 8, 2, 64)]


@pytest.mark.parametrize("name,rows,TL,W,H,dh", KERNEL_SHAPES)
def test_rope_emb_fwd_and_bwd_are_the_float32_expression_bit_for_bit(ops, name, rows, TL, W, H, dh):
    table = _table(TL, W, dh)
    S, n = TL + W * W, table.shape[2]
    x = _qkv(rows, H, dh, rows + dh)
    for inv, fn in ((False, ops.rope_emb_fwd), (True, ops.rope_emb_bwd)):
        y = x.clone()
        fn(y, table, S, H, dh)
        want = torch_rope_emb(x, table, H, dh, S=S, inv=inv)
        torch.cuda.synchronize()
        assert _bits_equal(y, want), (name, inv)
        v3, x3 = y.view(rows, 3, H, dh), x.view(rows, 3, H, dh)
        assert _bits_equal(v3[..., 2 * n:], x3[..., 2 * n:])
        for part in range(3):                                   # q, k and v are all rotated
            assert not _bits_equal(v3[:, part, :, :2 * n], x3[:, part, :, :2 * n])
    print(f"[{TAG}] rope_emb_fwd / _bwd {name} rows {rows} S {S} H {H} dh {dh} pairs {n}: bit for bit")


@pytest.mark.parametrize("dh", [128, 64])
def test_rope_emb_bwd_is_the_adjoint_of_rope_emb_fwd_in_float64(ops, dh):
    rows, TL, W, H = 1280 * 2, 256, 32, 512 // dh
    S = TL + W * W
    table = _table(TL, W, dh)
    x, y = _qkv(rows, H, dh, 1), _qkv(rows, H, dh, 2)
    rx, rty, ry = x.clone(), y.clone(), y.clone()
    ops.rope_emb_fwd(rx, table, S, H, dh)
    ops.rope_emb_bwd(rty, table, S, H, dh)
    ops.rope_emb_fwd(ry, table, S, H, dh)
    torch.cuda.synchronize()
    d = lambda a, b: (a.double() * b.double()).sum().item()          # noqa: E731
    lhs, rhs, wrong = d(rx, y), d(x, rty), d(x, ry)
    tol = 2.0 ** -7 * (x.double().abs() * y.double().abs()).sum().item() / math.sqrt(x.numel())
    print(f"[{TAG}] adjoint dh {dh}: |<Rx,y> - <x,R^T y>| {abs(lhs - rhs):.3e} (tol {tol:.3e}), against R y "
          f"{abs(lhs - wrong):.3e}")
    assert abs(lhs - rhs) <= tol
    assert abs(lhs - wrong) > 10 * tol


@pytest.mark.parametrize("rows,TL,W,H,dh", [(32, 256, 32, 4, 128), (32, 256, 32, 16, 64), (32, 128, 32, 32, 128),
                                            (3, 24, 4, 2, 64)])
def test_decode_variants_at_the_sequence_boundaries(ops, rows, TL, W, H, dh):
    """rope_emb_decode against the float32 expression at positions 0, TL - 1, TL, the row ends and S - 1;
    rope_emb_decode_dev equals it bit for bit, eagerly and replayed from a captured graph."""
    S = TL + W * W
    table = _table(TL, W, dh)
    x = _qkv(rows, H, dh, S + dh)
    pos_dev = torch.zeros(1, dtype=I32, device=DEV)
    buf = x.clone()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.rope_emb_decode_dev(buf, table, pos_dev, H, dh)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        ops.rope_emb_decode_dev(buf, table, pos_dev, H, dh)
    for pos in (0, TL - 1, TL, TL + W - 1, TL + W, S - W, S - 1):
        a, b = x.clone(), x.clone()
        ops.rope_emb_decode(a, table, pos, H, dh)
        pos_dev.fill_(pos)
        ops.rope_emb_decode_dev(b, table, pos_dev, H, dh)
        buf.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        want = torch_rope_emb(x, table, H, dh, pos=pos)
        assert _bits_equal(a, want) and _bits_equal(b, a) and _bits_equal(buf, a), pos
    pos_dev.fill_(S)                       # a device position outside [0, S) leaves the rows as they are
    b = x.clone()
    ops.rope_emb_decode_dev(b, table, pos_dev, H, dh)
    torch.cuda.synchronize()
    assert _bits_equal(b, x)


def test_entry_points_refuse_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    H, dh, S, n = 2, 128, 32, 63
    x = _qkv(8, H, dh, 0)
    t = _table(16, 4, dh)
    pos = torch.zeros(1, dtype=I32, device=DEV)
    s, px, pt = L.stream_ptr(), x.data_ptr(), t.data_ptr()
    E_INV, E_ALIGN = -1, -2
    for fn in (lib.db200_rope_emb_fwd, lib.db200_rope_emb_bwd):
        assert fn(s, None, pt, 8, S, H, dh, n) == E_INV
        assert fn(s, px, None, 8, S, H, dh, n) == E_INV
        for bad in ((0, S, H, dh, n), (8, 0, H, dh, n), (8, S, 0, dh, n), (8, S, H, 0, n), (8, S, H, dh, 0),
                    (8, S, H, dh, 65), (8, S, H, 127, n), (8, S, H, dh, -1)):
            assert fn(s, px, pt, *bad) == E_INV, bad
        assert fn(s, px + 2, pt, 8, S, H, dh, n) == E_ALIGN
        assert fn(s, px, pt + 2, 8, S, H, dh, n) == E_ALIGN
    assert lib.db200_rope_emb_decode(s, px, pt, 8, S, H, dh, n, S) == E_INV
    assert lib.db200_rope_emb_decode(s, px, pt, 8, S, H, dh, n, -1) == E_INV
    assert lib.db200_rope_emb_decode(s, None, pt, 8, S, H, dh, n, 0) == E_INV
    assert lib.db200_rope_emb_decode_dev(s, px, pt, 8, S, H, dh, n, None) == E_INV
    assert lib.db200_rope_emb_decode_dev(s, px, pt, 8, S, H, dh, 0, pos.data_ptr()) == E_INV
    assert lib.db200_rope_emb_decode_dev(s, px + 2, pt, 8, S, H, dh, n, pos.data_ptr()) == E_ALIGN
    torch.cuda.synchronize()
    assert _bits_equal(x, _qkv(8, H, dh, 0))                  # nothing ran
    for call in (lambda: ops.rope_emb_fwd(x[:, :100].contiguous(), t, S, H, dh),
                 lambda: ops.rope_emb_fwd(x.float(), t, S, H, dh),
                 lambda: ops.rope_emb_fwd(x, t, S + 1, H, dh),
                 lambda: ops.rope_emb_bwd(x, torch.zeros(S, 2, 65, device=DEV), S, H, dh),
                 lambda: ops.rope_emb_decode(x, t, S, H, dh),
                 lambda: ops.rope_emb_decode_dev(x, t, pos.long(), H, dh)):
        with pytest.raises(L.DB200Error):
            call()


# ------------------------------------------------------------------------------------------------ engine vs oracle
def _vs_oracle(types, B=3, seed=1, recompute=False, rates=None, adam=False, mutants=(), ts=24, shift=False,
               per_pos=False):
    """One rotary_emb engine step (forward, backward 1 / T) against oracle/dalle_rotary_emb.py in fp32 (the bounds)
    and with the reference's bf16 policy (the gradient scale): loss within 1e-3, loss rows within 5e-3, every gradient
    within 1.25 x the bf16 oracle's error + 1e-2 (tests/test_rotary_gpu.py's bounds); adam: one optimiser step against
    oracle/optim.py.  Each mutant's fp32 oracle must violate at least one of the same bounds.  types may hold
    "block_sparse" (the engine's layouts, tests/block_sparse_oracle.py's masks) and "mlp" (gMLP layers, unrotated);
    shift: the token shift; per_pos: per-position padding tokens (half of each caption padded)."""
    import block_sparse_oracle as OB
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_gmlp as OGM
    from oracle import dalle_input as I
    from oracle import dalle_rotary_emb as ORE
    from test_parity_baseline_gpu import _randomise_small_params
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    d, nl, H, tv, iv, isl = 256, len(types), 2, 300, 64, 64
    eng = DalleEngine(d, nl, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=types,
                      local_attention_radius=8, conv_attention_kernel=3, dropout=(rates or 0.0,) * 3,
                      dropout_seed=seed, per_position_padding=per_pos, shift_tokens=shift, rotary_emb=True)
    layouts = tuple(None if m is None else m.layout for m in eng.block_sparse)
    cfg = OB.BlockSparseConfig(d, nl, H, tv, iv, ts, isl, attention_types=tuple(types), local_attention_radius=8,
                               conv_attention_kernel=3, sparse_block_size=16, block_sparse_layouts=layouts)
    inp = I.InputConfig("absolute", per_pos, tv - 1 if per_pos else None)
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    if "mlp" in types:
        params = OGM.init_params(params, cfg, seed + 7)
    del params["positional_embedding/wpe"]
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    if per_pos:
        text[:, ts // 2:] = tv - 1
    tokens = I.assemble(text, torch.randint(0, iv, (B, isl), generator=g), cfg, inp)
    step = 3 if rates else None
    dropout = ((rates,) * 3, seed, step, 0) if rates else None

    def oracle(bf16, mutate=None):
        base = lambda p, t, c, dr, bf16=False, quirks=None: ORE.forward(  # noqa: E731
            p, t, c, dr, bf16=bf16, quirks=quirks, layers=OB, rotary_mutate=mutate, shift_tokens=shift)
        return I.loss_and_grads(params, tokens, cfg, inp, dropout, bf16, base=base)

    loss32, rows32, _, g32 = oracle(False)
    _, _, _, g16 = oracle(True)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=step)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    rows = eng._bufs["loss_rows"].view(B, -1).clone()
    grads = eng.export_params(eng.grads)
    assert set(grads) == set(params)

    def violations(l32, r32, gg32):
        bad, worst = [], [0.0, None]

        def bound(name, err, limit):
            if err > limit:
                bad.append((name, err, limit))
            if err / limit > worst[0]:
                worst[:] = [err / limit, name]
        bound("loss", abs(loss - l32.item()), 1e-3 * abs(l32.item()))
        bound("loss_rows", relfro(rows, r32), 5e-3)
        for k in gg32:
            if g32[k].any():
                bound("grad " + k, relfro(grads[k], gg32[k]), 1.25 * relfro(g16[k], g32[k]) + 1e-2)
        return bad, worst

    bad, worst = violations(loss32, rows32, g32)
    print(f"[{TAG}] engine types {types} recompute {recompute} rates {rates} shift {shift} per_pos {per_pos}: loss "
          f"{loss:.6f} oracle {loss32.item():.6f}, worst err/bound {worst[0]:.4f} ({worst[1]}), violations {bad}")
    assert not bad
    for m in mutants:
        ml, mr, _, mg = oracle(False, m)
        mbad, _ = violations(ml, mr, mg)
        print(f"[{TAG}]   mutant {m}: {len(mbad)} violated bounds, e.g. {mbad[:2]}")
        assert mbad, m
    if adam:
        from oracle import optim as OO
        hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
        zeros = {k: torch.zeros_like(v) for k, v in params.items()}
        newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
        eng.optimizer_step(lr)
        torch.cuda.synchronize()
        assert abs(eng.gnorm_sq.sqrt().item() - gn.item()) <= 1e-4 * gn.item()
        after = eng.export_params()
        for k in params:
            if (newp[k] - params[k]).norm() > 0:
                assert relfro(after[k] - params[k], newp[k] - params[k]) <= 1e-3, k


MUTANTS = ("no_v", "rotate_half", "swap_axes", "image_text_pos")
# the schedule of the issue: every attention-layer kind that reads the rotated q|k|v, and a gMLP layer that does not;
# S = 64 + 64 is a multiple of 64, as gMLP layers need
SCHEDULE = ["axial_row", "conv", "block_sparse", "mlp", "global"]


def test_engine_matches_the_oracle_and_not_its_mutants():
    _vs_oracle(["global", "global"], adam=True, mutants=MUTANTS)


@pytest.mark.parametrize("variant", [dict(recompute=True), dict(rates=0.1),
                                     dict(types=SCHEDULE, ts=64, adam=True, mutants=MUTANTS),
                                     dict(shift=True, per_pos=True, mutants=MUTANTS)],
                         ids=["recompute", "dropout", "schedule", "shift_per_pos"])
def test_engine_variants_match_the_oracle(variant):
    variant = dict(variant)
    _vs_oracle(variant.pop("types", ["global", "global"]), seed=2, **variant)


# ------------------------------------------------------------------------------------------------ invariances
def _small(seed=0):
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = O.init_params(cfg, seed)
    del params["positional_embedding/wpe"]
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


def test_steps_are_bit_identical_and_micro_batches_match():
    cfg, params, tok = _small(3)
    eng = _engine(cfg, rotary_emb=True, attention_types=["global", "axial_col"])
    eng.load_params(params)
    a, b = _step(eng, tok, 1.0 / tok.numel()), _step(eng, tok, 1.0 / tok.numel())
    assert torch.equal(a, b)
    c = _step(eng, tok, 1.0 / tok.numel(), split=2)
    n = eng.n_params_padded
    assert relfro(c[:n], a[:n]) < 1e-5


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion for the plain step (bit for bit), with rotary_emb and every feature:
    the layout without wpe moves the first gradient bucket and the decay segments, which its coverage check reads."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, rotary_emb=True)
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


def test_zero1_step_equals_the_replicated_step_bitwise():
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    grp = Loopback(2)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), rotary_emb=True) for r in range(2)]
    twin = _engine(cfg, rotary_emb=True)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    _twin_from(twin, twin.master[:n].clone(), ranks[0])
    g_ref = _step(twin, tok)
    for r, e in enumerate(ranks):
        assert_same_bits(_step(e, tok), g_ref, f"ZeRO-1 rank {r} rotary_emb gradients")
    twin.optimizer_step(1e-3)
    for e in ranks:
        e.optimizer_step(1e-3)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} parameters after the step")


def test_no_wpe_in_the_parameters_the_count_or_the_checkpoint():
    cfg, params, _ = _small(5)
    plain = _engine(cfg)
    rot = _engine(cfg, rotary_emb=True)
    S, d = plain.S, plain.d
    assert plain.n_params() - rot.n_params() == S * d
    assert plain.n_params_padded - rot.n_params_padded == S * d
    assert "wpe" not in rot.layout.entries and rot.embed_names == ("wte",)
    rot.init_params(seed=1)
    names = set(rot.export_params())
    assert "positional_embedding/wpe" not in names and names == set(params)
    assert not rot.pos_table.any()
    assert rot._decay_segments()[0][0] == 0


def test_checkpoints_of_the_other_position_kind_are_refused():
    from dalle_mtf_b200 import lib as L
    cfg, params, _ = _small(6)
    rot, plain = _engine(cfg, rotary_emb=True), _engine(cfg)
    with_wpe = dict(params, **{"positional_embedding/wpe": torch.zeros(plain.S, plain.d)})
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe"):
        rot.load_params(with_wpe)
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe: missing"):
        plain.load_params(params)
    rot.load_params(params)
    plain.load_params(with_wpe)


# ------------------------------------------------------------------------------------------------ generation
def _sharp_engine(d, L, H, tv, iv, ts, isl, **kw):
    """test_prefill_gpu.sharp_engine's oracle-initialised, sharpened weights (clear arg-maxima) without wpe, in a
    rotary_emb engine."""
    import conv_oracle as OC
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_gmlp as OGM
    types = kw.get("attention_types")
    cfg = OC.ConvConfig(d, L, H, tv, iv, ts, isl, attention_types=None if types is None else tuple(types))
    params = OGM.init_params(O.init_params(cfg, 3), cfg)       # gMLP layers: the engine's initialisation
    del params["positional_embedding/wpe"]
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, rotary_emb=True, **kw)
    eng.load_params(params)
    return eng


@pytest.mark.parametrize("types,ts", [(None, 16), (["global", "axial_col"], 16), (["block_sparse", "mlp"], 64)],
                         ids=["global", "axial_col", "block_sparse_mlp"])
def test_greedy_generation_follows_the_full_forward_and_the_caches_hold_rotated_k_and_v(types, ts):
    """Eager and graphed decoding, the prefill and layer 0's caches; the last schedule has a block-sparse layer and a
    gMLP layer, which stays unrotated in the full forward, the prefill and both decoders."""
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward
    S = ts + 64
    eng = _sharp_engine(256, 2, 2, 300, 64, ts, 64, attention_types=types)
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
    # layer 0's caches hold the keys and values of the teacher-forced forward, rotated, bit for bit; the prefill's too
    eng.logits(out)
    qkv = eng._bufs["layers"][0]["qkv"].view(3, S, 3, eng.H, eng.dh)
    assert _bits_equal(smp.kc[0][:, :S - 1], qkv[:, :S - 1, 1]) and _bits_equal(smp.vc[0][:, :S - 1], qkv[:, :S - 1, 2])
    for P in (ts, ts + 9):
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [None if c is None else torch.zeros_like(c) for c in smp.vc]   # a gMLP layer has no v cache
        logits = eng.prefill(out[:, :P].contiguous(), kc, vc).clone()
        assert _bits_equal(kc[0][:, :P], smp.kc[0][:, :P]) and _bits_equal(vc[0][:, :P], smp.vc[0][:, :P])
        ep = relfro(logits[:, :eng.V], step_logits[P - 1])
        print(f"[{TAG}] types {types}: decode vs full {e:.2e}, prefill P={P} vs decoding {ep:.2e}")
        assert ep < 2e-2, ep
    done = smp.complete(text, out[:, ts:ts + 8].contiguous() - eng.image_offset, temperature=0)
    greedy_agrees_with_full_forward(eng, done, ts + 8)
    torch.manual_seed(0)
    guided = smp.complete(text[:2], out[:2, ts:ts + 8].contiguous() - eng.image_offset, samples_per_prompt=2,
                          guidance_scale=3.0, top_k=16)
    assert guided.shape == (4, S)
    assert ((guided[:, ts:] >= eng.image_offset) & (guided[:, ts:] < eng.image_offset + 64)).all()


# ------------------------------------------------------------------------------------------------ model functions
def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def test_model_fn_checkpoint_resumes_bit_exactly_and_refuses_the_other_kind(tmp_path):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    img, cap = _batch()
    ROT = {"rotary_emb": True}
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    rot = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **ROT))
    assert rot.engine.rotary_emb and not plain.engine.rotary_emb
    rot.train_op(img, cap)
    st = rot.state_fn()
    assert "positional_embedding/wpe" not in st and "positional_embedding/wpe" in plain.state_fn()
    a = rot.train_op(img, cap).clone()
    sa = [t.clone() for t in (rot.engine.master, rot.engine.adam_m, rot.engine.adam_v)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **ROT))
    resumed.load_fn(st)
    b = resumed.train_op(img, cap)
    assert torch.equal(a, b)
    for x, y in zip(sa, (resumed.engine.master, resumed.engine.adam_m, resumed.engine.adam_v)):
        assert torch.equal(x, y)
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe"):
        plain.load_fn(st)
    with pytest.raises(L.DB200Error, match="positional_embedding/wpe"):
        resumed.load_fn(plain.state_fn())
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=64, n_layers=1, n_heads=2,
              mode="eval", params=ROT)
    assert m.engine.rotary_emb
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 64), generator=g)], 1)
    loss, loss_batch = m.forward({"tokens": tokens})
    assert math.isfinite(loss.item()) and loss_batch.shape == (2, 104)


def test_generate_cli_runs_on_a_tiny_rotary_emb_model(tmp_path):
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import save_checkpoint
    img, cap = _batch()
    p = _tiny_params(tmp_path, rotary_emb=True)
    spec = dalle_model_fn(img, cap, "train", p)
    spec.train_op(img, cap)
    vae = spec.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, spec.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "rotary_emb.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "rotary_emb.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, spec.engine.S) and len(list(out.glob("*.png"))) == 2
    io = spec.engine.image_offset
    assert ((toks[:, 12:] >= io) & (toks[:, 12:] < io + 64)).all()


# ------------------------------------------------------------------------------------------------ launches
def test_rotary_emb_off_launches_what_it_launched_before(monkeypatch):
    """Without rotary_emb (absent, None or False) forward, backward and the optimiser step call the same ops in the
    same order; with it, exactly 2 rope_emb_fwd and 2 rope_emb_bwd calls (one per layer) are added."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    from oracle import dalle as OD
    cfg, params, tok = _small(10)
    full = dict(params, **{"positional_embedding/wpe": OD.init_params(cfg, 10)["positional_embedding/wpe"]})
    calls = []
    names = [n for n, f in vars(O).items() if callable(f) and not n.startswith("_") and getattr(f, "__module__", "")
             == O.__name__]
    for n in names:
        f = getattr(O, n)
        monkeypatch.setattr(O, n, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(n, f))
    seqs, counts = [], []
    for kw in ({}, {"rotary_emb": None}, {"rotary_emb": False}, {"rotary_emb": True}):
        eng = _engine(cfg, **kw)
        eng.load_params(params if kw.get("rotary_emb") else full)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        counts.append(L.launch_count() - n0)
        seqs.append(list(calls))
    assert seqs[0] == seqs[1] == seqs[2] and counts[0] == counts[1] == counts[2]
    assert "rope_emb_fwd" not in seqs[0] and "rope_emb_bwd" not in seqs[0]
    assert [c for c in seqs[3] if not c.startswith("rope_emb_")] == seqs[0]
    assert seqs[3].count("rope_emb_fwd") == 2 and seqs[3].count("rope_emb_bwd") == 2
