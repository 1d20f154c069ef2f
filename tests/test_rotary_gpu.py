"""Rotary position embeddings on the GPU: the four rope kernels bit for bit against the float32 torch evaluation of
their expression (include/dalle_b200.h) at the engine's shapes, their adjoint in float64 and their argument checks;
the rotary engine against oracle/dalle_rotary.py (loss, loss rows, every gradient, one Adam update), with each oracle
mutant failing the same bounds; reproducibility, in-process ranks and micro-batches, ZeRO-1; greedy decoding, graph
replay, the caches and the prefill; the model functions and generate_dalle.py; and a launch census of a rotary model
at dalle_example, whose rope classes are replayed here.  Without rotary_dim the engine launches exactly what it
launched before."""
import math
import os

import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu
BF16, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
TAG = "rotary"


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _table(n_pos, r, base=10000.0):
    from dalle_mtf_b200.dalle_engine import rope_table
    return rope_table(n_pos, r, base).to(DEV)


def torch_rope(qkv, table, H, dh, r, S=None, pos=None, inv=False):
    """The kernels' expression in float32 torch, one rounded operation at a time: a copy of qkv (bf16 [rows, 3*H*dh])
    with the q and k heads rotated, row t at position t mod S (or every row at pos)."""
    rows, h = qkv.shape[0], r // 2
    x = qkv.view(rows, 3, H, dh).float()
    p = torch.arange(rows, device=qkv.device) % S if pos is None else torch.full((rows,), pos, device=qkv.device)
    c, s = table[p, 0][:, None, None, :], table[p, 1][:, None, None, :]
    a, b = x[:, :2, :, :h], x[:, :2, :, h:r]
    ac, bs, bc, as_ = a * c, b * s, b * c, a * s
    ao, bo = (ac + bs, bc - as_) if inv else (ac - bs, bc + as_)
    out = qkv.clone().view(rows, 3, H, dh)
    out[:, :2, :, :h] = ao.to(BF16)
    out[:, :2, :, h:r] = bo.to(BF16)
    return out.view(rows, 3 * H * dh)


def _qkv(rows, H, dh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(rows, 3 * H * dh, generator=g, device=DEV) * 2).to(BF16)


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------ kernels
# (name, rows, S, H, dh, r): dalle_example (T = 32 x 1280), dh 64 with r = 2, the 12B width on one slab of rows, and
# row counts that are not a multiple of S
KERNEL_SHAPES = [("dalle_example", 40960, 1280, 4, 128, 128), ("dalle_example", 40960, 1280, 4, 128, 32),
                 ("dalle_coco", 2560, 1280, 16, 64, 2), ("12B", 2560, 1280, 32, 128, 128),
                 ("12B", 2560, 1280, 32, 128, 24), ("partial", 1000, 384, 4, 128, 64), ("partial", 777, 90, 2, 64, 6)]


@pytest.mark.parametrize("name,rows,S,H,dh,r", KERNEL_SHAPES)
def test_rope_fwd_and_bwd_are_the_float32_expression_bit_for_bit(ops, name, rows, S, H, dh, r):
    table = _table(S, r)
    x = _qkv(rows, H, dh, rows + r)
    for inv, fn in ((False, ops.rope_fwd), (True, ops.rope_bwd)):
        y = x.clone()
        fn(y, table, S, H, dh, r)
        want = torch_rope(x, table, H, dh, r, S=S, inv=inv)
        torch.cuda.synchronize()
        assert _bits_equal(y, want), (name, inv)
        v3 = y.view(rows, 3, H, dh)
        x3 = x.view(rows, 3, H, dh)
        assert _bits_equal(v3[:, 2], x3[:, 2]) and _bits_equal(v3[:, :2, :, r:], x3[:, :2, :, r:])
        assert not _bits_equal(v3[:, :2, :, :r], x3[:, :2, :, :r])
    print(f"[{TAG}] rope_fwd / rope_bwd {name} rows {rows} S {S} H {H} dh {dh} r {r}: bit for bit")


@pytest.mark.parametrize("r", [128, 32, 2])
def test_rope_bwd_is_the_adjoint_of_rope_fwd_in_float64(ops, r):
    """<R x, y> = <x, R^T y> up to the bf16 rounding of the two outputs; the forward rotation used as its own
    "transpose" misses by far more."""
    rows, S, H, dh = 1280 * 2, 1280, 4, 128
    table = _table(S, r)
    x, y = _qkv(rows, H, dh, 1), _qkv(rows, H, dh, 2)
    rx, rty, ry = x.clone(), y.clone(), y.clone()
    ops.rope_fwd(rx, table, S, H, dh, r)
    ops.rope_bwd(rty, table, S, H, dh, r)
    ops.rope_fwd(ry, table, S, H, dh, r)
    torch.cuda.synchronize()
    d = lambda a, b: (a.double() * b.double()).sum().item()          # noqa: E731
    lhs, rhs, wrong = d(rx, y), d(x, rty), d(x, ry)
    tol = 2.0 ** -7 * (x.double().abs() * y.double().abs()).sum().item() / math.sqrt(x.numel())
    print(f"[{TAG}] adjoint r {r}: |<Rx,y> - <x,R^T y>| {abs(lhs - rhs):.3e} (tol {tol:.3e}), against R y "
          f"{abs(lhs - wrong):.3e}")
    assert abs(lhs - rhs) <= tol
    assert abs(lhs - wrong) > 10 * tol


@pytest.mark.parametrize("rows,TL,S,H,dh,r", [(3, 256, 1280, 4, 128, 128), (6, 256, 1280, 4, 128, 32),
                                              (4, 24, 88, 2, 64, 2), (2, 128, 1152, 32, 128, 64)])
def test_decode_variants_at_the_sequence_boundaries(ops, rows, TL, S, H, dh, r):
    """rope_decode against the float32 expression at positions 0, TL - 1, TL and S - 1; rope_decode_dev equals it bit
    for bit, eagerly and replayed from a captured graph."""
    table = _table(S, r)
    x = _qkv(rows, H, dh, S + r)
    pos_dev = torch.zeros(1, dtype=I32, device=DEV)
    buf = x.clone()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.rope_decode_dev(buf, table, pos_dev, H, dh, r)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        ops.rope_decode_dev(buf, table, pos_dev, H, dh, r)
    for pos in (0, TL - 1, TL, S - 1):
        a, b = x.clone(), x.clone()
        ops.rope_decode(a, table, pos, H, dh, r)
        pos_dev.fill_(pos)
        ops.rope_decode_dev(b, table, pos_dev, H, dh, r)
        buf.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        want = torch_rope(x, table, H, dh, r, pos=pos)
        assert _bits_equal(a, want) and _bits_equal(b, a) and _bits_equal(buf, a), pos
        if pos == 0:
            assert _bits_equal(a, x)          # position 0: cos 1, sin 0
    # a device position outside [0, S) leaves the rows as they are
    pos_dev.fill_(S)
    b = x.clone()
    ops.rope_decode_dev(b, table, pos_dev, H, dh, r)
    torch.cuda.synchronize()
    assert _bits_equal(b, x)


def test_entry_points_refuse_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    H, dh, S, r = 2, 128, 64, 32
    x = _qkv(8, H, dh, 0)
    t = _table(S, r)
    pos = torch.zeros(1, dtype=I32, device=DEV)
    s, px, pt = L.stream_ptr(), x.data_ptr(), t.data_ptr()
    E_INV, E_ALIGN = -1, -2
    for fn in (lib.db200_rope_fwd, lib.db200_rope_bwd):
        assert fn(s, None, pt, 8, S, H, dh, r) == E_INV
        assert fn(s, px, None, 8, S, H, dh, r) == E_INV
        for bad in ((0, S, H, dh, r), (8, 0, H, dh, r), (8, S, 0, dh, r), (8, S, H, 0, r), (8, S, H, dh, 0),
                    (8, S, H, dh, 3), (8, S, H, dh, -2), (8, S, H, dh, 130)):
            assert fn(s, px, pt, *bad) == E_INV, bad
        assert fn(s, px + 2, pt, 8, S, H, dh, r) == E_ALIGN
        assert fn(s, px, pt + 4, 8, S, H, dh, r) == E_ALIGN
    assert lib.db200_rope_decode(s, px, pt, 8, S, H, dh, r, S) == E_INV
    assert lib.db200_rope_decode(s, px, pt, 8, S, H, dh, r, -1) == E_INV
    assert lib.db200_rope_decode(s, None, pt, 8, S, H, dh, r, 0) == E_INV
    assert lib.db200_rope_decode(s, px, pt, 8, S, H, dh, 5, 0) == E_INV
    assert lib.db200_rope_decode_dev(s, px, pt, 8, S, H, dh, r, None) == E_INV
    assert lib.db200_rope_decode_dev(s, px, pt, 8, S, H, dh, 0, pos.data_ptr()) == E_INV
    assert lib.db200_rope_decode_dev(s, px + 2, pt, 8, S, H, dh, r, pos.data_ptr()) == E_ALIGN
    torch.cuda.synchronize()
    assert _bits_equal(x, _qkv(8, H, dh, 0))                  # nothing ran
    # the Python wrappers check shapes and dtypes first
    for call in (lambda: ops.rope_fwd(x[:, :100].contiguous(), t, S, H, dh, r),
                 lambda: ops.rope_fwd(x.float(), t, S, H, dh, r),
                 lambda: ops.rope_fwd(x, t, S + 1, H, dh, r),
                 lambda: ops.rope_bwd(x, t[:, :, :8].contiguous(), S, H, dh, r),
                 lambda: ops.rope_decode(x, t, S, H, dh, r),
                 lambda: ops.rope_decode_dev(x, t, pos.long(), H, dh, r)):
        with pytest.raises(L.DB200Error):
            call()


# ------------------------------------------------------------------------------------------------ engine vs oracle
MIXED = ["global", "local", "axial_row", "axial_col", "conv"]


def _rotary_vs_oracle(types, rotary, B=3, seed=1, recompute=False, rates=None, row_col=False, adam=False,
                      mutants=()):
    """One rotary engine step (forward, backward 1 / T) against oracle/dalle_rotary.py in fp32 (the bounds) and with
    the reference's bf16 policy (the gradient scale): loss within 1e-3, loss rows within 5e-3, every gradient within
    1.25 x the bf16 oracle's error + 1e-2 (test_logits_mask_gpu.py's bounds); adam: one optimiser step against
    oracle/optim.py.  Each mutant's fp32 oracle must violate at least one of the same bounds."""
    import conv_oracle as OC
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_input as I
    from oracle import dalle_rotary as OR
    from test_parity_baseline_gpu import _randomise_small_params
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    d, nl, H, tv, iv, ts, isl = 256, len(types), 2, 300, 64, 24, 64
    cfg = OC.ConvConfig(d, nl, H, tv, iv, ts, isl, attention_types=tuple(types), local_attention_radius=8,
                        conv_attention_kernel=3)
    inp = I.InputConfig("row_col" if row_col else "absolute", False, None)
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    tokens = I.assemble(text, torch.randint(0, iv, (B, isl), generator=g), cfg, inp)
    step = 3 if rates else None
    dropout = ((rates,) * 3, seed, step, 0) if rates else None

    def oracle(bf16, mutate=None):
        base = lambda p, t, c, dr, bf16=False, quirks=None: OR.forward(  # noqa: E731
            p, t, c, dr, bf16=bf16, quirks=quirks, layers=OC, rotary=rotary, rotary_mutate=mutate)
        return I.loss_and_grads(params, tokens, cfg, inp, dropout, bf16, base=base)

    loss32, rows32, _, g32 = oracle(False)
    _, _, _, g16 = oracle(True)
    eng = DalleEngine(d, nl, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=types,
                      local_attention_radius=8, conv_attention_kernel=3, dropout=(rates or 0.0,) * 3,
                      dropout_seed=seed, image_position_embedding=inp.image_position_embedding,
                      rotary_dim=rotary[0], rotary_base=rotary[1])
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
    print(f"[{TAG}] engine types {types} rotary {rotary} recompute {recompute} rates {rates} row_col {row_col}: loss "
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


@pytest.mark.parametrize("types,rotary", [(["global", "global"], (128, 10000.0)), (MIXED, (32, 10000.0))],
                         ids=["global", "mixed"])
def test_engine_matches_the_oracle_and_not_its_mutants(types, rotary):
    _rotary_vs_oracle(types, rotary, adam=True, mutants=("neg_theta", "interleaved", "shift"))


@pytest.mark.parametrize("variant", [dict(recompute=True), dict(rates=0.1), dict(row_col=True)],
                         ids=["recompute", "dropout", "row_col"])
@pytest.mark.parametrize("types,rotary", [(["global", "global"], (128, 10000.0)), (MIXED, (64, 500.0))],
                         ids=["global", "mixed"])
def test_engine_variants_match_the_oracle(types, rotary, variant):
    _rotary_vs_oracle(types, rotary, seed=2, **variant)


# ------------------------------------------------------------------------------------------------ invariances
def _small(seed=0):
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


def test_rotary_steps_are_bit_identical_and_micro_batches_match():
    cfg, params, tok = _small(3)
    eng = _engine(cfg, rotary_dim=64, attention_types=["global", "axial_col"])
    eng.load_params(params)
    a, b = _step(eng, tok, 1.0 / tok.numel()), _step(eng, tok, 1.0 / tok.numel())
    assert torch.equal(a, b)
    c = _step(eng, tok, 1.0 / tok.numel(), split=2)
    n = eng.n_params_padded
    assert relfro(c[:n], a[:n]) < 1e-5


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion for the plain step (bit for bit), with rotary and every feature."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, rotary_dim=64)
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


def test_zero1_rotary_step_equals_the_replicated_step_bitwise():
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    kw = dict(rotary_dim=32, rotary_base=500.0)
    grp = Loopback(2)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **kw) for r in range(2)]
    twin = _engine(cfg, **kw)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    _twin_from(twin, twin.master[:n].clone(), ranks[0])
    g_ref = _step(twin, tok)
    for r, e in enumerate(ranks):
        assert_same_bits(_step(e, tok), g_ref, f"ZeRO-1 rank {r} rotary gradients")
    twin.optimizer_step(1e-3)
    for e in ranks:
        e.optimizer_step(1e-3)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} parameters after the step")


# ------------------------------------------------------------------------------------------------ generation
@pytest.mark.parametrize("types", [None, ["global", "axial_col"]], ids=["global", "axial_col"])
def test_greedy_generation_follows_the_full_forward_and_the_caches_hold_rotated_keys(types):
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward, sharp_engine
    ts, S = 16, 80
    eng, _, _ = sharp_engine(256, 2, 2, 300, 64, ts, 64, rotary_dim=64, attention_types=types)
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
    # layer 0's cache holds the keys of the teacher-forced forward, rotated, bit for bit; the prefill's caches too
    eng.logits(out)
    qkv = eng._bufs["layers"][0]["qkv"].view(3, S, 3, eng.H, eng.dh)
    assert _bits_equal(smp.kc[0][:, :S - 1], qkv[:, :S - 1, 1]) and _bits_equal(smp.vc[0][:, :S - 1], qkv[:, :S - 1, 2])
    for P in (ts, ts + 9):
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [torch.zeros_like(c) for c in smp.vc]
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


def test_model_fn_checkpoint_resumes_bit_exactly_and_dalle_takes_the_key(tmp_path):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    img, cap = _batch()
    ROT = {"rotary_dim": 64, "rotary_base": 1000.0}
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    rot = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **ROT))
    assert rot.engine.rotary == (64, 1000.0) and plain.engine.rotary is None
    rot.train_op(img, cap)
    st = rot.state_fn()
    assert {k: tuple(v.shape) for k, v in st.items() if k != "global_step"} == \
        {k: tuple(v.shape) for k, v in plain.state_fn().items() if k != "global_step"}
    a = rot.train_op(img, cap).clone()
    sa = [t.clone() for t in (rot.engine.master, rot.engine.adam_m, rot.engine.adam_v)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **ROT))
    resumed.load_fn(st)
    b = resumed.train_op(img, cap)
    assert torch.equal(a, b)
    for x, y in zip(sa, (resumed.engine.master, resumed.engine.adam_m, resumed.engine.adam_v)):
        assert torch.equal(x, y)
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=88, n_layers=1, n_heads=2,
              mode="eval", params={"rotary_dim": 32})
    assert m.engine.rotary == (32, 10000.0)
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 88), generator=g)], 1)
    loss, loss_batch = m.forward({"tokens": tokens})
    assert math.isfinite(loss.item()) and loss_batch.shape == (2, 128)


def test_generate_cli_runs_on_a_tiny_rotary_model(tmp_path):
    """generate_dalle.py end to end on a tiny rotary model trained one step and checkpointed."""
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import save_checkpoint
    img, cap = _batch()
    p = _tiny_params(tmp_path, rotary_dim=32)
    spec = dalle_model_fn(img, cap, "train", p)
    spec.train_op(img, cap)
    vae = spec.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, spec.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "rotary.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "rotary.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, spec.engine.S) and len(list(out.glob("*.png"))) == 2
    io = spec.engine.image_offset
    assert ((toks[:, 12:] >= io) & (toks[:, 12:] < io + 64)).all()


# ------------------------------------------------------------------------------------------------ launches
def test_rotary_off_launches_what_it_launched_before(monkeypatch):
    """Without rotary_dim (absent or None) forward, backward and the optimiser step call the same ops in the same
    order with the same launch count; with it, exactly 2 rope_fwd and 2 rope_bwd calls (one per layer) are added."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    cfg, params, tok = _small(10)
    calls = []
    names = [n for n, f in vars(O).items() if callable(f) and not n.startswith("_") and getattr(f, "__module__", "")
             == O.__name__]
    for n in names:
        f = getattr(O, n)
        monkeypatch.setattr(O, n, (lambda n, f: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(n, f))
    seqs, counts = [], []
    for kw in ({}, {"rotary_dim": None}, {"rotary_dim": 64}):
        eng = _engine(cfg, **kw)
        eng.load_params(params)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        counts.append(L.launch_count() - n0)
        seqs.append(list(calls))
    assert seqs[0] == seqs[1] and counts[0] == counts[1]
    assert "rope_fwd" not in seqs[0] and "rope_bwd" not in seqs[0]
    assert [c for c in seqs[2] if not c.startswith("rope_")] == seqs[0]
    assert seqs[2].count("rope_fwd") == 2 and seqs[2].count("rope_bwd") == 2 and counts[2] == counts[0] + 4


def test_launch_census_of_a_rotary_model_adds_only_the_rope_classes(ops, monkeypatch):
    """dalle_example_b200 with and without rotary_dim recorded by test_dalle_config_launches_gpu.py's recorder
    (train, eval, eager and graphed decoding, prefill with guidance): the rotary model launches the plain model's
    classes plus rope_fwd, rope_bwd, rope_decode and rope_decode_dev classes and nothing else; each rope class is
    replayed here at its recorded shape against the float32 expression, bit for bit."""
    import launch_census as LC
    import test_dalle_config_launches_gpu as CL
    import test_dalle_kernels_gpu as DK
    base = DK._config("dalle_example_b200")
    recorded = {}
    for name, extra in (("plain", {}), ("rotary", {"rotary_dim": 32})):
        monkeypatch.setattr(DK, "_config", lambda c, extra=extra: dict(base, **extra))
        recorded[name] = set(CL.record_config("dalle_example_b200")[0])
    added = recorded["rotary"] - recorded["plain"]
    assert recorded["plain"] <= recorded["rotary"]
    entries = {c[0] for c in added}
    assert entries == {"rope_fwd", "rope_bwd", "rope_decode", "rope_decode_dev"}, entries
    for c in sorted(added, key=repr):
        f = LC.fields(c)
        (rows, width), _ = f.get("qkv") or f.get("dqkv")
        (n_pos, _, h), _ = f["table"]
        H, dh, r = f["H"], f["dh"], f["r"]
        assert width == 3 * H * dh and r == 2 * h == 32
        table = _table(n_pos, r)
        x = _qkv(rows, H, dh, rows)
        y = x.clone()
        if c[0] in ("rope_fwd", "rope_bwd"):
            getattr(ops, c[0])(y, table, f["S"], H, dh, r)
            want = torch_rope(x, table, H, dh, r, S=f["S"], inv=c[0] == "rope_bwd")
        else:
            pos = n_pos - 1
            if c[0] == "rope_decode":
                ops.rope_decode(y, table, pos, H, dh, r)
            else:
                ops.rope_decode_dev(y, table, torch.full((1,), pos, dtype=I32, device=DEV), H, dh, r)
            want = torch_rope(x, table, H, dh, r, pos=pos)
        torch.cuda.synchronize()
        assert _bits_equal(y, want), c
        print(f"[{TAG}] census class {c[0]} rows {rows} S {f.get('S')} H {H} dh {dh} r {r}: replayed bit for bit")
