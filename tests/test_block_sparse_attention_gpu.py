"""GPU tests of block-sparse attention layers (dalle_mtf_b200/csrc/attn_fa.cu, SPARSE; decode.cu).

Query i sees key j <= i iff layout[i // b][j // b] (dalle_engine.block_sparse_layout).  The kernels are checked
against float64 with the bounds of the causal kernels (test_axial_attention_gpu.py's masked_reference with the block
mask, outputs starting as NaN) at the (H, dh) of dalle_example, dalle_coco and the 12B config, S = 1279, a caption
length that is not a multiple of b, b = 16, 32 and 64, and R = 0, the default and nb.  With R = nb the layout is the
causal triangle, and the block-sparse kernels must return the causal kernels' out, lse and dqkv bit for bit.  Then a
dominating key in an unset block, prompt prefills, the decode kernels (host and device position, bit for bit), an
engine with every layer type against tests/block_sparse_oracle.py, reproducible training, generation and
dalle_model_fn.  The module prints its wall time and peak device memory.
"""
import math
import time

import numpy as np
import pytest
import torch

import block_sparse_oracle as OB
import float64_bounds
from float64_bounds import DEV, nan_like
from test_axial_attention_gpu import ratios
from test_local_attention_gpu import RATES, _gen, _qkv, decode_reference, relfro

pytestmark = pytest.mark.gpu

F64, F32, BF16, I32 = torch.float64, torch.float32, torch.bfloat16, torch.int32
TAG = "block-sparse"


@pytest.fixture(scope="module", autouse=True)
def _module_cost():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[{TAG}] module wall time {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB on {torch.cuda.get_device_name()}")


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def layout(S, TL, b=16, w=4, R=None, seed=0, owner=0):
    from dalle_mtf_b200.dalle_engine import block_sparse_layout
    return block_sparse_layout(S, TL, b, w, S // b // 4 if R is None else R, seed, owner)


def visible(S, lay, b):
    return ~OB.block_sparse_hidden(S, lay, b).to(DEV)


def run_bs(ops, qkv, dout, bs, scale=1.0):
    B, S, _, H, dh = qkv.shape
    out, lse = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, scale, block_sparse=bs)
    dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out, dout, lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv, B, S, H, dh, scale,
                 block_sparse=bs)
    return out, lse, dqkv


def check(ops, name, qkv, dout, bs, S, chunk):
    """The kernels against float64 on chunks of `chunk` sequences (the float64 reference of a whole batch is large)."""
    out, lse, dqkv = run_bs(ops, qkv, dout, bs)
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    vis = visible(S, bs.layout, bs.block)
    worst = {}
    for b0 in range(0, qkv.shape[0], chunk):
        sl = slice(b0, b0 + chunk)
        for n, v in ratios(qkv[sl], dout[sl], out[sl], lse[sl], dqkv[sl], vis).items():
            worst[n] = max(worst.get(n, 0.0), v)
    for n, v in worst.items():
        float64_bounds.report(f"{name} {n}", v, TAG)


# (name, B sequences per GPU, H, dh): dalle_example, dalle_coco and the 12B config at S = 1280, TL = 256
SHAPES = [("dalle_example", 32, 4, 128), ("dalle_coco", 8, 16, 64), ("12B", 2, 64, 64)]


@pytest.mark.parametrize("name,B,H,dh", SHAPES)
def test_kernels_at_the_config_shapes_against_float64(ops, name, B, H, dh):
    S, TL = 1280, 256
    qkv, dout = _qkv(B, S, H, dh, _gen(B + H + dh))
    bs = ops.BlockSparse(layout(S, TL), 16, S)
    check(ops, f"{name} B={B} H={H} dh={dh} S={S} b=16 R=20", qkv, dout, bs, S, max(1, 8 // H))


# (S, TL, b, w, R): S not a multiple of 64, TL not a multiple of b, b = 32 and 64, R = 0
GEOMS = [(1279, 256, 16, 4, None), (1280, 250, 16, 4, None), (1280, 256, 32, 4, None), (1280, 256, 64, 2, 3),
         (1280, 256, 16, 4, 0), (1030, 250, 16, 3, 5), (300, 7, 32, 1, 1)]


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S,TL,b,w,R", GEOMS)
def test_kernels_at_edge_geometries_against_float64(ops, S, TL, b, w, R, dh):
    B, H = 2, 2
    qkv, dout = _qkv(B, S, H, dh, _gen(S + TL + b + dh))
    bs = ops.BlockSparse(layout(S, TL, b, w, R), b, S)
    check(ops, f"S={S} TL={TL} b={b} w={w} R={R} dh={dh}", qkv, dout, bs, S, 1)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S,b", [(1280, 16), (1279, 32), (1000, 64)])
def test_full_layout_is_the_causal_kernel_bit_for_bit(ops, S, b, dh):
    B, H = 2, 4
    qkv, dout = _qkv(B, S, H, dh, _gen(S + b + dh))
    nb = -(-S // b)
    bs = ops.BlockSparse(layout(S, 256, b, 4, nb), b, S)
    assert bs.layout.sum() == nb * (nb + 1) // 2
    out, lse, dqkv = run_bs(ops, qkv, dout, bs)
    ref_out, ref_lse = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, ref_out, ref_lse, B, S, H, dh, 1.0)
    ref_dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, ref_out, dout, ref_lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), ref_dqkv, B, S, H,
                 dh, 1.0)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse) and torch.equal(dqkv, ref_dqkv)
    print(f"[{TAG}] S={S} b={b} dh={dh} R=nb: out, lse and dqkv bit for bit the causal kernels'")


@pytest.mark.parametrize("dh", [64, 128])
def test_a_dominating_key_in_an_unset_block_is_not_seen(ops, dh):
    S, TL, b, B, H = 1280, 256, 16, 1, 2
    lay = layout(S, TL, b, 4, 5)
    qkv, dout = _qkv(B, S, H, dh, _gen(77 + dh))
    q = torch.zeros(B, S, H, dh, device=DEV)
    q[..., 0] = 1.0
    key = torch.zeros(B, S, H, dh, device=DEV)
    key[..., 0] = 0.01 * torch.randn(B, S, H, device=DEV, generator=_gen(1))
    # every key whose block some later query block does not see dominates
    g = torch.arange(S, device=DEV) // b
    unset = torch.as_tensor([not lay[c:, c].all() for c in range(lay.shape[0])], device=DEV)
    key[:, unset[g], :, 0] = 8.0
    qkv[:, :, 0], qkv[:, :, 1] = q.to(BF16), key.to(BF16)
    bs = ops.BlockSparse(lay, b, S)
    out, lse, dqkv = run_bs(ops, qkv, dout, bs)
    res = ratios(qkv, dout, out, lse, dqkv, visible(S, lay, b))
    assert max(res.values()) < 1.0, res
    causal = torch.ones(S, S, dtype=torch.bool, device=DEV).tril()
    got = max(ratios(qkv, dout, out, lse, dqkv, causal).values())
    print(f"[{TAG}] dh={dh} dominating keys in unset blocks against the causal mask: worst {got:.1f}")
    assert got > 1.0


def test_prefill_lengths_use_the_full_length_tables(ops):
    """A prompt prefill runs the forward at S = P < the layout's length, with the tables of the full length."""
    import test_decode_kernels_gpu as DEC
    N, TL, B, H, dh = 1280, 256, 2, 4, 128
    bs = ops.BlockSparse(layout(N, TL), 16, N)
    qkv_full, dout_full = _qkv(B, N, H, dh, _gen(5))
    for P in sorted({TL - 5, TL, TL + 1, *DEC.PREFILL_P, N - 1, N}):
        qkv, dout = qkv_full[:, :P].contiguous(), dout_full[:, :P].contiguous()
        out, lse, dqkv = run_bs(ops, qkv, dout, bs)
        vis = visible(N, bs.layout, 16)[:P, :P]
        for n, v in ratios(qkv, dout, out, lse, dqkv, vis).items():
            float64_bounds.report(f"prefill P={P} {n}", v, TAG)


def test_invalid_arguments_are_rejected(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    B, S, H, dh = 1, 200, 1, 64
    bs = ops.BlockSparse(layout(S, 20), 16, S)
    qkv = torch.zeros(B, S, 3, H, dh, dtype=BF16, device=DEV)
    out, lse = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV), torch.zeros(B, H, S, device=DEV)
    kc = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV)
    step = torch.zeros(B, 3, H, dh, dtype=BF16, device=DEV)
    pos = torch.zeros(1, dtype=I32, device=DEV)
    s = L.stream_ptr()
    t, bl = bs.tiles.data_ptr(), bs.blocks.data_ptr()
    for tp, pitch in ((None, 4), (t, 3)):   # ceil(200 / 64) = 4 rows
        assert lib.db200_attn_block_sparse_fwd(s, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, S, H, dh, tp,
                                               pitch, 1.0) != 0
        assert lib.db200_attn_block_sparse_bwd(s, qkv.data_ptr(), out.data_ptr(), out.data_ptr(), lse.data_ptr(), None,
                                               lse.data_ptr(), qkv.data_ptr(), B, S, H, dh, tp, pitch, 1.0) != 0
    for bp, pitch in ((None, 14), (bl, 13)):   # ceil(200 / 16) + 1 = 14 entries per row
        assert lib.db200_attn_decode_block_sparse(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B,
                                                  S, H, dh, 3, bp, pitch, 1.0) != 0
        assert lib.db200_attn_decode_block_sparse_dev(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(),
                                                      B, S, H, dh, pos.data_ptr(), bp, pitch, 1.0) != 0
    for kw in ({"radius": 4}, {"conv": (4, 4, 2)}, {"dropout": L.make_dropout(0.1, 0, 0, 2, 0)}):
        with pytest.raises(L.DB200Error):
            ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, block_sparse=bs, **kw)
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, block_sparse=bs.tiles)
    small = ops.BlockSparse(layout(100, 20), 16, 100)
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, block_sparse=small)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- decode
@pytest.mark.parametrize("b,R,dh", [(16, None, 64), (16, None, 128), (32, 3, 128), (64, 0, 64)])
def test_attn_decode_block_sparse_against_float64(ops, b, R, dh):
    TL, S = 256, 1280
    B, H = 4, 512 // dh
    g = _gen(dh + b)
    bs = ops.BlockSparse(layout(S, TL, b, 4, R), b, S)
    vis = visible(S, bs.layout, b)
    for pos in (0, 15, 16, 100, TL - 1, TL, TL + 1, 700, 703, 1000, S - 17, S - 1):
        kc = (torch.randn(B, S, H, dh, generator=g, device=DEV) * 1.3 * dh ** -0.25).to(BF16)
        vc = torch.randn(B, S, H, dh, generator=g, device=DEV).to(BF16)
        step = torch.randn(B, 3, H, dh, generator=g, device=DEV)
        step[:, :2] *= 1.3 * dh ** -0.25
        step = step.to(BF16)
        kc2, vc2 = kc.clone(), vc.clone()
        out = nan_like((B, H, dh), BF16)
        ops.attn_decode(step, kc, vc, out, pos, 1.0, block_sparse=bs)
        assert torch.equal(kc[:, pos], step[:, 1]) and torch.equal(vc[:, pos], step[:, 2])
        keys = vis[pos].nonzero()[:, 0]
        ref, absref, bb = decode_reference(step[:, 0], kc[:, keys], vc[:, keys], 1.0)
        float64_bounds.check(f"attn_decode b={b} R={R} dh={dh} pos={pos}", out, ref, absref, b=bb, bf16_out=True,
                             tag=TAG)
        pos_dev = torch.full((1,), pos, dtype=I32, device=DEV)
        out_dev = nan_like((B, H, dh), BF16)
        ops.attn_decode_dev(step, kc2, vc2, out_dev, pos_dev, 1.0, block_sparse=bs)
        assert torch.equal(out_dev, out) and torch.equal(kc2, kc) and torch.equal(vc2, vc)


# ------------------------------------------------------------------------------------------------------- engine
# d, layers, H, text vocab, image vocab, text len, image len, B, layer types, block size
CASES = [(256, 4, 2, 1000, 100, 40, 100, 3, ("block_sparse", "axial_row", "global", "conv"), 16),
         (256, 3, 4, 1000, 100, 100, 196, 2, ("local", "block_sparse", "axial_col"), 32),
         (512, 2, 4, 3000, 512, 70, 256, 2, ("block_sparse", "block_sparse"), 64)]
SPARSE_KW = dict(sparse_local_window_blocks=2, sparse_random_blocks=1, sparse_layout_seed=3)


def _case(d, Ly, H, tv, iv, ts, isl, B, types, b, recompute=False, rates=(0.0, 0.0, 0.0), dseed=0, seed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, recompute_grad=recompute, dropout=rates, dropout_seed=dseed,
                      attention_types=types, local_attention_radius=48, conv_attention_kernel=3, sparse_block_size=b,
                      **SPARSE_KW)
    layouts = tuple(None if m is None else m.layout for m in eng.block_sparse)
    cfg = OB.BlockSparseConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=48,
                               conv_attention_kernel=3, sparse_block_size=b, block_sparse_layouts=layouts)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for n in params:
        if n.endswith("/b") or n.endswith("bias") or n.endswith("o_b"):
            params[n] = torch.randn(params[n].shape, generator=g) * 0.02
        if n.endswith("/g"):
            params[n] = 1 + torch.randn(params[n].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng.load_params(params)
    return cfg, params, tokens, eng


@pytest.mark.parametrize("rates", [(0.0, 0.0, 0.0), RATES], ids=["no-dropout", "dropout"])
@pytest.mark.parametrize("case", CASES)
def test_mixed_engine_matches_the_oracle_recompute_off_and_on(case, rates):
    step, row0, dseed = 6, 1, 11
    spec = (rates, dseed, step, row0)
    cfg, params, tokens, _ = _case(*case, rates=rates, dseed=dseed)
    loss32, _, logits32, g32 = OB.loss_and_grads(params, tokens, cfg, spec, bf16=False)
    _, _, logits16, g16 = OB.loss_and_grads(params, tokens, cfg, spec, bf16=True)
    tok = tokens.to(I32).cuda()
    T = tokens.numel()
    by_mode = []
    for recompute in (False, True):
        _, _, _, eng = _case(*case, recompute=recompute, rates=rates, dseed=dseed)
        eng.zero_grads()
        acc = eng.forward(tok, step=step, row0=row0)
        eng.backward(1.0 / T)
        torch.cuda.synchronize()
        assert abs(acc.item() / T - loss32.item()) / loss32.item() < 2e-3, recompute
        grads = eng.export_params(eng.grads)
        for n in g32:
            e_engine, e_ref = relfro(grads[n], g32[n]), relfro(g16[n], g32[n])
            assert e_engine <= 1.25 * e_ref + 1e-2, (recompute, n, e_engine, e_ref)
        by_mode.append(eng.grads.clone())
        if not any(rates):
            lg = eng.logits(tok)
            assert relfro(lg, logits32) <= 1.25 * relfro(logits16, logits32) + 1e-2
    assert torch.equal(by_mode[0], by_mode[1])
    # the block-sparse layers matter: the same weights with those layers global give other logits
    gtypes = tuple("global" if t == "block_sparse" else t for t in case[8])
    gcfg = OB.BlockSparseConfig(*case[:7], attention_types=gtypes, local_attention_radius=48, conv_attention_kernel=3)
    assert relfro(OB.forward(params, tokens, gcfg, spec)[2], logits32) > 1e-3


def _three_steps(types, rates=RATES, **kw):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 196, dropout=rates, dropout_seed=1, attention_types=types, **kw)
    eng.init_params(3)
    tok = torch.randint(0, 40, (4, eng.S), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV, dtype=I32)
    out = []
    for s in range(3):
        eng.zero_grads()
        acc = eng.forward(tok, step=s)
        eng.backward(1.0 / tok.numel())
        out.append((acc.clone(), eng.grads.clone()))
        eng.optimizer_step(1e-3)
    torch.cuda.synchronize()
    return out, eng.master.clone()


def test_training_is_bitwise_reproducible_and_calls_the_block_sparse_kernels(monkeypatch):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.dalle_engine import DalleEngine
    lib = L.load()
    seen = []
    for name in ("db200_attn_causal_fwd", "db200_attn_causal_fwd_ex", "db200_attn_causal_bwd",
                 "db200_attn_causal_bwd_ex", "db200_attn_block_sparse_fwd", "db200_attn_block_sparse_bwd"):
        fn = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _fn=fn, _n=name: (seen.append(_n), _fn(*a))[1])
    types = ["block_sparse", "global", "block_sparse"]
    a, pa = _three_steps(types, shared_attn_ids=[0, 1, 0])
    calls = list(seen)
    seen.clear()
    b, pb = _three_steps(types, shared_attn_ids=[0, 1, 0])
    for (la, ga), (lb, gb) in zip(a, b):
        assert torch.isfinite(ga).all() and torch.equal(la, lb) and torch.equal(ga, gb)
    assert torch.equal(pa, pb) and seen == calls
    one_step = ["db200_attn_block_sparse_fwd", "db200_attn_causal_fwd_ex", "db200_attn_block_sparse_fwd",
                "db200_attn_block_sparse_bwd", "db200_attn_causal_bwd_ex", "db200_attn_block_sparse_bwd"]
    assert calls == one_step * 3
    assert not torch.equal(_three_steps(["global"] * 3)[1], pa)
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 196, dropout=RATES, dropout_seed=1, attention_types=types,
                      shared_attn_ids=[0, 1, 0])
    dd = eng._dropout_descs(2, 0)
    assert dd["attn"][0] is None and dd["attn"][1] is not None and dd["attn"][2] is None
    assert eng.block_sparse[0] is eng.block_sparse[2] and eng.block_sparse[1] is None
    assert eng.block_sparse_kw[1] == {}


# ------------------------------------------------------------------------------------------------------- generation
GEN = [(256, 3, 2, 300, 64, 24, 100, 3, ("axial_row", "block_sparse", "global"), 16, 29),
       (256, 3, 4, 500, 100, 70, 196, 2, ("block_sparse", "local", "block_sparse"), 32, 77)]


def _sharp(d, Ly, H, tv, iv, ts, isl, types, b):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20,
                      sparse_block_size=b, **SPARSE_KW)
    cfg = OB.BlockSparseConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20,
                               sparse_block_size=b,
                               block_sparse_layouts=tuple(None if m is None else m.layout for m in eng.block_sparse))
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(9)
    for n in params:
        if n.endswith("/b") or n.endswith("bias") or n.endswith("o_b"):
            params[n] = torch.randn(params[n].shape, generator=g) * 0.02
        if "wte" in n or "wout" in n or n.endswith("kernel"):
            params[n] = params[n] * 4
    eng.load_params(params)
    return eng, params, cfg


@pytest.mark.parametrize("d,Ly,H,tv,iv,ts,isl,B,types,b,P", GEN)
def test_generation_follows_the_full_forward_pass(d, Ly, H, tv, iv, ts, isl, B, types, b, P):
    from dalle_mtf_b200.sampling import DalleSampler
    eng, params, cfg = _sharp(d, Ly, H, tv, iv, ts, isl, types, b)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, tv, (B, ts), generator=g).to(I32).cuda()
    smp = DalleSampler(eng)
    toks, step_logits = smp.generate(text, temperature=0, return_logits=True)
    S = ts + isl
    img = toks[:, ts:]
    assert (img >= tv).all() and (img < tv + iv).all()
    full = eng.logits(toks)
    dec = torch.stack(step_logits, 1)
    assert relfro(dec, full[:, :S - 1]) < 2e-2
    _, _, logits32, _ = OB.loss_and_grads(params, toks.cpu().long(), cfg, bf16=False)
    assert relfro(dec, logits32[:, :S - 1]) < 3e-2
    assert torch.equal(smp.generate_graphed(text, temperature=0.0), toks)
    kc = [torch.zeros_like(c) for c in smp.kc]
    vc = [torch.zeros_like(c) for c in smp.vc]
    smp.generate(text, temperature=0)
    logits = eng.prefill(toks[:, :P].contiguous(), kc, vc).clone()
    assert torch.equal(kc[0][:, :P], smp.kc[0][:, :P]) and torch.equal(vc[0][:, :P], smp.vc[0][:, :P])
    for i in range(1, Ly):
        assert relfro(kc[i][:, :P], smp.kc[i][:, :P]) <= 1e-2, i
        assert relfro(vc[i][:, :P], smp.vc[i][:, :P]) <= 1e-2, i
    assert relfro(logits[:, :eng.V], full[:, P - 1]) < 2e-2
    assert relfro(logits[:, :eng.V], logits32[:, P - 1]) < 3e-2
    out = smp.complete(text, toks[:, ts:P] - tv, temperature=0)
    assert torch.equal(out[:, :P], toks[:, :P]) and (out[:, P:] >= tv).all() and (out[:, P:] < tv + iv).all()


def test_guided_generation_runs_on_a_block_sparse_model():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, _, _ = _sharp(256, 3, 2, 300, 64, 24, 100, ("block_sparse", "global", "block_sparse"), 16)
    smp = DalleSampler(eng)
    text = torch.randint(0, 299, (3, 24), generator=torch.Generator().manual_seed(2)).to(I32).cuda()
    eager = smp.generate(text, temperature=0.0, guidance_scale=3.0)
    graphed = smp.generate_graphed(text, temperature=0.0, guidance_scale=3.0)
    assert torch.equal(eager, graphed) and torch.equal(eager[:, :24], text)
    assert ((eager[:, 24:] >= 300) & (eager[:, 24:] < 364)).all()
    torch.manual_seed(0)
    a = smp.complete(text, eager[:, 24:31] - 300, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    torch.manual_seed(0)
    b = smp.complete(text, eager[:, 24:31] - 300, samples_per_prompt=2, temperature=1.0, guidance_scale=3.0, top_k=8)
    assert torch.equal(a, b) and a.shape == (6, 124) and ((a[:, 24:] >= 300) & (a[:, 24:] < 364)).all()


def test_model_fn_trains_evaluates_and_round_trips_a_checkpoint(tmp_path):
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import dalle_model_fn
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 32}})

    def params(**extra):
        p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 32}, "train_batch_size": 4,
                                       "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                       "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                       "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                       "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                       "vae_params": vae, "vae_random_init": True, "seed": 5,
                                       "attention_dropout": 0.1, "residual_dropout": 0.1})
        p.update(extra)
        return p

    g = torch.Generator().manual_seed(3)
    img, cap = torch.rand(4, 32, 32, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)
    sparse = dict(attention_types=[[["block_sparse", "global"], 1]], sparse_block_size=16,
                  sparse_local_window_blocks=1, sparse_random_blocks=0)
    spec = dalle_model_fn(img, cap, "train", params(**sparse))
    eng = spec.engine
    assert eng.block_sparse[1] is None and eng.block_sparse[0].block == 16
    losses = [spec.train_op(img, cap).item() * spec.loss_scale for _ in range(2)]
    ev = spec.eval_op(img, cap).item() * spec.loss_scale
    assert all(math.isfinite(x) and 0 < x < 20 for x in losses + [ev])
    named = {k: v.clone() for k, v in eng.export_params().items()}
    again = dalle_model_fn(img, cap, "eval", params(**sparse))
    again.engine.load_params(named)
    assert again.eval_op(img, cap).item() == spec.eval_op(img, cap).item()
    plain = dalle_model_fn(img, cap, "eval", params())
    plain.engine.load_params(named)
    assert plain.eval_op(img, cap).item() != spec.eval_op(img, cap).item()
    with pytest.raises(ValueError, match="sparse_layout_seed"):
        dalle_model_fn(img, cap, "train", params(sparse_layout_seed=-1))
