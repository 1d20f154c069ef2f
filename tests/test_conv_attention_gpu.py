"""GPU tests of convolutional attention layers (dalle_mtf_b200/csrc/attn_fa.cu, CONV; decode.cu).

Text length TL, a W x W image grid, kernel size k: text queries are causal; the image query at (r, c) sees every text
key plus the image keys of the k x k window (r - k, r] x (c - k, c].  The kernels are checked against float64 with the
bounds of the causal kernels (test_axial_attention_gpu.py's masked_reference with the conv mask) at geometries that
break tile assumptions: windows that straddle 64-row tiles, W > 64, TL not a multiple of 64, W = 1, k > W.  Window-edge
tests make the keys just outside the window dominate and must fail against the oracle of kernel k - 1 and k + 1, and
against a raster band of the same reach.  Then prompt prefills at ragged lengths, the decode kernels (host and device
position, bit for bit), an engine with every layer type against tests/conv_oracle.py, the attention calls it makes,
generation and dalle_model_fn.  The module prints its wall time and peak device memory.
"""
import math
import time

import pytest
import torch

import conv_oracle as OC
import float64_bounds
from float64_bounds import DEV, nan_like
from test_axial_attention_gpu import ratios
from test_local_attention_gpu import RATES, _gen, _qkv, decode_reference, relfro

pytestmark = pytest.mark.gpu

F64, F32, BF16, I32 = torch.float64, torch.float32, torch.bfloat16, torch.int32
TAG = "conv-attention"


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


# ------------------------------------------------------------------------------------------------------- kernels
def visible(S, TL, W, k):
    return ~OC.conv_hidden(S, TL, W, k).to(DEV)


def band_visible(S, TL, W, k):
    """A wrong mask for the edge tests: the text prefix plus the raster band that reaches the window's top-left key."""
    i = torch.arange(S, device=DEV)[:, None]
    j = torch.arange(S, device=DEV)[None, :]
    return (j <= i) & ((j < TL) | (j >= i - (k - 1) * (W + 1)))


def run_conv(ops, qkv, dout, geom, scale=1.0):
    B, S, _, H, dh = qkv.shape
    out, lse = nan_like((B, S, H, dh), BF16), nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, scale, conv=geom)
    dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out, dout, lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv, B, S, H, dh, scale,
                 conv=geom)
    return out, lse, dqkv


# (TL, W, k, B, H): the dalle_example grid at k 5 and 11; W not dividing 64 and TL not a multiple of 64; W > 64;
# W = 1; k > W
GRIDS = [(256, 32, 5, 2, 2), (256, 32, 11, 2, 2), (100, 24, 3, 2, 2), (64, 80, 7, 1, 1), (7, 1, 1, 2, 2),
         (16, 8, 9, 2, 2)]


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("TL,W,k,B,H", GRIDS)
def test_conv_kernels_against_float64(ops, TL, W, k, B, H, dh):
    S = TL + W * W
    qkv, dout = _qkv(B, S, H, dh, _gen(TL * 7 + W + k + dh))
    out, lse, dqkv = run_conv(ops, qkv, dout, (TL, W, k))
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    for n, v in ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, k)).items():
        float64_bounds.report(f"conv TL={TL} W={W} k={k} dh={dh} {n}", v, TAG)


@pytest.mark.parametrize("TL,W,k,B,H", GRIDS)
def test_window_edges_are_exact(ops, TL, W, k, B, H):
    """q = 0: lse_i = log(#keys query i sees).  The kernel passes against the oracle and fails against the oracles of
    kernel size k - 1 and k + 1 wherever their masks differ."""
    S, dh = TL + W * W, 64
    qkv, dout = _qkv(B, S, H, dh, _gen(TL + 3 * W + k))
    qkv[:, :, 0] = 0
    out, lse, dqkv = run_conv(ops, qkv, dout, (TL, W, k))
    mask = visible(S, TL, W, k)
    assert max(ratios(qkv, dout, out, lse, dqkv, mask).values()) < 1.0
    assert (lse.to(F64) - torch.log(mask.sum(-1).to(F64))).abs().max() < 1e-5
    for kk in (k - 1, k + 1):
        if kk < 1 or torch.equal(visible(S, TL, W, kk), mask):
            continue
        got = max(ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, kk)).values())
        print(f"[{TAG}] TL={TL} W={W} k={k} against kernel {kk}: worst {got:.1f}")
        assert got > 1.0, kk


# keys made to dominate: whole grid rows r = 0 mod (k + 1) (each is key (r - k, c) of the queries k rows below), whole
# grid columns c = 0 mod (k + 1) (key (r, c - k) of the queries k columns right), anti-diagonals r + c = 0 mod (k + 1)
# (key (r - 1, c + 1) of the query on the same anti-diagonal)
EDGES = {"row": lambda r, c, k: r % (k + 1) == 0, "column": lambda r, c, k: c % (k + 1) == 0,
         "upper_right": lambda r, c, k: (r + c) % (k + 1) == 0}


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("edge", list(EDGES))
def test_dominating_keys_outside_the_window_are_not_seen(ops, edge, dh):
    TL, W, k, B, H = 100, 24, 5, 1, 2
    S = TL + W * W
    qkv, dout = _qkv(B, S, H, dh, _gen(5 + k + dh))
    q = torch.zeros(B, S, H, dh, device=DEV)
    q[..., 0] = 1.0
    key = torch.zeros(B, S, H, dh, device=DEV)
    key[..., 0] = 0.01 * torch.randn(B, S, H, device=DEV, generator=_gen(1))
    u = torch.arange(S, device=DEV) - TL
    dom = (u >= 0) & EDGES[edge](torch.div(u, W, rounding_mode="floor"), u % W, k)
    key[:, dom, :, 0] = 8.0
    qkv[:, :, 0], qkv[:, :, 1] = q.to(BF16), key.to(BF16)
    out, lse, dqkv = run_conv(ops, qkv, dout, (TL, W, k))
    res = ratios(qkv, dout, out, lse, dqkv, visible(S, TL, W, k))
    assert max(res.values()) < 1.0, res
    wrong = {"band": band_visible(S, TL, W, k)}
    if edge != "upper_right":
        wrong.update({f"k={kk}": visible(S, TL, W, kk) for kk in (k - 1, k + 1)})
    for name, m in wrong.items():
        got = max(ratios(qkv, dout, out, lse, dqkv, m).values())
        print(f"[{TAG}] {edge} dh={dh} dominating keys against the {name} mask: worst {got:.1f}")
        assert got > 1.0, name


@pytest.mark.parametrize("TL,W,k", [(256, 32, 5), (100, 24, 3), (64, 80, 7), (16, 8, 9)])
def test_prefill_lengths(ops, TL, W, k):
    """A prompt prefill runs the kernels at S = P <= TL + W^2: absent rows are neither seen nor stored."""
    N, B, H, dh = TL + W * W, 1, 2, 128
    qkv_full, dout_full = _qkv(B, N, H, dh, _gen(TL + W + k))
    for P in (TL - 5, TL, TL + 1, TL + W // 2, TL + 3 * W + W // 2, N - 1, N):
        qkv, dout = qkv_full[:, :P].contiguous(), dout_full[:, :P].contiguous()
        out, lse, dqkv = run_conv(ops, qkv, dout, (TL, W, k))
        assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
        for n, v in ratios(qkv, dout, out, lse, dqkv, visible(P, TL, W, k)).items():
            float64_bounds.report(f"prefill conv TL={TL} W={W} k={k} P={P} {n}", v, TAG)


def test_invalid_conv_arguments_are_rejected(ops):
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    B, S, H, dh = 1, 20, 1, 64
    qkv = torch.zeros(B, S, 3, H, dh, dtype=BF16, device=DEV)
    out, lse = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV), torch.zeros(B, H, S, device=DEV)
    kc = torch.zeros(B, S, H, dh, dtype=BF16, device=DEV)
    step = torch.zeros(B, 3, H, dh, dtype=BF16, device=DEV)
    pos = torch.zeros(1, dtype=I32, device=DEV)
    s = L.stream_ptr()
    for TL, W, k in ((4, 4, 0), (4, 4, -3), (4, 0, 2), (-1, 5, 2), (3, 4, 2)):   # last: S = 20 > 3 + 16
        assert lib.db200_attn_conv_fwd(s, qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, S, H, dh, TL, W, k,
                                       1.0) != 0
        assert lib.db200_attn_conv_bwd(s, qkv.data_ptr(), out.data_ptr(), out.data_ptr(), lse.data_ptr(), None,
                                       lse.data_ptr(), qkv.data_ptr(), B, S, H, dh, TL, W, k, 1.0) != 0
        assert lib.db200_attn_decode_conv(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S, H,
                                          dh, 3, TL, W, k, 1.0) != 0
        assert lib.db200_attn_decode_conv_dev(s, step.data_ptr(), kc.data_ptr(), kc.data_ptr(), out.data_ptr(), B, S,
                                              H, dh, pos.data_ptr(), TL, W, k, 1.0) != 0
    for kw in ({"radius": 4}, {"axial": (4, 4, 0)}, {"dropout": L.make_dropout(0.1, 0, 0, 2, 0)}):
        with pytest.raises(L.DB200Error):
            ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, conv=(4, 4, 2), **kw)
    with pytest.raises(L.DB200Error):
        ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0, conv=(4, 4, True))
    with pytest.raises(L.DB200Error):
        ops.attn_decode(step, kc, kc, torch.zeros(B, H, dh, dtype=BF16, device=DEV), 3, 1.0, conv=(4, 4, 2),
                        axial=(4, 4, 0))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------- decode
@pytest.mark.parametrize("k,dh", [(5, 64), (5, 128), (11, 128), (40, 64)])
def test_attn_decode_conv_against_float64(ops, k, dh):
    TL, W = 256, 32
    B, S, H = 4, TL + W * W, 512 // dh
    g = _gen(dh + k)
    vis = visible(S, TL, W, k)
    # text positions, TL - 1, TL, row starts and ends, r < k - 1 and c < k - 1, mid-grid, the last row, S - 1
    positions = (0, 100, TL - 1, TL, TL + 1, TL + 2 * W + 1, TL + W - 1, TL + W, TL + 5 * W, TL + 6 * W - 1,
                 TL + 17 * W + 2, TL + 17 * W + 9, S - W, S - 1)
    for pos in positions:
        kc = (torch.randn(B, S, H, dh, generator=g, device=DEV) * 1.3 * dh ** -0.25).to(BF16)
        vc = torch.randn(B, S, H, dh, generator=g, device=DEV).to(BF16)
        step = torch.randn(B, 3, H, dh, generator=g, device=DEV)
        step[:, :2] *= 1.3 * dh ** -0.25
        step = step.to(BF16)
        kc2, vc2 = kc.clone(), vc.clone()
        out = nan_like((B, H, dh), BF16)
        ops.attn_decode(step, kc, vc, out, pos, 1.0, conv=(TL, W, k))
        assert torch.equal(kc[:, pos], step[:, 1]) and torch.equal(vc[:, pos], step[:, 2])
        keys = vis[pos].nonzero()[:, 0]
        ref, absref, b = decode_reference(step[:, 0], kc[:, keys], vc[:, keys], 1.0)
        float64_bounds.check(f"attn_decode conv k={k} dh={dh} pos={pos}", out, ref, absref, b=b, bf16_out=True,
                             tag=TAG)
        pos_dev = torch.full((1,), pos, dtype=I32, device=DEV)
        out_dev = nan_like((B, H, dh), BF16)
        ops.attn_decode_dev(step, kc2, vc2, out_dev, pos_dev, 1.0, conv=(TL, W, k))
        assert torch.equal(out_dev, out) and torch.equal(kc2, kc) and torch.equal(vc2, vc)


# ------------------------------------------------------------------------------------------------------- engine
# d, layers, H, text vocab, image vocab, text len, image len (W^2), B, layer types, conv kernel
CASES = [(256, 4, 2, 1000, 100, 40, 25, 3, ("conv", "axial_row", "global", "local"), 2),
         (256, 3, 4, 1000, 100, 100, 64, 2, ("global", "conv", "axial_col"), 5),
         (512, 2, 4, 3000, 512, 70, 100, 2, ("axial_col", "conv"), 11)]


def _case(d, Ly, H, tv, iv, ts, isl, B, types, k, recompute=False, rates=(0.0, 0.0, 0.0), dseed=0, seed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = OC.ConvConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=48,
                        conv_attention_kernel=k)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for n in params:
        if n.endswith("/b") or n.endswith("bias") or n.endswith("o_b"):
            params[n] = torch.randn(params[n].shape, generator=g) * 0.02
        if n.endswith("/g"):
            params[n] = 1 + torch.randn(params[n].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, recompute_grad=recompute, dropout=rates, dropout_seed=dseed,
                      attention_types=types, local_attention_radius=48, conv_attention_kernel=k)
    eng.load_params(params)
    return cfg, params, tokens, eng


@pytest.mark.parametrize("rates", [(0.0, 0.0, 0.0), RATES], ids=["no-dropout", "dropout"])
@pytest.mark.parametrize("case", CASES)
def test_mixed_engine_matches_the_oracle_recompute_off_and_on(case, rates):
    step, row0, dseed = 6, 1, 11
    spec = (rates, dseed, step, row0)
    cfg, params, tokens, _ = _case(*case, rates=rates, dseed=dseed)
    loss32, _, logits32, g32 = OC.loss_and_grads(params, tokens, cfg, spec, bf16=False)
    _, _, logits16, g16 = OC.loss_and_grads(params, tokens, cfg, spec, bf16=True)
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
    # the conv layers matter: the same weights with those layers global give other logits
    gtypes = tuple("global" if t == "conv" else t for t in case[8])
    gcfg = OC.ConvConfig(*case[:7], attention_types=gtypes, local_attention_radius=48)
    assert relfro(OC.forward(params, tokens, gcfg, spec)[2], logits32) > 1e-3


def _three_steps(types, rates=RATES):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 64, dropout=rates, dropout_seed=1, attention_types=types)
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


def test_conv_training_is_bitwise_reproducible_and_calls_the_conv_kernels(monkeypatch):
    from dalle_mtf_b200 import lib as L, ops
    from dalle_mtf_b200.dalle_engine import DalleEngine
    lib = L.load()
    seen = []
    for name in ("db200_attn_causal_fwd", "db200_attn_causal_fwd_ex", "db200_attn_causal_bwd",
                 "db200_attn_causal_bwd_ex", "db200_attn_local_fwd", "db200_attn_local_bwd", "db200_attn_axial_fwd",
                 "db200_attn_axial_bwd", "db200_attn_conv_fwd", "db200_attn_conv_bwd"):
        fn = getattr(lib, name)
        # axial and conv calls are recorded with their geometry; every call with its B, S, H, dh
        monkeypatch.setattr(lib, name, lambda *a, _fn=fn, _n=name: (
            seen.append((_n,) + (tuple(a[-4:-1]) if "axial" in _n or "conv" in _n else ())), _fn(*a))[1])
    types = ["conv", "global", "axial_col"]
    a, pa = _three_steps(types)
    calls = list(seen)
    seen.clear()
    b, pb = _three_steps(types)
    for (la, ga), (lb, gb) in zip(a, b):
        assert torch.isfinite(ga).all() and torch.equal(la, lb) and torch.equal(ga, gb)
    assert torch.equal(pa, pb) and seen == calls
    # every step: the conv layer (kernel 5, the default), the global layer (with attention dropout), the column layer;
    # backward reversed
    one_step = [("db200_attn_conv_fwd", 60, 8, 5), ("db200_attn_causal_fwd_ex",), ("db200_attn_axial_fwd", 60, 8, 1),
                ("db200_attn_axial_bwd", 60, 8, 1), ("db200_attn_causal_bwd_ex",), ("db200_attn_conv_bwd", 60, 8, 5)]
    assert calls == one_step * 3
    # without the conv layer the other layers make the calls they made before
    seen.clear()
    _three_steps(["global", "global", "axial_col"])
    assert seen == [("db200_attn_causal_fwd_ex",), ("db200_attn_causal_fwd_ex",), ("db200_attn_axial_fwd", 60, 8, 1),
                    ("db200_attn_axial_bwd", 60, 8, 1), ("db200_attn_causal_bwd_ex",),
                    ("db200_attn_causal_bwd_ex",)] * 3
    assert not torch.equal(_three_steps(["global"] * 3)[1], pa)
    eng = DalleEngine(256, 3, 2, 500, 64, 60, 64, dropout=RATES, dropout_seed=1, attention_types=types)
    dd = eng._dropout_descs(2, 0)
    assert dd["attn"][0] is None and dd["attn"][1] is not None and dd["attn"][2] is None
    assert eng.conv == [(60, 8, 5), None, None] and eng.conv_kw[1] == {}
    assert ops.attn_pairs_conv(eng.S, 60, 8, 5) < ops.attn_pairs(eng.S)


# ------------------------------------------------------------------------------------------------------- generation
GEN = [(256, 3, 2, 300, 64, 24, 36, 3, ("axial_row", "conv", "global"), 3, 29),
       (256, 3, 4, 500, 100, 70, 81, 2, ("conv", "local", "axial_col"), 5, 77)]


def _sharp(d, Ly, H, tv, iv, ts, isl, types, k):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = OC.ConvConfig(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20,
                        conv_attention_kernel=k)
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(9)
    for n in params:
        if n.endswith("/b") or n.endswith("bias") or n.endswith("o_b"):
            params[n] = torch.randn(params[n].shape, generator=g) * 0.02
        if "wte" in n or "wout" in n or n.endswith("kernel"):
            params[n] = params[n] * 4
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, attention_types=types, local_attention_radius=20,
                      conv_attention_kernel=k)
    eng.load_params(params)
    return eng, params, cfg


@pytest.mark.parametrize("d,Ly,H,tv,iv,ts,isl,B,types,k,P", GEN)
def test_conv_generation_follows_the_full_forward_pass(d, Ly, H, tv, iv, ts, isl, B, types, k, P):
    from dalle_mtf_b200.sampling import DalleSampler
    eng, params, cfg = _sharp(d, Ly, H, tv, iv, ts, isl, types, k)
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
    rng = full[:, ts - 1:S - 1, tv:tv + iv]
    top2 = rng.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.05 * rng.abs().max()
    same = (rng.argmax(-1) + tv) == img
    assert (same | ~clear).all() and clear.float().mean() > 0.2 and same.float().mean() > 0.8
    _, _, logits32, _ = OC.loss_and_grads(params, toks.cpu().long(), cfg, bf16=False)
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


def test_guided_generation_runs_on_a_conv_model():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, _, _ = _sharp(256, 3, 2, 300, 64, 24, 36, ("axial_row", "axial_col", "conv"), 3)
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
    assert torch.equal(a, b) and a.shape == (6, 60) and ((a[:, 24:] >= 300) & (a[:, 24:] < 364)).all()
    assert torch.equal(a[:, 24:31], eager.repeat_interleave(2, 0)[:, 24:31])


def test_model_fn_trains_and_evaluates_with_conv_layers(tmp_path):
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import dalle_model_fn
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}})

    def params(**extra):
        p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                       "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                       "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                       "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                       "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                       "vae_params": vae, "vae_random_init": True, "seed": 5,
                                       "attention_dropout": 0.1, "residual_dropout": 0.1})
        p.update(extra)
        return p

    g = torch.Generator().manual_seed(3)
    img, cap = torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)
    conv = dict(attention_types=[[["axial_row", "conv"], 1]], conv_attention_kernel=2)
    spec = dalle_model_fn(img, cap, "train", params(**conv))
    W = math.isqrt(spec.engine.image_seq_len)
    assert spec.engine.conv == [None, (12, W, 2)] and spec.engine.axial == [(12, W, 0), None]
    losses = [spec.train_op(img, cap).item() * spec.loss_scale for _ in range(2)]
    ev = spec.eval_op(img, cap).item() * spec.loss_scale
    assert all(math.isfinite(x) and 0 < x < 20 for x in losses + [ev])
    plain = dalle_model_fn(img, cap, "eval", params())
    ev_conv = dalle_model_fn(img, cap, "eval", params(**conv)).eval_op(img, cap).item()
    assert ev_conv != plain.eval_op(img, cap).item()
    with pytest.raises(ValueError, match="conv_attention_kernel"):
        dalle_model_fn(img, cap, "train", params(conv_attention_kernel=1.5))
