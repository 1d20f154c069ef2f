"""The decoding step and the prompt prefill against float64 at the generation shapes of the three DALL-E configurations.

Method, helpers and bounds of test_dalle_kernels_gpu.py (DK) and float64_bounds.py: the kernel and a float64 torch
computation on the GPU get the same operands, and every output element must satisfy

    |got - ref| <= a |ref| + b absref (+ floor)

(bf16 outputs: half a bf16 ulp at |ref| instead of a |ref|).  Outputs start as NaN.  Each case prints one
`[decode-kernels] <case>: worst err/bound r` line, and r < 1 is required.  No new bound term is needed:
- A decoding step runs the training GEMM (STORE epilogue: b = (K + 9) UTC), LayerNorm forward and embedding kernels.
  Their bounds in DK do not depend on the row count.
- attn_decode takes the bound test_attn_decode derives (DK docstring, "attn_decode").
- The prefill runs the training forward at S = P: the GEMM, causal attention forward (O, lse) and LayerNorm bounds.
- The cache write of attn_decode, the embedding at one position and the hand-off copies are exact: bit for bit.

Shapes come from generation itself.  A recorder wraps the generation path's ops, as DK.engine_calls does, while a
one-layer DalleSampler of each configuration runs eager steps and complete() with an image prefix, 2 samples per prompt
and guidance.  The distinct calls are asserted against the expected set, then replayed with fresh operands:
- every step GEMM and LayerNorm at ROWS: predict_batch_size 1 / 32 / 128 and twice that with guidance, 2, and 65 pairs
  (M = 130: a second 128-row tile with 2 rows).  The logits product runs at N = Vpad with wout and the bias zero past
  V, and those columns must come out exactly 0;
- the prefill forward (4 GEMMs, causal attention, LayerNorm) at P in PREFILL_P and batch in PROMPTS.
attn_decode runs at each configuration's (H, dh) over a filled S = 1280 cache at the positions where its 8-warp key
split, the 32-key stride and the text / image boundary change what runs, with random and edge inputs.  The device-
position variant must match it bit for bit.  Live operands: every wrapped call of eager generation at LIVE_POS is
checked on the operands it actually read, right after the call.

On an H100 80GB HBM3 (132 SMs, 400 W power limit) the module takes 30 s of wall time including start-up, and its peak
device memory is 18.8 GiB (the attn_decode sweep at the 12B width: 130-row caches, their copies and float64 slabs).
"""
import contextlib
import types

import pytest
import torch

import float64_bounds
import test_dalle_kernels_gpu as DK
from float64_bounds import DEV, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "decode-kernels"
CONFIGS = list(DK.CONFIGS)
SLAB = DK.SLAB
ROWS = (1, 2, 32, 64, 65, 128, 130, 256)
PREFILL_P = (257, 300, 768, 1279)
PROMPTS = (1, 4)
DECODE_ROWS = (1, 64, 130)
DECODE_POS = (0, 1, 6, 7, 8, 31, 32, 33, 255, 256, 257, 1023, 1279)
DECODE_KINDS = ("random", "dominant newest key", "dominant first key", "equal keys", "exp underflow")
LIVE_POS = (0, 1, 31, 32, 255, 256, 257, 700, 1278)
TEXT_LEN, IMAGE_LEN = 256, 1024
S_MODEL = TEXT_LEN + IMAGE_LEN
STEP_ROWS = 3                        # rows of the recorded eager steps
REC_B, REC_N, REC_REP, REC_GS = 2, 44, 2, 3.0  # complete() of the recording: prompts, prefix codes, samples, guidance
LN_EPS = 1e-5

_PEAK = [0]


def report(name, r):
    return float64_bounds.report(name, r, TAG)


def bits(t):
    return t.view(torch.int16)


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    yield _ops
    print(f"[{TAG}] peak device memory of the module {_PEAK[0] / 2 ** 30:.1f} GiB")


@pytest.fixture(autouse=True)
def _peak_memory(request):
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------- engines
_ENGINE = {}


def sharp_engine(config, attention_types=None):
    """DalleEngine at the configuration's width, heads and vocabulary, with init_params weights sharpened as
    test_prefill_gpu.sharp_engine does: x4 on wte, wout and the layer kernels, biases and LayerNorm betas N(0, 0.02)
    (bout zero past V).  Attention is then peaked rather than uniform.  One layer, or one per entry of
    attention_types (local layers at the configuration's local_attention_radius, default 256; conv layers at
    its conv_attention_kernel, default 5).  One engine lives at a time."""
    key = (config, None if attention_types is None else tuple(attention_types))
    if key in _ENGINE:
        return _ENGINE[key]
    from dalle_mtf_b200.dalle_engine import DalleEngine
    _ENGINE.clear()
    torch.cuda.empty_cache()
    cfg = DK._config(config)
    n_layers = 1 if attention_types is None else len(attention_types)
    eng = DalleEngine(cfg["n_embd"], n_layers, cfg["n_heads"], cfg["text_vocab_size"], cfg["image_vocab_size"],
                      TEXT_LEN, IMAGE_LEN, attention_types=attention_types,
                      local_attention_radius=cfg.get("local_attention_radius", 256),
                      conv_attention_kernel=cfg.get("conv_attention_kernel", 5))
    eng.init_params(seed=3)
    g = DK._gen(9)
    for n in ("wte", "wout") + tuple(f"l{i}.{w}" for i in range(n_layers) for w in ("wqkv", "wo", "w1", "w2")):
        eng.P(n).mul_(4)
    for n in tuple(f"l{i}.{b}" for i in range(n_layers) for b in ("ln1_b", "o_b", "ln2_b", "b1", "b2")) + ("lnf_b",):
        eng.P(n).copy_(torch.randn(eng.P(n).shape, generator=g, device=DEV) * 0.02)
    eng.P("bout")[:eng.V].copy_(torch.randn(eng.V, generator=g, device=DEV) * 0.02)
    eng.refresh_shadow()
    _ENGINE[key] = eng
    return eng


# ------------------------------------------------------------------------------------------------------- recorder
GEN_OPS = ("gemm", "layernorm_fwd", "attn_fwd", "attn_decode", "attn_decode_dev", "embed_fwd", "embed_fwd_at",
           "embed_fwd_at_dev", "kv_cache_fill", "rows_repeat")


def describe(name, args, kw):
    """A call's shape descriptor.  Reads shapes and strides only, never tensor data (safe during graph capture)."""
    if name in ("gemm", "layernorm_fwd", "attn_fwd", "embed_fwd"):
        return DK._describe(name, args, kw)
    if name in ("attn_decode", "attn_decode_dev"):
        return (name,) + tuple(args[1].shape) + (float(args[5]), kw.get("radius"), kw.get("axial"), kw.get("conv"))
    if name == "embed_fwd_at":
        return (name, args[3].shape[0], args[1].shape[0], args[3].shape[1])
    if name == "embed_fwd_at_dev":
        return (name, args[3].shape[0], args[1].shape[0], args[3].shape[1], args[0].stride(0))
    rep = int(args[-1] if len(args) > (4 if name == "kv_cache_fill" else 2) else kw.get("rep", 1))
    if name == "kv_cache_fill":
        return (name, args[0].shape[0], tuple(args[1].shape), int(args[3]), rep)
    return (name, tuple(args[0].shape), args[0].stride(0), rep)


@contextlib.contextmanager
def wrapped(ops, hook):
    """ops.<GEN_OPS> replaced by hook(name, original, args, kw) inside the block."""
    orig = {n: getattr(ops, n) for n in GEN_OPS}

    def wrap(n):
        return lambda *args, **kw: hook(n, orig[n], args, kw)

    try:
        for n in GEN_OPS:
            setattr(ops, n, wrap(n))
        yield
    finally:
        for n in GEN_OPS:
            setattr(ops, n, orig[n])


_CALLS = {}


def generation_calls(ops, config, attention_types=None):
    """Distinct calls of (a) eager DalleSampler.step at STEP_ROWS rows and positions 0, 1, 256, and (b) complete() of
    REC_B prompts with a REC_N-code image prefix, REC_REP samples per prompt and guidance (the captured step at
    2 REC_B REC_REP rows and the prefill of 2 REC_B prompts), on sharp_engine(config, attention_types).  Also returns
    the engine's dimensions, its per-layer radii (None: global) and its per-layer attention geometry
    layers = ((radius, axial, conv), ...) as the attention ops take them (all None: causal)."""
    key = (config, None if attention_types is None else tuple(attention_types))
    if key in _CALLS:
        return _CALLS[key]
    from dalle_mtf_b200.sampling import DalleSampler
    eng = sharp_engine(config, attention_types)
    smp = DalleSampler(eng)
    seen = {"step": {}, "complete": {}}
    phase = ["step"]

    def record(n, f, args, kw):
        seen[phase[0]].setdefault(describe(n, args, kw), None)
        return f(*args, **kw)

    g = DK._gen(5)
    tv, iv = eng.text_vocab_size, eng.image_vocab_size
    with wrapped(ops, record):
        smp._alloc(STEP_ROWS)
        for pos in (0, 1, 256):
            smp.step(torch.randint(0, tv + iv, (STEP_ROWS,), generator=g, device=DEV, dtype=I32), pos)
        phase[0] = "complete"
        text = torch.randint(0, tv, (REC_B, TEXT_LEN), generator=g, device=DEV, dtype=I32)
        prefix = torch.randint(0, iv, (REC_B, REC_N), generator=g, device=DEV, dtype=I32)
        out = smp.complete(text, prefix, samples_per_prompt=REC_REP, temperature=0, guidance_scale=REC_GS)
        torch.cuda.synchronize()
    assert out.shape == (REC_B * REC_REP, eng.S)
    dims = types.SimpleNamespace(d=eng.d, H=eng.H, dh=eng.dh, V=eng.V, Vpad=eng.Vpad, S=eng.S, scale=eng.attn_scale,
                                 radii=tuple(eng.radii), layers=tuple(zip(eng.radii, eng.axial, eng.conv)))
    res = ({k: list(v) for k, v in seen.items()}, dims)
    del smp
    torch.cuda.empty_cache()
    _CALLS[key] = res
    return res


def _linear(M, N, K, *, bias=False, relu=False, res=False, f32=False):
    from dalle_mtf_b200 import lib as L
    return ("gemm", M, N, K, False, True, L.EPI_STORE, str(F32 if f32 else BF16), bias, relu, res, False, 1, 0, False,
            False)


def step_products(M, dm):
    """The 4 linear products of a layer and the fp32 logits product at M rows."""
    d = dm.d
    return [_linear(M, 3 * d, d), _linear(M, d, d, bias=True, res=True), _linear(M, 4 * d, d, bias=True, relu=True),
            _linear(M, d, 4 * d, bias=True, res=True), _linear(M, dm.Vpad, d, bias=True, f32=True)]


def expected_step_calls(rows, dm, graphed):
    """The distinct calls of one step at `rows` rows: one attn_decode(_dev) shape per distinct layer geometry
    (radius, axial, conv)."""
    s = set(step_products(rows, dm)) | {("layernorm_fwd", rows, dm.d)}
    if graphed:
        s |= {("attn_decode_dev", rows, dm.S, dm.H, dm.dh, dm.scale) + g for g in dm.layers}
        s |= {("embed_fwd_at_dev", rows, dm.V, dm.d, dm.S)}
    else:
        s |= {("attn_decode", rows, dm.S, dm.H, dm.dh, dm.scale) + g for g in dm.layers}
        s |= {("embed_fwd_at", rows, dm.V, dm.d)}
    return s


def expected_prefill_calls(dm):
    """The distinct calls complete() adds to its step's for the prefill of generation_calls: one attn_fwd shape per
    distinct layer geometry (radius, axial, conv), at S = P."""
    B2, P, R2 = 2 * REC_B, TEXT_LEN + REC_N, 2 * REC_B * REC_REP
    T = B2 * P
    return set(step_products(T, dm)[:4]) | {("attn_fwd", B2, P, dm.H, dm.dh, dm.scale, False) + g for g in dm.layers} | {
        ("layernorm_fwd", T, dm.d), ("embed_fwd", B2, P, False),
        ("kv_cache_fill", T, (R2, dm.S, dm.H, dm.dh), P, REC_REP), ("rows_repeat", (B2, dm.d), P * dm.d, REC_REP)}


@pytest.mark.parametrize("config", CONFIGS)
def test_generation_call_set(ops, config):
    """Per step: 4 linear GEMMs, the fp32 logits GEMM, 3 LayerNorm forwards (one shape), one attn_decode, one
    embed_fwd_at.  complete() adds the prefill: its embedding, LayerNorm, 4 GEMMs and attention at 2 REC_B prompts of
    P = 256 + REC_N, then kv_cache_fill, rows_repeat, the final LayerNorm and the logits GEMM at the step's rows."""
    calls, dm = generation_calls(ops, config)
    # the configurations' samplers run causal attention: no window, no axial and no conv geometry
    assert dm.radii == (None,) and dm.layers == ((None, None, None),)
    assert set(calls["step"]) == expected_step_calls(STEP_ROWS, dm, graphed=False), calls["step"]
    R2 = 2 * REC_B * REC_REP
    assert set(calls["complete"]) == expected_step_calls(R2, dm, graphed=True) | expected_prefill_calls(dm), \
        calls["complete"]
    print(f"[{TAG}] {config}: eager step {len(calls['step'])} distinct calls, complete() {len(calls['complete'])} "
          f"(d={dm.d} H={dm.H} dh={dm.dh} V={dm.V} Vpad={dm.Vpad})")


# ------------------------------------------------------------------------------------------------------- replays
def replay_gemm(ops, tag, desc, M, seed, n_valid=None):
    """A recorded product at M rows with fresh operands (DK.gemm_operands).  n_valid: B's columns and the bias are
    zero from n_valid on, as the engine pads wout / bout, and those output columns must be exactly 0."""
    (_, _, N, K, _, b_mn, mode, _, _, _, _, _, split_k, _, _, _) = desc
    splits = DK.gemm_splits(M, N, K, mode, split_k, DK._sm())
    tiles = -(-M // 128) * -(-N // 128) * splits
    name = DK.gemm_case_name(desc, M, N, K, splits, tiles, tag=tag)
    o = DK.gemm_operands(ops, desc, M, K, seed)
    if n_valid is not None:
        name += f" zero past {n_valid}"
        (o.b[:, n_valid:] if b_mn else o.b[n_valid:]).zero_()
        o.bias[n_valid:] = 0
    DK.run_gemm(ops, o)
    r = report(name, DK.check_gemm(name, o, splits, report=False))
    if n_valid is not None:
        assert (o.out[:, n_valid:] == 0).all(), f"{name}: padding columns are not exactly 0"
    return r


def replay_layernorm(ops, tag, rows, d, seed):
    x, gam, bet = DK.ln_operands(rows, d, DK._gen(seed))
    y, mean, rstd = nan_like((rows, d), BF16), nan_like((rows,), F32), nan_like((rows,), F32)
    ops.layernorm_fwd(x, gam, bet, y, mean, rstd, LN_EPS)
    rs = DK.check_layernorm_fwd(tag, x, gam, bet, y, mean, rstd, LN_EPS, report=False)
    return max(report(f"{tag} {n}", r) for n, r in rs.items())


@pytest.mark.parametrize("config", CONFIGS)
def test_step_products_at_the_generation_rows(ops, config):
    calls, dm = generation_calls(ops, config)
    gemms = [c for c in calls["step"] if c[0] == "gemm"]
    assert sorted(gemms) == sorted(step_products(STEP_ROWS, dm))
    kind = "wide" if dm.d == 4096 else "warp"
    worst = 0.0
    for i, desc in enumerate(gemms):
        logits = desc[2] == dm.Vpad
        for rows in ROWS:
            worst = max(worst, replay_gemm(ops, f"{config} step ", desc, rows, seed=100 * i + rows,
                                           n_valid=dm.V if logits else None))
    for rows in ROWS:
        worst = max(worst, replay_layernorm(ops, f"{config} step LN {kind} rows={rows} d={dm.d}", rows, dm.d,
                                            seed=rows))
    print(f"[{TAG}] {config} step products and LayerNorm at rows {ROWS}: worst err/bound {worst:.4f}")


@pytest.mark.parametrize("config", CONFIGS)
def test_prefill_forward_at_the_prompt_lengths(ops, config):
    calls, dm = generation_calls(ops, config)
    T_rec = 2 * REC_B * (TEXT_LEN + REC_N)
    gemms = [c for c in calls["complete"] if c[0] == "gemm" and c[1] == T_rec]
    assert sorted(gemms) == sorted(step_products(T_rec, dm)[:4])
    (att,) = [c for c in calls["complete"] if c[0] == "attn_fwd"]
    scale = att[5]
    kind = "wide" if dm.d == 4096 else "warp"
    worst = 0.0
    for B in PROMPTS:
        for P in PREFILL_P:
            M = B * P
            for i, desc in enumerate(gemms):
                worst = max(worst, replay_gemm(ops, f"{config} prefill ", desc, M, seed=10 * M + i))
            worst = max(worst, replay_layernorm(ops, f"{config} prefill LN {kind} rows={M} d={dm.d}", M, dm.d,
                                                seed=M))
            qkv, _ = DK._qkv(B, P, dm.H, dm.dh, DK._gen(M + 1))
            out, lse = nan_like((B, P, dm.H, dm.dh), BF16), nan_like((B, dm.H, P), F32)
            ops.attn_fwd(qkv, out, lse, B, P, dm.H, dm.dh, scale)
            tag = f"{config} prefill attention B={B} S={P} H={dm.H} dh={dm.dh}"
            rs = DK.check_attention(tag, B, P, dm.H, dm.dh, scale, qkv, out, lse, report=False)
            worst = max([worst] + [report(f"{tag} {n}", r) for n, r in rs.items()])
    print(f"[{TAG}] {config} prefill forward at P {PREFILL_P} x prompts {PROMPTS}: worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- attn_decode
def decode_operands(kind, rows, S, H, dh, g):
    """Step q|k|v [rows, 3, H, dh] (fp32, edited per position by decode_step) and filled bf16 caches [rows, S, H, dh].
    q, k at the spread of DK._qkv (logits of a few units at scale 1), v N(0, 1)."""
    sp = 1.3 * dh ** -0.25
    kc = DK._randn(rows, S, H, dh, g=g, scale=sp, dtype=BF16)
    vc = DK._randn(rows, S, H, dh, g=g, dtype=BF16)
    step = torch.randn(rows, 3, H, dh, generator=g, device=DEV)
    step[:, :2] *= sp
    if kind in ("dominant newest key", "dominant first key"):
        kc[..., 0] = 0
        step[:, 0, :, 0] = 4.0
        if kind == "dominant first key":
            kc[:, 0, :, 0] = 10.0               # every later key scores ~40 below key 0
    elif kind == "equal keys":
        kc.copy_(kc[:, :1].clone().expand_as(kc))
        step[:, 1] = kc[:, 0].float()
    elif kind == "exp underflow":
        # q = e_0: score_j = k_j[0], spread over [-110, 0] below the newest key's 0, so exponent arguments cross the
        # range where __expf's result is subnormal and flushed (arg < -87.3)
        step[:, 0] = 0
        step[:, 0, :, 0] = 1.0
        kc[..., 0] = (torch.rand(rows, S, H, generator=g, device=DEV) * -110).to(BF16)
        step[:, 1, :, 0] = 0.0
    return step, kc, vc


def decode_step(kind, step, pos):
    """The bf16 step operands at `pos` (the dominating key sits at pos, or at 0 from pos 1 on)."""
    s = step.clone()
    if kind == "dominant newest key":
        s[:, 1, :, 0] = 10.0
    elif kind == "dominant first key":
        s[:, 1, :, 0] = 10.0 if pos == 0 else 0.0
    return s.to(BF16)


def check_decode(w, step, kc, vc, out, pos, scale):
    """out of attn_decode at `pos` against float64 over the caches (which hold the step's k / v at pos), in row chunks
    of <= SLAB float64 elements per tensor.  Adds to the Worst w."""
    rows, _, H, dh = kc.shape
    chunk = max(1, SLAB // ((pos + 1) * H * dh))
    for r0 in range(0, rows, chunk):
        r1 = min(rows, r0 + chunk)
        ref, absref, b = DK.attn_decode_reference(step[r0:r1, 0], kc[r0:r1, :pos + 1], vc[r0:r1, :pos + 1], scale)
        w.add(out[r0:r1], ref, absref, b=b, bf16_out=True)
        del ref, absref, b


def assert_cache_write(name, kc, vc, kc0, vc0, step, pos):
    """Position pos of every row and head holds the step's k / v bit for bit; every other element is unchanged."""
    assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])), f"{name}: k not written at pos"
    assert torch.equal(bits(vc[:, pos]), bits(step[:, 2])), f"{name}: v not written at pos"
    for c, c0 in ((kc, kc0), (vc, vc0)):
        assert torch.equal(bits(c[:, :pos]), bits(c0[:, :pos])), f"{name}: cache changed below pos"
        assert torch.equal(bits(c[:, pos + 1:]), bits(c0[:, pos + 1:])), f"{name}: cache changed above pos"


@pytest.mark.parametrize("config", CONFIGS)
def test_attn_decode_sweep(ops, config):
    """attn_decode at each (rows, input kind, position), then attn_decode_dev with the same position in device memory
    on a copy of the caches as they were before the call: the same output and caches, bit for bit."""
    cfg = DK._config(config)
    H, dh = cfg["n_heads"], cfg["n_embd"] // cfg["n_heads"]
    S, scale = S_MODEL, 1.0
    worst = 0.0
    for rows in DECODE_ROWS:
        for ki, kind in enumerate(DECODE_KINDS):
            step32, kc, vc = decode_operands(kind, rows, S, H, dh, DK._gen(17 * rows + ki))
            w = DK.Worst(f"{config} attn_decode rows={rows} H={H} dh={dh} {kind} pos {DECODE_POS[0]}..{DECODE_POS[-1]}")
            for pos in DECODE_POS:
                step = decode_step(kind, step32, pos)
                kc0, vc0 = kc.clone(), vc.clone()
                out = nan_like((rows, H, dh), BF16)
                ops.attn_decode(step, kc, vc, out, pos, scale)
                name = f"{w.name} at pos={pos}"
                assert_cache_write(name, kc, vc, kc0, vc0, step, pos)
                check_decode(w, step, kc, vc, out, pos, scale)
                out_dev = nan_like((rows, H, dh), BF16)
                ops.attn_decode_dev(step, kc0, vc0, out_dev, torch.tensor([pos], dtype=I32, device=DEV), scale)
                assert torch.equal(bits(out_dev), bits(out)), f"{name}: attn_decode_dev output differs"
                assert torch.equal(bits(kc0), bits(kc)) and torch.equal(bits(vc0), bits(vc)), \
                    f"{name}: attn_decode_dev caches differ"
                # the edited keys go back to the kind's pattern for the next position
                kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
                del kc0, vc0
            worst = max(worst, report(w.name, w.r))
            del kc, vc
            torch.cuda.empty_cache()
    print(f"[{TAG}] {config} attn_decode sweep: worst err/bound {worst:.4f}")


@pytest.mark.parametrize("dh", [64, 128])
def test_attn_decode_shared_memory_limit(ops, dh):
    """The scores of one (row, head) live in up to 200 KiB of shared memory: S = 51 200 at pos = S - 1 runs (both
    variants, bit for bit equal) and passes the bound; S = 51 201 is refused on the host with DB200_E_UNSUPPORTED by
    both (the device variant's position is 0 < S and never read)."""
    from dalle_mtf_b200 import lib as L
    g = DK._gen(dh)
    S = 51200
    pos = S - 1
    step = DK._randn(1, 3, 1, dh, g=g, dtype=BF16)
    kc = DK._randn(1, S, 1, dh, g=g, scale=1.3 * dh ** -0.25, dtype=BF16)
    vc = DK._randn(1, S, 1, dh, g=g, dtype=BF16)
    kc0, vc0 = kc.clone(), vc.clone()
    out = nan_like((1, 1, dh), BF16)
    ops.attn_decode(step, kc, vc, out, pos, 1.0)
    name = f"attn_decode S={S} pos={pos} dh={dh}"
    assert_cache_write(name, kc, vc, kc0, vc0, step, pos)
    w = DK.Worst(name)
    check_decode(w, step, kc, vc, out, pos, 1.0)
    report(name, w.r)
    out_dev = nan_like((1, 1, dh), BF16)
    ops.attn_decode_dev(step, kc0, vc0, out_dev, torch.tensor([pos], dtype=I32, device=DEV), 1.0)
    assert torch.equal(bits(out_dev), bits(out)) and torch.equal(bits(kc0), bits(kc))
    lib, s = L.load(), L.stream_ptr()
    big = S + 1
    kb = torch.zeros(big * dh, dtype=BF16, device=DEV)
    vb = torch.zeros_like(kb)
    zero = torch.zeros(1, dtype=I32, device=DEV)
    args = (step.data_ptr(), kb.data_ptr(), vb.data_ptr(), out.data_ptr(), 1, big, 1, dh)
    assert lib.db200_attn_decode(s, *args, big - 1, 1.0) == -4                       # DB200_E_UNSUPPORTED
    assert lib.db200_attn_decode_dev(s, *args, zero.data_ptr(), 1.0) == -4
    torch.cuda.synchronize()
    print(f"[{TAG}] attn_decode dh={dh}: S={big} refused by both variants (DB200_E_UNSUPPORTED)")


# ------------------------------------------------------------------------------------------------------- embedding
@pytest.mark.parametrize("config", CONFIGS)
def test_embedding_at_one_position(ops, config):
    """embed_fwd_at and embed_fwd_at_dev equal bf16_rne(wte[id] + wpe[pos]) of float64 and the training embed_fwd on
    the same (id, pos), bit for bit, at the real vocabulary.  The _dev token matrix is a [B, S] view of a [B, S + 24]
    one (row stride != width) whose other columns hold other ids."""
    cfg = DK._config(config)
    d, tv, iv = cfg["n_embd"], cfg["text_vocab_size"], cfg["image_vocab_size"]
    V = tv + iv + 1
    g = DK._gen(V)
    wte = DK._randn(V, d, g=g, scale=0.02, dtype=BF16)
    wpe = DK._randn(S_MODEL, d, g=g, scale=0.01, dtype=BF16)
    ids = torch.tensor([0, tv - 1, tv, V - 1], dtype=I32, device=DEV)       # tv - 1: the padding id
    B = ids.numel()
    for pos in (0, 255, 256, 1279):
        ref = DK.bf16_rne(wte[ids.long()].to(F64) + wpe[pos].to(F64))
        out = nan_like((B, d), BF16)
        ops.embed_fwd_at(ids, wte, wpe, out, pos)
        wide = torch.randint(0, V, (B, S_MODEL + 24), generator=g, device=DEV, dtype=I32)
        wide[:, :S_MODEL] = (ids[:, None] + 1 + torch.arange(S_MODEL, device=DEV, dtype=I32)) % V
        wide[:, pos] = ids
        tokens = wide[:, :S_MODEL]
        assert tokens.stride(0) != tokens.shape[1]
        out_dev = nan_like((B, d), BF16)
        ops.embed_fwd_at_dev(tokens, wte, wpe, out_dev, torch.tensor([pos], dtype=I32, device=DEV))
        ids_full = torch.zeros(B, pos + 1, dtype=I32, device=DEV)
        ids_full[:, pos] = ids
        out_full = nan_like((B, pos + 1, d), BF16)
        ops.embed_fwd(ids_full, wte, wpe, out_full)
        for what, t in (("embed_fwd_at", out), ("embed_fwd_at_dev", out_dev), ("embed_fwd", out_full[:, pos])):
            assert torch.equal(bits(t), bits(ref)), f"{config} {what} pos={pos}: not bf16 RNE of wte[id] + wpe[pos]"
        print(f"{float64_bounds.prefix()}[{TAG}] {config} embedding at pos={pos} ids 0, {tv - 1}, {tv}, {V - 1}: "
              "embed_fwd_at, embed_fwd_at_dev and embed_fwd bit for bit (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- hand-off
@pytest.mark.parametrize("H,dh", [(32, 128), (16, 64)])
@pytest.mark.parametrize("P", [1, 257, 1279])
def test_hand_off_copies_at_production_widths(ops, H, dh, P):
    """kv_cache_fill into [B rep, 1280, H, dh] caches and rows_repeat from the strided last-position view of a
    [B, P, H dh] activation, bit for bit; cache positions >= P keep their sentinel."""
    B, S = 2, S_MODEL
    d = H * dh
    g = DK._gen(P + d)
    for rep in (1, 3):
        qkv = DK._randn(B * P, 3 * d, g=g, dtype=BF16)
        kc = torch.full((B * rep, S, H, dh), 7.0, dtype=BF16, device=DEV)
        vc = torch.full_like(kc, -7.0)
        ops.kv_cache_fill(qkv, kc, vc, P, rep)
        q5 = qkv.view(B, 1, P, 3, H, dh)
        for c, i, sentinel in ((kc, 1, 7.0), (vc, 2, -7.0)):
            c = c.view(B, rep, S, H, dh)
            assert torch.equal(bits(c[:, :, :P]), bits(q5[:, :, :, i].expand(B, rep, P, H, dh))), \
                f"kv_cache_fill H={H} dh={dh} P={P} rep={rep}: prompt positions"
            assert (c[:, :, P:] == sentinel).all(), f"kv_cache_fill H={H} dh={dh} P={P} rep={rep}: wrote past P"
        x = DK._randn(B, P, d, g=g, dtype=BF16)
        out = nan_like((B * rep, d), BF16)
        ops.rows_repeat(x[:, P - 1], out, rep)
        assert torch.equal(bits(out), bits(x[:, P - 1].repeat_interleave(rep, 0))), \
            f"rows_repeat d={d} P={P} rep={rep}"
        print(f"[{TAG}] kv_cache_fill / rows_repeat H={H} dh={dh} P={P} rep={rep}: bit for bit (worst err/bound 0)")


# ------------------------------------------------------------------------------------------------------- live operands
class LiveCheck:
    """Hook of `wrapped`: at positions in LIVE_POS, each call of an eager step is checked against float64 on the
    operands it read, right after it returns (no step call overwrites its own inputs; attn_decode writes position pos
    of the cache, which its reference includes).  Worst ratios are gathered per call shape."""

    def __init__(self, tag, dm):
        self.tag, self.dm, self.pos = tag, dm, None
        self.worst, self.count = {}, {}

    def add(self, key, r):
        self.worst[key] = max(self.worst.get(key, 0.0), r)

    def hook(self, n, f, args, kw):
        out = f(*args, **kw)
        if torch.cuda.is_current_stream_capturing() or self.pos not in LIVE_POS:
            return out
        key = getattr(self, "_" + n)(args, kw)
        self.count[key] = self.count.get(key, 0) + 1
        return out

    def _gemm(self, args, kw):
        from dalle_mtf_b200 import lib as L
        a, b, out, M, N, K = args[:6]
        assert int(kw.get("mode", L.EPI_STORE)) == L.EPI_STORE and kw.get("dropout") is None
        desc = DK._describe("gemm", args, kw)
        name = DK.gemm_case_name(desc, M, N, K, 1, -(-M // 128) * -(-N // 128), tag=f"{self.tag} ")
        o = types.SimpleNamespace(M=M, N=N, K=K, a=a, b=b, out=out, a_mn=bool(kw.get("a_mn")),
                                  b_mn=bool(kw.get("b_mn")), bias=kw.get("bias"), relu=bool(kw.get("relu")),
                                  res=kw.get("residual"), aux=None, base=None, keep=None, dropout=None, cs_base=None)
        self.add(name, DK.check_gemm(name, o, 1, report=False))
        if N == self.dm.Vpad:
            assert (out[:, self.dm.V:] == 0).all(), f"{name}: logits past V are not exactly 0"
        return name

    def _layernorm_fwd(self, args, kw):
        x, gam, bet, y, mean, rstd, eps = args
        name = f"{self.tag} LN rows={x.shape[0]} d={x.shape[1]}"
        for k, r in DK.check_layernorm_fwd(name, x, gam, bet, y, mean, rstd, eps, report=False).items():
            self.add(f"{name} {k}", r)
        return name

    def _attn_decode(self, args, kw):
        qkv, kc, vc, out, pos, scale = args
        rows, _, H, dh = kc.shape
        step = qkv.view(rows, 3, H, dh)
        name = f"{self.tag} attn_decode rows={rows} H={H} dh={dh}"
        assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])) and torch.equal(bits(vc[:, pos]), bits(step[:, 2])), \
            f"{name} pos={pos}: cache write"
        w = DK.Worst(name)
        check_decode(w, step, kc, vc, out.view(rows, H, dh), pos, scale)
        self.add(name, w.r)
        return name

    def _embed_fwd_at(self, args, kw):
        ids, wte, wpe, out, pos = args
        name = f"{self.tag} embed_fwd_at rows={ids.numel()}"
        ref = DK.bf16_rne(wte[ids.long()].to(F64) + wpe[pos].to(F64))
        assert torch.equal(bits(out), bits(ref)), f"{name} pos={pos}: not bf16 RNE of wte[id] + wpe[pos]"
        self.add(name, 0.0)
        return name

    def finish(self, rows):
        """One line per call shape; every step call was checked at every position of LIVE_POS."""
        n = len(LIVE_POS)
        want = {f"{self.tag} embed_fwd_at rows={rows}": n, f"{self.tag} LN rows={rows} d={self.dm.d}": 3 * n,
                f"{self.tag} attn_decode rows={rows} H={self.dm.H} dh={self.dm.dh}": n}
        gemm = {k: c for k, c in self.count.items() if k not in want}
        assert {k: c for k, c in self.count.items() if k in want} == want, self.count
        assert len(gemm) == 5 and set(gemm.values()) == {n}, gemm
        return max(report(f"{k} at pos {LIVE_POS}", r) for k, r in sorted(self.worst.items()))


@pytest.mark.parametrize("config", CONFIGS)
def test_live_operands_of_eager_generation(ops, config):
    """Eager greedy generate() of the sharpened one-layer engine with 1 row, and with guidance at 65 pairs (130 rows),
    every step call checked at LIVE_POS; then greedy generate_graphed() must return generate()'s tokens."""
    from dalle_mtf_b200.sampling import DalleSampler
    eng = sharp_engine(config)
    _, dm = generation_calls(ops, config)
    smp = DalleSampler(eng)
    tv = eng.text_vocab_size
    g = torch.Generator().manual_seed(21)
    worst = 0.0
    for label, B, gs in (("1 row", 1, None), ("65 pairs guided", 65, REC_GS)):
        rows = B if gs is None else 2 * B
        live = LiveCheck(f"{config} live {label}", dm)
        plain_step = smp.step

        def step(tokens, pos):
            live.pos = pos
            return plain_step(tokens, pos)

        text = torch.randint(0, tv, (B, TEXT_LEN), generator=g).to(I32).to(DEV)
        smp.step = step
        try:
            with wrapped(ops, live.hook):
                toks = smp.generate(text, temperature=0.0, guidance_scale=gs)
        finally:
            del smp.step
        assert ((toks[:, TEXT_LEN:] >= tv) & (toks[:, TEXT_LEN:] < tv + eng.image_vocab_size)).all()
        worst = max(worst, live.finish(rows))
    text = torch.randint(0, tv, (2, TEXT_LEN), generator=g).to(I32).to(DEV)
    eager = smp.generate(text, temperature=0.0)
    graphed = smp.generate_graphed(text, temperature=0.0)
    assert torch.equal(graphed, eager), "greedy generate_graphed differs from generate"
    print(f"[{TAG}] {config} live operands: worst err/bound {worst:.4f}; greedy generate_graphed == generate")
    del smp
    torch.cuda.empty_cache()
