"""Local (sliding-window) attention against float64 at the shapes the engine, the prefill and the decoder launch it.

Method, helpers and bounds of test_dalle_kernels_gpu.py (DK), test_decode_kernels_gpu.py (DEC) and float64_bounds.py:
the kernel and a float64 torch computation on the GPU get the same operands, and every output element must satisfy

    |got - ref| <= a |ref| + b absref (+ floor)

(bf16 outputs: half a bf16 ulp at |ref| instead of a |ref|).  Outputs start as NaN.  Each case prints one
`[local-kernels] <case>: worst err/bound r` line, and r < 1 is required.  In a local layer of radius r, query i sees
keys (i - r, i].

Bounds.  The training kernels take the causal attention bound of DK (module docstring, "Causal attention") with the band
in place of the lower triangle: test_local_attention_gpu.local_reference.  Its S-long sums over-count the keys a local
row adds, so the bound stays valid.  attn_decode takes DK's attn_decode bound over the window [lo, pos],
lo = max(0, pos - r + 1): test_local_attention_gpu.decode_reference.  The cache write, the device-position variant and
r >= S against the global entry point are checked bit for bit.

Edge inputs (S = 1280 and 1279, dh 64 and 128, r in 1, 2, 63-65, 127-129, 255-257 and S - 1):
- Dominators every r keys (r >= 2).  Every row has the same q, with q[0] = 4.  Keys 0, r, 2r, ... are one vector kd
  with kd[0] = 7.5, and every other key has k[0] = 0.  So a dominator's logit is about 30 above every other key.  Any
  r consecutive keys hold exactly one dominator, and row i sees the one at floor(i / r) r.  For rows i = r - 1 (mod r)
  it is the first key of the window, so a window one key too short sees none.  For rows i = 0 (mod r), i >= r, the
  previous dominator sits at i - r, one key below the window, so a window one key too long sees two, tied.  The kernel
  must pass against the oracle at r.  Against the oracle at r - 1 and at r + 1 its O must fail, and so must one of
  dQ / dK / dV.
- Large logits: q, k at 6 times the usual spread.  Rows whose first visited 64-key block lies wholly below their window
  start the online softmax from -inf.
- P rounded to nearest.  DK's test_attention_forward_rounds_p_to_nearest on the dominators-every-r layout: dominators
  have logit 0 and every other key -D, so every other weight is the same c.  The kernel rounds c to bf16 with RNE when
  the row's running max is already its dominator.  A key in a block it visits before the dominator's block enters
  with weight 1 (exact) and is rescaled by exp2(-D log2 e), so its weight is the fp32 c instead.  The reference follows
  both rules.  Dominator values cancel the rest in row n_e of column e (n_e < r) and in every row from r on, so a P
  rounded any other way is far outside the bound.  The bound is DK's without the 2^-8 term, with n_i, the keys of the
  blocks the kernel visits for row i (at most r + 127), in place of S:
      b_i = (n_i + 16) U + 2^-20 + 6 U D + (2 n_i + 64) UTC.

Shapes.  A recorder wraps the ops, as DK.engine_calls and DEC.generation_calls do, while a one-layer local DalleEngine
of dalle_example_local_b200 trains and a two-layer global / local DalleSampler generates.  Then:
- the training kernels run at r = 256, S = 1280 and each width's sequences per GPU (WIDTHS);
- the prefill's attention runs at P in DEC.PREFILL_P with 1 and 4 prompts;
- attn_decode runs at each configuration's (H, dh), DEC.DECODE_ROWS rows, DECODE_RADII and DEC.DECODE_POS plus
  r - 2 .. r + 1, over DEC's input kinds and a dominating key at lo and at lo - 1 (outside the window: no effect);
- the shared-memory rule: a local layer sizes scores for min(S, r) keys, so r = 256 runs on a 60 000-key cache that
  the global kernel refuses, and r = 51 201 is refused.

On an H100 80GB HBM3 (132 SMs, 700 W power limit) the module takes 28 s of wall time including start-up, and its peak
device memory is 8.2 GiB (the attn_decode sweep at the 12B width: 130-row caches, their pristine copies and float64
slabs).  The P-rounded-to-nearest cases measure 0.99 of their bound: with the 2^-8 term gone, the accumulation terms
are what they test.
"""
import pytest
import torch

import float64_bounds
import test_dalle_kernels_gpu as DK
import test_decode_kernels_gpu as DEC
import test_local_attention_gpu as LA
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "local-kernels"
CONFIG = "dalle_example_local_b200"
RADIUS = 256
S_MODEL = DEC.S_MODEL
# width -> sequences per GPU (DK.CONFIGS tokens / 1280), heads, head size
WIDTHS = {"dalle_example_local": (32, 4, 128), "dalle_coco": (16, 16, 64), "12B": (4, 32, 128)}
EDGE_S = (1280, 1279)
EDGE_RADII = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257)          # and S - 1
DECODE_RADII = (1, 2, 7, 8, 9, 31, 32, 33, 255, 256, 257)
DECODE_KINDS = DEC.DECODE_KINDS + ("dominant key at lo", "dominant key at lo - 1")
E_UNSUPPORTED = -4

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


# ------------------------------------------------------------------------------------------------------- call set
def test_engine_and_sampler_call_set(ops):
    """The local engine runs the global engine's calls except attention, and one local attention shape with r = 256
    and no dropout (also when the engine has dropout rates).  The mixed sampler decodes its local layer with r = 256
    and its global one with None, and its prefill runs local attn_fwd at S = P."""
    cfg = DK._config(CONFIG)
    r = cfg["local_attention_radius"]
    assert r == RADIUS
    H, dh = cfg["n_heads"], cfg["n_embd"] // cfg["n_heads"]
    base, _, _, _, S = DK.engine_calls(ops, "dalle_example_b200")
    calls, _, _, _, S_local = DK.engine_calls(ops, CONFIG, attention_types=["local"], local_attention_radius=r)
    assert S_local == S == S_MODEL
    is_att = lambda c: c[0] in ("attn_fwd", "attn_bwd")
    assert {c for c in calls if not is_att(c)} == {c for c in base if not is_att(c)}
    (scale,) = {c[5] for c in base if is_att(c)}
    want = {("attn_fwd", 1, S, H, dh, scale, False, r, None, None),
            ("attn_bwd", 1, S, H, dh, scale, False, r, None, None)}
    assert {c for c in calls if is_att(c)} == want, calls
    dropped = DK.engine_calls(ops, CONFIG, step=6, attention_types=["local"], local_attention_radius=r,
                              dropout=(0.1, 0.1, 0.1), dropout_seed=3)[0]
    assert any(c[0] == "gemm" and c[-1] for c in dropped)                  # the recording ran with dropout
    assert {c for c in dropped if is_att(c)} == want, dropped
    print(f"[{TAG}] {CONFIG} one local layer: {len(calls)} distinct calls, attention {sorted(want)}")

    gen, dm = DEC.generation_calls(ops, CONFIG, ["global", "local"])
    assert dm.radii == (None, r) and dm.layers == ((None, None, None), (r, None, None))
    assert set(gen["step"]) == DEC.expected_step_calls(DEC.STEP_ROWS, dm, graphed=False), gen["step"]
    R2 = 2 * DEC.REC_B * DEC.REC_REP
    assert set(gen["complete"]) == DEC.expected_step_calls(R2, dm, graphed=True) | DEC.expected_prefill_calls(dm), \
        gen["complete"]
    print(f"[{TAG}] {CONFIG} global / local sampler: attn_decode(_dev) with radius None and {r}, prefill attn_fwd "
          f"at S = {DEC.TEXT_LEN + DEC.REC_N} with both")


# ------------------------------------------------------------------------------------------------------- training
def check_local(tag, qkv, out, lse, r, dout=None, dqkv=None, *, scale=1.0, chunk=None, report_lines=True):
    """out / lse (and dqkv when dout is given) of the local kernels on [B, S, 3, H, dh] operands against
    local_reference at radius r, in chunks of sequences as DK.check_attention runs them (a [B, H, S, S] float64 tensor
    at B = 32 would take 1.7 GB).  report_lines=False returns {name: worst err/bound} without printing or asserting."""
    B, _, _, H, _ = qkv.shape
    chunk = chunk or max(1, 16 // H)
    names = ("O", "lse") + (("dQ", "dK", "dV") if dout is not None else ())
    ws = {n: DK.Worst(f"{tag} {n}") for n in names}
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        refs, b_fwd, b_bwd = LA.local_reference(qkv[sl, :, 0], qkv[sl, :, 1], qkv[sl, :, 2],
                                                None if dout is None else dout[sl], out[sl], scale, r)
        ws["O"].add(out[sl], *refs["O"], b=b_fwd, bf16_out=True, floor=2.0 ** -120)
        ws["lse"].add(lse[sl], *refs["lse"], a=0.0, b=1.0)
        if dout is not None:
            for i, n in enumerate(("dQ", "dK", "dV")):
                ws[n].add(dqkv[sl, :, i], *refs[n], b=b_bwd, bf16_out=True, floor=2.0 ** -120)
        del refs
    if not report_lines:
        return {n: w.r for n, w in ws.items()}
    return max(report(w.name, w.r) for w in ws.values())


@pytest.mark.parametrize("width", list(WIDTHS))
def test_local_attention_at_the_engine_shapes(ops, width):
    B, H, dh = WIDTHS[width]
    S, r = S_MODEL, RADIUS
    qkv, dout = DK._qkv(B, S, H, dh, DK._gen(B * H + r))
    out, lse, dqkv = LA.run_local(ops, qkv, dout, r)
    check_local(f"{width} local attention B={B} S={S} H={H} dh={dh} r={r}", qkv, out, lse, r, dout, dqkv)


# ------------------------------------------------------------------------------------------------------- edges
def _edge_radii(S):
    return EDGE_RADII + (S - 1,)


def dominators_every_r(S, H, dh, r, g):
    """One sequence: the same q in every row (q[0] = 4), keys 0, r, 2r, ... all kd (kd[0] = 7.5), every other key
    k[0] = 0 (module docstring)."""
    qkv, dout = DK._qkv(1, S, H, dh, g)
    qkv[:, :, 0] = qkv[:, :1, 0].clone()
    qkv[:, :, 0, :, 0] = 4.0
    qkv[:, :, 1, :, 0] = 0.0
    dom = torch.arange(0, S, r, device=DEV)
    qkv[:, dom, 1] = qkv[:, :1, 1].clone()
    qkv[:, dom, 1, :, 0] = 7.5
    return qkv, dout


def local_p_rounding(ops, S, dh, r):
    """The P-rounded-to-nearest case of the module docstring at radius r >= 2; returns the worst err/bound."""
    H = 2
    D, c = DK._exact_p_weight()
    cb = torch.tensor(c, dtype=F64).to(BF16).to(F64).item()
    pos = torch.arange(S, device=DEV)
    dom = pos % r == 0
    qkv = torch.zeros(1, S, 3, H, dh, device=DEV)
    qkv[:, :, 0, :, 0] = 1.0
    qkv[:, ~dom, 1, :, 0] = -D
    qkv[:, ~dom, 2] = 1.0
    n_e = 1 + torch.arange(dh, device=DEV) * (r - 2) // (dh - 1)          # 1 .. r - 1 others in row n_e
    qkv[:, 0, 2] = -(n_e * cb).float()
    qkv[:, dom & (pos > 0), 2] = -(r - 1) * cb                           # rows >= r see r - 1 others
    qkv = qkv.to(BF16)
    out, lse = nan_like((1, S, H, dh), BF16), nan_like((1, H, S), F32)
    ops.attn_fwd(qkv, out, lse, 1, S, H, dh, 1.0, radius=r)
    p_bf = DK.bf16_rne(torch.tensor([c], dtype=F64, device=DEV)).to(F64).item()
    assert p_bf == cb and cb > c
    i, j = pos[:, None], pos[None, :]
    vis = (j <= i) & (j > i - r)
    d_i = (pos // r) * r                                                  # the row's dominator
    early = (j // 64) < (d_i[:, None] // 64)                              # met before the dominator's block
    zero, one, cT, cbT = (torch.tensor(x, dtype=F64, device=DEV) for x in (0.0, 1.0, c, cb))
    w = torch.where(vis, torch.where(dom[None, :], one, torch.where(early, cT, cbT)), zero)
    tot = torch.where(vis, torch.where(dom[None, :], one, cT), zero).sum(-1)
    v = qkv[0, :, 2].to(F64).permute(1, 0, 2)                             # [H, S, dh]
    ref = ((w @ v) / tot[:, None]).permute(1, 0, 2)[None]
    absref = ((w @ v.abs()) / tot[:, None]).permute(1, 0, 2)[None]
    qb = pos // 64
    n_i = 64 * (qb - torch.clamp(64 * qb - r + 1, min=0) // 64 + 1)      # keys of the visited blocks
    assert int(n_i.max()) <= r + 127
    n_i = n_i.to(F64)
    b = ((n_i + 16) * U + 2.0 ** -20 + 6 * U * D + (2 * n_i + 64) * UTC)[None, :, None, None]
    print(f"[{TAG}] S={S} dh={dh} r={r} P rounded to nearest: {int((early & vis).any(-1).sum())} of {S} rows meet "
          "others before their dominator")
    return float64_bounds.worst_ratio("P rounded", out, ref, absref, b=b, bf16_out=True)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", EDGE_S)
def test_local_attention_edge_inputs(ops, S, dh):
    H = 2
    g = DK._gen(S + dh)
    for r in _edge_radii(S):
        if r >= 2:
            qkv, dout = dominators_every_r(S, H, dh, r, g)
            out, lse, dqkv = LA.run_local(ops, qkv, dout, r)
            report(f"local S={S} dh={dh} r={r} dominators every r", max(LA.ratios(qkv, dout, out, lse, dqkv, r).values()))
            for wrong in (r - 1, r + 1):
                if wrong < 1 or min(wrong, S) == min(r, S):
                    continue
                rs = LA.ratios(qkv, dout, out, lse, dqkv, wrong)
                bwd = max(rs["dQ"], rs["dK"], rs["dV"])
                print(f"[{TAG}] S={S} dh={dh} dominators every r: kernel r={r} against oracle r={wrong}: worst "
                      f"err/bound O {rs['O']:.1f} dQ {rs['dQ']:.1f} dK {rs['dK']:.1f} dV {rs['dV']:.1f}")
                assert rs["O"] > 1.0 and bwd > 1.0, (r, wrong, rs)
            report(f"local S={S} dh={dh} r={r} P rounded to nearest", local_p_rounding(ops, S, dh, r))
        qkv, dout = DK._qkv(1, S, H, dh, g, mag=6.0)
        out, lse, dqkv = LA.run_local(ops, qkv, dout, r)
        report(f"local S={S} dh={dh} r={r} large logits", max(LA.ratios(qkv, dout, out, lse, dqkv, r).values()))


# ------------------------------------------------------------------------------------------------------- prefill
@pytest.mark.parametrize("width", list(WIDTHS))
def test_prefill_local_attention_at_the_prompt_lengths(ops, width):
    _, H, dh = WIDTHS[width]
    worst = 0.0
    for B in DEC.PROMPTS:
        for P in DEC.PREFILL_P:
            qkv, _ = DK._qkv(B, P, H, dh, DK._gen(B * P + H))
            out, lse = nan_like((B, P, H, dh), BF16), nan_like((B, H, P), F32)
            ops.attn_fwd(qkv, out, lse, B, P, H, dh, 1.0, radius=RADIUS)
            worst = max(worst, check_local(f"{width} prefill local attention B={B} S={P} H={H} dh={dh} r={RADIUS}",
                                           qkv, out, lse, RADIUS))
    print(f"[{TAG}] {width} prefill local attention at P {DEC.PREFILL_P} x prompts {DEC.PROMPTS}: worst err/bound "
          f"{worst:.4f}")


# ------------------------------------------------------------------------------------------------------- decode
def check_window(w, step, kc, vc, out, pos, lo, scale):
    """out of a local attn_decode at `pos` against float64 over keys [lo, pos] of the caches, in row chunks of <= SLAB
    float64 elements per tensor.  Adds to the Worst w."""
    rows, _, H, dh = kc.shape
    chunk = max(1, DK.SLAB // ((pos + 1 - lo) * H * dh))
    for r0 in range(0, rows, chunk):
        r1 = min(rows, r0 + chunk)
        ref, absref, b = LA.decode_reference(step[r0:r1, 0], kc[r0:r1, lo:pos + 1], vc[r0:r1, lo:pos + 1], scale)
        w.add(out[r0:r1], ref, absref, b=b, bf16_out=True)
        del ref, absref, b


def _decode_positions(r):
    return sorted({p for p in DEC.DECODE_POS + (r - 2, r - 1, r, r + 1) if 0 <= p < S_MODEL})


def _decode_inputs(kind, rows, H, dh, g):
    """DEC.decode_operands; the two window kinds start from zero k[0] everywhere and q[0] = 4, and the sweep puts
    k[0] = 10 on the key at lo (or lo - 1) of each call."""
    if not kind.startswith("dominant key at lo"):
        return DEC.decode_operands(kind, rows, S_MODEL, H, dh, g)
    step, kc, vc = DEC.decode_operands("random", rows, S_MODEL, H, dh, g)
    kc[..., 0] = 0
    step[:, 0, :, 0] = 4.0
    step[:, 1, :, 0] = 0.0
    return step, kc, vc


@pytest.mark.parametrize("config", DEC.CONFIGS)
def test_attn_decode_local_sweep(ops, config):
    """attn_decode with radius r at each (rows, input kind, r, position) against float64 over [lo, pos]; the cache
    write bit for bit; attn_decode_dev on the caches as they were before the call, bit for bit; after each sweep the
    caches hold nothing but what they started with.  Then r = S against the global entry point, bit for bit."""
    cfg = DK._config(config)
    H, dh = cfg["n_heads"], cfg["n_embd"] // cfg["n_heads"]
    S, scale = S_MODEL, 1.0
    worst = 0.0
    for rows in DEC.DECODE_ROWS:
        for ki, kind in enumerate(DECODE_KINDS):
            step32, kc, vc = _decode_inputs(kind, rows, H, dh, DK._gen(31 * rows + ki))
            kc0, vc0 = kc.clone(), vc.clone()
            for r in DECODE_RADII:
                w = DK.Worst(f"{config} attn_decode_local rows={rows} H={H} dh={dh} r={r} {kind} pos "
                             f"{_decode_positions(r)[0]}..{_decode_positions(r)[-1]}")
                for pos in _decode_positions(r):
                    lo = max(0, pos - r + 1)
                    step = DEC.decode_step(kind, step32, pos)
                    edit = None
                    if kind == "dominant key at lo":
                        if lo < pos:
                            edit = lo
                        else:
                            step[:, 1, :, 0] = 10.0                      # the window is the newest key alone
                    elif kind == "dominant key at lo - 1" and lo > 0:
                        edit = lo - 1
                    if edit is not None:
                        kc[:, edit, :, 0] = 10.0
                    name = f"{w.name} at pos={pos}"
                    out = nan_like((rows, H, dh), BF16)
                    ops.attn_decode(step, kc, vc, out, pos, scale, radius=r)
                    assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])) and \
                        torch.equal(bits(vc[:, pos]), bits(step[:, 2])), f"{name}: cache write"
                    check_window(w, step, kc, vc, out, pos, lo, scale)
                    kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
                    out_dev = nan_like((rows, H, dh), BF16)
                    ops.attn_decode_dev(step, kc, vc, out_dev, torch.tensor([pos], dtype=I32, device=DEV), scale,
                                        radius=r)
                    assert torch.equal(bits(out_dev), bits(out)), f"{name}: attn_decode_dev output differs"
                    assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])) and \
                        torch.equal(bits(vc[:, pos]), bits(step[:, 2])), f"{name}: attn_decode_dev cache write"
                    kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
                    if edit is not None:
                        kc[:, edit] = kc0[:, edit]
                worst = max(worst, report(w.name, w.r))
            assert torch.equal(bits(kc), bits(kc0)) and torch.equal(bits(vc), bits(vc0)), \
                f"{config} rows={rows} {kind}: a call wrote outside its position"
            for pos in DEC.DECODE_POS:
                step = DEC.decode_step(kind, step32, pos)
                og, ol = nan_like((rows, H, dh), BF16), nan_like((rows, H, dh), BF16)
                ops.attn_decode(step, kc, vc, og, pos, scale)
                ops.attn_decode(step, kc, vc, ol, pos, scale, radius=S)
                assert torch.equal(bits(og), bits(ol)), f"{config} rows={rows} {kind} pos={pos}: r = S differs"
                kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
            del kc, vc, kc0, vc0
            torch.cuda.empty_cache()
    print(f"[{TAG}] {config} attn_decode_local sweep over r {DECODE_RADII}: worst err/bound {worst:.4f}; r = S equals "
          "the global kernel bit for bit")


@pytest.mark.parametrize("dh", [64, 128])
def test_attn_decode_local_shared_memory_rule(ops, dh):
    """Scores of a local layer take min(S, r) floats of shared memory.  On an S = 60 000 cache at pos = S - 1, r = 256
    and r = 51 200 run in both variants (bit for bit equal) and pass the bound, while the global kernel refuses the
    cache; r = 51 201 is refused with DB200_E_UNSUPPORTED by both variants (the device position is never read)."""
    from dalle_mtf_b200 import lib as L
    g = DK._gen(dh + 3)
    S = 60000
    pos = S - 1
    step = DK._randn(1, 3, 1, dh, g=g, dtype=BF16)
    step[:, :2] = (step[:, :2].float() * 1.3 * dh ** -0.25).to(BF16)
    kc = DK._randn(1, S, 1, dh, g=g, scale=1.3 * dh ** -0.25, dtype=BF16)
    vc = DK._randn(1, S, 1, dh, g=g, dtype=BF16)
    for r in (RADIUS, 51200):
        kc0, vc0 = kc.clone(), vc.clone()
        out = nan_like((1, 1, dh), BF16)
        ops.attn_decode(step, kc, vc, out, pos, 1.0, radius=r)
        name = f"attn_decode_local S={S} pos={pos} dh={dh} r={r}"
        DEC.assert_cache_write(name, kc, vc, kc0, vc0, step, pos)
        w = DK.Worst(name)
        check_window(w, step, kc, vc, out, pos, pos - r + 1, 1.0)
        report(name, w.r)
        out_dev = nan_like((1, 1, dh), BF16)
        ops.attn_decode_dev(step, kc0, vc0, out_dev, torch.tensor([pos], dtype=I32, device=DEV), 1.0, radius=r)
        assert torch.equal(bits(out_dev), bits(out)) and torch.equal(bits(kc0), bits(kc)), name
    lib, s = L.load(), L.stream_ptr()
    zero = torch.zeros(1, dtype=I32, device=DEV)
    args = (step.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), 1, S, 1, dh)
    assert lib.db200_attn_decode(s, *args, pos, 1.0) == E_UNSUPPORTED
    assert lib.db200_attn_decode_dev(s, *args, zero.data_ptr(), 1.0) == E_UNSUPPORTED
    assert lib.db200_attn_decode_local(s, *args, pos, 51201, 1.0) == E_UNSUPPORTED
    assert lib.db200_attn_decode_local_dev(s, *args, zero.data_ptr(), 51201, 1.0) == E_UNSUPPORTED
    torch.cuda.synchronize()
    print(f"[{TAG}] attn_decode dh={dh} S={S}: refused by the global kernel, r = 51201 refused by both local variants "
          "(DB200_E_UNSUPPORTED)")
