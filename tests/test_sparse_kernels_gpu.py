"""Axial (row / column) and convolutional attention against float64 at the shapes the engine, the prefill and the decoder
launch them.

Method, helpers and bounds of test_dalle_kernels_gpu.py (DK), test_decode_kernels_gpu.py (DEC) and float64_bounds.py:
the kernel and a float64 torch computation on the GPU get the same operands, and every output element must satisfy

    |got - ref| <= a |ref| + b absref (+ floor)

(bf16 outputs: half a bf16 ulp at |ref| instead of a |ref|).  Outputs start as NaN.  Each case prints one
`[sparse-kernels] <case>: worst err/bound r` line, and r < 1 is required.  Masks come from tests/axial_oracle.py and
tests/conv_oracle.py (TL text keys, a W x W image grid; conv layers of kernel size k).

Bounds.  The training kernels take DK's causal attention bound with the layer's mask in place of the lower triangle:
test_axial_attention_gpu.masked_reference.  Its S-long sums over-count the keys a sparse row adds, so the bound stays
valid.  attn_decode takes DK's attn_decode bound over the position's key list (test_local_attention_gpu.decode_reference).
The cache write and the device-position variant are checked bit for bit.

Shapes.  A recorder wraps the ops, as DK.engine_calls and DEC.generation_calls do, while one-layer axial and conv
DalleEngines of dalle_example_axial_b200 / dalle_example_conv_b200 train and a [global, axial_row, axial_col, conv]
DalleSampler generates.  Then:
- the training kernels run for both axes and conv at k = 5 and 11, at S = 1280 and each width's sequences per GPU
  (WIDTHS), checked in chunks of sequences;
- the prefill's attention runs at P in DEC.PREFILL_P with 1 and 4 prompts, both axes and conv at k = 5;
- attn_decode runs at each configuration's (H, dh), DEC.DECODE_ROWS rows and DECODE_POS over DEC's input kinds and one
  more: a dominating key just outside the position's key list (no effect);
- the shared-memory rules of attn_decode_launch: a 57 856-key cache the global kernel refuses, and the 51 200 / 51 201
  key boundary of both variants.

Edge inputs (S = 1280 and 1279, dh 64 and 128):
- Large logits: q, k at 6 times the usual spread.
- TL = 0, (TL, W) = (0, 24) and (0, 40) at S = W^2 and W^2 - 1, both axes and conv at k = 3 and 7.  Key 0 is no
  longer visible to every row, and some rows of a query block see nothing in the first key block the walk visits
  (axial W = 24: query block 1 starts at segment 48, so rows 72..127 see nothing in block 0).  They start the online
  softmax from -inf.
- P rounded to nearest, for axial_col and conv k = 5: DK's test_attention_forward_rounds_p_to_nearest with the layer's
  mask.  Key 0, a text key every row sees and the first key of the first block every query block visits, has logit 0
  and every other key -D, so every other weight is the same c, rounded to bf16 with RNE.  Value columns of key 0 cancel
  the rest in rows with m_e other keys, so a P rounded any other way is far outside the bound.  The bound is DK's
  without the 2^-8 term, with n_i, the keys of the blocks the kernel visits for row i (axial_oracle.key_blocks /
  conv_oracle.key_blocks of the row's kernel-order query block), in place of S:
      b_i = (n_i + 16) U + 2^-20 + 6 U D + (2 n_i + 64) UTC.
  These cases measure 0.989 of their bound on an H100: with the 2^-8 term gone, the accumulation terms are what they
  test.

On an H100 80GB HBM3 (132 SMs, 700 W power limit) the module takes 23 s of wall time including start-up, and its peak
device memory is 8.3 GiB (the attn_decode sweep at the 12B width: 130-row caches, their pristine copies and float64
slabs).
"""
import time

import pytest
import torch

import axial_oracle as OA
import conv_oracle as OC
import float64_bounds
import test_dalle_kernels_gpu as DK
import test_decode_kernels_gpu as DEC
from float64_bounds import DEV, U, UTC, nan_like
from test_axial_attention_gpu import masked_reference, ratios, run_axial
from test_conv_attention_gpu import run_conv
from test_local_attention_gpu import decode_reference

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
TAG = "sparse-kernels"
AXIAL_CONFIG, CONV_CONFIG = "dalle_example_axial_b200", "dalle_example_conv_b200"
TL, W = DEC.TEXT_LEN, 32
S_MODEL = DEC.S_MODEL
# width -> sequences per GPU (DK.CONFIGS tokens / 1280), heads, head size
WIDTHS = {"dalle_example": (32, 4, 128), "dalle_coco": (16, 16, 64), "12B": (4, 32, 128)}
# layer -> (attention keyword, geometry) at the dalle_example grid
LAYERS = {"axial_row": ("axial", (TL, W, 0)), "axial_col": ("axial", (TL, W, 1)), "conv k=5": ("conv", (TL, W, 5)),
          "conv k=11": ("conv", (TL, W, 11))}
EDGE_S = (1280, 1279)
# TL = 0: layer names and their (kind, axis or kernel)
ZERO_TEXT = {"axial_row": ("axial", 0), "axial_col": ("axial", 1), "conv k=3": ("conv", 3), "conv k=7": ("conv", 7)}
P_ROUNDING = ("axial_col", "conv k=5")
PREFILL_LAYERS = ("axial_row", "axial_col", "conv k=5")
DECODE_LAYERS = ("axial_row", "axial_col", "conv k=5")
# text positions (incl. the 8-warp key split's 7 / 8 / 31..33), TL - 1 / TL, row starts and ends, r < k - 1 and
# c < k - 1 (TL + 2 W + 1), mid-grid, the last row and S - 1
DECODE_POS = (0, 1, 7, 8, 31, 32, 33, 100, TL - 1, TL, TL + 1, TL + 2 * W + 1, TL + W - 1, TL + W, TL + 5 * W,
              TL + 6 * W - 1, TL + 17 * W + 2, TL + 17 * W + 9, S_MODEL - W, S_MODEL - 1)
DECODE_KINDS = DEC.DECODE_KINDS + ("dominant key outside",)
SMEM_KEYS = 51200                                      # 200 KiB of fp32 scores
# (kind, geometry whose widest key list and device sizing are exactly SMEM_KEYS keys, its twin one key over)
BOUNDARY = [("axial", (51000, 200, 0), (51000, 201, 0)), ("axial", (51192, 8, 1), (51193, 8, 1)),
            ("conv", (51100, 16, 10), (51101, 16, 10)), ("conv", (51136, 8, 9), (51137, 8, 9))]
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
    t0 = time.perf_counter()
    yield _ops
    torch.cuda.synchronize()
    print(f"\n[{TAG}] module wall time {time.perf_counter() - t0:.1f} s, peak device memory of the module "
          f"{_PEAK[0] / 2 ** 30:.1f} GiB on {torch.cuda.get_device_name()}")


@pytest.fixture(autouse=True)
def _peak_memory(request):
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------- geometry
def visible(kind, geom, S):
    """[S, S] bool on the device, sequence order: True where query i sees key j."""
    hidden = OA.axial_hidden(S, *geom) if kind == "axial" else OC.conv_hidden(S, *geom)
    return ~hidden.to(DEV)


def key_list(kind, geom, pos):
    """The keys the query of `pos` sees, restated from the layer's definition (no [S, S] mask): the text run, then the
    grid row's columns <= c / the grid column's rows <= r (axial), or the k x k window rows (conv)."""
    text_len, w, p = geom
    if pos < text_len:
        return torch.arange(pos + 1, device=DEV)
    r, c = divmod(pos - text_len, w)
    text = torch.arange(text_len, device=DEV)
    if kind == "axial":
        img = r * w + torch.arange(c + 1, device=DEV) if p == 0 else torch.arange(r + 1, device=DEV) * w + c
    else:
        rr = torch.arange(max(0, r - p + 1), r + 1, device=DEV)[:, None]
        cc = torch.arange(max(0, c - p + 1), c + 1, device=DEV)[None, :]
        img = (rr * w + cc).flatten()
    return torch.cat([text, text_len + img])


def outside_key(kind, geom, pos):
    """A key just outside the key list of `pos`, or None: the previous row's last token (row layer), the token one
    column left (column layer), the key one column left of the window or else one row above it (conv)."""
    text_len, w, p = geom
    if pos < text_len:
        return None
    r, c = divmod(pos - text_len, w)
    if kind == "axial":
        j = pos - c - 1 if p == 0 else pos - 1
        return j if j >= text_len else None
    if c >= p:
        return pos - p
    return pos - p * w if r >= p else None


def run_layer(ops, kind, geom, qkv, dout):
    return (run_axial if kind == "axial" else run_conv)(ops, qkv, dout, geom)


def kernel_rows(kind, geom, S):
    """Kernel-order row of each sequence position < S (a column layer walks its image rows column-major)."""
    text_len, w, p = geom
    if kind != "axial" or p == 0:
        return torch.arange(S)
    perm = OA.kernel_order(S, text_len, w, 1)
    t = torch.empty(S, dtype=torch.long)
    ok = perm < S
    t[perm[ok]] = torch.arange(perm.numel())[ok]
    return t


def walk(kind, geom, S, qb):
    """Key blocks the forward kernel visits for query block qb (axial_oracle / conv_oracle key_blocks)."""
    text_len, w, p = geom
    return OA.key_blocks(S, text_len, w, qb) if kind == "axial" else OC.key_blocks(S, text_len, w, p, qb)


def check_sparse(tag, qkv, out, lse, mask, dout=None, dqkv=None, *, scale=1.0, chunk=None, report_lines=True):
    """out / lse (and dqkv when dout is given) of a sparse layer on [B, S, 3, H, dh] operands against masked_reference
    with the [S, S] mask, in chunks of sequences as DK.check_attention runs them.  report_lines=False returns
    {name: worst err/bound} without printing or asserting."""
    B, _, _, H, _ = qkv.shape
    chunk = chunk or max(1, 16 // H)
    names = ("O", "lse") + (("dQ", "dK", "dV") if dout is not None else ())
    ws = {n: DK.Worst(f"{tag} {n}") for n in names}
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        refs, b_fwd, b_bwd = masked_reference(qkv[sl, :, 0], qkv[sl, :, 1], qkv[sl, :, 2],
                                              None if dout is None else dout[sl], out[sl], scale, mask)
        ws["O"].add(out[sl], *refs["O"], b=b_fwd, bf16_out=True, floor=2.0 ** -120)
        ws["lse"].add(lse[sl], *refs["lse"], a=0.0, b=1.0)
        if dout is not None:
            for i, n in enumerate(("dQ", "dK", "dV")):
                ws[n].add(dqkv[sl, :, i], *refs[n], b=b_bwd, bf16_out=True, floor=2.0 ** -120)
        del refs
    if not report_lines:
        return {n: w.r for n, w in ws.items()}
    return max(report(w.name, w.r) for w in ws.values())


# ------------------------------------------------------------------------------------------------------- call set
def test_engine_and_sampler_call_set(ops):
    """One-layer axial_row, axial_col and conv engines run the global engine's calls except attention, and one
    attention shape with their (TL, W, axis) / (TL, W, 5) and no dropout (also when the engine has dropout rates).  A
    [global, axial_row, axial_col, conv] sampler decodes and prefills each layer with that layer's geometry."""
    k = DK._config(CONV_CONFIG).get("conv_attention_kernel", 5)
    assert k == 5
    cfg = DK._config(AXIAL_CONFIG)
    H, dh = cfg["n_heads"], cfg["n_embd"] // cfg["n_heads"]
    base, _, _, _, S = DK.engine_calls(ops, "dalle_example_b200")
    is_att = lambda c: c[0] in ("attn_fwd", "attn_bwd")
    (scale,) = {c[5] for c in base if is_att(c)}
    for config, layer, geo in ((AXIAL_CONFIG, "axial_row", (None, (TL, W, 0), None)),
                               (AXIAL_CONFIG, "axial_col", (None, (TL, W, 1), None)),
                               (CONV_CONFIG, "conv", (None, None, (TL, W, k)))):
        kw = dict(attention_types=[layer], conv_attention_kernel=k)
        calls, _, _, _, S_layer = DK.engine_calls(ops, config, **kw)
        assert S_layer == S == S_MODEL
        assert {c for c in calls if not is_att(c)} == {c for c in base if not is_att(c)}, layer
        want = {("attn_fwd", 1, S, H, dh, scale, False) + geo, ("attn_bwd", 1, S, H, dh, scale, False) + geo}
        assert {c for c in calls if is_att(c)} == want, calls
        dropped = DK.engine_calls(ops, config, step=6, dropout=(0.1, 0.1, 0.1), dropout_seed=3, **kw)[0]
        assert any(c[0] == "gemm" and c[-1] for c in dropped)                # the recording ran with dropout
        assert {c for c in dropped if is_att(c)} == want, dropped
        print(f"[{TAG}] {config} one {layer} layer: {len(calls)} distinct calls, attention {sorted(want)}")

    types = ["global", "axial_row", "axial_col", "conv"]
    gen, dm = DEC.generation_calls(ops, CONV_CONFIG, types)
    assert dm.layers == ((None, None, None), (None, (TL, W, 0), None), (None, (TL, W, 1), None),
                         (None, None, (TL, W, k)))
    assert set(gen["step"]) == DEC.expected_step_calls(DEC.STEP_ROWS, dm, graphed=False), gen["step"]
    R2 = 2 * DEC.REC_B * DEC.REC_REP
    assert set(gen["complete"]) == DEC.expected_step_calls(R2, dm, graphed=True) | DEC.expected_prefill_calls(dm), \
        gen["complete"]
    print(f"[{TAG}] {CONV_CONFIG} {'/'.join(types)} sampler: attn_decode(_dev) and prefill attn_fwd at S = "
          f"{DEC.TEXT_LEN + DEC.REC_N} with each layer's geometry")


# ------------------------------------------------------------------------------------------------------- training
@pytest.mark.parametrize("layer", list(LAYERS))
@pytest.mark.parametrize("width", list(WIDTHS))
def test_sparse_attention_at_the_engine_shapes(ops, width, layer):
    B, H, dh = WIDTHS[width]
    kind, geom = LAYERS[layer]
    S = S_MODEL
    qkv, dout = DK._qkv(B, S, H, dh, DK._gen(B * H + geom[2] + 17 * (kind == "conv")))
    out, lse, dqkv = run_layer(ops, kind, geom, qkv, dout)
    check_sparse(f"{width} {layer} attention B={B} S={S} H={H} dh={dh}", qkv, out, lse, visible(kind, geom, S), dout,
                 dqkv)


# ------------------------------------------------------------------------------------------------------- edges
def p_rounding(ops, kind, geom, S, dh):
    """The P-rounded-to-nearest case of the module docstring; returns the worst err/bound."""
    H = 2
    D, c = DK._exact_p_weight()
    cb = torch.tensor(c, dtype=F64).to(BF16).to(F64).item()
    vis = visible(kind, geom, S)
    others = vis.sum(-1) - 1                                              # visible keys besides key 0, per row
    counts = torch.unique(others)
    m_e = counts[torch.arange(dh, device=DEV) * (counts.numel() - 1) // (dh - 1)]
    qkv = torch.zeros(1, S, 3, H, dh, device=DEV)
    qkv[:, :, 0, :, 0] = 1.0
    qkv[:, 1:, 1, :, 0] = -D
    qkv[:, 1:, 2] = 1.0
    qkv[:, 0, 2] = -(m_e * cb).float()                                    # row i cancels in columns m_e = others_i
    qkv = qkv.to(BF16)
    out, lse = nan_like((1, S, H, dh), BF16), nan_like((1, H, S), F32)
    ops.attn_fwd(qkv, out, lse, 1, S, H, dh, 1.0, **{kind: geom})
    p_bf = DK.bf16_rne(torch.tensor([c], dtype=F64, device=DEV)).to(F64).item()
    assert p_bf == cb and cb > c
    first = (torch.arange(S, device=DEV) == 0)[None, :]
    zero, one, cT, cbT = (torch.tensor(x, dtype=F64, device=DEV) for x in (0.0, 1.0, c, cb))
    w = torch.where(vis, torch.where(first, one, cbT), zero)
    tot = torch.where(vis, torch.where(first, one, cT), zero).sum(-1)
    v = qkv[0, :, 2].to(F64).permute(1, 0, 2)                             # [H, S, dh]
    ref = ((w @ v) / tot[:, None]).permute(1, 0, 2)[None]
    absref = ((w @ v.abs()) / tot[:, None]).permute(1, 0, 2)[None]
    qb = kernel_rows(kind, geom, S) // 64
    blocks = {int(b): len(walk(kind, geom, S, int(b))) for b in torch.unique(qb)}
    assert all(walk(kind, geom, S, b)[0] == 0 for b in blocks)            # key 0's block comes first
    n_i = torch.tensor([64.0 * blocks[int(b)] for b in qb], dtype=F64, device=DEV)
    b = ((n_i + 16) * U + 2.0 ** -20 + 6 * U * D + (2 * n_i + 64) * UTC)[None, :, None, None]
    print(f"[{TAG}] {kind} {geom} S={S} dh={dh} P rounded to nearest: visited keys per row {int(n_i.min())}.."
          f"{int(n_i.max())}, others per row {int(others.min())}..{int(others.max())}")
    return float64_bounds.worst_ratio("P rounded", out, ref, absref, b=b, bf16_out=True)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", EDGE_S)
def test_sparse_attention_edge_inputs(ops, S, dh):
    H = 2
    for layer, (kind, geom) in LAYERS.items():
        qkv, dout = DK._qkv(1, S, H, dh, DK._gen(S + dh + geom[2]), mag=6.0)
        out, lse, dqkv = run_layer(ops, kind, geom, qkv, dout)
        report(f"{layer} S={S} dh={dh} large logits",
               max(ratios(qkv, dout, out, lse, dqkv, visible(kind, geom, S)).values()))
    for layer in P_ROUNDING:
        kind, geom = LAYERS[layer]
        report(f"{layer} S={S} dh={dh} P rounded to nearest", p_rounding(ops, kind, geom, S, dh))


def empty_first_block_rows(kind, geom, S):
    """Rows (kernel order) that see no key in the first key block their query block visits."""
    text_len, w, p = geom
    hidden = OA.segment_hidden(S, text_len, w) if kind == "axial" else OC.conv_hidden(S, *geom)
    n = 0
    for qb in range(-(-S // 64)):
        j = walk(kind, geom, S, qb)[0]
        n += int((~hidden[64 * qb:64 * qb + 64, 64 * j:64 * j + 64]).any(-1).logical_not().sum())
    return n


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("grid_w", [24, 40])
def test_zero_text_length(ops, grid_w, dh):
    """TL = 0 at S = W^2 and W^2 - 1: forward and backward against float64, with some rows starting from -inf."""
    H = 2
    for layer, (kind, p) in ZERO_TEXT.items():
        geom = (0, grid_w, p)
        n_empty = empty_first_block_rows(kind, geom, grid_w * grid_w)
        assert n_empty > 0, layer
        for S in (grid_w * grid_w, grid_w * grid_w - 1):
            for mag in (1.0, 6.0):
                qkv, dout = DK._qkv(2, S, H, dh, DK._gen(S + dh + p + int(mag)), mag=mag)
                out, lse, dqkv = run_layer(ops, kind, geom, qkv, dout)
                report(f"{layer} TL=0 W={grid_w} S={S} dh={dh} spread x{mag:g} ({n_empty} rows see nothing in their "
                       "first key block)", max(ratios(qkv, dout, out, lse, dqkv, visible(kind, geom, S)).values()))


# ------------------------------------------------------------------------------------------------------- prefill
@pytest.mark.parametrize("width", list(WIDTHS))
def test_prefill_sparse_attention_at_the_prompt_lengths(ops, width):
    _, H, dh = WIDTHS[width]
    worst = 0.0
    for layer in PREFILL_LAYERS:
        kind, geom = LAYERS[layer]
        for B in DEC.PROMPTS:
            for P in DEC.PREFILL_P:
                qkv, _ = DK._qkv(B, P, H, dh, DK._gen(B * P + H + geom[2]))
                out, lse = nan_like((B, P, H, dh), BF16), nan_like((B, H, P), F32)
                ops.attn_fwd(qkv, out, lse, B, P, H, dh, 1.0, **{kind: geom})
                worst = max(worst, check_sparse(f"{width} prefill {layer} attention B={B} S={P} H={H} dh={dh}",
                                                qkv, out, lse, visible(kind, geom, P)))
    print(f"[{TAG}] {width} prefill {'/'.join(PREFILL_LAYERS)} attention at P {DEC.PREFILL_P} x prompts {DEC.PROMPTS}: "
          f"worst err/bound {worst:.4f}")


# ------------------------------------------------------------------------------------------------------- decode
def check_keys(w, step, kc, vc, out, keys, scale):
    """out of attn_decode against float64 over the key rows `keys` of the caches, in row chunks of <= SLAB float64
    elements per tensor.  Adds to the Worst w."""
    rows, _, H, dh = kc.shape
    chunk = max(1, DK.SLAB // (keys.numel() * H * dh))
    for r0 in range(0, rows, chunk):
        r1 = min(rows, r0 + chunk)
        ref, absref, b = decode_reference(step[r0:r1, 0], kc[r0:r1, keys], vc[r0:r1, keys], scale)
        w.add(out[r0:r1], ref, absref, b=b, bf16_out=True)
        del ref, absref, b


def _decode_inputs(kind, rows, H, dh, g):
    """DEC.decode_operands; "dominant key outside" starts from zero k[0] everywhere and q[0] = 4, and the sweep puts
    k[0] = 10 on the key just outside each call's key list."""
    if kind != "dominant key outside":
        return DEC.decode_operands(kind, rows, S_MODEL, H, dh, g)
    step, kc, vc = DEC.decode_operands("random", rows, S_MODEL, H, dh, g)
    kc[..., 0] = 0
    step[:, 0, :, 0] = 4.0
    step[:, 1, :, 0] = 0.0
    return step, kc, vc


@pytest.mark.parametrize("config", DEC.CONFIGS)
def test_attn_decode_sparse_sweep(ops, config):
    """attn_decode of each layer at each (rows, input kind, position) against float64 over the position's key list;
    the cache write bit for bit; attn_decode_dev on the caches as they were before the call, bit for bit; after each
    sweep the caches hold nothing but what they started with."""
    cfg = DK._config(config)
    H, dh = cfg["n_heads"], cfg["n_embd"] // cfg["n_heads"]
    S, scale = S_MODEL, 1.0
    keys = {}
    for layer in DECODE_LAYERS:
        kind, geom = LAYERS[layer]
        vis = visible(kind, geom, S)
        keys[layer] = {pos: vis[pos].nonzero()[:, 0] for pos in DECODE_POS}
        for pos in DECODE_POS:
            assert torch.equal(keys[layer][pos], key_list(kind, geom, pos)), (layer, pos)
            out_key = outside_key(kind, geom, pos)
            assert out_key is None or not vis[pos, out_key], (layer, pos)
    worst = 0.0
    for rows in DEC.DECODE_ROWS:
        for ki, kind_in in enumerate(DECODE_KINDS):
            step32, kc, vc = _decode_inputs(kind_in, rows, H, dh, DK._gen(37 * rows + ki))
            kc0, vc0 = kc.clone(), vc.clone()
            for layer in DECODE_LAYERS:
                kind, geom = LAYERS[layer]
                kw = {kind: geom}
                w = DK.Worst(f"{config} attn_decode {layer} rows={rows} H={H} dh={dh} {kind_in} pos "
                             f"{DECODE_POS[0]}..{DECODE_POS[-1]}")
                for pos in DECODE_POS:
                    step = DEC.decode_step(kind_in, step32, pos)
                    edit = outside_key(kind, geom, pos) if kind_in == "dominant key outside" else None
                    if edit is not None:
                        kc[:, edit, :, 0] = 10.0
                    name = f"{w.name} at pos={pos}"
                    out = nan_like((rows, H, dh), BF16)
                    ops.attn_decode(step, kc, vc, out, pos, scale, **kw)
                    assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])) and \
                        torch.equal(bits(vc[:, pos]), bits(step[:, 2])), f"{name}: cache write"
                    check_keys(w, step, kc, vc, out, keys[layer][pos], scale)
                    kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
                    out_dev = nan_like((rows, H, dh), BF16)
                    ops.attn_decode_dev(step, kc, vc, out_dev, torch.tensor([pos], dtype=I32, device=DEV), scale, **kw)
                    assert torch.equal(bits(out_dev), bits(out)), f"{name}: attn_decode_dev output differs"
                    assert torch.equal(bits(kc[:, pos]), bits(step[:, 1])) and \
                        torch.equal(bits(vc[:, pos]), bits(step[:, 2])), f"{name}: attn_decode_dev cache write"
                    kc[:, pos], vc[:, pos] = kc0[:, pos], vc0[:, pos]
                    if edit is not None:
                        kc[:, edit] = kc0[:, edit]
                worst = max(worst, report(w.name, w.r))
            assert torch.equal(bits(kc), bits(kc0)) and torch.equal(bits(vc), bits(vc0)), \
                f"{config} rows={rows} {kind_in}: a call wrote outside its position"
            del kc, vc, kc0, vc0
            torch.cuda.empty_cache()
    print(f"[{TAG}] {config} attn_decode {'/'.join(DECODE_LAYERS)} sweep: worst err/bound {worst:.4f}")


def _one_row_cache(S, dh, g):
    step = DK._randn(1, 3, 1, dh, g=g, dtype=BF16)
    step[:, :2] = (step[:, :2].float() * 1.3 * dh ** -0.25).to(BF16)
    kc = DK._randn(1, S, 1, dh, g=g, scale=1.3 * dh ** -0.25, dtype=BF16)
    vc = DK._randn(1, S, 1, dh, g=g, dtype=BF16)
    return step, kc, vc


def _decode_both(ops, name, kind, geom, step, kc, vc, pos):
    """attn_decode at pos against float64 over key_list, its cache write, and attn_decode_dev on the caches as they
    were before the call, bit for bit."""
    kc0, vc0 = kc.clone(), vc.clone()
    dh = kc.shape[-1]
    out = nan_like((1, 1, dh), BF16)
    ops.attn_decode(step, kc, vc, out, pos, 1.0, **{kind: geom})
    DEC.assert_cache_write(name, kc, vc, kc0, vc0, step, pos)
    w = DK.Worst(name)
    check_keys(w, step, kc, vc, out, key_list(kind, geom, pos), 1.0)
    report(name, w.r)
    out_dev = nan_like((1, 1, dh), BF16)
    ops.attn_decode_dev(step, kc0, vc0, out_dev, torch.tensor([pos], dtype=I32, device=DEV), 1.0, **{kind: geom})
    assert torch.equal(bits(out_dev), bits(out)) and torch.equal(bits(kc0), bits(kc)), name


def _widest(kind, geom):
    """The position with the longest key list of a grid."""
    text_len, w, p = geom
    if kind == "axial":
        return text_len + (w - 1 if p == 0 else (w - 1) * w)
    m = min(p, w) - 1
    return text_len + m * w + m


def _raw_decode(kind, dev):
    from dalle_mtf_b200 import lib as L
    return getattr(L.load(), f"db200_attn_decode_{kind}{'_dev' if dev else ''}")


@pytest.mark.parametrize("dh", [64, 128])
def test_attn_decode_sparse_shared_memory_rules(ops, dh):
    """Scores of an axial / conv layer take the position's key list of shared memory (host variant) or
    min(S, TL + W) / min(S, TL + k min(k, W)) floats (device variant).  TL = 256, W = 240 (S = 57 856): both axes and
    conv run at pos = S - 1 and pass the bound, while the global kernel refuses the cache.  At each BOUNDARY grid the
    widest key list and the device sizing are exactly 51 200 keys: both variants run and pass; on its twin both are
    refused with DB200_E_UNSUPPORTED (the device position is never read).  (51 136, 8, 9) is k > W: the device sizing
    k min(k, W) = 72 exceeds the W^2 = 64 image keys, so S itself sizes it."""
    from dalle_mtf_b200 import lib as L
    g = DK._gen(dh + 5)
    S = 256 + 240 * 240
    step, kc, vc = _one_row_cache(S, dh, g)
    for kind, geom in (("axial", (256, 240, 0)), ("axial", (256, 240, 1)), ("conv", (256, 240, 5))):
        _decode_both(ops, f"attn_decode {kind} {geom} S={S} pos={S - 1} dh={dh}", kind, geom, step, kc, vc, S - 1)
    lib, s = L.load(), L.stream_ptr()
    zero = torch.zeros(1, dtype=I32, device=DEV)
    out = nan_like((1, 1, dh), BF16)
    args = (step.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), 1, S, 1, dh)
    assert lib.db200_attn_decode(s, *args, S - 1, 1.0) == E_UNSUPPORTED
    assert lib.db200_attn_decode_dev(s, *args, zero.data_ptr(), 1.0) == E_UNSUPPORTED
    del kc, vc
    for kind, ok, over in BOUNDARY:
        for geom, accept in ((ok, True), (over, False)):
            text_len, w, p = geom
            pos = _widest(kind, geom)
            n = key_list(kind, geom, pos).numel()
            assert n == SMEM_KEYS + (not accept), (geom, n)
            S = min(text_len + w * w, max(pos + 1, SMEM_KEYS + 1))          # the device sizing, not S, is at the edge
            dev_keys = min(S, text_len + (w if kind == "axial" else p * min(p, w)))
            assert dev_keys == SMEM_KEYS + (not accept), (geom, S, dev_keys)
            step, kc, vc = _one_row_cache(S, dh, g)
            name = f"attn_decode {kind} {geom} S={S} pos={pos} dh={dh} ({n} keys)"
            if accept:
                _decode_both(ops, name, kind, geom, step, kc, vc, pos)
            else:
                args = (step.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), 1, S, 1, dh)
                assert _raw_decode(kind, False)(s, *args, pos, *geom, 1.0) == E_UNSUPPORTED, name
                assert _raw_decode(kind, True)(s, *args, zero.data_ptr(), *geom, 1.0) == E_UNSUPPORTED, name
                print(f"[{TAG}] {name}: refused by both variants (DB200_E_UNSUPPORTED)")
            del kc, vc
    torch.cuda.synchronize()
