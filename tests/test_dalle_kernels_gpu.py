"""DALL-E transformer kernels against float64 references of the same operation on the same operands.

Method as in test_vae_kernels_gpu.py (helpers in float64_bounds.py): the kernel and a float64 torch computation on the
GPU get the SAME rounded operands, and every output element must satisfy

    |got - ref| <= a |ref| + b absref (+ floor)

with absref the same operation in float64 on |operands| (it bounds every partial sum the kernel can form); bf16 outputs
take half a bf16 ulp at |ref| instead of a |ref|.  Written outputs start as NaN; accumulated outputs (dw, colsum,
dg / db / dxsum, dwte / dwpe, loss_sum, gnorm_sq) start from a non-zero base the reference adds too.  One
`[dalle-kernels] <case>: worst err/bound r` line per case; r < 1 is required.  U = 2^-24 (fp32), UTC = 2^-23 (one
wgmma accumulation step, which may truncate), u_bf = 2^-8 (bf16 unit roundoff).

GEMM (every epilogue).  b = (K + 8 + splits) UTC: K accumulation steps, the bias / residual / alpha / red.add
  operations and one add per split-K slice.  RELU_BWD multiplies by an exact 0/1 mask.  colsum (RELU_BWD, CE_GRAD) is
  checked against float64 column sums of the bf16 values the kernel wrote: 32-row blocks of two 16-long chains, then
  the row blocks added in order onto the base, b = (32 + M/32 + 8) U.  The dropout STORE takes the keep mask of
  ops.dropout_mask and one more rounding for the scale (+ 2 U).
Cross-entropy (CE_STATS -> ce_finish -> CE_GRAD).  Every logit z_j carries delta_j <= (K + 8) UTC absref_j.
  lse = m + log(sum_j exp(z_j - m)) moves by at most max_j delta_j; the exponent arguments z log2e - m log2e are
  formed with three fp32 roundings, <= 5 U max|z| in natural units; ex2.approx.ftz has <= 2 ulp relative error
  (2^-22, PTX ISA) at two sites, expf <= 2 ulp at two sites, logf <= 1 ulp of |log s| <= 16: 2^-19 covers them all;
  the partial sums are n_parts / 8 long per finishing warp plus 16-long chunk chains and the merges: (n_parts/8 + 40) U
  relative, and the final add 4 U |lse|:
      eps_lse = max_j delta_j + 5 U max|z| + 2^-19 + (n_parts/8 + 40) U + 4 U |lse|.
  loss_rows = lse - z_label adds delta_label + 2 U |loss|.  dlogits_j = alpha (p_j - [j = label]) with the kernel's lse:
      |err| <= 1.01 alpha p_j (delta_j + eps_lse + eps_exp_j) + U alpha (p_j + [j = label]) + half a bf16 ulp,
  eps_exp_j = 2^-21 + 5 U (|z_j| + |lse|) + 2 U |ln alpha| (ex2.approx, the folded log2f(alpha), the fma).  Padding
  columns must be exactly 0.  loss_sum adds the row bounds plus (T/32 + 48) U sum|loss|.
Causal attention.  Logit s_ij = scale q_i.k_j carries eps_s = (dh + 8) UTC scale |q_i|.|k_j| + 3 U (|s_ij| + |m_i|)
  (the wgmma sum, the fp32 scale * log2e product and the subtraction of the running max m); eps_row = max_j eps_s.
  lse: eps_lse = eps_row + (S + 32) U + (nblk + 4) 2^-21 + 2 U |lse| (the sum of S exp2f terms of 2 ulp each and one
  rescale per 64-key block).  O = sum_j bf16(p_j) v_j / l: b = 2^-8 (P rounded to bf16 before PV) + 2 eps_row +
  (2 nblk + 2) 2^-21 + (2 S + 2 nblk + 32) UTC on absref = P |V|.  Backward, with delta = rowsum(dO * O) of the
  kernel's own bf16 O (the operand the kernel uses): dS = P (dP - delta), absref |dS| <= P (|dO||V|^T +
  rowsum(|dO||O|)), dQ = scale dS K, dK = scale dS^T Q, dV = P^T dO on the matching |.| graphs, and
  b = max(eps_s + eps_lse) + 2^-20 + 2^-8 (P or dS rounded to bf16) + (S + dh + 24) UTC.  Dropout multiplies P by
  the keep mask * scale in every graph (+ 2 U).  A case with one key above the others gives every other key the same
  weight c, chosen at 0.85 ulp inside a bf16 interval: the reference rounds that P to bf16 exactly as RNE does, so the
  2^-8 term drops out, and values v_0 that cancel the rest make some outputs small: a truncating P is caught there.
  attn_decode: the same bound on one query row (P rounded to bf16; __expf has 2 + 1.17 |arg| ulp, within
  3 U (|s| + |m|) + 2^-20).
LayerNorm.  mean: the sum chain of d/32 (+ 16 tree) terms, dm <= (d/32 + 16) U mean|x| + U |mean|.  var (two-pass:
  the mean error enters squared): eps_v = (d/32 + 24) U + dm^2 / (var + eps), rsqrtf 2 ulp, eps_r = eps_v / 2 + 2^-22 +
  2 U.  y: |g| rstd dm + |g| |xhat| (eps_r + 4 U) + 2 U |b| + half a bf16 ulp.  Backward on the kernel's mean / rstd:
  dx absref = rstd (|t| + mean|t| + |xhat| mean|t xhat|) + |dres| with t = dy g, b = (d/32 + 24) U.  dg / db / dxsum
  accumulate rows_per_chain rows per thread, then the block tree and the grid partials in order: gamma_n with
  n = rows_per_chain + grid + 16.
Embedding.  The forward is exact: bf16 RNE of the exact wte[id] + wpe[s].  dwte: runs of equal ids inside 32-token
  strips are summed in fp32 (<= 31 U of their absolute sum), each run is rounded to the 2^-40 fixed-point grid
  (<= 2^-41 each: count * 2^-41 with count the number of runs that hit the row) and the total is cast and added in
  fp32 (a = 2 U).  dwpe: B - 1 fp32 adds onto the base.
Adam.  Restated in float64 from oracle/optim.py with the kernel's fp32 constants.  The clip factor has 5 fp32
  roundings, g_s 6 U; m' = b1 m + (1 - b1) g_s within 9 U (b1 |m| + (1 - b1) |g_s|); v' within 16 U v'; the
  denominator sqrt(v') + eps within 10 U; the update lr (m'/den + wd p) within lr (20 U mA / den + 2 U wd |p|) +
  3 U |update| + U |p'| (the rounding of p' itself).  The bf16 shadow is bf16 RNE of the new p, bit for bit.

Shapes come from the engine: a recorder wraps ops.gemm / attn_* / layernorm_* / embed_* while a one-layer DalleEngine
of each configuration runs forward + backward + logits() at S = 1280 (the product shapes do not depend on the layer
count), and every distinct call is replayed at the tokens-per-GPU of the configuration with fresh operands.
"""
import functools
import json
import math
import os
import types

import pytest
import torch

import float64_bounds
from float64_bounds import DEV, U, UTC, nan_like

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = "dalle-kernels"
check = functools.partial(float64_bounds.check, tag=TAG)
UBF = 2.0 ** -8
SLAB = 1 << 26                      # float64 elements per comparison slab (512 MiB per tensor)

# config -> tokens per GPU of the replay (dalle_example: the bench shape)
CONFIGS = {"dalle_example_b200": 40960, "dalle_coco_b200": 20480, "dalle_12b_b200": 5120}
# split-K wgrads (M, N) whose work-tile count does not depend on T and stays below 2 x SM on a 132-SM H100
WGRAD_EXCEPTIONS = {
    "dalle_example_b200": {(512, 1536), (512, 512), (512, 2048), (2048, 512)},
    "dalle_coco_b200": {(1024, 3072), (1024, 1024), (1024, 4096), (4096, 1024)},
    "dalle_12b_b200": set(),
}


_PEAK = [0]


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    yield _ops
    print(f"[{TAG}] peak device memory of the module {_PEAK[0] / 2 ** 30:.1f} GiB")


@pytest.fixture(autouse=True)
def _peak_memory(request):
    """The comparisons run in row slabs so that no case needs more than a fraction of the device (shared machines)."""
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: peak device memory {peak / 2 ** 30:.1f} GiB")


def _sm():
    return float64_bounds.sm_count()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, g, scale=1.0, dtype=F32):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _config(name):
    with open(os.path.join(ROOT, "configs", name + ".json")) as f:
        return json.load(f)


def _slabs(rows, cols):
    step = max(1, SLAB // max(cols, 1))
    return [(r, min(rows, r + step)) for r in range(0, rows, step)]


class Worst:
    """Worst err/bound of one case over several slabs; report() prints the case line and asserts r < 1."""

    def __init__(self, name):
        self.name, self.r = name, 0.0

    def add(self, got, ref, absref, **kw):
        self.r = max(self.r, float64_bounds.worst_ratio(self.name, got, ref, absref, **kw))

    def report(self):
        return float64_bounds.report(self.name, self.r, TAG)


def bf16_rne(x):
    """bf16 round-to-nearest-even of float64 x in one rounding (x -> fp32 -> bf16 would round twice)."""
    x32 = x.float()
    inexact = x32.double() != x
    mid = (x32.view(I32) & 0xFFFF) == 0x8000          # the fp32 value sits on a bf16 midpoint
    toward = torch.where(x > x32.double(), torch.full_like(x32, math.inf), torch.full_like(x32, -math.inf))
    x32 = torch.where(inexact & mid, torch.nextafter(x32, toward), x32)
    return x32.to(BF16)


def synthetic_tokens(cfg, B, g):
    """Captions as the synthetic input pipeline makes them (5..64 ids, right-padded with one id to 256) followed by
    image codes offset by the text vocabulary."""
    from dalle_mtf_b200.input_fns import synthetic_captions
    tv, iv = cfg["text_vocab_size"], cfg["image_vocab_size"]
    cap = synthetic_captions(B, 256, 50257, torch.Generator().manual_seed(B), vocab=min(50257, tv)).to(DEV)
    img = torch.randint(tv, tv + iv, (B, 1024), generator=g, device=DEV, dtype=I32)
    return torch.cat([cap, img], 1).contiguous()


# ------------------------------------------------------------------------------------------------------- recorder
RECORDED = ("gemm", "attn_fwd", "attn_bwd", "layernorm_fwd", "layernorm_bwd", "embed_fwd", "embed_bwd")
_RECORDS = {}


def _describe(name, args, kw):
    if name == "gemm":
        M, N, K = args[3:6]
        out = args[2]
        return ("gemm", M, N, K, bool(kw.get("a_mn")), bool(kw.get("b_mn")), int(kw.get("mode", 0)),
                None if out is None else str(out.dtype), kw.get("bias") is not None, bool(kw.get("relu")),
                kw.get("residual") is not None, kw.get("aux") is not None, int(kw.get("split_k", 1)),
                int(kw.get("n_valid", 0)), kw.get("colsum") is not None, kw.get("dropout") is not None)
    if name in ("attn_fwd", "attn_bwd"):
        B, S, H, dh = args[3:7] if name == "attn_fwd" else args[7:11]
        scale = args[7] if name == "attn_fwd" and len(args) > 7 else (args[11] if len(args) > 11 else kw["scale"])
        return (name, B, S, H, dh, float(scale), kw.get("dropout") is not None, kw.get("radius"), kw.get("axial"),
                kw.get("conv"))
    if name == "layernorm_fwd":
        return (name,) + tuple(args[0].shape)
    if name == "layernorm_bwd":
        return (name,) + tuple(args[1].shape) + (args[5] is not None, kw.get("dxsum") is not None,
                                                  kw.get("dropout") is not None)
    ids = args[0]
    return (name,) + tuple(ids.shape) + (kw.get("wte_drop") is not None,)


def engine_calls(ops, config, step=None, **engine_kw):
    """Distinct kernel calls of one forward + backward + logits() of a one-layer DalleEngine of `config` at B = 1,
    S = 1280, and the standard deviation of the gradient that reaches the embedding.  engine_kw go to the engine
    (attention_types, local_attention_radius, dropout rates); step goes to forward() (dropout runs with a step)."""
    key = (config, step, repr(sorted(engine_kw.items())))
    if key in _RECORDS:
        return _RECORDS[key]
    from dalle_mtf_b200.dalle_engine import DalleEngine
    cfg = _config(config)
    eng = DalleEngine(cfg["n_embd"], 1, cfg["n_heads"], cfg["text_vocab_size"], cfg["image_vocab_size"], 256, 1024,
                      **engine_kw)
    eng.init_params(seed=1)
    seen, extra = {}, {}
    orig = {n: getattr(ops, n) for n in RECORDED}

    def wrap(n):
        def rec(*args, **kw):
            seen.setdefault(_describe(n, args, kw), None)
            if n == "embed_bwd":
                extra["dx_std"] = float(args[1].float().std())
            return orig[n](*args, **kw)
        return rec

    try:
        for n in RECORDED:
            setattr(ops, n, wrap(n))
        tokens = synthetic_tokens(cfg, 1, _gen(1))
        eng.zero_grads()
        eng.forward(tokens, step=step)
        eng.backward(1.0 / tokens.numel())
        eng.logits(tokens)
        torch.cuda.synchronize()
    finally:
        for n in RECORDED:
            setattr(ops, n, orig[n])
    res = (list(seen), extra, eng.V, eng.Vpad, eng.S)
    del eng
    torch.cuda.empty_cache()
    _RECORDS[key] = res
    return res


# ------------------------------------------------------------------------------------------------------- GEMM
def gemm_splits(M, N, K, mode, split_k, sm):
    """gemm.cu gemm_splits: the K slices of an ATOMIC product (1 otherwise)."""
    from dalle_mtf_b200 import lib as L
    if mode != L.EPI_ATOMIC:
        return 1
    kb = -(-K // 64)
    s = split_k
    if s <= 0:
        s = sm // max(1, -(-M // 128) * -(-N // 128))
        s = min(s, kb // 4)
        s = max(s, 1)
    s = max(1, min(s, kb))
    per = -(-kb // s)
    return -(-kb // per)


def _mode_name(mode):
    from dalle_mtf_b200 import lib as L
    return {L.EPI_STORE: "STORE", L.EPI_ATOMIC: "ATOMIC", L.EPI_RELU_BWD: "RELU_BWD", L.EPI_CE_STATS: "CE_STATS",
            L.EPI_CE_GRAD: "CE_GRAD"}[mode]


def gemm_case_name(desc, M, N, K, splits, tiles, dropout=None, tag=""):
    from dalle_mtf_b200 import lib as L
    (_, _, _, _, a_mn, b_mn, mode, out_dt, has_bias, relu, has_res, _, _, _, has_colsum, _) = desc
    return f"{tag}{_mode_name(mode)} {M}x{N}x{K} aT={int(a_mn)} bT={int(b_mn)}" + \
        "".join(f" {f}" for f, on in (("bias", has_bias), ("relu", relu), ("res", has_res), ("colsum", has_colsum),
                                      ("f32", out_dt == "torch.float32" and mode == L.EPI_STORE),
                                      ("dropout", dropout is not None)) if on) + f" splits={splits} tiles={tiles}"


def gemm_operands(ops, desc, M, K, seed, dropout=None):
    """Fresh operands of the recorded product `desc` at M rows and depth K: bf16 A and B (B at K^-1/2, so products
    are O(1)), the epilogue inputs the recorded call had, the output NaN-filled (ATOMIC: a random base, also kept in
    `base`), and the dropout keep mask.  Fields as check_gemm reads them."""
    from dalle_mtf_b200 import lib as L
    (_, _, N, _, a_mn, b_mn, mode, out_dt, has_bias, relu, has_res, has_aux, split_k, _, has_colsum, _) = desc
    g = _gen(seed)
    o = types.SimpleNamespace(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, mode=mode, relu=relu, split_k=split_k,
                              dropout=dropout)
    o.a = _randn(*((K, M) if a_mn else (M, K)), g=g, dtype=BF16)
    o.b = _randn(*((K, N) if b_mn else (N, K)), g=g, scale=K ** -0.5, dtype=BF16)
    o.bias = _randn(N, g=g, scale=0.1) if has_bias else None
    o.res = _randn(M, N, g=g, dtype=BF16) if has_res else None
    o.aux = _randn(M, N, g=g, dtype=BF16) if has_aux else None
    o.cs_base = _randn(N, g=g, scale=math.sqrt(M)) if has_colsum else None
    o.colsum = o.cs_base.clone() if has_colsum else None
    if mode == L.EPI_ATOMIC:
        o.base = _randn(M, N, g=g)
        o.out = o.base.clone()
    else:
        o.base = None
        o.out = nan_like((M, N), F32 if out_dt == "torch.float32" else BF16)
    o.keep = None
    if dropout is not None:
        o.keep = torch.empty(M, N, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(dropout, L.DROPOUT_ELEMENTWISE, (M, N), o.keep)
    return o


def run_gemm(ops, o):
    ops.gemm(o.a, o.b, o.out, o.M, o.N, o.K, a_mn=o.a_mn, b_mn=o.b_mn, mode=o.mode, bias=o.bias, relu=o.relu,
             residual=o.res, aux=o.aux, split_k=o.split_k, colsum=o.colsum, dropout=o.dropout)


def check_gemm(name, o, splits, report=True):
    """o.out (and o.colsum) against float64 on the operands in o (fields of gemm_operands; keep / base / cs_base None
    where the call had none), in slabs.  report=False returns the worst err/bound of o.out without printing or
    asserting, for callers that gather many calls into one case line."""
    M, N, K = o.M, o.N, o.K
    A = o.a.t() if o.a_mn else o.a                   # [M, K]
    Bm = o.b if o.b_mn else o.b.t()                  # [K, N]
    bias, res, aux, base, keep, out = o.bias, o.res, o.aux, o.base, o.keep, o.out
    has_colsum = o.cs_base is not None
    w = Worst(name)
    bnd = (K + 8 + splits) * UTC
    cs_ref, cs_abs = (o.cs_base.to(F64), o.cs_base.to(F64).abs()) if has_colsum else (None, None)
    bf = out.dtype == BF16
    for c0, c1 in _slabs(N, K):                      # column slabs of B, row slabs of A: float64 tiles <= SLAB
        B64 = Bm[:, c0:c1].to(F64)
        Ba = B64.abs()
        for r0, r1 in _slabs(M, max(c1 - c0, K)):
            A64 = A[r0:r1].to(F64)
            ref, absref = A64 @ B64, A64.abs() @ Ba
            if bias is not None:
                ref, absref = ref + bias[c0:c1].to(F64), absref + bias[c0:c1].abs().to(F64)
            if o.relu:
                ref = ref.clamp_min(0)
            if keep is not None:
                kk = keep[r0:r1, c0:c1].to(F64) * o.dropout.scale
                ref, absref = ref * kk, absref * kk
            if res is not None:
                ref, absref = ref + res[r0:r1, c0:c1].to(F64), absref + res[r0:r1, c0:c1].abs().to(F64)
            if aux is not None:
                m = (aux[r0:r1, c0:c1] > 0).to(F64)
                ref, absref = ref * m, absref * m
            if base is not None:
                ref, absref = ref + base[r0:r1, c0:c1].to(F64), absref + base[r0:r1, c0:c1].abs().to(F64)
            w.add(out[r0:r1, c0:c1], ref, absref, a=2 * U, b=bnd + (2 * U if keep is not None else 0.0), bf16_out=bf)
            if has_colsum:
                o64 = out[r0:r1, c0:c1].to(F64)
                cs_ref[c0:c1] += o64.sum(0)
                cs_abs[c0:c1] += o64.abs().sum(0)
            del ref, absref, A64
        del B64, Ba
    if not report:
        return w.r
    r = w.report()
    if has_colsum:
        r = max(r, check(name + " colsum", o.colsum, cs_ref, cs_abs, a=0.0, b=(32 + M / 32 + 8) * U))
    return r


def run_gemm_case(ops, desc, T_rec, T, seed, dropout=None, tag=""):
    """Replay one recorded product with T tokens: fresh operands, NaN-filled or based outputs, float64 reference."""
    (_, M, N, K, _, _, mode, _, _, _, _, _, split_k, _, _, _) = desc
    M, K = (T if M == T_rec else M), (T if K == T_rec else K)
    splits = gemm_splits(M, N, K, mode, split_k, _sm())
    tiles = -(-M // 128) * -(-N // 128) * splits
    o = gemm_operands(ops, desc, M, K, seed, dropout)
    run_gemm(ops, o)
    return check_gemm(gemm_case_name(desc, M, N, K, splits, tiles, dropout, tag), o, splits), tiles, (M, N)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_gemm_products_of_the_engine(ops, config):
    from dalle_mtf_b200 import lib as L
    calls, _, V, Vpad, S = engine_calls(ops, config)
    T_rec, T = S, CONFIGS[config]
    gemms = [c for c in calls if c[0] == "gemm"]
    assert len(gemms) == 17, gemms                   # 12 per layer + CE_STATS, CE_GRAD, wout dgrad / wgrad, logits()
    modes = [c[6] for c in gemms]
    assert modes.count(L.EPI_ATOMIC) == 5 and modes.count(L.EPI_RELU_BWD) == 1
    assert modes.count(L.EPI_CE_STATS) == 1 and modes.count(L.EPI_CE_GRAD) == 1
    sm = _sm()
    worst = 0.0
    for i, desc in enumerate(gemms):
        if desc[6] in (L.EPI_CE_STATS, L.EPI_CE_GRAD):
            continue                                   # test_cross_entropy_at_the_real_vocabulary
        r, tiles, (M, N) = run_gemm_case(ops, desc, T_rec, T, seed=i, tag=f"{config} ")
        worst = max(worst, r)
        if tiles < 2 * sm:
            assert desc[6] == L.EPI_ATOMIC and (M, N) in WGRAD_EXCEPTIONS[config], (desc, tiles)
            print(f"[{TAG}] {config} wgrad {M}x{N}: {tiles} work tiles at any T (below 2 x {sm} SMs)")
    # residual dropout on the STORE epilogue, once per configuration: the wo product (bias + residual)
    wo = [c for c in gemms if c[6] == L.EPI_STORE and c[10] and c[3] == c[2] == _config(config)["n_embd"]]
    assert len(wo) == 1
    drop = L.make_dropout(0.1, 7, 3, L.dropout_site_attn_out(0), 0)
    r, _, _ = run_gemm_case(ops, wo[0], T_rec, T, seed=99, dropout=drop, tag=f"{config} ")
    print(f"[{TAG}] {config} GEMM: worst err/bound {max(worst, r):.4f}")


# ------------------------------------------------------------------------------------------------------- cross-entropy
def run_cross_entropy(ops, tag, T, K, V, Vpad, *, labels, h, W, bias, n_valid=None, alpha=None, colsum=True, dl=None):
    """CE_STATS -> ce_finish -> CE_GRAD as the engine runs them, checked per element in row slabs.  dl: the NaN-filled
    [T, Vpad] bf16 gradient to write (default: a fresh one), for callers that read it afterwards."""
    from dalle_mtf_b200 import lib as L
    n_valid = V if n_valid is None else n_valid
    alpha = 1.0 / T if alpha is None else alpha
    nt = ops.ce_tiles(Vpad)
    pm, ps = nan_like((nt, T), F32), nan_like((nt, T), F32)
    ll, lse, lr = nan_like((T,), F32), nan_like((T,), F32), nan_like((T,), F32)
    lsum_base = 0.75
    lsum = torch.full((1,), lsum_base, device=DEV)
    ops.gemm(h, W, None, T, Vpad, K, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS, bias=bias, labels=labels,
             part_max=pm, part_sum=ps, label_logit=ll, n_valid=n_valid)
    ops.ce_finish(pm, ps, ll, lse, lr, lsum)
    del pm, ps
    dl = nan_like((T, Vpad), BF16) if dl is None else dl
    cs_base = torch.randn(Vpad, generator=_gen(T + Vpad), device=DEV) * 1e-3 if colsum else None
    cs = cs_base.clone() if colsum else None
    ops.gemm(h, W, dl, T, Vpad, K, a_mn=False, b_mn=True, mode=L.EPI_CE_GRAD, alpha=alpha, bias=bias, labels=labels,
             lse=lse, n_valid=n_valid, colsum=cs)
    W64 = W[:, :n_valid].to(F64)
    Wa = W64.abs()
    b64 = bias[:n_valid].to(F64)
    al = float(torch.tensor(alpha, dtype=F32))
    names = ("lse", "label_logit", "loss_rows", "dlogits")
    ws = {n: Worst(f"{tag} {n}") for n in names}
    loss_ref, loss_abs, loss_bnd = 0.0, 0.0, 0.0
    cs_ref = cs_base.to(F64) if colsum else None
    cs_abs = cs_base.abs().to(F64) if colsum else None
    pad_ok = True
    for r0, r1 in _slabs(T, Vpad):
        h64 = h[r0:r1].to(F64)
        z = h64 @ W64 + b64
        za = h64.abs() @ Wa + b64.abs()
        delta = (K + 8) * UTC * za
        lse_ref = torch.logsumexp(z, 1)
        zmax = z.abs().max(1).values
        eps_lse = delta.max(1).values + 5 * U * zmax + 2.0 ** -19 + (nt / 8 + 40) * U + 4 * U * lse_ref.abs()
        ws["lse"].add(lse[r0:r1], lse_ref, eps_lse, a=0.0, b=1.0)
        lab = labels[r0:r1].long()
        zl = z.gather(1, lab[:, None])[:, 0]
        dll = delta.gather(1, lab[:, None])[:, 0]
        ws["label_logit"].add(ll[r0:r1], zl, dll, a=U, b=1.0)
        loss = lse_ref - zl
        lb = eps_lse + dll + 2 * U * loss.abs()
        ws["loss_rows"].add(lr[r0:r1], loss, lb, a=0.0, b=1.0)
        loss_ref += loss.sum().item()
        loss_abs += loss.abs().sum().item()
        loss_bnd += lb.sum().item()
        p = torch.exp(z - lse_ref[:, None])
        onehot = torch.zeros_like(p).scatter_(1, lab[:, None], 1.0)
        ref = al * (p - onehot)
        eps_exp = 2.0 ** -21 + 5 * U * (z.abs() + lse_ref.abs()[:, None]) + 2 * U * abs(math.log(al))
        acc = 1.01 * al * p * (delta + eps_lse[:, None] + eps_exp) + U * al * (p + onehot)
        ws["dlogits"].add(dl[r0:r1, :n_valid], ref, acc, b=1.0, bf16_out=True, floor=2.0 ** -126)
        pad_ok &= bool((dl[r0:r1, n_valid:] == 0).all())
        if colsum:
            o64 = dl[r0:r1].to(F64)
            cs_ref, cs_abs = cs_ref + o64.sum(0), cs_abs + o64.abs().sum(0)
        del z, za, delta, p, onehot, ref, acc, eps_exp, h64
    worst = max(w.report() for w in ws.values())
    assert pad_ok, f"{tag}: padding columns of dlogits are not exactly 0"
    worst = max(worst, check(f"{tag} loss_sum", lsum, torch.tensor([lsum_base + loss_ref], dtype=F64, device=DEV),
                             torch.tensor([lsum_base + loss_abs], dtype=F64, device=DEV), a=0.0,
                             b=(T / 32 + 48) * U, floor=loss_bnd))
    if colsum:
        worst = max(worst, check(f"{tag} dbias colsum", cs, cs_ref, cs_abs, a=0.0, b=(32 + T / 32 + 8) * U))
    return worst


def ce_operands(T, K, V, Vpad, g, *, dominate_cols=(), bias_scale=0.1):
    """LayerNorm-output-like h, wout at its init scale (pad columns 0), a non-zero bias.  Rows r = 5 (mod 97) get a
    one-hot selector in the first 16 features, which meet a weight of 100 in the column they select: that logit then
    dominates the row by > 90 (every other p underflows)."""
    h = _randn(T, K, g=g)
    W = torch.zeros(K, Vpad, device=DEV)
    W[:, :V] = torch.randn(K, V, generator=g, device=DEV) * 0.02
    bias = torch.zeros(Vpad, device=DEV)
    bias[:V] = torch.randn(V, generator=g, device=DEV) * bias_scale
    sel_rows = torch.arange(5, T, 97, device=DEV)
    cols = list(dominate_cols)
    if cols:
        h[:, :len(cols)] = 0
        c = torch.arange(sel_rows.numel(), device=DEV) % len(cols)
        h[sel_rows, c] = 1.0
        for i, j in enumerate(cols):
            W[i, j] = 100.0
    return h.to(BF16), W.to(BF16), bias, sel_rows, cols


@pytest.mark.parametrize("config", list(CONFIGS))
def test_cross_entropy_at_the_real_vocabulary(ops, config):
    """The vocabulary head at each configuration's V / Vpad and width: labels from the engine's shift_labels (EOS = V-1
    closes every sequence, in the last, ragged vocabulary tile), labels 0 and at tile boundaries, rows that one logit
    dominates (also at EOS and in the last half tile), a non-zero bias.  dalle_coco runs T = 40 960 rows, so dlogits
    has more than 2^31 elements."""
    T = 40960 if config == "dalle_coco_b200" else CONFIGS[config]
    if config == "dalle_coco_b200":
        assert T * engine_calls(ops, config)[3] > 2 ** 31
    real_vocabulary_cross_entropy(ops, config, T)


def real_vocabulary_cross_entropy(ops, config, T):
    """run_cross_entropy at the configuration's V / Vpad / width with T rows (see the test above)."""
    K, V, Vpad, h, W, bias, labels = real_vocabulary_operands(ops, config, T)
    return run_cross_entropy(ops, f"{config} CE T={T} V={V}", T, K, V, Vpad, labels=labels, h=h, W=W, bias=bias)


def real_vocabulary_operands(ops, config, T):
    """(K, V, Vpad, h, W, bias, labels) of the vocabulary head of `config` with T rows: ce_operands with dominating
    logits at the edge columns, labels of the engine's shift_labels with edge columns on every 101st row."""
    cfg = _config(config)
    calls, _, V, Vpad, S = engine_calls(ops, config)
    assert any(c[0] == "gemm" and c[13] == V for c in calls)          # the engine's n_valid is V
    K = cfg["n_embd"]
    g = _gen(Vpad + T)
    last = (V - 1) // 128 * 128
    edge = sorted({0, 1, 63, 64, 127, 128, V // 2, last - 1, last, last + 63, last + 64, V - 20, V - 19, V - 2, V - 1,
                   (V - 1) // 64 * 64})
    edge = [j for j in edge if 0 <= j < V][:16]
    h, W, bias, sel_rows, cols = ce_operands(T, K, V, Vpad, g, dominate_cols=edge)
    tokens = synthetic_tokens(cfg, T // S, g)
    labels = torch.empty_like(tokens)
    ops.shift_labels(tokens, labels, V - 1)
    labels = labels.view(T)
    assert (labels.view(-1, S)[:, -1] == V - 1).all()
    rows = torch.arange(7, T, 101, device=DEV)
    labels[rows] = torch.tensor(edge, dtype=I32, device=DEV)[torch.arange(rows.numel(), device=DEV) % len(edge)]
    labels[sel_rows] = torch.tensor(cols, dtype=I32, device=DEV)[torch.arange(sel_rows.numel(), device=DEV) % len(cols)]
    return K, V, Vpad, h, W, bias, labels.contiguous()


@pytest.mark.parametrize("n_valid", [130, 1, 200])
def test_cross_entropy_abi_edges(ops, n_valid):
    """n_valid the engine cannot produce: 130 of 256 columns leave the whole half tile [192, 256) padded, 1 leaves a
    single valid column; ce_finish then merges (-inf, 0) partials.  Rows with h = 0 and no bias have all logits
    equal; rows with a dominating logit as above."""
    T, K, Vpad = 3000, 128, 256
    g = _gen(n_valid)
    h, W, bias, sel_rows, cols = ce_operands(T, K, n_valid, Vpad, g, dominate_cols=[0, n_valid - 1])
    bias.zero_()
    h[100:300] = 0                                            # every logit of these rows equal
    labels = torch.randint(0, n_valid, (T,), generator=g, device=DEV, dtype=I32)
    labels[sel_rows] = torch.tensor(cols, dtype=I32, device=DEV)[torch.arange(sel_rows.numel(), device=DEV) % 2]
    run_cross_entropy(ops, f"CE edge n_valid={n_valid}", T, K, n_valid, Vpad, labels=labels, h=h, W=W, bias=bias)


# ------------------------------------------------------------------------------------------------------- attention
def attn_reference(q, k, v, do, o, scale, keep=None, kscale=1.0):
    """float64 causal attention forward / backward and the |.| graphs on [B, S, H, dh] operands (o: the kernel's
    output, used in delta as the kernel uses it).  Returns dicts of ref, abs and the per-row exponent errors.
    do = None: the forward only (O and lse; b_bwd is None)."""
    q, k, v = (t.to(F64).permute(0, 2, 1, 3) for t in (q, k, v))                    # [B, H, S, dh]
    S, dh = q.shape[2], q.shape[3]
    mask = torch.ones(S, S, dtype=torch.bool, device=DEV).tril()
    s = scale * q @ k.transpose(-1, -2)
    sa = scale * q.abs() @ k.abs().transpose(-1, -2)
    s = s.masked_fill(~mask, -math.inf)
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    m = s.max(-1).values
    eps_s = ((dh + 8) * UTC * sa + 3 * U * (s.abs() + m.abs()[..., None])).masked_fill(~mask, 0)
    eps_row = eps_s.max(-1).values
    nblk = -(-S // 64)
    eps_lse = eps_row + (S + 32) * U + (nblk + 4) * 2.0 ** -21 + 2 * U * lse.abs()
    Pk = P if keep is None else P * keep.to(F64) * kscale
    out = {"O": (Pk @ v, Pk @ v.abs()), "lse": (lse, eps_lse)}
    b_fwd = UBF + 2 * eps_row + (2 * nblk + 2) * 2.0 ** -21 + (2 * S + 2 * nblk + 32) * UTC
    b_bwd = None
    if do is not None:
        do, o = do.to(F64).permute(0, 2, 1, 3), o.to(F64).permute(0, 2, 1, 3)
        dP = do @ v.transpose(-1, -2)
        dPa = do.abs() @ v.abs().transpose(-1, -2)
        if keep is not None:
            dP, dPa = dP * keep.to(F64) * kscale, dPa * keep.to(F64) * kscale
        delta = (do * o).sum(-1, keepdim=True)
        deltaa = (do * o).abs().sum(-1, keepdim=True)
        dS = P * (dP - delta)
        dSa = P * (dPa + deltaa)
        out["dQ"] = (scale * dS @ k, scale * dSa @ k.abs())
        out["dK"] = (scale * dS.transpose(-1, -2) @ q, scale * dSa.transpose(-1, -2) @ q.abs())
        out["dV"] = (Pk.transpose(-1, -2) @ do, Pk.transpose(-1, -2) @ do.abs())
        b_bwd = (eps_s + eps_lse[..., None]).masked_fill(~mask, 0).max().item() + 2.0 ** -20 + UBF + \
            (S + dh + 24) * UTC
    out = {n: (r.permute(0, 2, 1, 3) if r.dim() == 4 else r, a.permute(0, 2, 1, 3) if a.dim() == 4 else a)
           for n, (r, a) in out.items()}
    return out, b_fwd.permute(0, 2, 1)[..., None], b_bwd


def check_attention(tag, B, S, H, dh, scale, qkv, out, lse, dout=None, dqkv=None, *, keep_all=None, kscale=1.0,
                    chunk=None, report=True):
    """out / lse (and dqkv when dout is given) of attn_fwd / attn_bwd on the [B, S, 3, H, dh] operands qkv against
    float64, in chunks of sequences; keep_all: the [B, H, S, S] dropout keep mask (kscale its fp32 scale).
    report=False returns {name: worst err/bound} without printing or asserting."""
    extra = 2 * U if keep_all is not None else 0.0
    chunk = chunk or max(1, 16 // H)
    names = ("O", "lse") + (("dQ", "dK", "dV") if dout is not None else ())
    ws = {n: Worst(f"{tag} {n}") for n in names}
    for b0 in range(0, B, chunk):
        b1 = min(B, b0 + chunk)
        q, k, v = qkv[b0:b1, :, 0], qkv[b0:b1, :, 1], qkv[b0:b1, :, 2]
        keep = keep_all[b0:b1] if keep_all is not None else None
        do = dout[b0:b1] if dout is not None else None
        refs, b_fwd, b_bwd = attn_reference(q, k, v, do, out[b0:b1], scale, keep, kscale)
        ref, absref = refs["O"]
        ws["O"].add(out[b0:b1], ref, absref, b=b_fwd + extra, bf16_out=True, floor=2.0 ** -120)
        ref, bnd = refs["lse"]
        ws["lse"].add(lse[b0:b1], ref, bnd, a=0.0, b=1.0)
        if dout is not None:
            for i, n in enumerate(("dQ", "dK", "dV")):
                ref, absref = refs[n]
                ws[n].add(dqkv[b0:b1, :, i], ref, absref, b=b_bwd + extra, bf16_out=True, floor=2.0 ** -120)
        del refs
    if not report:
        return {n: w.r for n, w in ws.items()}
    return max(w.report() for w in ws.values())


def run_attention(ops, tag, B, S, H, dh, scale, qkv, dout, *, dropout=None, chunk=None):
    """attn_fwd + attn_bwd on [B, S, 3, H, dh] bf16 operands, checked in chunks of sequences."""
    from dalle_mtf_b200 import lib as L
    out = nan_like((B, S, H, dh), BF16)
    lse = nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, scale, dropout=dropout)
    dqkv = nan_like((B, S, 3, H, dh), BF16)
    ops.attn_bwd(qkv, out, dout, lse, torch.zeros(1, device=DEV), nan_like((B, H, S), F32), dqkv, B, S, H, dh, scale,
                 dropout=dropout)
    keep_all = None
    if dropout is not None:
        keep_all = torch.empty(B, H, S, S, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(dropout, L.DROPOUT_ATTENTION, (B, H, S), keep_all)
    kscale = float(torch.tensor(dropout.scale, dtype=F32)) if dropout is not None else 1.0
    return check_attention(tag, B, S, H, dh, scale, qkv, out, lse, dout, dqkv, keep_all=keep_all, kscale=kscale,
                           chunk=chunk)


def _qkv(B, S, H, dh, g, mag=1.0):
    """q, k at a spread that gives logits of a few units (scale 1, as the engine's attn_scale), v and dO N(0, 1)."""
    qkv = torch.randn(B, S, 3, H, dh, generator=g, device=DEV)
    qkv[:, :, :2] *= mag * 1.3 * dh ** -0.25
    return qkv.to(BF16), _randn(B, S, H, dh, g=g, dtype=BF16)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_attention_at_the_engine_shapes(ops, config):
    calls, _, _, _, S = engine_calls(ops, config)
    att = [c for c in calls if c[0] in ("attn_fwd", "attn_bwd")]
    assert {c[0] for c in att} == {"attn_fwd", "attn_bwd"} and len({c[1:] for c in att}) == 1
    _, _, S_, H, dh, scale, dropout, radius, axial, conv = att[0]
    # the configurations' engines run causal attention: no window, no axial and no conv geometry
    assert not dropout and radius is None and axial is None and conv is None
    B = CONFIGS[config] // S
    qkv, dout = _qkv(B, S, H, dh, _gen(B * H))
    run_attention(ops, f"{config} attention B={B} S={S} H={H} dh={dh}", B, S, H, dh, scale, qkv, dout)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("S", [1, 63, 65, 1279])
def test_attention_ragged_lengths(ops, S, dh):
    qkv, dout = _qkv(2, S, 2, dh, _gen(S + dh))
    run_attention(ops, f"attention S={S} dh={dh}", 2, S, 2, dh, 1.0, qkv, dout)


@pytest.mark.parametrize("dh", [64, 128])
def test_attention_edge_inputs(ops, dh):
    B, S, H = 2, 1280, 2
    g = _gen(dh)
    # large-magnitude rows: logits of tens of units, most keys underflow
    qkv, dout = _qkv(B, S, H, dh, g, mag=6.0)
    run_attention(ops, f"attention large logits dh={dh}", B, S, H, dh, 1.0, qkv, dout)
    # constant keys: uniform P over the visible keys
    qkv, dout = _qkv(B, S, H, dh, g)
    qkv[:, :, 1] = qkv[:, :1, 1]
    run_attention(ops, f"attention constant keys dh={dh}", B, S, H, dh, 1.0, qkv, dout)
    # one key (position 0) dominates every row by ~40
    qkv, dout = _qkv(B, S, H, dh, g)
    qkv[:, :, 0, :, 0] = 4.0
    qkv[:, :, 1, :, 0] = 0.0
    qkv[:, 0, 1, :, 0] = 10.0
    run_attention(ops, f"attention dominating key dh={dh}", B, S, H, dh, 1.0, qkv, dout)


@pytest.mark.parametrize("dh,H", [(64, 16), (128, 4)])
def test_attention_dropout(ops, dh, H):
    from dalle_mtf_b200 import lib as L
    B, S = 2, 1280
    qkv, dout = _qkv(B, S, H, dh, _gen(dh + 1))
    drop = L.make_dropout(0.1, 5, 11, L.dropout_site_attn(0), 3)
    run_attention(ops, f"attention dropout dh={dh} H={H}", B, S, H, dh, 1.0, qkv, dout, dropout=drop)


def _exact_p_weight():
    """A bf16 logit gap D whose weight c = exp(-D) lies 0.8-0.9 ulp into its bf16 interval: bf16 RNE rounds it up by
    ~0.15 ulp, truncation down by ~0.85 ulp, and no fp32 error of the kernel can move it across the midpoint."""
    for i in range(4000):
        D = torch.tensor(0.2 + i * 1e-4, dtype=F64).to(BF16).to(F64)
        c = torch.exp(-D)
        ulp = 2.0 ** (math.floor(math.log2(c.item())) - 7)
        frac = (c.item() % ulp) / ulp
        if 0.8 < frac < 0.9:
            return D.item(), c.item()
    raise AssertionError("no suitable gap")


@pytest.mark.parametrize("dh", [64, 128])
def test_attention_forward_rounds_p_to_nearest(ops, dh):
    """Key 0 is above every other key by D, so every other weight is the same c (the running max is key 0 from the
    first block on).  The reference rounds c to bf16 with RNE, as the kernel must; v_0 = -n_e c_bf16 in column e makes
    row n_e's output cancel to ~0, where a P rounded any other way is far outside the bound."""
    B, S, H = 1, 1280, 2
    D, c = _exact_p_weight()
    qkv = torch.zeros(B, S, 3, H, dh, device=DEV)
    qkv[:, :, 0, :, 0] = 1.0
    qkv[:, 1:, 1, :, 0] = -D
    qkv[:, 1:, 2] = 1.0
    cb = torch.tensor(c, dtype=F64).to(BF16).to(F64).item()
    n_e = torch.arange(dh, device=DEV) * ((S - 2) // dh) + 1
    qkv[:, 0, 2, :, :] = -(n_e * cb).float()
    qkv = qkv.to(BF16)
    out = nan_like((B, S, H, dh), BF16)
    lse = nan_like((B, H, S), F32)
    ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0)
    v = qkv[:, :, 2].to(F64).permute(0, 2, 1, 3)
    pos = torch.arange(S, device=DEV)
    pu = torch.where(pos == 0, torch.tensor(1.0, dtype=F64, device=DEV), torch.tensor(c, dtype=F64, device=DEV))
    p_bf = bf16_rne(pu).to(F64)
    assert (p_bf[1:] == cb).all() and cb > c
    mask = torch.ones(S, S, dtype=torch.bool, device=DEV).tril()
    Pn = torch.where(mask, p_bf[None, :], torch.zeros((), dtype=F64, device=DEV))
    tot = torch.where(mask, pu[None, :], torch.zeros((), dtype=F64, device=DEV)).sum(-1, keepdim=True)
    ref = (Pn @ v) / tot
    absref = (Pn @ v.abs()) / tot
    b = (S + 16) * U + 2.0 ** -20 + 6 * U * D + (2 * S + 64) * UTC
    check(f"attention P rounded to nearest dh={dh}", out, ref.permute(0, 2, 1, 3), absref.permute(0, 2, 1, 3), b=b,
          bf16_out=True)


@pytest.mark.parametrize("dh", [64, 128])
def test_attn_decode(ops, dh):
    """One decoding step at S = 1280 over a filled cache: the new k, v are appended at pos, then the query attends to
    keys <= pos.  Same bound as the forward (P rounded to bf16, __expf), checked at the last position and a middle one."""
    B, S, H = 4, 1280, 1024 // dh
    g = _gen(dh + 7)
    for pos in (S - 1, 700):
        kc, vc = _randn(B, S, H, dh, g=g, scale=1.3 * dh ** -0.25, dtype=BF16), _randn(B, S, H, dh, g=g, dtype=BF16)
        step = _randn(B, 3, H, dh, g=g, dtype=BF16)
        step[:, :2] = (step[:, :2].float() * 1.3 * dh ** -0.25).to(BF16)
        out = nan_like((B, H, dh), BF16)
        ops.attn_decode(step, kc, vc, out, pos, 1.0)
        assert torch.equal(kc[:, pos], step[:, 1]) and torch.equal(vc[:, pos], step[:, 2])
        ref, absref, b = attn_decode_reference(step[:, 0], kc[:, :pos + 1], vc[:, :pos + 1], 1.0)
        check(f"attn_decode dh={dh} pos={pos}", out, ref, absref, b=b, bf16_out=True)


def attn_decode_reference(q, k, v, scale):
    """float64 softmax_j(scale q.k_j) v_j of q [B, H, dh] over the keys k, v [B, n, H, dh], its |.| graph and the b of
    the attn_decode bound (module docstring) per (b, h): ref, absref [B, H, dh] and b [B, H, 1]."""
    dh = q.shape[-1]
    q = q.to(F64)
    k = k.to(F64).permute(0, 2, 1, 3)                         # [B, H, n, dh]
    v = v.to(F64).permute(0, 2, 1, 3)
    s = scale * (k @ q[..., None])[..., 0]
    sa = abs(scale) * (k.abs() @ q.abs()[..., None])[..., 0]
    P = torch.softmax(s, -1)
    eps = ((dh + 8) * U * sa + 3 * U * (s.abs() + s.max(-1, keepdim=True).values.abs())).max(-1).values
    n = k.shape[2]
    b = UBF + 2 * eps + 2.0 ** -20 + (n / 8 + 40) * U
    return (P[..., None, :] @ v)[..., 0, :], (P[..., None, :] @ v.abs())[..., 0, :], b[..., None]


# ------------------------------------------------------------------------------------------------------- LayerNorm
def ln_inputs(rows, d, g):
    """Residual-stream-like rows N(0, 1), rows with |mean| >> std (64 + N(0, 0.5)) and constant rows."""
    x = torch.randn(rows, d, generator=g, device=DEV)
    x[1::7] = 64 + torch.randn(x[1::7].shape, generator=g, device=DEV) * 0.5
    x[3::97] = torch.randn(x[3::97].shape[0], 1, generator=g, device=DEV)
    return x.to(BF16)


def ln_operands(rows, d, g):
    """ln_inputs rows, gamma 1 + N(0, 0.1), beta N(0, 0.1)."""
    x = ln_inputs(rows, d, g)
    gam = 1 + torch.randn(d, generator=g, device=DEV) * 0.1
    bet = torch.randn(d, generator=g, device=DEV) * 0.1
    return x, gam, bet


def check_layernorm_fwd(tag, x, gam, bet, y, mean, rstd, eps, report=True):
    """y / mean / rstd of layernorm_fwd on x [rows, d] against float64 (the LayerNorm bound), in row slabs.
    report=False returns {name: worst err/bound} without printing or asserting."""
    rows, d = x.shape
    g64, b64 = gam.to(F64), bet.to(F64)
    ws = {n: Worst(f"{tag} {n}") for n in ("y", "mean", "rstd")}
    for r0, r1 in _slabs(rows, d):
        x64 = x[r0:r1].to(F64)
        mu = x64.mean(1, keepdim=True)
        var = ((x64 - mu) ** 2).mean(1, keepdim=True)
        r = 1 / torch.sqrt(var + eps)
        dm = (d / 32 + 16) * U * x64.abs().mean(1, keepdim=True) + U * mu.abs()
        eps_r = ((d / 32 + 24) * U * var + dm ** 2) / (var + eps) / 2 + 2.0 ** -22 + 2 * U
        xh = (x64 - mu) * r
        ws["mean"].add(mean[r0:r1], mu[:, 0], dm[:, 0], a=0.0, b=1.0)
        ws["rstd"].add(rstd[r0:r1], r[:, 0], (eps_r * r)[:, 0], a=0.0, b=1.0)
        ws["y"].add(y[r0:r1], xh * g64 + b64, g64.abs() * r * dm + g64.abs() * xh.abs() * (eps_r + 4 * U)
                    + 2 * U * b64.abs(), b=1.0, bf16_out=True)
        del x64, mu, var, r, dm, eps_r, xh
    if not report:
        return {n: w.r for n, w in ws.items()}
    return max(w.report() for w in ws.values())


def run_layernorm(ops, tag, rows, d, *, dres=True, dxsum=True, dropout=None, seed=0):
    from dalle_mtf_b200 import lib as L
    g = _gen(seed)
    eps = 1e-5
    x, gam, bet = ln_operands(rows, d, g)
    y, mean, rstd = nan_like((rows, d), BF16), nan_like((rows,), F32), nan_like((rows,), F32)
    ops.layernorm_fwd(x, gam, bet, y, mean, rstd, eps)
    worst = check_layernorm_fwd(tag, x, gam, bet, y, mean, rstd, eps)
    dy = _randn(rows, d, g=g, dtype=BF16)
    dr = _randn(rows, d, g=g, dtype=BF16) if dres else None
    dx = nan_like((rows, d), BF16)
    dxm = nan_like((rows, d), BF16) if dropout is not None else None
    base = [_randn(d, g=g, scale=math.sqrt(rows)) for _ in range(3)]
    dg, db = base[0].clone(), base[1].clone()
    dxs = base[2].clone() if dxsum else None
    ops.layernorm_bwd(dy, x, gam, mean, rstd, dr, dx, dg, db, dxsum=dxs, dxm=dxm, dropout=dropout)
    keep = None
    if dropout is not None:
        keep = torch.empty(rows, d, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(dropout, L.DROPOUT_ELEMENTWISE, (rows, d), keep)
    grid = min(rows if d == 4096 else -(-rows // 4), 4 * _sm())
    chain = -(-rows // grid) if d == 4096 else -(-rows // (4 * grid))
    n_acc = chain + grid + 16
    gam_n = n_acc * U / (1 - n_acc * U)
    g64 = gam.to(F64)
    names = ["dx"] + (["dxm"] if dropout is not None else [])
    ws = {n: Worst(f"{tag} {n}") for n in names}
    sums = {n: [bb.to(F64), bb.abs().to(F64)] for n, bb in zip(("dg", "db", "dxsum"), base)}
    for r0, r1 in _slabs(rows, d):
        x64 = x[r0:r1].to(F64)
        # backward on the kernel's own statistics
        m32, r32 = mean[r0:r1, None].to(F64), rstd[r0:r1, None].to(F64)
        h = (x64 - m32) * r32
        dy64 = dy[r0:r1].to(F64)
        t = dy64 * g64
        c1, c2 = t.mean(1, keepdim=True), (t * h).mean(1, keepdim=True)
        ref = (t - c1 - h * c2) * r32
        absref = r32 * (t.abs() + t.abs().mean(1, keepdim=True) + h.abs() * (t * h).abs().mean(1, keepdim=True))
        if dr is not None:
            ref, absref = ref + dr[r0:r1].to(F64), absref + dr[r0:r1].abs().to(F64)
        ws["dx"].add(dx[r0:r1], ref, absref, b=(d / 32 + 24) * U, bf16_out=True)
        got = dx[r0:r1].to(F64)
        if keep is not None:
            km = keep[r0:r1].to(F64) * float(torch.tensor(dropout.scale, dtype=F32))
            ws["dxm"].add(dxm[r0:r1], got * km, got.abs() * km, b=2 * U, bf16_out=True)
            got = dxm[r0:r1].to(F64)
        for n, v, va in (("dg", (dy64 * h).sum(0), (dy64 * h).abs().sum(0)), ("db", dy64.sum(0), dy64.abs().sum(0)),
                         ("dxsum", got.sum(0), got.abs().sum(0))):
            sums[n][0] += v
            sums[n][1] += va
    worst = max([worst] + [w.report() for w in ws.values()])
    for n, t in (("dg", dg), ("db", db), ("dxsum", dxs)):
        if t is not None:
            worst = max(worst, check(f"{tag} {n}", t, sums[n][0], sums[n][1], a=0.0, b=gam_n + 4 * U))
    return worst


@pytest.mark.parametrize("config", list(CONFIGS))
def test_layernorm_at_the_engine_shapes(ops, config):
    calls, _, _, _, S = engine_calls(ops, config)
    d = _config(config)["n_embd"]
    fw = {c for c in calls if c[0] == "layernorm_fwd"}
    bw = {c for c in calls if c[0] == "layernorm_bwd"}
    assert fw == {("layernorm_fwd", S, d)}
    assert ("layernorm_bwd", S, d, True, True, False) in bw and ("layernorm_bwd", S, d, False, True, False) in bw
    rows = CONFIGS[config]
    kind = "wide" if d == 4096 else "warp"
    run_layernorm(ops, f"{config} LN {kind} rows={rows} d={d} +dres", rows, d, seed=d)
    run_layernorm(ops, f"{config} LN {kind} rows={rows} d={d} no dres", rows, d, dres=False, seed=d + 1)


@pytest.mark.parametrize("d", [512, 1024, 4096])
def test_layernorm_backward_with_residual_dropout(ops, d):
    from dalle_mtf_b200 import lib as L
    drop = L.make_dropout(0.1, 9, 4, L.dropout_site_mlp_out(0), 1280)
    run_layernorm(ops, f"LN dropout rows=5120 d={d}", 5120, d, dropout=drop, seed=d + 2)


# ------------------------------------------------------------------------------------------------------- embedding
def fixed_point_runs(ids, V):
    """Number of 2^-40 fixed-point additions that reach each wte row: one per run of equal ids inside a 32-token strip
    (rowops.cu embed_bwd_wte_kernel)."""
    flat = ids.reshape(-1).long()
    t = torch.arange(flat.numel(), device=DEV)
    start = (t % 32 == 0) | torch.cat([torch.ones(1, dtype=torch.bool, device=DEV), flat[1:] != flat[:-1]])
    return torch.bincount(flat[start], minlength=V)


def run_embedding(ops, tag, ids, V, d, dx_scale, g, wte_drop=None, wpe_drop=None):
    """embed_fwd / embed_bwd against float64.  With the dropout descriptors (both or neither) every term carries its
    keep mask * scale: the forward is then a bound (one fp32 rounding per product and one for the sum, then bf16)
    instead of bit for bit, and the backward adds one rounding per masked gradient element (+ U)."""
    from dalle_mtf_b200 import lib as L
    B, S = ids.shape
    wte = _randn(V, d, g=g, scale=0.02, dtype=BF16)
    wpe = _randn(S, d, g=g, scale=0.01, dtype=BF16)
    mt = mp = None
    if wte_drop is not None:
        mt = torch.empty(B * S, d, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(wte_drop, L.DROPOUT_ELEMENTWISE, (B * S, d), mt)
        mp = torch.empty(S, d, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(wpe_drop, L.DROPOUT_ELEMENTWISE, (S, d), mp)
        mt = mt.view(B, S, d).to(F64) * _f32(wte_drop.scale)
        mp = mp.to(F64) * _f32(wpe_drop.scale)
    out = nan_like((B, S, d), BF16)
    ops.embed_fwd(ids, wte, wpe, out, wte_drop=wte_drop, wpe_drop=wpe_drop)
    if mt is None:
        for b0 in range(0, B, 8):
            ref = wte.to(F64)[ids[b0:b0 + 8].long()] + wpe.to(F64)[None]
            assert torch.equal(out[b0:b0 + 8].view(torch.int16), bf16_rne(ref).view(torch.int16)), f"{tag} forward"
        print(f"{float64_bounds.prefix()}[{TAG}] {tag} embed_fwd: bf16 RNE of the exact sum, bit for bit "
              "(worst err/bound 0)")
    else:
        a, p = wte.to(F64)[ids.long()] * mt, wpe.to(F64)[None] * mp[None]
        check(f"{tag} embed_fwd", out, a + p, a.abs() + p.abs(), b=2 * U, bf16_out=True)
    dx = _randn(B, S, d, g=g, scale=dx_scale, dtype=BF16)
    base_t = _randn(V, d, g=g, scale=dx_scale)
    base_p = _randn(S, d, g=g, scale=dx_scale)
    dwte, dwpe = base_t.clone(), base_p.clone()
    ops.embed_bwd(ids, dx, dwte, dwpe, wte_drop=wte_drop, wpe_drop=wpe_drop)
    flat = ids.reshape(-1).long()
    dx2 = (dx.to(F64) * (1.0 if mt is None else mt)).reshape(-1, d)
    runs = fixed_point_runs(ids, V).to(F64)
    share = torch.zeros(V, dtype=F64, device=DEV)        # the fixed-point term's share of the bound, per row
    b_run = (31 if mt is None else 32) * U
    w = Worst(f"{tag} dwte")
    for v0, v1 in _slabs(V, d):
        sel = (flat >= v0) & (flat < v1)
        idx, rows = flat[sel] - v0, dx2[sel]
        ref = base_t[v0:v1].to(F64).index_add_(0, idx, rows)
        absref = base_t[v0:v1].abs().to(F64).index_add_(0, idx, rows.abs())
        fixed = runs[v0:v1, None] * 2.0 ** -41
        w.add(dwte[v0:v1], ref, absref, a=2 * U, b=b_run, floor=fixed)
        fp32 = (b_run * absref + 2 * U * ref.abs()).mean(1)
        share[v0:v1] = fixed[:, 0] / (fixed[:, 0] + fp32).clamp_min(1e-300)
        del ref, absref, rows
    r = w.report()
    pad = int(torch.bincount(flat, minlength=V).argmax())
    touched = runs > 0
    print(f"{float64_bounds.prefix()}[{TAG}] {tag} dwte: fixed-point term {share[pad].item():.4f} of the bound at "
          f"the padding row ({int(runs[pad])} runs, {int((flat == pad).sum())} tokens), "
          f"median {share[touched].median().item():.4f}, max {share.max().item():.4f} over the {int(touched.sum())} "
          "rows hit")
    dref = base_p.to(F64) + dx.to(F64).sum(0) * (1.0 if mp is None else mp)
    dabs = base_p.abs().to(F64) + dx.to(F64).abs().sum(0) * (1.0 if mp is None else mp)
    r = max(r, check(f"{tag} dwpe", dwpe, dref, dabs, a=2 * U, b=(B + 2 + (mp is not None)) * U))
    return r


@pytest.mark.parametrize("config", list(CONFIGS))
def test_embedding_at_the_real_vocabulary(ops, config):
    """The synthetic input's token distribution (one padding id fills most of every caption) at the real (V, d): with
    gradients at the scale the engine produces at this T (the recorded embedding gradient, rescaled by the tokens of
    the recording over T through grad_scale = 1/T), and N(0, 1)."""
    cfg = _config(config)
    calls, extra, V, _, S = engine_calls(ops, config)
    d, T = cfg["n_embd"], CONFIGS[config]
    assert ("embed_fwd", 1, S, False) in calls and ("embed_bwd", 1, S, False) in calls
    g = _gen(V + T)
    ids = synthetic_tokens(cfg, T // S, g)
    scale = extra["dx_std"] * S / T
    print(f"[{TAG}] {config}: engine embedding gradient std {scale:.3g} at T={T}")
    run_embedding(ops, f"{config} embedding T={T} grad std {scale:.2g}", ids, V, d, scale, g)
    run_embedding(ops, f"{config} embedding T={T} grad N(0,1)", ids, V, d, 1.0, g)


# ------------------------------------------------------------------------------------------------------- optimiser
def _f32(x):
    return float(torch.tensor(x, dtype=F32))


def check_adam_update(tag, inputs, outputs, lr, b1, b2, eps, wd, clip, gscale, bc, step):
    """One db200_adam_step against the float64 restatement of oracle/optim.py (adam_mtf_step / adam_tf_step,
    clip_by_global_norm) on the kernel's fp32 constants, with the bounds of the module docstring.  inputs = (p, m, v,
    g, gnorm_sq) as the kernel read them (gnorm_sq unused without clipping), outputs = (p', m', v', bf16 shadow) as it
    wrote them.  Returns whether the clip scaled the gradient down."""
    p, m, v, gr, gn = inputs
    pd, md, vd, p16 = outputs
    B1, B2, EPS, LR, WD, CL, GS = map(_f32, (b1, b2, eps, lr, wd, clip, gscale))
    gmul, clipped = GS, False
    if clip:
        gnorm = math.sqrt(float(gn)) * GS
        gmul = GS * CL / max(gnorm, CL)
        clipped = gnorm > CL
    gs = gr.to(F64) * gmul
    m2 = B1 * m.to(F64) + _f32(1 - B1) * gs
    mA = B1 * m.to(F64).abs() + _f32(1 - B1) * gs.abs()
    v2 = B2 * v.to(F64) + _f32(1 - B2) * gs * gs
    den = torch.sqrt(v2) + EPS
    lr_eff = _f32(LR * math.sqrt(1 - B2 ** step) / (1 - B1 ** step)) if bc else LR
    upd = m2 / den + (WD * p.to(F64) if wd else 0.0)
    ref_u = -lr_eff * upd
    p_new = p.to(F64) + ref_u
    check(f"adam m ({tag})", md, m2, mA, a=0.0, b=9 * U)
    check(f"adam v ({tag})", vd, v2, v2, a=0.0, b=16 * U)
    check(f"adam update p'-p ({tag})", pd.to(F64) - p.to(F64), ref_u,
          lr_eff * (mA / den + WD * p.to(F64).abs()), a=3 * U, b=20 * U, floor=U * p_new.abs())
    assert torch.equal(p16.view(torch.int16), pd.to(BF16).view(torch.int16)), "bf16 shadow is not RNE of the new p"
    return clipped


@pytest.mark.parametrize("case", ["clip active", "clip inactive", "bias correction", "weight decay", "zero_grad"])
def test_sqnorm_and_adam_update(ops, case):
    n = 1_000_003
    g = _gen(len(case))
    sign = lambda: torch.where(torch.rand(n, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    logu = lambda lo, hi: torch.exp(torch.empty(n, device=DEV).uniform_(math.log(lo), math.log(hi), generator=g))
    p = torch.randn(n, generator=g, device=DEV) * 0.05
    gr = sign() * logu(1e-8, 1e-3)
    m = sign() * logu(1e-9, 1e-4)
    v = logu(1e-18, 1e-8)                              # sqrt(v) from 1e-9 to 1e-4: eps = 1e-6 matters
    lr, b1, b2, eps, wd, clip, gscale, bc, step = 1e-3, 0.9, 0.999, 1e-6, 0.0, 0.0, 1.0, False, 0
    if case == "clip active":
        clip = 0.05
    elif case == "clip inactive":
        clip = 10.0
    elif case == "bias correction":
        bc, step, eps, gscale = True, 3, 1e-8, 0.5
    elif case == "weight decay":
        wd, clip = 0.01, 1.0
    gn_base = 1e-3
    gn = torch.full((1,), gn_base, device=DEV)
    ops.sqnorm(gr, gn)
    sq = gn_base + (gr.to(F64) ** 2).sum()
    blocks = min(-(-(n // 4) // 256), 8 * _sm())
    depth = 4 * -(-(n // 4) // (blocks * 256)) + 5 + 8 + blocks + 8
    check(f"sqnorm n={n} ({case})", gn, sq.reshape(1), sq.reshape(1), a=0.0, b=depth * U)
    pd, md, vd, gd = p.clone(), m.clone(), v.clone(), gr.clone()
    p16 = nan_like((n,), BF16)
    ops.adam_step(pd, md, vd, gd, p16, lr, b1, b2, eps, wd, gn if clip else None, clip, gscale, bc, step,
                  zero_grad=case == "zero_grad")
    clipped = check_adam_update(case, (p, m, v, gr, gn), (pd, md, vd, p16), lr, b1, b2, eps, wd, clip, gscale, bc,
                                step)
    assert clipped == (case == "clip active")
    if case == "zero_grad":
        assert (gd == 0).all()
    else:
        assert torch.equal(gd, gr)
