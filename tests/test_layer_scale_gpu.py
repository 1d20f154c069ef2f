"""LayerScale and the stable option on the GPU: db200_layer_scale_residual_fwd, db200_layernorm_scale_residual_fwd,
db200_layer_scale_bwd, db200_layernorm_divmax_fwd / _bwd and db200_embed_bwd_scaled against float64 at the
dalle_example, dalle_coco and 12B widths (with and without dropout and the sandwich LayerNorm, DivideMax rows where
the division matters and with tied maxima, bit-reproducible, the dropout mask the existing sites draw); the engine
against oracle/dalle_layer_scale.py (loss, logits, every gradient including both scales and the embedding tables, one
Adam update) with the oracle's mutants failing the same bounds; reproducibility, in-process ranks, ZeRO-1, decoding,
the prefill, guidance, checkpoints, generate_dalle.py and the launches with the keys off."""
import math

import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro
from test_sandwich_norm_gpu import bf16_ulp

pytestmark = pytest.mark.gpu
BF16, F32, I32, F64 = torch.bfloat16, torch.float32, torch.int32, torch.float64
TAG = "layer_scale"


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def _rand(rows, d, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(rows, d, generator=g, device=DEV) * scale).to(BF16)


def _vec(d, seed, base=0.0, scale=0.3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(d, generator=g, device=DEV) * scale + base


def _within_ulp(y, y64, slack, what):
    """|y - y64| <= one bf16 ulp of y64 plus `slack` (the fp32 evaluation's own rounding)."""
    excess = ((y.double() - y64).abs() - bf16_ulp(y64) - slack).max().item()
    assert excess <= 0, (what, excess)


# ------------------------------------------------------------------------------------------------ kernels
WIDTHS = (512, 1024, 4096)                    # dalle_example, dalle_coco, 12B
SHAPES = [(rows, d) for d in WIDTHS for rows in (1, 37, 1000)] + [(40960, 512), (10240, 1024), (5120, 4096)]
IDS = [f"{r}x{d}" for r, d in SHAPES]


@pytest.mark.parametrize("rows,d", SHAPES, ids=IDS)
def test_residual_fwd_matches_float64(ops, rows, d):
    check_residual_fwd(ops, rows, d)


def check_residual_fwd(ops, rows, d):
    o, x, s = _rand(rows, d, 1), _rand(rows, d, 2, 4.0), _vec(d, 3, 0.1)
    y = torch.empty_like(o)
    ops.layer_scale_residual_fwd(o, x, s, y)
    y64 = x.double() + s.double() * o.double()
    _within_ulp(y, y64, 2 * 2.0 ** -24 * (x.double().abs() + (s.double() * o.double()).abs()), (rows, d))


@pytest.mark.parametrize("rows,d", SHAPES + [(37, w) for w in (256, 768, 2048)],
                         ids=IDS + [f"37x{w}" for w in (256, 768, 2048)])
def test_layernorm_scale_residual_fwd_matches_layernorm_and_float64(ops, rows, d):
    check_ln_scale_residual_fwd(ops, rows, d)


def check_ln_scale_residual_fwd(ops, rows, d):
    o, x = _rand(rows, d, 4, 2.0), _rand(rows, d, 5)
    g, b, s = _vec(d, 6, 1.0), _vec(d, 7), _vec(d, 8, 0.5)
    y, mean, rstd = torch.empty_like(o), torch.empty(rows, dtype=F32, device=DEV), torch.empty(rows, dtype=F32,
                                                                                                device=DEV)
    ops.layernorm_scale_residual_fwd(o, x, g, b, s, y, mean, rstd)
    y0, mean0, rstd0 = torch.empty_like(o), torch.empty_like(mean), torch.empty_like(rstd)
    ops.layernorm_fwd(o, g, b, y0, mean0, rstd0)
    assert torch.equal(mean, mean0) and torch.equal(rstd, rstd0)
    n64 = (o.double() - mean.double()[:, None]) * rstd.double()[:, None] * g.double() + b.double()
    y64 = x.double() + s.double() * n64
    terms = ((o.double().abs() + mean.double().abs()[:, None]) * rstd.double()[:, None] * g.double().abs() +
             b.double().abs()) * s.double().abs()
    _within_ulp(y, y64, 4 * 2.0 ** -24 * (x.double().abs() + terms), (rows, d))


def _bwd64(dy, v, s, keep_scale=None, norm=None):
    """float64 reference of layer_scale_bwd: (dv before its bf16 rounding, ds, the scaled value v)."""
    v64 = v.double()
    if norm is not None:
        g, b, mean, rstd = norm
        v64 = (v64 - mean.double()[:, None]) * rstd.double()[:, None] * g.double() + b.double()
    dv = s.double() * dy.double()
    if keep_scale is not None:
        dv = dv * keep_scale
    return dv, (dy.double() * v64).sum(0), v64


def _check_bwd(ops, rows, d, drop=None, sandwich=False):
    from dalle_mtf_b200 import lib as L
    dy, o = _rand(rows, d, 11), _rand(rows, d, 12, 2.0)
    s = _vec(d, 13, 0.2)
    norm = None
    if sandwich:
        g, b = _vec(d, 14, 1.0), _vec(d, 15)
        mean, rstd = torch.empty(rows, dtype=F32, device=DEV), torch.empty(rows, dtype=F32, device=DEV)
        ops.layernorm_fwd(o, g, b, torch.empty_like(o), mean, rstd)
        norm = (g, b, mean, rstd)
    keep_scale = None
    if drop is not None:
        keep = torch.empty(rows, d, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(drop, L.DROPOUT_ELEMENTWISE, (rows, d), keep)
        keep_scale = keep.double() * drop.scale
    ds0, db0 = _vec(d, 16), _vec(d, 17)                       # both accumulate
    ds, db, dv = ds0.clone(), db0.clone(), torch.empty_like(dy)
    ops.layer_scale_bwd(dy, o, s, dv, ds, db=None if sandwich else db, dropout=drop, norm=norm)
    dv64, ds64, _ = _bwd64(dy, o, s, keep_scale, norm)
    _within_ulp(dv, dv64, 2 * 2.0 ** -24 * dv64.abs(), ("dv", rows, d))
    if drop is not None:
        assert torch.equal(dv == 0, (keep == 0) | (dy == 0)), "dropped entries"
    # fp32 sums over `rows` terms: error bounded by rows * eps * sum |terms| (a loose, order-free bound)
    vabs = o.double().abs()
    if sandwich:   # the fp32 recomputation of v rounds its terms, which can cancel
        vabs = (vabs + mean.double().abs()[:, None]) * rstd.double()[:, None] * g.double().abs() + b.double().abs()
    absterm = (dy.double().abs() * vabs).sum(0)
    assert ((ds.double() - ds0.double() - ds64).abs() <= (2 * rows + 8) * 2.0 ** -24 * absterm + 1e-6).all()
    if not sandwich:
        dbs = dv.double().sum(0)                                # the column sum of the stored bf16 values
        assert ((db.double() - db0.double() - dbs).abs() <= 2 * rows * 2.0 ** -24 * dv.double().abs().sum(0) +
                1e-6).all()
    else:
        assert torch.equal(db, db0)
    # bit-reproducible: the same call again
    ds2, db2, dv2 = ds0.clone(), db0.clone(), torch.empty_like(dy)
    ops.layer_scale_bwd(dy, o, s, dv2, ds2, db=None if sandwich else db2, dropout=drop, norm=norm)
    assert torch.equal(dv, dv2) and torch.equal(ds, ds2) and torch.equal(db, db2)


@pytest.mark.parametrize("rows,d", SHAPES, ids=IDS)
def test_bwd_matches_float64(ops, rows, d):
    _check_bwd(ops, rows, d)


@pytest.mark.parametrize("rows,d", [(37, 512), (1000, 1024), (40960, 512), (5120, 4096)])
def test_bwd_with_dropout_matches_float64_and_the_site_mask(ops, rows, d):
    from dalle_mtf_b200 import lib as L
    _check_bwd(ops, rows, d, drop=L.make_dropout(0.1, 5, 3, L.dropout_site_mlp_out(2), 0))


@pytest.mark.parametrize("rows,d", SHAPES, ids=IDS)
def test_bwd_sandwich_form_matches_float64(ops, rows, d):
    _check_bwd(ops, rows, d, sandwich=True)


def test_argument_checks(ops):
    from dalle_mtf_b200 import lib as L
    o, s = _rand(8, 512, 1), _vec(512, 2)
    with pytest.raises(L.DB200Error):
        ops.layer_scale_residual_fwd(o, o, s[:256], torch.empty_like(o))
    with pytest.raises(L.DB200Error):
        ops.layer_scale_residual_fwd(o, o[:4], s, torch.empty_like(o))
    with pytest.raises(L.DB200Error, match="multiple of 256"):
        x = _rand(8, 264, 1)
        ops.layer_scale_bwd(x, x, _vec(264, 3), torch.empty_like(x), _vec(264, 4))
    with pytest.raises(L.DB200Error, match="no dropout"):
        norm = (s, s, _vec(8, 5), _vec(8, 6))
        ops.layer_scale_bwd(o, o, s, torch.empty_like(o), s.clone(), dropout=L.make_dropout(0.1, 1, 1, 4, 0),
                            norm=norm)
    with pytest.raises(L.DB200Error, match="d=640"):
        x = _rand(8, 640, 1)
        v = _vec(640, 1)
        ops.layernorm_scale_residual_fwd(x, x, v, v, v, torch.empty_like(x), _vec(8, 1), _vec(8, 2))


# ------------------------------------------------------------------------------------------------ stable kernels
def _rows(kind, rows, d, seed):
    """bf16 rows: "random" N(0, 1); "c+100" / "c-100": +-100 + N(0, 0.3), where sigma / m is near sqrt(eps) and the
    division matters (a negative m flips the row); "tied": integers in [-3, 3], every row's maximum repeated."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "tied":
        return torch.randint(-3, 4, (rows, d), generator=g, device=DEV).to(BF16)
    c = {"random": 0.0, "c+100": 100.0, "c-100": -100.0}[kind]
    return (c + torch.randn(rows, d, generator=g, device=DEV) * (1.0 if c == 0 else 0.3)).to(BF16)


KINDS = ("random", "c+100", "c-100", "tied")
DM_SHAPES = [(rows, d) for d in WIDTHS for rows in (1, 37, 1000)] + [(37, w) for w in (256, 768, 2048)] + \
    [(40960, 512), (10240, 1024), (5120, 4096)]
DM_IDS = [f"{r}x{d}" for r, d in DM_SHAPES]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rows,d", DM_SHAPES, ids=DM_IDS)
def test_divmax_fwd_matches_float64(ops, rows, d, kind):
    check_divmax_fwd(ops, rows, d, kind)


def check_divmax_fwd(ops, rows, d, kind):
    x = _rows(kind, rows, d, 21)
    g, b = _vec(d, 22, 1.0), _vec(d, 23)
    y, mean, rstd, m = (torch.empty_like(x), *(torch.empty(rows, dtype=F32, device=DEV) for _ in range(3)))
    ops.layernorm_divmax_fwd(x, g, b, y, mean, rstd, m)
    assert torch.equal(m, x.float().amax(1))
    u64 = x.double() / m.double()[:, None]
    m64 = u64.mean(1)
    r64 = torch.rsqrt(((u64 - m64[:, None]) ** 2).mean(1) + 1e-5)
    assert (mean.double() - m64).abs().max().item() <= 1e-6 * (1 + m64.abs().max().item()), kind
    assert relfro(rstd, r64) < 1e-4, (kind, relfro(rstd, r64))
    # y from the kernel's statistics: one bf16 ulp plus the fp32 rounding of u = x / m and of the affine terms
    y64 = (u64 - mean.double()[:, None]) * rstd.double()[:, None] * g.double() + b.double()
    terms = (u64.abs() + mean.double().abs()[:, None]) * rstd.double()[:, None] * g.double().abs() + b.double().abs()
    _within_ulp(y, y64, 8 * 2.0 ** -24 * terms, (rows, d, kind))


def _divmax_bwd64(dy, x, g, m, detach=True):
    """float64 dx, dg, db of y = LN(x / m) g + b, m the row maximum (held constant unless detach=False)."""
    x64 = x.double().requires_grad_(True)
    g64 = g.double().requires_grad_(True)
    b64 = torch.zeros_like(g64, requires_grad=True)
    mm = m.double()[:, None] if detach else x64.amax(1, keepdim=True)
    u = x64 / mm
    mu = u.mean(1, keepdim=True)
    y = (u - mu) / torch.sqrt(((u - mu) ** 2).mean(1, keepdim=True) + 1e-5) * g64 + b64
    y.backward(dy.double())
    return x64.grad, g64.grad, b64.grad


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rows,d", [(37, w) for w in (256, 512, 768, 1024, 2048, 4096)] +
                         [(1000, 512), (40960, 512), (5120, 4096)])
def test_divmax_bwd_matches_float64_with_m_held_constant(ops, rows, d, kind):
    """dx = LN'(x / m)^T dy / m with the residual term, dg and db within fp32 sums of float64; against the gradient
    through the maximum (a mutant) the error at the rows' argmax is larger than the kernel's own error."""
    x, dy, dres = _rows(kind, rows, d, 31), _rand(rows, d, 32), _rand(rows, d, 33)
    g, b = _vec(d, 34, 1.0), _vec(d, 35)
    y, mean, rstd, m = (torch.empty_like(x), *(torch.empty(rows, dtype=F32, device=DEV) for _ in range(3)))
    ops.layernorm_divmax_fwd(x, g, b, y, mean, rstd, m)
    dx, dg, db = torch.empty_like(x), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    ops.layernorm_divmax_bwd(dy, x, g, mean, rstd, m, None, dx, dg, db)
    dx64, dg64, db64 = _divmax_bwd64(dy, x, g, m)
    assert relfro(dx, dx64) < 1e-2, (kind, relfro(dx, dx64))
    assert relfro(dg, dg64) < 1e-3 and relfro(db, db64) < 1e-4, (relfro(dg, dg64), relfro(db, db64))
    dxr = torch.empty_like(x)                            # the residual term is added before the one rounding
    ops.layernorm_divmax_bwd(dy, x, g, mean, rstd, m, dres, dxr, torch.zeros_like(dg), torch.zeros_like(db))
    assert ((dxr.double() - dres.double() - dx.double()).abs() <= bf16_ulp(dxr.double()) +
            bf16_ulp(dx.double())).all()
    if kind in ("c+100", "c-100") and rows <= 1000:      # the gradient through m moves the rows' argmax entries
        dx_thr = _divmax_bwd64(dy, x, g, m, detach=False)[0]
        am = x.float() == m[:, None]
        err = (dx.double() - dx64)[am].norm().item()
        err_thr = (dx.double() - dx_thr)[am].norm().item()
        assert err_thr > 2 * err, (err, err_thr)


@pytest.mark.parametrize("rows,d", [(37, 512), (1000, 1024), (40960, 512), (5120, 4096), (37, 2048)])
def test_divmax_bwd_keeps_the_dropout_and_bias_fusions(ops, rows, d):
    check_divmax_bwd_fusions(ops, rows, d)


def check_divmax_bwd_fusions(ops, rows, d):
    """With the last block's residual-dropout site: dxm = bf16(dx keep scale) bit for bit, dxsum = colsum(dxm) (the
    b2 gradient), dx as without dropout and within float64's bound; twice the same call gives the same bits."""
    from dalle_mtf_b200 import lib as L
    x, dy = _rows("c-100", rows, d, 41), _rand(rows, d, 42)
    g, b = _vec(d, 43, 1.0), _vec(d, 44)
    y, mean, rstd, m = (torch.empty_like(x), *(torch.empty(rows, dtype=F32, device=DEV) for _ in range(3)))
    ops.layernorm_divmax_fwd(x, g, b, y, mean, rstd, m)
    drop = L.make_dropout(0.1, 3, 5, L.dropout_site_mlp_out(5), 0)
    keep = torch.empty(rows, d, dtype=torch.uint8, device=DEV)
    ops.dropout_mask(drop, L.DROPOUT_ELEMENTWISE, (rows, d), keep)

    def run(dropout):
        dx, dxm = torch.empty_like(x), torch.empty_like(x)
        dg, db, dxs = (torch.zeros(d, device=DEV) for _ in range(3))
        ops.layernorm_divmax_bwd(dy, x, g, mean, rstd, m, None, dx, dg, db, dxsum=dxs,
                                 dxm=dxm if dropout else None, dropout=drop if dropout else None)
        return dx, dxm, dg, db, dxs
    dx0, _, dg0, db0, dxs0 = run(False)
    assert relfro(dx0, _divmax_bwd64(dy, x, g, m)[0]) < 1e-2
    dx, dxm, dg, db, dxs = run(True)
    assert torch.equal(dx, dx0) and torch.equal(dg, dg0) and torch.equal(db, db0)
    assert torch.equal(dxm, (dx.float() * (keep.float() * drop.scale)).to(BF16))
    assert relfro(dxs, dxm.double().sum(0)) < 1e-5 and relfro(dxs0, dx0.double().sum(0)) < 1e-5
    again = run(True)
    assert all(torch.equal(p, q) for p, q in zip(again, (dx, dxm, dg, db, dxs)))


def check_embed_bwd_scaled(ops, B, S, d, V, dropout, alpha=0.1):
    """embed_bwd with the gradient shrink against a float64 scatter-add of alpha dx (times the embedding dropout's
    keep masks): each bf16 dx element times alpha in fp32, runs of up to 32 tokens of one id summed in fp32 before the
    exact fixed-point sum (each add within 2^-24 of the run's sum of |terms|), the result rounded to fp32."""
    from dalle_mtf_b200 import lib as L
    g = torch.Generator(device=DEV).manual_seed(51)
    ids = torch.randint(0, V, (B, S), generator=g, device=DEV, dtype=I32)
    ids[:, 10:40] = min(7, V - 1)                       # runs of one id, as caption padding makes
    dx = _rand(B * S, d, 52).view(B, S, d)
    kw, mw, mp = {}, 1.0, 1.0
    if dropout:
        kw = dict(wte_drop=L.make_dropout(0.1, 1, 2, L.SITE_WTE, 0), wpe_drop=L.make_dropout(0.1, 1, 2, L.SITE_WPE, 0))
        kt = torch.empty(B * S, d, dtype=torch.uint8, device=DEV)
        kp = torch.empty(S, d, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(kw["wte_drop"], L.DROPOUT_ELEMENTWISE, (B * S, d), kt)
        ops.dropout_mask(kw["wpe_drop"], L.DROPOUT_ELEMENTWISE, (S, d), kp)
        mw, mp = kt.double() * kw["wte_drop"].scale, kp.double() * kw["wpe_drop"].scale
    dwte, dwpe = torch.zeros(V, d, device=DEV), torch.zeros(S, d, device=DEV)
    ops.embed_bwd(ids, dx, dwte, dwpe, alpha=alpha, **kw)
    a64 = alpha * dx.double().view(B * S, d)
    flat = ids.view(-1).long()
    want_te = torch.zeros(V, d, dtype=F64, device=DEV).index_add_(0, flat, a64 * mw)
    abs_te = torch.zeros(V, d, dtype=F64, device=DEV).index_add_(0, flat, (a64 * mw).abs())
    want_pe = a64.view(B, S, d).sum(0) * mp
    abs_pe = a64.abs().view(B, S, d).sum(0) * (mp if dropout else 1.0)
    for got, want, absum in ((dwte, want_te, abs_te), (dwpe, want_pe, abs_pe)):
        lim = 40 * 2.0 ** -24 * absum + 2.0 ** -24 * want.abs() + 1e-10
        assert ((got.double() - want).abs() <= lim).all()
        assert got.any()


@pytest.mark.parametrize("dropout", [False, True], ids=["plain", "dropout"])
@pytest.mark.parametrize("B,S,d,V", [(4, 1280, 512, 50771), (2, 1280, 1024, 58451), (1, 320, 4096, 1000)])
def test_embed_bwd_scaled_matches_a_float64_scatter_add(ops, B, S, d, V, dropout):
    check_embed_bwd_scaled(ops, B, S, d, V, dropout)


# ------------------------------------------------------------------------------------------------ engine vs oracle
VARIANTS = {
    "plain": dict(types=("global", "global")),
    "sandwich": dict(types=("global", "global"), sandwich_norm=True),
    "global_mlp": dict(types=("global", "mlp")),
    "global_mlp_sandwich": dict(types=("global", "mlp"), sandwich_norm=True),
    "dropout": dict(types=("global", "axial_row"), dropout=(0.1, 0.1, 0.2)),
    "dropout_sandwich": dict(types=("global", "global"), dropout=(0.1, 0.1, 0.2), sandwich_norm=True),
    "recompute": dict(types=("global", "mlp"), recompute_grad=True),
    "geglu_rotary_shift": dict(types=("global", "axial_col"), gated_mlp=True, activation="gelu", rotary_dim=32,
                               shift_tokens=True),
    # stable, with the last layer's b2 a large constant so that the division by the row maximum matters
    "stable_pos": dict(types=("global", "global"), layer_scale=None, stable=True, b2=60.0),
    "stable_neg": dict(types=("global", "global"), layer_scale=None, stable=True, b2=-60.0),
    "stable_dropout": dict(types=("global", "axial_row"), layer_scale=None, stable=True, b2=60.0,
                           dropout=(0.1, 0.1, 0.2)),
    "stable_recompute": dict(types=("global", "mlp"), layer_scale=None, stable=True, b2=-60.0, recompute_grad=True),
    "both": dict(types=("global", "mlp"), stable=True, b2=-60.0, sandwich_norm=True),
}
MUTANTS = {"plain": ("post_residual", "swapped"), "sandwich": ("post_residual", "swapped", "scale_before_norm"),
           "global_mlp": ("swapped",), "dropout": ("post_residual", "swapped"),
           "stable_pos": ("norm_then_divide", "no_shrink"), "stable_neg": ("max_abs", "norm_then_divide", "no_shrink"),
           "both": ("swapped", "no_shrink")}


def _model(types, seed=3, d=256, H=2, TL=28, W=10, sandwich=False, gated=False, b2=None):
    import axial_oracle as AX
    from oracle import dalle as O, dalle_glu as OGL, dalle_gmlp as OM, dalle_layer_scale as OLS
    from oracle import dalle_local as OL, dalle_sandwich as OSW
    cfg = OL.LocalConfig(d, len(types), H, 300, 64, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    tokens = O.assemble_tokens(torch.randint(0, 299, (2, TL), generator=g),
                               torch.randint(0, 64, (2, W * W), generator=g), 300)
    if sandwich:
        params = OSW.init_params(params, cfg, seed + 11)
    if gated:
        params = OGL.init_params(params, cfg, seed + 12)
    params = OLS.init_params(params, cfg, seed=seed + 13)
    if b2 is not None:
        params[f"layer_{len(types) - 1}/mlp/mlp_linear_2/bias"] = torch.full((d,), b2)
    return AX.AxialConfig(**{**cfg.__dict__}), params, tokens


def _vs_oracle(variant, adam=False, seed=3):
    import axial_oracle as AX
    from oracle import dalle_layer_scale as OLS
    v = {"layer_scale": True, **VARIANTS[variant]}
    types = v.pop("types")
    cfg, params, tokens = _model(types, seed, sandwich=v.get("sandwich_norm", False), gated=v.get("gated_mlp", False),
                                 b2=v.pop("b2", None))
    if not v["layer_scale"]:
        params = {k: x for k, x in params.items() if not k.endswith("/layer_scale")}
    kw = {"layers": AX, "layer_scale": bool(v["layer_scale"]), "sandwich_norm": v.get("sandwich_norm", False),
          "shift_tokens": v.get("shift_tokens", False), "stable": v.get("stable", False)}
    if v.get("gated_mlp"):
        kw.update(gated=True, activation="gelu", rotary=(v["rotary_dim"], 10000.0))
    dropout = (v["dropout"], 7, 3, 0) if "dropout" in v else None
    def oracle(bf16, m=None):
        which = "stable_mutate" if m in OLS.STABLE_MUTATIONS else "scale_mutate"
        return OLS.loss_and_grads(params, tokens, cfg, dropout=dropout, bf16=bf16, **{which: m}, **kw)
    loss32, rows32, logits32, g32 = oracle(False)
    loss16, rows16, logits16, g16 = oracle(True)
    eng = _engine(cfg, attention_types=list(types), conv_attention_kernel=3, dropout_seed=7, **v)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=3 if dropout else None)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    rows = eng._bufs["loss_rows"].view(2, -1).clone()
    grads = eng.export_params(eng.grads)
    assert set(params) == set(grads)

    # every bound: 1.25 x the bf16-policy oracle's own distance from the fp32 oracle, plus a floor
    loss_lim = 1.25 * abs(loss16.item() - loss32.item()) + 1e-3 * abs(loss32.item())
    rows_lim = 1.25 * relfro(rows16, rows32) + 5e-3

    def violations(l32, r32, gg32):
        bad = []
        if abs(loss - l32.item()) > loss_lim:
            bad.append(("loss", loss, l32.item()))
        if relfro(rows, r32) > rows_lim:
            bad.append(("loss_rows", relfro(rows, r32)))
        for k in gg32:
            if g32[k].any():
                lim = 1.25 * relfro(g16[k], g32[k]) + 1e-2
                if relfro(grads[k], gg32[k]) > lim:
                    bad.append((k, relfro(grads[k], gg32[k]), lim))
        return bad

    bad = violations(loss32, rows32, g32)
    print(f"[{TAG}] {variant}: loss {loss:.6f} oracle {loss32.item():.6f}, violations {bad}")
    assert not bad
    for name in OLS.scale_names(cfg) if kw["layer_scale"] else ():   # both scales of every layer trained
        assert grads[name].any(), name
    if not dropout:   # the logits within the gradients' bound
        e = relfro(eng.logits(tok), logits32)
        assert e <= 1.25 * relfro(logits16, logits32) + 1e-2, e
    for m in MUTANTS.get(variant, ()):
        ml, mr, _, mg = oracle(False, m)
        mbad = violations(ml, mr, mg)
        print(f"[{TAG}]   mutant {m}: {len(mbad)} violated bounds, e.g. {mbad[:2]}")
        assert mbad, m
    if adam:
        from oracle import optim as OO
        hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
        zeros = {k: torch.zeros_like(x) for k, x in params.items()}
        newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
        eng.optimizer_step(lr)
        torch.cuda.synchronize()
        assert abs(eng.gnorm_sq.sqrt().item() - gn.item()) <= 1e-4 * gn.item()
        after = eng.export_params()
        for k in params:
            if (newp[k] - params[k]).norm() > 0:
                assert relfro(after[k] - params[k], newp[k] - params[k]) <= 1e-3, k


def test_engine_matches_the_oracle_with_an_adam_step_and_not_its_mutants():
    _vs_oracle("plain", adam=True)


@pytest.mark.parametrize("variant", [v for v in VARIANTS if v != "plain"])
def test_engine_variants_match_the_oracle_and_not_its_mutants(variant):
    _vs_oracle(variant)


INPUT_VARIANTS = {
    "logits_mask_scale": dict(mask=True), "logits_mask_stable": dict(mask=True, ls=False, stable=True),
    "weighted_scale": dict(weights=((1.0, 7.0), 1e-4)), "weighted_stable": dict(weights=((1.0, 7.0), 1e-4), ls=False,
                                                                               stable=True),
    "row_col_scale": dict(row_col=True), "row_col_stable": dict(row_col=True, ls=False, stable=True),
}


@pytest.mark.parametrize("variant", list(INPUT_VARIANTS))
def test_engine_with_the_logits_mask_weighted_loss_and_row_col_positions_matches_the_oracle(variant):
    """The engine's objective and input-embedding variants against oracle/dalle_layer_scale.py through
    oracle/dalle_input.py and oracle/logits_mask.py, each with layer_scale and with stable (the last layer's b2 a large
    constant so that the division matters): loss, loss rows, logits and every gradient (image_row / image_col
    included: the gradient shrink passes through pos_fold) within the bounds of _vs_oracle, and the mutants failing
    them."""
    import conv_oracle as OC
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_input as I, dalle_layer_scale as OLS, logits_mask as OLM
    from test_parity_baseline_gpu import _randomise_small_params
    v = {"ls": True, "stable": False, "mask": False, "weights": None, "row_col": False, **INPUT_VARIANTS[variant]}
    B, seed, d, H, ts, W, tv, iv = 3, 2, 256, 2, 24, 8, 300, 64
    types = ["global", "global"]
    cfg = OC.ConvConfig(d, 2, H, tv, iv, ts, W * W, attention_types=tuple(types), local_attention_radius=8,
                        conv_attention_kernel=3)
    inp = I.InputConfig("row_col" if v["row_col"] else "absolute", False, None)
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    if v["ls"]:
        params = OLS.init_params(params, cfg, seed=seed + 13)
    if v["stable"]:
        params["layer_1/mlp/mlp_linear_2/bias"] = torch.full((d,), -60.0)
    tokens = I.assemble(torch.randint(0, tv - 1, (B, ts), generator=g), torch.randint(0, iv, (B, W * W), generator=g),
                        cfg, inp)
    off, _ = I.vocab(cfg, inp)
    w, z = v["weights"] if v["weights"] else (None, 0.0)

    def oracle(bf16, m=None):
        which = "stable_mutate" if m in OLS.STABLE_MUTATIONS else "scale_mutate"
        base = lambda p, t, c, dr, bf16=False, quirks=None: OLS.forward(  # noqa: E731
            p, t, c, dr, bf16=bf16, quirks=quirks, layers=OC, layer_scale=v["ls"], stable=v["stable"], **{which: m})
        if not v["mask"] and w is None:
            loss, rows, logits, grads = I.loss_and_grads(params, tokens, cfg, inp, None, bf16, base=base)
            return loss, rows, logits, grads
        fwd = lambda p, t: I.forward(p, t, cfg, inp, None, bf16, base=base)  # noqa: E731
        loss, rows, _, logits, grads = OLM.loss_and_grads(params, tokens, I._model_cfg(cfg, inp), off, weights=w, z=z,
                                                          forward=fwd, mask=v["mask"])
        return loss, rows, logits, grads

    loss32, rows32, logits32, g32 = oracle(False)
    loss16, rows16, logits16, g16 = oracle(True)
    kw = dict(loss_weights=w, z_loss=z) if w else {}
    eng = DalleEngine(d, 2, H, tv, iv, ts, W * W, attention_types=types,
                      image_position_embedding=inp.image_position_embedding, logits_mask=v["mask"],
                      layer_scale=True if v["ls"] else None, stable=v["stable"], **kw)
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok)
    if w:
        eng.backward(1.0)
        torch.cuda.synchronize()
        loss = acc[0].item()
    else:
        eng.backward(1.0 / T)
        torch.cuda.synchronize()
        loss = acc.item() / T
    rows = eng._bufs["loss_rows"].view(B, -1).clone()
    grads = eng.export_params(eng.grads)
    assert set(params) == set(grads)
    if v["row_col"]:
        assert grads["positional_embedding/image_row"].any() and grads["positional_embedding/image_col"].any()
    loss_lim = 1.25 * abs(loss16.item() - loss32.item()) + 1e-3 * abs(loss32.item())
    rows_lim = 1.25 * relfro(rows16, rows32) + 5e-3

    def violations(l32, r32, gg32):
        bad = []
        if abs(loss - l32.item()) > loss_lim:
            bad.append(("loss", loss, l32.item()))
        if relfro(rows, r32) > rows_lim:
            bad.append(("loss_rows", relfro(rows, r32)))
        for k in gg32:
            if g32[k].any():
                lim = 1.25 * relfro(g16[k], g32[k]) + 1e-2
                if relfro(grads[k], gg32[k]) > lim:
                    bad.append((k, relfro(grads[k], gg32[k]), lim))
        return bad

    bad = violations(loss32, rows32, g32)
    print(f"[{TAG}] {variant}: loss {loss:.6f} oracle {loss32.item():.6f}, violations {bad}")
    assert not bad
    got = eng.logits(tok)                                 # the logits mask: -inf outside each row's window
    fin = torch.isfinite(got).cpu()
    assert fin.any()
    e = relfro(got.cpu()[fin], logits32[fin])
    assert e <= 1.25 * relfro(logits16[fin], logits32[fin]) + 1e-2, e
    mutants = ("norm_then_divide", "no_shrink") if v["stable"] else ("post_residual", "swapped")
    for m in mutants:
        ml, mr, _, mg = oracle(False, m)
        mbad = violations(ml, mr, mg)
        print(f"[{TAG}]   mutant {m}: {len(mbad)} violated bounds, e.g. {mbad[:2]}")
        assert mbad, m
    if v["row_col"] and v["stable"]:   # the shrink reaches the row / column tables: without it they are 10x off
        _, _, _, ns = oracle(False, "no_shrink")
        for k in ("positional_embedding/image_row", "positional_embedding/image_col"):
            assert relfro(grads[k], g32[k]) < 0.1 < relfro(grads[k], ns[k]), k


def test_engine_initialises_by_depth_on_both_paths():
    """init_params and ZeRO-1's sharded initialisation write the depth schedule (L = 25 reaches all three values)."""
    from oracle import dalle as O
    from oracle import dalle_layer_scale as OLS
    from test_zero1_gpu import Loopback
    cfg = O.DalleConfig(256, 25, 2, 50, 16, 8, 16)
    want = OLS.init_params({}, cfg)
    eng = _engine(cfg, layer_scale=True)
    eng.init_params(seed=1)
    grp = Loopback(2)
    grp.engines = ranks = [_engine(cfg, layer_scale=True, zero=grp.member(r)) for r in range(2)]
    for e in ranks:
        e.init_params(seed=1)
    for e in [eng] + ranks:
        got = e.export_params()
        for k, v in want.items():
            assert torch.equal(got[k], v.to(BF16).float() if e.zero is not None else v), k
    sharded = ranks[0].export_params()
    for k, v in eng.export_params().items():
        assert torch.equal(sharded[k], v.to(BF16).float()), k


# ------------------------------------------------------------------------------------------------ steps
def _small(seed=0, sandwich=False):
    from oracle import dalle as O, dalle_layer_scale as OLS, dalle_sandwich as OSW
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 64)
    params = O.init_params(cfg, seed)
    if sandwich:
        params = OSW.init_params(params, cfg, seed + 5)
    params = OLS.init_params(params, cfg, seed=seed + 6)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.cat([torch.randint(0, 300, (4, 40), generator=g), torch.randint(300, 360, (4, 64), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


@pytest.mark.parametrize("sandwich", [False, True], ids=["plain", "sandwich"])
def test_steps_are_bit_identical_and_micro_batches_match(sandwich):
    cfg, params, tok = _small(3, sandwich)
    eng = _engine(cfg, layer_scale=True, sandwich_norm=sandwich, attention_types=["global", "axial_col"],
                  dropout=(0.1, 0.1, 0.1))
    eng.load_params(params)

    def step(split=1):
        eng.zero_grads()
        mb = tok.shape[0] // split
        for i in range(split):
            eng.forward(tok[i * mb:(i + 1) * mb], step=4, row0=i * mb)
            eng.backward(1.0 / tok.numel())
        torch.cuda.synchronize()
        return eng.grads.clone()
    a, b = step(), step()
    assert torch.equal(a, b)
    n = eng.n_params_padded
    assert relfro(step(2)[:n], a[:n]) < 1e-5


def test_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion for the plain step (bit for bit), with the key and every feature."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, layer_scale=True, sandwich_norm=True, stable=True)
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


@pytest.mark.parametrize("world", [2, 3])
def test_zero1_step_equals_the_replicated_step_bitwise(ops, world):
    """Three Adam steps of W ranks with sharded optimiser state (the scales in the fp32 vector table) against the
    replicated optimiser stepped on the full buffer, bit for bit (test_zero1_gpu.py's emulation)."""
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    params = {k: v.to(BF16).float() for k, v in params.items()}
    grp = Loopback(world)
    kw = dict(layer_scale=True, stable=True, attention_types=["global", "axial_row"])
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **kw) for r in range(world)]
    twin = _engine(cfg, **kw)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    P = twin.master[:n].clone()
    M, V = torch.zeros_like(P), torch.zeros_like(P)
    gn = torch.zeros(1, dtype=F32, device=DEV)
    for step in range(3):
        _twin_from(twin, P, ranks[0])
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
    ex = ranks[0].export_params()
    for k in ("layer_0/attn/layer_scale", "layer_1/mlp/layer_scale"):
        assert not torch.equal(ex[k], params[k]), k                       # the scales trained


# ------------------------------------------------------------------------------------------------ generation
def test_decoding_follows_the_full_forward_and_the_prefill():
    from dalle_mtf_b200.sampling import DalleSampler
    from oracle import dalle as O, dalle_layer_scale as OLS, dalle_sandwich as OSW
    from test_prefill_gpu import greedy_agrees_with_full_forward
    ts, W = 16, 8
    S = ts + W * W
    for sandwich, stable in ((False, False), (True, False), (False, True)):
        cfg = O.DalleConfig(256, 3, 2, 300, 64, ts, W * W)
        params = O.init_params(cfg, 3)
        if sandwich:
            params = OSW.init_params(params, cfg, 4)
        params = OLS.init_params(params, cfg, seed=5)
        g = torch.Generator().manual_seed(9)
        for k in params:
            if k.endswith("bias") or k.endswith("o_b"):
                params[k] = torch.randn(params[k].shape, generator=g) * 0.02
            if "wte" in k or "linear_out" in k or k.endswith("kernel"):
                params[k] = params[k] * 4
        if stable:   # rows whose maximum matters: sigma / m near sqrt(eps)
            params["layer_2/mlp/mlp_linear_2/bias"] = torch.full((256,), -40.0)
        eng = _engine(cfg, layer_scale=True, sandwich_norm=sandwich, stable=stable,
                      attention_types=["global", "axial_col", "conv"])
        eng.load_params(params)
        text = torch.randint(0, 299, (3, ts), generator=g).to(I32).to(DEV)
        smp = DalleSampler(eng)
        out, step_logits = smp.generate(text, 0.0, return_logits=True)
        assert torch.equal(smp.generate_graphed(text, temperature=0.0), out)
        greedy_agrees_with_full_forward(eng, out, ts)
        full = eng.logits(out)
        e = relfro(torch.stack(step_logits, 1), full[:, :S - 1])
        assert e < 2e-2, e
        for P in (ts, ts + W + 3, S - 1):
            kc = [torch.zeros_like(c) for c in smp.kc]
            vc = [torch.zeros_like(c) for c in smp.vc]
            logits = eng.prefill(out[:, :P].contiguous(), kc, vc).clone()
            ep = relfro(logits[:, :eng.V], step_logits[P - 1])
            print(f"[{TAG}] sandwich {sandwich} stable {stable}: decode vs full {e:.2e}, prefill P={P} vs decoding "
                  f"{ep:.2e}")
            assert ep < 2e-2, ep
        done = smp.complete(text, out[:, ts:ts + W + 3].contiguous() - eng.image_offset, temperature=0)
        greedy_agrees_with_full_forward(eng, done, ts + W + 3)
        torch.manual_seed(0)
        guided = smp.complete(text[:2], out[:2, ts:ts + W + 3].contiguous() - eng.image_offset, samples_per_prompt=2,
                              guidance_scale=3.0, top_k=16)
        assert guided.shape == (4, S)
        assert ((guided[:, ts:] >= eng.image_offset) & (guided[:, ts:] < eng.image_offset + 64)).all()
        assert torch.equal(smp.generate_graphed(text[:2], temperature=0.0, guidance_scale=2.0),
                           smp.generate(text[:2], 0.0, guidance_scale=2.0))


# ------------------------------------------------------------------------------------------------ checkpoints
def test_export_load_round_trip_and_mismatched_checkpoints_are_refused():
    from dalle_mtf_b200 import lib as L
    from oracle import dalle_layer_scale as OLS
    cfg, params, tok = _small(7)
    eng = _engine(cfg, layer_scale=True)
    eng.load_params(params)
    ex = eng.export_params()
    assert set(ex) == set(params)
    for k in params:
        assert torch.equal(ex[k], params[k].float()), k
    plain_params = {k: v for k, v in params.items() if not k.endswith("/layer_scale")}
    assert set(params) - set(plain_params) == set(OLS.scale_names(cfg))
    with pytest.raises(L.DB200Error, match="layer_0/attn/layer_scale"):
        eng.load_params(plain_params)
    plain = _engine(cfg)
    with pytest.raises(L.DB200Error, match="layer_0/attn/layer_scale"):
        plain.load_params(params)
    with pytest.raises(L.DB200Error, match="layer_1/mlp/layer_scale"):
        eng.load_params({k: v for k, v in params.items() if k != "layer_1/mlp/layer_scale"})
    with pytest.raises(L.DB200Error, match="layer_1/mlp/layer_scale"):
        plain.load_params({**plain_params, "layer_1/mlp/layer_scale": params["layer_1/mlp/layer_scale"]})
    plain.load_params(plain_params)
    assert set(plain.export_params()) == set(plain_params)


def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def test_model_fn_checkpoint_resumes_bit_exactly_and_generate_runs(tmp_path):
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    from dalle_mtf_b200.utils import save_checkpoint
    key = {"layer_scale": True, "sandwich_norm": True, "stable": True}
    img, cap = _batch()
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    p = _tiny_params(tmp_path, **key)
    ls = dalle_model_fn(img, cap, "train", p)
    assert ls.engine.layer_scale is True and plain.engine.layer_scale is None
    assert ls.engine.stable and not plain.engine.stable
    assert ls.engine.n_params() - plain.engine.n_params() == (4 + 2) * 256 * 2
    ls.train_op(img, cap)
    st = ls.state_fn()
    assert {k for k in st if k.endswith("/layer_scale")} == \
        {f"layer_{i}/{b}/layer_scale" for i in range(2) for b in ("attn", "mlp")}
    a = ls.train_op(img, cap).clone()
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **key))
    resumed.load_fn(st)
    assert torch.equal(a, resumed.train_op(img, cap))
    with pytest.raises(L.DB200Error, match="layer_scale|norm_out"):
        plain.load_fn(st)
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=64, n_layers=1, n_heads=2,
              mode="eval", params={"layer_scale": 0.5, "stable": True})
    assert m.engine.layer_scale == 0.5 and m.engine.stable
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 64), generator=g)], 1)
    loss, loss_batch = m.forward({"tokens": tokens})
    assert math.isfinite(loss.item()) and loss_batch.shape == (2, 104)
    # generate_dalle.py end to end on the trained checkpoint
    vae = ls.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, ls.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "ls.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "ls.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, ls.engine.S) and len(list(out.glob("*.png"))) == 2


# ------------------------------------------------------------------------------------------------ launches
@pytest.mark.parametrize("recompute", [False, True], ids=["saved", "recompute"])
def test_key_off_runs_no_new_kernel_and_the_key_adds_the_expected_launches(monkeypatch, recompute):
    """With the keys absent or false no new op runs and the op sequence is the same; with layer_scale on, every layer
    adds one layer_scale_residual_fwd per branch in forward (twice with recompute_grad) and one layer_scale_bwd per
    branch in backward, and every other op runs as without it; stable replaces the final LayerNorm's two ops."""
    from dalle_mtf_b200 import ops as O
    cfg, params, tok = _small(2)
    names = [n for n in dir(O) if not n.startswith("_") and callable(getattr(O, n)) and
             getattr(getattr(O, n), "__module__", "") == O.__name__]
    calls = []
    for n in names:
        f = getattr(O, n)
        monkeypatch.setattr(O, n, (lambda f, n: lambda *a, **k: (calls.append(n), f(*a, **k))[1])(f, n))

    def run(**kw):
        eng = _engine(cfg, recompute_grad=recompute, **kw)
        eng.load_params(params if kw.get("layer_scale") else
                        {k: v for k, v in params.items() if not k.endswith("/layer_scale")})
        calls.clear()
        _step(eng, tok)
        eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        return list(calls)
    absent, off, on = run(), run(layer_scale=False, stable=False), run(layer_scale=True)
    assert absent == off
    new = {"layer_scale_residual_fwd", "layer_scale_bwd", "layernorm_scale_residual_fwd", "layernorm_divmax_fwd",
           "layernorm_divmax_bwd"}
    assert not new & set(off)
    Lyr = cfg.n_layers
    assert on.count("layer_scale_residual_fwd") == 2 * Lyr * (2 if recompute else 1)
    assert on.count("layer_scale_bwd") == 2 * Lyr
    assert [c for c in on if c not in ("layer_scale_residual_fwd", "layer_scale_bwd")] == off
    # stable: the final LayerNorm's forward and backward are the DivideMax ones, nothing else changes
    st = run(layer_scale=True, stable=True)
    swap = {"layernorm_divmax_fwd": "layernorm_fwd", "layernorm_divmax_bwd": "layernorm_bwd"}
    assert st.count("layernorm_divmax_fwd") == 1 and st.count("layernorm_divmax_bwd") == 1
    assert [swap.get(c, c) for c in st] == on


def _replay_store_gemm(ops, f, c):
    """A STORE product without a residual (Wo / W2 / gMLP W_out writing o) against float64."""
    from dalle_mtf_b200 import lib as L
    M, N, K = f["M"], f["N"], f["K"]
    assert not f["residual"] and f["mode"] == L.EPI_STORE and not f["a_mn"] and f["b_mn"], c
    x, w = _rand(M, K, M, scale=0.5), _rand(K, N, K, scale=0.05)
    bias = _vec(N, N, 0.0) if f["bias"] else None
    site = L.make_dropout(0.1, 1, 2, L.dropout_site_attn_out(0), 0) if f["dropout"] else None
    out = torch.empty(M, N, dtype=BF16, device=DEV)
    ops.linear_fwd(x, w, out, bias=bias, dropout=site)
    want = x.double() @ w.double() + (bias.double() if bias is not None else 0)
    if site is not None:
        keep = torch.empty(M, N, dtype=torch.uint8, device=DEV)
        ops.dropout_mask(site, L.DROPOUT_ELEMENTWISE, (M, N), keep)
        want = want * keep.double() * site.scale
    torch.cuda.synchronize()
    assert relfro(out, want) < 1e-2, c


def test_launch_census_of_dalle_example_with_the_keys_replays_its_new_classes(ops, monkeypatch):
    """dalle_example_b200 recorded by test_dalle_config_launches_gpu.py's recorder (train, eval, eager and graphed
    decoding, prefill with guidance) plain, with {layer_scale, stable} and with {layer_scale, stable, sandwich_norm}:
    the keyed models launch the plain model's classes plus the new kernels' classes (at the training, prefill and
    decoder row counts), the LayerNorm backwards and STORE products whose fusions the keys move, and the optimiser's
    classes at the new parameter count.  Each added class is replayed at its recorded shape against float64, and so
    is the scaled embedding backward at the recorded B / S / V (its class does not record alpha)."""
    import launch_census as LC
    import test_dalle_config_launches_gpu as CL
    import test_dalle_kernels_gpu as DK
    from dalle_mtf_b200 import lib as L
    from test_sandwich_norm_gpu import _ln_bwd_reference, _replay_optimizer_class
    base = DK._config("dalle_example_b200")
    recorded = {}
    for name, extra in (("plain", {}), ("keys", {"layer_scale": True, "stable": True}),
                        ("keys_sandwich", {"layer_scale": True, "stable": True, "sandwich_norm": True})):
        monkeypatch.setattr(DK, "_config", lambda c, extra=extra: dict(base, **extra))
        recorded[name] = set(CL.record_config("dalle_example_b200")[0])
    added = (recorded["keys"] | recorded["keys_sandwich"]) - recorded["plain"]
    entries = {c[0] for c in added}
    new = {"layer_scale_residual_fwd", "layernorm_scale_residual_fwd", "layer_scale_bwd", "layernorm_divmax_fwd",
           "layernorm_divmax_bwd"}
    assert new <= entries <= new | {"layernorm_bwd", "gemm", "sqnorm", "adam_step", "cast_f32_to_bf16"}, entries
    assert not {c[0] for c in recorded["plain"]} & new
    rows_seen = {e: sorted({LC.fields(c)["o" if "residual" in e else "v" if e == "layer_scale_bwd" else "x"][0][0]
                            for c in added if c[0] == e}) for e in new}
    print(f"[{TAG}] census rows of the new entries: {rows_seen}")
    # the forwards run at the training rows and at the decoder's (and guidance's) rows, the backwards in training only
    assert all(len(r) >= 3 for e, r in rows_seen.items() if not e.endswith("_bwd")), rows_seen
    for c in sorted(added, key=repr):
        f = LC.fields(c)
        if c[0] == "layer_scale_residual_fwd":
            check_residual_fwd(ops, *f["o"][0])
        elif c[0] == "layernorm_scale_residual_fwd":
            check_ln_scale_residual_fwd(ops, *f["o"][0])
        elif c[0] == "layer_scale_bwd":
            rows, d = f["v"][0]
            drop = L.make_dropout(0.1, 5, 3, L.dropout_site_mlp_out(2), 0) if f["dropout"] is not None else None
            assert (f["db"] is None) == (f["norm"] is not None), c       # db is fused only without the sandwich
            _check_bwd(ops, rows, d, drop=drop, sandwich=f["norm"] is not None)
        elif c[0] == "layernorm_divmax_fwd":
            for kind in ("random", "c-100"):
                check_divmax_fwd(ops, *f["x"][0], kind)
        elif c[0] == "layernorm_divmax_bwd":
            check_divmax_bwd_fusions(ops, *f["x"][0])
        elif c[0] in ("sqnorm", "adam_step", "cast_f32_to_bf16"):
            _replay_optimizer_class(ops, c[0], f)
        elif c[0] == "layernorm_bwd":
            rows, d = f["rows"], f["d"]
            x, dy = _rand(rows, d, rows, scale=2.0), _rand(rows, d, rows + 1)
            dres = _rand(rows, d, rows + 2) if f["dres"] else None
            g = _vec(d, 3, 1.0)
            mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
            ops.layernorm_fwd(x, g, torch.zeros(d, device=DEV), torch.empty_like(x), mean, rstd)
            dx, dg, db = torch.empty_like(x), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
            dxsum = torch.zeros(d, device=DEV) if f["dxsum"] else None
            site = L.make_dropout(0.1, 1, 2, L.dropout_site_mlp_out(0), 0) if f["dropout"] else None
            dxm = torch.empty_like(x) if site is not None else None
            ops.layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db, dxsum=dxsum, dxm=dxm, dropout=site)
            torch.cuda.synchronize()
            rdx, rdg, rdb = _ln_bwd_reference(dy, x, g, mean, rstd, dres)
            assert relfro(dx, rdx) < 1e-2 and relfro(dg, rdg) < 1e-4 and relfro(db, rdb) < 1e-4, c
            if dxsum is not None:
                assert relfro(dxsum, (dxm if dxm is not None else dx).double().sum(0)) < 1e-4, c
        else:
            _replay_store_gemm(ops, f, c)
        print(f"[{TAG}] census class {c[0]} {f}: replayed against float64")
    embeds = [LC.fields(c) for c in recorded["keys"] if c[0] == "embed_bwd"]
    assert embeds
    for f in embeds:
        check_embed_bwd_scaled(ops, f["B"], f["S"], f["d"], f["V"], f["dropout"])
        print(f"[{TAG}] embed_bwd with alpha at {f}: replayed against float64")


def test_checkpoint_refusals_name_a_layer_kind_mismatch_first_and_take_malformed_names():
    from dalle_mtf_b200 import lib as L
    from oracle import dalle as O, dalle_gmlp as OM, dalle_layer_scale as OLS, dalle_local as OL
    cfg = OL.LocalConfig(256, 2, 2, 300, 64, 64, 64, attention_types=("global", "mlp"))
    params = OLS.init_params(OM.init_params(O.init_params(cfg, 1), cfg, 2), cfg)
    attn = _engine(cfg, attention_types=["global", "global"], layer_scale=True)
    with pytest.raises(L.DB200Error, match="layer_1/gmlp/.*attention layer"):   # the kind, not a missing scale
        attn.load_params(params)
    eng = _engine(cfg, attention_types=["global", "mlp"], layer_scale=True, stable=None)
    eng.load_params(params)
    assert eng.stable is False
    with pytest.raises(L.DB200Error, match="layer_x/mlp/layer_scale"):
        eng.load_params({**params, "layer_x/mlp/layer_scale": torch.ones(256)})
