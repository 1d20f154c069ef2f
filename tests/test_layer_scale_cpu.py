"""CPU side of LayerScale and the stable option: the layer_scale and stable keys at every place a model is built (true
is not the number 1), generate_dalle.py handing them to the engine, the parameter layout (names, shapes, bucket
spans, the fp32 vector table, weight decay), the count, the initial values by depth, DivideMax's LayerNorm identity
and the embedding gradient shrink in float64, and the oracle (bit for bit the gMLP oracle with both keys off, and
mutants that change the output)."""
import math

import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import DalleEngine, layer_mlp, layer_scale_init, param_layout, validate_layer_scale
from dalle_mtf_b200.model_fns import dalle_model_fn, layer_scale
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_gmlp as OM
from oracle import dalle_layer_scale as OLS
from oracle import dalle_local as OL
from oracle import dalle_sandwich as OSW
from test_gelu_cpu import _Built, _generate_config

NEW = ("lsa", "lsm")


# ------------------------------------------------------------------------------------------------ config values
ACCEPTED = [({}, None), ({"layer_scale": None}, None), ({"layer_scale": False}, None), ({"layer_scale": True}, True),
            ({"layer_scale": 1}, 1.0), ({"layer_scale": 0.1}, 0.1), ({"layer_scale": 1e-6}, 1e-6)]
REJECTED = [0, 0.0, -0.1, -1, math.nan, math.inf, -math.inf, "true", "0.1", "", [], [True], {"on": True}]


@pytest.mark.parametrize("params,want", ACCEPTED, ids=[repr(p) for p, _ in ACCEPTED])
def test_accepted_values(params, want):
    got = layer_scale(params)
    assert got == want and type(got) is type(want)


def test_true_is_the_depth_schedule_and_not_the_number_one():
    assert layer_scale({"layer_scale": True}) is True
    assert layer_scale({"layer_scale": 1}) == 1.0 and layer_scale({"layer_scale": 1}) is not True
    assert [layer_scale_init(True, i) for i in (0, 5)] == [0.1, 0.1]
    assert [layer_scale_init(1.0, i) for i in (0, 30)] == [1.0, 1.0]


@pytest.mark.parametrize("value", REJECTED, ids=[repr(v) for v in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    p = {"layer_scale": value}
    with pytest.raises(ValueError, match="layer_scale"):
        layer_scale(p)
    with pytest.raises(ValueError, match="layer_scale"):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="layer_scale"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match="layer_scale"):
        G.main(_generate_config(tmp_path, p))


def test_engine_validates_its_argument_before_any_device_work():
    for v, want in ((None, None), (False, None), (True, True), (0.5, 0.5), (2, 2.0)):
        assert validate_layer_scale(v) == want
    for bad in REJECTED:
        with pytest.raises(ValueError, match="layer_scale"):
            validate_layer_scale(bad)
        with pytest.raises(ValueError, match="layer_scale"):
            DalleEngine(256, 1, 2, 10, 16, 4, 16, layer_scale=bad)


@pytest.mark.parametrize("extra,want", [({}, None), ({"layer_scale": None}, None), ({"layer_scale": True}, True),
                                        ({"layer_scale": 0.25}, 0.25)])
def test_generate_cli_builds_the_engine_with_the_config_key(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the LayerScale it was trained with (device work stubbed)."""
    import types
    from dalle_mtf_b200 import dalle_engine, lib as L, model_fns
    seen = {}

    def engine(*a, **k):
        seen.update(k)
        raise _Built

    vae = types.SimpleNamespace(K=64, image_seq_len=16, load_params=lambda state: None)
    monkeypatch.setattr(L, "require_device", lambda: None)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(model_fns, "load_vae_model", lambda params, device: (vae, None))
    monkeypatch.setattr(dalle_engine, "DalleEngine", engine)
    with pytest.raises(_Built):
        G.main(_generate_config(tmp_path, extra))
    assert seen["layer_scale"] == want and type(seen["layer_scale"]) is type(want)


# ------------------------------------------------------------------------------------------------ layout
def _bare_engine(d, types, scale, sandwich=False, tl=64, il=64):
    """A DalleEngine with only the fields n_params / _ref_names / _decay_segments / layer_last read (no device)."""
    e = DalleEngine.__new__(DalleEngine)
    Lyr = len(types)
    e.d, e.L, e.text_seq_len, e.image_seq_len = d, Lyr, tl, il
    e.V, e.S = 300 + 64 + 1, tl + il
    e.row_col, e.grid_w, e.gated_mlp, e.sandwich_norm, e.layer_scale = False, None, False, sandwich, scale
    e.mlp = layer_mlp(types, Lyr, e.S, d)
    e.layout = param_layout(d, Lyr, e.V, e.S, sandwich_norm=sandwich, mlp_layers=e.mlp,
                            layer_scale=scale is not None)
    return e


@pytest.mark.parametrize("sandwich", [False, True], ids=["plain", "sandwich"])
@pytest.mark.parametrize("types", [["global", "global"], ["global", "mlp", "axial_row"]], ids=["global", "mixed"])
def test_layout_names_spans_and_count(types, sandwich):
    d, Lyr = 256, len(types)
    plain = _bare_engine(d, types, None, sandwich)
    e = _bare_engine(d, types, True, sandwich)
    lay = e.layout
    added = [k for k in lay.order if k not in plain.layout.entries]
    assert added == [f"l{i}.{n}" for i in range(Lyr) for n in NEW]
    assert [k for k in lay.order if k in plain.layout.entries] == plain.layout.order
    assert all(lay.entries[k][1] == (d,) and lay.entries[k][0] % 64 == 0 for k in added)
    assert e.n_params() - plain.n_params() == Lyr * 2 * d
    for i in range(Lyr):   # the two vectors end each layer, inside its data-parallel bucket
        assert [k for k in lay.order if k.startswith(f"l{i}.")][-2:] == [f"l{i}.lsa", f"l{i}.lsm"]
        assert e.layer_last(i) == f"l{i}.lsm"
        s, end = lay.span(f"l{i}.ln1_g", e.layer_last(i))
        assert end == lay.entries[f"l{i + 1}.ln1_g" if i + 1 < Lyr else "lnf_g"][0]
    assert plain.layer_last(0) == ("l0.lnm_b" if sandwich else "l0.b2")
    names = [rn for i in range(Lyr) for k, rn in e._layer_ref_names(i).items() if k in NEW]
    cfg = OL.LocalConfig(d, Lyr, 2, 300, 64, 64, 64, attention_types=tuple(types))
    assert names == OLS.scale_names(cfg)
    assert ("layer_1/gmlp/layer_scale" in names) == (types[1] == "mlp")
    assert all(k not in NEW for i in range(Lyr) for k in plain._layer_ref_names(i))


def test_scales_are_vector_parameters_and_are_not_decayed():
    e = _bare_engine(256, ["global", "mlp", "global"], 0.5, sandwich=True)
    plain = _bare_engine(256, ["global", "mlp", "global"], None, sandwich=True)
    assert set(NEW) <= set(DalleEngine.VECTOR_PARAMS)
    for name in e.layout.order:
        if name.split(".")[-1] in NEW:
            o, _ = e.layout.entries[name]
            assert [dec for s, t, dec in e._decay_segments() if s <= o < t] == [False], name
    decayed = lambda eng: sum(t - s for s, t, dec in eng._decay_segments() if dec)   # noqa: E731
    assert decayed(e) == decayed(plain)


def test_initial_values_follow_the_depth_schedule():
    """true: 0.1 up to depth 18, 1e-5 up to 24, 1e-6 beyond (L = 30 reaches all three); the engine's values equal the
    oracle's, and CaiT's rule by total depth (the depth_by_L mutant) differs from them."""
    got = [layer_scale_init(True, i) for i in range(30)]
    assert got == [0.1] * 18 + [1e-5] * 6 + [1e-6] * 6
    assert got == [OLS.depth_value(i + 1) for i in range(30)]
    cfg = O.DalleConfig(64, 30, 2, 50, 16, 4, 16)
    ref = OLS.init_params({}, cfg)
    mut = OLS.init_params({}, cfg, mutate="depth_by_L")
    for i in range(30):
        for b in ("attn", "mlp"):
            assert torch.equal(ref[f"layer_{i}/{b}/layer_scale"], torch.full((64,), got[i]))
    assert any(not torch.equal(ref[k], mut[k]) for k in ref)
    assert all(torch.equal(v, torch.full((64,), 0.25)) for v in OLS.init_params({}, cfg, value=0.25).values())


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, types=("global", "global"), d=64, H=2, TL=8, W=4):
    cfg = OL.LocalConfig(d, len(types), H, 50, 16, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 1)
    params = OSW.init_params(params, cfg, seed + 2)
    g = torch.Generator().manual_seed(seed + 3)
    for k in params:
        if k.endswith("o_b") or k.endswith("mlp_linear_2/bias"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.05
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, TL), generator=g),
                               torch.randint(0, 16, (2, W * W), generator=g), 50)
    return cfg, OLS.init_params(params, cfg, seed=seed + 4), tokens


@pytest.mark.parametrize("variant", [dict(), dict(sandwich_norm=True), dict(gated=True, activation="gelu",
                                                                             rotary=(16, 10000.0), shift_tokens=True)],
                         ids=["plain", "sandwich", "geglu_rotary_shift"])
@pytest.mark.parametrize("types", [("global", "global"), ("global", "mlp")], ids=["global", "global_mlp"])
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_oracle_without_the_key_is_the_gmlp_oracle_bit_for_bit(types, variant, bf16):
    from oracle import dalle_glu as OGL
    cfg, params, tokens = _model(3, types)
    if variant.get("gated"):
        params = OGL.init_params(params, cfg, 4)
    base = {k: v for k, v in params.items() if not k.endswith("/layer_scale")}
    if not variant.get("sandwich_norm"):
        base = {k: v for k, v in base.items() if "/norm_out/" not in k}
    a = OLS.loss_and_grads(params, tokens, cfg, layer_scale=False, bf16=bf16, **variant)
    b = OM.loss_and_grads(base, tokens, cfg, bf16=bf16, **variant)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert all(torch.equal(a[3][k], b[3][k]) for k in b[3])
    assert all(not a[3][k].any() for k in OLS.scale_names(cfg))


def test_oracle_with_dropout_and_without_the_key_is_the_gmlp_oracle_bit_for_bit():
    cfg, params, tokens = _model(4, ("global", "mlp"))
    dropout = ((0.1, 0.1, 0.2), 7, 3, 0)
    base = {k: v for k, v in params.items() if not k.endswith("/layer_scale") and "/norm_out/" not in k}
    a = OLS.forward(params, tokens, cfg, dropout, layer_scale=False)
    b = OM.forward(base, tokens, cfg, dropout)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_the_scales_and_each_mutant_change_the_output():
    cfg, params, tokens = _model(5, ("global", "mlp"), d=128)
    for sandwich in (False, True):
        off = OLS.forward(params, tokens, cfg, sandwich_norm=sandwich)[2]
        ref = OLS.forward(params, tokens, cfg, sandwich_norm=sandwich, layer_scale=True)[2]
        assert ((ref - off).norm() / off.norm()).item() > 1e-3
        for m in ("post_residual", "swapped") + (("scale_before_norm",) if sandwich else ()):
            mut = OLS.forward(params, tokens, cfg, sandwich_norm=sandwich, layer_scale=True, scale_mutate=m)[2]
            rel = ((mut - ref).norm() / ref.norm()).item()
            assert rel > 1e-3, (sandwich, m, rel)
    for bad in (dict(scale_mutate="nope", layer_scale=True), dict(scale_mutate="swapped"),
                dict(scale_mutate="scale_before_norm", layer_scale=True), dict(scale_mutate="depth_by_L",
                                                                               layer_scale=True)):
        with pytest.raises(ValueError):
            OLS.forward(params, tokens, cfg, **bad)


def test_scale_gradient_is_the_column_sum_of_dy_times_the_branch_in_float64():
    """The adjoint the backward kernel implements: for y = x + s * v, ds = sum_rows dy v and dv = s dy (float64)."""
    g = torch.Generator().manual_seed(0)
    x, v, dy = (torch.randn(37, 64, generator=g, dtype=torch.float64) for _ in range(3))
    s = (torch.rand(64, generator=g, dtype=torch.float64) + 0.1).requires_grad_(True)
    v = v.requires_grad_(True)
    (x + s * v).backward(dy)
    assert torch.allclose(s.grad, (dy * v).sum(0).detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(v.grad, s.detach() * dy, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ stable
STABLE_REJECTED = [1, 0, 1.0, "true", "", [], [True], {"on": True}]


@pytest.mark.parametrize("params,want", [({}, False), ({"stable": None}, False), ({"stable": False}, False),
                                         ({"stable": True}, True)])
def test_stable_accepted_values(params, want):
    from dalle_mtf_b200.dalle_engine import validate_stable
    from dalle_mtf_b200.model_fns import stable
    assert stable(params) is want
    assert validate_stable(params.get("stable")) is want       # the engine takes null as off too


@pytest.mark.parametrize("value", STABLE_REJECTED, ids=[repr(v) for v in STABLE_REJECTED])
def test_stable_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    from dalle_mtf_b200.dalle_engine import validate_stable
    from dalle_mtf_b200.model_fns import stable
    p = {"stable": value}
    for build in (lambda: stable(p), lambda: validate_stable(value),
                  lambda: DalleEngine(256, 1, 2, 10, 16, 4, 16, stable=value),
                  lambda: dalle_model_fn(None, None, "train", dict(p)),
                  lambda: DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16,
                                n_layers=1, n_heads=2, params=dict(p)),
                  lambda: G.main(_generate_config(tmp_path, p))):
        with pytest.raises(ValueError, match="stable"):
            build()


@pytest.mark.parametrize("extra,want", [({}, False), ({"stable": True}, True)])
def test_generate_cli_hands_stable_to_the_engine(tmp_path, monkeypatch, extra, want):
    import types
    from dalle_mtf_b200 import dalle_engine, lib as L, model_fns
    seen = {}

    def engine(*a, **k):
        seen.update(k)
        raise _Built

    vae = types.SimpleNamespace(K=64, image_seq_len=16, load_params=lambda state: None)
    monkeypatch.setattr(L, "require_device", lambda: None)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(model_fns, "load_vae_model", lambda params, device: (vae, None))
    monkeypatch.setattr(dalle_engine, "DalleEngine", engine)
    with pytest.raises(_Built):
        G.main(_generate_config(tmp_path, extra))
    assert seen["stable"] is want


def _ln64(x, g, b, eps):
    mu = x.mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps) * g + b


@pytest.mark.parametrize("c", [100.0, -100.0, 0.0])
def test_divide_max_layernorm_identity_and_sign_flip_in_float64(c):
    """LN(x / m) = sign(m) (x - mu) / sqrt(sigma^2 + eps m^2) g + b: the division matters where sigma / m is near
    sqrt(eps) (x = c + small noise, c = +-100) and a negative m flips the sign of the normalised row."""
    g0 = torch.Generator().manual_seed(1)
    eps = 1e-5
    x = (c + 0.3 * torch.randn(16, 512, generator=g0, dtype=torch.float64)).to(torch.bfloat16).double()
    g, b = 1 + 0.3 * torch.randn(512, generator=g0, dtype=torch.float64), 0.1 * torch.randn(512, generator=g0,
                                                                                             dtype=torch.float64)
    m = x.amax(-1, keepdim=True)
    lhs = _ln64(x / m, g, b, eps)
    mu, var = x.mean(-1, keepdim=True), ((x - x.mean(-1, keepdim=True)) ** 2).mean(-1, keepdim=True)
    rhs = torch.sign(m) * (x - mu) / torch.sqrt(var + eps * m ** 2) * g + b
    assert torch.allclose(lhs, rhs, rtol=1e-9, atol=1e-9)
    plain = _ln64(x, g, b, eps)
    corr = ((lhs - b) * (plain - b)).sum(-1)
    assert ((corr < 0) if c < 0 else (corr > 0)).all()     # m < 0 flips the normalised row, m > 0 keeps its sign
    if c != 0:  # sigma / m ~ sqrt(eps): the division changes the result
        assert ((lhs - torch.sign(m) * (plain - b) - b).abs().max() > 1e-2)
    else:       # ordinary rows: LN(x / m) ~ LN(x)
        assert torch.allclose(lhs, plain, atol=1e-3)


def test_stable_shrinks_every_embedding_gradient_by_alpha_in_float64():
    """The forward is unchanged; the wte / wpe gradients are alpha times those without the shrink; every other
    gradient is the same (float64)."""
    cfg, params, tokens = _model(6, ("global", "mlp"))
    p64 = {k: v.double() for k, v in params.items()}
    a = OLS.loss_and_grads(p64, tokens, cfg, stable=True, layer_scale=True)
    b = OLS.loss_and_grads(p64, tokens, cfg, stable=True, layer_scale=True, stable_mutate="no_shrink")
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    for k in a[3]:
        if k.startswith(("embedding/", "positional_embedding/")):
            assert torch.allclose(a[3][k], OLS.ALPHA * b[3][k], rtol=1e-12, atol=1e-15), k
        else:
            assert torch.equal(a[3][k], b[3][k]), k


def test_stable_and_each_of_its_mutants_change_the_model():
    cfg, params, tokens = _model(7, ("global", "global"))
    for c in (200.0, -200.0):
        p = dict(params)
        p[f"layer_{cfg.n_layers - 1}/mlp/mlp_linear_2/bias"] = torch.full((cfg.n_embd,), c)
        off = OLS.loss_and_grads(p, tokens, cfg, layer_scale=True)
        on = OLS.loss_and_grads(p, tokens, cfg, layer_scale=True, stable=True)
        assert ((on[2] - off[2]).norm() / off[2].norm()).item() > 1e-4
        for m in OLS.STABLE_MUTATIONS:
            mut = OLS.loss_and_grads(p, tokens, cfg, layer_scale=True, stable=True, stable_mutate=m)
            dl = ((mut[2] - on[2]).norm() / on[2].norm()).item()
            dg = max(((mut[3][k] - on[3][k]).norm() / on[3][k].norm()).item() for k in on[3] if on[3][k].any())
            if m == "max_abs" and c > 0:   # all positive rows: max |x| is max x
                assert dl == 0 and dg == 0
            else:
                assert dl > 1e-4 or dg > 1e-6, (c, m, dl, dg)
    with pytest.raises(ValueError):
        OLS.forward(params, tokens, cfg, stable_mutate="max_abs")
