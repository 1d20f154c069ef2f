"""gMLP token-mixing layers ("mlp" in attention_types) without a GPU: parsing and refusals, the parameter layout and
names, the oracle's properties and mutants (oracle/dalle_gmlp.py)."""
import pytest
import torch

from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.dalle_engine import ATTENTION_TYPES, DalleEngine, layer_mlp, param_layout
from dalle_mtf_b200.model_fns import attention_layers
from oracle import dalle as O
from oracle import dalle_gmlp as OM
from oracle import dalle_local as OL
from oracle import dalle_sandwich as OSW

GMLP = ("gm_win", "gm_bin", "sgu_g", "sgu_b", "sgu_w", "sgu_c", "gm_wout", "gm_bout")


# ------------------------------------------------------------------------------------------------ parsing, refusals
@pytest.mark.parametrize("other", ["global", "local", "axial_row", "axial_col", "conv"])
def test_mlp_mixes_with_every_other_type(other):
    assert "mlp" in ATTENTION_TYPES
    types, _ = attention_layers({"n_layers": 4, "attention_types": [[[other, "mlp"], 2]]})
    assert list(types) == [other, "mlp"] * 2
    assert layer_mlp(types, 4, 128, 256) == [False, True, False, True]


def test_sparse_stays_refused():
    with pytest.raises(ValueError, match="sparse"):
        attention_layers({"n_layers": 1, "attention_types": [[["sparse"], 1]]})


@pytest.mark.parametrize("S", [63, 65, 100, 1000])
def test_sequence_length_not_a_multiple_of_64_is_refused(S):
    with pytest.raises(L.DB200Error, match="multiple of 64"):
        layer_mlp(["global", "mlp"], 2, S, 256)
    assert layer_mlp(["global", "global"], 2, S, 256) == [False, False]   # no gMLP layer: no rule


@pytest.mark.parametrize("d", [768, 4096])
def test_sgu_width_outside_the_layernorm_widths_is_refused(d):
    with pytest.raises(L.DB200Error, match="spatial gating unit"):
        layer_mlp(["mlp"], 1, 128, d)


@pytest.mark.parametrize("d", [128, 256, 512, 1024, 2048])
def test_sgu_widths_the_layernorm_kernels_cover_are_accepted(d):
    assert layer_mlp(["mlp"], 1, 1280, d) == [True]


# ------------------------------------------------------------------------------------------------ layout, names
def _bare_engine(d, types, tl=64, il=64, sandwich=False):
    """A DalleEngine with only the fields n_params / _ref_names / _decay_segments / _check_layer_kinds read."""
    e = DalleEngine.__new__(DalleEngine)
    Lyr = len(types)
    e.d, e.L, e.text_seq_len, e.image_seq_len = d, Lyr, tl, il
    e.V, e.S = 300 + 64 + 1, tl + il
    e.row_col, e.grid_w, e.gated_mlp, e.sandwich_norm = False, None, False, sandwich
    e.mlp = layer_mlp(types, Lyr, e.S, d)
    e.layout = param_layout(d, Lyr, e.V, e.S, sandwich_norm=sandwich, mlp_layers=e.mlp)
    return e


@pytest.mark.parametrize("sandwich", [False, True])
def test_layout_spans_counts_and_decay(sandwich):
    d, types = 256, ["global", "mlp", "axial_row", "mlp"]
    e = _bare_engine(d, types, sandwich=sandwich)
    lay, S = e.layout, e.S
    last = "lnm_b" if sandwich else "b2"
    for i, t in enumerate(types):
        names = [k.split(".")[1] for k in lay.order if k.startswith(f"l{i}.")]
        if t == "mlp":
            assert names[2:10] == list(GMLP) and "wqkv" not in names
            assert lay.entries[f"l{i}.sgu_w"][1] == (S, S)
        else:
            assert "wqkv" in names and not set(GMLP) & set(names)
        s, end = lay.span(f"l{i}.ln1_g", f"l{i}.{last}")
        assert all(s <= lay.entries[f"l{i}.{n}"][0] < end for n in names)   # one contiguous bucket per layer
    assert all(off % 64 == 0 for off, _ in lay.entries.values())
    count = sum(torch.Size(s).numel() for k, (_, s) in lay.entries.items() if k not in ("wout", "bout"))
    assert e.n_params() == count + d * e.V + e.V
    plain = _bare_engine(d, ["global"] * 4, sandwich=sandwich)
    gmlp = 4 * d * d + 4 * d + 2 * 2 * d + S * S + S + 2 * d * d + d
    attn = 4 * d * d + d
    assert e.n_params() - plain.n_params() == 2 * (gmlp - attn)
    assert {"gm_bin", "sgu_g", "sgu_b", "sgu_c", "gm_bout"} <= set(DalleEngine.VECTOR_PARAMS)
    for name in lay.order:   # mtf's exclude_from_weight_decay=["norm", "bias"], by reference name
        leaf = name.split(".")[-1]
        if leaf in GMLP:
            o, _ = lay.entries[name]
            dec = [x for s, t, x in e._decay_segments() if s <= o < t]
            assert dec == [leaf in ("gm_win", "sgu_w", "gm_wout")], name


def test_reference_names_of_a_gmlp_layer():
    e = _bare_engine(256, ["global", "mlp"])
    names = e._layer_ref_names(1)
    assert "wo" not in names and "o_b" not in names
    assert {names[k] for k in GMLP} == {f"layer_1/gmlp/{v}" for v in OM.GMLP_VARS}
    assert "wo" in e._layer_ref_names(0)


def _named(types, d=256, tl=64, il=64, seed=0):
    cfg = OL.LocalConfig(d, len(types), 2, 300, 64, tl, il, attention_types=tuple(types))
    return OM.init_params(O.init_params(cfg, seed), cfg)


def test_checkpoint_of_another_layer_kind_is_refused_naming_the_variable():
    e = _bare_engine(256, ["global", "mlp"])
    e._check_layer_kinds(_named(["global", "mlp"]))                     # its own kind: accepted
    with pytest.raises(L.DB200Error, match="layer_1/attn/q"):
        e._check_layer_kinds(_named(["global", "global"]))
    with pytest.raises(L.DB200Error, match="layer_0/gmlp/proj_in/bias"):
        _bare_engine(256, ["global", "global"])._check_layer_kinds(_named(["mlp", "global"]))
    named = _named(["global", "mlp"])
    del named["layer_1/gmlp/sgu/bias"]
    with pytest.raises(L.DB200Error, match="layer_1/gmlp/sgu/bias"):
        e._check_layer_kinds(named)


def test_checkpoint_with_a_non_causal_mixing_weight_is_refused():
    e = _bare_engine(256, ["global", "mlp"])
    named = _named(["global", "mlp"])
    named["layer_1/gmlp/sgu/weight"][3, 4] = 1e-30
    with pytest.raises(L.DB200Error, match="upper triangle"):
        e._check_layer_kinds(named)


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, types=("global", "mlp"), d=64, TL=28, W=6):
    cfg = OL.LocalConfig(d, len(types), 2, 50, 16, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 2)
    g = torch.Generator().manual_seed(seed + 1)
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, TL), generator=g),
                               torch.randint(0, 16, (2, W * W), generator=g), 50)
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_oracle_without_gmlp_layers_is_the_sandwich_oracle_bit_for_bit(bf16):
    cfg, params, tokens = _model(3, types=("global", "local"))
    a = OM.forward(params, tokens, cfg, bf16=bf16)
    b = OSW.forward(params, tokens, cfg, bf16=bf16, sandwich_norm=False)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_perturbing_a_token_leaves_every_earlier_output_bit_identical(bf16):
    cfg, params, tokens = _model(5, types=("mlp", "mlp"))
    _, _, base = OM.forward(params, tokens, cfg, bf16=bf16)
    for j in (5, 30, 63):
        t2 = tokens.clone()
        t2[:, j] = (t2[:, j] + 1) % cfg.total_tokens
        _, _, pert = OM.forward(params, t2, cfg, bf16=bf16)
        assert torch.equal(pert[:, :j], base[:, :j])
        assert not torch.equal(pert[:, j:], base[:, j:])


def test_zero_mixing_weight_and_unit_bias_give_res():
    g = torch.Generator().manual_seed(0)
    u = torch.randn(2, 64, 32, generator=g)
    h, mixed = OM.sgu(u, torch.ones(16), torch.zeros(16), torch.zeros(64, 64), torch.ones(64), 1e-5)
    assert torch.equal(h, u[..., :16]) and torch.equal(mixed, torch.ones_like(mixed))


@pytest.mark.parametrize("mutate", OM.MUTATIONS)
def test_each_mutant_differs_from_the_oracle(mutate):
    cfg, params, tokens = _model(7)
    if mutate == "unmasked":   # a weight that breaks causality: only then does the mask matter
        params = dict(params)
        params["layer_1/gmlp/sgu/weight"] = params["layer_1/gmlp/sgu/weight"] + 0.1 * torch.triu(
            torch.ones(cfg.seq_len, cfg.seq_len), 1)
    ref = OM.forward(params, tokens, cfg)[2]
    mut = OM.forward(params, tokens, cfg, gmlp_mutate=mutate)[2]
    assert (mut - ref).abs().max() > 1e-4


def test_engine_initialisation_starts_near_the_identity_gate():
    cfg = OL.LocalConfig(64, 1, 2, 50, 16, 28, 36, attention_types=("mlp",))
    p = OM.init_params(O.init_params(cfg, 0), cfg)
    w = p["layer_0/gmlp/sgu/weight"]
    assert torch.equal(torch.triu(w, 1), torch.zeros_like(w)) and w.abs().max() <= 1e-3 / 64
    assert torch.equal(p["layer_0/gmlp/sgu/bias"], torch.ones(64))
