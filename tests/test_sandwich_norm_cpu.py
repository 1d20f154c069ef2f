"""CPU side of the sandwich LayerNorm: the sandwich_norm key at every place a model is built, generate_dalle.py handing
it to the engine, the parameter layout (names, shapes, bucket spans, the fp32 vector table, weight decay) and count,
and the oracle (bit for bit the token-shift oracle with the key off, and four mutants that change the output)."""
import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import DalleEngine, param_layout, validate_sandwich_norm
from dalle_mtf_b200.model_fns import dalle_model_fn, sandwich_norm
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_glu as OGL
from oracle import dalle_sandwich as OSW
from oracle import dalle_shift as OS
from test_gelu_cpu import _Built, _generate_config

NEW = ("lna_g", "lna_b", "lnm_g", "lnm_b")


# ------------------------------------------------------------------------------------------------ config values
ACCEPTED = [({}, False), ({"sandwich_norm": None}, False), ({"sandwich_norm": False}, False),
            ({"sandwich_norm": True}, True)]
REJECTED = [1, 0, 1.0, "true", "false", "", [], [True], {"on": True}]


@pytest.mark.parametrize("params,want", ACCEPTED)
def test_accepted_values(params, want):
    assert sandwich_norm(params) is want


@pytest.mark.parametrize("value", REJECTED, ids=[repr(v) for v in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    p = {"sandwich_norm": value}
    with pytest.raises(ValueError, match="sandwich_norm"):
        sandwich_norm(p)
    with pytest.raises(ValueError, match="sandwich_norm"):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="sandwich_norm"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match="sandwich_norm"):
        G.main(_generate_config(tmp_path, p))


def test_engine_validates_its_argument_before_any_device_work():
    for v in (True, False):
        assert validate_sandwich_norm(v) is v
    for bad in [None, 1, 0, "true", [], [True]]:
        with pytest.raises(ValueError, match="sandwich_norm"):
            validate_sandwich_norm(bad)
        with pytest.raises(ValueError, match="sandwich_norm"):
            DalleEngine(256, 1, 2, 10, 16, 4, 16, sandwich_norm=bad)


@pytest.mark.parametrize("extra,want", [({}, False), ({"sandwich_norm": None}, False),
                                        ({"sandwich_norm": True}, True)])
def test_generate_cli_builds_the_engine_with_the_config_key(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the sandwich LayerNorm it was trained with (device work stubbed)."""
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
    assert seen["sandwich_norm"] is want


# ------------------------------------------------------------------------------------------------ layout
def _bare_engine(d, Lyr, tv, iv, tl, il, sandwich, gated=False):
    """A DalleEngine with only the fields n_params / _ref_names / _decay_segments read (no device)."""
    e = DalleEngine.__new__(DalleEngine)
    e.d, e.L, e.text_seq_len, e.image_seq_len = d, Lyr, tl, il
    e.V, e.S = tv + iv + 1, tl + il
    e.row_col, e.grid_w, e.gated_mlp, e.sandwich_norm = False, None, gated, sandwich
    e.layout = param_layout(d, Lyr, e.V, e.S, gated_mlp=gated, sandwich_norm=sandwich)
    return e


@pytest.mark.parametrize("d,Lyr,gated", [(256, 2, False), (512, 6, False), (4096, 1, True)])
def test_layout_names_and_count(d, Lyr, gated):
    V, S = 300 + 64 + 1, 88
    plain = param_layout(d, Lyr, V, S, gated_mlp=gated)
    sand = param_layout(d, Lyr, V, S, gated_mlp=gated, sandwich_norm=True)
    added = [k for k in sand.order if k not in plain.entries]
    assert added == [f"l{i}.{n}" for i in range(Lyr) for n in NEW]
    assert [k for k in sand.order if k in plain.entries] == plain.order
    assert all(sand.entries[k][1] == (d,) for k in added)
    assert all(sand.entries[k][0] % 64 == 0 for k in sand.order)
    n0 = _bare_engine(d, Lyr, 300, 64, 24, 64, False, gated).n_params()
    n1 = _bare_engine(d, Lyr, 300, 64, 24, 64, True, gated).n_params()
    assert n1 - n0 == Lyr * 4 * d
    count = lambda lay: sum(torch.Size(s).numel() for k, (_, s) in lay.entries.items() if k not in ("wout", "bout"))
    assert n1 == count(sand) + d * V + V
    e = _bare_engine(d, Lyr, 300, 64, 24, 64, True, gated)
    names = [rn for i in range(Lyr) for k, rn in e._layer_ref_names(i).items() if k in NEW]
    assert names == OSW.norm_names(Lyr)
    assert all(k not in NEW for i in range(Lyr) for k in e._ref_names(i))      # the plain model's names unchanged


def test_new_vectors_sit_in_their_layer_bucket_in_the_vector_table_and_are_not_decayed():
    d, Lyr = 256, 3
    e = _bare_engine(d, Lyr, 300, 64, 24, 64, True)
    lay = e.layout
    for i in range(Lyr):
        s, end = lay.span(f"l{i}.ln1_g", f"l{i}.lnm_b")
        for n in NEW:
            o, shp = lay.entries[f"l{i}.{n}"]
            assert s <= o and o + shp[0] <= end, n
        if i + 1 < Lyr:
            assert end <= lay.entries[f"l{i + 1}.ln1_g"][0]          # buckets of adjacent layers do not overlap
    assert end <= lay.entries["lnf_g"][0]
    assert set(NEW) <= set(DalleEngine.VECTOR_PARAMS)
    for name in lay.order:
        if name.split(".")[-1] in NEW:
            o, _ = lay.entries[name]
            assert any(s <= o < t and not decays for s, t, decays in e._decay_segments()), name
    decayed = sum(t - s for s, t, dec in e._decay_segments() if dec)
    plain = _bare_engine(d, Lyr, 300, 64, 24, 64, False)
    assert decayed == sum(t - s for s, t, dec in plain._decay_segments() if dec)


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, d=64, Lyr=2, H=2, TL=6, W=3):
    cfg = O.DalleConfig(d, Lyr, H, 50, 16, TL, W * W)
    params = OSW.init_params(O.init_params(cfg, seed), cfg, seed + 2)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("o_b") or k.endswith("mlp_linear_2/bias"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.05
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, TL), generator=g),
                               torch.randint(0, 16, (2, W * W), generator=g), 50)
    return cfg, params, tokens


@pytest.mark.parametrize("variant", [dict(), dict(gated=True, activation="gelu", rotary=(16, 10000.0)),
                                     dict(shift_tokens=True)], ids=["plain", "geglu_rotary", "shift"])
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_oracle_without_the_key_is_the_shift_oracle_bit_for_bit(variant, bf16):
    cfg, params, tokens = _model(3)
    if variant.get("gated"):
        params = OGL.init_params(params, cfg, 4)
    base = {k: v for k, v in params.items() if "/norm_out/" not in k}
    kw = dict(bf16=bf16, **{"shift_tokens": False, **variant})
    a = OSW.loss_and_grads(params, tokens, cfg, sandwich_norm=False, **kw)
    b = OS.loss_and_grads(base, tokens, cfg, **kw)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert all(torch.equal(a[3][k], b[3][k]) for k in b[3])
    assert all(not a[3][k].any() for k in OSW.norm_names(cfg.n_layers))


def test_oracle_with_dropout_and_without_the_key_is_the_shift_oracle_bit_for_bit():
    cfg, params, tokens = _model(4)
    dropout = ((0.1, 0.1, 0.2), 7, 3, 0)
    base = {k: v for k, v in params.items() if "/norm_out/" not in k}
    a = OSW.forward(params, tokens, cfg, dropout, sandwich_norm=False)
    b = OS.forward(base, tokens, cfg, dropout, shift_tokens=False)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_the_norms_and_each_mutant_change_the_output():
    cfg, params, tokens = _model(5, d=128)
    dropout = ((0.0, 0.0, 0.3), 11, 2, 0)            # residual dropout: norm_before_drop differs only with it
    off = OSW.forward(params, tokens, cfg, dropout, sandwich_norm=False)[2]
    ref = OSW.forward(params, tokens, cfg, dropout)[2]
    assert ((ref - off).norm() / off.norm()).item() > 1e-3
    for m in OSW.MUTATIONS:
        mut = OSW.forward(params, tokens, cfg, dropout, sandwich_mutate=m)[2]
        rel = ((mut - ref).norm() / ref.norm()).item()
        assert rel > 1e-3, (m, rel)
    ign = OSW.forward(params, tokens, cfg, dropout, sandwich_mutate="ignored")[2]
    assert torch.equal(ign, off)
    with pytest.raises(ValueError):
        OSW.forward(params, tokens, cfg, sandwich_mutate="nope")
    with pytest.raises(ValueError):
        OSW.forward(params, tokens, cfg, sandwich_norm=False, sandwich_mutate="swapped")


def test_unit_norms_at_initialisation_still_normalise_the_branch():
    """g = 1, b = 0 (the engine's initialisation) is not the identity: each branch output enters the residual stream
    with zero mean and unit variance per row."""
    cfg, params, tokens = _model(6)
    params = OSW.init_params({k: v for k, v in params.items() if "/norm_out/" not in k}, cfg)
    assert all(torch.equal(params[k], torch.ones(cfg.n_embd) if k.endswith("/g") else torch.zeros(cfg.n_embd))
               for k in OSW.norm_names(cfg.n_layers))
    off = OSW.forward(params, tokens, cfg, sandwich_norm=False)[2]
    on = OSW.forward(params, tokens, cfg)[2]
    assert ((on - off).norm() / off.norm()).item() > 1e-3
