"""CPU side of the gated MLP: the gated_mlp key at every place a model is built, the engine's argument check,
generate_dalle.py handing the key to the engine, the parameter layout and count, and the oracle (DALLE-pytorch's
chunk order in float64, bit for bit the ungated oracle with the key off, and two mutants that change the output)."""

import pytest
import torch
import torch.nn.functional as F

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import ACTIVATIONS, DalleEngine, param_layout, validate_gated_mlp
from dalle_mtf_b200.model_fns import dalle_model_fn, gated_mlp
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_gelu as OG
from oracle import dalle_glu as OGL
from test_gelu_cpu import _Built, _generate_config

ACCEPTED = [({}, False), ({"gated_mlp": None}, False), ({"gated_mlp": False}, False), ({"gated_mlp": True}, True)]
REJECTED = [1, 0, 1.0, "true", "false", "", [True], {"on": True}]


@pytest.mark.parametrize("params,want", ACCEPTED)
def test_accepted_values(params, want):
    assert gated_mlp(params) is want


@pytest.mark.parametrize("value", REJECTED, ids=[repr(v) for v in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    p = {"gated_mlp": value}
    with pytest.raises(ValueError, match="gated_mlp"):
        gated_mlp(p)
    with pytest.raises(ValueError, match="gated_mlp"):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="gated_mlp"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match="gated_mlp"):
        G.main(_generate_config(tmp_path, p))


def test_engine_validates_its_argument_before_any_device_work():
    assert ACTIVATIONS == ("relu", "gelu")                     # the key composes with activation_function
    for v in (True, False):
        assert validate_gated_mlp(v) is v
    for bad in [None, 1, 0, "true", [True]]:
        with pytest.raises(ValueError, match="gated_mlp"):
            validate_gated_mlp(bad)
        with pytest.raises(ValueError, match="gated_mlp"):
            DalleEngine(256, 1, 2, 10, 16, 4, 16, gated_mlp=bad)


@pytest.mark.parametrize("extra,want", [({}, False), ({"gated_mlp": True}, True),
                                        ({"gated_mlp": True, "activation_function": "gelu"}, True)])
def test_generate_cli_builds_the_engine_with_the_config_key(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the MLP it was trained with (the device work is stubbed out)."""
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
    assert seen["gated_mlp"] is want
    assert seen["activation"] == extra.get("activation_function", "relu")


# ------------------------------------------------------------------------------------------------ parameters
def _bare_engine(d, Lyr, tv, iv, tl, il, gated):
    """A DalleEngine with only the attributes n_params reads (no device)."""
    e = DalleEngine.__new__(DalleEngine)
    e.d, e.L, e.text_seq_len = d, Lyr, tl
    e.V, e.S = tv + iv + 1, tl + il
    e.row_col, e.grid_w, e.gated_mlp = False, None, gated
    return e


@pytest.mark.parametrize("d,Lyr", [(256, 2), (512, 6), (4096, 1)])
def test_layout_and_count_grow_by_the_gate_half(d, Lyr):
    V, S = 300 + 64 + 1, 88
    plain, gated = param_layout(d, Lyr, V, S), param_layout(d, Lyr, V, S, gated_mlp=True)
    for i in range(Lyr):
        assert plain.entries[f"l{i}.w1"][1] == (d, 4 * d) and plain.entries[f"l{i}.b1"][1] == (4 * d,)
        assert gated.entries[f"l{i}.w1"][1] == (d, 8 * d) and gated.entries[f"l{i}.b1"][1] == (8 * d,)
        assert gated.entries[f"l{i}.w2"][1] == (4 * d, d)
    assert list(gated.entries) == list(plain.entries)
    assert {k: v[1] for k, v in gated.entries.items() if not k.endswith((".w1", ".b1"))} == \
        {k: v[1] for k, v in plain.entries.items() if not k.endswith((".w1", ".b1"))}
    n0 = _bare_engine(d, Lyr, 300, 64, 24, 64, False).n_params()
    n1 = _bare_engine(d, Lyr, 300, 64, 24, 64, True).n_params()
    assert n1 - n0 == Lyr * (4 * d * d + 4 * d)
    count = lambda lay: sum(torch.Size(s).numel() for k, (_, s) in lay.entries.items() if k not in ("wout", "bout"))
    assert n0 == count(plain) + d * V + V and n1 == count(gated) + d * V + V


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, d=64, Lyr=2, H=2):
    cfg = O.DalleConfig(d, Lyr, H, 50, 16, 6, 10)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("mlp_linear_1/kernel"):
            params[k] = params[k] * 50.0        # z with std ~1: the curved part of GELU
        if k.endswith("mlp_linear_1/bias"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.5
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, 6), generator=g), torch.randint(0, 16, (2, 10), generator=g),
                               50)
    return cfg, params, tokens


def test_oracle_gelu_gate_is_dallepytorch_chunk_order_in_float64():
    """gated_mlp(y) of the oracle equals DALLE-pytorch's `x, g = y.chunk(2, -1); x * F.gelu(g, approximate="tanh")`
    restated in float64, which pins the value half first and the gate half second."""
    g = torch.Generator().manual_seed(0)
    y = torch.randn(5, 7, 2 * 256, generator=g, dtype=torch.float64) * 3
    x, gate = y.chunk(2, dim=-1)
    want = x * F.gelu(gate, approximate="tanh")
    got = OGL.gated_mlp(y, "gelu")
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-13)   # 1 + tanh(u) cancels in torch's negative tail
    assert not torch.allclose(gate * F.gelu(x, approximate="tanh"), want, rtol=1e-3)
    assert torch.equal(OGL.gated_mlp(y, "relu"), x * torch.relu(gate))


@pytest.mark.parametrize("act", ACTIVATIONS)
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_oracle_without_the_gate_is_the_ungated_oracle_bit_for_bit(act, bf16):
    cfg, params, tokens = _model(3)
    a = OGL.loss_and_grads(params, tokens, cfg, bf16=bf16, activation=act, gated=False)
    b = OG.loss_and_grads(params, tokens, cfg, bf16=bf16, activation=act)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert a[3].keys() == b[3].keys() and all(torch.equal(a[3][k], b[3][k]) for k in a[3])


@pytest.mark.parametrize("act", ACTIVATIONS)
def test_both_mutants_change_the_output(act):
    cfg, params, tokens = _model(4, d=128)
    params = OGL.init_params(params, cfg, 5)
    for k in params:
        if k.endswith("mlp_linear_1/kernel"):
            params[k][:, 4 * 128:] = params[k][:, 4 * 128:] * 50.0
    assert params["layer_0/mlp/mlp_linear_1/kernel"].shape == (128, 1024)
    ref = OGL.forward(params, tokens, cfg, activation=act)
    for m in OGL.MUTATIONS:
        mut = OGL.forward(params, tokens, cfg, activation=act, mutate=m)
        rel = ((mut[2] - ref[2]).norm() / ref[2].norm()).item()
        assert rel > 1e-3, (m, rel)
    with pytest.raises(ValueError):
        OGL.forward(params, tokens, cfg, activation=act, mutate="nope")
