"""CPU side of the GELU MLP: the activation_function key at the three places a model is built, the engine's argument
check, generate_dalle.py handing the key to the engine, and the oracle's GELU (against torch's float64 tanh GELU and
its closed-form derivative) and ReLU (bit for bit what the oracles computed before the switch existed)."""
import json
import math

import pytest
import torch
import torch.nn.functional as F

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import ACTIVATIONS, DalleEngine, validate_activation
from dalle_mtf_b200.model_fns import activation_function, dalle_model_fn
from dalle_mtf_b200.models import DALLE
from dalle_mtf_b200.utils import save_checkpoint
from oracle import dalle as O
from oracle import dalle_dropout as OD
from oracle import dalle_gelu as OG
from oracle import dalle_local as OL

ACCEPTED = [({}, "relu"), ({"activation_function": None}, "relu"), ({"activation_function": "relu"}, "relu"),
            ({"activation_function": "gelu"}, "gelu")]
REJECTED = ["GELU", "Gelu", "swish", "gelu_new", "tanh", "", True, False, 0, 1, 1.0, ["gelu"]]


@pytest.mark.parametrize("params,want", ACCEPTED)
def test_accepted_values(params, want):
    assert activation_function(params) == want


@pytest.mark.parametrize("value", REJECTED, ids=[repr(v) for v in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    p = {"activation_function": value}
    with pytest.raises(ValueError, match="activation_function"):
        activation_function(p)
    with pytest.raises(ValueError, match="activation_function"):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="activation_function"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match="activation_function"):
        G.main(_generate_config(tmp_path, p))


def test_engine_validates_its_argument_before_any_device_work():
    assert ACTIVATIONS == ("relu", "gelu")
    for a in ACTIVATIONS:
        assert validate_activation(a) == a
    for bad in [None, "GELU", "swish", True, 1]:
        with pytest.raises(ValueError, match="activation"):
            validate_activation(bad)
        with pytest.raises(ValueError, match="activation"):
            DalleEngine(256, 1, 2, 10, 16, 4, 16, activation=bad)


def test_a_custom_activation_fn_stays_rejected():
    from dalle_mtf_b200 import lib as L
    with pytest.raises(L.DB200Error, match="activation_function"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              activation_fn=torch.relu)


def _generate_config(tmp_path, extra):
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, "n_embd": 256, "n_layers": 1, "n_heads": 2, **extra}
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    import numpy as np
    np.save(tmp_path / "ids.npy", np.zeros((1, 4), np.int32))
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})
    return ["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
            "--caption_ids", str(tmp_path / "ids.npy")]


class _Built(Exception):
    pass


@pytest.mark.parametrize("extra,want", [({}, "relu"), ({"activation_function": "gelu"}, "gelu")])
def test_generate_cli_builds_the_engine_with_the_config_activation(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the activation it was trained with: the engine it builds gets the
    config's key (the device work that follows is stubbed out)."""
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
    assert seen["activation"] == want


def test_example_gelu_config_is_the_example_plus_the_key():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "dalle_example_b200.json")) as f:
        base = json.load(f)
    with open(os.path.join(root, "configs", "dalle_example_gelu_b200.json")) as f:
        gelu = json.load(f)
    assert gelu.pop("activation_function") == "gelu"
    assert gelu.pop("model_path") != base.pop("model_path")
    assert gelu == base


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_gelu_is_torch_tanh_gelu_and_its_derivative_the_closed_form():
    z = torch.linspace(-12, 12, 20001, dtype=torch.float64)
    assert torch.allclose(OG.gelu(z), F.gelu(z, approximate="tanh"), rtol=1e-12, atol=1e-15)
    zz = z.clone().requires_grad_(True)
    F.gelu(zz, approximate="tanh").sum().backward()
    assert torch.allclose(OG.gelu_grad(z), zz.grad, rtol=1e-10, atol=1e-12)
    # the activation helper: gelu of the bf16-rounded pre-activation with bf16, plain gelu without
    y = torch.randn(1000, dtype=torch.float64) * 3
    assert torch.equal(OG.mlp_activation(y, "gelu"), OG.gelu(y))
    r = y.float().to(torch.bfloat16).float()
    assert torch.equal(OG.mlp_activation(y.float(), "gelu", bf16=True), OG.gelu(r))
    # the mutant drops the cubic term: about 0.03 at x = 2
    two = torch.tensor([2.0], dtype=torch.float64)
    diff = (OG.mlp_activation(two, "gelu") - OG.mlp_activation(two, "gelu", mutate="gelu_no_cubic")).item()
    assert 0.02 < abs(diff) < 0.04, diff
    with pytest.raises(ValueError):
        OG.mlp_activation(y, "swish")
    with pytest.raises(ValueError):
        OG.mlp_activation(y, "gelu", mutate="other")


def test_relu_rounding_commutes_with_the_nonlinearity():
    g = torch.Generator().manual_seed(0)
    y = torch.randn(100000, generator=g) * torch.logspace(-40, 38, 100000).float()
    y = torch.cat([y, -y, torch.tensor([0.0, -0.0, float("inf"), -float("inf")])])
    a = O._r(torch.relu(y), True)
    b = O._r(OG.mlp_activation(y, "relu", bf16=True), True)
    nz = a != 0          # zeros may differ in sign only (relu(-0) keeps -0); every other value bit for bit
    assert torch.equal(a, b) and torch.equal(a[nz].view(torch.int32), b[nz].view(torch.int32))


def _tiny():
    cfg = O.DalleConfig(64, 2, 2, 50, 16, 6, 10)
    p = O.init_params(cfg, 1)
    g = torch.Generator().manual_seed(2)
    for k in p:
        if k.endswith("bias") or k.endswith("/b"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (2, cfg.seq_len), generator=g)
    return cfg, p, tokens


def _bitwise(a, b):
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k


@pytest.mark.parametrize("bf16", [False, True])
def test_relu_is_bit_identical_to_every_oracle_forward_that_restates_the_mlp(bf16):
    """With activation "relu" the parameterised forward computes bit for bit what the unchanged oracles compute (so the
    golden fixtures, which those oracles produce, are untouched): oracle.dalle, oracle.dalle_dropout,
    oracle.dalle_local and the axial and conv oracles of tests/."""
    import axial_oracle as OA
    import conv_oracle as OC
    cfg, p, tokens = _tiny()
    _bitwise(OG.loss_and_grads(p, tokens, cfg, bf16=bf16), O.loss_and_grads(p, tokens, cfg, bf16=bf16))
    spec = ((0.1, 0.1, 0.1), 5, 2, 0)
    _bitwise(OG.loss_and_grads(p, tokens, cfg, spec, bf16=bf16), OD.loss_and_grads(p, tokens, cfg, spec, bf16=bf16))
    lcfg = OL.LocalConfig(64, 2, 2, 50, 16, 6, 10, attention_types=("global", "local"), local_attention_radius=3)
    for sp in (None, spec):
        _bitwise(OG.loss_and_grads(p, tokens, lcfg, sp, bf16=bf16), OL.loss_and_grads(p, tokens, lcfg, sp, bf16=bf16))
    ctok = torch.randint(0, cfg.total_tokens - 1, (2, 7 + 9), generator=torch.Generator().manual_seed(3))
    acfg = OA.AxialConfig(64, 2, 2, 50, 16, 7, 9, attention_types=("axial_row", "axial_col"), local_attention_radius=3)
    ccfg = OC.ConvConfig(64, 2, 2, 50, 16, 7, 9, attention_types=("axial_row", "conv"), local_attention_radius=3,
                         conv_attention_kernel=2)
    for sp in (None, spec):
        _bitwise(OG.loss_and_grads(p, ctok, acfg, sp, bf16=bf16, layers=OA),
                 OA.loss_and_grads(p, ctok, acfg, sp, bf16=bf16))
        _bitwise(OG.loss_and_grads(p, ctok, ccfg, sp, bf16=bf16, layers=OC),
                 OC.loss_and_grads(p, ctok, ccfg, sp, bf16=bf16))


def test_gelu_and_its_mutant_change_the_forward_and_arguments_are_checked():
    import conv_oracle as OC
    cfg, p, tokens = _tiny()
    relu = OG.forward(p, tokens, cfg)[0]
    gelu = OG.forward(p, tokens, cfg, activation="gelu")[0]
    mut = OG.forward(p, tokens, cfg, activation="gelu", mutate="gelu_no_cubic")[0]
    assert torch.equal(relu, O.forward(p, tokens, cfg)[0])
    assert not torch.equal(gelu, relu) and not torch.equal(mut, gelu) and math.isfinite(gelu.item())
    # with dropout rates of 0 the dropout path is the same computation
    assert torch.equal(OG.forward(p, tokens, cfg, ((0.0, 0.0, 0.0), 0, 0, 0), activation="gelu")[0], gelu)
    for kw in ({"activation": "swish"}, {"activation": "relu", "mutate": "gelu_no_cubic"},
               {"activation": "gelu", "mutate": "other"}):
        with pytest.raises(ValueError):
            OG.forward(p, tokens, cfg, **kw)
    ccfg = OC.ConvConfig(64, 2, 2, 50, 16, 7, 9, attention_types=("axial_row", "conv"), conv_attention_kernel=2)
    with pytest.raises(ValueError, match="layers="):   # a config whose attention masks live elsewhere
        OG.forward(p, tokens[:, :16], ccfg)
