"""CPU tests of local (sliding-window) attention layers: the attention_types / local_attention_radius config keys, the
oracle's per-layer window (src/dalle_mtf/models.py:257-273: query i sees keys (i - r, i]), the absence of attention
dropout in local layers, and the plumbing of both keys from models.DALLE and generate_dalle.py into DalleEngine."""
import json
import os
from collections import defaultdict

import numpy as np
import pytest
import torch

from dalle_mtf_b200.dalle_engine import layer_radii
from dalle_mtf_b200.model_fns import attention_layers
from oracle import dalle as O
from oracle import dalle_dropout as D
from oracle import dalle_local as OL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------- config
def test_attention_types_expand_in_gpt_neo_form():
    p = {"n_layers": 6, "attention_types": [[["global", "local"], 3]]}
    assert attention_layers(p) == (["global", "local"] * 3, 256)
    p = {"n_layers": 5, "attention_types": [[["local"], 2], [["global", "local", "global"], 1]],
         "local_attention_radius": 64}
    assert attention_layers(p) == (["local", "local", "global", "local", "global"], 64)


def test_missing_or_null_keys_mean_every_layer_global_with_radius_256():
    assert attention_layers({"n_layers": 3}) == (None, 256)
    assert attention_layers(defaultdict(lambda: None, {"n_layers": 3})) == (None, 256)
    assert attention_layers({"n_layers": 3, "local_attention_radius": 1}) == (None, 1)
    assert layer_radii(None, 256, 3) == [None, None, None]
    assert layer_radii(["local", "global"], 7, 2) == [7, None]


@pytest.mark.parametrize("extra", [
    {"local_attention_radius": 0},
    {"local_attention_radius": -3},
    {"local_attention_radius": 2.5},
    {"local_attention_radius": True},
    {"local_attention_radius": "256"},
    {"attention_types": "local"},                                  # not a list of items
    {"attention_types": [["global", "local"], 2]},                 # item is not [[types], count]
    {"attention_types": [[["global", "local"], 1]]},               # expands to 2 layers, n_layers 4
    {"attention_types": [[["global", "local"], 3]]},               # 6 layers
    {"attention_types": [[["global", "sparse"], 2]]},              # unknown type
    {"attention_types": [[["global", "local"], 0], [["local"], 4]]},
    {"attention_types": [[["global", "local"], 2.0]]},
    {"attention_types": [[["global", "local"], True], [["local"], 3]]},
])
def test_bad_attention_config_is_rejected_with_a_message(extra):
    with pytest.raises(ValueError, match="attention_types|local_attention_radius"):
        attention_layers({"n_layers": 4, **extra})


def test_engine_rejects_bad_layer_types():
    for types, r in ((["global"], 4), (["global", "dense"], 4), (["local", "local"], 0), (["local", "local"], 1.5)):
        with pytest.raises(ValueError):
            layer_radii(types, r, 2)


def test_the_example_config_is_the_measured_workload():
    with open(os.path.join(ROOT, "configs", "dalle_example_local_b200.json")) as f:
        local = json.load(f)
    with open(os.path.join(ROOT, "configs", "dalle_example_b200.json")) as f:
        base = json.load(f)
    assert attention_layers(local) == (["global", "local"] * 3, 256)
    differ = {k for k in set(local) | set(base) if local.get(k) != base.get(k)}
    assert differ == {"attention_types", "local_attention_radius", "model_path"}


# ------------------------------------------------------------------------------------------------------- oracle
def _case(types=None, radius=256, seed=0, B=2, ts=12, isl=20, L=2, dtype=torch.float32):
    cfg = OL.LocalConfig(64, L, 2, 100, 30, ts, isl, attention_types=types, local_attention_radius=radius)
    params = {k: v.to(dtype) for k, v in O.init_params(cfg, seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True])
def test_radius_at_least_s_is_global_attention_bit_for_bit(bf16):
    cfg, params, tokens = _case()
    S = cfg.seq_len
    _, lb, logits = O.forward(params, tokens, cfg, bf16=bf16)
    for r in (S, S + 1, 10 * S):
        for types in (("local", "local"), ("global", "local")):
            lcfg = OL.LocalConfig(*[getattr(cfg, f) for f in ("n_embd", "n_layers", "n_heads", "text_vocab_size",
                                                              "image_vocab_size", "text_seq_len", "image_seq_len")],
                                  attention_types=types, local_attention_radius=r)
            _, lb2, logits2 = OL.forward(params, tokens, lcfg, bf16=bf16)
            assert torch.equal(logits, logits2) and torch.equal(lb, lb2)
    # no attention_types, and an explicit all-global list, are oracle.dalle.forward bit for bit
    assert torch.equal(OL.forward(params, tokens, _case()[0], bf16=bf16)[2], logits)
    gcfg = OL.LocalConfig(64, 2, 2, 100, 30, 12, 20, attention_types=("global", "global"), local_attention_radius=3)
    assert torch.equal(OL.forward(params, tokens, gcfg, bf16=bf16)[2], logits)
    assert not torch.equal(OL.forward(params, tokens, _case(("global", "local"), 3)[0], bf16=bf16)[2], logits)


def test_radius_one_attends_to_itself_only():
    cfg = _case(("local",), radius=1, L=1)[0]
    S = cfg.seq_len
    mask = OL.attention_mask(cfg, 0, S, O.Quirks())
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(2, S, 2, 32, generator=g) * 3 for _ in range(3))
    p = torch.softmax(torch.einsum("bihe,bjhe->bhij", q, k) + mask, dim=-1)
    assert torch.equal(p, torch.eye(S).expand_as(p))
    assert torch.equal(torch.einsum("bhij,bjhe->bihe", p, v), v)


@pytest.mark.parametrize("radius", [1, 2, 5, 31, 32])
def test_window_matches_brute_force_masked_softmax(radius):
    """A one-layer local model in float64 against a restatement that computes every query's softmax over the keys
    max(0, i - r + 1) .. i by explicit slicing."""
    cfg, params, tokens = _case(("local",), radius, L=1, dtype=torch.float64)
    B, S = tokens.shape
    H, dh = cfg.n_heads, cfg.head_dim
    _, _, logits = OL.forward(params, tokens, cfg)
    P = params
    x = P["embedding/wte"][tokens] + P["positional_embedding/wpe"][:S]
    h = O.layer_norm(x, P["layer_0/norm_1/g"], P["layer_0/norm_1/b"], 1e-5)
    q, k, v = ((h @ P[f"layer_0/attn/{n}"]).view(B, S, H, dh) for n in "qkv")
    a = torch.empty(B, S, H, dh, dtype=torch.float64)
    for i in range(S):
        lo = max(0, i - radius + 1)
        w = torch.softmax(torch.einsum("bhe,bjhe->bhj", q[:, i], k[:, lo:i + 1]), -1)
        a[:, i] = torch.einsum("bhj,bjhe->bhe", w, v[:, lo:i + 1])
    x = x + a.reshape(B, S, H * dh) @ P["layer_0/attn/o"] + P["layer_0/attn/compute_output_bias/o_b"]
    h = O.layer_norm(x, P["layer_0/norm_2/g"], P["layer_0/norm_2/b"], 1e-5)
    x = x + torch.relu(h @ P["layer_0/mlp/mlp_linear_1/kernel"] + P["layer_0/mlp/mlp_linear_1/bias"]) @ \
        P["layer_0/mlp/mlp_linear_2/kernel"] + P["layer_0/mlp/mlp_linear_2/bias"]
    hf = O.layer_norm(x, P["to_logits/layer_norm/g"], P["to_logits/layer_norm/b"], 1e-5)
    ref = hf @ P["to_logits/linear_out/kernel"] + P["to_logits/linear_out/bias"]
    assert torch.allclose(logits, ref, rtol=1e-10, atol=1e-10)


def test_local_layers_have_no_attention_dropout_and_keep_residual_dropout():
    types = ("global", "local")
    cfg, params, tokens = _case(types, radius=4)
    B = tokens.shape[0]
    spec = lambda rates: (rates, 7, 3, 1)
    dm = OL.dropout_masks(spec((0.1, 0.3, 0.2)), B, cfg)
    assert dm["attn"][0] is not None and dm["attn"][1] is None
    assert all(m is not None for m in dm["attn_out"] + dm["mlp_out"])
    # the global layer's masks are those of an all-global model: site numbers do not move
    gm = D.dropout_masks(spec((0.1, 0.3, 0.2)), B, _case()[0])
    assert torch.equal(dm["attn"][0], gm["attn"][0]) and torch.equal(dm["attn_out"][1], gm["attn_out"][1])
    # all-local: attention dropout changes nothing, residual dropout does
    lcfg = _case(("local", "local"), radius=4)[0]
    plain = OL.forward(params, tokens, lcfg, spec((0.0, 0.0, 0.0)))[2]
    assert torch.equal(OL.forward(params, tokens, lcfg, spec((0.0, 0.5, 0.0)))[2], plain)
    assert not torch.equal(OL.forward(params, tokens, lcfg, spec((0.0, 0.0, 0.3)))[2], plain)
    # with every rate 0 the dropout path is the eval path, local layers included
    assert torch.equal(plain, OL.forward(params, tokens, lcfg)[2])
    # and the mixed model's global layer still drops attention weights
    mixed = _case(types, radius=4)[0]
    assert not torch.equal(OL.forward(params, tokens, mixed, spec((0.0, 0.5, 0.0)))[2],
                           OL.forward(params, tokens, mixed, spec((0.0, 0.0, 0.0)))[2])
    # with every layer global the module is oracle.dalle_dropout.forward bit for bit
    for bf16 in (False, True):
        for rates in ((0.1, 0.3, 0.2), (0.0, 0.0, 0.0)):
            want = D.forward(params, tokens, _case()[0], spec(rates), bf16=bf16)
            got = OL.forward(params, tokens, _case()[0], spec(rates), bf16=bf16)
            assert all(torch.equal(a, b) for a, b in zip(want, got))


# ------------------------------------------------------------------------------------------------------- plumbing
class _Stop(Exception):
    pass


class _FakeEngine:
    calls = []

    def __init__(self, *args, **kw):
        _FakeEngine.calls.append((args, kw))
        if kw.pop("_stop", True):
            raise _Stop

    def init_params(self, seed=0):
        pass


def test_dalle_class_passes_the_layer_types_to_the_engine(monkeypatch):
    from dalle_mtf_b200 import models

    class Eng(_FakeEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, _stop=False, **kw)

    monkeypatch.setattr(models, "DalleEngine", Eng)
    _FakeEngine.calls.clear()
    models.DALLE(256, n_layers=4, params={"attention_types": [[["local", "global"], 2]], "local_attention_radius": 64})
    models.DALLE(256, n_layers=2, params={})
    (_, kw1), (_, kw2) = _FakeEngine.calls
    assert kw1["attention_types"] == ["local", "global", "local", "global"] and kw1["local_attention_radius"] == 64
    assert kw2["attention_types"] is None and kw2["local_attention_radius"] == 256
    with pytest.raises(ValueError, match="attention_types"):
        models.DALLE(256, n_layers=3, params={"attention_types": [[["local", "global"], 2]]})


def test_generate_dalle_builds_the_engine_with_the_trained_layer_types(tmp_path, monkeypatch):
    import generate_dalle as G
    from dalle_mtf_b200 import dalle_engine, lib, model_fns
    from dalle_mtf_b200.utils import save_checkpoint
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, "n_embd": 256, "n_layers": 4, "n_heads": 2,
             "attention_types": [[["global", "local"], 2]], "local_attention_radius": 9}
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    np.save(tmp_path / "ids.npy", np.zeros((1, 4), np.int32))
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})

    class Vae:
        K, image_seq_len = 64, 16

        def load_params(self, named):
            pass

    monkeypatch.setattr(lib, "require_device", lambda: None)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(model_fns, "load_vae_model", lambda params, device: (Vae(), None))
    monkeypatch.setattr(dalle_engine, "DalleEngine", _FakeEngine)
    _FakeEngine.calls.clear()
    with pytest.raises(_Stop):
        G.main(["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
                "--caption_ids", str(tmp_path / "ids.npy")])
    (args, kw), = _FakeEngine.calls
    assert args[:3] == (256, 4, 2)
    assert kw["attention_types"] == ["global", "local", "global", "local"] and kw["local_attention_radius"] == 9
    dalle["attention_types"] = [[["global", "local"], 1]]                  # 2 types for 4 layers
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    with pytest.raises(ValueError, match="n_layers"):
        G.main(["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
                "--caption_ids", str(tmp_path / "ids.npy")])
