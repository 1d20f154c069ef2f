"""CPU tests of axial (row and column) attention layers: parsing of the "axial_row" / "axial_col" attention types, the
reference masks against a brute-force definition from grid coordinates, the kernels' transposed ("kernel order")
formulation of the column mask, the absence of attention dropout in axial layers, the pair count the attention
profiler uses, and the plumbing of the layer types from models.DALLE and generate_dalle.py into DalleEngine."""
import json

import numpy as np
import pytest
import torch

import axial_oracle as OA
from dalle_mtf_b200 import dalle_engine, lib, ops
from dalle_mtf_b200.dalle_engine import layer_axial, layer_radii
from dalle_mtf_b200.model_fns import attention_layers
from oracle import dalle as O
from oracle import dalle_dropout as D
from oracle import dalle_local as OL


# ------------------------------------------------------------------------------------------------------- config
def test_axial_types_parse_and_mix_with_global_and_local_layers():
    p = {"n_layers": 6, "attention_types": [[["axial_row", "axial_col", "global"], 2]]}
    assert attention_layers(p) == (["axial_row", "axial_col", "global"] * 2, 256)
    p = {"n_layers": 4, "attention_types": [[["local", "axial_col"], 1], [["axial_row"], 2]],
         "local_attention_radius": 64}
    types, r = attention_layers(p)
    assert types == ["local", "axial_col", "axial_row", "axial_row"] and r == 64
    assert layer_radii(types, r, 4) == [64, None, None, None]
    assert layer_axial(types, 256, 1024, 4) == [None, (256, 32, 1), (256, 32, 0), (256, 32, 0)]
    assert layer_axial(["global", "local"], 256, 1000, 2) == [None, None]   # no axial layer: any image length
    assert layer_axial(None, 256, 1000, 3) == [None] * 3


@pytest.mark.parametrize("name", ["axial", "axial_rows", "row", "conv_like", "Axial_Row", "sparse"])
def test_unknown_attention_type_is_rejected(name):
    with pytest.raises(ValueError, match="attention_types"):
        attention_layers({"n_layers": 2, "attention_types": [[["axial_row", name], 1]]})
    with pytest.raises(ValueError, match="attention_types"):
        layer_radii(["axial_row", name], 256, 2)


@pytest.mark.parametrize("image_seq_len", [1000, 2, 15, 1023])
def test_axial_layers_reject_a_non_square_image_grid(image_seq_len, monkeypatch):
    with pytest.raises(ValueError, match="square"):
        layer_axial(["global", "axial_col"], 256, image_seq_len, 2)
    monkeypatch.setattr(lib, "require_device", lambda: None)
    with pytest.raises(ValueError, match="square"):
        dalle_engine.DalleEngine(256, 2, 2, 300, 64, 8, image_seq_len, attention_types=["axial_row", "global"])


def test_the_axial_example_config_is_dalle_example_with_axial_layers():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "dalle_example_axial_b200.json")) as f:
        axial = json.load(f)
    with open(os.path.join(root, "configs", "dalle_example_b200.json")) as f:
        base = json.load(f)
    assert attention_layers(axial) == (["axial_row", "axial_col", "global"] * 2, 256)
    assert {k for k in set(axial) | set(base) if axial.get(k) != base.get(k)} == {"attention_types", "model_path"}


# ------------------------------------------------------------------------------------------------------- masks
def _brute_force_visible(S, TL, W, axis):
    vis = torch.zeros(S, S, dtype=torch.bool)
    for i in range(S):
        for j in range(i + 1):
            if i < TL or j < TL:
                vis[i, j] = True
                continue
            (ri, ci), (rj, cj) = divmod(i - TL, W), divmod(j - TL, W)
            vis[i, j] = (ri == rj and cj <= ci) if axis == 0 else (ci == cj and rj <= ri)
    return vis


GEOMETRIES = [(12, 4, 16), (0, 3, 9), (5, 1, 6), (7, 5, 25), (7, 5, 19), (3, 6, 20), (16, 4, 10)]


@pytest.mark.parametrize("TL,W,S", GEOMETRIES)
@pytest.mark.parametrize("axis", [0, 1])
def test_oracle_mask_matches_the_grid_definition(TL, W, S, axis):
    cfg = OA.AxialConfig(64, 1, 2, 100, 30, TL, W * W, attention_types=(["axial_row", "axial_col"][axis],))
    mask = OA.attention_mask(cfg, 0, S, O.Quirks())
    want = _brute_force_visible(S, TL, W, axis)
    assert torch.equal(mask == 0, want)
    assert torch.equal(mask[~want], torch.full((int((~want).sum()),), O.Quirks().mask_value))


@pytest.mark.parametrize("TL,W,S", GEOMETRIES)
@pytest.mark.parametrize("axis", [0, 1])
def test_pair_count_matches_the_counted_mask(TL, W, S, axis):
    assert ops.attn_pairs_axial(S, TL, W, axis) == float(_brute_force_visible(S, TL, W, axis).sum())


def test_pair_count_at_dalle_example():
    # 256 text rows, a 32 x 32 grid: text triangle + every image row's text prefix + 32 triangles of 32 per grid line
    want = 256 * 257 // 2 + 1024 * 256 + 32 * (32 * 33 // 2)
    assert ops.attn_pairs_axial(1280, 256, 32, 0) == ops.attn_pairs_axial(1280, 256, 32, 1) == want


@pytest.mark.parametrize("TL,W", [(12, 4), (0, 3), (5, 1), (7, 5), (3, 6)])
def test_column_layer_is_the_segment_mask_in_kernel_order(TL, W):
    """Permuting the sequence by the column map and applying "text prefix + causal within segments of W" gives the
    reference's column-layer attention, output row for output row."""
    S = TL + W * W
    g = torch.Generator().manual_seed(TL * 31 + W)
    q, k, v = (torch.randn(S, 8, generator=g, dtype=torch.float64) for _ in range(3))
    col = OA.axial_hidden(S, TL, W, 1)
    want = torch.softmax((q @ k.T).masked_fill(col, float("-inf")), -1) @ v
    perm = OA.kernel_order(S, TL, W, 1)
    assert sorted(perm.tolist()) == list(range(S))
    seg = OA.segment_hidden(S, TL, W)
    got_k = torch.softmax((q[perm] @ k[perm].T).masked_fill(seg, float("-inf")), -1) @ v[perm]
    got = torch.empty_like(got_k)
    got[perm] = got_k
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    # in kernel order the row layer is the same segment mask without a permutation
    assert torch.equal(OA.axial_hidden(S, TL, W, 0), seg)


@pytest.mark.parametrize("TL,W", [(256, 32), (100, 24), (64, 80), (7, 1), (0, 24), (0, 40), (0, 3)])
def test_key_block_walk_covers_every_visible_pair(TL, W):
    """axial_oracle.key_blocks (the forward / dQ walk) visits each key block once, never past the query block, and
    every 64 x 64 tile of the kernel-order mask that holds a visible pair.  With TL = 0 and W = 24 query block 1 starts
    its walk at block 0, where its rows 72..127 see nothing."""
    S = TL + W * W
    n = -(-S // 64)
    pad = torch.zeros(n * 64, n * 64, dtype=torch.bool)
    pad[:S, :S] = ~OA.segment_hidden(S, TL, W)
    need = pad.view(n, 64, n, 64).any(3).any(1)
    for qb in range(n):
        blocks = OA.key_blocks(S, TL, W, qb)
        assert len(set(blocks)) == len(blocks) and all(0 <= j <= qb for j in blocks)
        assert set(need[qb].nonzero()[:, 0].tolist()) <= set(blocks), qb
    if (TL, W) == (0, 24):
        assert OA.key_blocks(S, 0, 24, 1) == [0, 1] and not pad[72:128, :64].any() and pad[64:72, 48:64].all()


# ------------------------------------------------------------------------------------------------------- oracle
def _case(types, seed=0, B=2, ts=5, isl=16, L=3, dtype=torch.float32):
    cfg = OA.AxialConfig(64, L, 2, 100, 30, ts, isl, attention_types=types, local_attention_radius=3)
    params = {k: v.to(dtype) for k, v in O.init_params(cfg, seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True])
def test_global_and_local_models_are_unchanged_bit_for_bit(bf16):
    for types in (None, ("global", "global", "global"), ("local", "global", "local")):
        cfg, params, tokens = _case(types)
        lcfg = OL.LocalConfig(*[getattr(cfg, f) for f in ("n_embd", "n_layers", "n_heads", "text_vocab_size",
                                                          "image_vocab_size", "text_seq_len", "image_seq_len")],
                              attention_types=types, local_attention_radius=3)
        spec = ((0.1, 0.3, 0.2), 7, 3, 1)
        for dropout in (None, spec):
            want = OL.forward(params, tokens, lcfg, dropout, bf16=bf16)
            got = OA.forward(params, tokens, cfg, dropout, bf16=bf16)
            assert all(torch.equal(a, b) for a, b in zip(want, got))
        if types is None:
            assert torch.equal(OA.forward(params, tokens, cfg, bf16=bf16)[2], O.forward(params, tokens, cfg,
                                                                                         bf16=bf16)[2])
    cfg, params, tokens = _case(("global", "axial_row", "axial_col"))
    assert not torch.equal(OA.forward(params, tokens, cfg)[2], OA.forward(params, tokens, _case(None)[0])[2])


def test_axial_layers_have_no_attention_dropout_and_keep_residual_dropout():
    types = ("global", "axial_row", "axial_col")
    cfg, params, tokens = _case(types)
    B = tokens.shape[0]
    spec = lambda rates: (rates, 7, 3, 1)
    dm = OA.dropout_masks(spec((0.1, 0.3, 0.2)), B, cfg)
    assert dm["attn"][0] is not None and dm["attn"][1] is None and dm["attn"][2] is None
    assert all(m is not None for m in dm["attn_out"] + dm["mlp_out"])
    gm = D.dropout_masks(spec((0.1, 0.3, 0.2)), B, _case(None)[0])         # site numbers do not move
    assert torch.equal(dm["attn"][0], gm["attn"][0])
    assert all(torch.equal(a, b) for a, b in zip(dm["attn_out"] + dm["mlp_out"], gm["attn_out"] + gm["mlp_out"]))
    acfg = _case(("axial_row", "axial_col", "axial_row"))[0]
    plain = OA.forward(params, tokens, acfg, spec((0.0, 0.0, 0.0)))[2]
    assert torch.equal(OA.forward(params, tokens, acfg, spec((0.0, 0.5, 0.0)))[2], plain)
    assert not torch.equal(OA.forward(params, tokens, acfg, spec((0.0, 0.0, 0.3)))[2], plain)
    assert torch.equal(plain, OA.forward(params, tokens, acfg)[2])
    assert not torch.equal(OA.forward(params, tokens, cfg, spec((0.0, 0.5, 0.0)))[2],
                           OA.forward(params, tokens, cfg, spec((0.0, 0.0, 0.0)))[2])


def test_engine_drops_attention_weights_only_in_global_layers():
    eng = dalle_engine.DalleEngine.__new__(dalle_engine.DalleEngine)
    eng.dropout, eng.dropout_seed, eng.S, eng.L = (0.1, 0.2, 0.3), 5, 21, 4
    eng.radii = [None, 3, None, None]
    eng.axial = [None, None, (5, 4, 0), (5, 4, 1)]
    dd = eng._dropout_descs(step=2, row0=0)
    assert dd["attn"][0] is not None and dd["attn"][1:] == [None, None, None]
    assert all(d is not None for d in dd["attn_out"] + dd["mlp_out"])


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


def test_dalle_class_passes_the_axial_types_to_the_engine(monkeypatch):
    from dalle_mtf_b200 import models

    class Eng(_FakeEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, _stop=False, **kw)

    monkeypatch.setattr(models, "DalleEngine", Eng)
    _FakeEngine.calls.clear()
    models.DALLE(256, n_layers=3, params={"attention_types": [[["axial_row", "axial_col", "global"], 1]]})
    (_, kw), = _FakeEngine.calls
    assert kw["attention_types"] == ["axial_row", "axial_col", "global"]
    with pytest.raises(ValueError, match="attention_types"):
        models.DALLE(256, n_layers=2, params={"attention_types": [[["axial_row", "axial_diag"], 1]]})


def test_generate_dalle_builds_the_engine_with_the_trained_axial_types(tmp_path, monkeypatch):
    import generate_dalle as G
    from dalle_mtf_b200 import model_fns
    from dalle_mtf_b200.utils import save_checkpoint
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, "n_embd": 256, "n_layers": 3, "n_heads": 2,
             "attention_types": [[["axial_row", "axial_col", "global"], 1]]}
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
    assert args[:3] == (256, 3, 2) and args[6] == 16
    assert kw["attention_types"] == ["axial_row", "axial_col", "global"]
