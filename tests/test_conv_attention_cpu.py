"""CPU tests of convolutional attention layers: parsing of the "conv" attention type and of conv_attention_kernel, the
reference mask against a brute-force definition and against DALLE-pytorch's unfold construction, the pair count the
attention profiler uses, the kernels' tile walks, the absence of attention dropout in conv layers, and the plumbing of
the layer types and the kernel size from models.DALLE and generate_dalle.py into DalleEngine."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import axial_oracle as OA
import conv_oracle as OC
from dalle_mtf_b200 import dalle_engine, lib, ops
from dalle_mtf_b200.dalle_engine import layer_axial, layer_conv, layer_radii
from dalle_mtf_b200.model_fns import attention_layers, conv_kernel
from oracle import dalle as O
from oracle import dalle_dropout as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------- config
def test_conv_type_parses_and_mixes_with_every_other_type():
    p = {"n_layers": 6, "attention_types": [[["axial_row", "axial_col"], 2], [["axial_row", "conv"], 1]]}
    assert attention_layers(p) == (["axial_row", "axial_col"] * 2 + ["axial_row", "conv"], 256)
    types = ["global", "local", "axial_row", "axial_col", "conv"]
    p = {"n_layers": 5, "attention_types": [[types, 1]], "local_attention_radius": 64, "conv_attention_kernel": 3}
    assert attention_layers(p) == (types, 64) and conv_kernel(p) == 3
    assert layer_radii(types, 64, 5) == [None, 64, None, None, None]
    assert layer_axial(types, 256, 1024, 5) == [None, None, (256, 32, 0), (256, 32, 1), None]
    assert layer_conv(types, 256, 1024, 3, 5) == [None, None, None, None, (256, 32, 3)]
    assert layer_conv(["global", "axial_row"], 256, 1024, 5, 2) == [None, None]
    assert layer_conv(["global", "local"], 256, 1000, 5, 2) == [None, None]   # no conv layer: any image length
    assert layer_conv(None, 256, 1000, 5, 3) == [None] * 3


def test_conv_attention_kernel_defaults_to_five():
    assert conv_kernel({}) == 5 and conv_kernel({"conv_attention_kernel": None}) == 5
    assert conv_kernel({"conv_attention_kernel": 1}) == 1 and conv_kernel({"conv_attention_kernel": 40}) == 40
    assert conv_kernel({"conv_attention_kernel": np.int64(7)}) == 7


@pytest.mark.parametrize("value", [0, -1, 2.0, 2.5, True, False, "5", [5]])
def test_malformed_conv_attention_kernel_is_rejected(value, monkeypatch):
    with pytest.raises(ValueError, match="conv_attention_kernel"):
        conv_kernel({"conv_attention_kernel": value})
    with pytest.raises(ValueError, match="conv_attention_kernel"):
        layer_conv(["conv"], 8, 16, value, 1)
    monkeypatch.setattr(lib, "require_device", lambda: None)
    with pytest.raises(ValueError, match="conv_attention_kernel"):
        dalle_engine.DalleEngine(256, 1, 2, 300, 64, 8, 16, attention_types=["conv"], conv_attention_kernel=value)


@pytest.mark.parametrize("name", ["conv_like", "Conv", "convolution", "conv2d"])
def test_other_conv_names_stay_unknown(name):
    with pytest.raises(ValueError, match="attention_types"):
        attention_layers({"n_layers": 2, "attention_types": [[["conv", name], 1]]})
    with pytest.raises(ValueError, match="attention_types"):
        layer_radii(["conv", name], 256, 2)


@pytest.mark.parametrize("image_seq_len", [1000, 2, 15, 1023])
def test_conv_layers_reject_a_non_square_image_grid(image_seq_len, monkeypatch):
    with pytest.raises(ValueError, match="square"):
        layer_conv(["global", "conv"], 256, image_seq_len, 5, 2)
    monkeypatch.setattr(lib, "require_device", lambda: None)
    with pytest.raises(ValueError, match="square"):
        dalle_engine.DalleEngine(256, 2, 2, 300, 64, 8, image_seq_len, attention_types=["conv", "global"])


def test_the_conv_example_config_is_dalle_example_with_a_conv_last_layer():
    with open(os.path.join(ROOT, "configs", "dalle_example_conv_b200.json")) as f:
        conv = json.load(f)
    with open(os.path.join(ROOT, "configs", "dalle_example_b200.json")) as f:
        base = json.load(f)
    types, _ = attention_layers(conv)
    assert types == ["axial_row", "axial_col", "axial_row", "axial_col", "axial_row", "conv"]
    assert conv_kernel(conv) == 5
    assert {k for k in set(conv) | set(base) if conv.get(k) != base.get(k)} == {"attention_types", "model_path"}


# ------------------------------------------------------------------------------------------------------- masks
def _brute_force_visible(S, TL, W, k):
    vis = torch.zeros(S, S, dtype=torch.bool)
    for i in range(S):
        for j in range(i + 1):
            if j < TL:
                vis[i, j] = True
                continue
            (ri, ci), (rj, cj) = divmod(i - TL, W), divmod(j - TL, W)
            vis[i, j] = ri - k < rj <= ri and ci - k < cj <= ci
    return vis


def _unfold_visible(S, TL, W, k):
    """DALLE-pytorch's construction: pad the grid of image positions top and left by k - 1 and unfold k x k windows;
    each window lists the image keys its bottom-right query sees (padding: none)."""
    grid = torch.arange(W * W, dtype=torch.float64).view(1, 1, W, W)
    padded = F.pad(grid + 1, (k - 1, 0, k - 1, 0))                       # 0 marks padding
    win = F.unfold(padded, k).squeeze(0).T.long() - 1                     # [W*W query][k*k key] image index or -1
    vis = torch.zeros(S, S, dtype=torch.bool)
    for i in range(S):
        vis[i, :min(i + 1, TL)] = True
        if i >= TL:
            keys = win[i - TL]
            keys = keys[keys >= 0] + TL
            vis[i, keys[keys < S]] = True
    return vis


# (TL, W, S, k): full and ragged lengths, k = 1, k = W, k > W, TL = 0, W = 1
GEOMETRIES = [(12, 4, 28, 2), (0, 3, 9, 2), (5, 1, 6, 1), (5, 1, 6, 3), (7, 5, 32, 3), (7, 5, 19, 5), (3, 6, 20, 9),
              (16, 4, 25, 1), (4, 7, 53, 4)]


@pytest.mark.parametrize("TL,W,S,k", GEOMETRIES)
def test_oracle_mask_matches_the_grid_definition_and_the_unfold_construction(TL, W, S, k):
    cfg = OC.ConvConfig(64, 1, 2, 100, 30, TL, W * W, attention_types=("conv",), conv_attention_kernel=k)
    mask = OC.attention_mask(cfg, 0, S, O.Quirks())
    want = _brute_force_visible(S, TL, W, k)
    assert torch.equal(mask == 0, want)
    assert torch.equal(mask[~want], torch.full((int((~want).sum()),), O.Quirks().mask_value))
    assert torch.equal(_unfold_visible(S, TL, W, k), want)
    assert torch.equal(~OC.conv_hidden(S, TL, W, k), want)


def test_the_window_is_not_a_band():
    """(r - 1, c + 1) precedes (r, c) in raster order but is outside its window; k >= W sees the whole quadrant."""
    TL, W, k = 4, 6, 3
    vis = ~OC.conv_hidden(TL + W * W, TL, W, k)
    pos = lambda r, c: TL + r * W + c
    assert not vis[pos(3, 2), pos(2, 3)] and vis[pos(3, 2), pos(2, 2)] and vis[pos(3, 2), pos(1, 0)]
    assert not vis[pos(3, 2), pos(0, 2)] and not vis[pos(3, 3), pos(3, 0)] and vis[pos(3, 3), pos(3, 1)]
    full = ~OC.conv_hidden(TL + W * W, TL, W, W)
    assert torch.equal(full, ~OC.conv_hidden(TL + W * W, TL, W, W + 5))
    assert full[pos(5, 5), pos(0, 0)] and not full[pos(4, 2), pos(0, 3)]


@pytest.mark.parametrize("TL,W,S,k", GEOMETRIES)
def test_pair_count_matches_the_counted_mask(TL, W, S, k):
    assert ops.attn_pairs_conv(S, TL, W, k) == float(_brute_force_visible(S, TL, W, k).sum())


def test_pair_count_at_dalle_example():
    S = 1280
    for k, want in ((5, 317540), (11, 383249)):
        assert ops.attn_pairs_conv(S, 256, 32, k) == want == float((~OC.conv_hidden(S, 256, 32, k)).sum())
    assert abs(317540 / (S * (S + 1) / 2) - 0.387) < 1e-3 and abs(383249 / (S * (S + 1) / 2) - 0.467) < 1e-3


# ------------------------------------------------------------------------------------------------------- tile walks
WALKS = [(256, 32, 1280, 5), (256, 32, 1280, 11), (100, 24, 676, 3), (64, 80, 6464, 7), (7, 1, 8, 1), (16, 8, 80, 9),
         (256, 32, 300, 5), (256, 32, 777, 5), (0, 16, 256, 4), (100, 24, 150, 24)]


def _tile_any(vis, S):
    n = -(-S // 64)
    pad = torch.zeros(n * 64, n * 64, dtype=torch.bool)
    pad[:S, :S] = vis
    return pad.view(n, 64, n, 64).any(3).any(1)


@pytest.mark.parametrize("TL,W,S,k", WALKS)
def test_tile_walks_cover_every_visible_pair(TL, W, S, k):
    vis = ~OC.conv_hidden(S, TL, W, k)
    need = _tile_any(vis, S)                            # [query block][key block]
    n = need.shape[0]
    fwd = torch.zeros(n, n, dtype=torch.bool)
    for qb in range(n):
        blocks = OC.key_blocks(S, TL, W, k, qb)
        assert len(set(blocks)) == len(blocks) and all(0 <= j <= qb for j in blocks)
        fwd[qb, blocks] = True
    dkv = torch.zeros(n, n, dtype=torch.bool)
    for kb in range(n):
        dkv[OC.query_blocks(S, TL, W, k, kb), kb] = True
    assert not (need & ~fwd).any() and not (need & ~dkv).any()


@pytest.mark.parametrize("k,tiles", [(5, 119), (11, 155)])
def test_forward_walk_at_dalle_example_visits_only_tiles_with_pairs(k, tiles):
    TL, W, S = 256, 32, 1280
    need = _tile_any(~OC.conv_hidden(S, TL, W, k), S)
    visited = [(qb, j) for qb in range(S // 64) for j in OC.key_blocks(S, TL, W, k, qb)]
    assert len(visited) == tiles and all(need[qb, j] for qb, j in visited)
    assert (S // 64) * (S // 64 + 1) // 2 == 210


# ------------------------------------------------------------------------------------------------------- oracle
def _case(types, seed=0, B=2, ts=5, isl=16, L=3, k=2, dtype=torch.float32):
    cfg = OC.ConvConfig(64, L, 2, 100, 30, ts, isl, attention_types=types, local_attention_radius=3,
                        conv_attention_kernel=k)
    params = {n: v.to(dtype) for n, v in O.init_params(cfg, seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True])
def test_models_without_conv_layers_are_the_axial_oracle_bit_for_bit(bf16):
    for types in (None, ("global", "global", "global"), ("local", "global", "local"),
                  ("axial_row", "global", "axial_col")):
        cfg, params, tokens = _case(types)
        acfg = OA.AxialConfig(*[getattr(cfg, f) for f in ("n_embd", "n_layers", "n_heads", "text_vocab_size",
                                                          "image_vocab_size", "text_seq_len", "image_seq_len")],
                              attention_types=types, local_attention_radius=3)
        for dropout in (None, ((0.1, 0.3, 0.2), 7, 3, 1)):
            want = OA.forward(params, tokens, acfg, dropout, bf16=bf16)
            got = OC.forward(params, tokens, cfg, dropout, bf16=bf16)
            assert all(torch.equal(a, b) for a, b in zip(want, got))
    cfg, params, tokens = _case(("global", "conv", "axial_row"))
    assert not torch.equal(OC.forward(params, tokens, cfg)[2], OC.forward(params, tokens, _case(None)[0])[2])
    # the kernel size matters
    assert not torch.equal(OC.forward(params, tokens, cfg)[2], OC.forward(params, tokens, _case(cfg.attention_types,
                                                                                                 k=3)[0])[2])


def test_conv_layers_have_no_attention_dropout_and_keep_residual_dropout():
    types = ("global", "conv", "axial_col")
    cfg, params, tokens = _case(types)
    B = tokens.shape[0]
    spec = lambda rates: (rates, 7, 3, 1)
    dm = OC.dropout_masks(spec((0.1, 0.3, 0.2)), B, cfg)
    assert dm["attn"][0] is not None and dm["attn"][1] is None and dm["attn"][2] is None
    assert all(m is not None for m in dm["attn_out"] + dm["mlp_out"])
    gm = D.dropout_masks(spec((0.1, 0.3, 0.2)), B, _case(None)[0])         # site numbers do not move
    assert torch.equal(dm["attn"][0], gm["attn"][0])
    assert all(torch.equal(a, b) for a, b in zip(dm["attn_out"] + dm["mlp_out"], gm["attn_out"] + gm["mlp_out"]))
    ccfg = _case(("conv", "conv", "conv"))[0]
    plain = OC.forward(params, tokens, ccfg, spec((0.0, 0.0, 0.0)))[2]
    assert torch.equal(OC.forward(params, tokens, ccfg, spec((0.0, 0.5, 0.0)))[2], plain)
    assert not torch.equal(OC.forward(params, tokens, ccfg, spec((0.0, 0.0, 0.3)))[2], plain)
    assert torch.equal(plain, OC.forward(params, tokens, ccfg)[2])


def test_engine_drops_attention_weights_only_in_global_layers():
    eng = dalle_engine.DalleEngine.__new__(dalle_engine.DalleEngine)
    eng.dropout, eng.dropout_seed, eng.S, eng.L = (0.1, 0.2, 0.3), 5, 21, 5
    eng.radii = [None, 3, None, None, None]
    eng.axial = [None, None, (5, 4, 0), (5, 4, 1), None]
    eng.conv = [None, None, None, None, (5, 4, 3)]
    dd = eng._dropout_descs(step=2, row0=0)
    assert dd["attn"][0] is not None and dd["attn"][1:] == [None] * 4
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


def test_dalle_class_passes_the_conv_types_and_kernel_to_the_engine(monkeypatch):
    from dalle_mtf_b200 import models

    class Eng(_FakeEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, _stop=False, **kw)

    monkeypatch.setattr(models, "DalleEngine", Eng)
    _FakeEngine.calls.clear()
    models.DALLE(256, n_layers=3, params={"attention_types": [[["axial_row", "conv", "global"], 1]],
                                          "conv_attention_kernel": 7})
    models.DALLE(256, n_layers=2, params={"attention_types": [[["conv"], 2]]})
    (_, kw), (_, kw2) = _FakeEngine.calls
    assert kw["attention_types"] == ["axial_row", "conv", "global"] and kw["conv_attention_kernel"] == 7
    assert kw2["attention_types"] == ["conv", "conv"] and kw2["conv_attention_kernel"] == 5
    with pytest.raises(ValueError, match="conv_attention_kernel"):
        models.DALLE(256, n_layers=1, params={"attention_types": [[["conv"], 1]], "conv_attention_kernel": 0})


def test_generate_dalle_builds_the_engine_with_the_trained_conv_layers(tmp_path, monkeypatch):
    import generate_dalle as G
    from dalle_mtf_b200 import model_fns
    from dalle_mtf_b200.utils import save_checkpoint
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, "n_embd": 256, "n_layers": 3, "n_heads": 2,
             "attention_types": [[["axial_row", "axial_col", "conv"], 1]], "conv_attention_kernel": 3}
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
    assert kw["attention_types"] == ["axial_row", "axial_col", "conv"] and kw["conv_attention_kernel"] == 3
