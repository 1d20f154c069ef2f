"""CPU tests of block-sparse attention layers: parsing of the "block_sparse" attention type and of its four keys, the
layout against a brute-force restatement of its three rules, its determinism and its sharing between layers that
share attention, the tables the kernels read, the pair count the attention profiler uses, the oracle, and the plumbing
of the keys from models.DALLE and generate_dalle.py into DalleEngine."""
import json

import numpy as np
import pytest
import torch

import block_sparse_oracle as OB
import conv_oracle as OC
from dalle_mtf_b200 import dalle_engine, lib, ops
from dalle_mtf_b200.dalle_engine import block_sparse_layout, layer_block_sparse, validate_block_sparse
from dalle_mtf_b200.model_fns import attention_layers, block_sparse_options
from oracle import dalle as O
from test_conv_attention_cpu import _FakeEngine, _Stop

KEYS = ("sparse_block_size", "sparse_local_window_blocks", "sparse_random_blocks", "sparse_layout_seed")


# ------------------------------------------------------------------------------------------------------- config
def test_block_sparse_type_parses_and_mixes_with_every_other_type():
    types = ["global", "local", "axial_row", "axial_col", "conv", "mlp", "block_sparse"]
    assert attention_layers({"n_layers": 7, "attention_types": [[types, 1]]}) == (types, 256)
    p = {"n_layers": 6, "attention_types": [[["block_sparse", "global"], 3]]}
    assert attention_layers(p)[0] == ["block_sparse", "global"] * 3


@pytest.mark.parametrize("name", ["sparse", "Block_sparse", "blocksparse", "block-sparse"])
def test_other_sparse_names_stay_unknown(name):
    with pytest.raises(ValueError, match="attention_types"):
        attention_layers({"n_layers": 1, "attention_types": [[[name], 1]]})
    with pytest.raises(ValueError, match="attention_types"):
        dalle_engine.layer_radii([name], 256, 1)


def test_defaults_are_dalle_pytorchs():
    assert validate_block_sparse(None, None, None, None, 1280) == (16, 4, 20, 0)
    assert validate_block_sparse(32, None, None, None, 1280) == (32, 4, 10, 0)
    assert validate_block_sparse(64, 2, 0, 7, 1280) == (64, 2, 0, 7)
    assert block_sparse_options({}) == dict.fromkeys(KEYS)
    opts = {"sparse_block_size": 32, "sparse_local_window_blocks": 1, "sparse_random_blocks": 0,
            "sparse_layout_seed": 3}
    assert block_sparse_options(opts) == opts


@pytest.mark.parametrize("key,value", [("sparse_block_size", v) for v in (8, 48, 128, 0, True, 16.0, "16")] +
                         [("sparse_local_window_blocks", v) for v in (0, -1, True, 2.0, "4", [4])] +
                         [("sparse_random_blocks", v) for v in (-1, False, 1.5, "20")] +
                         [("sparse_layout_seed", v) for v in (-1, True, 0.0, "0")])
def test_malformed_keys_are_refused_with_the_key_named(key, value):
    with pytest.raises(ValueError, match=key):
        block_sparse_options({key: value})
    with pytest.raises(ValueError, match=key):
        layer_block_sparse(["block_sparse"], 256, 1024, 1, **_engine_kw(key, value))


def _engine_kw(key, value):
    names = {"sparse_block_size": "block_size", "sparse_local_window_blocks": "local_window_blocks",
             "sparse_random_blocks": "random_blocks", "sparse_layout_seed": "layout_seed"}
    return {names[key]: value}


# ------------------------------------------------------------------------------------------------------- layout
def _brute_force(S, TL, b, w, R, seed, owner):
    nb = -(-S // b)
    rng = np.random.Generator(np.random.PCG64(np.random.SeedSequence([seed, owner])))
    rand = [set(rng.choice(r + 1, min(R, r + 1), replace=False).tolist()) for r in range(nb)]
    g = -(-TL // b)
    return np.array([[c <= r and (c < g or c // w == r // w or c in rand[r]) for c in range(nb)] for r in range(nb)])


GEOMETRIES = [(1280, 256, 16, 4, 20), (1280, 256, 16, 4, 0), (1280, 256, 16, 4, 80), (1279, 256, 32, 4, 10),
              (1030, 250, 16, 3, 5), (1280, 256, 64, 1, 2), (300, 7, 16, 2, 1)]


@pytest.mark.parametrize("S,TL,b,w,R", GEOMETRIES)
@pytest.mark.parametrize("seed,owner", [(0, 0), (5, 2)])
def test_layout_is_the_three_rules(S, TL, b, w, R, seed, owner):
    lay = block_sparse_layout(S, TL, b, w, R, seed, owner)
    assert np.array_equal(lay, _brute_force(S, TL, b, w, R, seed, owner))
    assert lay.diagonal().all() and not np.triu(lay, 1).any()
    rand = lay.sum(1)
    assert (rand >= np.minimum(R, np.arange(lay.shape[0]) + 1)).all()   # every row gets its R blocks where it can


def test_full_random_rows_give_the_causal_triangle():
    nb = 1280 // 16
    assert np.array_equal(block_sparse_layout(1280, 256, 16, 4, nb, 0, 0), np.tril(np.ones((nb, nb), bool)))


def test_layout_is_deterministic_per_seed_and_owner_and_shared_by_sharing_layers():
    a = block_sparse_layout(1280, 256, 16, 4, 20, 0, 0)
    assert np.array_equal(a, block_sparse_layout(1280, 256, 16, 4, 20, 0, 0))
    assert not np.array_equal(a, block_sparse_layout(1280, 256, 16, 4, 20, 1, 0))
    assert not np.array_equal(a, block_sparse_layout(1280, 256, 16, 4, 20, 0, 1))
    types = ["block_sparse", "global", "block_sparse", "block_sparse"]
    own = layer_block_sparse(types, 256, 1024, 4)
    assert own[1] is None and not np.array_equal(own[0], own[2]) and not np.array_equal(own[2], own[3])
    shared = layer_block_sparse(types, 256, 1024, 4, attn_owner=[0, 1, 0, 3])
    assert shared[0] is shared[2] and np.array_equal(shared[0], own[0]) and np.array_equal(shared[3], own[3])
    assert layer_block_sparse(None, 256, 1024, 3) == [None] * 3


def test_layout_does_not_depend_on_the_training_seed():
    """The engine's layout is a function of the four keys and the owner only (dropout_seed is not among them)."""
    a = layer_block_sparse(["block_sparse"], 256, 1024, 1, layout_seed=4)
    assert np.array_equal(a[0], block_sparse_layout(1280, 256, 16, 4, 20, 4, 0))


# ------------------------------------------------------------------------------------------------------- tables
def _decode_tables(bs):
    tiles = bs.tiles.cpu().numpy().view(np.uint16).astype(np.int64)
    return tiles, bs.blocks.cpu().numpy()


@pytest.mark.parametrize("S,TL,b,w,R", GEOMETRIES)
def test_tables_restate_the_layout_at_16_token_granularity(S, TL, b, w, R):
    lay = block_sparse_layout(S, TL, b, w, R, 0, 0)
    bs = ops.BlockSparse(lay, b, S, device="cpu")
    tiles, blocks = _decode_tables(bs)
    vis = ~OB.block_sparse_hidden(S, lay, b).numpy()
    nt, ng = -(-S // 64), -(-S // 16)
    assert tiles.shape == (nt, nt) and blocks.shape == (ng, ng + 1)
    for qt in range(nt):
        for kt in range(nt):
            for a in range(4):
                for c in range(4):
                    bit = (tiles[qt, kt] >> (4 * a + c)) & 1
                    i0, j0 = 64 * qt + 16 * a, 64 * kt + 16 * c
                    want = i0 < S and j0 <= i0 and lay[i0 // b, j0 // b]
                    assert bit == want, (qt, kt, a, c)
    for g in range(ng):
        n = blocks[g, 0]
        listed = blocks[g, 1:1 + n]
        assert (np.diff(listed) > 0).all() and (listed <= g).all()
        keys = np.concatenate([np.arange(16 * c, min(16 * c + 16, 16 * g + 1)) for c in listed])
        assert np.array_equal(np.flatnonzero(vis[16 * g]), keys)


def test_tables_refuse_a_layout_of_the_wrong_shape():
    with pytest.raises(lib.DB200Error):
        ops.BlockSparse(np.ones((10, 10), bool), 16, 1280, device="cpu")
    with pytest.raises(lib.DB200Error):
        ops.BlockSparse(np.ones((80, 80), bool), 16, 1280, device="cpu")   # not lower triangular


def test_tile_counts_at_dalle_example():
    """The shares of causal pairs and 64 x 64 tiles visited at S 1280, TL 256, b 16 (DESIGN.md's table)."""
    S, TL = 1280, 256
    for R, share, tiles in ((0, 0.40, 90), (5, 0.46, 177), (20, 0.61, 210)):
        lay = block_sparse_layout(S, TL, 16, 4, R, 0, 0)
        t, _ = _decode_tables(ops.BlockSparse(lay, 16, S, device="cpu"))
        assert np.count_nonzero(np.tril(t)) == tiles
        assert abs(ops.attn_pairs_block_sparse(S, lay, 16) / (S * (S + 1) / 2) - share) < 0.005


@pytest.mark.parametrize("S,TL,b,w,R", GEOMETRIES)
def test_pair_count_matches_the_counted_mask(S, TL, b, w, R):
    lay = block_sparse_layout(S, TL, b, w, R, 0, 0)
    for P in (S, S - 1, S // 2 + 3):
        assert ops.attn_pairs_block_sparse(P, lay, b) == (~OB.block_sparse_hidden(P, lay, b)).sum().item()


# ------------------------------------------------------------------------------------------------------- oracle
def _case(types, seed=0, B=2, ts=5, isl=59, Ly=3):
    layouts = tuple(block_sparse_layout(ts + isl, ts, 16, 1, 0, 0, l) if t == "block_sparse" else None
                    for l, t in enumerate(types))
    cfg = OB.BlockSparseConfig(256, Ly, 2, 100, 50, ts, isl, attention_types=types, local_attention_radius=8,
                               conv_attention_kernel=2, block_sparse_layouts=layouts)
    params = O.init_params(cfg, seed)
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=torch.Generator().manual_seed(seed))
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True])
def test_models_without_block_sparse_layers_are_the_conv_oracle_bit_for_bit(bf16):
    cfg, params, tokens = _case(("global", "local", "global"))
    ccfg = OC.ConvConfig(256, 3, 2, 100, 50, 5, 59, attention_types=("global", "local", "global"),
                         local_attention_radius=8, conv_attention_kernel=2)
    a = OB.forward(params, tokens, cfg, bf16=bf16)[2]
    b = OC.forward(params, tokens, ccfg, bf16=bf16)[2]
    assert torch.equal(a, b)


def test_block_sparse_layers_change_the_output_and_have_no_attention_dropout():
    cfg, params, tokens = _case(("block_sparse", "global", "global"))
    gcfg, _, _ = _case(("global", "global", "global"))
    assert not torch.equal(OB.forward(params, tokens, cfg)[2], OB.forward(params, tokens, gcfg)[2])
    dm = OB.dropout_masks(((0.1, 0.2, 0.15), 3, 1, 0), 2, cfg)
    assert dm["attn"][0] is None and dm["attn"][1] is not None and dm["attn_out"][0] is not None
    # with the full causal layout the block-sparse layer is a global layer without dropout
    nb = 4
    full = OB.BlockSparseConfig(256, 3, 2, 100, 50, 5, 59, attention_types=("block_sparse", "global", "global"),
                                block_sparse_layouts=(np.tril(np.ones((nb, nb), bool)), None, None))
    assert torch.equal(OB.forward(params, tokens, full)[2], OB.forward(params, tokens, gcfg)[2])


# ------------------------------------------------------------------------------------------------------- plumbing
def test_dalle_class_passes_the_block_sparse_keys_to_the_engine(monkeypatch):
    from dalle_mtf_b200 import models

    class Eng(_FakeEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, _stop=False, **kw)

    monkeypatch.setattr(models, "DalleEngine", Eng)
    _FakeEngine.calls.clear()
    opts = {"sparse_block_size": 32, "sparse_local_window_blocks": 2, "sparse_random_blocks": 3,
            "sparse_layout_seed": 9}
    models.DALLE(256, n_layers=2, params={"attention_types": [[["block_sparse", "global"], 1]], **opts})
    models.DALLE(256, n_layers=1, params={"attention_types": [[["block_sparse"], 1]]})
    (_, kw), (_, kw2) = _FakeEngine.calls
    assert kw["attention_types"] == ["block_sparse", "global"] and all(kw[k] == v for k, v in opts.items())
    assert all(kw2[k] is None for k in KEYS)
    with pytest.raises(ValueError, match="sparse_block_size"):
        models.DALLE(256, n_layers=1, params={"attention_types": [[["block_sparse"], 1]], "sparse_block_size": 24})


def test_model_fn_refuses_malformed_keys_before_touching_the_device(monkeypatch):
    from dalle_mtf_b200 import model_fns
    monkeypatch.setattr(lib, "require_device", lambda: (_ for _ in ()).throw(AssertionError("device touched")))
    with pytest.raises(ValueError, match="sparse_random_blocks"):
        model_fns.dalle_model_fn(None, None, "train", {"n_layers": 1, "sparse_random_blocks": -2})


def test_generate_dalle_builds_the_engine_with_the_trained_layout_keys(tmp_path, monkeypatch):
    import generate_dalle as G
    from dalle_mtf_b200 import model_fns
    from dalle_mtf_b200.utils import save_checkpoint
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, "n_embd": 256, "n_layers": 2, "n_heads": 2,
             "attention_types": [[["block_sparse", "global"], 1]], "sparse_block_size": 16,
             "sparse_local_window_blocks": 2, "sparse_random_blocks": 1, "sparse_layout_seed": 11}
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
    assert kw["attention_types"] == ["block_sparse", "global"]
    assert [kw[k] for k in KEYS] == [16, 2, 1, 11]
