"""CPU tests of the DALL-E paper's input embedding (row / column image positions, per-position padding): the oracle
(oracle/dalle_input.py) against brute-force per-position definitions and against the forwards it wraps, its autograd
gradients against the fold definition, the pad mapping with and without caption dropout, the validation of both
config keys (model_fn, models.DALLE, generate_dalle.py), and the engine's parameter layout, vocabulary and names."""
import json
import math

import numpy as np
import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import DalleEngine, image_grid_side, param_layout, validate_per_position_padding, \
    validate_position_embedding
from dalle_mtf_b200.model_fns import dalle_model_fn, input_embedding
from dalle_mtf_b200.models import DALLE
from dalle_mtf_b200.utils import save_checkpoint
from oracle import dalle as O
from oracle import dalle_dropout as OD
from oracle import dalle_input as I
from oracle import dalle_local as OL
from oracle.guidance import caption_dropped

ROW_COL = I.InputConfig("row_col", False, None)
BOTH = I.InputConfig("row_col", True, 7)
OFF = I.InputConfig()


def _cfg(TL=6, W=3, d=32, L=2, tv=50, iv=16, types=None):
    return OL.LocalConfig(d, L, 2, tv, iv, TL, W * W, attention_types=types)


def _tokens(cfg, inp, B=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, cfg.text_vocab_size, (B, cfg.text_seq_len), generator=g)
    if inp.padding_id is not None:
        text[:, cfg.text_seq_len // 2:] = inp.padding_id
    img = torch.randint(0, cfg.image_vocab_size, (B, cfg.image_seq_len), generator=g)
    return I.assemble(text, img, cfg, inp)


# ------------------------------------------------------------------------------------------------ oracle definitions
@pytest.mark.parametrize("bf16", [False, True])
def test_composed_table_is_the_per_position_definition(bf16):
    cfg = _cfg(TL=5, W=4, d=16)
    p = I.init_params(cfg, ROW_COL, seed=1)
    table = I.compose_positions(p, cfg, bf16=bf16)
    r16 = (lambda x: x.to(torch.bfloat16).float()) if bf16 else (lambda x: x)
    wpe, row, col = (r16(p["positional_embedding/" + n]) for n in ("wpe", "image_row", "image_col"))
    assert table.shape == (cfg.seq_len, cfg.n_embd)
    for pos in range(cfg.seq_len):
        if pos < cfg.text_seq_len:
            want = wpe[pos]
        else:
            r, c = divmod(pos - cfg.text_seq_len, 4)
            want = r16(row[r] + col[c])
        assert torch.equal(table[pos], want), pos
    if bf16:   # each image row is one bf16 rounding of the fp32 sum of two bf16 values
        assert torch.equal(table, table.to(torch.bfloat16).float())


def test_mutated_tables_differ_from_the_definition():
    cfg = _cfg(TL=5, W=4, d=16)
    p = I.init_params(cfg, ROW_COL, seed=2)
    base = I.compose_positions(p, cfg)
    for m in ("transpose", "shift_origin"):
        got = I.compose_positions(p, cfg, mutate=m)
        assert torch.equal(got[:cfg.text_seq_len], base[:cfg.text_seq_len])
        assert not torch.equal(got, base), m
    # transposed: token (r, c) carries row[c] + col[r]
    t = I.compose_positions(p, cfg, mutate="transpose")
    assert torch.equal(t[5 + 1 * 4 + 2], p["positional_embedding/image_row"][2] + p["positional_embedding/image_col"][1])


def test_row_and_column_gradients_are_the_fold_of_the_table_gradient():
    cfg = _cfg(TL=6, W=3, d=32, L=1)
    p = I.init_params(cfg, ROW_COL, seed=3)
    tokens = _tokens(cfg, ROW_COL)
    p64 = {k: v.double() for k, v in p.items()}
    _, _, _, g = I.loss_and_grads(p64, tokens, cfg, ROW_COL)
    # the gradient of the composed table, from the absolute-position model run on that table
    pa = dict(p64)
    pa["positional_embedding/wpe"] = I.compose_positions(p64, cfg).detach()
    _, _, _, ga = OL.loss_and_grads(pa, tokens, I._model_cfg(cfg, ROW_COL))
    dpos = ga["positional_embedding/wpe"]
    TL, W = 6, 3
    img = dpos[TL:].view(W, W, -1)
    assert torch.allclose(g["positional_embedding/wpe"], dpos[:TL], rtol=0, atol=1e-15)
    assert torch.allclose(g["positional_embedding/image_row"], img.sum(1), rtol=1e-12, atol=1e-15)
    assert torch.allclose(g["positional_embedding/image_col"], img.sum(0), rtol=1e-12, atol=1e-15)
    for k in g:
        if not k.startswith("positional_embedding/"):
            assert torch.allclose(g[k], ga[k], rtol=1e-12, atol=1e-15), k


def test_with_both_keys_off_the_oracle_is_the_forward_it_wraps():
    cfg = _cfg(TL=6, W=3, d=32)
    p = O.init_params(cfg, seed=4)
    assert I.init_params(cfg, OFF, seed=4).keys() == p.keys()
    assert all(torch.equal(I.init_params(cfg, OFF, seed=4)[k], p[k]) for k in p)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, cfg.text_vocab_size, (2, 6), generator=g)
    img = torch.randint(0, cfg.image_vocab_size, (2, 9), generator=g)
    tokens = I.assemble(text, img, cfg, OFF)
    assert torch.equal(tokens, O.assemble_tokens(text, img, cfg.text_vocab_size))
    for bf16 in (False, True):
        got = I.forward(p, tokens, cfg, OFF, bf16=bf16)
        for want in (O.forward(p, tokens, cfg, bf16=bf16), OL.forward(p, tokens, cfg, bf16=bf16)):
            assert all(torch.equal(a, b) for a, b in zip(got, want))
        drop = ((0.1, 0.1, 0.1), 5, 3, 0)
        got = I.forward(p, tokens, cfg, OFF, dropout=drop, bf16=bf16)
        want = OD.forward(p, tokens, cfg, drop, bf16=bf16)
        assert all(torch.equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------------ pad mapping
def test_pad_mapping_per_position():
    cfg = _cfg(TL=6, tv=50)
    text = torch.tensor([[1, 2, 7, 7, 7, 7], [7, 3, 7, 4, 7, 7], [5, 6, 8, 9, 10, 11]])
    got = I.map_pads(text, cfg, BOTH)
    want = text.clone()
    for b in range(3):
        for t in range(6):
            if text[b, t] == 7:
                want[b, t] = 50 + t
    assert torch.equal(got, want)
    assert torch.equal(I.map_pads(text, cfg, BOTH, mutate="pad_plus_one"), torch.where(text == 7, want + 1, want))
    off, V = I.vocab(cfg, BOTH)
    assert (off, V) == (50 + 6, 50 + 6 + 16 + 1)
    img = torch.arange(9).view(1, 9).repeat(3, 1)
    assert torch.equal(I.assemble(text, img, cfg, BOTH)[:, 6:], img + off)


def test_pad_mapping_with_caption_dropout():
    cfg = _cfg(TL=6, tv=50)
    B = 64
    g = torch.Generator().manual_seed(5)
    text = torch.randint(0, 50, (B, 6), generator=g)
    img = torch.zeros(B, 9, dtype=torch.long)
    rate, seed, step, row0 = 0.3, 11, 4, 8
    dropped = torch.from_numpy(caption_dropped(rate, seed, step, B, row0))
    assert 0 < int(dropped.sum()) < B
    got = I.assemble(text, img, cfg, BOTH, caption_drop=(rate, seed, step, row0))
    pads = 50 + torch.arange(6)
    for b in range(B):
        if dropped[b]:
            assert torch.equal(got[b, :6], pads)          # a dropped caption is the TL per-position pads
        else:
            assert torch.equal(got[b, :6], torch.where(text[b] == 7, pads, text[b]))
    # without per-position padding a dropped caption is padding_id everywhere
    single = I.InputConfig("absolute", False, 7)
    got = I.assemble(text, img, cfg, single, caption_drop=(rate, seed, step, row0))
    assert torch.equal(got[:, :6], torch.where(dropped[:, None], torch.full_like(text, 7), text))


# ------------------------------------------------------------------------------------------------ key validation
def test_key_validation():
    assert validate_position_embedding(None) == "absolute"
    assert validate_position_embedding("absolute") == "absolute"
    assert validate_position_embedding("row_col") == "row_col"
    for bad in ("rowcol", "ROW_COL", "", 1, True, ["row_col"], "axial"):
        with pytest.raises(ValueError, match="image_position_embedding"):
            validate_position_embedding(bad)
    assert validate_per_position_padding(None) is False
    assert validate_per_position_padding(False) is False and validate_per_position_padding(True) is True
    for bad in (0, 1, "true", 1.0, []):
        with pytest.raises(ValueError, match="per_position_padding"):
            validate_per_position_padding(bad)
    assert image_grid_side(1024) == 32 and image_grid_side(256) == 16
    for bad in (1000, 1023, 2):
        with pytest.raises(ValueError, match="square image-token grid"):
            image_grid_side(bad)


def test_config_helper():
    assert input_embedding({}) == ("absolute", False, None)
    assert input_embedding({"image_position_embedding": None, "per_position_padding": None}) == \
        ("absolute", False, None)
    assert input_embedding({"per_position_padding": False, "padding_id": 3}) == ("absolute", False, None)
    assert input_embedding({"image_position_embedding": "row_col", "per_position_padding": True, "padding_id": 9,
                            "text_vocab_size": 10}) == ("row_col", True, 9)
    bad = [
        {"image_position_embedding": "learned"},
        {"image_position_embedding": 0},
        {"per_position_padding": "yes"},
        {"per_position_padding": 1},
        {"per_position_padding": True, "text_vocab_size": 10},                        # no padding_id
        {"per_position_padding": True, "padding_id": 10, "text_vocab_size": 10},     # outside the vocabulary
        {"per_position_padding": True, "padding_id": -1, "text_vocab_size": 10},
        {"per_position_padding": True, "padding_id": 2.5, "text_vocab_size": 10},
        {"per_position_padding": True, "padding_id": True, "text_vocab_size": 10},
    ]
    for p in bad:
        with pytest.raises(ValueError):
            input_embedding(p)
        with pytest.raises(ValueError):                 # raised when the model_fn is built, before any GPU work
            dalle_model_fn(None, None, "train", dict(p))
        with pytest.raises(ValueError):
            DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1,
                  n_heads=2, params=dict(p))


def test_engine_rejects_bad_keys_and_a_non_square_grid_before_any_device_work():
    with pytest.raises(ValueError, match="square image-token grid"):
        DalleEngine(256, 1, 2, 10, 16, 4, 15, image_position_embedding="row_col")
    with pytest.raises(ValueError, match="image_position_embedding"):
        DalleEngine(256, 1, 2, 10, 16, 4, 16, image_position_embedding="rows")
    with pytest.raises(ValueError, match="per_position_padding"):
        DalleEngine(256, 1, 2, 10, 16, 4, 16, per_position_padding="on")


def _generate_config(tmp_path, extra):
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64, **extra}
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    np.save(tmp_path / "ids.npy", np.zeros((1, 4), np.int32))
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})
    return ["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
            "--caption_ids", str(tmp_path / "ids.npy")]


@pytest.mark.parametrize("extra", [{"image_position_embedding": "rows"}, {"per_position_padding": 1},
                                   {"per_position_padding": True}, {"per_position_padding": True, "padding_id": 300}])
def test_generate_cli_rejects_bad_keys(tmp_path, extra):
    with pytest.raises(ValueError):
        G.main(_generate_config(tmp_path, extra))


def test_generate_cli_pads_captions_with_the_config_padding_id():
    out = G.pad_captions([[1, 2]], 4, 300, pad=9)
    assert out.tolist() == [[1, 2, 9, 9]]
    assert G.pad_captions([[1, 2]], 4, 60000).tolist() == [[1, 2, G.PADDING_ID, G.PADDING_ID]]


# ------------------------------------------------------------------------------------------------ layout and names
def _layout_names(lay):
    return list(lay.order)


def test_layout_without_the_keys_is_unchanged():
    d, Lyr, V, S = 512, 6, 50258 + 512 + 1, 1280
    lay = param_layout(d, Lyr, V, S)
    assert lay.order[:2] == ["wte", "wpe"] and lay.entries["wpe"][1] == (S, d)
    assert lay.span("wte", "wpe") == (0, lay.entries["l0.ln1_g"][0])
    assert "image_row" not in lay.entries


def test_row_col_layout_offsets_and_last_bucket():
    d, Lyr, TL, W = 512, 6, 256, 32
    V = 50258 + TL + 512 + 1
    lay = param_layout(d, Lyr, V, TL + W * W, TL, W)
    assert lay.order[:4] == ["wte", "wpe", "image_row", "image_col"] and lay.order[4] == "l0.ln1_g"
    off = 0
    for name, shape in (("wte", (V, d)), ("wpe", (TL, d)), ("image_row", (W, d)), ("image_col", (W, d))):
        assert lay.entries[name] == (off, shape)
        off += -(-shape[0] * shape[1] // 64) * 64
    # the last gradient bucket backward hands over is span(wte .. image_col): everything before layer 0
    assert lay.span("wte", "image_col") == (0, lay.entries["l0.ln1_g"][0]) == (0, off)
    base = param_layout(d, Lyr, V, TL + W * W)
    assert lay.size == base.size - (TL + W * W) * d + (TL + 2 * W) * d
    # every other entry keeps its shape; names that decay (neither "norm" nor "bias" in the reference name) include
    # the new matrices
    assert [n for n in lay.order if n not in ("wpe", "image_row", "image_col")] == \
        [n for n in base.order if n != "wpe"]


def test_vocabulary_and_image_offsets():
    tv, iv, TL = 50258, 512, 256
    # per-position pads come right after the caption vocabulary; the image codes and EOS follow them
    _, V = I.vocab(_cfg(TL=TL, W=32, tv=tv, iv=iv), BOTH)
    assert V == tv + TL + iv + 1
    assert I.vocab(_cfg(TL=TL, W=32, tv=tv, iv=iv), OFF) == (tv, tv + iv + 1)


def test_n_params_formula_counts_the_reference_style_variables():
    cfg = _cfg(TL=6, W=3, d=32, L=2, tv=50, iv=16)
    for inp in (OFF, ROW_COL, BOTH):
        p = I.init_params(cfg, inp)
        eng = DalleEngine.__new__(DalleEngine)
        eng.d, eng.L, eng.S, eng.text_seq_len = cfg.n_embd, cfg.n_layers, cfg.seq_len, cfg.text_seq_len
        eng.V = I.vocab(cfg, inp)[1]
        eng.row_col = inp.image_position_embedding == "row_col"
        eng.grid_w = 3 if eng.row_col else None
        assert eng.n_params() == sum(v.numel() for v in p.values()), inp


def test_checkpoint_names():
    cfg = _cfg(TL=6, W=3, d=32, L=2)
    off = set(I.init_params(cfg, OFF))
    rc = set(I.init_params(cfg, ROW_COL))
    assert rc - off == {"positional_embedding/image_row", "positional_embedding/image_col"}
    assert off - rc == set()
    names = DalleEngine.EMBED_REF_NAMES
    assert names["image_row"] == "positional_embedding/image_row"
    assert names["image_col"] == "positional_embedding/image_col"
    for n in ("image_row", "image_col", "wpe", "wte"):
        assert "norm" not in names[n] and "bias" not in names[n]
    assert math.isqrt(cfg.image_seq_len) == 3
