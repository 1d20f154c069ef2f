"""CPU tests of classifier-free guidance and caption dropout: the float32 guidance oracle and the caption-dropout
decisions (oracle/guidance.py), the config and argument validation in front of them, and the
--guidance_scale option of generate_dalle.py."""
import math
import os

import numpy as np
import pytest

import generate_dalle as G
from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.model_fns import caption_dropout, dalle_model_fn
from dalle_mtf_b200.sampling import DalleSampler
from dalle_mtf_b200.utils import save_checkpoint
from oracle import guidance as CG
from oracle import philox as X
from oracle.guidance import guided_logits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ guidance oracle
def test_scale_zero_gives_the_unconditional_row_exactly():
    g = np.random.default_rng(0)
    c = (g.standard_normal((4, 1000)) * 5).astype(np.float32)
    u = (g.standard_normal((4, 1000)) * 5).astype(np.float32)
    u[0, :10] = -0.0
    assert np.array_equal(guided_logits(c, u, 0.0), u)
    assert guided_logits(c, u, 0.0).dtype == np.float32


def test_guided_logits_round_every_op_to_float32():
    g = np.random.default_rng(1)
    c = (g.standard_normal(4096) * 3).astype(np.float32)
    u = (g.standard_normal(4096) * 3).astype(np.float32)
    for s in (0.5, 3.0, 7.5):
        d = np.float32(c - u)                                       # each op rounded, never fused
        want = np.float32(u + np.float32(np.float32(s) * d))
        assert np.array_equal(guided_logits(c, u, s), want)
        # differs from the unrounded mix somewhere: the rounding is what the kernel must reproduce
        assert not np.array_equal(guided_logits(c, u, s).astype(np.float64),
                                  u.astype(np.float64) + s * (c.astype(np.float64) - u.astype(np.float64)))


def test_guided_logits_non_finite_rules():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    c = np.array([inf, inf, 1.0, nan, 2.0, -inf], dtype=np.float32)
    u = np.array([0.0, inf, -inf, 0.0, 2.0, 0.0], dtype=np.float32)
    got = guided_logits(c, u, 3.0)
    assert got[0] == inf                   # c = +inf: +inf
    assert np.isnan(got[1])                # inf - inf
    assert np.isnan(got[2])                # -inf + inf
    assert np.isnan(got[3])
    assert got[4] == 2.0                   # c == u: u
    assert got[5] == -inf
    assert np.isnan(guided_logits(c, u, 0.0)[0])                       # 0 * inf


# ------------------------------------------------------------------------------------------------ caption dropout
def test_caption_site_is_out_of_reach_of_the_layer_sites():
    assert CG.SITE_CAPTION == L.SITE_CAPTION == 0xFFFFFFFF
    with open(os.path.join(ROOT, "include", "dalle_b200.h")) as f:
        assert "#define DB200_SITE_CAPTION 0xFFFFFFFFu" in f.read()
    for layer in range(4096):
        assert CG.SITE_CAPTION not in (X.site_attn(layer), X.site_attn_out(layer), X.site_mlp_out(layer))


def test_drop_fraction_is_binomial():
    n = 100_000
    for rate in (0.1, 0.5):
        k = int(CG.caption_dropped(rate, 1234, 3, n).sum())
        sigma = math.sqrt(n * rate * (1 - rate))
        assert abs(k - n * rate) < 5 * sigma, (rate, k)
    assert not CG.caption_dropped(0.0, 1234, 3, n).any()


def test_decisions_depend_on_the_global_index_only():
    for seed, step in ((0, 0), (5, 7), (2 ** 40 + 3, 123456)):
        whole = CG.caption_dropped(0.5, seed, step, 8, row0=0)
        split = np.concatenate([CG.caption_dropped(0.5, seed, step, 4, row0=0),
                                CG.caption_dropped(0.5, seed, step, 4, row0=4)])
        assert np.array_equal(whole, split)
        assert np.array_equal(CG.caption_dropped(0.5, seed, step, 3, row0=5), whole[5:8])
    # the step and the seed change the decisions
    a = CG.caption_dropped(0.5, 5, 1, 256)
    assert not np.array_equal(a, CG.caption_dropped(0.5, 5, 2, 256))
    assert not np.array_equal(a, CG.caption_dropped(0.5, 6, 1, 256))


def test_decision_layout_is_the_elementwise_one_with_one_column():
    seed, step, rate = 2 ** 33 + 9, 4, 0.3
    thr = int(rate * 2 ** 32)
    got = CG.caption_dropped(rate, seed, step, 11, row0=6)
    for b in range(11):
        e = 6 + b
        words = X.philox4x32_10(e >> 2, 0, CG.SITE_CAPTION, step, seed & 0xFFFFFFFF, seed >> 32)
        assert got[b] == (int(words[e & 3]) < thr)


def test_caption_dropout_config():
    assert caption_dropout({}) == (0.0, None)
    assert caption_dropout({"caption_dropout": None, "padding_id": 50257}) == (0.0, None)
    assert caption_dropout({"caption_dropout": 0.2, "padding_id": 50257, "text_vocab_size": 50258}) == (0.2, 50257)
    bad = [
        {"caption_dropout": 1.0, "padding_id": 1, "text_vocab_size": 10},
        {"caption_dropout": -0.1, "padding_id": 1, "text_vocab_size": 10},
        {"caption_dropout": float("nan"), "padding_id": 1, "text_vocab_size": 10},
        {"caption_dropout": 0.1, "text_vocab_size": 10},                         # no padding_id
        {"caption_dropout": 0.1, "padding_id": None, "text_vocab_size": 10},
        {"caption_dropout": 0.1, "padding_id": 10, "text_vocab_size": 10},       # outside the text vocabulary
        {"caption_dropout": 0.1, "padding_id": -1, "text_vocab_size": 10},
        {"caption_dropout": 0.1, "padding_id": 2.5, "text_vocab_size": 10},
        {"caption_dropout": 0.1, "padding_id": True, "text_vocab_size": 10},
    ]
    for p in bad:
        with pytest.raises(ValueError):
            caption_dropout(p)
        with pytest.raises(ValueError):                      # raised when the model_fn is built, before any GPU work
            dalle_model_fn(None, None, "train", p)
        with pytest.raises(ValueError):
            dalle_model_fn(None, None, "eval", p)


# ------------------------------------------------------------------------------------------------ sampler arguments
class _Engine:
    text_vocab_size = 300


def test_guidance_scale_and_padding_id_validation():
    assert DalleSampler._guidance(None) is None
    assert DalleSampler._guidance(1.0) is None and DalleSampler._guidance(1) is None      # 1 = the plain sampler
    assert DalleSampler._guidance(0) == 0.0 and DalleSampler._guidance(3) == 3.0
    assert DalleSampler._guidance(np.float32(7.5)) == 7.5
    for bad in (-0.5, float("nan"), float("inf"), True, "3", [3.0]):
        with pytest.raises(ValueError):
            DalleSampler._guidance(bad)
    assert DalleSampler(_Engine()).padding_id == 299
    assert DalleSampler(_Engine(), padding_id=0).padding_id == 0
    for bad in (300, -1, 1.5, True):
        with pytest.raises(ValueError):
            DalleSampler(_Engine(), padding_id=bad)


# ------------------------------------------------------------------------------------------------ generate_dalle.py
BASE = ["--model", "m", "--out", "o", "--caption_ids", "c.npy"]


def test_guidance_scale_argument():
    assert G.parse_args(BASE).guidance_scale is None
    assert G.parse_args(BASE + ["--guidance_scale", "3"]).guidance_scale == 3.0
    assert G.parse_args(BASE + ["--guidance_scale", "0"]).guidance_scale == 0.0
    for bad in ("-1", "-0.01", "nan", "inf", "x"):
        with pytest.raises(SystemExit):
            G.parse_args(BASE + ["--guidance_scale", bad])


def test_guidance_padding_id_comes_from_the_config(tmp_path):
    assert G.padding_id({"padding_id": 7}) == 7
    assert G.padding_id({}) == G.PADDING_ID == 50257
    # a config whose text vocabulary does not hold the padding id is refused before any GPU work
    import json
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64}
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    np.save(tmp_path / "ids.npy", np.zeros((1, 4), np.int32))
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})
    argv = ["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
            "--caption_ids", str(tmp_path / "ids.npy"), "--guidance_scale", "3"]
    with pytest.raises(SystemExit, match="padding id 50257"):
        G.main(argv)
