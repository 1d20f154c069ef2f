"""CPU tests of generate_dalle.py's host side: arguments, caption ids, the prompt-rows arithmetic, the uint8 conversion
and the errors a user meets before any GPU work (missing checkpoints, missing GPT-2 BPE files)."""
import json
from collections import defaultdict

import numpy as np
import pytest

import generate_dalle as G
from dalle_mtf_b200.tokenizer import _PaddingOnlyTokenizer
from dalle_mtf_b200.utils import save_checkpoint

BASE = ["--model", "m", "--out", "o"]


def test_arguments():
    a = G.parse_args(BASE + ["--caption_ids", "c.npy"])
    assert a.samples_per_prompt == 1 and a.temperature == 1.0 and a.seed == 0
    assert a.batch_size is None and a.top_k is None and a.top_p is None and a.image_prompt is None
    a = G.parse_args(BASE + ["--captions", "c.txt", "--image_prompt", "x.png", "y.png", "--prompt_rows", "3",
                             "--samples_per_prompt", "4", "--top_k", "5", "--top_p", "0.9", "--batch_size", "8"])
    assert a.image_prompt == ["x.png", "y.png"] and a.prompt_rows == 3 and a.samples_per_prompt == 4
    assert (a.top_k, a.top_p, a.batch_size) == (5, 0.9, 8)
    bad = [
        BASE,                                                                      # no captions
        BASE + ["--captions", "c.txt", "--caption_ids", "c.npy"],                  # both sources
        ["--out", "o", "--caption_ids", "c.npy"],                                  # no model
        BASE + ["--caption_ids", "c.npy", "--image_prompt", "x.png"],              # prompt without rows
        BASE + ["--caption_ids", "c.npy", "--prompt_rows", "2"],                   # rows without prompt
        BASE + ["--caption_ids", "c.npy", "--samples_per_prompt", "0"],
        BASE + ["--caption_ids", "c.npy", "--batch_size", "0"],
        BASE + ["--caption_ids", "c.npy", "--top_k", "0"],
        BASE + ["--caption_ids", "c.npy", "--top_p", "0"],
        BASE + ["--caption_ids", "c.npy", "--top_p", "1.5"],
    ]
    for argv in bad:
        with pytest.raises(SystemExit):
            G.parse_args(argv)


def test_caption_ids_are_padded_and_truncated_like_training(tmp_path):
    p = tmp_path / "ids.npy"
    np.save(p, np.array([[1, 2, 3], [4, 5, 6]], dtype=np.int64))
    got = G.load_caption_ids(str(p), 5, 50258)
    assert got.dtype == np.int32 and (got == [[1, 2, 3, 50257, 50257], [4, 5, 6, 50257, 50257]]).all()
    assert (G.load_caption_ids(str(p), 2, 50258) == [[1, 2], [4, 5]]).all()
    np.save(p, np.array([7, 8], dtype=np.int32))                                   # one caption
    assert (G.load_caption_ids(str(p), 3, 50258) == [[7, 8, 50257]]).all()
    for bad in (np.zeros((1, 2, 3), np.int32), np.zeros((2, 3), np.float32), np.array([[1, 300]]),
                np.array([[-1, 2]]), np.zeros((0, 3), np.int32)):
        np.save(p, bad)
        with pytest.raises(SystemExit):
            G.load_caption_ids(str(p), 4, 300)


def test_captions_without_bpe_files_point_at_caption_ids():
    with pytest.raises(SystemExit, match="--caption_ids"):
        G.encode_captions(["a cat"], _PaddingOnlyTokenizer(), 8, 50258)

    class Tok:
        def encode(self, s):
            return [len(w) for w in s.split()]
    assert (G.encode_captions(["ab c", "abcd"], Tok(), 3, 50258) == [[2, 1, 50257], [4, 50257, 50257]]).all()


def _params(image_size, convblocks=None, stack_factor=None):
    p = defaultdict(lambda: None, {"dataset": {"image_size": image_size}})
    vp = {}
    if convblocks is not None:
        vp["convblocks"] = convblocks
    if stack_factor is not None:
        vp["stack_factor"] = stack_factor
    p["vae_params"] = defaultdict(lambda: None, vp)
    return p


def test_prompt_rows_to_prefix_length():
    p = _params(256)                                                  # default convblocks: 3 halvings -> 32 x 32
    assert G.token_grid_side(p) == 32 and G.prefix_length(p, 16) == 512 and G.prefix_length(p, 1) == 32
    p = _params(256, [[2, 64], [2, 128]], stack_factor=2)             # 256 / 2 / 4 -> 32
    assert G.token_grid_side(p) == 32 and G.prefix_length(p, 3) == 96
    p = _params(32, [[2, 64], [2, 128]])
    assert G.token_grid_side(p) == 8 and G.prefix_length(p, 7) == 56
    for r in (0, 8, -1):
        with pytest.raises(SystemExit):
            G.prefix_length(p, r)


def test_uint8_conversion():
    x = np.array([-2.0, -1.0, -0.5, 0.0, 0.001, 0.5, 1.0, 3.0], dtype=np.float32)
    got = G.to_uint8(x)
    assert got.dtype == np.uint8
    assert got.tolist() == [0, 0, 64, 128, 128, 191, 255, 255]


def _write_configs(tmp_path, vae_ckpt_dir=True):
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64}
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    np.save(tmp_path / "ids.npy", np.zeros((1, 4), np.int32))
    return ["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
            "--caption_ids", str(tmp_path / "ids.npy")]


def test_missing_checkpoints_are_reported_before_any_gpu_work(tmp_path):
    argv = _write_configs(tmp_path)
    with pytest.raises(SystemExit, match="no DALL-E checkpoint"):
        G.main(argv)
    with pytest.raises(SystemExit, match="no DALL-E checkpoint"):
        G.main(argv + ["--checkpoint", str(tmp_path / "nope.pt")])
    save_checkpoint(str(tmp_path / "dalle_run"), 5, {"global_step": 5})
    with pytest.raises(SystemExit, match="no VAE checkpoint"):
        G.main(argv)
    params = G.load_params(str(tmp_path / "dalle.json"))
    save_checkpoint(str(tmp_path / "vae_run"), 2, {"global_step": 2})
    save_checkpoint(str(tmp_path / "vae_run"), 9, {"global_step": 9})
    ckpt, vae_ckpt = G.find_checkpoints(params)
    assert ckpt.endswith("model.ckpt-5.pt") and vae_ckpt.endswith("model.ckpt-9.pt")
    params["vae_checkpoint_path"] = str(tmp_path / "missing.pt")
    with pytest.raises(SystemExit, match="no VAE checkpoint"):
        G.find_checkpoints(params)


def test_prompt_images_must_match_the_captions(tmp_path):
    argv = _write_configs(tmp_path)
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})
    with pytest.raises(SystemExit, match="prompt images"):
        G.main(argv + ["--image_prompt", "a.png", "b.png", "--prompt_rows", "2"])
    with pytest.raises(SystemExit, match="prompt_rows"):
        G.main(argv + ["--image_prompt", "a.png", "--prompt_rows", "8"])


def test_a_non_dalle_config_is_refused(tmp_path):
    (tmp_path / "v.json").write_text(json.dumps({"model_type": "vae"}))
    with pytest.raises(SystemExit, match="not a DALL-E config"):
        G.load_params(str(tmp_path / "v.json"))
