"""CPU tests of caption generation (DalleSampler.generate_texts, generate_dalle.py --gentxt): the numpy statement of
db200_caption_next that the GPU tests compare the kernel with, the prefix lengths and argument errors a user meets
before any device work, and the command's --gentxt handling."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200.sampling import FILTER_MAX_IDS, DalleSampler
from dalle_mtf_b200.utils import save_checkpoint


# ------------------------------------------------------------------------------------------------ caption_next oracle
def caption_next_ref(tokens, prefix, lens, pos, text_len, text_vocab_size, padding_id, pad_base=None):
    """db200_caption_next on host arrays: a copy of tokens int [rows, >= text_len] with text column c = pos + 1 of
    every row finished (include/dalle_b200.h).  pad_base None: no per-position padding."""
    out = np.array(tokens, dtype=np.int64, copy=True)
    c = pos + 1
    if not 1 <= c < text_len:
        return out

    def is_pad(i):
        return i == padding_id or (pad_base is not None and i >= text_vocab_size)

    for b in range(out.shape[0]):
        if c < lens[b]:
            out[b, c] = prefix[b, c]
        elif is_pad(out[b, c - 1]) or is_pad(out[b, c]):
            out[b, c] = padding_id if pad_base is None else pad_base + c
    return out


def complete_ref(prefix, lens, draws, text_vocab_size, padding_id, pad_base=None):
    """The text columns generate_texts produces when the draw for column c of row b is draws[b, c]: the prompt matrix,
    then for c = P .. text_len - 1 the draw followed by caption_next (P = min lens)."""
    TL = prefix.shape[1]
    tok = np.array(prefix, dtype=np.int64, copy=True)
    for c in range(int(min(lens)), TL):
        tok[:, c] = draws[:, c]
        tok = caption_next_ref(tok, prefix, lens, c - 1, TL, text_vocab_size, padding_id, pad_base)
    return tok


TV, PAD, TL = 20, 19, 8


def test_oracle_keeps_the_prompt_below_its_length():
    prefix = np.array([[1, 2, 3, 4, 5, 6, 7, 8], [1, 2, 3, PAD, PAD, PAD, PAD, PAD]])
    lens = [6, 3]
    tok = np.array([[1, 2, 3, 11, 12, 13, 14, 15], [1, 2, 3, 11, 12, 13, 14, 15]])
    got = caption_next_ref(tok, prefix, lens, 2, TL, TV, PAD)      # column 3
    assert got[0].tolist() == [1, 2, 3, 4, 12, 13, 14, 15]          # forced: 3 < 6
    assert got[1].tolist() == tok[1].tolist()                       # drawn: kept
    assert (np.delete(got, 3, 1) == np.delete(tok, 3, 1)).all()     # no other column changes


def test_oracle_pads_after_a_padding_token():
    prefix = np.full((3, TL), PAD)
    prefix[:, :2] = [[1, 2], [3, 4], [5, 6]]
    lens = [2, 2, 2]
    # row 0 draws padding at the prefix boundary (column 2), row 1 at column 5, row 2 never
    draws = np.array([[0, 0, PAD, 7, 8, 9, 10, 11], [0, 0, 7, 8, 9, PAD, 3, 4], [0, 0, 7, 8, 9, 10, 11, 12]])
    got = complete_ref(prefix, lens, draws, TV, PAD)
    assert got.tolist() == [[1, 2, PAD, PAD, PAD, PAD, PAD, PAD],
                            [3, 4, 7, 8, 9, PAD, PAD, PAD],
                            [5, 6, 7, 8, 9, 10, 11, 12]]


def test_oracle_per_position_pads():
    base = TV                                                       # pads TV + c, text window [0, TV + TL)
    prefix = np.array([[1, 2, 3, base + 3, base + 4, base + 5, base + 6, base + 7],
                       [4, 5, 6, 7, 8, 9, 10, 11],
                       [1, base + 1, base + 2, base + 3, base + 4, base + 5, base + 6, base + 7]])
    lens = [3, TL, 1]
    # row 0 draws a pad of another column (base + 1) at column 4, row 2 draws padding_id itself at column 2
    draws = np.array([[0, 0, 0, 9, base + 1, 9, 9, 9], [0] * TL, [0, 3, PAD, 4, 5, 6, 7, 8]])
    got = complete_ref(prefix, lens, draws, TV, PAD, base)
    assert got.tolist() == [[1, 2, 3, 9, base + 4, base + 5, base + 6, base + 7],
                            [4, 5, 6, 7, 8, 9, 10, 11],              # n = text_seq_len: unchanged
                            [1, 3, base + 2, base + 3, base + 4, base + 5, base + 6, base + 7]]
    # padding_id is a padding token with per-position padding too, and a pad in column c - 1 pads column c
    tok = np.array([[1, PAD, 5, 0, 0, 0, 0, 0]])
    assert caption_next_ref(tok, tok, [1], 1, TL, TV, PAD, base)[0, 2] == base + 2


def test_oracle_rows_at_full_length_and_columns_out_of_range():
    prefix = np.arange(2 * TL).reshape(2, TL) % 10
    tok = np.zeros_like(prefix)
    for pos in range(TL - 1):
        tok = caption_next_ref(tok, prefix, [TL, TL], pos, TL, TV, PAD)
    assert (tok[:, 1:] == prefix[:, 1:]).all() and (tok[:, 0] == 0).all()
    for pos in (-1, TL - 1, TL + 3):                                  # column 0 and columns past the text: untouched
        assert (caption_next_ref(tok, prefix, [1, 1], pos, TL, TV, PAD) == tok).all()


# ------------------------------------------------------------------------------------------------ sampler arguments
def _sampler(text_vocab_size=TV, text_seq_len=TL, per_position_padding=False, padding_id=PAD):
    """A DalleSampler over a stand-in engine: generate_texts validates before it touches the engine's device."""
    off = text_vocab_size + (text_seq_len if per_position_padding else 0)
    eng = SimpleNamespace(text_vocab_size=text_vocab_size, text_seq_len=text_seq_len, image_vocab_size=16,
                          image_offset=off, per_position_padding=per_position_padding)
    return DalleSampler(eng, padding_id=padding_id)


def test_prefix_lengths():
    s = _sampler()
    ids = torch.tensor([[1, 2, 3, 4, 5, 6, 7, 8], [1, PAD, 3, 4, 5, 6, 7, 8], [1, 2, 3, 4, 5, 6, 7, PAD],
                        [0, 0, PAD, PAD, PAD, PAD, PAD, PAD]])
    lens = s.caption_lengths(ids)
    assert lens.dtype == torch.int32 and lens.tolist() == [TL, 1, 7, 2]
    assert s.caption_lengths(ids.to(torch.int64)).tolist() == [TL, 1, 7, 2]
    # generate_dalle.pad_captions pads as the sampler reads: the prefix is the caption given
    caps = G.pad_captions([[3, 1, 4], [1, 5, 9, 2, 6, 5, 3, 5, 8]], TL, TV, PAD)
    assert s.caption_lengths(torch.from_numpy(caps)).tolist() == [3, TL]


def test_generate_texts_refuses_bad_prompts():
    s = _sampler()
    ok = torch.tensor([[1, 2, PAD, PAD, PAD, PAD, PAD, PAD]])
    for bad in (ok[0], ok[:, :-1], ok[:0], ok.float(), torch.full((1, TL), PAD), ok - 2, ok + TV, [[1] * TL]):
        with pytest.raises(ValueError):
            s.generate_texts(bad)
    with pytest.raises(ValueError, match="empty prefix"):
        s.generate_texts(torch.tensor([[1, 2, 3, 4, 5, 6, 7, 8], [PAD, 2, 3, 4, 5, 6, 7, 8]]))
    for k, p in ((0, None), (-1, None), (1.5, None), (True, None), (None, 0.0), (None, 1.5)):
        with pytest.raises(ValueError):
            s.generate_texts(ok, top_k=k, top_p=p)


def test_text_filter_is_checked_against_the_text_window():
    # window = text_vocab_size (+ text_seq_len pads): top_k at or past it filters nothing
    s = _sampler(per_position_padding=True)
    assert s._filter(TV + TL - 1, None, n_text=TV + TL) == (TV + TL - 1, 1.0)
    assert s._filter(TV + TL, None, n_text=TV + TL) is None
    # the image draw keeps comparing with image_vocab_size (16)
    assert s._filter(TV, None) is None and s._filter(15, None) == (15, 1.0)
    # 50 258 GPT-2 ids (+ 256 pads) fit the filtered kernel; a wider window refuses a filter and nothing else
    for tv, tl, pp in ((50258, 256, False), (50258, 256, True)):
        assert _sampler(tv, tl, pp)._filter(64, 0.9, n_text=tv + (tl if pp else 0)) == (64, 0.9)
    wide = _sampler(FILTER_MAX_IDS, 4, True, padding_id=0)
    prompt = torch.tensor([[1, 0, 0, 0]])
    for k, p in ((64, None), (None, 0.9), (FILTER_MAX_IDS, None)):
        with pytest.raises(ValueError, match="text window"):
            wide.generate_texts(prompt, top_k=k, top_p=p)
    assert wide._filter(None, None, n_text=FILTER_MAX_IDS + 4) is None


# ------------------------------------------------------------------------------------------------ generate_dalle.py
BASE = ["--model", "m", "--out", "o", "--caption_ids", "c.npy"]


def test_gentxt_argument():
    assert G.parse_args(BASE).gentxt is False
    a = G.parse_args(BASE + ["--gentxt", "--top_k", "64", "--temperature", "0.7"])
    assert a.gentxt is True and a.top_k == 64 and a.temperature == 0.7
    with pytest.raises(SystemExit):
        G.parse_args(BASE + ["--gentxt", "yes"])


def test_empty_captions_are_refused():
    caps = np.array([[1, 2, PAD, PAD], [PAD, PAD, PAD, PAD], [3, PAD, PAD, PAD], [PAD, 4, 5, 6]])
    with pytest.raises(SystemExit, match=r"\[1, 3\]"):
        G.check_caption_prefixes(caps, PAD)
    G.check_caption_prefixes(caps[[0, 2]], PAD)


def test_captions_npy_and_txt(tmp_path):
    caps = np.array([[5, 6, 7, PAD, PAD], [8, 9, 10, 11, 12], [13, PAD, PAD, PAD, PAD]], dtype=np.int64)

    class Tok:   # stands in for the GPT-2 tokenizer: id i decodes to word w<i>
        def decode(self, ids):
            return " ".join(f"w{i}" for i in ids)

    G.write_captions(str(tmp_path), caps, PAD, Tok())
    got = np.load(tmp_path / "captions.npy")
    assert got.dtype == np.int32 and (got == caps).all()
    assert (tmp_path / "captions.txt").read_text().splitlines() == ["w5 w6 w7", "w8 w9 w10 w11 w12", "w13"]
    # without BPE files (the stand-in tokenizer cannot decode) only captions.npy is written
    from dalle_mtf_b200.tokenizer import _PaddingOnlyTokenizer
    other = tmp_path / "no_bpe"
    other.mkdir()
    G.write_captions(str(other), caps, PAD, _PaddingOnlyTokenizer())
    assert (other / "captions.npy").exists() and not (other / "captions.txt").exists()


def _configs(tmp_path, caption_ids, padding_id=None):
    vae = {"model_type": "vae", "num_tokens": 64, "model_path": str(tmp_path / "vae_run")}
    dalle = {"model_type": "dalle", "dataset": {"image_size": 32}, "model_path": str(tmp_path / "dalle_run"),
             "vae_model": str(tmp_path / "vae.json"), "text_seq_len": 4, "text_vocab_size": 300,
             "image_vocab_size": 64}
    if padding_id is not None:
        dalle["padding_id"] = padding_id
    (tmp_path / "vae.json").write_text(json.dumps(vae))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle))
    np.save(tmp_path / "ids.npy", np.asarray(caption_ids, np.int32))
    save_checkpoint(str(tmp_path / "dalle_run"), 1, {"global_step": 1})
    save_checkpoint(str(tmp_path / "vae_run"), 1, {"global_step": 1})
    return ["--model", str(tmp_path / "dalle.json"), "--out", str(tmp_path / "out"),
            "--caption_ids", str(tmp_path / "ids.npy"), "--gentxt"]


def test_gentxt_errors_come_before_any_gpu_work(tmp_path):
    # a caption with no ids (here: all padding, and one padded from an empty row) cannot be continued
    argv = _configs(tmp_path, [[7, 8, 299, 299], [299, 299, 299, 299]], padding_id=299)
    with pytest.raises(SystemExit, match="no ids before the padding id"):
        G.main(argv)
    # the captions end at the config's padding_id, which must be a text id
    argv = _configs(tmp_path, [[7, 8, 9, 10]])
    with pytest.raises(SystemExit, match="--gentxt: padding id 50257"):
        G.main(argv)
