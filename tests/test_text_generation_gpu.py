"""GPU tests of caption generation: db200_caption_next(_at) against the numpy statement in
test_text_generation_cpu.py, the samplers over the GPT-2 text window, DalleEngine.prefill at prompts shorter than the
caption against the teacher-forced decoder, DalleSampler.generate_texts / DALLE.generate_texts and
generate_dalle.py --gentxt end to end."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.sampling import boundary_margin, keep_mask
from test_sampling_filter_gpu import MARGIN, check_selection, perturbed, scaled
from test_text_generation_cpu import caption_next_ref

pytestmark = pytest.mark.gpu

DEV = "cuda"


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ caption_next
@pytest.mark.parametrize("per_position", [False, True])
def test_caption_next_matches_the_oracle(ops, per_position):
    B, TL, TV = 32, 256, 50258
    PAD = TV - 1
    base = TV if per_position else None
    rng = np.random.default_rng(5 + per_position)
    lens = rng.integers(1, TL + 1, B)
    lens[:3] = (1, TL, TL - 1)
    prefix = rng.integers(0, TV - 1, (B, TL))
    for b in range(B):   # the prompt in token form: its padding is padding_id, or each column's pad
        prefix[b, lens[b]:] = base + np.arange(lens[b], TL) if per_position else PAD
    # a token matrix of draws over the text window with padding tokens sprinkled in: padding_id, and with per-position
    # padding pads of the right and of other columns
    hi = TV + (TL if per_position else 0)
    tok = rng.integers(0, hi, (B, TL + 5))
    tok[rng.random((B, TL + 5)) < 0.05] = PAD
    ld_prefix = TL + 3
    pre = np.zeros((B, ld_prefix), np.int64)
    pre[:, :TL] = prefix
    t_dev = torch.from_numpy(tok.astype(np.int32)).to(DEV)
    p_dev = torch.from_numpy(pre.astype(np.int32)).to(DEV)
    l_dev = torch.from_numpy(lens.astype(np.int32)).to(DEV)
    pos_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    want = tok.copy()
    t_at = t_dev.clone()
    for pos in range(TL - 1):   # every column in turn, as generation runs them; the two variants side by side
        want = caption_next_ref(want, prefix, lens, pos, TL, TV, PAD, base)
        ops.caption_next(t_dev, p_dev, l_dev, pos, TL, TV, PAD, base)
        pos_dev.fill_(pos)
        ops.caption_next_at(t_at, p_dev, l_dev, pos_dev, TL, TV, PAD, base)
        if pos in (0, 1, 37, TL - 2):
            assert np.array_equal(t_dev.cpu().numpy(), want), pos
    assert np.array_equal(t_dev.cpu().numpy(), want) and torch.equal(t_at, t_dev)
    assert np.array_equal(want[:, TL:], tok[:, TL:]) and np.array_equal(want[:, 0], tok[:, 0])
    # the completed rows: prompt kept, everything after a padding token padded
    for b in range(B):
        row = want[b, :TL]
        assert np.array_equal(row[1:lens[b]], prefix[b, 1:lens[b]])
        padded = (row == PAD) | ((row >= TV) if per_position else False)
        first = np.argmax(padded[lens[b]:]) + lens[b] if padded[lens[b]:].any() else TL
        assert padded[first:].all()
    # a device position past the text leaves the matrix alone
    pos_dev.fill_(TL - 1)
    ops.caption_next_at(t_at, p_dev, l_dev, pos_dev, TL, TV, PAD, base)
    assert torch.equal(t_at, t_dev)


def test_caption_next_refuses_bad_arguments():
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    L.require_device()
    s = L.stream_ptr()
    t = torch.zeros(4, 8, dtype=torch.int32, device=DEV)
    n = torch.ones(4, dtype=torch.int32, device=DEV)
    T, N = t.data_ptr(), n.data_ptr()
    assert lib.db200_caption_next(s, T, 8, T, 8, N, 4, 8, 20, 19, -1, 0) == 0
    assert lib.db200_caption_next(s, T, 8, T, 8, N, 4, 8, 20, 19, 20, 6) == 0
    for args in ((8, 8, 4, 8, 20, 19, -1, 7), (8, 8, 4, 8, 20, 19, -1, -1), (7, 8, 4, 8, 20, 19, -1, 0),
                 (8, 7, 4, 8, 20, 19, -1, 0), (8, 8, 0, 8, 20, 19, -1, 0), (8, 8, 4, 8, 20, 20, -1, 0),
                 (8, 8, 4, 8, 20, 19, 19, 0)):
        ld, ldp, rows, tl, tv, pad, base, pos = args
        assert lib.db200_caption_next(s, T, ld, T, ldp, N, rows, tl, tv, pad, base, pos) == -1, args
    assert lib.db200_caption_next(s, None, 8, T, 8, N, 4, 8, 20, 19, -1, 0) == -1
    assert lib.db200_caption_next_at(s, T, 8, T, 8, N, 4, 8, 20, 19, -1, None) == -1
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ text-window draws
@pytest.mark.parametrize("n", [50258, 50514])
def test_samplers_over_the_text_window_match_the_oracle(ops, n):
    rows, ld = 32, n + 46          # ld: the vocabulary rows padded past the window, as the logits buffer is
    g = torch.Generator(device=DEV).manual_seed(n)
    scale = torch.exp(torch.empty(rows, 1, device=DEV).uniform_(np.log(2.5), np.log(10.0), generator=g))
    logits = torch.randn(rows, ld, device=DEV, generator=g) * scale
    logits[:, n:] = 100.0                                       # past the window: never drawn
    u = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    idx = torch.empty(rows, dtype=torch.int32, device=DEV)
    kept = torch.empty(rows, dtype=torch.int32, device=DEV)
    tokens = torch.zeros(rows, 9, dtype=torch.int32, device=DEV)
    pos_dev = torch.full((1,), 4, dtype=torch.int32, device=DEV)
    compared = decisions = 0
    for inv_temp in (1.0, 1.4):
        pert = perturbed(logits[:, :n], u, inv_temp)
        x = scaled(logits[:, :n], inv_temp)
        every = np.ones((rows, n), bool)
        for noise in (None, u):      # the unfiltered kernel: the first maximum of x (+ noise)
            ops.sample_rows(logits, noise, idx, 0, n, inv_temp)
            ops.sample_rows_at(logits, noise, tokens, 0, n, inv_temp, pos_dev)
            assert torch.equal(tokens[:, 5], idx)
            want = pert if noise is not None else torch.from_numpy(x)
            assert check_selection(idx.cpu().long(), 0, every, want, np.ones(rows, bool)) >= rows - 1
        for k, p in ((64, 1.0), (0, 0.9), (64, 0.9), (1, 1.0), (n - 1, 0.999)):
            pf = float(np.float32(p))
            mask = keep_mask(x, k, pf)
            ok = boundary_margin(x, k, pf) > MARGIN
            ops.sample_rows_filtered(logits, u, idx, 0, n, inv_temp, k, p, kept=kept)
            assert np.array_equal(kept.cpu().numpy()[ok], mask.sum(-1)[ok]), (k, p)
            assert check_selection(idx.cpu().long(), 0, mask, pert, ok) >= 0.99 * ok.sum()
            ops.sample_rows_filtered_at(logits, u, tokens, 0, n, inv_temp, k, p, pos_dev)
            assert torch.equal(tokens[:, 5], idx)
            compared, decisions = compared + int(ok.sum()), decisions + rows
    assert compared >= 0.75 * decisions     # rows within MARGIN of a top-p tie are not compared


# ------------------------------------------------------------------------------------------------ engines
D, TS, ISL, TV, IV = 256, 112, 16, 300, 32          # S = 128: a gMLP layer's multiple of 64, a 4 x 4 image grid
CONFIGS = {
    "plain": dict(n_layers=2),
    "pp_mask": dict(n_layers=2, per_position_padding=True, logits_mask=True),
    "rotary_emb_shift_sandwich": dict(n_layers=2, rotary_emb=True, shift_tokens=True, sandwich_norm=True),
    "rotary_dim": dict(n_layers=2, rotary_dim=32),
    "stable_tied": dict(n_layers=2, stable=True, share_input_output_emb=True),
    "layer_mix": dict(n_layers=6, attention_types=["mlp", "local", "axial_row", "axial_col", "conv", "block_sparse"],
                      local_attention_radius=5, conv_attention_kernel=3),
}
_ENGINES = {}


def engine(name):
    """An engine of configuration `name` at random initialisation with its embedding and output projection scaled by
    4, so that most greedy decisions are clear of a tie (cached per module)."""
    if name not in _ENGINES:
        from dalle_mtf_b200.dalle_engine import DalleEngine
        kw = dict(CONFIGS[name])
        Lyr = kw.pop("n_layers")
        eng = DalleEngine(D, Lyr, 2, TV, IV, TS, ISL, **kw)
        eng.init_params(7)
        for nm in ("wte", "wout"):
            if nm in eng.layout.entries and nm not in eng.layout.aliases:
                eng.layout.view(eng.master, nm).mul_(4)
        eng.refresh_shadow()
        _ENGINES[name] = eng
    return _ENGINES[name]


def token_rows(eng, smp, captions):
    """[B, S] token rows of caption ids (token form) followed by image code 0: what DalleEngine.logits reads."""
    B = captions.shape[0]
    img = torch.full((B, eng.image_seq_len), eng.image_offset, dtype=torch.int32, device=DEV)
    return torch.cat([smp._captions(captions.to(DEV).to(torch.int32)), img], 1).contiguous()


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_prefill_shorter_than_the_caption(name):
    from dalle_mtf_b200.sampling import DalleSampler
    eng = engine(name)
    B = 3
    g = torch.Generator().manual_seed(3)
    text = torch.randint(0, TV - 1, (B, TS), generator=g).to(torch.int32).to(DEV)
    smp = DalleSampler(eng)
    toks = smp.generate(text, temperature=0)             # teacher-forced caches of every text position
    full = eng.logits(toks)
    mlp = [eng._is_mlp(i) for i in range(eng.L)]
    for P in (1, 7, 64, TS - 1):
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [None if c is None else torch.zeros_like(c) for c in smp.vc]
        sc = [torch.zeros_like(c) for c in smp.sc] if eng.shift_tokens else None
        logits = eng.prefill(toks[:, :P].contiguous(), kc, vc, shift_caches=sc).clone()
        torch.cuda.synchronize()
        # layer 0's K / V, SGU cache (a gMLP layer) and LN1 shift cache: the same per-row arithmetic on the embedding
        assert torch.equal(kc[0][:, :P], smp.kc[0][:, :P]), P
        if not mlp[0]:
            assert torch.equal(vc[0][:, :P], smp.vc[0][:, :P]), P
        if sc is not None:
            assert torch.equal(sc[0][:, :P], smp.sc[0][:, :P]), P
            # LN2 of layer 0 onwards reads the token mixer's output: flash attention vs the decode kernel
            for j in range(1, 2 * eng.L):
                assert relfro(sc[j][:, :P], smp.sc[j][:, :P]) <= 1e-2, (P, j)
        for i in range(1, eng.L):   # deeper layers: flash attention vs the decode kernels
            assert relfro(kc[i][:, :P], smp.kc[i][:, :P]) <= 1e-2, (P, i)
            if not mlp[i]:
                assert relfro(vc[i][:, :P], smp.vc[i][:, :P]) <= 1e-2, (P, i)
        for c in kc + vc + (sc or []):
            assert c is None or not c[:, P:].any()
        w = eng.image_offset                               # a text row: its window
        assert relfro(logits[:, :w], full[:, P - 1, :w]) < 2e-2, P


def clear_argmax(full, c, window):
    """(argmax, clear) of the logits window of position c - 1: clear when its top-2 gap exceeds 5 % of the largest
    magnitude (the criterion of test_prefill_gpu.py)."""
    rng = full[:, c - 1, :window]
    top2 = rng.topk(2, -1).values
    return rng.argmax(-1), (top2[:, 0] - top2[:, 1]) > 0.05 * rng.abs().max(-1).values


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_greedy_caption_follows_the_model(name):
    from dalle_mtf_b200.sampling import DalleSampler
    eng = engine(name)
    smp = DalleSampler(eng)
    pad, tv, W = smp.padding_id, eng.text_vocab_size, eng.image_offset
    lens = [5, 1, 40, TS, 2]
    g = torch.Generator().manual_seed(11)
    text = torch.randint(0, pad, (len(lens), TS), generator=g).to(torch.int32)
    for b, n in enumerate(lens):
        text[b, n:] = pad
    out = smp.generate_texts(text.to(DEV), temperature=0)
    assert out.shape == text.shape and out.dtype == torch.int32 and out.device.type == "cuda"
    out_h = out.cpu()
    full = eng.logits(token_rows(eng, smp, out))
    is_pad = lambda t: (t == pad) | (t >= tv)
    total = same = clear = 0
    for b, n in enumerate(lens):
        assert torch.equal(out_h[b, :n], text[b, :n])                 # the prefix, bit for bit
        assert ((out_h[b, n:] >= 0) & (out_h[b, n:] < tv)).all()       # caption ids: pads come back as padding_id
        padded = is_pad(out_h[b])
        first = int(padded[n:].to(torch.int32).argmax()) + n if padded[n:].any() else TS
        assert padded[first:].all()                                    # padding ends the caption
        for c in range(n, min(first + 1, TS)):
            am, ok = clear_argmax(full[b:b + 1], c, W)
            hit = bool(is_pad(am)[0]) if c == first else int(am[0]) == int(out_h[b, c])
            assert hit or not bool(ok[0]), (b, c)
            total, same, clear = total + 1, same + hit, clear + bool(ok[0])
    assert clear > 0.2 * total and same > 0.8 * total, (name, total, same, clear)
    # each row alone: the same caption, except after a decision the full forward pass calls a near tie
    for b, n in enumerate(lens):
        alone = smp.generate_texts(text[b:b + 1].to(DEV), temperature=0).cpu()[0]
        diff = (alone != out_h[b]).nonzero().flatten()
        if len(diff):
            c = int(diff[0])
            _, ok = clear_argmax(full[b:b + 1], c, W)
            assert c >= n and not bool(ok[0]), (name, b, c)


def test_seeded_sampling_repeats_and_top1_is_greedy():
    from dalle_mtf_b200.models import DALLE
    from dalle_mtf_b200.sampling import DalleSampler
    eng = engine("pp_mask")
    smp = DalleSampler(eng)
    pad = smp.padding_id
    text = torch.full((6, TS), pad, dtype=torch.int32, device=DEV)
    text[:, :3] = torch.arange(3 * 6, dtype=torch.int32, device=DEV).view(6, 3) + 10
    text[4, 3:20] = 7
    runs = []
    for kw in (dict(), dict(top_k=64), dict(top_p=0.9)):
        torch.manual_seed(5)
        a = smp.generate_texts(text, temperature=1.3, **kw)        # captures
        torch.manual_seed(5)
        b = smp.generate_texts(text, temperature=1.3, **kw)        # replays the same graph
        assert torch.equal(a, b), kw
        assert torch.equal(a[:, :3], text[:, :3]) and torch.equal(a[4, :20], text[4, :20])
        runs.append(a)
    torch.manual_seed(5)
    assert torch.equal(DalleSampler(eng).generate_texts(text, temperature=1.3), runs[0])   # a fresh capture
    greedy = smp.generate_texts(text, temperature=0)
    assert torch.equal(smp.generate_texts(text, temperature=1.0, top_k=1), greedy)
    # image sampling after text sampling (and back) runs its own graphs over the same caches
    img = smp.complete(greedy, temperature=0)
    assert torch.equal(img[:, :TS], smp._captions(greedy))
    assert torch.equal(smp.generate_texts(text, temperature=0), greedy)
    # the model class forwards to the sampler
    m = DALLE(256, text_vocab_size=200, image_vocab_size=32, text_seq_len=8, image_seq_len=16, n_layers=1, n_heads=2)
    t = torch.tensor([[5, 6, 199, 199, 199, 199, 199, 199], [1, 2, 3, 4, 5, 6, 7, 8]], dtype=torch.int32)
    out = m.generate_texts(t, temperature=0)
    assert out.shape == (2, 8) and torch.equal(out[:, :2].cpu(), t[:, :2]) and torch.equal(out[1].cpu(), t[1])


# ------------------------------------------------------------------------------------------------ command
def test_generate_dalle_gentxt_end_to_end(tmp_path):
    import generate_dalle
    from PIL import Image
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.utils import save_checkpoint
    from dalle_mtf_b200.vae_engine import VaeEngine

    size, convblocks, K = 32, [[2, 64], [2, 128]], 64
    tv, ts, pad = 300, 12, 299
    vae_cfg = {"model_type": "vae", "dataset": {"image_size": size}, "num_tokens": K, "convblocks": convblocks,
               "model_path": str(tmp_path / "vae_run"), "use_bf16": True}
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": size}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts, "padding_id": pad,
                 "vae_model": str(tmp_path / "vae.json")}
    (tmp_path / "vae.json").write_text(json.dumps(vae_cfg))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    vae = VaeEngine(K, size, convblocks, 3, True, False, 1)
    vae.init_params(4)
    st = {"vae/" + k: v for k, v in vae.export_params().items()}
    st.update({"vae/" + k + "/Adam": v for k, v in vae.export_params(vae.adam_m).items()})
    st.update({"vae/" + k + "/Adam_1": v for k, v in vae.export_params(vae.adam_v).items()})
    st["global_step"] = 7
    save_checkpoint(vae_cfg["model_path"], 7, st)
    hw = size // 4
    eng = DalleEngine(256, 2, 2, tv, K, ts, hw * hw)
    eng.init_params(5)
    st = dict(eng.export_params())
    st.update({k + "/adam_m": v for k, v in eng.export_params(eng.adam_m).items()})
    st.update({k + "/adam_v": v for k, v in eng.export_params(eng.adam_v).items()})
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)

    caps = np.full((3, ts), pad, np.int32)
    caps[0, :2], caps[1, :5], caps[2, :] = [4, 5], [6, 7, 8, 9, 10], np.arange(ts) + 20
    np.save(tmp_path / "caps.npy", caps)
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out), "--caption_ids",
                         str(tmp_path / "caps.npy"), "--gentxt", "--samples_per_prompt", "2", "--seed", "1",
                         "--top_k", "50"])
    done = np.load(out / "captions.npy")
    assert done.shape == (3, ts) and done.dtype == np.int32
    for b, n in enumerate((2, 5, ts)):
        assert (done[b, :n] == caps[b, :n]).all()
    assert ((done >= 0) & (done < tv)).all()
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (6, ts + hw * hw)
    assert (toks[:, :ts] == np.repeat(done, 2, 0)).all()
    assert ((toks[:, ts:] >= tv) & (toks[:, ts:] < tv + K)).all()
    pngs = sorted(p for p in os.listdir(out) if p.endswith(".png"))
    assert pngs == [f"{c:05d}_{s:02d}.png" for c in range(3) for s in range(2)]
    for p in pngs:
        assert Image.open(out / p).size == (size, size)
