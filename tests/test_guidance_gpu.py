"""GPU tests of classifier-free guidance and caption dropout: db200_sample_rows_guided against the float32 guidance
oracle (oracle/guidance.py) followed by the keep-mask / Gumbel-max oracle (oracle/sampling.py), the guided decoder (DalleSampler generate /
generate_graphed / complete, DALLE.sample) against step-by-step references, and db200_assemble_tokens_ex plus the
caption_dropout wiring of dalle_model_fn against oracle/guidance.py's decisions."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import guidance as CG
from oracle.guidance import guided_logits
from oracle.sampling import boundary_margin, keep_mask
from test_sampling_filter_gpu import MARGIN, check_selection, sharp_engine

pytestmark = pytest.mark.gpu

DEV = "cuda"
SCALES = (0.0, 0.5, 3.0, 7.5)
FILTERS = ((0, 1.0), (64, 1.0), (0, 0.9), (64, 0.9))


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import ops as o
    return o


def guided_x(logits, rows, lo, hi, s, inv_temp):
    """float32 x = guided_logits(c, u, s) * inv_temp of every pair (host numpy), from [2 rows, ld] device logits."""
    lg = logits[:, lo:hi].cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        return (guided_logits(lg[:rows], lg[rows:], s) * np.float32(inv_temp)).astype(np.float32)


def first_argmax(x, mask):
    """First index of the maximum of x over mask per row (0 where the mask is empty)."""
    xs = np.where(mask, x.astype(np.float64), -np.inf)
    return np.where(mask.any(-1), np.argmax(xs, -1), 0)


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("rows,n", [(1, 512), (32, 512), (130, 512), (1, 8192), (32, 8192), (130, 8192),
                                    (1, 32768), (32, 32768), (130, 32768)])
def test_guided_draws_match_the_float32_oracle(ops, rows, n):
    check_guided_rows(ops, rows, n)


def check_guided_rows(ops, rows, n):
    """sample_rows_guided over n ids at lo = 7 of rows pairs with ld = lo + n + 5, for every guidance scale, two
    temperatures and the filters: greedy draws are the oracle's first maximum of the kept set, kept counts equal the
    oracle's, noisy draws the first Gumbel-max, both rows of a pair get the draw and no other column is written."""
    g = torch.Generator(device=DEV).manual_seed(rows * 13 + n)
    lo = 7
    hi, ld = lo + n, lo + n + 5
    scale = torch.exp(torch.empty(2 * rows, 1, device=DEV).uniform_(math.log(1.0), math.log(4.0), generator=g))
    logits = torch.randn(2 * rows, ld, device=DEV, generator=g) * scale
    noise = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    tokens = torch.full((2 * rows, 3), -5, dtype=torch.int32, device=DEV)
    kept = torch.empty(rows, dtype=torch.int32, device=DEV)
    compared = near = exact = 0
    for s in SCALES:
        for inv_temp in (1.0, 0.8):
            x = guided_x(logits, rows, lo, hi, s, inv_temp)
            pert = torch.from_numpy(x).to(DEV) + -torch.log(-torch.log(noise))
            for k, p in FILTERS:
                pf = float(np.float32(p))
                mask = keep_mask(x.astype(np.float64), k, pf)
                ok = boundary_margin(x.astype(np.float64), k, pf) > MARGIN
                filtered = (k, p) != (0, 1.0)
                # greedy: the first maximum of the kept set, exactly
                ops.sample_rows_guided(logits, None, tokens[:, 1:2], lo, hi, inv_temp, s, k, p,
                                       kept=kept if filtered else None)
                t = tokens.cpu().numpy()
                assert (t[:rows, 1] == t[rows:, 1]).all(), "both rows of a pair receive the draw"
                assert (t[:, 0] == -5).all() and (t[:, 2] == -5).all(), "only the addressed column is written"
                want = first_argmax(x, mask) + lo
                assert (t[:rows, 1][ok] == want[ok]).all(), (s, inv_temp, k, p)
                if filtered:
                    assert (kept.cpu().numpy()[ok] == mask.sum(-1)[ok]).all(), (s, inv_temp, k, p)
                # with noise: a kept id maximising x + Gumbel (torch's log may differ from logf in the last bit)
                ops.sample_rows_guided(logits, noise, tokens[:, 1:2], lo, hi, inv_temp, s, k, p)
                t = tokens[:, 1].cpu()
                assert torch.equal(t[:rows], t[rows:])
                exact += check_selection(t[:rows].long(), lo, mask, pert, ok)
                compared += int(ok.sum())
                near += int((~ok).sum())
    assert near <= 0.25 * (compared + near)
    assert exact >= 0.999 * compared


@pytest.mark.parametrize("n", [512, 8192])
def test_scale_zero_is_the_plain_sampler_on_the_unconditional_rows(ops, n):
    g = torch.Generator(device=DEV).manual_seed(n)
    rows, lo = 32, 3
    hi = lo + n
    logits = torch.randn(2 * rows, hi + 1, device=DEV, generator=g) * 3
    noise = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    tokens = torch.empty(2 * rows, 1, dtype=torch.int32, device=DEV)
    ref = torch.empty(rows, dtype=torch.int32, device=DEV)
    for u in (None, noise):
        for inv_temp in (1.0, 0.7):
            ops.sample_rows(logits[rows:], u, ref, lo, hi, inv_temp)
            ops.sample_rows_guided(logits, u, tokens, lo, hi, inv_temp, 0.0)
            assert torch.equal(tokens[:rows, 0], ref) and torch.equal(tokens[rows:, 0], ref)
            for k, p in FILTERS[1:]:
                ops.sample_rows_filtered(logits[rows:], u, ref, lo, hi, inv_temp, k, p)
                ops.sample_rows_guided(logits, u, tokens, lo, hi, inv_temp, 0.0, k, p)
                assert torch.equal(tokens[:rows, 0], ref), (u is None, inv_temp, k, p)


def test_device_position_writes_column_pos_plus_one_of_both_rows(ops):
    g = torch.Generator(device=DEV).manual_seed(2)
    rows, lo, n, S = 16, 50, 8192, 40
    logits = torch.randn(2 * rows, lo + n, device=DEV, generator=g)
    noise = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    ids = torch.empty(2 * rows, 1, dtype=torch.int32, device=DEV)
    pos = torch.tensor([21], dtype=torch.int32, device=DEV)
    for k, p in FILTERS:
        ops.sample_rows_guided(logits, noise, ids, lo, lo + n, 1.2, 3.0, k, p)
        tokens = torch.full((2 * rows, S), -7, dtype=torch.int32, device=DEV)
        ops.sample_rows_guided(logits, noise, tokens, lo, lo + n, 1.2, 3.0, k, p, pos_dev=pos)
        want = torch.full_like(tokens, -7)
        want[:, 22] = ids[:, 0]
        assert torch.equal(tokens, want), (k, p)
        again = torch.full_like(tokens, -7)
        ops.sample_rows_guided(logits, noise, again, lo, lo + n, 1.2, 3.0, k, p, pos_dev=pos)
        assert torch.equal(again, tokens)                                   # bit-reproducible


# rows of (c, u): the guided value per id is the oracle's; NaN is never selected, +inf wins, no usable id gives lo
INF, NAN = math.inf, math.nan
HAND = [
    ("nan_skipped", [NAN, 1.0, 5.0, 2.0], [0.0, 0.0, 0.0, 0.0]),
    ("inf_minus_inf", [INF, 1.0, 2.0, 0.5], [INF, 0.0, 0.0, 0.0]),          # id 0 is NaN, not +inf
    ("neg_inf_uncond", [9.0, 1.0, 2.0, 0.5], [-INF, 0.0, 0.0, 0.0]),       # -inf + inf = NaN
    ("pos_inf_wins", [1.0, INF, 2.0, INF], [0.0, 0.0, 0.0, 0.0]),
    ("ties", [2.0, 3.0, 3.0, 1.0], [1.0, 3.0, 3.0, 0.0]),
    ("all_nan", [INF, INF, INF, INF], [INF, INF, INF, INF]),
    ("neg_inf_cond", [-INF, 1.0, -INF, 0.0], [0.0, 0.0, 0.0, 0.0]),
]


@pytest.mark.parametrize("name,c,u", HAND, ids=[h[0] for h in HAND])
def test_hand_built_rows_follow_the_rules(ops, name, c, u):
    n, lo, s = len(c), 2, 3.0
    logits = torch.full((2, lo + n + 1), 100.0)                              # out-of-range ids are never selected
    logits[0, lo:lo + n] = torch.tensor(c)
    logits[1, lo:lo + n] = torch.tensor(u)
    logits = logits.to(DEV)
    x = guided_x(logits, 1, lo, lo + n, s, 1.0)
    noise = torch.empty(1, n, device=DEV).uniform_(1e-9, 1.0, generator=torch.Generator(device=DEV).manual_seed(1))
    tokens = torch.empty(2, 1, dtype=torch.int32, device=DEV)
    for k, p in ((0, 1.0), (2, 1.0), (0, 0.5)):
        mask = keep_mask(x.astype(np.float64), k, p)
        for u_ in (None, noise):
            ops.sample_rows_guided(logits, u_, tokens, lo, lo + n, 1.0, s, k, p)
            got = tokens[:, 0].cpu().tolist()
            assert got[0] == got[1]
            if not mask.any():
                assert got[0] == lo, (name, k, p)                           # no usable id: the first allowed id
            elif u_ is None:
                assert got[0] == lo + int(first_argmax(x, mask)[0]), (name, k, p)
            else:
                assert mask[0, got[0] - lo] and not np.isnan(x[0, got[0] - lo]), (name, k, p)


def test_invalid_arguments_raise(ops):
    from dalle_mtf_b200 import lib as L
    logits = torch.randn(4, 64, device=DEV)
    tokens = torch.zeros(4, 1, dtype=torch.int32, device=DEV)
    kept = torch.empty(2, dtype=torch.int32, device=DEV)
    good = dict(inv_temp=1.0, guidance_scale=3.0, top_k=4, top_p=0.9)
    bad = [dict(guidance_scale=-0.1), dict(guidance_scale=math.nan), dict(guidance_scale=math.inf),
           dict(top_k=-1), dict(top_p=0.0), dict(top_p=1.5), dict(top_p=math.nan), dict(inv_temp=0.0),
           dict(inv_temp=-1.0, top_k=0, top_p=1.0), dict(guidance_scale=-1.0, top_k=0, top_p=1.0)]
    for b in bad:
        a = {**good, **b}
        with pytest.raises(L.DB200Error):
            ops.sample_rows_guided(logits, None, tokens, 0, 64, a["inv_temp"], a["guidance_scale"], a["top_k"],
                                   a["top_p"])
    with pytest.raises(L.DB200Error):
        ops.sample_rows_guided(logits, None, tokens, 10, 10, 1.0, 3.0)                     # empty range
    with pytest.raises(L.DB200Error):
        ops.sample_rows_guided(logits, None, tokens, 0, 64, 1.0, 3.0, kept=kept)           # kept needs a filter
    with pytest.raises(L.DB200Error):
        ops.sample_rows_guided(logits[:3], None, tokens[:3], 0, 64, 1.0, 3.0)              # odd row count
    lib, s = L.load(), torch.cuda.current_stream().cuda_stream
    assert lib.db200_sample_rows_guided(s, logits.data_ptr(), 64, None, tokens.data_ptr(), 0, None, 2, 0, 64, 1.0,
                                        3.0, 0, 1.0, None) != 0                             # ld_tokens 0
    assert lib.db200_sample_rows_guided(s, None, 64, None, tokens.data_ptr(), 1, None, 2, 0, 64, 1.0, 3.0, 0, 1.0,
                                        None) != 0                                          # null logits
    wide = torch.randn(2, 51201, device=DEV)
    with pytest.raises(L.DB200Error):
        ops.sample_rows_guided(wide, None, torch.zeros(2, 1, dtype=torch.int32, device=DEV), 0, 51201, 1.0, 3.0, 8)


# ------------------------------------------------------------------------------------------------ decoder
def reference_guided_greedy(eng, text, s, pad):
    """Guided greedy decoding by hand: DalleSampler.step on the 2B rows, logits combined with torch float32 ops, first
    maximum over the image range."""
    from dalle_mtf_b200.sampling import DalleSampler
    tv, iv, TL, S = eng.text_vocab_size, eng.image_vocab_size, eng.text_seq_len, eng.S
    B = text.shape[0]
    smp = DalleSampler(eng)
    smp._alloc(2 * B)
    toks = torch.zeros(2 * B, S, dtype=torch.int32, device=DEV)
    toks[:B, :TL] = text
    toks[B:, :TL] = pad
    st = torch.tensor(s, dtype=torch.float32, device=DEV)
    for pos in range(S - 1):
        logits = smp.step(toks[:, pos].contiguous(), pos)
        if pos + 1 < TL:
            continue
        c, u = logits[:B, tv:tv + iv], logits[B:, tv:tv + iv]
        g = u + st * (c - u)
        nxt = (g.argmax(-1) + tv).to(torch.int32)
        toks[:B, pos + 1] = nxt
        toks[B:, pos + 1] = nxt
    return toks[:B]


def test_guided_generate_matches_the_step_by_step_reference():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text = sharp_engine()
    smp = DalleSampler(eng)
    for s in (0.0, 3.0, 7.5):
        want = reference_guided_greedy(eng, text, s, eng.text_vocab_size - 1)
        eager = smp.generate(text, temperature=0, guidance_scale=s)
        assert torch.equal(eager, want), s
        graphed = smp.generate_graphed(text, temperature=0, guidance_scale=s)
        assert torch.equal(graphed, eager), s
    # guidance changes the result, and a different padding id changes the unconditional rows
    plain = smp.generate(text, temperature=0)
    assert not torch.equal(plain, smp.generate(text, temperature=0, guidance_scale=7.5))
    other = DalleSampler(eng, padding_id=5)
    assert torch.equal(other.generate(text, temperature=0, guidance_scale=3.0),
                       reference_guided_greedy(eng, text, 3.0, 5))
    # return_logits: all 2B rows of each step, conditional first
    out, lg = smp.generate(text, temperature=0, guidance_scale=3.0, return_logits=True)
    assert out.shape == (3, eng.S) and lg[0].shape == (6, eng.V)
    # seeded noise with a filter is reproducible, within the image range, and the graphed path runs it too
    g = torch.Generator(device=DEV)
    a = smp.generate(text, temperature=1.0, generator=g.manual_seed(3), top_k=8, top_p=0.9, guidance_scale=3.0)
    b = smp.generate(text, temperature=1.0, generator=g.manual_seed(3), top_k=8, top_p=0.9, guidance_scale=3.0)
    assert torch.equal(a, b)
    tv, iv, ts = eng.text_vocab_size, eng.image_vocab_size, eng.text_seq_len
    c = smp.generate_graphed(text, temperature=1.0, top_k=8, guidance_scale=3.0)
    for t in (a, c):
        assert torch.equal(t[:, :ts], text) and ((t[:, ts:] >= tv) & (t[:, ts:] < tv + iv)).all()
    for bad in (-1.0, math.nan, math.inf):
        for fn in (smp.generate, smp.generate_graphed, smp.complete):
            with pytest.raises(ValueError):
                fn(text, guidance_scale=bad)


def test_scale_none_and_one_run_the_plain_path():
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text = sharp_engine()
    B = text.shape[0]
    smp = DalleSampler(eng)
    for name, kw in (("generate", dict(temperature=0)), ("generate_graphed", dict(temperature=0)),
                     ("complete", dict(temperature=1.0, top_k=8))):
        fn = getattr(smp, name)
        results, launches = [], []
        for extra in ({}, {"guidance_scale": None}, {"guidance_scale": 1.0}, {"guidance_scale": 1}):
            fn(text, **kw, **extra)                                 # capture / warm-up
            torch.manual_seed(4)
            n0 = L.launch_count()
            results.append(fn(text, **kw, **extra))
            launches.append(L.launch_count() - n0)
            assert smp._B == B and smp.kc[0].shape[0] == B, (name, extra)        # no 2B-row buffers
            if name != "generate":
                assert smp.tokens.shape[0] == B and smp._graph_key[-1] is None
        assert all(torch.equal(r, results[0]) for r in results), name
        assert len(set(launches)) == 1, (name, launches)


def test_guided_complete_is_seeded_whether_or_not_it_captured():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text = sharp_engine()
    iv = eng.image_vocab_size
    prefix = torch.randint(0, iv, (3, 6), generator=torch.Generator().manual_seed(2)).to(torch.int32).cuda()
    kw = dict(samples_per_prompt=2, temperature=1.0, top_p=0.95, guidance_scale=3.0)
    fresh = DalleSampler(eng)
    torch.manual_seed(9)
    a = fresh.complete(text, prefix, **kw)                           # captures inside the call
    warm = DalleSampler(eng)
    warm.complete(text, prefix, **kw)
    torch.manual_seed(9)
    b = warm.complete(text, prefix, **kw)                            # replays the graphs captured before
    assert torch.equal(a, b)
    assert a.shape == (6, eng.S)
    ts = eng.text_seq_len
    assert torch.equal(a[:, :ts], text.repeat_interleave(2, 0))
    assert torch.equal(a[:, ts:ts + 6], prefix.repeat_interleave(2, 0) + eng.text_vocab_size)


# ------------------------------------------------------------------------------------------------ prefill
def test_guided_complete_first_token_is_the_oracle_on_two_separate_prefills():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text = sharp_engine()
    tv, iv, ts, S = eng.text_vocab_size, eng.image_vocab_size, eng.text_seq_len, eng.S
    B, n, pad = text.shape[0], 5, 17
    prefix = torch.randint(0, iv, (B, n), generator=torch.Generator().manual_seed(6)).to(torch.int32).cuda()
    cond = torch.cat([text, prefix + tv], 1)
    unc = cond.clone()
    unc[:, :ts] = pad
    caches = lambda: ([torch.zeros(B, S, eng.H, eng.dh, dtype=torch.bfloat16, device=DEV) for _ in range(eng.L)],
                      [torch.zeros(B, S, eng.H, eng.dh, dtype=torch.bfloat16, device=DEV) for _ in range(eng.L)])
    lc = eng.prefill(cond, *caches())[:, tv:tv + iv].clone()
    lu = eng.prefill(unc, *caches())[:, tv:tv + iv].clone()
    smp = DalleSampler(eng, padding_id=pad)
    for s in (0.0, 3.0, 7.5):
        x = guided_logits(lc.cpu().numpy(), lu.cpu().numpy(), s)
        want = torch.from_numpy(np.argmax(x, -1) + tv).to(torch.int32)
        out = smp.complete(text, prefix, temperature=0, guidance_scale=s)
        assert torch.equal(out[:, ts + n].cpu(), want), s
        # replicas of a greedy guided completion are identical
        many = smp.complete(text, prefix, samples_per_prompt=3, temperature=0, guidance_scale=s)
        assert torch.equal(many, out.repeat_interleave(3, 0)), s


def test_dalle_class_passes_guidance_and_padding_id_through():
    from dalle_mtf_b200.models import DALLE
    from dalle_mtf_b200.sampling import DalleSampler
    kw = dict(text_vocab_size=200, image_vocab_size=32, text_seq_len=8, image_seq_len=16, n_layers=1, n_heads=2)
    text = torch.randint(0, 200, (2, 8), dtype=torch.int32)
    m = DALLE(256, params={"padding_id": 150}, **kw)
    got = m.sample(text, temperature=0.0, guidance_scale=3.0)
    assert m._sampler.padding_id == 150
    assert torch.equal(got, DalleSampler(m.engine, padding_id=150).generate(text.cuda(), 0.0, guidance_scale=3.0))
    out = m.complete(text, samples_per_prompt=2, temperature=0.0, guidance_scale=3.0)
    assert out.shape == (4, 24) and ((out[:, 8:] >= 200) & (out[:, 8:] < 232)).all()
    assert DALLE(256, **kw)._get_sampler().padding_id == 199                 # default: text_vocab_size - 1
    with pytest.raises(ValueError):
        m.sample(text, guidance_scale=-2.0)


# ------------------------------------------------------------------------------------------------ training
def test_assemble_tokens_caption_drop_matches_the_oracle(ops):
    from dalle_mtf_b200 import lib as L
    g = torch.Generator().manual_seed(0)
    B, Tt, Ti, tv, pad = 300, 12, 20, 500, 499
    text = torch.randint(0, pad, (B, Tt), generator=g).to(torch.int32)
    img = torch.randint(0, 64, (B, Ti), generator=g).to(torch.int32)
    out = torch.empty(B, Tt + Ti, dtype=torch.int32, device=DEV)
    for rate, seed, step, row0 in ((0.5, 5, 0, 0), (0.1, 2 ** 40 + 3, 17, 1000), (0.9, 7, 3, 2 ** 33 + 1)):
        drop = L.make_dropout(rate, seed, step, L.SITE_CAPTION, row0)
        ops.assemble_tokens(text.to(DEV), img.to(DEV), out, tv, caption_drop=drop, pad_id=pad)
        dropped = torch.from_numpy(CG.caption_dropped(rate, seed, step, B, row0))
        want = torch.cat([text, img + tv], 1)
        want[dropped, :Tt] = pad
        assert torch.equal(out.cpu(), want), (rate, seed, step, row0)
        assert 0 < int(dropped.sum()) < B
    # no drop descriptor, or rate 0: the plain assembly
    ops.assemble_tokens(text.to(DEV), img.to(DEV), out, tv, caption_drop=None, pad_id=pad)
    assert torch.equal(out.cpu(), torch.cat([text, img + tv], 1))
    assert L.make_dropout(0.0, 5, 0, L.SITE_CAPTION, 0) is None
    lib, s = L.load(), torch.cuda.current_stream().cuda_stream
    bad = L.make_dropout(0.5, 5, 0, L.SITE_CAPTION, 0)
    assert lib.db200_assemble_tokens_ex(s, text.to(DEV).data_ptr(), img.to(DEV).data_ptr(), out.data_ptr(), B, Tt, Ti,
                                        tv, -1, ctypes.byref(bad)) != 0                     # negative pad id


def _host_dropped(cap, rate, seed, step, pad, row0=0):
    cap = cap.clone()
    cap[torch.from_numpy(CG.caption_dropped(rate, seed, step, cap.shape[0], row0))] = pad
    return cap


def test_model_fn_caption_dropout_equals_host_padded_captions(tmp_path, monkeypatch):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from test_dropout_gpu import _batch, _tiny_dalle_params
    img, cap = _batch()
    pad, seed, rate = 299, 5, 0.5
    steps = 3
    dropped = [CG.caption_dropped(rate, seed, i, 4) for i in range(steps)]
    assert any(d.any() for d in dropped) and any((~d).any() for d in dropped)
    for mb in (None, 2 * 28):                     # the drops are drawn before micro-batching: the same either way
        extra = {"tokens_per_mb_per_replica": mb} if mb else {}
        dev = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, caption_dropout=rate, padding_id=pad,
                                                                   **extra))
        host = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, padding_id=pad, **extra))
        for i in range(steps):
            a = dev.train_op(img, cap).clone()
            b = host.train_op(img, _host_dropped(cap, rate, seed, i, pad)).clone()
            assert torch.equal(a, b), (mb, i)
        torch.cuda.synchronize()
        assert torch.equal(dev.engine.master, host.engine.master), mb
    # eval_op never drops
    ev = dalle_model_fn(img, cap, "eval", _tiny_dalle_params(tmp_path, caption_dropout=rate, padding_id=pad))
    ev0 = dalle_model_fn(img, cap, "eval", _tiny_dalle_params(tmp_path))
    assert torch.equal(ev.eval_op(img, cap).clone(), ev0.eval_op(img, cap).clone())
    # rate 0 (or no key): the plain assembly kernel, the same launches
    calls = []
    orig = O.assemble_tokens

    def spy(*a, **kw):
        calls.append(kw.get("caption_drop"))
        return orig(*a, **kw)
    monkeypatch.setattr(O, "assemble_tokens", spy)
    counts = []
    for extra in ({}, {"caption_dropout": 0.0}, {"caption_dropout": None, "padding_id": pad}):
        spec = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, **extra))
        spec.train_op(img, cap)
        torch.cuda.synchronize()
        n0 = L.launch_count()
        spec.train_op(img, cap)
        counts.append(L.launch_count() - n0)
    assert calls and all(c is None for c in calls)
    assert len(set(counts)) == 1, counts
