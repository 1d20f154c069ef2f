"""GPU tests of top-k / nucleus (top-p) filtered sampling: db200_sample_rows_filtered(_at) against the float64
statement in oracle/sampling.py, and the sampler options built on it (DalleSampler.generate / generate_graphed
top_k, top_p; DALLE.sample)."""
import math

import numpy as np
import pytest
import torch

from oracle.sampling import boundary_margin, keep_mask
from test_sampling_filter_cpu import ADVERSARIAL

pytestmark = pytest.mark.gpu

DEV = "cuda"
MARGIN = 1e-5      # rows whose top-p decision lies closer than this (relative to Z) to a tie are not compared


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import ops as o
    return o


def scaled(logits, inv_temp):
    """x = logits * inv_temp in fp32, as the kernels compute it (on the device, then widened to float64)."""
    return (logits * torch.tensor(inv_temp, dtype=torch.float32, device=logits.device)).double().cpu().numpy()


def perturbed(logits, u, inv_temp):
    """The fp32 Gumbel-perturbed values x + (-log(-log u)) the kernels maximise, on the device."""
    x = logits * torch.tensor(inv_temp, dtype=torch.float32, device=logits.device)
    return x + -torch.log(-torch.log(u)) if u is not None else x


def check_selection(idx, lo, mask, pert, rows_ok):
    """idx (host, minus lo) is in the kept set and is the first argmax of pert over it; pert is computed by torch, which
    may differ from the kernel's logf in the last bit, so a different index must tie to 1e-6.  Returns the number of
    rows where the index is exactly torch's."""
    got = idx - lo
    m = torch.from_numpy(mask)
    p = pert.cpu().masked_fill(~m, -math.inf)
    want = p.argmax(-1)
    r = torch.from_numpy(np.nonzero(rows_ok)[0])
    assert m[r, got[r]].all(), "sampled an id outside the kept set"
    pg, pw = p[r, got[r]], p[r, want[r]]
    assert ((pg - pw).abs() <= 1e-6 * (1 + pw.abs())).all()
    return int((got[r] == want[r]).sum())


@pytest.mark.parametrize("rows,n", [(1, 512), (32, 512), (130, 512), (1, 8192), (32, 8192), (130, 8192),
                                    (1, 32768), (32, 32768), (130, 32768)])
def test_kept_set_and_selection_match_the_float64_oracle(ops, rows, n):
    check_filtered_rows(ops, rows, n)


def check_filtered_rows(ops, rows, n):
    """sample_rows_filtered over n ids at lo = 5 of rows with ld = lo + n + 3, at three temperatures and a grid of
    top_k / top_p: the kept counts equal the oracle's and every draw is the first Gumbel-max of the kept set, except on
    rows whose top-p decision lies within MARGIN of a tie (at most a quarter of them)."""
    g = torch.Generator(device=DEV).manual_seed(rows * 7 + n)
    lo = 5
    hi, ld = lo + n, lo + n + 3
    # row scales log-uniform in [2.5, 10]: from broad to sharply peaked distributions
    scale = torch.exp(torch.empty(rows, 1, device=DEV).uniform_(math.log(2.5), math.log(10.0), generator=g))
    logits = torch.randn(rows, ld, device=DEV, generator=g) * scale
    u = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    idx = torch.empty(rows, dtype=torch.int32, device=DEV)
    kept = torch.empty(rows, dtype=torch.int32, device=DEV)
    total = near = exact = 0
    for inv_temp in (0.7, 1.0, 1.5):
        x = scaled(logits[:, lo:hi], inv_temp)
        pert = perturbed(logits[:, lo:hi], u, inv_temp)
        for k in (0, 1, 50, n - 1):
            for p in (0.5, 0.9, 0.999, 1.0):
                pf = float(np.float32(p))                        # the kernel compares against the fp32 top_p
                mask = keep_mask(x, k, pf)
                ok = boundary_margin(x, k, pf) > MARGIN
                ops.sample_rows_filtered(logits, u, idx, lo, hi, inv_temp, k, p, kept=kept)
                kc = kept.cpu().numpy()
                assert np.array_equal(kc[ok], mask.sum(-1)[ok]), (inv_temp, k, p)
                exact += check_selection(idx.cpu().long(), lo, mask, pert, ok)
                total += rows
                near += int((~ok).sum())
    print(f"rows={rows} n={n}: {near} of {total} row decisions within {MARGIN} of a top-p tie (not compared)")
    # near ties come mostly from p = 0.999 on the broader rows, where each id around the cut carries < 1e-5 of Z
    # (11-17 % of the decisions at n >= 8192)
    assert near <= 0.25 * total
    assert exact >= 0.999 * (total - near)


@pytest.mark.parametrize("name,x,k,p,want", ADVERSARIAL, ids=[a[0] for a in ADVERSARIAL])
def test_hand_built_rows_match_the_oracle_exactly(ops, name, x, k, p, want):
    n = len(x)
    lo = 3
    logits = torch.full((2, lo + n + 2), 50.0)                       # out-of-range ids are large: never selected
    logits[:, lo:lo + n] = torch.tensor(x, dtype=torch.float32)
    logits = logits.to(DEV)
    mask = keep_mask(np.array(x), k, p)
    assert mask.tolist() == [bool(v) for v in want]
    idx = torch.empty(2, dtype=torch.int32, device=DEV)
    kept = torch.empty(2, dtype=torch.int32, device=DEV)
    u = torch.empty(2, n, device=DEV).uniform_(1e-9, 1.0, generator=torch.Generator(device=DEV).manual_seed(n))
    for noise in (None, u):
        ops.sample_rows_filtered(logits, noise, idx, lo, lo + n, 1.0, k, p, kept=kept)
        got, kc = idx.cpu().tolist(), kept.cpu().tolist()
        assert kc == [int(mask.sum())] * 2, name
        for i in got:
            if mask.any():
                assert mask[i - lo], (name, i)
            else:
                assert i == lo, (name, i)                                  # no finite entry: the first allowed id
        if noise is None and mask.any():
            xs = np.where(mask, np.array(x), -np.inf)
            assert got == [lo + int(np.argmax(xs))] * 2                     # greedy: first maximum of the kept set


def test_filter_off_equals_sample_rows(ops):
    g = torch.Generator(device=DEV).manual_seed(11)
    rows, lo, n = 64, 17, 1000
    hi, ld = lo + n, lo + n + 9
    logits = torch.randn(rows, ld, device=DEV, generator=g) * 3
    logits[:, lo + 100] = logits[:, lo + 900] = 9.0                   # ties of the maximum
    logits[::3, lo + 40] = -0.0
    logits[::5, lo + 41] = float("nan")
    logits[::7, lo + 42] = float("-inf")
    logits[3, lo:hi] = torch.round(logits[3, lo:hi])                  # a row full of ties
    u = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    a = torch.empty(rows, dtype=torch.int32, device=DEV)
    b = torch.empty_like(a)
    for noise in (None, u):
        for inv_temp in (0.5, 1.0):
            ops.sample_rows(logits, noise, a, lo, hi, inv_temp)
            for k in (0, n, n + 5):
                ops.sample_rows_filtered(logits, noise, b, lo, hi, inv_temp, k, 1.0)
                assert torch.equal(a, b), (noise is None, inv_temp, k)
    # top_k = 1 on tie-free rows is greedy whatever the noise
    tie_free = torch.randn(rows, ld, device=DEV, generator=g)
    ops.sample_rows(tie_free, None, a, lo, hi, 1.0)
    for p in (1.0, 0.3):
        ops.sample_rows_filtered(tie_free, u, b, lo, hi, 1.0, 1, p)
        assert torch.equal(a, b)


@pytest.mark.parametrize("k,p", [(3, 1.0), (0, 0.8), (5, 0.9)])
def test_sampling_distribution_is_the_renormalised_filtered_softmax(ops, k, p):
    n, K = 20000, 8
    lg = torch.tensor([0.0, 1.0, 2.0, -1.0, 0.5, 3.0, -2.0, 1.5])
    big = lg.repeat(n, 1).to(DEV)
    uu = torch.empty(n, K, device=DEV).uniform_(1e-9, 1.0, generator=torch.Generator(device=DEV).manual_seed(3))
    out = torch.empty(n, dtype=torch.int32, device=DEV)
    kept = torch.empty(n, dtype=torch.int32, device=DEV)
    ops.sample_rows_filtered(big, uu, out, 0, K, 1.0, k, p, kept=kept)
    mask = torch.from_numpy(keep_mask(lg.double().numpy(), k, p))
    assert (kept.cpu() == int(mask.sum())).all()
    freq = torch.bincount(out.cpu().long(), minlength=K).double() / n
    want = torch.softmax(lg.double().masked_fill(~mask, -math.inf), 0)
    assert (freq - want).abs().max() < 0.02                          # sigma <= 0.0035 at n = 20000
    assert (freq[~mask] == 0).all()


def test_repeated_launches_are_identical_and_the_device_position_variant_writes_one_column(ops):
    g = torch.Generator(device=DEV).manual_seed(4)
    rows, lo, n, S = 32, 100, 32768, 40
    logits = torch.randn(rows, lo + n, device=DEV, generator=g) * 2
    u = torch.empty(rows, n, device=DEV).uniform_(1e-9, 1.0, generator=g)
    for k, p in ((0, 0.9), (64, 0.95), (500, 1.0)):
        i1, i2 = (torch.empty(rows, dtype=torch.int32, device=DEV) for _ in range(2))
        k1, k2 = (torch.empty(rows, dtype=torch.int32, device=DEV) for _ in range(2))
        ops.sample_rows_filtered(logits, u, i1, lo, lo + n, 1.3, k, p, kept=k1)
        ops.sample_rows_filtered(logits, u, i2, lo, lo + n, 1.3, k, p, kept=k2)
        assert torch.equal(i1, i2) and torch.equal(k1, k2)
        tokens = torch.full((rows, S), -7, dtype=torch.int32, device=DEV)
        pos = torch.tensor([17], dtype=torch.int32, device=DEV)
        k3 = torch.empty(rows, dtype=torch.int32, device=DEV)
        ops.sample_rows_filtered_at(logits, u, tokens, lo, lo + n, 1.3, k, p, pos, kept=k3)
        want = torch.full_like(tokens, -7)
        want[:, 18] = i1
        assert torch.equal(tokens, want) and torch.equal(k3, k1)


def test_invalid_arguments_raise(ops):
    from dalle_mtf_b200.lib import DB200Error
    logits = torch.randn(2, 64, device=DEV)
    idx = torch.empty(2, dtype=torch.int32, device=DEV)
    good = dict(inv_temp=1.0, top_k=4, top_p=0.9)
    bad = [dict(top_k=-1), dict(top_p=float("nan")), dict(top_p=0.0), dict(top_p=-0.5), dict(top_p=1.5),
           dict(inv_temp=0.0), dict(inv_temp=-1.0)]
    for b in bad:
        a = {**good, **b}
        with pytest.raises(DB200Error):
            ops.sample_rows_filtered(logits, None, idx, 0, 64, a["inv_temp"], a["top_k"], a["top_p"])
    with pytest.raises(DB200Error):
        ops.sample_rows_filtered(logits, None, idx, 10, 10, 1.0, 4, 0.9)              # empty range
    tokens = torch.zeros(2, 8, dtype=torch.int32, device=DEV)
    pos = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(DB200Error):
        ops.sample_rows_filtered_at(logits, None, tokens, 0, 64, 1.0, -3, 0.9, pos)
    wide = torch.randn(1, 51201, device=DEV)                            # one id more than a CTA holds
    one = torch.empty(1, dtype=torch.int32, device=DEV)
    with pytest.raises(DB200Error):
        ops.sample_rows_filtered(wide, None, one, 0, 51201, 1.0, 8, 0.9)
    ops.sample_rows_filtered(wide, None, one, 1, 51201, 1.0, 8, 0.9)    # 51 200 ids: supported
    assert one.item() == int(wide[0, 1:].argmax()) + 1


def sharp_engine(d=256, L=2, H=2, tv=300, iv=64, ts=24, isl=40):
    """The small engine of test_sampling_gpu.py's cached-decoding test, with sharpened weights."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, L, H, tv, iv, ts, isl)
    eng.load_params(params)
    text = torch.randint(0, tv, (3, ts), generator=g).to(torch.int32).cuda()
    return eng, text


def test_sampler_top_k_and_top_p():
    from dalle_mtf_b200.sampling import DalleSampler
    eng, text = sharp_engine()
    tv, iv, ts = eng.text_vocab_size, eng.image_vocab_size, eng.text_seq_len
    smp = DalleSampler(eng)
    greedy = smp.generate(text, temperature=0)
    g = torch.Generator(device=DEV).manual_seed(5)
    assert torch.equal(smp.generate(text, temperature=1.0, generator=g, top_k=1), greedy)
    assert torch.equal(smp.generate_graphed(text, temperature=1.0, top_k=1), greedy)
    # every sampled token lies in the kept set of the logits it was drawn from
    g.manual_seed(6)
    toks, step_logits = smp.generate(text, temperature=1.0, generator=g, top_k=8, top_p=0.9, return_logits=True)
    checked = 0
    for pos in range(ts - 1, eng.S - 1):
        x = step_logits[pos][:, tv:tv + iv].double().cpu().numpy()
        mask = keep_mask(x, 8, float(np.float32(0.9)))
        ok = boundary_margin(x, 8, float(np.float32(0.9))) > MARGIN
        tok = toks[:, pos + 1].cpu().numpy() - tv
        assert ((0 <= tok) & (tok < iv)).all()
        assert mask[np.arange(len(tok)), tok][ok].all(), pos
        checked += int(ok.sum())
    assert checked >= 0.9 * 3 * (eng.S - ts)
    g.manual_seed(6)
    assert torch.equal(smp.generate(text, temperature=1.0, generator=g, top_k=8, top_p=0.9), toks)
    # changing the filter re-captures the graphed step
    a = smp.generate_graphed(text, temperature=1.0, top_k=8)
    key_k = smp._graph_key
    b = smp.generate_graphed(text, temperature=1.0, top_p=0.9)
    assert smp._graph_key != key_k
    for t in (a, b):
        assert torch.equal(t[:, :ts], text) and ((t[:, ts:] >= tv) & (t[:, ts:] < tv + iv)).all()
    # no active filter keeps the unfiltered kernels (and graphs): top_k >= image vocabulary and top_p = 1 are off
    smp.generate_graphed(text, temperature=0.0)
    key_off = smp._graph_key
    assert torch.equal(smp.generate_graphed(text, temperature=0.0, top_k=iv, top_p=1.0), greedy)
    assert smp._graph_key == key_off
    for bad in (dict(top_k=0), dict(top_k=-2), dict(top_k=2.5), dict(top_p=0.0), dict(top_p=1.01),
                dict(top_p=float("nan"))):
        with pytest.raises(ValueError):
            smp.generate(text, **bad)
        with pytest.raises(ValueError):
            smp.generate_graphed(text, **bad)


def test_dalle_sample_passes_the_filter_through():
    from dalle_mtf_b200.models import DALLE
    m = DALLE(256, text_vocab_size=200, image_vocab_size=32, text_seq_len=8, image_seq_len=16, n_layers=1, n_heads=2)
    text = torch.randint(0, 200, (2, 8), dtype=torch.int32)
    greedy = m.sample(text, temperature=0.0)
    out = m.sample(text, temperature=1.0, generator=torch.Generator(device=DEV).manual_seed(1), top_k=1)
    assert torch.equal(out, greedy)
    out = m.sample(text, temperature=1.0, top_k=5, top_p=0.8)
    assert out.shape == (2, 24) and (out[:, 8:] >= 200).all() and (out[:, 8:] < 232).all()
    for bad in (dict(top_k=0), dict(top_p=0.0), dict(top_p=2.0)):
        with pytest.raises(ValueError):
            m.sample(text, **bad)
