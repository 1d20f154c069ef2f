"""CPU tests of the dropout masks (oracle/philox.py), of the oracle under dropout and of the host-side key parsing."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import dalle as O
from oracle import dalle_dropout as D
from oracle import philox as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_philox_known_answer_vectors():
    """Random123's kat_vectors for philox4x32_10 (the toolkit's curand_Philox4x32_10 computes the same rounds)."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = tuple(int(w) for w in X.philox4x32_10(*ctr, *key))
        assert got == want, [hex(w) for w in got]


def _binomial_ok(keep, rate):
    n = keep.size
    p = 1.0 - rate
    return abs(keep.mean() - p) <= 6 * math.sqrt(p * (1 - p) / n)


@pytest.mark.parametrize("rate", [0.1, 0.5])
def test_kept_fraction_is_within_binomial_bounds(rate):
    assert _binomial_ok(X.keep_elementwise(rate, 7, 3, 5, 300, 256, row0=11), rate)
    assert _binomial_ok(X.keep_attention(rate, 7, 3, 2, 3, 4, 97, row0=2), rate)
    # different sites, steps and seeds draw different masks
    a = X.keep_elementwise(rate, 7, 3, 5, 64, 64)
    for other in (X.keep_elementwise(rate, 7, 3, 6, 64, 64), X.keep_elementwise(rate, 7, 4, 5, 64, 64),
                  X.keep_elementwise(rate, 8, 3, 5, 64, 64)):
        assert (a != other).mean() > 0.05


def test_rate_zero_keeps_everything_and_threshold_rule():
    assert X.keep_elementwise(0.0, 1, 2, 3, 8, 16).all()
    assert X.threshold_scale(0.1) == (429496729, float(np.float32(1 / 0.9)))
    assert X.threshold_scale(0.5)[0] == 2 ** 31
    for bad in (-0.1, 1.0, 1.5):
        with pytest.raises(ValueError):
            X.threshold_scale(bad)


def test_row_slices_equal_the_full_batch_masks():
    """Rows [r0, r0 + n) drawn on their own (one rank or micro-batch) equal that slice of the full-batch masks."""
    S, d, B, H = 13, 32, 6, 2
    full = X.keep_elementwise(0.3, 5, 9, 4, B * S, d)
    att = X.keep_attention(0.3, 5, 9, 2, B, H, S)
    for r0, n in ((0, 2), (2, 3), (5, 1)):
        assert np.array_equal(X.keep_elementwise(0.3, 5, 9, 4, n * S, d, row0=r0 * S), full[r0 * S:(r0 + n) * S])
        assert np.array_equal(X.keep_attention(0.3, 5, 9, 2, n, H, S, row0=r0), att[r0:r0 + n])


def test_attention_layout_uses_two_by_two_blocks():
    """(i, j), (i, j^1), (i^1, j), (i^1, j^1) read the four words of one Philox call."""
    seed, step, site, H, S = 3, 1, 2, 2, 9
    b, h, i, j = 1, 1, 4, 6
    S2 = (S + 1) // 2
    n = ((b * H + h) * S2 + i // 2) * S2 + j // 2
    words = [int(w) for w in X.philox4x32_10(n & 0xFFFFFFFF, n >> 32, site, step, seed, 0)]
    rate = 0.5
    keep = X.keep_attention(rate, seed, step, site, b + 1, H, S)
    for di in (0, 1):
        for dj in (0, 1):
            assert keep[b, h, i + di, j + dj] == (words[2 * di + dj] >= 2 ** 31)


def test_wpe_mask_is_shared_by_the_batch():
    cfg = O.DalleConfig(32, 1, 2, 20, 8, 5, 4)
    dm = D.dropout_masks(((0.2, 0.0, 0.0), 1, 0, 0), 3, cfg)
    assert tuple(dm["wpe"].shape) == (cfg.seq_len, cfg.n_embd)
    assert tuple(dm["wte"].shape) == (3, cfg.seq_len, cfg.n_embd)
    assert not torch.equal(dm["wte"][0], dm["wte"][1])      # wte: i.i.d. over the full [B, S, d] shape


def _case():
    cfg = O.DalleConfig(32, 2, 2, 20, 8, 5, 4)
    p = O.init_params(cfg, 1)
    t = torch.randint(0, cfg.total_tokens - 1, (3, cfg.seq_len), generator=torch.Generator().manual_seed(1))
    return cfg, p, t


def test_rates_zero_give_the_oracle_without_dropout():
    cfg, p, t = _case()
    for bf16 in (False, True):
        l0, lb0, lg0, g0 = O.loss_and_grads(p, t, cfg, bf16=bf16)
        l1, lb1, lg1, g1 = D.loss_and_grads(p, t, cfg, ((0.0, 0.0, 0.0), 5, 3, 0), bf16=bf16)
        assert torch.equal(l0, l1) and torch.equal(lb0, lb1) and torch.equal(lg0, lg1)
        for k in g0:
            assert torch.equal(g0[k], g1[k]), k


def test_dropout_changes_the_loss_and_depends_on_step_and_seed():
    cfg, p, t = _case()
    l0 = O.forward(p, t, cfg)[0]
    la = D.forward(p, t, cfg, ((0.1, 0.2, 0.15), 5, 3, 0))[0]
    lb = D.forward(p, t, cfg, ((0.1, 0.2, 0.15), 5, 4, 0))[0]
    lc = D.forward(p, t, cfg, ((0.1, 0.2, 0.15), 6, 3, 0))[0]
    assert la != l0 and la != lb and la != lc
    assert torch.equal(la, D.forward(p, t, cfg, ((0.1, 0.2, 0.15), 5, 3, 0))[0])


def test_oracle_row0_equals_the_matching_slice_of_the_batch():
    """Per-token losses of sequences [1, 3) run alone with row0 = 1 equal those rows of the full-batch run."""
    cfg, p, t = _case()
    spec = lambda r0: ((0.1, 0.2, 0.15), 5, 3, r0)
    full = D.forward(p, t, cfg, spec(0))[1]
    part = D.forward(p, t[1:3], cfg, spec(1))[1]
    assert torch.allclose(part, full[1:3], rtol=1e-5, atol=1e-6)


def test_autograd_matches_finite_differences_with_dropout():
    cfg = O.DalleConfig(16, 1, 2, 10, 5, 3, 2)
    p = {k: v.double() for k, v in O.init_params(cfg, 3).items()}
    t = torch.randint(0, cfg.total_tokens - 1, (2, cfg.seq_len), generator=torch.Generator().manual_seed(3))
    spec = ((0.3, 0.3, 0.3), 11, 2, 0)
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    D.forward(leaves, t, cfg, spec)[0].backward()
    for name in ("layer_0/attn/q", "layer_0/attn/v", "layer_0/mlp/mlp_linear_2/kernel", "positional_embedding/wpe",
                 "to_logits/linear_out/bias", "embedding/wte"):
        w = p[name]
        idx = tuple(int(i) for i in torch.tensor(w.shape) // 2)
        if name == "embedding/wte":
            idx = (int(t[0, 0]), 1)
        eps = 1e-5
        wp = {k: v.clone() for k, v in p.items()}
        wm = {k: v.clone() for k, v in p.items()}
        wp[name][idx] += eps
        wm[name][idx] -= eps
        fd = (D.forward(wp, t, cfg, spec)[0] - D.forward(wm, t, cfg, spec)[0]) / (2 * eps)
        assert abs(fd.item() - leaves[name].grad[idx].item()) < 1e-6 * max(1, abs(fd.item())), name


def test_dropout_keys_are_parsed_and_validated():
    from dalle_mtf_b200.model_fns import dropout_rates
    assert dropout_rates({}) == (0.0, 0.0, 0.0)
    assert dropout_rates({"embed_dropout": 0.1, "attention_dropout": None, "residual_dropout": 0.2}) == \
        (0.1, 0.0, 0.2)
    for bad in (-0.1, 1.0, 2):
        with pytest.raises(ValueError):
            dropout_rates({"attention_dropout": bad})


def test_host_descriptors_follow_the_mask_rule():
    from dalle_mtf_b200 import lib as L
    assert L.make_dropout(0.0, 1, 2, 3, 4) is None
    d = L.make_dropout(0.1, 2 ** 40 + 5, 7, L.dropout_site_mlp_out(2), 96)
    assert (d.seed, d.step, d.site, d.row0) == (2 ** 40 + 5, 7, 10, 96)
    assert (d.threshold, d.scale) == X.threshold_scale(0.1)
    assert (L.dropout_site_attn(0), L.dropout_site_attn_out(0), L.SITE_WPE) == (X.site_attn(0), X.site_attn_out(0),
                                                                                  X.SITE_WPE)
    with pytest.raises(ValueError):
        L.make_dropout(1.0, 0, 0, 0, 0)


def test_dropout_struct_mirror_matches_header(tmp_path):
    from dalle_mtf_b200.lib import Dropout
    names = [n for n, _ in Dropout._fields_]
    src = ["#include <stdio.h>", "#include <stddef.h>", '#include "dalle_b200.h"', "int main(void) {",
           '  printf("size %zu\\n", sizeof(db200_dropout));']
    src += [f'  printf("{n} %zu\\n", offsetof(db200_dropout, {n}));' for n in names]
    src += ["  return 0;", "}"]
    c = tmp_path / "dropout_sizes.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "dropout_sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True,
                                                  text=True).stdout.splitlines())
    assert ctypes.sizeof(Dropout) == int(out["size"]) == 32
    for n in names:
        assert getattr(Dropout, n).offset == int(out[n]), n
