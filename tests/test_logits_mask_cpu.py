"""CPU tests of the modality logits mask: the oracle (windowed cross-entropy, its explicit gradient, finite
differences, the two mutants) and the config key.  The kernels are tested in test_logits_mask_gpu.py
(db200_logits_mask_partition, db200_logits_mask_scatter)."""
import pytest
import torch

from oracle import dalle as O
from oracle import logits_mask as OM

F64 = torch.float64


def _case(seed=0, B=2, TL=5, IL=6, off=13, n_image=4):
    """float64 logits [B, S, V] and labels that follow the windows: captions < off, codes < n_image, EOS last."""
    g = torch.Generator().manual_seed(seed)
    V = off + n_image + 1
    S = TL + IL
    logits = torch.randn(B, S, V, generator=g, dtype=F64) * 2
    tokens = torch.cat([torch.randint(0, off, (B, TL), generator=g),
                        torch.randint(0, n_image, (B, IL), generator=g) + off], 1)
    return logits, O.shift_labels(tokens, V - 1), TL, IL, off, V


def _direct_rows(logits, labels, TL, off, z=0.0):
    """Each row's loss from the slice of its window (no -inf anywhere)."""
    rows = torch.empty(labels.shape, dtype=logits.dtype)
    for t in range(logits.shape[1]):
        lo, hi = (0, off) if t < TL - 1 else (off, logits.shape[2])
        w = logits[:, t, lo:hi]
        lse = torch.logsumexp(w, -1)
        rows[:, t] = lse - w.gather(-1, (labels[:, t] - lo)[:, None]).squeeze(-1) + z * lse * lse
    return rows


@pytest.mark.parametrize("weights,z", [(None, 0.0), ((1.0, 7.0), 0.0), ((1.0, 7.0), 1e-2), ((0.0, 1.0), 1e-3)])
def test_windowed_ce_equals_the_ce_of_each_window(weights, z):
    logits, labels, TL, IL, off, V = _case(1)
    loss, rows, parts = OM.masked_loss(logits, labels, TL, IL, off, weights, z)
    direct = _direct_rows(logits, labels, TL, off, z)
    assert torch.allclose(rows, direct, rtol=1e-13, atol=1e-13)
    assert torch.isfinite(loss)
    # the same objective as the full CE of logits set to -inf outside the windows
    ml = logits.clone()
    ml[:, :TL - 1, off:] = -float("inf")
    ml[:, TL - 1:, :off] = -float("inf")
    full = torch.logsumexp(ml, -1) - ml.gather(-1, labels[..., None]).squeeze(-1)
    full = full + z * torch.logsumexp(ml, -1) ** 2
    assert torch.allclose(rows, full, rtol=1e-13, atol=1e-13)
    # and it differs from the unmasked objective
    from oracle import loss_weights as OW
    plain, _, _ = OW.weighted_loss(logits, labels, TL, IL, weights, z)
    assert loss < plain


@pytest.mark.parametrize("weights,z", [(None, 0.0), ((1.0, 7.0), 1e-2)])
def test_autograd_equals_the_explicit_gradient_and_finite_differences(weights, z):
    logits, labels, TL, IL, off, V = _case(2)
    B, S, _ = logits.shape
    x = logits.clone().requires_grad_(True)
    loss, _, _ = OM.masked_loss(x, labels, TL, IL, off, weights, z)
    loss.backward()
    explicit = OM.dlogits(logits.reshape(B * S, V), labels.reshape(-1), TL, IL, off, weights, z).view(B, S, V)
    assert torch.allclose(x.grad, explicit, rtol=1e-12, atol=1e-15)
    # exactly 0 outside the windows
    assert (explicit[:, :TL - 1, off:] == 0).all() and (explicit[:, TL - 1:, :off] == 0).all()
    # central differences on a few entries inside and outside the windows
    h = 1e-6
    for (b, t, v) in ((0, 0, 3), (1, TL - 2, off - 1), (0, TL - 1, off), (1, S - 1, V - 1), (0, S - 2, off + 1),
                      (1, 1, off + 2), (0, TL, 2)):
        e = torch.zeros_like(logits)
        e[b, t, v] = h
        lp, _, _ = OM.masked_loss(logits + e, labels, TL, IL, off, weights, z)
        lm, _, _ = OM.masked_loss(logits - e, labels, TL, IL, off, weights, z)
        fd = (lp - lm).item() / (2 * h)
        assert abs(fd - explicit[b, t, v].item()) <= 1e-7, (b, t, v, fd, explicit[b, t, v].item())


@pytest.mark.parametrize("quirks", [OM.Quirks(text_rows_offset=0), OM.Quirks(eos_in_image_window=False)])
def test_both_mutants_change_the_loss(quirks):
    logits, labels, TL, IL, off, V = _case(3)
    ref, _, _ = OM.masked_loss(logits, labels, TL, IL, off)
    bad, _, _ = OM.masked_loss(logits, labels, TL, IL, off, quirks=quirks)
    assert not torch.isclose(bad, ref), quirks
    B, S, _ = logits.shape
    g_ref = OM.dlogits(logits.reshape(B * S, V), labels.reshape(-1), TL, IL, off)
    g_bad = OM.dlogits(logits.reshape(B * S, V), labels.reshape(-1), TL, IL, off, quirks=quirks)
    assert (g_bad - g_ref).abs().max() > 1e-3


def test_single_text_position_has_no_text_rows():
    """text_seq_len 1: every row is an image row."""
    logits, labels, _, _, off, V = _case(4, TL=1, IL=7)
    _, rows, _ = OM.masked_loss(logits, labels, 1, 7, off)
    assert torch.allclose(rows, _direct_rows(logits, labels, 1, off), rtol=1e-13, atol=1e-13)
    assert not OM.window_mask(8, 1, off, V)[:, :off].any()


def test_loss_and_grads_on_the_model_matches_the_windowed_loss():
    cfg = O.DalleConfig(n_embd=32, n_layers=1, n_heads=2, text_vocab_size=21, image_vocab_size=6, text_seq_len=4,
                        image_seq_len=5)
    params = {k: v.double() for k, v in O.init_params(cfg, 0).items()}
    g = torch.Generator().manual_seed(5)
    tokens = torch.cat([torch.randint(0, 21, (2, 4), generator=g), torch.randint(0, 6, (2, 5), generator=g) + 21], 1)
    loss, rows, _, logits, grads = OM.loss_and_grads(params, tokens, cfg, 21)
    labels = O.shift_labels(tokens, cfg.eos_token_id)
    assert torch.allclose(rows, _direct_rows(logits, labels, 4, 21), rtol=1e-12, atol=1e-12)
    assert torch.isclose(loss, rows.mean())
    # d loss / d bias = the sum over rows of the explicit gradient (which carries the 1 / (B S) of the mean)
    T = tokens.numel()
    dl = OM.dlogits(logits.reshape(T, -1), labels.reshape(-1), 4, 5, 21)
    assert torch.allclose(grads["to_logits/linear_out/bias"], dl.sum(0), rtol=1e-10, atol=1e-14)


# ------------------------------------------------------------------------------------------------------ config key
@pytest.mark.parametrize("value,expected", [(True, True), (False, False), (None, False)])
def test_config_key_accepts_true_false_and_null(value, expected):
    from dalle_mtf_b200.model_fns import logits_mask
    assert logits_mask({"logits_mask": value}) is expected
    assert logits_mask({}) is False


@pytest.mark.parametrize("value", ["true", "yes", 1, 0, 1.0, [True], {"on": True}])
def test_config_key_rejects_other_values(value):
    from dalle_mtf_b200.model_fns import logits_mask
    with pytest.raises(ValueError, match="logits_mask"):
        logits_mask({"logits_mask": value})


def test_example_config_is_the_example_plus_the_key():
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "dalle_example_b200.json")) as f:
        base = json.load(f)
    with open(os.path.join(root, "configs", "dalle_example_logits_mask_b200.json")) as f:
        masked = json.load(f)
    assert masked.pop("logits_mask") is True
    masked.pop("model_path"), base.pop("model_path")
    assert masked == base
