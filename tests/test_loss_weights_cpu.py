"""CPU tests of the weighted DALL-E loss (text_loss_weight / image_loss_weight / z_loss): the oracle against
oracle.dalle and float64 finite differences, the config validation, and the coefficients' independence of how the
global batch is split."""
import json
import math
import os

import pytest
import torch

from dalle_mtf_b200.dalle_engine import loss_coefficients
from dalle_mtf_b200.model_fns import loss_weights
from oracle import dalle as O
from oracle import loss_weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _tiny(seed=0, dtype=F64):
    cfg = O.DalleConfig(n_embd=16, n_layers=1, n_heads=2, text_vocab_size=20, image_vocab_size=8, text_seq_len=5,
                        image_seq_len=6)
    params = {k: v.to(dtype) for k, v in O.init_params(cfg, seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:   # non-zero biases and larger logits, so that lse and the class terms differ between rows
        if k.endswith("bias") or k.endswith("/b"):
            params[k] = torch.randn(params[k].shape, generator=g, dtype=dtype) * 0.3
    params["to_logits/linear_out/kernel"] = params["to_logits/linear_out/kernel"] * 40
    text = torch.randint(0, cfg.text_vocab_size, (3, cfg.text_seq_len), generator=g)
    img = torch.randint(0, cfg.image_vocab_size, (3, cfg.image_seq_len), generator=g)
    return cfg, params, O.assemble_tokens(text, img, cfg.text_vocab_size)


def test_reference_ratio_without_z_is_the_reference_loss():
    cfg, params, tokens = _tiny()
    ratio = (cfg.text_seq_len - 1, cfg.image_seq_len + 1)
    loss0, rows0, _, g0 = O.loss_and_grads(params, tokens, cfg)
    loss, rows, parts, _, g = W.loss_and_grads(params, tokens, cfg, ratio, 0.0)
    assert torch.allclose(loss, loss0, rtol=1e-13, atol=0) and torch.equal(rows, rows0)
    for k in g0:
        assert torch.allclose(g[k], g0[k], rtol=1e-10, atol=1e-15), k
    a_t, a_i = W.coefficients(ratio, cfg.text_seq_len, cfg.image_seq_len, tokens.shape[0])
    assert math.isclose(a_t, a_i, rel_tol=1e-15) and math.isclose(a_t, 1 / tokens.numel(), rel_tol=1e-15)
    # the parts: text-row and image-row means of the CE, the z-term 0
    mask = W.text_mask(cfg.seq_len, cfg.text_seq_len)
    assert torch.allclose(parts[0], rows0[:, mask].mean()) and torch.allclose(parts[1], rows0[:, ~mask].mean())
    assert parts[2] == 0


@pytest.mark.parametrize("weights,z", [((1.0, 7.0), 0.0), ((1.0, 7.0), 0.05), (None, 0.05), ((0.0, 1.0), 0.02),
                                       ((2.0, 0.0), 0.0)])
def test_autograd_matches_finite_differences_and_the_explicit_gradient(weights, z):
    cfg, params, tokens = _tiny(seed=2)
    loss, rows, parts, logits, g = W.loss_and_grads(params, tokens, cfg, weights, z)
    # the explicit dlogits (what the CE_GRAD epilogue computes) equals autograd's gradient with respect to the logits
    lg = logits.clone().requires_grad_(True)
    labels = O.shift_labels(tokens, cfg.eos_token_id)
    W.weighted_loss(lg, labels, cfg.text_seq_len, cfg.image_seq_len, weights, z)[0].backward()
    V = logits.shape[-1]
    explicit = W.dlogits(logits.view(-1, V), labels.view(-1), cfg.text_seq_len, cfg.image_seq_len, weights, z)
    assert torch.allclose(explicit, lg.grad.view(-1, V), rtol=1e-10, atol=1e-16)
    # a class of weight 0 has exactly zero gradient rows
    if weights is not None and 0.0 in weights:
        zero_text = weights[0] == 0
        mask = W.text_mask(cfg.seq_len, cfg.text_seq_len).repeat(tokens.shape[0])
        assert (explicit[mask if zero_text else ~mask] == 0).all()
    # central differences of the loss on a few parameter entries, float64
    h = 1e-6
    for name, idx in (("to_logits/linear_out/kernel", (3, 5)), ("to_logits/linear_out/bias", (7,)),
                      ("layer_0/attn/q", (1, 2)), ("embedding/wte", (int(tokens[0, 2]), 4))):
        def f(delta):
            p = dict(params)
            p[name] = params[name].clone()
            p[name][idx] += delta
            _, _, lgt = O.forward(p, tokens, cfg)
            return W.weighted_loss(lgt, labels, cfg.text_seq_len, cfg.image_seq_len, weights, z)[0].item()
        fd = (f(h) - f(-h)) / (2 * h)
        assert abs(fd - g[name][idx].item()) <= 1e-6 * max(1.0, abs(fd)), (name, fd, g[name][idx].item())


def test_mutant_oracles_differ():
    """The class boundary at TL instead of TL - 1, or the z gradient without its factor 2, changes the gradient."""
    cfg, params, tokens = _tiny(seed=3)
    _, _, _, logits, _ = W.loss_and_grads(params, tokens, cfg, (1.0, 7.0), 0.05)
    labels = O.shift_labels(tokens, cfg.eos_token_id).view(-1)
    lg = logits.view(-1, logits.shape[-1])
    ok = W.dlogits(lg, labels, cfg.text_seq_len, cfg.image_seq_len, (1.0, 7.0), 0.05)
    for q in (W.LossQuirks(text_rows_offset=0), W.LossQuirks(z_grad_factor=1.0)):
        bad = W.dlogits(lg, labels, cfg.text_seq_len, cfg.image_seq_len, (1.0, 7.0), 0.05, quirks=q)
        assert (bad - ok).abs().max() > 1e-3 * ok.abs().max()


@pytest.mark.parametrize("extra", [
    {"text_loss_weight": 1.0},                                  # only one weight
    {"image_loss_weight": 7},
    {"text_loss_weight": 0, "image_loss_weight": 0.0},          # both 0
    {"text_loss_weight": True, "image_loss_weight": 7},         # a bool
    {"text_loss_weight": 1, "image_loss_weight": -7},           # negative
    {"text_loss_weight": float("nan"), "image_loss_weight": 7},  # non-finite
    {"text_loss_weight": 1, "image_loss_weight": float("inf")},
    {"text_loss_weight": "1", "image_loss_weight": 7},          # not a number
    {"z_loss": -1e-4}, {"z_loss": float("nan")}, {"z_loss": float("inf")}, {"z_loss": False}, {"z_loss": "1e-4"},
])
def test_malformed_keys_are_rejected(extra):
    with pytest.raises(ValueError):
        loss_weights(extra)


def test_accepted_keys():
    assert loss_weights({}) == (None, 0.0)
    assert loss_weights({"z_loss": 0}) == (None, 0.0)
    assert loss_weights({"text_loss_weight": 1, "image_loss_weight": 7, "z_loss": 1e-4}) == ((1.0, 7.0), 1e-4)
    assert loss_weights({"text_loss_weight": 0, "image_loss_weight": 2}) == ((0.0, 2.0), 0.0)   # a class of weight 0
    with open(os.path.join(ROOT, "configs", "dalle_example_weighted_b200.json")) as f:
        cfg = json.load(f)
    assert loss_weights(cfg) == ((1.0, 7.0), 1e-4) and cfg["caption_dropout"] > 0


@pytest.mark.parametrize("weights", [None, (1.0, 7.0), (0.0, 1.0), (3.0, 0.5)])
def test_coefficients_depend_on_the_global_batch_only(weights):
    """Every rank and micro-batch adds sum_t a_t l_t with the global batch's coefficients: the sum over any split of
    the batch is the loss of the whole batch."""
    TL, IL, Bg = 256, 1024, 8
    a = loss_coefficients(weights, TL, IL, Bg)
    ao = W.coefficients(weights, TL, IL, Bg)
    assert all(math.isclose(x, y, rel_tol=1e-15) for x, y in zip(a, ao))
    g = torch.Generator().manual_seed(0)
    rows = torch.rand(Bg, TL + IL, generator=g, dtype=F64) * 10
    coef = torch.tensor([a[0]] * (TL - 1) + [a[1]] * (IL + 1), dtype=F64)
    whole = W.weighted_loss(torch.log_softmax(torch.zeros(Bg, TL + IL, 2, dtype=F64), -1), torch.zeros(Bg, TL + IL,
                            dtype=torch.long), TL, IL, weights, 0.0)[0]    # log 2 per row: a known loss
    assert math.isclose(whole.item(), (coef * math.log(2)).sum().item() * Bg, rel_tol=1e-12)
    ref = (rows * coef).sum().item()
    for ranks in (1, 2, 4):
        for mb in (1, 2):
            local = Bg // ranks
            total = sum((rows[r * local + i * (local // mb):r * local + (i + 1) * (local // mb)] * coef).sum().item()
                        for r in range(ranks) for i in range(mb))
            assert math.isclose(total, ref, rel_tol=1e-13), (ranks, mb)
    if weights is not None:   # the loss is the weighted mean of the class means
        wt, wi = weights
        means = rows[:, :TL - 1].mean().item(), rows[:, TL - 1:].mean().item()
        assert math.isclose(ref, (wt * means[0] + wi * means[1]) / (wt + wi), rel_tol=1e-12)
