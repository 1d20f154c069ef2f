"""CPU tests of the discrete VAE's logit-Laplace reconstruction loss: the oracle (oracle/vae_logit_laplace.py) against
numerical integration and the closed-form gradients, its mutations, the reconstruction_loss key's validation, the
beta conversion from the paper's per-image ELB and the estimator's log lines."""
import math
from collections import defaultdict

import pytest
import torch
from scipy import integrate

from oracle import vae_logit_laplace as OL


@pytest.mark.parametrize("mu,b", [(0.0, 1.0), (1.5, 0.3), (-2.0, 0.05), (0.3, 4.0), (3.0, 1e-2)])
def test_oracle_density_integrates_to_one_over_the_unit_interval(mu, b):
    """exp(-nll) with the Jacobian 1 / (y (1 - y)) of t = logit(y) is a density of y on (0, 1)."""
    u0 = 1.0 / (1.0 + math.exp(-mu))
    total = 0.0
    for lo, hi in ((0.0, u0), (u0, 1.0)):       # split at the cusp y = sigmoid(mu)
        v, _ = integrate.quad(OL.density, lo, hi, args=(mu, b), limit=400, epsabs=1e-13, epsrel=1e-11)
        total += v
    assert abs(total - 1.0) < 1e-8


def test_oracle_nll_is_the_negative_log_density():
    g = torch.Generator().manual_seed(0)
    stats = torch.randn(50, 6, generator=g, dtype=torch.float64)
    x = torch.rand(50, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8
    got = OL.nll(stats, x)
    y, _ = OL.target(x)
    for i in range(0, 50, 7):
        for c in range(3):
            ref = -math.log(OL.density(y[i, c].item(), stats[i, c].item(), math.exp(stats[i, 3 + c].item())))
            assert abs(got[i, c].item() - ref) < 1e-10


def test_oracle_autograd_gradients_equal_the_closed_forms():
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 4, 4, 3, generator=g, dtype=torch.float64) * 2 - 1
    x[0, 0, 0] = torch.tensor([-1.0, 1.0, 1.3])           # the ends of the range and beyond (clamped)
    _, t = OL.target(x)
    mu = torch.randn(2, 4, 4, 3, generator=g, dtype=torch.float64)
    mu[1, 2, 2] = t[1, 2, 2]                               # t = mu exactly: d mu = 0 (sign(0) = 0)
    lb = torch.rand(2, 4, 4, 3, generator=g, dtype=torch.float64) * 12 - 8
    stats = torch.cat([mu, lb], -1).requires_grad_(True)
    OL.nll(stats, x).mean().backward()
    dmu, dlb = OL.grads(stats.detach(), x, 1.0 / x.numel())
    assert torch.allclose(stats.grad, torch.cat([dmu, dlb], -1), rtol=1e-12, atol=1e-15)
    assert (stats.grad[1, 2, 2, :3] == 0).all()


def test_oracle_image_maps_t_equal_mu_back_to_the_target():
    x = torch.linspace(-1, 1, 101, dtype=torch.float64).view(1, 1, 101, 1)
    _, t = OL.target(x)
    stats = torch.cat([t, torch.zeros_like(t)], -1)
    assert torch.allclose(OL.image(stats), x, rtol=0, atol=1e-12)
    extreme = torch.tensor([[-50.0, 0.0], [50.0, 0.0]], dtype=torch.float64)
    assert OL.image(extreme).flatten().tolist() == [-1.0, 1.0]      # clamped into [-1, 1]


def test_oracle_mutations_change_value_or_gradient():
    g = torch.Generator().manual_seed(2)
    stats = torch.randn(3, 3, 3, 6, generator=g, dtype=torch.float64, requires_grad=True)
    x = torch.rand(3, 3, 3, 3, generator=g, dtype=torch.float64) * 2 - 1

    def run(m):
        stats.grad = None
        v = OL.nll(stats, x, m).mean()
        v.backward()
        return v.detach(), stats.grad.clone(), OL.image(stats.detach(), m)
    v0, g0, i0 = run(None)
    for m in OL.MUTATIONS:
        v, gm, im = run(m)
        assert not (torch.allclose(v, v0) and torch.allclose(gm, g0) and torch.allclose(im, i0)), m
    assert not torch.allclose(run("wrong_eps")[0], v0) and not torch.allclose(run("swap_halves")[1], g0)
    assert not torch.allclose(run("no_jacobian")[0], v0) and not torch.allclose(run("mu_pixel_space")[2], i0)


def test_oracle_forward_with_kl_adds_the_kl_term():
    from oracle import vae_kl as OK
    cb, K, size, B = [[1, 16], [1, 16]], 32, 8, 2
    p = OL.init_params(cb, K, seed=3)
    assert p["decoder/conv2d/kernel"].shape == (1, 1, 16, 6) and p["decoder/conv2d/bias"].shape == (6,)
    g = torch.Generator().manual_seed(3)
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    u = torch.rand(B, 2, 2, K, generator=g).clamp_(1e-9, 1.0)
    loss, rec, mse, kl, xhat, logits = OL.forward(p, img, u, cb, 0.7, True, kl_weight=0.25)
    assert torch.allclose(loss, rec + 0.25 * OK.kl_uniform(logits))
    assert torch.allclose(mse, ((xhat - img) ** 2).mean())
    loss0, rec0, _, kl0, _, _ = OL.forward(p, img, u, cb, 0.7, True)
    assert kl0 is None and torch.equal(loss0, rec0) and torch.equal(rec0, rec)


def test_oracle_stack_factor_keeps_the_packed_channel_order():
    from oracle import vae as OV
    cb, K, size, B, s = [[1, 16], [1, 16]], 32, 16, 1, 2
    p = OL.init_params(cb, K, stack_factor=s, seed=4)
    assert p["decoder/conv2d/kernel"].shape[-1] == 24
    g = torch.Generator().manual_seed(4)
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    u = torch.rand(B, 2, 2, K, generator=g).clamp_(1e-9, 1.0)
    _, rec, _, _, xhat, logits = OL.forward(p, img, u, cb, 1.0, True, stack_factor=s)
    stats = OV.decoder(p, OV.gumbel_softmax(logits, u, 1.0, True), cb, stack_factor=1)
    assert torch.allclose(rec, OL.nll(stats, OV.space_to_depth(img, s)).mean())
    assert torch.allclose(xhat, OV.depth_to_space(OL.image(stats), s))


def test_beta_conversion_at_the_vae_coco_geometry():
    """The paper's per-image ELB / (H W C) = mean nll + beta h w / (H W C) mean KL; vae_coco: 256^2 x 3, 32 x 32."""
    assert OL.beta_from_paper(6.6, 256, 3, 32) == pytest.approx(0.034375, rel=1e-15)
    import json
    import os
    cfg = json.load(open(os.path.join(os.path.dirname(__file__), "..", "configs", "vae_coco_elb_b200.json")))
    grid = cfg["dataset"]["image_size"] // 2 ** len(cfg["convblocks"])
    assert cfg["kl_loss_weight"] == pytest.approx(OL.beta_from_paper(6.6, cfg["dataset"]["image_size"], 3, grid),
                                                  rel=1e-15)
    assert cfg["reconstruction_loss"] == "logit_laplace"
    # the identity itself, on a small per-image ELB: sum nll + beta sum KL over one image's h w rows
    g = torch.Generator().manual_seed(5)
    nll = torch.rand(8, 8, 3, generator=g, dtype=torch.float64)
    kl_rows = torch.rand(2, 2, generator=g, dtype=torch.float64)
    elb = nll.sum() + 6.6 * kl_rows.sum()
    assert torch.allclose(elb / nll.numel(), nll.mean() + OL.beta_from_paper(6.6, 8, 3, 2) * kl_rows.mean())


# ------------------------------------------------------------------------------------------------------ the key
@pytest.mark.parametrize("value,expected", [("mse", "mse"), ("logit_laplace", "logit_laplace"), (None, "mse")])
def test_reconstruction_loss_key_accepts(value, expected):
    from dalle_mtf_b200.model_fns import reconstruction_loss
    assert reconstruction_loss(value) == expected


@pytest.mark.parametrize("value", ["logit_laplase", "MSE", "", True, 1, 0.5, ["mse"]])
def test_reconstruction_loss_key_rejects(value):
    from dalle_mtf_b200.model_fns import reconstruction_loss
    with pytest.raises(ValueError):
        reconstruction_loss(value)


def _vae_params(**extra):
    d = {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]], "dataset": {"image_size": 16},
         "train_batch_size": 4, "eval_batch_size": 4, "lr": 1e-3}
    d.update(extra)
    return defaultdict(lambda: None, d)


@pytest.mark.parametrize("value", ["logit-laplace", False, 2])
def test_every_builder_rejects_a_bad_key_before_touching_a_device(value):
    from dalle_mtf_b200.model_fns import TRAIN, load_vae_model, vae_model_fn
    from dalle_mtf_b200.models import DiscreteVAE
    with pytest.raises(ValueError, match="reconstruction_loss"):
        vae_model_fn(None, None, TRAIN, _vae_params(reconstruction_loss=value))
    with pytest.raises(ValueError, match="reconstruction_loss"):
        load_vae_model({"dataset": {"image_size": 16}, "vae_params": _vae_params(reconstruction_loss=value)}, "cpu")
    with pytest.raises(ValueError, match="reconstruction_loss"):
        DiscreteVAE(64, 16, [[2, 64], [2, 64]], reconstruction_loss=value)


# ------------------------------------------------------------------------------------------------- estimator lines
def test_vae_log_lines_with_logit_laplace(tmp_path):
    from dalle_mtf_b200.model_fns import VAE_LL_KL_PARTS_FORMAT, VAE_LL_PARTS_FORMAT
    from test_vae_kl_cpu import _log_lines

    def ll(spec):
        spec.loss_parts = torch.tensor([-1.25, 0.0625])
        spec.loss_parts_format = VAE_LL_PARTS_FORMAT
    assert _log_lines(tmp_path / "a", ll)[1] == "step 2 loss 1.50000 recon_nll -1.25000 recon_mse 0.06250"

    def ll_kl(spec):
        spec.loss_parts = torch.tensor([-1.25, 0.0625, 0.5])
        spec.loss_parts_format = VAE_LL_KL_PARTS_FORMAT
        spec.codebook_usage = lambda: (37, 21.456)
    assert _log_lines(tmp_path / "b", ll_kl)[1] == \
        "step 2 loss 1.50000 recon_nll -1.25000 recon_mse 0.06250 kl 0.50000 codes_used 37 perplexity 21.46"
