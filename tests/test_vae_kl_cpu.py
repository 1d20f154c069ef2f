"""CPU tests of the discrete VAE's KL term: the oracle (oracle/vae_kl.py) against torch's own KL and the closed-form
gradient, the anneal schedule, the config validation, the codebook-usage statistics and the estimator's log lines."""
import math
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from oracle import vae_kl as OK


def test_oracle_kl_equals_torch_kl_div_against_the_uniform_prior():
    g = torch.Generator().manual_seed(0)
    for rows, K in ((1, 1), (5, 7), (64, 512)):
        logits = torch.randn(rows, K, generator=g, dtype=torch.float64) * 3
        ref = F.kl_div(torch.tensor(math.log(1.0 / K), dtype=torch.float64), F.log_softmax(logits, -1),
                       log_target=True, reduction="sum") / rows
        assert torch.allclose(OK.kl_uniform(logits), ref, rtol=1e-12, atol=1e-12)


def test_oracle_kl_is_zero_on_constant_logits_and_log_k_on_a_one_hot_limit():
    K = 100
    assert OK.kl_uniform(torch.full((3, K), 2.5, dtype=torch.float64)).abs().item() < 1e-14
    one_hot = torch.zeros(4, K, dtype=torch.float64)
    one_hot[:, 7] = 1e4          # q underflows to 0 on the other codes: l - lse is used, never log q
    kl = OK.kl_uniform(one_hot)
    assert torch.isfinite(kl) and abs(kl.item() - math.log(K)) < 1e-12


def test_oracle_autograd_gradient_equals_the_closed_form():
    g = torch.Generator().manual_seed(1)
    logits = (torch.randn(2, 3, 3, 50, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    rows = 18
    OK.kl_uniform(logits).backward()
    assert torch.allclose(logits.grad, OK.kl_grad(logits.detach(), 1.0 / rows), rtol=1e-10, atol=1e-14)


def test_oracle_mutations_change_value_or_gradient():
    g = torch.Generator().manual_seed(2)
    logits = (torch.randn(2, 2, 2, 16, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    OK.kl_uniform(logits).backward()
    good = logits.grad.clone()
    logits.grad = None
    OK.kl_uniform(logits, "no_centring").backward()
    assert torch.allclose(OK.kl_uniform(logits, "no_centring"), OK.kl_uniform(logits))   # same value
    assert not torch.allclose(logits.grad, good)                                         # other gradient
    assert torch.allclose(OK.kl_uniform(logits, "per_image"), OK.kl_uniform(logits) * 4)  # 4 rows per image


def test_oracle_without_kl_weight_is_oracle_vae_bit_for_bit():
    from oracle import vae as OV
    cb, K, size, B = [[1, 16], [1, 16]], 32, 8, 2
    p = OV.init_params(cb, K, seed=3)
    g = torch.Generator().manual_seed(3)
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    u = torch.rand(B, 2, 2, K, generator=g).clamp_(1e-9, 1.0)
    loss, out, logits, grads = OV.loss_and_grads(p, img, u, cb, 0.7, True)
    loss2, mse, kl, out2, logits2, grads2 = OK.loss_and_grads(p, img, u, cb, 0.7, True)
    assert kl is None and torch.equal(loss, loss2) and torch.equal(mse, loss) and torch.equal(out, out2)
    assert all(torch.equal(grads[k], grads2[k]) for k in grads)
    # with the term, the loss is recon + beta * KL of the raw logits
    lossk, msek, klk, _, logitsk, _ = OK.loss_and_grads(p, img, u, cb, 0.7, True, kl_weight=0.5)
    assert torch.equal(msek, loss) and torch.allclose(lossk, msek + 0.5 * OK.kl_uniform(logitsk))


@pytest.mark.parametrize("step,expect", [(0, 0.0), (50, 0.25), (100, 0.5), (250, 0.5)])
def test_beta_schedule(step, expect):
    from dalle_mtf_b200.model_fns import vae_kl_weight
    params = {"kl_loss_weight": 0.5, "kl_anneal_steps": 100}
    assert vae_kl_weight(step, params) == pytest.approx(expect) == OK.kl_weight(step, params)
    assert vae_kl_weight(step, {"kl_loss_weight": 0.5}) == 0.5
    assert vae_kl_weight(step, {}) is None


def test_beta_schedule_continues_across_a_resume():
    """The schedule is a function of global_step: a run resumed at step s sees the betas an uninterrupted run sees."""
    from dalle_mtf_b200.model_fns import vae_kl_weight
    params = {"kl_loss_weight": 2.0, "kl_anneal_steps": 10}
    straight = [vae_kl_weight(s, params) for s in range(20)]
    resumed = [vae_kl_weight(s, params) for s in range(7)] + [vae_kl_weight(s, dict(params)) for s in range(7, 20)]
    assert straight == resumed and straight[5] == 1.0 and straight[15] == 2.0


@pytest.mark.parametrize("beta,anneal", [
    (True, None), (False, None), ("0.1", None), (float("nan"), None), (float("inf"), None), (-float("inf"), None),
    (-0.1, None), (0.1, 0), (0.1, -3), (0.1, 2.5), (0.1, True), (0.1, "10"), (None, 10)])
def test_malformed_kl_keys_are_rejected(beta, anneal):
    from dalle_mtf_b200.model_fns import kl_loss_weight
    params = defaultdict(lambda: None, {"kl_loss_weight": beta, "kl_anneal_steps": anneal})
    with pytest.raises(ValueError):
        kl_loss_weight(params)


@pytest.mark.parametrize("beta,anneal", [(0, None), (0.0, 1), (1, 1000), (6.6, None)])
def test_wellformed_kl_keys_are_accepted(beta, anneal):
    from dalle_mtf_b200.model_fns import kl_loss_weight
    assert kl_loss_weight({"kl_loss_weight": beta, "kl_anneal_steps": anneal}) == (float(beta), anneal)
    assert kl_loss_weight(defaultdict(lambda: None)) == (None, None)


def test_codebook_usage_uniform_and_single_code():
    from dalle_mtf_b200.vae_engine import codebook_usage
    K = 64
    uniform = torch.full((K,), 5, dtype=torch.int32)
    single = torch.zeros(K, dtype=torch.int32)
    single[9] = 320
    for fn in (codebook_usage, OK.usage_of_counts):
        used, ppl = fn(uniform)
        assert used == K and ppl == pytest.approx(K, rel=1e-12)
        used, ppl = fn(single)
        assert used == 1 and ppl == pytest.approx(1.0, abs=1e-12)


def test_oracle_codes_follow_the_first_maximum_and_send_nan_rows_to_code_0():
    logits = torch.tensor([[1.0, 3.0, 3.0, 0.0], [float("nan"), 5.0, 1.0, 1.0], [-math.inf] * 4,
                           [0.0, 0.0, 0.0, 2.0], [1.0, float("nan"), 9.0, 0.0]])
    assert OK.first_max_codes(logits).tolist() == [1, 0, 0, 3, 0]
    counts, used, ppl = OK.codebook_usage(logits)
    assert counts.tolist() == [3, 1, 0, 1] and used == 3


# ------------------------------------------------------------------------------------------------- estimator lines
class _DP:
    rank, world, enabled = 0, 1, False

    def barrier(self):
        pass


def _log_lines(tmp_path, configure):
    """Train two steps through the Estimator on a fake spec configured by `configure(spec)`; returns the step lines."""
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import StepSpec

    lines = []

    class _Log:
        def info(self, msg):
            lines.append(msg)

    def fake_model_fn(features, labels, mode, params):
        spec = StepSpec(mode, engine=None, dp=_DP())

        def train_op(f, l):
            spec.global_step += 1
            spec.loss_sum, spec.loss_scale = torch.tensor([1.5]), 1.0
            configure(spec)
            return spec.loss_sum
        spec.train_op = train_op
        spec.state_fn = lambda: {"global_step": spec.global_step}
        spec.load_fn = lambda st: None
        return spec

    params = defaultdict(lambda: None, {"dataset": {"image_size": 8, "train_path": "synthetic"}, "train_batch_size": 2,
                                        "model_path": str(tmp_path / "m"), "iterations": 1})
    est = Estimator(fake_model_fn, params, logger=_Log())
    est.train(partial(vae_input_fn, eval=False), max_steps=2)
    est.close()
    return [ln.split(" global_step/sec")[0] for ln in lines if ln.startswith("step ")]


def test_dalle_log_lines_are_unchanged(tmp_path):
    plain = _log_lines(tmp_path / "a", lambda spec: None)
    assert plain == ["step 1 loss 1.50000", "step 2 loss 1.50000"]

    def weighted(spec):
        spec.loss_parts = torch.tensor([2.0, 3.25, 1.5e-4])
    assert _log_lines(tmp_path / "b", weighted)[0] == \
        "step 1 loss 1.50000 text_ce 2.00000 image_ce 3.25000 z_term 0.00015"


def test_vae_log_line_carries_recon_kl_and_codebook_usage(tmp_path):
    from dalle_mtf_b200.model_fns import VAE_PARTS_FORMAT

    calls = []

    def kl(spec):
        spec.loss_parts = torch.tensor([0.125, 0.5])
        spec.loss_parts_format = VAE_PARTS_FORMAT
        spec.codebook_usage = lambda: calls.append(1) or (37, 21.456)
    lines = _log_lines(tmp_path, kl)
    assert lines[1] == "step 2 loss 1.50000 recon_mse 0.12500 kl 0.50000 codes_used 37 perplexity 21.46"
    assert len(calls) == 2     # the usage reduction runs at log steps only
