"""GPU parity tests of the engines and of the drop-in boundary (model_fns) against the oracle.

Tolerances:
  * loss (mean over B*S fp32 per-token losses): 2e-3 relative vs the fp32 oracle (north_star: 1e-3 rel in bf16 is met
    in practice — measured ~1e-5 — the bound leaves room for other seeds).
  * logits: relative Frobenius error <= 2e-2 vs fp32 oracle (every activation is rounded to bf16, 2^-8 per op).
  * gradients: the reference's own bf16 policy (oracle with bf16 cast points) deviates from fp32 math by e_ref(k) per
    tensor; the engine must be no worse than 1.25 * e_ref(k) + 1e-2 — i.e. within the reference's bf16 rounding noise.
  * VAE in fp32 mode: 1e-4 (fp32 kernels), token / code indices bit-exact.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _dalle_case(d, L, H, tv, iv, ts, isl, B, recompute, seed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:   # non-trivial biases / gains so that their use and gradients are exercised
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, recompute_grad=recompute)
    eng.load_params(params)
    return cfg, params, tokens, eng


@pytest.mark.parametrize("d,L,H,tv,iv,ts,isl,B,recompute", [
    (256, 2, 2, 1000, 100, 40, 24, 3, False),     # dh=128, S=64
    (256, 2, 4, 1000, 100, 100, 60, 2, False),    # dh=64,  S=160 (ragged 128-row tiles)
    (512, 2, 4, 3000, 512, 200, 100, 2, True),    # recompute_grad path, S=300
])
def test_dalle_forward_backward_optimizer_match_oracle(d, L, H, tv, iv, ts, isl, B, recompute):
    from oracle import dalle as O
    from oracle import optim as OO
    cfg, params, tokens, eng = _dalle_case(d, L, H, tv, iv, ts, isl, B, recompute)
    loss32, _, logits32, g32 = O.loss_and_grads(params, tokens, cfg, bf16=False)
    _, _, _, g16 = O.loss_and_grads(params, tokens, cfg, bf16=True)
    tok = tokens.to(torch.int32).cuda()
    T = tokens.numel()
    eng.zero_grads()
    acc = eng.forward(tok)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    assert abs(acc.item() / T - loss32.item()) / loss32.item() < 2e-3
    assert relfro(eng.logits(tok), logits32) < 2e-2
    grads = eng.export_params(eng.grads)
    for k in g32:
        e_engine, e_ref = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
        assert e_engine <= 1.25 * e_ref + 1e-2, (k, e_engine, e_ref)
    # the padded vocabulary columns never receive gradient
    assert (eng.G("wout")[:, eng.V:] == 0).all() and (eng.G("bout")[eng.V:] == 0).all()
    # one optimiser step applied to the ENGINE's gradients: isolates schedule + clip + Adam
    hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
    zeros = {k: torch.zeros_like(v) for k, v in params.items()}
    newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
    eng.optimizer_step(lr)
    torch.cuda.synchronize()
    assert abs(eng.gnorm_sq.sqrt().item() - gn.item()) / gn.item() < 1e-4
    after = eng.export_params()
    for k in params:
        if (newp[k] - params[k]).norm() > 0:
            assert relfro(after[k] - params[k], newp[k] - params[k]) < 1e-3, k


def test_dalle_training_curve_tracks_oracle_for_several_steps():
    """Loss curve on a fixed batch: 6 optimiser steps, engine (bf16) vs oracle (fp32), each loss within 1e-2 relative.
    (Bias-correction-free Adam takes sign-like steps of size lr while v is tiny, so bf16 gradient noise is amplified
    step after step; with lr = 2e-3 the two trajectories drift apart by 9 % after six steps although every single-step
    quantity matches — hence a moderate lr here and a per-step bound that grows from 2e-3 to 2e-2;
    measured drift: 3e-7, 2e-5, 3e-4, 2e-3, 3e-3, 1e-2.)"""
    from oracle import dalle as O
    from oracle import optim as OO
    cfg, params, tokens, eng = _dalle_case(256, 2, 2, 300, 60, 20, 12, 4, False, seed=3)
    hp = {"lr": 4e-4, "train_steps": 100, "warmup_steps": 2}
    m = {k: torch.zeros_like(v) for k, v in params.items()}
    v = {k: torch.zeros_like(v_) for k, v_ in params.items()}
    p = params
    tok = tokens.to(torch.int32).cuda()
    T = tokens.numel()
    ref_losses, eng_losses = [], []
    for step in range(1, 7):
        loss, _, _, grads = O.loss_and_grads(p, tokens, cfg)
        ref_losses.append(loss.item())
        p, m, v, lr, _ = OO.dalle_train_step(p, m, v, grads, step, hp)
        eng.zero_grads()
        acc = eng.forward(tok)
        eng.backward(1.0 / T)
        eng.optimizer_step(lr)
        eng_losses.append(acc.item() / T)
    assert ref_losses[-1] < ref_losses[0] - 0.05            # it actually trains
    for i, (a, b) in enumerate(zip(eng_losses, ref_losses)):
        assert abs(a - b) / b < (2e-3, 2e-3, 5e-3, 1e-2, 1e-2, 2e-2)[i], (eng_losses, ref_losses)


def test_dalle_class_mirrors_reference_forward_signature():
    from dalle_mtf_b200.models import DALLE
    m = DALLE(n_embd=256, text_vocab_size=100, image_vocab_size=20, text_seq_len=8, image_seq_len=8, n_layers=1,
              n_heads=2, batch_size=2, bf_16=True, mode="train", params={})
    tokens = torch.randint(0, 120, (2, 16))
    loss, loss_batch = m.forward({"tokens": tokens}, return_loss=True)
    assert loss.shape == (1,) and loss_batch.shape == (2, 16) and torch.isfinite(loss).all()
    assert abs(loss.item() - loss_batch.mean().item()) < 1e-4
    loss, loss_batch, logits = m.forward({"tokens": tokens}, return_loss=True, return_logits=True)
    assert logits.shape == (2, 16, 121)                                       # total_tokens = 100 + 20 + 1
    assert m.forward({"tokens": tokens}, return_loss=False).shape == (2, 16, 121)


# ------------------------------------------------------------------------------------------------------- VAE
@pytest.mark.parametrize("N,H,Cin,Cout,k,stride,transposed", [
    (2, 8, 16, 24, 3, 1, False), (2, 9, 5, 70, 3, 1, False), (2, 8, 3, 32, 4, 2, False), (3, 12, 20, 36, 4, 2, False),
    (2, 6, 24, 16, 4, 2, True), (1, 5, 70, 9, 4, 2, True), (2, 8, 16, 3, 1, 1, False),
    # channel counts that are multiples of 64 run on wgmma through the three-way bf16 split (conv_f32_tc.cu)
    (2, 8, 64, 64, 3, 1, False), (3, 9, 128, 64, 3, 1, False), (2, 8, 64, 128, 4, 2, False),
    (2, 6, 128, 64, 4, 2, True), (1, 4, 256, 256, 3, 1, False), (2, 8, 64, 512, 1, 1, False),
    (5, 16, 64, 64, 3, 1, False)])
def test_direct_conv_fwd_dgrad_wgrad_fp32(N, H, Cin, Cout, k, stride, transposed):
    from dalle_mtf_b200 import ops
    from oracle import vae as OV
    g = torch.Generator().manual_seed(N * 100 + H)
    x = torch.randn(N, H, H, Cin, generator=g)
    w = torch.randn(*((k, k, Cout, Cin) if transposed else (k, k, Cin, Cout)), generator=g) * 0.1
    bias = torch.randn(Cout, generator=g) * 0.1
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    y = OV.conv2d_transpose_same(xr, wr, br) if transposed else OV.conv2d_same(xr, wr, br, stride)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    c = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, transposed=transposed, act_f32=True)
    xd, wd, bd, dyd = x.to(DEV), w.to(DEV), bias.to(DEV), dy.to(DEV)
    yd, dxd = torch.empty(y.shape, device=DEV), torch.empty(x.shape, device=DEV)
    dwd, dbd = torch.zeros(w.shape, device=DEV), torch.zeros(Cout, device=DEV)
    ops.conv2d_fwd(c, xd, wd, bd, None, yd)
    ops.conv2d_dgrad(c, dyd, wd, None, None, dxd)
    ops.conv2d_wgrad(c, xd, dyd, dwd, dbd)
    # CUDA-core path: fp32 FMA chains (1e-5).  wgmma path (channels % 64 == 0): products are exact to ~2^-24 through the
    # three-way split, but the tensor core adds partial sums with truncation, so long contractions (K = 9 x 256) sit at
    # ~1e-5 relative — still two orders below one bf16 rounding (4e-3)
    tol = 3e-5 if (Cin % 64 == 0 and Cout % 64 == 0) else 1e-5
    assert relfro(yd, y) < tol and relfro(dxd, xr.grad) < tol
    assert relfro(dwd, wr.grad) < tol and relfro(dbd, br.grad) < 1e-5


@pytest.mark.parametrize("N,H,Cin,Cout,k,stride,relu,res", [
    (2, 16, 64, 64, 3, 1, True, False), (2, 16, 128, 128, 3, 1, False, True), (3, 12, 64, 128, 3, 1, False, False),
    (2, 16, 64, 128, 4, 2, False, False), (5, 8, 128, 256, 4, 2, False, False), (2, 4, 256, 256, 3, 1, True, True),
    (1, 32, 256, 64, 3, 1, False, False)])
def test_tensor_core_conv_forward_bf16(N, H, Cin, Cout, k, stride, relu, res):
    from dalle_mtf_b200 import ops
    from oracle import vae as OV
    g = torch.Generator().manual_seed(Cin + Cout + H)
    x = torch.randn(N, H, H, Cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(k, k, Cin, Cout, generator=g) * (k * k * Cin) ** -0.5).to(torch.bfloat16)
    bias = torch.randn(Cout, generator=g) * 0.1
    y = OV.conv2d_same(x.float(), w.float(), bias, stride)
    y = torch.relu(y) if relu else y
    r = torch.randn(y.shape, generator=g).to(torch.bfloat16) if res else None
    y = y + r.float() if res else y
    c = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, act_f32=False, relu=relu)
    yd = torch.zeros(y.shape, dtype=torch.bfloat16, device=DEV)
    ops.conv2d_fwd_tc(c, x.to(DEV), w.to(DEV).view(-1, Cout), bias.to(DEV), None if r is None else r.to(DEV), yd)
    assert relfro(yd, y) < 1e-2


@pytest.mark.parametrize("N,H,Cin,Cout,k,stride,transposed", [
    (2, 16, 64, 64, 3, 1, False), (2, 16, 128, 64, 3, 1, False), (3, 12, 64, 128, 3, 1, False),
    (2, 16, 64, 128, 4, 2, False), (2, 8, 128, 64, 4, 2, True), (5, 4, 256, 128, 4, 2, True),
    (1, 32, 256, 256, 3, 1, False)])
def test_tensor_core_conv_training_kernels_bf16(N, H, Cin, Cout, k, stride, transposed):
    """conv-transpose forward, dgrad (with ReLU mask + residual-gradient add) and wgrad on wgmma vs autograd."""
    from dalle_mtf_b200 import ops
    from oracle import vae as OV
    g = torch.Generator().manual_seed(Cin * 7 + Cout + H)
    bf = lambda t: t.to(torch.bfloat16)
    x = bf(torch.randn(N, H, H, Cin, generator=g))
    wshape = (k, k, Cout, Cin) if transposed else (k, k, Cin, Cout)
    w = bf(torch.randn(*wshape, generator=g) * (k * k * Cin) ** -0.5)
    bias = torch.randn(Cout, generator=g) * 0.1
    xr, wr = x.float().requires_grad_(True), w.float().requires_grad_(True)
    y = OV.conv2d_transpose_same(xr, wr, bias) if transposed else OV.conv2d_same(xr, wr, bias, stride)
    dy = bf(torch.randn(y.shape, generator=g))
    y.backward(dy.float())
    c = ops.conv_desc(N, H, H, Cin, Cout, k, k, stride, transposed=transposed, act_f32=False)
    xd, wd, dyd = x.to(DEV), w.to(DEV), dy.to(DEV)
    yd = torch.zeros(y.shape, dtype=torch.bfloat16, device=DEV)
    ops.conv2d_fwd_tc(c, xd, wd, bias.to(DEV), None, yd)
    assert relfro(yd, y) < 1e-2
    mask = bf(torch.randn(x.shape, generator=g))
    dres = bf(torch.randn(x.shape, generator=g))
    dxd = torch.zeros(x.shape, dtype=torch.bfloat16, device=DEV)
    ops.conv2d_dgrad_tc(c, dyd, wd, mask.to(DEV), dres.to(DEV), dxd)
    assert relfro(dxd, xr.grad * (mask.float() > 0) + dres.float()) < 1e-2
    dwd = torch.ones(wshape, device=DEV)
    ops.conv2d_wgrad_tc(c, xd, dyd, dwd)
    assert relfro(dwd, 1.0 + wr.grad) < 1e-4        # bf16 inputs are exact in the reference too; fp32 accumulate


def test_vae_engine_bf16_training_step_on_tensor_cores():
    """Whole VAE step with bf16 activations (wgmma conv fwd/dgrad/wgrad): loss and gradients vs the fp32 oracle."""
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    cb, K, size, B = [[2, 64], [2, 128]], 128, 32, 4
    g = torch.Generator().manual_seed(77)
    p = OV.init_params(cb, K, seed=5)
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // 4
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    loss, out, logits, grads = OV.loss_and_grads(p, img, u.view(B, hw, hw, K), cb, 1.0, False)
    _, _, _, g16 = OV.loss_and_grads(p, img, u.view(B, hw, hw, K), cb, 1.0, False, bf16=True)
    eng = VaeEngine(K, size, cb, use_bf16=True)
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(1, device=DEV)
    eng.forward(img.to(DEV), u.to(DEV), 1.0, False, loss_accum=acc)
    eng.backward()
    torch.cuda.synchronize()
    assert relfro(acc, loss.reshape(1)) < 2e-2
    eg = eng.export_params(eng.grads)
    for k in grads:   # no worse than the reference's own bf16 policy (+ slack)
        e_engine, e_ref = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        assert e_engine <= 1.5 * e_ref + 2e-2, (k, e_engine, e_ref)


@pytest.mark.parametrize("convblocks,K,size,B,hard,tau", [
    ([[2, 32], [2, 64]], 64, 16, 4, True, 1.0), ([[2, 32], [2, 64]], 64, 16, 4, False, 0.5),
    ([[3, 64], [3, 128], [3, 256]], 512, 32, 8, True, 1.0)])          # last = vae_example geometry
def test_vae_engine_fp32_matches_oracle_exactly_enough(convblocks, K, size, B, hard, tau):
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    g = torch.Generator().manual_seed(K + size)
    p = OV.init_params(convblocks, K, seed=K)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // (2 ** len(convblocks))
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    loss, out, logits, grads = OV.loss_and_grads(p, img, u.view(B, hw, hw, K), convblocks, tau, hard)
    eng = VaeEngine(K, size, convblocks)
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(1, device=DEV)
    recon = eng.forward(img.to(DEV), u.to(DEV), tau, hard, loss_accum=acc)
    eng.backward()
    torch.cuda.synchronize()
    assert relfro(eng._b["logits"], logits.reshape(-1, K)) < 1e-4
    idx_ref = OV.gumbel_softmax(logits, u.view(B, hw, hw, K), tau, True).argmax(-1).flatten()
    assert torch.equal(eng._b["idx"].cpu().long(), idx_ref)                    # sampled codes: bit-exact
    assert torch.equal(eng.encode_tokens(img.to(DEV)).cpu().long(), OV.encode_tokens(p, img, convblocks))
    assert relfro(recon, out) < 1e-4 and relfro(acc, loss.reshape(1)) < 1e-4
    eg = eng.export_params(eng.grads)
    for k in grads:
        # fp32 atomics order + tensor-core accumulation order; the hard-Gumbel encoder / codebook gradients are sums
        # of ~1e-3 terms that cancel to ~1e-6 values, so their RELATIVE error amplifies the 1e-5 of the convolutions
        assert relfro(eg[k], grads[k]) < 2e-2, k
    # TF-style Adam (bias-corrected) on the engine's gradients
    from oracle import optim as OO
    eng.optimizer_step(1e-3, step=1)
    after = eng.export_params()
    for k in ("codebook/codebook", "decoder/conv2d/kernel"):
        ref, _, _ = OO.adam_tf_step(p[k], torch.zeros_like(p[k]), torch.zeros_like(p[k]), eg[k], 1e-3, 1)
        assert relfro(after[k] - p[k], ref - p[k]) < 1e-3


@pytest.mark.parametrize("N,H,Cout", [(2, 16, 64), (3, 24, 128), (1, 256, 64)])
def test_first_layer_conv_kernel(N, H, Cout):
    from dalle_mtf_b200 import ops
    from oracle import vae as OV
    g = torch.Generator().manual_seed(H)
    x = torch.rand(N, H, H, 3, generator=g) * 2 - 1
    w = torch.randn(4, 4, 3, Cout, generator=g) * 0.2
    bias = torch.randn(Cout, generator=g) * 0.1
    y = OV.conv2d_same(x, w, bias, 2)
    yd = torch.zeros(N, H // 2, H // 2, Cout, dtype=torch.bfloat16, device=DEV)
    ops.conv2d_first_fwd(x.to(DEV), w.to(DEV), bias.to(DEV), yd)
    assert relfro(yd, y) < 5e-3      # fp32 math, bf16 output rounding only


def test_bf16_tensor_core_tokenizer_agrees_with_fp32_oracle_up_to_near_ties():
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    cb = [[3, 64], [3, 128], [3, 256]]
    p = OV.init_params(cb, 512, seed=30)
    g = torch.Generator().manual_seed(30)
    img = (torch.randint(0, 256, (4, 64, 64, 3), generator=g).float() - 127.5) / 127.5
    logits = OV.encoder(p, img, cb).reshape(-1, 512)
    eng = VaeEngine(512, 64, cb, use_bf16=True)
    eng.load_params(p)
    tok = eng.encode_tokens(img.to(DEV)).cpu().long().flatten()
    assert relfro(eng._b["logits"], logits) < 3e-2
    ref = logits.argmax(-1)
    top2 = logits.topk(2, -1).values
    margin = top2[:, 0] - top2[:, 1]
    mism = tok != ref
    assert (~mism).float().mean() > 0.97
    if mism.any():   # every disagreement is a near-tie of the fp32 logits
        assert margin[mism].max() < 0.1 * margin.median() + 1e-3 or margin[mism].max() < 0.05


# ------------------------------------------------------------------------------------------------------- boundary
def _tiny_params(tmp_path, vae_bf16=False):
    from collections import defaultdict
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}, "train_batch_size": 4, "eval_batch_size": 4,
                                     "lr": 1e-3, "model_path": str(tmp_path / "vae"), "n_channels": 3,
                                     "train_gumbel_hard": True, "use_bf16": vae_bf16, "iterations": 2,
                                     "steps_per_checkpoint": 3, "train_steps": 6})
    dalle = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                       "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                       "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                       "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                       "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                       "iterations": 2, "steps_per_checkpoint": 4, "n_channels": 3, "padding_id": 299,
                                       "vae_params": vae})
    return vae, dalle


def test_two_stage_run_vae_checkpoint_feeds_dalle_model_fn(tmp_path):
    """train_vae_tf-style run -> checkpoint -> dalle_model_fn loads it by vae_params.model_path (model_fns.py:35-52),
    tokens produced inside the step equal the oracle's argmax tokens bit-exactly, loss decreases, resume works."""
    from functools import partial
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import dalle_input_fn, vae_input_fn
    from dalle_mtf_b200.model_fns import dalle_model_fn, vae_model_fn
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint, load_global_step_from_checkpoint_dir
    from oracle import vae as OV
    vae_p, dalle_p = _tiny_params(tmp_path)
    est = Estimator(vae_model_fn, vae_p)
    est.train(partial(vae_input_fn, eval=False), max_steps=6)
    assert load_global_step_from_checkpoint_dir(vae_p["model_path"]) == 6
    st = load_checkpoint(latest_checkpoint(vae_p["model_path"]))
    vae_weights = {k[len("vae/"):]: v for k, v in st.items()
                   if k.startswith("vae/") and not k.endswith("/Adam") and not k.endswith("/Adam_1")}
    # DALL-E stage
    est2 = Estimator(dalle_model_fn, dalle_p)
    spec = est2.train(partial(dalle_input_fn, eval=False), max_steps=4)
    img, cap = next(iter(dalle_input_fn(dalle_p)))
    toks = spec.assemble(img, cap).cpu().long()
    ref_img_tokens = OV.encode_tokens(vae_weights, img, [[2, 64], [2, 64]])
    assert torch.equal(toks[:, :12], cap.long())
    assert torch.equal(toks[:, 12:], ref_img_tokens + 300)                     # token indices: bit-exact
    # a few more steps: loss goes down on average, and a fresh Estimator resumes at the saved step
    l0 = float(spec.loss_sum.item()) * spec.loss_scale
    for _ in range(12):
        spec.train_op(img, cap)
    l1 = float(spec.loss_sum.item()) * spec.loss_scale
    assert l1 < l0
    est3 = Estimator(dalle_model_fn, dalle_p)
    spec3 = est3._spec("train", img, cap)
    assert spec3.global_step == 4


def test_full_size_step_is_finite_and_starts_near_log_vocab():
    """One step at the BASELINE shape (B=8 of S=1280 to keep the test short): loss ~ ln(50771) = 10.8 at init."""
    import math
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    g = torch.Generator(device=DEV).manual_seed(0)
    tok = torch.randint(0, eng.V - 1, (8, eng.S), generator=g, device=DEV, dtype=torch.int32)
    eng.zero_grads()
    acc = eng.forward(tok)
    eng.backward(1.0 / tok.numel())
    loss0 = acc.item() / tok.numel()
    assert abs(loss0 - math.log(eng.V)) < 0.3
    assert torch.isfinite(eng.grads).all()
    eng.optimizer_step(1e-3)
    for _ in range(3):
        eng.zero_grads(); acc = eng.forward(tok); eng.backward(1.0 / tok.numel()); eng.optimizer_step(1e-3)
    assert acc.item() / tok.numel() < loss0


def test_vae_stack_factor_2_matches_oracle():
    """stack_factor > 1 (src/vae_tf/models.py:85-86, 155-161): space_to_depth on the way in, depth_to_space on the way
    out, image_seq_len divided by stack_factor^2 (src/model_fns.py:68); fp32 mode, loss / logits / tokens / gradients."""
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    cb, K, size, B, sf = [[2, 32], [2, 64]], 64, 32, 3, 2
    g = torch.Generator().manual_seed(5)
    p = OV.init_params(cb, K, stack_factor=sf, seed=9)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // sf // 4
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    leaves = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss, out, logits = OV.forward(leaves, img, u.view(B, hw, hw, K), cb, 1.0, True, stack_factor=sf)
    loss.backward()
    eng = VaeEngine(K, size, cb, stack_factor=sf)
    assert eng.image_seq_len == OV.image_seq_len(size, cb, sf) == hw * hw
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(1, device=DEV)
    recon = eng.forward(img.to(DEV), u.to(DEV), 1.0, True, loss_accum=acc)
    eng.backward()
    torch.cuda.synchronize()
    assert tuple(recon.shape) == (B, size, size, 3)
    assert relfro(eng._b["logits"], logits.reshape(-1, K)) < 1e-4
    assert relfro(recon, out) < 1e-4 and relfro(acc, loss.reshape(1)) < 1e-4
    assert torch.equal(eng.encode_tokens(img.to(DEV)).cpu().long(), OV.encode_tokens(p, img, cb, stack_factor=sf))
    eg = eng.export_params(eng.grads)
    for k in p:
        assert relfro(eg[k], leaves[k].grad) < 2e-2, k


def test_training_step_is_bitwise_reproducible():
    """Two engines from the same weights, fed the same tokens, agree bit for bit after three steps.  The shape takes the
    split-K wgrad path (T = 512 tokens: two K splits), repeats token ids (embedding scatter onto shared rows) and runs
    every ordered reduction of the step (LayerNorm dg / db, bias column sums, gradient norm, loss)."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    runs = []
    for _ in range(2):
        eng = DalleEngine(256, 2, 2, 500, 64, 64, 64)
        eng.init_params(3)
        tok = torch.randint(0, 40, (4, eng.S), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV,
                            dtype=torch.int32)
        losses, grads = [], []
        for _ in range(3):
            eng.zero_grads()
            acc = eng.forward(tok)
            eng.backward(1.0 / tok.numel())
            grads.append(eng.grads.clone())
            losses.append(acc.clone())
            eng.optimizer_step(1e-3)
        torch.cuda.synchronize()
        runs.append((losses, grads, eng.master.clone()))
    (l0, g0, p0), (l1, g1, p1) = runs
    for a, b in zip(l0, l1):
        assert torch.equal(a, b)
    for a, b in zip(g0, g1):
        assert torch.isfinite(a).all() and torch.equal(a, b)
    assert torch.equal(p0, p1)
