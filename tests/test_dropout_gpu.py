"""GPU tests of embed / attention / residual dropout: the fused kernels against the oracle's masks (oracle/philox.py),
each dropout variant against torch math on the materialised masks, and the engine / model_fn properties the masks
must keep (bit-reproducibility, micro-batch and rank invariance, resume, no dropout outside training).
Tolerances are those of the tests without dropout (test_kernels_gpu.py, test_engine_gpu.py)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = "cuda"
RATES = (0.1, 0.2, 0.15)


@pytest.fixture(scope="module")
def L():
    from dalle_mtf_b200 import lib
    lib.require_device()
    return lib


def relmax(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert torch.isfinite(got).all()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-30)).item()


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def bf(x):
    return x.to(torch.bfloat16)


def _mask(L, desc, layout, dims):
    from dalle_mtf_b200 import ops
    shape = dims if layout == L.DROPOUT_ELEMENTWISE else (dims[0], dims[1], dims[2], dims[2])
    keep = torch.empty(shape, dtype=torch.uint8, device=DEV)
    ops.dropout_mask(desc, layout, dims, keep)
    return keep.cpu()


# ------------------------------------------------------------------------------------------------------- masks
@pytest.mark.parametrize("rate,seed,step,site,rows,cols,row0", [(0.1, 0, 0, 0, 65, 256, 0),
                                                                (0.5, 2 ** 40 + 3, 17, 7, 300, 512, 1300)])
def test_elementwise_mask_matches_oracle(L, rate, seed, step, site, rows, cols, row0):
    from oracle import philox as X
    d = L.make_dropout(rate, seed, step, site, row0)
    got = _mask(L, d, L.DROPOUT_ELEMENTWISE, (rows, cols)).numpy().astype(bool)
    assert np.array_equal(got, X.keep_elementwise(rate, seed, step, site, rows, cols, row0))


@pytest.mark.parametrize("rate,B,H,S,row0", [(0.2, 2, 3, 77, 0), (0.5, 3, 2, 130, 5), (0.1, 1, 1, 64, 2)])
def test_attention_mask_matches_oracle(L, rate, B, H, S, row0):
    from oracle import philox as X
    d = L.make_dropout(rate, 9, 4, 5, row0)
    got = _mask(L, d, L.DROPOUT_ATTENTION, (B, H, S)).numpy().astype(bool)
    assert np.array_equal(got, X.keep_attention(rate, 9, 4, 5, B, H, S, row0))


# ------------------------------------------------------------------------------------------------------- attention
def _ref_attn_drop(qkv, scale, mult):
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    s = torch.einsum("bihe,bjhe->bhij", q, k) * scale
    S = q.shape[1]
    s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool), 1), float("-inf"))
    return torch.einsum("bhij,bjhe->bihe", torch.softmax(s, -1) * mult, v), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,S,H,dh,scale,mag,row0", [(1, 128, 1, 128, 1.0, 0.3, 0), (1, 128, 1, 64, 1.0, 0.4, 3),
                                                     (2, 256, 2, 128, 1.0, 0.3, 1), (1, 300, 3, 64, 0.125, 1.0, 0),
                                                     (1, 333, 2, 128, 0.0884, 1.0, 7), (1, 129, 1, 128, 1.0, 0.5, 0),
                                                     (2, 1280, 3, 64, 0.125, 1.0, 2)])
def test_attention_dropout_fwd_bwd_match_reference(L, B, S, H, dh, scale, mag, row0):
    from dalle_mtf_b200 import ops
    rate = 0.2
    d = L.make_dropout(rate, 123, 5, 2, row0)
    keep = _mask(L, d, L.DROPOUT_ATTENTION, (B, H, S)).float()
    g = torch.Generator().manual_seed(S + dh)
    qkv = bf(torch.randn(B, S, 3, H, dh, generator=g) * mag)
    dout = bf(torch.randn(B, S, H, dh, generator=g))
    qf = qkv.float().requires_grad_(True)
    o_ref, lse_ref = _ref_attn_drop(qf, scale, keep * d.scale)
    o_ref.backward(dout.float())
    qd, dd = qkv.to(DEV), dout.to(DEV)
    out = torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, H, S, device=DEV)
    ops.attn_fwd(qd, out, lse, B, S, H, dh, scale, dropout=d)
    assert relmax(out, o_ref) < 1e-2 and relmax(lse, lse_ref) < 1e-3
    dqkv = torch.zeros_like(qd)
    ops.attn_bwd(qd, out, dd, lse, torch.zeros(1, device=DEV), torch.zeros(B, H, S, device=DEV), dqkv, B, S, H, dh,
                 scale, dropout=d)
    for i in range(3):
        assert relmax(dqkv[:, :, i], qf.grad[:, :, i]) < 2e-2, i


@pytest.mark.parametrize("dh", [64, 128])
def test_attention_ex_with_null_or_zero_rate_is_the_old_entry_point(L, dh):
    import ctypes
    from dalle_mtf_b200.lib import ptr, stream_ptr
    B, S, H = 2, 200, 2
    g = torch.Generator(device=DEV).manual_seed(dh)
    qkv = bf(torch.randn(B, S, 3, H, dh, generator=g, device=DEV) * 0.5)
    dout = bf(torch.randn(B, S, H, dh, generator=g, device=DEV))
    lib = L.load()
    zero = L.Dropout()
    zero.scale = 1.0
    res = []
    for desc in ("old", None, zero):
        out = torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV)
        lse = torch.zeros(B, H, S, device=DEV)
        dqkv = torch.zeros_like(qkv)
        delta, dq = torch.zeros(B, H, S, device=DEV), torch.zeros(1, device=DEV)
        a = (stream_ptr(), ptr(qkv), ptr(out), ptr(lse), B, S, H, dh, 1.0)
        b = (stream_ptr(), ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dq), ptr(delta), ptr(dqkv), B, S, H, dh, 1.0)
        if desc == "old":
            L.check(lib.db200_attn_causal_fwd(*a)); L.check(lib.db200_attn_causal_bwd(*b))
        else:
            r = None if desc is None else ctypes.byref(desc)
            L.check(lib.db200_attn_causal_fwd_ex(*a, r)); L.check(lib.db200_attn_causal_bwd_ex(*b, r))
        torch.cuda.synchronize()
        res.append((out, lse, dqkv))
    for other in res[1:]:
        for x, y in zip(res[0], other):
            assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------------- GEMM / rows
@pytest.mark.parametrize("M,N,K,row0", [(300, 256, 128, 0), (1000, 512, 256, 640), (77, 264, 72, 3)])
def test_gemm_store_with_dropout(L, M, N, K, row0):
    from dalle_mtf_b200 import ops
    g = torch.Generator().manual_seed(M + N)
    x = bf(torch.randn(M, K, generator=g))
    w = bf(torch.randn(K, N, generator=g) * K ** -0.5)
    bias = torch.randn(N, generator=g) * 0.1
    res = bf(torch.randn(M, N, generator=g))
    d = L.make_dropout(0.15, 77, 3, 4, row0)
    mult = _mask(L, d, L.DROPOUT_ELEMENTWISE, (M, N)).float() * d.scale
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.linear_fwd(x.to(DEV), w.to(DEV), out, bias=bias.to(DEV), residual=res.to(DEV), dropout=d)
    ref = res.float() + mult * (x.float() @ w.float() + bias)
    assert relmax(out, ref) < 1e-2
    # rate 0 runs the kernel without dropout: bit-identical to the plain call
    a = torch.empty_like(out)
    ops.linear_fwd(x.to(DEV), w.to(DEV), a, bias=bias.to(DEV), residual=res.to(DEV))
    b = torch.empty_like(out)
    zero = L.Dropout()      # threshold 0 through db200_gemm_bf16_ex
    zero.scale = 1.0
    ops.linear_fwd(x.to(DEV), w.to(DEV), b, bias=bias.to(DEV), residual=res.to(DEV), dropout=zero)
    assert torch.equal(a, b)


@pytest.mark.parametrize("rows,d,row0", [(300, 256, 0), (129, 512, 64), (70, 4096, 5)])
def test_layernorm_bwd_dropout_variant(L, rows, d, row0):
    from dalle_mtf_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(rows + d)
    x = bf(torch.randn(rows, d, generator=g, device=DEV))
    dy = bf(torch.randn(rows, d, generator=g, device=DEV))
    dres = bf(torch.randn(rows, d, generator=g, device=DEV))
    gam = 1 + 0.1 * torch.randn(d, generator=g, device=DEV)
    mean, rstd = x.float().mean(-1), torch.rsqrt(x.float().var(-1, unbiased=False) + 1e-5)
    drop = L.make_dropout(0.3, 5, 2, 6, row0)
    outs = []
    for with_drop in (False, True):
        dx = torch.empty(rows, d, dtype=torch.bfloat16, device=DEV)
        dxm = torch.empty_like(dx) if with_drop else None
        dg, db, dxsum = (torch.zeros(d, device=DEV) for _ in range(3))
        ops.layernorm_bwd(dy, x, gam, mean, rstd, dres, dx, dg, db, dxsum=dxsum, dxm=dxm,
                          dropout=drop if with_drop else None)
        outs.append((dx, dxm, dg, db, dxsum))
    (dx0, _, dg0, db0, _), (dx1, dxm, dg1, db1, dxsum) = outs
    assert torch.equal(dg0, dg1) and torch.equal(db0, db1)
    # dx is the same math; the compiler may contract a few elements differently in the two instantiations (one bf16 ulp)
    assert ((dx1.float() - dx0.float()).abs() <= dx0.float().abs() * 2 ** -7).all()
    mult = _mask(L, drop, L.DROPOUT_ELEMENTWISE, (rows, d)).to(DEV).float() * drop.scale
    assert torch.equal(dxm, bf(dx1.float() * mult))
    assert relmax(dxsum, dxm.float().sum(0)) < 1e-5


@pytest.mark.parametrize("B,S,d,V,row0", [(3, 77, 256, 500, 0), (2, 64, 512, 100, 4)])
def test_embedding_dropout_fwd_bwd(L, B, S, d, V, row0):
    from dalle_mtf_b200 import ops
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(0, 40, (B, S), generator=g, dtype=torch.int32)   # repeated ids: scatter onto shared rows
    wte = bf(torch.randn(V, d, generator=g))
    wpe = bf(torch.randn(S, d, generator=g))
    dx = bf(torch.randn(B, S, d, generator=g))
    dw = L.make_dropout(0.25, 3, 8, L.SITE_WTE, row0 * S)
    dp = L.make_dropout(0.25, 3, 8, L.SITE_WPE, 0)
    mw = _mask(L, dw, L.DROPOUT_ELEMENTWISE, (B * S, d)).float().view(B, S, d) * dw.scale
    mp_ = _mask(L, dp, L.DROPOUT_ELEMENTWISE, (S, d)).float() * dp.scale
    out = torch.empty(B, S, d, dtype=torch.bfloat16, device=DEV)
    ops.embed_fwd(ids.to(DEV), wte.to(DEV), wpe.to(DEV), out, wte_drop=dw, wpe_drop=dp)
    ref = wte.float()[ids.long()] * mw + wpe.float() * mp_
    assert relmax(out, ref) < 1e-2
    dwte, dwpe = torch.zeros(V, d, device=DEV), torch.zeros(S, d, device=DEV)
    ops.embed_bwd(ids.to(DEV), dx.to(DEV), dwte, dwpe, wte_drop=dw, wpe_drop=dp)
    rw = torch.zeros(V, d).index_add_(0, ids.long().flatten(), (dx.float() * mw).view(-1, d))
    assert relmax(dwte, rw) < 1e-5
    assert relmax(dwpe, dx.float().sum(0) * mp_) < 1e-5


# ------------------------------------------------------------------------------------------------------- engine
def _dalle_case(d, Ly, H, tv, iv, ts, isl, B, recompute, seed=0, rates=RATES, dseed=0):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    cfg = O.DalleConfig(d, Ly, H, tv, iv, ts, isl)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.05
    tokens = torch.randint(0, cfg.total_tokens - 1, (B, cfg.seq_len), generator=g)
    eng = DalleEngine(d, Ly, H, tv, iv, ts, isl, recompute_grad=recompute, dropout=rates, dropout_seed=dseed)
    eng.load_params(params)
    return cfg, params, tokens, eng


CASES = [(256, 2, 2, 1000, 100, 40, 24, 3), (256, 2, 4, 1000, 100, 100, 60, 2), (512, 2, 4, 3000, 512, 200, 100, 2)]


@pytest.mark.parametrize("case", CASES)
def test_engine_with_dropout_matches_oracle_recompute_off_and_on(case):
    from oracle import dalle_dropout as D
    from oracle import optim as OO
    step, row0, dseed = 6, 1, 11
    spec = (RATES, dseed, step, row0)
    cfg, params, tokens, _ = _dalle_case(*case, False, dseed=dseed)
    loss32, _, _, g32 = D.loss_and_grads(params, tokens, cfg, spec, bf16=False)
    _, _, _, g16 = D.loss_and_grads(params, tokens, cfg, spec, bf16=True)
    tok = tokens.to(torch.int32).cuda()
    T = tokens.numel()
    grads_by_mode = []
    for recompute in (False, True):
        _, _, _, eng = _dalle_case(*case, recompute, dseed=dseed)
        eng.zero_grads()
        acc = eng.forward(tok, step=step, row0=row0)
        eng.backward(1.0 / T)
        torch.cuda.synchronize()
        assert abs(acc.item() / T - loss32.item()) / loss32.item() < 2e-3, recompute
        grads = eng.export_params(eng.grads)
        for k in g32:
            e_engine, e_ref = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
            assert e_engine <= 1.25 * e_ref + 1e-2, (recompute, k, e_engine, e_ref)
        grads_by_mode.append(eng.grads.clone())
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
    assert torch.equal(grads_by_mode[0], grads_by_mode[1])   # recompute regenerates the forward's masks


def _three_steps(step0=0, dseed=0, rates=RATES):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 2, 2, 500, 64, 64, 64, dropout=rates, dropout_seed=dseed)
    eng.init_params(3)
    tok = torch.randint(0, 40, (4, eng.S), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV,
                        dtype=torch.int32)
    losses, grads = [], []
    for s in range(3):
        eng.zero_grads()
        acc = eng.forward(tok, step=step0 + s)
        eng.backward(1.0 / tok.numel())
        grads.append(eng.grads.clone())
        losses.append(acc.clone())
        eng.optimizer_step(1e-3)
    torch.cuda.synchronize()
    return losses, grads, eng.master.clone()


def test_training_with_dropout_is_bitwise_reproducible_and_depends_on_step_and_seed():
    (l0, g0, p0), (l1, g1, p1) = _three_steps(), _three_steps()
    for a, b in zip(l0, l1):
        assert torch.equal(a, b)
    for a, b in zip(g0, g1):
        assert torch.isfinite(a).all() and torch.equal(a, b)
    assert torch.equal(p0, p1)
    assert not torch.equal(_three_steps(step0=1)[0][0], l0[0])
    assert not torch.equal(_three_steps(dseed=1)[0][0], l0[0])
    assert not torch.equal(_three_steps(rates=(0, 0, 0))[0][0], l0[0])


def test_forward_without_step_and_logits_equal_a_model_without_dropout():
    _, _, tokens, eng = _dalle_case(256, 2, 2, 300, 60, 20, 12, 2, False)
    _, _, _, ref = _dalle_case(256, 2, 2, 300, 60, 20, 12, 2, False, rates=(0.0, 0.0, 0.0))
    tok = tokens.to(torch.int32).cuda()
    a, b = (torch.zeros(1, device=DEV) for _ in range(2))
    eng.forward(tok, loss_accum=a)
    ref.forward(tok, loss_accum=b)
    assert torch.equal(a, b)
    eng.forward(tok, loss_accum=torch.zeros(1, device=DEV), step=3)     # a training forward in between
    assert torch.equal(eng.logits(tok), ref.logits(tok))


def test_dalle_class_applies_dropout_in_train_mode_only():
    from dalle_mtf_b200.models import DALLE
    kw = dict(n_embd=256, text_vocab_size=100, image_vocab_size=20, text_seq_len=8, image_seq_len=8, n_layers=1,
              n_heads=2, batch_size=2, bf_16=True)
    p = {"embed_dropout": 0.1, "attention_dropout": 0.1, "residual_dropout": 0.1}
    tokens = torch.randint(0, 120, (2, 16), generator=torch.Generator().manual_seed(0))
    plain = DALLE(mode="train", params={}, **kw).forward({"tokens": tokens})[0]
    ev = DALLE(mode="eval", params=p, **kw).forward({"tokens": tokens})[0]
    assert torch.equal(ev, plain)
    tr = DALLE(mode="train", params=p, **kw)
    l1, l2 = tr.forward({"tokens": tokens})[0], tr.forward({"tokens": tokens})[0]   # steps 0 and 1
    assert not torch.equal(l1, plain) and not torch.equal(l1, l2)
    with pytest.raises(ValueError):
        DALLE(mode="train", params={"residual_dropout": 1.0}, **kw)


def test_two_microbatches_draw_the_masks_of_one_batch():
    _, _, tokens, eng = _dalle_case(256, 2, 2, 300, 60, 20, 12, 4, False)
    tok = tokens.to(torch.int32).cuda()
    T = tok.numel()
    eng.zero_grads()
    a = eng.forward(tok, loss_accum=torch.zeros(1, device=DEV), step=2).clone()
    eng.backward(1.0 / T)
    g_one = eng.grads[:eng.n_params_padded].clone()
    eng.zero_grads()
    b = torch.zeros(1, device=DEV)
    for i in range(2):
        eng.forward(tok[2 * i:2 * i + 2], loss_accum=b, step=2, row0=2 * i)
        eng.backward(1.0 / T)
    g_two = eng.grads[:eng.n_params_padded].clone()
    torch.cuda.synchronize()
    assert abs(a.item() - b.item()) / a.item() < 1e-5
    assert relfro(g_two, g_one) < 2e-3


# ------------------------------------------------------------------------------------------------------- model_fn
def _tiny_dalle_params(tmp_path, **extra):
    from collections import defaultdict
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}})
    p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                   "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                   "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 2e-3,
                                   "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1",
                                   "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                   "vae_params": vae, "vae_random_init": True, "seed": 5})
    p.update(extra)
    return p


def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def test_model_fn_eval_op_ignores_dropout_and_resume_keeps_the_masks(tmp_path):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    img, cap = _batch()
    drop = dict(embed_dropout=0.1, attention_dropout=0.2, residual_dropout=0.15)
    ev = dalle_model_fn(img, cap, "eval", _tiny_dalle_params(tmp_path, **drop)).eval_op(img, cap).clone()
    ev0 = dalle_model_fn(img, cap, "eval", _tiny_dalle_params(tmp_path)).eval_op(img, cap).clone()
    assert torch.equal(ev, ev0)
    # uninterrupted: 3 steps;  resumed: 2 steps, checkpoint, fresh model_fn, 1 step
    full = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, **drop))
    losses = [full.train_op(img, cap).clone() for _ in range(3)]
    first = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, **drop))
    for _ in range(2):
        first.train_op(img, cap)
    state = first.state_fn()
    resumed = dalle_model_fn(img, cap, "train", _tiny_dalle_params(tmp_path, **drop))
    resumed.load_fn(state)
    assert resumed.global_step == 2
    assert torch.equal(resumed.train_op(img, cap), losses[2])
    # tokens_per_mb_per_replica splits the batch into micro-batches: same masks, same loss up to summation order
    p_mb = _tiny_dalle_params(tmp_path, tokens_per_mb_per_replica=2 * 28, **drop)   # S = 12 + 4 * 4
    mb = dalle_model_fn(img, cap, "train", p_mb)
    assert p_mb["num_microbatches"] == 2
    l_mb = mb.train_op(img, cap).item()
    assert abs(l_mb - losses[0].item()) / losses[0].item() < 1e-5


# ------------------------------------------------------------------------------------------------------- 2 ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    dev = torch.device("cuda", rank)
    args = (256, 2, 2, 500, 64, 24, 40)
    g = torch.Generator().manual_seed(0)
    global_tokens = torch.randint(0, 500 + 64, (4, 64), generator=g, dtype=torch.int32)
    T = global_tokens.numel()
    eng = DalleEngine(*args, device=dev, dropout=RATES, dropout_seed=4)
    eng.init_params(seed=7)
    start, per = dp.shard(4)
    eng.zero_grads()
    eng.forward(global_tokens[start:start + per].to(dev), step=3, row0=start)
    eng.backward(1.0 / T, on_bucket_ready=dp.make_bucket_hook(eng.grads))
    dp.wait()
    g_dp = eng.grads[:eng.n_params_padded].clone()
    eng.optimizer_step(1e-3)
    torch.cuda.synchronize()
    loss_dp = eng.grads[eng.aux_off].item() / T
    ref = DalleEngine(*args, device=dev, dropout=RATES, dropout_seed=4)
    ref.init_params(seed=7)
    ref.zero_grads()
    ref.forward(global_tokens.to(dev), step=3)
    ref.backward(1.0 / T)
    g_ref = ref.grads[:ref.n_params_padded].clone()
    ref.optimizer_step(1e-3)
    torch.cuda.synchronize()
    loss_ref = ref.grads[ref.aux_off].item() / T
    n = eng.n_params_padded
    gerr = ((g_dp - g_ref).norm() / g_ref.norm()).item()
    perr = ((eng.master[:n] - ref.master[:n]).norm() / ref.master[:n].norm()).item()
    dp.barrier()
    out.put((rank, loss_dp, loss_ref, gerr, perr))
    dp.shutdown()


def test_two_rank_dropout_step_equals_single_rank_step_on_concatenated_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, loss_dp, loss_ref, gerr, perr in res:
        assert abs(loss_dp - loss_ref) / loss_ref < 1e-5, res
        assert gerr < 2e-3, res
        assert perr < 1e-5, res
