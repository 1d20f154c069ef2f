"""GPU tests of the modality logits mask (config key logits_mask).

Kernels.  db200_logits_mask_partition / db200_logits_mask_scatter against torch indexing, bit for bit.  The windowed
cross-entropy: partition -> CE_STATS -> ce_finish(_weighted) -> CE_GRAD on each block, checked per element against
float64 over the block's window with the bounds of test_loss_weights_gpu.py (its module docstring; unweighted rows take
the coefficient alpha = a).  Outside its window a row's dlogits must be exactly 0: the ≤ 7 text columns the image block
covers get -inf from the window bias, the columns past n_valid are pad columns.  Both mutants of oracle/logits_mask.py
(the class boundary at TL, EOS out of the image window) must fail the same bounds.

Engine.  The masked step against oracle/logits_mask.py with the bounds of test_parity_baseline_gpu.py (loss within
1e-3, loss_rows 5e-3, every gradient within 1.25 x the oracle's bf16 policy + 1e-2); structural zeros; bit-identical
repeats; micro-batching, reserved SMs, ZeRO-1 and in-process ranks against the one-rank step under the criteria the
plain-step tests apply; the model functions, DALLE, checkpoints and generation; and the unmasked step's launches.
"""
import math
import os

import pytest
import torch

import float64_bounds
from float64_bounds import DEV, U, UTC, nan_like
from test_dalle_kernels_gpu import Worst, _gen, _slabs, ce_operands
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu

F32, F64, BF16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int32


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


# ------------------------------------------------------------------------------------------------ partition / scatter
@pytest.mark.parametrize("B,TL,IL,d", [(3, 1, 37, 64), (5, 2, 23, 512), (3, 256, 17, 4096), (1, 256, 1024, 512)])
def test_partition_and_scatter_are_torch_indexing(ops, B, TL, IL, d):
    """Odd B S in every case; TL 1 has no text block."""
    g = _gen(B * 1000 + TL + d)
    S = TL + IL
    T = B * S
    tv, iv = 997, 61
    io, V = tv + 3, tv + 3 + iv + 1          # image_offset = 1000: c0 = 1000 - 0, and 1002 below
    hf = torch.randn(T, d, generator=g, device=DEV).to(BF16)
    tokens = torch.cat([torch.randint(0, io, (B, TL), generator=g, device=DEV, dtype=I32),
                        torch.randint(io, io + iv, (B, IL), generator=g, device=DEV, dtype=I32)], 1)
    labels = torch.empty_like(tokens)
    ops.shift_labels(tokens, labels, V - 1)
    labels = labels.view(-1)
    bias = torch.randn((V + 63) // 64 * 64, generator=g, device=DEV)
    nt = TL - 1
    text = torch.arange(S, device=DEV) < nt
    rows_t = text.repeat(B)
    for io_ in (io, io + 2):
        c0 = io_ // 8 * 8
        n_bias = (V - c0 + 7) // 8 * 8
        hf_t = nan_like((B * nt, d), BF16) if nt else None
        lab_t = torch.full((B * nt,), -7, dtype=I32, device=DEV) if nt else None
        hf_i = nan_like((B * (S - nt), d), BF16)
        lab_i = torch.full((B * (S - nt),), -7, dtype=I32, device=DEV)
        bias_i = nan_like((n_bias,), F32)
        ops.logits_mask_partition(hf, labels, bias, hf_t, hf_i, lab_t, lab_i, bias_i, B, S, nt, c0, io_, V)
        if nt:
            assert torch.equal(hf_t.view(torch.int16), hf[rows_t].view(torch.int16))
            assert torch.equal(lab_t, labels[rows_t])
        assert torch.equal(hf_i.view(torch.int16), hf[~rows_t].view(torch.int16))
        assert torch.equal(lab_i, labels[~rows_t] - c0)
        want = torch.zeros(n_bias, device=DEV)
        want[:io_ - c0] = -math.inf
        want[io_ - c0:V - c0] = bias[io_:V]
        assert torch.equal(bias_i, want)
    # scatter: dx and loss_rows back into [T] order, either part alone
    dx_t = torch.randn(B * nt, d, generator=g, device=DEV).to(BF16) if nt else None
    dx_i = torch.randn(B * (S - nt), d, generator=g, device=DEV).to(BF16)
    l_t = torch.randn(B * nt, generator=g, device=DEV) if nt else None
    l_i = torch.randn(B * (S - nt), generator=g, device=DEV)
    dx, lr = nan_like((T, d), BF16), nan_like((T,), F32)
    ops.logits_mask_scatter(B, S, nt, dx_text=dx_t, dx_image=dx_i, dx=dx)
    assert torch.isnan(lr).all()
    ops.logits_mask_scatter(B, S, nt, loss_text=l_t, loss_image=l_i, loss_rows=lr)
    want_dx = torch.empty(T, d, dtype=BF16, device=DEV)
    want_l = torch.empty(T, device=DEV)
    if nt:
        want_dx[rows_t], want_l[rows_t] = dx_t, l_t
    want_dx[~rows_t], want_l[~rows_t] = dx_i, l_i
    assert torch.equal(dx.view(torch.int16), want_dx.view(torch.int16)) and torch.equal(lr, want_l)


def test_partition_and_scatter_reject_bad_arguments(ops):
    from dalle_mtf_b200 import lib as L
    lib, s = L.load(), torch.cuda.current_stream().cuda_stream
    x = torch.zeros(4096, device=DEV)
    p = x.data_ptr()
    ok = (p, p, p, p, p, p, p, p)
    assert lib.db200_logits_mask_partition(s, *ok, 2, 10, 3, 64, 8, 10, 20) == 0
    torch.cuda.synchronize()
    for args in ((2, 10, 10, 64, 8, 10, 20), (2, 10, 3, 60, 8, 10, 20), (2, 10, 3, 64, 4, 10, 20),
                 (2, 10, 3, 64, 16, 10, 20), (2, 10, 3, 64, 8, 20, 20)):
        assert lib.db200_logits_mask_partition(s, *ok, *args) != 0, args
    assert lib.db200_logits_mask_partition(s, p + 2, *ok[1:], 2, 10, 3, 64, 8, 10, 20) != 0
    assert lib.db200_logits_mask_scatter(s, p, p, None, p, p, None, 2, 10, 3, 64) != 0
    assert lib.db200_logits_mask_scatter(s, p, p, p, p, p, p, 2, 10, 10, 64) != 0
    assert lib.db200_logits_mask_scatter(s, None, p, p, None, None, None, 2, 10, 3, 64) != 0


# ------------------------------------------------------------------------------------------------ windowed CE
def run_windowed_ce(ops, tag, B, S, TL, K, io, iv, *, weights=None, z=0.0, mutants=(), seed=0):
    """One masked forward + backward of the vocabulary products on synthetic operands; per element against float64.
    Returns the worst err/bound."""
    from dalle_mtf_b200 import lib as L
    from oracle import logits_mask as OM
    from oracle import loss_weights as OW
    V = io + iv + 1
    Vpad = (V + 63) // 64 * 64
    T, nt = B * S, TL - 1
    c0 = io // 8 * 8
    g = _gen(seed + T + K + io)
    h, W, bias, _, _ = ce_operands(T, K, V, Vpad, g)
    p = torch.arange(S, device=DEV).repeat(B)
    text = p < nt
    labels = torch.where(text, torch.randint(0, io, (T,), generator=g, device=DEV),
                         torch.randint(io, V - 1, (T,), generator=g, device=DEV))
    labels[p == S - 1] = V - 1                                   # EOS
    labels = labels.to(I32)
    weighted = weights is not None or z > 0
    a_text, a_image = OW.coefficients(weights, TL, S - TL, B)
    blocks = []
    for rows, lo, N, n_valid in ((B * nt, 0, (io + 7) // 8 * 8, io), (B * (S - nt), c0, (V - c0 + 7) // 8 * 8, V - c0)):
        blocks.append(None if rows == 0 else dict(rows=rows, lo=lo, N=N, n_valid=n_valid,
                                                  hf=nan_like((rows, K), BF16),
                                                  lab=torch.full((rows,), -1, dtype=I32, device=DEV)))
    bias_i = nan_like((blocks[1]["N"],), F32)
    ops.logits_mask_partition(h, labels, bias, blocks[0]["hf"] if nt else None, blocks[1]["hf"],
                              blocks[0]["lab"] if nt else None, blocks[1]["lab"], bias_i, B, S, nt, c0, io, V)
    base = torch.tensor([0.5, 0.25, -0.75, 0.125], device=DEV)
    sums = base.clone() if weighted else base[:1].clone()
    cs_base = torch.randn(Vpad, generator=g, device=DEV) * 1e-3
    cs = cs_base.clone()
    # one coefficient per row in each block: the plain loss back-propagates sum / T (alpha)
    for k, blk in enumerate(blocks):
        if blk is None:
            continue
        N, rows = blk["N"], blk["rows"]
        b_ = bias if k == 0 else bias_i
        nb = ops.ce_tiles(N)
        pm, ps = nan_like((nb, rows), F32), nan_like((nb, rows), F32)
        blk["ll"], blk["lse"], blk["lr"] = nan_like((rows,), F32), nan_like((rows,), F32), nan_like((rows,), F32)
        Wb = W[:, blk["lo"]:blk["lo"] + N]
        ops.gemm(blk["hf"], Wb, None, rows, N, K, a_mn=False, b_mn=True, mode=L.EPI_CE_STATS, bias=b_,
                 labels=blk["lab"], part_max=pm, part_sum=ps, label_logit=blk["ll"], n_valid=blk["n_valid"])
        cew = L.make_ce_weights(1, 1 - k, a_text, a_image, z) if weighted else None
        if weighted:
            ops.ce_finish_weighted(pm, ps, blk["ll"], blk["lse"], blk["lr"], sums, cew)
        else:
            ops.ce_finish(pm, ps, blk["ll"], blk["lse"], blk["lr"], sums)
        blk["dl"] = nan_like((rows, N), BF16)
        ops.gemm(blk["hf"], Wb, blk["dl"], rows, N, K, a_mn=False, b_mn=True, mode=L.EPI_CE_GRAD, alpha=a_text,
                 bias=b_, labels=blk["lab"], lse=blk["lse"], n_valid=blk["n_valid"],
                 colsum=cs[blk["lo"]:blk["lo"] + N], ce_weights=cew)
    # exact zeros outside each block's window
    t_blk, i_blk = blocks
    if t_blk is not None:
        assert (t_blk["dl"][:, io:] == 0).all(), f"{tag}: text block columns past image_offset are not 0"
    assert (i_blk["dl"][:, :io - c0] == 0).all(), f"{tag}: image block text columns are not 0"
    assert (i_blk["dl"][:, V - c0:] == 0).all(), f"{tag}: image block pad columns are not 0"
    # scatter the blocks back to [T] order (torch) and check per element in row slabs over the full vocabulary
    lse = torch.empty(T, device=DEV)
    lr = torch.empty(T, device=DEV)
    dense = torch.zeros(T, V, dtype=BF16, device=DEV)
    if t_blk is not None:
        lse[text], lr[text] = t_blk["lse"], t_blk["lr"]
        dense[text, :io] = t_blk["dl"][:, :io]
    lse[~text], lr[~text] = i_blk["lse"], i_blk["lr"]
    dense[~text, c0:] = i_blk["dl"][:, :V - c0]
    W64, b64 = W[:, :V].to(F64), bias[:V].to(F64)
    Wa = W64.abs()
    win = OM.window_mask(S, TL, io, V, device=DEV)
    a32 = torch.tensor([a_text, a_image], dtype=F32, device=DEV).to(F64)
    z32 = float(torch.tensor(z, dtype=F32))
    nb = ops.ce_tiles(Vpad)
    ws = {n: Worst(f"{tag} {n}") for n in ("lse", "loss_rows", "dlogits")}
    mut = [0.0] * len(mutants)
    s_ref, s_abs, s_bnd = (torch.zeros(4, dtype=F64, device=DEV) for _ in range(3))
    cs_ref, cs_abs = cs_base.to(F64), cs_base.abs().to(F64)
    for r0, r1 in _slabs(T, Vpad):
        m = win[p[r0:r1]]
        zf = h[r0:r1].to(F64) @ W64 + b64
        z_ = torch.where(m, zf, -math.inf)
        delta = torch.where(m, (K + 8) * UTC * (h[r0:r1].to(F64).abs() @ Wa + b64.abs()), 0.0)
        lse_ref = torch.logsumexp(z_, 1)
        zmax = torch.where(m, zf.abs(), 0.0).max(1).values
        eps_lse = delta.max(1).values + 5 * U * zmax + 2.0 ** -19 + (nb / 8 + 40) * U + 4 * U * lse_ref.abs()
        ws["lse"].add(lse[r0:r1], lse_ref, eps_lse, a=0.0, b=1.0)
        lab = labels[r0:r1].long()
        ce = lse_ref - zf.gather(1, lab[:, None])[:, 0]
        zt = z32 * lse_ref ** 2
        loss = ce + zt
        eps_ce = eps_lse + delta.gather(1, lab[:, None])[:, 0] + 2 * U * ce.abs()
        lb = eps_ce + z32 * (2 * lse_ref.abs() * eps_lse + 3 * U * lse_ref ** 2) + 2 * U * loss.abs()
        ws["loss_rows"].add(lr[r0:r1], loss, lb, a=0.0, b=1.0)
        tx = text[r0:r1]
        a = torch.where(tx, a32[0], a32[1])
        for i, (v, b) in enumerate(((a * loss, a * lb), (torch.where(tx, ce, 0.0), torch.where(tx, eps_ce, 0.0)),
                                    (torch.where(tx, 0.0, ce), torch.where(tx, 0.0, eps_ce)),
                                    (zt, z32 * (2 * lse_ref.abs() * eps_lse + 3 * U * lse_ref ** 2)))):
            s_ref[i] += v.sum() if weighted or i else loss.sum()
            s_abs[i] += v.abs().sum() if weighted or i else loss.abs().sum()
            s_bnd[i] += b.sum() if weighted or i else lb.sum()
        pr = torch.exp(z_ - lse_ref[:, None])
        onehot = torch.zeros_like(pr).scatter_(1, lab[:, None], 1.0)
        c = a * (1 + 2 * z32 * lse_ref)
        ref = c[:, None] * pr - a[:, None] * onehot
        eps_exp = 2.0 ** -21 + 5 * U * (torch.where(m, zf.abs(), 0.0) + lse_ref.abs()[:, None]) + \
            2 * U * torch.log(c.abs().clamp_min(1e-300)).abs()[:, None]
        acc = (1.01 * c.abs()[:, None] * (delta + eps_lse[:, None] + eps_exp) + 2 * (a * z32 * eps_lse)[:, None]
               + 4 * U * c.abs()[:, None]) * pr + U * a[:, None] * onehot
        ws["dlogits"].add(dense[r0:r1], ref, acc, b=1.0, bf16_out=True, floor=2.0 ** -126)
        for i, q in enumerate(mutants):
            bad = OM.dlogits(zf, lab, TL, S - TL, io, weights, z32, B, quirks=q)
            bad = torch.nan_to_num(bad, nan=0.0)
            mut[i] = max(mut[i], float64_bounds.worst_ratio(f"{tag} mutant", dense[r0:r1], bad, acc, b=1.0,
                                                            bf16_out=True, floor=2.0 ** -126))
        o64 = dense[r0:r1].to(F64)
        cs_ref, cs_abs = cs_ref + torch.nn.functional.pad(o64.sum(0), (0, Vpad - V)), \
            cs_abs + torch.nn.functional.pad(o64.abs().sum(0), (0, Vpad - V))
        del zf, z_, delta, pr, onehot, ref, acc, eps_exp, o64
    worst = max(w.report() for w in ws.values())
    n_sums = 4 if weighted else 1
    for i in range(n_sums):
        # the two blocks' finishes each add their block partials onto the accumulator: (M / 32 + 48) U per block
        worst = max(worst, float64_bounds.check(f"{tag} sum {i}", sums[i:i + 1], base[i:i + 1].to(F64) + s_ref[i:i + 1],
                                                base[i:i + 1].abs().to(F64) + s_abs[i:i + 1], a=0.0,
                                                b=(T / 32 + 2 * 48) * U, floor=s_bnd[i].item() + 1e-30))
    # column sums: the overlap columns [c0, io + 7] receive one (exactly zero) contribution from each block
    worst = max(worst, float64_bounds.check(f"{tag} dbias colsum", cs, cs_ref, cs_abs, a=0.0,
                                            b=(2 * 32 + T / 32 + 16) * U))
    for q, r in zip(mutants, mut):
        print(f"[logits-mask] {tag} mutant {q}: worst err/bound {r:.3g} (must exceed 1)")
        assert r > 1.0, f"{tag}: the kernels also satisfy the mutant oracle {q}"
    return worst


MUTANTS = "both"


@pytest.mark.parametrize("B,S,TL,K,io,iv,weights,z", [
    (2, 1280, 256, 512, 50258, 512, None, 0.0),             # dalle_example: image_offset = 2 (mod 8)
    (2, 1280, 256, 512, 50258, 512, (1.0, 7.0), 1e-4),
    (3, 96, 32, 256, 3000, 60, None, 0.0),                  # image_offset = 0 (mod 8): no overlap column
    (3, 96, 32, 256, 3007, 60, (2.0, 1.0), 1e-3),           # image_offset = 7 (mod 8)
    (3, 96, 1, 256, 3002, 60, (1.0, 7.0), 0.0),             # TL = 1: no text block
    (1, 1280, 256, 1024, 50258, 8192, (0.0, 1.0), 0.0),     # dalle_coco width, a zero-weight text class
])
def test_windowed_cross_entropy_against_float64(ops, B, S, TL, K, io, iv, weights, z):
    from oracle import logits_mask as OM
    mutants = (OM.Quirks(text_rows_offset=0), OM.Quirks(eos_in_image_window=False)) if TL > 1 and iv == 512 else ()
    run_windowed_ce(ops, f"windowed CE B={B} S={S} TL={TL} K={K} io={io} w={weights} z={z}", B, S, TL, K, io, iv,
                    weights=weights, z=z, mutants=mutants)


# ------------------------------------------------------------------------------------------------ engine vs oracle
def _engine_vs_oracle(d, nl, H, tv, iv, ts, isl, B, *, seed, recompute=False, types=None, rates=None, gelu=False,
                      weights=None, z=0.0, pp=False, row_col=False, drop_caption=False, radius=8, kernel=3, mask=True,
                      adam=False):
    """One masked engine step (forward, backward 1.0 with the weighted loss, else 1 / T) against
    oracle/logits_mask.py over the oracle composed from the flags; returns (the list of violated bounds, the worst
    err / bound of any check).  mask False: the same step without the logits mask, against the same oracle unmasked.
    adam: also one optimiser step on the engine's gradients against oracle/optim.py (test_engine_gpu.py's bounds:
    the global norm within 1e-4, every parameter's update within 1e-3, relative)."""
    import conv_oracle as OC
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle_gelu as OG
    from oracle import dalle_input as I
    from oracle import logits_mask as OM
    from test_parity_baseline_gpu import _randomise_small_params
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    types = types or ["global"] * nl
    cfg = OC.ConvConfig(d, nl, H, tv, iv, ts, isl, attention_types=tuple(types), local_attention_radius=radius,
                        conv_attention_kernel=kernel)
    inp = I.InputConfig("row_col" if row_col else "absolute", pp, tv - 1 if pp else None)
    io, V = I.vocab(cfg, inp)
    params = I.init_params(cfg, inp, seed)
    g = torch.Generator().manual_seed(seed + 1)
    _randomise_small_params(params, g)
    text = torch.randint(0, tv - 1, (B, ts), generator=g)
    text[:, ts // 2:] = tv - 1
    if drop_caption:
        text[0] = tv - 1                                             # a dropped caption: pads at every position
    img = torch.randint(0, iv, (B, isl), generator=g)
    tokens = I.assemble(text, img, cfg, inp)
    step = 3 if rates else None
    dropout = ((rates,) * 3, seed, step, 0) if rates else None
    act = "gelu" if gelu else "relu"
    base = lambda p, t, c, dr, bf16=False, quirks=None: OG.forward(p, t, c, dr, bf16=bf16, quirks=quirks,  # noqa
                                                                     activation=act, layers=OC)
    fwd = lambda bf16: (lambda p, t: I.forward(p, t, cfg, inp, dropout, bf16, base=base))  # noqa: E731
    loss32, rows32, parts32, _, g32 = OM.loss_and_grads(params, tokens, cfg, io, weights, z, forward=fwd(False),
                                                        mask=mask)
    _, _, _, _, g16 = OM.loss_and_grads(params, tokens, cfg, io, weights, z, forward=fwd(True), mask=mask)
    eng = DalleEngine(d, nl, H, tv, iv, ts, isl, recompute_grad=recompute, attention_types=types,
                      local_attention_radius=radius, conv_attention_kernel=kernel, dropout=(rates or 0.0,) * 3,
                      dropout_seed=seed, image_position_embedding=inp.image_position_embedding,
                      per_position_padding=pp, activation=act, logits_mask=mask,
                      loss_weights=weights, z_loss=z)
    assert eng.image_offset == io and eng.V == V
    eng.load_params(params)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=step)
    eng.backward(1.0 if eng.weighted_loss else 1.0 / T)
    torch.cuda.synchronize()
    loss = acc[0].item() if eng.weighted_loss else acc.item() / T
    bad, worst = [], [0.0, None]

    def bound(name, err, limit, *info):
        if err > limit:
            bad.append((name, err, *info))
        if err / limit > worst[0]:
            worst[:] = [err / limit, name]

    bound("loss", abs(loss - loss32.item()), 1e-3 * abs(loss32.item()), loss, loss32.item())
    bound("loss_rows", relfro(eng._bufs["loss_rows"].view(B, -1), rows32), 5e-3)
    if eng.weighted_loss:
        scales = eng.loss_part_scales(B)
        for i in range(3):
            bound(f"part {i}", abs(acc[i + 1].item() * scales[i] - parts32[i].item()),
                  1e-3 * abs(parts32[i].item()) + 1e-7, acc[i + 1].item() * scales[i], parts32[i].item())
    grads = eng.export_params(eng.grads)
    assert set(grads) == set(g32)
    total = math.sqrt(sum(v.double().norm().item() ** 2 for v in g32.values()))
    for k in g32:
        if g32[k].any():
            ee, er = relfro(grads[k], g32[k]), relfro(g16[k], g32[k])
        else:   # exactly 0 (a radius-1 layer's dq and dk: softmax over one key): rounding relative to the gradient
            ee, er = grads[k].double().norm().item() / total, g16[k].double().norm().item() / total
        bound("grad " + k, ee, 1.25 * er + 1e-2, er)
    if not ((eng.G("wout")[:, V:] == 0).all() and (eng.G("bout")[V:] == 0).all()):
        bad.append("pad columns of the gradient")
    if adam:   # one optimiser step applied to the engine's gradients: isolates schedule + clip + Adam
        from oracle import optim as OO
        hp = {"lr": 1e-3, "train_steps": 1000, "warmup_steps": 10}
        zeros = {k: torch.zeros_like(v) for k, v in params.items()}
        newp, _, _, lr, gn = OO.dalle_train_step(params, zeros, zeros, grads, 5, hp)
        eng.optimizer_step(lr)
        torch.cuda.synchronize()
        bound("global norm", abs(eng.gnorm_sq.sqrt().item() - gn.item()), 1e-4 * gn.item())
        after = eng.export_params()
        for k in params:
            if (newp[k] - params[k]).norm() > 0:
                bound("adam " + k, relfro(after[k] - params[k], newp[k] - params[k]), 1e-3)
    print(f"[logits-mask] engine d{d} L{nl} types {types} rates {rates} gelu {gelu} w {weights} z {z} pp {pp} "
          f"row_col {row_col} recompute {recompute} mask {mask}: loss {loss:.6f} oracle {loss32.item():.6f}, "
          f"worst err/bound {worst[0]:.4f} ({worst[1]}), violations {bad}")
    return bad, worst[0]


def test_tiny_masked_step_matches_the_oracle():
    assert not _engine_vs_oracle(256, 2, 2, 300, 64, 24, 64, 3, seed=1)[0]


def test_masked_step_with_every_feature_matches_the_oracle():
    """Per-position padding + row / column positions, weights + z-loss + a dropped caption, GELU + dropout, global /
    local / axial / conv layers and recompute_grad in one step."""
    assert not _engine_vs_oracle(256, 4, 2, 300, 64, 24, 64, 3, seed=2, recompute=True, rates=0.1, gelu=True,
                                 types=["global", "local", "axial_row", "conv"], weights=(1.0, 7.0), z=1e-3,
                                 pp=True, row_col=True, drop_caption=True)[0]


def test_dalle_example_shape_masked_step_matches_the_oracle():
    """d512 / L6 / H4 / S = 256 + 1024 / V 50 771, B = 2."""
    assert not _engine_vs_oracle(512, 6, 4, 50258, 512, 256, 1024, 2, seed=3)[0]


def test_dalle_example_shape_weighted_masked_step_matches_the_oracle():
    assert not _engine_vs_oracle(512, 2, 4, 50258, 512, 256, 1024, 2, seed=4, weights=(1.0, 7.0), z=1e-4,
                                 drop_caption=True)[0]


def test_oracle_mutants_fail_the_engine_bounds():
    """The engine's masked loss rows against the two mutated windows: each changes rows by far more than the bound."""
    from oracle import dalle as O
    from oracle import logits_mask as OM
    cfg = O.DalleConfig(256, 2, 2, 300, 64, 24, 64)
    params = O.init_params(cfg, 5)
    g = torch.Generator().manual_seed(6)
    tokens = torch.cat([torch.randint(0, 300, (2, 24), generator=g), torch.randint(300, 364, (2, 64), generator=g)], 1)
    eng = _engine(cfg, logits_mask=True)
    eng.load_params(params)
    eng.zero_grads()
    eng.forward(tokens.to(I32).to(DEV))
    eng.backward(1.0 / tokens.numel())
    torch.cuda.synchronize()
    for q in (OM.Quirks(text_rows_offset=0), OM.Quirks(eos_in_image_window=False)):
        _, rows, _, _, gq = OM.loss_and_grads(params, tokens, cfg, 300, quirks=q)
        err = relfro(eng._bufs["loss_rows"].view(2, -1), torch.nan_to_num(rows, posinf=1e30))
        assert err > 5e-3, q


# ------------------------------------------------------------------------------------------------ structure
def _small(seed=0, TL=40):
    from oracle import dalle as O
    cfg = O.DalleConfig(256, 2, 2, 300, 60, TL, 88)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    text = torch.randint(0, 300, (4, TL), generator=g)
    text[:, 20:] = 299
    tokens = torch.cat([text, torch.randint(300, 360, (4, 88), generator=g)], 1)
    return cfg, params, tokens.to(I32).to(DEV)


@pytest.mark.parametrize("weights,zero", [((0.0, 1.0), "text"), ((1.0, 0.0), "image")])
def test_a_zero_weight_class_leaves_its_window_exactly_zero(weights, zero):
    cfg, params, tok = _small(7)
    eng = _engine(cfg, logits_mask=True, loss_weights=weights)
    eng.load_params(params)
    _step(eng, tok)
    io, c0 = eng.image_offset, eng.mask_c0
    gw, gb = eng.G("wout"), eng.G("bout")
    if zero == "image":
        assert (gw[:, io:eng.V] == 0).all() and (gb[io:eng.V] == 0).all()
        assert (gw[:, :io] != 0).any()
    else:
        assert (gw[:, :io] == 0).all() and (gb[:io] == 0).all()
        assert (gw[:, io:eng.V] != 0).any()
    assert c0 < io


def test_masked_steps_are_bit_identical_and_splits_match():
    """Two masked steps bit-identical; two micro-batches and 16 reserved SMs within the plain step's criteria
    (test_loss_weights_gpu.py); TL = 1 (no text rows) runs and matches its oracle loss."""
    cfg, params, tok = _small(8)
    for kw in ({}, {"loss_weights": (1.0, 7.0), "z_loss": 1e-4}):
        eng = _engine(cfg, logits_mask=True, **kw)
        eng.load_params(params)
        a, b = _step(eng, tok), _step(eng, tok)
        assert torch.equal(a, b)
        n = eng.n_params_padded
        c = _step(eng, tok, split=2)
        assert relfro(c[:n], a[:n]) < 1e-5
        assert torch.allclose(c[eng.aux_off:eng.aux_off + 4], a[eng.aux_off:eng.aux_off + 4], rtol=1e-5, atol=0)
        with float64_bounds.reserved_sms(16):
            r = _step(eng, tok)
        assert relfro(r[:n], a[:n]) < 1e-5
        assert torch.allclose(r[eng.aux_off:eng.aux_off + 4], a[eng.aux_off:eng.aux_off + 4], rtol=1e-5, atol=0)
    from oracle import logits_mask as OM
    cfg1, params1, tok1 = _small(9, TL=1)
    eng = _engine(cfg1, logits_mask=True)
    eng.load_params(params1)
    eng.zero_grads()
    acc = eng.forward(tok1)
    eng.backward(1.0 / tok1.numel())
    torch.cuda.synchronize()
    loss, _, _, _, g32 = OM.loss_and_grads(params1, tok1.long().cpu(), cfg1, 300)
    assert abs(acc.item() / tok1.numel() - loss.item()) <= 1e-3 * loss.item()
    k = "to_logits/linear_out/kernel"
    assert relfro(eng.export_params(eng.grads)[k], g32[k]) < 3e-2


def test_unmasked_step_launches_what_it_launched_before(monkeypatch):
    """Without the key (absent or False): the vocabulary GEMMs over [T, Vpad] with n_valid = V, no partition or
    scatter, and the same launch count either way."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200 import ops as O
    cfg, params, tok = _small(10)
    calls = []
    orig = {n: getattr(O, n) for n in ("gemm", "logits_mask_partition", "logits_mask_scatter", "ce_finish")}

    def spy(name):
        def f(*a, **kw):
            calls.append((name, tuple(x for x in a if isinstance(x, int)), kw.get("mode"), kw.get("n_valid"),
                          kw.get("ldb")))
            return orig[name](*a, **kw)
        return f
    for n in orig:
        monkeypatch.setattr(O, n, spy(n))
    counts, lists = [], []
    for kw in ({}, {"logits_mask": False}, {"logits_mask": None}):
        eng = _engine(cfg, **kw)
        eng.load_params(params)
        _step(eng, tok, 1.0 / tok.numel())
        calls.clear()
        n0 = L.launch_count()
        _step(eng, tok, 1.0 / tok.numel())
        counts.append(L.launch_count() - n0)
        lists.append(list(calls))
    assert len(set(counts)) == 1 and all(x == lists[0] for x in lists), counts
    names = [c[0] for c in lists[0]]
    assert "logits_mask_partition" not in names and "logits_mask_scatter" not in names
    T = tok.numel()
    assert ("gemm", (T, eng.Vpad, cfg.n_embd), L.EPI_CE_STATS, eng.V, None) in lists[0]
    assert ("gemm", (T, eng.Vpad, cfg.n_embd), L.EPI_CE_GRAD, eng.V, None) in lists[0]
    # with the key: one partition (forward), two scatters (loss rows, dgrads), no [T, Vpad] product
    eng = _engine(cfg, logits_mask=True)
    eng.load_params(params)
    calls.clear()
    _step(eng, tok, 1.0 / T)
    names = [c[0] for c in calls]
    assert names.count("logits_mask_partition") == 1 and names.count("logits_mask_scatter") == 2
    assert not any(c[0] == "gemm" and c[1][:2] == (T, eng.Vpad) for c in calls)
    assert "dlogits" not in eng._bufs and "part_max" not in eng._bufs


# ------------------------------------------------------------------------------------------------ ranks, ZeRO-1
def test_two_in_process_ranks_equal_one_rank_with_micro_batches_bitwise(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion for the plain step (bit for bit), with the key and every feature."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    rec = _Rec(monkeypatch)
    extra = dict(FEATURES, logits_mask=True)
    W, B = 2, 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()


def test_zero1_masked_step_equals_the_replicated_step_bitwise():
    """Optimizer-state sharding over 2 loopback ranks, each on the whole batch: the gradients and the bf16 parameters
    after one masked step are those of the replicated twin, bit for bit (test_zero1_gpu.py's criterion)."""
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    cfg, params, tok = _small(11)
    kw = dict(logits_mask=True, loss_weights=(1.0, 7.0), z_loss=1e-4)
    grp = Loopback(2)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **kw) for r in range(2)]
    twin = _engine(cfg, **kw)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    _twin_from(twin, twin.master[:n].clone(), ranks[0])
    g_ref = _step(twin, tok)
    for r, e in enumerate(ranks):
        assert_same_bits(_step(e, tok), g_ref, f"ZeRO-1 rank {r} masked gradients")
    twin.optimizer_step(1e-3)
    for e in ranks:
        e.optimizer_step(1e-3)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} parameters after the step")


# ------------------------------------------------------------------------------------------------ surface
MASKED = {"logits_mask": True, "text_loss_weight": 1, "image_loss_weight": 7, "z_loss": 1e-4, "caption_dropout": 0.5,
          "padding_id": 299}


def _batch():
    g = torch.Generator().manual_seed(3)
    return torch.rand(4, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (4, 12), generator=g)


def _masked_rows(logits, toks, eng, weights=None, z=0.0):
    from oracle import logits_mask as OM
    labels = torch.cat([toks[:, 1:], torch.full_like(toks[:, :1], eng.eos_token_id)], 1).long().cpu()
    return OM.masked_loss(logits, labels, eng.text_seq_len, eng.image_seq_len, eng.image_offset, weights, z)


def test_model_fn_and_dalle_report_the_masked_loss_and_minus_inf_logits(tmp_path):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.models import DALLE
    img, cap = _batch()
    spec = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **MASKED))
    assert spec.engine.logits_mask
    loss = spec.train_op(img, cap).item()
    assert math.isfinite(loss) and spec.loss_parts.shape == (3,)
    ev = dalle_model_fn(img, cap, "eval", _tiny_params(tmp_path, **MASKED))
    el = ev.eval_op(img, cap).item()
    eng = ev.engine
    toks = ev.assemble(img, cap).clone()
    logits = eng.logits(toks)
    nt, io = eng.text_rows, eng.image_offset
    assert torch.isinf(logits[:, :nt, io:]).all() and (logits[:, :nt, io:] < 0).all()
    assert torch.isinf(logits[:, nt:, :io]).all() and torch.isfinite(logits[:, :nt, :io]).all()
    assert torch.isfinite(logits[:, nt:, io:]).all()
    ref, rows, parts = _masked_rows(logits.double().cpu(), toks, eng, (1.0, 7.0), 1e-4)
    assert math.isclose(el, ref.item(), rel_tol=1e-4), (el, ref.item())
    ev.eval_op(img, cap)
    assert relfro(eng._bufs["loss_rows"].view(4, -1), rows) < 1e-4
    for a, b in zip(ev.loss_parts.tolist(), parts):
        assert math.isclose(a, b.item(), rel_tol=1e-4, abs_tol=1e-7)
    # DALLE.forward: the masked loss, loss_batch in [B, S] order, -inf logits outside the windows
    m = DALLE(256, text_vocab_size=300, image_vocab_size=60, text_seq_len=40, image_seq_len=88, n_layers=1, n_heads=2,
              mode="eval", params={"logits_mask": True})
    g = torch.Generator().manual_seed(9)
    tokens = torch.cat([torch.randint(0, 300, (2, 40), generator=g), torch.randint(300, 360, (2, 88), generator=g)], 1)
    loss, loss_batch, lg = m.forward({"tokens": tokens}, return_logits=True)
    ref, rows, _ = _masked_rows(lg.double().cpu(), tokens, m.engine)
    assert loss_batch.shape == (2, 128)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-4) and relfro(loss_batch, rows) < 1e-4
    assert torch.isinf(m.forward({"tokens": tokens}, return_loss=False)[:, :39, 300:]).all()
    with pytest.raises(ValueError, match="logits_mask"):
        dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, logits_mask="yes"))


def test_checkpoint_has_the_same_names_and_resumes_bit_exactly(tmp_path):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    img, cap = _batch()
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    masked = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **MASKED))
    masked.train_op(img, cap)
    st = masked.state_fn()
    ps = plain.state_fn()
    assert {k: tuple(v.shape) for k, v in st.items() if k != "global_step"} == \
        {k: tuple(v.shape) for k, v in ps.items() if k != "global_step"}
    a = masked.train_op(img, cap).clone()
    sa = [t.clone() for t in (masked.engine.master, masked.engine.adam_m, masked.engine.adam_v)]
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **MASKED))
    resumed.load_fn(st)
    b = resumed.train_op(img, cap)
    assert torch.equal(a, b)
    for x, y in zip(sa, (resumed.engine.master, resumed.engine.adam_m, resumed.engine.adam_v)):
        assert torch.equal(x, y)
    plain.load_fn(st)                          # and the plain model loads it too
    plain.eval_op(img, cap)


def test_greedy_generation_is_the_argmax_of_the_masked_forward():
    """Greedy sample and complete of a masked model follow the argmax over the image ids of the masked full forward
    pass, with test_prefill_gpu.py's criterion (every token where the top-2 margin is clear)."""
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward, sharp_engine
    eng, _, _ = sharp_engine(256, 2, 2, 300, 64, 16, 64, logits_mask=True)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, 299, (3, 16), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    out = smp.generate(text, 0.0)
    greedy_agrees_with_full_forward(eng, out, 16)
    assert torch.isinf(eng.logits(out)[:, 15:, :300]).all()
    done = smp.complete(text, out[:, 16:24].contiguous() - eng.image_offset, temperature=0)
    greedy_agrees_with_full_forward(eng, done, 24)


def test_generate_cli_runs_on_a_tiny_masked_model(tmp_path):
    """generate_dalle.py end to end on a tiny masked model trained one step and checkpointed."""
    import json
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from dalle_mtf_b200.utils import save_checkpoint
    img, cap = _batch()
    p = _tiny_params(tmp_path, **MASKED)
    spec = dalle_model_fn(img, cap, "train", p)
    spec.train_op(img, cap)
    vae = spec.extra["vae"]
    save_checkpoint(str(tmp_path / "vae"), 1, {"vae/" + k: v for k, v in vae.export_params().items()})
    save_checkpoint(str(tmp_path / "dalle"), 1, spec.state_fn())
    vcfg = dict(p["vae_params"], model_path=str(tmp_path / "vae"))
    (tmp_path / "vae.json").write_text(json.dumps(vcfg))
    cfg = {k: v for k, v in p.items() if k != "vae_params"}
    cfg.update(vae_model=str(tmp_path / "vae.json"), model_path=str(tmp_path / "dalle"), predict_batch_size=2)
    (tmp_path / "masked.json").write_text(json.dumps(cfg))
    np.save(tmp_path / "ids.npy", np.array([[1, 2, 3] + [299] * 9, [4, 5] + [299] * 10], dtype=np.int64))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "masked.json"), "--caption_ids", str(tmp_path / "ids.npy"),
                         "--out", str(out), "--temperature", "0"])
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (2, spec.engine.S) and len(list(out.glob("*.png"))) == 2
    io = spec.engine.image_offset
    assert ((toks[:, 12:] >= io) & (toks[:, 12:] < io + 64)).all()
