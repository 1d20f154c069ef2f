"""GPU tests of image-prompted generation: the prefill hand-off kernels (db200_kv_cache_fill, db200_rows_repeat),
DalleEngine.prefill against the teacher-forced decode path and the fp32 oracle, DalleSampler.complete / DALLE.complete,
and generate_dalle.py end to end on a tiny VAE + DALL-E pair."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def relfro(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import ops as o
    return o


# the tiny engines of test_sampling_gpu.py (dh 128 and 64), each with an odd prompt length P
SHAPES = [(256, 2, 2, 300, 64, 24, 40, 3, 29), (256, 2, 4, 500, 100, 70, 90, 2, 77)]


def sharp_engine(d, L, H, tv, iv, ts, isl, **kw):
    """Oracle-initialised engine with sharpened weights (clear arg-maxima), as in test_sampling_gpu.py.  With the
    image_position_embedding / per_position_padding keywords the parameters are oracle/dalle_input.py's."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from oracle import dalle as O
    from oracle import dalle_input as I
    cfg = O.DalleConfig(d, L, H, tv, iv, ts, isl)
    pp = bool(kw.get("per_position_padding"))
    inp = I.InputConfig(kw.get("image_position_embedding") or "absolute", pp, tv - 1 if pp else None)
    params = I.init_params(cfg, inp, 3)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        if "wte" in k or "wout" in k or k.endswith("kernel"):
            params[k] = params[k] * 4
    eng = DalleEngine(d, L, H, tv, iv, ts, isl, **kw)
    eng.load_params(params)
    return eng, params, cfg


# ------------------------------------------------------------------------------------------------ hand-off kernels
@pytest.mark.parametrize("rep", [1, 3])
@pytest.mark.parametrize("B,P,S,H,dh", [(3, 29, 40, 2, 128), (2, 77, 90, 4, 64)])
def test_kv_cache_fill_and_rows_repeat_equal_indexing(ops, rep, B, P, S, H, dh):
    g = torch.Generator().manual_seed(P + rep)
    qkv = torch.randn(B, P, 3, H, dh, generator=g).to(torch.bfloat16)
    kc = torch.full((B * rep, S, H, dh), 7.0, dtype=torch.bfloat16, device=DEV)
    vc = torch.full_like(kc, -7.0)
    ops.kv_cache_fill(qkv.to(DEV).view(B * P, 3 * H * dh), kc, vc, P, rep)
    want_k = torch.full((B, rep, S, H, dh), 7.0, dtype=torch.bfloat16)
    want_v = torch.full_like(want_k, -7.0)
    want_k[:, :, :P] = qkv[:, None, :, 1]
    want_v[:, :, :P] = qkv[:, None, :, 2]
    assert torch.equal(kc.cpu(), want_k.view(B * rep, S, H, dh))        # positions >= P keep the sentinel
    assert torch.equal(vc.cpu(), want_v.view(B * rep, S, H, dh))
    d = H * dh
    x = torch.randn(B, P, d, generator=g).to(torch.bfloat16).to(DEV)
    out = torch.empty(B * rep, d, dtype=torch.bfloat16, device=DEV)
    ops.rows_repeat(x[:, P - 1], out, rep)
    assert torch.equal(out.cpu(), x[:, P - 1].cpu().repeat_interleave(rep, 0))


def test_hand_off_kernels_reject_bad_arguments():
    from dalle_mtf_b200 import lib as L
    lib = L.load()
    L.require_device()
    s = L.stream_ptr()
    B, P, S, H, dh = 2, 5, 8, 2, 64
    qkv = torch.zeros(B * P * 3 * H * dh + 64, dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros(B * S * H * dh + 64, dtype=torch.bfloat16, device=DEV)
    vc = torch.zeros_like(kc)
    q, k, v = qkv.data_ptr(), kc.data_ptr(), vc.data_ptr()
    assert lib.db200_kv_cache_fill(s, q, k, v, B, P, H, dh, S, 1) == 0
    for args in ((B, S + 1, H, dh, S, 1), (B, P, H, dh, S, 0), (0, P, H, dh, S, 1), (B, P, H, 0, S, 1)):
        assert lib.db200_kv_cache_fill(s, q, k, v, *args) == -1, args          # DB200_E_INVALID
    assert lib.db200_kv_cache_fill(s, q + 2, k, v, B, P, H, dh, S, 1) == -2    # DB200_E_ALIGN
    assert lib.db200_kv_cache_fill(s, q, k, v + 2, B, P, H, dh, S, 1) == -2
    with pytest.raises(L.DB200Error):
        L.check(lib.db200_kv_cache_fill(s, q, None, v, B, P, H, dh, S, 1), "kv_cache_fill")
    assert lib.db200_rows_repeat(s, q, P * 128, k, B, 128, 3) == 0
    assert lib.db200_rows_repeat(s, q, P * 128, k, B, 128, 0) == -1
    assert lib.db200_rows_repeat(s, q, 64, k, B, 128, 1) == -1                  # rows overlap: ld < d
    assert lib.db200_rows_repeat(s, q, P * 128 + 4, k, B, 128, 1) == -2
    assert lib.db200_rows_repeat(s, q, P * 128, k + 2, B, 128, 1) == -2
    with pytest.raises(L.DB200Error):
        L.check(lib.db200_rows_repeat(s, q, P * 128, k, B, 128, -1), "rows_repeat")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ prefill
@pytest.mark.parametrize("d,L,H,tv,iv,ts,isl,B,P", SHAPES)
def test_prefill_matches_teacher_forcing_and_the_oracle(d, L, H, tv, iv, ts, isl, B, P):
    from dalle_mtf_b200.sampling import DalleSampler
    from oracle import dalle as O
    eng, params, cfg = sharp_engine(d, L, H, tv, iv, ts, isl)
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, tv, (B, ts), generator=g).to(torch.int32).cuda()
    smp = DalleSampler(eng)
    toks = smp.generate(text, temperature=0)            # teacher-forced caches of every position of toks
    kc = [torch.zeros_like(c) for c in smp.kc]
    vc = [torch.zeros_like(c) for c in smp.vc]
    logits = eng.prefill(toks[:, :P].contiguous(), kc, vc).clone()
    torch.cuda.synchronize()
    # layer 0: embedding, LayerNorm and the q|k|v GEMM do the same per-row arithmetic at any row count
    assert torch.equal(kc[0][:, :P], smp.kc[0][:, :P]) and torch.equal(vc[0][:, :P], smp.vc[0][:, :P])
    for i in range(1, L):   # deeper layers see attention outputs: flash attention vs the decode kernel
        assert relfro(kc[i][:, :P], smp.kc[i][:, :P]) <= 1e-2, i
        assert relfro(vc[i][:, :P], smp.vc[i][:, :P]) <= 1e-2, i
    for c in kc + vc:
        assert not c[:, P:].any()                        # nothing written past the prompt
    full = eng.logits(toks)
    assert relfro(logits[:, :eng.V], full[:, P - 1]) < 2e-2
    _, _, logits32, _ = O.loss_and_grads(params, toks.cpu().long(), cfg, bf16=False)
    assert relfro(logits[:, :eng.V], logits32[:, P - 1]) < 3e-2
    # replicas: rep copies of each prompt's caches and logits
    kc3 = [torch.zeros(B * 3, *c.shape[1:], dtype=c.dtype, device=DEV) for c in kc]
    vc3 = [torch.zeros_like(c) for c in kc3]
    logits3 = eng.prefill(toks[:, :P].contiguous(), kc3, vc3, rep=3)
    assert torch.equal(logits3, logits.repeat_interleave(3, 0))
    for a, b in zip(kc3 + vc3, kc + vc):
        assert torch.equal(a, b.repeat_interleave(3, 0))
    with pytest.raises(ValueError):
        eng.prefill(toks, kc, vc)                        # P = S: nothing left to predict
    with pytest.raises(ValueError):
        eng.prefill(toks[:, :P].contiguous(), kc3, vc3)  # caches sized for another row count


def test_prefill_between_forward_and_backward_leaves_the_gradients_alone():
    d, L, H, tv, iv, ts, isl, B, P = SHAPES[0]
    eng, _, _ = sharp_engine(d, L, H, tv, iv, ts, isl, dropout=(0.1, 0.1, 0.1), dropout_seed=5)
    g = torch.Generator().manual_seed(6)
    toks = torch.randint(0, tv + iv, (B, ts + isl), generator=g).to(torch.int32).cuda()
    kc = [torch.zeros(B, ts + isl, H, d // H, dtype=torch.bfloat16, device=DEV) for _ in range(L)]
    vc = [torch.zeros_like(c) for c in kc]
    T = toks.numel()
    eng.zero_grads()
    eng.forward(toks, step=3)
    eng.backward(1.0 / T)
    ref = eng.grads.clone()
    eng.zero_grads()
    eng.forward(toks, step=3)
    eng.prefill(toks[:, :P].contiguous(), kc, vc, rep=1)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    assert torch.equal(eng.grads, ref)


# ------------------------------------------------------------------------------------------------ complete
def greedy_agrees_with_full_forward(eng, out, P):
    """Every sampled token equals the full forward pass's argmax wherever its top-2 margin is clear (the criterion of
    test_sampling_gpu.py)."""
    io, iv, S = eng.image_offset, eng.image_vocab_size, eng.S
    full = eng.logits(out)
    if iv == 1:   # one image code: every draw is it
        assert (out[:, P:] == io).all()
        return
    rng = full[:, P - 1:S - 1, io:io + iv]
    top2 = rng.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 0.05 * rng.abs().max()
    same = (rng.argmax(-1) + io) == out[:, P:]
    assert (same | ~clear).all() and clear.float().mean() > 0.2 and same.float().mean() > 0.8


@pytest.mark.parametrize("d,L,H,tv,iv,ts,isl,B,P", SHAPES)
def test_complete_greedy_follows_the_model(d, L, H, tv, iv, ts, isl, B, P):
    from dalle_mtf_b200.sampling import DalleSampler
    eng, _, _ = sharp_engine(d, L, H, tv, iv, ts, isl)
    g = torch.Generator().manual_seed(8)
    text = torch.randint(0, tv, (B, ts), generator=g).to(torch.int32).cuda()
    n = P - ts
    prefix = torch.randint(0, iv, (B, n), generator=g).to(torch.int32).cuda()
    smp = DalleSampler(eng)
    for pre, p in ((None, ts), (prefix, P)):
        out = smp.complete(text, pre, temperature=0)
        assert out.shape == (B, ts + isl) and out.dtype == torch.int32
        assert torch.equal(out[:, :ts], text)
        if pre is not None:
            assert torch.equal(out[:, ts:P], prefix + tv)                      # the prefix comes back verbatim
        assert ((out[:, p:] >= tv) & (out[:, p:] < tv + iv)).all()
        greedy_agrees_with_full_forward(eng, out, p)
    # greedy replicas are the prompts repeated, bit for bit
    rep = 3
    many = smp.complete(text, prefix, samples_per_prompt=rep, temperature=0)
    assert torch.equal(many, smp.complete(text.repeat_interleave(rep, 0), prefix.repeat_interleave(rep, 0),
                                          temperature=0))
    # top-1 and a tiny nucleus keep only the maximum: sampling with noise then equals greedy
    greedy = smp.complete(text, prefix, temperature=0)
    assert torch.equal(smp.complete(text, prefix, temperature=1.0, top_k=1), greedy)
    assert torch.equal(smp.complete(text, prefix, temperature=1.0, top_p=1e-6), greedy)


def test_complete_sampling_is_seeded_and_filtered():
    from dalle_mtf_b200.sampling import DalleSampler
    d, L, H, tv, iv, ts, isl, B, P = SHAPES[0]
    eng, _, _ = sharp_engine(d, L, H, tv, iv, ts, isl)
    smp = DalleSampler(eng)
    g = torch.Generator().manual_seed(10)
    text = torch.randint(0, tv, (B, ts), generator=g).to(torch.int32).cuda()
    prefix = torch.randint(0, iv, (B, P - ts), generator=g).to(torch.int32).cuda()
    torch.manual_seed(11)
    a = smp.complete(text, prefix, samples_per_prompt=4, temperature=1.5)
    torch.manual_seed(11)
    b = smp.complete(text, prefix, samples_per_prompt=4, temperature=1.5)
    assert torch.equal(a, b)
    assert a.shape == (B * 4, ts + isl)
    assert torch.equal(a[:, :P], torch.cat([text, prefix + tv], 1).repeat_interleave(4, 0))
    img = a[:, P:].view(B, 4, -1)
    for bi in range(B):                                   # independent noise per replica
        assert len({tuple(r.tolist()) for r in img[bi]}) > 1
    # top-k: every sampled id lies in the top k of the full forward pass's distribution at its position
    k = 3
    out = smp.complete(text, prefix, samples_per_prompt=2, temperature=2.0, top_k=k)
    full = eng.logits(out)[:, P - 1:-1, tv:tv + iv]
    kth = full.topk(k, -1).values[..., -1:]
    chosen = full.gather(-1, (out[:, P:] - tv).long()[..., None])
    # the full forward's logits differ from the decode step's by bf16 rounding: allow that much slack at the threshold
    assert (chosen >= kth - 0.02 * full.abs().max()).all()


def test_complete_rejects_bad_arguments():
    from dalle_mtf_b200.sampling import DalleSampler
    d, L, H, tv, iv, ts, isl, B, P = SHAPES[0]
    eng, _, _ = sharp_engine(d, L, H, tv, iv, ts, isl)
    smp = DalleSampler(eng)
    text = torch.zeros(B, ts, dtype=torch.int32, device=DEV)
    pre = torch.zeros(B, 4, dtype=torch.int32, device=DEV)
    bad = [
        dict(text_ids=text[:, :-1]),                                              # text shape
        dict(text_ids=text[0]),
        dict(text_ids=text, image_prefix=pre[:1]),                                # prefix batch
        dict(text_ids=text, image_prefix=pre[0]),
        dict(text_ids=text, image_prefix=pre[:, :0]),                             # n = 0
        dict(text_ids=text, image_prefix=torch.zeros(B, isl, dtype=torch.int32, device=DEV)),   # n = image_seq_len
        dict(text_ids=text, image_prefix=pre - 1),                                # code < 0
        dict(text_ids=text, image_prefix=pre + iv),                               # code >= image_vocab_size
        dict(text_ids=text, samples_per_prompt=0),
        dict(text_ids=text, samples_per_prompt=1.5),
        dict(text_ids=text, top_k=0),
        dict(text_ids=text, top_p=0.0),
        dict(text_ids=text, top_p=1.5),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            smp.complete(**kw)


def test_dalle_model_class_complete():
    from dalle_mtf_b200.models import DALLE
    m = DALLE(256, text_vocab_size=200, image_vocab_size=32, text_seq_len=8, image_seq_len=16, n_layers=1, n_heads=2)
    text = torch.randint(0, 200, (2, 8), dtype=torch.int32)
    prefix = torch.randint(0, 32, (2, 5), dtype=torch.int32)
    out = m.complete(text, prefix, samples_per_prompt=2, temperature=0.0)
    assert out.shape == (4, 24)
    assert torch.equal(out[:, :8].cpu(), text.repeat_interleave(2, 0))
    assert torch.equal(out[:, 8:13].cpu(), prefix.repeat_interleave(2, 0) + 200)
    assert ((out[:, 13:] >= 200) & (out[:, 13:] < 232)).all()


# ------------------------------------------------------------------------------------------------ command
def test_generate_dalle_end_to_end(tmp_path):
    import generate_dalle
    from PIL import Image
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.data_pipeline import device_stage, host_stage
    from dalle_mtf_b200.utils import save_checkpoint
    from dalle_mtf_b200.vae_engine import VaeEngine
    from concurrent.futures import ThreadPoolExecutor

    size, convblocks, K = 32, [[2, 64], [2, 128]], 64
    tv, ts = 300, 12
    vae_cfg = {"model_type": "vae", "dataset": {"image_size": size}, "num_tokens": K, "convblocks": convblocks,
               "model_path": str(tmp_path / "vae_run"), "use_bf16": True}
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": size}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts,
                 "vae_model": str(tmp_path / "vae.json")}
    (tmp_path / "vae.json").write_text(json.dumps(vae_cfg))
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    # checkpoints under the keys the model functions' state_fn write
    vae = VaeEngine(K, size, convblocks, 3, True, False, 1)
    vae.init_params(4)
    st = {"vae/" + k: v for k, v in vae.export_params().items()}
    st.update({"vae/" + k + "/Adam": v for k, v in vae.export_params(vae.adam_m).items()})
    st.update({"vae/" + k + "/Adam_1": v for k, v in vae.export_params(vae.adam_v).items()})
    st["global_step"] = 7
    save_checkpoint(vae_cfg["model_path"], 7, st)
    hw = size // 4
    eng = DalleEngine(256, 2, 2, tv, K, ts, hw * hw)
    eng.init_params(5)
    st = dict(eng.export_params())
    st.update({k + "/adam_m": v for k, v in eng.export_params(eng.adam_m).items()})
    st.update({k + "/adam_v": v for k, v in eng.export_params(eng.adam_v).items()})
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)

    g = np.random.default_rng(0)
    Image.fromarray(g.integers(0, 256, (48, 48, 3), dtype=np.uint8)).save(tmp_path / "prompt.png")
    np.save(tmp_path / "caps.npy", g.integers(0, tv, (3, ts)).astype(np.int32))
    out = tmp_path / "out"
    rows = 3
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out),
                         "--caption_ids", str(tmp_path / "caps.npy"), "--image_prompt", str(tmp_path / "prompt.png"),
                         "--prompt_rows", str(rows), "--samples_per_prompt", "2", "--seed", "1"])
    pngs = sorted(p for p in os.listdir(out) if p.endswith(".png"))
    assert pngs == [f"{c:05d}_{s:02d}.png" for c in range(3) for s in range(2)]
    for p in pngs:
        assert Image.open(out / p).size == (size, size)
    toks = np.load(out / "tokens.npy")
    assert toks.shape == (6, ts + hw * hw) and toks.dtype == np.int32
    assert (toks[:, :ts] == np.repeat(np.load(tmp_path / "caps.npy"), 2, 0)).all()
    # the prefix is the prompt image's first rows of codes (training input transform + encoder), offset by tv
    params = generate_dalle.load_params(str(tmp_path / "dalle.json"))
    with ThreadPoolExecutor(1) as pool:
        hb = host_stage([str(tmp_path / "prompt.png")], params, labeled=False, tfrecords=False, pool=pool)
    codes = vae.encode_tokens(device_stage(hb, params, torch.device(DEV))).cpu().numpy()
    n = rows * hw
    assert (toks[:, ts:ts + n] == codes[:, :n] + tv).all()
    assert ((toks[:, ts + n:] >= tv) & (toks[:, ts + n:] < tv + K)).all()
