"""GPU tests of Gumbel-quantised VQGANs ("quantizer": "gumbel", taming's GumbelVQ) and of the long-sequence attention
kernel their 32 x 32 grids need: the kernel against float64 at every (S, C) the Gumbel geometries launch and at the
edges of its range, its reproducibility, the engine's codes and decoded images against oracle/vqgan.py, a launch census
at the f8 geometry, and the DALL-E boundary.

Bounds, eps = 2^-24 (f32 roundoff), bf16 outputs with half a bf16 ulp at |ref| (tests/float64_bounds.py):
  * long attention (db200_attn_noncausal_long_fwd): a score s_ij = scale sum_c q_c k_c of exact bf16 products summed
    on the tensor cores (each step may truncate: 2^-23) in two halves added in f32, then scaled by scale log2(e) in f32,
    is within e_ij = (C + 4) 2^-23 scale sum_c |q_c k_c| of exact; the softmax weights then move by at most
    2 max_j e_ij + 8 eps relative.  The online softmax rescales the running sums once per 64-key tile (exp2f and a
    multiply, 4 eps each), S / 16 eps in all.  The weights are rounded to bf16 for P v, at most 2^-8 relative each (half
    a bf16 ulp of a value in [2^e, 2^(e+1)) is 2^(e-8)), while the row sum uses the unrounded weights; the weighted sum
    is accumulated on the tensor cores, (S + 2) 2^-23.  So |do_i| <= (2 max_j e_ij + 2^-8 + (S / 16 + S + 10) 2^-23)
    sum_j p_ij |v_j|;
  * GroupNorm at the widths the f8 geometry adds: test_vqgan_gpu.py's bounds;
  * codes: see test_gumbel_codes_agree_with_the_oracle_where_the_gap_decides_them;
  * decoded images: L 2^-9 relative as in test_vqgan_gpu.py, L the decoder's bf16 roundings on its longest path.
"""
import json

import pytest
import torch

import float64_bounds as FB
import test_vqgan_gpu as V
from dalle_mtf_b200 import ops
from oracle import vqgan as O
from oracle import vqgan_gumbel as OG

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
UTC = 2.0 ** -23
F64 = torch.float64
GEOS = {"gumbel_f8": OG.GEOMETRY_GUMBEL_F8, "gumbel_test": OG.GEOMETRY_GUMBEL_TEST}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _engine(geo):
    from dalle_mtf_b200.vqgan_engine import VqganEngine
    return VqganEngine(geo["num_tokens"], geo["resolution"], geo["ch"], geo["ch_mult"], geo["num_res_blocks"],
                       geo["attn_resolutions"], geo["z_channels"], geo["embed_dim"], quantizer=geo["quantizer"])


def long_attention_reference(qkv, C, scale):
    """float64 reference and per-element tolerance (the module docstring's bound) of the long attention for the
    bf16 q | k | v [B, S, 3C] the kernel reads: (ref, coef * sum_j p_ij |v_j|)."""
    qd, kd, vd = (t.to(F64) for t in qkv.split(C, -1))
    S = qd.shape[1]
    p = torch.softmax(scale * qd @ kd.transpose(1, 2), -1)
    e = (C + 4) * UTC * scale * (qd.abs() @ kd.abs().transpose(1, 2))
    coef = 2 * e.amax(-1, keepdim=True) + 8 * EPS + 2.0 ** -8 + (S / 16 + S + 10) * UTC
    return p @ vd, coef * (p @ vd.abs())


def _attn_inputs(B, S, C, seed):
    """Rows of ordinary, large (|scores| up to ~50, nearly one-hot weights) and near-uniform scores, as
    test_vqgan_gpu.py's attention test."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, S, C, generator=g, device=DEV)
    q[:, 1::3] *= 12.0 * C ** -0.25
    q[:, 2::3] *= 1e-3
    k, v = torch.randn(B, S, C, generator=g, device=DEV), torch.randn(B, S, C, generator=g, device=DEV)
    return torch.cat([q, k, v], -1).to(torch.bfloat16).contiguous()


def _long_shapes(geo):
    return {(S, C) for S, C in V._shapes(geo)[1] if S > 256}


LONG_SHAPES = sorted(set().union(*(_long_shapes(g) for g in GEOS.values())) | {(320, 512), (4096, 512)})
LONG_CASES = [(S, C, B) for S, C in LONG_SHAPES for B in (1, V.TOKENIZE_B, 64)]


@pytest.mark.parametrize("S,C,B", LONG_CASES)
def test_long_attention_against_float64(S, C, B):
    qkv = _attn_inputs(B, S, C, S + C + B)
    out = torch.full((B, S, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    scale = C ** -0.5
    ops.attn_noncausal_long(qkv, out, B, S, C, scale)
    worst = 0.0
    step = max(1, 2 ** 26 // (S * S))             # float64 score matrices of at most 512 MiB at once
    for i in range(0, B, step):
        ref, tol = long_attention_reference(qkv[i:i + step], C, scale)
        worst = max(worst, FB.worst_ratio(f"attn_noncausal_long S={S} C={C} B={B}", out[i:i + step], ref, tol,
                                          a=0, b=1.0, bf16_out=True))
    FB.report(f"attn_noncausal_long S={S} C={C} B={B}", worst)


def test_long_attention_refuses_what_it_does_not_cover():
    from dalle_mtf_b200 import lib as L
    for S, C in ((256, 512), (4160, 512), (1024, 256), (352, 512), (1024, 576)):
        qkv = torch.zeros(1, S, 3 * C, dtype=torch.bfloat16, device=DEV)
        with pytest.raises(L.DB200Error, match="code -4"):
            ops.attn_noncausal_long(qkv, torch.empty(1, S, C, dtype=torch.bfloat16, device=DEV), 1, S, C, 1.0)


def test_long_attention_is_reproducible_and_independent_of_the_batch():
    S, C, B = 1024, 512, V.TOKENIZE_B
    qkv = _attn_inputs(B, S, C, 11)
    a, b = (torch.empty(B, S, C, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    ops.attn_noncausal_long(qkv, a, B, S, C, C ** -0.5)
    ops.attn_noncausal_long(qkv, b, B, S, C, C ** -0.5)
    assert torch.equal(a, b)
    for i in (0, 5, B - 1):
        one = torch.empty(1, S, C, dtype=torch.bfloat16, device=DEV)
        ops.attn_noncausal_long(qkv[i:i + 1].contiguous(), one, 1, S, C, C ** -0.5)
        assert torch.equal(one, a[i:i + 1])


GN_NEW = sorted({(r, C) for g in GEOS.values() for r, C in V._shapes(g)[0]} - V.GN_SHAPES)


@pytest.mark.parametrize("res,C", GN_NEW)
@pytest.mark.parametrize("swish", [False, True])
def test_groupnorm_at_the_gumbel_widths_against_float64(res, C, swish):
    for B in (1, 3):
        V._check_groupnorm(res, C, B, swish, 1.5, 3.0)
    V._check_groupnorm(res, C, 2, False, 64.0, 0.5)


# ------------------------------------------------------------------------------------------------------ engine
def _setup(gname, seed=0, edit=None):
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    geo = GEOS[gname]
    sd = OG.random_state_dict(geo, seed)
    if edit is not None:
        edit(sd)
    eng = _engine(geo)
    eng.load_params(import_taming_state_dict(sd, geo))
    return geo, sd, eng


def gumbel_decided(sd, z_ref, z_eng):
    """(oracle codes, rows the oracle's logit gap decides) for latent rows z [rows, D] (float64, CPU).  Code b beats
    code n by gap_bn = l_b - l_n; the engine's z moves it by at most ||dz|| ||w_b - w_n|| and the logits' split-product
    rounding (3 2^-16 sum_c |z_c w_nc| for the dropped lo x lo product and the splits' residuals, (D + 2) 2^-23 of it
    for the f32 sums and the bias) by that much again for each of the two codes."""
    w = sd["quantize.proj.weight"][:, :, 0, 0].to(F64).cpu()
    lg = OG.logits({k: v.to(F64).cpu() for k, v in sd.items() if k.startswith("quantize.")}, z_ref)
    two = lg.topk(2, dim=1)
    best = two.indices[:, 0]
    sq = (w * w).sum(1)
    spread = (sq[best][:, None] + sq[None, :] - 2 * w[best] @ w.T).clamp_min(0).sqrt().amax(-1)
    D = w.shape[1]
    rnd = 2 * (3 * 2.0 ** -16 + (D + 2) * 2.0 ** -23) * (z_ref.abs() @ w.abs().T).amax(-1)
    dz = (z_eng - z_ref).norm(dim=-1)
    return best, two.values[:, 0] - two.values[:, 1] > 2 * dz * spread + rnd


@pytest.mark.parametrize("gname,B", [("gumbel_test", 4), ("gumbel_f8", 2)])
def test_gumbel_codes_agree_with_the_oracle_where_the_gap_decides_them(gname, B):
    """Codes are the argmax of the logits z . proj_n + bias_n (the mode of taming's draw).  Rows whose oracle gap
    exceeds what the engine's z error and the split-product rounding can move must agree; the others are reported."""
    geo, sd, eng = _setup(gname)
    img = V._images(B, geo["resolution"], 1)
    codes = eng.encode_tokens(img.to(DEV)).clone().cpu().long().view(-1)
    assert codes.numel() == B * 1024
    z_eng = eng._b["z"].double().cpu()
    z_ref = O.encode_z(O.to(sd, F64, DEV), geo, img.to(DEV, F64)).reshape(-1, geo["embed_dim"]).cpu()
    best, decided = gumbel_decided(sd, z_ref, z_eng)
    print(f"[vqgan-gumbel] {gname} B={B}: {int((~decided).sum())} of {decided.numel()} rows excluded (gap below the "
          f"bound)")
    assert decided.any()
    assert torch.equal(codes[decided], best[decided])
    rel = ((z_eng - z_ref).norm() / z_ref.norm()).item()
    bound = V._encoder_roundings(geo) * 2.0 ** -9
    print(f"[vqgan-gumbel] {gname}: z rel-fro {rel:.3e} (bound {bound:.3e})")
    assert rel < bound
    own, own_ok = gumbel_decided(sd, z_eng, z_eng)
    assert own_ok.any() and torch.equal(codes[own_ok], own[own_ok])


def test_gumbel_codes_take_the_first_of_tied_logits():
    """A proj whose odd rows and biases repeat the even ones before them: every logit ties in pairs, and the engine
    must return the first (even) index, as torch.argmax does."""
    def tie(sd):
        sd["quantize.proj.weight"][1::2] = sd["quantize.proj.weight"][0::2]
        sd["quantize.proj.bias"][1::2] = sd["quantize.proj.bias"][0::2]
    geo, _, eng = _setup("gumbel_test", 8, tie)
    codes = eng.encode_tokens(V._images(4, geo["resolution"], 6).to(DEV)).clone().cpu()
    print(f"[vqgan-gumbel] ties: {len(set(codes.view(-1).tolist()))} distinct codes, all must be even")
    assert (codes % 2 == 0).all()


@pytest.mark.parametrize("gname", ["gumbel_test", "gumbel_f8"])
def test_gumbel_codes_are_reproducible_and_independent_of_the_batch(gname):
    geo, _, eng = _setup(gname, 5)
    img = V._images(V.TOKENIZE_B, geo["resolution"], 4).to(DEV)
    a = eng.encode_tokens(img).clone()
    assert torch.equal(eng.encode_tokens(img).clone(), a)
    for i in (0, 7, V.TOKENIZE_B - 1):
        assert torch.equal(eng.encode_tokens(img[i:i + 1].contiguous()).clone(), a[i:i + 1])


@pytest.mark.parametrize("gname,B", [("gumbel_test", 3), ("gumbel_f8", 2)])
def test_gumbel_decode_tokens_against_the_oracle(gname, B):
    geo, sd, eng = _setup(gname, 6)
    codes = torch.randint(0, geo["num_tokens"], (B, eng.image_seq_len), generator=torch.Generator().manual_seed(9))
    off = 1000
    got = eng.decode_tokens((codes + off).to(torch.int32).to(DEV), offset=off).clone()
    ref = OG.decode(O.to(sd, F64, DEV), geo, codes.to(DEV))
    rel = ((got.double() - ref).norm() / ref.norm()).item()
    bound = V._decoder_roundings(geo) * 2.0 ** -9
    print(f"[vqgan-gumbel] {gname} decode B={B}: rel-fro {rel:.3e} (bound {bound:.3e})")
    assert rel < bound and got.abs().max() <= 1
    one = torch.cat([eng.decode_tokens((codes[i:i + 1] + off).to(torch.int32).to(DEV), offset=off).clone()
                     for i in range(B)])
    assert torch.equal(one, got)


# ------------------------------------------------------------------------------------------------------ census
def _describe(entry, A):
    import launch_census as LC
    if entry == "attn_noncausal_long":
        return LC.launch_class(entry, S=A["S"], C=A["C"], B=A["B"]), None
    return V._describe(entry, A)


GN_ALL = V.GN_SHAPES | set(GN_NEW)
CHECKERS = [
    ("test_groupnorm_against_float64", lambda c: c[0] == "groupnorm" and (V.LCf(c)["res"], V.LCf(c)["C"]) in V.GN_SHAPES),
    ("test_groupnorm_at_the_gumbel_widths_against_float64",
     lambda c: c[0] == "groupnorm" and (V.LCf(c)["res"], V.LCf(c)["C"]) in GN_ALL),
    ("test_long_attention_against_float64",
     lambda c: c[0] == "attn_noncausal_long" and (V.LCf(c)["S"], V.LCf(c)["C"]) in set(LONG_SHAPES)),
] + [ck for ck in V.CHECKERS if ck[0] not in ("test_groupnorm_against_float64", "test_attention_against_float64")]
PRESENT = {"test_groupnorm_at_the_gumbel_widths_against_float64", "test_long_attention_against_float64"} | \
    {n for n, _ in V.CHECKERS}


def test_launch_census_of_gumbel_f8_encode_and_decode():
    """Encoding a batch of 16 and decoding 128 images in passes at GEOMETRY_GUMBEL_F8 with synthetic weights: every
    launch class is checked against float64 by a test at its shape (here or in test_vqgan_gpu.py) or exempted there."""
    import launch_census as LC
    geo = OG.GEOMETRY_GUMBEL_F8
    eng = _engine(geo)
    eng.init_params(0)
    img = V._images(V.TOKENIZE_B, geo["resolution"], 0).to(DEV)
    with LC.OpsRecorder(_describe) as rec:
        eng.encode_tokens(img)
        eng.decode_tokens(torch.zeros(V.DECODE_B, eng.image_seq_len, dtype=torch.int32, device=DEV))
    census = LC.Census(CHECKERS, V.EXEMPT, present=PRESENT)
    checked, exempt, unchecked, stale = census.classify(rec.classes())
    print(f"[vqgan-gumbel] census: {len(checked)} checked, {len(exempt)} exempt, passes of "
          f"{eng.decode_pass_images()} images")
    assert any(c[0] == "attn_noncausal_long" for c in checked)
    assert not unchecked, unchecked
    assert not stale, stale


# ------------------------------------------------------------------------------------------------------ boundary
def _import(tmp_path, seed=0, geo=OG.GEOMETRY_GUMBEL_TEST):
    """A synthetic GumbelVQ checkpoint imported with tools/import_vqgan.py; returns (config path, state dict)."""
    from tools import import_vqgan
    cfg = dict(V._vqgan_cfg(tmp_path, geo), quantizer="gumbel")
    (tmp_path / "vqgan.json").write_text(json.dumps(cfg))
    sd = OG.random_state_dict(geo, seed)
    torch.save({"state_dict": sd}, tmp_path / "last.ckpt")
    import_vqgan.main(["--model", str(tmp_path / "vqgan.json"), "--ckpt", str(tmp_path / "last.ckpt")])
    return str(tmp_path / "vqgan.json"), sd


def test_dalle_model_fn_trains_on_gumbel_codes(tmp_path):
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    vae_json, _ = _import(tmp_path)
    K, tv, ts = OG.GEOMETRY_GUMBEL_TEST["num_tokens"], 300, 12

    def params():
        return defaultdict(lambda: None, {
            "model_type": "dalle", "dataset": {"image_size": 64}, "train_batch_size": 2, "n_embd": 256,
            "n_layers": 2, "n_heads": 2, "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts, "lr": 2e-3,
            "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1", "layout": "batch_dim:data",
            "model_path": None, "n_channels": 3, "vae_params": fetch_model_params(vae_json)})
    img = V._images(2, 64, 3)
    cap = torch.randint(0, tv, (2, ts), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
    runs = []
    for _ in range(2):
        spec = dalle_model_fn(img, cap, TRAIN, params())
        vae = spec.extra["vae"]
        assert type(vae).__name__ == "VqganEngine" and vae.gumbel and vae.image_seq_len == 1024
        toks = spec.assemble(img, cap).clone()
        assert toks.shape == (2, ts + 1024)
        assert torch.equal(toks[:, ts:].long() - tv, vae.encode_tokens(img.to(DEV)).clone().long())
        for _ in range(2):
            spec.train_op(img, cap)
        runs.append(spec.engine.export_params())
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])


def test_generate_dalle_writes_pngs_through_the_gumbel_decoder(tmp_path):
    import os
    import numpy as np
    import generate_dalle
    from PIL import Image
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import load_vae_model
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint, save_checkpoint
    vae_json, _ = _import(tmp_path, 2)
    K, tv, ts = OG.GEOMETRY_GUMBEL_TEST["num_tokens"], 300, 12
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": 64}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts, "vae_model": vae_json}
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    params = generate_dalle.load_params(str(tmp_path / "dalle.json"))
    assert generate_dalle.token_grid_side(params) == 32
    eng = DalleEngine(256, 2, 2, tv, K, ts, 1024)
    eng.init_params(5)
    st = dict(eng.export_params())
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)
    np.save(tmp_path / "caps.npy", np.random.default_rng(0).integers(0, tv, (2, ts)).astype(np.int32))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out),
                         "--caption_ids", str(tmp_path / "caps.npy"), "--samples_per_prompt", "1", "--seed", "1"])
    pngs = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(pngs) == 2
    vae, _ = load_vae_model(params, torch.device(DEV))
    vae.load_params({k[4:]: v for k, v in load_checkpoint(latest_checkpoint(str(tmp_path / "vqgan"))).items()
                     if k.startswith("vae/")})
    toks = torch.from_numpy(np.load(out / "tokens.npy")).to(DEV)
    want = generate_dalle.to_uint8(vae.decode_tokens(toks[:, ts:].contiguous(), offset=tv).cpu().numpy())
    for j, f in enumerate(pngs):
        assert np.array_equal(np.asarray(Image.open(out / f)), want[j])


def test_gumbel_vqgan_vae_round_trip(tmp_path):
    from dalle_mtf_b200.models import VQGanVAE
    vae_json, sd = _import(tmp_path, 4)
    m = VQGanVAE(vae_json)
    img = V._images(2, 64, 5)
    ids = m.get_codebook_indices(img)
    assert ids.dtype == torch.int32 and ids.shape == (2, 1024)
    assert ((ids >= 0) & (ids < 512)).all()
    ref_ids = OG.encode_codes(O.to(sd, F64, DEV), OG.GEOMETRY_GUMBEL_TEST, img.to(DEV, F64)).cpu()
    print(f"[vqgan-gumbel] VQGanVAE: {int((ids.cpu().long() == ref_ids).sum())} of {ids.numel()} codes equal the "
          "oracle's")
    out = m.decode(ids)
    assert out.shape == (2, 64, 64, 3) and out.abs().max() <= 1
    assert torch.equal(m.decode(ids + 7, offset=7), out)
    ref = OG.decode(O.to(sd, F64, DEV), OG.GEOMETRY_GUMBEL_TEST, ids.long())
    assert ((out.double() - ref).norm() / ref.norm()).item() < V._decoder_roundings(OG.GEOMETRY_GUMBEL_TEST) * 2.0 ** -9
