"""GPU tests of the VQGAN tokenizer (architecture "vqgan"): the K14 kernels against float64 at every shape the f16 and
test geometries launch, the stride-2 and small-channel convolutions against the oracle's padding, the engine's codes and
decoded images against oracle/vqgan.py, reproducibility, a launch census, and the DALL-E boundary.

Bounds, eps = 2^-24 (f32 roundoff), bf16 outputs with half a bf16 ulp at |ref| (tests/float64_bounds.py):
  * groupnorm statistics: fp32 Welford / Chan combinations over n <= 2^21 values of one group; the computed mean is
    within 2^-16 (|mean| + std) and rstd within 2^-16 + 2^-20 |mean| / std relative (centred sums: an f32 mean off by a
    few eps |mean| moves the variance by ~ eps |mean| / std; E[x^2] - E[x]^2 would move it by ~ eps mean^2 / var, which
    the large-mean case, |mean| / std = 128, rejects);
  * groupnorm apply: v = (x - mean) rstd gamma + beta in f32 (a few eps) from those statistics: |dv| <= 2^-16
    ((|x| + |mean|) rstd |gamma| + |beta|); swish multiplies by at most 1.1 and adds __expf's 2^-21 relative error;
  * attention: a score s_ij = scale sum_c q_c k_c of exact bf16 products summed in f32 is within e_ij = (C + 2) eps
    scale sum_c |q_c k_c|; the softmax weights then move by at most 2 max_j e_ij + 8 eps relative, the f32 weighted sum
    by (S + 2) eps: |do_i| <= (2 max_j e_ij + (S + 10) eps) sum_j p_ij |v_j|;
  * convolutions: n = 9 Cin exact products (bf16 x bf16 on the tensor cores, bf16 x f32 on the direct kernel, one f32
    rounding each) summed in f32: (n + 2) 2^-23 sum |x w| (2^-23: the tensor core may truncate);
  * codes: see test_codes_agree_with_the_oracle_where_the_gap_decides_them;
  * decoded images: every bf16 rounding of an activation moves it by at most 2^-9 relative; on the longest path of the
    decoder (L roundings) the first-order sum is L 2^-9 of the output's scale, which bounds the relative error.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import float64_bounds as FB
from dalle_mtf_b200 import ops
from oracle import vqgan as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
F64 = torch.float64
TOKENIZE_B, DECODE_B = 16, 128       # dalle_coco_b200's per-GPU batch and its predict batch
GEOS = {"f16": O.GEOMETRY_F16, "test": O.GEOMETRY_TEST}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _engine(geo):
    from dalle_mtf_b200.vqgan_engine import VqganEngine
    return VqganEngine(geo["num_tokens"], geo["resolution"], geo["ch"], geo["ch_mult"], geo["num_res_blocks"],
                       geo["attn_resolutions"], geo["z_channels"], geo["embed_dim"])


def _shapes(geo):
    """(res, C) of every GroupNorm and of every attention the engine of `geo` launches."""
    from dalle_mtf_b200.vqgan_engine import network
    enc, dec, _ = network(geo)
    gn, attn = set(), set()
    top, bottom = geo["ch"] * geo["ch_mult"][-1], geo["ch"] * geo["ch_mult"][0]
    hw = geo["resolution"] // 2 ** (len(geo["ch_mult"]) - 1)
    gn |= {(hw, top), (geo["resolution"], bottom)}
    for s in enc + dec:
        if s[0] == "res":
            gn |= {(s[2], s[3]), (s[2], s[4])}
        elif s[0] == "attn":
            gn.add((s[2], s[3]))
            attn.add((s[2] * s[2], s[3]))
    return sorted(gn), sorted(attn)


GN_CASES = sorted({(r, C, B) for g in GEOS.values() for r, C in _shapes(g)[0] for B in (1, 3, TOKENIZE_B)
                   if B * r * r * C <= 2 ** 28})
ATTN_CASES = sorted({(S, C, B) for g in GEOS.values() for S, C in _shapes(g)[1] for B in (1, TOKENIZE_B, 64)})


def _images(B, size, seed):
    """Smooth random images in [-1, 1] (low-frequency noise upsampled, so the codes are not all ties)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(B, 3, size // 8, size // 8, generator=g) * 2 - 1
    img = F.interpolate(low, size=(size, size), mode="bilinear", align_corners=False)
    img = img + 0.1 * (torch.rand(B, 3, size, size, generator=g) * 2 - 1)
    return img.clamp(-1, 1).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------------ kernels
def _check_groupnorm(res, C, B, swish, mu, sigma):
    g = torch.Generator(device=DEV).manual_seed(res * 7 + C + B)
    x = (torch.randn(B, res, res, C, generator=g, device=DEV) * sigma + mu).to(torch.bfloat16)
    gamma = 1 + 0.5 * torch.randn(C, generator=g, device=DEV)
    beta = 0.5 * torch.randn(C, generator=g, device=DEV)
    mean, rstd = FB.nan_like((B, 32), torch.float32), FB.nan_like((B, 32), torch.float32)
    y = torch.full_like(x, float("nan"))
    ops.groupnorm_stats(x, mean, rstd, 32, 1e-6)
    ops.groupnorm_apply(x, mean, rstd, gamma, beta, y, 32, swish)
    xg = x.to(F64).view(B, res * res, 32, C // 32)
    m = xg.mean(dim=(1, 3))
    var = ((xg - m[:, None, :, None]) ** 2).mean(dim=(1, 3))
    sd = var.sqrt()
    tag = f"groupnorm res={res} C={C} B={B} swish={swish} x~N({mu}, {sigma}^2)"
    FB.check(tag + " mean", mean, m, m.abs() + sd, a=0, b=2 ** -16)
    r = 1 / torch.sqrt(var + 1e-6)
    # centred sums: an f32 mean off by a few eps |m| moves the variance by ~ eps |m| / sd relative (16 eps allowed);
    # E[x^2] - E[x]^2 would move it by ~ eps m^2 / var, which this bound rejects once |m| / sd >> 16
    FB.check(tag + " rstd", rstd, r, r * (1 + 2 ** -4 * m.abs() / sd), a=0, b=2 ** -16)
    mm, rr = m.repeat_interleave(C // 32, 1)[:, None, None, :], r.repeat_interleave(C // 32, 1)[:, None, None, :]
    gd, bd = gamma.to(F64), beta.to(F64)
    v = (x.to(F64) - mm) * rr * gd + bd
    absv = (x.to(F64).abs() + mm.abs()) * rr * gd.abs() + bd.abs()
    if swish:
        FB.check(tag, y, v * torch.sigmoid(v), absv, b=1.1 * 2 ** -16 + 2 ** -20, bf16_out=True)
    else:
        FB.check(tag, y, v, absv, b=2 ** -16, bf16_out=True)


@pytest.mark.parametrize("res,C,B", GN_CASES)
@pytest.mark.parametrize("swish", [False, True])
def test_groupnorm_against_float64(res, C, B, swish):
    _check_groupnorm(res, C, B, swish, 1.5, 3.0)


@pytest.mark.parametrize("res,C", sorted({(r, C) for r, C, _ in GN_CASES}))
def test_groupnorm_variance_of_a_large_mean_against_float64(res, C):
    """mean 64, std 0.5 (|m| / sd = 128): the variance must come from centred sums, not E[x^2] - E[x]^2."""
    _check_groupnorm(res, C, 2, False, 64.0, 0.5)


@pytest.mark.parametrize("S,C,B", ATTN_CASES)
def test_attention_against_float64(S, C, B):
    """Rows of ordinary, large (|scores| up to ~50, nearly one-hot weights) and near-uniform scores."""
    g = torch.Generator(device=DEV).manual_seed(S + C + B)
    q = torch.randn(B, S, C, generator=g, device=DEV)
    q[:, 1::3] *= 12.0 * C ** -0.25        # large scores
    q[:, 2::3] *= 1e-3                      # near-uniform
    k, v = torch.randn(B, S, C, generator=g, device=DEV), torch.randn(B, S, C, generator=g, device=DEV)
    qkv = torch.cat([q, k, v], -1).to(torch.bfloat16).contiguous()
    out = torch.full((B, S, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    scale = C ** -0.5
    ops.attn_noncausal(qkv, out, B, S, C, scale)
    qd, kd, vd = (t.to(F64) for t in qkv.split(C, -1))
    p = torch.softmax(scale * qd @ kd.transpose(1, 2), -1)
    ref = p @ vd
    e = (C + 2) * EPS * scale * (qd.abs() @ kd.abs().transpose(1, 2))
    coef = 2 * e.amax(-1, keepdim=True) + (S + 10) * EPS
    FB.check(f"attn_noncausal S={S} C={C} B={B}", out, ref, coef * (p @ vd.abs()), a=0, b=1.0, bf16_out=True)


def test_attention_refuses_what_it_does_not_cover():
    from dalle_mtf_b200 import lib as L
    for S, C in ((320, 128), (96, 128), (256, 576), (256, 96)):
        qkv = torch.zeros(1, S, 3 * C, dtype=torch.bfloat16, device=DEV)
        with pytest.raises(L.DB200Error, match="code -4"):
            ops.attn_noncausal(qkv, torch.empty(1, S, C, dtype=torch.bfloat16, device=DEV), 1, S, C, 1.0)


def test_gather_rows_split_is_exact_and_zero_outside_the_codebook():
    g = torch.Generator(device=DEV).manual_seed(0)
    table = torch.randn(100, 64, generator=g, device=DEV)
    idx = torch.tensor([5, 7, 99 + 10, 10, 3, 110, 200], dtype=torch.int32, device=DEV)
    hi, lo = (torch.full((7, 64), float("nan"), dtype=torch.bfloat16, device=DEV) for _ in range(2))
    ops.gather_rows_split(idx, table, hi, lo, offset=10)
    want = torch.zeros(7, 64, dtype=F64, device=DEV)
    ok = (idx >= 10) & (idx < 110)
    want[ok] = table[(idx[ok] - 10).long()].to(F64)
    hl = hi.to(F64) + lo.to(F64)
    assert ((hl - want).abs() <= 2.0 ** -16 * want.abs()).all()
    assert torch.equal(hi.float(), want.float().to(torch.bfloat16).float())


def test_clamp_bf16_to_f32():
    x = torch.linspace(-3, 3, 1001, device=DEV).to(torch.bfloat16)
    y = torch.full((1001,), float("nan"), device=DEV)
    ops.clamp_bf16_to_f32(x, y)
    assert torch.equal(y, x.float().clamp(-1, 1))


def _conv_cases():
    """(name, B, res, cin, cout, k, stride): the downsampling convs and the 3 -> ch / ch -> 3 convs of both
    geometries."""
    out = []
    for gname, geo in GEOS.items():
        H, ch = geo["resolution"], geo["ch"]
        for B in (1, 2):
            out.append((gname + " conv_in", B, H, 3, ch, 3, 1))
            out.append((gname + " conv_out", B, H, ch * geo["ch_mult"][0], 3, 3, 1))
            res = H
            for i, m in enumerate(geo["ch_mult"][:-1]):
                out.append((f"{gname} down.{i}", B, res, ch * m, ch * m, 3, 2))
                res //= 2
    return out


CONV_CASES = _conv_cases()


@pytest.mark.parametrize("name,B,res,cin,cout,k,stride", CONV_CASES)
def test_convolutions_against_the_oracle_padding(name, B, res, cin, cout, k, stride):
    """The engine's convolution (TF SAME on K11) against taming's: padding 1 for stride 1, an explicit (0, 1, 0, 1)
    pad then no padding for the stride-2 Downsample."""
    from dalle_mtf_b200.vqgan_engine import VqganEngine   # noqa: F401 (the engine's _conv picks the kernel)
    g = torch.Generator(device=DEV).manual_seed(res + cin + cout)
    x = torch.randn(B, res, res, cin, generator=g, device=DEV).to(torch.bfloat16)
    w = torch.randn(cout, cin, k, k, generator=g, device=DEV) / math.sqrt(cin * k * k)
    bias = 0.1 * torch.randn(cout, generator=g, device=DEV)
    dsc = ops.conv_desc(B, res, res, cin, cout, k, k, stride, act_f32=False)
    y = torch.full((B, dsc.Ho, dsc.Wo, cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    w_hwio = w.permute(2, 3, 1, 0).contiguous()
    if ops.conv_tc_supported(dsc):
        w16 = w_hwio.to(torch.bfloat16)
        ops.conv2d_fwd_tc(dsc, x, w16, bias, None, y)
        wd = w16.to(F64).permute(3, 2, 0, 1)
    else:
        ops.conv2d_fwd(dsc, x, w_hwio, bias, None, y)
        wd = w.to(F64)
    xd = x.to(F64).permute(0, 3, 1, 2)
    if stride == 2:
        ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wd, bias.to(F64), stride=2)
        absref = F.conv2d(F.pad(xd.abs(), (0, 1, 0, 1)), wd.abs(), bias.to(F64).abs(), stride=2)
    else:
        ref = F.conv2d(xd, wd, bias.to(F64), padding=k // 2)
        absref = F.conv2d(xd.abs(), wd.abs(), bias.to(F64).abs(), padding=k // 2)
    n = k * k * cin
    FB.check(f"conv {name} B={B}", y, ref.permute(0, 2, 3, 1), absref.permute(0, 2, 3, 1), a=0,
             b=(n + 2) * 2.0 ** -23, bf16_out=True)


# ------------------------------------------------------------------------------------------------------ engine
def _setup(gname, seed=0):
    geo = GEOS[gname]
    sd = O.random_state_dict(geo, seed)
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    eng = _engine(geo)
    eng.load_params(import_taming_state_dict(sd, geo))
    return geo, sd, eng


@pytest.mark.parametrize("gname,B", [("test", 4), ("f16", 2)])
def test_codes_agree_with_the_oracle_where_the_gap_decides_them(gname, B):
    """Row r's code is decided by the oracle's gap g_r between its best and second-best distance when
    g_r > 2 ||z_eng,r - z_ref,r|| max_n ||e_best - e_n|| + the score's rounding bound (the engine's scores
    z . e_n - ||e_n||^2 / 2 on hi + lo split operands: the dropped lo x lo product and the splits' residuals are
    3 2^-16 sum_c |z_c e_nc|, the f32 sums (D + 2) 2^-23 of it, doubled for distances, for both codes).  Such rows must
    agree; the others are counted and reported.  Separately, the engine's codes are the exact nearest codes of its own
    z wherever that gap exceeds the rounding bound."""
    geo, sd, eng = _setup(gname)
    img = _images(B, geo["resolution"], 1)
    codes = eng.encode_tokens(img.to(DEV)).clone().cpu().long().view(-1)
    z_eng = eng._b["z"].double().cpu()
    sd64 = O.to(sd, F64, DEV)
    z_ref = O.encode_z(sd64, geo, img.to(DEV, F64)).reshape(-1, geo["embed_dim"]).cpu()
    E = sd64["quantize.embedding.weight"].cpu()
    D = geo["embed_dim"]

    def gap_and_bound(z):
        d = O.distances(z, E)
        two = d.topk(2, dim=1, largest=False)
        best = two.indices[:, 0]
        spread = (E[best][:, None, :] - E[None, :, :]).norm(dim=-1).amax(-1) if E.shape[0] <= 4096 else \
            torch.stack([(E[b] - E).norm(dim=-1).max() for b in best.tolist()])
        rnd = 2 * 2 * (3 * 2.0 ** -16 + (D + 2) * 2.0 ** -23) * (z.abs() @ E.abs().T).amax(-1)
        return best, two.values[:, 1] - two.values[:, 0], spread, rnd

    best, gap, spread, rnd = gap_and_bound(z_ref)
    dz = (z_eng - z_ref).norm(dim=-1)
    decided = gap > 2 * dz * spread + rnd
    n = decided.numel()
    print(f"[vqgan] {gname} B={B}: {int((~decided).sum())} of {n} rows excluded (gap below the bound); "
          f"max |z_eng - z_ref| / |z_ref| {float((dz / z_ref.norm(dim=-1)).max()):.3e}")
    assert torch.equal(codes[decided], best[decided])
    rel = ((z_eng - z_ref).norm() / z_ref.norm()).item()
    print(f"[vqgan] {gname}: z rel-fro {rel:.3e} (bound {_encoder_roundings(geo) * 2.0 ** -9:.3e})")
    assert rel < _encoder_roundings(geo) * 2.0 ** -9
    own, own_gap, _, own_rnd = gap_and_bound(z_eng)
    own_ok = own_gap > own_rnd
    print(f"[vqgan] {gname}: codes against the engine's own z: {int(own_ok.sum())} of {n} rows decided")
    assert own_ok.any() and torch.equal(codes[own_ok], own[own_ok])


@pytest.mark.parametrize("gname", ["test", "f16"])
def test_codes_take_the_first_of_tied_codes(gname):
    """A codebook whose odd rows repeat the even rows before them: every distance ties in pairs, and the engine must
    return the first (even) index, as torch.argmin does."""
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    geo = GEOS[gname]
    sd = O.random_state_dict(geo, 8)
    E = sd["quantize.embedding.weight"]
    E[1::2] = E[0::2]
    eng = _engine(geo)
    eng.load_params(import_taming_state_dict(sd, geo))
    codes = eng.encode_tokens(_images(4, geo["resolution"], 6).to(DEV)).clone().cpu()
    print(f"[vqgan] {gname} ties: {len(set(codes.view(-1).tolist()))} distinct codes, all must be even")
    assert (codes % 2 == 0).all()


@pytest.mark.parametrize("gname", ["test", "f16"])
def test_codes_are_reproducible_and_independent_of_the_batch(gname):
    geo, _, eng = _setup(gname, 5)
    img = _images(TOKENIZE_B, geo["resolution"], 4).to(DEV)
    a = eng.encode_tokens(img).clone()
    b = eng.encode_tokens(img).clone()
    assert torch.equal(a, b)
    for i in (0, 7, TOKENIZE_B - 1):
        assert torch.equal(eng.encode_tokens(img[i:i + 1].contiguous()).clone(), a[i:i + 1])


def _encoder_roundings(geo):
    """bf16 roundings on the encoder's longest path to z: the image, conv_in, 4 per ResnetBlock and AttnBlock, 1 per
    Downsample, norm_out and conv_out (quant_conv is fp32-accurate)."""
    from dalle_mtf_b200.vqgan_engine import network
    return 3 + sum({"res": 4, "attn": 4, "down": 1}[s[0]] for s in network(geo)[0])


def _decoder_roundings(geo):
    """bf16 roundings on the decoder's longest path: per ResnetBlock 4 (GN1, conv1, GN2, conv2), per AttnBlock 4
    (GN, q|k|v, o, proj_out), per Upsample 2 (the copy is exact; its conv 1), plus post_quant_conv, conv_in, norm_out
    and conv_out."""
    from dalle_mtf_b200.vqgan_engine import network
    n = 4
    for s in network(geo)[1]:
        n += {"res": 4, "attn": 4, "up": 1}[s[0]]
    return n


@pytest.mark.parametrize("gname,B", [("test", 3), ("f16", 2)])
def test_decode_tokens_against_the_oracle(gname, B):
    geo, sd, eng = _setup(gname, 6)
    g = torch.Generator().manual_seed(9)
    codes = torch.randint(0, geo["num_tokens"], (B, eng.image_seq_len), generator=g)
    off = 1000
    got = eng.decode_tokens((codes + off).to(torch.int32).to(DEV), offset=off).clone()
    ref = O.decode(O.to(sd, F64, DEV), geo, codes.to(DEV))
    rel = ((got.double() - ref).norm() / ref.norm()).item()
    bound = _decoder_roundings(geo) * 2.0 ** -9
    print(f"[vqgan] {gname} decode B={B}: rel-fro {rel:.3e} (bound {bound:.3e})")
    assert rel < bound and got.abs().max() <= 1
    # independent of the pass size
    one = torch.cat([eng.decode_tokens((codes[i:i + 1] + off).to(torch.int32).to(DEV), offset=off).clone()
                     for i in range(B)])
    assert torch.equal(one, got)


# ------------------------------------------------------------------------------------------------------ census
def _describe(entry, A):
    """A launch class per ops entry, with the fields its float64 check is parametrised by."""
    import launch_census as LC
    if entry in ("conv_desc", "conv_tc_supported"):       # host helpers, no launch
        return None
    if entry == "groupnorm":
        x = A["x"]
        return LC.launch_class(entry, res=x.shape[1], C=x.shape[-1], B=x.shape[0]), None
    if entry == "attn_noncausal":
        return LC.launch_class(entry, S=A["S"], C=A["C"], B=A["B"]), None
    if entry in ("conv2d_fwd", "conv2d_fwd_tc"):
        c = A["c"]
        return LC.launch_class(entry, B=c.N, res=c.H, cin=c.Cin, cout=c.Cout, k=c.KH, stride=c.stride), None
    return LC.launch_class(entry), None


def _census(B_enc, B_dec, gname="f16"):
    import launch_census as LC
    geo, _, eng = _setup(gname, 0)
    img = _images(B_enc, geo["resolution"], 0).to(DEV)
    with LC.OpsRecorder(_describe) as rec:
        eng.encode_tokens(img)
        eng.decode_tokens(torch.zeros(B_dec, eng.image_seq_len, dtype=torch.int32, device=DEV))
    return rec.classes(), eng


GN_SHAPES = {(r, C) for r, C, _ in GN_CASES}
ATTN_SHAPES = {(S, C) for S, C, _ in ATTN_CASES}
CONV_SHAPES = {(res, cin, cout, k, stride) for _, _, res, cin, cout, k, stride in CONV_CASES}
CHECKERS = [
    ("test_groupnorm_against_float64", lambda c: c[0] == "groupnorm" and (LCf(c)["res"], LCf(c)["C"]) in GN_SHAPES),
    ("test_attention_against_float64", lambda c: c[0] == "attn_noncausal" and (LCf(c)["S"], LCf(c)["C"]) in ATTN_SHAPES),
    ("test_convolutions_against_the_oracle_padding", lambda c: c[0] in ("conv2d_fwd", "conv2d_fwd_tc") and
     tuple(LCf(c)[k] for k in ("res", "cin", "cout", "k", "stride")) in CONV_SHAPES),
    ("test_gather_rows_split_is_exact_and_zero_outside_the_codebook", lambda c: c[0] == "gather_rows_split"),
    ("test_clamp_bf16_to_f32", lambda c: c[0] == "clamp_bf16_to_f32"),
]
# the other launches run kernels whose float64 tests live elsewhere; at this network's shapes the engine tests compare
# their composition with the oracle
EXEMPT = {
    "conv2d_fwd_tc": ("tests/test_vqgan_gpu.py::test_decode_tokens_against_the_oracle", "stride-1 3x3 / 1x1 wgmma "
                      "convolutions (float64 tests: test_vae_config_launches_gpu.py); composed here against the oracle"),
    "linear_fwd": ("tests/test_vqgan_gpu.py::test_decode_tokens_against_the_oracle", "AttnBlock q|k|v and proj_out"),
    "gemm": ("tests/test_vqgan_gpu.py::test_codes_agree_with_the_oracle_where_the_gap_decides_them",
             "split products of quant_conv, the code scores and post_quant_conv"),
    "split_f32": ("tests/test_vqgan_gpu.py::test_codes_agree_with_the_oracle_where_the_gap_decides_them", "exact split"),
    "argmax_rows": ("tests/test_vqgan_gpu.py::test_codes_agree_with_the_oracle_where_the_gap_decides_them",
                    "first maximum"),
    "cast_f32_to_bf16": ("tests/test_vqgan_gpu.py::test_decode_tokens_against_the_oracle", "rounding cast"),
    "upsample2x_fwd": ("tests/test_vae_paper_gpu.py::test_upsample_fwd_exact_bwd_against_float64", "exact copy"),
}


def LCf(c):
    import launch_census as LC
    return LC.fields(c)


def test_launch_census_of_encode_and_decode():
    """Encoding the tokenize batch of 16 and decoding the predict batch of 128 in passes at the f16 geometry: every
    launch class is checked against float64 by a test of this module or exempted to a named test."""
    import launch_census as LC
    classes, eng = _census(TOKENIZE_B, DECODE_B)
    census = LC.Census(CHECKERS, EXEMPT, present={n for n, _ in CHECKERS})
    checked, exempt, unchecked, stale = census.classify(classes)
    print(f"[vqgan] census: {len(checked)} checked, {len(exempt)} exempt, passes of {eng.decode_pass_images()} images")
    assert not unchecked, unchecked
    assert not stale, stale


# ------------------------------------------------------------------------------------------------------ boundary
def _vqgan_cfg(tmp_path, geo=O.GEOMETRY_TEST):
    return {"model_type": "vae", "dataset": {"image_size": geo["resolution"]}, "architecture": "vqgan",
            "num_tokens": geo["num_tokens"], "use_bf16": True, "model_path": str(tmp_path / "vqgan"),
            "predict_batch_size": 4, **{k: geo[k] for k in ("ch", "ch_mult", "num_res_blocks", "attn_resolutions",
                                                             "z_channels", "embed_dim", "resolution")}}


def _import(tmp_path, seed=0):
    """A synthetic taming checkpoint imported with tools/import_vqgan.py; returns (config path, state dict)."""
    import json
    from tools import import_vqgan
    cfg = _vqgan_cfg(tmp_path)
    (tmp_path / "vqgan.json").write_text(json.dumps(cfg))
    sd = O.random_state_dict(O.GEOMETRY_TEST, seed)
    torch.save({"state_dict": {**sd, "loss.discriminator.main.0.weight": torch.zeros(2)}}, tmp_path / "last.ckpt")
    import_vqgan.main(["--model", str(tmp_path / "vqgan.json"), "--ckpt", str(tmp_path / "last.ckpt")])
    return str(tmp_path / "vqgan.json"), sd


def test_dalle_model_fn_trains_on_vqgan_codes(tmp_path):
    from collections import defaultdict
    from dalle_mtf_b200.model_fns import TRAIN, dalle_model_fn
    from dalle_mtf_b200.utils import fetch_model_params
    vae_json, _ = _import(tmp_path)
    K, tv, ts = O.GEOMETRY_TEST["num_tokens"], 300, 12

    def params():
        return defaultdict(lambda: None, {
            "model_type": "dalle", "dataset": {"image_size": 64}, "train_batch_size": 4, "n_embd": 256,
            "n_layers": 2, "n_heads": 2, "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts, "lr": 2e-3,
            "train_steps": 100, "warmup_steps": 2, "bf_16": True, "mesh_shape": "data:1", "layout": "batch_dim:data",
            "model_path": None, "n_channels": 3, "vae_params": fetch_model_params(vae_json)})
    img = _images(4, 64, 3)
    cap = torch.randint(0, tv, (4, ts), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
    runs = []
    for _ in range(2):
        spec = dalle_model_fn(img, cap, TRAIN, params())
        vae = spec.extra["vae"]
        assert type(vae).__name__ == "VqganEngine"
        toks = spec.assemble(img, cap).clone()
        want = vae.encode_tokens(img.to(DEV)).clone()
        assert torch.equal(toks[:, ts:].long() - tv, want.long())
        for _ in range(2):
            spec.train_op(img, cap)
        runs.append(spec.engine.export_params())
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])


def test_generate_dalle_writes_pngs_through_the_vqgan_decoder(tmp_path):
    import json
    import os
    import numpy as np
    import generate_dalle
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import load_vae_model
    from dalle_mtf_b200.utils import save_checkpoint
    vae_json, _ = _import(tmp_path, 2)
    K, tv, ts = O.GEOMETRY_TEST["num_tokens"], 300, 12
    dalle_cfg = {"model_type": "dalle", "dataset": {"image_size": 64}, "predict_batch_size": 2,
                 "model_path": str(tmp_path / "dalle_run"), "n_embd": 256, "n_layers": 2, "n_heads": 2,
                 "text_vocab_size": tv, "image_vocab_size": K, "text_seq_len": ts, "vae_model": vae_json}
    (tmp_path / "dalle.json").write_text(json.dumps(dalle_cfg))
    params = generate_dalle.load_params(str(tmp_path / "dalle.json"))
    assert generate_dalle.token_grid_side(params) == 16
    eng = DalleEngine(256, 2, 2, tv, K, ts, 256)
    eng.init_params(5)
    st = dict(eng.export_params())
    st["global_step"] = 3
    save_checkpoint(dalle_cfg["model_path"], 3, st)
    np.save(tmp_path / "caps.npy", np.random.default_rng(0).integers(0, tv, (3, ts)).astype(np.int32))
    out = tmp_path / "out"
    generate_dalle.main(["--model", str(tmp_path / "dalle.json"), "--out", str(out),
                         "--caption_ids", str(tmp_path / "caps.npy"), "--samples_per_prompt", "1", "--seed", "1"])
    pngs = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(pngs) == 3
    from PIL import Image
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    vae, ckpt = load_vae_model(params, torch.device(DEV))
    vae.load_params({k[4:]: v for k, v in load_checkpoint(latest_checkpoint(str(tmp_path / "vqgan"))).items()
                     if k.startswith("vae/")})
    toks = torch.from_numpy(np.load(out / "tokens.npy")).to(DEV)
    want = generate_dalle.to_uint8(vae.decode_tokens(toks[:, ts:].contiguous(), offset=tv).cpu().numpy())
    for j, f in enumerate(pngs):
        assert np.array_equal(np.asarray(Image.open(out / f)), want[j])


def test_vqgan_vae_round_trip(tmp_path):
    from dalle_mtf_b200.models import VQGanVAE
    vae_json, sd = _import(tmp_path, 4)
    m = VQGanVAE(vae_json)
    img = _images(2, 64, 5)
    ids = m.get_codebook_indices(img)
    assert ids.dtype == torch.int32 and ids.shape == (2, 256)
    assert ((ids >= 0) & (ids < 512)).all()
    out = m.decode(ids)
    assert out.shape == (2, 64, 64, 3) and out.abs().max() <= 1
    assert torch.equal(m.decode(ids + 7, offset=7), out)
    ref = O.decode(O.to(sd, F64, DEV), O.GEOMETRY_TEST, ids.long())
    assert ((out.double() - ref).norm() / ref.norm()).item() < _decoder_roundings(O.GEOMETRY_TEST) * 2.0 ** -9
