"""CPU side of the token shift: the oracle's shift against a literal restatement of DALLE-pytorch's PreShiftToken, the
adjoint the backward kernel implements (float64), the shift_tokens key at every place a model is built (including the
refusal of a non-square image grid), generate_dalle.py handing the key to the engine, and the oracle (bit for bit the
unshifted oracle with the key off, and three mutants that change the output)."""
import pytest
import torch
import torch.nn.functional as F

import generate_dalle as G
from dalle_mtf_b200.dalle_engine import DalleEngine, validate_shift_tokens
from dalle_mtf_b200.model_fns import dalle_model_fn, shift_tokens
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_glu as OGL
from oracle import dalle_shift as OS
from test_gelu_cpu import _Built, _generate_config

F64 = torch.float64


# ------------------------------------------------------------------------------------------------ the definition
def pre_shift_token(x, text_len, image_size):
    """DALLE-pytorch's PreShiftToken.forward (before its fn) restated on x [b, n, d], n <= text_len + image_size^2:
    the text part shifts chunk(2)[0] by one position, the image part, padded to the full grid, chunk(4)[0] from the
    top and chunk(4)[1] from the left, both with zero padding."""
    b, n, _ = x.shape
    x_text, x_img = x[:, :text_len], x[:, text_len:]
    padding = image_size ** 2 - x_img.shape[1]
    x_img = F.pad(x_img, (0, 0, 0, padding))
    x_img = x_img.reshape(b, image_size, image_size, -1)
    x_text_shift, x_text_pass = x_text.chunk(2, dim=-1)
    x_text_shift = F.pad(x_text_shift, (0, 0, 1, -1))
    x_text = torch.cat((x_text_shift, x_text_pass), dim=-1)
    top, left, *rest = x_img.chunk(4, dim=-1)
    left = F.pad(left, (0, 0, 1, -1))
    top = F.pad(top, (0, 0, 0, 0, 1, -1))
    x_img = torch.cat((top, left, *rest), dim=-1).reshape(b, image_size ** 2, -1)
    return torch.cat((x_text, x_img[:, :max(n - text_len, 0)]), dim=1)


def shift_transpose(g, text_len, grid_w):
    """The transpose of the shift as include/dalle_b200.h states it for shift_tokens_bwd, one position at a time."""
    S, d = g.shape[-2], g.shape[-1]
    c = d // 4
    out = torch.zeros_like(g)
    out[..., 2 * c:] = g[..., 2 * c:]
    for p in range(S):
        if p < text_len:
            if p + 1 < min(text_len, S):
                out[..., p, :2 * c] = g[..., p + 1, :2 * c]
            continue
        u = p - text_len
        if u // grid_w + 1 < grid_w and p + grid_w < S:
            out[..., p, :c] = g[..., p + grid_w, :c]
        if u % grid_w + 1 < grid_w and p + 1 < S:
            out[..., p, c:2 * c] = g[..., p + 1, c:2 * c]
    return out


GEOMETRIES = [(4, 3), (1, 4), (5, 1), (3, 2), (16, 8)]   # (text_len, grid_w): TL = 1, W = 1 and W = 2 among them


@pytest.mark.parametrize("TL,W", GEOMETRIES)
def test_oracle_shift_is_dallepytorch_pre_shift_token(TL, W):
    """With a zero <bos> row in front, DALLE-pytorch's text part is [<bos>, caption] (TL + 1 long) and its grid holds
    all W^2 codes: its PreShiftToken then computes, on the caption and the codes, what the oracle's shift computes.
    A prefix (the prefill) shifts as the prefix of the whole sequence does."""
    g = torch.Generator().manual_seed(TL * 100 + W)
    S, d = TL + W * W, 64
    y = torch.randn(3, S, d, generator=g, dtype=F64)
    with_bos = torch.cat([torch.zeros(3, 1, d, dtype=F64), y], 1)
    want = pre_shift_token(with_bos, TL + 1, W)[:, 1:]
    got = OS.shift(y, TL, W)
    assert torch.equal(got, want)
    for P in sorted({1, max(TL - 1, 1), TL, TL + 1, TL + W - 1, TL + W, S - 1, S} & set(range(1, S + 1))):
        assert torch.equal(OS.shift(y[:, :P], TL, W), got[:, :P]), P
        bos_p = torch.cat([torch.zeros(3, 1, d, dtype=F64), y[:, :P]], 1)
        assert torch.equal(pre_shift_token(bos_p, TL + 1, W)[:, 1:], got[:, :P]), P
    # the first image token reads zeros in both chunks, text never reads image and image never reads text
    c = d // 4
    assert not got[:, TL, :2 * c].any()
    if TL >= 1:
        z = y.clone()
        z[:, :TL] = 0
        assert torch.equal(OS.shift(z, TL, W)[:, TL:], got[:, TL:])
        z = y.clone()
        z[:, TL:] = 0
        assert torch.equal(OS.shift(z, TL, W)[:, :TL], got[:, :TL])


@pytest.mark.parametrize("TL,W", GEOMETRIES)
def test_the_stated_transpose_is_the_adjoint_in_float64(TL, W):
    """<shift(y), g> = <y, shift^T(g)> for the transpose stated for shift_tokens_bwd, at full length and at prefill
    lengths; it is also autograd's vector-Jacobian product of the oracle's shift."""
    g = torch.Generator().manual_seed(7 + TL + W)
    S, d = TL + W * W, 32
    for n in sorted({S, max(S - 1, 1), TL + W, 1} & set(range(1, S + 1))):
        y = torch.randn(2, n, d, generator=g, dtype=F64, requires_grad=True)
        gr = torch.randn(2, n, d, generator=g, dtype=F64)
        lhs = (OS.shift(y, TL, W) * gr).sum()
        rhs = (y * shift_transpose(gr, TL, W)).sum()
        assert abs(lhs.item() - rhs.item()) <= 1e-12 * (1 + abs(lhs.item())), n
        (vjp,) = torch.autograd.grad(lhs, y)
        assert torch.equal(vjp, shift_transpose(gr, TL, W)), n


# ------------------------------------------------------------------------------------------------ config values
ACCEPTED = [({}, False), ({"shift_tokens": None}, False), ({"shift_tokens": False}, False),
            ({"shift_tokens": True}, True)]
REJECTED = [1, 0, 1.0, "true", "false", "", [True], {"on": True}]


@pytest.mark.parametrize("params,want", ACCEPTED)
def test_accepted_values(params, want):
    assert shift_tokens(params) is want
    assert shift_tokens(params, 16) is want


@pytest.mark.parametrize("value", REJECTED, ids=[repr(v) for v in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, value):
    p = {"shift_tokens": value}
    with pytest.raises(ValueError, match="shift_tokens"):
        shift_tokens(p)
    with pytest.raises(ValueError, match="shift_tokens"):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="shift_tokens"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match="shift_tokens"):
        G.main(_generate_config(tmp_path, p))


def test_engine_validates_its_argument_before_any_device_work():
    for v in (True, False):
        assert validate_shift_tokens(v, 16) is v
    assert validate_shift_tokens(False, 24) is False             # off: any image length
    for bad in [None, 1, 0, "true", [True]]:
        with pytest.raises(ValueError, match="shift_tokens"):
            validate_shift_tokens(bad, 16)
        with pytest.raises(ValueError, match="shift_tokens"):
            DalleEngine(256, 1, 2, 10, 16, 4, 16, shift_tokens=bad)


@pytest.mark.parametrize("image_seq_len", [24, 15, 2])
def test_a_non_square_image_grid_is_refused_with_the_key_on(image_seq_len):
    with pytest.raises(ValueError, match="shift_tokens"):
        validate_shift_tokens(True, image_seq_len)
    with pytest.raises(ValueError, match="shift_tokens"):
        shift_tokens({"shift_tokens": True}, image_seq_len)
    with pytest.raises(ValueError, match="shift_tokens"):
        DalleEngine(256, 1, 2, 10, 16, 4, image_seq_len, shift_tokens=True)
    with pytest.raises(ValueError, match="shift_tokens"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=image_seq_len, n_layers=1,
              n_heads=2, params={"shift_tokens": True})


@pytest.mark.parametrize("extra,want", [({}, False), ({"shift_tokens": None}, False), ({"shift_tokens": True}, True)])
def test_generate_cli_builds_the_engine_with_the_config_key(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the token shift it was trained with (device work stubbed out)."""
    import types
    from dalle_mtf_b200 import dalle_engine, lib as L, model_fns
    seen = {}

    def engine(*a, **k):
        seen.update(k)
        raise _Built

    vae = types.SimpleNamespace(K=64, image_seq_len=16, load_params=lambda state: None)
    monkeypatch.setattr(L, "require_device", lambda: None)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(model_fns, "load_vae_model", lambda params, device: (vae, None))
    monkeypatch.setattr(dalle_engine, "DalleEngine", engine)
    with pytest.raises(_Built):
        G.main(_generate_config(tmp_path, extra))
    assert seen["shift_tokens"] is want


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, d=64, Lyr=2, H=2, TL=6, W=3):
    cfg = O.DalleConfig(d, Lyr, H, 50, 16, TL, W * W)
    params = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.3
        if k.endswith("attn/q") or k.endswith("attn/k"):
            params[k] = params[k] * 20.0           # sharp attention: the shifted features matter
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, TL), generator=g),
                               torch.randint(0, 16, (2, W * W), generator=g), 50)
    return cfg, params, tokens


@pytest.mark.parametrize("gated", [False, True], ids=["plain", "gated"])
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_oracle_without_the_shift_is_the_glu_oracle_bit_for_bit(gated, bf16):
    cfg, params, tokens = _model(3)
    if gated:
        params = OGL.init_params(params, cfg, 4)
    kw = dict(bf16=bf16, activation="gelu", gated=gated, rotary=(16, 10000.0))
    a = OS.loss_and_grads(params, tokens, cfg, shift_tokens=False, **kw)
    b = OGL.loss_and_grads(params, tokens, cfg, **kw)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert a[3].keys() == b[3].keys() and all(torch.equal(a[3][k], b[3][k]) for k in a[3])


def test_the_shift_and_each_mutant_change_the_output():
    cfg, params, tokens = _model(5, d=128)
    off = OS.forward(params, tokens, cfg, shift_tokens=False)[2]
    ref = OS.forward(params, tokens, cfg)[2]
    assert ((ref - off).norm() / off.norm()).item() > 1e-3
    for m in OS.MUTATIONS:
        mut = OS.forward(params, tokens, cfg, shift_mutate=m)[2]
        rel = ((mut - ref).norm() / ref.norm()).item()
        assert rel > 1e-3, (m, rel)
    with pytest.raises(ValueError):
        OS.forward(params, tokens, cfg, shift_mutate="nope")
    with pytest.raises(ValueError):
        OS.forward(params, tokens, cfg, shift_tokens=False, shift_mutate="swap")
