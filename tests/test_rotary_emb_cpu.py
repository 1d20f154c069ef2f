"""CPU side of DALLE-pytorch's rotary embedding (rotary_emb): the key at the four places a model is built (DalleEngine,
dalle_model_fn, models.DALLE, generate_dalle.py), the angle table against a literal restatement of DALLE-pytorch's
and rotary-embedding-torch's recipe, the oracle's rotation against rotary-embedding-torch's apply_rotary_emb, the
oracle with zero angles against the GELU oracle with a zero wpe, and the parameter layout without wpe."""
import math

import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.dalle_engine import DalleEngine, param_layout, rotary_emb_table, validate_rotary, \
    validate_rotary_emb
from dalle_mtf_b200.model_fns import dalle_model_fn, rotary_emb, rotary_embedding
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_gelu as OG
from oracle import dalle_rotary_emb as ORE
from test_gelu_cpu import _Built, _generate_config

ACCEPTED = [({}, False), ({"rotary_emb": None}, False), ({"rotary_emb": False}, False), ({"rotary_emb": True}, True),
            ({"rotary_emb": False, "rotary_dim": 64}, False), ({"rotary_emb": True, "image_position_embedding": None},
                                                                True)]
REJECTED = [{"rotary_emb": 1}, {"rotary_emb": 0}, {"rotary_emb": "true"}, {"rotary_emb": [True]}, {"rotary_emb": 1.0},
            {"rotary_emb": True, "rotary_dim": 64}, {"rotary_emb": True, "rotary_base": 500.0},
            {"rotary_emb": True, "image_position_embedding": "absolute"},
            {"rotary_emb": True, "image_position_embedding": "row_col"}]
MODEL = {"n_embd": 256, "n_heads": 2}


@pytest.mark.parametrize("params,want", ACCEPTED, ids=[repr(p) for p, _ in ACCEPTED])
def test_accepted_values(params, want):
    assert rotary_emb({**MODEL, **params}) is want
    assert rotary_emb({**MODEL, **params}, 16) is want
    # the GPT-NeoX keys keep their meaning and their exact return values
    assert rotary_embedding({**MODEL, **params}) == ((None, None) if "rotary_dim" not in params else (64, 10000.0))
    assert validate_rotary(None, None, 128) is None


@pytest.mark.parametrize("params", REJECTED, ids=[repr(p) for p in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, params):
    with pytest.raises(ValueError, match="rotary"):
        rotary_emb({**MODEL, **params})
    with pytest.raises(ValueError, match="rotary"):        # before any GPU work
        dalle_model_fn(None, None, "train", {**MODEL, **params})
    with pytest.raises(ValueError, match="rotary"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(params))
    with pytest.raises(ValueError, match="rotary"):
        DalleEngine(256, 1, 2, 10, 16, 4, 16, rotary_dim=params.get("rotary_dim"),
                    rotary_base=params.get("rotary_base"), rotary_emb=params.get("rotary_emb"),
                    image_position_embedding=params.get("image_position_embedding"))
    with pytest.raises(ValueError, match="rotary"):
        G.main(_generate_config(tmp_path, params))


def test_a_non_square_grid_is_refused():
    with pytest.raises(ValueError, match="square"):
        validate_rotary_emb(True, 15)
    with pytest.raises(ValueError, match="square"):
        rotary_emb({"rotary_emb": True}, 24)
    with pytest.raises(ValueError, match="square"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=15, n_layers=1, n_heads=2,
              params={"rotary_emb": True})
    with pytest.raises(ValueError, match="square"):
        DalleEngine(256, 1, 2, 10, 16, 4, 15, rotary_emb=True)
    with pytest.raises(L.DB200Error):       # the arguments pass; there is no device here
        DalleEngine(256, 1, 2, 10, 16, 4, 16, rotary_emb=True)


@pytest.mark.parametrize("extra,want", [({}, False), ({"rotary_emb": True}, True)])
def test_generate_cli_builds_the_engine_with_the_config_key(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the rotary_emb of its config (device work stubbed out)."""
    import types
    from dalle_mtf_b200 import dalle_engine, model_fns
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
    assert seen["rotary_emb"] is want
    assert seen["image_position_embedding"] == (None if want else "absolute")


# ------------------------------------------------------------------------------------------------ the table
def dallepytorch_freqs(dh, text_len, fmap):
    """DALLE-pytorch's pos_emb [S, 6 nf] restated: rotary-embedding-torch's RotaryEmbedding(dim = dh // 3) with
    freqs_for 'lang' (theta 10000) and 'pixel' (max_freq 10), forward(t) = repeat(t * freqs, '... n -> ... (n r)',
    r = 2); text positions 0 .. TL-1, image tokens at 8192; the axial part broadcat of the row and column frequencies
    of linspace(-1, 1, fmap), text tokens at -10.  (Text positions here start at 0: this repository has no BOS.)"""
    rot = dh // 3
    lang = 1. / (10000 ** (torch.arange(0, rot, 2)[:(rot // 2)].float() / rot))
    pixel = torch.linspace(1., 10 / 2, rot // 2) * math.pi

    def emb(t, freqs):   # einsum('..., f -> ... f', t, freqs) then repeat (n r), r = 2
        f = torch.einsum("..., f -> ... f", t.type(freqs.dtype), freqs)
        return f.repeat_interleave(2, dim=-1)
    img_len = fmap ** 2
    text_freqs = torch.cat((emb(torch.arange(text_len), lang), emb(torch.full((img_len,), 8192), lang)), dim=0)
    axial = emb(torch.linspace(-1, 1, steps=fmap), pixel)
    img = torch.cat((axial[:, None, :].expand(fmap, fmap, -1), axial[None, :, :].expand(fmap, fmap, -1)), dim=-1)
    img = img.reshape(fmap * fmap, -1)
    text_axial = emb(torch.full((text_len,), -10.), pixel)
    img_freqs = torch.cat((torch.cat((text_axial, text_axial), dim=-1), img), dim=0)
    return torch.cat((text_freqs, img_freqs), dim=-1)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("W", [4, 16, 32])
def test_table_is_dallepytorchs_recipe_bit_for_bit(dh, W):
    TL = 256 if W == 32 else 24
    freqs = dallepytorch_freqs(dh, TL, W)
    nf = dh // 3 // 2
    assert freqs.shape == (TL + W * W, 6 * nf)
    assert torch.equal(freqs[:, 0::2], freqs[:, 1::2])          # each angle covers one interleaved pair
    want = freqs[:, 0::2]
    assert torch.equal(ORE.angles(TL, W, dh), want)
    t = rotary_emb_table(TL, W, dh)
    assert t.dtype == torch.float32 and tuple(t.shape) == (TL + W * W, 2, 3 * nf)
    c, s = torch.cos(want.double()).float(), torch.sin(want.double()).float()
    assert torch.equal(t[:, 0], c) and torch.equal(t[:, 1], s)
    oc, os_ = ORE.table(TL, W, dh)
    assert torch.equal(oc, c) and torch.equal(os_, s)
    # the float64 evaluation of the float32 angle differs from a float32 one (up to ~5e-4 rad at 8192)
    assert not torch.equal(torch.cos(want), c) or dh == 64 and W == 4


@pytest.mark.parametrize("m", ORE.MUTATIONS)
def test_every_mutant_changes_the_angles_or_the_rotation(m):
    if m in ("no_v", "rotate_half"):
        return   # not a table mutation: forward() applies them (checked below)
    assert not torch.equal(ORE.angles(16, 4, 128, m), ORE.angles(16, 4, 128))


# ------------------------------------------------------------------------------------------------ oracle
def apply_rotary_emb(freqs, t):
    """rotary-embedding-torch's apply_rotary_emb restated: t * cos + rotate_half(t) * sin over the first
    freqs.shape[-1] dims, rotate_half interleaved: (x1, x2) pairs -> (-x2, x1)."""
    rot_dim = freqs.shape[-1]
    t_mid, t_right = t[..., :rot_dim], t[..., rot_dim:]
    x = t_mid.unflatten(-1, (-1, 2))
    x1, x2 = x.unbind(dim=-1)
    rot_half = torch.stack((-x2, x1), dim=-1).flatten(-2)
    t_mid = (t_mid * freqs.cos()) + (rot_half * freqs.sin())
    return torch.cat((t_mid, t_right), dim=-1)


@pytest.mark.parametrize("dh,W", [(128, 4), (64, 4), (128, 16)])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_oracle_rotation_is_apply_rotary_emb(dh, W, dtype):
    TL, B, H = 20, 2, 3
    S = TL + W * W
    g = torch.Generator().manual_seed(dh + W)
    x = torch.randn(B, S, H, dh, generator=g, dtype=dtype)
    freqs = dallepytorch_freqs(dh, TL, W)                    # [S, 6 nf]
    c, s = torch.cos(freqs.double()).to(dtype), torch.sin(freqs.double()).to(dtype)
    # apply_rotary_emb with the table's rounding of cos / sin: x [B, H, S, dh] as DALLE-pytorch holds it
    want = apply_rotary_emb_with(c, s, x.transpose(1, 2)).transpose(1, 2)
    oc, os_ = ORE.table(TL, W, dh, dtype)
    got = ORE.rotate(x, oc, os_)
    assert torch.equal(got, want)
    # and with float64 cos / sin of the angle, apply_rotary_emb itself
    if dtype == torch.float64:
        assert torch.allclose(ORE.rotate(x, torch.cos(freqs[:, 0::2].double()), torch.sin(freqs[:, 0::2].double())),
                              apply_rotary_emb(freqs.double(), x.transpose(1, 2)).transpose(1, 2), rtol=0, atol=1e-12)
    assert torch.equal(got[..., 6 * (dh // 6):], x[..., 6 * (dh // 6):])


def apply_rotary_emb_with(cos, sin, t):
    """apply_rotary_emb with given cos / sin [S, rot_dim] (each rounded once from the float64 evaluation)."""
    rot_dim = cos.shape[-1]
    t_mid, t_right = t[..., :rot_dim], t[..., rot_dim:]
    x1, x2 = t_mid.unflatten(-1, (-1, 2)).unbind(dim=-1)
    rot_half = torch.stack((-x2, x1), dim=-1).flatten(-2)
    return torch.cat(((t_mid * cos) + (rot_half * sin), t_right), dim=-1)


def _params_no_wpe(cfg, seed):
    p = O.init_params(cfg, seed=seed)
    return {k: v for k, v in p.items() if k != "positional_embedding/wpe"}


@pytest.mark.parametrize("bf16", [False, True])
def test_zero_angles_are_the_gelu_oracle_with_a_zero_wpe_bit_for_bit(bf16):
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        cfg = O.DalleConfig(256, 2, 2, 300, 64, 24, 64)
        params = _params_no_wpe(cfg, 3)
        g = torch.Generator().manual_seed(4)
        tokens = torch.cat([torch.randint(0, 300, (2, 24), generator=g), torch.randint(300, 364, (2, 64), generator=g)],
                           1)
        zero_wpe = dict(params, **{"positional_embedding/wpe": torch.zeros(cfg.text_seq_len + cfg.image_seq_len, 256)})
        ref = OG.forward(zero_wpe, tokens, cfg, bf16=bf16, activation="gelu")
        S, n = tokens.shape[1], 3 * (128 // 3 // 2)
        zero = (torch.ones(S, n), torch.zeros(S, n))
        got = ORE.forward(params, tokens, cfg, bf16=bf16, activation="gelu", tables=zero)
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
        rotated = ORE.forward(params, tokens, cfg, bf16=bf16, activation="gelu")
        assert not torch.equal(rotated[1], ref[1])
        for m in ORE.MUTATIONS:
            assert not torch.equal(ORE.forward(params, tokens, cfg, bf16=bf16, activation="gelu", rotary_mutate=m)[1],
                                   rotated[1]), m
    finally:
        torch.use_deterministic_algorithms(det)


# ------------------------------------------------------------------------------------------------ layout
@pytest.mark.parametrize("d,S", [(256, 40), (512, 1280)])
def test_layout_has_no_wpe_and_shrinks_by_s_d(d, S):
    with_pos = param_layout(d, 2, 1000, S)
    without = param_layout(d, 2, 1000, S, wpe=False)
    assert "wpe" in with_pos.entries and "wpe" not in without.entries
    assert with_pos.size - without.size == S * d
    assert without.order[:2] == ["wte", "l0.ln1_g"]
    assert [n for n in with_pos.order if n != "wpe"] == without.order
