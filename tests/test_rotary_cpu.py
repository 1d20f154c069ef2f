"""CPU side of rotary position embeddings: the rotary_dim / rotary_base keys at the four places a model is built
(DalleEngine, dalle_model_fn, models.DALLE, generate_dalle.py), the engine's cos / sin table against a direct float64
evaluation, and the oracle: relative positions in float64, no rotation bit for bit the GELU oracle's forward, and
transformers' GPT-NeoX apply_rotary_pos_emb."""
import math

import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.dalle_engine import DalleEngine, rope_table, validate_rotary
from dalle_mtf_b200.model_fns import dalle_model_fn, rotary_embedding
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_gelu as OG
from oracle import dalle_rotary as OR
from test_gelu_cpu import _Built, _generate_config

# n_embd 256, n_heads 2: head dim 128
ACCEPTED = [({}, (None, None)), ({"rotary_dim": None}, (None, None)),
            ({"rotary_dim": None, "rotary_base": None}, (None, None)),
            ({"rotary_dim": 2}, (2, 10000.0)), ({"rotary_dim": 32}, (32, 10000.0)), ({"rotary_dim": 128}, (128, 10000.0)),
            ({"rotary_dim": 64, "rotary_base": 500}, (64, 500.0)), ({"rotary_dim": 64, "rotary_base": 1.5}, (64, 1.5)),
            ({"rotary_dim": 64, "rotary_base": None}, (64, 10000.0))]
REJECTED = [{"rotary_dim": 3}, {"rotary_dim": 0}, {"rotary_dim": -2}, {"rotary_dim": 130}, {"rotary_dim": 256},
            {"rotary_dim": True}, {"rotary_dim": False}, {"rotary_dim": 32.0}, {"rotary_dim": "32"},
            {"rotary_dim": [32]}, {"rotary_dim": 32, "rotary_base": 1}, {"rotary_dim": 32, "rotary_base": 0.5},
            {"rotary_dim": 32, "rotary_base": -10000}, {"rotary_dim": 32, "rotary_base": float("inf")},
            {"rotary_dim": 32, "rotary_base": float("nan")}, {"rotary_dim": 32, "rotary_base": "10000"},
            {"rotary_dim": 32, "rotary_base": True}, {"rotary_base": 10000}, {"rotary_dim": None, "rotary_base": 500}]
MODEL = {"n_embd": 256, "n_heads": 2}


@pytest.mark.parametrize("params,want", ACCEPTED, ids=[repr(p) for p, _ in ACCEPTED])
def test_accepted_values(params, want):
    assert rotary_embedding({**MODEL, **params}) == want
    got = validate_rotary(params.get("rotary_dim"), params.get("rotary_base"), 128)
    assert got == (None if want[0] is None else want)


@pytest.mark.parametrize("params", REJECTED, ids=[repr(p) for p in REJECTED])
def test_other_values_are_rejected_where_a_model_is_built(tmp_path, params):
    with pytest.raises(ValueError, match="rotary"):
        rotary_embedding({**MODEL, **params})
    with pytest.raises(ValueError, match="rotary"):        # before any GPU work
        dalle_model_fn(None, None, "train", {**MODEL, **params})
    with pytest.raises(ValueError, match="rotary"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(params))
    with pytest.raises(ValueError, match="rotary"):
        DalleEngine(256, 1, 2, 10, 16, 4, 16, rotary_dim=params.get("rotary_dim"),
                    rotary_base=params.get("rotary_base"))
    with pytest.raises(ValueError, match="rotary"):
        G.main(_generate_config(tmp_path, params))


def test_rotary_dim_is_bounded_by_each_models_head_dim():
    """DALLE and DalleEngine take the head dim from their own n_embd / n_heads: 128 is valid at 256 / 2, not 256 / 4."""
    with pytest.raises(ValueError, match="rotary_dim"):
        DalleEngine(256, 1, 4, 10, 16, 4, 16, rotary_dim=128)
    with pytest.raises(ValueError, match="rotary_dim"):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=4,
              params={"rotary_dim": 128})
    for kw in ({}, {"rotary_dim": 128}, {"rotary_dim": 64, "rotary_base": 100.0}):
        with pytest.raises(L.DB200Error):       # the arguments pass; there is no device here
            DalleEngine(256, 1, 2, 10, 16, 4, 16, **kw)


@pytest.mark.parametrize("extra,want", [({}, (None, None)), ({"rotary_dim": 64}, (64, 10000.0)),
                                        ({"rotary_dim": 2, "rotary_base": 500}, (2, 500.0))])
def test_generate_cli_builds_the_engine_with_the_config_rotary(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the rotary embedding of its config (device work stubbed out)."""
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
    assert (seen["rotary_dim"], seen["rotary_base"]) == want


@pytest.mark.parametrize("S,r,base", [(1280, 128, 10000.0), (1280, 32, 10000.0), (1280, 2, 10000.0), (300, 64, 500.0),
                                      (2080, 128, 10000.0)])
def test_table_is_the_float64_evaluation_rounded_once(S, r, base):
    t = rope_table(S, r, base)
    assert t.dtype == torch.float32 and tuple(t.shape) == (S, 2, r // 2)
    h = r // 2
    c = torch.tensor([[math.cos(p * base ** (-2.0 * j / r)) for j in range(h)] for p in range(S)], dtype=torch.float64)
    s = torch.tensor([[math.sin(p * base ** (-2.0 * j / r)) for j in range(h)] for p in range(S)], dtype=torch.float64)
    for got, want in ((t[:, 0], c), (t[:, 1], s)):
        want32 = want.float()
        # libm and torch may differ in the last float64 bit; after the one rounding to fp32 at most a tie moves
        ulp = torch.finfo(torch.float32).eps * want32.abs().clamp_min(torch.finfo(torch.float32).tiny)
        assert ((got.double() - want).abs() <= ulp.double()).all()
        assert (got == want32).double().mean() > 0.9999
    assert torch.equal(t[:, 0], OR.table(S, r, base)[0]) and torch.equal(t[:, 1], OR.table(S, r, base)[1])
    assert torch.equal(t[0, 0], torch.ones(h)) and torch.equal(t[0, 1], torch.zeros(h))


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("r,base", [(128, 10000.0), (32, 10000.0), (2, 10000.0), (64, 77.0)])
def test_rotated_scores_depend_only_on_the_offset(r, base):
    """In float64, q_i . k_j after the rotation is a function of i - j: the same q and k vectors placed at every
    position give scores constant along each diagonal."""
    g = torch.Generator().manual_seed(r)
    S, H, dh = 48, 2, 128
    q = torch.randn(1, 1, H, dh, generator=g, dtype=torch.float64).expand(1, S, H, dh)
    k = torch.randn(1, 1, H, dh, generator=g, dtype=torch.float64).expand(1, S, H, dh)
    qr, kr = OR.rotate(q, r, base), OR.rotate(k, r, base)
    scores = torch.einsum("bihe,bjhe->bhij", qr, kr)[0]
    for off in range(-S + 1, S):
        dg = torch.diagonal(scores, offset=off, dim1=1, dim2=2)
        assert torch.allclose(dg, dg[:, :1].expand_as(dg), rtol=1e-10, atol=1e-10), off
    # the pass-through dims and v are untouched, and a rotation keeps each pair's norm
    assert torch.equal(qr[..., r:], q[..., r:])
    h = r // 2
    assert torch.allclose(qr[..., :h] ** 2 + qr[..., h:r] ** 2, q[..., :h] ** 2 + q[..., h:r] ** 2, rtol=1e-12)
    # every mutant changes the value (at r = 2 the two pair layouts are the same pair (x_0, x_1))
    for m in OR.MUTATIONS if r > 2 else ("neg_theta", "shift"):
        assert not torch.allclose(OR.rotate(q, r, base, m), qr, rtol=1e-6, atol=1e-9), m


@pytest.mark.parametrize("r,dh", [(128, 128), (32, 128), (2, 64), (24, 64)])
def test_oracle_is_gpt_neox_apply_rotary_pos_emb(r, dh):
    mod = pytest.importorskip("transformers.models.gpt_neox.modeling_gpt_neox")
    g = torch.Generator().manual_seed(dh + r)
    B, S, H = 2, 40, 3
    q = torch.randn(B, S, H, dh, generator=g, dtype=torch.float64)
    k = torch.randn(B, S, H, dh, generator=g, dtype=torch.float64)
    c, s = OR.table(S, r, 10000.0, torch.float64)
    cos, sin = torch.cat([c, c], -1)[None], torch.cat([s, s], -1)[None]          # [1, S, r]: emb = cat(freqs, freqs)
    qn, kn = mod.apply_rotary_pos_emb(q, k, cos, sin, unsqueeze_dim=2)
    assert torch.allclose(OR.rotate(q, r), qn, rtol=1e-12, atol=1e-12)
    assert torch.allclose(OR.rotate(k, r), kn, rtol=1e-12, atol=1e-12)
    # transformers' inverse frequencies: 1 / base^(arange(0, r, 2) / r)
    inv = 1.0 / (10000.0 ** (torch.arange(0, r, 2, dtype=torch.float64) / r))
    assert torch.allclose(torch.cos(torch.arange(S, dtype=torch.float64)[:, None] * inv), c, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("bf16", [False, True])
def test_no_rotation_is_the_gelu_oracle_bit_for_bit(bf16):
    """rotary None and r = 0 compute exactly oracle/dalle_gelu.forward (loss rows, logits and every gradient; torch's
    deterministic algorithms, without which the CPU index backward of wte is not bit-reproducible)."""
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _no_rotation_case(bf16)
    finally:
        torch.use_deterministic_algorithms(det)


def _no_rotation_case(bf16):
    cfg = O.DalleConfig(256, 2, 2, 300, 64, 24, 40)
    params = O.init_params(cfg, seed=3)
    g = torch.Generator().manual_seed(4)
    tokens = torch.cat([torch.randint(0, 300, (2, 24), generator=g), torch.randint(300, 364, (2, 40), generator=g)], 1)
    ref = OG.loss_and_grads(params, tokens, cfg, bf16=bf16, activation="gelu")
    for rot in (None, (0, 10000.0)):
        got = OR.loss_and_grads(params, tokens, cfg, bf16=bf16, activation="gelu", rotary=rot)
        for a, b in zip(got[:3], ref[:3]):
            assert torch.equal(a, b)
        assert all(torch.equal(got[3][k], ref[3][k]) for k in ref[3])
    # and a rotation changes the loss
    rotated = OR.loss_and_grads(params, tokens, cfg, bf16=bf16, activation="gelu", rotary=(128, 10000.0))
    assert not torch.equal(rotated[1], ref[1])
