"""GPU tests of DalleEngine across the configurations its constructor accepts: every row of the edge table of
tests/test_dalle_config_space_cpu.py.

Accepted rows, each with and without the logits mask:
  * one training step (loss, loss rows, every gradient, one Adam update) against the float64-composed oracle of
    test_logits_mask_gpu._engine_vs_oracle, with its bounds (a gradient's relfro within 1.25 x the bf16 oracle's +
    1e-2); each prints its worst err / bound;
  * generation on the row's geometry with sharpened weights: greedy eager and graph-replayed generation are the same
    tokens and the argmax of the full forward (test_prefill_gpu.greedy_agrees_with_full_forward), and the prefill at P
    gives the logits of decoding to P.
Filtered sampling at its limit: with 51 200 image codes a filtered draw, guided and unguided, keeps to the kept set of
oracle/sampling.py; with 51 201 the sampler refuses a filter and plain sampling still runs.
Refused rows: DalleEngine raises before any CUDA allocation, and dalle_model_fn raises the same error from the
constructor.
"""
import traceback

import numpy as np
import pytest
import torch

from test_dalle_config_space_cpu import EDGE_REFUSED, EDGE_ROWS
from test_guidance_gpu import guided_x
from test_logits_mask_gpu import _engine_vs_oracle
from test_prefill_gpu import greedy_agrees_with_full_forward, relfro, sharp_engine
from test_sampling_filter_gpu import MARGIN

pytestmark = pytest.mark.gpu

DEV = "cuda"
I32 = torch.int32
GEN_B = 4


@pytest.mark.parametrize("mask", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_training_step_matches_the_oracle(name, mask):
    (d, nl, H, tv, iv, ts, isl, B), kw = EDGE_ROWS[name]
    bad, worst = _engine_vs_oracle(d, nl, H, tv, iv, ts, isl, B, seed=len(name), mask=mask, adam=True, **kw)
    print(f"[config-space] {name} mask {mask}: worst err/bound {worst:.4f}")
    assert not bad, bad


def _engine_keywords(kw, mask):
    out = {"logits_mask": mask}
    if "types" in kw:
        out.update(attention_types=kw["types"], local_attention_radius=kw.get("radius", 8),
                   conv_attention_kernel=kw.get("kernel", 3))
    if kw.get("row_col"):
        out["image_position_embedding"] = "row_col"
    if kw.get("pp"):
        out["per_position_padding"] = True
    return out


@pytest.mark.parametrize("mask", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("name", list(EDGE_ROWS))
def test_generation_follows_the_full_forward(name, mask):
    from dalle_mtf_b200.sampling import DalleSampler
    (d, nl, H, tv, iv, ts, isl, _), kw = EDGE_ROWS[name]
    eng, _, _ = sharp_engine(d, nl, H, tv, iv, ts, isl, **_engine_keywords(kw, mask))
    g = torch.Generator().manual_seed(len(name))
    text = torch.randint(0, tv, (GEN_B, ts), generator=g).to(I32).to(DEV)
    smp = DalleSampler(eng)
    eager, step_logits = smp.generate(text, temperature=0, return_logits=True)
    graphed = smp.generate_graphed(text, temperature=0)
    torch.cuda.synchronize()
    assert torch.equal(eager, graphed)
    assert torch.equal(eager[:, :ts], smp._captions(text))
    io = eng.image_offset
    assert ((eager[:, ts:] >= io) & (eager[:, ts:] < io + iv)).all()
    greedy_agrees_with_full_forward(eng, eager, ts)
    dec = torch.stack(step_logits, 1)                      # [B, S - 1, V]: the logits after each position
    S = ts + isl
    for P in sorted({ts, (ts + S) // 2, S - 1}):
        if P >= S:
            continue
        kc = [torch.zeros_like(c) for c in smp.kc]
        vc = [torch.zeros_like(c) for c in smp.vc]
        logits = eng.prefill(eager[:, :P].contiguous(), kc, vc)
        err = relfro(logits[:, :eng.V], dec[:, P - 1])
        assert err < 2e-2, (P, err)
    print(f"[config-space] {name} mask {mask}: greedy generation and prefill agree")


# ------------------------------------------------------------------------------------------------ filtered sampling
def _wide_engine(iv):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    eng = DalleEngine(256, 1, 2, 64, iv, 4, 4)
    eng.init_params(5)
    return eng


def test_filtered_draws_at_the_limit_keep_to_the_oracle_kept_set():
    from dalle_mtf_b200.sampling import FILTER_MAX_IDS, DalleSampler
    from oracle.sampling import boundary_margin, keep_mask
    eng = _wide_engine(FILTER_MAX_IDS)
    ts, tv, iv, S = 4, 64, FILTER_MAX_IDS, eng.S
    text = torch.randint(0, tv, (2, ts), generator=torch.Generator().manual_seed(1)).to(I32).to(DEV)
    smp = DalleSampler(eng)
    k, p = 8, float(np.float32(0.9))
    for gs in (None, 3.0):
        gen = torch.Generator(device=DEV).manual_seed(2)
        toks, step_logits = smp.generate(text, temperature=1.0, generator=gen, top_k=k, top_p=0.9,
                                         guidance_scale=gs, return_logits=True)
        checked = 0
        for pos in range(ts - 1, S - 1):
            x = (guided_x(step_logits[pos], 2, tv, tv + iv, gs, 1.0) if gs is not None
                 else step_logits[pos][:, tv:tv + iv].cpu().numpy()).astype(np.float64)
            mask = keep_mask(x, k, p)
            ok = boundary_margin(x, k, p) > MARGIN
            tok = toks[:, pos + 1].cpu().numpy() - tv
            assert ((0 <= tok) & (tok < iv)).all()
            assert mask[np.arange(len(tok)), tok][ok].all(), (gs, pos)
            checked += int(ok.sum())
        assert checked >= 0.9 * 2 * (S - ts), (gs, checked)
        graphed = smp.generate_graphed(text, temperature=1.0, top_k=k, top_p=0.9, guidance_scale=gs)
        assert ((graphed[:, ts:] >= tv) & (graphed[:, ts:] < tv + iv)).all()
    # top-1 keeps the maximum only: the filtered draw is the greedy one
    assert torch.equal(smp.generate(text, temperature=1.0, top_k=1), smp.generate(text, temperature=0))
    print(f"[config-space] image_vocab_size {iv}: filtered draws, guided and unguided, keep to the kept set")


def test_past_the_limit_the_sampler_refuses_a_filter_and_plain_sampling_runs():
    from dalle_mtf_b200.sampling import FILTER_MAX_IDS, DalleSampler
    eng = _wide_engine(FILTER_MAX_IDS + 1)
    tv, iv, ts = 64, FILTER_MAX_IDS + 1, 4
    text = torch.randint(0, tv, (2, ts), generator=torch.Generator().manual_seed(3)).to(I32).to(DEV)
    smp = DalleSampler(eng)
    for flt in (dict(top_k=8), dict(top_p=0.9), dict(top_k=8, guidance_scale=3.0)):
        for call in (smp.generate, smp.generate_graphed, smp.complete):
            with pytest.raises(ValueError, match="image_vocab_size"):
                call(text, temperature=1.0, **flt)
    for gs in (None, 3.0):
        out = smp.generate(text, temperature=1.0, guidance_scale=gs)
        graphed = smp.generate_graphed(text, temperature=1.0, guidance_scale=gs, top_k=iv)   # top_k >= iv: no filter
        for o in (out, graphed):
            assert torch.equal(o[:, :ts], text) and ((o[:, ts:] >= tv) & (o[:, ts:] < tv + iv)).all()
    assert torch.equal(smp.generate(text, temperature=0), smp.generate_graphed(text, temperature=0))


# ------------------------------------------------------------------------------------------------ refused rows
def _raised_in_the_constructor(excinfo):
    """The error came from validate_geometry, called by DalleEngine.__init__ before its first allocation."""
    frames = [f.name for f in traceback.extract_tb(excinfo.tb)]
    assert frames[-1] == "validate_geometry" and frames[-2] == "__init__", frames


@pytest.mark.parametrize("name", sorted(EDGE_REFUSED))
def test_refused_geometry_raises_before_allocating(name):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    (d, H, ts, isl, tv, iv), exc = EDGE_REFUSED[name]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(exc) as e:
        DalleEngine(d, 2, H, tv, iv, ts, isl)
    assert torch.cuda.memory_allocated() == before
    _raised_in_the_constructor(e)


@pytest.mark.parametrize("name", sorted(EDGE_REFUSED))
def test_refused_geometry_through_the_model_fn(name, tmp_path, monkeypatch):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from test_engine_gpu import _tiny_params
    (d, H, ts, _, tv, iv), exc = EDGE_REFUSED[name]
    _, params = _tiny_params(tmp_path)
    params.update(n_embd=d, n_heads=H, text_seq_len=ts, text_vocab_size=tv, image_vocab_size=iv,
                  vae_random_init=True)
    built = []
    init = DalleEngine.__init__

    def spy(self, *a, **k):
        built.append(self)
        init(self, *a, **k)

    monkeypatch.setattr(DalleEngine, "__init__", spy)
    with pytest.raises(exc) as e:
        dalle_model_fn(None, None, "train", params)
    monkeypatch.undo()
    _raised_in_the_constructor(e)
    assert len(built) == 1 and not hasattr(built[0], "grads")   # the engine got no buffer
    with pytest.raises(exc) as direct:
        DalleEngine(d, 2, H, tv, iv, ts, 16)
    assert str(e.value) == str(direct.value)
