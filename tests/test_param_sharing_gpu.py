"""Parameter sharing on the GPU (share_input_output_emb, shared_attn_ids, shared_ff_ids).

Kernels: the tied vocabulary products read wte [Vpad, d] as a K-major B.  CE_STATS, CE_GRAD, the weighted CE_GRAD
(the new gemm_tc_kernel<0, 0, false, true>), the wgrad (dlogits^T hf, both MN-major) and the dgrad (dlogits wte, B
MN-major) are checked against float64 with test_dalle_kernels_gpu.py's and test_loss_weights_gpu.py's bounds at the
dalle_example, dalle_coco and 12B vocabularies and widths, by running those checks with every vocabulary B operand
handed over transposed (K-major).  Every vocabulary-product class a tied engine launches (recorded with
launch_census.OpsRecorder) is one of the checked ones.

Engine: against oracle/dalle_sharing.py (loss, loss rows, logits, every gradient) with its mutants failing the same
bounds; against unshared / untied twins holding copies of the shared weights; wte's pad rows under Adam; in-process
data-parallel ranks (bit for bit except the slots that sum several contributions) and ZeRO-1 bit for bit; checkpoints through dalle_model_fn; decoding, graph replay, the prefill and
guided completion."""
import pytest
import torch

from float64_bounds import DEV
from test_loss_weights_gpu import _engine, _step, _tiny_params, relfro

pytestmark = pytest.mark.gpu
BF16, F32, I32 = torch.bfloat16, torch.float32, torch.int32
TAG = "param_sharing"


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


# ------------------------------------------------------------------------------------------------ kernels
class KMajorVocab:
    """`ops` with every vocabulary product's B operand (a [K, N] MN-major weight of a product with N > K) handed to the
    GEMM transposed, K-major, as a tied wte is.  `modes` records the epilogues that went through it."""

    def __init__(self, ops):
        self._ops, self.modes = ops, []

    def __getattr__(self, name):
        return getattr(self._ops, name)

    def gemm(self, a, b, out, M, N, K, *, b_mn=False, **kw):
        if b_mn and tuple(b.shape) == (K, N) and N > K and not kw.get("a_mn"):
            self.modes.append((kw.get("mode"), kw.get("ce_weights") is not None))
            return self._ops.gemm(a, b.t().contiguous(), out, M, N, K, b_mn=False, **kw)
        return self._ops.gemm(a, b, out, M, N, K, b_mn=b_mn, **kw)


@pytest.mark.parametrize("config", ["dalle_example_b200", "dalle_coco_b200", "dalle_12b_b200"])
def test_k_major_cross_entropy_at_the_real_vocabulary(ops, config):
    from dalle_mtf_b200 import lib as L
    from test_dalle_kernels_gpu import CONFIGS, real_vocabulary_operands, run_cross_entropy
    shim = KMajorVocab(ops)
    T = CONFIGS[config]
    K, V, Vpad, h, W, bias, labels = real_vocabulary_operands(ops, config, T)
    run_cross_entropy(shim, f"{config} K-major CE T={T} V={V}", T, K, V, Vpad, labels=labels, h=h, W=W, bias=bias)
    assert {m for m, _ in shim.modes} == {L.EPI_CE_STATS, L.EPI_CE_GRAD}


@pytest.mark.parametrize("config,T,weights,z", [("dalle_example_b200", 40960, (1.0, 7.0), 1e-4),
                                                ("dalle_coco_b200", 20480, (1.0, 7.0), 0.0),
                                                ("dalle_example_b200", 2 * 1280 + 333, (0.0, 1.0), 1e-4)])
def test_k_major_weighted_cross_entropy_against_float64(ops, config, T, weights, z):
    from oracle import loss_weights as OW
    from test_dalle_kernels_gpu import _config, _gen, ce_operands
    from test_loss_weights_gpu import _labels, run_weighted_ce
    cfg = _config(config)
    K, V = cfg["n_embd"], cfg["text_vocab_size"] + cfg["image_vocab_size"] + 1
    Vpad, S, TL = (V + 63) // 64 * 64, 1280, cfg["text_seq_len"]
    g = _gen(T + K)
    h, W, bias, _, _ = ce_operands(T, K, V, Vpad, g)
    labels = _labels(ops, cfg, T, S, g)
    shim = KMajorVocab(ops)
    mutants = (OW.LossQuirks(text_rows_offset=0),) if weights == (1.0, 7.0) else ()
    run_weighted_ce(shim, f"{config} K-major weighted CE T={T} w={weights} z={z}", T, K, V, Vpad, S, TL,
                    labels=labels, h=h, W=W, bias=bias, weights=weights, z=z, global_batch=max(1, T // S),
                    mutants=mutants)
    assert any(w for _, w in shim.modes)


def _tied_products(d, T, Vpad):
    """The tied backward's wgrad (M = Vpad, N = d, K = T, both MN-major, ATOMIC split-K) and dgrad (M = T, N = d,
    K = Vpad, A K-major, B MN-major, STORE), and the fp32 logits with bias of logits(), the prefill and the decoder
    (M = 4096 rows, N = Vpad, K = d, B K-major) in test_dalle_kernels_gpu's descriptor form."""
    from dalle_mtf_b200 import lib as L
    wgrad = ("gemm", Vpad, d, T, 1, 1, L.EPI_ATOMIC, "torch.float32", False, False, False, False, 0, 0, False, None)
    dgrad = ("gemm", T, d, Vpad, 0, 1, L.EPI_STORE, "torch.bfloat16", False, False, False, False, 1, 0, False, None)
    logits = ("gemm", 4096, Vpad, d, 0, 0, L.EPI_STORE, "torch.float32", True, False, False, False, 1, 0, False, None)
    return (("wgrad", wgrad), ("dgrad", dgrad), ("logits", logits))


@pytest.mark.parametrize("config", ["dalle_example_b200", "dalle_coco_b200", "dalle_12b_b200"])
def test_tied_wgrad_and_dgrad_against_float64(ops, config):
    from test_dalle_kernels_gpu import CONFIGS, _config, _sm, check_gemm, gemm_operands, gemm_splits, run_gemm
    cfg = _config(config)
    d, V = cfg["n_embd"], cfg["text_vocab_size"] + cfg["image_vocab_size"] + 1
    Vpad, T = (V + 63) // 64 * 64, CONFIGS[config]
    for k, (what, desc) in enumerate(_tied_products(d, T, Vpad)):
        M, K = desc[1], desc[3]
        o = gemm_operands(ops, desc, M, K, seed=11 + k)
        run_gemm(ops, o)
        splits = gemm_splits(M, desc[2], K, desc[6], desc[12], _sm())
        check_gemm(f"{config} tied {what} M={M} N={desc[2]} K={K}", o, splits)


def test_every_vocabulary_product_class_of_a_tied_engine_is_checked(ops):
    """Record a tied dalle_example-shaped step (plain, weighted, logits mask) and its logits / prefill / decoding: every
    GEMM whose B is wte or which writes G(wte) is of a class the tests above check (K-major B CE_STATS / CE_GRAD /
    weighted CE_GRAD / STORE, the MN-major ATOMIC wgrad and STORE dgrad)."""
    from launch_census import OpsRecorder
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.sampling import DalleSampler
    seen = set()
    state = {}

    def describe(entry, A):
        if entry != "gemm":
            return None
        e = state["eng"]
        w, gw = e.W("wte"), e.G("wte")
        touches = lambda t: t is not None and t.data_ptr() >= w.data_ptr() and \
            t.data_ptr() < w.data_ptr() + w.numel() * w.element_size()   # noqa: E731
        touches_g = lambda t: t is not None and gw.data_ptr() <= t.data_ptr() < \
            gw.data_ptr() + gw.numel() * gw.element_size()   # noqa: E731
        if not (touches(A["b"]) or touches_g(A["out"])):
            return None
        cls = (A["mode"], int(A["a_mn"]), int(A["b_mn"]), A["ce_weights"] is not None)
        return cls, None

    d, tv, iv = 512, 50258, 512
    for kw in (dict(), dict(loss_weights=(1.0, 7.0), z_loss=1e-4), dict(logits_mask=True)):
        eng = state["eng"] = _Cfg.engine(d, 2, 4, tv, iv, 64, 64, share_input_output_emb=True, **kw)
        eng.init_params(1)
        tok = _tokens(eng, 2, 5)
        with OpsRecorder(describe, nested=("gemm",)) as rec:
            _step(eng, tok, 1.0 / tok.numel())
            eng.logits(tok[:1])
            smp = DalleSampler(eng)
            smp.generate(tok[:1, :64].contiguous(), 0.0)
        seen |= set(rec.classes())
    checked = {(L.EPI_CE_STATS, 0, 0, False), (L.EPI_CE_GRAD, 0, 0, False), (L.EPI_CE_GRAD, 0, 0, True),
               (L.EPI_STORE, 0, 0, False), (L.EPI_ATOMIC, 1, 1, False), (L.EPI_STORE, 0, 1, False)}
    print(f"[{TAG}] tied vocabulary classes {sorted(seen)}")
    assert seen <= checked and (L.EPI_CE_GRAD, 0, 0, True) in seen and (L.EPI_ATOMIC, 1, 1, False) in seen


class _Cfg:
    @staticmethod
    def engine(d, Lyr, H, tv, iv, ts, isl, **kw):
        from dalle_mtf_b200.dalle_engine import DalleEngine
        return DalleEngine(d, Lyr, H, tv, iv, ts, isl, **kw)


def _tokens(eng, B, seed):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, eng.text_vocab_size - 1, (B, eng.text_seq_len), generator=g)
    image = torch.randint(0, eng.image_vocab_size, (B, eng.image_seq_len), generator=g) + eng.image_offset
    return torch.cat([text, image], 1).to(I32).to(DEV)


# ------------------------------------------------------------------------------------------------ engine vs oracle
VARIANTS = {
    "tied": dict(types=("global", "global"), tie=True, mutants=("untied_grad",)),
    "tied_stable": dict(types=("global", "global"), tie=True, stable=True, b2=-60.0,
                        mutants=("untied_grad", "shrink_output")),
    "shared": dict(types=("global", "axial_row", "global"), attn=[0, 1], ff=[0, 1],
                   mutants=("shared_norms", "last_owner", "no_cycle")),
    "mixed_gmlp": dict(types=("axial_row", "axial_col", "mlp") * 2, attn=[0, 1, 2], ff=[0], tie=True,
                       sandwich_norm=True, layer_scale=True, mutants=("shared_norms", "last_owner", "untied_grad")),
    "recompute_dropout": dict(types=("global", "axial_col", "global", "axial_col"), attn=[0, 1], ff=[0], tie=True,
                              recompute_grad=True, dropout=(0.1, 0.1, 0.1), mutants=("shared_norms",)),
    "gated_rotary_shift": dict(types=("global", "global"), attn=[0], ff=[0], tie=True, gated_mlp=True,
                               rotary_dim=16, shift_tokens=True, mutants=("last_owner",)),
}


def _model(types, seed=3, d=256, H=2, TL=28, W=10, gated=False, b2=None, sandwich=False, scale=False):
    import axial_oracle as AX
    from oracle import dalle as O, dalle_glu as OGL, dalle_gmlp as OM, dalle_layer_scale as OLS
    from oracle import dalle_local as OL, dalle_sandwich as OSW
    cfg = OL.LocalConfig(d, len(types), H, 300, 64, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 1)
    if sandwich:
        params = OSW.init_params(params, cfg, seed + 11)
    if gated:
        params = OGL.init_params(params, cfg, seed + 12)
    if scale:
        params = OLS.init_params(params, cfg, seed=seed + 13)
    g = torch.Generator().manual_seed(seed + 2)
    for k in params:   # every layer's norms and biases differ, so that sharing a norm is visible
        if k.endswith("norm_1/g") or k.endswith("norm_2/g"):
            params[k] = 1 + 0.3 * torch.randn(params[k].shape, generator=g)
        elif k.endswith("norm_1/b") or k.endswith("norm_2/b") or k.endswith("o_b") or k.endswith("bias"):
            params[k] = 0.05 * torch.randn(params[k].shape, generator=g)
    if b2 is not None:
        params[f"layer_{len(types) - 1}/mlp/mlp_linear_2/bias"] = torch.full((d,), b2)
    tokens = O.assemble_tokens(torch.randint(0, 299, (2, TL), generator=g),
                               torch.randint(0, 64, (2, W * W), generator=g), 300)
    return AX.AxialConfig(**{**cfg.__dict__}), params, tokens


def _variant(name):
    v = dict(VARIANTS[name])
    types, mutants = v.pop("types"), v.pop("mutants")
    tie, attn, ff = v.pop("tie", False), v.pop("attn", None), v.pop("ff", None)
    return types, mutants, tie, attn, ff, v


def _violations(loss, rows, grads, ref32, ref16):
    """The bounds of test_layer_scale_gpu._vs_oracle: 1.25 x the bf16-policy oracle's own distance from the fp32 oracle
    plus a floor; a gradient the engine does not have (another naming) is a violation."""
    l32, r32, g32 = ref32
    l16, r16, g16 = ref16
    bad = []
    if abs(loss - l32.item()) > 1.25 * abs(l16.item() - l32.item()) + 1e-3 * abs(l32.item()):
        bad.append(("loss", loss, l32.item()))
    if relfro(rows, r32) > 1.25 * relfro(r16, r32) + 5e-3:
        bad.append(("loss_rows", relfro(rows, r32)))
    return bad + [(k, "missing") for k in g32 if k not in grads]


def _grad_violations(grads, g32, g16, gm=None):
    gm = g32 if gm is None else gm
    bad = []
    for k in gm:
        if k in grads and g32.get(k) is not None and g32[k].any():
            lim = 1.25 * relfro(g16[k], g32[k]) + 1e-2
            if relfro(grads[k], gm[k]) > lim:
                bad.append((k, relfro(grads[k], gm[k]), lim))
    return bad


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_engine_matches_the_oracle_and_not_its_mutants(variant):
    import axial_oracle as AX
    from oracle import dalle_layer_scale as OLS, dalle_sharing as OSH
    types, mutants, tie, attn, ff, v = _variant(variant)
    cfg, params, tokens = _model(types, gated=v.get("gated_mlp", False), b2=v.pop("b2", None),
                                 sandwich=v.get("sandwich_norm", False), scale=v.get("layer_scale", False))
    dropout = (v["dropout"], 7, 3, 0) if "dropout" in v else None
    okw = dict(layers=AX, sandwich_norm=v.get("sandwich_norm", False), layer_scale=v.get("layer_scale", False),
               stable=v.get("stable", False), shift_tokens=v.get("shift_tokens", False), dropout=dropout)
    if v.get("gated_mlp"):
        okw.update(gated=True, activation="gelu", rotary=(v["rotary_dim"], 10000.0))
        v["activation"] = "gelu"

    def oracle(bf16, m=None):
        loss, rows, logits, grads = OSH.loss_and_grads(params, tokens, cfg, tie, attn, ff, m, forward=OLS.forward,
                                                       bf16=bf16, **okw)
        return loss, rows, logits, grads

    ref32, ref16 = oracle(False), oracle(True)
    shared = OSH.share(params, cfg, tie, attn, ff)
    eng = _engine(cfg, attention_types=list(types), conv_attention_kernel=3, local_attention_radius=8, dropout_seed=7,
                  share_input_output_emb=tie, shared_attn_ids=attn, shared_ff_ids=ff, **v)
    eng.load_params(shared)
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok, step=3 if dropout else None)
    eng.backward(1.0 / T)
    torch.cuda.synchronize()
    loss, rows = acc.item() / T, eng._bufs["loss_rows"].view(2, -1).clone()
    grads = eng.export_params(eng.grads)
    assert set(grads) == set(shared) == set(ref32[3])
    bad = _violations(loss, rows, grads, (ref32[0], ref32[1], ref32[3]), (ref16[0], ref16[1], ref16[3])) + \
        _grad_violations(grads, ref32[3], ref16[3])
    print(f"[{TAG}] {variant}: loss {loss:.6f} oracle {ref32[0].item():.6f}, violations {bad}")
    assert not bad
    if not dropout:
        e = relfro(eng.logits(tok), ref32[2])
        assert e <= 1.25 * relfro(ref16[2], ref32[2]) + 1e-2, e
    for m in mutants:
        ml, mr, _, mg = oracle(False, m)
        mbad = _violations(loss, rows, grads, (ml, mr, mg), (ref16[0], ref16[1], ref16[3])) + \
            _grad_violations(grads, ref32[3], ref16[3], mg) + [(k, "extra") for k in grads if k not in mg]
        print(f"[{TAG}]   mutant {m}: {len(mbad)} violated bounds, e.g. {mbad[:2]}")
        assert mbad, m


@pytest.mark.parametrize("mask,weights", [(True, None), (False, ((1.0, 7.0), 1e-4)), (True, ((1.0, 7.0), 1e-4))],
                         ids=["logits_mask", "weighted", "mask_weighted"])
def test_tied_engine_with_the_logits_mask_and_the_weighted_loss_matches_the_oracle(mask, weights):
    """The masked windows become row windows of the tied wte (the image window's rows past V in its zero pad)."""
    import axial_oracle as AX
    from oracle import dalle_layer_scale as OLS, dalle_sharing as OSH, logits_mask as OLM
    types, tie, attn, ff = ("global", "global", "global"), True, [0], [0, 1]
    cfg, params, tokens = _model(types, seed=5)
    w, z = weights if weights else (None, 0.0)

    def oracle(bf16, m=None):
        fwd = OSH.wrap(OLS.forward, cfg, tie, attn, ff, m)
        loss, rows, _, logits, grads = OLM.loss_and_grads(OSH.share(params, cfg, tie, attn, ff, m), tokens, cfg, 300,
                                                          weights=w, z=z, mask=mask,
                                                          forward=lambda p, t: fwd(p, t, cfg, layers=AX, bf16=bf16))
        return loss, rows, logits, grads

    ref32, ref16 = oracle(False), oracle(True)
    eng = _engine(cfg, attention_types=list(types), logits_mask=mask, share_input_output_emb=tie, shared_attn_ids=attn,
                  shared_ff_ids=ff, **(dict(loss_weights=w, z_loss=z) if w else {}))
    eng.load_params(OSH.share(params, cfg, tie, attn, ff))
    tok = tokens.to(I32).to(DEV)
    T = tok.numel()
    eng.zero_grads()
    acc = eng.forward(tok)
    eng.backward(1.0 if w else 1.0 / T)
    torch.cuda.synchronize()
    loss = acc[0].item() if w else acc.item() / T
    rows = eng._bufs["loss_rows"].view(2, -1).clone()
    grads = eng.export_params(eng.grads)
    bad = _violations(loss, rows, grads, (ref32[0], ref32[1], ref32[3]), (ref16[0], ref16[1], ref16[3])) + \
        _grad_violations(grads, ref32[3], ref16[3])
    print(f"[{TAG}] mask {mask} weights {weights}: loss {loss:.6f} oracle {ref32[0].item():.6f}, violations {bad}")
    assert not bad
    got = eng.logits(tok)
    fin = torch.isfinite(got).cpu()
    assert relfro(got.cpu()[fin], ref32[2][fin]) <= 1.25 * relfro(ref16[2][fin], ref32[2][fin]) + 1e-2
    ml, mr, _, mg = oracle(False, "untied_grad")
    assert _violations(loss, rows, grads, (ml, mr, mg), (ref16[0], ref16[1], ref16[3])) + \
        _grad_violations(grads, ref32[3], ref16[3], mg)


# ------------------------------------------------------------------------------------------------ twins
def _twin_pair(tie, attn, ff, types=("global", "global", "global", "global"), seed=4, **kw):
    """A shared engine and its unshared twin holding copies of the shared weights (same oracle dict expanded)."""
    from oracle import dalle_sharing as OSH
    cfg, params, tokens = _model(types, seed=seed, TL=24, W=8)
    shared = OSH.share(params, cfg, tie, attn, ff)
    full = {k: v.detach().clone() for k, v in OSH.expand(shared, cfg, tie, attn, ff).items()}
    eng = _engine(cfg, attention_types=list(types), share_input_output_emb=tie, shared_attn_ids=attn,
                  shared_ff_ids=ff, **kw)
    twin = _engine(cfg, attention_types=list(types), **kw)
    eng.load_params(shared)
    twin.load_params(full)
    return cfg, eng, twin, tokens.to(I32).to(DEV)


@pytest.mark.parametrize("recompute", [False, True], ids=["saved", "recompute"])
def test_shared_model_equals_its_unshared_twin(recompute):
    """Same weights: bit-identical loss rows, logits and unshared gradients; each shared gradient is the fp32 sum of
    the twin's per-layer gradients within fp32 reassociation: the shared slot adds each layer's split-K slices and
    column-sum partials into one running sum where the twin sums them per layer, so per element
    |g - sum_j g_j| <= 8 n 2^-24 sum_j |g_j| + 1e-6 max |sum_j g_j|, n the number of users."""
    from dalle_mtf_b200.dalle_engine import ATTN_MODULE, FF_MODULE
    attn, ff = [0, 1], [0]
    cfg, eng, twin, tok = _twin_pair(False, attn, ff, recompute_grad=recompute)
    T = tok.numel()
    ge, gt = _step(eng, tok, 1.0 / T), _step(twin, tok, 1.0 / T)
    assert torch.equal(eng._bufs["loss_rows"], twin._bufs["loss_rows"])
    assert torch.equal(eng.logits(tok), twin.logits(tok))
    worst = 0.0
    for name in twin.layout.order:
        p, k = (name.split(".") + [None])[:2] if name.startswith("l") and "." in name else (None, None)
        if k in ATTN_MODULE + FF_MODULE:
            i = int(p[1:])
            owners = eng.ff_owner if k in FF_MODULE else eng.attn_owner
            if owners[i] != i:
                continue
            users = [j for j in range(eng.L) if owners[j] == i]
            parts = [twin.G(f"l{j}.{k}") for j in users]
            want = sum(x.double() for x in parts)
            bound = 8 * len(users) * 2.0 ** -24 * sum(x.double().abs() for x in parts) + 1e-6 * want.abs().max()
            err = (eng.G(name).double() - want).abs()
            assert (err <= bound).all(), name
            worst = max(worst, (err / bound.clamp_min(1e-300)).max().item())
        else:
            assert torch.equal(eng.G(name), twin.G(name)), name
    print(f"[{TAG}] twin recompute={recompute}: shared gradients within {worst:.3f} of the reassociation bound")
    del ge, gt


def test_tied_model_against_its_untied_twin():
    """wout[:, :V] = wte^T: the forward differs only in the B descriptor's transpose bit.  Reported: whether the
    losses and logits are bit-identical; required: both within the float64-anchored oracle bounds of
    test_engine_matches_the_oracle_and_not_its_mutants (the tied variant), and wte's gradient equal to the twin's
    embedding gradient plus its wout gradient transposed within fp32 rounding of the sum."""
    cfg, eng, twin, tok = _twin_pair(True, None, None)
    T = tok.numel()
    _step(eng, tok, 1.0 / T)
    _step(twin, tok, 1.0 / T)
    same_rows = torch.equal(eng._bufs["loss_rows"], twin._bufs["loss_rows"])
    le, lt = eng.logits(tok), twin.logits(tok)
    print(f"[{TAG}] tied vs untied twin: loss rows bit-identical {same_rows}, logits bit-identical "
          f"{torch.equal(le, lt)}, max |diff| {(le - lt).abs().max().item():.3e}")
    assert relfro(le, lt) < 1e-5
    V = eng.V
    ge = eng.G("wte")[:V].double()
    want = twin.G("wte").double() + twin.G("wout")[:, :V].t().double()
    bound = 2.0 ** -23 * (twin.G("wte").double().abs() + twin.G("wout")[:, :V].t().double().abs()) + 1e-12
    assert ((ge - want).abs() <= bound + 1e-3 * want.abs().max()).all()


def test_pad_rows_of_a_tied_wte_stay_exactly_zero_through_adam():
    cfg, eng, _, tok = _twin_pair(True, [0], [0])
    for wd in (0.0, 0.01):
        for _ in range(3):
            _step(eng, tok, 1.0 / tok.numel())
            eng.optimizer_step(1e-3, weight_decay=wd)
        torch.cuda.synchronize()
        V = eng.V
        assert eng.layout.entries["wte"][1][0] == eng.Vpad > V
        for buf in (eng.master, eng.adam_m, eng.adam_v, eng.grads):
            assert not eng.layout.view(buf, "wte")[V:].any()
        assert not eng.W("wte")[V:].float().any()
        assert eng.W("wte")[:V].float().abs().sum() > 0


# ------------------------------------------------------------------------------------------------ parallel
def test_in_process_ranks_equal_one_rank_with_micro_batches(monkeypatch, tmp_path):
    """tests/test_data_parallel_gpu.py's criterion with every key, W = 2 and 3.  The group fails a bucket whose range
    changes after its all-reduce was launched (a shared module in the wrong bucket would) and checks that the buckets
    cover the buffer.  Tokens, loss rows, the loss and every gradient slot with one contribution per micro-batch are
    bit-identical.  A slot several layers (or, tied, the gather and the vocabulary product) add into is not: one rank
    adds every contribution of every micro-batch into one running fp32 sum, while W ranks add each rank's own
    contributions first and all-reduce those partial sums, a different association.  So those slots (wte and the
    shared modules) are the only ones allowed to differ at the first step, and only in the gradient and the state that
    follows."""
    from test_data_parallel_gpu import FEATURES, _Rec, _check_coverage, _dalle_data, _dalle_params, _dalle_ranks, \
        _dalle_reference, _seq_len, STEPS
    shared = {"wte"} | {f"l{i}.{k}" for i in (0, 1) for k in ("wqkv", "wo", "o_b")} | \
        {f"l0.{k}" for k in ("w1", "b1", "w2", "b2")}
    for W in (2, 3):
        rec = _Rec(monkeypatch)
        # 4 layers: attention ids 0 1 0 1 (owners 0, 1), MLP ids 1 0 2 1 (layers 0 and 3 share, owner 0)
        extra = dict(FEATURES, attention_types=[[["global", "axial_row"], 2]], share_input_output_emb=True,
                     shared_attn_ids=[0, 1], shared_ff_ids=[1, 0, 2])
        B = 12
        make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
        p = make()
        feats, caps = _dalle_data(p, B, seed=W)
        ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
        group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
        assert (n_r, aux_r) == (n, aux_off)
        _check_coverage(group.trace, n, aux_off, STEPS)
        # the first step: nothing but those slots' gradients and the state they update (later steps start from that
        # state, so their forward may differ in the last bits too)
        assert {kind for kind, v in chk.failed.items() if any(k == 0 for _, k in v)} <= {"gradient", "state"}, \
            chk.failed
        for (what, rank, k), names in chk.detail.items():
            if what == "gradient" and k == 0:
                assert set(names) <= shared, (rank, names)
        monkeypatch.undo()


@pytest.mark.parametrize("world", [2, 3])
def test_zero1_step_equals_the_replicated_step_bitwise(ops, world):
    from test_zero1_gpu import Loopback, _twin_from, assert_same_bits
    from oracle import dalle_sharing as OSH
    types = ("global", "mlp", "global", "mlp")
    cfg, params, tokens = _model(types, seed=11, TL=64, W=8)
    kw = dict(share_input_output_emb=True, shared_attn_ids=[0, 1], shared_ff_ids=[0], attention_types=list(types))
    params = {k: v.to(BF16).float() for k, v in OSH.share(params, cfg, True, [0, 1], [0]).items()}
    tok = tokens.to(I32).to(DEV)
    grp = Loopback(world)
    grp.engines = ranks = [_engine(cfg, zero=grp.member(r), **kw) for r in range(world)]
    twin = _engine(cfg, **kw)
    for e in [twin] + ranks:
        e.load_params(params)
    n = twin.n_params_padded
    P = twin.master[:n].clone()
    M, V = torch.zeros_like(P), torch.zeros_like(P)
    gn = torch.zeros(1, dtype=F32, device=DEV)
    for step in range(3):
        _twin_from(twin, P, ranks[0])
        g_ref = _step(twin, tok, 1e-2)
        for r, e in enumerate(ranks):
            assert_same_bits(_step(e, tok, 1e-2), g_ref, f"ZeRO-1 rank {r} step {step} gradients")
        for e in ranks:
            e.optimizer_step(1e-3, clip=1.0)
        gn.zero_()
        ops.sqnorm(g_ref[:n], gn)
        ops.adam_step(P, M, V, g_ref[:n], twin.shadow[:n], 1e-3, 0.9, 0.999, 1e-6, 0.0, gn, 1.0, 1.0, False, 0)
        for r, e in enumerate(ranks):
            lo, hi = e.shard
            assert_same_bits(e.master[:hi - lo], P[lo:hi], f"ZeRO-1 rank {r} step {step} fp32 slice")
            assert_same_bits(e.shadow[:n], twin.shadow[:n], f"ZeRO-1 rank {r} step {step} parameters")
    # the sharded initialisation equals the replicated one
    rep = _engine(cfg, **kw)
    rep.init_params(seed=3)
    for e in ranks:
        e.init_params(seed=3)
    got, want = ranks[0].export_params(), rep.export_params()
    assert set(got) == set(want) and "to_logits/linear_out/kernel" not in got
    for k in want:
        assert torch.equal(got[k], want[k].to(BF16).float()), k


# ------------------------------------------------------------------------------------------------ checkpoints
def test_checkpoint_round_trip_refusals_and_resume_through_the_model_fn(tmp_path):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import dalle_model_fn
    from test_layer_scale_gpu import _batch
    key = {"share_input_output_emb": True, "shared_attn_ids": [0], "shared_ff_ids": [0]}
    img, cap = _batch()
    plain = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path))
    sh = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **key))
    d, V = 256, sh.engine.V
    assert plain.engine.n_params() - sh.engine.n_params() == d * V + (12 * d * d + 6 * d)
    sh.train_op(img, cap)
    st = sh.state_fn()
    assert "to_logits/linear_out/kernel" not in st and "layer_1/attn/q" not in st and "layer_0/attn/q" in st
    assert tuple(st["embedding/wte"].shape) == (V, d)
    a = sh.train_op(img, cap).clone()
    resumed = dalle_model_fn(img, cap, "train", _tiny_params(tmp_path, **key))
    resumed.load_fn(st)
    assert torch.equal(a, resumed.train_op(img, cap))
    ex = sh.engine.export_params()
    e2 = sh.engine
    e2.load_params(ex)
    assert all(torch.equal(e2.export_params()[k], ex[k]) for k in ex)
    with pytest.raises(L.DB200Error, match="to_logits/linear_out/kernel: missing"):
        plain.engine.load_params(ex)
    pe = plain.engine.export_params()
    with pytest.raises(L.DB200Error, match="to_logits/linear_out/kernel: an output projection"):
        e2.load_params(pe)
    with pytest.raises(L.DB200Error, match="layer_1/attn/q: layer 1 uses the token mixer"):
        e2.load_params({k: v for k, v in pe.items() if k != "to_logits/linear_out/kernel"})
    with pytest.raises(L.DB200Error, match="layer_0/mlp/mlp_linear_2/bias: missing"):
        e2.load_params({k: v for k, v in ex.items() if k != "layer_0/mlp/mlp_linear_2/bias"})


# ------------------------------------------------------------------------------------------------ decoding
def test_decoding_follows_the_full_forward_and_the_prefill():
    from dalle_mtf_b200.sampling import DalleSampler
    from test_prefill_gpu import greedy_agrees_with_full_forward
    from oracle import dalle_sharing as OSH
    ts, W = 16, 8
    S = ts + W * W
    types = ("global", "axial_col", "global", "axial_col")
    for tie, attn, ff in ((True, None, None), (True, [0, 1], [0]), (False, [0, 1], [1, 0])):
        cfg, params, _ = _model(types, seed=6, TL=ts, W=W)
        g = torch.Generator().manual_seed(9)
        for k in params:
            if "wte" in k or "linear_out" in k or k.endswith("kernel"):
                params[k] = params[k] * 4
        eng = _engine(cfg, attention_types=list(types), share_input_output_emb=tie, shared_attn_ids=attn,
                      shared_ff_ids=ff)
        eng.load_params(OSH.share(params, cfg, tie, attn, ff))
        text = torch.randint(0, 299, (3, ts), generator=g).to(I32).to(DEV)
        smp = DalleSampler(eng)
        out, step_logits = smp.generate(text, 0.0, return_logits=True)
        assert torch.equal(smp.generate_graphed(text, temperature=0.0), out)
        greedy_agrees_with_full_forward(eng, out, ts)
        full = eng.logits(out)
        e = relfro(torch.stack(step_logits, 1), full[:, :S - 1])
        assert e < 2e-2, e
        for P in (ts, ts + W + 3, S - 1):
            kc = [torch.zeros_like(c) for c in smp.kc]
            vc = [torch.zeros_like(c) for c in smp.vc]
            logits = eng.prefill(out[:, :P].contiguous(), kc, vc).clone()
            ep = relfro(logits[:, :eng.V], step_logits[P - 1])
            print(f"[{TAG}] tie {tie} attn {attn} ff {ff}: decode vs full {e:.2e}, prefill P={P} vs decoding {ep:.2e}")
            assert ep < 2e-2, ep
        done = smp.complete(text, out[:, ts:ts + W + 3].contiguous() - eng.image_offset, temperature=0)
        greedy_agrees_with_full_forward(eng, done, ts + W + 3)
        torch.manual_seed(0)
        guided = smp.complete(text[:2], out[:2, ts:ts + W + 3].contiguous() - eng.image_offset, samples_per_prompt=2,
                              guidance_scale=3.0, top_k=16)
        assert guided.shape == (4, S)
        assert ((guided[:, ts:] >= eng.image_offset) & (guided[:, ts:] < eng.image_offset + 64)).all()
        assert torch.equal(smp.generate_graphed(text[:2], temperature=0.0, guidance_scale=2.0),
                           smp.generate(text[:2], 0.0, guidance_scale=2.0))
