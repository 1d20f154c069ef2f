"""CPU side of parameter sharing (share_input_output_emb, shared_attn_ids, shared_ff_ids): the keys at every place a
model is built, the cycling of the ids, the parameter layout (aliases at their owner's offset, each slot once in
`order`, data-parallel bucket spans that are disjoint and cover the buffer, the parameter count, weight decay), the
reference names and the checkpoint refusals, and the oracle (bit for bit the plain oracle with nothing shared, autograd
summing the uses, and mutants that change the result)."""
import math

import pytest
import torch

import generate_dalle as G
from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.dalle_engine import ATTN_MODULE, FF_MODULE, GMLP_MODULE, DalleEngine, layer_mlp, param_layout, \
    sharing_owners, validate_shared_ids
from dalle_mtf_b200.model_fns import dalle_model_fn, share_input_output_emb, shared_attn_ids, shared_ff_ids
from dalle_mtf_b200.models import DALLE
from oracle import dalle as O
from oracle import dalle_gmlp as OM
from oracle import dalle_layer_scale as OLS
from oracle import dalle_local as OL
from oracle import dalle_sharing as OSH
from test_gelu_cpu import _Built, _generate_config


# ------------------------------------------------------------------------------------------------ config values
def test_ids_are_cycled_to_the_depth():
    assert validate_shared_ids([0, 1], 6, "x") == [0, 1, 0, 1, 0, 1]
    assert validate_shared_ids((3,), 4, "x") == [3, 3, 3, 3]
    assert validate_shared_ids([0, 1, 2, 3, 4, 5, 6], 3, "x") == [0, 1, 2]
    assert validate_shared_ids(None, 3, "x") is None
    assert sharing_owners([0, 1], [5, 5, 7], 6) == ([0, 1, 0, 1, 0, 1], [0, 0, 2, 0, 0, 2])
    assert sharing_owners(None, None, 3) == ([0, 1, 2], [0, 1, 2])
    assert sharing_owners([2, 1, 2], None, 3) == ([0, 1, 0], [0, 1, 2])


BAD_IDS = [[], [True], [0, False], [-1], [0.0], [1.5], ["0"], "01", 0, {"a": 0}, [[0]], [None]]


@pytest.mark.parametrize("value", BAD_IDS, ids=[repr(v) for v in BAD_IDS])
@pytest.mark.parametrize("key", ["shared_attn_ids", "shared_ff_ids"])
def test_bad_ids_are_rejected_where_a_model_is_built(tmp_path, key, value):
    p = {key: value}
    reader = shared_attn_ids if key == "shared_attn_ids" else shared_ff_ids
    with pytest.raises(ValueError, match=key):
        reader(p)
    with pytest.raises(ValueError, match=key):        # before any GPU work
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match=key):
        DALLE(256, text_vocab_size=10, image_vocab_size=16, text_seq_len=4, image_seq_len=16, n_layers=1, n_heads=2,
              params=dict(p))
    with pytest.raises(ValueError, match=key):
        G.main(_generate_config(tmp_path, p))
    with pytest.raises(ValueError, match=key):
        DalleEngine(256, 2, 2, 10, 16, 4, 16, **{key: value})


@pytest.mark.parametrize("value", [1, 0, "true", [], [True]])
def test_share_input_output_emb_takes_a_bool_only(tmp_path, value):
    for ok, want in (({}, False), ({"share_input_output_emb": None}, False), ({"share_input_output_emb": False}, False),
                     ({"share_input_output_emb": True}, True)):
        assert share_input_output_emb(ok) is want
    p = {"share_input_output_emb": value}
    with pytest.raises(ValueError, match="share_input_output_emb"):
        share_input_output_emb(p)
    with pytest.raises(ValueError, match="share_input_output_emb"):
        dalle_model_fn(None, None, "train", dict(p))
    with pytest.raises(ValueError, match="share_input_output_emb"):
        G.main(_generate_config(tmp_path, p))
    with pytest.raises(ValueError, match="share_input_output_emb"):
        DalleEngine(256, 1, 2, 10, 16, 4, 16, share_input_output_emb=value)


def test_layers_sharing_an_attention_id_must_have_one_attention_type():
    with pytest.raises(ValueError, match="layers 0 and 2 share attention id 0"):
        DalleEngine(256, 3, 2, 10, 16, 4, 16, attention_types=["global", "axial_row", "mlp"], shared_attn_ids=[0, 1])
    with pytest.raises(ValueError, match="different attention types"):
        sharing_owners([0], None, 2, ["global", "local"])
    # the MLPs of layers of different types may be shared, and so may equal-type token mixers
    assert sharing_owners([0, 1, 2], [0], 3, ["global", "axial_row", "mlp"]) == ([0, 1, 2], [0, 0, 0])
    assert sharing_owners([0, 1, 2, 0, 1, 2], None, 6, ["axial_row", "axial_col", "mlp"] * 2)[0] == [0, 1, 2, 0, 1, 2]


@pytest.mark.parametrize("extra,want", [({}, (False, None, None)),
                                        ({"share_input_output_emb": True, "shared_attn_ids": [0, 1],
                                          "shared_ff_ids": [0]}, (True, [0, 1], [0]))])
def test_generate_cli_builds_the_engine_with_the_config_keys(tmp_path, monkeypatch, extra, want):
    """generate_dalle.py samples a checkpoint with the sharing it was trained with (device work stubbed)."""
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
    assert (seen["share_input_output_emb"], seen["shared_attn_ids"], seen["shared_ff_ids"]) == want


# ------------------------------------------------------------------------------------------------ layout
def _bare_engine(d, types, tied=False, attn_ids=None, ff_ids=None, sandwich=False, scale=None, tl=64, il=64):
    """A DalleEngine with only the fields the layout, the count, the names and the checkpoint checks read."""
    e = DalleEngine.__new__(DalleEngine)
    Lyr = len(types)
    e.d, e.L, e.text_seq_len, e.image_seq_len = d, Lyr, tl, il
    e.V, e.S = 300 + 64 + 1, tl + il
    e.row_col, e.grid_w, e.gated_mlp, e.sandwich_norm, e.layer_scale = False, None, False, sandwich, scale
    e.mlp = layer_mlp(types, Lyr, e.S, d)
    e.tied = tied
    e.attn_owner, e.ff_owner = sharing_owners(attn_ids, ff_ids, Lyr, types)
    e.layout = param_layout(d, Lyr, e.V, e.S, sandwich_norm=sandwich, mlp_layers=e.mlp if any(e.mlp) else None,
                            layer_scale=scale is not None, tied=tied, attn_owner=e.attn_owner, ff_owner=e.ff_owner)
    return e


CASES = {
    "tied": dict(types=["global"] * 3, tied=True),
    "attn_0": dict(types=["global"] * 3, attn_ids=[0]),
    "ff_01": dict(types=["global"] * 4, ff_ids=[0, 1]),
    "both_sandwich_scale": dict(types=["global"] * 4, tied=True, attn_ids=[0, 1], ff_ids=[0], sandwich=True,
                                scale=0.1),
    "mixed_gmlp": dict(types=["axial_row", "axial_col", "mlp"] * 2, attn_ids=[0, 1, 2], ff_ids=[7]),
    "mixed_ff_only": dict(types=["axial_row", "axial_col", "mlp"] * 2, ff_ids=[0, 1]),
}


def _numel(shape):
    return math.prod(shape)


@pytest.mark.parametrize("case", list(CASES))
def test_layout_aliases_buckets_and_count(case):
    c = CASES[case]
    e = _bare_engine(256, **c)
    plain = _bare_engine(256, c["types"], sandwich=c.get("sandwich", False), scale=c.get("scale"))
    lay = e.layout
    # every alias points at its owner's entry, and only non-owners have aliases
    for name, owner in lay.aliases.items():
        assert lay.entries[name] == lay.entries[owner] and name not in lay.order and owner in lay.order
        i, k = int(name.split(".")[0][1:]), name.split(".")[1]
        own = e.ff_owner[i] if k in FF_MODULE else e.attn_owner[i]
        assert own < i and owner == f"l{own}.{k}"
    want_aliases = {f"l{i}.{k}" for i in range(e.L) for k in FF_MODULE if e.ff_owner[i] != i} | \
        {f"l{i}.{k}" for i in range(e.L) for k in (GMLP_MODULE if e.mlp[i] else ATTN_MODULE) if e.attn_owner[i] != i}
    assert set(lay.aliases) == want_aliases
    # order holds each slot once: offsets strictly increase, each entry ends where the next begins
    offs = [lay.entries[n][0] for n in lay.order]
    assert offs == sorted(set(offs)) and offs[0] == 0
    assert all(lay.span(a, a)[1] == lay.entries[b][0] for a, b in zip(lay.order, lay.order[1:]))
    assert lay.span(lay.order[-1], lay.order[-1])[1] == lay.size
    # the engine's data-parallel buckets: embeddings, each layer's own entries, the head; disjoint and covering
    buckets = [lay.span("wte", "wpe")] + [lay.span(f"l{i}.ln1_g", e.layer_last(i)) for i in range(e.L)] + \
        [lay.span("lnf_g", "bout")]
    assert buckets[0][0] == 0 and buckets[-1][1] == lay.size
    assert all(a[1] == b[0] for a, b in zip(buckets, buckets[1:]))
    for i in range(e.L):   # a bucket holds exactly the entries layer i owns, and every alias is in its owner's
        s, t = buckets[1 + i]
        inside = [n for n in lay.order if s <= lay.entries[n][0] < t]
        assert inside == [n for n in lay.order if n.startswith(f"l{i}.")]
    # tied: wte has Vpad rows and there is no wout
    assert lay.entries["wte"][1] == ((e.V + 63) // 64 * 64 if c.get("tied") else e.V, 256)
    assert ("wout" in lay.entries) == (not c.get("tied"))
    # the count: each parameter once (a tied wte's V rows, no pad), what the unshared model has minus the aliases
    counted = sum(_numel(lay.entries[n][1]) for n in lay.order if n not in ("wte", "wout", "bout")) + \
        e.V * 256 + (0 if c.get("tied") else e.V * 256) + e.V
    assert e.n_params() == counted
    assert plain.n_params() - e.n_params() == sum(_numel(lay.entries[n][1]) for n in lay.aliases) + \
        (e.V * 256 if c.get("tied") else 0)
    # weight decay iterates `order`: the shared slots once, and the decayed total shrinks by exactly the aliases
    decayed = lambda eng: sum(t - s for s, t, dec in eng._decay_segments() if dec)   # noqa: E731
    shared = sum(lay.span(n, n)[1] - lay.span(n, n)[0] for n in lay.aliases
                 if n.split(".")[1] in ("wqkv", "wo", "w1", "w2", "gm_win", "sgu_w", "gm_wout"))
    assert decayed(plain) - decayed(e) == shared + (e.V * 256 if c.get("tied") else 0)   # tied: wout's d x V


def test_the_savings_stated_in_the_docs():
    """The README's counts: dalle_example (d 512, L 6, V 50 771) has 71.6 M parameters, the output projection holds
    26.0 M of them and one attention + MLP module for all layers saves 15.7 M more; at the dalle_coco width (d 1024,
    L 12, 1 280 positions) 52.0 M of 256.5 M, and 138.5 M."""
    def count(d, Lyr, **kw):
        e = _bare_engine(d, ["global"] * Lyr, tl=256, il=1024, **kw)
        e.V = 50258 + 512 + 1
        e.layout = param_layout(d, Lyr, e.V, e.S, tied=kw.get("tied", False), attn_owner=e.attn_owner,
                                ff_owner=e.ff_owner)
        return e.n_params()
    for d, Lyr, total, out, modules in ((512, 6, 71.6, 26.0, 15.7), (1024, 12, 256.5, 52.0, 138.5)):
        base = count(d, Lyr)
        assert base - count(d, Lyr, tied=True) == d * 50771
        assert base - count(d, Lyr, attn_ids=[0], ff_ids=[0]) == (Lyr - 1) * (12 * d * d + 6 * d)
        assert [round(x / 1e6, 1) for x in (base, d * 50771, (Lyr - 1) * (12 * d * d + 6 * d))] == \
            [total, out, modules]


# ------------------------------------------------------------------------------------------------ names
def _cfg(types, d=64):
    return OL.LocalConfig(d, len(types), 2, 50, 16, 8, 16, attention_types=tuple(types))


def _full_names(e):
    """Every reference name of the unshared twin of a bare engine, in the engine's export order."""
    twin = _bare_engine(e.d, [("mlp" if m else "global") for m in e.mlp], sandwich=e.sandwich_norm,
                        scale=e.layer_scale, tl=e.text_seq_len, il=e.image_seq_len)
    out = ["embedding/wte", "positional_embedding/wpe"]
    for i in range(e.L):
        out += list(twin._layer_ref_names(i).values())
        if not twin._is_mlp(i):
            out += [f"layer_{i}/attn/{x}" for x in "qkv"]
    return out + ["to_logits/layer_norm/g", "to_logits/layer_norm/b", OSH.OUT_KERNEL, "to_logits/linear_out/bias"]


def _engine_names(e):
    out = ["embedding/wte", "positional_embedding/wpe"]
    for i in range(e.L):
        out += list(e._layer_ref_names(i).values())
        if not e._is_mlp(i) and e._owns_mixer(i):
            out += [f"layer_{i}/attn/{x}" for x in "qkv"]
    out += ["to_logits/layer_norm/g", "to_logits/layer_norm/b", "to_logits/linear_out/bias"]
    return out + ([] if e.tied else [OSH.OUT_KERNEL])


@pytest.mark.parametrize("case", list(CASES))
def test_reference_names_are_the_owners_and_match_the_oracle(case):
    c = CASES[case]
    e = _bare_engine(256, **c)
    cfg = _cfg(["mlp" if m else "global" for m in e.mlp])
    kw = dict(tie=c.get("tied", False), attn_ids=c.get("attn_ids"), ff_ids=c.get("ff_ids"))
    want = OSH.names(_full_names(e), cfg, **kw)
    assert sorted(_engine_names(e)) == sorted(want)
    for m in ("last_owner", "no_cycle"):   # naming mutants: different variables whenever something is shared
        if m == "no_cycle" and all(len(v or [0] * e.L) >= e.L for v in (c.get("attn_ids"), c.get("ff_ids"))):
            continue
        if c.get("attn_ids") is None and c.get("ff_ids") is None:
            continue
        assert sorted(OSH.names(_full_names(e), cfg, **kw, mutate=m)) != sorted(want), m


def _named(e):
    return {n: torch.zeros(1) for n in _engine_names(e)}


def test_checkpoint_refusals_name_the_first_mismatched_variable():
    types = ["global", "mlp", "global", "mlp"]
    e = _bare_engine(256, types, tied=True, attn_ids=[0, 1], ff_ids=[0])
    good = _named(e)
    e._check_sharing_names(good)
    e._check_layer_kinds({k: v for k, v in good.items()
                          if not k.endswith("gmlp/sgu/weight")} | {"layer_1/gmlp/sgu/weight": torch.zeros(128, 128)})
    with pytest.raises(L.DB200Error, match="to_logits/linear_out/kernel: an output projection"):
        e._check_sharing_names({**good, OSH.OUT_KERNEL: torch.zeros(1)})
    untied = _bare_engine(256, types, attn_ids=[0, 1], ff_ids=[0])
    with pytest.raises(L.DB200Error, match="to_logits/linear_out/kernel: missing"):
        untied._check_sharing_names(good)
    with pytest.raises(L.DB200Error, match="layer_2/attn/q: layer 2 uses the token mixer .* of layer 0"):
        e._check_sharing_names({**good, "layer_2/attn/q": torch.zeros(1), "layer_3/gmlp/proj_in/kernel": 0})
    with pytest.raises(L.DB200Error, match="layer_1/mlp/mlp_linear_1/kernel: layer 1 uses the MLP .* of layer 0"):
        e._check_sharing_names({**good, "layer_1/mlp/mlp_linear_1/kernel": torch.zeros(1)})
    with pytest.raises(L.DB200Error, match="layer_1/gmlp/sgu/bias: missing from the checkpoint, and layer 1 owns"):
        e._check_sharing_names({k: v for k, v in good.items() if k != "layer_1/gmlp/sgu/bias"})
    with pytest.raises(L.DB200Error, match="layer_0/mlp/mlp_linear_2/bias: missing"):
        e._check_sharing_names({k: v for k, v in good.items() if k != "layer_0/mlp/mlp_linear_2/bias"})
    # an unshared model given the shared checkpoint: the first variable it owns and misses
    plain = _bare_engine(256, types, tied=True)
    with pytest.raises(L.DB200Error, match="layer_1/mlp/mlp_linear_1/kernel: missing"):
        plain._check_sharing_names(good)


# ------------------------------------------------------------------------------------------------ oracle
def _model(seed, types=("global", "global", "global"), d=64, H=2, TL=8, W=4):
    cfg = OL.LocalConfig(d, len(types), H, 50, 16, TL, W * W, attention_types=tuple(types))
    params = OM.init_params(O.init_params(cfg, seed), cfg, seed + 1)
    g = torch.Generator().manual_seed(seed + 3)
    for k in params:   # every bias, norm and the gMLP's mixing weight non-trivial
        if k.endswith("/b") or k.endswith("bias") or k.endswith("o_b"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.05
        if k.endswith("/g"):
            params[k] = 1 + torch.randn(params[k].shape, generator=g) * 0.2
    tokens = O.assemble_tokens(torch.randint(0, 49, (2, TL), generator=g),
                               torch.randint(0, 16, (2, W * W), generator=g), 50)
    return cfg, params, tokens


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("types", [("global", "global", "global"), ("global", "mlp", "local")],
                         ids=["global", "mixed"])
def test_oracle_with_nothing_shared_is_the_plain_oracle_bit_for_bit(types, bf16):
    cfg, params, tokens = _model(3, types)
    a = OSH.loss_and_grads(params, tokens, cfg, attn_ids=list(range(len(types))), ff_ids=[5, 6, 7], bf16=bf16)
    b = OLS.loss_and_grads(params, tokens, cfg, bf16=bf16)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert set(a[3]) == set(b[3]) and all(torch.equal(a[3][k], b[3][k]) for k in b[3])


def test_shared_gradients_are_the_sums_of_the_twins_per_layer_gradients():
    """float64: with the twin's per-layer copies equal to the owner's, the shared model's loss is the twin's and each
    shared gradient the sum of the twin's per-layer ones; a tied wte's gradient is the twin's wte gradient plus its
    output projection's (transposed)."""
    cfg, params, tokens = _model(5, ("global", "mlp", "global", "mlp"))
    params = {k: v.double() for k, v in params.items()}
    tie, attn, ff = True, [0, 1], [0]
    twin = dict(OSH.expand(OSH.share(params, cfg, tie, attn, ff), cfg, tie, attn, ff))
    twin = {k: v.detach().clone() for k, v in twin.items()}
    ls, _, logits_s, gs = OSH.loss_and_grads(params, tokens, cfg, tie, attn, ff)
    lt, _, logits_t, gt = OLS.loss_and_grads(twin, tokens, cfg)
    assert torch.allclose(ls, lt, rtol=1e-12) and torch.allclose(logits_s, logits_t, rtol=1e-12, atol=1e-12)
    ao, fo = OSH.owners(attn, 4), OSH.owners(ff, 4)
    for k in gs:
        if k == "embedding/wte":
            want = gt[k] + gt[OSH.OUT_KERNEL].t()
        elif k.startswith("layer_"):
            l, v = int(k.split("/")[0][6:]), k.split("/", 1)[1]
            owner = fo if v in OSH.FF_VARS else ao if v in OSH.mixer_vars(cfg, l) else None
            users = [j for j in range(4) if owner is not None and owner[j] == l] or [l]
            want = sum(gt[f"layer_{j}/{v}"] for j in users)
        else:
            want = gt[k]
        assert torch.allclose(gs[k], want, rtol=1e-10, atol=1e-14), k


@pytest.mark.parametrize("mutate", OSH.MUTATIONS)
def test_each_mutant_changes_the_loss_or_a_gradient(mutate):
    cfg, params, tokens = _model(7, ("global", "mlp", "global", "mlp"))
    kw = dict(tie=True, attn_ids=[0, 1], ff_ids=[0, 1, 1], stable=True)
    ref = OSH.loss_and_grads(params, tokens, cfg, **kw)
    mut = OSH.loss_and_grads(params, tokens, cfg, **kw, mutate=mutate)
    differs = not torch.equal(ref[0], mut[0]) or set(ref[3]) != set(mut[3]) or \
        any(not torch.equal(ref[3][k], mut[3][k]) for k in ref[3])
    assert differs, mutate
    with pytest.raises(ValueError, match="mutation"):
        OSH.expand(params, cfg, mutate="nope")
