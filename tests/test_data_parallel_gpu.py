"""Data-parallel training on one GPU: W in-process ranks (tests/rank_group.py) through dalle_model_fn and vae_model_fn.

Each rank gets its own params dict with `_dp` = a RankGroup member, so the model functions run their own sharding,
bucket hooks, overlap calls and eval reductions; the group checks at every rendezvous that all ranks launched the
same ranges and that no range changed after its launch, and sums each range in fp32 in rank order.

DALL-E, bit for bit.  W ranks with one micro-batch of B/W rows each equal one rank with W micro-batches of B/W rows
(tokens_per_mb_per_replica = (B/W) S): the same rows in the same groups, in rank order.  Every gradient-accumulating
kernel adds one fully formed contribution per element and call (split-K partials and row / column sums are formed
first, then D += s; the embedding gradient is converted from its fixed-point accumulator once per call), so the one-rank
buffer after micro-batch i is fl(... fl(s0 + s1) ... + si), which is the rank-order sum; the dropout masks and caption
drops are indexed by the global row; and the split-K, LayerNorm and column-sum grids depend only on the per-call row
count, which is the same in both runs.  So the assembled tokens, every rank's loss_rows, the reduced gradient buffer
(aux slots included), master / Adam slots / bf16 copy after each step and the reported loss are compared bitwise.
Steps 0, 1, 2 run with clip-by-global-norm active, inactive and off (the clip value is set per step by wrapping
DalleEngine.optimizer_step in the test).

The eval reduction sums per-row losses through ce_finish(_weighted)'s partial-sum chain (a 5-level warp tree, the
per-block partials in block order onto the accumulator) and then W rank additions: its sums are bounded per slot by
gamma_k sum |v| against the float64 sum of the one-rank per-row values, k = (roundings of a row's value) + 5 +
blocks + 1 + W.

VAE, against the oracle of the global batch.  Its convolution wgrads use float atomics, so a one-rank run is not
bitwise comparable; each step the objective, loss_parts and the reduced gradient / W are compared with the oracle at
the engine's current parameters, with the tolerances of the one-rank engine tests (fp32: test_engine_gpu.py's
test_vae_engine_fp32_matches_oracle_exactly_enough and test_vae_logit_laplace_gpu.py's model_fn test; bf16: the bf16
policy of those modules).  The gradient Adam consumed, recovered from adam_m, must be the reduced gradient / W.
codebook_usage() must agree on every rank and equal the usage of the first-maximum codes of the global batch (the
oracle's fp32 logits; with bf16 activations the engines' own logits, which the bf16 encoder rounds differently near
ties).

Mutation tests apply a fault with monkeypatch and assert that the named check catches it.
"""
import gc
import time
from collections import defaultdict

import pytest
import torch

import float64_bounds as FB
from rank_group import RankGroup, RankGroupError, RankMember
from test_loss_weights_gpu import _tiny_params
from test_vae_logit_laplace_gpu import _vae_params, near, relfro
from test_zero1_gpu import CLIPS

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAG = "dp"
F32, F64, BF16, I16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int16, torch.int32
STEPS = len(CLIPS)
_PEAK = [0]


@pytest.fixture(scope="module", autouse=True)
def _module_cost():
    from dalle_mtf_b200 import lib as L
    L.require_device()
    t0 = time.time()
    yield
    print(f"[{TAG}] module: {time.time() - t0:.1f} s, peak device memory {_PEAK[0] / 2 ** 30:.2f} GiB")


@pytest.fixture(autouse=True)
def _cost(request):
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    gc.collect()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: {time.time() - t0:.1f} s, peak device memory {peak / 2 ** 30:.2f} GiB")


def _bits(t):
    return t.view({F32: I32, BF16: I16}.get(t.dtype, t.dtype))


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and bool(torch.equal(_bits(a), _bits(b)))


class _Checks:
    """Named checks; a failure is recorded (name -> {(rank, step)}) rather than raised, so one run reports every check
    and a mutation test can assert which one caught its fault."""

    def __init__(self):
        self.failed = defaultdict(set)
        self.detail = {}
        self.bitwise = 0

    def same(self, name, rank, step, got, ref):
        self.bitwise += 1
        if not _same(got, ref):
            self.failed[name].add((rank, step))

    def ok(self, name, rank, step, cond):
        if not cond:
            self.failed[name].add((rank, step))

    def assert_clean(self):
        assert not self.failed, ({k: sorted(v) for k, v in self.failed.items()}, self.detail)


class _Rec:
    """Test-side wrappers of DalleEngine.forward / optimizer_step: per engine, (tokens, loss_rows) of every forward and
    the gradient buffer every optimizer_step consumes; clip[engine] replaces the clip value of that engine's steps (per
    engine: a rank's optimizer_step runs after the next rank has started its step)."""

    def __init__(self, monkeypatch):
        from dalle_mtf_b200.dalle_engine import DalleEngine
        self.fwd, self.grads, self.clip = defaultdict(list), defaultdict(list), {}
        fwd0, step0 = DalleEngine.forward, DalleEngine.optimizer_step
        rec = self

        def forward(eng, tokens, *a, **k):
            out = fwd0(eng, tokens, *a, **k)
            rec.fwd[eng].append((tokens.clone(), eng._bufs["loss_rows"][:tokens.numel()].clone()))
            return out

        def optimizer_step(eng, lr, **k):
            rec.grads[eng].append(eng.grads.clone())
            if eng in rec.clip:
                k["clip"] = rec.clip[eng]
            return step0(eng, lr, **k)

        monkeypatch.setattr(DalleEngine, "forward", forward)
        monkeypatch.setattr(DalleEngine, "optimizer_step", optimizer_step)


@pytest.fixture
def rec(monkeypatch):
    r = _Rec(monkeypatch)
    yield r
    r.fwd.clear()
    r.grads.clear()


def _state(eng):
    return [t.clone() for t in (eng.master, eng.adam_m, eng.adam_v, eng.shadow) if t is not None]


def _check_coverage(trace, n, aux_off, steps):
    """(A) the hook ranges of every training step (the waits of `trace` with more than one range): pairwise disjoint,
    launched in descending start order, union [0, n) + [aux_off, aux_off + 64), the range at 0 launched last and the
    only exposed one.  Returns the number of ranges per step."""
    waits = [e["ranges"] for e in trace if e["kind"] == "wait" and len(e["ranges"]) > 1]
    assert len(waits) == steps, [(e["kind"], len(e["ranges"])) for e in trace]
    for ranges in waits:
        spans = [(off, off + numel) for off, numel, dtype, _ in ranges]
        assert all(dtype == F32 for _, _, dtype, _ in ranges)
        assert [s for s, _ in spans] == sorted((s for s, _ in spans), reverse=True), spans
        assert ranges[-1][0] == 0 and ranges[-1][3] and not any(x[3] for x in ranges[:-1]), ranges
        cover = sorted(spans)
        assert all(a[1] <= b[0] for a, b in zip(cover, cover[1:])), cover
        merged = []
        for s, e in cover:
            if merged and merged[-1][1] == s:
                merged[-1][1] = e
            else:
                merged.append([s, e])
        expect = [[0, n], [aux_off, aux_off + 64]] if aux_off > n else [[0, aux_off + 64]]
        assert merged == expect, (merged, expect)
    return len(waits[0])


# ====================================================================================================== DALL-E
FEATURES = dict(embed_dropout=0.1, attention_dropout=0.1, residual_dropout=0.1, caption_dropout=0.5, padding_id=299,
                text_loss_weight=1, image_loss_weight=7, z_loss=1e-3, recompute_grad=True, n_layers=4,
                attention_types=[[["global", "local", "axial_row", "conv"], 1]], local_attention_radius=8,
                conv_attention_kernel=3)
EXAMPLE = dict(n_embd=512, n_layers=2, n_heads=4, text_vocab_size=50258, image_vocab_size=512, text_seq_len=256,
               dataset={"image_size": 64},
               vae_params={"model_type": "vae", "num_tokens": 512, "convblocks": [[1, 32]],
                           "dataset": {"image_size": 64}})
DALLE_CASES = [("tiny", W, 12, {}) for W in (2, 3, 4)] + [("tiny-features", W, 12, FEATURES) for W in (2, 3)] + \
              [("dalle_example-width", W, 8, EXAMPLE) for W in (2, 4)]


def _dalle_params(tmp_path, extra, **kw):
    from collections import defaultdict as dd
    extra = dict(extra)
    if "vae_params" in extra:
        extra["vae_params"] = dd(lambda: None, extra["vae_params"])
    return _tiny_params(tmp_path, model_path=None, **extra, **kw)


def _seq_len(p):
    vp = p["vae_params"]
    return p["text_seq_len"] + (p["dataset"]["image_size"] // 2 ** len(vp["convblocks"])) ** 2


def _dalle_data(p, B, seed):
    g = torch.Generator().manual_seed(seed)
    size = p["dataset"]["image_size"]
    return (torch.rand(B, size, size, 3, generator=g) * 2 - 1,
            torch.randint(0, p["text_vocab_size"] - 1, (B, p["text_seq_len"]), generator=g))


def _dalle_reference(rec, params, feats, caps, W, steps=STEPS):
    """One rank, W micro-batches of B/W rows: per step the micro-batches' tokens and loss_rows, the gradient buffer
    its optimizer_step consumes, the state after the step and the reported loss."""
    from dalle_mtf_b200.model_fns import dalle_model_fn
    spec = dalle_model_fn(feats, caps, "train", params)
    assert params["num_microbatches"] == W
    eng = spec.engine
    n = eng.n_params_padded
    ref = []
    for k in range(steps):
        rec.clip[eng] = CLIPS[k]
        spec.train_op(feats, caps)
        fw = rec.fwd.pop(eng)
        assert len(fw) == W
        g = rec.grads.pop(eng)[-1]
        ref.append(dict(tokens=[t for t, _ in fw], loss_rows=[r for _, r in fw], grads=g, state=_state(eng),
                        loss=(spec.loss_sum * spec.loss_scale).clone(),
                        parts=None if spec.loss_parts is None else spec.loss_parts.clone()))
    gn = [ref[k]["grads"][:n].double().norm().item() for k in range(steps)]
    assert gn[0] > CLIPS[0] and gn[1] < CLIPS[1], gn            # clip active, then inactive
    return ref, n, eng.aux_off


def _dalle_ranks(rec, make, feats, caps, W, ref, steps=STEPS, group=None):
    """W ranks, one micro-batch each, checked against `ref` after every step (_Checks names: tokens, loss_rows,
    gradient, aux, state, loss)."""
    from dalle_mtf_b200.model_fns import dalle_model_fn
    group = group or RankGroup(W, keep_inputs=False)
    chk = _Checks()
    b = feats.shape[0] // W

    def fn(rank, dp):
        p = make()
        p["_dp"] = dp
        f, c = feats[rank * b:(rank + 1) * b], caps[rank * b:(rank + 1) * b]
        spec = dalle_model_fn(f, c, "train", p)
        eng = spec.engine
        n = eng.n_params_padded
        for k in range(steps):
            rec.clip[eng] = CLIPS[k]
            spec.train_op(f, c)
            r = ref[k]
            (tok, rows), = rec.fwd.pop(eng)
            chk.same("tokens", rank, k, tok, r["tokens"][rank])
            chk.same("loss_rows", rank, k, rows, r["loss_rows"][rank])
            g = rec.grads.pop(eng)[-1]
            chk.same("gradient", rank, k, g[:n], r["grads"][:n])
            if not _same(g[:n], r["grads"][:n]):
                chk.detail[("gradient", rank, k)] = [
                    nm for nm in eng.layout.order
                    if not _same(eng.layout.view(g, nm), eng.layout.view(r["grads"], nm))]
            chk.same("aux", rank, k, g[n:], r["grads"][n:])
            for got, exp in zip(_state(eng), r["state"]):
                chk.same("state", rank, k, got, exp)
            chk.same("loss", rank, k, spec.loss_sum * spec.loss_scale, r["loss"])
            if r["parts"] is not None:
                chk.same("loss", rank, k, spec.loss_parts, r["parts"])
        return n, eng.aux_off

    res = group.run(fn)
    return group, chk, res[0]


@pytest.mark.parametrize("name,W,B,extra", DALLE_CASES, ids=[f"{c[0]}-W{c[1]}" for c in DALLE_CASES])
def test_dalle_ranks_equal_one_rank_with_micro_batches_bitwise(rec, tmp_path, name, W, B, extra):
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, n, aux_off = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W)
    group, chk, (n_r, aux_r) = _dalle_ranks(rec, make, feats, caps, W, ref)
    assert (n_r, aux_r) == (n, aux_off)
    buckets = _check_coverage(group.trace, n, aux_off, STEPS)
    chk.assert_clean()
    print(f"[{TAG}] dalle {name} W={W} B={B}: {STEPS} steps (clip {CLIPS}), {chk.bitwise} tensors bitwise "
          f"(tokens, loss_rows, gradient + aux, master / adam_m / adam_v / shadow, loss), {buckets} buckets per step "
          f"cover the buffer, none written after launch")


class _ShardOnly(RankMember):
    """Rank r of W that reduces nothing: its shard's gradient, as the rank computes it before the all-reduce."""

    def make_bucket_hook(self, flat):
        return None

    def wait(self):
        pass


def test_dalle_micro_batches_inside_ranks_reduce_once(rec, tmp_path):
    """(C) W = 2, two micro-batches per rank: the reduced gradient is the rank-order fp32 sum of each rank's shard
    gradient computed with the same micro-batching and no reduction; a hook on a non-last micro-batch would reduce a
    partial gradient and show here (and in the group's snapshot check)."""
    from dalle_mtf_b200.model_fns import dalle_model_fn
    W, B = 2, 8
    p = _dalle_params(tmp_path, FEATURES)
    make = lambda **kw: _dalle_params(tmp_path, FEATURES, train_batch_size=B,                  # noqa: E731
                                      tokens_per_mb_per_replica=(B // W // 2) * _seq_len(p), **kw)
    feats, caps = _dalle_data(p, B, seed=11)
    b = B // W
    shard_grads = []
    for r in range(W):
        pr = make()
        pr["_dp"] = _ShardOnly(RankGroup(W), r)
        spec = dalle_model_fn(feats[r * b:(r + 1) * b], caps[r * b:(r + 1) * b], "train", pr)
        assert pr["num_microbatches"] == 2
        rec.clip[spec.engine] = CLIPS[0]
        spec.train_op(feats[r * b:(r + 1) * b], caps[r * b:(r + 1) * b])
        shard_grads.append(rec.grads.pop(spec.engine)[-1])
        del spec
    expect = shard_grads[0].clone()
    expect += shard_grads[1]
    group = RankGroup(W, keep_inputs=True)
    chk = _Checks()

    def fn(rank, dp):
        pr = make()
        pr["_dp"] = dp
        f, c = feats[rank * b:(rank + 1) * b], caps[rank * b:(rank + 1) * b]
        spec = dalle_model_fn(f, c, "train", pr)
        assert pr["num_microbatches"] == 2
        spec.train_op(f, c)
        chk.same("gradient", rank, 0, rec.grads.pop(spec.engine)[-1], expect)
        return spec.engine.n_params_padded, spec.engine.aux_off

    (n, aux_off), _ = group.run(fn)
    _check_coverage(group.trace, n, aux_off, 1)
    for j, red in enumerate(group.last_reduce):       # what each rank launched is its own shard gradient
        off, numel, _, _ = red["sig"]
        for r in range(W):
            chk.same("launched", r, 0, red["inputs"][r], shard_grads[r][off:off + numel])
    chk.assert_clean()
    print(f"[{TAG}] dalle micro-batches in ranks W={W} B={B} (2 per rank): {chk.bitwise} tensors bitwise")


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("weighted", [False, True], ids=["plain", "weighted"])
def test_dalle_eval_op_reduces_the_global_sums(rec, tmp_path, W, weighted):
    """(C) eval_op at W ranks: per-row losses bitwise equal to the one-rank eval; the reduced sums (1 or 4 slots)
    within gamma_k sum |v| of the float64 sums of the one-rank per-row values."""
    from dalle_mtf_b200.model_fns import dalle_model_fn
    B = 12
    extra = {"text_loss_weight": 1, "image_loss_weight": 7, "z_loss": 1e-3} if weighted else {}
    make = lambda: _dalle_params(tmp_path, extra, eval_batch_size=B)                          # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=20 + W)
    one = dalle_model_fn(feats, caps, "eval", p)
    one.eval_op(feats, caps)
    eng = one.engine
    (_, rows_ref), = rec.fwd.pop(eng)
    T = rows_ref.numel()
    lse = eng._bufs["lse_v"][:T].double().cpu()
    lab = eng._bufs["label_logit"][:T].double().cpu()
    rows64 = rows_ref.double().cpu()
    S = eng.S
    b = B // W
    nb = -(-(b * S) // 32)          # ce_finish blocks of one rank's forward
    if weighted:
        w = eng._cew
        text = (torch.arange(T) % w.period) < w.text_rows
        a = torch.where(text, torch.tensor(w.a_text, dtype=F64), torch.tensor(w.a_image, dtype=F64))
        ce = lse - lab
        values = [(a * rows64, 1), (torch.where(text, ce, 0.0), 1), (torch.where(text, 0.0, ce), 1),
                  (float(w.z_loss) * lse * lse, 2)]
    else:
        values = [(rows64, 0)]
    del one, eng
    group = RankGroup(W)
    chk = _Checks()
    sums = {}

    def fn(rank, dp):
        pr = make()
        pr["_dp"] = dp
        f, c = feats[rank * b:(rank + 1) * b], caps[rank * b:(rank + 1) * b]
        spec = dalle_model_fn(f, c, "eval", pr)
        spec.eval_op(f, c)
        (_, rows), = rec.fwd.pop(spec.engine)
        chk.same("loss_rows", rank, 0, rows, rows_ref[rank * b * S:(rank + 1) * b * S])
        red, = group.last_reduce
        chk.same("loss", rank, 0, spec.loss_sum, red["result"][:1])
        sums[rank] = red["result"].double().cpu()

    group.run(fn)
    chk.assert_clean()
    assert group.trace[-1]["ranges"] == [(0, 4 if weighted else 1, F32, True)]
    worst = 0.0
    for slot, (v, k_row) in enumerate(values):
        k = k_row + 5 + nb + 1 + W
        gamma = k * FB.U / (1 - k * FB.U)
        worst = max(worst, FB.check(f"dalle eval W={W} {'weighted' if weighted else 'plain'} slot {slot}",
                                    sums[0][slot:slot + 1], v.sum().reshape(1), v.abs().sum().reshape(1),
                                    a=0.0, b=gamma, tag=TAG))
    print(f"[{TAG}] dalle eval W={W} {'weighted' if weighted else 'plain'}: {chk.bitwise} tensors bitwise, "
          f"{len(values)} reduced sums, worst err/bound {worst:.3f}")


# ====================================================================================================== VAE
VAE_CASES = {
    "fp32-mse": dict(reconstruction_loss=None),
    "logit-laplace-kl": dict(kl_loss_weight=0.8, kl_anneal_steps=2),
    "bf16-s2-kl": dict(reconstruction_loss=None, use_bf16=True, stack_factor=2, kl_loss_weight=0.8,
                       dataset={"image_size": 32}),
}
VAE_B = 4
ADAM_B1 = 0.9


def _vae_oracle(case, p, named, img, uv, step, hard=True):
    """dict(objective, parts [in loss_parts order] , grads, logits, bf16 refs when the case runs bf16)."""
    from oracle import vae as OV
    from oracle import vae_kl as OK
    from oracle import vae_logit_laplace as OL
    cb = p["convblocks"]
    beta = OK.kl_weight(step, p)
    if p["reconstruction_loss"] == "logit_laplace":
        loss, rec_, mse, kl, _, logits, grads = OL.loss_and_grads(named, img, uv, cb, 1.0, hard, kl_weight=beta)
        return dict(objective=loss, parts=[rec_, mse] + ([kl] if beta is not None else []), grads=grads,
                    logits=logits)
    if not p["use_bf16"]:
        loss, _, logits, grads = OV.loss_and_grads(named, img, uv, cb, 1.0, hard)
        return dict(objective=loss, parts=None, grads=grads, logits=logits)
    out = {}
    for bf16 in (False, True):      # oracle.vae_kl.forward with the stack factor, fp32 and the bf16 policy
        leaves = {k: v.clone().requires_grad_(True) for k, v in named.items()}
        loss, mse, kl, _, logits = OK.forward(leaves, img, uv, cb, 1.0, hard, bf16, p["stack_factor"], kl_weight=beta)
        loss.backward()
        out[bf16] = dict(objective=loss.detach(), parts=[mse.detach(), kl.detach()],
                         grads={k: v.grad for k, v in leaves.items()}, logits=logits.detach())
    out[False]["bf16"] = out[True]
    return out[False]


def _vae_check_step(chk, case, p, orc, k, obj, parts, eg=None):
    """Objective, loss_parts and per-tensor gradients (eg; None: eval, no gradients) against the oracle at the
    tolerances of the one-rank tests."""
    grads = orc["grads"] if eg is not None else {}
    if p["use_bf16"]:
        ref16 = orc["bf16"]
        lo, l16 = orc["objective"].item(), ref16["objective"].item()
        chk.ok("objective", 0, k, abs(obj - lo) <= 1.5 * abs(l16 - lo) + 2e-2 * max(abs(lo), 1.0))
        for i, (got, r, r16) in enumerate(zip(parts, orc["parts"], ref16["parts"])):
            chk.ok("loss_parts", 0, k, abs(got - r.item()) <= 1.5 * abs(r16.item() - r.item()) + 2e-2 * max(abs(r.item()), 1.0))
        for name, g in grads.items():
            chk.ok("gradient", 0, k, relfro(eg[name], g) <= 1.5 * relfro(ref16["grads"][name], g) + 2e-2)
        return
    if p["reconstruction_loss"] == "logit_laplace":
        chk.ok("objective", 0, k, near(torch.tensor(obj), orc["objective"]))
        chk.ok("loss_parts", 0, k, near(torch.tensor(parts[0]), orc["parts"][0]))
        for got, r in zip(parts[1:], orc["parts"][1:]):
            chk.ok("loss_parts", 0, k, relfro(torch.tensor([got]), r.reshape(1)) < 1e-4)
    else:
        chk.ok("objective", 0, k, relfro(torch.tensor([obj]), orc["objective"].reshape(1)) < 1e-4)
    for name, g in grads.items():
        chk.ok("gradient", 0, k, relfro(eg[name], g) < 2e-2)


def _vae_run(tmp_path, case, W, steps=3, group=None, with_eval=False):
    from dalle_mtf_b200.model_fns import EVAL, TRAIN, vae_model_fn
    from oracle import vae_kl as OK
    make = lambda: _vae_params(tmp_path, model_path=None, **VAE_CASES[case])                # noqa: E731
    p = make()
    size, K, s = p["dataset"]["image_size"], p["num_tokens"], p["stack_factor"] or 1
    hw = size // s // 2 ** len(p["convblocks"])
    g = torch.Generator().manual_seed(17 + W)
    img = torch.rand(VAE_B, size, size, 3, generator=g) * 2 - 1
    u = torch.rand(VAE_B * hw * hw, K, generator=g).clamp_(1e-9, 1.0)
    uv = u.view(VAE_B, hw, hw, K)
    b = VAE_B // W
    rows = b * hw * hw
    kl_on = p["kl_loss_weight"] is not None
    group = group or RankGroup(W)
    chk = _Checks()
    shared = {"state": {}, "obj": {}, "usage": defaultdict(dict), "logits": defaultdict(dict), "orc_logits": {}}

    def fn(rank, dp):
        pr = make()
        pr["_dp"] = dp
        pr["_gumbel_u"] = u[rank * rows:(rank + 1) * rows].to(DEV)
        x = img[rank * b:(rank + 1) * b]
        spec = vae_model_fn(x, x, TRAIN, pr)
        eng = spec.engine
        n = eng.n_params_padded
        for k in range(steps):
            if rank == 0:
                orc = _vae_oracle(case, p, eng.export_params(), img, uv, k)
                shared["orc_logits"][k] = orc["logits"]
                m_old = eng.adam_m[:n].double()
            spec.train_op(x)
            obj = float(spec.loss_sum.item()) * spec.loss_scale
            if rank == 0:
                parts = [] if spec.loss_parts is None else spec.loss_parts.tolist()
                full = torch.zeros_like(eng.grads)
                for red in group.last_reduce:
                    off, numel, _, _ = red["sig"]
                    full[off:off + numel] = red["result"]
                full *= 1.0 / W
                _vae_check_step(chk, case, p, orc, k, obj, parts, eng.export_params(full))
                # the gradient Adam consumed: (m_new - b1 m_old) / (1 - b1) = the reduced gradient / W
                m_new = eng.adam_m[:n].double()
                g_adam = (m_new - ADAM_B1 * m_old) / (1 - ADAM_B1)
                bound = 2.0 ** -20 * (m_new.abs() + m_old.abs()) / (1 - ADAM_B1) + 1e-30
                chk.ok("adam_gradient", 0, k, bool(((g_adam - full[:n].double()).abs() <= bound).all()))
                shared["state"][k] = _state(eng)
                shared["obj"][k] = obj
            else:
                for got, exp in zip(_state(eng), shared["state"][k]):
                    chk.same("state", rank, k, got, exp)
                chk.ok("objective_ranks", rank, k, obj == shared["obj"][k])
            if kl_on:
                shared["logits"][k][rank] = eng._b["logits"][:rows].float().cpu()
                shared["usage"][k][rank] = spec.codebook_usage()
        if with_eval:
            pe = make()
            pe["_dp"] = dp
            pe["_gumbel_u"] = pr["_gumbel_u"]
            ev = vae_model_fn(x, x, EVAL, pe)
            ev.engine.copy_params_from(eng)
            ev.global_step = spec.global_step
            if rank == 0:
                orc = _vae_oracle(case, p, eng.export_params(), img, uv, spec.global_step)
            ev.eval_op(x)
            if rank == 0:
                got = float(ev.loss_sum.item()) * ev.loss_scale
                _vae_check_step(chk, case, p, orc, "eval", got, ev.loss_parts.tolist())
        return n, eng.aux_off

    (n, aux_off) = group.run(fn)[0]
    if kl_on:
        for k in range(steps):
            us = shared["usage"][k]
            own = OK.codebook_usage(torch.cat([shared["logits"][k][r] for r in range(W)]))[1:]
            chk.ok("codebook_usage", 0, k, all(us[r] == us[0] for r in range(W)) and us[0] == own)
            if not p["use_bf16"]:
                chk.ok("codebook_usage", 0, k, us[0] == OK.codebook_usage(shared["orc_logits"][k])[1:])
    return group, chk, n, aux_off


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("case", list(VAE_CASES))
def test_vae_ranks_match_the_oracle_of_the_global_batch(tmp_path, case, W):
    steps = 3
    group, chk, n, aux_off = _vae_run(tmp_path, case, W, steps, with_eval=(case == "logit-laplace-kl"))
    waits = [e for e in group.trace if e["kind"] == "wait"]
    buckets = _check_coverage(group.trace, n, aux_off, steps)
    assert buckets == 3                       # decoder + aux slots, codebook, encoder
    chk.assert_clean()
    print(f"[{TAG}] vae {case} W={W} B={VAE_B}: {steps} steps against the oracle of the global batch, "
          f"{chk.bitwise} state tensors bitwise across ranks, "
          f"{sum(1 for e in waits if len(e['ranges']) == 1)} single-range reductions (codebook usage / eval)")


# ====================================================================================================== Estimator
def _estimator_ranks(tmp_path, make, batches, W, max_steps, monkeypatch, group=None, per_rank=None):
    """One Estimator per rank, each with its own shard of the fixed global batches; returns the group, per-rank specs
    and log messages, and the ranks that called save_checkpoint."""
    from dalle_mtf_b200 import estimator as E
    group = group or RankGroup(W)
    saved = []
    save0 = E.save_checkpoint

    def save(*a, **k):
        saved.append(group.current_rank())
        return save0(*a, **k)

    monkeypatch.setattr(E, "save_checkpoint", save)
    logs = defaultdict(list)

    class _Log:
        def __init__(self, rank):
            self.rank = rank

        def info(self, msg):
            logs[self.rank].append(msg)

    def fn(rank, dp):
        p = make()
        p["_dp"] = dp
        if per_rank is not None:
            per_rank(p, rank)

        def input_fn(params):
            start = params.get("_data_seed_offset") or 0      # a resumed run continues with the next batches
            b = batches[0][0].shape[0] // W
            return iter([(f[rank * b:(rank + 1) * b], c[rank * b:(rank + 1) * b]) for f, c in batches[start:]])

        est = E.Estimator(p["_model_fn"], p, logger=_Log(rank))
        spec = est.train(input_fn, max_steps=max_steps)
        est.close()
        return spec

    specs = group.run(fn)
    monkeypatch.setattr(E, "save_checkpoint", save0)
    return group, specs, logs, saved


def test_estimator_two_ranks_save_log_and_resume_bitwise(tmp_path, monkeypatch):
    from dalle_mtf_b200.model_fns import dalle_model_fn
    W, B = 2, 4
    p0 = _dalle_params(tmp_path, {})
    batches = [_dalle_data(p0, B, seed=40 + i) for i in range(4)]

    def make(path):
        return lambda: _tiny_params(tmp_path, train_batch_size=B, model_path=str(tmp_path / path),
                                    steps_per_checkpoint=2, iterations=2, _model_fn=dalle_model_fn)

    _, full, logs, saved = _estimator_ranks(tmp_path, make("full"), batches, W, 4, monkeypatch)
    assert saved == [0, 0], saved
    assert not logs[1], logs[1]
    assert sum(m.startswith("step ") for m in logs[0]) == 2 and sum(m.startswith("saved ") for m in logs[0]) == 2
    _, first, _, saved1 = _estimator_ranks(tmp_path, make("resumed"), batches, W, 2, monkeypatch)
    assert saved1 == [0] and all(s.global_step == 2 for s in first)
    _, resumed, logs2, saved2 = _estimator_ranks(tmp_path, make("resumed"), batches, W, 4, monkeypatch)
    assert saved2 == [0] and any(m.startswith("restored ") for m in logs2[0]) and not logs2[1]
    count = 0
    for r in range(W):
        assert resumed[r].global_step == full[r].global_step == 4
        for got, exp in zip(_state(resumed[r].engine), _state(full[r].engine)):
            assert _same(got, exp), r
            count += 1
    print(f"[{TAG}] estimator W={W}: rank 0 alone saved (steps 2, 4) and logged; resumed at step 2, step 4 equals the "
          f"uninterrupted run ({count} state tensors bitwise)")


def test_estimator_vae_log_line_reports_the_collective_codebook_usage(tmp_path, monkeypatch):
    from dalle_mtf_b200.model_fns import vae_model_fn
    from oracle import vae_kl as OK
    W = 2
    g = torch.Generator().manual_seed(5)
    img = torch.rand(VAE_B, 16, 16, 3, generator=g) * 2 - 1
    u = torch.rand(VAE_B * 16, 64, generator=g).clamp_(1e-9, 1.0)
    rows = VAE_B // W * 16
    logits = {}
    model_fn0 = vae_model_fn

    def model_fn(features, labels, mode, params):
        spec = model_fn0(features, labels, mode, params)
        usage0 = spec.codebook_usage

        def usage():     # the engines' logits of the logged step, read before the collective
            logits[params["_dp"].rank] = spec.engine._b["logits"][:rows].float().cpu()
            return usage0()
        spec.codebook_usage = usage
        return spec

    def make():
        return _vae_params(tmp_path, model_path=str(tmp_path / "vae"), kl_loss_weight=0.5, steps_per_checkpoint=2,
                           iterations=2, _model_fn=model_fn)

    def own_noise(p, rank):
        p["_gumbel_u"] = u[rank * rows:(rank + 1) * rows].to(DEV)

    group = RankGroup(W)
    batches = [(img, img)] * 2
    _, specs, logs, saved = _estimator_ranks(tmp_path, make, batches, W, 2, monkeypatch, group=group,
                                             per_rank=own_noise)
    assert saved == [0] and not logs[1]
    line = [m for m in logs[0] if m.startswith("step 2 ")]
    assert len(line) == 1, logs[0]
    used, ppl = OK.codebook_usage(torch.cat([logits[r] for r in range(W)]))[1:]
    assert f" codes_used {used} perplexity {ppl:.2f}" in line[0], (line[0], used, ppl)
    usage_reductions = [e for e in group.trace if e["kind"] == "wait" and e["ranges"] == [(0, 64, F32, True)]]
    assert len(usage_reductions) == 1
    print(f"[{TAG}] estimator vae W={W}: {line[0]!r}")


# ====================================================================================================== mutations
def _hook_mutant(monkeypatch, change):
    base = RankMember.make_bucket_hook

    def make_bucket_hook(self, flat):
        hook = base(self, flat)
        n = flat.numel()

        def mutated(start, end):
            r = change(start, end, n)
            if r is not None:
                hook(*r)
        return mutated

    monkeypatch.setattr(RankMember, "make_bucket_hook", make_bucket_hook)


def _dalle_mutant_run(rec, tmp_path, extra, W, mutate, steps=1, group=None):
    B = 12
    make = lambda **kw: _dalle_params(tmp_path, extra, train_batch_size=B, **kw)      # noqa: E731
    p = make()
    feats, caps = _dalle_data(p, B, seed=W)
    ref, _, _ = _dalle_reference(rec, make(tokens_per_mb_per_replica=(B // W) * _seq_len(p)), feats, caps, W,
                                 steps=2)
    mutate()
    _, chk, _ = _dalle_ranks(rec, make, feats, caps, W, ref, steps=steps, group=group)
    return chk


DROP_ZERO = lambda s, e, n: None if s == 0 else (s, e)                    # noqa: E731
CLIP_AUX = lambda s, e, n: (s, min(e, n - 64))                            # noqa: E731


@pytest.mark.parametrize("mutant", ["drop-range-0", "aux-not-reduced"])
def test_mutant_bucket_ranges_are_caught(rec, tmp_path, monkeypatch, mutant):
    change, dalle_check, vae_check = {"drop-range-0": (DROP_ZERO, "gradient", "gradient"),
                                      "aux-not-reduced": (CLIP_AUX, "loss", "objective")}[mutant]
    chk = _dalle_mutant_run(rec, tmp_path, {}, 2, lambda: _hook_mutant(monkeypatch, change))
    assert dalle_check in chk.failed, dict(chk.failed)
    _, vchk, _, _ = _vae_run(tmp_path, "fp32-mse", 2, steps=1)
    assert vae_check in vchk.failed, dict(vchk.failed)
    print(f"[{TAG}] mutant {mutant}: DALL-E {sorted(chk.failed)}, VAE {sorted(vchk.failed)} fail")


def test_mutant_row_offsets_are_caught(rec, tmp_path, monkeypatch):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.dalle_engine import DalleEngine
    drop = dict(embed_dropout=0.1, attention_dropout=0.1, residual_dropout=0.1)

    def no_rank_offset():
        fwd = DalleEngine.forward

        def forward(eng, tokens, loss_accum=None, step=None, row0=0, global_batch=None):
            return fwd(eng, tokens, loss_accum=loss_accum, step=step, row0=row0 % tokens.shape[0],
                       global_batch=global_batch)
        monkeypatch.setattr(DalleEngine, "forward", forward)

    chk = _dalle_mutant_run(rec, tmp_path, drop, 2, no_rank_offset)
    assert "loss_rows" in chk.failed, dict(chk.failed)
    monkeypatch.undo()
    rec2 = _Rec(monkeypatch)

    def caption_without_first_row():
        make = L.make_dropout

        def make_dropout(rate, seed, step, site, row0=0):
            return make(rate, seed, step, site, 0 if site == L.SITE_CAPTION else row0)
        monkeypatch.setattr(L, "make_dropout", make_dropout)

    chk2 = _dalle_mutant_run(rec2, tmp_path, {"caption_dropout": 0.5, "padding_id": 299}, 2,
                             caption_without_first_row)
    assert "tokens" in chk2.failed, dict(chk2.failed)
    print(f"[{TAG}] mutant row0 without the rank offset: {sorted(chk.failed)} fail; caption drops without first_row: "
          f"{sorted(chk2.failed)} fail")


def test_mutant_vae_adam_scale_is_caught(tmp_path, monkeypatch):
    from dalle_mtf_b200.vae_engine import VaeEngine
    step0 = VaeEngine.optimizer_step
    monkeypatch.setattr(VaeEngine, "optimizer_step",
                        lambda self, lr, step, grad_scale=1.0, **k: step0(self, lr, step, grad_scale=1.0, **k))
    _, chk, _, _ = _vae_run(tmp_path, "fp32-mse", 2, steps=1)
    assert "adam_gradient" in chk.failed, dict(chk.failed)
    print(f"[{TAG}] mutant VAE Adam grad_scale 1: {sorted(chk.failed)} fail")


def test_mutant_write_after_launch_is_caught(rec, tmp_path, monkeypatch):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    bwd = DalleEngine._block_bwd

    def block_bwd(eng, i, *a, **k):
        out = bwd(eng, i, *a, **k)
        if i + 1 < eng.L:       # block i+1's range was launched before this block's backward
            eng.G(f"l{i + 1}.b2").view(-1)[0] += 1.0
        return out

    with pytest.raises(RankGroupError, match=r"written after its all-reduce was launched"):
        _dalle_mutant_run(rec, tmp_path, {}, 2, lambda: monkeypatch.setattr(DalleEngine, "_block_bwd", block_bwd))
    print(f"[{TAG}] mutant write after launch: the group's snapshot check fails")


def test_mutant_reversed_rank_order_is_caught(rec, tmp_path):
    group = RankGroup(3, keep_inputs=False)
    group.reduce_order = lambda: [2, 1, 0]
    chk = _dalle_mutant_run(rec, tmp_path, {}, 3, lambda: None, group=group)
    assert "gradient" in chk.failed, dict(chk.failed)
    print(f"[{TAG}] mutant reversed rank order W=3: {sorted(chk.failed)} fail")
