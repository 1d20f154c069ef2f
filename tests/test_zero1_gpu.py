"""ZeRO-1 optimizer-state sharding (DalleEngine(zero=...), the `optimizer_state_sharding` key) on one GPU, bit for bit.

W ranks run in one process.  A loopback group hands rank r's engine a stand-in with world = W and rank = r:
  * all_gather_inplace(buf, chunk) completes once every rank has entered it: slice r of rank r's buffer is copied
    into every rank's buffer.  Ranks whose call returned before the last one entered rebuild their fp32 vector
    parameters (vec32) then, as they would after a real collective returns; the last rank to enter rebuilds its own in
    optimizer_step.  The order in which the ranks step rotates every step, so each rank's own rebuild is exercised.
  * the gradient all-reduce is an fp32 sum over the ranks in rank order, written into every rank's `grads` (aux slots
    included): every rank sees the same reduced gradient, as NCCL guarantees.

Against this, the sharded state must equal a full fp32 P / M / V stepped with the same ops.adam_step call the
replicated optimizer_step makes, bitwise; every rank's bf16 copy must be bf16(P) and vec32 float(bf16(P)); and a
replicated twin engine whose master is P with the vector parameters replaced by vec32 must produce the rank's logits,
loss sums and gradient buffer bitwise: ZeRO-1 is the replicated step on bf16-rounded vector parameters, exactly.

Also here: db200_gather_cast_bf16_f32 against the exact bf16 -> fp32 widening (64-bit source offsets included), the
ZeRO-1 checkpoint restore of dalle_model_fn and the Estimator's evaluation of the weights being trained.
"""
import gc
import itertools
import math
import time

import pytest
import torch

from test_dalle_kernels_gpu import check_adam_update
from test_parity_baseline_gpu import _randomise_small_params

pytestmark = pytest.mark.gpu

F32, F64, BF16, I16, I32 = torch.float32, torch.float64, torch.bfloat16, torch.int16, torch.int32
DEV = "cuda"
TAG = "zero1"
ADAM_SLAB = 1 << 24          # float64 elements per slab of the float64 Adam check

# geometry = DalleEngine's leading arguments (n_embd, n_layers, n_heads, text_vocab, image_vocab, text_len, image_len)
EXAMPLE = (512, 6, 4, 50258, 512, 256, 1024)        # dalle_example: V 50 771, S 1280
WIDE = (4096, 1, 32, 3000, 570, 64, 256)            # 12B width, the reduced vocabulary of the 12B parity test
TINY = (256, 2, 2, 226, 64, 16, 16)                 # W = 2 puts the shard boundary inside l1.ln1_g
TINY_FEATURES = dict(loss_weights=(1.0, 7.0), z_loss=1e-3, dropout=(0.1, 0.1, 0.1), dropout_seed=3,
                     attention_types=["global", "local"], local_attention_radius=8, recompute_grad=True)
CASES = [("dalle_example", EXAMPLE, 2, {}), ("dalle_example", EXAMPLE, 3, {}), ("dalle_example", EXAMPLE, 8, {}),
         ("12B-width", WIDE, 2, {}), ("12B-width", WIDE, 4, {}), ("tiny features", TINY, 2, TINY_FEATURES)]
# step k of every case: clip active (asserted), clip inactive (asserted), clipping disabled
CLIPS = (1e-3, 1e4, None)
LR = 4e-3


_PEAK = [0]


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    yield _ops
    print(f"[{TAG}] peak device memory of the module {_PEAK[0] / 2 ** 30:.2f} GiB")


@pytest.fixture(autouse=True)
def _cost(request):
    gc.collect()        # a loopback group and its engines form a reference cycle: free the previous test's now
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f"[{TAG}] {request.node.name}: {time.time() - t0:.1f} s, peak device memory {peak / 2 ** 30:.2f} GiB")


def _engine(geom, **kw):
    from dalle_mtf_b200.dalle_engine import DalleEngine
    return DalleEngine(*geom, device=DEV, **kw)


def _bits(t):
    return t.view({F32: I32, BF16: I16}[t.dtype])


def assert_same_bits(got, ref, what):
    """Bitwise equality (-0 != +0, NaN payloads compared), with the first differing element on failure."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    diff = _bits(got) != _bits(ref)
    if bool(diff.any()):
        i = int(diff.nonzero()[0, 0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {got.numel()} elements differ, first at {i}: "
                             f"{got[i].item()!r} != {ref[i].item()!r}")


# ------------------------------------------------------------------------------------------------------ loopback group
class Loopback:
    """W data-parallel ranks inside one process; `engines[r]` is rank r's DalleEngine (built with member(r))."""

    def __init__(self, world):
        self.world = world
        self.engines = []
        self._entered = {}

    def member(self, rank):
        return _Member(self, rank)

    def all_gather(self, rank, buf, chunk):
        self._entered[rank] = (buf, chunk)
        if len(self._entered) < self.world:
            return
        entered, self._entered = self._entered, {}
        assert len({c for _, c in entered.values()}) == 1, "ranks disagree on the slice size"
        for r, (src, c) in entered.items():
            for q, (dst, _) in entered.items():
                if q != r:
                    dst[r * c:(r + 1) * c].copy_(src[r * c:(r + 1) * c])
        for r in entered:          # their calls returned before the data arrived
            if r != rank:
                self.engines[r]._refresh_vecs()

    def all_reduce_grads(self):
        total = self.engines[0].grads          # summed in rank order in place, then handed to every other rank
        for e in self.engines[1:]:
            total += e.grads
        for e in self.engines[1:]:
            e.grads.copy_(total)


class _Member:
    enabled = True

    def __init__(self, group, rank):
        self.group, self.rank, self.world = group, rank, group.world

    def all_gather_inplace(self, buf, count_per_rank):
        self.group.all_gather(self.rank, buf, count_per_rank)
        return buf


def _layout_of(geom):
    from dalle_mtf_b200.dalle_engine import param_layout
    d, n_layers, _, tv, iv, tl, il = geom
    return param_layout(d, n_layers, tv + iv + 1, tl + il)


def _chunk(size, world):
    """DalleEngine's elements per rank: ceil(size / world) rounded up to 64 (equal slices for the in-place gather)."""
    return (-(-size // world) + 63) // 64 * 64


def _boundary_cuts(lay, world):
    """Names of the parameters that a shard boundary of `world` ranks cuts strictly inside."""
    chunk = _chunk(lay.size, world)
    return {name for r in range(1, world) for name, (off, shape) in lay.entries.items()
            if off < r * chunk < off + math.prod(shape)}


def test_chosen_cases_cut_a_vector_parameter_wout_and_wte():
    """The cases below put a shard boundary strictly inside a vector parameter, inside the (column-padded) vocabulary
    projection and inside the embedding table, and at least one leaves the last shard shorter than the others."""
    from dalle_mtf_b200.dalle_engine import DalleEngine
    cuts, short = set(), []
    for name, geom, world, _ in CASES:
        lay = _layout_of(geom)
        cuts |= _boundary_cuts(lay, world)
        if world * _chunk(lay.size, world) > lay.size:
            short.append(f"{name} W={world}: last shard {world * _chunk(lay.size, world) - lay.size} short")
    assert {c for c in cuts if c.split(".")[-1] in DalleEngine.VECTOR_PARAMS}, cuts
    assert "wout" in cuts and "wte" in cuts, cuts
    assert short
    print(f"[{TAG}] shard boundaries cut {sorted(cuts)}; {'; '.join(short)}")


# ------------------------------------------------------------------------------------------------------ state checks
def _vector_names(eng):
    return [n for n in eng.layout.order if n.split(".")[-1] in eng.VECTOR_PARAMS]


def assert_state(tag, ranks, P, M=None, V=None):
    """The sharded state of `ranks` against the full fp32 buffers P (and M, V): concatenated slices bitwise, every
    rank's bf16 copy bf16(P) with zeros behind the layout, vec32 float(bf16(P)) of every vector parameter."""
    lay = ranks[0].layout
    n, W, chunk = lay.size, len(ranks), ranks[0].chunk
    for e in ranks:
        assert e.master.numel() == chunk and e.shard == (min(e.zero.rank * chunk, n), min((e.zero.rank + 1) * chunk, n))
    for name, full in (("master", P), ("adam_m", M), ("adam_v", V)):
        if full is not None:
            cat = torch.cat([getattr(e, name)[:e.shard[1] - e.shard[0]] for e in ranks])
            assert_same_bits(cat, full, f"{tag}: concatenated {name} slices")
    P16 = P.to(BF16)
    for r, e in enumerate(ranks):
        assert_same_bits(e.shadow[:n], P16, f"{tag}: rank {r} bf16 parameters")
        tail = e.shadow[n:W * chunk]
        assert not bool((_bits(tail) != 0).any()), f"{tag}: rank {r} bf16 copy is not zero behind the layout"
        for name in _vector_names(e):
            assert_same_bits(e.P(name), lay.view(P16, name).float(), f"{tag}: rank {r} vec32 {name}")


def _make_ranks(geom, world, kw):
    grp = Loopback(world)
    grp.engines = [_engine(geom, zero=grp.member(r), **kw) for r in range(world)]
    return grp, grp.engines


def _twin_from(twin, P, zero_engine):
    """The replicated twin: master = P with every vector parameter replaced by the ZeRO engine's vec32."""
    n = twin.n_params_padded
    twin.master[:n].copy_(P)
    for name in _vector_names(twin):
        twin.P(name).copy_(zero_engine.P(name))
    twin.refresh_shadow()


def _adam_f64_slabs(tag, before, after, gn, clip):
    """check_adam_update on slabs of one rank's slice (the float64 temporaries stay small); returns whether the clip
    scaled the gradient."""
    n = before[0].numel()
    clipped = set()
    for s in range(0, n, ADAM_SLAB):
        e = min(n, s + ADAM_SLAB)
        ins = tuple(t[s:e] for t in before) + (gn,)
        outs = tuple(t[s:e] for t in after)
        clipped.add(check_adam_update(f"{tag} [{s}:{e})", ins, outs, LR, 0.9, 0.999, 1e-6, 0.0, clip or 0.0, 1.0,
                                      False, 0))
    assert len(clipped) == 1
    return clipped.pop()


@pytest.mark.parametrize("name,geom,world,kw", CASES, ids=[f"{c[0]}-W{c[2]}" for c in CASES])
def test_zero1_sharded_state_equals_replicated_bitwise(ops, name, geom, world, kw):
    from oracle import dalle as O
    tag = f"{name} W={world}"
    grp, ranks = _make_ranks(geom, world, kw)
    twin = _engine(geom, **kw)
    n = twin.n_params_padded
    assert ranks[0].chunk == _chunk(n, world) and twin.layout.entries == _layout_of(geom).entries

    # ---- init and load
    twin.init_params(seed=11)
    for e in ranks:
        e.init_params(seed=11)
    assert_state(f"{tag} init_params", ranks, twin.master[:n])
    exp_rep, exp_z = twin.export_params(), ranks[-1].export_params()
    assert exp_rep.keys() == exp_z.keys()
    for k in exp_rep:
        assert_same_bits(exp_z[k], exp_rep[k].to(BF16).float(), f"{tag}: export {k}")
    del exp_rep, exp_z
    cfg = O.DalleConfig(*geom)
    named = O.init_params(cfg, seed=5)
    _randomise_small_params(named, torch.Generator().manual_seed(6))
    twin.load_params(named)
    for e in ranks:
        e.load_params(named)
    del named
    assert_state(f"{tag} load_params", ranks, twin.master[:n])
    P = twin.master[:n].clone()
    M, V = torch.zeros_like(P), torch.zeros_like(P)
    gn = torch.zeros(1, dtype=F32, device=DEV)

    # ---- K optimizer steps on the global batch
    b, S = 1, twin.S
    g = torch.Generator(device=DEV).manual_seed(world)
    weighted = twin.weighted_loss
    scale = 1.0 if weighted else 1.0 / (world * b * S)
    for k, clip in enumerate(CLIPS):
        tok = torch.randint(0, twin.V - 1, (world * b, S), generator=g, device=DEV, dtype=I32)
        _twin_from(twin, P, ranks[0])
        assert_same_bits(twin.shadow[:n], ranks[0].shadow[:n], f"{tag} step {k}: twin bf16 parameters")
        for r, e in enumerate(ranks):
            shard = tok[r * b:(r + 1) * b]
            for eng in (e, twin):
                eng.zero_grads()
                eng.forward(shard, step=k, row0=r * b, global_batch=world * b)
                eng.backward(scale)
            # gradients and the loss sums in the aux slots behind them, before the all-reduce
            assert_same_bits(e.grads, twin.grads, f"{tag} step {k}: rank {r} gradients + loss sums vs the twin")
            assert_same_bits(e.logits(shard), twin.logits(shard), f"{tag} step {k}: rank {r} logits vs the twin")
        grp.all_reduce_grads()
        G = ranks[0].grads[:n]          # the ZeRO-1 Adam step reads its slice and leaves the buffer as it is
        if clip:
            gn.zero_()
            ops.sqnorm(G, gn)
            gnorm = math.sqrt(gn.item())
            assert (gnorm > clip) == (k == 0), (tag, k, gnorm, clip)
        order = [(k + i) % world for i in range(world)]     # the last rank to enter the gather rotates
        for r in order:
            ranks[r].optimizer_step(LR, clip=clip)
        if clip:
            for r, e in enumerate(ranks):
                assert_same_bits(e.gnorm_sq, gn, f"{tag} step {k}: rank {r} gnorm_sq")
        if k == 0:      # each rank's slice against float64 Adam on the state before the step
            for r, e in enumerate(ranks):
                lo, hi = e.shard
                m = hi - lo
                assert _adam_f64_slabs(f"{tag} step 0 rank {r}", (P[lo:hi], M[lo:hi], V[lo:hi], G[lo:hi]),
                                       (e.master[:m], e.adam_m[:m], e.adam_v[:m], e.shadow[lo:hi]), gn, clip)
        # the twin's bf16 copy takes the bf16 output (it is rebuilt from P at the next step)
        ops.adam_step(P, M, V, G, twin.shadow[:n], LR, 0.9, 0.999, 1e-6, 0.0, gn if clip else None, clip or 0.0, 1.0, False, 0)
        assert_state(f"{tag} step {k} (clip {clip})", ranks, P, M, V)
    moved = (_bits(P.to(BF16)) != _bits(twin.master[:n].to(BF16))).float().mean().item()
    print(f"[{TAG}] {tag}: {len(CLIPS)} steps bitwise; the last step changed {moved:.1%} of the bf16 parameters")


def test_zero1_refuses_weight_decay(ops):
    from dalle_mtf_b200 import lib as L
    grp, ranks = _make_ranks(TINY, 2, {})
    for e in ranks:
        e.init_params(seed=1)
    with pytest.raises(L.DB200Error, match="weight_decay"):
        ranks[0].optimizer_step(1e-3, weight_decay=0.01)


# ------------------------------------------------------------------------------------------------------ gather_cast
SEGMENT_LENGTHS = (1, 63, 64, 255, 256, 257, 4096, 16384, 50816)
SENTINEL = 0x7FBADBAD      # a NaN that no bf16 value widens to (its low 16 bits are not zero)


def _widen_bits(src):
    """The exact bf16 -> fp32 widening as int32 bit patterns: the 16 bits move to the top, the rest are zero."""
    return _bits(src).to(I32) << 16


def _special_bf16(n, gen):
    """Random bf16 bit patterns (every class: normals, subnormals, NaN payloads) with +-0, +-min subnormal, +-max
    subnormal, +-inf, quiet and signalling NaNs of both signs at the front."""
    bits = torch.randint(-32768, 32768, (n,), generator=gen, device=DEV, dtype=I32).to(I16)
    special = [0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x807F, 0x7F80, 0xFF80, 0x7FC0, 0xFFC1, 0x7F81, 0xFFBF,
               0x0080, 0x7F7F, 0xFF7F]
    sp = torch.tensor([s - 65536 if s >= 32768 else s for s in special], dtype=I16, device=DEV)
    k = min(n, sp.numel())
    bits[:k] = sp[:k]
    return bits.view(BF16)


def _run_gather_cast(ops, src, segments, dst_len):
    """segments = [(src_off, dst_off, n)]; returns dst after one launch over a NaN-sentinel buffer."""
    dst = torch.full((dst_len,), SENTINEL, dtype=I32, device=DEV).view(F32)
    table = torch.tensor([x for s in segments for x in s], dtype=torch.int64, device=DEV)
    ops.gather_cast(src, dst, table, len(segments))
    torch.cuda.synchronize()
    return dst


def _check_gather_cast(src, segments, dst, what):
    expect = torch.full_like(dst, 0).view(I32).fill_(SENTINEL)
    for so, do, n in segments:
        expect[do:do + n] = _widen_bits(src[so:so + n])
    diff = (_bits(dst) != expect)
    if bool(diff.any()):
        i = int(diff.nonzero()[0, 0])
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at dst {i}: "
                             f"{int(_bits(dst)[i]) & 0xFFFFFFFF:#010x} != {int(expect[i]) & 0xFFFFFFFF:#010x}")


def test_gather_cast_bf16_f32_segments_special_values_and_gaps(ops):
    gen = torch.Generator(device=DEV).manual_seed(17)
    src = _special_bf16(1 << 18, gen)
    # torch's widening agrees with the bit-level definition on every non-NaN value
    finite = ~torch.isnan(src)
    assert torch.equal(_bits(src.float())[finite], _widen_bits(src)[finite])
    # unaligned, unordered source offsets (one range read twice), destinations separated by sentinel gaps of 1..65
    segments, do = [], 3
    for i, n in enumerate(SEGMENT_LENGTHS):
        so = (i * 40503 + 7 * n + 1) % (src.numel() - n)
        segments.append((so, do, n))
        do += n + 1 + (i * 29) % 65
    segments.append((segments[3][0], do, SEGMENT_LENGTHS[3]))          # the same source range again
    do += SEGMENT_LENGTHS[3] + 5
    segments.append((0, do, 15))                                        # the special values themselves
    do += 15 + 2
    dst = _run_gather_cast(ops, src, segments, do)
    _check_gather_cast(src, segments, dst, "gather_cast")
    print(f"[{TAG}] gather_cast: {len(segments)} segments, lengths {sorted({s[2] for s in segments})}, bitwise")
    # no segments: OK and nothing written
    before = dst.clone()
    ops.gather_cast(src, dst, torch.zeros(3, dtype=torch.int64, device=DEV), 0)
    torch.cuda.synchronize()
    assert_same_bits(dst, before, "gather_cast with 0 segments")


def test_gather_cast_bf16_f32_source_offsets_beyond_32_bits(ops):
    """The 12B layout puts vector parameters near element 8.5e9 of the bf16 copy.  Offsets >= 2^32 elements: a kernel
    that kept 32-bit offsets would read the low elements, which hold different values, inside the buffer."""
    base, span = 1 << 32, 1 << 17
    big = torch.empty(base + span, dtype=BF16, device=DEV)       # 8 GiB + 256 KiB, freed below
    try:
        gen = torch.Generator(device=DEV).manual_seed(23)
        big[:span] = _special_bf16(span, gen)
        big[base:] = _special_bf16(span, gen)
        big[base:base + 15] = big[base + 15:base + 30]               # the truncated reads differ from the first elements
        segments = [(base + 12345, 0, 4096), (base + span - 257, 4100, 257), (base, 4400, 64), (7, 4500, 300),
                    ((1 << 31) - 5, 4900, 10)]
        dst = _run_gather_cast(ops, big, segments, 4910)
        _check_gather_cast(big, segments, dst, "gather_cast 64-bit source offsets")
        print(f"[{TAG}] gather_cast: source offsets up to {base + span - 1} (>= 2^32), bitwise")
    finally:
        del big
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------ model_fn / Estimator
class _IdentityGroup:
    """Rank 0 of a 2-rank data-parallel group whose collectives leave every buffer as it is: enough to run the ZeRO-1
    code paths of dalle_model_fn and the Estimator in one process (no real 2-rank trajectory)."""
    world, rank, enabled = 2, 0, True

    def shard(self, global_batch):
        return 0, global_batch // self.world

    def hint_tokens_per_gpu(self, tokens):
        pass

    def make_bucket_hook(self, flat):
        return None

    def begin_overlap(self):
        pass

    def wait(self):
        pass

    def all_reduce_now(self, t):
        return t

    def all_gather_inplace(self, buf, count_per_rank):
        return buf

    def barrier(self):
        pass


def _params(tmp_path, **extra):
    from collections import defaultdict
    vae = defaultdict(lambda: None, {"model_type": "vae", "num_tokens": 64, "convblocks": [[2, 64], [2, 64]],
                                     "dataset": {"image_size": 16}})
    p = defaultdict(lambda: None, {"model_type": "dalle", "dataset": {"image_size": 16}, "train_batch_size": 4,
                                   "eval_batch_size": 4, "n_embd": 256, "n_layers": 2, "n_heads": 2,
                                   "text_vocab_size": 300, "image_vocab_size": 64, "text_seq_len": 12, "lr": 1e-2,
                                   "train_steps": 100, "warmup_steps": 0, "bf_16": True, "mesh_shape": "data:1",
                                   "layout": "batch_dim:data", "model_path": str(tmp_path / "dalle"),
                                   "iterations": 100, "vae_params": vae, "vae_random_init": True, "seed": 5})
    p.update(extra)
    return p


def _feed(batch):
    return lambda params: itertools.repeat(batch)


def _local_batch(params):
    local = params["train_batch_size"] // (params["_dp"].world if params.get("_dp") else 1)
    g = torch.Generator().manual_seed(3)
    return torch.rand(local, 16, 16, 3, generator=g) * 2 - 1, torch.randint(0, 299, (local, 12), generator=g)


def test_zero1_checkpoint_restores_for_evaluation_and_refuses_a_training_restart(tmp_path):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.model_fns import EVAL, dalle_model_fn
    params = _params(tmp_path, optimizer_state_sharding=True, _dp=_IdentityGroup())
    batch = _local_batch(params)
    est = Estimator(dalle_model_fn, params)
    train = est.train(_feed(batch), max_steps=2)              # saves a checkpoint at step 2
    assert train.engine.zero is not None and train.global_step == 2
    est.evaluate(_feed(batch), steps=1)                       # train_dalle.py's eval: loads that checkpoint
    # a fresh process evaluating the checkpoint: the loaded weights are the trained ones, bit for bit
    fresh = Estimator(dalle_model_fn, params)
    fresh.evaluate(_feed(batch), steps=1)
    ev = fresh._specs[EVAL]
    assert ev.engine.zero is not None and ev.global_step == train.global_step
    n = train.engine.n_params_padded
    assert_same_bits(ev.engine.shadow[:n], train.engine.shadow[:n], "loaded bf16 parameters")
    assert_same_bits(ev.engine.vec32, train.engine.vec32, "loaded vec32")
    # resuming training would restart Adam's moments from zero: refused
    with pytest.raises(L.DB200Error, match="Adam slots"):
        Estimator(dalle_model_fn, params).train(_feed(batch), max_steps=3)
    est.close(); fresh.close()


@pytest.mark.parametrize("mode", ["replicated", "zero1"])
def test_evaluate_reads_the_weights_being_trained(tmp_path, mode):
    """Two steps that visibly move the weights, then evaluate: the eval loss is the train engine's own forward on the
    batch, bitwise, and differs from the initial weights' loss.  No model_path: nothing is saved or restored, so the
    eval engine only has the weights it is handed."""
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.model_fns import dalle_model_fn
    extra = {"optimizer_state_sharding": True, "_dp": _IdentityGroup()} if mode == "zero1" else {}
    params = _params(tmp_path, model_path=None, **extra)
    batch = _local_batch(params)
    initial = dalle_model_fn(*batch, "eval", params)
    loss0 = initial.eval_op(*batch).item() * initial.loss_scale
    est = Estimator(dalle_model_fn, params)
    train = est.train(_feed(batch), max_steps=2)
    loss = est.evaluate(_feed(batch), steps=1)["loss"]
    # the train engine's own forward on the same batch (no dropout, same kernels)
    acc = torch.zeros(1, dtype=F32, device=DEV)
    train.engine.forward(train.assemble(*batch), loss_accum=acc, global_batch=params["eval_batch_size"])
    expect = float(acc.item()) * train.loss_scale
    print(f"[{TAG}] evaluate ({mode}): initial weights {loss0:.6f}, after 2 steps {loss:.6f}, train engine {expect:.6f}")
    assert loss != loss0, "evaluation read the initial weights"
    assert loss == expect
    est.close()
