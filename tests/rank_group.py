"""W data-parallel ranks in one process: an in-process stand-in for the collectives of dalle_mtf_b200.dist.

`RankGroup(world).member(rank)` is a `DataParallel` with world = W, rank = r and no communicator.  It keeps the
package's own shard / make_bucket_hook / all_reduce_now / begin_overlap / hint_tokens_per_gpu and replaces only the
transport: `_launch`, `wait`, `all_gather_inplace`, `barrier` and `max_over_ranks`.  So what a test sees is the bucket
bookkeeping the model functions really do.

`group.run(fn)` runs fn(rank, member) on one thread per rank, serially: exactly one rank thread runs at a time.  A rank
hands the baton to the next one when it enters a collective (or returns from fn); ranks enter in order 0..W-1, the last
one to enter performs the collective and the ranks then resume in order 0..W-1.  CUDA is never used from two threads
at once, the run is deterministic, and the package needs no locking.

What the rendezvous of `wait()` checks and does, each violation breaking the group with a RankGroupError:
  (a) every rank launched the same ranges: the same (offset, numel, dtype, exposed) sequence;
  (b) every range still holds, bitwise, what it held when its all-reduce was launched (a snapshot taken then, after a
      synchronize): nothing may write into a range once NCCL may be reading it;
  (c) each range is summed in fp32 in rank order, ((x0 + x1) + x2) + ..., and the sum is written into every rank's
      range, as NCCL's in-place all-reduce leaves the same result on every rank.  The per-rank inputs and the result
      are kept in `group.last_reduce`.
`all_reduce_now` goes through the same path (it is `_launch` + `wait`); `all_gather_inplace` copies slice r of rank r
into every rank's buffer.  `group.trace` lists every collective: its kind and the ranges it reduced.

A rank that raises, ranks that disagree on the collective they are in (one returns while another waits), or no
progress within `timeout_s` break the group: every waiting rank raises RankGroupError naming what each rank is blocked
in, `run` joins every thread and re-raises the first error.  A missing collective fails instead of hanging.
"""
import threading
import time

import torch

from dalle_mtf_b200.dist import DataParallel

_INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}


class RankGroupError(RuntimeError):
    """The group is broken: a rank raised, the ranks disagree on a collective, or a rendezvous timed out."""


def _bits(t):
    return t.view(_INT_VIEW[t.dtype]) if t.dtype in _INT_VIEW else t


def _sync():
    if torch.cuda.is_available():
        torch.cuda.synchronize()


class _Launch:
    """One pending range: the view, where it sits in its buffer, and a bitwise snapshot taken at launch."""

    def __init__(self, t, exposed):
        self.view = t
        self.sig = (t.storage_offset(), t.numel(), t.dtype, bool(exposed))
        _sync()
        self.snapshot = t.clone()


class RankMember(DataParallel):
    """Rank `rank` of a RankGroup: the package's DataParallel bookkeeping over the group's in-process transport."""

    def __init__(self, group, rank):
        super().__init__()
        self.group = group
        self.world, self.rank, self.local_rank = group.world, rank, 0
        self.enabled = True
        self.comm = self.comm_tail = None
        self._want_comm = False
        self._pending = []

    def _launch(self, t, exposed=False):
        if t.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"all-reduce of a {t.dtype} tensor: the data plane carries fp32 and bf16 only")
        if not t.is_contiguous():
            raise ValueError("all-reduce of a non-contiguous view")
        self._pending.append(_Launch(t, exposed))

    def wait(self):
        pending, self._pending = self._pending, []
        self.group._collective(self.rank, "wait", pending)

    def all_gather_inplace(self, buf, count_per_rank):
        self.group._collective(self.rank, "all_gather", (buf, count_per_rank))
        return buf

    def barrier(self):
        self.group._collective(self.rank, "barrier", None)

    def max_over_ranks(self, value):
        return self.group._collective(self.rank, "max_over_ranks", float(value))


class RankGroup:
    def __init__(self, world, timeout_s=120, keep_inputs=True):
        if world < 1:
            raise ValueError(f"world = {world}")
        self.world = world
        self.timeout_s = timeout_s
        self.keep_inputs = keep_inputs      # False: last_reduce keeps only the results (saves W copies of the buffer)
        self.trace = []                     # [{"kind": ..., "ranges": [(offset, numel, dtype, exposed), ...]}]
        self.last_reduce = []               # [{"sig": (offset, numel, dtype, exposed), "inputs": [...], "result": t}]
        self._members = [RankMember(self, r) for r in range(world)]
        self._cv = threading.Condition()
        self._tls = threading.local()
        self._reset()

    def member(self, rank):
        return self._members[rank]

    def reduce_order(self):
        """The order in which the ranks' contributions are added (rank order)."""
        return list(range(self.world))

    def current_rank(self):
        """The rank whose thread calls this (None outside run)."""
        return getattr(self._tls, "rank", None)

    # ------------------------------------------------------------------------------------------------ run
    def _reset(self):
        self._turn = 0
        self._phase = 0
        self._state = ["not started"] * self.world
        self._entered = [None] * self.world
        self._results = [None] * self.world
        self._returns = [None] * self.world
        self._errors = []
        self._broken = None
        self._progress = time.monotonic()
        for m in self._members:
            m._pending = []

    def run(self, fn):
        """fn(rank, member) on one thread per rank, serially (see the module docstring); returns [fn's result per
        rank].  Joins every thread before it returns or re-raises the first error."""
        self._reset()
        threads = [threading.Thread(target=self._main, args=(r, fn), name=f"rank-{r}", daemon=True)
                   for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if self._errors:
            raise self._errors[0][1]
        return list(self._returns)

    def _main(self, rank, fn):
        self._tls.rank = rank
        try:
            with self._cv:
                self._await(rank, lambda: self._phase == 0 and self._turn == rank, "its first turn")
                self._state[rank] = "running"
            if torch.cuda.is_available():
                torch.cuda.set_device(0)
            self._returns[rank] = fn(rank, self._members[rank])
            with self._cv:
                self._arrive(rank, "returned", None)
        except BaseException as e:          # noqa: BLE001 - handed to run()
            with self._cv:
                self._errors.append((rank, e))
                self._state[rank] = f"raised {type(e).__name__}"
                if self._broken is None:
                    self._break(f"rank {rank} raised {type(e).__name__}: {e}")

    # ------------------------------------------------------------------------------------------------ baton
    def _describe(self):
        return "; ".join(f"rank {r}: {s}" for r, s in enumerate(self._state))

    def _break(self, why):
        self._broken = f"{why} [{self._describe()}]"
        self._cv.notify_all()

    def _await(self, rank, cond, what):
        while not cond():
            if self._broken is not None:
                raise RankGroupError(f"rank {rank} waiting for {what}: group broken: {self._broken}")
            left = self.timeout_s - (time.monotonic() - self._progress)
            if left <= 0:
                self._break(f"no progress within {self.timeout_s} s while rank {rank} waited for {what}")
                continue
            self._cv.wait(timeout=min(left, 1.0))
        if self._broken is not None:
            raise RankGroupError(f"rank {rank} waiting for {what}: group broken: {self._broken}")

    def _arrive(self, rank, kind, payload):
        """Rank `rank` (holding the baton) enters collective `kind` or returns from fn; hands the baton on or, as the
        last rank, completes the phase."""
        if self._broken is not None:
            raise RankGroupError(f"rank {rank} entering {kind}: group broken: {self._broken}")
        assert self._turn == rank, (rank, self._turn)
        self._entered[rank] = (kind, payload)
        self._state[rank] = f"in {kind}()" if kind != "returned" else "returned"
        self._progress = time.monotonic()
        if rank + 1 < self.world:
            self._turn = rank + 1
            self._cv.notify_all()
            return
        kinds = [k for k, _ in self._entered]
        if len(set(kinds)) != 1:
            self._break("the ranks are not in the same collective")
            raise RankGroupError(f"rank {rank}: group broken: {self._broken}")
        if kind != "returned":
            try:
                self._perform(kind, [p for _, p in self._entered])
            except RankGroupError as e:
                self._break(str(e))
                raise RankGroupError(f"rank {rank}: group broken: {self._broken}") from None
        self._entered = [None] * self.world
        self._phase += 1
        self._turn = 0
        self._cv.notify_all()

    def _collective(self, rank, kind, payload):
        with self._cv:
            phase = self._phase
            self._arrive(rank, kind, payload)
            self._await(rank, lambda: self._phase > phase and self._turn == rank, f"the other ranks in {kind}()")
            self._state[rank] = "running"
            res, self._results[rank] = self._results[rank], None
            if rank + 1 == self.world:
                self._progress = time.monotonic()
            return res

    # ------------------------------------------------------------------------------------------------ collectives
    def _perform(self, kind, payloads):
        W = self.world
        _sync()
        if kind == "wait":
            sigs = [[p.sig for p in pend] for pend in payloads]
            for r in range(1, W):
                if sigs[r] != sigs[0]:
                    raise RankGroupError(f"ranks 0 and {r} launched different ranges: {sigs[0]} != {sigs[r]}")
            for r, pend in enumerate(payloads):
                for p in pend:
                    diff = _bits(p.view) != _bits(p.snapshot)
                    if bool(diff.any()):
                        i = int(diff.nonzero()[0, 0])
                        off, n, _, _ = p.sig
                        raise RankGroupError(
                            f"rank {r}: range [{off}, {off + n}) was written after its all-reduce was launched: "
                            f"{int(diff.sum())} elements differ, first at offset {off + i}")
            order = self.reduce_order()
            assert sorted(order) == list(range(W)), order
            reduced = []
            for j, sig in enumerate(sigs[0]):
                views = [payloads[r][j].view for r in range(W)]
                inputs = [v.clone() for v in views] if self.keep_inputs else None
                total = views[order[0]].float().clone()
                for r in order[1:]:
                    total += views[r].float()
                for v in views:
                    v.copy_(total.to(v.dtype))
                reduced.append({"sig": sig, "inputs": inputs, "result": views[0].clone()})
            self.last_reduce = reduced
            self.trace.append({"kind": kind, "ranges": sigs[0]})
            _sync()
            return
        if any(m._pending for m in self._members):
            raise RankGroupError(f"{kind}() with all-reduces launched but not waited for")
        if kind == "all_gather":
            counts = {c for _, c in payloads}
            if len(counts) != 1:
                raise RankGroupError(f"ranks disagree on the all-gather slice size: {sorted(counts)}")
            c = counts.pop()
            for r, (src, _) in enumerate(payloads):
                for q, (dst, _) in enumerate(payloads):
                    if q != r:
                        dst[r * c:(r + 1) * c].copy_(src[r * c:(r + 1) * c])
            self.trace.append({"kind": kind, "ranges": [(0, W * c, payloads[0][0].dtype, True)]})
        elif kind == "max_over_ranks":
            m = max(payloads)
            for r in range(W):
                self._results[r] = m
            self.trace.append({"kind": kind, "ranges": []})
        elif kind == "barrier":
            self.trace.append({"kind": kind, "ranges": []})
        else:
            raise AssertionError(kind)
        _sync()
