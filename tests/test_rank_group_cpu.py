"""The in-process rank group of tests/rank_group.py on CPU tensors: the reduction it performs, the all-gather, and the
violations it must report (a write after launch, ranks that launched different ranges, a skipped collective, a rank
that raises) without leaving a thread behind."""
import threading
import time

import pytest
import torch

from rank_group import RankGroup, RankGroupError

F32 = torch.float32


def _rank_threads():
    return [t for t in threading.enumerate() if t.name.startswith("rank-")]


def _bits(t):
    return t.view(torch.int32)


def test_sum_is_in_rank_order_bitwise_at_three_ranks():
    """1 + 2^-24 rounds to 1 (ties to even), so ((1 + u) + u) = 1 while 1 + (u + u) = 1 + 2^-23: the association shows.
    Random rows must equal ((x0 + x1) + x2) bitwise on every rank, and the ranges outside the launched ones stay."""
    W, n = 3, 1000
    u = 2.0 ** -24
    g = torch.Generator().manual_seed(0)
    data = [torch.randn(n, generator=g) * 10 ** torch.randint(-3, 4, (n,), generator=g) for _ in range(W)]
    data[0][0], data[1][0], data[2][0] = 1.0, u, u
    expect = ((data[0] + data[1]) + data[2])
    assert expect[0].item() == 1.0 and (data[0][0] + (data[1][0] + data[2][0])).item() != 1.0
    group = RankGroup(W)
    bufs = [torch.cat([d, torch.full((64,), float(r))]) for r, d in enumerate(data)]
    order = []

    def fn(rank, dp):
        order.append(("start", rank))
        hook = dp.make_bucket_hook(bufs[rank])
        hook(500, n + 64)                 # clipped to the buffer's end, as the engines' first range is
        hook(0, 500)
        dp.wait()
        order.append(("after", rank))
        return dp.max_over_ranks(rank * 1.5)

    assert group.run(fn) == [3.0] * W
    assert order == [("start", 0), ("start", 1), ("start", 2), ("after", 0), ("after", 1), ("after", 2)]
    full = torch.cat([expect, torch.full((64,), 0.0 + 1.0 + 2.0)])
    for r in range(W):
        assert torch.equal(_bits(bufs[r]), _bits(full)), r
    assert [e["kind"] for e in group.trace] == ["wait", "max_over_ranks"]
    assert group.trace[0]["ranges"] == [(500, n + 64 - 500, F32, False), (0, 500, F32, True)]
    red = group.last_reduce
    assert [x["sig"] for x in red] == group.trace[0]["ranges"]
    assert torch.equal(red[1]["inputs"][2], data[2][:500]) and torch.equal(red[1]["result"], expect[:500])
    assert not _rank_threads()


def test_reduce_order_is_what_the_sum_follows():
    W = 3
    u = 2.0 ** -24
    group = RankGroup(W)
    group.reduce_order = lambda: [2, 1, 0]
    bufs = [torch.tensor([1.0 if r == 0 else u]) for r in range(W)]

    def fn(rank, dp):
        dp.all_reduce_now(bufs[rank])

    group.run(fn)
    assert bufs[0].item() == 1.0 + 2 * u


def test_all_gather_copies_slice_r_of_rank_r_everywhere():
    W, c = 3, 5
    bufs = [torch.full((W * c + 2,), -1.0) for _ in range(W)]
    for r in range(W):
        bufs[r][r * c:(r + 1) * c] = torch.arange(c, dtype=F32) + 10 * r
    tail = [b[W * c:].clone() for b in bufs]
    group = RankGroup(W)
    group.run(lambda rank, dp: dp.all_gather_inplace(bufs[rank], c))
    expect = torch.cat([torch.arange(c, dtype=F32) + 10 * r for r in range(W)])
    for r in range(W):
        assert torch.equal(bufs[r][:W * c], expect) and torch.equal(bufs[r][W * c:], tail[r])
    assert group.trace[-1]["kind"] == "all_gather"


def test_a_write_after_launch_is_reported():
    W = 2
    bufs = [torch.ones(128) for _ in range(W)]

    def fn(rank, dp):
        hook = dp.make_bucket_hook(bufs[rank])
        hook(64, 128)
        if rank == 1:
            bufs[rank][100] += 1.0            # the range is already being reduced
        hook(0, 64)
        dp.wait()

    with pytest.raises(RankGroupError, match=r"rank 1: range \[64, 128\) was written after .* first at offset 100"):
        RankGroup(W).run(fn)
    assert not _rank_threads()


def test_different_pending_lists_are_reported():
    W = 3
    bufs = [torch.ones(128) for _ in range(W)]

    def fn(rank, dp):
        hook = dp.make_bucket_hook(bufs[rank])
        hook(64, 128 if rank != 2 else 120)
        hook(0, 64)
        dp.wait()

    with pytest.raises(RankGroupError, match="ranks 0 and 2 launched different ranges"):
        RankGroup(W).run(fn)
    assert not _rank_threads()


@pytest.mark.parametrize("skipper", [0, 1])
def test_a_skipped_collective_fails_within_the_timeout(skipper):
    """One rank returns without the all-reduce its peer waits in: RankGroupError naming what each rank is in, well
    within the timeout, and no rank thread outlives run()."""
    W, timeout = 2, 20
    bufs = [torch.ones(8) for _ in range(W)]

    def fn(rank, dp):
        if rank != skipper:
            dp.all_reduce_now(bufs[rank])

    t0 = time.monotonic()
    with pytest.raises(RankGroupError, match=r"not in the same collective.*(in wait\(\).*returned|returned.*in wait)"):
        RankGroup(W, timeout_s=timeout).run(fn)
    assert time.monotonic() - t0 < timeout
    assert not _rank_threads()


def test_a_rendezvous_that_never_completes_times_out():
    """A rank blocked outside any collective: the rank waiting for it gives up after timeout_s."""
    def fn(rank, dp):
        if rank == 0:
            dp.barrier()                       # waits for rank 1, which is blocked below
        else:
            time.sleep(3)

    t0 = time.monotonic()
    group = RankGroup(2, timeout_s=1)
    with pytest.raises(RankGroupError, match=r"no progress within 1 s.*rank 0: in barrier\(\); rank 1: running"):
        group.run(fn)
    assert time.monotonic() - t0 < 10
    assert not _rank_threads()


def test_an_exception_in_one_rank_reaches_the_caller():
    W = 3
    seen = []

    def fn(rank, dp):
        seen.append(rank)
        if rank == 1:
            raise ValueError("boom in rank 1")
        dp.barrier()

    with pytest.raises(ValueError, match="boom in rank 1"):
        RankGroup(W).run(fn)
    assert seen == [0, 1]                      # rank 2 never started: the group broke first
    assert not _rank_threads()
