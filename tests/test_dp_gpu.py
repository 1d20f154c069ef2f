"""Data-parallel equivalence on real GPUs (needs >= 2 devices; skipped otherwise):
an N-rank step on batch shards must equal a 1-rank step on the concatenated batch — mtf semantics: the loss is the
mean over the GLOBAL batch and weight gradients are SUMMED over the `data` mesh axis (SURVEY.md §4, §8e)."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    dev = torch.device("cuda", rank)
    args = (256, 2, 2, 500, 64, 24, 40)
    g = torch.Generator().manual_seed(0)
    global_tokens = torch.randint(0, 500 + 64, (4, 64), generator=g, dtype=torch.int32)
    T = global_tokens.numel()
    # N-rank run on shards
    eng = DalleEngine(*args, device=dev)
    eng.init_params(seed=7)
    start, per = dp.shard(4)
    eng.zero_grads()
    eng.forward(global_tokens[start:start + per].to(dev))
    eng.backward(1.0 / T, on_bucket_ready=dp.make_bucket_hook(eng.grads))
    dp.wait()
    g_dp = eng.grads[:eng.n_params_padded].clone()     # the optimiser step zeroes the buffer behind itself
    eng.optimizer_step(1e-3)
    torch.cuda.synchronize()
    loss_dp = eng.grads[eng.aux_off].item() / T
    # 1-rank reference on the concatenated batch (same device, no communication)
    ref = DalleEngine(*args, device=dev)
    ref.init_params(seed=7)
    ref.zero_grads()
    ref.forward(global_tokens.to(dev))
    ref.backward(1.0 / T)
    g_ref = ref.grads[:ref.n_params_padded].clone()
    ref.optimizer_step(1e-3)
    torch.cuda.synchronize()
    loss_ref = ref.grads[ref.aux_off].item() / T
    n = eng.n_params_padded
    gerr = ((g_dp - g_ref).norm() / g_ref.norm()).item()
    perr = ((eng.master[:n] - ref.master[:n]).norm() / ref.master[:n].norm()).item()
    dp.barrier()
    out.put((rank, loss_dp, loss_ref, gerr, perr))
    dp.shutdown()


def test_two_rank_step_equals_single_rank_step_on_concatenated_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, loss_dp, loss_ref, gerr, perr in res:
        assert abs(loss_dp - loss_ref) / loss_ref < 1e-5, res       # loss = global mean on every rank
        assert gerr < 2e-3, res     # same math, different summation order (per-rank partial sums, fp32 atomics)
        assert perr < 1e-5, res
    assert abs(res[0][1] - res[1][1]) < 1e-7                        # ranks agree exactly after the all-reduce


def _zero_worker(rank, world, port, out):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init()
    dev = torch.device("cuda", rank)
    args = (256, 2, 2, 500, 64, 24, 40)
    g = torch.Generator().manual_seed(1)
    global_tokens = torch.randint(0, 500 + 64, (4, 64), generator=g, dtype=torch.int32)
    T = global_tokens.numel()
    start, per = dp.shard(4)
    engines = []
    for zero in (None, dp):      # replicated optimiser state vs ZeRO-1 (sharded master / m / v + all-gathered bf16)
        eng = DalleEngine(*args, device=dev, zero=zero)
        eng.init_params(seed=7)
        for step in range(3):
            eng.zero_grads()
            eng.forward(global_tokens[start:start + per].to(dev))
            eng.backward(1.0 / T, on_bucket_ready=dp.make_bucket_hook(eng.grads))
            dp.wait()
            eng.optimizer_step(2e-3)
        torch.cuda.synchronize()
        engines.append(eng)
    rep, z = engines
    n = rep.n_params_padded
    # same random stream -> same initial weights; after 3 steps the bf16 compute copies must agree up to the one
    # difference between the modes: ZeRO feeds LayerNorm gains / biases to the kernels bf16-rounded (reference policy)
    werr = ((z.shadow[:n].float() - rep.shadow[:n].float()).norm() / rep.shadow[:n].float().norm()).item()
    lo, hi = z.shard
    merr = ((z.master[:hi - lo] - rep.master[lo:hi]).norm() / rep.master[lo:hi].norm()).item()
    loss_rep, loss_z = rep.grads[rep.aux_off].item() / T, z.grads[z.aux_off].item() / T
    dp.barrier()
    out.put((rank, werr, merr, loss_rep, loss_z, int(z.master.numel()), int(rep.master.numel())))
    dp.shutdown()


def test_zero1_sharded_optimizer_matches_replicated_optimizer():
    """ZeRO-1 (optimiser-state sharding for the 12 B configuration, SURVEY.md §7): three steps with sharded
    master / Adam slots + in-place all-gather of the bf16 parameters == three steps with replicated state."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_zero_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, werr, merr, loss_rep, loss_z, nz, nrep in res:
        assert nz <= nrep // 2 + 64                                 # fp32 state really is halved
        # ZeRO-1 rebuilds the fp32 vector parameters (LayerNorm g / b, biases) from the all-gathered bf16 values — the
        # reference's own activation-dtype cast of every variable — so the two runs differ by bf16 roundings
        assert werr < 1.5e-2 and merr < 1.5e-2, res
        assert abs(loss_rep - loss_z) / loss_rep < 2e-3, res
