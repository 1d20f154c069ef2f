"""Data parallelism: one process per GPU, NCCL over NVLink / NVSwitch, bucketed gradient all-reduce that overlaps
with the rest of backward.

The reference's only parallelism is the layout rule "batch_dim:data" (configs/dalle_example.json:20-21): mtf lowers
every weight gradient to an all-reduce SUM across the `data` mesh axis (src/optimizers.py:34, src/model_fns.py:189),
one collective per variable and no overlap control.  Here the gradients live in ONE flat fp32 buffer in forward order;
backward completes it from the tail, and each finished contiguous range ("bucket": the vocabulary projection, then
one transformer layer at a time, then the embeddings) is all-reduced asynchronously on NCCL's own stream while the
earlier layers are still back-propagating.  The loss scalar rides in the first bucket.  The optimiser waits on the
handles; clip-by-global-norm is computed after the reduce, identically on every rank (src/optimizers.py:101-102), so
there is no second collective.
"""
import ctypes
import os

import torch
import torch.distributed as dist


def _libnccl_path():
    """The libnccl.so.2 that ships next to torch (nvidia-nccl wheel); None -> the dynamic loader's default."""
    try:
        import nvidia.nccl
        p = os.path.join(list(nvidia.nccl.__path__)[0], "lib", "libnccl.so.2")
        return p if os.path.exists(p) else None
    except Exception:  # noqa: BLE001
        return None


class DataParallel:
    """Rank bookkeeping + the gradient collectives.

    Data plane on a GPU box: the communicator of libdalle_b200.so (db200_comm_*: ncclCommInitRankConfig, a dedicated
    high-priority stream, event hand-offs, CTA cap) — torch.distributed is only the side channel that ships the NCCL
    unique id and provides barrier / scalar reductions for logging (control plane, "gloo" for CPU tensors).
    Without a GPU (the world-size-2 CPU tests of the bucket logic) the collectives go through torch.distributed/gloo.
    """

    # CTAs NCCL may occupy while the persistent one-CTA-per-SM wgmma grids of backward are running (0 = NCCL's default).
    # The same number of SMs is taken out of the persistent kernels' grids (db200_set_reserved_sms), so that the two fit
    # side by side; the overlapped all-reduce only has to move 287 MB during ~10 ms of backward: four CTAs are plenty.
    MAX_CTAS = int(os.environ.get("DB200_NCCL_MAX_CTAS", "4"))
    # A second communicator without that cap carries the collectives that run when no compute is left to overlap with:
    # the last gradient bucket ([wte | wpe], finished by the final kernel of backward), the ZeRO-1 parameter
    # all-gather and the eval-loss reduction.  -1 disables it (everything on the capped communicator).
    TAIL_CTAS = int(os.environ.get("DB200_NCCL_TAIL_CTAS", "0"))

    def __init__(self):
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.handles = []
        self.enabled = self.world > 1
        self.comm = None          # db200_comm* (ctypes void pointer) when the C-ABI communicator is in use
        self.comm_tail = None     # uncapped communicator for the exposed collectives (None: use self.comm)
        self._reserve = 0         # SMs the persistent kernels leave free while bucket all-reduces may be in flight
        self.registered = False

    def init(self, backend=None):
        cuda = torch.cuda.is_available()
        if cuda:
            torch.cuda.set_device(self.local_rank)
        if self.enabled and not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            # control plane: gloo for host tensors; torch's own NCCL group is declared for CUDA tensors but stays
            # uninitialised unless somebody uses it (the data plane below does not)
            backend = backend or ("cpu:gloo,cuda:nccl" if cuda else "gloo")
            dist.init_process_group(backend=backend, rank=self.rank, world_size=self.world)
        # the NCCL communicators are created at first use (every rank reaches it at the same point of its first step),
        # after the model function had the chance to size the CTA cap for its step (hint_tokens_per_gpu)
        self._want_comm = bool(self.enabled and cuda and os.environ.get("DB200_DP_BACKEND", "cabi") == "cabi")
        return self

    def hint_tokens_per_gpu(self, tokens):
        """Sizes the CTA cap of the overlapped communicator (unless DB200_NCCL_MAX_CTAS is set): the gradient volume
        is fixed by the model, the time to hide it behind shrinks with the per-GPU batch.  A long backward (weak
        scaling, >= 16 k tokens per GPU) hides 287 MB behind 4 CTAs; a short one (strong scaling) needs more."""
        if self.comm is None and "DB200_NCCL_MAX_CTAS" not in os.environ:
            self.MAX_CTAS = 4 if tokens >= 16384 else 16

    def _ensure_comm(self):
        if getattr(self, "_want_comm", False) and self.comm is None:
            self._create_comm()

    def _create_comm(self):
        from . import lib as L
        lib = L.load()
        path = _libnccl_path()
        L.check(lib.db200_comm_load_nccl(path.encode() if path else None), "comm_load_nccl")

        def create(max_ctas):
            uid = ctypes.create_string_buffer(128)
            if self.rank == 0:
                L.check(lib.db200_comm_unique_id(uid, 128), "comm_unique_id")
            box = [uid.raw]
            dist.broadcast_object_list(box, src=0)            # side channel (gloo): 128 bytes
            uid = ctypes.create_string_buffer(box[0], 128)
            comm = ctypes.c_void_p()
            L.check(lib.db200_comm_create(torch.cuda.current_device(), self.rank, self.world, uid, max_ctas,
                                          ctypes.byref(comm)), "comm_create")
            return comm

        self.comm = create(self.MAX_CTAS)
        self._reserve = self.MAX_CTAS if (self.MAX_CTAS > 0 and os.environ.get("DB200_RESERVE_SMS", "1") != "0") else 0
        if self.TAIL_CTAS >= 0 and self.TAIL_CTAS != self.MAX_CTAS:
            self.comm_tail = create(self.TAIL_CTAS)

    def shard(self, global_batch):
        """Rows [rank*B/N, (rank+1)*B/N) of the global batch (SURVEY.md §8e)."""
        if global_batch % self.world != 0:
            raise ValueError(f"global batch {global_batch} is not divisible by the data-parallel size {self.world}")
        per = global_batch // self.world
        return self.rank * per, per

    # --- gradient buckets ------------------------------------------------------------------------------
    def _exposed_comm(self):
        return self.comm_tail if self.comm_tail is not None else self.comm

    def _launch(self, t, exposed=False):
        """Asynchronous in-place SUM all-reduce of a contiguous fp32 / bf16 tensor (a slice of a flat buffer).
        exposed: nothing is left to overlap with — use the communicator without the CTA cap."""
        self._ensure_comm()
        if self.comm is not None:
            from . import lib as L
            dt = {torch.float32: 0, torch.bfloat16: 1}[t.dtype]
            comm = self._exposed_comm() if exposed else self.comm
            L.check(L.load().db200_bucket_allreduce_launch(comm, L.stream_ptr(), t.data_ptr(), t.numel(), dt),
                    "bucket_allreduce_launch")
        else:
            self.handles.append(dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=True))

    def register(self, flat):
        """ncclCommRegister of a long-lived flat buffer (best effort; once)."""
        self._ensure_comm()
        if self.comm is not None and not self.registered:
            from . import lib as L
            ok = ctypes.c_int(0)
            L.check(L.load().db200_comm_register(self.comm, flat.data_ptr(), flat.numel() * flat.element_size(),
                                                 ctypes.byref(ok)), "comm_register")
            self.registered = True

    def begin_overlap(self):
        """Call right before the backward pass whose buckets are all-reduced on the fly: from here until wait() the
        persistent kernels size their grids to (SM count - CTA cap), so the collective's CTAs and theirs fit side by
        side (grids are sized on the host at launch time; forward / optimizer kernels keep all SMs)."""
        self._ensure_comm()
        if self.comm is not None and self._reserve:
            from . import lib as L
            L.check(L.load().db200_set_reserved_sms(self._reserve), "set_reserved_sms")

    def make_bucket_hook(self, flat):
        """Returns on_bucket_ready(start, end) for the engines' backward: async all-reduce(SUM) of flat[start:end],
        ordered after the kernels already enqueued on the current stream, overlapping with whatever comes next."""
        if not self.enabled:
            return None
        self.register(flat)

        def hook(start, end):
            end = min(end, flat.numel())
            # the flat buffers are laid out in forward order and backward finalises them from the tail: the range that
            # starts at offset 0 is the last one, launched after the final kernel of backward
            self._launch(flat[start:end], exposed=(start == 0))

        return hook

    def all_reduce_now(self, t):
        if self.enabled:
            self._launch(t, exposed=True)
            self.wait()
        return t

    def all_gather_inplace(self, buf, count_per_rank):
        """In-place all-gather of equal slices: rank r's data is buf[r*count : (r+1)*count] (ZeRO-1 parameter refresh);
        the current stream waits for it."""
        if not self.enabled:
            return buf
        mine = buf[self.rank * count_per_rank:(self.rank + 1) * count_per_rank]
        self._ensure_comm()
        if self.comm is not None:
            from . import lib as L
            dt = {torch.float32: 0, torch.bfloat16: 1}[buf.dtype]
            L.check(L.load().db200_bucket_all_gather_launch(self._exposed_comm(), L.stream_ptr(), mine.data_ptr(),
                                                            buf.data_ptr(), count_per_rank, dt), "bucket_all_gather_launch")
            self.wait()
        else:
            dist.all_gather_into_tensor(buf[:self.world * count_per_rank], mine.clone())
        return buf

    def wait(self):
        """Make the current stream wait for every outstanding bucket (on the device; no host block with NCCL)."""
        if self.comm is not None:
            from . import lib as L
            L.check(L.load().db200_bucket_allreduce_wait(self.comm, L.stream_ptr()), "bucket_allreduce_wait")
            if self.comm_tail is not None:
                L.check(L.load().db200_bucket_allreduce_wait(self.comm_tail, L.stream_ptr()), "bucket_allreduce_wait")
            if self._reserve:
                L.check(L.load().db200_set_reserved_sms(0), "set_reserved_sms")
        for h in self.handles:
            h.wait()
        self.handles = []

    def barrier(self):
        if self.enabled:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            dist.barrier()

    def max_over_ranks(self, value):
        if not self.enabled:
            return value
        t = torch.tensor([value], dtype=torch.float64)       # host tensor: control plane (gloo)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def shutdown(self):
        if self.comm is not None:
            from . import lib as L
            torch.cuda.synchronize()
            if self.comm_tail is not None:
                L.load().db200_comm_destroy(self.comm_tail)
                self.comm_tail = None
            L.load().db200_comm_destroy(self.comm)
            self.comm = None
        if self.enabled and dist.is_initialized():
            dist.destroy_process_group()
