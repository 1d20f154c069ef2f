"""Step assembly — the drop-in boundary.  Mirrors src/model_fns.py (dalle_model_fn) and src/model_fns_tf.py
(vae_model_fn): same signature ``model_fn(features, labels, mode, params)``, same parameter keys, PREDICT raises
NotImplementedError (src/model_fns.py:135-136, src/model_fns_tf.py:29-30).

Where the reference returns a TPUEstimatorSpec wiring TF ops, these return a ``StepSpec``: the model_fn is called
ONCE (like the Estimator's graph build) and ``spec.train_op(features, labels)`` runs one optimisation step on a
batch (host or device tensors), returning the device scalar with the global-mean loss.  One process per GPU: each
rank passes ITS shard of the global batch (rows rank*B/N..., the reference's "batch_dim:data" layout).
"""
import torch

from . import lib as L
from . import ops
from .dalle_engine import DalleEngine
from .dist import DataParallel
from .optimizers import OptimizerConfig
from .utils import latest_checkpoint, load_checkpoint, local_path, parse_mesh, print_n_params
from .vae_engine import VaeEngine

TRAIN, EVAL, PREDICT = "train", "eval", "predict"   # tf.estimator.ModeKeys values


def mode_to_str(mode):
    """src/utils/utils.py:29-37."""
    if mode in (TRAIN, EVAL, PREDICT):
        return mode
    raise ValueError(f"Invalid mode {mode}")


class StepSpec:
    """What model_fn hands back to the training loop (stands in for TPUEstimatorSpec)."""

    def __init__(self, mode, engine, train_op=None, eval_op=None, state_fn=None, load_fn=None, dp=None, extra=None):
        self.mode = mode
        self.engine = engine
        self.train_op = train_op      # (features, labels) -> device scalar loss (global mean)
        self.eval_op = eval_op        # (features, labels) -> device scalar loss
        self.state_fn = state_fn      # () -> checkpoint dict
        self.load_fn = load_fn        # (dict) -> None
        self.dp = dp
        self.global_step = 0
        self.extra = extra or {}
        self.loss = None              # device scalar of the last step (read it only when logging: it syncs)


def _to_device(t, dtype, device):
    """Host -> device copy of a step's inputs (pinned host tensors make it asynchronous)."""
    if not torch.is_tensor(t):
        t = torch.as_tensor(t)
    if t.device.type != "cuda":
        t = t.to(device, non_blocking=True)
    if t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()


# =====================================================================================================================
# DALL-E
# =====================================================================================================================
def load_vae_model(params, device):
    """src/model_fns.py:35-52: build the (frozen) VAE from params["vae_params"] and locate its checkpoint."""
    vae_params = params.get("vae_params")
    assert vae_params is not None, "vae model config must be supplied"        # model_fns.py:38
    D = params["dataset"]["image_size"]
    convblocks = vae_params.get("convblocks") or [(3, 64), (3, 128), (3, 256)]
    vae = VaeEngine(num_tokens=vae_params["num_tokens"], image_size=D, convblocks=convblocks,
                    input_channels=vae_params.get("input_channels") or 3,
                    use_bf16=bool(vae_params.get("use_bf16")),   # bf16 -> wgmma implicit-GEMM convolutions
                    stack_factor=vae_params.get("stack_factor") or 1, device=device)
    ckpt = params.get("vae_checkpoint_path")
    if ckpt is None:
        ckpt = latest_checkpoint(vae_params["model_path"]) if vae_params.get("model_path") else None
    return vae, ckpt


def dalle_model_fn(features, labels, mode, params):
    """src/model_fns.py:55-236.  features: images f32 [B,H,W,C] in [-1,1] (NHWC); labels: caption ids i32
    [B, text_seq_len].  (The reference's own comment has them swapped; the code uses them this way.)"""
    mode_str = mode_to_str(mode)
    if mode == PREDICT:
        raise NotImplementedError                                             # model_fns.py:135-136
    L.require_device()
    dp = params.get("_dp") or DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    mesh, _ = parse_mesh(params["mesh_shape"], params["layout"])            # model_fns.py:81-82
    if mesh.get("model", 1) != 1 and dp.rank == 0:
        print(f"note: mesh axis model:{mesh['model']} has no layout rule in the reference either (pure replication); "
              f"this engine runs data:{dp.world} and does not duplicate work")

    # ---- frozen VAE tokenizer (model_fns.py:63-77)
    vae, vae_ckpt = load_vae_model(params, device)
    if vae_ckpt is not None:
        state = load_checkpoint(local_path(vae_ckpt))
        vae.load_params({k[len("vae/"):]: v for k, v in state.items() if k.startswith("vae/")})
    elif params.get("vae_random_init"):
        vae.init_params(seed=params.get("vae_seed") or 0)   # extension key: throughput runs without a checkpoint
    else:
        raise AssertionError("pretrained vae needed for training")              # model_fns.py:41
    image_seq_len = vae.image_seq_len                                           # model_fns.py:68
    global_batch = params[f"{mode_str}_batch_size"]                             # model_fns.py:69
    _, local_batch = dp.shard(global_batch)

    model = DalleEngine(n_embd=params["n_embd"], n_layers=params["n_layers"], n_heads=params["n_heads"],
                        text_vocab_size=params["text_vocab_size"], image_vocab_size=params["image_vocab_size"],
                        text_seq_len=params["text_seq_len"], image_seq_len=image_seq_len, device=device,
                        recompute_grad=bool(params.get("recompute_grad")) and mode == TRAIN,   # models.py:342
                        # extension key: shard fp32 master + Adam slots across the data-parallel ranks (ZeRO-1) —
                        # what lets the d = 4096 configuration fit 80 GB GPUs in pure data parallelism
                        zero=dp if (params.get("optimizer_state_sharding") and dp.enabled) else None)
    if params["bf_16"] is False and dp.rank == 0:
        print("note: bf_16=false — the engine still runs activations and matmul operands in bf16 with fp32 "
              "accumulation, fp32 master weights / optimiser state (there is no fp32 tensor-core path yet)")
    if vae.K > params["image_vocab_size"]:
        raise ValueError(f"vae num_tokens {vae.K} exceeds image_vocab_size {params['image_vocab_size']}: image ids "
                         "would index past the embedding table (SURVEY.md Appendix C.4)")
    model.init_params(seed=params.get("seed") or 0)
    if dp.rank == 0:
        print_n_params(model.n_params())                                        # get_graph_info, model_fns.py:186

    S = model.S
    tokens = torch.empty(local_batch, S, dtype=torch.int32, device=device)
    total_tokens_global = global_batch * S
    # micro-batching (model_fns.py:144-166): tokens_per_mb_per_replica -> number of sequential micro-batches
    tpmb = params.get("tokens_per_mb_per_replica")
    num_microbatches = 1
    if mode == TRAIN and tpmb:
        seqs_per_mb = max(1, int(tpmb) // S)
        num_microbatches = max(1, -(-local_batch // seqs_per_mb))
        while local_batch % num_microbatches:
            num_microbatches += 1
    params["num_microbatches"] = num_microbatches                               # model_fns.py:154
    opt = OptimizerConfig(params) if mode == TRAIN else None
    spec = StepSpec(mode, model, dp=dp, extra={"vae": vae})

    def assemble(features, labels):
        img = _to_device(features, torch.float32, device).view(local_batch, vae.img_H, vae.img_W, vae.img_C)
        text = _to_device(labels, torch.int32, device).view(local_batch, params["text_seq_len"])
        img_ids = vae.encode_tokens(img)                                        # model_fns.py:72-77
        ops.assemble_tokens(text, img_ids, tokens, model.text_vocab_size)       # model_fns.py:117-122
        return tokens

    def loss_value():
        # sum of per-token losses over all ranks (all-reduced with the gradients) / global token count
        return model.grads[model.aux_off:model.aux_off + 1]

    dp.hint_tokens_per_gpu(local_batch * S)

    def train_op(features, labels):
        toks = assemble(features, labels)
        model.zero_grads()
        mb = local_batch // num_microbatches
        hook = dp.make_bucket_hook(model.grads)
        for i in range(num_microbatches):
            model.forward(toks[i * mb:(i + 1) * mb])
            last = i == num_microbatches - 1
            if last:
                dp.begin_overlap()
            # loss = mean over the GLOBAL batch (models.py:353-354): every rank back-props local_sum / (B*S) and the
            # all-reduce SUMs the shard partials (mtf semantics, SURVEY.md §8e)
            model.backward(1.0 / total_tokens_global, on_bucket_ready=hook if last else None)
        dp.wait()
        lr = opt.learning_rate(spec.global_step)                                # step counter before the increment
        model.optimizer_step(lr, beta1=opt.beta_1, beta2=opt.beta_2, eps=opt.epsilon,
                             weight_decay=opt.weight_decay, clip=opt.gradient_clipping)
        spec.global_step += 1                                                   # model_fns.py:201
        spec.lr = lr
        spec.loss_sum = loss_value()
        spec.loss_scale = 1.0 / total_tokens_global
        return spec.loss_sum

    def eval_op(features, labels):
        toks = assemble(features, labels)
        acc = torch.zeros(1, dtype=torch.float32, device=device)
        model.forward(toks, loss_accum=acc)
        dp.all_reduce_now(acc)
        spec.loss_sum, spec.loss_scale = acc, 1.0 / total_tokens_global
        return acc

    def state_fn():
        st = {k: v for k, v in model.export_params().items()}
        if model.zero is not None:      # sharded Adam slots are not gathered into rank 0's checkpoint (throughput config)
            st["global_step"] = spec.global_step
            return st
        st.update({k + "/adam_m": v for k, v in model.export_params(model.adam_m).items()})   # optimizers.py:139
        st.update({k + "/adam_v": v for k, v in model.export_params(model.adam_v).items()})   # optimizers.py:147
        st["global_step"] = spec.global_step
        return st

    def load_fn(st):
        names = [k for k in st if not k.endswith("/adam_m") and not k.endswith("/adam_v") and k != "global_step"]
        model.load_params({k: st[k] for k in names})                                # master + bf16 shadow
        for suffix, flat in (("/adam_m", model.adam_m), ("/adam_v", model.adam_v)):
            model.load_flat(flat, {k: st[k + suffix] for k in names})
        spec.global_step = int(st.get("global_step", 0))

    spec.train_op = train_op if mode == TRAIN else None
    spec.eval_op = eval_op
    spec.state_fn, spec.load_fn = state_fn, load_fn
    spec.tokens_per_step = total_tokens_global
    spec.assemble = assemble
    return spec


# =====================================================================================================================
# discrete VAE
# =====================================================================================================================
def vae_temperature(step, params):
    """src/model_fns_tf.py:40-45."""
    if params.get("temp_anneal_steps"):
        frac = min(step / params["temp_anneal_steps"], 1.0)
        return params["temp_start"] - frac * (params["temp_start"] - params["temp"])
    t = params.get("temp")
    return 1.0 if t is None else t


def vae_model_fn(features, labels, mode, params):
    """src/model_fns_tf.py:9-114.  features = labels = images f32 [B,H,W,C] in [-1,1]."""
    mode_str = mode_to_str(mode)
    if mode == PREDICT:
        raise NotImplementedError                                             # model_fns_tf.py:29-30
    L.require_device()
    dp = params.get("_dp") or DataParallel().init()
    device = torch.device("cuda", torch.cuda.current_device())
    H = params["dataset"]["image_size"]                                       # model_fns_tf.py:13
    global_batch = params[f"{mode_str}_batch_size"]
    _, local_batch = dp.shard(global_batch)
    model = VaeEngine(num_tokens=params["num_tokens"], image_size=H,
                      convblocks=params.get("convblocks") or [(3, 64), (3, 128), (3, 256)],
                      input_channels=params.get("input_channels") or 3,
                      recompute_grad=bool(params.get("recompute_grad")), use_bf16=bool(params.get("use_bf16")),
                      stack_factor=params.get("stack_factor") or 1, device=device)
    model.init_params(seed=params.get("seed") or 0)
    if dp.rank == 0:
        print_n_params(model.n_params())
        if params.get("recompute_grad"):
            print("note: recompute_grad=true (src/vae_tf/models.py:8-43) — the engine keeps the residual-pair "
                  "activations instead of recomputing them (they fit in HBM many times over); gradients are identical")
    tg = params.get("train_gumbel_hard")
    eg = params.get("eval_gumbel_hard")
    train_gumbel = True if tg is None else tg                                 # model_fns_tf.py:32
    eval_gumbel = True if eg is None else eg                                  # model_fns_tf.py:33
    hard = train_gumbel if mode == TRAIN else eval_gumbel
    rows = local_batch * model.hw * model.hw
    noise = torch.empty(rows, model.K, dtype=torch.float32, device=device)
    gen = torch.Generator(device=device).manual_seed(1234 + dp.rank)
    spec = StepSpec(mode, model, dp=dp)
    n_global = global_batch * H * H * model.img_C

    def draw_noise():
        # tf.random_uniform(minval=1e-9, maxval=1.) (src/vae_tf/layers.py:8-13); RNG stream is ours (SURVEY §7)
        noise.uniform_(1e-9, 1.0, generator=gen)
        return noise

    def run(features, train):
        img = _to_device(features, torch.float32, device).view(local_batch, H, H, model.img_C)
        temp = vae_temperature(spec.global_step, params)
        u = params.get("_gumbel_u")
        u = draw_noise() if u is None else u
        model.zero_grads()
        recon = model.forward(img, u, temp, hard)       # adds sum((img-out)^2)/local_numel into the aux slot
        return recon

    def train_op(features, labels=None):
        run(features, True)
        # CrossShardOptimizer: cross-replica MEAN of the gradients (model_fns_tf.py:61) = bucketed SUM all-reduce that
        # overlaps with the rest of backward (decoder, codebook, encoder ranges), then 1/N inside the Adam kernel
        dp.begin_overlap()
        model.backward(on_bucket_ready=dp.make_bucket_hook(model.grads))
        dp.wait()
        spec.global_step += 1
        model.optimizer_step(params["lr"], spec.global_step, grad_scale=1.0 / dp.world)   # model_fns_tf.py:58-60
        spec.loss_sum = model.grads[model.aux_off:model.aux_off + 1]
        spec.loss_scale = 1.0 / dp.world    # each rank's aux slot holds its local mean; the SUM over ranks / N
        return spec.loss_sum

    def eval_op(features, labels=None):
        run(features, False)
        acc = model.grads[model.aux_off:model.aux_off + 1].clone()
        dp.all_reduce_now(acc)
        spec.loss_sum, spec.loss_scale = acc, 1.0 / dp.world
        return acc

    def state_fn():
        st = {"vae/" + k: v for k, v in model.export_params().items()}
        st.update({"vae/" + k + "/Adam": v for k, v in model.export_params(model.adam_m).items()})
        st.update({"vae/" + k + "/Adam_1": v for k, v in model.export_params(model.adam_v).items()})
        st["global_step"] = spec.global_step
        return st

    def load_fn(st):
        # master weights (+ the bf16 shadow / split codebook derived from them), then the Adam slots straight into
        # their flat buffers: the compute copies must never be refreshed from anything but the weights
        model.load_params({k[len("vae/"):]: v for k, v in st.items()
                           if k.startswith("vae/") and not k.endswith("/Adam") and not k.endswith("/Adam_1")})
        for suffix, flat in (("/Adam", model.adam_m), ("/Adam_1", model.adam_v)):
            model.load_flat(flat, {k[len("vae/"):-len(suffix)]: v for k, v in st.items() if k.endswith(suffix)})
        spec.global_step = int(st.get("global_step", 0))

    spec.train_op = train_op if mode == TRAIN else None
    spec.eval_op = eval_op
    spec.state_fn, spec.load_fn = state_fn, load_fn
    spec.images_per_step = global_batch
    spec.n_global = n_global
    return spec
