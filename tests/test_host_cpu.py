"""CPU tests of the host-side logic and of the C-ABI surface (no GPU: symbols load, nothing computes)."""
import ctypes
import json
import os
import re
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build_once():
    from dalle_mtf_b200 import lib as L
    if not os.path.exists(L.LIB_PATH):
        from dalle_mtf_b200.build import build
        build()
    return L


# ------------------------------------------------------------------------------------------------ C ABI
def test_library_exports_every_symbol_declared_in_the_header():
    L = _build_once()
    hdr = open(os.path.join(ROOT, "include", "dalle_b200.h")).read()
    declared = set(re.findall(r"\b(db200_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"db200_stream_t"}
    assert len(declared) >= 30
    lib = ctypes.CDLL(L.LIB_PATH)
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"symbols declared in include/dalle_b200.h but not exported: {missing}"
    L.load()
    assert L.MISSING_SYMBOLS == []
    assert set(L.EXPORTED_SYMBOLS) == declared, set(L.EXPORTED_SYMBOLS) ^ declared


def test_struct_mirrors_match_header_sizes(tmp_path):
    """The ctypes mirrors must have the size AND field offsets the C compiler gives the structs of the header."""
    import subprocess
    from dalle_mtf_b200.lib import ConvDesc, GemmEpilogue
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = {"db200_gemm_epilogue": [n for n, _ in GemmEpilogue._fields_],
              "db200_conv_desc": [n for n, _ in ConvDesc._fields_]}
    src = ["#include <stdio.h>", "#include <stddef.h>", '#include "dalle_b200.h"', "int main(void) {"]
    for st, names in fields.items():
        src.append(f'  printf("{st} %zu\\n", sizeof({st}));')
        for n in names:
            src.append(f'  printf("{st}.{n} %zu\\n", offsetof({st}, {n}));')
    src += ["  return 0;", "}"]
    c = tmp_path / "sizes.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for st, cls in (("db200_gemm_epilogue", GemmEpilogue), ("db200_conv_desc", ConvDesc)):
        assert ctypes.sizeof(cls) == int(out[st]), st
        for n, _ in cls._fields_:
            assert getattr(cls, n).offset == int(out[f"{st}.{n}"]), f"{st}.{n}"


def test_no_cpu_fallback_ops_raise_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dalle_mtf_b200 import lib as L, ops
    with pytest.raises(L.DB200Error):
        ops.sqnorm(torch.zeros(8), torch.zeros(1))
    with pytest.raises(L.DB200Error):
        from dalle_mtf_b200.dalle_engine import DalleEngine
        DalleEngine(256, 1, 2, 10, 4, 4, 4)


def test_last_error_and_version_are_callable_without_gpu():
    L = _build_once()
    lib = L.load()
    assert lib.db200_version() >= 100
    assert isinstance(lib.db200_last_error(), bytes)
    assert L.launch_count() >= 0


# ------------------------------------------------------------------------------------------------ config surface
def test_fetch_model_params_none_on_missing_and_get_default():
    from dalle_mtf_b200.utils import fetch_model_params
    p = fetch_model_params("dalle_example")
    assert p["n_embd"] == 512 and p.get("no_such_key", 7) == 7          # utils.py:13-17: .get still honours defaults
    assert p["no_such_key"] is None                                      # [] on a missing key reads None ...
    assert p.get("no_such_key", 7) is None                               # ... and (defaultdict) inserts it
    q = fetch_model_params(os.path.join(ROOT, "configs", "vae_example.json"))
    assert q["convblocks"] == [[3, 64], [3, 128], [3, 256]] and q["model_type"] == "vae"


def test_reference_config_values_are_preserved():
    ref = {
        "dalle_example": dict(n_embd=512, n_layers=6, n_heads=4, text_vocab_size=50258, image_vocab_size=512,
                              text_seq_len=256, train_batch_size=32, lr=0.001, bf_16=False, vae_model="vae_example",
                              mesh_shape="data:16,model:2", layout="batch_dim:data", iterations=500),
        "dalle_coco": dict(n_embd=1024, n_layers=12, n_heads=8, recompute_grad=True, lr=0.0001, train_batch_size=128),
        "vae_coco": dict(num_tokens=2048, use_bf16=True, temp_start=1, temp=0.05, temp_anneal_steps=25000,
                         train_gumbel_hard=False, eval_gumbel_hard=True, convblocks=[[2, 128], [3, 256], [5, 512]]),
        "vae_example": dict(num_tokens=512, dim=512, hidden_dim=64, lr=0.001, train_gumbel_hard=True),
    }
    for name, kv in ref.items():
        d = json.load(open(os.path.join(ROOT, "configs", name + ".json")))
        for k, v in kv.items():
            assert d[k] == v, (name, k)


def test_parse_mesh_accepts_data_parallel_only():
    from dalle_mtf_b200.utils import parse_mesh
    mesh, rules = parse_mesh("data:16,model:2", "batch_dim:data")
    assert mesh == {"data": 16, "model": 2} and rules == {"batch_dim": "data"}
    with pytest.raises(ValueError):
        parse_mesh("data:4,model:2", "batch_dim:data,heads:model")


def test_predict_mode_raises_not_implemented():
    from dalle_mtf_b200.model_fns import PREDICT, dalle_model_fn, vae_model_fn
    with pytest.raises(NotImplementedError):
        dalle_model_fn(None, None, PREDICT, {})
    with pytest.raises(NotImplementedError):
        vae_model_fn(None, None, PREDICT, {})


def test_entry_points_and_reference_import_paths():
    sys.path.insert(0, ROOT)
    import train_dalle, train_vae_tf  # noqa: F401,E401
    from src.model_fns import dalle_model_fn  # noqa: F401
    from src.model_fns_tf import vae_model_fn  # noqa: F401
    from src.optimizers import get_optimizer  # noqa: F401
    from src.input_fns import dalle_input_fn, vae_input_fn  # noqa: F401
    from src.dalle_mtf import DALLE  # noqa: F401
    from src.vae_tf import DiscreteVAE  # noqa: F401
    from src.data import get_tokenizer
    tok = get_tokenizer(None)
    assert len(tok) == 50258 and tok.pad_token_id == 50257     # train_dalle.py:47-49


# ------------------------------------------------------------------------------------------------ optimiser host math
def test_lr_schedule_matches_the_oracle():
    from dalle_mtf_b200.optimizers import OptimizerConfig
    from oracle import optim as OO
    for hp in ({"lr": 1e-3, "train_steps": 100000}, {"lr": 3e-4, "train_steps": 5000, "warmup_steps": 100},
               {"lr": 1e-3, "train_steps": 1000, "lr_decay": "linear", "warmup_steps": 0, "lr_decay_end": 500}):
        cfg = OptimizerConfig(hp)
        for s in (0, 1, 50, 99, 100, 499, 500, 2999, 3000, 4999, 5000, 99999, 100000, 150000):
            assert abs(cfg.learning_rate(s) - OO.learning_rate(s, hp)) <= 1e-15
    cfg = OptimizerConfig({"lr": 1.0, "train_steps": 10})
    assert (cfg.gradient_clipping, cfg.epsilon, cfg.beta_1, cfg.beta_2, cfg.warmup_steps) == (1.0, 1e-6, 0.9, 0.999, 3000)
    with pytest.raises(ValueError):
        OptimizerConfig({"lr": 1.0, "train_steps": 10, "optimizer": "adafactor"})


def test_param_layout_offsets_and_spans():
    from dalle_mtf_b200.dalle_engine import ParamLayout
    lay = ParamLayout()
    lay.add("a", (3, 5)); lay.add("b", (64,)); lay.add("c", (2, 2))
    assert lay.entries["a"][0] == 0 and lay.entries["b"][0] == 64 and lay.entries["c"][0] == 128 and lay.size == 192
    flat = torch.arange(192.0)
    assert lay.view(flat, "b")[0] == 64 and lay.view(flat, "a").shape == (3, 5)
    assert lay.span("b", "c") == (64, 192)


# ------------------------------------------------------------------------------------------------ input contract
def test_input_fns_honour_the_reference_output_contract():
    from dalle_mtf_b200.input_fns import dalle_input_fn, vae_input_fn
    params = {"train_batch_size": 4, "eval_batch_size": 2, "dataset": {"image_size": 32}, "n_channels": 3,
              "text_seq_len": 256, "padding_id": 50257, "text_vocab_size": 50258}
    img, cap = next(iter(dalle_input_fn(params)))
    assert img.shape == (4, 32, 32, 3) and img.dtype == torch.float32 and img.min() >= -1 and img.max() <= 1
    assert cap.shape == (4, 256) and cap.dtype == torch.int32
    # (x - 127.5) / 127.5 of integer pixels                                                   input_fns.py:20
    px = img * 127.5 + 127.5
    assert torch.allclose(px, px.round(), atol=1e-3)
    for row in cap:  # right-padded with padding_id, ids below the GPT-2 vocabulary           input_fns.py:32-38
        n = int((row != 50257).sum())
        assert 5 <= n <= 64 and (row[n:] == 50257).all() and (row[:n] < 50257).all()
    a, b = next(iter(vae_input_fn(params, eval=True)))
    assert a.shape == (2, 32, 32, 3) and a is b                                               # input_fns.py:64


# ------------------------------------------------------------------------------------------------ checkpoints
def test_checkpoint_roundtrip_latest_and_retention(tmp_path):
    from dalle_mtf_b200.utils import (latest_checkpoint, list_checkpoints, load_checkpoint,
                                      load_global_step_from_checkpoint_dir, save_checkpoint)
    d = str(tmp_path / "run")
    assert load_global_step_from_checkpoint_dir(d) == 0 and latest_checkpoint(d) is None
    for step in (10, 20, 30, 40):
        save_checkpoint(d, step, {"w": torch.full((2,), float(step)), "global_step": step}, max_to_keep=2)
    assert [s for s, _ in list_checkpoints(d)] == [30, 40]
    assert load_global_step_from_checkpoint_dir(d) == 40
    st = load_checkpoint(latest_checkpoint(d))
    assert st["global_step"] == 40 and torch.equal(st["w"], torch.full((2,), 40.0))


def test_local_path_maps_gs_urls(monkeypatch):
    from dalle_mtf_b200.utils import local_path
    monkeypatch.setenv("DB200_GS_ROOT", "/tmp/gsroot")
    assert local_path("gs://neo-models/dalle_test/") == "/tmp/gsroot/neo-models/dalle_test/"
    assert local_path("./runs/x") == "./runs/x"


def test_usable_cores_is_positive():
    sys.path.insert(0, ROOT)
    import bench
    assert 1 <= bench.usable_cores() <= (os.cpu_count() or 1)


# ------------------------------------------------------------------------------------------------ data parallel (gloo)
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dp_worker(rank, world, port, out):
    # the host-only path under test: hide any GPU (a machine with fewer GPUs than ranks must still run this test)
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "CUDA_VISIBLE_DEVICES": ""})
    from dalle_mtf_b200.dist import DataParallel
    dp = DataParallel().init(backend="gloo")
    assert dp.shard(8) == (rank * 4, 4)
    flat = torch.full((300,), float(rank + 1))
    hook = dp.make_bucket_hook(flat)
    # backward finishes buckets from the tail: [200,300), then [100,200); [0,100) is left un-reduced on purpose
    dp.hint_tokens_per_gpu(40960)          # sizes the CTA cap of the (here absent) NCCL communicator: host logic only
    assert dp.MAX_CTAS == 4 or "DB200_NCCL_MAX_CTAS" in os.environ
    dp.hint_tokens_per_gpu(5120)
    assert dp.MAX_CTAS == 16 or "DB200_NCCL_MAX_CTAS" in os.environ
    dp.begin_overlap()                     # no C-ABI communicator on CPU: a no-op
    hook(200, 364)      # end beyond the buffer is clipped
    hook(100, 200)
    dp.wait()
    ok = bool((flat[100:] == 3.0).all() and (flat[:100] == float(rank + 1)).all())
    mx = dp.max_over_ranks(float(rank))
    dp.barrier()
    out.put((rank, ok, mx))
    dp.shutdown()


def test_bucketed_allreduce_world_size_2_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res == [(0, True, 1.0), (1, True, 1.0)]


# ------------------------------------------------------------------------------------------------- estimator loop
def test_estimator_keeps_one_input_stream_across_train_calls(tmp_path):
    """train_dalle.py / train_vae_tf.py call train() once per steps_per_checkpoint chunk: the input stream must
    continue (not restart from its seed), and a run resumed from a checkpoint must not replay the first batches."""
    from collections import defaultdict
    from functools import partial
    import torch
    from dalle_mtf_b200.estimator import Estimator
    from dalle_mtf_b200.input_fns import vae_input_fn
    from dalle_mtf_b200.model_fns import StepSpec

    seen, created = [], []

    class _DP:
        rank, world, enabled = 0, 1, False

        def barrier(self):
            pass

    def fake_model_fn(features, labels, mode, params):
        spec = StepSpec(mode, engine=None, dp=_DP())

        def train_op(f, l):
            seen.append(float(f.double().sum()))
            spec.global_step += 1
            spec.loss_sum, spec.loss_scale = torch.zeros(1), 1.0
            return spec.loss_sum
        spec.train_op = train_op
        spec.state_fn = lambda: {"global_step": spec.global_step}
        spec.load_fn = lambda st: setattr(spec, "global_step", int(st["global_step"]))
        created.append(mode)
        return spec

    params = defaultdict(lambda: None, {"dataset": {"image_size": 8, "train_path": "synthetic"}, "train_batch_size": 2,
                                        "model_path": str(tmp_path / "m"), "steps_per_checkpoint": 2, "iterations": 100})
    est = Estimator(fake_model_fn, params)
    fn = partial(vae_input_fn, eval=False)
    est.train(fn, max_steps=2)
    est.train(fn, max_steps=4)
    assert created == ["train"] and len(seen) == 4
    assert len(set(seen)) == 4, "the second train() call replayed batches of the first"
    # a fresh process resuming at step 4 draws from a different stream than a fresh run did at step 0
    first_run = list(seen)
    seen.clear()
    est2 = Estimator(fake_model_fn, params)
    est2.train(fn, max_steps=6)
    assert len(seen) == 2 and not set(seen) & set(first_run)
    est.close(); est2.close()


def test_optimizer_config_distinguishes_missing_from_null_clipping():
    """params.get("gradient_clipping", 1.0) on the reference's defaultdict (src/optimizers.py:27,101)."""
    from collections import defaultdict
    from dalle_mtf_b200.optimizers import OptimizerConfig
    base = {"lr": 1e-3, "train_steps": 10}
    assert OptimizerConfig(defaultdict(lambda: None, base)).gradient_clipping == 1.0
    assert OptimizerConfig(defaultdict(lambda: None, dict(base, gradient_clipping=None))).gradient_clipping is None
    assert OptimizerConfig(defaultdict(lambda: None, dict(base, gradient_clipping=0.5))).gradient_clipping == 0.5
    import pytest
    with pytest.raises(ValueError):
        OptimizerConfig(defaultdict(lambda: None, dict(base, weight_decay=-1)))


def test_tokenizer_loads_bpe_files_from_a_local_directory(tmp_path):
    """src/data/tokenizer_utils.py:4-16 offline: vocab.json + merges.txt from a directory, `<|padding|>` appended as
    the last id (the real GPT-2 files give len 50258 / pad id 50257; a toy vocabulary is used here)."""
    import json
    from dalle_mtf_b200.tokenizer import get_tokenizer
    vocab = {c: i for i, c in enumerate(["a", "b", "c", "ab", "abc", "Ġ", "Ġa", "<|endoftext|>"])}
    (tmp_path / "vocab.json").write_text(json.dumps(vocab))
    (tmp_path / "merges.txt").write_text("#version: 0.2\na b\nab c\nĠ a\n")
    for kind in (None, "hf_gp2tokenizer"):
        tok = get_tokenizer(kind, vocab_dir=str(tmp_path))
        assert len(tok) == len(vocab) + 1 and tok.pad_token_id == len(vocab)
        assert tok.encode("abc") == [vocab["abc"]] and tok.encode("ab a") == [vocab["ab"], vocab["Ġa"]]
    import pytest
    with pytest.raises(FileNotFoundError):
        get_tokenizer(None, vocab_dir=str(tmp_path / "missing"))


def test_bench_helpers_flop_counts_and_scaling_modes():
    """SURVEY.md §8d figures: vae_example 4.03 GFLOP / image, vae_coco (K = 8192) 1 221.6; strong scaling keeps the
    config's global batch (32 -> 4 per GPU at N = 8), weak scaling the per-GPU batch."""
    import bench
    assert abs(bench.vae_train_flops_per_image([[3, 64], [3, 128], [3, 256]], 32, 512) / 1e9 - 4.032) < 0.01
    assert abs(bench.vae_train_flops_per_image([[2, 128], [3, 256], [5, 512]], 256, 8192) / 1e9 - 1221.6) < 0.1
    assert bench.per_gpu_batch_for("dalle_example", 8, "weak") == 32
    assert bench.per_gpu_batch_for("dalle_example", 8, "strong") == 4
    p = bench.load_params(8, "dalle_example", "strong")
    assert p["train_batch_size"] == 32 and p["mesh_shape"] == "data:8"
    assert bench.load_params(8, "dalle_12b")["optimizer_state_sharding"] is True
    assert len(bench.csrc_hash()) == 16
