"""Minimal stand-in for the TPUEstimator loop the reference entry points drive (train_dalle.py:57-98,
train_vae_tf.py:51-93): build once via model_fn, restore the latest checkpoint, run steps from input_fn, save every
`steps_per_checkpoint`, log every `iterations` steps (log_step_count_steps) without syncing the GPU in between.
"""
import time

from .model_fns import DALLE_PARTS_FORMAT, EVAL, TRAIN
from .utils import (latest_checkpoint, load_checkpoint, load_global_step_from_checkpoint_dir, save_checkpoint)


class Estimator:
    def __init__(self, model_fn, params, logger=None):
        self.model_fn = model_fn
        self.params = params
        self.logger = logger
        self._specs = {}
        self._iters = {}      # mode -> (input_fn identity, live iterator)

    def _batches(self, mode, input_fn):
        """ONE persistent input iterator per mode.  train_dalle.py / train_vae_tf.py call train() once per
        steps_per_checkpoint chunk; re-creating a (seeded) pipeline on every call would replay the same file order and
        batches from the start each time and leave the previous producer thread alive (the reference's tf.data
        pipelines are unseeded and simply continue).  A different input_fn replaces, and closes, the old stream."""
        key = getattr(input_fn, "func", input_fn), repr(getattr(input_fn, "keywords", None))
        cur = self._iters.get(mode)
        if cur is None or cur[0] != key:
            if cur is not None and hasattr(cur[1], "close"):
                cur[1].close()
            # a resumed run must not replay the first epoch's order either: the pipelines add this offset to their
            # seeds (every rank reads the same checkpoint directory, so the offset is identical on all ranks)
            if self.params.get("model_path"):
                self.params["_data_seed_offset"] = load_global_step_from_checkpoint_dir(self.params["model_path"])
            cur = (key, iter(input_fn(self.params)))
            self._iters[mode] = cur
        return cur[1]

    def close(self):
        for _, it in self._iters.values():
            if hasattr(it, "close"):
                it.close()
        self._iters = {}

    def _log(self, msg):
        if self.logger is not None:
            self.logger.info(msg)
        else:
            print(msg, flush=True)

    def _spec(self, mode, features, labels):
        if mode not in self._specs:
            spec = self.model_fn(features, labels, mode, self.params)
            ckpt = latest_checkpoint(self.params["model_path"]) if self.params.get("model_path") else None
            if ckpt is not None:
                spec.load_fn(load_checkpoint(ckpt))            # MtfRestoreHook / Saver restore (model_fns.py:206)
                if spec.dp.rank == 0:
                    self._log(f"restored {ckpt} at global step {spec.global_step}")
            self._specs[mode] = spec
        return self._specs[mode]

    def _save(self, spec):
        if spec.dp.rank == 0 and self.params.get("model_path"):
            path = save_checkpoint(self.params["model_path"], spec.global_step, spec.state_fn(),
                                   max_to_keep=self.params.get("max_checkpoints") or 5)   # model_fns.py:212
            self._log(f"saved {path}")
        spec.dp.barrier()

    def train(self, input_fn, max_steps):
        it = self._batches(TRAIN, input_fn)
        features, labels = next(it)
        spec = self._spec(TRAIN, features, labels)
        log_every = self.params.get("iterations") or 100
        ckpt_every = self.params.get("steps_per_checkpoint") or 0
        t0, s0 = time.time(), spec.global_step
        while spec.global_step < max_steps:
            spec.train_op(features, labels)
            if spec.global_step % log_every == 0 or spec.global_step == max_steps:
                loss = float(spec.loss_sum.item()) * spec.loss_scale      # the only host sync
                parts = getattr(spec, "loss_parts", None)
                parts = "" if parts is None else \
                    getattr(spec, "loss_parts_format", DALLE_PARTS_FORMAT).format(*parts.tolist())
                usage = getattr(spec, "codebook_usage", None)
                if usage is not None:   # a collective: every rank runs this branch
                    codes_used, perplexity = usage()
                    parts += f" codes_used {codes_used} perplexity {perplexity:.2f}"
                dt = time.time() - t0
                if spec.dp.rank == 0:
                    self._log(f"step {spec.global_step} loss {loss:.5f}{parts} "
                              f"global_step/sec {(spec.global_step - s0) / max(dt, 1e-9):.3f}")
                t0, s0 = time.time(), spec.global_step
            if ckpt_every and spec.global_step % ckpt_every == 0:
                self._save(spec)
            if spec.global_step < max_steps:
                features, labels = next(it)
        if not ckpt_every or spec.global_step % ckpt_every != 0:
            self._save(spec)
        return spec

    def evaluate(self, input_fn, steps):
        it = self._batches(EVAL, input_fn)
        features, labels = next(it)
        spec = self._spec(EVAL, features, labels)
        train_spec = self._specs.get(TRAIN)
        if train_spec is not None:  # evaluate the weights being trained
            spec.engine.copy_params_from(train_spec.engine)
            spec.global_step = train_spec.global_step
        total = 0.0
        for i in range(steps):
            spec.eval_op(features, labels)
            total += float(spec.loss_sum.item()) * spec.loss_scale
            if i + 1 < steps:
                features, labels = next(it)
        loss = total / max(steps, 1)
        if spec.dp.rank == 0:
            self._log(f"eval loss {loss:.5f} over {steps} steps")
        return {"loss": loss}
