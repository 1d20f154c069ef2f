"""Host-side mirror of src/optimizers.py: hyper-parameter defaults, learning-rate schedule, optimiser wiring.

The schedule is a handful of scalar flops per step and is evaluated on the host from the integer step counter (no
device sync); clip-by-global-norm and Adam themselves are the K9/K10 kernels (csrc/optim.cu).
"""
import math


class OptimizerConfig:
    """Defaults exactly as src/optimizers.py:24-28, 84-87."""

    def __init__(self, params):
        self.lr = params["lr"]
        self.end_step = params.get("lr_decay_end") or params["train_steps"]   # optimizers.py:24
        self.lr_decay = params.get("lr_decay") or "cosine"                    # optimizers.py:25
        ws = params.get("warmup_steps")
        self.warmup_steps = 3000 if ws is None else ws                        # optimizers.py:26
        # optimizers.py:27,101: a MISSING key means 1.0, an explicit `null` disables clipping (`params.get(k, 1.0)` on the
        # reference's defaultdict returns the default only when the key is absent)
        self.gradient_clipping = params["gradient_clipping"] if "gradient_clipping" in params else 1.0
        self.optimizer = (params.get("optimizer") or "adam").lower()          # optimizers.py:28
        self.weight_decay = params.get("weight_decay") or 0.0                 # optimizers.py:84
        self.beta_1 = params.get("beta_1") or 0.9
        self.beta_2 = params.get("beta_2") or 0.999
        self.epsilon = params.get("epsilon") or 1e-6
        if not (isinstance(self.weight_decay, (int, float)) and self.weight_decay >= 0):
            raise ValueError(f"weight_decay must be a non-negative number, got {self.weight_decay!r}")
        if self.optimizer != "adam":
            # the Adafactor branch (optimizers.py:90-97) is selected by no reference config (SURVEY.md §2 row 7)
            raise ValueError(f"{self.optimizer} not recognized (only 'adam' is implemented)")

    def learning_rate(self, step):
        """Value used for the update taken at global step `step` (the step counter before the increment,
        src/model_fns.py:201).  cosine: tf.train.cosine_decay(alpha=0.1); linear: polynomial_decay to 0.1*lr;
        then linear warm-up (optimizers.py:46-76)."""
        s = min(step, self.end_step)
        if self.lr_decay == "linear":
            lr = (self.lr - 0.1 * self.lr) * (1.0 - s / self.end_step) + 0.1 * self.lr
        elif self.lr_decay == "cosine":
            lr = self.lr * (0.9 * 0.5 * (1.0 + math.cos(math.pi * s / self.end_step)) + 0.1)
        else:
            lr = self.lr
        if self.warmup_steps > 0 and step < self.warmup_steps:
            lr = lr * (step / self.warmup_steps)
        return lr


def get_optimizer(mesh, loss, params, variable_dtype=None, inp_var_grads=None):
    """Same signature as the reference's get_optimizer(mesh, loss, params, variable_dtype, inp_var_grads=None)
    (src/optimizers.py:19) and the same 3-tuple back: (learning_rate, update_ops, var_grads).

    What the arguments are here: `mesh` is the engine that owns the variables (the mtf mesh's role: it holds the flat
    fp32 master / gradient / Adam buffers); `loss` is the device scalar the engine's forward produced — gradients
    already sit in the engine's flat buffer after backward(), so it is not differentiated again (mtf.gradients,
    optimizers.py:34); `variable_dtype` is accepted for signature parity (slices are always fp32, ops.py:76-82);
    `inp_var_grads`, when given, is a dict of reference-named gradient tensors that replaces the engine's own.
    learning_rate is a function of the integer global step (host scalar math, no device sync); update_ops(step)
    applies clip-by-global-norm + Adam on the device and returns the learning rate it used."""
    engine = mesh
    cfg = OptimizerConfig(params)
    if inp_var_grads is not None:
        engine.load_flat(engine.grads, inp_var_grads)

    def update_ops(step):
        lr = cfg.learning_rate(step)
        engine.optimizer_step(lr, beta1=cfg.beta_1, beta2=cfg.beta_2, eps=cfg.epsilon,
                              weight_decay=cfg.weight_decay, clip=cfg.gradient_clipping)
        return lr

    return cfg.learning_rate, update_ops, engine.grads
