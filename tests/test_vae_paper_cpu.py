"""CPU tests of the DALL-E paper's discrete-VAE network (architecture "dalle_paper"): the oracle's definition
(oracle/vae_paper.py) — parameter names, shapes and counts, the max-pool tie rule, the gain, the token grid — and the
config validation the model functions and generate_dalle.py share."""
import math

import pytest
import torch

from oracle import vae_paper as P


def test_parameter_count_at_the_paper_geometry():
    shapes = P.param_shapes(8192, logit_laplace=True)
    enc = sum(math.prod(s) for n, s in shapes.items() if n.startswith("encoder/"))
    dec = sum(math.prod(s) for n, s in shapes.items() if n.startswith("decoder/"))
    assert (enc, dec) == (53_786_240, 43_829_766)
    mse = P.param_shapes(8192, logit_laplace=False)
    assert sum(math.prod(s) for s in mse.values()) == enc + dec - 256 * 3 - 3


def test_parameter_names_shapes_and_order():
    shapes = P.param_shapes(8192)
    names = list(shapes)
    assert names[:2] == ["encoder/input/kernel", "encoder/input/bias"]
    assert shapes["encoder/input/kernel"] == (7, 7, 3, 256)
    assert names.index("encoder/output/conv/bias") + 1 == names.index("decoder/input/kernel")
    assert names[-2:] == ["decoder/output/conv/kernel", "decoder/output/conv/bias"]
    assert shapes["encoder/output/conv/kernel"] == (1, 1, 2048, 8192)
    assert shapes["decoder/input/kernel"] == (1, 1, 8192, 128)
    assert shapes["decoder/output/conv/kernel"] == (1, 1, 256, 6)
    # encoder block: 3x3, 3x3, 3x3, 1x1 with h = n_out / 4; id_path only where the width changes, before res_path
    assert "encoder/group_1/block_1/id_path/kernel" not in shapes
    assert shapes["encoder/group_2/block_1/id_path/kernel"] == (1, 1, 256, 512)
    assert names.index("encoder/group_2/block_1/id_path/bias") < names.index("encoder/group_2/block_1/res_path/conv_1/kernel")
    assert [shapes[f"encoder/group_2/block_1/res_path/conv_{j}/kernel"] for j in (1, 2, 3, 4)] == \
        [(3, 3, 256, 128), (3, 3, 128, 128), (3, 3, 128, 128), (1, 1, 128, 512)]
    # decoder block: 1x1, 3x3, 3x3, 3x3; group 1 reads the n_init channels and is 2^(G-1) n_hid wide
    assert [shapes[f"decoder/group_1/block_1/res_path/conv_{j}/kernel"] for j in (1, 2, 3, 4)] == \
        [(1, 1, 128, 512), (3, 3, 512, 512), (3, 3, 512, 512), (3, 3, 512, 2048)]
    assert shapes["decoder/group_1/block_1/id_path/kernel"] == (1, 1, 128, 2048)
    assert shapes["decoder/group_4/block_2/res_path/conv_4/kernel"] == (3, 3, 64, 256)
    blocks = {n.split("/res_path")[0] for n in names if "/res_path/" in n}
    assert len(blocks) == 2 * 4 * 2


def test_init_is_normal_with_fan_in_std_and_zero_biases():
    p = P.init_params(512, n_hid=64, group_count=2, n_init=64, seed=3)
    w = p["encoder/group_1/block_1/res_path/conv_2/kernel"]            # fan-in 3 * 3 * 16
    assert w.std().item() == pytest.approx(1 / math.sqrt(144), rel=0.1)
    assert all(v.abs().sum() == 0 for k, v in p.items() if k.endswith("/bias"))


def test_max_pool_tie_rule_first_maximum_in_raster_order():
    # every window [[a, b], [c, d]] of 4 values from {0, 1}: the gradient lands on the first maximal one
    wins = torch.tensor([[(i >> 3) & 1, (i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(16)], dtype=torch.float32)
    x = wins.view(16, 2, 2).permute(1, 0, 2).reshape(1, 2, 32, 1)   # 16 windows side by side, x[0, dy, 2 j + dx, 0]
    x = x.clone().requires_grad_(True)
    y = P.max_pool(x)
    y.sum().backward()
    g = x.grad.view(2, 16, 2).permute(1, 0, 2).reshape(16, 4)
    first = [int(torch.argmax(w)) for w in wins]                         # torch.argmax: first maximal index
    assert torch.equal(g.argmax(-1), torch.tensor(first)) and torch.equal(g.sum(-1), torch.ones(16))
    for i, w in enumerate(wins):
        m = w.max()
        assert g[i, [j for j in range(4) if w[j] == m][0]] == 1
    x.grad = None
    P.max_pool(x, "tie_last").sum().backward()
    g2 = x.grad.view(2, 16, 2).permute(1, 0, 2).reshape(16, 4)
    tied = (wins == wins.max(-1, keepdim=True).values).sum(-1) > 1
    assert (g2.argmax(-1) != g.argmax(-1))[tied].all()


def test_max_pool_values_equal_torch_and_its_tie_rule_is_pinned():
    g = torch.Generator().manual_seed(0)
    x = torch.randint(-2, 3, (3, 6, 10, 5), generator=g).to(torch.float32)   # many exact ties
    xr = x.clone().requires_grad_(True)
    y = P.max_pool(xr)
    ref = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    assert torch.equal(y.detach(), ref)
    y.sum().backward()
    win = x.reshape(3, 3, 2, 5, 2, 5).permute(0, 1, 3, 5, 2, 4).reshape(3, 3, 5, 5, 4)
    first = (win == win.max(-1, keepdim=True).values).to(torch.int64).argmax(-1)
    grad = xr.grad.reshape(3, 3, 2, 5, 2, 5).permute(0, 1, 3, 5, 2, 4).reshape(3, 3, 5, 5, 4)
    assert torch.equal(grad.argmax(-1), first) and torch.equal(grad.sum(-1), torch.ones(3, 3, 5, 5))
    # torch's own max_pool2d backward on the same input: record where it puts each window's gradient
    xt = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    torch.nn.functional.max_pool2d(xt, 2).sum().backward()
    gt = xt.grad.permute(0, 2, 3, 1).reshape(3, 3, 2, 5, 2, 5).permute(0, 1, 3, 5, 2, 4).reshape(3, 3, 5, 5, 4)
    assert torch.equal(gt.sum(-1), torch.ones(3, 3, 5, 5))
    assert torch.equal(gt.argmax(-1), first), "torch's CPU max_pool2d no longer picks the first maximum"


def test_gain_and_grid():
    assert P.gain(2, 4) == 1 / 64
    assert P.gain(1, 3) == 1 / 9
    assert P.grid_size(256, 4) == 32 and P.grid_size(32, 2) == 16


def test_block_applies_the_gain_to_the_whole_residual_path():
    p = P.init_params(64, n_hid=64, n_blk_per_group=1, group_count=1, n_init=64, seed=1)
    for k in p:
        if k.endswith("/bias"):
            p[k] = torch.full_like(p[k], 0.5)
    x = torch.randn(1, 4, 4, 64, generator=torch.Generator().manual_seed(2))
    blk = ("encoder/group_1/block_1/", 64, 64, (3, 3, 3, 1))
    y = P._block(p, x, *blk, 0.25, False, None)
    y1 = P._block(p, x, *blk, 1.0, False, None)
    assert torch.allclose(y - x, 0.25 * (y1 - x), atol=1e-6)
    # no pre-activation: conv_1 reads x itself
    assert not torch.allclose(P._block(p, x, *blk, 0.25, False, "no_preact"), y)


def _params(**kw):
    from collections import defaultdict
    d = {"num_tokens": 64, "dataset": {"image_size": 32}, "architecture": "dalle_paper", "n_hid": 64,
         "group_count": 2}
    d.update(kw)
    return defaultdict(lambda: None, d)


def test_architecture_key_values():
    from dalle_mtf_b200.model_fns import vae_architecture
    assert vae_architecture(_params(architecture=None), 32) is None
    assert vae_architecture(_params(architecture="reference"), 32) is None
    assert vae_architecture(_params(), 32) == {"n_hid": 64, "n_blk_per_group": 2, "group_count": 2, "n_init": 128}
    assert vae_architecture({"architecture": "dalle_paper"}, 256) == \
        {"n_hid": 256, "n_blk_per_group": 2, "group_count": 4, "n_init": 128}
    for bad in ("paper", "DALLE_PAPER", 1, True):
        with pytest.raises(ValueError, match="architecture"):
            vae_architecture(_params(architecture=bad), 32)


@pytest.mark.parametrize("kw,msg", [
    ({"convblocks": [[2, 64]]}, "convblocks"),
    ({"stack_factor": 2}, "stack_factor"),
    ({"group_count": 4}, "divisible"),            # 32 / 2^3 = 4 ok; use 33 below for the odd case
    ({"n_hid": 60}, "n_hid"),
    ({"n_hid": 56}, "n_hid"),
    ({"n_init": 100}, "n_init"),
    ({"n_blk_per_group": 0}, "n_blk_per_group"),
])
def test_invalid_combinations_are_rejected(kw, msg):
    from dalle_mtf_b200.model_fns import vae_architecture
    size = 36 if kw.get("group_count") == 4 else 32
    with pytest.raises(ValueError, match=msg):
        vae_architecture(_params(**kw), size)


def test_stack_factor_one_and_absent_convblocks_are_accepted():
    from dalle_mtf_b200.model_fns import vae_architecture
    assert vae_architecture(_params(stack_factor=1), 32) is not None
    assert vae_architecture(_params(convblocks=None), 32) is not None


def test_vae_model_fn_rejects_before_touching_a_device():
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn
    with pytest.raises(ValueError, match="convblocks"):
        vae_model_fn(None, None, TRAIN, _params(convblocks=[[2, 64]], train_batch_size=2))


def test_generate_dalle_sizes_the_grid_from_the_architecture():
    import generate_dalle
    ref = {"dataset": {"image_size": 256}, "vae_params": {"convblocks": [[2, 128], [3, 256], [5, 512]]}}
    paper = {"dataset": {"image_size": 256}, "vae_params": {"architecture": "dalle_paper", "group_count": 4}}
    paper3 = {"dataset": {"image_size": 64}, "vae_params": {"architecture": "dalle_paper", "group_count": 3,
                                                            "n_hid": 64}}
    assert generate_dalle.token_grid_side(ref) == 32
    assert generate_dalle.token_grid_side(paper) == 32
    assert generate_dalle.token_grid_side(paper3) == 16
    assert generate_dalle.prefix_length(paper3, 3) == 48


def test_configs_name_the_paper_geometry():
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    vae = json.load(open(os.path.join(root, "configs", "vae_paper_b200.json")))
    assert (vae["architecture"], vae["n_hid"], vae["n_blk_per_group"], vae["group_count"], vae["n_init"],
            vae["num_tokens"], vae["dataset"]["image_size"]) == ("dalle_paper", 256, 2, 4, 128, 8192, 256)
    assert vae["use_bf16"] and vae["reconstruction_loss"] == "logit_laplace" and vae["train_gumbel_hard"] is False
    assert (vae["kl_loss_weight"], vae["kl_anneal_steps"], vae["temp_start"], vae["temp"],
            vae["temp_anneal_steps"]) == (0.034375, 5000, 1, 0.0625, 150000)
    assert vae["mesh_shape"] == "data:8" and vae["train_batch_size"] == 64 and "convblocks" not in vae
    dalle = json.load(open(os.path.join(root, "configs", "dalle_coco_paper_vae_b200.json")))
    base = json.load(open(os.path.join(root, "configs", "dalle_coco_b200.json")))
    assert dalle["vae_model"] == "vae_paper_b200"
    assert {k: v for k, v in dalle.items() if k not in ("vae_model", "model_path")} == \
        {k: v for k, v in base.items() if k not in ("vae_model", "model_path")}
