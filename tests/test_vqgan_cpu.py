"""CPU tests of the VQGAN tokenizer (architecture "vqgan"): config validation and its refusals, the taming importer, the
grid size, meta-device buffer bytes, and the oracle's mutants (each must make a comparison of tests/test_vqgan_gpu.py
fail)."""
import json
import os
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from oracle import vqgan as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _cfg(**extra):
    geo = O.GEOMETRY_TEST
    d = {"model_type": "vae", "dataset": {"image_size": 64}, "architecture": "vqgan", "num_tokens": geo["num_tokens"],
         **{k: geo[k] for k in ("ch", "ch_mult", "num_res_blocks", "attn_resolutions", "z_channels", "embed_dim",
                                "resolution")}}
    d.update(extra)
    return defaultdict(lambda: None, d)


@pytest.fixture
def meta(monkeypatch):
    from dalle_mtf_b200 import lib as L
    monkeypatch.setattr(L, "require_device", lambda: None)


def test_geometry_grid_and_sequence_length(meta):
    from dalle_mtf_b200.model_fns import build_vae_engine, vae_architecture, vae_grid_size
    cfg = json.load(open(os.path.join(ROOT, "configs", "vae_vqgan_f16_16384_b200.json")))
    assert vae_grid_size(cfg, 256) == 16
    eng = build_vae_engine(cfg, 256, torch.device("meta"))
    assert (eng.K, eng.image_seq_len, eng.hw, eng.img_H, eng.img_W, eng.img_C) == (16384, 256, 16, 256, 256, 3)
    assert vae_architecture(cfg, 256)["ch_mult"] == [1, 1, 2, 2, 4]
    assert vae_grid_size(_cfg(), 64) == 16
    small = build_vae_engine(_cfg(), 64, torch.device("meta"))
    assert small.image_seq_len == 256
    # the other architectures keep their contract
    assert vae_architecture({"architecture": "dalle_paper"}, 256) == {"n_hid": 256, "n_blk_per_group": 2,
                                                                      "group_count": 4, "n_init": 128}
    assert vae_grid_size({"architecture": "dalle_paper"}, 256) == 32
    assert vae_architecture({}, 256) is None and vae_grid_size({}, 256) == 32


def test_meta_buffer_bytes_count_the_live_layers_only(meta):
    from dalle_mtf_b200.model_fns import build_vae_engine
    from dalle_mtf_b200.vae_engine import DECODE_PASS_BYTES
    cfg = json.load(open(os.path.join(ROOT, "configs", "vae_vqgan_f16_16384_b200.json")))
    eng = build_vae_engine(cfg, 256, torch.device("meta"))
    one, many = eng.buffer_bytes(1), eng.buffer_bytes(16)
    # the largest activation is [256, 256, 128] bf16 = 16 MiB per image; a few of them plus the scores
    assert 3 * 2 ** 24 < one < 2 ** 28 and many == pytest.approx(16 * one, rel=0.01)
    n = eng.decode_pass_images()
    assert n >= cfg["predict_batch_size"] and eng.buffer_bytes(n) <= DECODE_PASS_BYTES


@pytest.mark.parametrize("change,match", [
    ({"ch": 96}, "ch = 96"),
    ({"z_channels": 96}, "z_channels"),
    ({"embed_dim": 32}, "embed_dim"),
    ({"resolution": 128}, "resolution"),
    ({"ch_mult": [1, 2, 2, 2, 2, 2, 2, 2]}, "image_size"),
    ({"attn_resolutions": [32]}, "attn_resolutions"),
    ({"ch_mult": [1, 2]}, "mid AttnBlock"),
    ({"ch": 384}, "channels"),
    ({"convblocks": [[2, 64]]}, "convblocks"),
    ({"n_hid": 64}, "n_hid"),
    ({"stack_factor": 2}, "stack_factor"),
    ({"use_bf16": False}, "use_bf16"),
    ({"embed_dim": None}, "embed_dim"),
    ({"kl_loss_weight": 0.1}, "kl_loss_weight"),
])
def test_config_validation_names_the_key(change, match):
    from dalle_mtf_b200.model_fns import vae_architecture
    with pytest.raises(ValueError, match=match):
        vae_architecture(_cfg(**change), 64)


def test_vae_model_fn_refuses_a_vqgan_before_any_device_work(monkeypatch):
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import TRAIN, vae_model_fn

    def no_device():
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(L, "require_device", no_device)
    with pytest.raises(ValueError, match="vqgan"):
        vae_model_fn(None, None, TRAIN, _cfg(train_batch_size=2))


# ------------------------------------------------------------------------------------------------------ importer
def test_import_maps_names_and_shapes():
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict, network
    geo = O.GEOMETRY_TEST
    sd = O.random_state_dict(geo, 1)
    named = import_taming_state_dict({**sd, "loss.discriminator.main.0.weight": torch.zeros(3)}, geo)
    assert list(named) == network(geo)[2].order
    assert len(named) == len(sd)
    w = sd["encoder.down.1.block.0.conv1.weight"]                      # OIHW [128, 64, 3, 3]
    assert torch.equal(named["encoder/down/1/block/0/conv1/weight"], w.permute(2, 3, 1, 0))
    assert named["encoder/down/1/block/0/nin_shortcut/weight"].shape == (1, 1, 64, 128)
    assert torch.equal(named["quantize/embedding/weight"], sd["quantize.embedding.weight"])
    assert torch.equal(named["decoder/up/2/attn/1/q/weight"].view(128, 128), sd["decoder.up.2.attn.1.q.weight"][:, :, 0, 0].T)
    assert "decoder/up/0/upsample/conv/weight" not in named and "decoder/up/1/upsample/conv/weight" in named
    assert "encoder/down/2/downsample/conv/weight" not in named


@pytest.mark.parametrize("edit,match", [
    (lambda sd: sd.pop("decoder.mid.attn_1.k.bias"), "decoder.mid.attn_1.k.bias: missing"),
    (lambda sd: sd.__setitem__("encoder.extra.weight", torch.zeros(1)), "encoder.extra.weight: not a tensor"),
    (lambda sd: sd.__setitem__("quant_conv.weight", torch.zeros(64, 64, 3, 3)), "quant_conv.weight: shape"),
    (lambda sd: sd.__setitem__("quantize.embed.weight", torch.zeros(512, 64)), "quantize.embed.weight: a Gumbel"),
    (lambda sd: sd.__setitem__("quantize.proj.weight", torch.zeros(512, 64, 1, 1)), "quantize.proj.weight: a Gumbel"),
    (lambda sd: sd.__setitem__("encoder.conv_out.weight", torch.zeros(128, 128, 3, 3)), "double_z"),
])
def test_import_refusals_name_the_variable(edit, match):
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    sd = O.random_state_dict(O.GEOMETRY_TEST, 2)
    edit(sd)
    with pytest.raises(ValueError, match=match):
        import_taming_state_dict(sd, O.GEOMETRY_TEST)


@pytest.mark.parametrize("lightning", [True, False])
def test_import_cli_writes_a_checkpoint(tmp_path, lightning):
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    from tools import import_vqgan
    cfg = dict(_cfg(model_path=str(tmp_path / "run")))
    (tmp_path / "vq.json").write_text(json.dumps(cfg))
    sd = O.random_state_dict(O.GEOMETRY_TEST, 3)
    torch.save({"state_dict": sd, "epoch": 3} if lightning else sd, tmp_path / "in.ckpt")
    import_vqgan.main(["--model", str(tmp_path / "vq.json"), "--ckpt", str(tmp_path / "in.ckpt")])
    st = load_checkpoint(latest_checkpoint(str(tmp_path / "run")))
    assert st["global_step"] == 0
    assert torch.equal(st["vae/encoder/conv_in/weight"], sd["encoder.conv_in.weight"].permute(2, 3, 1, 0))
    assert len([k for k in st if k.startswith("vae/")]) == len(sd)


class _Opaque:
    """An object a Lightning checkpoint may pickle (its hyper-parameters) that weights_only loading refuses."""


def test_import_cli_explains_a_checkpoint_it_cannot_read_safely(tmp_path):
    from tools import import_vqgan
    (tmp_path / "vq.json").write_text(json.dumps(dict(_cfg(model_path=str(tmp_path / "run")))))
    torch.save({"state_dict": O.random_state_dict(O.GEOMETRY_TEST, 3), "cfg": _Opaque()}, tmp_path / "in.ckpt")
    with pytest.raises(SystemExit, match="weights_only=False.*state_dict"):
        import_vqgan.main(["--model", str(tmp_path / "vq.json"), "--ckpt", str(tmp_path / "in.ckpt")])


# ------------------------------------------------------------------------------------------------------ oracle
def _images(B, size, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(B, 3, size // 8, size // 8, generator=g) * 2 - 1
    img = F.interpolate(low, size=(size, size), mode="bilinear", align_corners=False)
    return img.clamp(-1, 1).permute(0, 2, 3, 1).contiguous().double()


@pytest.mark.parametrize("mut", O.MUTANTS)
def test_oracle_mutants_fail_the_gpu_comparisons(mut):
    """Each mutant, standing in for the engine, fails what tests/test_vqgan_gpu.py asserts: a code that differs on a
    row the gap decides or a z further from the oracle's than test_codes_agree_with_the_oracle_where_the_gap_decides_them
    allows, or a decoded image
    further from the oracle than test_decode_tokens_against_the_oracle's bound.  For the GroupNorm eps the network's
    activations are scaled down until the eps matters (conv_in's weights x 1e-3)."""
    import test_vqgan_gpu as G
    geo = O.GEOMETRY_TEST
    sd = O.to(O.random_state_dict(geo, 7), F64)
    if mut == "gn_eps":
        sd["encoder.conv_in.weight"] = sd["encoder.conv_in.weight"] * 1e-3
        sd["encoder.conv_in.bias"] = sd["encoder.conv_in.bias"] * 1e-3
    img = _images(2, 64, 8)
    E = sd["quantize.embedding.weight"]
    if mut == "tie_last":
        z = torch.cat([E[:1], E[:1]])
        Et = torch.cat([E[:4], E[:1]])               # code 4 ties with code 0
        assert O.nearest_codes(z, Et).tolist() == [0, 0] and O.nearest_codes(z, Et, mut).tolist() == [4, 4]
        return
    z = O.encode_z(sd, geo, img).reshape(-1, geo["embed_dim"])
    zm = O.encode_z(sd, geo, img, mut).reshape(-1, geo["embed_dim"])
    d = O.distances(z, E)
    two = d.topk(2, dim=1, largest=False)
    best, gap = two.indices[:, 0], two.values[:, 1] - two.values[:, 0]
    spread = (E[best][:, None, :] - E[None, :, :]).norm(dim=-1).amax(-1)
    rnd = 4 * (3 * 2.0 ** -16 + (geo["embed_dim"] + 2) * 2.0 ** -23) * (zm.abs() @ E.abs().T).amax(-1)
    decided = gap > 2 * (zm - z).norm(dim=-1) * spread + rnd
    codes_fail = not torch.equal(O.nearest_codes(zm, E)[decided], best[decided])
    codes = best.view(2, -1)
    ref, dm = O.decode(sd, geo, codes), O.decode(sd, geo, codes, mut)
    decode_fail = ((dm - ref).norm() / ref.norm()).item() >= G._decoder_roundings(geo) * 2.0 ** -9
    z_fail = ((zm - z).norm() / z.norm()).item() >= G._encoder_roundings(geo) * 2.0 ** -9
    assert z_fail or codes_fail or decode_fail, mut


# ------------------------------------------------------------------------------------------------------ buffers
# launches of the engine: name -> (positions of the inputs a launch reads, position of the output it writes)
_LAUNCHES = {"conv2d_fwd": ((1, 4), 5), "conv2d_fwd_tc": ((1, 4), 5), "groupnorm": ((0,), 5),
             "linear_fwd": ((0, "residual"), 2), "attn_noncausal": ((0,), 1), "upsample2x_fwd": ((0,), 1),
             "gemm": ((0,), 2), "cast_f32_to_bf16": ((0,), 1), "clamp_bf16_to_f32": ((0,), 1)}


@pytest.mark.parametrize("geo", [
    dict(ch=64, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[], z_channels=128, embed_dim=64, num_tokens=64,
         resolution=32),                                           # z_channels == ch * ch_mult[-1]
    dict(ch=64, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[], z_channels=64, embed_dim=64, num_tokens=64,
         resolution=32),
    dict(ch=64, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2, attn_resolutions=[16], z_channels=256, embed_dim=64,
         num_tokens=64, resolution=256),                           # z_channels == ch * ch_mult[-1] with attention
    dict(ch=64, ch_mult=[1, 1, 2, 2, 2], num_res_blocks=1, attn_resolutions=[16], z_channels=64, embed_dim=64,
         num_tokens=64, resolution=128),                           # one width attending at S = 256 and S = 64
    O.GEOMETRY_TEST,
])
def test_no_launch_writes_a_buffer_it_reads(meta, monkeypatch, geo):
    """The engine's encode and decode with every launch replaced by a check: no output shares memory with an input of
    the same launch, and every output holds the rows its input has."""
    from dalle_mtf_b200 import ops
    from dalle_mtf_b200.vqgan_engine import VqganEngine
    seen = []

    def stub(name, pos_in, pos_out):
        def f(*a, **k):
            out = a[pos_out]
            for p in pos_in:
                x = k.get(p) if isinstance(p, str) else a[p]
                if x is None:
                    continue
                assert x.data_ptr() != out.data_ptr(), f"{name} writes its input"
                if name in ("linear_fwd", "gemm", "attn_noncausal"):
                    assert x.shape[0] == out.shape[0], f"{name}: {tuple(x.shape)} -> {tuple(out.shape)}"
            seen.append(name)
            return out
        return f
    for name, (pos_in, pos_out) in _LAUNCHES.items():
        monkeypatch.setattr(ops, name, stub(name, pos_in, pos_out))
    for name in ("split_f32", "argmax_rows", "gather_rows_split"):
        monkeypatch.setattr(ops, name, lambda *a, **k: None)
    eng = VqganEngine(geo["num_tokens"], geo["resolution"], geo["ch"], geo["ch_mult"], geo["num_res_blocks"],
                      geo["attn_resolutions"], geo["z_channels"], geo["embed_dim"], device="cpu")
    H = geo["resolution"]
    for B in (1, 2):
        eng.encode_tokens(torch.zeros(B, H, H, 3))
        eng.decode_tokens(torch.zeros(B, eng.image_seq_len, dtype=torch.int32))
    assert seen.count("conv2d_fwd_tc") > 0 and seen.count("groupnorm") > 0
