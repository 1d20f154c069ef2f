"""CPU tests of Gumbel-quantised VQGANs ("quantizer": "gumbel", taming's GumbelVQ): config validation and the long
attention range, the importer and its CLI, the grid size, meta-device buffer bytes, the stubbed-launch buffer check on
the Gumbel geometries, and the oracle's Gumbel mutants (each must make a comparison of tests/test_vqgan_gumbel_gpu.py
fail), as must the existing attention mutants against the long-attention bound."""
import json
import os
from collections import defaultdict

import pytest
import torch

import test_vqgan_cpu as VC
from oracle import vqgan as O
from oracle import vqgan_gumbel as OG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
GUMBEL_CFG = os.path.join(ROOT, "configs", "vae_vqgan_gumbel_f8_8192_b200.json")


def _cfg(geo=OG.GEOMETRY_GUMBEL_TEST, **extra):
    d = {"model_type": "vae", "dataset": {"image_size": geo["resolution"]}, "architecture": "vqgan",
         "num_tokens": geo["num_tokens"], "quantizer": geo.get("quantizer"),
         **{k: geo[k] for k in ("ch", "ch_mult", "num_res_blocks", "attn_resolutions", "z_channels", "embed_dim",
                                "resolution")}}
    d.update(extra)
    return defaultdict(lambda: None, d)


meta = VC.meta


# ------------------------------------------------------------------------------------------------------ config
def test_quantizer_key_selects_the_layout():
    from dalle_mtf_b200.model_fns import vqgan_geometry
    from dalle_mtf_b200.vqgan_engine import network
    assert vqgan_geometry(_cfg(), 64)["quantizer"] == "gumbel"
    assert vqgan_geometry(_cfg(quantizer=None), 64)["quantizer"] == "vq"
    assert vqgan_geometry(_cfg(quantizer="vq"), 64)["quantizer"] == "vq"
    lay = network(OG.GEOMETRY_GUMBEL_TEST)[2]
    assert lay.entries["quantize/proj/weight"][1] == (1, 1, 64, 512)
    assert lay.entries["quantize/proj/bias"][1] == (512,)
    assert lay.entries["quantize/embed/weight"][1] == (512, 64)
    assert "quantize/embedding/weight" not in lay.entries
    assert "quant_conv/weight" in lay.entries and "post_quant_conv/weight" in lay.entries


@pytest.mark.parametrize("change,match", [
    ({"quantizer": "ema"}, "quantizer"),
    ({"quantizer": True}, "quantizer"),
    ({"embed_dim": 128}, "embed_dim"),
    ({"attn_resolutions": [32], "ch_mult": [1, 2]}, "attn_resolutions"),          # S = 1024 at C = 256
    ({"ch_mult": [1, 2], "attn_resolutions": []}, "mid AttnBlock"),                # the mid block at C = 256
    ({"dataset": {"image_size": 144}, "resolution": 144, "ch_mult": [1, 4], "attn_resolutions": []},
     "mid AttnBlock"),                                                           # S = 72^2 = 5184 > 4096
])
def test_gumbel_config_validation_names_the_key(change, match):
    from dalle_mtf_b200.model_fns import vae_architecture
    cfg = _cfg(**change)
    with pytest.raises(ValueError, match=match):
        vae_architecture(cfg, cfg["dataset"]["image_size"])


def test_long_attention_range_at_its_edges():
    from dalle_mtf_b200.model_fns import vae_architecture
    from dalle_mtf_b200.vqgan_engine import attention_in_range
    assert attention_in_range(320, 512) and attention_in_range(4096, 512) and attention_in_range(1024, 512)
    assert not attention_in_range(4160, 512) and not attention_in_range(1024, 256)
    assert not attention_in_range(352, 512) and not attention_in_range(1024, 576)
    assert attention_in_range(256, 512) and attention_in_range(256, 128) and not attention_in_range(320, 128)
    # through a geometry: a 64 x 64 mid block at C = 512 (S = 4096) is accepted, a 24 x 24 one (S = 576) too
    for size in (128, 48):
        cfg = _cfg(dataset={"image_size": size}, resolution=size, ch_mult=[1, 4], attn_resolutions=[])
        assert vae_architecture(cfg, size)["resolution"] == size


# ------------------------------------------------------------------------------------------------------ importer
def test_gumbel_import_maps_names_and_shapes():
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict, network
    geo = OG.GEOMETRY_GUMBEL_TEST
    sd = OG.random_state_dict(geo, 1)
    assert tuple(sd["quantize.proj.weight"].shape) == (512, 64, 1, 1) and "quantize.embedding.weight" not in sd
    named = import_taming_state_dict({**sd, "loss.discriminator.main.0.weight": torch.zeros(3)}, geo)
    assert list(named) == network(geo)[2].order and len(named) == len(sd)
    assert torch.equal(named["quantize/proj/weight"].view(64, 512), sd["quantize.proj.weight"][:, :, 0, 0].T)
    assert torch.equal(named["quantize/proj/bias"], sd["quantize.proj.bias"])
    assert torch.equal(named["quantize/embed/weight"], sd["quantize.embed.weight"])
    assert named["decoder/up/1/attn/1/q/weight"].shape == (1, 1, 512, 512)


@pytest.mark.parametrize("edit,match", [
    (lambda sd: sd.__setitem__("quantize.embedding.weight", torch.zeros(512, 64)),
     "quantize.embedding.weight: a VectorQuantizer.*\"quantizer\": \"vq\""),
    (lambda sd: sd.pop("quantize.proj.bias"), "quantize.proj.bias: missing"),
    (lambda sd: sd.__setitem__("quantize.proj.weight", torch.zeros(512, 128, 1, 1)), "quantize.proj.weight: shape"),
    (lambda sd: sd.__setitem__("quantize.embed.weight", torch.zeros(256, 64)), "quantize.embed.weight: shape"),
])
def test_gumbel_import_refusals_name_the_variable(edit, match):
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    sd = OG.random_state_dict(OG.GEOMETRY_GUMBEL_TEST, 2)
    edit(sd)
    with pytest.raises(ValueError, match=match):
        import_taming_state_dict(sd, OG.GEOMETRY_GUMBEL_TEST)


def test_vq_import_of_a_gumbel_checkpoint_points_to_the_config_key():
    from dalle_mtf_b200.vqgan_engine import import_taming_state_dict
    geo = dict(OG.GEOMETRY_GUMBEL_TEST, quantizer="vq")
    with pytest.raises(ValueError, match="quantize.proj.weight: a Gumbel.*\"quantizer\": \"gumbel\""):
        import_taming_state_dict(OG.random_state_dict(OG.GEOMETRY_GUMBEL_TEST, 2), geo)


def test_import_cli_writes_a_gumbel_checkpoint(tmp_path):
    from dalle_mtf_b200.utils import latest_checkpoint, load_checkpoint
    from tools import import_vqgan
    (tmp_path / "vq.json").write_text(json.dumps(dict(_cfg(model_path=str(tmp_path / "run")))))
    sd = OG.random_state_dict(OG.GEOMETRY_GUMBEL_TEST, 3)
    torch.save({"state_dict": sd, "epoch": 3}, tmp_path / "in.ckpt")
    import_vqgan.main(["--model", str(tmp_path / "vq.json"), "--ckpt", str(tmp_path / "in.ckpt")])
    st = load_checkpoint(latest_checkpoint(str(tmp_path / "run")))
    assert torch.equal(st["vae/quantize/embed/weight"], sd["quantize.embed.weight"])
    assert torch.equal(st["vae/quantize/proj/weight"], sd["quantize.proj.weight"].permute(2, 3, 1, 0))
    assert len([k for k in st if k.startswith("vae/")]) == len(sd)
    with pytest.raises(SystemExit, match="quantize.proj.weight: a Gumbel"):      # the same file under "vq"
        (tmp_path / "vq2.json").write_text(json.dumps(dict(_cfg(model_path=str(tmp_path / "r2"), quantizer="vq"))))
        import_vqgan.main(["--model", str(tmp_path / "vq2.json"), "--ckpt", str(tmp_path / "in.ckpt")])


# ------------------------------------------------------------------------------------------------------ engine
def test_gumbel_grid_and_sequence_length(meta):
    from dalle_mtf_b200.model_fns import build_vae_engine, vae_grid_size
    cfg = json.load(open(GUMBEL_CFG))
    assert vae_grid_size(cfg, 256) == 32
    eng = build_vae_engine(cfg, 256, torch.device("meta"))
    assert (eng.K, eng.image_seq_len, eng.hw, eng.img_H, eng.gumbel) == (8192, 1024, 32, 256, True)
    assert eng.codebook == "quantize/embed/weight"
    assert vae_grid_size(_cfg(), 64) == 32
    assert build_vae_engine(_cfg(), 64, torch.device("meta")).image_seq_len == 1024
    # dalle_coco_b200's image tokens and image vocabulary match the f8 tokenizer
    coco = json.load(open(os.path.join(ROOT, "configs", "dalle_coco_b200.json")))
    assert coco["image_vocab_size"] == eng.K


def test_gumbel_meta_buffer_bytes(meta):
    from dalle_mtf_b200.model_fns import build_vae_engine
    from dalle_mtf_b200.vae_engine import DECODE_PASS_BYTES
    cfg = json.load(open(GUMBEL_CFG))
    eng = build_vae_engine(cfg, 256, torch.device("meta"))
    one, many = eng.buffer_bytes(1), eng.buffer_bytes(16)
    # [256, 256, 128] bf16 activations of 16 MiB per image, the [1024, 8192] f32 logits of 32 MiB
    assert 2 ** 25 + 3 * 2 ** 24 < one < 2 ** 28 and many == pytest.approx(16 * one, rel=0.01)
    n = eng.decode_pass_images()
    assert eng.buffer_bytes(n) <= DECODE_PASS_BYTES < eng.buffer_bytes(n + 1)


@pytest.mark.parametrize("geo", [OG.GEOMETRY_GUMBEL_TEST, OG.GEOMETRY_GUMBEL_F8,
                                 dict(OG.GEOMETRY_GUMBEL_TEST, ch_mult=[1, 4, 4])])   # C = 512 at S = 1024 and 256
def test_no_launch_writes_a_buffer_it_reads_on_gumbel_geometries(meta, monkeypatch, geo):
    """test_vqgan_cpu.py's stubbed-launch check with the long attention in the stub table."""
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
                if name in ("linear_fwd", "gemm", "attn_noncausal", "attn_noncausal_long"):
                    assert x.shape[0] == out.shape[0], f"{name}: {tuple(x.shape)} -> {tuple(out.shape)}"
            seen.append(name)
            return out
        return f
    launches = dict(VC._LAUNCHES, attn_noncausal_long=((0,), 1))
    for name, (pos_in, pos_out) in launches.items():
        monkeypatch.setattr(ops, name, stub(name, pos_in, pos_out))
    for name in ("split_f32", "argmax_rows", "gather_rows_split"):
        monkeypatch.setattr(ops, name, lambda *a, **k: None)
    eng = VqganEngine(geo["num_tokens"], geo["resolution"], geo["ch"], geo["ch_mult"], geo["num_res_blocks"],
                      geo["attn_resolutions"], geo["z_channels"], geo["embed_dim"], device="cpu",
                      quantizer=geo["quantizer"])
    H = geo["resolution"]
    for B in (1, 2):
        eng.encode_tokens(torch.zeros(B, H, H, 3))
        eng.decode_tokens(torch.zeros(B, eng.image_seq_len, dtype=torch.int32))
    assert seen.count("attn_noncausal_long") > 0 and seen.count("conv2d_fwd_tc") > 0
    assert ("attn_noncausal" in seen) == (geo["ch_mult"] == [1, 4, 4])


# ------------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("mut", OG.GUMBEL_MUTANTS)
def test_gumbel_mutants_fail_the_gpu_comparisons(mut):
    """Each Gumbel mutant, standing in for the engine, fails what tests/test_vqgan_gumbel_gpu.py asserts: a code that
    differs on a row the logit gap decides, a tie that does not go to the first index, or a decoded image further from
    the oracle than the decode test's bound."""
    import test_vqgan_gpu as G
    import test_vqgan_gumbel_gpu as GG
    geo = OG.GEOMETRY_GUMBEL_TEST
    sd = O.to(OG.random_state_dict(geo, 7), F64)
    if mut == "gumbel_tie_last":
        w, b = sd["quantize.proj.weight"], sd["quantize.proj.bias"]
        w[1::2], b[1::2] = w[0::2], b[0::2]
        z = torch.randn(16, geo["embed_dim"], dtype=F64, generator=torch.Generator().manual_seed(1))
        assert (OG.codes(sd, z) % 2 == 0).all() and (OG.codes(sd, z, mut) % 2 == 1).all()
        return
    if mut == "gumbel_no_bias":
        z = O.encode_z(sd, geo, VC._images(1, 64, 8)).reshape(-1, geo["embed_dim"])
        best, decided = GG.gumbel_decided(sd, z, z)
        assert not torch.equal(OG.codes(sd, z, mut)[decided], best[decided])
        return
    codes = torch.randint(0, geo["num_tokens"], (1, 1024), generator=torch.Generator().manual_seed(2))
    ref, dm = OG.decode(sd, geo, codes), OG.decode(sd, geo, codes, mut)
    assert ((dm - ref).norm() / ref.norm()).item() >= G._decoder_roundings(geo) * 2.0 ** -9


@pytest.mark.parametrize("mut", ["no_scale", "softmax_queries"])
def test_attention_mutants_fail_the_long_attention_bound(mut):
    """The oracle's attention mutants at S = 1024, C = 512 land outside test_long_attention_against_float64's bound
    around the correct attention, computed on the same bf16 inputs."""
    import test_vqgan_gumbel_gpu as GG
    S, C = 1024, 512
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(1, S, C, generator=g) for _ in range(3))
    qkv = torch.cat([q, k, v], -1).to(torch.bfloat16)
    ref, tol = GG.long_attention_reference(qkv, C, C ** -0.5)
    qd, kd, vd = (t.to(F64) for t in qkv.split(C, -1))
    s = qd @ kd.transpose(1, 2)
    p = torch.softmax(s, -1) if mut == "no_scale" else torch.softmax(s * C ** -0.5, 1)
    out = (p @ vd).to(torch.bfloat16).to(F64)
    import float64_bounds as FB
    assert FB.worst_ratio(mut, out, ref, tol, a=0, b=1.0, bf16_out=True) > 1.0
