"""The conv-dVAE launch census (test_vae_config_launches_gpu.py) without a GPU: its routing on synthetic classes, its
exemptions against pytest's collection, the batches it records against the ones the DALL-E configurations run, and the
buffers of every decode pass against the engines' byte budget (counted on the meta device)."""
import glob
import json
import os
import subprocess
import sys

import pytest
import torch

import launch_census as LC
import test_vae_config_launches_gpu as VC
import test_vae_kernels_gpu as VK
import test_vae_paper_kernels_gpu as VPK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def meta_engine(monkeypatch):
    """engine(vae config name) -> its engine on the meta device (shapes and bytes, no device memory)."""
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.model_fns import build_vae_engine
    monkeypatch.setattr(L, "require_device", lambda: None)

    def make(name):
        cfg = VC._config(name)
        return build_vae_engine(cfg, cfg["dataset"]["image_size"], torch.device("meta"))
    return make


def passes(B, n):
    """The images of each pass decode_tokens runs for B images in passes of at most n."""
    return [min(n, B - i) for i in range(0, B, n)]


def test_every_checker_names_a_test_of_the_gpu_module():
    for name, _ in VC.CHECKERS:
        assert callable(getattr(VC, name, None)), name


def test_every_exemption_names_a_collected_test():
    ids = [t for t, *_ in VC.EXEMPT.values()]
    mods = sorted({t.split("::")[0] for t in ids})
    out = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider"] +
                         [os.path.join("tests", m) for m in mods], cwd=ROOT, capture_output=True, text=True)
    collected = {ln.strip()[len("tests/"):] for ln in out.stdout.splitlines() if ln.startswith("tests/")}
    assert collected, out.stdout + out.stderr
    for t in ids:
        hit = t in collected if "[" in t else any(c == t or c.startswith(t + "[") for c in collected)
        assert hit, f"exemption names {t}, which pytest does not collect"


def test_an_exemption_covers_only_the_shapes_its_test_runs():
    cen = VC.make_census()
    f32 = "float32"
    kl = lambda rows, K: LC.launch_class("vae_kl_stats", logits=((rows, K), f32), rows=rows, K=K, scale=1.0 / rows)
    bkl = lambda rows, K: LC.launch_class("gumbel_softmax_bwd_kl", rows=rows, K=K, tau=1.0, c=0.1)
    mse = lambda n: LC.launch_class("mse_fwd_bwd", pred=((n // 3, 3), f32), scale=1.0 / n)
    ll = lambda n_pix, Cp, train: LC.launch_class("logit_laplace", target=((n_pix, Cp), f32) if train else None,
                                                  n_pix=n_pix, Cp=Cp)
    ok = [kl(16384, 8192), kl(32768, 512), bkl(16384, 8192), bkl(4096, 512), mse(16 * 256 * 256 * 3),
          ll(16 * 256 * 256, 3, True)]
    out = [kl(16385, 8192), kl(100, 4096), bkl(32768, 8192), bkl(4096, 1024), mse(64 * 256 * 256 * 3),
           ll(64 * 256 * 256, 3, True), ll(16 * 256 * 256, 6, True), ll(16 * 256 * 256, 3, False)]
    _, exempted, unchecked, _ = cen.classify(ok + out)
    assert set(exempted) == set(ok) and unchecked == out


def test_census_reports_unknown_classes_and_stale_exemptions():
    unknown = LC.launch_class("a_kernel_nobody_knows", n=3)
    conv = LC.launch_class("conv2d_fwd", N=32, H=256, W=256, Cin=64, Cout=3, k=1, stride=1, transposed=False,
                           f32=False, kernel="direct", relu=False, bias=True, residual=False)
    exempt = dict(VC.EXEMPT, retired_kernel=("test_vae_kernels_gpu.py::test_rowmatmul", "no longer launched"))
    checked, _, unchecked, stale = LC.Census(VC.CHECKERS, exempt, set(vars(VC))).classify([conv, unknown])
    assert checked == {conv: "test_convolution_classes"} and unchecked == [unknown]
    assert set(stale) == set(exempt)
    present = set(vars(VC)) - {"test_convolution_classes"}
    _, _, unchecked, _ = LC.Census(VC.CHECKERS, VC.EXEMPT, present).classify([conv])
    assert unchecked == [conv]


def test_the_census_covers_every_conv_vae_configuration():
    paths = sorted(glob.glob(os.path.join(ROOT, "configs", "vae_*_b200.json")))
    conv = [VC._name(p) for p in paths if json.load(open(p)).get("architecture") in (None, "reference")]
    assert conv and VC.CONFIGS == conv
    assert "vae_paper_b200" not in VC.CONFIGS


def test_every_dalle_configuration_has_its_tokenizer_batches_recorded(meta_engine):
    """For each configs/dalle_*_b200.json, its VAE's tokenize batch (the per-GPU train batch) and the pass sizes of
    decoding its predict_batch_size are recorded by the census that owns that network: test_vae_config_launches_gpu.py
    for the convolutional one, test_vae_paper_kernels_gpu.py for the paper's."""
    for dalle in VC.DALLE_CONFIGS:
        cfg = VC._config(dalle)
        vae = cfg["vae_model"]
        eng = meta_engine(vae)
        n = eng.decode_pass_images()
        tok = cfg["train_batch_size"] // VC.data_axis(cfg)
        dec = set(passes(cfg["predict_batch_size"], n))
        if vae in VC.CONFIGS:
            b = VC.phase_batches(vae)
            rec_tok, rec_dec = set(b["tokenize"]), {p for B in b["decode"] for p in passes(B, n)}
        else:
            assert VC._config(vae).get("architecture") == "dalle_paper", vae
            rec_tok, rec_dec = {VPK.TOKENIZE_B}, set(passes(VPK.DECODE_B, n))
        assert tok in rec_tok, (dalle, vae, tok, rec_tok)
        assert dec <= rec_dec, (dalle, vae, dec, rec_dec)


def test_codebook_products_run_at_every_recorded_batch(meta_engine):
    """test_vae_kernels_gpu.test_codebook_products_of_split_operands runs at every batch the census records for a
    network of the same codebook geometry (n_hid, K)."""
    geo = lambda name: (VC._config(name)["convblocks"][-1][1], VC._config(name)["num_tokens"])
    cases = {(geo(c), B) for c, B in VK.CODEBOOK_CASES}
    for vae in VC.CONFIGS:
        b = VC.phase_batches(vae)
        n = meta_engine(vae).decode_pass_images()
        batches = set(b["train"] + b["eval"] + b["tokenize"]) | {p for B in b["decode"] for p in passes(B, n)}
        missing = {B for B in batches if (geo(vae), B) not in cases}
        assert not missing, (vae, missing)


def test_every_decode_pass_fits_the_byte_budget(meta_engine):
    """_alloc's bytes on the meta device for each shipped VAE at every decode pass size it runs: the predict batch of
    each DALL-E configuration that uses it and its own.  One decode_tokens call at 128 images used to allocate them all
    at once: 182 GiB for the paper network."""
    from dalle_mtf_b200.vae_engine import DECODE_PASS_BYTES
    for path in sorted(glob.glob(os.path.join(ROOT, "configs", "vae_*.json"))):
        vae = VC._name(path)
        eng = meta_engine(vae)
        n = eng.decode_pass_images()
        batches = {VC._config(vae)["predict_batch_size"]} | \
            {VC._config(d)["predict_batch_size"] for d in VC.DALLE_CONFIGS if VC._config(d)["vae_model"] == vae}
        for B in sorted(batches):
            for p in sorted(set(passes(B, n))):
                nbytes = eng.buffer_bytes(p)
                print(f"{vae}: decode B={B} pass of {p}: {nbytes / 2 ** 30:.2f} GiB "
                      f"(one pass of {B}: {eng.buffer_bytes(B) / 2 ** 30:.1f} GiB)")
                assert nbytes <= DECODE_PASS_BYTES, (vae, B, p, nbytes)
    assert meta_engine("vae_paper_b200").buffer_bytes(128) > 80 * 10 ** 9
