"""The class matching of the DALL-E launch census (test_dalle_config_launches_gpu.py) on synthetic records, without a
GPU: launch classes are described from CPU tensors with the GPU module's own describe(), and routed by its own
CHECKERS and EXEMPT.  A census that cannot report an unknown class, a class that differs from a checked one only in a
pitch, a stale exemption or a deleted replay test would pass vacuously."""
import inspect
import os
import subprocess
import sys

import torch

import launch_census as LC
import test_dalle_config_launches_gpu as CL


def bound(entry, *args, **kw):
    from dalle_mtf_b200 import ops
    ba = inspect.signature(getattr(ops, entry)).bind(*args, **kw)
    ba.apply_defaults()
    return dict(ba.arguments)


def cls(entry, *args, **kw):
    return CL.describe(entry, bound(entry, *args, **kw))[0]


def gemm_pair():
    """A plain product with a bias and the same product whose B is a window of a wider buffer (only ldb differs):
    no replay here takes a windowed B with a bias epilogue."""
    x = torch.zeros(64, 520, dtype=torch.bfloat16)
    w = torch.zeros(512, 520, dtype=torch.bfloat16)
    wide = torch.zeros(512, 50816, dtype=torch.bfloat16)
    out = torch.zeros(64, 512, dtype=torch.bfloat16)
    bias = torch.zeros(512)
    plain = cls("gemm", x, w, out, 64, 512, 520, bias=bias)
    window = cls("gemm", x, wide[:, :520], out, 64, 512, 520, bias=bias)
    return plain, window


def test_a_window_differs_from_its_plain_product_only_in_the_pitch():
    plain, window = gemm_pair()
    fp, fw = LC.fields(plain), LC.fields(window)
    assert {k for k in fp if fp[k] != fw[k]} == {"b_strided"}
    assert CL.is_plain_gemm(plain) and not CL.is_plain_gemm(window) and not CL.is_window_gemm(window)
    # without the bias it is a window product (the logits mask's vocabulary dgrad)
    x = torch.zeros(64, 520, dtype=torch.bfloat16)
    W = torch.zeros(512, 50816, dtype=torch.bfloat16)
    assert CL.is_window_gemm(cls("gemm", x, W[:, 50256:50776], torch.zeros(64, 512, dtype=torch.bfloat16), 64, 512,
                                 520))
    # the logits mask's wgrad window: D strided and at the image offset's alignment
    h = torch.zeros(64, 512, dtype=torch.bfloat16)
    dl = torch.zeros(64, 520, dtype=torch.bfloat16)
    G = torch.zeros(512, 50816)
    c = cls("gemm", h, dl, G[:, 50256:50776], 512, 520, 64, a_mn=True, b_mn=True, mode=CL._lib().EPI_ATOMIC,
            split_k=0)
    f = LC.fields(c)
    assert f["d_strided"] and f["d_off"] == 50256 % 128 and CL.is_window_gemm(c)


def test_census_reports_unknown_classes_pitch_variants_and_stale_exemptions():
    plain, window = gemm_pair()
    unknown = LC.launch_class("a_kernel_nobody_knows", n=3)
    exempt = dict(CL.EXEMPT, retired_kernel=("test_kernels_gpu.py::test_gemm_epilogues", "no longer launched"))
    cen = LC.Census(CL.CHECKERS, exempt, set(vars(CL)))
    recorded = [plain, window, unknown, cls("shift_labels", torch.zeros(2, 5, dtype=torch.int32),
                                            torch.zeros(2, 5, dtype=torch.int32), 7)]
    checked, exempted, unchecked, stale = cen.classify(recorded)
    assert checked == {plain: "test_plain_gemm_classes"}
    assert set(exempted) == {recorded[3]}
    assert unchecked == [window, unknown]
    assert "retired_kernel" in stale
    # an entry:kind exemption is more specific than the entry's own
    dec = LC.launch_class("attn_decode", kind="local", rows=32, S=1280, H=4, dh=128, scale=1.0, radius=256, axial=None,
                          conv=None)
    assert cen.exemption(dec) == "attn_decode:local"


def test_deleting_a_replay_test_or_an_exemption_leaves_its_classes_unchecked():
    plain, _ = gemm_pair()
    sl = cls("shift_labels", torch.zeros(2, 5, dtype=torch.int32), torch.zeros(2, 5, dtype=torch.int32), 7)
    present = set(vars(CL)) - {"test_plain_gemm_classes"}
    _, _, unchecked, _ = LC.Census(CL.CHECKERS, CL.EXEMPT, present).classify([plain])
    assert unchecked == [plain]
    exempt = {k: v for k, v in CL.EXEMPT.items() if k != "shift_labels"}
    _, _, unchecked, _ = LC.Census(CL.CHECKERS, exempt, set(vars(CL))).classify([sl])
    assert unchecked == [sl]


def test_every_checker_names_a_test_of_the_gpu_module():
    for name, _ in CL.CHECKERS:
        assert callable(getattr(CL, name, None)), name


def test_an_exemption_covers_only_the_shapes_its_test_runs():
    cen = LC.Census(CL.CHECKERS, CL.EXEMPT, set(vars(CL)))
    dec = dict(kind="causal", rows=64, S=1280, H=4, dh=128, scale=1.0, radius=None, axial=None, conv=None)
    ok = LC.launch_class("attn_decode", **dec)
    wide = LC.launch_class("attn_decode", **dict(dec, rows=1024))
    _, exempted, unchecked, _ = cen.classify([ok, wide])
    assert set(exempted) == {ok} and unchecked == [wide]


def test_every_exemption_names_a_collected_test():
    """Each EXEMPT id (with its parameter ids, when it gives them) is a test pytest collects."""
    ids = [t for t, *_ in CL.EXEMPT.values()]
    mods = sorted({t.split("::")[0] for t in ids})
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider"] +
                         [os.path.join("tests", m) for m in mods], cwd=root, capture_output=True, text=True)
    collected = {ln.strip()[len("tests/"):] for ln in out.stdout.splitlines() if ln.startswith("tests/")}
    assert collected, out.stdout + out.stderr
    for t in ids:
        hit = t in collected if "[" in t else any(c == t or c.startswith(t + "[") for c in collected)
        assert hit, f"exemption names {t}, which pytest does not collect"
