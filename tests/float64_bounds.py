"""Shared pieces of the float64-reference kernel tests (test_vae_kernels_gpu.py, test_dalle_kernels_gpu.py).

Each output element of a kernel must satisfy |got - ref| <= a |ref| + b absref + floor, where ref is the same operation
in float64 on the operands the kernel saw and absref the same operation on |operands|; bf16 outputs take half a bf16
ulp at |ref| in place of a |ref|.  The test modules derive their a, b and floor.

Bounds that depend on a grid or split count read sm_count(), which follows a reservation made through reserved_sms()
as the library's launch rules do; case lines printed under a reservation start with `[reserved-sms k=<k> sm=<n>]`.
"""
import contextlib

import torch

DEV = "cuda"
F64 = torch.float64
NAN = float("nan")

U = 2.0 ** -24          # fp32 unit roundoff
UTC = 2.0 ** -23        # one wgmma accumulation step (the tensor core may truncate instead of rounding)

_RESERVED = [0]         # SMs currently reserved through reserved_sms()


def sm_count():
    """common.cu sm_count(): the device's SMs minus the current reservation (db200_set_reserved_sms), at least 16.
    Every host launch rule (persistent grids, split-K and pixel splits, LayerNorm / colsum / sqnorm grids) reads it."""
    n = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count - _RESERVED[0]
    return max(n, 16)


@contextlib.contextmanager
def reserved_sms(k):
    """Run the body with k SMs reserved, as DataParallel.begin_overlap() runs the backward of a data-parallel step;
    yields sm_count().  The reservation goes back to 0 on the way out, also when the body fails."""
    from dalle_mtf_b200 import lib as L
    L.check(L.load().db200_set_reserved_sms(k), f"set_reserved_sms({k})")
    _RESERVED[0] = k
    try:
        yield sm_count()
    finally:
        _RESERVED[0] = 0
        L.check(L.load().db200_set_reserved_sms(0), "set_reserved_sms(0)")


def reservation():
    """SMs currently reserved through reserved_sms()."""
    return _RESERVED[0]


def prefix():
    """`[reserved-sms k=<k> sm=<n>] ` while SMs are reserved, empty otherwise: the start of every case line."""
    return f"[reserved-sms k={_RESERVED[0]} sm={sm_count()}] " if _RESERVED[0] else ""


def half_ulp_bf16(x):
    """Half an ulp of bf16 at |x| (float64, x >= 0): the largest error of rounding a value of that size to bf16."""
    return torch.exp2(torch.floor(torch.log2(x.clamp_min(2.0 ** -133))) - 8)


def worst_ratio(name, got, ref, absref, *, a=2 * U, b=0.0, bf16_out=False, floor=0.0):
    """max over elements of |got - ref| / (a |ref| + b absref + floor), bf16 outputs with half a bf16 ulp instead of
    a |ref|.  Every output must be finite (outputs start as NaN, so an element never written fails here)."""
    got = got.to(F64)
    bad = (~torch.isfinite(got)).sum().item()
    assert bad == 0, f"{name}: {bad} outputs are not finite (never written over the NaN sentinel?)"
    acc = b * absref + floor
    rnd = half_ulp_bf16(ref.abs() + acc) if bf16_out else a * ref.abs()
    return ((got - ref).abs() / (rnd + acc).clamp_min(1e-300)).max().item()


def report(name, ratio, tag="kernels"):
    print(f"{prefix()}[{tag}] {name}: worst err/bound {ratio:.4f}")
    assert ratio < 1.0, f"{name}: worst err/bound {ratio:.4f}"
    return ratio


def check(name, got, ref, absref, *, a=2 * U, b=0.0, bf16_out=False, floor=0.0, tag="kernels"):
    """Per element |got - ref| <= a |ref| + b absref + floor (bf16 outputs: half a bf16 ulp instead of a |ref|).
    Prints one `[tag] name: worst err/bound r` line and returns r (< 1 or the assertion fails)."""
    return report(name, worst_ratio(name, got, ref, absref, a=a, b=b, bf16_out=bf16_out, floor=floor), tag)


def nan_like(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)
