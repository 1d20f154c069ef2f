"""Shared pieces of the float64-reference kernel tests (test_vae_kernels_gpu.py, test_dalle_kernels_gpu.py).

Each output element of a kernel must satisfy |got - ref| <= a |ref| + b absref + floor, where ref is the same operation
in float64 on the operands the kernel saw and absref the same operation on |operands|; bf16 outputs take half a bf16
ulp at |ref| in place of a |ref|.  The test modules derive their a, b and floor.
"""
import torch

DEV = "cuda"
F64 = torch.float64
NAN = float("nan")

U = 2.0 ** -24          # fp32 unit roundoff
UTC = 2.0 ** -23        # one wgmma accumulation step (the tensor core may truncate instead of rounding)


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
    print(f"[{tag}] {name}: worst err/bound {ratio:.4f}")
    assert ratio < 1.0, f"{name}: worst err/bound {ratio:.4f}"
    return ratio


def check(name, got, ref, absref, *, a=2 * U, b=0.0, bf16_out=False, floor=0.0, tag="kernels"):
    """Per element |got - ref| <= a |ref| + b absref + floor (bf16 outputs: half a bf16 ulp instead of a |ref|).
    Prints one `[tag] name: worst err/bound r` line and returns r (< 1 or the assertion fails)."""
    return report(name, worst_ratio(name, got, ref, absref, a=a, b=b, bf16_out=bf16_out, floor=floor), tag)


def nan_like(shape, dtype):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)
