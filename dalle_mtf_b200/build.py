"""In-tree build of libdalle_b200.so with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))


def build(verbose=False, jobs=8):
    csrc = os.path.join(_HERE, "csrc")
    cmd = ["make", "-C", csrc, f"-j{jobs}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout)
    if r.returncode != 0:
        raise RuntimeError("building libdalle_b200.so failed (see output above)")
    path = os.path.join(_HERE, "libdalle_b200.so")
    if not os.path.exists(path):
        raise RuntimeError(f"{path} missing after build")
    return path
