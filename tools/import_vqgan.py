"""Import a taming-transformers VQGAN checkpoint as this project's VAE checkpoint.

    python tools/import_vqgan.py --model vae_vqgan_f16_16384_b200 --ckpt last.ckpt

reads a Lightning .ckpt (its "state_dict") or a bare state dict with torch.load(weights_only=True), converts it for the
config's geometry (dalle_mtf_b200.vqgan_engine.import_taming_state_dict: names "." -> "/", conv kernels OIHW -> HWIO,
taming's loss.* entries dropped) and writes model.ckpt-<step>.pt (vae/<name> tensors + global_step) under the config's
model_path, where load_vae_model, dalle_model_fn and generate_dalle.py find it.  No GPU is needed.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dalle_mtf_b200.model_fns import vqgan_geometry                                    # noqa: E402
from dalle_mtf_b200.utils import fetch_model_params, save_checkpoint                   # noqa: E402
from dalle_mtf_b200.vqgan_engine import import_taming_state_dict, load_taming_checkpoint  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--model", required=True, help="VAE config name (configs/<name>.json) or path with architecture "
                                                   "\"vqgan\"")
    ap.add_argument("--ckpt", required=True, help="taming checkpoint: Lightning .ckpt or a bare state dict")
    ap.add_argument("--step", type=int, default=0, help="global_step recorded in the written checkpoint")
    args = ap.parse_args(argv)
    params = fetch_model_params(args.model)
    if params.get("architecture") != "vqgan":
        raise SystemExit(f"{args.model}: architecture = {params.get('architecture')!r}, expected \"vqgan\"")
    geo = dict(vqgan_geometry(params, params["dataset"]["image_size"]), num_tokens=params["num_tokens"])
    try:
        named = import_taming_state_dict(load_taming_checkpoint(args.ckpt), geo)
    except ValueError as e:
        raise SystemExit(f"import_vqgan: {e}")
    state = {"vae/" + k: v for k, v in named.items()}
    state["global_step"] = int(args.step)
    path = save_checkpoint(params["model_path"], args.step, state)
    print(f"wrote {path}: {len(named)} tensors, {sum(v.numel() for v in named.values()):,} parameters")
    return path


if __name__ == "__main__":
    main()
