"""DALL-E training entry point — same flags and config surface as the reference's train_dalle.py
(--tpu --gpu_ids --model --new; configs/*.json with the same keys), CUDA engine underneath.

Launch one process per GPU:   python train_dalle.py --model dalle_example_b200
                              torchrun --nproc-per-node 8 --master-addr 127.0.0.1 train_dalle.py --model ...
"""
import argparse
from functools import partial

from src.utils import *  # noqa: F401,F403  (same import surface as the reference)
from src.model_fns import dalle_model_fn
from src.input_fns import dalle_input_fn
from src.data import get_tokenizer
from dalle_mtf_b200.estimator import Estimator
from dalle_mtf_b200.dist import DataParallel


def parse_args():
    parser = argparse.ArgumentParser()
    parser.add_argument("--tpu", type=str, help="Accepted for compatibility; there is no TPU path (ignored).")
    parser.add_argument("--gpu_ids", nargs="+", type=str, default=["device:GPU:0"],
                        help="Accepted for compatibility; GPUs are chosen by the launcher (one process per GPU).")
    parser.add_argument("--model", type=str, default=None, help="JSON file that contains model parameters.")
    parser.add_argument("--new", action="store_true", help="If set, deletes previous checkpoint, if it exists, and "
                                                           "starts a new training run")
    args = parser.parse_args()
    assert args.model is not None, "Model must be set"
    return args


def main():
    args = parse_args()
    logging = setup_logging(args)
    params = fetch_model_params(args.model)
    params["vae_params"] = fetch_model_params(params["vae_model"])
    assert params["model_type"].lower() == "dalle", f'model_type {params["model_type"]} not recognized'
    dp = DataParallel().init()
    params["_dp"] = dp

    if args.new and dp.rank == 0:
        maybe_remove_gs_or_filepath(params["model_path"])
    dp.barrier()

    current_step = int(load_global_step_from_checkpoint_dir(params["model_path"]))
    logging.info(f"Current step: {current_step}")

    mesh, _ = parse_mesh(params["mesh_shape"], params["layout"])
    params["num_cores"] = dp.world
    params["use_tpu"] = False
    params["gpu_ids"] = args.gpu_ids
    tokenizer = get_tokenizer(params["tokenizer"])
    assert len(tokenizer) == params["text_vocab_size"], \
        f"tokenizer vocab size {len(tokenizer)} must equal model vocab size {params['text_vocab_size']}"
    params["padding_id"] = tokenizer.pad_token_id

    estimator = Estimator(model_fn=dalle_model_fn, params=params, logger=logging)
    has_predict_or_eval_steps = params["predict_steps"] > 0 or params["eval_steps"] > 0
    if has_predict_or_eval_steps:
        while current_step < params["train_steps"]:
            next_checkpoint = min(current_step + params["steps_per_checkpoint"], params["train_steps"])
            estimator.train(input_fn=partial(dalle_input_fn, eval=False), max_steps=next_checkpoint)
            current_step = next_checkpoint
            if params["predict_steps"] > 0:
                raise NotImplementedError
            if params["eval_steps"] > 0:
                estimator.evaluate(input_fn=partial(dalle_input_fn, eval=True), steps=params["eval_steps"])
        return
    while current_step < params["train_steps"]:
        spec = estimator.train(input_fn=partial(dalle_input_fn, eval=False), max_steps=params["train_steps"])
        current_step = spec.global_step
    dp.shutdown()


if __name__ == "__main__":
    main()
