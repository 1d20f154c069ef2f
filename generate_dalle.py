"""Image generation from a trained DALL-E run: loads the config and checkpoints the way train_dalle.py does, samples
image tokens for each caption (optionally completing the top rows of a prompt image) and decodes them with the VAE.

    python generate_dalle.py --model dalle_example_b200 --out DIR (--captions FILE | --caption_ids FILE.npy)
        [--checkpoint PATH] [--image_prompt IMG ...] [--prompt_rows R] [--samples_per_prompt N]
        [--temperature T] [--top_k K] [--top_p P] [--guidance_scale G] [--batch_size B] [--seed S] [--gentxt]

Writes DIR/{caption:05d}_{sample:02d}.png and DIR/tokens.npy (int32 [captions * samples_per_prompt, S]: caption ids,
then image-token ids offset as in training: by text_vocab_size, or with per_position_padding by text_vocab_size +
text_seq_len, the caption's padding then shown as the per-position pad tokens the model saw).  One process, one GPU.

--gentxt (DALLE-pytorch's flag) first completes every caption with the model's text half (DalleSampler.generate_texts,
with the run's --temperature, --top_k and --top_p; the caption ends where the config's padding_id begins) and writes
DIR/captions.npy (int32 [captions, text_seq_len]) and, when the GPT-2 BPE files are available, DIR/captions.txt (one
decoded caption per line, padding dropped); the images are then drawn for the completed captions.
"""
import argparse
import math
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from dalle_mtf_b200.data_pipeline import truncate_or_pad_label
from dalle_mtf_b200.model_fns import activation_function, attention_layers, block_sparse_options, conv_kernel, \
    gated_mlp, input_embedding, layer_scale, logits_mask, rotary_emb, rotary_embedding, sandwich_norm, \
    share_input_output_emb, shared_attn_ids, shared_ff_ids, shift_tokens, stable, \
    vae_checkpoint, vae_grid_size
from dalle_mtf_b200.utils import fetch_model_params, latest_checkpoint, load_checkpoint, local_path

PADDING_ID = 50257   # GPT-2 vocabulary + <|padding|> (src/data/tokenizer_utils.py), what training pads captions with


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Sample images from a trained DALL-E checkpoint.")
    p.add_argument("--model", required=True, help="DALL-E config name (configs/NAME.json) or path to a .json file.")
    p.add_argument("--out", required=True, help="Output directory for the PNGs and tokens.npy.")
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument("--captions", help="Text file, one caption per line (needs local GPT-2 BPE files).")
    src.add_argument("--caption_ids", help=".npy file of token ids, [N, <= text_seq_len] (or [L] for one caption).")
    p.add_argument("--checkpoint", help="DALL-E checkpoint (default: the latest model.ckpt-N.pt under model_path).")
    p.add_argument("--image_prompt", nargs="+", help="Prompt image(s): one per caption, or one for all captions.")
    p.add_argument("--prompt_rows", type=int, help="Rows of the prompt image's token grid to keep (0 < R < grid side).")
    p.add_argument("--samples_per_prompt", type=int, default=1)
    p.add_argument("--temperature", type=float, default=1.0, help="0 = greedy.")
    p.add_argument("--top_k", type=int)
    p.add_argument("--top_p", type=float)
    p.add_argument("--guidance_scale", type=float,
                   help="Classifier-free guidance scale (>= 0; 1 or unset = unguided).  Needs a model trained with "
                        "caption_dropout > 0.")
    p.add_argument("--batch_size", type=int, help="Captions per sampling call (default: predict_batch_size).")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--gentxt", action="store_true",
                   help="Complete each caption with the model before drawing its images (writes captions.npy and, "
                        "with local GPT-2 BPE files, captions.txt).")
    args = p.parse_args(argv)
    if (args.image_prompt is None) != (args.prompt_rows is None):
        p.error("--image_prompt and --prompt_rows go together")
    if args.samples_per_prompt < 1:
        p.error("--samples_per_prompt must be >= 1")
    if args.batch_size is not None and args.batch_size < 1:
        p.error("--batch_size must be >= 1")
    if args.top_k is not None and args.top_k < 1:
        p.error("--top_k must be >= 1")
    if args.top_p is not None and not 0.0 < args.top_p <= 1.0:
        p.error("--top_p must lie in (0, 1]")
    if args.guidance_scale is not None and not (math.isfinite(args.guidance_scale) and args.guidance_scale >= 0):
        p.error("--guidance_scale must be a finite number >= 0")
    return args


def padding_id(params):
    """Caption id of the unconditional rows of guided sampling: the config's padding_id, else what captions are padded
    with here."""
    pad = params.get("padding_id")
    return PADDING_ID if pad is None else pad


def load_params(model):
    """The config as train_dalle.py loads it, with the VAE's config under vae_params."""
    params = fetch_model_params(model)
    if (params["model_type"] or "").lower() != "dalle":
        raise SystemExit(f"{model}: model_type {params['model_type']!r} is not a DALL-E config")
    params["vae_params"] = fetch_model_params(params["vae_model"])
    return params


def find_checkpoints(params, checkpoint=None):
    """(DALL-E checkpoint, VAE checkpoint) paths; a clear error when either is missing."""
    ckpt = checkpoint or latest_checkpoint(params["model_path"])
    if ckpt is None or not os.path.exists(local_path(ckpt)):
        raise SystemExit(f"no DALL-E checkpoint: {checkpoint or 'no model.ckpt-N.pt under ' + str(params['model_path'])}"
                         " (train with train_dalle.py or pass --checkpoint)")
    vae_ckpt = vae_checkpoint(params)
    if vae_ckpt is None or not os.path.exists(local_path(vae_ckpt)):
        where = vae_ckpt or f"no model.ckpt-N.pt under {params['vae_params']['model_path']}"
        raise SystemExit(f"no VAE checkpoint: {where} (set vae_checkpoint_path or train the VAE with train_vae_tf.py)")
    return local_path(ckpt), local_path(vae_ckpt)


def pad_captions(rows, text_seq_len, text_vocab_size, pad=PADDING_ID):
    """Captions (lists of ids) -> int32 [N, text_seq_len], padded with `pad` / truncated as in training."""
    if len(rows) == 0:
        raise SystemExit("no captions given")
    out = np.stack([truncate_or_pad_label(r, text_seq_len, pad) for r in rows])
    if out.min() < 0 or out.max() >= text_vocab_size:
        raise SystemExit(f"caption ids must lie in [0, {text_vocab_size})")
    return out


def load_caption_ids(path, text_seq_len, text_vocab_size, pad=PADDING_ID):
    ids = np.load(path)
    if ids.ndim == 1:
        ids = ids[None]
    if ids.ndim != 2 or not np.issubdtype(ids.dtype, np.integer):
        raise SystemExit(f"{path}: expected an integer array [N, <= {text_seq_len}], got {ids.dtype} {ids.shape}")
    return pad_captions(list(ids), text_seq_len, text_vocab_size, pad)


def encode_captions(lines, tokenizer, text_seq_len, text_vocab_size, pad=PADDING_ID):
    try:
        rows = [tokenizer.encode(line) for line in lines]
    except NotImplementedError as err:
        raise SystemExit(f"cannot tokenise captions ({err}); pass pre-tokenised ids with --caption_ids") from None
    return pad_captions(rows, text_seq_len, text_vocab_size, pad)


def check_caption_prefixes(captions, pad):
    """--gentxt continues each caption after its prefix (the ids before the first `pad`): an empty one has nothing to
    continue from."""
    empty = np.flatnonzero(captions[:, 0] == pad)
    if len(empty):
        raise SystemExit(f"--gentxt: caption(s) {empty.tolist()} have no ids before the padding id {pad}; give each "
                         "caption at least one token to complete")


def write_captions(out_dir, captions, pad, tokenizer=None):
    """DIR/captions.npy (int32 [N, text_seq_len]) and, with a tokenizer that decodes, DIR/captions.txt: one caption per
    line, its ids before the first `pad`."""
    np.save(os.path.join(out_dir, "captions.npy"), captions.astype(np.int32))
    if tokenizer is None or not hasattr(tokenizer, "decode"):
        return
    with open(os.path.join(out_dir, "captions.txt"), "w") as f:
        for row in captions:
            n = int(np.argmax(row == pad)) if (row == pad).any() else len(row)
            f.write(tokenizer.decode([int(i) for i in row[:n]]).replace("\n", " ") + "\n")


def token_grid_side(params):
    """Side of the VAE's token grid: image_size / 2^(group_count - 1) for the DALL-E paper's network, image_size /
    stack_factor / 2^len(convblocks) for the reference's."""
    return vae_grid_size(params["vae_params"], params["dataset"]["image_size"])


def prefix_length(params, prompt_rows):
    """Number of prompt-image tokens kept by --prompt_rows R: R whole rows of the hw x hw grid, 0 < R < hw."""
    hw = token_grid_side(params)
    if not 0 < prompt_rows < hw:
        raise SystemExit(f"--prompt_rows must lie in (0, {hw}) for a {hw}x{hw} token grid, got {prompt_rows}")
    return prompt_rows * hw


def to_uint8(img):
    """fp32 decoder output in [-1, 1] -> uint8 (values outside are clipped)."""
    return np.round(np.clip(img, -1.0, 1.0) * 127.5 + 127.5).astype(np.uint8)


def encode_image_prompts(paths, params, vae, device):
    """Image files -> VAE codes int32 [len(paths), image_seq_len] through the training input transform."""
    from dalle_mtf_b200.data_pipeline import device_stage, host_stage
    with ThreadPoolExecutor(4) as pool:
        hb = host_stage(paths, params, labeled=False, tfrecords=False, pool=pool)
    return vae.encode_tokens(device_stage(hb, params, device)).clone()


def main(argv=None):
    args = parse_args(argv)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("generate_dalle.py is a single process on one GPU; do not launch it with torchrun")
    params = load_params(args.model)
    ckpt, vae_ckpt = find_checkpoints(params, args.checkpoint)
    tl, tv, iv = params["text_seq_len"], params["text_vocab_size"], params["image_vocab_size"]
    attention_types, local_radius = attention_layers(params)    # the layer types the checkpoint was trained with
    conv_k = conv_kernel(params)
    sparse = block_sparse_options(params)              # and the block-sparse layout (not stored in the checkpoint)
    pos_scheme, per_pos, _ = input_embedding(params)   # the input embedding the checkpoint was trained with
    activation = activation_function(params)           # and its MLP nonlinearity
    gated = gated_mlp(params)                           # and whether that MLP is gated
    shift = shift_tokens(params)                        # and whether its LayerNorm outputs are token-shifted
    sandwich = sandwich_norm(params)                    # and whether its branch outputs are normalised
    scale = layer_scale(params)                         # and whether they are LayerScaled
    stab = stable(params)                               # and whether its final LayerNorm divides by the row maximum
    tied = share_input_output_emb(params)               # and whether its output projection is the embedding
    attn_ids, ff_ids = shared_attn_ids(params), shared_ff_ids(params)   # and which layers share their modules
    mask = logits_mask(params)                         # and its objective (sampling draws image ids either way)
    rotary_dim, rotary_base = rotary_embedding(params)  # and its rotary position embeddings
    # or DALLE-pytorch's rotary embedding in place of learned positions
    rot_emb = rotary_emb(params) and rotary_emb(params, token_grid_side(params) ** 2)
    # with per-position padding the captions are padded with the config's padding_id, which the sampler maps to the
    # per-position pads as training does
    # (--gentxt: a caption ends where the config's padding_id begins, the id the sampler then draws to end one)
    pad = padding_id(params) if (per_pos or args.gentxt) else PADDING_ID
    for flag, on in (("--guidance_scale", args.guidance_scale is not None), ("--gentxt", args.gentxt)):
        if on and not 0 <= padding_id(params) < tv:
            raise SystemExit(f"{flag}: padding id {padding_id(params)} outside [0, {tv}); set padding_id in the config")
    tokenizer = None
    if args.caption_ids:
        captions = load_caption_ids(args.caption_ids, tl, tv, pad)
    else:
        from dalle_mtf_b200.tokenizer import get_tokenizer
        with open(args.captions) as f:
            lines = [ln.rstrip("\n") for ln in f if ln.strip()]
        tokenizer = get_tokenizer(params["tokenizer"])
        captions = encode_captions(lines, tokenizer, tl, tv, pad)
    if args.gentxt:
        check_caption_prefixes(captions, pad)
    N = len(captions)
    n = 0
    if args.image_prompt:
        if len(args.image_prompt) not in (1, N):
            raise SystemExit(f"{len(args.image_prompt)} prompt images for {N} captions: give one per caption or one")
        n = prefix_length(params, args.prompt_rows)

    import torch
    from PIL import Image
    from dalle_mtf_b200 import lib as L
    from dalle_mtf_b200.dalle_engine import DalleEngine
    from dalle_mtf_b200.model_fns import load_vae_model
    from dalle_mtf_b200.sampling import DalleSampler

    L.require_device()
    device = torch.device("cuda", torch.cuda.current_device())
    vae, _ = load_vae_model(params, device)
    state = load_checkpoint(vae_ckpt)
    vae.load_params({k[len("vae/"):]: v for k, v in state.items() if k.startswith("vae/")})
    if vae.K < iv:
        raise SystemExit(f"VAE has {vae.K} codes but image_vocab_size is {iv}: a sampled id would index past the "
                         "codebook")
    eng = DalleEngine(params["n_embd"], params["n_layers"], params["n_heads"], tv, iv, tl, vae.image_seq_len,
                      device=device, attention_types=attention_types, local_attention_radius=local_radius,
                      conv_attention_kernel=conv_k, image_position_embedding=None if rot_emb else pos_scheme,
                      per_position_padding=per_pos, activation=activation, logits_mask=mask, rotary_dim=rotary_dim,
                      rotary_base=rotary_base, gated_mlp=gated, shift_tokens=shift, sandwich_norm=sandwich,
                      layer_scale=scale, stable=stab, share_input_output_emb=tied, shared_attn_ids=attn_ids,
                      shared_ff_ids=ff_ids, rotary_emb=rot_emb, **sparse)
    state = load_checkpoint(ckpt)
    eng.load_params({k: v for k, v in state.items()
                     if not k.endswith("/adam_m") and not k.endswith("/adam_v") and k != "global_step"})
    del state
    prefix = None
    if n:
        prefix = encode_image_prompts(args.image_prompt, params, vae, device)[:, :n]
        if len(prefix) == 1:
            prefix = prefix.expand(N, n)
    sampler = DalleSampler(eng, padding_id=padding_id(params) if (args.guidance_scale is not None or per_pos or
                                                                  args.gentxt) else None)
    torch.manual_seed(args.seed)
    rep = args.samples_per_prompt
    bs = args.batch_size or params["predict_batch_size"] or 1
    os.makedirs(args.out, exist_ok=True)
    if args.gentxt:
        captions = np.concatenate([
            sampler.generate_texts(torch.from_numpy(captions[c0:c0 + bs]).to(device), temperature=args.temperature,
                                   top_k=args.top_k, top_p=args.top_p).cpu().numpy() for c0 in range(0, N, bs)])
        if tokenizer is None:
            from dalle_mtf_b200.tokenizer import get_tokenizer
            tokenizer = get_tokenizer(params.get("tokenizer"))
        write_captions(args.out, captions, pad, tokenizer)
    all_tokens = []
    for c0 in range(0, N, bs):
        text = torch.from_numpy(captions[c0:c0 + bs]).to(device)
        pre = prefix[c0:c0 + bs].contiguous() if prefix is not None else None
        toks = sampler.complete(text, pre, samples_per_prompt=rep, temperature=args.temperature, top_k=args.top_k,
                                top_p=args.top_p, guidance_scale=args.guidance_scale)
        imgs = to_uint8(vae.decode_tokens(toks[:, tl:].contiguous(), offset=eng.image_offset).cpu().numpy())
        for j, im in enumerate(imgs):
            c, s = c0 + j // rep, j % rep
            Image.fromarray(im if im.shape[-1] == 3 else im[..., 0]).save(
                os.path.join(args.out, f"{c:05d}_{s:02d}.png"))
        all_tokens.append(toks.cpu().numpy())
    np.save(os.path.join(args.out, "tokens.npy"), np.concatenate(all_tokens).astype(np.int32))
    print(f"wrote {N * rep} images to {args.out}")


if __name__ == "__main__":
    main(sys.argv[1:])
