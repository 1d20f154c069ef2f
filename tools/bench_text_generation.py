"""Cost of caption generation (DalleSampler.generate_texts), on one GPU.  Prints JSON lines:

  * device time per text position of the captured text step (step, noise, draw over the 50 258-id text window,
    caption_next_at, position advance) with no filter, top_k=64 and top_p=0.9, next to the captured image step (no
    filter, 512 image ids): 247 replays of each graph timed with CUDA events, 3 rounds, the variants alternated;
  * per-launch device time of db200_caption_next_at: 1000 launches captured in one CUDA graph, 3 rounds;
  * generate_texts captions/s from an 8-token prefix (one prefill of 8 positions, then 247 replayed text steps), per
    variant, 3 rounds alternated.
The model is the dalle_example_b200 shape (d=512, L=6, H=4, 256 text + 1024 image positions, GPT-2 vocabulary) at
random initialisation, batch 32.  Every line carries the GPU name and its power limit."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dalle_mtf_b200 import lib as L  # noqa: E402
from dalle_mtf_b200 import ops  # noqa: E402
from dalle_mtf_b200.dalle_engine import DalleEngine  # noqa: E402
from dalle_mtf_b200.sampling import DalleSampler  # noqa: E402
from tools.bench_sampling_filter import gpu_info, time_graph  # noqa: E402

ROUNDS, PREFIX, BATCH = 3, 8, 32
VARIANTS = {"none": {}, "top_k=64": {"top_k": 64}, "top_p=0.9": {"top_p": 0.9}}


def events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def replay_ms(graph, pos, first, n):
    """Device ms per replay of n replays of a step graph starting at position `first` (pos: its device position)."""
    pos.fill_(first)
    e0, e1 = events()
    e0.record()
    for _ in range(n):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    L.require_device()
    info = gpu_info()
    eng = DalleEngine(512, 6, 4, 50258, 512, 256, 1024)
    eng.init_params(0)
    TL = eng.text_seq_len
    g = torch.Generator().manual_seed(0)
    prompt = torch.full((BATCH, TL), 50257, dtype=torch.int32)
    prompt[:, :PREFIX] = torch.randint(0, 50257, (BATCH, PREFIX), generator=g)
    prompt = prompt.cuda()
    samplers = {name: DalleSampler(eng) for name in VARIANTS}
    for name, kw in VARIANTS.items():                  # captures and warms up every graph
        samplers[name].generate_texts(prompt, temperature=1.0, **kw)
    image = DalleSampler(eng)
    image.generate_graphed(prompt, temperature=1.0)
    torch.cuda.synchronize()

    n = TL - 1 - PREFIX
    step = {name: [] for name in list(VARIANTS) + ["image"]}
    for _ in range(ROUNDS):
        for name, s in samplers.items():
            step[name].append(replay_ms(s.g_text, s.t_pos, PREFIX, n))
        step["image"].append(replay_ms(image.g_sample, image.pos_dev, TL, n))
    for name, t in step.items():
        print(json.dumps({"metric": "ms_per_position", "step": "image" if name == "image" else "text",
                          "filter": "none" if name == "image" else name, "batch": BATCH, "replays": n,
                          "rounds": [round(v, 4) for v in t], "min": round(min(t), 4), **info}))

    s = samplers["none"]
    s.t_pos.fill_(PREFIX)
    graph = time_graph(lambda: ops.caption_next_at(s.t_tokens, s.t_prefix, s.t_lens, s.t_pos, TL, eng.text_vocab_size,
                                                   s.padding_id, eng.pad_base))
    us = []
    for _ in range(ROUNDS):
        e0, e1 = events()
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        us.append(e0.elapsed_time(e1) * 1000.0 / 1000)
    print(json.dumps({"metric": "us_per_launch", "kernel": "caption_next_kernel", "rows": BATCH,
                      "rounds": [round(v, 3) for v in us], "min": round(min(us), 3), **info}))
    del graph

    rate = {name: [] for name in VARIANTS}
    for _ in range(ROUNDS):
        for name, kw in VARIANTS.items():
            e0, e1 = events()
            e0.record()
            out = samplers[name].generate_texts(prompt, temperature=1.0, **kw)
            e1.record()
            torch.cuda.synchronize()
            assert out.shape == (BATCH, TL) and torch.equal(out[:, :PREFIX], prompt[:, :PREFIX])
            rate[name].append(BATCH * 1000.0 / e0.elapsed_time(e1))
    for name, r in rate.items():
        print(json.dumps({"metric": "captions_per_sec", "filter": name, "batch": BATCH, "prefix": PREFIX,
                          "rounds": [round(v, 2) for v in r], "max": round(max(r), 2), **info}))


if __name__ == "__main__":
    main()
