#!/usr/bin/env python
"""Speed of teacher-forced scoring (``GPT.score``, ctb_gpt_score) against sampling the same tokens.

    python tools/score_time.py [--repeats 5]

On the synthetic model (fp32), each arm timed with CUDA events around the call after one warm-up call of the same
shape, ``--repeats`` times:
  code32   32 rows of a 100-token prompt + 500 given codes (one call, 599 columns per row)
  long1    1 row of a 100-token prompt + 3,000 given codes (3,099 columns: the tiled attention)
  text32   32 rows of a 100-token prompt + 200 given text ids (the text head's 21,178 columns)
  gen32    generating the same 32 x 500 codes on a 32-slot fp32 slot engine, every request forced to 500 tokens
Tokens per second count given tokens (code frames of num_vq ids, or text ids).  Prints one JSON line with the
medians, every sample, and the card, its power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20)
        return [x.strip() for x in out.stdout.strip().split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0)]


def timed(fn, repeats):
    fn()  # warm-up: the same shapes as the timed calls
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("score_time: no CUDA device")
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import Request
    from chattts_b200.gpt import GPT
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    cfg = Config()
    embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                  cfg.embed.num_vq).load_state_dict(synth_embed_state(1)).to("cuda")
    gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=32, max_context=3200)
    gpt.load_state(synth_gpt_state(0))
    g = torch.Generator().manual_seed(0)
    d = cfg.gpt.hidden_size

    def prompts(n):
        return [torch.randn(100, d, generator=g).mul_(0.02).cuda() for _ in range(n)]

    def codes(n, k):
        return [torch.randint(0, 626, (k, 4), generator=g) for _ in range(n)]

    p32, c32 = prompts(32), codes(32, 500)
    p1, c1 = prompts(1), codes(1, 3000)
    t32 = [torch.randint(0, 21178, (200,), generator=g) for _ in range(32)]
    arms = {
        "code32": (lambda: gpt.score(p32, c32), 32 * 500),
        "long1": (lambda: gpt.score(p1, c1), 3000),
        "text32": (lambda: gpt.score(p32, t32, infer_text=True), 32 * 200),
    }
    reqs = [Request(emb=p, temperature=[0.7] * 4, eos_token=625, max_new_token=500, min_new_token=500, manual_seed=i)
            for i, p in enumerate(p32)]
    arms["gen32"] = (lambda: list(gpt.generate_continuous(reqs, slots=32, return_hidden=False)), 32 * 500)
    res = {"card": card(), "repeats": args.repeats}
    for name, (fn, tokens) in arms.items():
        ms = timed(fn, args.repeats)
        res[name] = {"ms_median": statistics.median(ms), "tokens": tokens,
                     "tokens_per_s": tokens / statistics.median(ms) * 1e3, "ms": ms}
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
