#!/usr/bin/env python
"""Decode-step time of the slot engine, fp32 against the half-precision engine (fp16 layer weights and KV cache).

    python tools/engine_step_time.py [--slots 8,16,32] [--contexts 300,1000] [--steps 64] [--repeats 3]

For each slot count S and context T: S seeded requests with T-token prompts are admitted into an S-slot engine
(every slot running, forced lengths), then ``--steps`` decode steps are timed with CUDA events, ``--repeats`` times,
the fp32 and fp16 engines alternating.  Prints one JSON line with the median milliseconds per step of each, the card,
its power limit and SM clock read in the same run, and the bytes one step must read (layer weights + heads + KV).
"""
import argparse
import json
import os
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="8,16,32")
    ap.add_argument("--contexts", default="300,1000")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("engine_step_time: needs a CUDA device")

    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    slots = [int(x) for x in args.slots.split(",")]
    contexts = [int(x) for x in args.contexts.split(",")]
    cap = args.steps + 8
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to("cuda")
    gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=max(slots),
              max_context=max(contexts) + cap + 8)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)

    def requests(S, T):
        out = []
        for i in range(S):
            ids, _, tmask = synth_prompt_batch([T], seed=100 + i)
            out.append(Request(emb=embed(ids, tmask)[0], temperature=[0.3] * 4, eos_token=625, max_new_token=cap,
                               min_new_token=cap, logits_processors=(*proc, *warp), manual_seed=7 + i))
        return out

    def step_ms(S, T, flags):
        reqs = requests(S, T)
        dev = EngineDevice(gpt, reqs, S, cap, True, flags)
        dev.admit([(s, s) for s in range(S)])
        dev.decode(2)  # graph capture and first launches
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dev.decode(args.steps)
        b.record()
        b.synchronize()
        st = dev.status()
        assert all(s == 1 for s in st.state), "every slot must still be running in the timed window"
        return a.elapsed_time(b) / args.steps

    rows = []
    for S in slots:
        for T in contexts:
            t = {0: [], 3: []}
            for flags in (0, 3):  # warm-up of both shapes
                step_ms(S, T, flags)
            for _ in range(args.repeats):
                for flags in (0, 3):
                    t[flags].append(step_ms(S, T, flags))
            med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
            ctx = T + args.steps // 2 + 2  # mean context over the timed steps
            kv = 20 * 2 * 768 * ctx * S
            rows.append({"slots": S, "context": T, "fp32_ms": round(med[0], 4), "fp16_ms": round(med[3], 4),
                         "fp32_over_fp16": round(med[0] / med[3], 3),
                         "fp32_all": [round(x, 4) for x in t[0]], "fp16_all": [round(x, 4) for x in t[3]],
                         "bytes_fp32": 755e6 + 7.7e6 + 4 * kv, "bytes_fp16": 377.5e6 + 7.7e6 + 2 * kv})
    print(json.dumps({"metric": "engine_decode_step_ms", "card": card(), "steps": args.steps,
                      "repeats": args.repeats, "rows": rows}))


if __name__ == "__main__":
    main()
