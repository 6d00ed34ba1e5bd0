#!/usr/bin/env python
"""Decode-step time of the slot engine with and without the top log-probability buffers (ctb_gpt_engine_top_logprobs).

    python tools/top_logprob_time.py [--slots 8,32,64] [--contexts 300,1000] [--tops 5,20] [--steps 64] [--repeats 3]

For each slot count S, context T, precision (fp32, fp16 weights and KV) and N: S seeded code requests with T-token
prompts are admitted into an S-slot engine (every slot running, forced lengths), then ``--steps`` decode steps are
timed with CUDA events, ``--repeats`` times, the engines without and with the buffers (top_logprobs=N) alternating.
S = 8 runs the fp32 engine on the PDL chain, 32 and 64 the wgmma step.  Prints one JSON line with the median
milliseconds per step of each arm, their ratio, every sample, and the card, its power limit and SM clock read in the
same run.  The attached arm also checks that its ids equal the other arm's.
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
    ap.add_argument("--slots", default="8,32,64")
    ap.add_argument("--contexts", default="300,1000")
    ap.add_argument("--tops", default="5,20")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("top_logprob_time: needs a CUDA device")

    from chattts_b200 import _lib
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    slots = [int(x) for x in args.slots.split(",")]
    contexts = [int(x) for x in args.contexts.split(",")]
    tops = [int(x) for x in args.tops.split(",")]
    cap = args.steps + 8
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to("cuda")
    gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=max(slots),
              max_context=max(contexts) + cap + 8)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    fp16 = _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV

    def requests(S, T):
        out = []
        for i in range(S):
            ids, _, tmask = synth_prompt_batch([T], seed=100 + i)
            out.append(Request(emb=embed(ids, tmask)[0], temperature=[0.3] * 4, eos_token=625, max_new_token=cap,
                               min_new_token=cap, logits_processors=(*proc, *warp), manual_seed=7 + i))
        return out

    def step_ms(S, T, flags, top):
        dev = EngineDevice(gpt, requests(S, T), S, cap, True, flags, top_logprobs=top)
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
        return a.elapsed_time(b) / args.steps, dev.ids_out[:, : args.steps + 3].cpu()

    rows = []
    for S in slots:
        for T in contexts:
            for flags in (0, fp16):
                for N in tops:
                    t = {0: [], N: []}
                    ids = {}
                    for top in (0, N):  # warm-up of both arms
                        step_ms(S, T, flags, top)
                    for _ in range(args.repeats):
                        for top in (0, N):
                            ms, ids[top] = step_ms(S, T, flags, top)
                            t[top].append(ms)
                    assert torch.equal(ids[0], ids[N]), (S, T, flags, N)
                    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
                    rows.append({"slots": S, "context": T, "dtype": "fp16" if flags else "fp32", "top": N,
                                 "step": "wgmma" if flags or 9 <= S <= 64 else "pdl_chain",
                                 "without_ms": round(med[0], 4), "with_ms": round(med[N], 4),
                                 "with_over_without": round(med[N] / med[0], 4),
                                 "without_all": [round(x, 4) for x in t[0]],
                                 "with_all": [round(x, 4) for x in t[N]]})
    print(json.dumps({"metric": "engine_decode_step_ms_top_logprobs", "card": card(), "steps": args.steps,
                      "repeats": args.repeats, "rows": rows}))


if __name__ == "__main__":
    main()
