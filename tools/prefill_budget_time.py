#!/usr/bin/env python
"""What a prefill budget buys the running slots: poll wall times of a busy slot engine while long prompts are
admitted, with the whole prompt prefilled at one poll (no budget) and in chunks of ``--budget`` columns.

    python tools/prefill_budget_time.py [--budget 1024] [--repeats 3] [--chunk 24]

A 32-slot engine (fp32, and fp16 weights + KV), driven by the engine's own scheduling loop with an open request
source.  The running requests decode 64-token prompts; after a few warm polls the arrival is submitted:
* (a) one 4,000-token prompt, 31 slots decoding;
* (b) eight 520-token prompts (the size of a voice-cloning prompt: a 10 s speaker sample is about 470 codes) arriving
  at one poll, 24 slots decoding, so that all eight find a free slot.
Each arm runs with and without the budget, the two alternating inside each repeat, engines and scenarios in turn.
Per arm: the median and worst poll wall time while the admission is in progress (from the poll that takes the
arrival to the one whose status read first shows every arrival decoding), the time the running slots lose in all
(those polls' excess over the median warm poll), and each arrival's time to its first token (submission to that
status read).  A poll's wall time runs from one status read to the next: ``--chunk`` decode steps, then the
prefill work the policy issues, ended by the status read's synchronise.  Prints one JSON line with the card, its power
limit and SM clock read in the same run; medians and min..max spreads over the repeats.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.long_prompt_time import card, spread  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefill_budget_time: needs a CUDA device")

    from chattts_b200 import _lib
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import Arrivals, EngineDevice, Request, ScheduleStats, _poll_cycles
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    cfg = Config().gpt
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to("cuda")
    gpt = GPT(cfg, embed, device="cuda", device_gpt="cuda", max_batch=32, max_context=4096)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    engines = {"fp32": 0, "fp16": _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV}
    scenarios = {"a_one_4000": (31, [4000]), "b_eight_520": (24, [520] * 8)}
    warm, cap = 4, 512

    def request(T, max_new, seed):
        ids = synth_prompt_batch([T], seed=seed)[0]
        return Request(emb=embed(ids, torch.ones(1, T, dtype=torch.bool))[0], temperature=[0.3] * 4, eos_token=625,
                       max_new_token=max_new, min_new_token=max_new, logits_processors=(*proc, *warp),
                       manual_seed=seed)

    def arm(flags, running, arrivals, budget):
        reqs = []
        src = Arrivals()
        dev = EngineDevice(gpt, reqs, 32, cap, True, flags)
        stats = ScheduleStats()
        src.submit_all([(k, request(64, cap, 700 + k)) for k in range(running)])
        polls, t_prev, t_sub, first, waiting = [], None, None, {}, None
        for n_poll, (st, polled, _) in enumerate(_poll_cycles(reqs, dev, args.chunk, stats=stats, source=src,
                                                               prefill_budget=budget)):
            t = time.perf_counter()
            if t_prev is not None:
                polls.append(t - t_prev)
            t_prev = t
            if waiting is not None:
                for s, i in enumerate(polled):
                    if i in waiting and i not in first:
                        assert st.state[s] in (_lib.SLOT_RUNNING, _lib.SLOT_FINISHED)
                        first[i] = (t - t_sub, len(polls))
                if len(first) == len(waiting):
                    break
            if n_poll == warm:
                ids = [running + k for k in range(len(arrivals))]
                waiting = set(ids)
                t_sub = time.perf_counter()
                src.submit_all([(i, request(T, 64, 900 + k)) for k, (i, T) in enumerate(zip(ids, arrivals))])
                k_sub = len(polls)  # the next poll takes them
        src.close()
        assert all(s == _lib.SLOT_RUNNING for s in dev.status().state[:running])
        base = statistics.median(polls[1:k_sub])
        busy = polls[k_sub:max(p for _, p in first.values())]
        return {"base": base * 1e3, "busy": [x * 1e3 for x in busy], "lost": sum(x - base for x in busy) * 1e3,
                "ttft": [ms * 1e3 for ms, _ in first.values()], "max_cols": max(stats.prefill_cols[k_sub:] or [0]),
                "chunks": stats.chunks}

    result = {"card_before": card(), "budget": args.budget, "chunk": args.chunk, "repeats": args.repeats,
              "slots": 32}
    raw = {}
    with torch.cuda.device(gpt.device_gpt), torch.no_grad():
        for e, flags in engines.items():  # warm every shape
            for sc, (running, arrivals) in scenarios.items():
                for b in (None, args.budget):
                    arm(flags, running, arrivals, b)
        for rep in range(args.repeats):
            for e, flags in engines.items():
                for sc, (running, arrivals) in scenarios.items():
                    for b in ((None, args.budget) if rep % 2 == 0 else (args.budget, None)):
                        raw.setdefault((e, sc, b), []).append(arm(flags, running, arrivals, b))
    out = {}
    for (e, sc, b), runs in raw.items():
        key = f"{e}/{sc}/{'budget' if b else 'whole'}"
        out[key] = {
            "running": scenarios[sc][0],
            "poll_ms_warm": spread([r["base"] for r in runs]),
            "polls_in_progress": spread([len(r["busy"]) for r in runs]),
            "poll_ms_in_progress_median": spread([statistics.median(r["busy"]) for r in runs]),
            "poll_ms_in_progress_worst": spread([max(r["busy"]) for r in runs]),
            "lost_ms_total": spread([r["lost"] for r in runs]),
            "ttft_ms_median": spread([statistics.median(r["ttft"]) for r in runs]),
            "ttft_ms_last": spread([max(r["ttft"]) for r in runs]),
            "max_prefill_cols_per_poll": max(r["max_cols"] for r in runs) if b else None,  # recorded with a budget
        }
    result["arms"] = out
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
