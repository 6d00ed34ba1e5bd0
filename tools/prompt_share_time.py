#!/usr/bin/env python
"""Shared prompts (``Request.prompt_key``) against the same requests without a key; one JSON line per measurement.

    python tools/prompt_share_time.py [--reps 3] [--parts first,serve,copy]

``first``: n = 2, 4 and 8 seeded takes of one prompt of 500, 1,500 and 4,000 tokens arrive at an idle 32-slot engine
(fixed, and paged with a pool as large as the fixed reservation).  Time until every take has its first token: a host
clock around the first poll of the scheduling policy (admissions, shares, final chunks and the status read that
synchronises the stream).  The keyed and unkeyed arms alternate, ``--reps`` times each, after one untimed warm-up
of each; every arm pair must give equal ids.

``serve``: 32 texts x 4 takes with speaker-sample prompts of 1,000..3,990 tokens (100 new tokens each) on a paged
32-slot engine whose pool is 1/4 of the fixed reservation: useful tokens/s (host clock around the whole run), peak
physical pages, peak shared pages, shares and suspensions, keyed against unkeyed, alternating.

``copy``: ``k_kv_copy``'s kernel time (torch.profiler, 20 calls) for a 4,000-token prompt on the fixed engine (fp32 and
fp16) and its achieved bandwidth, 2 x bytes copied over kernel time.

The card, its power limit and SM clocks are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parts", default="first,serve,copy")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prompt_share_time: needs a CUDA device")

    from chattts_b200 import _lib
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request, ScheduleStats, _poll_cycles, shared_prompt_cols
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    name, power, sm, sm_max = card()
    cfg = Config()
    embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                  cfg.embed.num_vq).load_state_dict(synth_embed_state(1)).to("cuda")
    CTX, S = 4096, 32
    gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=S, max_context=CTX)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    page = 2 * 12 * 16 * 64 * 4 * 20
    fixed_pages = S * -(-CTX // 16) + 1

    def prompt(T, seed):
        ids, _, tmask = synth_prompt_batch([T], seed=seed)
        return embed(ids, tmask)[0]

    def takes(emb, n, key, max_new, seed):
        return [Request(emb=emb, temperature=[0.3, 0.5, 0.7, 1.0], eos_token=625, max_new_token=max_new,
                        min_new_token=max_new, logits_processors=(*proc, *warp), manual_seed=seed,
                        noise_batch=(n, k), prompt_key=key) for k in range(n)]

    def emit(d):
        d.update(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
        print(json.dumps(d), flush=True)

    def drain(dev, gen, reqs, out):
        for _, _, ended in gen:
            for i, s, n, _ in ended:
                out[i] = dev.harvest(s, n).ids[0].cpu() if s is not None else None

    parts = args.parts.split(",")
    with torch.no_grad():
        if "first" in parts:
            for pool in (None, fixed_pages):
                for T in (500, 1500, 4000):
                    for n in (2, 4, 8):
                        emb = prompt(T, 900 + T)
                        times = {True: [], False: []}
                        ids = {}
                        for rep in range(args.reps + 1):
                            for keyed in (True, False):
                                reqs = takes(emb, n, "k" if keyed else None, 2, 77)
                                dev = EngineDevice(gpt, reqs, S, 8, False, 0, kv_pool_pages=pool)
                                stats = ScheduleStats()
                                gen = _poll_cycles(reqs, dev, 8, stats=stats)
                                torch.cuda.synchronize()
                                t0 = time.perf_counter()
                                first = next(gen)  # admissions, shares and the status read that synchronises
                                dt = time.perf_counter() - t0
                                out = {}
                                for i, s, m, _ in first[2]:
                                    out[i] = dev.harvest(s, m).ids[0].cpu()
                                drain(dev, gen, reqs, out)
                                if rep:
                                    times[keyed].append(dt * 1e3)
                                ids[keyed] = out
                                assert stats.shares == (n - 1 if keyed else 0), stats.shares
                        equal = all(torch.equal(ids[True][i], ids[False][i]) for i in range(n))
                        assert equal, (T, n)
                        emit(dict(part="first", engine="paged" if pool else "fixed", T=T, takes=n,
                                  c0=shared_prompt_cols(T), keyed_ms=[round(t, 2) for t in times[True]],
                                  unkeyed_ms=[round(t, 2) for t in times[False]],
                                  keyed_median_ms=round(statistics.median(times[True]), 2),
                                  unkeyed_median_ms=round(statistics.median(times[False]), 2), ids_equal=equal))
        if "serve" in parts:
            import random

            rnd = random.Random(3)
            texts = [(rnd.randint(1000, 3990), 5000 + t) for t in range(32)]
            embs = [prompt(T, seed) for T, seed in texts]
            quarter = (fixed_pages - 1) // 4 + 1
            res = {True: [], False: []}
            ids = {}
            for rep in range(max(2, args.reps - 1)):
                for keyed in (True, False):
                    reqs = [r for t, emb in enumerate(embs) for r in takes(emb, 4, t if keyed else None, 100, 60 + t)]
                    dev = EngineDevice(gpt, reqs, S, 100, False, 0, kv_pool_pages=quarter)
                    stats = ScheduleStats()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = {}
                    drain(dev, _poll_cycles(reqs, dev, 16, stats=stats), reqs, out)
                    dt = time.perf_counter() - t0
                    ids[keyed] = out
                    res[keyed].append(dict(tok_s=round(100 * len(reqs) / dt, 1), s=round(dt, 3),
                                           peak_pages=stats.peak_pages, peak_shared_pages=stats.peak_shared_pages,
                                           shares=stats.shares, suspensions=stats.suspensions))
            equal = all(torch.equal(ids[True][i], ids[False][i]) for i in ids[False])
            assert equal
            emit(dict(part="serve", texts=32, takes=4, pool_pages=quarter, pool_GB=round(quarter * page / 1e9, 2),
                      keyed=res[True], unkeyed=res[False], ids_equal=equal))
        if "copy" in parts:
            for flags in (0, _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV):
                T = 4000
                c0 = shared_prompt_cols(T)
                reqs = takes(prompt(T, 4), 2, "k", 8, 5)
                dev = EngineDevice(gpt, reqs, 2, 8, False, flags)
                dev.admit([(0, 0)])
                lib, h = dev.lib, gpt._handle
                for _ in range(3):  # warm-up
                    _lib.check(lib.ctb_gpt_engine_share_prompt(h, 0, 1, T, c0, dev.stream))
                    dev.cancel([1])
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(20):
                        _lib.check(lib.ctb_gpt_engine_share_prompt(h, 0, 1, T, c0, dev.stream))
                        dev.cancel([1])
                    torch.cuda.synchronize()
                us = [e.device_time for e in prof.events() if "k_kv_copy" in e.name]
                elem = 2 if flags else 4
                nbytes = 20 * (c0 // 16) * 2 * 12 * 16 * 64 * elem
                med = statistics.median(us)
                emit(dict(part="copy", kv="fp16" if flags else "fp32", T=T, c0=c0, calls=len(us),
                          kernel_us_median=round(med, 1), kernel_us_min=round(min(us), 1),
                          kernel_us_max=round(max(us), 1), bytes_copied=nbytes,
                          achieved_GBs=round(2 * nbytes / (med * 1e-6) / 1e9, 1)))


if __name__ == "__main__":
    main()
