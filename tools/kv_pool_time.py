#!/usr/bin/env python
"""KV pages on demand against the fixed engine, on tools/bench_continuous.py's workload; one JSON line per arm.

    python tools/kv_pool_time.py [--requests 128] [--slots 32,64] [--dtype float32,float16] [--max-context 4096]

N seeded requests (prompts of 8..128 tokens, forced lengths of 64..1024 tokens: ``bench_continuous.continuous_workload``)
through ``GPT.generate_continuous`` on a handle of ``--max-context`` tokens per slot, in five arms per (slots, dtype):
the fixed engine (every slot owns max_context tokens of pages from ``begin``), a pool as large as the fixed one (it
never suspends), and pools of 1/2, 1/4 and 1/8 of it.  Per arm: useful speech-tokens/s (the tokens the requests asked
for, host clock around work that ends in a device synchronise), the KV pool the engine holds from ``begin`` (constant
until the engine ends) and the device memory in use after ``begin`` (total - free), the peak pages mapped and their
bytes, suspensions and resumes, and per suspend / resume the device time of its copies (CUDA events around the call)
and the MB moved.  The arms are run once each after one untimed warm-up run of the first arm, and every arm's ids are
checked equal to the fixed engine's.

The last line compares the two ways of moving a slot's KV to pinned host memory for the same bytes: the engine's
``k_kv_pack`` storing straight into mapped pinned memory (from the suspensions above), against a device staging buffer:
a device-to-device copy of the same bytes (standing in for the gather into it) plus one ``cudaMemcpyAsync`` to pinned
memory, each timed with CUDA events.  The card, its power limit and SM clocks are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
    return [x.strip() for x in out.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--slots", default="32,64")
    ap.add_argument("--dtype", default="float32,float16")
    ap.add_argument("--max-context", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_pool_time: needs a CUDA device")

    from bench_continuous import continuous_workload
    from chattts_b200 import _lib
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    slot_counts = [int(x) for x in args.slots.split(",")]
    n = args.requests
    plen, tok = continuous_workload(n, seed=7)
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to(dev)
    gpt = GPT(Config().gpt, embed, device=dev, device_gpt=dev, max_batch=max(slot_counts), max_context=args.max_context)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    reqs = []
    for i, L in enumerate(plen):
        ids, _, tmask = synth_prompt_batch([L], seed=1000 + i)
        reqs.append(Request(emb=embed(ids, tmask)[0], temperature=[0.3] * 4, eos_token=625, max_new_token=tok[i],
                            min_new_token=tok[i], logits_processors=(*proc, *warp), manual_seed=5000 + i))
    useful = sum(tok)
    name, limit, sm, sm_max = card()
    pages_per_slot = -(-args.max_context // 16)
    moves = []  # (kind, bytes, ms)

    # time every suspend / resume with events around the call (both synchronise the stream before they enqueue)
    suspend, resume = EngineDevice.suspend, EngineDevice.resume

    def timed(fn, kind):
        def call(self, *a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(self, *a)
            e1.record()
            image = out if kind == "suspend" else a[1]
            moves.append((kind, image.nbytes, e0, e1))
            return out
        return call

    EngineDevice.suspend, EngineDevice.resume = timed(suspend, "suspend"), timed(resume, "resume")

    def arm(S, dtype, frac):
        flags = _lib.engine_flags(dtype)
        page = 2 * 12 * 16 * 64 * (2 if flags else 4) * 20
        fixed_pages = S * pages_per_slot
        pool = None if frac is None else int(fixed_pages * frac) * page
        moves.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = {}
        gen = gpt.generate_continuous(reqs, slots=S, return_hidden=False, dtype=dtype, kv_pool_bytes=pool)
        first = True
        for i, o in gen:
            if first:  # the engine has begun: its pool is allocated
                free, total = torch.cuda.mem_get_info(dev)
                first = False
            out[i] = o.ids[0]
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        st = gpt.last_schedule_stats
        held = fixed_pages * page * 9 // 8 if pool is None else pool  # kv_reserve keeps 1/8 head-room
        sus = [(b, a.elapsed_time(e)) for k, b, a, e in moves if k == "suspend"]
        res = [(b, a.elapsed_time(e)) for k, b, a, e in moves if k == "resume"]

        def per(xs):
            if not xs:
                return None
            ms, mb = sum(t for _, t in xs) / len(xs), sum(b for b, _ in xs) / len(xs) / 1e6
            return {"ms": round(ms, 3), "MB": round(mb, 2), "GB_per_s": round(mb / ms, 2)}

        return out, dt, {
            "slots": S, "dtype": str(dtype).replace("torch.", ""), "arm": "fixed" if frac is None else f"pool {frac:g}",
            "useful_tokens_per_s": round(useful / dt, 1), "wall_s": round(dt, 3),
            "kv_pool_GB": round(held / 1e9, 3), "device_used_GB_after_begin": round((total - free) / 1e9, 2),
            "peak_pages": st.peak_pages if pool is not None else fixed_pages,
            "peak_mapped_GB": round((st.peak_pages if pool is not None else fixed_pages) * page / 1e9, 3),
            "suspensions": st.suspensions, "resumes": st.resumes,
            "peak_host_MB": round(max(st.host_bytes, default=0) / 1e6, 1),
            "suspend": per(sus), "resume": per(res), "decode_steps": st.decode_steps,
            "card": name, "power_limit": limit, "sm_clock": sm, "sm_clock_max": sm_max}

    mapped_rates = []
    for S in slot_counts:
        for dname in args.dtype.split(","):
            dtype = getattr(torch, dname)
            arm(S, dtype, None)  # warm-up: weights, graphs, scratch
            ref = None
            for frac in (None, 1.0, 0.5, 0.25, 0.125):
                out, _, row = arm(S, dtype, frac)
                if ref is None:
                    ref = out
                row["ids_equal_fixed"] = sorted(out) == sorted(ref) and all(torch.equal(out[i], ref[i]) for i in ref)
                if row["suspend"]:
                    mapped_rates.append(row["suspend"]["GB_per_s"])
                print(json.dumps(row), flush=True)

    # the staging alternative for the same bytes: a device-to-device copy (the gather) plus one copy to pinned memory
    nbytes = 4008 * 2 * 12 * 64 * 4 * 20  # a 4,000-token fp32 slot's KV (491 MB)
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    stage = torch.empty_like(src)
    host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    d2d, d2h = [], []
    for _ in range(6):
        e[0].record()
        stage.copy_(src)
        e[1].record()
        host.copy_(stage, non_blocking=True)
        e[2].record()
        torch.cuda.synchronize()
        d2d.append(e[0].elapsed_time(e[1]))
        d2h.append(e[1].elapsed_time(e[2]))
    d2d, d2h = sorted(d2d[1:])[2], sorted(d2h[1:])[2]
    print(json.dumps({
        "staging_MB": round(nbytes / 1e6, 1), "staging_gather_ms": round(d2d, 3), "staging_d2h_ms": round(d2h, 3),
        "staging_GB_per_s": round(nbytes / 1e6 / (d2d + d2h), 2),
        "mapped_suspend_GB_per_s_range": [min(mapped_rates), max(mapped_rates)] if mapped_rates else None,
        "card": name, "power_limit": limit, "sm_clock": sm, "sm_clock_max": sm_max}), flush=True)


if __name__ == "__main__":
    main()
