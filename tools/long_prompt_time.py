#!/usr/bin/env python
"""Long prompts on the slot engine: admission time, the tiled prefill attention beside the prefill GEMMs, and the stall
a long admission causes for the running slots.  fp32 and half-precision (fp16 weights + KV) engines.

    python tools/long_prompt_time.py [--lengths 1025,2048,4000] [--repeats 5] [--out DIR]

* admission: one prompt of each length admitted alone into an idle 2-slot engine (``max_new_token`` 1, so the slot is
  free again at once), wall time around the admission call ending in a device synchronise; ``--repeats`` rounds, the
  lengths and the two engines alternating inside each round, after one warm-up round.
* split: one admission of the longest prompt under ``torch.profiler`` (a run of its own); device time per kernel
  family, divided by the 20 layers, with the attention's share of its FLOP floor (pairs x 256 FLOP x 12 heads x 20
  layers at 67 TFLOP/s FP32) and the GEMMs' (3 x their FLOP at 495 TFLOP/s TF32).
* stall: a 32-slot engine with 31 slots decoding (64-token prompts); a poll of ``--chunk`` decode steps is timed alone
  and with the admission of the longest prompt into the free slot in front of it, alternating.  The extra wall time and
  the decode steps it is worth are reported.
Prints one JSON line with the card, its power limit and SM clock read in the same run; medians and min..max spreads.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20)
        return [x.strip() for x in out.stdout.strip().split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0)]


def spread(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", default="1025,2048,4000")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=24)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_prompt_time: needs a CUDA device")

    from chattts_b200 import _lib
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    lengths = [int(x) for x in args.lengths.split(",")]
    longest = max(lengths)
    cfg = Config().gpt
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to("cuda")
    gpt = GPT(cfg, embed, device="cuda", device_gpt="cuda", max_batch=32, max_context=4096)
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    engines = {"fp32": 0, "fp16": _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV}

    def request(T, max_new, seed):
        ids = synth_prompt_batch([T], seed=seed)[0]
        return Request(emb=embed(ids, torch.ones(1, T, dtype=torch.bool))[0], temperature=[0.3] * 4, eos_token=625,
                       max_new_token=max_new, min_new_token=max_new, logits_processors=(*proc, *warp),
                       manual_seed=seed)

    def admit(dev, slot, index):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dev._admit([(slot, index)], True, False, {})
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    result = {"card": card(), "lengths": lengths, "repeats": args.repeats}

    # ---- admission wall time of single prompts
    reqs = [request(T, 1, 100 + T) for T in lengths]
    admit_ms = {k: {T: [] for T in lengths} for k in engines}
    devs = {}
    with torch.cuda.device(gpt.device_gpt):
        for rnd in range(args.repeats + 1):
            for k, flags in engines.items():
                dev = EngineDevice(gpt, reqs, 2, 8, True, flags)  # one engine per handle at a time
                for i, T in enumerate(lengths):
                    ms = admit(dev, 0, i)
                    if rnd:  # round 0 warms up every shape
                        admit_ms[k][T].append(ms)
                del dev
    result["admit_ms"] = {k: {str(T): spread(v) for T, v in d.items()} for k, d in admit_ms.items()}

    # ---- kernel split of one admission of the longest prompt
    from torch.profiler import ProfilerActivity, profile

    T = longest
    pairs = T * (T + 1) / 2
    attn_floor_ms = pairs * 256 * cfg.num_attention_heads * cfg.num_hidden_layers / 67e12 * 1e3
    d, I = cfg.hidden_size, cfg.intermediate_size
    gemm_flop = 2 * T * d * (3 * d + d + 2 * I + I) * cfg.num_hidden_layers
    gemm_floor_ms = 3 * gemm_flop / 495e12 * 1e3
    split = {}
    with torch.cuda.device(gpt.device_gpt):
        for k, flags in engines.items():
            dev = EngineDevice(gpt, [reqs[lengths.index(longest)]], 2, 8, True, flags)
            admit(dev, 0, 0)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                admit(dev, 0, 0)
            fam = {"attention": 0.0, "gemm": 0.0, "other": 0.0}
            rows = []
            for ev in prof.key_averages():
                us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                if us <= 0:
                    continue
                rows.append((ev.key, us, ev.count))
                f = "attention" if "prefill_attn" in ev.key else "gemm" if "k_tc_gemm" in ev.key else "other"
                fam[f] += us / 1e3
            split[k] = {
                "attention_ms": round(fam["attention"], 3), "gemm_ms": round(fam["gemm"], 3),
                "other_ms": round(fam["other"], 3),
                "attention_ms_per_layer": round(fam["attention"] / cfg.num_hidden_layers, 4),
                "gemm_ms_per_layer": round(fam["gemm"] / cfg.num_hidden_layers, 4),
                "attention_share_of_floor": round(attn_floor_ms / fam["attention"], 3) if fam["attention"] else None,
                "gemm_share_of_floor": round(gemm_floor_ms / fam["gemm"], 3) if fam["gemm"] else None,
            }
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, f"long_prompt_kernels_{k}.txt"), "w") as f:
                    for name, us, cnt in sorted(rows, key=lambda r: -r[1]):
                        f.write(f"{us / 1e3:10.3f} ms  {cnt:6d}  {name}\n")
            del dev
    result["split"] = split
    result["floors_ms"] = {"attention_fp32": round(attn_floor_ms, 3), "gemm_3xtf32": round(gemm_floor_ms, 3)}

    # ---- decode stall of a 32-slot engine when the longest prompt is admitted
    stall = {}
    steps = args.chunk
    rounds = args.repeats * 2
    max_new = (rounds + 2) * 2 * steps + 64
    running = [request(64, max_new, 700 + i) for i in range(31)]
    with torch.cuda.device(gpt.device_gpt):
        for k, flags in engines.items():
            rs = running + [request(longest, 1, 900)]
            dev = EngineDevice(gpt, rs, 32, max_new, True, flags)
            dev._admit([(s, s) for s in range(31)], True, False, {})
            dev.decode(2 * steps)
            admit(dev, 31, 31)  # warm the long shape
            base, withp = [], []
            for rnd in range(rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dev.decode(steps)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                dev._admit([(31, 31)], True, False, {})
                dev.decode(steps)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                base.append((t1 - t0) * 1e3)
                withp.append((t2 - t1) * 1e3)
            st = dev.status()
            assert all(s == _lib.SLOT_RUNNING for s in st.state[:31]), st.state
            b, w = statistics.median(base), statistics.median(withp)
            stall[k] = {"poll_ms": spread(base), "poll_with_admission_ms": spread(withp),
                        "extra_ms": round(w - b, 3), "step_ms": round(b / steps, 4),
                        "equivalent_steps": round((w - b) / (b / steps), 1)}
            del dev
    result["stall"] = {"slots": 32, "running": 31, "chunk": steps, **stall}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
