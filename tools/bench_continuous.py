#!/usr/bin/env python
"""Continuous-batching benchmark: the slot engine against static batches, one JSON line.

    python tools/bench_continuous.py [--requests N] [--slots S] [--steps K] [--warmup W] [--dump-outputs DIR]

N requests (default 128), each one utterance with its own seeded prompt (8..128 tokens) and forced length (64..1024
tokens, min_new = max_new: synthetic weights have no meaningful EOS), run through the slot engine with S slots
(``GPT.generate_continuous``) and, in the same process, through the static path as consecutive S-row batches that each
run to their longest row (``GPT.generate``).  Reports useful speech-tokens/s of both arms (the tokens the requests
asked for), mean slot occupancy, the card and its power limit.  ``--steps`` = timed repeats of each arm, alternating.
``--dump-outputs DIR`` writes both arms' ids (concatenated in request order) and the lengths as DIR/<name>.npy.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def dump_outputs(path, arrays):
    import numpy as np

    if not path:
        return
    os.makedirs(path, exist_ok=True)
    for name, a in arrays.items():
        a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        np.save(os.path.join(path, name + ".npy"), a)


def gpu_card(index: int):
    """(name, power limit) of the card, read in the same process as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")[:2]]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(index), None


def continuous_workload(n: int, seed: int):
    """Seeded prompt lengths (8..128 tokens) and forced output lengths (64..1024 tokens) of n requests."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(8, 129, (n,), generator=g).tolist(), torch.randint(64, 1025, (n,), generator=g).tolist()


def run_continuous(args, local_rank: int = 0):
    """N requests (one utterance each, its own forced length) through the slot engine with S slots
    (GPT.generate_continuous) and through the static path as consecutive S-row batches, each running to its longest
    row (GPT.generate).  Both arms are timed in this run, alternating, with a host clock around work that ends in a
    device synchronise; `useful` tokens are the ones the requests asked for."""
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    n, S = args.requests, args.slots
    plen, tok = continuous_workload(n, seed=7)
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to(dev)
    gpt = GPT(Config().gpt, embed, device=dev, device_gpt=dev, max_batch=S, max_context=max(plen) + max(tok))
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    procs, temp = (*proc, *warp), [0.3] * 4
    embs = []
    for i, L in enumerate(plen):
        ids, _, tmask = synth_prompt_batch([L], seed=1000 + i)
        embs.append(embed(ids, tmask)[0])
    reqs = [Request(emb=embs[i], temperature=temp, eos_token=625, max_new_token=tok[i], min_new_token=tok[i],
                    logits_processors=procs, manual_seed=5000 + i) for i in range(n)]

    def engine_arm(rs):
        out = {i: o.ids[0] for i, o in gpt.generate_continuous(rs, slots=S, return_hidden=False)}
        torch.cuda.synchronize()
        return out, gpt.last_schedule_stats

    def static_arm(idx_all, lengths):
        out, steps = {}, 0
        for lo in range(0, len(idx_all), S):
            idx = idx_all[lo: lo + S]
            T0, mx = max(plen[i] for i in idx), max(lengths[i] for i in idx)
            emb = torch.zeros(len(idx), T0, 768, device=dev)
            mask = torch.zeros(len(idx), T0, dtype=torch.bool)
            for k, i in enumerate(idx):  # left padding, as the tokenizer batches prompts
                emb[k, T0 - plen[i]:] = embs[i]
                mask[k, T0 - plen[i]:] = True
            o = list(gpt.generate(emb, torch.zeros(len(idx), T0, 4, dtype=torch.long), temperature=torch.tensor(temp),
                                  eos_token=625, attention_mask=mask, max_new_token=mx, min_new_token=mx,
                                  logits_processors=procs, return_hidden=False, show_tqdm=False,
                                  manual_seed=5000 + lo))[-1]
            out.update({i: o.ids[k][: lengths[i]] for k, i in enumerate(idx)})
            steps += mx
        torch.cuda.synchronize()
        return out, steps

    # warm-up: both arms on a short version of the workload (graph capture, buffer growth, module loads)
    short = [min(t, 64) for t in tok]
    for _ in range(max(1, min(args.warmup, 2))):
        engine_arm([Request(emb=r.emb, temperature=temp, eos_token=625, max_new_token=64, min_new_token=64,
                            logits_processors=procs, manual_seed=r.manual_seed) for r in reqs[: 2 * S]])
        static_arm(list(range(2 * S)), short)
    useful = sum(tok)
    t_eng, t_sta = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        eng, stats = engine_arm(reqs)
        t_eng.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        sta, static_steps = static_arm(list(range(n)), tok)
        t_sta.append(time.perf_counter() - t0)
    assert all(int(eng[i].shape[0]) == tok[i] and int(sta[i].shape[0]) == tok[i] for i in range(n))
    dump_outputs(args.dump_outputs, {"engine_ids": torch.cat([eng[i] for i in range(n)]),
                                     "static_ids": torch.cat([sta[i] for i in range(n)]),
                                     "lengths": torch.tensor(tok)})
    name, limit = gpu_card(local_rank)
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    te, ts = med(t_eng), med(t_sta)
    return {
        "metric": "continuous_useful_speech_tokens_per_s", "unit": "tokens/s", "card": name, "power_limit": limit,
        "requests": n, "slots": S, "prompt_tokens": [min(plen), max(plen)], "forced_tokens": [min(tok), max(tok)],
        "useful_tokens": useful, "repeats": args.steps,
        "engine": {"tokens_per_s": round(useful / te, 1), "seconds": round(te, 3),
                   "seconds_all": [round(t, 3) for t in t_eng], "decode_steps": stats.decode_steps,
                   "admissions": stats.admissions,
                   "mean_slot_occupancy": round((useful - n) / (S * max(1, stats.decode_steps)), 4)},
        "static": {"tokens_per_s": round(useful / ts, 1), "seconds": round(ts, 3),
                   "seconds_all": [round(t, 3) for t in t_sta], "decode_steps": static_steps,
                   "mean_slot_occupancy": round(useful / (S * static_steps), 4)},
        "speedup": round(ts / te, 3),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--slots", type=int, default=32, help="engine slots = static batch rows")
    ap.add_argument("--steps", type=int, default=3, help="timed repeats of each arm")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dump-outputs", default=None, metavar="DIR")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    print(json.dumps(run_continuous(args, int(os.environ.get("LOCAL_RANK", "0")))), flush=True)


if __name__ == "__main__":
    main()
