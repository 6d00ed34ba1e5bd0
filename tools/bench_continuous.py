#!/usr/bin/env python
"""Continuous-batching benchmark: the slot engine against static batches, one JSON line.

    python tools/bench_continuous.py [--requests N] [--slots S] [--steps K] [--warmup W] [--dump-outputs DIR] [--stream]
                                     [--dtype float16]
                                     [--refine] [--online RATE[,RATE...] [--cancel FRACTION]]
    python tools/bench_continuous.py --paragraphs N [--refine] [--slots S] [--steps K] [--warmup W]

N requests (default 128), each one utterance with its own seeded prompt (8..128 tokens) and forced length (64..1024
tokens, min_new = max_new: synthetic weights have no meaningful EOS), run through the slot engine with S slots
(``GPT.generate_continuous``) and, in the same process, through the static path as consecutive S-row batches that each
run to their longest row (``GPT.generate``).  Reports useful speech-tokens/s of both arms (the tokens the requests
asked for), mean slot occupancy, the card and its power limit.  ``--steps`` = timed repeats of each arm, alternating.
``--dump-outputs DIR`` writes both arms' ids (concatenated in request order) and the lengths as DIR/<name>.npy.
``--dtype float16`` adds a third arm, alternated with the others: the half-precision slot engine (fp16 layer weights
and KV cache) on the same requests.

``--refine`` prints one more JSON line: each request is a text-refinement stage (16..160 forced text tokens) followed by
its speech codes (the forced lengths above), through S slots, timed alternately in three arms: (a) both stages on the
engine, the speech request admitted as the request's refinement ends (``Request.then``); (b) what
``Chat.infer_continuous(skip_refine_text=False)`` does by default: static refinement in batches of S texts, then the
speech codes on the engine; (c) the speech codes alone on the engine (the first line's workload).  Per arm: wall time,
useful speech-tokens/s, decode steps, mean slot occupancy and the time from start to each request's first speech token
(p50 / p95 / max; the token is sampled by the admission's prefill and counted at the status read that follows it).

``--paragraphs N`` prints only one JSON line: N split-text paragraphs on the open engine (see ``run_paragraphs``);
with ``--refine`` every sentence is refined first, against ``Chat.infer``'s default mode (``run_paragraphs_refine``).

``--stream`` then prints a second JSON line: the same requests streamed as audio (hidden path, DVAE decoder and Vocos
from synthetic weights, InferCodeParams' default stream_batch / stream_speed / pass_first_n_batches), timed
alternately in two arms: (a) every request a streaming job of one open engine (``ChatEngine``), all submitted at once,
with one ragged ``decode_rows`` call per poll, (c) the non-streaming engine without path 2.  For (a): wall time,
useful speech-tokens/s, seconds of audio delivered per wall second, time to first chunk from admission and from start
(p50 / p95 / max), playback underruns (chunks that arrive after the request's earlier chunks have finished playing,
counted from its first chunk) and the share of wall time in path 2 (host time in ``core._decode_windows``).  With
``--dump-outputs`` the chunks of (a) are written as stream_chunks.npy (concatenated in yield order),
stream_chunk_index.npy and stream_chunk_lengths.npy.

``--online 12,24`` prints one more line per rate: the same requests streamed (hidden path, 32 slots, InferCodeParams'
defaults) but arriving over time, seeded Poisson arrivals at that many requests/s; (a) the open engine, each request
submitted at its arrival, against (b) one open engine after another, each starting every request that arrived while
the previous one ran (all submitted, then closed).  Per arm: time from arrival to first and to last chunk (p50 / p95 / max), useful tokens/s
over the span from the first arrival to the last chunk, decode steps, mean slot occupancy and underruns.  ``--cancel F``
adds a line with a seeded fraction F of the requests cancelled 0..1 s after their first chunk (open engine, highest
rate), against the same arrivals without cancellation: decode steps and span.
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


def request_job(eng, request, p, sink=None):
    """``request`` (an engine ``Request``) as one streaming job of ``eng`` (a ``ChatEngine``) with the windows of ``p``
    (``InferCodeParams``), not queued yet: ``(Job, request)`` for ``eng._enqueue``."""
    from chattts_b200.core import _Paragraph

    para = _Paragraph(1, p, sink)
    para.order[request] = 0
    para.job = eng._new_job(request, True, para)
    return para.job, request


def stream_requests(eng, requests, p):
    """Every request one streaming job of ``eng``, all queued in one step: generator of ``(position, chunk)`` as the
    chunks come, until every job has ended."""
    import queue

    out = queue.Queue()
    eng._enqueue([request_job(eng, r, p, (out, k)) for k, r in enumerate(requests)])
    left = len(requests)
    while left:
        k, item = out.get(timeout=600)
        if item is None:
            left -= 1
        else:
            yield k, item[0]


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

    def engine_arm(rs, dtype=torch.float32):
        out = {i: o.ids[0] for i, o in gpt.generate_continuous(rs, slots=S, return_hidden=False, dtype=dtype)}
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
    fp16 = args.dtype == "float16"  # a third arm: the half-precision engine on the same requests
    for _ in range(max(1, min(args.warmup, 2))):
        warm = [Request(emb=r.emb, temperature=temp, eos_token=625, max_new_token=64, min_new_token=64,
                        logits_processors=procs, manual_seed=r.manual_seed) for r in reqs[: 2 * S]]
        engine_arm(warm)
        if fp16:
            engine_arm(warm, torch.float16)
        static_arm(list(range(2 * S)), short)
    useful = sum(tok)
    t_eng, t_sta, t_e16 = [], [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        eng, stats = engine_arm(reqs)
        t_eng.append(time.perf_counter() - t0)
        if fp16:
            t0 = time.perf_counter()
            eng16, stats16 = engine_arm(reqs, torch.float16)
            t_e16.append(time.perf_counter() - t0)
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
    extra = {}
    if fp16:
        t16 = med(t_e16)
        extra = {"engine_fp16": {"tokens_per_s": round(useful / t16, 1), "seconds": round(t16, 3),
                                 "seconds_all": [round(t, 3) for t in t_e16], "decode_steps": stats16.decode_steps,
                                 "admissions": stats16.admissions,
                                 "ids_equal_to_fp32_engine": sum(torch.equal(eng16[i], eng[i]) for i in range(n))},
                 "fp16_over_fp32_engine": round(te / t16, 3)}
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
        "speedup": round(ts / te, 3), **extra,
    }


def run_stream(args, local_rank: int = 0):
    """Streamed audio on the slot engine, two arms timed alternately in this process (see the module docstring)."""
    import types

    import numpy as np

    import chattts_b200.core as core
    from chattts_b200.config import Config
    from chattts_b200.core import Chat, ChatEngine
    from chattts_b200.decoder import DVAE, Vocos
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_dvae_state, synth_embed_state, synth_gpt_state, synth_vocos_state

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    n, S, cfg = args.requests, args.slots, Config()
    plen, tok = continuous_workload(n, seed=7)
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to(dev)
    gpt = GPT(cfg.gpt, embed, device=dev, device_gpt=dev, max_batch=S, max_context=max(plen) + max(tok))
    gpt.load_state(synth_gpt_state(0))
    voc = Vocos(cfg.vocos, dev, max_batch=S, max_tokens=256).load_state_dict(synth_vocos_state(5))
    dec = DVAE(cfg.decoder, dim=cfg.decoder.idim, device=dev, vocos=voc, max_batch=S, max_tokens=256)
    dec.load_state_dict(synth_dvae_state(2, cfg.decoder, cfg.decoder.idim))
    p = Chat.InferCodeParams()
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    procs, temp = (*proc, *warp), [0.3] * 4
    embs = []
    for i, L in enumerate(plen):
        ids, _, tmask = synth_prompt_batch([L], seed=1000 + i)
        embs.append(embed(ids, tmask)[0])

    def requests(lengths):
        return [Request(emb=embs[i], temperature=temp, eos_token=625, max_new_token=lengths[i],
                        min_new_token=lengths[i], logits_processors=procs, manual_seed=5000 + i,
                        stream_batch=p.stream_batch) for i in range(len(lengths))]

    admitted = {}
    admit = EngineDevice.admit

    def timed_admit(self, batch):  # admission time of each request, for the time to first chunk
        t = time.perf_counter()
        for _, i in batch:
            admitted.setdefault(i, t)
        admit(self, batch)

    EngineDevice.admit = timed_admit
    path2 = [0.0]
    decode_windows = core._decode_windows

    def timed_windows(*a, **kw):  # the host time of each poll's path-2 work: decode and copy the audio
        t = time.perf_counter()
        out = decode_windows(*a, **kw)
        path2[0] += time.perf_counter() - t
        return out

    core._decode_windows = timed_windows
    models = types.SimpleNamespace(decoder=dec, dvae=dec)  # what ChatEngine reads of a Chat

    def stream_arm(lengths):
        admitted.clear()
        path2[0] = 0.0
        chunks, arrive = [], []
        t0 = time.perf_counter()
        with gpt._open_slot_engine(ChatEngine, S, max(lengths), True, p.stream_batch, models, True) as eng:
            for i, chunk in stream_requests(eng, requests(lengths), p):
                chunks.append((i, chunk))
                arrive.append(time.perf_counter())
        wall = time.perf_counter() - t0
        return dict(wall=wall, t0=t0, chunks=chunks, arrive=arrive, admitted=dict(admitted), path2=path2[0])

    def plain_arm(lengths):
        t0 = time.perf_counter()
        for _ in gpt.generate_continuous(requests(lengths), slots=S, return_hidden=True):
            pass
        torch.cuda.synchronize()
        return dict(wall=time.perf_counter() - t0)

    short = [min(t, 96) for t in tok[: 2 * S]]
    for _ in range(max(1, min(args.warmup, 2))):
        stream_arm(short)
        plain_arm(short)
    runs = {"a": [], "c": []}
    for _ in range(args.steps):
        runs["a"].append(stream_arm(tok))
        runs["c"].append(plain_arm(tok))
    ca = runs["a"][-1]["chunks"]
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {
            "stream_chunks": np.concatenate([c[0] for _, c in ca]) if ca else np.zeros(0, np.float32),
            "stream_chunk_index": np.array([i for i, _ in ca], dtype=np.int64),
            "stream_chunk_lengths": np.array([c.shape[1] for _, c in ca], dtype=np.int64)})
    sr = 24000.0
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    pct = lambda v, q: float(np.percentile(np.asarray(v), q)) if v else None  # noqa: E731
    useful = sum(tok)

    def summary(r):
        first, under = {}, 0
        played = {}
        for (i, c), t in zip(r["chunks"], r["arrive"]):
            if c.shape[1] == 0:
                continue
            if i not in first:
                first[i], played[i] = t, 0.0
            elif t > first[i] + played[i]:
                under += 1
            played[i] += c.shape[1] / sr
        ttfc_adm = [first[i] - r["admitted"][i] for i in first]
        ttfc_start = [first[i] - r["t0"] for i in first]
        audio = sum(c.shape[1] for _, c in r["chunks"]) / sr
        q = lambda v: {"p50": round(pct(v, 50), 4), "p95": round(pct(v, 95), 4), "max": round(max(v), 4)}  # noqa: E731
        return {"seconds": round(r["wall"], 3), "tokens_per_s": round(useful / r["wall"], 1),
                "audio_s_per_wall_s": round(audio / r["wall"], 2), "chunks": len(r["chunks"]),
                "ttfc_from_admission_s": q(ttfc_adm), "ttfc_from_start_s": q(ttfc_start), "underruns": under,
                "path2_share": round(r["path2"] / r["wall"], 4)}

    out = {"metric": "continuous_stream", "card": None, "power_limit": None, "requests": n, "slots": S,
           "stream_batch": p.stream_batch, "stream_speed": p.stream_speed,
           "pass_first_n_batches": p.pass_first_n_batches, "useful_tokens": useful, "repeats": args.steps}
    rs = runs["a"]
    out["a"] = summary(sorted(rs, key=lambda r: r["wall"])[len(rs) // 2])  # the median run
    out["a"]["seconds_all"] = [round(r["wall"], 3) for r in rs]
    tc = med([r["wall"] for r in runs["c"]])
    out["c"] = {"seconds": round(tc, 3), "tokens_per_s": round(useful / tc, 1),
                "seconds_all": [round(r["wall"], 3) for r in runs["c"]]}
    out["card"], out["power_limit"] = gpu_card(local_rank)
    EngineDevice.admit = admit
    core._decode_windows = decode_windows
    return out


def run_refine(args, local_rank: int = 0):
    """Text refinement followed by speech codes, three arms timed alternately in this process (module docstring)."""
    import numpy as np

    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.engine import EngineDevice, Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    n, S = args.requests, args.slots
    plen, tok = continuous_workload(n, seed=7)
    tlen = torch.randint(16, 161, (n,), generator=torch.Generator().manual_seed(11)).tolist()
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to(dev)
    gpt = GPT(Config().gpt, embed, device=dev, device_gpt=dev, max_batch=S, max_context=max(plen) + max(tok))
    gpt.load_state(synth_gpt_state(0))
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    cprocs, ctemp = (*proc, *warp), [0.3] * 4
    warp, proc = gen_logits(num_code=21178, top_P=0.7, top_K=20, repetition_penalty=1.0)  # RefineTextParams()
    tprocs = (*proc, *warp)
    embs = []
    for i, L in enumerate(plen):
        ids, _, tmask = synth_prompt_batch([L], seed=1000 + i)
        embs.append(embed(ids, tmask)[0])

    # synthetic weights refine to no meaningful text, so each speech stage reuses its utterance's seeded prompt: the
    # arms differ in scheduling only
    def code_req(i, lengths):
        return Request(emb=embs[i], temperature=ctemp, eos_token=625, max_new_token=lengths[i],
                       min_new_token=lengths[i], logits_processors=cprocs, manual_seed=5000 + i)

    def text_req(i, tl, lengths):
        return Request(emb=embs[i], temperature=[0.7], eos_token=21001, max_new_token=tl[i], min_new_token=tl[i],
                       logits_processors=tprocs, manual_seed=9000 + i, infer_text=True,
                       then=lambda out, i=i: code_req(i, lengths))

    first, pending = {}, []
    admit, status = EngineDevice.admit, EngineDevice.status

    def timed_admit(self, batch):  # speech requests admitted now have sampled their first token at the next status
        pending.extend(self.requests[i].manual_seed - 5000 for _, i in batch if not self.requests[i].infer_text)
        admit(self, batch)

    def timed_status(self):
        st = status(self)  # synchronises the stream: the admission's prefill and first token are done
        t = time.perf_counter()
        for k in pending:
            first.setdefault(k, t)
        pending.clear()
        return st

    EngineDevice.admit, EngineDevice.status = timed_admit, timed_status

    def engine_run(reqs, cap):
        for _ in gpt.generate_continuous(reqs, slots=S, return_hidden=False, max_new_cap=cap):
            pass
        torch.cuda.synchronize()
        return gpt.last_schedule_stats

    def arm_a(tl, lengths):  # refinement and speech on the engine
        first.clear()
        t0 = time.perf_counter()
        st = engine_run([text_req(i, tl, lengths) for i in range(len(lengths))], max(max(lengths), max(tl)))
        return dict(wall=time.perf_counter() - t0, t0=t0, first=dict(first), steps=st.decode_steps,
                    row_tokens=sum(tl) + sum(lengths) - 2 * len(lengths))

    def arm_b(tl, lengths):  # infer_continuous(skip_refine_text=False) today: static refinement, then the engine
        first.clear()
        t0 = time.perf_counter()
        steps = 0
        for lo in range(0, len(lengths), S):
            idx = list(range(lo, min(lo + S, len(lengths))))
            T0, mx = max(plen[i] for i in idx), max(tl[i] for i in idx)
            emb = torch.zeros(len(idx), T0, 768, device=dev)
            mask = torch.zeros(len(idx), T0, dtype=torch.bool)
            for k, i in enumerate(idx):
                emb[k, T0 - plen[i]:] = embs[i]
                mask[k, T0 - plen[i]:] = True
            list(gpt.generate(emb, torch.zeros(len(idx), T0, 4, dtype=torch.long), temperature=torch.tensor([0.7]),
                              eos_token=21001, attention_mask=mask, max_new_token=mx, min_new_token=mx,
                              logits_processors=tprocs, infer_text=True, show_tqdm=False, manual_seed=9000 + lo))
            steps += mx
        st = engine_run([code_req(i, lengths) for i in range(len(lengths))], max(lengths))
        # the static batches' rows count the tokens their requests asked for, decode steps their longest rows
        return dict(wall=time.perf_counter() - t0, t0=t0, first=dict(first), steps=steps + st.decode_steps,
                    row_tokens=sum(tl) + sum(lengths) - 2 * len(lengths))

    def arm_c(tl, lengths):  # the code-only engine workload of the first line
        first.clear()
        t0 = time.perf_counter()
        st = engine_run([code_req(i, lengths) for i in range(len(lengths))], max(lengths))
        return dict(wall=time.perf_counter() - t0, t0=t0, first=dict(first), steps=st.decode_steps,
                    row_tokens=sum(lengths) - len(lengths))

    arms = {"a": arm_a, "b": arm_b, "c": arm_c}
    for _ in range(max(1, min(args.warmup, 2))):
        for f in arms.values():
            f([min(t, 32) for t in tlen[: 2 * S]], [min(t, 64) for t in tok[: 2 * S]])
    runs = {k: [] for k in arms}
    for _ in range(args.steps):
        for k, f in arms.items():
            runs[k].append(f(tlen, tok))
    EngineDevice.admit, EngineDevice.status = admit, status
    useful = sum(tok)

    def summary(rs):
        r = sorted(rs, key=lambda x: x["wall"])[len(rs) // 2]  # the median run
        ft = [r["first"][i] - r["t0"] for i in range(n)]
        out = {"seconds": round(r["wall"], 3), "seconds_all": [round(x["wall"], 3) for x in rs],
               "tokens_per_s": round(useful / r["wall"], 1), "decode_steps": r["steps"],
               "mean_slot_occupancy": round(r["row_tokens"] / (S * max(1, r["steps"])), 4),
               "first_speech_token_s": {"p50": round(float(np.percentile(ft, 50)), 3),
                                        "p95": round(float(np.percentile(ft, 95)), 3), "max": round(max(ft), 3)}}
        return out

    name, limit = gpu_card(local_rank)
    out = {"metric": "continuous_refine", "card": name, "power_limit": limit, "requests": n, "slots": S,
           "text_tokens": [min(tlen), max(tlen)], "forced_tokens": [min(tok), max(tok)], "useful_tokens": useful,
           "repeats": args.steps}
    for k in arms:
        out[k] = summary(runs[k])
    out["a_over_b_speedup"] = round(out["b"]["seconds"] / out["a"]["seconds"], 3)
    return out


def run_online(args, local_rank: int = 0):
    """Requests arriving over time (seeded Poisson arrivals at each rate of ``--online``), streamed as audio: (a) the
    open engine (``GPT.open_engine`` / ``ChatEngine``: every request submitted at its arrival) against (b) what a
    server can do without it: the requests that arrived while one engine ran start together on the next one.  Arms alternate, ``--steps`` repeats each; the median run by span is reported.  One JSON line per rate,
    and with ``--cancel F`` one more: arm (a) at the highest rate with a seeded fraction F of the requests cancelled
    at a seeded time (0..1 s) after their first chunk, against the same arrivals without cancellation."""
    import threading
    import types

    import numpy as np

    from chattts_b200.config import Config
    from chattts_b200.core import Chat, ChatEngine
    from chattts_b200.decoder import DVAE, Vocos
    from chattts_b200.embed import Embed
    from chattts_b200.engine import Request
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_dvae_state, synth_embed_state, synth_gpt_state, synth_vocos_state

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    n, S, cfg = args.requests, args.slots, Config()
    plen, tok = continuous_workload(n, seed=7)
    cap = max(tok)
    embed = Embed(768, 626, 21178, 4).load_state_dict(synth_embed_state(1)).to(dev)
    gpt = GPT(cfg.gpt, embed, device=dev, device_gpt=dev, max_batch=S, max_context=max(plen) + max(tok))
    gpt.load_state(synth_gpt_state(0))
    voc = Vocos(cfg.vocos, dev, max_batch=S, max_tokens=256).load_state_dict(synth_vocos_state(5))
    dec = DVAE(cfg.decoder, dim=cfg.decoder.idim, device=dev, vocos=voc, max_batch=S, max_tokens=256)
    dec.load_state_dict(synth_dvae_state(2, cfg.decoder, cfg.decoder.idim))
    models = types.SimpleNamespace(decoder=dec, dvae=dec)  # what ChatEngine reads of a Chat
    p = Chat.InferCodeParams()
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    procs, temp = (*proc, *warp), [0.3] * 4
    embs = []
    for i, L in enumerate(plen):
        ids, _, tmask = synth_prompt_batch([L], seed=1000 + i)
        embs.append(embed(ids, tmask)[0])
    torch.cuda.synchronize()

    def request(i, lengths):
        return Request(emb=embs[i], temperature=temp, eos_token=625, max_new_token=lengths[i],
                       min_new_token=lengths[i], logits_processors=procs, manual_seed=5000 + i,
                       stream_batch=p.stream_batch)

    def arrivals(rate, count, seed):
        g = np.random.default_rng(seed)
        return np.cumsum(g.exponential(1.0 / rate, count)).tolist()

    def open_arm(at, lengths, cancel_after=None):
        """(a): each request submitted at its arrival; one consumer thread per job records its chunks."""
        chunks = {i: [] for i in range(len(at))}
        eng = gpt._open_slot_engine(ChatEngine, S, cap, True, None, models, True)
        threads, jobs = [], []
        t0 = time.perf_counter()

        def consume(i, job):
            for c, _ in job:
                chunks[i].append((time.perf_counter() - t0, c.shape[1]))
                if cancel_after is not None and i in cancel_after and len(chunks[i]) == 1:
                    threading.Timer(cancel_after[i], job.cancel).start()

        for i, a in enumerate(at):
            time.sleep(max(0.0, a - (time.perf_counter() - t0)))
            job, r = request_job(eng, request(i, lengths), p)
            eng._enqueue([(job, r)])
            jobs.append(job)
            th = threading.Thread(target=consume, args=(i, job))
            th.start()
            threads.append(th)
        for th in threads:
            th.join()
        eng.close()
        return dict(chunks=chunks, steps=eng.stats.decode_steps, cancelled=sum(j.cancelled() for j in jobs))

    def call_arm(at, lengths):
        """(b): the requests that arrived while one engine ran start together on the next one (all submitted, then
        closed)."""
        chunks = {i: [] for i in range(len(at))}
        steps, nxt = 0, 0
        t0 = time.perf_counter()
        while nxt < len(at):
            time.sleep(max(0.0, at[nxt] - (time.perf_counter() - t0)))
            now = time.perf_counter() - t0
            batch = [i for i in range(nxt, len(at)) if at[i] <= now]
            nxt = batch[-1] + 1
            with gpt._open_slot_engine(ChatEngine, S, cap, True, None, models, True) as eng:
                for k, c in stream_requests(eng, [request(i, lengths) for i in batch], p):
                    chunks[batch[k]].append((time.perf_counter() - t0, c.shape[1]))
            steps += eng.stats.decode_steps
        return dict(chunks=chunks, steps=steps, cancelled=0)

    sr = 24000.0
    pct = lambda v, q: round(float(np.percentile(np.asarray(v), q)), 4)  # noqa: E731

    def summary(r, at, lengths):
        first, done, under = [], [], 0
        for i, ch in r["chunks"].items():
            ch = [(t, m) for t, m in ch if m > 0]
            if not ch:
                continue
            first.append(ch[0][0] - at[i])
            done.append(ch[-1][0] - at[i])
            played = ch[0][1] / sr  # audio handed out before each later chunk, played from the first chunk on
            for t, m in ch[1:]:
                under += t > ch[0][0] + played
                played += m / sr
        span = max(t for ch in r["chunks"].values() for t, _ in ch) - at[0]
        useful = sum(lengths)
        q = lambda v: {"p50": pct(v, 50), "p95": pct(v, 95), "max": round(max(v), 4)}  # noqa: E731
        return {"span_s": round(span, 3), "first_chunk_s": q(first), "last_chunk_s": q(done),
                "tokens_per_s": round(useful / span, 1), "decode_steps": r["steps"],
                "mean_slot_occupancy": round((useful - len(lengths)) / (S * max(1, r["steps"])), 4),
                "underruns": under, "cancelled": r["cancelled"]}

    def median_run(rs):
        return sorted(rs, key=lambda x: x["span_s"])[len(rs) // 2]

    short = [min(t, 96) for t in tok[: 2 * S]]
    for _ in range(max(1, min(args.warmup, 2))):
        open_arm([0.0] * len(short), short)
        call_arm([0.0] * len(short), short)
    name, limit = gpu_card(local_rank)
    rates = [float(x) for x in args.online.split(",")]
    lines = []
    for k, rate in enumerate(rates):
        at = arrivals(rate, n, seed=11 + k)
        runs = {"a": [], "b": []}
        for _ in range(args.steps):
            runs["a"].append(summary(open_arm(at, tok), at, tok))
            runs["b"].append(summary(call_arm(at, tok), at, tok))
        line = {"metric": "continuous_online", "card": name, "power_limit": limit, "rate_per_s": rate,
                "requests": n, "slots": S, "useful_tokens": sum(tok), "repeats": args.steps,
                "stream_batch": p.stream_batch, "stream_speed": p.stream_speed,
                "pass_first_n_batches": p.pass_first_n_batches}
        for arm in ("a", "b"):
            line[arm] = median_run(runs[arm])
            line[arm]["span_all_s"] = [r["span_s"] for r in runs[arm]]
        lines.append(line)
    if args.cancel is not None:
        rate = max(rates)
        at = arrivals(rate, n, seed=11 + rates.index(rate))
        g = np.random.default_rng(23)
        victims = sorted(g.choice(n, int(round(args.cancel * n)), replace=False).tolist())
        after = {i: float(g.uniform(0.0, 1.0)) for i in victims}
        runs = {"cancel": [], "full": []}
        for _ in range(args.steps):
            runs["cancel"].append(summary(open_arm(at, tok, after), at, tok))
            runs["full"].append(summary(open_arm(at, tok), at, tok))
        line = {"metric": "continuous_online_cancel", "card": name, "power_limit": limit, "rate_per_s": rate,
                "requests": n, "slots": S, "cancel_fraction": args.cancel, "cancelled_requests": len(victims),
                "repeats": args.steps}
        for arm in ("cancel", "full"):
            r = median_run(runs[arm])
            line[arm] = {"span_s": r["span_s"], "decode_steps": r["decode_steps"], "cancelled": r["cancelled"],
                         "span_all_s": [x["span_s"] for x in runs[arm]]}
        lines.append(line)
    return lines


class _CharTokenizer:
    """A tokenizer stand-in for ``--paragraphs`` (the real one needs the model assets): one id per character."""
    len, break_0_ids, eos_token, spk_emb_ids = 21178, 21150, 21001, 21143

    def encode(self, text, num_vq, prompt=None, device="cpu"):
        rows = [[(ord(ch) * 37 + 11) % 20000 + 1 for ch in t] or [1] for t in text]
        P = 0 if prompt is None else int(prompt.size(1))
        T = max(len(r) for r in rows) + P
        ids = torch.zeros(len(rows), T, num_vq, dtype=torch.long)
        mask = torch.zeros(len(rows), T, dtype=torch.bool)
        for b, r in enumerate(rows):
            ids[b, T - P - len(r): T - P] = torch.tensor(r)[:, None]
            mask[b, T - P - len(r):] = True
        text_mask = mask.clone()
        if P:
            ids[:, T - P:] = prompt.t().long()[None]
            text_mask[:, T - P:] = False
        return ids.to(device), mask.to(device), text_mask.to(device)

    def decode(self, tokens):
        return ["".join(chr(97 + int(t) % 26) for t in row) for row in tokens]


def run_paragraphs(args, local_rank: int = 0):
    """Paragraphs of 2-6 sentences (seeded; each paragraph's sentences forced to one seeded length of 48..256 tokens),
    all submitted at once.  Arms, alternated, ``--steps`` repeats each: (a) ``ChatEngine.submit(split_text=True,
    stream=True)`` on one open engine of S slots; (b) the same with one lone ``encode`` per speaker sample instead of
    one ``encode_rows`` call per poll; (c) ``Chat.infer(paragraph, stream=True)`` one paragraph after another.
    Per arm (median repeat by wall time): wall time, first- and last-chunk latency per paragraph, and for (a)/(b) the
    share of the wall time spent in the speaker-sample encode (device-synchronised around each call)."""
    import numpy as np

    from chattts_b200 import Chat
    from chattts_b200.core import split_sentences
    from chattts_b200.speaker import Speaker
    from chattts_b200.synth import synth_all

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    S, n = args.slots, args.paragraphs
    g = np.random.default_rng(31)
    texts, lengths = [], []
    for k in range(n):
        m = int(g.integers(2, 7))
        texts.append(" ".join(f"sentence {j} of paragraph {k} says something." for j in range(m)))
        lengths.append(int(g.integers(48, 257)))
    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=_CharTokenizer(), speaker=Speaker(768, None), device=dev,
                         max_batch=S, max_context=1024)
    enc = c.dvae.audio_encoder
    batched = enc.encode_rows
    encode_s = [0.0]

    def timed(fn):
        def call(wavs, *a, **kw):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = fn(wavs, *a, **kw)
            torch.cuda.synchronize()
            encode_s[0] += time.perf_counter() - t
            return out
        return call

    def lone(wavs, *a, **kw):  # arm (b): what the engine would do without the ragged encode
        return [enc.encode(w) for w in wavs]

    def params(k):
        return c.InferCodeParams(manual_seed=900 + k, max_new_token=lengths[k], min_new_token=lengths[k],
                                 show_tqdm=False)

    def engine_arm(rows):
        enc.encode_rows = timed(rows)
        encode_s[0] = 0.0
        times = {k: [] for k in range(n)}
        t0 = time.perf_counter()
        try:
            with c.open_engine(slots=S, max_new_cap=max(lengths)) as eng:
                jobs = [eng.submit(t, params_infer_code=params(k), stream=True, split_text=True)
                        for k, t in enumerate(texts)]
                threads = []
                for k, job in enumerate(jobs):
                    def consume(k=k, job=job):
                        for ch, _ in job:
                            if ch.shape[1]:
                                times[k].append(time.perf_counter() - t0)
                    threads.append(threading.Thread(target=consume))
                    threads[-1].start()
                for th in threads:
                    th.join()
        finally:
            del enc.encode_rows
        return times, time.perf_counter() - t0, encode_s[0]

    def infer_arm():
        times = {k: [] for k in range(n)}
        t0 = time.perf_counter()
        for k, t in enumerate(texts):
            for ch in c.infer(t, stream=True, skip_refine_text=True, params_infer_code=params(k)):
                if ch.shape[1]:
                    times[k].append(time.perf_counter() - t0)
        return times, time.perf_counter() - t0, None

    def summary(r):
        times, wall, enc_s = r
        q = lambda v: {"p50": round(float(np.percentile(v, 50)), 4), "p95": round(float(np.percentile(v, 95)), 4),
                       "max": round(float(max(v)), 4)}  # noqa: E731
        out = {"wall_s": round(wall, 3), "first_chunk_s": q([t[0] for t in times.values() if t]),
               "last_chunk_s": q([t[-1] for t in times.values() if t])}
        if enc_s is not None:
            out["encode_s"] = round(enc_s, 4)
            out["encode_share"] = round(enc_s / wall, 4)
        return out

    import threading

    for _ in range(max(1, args.warmup)):
        engine_arm(batched)
        engine_arm(lone)
    runs = {"a": [], "b": [], "c": []}
    for _ in range(args.steps):
        runs["a"].append(summary(engine_arm(batched)))
        runs["b"].append(summary(engine_arm(lone)))
        runs["c"].append(summary(infer_arm()))
    name, limit = gpu_card(local_rank)
    line = {"metric": "continuous_paragraphs", "card": name, "power_limit": limit, "paragraphs": n, "slots": S,
            "sentences": sum(len(split_sentences(t)) for t in texts), "forced_tokens": [min(lengths), max(lengths)],
            "repeats": args.steps}
    for arm, rs in runs.items():
        line[arm] = sorted(rs, key=lambda x: x["wall_s"])[len(rs) // 2]
        line[arm]["wall_all_s"] = [x["wall_s"] for x in rs]
    return line


def run_paragraphs_refine(args, local_rank: int = 0):
    """``--paragraphs N --refine``: the paragraphs of ``run_paragraphs``, each sentence refined first (seeded, forced to
    one seeded length of 16..48 tokens per paragraph).  Arms, alternated, ``--steps`` repeats each: (a)
    ``ChatEngine.submit(split_text=True, skip_refine_text=False, max_split_batch=4, stream=True)`` on one open engine
    of S slots; (b) ``Chat.infer(paragraph, stream=True)`` with its default arguments (the same refinement and batches
    of 4 sentences), one paragraph after another.  Per arm (median repeat by wall time): wall time, first- and
    last-chunk latency per paragraph, and the host time spent building seeded Exp(1) noise (``exp_noise``)."""
    import threading

    import numpy as np

    import chattts_b200.engine as engine_mod
    import chattts_b200.gpt as gpt_mod
    from chattts_b200 import Chat
    from chattts_b200.core import split_sentences
    from chattts_b200.speaker import Speaker
    from chattts_b200.synth import synth_all

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    S, n = args.slots, args.paragraphs
    g = np.random.default_rng(31)
    texts, lengths, rlengths = [], [], []
    for k in range(n):
        m = int(g.integers(2, 7))
        texts.append(" ".join(f"sentence {j} of paragraph {k} says something." for j in range(m)))
        lengths.append(int(g.integers(48, 257)))
        rlengths.append(int(g.integers(16, 49)))
    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=_CharTokenizer(), speaker=Speaker(768, None), device=dev,
                         max_batch=S, max_context=1024)
    noise_s = [0.0]

    def timed_noise(fn):
        def call(*a, **kw):
            t = time.perf_counter()
            out = fn(*a, **kw)
            noise_s[0] += time.perf_counter() - t
            return out
        return call

    def params(k):
        return c.InferCodeParams(manual_seed=900 + k, max_new_token=lengths[k], min_new_token=lengths[k],
                                 show_tqdm=False)

    def refine(k):
        return c.RefineTextParams(manual_seed=500 + k, max_new_token=rlengths[k], min_new_token=rlengths[k],
                                  show_tqdm=False)

    def engine_arm():
        times = {k: [] for k in range(n)}
        t0 = time.perf_counter()
        cap = max(max(lengths), max(rlengths))
        with c.open_engine(slots=S, max_new_cap=cap) as eng:
            jobs = [eng.submit(t, params_infer_code=params(k), stream=True, split_text=True, skip_refine_text=False,
                               params_refine_text=refine(k), max_split_batch=4) for k, t in enumerate(texts)]
            threads = []
            for k, job in enumerate(jobs):
                def consume(k=k, job=job):
                    for ch, _ in job:
                        if ch.shape[1]:
                            times[k].append(time.perf_counter() - t0)
                threads.append(threading.Thread(target=consume))
                threads[-1].start()
            for th in threads:
                th.join()
        return times, time.perf_counter() - t0

    def infer_arm():
        times = {k: [] for k in range(n)}
        t0 = time.perf_counter()
        for k, t in enumerate(texts):
            for ch in c.infer(t, stream=True, params_refine_text=refine(k), params_infer_code=params(k)):
                if ch.shape[1]:
                    times[k].append(time.perf_counter() - t0)
        return times, time.perf_counter() - t0

    def run(arm, module):
        real = module.exp_noise
        module.exp_noise = timed_noise(real)
        noise_s[0] = 0.0
        try:
            times, wall = arm()
        finally:
            module.exp_noise = real
        q = lambda v: {"p50": round(float(np.percentile(v, 50)), 4), "p95": round(float(np.percentile(v, 95)), 4),
                       "max": round(float(max(v)), 4)}  # noqa: E731
        return {"wall_s": round(wall, 3), "first_chunk_s": q([t[0] for t in times.values() if t]),
                "last_chunk_s": q([t[-1] for t in times.values() if t]), "noise_s": round(noise_s[0], 4)}

    for _ in range(max(1, args.warmup)):
        run(engine_arm, engine_mod)
        run(infer_arm, gpt_mod)
    runs = {"a": [], "b": []}
    for _ in range(args.steps):
        runs["a"].append(run(engine_arm, engine_mod))
        runs["b"].append(run(infer_arm, gpt_mod))
    name, limit = gpu_card(local_rank)
    line = {"metric": "continuous_paragraphs_refine", "card": name, "power_limit": limit, "paragraphs": n,
            "slots": S, "sentences": sum(len(split_sentences(t)) for t in texts),
            "forced_tokens": [min(lengths), max(lengths)], "forced_refine_tokens": [min(rlengths), max(rlengths)],
            "max_split_batch": 4, "repeats": args.steps}
    for arm, rs in runs.items():
        line[arm] = sorted(rs, key=lambda x: x["wall_s"])[len(rs) // 2]
        line[arm]["wall_all_s"] = [x["wall_s"] for x in rs]
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--slots", type=int, default=32, help="engine slots = static batch rows")
    ap.add_argument("--steps", type=int, default=3, help="timed repeats of each arm")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dtype", choices=("float32", "float16"), default="float32",
                    help="float16: also time the half-precision slot engine on the same requests (a third arm)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR")
    ap.add_argument("--stream", action="store_true", help="also measure streamed audio (a second JSON line)")
    ap.add_argument("--refine", action="store_true", help="also measure refinement + speech (one more JSON line); "
                    "with --paragraphs: refine every sentence (the paragraphs line of run_paragraphs_refine)")
    ap.add_argument("--online", default=None, metavar="RATE[,RATE...]",
                    help="also measure streamed requests arriving at these rates (requests/s; one JSON line each)")
    ap.add_argument("--cancel", type=float, default=None, metavar="FRACTION",
                    help="with --online: one more line with this fraction of the requests cancelled")
    ap.add_argument("--paragraphs", type=int, default=None, metavar="N",
                    help="only measure N split-text paragraphs on the open engine (one JSON line)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.paragraphs:
        run = run_paragraphs_refine if args.refine else run_paragraphs
        print(json.dumps(run(args, rank)), flush=True)
        return
    print(json.dumps(run_continuous(args, rank)), flush=True)
    if args.stream:
        print(json.dumps(run_stream(args, rank)), flush=True)
    if args.refine:
        print(json.dumps(run_refine(args, rank)), flush=True)
    if args.online:
        for line in run_online(args, rank):
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
