#!/usr/bin/env python
"""Wall time and output digests of ``Chat.infer_continuous*`` on a synthetic ``Chat``, one JSON line.

    python tools/chat_continuous_time.py [--tree DIR] [--requests N] [--paragraphs P] [--slots S] [--warmup W]
    python tools/chat_continuous_time.py --compare A.json B.json

The ``Chat`` is built as ``bench_continuous.py --paragraphs`` builds it (``synth_all`` weights, a character tokenizer)
and only public calls are timed, each with a host clock around a call that ends in a device synchronise:

* ``plain``: ``infer_continuous`` on N texts (default 128) with seeded forced lengths of 64..1024 tokens, hidden path;
* ``stream``: ``infer_continuous_stream`` on the same texts;
* ``paragraphs``: ``infer_continuous(split_text=True)`` on the P paragraphs (default 48) of ``--paragraphs``.

The engine slots and poll interval are the calls' defaults (``max_batch`` = S, default 32).  ``--tree DIR`` imports
``chattts_b200`` from another checkout (its library built), so two versions can be timed alternately on one card.
The line carries a sha256 per waveform and per text's chunk sequence; ``--compare`` checks that two lines hold the
same digests, i.e. bitwise equal outputs.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _digest(arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(str(a.shape).encode() + a.tobytes())
    return h.hexdigest()


def compare(a_path: str, b_path: str) -> int:
    a, b = (json.load(open(p)) for p in (a_path, b_path))
    bad = {arm: sum(x != y for x, y in zip(a["digests"][arm], b["digests"][arm])) +
           abs(len(a["digests"][arm]) - len(b["digests"][arm])) for arm in a["digests"]}
    print(json.dumps({"compare": [a_path, b_path], "differing_outputs": bad}), flush=True)
    return 1 if any(bad.values()) else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--paragraphs", type=int, default=48)
    ap.add_argument("--slots", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--compare", nargs=2, default=None, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    sys.path.insert(0, os.path.abspath(args.tree))
    sys.path.insert(0, os.path.join(ROOT, "tools"))

    import numpy as np
    import torch

    import chattts_b200
    from bench_continuous import _CharTokenizer, continuous_workload, gpu_card
    from chattts_b200 import Chat
    from chattts_b200.speaker import Speaker
    from chattts_b200.synth import synth_all

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    S, n = args.slots, args.requests
    _, tok = continuous_workload(n, seed=7)
    texts = [f"utterance {i} of the continuous workload." for i in range(n)]
    g = np.random.default_rng(31)  # the --paragraphs workload of bench_continuous.py
    ptexts, plens = [], []
    for k in range(args.paragraphs):
        m = int(g.integers(2, 7))
        ptexts.append(" ".join(f"sentence {j} of paragraph {k} says something." for j in range(m)))
        plens.append(int(g.integers(48, 257)))
    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=_CharTokenizer(), speaker=Speaker(768, None), device=dev,
                         max_batch=S, max_context=1280)

    def params(lengths, seed0):
        return [c.InferCodeParams(manual_seed=seed0 + i, max_new_token=L, min_new_token=L, show_tqdm=False)
                for i, L in enumerate(lengths)]

    def plain(ts, lengths):
        return {i: [w] for i, w in c.infer_continuous(ts, params_infer_code=params(lengths, 5000))}

    def stream(ts, lengths):
        out = {}
        for i, chunk, _ in c.infer_continuous_stream(ts, params_infer_code=params(lengths, 5000)):
            out.setdefault(i, []).append(chunk)
        return out

    def paragraphs(ts, lengths):
        return {i: [w] for i, w in c.infer_continuous(ts, params_infer_code=params(lengths, 900), split_text=True)}

    arms = {"plain": (plain, texts, tok), "stream": (stream, texts, tok), "paragraphs": (paragraphs, ptexts, plens)}
    for _ in range(args.warmup):
        for fn, ts, lengths in arms.values():
            fn(ts[: 2 * S], [min(L, 96) for L in lengths[: 2 * S]])
    line = {"tree": os.path.abspath(os.path.dirname(chattts_b200.__file__)), "requests": n, "slots": S,
            "forced_tokens": [min(tok), max(tok)], "paragraphs": args.paragraphs, "seconds": {}, "digests": {}}
    for name, (fn, ts, lengths) in arms.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(ts, lengths)
        torch.cuda.synchronize()
        line["seconds"][name] = round(time.perf_counter() - t0, 3)
        assert sorted(out) == list(range(len(ts))), name
        line["digests"][name] = [_digest(out[i]) for i in range(len(ts))]
    line["card"], line["power_limit"] = gpu_card(0)
    text = json.dumps(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps({k: v for k, v in line.items() if k != "digests"}), flush=True)


if __name__ == "__main__":
    main()
