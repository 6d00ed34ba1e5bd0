#!/usr/bin/env python
"""Per-edge timing of the batch-1 dataflow step k_flow<1> (csrc/flow.cuh) on the GPU.

Runs the bench workload (B = 1, 16-token prompt, greedy forced tokens) until the last step attends over about
--context keys, with CTB_MEGA_TRACE=1, and reads the per-CTA event stamps (FL_EV) of layer 10 of that step.  For every
exchange it prints when the last producer CTA had finished and when the last consumer CTA had its inputs, the spread
over CTAs, and for the weight-streaming phases how long CTAs still waited for their ring slot after the inputs were in.
Each number is the median over --reps traced runs (the global timer ticks in tens of nanoseconds to a microsecond).

    python tools/flow_trace.py [--context 300] [--reps 7] [--save DIR]

--save DIR also writes the ids and hidden states of a seeded GPT.generate at B = 2 and B = 4 (k_flow forced,
CTB_FLOW_MAX_BATCH=4, 300 steps) to DIR/flow_B2.pt and DIR/flow_B4.pt, for comparing two builds with torch.equal.
"""
import argparse
import ctypes as C
import os
import re
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from flow_check import gen, make, time_steps  # noqa: E402

HEADS = 12
# FL_EV indices (flow.cuh)
A_START, X_STAGED, Q_SLOT, A_END, Q_ARRIVED, B_END, C_MERGED, O_SLOT, C_END, XO_STAGED, D_END, ACT_POLLED, E_PARTIAL, \
    E_END, B_PARTIAL, B_STORED, GU_SLOT, D_SLOT = range(18)


def flow_consts():
    src = open(os.path.join(os.path.dirname(ROOT), "chattts_b200", "csrc", "flow.cuh")).read()
    get = lambda name: int(re.search(r"\b%s = (\d+)" % name, src).group(1))  # noqa: E731
    ev0, evn = get("FL_TR_EV"), get("FL_TR_EVN")
    return get("FL_SMAX"), ev0, evn, ev0 + 192 * evn  # FL_TR_WORDS


def one_trace(lib, tr, embed, tokens, consts):
    from chattts_b200 import _lib

    smax, ev0, evn, words = consts
    time_steps(tr, embed, 1, tokens, reps=1)
    buf = (C.c_ulonglong * words)()
    _lib.check(lib.ctb_gpt_debug_trace(tr._handle, buf, words))
    G = torch.cuda.get_device_properties(0).multi_processor_count
    ev = np.array([[buf[ev0 + c * evn + k] for k in range(18)] for c in range(G)], dtype=np.int64)
    t0 = ev[:, A_START][ev[:, A_START] > 0].min()
    ev = np.where(ev >= t0, ev - t0, -1)  # -1: not recorded in this step (or a stale stamp of an earlier one)
    return ev, min(smax, G // HEADS)


def edges(ev, S):
    """Named numbers (ns after the first CTA entered layer 10) of one trace."""
    cta = np.arange(ev.shape[0])
    unit = ev[:, B_PARTIAL] >= 0
    split = cta % S
    head = (cta // S) % HEADS
    r = {}

    def mx(k, sel=None):
        col = ev[:, k] if sel is None else ev[sel, k]
        col = col[col >= 0]
        return float(col.max()) if len(col) else float("nan")

    def spread(k, sel=None):
        col = ev[:, k] if sel is None else ev[sel, k]
        col = col[col >= 0]
        return float(col.max() - col.min()) if len(col) else float("nan")

    def late(k_slot, k_in):  # how long the CTA still waited for its weights after its inputs were staged (max over CTAs)
        ok = (ev[:, k_slot] >= 0) & (ev[:, k_in] >= 0)
        return float((ev[ok, k_slot] - ev[ok, k_in]).max()) if ok.any() else float("nan")

    r["X: prev. layer down done (last CTA)"] = mx(A_START)
    r["X: staged by QKV (last CTA)"] = mx(X_STAGED)
    r["X: spread of staging over CTAs"] = spread(X_STAGED)
    r["X: QKV weights late after staging (max CTA)"] = late(Q_SLOT, X_STAGED)
    r["QKV: stored (last CTA)"] = mx(A_END)
    r["QKV: q arrived at unit (last unit)"] = mx(Q_ARRIVED, unit)
    r["attn: last partial computed (last unit)"] = mx(B_PARTIAL, unit)
    r["attn: last partial stored (last unit)"] = mx(B_STORED, unit)
    nsplit = split[unit].max() + 1 if unit.any() else 0
    if nsplit > 1:  # per head: the split-0 unit's store after the last store of the head's other splits
        d = []
        for h in range(HEADS):
            s0 = unit & (head == h) & (split == 0)
            so = unit & (head == h) & (split > 0)
            if s0.any() and so.any():
                d.append(ev[s0, B_STORED].max() - ev[so, B_STORED].max())
        r["P: split-0 store after its head's last partial (median head)"] = float(np.median(d))
    r["AO: O-proj inputs staged (last CTA)"] = mx(C_MERGED)
    r["AO: spread of staging over CTAs"] = spread(C_MERGED)
    r["AO: O weights late after staging (max CTA)"] = late(O_SLOT, C_MERGED)
    r["P+AO: last partial computed -> O-proj inputs staged"] = r["AO: O-proj inputs staged (last CTA)"] - \
        r["attn: last partial computed (last unit)"]
    r["XO: O-proj stored (last CTA)"] = mx(C_END)
    r["XO: staged by gate/up (last CTA)"] = mx(XO_STAGED)
    r["XO: spread of staging over CTAs"] = spread(XO_STAGED)
    r["XO: gate/up weights late after staging (max CTA)"] = late(GU_SLOT, XO_STAGED)
    r["ACT: gate/up stored (last CTA)"] = mx(D_END)
    r["ACT: polled by down (last CTA)"] = mx(ACT_POLLED)
    r["ACT: spread of polling over CTAs"] = spread(ACT_POLLED)
    r["ACT: down weights late after polling (max CTA)"] = late(D_SLOT, ACT_POLLED)
    r["down: stored (last CTA) = layer end"] = mx(E_END)
    return r


def save_parity(embed, out_dir):
    gpt, _ = make({"CTB_FLOW_MAX_BATCH": "4"})
    os.makedirs(out_dir, exist_ok=True)
    for B, lengths in ((2, [16, 5]), (4, [16, 5, 11, 9])):
        o = gen(gpt, embed, lengths, 300)
        torch.save({"ids": [t.cpu() for t in o.ids], "hiddens": [t.cpu() for t in o.hiddens]},
                   os.path.join(out_dir, f"flow_B{B}.pt"))
        print(f"saved {out_dir}/flow_B{B}.pt", flush=True)
    del gpt
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--context", type=int, default=300, help="keys attended by the traced (last) step, about")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--save", default=None, help="directory for the B = 2 / 4 ids and hidden states")
    a = ap.parse_args()
    from chattts_b200 import _lib

    lib = _lib.load()
    consts = flow_consts()
    tr, embed = make({"CTB_MEGA_TRACE": "1"})
    tokens = a.context - 16
    runs = []
    for _ in range(a.reps):
        ev, S = one_trace(lib, tr, embed, tokens, consts)
        runs.append(edges(ev, S))
    print(f"k_flow<1> layer 10 at ~{a.context} keys ({S} splits per head, {int((ev[:, B_PARTIAL] >= 0).sum())} attention "
          f"units), ns after the first CTA entered the layer, median over {a.reps} runs:")
    for k in runs[0]:
        vals = [r.get(k, float("nan")) for r in runs]
        print(f"  {k:66s} {np.nanmedian(vals):8.0f}   (min {np.nanmin(vals):.0f}, max {np.nanmax(vals):.0f})", flush=True)
    del tr
    torch.cuda.empty_cache()
    if a.save:
        save_parity(embed, a.save)


if __name__ == "__main__":
    main()
