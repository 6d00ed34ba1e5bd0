#!/usr/bin/env python
"""Development check of the dataflow decode step (csrc/flow.cuh) on the GPU: ids/hiddens against the older one-kernel
step (CTB_NO_FLOW=1) for B = 1..4, per-step time for a sweep of replica counts, per-phase trace of CTA 0.

    python tools/flow_check.py [--steps 96] [--tokens 512]
"""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def make(env, max_batch=4, max_context=640):
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.gpt import GPT
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        es = synth_embed_state(1)
        embed = Embed(768, 626, 21178, 4).load_state_dict(es).to("cuda")
        gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
        gpt.load_state(synth_gpt_state(0))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return gpt, embed


def gen(gpt, embed, lengths, steps, greedy=True):
    from chattts_b200.processors import ArgmaxOnly, gen_logits
    from chattts_b200.prompts import synth_prompt_batch

    ids, mask, tmask = synth_prompt_batch(lengths, seed=9)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    extra = (ArgmaxOnly(exclude_eos=True),) if greedy else ()
    out = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([0.3] * 4), eos_token=625,
                            attention_mask=mask, max_new_token=steps, min_new_token=steps,
                            logits_processors=(*proc, *warp, *extra), return_hidden=True, show_tqdm=False,
                            manual_seed=1234))[-1]
    return out


def time_steps(gpt, embed, B, tokens, reps=3):
    from chattts_b200.processors import ArgmaxOnly, build_sampler_config, exp_noise, gen_logits
    from chattts_b200.prompts import synth_prompt_batch

    ids, mask, tmask = synth_prompt_batch([16] * B, seed=1)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    cfg = build_sampler_config((*proc, *warp, ArgmaxOnly(exclude_eos=True)), [0.3] * 4, 625, tokens)
    q = exp_noise(B * 4, 626, 1234).cuda()
    emb = embed(ids, tmask)
    mask_d = mask.cuda().to(torch.uint8)
    ids_out = torch.zeros(B, tokens, 4, dtype=torch.int32, device="cuda")
    for _ in range(2):
        gpt.enqueue_generate(emb, mask_d, cfg, q, tokens, False, ids_out, None)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        gpt.enqueue_generate(emb, mask_d, cfg, q, tokens, False, ids_out, None)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * tokens)  # us per emitted token-step (prefill included)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=96)
    ap.add_argument("--tokens", type=int, default=512)
    ap.add_argument("--sweep", default="1,2,4,8,16")
    ap.add_argument("--batches", default="1,2,3,4")
    a = ap.parse_args()
    from chattts_b200 import _lib

    lib = _lib.load()
    ref, embed = make({"CTB_NO_FLOW": "1"})
    new, _ = make({"CTB_FLOW_MAX_BATCH": "4"})
    ok = True
    for B in [int(x) for x in a.batches.split(",")]:
        lengths = [16, 5, 11, 9][:B]
        r = gen(ref, embed, lengths, a.steps)
        try:
            n = gen(new, embed, lengths, a.steps)
        except Exception as e:  # watchdog / launch error: report and stop
            print(f"B={B}: flow FAILED: {e}", flush=True)
            ok = False
            break
        for b in range(B):
            same = torch.equal(r.ids[b], n.ids[b])
            first = int((r.ids[b] != n.ids[b]).any(-1).float().argmax()) if not same else -1
            hd = float((r.hiddens[b] - n.hiddens[b]).abs().max())
            hd0 = float((r.hiddens[b][0] - n.hiddens[b][0]).abs().max())
            print(f"B={B} row {b}: ids_equal={same} first_diff_step={first} max|dh|={hd:.3e} step0|dh|={hd0:.3e}", flush=True)
            ok &= same
    # sampled (top-p) run too
    r = gen(ref, embed, [16, 7], 48, greedy=False)
    n = gen(new, embed, [16, 7], 48, greedy=False)
    print("top-p B=2 ids equal:", [bool(torch.equal(r.ids[b], n.ids[b])) for b in range(2)], flush=True)
    print("PARITY", "OK" if ok else "MISMATCH", flush=True)

    print(f"old k_step  B=1: {time_steps(ref, embed, 1, a.tokens):8.1f} us/step", flush=True)
    for R in [int(x) for x in a.sweep.split(",")]:
        for l2a in (0, 1):
            g, _ = make({"CTB_FLOW_R": str(R), "CTB_FLOW_MAX_BATCH": "4", "CTB_FLOW_L2_AHEAD": str(l2a)})
            t = {B: time_steps(g, embed, B, a.tokens) for B in (1, 2, 4)}
            print(f"flow R={R:2d} l2_ahead={l2a}: " + "  ".join(f"B={B}: {t[B]:7.1f} us/step" for B in t), flush=True)
            del g
            torch.cuda.empty_cache()

    # per-phase trace of CTA 0 (last step)
    tr, _ = make({"CTB_MEGA_TRACE": "1", "CTB_FLOW_R": "1", "CTB_FLOW_L2_AHEAD": os.environ.get("TRACE_L2_AHEAD", "1")})
    time_steps(tr, embed, 1, 64, reps=1)
    buf = (C.c_ulonglong * 256)()
    _lib.check(lib.ctb_gpt_debug_trace(tr._handle, buf, 256))
    t = [buf[i] for i in range(103)]
    names = ["qkv", "attn", "oproj", "gateup", "down"]
    # stamps: [0]=start, then per layer 5 stamps (after A,B,C,D,E), then final
    per = [[(t[1 + 5 * l + k] - t[5 * l + k]) for k in range(5)] for l in range(20)]
    avg = [sum(per[l][k] for l in range(2, 20)) / 18 for k in range(5)]
    print("trace ns/phase (avg layers 2..19): " + "  ".join(f"{nm}={v:.0f}" for nm, v in zip(names, avg)),
          f" layer={sum(avg):.0f}  heads={t[101] - t[100]}  total={t[101] - t[0]}", flush=True)
    print("layer0:", per[0], "layer1:", per[1], flush=True)
    # per-CTA event stamps of layer 10 (see FL_EV in flow.cuh)
    from flow_trace import flow_consts
    _, ev0, evn, words = flow_consts()
    buf2 = (C.c_ulonglong * words)()
    _lib.check(lib.ctb_gpt_debug_trace(tr._handle, buf2, words))
    import numpy as np
    ev = np.array([[buf2[ev0 + c * evn + k] for k in range(14)] for c in range(132)], dtype=np.int64)
    t0 = ev[:, 0].min()
    names = ["A.start", "X.staged", "Q.slot", "A.end", "q.arrived", "B.end", "C.merged", "O.slot", "C.end", "XO.staged",
             "D.end", "ACT.polled", "E.partial", "E.end"]
    print("layer-10 events, ns after the first CTA entered the layer: min / median / max over CTAs (0 = not recorded)")
    for k, nm in enumerate(names):
        col = ev[:, k]
        col = col[col > 0] - t0
        if len(col):
            print(f"  {k:2d} {nm:11s} n={len(col):3d}  min={col.min():6d}  med={int(np.median(col)):6d}  max={col.max():6d}  argmax_cta={int(np.argmax(ev[:, k]))}")
    ck = [int(buf2[3000 + k]) for k in range(12)]
    print("  GU (all tasks) of CTA0/warp0, cycles: wait=%d dot=%d reduce=%d silu+store=%d release=%d | stage=%d load_x=%d norm=%d" % (
        ck[1] - ck[0], ck[2] - ck[1], ck[3] - ck[2], ck[5] - ck[3], ck[6] - ck[5], ck[9] - ck[8], ck[10] - ck[9], ck[11] - ck[10]))
    print("  L2 probe (cycles per 8 dependent loads): relaxed.gpu=%d ldcg=%d volatile=%d | 8 stores issue=%d" % tuple(int(buf2[3020 + k]) for k in range(4)))
    print("  ACT poll of CTA0/warp0, cycles: enter->sentinel=%d sentinel->full=%d  iterations: sentinel=%d full=%d" % (
        int(buf2[3013]) - int(buf2[3012]), int(buf2[3014]) - int(buf2[3013]), int(buf2[3015]), int(buf2[3016])))
    print("  CTA 0:", (ev[0] - t0).tolist())
    print("  CTA 100:", (ev[100] - t0).tolist())
    print("  CTA 131:", (ev[131] - t0).tolist(), flush=True)


if __name__ == "__main__":
    main()
