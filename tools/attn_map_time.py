#!/usr/bin/env python
"""Time of the attention-map pass of ``GPT.generate(return_attn=True)`` (ctb_gpt_attention_maps) against the decode.

    python tools/attn_map_time.py [--batch 1] [--prompt 100] [--steps 512] [--chunk 24] [--repeats 3]

A seeded code run of ``--steps`` forced steps on the synthetic model: the whole run without maps (decode time), the
same run's maps computed once at the end (the non-stream pass), and the pass per stream chunk of ``--chunk`` steps
(the cost added to each ``stream=True`` yield), each timed with a host clock around work that ends in a device
synchronise, ``--repeats`` times.  Bytes written are the maps' floats x 4; their rate is set against the H100 SXM data
sheet's 3.35 TB/s.  Prints one JSON line with the medians, every sample, and the card, its power limit and SM clock
read in the same run.
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
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20)
        return [x.strip() for x in out.stdout.strip().split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--prompt", type=int, default=100)
    ap.add_argument("--steps", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_map_time: no CUDA device")
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.gpt import GPT
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    cfg = Config()
    es = synth_embed_state(1)
    embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                  cfg.embed.num_vq).load_state_dict(es).to("cuda")
    gpt = GPT(cfg.gpt, embed, max_batch=max(args.batch, 2), max_context=args.prompt + args.steps + 16)
    gpt.load_state(synth_gpt_state(0))
    ids, mask, tmask = synth_prompt_batch([args.prompt] * args.batch, seed=1)
    emb = embed(ids, tmask)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    L, H, B, T0, n = cfg.gpt.num_hidden_layers, cfg.gpt.num_attention_heads, args.batch, ids.shape[1], args.steps

    def run(return_attn):
        return list(gpt.generate(emb, ids, temperature=torch.tensor([0.3] * 4), eos_token=625, attention_mask=mask,
                                 max_new_token=n, min_new_token=n, logits_processors=(*proc, *warp),
                                 return_attn=return_attn, show_tqdm=False, manual_seed=3))[-1]

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t, r

    # the pass on the handle as a finished run leaves it (every step fed), in one call or per stream chunk
    mask_d = mask.cuda().to(torch.uint8).contiguous()
    stream = torch.cuda.current_stream().cuda_stream

    def maps(i0, i1):
        att = [None] * i0
        gpt._extend_attention_maps(att, i1, emb, mask_d, ids_out, False, stream)
        return att

    decode, whole, chunked, with_maps = [], [], [], []
    for _ in range(args.repeats + 1):
        t_dec, out = timed(lambda: run(False))
        ids_out = torch.zeros(B, n, 4, dtype=torch.int32, device="cuda")
        for b in range(B):
            ids_out[b, : len(out.ids[b])] = out.ids[b].to(torch.int32)
        t_whole, _ = timed(lambda: maps(0, n))
        per_chunk = [timed(lambda: maps(i, min(i + args.chunk, n)))[0] for i in range(args.chunk, n, args.chunk)]
        t_both, _ = timed(lambda: run(True))
        decode.append(t_dec); whole.append(t_whole); chunked.append(statistics.median(per_chunk)); with_maps.append(t_both)
    decode, whole, chunked, with_maps = decode[1:], whole[1:], chunked[1:], with_maps[1:]  # the first is warm-up
    floats = L * B * H * (T0 * T0 + sum(T0 + i for i in range(1, n)))
    chunk_floats = L * B * H * args.chunk * (T0 + n // 2)
    med = statistics.median
    print(json.dumps({
        "card": card(), "batch": B, "prompt": T0, "steps": n, "chunk": args.chunk,
        "decode_s": med(decode), "maps_whole_s": med(whole), "maps_over_decode": med(whole) / med(decode),
        "generate_with_maps_s": med(with_maps), "maps_chunk_s": med(chunked),
        "maps_bytes": 4 * floats, "maps_write_GBps": 4 * floats / med(whole) / 1e9,
        "maps_write_share_of_3.35TBps": 4 * floats / med(whole) / HBM_BYTES_PER_S,
        "chunk_write_GBps_mid_run": 4 * chunk_floats / med(chunked) / 1e9,
        "samples": {"decode": decode, "whole": whole, "chunk": chunked, "with_maps": with_maps}}))


if __name__ == "__main__":
    main()
