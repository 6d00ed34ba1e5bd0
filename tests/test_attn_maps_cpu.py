"""Attention maps without a GPU: the float64 oracle (tests/attn_oracle.py) against the reference's own eager maps
(tests/golden/gpt_attn.npz, tools/make_attn_golden.py), the views ``GPT.generate(return_attn=True)`` hands out, and
the ABI entry."""
import os

import numpy as np
import pytest
import torch

from attn_oracle import oracle_maps, step_offsets
from chattts_b200 import _lib
from chattts_b200.embed import Embed
from chattts_b200.config import Config
from chattts_b200.gpt import attention_map_views
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from f64_oracle import F64Oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gpt_attn.npz")


@pytest.mark.parametrize("case,text", [("audio_b3", False), ("text_b2", True)])
def test_oracle_matches_reference_eager_maps(case, text):
    g = np.load(GOLD)
    lengths = g[f"{case}_lengths"].tolist()
    steps = int(g[f"{case}_steps"])
    ids, mask, tmask = synth_prompt_batch(lengths, seed=int(g[f"{case}_prompt_seed"]))
    cfg = Config()
    es = synth_embed_state(1)
    embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                  cfg.embed.num_vq).load_state_dict(es)
    with torch.no_grad():
        emb = embed(ids, tmask)
    orc = F64Oracle(synth_gpt_state(0), es)
    gen = [torch.from_numpy(g[f"{case}_ids"][b]) for b in range(len(lengths))]
    got = oracle_maps(orc, emb, mask, gen, g[f"{case}_n"].tolist(), steps, text)
    ref = torch.from_numpy(g[f"{case}_maps"]).double()
    assert got.shape == ref.shape
    T0 = ids.shape[1]
    # eager attention's padding: padded key columns exactly 0, padded prompt rows exactly uniform
    for b, n in enumerate(lengths):
        pad = T0 - n
        for o, r, c in step_offsets(T0, steps):
            blk = ref[:, b, :, o: o + r * c].view(ref.shape[0], -1, r, c)
            assert (blk[..., :pad] == 0).all() if r == 1 else (blk[:, :, pad:, :pad] == 0).all()
            if r > 1:
                assert (blk[:, :, :pad, :] == torch.tensor(1.0 / T0, dtype=torch.float32).double()).all()
    assert (got - ref).abs().max().item() < 2e-6


def test_views_are_the_reference_shapes_in_one_buffer():
    L, B, H, T0 = 3, 2, 4, 5
    floats = L * B * H * (T0 * T0 + (T0 + 1) + (T0 + 2))
    buf = torch.arange(floats, dtype=torch.float32)
    steps = attention_map_views(buf, L, B, H, T0, 0, 3)
    assert len(steps) == 3 and all(len(s) == L for s in steps)
    assert [tuple(s[0].shape) for s in steps] == [(B, H, T0, T0), (B, H, 1, T0 + 1), (B, H, 1, T0 + 2)]
    assert all(t.data_ptr() >= buf.data_ptr() for s in steps for t in s)  # views, no copies
    # step blocks in order, each [L, B, H, rows, cols] row-major
    assert steps[1][0][0, 0, 0, 0].item() == L * B * H * T0 * T0
    assert steps[0][1][0, 0, 0, 0].item() == B * H * T0 * T0
    later = attention_map_views(buf[L * B * H * T0 * T0:], L, B, H, T0, 1, 3)
    assert all(torch.equal(a, b) for s, t in zip(steps[1:], later) for a, b in zip(s, t))


def test_abi_entry_is_exported_and_declared():
    assert "ctb_gpt_attention_maps" in _lib.EXPORTS
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "chattts_b200.h")).read()
    assert "int ctb_gpt_attention_maps(ctb_gpt* h, int32_t B, int32_t T0, int32_t q0, int32_t n," in hdr
