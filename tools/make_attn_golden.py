"""Write tests/golden/gpt_attn.npz: the reference's own ``GPT.generate(return_attn=True)`` on the seeded synthetic
weights, with its Llama model switched to eager attention (the path ``output_attentions=True`` takes in the
transformers versions the reference's requirements allow; with sdpa, newer versions return no maps).

    python tools/make_attn_golden.py

Needs the reference sources (oracle/ref_import.py) and runs on the CPU.  Two cases: audio rows of ragged prompts
(left padding) and text rows.  Per case it stores the prompt lengths and seeds, the ids the reference sampled, and
each step's maps concatenated over steps: ``maps`` [L, B, H, sum of rows * cols] fp32, step 0 [T0, T0] and step i
[1, T0 + i] row-major, the layout ``GPT.generate`` returns as views."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chattts_b200.prompts import synth_prompt_batch  # noqa: E402
from chattts_b200.synth import synth_embed_state, synth_gpt_state  # noqa: E402
from oracle.ref_models import build_reference_gpt  # noqa: E402

# name: (lengths, prompt_seed, sampler_seed, steps, text)
CASES = {"audio_b3": ([5, 12, 9], 1, 42, 12, False), "text_b2": ([7, 4], 3, 7, 8, True)}


def main():
    gpt, embed = build_reference_gpt(synth_gpt_state(0), synth_embed_state(1))
    from ChatTTS.model import gen_logits

    gpt.gpt.config._attn_implementation = "eager"
    out = {}
    for name, (lengths, pseed, sseed, steps, text) in CASES.items():
        ids, mask, tmask = synth_prompt_batch(lengths, seed=pseed)
        warp, proc = gen_logits(num_code=21178 if text else 625, top_P=0.7, top_K=20,
                                repetition_penalty=1.0 if text else 1.05)
        res = next(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([0.7] if text else [0.3] * 4),
                                eos_token=21001 if text else 625, attention_mask=mask, max_new_token=steps,
                                min_new_token=0 if text else steps, logits_processors=(*proc, *warp),
                                infer_text=text, return_attn=True, show_tqdm=False, manual_seed=sseed))
        assert len(res.attentions) == steps and all(len(a) == 20 for a in res.attentions), "no eager maps"
        maps = torch.cat([torch.stack(a).flatten(3) for a in res.attentions], 3)  # [L, B, H, sum rows * cols]
        B = len(lengths)
        n = np.array([len(t) for t in res.ids])
        pad = np.full((B, steps, 4), -1, np.int64)
        for b, t in enumerate(res.ids):
            pad[b, : len(t)] = t.numpy() if t.dim() == 2 else t.numpy()[:, None]
        out.update({f"{name}_lengths": np.array(lengths), f"{name}_prompt_seed": pseed, f"{name}_sampler_seed": sseed,
                    f"{name}_steps": steps, f"{name}_ids": pad, f"{name}_n": n,
                    f"{name}_maps": maps.float().numpy()})
        print(name, "T0", ids.shape[1], "n", n.tolist(), "maps", tuple(maps.shape))
    path = os.path.join(ROOT, "tests", "golden", "gpt_attn.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
