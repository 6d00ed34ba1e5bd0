"""Attention maps of ``GPT.generate(return_attn=True)`` in float64, teacher-forced on the ids a run produced.

For each row, ONE causal pass of ``F64Oracle`` over the row's valid prompt embeddings followed by the embeddings of
the ids it fed (positions 0 .. its last query) gives every layer's Q and K; softmax(Q K^T / 8) over the causal keys is
then placed where the reference's eager attention puts it: key column = position + the row's left padding, padded key
columns 0, padded prompt rows uniform (1 / T0), and the steps after the row's end 0.  The layout is the packed one of
``pack_maps``: [L, B, H, sum over steps of rows * cols], step 0 [T0, T0] then step i [1, T0 + i], row-major."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def pack_maps(attentions) -> torch.Tensor:
    """``GenerationOutputs.attentions`` (a list of per-step tuples of [B, H, rows, cols]) -> [L, B, H, S]."""
    return torch.cat([torch.stack(a).flatten(3) for a in attentions], 3)


def step_offsets(T0: int, steps: int):
    """(offset, rows, cols) of each step's block along the packed axis."""
    out, off = [], 0
    for i in range(steps):
        r, c = (T0, T0) if i == 0 else (1, T0 + i)
        out.append((off, r, c))
        off += r * c
    return out


@torch.no_grad()
def oracle_maps(orc, prompt_emb: torch.Tensor, mask: torch.Tensor, ids, end, steps: int, infer_text: bool):
    """Packed maps [L, B, H, S] (float64, on the oracle's device) of a run of ``steps`` steps over the prompt
    embeddings ``prompt_emb`` [B, T0, d] with left-padding ``mask`` [B, T0], whose rows sampled ``ids[b]`` ([n] text
    or [n, num_vq] codes) and ended at ``end[b]`` (the ``end_idx`` of the outputs: steps > end[b] are 0)."""
    B, T0 = int(prompt_emb.shape[0]), int(prompt_emb.shape[1])
    offs = step_offsets(T0, steps)
    out = torch.zeros(orc.L, B, orc.H, offs[-1][0] + offs[-1][1] * offs[-1][2], dtype=torch.float64, device=orc.device)
    for b in range(B):
        pad = T0 - int(mask[b].sum())
        fed = min(int(end[b]), steps - 1)  # generated ids fed as queries: steps 1 .. fed
        g = ids[b][:fed].to(orc.device).long()
        if infer_text:
            gen = F.embedding(g if g.dim() == 1 else g[:, 0], orc.emb_text)
        else:
            gen = orc.embed_codes(g) if fed else g.new_zeros(0, orc.emb_text.shape[1], dtype=orc.dtype)
        x = torch.cat([prompt_emb[b, pad:].to(orc.device, orc.dtype), gen.to(orc.dtype)])
        _, qkvs = orc.forward(x, return_qkv=True)
        P = x.shape[0]
        future = torch.ones(P, P, dtype=torch.bool, device=orc.device).triu(1)
        for l, (q, k, _) in enumerate(qkvs):
            p = torch.softmax((q @ k.transpose(1, 2) * orc.hd ** -0.5).masked_fill_(future, -float("inf")), -1)
            o, r, c = offs[0]
            blk = out[l, b, :, o: o + r * c].view(orc.H, r, c)
            blk[:, :pad, :] = 1.0 / T0
            blk[:, pad:, pad:] = p[:, : T0 - pad, : T0 - pad]
            for i in range(1, fed + 1):
                o, r, c = offs[i]
                t = T0 - pad + i - 1  # the query's position
                out[l, b, :, o + pad: o + c] = p[:, t, : t + 1]
    return out
