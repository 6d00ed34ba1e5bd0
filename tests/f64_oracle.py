"""The decode model in float64: a teacher-forced reference for long GPU runs.

``GPTOracle`` (oracle/gpt_oracle.py) restated with float64 states, embeddings, residual, softmax and K/V cache.  What
the model defines in fp32 is computed in fp32 and then widened: the RoPE cos/sin tables (``rope_cos_sin``; at position
2000 the fp32 angle is ~1e-4 rad from the float64 one, and the device tables are the fp32 ones) and, in the fp16
variant, the folded layer matrices rounded to fp16 (``fp16_oracle.fp16_layer_state``).  The fp16 variant also rounds
K (after RoPE) and V to fp16, which is the model ``fp16_oracle.GPTOracleFp16`` defines.

A request runs teacher-forced: once the GPU has produced its ids, ONE causal forward over the prompt embeddings followed
by the embeddings of the generated ids (positions 0 .. T0 + n - 2; the engine admits every request as a batch of one)
gives all n step hidden states at once: the output at position T0 - 1 + i is step i's.  K/V rounding is per position,
so this is the same function as the step-by-step decode loop.  ``sample_trace`` then samples each step's ids from its
logits with the request's own noise and the generated ids before that step as the repetition window, and records
its decision margins beside them (``decision_margins``, and the top-k cut's).

The arithmetic is that of ``dtype`` (float64 by default) on whichever device the oracle is built on; the GPU tests put
it on the GPU, where torch's own float64 kernels (nothing of this project's) run a 2048-token forward in well under a
second.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from fp16_oracle import fp16_layer_state
from oracle.gpt_oracle import (SamplerParams, apply_temperature, decision_margins, fold_weight_norm, repetition_penalty,
                               rope_cos_sin, rotate_half, sample_step, top_p_filter)


def peaked_state(gpt_state, scale=4.0):
    """The model with q_proj and k_proj scaled by ``scale``: every attention score scaled by scale**2 (the synthetic
    model's near-uniform attention, score std ~0.3, becomes peaked, std ~5 at scale 4)."""
    s = dict(gpt_state)
    for k in gpt_state:
        if k.endswith(("self_attn.q_proj.weight", "self_attn.k_proj.weight")):
            s[k] = gpt_state[k] * scale
    return s


class F64Oracle:
    """The ChatTTS GPT of ``gpt_state`` / ``embed_state`` in ``dtype``; ``fp16_layers`` / ``fp16_kv`` select the two
    parts of the half-precision engine's model independently."""

    def __init__(self, gpt_state, embed_state, *, fp16_layers=False, fp16_kv=False, dtype=torch.float64,
                 device="cpu", num_heads=12, head_dim=64, eps=1e-6, theta=10000.0, num_vq=4):
        src = fp16_layer_state(gpt_state) if fp16_layers else gpt_state
        self.dtype, self.device = dtype, torch.device(device)
        self.s = {k: v.to(self.device, dtype) for k, v in src.items()}
        self.L = 1 + max(int(k.split(".")[1]) for k in src if k.startswith("layers."))
        self.H, self.hd, self.eps, self.theta, self.num_vq = num_heads, head_dim, eps, theta, num_vq
        self.fp16_kv = fp16_kv
        w = lambda k: embed_state[k].to(self.device, dtype)  # noqa: E731
        self.emb_text = w("emb_text.weight")
        self.emb_code = [w(f"emb_code.{q}.weight") for q in range(num_vq)]
        self.head_code = [fold_weight_norm(w(f"head_code.{q}.parametrizations.weight.original0"),
                                           w(f"head_code.{q}.parametrizations.weight.original1"))
                          for q in range(num_vq)]
        self.head_text = fold_weight_norm(w("head_text.parametrizations.weight.original0"),
                                          w("head_text.parametrizations.weight.original1"))

    def _rms(self, x, w):
        return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps))

    def _kv_round(self, t):
        return t.half().to(self.dtype) if self.fp16_kv else t

    def embed_prompt(self, prompt_ids: torch.Tensor) -> torch.Tensor:
        """A text prompt [T] (or [T, num_vq], text id replicated) -> [T, d]."""
        ids = prompt_ids if prompt_ids.dim() == 1 else prompt_ids[:, 0]
        return F.embedding(ids.to(self.device), self.emb_text)

    def embed_codes(self, ids: torch.Tensor) -> torch.Tensor:
        """Generated code ids [n, num_vq] -> [n, d]."""
        ids = ids.to(self.device).long()
        return sum(F.embedding(ids[:, q], self.emb_code[q]) for q in range(self.num_vq))

    @torch.no_grad()
    def forward(self, x: torch.Tensor, return_qkv: bool = False):
        """One causal pass over x [T, d] at positions 0 .. T - 1 -> the final-normed hidden states [T, d] (and, with
        ``return_qkv``, each layer's attention inputs (Q, K, V) [H, T, hd], K and V as cached)."""
        T = x.shape[0]
        x = x.to(self.device, self.dtype)
        cos, sin = rope_cos_sin(torch.arange(T, dtype=torch.float32)[None], self.hd, self.theta)
        cos, sin = cos[0].to(self.device, self.dtype), sin[0].to(self.device, self.dtype)  # [T, hd]
        future = torch.ones(T, T, dtype=torch.bool, device=self.device).triu(1)
        s, H, hd = self.s, self.H, self.hd
        qkvs = []
        for l in range(self.L):
            p = f"layers.{l}."
            h = self._rms(x, s[p + "input_layernorm.weight"])
            q = F.linear(h, s[p + "self_attn.q_proj.weight"]).view(T, H, hd).transpose(0, 1)
            k = F.linear(h, s[p + "self_attn.k_proj.weight"]).view(T, H, hd).transpose(0, 1)
            v = F.linear(h, s[p + "self_attn.v_proj.weight"]).view(T, H, hd).transpose(0, 1)
            q = q * cos + rotate_half(q) * sin
            k = self._kv_round(k * cos + rotate_half(k) * sin)
            v = self._kv_round(v)
            if return_qkv:
                qkvs.append((q, k, v))
            w = torch.matmul(q, k.transpose(1, 2)) * (hd ** -0.5)
            w = torch.softmax(w.masked_fill_(future, -float("inf")), dim=-1)
            a = torch.matmul(w, v).transpose(0, 1).reshape(T, H * hd)
            del w
            x = x + F.linear(a, s[p + "self_attn.o_proj.weight"])
            h = self._rms(x, s[p + "post_attention_layernorm.weight"])
            m = F.silu(F.linear(h, s[p + "mlp.gate_proj.weight"])) * F.linear(h, s[p + "mlp.up_proj.weight"])
            x = x + F.linear(m, s[p + "mlp.down_proj.weight"])
        out = self._rms(x, s["norm.weight"])
        return (out, qkvs) if return_qkv else out

    def logits_rows(self, hidden: torch.Tensor) -> torch.Tensor:
        """Hidden states [n, d] -> code logits [n, num_vq, V]."""
        return torch.stack([F.linear(hidden, w) for w in self.head_code], dim=1)

    @torch.no_grad()
    def teacher_forced(self, prompt_emb: torch.Tensor, ids: torch.Tensor):
        """The n steps of a request whose prompt embeds to ``prompt_emb`` [T0, d] and which generated ``ids``
        [n, num_vq]: (hidden states [n, d], logits [n, num_vq, V]), on the oracle's device."""
        n, T0 = int(ids.shape[0]), int(prompt_emb.shape[0])
        x = torch.cat([prompt_emb.to(self.device, self.dtype), self.embed_codes(ids[: n - 1])])
        hid = self.forward(x)[T0 - 1:]
        return hid, self.logits_rows(hid)

    @torch.no_grad()
    def teacher_forced_text(self, prompt_emb: torch.Tensor, ids: torch.Tensor):
        """``teacher_forced`` for a text request (infer_text): ``ids`` [n] the generated text ids, each fed back through
        emb_text.  Returns (hidden states [n, d], text-head logits [n, 1, num_text]): one sampler row per step."""
        n, T0 = int(ids.shape[0]), int(prompt_emb.shape[0])
        x = torch.cat([prompt_emb.to(self.device, self.dtype), F.embedding(ids[: n - 1].to(self.device).long(),
                                                                           self.emb_text)])
        hid = self.forward(x)[T0 - 1:]
        return hid, F.linear(hid, self.head_text)[:, None]


def top_k_margin(logits: torch.Tensor, generated: torch.Tensor, temperature: torch.Tensor, sp: SamplerParams) -> float:
    """How close the top-k cut is to flipping: the smallest gap, over the rows, between the k-th and (k+1)-th largest
    scores the top-k filter sees (after temperature, repetition penalty and top-p).  ``decision_margins`` does not
    measure this cut, and a near-tie there lets either token into the sampled set."""
    if sp.top_k is None:
        return float("inf")
    x = apply_temperature(logits, temperature)
    if sp.repetition_penalty is not None and sp.repetition_penalty != 1:
        x = repetition_penalty(generated, x, sp.repetition_penalty, sp.penalty_max_ids, sp.penalty_window)
    if sp.top_p is not None:
        x = top_p_filter(x, sp.top_p, sp.min_keep)
    k = min(max(sp.top_k, sp.min_keep), x.shape[-1] - 1)
    top = torch.topk(x, k + 1, dim=-1)[0]
    gap = (top[:, k - 1] - top[:, k])[torch.isfinite(top[:, k])]
    return float(gap.min()) if gap.numel() else float("inf")


def sample_trace(logits: torch.Tensor, ids: torch.Tensor, temperature: torch.Tensor, sp: SamplerParams,
                 q: torch.Tensor, eos: int, min_new: int):
    """Sample every step of a teacher-forced request: ``logits`` [n, rows, V], ``ids`` [n, rows] the ids the GPU
    generated (step i's repetition window is ids[:i]), ``q`` [rows, V] the request's Exp(1) noise.  Returns (the
    sampled ids [n, rows], per step the smallest of ``decision_margins``' two margins and ``top_k_margin``)."""
    logits, ids = logits.cpu(), ids.cpu().long()
    n = int(logits.shape[0])
    sampled = torch.zeros(n, ids.shape[1], dtype=torch.long)
    margins = torch.zeros(n, dtype=torch.float64)
    for i in range(n):
        gen = ids[:i].T  # [rows, i]
        ban = i < min_new
        sampled[i] = sample_step(logits[i], gen, temperature, sp, q, eos, ban)
        am, pm = decision_margins(logits[i], gen, temperature, sp, q, eos, ban)
        margins[i] = min(am, pm, top_k_margin(logits[i], gen, temperature, sp))
    return sampled, margins
