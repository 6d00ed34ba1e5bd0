"""The half-precision slot engine's model (ctb_gpt_engine_begin_ex, CTB_ENGINE_FP16_*) restated on the CPU oracle.

* fp16 layers: Wqkv and [Wgate; Wup] are ``fp16_rne(fp32(W * ln))`` with the layer's input / post-attention norm
  weight folded into their columns in fp32 first, and the norms then act with unit weights (``x * rsqrt(...)``); Wo
  and Wdown are ``fp16_rne(W)``.  The heads and the final norm stay fp32.
* fp16 KV: K (after RoPE) and V are rounded to fp16 before they are cached, and every attention, the prompt's and a
  token's attention to itself included, reads the rounded values.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.gpt_oracle import GPTOracle, State, rms_norm, rope_cos_sin, rotate_half

FOLDED = (("self_attn.q_proj", "input_layernorm"), ("self_attn.k_proj", "input_layernorm"),
          ("self_attn.v_proj", "input_layernorm"), ("mlp.gate_proj", "post_attention_layernorm"),
          ("mlp.up_proj", "post_attention_layernorm"))
RAW = ("self_attn.o_proj", "mlp.down_proj")


def fp16_round(x: torch.Tensor) -> torch.Tensor:
    return x.half().float()


def fp16_layer_state(gpt_state: State) -> State:
    """The state whose fp32 model is the fp16-layer model: rounded (folded) layer matrices, unit layer norms."""
    s = dict(gpt_state)
    L = 1 + max(int(k.split(".")[1]) for k in gpt_state if k.startswith("layers."))
    for l in range(L):
        p = f"layers.{l}."
        for m, norm in FOLDED:
            s[p + m + ".weight"] = fp16_round(gpt_state[p + m + ".weight"] * gpt_state[p + norm + ".weight"][None, :])
        for m in RAW:
            s[p + m + ".weight"] = fp16_round(gpt_state[p + m + ".weight"])
        for norm in ("input_layernorm", "post_attention_layernorm"):
            s[p + norm + ".weight"] = torch.ones_like(gpt_state[p + norm + ".weight"])
    return s


class GPTOracleFp16(GPTOracle):
    """``GPTOracle`` of the fp16 model; ``fp16_layers`` / ``fp16_kv`` select its two parts independently."""

    def __init__(self, gpt_state: State, embed_state: State, *, fp16_layers=False, fp16_kv=False, **kw):
        super().__init__(fp16_layer_state(gpt_state) if fp16_layers else gpt_state, embed_state, **kw)
        self.fp16_kv = fp16_kv

    def forward(self, x, positions, key_mask, past):
        """``GPTOracle.forward`` with K and V rounded to fp16 (when ``fp16_kv``) right after RoPE."""
        B, t, d = x.shape
        cos, sin = rope_cos_sin(positions, self.hd, self.theta)
        cos, sin = cos[:, None], sin[:, None]
        Ttot = key_mask.shape[1]
        causal = torch.ones(t, Ttot, dtype=torch.bool).tril(diagonal=Ttot - t)
        allow = causal[None, None] & key_mask[:, None, None, :]
        add = torch.zeros(B, 1, t, Ttot).masked_fill(~allow, -float("inf"))
        new_past = []
        s = self.s
        for l in range(self.L):
            p = f"layers.{l}."
            h = rms_norm(x, s[p + "input_layernorm.weight"], self.eps)
            q = F.linear(h, s[p + "self_attn.q_proj.weight"]).view(B, t, self.H, self.hd).transpose(1, 2)
            k = F.linear(h, s[p + "self_attn.k_proj.weight"]).view(B, t, self.H, self.hd).transpose(1, 2)
            v = F.linear(h, s[p + "self_attn.v_proj.weight"]).view(B, t, self.H, self.hd).transpose(1, 2)
            q = q * cos + rotate_half(q) * sin
            k = k * cos + rotate_half(k) * sin
            if self.fp16_kv:
                k, v = fp16_round(k), fp16_round(v)
            if past is not None:
                k = torch.cat([past[l][0], k], dim=2)
                v = torch.cat([past[l][1], v], dim=2)
            new_past.append((k, v))
            w = torch.matmul(q, k.transpose(2, 3)) * (self.hd ** -0.5) + add
            w = torch.softmax(w, dim=-1, dtype=torch.float32)
            w = torch.nan_to_num(w)
            a = torch.matmul(w, v).transpose(1, 2).reshape(B, t, self.H * self.hd)
            x = x + F.linear(a, s[p + "self_attn.o_proj.weight"])
            h = rms_norm(x, s[p + "post_attention_layernorm.weight"], self.eps)
            m = F.silu(F.linear(h, s[p + "mlp.gate_proj.weight"])) * F.linear(h, s[p + "mlp.up_proj.weight"])
            x = x + F.linear(m, s[p + "mlp.down_proj.weight"])
        return rms_norm(x, s["norm.weight"], self.eps), new_past
