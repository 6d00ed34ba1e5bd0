"""Host side of hot path 1: drop-in for the reference's ``GPT`` (ChatTTS/model/gpt.py).

Same constructor, ``generate`` signature, ``GenerationOutputs`` and ``Context`` as the
reference (gpt.py:21-57,103-111,276-337); the per-token Python loop (gpt.py:394-596) is
replaced by ``ctb_gpt_begin`` / ``ctb_gpt_decode`` (include/chattts_b200.h) which run the
whole step - embedding sum, 20 decoder layers with paged KV, the four heads, the sampling
filters, multinomial and finish bookkeeping - as CUDA kernels replayed from a CUDA graph.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
import weakref
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple, Union

import torch

from . import _lib
from .config import GPTConfig
from .embed import Embed
from .processors import build_sampler_config, exp_noise


def _rope_tables(max_pos: int, head_dim: int, theta: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos/sin exactly as HF LlamaRotaryEmbedding computes them on the CPU in fp32
    ([3p]; in-tree statement examples/onnx/modeling_llama.py:119-162).  Built on the host so
    the kernel reads bit-identical values to the fp32 CPU reference."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).float() / head_dim))
    pos = torch.arange(max_pos, dtype=torch.float32)
    freqs = (inv_freq[None, :, None] @ pos[None, None, :]).transpose(1, 2)[0]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().contiguous(), emb.sin().contiguous()


def _del_all(x):
    if isinstance(x, list):
        x.clear()


def _attention_step_shapes(T0: int, i0: int, i1: int) -> List[Tuple[int, int]]:
    """(rows, cols) of each step's map in [i0, i1): the prompt's [T0, T0] at step 0, then [1, T0 + i]."""
    return [(T0, T0) if i == 0 else (1, T0 + i) for i in range(i0, i1)]


def attention_map_views(buf: torch.Tensor, L: int, B: int, H: int, T0: int, i0: int, i1: int):
    """The entries of steps i0 .. i1 - 1 of ``GenerationOutputs.attentions``, views into ``buf``, the output of one
    ``ctb_gpt_attention_maps`` call: per step, a tuple of ``L`` tensors ``[B, H, rows, cols]`` (one per layer)."""
    out, off = [], 0
    for r, c in _attention_step_shapes(T0, i0, i1):
        size = L * B * H * r * c
        out.append(tuple(buf.narrow(0, off, size).view(L, B, H, r, c).unbind(0)))
        off += size
    assert off == buf.numel()
    return out


def score_groups(widths: List[int], max_batch: int) -> List[Tuple[List[int], int]]:
    """The ``ctb_gpt_score`` calls ``GPT.score`` makes for rows of ``widths`` columns (prompt + given tokens - 1), as
    ``[(row indices, padded width)]``, by the slot engine's admission rule: rows of up to ``LONG_PROMPT_COLS`` columns
    share one width (at least ``MIN_PROMPT_COLS``) in calls of at most ``ADMIT_MAX_ROWS`` (row, column) pairs and
    ``max_batch`` rows (``engine.admission_chunks``); a longer row is scored on its own, after them."""
    from .engine import LONG_PROMPT_COLS, MIN_PROMPT_COLS, admission_chunks

    short = [i for i, w in enumerate(widths) if w <= LONG_PROMPT_COLS]
    out = []
    if short:
        T = max(MIN_PROMPT_COLS, max(widths[i] for i in short))
        for part in admission_chunks(short, T):
            out += [(part[k: k + max_batch], T) for k in range(0, len(part), max_batch)]
    return out + [([i], w) for i, w in enumerate(widths) if w > LONG_PROMPT_COLS]


class GPT:
    class Context:
        """gpt.py:103-111 - interrupt flag polled between decode chunks."""

        def __init__(self):
            self._interrupt = False

        def set(self, v: bool):
            self._interrupt = v

        def get(self) -> bool:
            return self._interrupt

    @dataclass(repr=False, eq=False)
    class GenerationOutputs:
        """gpt.py:276-285."""

        ids: List[torch.Tensor]
        attentions: List[Optional[Tuple[torch.FloatTensor, ...]]]
        hiddens: List[torch.Tensor]
        cancelled: bool = False  # an open engine's job that was cancelled: the outputs are the prefix it had
        # a slot engine opened with logprobs=True: per item, log p of each returned id under the model's logits at
        # temperature 1 ([n, num_vq] fp32 for codes, [n] for text), aligned with ``ids``; otherwise empty
        logprobs: List[torch.Tensor] = field(default_factory=list)
        # a slot engine opened with top_logprobs=N: per item, (ids, lp) of the N most likely ids at each returned token
        # under the same logits, z descending (int64 and fp32, [n, num_vq, N] for codes, [n, N] for text), aligned
        # with ``ids``; otherwise empty
        top_logprobs: List[Tuple[torch.Tensor, torch.Tensor]] = field(default_factory=list)

        def destroy(self):
            _del_all(self.ids)
            _del_all(self.attentions)
            _del_all(self.hiddens)
            _del_all(self.logprobs)
            _del_all(self.top_logprobs)

    def __init__(self, gpt_config: Union[dict, GPTConfig], embed: Embed, use_flash_attn=False, use_vllm=False,
                 device=torch.device("cuda"), device_gpt=torch.device("cuda"),
                 logger=logging.getLogger(__name__), max_batch: int = 32, max_context: int = 2560):
        self.logger = logger
        self.device = torch.device(device)
        self.device_gpt = torch.device(device_gpt)
        if isinstance(gpt_config, dict):
            known = {f for f in GPTConfig.__dataclass_fields__}
            gpt_config = GPTConfig(**{k: v for k, v in gpt_config.items() if k in known})
        self.config = gpt_config
        self.num_vq = int(gpt_config.num_vq)
        self.num_audio_tokens = int(gpt_config.num_audio_tokens)
        self.num_text_tokens = int(gpt_config.num_text_tokens)
        # accepted for signature compatibility, ignored (SURVEY.md quirk Q14): there is one back end
        self.use_flash_attn, self.is_vllm, self.is_te_llama = use_flash_attn, False, False
        self.embed = embed
        self.max_batch, self.max_context = max_batch, max_context
        self._handle = C.c_void_p()
        self._weights: Optional[torch.Tensor] = None
        self._stream_keepalive = []
        self._open = None  # the open engine (open_engine) that owns the handle until it is closed

    # ------------------------------------------------------------------ loading
    def load_pretrained(self, gpt_folder: str, embed_file_path: str, experimental=False):
        """gpt.py:59-101: HF folder -> state dict (the reference's loader), then pack."""
        from transformers import LlamaModel

        model = LlamaModel.from_pretrained(gpt_folder)
        cfg = model.config  # quirk Q22: hyper-parameters come from asset/gpt/config.json
        rope = getattr(cfg, "rope_parameters", None) or {}
        self.config = GPTConfig(
            hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
            num_attention_heads=cfg.num_attention_heads,
            num_key_value_heads=getattr(cfg, "num_key_value_heads", cfg.num_attention_heads),
            head_dim=getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads,
            num_hidden_layers=cfg.num_hidden_layers, max_position_embeddings=cfg.max_position_embeddings,
            rms_norm_eps=cfg.rms_norm_eps, rope_theta=rope.get("rope_theta", getattr(cfg, "rope_theta", 10000.0)),
            num_audio_tokens=self.num_audio_tokens, num_text_tokens=self.num_text_tokens, num_vq=self.num_vq)
        state = {k: v for k, v in model.state_dict().items() if not k.startswith("embed_tokens")}
        self.load_state(state)

    def load_state(self, gpt_state: Dict[str, torch.Tensor], weights_blob: Optional[torch.Tensor] = None):
        """Pack the checkpoint into the blob layout of ``ctb_gpt_layout_query`` and create the handle.

        ``weights_blob``: an already packed device tensor (e.g. received by NCCL broadcast,
        chattts_b200/dist.py) - then ``gpt_state`` may be None."""
        _lib.require_cuda()
        lib = _lib.load()
        cc, lay = self.query_layout()
        if weights_blob is None:
            weights_blob = self.pack_weights(gpt_state, lay).to(self.device_gpt)
        assert weights_blob.numel() == lay.total and weights_blob.dtype == torch.float32
        self._weights = weights_blob.contiguous()
        if self._handle:
            lib.ctb_gpt_destroy(self._handle)
            self._handle = C.c_void_p()
        with torch.cuda.device(self.device_gpt):
            _lib.check(lib.ctb_gpt_create(C.byref(cc), C.c_void_p(self._weights.data_ptr()), C.byref(self._handle)))
        self.embed._gpt = self  # Embed.forward now runs as ctb_gpt_embed_prompt on this handle's tables

    @torch.inference_mode()
    def embed_prompt(self, input_ids: torch.Tensor, text_mask: torch.Tensor) -> torch.Tensor:
        """Embed.forward (embed.py:51-79) on the device: [B, T, num_vq] ids + text mask -> [B, T, d] fp32."""
        lib = _lib.load()
        dev = self.device_gpt
        ids = input_ids.to(dev, torch.int64).contiguous()
        tm = text_mask.to(dev).to(torch.uint8).contiguous()
        B, T = int(ids.shape[0]), int(ids.shape[1])
        out = torch.empty(B, T, self.config.hidden_size, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.ctb_gpt_embed_prompt(self._handle, C.c_void_p(ids.data_ptr()), C.c_void_p(tm.data_ptr()), B, T,
                                                C.c_void_p(out.data_ptr()),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out

    def query_layout(self):
        """(ctb_gpt_config, ctb_gpt_layout) for this model shape - the C side owns the blob layout."""
        lib = _lib.load()
        c = self.config
        cc = _lib.GptConfig(c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.num_attention_heads,
                            c.num_key_value_heads, c.head_dim, c.num_vq, c.num_audio_tokens, c.num_text_tokens,
                            c.max_position_embeddings, c.rms_norm_eps, self.max_batch, self.max_context)
        lay = _lib.GptLayout()
        _lib.check(lib.ctb_gpt_layout_query(C.byref(cc), C.byref(lay)))
        self._cc, self._layout = cc, lay
        return cc, lay

    def pack_weights(self, s: Dict[str, torch.Tensor], lay) -> torch.Tensor:
        c = self.config
        blob = torch.empty(lay.total, dtype=torch.float32)

        def put(off, t):
            t = t.detach().to("cpu", torch.float32).contiguous().view(-1)
            blob[off: off + t.numel()] = t

        for l in range(c.num_hidden_layers):
            base, p = lay.layer0 + l * lay.layer_stride, f"layers.{l}."
            put(base + lay.wqkv, torch.cat([s[p + "self_attn.q_proj.weight"], s[p + "self_attn.k_proj.weight"],
                                            s[p + "self_attn.v_proj.weight"]], 0))
            put(base + lay.wo, s[p + "self_attn.o_proj.weight"])
            put(base + lay.wgate_up, torch.cat([s[p + "mlp.gate_proj.weight"], s[p + "mlp.up_proj.weight"]], 0))
            put(base + lay.wdown, s[p + "mlp.down_proj.weight"])
            put(base + lay.ln1, s[p + "input_layernorm.weight"])
            put(base + lay.ln2, s[p + "post_attention_layernorm.weight"])
        put(lay.final_norm, s["norm.weight"])
        e = self.embed
        put(lay.head_code, torch.cat([e.folded_head(f"head_code.{q}").cpu() for q in range(c.num_vq)], 0))
        put(lay.head_text, e.folded_head("head_text").cpu())
        put(lay.emb_code, torch.cat([e.state[f"emb_code.{q}.weight"].cpu() for q in range(c.num_vq)], 0))
        put(lay.emb_text, e.state["emb_text.weight"].cpu())
        cos, sin = _rope_tables(c.max_position_embeddings, c.head_dim, c.rope_theta)
        put(lay.rope_cos, cos)
        put(lay.rope_sin, sin)
        return blob

    def prepare(self, compile=False):
        """gpt.py:131-139 compiled the HF model with inductor; nothing to do here (quirk Q14)."""

    def eval(self):
        return self

    def __del__(self):
        try:
            if self._handle:
                _lib.load().ctb_gpt_destroy(self._handle)
        except Exception:
            pass

    # ------------------------------------------------------------------ outputs
    @torch.no_grad()
    def _prepare_generation_outputs(self, inputs_ids: torch.Tensor, start_idx: int, end_idx: torch.Tensor,
                                    attentions, hiddens, infer_text: bool) -> "GPT.GenerationOutputs":
        """gpt.py:287-313 (``hiddens`` here is already a [B, n, d] tensor or an empty list)."""
        ids = [inputs_ids[i].narrow(0, start_idx, int(n)) for i, n in enumerate(end_idx)]
        if infer_text:
            ids = [i.narrow(1, 0, 1).squeeze_(1) for i in ids]
        if isinstance(hiddens, list) and len(hiddens) > 0:
            hiddens = torch.stack(hiddens, 1)
        if isinstance(hiddens, torch.Tensor):
            hiddens = [hiddens[i].narrow(0, 0, int(n)) for i, n in enumerate(end_idx.int())]
        return self.GenerationOutputs(ids=ids, attentions=attentions, hiddens=hiddens)

    # ------------------------------------------------------------------ device-resident entry
    def enqueue_generate(self, emb_d: torch.Tensor, mask_d: torch.Tensor, cfg, q_d: Optional[torch.Tensor],
                         max_new_token: int, infer_text: bool, ids_out: torch.Tensor,
                         hid_out: Optional[torch.Tensor], n_steps: Optional[int] = None) -> None:
        """Enqueue prefill + ``n_steps`` loop iterations on the current stream with every buffer
        already resident on the device; never synchronises (bench.py times this with CUDA events)."""
        lib = _lib.load()
        B, T0 = int(emb_d.shape[0]), int(emb_d.shape[1])
        stream_ptr = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(lib.ctb_gpt_begin(
            self._handle, B, T0, C.c_void_p(emb_d.data_ptr()), C.c_void_p(mask_d.data_ptr()), C.byref(cfg),
            C.c_void_p(q_d.data_ptr()) if q_d is not None else None, max_new_token, int(bool(infer_text)),
            C.c_void_p(ids_out.data_ptr()), C.c_void_p(hid_out.data_ptr()) if hid_out is not None else None,
            stream_ptr))
        n = max_new_token - 1 if n_steps is None else n_steps
        if n > 0:
            _lib.check(lib.ctb_gpt_decode(self._handle, n, stream_ptr))

    def _extend_attention_maps(self, attentions: list, steps: int, emb_d: torch.Tensor, mask_d: torch.Tensor,
                               ids_out: torch.Tensor, infer_text: bool, stream_ptr) -> None:
        """Append to ``attentions`` the maps of steps ``len(attentions)`` .. ``steps - 1`` of the static batch in flight:
        ctb_gpt_attention_maps over their query columns, whose embeddings are the prompt's (step 0) and
        ctb_gpt_embed_prompt of the ids fed at steps 1, 2, ... (step i feeds the id sampled at step i - 1)."""
        i0 = len(attentions)
        if steps <= i0:
            return
        c = self.config
        B, T0 = int(emb_d.shape[0]), int(emb_d.shape[1])
        L, H = c.num_hidden_layers, c.num_attention_heads
        parts = [emb_d] if i0 == 0 else []
        g0, g1 = max(i0, 1) - 1, steps - 1
        if g1 > g0:
            ids = ids_out[:, g0:g1].to(torch.int64)
            parts.append(self.embed_prompt(ids, torch.full(ids.shape[:2], bool(infer_text), device=ids.device)))
        emb = torch.cat(parts, 1) if len(parts) > 1 else parts[0].contiguous()
        q0 = 0 if i0 == 0 else T0 + i0 - 1
        floats = L * B * H * sum(r * k for r, k in _attention_step_shapes(T0, i0, steps))
        buf = torch.empty(floats, dtype=torch.float32, device=emb_d.device)
        _lib.check(_lib.load().ctb_gpt_attention_maps(
            self._handle, B, T0, q0, int(emb.shape[1]), C.c_void_p(emb.data_ptr()), C.c_void_p(mask_d.data_ptr()),
            C.c_void_p(buf.data_ptr()), stream_ptr))
        attentions.extend(attention_map_views(buf, L, B, H, T0, i0, steps))

    # ------------------------------------------------------------------ teacher-forced scoring
    @torch.no_grad()
    def score(self, prompts, targets, infer_text: bool = False, top_logprobs: int = 0) -> list:
        """The model's log-probability of given tokens: for each row, ``log softmax(z)[token]`` of every token of
        ``targets[i]`` after ``prompts[i]`` and the tokens before it (teacher forcing), at temperature 1 on the raw
        head logits ``z``, the quantity ``GenerationOutputs.logprobs`` holds for sampled ids.

        ``prompts``: per row, the prompt embedding ``[P, d]`` with every position valid (``Request.emb``).
        ``targets``: per row, ids ``[n, num_vq]`` of audio codes, or ``[n]`` text ids with ``infer_text``
        (``GenerationOutputs.ids``).  Returns per row an fp32 device tensor ``[n, num_vq]`` (``[n]`` for text).

        One causal prefill pass per call of ``ctb_gpt_score`` on the fp32 model, rows grouped as the slot engine
        admits prompts (``score_groups``).  ValueError for an id outside the vocabulary or ``P + n - 1`` over
        ``max_context``; RuntimeError while an open engine owns the handle.  A static ``generate`` stream in flight
        ends (resuming it raises ``CtbError``).

        ``top_logprobs=N`` (1..20; ctb_gpt_score_ex) makes each row ``(lp, top_ids, top_lp)``: besides ``lp`` as above,
        the N ids with the largest ``z`` at every scored position (z descending, the smaller id first among equal z;
        int64 ``[n, num_vq, N]``, ``[n, N]`` for text) and their log-probabilities (fp32, same shape), the quantity
        ``GenerationOutputs.top_logprobs`` holds.  ``lp`` is bit-equal to that of a call without it."""
        from .engine import check_top_logprobs

        top_n = check_top_logprobs(top_logprobs)
        self._check_free("score")
        if not self._handle:
            raise _lib.CtbError("GPT weights not loaded")
        prompts, targets = list(prompts), list(targets)
        if len(prompts) != len(targets):
            raise ValueError(f"score: {len(prompts)} prompts and {len(targets)} target rows")
        dev, d = self.device_gpt, self.config.hidden_size
        rpi = 1 if infer_text else self.num_vq
        V = self.num_text_tokens if infer_text else self.num_audio_tokens
        rows = []
        for i, (p, t) in enumerate(zip(prompts, targets)):
            t = torch.as_tensor(t)
            if p.dim() != 2 or int(p.shape[1]) != d or int(p.shape[0]) < 1:
                raise ValueError(f"score: prompt {i} has shape {tuple(p.shape)}, expected [P >= 1, {d}]")
            if (t.dim() != 1) if infer_text else (t.dim() != 2 or int(t.shape[1]) != rpi):
                raise ValueError(f"score: targets {i} have shape {tuple(t.shape)}, expected "
                                 f"{'[n]' if infer_text else f'[n, {rpi}]'}")
            P, n = int(p.shape[0]), int(t.shape[0])
            if n and (int(t.min()) < 0 or int(t.max()) >= V):
                raise ValueError(f"score: targets {i} hold ids outside [0, {V})")
            if P + n - 1 > self.max_context:
                raise ValueError(f"score: row {i}: prompt {P} + {n} tokens - 1 exceed max_context={self.max_context}")
            rows.append((p, t.reshape(n, rpi), P, n))
        out = [torch.empty((n, rpi) if rpi > 1 else (n,), dtype=torch.float32, device=dev) for _, _, _, n in rows]
        top_shape = [((n, rpi, top_n) if rpi > 1 else (n, top_n)) for _, _, _, n in rows]
        top_ids = [torch.empty(t, dtype=torch.int64, device=dev) for t in top_shape] if top_n else []
        top_lp = [torch.empty(t, dtype=torch.float32, device=dev) for t in top_shape] if top_n else []
        result = list(zip(out, top_ids, top_lp)) if top_n else out
        live = [i for i, r in enumerate(rows) if r[3] > 0]
        if not live:
            return result
        lib = _lib.load()
        with torch.cuda.device(dev):
            stream_ptr = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            for group, T in score_groups([rows[i][2] + rows[i][3] - 1 for i in live], self.max_batch):
                idx = [live[g] for g in group]
                B = len(idx)
                emb = torch.zeros(B, T, d, dtype=torch.float32, device=dev)
                for b, i in enumerate(idx):
                    p, t, P, n = rows[i]
                    c0 = T - (P + n - 1)
                    emb[b, c0: c0 + P] = p.to(dev, torch.float32)
                    if n > 1:
                        ids = t[: n - 1].to(dev, torch.int64).expand(n - 1, self.num_vq)[None].contiguous()
                        emb[b, c0 + P:] = self.embed_prompt(ids, torch.full((1, n - 1), bool(infer_text), device=dev))[0]
                tgt = torch.cat([rows[i][1] for i in idx]).to(dev, torch.int32).contiguous()
                res = torch.empty(tgt.shape, dtype=torch.float32, device=dev)
                n_prompt = (C.c_int32 * B)(*[rows[i][2] for i in idx])
                n_given = (C.c_int32 * B)(*[rows[i][3] for i in idx])
                if not top_n:
                    _lib.check(lib.ctb_gpt_score(self._handle, B, T, C.c_void_p(emb.data_ptr()), n_prompt, n_given,
                                                 C.c_void_p(tgt.data_ptr()), int(bool(infer_text)),
                                                 C.c_void_p(res.data_ptr()), stream_ptr))
                else:
                    t_ids = torch.empty(*tgt.shape, top_n, dtype=torch.int32, device=dev)
                    t_lp = torch.empty(*tgt.shape, top_n, dtype=torch.float32, device=dev)
                    _lib.check(lib.ctb_gpt_score_ex(self._handle, B, T, C.c_void_p(emb.data_ptr()), n_prompt, n_given,
                                                    C.c_void_p(tgt.data_ptr()), int(bool(infer_text)),
                                                    C.c_void_p(res.data_ptr()), top_n, C.c_void_p(t_ids.data_ptr()),
                                                    C.c_void_p(t_lp.data_ptr()), stream_ptr))
                    sizes = [rows[i][3] for i in idx]
                    for i, a, b in zip(idx, t_ids.split(sizes), t_lp.split(sizes)):
                        top_ids[i].copy_(a.view(top_shape[i]))
                        top_lp[i].copy_(b.view(top_shape[i]))
                for i, r in zip(idx, res.split([rows[i][3] for i in idx])):
                    out[i].copy_(r.view(out[i].shape))
        return result

    # ------------------------------------------------------------------ continuous batching
    @torch.no_grad()
    def generate_continuous(self, requests, slots: Optional[int] = None, return_hidden=True, infer_text=False,
                            stream=False, return_attn=False, context=None, chunk: Optional[int] = None,
                            max_new_cap: Optional[int] = None, dtype=torch.float32,
                            prefill_budget: Optional[int] = None, kv_pool_bytes: Optional[int] = None,
                            logprobs: bool = False, top_logprobs: int = 0):
        """Generate audio codes or text for many utterances on a slot engine (chattts_b200.engine): up to ``slots``
        requests (default: ``max_batch``, at most the number of requests) decode together, and a waiting request takes
        the place of a finished one at the next poll (every ``chunk`` steps, default CTB_DECODE_CHUNK or 32).  Each
        ``Request`` chooses its mode (``Request.infer_text``); code and text requests share the engine.  ``slots`` may
        be up to the handle's ``max_batch``: engines of 9..64 slots run the wgmma decode step, wider ones the PDL chain.

        Generator of ``(request_index, GenerationOutputs)`` in completion order.  A prompt may be up to ``max_context``
        - ``max_new_token`` tokens.  Up to 1,024 tokens, each request's ids equal, bit for bit, ``generate`` on that
        request alone with the same arguments and ``manual_seed``.  A longer prompt is prefilled on its own with a tiled
        attention kernel, while ``generate`` walks such a prompt's columns: the two agree within float rounding, so
        their ids can differ where the sampler's decision is a near-tie (DESIGN.md §4, "Long prompts").  A seeded request that
        samples EOS first yields empty outputs (``generate`` yields nothing then); an unseeded one with
        ``ensure_non_empty`` runs again.  The handle serves one generator at a time; ``generate`` may be called again
        once it is exhausted.

        Follow-ups (``Request.then``) are yielded under new indices, ``len(requests)`` on; ``last_schedule_stats
        .children`` maps each request index to its follow-up's.  ``max_new_cap`` (default: the largest
        ``max_new_token`` of ``requests``) bounds every request's ``max_new_token``, follow-ups included: the engine's
        output buffers are sized by it.

        ``dtype=torch.float16`` runs a half-precision engine (ctb_gpt_engine_begin_ex): the four matrices of every
        layer and the KV cache in fp16, everything else fp32 (the model the reference serves with
        ``Chat.load(use_vllm=True)``).  Its ids then follow that model, not ``generate``'s fp32 one.  It serves up to
        64 slots (``CtbError`` above).

        ``prefill_budget`` (prompt columns per poll, at least 128; default None: every admission is prefilled whole)
        bounds the prefill the running slots wait for at each poll: a prompt that does not fit is prefilled in chunks
        of multiples of 128 columns over the next polls (``engine._poll_cycles``), and its outputs are bit for bit
        those of its admission in one call.  The yields are the same; a long prompt's first token comes later.

        ``kv_pool_bytes`` (default None: every slot owns ``max_context`` tokens of KV pages from the start) bounds the
        engine's KV memory: slots take 16-token pages from a pool of that many bytes as they grow, and when it runs
        short the running request admitted last is suspended to pinned host memory and resumed later, in any slot, bit
        for bit as if it had not moved (``engine._poll_cycles``).  A request whose prompt + ``max_new_token`` does not
        fit in the pool alone is refused.  ``last_schedule_stats`` records pages, suspensions and resumes.

        Requests with equal ``Request.prompt_key`` (several takes of one utterance) must have equal prompts
        (``ValueError`` otherwise).  While one of them runs, another is admitted by taking that slot's KV for all but
        the last chunk of at most 128 prompt columns and prefilling only that chunk (``engine._poll_cycles``), with
        the same outputs; a paged engine shares the pages themselves.  ``last_schedule_stats`` records the shares.

        ``logprobs=True`` fills ``GenerationOutputs.logprobs``: for each returned id, its log-probability under the
        head logits the sampler read, at temperature 1 and before the repetition penalty, top-P, top-K and the EOS ban
        (ctb_gpt_engine_logprobs).  Ids and hidden states are the same with or without it.

        ``top_logprobs=N`` (1..20; 0 is off) fills ``GenerationOutputs.top_logprobs``: for each returned token, the N
        ids with the largest head logits ``z`` (z descending, the smaller id first among equal z) and their
        log-probabilities, of the distribution ``logprobs`` uses (ctb_gpt_engine_top_logprobs).  Where the sampled id
        is among them its entry equals its ``logprobs`` value bit for bit.  Independent of ``logprobs``; ids, hidden
        states and log-probabilities are the same with or without it."""
        from .engine import ScheduleStats, check_prefill_budget, check_top_logprobs, kv_pool_pages, schedule

        check_top_logprobs(top_logprobs)
        flags = _lib.engine_flags(dtype)
        prefill_budget = check_prefill_budget(prefill_budget)
        pool = kv_pool_pages(self.config, kv_pool_bytes, flags)

        if stream:
            raise ValueError("generate_continuous: stream=True is not supported; results are yielded per request "
                             "(generate_continuous_stream streams)")
        requests, S, chunk, context, cap, check = self._engine_args(
            "generate_continuous", requests, slots, infer_text, return_attn, context, chunk, 32, max_new_cap, pool)
        if not requests:
            return
        with torch.cuda.device(self.device_gpt):
            dev = self._engine_device(requests, S, cap, return_hidden, flags, pool, logprobs, top_logprobs)
            self.last_schedule_stats = stats = ScheduleStats()  # admissions, decode steps (tools/bench_continuous.py)
            for i, slot, n in schedule(requests, dev, chunk, context, stats, check, prefill_budget):
                yield i, (dev.empty(i) if slot is None else dev.harvest(slot, n))
            if stats.interrupted:
                self.logger.warning("generation is interrupted")

    @torch.no_grad()
    def generate_continuous_stream(self, requests, slots: Optional[int] = None, return_hidden=True, context=None,
                                   chunk: Optional[int] = None, infer_text=False, return_attn=False,
                                   max_new_cap: Optional[int] = None, dtype=torch.float32,
                                   prefill_budget: Optional[int] = None, kv_pool_bytes: Optional[int] = None,
                                   logprobs: bool = False, top_logprobs: int = 0):
        """Streaming form of ``generate_continuous``: generator of ``(request_index, GenerationOutputs, last)``.

        For each request the yields are exactly those ``generate(stream=True, stream_batch=r.stream_batch)`` makes for
        it alone, in the same order: cumulative outputs every ``stream_batch`` steps while unfinished, the repeated
        boundary when EOS follows it on the next step, then the final yield, which alone has ``last=True``.  Yields of
        different requests interleave in poll order.  The engine polls every ``chunk`` steps (default:
        CTB_DECODE_CHUNK, or the smallest ``stream_batch`` among the requests); the yields do not depend on it.
        A seeded request that samples EOS first yields one empty final output.  Text requests and follow-ups are
        served as in ``generate_continuous``.

        ``ids`` are copies.  ``hiddens`` are views into the engine's buffer, like the narrowed views ``generate``
        hands out: they stay valid until this generator is resumed (copy them to keep them).  ``dtype``,
        ``prefill_budget`` and ``kv_pool_bytes`` as in ``generate_continuous``: none changes a request's yields.
        ``logprobs`` and ``top_logprobs`` as there: each yield carries copies of the rows of the ids it carries."""
        from .engine import ScheduleStats, check_prefill_budget, check_top_logprobs, kv_pool_pages, stream_schedule

        check_top_logprobs(top_logprobs)
        flags = _lib.engine_flags(dtype)
        prefill_budget = check_prefill_budget(prefill_budget)
        pool = kv_pool_pages(self.config, kv_pool_bytes, flags)
        requests, S, chunk, context, cap, check = self._engine_args(
            "generate_continuous_stream", requests, slots, infer_text, return_attn, context, chunk, None, max_new_cap,
            pool)
        if not requests:
            return
        with torch.cuda.device(self.device_gpt):
            dev = self._engine_device(requests, S, cap, return_hidden, flags, pool, logprobs, top_logprobs)
            self.last_schedule_stats = stats = ScheduleStats()
            for batch in stream_schedule(requests, dev, chunk, context, stats, check, prefill_budget=prefill_budget):
                for i, slot, n, last in batch:
                    yield i, (dev.empty(i) if slot is None else dev.harvest(slot, n, copy=False)), last
            if stats.interrupted:
                self.logger.warning("generation is interrupted")

    def open_engine(self, slots: int, max_new_cap: int, return_hidden=True, chunk: Optional[int] = None,
                    dtype=torch.float32, prefill_budget: Optional[int] = None, kv_pool_bytes: Optional[int] = None,
                    logprobs: bool = False, top_logprobs: int = 0):
        """A slot engine that takes requests while it decodes: ``submit(request, stream=False) -> engine.Job`` from
        any thread, ``Job.cancel()`` for one request, ``close(cancel=False)`` (or a ``with`` block) to drain it.

        A job's ``result()`` is the request's ``GenerationOutputs``, bit for bit what ``generate_continuous`` yields
        for it; a cancelled job's result is the prefix it had at the poll that stopped it, with ``cancelled=True``.  A
        streaming job iterates ``(GenerationOutputs, last)``, the yields ``generate_continuous_stream`` makes for it
        (copies), and simply ends when cancelled.  ``submit`` checks the request against this handle and
        ``max_new_cap`` in the caller's thread: prompt + ``max_new_token`` within ``max_context``.  A prompt over
        1,024 tokens is prefilled on its own; the running slots wait for that prefill, unless ``prefill_budget``
        bounds each poll's prefill (``generate_continuous``; a job cancelled while its prompt is in progress frees its
        slot at the next poll).  One worker thread owns the handle and its stream; while the engine
        is open ``generate``, ``generate_continuous*`` and another ``open_engine`` raise.  The poll interval is
        ``chunk`` steps (default CTB_DECODE_CHUNK, else 24).  ``slots`` and ``dtype`` as in ``generate_continuous``
        (up to ``max_batch`` slots; a half-precision engine up to 64).  ``kv_pool_bytes`` as in
        ``generate_continuous``: ``submit`` refuses a request that does not fit in the pool alone, and a job cancelled
        while suspended ends with the tokens it had.  ``logprobs`` and ``top_logprobs`` as in
        ``generate_continuous``."""
        from .engine import GptEngine

        return self._open_slot_engine(GptEngine, slots, max_new_cap, return_hidden, chunk,
                                      flags=_lib.engine_flags(dtype), prefill_budget=prefill_budget,
                                      kv_pool_bytes=kv_pool_bytes, logprobs=logprobs, top_logprobs=top_logprobs)

    def _open_slot_engine(self, cls, slots, max_new_cap, return_hidden, chunk, *args, flags=0, prefill_budget=None,
                          kv_pool_bytes=None, logprobs=False, top_logprobs=0):
        """An ``engine.OpenEngine`` subclass ``cls`` that owns this handle until it is closed (``flags``: the
        ctb_gpt_engine_begin_ex precision flags; ``prefill_budget``: the engine's bound on each poll's prefill;
        ``kv_pool_bytes``: its KV pool, None for fixed pages; ``logprobs``: outputs carry token log-probabilities;
        ``top_logprobs``: and the N most likely ids at each token)."""
        from .engine import check_prefill_budget, check_top_logprobs, kv_pool_pages

        check_top_logprobs(top_logprobs)
        prefill_budget = check_prefill_budget(prefill_budget)
        pool = kv_pool_pages(self.config, kv_pool_bytes, flags)
        _, S, chunk, _, cap, check = self._engine_args("open_engine", [], slots, False, False, None, chunk, None,
                                                       max_new_cap, pool)
        kw = {"slots": S} if prefill_budget is None else {"prefill_budget": prefill_budget, "slots": S}
        engine = cls(lambda requests: self._engine_device(requests, S, cap, return_hidden, flags, pool, logprobs,
                                                          top_logprobs), chunk, check,
                     self.device_gpt, self._close_engine, *args, max_new_cap=cap, **kw)
        self._open = engine
        return engine

    def _engine_device(self, requests, S, cap, return_hidden, flags, pool_pages=None, logprobs=False, top_logprobs=0):
        """The ``engine.EngineDevice`` of one slot engine; an fp32 engine with fixed pages gets the five-argument form
        that stand-in devices implement."""
        from . import engine

        if top_logprobs:
            return engine.EngineDevice(self, requests, S, cap, return_hidden, flags=flags, kv_pool_pages=pool_pages,
                                       logprobs=logprobs, top_logprobs=top_logprobs)
        if logprobs:
            return engine.EngineDevice(self, requests, S, cap, return_hidden, flags=flags, kv_pool_pages=pool_pages,
                                       logprobs=True)
        if pool_pages is not None:
            return engine.EngineDevice(self, requests, S, cap, return_hidden, flags=flags, kv_pool_pages=pool_pages)
        if flags:
            return engine.EngineDevice(self, requests, S, cap, return_hidden, flags=flags)
        return engine.EngineDevice(self, requests, S, cap, return_hidden)

    def _close_engine(self):
        self._open = None

    def _check_free(self, name):
        if self._open is not None:
            raise RuntimeError(f"{name}: an open engine owns this handle; close it first")

    def _engine_args(self, name, requests, slots, infer_text, return_attn, context, chunk, default_chunk,
                     max_new_cap=None, pool_pages=None):
        """Checks shared by the slot-engine generators -> (requests, slots, chunk, context, max_new_cap, check), where
        ``check`` validates a follow-up request as the up-front ones are (with a KV pool of ``pool_pages`` pages, also
        that it fits in the pool alone; with a ``prompt_key``, that its prompt is that of the key's first live
        request).  The poll interval is `chunk`, else CTB_DECODE_CHUNK, else `default_chunk`
        (None: the smallest ``stream_batch``)."""
        from .engine import MIN_PROMPT_COLS, Request, check_noise_batch, check_prompt_key, pool_pages_needed

        self._check_free(name)
        if infer_text:
            raise ValueError(f"{name}: the mode is chosen per request: set Request.infer_text for text generation")
        if return_attn:
            raise ValueError(f"{name}: return_attn is not supported")
        if not self._handle:
            raise _lib.CtbError("GPT weights not loaded")
        requests = list(requests)
        if not all(isinstance(r, Request) for r in requests):
            raise TypeError("requests must be chattts_b200.engine.Request objects")
        S = min(self.max_batch, len(requests)) if slots is None else int(slots)
        S = max(S, 2)
        if S > self.max_batch:
            raise ValueError(f"slots={S} exceed this handle's max_batch={self.max_batch}")
        cap = max((r.max_new_token for r in requests), default=1) if max_new_cap is None else int(max_new_cap)
        if cap < 1 or cap >= self.max_context:
            raise ValueError(f"max_new_cap={cap} outside [1, max_context={self.max_context})")
        keyed = weakref.WeakValueDictionary()  # prompt key -> the first of its requests still alive

        def check(r):
            if not isinstance(r, Request):
                raise TypeError("requests must be chattts_b200.engine.Request objects")
            T0 = max(MIN_PROMPT_COLS, int(r.emb.shape[0]))
            if T0 + r.max_new_token > self.max_context:
                raise ValueError(f"prompt {int(r.emb.shape[0])} + max_new_token {r.max_new_token} exceed this handle's "
                                 f"max_context={self.max_context}")
            if r.max_new_token > cap:
                raise ValueError(f"max_new_token {r.max_new_token} exceeds max_new_cap={cap}")
            if pool_pages is not None and pool_pages_needed(r) > pool_pages - 1:
                raise ValueError(f"prompt {int(r.emb.shape[0])} + max_new_token {r.max_new_token} need "
                                 f"{pool_pages_needed(r)} KV pages; the pool has {pool_pages - 1} (kv_pool_bytes)")
            check_noise_batch(r, 1 if r.infer_text else self.num_vq, self.max_batch)
            check_prompt_key(r, keyed)

        for r in requests:
            check(r)
        if default_chunk is None:
            default_chunk = min((r.stream_batch for r in requests), default=24)
        env = os.environ.get("CTB_DECODE_CHUNK")
        chunk = (int(env) if env else default_chunk) if chunk is None else int(chunk)
        return requests, S, chunk, (context if context is not None else GPT.Context()), cap, check

    # ------------------------------------------------------------------ the loop
    @torch.no_grad()
    def generate(self, emb: torch.Tensor, inputs_ids: torch.Tensor, temperature: torch.Tensor,
                 eos_token: Union[int, torch.Tensor], attention_mask: Optional[torch.Tensor] = None,
                 max_new_token=2048, min_new_token=0,
                 logits_processors: Tuple[Callable[[torch.LongTensor, torch.FloatTensor], torch.FloatTensor]] = (),
                 infer_text=False, return_attn=False, return_hidden=False, stream=False, show_tqdm=True,
                 ensure_non_empty=True, stream_batch=24, manual_seed: Optional[int] = None,
                 context=Context()):
        """Generator with the reference's contract (gpt.py:315-618).

        ``return_attn=True`` fills ``GenerationOutputs.attentions`` as the reference with eager attention does: one
        entry per step run, each a tuple of ``num_hidden_layers`` fp32 device tensors of softmax probabilities,
        ``[B, heads, T0, T0]`` for the prompt (step 0) and ``[B, heads, 1, T0 + i]`` for step i, whose query is the id
        sampled at step i - 1; columns are the reference's, left padding included.  A padded key column is 0 and a
        padded prompt row uniform (1 / T0); a row's entries for steps after its end (``end_idx``) are 0 (SURVEY.md
        quirk list).  They are computed by a query-only pass over the K / V the decode wrote
        (ctb_gpt_attention_maps), so ids and hidden states are the same with or without them.  With ``stream`` every
        yield carries the steps done so far and the list is extended in place.  The maps take
        ``4 * L * heads * B * (T0**2 + sum(T0 + i for i in 1 .. n - 1))`` bytes of device memory for n steps: about
        170 MB for B = 1, T0 = 100 and 500 steps."""
        self._check_free("generate")
        if not self._handle:
            raise _lib.CtbError("GPT weights not loaded")
        lib = _lib.load()
        dev = self.device_gpt
        B, T0 = int(inputs_ids.shape[0]), int(inputs_ids.shape[1])
        eos = int(eos_token)
        if B > self.max_batch or T0 + max_new_token > self.max_context:
            raise ValueError(f"batch {B} / context {T0}+{max_new_token} exceed this handle "
                             f"(max_batch={self.max_batch}, max_context={self.max_context})")
        rows_per_item = 1 if infer_text else self.num_vq
        V = self.num_text_tokens if infer_text else self.num_audio_tokens
        temps = [float(t) for t in torch.as_tensor(temperature).flatten().tolist()]
        seed = manual_seed
        philox = int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else 0
        cfg = build_sampler_config(logits_processors, temps, eos, min_new_token, philox)
        if cfg.penalty_on and cfg.penalty_max_ids < B * rows_per_item:
            pass  # rows >= max_input_ids silently lose the penalty, like processors.py:24-27

        with torch.cuda.device(dev):
            stream_ptr = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            emb_d = emb.to(dev, torch.float32).contiguous()
            if attention_mask is None:
                attention_mask = torch.ones(B, T0, dtype=torch.bool)
            mask_d = attention_mask.to(dev).to(torch.uint8).contiguous()
            # left padding (tokenizer.py:79-110): every row's valid tokens are a contiguous suffix ending in the last column
            if not bool(mask_d[:, -1].all()) or (T0 > 1 and bool((mask_d[:, 1:] < mask_d[:, :-1]).any())):
                raise ValueError("attention_mask must be left padded: each row 0...0 1...1 with the last column valid")
            q_d = None
            if seed is not None:
                q_d = exp_noise(B * rows_per_item, V, seed).to(dev, non_blocking=True)
            ids_out = torch.zeros(B, max_new_token, self.num_vq, dtype=torch.int32, device=dev)
            hid_out = (torch.zeros(B, max_new_token, self.config.hidden_size, dtype=torch.float32, device=dev)
                       if return_hidden else None)
            end_idx = torch.zeros(B, dtype=torch.int32)
            finish = torch.zeros(B, dtype=torch.uint8)
            st = _lib.GptStatus()

            def query():
                _lib.check(lib.ctb_gpt_status_query(self._handle, C.byref(st), C.c_void_p(end_idx.data_ptr()),
                                                    C.c_void_p(finish.data_ptr()), stream_ptr))

            attentions: List[Optional[Tuple[torch.FloatTensor, ...]]] = []

            def outputs():
                if return_attn:
                    self._extend_attention_maps(attentions, steps, emb_d, mask_d, ids_out, infer_text, stream_ptr)
                ids64 = ids_out.to(torch.int64)
                if inputs_ids.device != ids64.device:
                    ids64 = ids64.to(inputs_ids.device)
                return self._prepare_generation_outputs(ids64, 0, end_idx.clone().long(), attentions,
                                                        hid_out if return_hidden else [], infer_text)

            pbar = None
            if show_tqdm:
                from tqdm import tqdm

                pbar = tqdm(total=max_new_token, desc="text" if infer_text else "code",
                            bar_format="{l_bar}{bar}| {n_fmt}/{total_fmt}(max) [{elapsed}, {rate_fmt}{postfix}]")

            _lib.check(lib.ctb_gpt_begin(
                self._handle, B, T0, C.c_void_p(emb_d.data_ptr()), C.c_void_p(mask_d.data_ptr()), C.byref(cfg),
                C.c_void_p(q_d.data_ptr()) if q_d is not None else None, max_new_token, int(bool(infer_text)),
                C.c_void_p(ids_out.data_ptr()), C.c_void_p(hid_out.data_ptr()) if hid_out is not None else None,
                stream_ptr))
            query()
            if st.any_finished_first_step:
                # gpt.py:527-570
                self.logger.warning("unexpected end at index %s", str([i for i in range(B) if finish[i]]))
                if ensure_non_empty and manual_seed is None:
                    if pbar is not None:
                        pbar.close()
                    self.logger.warning("regenerate in order to ensure non-empty")
                    yield from self.generate(emb, inputs_ids, temperature, eos_token, attention_mask, max_new_token,
                                             min_new_token, logits_processors, infer_text, return_attn,
                                             return_hidden, stream, show_tqdm, ensure_non_empty, stream_batch,
                                             manual_seed, context)
                return

            steps = 1
            chunk = int(stream_batch) if stream else int(os.environ.get("CTB_DECODE_CHUNK", "32"))
            interrupted = False
            while not st.all_finished and steps < max_new_token:
                if context.get():
                    interrupted = True
                    break
                n = min(chunk - (steps % chunk) if stream else chunk, max_new_token - steps)
                _lib.check(lib.ctb_gpt_decode(self._handle, n, stream_ptr))
                query()
                done = st.steps_done
                if done <= steps and not st.all_finished:
                    raise _lib.CtbError(f"decode made no progress (steps_done={done}); device loop state is corrupt")
                if pbar is not None:
                    pbar.update(done - steps)
                steps = done
                # gpt.py:578-589: cumulative yield every `stream_batch` unfinished steps
                if stream and not st.all_finished and steps % stream_batch == 0:
                    yield outputs()
            if pbar is not None:
                pbar.close()
            if stream and st.all_finished and steps - 1 > 0 and (steps - 1) % stream_batch == 0:
                # gpt.py:578-589 quirk: the finishing step does not advance stream_iter, so a boundary
                # reached on the previous step is yielded a second time before the final yield
                yield outputs()
            if not st.all_finished:
                if interrupted or context.get():
                    self.logger.warning("generation is interrupted")
                else:
                    self.logger.warning(f"incomplete result. hit max_new_token: {max_new_token}")
            yield outputs()
