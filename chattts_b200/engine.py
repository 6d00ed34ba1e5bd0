"""Continuous batching of audio-code and text generation: a slot engine on one GPT handle.

The handle's decode rows become ``S`` slots (``ctb_gpt_engine_*`` in include/chattts_b200.h).  Each request - one
utterance: a prompt embedding with its own sampling parameters, seed and token limits, generating audio codes or
(``infer_text``) text tokens - enters a free slot between decode chunks, and its slot is reused as soon as it finishes.
A request's token ids are bit for bit what ``GPT.generate`` returns for it alone (B = 1, same ``manual_seed``, same
``infer_text``), whatever else is in flight.  A request may name a follow-up (``then``), which is queued ahead of
every waiting request when it ends: text refinement followed by the speech codes of the refined text.

The scheduling policy (``schedule``) is plain Python over a small device interface, so it can be driven by a stub.
``stream_schedule`` runs the same policy and reconstructs, per request, the cumulative yields of
``GPT.generate(stream=True)`` from the slots' token counts at each poll.
"""
from __future__ import annotations

import ctypes as C
from collections import deque
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .processors import build_sampler_config, exp_noise

#: shortest prompt the token-parallel prefill takes; shorter prompts are left padded with masked columns
MIN_PROMPT_COLS = 8


@dataclass(eq=False)
class Request:
    """One utterance for ``GPT.generate_continuous``.

    ``emb``: [T, d] prompt embedding (every position valid, as a batch of one has no padding) or [1, T, d].
    The other fields mean what the ``GPT.generate`` arguments of the same name mean; ``infer_text=True`` generates
    text tokens (one temperature, ``eos_token`` the tokenizer's EOS) and its outputs are those of
    ``GPT.generate(infer_text=True)`` for one row: 1-D int64 ids and no hidden states.

    ``then``: called with the request's outputs when it ends at EOS or ``max_new_token`` (a seeded request that ended
    empty included; not on an interrupt); the ``Request`` it returns, if any, is queued ahead of every waiting request
    under the next unused request index."""

    emb: torch.Tensor
    temperature: Sequence[float]
    eos_token: int
    max_new_token: int = 2048
    min_new_token: int = 0
    logits_processors: tuple = ()
    manual_seed: Optional[int] = None
    ensure_non_empty: bool = True
    stream_batch: int = 24
    infer_text: bool = False
    then: Optional[Callable[[object], Optional["Request"]]] = None

    def __post_init__(self):
        if self.emb.dim() == 3:
            if self.emb.shape[0] != 1:
                raise ValueError("Request.emb holds one prompt: [T, d] or [1, T, d]")
            self.emb = self.emb[0]
        if self.emb.dim() != 2 or self.emb.shape[0] < 1:
            raise ValueError("Request.emb must be [T, d] with T >= 1")
        if self.max_new_token < 1:
            raise ValueError("max_new_token must be >= 1")
        if self.stream_batch < 1:
            raise ValueError("stream_batch must be >= 1")
        if self.infer_text and torch.as_tensor(self.temperature).numel() != 1:
            raise ValueError("a text request takes one temperature")


@dataclass
class SlotStatus:
    state: List[int]
    end_idx: List[int]
    finish: List[int]
    steps_done: int = 0


@dataclass
class ScheduleStats:
    """What one ``schedule`` run did: admissions, (device) decode steps and harvested tokens."""

    admissions: int = 0
    admitted: int = 0
    requeued: int = 0
    decode_steps: int = 0
    tokens: int = 0
    interrupted: bool = False
    children: Dict[int, int] = field(default_factory=dict)  # request index -> index of the follow-up it returned


def _follow_up(requests: List[Request], i: int, slot: Optional[int], n: int, dev, check, stats: ScheduleStats):
    """Request ``i`` ended: its follow-up's index as a list (empty without one)."""
    then = requests[i].then
    if then is None:
        return []
    child = then(dev.empty(i) if slot is None else dev.harvest(slot, n))
    if child is None:
        return []
    if not isinstance(child, Request):
        raise TypeError("Request.then must return a Request or None")
    if check is not None:
        check(child)
    requests.append(child)
    stats.children[i] = len(requests) - 1
    return [len(requests) - 1]


def _poll_cycles(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
                 check: Optional[Callable[[Request], None]] = None
                 ) -> Iterator[Tuple[SlotStatus, List[Optional[int]], list]]:
    """The scheduling policy of ``schedule``: yields once per poll ``(status, owner, ended)`` - the slots' status, the
    request each slot held when it was read, and the requests that ended at this poll as ``(request_index, slot or
    None, n_tokens, eos)``.  The slots of the ended requests are refilled only after the generator is resumed.

    A request's follow-up (``Request.then``, called here while the slot's outputs are valid and checked by ``check``)
    is appended to ``requests`` and queued ahead of the waiting requests, so the refill after this poll admits it."""
    stats = stats if stats is not None else ScheduleStats()
    waiting = deque(range(len(requests)))
    owner: List[Optional[int]] = [None] * dev.slots
    while True:
        free = [s for s in range(dev.slots) if owner[s] is None]
        batch = []
        while free and waiting:
            s, i = free.pop(0), waiting.popleft()
            owner[s] = i
            batch.append((s, i))
        if batch:
            dev.admit(batch)
            stats.admissions += 1
            stats.admitted += len(batch)
        st = dev.status()
        stats.decode_steps = st.steps_done
        polled = list(owner)
        ended = []
        follow: List[int] = []
        freed = False
        for s in range(dev.slots):
            i = owner[s]
            if i is None or st.state[s] != _lib.SLOT_FINISHED:
                continue
            owner[s] = None
            freed = True
            if st.end_idx[s] == 0 and st.finish[s]:
                r = requests[i]
                if r.manual_seed is None and r.ensure_non_empty:
                    waiting.appendleft(i)  # regenerate (gpt.py:527-570); a fresh Philox seed is drawn at admission
                    stats.requeued += 1
                    continue
                ended.append((i, None, 0, True))
                follow += _follow_up(requests, i, None, 0, dev, check, stats)
                continue
            stats.tokens += st.end_idx[s]
            ended.append((i, s, st.end_idx[s], bool(st.finish[s])))
            follow += _follow_up(requests, i, s, st.end_idx[s], dev, check, stats)
        waiting.extendleft(reversed(follow))  # ahead of the waiting requests, in slot order
        if freed and waiting:
            yield st, polled, ended
            continue  # refill the freed slots before the next chunk
        running = [s for s in range(dev.slots) if owner[s] is not None]
        interrupted = bool(running) and context is not None and context.get()
        if interrupted:
            stats.interrupted = True
            for s in running:
                stats.tokens += st.end_idx[s]
                ended.append((owner[s], s, st.end_idx[s], False))
        yield st, polled, ended
        if not running or interrupted:
            return
        dev.decode(chunk)


def schedule(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
             check: Optional[Callable[[Request], None]] = None) -> Iterator[Tuple[int, Optional[int], int]]:
    """Drive ``dev`` (``slots``, ``admit([(slot, request_index)])``, ``decode(n)``, ``status() -> SlotStatus``) until
    every request has finished; yields ``(request_index, slot, n_tokens)`` as each one completes - the caller harvests
    the slot's first ``n_tokens`` outputs before resuming the generator - or ``(request_index, None, 0)`` for a seeded
    request whose first token is EOS (it ends empty, gpt.py:527).  An unseeded one with ``ensure_non_empty`` is queued
    again instead.

    Waiting requests enter free slots in order, lowest slot first, at every poll (every ``chunk`` decode steps).  On a
    ``context`` interrupt the running requests are yielded with what they have so far and the waiting ones are dropped.
    Follow-ups (``Request.then``) need ``dev.harvest(slot, n)`` and ``dev.empty(request_index)``; see ``_poll_cycles``.
    """
    for _, _, ended in _poll_cycles(requests, dev, chunk, context, stats, check):
        for i, s, n, _ in ended:
            yield i, s, n


def stream_schedule(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
                    check: Optional[Callable[[Request], None]] = None
                    ) -> Iterator[List[Tuple[int, Optional[int], int, bool]]]:
    """``schedule``'s policy, yielding once per poll the list of ``(request_index, slot, n_tokens, last)``: for each
    request, the yields ``GPT.generate(stream=True, stream_batch=r.stream_batch)`` makes for it alone, in its order,
    as cumulative token counts (the slot's first ``n_tokens`` outputs; slot None: a seeded request that ended empty).

    The static loop (gpt.py here, generate) yields at every multiple of ``stream_batch`` (from step 2 on) that the row
    reaches unfinished, yields a boundary a second time when EOS follows it on the very next step, and ends with the
    final yield; a row that stops at ``max_new_token`` is not finished there, so it gets no second yield.  Tokens only
    ever append to a slot, so each poll rebuilds every boundary a slot crossed since the last one from its token count:
    the yields do not depend on ``chunk``.  The slots' outputs stay in place until the generator is resumed."""
    sent: Dict[int, int] = {}  # last boundary yielded per request
    for st, owner, ended in _poll_cycles(requests, dev, chunk, context, stats, check):
        out = []
        for s, i in enumerate(owner):
            if i is None:
                continue
            sb = requests[i].stream_batch
            nxt = sent.get(i, 0) + sb
            if nxt < 2:  # step 1 (the prefill's token) is never a boundary
                nxt += sb
            # running: end_idx steps so far, all unfinished; EOS at step end_idx + 1; max_new: end_idx = max_new
            while nxt <= st.end_idx[s]:
                out.append((i, s, nxt, False))
                sent[i] = nxt
                nxt += sb
        for i, s, n, eos in ended:
            if s is not None and eos and n > 0 and n % requests[i].stream_batch == 0:
                out.append((i, s, n, False))  # the boundary before the finishing step, again (gpt.py:381-384)
            out.append((i, s, n, True))
        if out:
            yield out


class EngineDevice:
    """The device layer of ``schedule`` on a GPT handle (ctb_gpt_engine_begin / _admit / _status, ctb_gpt_decode)."""

    def __init__(self, gpt, requests: Sequence[Request], slots: int, max_new_cap: int, return_hidden: bool = True):
        self.gpt, self.requests, self.slots = gpt, requests, slots
        self.lib = _lib.load()
        dev = gpt.device_gpt
        self.dev = dev
        self.stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        self.ids_out = torch.zeros(slots, max_new_cap, gpt.num_vq, dtype=torch.int32, device=dev)
        self.hid_out = (torch.zeros(slots, max_new_cap, gpt.config.hidden_size, dtype=torch.float32, device=dev)
                        if return_hidden else None)
        _lib.check(self.lib.ctb_gpt_engine_begin(
            gpt._handle, slots, max_new_cap, C.c_void_p(self.ids_out.data_ptr()),
            C.c_void_p(self.hid_out.data_ptr()) if self.hid_out is not None else None, self.stream))
        self._state = (C.c_int32 * slots)()
        self._end = torch.zeros(slots, dtype=torch.int32)
        self._fin = torch.zeros(slots, dtype=torch.uint8)
        self._text = [False] * slots  # mode of the request each slot was last given

    def admit(self, batch: List[Tuple[int, int]]) -> None:
        # one prefill per kind: seeded requests bring their Exp(1) rows, unseeded ones sample with device Philox; code
        # and text requests are admitted by separate calls
        for seeded, text in ((True, False), (True, True), (False, False), (False, True)):
            group = [(s, i) for s, i in batch if (self.requests[i].manual_seed is not None) == seeded
                     and bool(self.requests[i].infer_text) == text]
            if not group:
                continue
            # the prompts share one padded width; a request whose max_new no longer fits its slot's max_context
            # next to that width is admitted on its own
            T0 = max(MIN_PROMPT_COLS, max(int(self.requests[i].emb.shape[0]) for _, i in group))
            alone = [(s, i) for s, i in group if T0 + self.requests[i].max_new_token > self.gpt.max_context]
            rest = [p for p in group if p not in alone]
            for part in ([rest] if rest else []) + [[p] for p in alone]:
                self._admit(part, seeded, text)

    def _admit(self, group, seeded: bool, text: bool) -> None:
        gpt, n = self.gpt, len(group)
        reqs = [self.requests[i] for _, i in group]
        T0 = max(MIN_PROMPT_COLS, max(int(r.emb.shape[0]) for r in reqs))
        d = gpt.config.hidden_size
        emb = torch.zeros(n, T0, d, dtype=torch.float32, device=self.dev)
        mask = torch.zeros(n, T0, dtype=torch.uint8, device=self.dev)
        for k, r in enumerate(reqs):  # left padding: the prompt is a suffix of its row
            T = int(r.emb.shape[0])
            emb[k, T0 - T:] = r.emb.to(self.dev, torch.float32)
            mask[k, T0 - T:] = 1
        cfgs = (_lib.SamplerConfig * n)()
        for k, r in enumerate(reqs):
            temps = [float(t) for t in torch.as_tensor(r.temperature).flatten().tolist()]
            philox = 0 if seeded else int(torch.randint(0, 2 ** 62, (1,)).item())
            cfgs[k] = build_sampler_config(r.logits_processors, temps, int(r.eos_token), r.min_new_token, philox)
        noise = None
        if seeded:  # the rows GPT.generate draws for a batch of one with this seed
            rows, cols = (1, gpt.num_text_tokens) if text else (gpt.num_vq, gpt.num_audio_tokens)
            noise = torch.cat([exp_noise(rows, cols, r.manual_seed) for r in reqs]).to(self.dev)
        slots = (C.c_int32 * n)(*[s for s, _ in group])
        max_new = (C.c_int32 * n)(*[r.max_new_token for r in reqs])
        for s, _ in group:
            self._text[s] = text
        admit = self.lib.ctb_gpt_engine_admit_text if text else self.lib.ctb_gpt_engine_admit
        _lib.check(admit(
            gpt._handle, n, slots, T0, C.c_void_p(emb.data_ptr()), C.c_void_p(mask.data_ptr()), cfgs,
            C.c_void_p(noise.data_ptr()) if noise is not None else None, max_new, self.stream))

    def decode(self, n: int) -> None:
        _lib.check(self.lib.ctb_gpt_decode(self.gpt._handle, n, self.stream))

    def status(self) -> SlotStatus:
        st = _lib.GptStatus()
        _lib.check(self.lib.ctb_gpt_engine_status(self.gpt._handle, C.byref(st), self._state,
                                                  C.c_void_p(self._end.data_ptr()), C.c_void_p(self._fin.data_ptr()),
                                                  self.stream))
        return SlotStatus(list(self._state), self._end.tolist(), self._fin.tolist(), int(st.steps_done))

    def harvest(self, slot: int, n: int, copy: bool = True):
        """GenerationOutputs of the request in ``slot``: its first ``n`` ids (int64 copies) and hidden states (copies,
        or with ``copy=False`` views into the engine buffer, valid until the engine decodes or admits again).  A text
        request's ids are 1-D and it has no hidden states, as ``GPT.generate(infer_text=True)`` returns them."""
        from .gpt import GPT

        if self._text[slot]:
            return GPT.GenerationOutputs(ids=[self.ids_out[slot, :n, 0].to(torch.int64)], attentions=[], hiddens=[])
        ids = self.ids_out[slot, :n].to(torch.int64)
        hid = ([self.hid_out[slot, :n].clone() if copy else self.hid_out[slot, :n]] if self.hid_out is not None
               else [])
        return GPT.GenerationOutputs(ids=[ids], attentions=[], hiddens=hid)

    def empty(self, index: Optional[int] = None):
        """The outputs of request ``index`` (default: a code request) when it ended empty (a seeded request whose
        first token was EOS)."""
        from .gpt import GPT

        if index is not None and self.requests[index].infer_text:
            return GPT.GenerationOutputs(ids=[torch.zeros(0, dtype=torch.int64, device=self.dev)], attentions=[],
                                         hiddens=[])
        ids = torch.zeros(0, self.gpt.num_vq, dtype=torch.int64, device=self.dev)
        hid = ([torch.zeros(0, self.gpt.config.hidden_size, dtype=torch.float32, device=self.dev)]
               if self.hid_out is not None else [])
        return GPT.GenerationOutputs(ids=[ids], attentions=[], hiddens=hid)
