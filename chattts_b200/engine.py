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

An opt-in prefill budget (``prefill_budget``, prompt columns per poll) bounds the prefill work the running slots wait
for at each poll: a prompt that does not fit is prefilled in chunks over several polls (``ctb_gpt_engine_prefill_chunk``),
with the same bits as one admission of it.

An opt-in KV pool (``kv_pool_bytes``) bounds the engine's KV memory: slots take 16-token pages from a shared pool as
they grow, and when the pool runs short a running request is suspended to host memory and later resumed, in any
slot, bit for bit as if it had never moved (``_poll_cycles`` has the policy).
"""
from __future__ import annotations

import ctypes as C
import itertools
import logging
import queue
import threading
import weakref
from collections import deque
from concurrent.futures import Future
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Set, Tuple

import torch

from . import _lib
from .processors import build_sampler_config, exp_noise

#: shortest prompt the token-parallel prefill takes; shorter prompts are left padded with masked columns
MIN_PROMPT_COLS = 8
#: widest prefill whose attention keeps the short-prompt kernel (k_prefill_attn); a longer prompt takes the tiled
#: kernel and is prefilled on its own (``admission_groups``)
LONG_PROMPT_COLS = 1024
#: most prompt rows (prompts x padded width) one admission prefill takes.  Its activation scratch is sized per call and
#: kept by the handle (3.8 GB for 64 prompts of 1,024 tokens); larger admissions run as consecutive prefills of up to
#: this many rows, so an engine of 64 slots needs no more of it (1.9 GB) than one of 32 did.
ADMIT_MAX_ROWS = 32 * 1024
#: a prompt prefilled in chunks: every chunk starts at a multiple of this many columns, and every chunk but its last
#: is a multiple of it (``ctb_gpt_engine_prefill_chunk``)
PREFILL_CHUNK_ALIGN = _lib.PREFILL_CHUNK_ALIGN


def admission_chunks(group: list, T0: int) -> List[list]:
    """``group`` (one admission's prompts, padded to ``T0`` columns) as consecutive runs of at most
    ``ADMIT_MAX_ROWS // T0`` prompts."""
    n = max(1, ADMIT_MAX_ROWS // T0)
    return [group[i: i + n] for i in range(0, len(group), n)]


def admission_prefills(batch: list, requests: Sequence["Request"], max_context: int) -> List[Tuple[list, int, bool, bool]]:
    """The prefill calls ``EngineDevice.admit(batch)`` makes, in order: ``[(pairs, T0, seeded, text)]``.  Seeded
    requests bring their Exp(1) rows, unseeded ones sample with device Philox, and code and text requests are
    admitted by separate calls; each kind is split by ``admission_groups`` and ``admission_chunks``."""
    out = []
    for seeded, text in ((True, False), (True, True), (False, False), (False, True)):
        group = [(s, i) for s, i in batch if (requests[i].manual_seed is not None) == seeded
                 and bool(requests[i].infer_text) == text]
        if not group:
            continue
        for part, T0 in admission_groups(group, requests, max_context):
            for chunk in admission_chunks(part, T0):  # each prompt's results do not depend on its batch
                out.append((chunk, T0, seeded, text))
    return out


def admission_cols(batch: list, requests: Sequence["Request"], max_context: int) -> int:
    """Padded prompt columns ``EngineDevice.admit(batch)`` prefills: prompts x ``T0`` of each of its calls."""
    return sum(len(pairs) * T0 for pairs, T0, _, _ in admission_prefills(batch, requests, max_context))


def check_prefill_budget(budget: Optional[int]) -> Optional[int]:
    """``budget`` as an int of at least ``PREFILL_CHUNK_ALIGN`` (128) prompt columns, or None; ValueError otherwise."""
    if budget is None:
        return None
    if int(budget) != budget or int(budget) < PREFILL_CHUNK_ALIGN:
        raise ValueError(f"prefill_budget={budget!r}: an int of at least {PREFILL_CHUNK_ALIGN} prompt columns, or None")
    return int(budget)


TOP_LOGPROBS_MAX = 20  # the most alternatives per token ctb_gpt_engine_top_logprobs and ctb_gpt_score_ex return


def check_top_logprobs(n) -> int:
    """``top_logprobs`` as an int in [0, 20] (0: off); ValueError otherwise."""
    if isinstance(n, bool) or not isinstance(n, int) or not 0 <= n <= TOP_LOGPROBS_MAX:
        raise ValueError(f"top_logprobs={n!r}: an int in [0, {TOP_LOGPROBS_MAX}] (0: off)")
    return n


def kv_pool_pages(gpt_config, kv_pool_bytes: Optional[int], flags: int) -> Optional[int]:
    """The pages (16 tokens of K and V of every layer; page 0 is the zero page) a pool of ``kv_pool_bytes`` holds on an
    engine of precision ``flags``, or None for None.  ValueError when it holds fewer than two."""
    if kv_pool_bytes is None:
        return None
    c = gpt_config
    elem = 2 if flags & _lib.ENGINE_FP16_KV else 4
    page = 2 * c.num_key_value_heads * _lib.PAGE_TOKENS * c.head_dim * elem
    pages = int(kv_pool_bytes) // (page * c.num_hidden_layers)
    if int(kv_pool_bytes) != kv_pool_bytes or pages < 2:
        raise ValueError(f"kv_pool_bytes={kv_pool_bytes!r}: an int of at least two pages "
                         f"({2 * page * c.num_hidden_layers} bytes), or None")
    return pages


def pool_pages_needed(r: "Request") -> int:
    """Pages request ``r`` holds at most on a paged engine: its prompt plus ``max_new_token`` positions."""
    return -(-(int(r.emb.shape[0]) + r.max_new_token) // _lib.PAGE_TOKENS)


def admission_groups(group: list, requests: Sequence["Request"], max_context: int) -> List[Tuple[list, int]]:
    """``group`` (one admission's ``(slot, request index)`` pairs of one kind) as the prefills it runs as, each with
    its padded width: ``[(pairs, T0)]``.

    Prompts of up to ``LONG_PROMPT_COLS`` tokens share one width, and a request whose ``max_new_token`` no longer fits
    its slot's ``max_context`` next to that width is admitted on its own.  A longer prompt is always prefilled on its
    own, after them, so it never pads a short prompt to its width."""
    def cols(pairs):
        return max(MIN_PROMPT_COLS, max(int(requests[i].emb.shape[0]) for _, i in pairs))

    short = [(s, i) for s, i in group if int(requests[i].emb.shape[0]) <= LONG_PROMPT_COLS]
    out = []
    if short:
        T0 = cols(short)
        alone = [(s, i) for s, i in short if T0 + requests[i].max_new_token > max_context]
        rest = [p for p in short if p not in alone]
        out += [(part, T0) for part in ([rest] if rest else [])] + [([p], T0) for p in alone]
    return out + [([p], cols([p])) for p in group if int(requests[p[1]].emb.shape[0]) > LONG_PROMPT_COLS]


@dataclass(eq=False)
class Request:
    """One utterance for ``GPT.generate_continuous``.

    ``emb``: [T, d] prompt embedding (every position valid, as a batch of one has no padding) or [1, T, d];
    ``T + max_new_token`` at most the handle's ``max_context``.  A prompt of more than ``LONG_PROMPT_COLS`` (1,024)
    tokens is prefilled on its own with the tiled attention kernel (``GPT.generate_continuous`` on what that means
    for equality with ``GPT.generate``).
    The other fields mean what the ``GPT.generate`` arguments of the same name mean; ``infer_text=True`` generates
    text tokens (one temperature, ``eos_token`` the tokenizer's EOS) and its outputs are those of
    ``GPT.generate(infer_text=True)`` for one row: 1-D int64 ids and no hidden states.

    ``then``: called with the request's outputs when it ends at EOS or ``max_new_token`` (a seeded request that ended
    empty included; not on an interrupt); the ``Request`` it returns, if any, is queued ahead of every waiting request
    under the next unused request index.  It may also return a list of requests (a fan-out): all of them are queued
    ahead of the waiting requests, in list order, under consecutive indices.

    ``prepare``: per-poll device work the follow-ups depend on.  When requests with a ``then`` end at a poll, each
    distinct ``prepare`` among them is called once, before any of their ``then``, as ``prepare(dev, [(request, slot,
    n_tokens)])`` with every one of them that names it (slot None for a seeded request that ended empty); the slots'
    outputs are valid in ``dev``'s buffers.  This is how the work of every request ending at one poll is batched.

    ``noise_batch``: ``(B, b)`` - a seeded request samples as row ``b`` of a static ``GPT.generate`` batch of ``B``
    with the same seed: it draws rows ``b * rows ... (b + 1) * rows - 1`` of that batch's Exp(1) noise (``rows``: 1
    for text, ``num_vq`` for codes) instead of the rows of a batch of one.  Nothing else the sampler computes depends
    on the row, as long as the repetition penalty covers the row (``check_noise_batch``).  ``None`` and ``(1, 0)`` are
    a batch of one; an unseeded request ignores it.

    ``prompt_key``: any hashable (default None: none).  Requests with equal keys promise the same ``emb`` and
    ``infer_text`` (checked against the first live request of the key when they are submitted): several takes of one
    utterance.  When one of them is running in a slot, a waiting one is admitted by sharing that slot's KV for prompt
    columns ``[0, c0)``, ``c0 = 128 * floor((T - 1) / 128)`` (``shared_prompt_cols``), and prefilling only ``[c0, T)``
    (``ctb_gpt_engine_share_prompt`` and the final prefill chunk); its outputs are bit for bit those of its normal
    admission.  Prompts of 128 tokens or fewer are admitted as usual."""

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
    then: Optional[Callable[[object], object]] = None
    prepare: Optional[Callable[[object, list], None]] = None
    noise_batch: Optional[Tuple[int, int]] = None
    prompt_key: object = None

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
        if self.noise_batch is not None:
            B, b = (int(x) for x in self.noise_batch)
            self.noise_batch = (B, b)
            check_noise_batch(self, 1 if self.infer_text else None)


def shared_prompt_cols(T: int) -> int:
    """Columns of a prompt of ``T`` tokens that a request sharing another slot's prompt takes from it: the last chunk
    boundary (a multiple of ``PREFILL_CHUNK_ALIGN``) before its last column, 0 for prompts of up to 128 tokens."""
    return (T - 1) // PREFILL_CHUNK_ALIGN * PREFILL_CHUNK_ALIGN


def check_prompt_key(r: Request, first: "weakref.WeakValueDictionary") -> None:
    """Raise ``ValueError`` unless ``r`` has the prompt (``emb``, ``infer_text``) of ``first[r.prompt_key]``, the first
    request of its key still alive; ``r`` becomes that one when there is none."""
    if r.prompt_key is None:
        return
    f = first.get(r.prompt_key)
    if f is None:
        first[r.prompt_key] = r
        return
    if (f.emb.shape != r.emb.shape or bool(f.infer_text) != bool(r.infer_text)
            or not torch.equal(f.emb, r.emb.to(f.emb.device, f.emb.dtype))):
        raise ValueError(f"prompt_key {r.prompt_key!r}: the request's prompt differs from that of the key's first "
                         f"request (same emb and infer_text required)")


def check_noise_batch(r: Request, rows: Optional[int], max_batch: Optional[int] = None) -> None:
    """Raise ``ValueError`` unless ``r.noise_batch`` = ``(B, b)`` names a row of a static batch the request can sample
    as: ``0 <= b < B``, ``B`` at most ``max_batch``, and with a repetition penalty every one of the row's ``rows``
    noise rows below the penalty's ``max_input_ids`` (the static sampler drops the penalty from rows at or past it,
    the engine never does).  ``rows`` None skips the penalty check."""
    if r.noise_batch is None:
        return
    B, b = r.noise_batch
    if B < 1 or not 0 <= b < B:
        raise ValueError(f"noise_batch {r.noise_batch}: needs 0 <= b < B")
    if max_batch is not None and B > max_batch:
        raise ValueError(f"noise_batch {r.noise_batch}: B exceeds this handle's max_batch={max_batch}")
    if rows is None:
        return
    for proc in r.logits_processors:
        if hasattr(proc, "penalty") and hasattr(proc, "past_window") and hasattr(proc, "max_input_ids"):
            if (b + 1) * rows > int(proc.max_input_ids):
                raise ValueError(f"noise_batch {r.noise_batch}: row {b} of the static batch would lose its repetition "
                                 f"penalty (rows {b * rows}..{(b + 1) * rows - 1}, max_input_ids "
                                 f"{proc.max_input_ids})")


def noise_rows(reqs: Sequence[Request], rows: int, cols: int, cache: Dict[tuple, torch.Tensor]) -> torch.Tensor:
    """The Exp(1) noise of the seeded requests ``reqs`` ([len(reqs) * rows, cols], on the host): for each one, rows
    ``b * rows ... (b + 1) * rows - 1`` of ``exp_noise(B * rows, cols, manual_seed)``, ``(B, b)`` its ``noise_batch``
    (default a batch of one).  The full batch's noise is built once per ``(B, rows, cols, seed)`` in ``cache`` and the
    rows are sliced from it."""
    parts = []
    for r in reqs:
        B, b = r.noise_batch or (1, 0)
        key = (B, rows, cols, r.manual_seed)
        if key not in cache:
            cache[key] = exp_noise(B * rows, cols, r.manual_seed)
        parts.append(cache[key][b * rows: (b + 1) * rows])
    return torch.cat(parts)


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
    fanout: Dict[int, List[int]] = field(default_factory=dict)  # request index -> indices of the list ``then`` returned
    cancelled: Set[int] = field(default_factory=set)  # request indices stopped by an ``Arrivals.cancel``
    # with a prefill budget: the prompt columns prefilled in each poll (the admissions and chunks between two decode
    # chunks), and the number of prompt chunks issued
    prefill_cols: List[int] = field(default_factory=list)
    chunks: int = 0
    # with a KV pool: pages mapped at each poll (as its decode chunk starts), their peak, requests suspended and
    # resumed, and host bytes their images held at each poll
    pages: List[int] = field(default_factory=list)
    peak_pages: int = 0
    suspensions: int = 0
    resumes: int = 0
    host_bytes: List[int] = field(default_factory=list)
    # shared prompts (Request.prompt_key): requests admitted by sharing another slot's prompt, the prompt columns they
    # did not prefill, and (KV pool) the peak of pages mapped by more than one slot
    shares: int = 0
    shared_cols: int = 0
    peak_shared_pages: int = 0
    keys: Dict[int, object] = field(default_factory=dict)  # open source: index of a submitted request -> its key
    failed: Dict[int, BaseException] = field(default_factory=dict)  # open source: request index -> its follow-up's error


class Arrivals:
    """The request source of an open engine: requests submitted and cancelled from any thread, taken by the scheduling
    loop at each poll.  Each submission carries a key (an open engine's ``Job``; by default the request itself), so one
    ``Request`` may be submitted several times under different keys; ``cancel(key)`` stops every stage of that
    submission that is live (its follow-ups and fan-outs included).  A submission may be a list of requests, queued
    in list order, which are stages of one submission from the start."""

    def __init__(self):
        self._cv = threading.Condition()
        self._new: List[Tuple[object, object]] = []  # (key, Request or list of Requests)
        self._cancel: List[object] = []
        self.closed = False

    def submit(self, r, key=None) -> None:
        self.submit_all([(r if key is None else key, r)])

    def submit_all(self, items: List[Tuple[object, object]]) -> None:
        """Queue ``[(key, request or list of requests)]`` in one step: the loop takes all of them at the same poll."""
        with self._cv:
            if self.closed:
                raise RuntimeError("the engine is closed")
            self._new += items
            self._cv.notify()

    def cancel(self, key) -> None:
        with self._cv:
            self._cancel.append(key)
            self._cv.notify()

    def close(self) -> None:
        with self._cv:
            self.closed = True
            self._cv.notify()

    def take(self, block: bool) -> Tuple[List[Tuple[object, object]], List[object], bool]:
        """``([(key, request)] submitted, [key] cancelled, closed)`` since the last call; with ``block``, waits until
        there is one of them."""
        with self._cv:
            while block and not self._new and not self._cancel and not self.closed:
                self._cv.wait()
            new, cancel, self._new, self._cancel = self._new, self._cancel, [], []
            return new, cancel, self.closed


def _prepare(requests: List[Request], done, dev, stats: ScheduleStats, source: Optional[Arrivals] = None) -> None:
    """One call of each distinct ``Request.prepare`` among the requests ``done`` (``(index, slot, n_tokens, _)``) that
    ended at this poll with a ``then``.  With an open ``source`` a failure is recorded in ``stats.failed`` for every
    request of that call (their ``then`` is not called) instead of stopping the loop."""
    groups: Dict[Callable, list] = {}
    for i, s, n, _ in done:
        r = requests[i]
        if r.then is not None and r.prepare is not None:
            groups.setdefault(r.prepare, []).append((i, s, n))
    for fn, items in groups.items():
        try:
            fn(dev, [(requests[i], s, n) for i, s, n in items])
        except Exception as e:
            if source is None:
                raise
            for i, _, _ in items:
                stats.failed[i] = e


def _follow_up(requests: List[Request], i: int, slot: Optional[int], n: int, dev, check, stats: ScheduleStats,
               source: Optional[Arrivals] = None):
    """Request ``i`` ended: the indices of its follow-ups (empty without one).  With an open ``source`` a follow-up
    that fails (``then`` raises or ``check`` rejects one of a fan-out) is recorded in ``stats.failed`` instead of
    stopping the loop."""
    then = requests[i].then
    if then is None or i in stats.failed:
        return []
    try:
        child = then(dev.empty(i) if slot is None else dev.harvest(slot, n))
        if child is None:
            return []
        kids = list(child) if isinstance(child, (list, tuple)) else [child]
        if not all(isinstance(c, Request) for c in kids):
            raise TypeError("Request.then must return a Request, a list of Requests or None")
        if check is not None:
            for c in kids:
                check(c)
    except Exception as e:
        if source is None:
            raise
        stats.failed[i] = e
        return []
    if not kids:
        return []
    first = len(requests)
    for c in kids:
        requests.append(c)
    idx = list(range(first, first + len(kids)))
    if isinstance(child, Request):
        stats.children[i] = idx[0]
    else:
        stats.fanout[i] = idx
    return idx


def _poll_cycles(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
                 check: Optional[Callable[[Request], None]] = None, source: Optional[Arrivals] = None,
                 prefill_budget: Optional[int] = None) -> Iterator[Tuple[SlotStatus, List[Optional[int]], list]]:
    """The scheduling policy of ``schedule``: yields once per poll ``(status, owner, ended)`` - the slots' status, the
    request each slot held when it was read, and the requests that ended at this poll as ``(request_index, slot or
    None, n_tokens, eos)``.  The slots of the ended requests are refilled only after the generator is resumed.

    A request's follow-up (``Request.then``, called here while the slot's outputs are valid and checked by ``check``)
    is appended to ``requests`` and queued ahead of the waiting requests, so the refill after this poll admits it.

    ``source`` (open engine): every poll first takes the requests submitted since the last one (appended to
    ``requests`` and queued behind the waiting ones; ``stats.keys`` maps each one's index to its submission key) and
    the cancellations.  A cancelled waiting request leaves the
    queue and ends empty without touching a slot; a cancelled running request is stopped with ``dev.cancel`` right
    after the status read, so it ends with the ``end_idx`` tokens that read reported (a request the same read shows
    finished is finished); neither calls its ``then``, and cancelling a request whose follow-up was already made
    cancels the follow-up.  A submission's live stages are all cancelled together (a fan-out runs several).  Cancelled
    requests are listed in ``stats.cancelled``.  With nothing running and nothing
    waiting the loop blocks in ``source.take`` instead of decoding, and it ends once the source is closed and drained.

    ``prefill_budget`` (prompt columns, at least 128; None: no bound) bounds the prefill of each poll - the admissions
    and chunks between two decode chunks - with ``dev.prefill_chunk(slot, index, c0, n)`` and ``dev.max_context``:

    1. A prompt in progress (at most one) first advances by ``min(remaining, budget left rounded down to 128)``
       columns; its final chunk admits the request.
    2. With no prompt in progress, waiting requests then enter free slots in order, lowest slot first, while the
       padded columns of the poll's admission (``admission_cols``) stay within the budget left.
    3. The first request that does not fit takes a free slot and becomes the prompt in progress, starting with the
       budget left over (rounded down to 128) if that is at least 128 columns, else at the next poll; the requests
       behind it wait.
    4. Its slot is reserved: not refilled, and its status is not read for it until its final chunk.  A cancel frees
       the slot at the next poll (``dev.cancel`` drops the prompt in progress; the request ends empty, without a
       follow-up); an interrupt drops it as it drops the waiting requests.

    ``stats.prefill_cols`` records each poll's prefilled columns, ``stats.chunks`` the chunks.

    A device with a KV pool (``dev.pool_pages`` not None: ``dev.reserve(slots, tokens) -> bool``, ``dev.release(slots)``,
    ``dev.suspend(slot) -> image``, ``dev.resume(slot, image)``, ``dev.pages_in_use``, ``dev.host_bytes``) maps pages
    as the slots grow.  A request of prompt ``T`` never holds more than ``T + max_new_token`` positions, and every
    mapping below is capped there:

    1. Before an admission, or a chunk ending at column ``c``, the slot is mapped up to ``T`` (``c``) plus ``chunk``
       positions.  When the pool cannot cover it, the request waits at the head of the queue (a chunk waits for the
       next poll).
    2. Before each decode chunk every running slot is mapped up to ``seq_len + chunk + 1`` positions (``T`` plus its
       tokens plus ``chunk``), all in one call.  When the pool cannot cover them all, the running request admitted
       last is suspended (``dev.suspend``: its state and KV go to host memory, its slot and pages are freed) and the
       call is repeated, until the rest fit.  A prompt in progress is never suspended.
    3. Suspended requests are served before the waiting queue: at each poll, in admission order, each takes the
       lowest free slot as soon as its tokens plus ``chunk`` fit together with one more chunk for every running slot
       (mapped in the same call, so the decode that follows cannot suspend it again at once), and no waiting request
       is admitted while one is suspended.  A resumed request continues bit for bit as if it had not moved.
    4. Pages are released when a slot's request ends (harvest, cancel, requeue) or its prompt in progress is dropped.
    5. A cancelled suspended request ends with the tokens it had (its image becomes the ``slot`` of its ``ended``
       entry: ``dev.harvest`` reads it); an interrupt ends suspended requests as it ends running ones.

    ``stats`` records the pages mapped at each poll and their peak, the suspensions, the resumes and the host bytes
    held by images.  Without a pool none of these calls are made.

    Shared prompts (``Request.prompt_key``; ``dev.share(src, dst, index, c0) -> bool``, ``dev.shared_pages``): a
    holder of a key is a running slot (not suspended, not resumed) whose request has the key and whose prompt was
    prefilled there, wholly or by chunks, or shared.  A waiting keyed request of ``T > 128`` tokens whose key has a
    holder takes its place in the queue as usual, but is admitted by ``dev.share(holder, slot, index, c0)`` (``c0 =
    shared_prompt_cols(T)``) and the final chunk ``dev.prefill_chunk(slot, index, c0, T - c0)``.  Several members
    waiting at one poll with no holder: the first is admitted normally and the others share from it at the same poll.
    The shares of a poll follow its admission call on the same stream.  A member that finds no holder is an
    ordinary request.  A share's final chunk costs ``T - c0`` columns of the prefill budget; when they do not fit, the
    member waits at the head of the queue for the next poll.  With a KV pool, a share needs pages for positions
    ``[c0, T + chunk)`` only: when the pool (counted in physical pages) cannot cover them, it waits at the head of the
    queue.  A suspended member resumes into pages of its own, and a resumed request is no holder.  ``stats`` records
    the shares, the prompt columns they did not prefill, and the peak of shared pages."""
    stats = stats if stats is not None else ScheduleStats()
    pool = getattr(dev, "pool_pages", None)
    admitted_at: Dict[int, int] = {}  # request index -> admission number (suspension victims: the highest)
    suspended: List[list] = []  # [request index, image, tokens], in admission order

    mapped: Dict[int, int] = {}  # slot -> positions its pages hold

    def reserve(slots: List[int], tokens: List[int]) -> bool:
        if not dev.reserve(slots, tokens):
            return False
        for s, t in zip(slots, tokens):
            mapped[s] = max(mapped.get(s, 0), t)
        return True

    def limit(i: int, n: int) -> int:  # n positions plus one chunk, capped at what request i can ever hold
        r = requests[i]
        return min(n + chunk, int(r.emb.shape[0]) + r.max_new_token)

    def held(i: int, n: int) -> int:  # positions request i holds with n tokens generated (and one more appended)
        return int(requests[i].emb.shape[0]) + n

    admission_no = itertools.count()

    def note_admitted(i: int) -> None:
        admitted_at[i] = next(admission_no)

    holders: Dict[int, Tuple[object, int]] = {}  # slot -> (prompt key, request index) of a request admitted there

    def holder(key) -> Optional[int]:
        for s, (k, i) in holders.items():
            if k == key and owner[s] == i:
                return s
        return None
    budget = prefill_budget
    prog: Optional[List[int]] = None  # the prompt in progress: [slot, request index, columns done]
    left = budget  # prompt columns this poll may still prefill

    def advance() -> None:  # the prompt in progress by one chunk of the budget left
        nonlocal prog, left
        s, i, c0 = prog
        T = int(requests[i].emb.shape[0])
        n = min(T - c0, left // PREFILL_CHUNK_ALIGN * PREFILL_CHUNK_ALIGN)
        if n <= 0 or (pool is not None and not reserve([s], [limit(i, c0 + n)])):
            return
        dev.prefill_chunk(s, i, c0, n)
        stats.chunks += 1
        left -= max(MIN_PROMPT_COLS, n) if c0 == 0 and n == T else n  # a whole prompt is padded as an admission
        if c0 + n == T:
            prog = None
            stats.admitted += 1
            if requests[i].prompt_key is not None:
                holders[s] = (requests[i].prompt_key, i)
            if pool is not None:
                note_admitted(i)
        else:
            prog[2] = c0 + n

    waiting = deque(range(len(requests)))
    owner: List[Optional[int]] = [None] * dev.slots
    live: Dict[object, Set[int]] = {}  # open source: submission key -> indices of its live stages
    root: Dict[int, object] = {}  # and back

    def retire(i: int) -> Set[int]:  # stage i is no longer live: the submission's remaining live stages
        key = root.pop(i)
        stages = live[key]
        stages.discard(i)
        if not stages:
            del live[key]
        return stages

    doomed: Set[int] = set()  # running requests to stop after the next status read
    while True:
        taken: list = []
        if source is not None:
            idle = not waiting and not suspended and all(o is None for o in owner)
            new, cancels, closed = source.take(block=idle)
            for key, r in new:
                stages = live.setdefault(key, set())
                for x in (r if isinstance(r, (list, tuple)) else [r]):
                    requests.append(x)
                    i = len(requests) - 1
                    stages.add(i)
                    root[i], stats.keys[i] = key, key
                    waiting.append(i)
            for key in cancels:
                for i in sorted(live.get(key, ())):  # nothing left when it ended already
                    if i in waiting:
                        waiting.remove(i)
                        retire(i)
                        stats.cancelled.add(i)
                        taken.append((i, None, 0, False))
                    elif prog is not None and prog[1] == i:  # mid-prefill: no final chunk, the slot is free again
                        dev.cancel([prog[0]])
                        if pool is not None:
                            dev.release([prog[0]])
                            mapped.pop(prog[0], None)
                        owner[prog[0]] = None
                        prog = None
                        retire(i)
                        stats.cancelled.add(i)
                        taken.append((i, None, 0, False))
                    elif any(e[0] == i for e in suspended):  # its image ends it with the tokens it had
                        e = next(e for e in suspended if e[0] == i)
                        suspended.remove(e)
                        retire(i)
                        stats.cancelled.add(i)
                        stats.tokens += e[2]
                        taken.append((i, e[1], e[2], False))
                    else:
                        doomed.add(i)
            if idle and closed and not new and not taken:
                return
        free = [s for s in range(dev.slots) if owner[s] is None]
        # a suspended request resumes only if the running slots' pages for their next chunk fit beside it, so the
        # decode that follows does not suspend it again before it has moved
        ahead = [s for s in range(dev.slots) if owner[s] is not None and (prog is None or s != prog[0])]
        while suspended and free and reserve([free[0]] + ahead, [limit(suspended[0][0], held(*suspended[0][::2]))] +
                                             [limit(owner[s], mapped.get(s, 0)) for s in ahead]):
            i, image, _ = suspended.pop(0)
            s = free.pop(0)
            dev.resume(s, image)
            owner[s] = i
            ahead.append(s)
            stats.resumes += 1
        batch = []
        shares = []  # (slot, request index, source slot, c0): after the admission of `batch`
        share_cols = share_pages = 0  # the shares' final chunks' columns, and the pages they will map
        created = False
        if prog is not None:
            advance()
        # the requests behind a prompt in progress, or behind a suspended request, wait for it
        while free and waiting and prog is None and not suspended:
            s, i = free.pop(0), waiting.popleft()
            r = requests[i]
            T = int(r.emb.shape[0])
            if r.prompt_key is not None and shared_prompt_cols(T) > 0:
                src = holder(r.prompt_key)
                if src is None:  # a member admitted at this poll
                    src = next((t for t, j in batch if requests[j].prompt_key == r.prompt_key), None)
                if src is not None:
                    c0 = shared_prompt_cols(T)
                    need = -(-limit(i, T) // _lib.PAGE_TOKENS) - c0 // _lib.PAGE_TOKENS
                    if ((budget is not None
                         and admission_cols(batch, requests, dev.max_context) + share_cols + T - c0 > left)
                            or (pool is not None and dev.pages_in_use + share_pages + need > pool - 1)):
                        waiting.appendleft(i)  # the budget or the pool is short: it waits at the head of the queue
                        break
                    owner[s] = i
                    shares.append((s, i, src, c0))
                    share_cols += T - c0
                    share_pages += need
                    continue
            # no budget, no bound: admission_cols (quadratic in the admission's size) is not evaluated
            if budget is not None and admission_cols(batch + [(s, i)], requests, dev.max_context) + share_cols > left:
                owner[s] = i
                prog, created = [s, i, 0], True  # the first request that does not fit
                break
            if pool is not None and share_pages and (
                    dev.pages_in_use + share_pages + -(-limit(i, T) // _lib.PAGE_TOKENS) > pool - 1):
                waiting.appendleft(i)  # the pages the shares ahead of it need come first
                break
            if pool is not None and not reserve([s], [limit(i, T)]):
                waiting.appendleft(i)  # the pool is short: it waits for pages at the head of the queue
                break
            owner[s] = i
            batch.append((s, i))
        if budget is not None:
            left -= admission_cols(batch, requests, dev.max_context) + share_cols
        if batch:
            dev.admit(batch)
            stats.admissions += 1
            stats.admitted += len(batch)
            for s, i in batch:
                if pool is not None:
                    note_admitted(i)
                if requests[i].prompt_key is not None:
                    holders[s] = (requests[i].prompt_key, i)
        for s, i, src, c0 in shares:
            T = int(requests[i].emb.shape[0])
            if not dev.share(src, s, i, c0) or (pool is not None and not reserve([s], [limit(i, T)])):
                raise RuntimeError("a shared prompt's pages were counted and did not fit")  # share_pages covers them
            if pool is not None:
                note_admitted(i)
            dev.prefill_chunk(s, i, c0, T - c0)
            holders[s] = (requests[i].prompt_key, i)
            stats.shares += 1
            stats.shared_cols += c0
            stats.admitted += 1
        if created:  # its first chunk, from the budget left over
            advance()
        st = dev.status()
        stats.decode_steps = st.steps_done
        polled = list(owner)
        if prog is not None:  # reserved: the slot's status is not its request's yet
            polled[prog[0]] = None
        ended = taken
        follow: List[int] = []
        done = []  # (index, slot, n_tokens, cancelled at this read) of the requests that may have a follow-up
        freed = False
        released: List[int] = []
        stop = [s for s in range(dev.slots) if owner[s] in doomed and st.state[s] != _lib.SLOT_FINISHED]
        if stop:
            dev.cancel(stop)
        for s in range(dev.slots):
            i = polled[s]
            if i is None or (st.state[s] != _lib.SLOT_FINISHED and s not in stop):
                continue
            owner[s] = None
            freed = True
            released.append(s)
            admitted_at.pop(i, None)
            was_doomed = i in doomed
            doomed.discard(i)
            if s in stop:  # no follow-up after a cancel
                retire(i)
                stats.cancelled.add(i)
                stats.tokens += st.end_idx[s]
                ended.append((i, s, st.end_idx[s], False))
                continue
            if st.end_idx[s] == 0 and st.finish[s]:
                r = requests[i]
                if r.manual_seed is None and r.ensure_non_empty:
                    waiting.appendleft(i)  # regenerate (gpt.py:527-570); a fresh Philox seed is drawn at admission
                    stats.requeued += 1
                    continue
                ended.append((i, None, 0, True))
                done.append((i, None, 0, was_doomed))
            else:
                stats.tokens += st.end_idx[s]
                ended.append((i, s, st.end_idx[s], bool(st.finish[s])))
                done.append((i, s, st.end_idx[s], was_doomed))
        if pool is not None and released:
            dev.release(released)
            for s in released:
                mapped.pop(s, None)
        _prepare(requests, done, dev, stats, source)
        for i, s, n, was_doomed in done:
            kids = _follow_up(requests, i, s, n, dev, check, stats, source)
            if i in root:  # the submitted request's live stage moves on to its follow-ups, or it is done
                key = root[i]
                retire(i)
                if kids and was_doomed:  # finished at the read that applies its cancel: the follow-ups are cancelled
                    for k in kids:
                        stats.cancelled.add(k)
                        ended.append((k, None, 0, False))
                    kids = []
                for k in kids:
                    live.setdefault(key, set()).add(k)
                    root[k] = key
            follow += kids
        waiting.extendleft(reversed(follow))  # ahead of the waiting requests, in slot order
        if freed and waiting:
            yield st, polled, ended
            continue  # refill the freed slots before the next chunk
        running = [s for s in range(dev.slots) if owner[s] is not None and (prog is None or s != prog[0])]
        interrupted = (bool(running) or prog is not None or bool(suspended)) and context is not None and context.get()
        if interrupted:
            stats.interrupted = True
            for s in running:
                stats.tokens += st.end_idx[s]
                ended.append((owner[s], s, st.end_idx[s], False))
            for i, image, n in suspended:
                stats.tokens += n
                ended.append((i, image, n, False))
        yield st, polled, ended
        if budget is not None:  # the poll ends here: the next one has the whole budget
            stats.prefill_cols.append(budget - left)
            left = budget
        if interrupted or (not running and source is None and prog is None and not suspended):
            return
        while pool is not None and running:  # map every running slot for the chunk, suspending the last admitted
            if reserve(running, [limit(owner[s], held(owner[s], st.end_idx[s])) for s in running]):
                break
            s = max(running, key=lambda s: admitted_at[owner[s]])
            i = owner[s]
            suspended.append([i, dev.suspend(s), st.end_idx[s]])
            mapped.pop(s, None)
            holders.pop(s, None)
            suspended.sort(key=lambda e: admitted_at[e[0]])
            owner[s] = None
            running.remove(s)
            stats.suspensions += 1
        if pool is not None:
            stats.pages.append(dev.pages_in_use)
            stats.peak_pages = max(stats.peak_pages, dev.pages_in_use)
            stats.host_bytes.append(dev.host_bytes)
            stats.peak_shared_pages = max(stats.peak_shared_pages, getattr(dev, "shared_pages", 0))
        if running:
            dev.decode(chunk)


def schedule(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
             check: Optional[Callable[[Request], None]] = None, prefill_budget: Optional[int] = None
             ) -> Iterator[Tuple[int, Optional[int], int]]:
    """Drive ``dev`` (``slots``, ``admit([(slot, request_index)])``, ``decode(n)``, ``status() -> SlotStatus``) until
    every request has finished; yields ``(request_index, slot, n_tokens)`` as each one completes - the caller harvests
    the slot's first ``n_tokens`` outputs before resuming the generator - or ``(request_index, None, 0)`` for a seeded
    request whose first token is EOS (it ends empty, gpt.py:527).  An unseeded one with ``ensure_non_empty`` is queued
    again instead.

    Waiting requests enter free slots in order, lowest slot first, at every poll (every ``chunk`` decode steps).  On a
    ``context`` interrupt the running requests are yielded with what they have so far and the waiting ones are dropped.
    Follow-ups (``Request.then``) need ``dev.harvest(slot, n)`` and ``dev.empty(request_index)``; see ``_poll_cycles``,
    which also describes the policy of a ``prefill_budget`` (``dev.prefill_chunk``, ``dev.max_context``).
    """
    for _, _, ended in _poll_cycles(requests, dev, chunk, context, stats, check, None, prefill_budget):
        for i, s, n, _ in ended:
            yield i, s, n


def stream_schedule(requests: List[Request], dev, chunk: int, context=None, stats: Optional[ScheduleStats] = None,
                    check: Optional[Callable[[Request], None]] = None, source: Optional[Arrivals] = None,
                    prefill_budget: Optional[int] = None) -> Iterator[List[Tuple[int, Optional[int], int, bool]]]:
    """``schedule``'s policy, yielding once per poll the list of ``(request_index, slot, n_tokens, last)``: for each
    request, the yields ``GPT.generate(stream=True, stream_batch=r.stream_batch)`` makes for it alone, in its order,
    as cumulative token counts (the slot's first ``n_tokens`` outputs; slot None: a seeded request that ended empty).

    The static loop (gpt.py here, generate) yields at every multiple of ``stream_batch`` (from step 2 on) that the row
    reaches unfinished, yields a boundary a second time when EOS follows it on the very next step, and ends with the
    final yield; a row that stops at ``max_new_token`` is not finished there, so it gets no second yield.  Tokens only
    ever append to a slot, so each poll rebuilds every boundary a slot crossed since the last one from its token count:
    the yields do not depend on ``chunk``.  The slots' outputs stay in place until the generator is resumed.

    With an open ``source`` (see ``_poll_cycles``) a cancelled request gets a final yield of what it has, and
    ``stats.cancelled`` tells it apart.  A request yields nothing before its first token, so a ``prefill_budget``
    leaves every request's yields as they are."""
    sent: Dict[int, int] = {}  # last boundary yielded per request
    for st, owner, ended in _poll_cycles(requests, dev, chunk, context, stats, check, source, prefill_budget):
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
            sent.pop(i, None)
        if out:
            yield out


class SlotImage:
    """A suspended request (``EngineDevice.suspend``): its slot's image in pinned host memory (ctb_slot_image), until
    ``EngineDevice.resume`` restores it into a slot.  ``row(hidden)`` and ``outputs(n)`` read its first tokens' ids and
    hidden states, as the slot held them, once the copies that filled it are complete (``ready``).  ``logprobs``: the
    slot's log-probabilities [n_gen, num_vq] in pinned host memory (an engine with logprobs; they are not part of the
    device image), else None.  ``top``: likewise its top log-probabilities, (ids, lp) [n_gen, num_vq, N] (an engine
    with top_logprobs), else None."""

    top: Optional[Tuple[torch.Tensor, torch.Tensor]] = None

    def __init__(self, buf: torch.Tensor, text: bool, device, num_vq: int, hidden_size: int, stream,
                 logprobs: Optional[torch.Tensor] = None, top: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        self.buf, self.text, self.device, self.num_vq, self.hidden_size = buf, text, device, num_vq, hidden_size
        self.logprobs, self.top = logprobs, top
        self.ready = torch.cuda.Event()
        self.ready.record(stream)  # after the copies that fill the image
        self.header = _lib.SlotImage.from_address(buf.data_ptr())

    @property
    def nbytes(self) -> int:
        return int(self.buf.numel())

    def row(self, hidden: bool) -> torch.Tensor:
        """The slot's hidden states [n_gen, d] (fp32) or ids [n_gen, num_vq] (int32), on the device."""
        self.ready.synchronize()
        h = self.header
        if hidden:
            off, n = h.off_hiddens, h.n_gen * self.hidden_size
            return self.buf[off: off + 4 * n].view(torch.float32).view(h.n_gen, self.hidden_size).to(self.device)
        off, n = h.off_ids, h.n_gen * self.num_vq
        return self.buf[off: off + 4 * n].view(torch.int32).view(h.n_gen, self.num_vq).to(self.device)

    def outputs(self, n: int, return_hidden: bool):
        """GenerationOutputs of the first ``n`` tokens, as ``EngineDevice.harvest`` gives them for a slot."""
        from .gpt import GPT

        ids = self.row(False)[:n].to(torch.int64)
        lp = [] if self.logprobs is None else [self.logprobs[:n, 0] if self.text else self.logprobs[:n]]
        lp = [t.to(self.device) for t in lp]
        top = []
        if self.top is not None:
            i, v = (t[:n, 0] if self.text else t[:n] for t in self.top)
            top = [(i.to(self.device, torch.int64), v.to(self.device))]
        if self.text:
            return GPT.GenerationOutputs(ids=[ids[:, 0].contiguous()], attentions=[], hiddens=[], logprobs=lp,
                                         top_logprobs=top)
        hid = [self.row(True)[:n]] if return_hidden else []
        return GPT.GenerationOutputs(ids=[ids], attentions=[], hiddens=hid, logprobs=lp, top_logprobs=top)


class EngineDevice:
    """The device layer of ``schedule`` on a GPT handle (ctb_gpt_engine_begin / _admit / _status, ctb_gpt_decode).
    ``kv_pool_pages`` (``kv_pool_pages()``) makes a paged engine (ctb_gpt_engine_begin_paged) with the pool interface
    ``_poll_cycles`` describes; None keeps every slot's fixed pages.  ``logprobs`` attaches a buffer of token
    log-probabilities (ctb_gpt_engine_logprobs) beside ``ids_out``: outputs then carry them (``GenerationOutputs
    .logprobs``), and suspended requests take theirs along in their ``SlotImage``.  ``top_logprobs`` (N > 0) attaches
    the two buffers of ctb_gpt_engine_top_logprobs, the N most likely ids of every sampled row and their
    log-probabilities, which outputs (``GenerationOutputs.top_logprobs``) and suspended requests carry in the same way."""

    top_ids_out: Optional[torch.Tensor] = None  # [S, max_new_cap, num_vq, N] int32 with top_logprobs
    top_lp_out: Optional[torch.Tensor] = None   # [S, max_new_cap, num_vq, N] fp32

    def __init__(self, gpt, requests: Sequence[Request], slots: int, max_new_cap: int, return_hidden: bool = True,
                 flags: int = 0, kv_pool_pages: Optional[int] = None, logprobs: bool = False, top_logprobs: int = 0):
        self.gpt, self.requests, self.slots = gpt, requests, slots
        self.max_context = gpt.max_context
        self.lib = _lib.load()
        dev = gpt.device_gpt
        self.dev = dev
        self._torch_stream = torch.cuda.current_stream(dev)  # every device call of this engine is enqueued on it
        self.stream = C.c_void_p(self._torch_stream.cuda_stream)
        self.ids_out = torch.zeros(slots, max_new_cap, gpt.num_vq, dtype=torch.int32, device=dev)
        self.hid_out = (torch.zeros(slots, max_new_cap, gpt.config.hidden_size, dtype=torch.float32, device=dev)
                        if return_hidden else None)
        self.lp_out = (torch.zeros(slots, max_new_cap, gpt.num_vq, dtype=torch.float32, device=dev) if logprobs
                       else None)
        top_n = check_top_logprobs(top_logprobs)
        shape = (slots, max_new_cap, gpt.num_vq, top_n)
        self.top_ids_out = torch.zeros(shape, dtype=torch.int32, device=dev) if top_n else None
        self.top_lp_out = torch.zeros(shape, dtype=torch.float32, device=dev) if top_n else None
        hid = C.c_void_p(self.hid_out.data_ptr()) if self.hid_out is not None else None
        self.pool_pages = kv_pool_pages
        if kv_pool_pages is None:
            _lib.check(self.lib.ctb_gpt_engine_begin_ex(
                gpt._handle, slots, max_new_cap, flags, C.c_void_p(self.ids_out.data_ptr()), hid, self.stream))
        else:
            _lib.check(self.lib.ctb_gpt_engine_begin_paged(
                gpt._handle, slots, max_new_cap, flags, kv_pool_pages, C.c_void_p(self.ids_out.data_ptr()), hid,
                self.stream))
        if self.lp_out is not None:
            _lib.check(self.lib.ctb_gpt_engine_logprobs(gpt._handle, C.c_void_p(self.lp_out.data_ptr()), self.stream))
        if top_n:
            _lib.check(self.lib.ctb_gpt_engine_top_logprobs(gpt._handle, top_n, C.c_void_p(self.top_ids_out.data_ptr()),
                                                            C.c_void_p(self.top_lp_out.data_ptr()), self.stream))
        # the images of suspended requests, by id, while anything holds them (a cancelled one's ends with its outputs)
        self._images: "weakref.WeakValueDictionary[int, SlotImage]" = weakref.WeakValueDictionary()
        self._resumed: List[SlotImage] = []  # read by the device until the next status read
        self._state = (C.c_int32 * slots)()
        self._end = torch.zeros(slots, dtype=torch.int32)
        self._fin = torch.zeros(slots, dtype=torch.uint8)
        self._text = [False] * slots  # mode of the request each slot was last given

    def admit(self, batch: List[Tuple[int, int]]) -> None:
        noise: Dict[tuple, torch.Tensor] = {}  # one static batch's noise per (B, rows, cols, seed) in this admission
        for chunk, _, seeded, text in admission_prefills(batch, self.requests, self.gpt.max_context):
            self._admit(chunk, seeded, text, noise)

    def prefill_chunk(self, slot: int, index: int, c0: int, n: int) -> None:
        """Prompt columns ``[c0, c0 + n)`` of request ``index`` into ``slot`` (ctb_gpt_engine_prefill_chunk); the
        final chunk admits the request.  A whole prompt (``c0 == 0``, ``n`` its length) is one ordinary admission."""
        r = self.requests[index]
        T, seeded, text = int(r.emb.shape[0]), r.manual_seed is not None, bool(r.infer_text)
        if c0 == 0 and n == T:
            self._admit([(slot, index)], seeded, text, {})
            return
        emb = r.emb[c0: c0 + n].to(self.dev, torch.float32).contiguous()
        cfg, noise = None, None
        if c0 + n == T:
            cfgs, noise = self._sampling([r], seeded, text, {})
            cfg = C.byref(cfgs[0])
            self._text[slot] = text
        _lib.check(self.lib.ctb_gpt_engine_prefill_chunk(
            self.gpt._handle, slot, T, c0, n, C.c_void_p(emb.data_ptr()), int(text), cfg,
            C.c_void_p(noise.data_ptr()) if noise is not None else None, r.max_new_token, self.stream))

    def _sampling(self, reqs: List[Request], seeded: bool, text: bool, cache: Dict[tuple, torch.Tensor]):
        """The sampler configs (host array) and seeded Exp(1) rows (device, or None) of an admission of ``reqs``."""
        gpt, n = self.gpt, len(reqs)
        cfgs = (_lib.SamplerConfig * n)()
        for k, r in enumerate(reqs):
            temps = [float(t) for t in torch.as_tensor(r.temperature).flatten().tolist()]
            philox = 0 if seeded else int(torch.randint(0, 2 ** 62, (1,)).item())
            cfgs[k] = build_sampler_config(r.logits_processors, temps, int(r.eos_token), r.min_new_token, philox)
        noise = None
        if seeded:  # the rows GPT.generate draws for this request's row of its batch (noise_batch) with this seed
            rows, cols = (1, gpt.num_text_tokens) if text else (gpt.num_vq, gpt.num_audio_tokens)
            noise = noise_rows(reqs, rows, cols, cache).to(self.dev)
        return cfgs, noise

    def _admit(self, group, seeded: bool, text: bool, cache: Dict[tuple, torch.Tensor]) -> None:
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
        cfgs, noise = self._sampling(reqs, seeded, text, cache)
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

    # ---------------------------------------------------------------- KV pool (paged engines)
    def _page_counts(self) -> Tuple[int, int]:
        used, shared = C.c_int32(), C.c_int32()
        _lib.check(self.lib.ctb_gpt_engine_pages(self.gpt._handle, C.byref(used), C.byref(shared)))
        return used.value, shared.value

    @property
    def pages_in_use(self) -> int:
        """Pages mapped, each counted once however many slots share it (ctb_gpt_engine_pages)."""
        return self._page_counts()[0]

    @property
    def shared_pages(self) -> int:
        """Pages more than one slot maps (shared prompts)."""
        return self._page_counts()[1]

    @property
    def host_bytes(self) -> int:
        """Bytes of the images of suspended requests.  They live in pinned blocks of torch's caching host allocator,
        which rounds each block up to a power of two and keeps freed blocks for reuse: the process can hold up to about
        twice the peak of this figure pinned until it exits."""
        return sum(im.nbytes for im in self._images.values())

    def reserve(self, slots: List[int], tokens: List[int]) -> bool:
        """Map pages so that each slot holds positions [0, tokens[i]) (ctb_gpt_engine_reserve); False, with nothing
        mapped, when the pool cannot cover them all."""
        n = len(slots)
        rc = self.lib.ctb_gpt_engine_reserve(self.gpt._handle, n, (C.c_int32 * n)(*slots), (C.c_int32 * n)(*tokens),
                                             self.stream)
        if rc == _lib.ERR_POOL:
            return False
        _lib.check(rc)
        return True

    def release(self, slots: List[int]) -> None:
        """Return the pages of idle or finished slots to the pool (ctb_gpt_engine_release)."""
        _lib.check(self.lib.ctb_gpt_engine_release(self.gpt._handle, len(slots), (C.c_int32 * len(slots))(*slots),
                                                   self.stream))

    def suspend(self, slot: int) -> SlotImage:
        """Move the running request in ``slot`` to a pinned host image (ctb_gpt_engine_suspend); the slot and its pages
        are free afterwards."""
        nbytes = C.c_uint64()
        _lib.check(self.lib.ctb_gpt_engine_suspend_bytes(self.gpt._handle, slot, C.byref(nbytes), self.stream))
        buf = torch.empty(nbytes.value, dtype=torch.uint8, pin_memory=True)
        _lib.check(self.lib.ctb_gpt_engine_suspend(self.gpt._handle, slot, C.c_void_p(buf.data_ptr()), nbytes.value,
                                                   self.stream))
        lp = top = None
        n = _lib.SlotImage.from_address(buf.data_ptr()).n_gen  # the header is written: n_gen is known on the host
        if self.lp_out is not None:
            lp = torch.empty(n, self.gpt.num_vq, dtype=torch.float32, pin_memory=True)
            with torch.cuda.stream(self._torch_stream):
                lp.copy_(self.lp_out[slot, :n], non_blocking=True)
        if self.top_ids_out is not None:
            top = tuple(torch.empty(t[slot, :n].shape, dtype=t.dtype, pin_memory=True)
                        for t in (self.top_ids_out, self.top_lp_out))
            with torch.cuda.stream(self._torch_stream):
                for h, t in zip(top, (self.top_ids_out, self.top_lp_out)):
                    h.copy_(t[slot, :n], non_blocking=True)
        image = SlotImage(buf, self._text[slot], self.dev, self.gpt.num_vq, self.gpt.config.hidden_size,
                          self._torch_stream, lp, top)
        self._images[id(image)] = image
        return image

    def resume(self, slot: int, image: SlotImage) -> None:
        """Restore a suspended request into ``slot``, whose pages already cover it (ctb_gpt_engine_resume)."""
        _lib.check(self.lib.ctb_gpt_engine_resume(self.gpt._handle, slot, C.c_void_p(image.buf.data_ptr()),
                                                  image.nbytes, self.stream))
        if self.lp_out is not None:
            with torch.cuda.stream(self._torch_stream):
                self.lp_out[slot, :image.logprobs.shape[0]].copy_(image.logprobs, non_blocking=True)
        if self.top_ids_out is not None:
            with torch.cuda.stream(self._torch_stream):
                for t, h in zip((self.top_ids_out, self.top_lp_out), image.top):
                    t[slot, :h.shape[0]].copy_(h, non_blocking=True)
        self._text[slot] = image.text
        self._images.pop(id(image), None)
        self._resumed.append(image)  # the copies read it until the stream passes them

    def share(self, src: int, dst: int, index: int, c0: int) -> bool:
        """Set up ``dst`` for request ``index`` with prompt columns ``[0, c0)`` taken from the prompt of the request in
        ``src`` (ctb_gpt_engine_share_prompt); ``prefill_chunk(dst, index, c0, T - c0)`` then admits it.  A paged
        engine maps ``src``'s pages for them, and pages of ``dst``'s own up to the prompt's end: False, with nothing
        changed, when the pool cannot cover those."""
        T = int(self.requests[index].emb.shape[0])
        rc = self.lib.ctb_gpt_engine_share_prompt(self.gpt._handle, src, dst, T, c0, self.stream)
        if rc == _lib.ERR_POOL:
            return False
        _lib.check(rc)
        return True

    def cancel(self, slots: List[int]) -> None:
        """Stop the requests in ``slots`` (ctb_gpt_engine_cancel): each keeps the tokens it has."""
        _lib.check(self.lib.ctb_gpt_engine_cancel(self.gpt._handle, len(slots), (C.c_int32 * len(slots))(*slots),
                                                  self.stream))

    def status(self) -> SlotStatus:
        st = _lib.GptStatus()
        _lib.check(self.lib.ctb_gpt_engine_status(self.gpt._handle, C.byref(st), self._state,
                                                  C.c_void_p(self._end.data_ptr()), C.c_void_p(self._fin.data_ptr()),
                                                  self.stream))
        self._resumed.clear()  # the status read synchronised the stream
        return SlotStatus(list(self._state), self._end.tolist(), self._fin.tolist(), int(st.steps_done))

    def harvest(self, slot: int, n: int, copy: bool = True):
        """GenerationOutputs of the request in ``slot``: its first ``n`` ids (int64 copies) and hidden states (copies,
        or with ``copy=False`` views into the engine buffer, valid until the engine decodes or admits again).  A text
        request's ids are 1-D and it has no hidden states, as ``GPT.generate(infer_text=True)`` returns them."""
        from .gpt import GPT

        if isinstance(slot, SlotImage):  # a suspended request that was cancelled or interrupted
            self._images.pop(id(slot), None)
            return slot.outputs(n, self.hid_out is not None)
        text = self._text[slot]
        lp = [] if self.lp_out is None else [(self.lp_out[slot, :n, 0] if text else self.lp_out[slot, :n]).clone()]
        top = []
        if self.top_ids_out is not None:
            i, v = (t[slot, :n, 0] if text else t[slot, :n] for t in (self.top_ids_out, self.top_lp_out))
            top = [(i.to(torch.int64), v.clone())]
        if text:
            return GPT.GenerationOutputs(ids=[self.ids_out[slot, :n, 0].to(torch.int64)], attentions=[], hiddens=[],
                                         logprobs=lp, top_logprobs=top)
        ids = self.ids_out[slot, :n].to(torch.int64)
        hid = ([self.hid_out[slot, :n].clone() if copy else self.hid_out[slot, :n]] if self.hid_out is not None
               else [])
        return GPT.GenerationOutputs(ids=[ids], attentions=[], hiddens=hid, logprobs=lp, top_logprobs=top)

    def empty(self, index: Optional[int] = None):
        """The outputs of request ``index`` (default: a code request) when it ended empty (a seeded request whose
        first token was EOS)."""
        from .gpt import GPT

        text = index is not None and self.requests[index].infer_text
        lp = ([] if self.lp_out is None else
              [torch.zeros((0,) if text else (0, self.gpt.num_vq), dtype=torch.float32, device=self.dev)])
        top = []
        if self.top_ids_out is not None:
            shape = (0, self.top_ids_out.shape[3]) if text else (0, self.gpt.num_vq, self.top_ids_out.shape[3])
            top = [(torch.zeros(shape, dtype=torch.int64, device=self.dev),
                    torch.zeros(shape, dtype=torch.float32, device=self.dev))]
        if text:
            return GPT.GenerationOutputs(ids=[torch.zeros(0, dtype=torch.int64, device=self.dev)], attentions=[],
                                         hiddens=[], logprobs=lp, top_logprobs=top)
        ids = torch.zeros(0, self.gpt.num_vq, dtype=torch.int64, device=self.dev)
        hid = ([torch.zeros(0, self.gpt.config.hidden_size, dtype=torch.float32, device=self.dev)]
               if self.hid_out is not None else [])
        return GPT.GenerationOutputs(ids=[ids], attentions=[], hiddens=hid, logprobs=lp, top_logprobs=top)


_END = object()  # closes a streaming job's iterator
_log = logging.getLogger(__name__)


class _RequestTable:
    """An open engine's requests by index (the ``requests`` of ``_poll_cycles``): indices are never reused, and an entry
    is dropped once its request has been served, so a long-lived engine holds only the requests still in it."""

    def __init__(self):
        self._items: Dict[int, Request] = {}
        self._next = 0

    def append(self, r: Request) -> None:
        self._items[self._next] = r
        self._next += 1

    def __len__(self) -> int:  # the next index
        return self._next

    def __getitem__(self, i: int) -> Request:
        return self._items[i]

    def __delitem__(self, i: int) -> None:
        del self._items[i]

    def held(self) -> int:
        return len(self._items)


class Job:
    """A request submitted to an open engine (``GPT.open_engine``, ``Chat.open_engine``).

    ``result(timeout)`` waits for it to end; ``cancel()`` stops it at the engine's next poll; a streaming job
    (``submit(..., stream=True)``) is also an iterator of its yields, which simply ends when the job is cancelled.
    Results and yields are handed over on the caller's current CUDA stream: whatever the engine copied for them is
    complete before the caller's later work on that stream reads it."""

    def __init__(self, engine: "OpenEngine", stream: bool):
        self._engine, self.stream = engine, stream
        self._future: Future = Future()
        self._items: Optional[queue.Queue] = queue.Queue() if stream else None
        self._cancelled = False
        self.state = None
        self.spk_smp: Optional[str] = None  # Chat.open_engine paragraphs: the speaker sampled from sentence 0
        self.refined: Optional[List[Optional[str]]] = None  # refined paragraphs: each sentence's text once refined
        self.logprobs = None  # Chat.open_engine(logprobs=True): the speech tokens' log-probabilities once it has ended
        self.top_logprobs = None  # Chat.open_engine(top_logprobs=N): their N most likely ids and log p, likewise

    def cancel(self) -> None:
        self._engine._source.cancel(self)

    def result(self, timeout: Optional[float] = None):
        return self._engine._receive(*self._future.result(timeout))

    def done(self) -> bool:
        return self._future.done()

    def cancelled(self) -> bool:
        return self._cancelled or self._future.cancelled()

    def __iter__(self):
        if self._items is None:
            raise TypeError("only a job submitted with stream=True is iterable")
        while True:
            item = self._items.get()
            if item is _END:
                return
            if isinstance(item, BaseException):
                raise item
            yield self._engine._receive(*item)

    # worker side
    def _put(self, value, event=None) -> None:
        self._items.put((value, event))

    def _finish(self, value, event=None) -> None:
        if self._items is not None:
            self._items.put(_END)
        self._future.set_result((value, event))

    def _stop(self) -> None:
        """Cancelled: a streaming job's iterator ends and ``result()`` raises ``CancelledError``."""
        self._cancelled = True
        if self._items is not None:
            self._items.put(_END)
        self._future.cancel()

    def _fail(self, e: BaseException) -> None:
        if self._items is not None:
            self._items.put(e)
        if not self._future.done():
            self._future.set_exception(e)


class OpenEngine:
    """A slot engine that takes requests while it decodes (``schedule``'s policy with an ``Arrivals`` source).

    One worker thread owns the device: it makes the device layer with ``make_device(requests)`` and issues every
    admission, decode, status read, cancellation and harvest copy on the engine's CUDA stream.  ``submit`` and
    ``Job.cancel`` only queue under a lock, from any thread.  ``check`` validates a request in the caller's thread at
    ``submit`` (and each follow-up in the worker, where a failure fails that job only).  An error in the worker fails
    every pending job with it, stops the engine and is raised again by ``close``.  With a ``context`` (``GPT.Context``)
    an interrupt is ``schedule``'s: at the first poll that sees it the running requests end with what they have, the
    engine stops, and every job that has not ended by then is cancelled.  Subclasses turn each poll's yields into job
    results (``_serve``).  ``prefill_budget``: ``_poll_cycles``' bound on each poll's prompt columns (None: none).
    ``slots``: the device's slot count, when known."""

    def __init__(self, make_device: Callable[[List[Request]], object], chunk: int,
                 check: Optional[Callable[[Request], None]] = None, device=None,
                 on_close: Optional[Callable[[], None]] = None, max_new_cap: Optional[int] = None, context=None,
                 prefill_budget: Optional[int] = None, slots: Optional[int] = None):
        self._make_device, self.chunk, self._check, self._on_close = make_device, int(chunk), check, on_close
        self.slots = slots
        self.prefill_budget = check_prefill_budget(prefill_budget)
        self.device, self.max_new_cap, self._context = device, max_new_cap, context
        cuda = device is not None and torch.device(device).type == "cuda"
        self._stream = torch.cuda.Stream(device) if cuda else None
        self._source = Arrivals()
        self._lock = threading.Lock()
        self._pending: Set[Job] = set()  # submitted jobs, until each one ends
        self._job_at: Dict[int, Job] = {}  # request index (a stage) -> its job, while the stage is live
        self._error: Optional[BaseException] = None
        self._stopped = False
        self.stats = ScheduleStats()
        self._requests = _RequestTable()
        self._thread = threading.Thread(target=self._run, name="ctb-open-engine", daemon=True)
        self._thread.start()

    # ---------------------------------------------------------------- callers
    def submit(self, request, stream: bool = False, state=None) -> Job:
        """Queue ``request`` (or a non-empty list of requests, stages of one job from the start); ``state`` is kept on
        the job for ``_serve`` (``Job.state``)."""
        job = self._new_job(request, stream, state)
        self._enqueue([(job, request)])
        return job

    def _new_job(self, request, stream: bool, state) -> Job:
        """The job of ``submit(request, stream, state)``, its requests checked, not queued yet."""
        reqs = list(request) if isinstance(request, (list, tuple)) else [request]
        if not reqs or not all(isinstance(r, Request) for r in reqs):
            raise TypeError("requests must be chattts_b200.engine.Request objects")
        if self._check is not None:
            for r in reqs:
                self._check(r)
        job = Job(self, stream)
        job.state = state
        return job

    def _enqueue(self, subs: List[Tuple[Job, object]]) -> None:
        """Queue ``[(job, request or list of requests)]`` in one step: the worker takes all of them at the same poll."""
        with self._lock:
            if self._stopped:
                raise RuntimeError("the engine is closed") from self._error
            if self._stream is not None:  # the prompts were made on the caller's stream
                self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._pending.update(job for job, _ in subs)
            self._source.submit_all(subs)

    def close(self, cancel: bool = False) -> None:
        """Wait for every submitted job (``cancel=True``: cancel them all first), then join the worker.  Raises the
        worker's error, if it had one."""
        if cancel:
            with self._lock:
                for job in list(self._pending):
                    self._source.cancel(job)
        self._source.close()
        self._thread.join()
        if self._on_close is not None:
            self._on_close()
            self._on_close = None
        if self._error is not None:
            raise self._error

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.close()
            return
        try:  # the block's own exception is the one to propagate; a worker error is only logged beside it
            self.close(cancel=True)
        except Exception:
            _log.exception("the open engine had failed as well")

    def _receive(self, value, event):
        """A job's result or yield in the caller's thread (``event``: recorded by ``_serve`` after its copies)."""
        return value

    # ---------------------------------------------------------------- worker
    def _run(self) -> None:
        requests = self._requests
        try:
            if self._stream is not None:
                with torch.cuda.device(self.device), torch.cuda.stream(self._stream), torch.no_grad():
                    self._loop(requests)
            else:
                self._loop(requests)
        except BaseException as e:
            self._error = e
        finally:
            with self._lock:
                self._stopped = True
                self._source.close()
                jobs = list(self._pending)
                self._pending.clear()
            for job in jobs:  # without an error the loop ended early only on an interrupt
                if job.done():
                    continue
                if self._error is not None:
                    job._fail(self._error)
                else:
                    job._stop()

    def _loop(self, requests: _RequestTable) -> None:
        dev = self._make_device(requests)
        for batch in stream_schedule(requests, dev, self.chunk, self._context, self.stats, self._check, self._source,
                                     self.prefill_budget):
            jobs = []
            for i, s, n, last in batch:
                job = self._job_at.get(i)
                if job is None:  # a submitted request's first yield
                    job = self._job_at[i] = self.stats.keys.pop(i)
                kids = []
                if last:
                    child = self.stats.children.get(i)
                    kids = ([] if child is None else [child]) + self.stats.fanout.get(i, [])
                for c in kids:
                    self._job_at[c] = job
                jobs.append((job, not kids))
            self._serve(dev, requests, batch, jobs)
            for (i, _, _, last), (job, final) in zip(batch, jobs):
                if last:  # every stage's outputs are handed out once its final yield is served: release it
                    del self._job_at[i], requests[i]
                    self.stats.children.pop(i, None)
                    self.stats.fanout.pop(i, None)
                    self.stats.cancelled.discard(i)
                    if self.stats.failed.pop(i, None) is not None:
                        self._source.cancel(job)  # a failed job's other live stages are stopped at the next poll
                    if final and job.done():  # a job of several final stages (a fan-out) ends with the last one
                        with self._lock:
                            self._pending.discard(job)

    def _serve(self, dev, requests, batch, jobs) -> None:
        """Hand one poll's yields ``batch`` (``stream_schedule``) to their ``jobs``: ``(job, final)`` per yield,
        ``final`` False on the last yield of a stage that has a follow-up.  The slots' outputs are valid here."""
        raise NotImplementedError


class GptEngine(OpenEngine):
    """``GPT.open_engine``: a job's result is its ``GenerationOutputs``, the outputs ``GPT.generate`` gives the request
    alone; a streaming job yields ``(GenerationOutputs, last)``, the yields of ``GPT.generate_continuous_stream`` for
    it (for a request with a follow-up: every stage's, ``last`` only on the final one)."""

    def _receive(self, value, event):
        # the harvest copies were made on the engine's stream: order the caller's stream after them, and tell the
        # caching allocator that the caller's stream uses the tensors
        if event is not None:
            out = value[0] if isinstance(value, tuple) else value
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(event)
            for t in [*out.ids, *out.hiddens, *out.logprobs, *(t for pair in out.top_logprobs for t in pair)]:
                t.record_stream(cur)
        return value

    def _serve(self, dev, requests, batch, jobs) -> None:
        done = []
        for (i, s, n, last), (job, final) in zip(batch, jobs):
            if i in self.stats.failed:
                job._fail(self.stats.failed[i])
                continue
            if job.done():
                continue
            # a cancelled request's final yield ends its job; the stream boundaries it crossed at the same poll
            # come before it and are ordinary yields
            cancelled = last and i in self.stats.cancelled
            if not (job.stream or (last and final) or cancelled):
                continue
            out = dev.empty(i) if s is None else dev.harvest(s, n)
            out.cancelled = cancelled
            done.append((job, out, last and final, cancelled))
        event = None
        if done and self._stream is not None:
            event = torch.cuda.Event()
            event.record(self._stream)
        for job, out, last, cancelled in done:
            if cancelled:
                job._cancelled = True
                job._finish(out, event)
                continue
            if job.stream:
                job._put((out, last), event)
            if last:
                job._finish(out, event)
