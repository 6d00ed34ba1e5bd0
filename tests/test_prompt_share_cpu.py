"""Shared prompts (``Request.prompt_key``), host side: the policy of ``engine._poll_cycles`` against stub devices that
model ``ctb_gpt_engine_share_prompt`` - a fixed engine, and a paged one with page reference counts - and assert what
the device refuses or must never see: a share without a running holder of at least ``c0`` columns, a write to a page
more than one slot maps, and a pool overdrawn in physical pages.  Also the checks at submission and
``ChatEngine.submit(takes=n)``.  No GPU needed."""
import random

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.core import Chat
from chattts_b200.engine import (PREFILL_CHUNK_ALIGN, Arrivals, ScheduleStats, _poll_cycles, pool_pages_needed,
                                 schedule, shared_prompt_cols)
from test_kv_pool_cpu import PagedStub
from test_paragraph_refine_cpu import _FakeChat, _open
from test_prefill_budget_cpu import ChunkStub, _req

P = _lib.PAGE_TOKENS


class ShareStub(PagedStub):
    """``PagedStub`` (``pool_pages`` None: a fixed engine, ``ChunkStub``'s checks only) with ``share`` and page
    reference counts: each slot's entries are page ids, ``refs`` counts the entries that map each page."""

    def __init__(self, slots, requests, length, pool_pages=None):
        super().__init__(slots, requests, length, pool_pages)
        self.pages = [[] for _ in range(slots)]
        self.refs = {}
        self.ids = iter(range(1, 10 ** 9))
        self.prompt_at = {}  # slot -> request index whose prompt was prefilled (or shared) there
        self.shares = []  # (src, dst, request index, c0)
        self.peak_shared = 0
        self.starts = []  # per call that starts requests (admit, share): their indices

    # ---- page accounting
    @property
    def pages_in_use(self):
        return len(self.refs)

    @property
    def shared_pages(self):
        return sum(1 for n in self.refs.values() if n > 1)

    def _map(self, s, pages):
        for p in pages:
            self.refs[p] = self.refs.get(p, 0) + 1
        self.pages[s] += pages
        self.mapped[s] = len(self.pages[s])
        assert len(self.refs) <= self.pool_pages - 1, "the pool is overdrawn"
        self.peak = max(self.peak, len(self.refs))
        self.peak_shared = max(self.peak_shared, self.shared_pages)

    def _unmap(self, s):
        for p in self.pages[s]:
            self.refs[p] -= 1
            if not self.refs[p]:
                del self.refs[p]
        self.pages[s] = []
        self.mapped[s] = 0

    def _private(self, s, lo, hi):
        if self.pool_pages is None:
            return
        for k in range(lo // P, min(-(-hi // P), len(self.pages[s]))):
            assert self.refs[self.pages[s][k]] == 1, f"slot {s} writes positions [{lo},{hi}) into a shared page"

    def reserve(self, slots, tokens):
        self.calls.append(["reserve", list(slots), list(tokens)])
        new = [max(0, -(-t // P) - len(self.pages[s])) for s, t in zip(slots, tokens)]
        if len(self.refs) + sum(new) > self.pool_pages - 1:
            return False
        for s, k in zip(slots, new):
            self._map(s, [next(self.ids) for _ in range(k)])
        return True

    def release(self, slots):
        super().release(slots)
        for s in slots:
            self._unmap(s)
            self.prompt_at.pop(s, None)

    # ---- device calls
    def admit(self, batch):
        for s, i in batch:
            self._private(s, 0, self._T(i))
        (ChunkStub if self.pool_pages is None else PagedStub).admit(self, batch)
        for s, i in batch:
            self.prompt_at[s] = i
        self.starts.append([i for _, i in batch])

    def prefill_chunk(self, s, i, c0, n):
        self._private(s, c0, c0 + n)
        if c0 + n < self._T(i) or c0 == 0:
            self.prompt_at.pop(s, None)
        (ChunkStub if self.pool_pages is None else PagedStub).prefill_chunk(self, s, i, c0, n)
        if c0 + n == self._T(i):
            self.prompt_at[s] = i

    def share(self, src, dst, i, c0):
        self.calls.append(["share", src, dst, i, c0])
        T = self._T(i)
        j = self.prompt_at.get(src)
        assert j is not None and self.owner[src] == j and self.state[src] != _lib.SLOT_IDLE, "no holder in src"
        assert self.requests[j].prompt_key == self.requests[i].prompt_key and src not in self.prog
        assert c0 == shared_prompt_cols(T) > 0 and self._T(j) >= c0, "the holder's prompt is shorter than c0"
        assert (T > 1024) == (self._T(j) > 1024)
        assert self.state[dst] != _lib.SLOT_RUNNING and dst not in self.prog and src != dst
        if self.pool_pages is not None:
            assert not self.pages[dst], "dst has pages mapped"
            own = -(-T // P) - c0 // P
            if len(self.refs) + own > self.pool_pages - 1:
                return False
            self._map(dst, self.pages[src][:c0 // P] + [next(self.ids) for _ in range(own)])
        self.prog[dst] = [i, T, c0]
        self.prompt_at.pop(dst, None)
        self.shares.append((src, dst, i, c0))
        self.starts.append([i])
        return True

    def decode(self, n):
        for s in range(self.slots):
            if self.state[s] == _lib.SLOT_RUNNING:
                i = self.owner[s]
                hi = min(self._T(i) + self.done[s] - 1 + n, self._T(i) + self.requests[i].max_new_token - 1)
                self._private(s, self._T(i) + self.done[s] - 1, hi)
        (ChunkStub if self.pool_pages is None else PagedStub).decode(self, n)

    def suspend(self, s):
        image = super().suspend(s)
        self._unmap(s)
        self.prompt_at.pop(s, None)
        return image

    def resume(self, s, image):
        super().resume(s, image)
        self._private(s, 0, self.mapped[s] * P)  # a resumed request holds private pages only


def _keyed(Ts, takes, seed0=0, max_new=(20, 64, 200), rnd=None, unkeyed=0):
    """``takes`` keyed requests per prompt length in ``Ts`` (consecutive), then ``unkeyed`` ordinary ones."""
    rnd = rnd or random.Random(0)
    reqs = []
    for g, T in enumerate(Ts):
        for k in range(takes):
            r = _req(T, seed=seed0 + 100 * g + k, max_new=rnd.choice(max_new))
            r.prompt_key = ("utt", g)
            reqs.append(r)
    reqs += [_req(rnd.choice([40, 200, 1500]), seed=9000 + k, max_new=rnd.choice(max_new)) for k in range(unkeyed)]
    return reqs


def _unkeyed(reqs):
    out = []
    for r in reqs:
        c = _req(int(r.emb.shape[0]), seed=r.manual_seed, max_new=r.max_new_token, text=r.infer_text)
        out.append(c)
    return out


def _fifo(dev):
    """The requests in the order they started, poll by poll (within a poll the shares follow the admission); asserts
    that no request starts at an earlier poll than one queued before it."""
    polls, cur = [], []
    for c in dev.calls:
        if c[0] == "decode":
            polls.append(sorted(cur))
            cur = []
        elif c[0] == "admit":
            cur += [i for _, i in c[1]]
        elif c[0] == "share" or (c[0] == "chunk" and c[3] == 0):
            cur.append(c[3] if c[0] == "share" else c[2])
    order = [i for p in polls + [sorted(cur)] for i in p]
    assert order == sorted(order), polls
    return order


def _run(reqs, length, slots, pool=None, chunk=8, budget=None):
    dev = ShareStub(slots, reqs, length, pool)
    stats = ScheduleStats()
    out = list(schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget))
    return dev, stats, sorted((i, n) for i, _, n in out)


@pytest.mark.parametrize("seed", range(10))
def test_shares_give_the_results_of_the_unkeyed_workload(seed):
    """Random keyed groups mixed with ordinary requests, fixed and paged, with and without a budget: every request ends
    as in the same workload without keys, every share has a holder (asserted by the stub), no write reaches a shared
    page, and the pool bound holds in physical pages."""
    rnd = random.Random(seed)
    Ts = [rnd.choice([100, 200, 700, 1024, 1500, 4000]) for _ in range(rnd.randint(1, 4))]
    reqs = _keyed(Ts, rnd.choice([2, 5, 12]), rnd=rnd, unkeyed=rnd.randint(0, 6))
    lengths = [rnd.choice([0, 1, 2, 30, 64, 200]) for _ in reqs]
    length = (lambda i: min(lengths[i], reqs[i].max_new_token) if i < len(reqs) else 9)
    slots = rnd.choice([4, 8, 16])
    budget = rnd.choice([None, 128, 1024])
    _, _, want = _run(_unkeyed(reqs), length, slots, None, budget=budget)
    for pool in (None, max(pool_pages_needed(r) for r in reqs) + 1 + rnd.choice([0, 40]), 10 ** 6):
        dev, stats, got = _run(reqs, length, slots, pool, budget=budget)
        assert got == want
        assert stats.shares == len(dev.shares) and stats.shared_cols == sum(c0 for *_, c0 in dev.shares)
        if pool is not None:
            assert dev.peak <= pool - 1 and stats.peak_pages <= pool - 1
            assert stats.peak_shared_pages <= dev.peak_shared
            assert stats.suspensions == stats.resumes
        if budget is not None:
            assert max(dev.polls) <= budget
        if not any(lengths[i] == 0 for i in range(len(reqs))):  # no unseeded requeues either: all seeded
            _fifo(dev)
        if pool == 10 ** 6 or pool is None:
            shareable = sum(1 for r in reqs if r.prompt_key is not None and int(r.emb.shape[0]) > PREFILL_CHUNK_ALIGN)
            assert stats.shares <= shareable


def test_members_waiting_together_share_from_the_first_at_the_same_poll():
    reqs = _keyed([700], 4) + _keyed([100], 2, seed0=50)  # the 100-token prompts never share
    for r in reqs[4:]:
        r.prompt_key = "short"
    dev, stats, _ = _run(reqs, lambda i: 30, 8)
    # requests take slots in FIFO order; the shares follow the poll's admission, in order
    assert dev.calls[0] == ["admit", [[0, 0], [4, 4], [5, 5]]]
    assert dev.calls[1:7] == [c for k in (1, 2, 3) for c in (["share", 0, k, k, 640], ["chunk", k, k, 640, 60])]
    assert stats.shares == 3 and stats.shared_cols == 3 * 640 and stats.admissions == 1


def test_fifo_order_and_the_budget():
    """Budget 128: each poll prefills at most 128 columns; the members wait for the first take's chunks and then share
    (their final chunks are 60 columns); requests start in FIFO order."""
    reqs = _keyed([700], 3) + [_req(40, seed=77)]
    dev, stats, got = _run(reqs, lambda i: 200, 4, budget=128)
    assert max(dev.polls) <= 128
    assert _fifo(dev) == [0, 1, 2, 3]
    assert stats.shares == 2 and stats.chunks >= 6
    assert got == _run(_unkeyed(reqs), lambda i: 200, 4, budget=128)[2]


def test_a_member_without_a_holder_is_an_ordinary_request_and_becomes_the_holder():
    """Two slots: take 0 ends before take 1 is admitted, so take 1 is admitted normally; take 2 then shares from it."""
    takes = _keyed([300], 3)
    reqs = [takes[0], _req(40, seed=5), takes[1], takes[2]]
    dev, stats, got = _run(reqs, lambda i: [2, 9, 200, 10][i], 2)
    assert dev.calls[0] == ["admit", [[0, 0], [1, 1]]] and ["admit", [[0, 2]]] in dev.calls
    assert dev.shares == [(0, 1, 3, 256)]
    assert got == [(0, 2), (1, 9), (2, 200), (3, 10)]


def test_cancelling_a_holder_keeps_the_members_pages_and_results():
    """Take 0 is cancelled while takes 1..3 read its pages: the shared pages stay mapped until the last slot that maps
    them is released, and the other takes end with all their tokens."""
    reqs = _keyed([1500], 4, max_new=(200,))
    dev = ShareStub(4, reqs, lambda i: 200, pool_pages_needed(reqs[0]) * 4 + 1)
    src = Arrivals()
    stats = ScheduleStats()
    gen = _poll_cycles([], dev, 8, stats=stats, source=src)
    src.submit_all([(k, r) for k, r in enumerate(reqs)])
    next(gen)  # take 0 admitted, takes 1..3 share from it
    assert stats.shares == 3 and dev.shared_pages == 1408 // P
    src.cancel(0)
    ended = []
    while 0 not in stats.cancelled:
        ended += next(gen)[2]
    assert dev.shared_pages == 1408 // P and not dev.pages[0]  # released by take 0, still mapped by three slots
    src.close()
    for _, _, e in gen:
        ended += e
    assert sorted((i, n) for i, _, n, _ in ended if i != 0) == [(1, 200), (2, 200), (3, 200)]
    assert not dev.refs  # every page back once the last take was released


def test_suspended_members_resume_into_private_pages():
    """A pool that holds fewer than all the takes once they grow: members are suspended (last admitted first), resumed
    into pages of their own (asserted by the stub) and end as without keys."""
    reqs = _keyed([700], 6, max_new=(300,))
    need = pool_pages_needed(reqs[0])
    length = (lambda i: 300)
    want = _run(_unkeyed(reqs), length, 6, 10 ** 6)[2]
    dev, stats, got = _run(reqs, length, 6, 2 * need + 1)
    assert got == want
    assert stats.suspensions > 0 and stats.resumes == stats.suspensions and stats.shares > 0
    assert dev.peak <= 2 * need


def test_the_pool_counts_physical_pages():
    """Eight takes of a 4,000-token prompt in a pool that holds one private copy and the takes' own pages only: they
    all run at once, which only physical counting allows."""
    reqs = _keyed([4000], 8, max_new=(20,))
    c0 = shared_prompt_cols(4000)
    own = -(-(4000 + 20) // P) - c0 // P
    pool = pool_pages_needed(reqs[0]) + 7 * own + 1
    dev, stats, got = _run(reqs, lambda i: 20, 8, pool, chunk=32)
    assert stats.shares == 7 and stats.suspensions == 0
    assert stats.peak_pages <= pool - 1 and stats.peak_shared_pages == c0 // P
    assert got == [(i, 20) for i in range(8)]


def test_submit_refuses_a_mismatched_prompt_and_too_many_takes():
    from chattts_b200.gpt import GPT

    gpt = GPT.__new__(GPT)
    gpt._open, gpt._handle, gpt.max_batch, gpt.max_context, gpt.num_vq = None, 1, 8, 4096, 4
    a, b, c = _req(300, seed=1), _req(300, seed=2), _req(300, seed=3)
    b.emb = b.emb + 1
    c.emb = torch.zeros(301, 4)
    try:
        for r in (a, b, c):
            r.prompt_key = "k"
        gpt._engine_args("t", [a, _req(300, seed=4)], 2, False, False, None, 8, 8)
        for bad in (b, c):
            with pytest.raises(ValueError, match="prompt_key"):
                gpt._engine_args("t", [a, bad], 2, False, False, None, 8, 8)
        *_, check = gpt._engine_args("t", [a], 2, False, False, None, 8, 8)
        with pytest.raises(ValueError, match="prompt_key"):
            check(b)  # a submission to an open engine is checked against the key's first live request
    finally:
        gpt._handle = None

    chat = _TakesChat()
    eng, _ = _open(chat, slots=4)
    with eng:
        p = Chat.InferCodeParams(manual_seed=3, max_new_token=200)
        with pytest.raises(ValueError, match="takes"):
            eng.submit("a", p, takes=5)  # above the slot count
        for kw in ({"stream": True}, {"split_text": True}, {"skip_refine_text": False}):
            with pytest.raises(ValueError, match="takes"):
                eng.submit("a", p, takes=2, **kw)


class _TakesChat(_FakeChat):
    """``_FakeChat`` whose code requests of any text yield 9 + 8 * b tokens for take b of their batch."""

    def __init__(self):
        super().__init__({}, {})

    def length(self, r):
        return 9 + 8 * (r.noise_batch or (1, 0))[1]


def test_chat_engine_takes_return_one_waveform_per_take_and_cancel_together():
    chat = _TakesChat()
    eng, devs = _open(chat, slots=4)
    with eng:
        p = Chat.InferCodeParams(manual_seed=3, max_new_token=200)
        wavs = eng.submit("a", p, takes=3).result(timeout=30)
    assert isinstance(wavs, list) and [w.shape[0] for w in wavs] == [512 * (9 + 8 * k) - 256 for k in range(3)]
    assert all(isinstance(w, np.ndarray) for w in wavs)
    assert len(chat.codes) == 1  # one prompt, embedded once
    with _open(chat, slots=4)[0] as eng2:
        job = eng2.submit("a", Chat.InferCodeParams(max_new_token=200), takes=3)
        job.cancel()
        with pytest.raises(Exception):
            job.result(timeout=30)
        assert job.cancelled()
