"""KV pages on demand (``kv_pool_bytes``), host side: the pool policy of ``engine._poll_cycles`` against a stub device
that holds the pool's page accounting and asserts what the paged engine refuses or must never see: a prompt, chunk
or decode chunk that writes past its slot's pages, a pool overdrawn, a suspension that is not of the running request
admitted last or that finds the request where its last resume left it, and an admission while a request is
suspended.  No GPU needed."""
import random

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import (Arrivals, Request, ScheduleStats, _poll_cycles, kv_pool_pages, pool_pages_needed,
                                 schedule, stream_schedule)
from test_prefill_budget_cpu import ChunkStub, _req

P = _lib.PAGE_TOKENS


class PagedStub(ChunkStub):
    """``ChunkStub`` with a pool of ``pool_pages`` pages (page 0 the zero page)."""

    def __init__(self, slots, requests, length, pool_pages):
        super().__init__(slots, requests, length)
        self.pool_pages = pool_pages
        self.mapped = [0] * slots
        self.peak = 0
        self.admitted = []  # request indices in admission order
        self.images = {}  # id -> image of each suspended request
        self.suspended_slots = []  # (request index, slot it left)
        self.resumed_slots = []  # (request index, slot it entered)
        self.resumed_at = {}  # request index -> its tokens when it was last resumed

    @property
    def pages_in_use(self):
        return sum(self.mapped)

    @property
    def host_bytes(self):
        return 1000 * len(self.images)

    def _T(self, i):
        return int(self.requests[i].emb.shape[0])

    def reserve(self, slots, tokens):
        self.calls.append(["reserve", list(slots), list(tokens)])
        want = [max(self.mapped[s], -(-t // P)) for s, t in zip(slots, tokens)]
        if self.pages_in_use + sum(w - self.mapped[s] for s, w in zip(slots, want)) > self.pool_pages - 1:
            return False
        for s, w in zip(slots, want):
            self.mapped[s] = w
        self.peak = max(self.peak, self.pages_in_use)
        return True

    def release(self, slots):
        self.calls.append(["release", list(slots)])
        for s in slots:
            assert self.state[s] != _lib.SLOT_RUNNING and s not in self.prog, "pages of a live slot released"
            self.mapped[s] = 0

    def admit(self, batch):
        assert not self.images, "a waiting request was admitted while one is suspended"
        for s, i in batch:
            assert self.mapped[s] * P >= self._T(i), "admission past the slot's pages"
        super().admit(batch)
        self.admitted += [i for _, i in batch]

    def prefill_chunk(self, s, i, c0, n):
        assert self.mapped[s] * P >= c0 + n, "chunk past the slot's pages"
        super().prefill_chunk(s, i, c0, n)
        if c0 + n == self._T(i):
            self.admitted.append(i)

    def decode(self, n):
        for s in range(self.slots):
            if self.state[s] == _lib.SLOT_RUNNING:  # positions after n steps: T + tokens - 1 + n, at most T + max_new - 1
                i = self.owner[s]
                need = min(self._T(i) + self.done[s] - 1 + n, self._T(i) + self.requests[i].max_new_token - 1)
                assert self.mapped[s] * P >= need, "decode chunk past the slot's pages"
        super().decode(n)

    def suspend(self, s):
        self.calls.append(["suspend", s])
        assert self.state[s] == _lib.SLOT_RUNNING and s not in self.prog
        running = [self.owner[b] for b in range(self.slots) if self.state[b] == _lib.SLOT_RUNNING and b not in self.prog]
        assert max(running, key=self.admitted.index) == self.owner[s], "the victim is not the last admitted"
        assert self.done[s] > self.resumed_at.get(self.owner[s], -1), "suspended again before it moved"
        image = (self.owner[s], self.done[s], self.target[s])
        self.images[id(image)] = image
        self.suspended_slots.append((self.owner[s], s))
        self.state[s], self.owner[s], self.mapped[s] = _lib.SLOT_IDLE, None, 0
        return image

    def resume(self, s, image):
        self.calls.append(["resume", s])
        assert self.state[s] != _lib.SLOT_RUNNING and s not in self.prog
        i, done, target = self.images.pop(id(image))
        assert self.mapped[s] * P >= self._T(i) + done - 1, "resume past the slot's pages"
        self.owner[s], self.done[s], self.target[s] = i, done, target
        self.state[s], self.fin[s] = _lib.SLOT_RUNNING, 0
        self.resumed_slots.append((i, s))
        self.resumed_at[i] = done

    def harvest(self, s, n, copy=True):
        if isinstance(s, tuple):  # an image: a suspended request cancelled or interrupted
            self.images.pop(id(s), None)
            return ("out", s[0], n)
        return super().harvest(s, n, copy)


def _workload(rnd, n, max_T=300):
    reqs = [_req(rnd.choice([5, 8, 40, 130, max_T]), seed=k, max_new=rnd.choice([20, 64, 200]),
                 text=rnd.random() < 0.2) for k in range(n)]
    lengths = [rnd.choice([0, 1, 2, 30, 64, 200]) for _ in range(n)]
    return reqs, (lambda i: min(lengths[i], reqs[i].max_new_token) if i < n else 9)


def _run(reqs, length, slots, pool, chunk=8, budget=None, stream=False, **kw):
    dev = PagedStub(slots, reqs, length, pool)
    stats = ScheduleStats()
    if stream:
        out = [y for batch in stream_schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget, **kw)
               for y in batch]
    else:
        out = list(schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget, **kw))
    return dev, stats, out


def _fits(reqs):
    return max(pool_pages_needed(r) for r in reqs) + 1


@pytest.mark.parametrize("seed", range(8))
def test_pool_bounds_coverage_and_results(seed):
    """Every request ends with the tokens of the fixed-page run, the pages never exceed the pool, every prompt, chunk,
    decode chunk and resume is covered (asserted by the stub), and the stats record what happened."""
    rnd = random.Random(seed)
    reqs, length = _workload(rnd, rnd.randint(4, 24))
    slots = rnd.choice([2, 3, 8])
    budget = rnd.choice([None, 128])
    _, _, want = _run(reqs, length, slots, 10 ** 6, budget=budget)
    for pool in (_fits(reqs), _fits(reqs) + 7, 10 ** 6):
        dev, stats, got = _run(reqs, length, slots, pool, budget=budget)
        assert sorted((i, n) for i, _, n in got) == sorted((i, n) for i, _, n in want)  # slots may differ
        assert dev.peak <= pool - 1 and stats.peak_pages == max(stats.pages) <= pool - 1
        assert stats.suspensions == stats.resumes == len(dev.suspended_slots)
        assert not dev.images
        if pool == 10 ** 6:
            assert stats.suspensions == 0


def test_small_pool_suspends_last_admitted_and_resumes_first():
    """A pool that holds two of four long requests: the later admissions are suspended (last admitted first, checked by
    the stub), resumed before the waiting requests are admitted (checked by the stub), and all end as without a pool."""
    reqs = [_req(40, seed=k, max_new=200) for k in range(6)]
    length = (lambda i: 200)
    _, _, want = _run(reqs, length, 4, 10 ** 6)
    dev, stats, got = _run(reqs, length, 4, 2 * pool_pages_needed(reqs[0]) + 1)
    assert sorted((i, n) for i, _, n in got) == sorted((i, n) for i, _, n in want)
    assert stats.suspensions >= 2 and stats.resumes == stats.suspensions
    assert max(stats.host_bytes) > 0 and stats.host_bytes[-1] == 0


def test_one_request_needing_the_whole_pool_does_not_livelock():
    reqs = [_req(100, seed=k, max_new=300) for k in range(5)]
    dev, stats, got = _run(reqs, lambda i: 300, 3, _fits(reqs))
    assert sorted(i for i, _, _ in got) == list(range(5)) and all(n == 300 for _, _, n in got)
    assert dev.peak <= _fits(reqs) - 1


def test_prompt_in_progress_is_never_suspended():
    reqs = [_req(40, seed=0, max_new=200), _req(1000, seed=1, max_new=64), _req(40, seed=2, max_new=200)]
    dev, stats, got = _run(reqs, lambda i: reqs[i].max_new_token, 3, _fits(reqs) + 4, budget=128)
    assert sorted(i for i, _, _ in got) == [0, 1, 2]
    assert stats.suspensions > 0  # none of them while the long prompt was in progress (asserted by the stub)
    assert stats.chunks > 1


def test_streamed_yields_equal_the_unsuspended_run():
    rnd = random.Random(5)
    reqs, length = _workload(rnd, 16)
    _, _, want = _run(reqs, length, 4, 10 ** 6, stream=True)
    dev, stats, got = _run(reqs, length, 4, _fits(reqs), stream=True)
    assert stats.suspensions > 0

    def per_request(ys):
        out = {}
        for i, _, n, last in ys:
            out.setdefault(i, []).append((n, last))
        return out

    assert per_request(got) == per_request(want)


def test_follow_ups_run_after_a_suspension():
    kids = {}

    def then(k):
        def f(out):
            kids[k] = out
            return _req(8, seed=100 + k, max_new=20)
        return f

    reqs = [_req(40, seed=k, max_new=200, then=then(k)) for k in range(4)]
    stats = ScheduleStats()
    dev = PagedStub(4, reqs, lambda i: reqs[i].max_new_token, 2 * pool_pages_needed(reqs[0]) + 1)
    got = list(schedule(reqs, dev, 8, stats=stats))
    assert stats.suspensions > 0 and sorted(kids) == [0, 1, 2, 3]
    assert sorted(i for i, _, _ in got) == list(range(8))


def test_cancel_and_interrupt_end_a_suspended_request_with_its_tokens():
    reqs = [_req(40, seed=k, max_new=200) for k in range(4)]
    dev = PagedStub(4, reqs, lambda i: 200, 2 * pool_pages_needed(reqs[0]) + 1)
    src = Arrivals()
    stats = ScheduleStats()
    gen = _poll_cycles([], dev, 8, stats=stats, source=src)
    for k, r in enumerate(reqs):
        src.submit(r, key=k)
    while not dev.images:
        next(gen)
    (i, _, _), = dev.images.values()
    src.cancel(i)
    ended = []
    while i not in stats.cancelled:
        ended += next(gen)[2]
    (n,) = [n for j, s, n, _ in ended if j == i and isinstance(s, tuple)]
    assert n > 0
    assert dev.harvest(next(s for j, s, _, _ in ended if j == i), n) == ("out", i, n)
    assert all(im[0] != i for im in dev.images.values())
    src.close()
    for _ in gen:
        pass

    class Ctx:
        flag = False

        def get(self):
            return self.flag

    ctx = Ctx()
    dev = PagedStub(4, reqs, lambda i: 200, 2 * pool_pages_needed(reqs[0]) + 1)
    gen = _poll_cycles(list(reqs), dev, 8, context=ctx)
    while not dev.images:
        next(gen)
    ctx.flag = True
    _, _, ended = next(gen)
    parked = [(j, n) for j, s, n, _ in ended if isinstance(s, tuple)]
    assert parked and all(n > 0 for _, n in parked)
    assert {j for j, _, _, _ in ended} >= {j for j, _ in parked}


def test_submit_check_and_pool_size():
    from types import SimpleNamespace

    from chattts_b200.gpt import GPT

    cfg = SimpleNamespace(num_key_value_heads=12, head_dim=64, num_hidden_layers=20)
    page32 = 2 * 12 * 16 * 64 * 4 * 20
    assert kv_pool_pages(cfg, None, 0) is None
    assert kv_pool_pages(cfg, 10 * page32 + 5, 0) == 10
    assert kv_pool_pages(cfg, 10 * page32, _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV) == 20
    with pytest.raises(ValueError):
        kv_pool_pages(cfg, page32, 0)
    gpt = GPT.__new__(GPT)
    gpt._open, gpt._handle, gpt.max_batch, gpt.max_context, gpt.num_vq = None, 1, 8, 4096, 4
    ok, big = _req(100, max_new=60), _req(100, max_new=400)  # 10 and 32 pages
    try:
        gpt._engine_args("t", [ok], 2, False, False, None, 8, 8, None, 11)
        with pytest.raises(ValueError, match="KV pages"):
            gpt._engine_args("t", [ok, big], 2, False, False, None, 8, 8, None, 11)
        *_, check = gpt._engine_args("t", [ok], 2, False, False, None, 8, 8, 400, 11)
        with pytest.raises(ValueError, match="KV pages"):
            check(big)  # a follow-up or a submission is refused as well
    finally:
        gpt._handle = None  # a stand-in: nothing to destroy
