"""The slot engine's prefill budget (``prefill_budget``), host side: the scheduling policy of ``engine._poll_cycles``
against a stub device that records every device call and checks the chunk contract of
``ctb_gpt_engine_prefill_chunk``.  No GPU needed."""
import json
import os
import random

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import (MIN_PROMPT_COLS, PREFILL_CHUNK_ALIGN, Arrivals, Request, ScheduleStats,
                                 SlotStatus, _poll_cycles, admission_cols, check_prefill_budget, schedule,
                                 stream_schedule)

MAX_CONTEXT = 8192
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "engine_calls_no_budget.json")


class ChunkStub:
    """Slot engine stand-in.  Request i yields ``length(i)`` tokens once admitted (0: EOS first).  Records the device
    calls in ``calls``; asserts what the device refuses or must never see: a chunk that does not continue its prompt
    or is misaligned, an admission or chunk into a running slot, and an admission into a slot whose prompt is in
    progress (a reserved slot)."""

    def __init__(self, slots, requests, length):
        self.slots, self.requests, self.length = slots, requests, length
        self.max_context = MAX_CONTEXT
        self.state = [_lib.SLOT_IDLE] * slots
        self.done = [0] * slots
        self.fin = [0] * slots
        self.target = [0] * slots
        self.owner = [None] * slots
        self.prog = {}  # slot -> [request index, T0, columns done]
        self.calls = []
        self.poll = []  # prefilled columns of each call of the poll in progress
        self.polls = []  # prefilled columns of each poll: up to a decode call, or a status read with nothing running
        self.started = []  # request indices in the order their prefill began
        self.steps = 0

    def _start(self, s, i):
        assert self.state[s] != _lib.SLOT_RUNNING, "admission into a running slot"
        length = self.length(i)
        self.owner[s], self.target[s] = i, length
        self.done[s], self.fin[s] = min(1, length), int(length == 0)
        self.state[s] = _lib.SLOT_RUNNING if length > 1 else _lib.SLOT_FINISHED

    def admit(self, batch):
        self.calls.append(["admit", [list(p) for p in batch]])
        for s, i in batch:
            assert s not in self.prog, "a reserved slot was refilled"
            self.started.append(i)
            self._start(s, i)
        self.poll.append(admission_cols(batch, self.requests, self.max_context))

    def prefill_chunk(self, s, i, c0, n):
        self.calls.append(["chunk", s, i, c0, n])
        T = int(self.requests[i].emb.shape[0])
        assert self.state[s] != _lib.SLOT_RUNNING, "chunk into a running slot"
        assert c0 % PREFILL_CHUNK_ALIGN == 0 and 0 < n and c0 + n <= T
        assert c0 + n == T or n % PREFILL_CHUNK_ALIGN == 0, "misaligned chunk"
        if c0 == 0:
            assert s not in self.prog, "a reserved slot was refilled"
            self.prog[s] = [i, T, 0]
            self.started.append(i)
        assert self.prog[s][:1] == [i] and self.prog[s][2] == c0, "the chunk does not continue its prompt"
        self.poll.append(max(MIN_PROMPT_COLS, n) if c0 == 0 and n == T else n)
        self.prog[s][2] = c0 + n
        if c0 + n == T:
            del self.prog[s]
            self._start(s, i)

    def cancel(self, slots):
        self.calls.append(["cancel", list(slots)])
        for s in slots:
            self.prog.pop(s, None)
            if self.state[s] == _lib.SLOT_RUNNING:
                self.state[s], self.fin[s] = _lib.SLOT_FINISHED, 0

    def decode(self, n):
        self.calls.append(["decode", n])
        self.polls.append(sum(self.poll))
        self.poll = []
        if any(st == _lib.SLOT_RUNNING for st in self.state):
            self.steps += n
        for s in range(self.slots):
            if self.state[s] == _lib.SLOT_RUNNING:
                self.done[s] = min(self.done[s] + n, self.target[s])
                if self.done[s] == self.target[s]:
                    self.state[s], self.fin[s] = _lib.SLOT_FINISHED, 1

    def status(self):
        self.calls.append(["status"])
        if not any(st == _lib.SLOT_RUNNING for st in self.state):  # no slot waits for the next poll's prefill
            self.polls.append(sum(self.poll))
            self.poll = []
        return SlotStatus(list(self.state), list(self.done), list(self.fin), self.steps)

    def harvest(self, s, n, copy=True):
        assert s not in self.prog, "a reserved slot was harvested"
        return ("out", self.owner[s], n)

    def empty(self, i=None):
        return ("empty", i, 0)


def _req(T, seed=0, max_new=64, then=None, text=False):
    return Request(emb=torch.zeros(T, 4), temperature=[0.3], eos_token=625, max_new_token=max_new, manual_seed=seed,
                   then=then, infer_text=text)


def _workload(rnd, n):
    """n seeded requests of mixed prompt lengths (short, speaker-sample sized and long), code and text"""
    Ts = [5, 8, 40, 130, 300, 470, 520, 1000, 1024, 1025, 2085, 4000]
    reqs = [_req(rnd.choice(Ts), seed=k, max_new=rnd.choice([1, 20, 64, 200]), text=rnd.random() < 0.2)
            for k in range(n)]
    lengths = [rnd.choice([0, 1, 2, 7, 30, 64, 150]) for _ in range(n)]
    return reqs, (lambda i: min(lengths[i], reqs[i].max_new_token) if i < n else 9)


def _run(reqs, length, slots, budget, chunk=8, stream=False, **kw):
    dev = ChunkStub(slots, reqs, length)
    stats = ScheduleStats()
    if stream:
        out = [y for batch in stream_schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget, **kw)
               for y in batch]
    else:
        out = list(schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget, **kw))
    dev.polls.append(sum(dev.poll))
    return dev, stats, out


def _golden_workloads():
    rnd = random.Random(11)
    return [(_workload(rnd, rnd.randint(1, 20)), rnd.choice([2, 3, 8]), rnd.choice([4, 8, 24])) for _ in range(12)]


def test_no_budget_issues_the_device_calls_of_before():
    """Device-call sequences recorded on seeded random workloads before the budget existed"""
    with open(GOLDEN) as f:
        golden = json.load(f)
    work = _golden_workloads()
    assert len(golden) == len(work)
    for k, ((reqs, length), slots, chunk) in enumerate(work):
        dev, _, _ = _run(reqs, length, slots, None, chunk)
        assert dev.calls == golden[k], k
        assert not any(c[0] in ("chunk", "cancel") for c in dev.calls)


@pytest.mark.parametrize("budget", [128, 640, 1024, 3000])
def test_budget_bounds_every_poll_and_changes_no_result(budget):
    rnd = random.Random(budget)
    for trial in range(40):
        reqs, length = _workload(rnd, rnd.randint(1, 24))
        slots, chunk = rnd.choice([2, 4, 8]), rnd.choice([4, 8, 24])
        dev, stats, out = _run(reqs, length, slots, budget, chunk)
        assert max(dev.polls) <= budget and max(stats.prefill_cols) <= budget, (trial, dev.polls)
        assert sum(dev.polls) == sum(stats.prefill_cols)
        assert stats.chunks == sum(c[0] == "chunk" for c in dev.calls)
        # a prompt wider than the budget is always chunked, never admitted whole
        assert all(int(reqs[i].emb.shape[0]) <= budget for c in dev.calls if c[0] == "admit" for _, i in c[1])
        # FIFO: every request's prefill begins in request order, and each ends once with its own tokens
        assert dev.started == list(range(len(reqs)))
        ref = _run(reqs, length, slots, None, chunk)[2]
        assert sorted((i, n) for i, _, n in out) == sorted((i, n) for i, _, n in ref)
        assert all(n == length(i) for i, _, n in out)
        assert not dev.prog


def test_every_poll_with_work_waiting_prefills():
    rnd = random.Random(5)
    for trial in range(30):
        reqs, length = _workload(rnd, rnd.randint(2, 16))
        dev = ChunkStub(rnd.choice([2, 4]), reqs, length)
        started, ended = set(), set()
        polls = []  # per poll: (waiting work at its start, prefilled something)
        orig_decode = dev.decode

        def decode(n):
            polls.append(dev.poll_start + (bool(dev.poll),))
            orig_decode(n)
            mark()

        def mark():
            free = any(dev.state[s] != _lib.SLOT_RUNNING and s not in dev.prog for s in range(dev.slots))
            waiting = len(dev.started) < len(reqs)
            dev.poll_start = (bool(dev.prog), free and waiting)

        dev.decode = decode
        mark()
        list(schedule(reqs, dev, 8, prefill_budget=rnd.choice([128, 1024])))
        assert polls
        for prog, free_and_waiting, prefilled in polls:
            if prog or free_and_waiting:
                assert prefilled, trial


def test_a_prompt_that_does_not_fit_is_chunked_from_the_budget_left_over():
    reqs = [_req(100, seed=k) for k in range(3)] + [_req(4000, seed=3), _req(50, seed=4)]
    dev, stats, out = _run(reqs, lambda i: 40, 8, 1024)
    prefill = [c for c in dev.calls if c[0] in ("admit", "chunk")]
    # 3 x 100 columns fit; the 4,000-token prompt starts with 1024 - 300 = 724 -> 640 columns, request 4 waits
    assert prefill[:2] == [["admit", [[0, 0], [1, 1], [2, 2]]], ["chunk", 3, 3, 0, 640]]
    assert prefill[2:5] == [["chunk", 3, 3, 640, 1024], ["chunk", 3, 3, 1664, 1024], ["chunk", 3, 3, 2688, 1024]]
    # the final chunk (288 columns) leaves room for request 4 at the same poll, in the next free slot
    assert prefill[5:] == [["chunk", 3, 3, 3712, 288], ["admit", [[4, 4]]]]
    assert stats.prefill_cols[:5] == [940, 1024, 1024, 1024, 288 + 50]
    assert sorted(i for i, _, _ in out) == list(range(5))


def test_left_over_under_128_columns_starts_the_prompt_at_the_next_poll():
    reqs = [_req(1000, seed=0), _req(2000, seed=1)]
    dev, stats, _ = _run(reqs, lambda i: 40, 2, 1024)
    prefill = [c for c in dev.calls if c[0] in ("admit", "chunk", "decode")]
    assert prefill[:4] == [["admit", [[0, 0]]], ["decode", 8], ["chunk", 1, 1, 0, 1024], ["decode", 8]]
    assert stats.prefill_cols[:2] == [1000, 1024]


def test_follow_ups_stay_ahead_of_waiting_requests():
    child = _req(200, seed=99)
    reqs = [_req(3000, seed=0, then=lambda out: child)] + [_req(600, seed=k) for k in range(1, 5)]
    dev, stats, out = _run(reqs, lambda i: 10, 2, 1024)
    assert stats.children == {0: 5}
    # request 0's follow-up starts before every request that was still waiting when 0 ended
    first = dev.started.index(5)
    assert all(dev.started.index(i) < first for i in range(len(reqs)) if i in dev.started[:first])
    waiting_then = [i for i in range(1, 5) if i not in dev.started[:first]]
    assert waiting_then and all(dev.started.index(i) > first for i in waiting_then)


def test_streamed_yields_are_those_without_a_budget():
    rnd = random.Random(9)
    for trial in range(20):
        reqs, length = _workload(rnd, rnd.randint(1, 12))
        for r in reqs:
            r.stream_batch = rnd.choice([4, 24])
        slots = rnd.choice([2, 4])
        got = _run(reqs, length, slots, rnd.choice([128, 1024]), stream=True)[2]
        ref = _run(reqs, length, slots, None, stream=True)[2]
        per = lambda ys: {i: [(n, last) for j, _, n, last in ys if j == i] for i in range(len(reqs))}  # noqa: E731
        assert per(got) == per(ref), trial


def test_cancel_frees_the_reserved_slot_without_a_final_chunk():
    reqs = []
    src = Arrivals()
    src.submit(_req(64, seed=0), key="a")
    src.submit(_req(4000, seed=1, then=lambda out: pytest.fail("no follow-up after a cancel")), key="long")
    dev = ChunkStub(2, reqs, lambda i: 200)
    stats = ScheduleStats()
    gen = _poll_cycles(reqs, dev, 8, stats=stats, source=src, prefill_budget=1024)
    next(gen)
    assert [c for c in dev.calls if c[0] == "chunk"] == [["chunk", 1, 1, 0, 896]]  # 1024 - 64 columns left
    src.cancel("long")
    src.submit(_req(64, seed=2), key="after")
    src.close()
    ended = [e for _, _, es in gen for e in es]
    assert [c for c in dev.calls if c[0] == "chunk"] == [["chunk", 1, 1, 0, 896]]  # no final chunk
    assert ["cancel", [1]] in dev.calls and 1 in stats.cancelled
    assert (1, None, 0, False) in ended  # ends empty
    assert ["admit", [[1, 2]]] in dev.calls  # the freed slot takes the next request
    assert sorted(e[0] for e in ended) == [0, 1, 2] and not dev.prog


def test_interrupt_drops_the_prompt_in_progress():
    from chattts_b200.gpt import GPT

    ctx = GPT.Context()
    reqs = [_req(64, seed=0), _req(4000, seed=1), _req(64, seed=2)]
    dev = ChunkStub(2, reqs, lambda i: 500)
    gen = _poll_cycles(reqs, dev, 8, context=ctx, prefill_budget=1024)
    ended = list(next(gen)[2])
    ctx.set(True)  # seen by the next poll, which advances the prompt in progress once more
    ended += [e for _, _, es in gen for e in es]
    assert [e[0] for e in ended] == [0]  # the running request ends; the prompt in progress and request 2 are dropped
    assert sum(c[0] == "chunk" for c in dev.calls) == 2 and dev.calls[-1] == ["status"]


@pytest.mark.parametrize("bad", [0, 127, 100.5, -1])
def test_budget_must_be_at_least_one_aligned_chunk(bad):
    with pytest.raises(ValueError):
        check_prefill_budget(bad)
    assert check_prefill_budget(None) is None and check_prefill_budget(128) == 128
