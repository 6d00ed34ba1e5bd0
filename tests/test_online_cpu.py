"""The open slot engine without a GPU: arrivals and cancellations in the scheduling policy (engine._poll_cycles with an
Arrivals source) against a stub device, and the threading of OpenEngine / GPT.open_engine (idle waiting, submit-time
checks, worker errors, close, one engine per handle)."""
import ctypes as C
import threading
import time

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import Arrivals, GptEngine, Request, ScheduleStats, _poll_cycles
from chattts_b200.gpt import GPT
from test_continuous_cpu import StubDevice


class _Lengths:
    """Request i yields requests[i].max_new_token tokens, unless `fixed` names its lengths (0: EOS first)."""

    def __init__(self, requests, fixed=None):
        self.requests, self.fixed = requests, fixed or {}

    def __getitem__(self, i):
        return self.fixed.get(i, self.requests[i].max_new_token)


class OnlineStub(StubDevice):
    """StubDevice with the open engine's extra calls: cancel, harvest, empty."""

    def __init__(self, slots, requests, fixed=None, fail_at_decode=None):
        super().__init__(slots, _Lengths(requests, fixed))
        self.requests = requests
        self.cancels, self.decodes = [], 0
        self.fail_at_decode = fail_at_decode

    def decode(self, n):
        self.decodes += 1
        if self.fail_at_decode is not None and self.decodes >= self.fail_at_decode:
            raise _lib.CtbError("device fault")
        super().decode(n)

    def cancel(self, slots):
        self.cancels.append(list(slots))
        for s in slots:
            if self.state[s] == _lib.SLOT_RUNNING:
                self.state[s] = _lib.SLOT_FINISHED

    def harvest(self, slot, n, copy=True):
        return GPT.GenerationOutputs(ids=[torch.arange(n)], attentions=[], hiddens=[])

    def empty(self, index=None):
        return GPT.GenerationOutputs(ids=[torch.zeros(0, dtype=torch.long)], attentions=[], hiddens=[])


def _req(n, seed=0, then=None, text=False):
    return Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=n, manual_seed=seed,
                   then=then, infer_text=text)


def _drain(gen, source):
    source.close()
    return [e for _, _, ended in gen for e in ended]


def test_arrivals_queue_behind_waiting_requests_and_follow_ups():
    requests, src, stats = [], Arrivals(), ScheduleStats()
    child = _req(20, seed=9)
    r0 = _req(6, then=lambda out: child, text=True)
    for r in (r0, _req(30), _req(8), _req(9)):
        src.submit(r)
    dev = OnlineStub(2, requests)
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    next(gen)
    assert dev.admissions == [[(0, 0), (1, 1)]]
    src.submit(_req(5))  # arrives while 2 and 3 wait: index 4, behind them
    _, _, ended = next(gen)  # request 0 ends; its follow-up (index 5) goes ahead of 2, 3 and 4
    assert ended == [(0, 0, 6, False)] and stats.children == {0: 5}
    ended = _drain(gen, src)
    assert dev.admissions[1] == [(0, 5)]
    assert [i for batch in dev.admissions for _, i in batch] == [0, 1, 5, 2, 3, 4]
    assert sorted(i for i, *_ in ended) == [1, 2, 3, 4, 5]
    assert all(n == requests[i].max_new_token for i, _, n, _ in ended)
    assert not stats.cancelled


def test_cancel_a_waiting_request_never_touches_a_slot():
    requests, src, stats = [], Arrivals(), ScheduleStats()
    r = [_req(100), _req(100), _req(7)]
    for x in r:
        src.submit(x)
    dev = OnlineStub(2, requests)
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    next(gen)
    src.cancel(r[2])
    _, _, ended = next(gen)
    assert ended == [(2, None, 0, False)] and stats.cancelled == {2}
    _drain(gen, src)
    assert all(i != 2 for batch in dev.admissions for _, i in batch) and not dev.cancels


def test_cancel_a_running_request_keeps_the_count_of_the_poll_that_applied_it():
    requests, src, stats = [], Arrivals(), ScheduleStats()
    seen = []
    r = [_req(100, then=lambda out: seen.append(out)), _req(40), _req(30)]
    for x in r:
        src.submit(x)
    dev = OnlineStub(2, requests)
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    next(gen)
    next(gen)  # 9 tokens each
    src.cancel(r[0])
    st, _, ended = next(gen)  # decode to 17, then the status read: request 0 is stopped at 17
    assert st.end_idx[0] == 17 and ended == [(0, 0, 17, False)]
    assert dev.cancels == [[0]] and stats.cancelled == {0}
    ended = _drain(gen, src)
    assert dev.admissions[1] == [(0, 2)]  # the freed slot is refilled
    assert sorted((i, n) for i, _, n, _ in ended) == [(1, 40), (2, 30)]
    assert seen == []  # no follow-up after a cancel


def test_cancel_of_a_request_that_finished_at_the_same_read_counts_as_finished():
    requests, src, stats = [], Arrivals(), ScheduleStats()
    child = _req(50, seed=3)
    r = [_req(9, then=lambda out: child), _req(100)]
    for x in r:
        src.submit(x)
    dev = OnlineStub(2, requests)
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    next(gen)
    src.cancel(r[0])
    _, _, ended = next(gen)  # request 0 reaches its 9 tokens in this chunk
    assert ended[0] == (0, 0, 9, False) and 0 not in stats.cancelled and not dev.cancels
    # its follow-up was made, and the cancel moves on to it: it never takes a slot
    assert stats.children == {0: 2} and ended[1] == (2, None, 0, False) and stats.cancelled == {2}
    src.cancel(r[1])
    ended = _drain(gen, src)
    assert ended == [(1, 1, 17, False)] and stats.cancelled == {1, 2}
    assert all(i != 2 for batch in dev.admissions for _, i in batch)


def test_cancel_after_a_first_step_requeue_does_not_run_it_again():
    requests, src, stats = [], Arrivals(), ScheduleStats()
    r = _req(20, seed=None)
    src.submit(r)
    src.submit(_req(30))
    dev = OnlineStub(2, requests, fixed={0: [0, 9]})
    gen = _poll_cycles(requests, dev, 8, stats=stats, source=src)
    next(gen)  # request 0 sampled EOS first: requeued
    assert stats.requeued == 1
    src.cancel(r)
    ended = _drain(gen, src)
    assert (0, None, 0, False) in ended and stats.cancelled == {0} and dev.draws[0] == 1


def test_idle_open_engine_does_not_decode_while_it_waits():
    devs, made = [], threading.Event()

    def make(requests):
        devs.append(OnlineStub(2, requests))
        made.set()
        return devs[-1]

    eng = GptEngine(make, 8)
    try:
        assert made.wait(timeout=10)
        time.sleep(0.2)  # the worker now waits for a submission
        assert devs[0].decodes == 0 and devs[0].admissions == []
        job = eng.submit(_req(20))
        out = job.result(timeout=10)
        assert torch.equal(out.ids[0], torch.arange(20)) and not out.cancelled and job.done()
        n = devs[0].decodes
        time.sleep(0.2)
        assert devs[0].decodes == n == 3  # ceil(19 / 8) chunks, then nothing while idle
    finally:
        eng.close()
    assert not eng._thread.is_alive()


class SlowStub(OnlineStub):
    def decode(self, n):
        time.sleep(0.002)  # a decode chunk takes time, so a cancel lands while the request runs
        super().decode(n)


def test_streaming_job_and_cancelled_jobs():
    with GptEngine(lambda requests: SlowStub(2, requests), 4) as eng:
        job = eng.submit(Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=10,
                                 manual_seed=1, stream_batch=4), stream=True)
        got = [(int(o.ids[0].shape[0]), last) for o, last in job]
        assert got == [(4, False), (8, False), (10, True)]
        assert int(job.result().ids[0].shape[0]) == 10
        long = eng.submit(_req(2000), stream=True)
        waiting = [eng.submit(_req(2000)) for _ in range(3)]
        it = iter(long)
        next(it)
        long.cancel()
        assert not any(last for _, last in it)  # a cancelled stream just ends
        out = long.result(timeout=10)
        assert long.cancelled() and out.cancelled and 0 < int(out.ids[0].shape[0]) < 2000
        eng.close(cancel=True)
    for j in waiting:
        assert j.cancelled() and j.result().cancelled


def test_submit_checks_in_the_callers_thread_and_follow_up_failures_fail_their_job(monkeypatch):
    import chattts_b200.engine as engine

    monkeypatch.setattr(engine, "EngineDevice", lambda g, requests, S, cap, hidden: OnlineStub(S, requests))
    gpt = GPT({"hidden_size": 4}, embed=None, device_gpt=torch.device("cpu"), max_batch=4, max_context=300)
    gpt._handle = C.c_void_p(1)  # never reaches the library: the device layer is a stub
    try:
        with gpt.open_engine(2, 100) as eng:
            with pytest.raises(ValueError, match="max_new_cap"):
                eng.submit(_req(101))
            with pytest.raises(ValueError, match="max_context"):
                eng.submit(Request(emb=torch.zeros(250, 4), temperature=[0.3], eos_token=625, max_new_token=60))
            with pytest.raises(RuntimeError, match="open engine"):
                gpt.open_engine(2, 100)
            with pytest.raises(RuntimeError, match="open engine"):
                next(gpt.generate_continuous([_req(5)]))
            with pytest.raises(RuntimeError, match="open engine"):
                next(gpt.generate(torch.zeros(1, 5, 4), torch.zeros(1, 5, 4, dtype=torch.long), [0.3], 625))
            bad = eng.submit(_req(5, then=lambda out: _req(150)))
            ok = eng.submit(_req(7))
            with pytest.raises(ValueError, match="max_new_cap"):
                bad.result(timeout=10)
            assert int(ok.result(timeout=10).ids[0].shape[0]) == 7
        eng2 = gpt.open_engine(2, 100)  # the handle is free again
        eng2.close()
    finally:
        gpt._handle = C.c_void_p()


class GatedStub(OnlineStub):
    gate = None

    def decode(self, n):
        self.gate.wait()  # the test submits every job before the device fails
        super().decode(n)


def test_worker_error_fails_every_pending_job_and_close_raises_it():
    gate = threading.Event()
    GatedStub.gate = gate
    eng = GptEngine(lambda requests: GatedStub(2, requests, fail_at_decode=2), 8)
    jobs = [eng.submit(_req(100)) for _ in range(3)]
    gate.set()
    for j in jobs:
        with pytest.raises(_lib.CtbError, match="device fault"):
            j.result(timeout=10)
    with pytest.raises(RuntimeError):
        eng.submit(_req(5))
    with pytest.raises(_lib.CtbError, match="device fault"):
        eng.close()
    assert not eng._thread.is_alive()


def test_no_thread_left_after_an_exception_in_the_with_block():
    with pytest.raises(KeyError):
        with GptEngine(lambda requests: SlowStub(2, requests), 8) as eng:
            jobs = [eng.submit(_req(5000)) for _ in range(4)]
            raise KeyError("client went away")
    assert not eng._thread.is_alive()
    assert all(j.cancelled() for j in jobs)
    assert not [t for t in threading.enumerate() if t.name == "ctb-open-engine"]


def test_one_request_submitted_twice_gives_two_jobs():
    with GptEngine(lambda requests: SlowStub(2, requests), 8) as eng:
        r = _req(40)
        a, b = eng.submit(r), eng.submit(r, stream=True)
        c = eng.submit(r)
        c.cancel()
        assert int(a.result(timeout=10).ids[0].shape[0]) == 40
        assert [int(o.ids[0].shape[0]) for o, _ in b] == [24, 40]
        assert c.result(timeout=10).cancelled and c.cancelled() and not a.cancelled() and not b.cancelled()


def test_a_long_lived_engine_keeps_nothing_of_served_requests():
    def check(r):
        if r.max_new_token > 100:
            raise ValueError("too long")

    child = lambda out: _req(6, seed=7)  # noqa: E731
    with GptEngine(lambda requests: OnlineStub(3, requests), 4, check) as eng:
        jobs = [eng.submit(_req(10 + k % 7, then=child if k % 3 == 0 else None), stream=k % 2 == 0) for k in range(40)]
        bad = eng.submit(_req(5, then=lambda out: _req(500)))  # its follow-up fails the check
        for j in jobs[::5]:
            j.cancel()
        with pytest.raises(ValueError):
            bad.result(timeout=10)
        for j in jobs:
            j.result(timeout=10)
    assert eng._requests.held() == 0 and len(eng._requests) > 40
    assert not eng._job_at and not eng._pending
    st = eng.stats
    assert not st.children and not st.cancelled and not st.failed and not st.keys


def test_the_with_blocks_exception_survives_a_failed_worker():
    gate = threading.Event()
    GatedStub.gate = gate
    with pytest.raises(KeyError, match="client went away"):
        with GptEngine(lambda requests: GatedStub(2, requests, fail_at_decode=1), 8) as eng:
            job = eng.submit(_req(100))
            gate.set()
            with pytest.raises(_lib.CtbError):
                job.result(timeout=10)
            raise KeyError("client went away")
    assert not eng._thread.is_alive()


def test_chat_engine_checks_the_speech_stage_limit_at_submit():
    import types

    from chattts_b200 import Chat
    from chattts_b200.core import ChatEngine

    chat = types.SimpleNamespace(decoder=None, dvae=None)  # the check comes before any model is used
    eng = ChatEngine(lambda requests: OnlineStub(2, requests), 8, None, None, None, chat, True, max_new_cap=100)
    try:
        with pytest.raises(ValueError, match="max_new_cap"):
            eng.submit("hello", params_infer_code=Chat.InferCodeParams(max_new_token=200), skip_refine_text=False)
    finally:
        eng.close()


def test_a_cancel_at_a_poll_that_crosses_stream_boundaries_ends_the_job_once():
    """stream_batch 2 and 4-step chunks: every poll crosses boundaries, so the poll that stops a cancelled request also
    yields its boundaries.  Those are ordinary yields; the job ends once, cancelled, with what it has (a second end
    would fail the worker, and close would raise it)."""
    def req():
        return Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=2000, manual_seed=1,
                       stream_batch=2)

    with GptEngine(lambda requests: SlowStub(2, requests), 4) as eng:
        streamed, plain = eng.submit(req(), stream=True), eng.submit(req())
        it = iter(streamed)
        next(it)
        streamed.cancel()
        plain.cancel()
        rest = [(int(o.ids[0].shape[0]), last) for o, last in it]
        assert not any(last for _, last in rest) and all(n % 2 == 0 for n, _ in rest), rest
        for job in (streamed, plain):
            out = job.result(timeout=10)
            assert job.cancelled() and out.cancelled and 0 < int(out.ids[0].shape[0]) < 2000
