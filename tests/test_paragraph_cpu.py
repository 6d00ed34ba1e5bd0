"""Split-text synthesis without a GPU: fan-out follow-ups and the per-poll ``prepare`` hook in the scheduling policy
(engine._poll_cycles against a stub device), cancelling every live stage of a submission, a failing child, the
in-order assembly of a paragraph's audio and the sentence split ``infer`` uses."""
import re

import numpy as np
import pytest

from chattts_b200.core import _Paragraph, split_sentences
from chattts_b200.engine import Arrivals, ScheduleStats, _poll_cycles
from test_online_cpu import OnlineStub, _drain, _req


def _run(requests, src, slots=2, check=None, chunk=8):
    stats = ScheduleStats()
    dev = OnlineStub(slots, requests)
    gen = _poll_cycles(requests, dev, chunk, stats=stats, source=src, check=check)
    return dev, stats, gen


def test_a_fan_out_is_queued_ahead_of_waiting_requests_in_order():
    requests, src = [], Arrivals()
    kids = [_req(5, seed=1), _req(6, seed=2), _req(7, seed=3)]
    r0 = _req(4, then=lambda out: kids)
    for r in (r0, _req(40), _req(8), _req(9)):
        src.submit(r)
    dev, stats, gen = _run(requests, src)
    next(gen)
    _, _, ended = next(gen)
    assert ended == [(0, 0, 4, False)] and stats.fanout == {0: [4, 5, 6]} and stats.children == {}
    assert [requests[i] for i in stats.fanout[0]] == kids
    _drain(gen, src)
    order = [i for batch in dev.admissions for _, i in batch]
    assert order == [0, 1, 4, 5, 6, 2, 3]


def test_a_single_follow_up_keeps_its_children_entry():
    requests, src = [], Arrivals()
    child = _req(5, seed=1)
    src.submit(_req(4, then=lambda out: child))
    src.submit(_req(30))
    dev, stats, gen = _run(requests, src)
    next(gen)
    next(gen)
    assert stats.children == {0: 2} and stats.fanout == {}
    _drain(gen, src)


def test_prepare_runs_once_per_poll_before_the_thens():
    requests, src = [], Arrivals()
    log = []

    def prepare(dev, items):
        log.append(("prepare", [(requests.index(r), s, n) for r, s, n in items]))

    def then(tag):
        return lambda out: log.append(("then", tag))

    for k in range(3):
        r = _req(4, then=then(k))
        r.prepare = prepare
        src.submit(r)
    src.submit(_req(4, then=then("plain")))  # no prepare: its then alone
    dev, stats, gen = _run(requests, src, slots=4)
    _drain(gen, src)
    assert log == [("prepare", [(0, 0, 4), (1, 1, 4), (2, 2, 4)]), ("then", 0), ("then", 1), ("then", 2),
                   ("then", "plain")]


def test_a_failing_prepare_fails_its_requests_only():
    requests, src = [], Arrivals()
    boom = ValueError("no sample")

    def prepare(dev, items):
        raise boom

    r = _req(4, then=lambda out: _req(3))
    r.prepare = prepare
    src.submit(r)
    src.submit(_req(4, then=lambda out: _req(3, seed=5)))
    dev, stats, gen = _run(requests, src)
    ended = _drain(gen, src)
    assert stats.failed == {0: boom} and stats.children == {1: 2}
    assert sorted(i for i, *_ in ended) == [0, 1, 2]


def _paragraph(key_src, n_sentences, length=6, stage0=4):
    """A paragraph submission: a reference stage whose then fans out to one request per sentence."""
    kids = [_req(length + k, seed=10 + k) for k in range(n_sentences)]
    return _req(stage0, then=lambda out: kids), kids


def test_cancel_during_stage_zero_cancels_the_paragraph_only():
    requests, src = [], Arrivals()
    para, kids = _paragraph(src, 3, stage0=30)
    other = _req(20)
    src.submit(para)
    src.submit(other)
    dev, stats, gen = _run(requests, src)
    next(gen)
    src.cancel(para)
    _, _, ended = next(gen)
    assert ended == [(0, 0, 9, False)] and stats.cancelled == {0} and stats.fanout == {}
    rest = _drain(gen, src)
    assert [(i, n) for i, _, n, _ in rest] == [(1, 20)] and not any(k in requests for k in kids)


def test_cancel_during_the_sentences_cancels_every_live_stage():
    requests, src = [], Arrivals()
    para, kids = _paragraph(src, 3, length=40)
    other = _req(60)
    src.submit(para)
    src.submit(other)
    dev, stats, gen = _run(requests, src)
    next(gen)
    next(gen)  # stage 0 ends: sentence 0 takes its slot, sentences 1 and 2 wait
    assert stats.fanout == {0: [2, 3, 4]}
    next(gen)
    src.cancel(para)
    _, _, ended = next(gen)
    assert sorted(i for i, *_ in ended) == [2, 3, 4] and stats.cancelled == {2, 3, 4}
    assert dev.cancels == [[0]]  # the running sentence is stopped; the waiting ones never touch a slot
    rest = _drain(gen, src)
    assert [(i, n) for i, _, n, _ in rest] == [(1, 60)]
    assert all(i in (0, 1, 2) for batch in dev.admissions for _, i in batch)


def test_a_child_that_fails_its_check_fails_only_its_job():
    requests, src = [], Arrivals()
    bad = _req(500, seed=1)

    def check(r):
        if r.max_new_token > 100:
            raise ValueError("too long")

    para = _req(4, then=lambda out: [_req(5, seed=2), bad])
    src.submit(para)
    src.submit(_req(6, then=lambda out: _req(7, seed=3)))
    dev, stats, gen = _run(requests, src, check=check)
    ended = _drain(gen, src)
    assert isinstance(stats.failed[0], ValueError) and stats.fanout == {} and stats.children == {1: 2}
    assert sorted((i, n) for i, _, n, _ in ended) == [(0, 4), (1, 6), (2, 7)]


class _FakeJob:
    def __init__(self):
        self.items, self.result = [], None

    def _put(self, item):
        self.items.append(item)

    def _finish(self, value):
        self.result = value


class _P:
    stream_speed, pass_first_n_batches = 6000, 0


def test_streamed_sentences_are_delivered_in_order():
    p = _Paragraph(3, _P())
    p.job = _FakeJob()
    c = [np.full((1, 2), float(k), np.float32) for k in range(8)]
    p.add(1, c[0], False)          # sentence 1 is held until sentence 0's final chunk
    p.add(2, c[1], True)
    assert p.job.items == []
    p.add(0, c[2], False)
    assert [x[0, 0] for x, _ in p.job.items] == [2.0]
    p.add(0, c[3], True)           # sentence 0 done: sentence 1's held chunk follows
    assert [x[0, 0] for x, _ in p.job.items] == [2.0, 3.0, 0.0] and not any(l for _, l in p.job.items)
    p.add(1, c[4], True)           # sentence 1 done: sentence 2 (already complete) follows, and only its end is last
    assert [x[0, 0] for x, _ in p.job.items] == [2.0, 3.0, 0.0, 4.0, 1.0]
    assert [l for _, l in p.job.items] == [False] * 4 + [True]


def test_whole_waveforms_are_concatenated_in_sentence_order():
    p = _Paragraph(3, None)
    p.job = _FakeJob()
    p.add(2, np.array([[5.0]], np.float32), True)
    p.add(0, np.array([[1.0, 2.0]], np.float32), True)
    assert p.job.result is None
    p.add(1, np.zeros((1, 0), np.float32), True)
    assert p.job.result.tolist() == [1.0, 2.0, 5.0]


def _old_rule(text):  # the split infer() has always made (reference core.py:237-241)
    if "\n" in text:
        return text.split("\n")
    return [t for t in re.split(r"(?<=。)|(?<=\.\s)", text) if t]


@pytest.mark.parametrize("text", ["one sentence", "a. b. c", "a.b. c", "end. ", "一。二。三", "x\ny. z", "\n", "",
                                  "first. second.\tthird. fourth", "trailing newline\n"])
def test_split_sentences_is_infer_s_rule(text):
    assert split_sentences(text) == _old_rule(text)
