"""Text requests and follow-ups on the slot engine without a GPU: the follow-up policy of engine._poll_cycles against a
stub device (admission at the same poll ahead of the waiting requests, index mapping, no follow-up after a requeue or
an interrupt, an empty seeded text stage), stream reconstruction with text requests, and Request validation."""
import pytest
import torch

from chattts_b200.engine import Request, ScheduleStats, schedule, stream_schedule
from test_continuous_cpu import StubDevice
from test_stream_cpu import StreamStub, static_yields


class HarvestStub(StubDevice):
    """StubDevice whose outputs can be harvested: slot s's request i produced ids 0..n-1 (1-D for a text request)."""

    def __init__(self, slots, lengths, requests):
        super().__init__(slots, lengths)
        self.requests = requests
        self.harvested = []

    def harvest(self, slot, n):
        i = self.req[slot][0]
        self.harvested.append((i, slot, n))
        ids = torch.arange(n) if self.requests[i].infer_text else torch.arange(n)[:, None].repeat(1, 4)
        return ("out", i, ids)

    def empty(self, index):
        self.harvested.append((index, None, 0))
        return ("out", index, torch.zeros(0, dtype=torch.long))


def _text(seed=0, max_new=100, then=None):
    return Request(emb=torch.zeros(5, 4), temperature=[0.7], eos_token=21001, max_new_token=max_new, manual_seed=seed,
                   infer_text=True, then=then)


def _code(seed=0, max_new=100):
    return Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=max_new, manual_seed=seed)


def test_follow_up_is_admitted_at_the_same_poll_ahead_of_waiting_requests():
    seen = []

    def then(out):
        seen.append(out)
        return _code(seed=50)

    # request 0 (text, 6 tokens) ends in the first chunk; requests 2 and 3 wait; its follow-up (index 4) goes first
    reqs = [_text(then=then), _code(1), _code(2), _code(3)]
    lengths = [6, 30, 8, 9, 20]
    dev = HarvestStub(2, lengths, reqs)
    stats = ScheduleStats()
    out = list(schedule(reqs, dev, 8, stats=stats))
    assert dev.admissions[0] == [(0, 0), (1, 1)]
    assert dev.admissions[1] == [(0, 4)]  # same poll the text stage ended at, its own (lowest free) slot
    assert seen[0][1] == 0 and torch.equal(seen[0][2], torch.arange(6))
    assert stats.children == {0: 4} and len(reqs) == 5
    assert sorted(i for i, _, _ in out) == [0, 1, 2, 3, 4]
    assert all(n == lengths[i] for i, _, n in out)


def test_follow_ups_keep_slot_order_and_chain():
    # two text stages end at the same poll: their follow-ups take slots 0 and 1 in that order, before request 2;
    # a follow-up may itself have a follow-up
    reqs = [_text(then=lambda o: _code(10)), _text(then=lambda o: _text(then=lambda o2: _code(11))), _code(2)]
    dev = HarvestStub(2, [4, 5, 7, 3, 6, 9], reqs)
    stats = ScheduleStats()
    list(schedule(reqs, dev, 8, stats=stats))
    assert dev.admissions[1] == [(0, 3), (1, 4)]
    assert stats.children == {0: 3, 1: 4, 4: 5}
    assert [a for adm in dev.admissions for a in adm][-2:] in ([(0, 2), (1, 5)], [(0, 5), (1, 2)])


def test_no_follow_up_after_a_requeue_or_an_interrupt():
    from chattts_b200.gpt import GPT

    calls = []
    # unseeded text stage whose first draw is EOS: queued again, and only its second run calls `then`
    reqs = [Request(emb=torch.zeros(5, 4), temperature=[0.7], eos_token=21001, max_new_token=50, infer_text=True,
                    then=lambda o: calls.append(o) or None), _code(1)]
    dev = HarvestStub(2, [[0, 9], 7], reqs)
    stats = ScheduleStats()
    list(schedule(reqs, dev, 4, stats=stats))
    assert stats.requeued == 1 and len(calls) == 1 and calls[0][2].shape == (9,)
    assert stats.children == {}

    calls.clear()
    ctx = GPT.Context()
    reqs = [_text(then=lambda o: calls.append(o) or _code()), _text(then=lambda o: calls.append(o) or _code())]
    dev = HarvestStub(2, [100, 100], reqs)
    gen = schedule(reqs, dev, 8, context=ctx)
    ctx.set(True)
    out = list(gen)
    assert sorted(i for i, _, _ in out) == [0, 1] and calls == [] and len(reqs) == 2


def test_empty_seeded_text_stage_still_calls_then():
    calls = []
    reqs = [_text(seed=3, then=lambda o: calls.append(o) or _code(9)), _code(1)]
    dev = HarvestStub(2, [0, 12, 5], reqs)
    out = list(schedule(reqs, dev, 4))
    assert (0, None, 0) in out
    assert calls[0][1] == 0 and calls[0][2].numel() == 0
    assert (2, 0, 5) in out


def test_follow_up_breaking_a_check_raises():
    def check(r):
        if r.max_new_token > 64:
            raise ValueError("max_new_token exceeds max_new_cap")

    reqs = [_text(max_new=32, then=lambda o: _code(max_new=128)), _code(1, max_new=40)]
    dev = HarvestStub(2, [5, 30, 9], reqs)
    with pytest.raises(ValueError):
        list(schedule(reqs, dev, 8, check=check))


class TextStreamStub(StreamStub):
    """StreamStub whose request behaviour is keyed by its manual_seed, so follow-ups need no index known in advance."""

    def _spec(self, i):
        return self.specs[self.requests[i].manual_seed]

    def harvest(self, slot, n):
        return ("out", self.req[slot][0], n)

    def empty(self, index):
        return ("out", index, 0)


SPECS = [(48, True), (30, True), (23, False), (72, False), (0, True), (40, True), (17, True), (25, True)]
MAX_NEW = [200, 200, 23, 72, 200, 200, 200, 200]
SBS = [24, 16, 24, 24, 16, 24, 16, 24]


def _mk(k, text, then=None):
    return Request(emb=torch.zeros(5, 4), temperature=[0.5], eos_token=1, max_new_token=MAX_NEW[k],
                   stream_batch=SBS[k], manual_seed=k, infer_text=text, then=then)


@pytest.mark.parametrize("chunk", [8, 24])
def test_stream_reconstruction_with_text_requests(chunk):
    """Text requests and their follow-ups stream exactly like code requests: the static loop is the same for both.
    Request 4 is a seeded text stage that ends empty; its follow-up still runs."""
    reqs = [_mk(0, True, lambda o: _mk(5, False, lambda o2: _mk(7, True))), _mk(1, False), _mk(2, True),
            _mk(3, False), _mk(4, True, lambda o: _mk(6, False))]
    dev = TextStreamStub(3, reqs, SPECS)
    stats = ScheduleStats()
    got = {}
    for batch in stream_schedule(reqs, dev, chunk, stats=stats):
        for i, s, n, last in batch:
            got.setdefault(i, []).append((n, last))
    assert len(reqs) == 8 and len(stats.children) == 3
    for i, r in enumerate(reqs):
        k = r.manual_seed
        length, eos = SPECS[k]
        ref = static_yields(length, eos, MAX_NEW[k], SBS[k]) or [(0, True)]
        assert got[i] == ref, (i, got[i], ref)


def test_text_request_validation():
    assert _text().infer_text and not _code().infer_text and _code().then is None
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(3, 4), temperature=[0.3, 0.3], eos_token=21001, infer_text=True)
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(3, 4), temperature=[0.3], eos_token=21001, infer_text=True, max_new_token=0)
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(2, 3, 4), temperature=[0.3], eos_token=21001, infer_text=True)
    Request(emb=torch.zeros(3, 4), temperature=0.7, eos_token=21001, infer_text=True)


def test_call_level_infer_text_points_at_the_request_field():
    from chattts_b200.config import Config
    from chattts_b200.gpt import GPT

    gpt = GPT(Config().gpt, embed=None)
    with pytest.raises(ValueError, match="Request.infer_text"):
        next(gpt.generate_continuous([_code(), _code()], infer_text=True))


def test_infer_continuous_rejects_misaligned_refine_params():
    from chattts_b200 import Chat

    with pytest.raises(ValueError):
        Chat().infer_continuous(["a", "b"], params_refine_text=[Chat.RefineTextParams()], skip_refine_text=False)
