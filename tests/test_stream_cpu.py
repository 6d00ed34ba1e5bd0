"""Streaming on the slot engine without a GPU: the per-request yield reconstruction of engine.stream_schedule against a
replay of the static streaming loop (GPT.generate(stream=True)), the Chat windowing (StreamWindows) against a replay of
the static hand-off, the shared scheduling policy against a stub device, and the rejected modes."""
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.core import StreamWindows
from chattts_b200.engine import Request, ScheduleStats, SlotStatus, stream_schedule


class StreamStub:
    """Slot device whose request i samples `length` tokens and then EOS (eos=True), or runs to its max_new_token."""

    def __init__(self, slots, requests, specs):
        self.slots, self.requests, self.specs = slots, requests, specs
        self.req = [None] * slots
        self.steps_in = [0] * slots
        self.admissions = []
        self.steps = 0
        self.draws = {}

    def _spec(self, i):
        spec = self.specs[i]
        if isinstance(spec, list):  # one (length, eos) per admission (a requeued request draws again)
            spec = spec[self.draws[i] - 1]
        return spec

    def admit(self, batch):
        self.admissions.append(list(batch))
        for s, i in batch:
            assert self.req[s] is None or self._finished(s)
            self.draws[i] = self.draws.get(i, 0) + 1
            self.req[s], self.steps_in[s] = (i, self._spec(i)), 1

    def _finished(self, s):
        i, (length, eos) = self.req[s]
        return (eos and self.steps_in[s] >= length + 1) or self.steps_in[s] >= self.requests[i].max_new_token

    def decode(self, n):
        if any(r is not None and not self._finished(s) for s, r in enumerate(self.req)):
            self.steps += n
        for s, r in enumerate(self.req):
            if r is None or self._finished(s):
                continue
            i, (length, eos) = r
            limit = min(length + 1, self.requests[i].max_new_token) if eos else self.requests[i].max_new_token
            self.steps_in[s] = min(self.steps_in[s] + n, limit)

    def status(self):
        state, end, fin = [], [], []
        for s, r in enumerate(self.req):
            if r is None:
                state.append(_lib.SLOT_IDLE), end.append(0), fin.append(0)
                continue
            i, (length, eos) = r
            done = self._finished(s)
            at_eos = done and eos and self.steps_in[s] >= length + 1
            state.append(_lib.SLOT_FINISHED if done else _lib.SLOT_RUNNING)
            end.append(length if at_eos else self.steps_in[s])
            fin.append(1 if at_eos else 0)
        return SlotStatus(state, end, fin, self.steps)


def static_yields(length, eos, max_new, sb):
    """(n_tokens, last) of GPT.generate(stream=True, stream_batch=sb) for one row, replaying its loop step by step:
    the row samples `length` tokens, then EOS (eos=True) or nothing until max_new."""
    finish_step = length + 1 if eos else None
    if finish_step == 1:
        return []  # first-step EOS of a seeded request: the static generator returns without a yield
    steps, finished, out = 1, False, []
    while not finished and steps < max_new:
        target = steps + min(sb - steps % sb, max_new - steps)
        if finish_step is not None and finish_step <= target:
            steps, finished = finish_step, True
        else:
            steps = target
        if not finished and steps % sb == 0:
            out.append((steps, False))
    if finished and steps - 1 > 0 and (steps - 1) % sb == 0:
        out.append((steps - 1, False))
    out.append((steps - 1 if finished else steps, True))
    return out


def _reqs(max_new, sb, seeded=True):
    return [Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=m, stream_batch=b,
                    manual_seed=i if seeded else None) for i, (m, b) in enumerate(zip(max_new, sb))]


def _run(specs, max_new, sb, slots, chunk, context=None, seeded=True, stats=None):
    reqs = _reqs(max_new, sb, seeded)
    dev = StreamStub(slots, reqs, specs)
    got = {i: [] for i in range(len(reqs))}
    polls = list(stream_schedule(reqs, dev, chunk, context, stats))
    for batch in polls:
        for i, s, n, last in batch:
            got[i].append((n, last))
    return got, dev, polls


def test_hand_worked_yields():
    # stream_batch 24: EOS after 48 tokens (step 49 = 24k + 1) repeats the 48 boundary; max_new 48 does not
    assert static_yields(48, True, 200, 24) == [(24, False), (48, False), (48, False), (48, True)]
    assert static_yields(48, False, 48, 24) == [(24, False), (48, False), (48, True)]
    assert static_yields(47, True, 200, 24) == [(24, False), (47, True)]
    assert static_yields(30, True, 200, 16) == [(16, False), (30, True)]
    assert static_yields(0, True, 100, 24) == []
    got, _, _ = _run([(48, True), (48, False), (47, True)], [200, 48, 200], [24, 24, 24], 3, 32)
    assert got[0] == [(24, False), (48, False), (48, False), (48, True)]
    assert got[1] == [(24, False), (48, False), (48, True)]
    assert got[2] == [(24, False), (47, True)]


SPECS = [(48, True), (72, False), (23, True), (24, True), (25, True), (16, True), (33, True), (95, False), (1, True),
         (0, True), (64, False), (2, False), (1, False), (47, False), (96, True), (17, True)]
MAX_NEW = [200, 72, 200, 200, 200, 200, 200, 95, 200, 200, 64, 2, 1, 47, 200, 18]


@pytest.mark.parametrize("chunk", [8, 24, 32])
@pytest.mark.parametrize("sb", [16, 24])
@pytest.mark.parametrize("slots", [2, 5])
def test_reconstruction_equals_the_static_loop_whatever_the_poll(chunk, sb, slots):
    got, _, _ = _run(SPECS, MAX_NEW, [sb] * len(SPECS), slots, chunk)
    for i, (length, eos) in enumerate(SPECS):
        ref = static_yields(length, eos, MAX_NEW[i], sb)
        if not ref:  # a seeded first-step EOS: one empty final output
            ref = [(0, True)]
        assert got[i] == ref, (i, got[i], ref)


def test_mixed_stream_batches_in_one_engine():
    sbs = [16, 24, 16, 24, 5, 1, 24, 16]
    specs = [(48, True), (72, False), (32, True), (24, True), (30, True), (6, True), (49, True), (17, False)]
    max_new = [200, 72, 200, 200, 200, 200, 200, 17]
    got, _, _ = _run(specs, max_new, sbs, 3, 7)
    for i, (length, eos) in enumerate(specs):
        assert got[i] == static_yields(length, eos, max_new[i], sbs[i]), i


def test_max_new_exactly_on_a_boundary():
    got, _, _ = _run([(200, False), (200, False)], [48, 72], [24, 24], 2, 32)
    assert got[0] == [(24, False), (48, False), (48, True)]
    assert got[1] == [(24, False), (48, False), (72, False), (72, True)]


def test_first_step_eos_seeded_ends_empty_unseeded_runs_again():
    got, _, _ = _run([(0, True), (30, True)], [100, 100], [24, 24], 2, 8)
    assert got[0] == [(0, True)] and got[1] == [(24, False), (30, True)]
    stats = ScheduleStats()
    got, dev, _ = _run([[(0, True), (26, True)], (30, True)], [100, 100], [24, 24], 2, 8, seeded=False, stats=stats)
    assert got[0] == [(24, False), (26, True)] and got[1] == [(24, False), (30, True)]
    assert stats.requeued == 1 and dev.draws[0] == 2


def test_slot_reuse_waits_for_the_finished_requests_yields():
    """A poll's yields all refer to the slots as they were when it was read: the freed slot is refilled only after
    the generator is resumed past them."""
    specs = [(10, True), (40, True), (5, True), (25, True)]
    reqs = _reqs([100] * 4, [8] * 4)
    dev = StreamStub(2, reqs, specs)
    gen = stream_schedule(reqs, dev, 4)
    seen = {}
    for batch in gen:
        for i, s, n, last in batch:
            if s is not None:
                assert dev.req[s][0] == i  # the slot still holds this request
            seen.setdefault(i, []).append((n, last))
    assert [a for adm in dev.admissions for a in adm] == [(0, 0), (1, 1), (0, 2), (0, 3)]
    for i, (length, eos) in enumerate(specs):
        assert seen[i] == static_yields(length, eos, 100, 8)


def test_interrupt_ends_running_requests_and_drops_waiting_ones():
    from chattts_b200.gpt import GPT

    ctx = GPT.Context()
    reqs = _reqs([100] * 3, [8] * 3)
    dev = StreamStub(2, reqs, [(90, True)] * 3)
    gen = stream_schedule(reqs, dev, 12, context=ctx)
    first = next(gen)  # poll after the first chunk: boundary 8 of both running requests
    assert first == [] or all(not last for *_, last in first)
    ctx.set(True)
    rest = [e for batch in gen for e in batch]
    finals = [(i, n) for i, _, n, last in rest if last]
    assert sorted(i for i, _ in finals) == [0, 1]
    assert all(not last for i, _, _, last in rest[: len(rest) - 2])  # the final yields close the stream
    assert 2 not in {i for i, *_ in rest}


def windows_replay(yield_tokens, speed, skip):
    """core.py:304-338 for one row: the (a, b) of every chunk, the flush last."""
    length, count, out = 0, 0, []
    for n in yield_tokens:
        count += 1
        total = 512 * n - 256
        if count <= skip:
            continue
        a, b = length, min(length + speed, total)
        length = b
        out.append((a, b, False))
    out.append((length, 512 * yield_tokens[-1] - 256, True))
    return out


@pytest.mark.parametrize("skip", [0, 2])
@pytest.mark.parametrize("speed", [6000, 12000, 30000])
@pytest.mark.parametrize("spec", [(48, True, 24), (72, False, 24), (150, True, 16), (16, True, 16), (3, True, 24)])
def test_windows_equal_the_static_hand_off(skip, speed, spec):
    length, eos, sb = spec
    ys = static_yields(length, eos, 200 if eos else length, sb)
    w = StreamWindows(speed, skip)
    got = [x for n, last in ys for x in w.windows(n, last)]
    assert got == windows_replay([n for n, _ in ys], speed, skip)


def test_windows_include_empty_ones():
    # a fast stream_speed catches up with the tokens: the later windows are empty and are still yielded
    w = StreamWindows(100000, 0)
    got = [x for n, last in [(24, False), (48, False), (48, False), (48, True)] for x in w.windows(n, last)]
    assert got == [(0, 512 * 24 - 256, False), (512 * 24 - 256, 512 * 48 - 256, False),
                   (512 * 48 - 256, 512 * 48 - 256, False), (512 * 48 - 256, 512 * 48 - 256, False),
                   (512 * 48 - 256, 512 * 48 - 256, True)]
    assert StreamWindows(6000, 2).windows(0, True) == [(0, 0, True)]


@pytest.mark.parametrize("kw", [dict(infer_text=True), dict(return_attn=True)])
def test_generate_continuous_stream_rejects_unsupported_modes(kw):
    from chattts_b200.config import Config
    from chattts_b200.gpt import GPT

    gpt = GPT(Config().gpt, embed=None)
    with pytest.raises(ValueError):
        next(gpt.generate_continuous_stream(_reqs([10, 10], [24, 24]), **kw))


def test_infer_continuous_stream_rejects_misaligned_params():
    from chattts_b200 import Chat

    with pytest.raises(ValueError):
        Chat().infer_continuous_stream(["a", "b"], params_infer_code=[Chat.InferCodeParams()])


def test_request_stream_batch_default_and_validation():
    assert Request(emb=torch.zeros(3, 4), temperature=[0.3], eos_token=625).stream_batch == 24
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(3, 4), temperature=[0.3], eos_token=625, stream_batch=0)
