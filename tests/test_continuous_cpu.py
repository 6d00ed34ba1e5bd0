"""Scheduling policy of the slot engine (chattts_b200.engine.schedule) against a stub device, and the input the engine
rejects.  No GPU needed."""
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import Request, ScheduleStats, SlotStatus, schedule


class StubDevice:
    """Slot b holds request i, which yields `lengths[i]` tokens (0: EOS as its first token)."""

    def __init__(self, slots, lengths):
        self.slots, self.lengths = slots, lengths
        self.req = [None] * slots
        self.done = [0] * slots
        self.state = [_lib.SLOT_IDLE] * slots
        self.admissions = []
        self.steps = 0
        self.draws = {}

    def admit(self, batch):
        self.admissions.append(list(batch))
        for s, i in batch:
            assert self.state[s] != _lib.SLOT_RUNNING
            n = self.draws.get(i, 0)
            self.draws[i] = n + 1
            length = self.lengths[i][n] if isinstance(self.lengths[i], list) else self.lengths[i]
            self.req[s], self.done[s] = (i, length), min(1, length)
            self.state[s] = _lib.SLOT_RUNNING if length > 1 else _lib.SLOT_FINISHED

    def decode(self, n):
        if any(st == _lib.SLOT_RUNNING for st in self.state):
            self.steps += n
        for s in range(self.slots):
            if self.state[s] == _lib.SLOT_RUNNING:
                self.done[s] = min(self.done[s] + n, self.req[s][1])
                if self.done[s] == self.req[s][1]:
                    self.state[s] = _lib.SLOT_FINISHED

    def status(self):
        fin = [1 if r is not None and r[1] == 0 else 0 for r in self.req]
        return SlotStatus(list(self.state), list(self.done), fin, self.steps)


def _reqs(n, seeded=True):
    return [Request(emb=torch.zeros(5, 4), temperature=[0.3], eos_token=625, max_new_token=100,
                    manual_seed=i if seeded else None) for i in range(n)]


def test_requests_fill_free_slots_in_order_and_slots_are_reused():
    lengths = [10, 40, 5, 25, 3, 12]
    dev = StubDevice(2, lengths)
    stats = ScheduleStats()
    out = list(schedule(_reqs(6), dev, 4, stats=stats))
    # both slots finish at step 40 of request 1 / request 3 (same chunk): yielded in slot order
    assert [i for i, _, _ in out] == [0, 2, 3, 1, 4, 5]
    assert all(n == lengths[i] for i, _, n in out)
    # a freed slot is refilled at the next poll, lowest free slot first
    assert dev.admissions == [[(0, 0), (1, 1)], [(0, 2)], [(0, 3)], [(0, 4), (1, 5)]]
    assert stats.admitted == 6 and stats.tokens == sum(lengths) and stats.decode_steps == dev.steps


def test_first_step_eos_seeded_ends_empty_unseeded_runs_again():
    dev = StubDevice(2, [0, 7])
    out = list(schedule(_reqs(2, seeded=True), dev, 4))
    assert (0, None, 0) in out and any(i == 1 and n == 7 for i, _, n in out)
    dev = StubDevice(2, [[0, 9], 7])
    stats = ScheduleStats()
    out = list(schedule(_reqs(2, seeded=False), dev, 4, stats=stats))
    assert sorted((i, n) for i, _, n in out) == [(0, 9), (1, 7)] and stats.requeued == 1


def test_interrupt_yields_running_requests_and_drops_waiting_ones():
    from chattts_b200.gpt import GPT

    ctx = GPT.Context()
    dev = StubDevice(2, [100, 100, 100])
    gen = schedule(_reqs(3), dev, 8, context=ctx)
    ctx.set(True)
    out = list(gen)
    assert sorted(i for i, _, _ in out) == [0, 1] and all(n == 1 for _, _, n in out)


@pytest.mark.parametrize("kw", [dict(infer_text=True), dict(stream=True), dict(return_attn=True)])
def test_generate_continuous_rejects_unsupported_modes(kw):
    from chattts_b200.config import Config
    from chattts_b200.gpt import GPT

    gpt = GPT(Config().gpt, embed=None)
    with pytest.raises(ValueError):
        next(gpt.generate_continuous(_reqs(2), **kw))


def test_infer_continuous_rejects_stream_and_misaligned_params():
    from chattts_b200 import Chat

    c = Chat()
    with pytest.raises(ValueError):
        c.infer_continuous(["a", "b"], stream=True)
    with pytest.raises(ValueError):
        c.infer_continuous(["a", "b"], params_infer_code=[Chat.InferCodeParams()])


def test_request_validation():
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(2, 3, 4), temperature=[0.3], eos_token=625)
    with pytest.raises(ValueError):
        Request(emb=torch.zeros(3, 4), temperature=[0.3], eos_token=625, max_new_token=0)
