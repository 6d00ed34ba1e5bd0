"""Token log-probabilities without a GPU: the engine's device layer is made exactly as before when they are off, the
host side carries a suspended request's rows (``SlotImage``) and harvests them, and ``Job.logprobs`` of
``Chat.open_engine(logprobs=True)`` has its documented shape for every kind of job (on the stand-ins of
``test_paragraph_refine_cpu``)."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from chattts_b200 import _lib, engine
from chattts_b200.engine import EngineDevice, SlotImage
from chattts_b200.gpt import GPT
from test_paragraph_refine_cpu import PARA, SENTENCES, ChatEngine, _chat, _FakeChat, _params, _Stub


# ---------------------------------------------------------------------------------------------------- device layer
@pytest.mark.parametrize("pool,flags", [(None, 0), (None, 3), (40, 0)])
def test_logprobs_off_makes_the_device_layer_as_before(monkeypatch, pool, flags):
    calls = []
    monkeypatch.setattr(engine, "EngineDevice", lambda *a, **kw: calls.append((a, kw)))
    gpt = SimpleNamespace()
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool)
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool, False)
    before = ((gpt, [], 4, 90, True), {} if pool is None and not flags else
              {"flags": flags, "kv_pool_pages": pool} if pool is not None else {"flags": flags})
    assert calls == [before, before]
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool, True)
    assert calls[-1] == ((gpt, [], 4, 90, True), {"flags": flags, "kv_pool_pages": pool, "logprobs": True})


def _host_device(text, slots=2, cap=8, num_vq=4, hidden=6, logprobs=True):
    """An EngineDevice's host side over CPU buffers: what harvest, empty and SlotImage read."""
    dev = EngineDevice.__new__(EngineDevice)
    dev.gpt = SimpleNamespace(num_vq=num_vq, config=SimpleNamespace(hidden_size=hidden))
    dev.dev = torch.device("cpu")
    dev.requests = [SimpleNamespace(infer_text=text)]
    dev.ids_out = torch.arange(slots * cap * num_vq, dtype=torch.int32).view(slots, cap, num_vq)
    dev.hid_out = torch.randn(slots, cap, hidden)
    dev.lp_out = -torch.rand(slots, cap, num_vq) if logprobs else None
    dev._text = [text] * slots
    dev._images = {}
    return dev


def _image(dev, slot, n):
    """The SlotImage a suspend of ``slot`` with ``n`` tokens leaves (its header, ids and hidden sections, and the rows
    EngineDevice.suspend copies beside it), as host memory."""
    num_vq, d = dev.gpt.num_vq, dev.gpt.config.hidden_size
    off_ids = C.sizeof(_lib.SlotImage)
    off_hid = off_ids + 4 * n * num_vq
    buf = torch.zeros(off_hid + 4 * n * d + 256, dtype=torch.uint8)
    h = _lib.SlotImage.from_address(buf.data_ptr())
    h.n_gen, h.off_ids, h.off_hiddens = n, off_ids, off_hid
    buf[off_ids: off_ids + 4 * n * num_vq] = dev.ids_out[slot, :n].contiguous().view(torch.uint8).view(-1)
    buf[off_hid: off_hid + 4 * n * d] = dev.hid_out[slot, :n].contiguous().view(torch.uint8).view(-1)
    im = SlotImage.__new__(SlotImage)
    im.buf, im.text, im.device, im.num_vq, im.hidden_size = buf, dev._text[slot], dev.dev, num_vq, d
    im.ready = SimpleNamespace(synchronize=lambda: None)
    im.header = h
    im.logprobs = dev.lp_out[slot, :n].clone() if dev.lp_out is not None else None
    return im


@pytest.mark.parametrize("text", [False, True])
def test_harvest_and_a_suspended_image_carry_the_rows(text):
    dev = _host_device(text)
    n = 5
    out = dev.harvest(1, n)
    want = dev.lp_out[1, :n, 0] if text else dev.lp_out[1, :n]
    assert len(out.logprobs) == 1 and torch.equal(out.logprobs[0], want)
    assert out.logprobs[0].shape == out.ids[0].shape
    im = _image(dev, 1, n)
    for k in (n, 3):  # a cancelled suspended request ends with the first k tokens of its image
        got = dev.harvest(im, k)
        assert torch.equal(got.ids[0], out.ids[0][:k]) and torch.equal(got.logprobs[0], want[:k])
    empty = dev.empty(0)
    assert empty.logprobs[0].shape == empty.ids[0].shape == ((0,) if text else (0, 4))
    off = _host_device(text, logprobs=False)
    assert off.harvest(1, n).logprobs == [] and off.empty(0).logprobs == []
    assert off.harvest(_image(off, 1, n), n).logprobs == []


def test_generation_outputs_default_to_no_logprobs():
    out = GPT.GenerationOutputs(ids=[], attentions=[], hiddens=[])
    assert out.logprobs == [] and not out.cancelled


# ---------------------------------------------------------------------------------------------------- Job.logprobs
class _TakesChat(_FakeChat):
    """_FakeChat whose takes (requests replaced from one code request) yield 5 + 3 k tokens, k the take."""

    def length(self, r):
        if r.prompt_key is not None:
            return 5 + 3 * r.noise_batch[1]
        return super().length(r)


class _LpStub(_Stub):
    """_Stub with a log-probability buffer: harvests carry rows of their token counts."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.lp_out = torch.zeros(self.slots, 256, 4)

    def harvest(self, slot, n, copy=True):
        out = super().harvest(slot, n, copy)
        out.logprobs = [-torch.arange(1, n + 1, dtype=torch.float32)[:, None].expand(n, 4).contiguous()]
        return out


def _open(chat, logprobs):
    devs = []

    def make(requests):
        devs.append((_LpStub if logprobs else _Stub)(4, requests, chat, lambda r: None))
        return devs[-1]

    return ChatEngine(make, 8, None, None, None, chat, False, max_new_cap=200), devs


def test_job_logprobs_for_every_kind_of_job():
    chat = _TakesChat(dict(zip(SENTENCES, (9, 9, 25, 41, 17))), dict(zip(SENTENCES, (9, 17, 25, 9, 33))))
    chat.code_len["one"] = 21
    p, r = _params()
    eng, _ = _open(chat, True)
    with eng:
        one = eng.submit("one", params_infer_code=p)
        takes = eng.submit("one", params_infer_code=p, takes=3)
        split = eng.submit(PARA, params_infer_code=p, split_text=True)
        refined = eng.submit(PARA, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r)
        for j in (one, takes, split, refined):
            j.result(timeout=30)
    assert isinstance(one.logprobs, torch.Tensor) and one.logprobs.shape == (21, 4)
    assert [t.shape for t in takes.logprobs] == [(5, 4), (8, 4), (11, 4)]  # take order
    for job in (split, refined):  # one row per sentence, in sentence order; no reference stage, no refinement
        assert [t.shape[0] for t in job.logprobs] == [chat.code_len[s] for s in SENTENCES]
        assert all(t.device.type == "cpu" for t in job.logprobs)


def test_without_logprobs_jobs_have_none_and_harvest_as_before():
    counts = []
    for logprobs in (False, True):
        chat = _chat()
        eng, devs = _open(chat, logprobs)
        with eng:
            job = eng.submit(PARA, params_infer_code=_params()[0], split_text=True)
            job.result(timeout=30)
        assert (job.logprobs is None) == (not logprobs)
        counts.append([d.decodes for d in devs])
    assert counts[0] == counts[1]
