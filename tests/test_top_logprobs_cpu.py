"""Top log-probabilities without a GPU: ``top_logprobs`` is checked before anything is built, the engine's device layer
is made exactly as before when it is off, the host side harvests the (ids, lp) rows, carries a suspended request's rows
(``SlotImage``) and hands streamed yields copies, ``Job.top_logprobs`` of ``Chat.open_engine(top_logprobs=N)`` has its
documented structure (on the stand-ins of ``test_paragraph_refine_cpu``), and ``GPT.score`` returns what it returned
before unless N > 0 (on the stand-in library of ``test_score_cpu``)."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from chattts_b200 import engine
from chattts_b200.engine import TOP_LOGPROBS_MAX, EngineDevice, check_top_logprobs
from chattts_b200.gpt import GPT
from test_logprobs_cpu import _host_device, _image, _TakesChat, _LpStub
from test_paragraph_refine_cpu import PARA, SENTENCES, ChatEngine, _chat, _params, _Stub
from test_score_cpu import NVQ, FakeLib, _codes, _prompt, fake  # noqa: F401 (fixture)

N = 3


# ---------------------------------------------------------------------------------------------------- arguments
@pytest.mark.parametrize("bad", [-1, 21, 2.0, 5.5, "3", True, None])
def test_bad_top_logprobs_are_value_errors(bad):
    with pytest.raises(ValueError, match="top_logprobs"):
        check_top_logprobs(bad)


def test_good_top_logprobs():
    assert [check_top_logprobs(n) for n in (0, 1, 20)] == [0, 1, 20] and TOP_LOGPROBS_MAX == 20


@pytest.mark.parametrize("bad", [21, 1.0])
def test_entry_points_refuse_before_touching_the_handle(bad):
    g = GPT.__new__(GPT)  # no handle, no weights: the check comes first
    with pytest.raises(ValueError, match="top_logprobs"):
        g.open_engine(4, 90, top_logprobs=bad)
    with pytest.raises(ValueError, match="top_logprobs"):
        next(g.generate_continuous([], top_logprobs=bad))
    with pytest.raises(ValueError, match="top_logprobs"):
        next(g.generate_continuous_stream([], top_logprobs=bad))
    with pytest.raises(ValueError, match="top_logprobs"):
        g.score([], [], top_logprobs=bad)


# ---------------------------------------------------------------------------------------------------- device layer
@pytest.mark.parametrize("pool,flags", [(None, 0), (None, 3), (40, 0)])
def test_top_logprobs_off_makes_the_device_layer_as_before(monkeypatch, pool, flags):
    calls = []
    monkeypatch.setattr(engine, "EngineDevice", lambda *a, **kw: calls.append((a, kw)))
    gpt = SimpleNamespace()
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool)
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool, False, 0)
    before = ((gpt, [], 4, 90, True), {} if pool is None and not flags else
              {"flags": flags, "kv_pool_pages": pool} if pool is not None else {"flags": flags})
    assert calls == [before, before]
    GPT._engine_device(gpt, [], 4, 90, True, flags, pool, True, 0)
    assert calls[-1] == ((gpt, [], 4, 90, True), {"flags": flags, "kv_pool_pages": pool, "logprobs": True})
    for lp in (False, True):
        GPT._engine_device(gpt, [], 4, 90, True, flags, pool, lp, 5)
        assert calls[-1] == ((gpt, [], 4, 90, True),
                             {"flags": flags, "kv_pool_pages": pool, "logprobs": lp, "top_logprobs": 5})


def _top_device(text, slots=2, cap=8, num_vq=4, logprobs=True):
    """_host_device with the two top buffers of an engine opened with top_logprobs=N."""
    dev = _host_device(text, slots, cap, num_vq, logprobs=logprobs)
    dev.top_ids_out = torch.randint(0, 626, (slots, cap, num_vq, N), dtype=torch.int32)
    dev.top_lp_out = -torch.rand(slots, cap, num_vq, N)
    return dev


def _top_image(dev, slot, n):
    im = _image(dev, slot, n)
    im.top = (dev.top_ids_out[slot, :n].clone(), dev.top_lp_out[slot, :n].clone())
    return im


@pytest.mark.parametrize("text", [False, True])
def test_harvest_shapes_and_a_suspended_image_carry_the_rows(text):
    dev = _top_device(text)
    n = 5
    out = dev.harvest(1, n)
    (ids, lp), = out.top_logprobs
    want_ids = dev.top_ids_out[1, :n, 0] if text else dev.top_ids_out[1, :n]
    want_lp = dev.top_lp_out[1, :n, 0] if text else dev.top_lp_out[1, :n]
    assert ids.dtype == torch.int64 and lp.dtype == torch.float32
    assert ids.shape == lp.shape == ((n, N) if text else (n, 4, N))
    assert ids.shape[:-1] == out.ids[0].shape
    assert torch.equal(ids, want_ids.long()) and torch.equal(lp, want_lp)
    assert torch.equal(out.logprobs[0], dev.lp_out[1, :n, 0] if text else dev.lp_out[1, :n])  # logprobs as before
    im = _top_image(dev, 1, n)
    for k in (n, 3):  # a cancelled suspended request ends with the first k tokens of its image
        got = dev.harvest(im, k)
        (gi, gl), = got.top_logprobs
        assert torch.equal(gi, ids[:k]) and torch.equal(gl, lp[:k]) and gi.dtype == torch.int64
        assert torch.equal(got.ids[0], out.ids[0][:k])
    empty = dev.empty(0)
    (ei, el), = empty.top_logprobs
    assert ei.shape == el.shape == ((0, N) if text else (0, 4, N))
    assert ei.dtype == torch.int64 and el.dtype == torch.float32


def test_top_logprobs_alone_and_off():
    dev = _top_device(False, logprobs=False)
    out = dev.harvest(0, 4)
    assert out.logprobs == [] and len(out.top_logprobs) == 1
    assert dev.empty(0).logprobs == [] and len(dev.empty(0).top_logprobs) == 1
    off = _host_device(False)  # an engine without top_logprobs: outputs as before
    assert off.harvest(1, 5).top_logprobs == [] and off.empty(0).top_logprobs == []
    assert off.harvest(_image(off, 1, 5), 5).top_logprobs == []
    assert GPT.GenerationOutputs(ids=[], attentions=[], hiddens=[]).top_logprobs == []


def test_streamed_yields_are_copies_of_the_prefix():
    """generate_continuous_stream harvests with copy=False: the rows a yield carries must not change as the engine
    writes on."""
    dev = _top_device(False)
    first = dev.harvest(0, 3, copy=False)
    (ids, lp), = first.top_logprobs
    ids0, lp0 = ids.clone(), lp.clone()
    dev.top_ids_out.add_(1)
    dev.top_lp_out.sub_(1)
    assert torch.equal(ids, ids0) and torch.equal(lp, lp0)
    later = dev.harvest(0, 6, copy=False)
    (i2, l2), = later.top_logprobs
    assert torch.equal(i2[:3], ids0 + 1) and torch.equal(l2[:3], lp0 - 1)


# ---------------------------------------------------------------------------------------------------- Job.top_logprobs
def _top_rows(n):
    ids = torch.arange(n * 4 * N, dtype=torch.int64).view(n, 4, N)
    return ids, -ids.float()


class _TopStub(_Stub):
    """_Stub with top buffers: harvests carry (ids, lp) rows of their token counts."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.top_ids_out = torch.zeros(self.slots, 256, 4, N, dtype=torch.int32)

    def harvest(self, slot, n, copy=True):
        out = super().harvest(slot, n, copy)
        out.top_logprobs = [_top_rows(n)]
        return out


class _BothStub(_LpStub, _TopStub):
    pass


def _open(chat, cls):
    devs = []

    def make(requests):
        devs.append(cls(4, requests, chat, lambda r: None))
        return devs[-1]

    return ChatEngine(make, 8, None, None, None, chat, False, max_new_cap=200), devs


@pytest.mark.parametrize("cls", [_TopStub, _BothStub])
def test_job_top_logprobs_for_every_kind_of_job(cls):
    chat = _TakesChat(dict(zip(SENTENCES, (9, 9, 25, 41, 17))), dict(zip(SENTENCES, (9, 17, 25, 9, 33))))
    chat.code_len["one"] = 21
    p, r = _params()
    eng, _ = _open(chat, cls)
    with eng:
        one = eng.submit("one", params_infer_code=p)
        takes = eng.submit("one", params_infer_code=p, takes=3)
        split = eng.submit(PARA, params_infer_code=p, split_text=True)
        refined = eng.submit(PARA, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r)
        for j in (one, takes, split, refined):
            j.result(timeout=30)
    ids, lp = one.top_logprobs
    assert ids.shape == lp.shape == (21, 4, N) and torch.equal(ids, _top_rows(21)[0])
    assert [t[0].shape for t in takes.top_logprobs] == [(5, 4, N), (8, 4, N), (11, 4, N)]  # take order
    for job in (split, refined):  # one pair per sentence, in sentence order; no reference stage, no refinement
        assert [t[0].shape[0] for t in job.top_logprobs] == [chat.code_len[s] for s in SENTENCES]
        assert all(t.device.type == "cpu" for pair in job.top_logprobs for t in pair)
    if cls is _BothStub:  # logprobs keep their own structure beside it
        assert one.logprobs.shape == (21, 4) and [t.shape for t in takes.logprobs] == [(5, 4), (8, 4), (11, 4)]
    else:
        assert one.logprobs is None and takes.logprobs is None


def test_without_top_logprobs_jobs_have_none_and_decode_as_before():
    counts = []
    for cls in (_Stub, _TopStub):
        chat = _chat()
        eng, devs = _open(chat, cls)
        with eng:
            job = eng.submit(PARA, params_infer_code=_params()[0], split_text=True)
            job.result(timeout=30)
        assert (job.top_logprobs is None) == (cls is _Stub)
        counts.append([d.decodes for d in devs])
    assert counts[0] == counts[1]


# ---------------------------------------------------------------------------------------------------- scoring
class TopFakeLib(FakeLib):
    """FakeLib with ctb_gpt_score_ex: ctb_gpt_score's entries, and for entry e and k < N the id e * N + k with
    log-probability -(e * N + k)."""

    def ctb_gpt_score_ex(self, h, B, T, emb, n_prompt, n_given, targets, text, out, n_top, ids, lp, stream):
        rc = self.ctb_gpt_score(h, B, T, emb, n_prompt, n_given, targets, text, out, stream)
        m = sum(self.calls[-1]["n"]) * (1 if text else NVQ)
        v = np.arange(m * n_top)
        np.ctypeslib.as_array((C.c_int32 * (m * n_top)).from_address(ids.value))[:] = v
        np.ctypeslib.as_array((C.c_float * (m * n_top)).from_address(lp.value))[:] = -v
        self.calls[-1]["n_top"] = n_top
        return rc


def test_score_without_top_logprobs_is_as_before(fake):
    g, lib = fake
    Ps, ns = [3, 20, 1100], [4, 1, 6]
    codes = [_codes(n, i) for i, n in enumerate(ns)]
    prompts = [_prompt(P, i) for i, P in enumerate(Ps)]
    a = g.score(prompts, codes)
    b = g.score(prompts, codes, top_logprobs=0)
    assert all(isinstance(t, torch.Tensor) for t in b) and len(a) == len(b)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not any("n_top" in c for c in lib.calls)


@pytest.mark.parametrize("text", [False, True])
def test_score_with_top_logprobs_rows_and_shapes(monkeypatch, fake, text):
    g, _ = fake
    lib = TopFakeLib()
    from chattts_b200 import _lib
    monkeypatch.setattr(_lib, "load", lambda *a, **k: lib)
    Ps, ns = [3, 20, 7, 1100], [4, 1, 0, 6]
    if text:
        targets = [torch.randint(0, 21178, (n,), generator=torch.Generator().manual_seed(i)) for i, n in enumerate(ns)]
    else:
        targets = [_codes(n, i) for i, n in enumerate(ns)]
    prompts = [_prompt(P, i) for i, P in enumerate(Ps)]
    plain = g.score(prompts, targets, infer_text=text)
    rows = g.score(prompts, targets, infer_text=text, top_logprobs=N)
    assert [c.get("n_top") for c in lib.calls] == [None, None, N, N]  # two groups per call
    rpi = 1 if text else NVQ
    start = {0: 0, 1: 4, 3: 0}  # each row's first entry in its group's call (rows 0, 1 | row 3 alone)
    for i, (lp, ids, tlp) in enumerate(rows):
        shape = (ns[i], N) if text else (ns[i], NVQ, N)
        assert torch.equal(lp, plain[i])
        assert ids.shape == tlp.shape == shape and ids.dtype == torch.int64 and tlp.dtype == torch.float32
        if ns[i]:
            want = torch.arange(start[i] * rpi * N, (start[i] + ns[i]) * rpi * N).view(shape)
            assert torch.equal(ids, want) and torch.equal(tlp, -want.float())
