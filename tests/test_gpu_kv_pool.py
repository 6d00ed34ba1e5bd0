"""KV pages on demand (ctb_gpt_engine_begin_paged, ``kv_pool_bytes``): where a request's KV lives, and whether it was
suspended to host memory and resumed in another slot, does not change one bit of its results.

1. A pool large enough never to suspend, S = 12 and 40, fp32 and fp16, code and text requests: ids and hidden states
   ``torch.equal`` to the fixed engine's.
2. The same with every slot's pages scattered and out of order and CTB_KV_POISON=1: equal, and every output finite.
3. A pool small enough to force at least 10 suspensions: every request equal to the fixed engine, one resumed into
   another slot; a streaming open engine with a text job under the same pool yields what the fixed engine yields; an
   open engine whose jobs are cancelled while one is suspended: that one ends with its image's tokens and hidden states,
   a prefix of its fixed-engine run; a prefill budget beside the pool, whose prompt in progress is never suspended.
4. A 4,000-token slot suspended, resumed into another slot and suspended again: both images byte-equal (the KV
   section page by page), fp32 and fp16, and the request then ends as on the fixed engine.
5. Refused calls leave the handle as it was: a reserve beyond the pool, a suspend of an idle slot or of a slot with a
   prompt in progress, a resume into a busy or unmapped slot, an admission into a slot whose pages do not cover the
   prompt.
6. ``Chat.open_engine(kv_pool_bytes=...)`` with split-text refined paragraphs under a pool that forces suspensions:
   every job's audio equals its audio on the fixed engine.
"""
import random

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.engine import EngineDevice, Request, ScheduleStats, pool_pages_needed, schedule
from chattts_b200.gpt import GPT
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from gpu_util import release_on_teardown

pytestmark = pytest.mark.gpu

FP16 = _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV
EOS, EOS_TEXT = 625, 21177
CAP = 48

_models = {}
_release = release_on_teardown(_models)


def _model(max_batch, max_context):
    key = (max_batch, max_context)
    if key not in _models:
        cfg = Config()
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(synth_embed_state(1)).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
        gpt.load_state(synth_gpt_state(0))
        _models[key] = (gpt, embed)
    return _models[key]


def _request(embed, T, k, text=False, max_new=CAP):
    ids, _, tmask = synth_prompt_batch([T], seed=800 + k)
    warp, proc = gen_logits(num_code=21178 if text else EOS, top_P=0.7, top_K=20, repetition_penalty=1.05)
    return Request(emb=embed(ids, tmask)[0], temperature=[0.7] if text else [0.3, 0.5, 0.7, 1.0],
                   eos_token=EOS_TEXT if text else EOS, max_new_token=max_new, min_new_token=max_new,
                   logits_processors=(*proc, *warp), manual_seed=5000 + k, infer_text=text)


def _workload(embed, n):
    return [_request(embed, 20 + 37 * (k % 5), k, text=k % 4 == 3, max_new=CAP - 4 * (k % 3)) for k in range(n)]


def _run(gpt, reqs, slots, flags, pool=None, prepare=None):
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, CAP, True, flags, kv_pool_pages=pool)
        if prepare is not None:
            prepare(dev)
        stats = ScheduleStats()
        for i, slot, n in schedule(reqs, dev, 8, stats=stats):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone() if o.hiddens else None)
            o.destroy()
    return got, stats, dev


def _equal(tag, got, ref):
    assert sorted(got) == sorted(ref), tag
    for i in ref:
        assert torch.equal(got[i][0], ref[i][0]), (tag, i)
        if ref[i][1] is not None:
            assert torch.equal(got[i][1], ref[i][1]), (tag, i)
            assert torch.isfinite(got[i][1]).all(), (tag, i)


def _scatter(dev):
    """Permute the free list: twice, the slots take one page each per round in a shuffled order for six rounds, then
    are released in a shuffled order.  The pages each slot then takes are spread over the pool and out of order (a
    model of the free list gives every slot of the first test a descending step among its first six pages)."""
    rnd = random.Random(dev.slots)
    order = list(range(dev.slots))
    for _ in range(2):
        for r in range(6):
            rnd.shuffle(order)
            for s in order:
                assert dev.reserve([s], [16 * (r + 1)])
        rnd.shuffle(order)
        dev.release(list(order))


@pytest.mark.parametrize("flags", [0, FP16])
@pytest.mark.parametrize("slots", [12, 40])
def test_large_pool_is_bit_identical(slots, flags, monkeypatch):
    gpt, embed = _model(40, 512)
    reqs = _workload(embed, slots + 8)
    ref, _, _ = _run(gpt, reqs, slots, flags)
    big = slots * 512 // 16 + 1
    got, stats, _ = _run(gpt, reqs, slots, flags, pool=big)
    _equal("large pool", got, ref)
    assert stats.suspensions == 0 and 0 < stats.peak_pages < big
    monkeypatch.setenv("CTB_KV_POISON", "1")
    got, stats, _ = _run(gpt, reqs, slots, flags, pool=big, prepare=_scatter)
    _equal("scattered, poisoned", got, ref)


@pytest.mark.parametrize("flags", [0, FP16])
def test_small_pool_suspends_and_resumes_bit_identically(flags, monkeypatch):
    gpt, embed = _model(40, 512)
    reqs = _workload(embed, 40)
    ref, _, _ = _run(gpt, reqs, 12, flags)
    monkeypatch.setenv("CTB_KV_POISON", "1")
    moves = []

    def prepare(dev):
        sus, res = dev.suspend, dev.resume
        dev.suspend = lambda s: (moves.append(("s", s)), sus(s))[1]
        dev.resume = lambda s, im: (moves.append(("r", s)), res(s, im))[1]

    pool = 2 * max(pool_pages_needed(r) for r in reqs) + 1
    got, stats, _ = _run(gpt, reqs, 12, flags, pool=pool, prepare=prepare)
    _equal("small pool", got, ref)
    assert stats.suspensions >= 10 and stats.resumes == stats.suspensions, stats.suspensions
    assert stats.peak_pages <= pool - 1
    sus = [s for k, s in moves if k == "s"]
    res = [s for k, s in moves if k == "r"]
    assert any(a != b for a, b in zip(sus, res)), "no request resumed into another slot"


def test_open_engine_streams_under_a_small_pool():
    gpt, embed = _model(40, 512)
    reqs = _workload(embed, 16)
    page = 2 * 12 * 16 * 64 * 4 * 20

    def serve(kv_pool_bytes):
        out = {}
        with gpt.open_engine(6, CAP, kv_pool_bytes=kv_pool_bytes) as eng:
            jobs = [eng.submit(r, stream=k % 3 == 0) for k, r in enumerate(reqs)]
            for k, job in enumerate(jobs):
                if job.stream:
                    out[k] = [(o.ids[0].cpu().clone(), last) for o, last in job]
                else:
                    o = job.result()
                    out[k] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone() if o.hiddens else None)
            stats = eng.stats
        return out, stats

    ref, _ = serve(None)
    got, stats = serve(3 * max(pool_pages_needed(r) for r in reqs) * page + page)
    assert stats.suspensions > 0
    for k in ref:
        if isinstance(ref[k], list):
            assert len(got[k]) == len(ref[k]) and all(torch.equal(a[0], b[0]) and a[1] == b[1]
                                                      for a, b in zip(got[k], ref[k])), k
        else:
            assert torch.equal(got[k][0], ref[k][0]), k
            assert (ref[k][1] is None) or torch.equal(got[k][1], ref[k][1]), k


@pytest.mark.parametrize("flags", [0, FP16])
def test_round_trip_of_a_4000_token_slot_is_byte_equal(flags):
    gpt, embed = _model(2, 4096)
    reqs = [_request(embed, 4000, 90, max_new=40)]
    ref, _, _ = _run(gpt, reqs, 2, flags)
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True, flags, kv_pool_pages=2 * 4096 // 16 + 1)
        assert dev.reserve([0], [4000 + 8])
        dev.admit([(0, 0)])
        dev.decode(7)
        assert dev.status().state[0] == _lib.SLOT_RUNNING
        one = dev.suspend(0)
        assert dev.reserve([1], [4000 + 8 + 32])
        dev.resume(1, one)
        two = dev.suspend(1)
        torch.cuda.synchronize()
        h = one.header
        assert h.npages == (4000 + 7 + 15) // 16 and h.seq_len == 4000 + 7
        assert one.nbytes == two.nbytes and torch.equal(one.buf, two.buf)  # header, sections, every page
        assert dev.reserve([0], [4000 + 40])
        dev.resume(0, two)
        st = dev.status()
        while st.state[0] == _lib.SLOT_RUNNING:
            dev.decode(8)
            st = dev.status()
        o = dev.harvest(0, st.end_idx[0])
        assert torch.equal(o.ids[0].cpu(), ref[0][0]) and torch.equal(o.hiddens[0].cpu(), ref[0][1])


def test_refused_calls_leave_the_handle_as_it_was():
    gpt, embed = _model(40, 512)
    reqs = _workload(embed, 3)
    ref, _, _ = _run(gpt, reqs, 2, 0)
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True, 0, kv_pool_pages=40)
        assert not dev.reserve([0, 1], [16 * 20, 16 * 20])  # 40 pages, 39 free: all or nothing
        assert dev.pages_in_use == 0
        with pytest.raises(_lib.CtbError, match="not running"):
            dev.suspend(0)
        with pytest.raises(_lib.CtbError, match="pages hold 0 positions"):
            dev.admit([(0, 0)])  # no pages for the prompt
        assert dev.reserve([0], [16 * 12])
        dev.admit([(0, 0)])
        dev.decode(4)
        dev.status()
        im = dev.suspend(0)
        with pytest.raises(_lib.CtbError, match="pages hold 0 positions"):
            dev.resume(1, im)  # unmapped
        assert dev.reserve([1], [16 * 12])
        dev.admit([(1, 1)])
        with pytest.raises(_lib.CtbError, match="still generating"):
            dev.resume(1, im)  # busy
        with pytest.raises(_lib.CtbError, match="outside"):
            dev.reserve([0], [10 ** 6])
        assert dev.reserve([0], [16 * 12])
        dev.resume(0, im)
        got = {}
        st = dev.status()
        while any(s == _lib.SLOT_RUNNING for s in st.state):
            assert dev.reserve([0, 1], [256, 256])
            dev.decode(8)
            st = dev.status()
        for s, i in ((0, 0), (1, 1)):
            o = dev.harvest(s, st.end_idx[s])
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
    for i in (0, 1):
        assert torch.equal(got[i][0], ref[i][0]) and torch.equal(got[i][1], ref[i][1]), i


def _finish(dev, slot):
    st = dev.status()
    while st.state[slot] == _lib.SLOT_RUNNING:
        dev.decode(8)
        st = dev.status()
    o = dev.harvest(slot, st.end_idx[slot])
    return o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone()


def test_suspend_refuses_a_prompt_in_progress():
    gpt, embed = _model(40, 512)
    reqs = [_request(embed, 300, 60, max_new=40)]
    ref, _, _ = _run(gpt, reqs, 2, 0)
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True, 0, kv_pool_pages=80)
        assert dev.reserve([0], [340])
        dev.prefill_chunk(0, 0, 0, 128)
        with pytest.raises(_lib.CtbError, match="prompt in progress"):
            dev.suspend(0)
        with pytest.raises(_lib.CtbError, match="prompt in progress"):
            dev.release([0])
        dev.prefill_chunk(0, 0, 128, 172)
        got = _finish(dev, 0)
    assert torch.equal(got[0], ref[0][0]) and torch.equal(got[1], ref[0][1])


def test_prefill_budget_beside_a_small_pool():
    """A prompt in progress is never suspended: the device refuses such a suspension, so a run that ends is one where
    the policy never tried."""
    gpt, embed = _model(40, 512)
    reqs = ([_request(embed, 150 + 10 * k, 72 + k) for k in range(6)] + [_request(embed, 420, 70, max_new=40)] +
            [_request(embed, 130 + 10 * k, 80 + k) for k in range(6)] + [_request(embed, 300, 71, text=True)])
    ref, _, _ = _run(gpt, reqs, 4, 0)
    got = {}
    pool = max(pool_pages_needed(r) for r in reqs) + 1  # one request alone fits
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 4, CAP, True, 0, kv_pool_pages=pool)
        stats = ScheduleStats()
        for i, slot, n in schedule(reqs, dev, 8, stats=stats, prefill_budget=128):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone() if o.hiddens else None)
    _equal("budget and pool", got, ref)
    assert stats.chunks > 2 and stats.suspensions > 0, (stats.chunks, stats.suspensions)


def test_cancelled_while_suspended_ends_with_its_image():
    """Every job is cancelled from inside the first suspension, so the cancel reaches the suspended request before it
    can resume: it ends with the tokens and hidden states of its image (served by ``EngineDevice.harvest``), a prefix
    of its run on the fixed engine, as does every other cancelled job."""
    gpt, embed = _model(40, 512)
    reqs = _workload(embed, 12)
    ref, _, _ = _run(gpt, reqs, 4, 0)
    page = 2 * 12 * 16 * 64 * 4 * 20
    served = []
    state = {}
    suspend, harvest = EngineDevice.suspend, EngineDevice.harvest

    def on_suspend(self, s):
        image = suspend(self, s)
        if not state.get("done"):
            state["done"] = True
            for job in list(state["eng"]._pending):
                job.cancel()
        return image

    def on_harvest(self, s, n, copy=True):
        if not isinstance(s, int):
            served.append(n)
        return harvest(self, s, n, copy)

    try:
        EngineDevice.suspend, EngineDevice.harvest = on_suspend, on_harvest
        with gpt.open_engine(4, CAP, kv_pool_bytes=(2 * max(pool_pages_needed(r) for r in reqs) + 1) * page) as eng:
            state["eng"] = eng
            jobs = [eng.submit(r, stream=k % 3 == 0) for k, r in enumerate(reqs)]
            outs = {}
            for k, job in enumerate(jobs):
                if job.stream:
                    ys = list(job)
                    outs[k] = ys[-1][0] if ys else None
                else:
                    try:
                        outs[k] = job.result()
                    except Exception:  # cancelled before it was admitted
                        outs[k] = None
    finally:
        EngineDevice.suspend, EngineDevice.harvest = suspend, harvest
    assert state.get("done") and served and all(n > 0 for n in served), served
    for k, o in outs.items():
        if o is None:
            continue
        n = o.ids[0].shape[0]
        assert torch.equal(o.ids[0].cpu(), ref[k][0][:n]), k
        if o.hiddens:
            assert torch.equal(o.hiddens[0].cpu(), ref[k][1][:n]), k


def test_chat_refined_paragraphs_under_a_small_pool(monkeypatch):
    from test_gpu_paragraph import PARAGRAPHS
    from test_gpu_paragraph_refine import _params, _refine
    from test_gpu_stream import chat

    c = chat()
    params = [_params(c, k) for k in range(len(PARAGRAPHS))]
    refine = [_refine(c, k) for k in range(len(PARAGRAPHS))]
    page = 2 * 12 * 16 * 64 * 4 * 20
    # polls every 4 steps, so a stage outgrows the chunk its admission mapped and the running stages compete for pages
    monkeypatch.setenv("CTB_DECODE_CHUNK", "4")
    sizes = []
    admit = EngineDevice.admit

    def sized(self, batch):  # the positions each stage can hold, from the run on the fixed engine
        sizes.extend(int(self.requests[i].emb.shape[0]) + self.requests[i].max_new_token for _, i in batch)
        return admit(self, batch)

    def run(kv_pool_bytes):
        with c.open_engine(slots=4, max_new_cap=64, use_decoder=False, kv_pool_bytes=kv_pool_bytes) as eng:
            jobs = [eng.submit(t, params_infer_code=p, split_text=True, skip_refine_text=False, params_refine_text=r,
                               max_split_batch=4) for t, p, r in zip(PARAGRAPHS, params, refine)]
            wavs = [j.result() for j in jobs]
            return wavs, eng.stats

    try:
        EngineDevice.admit = sized
        ref, _ = run(None)
    finally:
        EngineDevice.admit = admit
    got, stats = run((-(-max(sizes) // 16) + 1) * page)  # the largest stage alone fits
    assert stats.suspensions > 0 and stats.resumes == stats.suspensions
    for k in range(len(PARAGRAPHS)):
        assert np.array_equal(got[k], ref[k]), k
