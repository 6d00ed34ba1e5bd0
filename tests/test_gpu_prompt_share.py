"""Shared prompts on the slot engine (``Request.prompt_key``, ctb_gpt_engine_share_prompt): a request that takes a
running slot's KV for prompt columns [0, c0) and prefills only [c0, T) ends with exactly the ids, hidden states and
end index of its normal admission.

1. Keyed groups of 2, 5 and 12 takes of prompts of 100 (no sharing), 200, 700, 1,024, 1,500 and 4,000 tokens, one
   group of text requests, mixed with unkeyed requests: S = 12 and 40, fp32 and fp16, fixed and paged engines (paged
   under CTB_KV_POISON=1), each request ``torch.equal`` to the same workload without keys.  The short holders are
   admitted in one left-padded group, and each group's take 0 finishes first while the others still read its pages.
2. The same under ``prefill_budget=128``, and under a pool small enough that shared members are suspended and resumed.
3. On a paged engine, the suspend image of a shared slot is byte-equal to that of the same request admitted normally,
   at the same step.
4. Refused calls leave the handle as it was: the run that follows them gives the results of a run without them.
5. ``ChatEngine.submit(text, p, takes=n)``: take k equals, array for array, the waveform of
   ``chat._code_request(text, p, noise_batch=(n, k))`` run on the same engine without a key.
"""
import dataclasses

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import EngineDevice, ScheduleStats, pool_pages_needed, schedule, shared_prompt_cols
from test_gpu_kv_pool import FP16, _equal, _model, _request

pytestmark = pytest.mark.gpu

CAP = 48
CTX = 4096


def _workload(embed):
    """Keyed groups (T, takes, text) then unkeyed requests; take 0 of each group stops 40 tokens early."""
    groups = [(100, 2, False), (200, 5, False), (700, 12, False), (1024, 2, False), (1500, 5, False),
              (4000, 2, False), (300, 3, True)]
    reqs = []
    for g, (T, n, text) in enumerate(groups):
        first = _request(embed, T, 100 * g, text=text)
        for k in range(n):
            mx = 8 if k == 0 else CAP - 2 * (k % 3)
            reqs.append(dataclasses.replace(first, manual_seed=7000 + 100 * g + k, max_new_token=mx,
                                            min_new_token=mx, prompt_key=("utt", g)))
    reqs += [_request(embed, T, 50 + k, max_new=CAP - k) for k, T in enumerate((40, 260, 1030, 90))]
    return reqs


def _unkeyed(reqs):
    return [dataclasses.replace(r, prompt_key=None) for r in reqs]


def _run(gpt, reqs, slots, flags, pool=None, budget=None, chunk=8):
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, CAP, True, flags, kv_pool_pages=pool)
        stats = ScheduleStats()
        for i, slot, n in schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget):
            o = dev.empty(i) if slot is None else dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone() if o.hiddens else None)
    return got, stats


def _pool(reqs, slots):
    return slots * (-(-CTX // 16)) + 1


@pytest.mark.parametrize("flags", [0, FP16])
@pytest.mark.parametrize("slots", [12, 40])
def test_shared_prompts_are_bit_identical(slots, flags, monkeypatch):
    gpt, embed = _model(40, CTX)
    reqs = _workload(embed)
    ref, _ = _run(gpt, _unkeyed(reqs), slots, flags)
    got, stats = _run(gpt, reqs, slots, flags)
    _equal("fixed", got, ref)
    shareable = sum(n - 1 for T, n in ((200, 5), (700, 12), (1024, 2), (1500, 5), (4000, 2), (300, 3)))
    # with 40 slots every member is admitted at the first poll, beside its take 0
    assert stats.shares == shareable if slots == 40 else stats.shares > 0, stats.shares
    monkeypatch.setenv("CTB_KV_POISON", "1")
    got, stats = _run(gpt, reqs, slots, flags, pool=_pool(reqs, slots))
    _equal("paged", got, ref)
    assert (stats.shares == shareable if slots == 40 else stats.shares > 0) and stats.peak_shared_pages > 0
    assert stats.suspensions == 0


def test_budget_and_small_pool(monkeypatch):
    gpt, embed = _model(40, CTX)
    reqs = _workload(embed)
    ref, _ = _run(gpt, _unkeyed(reqs), 12, 0)
    got, stats = _run(gpt, reqs, 12, 0, budget=128)
    _equal("budget 128", got, ref)
    assert stats.shares > 0 and max(stats.prefill_cols) <= 128
    monkeypatch.setenv("CTB_KV_POISON", "1")
    got, stats = _run(gpt, reqs, 12, 0, pool=_pool(reqs, 12), budget=128)
    _equal("budget 128, paged", got, ref)
    small = 2 * max(pool_pages_needed(r) for r in reqs) + 1
    got, stats = _run(gpt, reqs, 12, 0, pool=small, chunk=4)
    _equal("small pool", got, ref)
    assert stats.shares > 0 and stats.suspensions > 0 and stats.resumes == stats.suspensions, \
        (stats.shares, stats.suspensions)


def _image(gpt, reqs, flags, share, steps=16):
    """Slot 0 holds reqs[0]; reqs[1] enters slot 1 by a share (or normally), decodes `steps` steps and is suspended:
    its image's bytes."""
    T = int(reqs[1].emb.shape[0])
    c0 = shared_prompt_cols(T)
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True, flags, kv_pool_pages=400)
        assert dev.reserve([0], [T + CAP])
        dev.admit([(0, 0)])
        if share:
            assert dev.share(0, 1, 1, c0)
            assert dev.reserve([1], [T + CAP])
            dev.prefill_chunk(1, 1, c0, T - c0)
        else:
            assert dev.reserve([1], [T + CAP])
            dev.admit([(1, 1)])
        dev.decode(steps)
        dev.status()
        im = dev.suspend(1)
        im.ready.synchronize()
        return im.buf.clone(), im.header.off_kv


@pytest.mark.parametrize("flags", [0, FP16])
def test_suspend_image_of_a_shared_slot_is_byte_equal(flags, monkeypatch):
    monkeypatch.setenv("CTB_KV_POISON", "1")
    gpt, embed = _model(40, CTX)
    first = _request(embed, 1500, 11, max_new=CAP)
    reqs = [dataclasses.replace(first, manual_seed=1, prompt_key="k"),
            dataclasses.replace(first, manual_seed=2, prompt_key="k")]
    a, off = _image(gpt, reqs, flags, share=False)
    b, _ = _image(gpt, reqs, flags, share=True)
    assert torch.equal(a[off:], b[off:]), "KV section"
    assert torch.equal(a, b)


@pytest.mark.parametrize("paged", [False, True])
def test_refused_calls_leave_the_handle_as_it_was(paged, monkeypatch):
    monkeypatch.setenv("CTB_KV_POISON", "1")
    gpt, embed = _model(40, CTX)
    first = _request(embed, 700, 21, max_new=CAP)
    reqs = [dataclasses.replace(first, manual_seed=30 + k, prompt_key="k") for k in range(3)]
    other = _request(embed, 300, 22, max_new=CAP)

    def run(refuse):
        out = {}
        with torch.cuda.device(gpt.device_gpt):
            dev = EngineDevice(gpt, reqs + [other], 4, CAP, True, 0, kv_pool_pages=300 if paged else None)
            lib, h = dev.lib, gpt._handle

            def share(src, dst, T0, c0):
                return lib.ctb_gpt_engine_share_prompt(h, src, dst, T0, c0, dev.stream)

            if paged:
                assert dev.reserve([0, 3], [700 + CAP, 300 + CAP])
            dev.admit([(0, 0), (3, 3)])
            if refuse:
                assert share(0, 0, 700, 640) != 0  # src == dst
                assert share(2, 1, 700, 640) != 0  # src idle
                assert share(0, 1, 700, 600) != 0  # c0 not a multiple of 128
                assert share(0, 1, 700, 0) != 0 and share(0, 1, 700, 768) != 0  # c0 not positive, not below T0
                assert share(3, 1, 700, 640) != 0  # src's prompt (300) shorter than c0
                assert share(0, 1, 1100, 640) != 0  # different prefill attention kernels
                assert share(0, 3, 700, 640) != 0  # dst running
                assert share(0, 4, 700, 640) != 0  # dst out of range
                if paged:
                    assert dev.reserve([1], [16])
                    assert share(0, 1, 700, 640) != 0  # dst has pages mapped
                    dev.release([1])
                    hog = [2]
                    assert dev.reserve(hog, [16 * (300 - 1 - dev.pages_in_use)])
                    assert share(0, 1, 700, 640) == _lib.ERR_POOL
                    dev.release(hog)
            assert dev.share(0, 1, 1, 640)
            if paged:
                assert dev.reserve([1], [700 + CAP])
            dev.prefill_chunk(1, 1, 640, 60)
            st = dev.status()
            while any(s == _lib.SLOT_RUNNING for s in st.state):
                if paged:
                    assert dev.reserve([0, 1, 3], [700 + CAP, 700 + CAP, 300 + CAP])
                dev.decode(8)
                st = dev.status()
            for s in (0, 1, 3):
                o = dev.harvest(s, st.end_idx[s])
                out[s] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
        return out

    ref = run(False)
    got = run(True)
    for s in ref:
        assert torch.equal(got[s][0], ref[s][0]) and torch.equal(got[s][1], ref[s][1]), s


def test_chat_takes_equal_their_rows():
    from chattts_b200.core import _Paragraph
    from test_gpu_stream import chat

    c = chat()
    text = "a rather long sentence to speak, " * 5  # about 170 prompt tokens: the takes share 128 columns
    p = c.InferCodeParams(manual_seed=9, max_new_token=40, min_new_token=8, temperature=0.5, show_tqdm=False)
    n = 3
    with c.open_engine(slots=4, max_new_cap=64, use_decoder=False) as eng:
        takes = eng.submit(text, p, takes=n, do_text_normalization=False, do_homophone_replacement=False).result()
        stats_shares = eng.stats.shares
        norm = c.normalizer(text, False, False, None)
        rows = []
        for k in range(n):  # the same request, unkeyed, as a job of one sentence
            r = c._code_request(norm, p, noise_batch=(n, k))
            para = _Paragraph(1, None)
            para.order[r] = 0
            para.job = eng._new_job([r], False, para)
            eng._enqueue([(para.job, [r])])
            rows.append(para.job.result())
    assert int(r.emb.shape[0]) > 128 and stats_shares == n - 1
    assert len(takes) == n
    for k in range(n):
        assert np.array_equal(takes[k], rows[k]), k
