"""Refusals of the slot engine's entry points: the exact return code of each refused call, on a fixed engine and on a
paged engine under CTB_KV_POISON=1, and a handle that then serves the workload with the ids and hidden states of a run
without any refused call.

Every entry point is refused with a bad argument, a bad state and, where both can occur, both at once: a call with
several faults returns the code of the check it reaches first.  An admission checks each slot in turn (range and
repetition, state, ``max_new``, sampler, pages), so ``[running slot, out-of-range slot]`` is a state error and the
reverse an argument error.  On the paged engine ``ctb_gpt_engine_pages`` follows the script: k pages reserved are k in
use, a share at c0 maps c0/16 shared pages, and releasing the holder frees only its unshared pages.

A decode step's shared-page refusal is not in the script: a slot that maps shared pages writes only at or past the
share's c0 (a source's positions start at the end of its prompt, which holds at least c0), so no call sequence reaches
it.
"""
import ctypes as C
import dataclasses

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import EngineDevice
from test_gpu_kv_pool import _model, _request

pytestmark = pytest.mark.gpu

OK, ARG, STATE, POOL = 0, -1, -3, _lib.ERR_POOL
S = 5      # slots 0-3 serve A, B, C and D; slot 4 stays idle
CAP = 48
CTX = 4096
POOL_PAGES = 300


def _requests(embed):
    """A (700 tokens, 8 new) holds the prompt that B shares at c0 = 640; C (300) and D (200) are admitted with A."""
    a = _request(embed, 700, 21, max_new=8)
    b = dataclasses.replace(a, manual_seed=31, max_new_token=CAP, min_new_token=CAP)
    return [a, b, _request(embed, 300, 22), _request(embed, 200, 23)]


def _pages(dev):
    used, shared = C.c_int32(-1), C.c_int32(-1)
    rc = dev.lib.ctb_gpt_engine_pages(dev.gpt._handle, C.byref(used), C.byref(shared))
    return rc, used.value, shared.value


def _script(gpt, embed, paged, refuse):
    """Admit A, C and D; share A's prompt with B; decode to the end (A ends first; on the paged engine it is then
    released, and C is suspended and resumed).  With ``refuse``, the refused calls on the way.  The outputs of A-D."""
    reqs = _requests(embed)
    T = [int(r.emb.shape[0]) for r in reqs]
    limit = [t + r.max_new_token for t, r in zip(T, reqs)]
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, S, CAP, True, 0, kv_pool_pages=POOL_PAGES if paged else None)
        lib, h, stream = dev.lib, gpt._handle, dev.stream
        cfgs, _ = dev._sampling([reqs[0], reqs[0]], False, False, {})
        bad = (_lib.SamplerConfig * 2)(*cfgs)
        bad[0].past_window = bad[1].past_window = 32
        emb = torch.zeros(2, CTX - 1, gpt.config.hidden_size, device=gpt.device_gpt)
        mask = torch.ones(2, CTX - 1, dtype=torch.uint8, device=gpt.device_gpt)
        pinned = torch.zeros(1 << 16, dtype=torch.uint8, pin_memory=True)
        unpinned = torch.zeros(1 << 16, dtype=torch.uint8)

        def i32(*v):
            return (C.c_int32 * len(v))(*v)

        def admit(slots, T0=700, max_new=None, sampler=cfgs, text=False, n=None):
            fn = lib.ctb_gpt_engine_admit_text if text else lib.ctb_gpt_engine_admit
            max_new = i32(*([CAP] * len(slots) if max_new is None else max_new))
            return fn(h, len(slots) if n is None else n, i32(*slots) if slots else None, T0,
                      C.c_void_p(emb.data_ptr()), C.c_void_p(mask.data_ptr()), sampler, None, max_new, stream)

        def chunk(slot, c0, n, T0=700, max_new=CAP, sampler=cfgs):
            return lib.ctb_gpt_engine_prefill_chunk(h, slot, T0, c0, n, C.c_void_p(emb.data_ptr()), 0, sampler, None,
                                                    max_new, stream)

        def share(src, dst, c0=640, T0=700):
            return lib.ctb_gpt_engine_share_prompt(h, src, dst, T0, c0, stream)

        def reserve(slots, tokens, n=None):
            return lib.ctb_gpt_engine_reserve(h, len(slots) if n is None else n, i32(*slots), i32(*tokens), stream)

        def release(slots, n=None):
            return lib.ctb_gpt_engine_release(h, len(slots) if n is None else n, i32(*slots), stream)

        def cancel(slots, n=None):
            return lib.ctb_gpt_engine_cancel(h, len(slots) if n is None else n, i32(*slots) if slots else None, stream)

        def suspend_bytes(slot):
            return lib.ctb_gpt_engine_suspend_bytes(h, slot, C.byref(C.c_uint64()), stream)

        def suspend(slot, buf=pinned, nbytes=1 << 16):
            return lib.ctb_gpt_engine_suspend(h, slot, C.c_void_p(buf.data_ptr()), nbytes, stream)

        def resume(slot, buf, nbytes):
            return lib.ctb_gpt_engine_resume(h, slot, C.c_void_p(buf.data_ptr()), nbytes, stream)

        def decode(n):
            return lib.ctb_gpt_decode(h, n, stream)

        def expect(rc, want, what):
            assert rc == want, (what, rc, want, lib.ctb_last_error().decode())

        # ---- every slot idle
        if refuse:
            expect(reserve([0], [16], n=0), ARG if paged else STATE, "reserve n=0")
            expect(release([0], n=S + 1), ARG if paged else STATE, "release n=S+1")
            expect(suspend_bytes(9), ARG if paged else STATE, "suspend_bytes of slot 9")
            expect(suspend(0, unpinned), STATE, "suspend of an idle slot into unpinned memory")
            expect(resume(9, pinned, 1 << 16), ARG if paged else STATE, "resume into slot 9")
            expect(cancel([], n=1), ARG, "cancel, null slots")
            expect(cancel([0], n=0), ARG, "cancel n=0")
            expect(cancel([0, 1, 2, 3, 4, 0]), ARG, "cancel n=S+1")
            expect(cancel([9]), ARG, "cancel slot 9")
            expect(cancel([1, 1]), ARG, "cancel, repeated slot")
            expect(chunk(9, 0, 128), ARG, "chunk into slot 9")
            expect(chunk(0, 0, 128, T0=7), ARG, "chunk, T0 below 8")
            expect(chunk(0, 640, 128), ARG, "chunk past the prompt")
            expect(chunk(0, 64, 128), ARG, "chunk at a misaligned c0")
            expect(chunk(0, 0, 100), ARG, "non-final chunk of a misaligned length")
            expect(chunk(0, 0, 128, max_new=0), ARG, "chunk, max_new 0")
            expect(chunk(0, 0, 700, sampler=None), ARG, "final chunk, null sampler")
            expect(chunk(0, 0, 700, sampler=bad), ARG, "final chunk, bad sampler")
            expect(chunk(0, 128, 128), STATE, "chunk at 128 without a prompt in progress")
            expect(chunk(0, 128, 572, sampler=bad), ARG, "final chunk at 128: its sampler before the prompt in progress")
            expect(chunk(9, 64, 128, max_new=0), ARG, "chunk: slot, c0 and max_new bad")
            expect(share(0, 1), STATE, "share from an idle slot")
            expect(share(0, 0, c0=600), ARG, "share: src == dst and a misaligned c0")
            if paged:
                expect(admit([0]), STATE, "admission into a slot without pages")
                expect(admit([0], sampler=bad), ARG, "admission without pages: the sampler first")
                expect(admit([1, 1]), STATE, "admission: a slot without pages, then the same slot")
                expect(chunk(0, 0, 128), STATE, "chunk into a slot without pages")
                expect(reserve([9], [16]), ARG, "reserve slot 9")
                expect(reserve([1, 1], [16, 16]), ARG, "reserve, repeated slot")
                expect(reserve([0], [-1]), ARG, "reserve of -1 tokens")
                expect(reserve([0], [CTX + 1]), ARG, "reserve past max_context")
                expect(reserve([0, 1], [16 * 200, 16 * 200]), POOL, "reserve beyond the pool")
                expect(reserve([0, 0], [10 ** 6, 10 ** 6]), ARG, "reserve: repeated slot and tokens out of range")
                expect(release([1, 1]), ARG, "release, repeated slot")
                expect(release([9]), ARG, "release slot 9")
                expect(suspend_bytes(0), STATE, "suspend_bytes of an idle slot")
                expect(_pages(dev), (OK, 0, 0), "pages of an empty pool")
            else:
                expect(admit([1, 1]), ARG, "admission, repeated slot")
                expect(reserve([0], [16]), STATE, "reserve on a fixed engine")
                expect(release([0]), STATE, "release on a fixed engine")
                expect(suspend_bytes(0), STATE, "suspend_bytes on a fixed engine")
                expect(suspend(0), STATE, "suspend on a fixed engine")
                expect(resume(0, pinned, 1 << 16), STATE, "resume on a fixed engine")
                expect(_pages(dev)[0], STATE, "pages on a fixed engine")

        if paged:  # 45 + 22 + 13 pages; D holds its prompt and 8 positions, 3 pages short of its 48 new tokens
            assert dev.reserve([0, 2, 3], [limit[0], limit[2], 208 if refuse else limit[3]])
            if refuse:
                expect(_pages(dev), (OK, 80, 0), "pages after reserving 80")
        dev.admit([(0, 0), (2, 2), (3, 3)])

        # ---- A, C and D running; slots 1 and 4 idle
        if refuse:
            expect(admit([0]), STATE, "admission into a running slot")
            expect(admit([0], text=True), STATE, "text admission into a running slot")
            expect(admit([0, 9]), STATE, "admission: a running slot, then slot 9")
            expect(admit([9, 0]), ARG, "admission: slot 9, then a running slot")
            expect(admit([], n=1), ARG, "admission, null slots")
            expect(admit([1], n=0), ARG, "admission n=0")
            expect(admit([1, 2, 3, 0, 4, 1]), ARG, "admission n=S+1")
            expect(admit([1], T0=7), ARG, "admission, T0 below 8")
            expect(admit([1], T0=CTX), ARG, "admission, T0 of max_context")
            expect(admit([1], max_new=[0]), ARG, "admission, max_new 0")
            expect(admit([1], max_new=[CAP + 1]), ARG, "admission, max_new over the capacity")
            expect(admit([1], T0=CTX - 10, max_new=[11]), ARG, "admission past max_context")
            expect(admit([1], sampler=bad), ARG, "admission, bad sampler")
            expect(admit([0], max_new=[0], sampler=bad), STATE, "admission: running slot, max_new and sampler bad")
            expect(chunk(0, 0, 128), STATE, "chunk into a running slot")
            expect(chunk(0, 0, 700), STATE, "final chunk into a running slot")
            expect(chunk(0, 128, 572), STATE, "final chunk at 128 into a running slot")
            expect(share(0, 0), ARG, "share src == dst")
            expect(share(0, 1, c0=600), ARG, "share at a misaligned c0")
            expect(share(0, 1, c0=0), ARG, "share at c0 = 0")
            expect(share(0, 1, c0=768), ARG, "share at a c0 past T0")
            expect(share(0, S), ARG, "share into slot S")
            expect(share(0, 1, T0=7), ARG, "share, T0 below 8")
            expect(share(2, 1), STATE, "share from a prompt shorter than c0")
            expect(share(0, 1, T0=1100), ARG, "share across prefill attention kernels")
            expect(share(0, 2), STATE, "share into a running slot")
            expect(share(1, 2, c0=600), ARG, "share: idle source, running target, misaligned c0")
            expect(share(1, 2), STATE, "share: idle source and running target")
            expect(release([0]), STATE, "release of a running slot")
            expect(suspend_bytes(1), STATE, "suspend_bytes of an idle slot")
            expect(cancel([0, 9]), ARG, "cancel: a running slot, then slot 9")
            if paged:
                expect(admit([1]), STATE, "admission into a slot without pages")
                expect(release([1, 0]), STATE, "release: an idle slot, then a running one")
                expect(suspend(2, unpinned), ARG, "suspend into unpinned memory")
                expect(suspend(2, pinned, 64), ARG, "suspend into too small a buffer")
                expect(suspend(9), ARG, "suspend of slot 9")
                assert dev.reserve([1], [16])
                expect(share(0, 1), STATE, "share into a slot with pages mapped")
                dev.release([1])
                assert dev.reserve([4], [16 * (POOL_PAGES - 1 - 80)])  # every free page
                expect(share(0, 1), POOL, "share beyond the pool")
                expect(reserve([1], [16]), POOL, "reserve from an empty free list")
                dev.release([4])
                expect(_pages(dev), (OK, 80, 0), "pages after the refusals")

        assert dev.share(0, 1, 1, 640)
        if refuse:
            expect(share(0, 1), STATE, "share into a slot with a prompt in progress")
            expect(release([1]), STATE, "release of a prompt in progress")
            expect(suspend_bytes(1), STATE, "suspend_bytes of a prompt in progress")
            expect(resume(1, unpinned, 64), STATE, "resume into a prompt in progress from unpinned memory")
            expect(chunk(1, 0, 128), STATE, "chunk that restarts the prompt in progress")
            expect(chunk(1, 512, 128), STATE, "chunk behind the prompt in progress")
            expect(chunk(1, 640, 60, sampler=bad), ARG, "final chunk, bad sampler")
            if paged:
                expect(_pages(dev), (OK, 84, 40), "pages after a share at 640")
                expect(admit([1]), STATE, "admission that writes shared pages")
                expect(admit([1], max_new=[0]), ARG, "admission that writes shared pages, max_new 0")
        if paged:
            assert dev.reserve([1], [limit[1]])
        dev.prefill_chunk(1, 1, 640, 60)
        if paged and refuse:
            expect(decode(16), STATE, "decode past D's pages")
            assert dev.reserve([3], [limit[3]])
            expect(_pages(dev), (OK, 90, 40), "pages with B and D reserved")

        # ---- decode to the end
        st = dev.status()
        first = True
        im = None
        while any(s == _lib.SLOT_RUNNING for s in st.state):
            run = [s for s in range(4) if st.state[s] == _lib.SLOT_RUNNING]
            if paged:
                assert dev.reserve(run, [limit[s] for s in run])
            dev.decode(8)
            st = dev.status()
            if refuse and first:
                first = False
                assert st.state[0] == _lib.SLOT_FINISHED and st.state[2] == _lib.SLOT_RUNNING
                if paged:
                    expect(_pages(dev), (OK, 90, 40), "pages before the holder's release")
                    dev.release([0])
                    expect(_pages(dev), (OK, 85, 0), "pages after the holder's release")
                    expect(share(0, 4), STATE, "share from a released slot")
                    expect(suspend_bytes(0), STATE, "suspend_bytes of a finished slot")
                    im = dev.suspend(2)
                    im.ready.synchronize()
                    nb = im.nbytes
                    expect(resume(2, im.buf, nb), STATE, "resume into a slot without pages")
                    expect(resume(2, unpinned, nb), ARG, "resume without pages from unpinned memory")
                    expect(resume(9, im.buf, nb), ARG, "resume into slot 9")
                    expect(resume(1, im.buf, nb), STATE, "resume into a running slot")
                    expect(resume(3, im.buf, nb), STATE, "resume into a running slot whose pages are short")
                    expect(resume(4, pinned, 1 << 16), ARG, "resume of a buffer that holds no image")
                    expect(resume(4, im.buf, 64), ARG, "resume of a buffer shorter than a header")
                    expect(resume(4, im.buf, nb - 1), ARG, "resume of a truncated image")
                    assert dev.reserve([2], [limit[2]])
                    dev.resume(2, im)
                    st = dev.status()
        out = {}
        for s in range(4):
            o = dev.harvest(s, st.end_idx[s])
            out[s] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
    return out


@pytest.mark.parametrize("paged", [False, True])
def test_refusals_return_their_codes_and_change_nothing(paged, monkeypatch):
    monkeypatch.setenv("CTB_KV_POISON", "1")
    gpt, embed = _model(40, CTX)
    ref = _script(gpt, embed, paged, refuse=False)
    got = _script(gpt, embed, paged, refuse=True)
    for s in ref:
        assert torch.equal(got[s][0], ref[s][0]) and torch.equal(got[s][1], ref[s][1]), s
        assert torch.isfinite(got[s][1]).all(), s
