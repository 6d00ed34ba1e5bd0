"""The open slot engine on the GPU: requests that arrive while the engine decodes and requests cancelled mid-decode keep
the engine contract (ids bit-identical to the request's B = 1 run, hidden states within 1e-4), a cancelled request's
ids are a prefix of its lone run, the text tail leaves the decode step once no text slot runs, and Chat.open_engine
jobs equal Chat.infer per text."""
import concurrent.futures

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.engine import Arrivals, EngineDevice, ScheduleStats, _poll_cycles
from oracle.gpt_oracle import GPTOracle
from test_gpu_continuous import DEFAULT, MIXED, _check, _oracle, _request, _spec
from test_gpu_refine_engine import _refine_params, _tcheck, _toracle, _trequest, _tspec, chat
from test_gpu_stream import TEXTS, _chat_params

pytestmark = pytest.mark.gpu


def _mixed(embed):
    """12 requests, text and code mixed, seeded, with different sampling parameters."""
    specs = [(i % 3 != 1, _tspec(i, MIXED[i % len(MIXED)]) if i % 3 != 1 else _spec(i, MIXED[i % len(MIXED)]))
             for i in range(12)]
    return specs, [_trequest(embed, s) if t else _request(embed, s) for t, s in specs]


def _drive(gpt, slots, reqs, plan, chunk=8, cancel_at=None, cap=90):
    """Run the open scheduling policy from this thread: ``plan[p]`` lists the requests (indices into ``reqs``)
    submitted after poll p (before poll 0 for p = -1), ``cancel_at[p]`` the ones cancelled then.  Returns
    ``({request: outputs}, stats, {request: slots it was admitted to})``."""
    src, stats, requests = Arrivals(), ScheduleStats(), []
    got, where = {}, {}
    last = max(max(plan), max(cancel_at or {-1: 0}))
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, requests, slots, cap)
        for k in plan.get(-1, []):
            src.submit(reqs[k])
        for poll, (st, owner, ended) in enumerate(_poll_cycles(requests, dev, chunk, stats=stats, source=src)):
            for s, i in enumerate(owner):
                if i is not None:
                    where.setdefault(requests[i], set()).add(s)
            for i, s, n, _ in ended:
                out = dev.empty(i) if s is None else dev.harvest(s, n)
                got[requests[i]] = out
            for k in plan.get(poll, []):
                src.submit(reqs[k])
            for k in (cancel_at or {}).get(poll, []):
                src.cancel(reqs[k])
            if poll == last:
                src.close()
    return got, stats, where


@pytest.mark.parametrize("slots", [3, 12])
def test_staggered_arrivals_match_b1_oracle(slots):
    """Requests submitted at five different polls through 3 slots (PDL chain) and 12 slots (wgmma step)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs, reqs = _mixed(embed)
    plan = {-1: [2, 0, 1], 0: [3, 4], 1: [5, 6, 7], 2: [8], 3: [9, 10, 11]}
    got, stats, _ = _drive(gpt, slots, reqs, plan)
    assert len(got) == len(reqs) and not stats.cancelled
    for k, (t, s) in enumerate(specs):
        if t:
            _tcheck(got[reqs[k]], _toracle(orc, s), (slots, k))
        else:
            _check(got[reqs[k]], _oracle(orc, s), (slots, k))


@pytest.mark.parametrize("slots", [4, 10])
def test_cancel_mid_decode_keeps_a_prefix_and_everyone_else_exact(slots):
    """Request 0 (forced to 90 tokens) is cancelled after poll 2; a request submitted then takes its slot.  S = 4 runs
    the PDL chain, S = 10 the wgmma step."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [_spec(2, DEFAULT)] + [_spec(i, DEFAULT) for i in (0, 1, 3, 4, 5, 6)] + [_spec(8, DEFAULT)]
    reqs = [_request(embed, s) for s in specs]
    n_first = min(slots, 7)
    plan = {-1: list(range(n_first)), 3: [7]}  # request 7 arrives after the poll that stopped request 0
    if n_first < 7:
        plan[1] = list(range(n_first, 7))
    got, stats, where = _drive(gpt, slots, reqs, plan, cancel_at={2: [0]})
    victim = got[reqs[0]]
    n = int(victim.ids[0].shape[0])
    ref = _oracle(orc, specs[0])
    assert 0 < n < 90 and victim is not None
    assert torch.equal(victim.ids[0].cpu(), ref.ids[0][:n])
    assert (victim.hiddens[0].cpu() - ref.hiddens[0][:n]).abs().max() < 1e-4
    assert where[reqs[0]] == {0} and any(0 in where[r] for r in reqs[1:])  # a later request takes its slot
    for k in range(1, len(reqs)):
        _check(got[reqs[k]], _oracle(orc, specs[k]), (slots, k))


def test_cancelling_the_only_text_slot_drops_the_text_tail():
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    lib = _lib.load()
    code, text = _spec(2, DEFAULT), _tspec(0, DEFAULT)
    reqs = [_request(embed, code), _trequest(embed, text)]

    def step():
        c0 = lib.ctb_launch_count()
        dev.decode(1)
        dev.status()
        return lib.ctb_launch_count() - c0

    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 4, 90)
        dev.admit([(0, 0)])
        dev.status()
        d_code = step()
        dev.admit([(1, 1)])
        dev.status()
        d_text = step()
        dev.cancel([1])
        st = dev.status()
        assert st.state[1] == _lib.SLOT_FINISHED and st.finish[1] == 0 and st.state[0] == _lib.SLOT_RUNNING
        n = st.end_idx[1]
        out = dev.harvest(1, n)
        d_after = step()
        steps = dev.status().steps_done
        dev.cancel([0, 1])  # a finished slot is left as it is
        st = dev.status()
        dev.decode(3)
        assert dev.status().steps_done == st.steps_done == steps  # nothing runs: no-op steps are not counted
    assert d_text > d_code and d_after == d_code, (d_code, d_text, d_after)
    ref = _toracle(orc, text)
    assert n == 2 and torch.equal(out.ids[0].cpu(), ref.ids[0][:n])


def test_gpt_open_engine_threads_and_single_owner():
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs, reqs = _mixed(embed)
    with gpt.open_engine(3, 90, chunk=8) as eng:
        with pytest.raises(RuntimeError):
            next(gpt.generate_continuous(reqs[:2]))
        jobs = [eng.submit(r, stream=k % 4 == 0) for k, r in enumerate(reqs[:6])]
        jobs[0].result(timeout=120)
        jobs += [eng.submit(r) for r in reqs[6:]]
        streams = {k: [o for o, _ in jobs[k]] for k in (0, 4)}
        outs = [j.result(timeout=300) for j in jobs]
    for k, (t, s) in enumerate(specs):
        (_tcheck if t else _check)(outs[k], (_toracle if t else _oracle)(orc, s), k)
    for k, ys in streams.items():
        assert torch.equal(ys[-1].ids[0].cpu(), outs[k].ids[0].cpu())
    got = dict(gpt.generate_continuous(reqs[:2], slots=2))  # the handle is free again
    assert sorted(got) == [0, 1]


# ---------------------------------------------------------------------------------------------------- Chat
def _same_wave(x, y, use_decoder, tag):
    assert x.shape == y.shape, (tag, x.shape, y.shape)
    if use_decoder:
        assert x.size == 0 or float(np.sqrt(np.mean((x - y) ** 2))) < 1e-4, tag
    else:
        assert np.array_equal(x, y), tag


@pytest.mark.parametrize("use_decoder", [False, True])
def test_chat_open_engine_equals_infer_per_text(use_decoder):
    c = chat()
    params, refine = _chat_params(c), _refine_params(c)
    with c.open_engine(slots=3, max_new_cap=200, use_decoder=use_decoder) as eng:
        plain = eng.submit(TEXTS[0], params_infer_code=params[0])
        streamed = eng.submit(TEXTS[1], params_infer_code=params[1], stream=True)
        refined = eng.submit(TEXTS[2], params_infer_code=params[2], skip_refine_text=False,
                             params_refine_text=refine[2])
        both = eng.submit(TEXTS[3], params_infer_code=params[3], stream=True)
        chunks = list(streamed)
        chunks3 = list(both)
        wav0, wav2 = plain.result(timeout=300), refined.result(timeout=300)
    ref0 = c.infer([TEXTS[0]], split_text=False, skip_refine_text=True, use_decoder=use_decoder,
                   params_infer_code=params[0])[0]
    _same_wave(wav0, ref0, use_decoder, "plain")
    ref2 = dict(c.infer_continuous([TEXTS[2]], params_infer_code=[params[2]], params_refine_text=[refine[2]],
                                   use_decoder=use_decoder, skip_refine_text=False, refine_on_engine=True))[0]
    _same_wave(wav2, ref2, use_decoder, "refined")
    for k, got in ((1, chunks), (3, chunks3)):
        ref = list(c.infer([TEXTS[k]], stream=True, split_text=False, skip_refine_text=True, use_decoder=use_decoder,
                           params_infer_code=params[k]))
        assert [last for _, last in got] == [False] * (len(ref) - 1) + [True]
        for (x, _), y in zip(got[:-1], ref[:-1]):
            _same_wave(x, y, use_decoder, k)
        if use_decoder:
            assert abs(got[-1][0].shape[1] - ref[-1].shape[1]) <= 2
        else:
            assert np.array_equal(got[-1][0], ref[-1])


def test_chat_open_engine_cancelled_jobs():
    c = chat()
    p = c.InferCodeParams(manual_seed=5, max_new_token=200, min_new_token=200, stream_batch=16, stream_speed=6000,
                          pass_first_n_batches=0, show_tqdm=False)
    with c.open_engine(slots=2, max_new_cap=200, use_decoder=False) as eng:
        s = eng.submit("one", params_infer_code=p, stream=True)
        a = eng.submit("two", params_infer_code=p)
        w = eng.submit("three", params_infer_code=p)  # waits for a slot
        r = eng.submit("four", params_infer_code=p, skip_refine_text=False,
                       params_refine_text=c.RefineTextParams(manual_seed=1, max_new_token=20, min_new_token=20,
                                                             show_tqdm=False))
        it = iter(s)
        next(it)
        for j in (s, a, w, r):
            j.cancel()
        rest = list(it)
        assert not any(last for _, last in rest)
        for j in (a, w, r):
            with pytest.raises(concurrent.futures.CancelledError):
                j.result(timeout=60)
            assert j.cancelled()
        ok = eng.submit("five", params_infer_code=c.InferCodeParams(manual_seed=9, max_new_token=30,
                                                                    show_tqdm=False))
        assert ok.result(timeout=120).ndim == 1
    assert s.cancelled()
