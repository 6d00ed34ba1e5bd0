"""Chunked prefill on the slot engine (ctb_gpt_engine_prefill_chunk, ``prefill_budget``): a prompt prefilled in
chunks over several polls gives the same bits as the same prompt admitted in one call.

1. Bit identity: seeded code and text requests with prompts of 136, 1,000, 1,024, 1,025, 2,085 and 4,000 tokens, run
   with budgets of 128, 512 and 1,024 columns (chunks of at most that many), fp32 and fp16 engines, short requests
   decoding between the chunks, the 4,000-token request first so its slot is reused: ids and hidden states
   ``torch.equal`` to the run without a budget, whose prompts are admitted in one call each.  The short requests
   (the neighbours) are equal too.  The code requests of up to 1,024 tokens also match ``GPT.generate`` alone (B = 1):
   ids bit for bit, hidden states within 1e-4.
2. Every CTB_ERR_STATE / CTB_ERR_ARG case of the entry point, then the same handle serves requests correctly.
3. ``GPT.open_engine`` and ``Chat.open_engine`` with ``prefill_budget=1024``: long and short jobs, streaming and
   not, one job cancelled while its prompt is in progress; every other job equals the run without a budget, and the
   cancelled job's slot serves the next job.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.engine import EngineDevice, Request, ScheduleStats, schedule
from chattts_b200.gpt import GPT
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from gpu_util import release_on_teardown

pytestmark = pytest.mark.gpu

FP16 = _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV
EOS, EOS_TEXT = 625, 21177
MAX_CONTEXT = 4096
CAP = 48
ERR_ARG, ERR_STATE = -1, -3
LONG = [136, 1000, 1024, 1025, 2085, 4000]

_models = {}
_release = release_on_teardown(_models)


def _model():
    if "plain" not in _models:
        cfg = Config()
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=8, max_context=MAX_CONTEXT)
        gpt.load_state(gs)
        _models["plain"] = (gpt, embed)
    return _models["plain"]


def _request(embed, T, k, text=False, max_new=CAP):
    ids, _, tmask = synth_prompt_batch([T], seed=700 + k)
    warp, proc = gen_logits(num_code=21178 if text else EOS, top_P=0.7, top_K=20, repetition_penalty=1.05)
    return Request(emb=embed(ids, tmask)[0], temperature=[0.7] if text else [0.3, 0.5, 0.7, 1.0],
                   eos_token=EOS_TEXT if text else EOS, max_new_token=max_new, min_new_token=max_new,
                   logits_processors=(*proc, *warp), manual_seed=9000 + k, infer_text=text)


def _workload(embed):
    """The 4,000-token request first (its slot is reused), then the others as code and text requests, with short
    requests among them that decode while the long ones are prefilled"""
    reqs = [_request(embed, 4000, 0)]
    for k, T in enumerate(LONG[:-1]):
        reqs.append(_request(embed, T, 10 + k))
        reqs.append(_request(embed, T, 20 + k, text=True))
        reqs.append(_request(embed, 40 + k, 30 + k, max_new=CAP - 8 * k))
    reqs.append(_request(embed, 4000, 40, text=True))
    return reqs


def _run(gpt, reqs, flags, budget, slots=4, dev=None):
    """Every request through one engine -> ({index: (ids, hiddens)}, stats, chunk calls)"""
    got, chunks = {}, []
    with torch.cuda.device(gpt.device_gpt):
        dev = dev or EngineDevice(gpt, reqs, slots, CAP, True, flags)
        one = dev.prefill_chunk
        dev.prefill_chunk = lambda s, i, c0, n: (chunks.append((s, i, c0, n)), one(s, i, c0, n))
        stats = ScheduleStats()
        for i, slot, n in schedule(reqs, dev, 8, stats=stats, prefill_budget=budget):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone() if o.hiddens else None)
            o.destroy()
        del dev.prefill_chunk
    return got, stats, chunks


def _equal(tag, got, ref):
    assert sorted(got) == sorted(ref), tag
    for i in ref:
        assert torch.equal(got[i][0], ref[i][0]), (tag, i)
        if ref[i][1] is not None:
            assert torch.equal(got[i][1], ref[i][1]), (tag, i, float((got[i][1] - ref[i][1]).abs().max()))


_refs = {}


def _reference(flags):
    if flags not in _refs:
        gpt, embed = _model()
        reqs = _workload(embed)
        _refs[flags] = (reqs, _run(gpt, reqs, flags, None)[0])
    return _refs[flags]


@pytest.mark.parametrize("flags", [0, FP16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("budget", [128, 512, 1024])
def test_chunked_prefill_is_bit_identical(flags, budget):
    gpt, _ = _model()
    reqs, ref = _reference(flags)
    got, stats, chunks = _run(gpt, reqs, flags, budget)
    assert max(stats.prefill_cols) <= budget
    long = {i for i, r in enumerate(reqs) if r.emb.shape[0] > budget}
    assert long <= {i for _, i, c0, n in chunks if n < reqs[i].emb.shape[0]}, "every prompt over the budget is chunked"
    assert max(n for *_, n in chunks) <= budget
    _equal(f"budget {budget}", got, ref)  # the chunked requests and their neighbours


def test_chunked_code_requests_match_static_generate():
    gpt, embed = _model()
    reqs, _ = _reference(0)
    got, _, _ = _run(gpt, reqs, 0, 128)
    for i, r in enumerate(reqs):
        T = int(r.emb.shape[0])
        if r.infer_text or T > 1024 or T < 128:
            continue
        ids = synth_prompt_batch([T], seed=700 + (10 + LONG.index(T)))[0]
        out = list(gpt.generate(r.emb[None], ids, temperature=torch.tensor(r.temperature), eos_token=EOS,
                                max_new_token=r.max_new_token, min_new_token=r.min_new_token,
                                logits_processors=r.logits_processors, return_hidden=True, show_tqdm=False,
                                manual_seed=r.manual_seed))[-1]
        assert torch.equal(out.ids[0].cpu().int(), got[i][0].long().int()), (i, T)
        assert (out.hiddens[0].cpu() - got[i][1]).abs().max() < 1e-4, (i, T)
        out.destroy()


def _chunk(dev, slot, T0, c0, n, max_new=8, sampler=True):
    gpt = dev.gpt
    emb = torch.zeros(n, 768, device="cuda")
    cfg = _lib.SamplerConfig()
    cfg.min_tokens_to_keep, cfg.eos_token = 1, EOS
    return dev.lib.ctb_gpt_engine_prefill_chunk(gpt._handle, slot, T0, c0, n, C.c_void_p(emb.data_ptr()), 0,
                                                C.byref(cfg) if sampler else None, None, max_new, dev.stream)


def test_errors_leave_the_handle_usable():
    gpt, embed = _model()
    reqs = [_request(embed, 1000, 50), _request(embed, 2085, 51), _request(embed, 40, 52)]
    ref = _run(gpt, reqs, 0, None, slots=2)[0]
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True)
        # arguments
        assert _chunk(dev, 2, 1000, 0, 128) == ERR_ARG  # slot out of range
        assert _chunk(dev, 0, 7, 0, 7) == ERR_ARG  # T0 under 8
        assert _chunk(dev, 0, MAX_CONTEXT, 0, 128) == ERR_ARG  # T0 over max_context - 1
        assert _chunk(dev, 0, 1000, 64, 128) == ERR_ARG  # c0 not aligned
        assert _chunk(dev, 0, 1000, 0, 100) == ERR_ARG  # a non-final n not aligned
        assert _chunk(dev, 0, 1000, 0, 1001) == ERR_ARG  # past the prompt
        assert _chunk(dev, 0, 4090, 0, 128, max_new=8) == ERR_ARG  # T0 + max_new over max_context
        assert _chunk(dev, 0, 1000, 896, 104, sampler=False) == ERR_ARG  # a final chunk without a sampler
        # state
        assert _chunk(dev, 0, 1000, 128, 128) == ERR_STATE  # a first chunk must start at 0
        assert _chunk(dev, 0, 1000, 0, 128) == 0
        assert _chunk(dev, 0, 1000, 256, 128) == ERR_STATE  # skips [128, 256)
        assert _chunk(dev, 0, 900, 128, 128) == ERR_STATE  # another T0
        assert _chunk(dev, 0, 1000, 0, 128) == ERR_STATE  # restarts without a cancel
        assert _chunk(dev, 0, 1000, 128, 128) == 0
        dev.cancel([0])  # drops the prompt in progress
        assert _chunk(dev, 0, 1000, 256, 128) == ERR_STATE
        assert _chunk(dev, 0, 1000, 0, 128) == 0
        dev.admit([(1, 2)])  # slot 1 runs
        assert _chunk(dev, 1, 1000, 0, 128) == ERR_STATE  # a running slot
        dev.admit([(0, 2)])  # drops slot 0's prompt in progress
        assert _chunk(dev, 0, 1000, 128, 128) == ERR_STATE
        dev.decode(CAP)
        st = dev.status()
        assert st.state[:2] == [_lib.SLOT_FINISHED] * 2
        dev.ids_out.zero_()
        dev.hid_out.zero_()
        got = _run(gpt, reqs, 0, 512, dev=dev)[0]
    _equal("after the errors", got, ref)


def _job_results(eng, reqs, cancel_index=None, stream_every=3):
    """Submit ``reqs`` at once (every ``stream_every``-th streaming) -> [result or streamed yields, or None if
    cancelled]"""
    jobs = [eng.submit(r, stream=(k % stream_every == 0)) for k, r in enumerate(reqs)]
    out = []
    for k, job in enumerate(jobs):
        if job.stream:
            ys = [(o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone(), last) for o, last in job]
            out.append(None if job.cancelled() else ys)
        else:
            try:
                o = job.result(timeout=600)
            except Exception:
                assert k == cancel_index
                out.append(None)
                continue
            out.append(None if job.cancelled() else (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone()))
    return out


def test_gpt_open_engine_cancel_mid_prefill(monkeypatch):
    gpt, embed = _model()
    reqs = [_request(embed, 64, 60), _request(embed, 3000, 61), _request(embed, 500, 62), _request(embed, 1500, 63),
            _request(embed, 2085, 64), _request(embed, 40, 65)]
    with gpt.open_engine(2, CAP) as eng:
        ref = _job_results(eng, reqs)
    victim = reqs[1]
    holder = {}
    one = EngineDevice.prefill_chunk

    def spy(self, slot, index, c0, n):  # cancel the 3,000-token job as soon as its first chunk is issued
        one(self, slot, index, c0, n)
        if self.requests[index] is victim and c0 == 0:
            holder["slot"] = slot
            holder["eng"]._source.cancel(holder["eng"].stats.keys[index])

    monkeypatch.setattr(EngineDevice, "prefill_chunk", spy)
    with gpt.open_engine(2, CAP, prefill_budget=1024) as eng:
        holder["eng"] = eng
        got = _job_results(eng, reqs, cancel_index=1)
        stats = eng.stats
    assert "slot" in holder and got[1] is None
    assert max(stats.prefill_cols) <= 1024
    for k in (0, 2, 3, 4, 5):
        if isinstance(ref[k], list):
            assert len(got[k]) == len(ref[k]), k
            for a, b in zip(got[k], ref[k]):
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2], k
        else:
            assert torch.equal(got[k][0], ref[k][0]) and torch.equal(got[k][1], ref[k][1]), k


def _chat():
    if "chat" not in _models:
        from chattts_b200 import Chat
        from chattts_b200.synth import synth_all
        from stubs import StubSpeaker, StubTokenizer

        c = Chat()
        assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                             max_batch=4, max_context=MAX_CONTEXT)
        _models["chat"] = c
    return _models["chat"]


def test_chat_open_engine_with_a_budget():
    from chattts_b200.speaker import Speaker

    c = _chat()
    g = torch.Generator().manual_seed(5)
    spk = Speaker.encode_prompt(torch.randint(0, 625, (4, 520), generator=g))
    texts = ["a first text", "the second text is spoken with a voice sample", "third", "and the fourth one"]
    params = [c.InferCodeParams(manual_seed=20 + k, max_new_token=40, min_new_token=40, show_tqdm=False,
                                spk_smp=spk if k % 2 else None, txt_smp="a sample" if k % 2 else None)
              for k in range(len(texts))]

    def run(budget):
        with c.open_engine(slots=2, max_new_cap=64, use_decoder=False, prefill_budget=budget) as eng:
            jobs = [eng.submit(t, params_infer_code=p, stream=(k == 1)) for k, (t, p) in enumerate(zip(texts, params))]
            out = [np.concatenate([ch for ch, _ in job], axis=1) if job.stream else job.result(timeout=600)
                   for job in jobs]
            return out, eng.stats

    ref, _ = run(None)
    got, stats = run(128)
    assert stats.chunks > 0 and max(stats.prefill_cols) <= 128
    for k in range(len(texts)):
        assert np.array_equal(got[k], ref[k]), k
