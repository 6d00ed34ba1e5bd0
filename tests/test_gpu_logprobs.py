"""Token log-probabilities on the slot engine (ctb_gpt_engine_logprobs, ctb_token_logprobs, ``logprobs=True``).

L1: attaching the buffer changes nothing: every request's ids and hidden states are bit-equal to the run without it
(fp32 at S = 4, 24, 64; fp16 at S = 24, 64; code and text, seeded and unseeded; a paged engine that suspends; a
prefill budget chunking a 2,085-token prompt; three takes sharing one prompt key).  L2: the stand-alone kernel against
float64 log_softmax of the same fp32 logits, and bit-reproducible.  L3: code rows against float64 heads applied to the
harvested hidden states; text rows against the teacher-forced float64 model.  L4: bookkeeping (lengths, a request
that ends empty, a cancelled prefix, suspension and resume, streamed prefixes, the ABI's refusals).  L5:
``Chat.open_engine(logprobs=True)`` on the stub components."""
import ctypes as C
import dataclasses
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.engine import Arrivals, EngineDevice, ScheduleStats, _poll_cycles, pool_pages_needed, schedule
from chattts_b200.gpt import GPT
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from f64_oracle import F64Oracle
from gpu_util import release_on_teardown
from oracle.gpt_oracle import fold_weight_norm
from test_gpu_fp16_engine import KV16, MIXED, W16, _request, _spec, _text_spec

pytestmark = pytest.mark.gpu

FP16 = W16 | KV16
CAP = 90
ERR_ARG, ERR_STATE = -1, -3
_handles, _refs = {}, {}
_release = release_on_teardown(_handles, _refs)


def _model(max_batch=64, max_context=640):
    key = (max_batch, max_context)
    if key not in _handles:
        cfg = Config()
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
        gpt.load_state(gs)
        _handles[key] = (gpt, embed, gs, es)
    return _handles[key]


def _mix(n=26):
    """Code requests (every fifth unseeded) with mixed sampling parameters, and two text requests."""
    specs = [_spec(i, MIXED[i % len(MIXED)], seeded=i % 5 != 4) for i in range(n)]
    specs[5:5] = [_text_spec(0)]
    return specs + [_text_spec(1)]


def _run(gpt, reqs, slots, flags=0, logprobs=False, pool=None, budget=None, cap=CAP, chunk=16):
    """Every request through one engine -> ({index: (ids, hiddens or None, logprobs or None, slot)}, stats).  Unseeded
    requests draw their Philox seeds from torch's generator, seeded here so that two runs draw the same ones."""
    torch.manual_seed(1234)
    got, stats = {}, ScheduleStats()
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, cap, True, flags, kv_pool_pages=pool, logprobs=logprobs)
        for i, slot, n in schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget):
            o = dev.empty(i) if slot is None else dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu(), o.hiddens[0].cpu() if o.hiddens else None,
                      o.logprobs[0].cpu() if o.logprobs else None, slot)
            assert bool(o.logprobs) == logprobs
            o.destroy()
    return got, stats


def _bookkeeping(tag, got):
    """L4: a row per request with its ids' length, [n, num_vq] for codes and [n] for text, finite and <= 0."""
    for i, (ids, _, lp, _) in got.items():
        assert lp.shape == ids.shape, (tag, i, lp.shape, ids.shape)
        assert lp.dtype == torch.float32 and torch.isfinite(lp).all() and (lp <= 0).all(), (tag, i)


def _same(tag, a, b):
    """L1: ids and hidden states bit-equal with and without the buffer."""
    assert sorted(a) == sorted(b), tag
    for i in a:
        assert torch.equal(a[i][0], b[i][0]), (tag, i)
        assert (a[i][1] is None) == (b[i][1] is None), (tag, i)
        if a[i][1] is not None:
            assert torch.equal(a[i][1], b[i][1]), (tag, i)


def _heads64(es):
    k = "head_code.{}.parametrizations.weight.original{}"
    return [fold_weight_norm(es[k.format(q, 0)].double(), es[k.format(q, 1)].double()).cuda() for q in range(4)]


def _code_error(specs, got, heads):
    """L3 for code requests: |lp - log_softmax(hidden64 @ W_head64^T)[id]| over every token, and over first tokens."""
    worst = first = 0.0
    for i, s in enumerate(specs):
        ids, hid, lp, _ = got[i]
        if s["text"] or ids.shape[0] == 0:
            continue
        h = hid.cuda().double()
        ref = torch.stack([F.log_softmax(h @ heads[q].t(), -1).gather(1, ids[:, q:q + 1].cuda().long())[:, 0]
                           for q in range(4)], 1).cpu()
        err = (lp.double() - ref).abs()
        worst, first = max(worst, float(err.max())), max(first, float(err[0].max()))
    return worst, first


# L3 bars, from the observed maxima (DESIGN.md §4, "Token log-probabilities")
CODE_BAR = 2e-5
TEXT_BAR = 1e-4


# ---------------------------------------------------------------------------------------------------- L1 / L3 / L4
@pytest.mark.parametrize("slots,flags", [(4, 0), (24, 0), (64, 0), (24, FP16), (64, FP16)])
def test_l1_attaching_changes_nothing_and_l3_code_rows_follow_the_heads(slots, flags):
    gpt, embed, gs, es = _model()
    specs = _mix(66 if slots == 64 else 26)
    reqs = [_request(embed, s) for s in specs]
    base, _ = _run(gpt, reqs, slots, flags)
    got, _ = _run(gpt, reqs, slots, flags, logprobs=True)
    _same((slots, flags), got, base)
    _bookkeeping((slots, flags), got)
    again, _ = _run(gpt, reqs, slots, flags, logprobs=True)
    assert all(torch.equal(got[i][2], again[i][2]) for i in got)  # the same run gives the same bits
    worst, first = _code_error(specs, got, _heads64(es))
    print(f"\nL3 S={slots} flags={flags}: max |lp - float64 heads| = {worst:.3e} (first tokens {first:.3e})")
    assert worst < CODE_BAR, (slots, flags, worst)


def test_l3_text_rows_follow_the_float64_model():
    gpt, embed, gs, es = _model()
    specs = [_text_spec(i) for i in range(4)] + [_spec(0, MIXED[0])]
    reqs = [_request(embed, s) for s in specs]
    got, _ = _run(gpt, reqs, 4, 0, logprobs=True)
    orc = F64Oracle(gs, es, device="cuda")
    k = "head_text.parametrizations.weight.original{}"
    head = fold_weight_norm(es[k.format(0)].double(), es[k.format(1)].double()).cuda()
    worst = 0.0
    for i, s in enumerate(specs[:4]):
        ids, _, lp, _ = got[i]
        n, T0 = ids.shape[0], reqs[i].emb.shape[0]
        assert n > 0
        x = torch.cat([reqs[i].emb.cuda().double(), orc.emb_text[ids[: n - 1].cuda()]])
        hid = orc.forward(x)[T0 - 1:]
        ref = F.log_softmax(hid @ head.t(), -1).gather(1, ids.cuda()[:, None])[:, 0].cpu()
        worst = max(worst, float((lp.double() - ref).abs().max()))
    print(f"\nL3 text: max |lp - teacher-forced float64| = {worst:.3e}")
    assert worst < TEXT_BAR, worst


def test_l1_paged_engine_that_suspends_keeps_the_rows_of_the_fixed_engine():
    """A pool of a third of what the requests need: requests are suspended and resumed, in other slots, and their
    rows equal those of the never-suspended run on a fixed engine."""
    gpt, embed, _, _ = _model()
    specs = _mix()
    reqs = [_request(embed, s) for s in specs]
    fixed, _ = _run(gpt, reqs, 24, 0, logprobs=True)
    pool = max(2 * max(pool_pages_needed(r) for r in reqs), sum(pool_pages_needed(r) for r in reqs) // 3)
    base, _ = _run(gpt, reqs, 24, 0, pool=pool)
    got, stats = _run(gpt, reqs, 24, 0, logprobs=True, pool=pool)
    assert stats.suspensions > 0 and stats.resumes > 0, (stats.suspensions, stats.resumes)
    _same("paged", got, base)
    for i in fixed:
        assert torch.equal(got[i][2], fixed[i][2]), i


def test_l1_prefill_budget_chunks_a_long_prompt():
    gpt, embed, _, _ = _model(4, 2304)
    specs = [dict(_spec(0, MIXED[0]), length=2085, max_new=48, min_new=48), _spec(1, MIXED[1]), _text_spec(2),
             dict(_spec(3, MIXED[2]), length=700)]
    reqs = [_request(embed, s) for s in specs]
    whole, _ = _run(gpt, reqs, 4, 0, logprobs=True, cap=64)
    base, _ = _run(gpt, reqs, 4, 0, budget=256, cap=64)
    got, stats = _run(gpt, reqs, 4, 0, logprobs=True, budget=256, cap=64)
    assert stats.chunks > 2
    _same("budget", got, base)
    _bookkeeping("budget", got)
    for i in whole:  # a chunked admission samples the first token from the same logits as a whole one
        assert torch.equal(got[i][2], whole[i][2]), i
    _handles.pop((4, 2304))
    gc.collect()
    torch.cuda.empty_cache()


def test_l1_takes_sharing_a_prompt_key():
    gpt, embed, _, _ = _model()
    first = _request(embed, dict(_spec(0, MIXED[0]), length=300))
    reqs = [dataclasses.replace(first, manual_seed=40 + k, prompt_key="utt") for k in range(3)]
    plain = [dataclasses.replace(r, prompt_key=None) for r in reqs]
    base, _ = _run(gpt, reqs, 4, 0)
    got, stats = _run(gpt, reqs, 4, 0, logprobs=True, chunk=4)
    ref, _ = _run(gpt, plain, 4, 0, logprobs=True)
    assert stats.shares > 0
    _same("takes", got, base)
    for i in ref:
        assert torch.equal(got[i][2], ref[i][2]), i


# ---------------------------------------------------------------------------------------------------- L2
def _ulp_bar(z, ids):
    """8 fp32 ulps of max(|z_id - max|, log(den), 1): the kernel rounds z_id - max once in fp32 (0.5 ulp of it), each
    expf is within 2 ulps relative, so den and log(den) are within ~2^-22 (summing in double adds nothing at these V),
    and the result is rounded once to fp32 (0.5 ulp of |lp| <= |z_id - max| + log(den))."""
    z64 = z.double()
    mx = z64.max(1).values
    scale = torch.maximum((z64.gather(1, ids[:, None].long())[:, 0] - mx).abs(), torch.logsumexp(z64 - mx[:, None], 1))
    return 8 * 2.0 ** -23 * scale.clamp_min(1.0)


@pytest.mark.parametrize("V", [626, 21178])
def test_l2_kernel_matches_float64_log_softmax(V):
    g = torch.Generator().manual_seed(V)
    rows = 64
    z = torch.randn(rows, V, generator=g) * 3
    z[16:32] = (torch.rand(16, V, generator=g) * 160 - 80)  # logits of +-80
    z[32:48] = torch.randn(16, V, generator=g)
    ids = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    for r in range(32, 48):  # exact ties at the maximum, the id among them or not
        m = float(z[r].max()) + 1.0
        tie = torch.randperm(V, generator=g)[:5]
        z[r, tie] = m
        if r % 2 == 0:
            ids[r] = int(tie[r % 5])
    ids[48:56] = z[48:56].argmax(1).int()  # the row's arg-max
    zd, idd = z.cuda(), ids.cuda()
    out = [torch.full((rows,), 7.0, device="cuda") for _ in range(2)]
    lib = _lib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for o in out:
        _lib.check(lib.ctb_token_logprobs(C.c_void_p(zd.data_ptr()), rows, V, C.c_void_p(idd.data_ptr()),
                                          C.c_void_p(o.data_ptr()), stream))
    torch.cuda.synchronize()
    got = out[0].cpu()
    ref = torch.log_softmax(z.double(), 1).gather(1, ids[:, None].long())[:, 0]
    err = (got.double() - ref).abs()
    bar = _ulp_bar(z, ids)
    print(f"\nL2 V={V}: max |lp - float64| = {float(err.max()):.3e}, max err / bar = {float((err / bar).max()):.3f}")
    assert (err <= bar).all(), (int((err / bar).argmax()), float((err / bar).max()))
    assert torch.equal(out[0], out[1])  # the same inputs give the same bits
    # an id outside [0, V) gives NaN; bad arguments are refused
    bad = torch.tensor([V, -1], dtype=torch.int32, device="cuda")
    o = torch.zeros(2, device="cuda")
    _lib.check(lib.ctb_token_logprobs(C.c_void_p(zd.data_ptr()), 2, V, C.c_void_p(bad.data_ptr()),
                                      C.c_void_p(o.data_ptr()), stream))
    assert torch.isnan(o).all()
    assert lib.ctb_token_logprobs(None, 2, V, C.c_void_p(bad.data_ptr()), C.c_void_p(o.data_ptr()), stream) == ERR_ARG
    assert lib.ctb_token_logprobs(C.c_void_p(zd.data_ptr()), 0, V, C.c_void_p(bad.data_ptr()),
                                  C.c_void_p(o.data_ptr()), stream) == ERR_ARG


# ---------------------------------------------------------------------------------------------------- L4
def test_l4_seeded_request_that_ends_empty_gives_an_empty_row():
    gpt, embed, _, _ = _model()
    s = dict(_spec(1, MIXED[1]), min_new=0)
    r = _request(embed, s)
    got, _ = _run(gpt, [r], 2, 0, logprobs=True)
    first = int(got[0][0][0, 0])
    empty = dataclasses.replace(r, eos_token=first)  # the same first step now samples EOS
    t = _request(embed, dict(_text_spec(3), min_new=0))
    tfirst = int(_run(gpt, [t], 2, 0, logprobs=True)[0][0][0][0])
    got, _ = _run(gpt, [empty, dataclasses.replace(t, eos_token=tfirst)], 2, 0, logprobs=True)
    assert got[0][3] is None and got[0][2].shape == (0, 4) and got[0][0].shape == (0, 4)
    assert got[1][3] is None and got[1][2].shape == (0,) and got[1][0].shape == (0,)


def test_l4_cancelled_request_keeps_its_prefix_and_streams_carry_prefixes():
    gpt, embed, _, _ = _model()
    specs = [_spec(i, MIXED[i % len(MIXED)]) for i in (2, 0, 1, 3)] + [_text_spec(1)]
    reqs = [_request(embed, s) for s in specs]
    full, _ = _run(gpt, reqs, 4, 0, logprobs=True)
    src, stats, requests, got = Arrivals(), ScheduleStats(), [], {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, requests, 4, CAP, logprobs=True)
        for r in reqs:
            src.submit(r)
        for poll, (_, _, ended) in enumerate(_poll_cycles(requests, dev, 8, stats=stats, source=src)):
            for i, s, n, _ in ended:
                o = dev.empty(i) if s is None else dev.harvest(s, n)
                got[next(k for k, r in enumerate(reqs) if r is requests[i])] = (o.ids[0].cpu(), o.logprobs[0].cpu())
            if poll == 2:
                src.cancel(reqs[0])
                src.close()
    ids, lp = got[0]
    n = ids.shape[0]
    assert 0 < n < full[0][0].shape[0] and lp.shape == ids.shape
    assert torch.equal(lp, full[0][2][:n])
    for k in range(1, len(reqs)):
        assert torch.equal(got[k][1], full[k][2]), k
    # streamed yields: each carries the rows of the ids it carries, a prefix of the final row
    torch.manual_seed(1234)
    finals, seen = {}, 0
    for i, o, last in gpt.generate_continuous_stream(reqs, slots=4, chunk=8, logprobs=True):
        lp = o.logprobs[0].cpu()
        assert lp.shape == o.ids[0].shape
        assert torch.equal(lp, full[i][2][: lp.shape[0]]), i
        seen += 1
        if last:
            finals[i] = lp
    assert seen > len(reqs) and all(torch.equal(finals[i], full[i][2]) for i in finals)


def test_l4_abi_refusals_leave_the_handle_usable():
    gpt, embed, _, _ = _model()
    lib = _lib.load()
    buf = torch.zeros(4, CAP, 4, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    reqs = [_request(embed, _spec(i, MIXED[i])) for i in range(3)]
    ref, _ = _run(gpt, reqs, 4, 0, logprobs=True)
    # a handle without an engine (after a static generate: the last begin was ctb_gpt_begin)
    gpt2, embed2 = _model(2, 64)[:2]
    from chattts_b200.prompts import synth_prompt_batch
    ids, mask, tmask = synth_prompt_batch([6], seed=1)
    list(gpt2.generate(embed2(ids, tmask), ids, temperature=torch.tensor([0.3] * 4), eos_token=625,
                       attention_mask=mask, max_new_token=4, show_tqdm=False, manual_seed=1))
    assert lib.ctb_gpt_engine_logprobs(gpt2._handle, C.c_void_p(buf.data_ptr()), stream) == ERR_STATE
    # null buffer, then a call after an admission, on a running engine
    torch.manual_seed(1234)
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 4, CAP, True, logprobs=True)
        assert lib.ctb_gpt_engine_logprobs(gpt._handle, None, dev.stream) == ERR_ARG
        assert lib.ctb_gpt_engine_logprobs(None, C.c_void_p(buf.data_ptr()), dev.stream) == ERR_ARG
        refused = []
        for i, slot, n in schedule(reqs, dev, 16):
            refused.append(lib.ctb_gpt_engine_logprobs(gpt._handle, C.c_void_p(buf.data_ptr()), dev.stream))
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu(), o.logprobs[0].cpu())
    assert refused and all(rc == ERR_STATE for rc in refused)
    for i in ref:
        assert torch.equal(got[i][0], ref[i][0]) and torch.equal(got[i][1], ref[i][2]), i
    assert float(buf.abs().sum()) == 0.0  # the refused buffer was never written
    _handles.pop((2, 64))


# ---------------------------------------------------------------------------------------------------- L5
def test_l5_chat_open_engine_with_logprobs():
    from chattts_b200 import Chat
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=8, max_context=256)
    p = c.InferCodeParams(manual_seed=7, max_new_token=40, min_new_token=8, show_tqdm=False)
    para = "first sentence here. second one. and a third"

    def jobs(logprobs):
        with c.open_engine(slots=8, max_new_cap=64, use_decoder=False, logprobs=logprobs) as eng:
            takes = eng.submit("several takes of this", params_infer_code=p, takes=3)
            one = eng.submit("one sentence", params_infer_code=p)
            split = eng.submit(para, params_infer_code=p, split_text=True)
            return [(j.result(timeout=300), j.logprobs) for j in (takes, one, split)]

    plain, lp = jobs(False), jobs(True)
    (tw, tl), (ow, ol), (sw, sl) = lp
    assert all(x is None for _, x in plain)
    assert all(np.array_equal(a, b) for a, b in zip(plain[0][0], tw))
    assert np.array_equal(plain[1][0], ow) and np.array_equal(plain[2][0], sw)
    assert isinstance(tl, list) and len(tl) == 3
    for w, t in zip(tw, tl):  # each take: 512 samples per token, less 256, before silence stripping
        assert t.device.type == "cpu" and t.shape[1] == 4 and 0 < t.shape[0] and w.shape[0] <= 512 * t.shape[0] - 256
    assert isinstance(ol, torch.Tensor) and ol.dim() == 2 and ol.shape[1] == 4
    from chattts_b200.core import split_sentences

    assert isinstance(sl, list) and len(sl) == len(split_sentences(para)) > 1 and all(t.dim() == 2 for t in sl)
    c.unload()
