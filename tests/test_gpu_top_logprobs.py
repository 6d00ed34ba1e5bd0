"""Top log-probabilities (ctb_gpt_engine_top_logprobs, ctb_token_top_logprobs, ctb_gpt_score_ex, ``top_logprobs=N``).

T1: attaching the buffers changes nothing: every request's ids, hidden states and log-probabilities are bit-equal to
the run without them (fp32 at S = 4, 24, 64; fp16 at S = 24, 64; code and text, seeded and unseeded; a paged engine
that suspends; a prefill budget chunking a 2,085-token prompt; three takes sharing one prompt key).  T2: the stand-alone
kernel against float64 log_softmax and a stable sort of the same fp32 rows.  T3: the sampled id's entry equals its
``logprobs`` value bit for bit; code rows against float64 heads applied to the harvested hidden states, text rows
against the teacher-forced float64 model.  T4: a request that ends empty, a cancelled prefix, streamed prefixes, the
ABI's refusals.  T5: ``Chat.open_engine(top_logprobs=5)``.  T6: ``GPT.score(top_logprobs=N)``."""
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
from test_gpu_logprobs import _heads64, _mix, _same, _ulp_bar

pytestmark = pytest.mark.gpu

FP16 = W16 | KV16
CAP = 90
ERR_ARG, ERR_STATE = -1, -3
# T3 bars: those of the sampled ids' log-probabilities (tests/test_gpu_logprobs.py, L3), whose arithmetic this is
CODE_BAR = 2e-5
TEXT_BAR = 1e-4
# T6 bars: the scoring pass's own (tests/test_gpu_score.py, S1)
SCORE_CODE_BAR = 1.2e-4
SCORE_TEXT_BAR = 1.5e-4
_handles = {}
_release = release_on_teardown(_handles)


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


def _drop(key):
    _handles.pop(key, None)
    gc.collect()
    torch.cuda.empty_cache()


def _run(gpt, reqs, slots, flags=0, top=0, logprobs=True, pool=None, budget=None, cap=CAP, chunk=16):
    """Every request through one engine -> ({index: (ids, hiddens, logprobs or None, (top ids, top lp) or None, slot)},
    stats).  Unseeded requests draw their Philox seeds from torch's generator, seeded here so that two runs draw the
    same ones."""
    torch.manual_seed(1234)
    got, stats = {}, ScheduleStats()
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, cap, True, flags, kv_pool_pages=pool, logprobs=logprobs, top_logprobs=top)
        for i, slot, n in schedule(reqs, dev, chunk, stats=stats, prefill_budget=budget):
            o = dev.empty(i) if slot is None else dev.harvest(slot, n)
            assert bool(o.logprobs) == logprobs and bool(o.top_logprobs) == bool(top)
            got[i] = (o.ids[0].cpu(), o.hiddens[0].cpu() if o.hiddens else None,
                      o.logprobs[0].cpu() if o.logprobs else None,
                      tuple(t.cpu() for t in o.top_logprobs[0]) if o.top_logprobs else None, slot)
            o.destroy()
    return got, stats


def _same_lp(tag, a, b):
    """T1: ids, hidden states and log-probabilities bit-equal."""
    _same(tag, a, b)
    for i in a:
        assert torch.equal(a[i][2], b[i][2]), (tag, i)


def _consistent(tag, got, N):
    """T3 / T4: shapes [n, num_vq, N] ([n, N] for text); ids distinct in each row, values non-increasing, finite and
    <= 0; where the sampled id is among the N its entry equals its log-probability bit for bit."""
    hits = 0
    for i, (ids, _, lp, (tid, tlp), _) in got.items():
        assert tid.shape == tlp.shape == (*ids.shape, N), (tag, i, tid.shape, ids.shape)
        assert tid.dtype == torch.int64 and tlp.dtype == torch.float32, (tag, i)
        if ids.numel() == 0:
            continue
        assert torch.isfinite(tlp).all() and (tlp <= 0).all(), (tag, i)
        assert (tlp[..., 1:] <= tlp[..., :-1]).all(), (tag, i)
        assert (tid.sort(-1).values.diff(dim=-1) > 0).all(), (tag, i)
        hit = tid == ids[..., None]
        assert (hit.sum(-1) <= 1).all()
        if lp is not None:
            assert torch.equal(tlp[hit], lp[hit.any(-1)]), (tag, i)
        hits += int(hit.sum())
    return hits


def _code_top_error(specs, got, heads):
    """T3 for code rows: the worst |top lp - float64 log_softmax(hidden64 @ W_head64^T)[top id]|, and the number of
    rows whose float64 top-2 margin exceeds CODE_BAR and whose entry 0 is not the float64 arg-max."""
    worst, wrong = 0.0, 0
    for i, s in enumerate(specs):
        ids, hid, _, (tid, tlp), _ = got[i]
        if s["text"] or ids.shape[0] == 0:
            continue
        h = hid.cuda().double()
        for q in range(4):
            z = h @ heads[q].t()
            ref = F.log_softmax(z, -1)
            err = (tlp[:, q].cuda().double() - ref.gather(1, tid[:, q].cuda())).abs()
            worst = max(worst, float(err.max()))
            top2 = z.topk(2, -1)
            clear = (top2.values[:, 0] - top2.values[:, 1]) > CODE_BAR
            wrong += int((clear & (top2.indices[:, 0].cpu() != tid[:, q, 0]).cuda()).sum())
    return worst, wrong


# ---------------------------------------------------------------------------------------------------- T1 / T3
@pytest.mark.parametrize("slots,flags,N", [(4, 0, 5), (24, 0, 5), (64, 0, 20), (24, FP16, 5), (64, FP16, 20)])
def test_t1_attaching_changes_nothing_and_t3_code_rows_follow_the_heads(slots, flags, N):
    gpt, embed, gs, es = _model()
    specs = _mix(66 if slots == 64 else 26)
    reqs = [_request(embed, s) for s in specs]
    base, _ = _run(gpt, reqs, slots, flags)
    got, _ = _run(gpt, reqs, slots, flags, top=N)
    _same_lp((slots, flags), got, base)
    hits = _consistent((slots, flags), got, N)
    assert hits > 0
    alone, _ = _run(gpt, reqs, slots, flags, top=N, logprobs=False)  # without logprobs: the same rows
    _same((slots, flags, "alone"), alone, base)
    for i in got:
        assert torch.equal(alone[i][3][0], got[i][3][0]) and torch.equal(alone[i][3][1], got[i][3][1]), i
    worst, wrong = _code_top_error(specs, got, _heads64(es))
    print(f"\nT3 S={slots} flags={flags} N={N}: max |top lp - float64 heads| = {worst:.3e}, sampled ids among the "
          f"top {hits}, arg-max misses {wrong}")
    assert worst < CODE_BAR and wrong == 0, (worst, wrong)


def test_t3_text_rows_follow_the_float64_model():
    gpt, embed, gs, es = _model()
    specs = [_text_spec(i) for i in range(4)] + [_spec(0, MIXED[0])]
    reqs = [_request(embed, s) for s in specs]
    N = 20
    got, _ = _run(gpt, reqs, 4, 0, top=N)
    _consistent("text", got, N)
    orc = F64Oracle(gs, es, device="cuda")
    k = "head_text.parametrizations.weight.original{}"
    head = fold_weight_norm(es[k.format(0)].double(), es[k.format(1)].double()).cuda()
    worst = 0.0
    for i in range(4):
        ids, _, _, (tid, tlp), _ = got[i]
        n, T0 = ids.shape[0], reqs[i].emb.shape[0]
        assert n > 0
        x = torch.cat([reqs[i].emb.cuda().double(), orc.emb_text[ids[: n - 1].cuda()]])
        ref = F.log_softmax(orc.forward(x)[T0 - 1:] @ head.t(), -1)
        worst = max(worst, float((tlp.cuda().double() - ref.gather(1, tid.cuda())).abs().max()))
    print(f"\nT3 text: max |top lp - teacher-forced float64| = {worst:.3e}")
    assert worst < TEXT_BAR, worst


def test_t1_paged_engine_that_suspends_keeps_the_rows_of_the_fixed_engine():
    gpt, embed, _, _ = _model()
    specs = _mix()
    reqs = [_request(embed, s) for s in specs]
    fixed, _ = _run(gpt, reqs, 24, 0, top=5)
    pool = max(2 * max(pool_pages_needed(r) for r in reqs), sum(pool_pages_needed(r) for r in reqs) // 3)
    base, _ = _run(gpt, reqs, 24, 0, pool=pool)
    got, stats = _run(gpt, reqs, 24, 0, top=5, pool=pool)
    assert stats.suspensions > 0 and stats.resumes > 0, (stats.suspensions, stats.resumes)
    _same_lp("paged", got, base)
    for i in fixed:
        assert torch.equal(got[i][3][0], fixed[i][3][0]) and torch.equal(got[i][3][1], fixed[i][3][1]), i


def test_t1_prefill_budget_chunks_a_long_prompt():
    gpt, embed, _, _ = _model(4, 2304)
    specs = [dict(_spec(0, MIXED[0]), length=2085, max_new=48, min_new=48), _spec(1, MIXED[1]), _text_spec(2),
             dict(_spec(3, MIXED[2]), length=700)]
    reqs = [_request(embed, s) for s in specs]
    whole, _ = _run(gpt, reqs, 4, 0, top=5, cap=64)
    base, _ = _run(gpt, reqs, 4, 0, budget=256, cap=64)
    got, stats = _run(gpt, reqs, 4, 0, top=5, budget=256, cap=64)
    assert stats.chunks > 2
    _same_lp("budget", got, base)
    _consistent("budget", got, 5)
    for i in whole:  # a chunked admission samples the first token from the same logits as a whole one
        assert torch.equal(got[i][3][0], whole[i][3][0]) and torch.equal(got[i][3][1], whole[i][3][1]), i
    _drop((4, 2304))


def test_t1_takes_sharing_a_prompt_key():
    gpt, embed, _, _ = _model()
    first = _request(embed, dict(_spec(0, MIXED[0]), length=300))
    reqs = [dataclasses.replace(first, manual_seed=40 + k, prompt_key="utt") for k in range(3)]
    plain = [dataclasses.replace(r, prompt_key=None) for r in reqs]
    base, _ = _run(gpt, reqs, 4, 0)
    got, stats = _run(gpt, reqs, 4, 0, top=5, chunk=4)
    ref, _ = _run(gpt, plain, 4, 0, top=5)
    assert stats.shares > 0
    _same_lp("takes", got, base)
    for i in ref:
        assert torch.equal(got[i][3][0], ref[i][3][0]) and torch.equal(got[i][3][1], ref[i][3][1]), i


# ---------------------------------------------------------------------------------------------------- T2
def _rows(V, g):
    """64 fp32 rows: ordinary, +-80, exact ties at the maximum, ties everywhere (values on a coarse grid, so tie groups
    straddle every N-th place), tie groups placed across places 1, 5 and 20, and constant rows."""
    z = torch.randn(64, V, generator=g) * 3
    z[8:16] = torch.rand(8, V, generator=g) * 160 - 80
    for r in range(16, 24):  # 5 ids tie at the maximum
        z[r, torch.randperm(V, generator=g)[:5]] = float(z[r].max()) + 1.0
    z[24:32] = (torch.randn(8, V, generator=g) * 2).round()
    for r, n in zip(range(32, 44), [1, 5, 20] * 4):  # n - 1 distinct leaders, then 4 ids tied at the n-th place
        lead = torch.randperm(V, generator=g)[: n + 3]
        top = float(z[r].max())
        z[r, lead[: n - 1]] = top + 2.0 + torch.arange(n - 1, 0, -1, dtype=torch.float32)
        z[r, lead[n - 1:]] = top + 1.0
    z[44:48] = torch.tensor([0.0, -3.5, 80.0, -80.0])[:, None]  # constant rows
    z[48, : V // 2] = -0.0  # signed zeros tie with +0.0
    z[48, V // 2:] = 0.0
    return z


@pytest.mark.parametrize("V", [626, 21178])
def test_t2_kernel_matches_float64_and_a_stable_sort(V):
    g = torch.Generator().manual_seed(V + 1)
    z = _rows(V, g)
    rows = z.shape[0]
    zd = z.cuda()
    lib = _lib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    order = torch.sort(-z, dim=1, stable=True).indices  # z descending, the smaller id first among equal z
    lsm = torch.log_softmax(z.double(), 1)
    for N in (1, 5, 20):
        outs = []
        for _ in range(2):
            ids = torch.full((rows, N), -7, dtype=torch.int32, device="cuda")
            lp = torch.full((rows, N), 7.0, device="cuda")
            _lib.check(lib.ctb_token_top_logprobs(C.c_void_p(zd.data_ptr()), rows, V, N, C.c_void_p(ids.data_ptr()),
                                                  C.c_void_p(lp.data_ptr()), stream))
            outs.append((ids, lp))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])  # the same bits
        ids, lp = outs[0][0].cpu().long(), outs[0][1].cpu()
        assert torch.equal(ids, order[:, :N]), (N, int((ids != order[:, :N]).any(1).nonzero()[0]))
        err = (lp.double() - lsm.gather(1, ids)).abs()
        bar = torch.stack([_ulp_bar(z, ids[:, k]) for k in range(N)], 1)
        print(f"\nT2 V={V} N={N}: max |lp - float64| = {float(err.max()):.3e}, max err / bar = "
              f"{float((err / bar).max()):.3f}")
        assert (err <= bar).all(), (N, float((err / bar).max()))
        # each entry is ctb_token_logprobs' value for its id, bit for bit
        for k in range(N):
            one = torch.empty(rows, device="cuda")
            kid = outs[0][0][:, k].contiguous()
            _lib.check(lib.ctb_token_logprobs(C.c_void_p(zd.data_ptr()), rows, V, C.c_void_p(kid.data_ptr()),
                                              C.c_void_p(one.data_ptr()), stream))
            assert torch.equal(one.cpu(), lp[:, k]), (N, k)
    # refusals
    ids = torch.zeros(rows, 20, dtype=torch.int32, device="cuda")
    lp = torch.zeros(rows, 20, device="cuda")
    args = (C.c_void_p(ids.data_ptr()), C.c_void_p(lp.data_ptr()), stream)
    for N in (0, 21, -1):
        assert lib.ctb_token_top_logprobs(C.c_void_p(zd.data_ptr()), rows, V, N, *args) == ERR_ARG
    assert lib.ctb_token_top_logprobs(None, rows, V, 5, *args) == ERR_ARG
    assert lib.ctb_token_top_logprobs(C.c_void_p(zd.data_ptr()), rows, V, 5, None, args[1], stream) == ERR_ARG
    assert lib.ctb_token_top_logprobs(C.c_void_p(zd.data_ptr()), 0, V, 5, *args) == ERR_ARG
    assert lib.ctb_token_top_logprobs(C.c_void_p(zd.data_ptr()), rows, 4, 5, *args) == ERR_ARG  # V < N


# ---------------------------------------------------------------------------------------------------- T4
def test_t4_seeded_request_that_ends_empty_gives_an_empty_row():
    gpt, embed, _, _ = _model()
    r = _request(embed, dict(_spec(1, MIXED[1]), min_new=0))
    first = int(_run(gpt, [r], 2, 0, top=5)[0][0][0][0, 0])
    t = _request(embed, dict(_text_spec(3), min_new=0))
    tfirst = int(_run(gpt, [t], 2, 0, top=5)[0][0][0][0])
    got, _ = _run(gpt, [dataclasses.replace(r, eos_token=first), dataclasses.replace(t, eos_token=tfirst)], 2, 0, top=5)
    assert got[0][4] is None and got[0][3][0].shape == got[0][3][1].shape == (0, 4, 5)
    assert got[1][4] is None and got[1][3][0].shape == got[1][3][1].shape == (0, 5)


def test_t4_cancelled_request_keeps_its_prefix_and_streams_carry_prefixes():
    gpt, embed, _, _ = _model()
    specs = [_spec(i, MIXED[i % len(MIXED)]) for i in (2, 0, 1, 3)] + [_text_spec(1)]
    reqs = [_request(embed, s) for s in specs]
    full, _ = _run(gpt, reqs, 4, 0, top=5)
    src, stats, requests, got = Arrivals(), ScheduleStats(), [], {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, requests, 4, CAP, top_logprobs=5)
        for r in reqs:
            src.submit(r)
        for poll, (_, _, ended) in enumerate(_poll_cycles(requests, dev, 8, stats=stats, source=src)):
            for i, s, n, _ in ended:
                o = dev.empty(i) if s is None else dev.harvest(s, n)
                got[next(k for k, r in enumerate(reqs) if r is requests[i])] = (
                    o.ids[0].cpu(), tuple(t.cpu() for t in o.top_logprobs[0]))
            if poll == 2:
                src.cancel(reqs[0])
                src.close()
    ids, (tid, tlp) = got[0]
    n = ids.shape[0]
    assert 0 < n < full[0][0].shape[0] and tid.shape == (n, 4, 5)
    assert torch.equal(tid, full[0][3][0][:n]) and torch.equal(tlp, full[0][3][1][:n])
    for k in range(1, len(reqs)):
        assert torch.equal(got[k][1][0], full[k][3][0]) and torch.equal(got[k][1][1], full[k][3][1]), k
    # streamed yields: each carries the rows of the ids it carries, a prefix of the final rows
    torch.manual_seed(1234)
    seen = 0
    held = []  # earlier yields' rows must stay as they were handed out
    for i, o, last in gpt.generate_continuous_stream(reqs, slots=4, chunk=8, top_logprobs=5):
        tid, tlp = o.top_logprobs[0]
        m = tid.shape[0]
        assert tid.shape[:-1] == o.ids[0].shape
        assert torch.equal(tid.cpu(), full[i][3][0][:m]) and torch.equal(tlp.cpu(), full[i][3][1][:m]), i
        held.append((i, m, tid, tlp))
        seen += 1
    assert seen > len(reqs)
    for i, m, tid, tlp in held:
        assert torch.equal(tid.cpu(), full[i][3][0][:m]) and torch.equal(tlp.cpu(), full[i][3][1][:m]), i


def test_t4_abi_refusals_leave_the_handle_usable():
    gpt, embed, _, _ = _model()
    lib = _lib.load()
    ids_buf = torch.zeros(4, CAP, 4, 5, dtype=torch.int32, device="cuda")
    lp_buf = torch.zeros(4, CAP, 4, 5, device="cuda")
    bufs = (C.c_void_p(ids_buf.data_ptr()), C.c_void_p(lp_buf.data_ptr()))
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    reqs = [_request(embed, _spec(i, MIXED[i])) for i in range(3)]
    ref, _ = _run(gpt, reqs, 4, 0, top=5)
    # a handle without an engine (after a static generate)
    gpt2, embed2 = _model(2, 64)[:2]
    from chattts_b200.prompts import synth_prompt_batch
    ids, mask, tmask = synth_prompt_batch([6], seed=1)
    list(gpt2.generate(embed2(ids, tmask), ids, temperature=torch.tensor([0.3] * 4), eos_token=625,
                       attention_mask=mask, max_new_token=4, show_tqdm=False, manual_seed=1))
    assert lib.ctb_gpt_engine_top_logprobs(gpt2._handle, 5, *bufs, stream) == ERR_STATE
    torch.manual_seed(1234)
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 4, CAP, True, top_logprobs=5)
        for N in (0, 21):
            assert lib.ctb_gpt_engine_top_logprobs(gpt._handle, N, *bufs, dev.stream) == ERR_ARG
        assert lib.ctb_gpt_engine_top_logprobs(gpt._handle, 5, None, bufs[1], dev.stream) == ERR_ARG
        assert lib.ctb_gpt_engine_top_logprobs(gpt._handle, 5, bufs[0], None, dev.stream) == ERR_ARG
        assert lib.ctb_gpt_engine_top_logprobs(None, 5, *bufs, dev.stream) == ERR_ARG
        refused = []
        for i, slot, n in schedule(reqs, dev, 16):
            refused.append(lib.ctb_gpt_engine_top_logprobs(gpt._handle, 5, *bufs, dev.stream))
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu(), tuple(t.cpu() for t in o.top_logprobs[0]))
    assert refused and all(rc == ERR_STATE for rc in refused)
    for i in ref:
        assert torch.equal(got[i][0], ref[i][0]), i
        assert torch.equal(got[i][1][0], ref[i][3][0]) and torch.equal(got[i][1][1], ref[i][3][1]), i
    assert int(ids_buf.abs().sum()) == 0 and float(lp_buf.abs().sum()) == 0.0  # the refused buffers were never written
    _drop((2, 64))


# ---------------------------------------------------------------------------------------------------- T5
def test_t5_chat_open_engine_with_top_logprobs():
    from chattts_b200 import Chat
    from chattts_b200.core import split_sentences
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=8, max_context=256)
    p = c.InferCodeParams(manual_seed=7, max_new_token=40, min_new_token=8, show_tqdm=False)
    para = "first sentence here. second one. and a third"

    def jobs(top):
        with c.open_engine(slots=8, max_new_cap=64, use_decoder=False, top_logprobs=top) as eng:
            takes = eng.submit("several takes of this", params_infer_code=p, takes=3)
            one = eng.submit("one sentence", params_infer_code=p)
            split = eng.submit(para, params_infer_code=p, split_text=True)
            return [(j.result(timeout=300), j.top_logprobs, j.logprobs) for j in (takes, one, split)]

    plain, top = jobs(0), jobs(5)
    assert all(x is None for _, x, _ in plain) and all(x is None for _, _, x in top)
    assert all(np.array_equal(a, b) for a, b in zip(plain[0][0], top[0][0]))
    assert np.array_equal(plain[1][0], top[1][0]) and np.array_equal(plain[2][0], top[2][0])
    (tw, tl, _), (_, ol, _), (_, sl, _) = top
    assert isinstance(tl, list) and len(tl) == 3
    for w, (i, v) in zip(tw, tl):
        assert i.device.type == v.device.type == "cpu" and i.shape == v.shape and i.shape[1:] == (4, 5)
        assert 0 < i.shape[0] and w.shape[0] <= 512 * i.shape[0] - 256
    assert isinstance(ol, tuple) and ol[0].shape[1:] == (4, 5) and ol[0].dtype == torch.int64
    assert isinstance(sl, list) and len(sl) == len(split_sentences(para)) > 1
    assert all(i.dim() == 3 and i.shape == v.shape for i, v in sl)
    c.unload()


# ---------------------------------------------------------------------------------------------------- T6
def _f64_rows(orc, prompt, ids, text):
    """The float64 teacher-forced model's log_softmax rows at each given token: [n, 4, V] or [n, V]."""
    n, P = int(ids.shape[0]), int(prompt.shape[0])
    ids = ids.cuda().long()
    prev = orc.emb_text[ids[: n - 1]] if text else orc.embed_codes(ids[: n - 1])
    hid = orc.forward(torch.cat([prompt.cuda().double(), prev]))[P - 1:]
    return F.log_softmax(hid @ orc.head_text.t() if text else orc.logits_rows(hid), -1)


def test_t6_scoring_with_top_logprobs():
    from chattts_b200.prompts import synth_prompt_batch

    gpt, embed, gs, es = _model(32, 1280)
    orc = F64Oracle(gs, es, device="cuda")
    k = "head_text.parametrizations.weight.original{}"
    orc.head_text = fold_weight_norm(es[k.format(0)].double(), es[k.format(1)].double()).cuda()

    def prompt(P, seed):
        ids, _, tmask = synth_prompt_batch([P], seed=seed)
        return embed(ids, tmask)[0]

    for text, bar in ((False, SCORE_CODE_BAR), (True, SCORE_TEXT_BAR)):
        V = 21178 if text else 626
        prompts = [prompt(P, 60 + i) for i, P in enumerate([8, 300, 57, 1000])]
        ns = [1, 200, 37, 150]  # the last row is over 1,024 columns: tiled attention
        g = torch.Generator().manual_seed(7 + text)
        targets = [torch.randint(0, V, (n,) if text else (n, 4), generator=g) for n in ns]
        # make some given tokens the model's own first choices, so that they appear in their top N
        plain = gpt.score(prompts, targets, infer_text=text)
        N = 20 if text else 5
        rows = gpt.score(prompts, targets, infer_text=text, top_logprobs=N)
        first = gpt.score(prompts, targets, infer_text=text, top_logprobs=N)
        hits, worst = 0, 0.0
        for r, (lp, tid, tlp) in enumerate(rows):
            assert torch.equal(lp, plain[r]), (text, r)
            assert torch.equal(tid, first[r][1]) and torch.equal(tlp, first[r][2])  # the same bits
            assert tid.shape == tlp.shape == (*targets[r].shape, N) and tid.dtype == torch.int64
            ref = _f64_rows(orc, prompts[r], targets[r], text)
            worst = max(worst, float((tlp.double() - ref.gather(-1, tid)).abs().max()))
            hit = tid == targets[r].cuda()[..., None]
            assert torch.equal(tlp[hit], lp[hit.any(-1)]), (text, r)
            hits += int(hit.sum())
        # tokens chosen as their position's own entry 0 are in their top N by construction
        forced = [rows[r][1][..., 0].cpu() for r in range(len(rows))]
        again = gpt.score(prompts, forced, infer_text=text, top_logprobs=N)
        for r, (lp, tid, tlp) in enumerate(again):
            if ns[r] == 1:  # a one-token row has no earlier token: the same distribution as before
                assert torch.equal(tid[0, ..., 0], forced[r][0].cuda())
            hit = tid == forced[r].cuda()[..., None]
            assert torch.equal(tlp[hit], lp[hit.any(-1)]), (text, r)
            hits += int(hit.sum())
        print(f"\nT6 {'text' if text else 'code'} N={N}: max |top lp - float64| = {worst:.3e}, given tokens in "
              f"their top N {hits}")
        assert worst < bar, (text, worst)
        assert hits > 0
    _drop((32, 1280))
