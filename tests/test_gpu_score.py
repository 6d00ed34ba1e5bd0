"""Teacher-forced scoring (``GPT.score``, ``Chat.score``, ctb_gpt_score) on one H100.

S1: code and text rows against the float64 teacher-forced model: a ragged batch, a row of more than 1,024 columns
(tiled attention), a row that fills ``max_context``, targets that include EOS.  S2: ids the fp32 slot engine sampled
with ``logprobs=True`` score to its log-probabilities, and ids of static ``generate`` at B = 1 and 24 score to the
float64 model.  S3: bit-reproducible, and a row scored alone agrees with the same row in a batch.  S4: the handle's
state around a score.  S5: ``Chat.score`` against ``Chat.open_engine(logprobs=True)``, and a recording's codes."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from chattts_b200 import _lib
from chattts_b200.engine import Request
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from f64_oracle import F64Oracle
import gpu_util
from gpu_util import build_gpt, release_on_teardown
from oracle.gpt_oracle import fold_weight_norm

pytestmark = pytest.mark.gpu

MAX_CONTEXT = 1280
EOS = 625
ERR_ARG, ERR_STATE = -1, -3
# S1 bars (DESIGN.md §4 "Scoring given tokens").  CPU evaluations of the same rows in fp32 and with 3xTF32 GEMMs came
# within 1.6e-6 of float64, but the device pass showed up to 3.6e-5 (code) and 4.7e-5 (text) on one H100; the bars are
# about 3x those observed maxima
CODE_BAR = 1.2e-4
TEXT_BAR = 1.5e-4
# the slot engine's own bar against the teacher-forced float64 model (tests/test_gpu_logprobs.py, text rows)
ENGINE_BAR = 1e-4
_cache = {}
_release = release_on_teardown(_cache)


def _model(max_batch=32):
    """The synthetic model of ``build_gpt`` on a handle this module owns: it leaves the shared cache, so that its
    device memory (the weights' copies, an engine's KV pool and the scoring scratch) is freed with ``_cache``."""
    key = ("model", max_batch)
    if key not in _cache:
        m = build_gpt(max_batch=max_batch, max_context=MAX_CONTEXT)
        for k in [k for k, v in gpu_util._cache.items() if v is m]:
            del gpu_util._cache[k]
        _cache[key] = m
    return _cache[key]


def _oracle():
    if "orc" not in _cache:
        _, _, gs, es = _model()
        orc = F64Oracle(gs, es, device="cuda")
        k = "head_text.parametrizations.weight.original{}"
        orc.head_text = fold_weight_norm(es[k.format(0)].double(), es[k.format(1)].double()).cuda()
        _cache["orc"] = orc
    return _cache["orc"]


def _prompt(embed, P, seed):
    ids, _, tmask = synth_prompt_batch([P], seed=seed)
    return embed(ids, tmask)[0]


def _codes(n, seed, eos_at=None):
    t = torch.randint(0, EOS + 1, (n, 4), generator=torch.Generator().manual_seed(seed))
    if eos_at is not None:
        t[eos_at] = EOS
    return t


def _text(n, seed):
    return torch.randint(0, 21178, (n,), generator=torch.Generator().manual_seed(seed))


def _f64(prompt, ids, text=False):
    """log softmax of the float64 teacher-forced model's logits at each given token: [n, 4] or [n]."""
    orc = _oracle()
    n, P = int(ids.shape[0]), int(prompt.shape[0])
    ids = ids.cuda().long()
    prev = orc.emb_text[ids[: n - 1]] if text else orc.embed_codes(ids[: n - 1])
    hid = orc.forward(torch.cat([prompt.cuda().double(), prev]))[P - 1:]
    if text:
        return F.log_softmax(hid @ orc.head_text.t(), -1).gather(1, ids[:, None])[:, 0]
    return F.log_softmax(orc.logits_rows(hid), -1).gather(2, ids[:, :, None])[..., 0]


def _err(got, prompt, ids, text=False):
    assert got.shape == ids.shape and got.dtype == torch.float32 and torch.isfinite(got).all()
    return float((got.double() - _f64(prompt, ids, text)).abs().max())


def test_s1_code_rows_against_float64():
    gpt, embed, _, _ = _model()
    Ps, ns = [8, 300, 57, 120, 13], [1, 400, 37, 200, 90]
    prompts = [_prompt(embed, P, 10 + i) for i, P in enumerate(Ps)]
    ids = [_codes(n, 20 + i, eos_at=n - 1 if i % 2 else None) for i, n in enumerate(ns)]
    long_p, long_ids = _prompt(embed, 1000, 31), _codes(150, 32, eos_at=149)        # 1,149 columns: tiled attention
    full_p, full_ids = _prompt(embed, 900, 33), _codes(MAX_CONTEXT - 899, 34)       # fills max_context
    got = gpt.score(prompts + [long_p, full_p], ids + [long_ids, full_ids])
    errs = [_err(g, p, i) for g, p, i in zip(got, prompts + [long_p, full_p], ids + [long_ids, full_ids])]
    print(f"\nS1 code: max |lp - float64| per row = {['%.2e' % e for e in errs]}")
    assert max(errs) < CODE_BAR, errs


def test_s1_text_rows_against_float64():
    gpt, embed, _, _ = _model()
    prompts = [_prompt(embed, 40, 40), _prompt(embed, 9, 41), _prompt(embed, 200, 42)]
    ids = [_text(80, 43), _text(1, 44), _text(300, 45)]
    ids[0][-1] = 21001  # the text EOS
    got = gpt.score(prompts, ids, infer_text=True)
    errs = [_err(g, p, i, text=True) for g, p, i in zip(got, prompts, ids)]
    print(f"\nS1 text: max |lp - float64| per row = {['%.2e' % e for e in errs]}")
    assert max(errs) < TEXT_BAR, errs


def _requests(embed, n, text=False, max_new=None):
    out = []
    for i in range(n):
        V = 21178 if text else 625
        warp, proc = gen_logits(num_code=V, top_P=0.7, top_K=20, repetition_penalty=1.05)
        out.append(Request(emb=_prompt(embed, 10 + 7 * i, 500 + i), temperature=[0.7] if text else [0.7] * 4,
                           eos_token=21001 if text else EOS, max_new_token=max_new[i] if max_new else 60,
                           min_new_token=max_new[i] if max_new else 8 + (i % 5) * 10,
                           logits_processors=(*proc, *warp), manual_seed=900 + i, infer_text=text))
    return out


@pytest.mark.parametrize("slots", [4, 24])
def test_s2_engine_logprobs(slots):
    gpt, embed, _, _ = _model()
    reqs = _requests(embed, slots + 2) + _requests(embed, 2, text=True)
    worst = {False: 0.0, True: 0.0}
    outs = dict(gpt.generate_continuous(reqs, slots=slots, logprobs=True))
    for text in (False, True):
        idx = [i for i, r in enumerate(reqs) if r.infer_text == text and outs[i].ids[0].shape[0] > 0]
        got = gpt.score([reqs[i].emb for i in idx], [outs[i].ids[0] for i in idx], infer_text=text)
        for i, g in zip(idx, got):
            worst[text] = max(worst[text], float((g.cpu().double() - outs[i].logprobs[0].cpu().double()).abs().max()))
    print(f"\nS2 S={slots}: max |score - engine logprobs| code {worst[False]:.2e} text {worst[True]:.2e}")
    assert worst[False] < CODE_BAR + ENGINE_BAR and worst[True] < TEXT_BAR + ENGINE_BAR, worst


@pytest.mark.parametrize("B", [1, 24])
def test_s2_static_generate_ids(B):
    gpt, embed, _, _ = _model()
    T0 = 30
    prompts = [_prompt(embed, T0, 600 + b) for b in range(B)]
    emb = torch.stack(prompts)
    (out,) = list(gpt.generate(emb, torch.zeros(B, T0, 4, dtype=torch.long), torch.tensor([0.7] * 4), EOS,
                               max_new_token=80, min_new_token=30, show_tqdm=False, manual_seed=77))
    got = gpt.score(prompts, out.ids)
    errs = [_err(g, p, i) for g, p, i in zip(got, prompts, out.ids)]
    print(f"\nS2 generate B={B}: max |lp - float64| = {max(errs):.2e}")
    assert max(errs) < CODE_BAR, errs


def test_s3_deterministic_and_independent_of_grouping():
    gpt, embed, _, _ = _model()
    prompts = [_prompt(embed, P, 70 + i) for i, P in enumerate([20, 150, 1050, 64])]
    ids = [_codes(n, 80 + i) for i, n in enumerate([50, 7, 120, 300])]
    a, b = gpt.score(prompts, ids), gpt.score(prompts, ids)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    alone = [gpt.score([p], [i])[0] for p, i in zip(prompts, ids)]
    diff = [float((x - y).abs().max()) for x, y in zip(a, alone)]
    print(f"\nS3 batch vs alone: max |diff| per row = {diff}, bit-equal: {[torch.equal(x, y) for x, y in zip(a, alone)]}")
    assert max(diff) < CODE_BAR, diff


def _lib_score(gpt, prompt, ids, targets=None):
    """ctb_gpt_score on one code row given ``ids`` (``targets``: other ids to score at the same columns) -> (rc, out)."""
    P, n = int(prompt.shape[0]), int(ids.shape[0])
    T = max(8, P + n - 1)
    emb = torch.zeros(1, T, 768, device="cuda")
    emb[0, T - (P + n - 1): T - n + 1] = prompt
    if n > 1:
        emb[0, T - n + 1:] = gpt.embed_prompt(ids[: n - 1][None].cuda(), torch.zeros(1, n - 1, dtype=torch.bool))[0]
    tgt = (ids if targets is None else targets).cuda().int().contiguous()
    out = torch.full(tgt.shape, 7.0, device="cuda")
    rc = _lib.load().ctb_gpt_score(gpt._handle, 1, T, C.c_void_p(emb.data_ptr()), (C.c_int32 * 1)(P),
                                   (C.c_int32 * 1)(n), C.c_void_p(tgt.data_ptr()), 0, C.c_void_p(out.data_ptr()),
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out


def test_s4_engine_refuses_and_keeps_serving():
    gpt, embed, _, _ = _model()
    reqs = _requests(embed, 6, max_new=[20, 120, 120, 120, 60, 60])  # forced lengths: slots 1-3 run past the first yield
    ref = {i: o.ids[0].cpu() for i, o in gpt.generate_continuous(reqs, slots=4, chunk=16)}
    p, ids = _prompt(embed, 20, 1), _codes(10, 2)
    gen = gpt.generate_continuous(reqs, slots=4, chunk=16)
    got, refused = {}, 0
    for i, o in gen:
        got[i] = o.ids[0].cpu()
        if len(got) == 1:  # the other slots are still running
            rc, out = _lib_score(gpt, p, ids)
            assert rc == ERR_STATE and (out == 7.0).all()
            refused += 1
    assert refused == 1 and all(torch.equal(got[i], ref[i]) for i in ref)
    with gpt.open_engine(slots=4, max_new_cap=64):
        with pytest.raises(RuntimeError, match="open engine"):
            gpt.score([p], [ids])
    assert torch.equal(gpt.score([p], [ids])[0], gpt.score([p], [ids])[0])


def test_s4_score_ends_a_static_batch_and_generate_is_unchanged():
    gpt, embed, _, _ = _model(max_batch=25)  # a handle of this test's own
    prompts = torch.stack([_prompt(embed, 40, 90 + b) for b in range(3)])

    def run():
        (o,) = list(gpt.generate(prompts, torch.zeros(3, 40, 4, dtype=torch.long), torch.tensor([0.7] * 4), EOS,
                                 max_new_token=50, min_new_token=10, show_tqdm=False, manual_seed=5,
                                 return_hidden=True))
        return [i.cpu() for i in o.ids], [h.cpu() for h in o.hiddens]

    fresh = run()
    stream = gpt.generate(prompts, torch.zeros(3, 40, 4, dtype=torch.long), torch.tensor([0.7] * 4), EOS,
                          max_new_token=200, min_new_token=100, show_tqdm=False, manual_seed=5, stream=True,
                          stream_batch=24)
    next(stream)
    gpt.score([prompts[0]], [_codes(30, 3)])
    lib, sp = _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.ctb_gpt_decode(gpt._handle, 1, sp) == ERR_STATE
    assert lib.ctb_gpt_status_query(gpt._handle, C.byref(_lib.GptStatus()), None, None, sp) == ERR_STATE
    with pytest.raises(_lib.CtbError):
        next(stream)
    after = run()
    assert all(torch.equal(a, b) for a, b in zip(fresh[0], after[0]))
    assert all(torch.equal(a, b) for a, b in zip(fresh[1], after[1]))


def test_s4_out_of_vocabulary_and_empty_rows():
    gpt, embed, _, _ = _model()
    p, ids = _prompt(embed, 25, 4), _codes(12, 5)
    with pytest.raises(ValueError):
        gpt.score([p], [torch.cat([ids[:-1], torch.tensor([[0, 1, 626, 2]])])])
    with pytest.raises(ValueError):
        gpt.score([p], [torch.tensor([21178])], infer_text=True)
    rc, good = _lib_score(gpt, p, ids)
    assert rc == 0
    bad = ids.clone()
    bad[3, 2], bad[7, 0] = 626, -1
    rc, out = _lib_score(gpt, p, ids, targets=bad)
    assert rc == 0
    nan = torch.zeros_like(out, dtype=torch.bool)
    nan[3, 2] = nan[7, 0] = True
    assert torch.isnan(out[nan]).all() and torch.equal(out[~nan], good[~nan])
    e = gpt.score([p, p], [torch.zeros(0, 4, dtype=torch.long), ids])
    assert e[0].shape == (0, 4) and torch.equal(e[1], good)
    assert gpt.score([p], [torch.zeros(0, dtype=torch.long)], infer_text=True)[0].shape == (0,)
    bad_args = [(0, 30, [25], [6]), (1, 7, [1], [1]), (1, MAX_CONTEXT + 1, [25], [6]), (1, 29, [25], [6]),
                (1, 30, [0], [6]), (1, 30, [25], [0])]
    buf = torch.zeros(1, MAX_CONTEXT + 1, 768, device="cuda")
    t = torch.zeros(64, device="cuda", dtype=torch.int32)
    for B, T, P, n in bad_args:
        rc = _lib.load().ctb_gpt_score(gpt._handle, B, T, C.c_void_p(buf.data_ptr()), (C.c_int32 * 1)(*P),
                                       (C.c_int32 * 1)(*n), C.c_void_p(t.data_ptr()), 0, C.c_void_p(buf.data_ptr()),
                                       None)
        assert rc == ERR_ARG, (B, T, P, n)


def test_s5_chat_score_matches_open_engine():
    from chattts_b200 import Chat
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=8, max_context=256)
    text = "one sentence to score"
    p = c.InferCodeParams(manual_seed=7, max_new_token=40, min_new_token=12, show_tqdm=False)
    with c.open_engine(slots=4, max_new_cap=64, use_decoder=False, logprobs=True) as eng:
        job = eng.submit(text, params_infer_code=p)
        wav = job.result(timeout=300)
        lp = job.logprobs
    req = c._code_request(c.normalizer(text, True, True, None), p)
    ((_, out),) = list(c.gpt.generate_continuous([req], slots=4, logprobs=True))
    assert out.logprobs[0].shape == lp.shape  # the same take
    (got,) = c.score([text], [out.ids[0]], params_infer_code=p)
    err = float((got.cpu().double() - lp.double()).abs().max())
    print(f"\nS5: max |Chat.score - Job.logprobs| = {err:.2e}")
    assert got.shape == lp.shape and err < CODE_BAR + ENGINE_BAR
    codes = c.dvae.sample_audio(torch.from_numpy(np.ascontiguousarray(np.asarray(wav, np.float32).reshape(-1)))).T
    (rec,) = c.score([text], [codes])
    assert rec.shape == (codes.shape[0], 4) and torch.isfinite(rec).all() and (rec <= 0).all()
    c.unload()
