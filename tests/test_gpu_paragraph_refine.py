"""Refined split-text paragraphs on the slot engine, on the GPU: a request with ``noise_batch=(B, b)`` samples exactly
as row b of a seeded static ``GPT.generate`` batch of B (text and codes, every static back end B selects), and
``ChatEngine.submit(split_text=True, skip_refine_text=False, max_split_batch=m)`` equals ``Chat.infer`` (bit for bit on
the code path; per sentence, given the engine's own speaker sample and refined sentences, on the hidden path), with
streams, the ``infer_continuous*`` entry points, and cancels in every phase from two threads beside ordinary jobs."""
import copy
import random
import threading
import time

import numpy as np
import pytest
import torch

from chattts_b200.core import split_sentences
from chattts_b200.engine import Request
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from test_gpu_paragraph import PARAGRAPHS
from test_gpu_stream import chat

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- noise_batch
def _static_rows(gpt, embed, B, text, seed):
    """A seeded, ragged static batch of B and one engine request per row with noise_batch=(B, b)."""
    g = np.random.default_rng(seed)
    lengths = [int(x) for x in g.integers(3, 41, B)]
    ids, mask, tmask = synth_prompt_batch(lengths, seed=seed)
    emb = embed(ids, tmask)
    if text:
        warp, proc = gen_logits(num_code=21178, top_P=0.7, top_K=20, repetition_penalty=1.05)
        temp, eos, max_new, min_new = [1.2], 21001, 30, 1
    else:
        warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
        temp, eos, max_new, min_new = [1.2] * 4, 625, 40, 2
    procs = (*proc, *warp)
    out = next(gpt.generate(emb, ids, temperature=torch.tensor(temp), eos_token=eos, attention_mask=mask,
                            max_new_token=max_new, min_new_token=min_new, logits_processors=procs, infer_text=text,
                            return_hidden=not text, show_tqdm=False, manual_seed=seed))
    reqs = [Request(emb=emb[b][mask[b].to(emb.device)], temperature=temp, eos_token=eos, max_new_token=max_new,
                    min_new_token=min_new, logits_processors=procs, manual_seed=seed, infer_text=text,
                    noise_batch=(B, b)) for b in range(B)]
    return out, reqs


@pytest.mark.parametrize("slots", [3, 12])
def test_noise_batch_rows_equal_the_static_batch(slots):
    from gpu_util import build_gpt

    gpt, embed, _, _ = build_gpt()
    static, reqs = [], []
    for B in (3, 5, 12):
        for text in (False, True):
            out, rs = _static_rows(gpt, embed, B, text, seed=700 + 10 * B + text)
            assert len({int(r.emb.shape[0]) for r in rs}) > 1, (B, text)  # ragged prompts
            static += [(out, b, text) for b in range(B)]
            reqs += rs
    order = list(range(len(reqs)))
    random.Random(slots).shuffle(order)
    got = dict(gpt.generate_continuous([reqs[i] for i in order], slots=slots, chunk=8))
    for j, i in enumerate(order):
        out, b, text = static[i]
        assert torch.equal(got[j].ids[0].cpu(), out.ids[b].cpu()), (slots, i)
        if not text:
            assert float((got[j].hiddens[0] - out.hiddens[b]).abs().max()) < 1e-4, (slots, i)


# ---------------------------------------------------------------------------------------------------- Chat
def _params(c, k, n=24, **kw):
    return c.InferCodeParams(manual_seed=7 + k, max_new_token=n, min_new_token=n, temperature=0.3 + 0.05 * k,
                             stream_batch=16, stream_speed=6000, pass_first_n_batches=[0, 2][k % 2], show_tqdm=False,
                             **kw)


def _refine(c, k, n=12):
    return c.RefineTextParams(manual_seed=50 + k, max_new_token=n, min_new_token=n, temperature=0.7 + 0.1 * (k % 3),
                              repetition_penalty=[1.0, 1.05][k % 2], show_tqdm=False)


def _same(x, y, use_decoder, tag):
    assert x.shape == y.shape, (tag, x.shape, y.shape)
    if use_decoder:
        assert x.size == 0 or float(np.sqrt(np.mean((x - y) ** 2))) < 1e-4, tag
    else:
        assert np.array_equal(x, y), tag


_runs = {}


def _engine_run(m, use_decoder=False, skip_refine_text=False):
    """Every paragraph through ChatEngine.submit on one engine of 3 slots -> (jobs, results)."""
    key = (m, use_decoder, skip_refine_text)
    if key not in _runs:
        c = chat()
        params = [_params(c, k) for k in range(len(PARAGRAPHS))]
        refine = [_refine(c, k) for k in range(len(PARAGRAPHS))]
        before = [copy.copy(p.__dict__) for p in params]
        with c.open_engine(slots=3, max_new_cap=64, use_decoder=use_decoder) as eng:
            jobs = [eng.submit(t, params_infer_code=p, split_text=True, skip_refine_text=skip_refine_text,
                               params_refine_text=r, max_split_batch=m)
                    for t, p, r in zip(PARAGRAPHS, params, refine)]
            wavs = [j.result(timeout=600) for j in jobs]
            assert eng._requests.held() == 0
        assert [p.__dict__ for p in params] == before  # the caller's params are not modified
        _runs[key] = (jobs, wavs, params, refine)
    return _runs[key]


@pytest.mark.parametrize("m", [1, 4])
def test_refined_paragraphs_equal_infer_on_the_code_path(m):
    c = chat()
    jobs, wavs, params, refine = _engine_run(m)
    for k, text in enumerate(PARAGRAPHS):
        ref = c.infer(text, use_decoder=False, max_split_batch=m, params_refine_text=refine[k],
                      params_infer_code=copy.copy(params[k]))[0]
        assert np.array_equal(wavs[k], ref), (m, k)
        refined = c.infer(text, refine_text_only=True, params_refine_text=refine[k]).split("\n")
        assert jobs[k].refined == refined, (m, k)
        assert (jobs[k].spk_smp is None) == (len(split_sentences(text)) == 1)


def test_unrefined_paragraphs_with_max_split_batch_equal_infer():
    c = chat()
    jobs, wavs, params, _ = _engine_run(4, skip_refine_text=True)
    for k, text in enumerate(PARAGRAPHS):
        ref = c.infer(text, skip_refine_text=True, max_split_batch=4, use_decoder=False,
                      params_infer_code=copy.copy(params[k]))[0]
        assert np.array_equal(wavs[k], ref), k
        assert jobs[k].refined is None


@pytest.mark.parametrize("m", [1, 4])
def test_hidden_path_per_sentence(m):
    c = chat()
    jobs, wavs, params, _ = _engine_run(m, use_decoder=True)
    for k, text in enumerate(PARAGRAPHS):
        refined = jobs[k].refined
        assert len(refined) == len(split_sentences(text)) and all(isinstance(t, str) for t in refined)
        p = copy.copy(params[k])
        if len(refined) > 1:
            p.spk_smp, p.txt_smp = jobs[k].spk_smp, refined[0]
        # infer's code batches of m, given the engine's sample and refined sentences
        ref = np.concatenate([w for lo in range(0, len(refined), m)
                              for w in c.infer(refined[lo: lo + m], split_text=False, skip_refine_text=True,
                                               use_decoder=True, params_infer_code=copy.copy(p))])
        _same(wavs[k], ref, True, (m, k))


def test_infer_continuous_and_its_stream_agree_with_submit():
    c = chat()
    jobs, wavs, params, refine = _engine_run(4)
    got = dict(c.infer_continuous(PARAGRAPHS, params_infer_code=params, params_refine_text=refine, use_decoder=False,
                                  split_text=True, skip_refine_text=False, max_split_batch=4, slots=3))
    assert sorted(got) == list(range(len(PARAGRAPHS)))
    for k in range(len(PARAGRAPHS)):
        assert np.array_equal(got[k], wavs[k]), k
    chunks = {k: [] for k in range(len(PARAGRAPHS))}
    for k, ch, last in c.infer_continuous_stream(PARAGRAPHS, params_infer_code=params, params_refine_text=refine,
                                                 use_decoder=False, split_text=True, skip_refine_text=False,
                                                 max_split_batch=4, slots=3):
        chunks[k].append((ch, last))
    with c.open_engine(slots=3, max_new_cap=64, use_decoder=False) as eng:
        sjobs = [eng.submit(t, params_infer_code=p, stream=True, split_text=True, skip_refine_text=False,
                            params_refine_text=r, max_split_batch=4) for t, p, r in zip(PARAGRAPHS, params, refine)]
        streamed = [list(j) for j in sjobs]
    for k, text in enumerate(PARAGRAPHS):
        assert [l for _, l in chunks[k]] == [False] * (len(chunks[k]) - 1) + [True], k
        assert len(streamed[k]) == len(chunks[k]) and all(
            np.array_equal(x, y) and a == b for (x, a), (y, b) in zip(streamed[k], chunks[k])), k


def test_streamed_refined_paragraph_is_each_sentence_s_stream_in_order():
    c = chat()
    jobs, _, params, refine = _engine_run(1)
    with c.open_engine(slots=3, max_new_cap=64, use_decoder=False) as eng:
        sjobs = [eng.submit(t, params_infer_code=p, stream=True, split_text=True, skip_refine_text=False,
                            params_refine_text=r) for t, p, r in zip(PARAGRAPHS, params, refine)]
        streamed = [list(j) for j in sjobs]
    for k, text in enumerate(PARAGRAPHS):
        refined = sjobs[k].refined
        assert refined == jobs[k].refined and sjobs[k].spk_smp == jobs[k].spk_smp, k
        p = copy.copy(params[k])
        if len(refined) > 1:
            p.spk_smp, p.txt_smp = sjobs[k].spk_smp, refined[0]
        ref = [ch for s in refined for ch in c.infer([s], stream=True, split_text=False, skip_refine_text=True,
                                                        use_decoder=False, params_infer_code=copy.copy(p))]
        assert [last for _, last in streamed[k]] == [False] * (len(ref) - 1) + [True], k
        for j, ((x, _), y) in enumerate(zip(streamed[k], ref)):
            _same(x, y, False, (k, j))


def test_refined_paragraphs_from_two_threads_beside_ordinary_jobs_with_cancels():
    c = chat()
    plain = ["hello there", "a somewhat longer sentence to speak", "ok"]
    pp = [_params(c, 10 + k, n=40) for k in range(len(plain))]
    lone = [c.infer([t], split_text=False, skip_refine_text=True, use_decoder=False,
                    params_infer_code=copy.copy(p))[0] for t, p in zip(plain, pp)]
    out, errors = {}, []

    def wait(cond, limit=120.0):
        t0 = time.perf_counter()
        while not cond() and time.perf_counter() - t0 < limit:
            time.sleep(0.002)

    with c.open_engine(slots=4, max_new_cap=64, use_decoder=False) as eng:
        def paragraphs(tag):
            try:
                long_refine = _refine(c, 3, n=48)
                jobs = {phase: eng.submit(PARAGRAPHS[2], params_infer_code=_params(c, 2, n=64), split_text=True,
                                          skip_refine_text=False, params_refine_text=long_refine, max_split_batch=4)
                        for phase in ("refinement", "reference", "code")}
                jobs["refinement"].cancel()
                j = jobs["reference"]
                wait(lambda: j.done() or j.refined[0] is not None)
                j.cancel()
                j = jobs["code"]
                wait(lambda: j.done() or j.spk_smp is not None)
                j.cancel()
                kept = eng.submit(PARAGRAPHS[1], params_infer_code=_params(c, 1), split_text=True,
                                  skip_refine_text=False, params_refine_text=_refine(c, 1), max_split_batch=4)
                out[tag] = (jobs, kept.result(timeout=600))
            except Exception as e:  # pragma: no cover - reported below
                errors.append(e)

        jobs = [eng.submit(t, params_infer_code=p) for t, p in zip(plain, pp)]
        threads = [threading.Thread(target=paragraphs, args=(n,)) for n in ("a", "b")]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=600)
        wavs = [j.result(timeout=600) for j in jobs]
    assert not errors and len(out) == 2
    assert eng._requests.held() == 0 and not eng._pending
    ref = c.infer(PARAGRAPHS[1], use_decoder=False, max_split_batch=4, params_refine_text=_refine(c, 1),
                  params_infer_code=_params(c, 1))[0]
    for jobs_, kept in out.values():
        assert all(j.done() for j in jobs_.values())
        assert jobs_["refinement"].cancelled()
        assert np.array_equal(kept, ref)
    for k, (w, r) in enumerate(zip(wavs, lone)):
        assert np.array_equal(w, r), k
