"""Split-text synthesis on the slot engine, on the GPU: the ragged batch encode (``ctb_dvae_encode_rows``) against each
row encoded alone on both back ends, paragraphs through ``infer_continuous*(split_text=True)`` and ``ChatEngine.submit``
against ``Chat.infer`` (bit-exact on the code path; per sentence, given the engine's own speaker sample, on the hidden
path), and one ``encode_rows`` call for every reference stage ending at one poll."""
import copy
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.core import split_sentences
from chattts_b200.synth import synth_speech_like
from test_gpu_encode import _state
from test_gpu_stream import chat

pytestmark = pytest.mark.gpu
MAX_SAMPLES = 24000 * 4
ERR_ARG = -1  # CTB_ERR_ARG (include/chattts_b200.h)
_enc = {}


def _encoder(fma: bool):
    if fma not in _enc:
        import os

        from chattts_b200.decoder import AudioEncoder, pack_dvae_encoder

        cfg = Config()
        old = os.environ.get("CTB_DECODER_FMA")
        if fma:
            os.environ["CTB_DECODER_FMA"] = "1"
        try:
            _enc[fma] = AudioEncoder(cfg.dvae.encoder, cfg.dvae.decoder.idim, cfg.dvae.vq,
                                     pack_dvae_encoder(_state(), cfg.dvae.encoder, cfg.dvae.decoder.idim, cfg.dvae.vq),
                                     "cuda", max_samples=MAX_SAMPLES)
        finally:
            if fma and old is None:
                del os.environ["CTB_DECODER_FMA"]
    return _enc[fma]


# 513: the shortest legal row (F = 3, one token); odd and even frame counts; a row at max_samples
LENGTHS = [513, 767, 768, 5000, 12345, 30000, MAX_SAMPLES]


@pytest.mark.parametrize("fma", [False, True])
def test_encode_rows_equal_lone_encodes(fma):
    enc = _encoder(fma)
    wavs = [synth_speech_like(4.0, 11 + k)[:n].cuda() for k, n in enumerate(LENGTHS)]
    assert sorted({(n // 256 + 1) % 2 for n in LENGTHS}) == [0, 1]
    lone = [enc.encode(w, want_margin=True) for w in wavs]
    for order in (list(range(len(wavs))), list(reversed(range(len(wavs)))), [3, 6, 0, 5, 1, 4, 2], [0], [6, 0]):
        got = enc.encode_rows([wavs[k] for k in order], want_margin=True)
        for (ids, margin), k in zip(got, order):
            assert ids.shape == lone[k][0].shape == (4, (LENGTHS[k] // 256 + 1) // 2), (fma, order, k)
            assert torch.equal(ids, lone[k][0]), (fma, order, k)
            assert torch.equal(margin, lone[k][1]), (fma, order, k)
    plain = enc.encode_rows(wavs[:3])
    assert all(torch.equal(a, b[0]) for a, b in zip(plain, lone[:3]))
    # the lone call still works after the scratch has grown for a batch
    assert torch.equal(enc.encode(wavs[4]), lone[4][0])


def test_encode_rows_reads_rows_in_place_from_one_buffer():
    enc = _encoder(False)
    buf = torch.zeros(3, 9000, device="cuda")
    ns = [9000, 600, 4097]
    for k, n in enumerate(ns):
        buf[k, :n] = synth_speech_like(1.0, 30 + k)[:n].cuda()
    got = enc.encode_rows([buf[k, :n] for k, n in enumerate(ns)])
    for k, n in enumerate(ns):
        assert torch.equal(got[k], enc.encode(buf[k, :n].clone()))


def test_encode_rows_argument_errors():
    enc = _encoder(False)
    lib = _lib.load()
    w = synth_speech_like(1.0, 3).cuda()
    with pytest.raises(_lib.CtbError):
        enc.encode_rows([w, w[:512]])                      # n <= 512
    with pytest.raises(_lib.CtbError):
        enc.encode_rows([torch.zeros(MAX_SAMPLES + 1, device="cuda")])
    ids = torch.empty(2, 4, 100, dtype=torch.int32, device="cuda")
    ptrs = (C.c_void_p * 2)(w.data_ptr(), w.data_ptr())
    ns = (C.c_int64 * 2)(w.numel(), w.numel())
    nt = (C.c_int32 * 2)()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    T = (w.numel() // 256 + 1) // 2
    assert lib.ctb_dvae_encode_rows(enc._handle, 2, ptrs, ns, C.c_void_p(ids.data_ptr()), T - 1, nt, None,
                                    stream) == ERR_ARG                       # T_k > ids_ld
    assert lib.ctb_dvae_encode_rows(enc._handle, 0, ptrs, ns, C.c_void_p(ids.data_ptr()), 100, nt, None,
                                    stream) == ERR_ARG
    assert lib.ctb_dvae_encode_rows(enc._handle, 2, ptrs, ns, None, 100, nt, None, stream) == ERR_ARG
    nulls = (C.c_void_p * 2)(w.data_ptr(), None)
    assert lib.ctb_dvae_encode_rows(enc._handle, 2, nulls, ns, C.c_void_p(ids.data_ptr()), 100, nt, None,
                                    stream) == ERR_ARG
    big = torch.empty(2, 4, T, dtype=torch.int32, device="cuda")
    assert lib.ctb_dvae_encode_rows(enc._handle, 2, ptrs, ns, C.c_void_p(big.data_ptr()), T, nt, None, stream) == 0
    assert list(nt) == [T, T]


# ---------------------------------------------------------------------------------------------------- Chat
PARAGRAPHS = [
    "just one sentence here",
    "first of two. and the second",
    "one. two is here. three comes next. and four. five ends it",
    "line one\nline two\nline three\nline four",
]


def _params(c, k, n=24, **kw):
    return c.InferCodeParams(manual_seed=7 + k, max_new_token=n, min_new_token=n, temperature=0.3 + 0.05 * k,
                             stream_batch=16, stream_speed=6000, pass_first_n_batches=[0, 2][k % 2], show_tqdm=False,
                             **kw)


def _same(x, y, use_decoder, tag):
    assert x.shape == y.shape, (tag, x.shape, y.shape)
    if use_decoder:
        assert x.size == 0 or float(np.sqrt(np.mean((x - y) ** 2))) < 1e-4, tag
    else:
        assert np.array_equal(x, y), tag


def test_split_rule_is_infer_s():
    assert [len(split_sentences(p)) for p in PARAGRAPHS] == [1, 2, 5, 4]


def test_infer_continuous_paragraphs_equal_infer_on_the_code_path():
    c = chat()
    params = [_params(c, k) for k in range(len(PARAGRAPHS))]
    before = [copy.copy(p.__dict__) for p in params]
    got = dict(c.infer_continuous(PARAGRAPHS, params_infer_code=params, use_decoder=False, split_text=True, slots=3))
    assert [p.__dict__ for p in params] == before  # the caller's params are not modified
    for k, text in enumerate(PARAGRAPHS):
        ref = c.infer(text, split_text=True, max_split_batch=1, skip_refine_text=True, use_decoder=False,
                      params_infer_code=copy.copy(params[k]))[0]
        assert np.array_equal(got[k], ref), k


def test_paragraph_stream_equals_per_sentence_streams():
    c = chat()
    for use_decoder in (False, True):
        params = [_params(c, k) for k in range(len(PARAGRAPHS))]
        got = {k: [] for k in range(len(PARAGRAPHS))}
        with c.open_engine(slots=3, max_new_cap=64, use_decoder=use_decoder) as eng:
            jobs = [eng.submit(t, params_infer_code=p, stream=True, split_text=True) for t, p in zip(PARAGRAPHS, params)]
            for k, job in enumerate(jobs):
                got[k] = list(job)
        for k, text in enumerate(PARAGRAPHS):
            sentences = split_sentences(text)
            p = copy.copy(params[k])
            if len(sentences) > 1:
                assert jobs[k].spk_smp is not None
                p.spk_smp, p.txt_smp = jobs[k].spk_smp, sentences[0]
            else:
                assert jobs[k].spk_smp is None
            ref = [ch for s in sentences for ch in c.infer([s], stream=True, split_text=False, skip_refine_text=True,
                                                            use_decoder=use_decoder, params_infer_code=copy.copy(p))]
            assert [last for _, last in got[k]] == [False] * (len(ref) - 1) + [True], (use_decoder, k)
            for j, ((x, _), y) in enumerate(zip(got[k], ref)):
                if use_decoder and x.shape != y.shape:  # a flushed tail may keep one more or fewer near-silent sample
                    assert abs(x.shape[1] - y.shape[1]) <= 2, (k, j)
                else:
                    _same(x, y, use_decoder, (k, j))


def test_hidden_path_per_sentence_and_where_margins_are_clear():
    c = chat()
    params = [_params(c, k) for k in range(len(PARAGRAPHS))]
    with c.open_engine(slots=4, max_new_cap=64, use_decoder=True) as eng:
        jobs = [eng.submit(t, params_infer_code=p, split_text=True) for t, p in zip(PARAGRAPHS, params)]
        wavs = [j.result(timeout=600) for j in jobs]
    for k, text in enumerate(PARAGRAPHS):
        sentences = split_sentences(text)
        p = copy.copy(params[k])
        if len(sentences) > 1:
            p.spk_smp, p.txt_smp = jobs[k].spk_smp, sentences[0]
        ref = np.concatenate([c.infer([s], split_text=False, skip_refine_text=True, use_decoder=True,
                                      params_infer_code=copy.copy(p))[0] for s in sentences])
        _same(wavs[k], ref, True, k)
        if len(sentences) > 1:  # end to end with infer() where infer's own stage-0 encode has clear margins
            res = next(c._infer_code(sentences[0], False, c.device, True, copy.copy(params[k])))
            wav0 = c._decode_to_wavs(res.hiddens, True)[0]
            res.destroy()
            _, margin = c.dvae.audio_encoder.encode(torch.from_numpy(wav0), want_margin=True)
            q = copy.copy(params[k])
            full = c.infer(text, split_text=True, max_split_batch=1, skip_refine_text=True, use_decoder=True,
                           params_infer_code=q)[0]
            if float(margin.min()) > 1e-3:
                assert q.spk_smp == jobs[k].spk_smp, k
                _same(wavs[k], full, True, ("e2e", k))


def test_one_encode_rows_call_per_poll():
    c = chat()
    enc = c.dvae.audio_encoder
    calls = []
    real = enc.encode_rows

    def spy(wavs, *a, **kw):
        calls.append(len(wavs))
        return real(wavs, *a, **kw)

    enc.encode_rows = spy
    try:
        with c.open_engine(slots=4, max_new_cap=64, use_decoder=False) as eng:
            # three reference stages of the same forced length, taken at one poll (the source is held while they are
            # submitted), admitted together: they end at one poll
            with eng._source._cv:
                jobs = [eng.submit(PARAGRAPHS[2], params_infer_code=_params(c, k), split_text=True) for k in range(3)]
            [j.result(timeout=600) for j in jobs]
    finally:
        del enc.encode_rows
    assert calls == [3]


def test_open_engine_paragraphs_from_two_threads_beside_ordinary_jobs_with_cancels():
    c = chat()
    plain = ["hello there", "a somewhat longer sentence to speak", "ok"]
    pp = [_params(c, 10 + k, n=40) for k in range(len(plain))]
    lone = [c.infer([t], split_text=False, skip_refine_text=True, use_decoder=False,
                    params_infer_code=copy.copy(p))[0] for t, p in zip(plain, pp)]
    out, errors = {}, []
    with c.open_engine(slots=4, max_new_cap=64, use_decoder=False) as eng:
        def paragraphs(tag, cancel_at):
            try:
                # the streamed paragraph's sentences run 64 steps and stream from step 16, so its first chunk comes
                # while they still run
                streamed = c.InferCodeParams(manual_seed=21, max_new_token=64, min_new_token=64, stream_batch=16,
                                             stream_speed=6000, pass_first_n_batches=0, show_tqdm=False)
                jobs = [eng.submit(PARAGRAPHS[2], params_infer_code=_params(c, 2), split_text=True),
                        eng.submit(PARAGRAPHS[3], params_infer_code=streamed, split_text=True, stream=True)]
                it = iter(jobs[1])
                next(it)  # sentence 0 of the streamed paragraph has started
                if cancel_at == "stage0":
                    jobs[0].cancel()
                else:
                    jobs[1].cancel()
                out[tag] = jobs
            except Exception as e:  # pragma: no cover - reported below
                errors.append(e)

        jobs = [eng.submit(t, params_infer_code=p) for t, p in zip(plain, pp)]
        threads = [threading.Thread(target=paragraphs, args=(n, n)) for n in ("stage0", "sentences")]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=600)
        wavs = [j.result(timeout=600) for j in jobs]
    assert not errors and len(out) == 2
    assert all(j.done() for jobs in out.values() for j in jobs)
    assert out["sentences"][1].cancelled()  # its stream had started: the cancel reached a live sentence
    for k, (w, ref) in enumerate(zip(wavs, lone)):
        assert np.array_equal(w, ref), k
