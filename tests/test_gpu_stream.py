"""Streaming on the GPU: the ragged token -> waveform decode (ctb_decode_rows) against each row decoded alone, the slot
engine's streamed yields against GPT.generate(stream=True) per request, and Chat.infer_continuous_stream against
Chat.infer(stream=True) per text."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.synth import synth_dvae_state, synth_vocos_state

pytestmark = pytest.mark.gpu
CFG = Config()
ROW_TOKENS = [1, 2, 7, 100, 300]
OFFSETS = [5, 0, 311, 40, 17]


def _decoders(max_batch, max_tokens, fma=False):
    from chattts_b200.decoder import DVAE, Vocos

    old = os.environ.pop("CTB_DECODER_FMA", None)
    if fma:
        os.environ["CTB_DECODER_FMA"] = "1"  # read when the handle is created
    try:
        voc = Vocos(CFG.vocos, "cuda", max_batch=max_batch, max_tokens=max_tokens).load_state_dict(synth_vocos_state(5))
        dec = DVAE(CFG.decoder, dim=CFG.decoder.idim, device="cuda", vocos=voc, max_batch=max_batch,
                   max_tokens=max_tokens).load_state_dict(synth_dvae_state(2, CFG.decoder, CFG.decoder.idim))
        dv = DVAE(CFG.dvae.decoder, None, CFG.dvae.vq, dim=CFG.dvae.decoder.idim, device="cuda", vocos=voc,
                  max_batch=max_batch, max_tokens=max_tokens)
        dv.load_state_dict(synth_dvae_state(3, CFG.dvae.decoder, CFG.dvae.decoder.idim, CFG.dvae.vq))
    finally:
        os.environ.pop("CTB_DECODER_FMA", None)
        if old is not None:
            os.environ["CTB_DECODER_FMA"] = old
    return dec.engine, dv.engine


def _engine_buffers():
    """Rows at offsets out of strided [S, cap, C] buffers, like slices of the GPT engine's outputs."""
    g = torch.Generator(device="cuda").manual_seed(11)
    S, cap = len(ROW_TOKENS), 640
    hid = torch.randn(S, cap, 768, device="cuda", generator=g) * 0.5
    ids = torch.randint(0, 625, (S, cap, 4), device="cuda", dtype=torch.int32, generator=g)
    hrows = [hid[s, o: o + n] for s, (o, n) in enumerate(zip(OFFSETS, ROW_TOKENS))]
    crows = [ids[s, o: o + n] for s, (o, n) in enumerate(zip(OFFSETS, ROW_TOKENS))]
    return hrows, crows


@pytest.mark.parametrize("fma", [False, True])
def test_decode_rows_bit_identical_to_each_row_alone(fma):
    dec, dv = _decoders(8, 301, fma)
    hrows, crows = _engine_buffers()
    for eng, rows, kind in ((dec, hrows, 1), (dv, crows, 2)):
        got = eng.decode_rows(rows, kind)
        assert len(got) == len(rows)
        for r, w in zip(rows, got):
            alone = eng.tokens_to_wav(r[None].contiguous(), 1) if kind == 1 else eng.tokens_to_wav(r.t()[None].contiguous(), 2)
            assert w.shape[0] == 256 * (2 * r.shape[0] - 1) == alone.shape[1]
            assert torch.equal(w, alone[0]), (kind, int(r.shape[0]), float((w - alone[0]).abs().max()))


def test_decode_rows_capacity():
    dec, _ = _decoders(1, 300)  # 600 frames: one 300-token row, or three 100-token rows, per call
    hrows, _ = _engine_buffers()
    lib = _lib.load()
    ptrs = (C.c_void_p * len(hrows))(*[r.data_ptr() for r in hrows])
    ns = (C.c_int32 * len(hrows))(*ROW_TOKENS)
    wav = torch.empty(len(hrows), 256 * 599, device="cuda")
    rc = lib.ctb_decode_rows(dec._handle, 1, len(hrows), ptrs, ns, C.c_void_p(wav.data_ptr()), 256 * 599,
                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc != 0 and b"exceed" in lib.ctb_last_error()
    got = dec.decode_rows(hrows, 1)  # the wrapper splits the batch into calls that fit
    for r, w in zip(hrows, got):
        assert torch.equal(w, dec.tokens_to_wav(r[None].contiguous(), 1)[0])


# ---------------------------------------------------------------------------------------------------- slot engine
def _gen_specs():
    # (prompt length, max_new, min_new, stream_batch, temperature): forced lengths ending on a boundary (48, 72 with
    # stream_batch 24), off a boundary, and hot seeded requests that end at EOS
    return [(9, 48, 48, 24, 0.3), (17, 72, 72, 24, 0.3), (5, 61, 61, 16, 0.3), (30, 90, 2, 24, 1.5),
            (12, 80, 2, 16, 1.5), (8, 33, 33, 24, 0.3), (21, 70, 2, 24, 1.5), (4, 40, 40, 16, 0.3)]


def _gen_request(embed, k, spec):
    from chattts_b200.engine import Request
    from chattts_b200.processors import gen_logits
    from chattts_b200.prompts import synth_prompt_batch

    L, mx, mn, sb, t = spec
    ids, mask, tmask = synth_prompt_batch([L], seed=400 + k)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    emb = embed(ids, tmask)
    req = Request(emb=emb[0], temperature=[t] * 4, eos_token=625, max_new_token=mx, min_new_token=mn,
                  logits_processors=(*proc, *warp), manual_seed=2000 + k, stream_batch=sb)
    return req, (emb, ids, mask)


@pytest.mark.parametrize("slots", [3, 12])
def test_generate_continuous_stream_matches_static_stream_per_request(slots):
    from gpu_util import build_gpt

    gpt, embed, _, _ = build_gpt()
    specs = _gen_specs()
    reqs, statics = zip(*[_gen_request(embed, k, s) for k, s in enumerate(specs)])
    got = {k: [] for k in range(len(reqs))}
    for i, out, last in gpt.generate_continuous_stream(list(reqs), slots=slots):
        got[i].append((out.ids[0].cpu(), out.hiddens[0].cpu().clone(), last))
    for k, r in enumerate(reqs):
        emb, ids, mask = statics[k]
        ref = [(o.ids[0].cpu(), o.hiddens[0].cpu().clone()) for o in gpt.generate(
            emb, ids, torch.tensor(r.temperature), 625, attention_mask=mask, max_new_token=r.max_new_token,
            min_new_token=r.min_new_token, logits_processors=r.logits_processors, return_hidden=True, stream=True,
            show_tqdm=False, stream_batch=r.stream_batch, manual_seed=r.manual_seed)]
        if not ref:  # seeded first-step EOS: generate yields nothing, the engine one empty final output
            assert len(got[k]) == 1 and got[k][0][0].shape[0] == 0 and got[k][0][2]
            continue
        assert len(got[k]) == len(ref), (k, [g[0].shape[0] for g in got[k]], [x[0].shape[0] for x in ref])
        assert [g[2] for g in got[k]] == [False] * (len(ref) - 1) + [True]
        for (gi, gh, _), (ri, rh) in zip(got[k], ref):
            assert torch.equal(gi, ri), k
            assert gh.shape == rh.shape and float((gh - rh).abs().max()) < 1e-4, k
    # the boundary-ending forced lengths give a boundary yield followed by a final yield of the same length
    assert [g[0].shape[0] for g in got[0]] == [24, 48, 48]
    assert [g[0].shape[0] for g in got[1]] == [24, 48, 72, 72]


# ---------------------------------------------------------------------------------------------------- Chat
_c = {}


def chat():
    if not _c:
        from chattts_b200 import Chat
        from chattts_b200.synth import synth_all
        from stubs import StubSpeaker, StubTokenizer

        c = Chat()
        assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                             max_batch=4, max_context=256)
        _c["chat"] = c
    return _c["chat"]


TEXTS = ["hello there", "hi", "a somewhat longer sentence to speak", "ok", "fifth text"]


def _chat_params(c):
    n = [48, 72, 61, 100, 37]
    return [c.InferCodeParams(manual_seed=3 + i, max_new_token=n[i], min_new_token=n[i], temperature=0.3 + 0.1 * i,
                              stream_batch=[16, 24, 16, 24, 16][i], stream_speed=[6000, 6000, 12000, 12000, 6000][i],
                              pass_first_n_batches=[0, 2, 0, 2, 2][i], show_tqdm=False)
            for i in range(len(TEXTS))]


@pytest.mark.parametrize("use_decoder", [True, False])
def test_infer_continuous_stream_equals_static_stream_per_text(use_decoder):
    c = chat()
    params = _chat_params(c)
    got = {i: [] for i in range(len(TEXTS))}
    for i, chunk, last in c.infer_continuous_stream(TEXTS, params_infer_code=params, slots=3, use_decoder=use_decoder):
        assert chunk.ndim == 2 and chunk.shape[0] == 1 and chunk.dtype == np.float32
        got[i].append((chunk, last))
    for i, t in enumerate(TEXTS):
        ref = list(c.infer([t], stream=True, split_text=False, skip_refine_text=True, use_decoder=use_decoder,
                           params_infer_code=params[i]))
        assert len(got[i]) == len(ref), (i, len(got[i]), len(ref))
        assert [last for _, last in got[i]] == [False] * (len(ref) - 1) + [True]
        for (x, _), y in zip(got[i], ref):
            if not use_decoder:  # ids are bit-exact, so every chunk is bit-identical
                assert np.array_equal(x, y), i
        for (x, _), y in zip(got[i][:-1], ref[:-1]):
            assert x.shape == y.shape, (i, x.shape, y.shape)
            if x.size:
                assert float(np.sqrt(np.mean((x - y) ** 2))) < 1e-4, i
        assert abs(got[i][-1][0].shape[1] - ref[-1].shape[1]) <= 2


def test_interrupt_ends_running_streams_with_a_final_chunk():
    c = chat()
    p = c.InferCodeParams(manual_seed=5, max_new_token=200, min_new_token=200, stream_batch=16, stream_speed=6000,
                          pass_first_n_batches=0, show_tqdm=False)
    gen = c.infer_continuous_stream(["one", "two", "three", "four"], params_infer_code=p, slots=2)
    events = [next(gen)]
    c.interrupt()
    events += list(gen)
    c.context.set(False)
    seen = {}
    for i, chunk, last in events:
        assert not seen.get(i, False), ("chunk after the final one", i)
        seen[i] = last
    assert sorted(seen) == [0, 1] and all(seen.values())
