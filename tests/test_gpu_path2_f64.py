"""Hot path 2 (DVAE decoder -> Vocos -> iSTFT) on the GPU against float64, at the lengths the product decodes.

Every case runs on both GEMM back ends - the wgmma 3xTF32 ``k_tc_gemm`` (default) and the fp32 FMA twin
(``CTB_DECODER_FMA=1``) - and is compared with ``tests/f64_path2.py``'s float64 evaluation of the same model, run on the
GPU by torch's own float64 kernels.  Bars (``f64_path2``): mel max-abs error / mel max-abs, waveform RMS error / signal
RMS and waveform max-abs error / signal max-abs; the wide-phase head has its own, looser waveform bars (an fp32 phase of
~1e2 carries ~1e-5 rad of rounding, in any fp32 implementation).  Every distance is printed (``pytest -s``).

A. full-length rows: T = 1024, 2048, 4096 tokens (``Chat`` makes its decoders with max_tokens = 4096; at 4096 a row is
   8192 frames = 64 M tiles of ``k_tc_gemm`` and 2 M samples of ``k_overlap_add``), hidden states through
   ``tokens_to_wav`` (token-major) and ``dvae_decode`` (channels-first), codes through both; the codes cover all 625 ids.
B. tile edges: T = 1 .. 300, frame counts at and just past multiples of the 128-frame M tile, two rows per call so the
   dilated k7 halo and the utterance boundary both cross tile edges.
C. the clipped head (most bins at clip(exp, 100)), the wide-phase head (|phase| ~ 1e2) and the loud DVAE (layer scale
   x 4).
D. ``decode_rows``: rows of 1, 65, 300, 2048 and 4096 tokens in one ragged call, read in place from an engine-like
   [rows, 4096, C] buffer; every row against its own float64 decode.
E. the encode branch at its full range: a 30 s encode, one of exactly ``max_samples`` (``Chat``'s 512 x 4096) and
   ``encode_rows`` with a 513-sample row beside a max-length row, against ``dvae_encode(precise_stft=True)``: codes
   exact wherever the oracle's decision margin is > 3e-3 and the earlier residual stages of the group agree.
"""
import gc
import os

import pytest
import torch

import f64_path2 as P
from chattts_b200.synth import synth_speech_like, synth_vocos_state
from gpu_util import release_on_teardown

pytestmark = pytest.mark.gpu

BACKENDS = ["wgmma", "fma"]
MAX_TOKENS = 4096
RAGGED = [300, 4096, 1, 2048, 65]
_h, _ref, _enc = {}, {}, {}
_release = release_on_teardown(_h, _ref, _enc)


def _states(model):
    """model: 'hidden' | 'codes' | 'clipped' | 'wide' | 'loud' -> (dvae state, vocos state, has_vq)."""
    vs = synth_vocos_state(5)
    if model == "codes":
        return P.code_state(), vs, True
    ds = P.hidden_state()
    if model == "clipped":
        return ds, P.clipped_vocos_state(), False
    if model == "wide":
        return ds, P.wide_phase_vocos_state(), False
    if model == "loud":
        return P.loud_dvae_state(ds), vs, False
    return ds, vs, False


def engine(model, backend, max_batch=2, max_tokens=MAX_TOKENS):
    key = (model, backend, max_batch, max_tokens)
    if key not in _h:
        from chattts_b200.decoder import DVAE, Vocos

        _h.clear()   # one handle alive at a time (each holds activations for up to 5 x 8192 frames)
        gc.collect()
        ds, vs, has_vq = _states(model)
        voc = Vocos(P.CFG.vocos, "cuda", max_batch=max_batch, max_tokens=max_tokens)
        voc.state = {k: v.float() for k, v in vs.items()}   # only its weights go into the DVAE handle
        stack = P.CFG.dvae.decoder if has_vq else P.CFG.decoder
        if backend == "fma":
            os.environ["CTB_DECODER_FMA"] = "1"
        try:
            dv = DVAE(stack, None, P.CFG.dvae.vq if has_vq else None, dim=stack.idim, device="cuda", vocos=voc,
                      max_batch=max_batch, max_tokens=max_tokens).load_state_dict(ds)
        finally:
            os.environ.pop("CTB_DECODER_FMA", None)
        _h[key] = dv.engine
    return _h[key]


def reference(model, key, inp):
    """(mel, wav) of inp ([B, 768, T] channels-first or codes [B, 4, T]) in float64, on the GPU; kept under ``key`` for
    the other back end."""
    ds, vs, has_vq = _states(model)
    key = (model, key)
    if key not in _ref:
        with torch.no_grad():
            mel = P.dvae_f64(inp, P.widen(ds, device="cuda"), has_vq)
            wav = P.vocos_f64(mel, P.widen(vs, device="cuda"))
        _ref[key] = (mel.cpu(), wav.cpu())
        del mel, wav
        torch.cuda.empty_cache()   # hand torch's float64 scratch back for the handles' own allocations
    return _ref[key]


def hidden_input(B, T, seed):
    return torch.randn(B, 768, T, generator=torch.Generator().manual_seed(seed))


def check(label, backend, d, wide=False):
    bars = {**P.BARS[backend], **(P.WIDE_BARS[backend] if wide else {})}
    print(f"\n[path2-f64] {label} {backend}: " + "  ".join(f"{k} {v:.2e}" for k, v in d.items()))
    for k, v in d.items():
        assert v <= bars[k], (label, backend, k, v, bars[k])


# ---------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("T", [1024, 2048, 4096])
@pytest.mark.parametrize("model", ["hidden", "codes"])
def test_full_length_rows(model, T, backend):
    eng = engine(model, backend)
    if model == "hidden":
        x = hidden_input(1, T, T)
        tm, layout = x.permute(0, 2, 1).contiguous(), 1
    else:
        x = P.all_codes(1, T, T)
        assert int(x.min()) == 0 and int(x.max()) == 624 and x.unique().numel() == 625
        tm, layout = x, 2
    mel_ref, wav_ref = reference(model, ("full", T), x)
    wav = eng.tokens_to_wav(tm.cuda(), layout)
    assert wav.shape == (1, 512 * T - 256) and bool(torch.isfinite(wav).all())
    check(f"{model} T={T} tokens_to_wav", backend, P.distances(None, None, wav, wav_ref))
    mel = eng.dvae_decode(x.cuda(), 0 if model == "hidden" else 2)
    check(f"{model} T={T} dvae_decode", backend, P.distances(mel, mel_ref, None, None))


# ---------------------------------------------------------------------------------------------------------------- B
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 300])
@pytest.mark.parametrize("model", ["hidden", "codes"])
def test_tile_edges(model, T, backend):
    eng = engine(model, backend)
    x = hidden_input(2, T, 100 + T) if model == "hidden" else P.all_codes(2, T, 100 + T)
    mel_ref, wav_ref = reference(model, ("edge", T), x)
    mel = eng.dvae_decode(x.cuda(), 0 if model == "hidden" else 2)
    wav = eng.vocos_decode(None)
    assert mel.shape == (2, 100, 2 * T) and wav.shape == (2, 256 * (2 * T - 1))
    for b in range(2):
        check(f"{model} T={T} row {b}", backend, P.distances(mel[b], mel_ref[b], wav[b], wav_ref[b]))


# ---------------------------------------------------------------------------------------------------------------- C
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("model", ["clipped", "wide", "loud"])
def test_head_and_residual_variants(model, backend):
    ds, vs, _ = _states(model)
    x = hidden_input(2, 300, 7)
    mel_ref, wav_ref = reference(model, "variant", x)
    with torch.no_grad():
        mag, phase = P.vocos_head(mel_ref.cuda(), P.widen(vs, device="cuda"))
    if model == "clipped":
        assert float((mag > torch.log(torch.tensor(100.0, dtype=torch.float64))).double().mean()) > 0.8
    elif model == "wide":
        assert float(phase.abs().max()) > 80
    eng = engine(model, backend)
    wav = eng.tokens_to_wav(x.permute(0, 2, 1).contiguous().cuda(), 1)
    mel = eng.dvae_decode(x.cuda(), 0)
    check(f"{model} T=300", backend, P.distances(mel, mel_ref, wav, wav_ref), wide=model == "wide")


# ---------------------------------------------------------------------------------------------------------------- D
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("model", ["hidden", "codes"])
def test_decode_rows_ragged_vs_f64(model, backend):
    eng = engine(model, backend, max_batch=len(RAGGED))
    g = torch.Generator().manual_seed(21)
    if model == "hidden":
        buf = torch.randn(len(RAGGED), MAX_TOKENS + 8, 768, generator=g).cuda()
        kind = 1
    else:
        buf = torch.randint(0, 625, (len(RAGGED), MAX_TOKENS + 8, 4), generator=g, dtype=torch.int32).cuda()
        kind = 2
    rows = [buf[k, :n] for k, n in enumerate(RAGGED)]
    assert all(r.is_contiguous() for r in rows)
    wavs = eng.decode_rows(rows, kind)
    for k, n in enumerate(RAGGED):
        assert wavs[k].data_ptr() - wavs[0].data_ptr() == k * 256 * (2 * max(RAGGED) - 1) * 4   # one call
        inp = rows[k].cpu().T[None].contiguous()
        _, wav_ref = reference(model, ("rows", k), inp.long() if kind == 2 else inp)
        check(f"decode_rows {model} n={n}", backend, P.distances(None, None, wavs[k][None], wav_ref))


# ---------------------------------------------------------------------------------------------------------------- E
ENC_MAX = 512 * MAX_TOKENS
CLEAR = 3e-3   # decision margin above which a code must equal the oracle's (see _check_codes)


def _encoder():
    if not _enc:
        from chattts_b200.decoder import AudioEncoder, pack_dvae_encoder
        from chattts_b200.synth import synth_dvae_state

        cfg = P.CFG
        st = synth_dvae_state(3, cfg.dvae.decoder, cfg.dvae.decoder.idim, cfg.dvae.vq, encoder=cfg.dvae.encoder)
        _enc["st"] = st
        _enc["enc"] = AudioEncoder(cfg.dvae.encoder, cfg.dvae.decoder.idim, cfg.dvae.vq,
                                   pack_dvae_encoder(st, cfg.dvae.encoder, cfg.dvae.decoder.idim, cfg.dvae.vq), "cuda",
                                   max_samples=max(ENC_MAX, 30 * 24000))
    return _enc["enc"], _enc["st"]


def _check_codes(label, ids, margin, wav, st):
    from oracle.dvae_oracle import dvae_encode

    ref_ids, ref_margin, _, _ = dvae_encode(wav, st, return_parts=True, precise_stft=True)
    assert tuple(ids.shape) == (4, (wav.numel() // 256 + 1) // 2) == tuple(ref_ids.shape[1:])
    same = ids.cpu() == ref_ids[0].int()
    # residual stage r quantises what stage r - 1 left: where an earlier stage of the group took the other side of a
    # near-tie (allowed), the later stages quantise a different residual, and neither their ids nor margins compare
    R = P.CFG.dvae.vq.R
    agree = torch.ones_like(same)
    for c in range(same.shape[0]):
        if c % R:
            agree[c] = agree[c - 1] & same[c - 1]
    # test_gpu_encode.py's 1e-3 holds to ~3 s of audio; over 30 - 87 s the GPU's margins are up to 2.2e-3 from the
    # oracle's (the wgmma accumulation, DESIGN.md path 2 against float64), so a code is exact where its margin is > 3e-3
    clear = (ref_margin[0] > CLEAR) & agree
    dm = float((margin.cpu() - ref_margin[0]).abs()[agree].max())
    print(f"\n[path2-f64] encode {label}: {ids.shape[1]} tokens, {int((~same).sum())} ids differ "
          f"({int((~agree).sum())} after a near-tie in an earlier stage); margin max-abs diff {dm:.1e}")
    assert bool(same[clear].all()), "an index with a clear decision margin differs from the oracle"
    assert float(same.float().mean()) > 0.99
    assert dm < CLEAR


@pytest.mark.parametrize("n", [30 * 24000, ENC_MAX])
def test_encode_full_range(n):
    enc, st = _encoder()
    wav = synth_speech_like(n / 24000 + 0.1, 9)[:n].contiguous()
    ids, margin = enc.encode(wav, want_margin=True)
    _check_codes(f"{n} samples", ids, margin, wav, st)


def test_encode_rows_shortest_and_longest():
    enc, st = _encoder()
    short = synth_speech_like(0.1, 4)[:513].contiguous()
    long = synth_speech_like(ENC_MAX / 24000 + 0.1, 10)[:ENC_MAX].contiguous()
    out = enc.encode_rows([short, long], want_margin=True)
    for (ids, margin), wav, label in zip(out, (short, long), ("rows: 513 samples", f"rows: {ENC_MAX} samples")):
        _check_codes(label, ids, margin, wav, st)
