"""GPU parity of hot path 2 (DVAE decode + Vocos + iSTFT) through the C ABI.
Tolerances: mel max-abs 1e-4 (fp32 reorder), waveform RMS 1e-4 (BASELINE.json north_star)."""
import numpy as np
import pytest
import torch

from chattts_b200.config import Config
from chattts_b200.synth import synth_dvae_state, synth_vocos_state
from oracle import dvae_oracle as O

pytestmark = pytest.mark.gpu
CFG = Config()
_c = {}


def models():
    if not _c:
        from chattts_b200.decoder import DVAE, Vocos

        vs = synth_vocos_state(5)
        ds = synth_dvae_state(2, CFG.decoder, CFG.decoder.idim)
        cs = synth_dvae_state(3, CFG.dvae.decoder, CFG.dvae.decoder.idim, CFG.dvae.vq)
        voc = Vocos(CFG.vocos, "cuda", max_batch=8, max_tokens=256).load_state_dict(vs)
        dec = DVAE(CFG.decoder, dim=CFG.decoder.idim, device="cuda", vocos=voc, max_batch=8, max_tokens=256)
        dec.load_state_dict(ds)
        dv = DVAE(CFG.dvae.decoder, None, CFG.dvae.vq, dim=CFG.dvae.decoder.idim, device="cuda", vocos=voc,
                  max_batch=8, max_tokens=256)
        dv.load_state_dict(cs)
        _c.update(vs=vs, ds=ds, cs=cs, voc=voc, dec=dec, dv=dv)
    return _c


def rms(a, b):
    return float((a - b).pow(2).mean().sqrt())


def assert_wave_close(wav, ref, rel=1e-4):
    """north_star: waveform within 1e-4 RMS.  The synthetic Vocos head is quiet (|wav| ~ 1e-3), so the absolute bound
    alone would accept a 20 % error: the bound that is asserted is RELATIVE to the signal (and the absolute one too)."""
    wav, ref = wav.detach().cpu().float(), ref.detach().cpu().float()
    sig = float(ref.pow(2).mean().sqrt())
    err = rms(wav, ref)
    assert err <= 1e-4, ("absolute RMS", err)
    assert err <= rel * sig + 1e-9, ("relative RMS", err / max(sig, 1e-30), sig)
    assert float((wav - ref).abs().max()) <= 1e-3 * float(ref.abs().max()) + 1e-8


def test_decoder_hidden_path_reference_fixture():
    from gpu_util import load_gold

    m = models()
    g = load_gold("dvae_decoder_hidden")
    mel = m["dec"](torch.from_numpy(g["x"]))
    assert mel.shape == (2, 100, 24)
    assert np.abs(mel.cpu().numpy() - g["mel"]).max() < 1e-4


@pytest.mark.parametrize("B,T", [(1, 1), (3, 37), (2, 130)])
def test_decoder_hidden_path_both_layouts(B, T):
    m = models()
    x = torch.randn(B, 768, T, generator=torch.Generator().manual_seed(T))
    ref = O.dvae_decode(x, m["ds"])
    mel_cf = m["dec"].engine.dvae_decode(x, 0)
    mel_tm = m["dec"].engine.dvae_decode(x.permute(0, 2, 1).contiguous(), 1)
    assert (mel_cf.cpu() - ref).abs().max() < 1e-4
    assert torch.equal(mel_cf, mel_tm)  # same arithmetic, only the staging differs


@pytest.mark.parametrize("B,T", [(1, 2), (4, 61)])
def test_dvae_code_path(B, T):
    m = models()
    ids = torch.randint(0, 625, (B, 4, T), generator=torch.Generator().manual_seed(B))
    ref = O.dvae_decode(ids, m["cs"], has_vq=True)
    mel = m["dv"](ids)
    assert mel.shape == (B, 100, 2 * T)
    assert (mel.cpu() - ref).abs().max() < 1e-4


@pytest.mark.parametrize("B,F", [(1, 2), (2, 9), (3, 150)])
def test_vocos_waveform_rms(B, F):
    m = models()
    mel = torch.randn(B, 100, F, generator=torch.Generator().manual_seed(F)) * 0.5
    ref = O.vocos_decode(mel, m["vs"])
    wav = m["voc"].decode(mel)
    assert wav.shape == (B, 256 * (F - 1))
    assert_wave_close(wav, ref)


def test_vocos_waveform_loud_weights():
    """Vocos head with O(1) magnitudes (bias shift +0.5 instead of -4): waveform RMS ~ 0.1, where north_star's
    absolute 1e-4 RMS is itself a 1e-3 relative bound."""
    from chattts_b200.decoder import Vocos

    vs = synth_vocos_state(5, mag_shift=0.5)
    voc = Vocos(CFG.vocos, "cuda", max_batch=2, max_tokens=128).load_state_dict(vs)
    mel = torch.randn(2, 100, 120, generator=torch.Generator().manual_seed(11)) * 0.5
    ref = O.vocos_decode(mel, vs)
    assert float(ref.pow(2).mean().sqrt()) > 0.02
    wav = voc.decode(mel)
    assert_wave_close(wav, ref)


@pytest.mark.parametrize("use_decoder", [True, False])
def test_decode_to_wavs_ragged_batch(use_decoder):
    """core.py:512-539 semantics incl. zero padding to the batch max length (quirk Q23)."""
    from chattts_b200.decoder import decode_to_wavs

    m = models()
    g = torch.Generator().manual_seed(7)
    lens = [33, 5, 21]
    if use_decoder:
        res = [torch.randn(n, 768, generator=g) for n in lens]
        ref = O.decode_to_wavs(res, True, m["ds"], m["vs"])
    else:
        res = [torch.randint(0, 625, (n, 4), generator=g) for n in lens]
        ref = O.decode_to_wavs(res, False, m["cs"], m["vs"])
    wav = decode_to_wavs([r.clone() for r in res], use_decoder, m["dec"], m["dv"])
    assert isinstance(wav, np.ndarray) and wav.dtype == np.float32 and wav.shape == (3, 512 * 33 - 256)
    assert_wave_close(torch.from_numpy(wav), ref)


def test_decode_to_wavs_empty():
    from chattts_b200.decoder import decode_to_wavs

    m = models()
    out = decode_to_wavs([], True, m["dec"], m["dv"])
    assert out.shape == (0,)


def test_full_size_properties_10s_batch():
    """BASELINE configs[3] scale (10 s = 469 tokens) on a small batch: length, finiteness, linearity of
    the iSTFT stage in the spectrum (zero mel frames at the tail do not leak NaNs), batch-row independence."""
    from chattts_b200.decoder import DVAE, Vocos

    m = models()
    voc = Vocos(CFG.vocos, "cuda", max_batch=4, max_tokens=469).load_state_dict(m["vs"])
    dec = DVAE(CFG.decoder, dim=384, device="cuda", vocos=voc, max_batch=4, max_tokens=469).load_state_dict(m["ds"])
    x = torch.randn(4, 469, 768, generator=torch.Generator().manual_seed(1))
    wav = dec.engine.tokens_to_wav(x, 1)
    assert wav.shape == (4, 512 * 469 - 256) and torch.isfinite(wav).all()
    solo = dec.engine.tokens_to_wav(x[2:3].contiguous(), 1)
    assert torch.equal(solo[0], wav[2])  # rows never interact (SURVEY.md 8e)
    ref = O.vocos_decode(O.dvae_decode(x[:1].permute(0, 2, 1).contiguous(), m["ds"]), m["vs"])
    assert_wave_close(wav[:1], ref)


def test_c4_full_size_batch64_rows_vs_oracle():
    """BASELINE configs[3] exactly: batch 64 x 469 tokens (10 s each) through DVAE decoder + Vocos + iSTFT in one call;
    8 of the 64 rows are checked against the CPU oracle (rows never interact, so the oracle decodes them alone)."""
    from chattts_b200.decoder import DVAE, Vocos

    m = models()
    voc = Vocos(CFG.vocos, "cuda", max_batch=64, max_tokens=469).load_state_dict(m["vs"])
    dec = DVAE(CFG.decoder, dim=384, device="cuda", vocos=voc, max_batch=64, max_tokens=469).load_state_dict(m["ds"])
    x = torch.randn(64, 469, 768, generator=torch.Generator().manual_seed(4))
    wav = dec.engine.tokens_to_wav(x, 1)
    assert wav.shape == (64, 512 * 469 - 256) and torch.isfinite(wav).all()
    for b in (0, 9, 18, 27, 36, 45, 54, 63):
        ref = O.vocos_decode(O.dvae_decode(x[b: b + 1].permute(0, 2, 1).contiguous(), m["ds"]), m["vs"])
        assert_wave_close(wav[b: b + 1], ref)


def test_tensor_core_path_matches_fma_path():
    """The wgmma 3xTF32 GEMMs (default) against the plain fp32 FMA GEMMs (CTB_DECODER_FMA=1) on the same
    handle configuration: fp32-equivalent accuracy is the contract of the hi/lo split."""
    import os

    from chattts_b200.decoder import DVAE, Vocos

    m = models()
    x = torch.randn(2, 300, 768, generator=torch.Generator().manual_seed(3))
    wav_tc = m["dec"].engine.tokens_to_wav(x, 1)
    os.environ["CTB_DECODER_FMA"] = "1"
    try:
        voc = Vocos(CFG.vocos, "cuda", max_batch=2, max_tokens=300).load_state_dict(m["vs"])
        dec = DVAE(CFG.decoder, dim=384, device="cuda", vocos=voc, max_batch=2, max_tokens=300).load_state_dict(m["ds"])
        wav_fma = dec.engine.tokens_to_wav(x, 1)
        mel_fma = dec.engine.dvae_decode(x, 1)
    finally:
        del os.environ["CTB_DECODER_FMA"]
    mel_tc = m["dec"].engine.dvae_decode(x, 1)
    assert (mel_tc - mel_fma).abs().max() < 2e-5 * max(1.0, float(mel_fma.abs().max()))
    assert rms(wav_tc, wav_fma) < 1e-5 * max(1e-3, float(wav_fma.pow(2).mean().sqrt())) + 1e-7


@pytest.mark.parametrize("use_decoder", [True, False])
def test_windowed_decode_equals_slices_of_the_full_decode(use_decoder):
    """SURVEY.md 8f N2: samples [a, b) decoded from the token window they depend on (halo 56 tokens each side) must be the
    samples [a, b) of the full decode, for ranges at the start, in the middle, across the end and for ragged rows."""
    from chattts_b200.decoder import decode_to_wavs, decode_to_wavs_window

    m = models()
    g = torch.Generator().manual_seed(13)
    lens = [250, 101, 187]
    res = [torch.randn(n, 768, generator=g) for n in lens] if use_decoder else \
          [torch.randint(0, 625, (n, 4), generator=g) for n in lens]
    full = decode_to_wavs([r.clone() for r in res], use_decoder, m["dec"], m["dv"])
    total = full.shape[1]
    assert total == 512 * 250 - 256
    for a, b in ((0, 12000), (12000, 24000), (60000, 72000), (512 * 100 - 300, 512 * 102), (total - 5000, total), (0, total)):
        win = decode_to_wavs_window([r.clone() for r in res], use_decoder, m["dec"], m["dv"], a, b)
        assert win.shape == (3, b - a)
        ref = full[:, a:b]
        assert np.abs(win - ref).max() <= 1e-6 * max(1.0, float(np.abs(ref).max())) + 1e-9, (a, b, float(np.abs(win - ref).max()))


def test_persistent_gemm_equals_the_one_tile_per_cta_twin_bit_for_bit():
    """k_tc_gemm with persistent CTAs (one per SM, walking tiles) runs the same MMAs in the same order as with one tile per
    CTA (CTB_TC_NONPERSISTENT=1): identical mel and waveform."""
    import os

    from chattts_b200.decoder import DVAE, Vocos

    m = models()
    x = torch.randn(3, 301, 768, generator=torch.Generator().manual_seed(4))      # 602 frames: a partial last M tile
    wav_p = m["dec"].engine.tokens_to_wav(x, 1)
    mel_p = m["dec"].engine.dvae_decode(x, 1)
    os.environ["CTB_TC_NONPERSISTENT"] = "1"
    try:
        voc = Vocos(CFG.vocos, "cuda", max_batch=3, max_tokens=301).load_state_dict(m["vs"])
        dec = DVAE(CFG.decoder, dim=384, device="cuda", vocos=voc, max_batch=3, max_tokens=301).load_state_dict(m["ds"])
        wav_t = dec.engine.tokens_to_wav(x, 1)
        mel_t = dec.engine.dvae_decode(x, 1)
    finally:
        del os.environ["CTB_TC_NONPERSISTENT"]
    assert torch.equal(mel_p, mel_t) and torch.equal(wav_p, wav_t)
