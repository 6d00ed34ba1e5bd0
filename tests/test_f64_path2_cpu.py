"""The float64 reference of hot path 2 (tests/f64_path2.py) on the CPU: that it is the oracle's model, that the fp32
oracle sits within ~1e-6 of it on every variant the GPU tests use, that the variants reach what they are for, and that
a one-GEMM loss of the 3xTF32 ``W_lo`` term lands above the GPU bars (so the bars can see a real regression)."""
import pytest
import torch

import f64_path2 as P
from chattts_b200.synth import synth_vocos_state
from oracle import dvae_oracle as O

T = 130
_c = {}


def base():
    if not _c:
        x = torch.randn(1, 768, T, generator=torch.Generator().manual_seed(0))
        ds, vs = P.hidden_state(), synth_vocos_state(5)
        mel = P.dvae_f64(x, P.widen(ds), False)
        _c.update(x=x, ds=ds, vs=vs, mel=mel, wav=P.vocos_f64(mel, P.widen(vs)))
    return _c


def test_vocos_f64_is_the_oracle_in_float64():
    b = base()
    assert torch.equal(P.vocos_f64(b["mel"], P.widen(b["vs"])), O.vocos_decode(b["mel"], P.widen(b["vs"])))


def test_gfsq_embed_float64_and_fp32_default():
    cs = P.code_state()
    ids = P.all_codes(1, 200, 1)
    assert ids.unique().numel() == 625
    f32 = O.gfsq_embed(ids, cs)
    f64 = O.gfsq_embed(ids, P.widen(cs))
    assert f32.dtype == torch.float32 and f64.dtype == torch.float64
    assert float((f32.double() - f64).abs().max()) < 1e-6


def test_istft_gemm_equals_torch_istft():
    """The GPU's inverse STFT formulation, with its fp32 basis and no other rounding, is torch.istft."""
    b = base()
    d = P.distances(None, None, P.vocos_f64(b["mel"], P.widen(b["vs"]), basis=P.gpu_basis(b["vs"]).double()), b["wav"])
    assert d["wav_rms"] < 1e-7 and d["wav_max"] < 1e-7


def test_tf32_rounding():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -(1.0 + 2 ** -11), 3.0 + 2 ** -12])
    assert P.tf32(x).tolist() == [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -(1.0 + 2 ** -10), 3.0]   # ties away from zero
    w = torch.randn(1000)
    assert float(((P.tf32(w) - w) / w).abs().max()) <= 2 ** -11


@pytest.mark.parametrize("model", ["hidden", "codes", "loud", "clipped", "wide"])
def test_fp32_oracle_is_within_1e6_of_float64(model):
    b = base()
    ds, vs, inp, has_vq = b["ds"], b["vs"], b["x"], False
    if model == "codes":
        ds, inp, has_vq = P.code_state(), P.all_codes(1, T, 1), True
    elif model == "loud":
        ds = P.loud_dvae_state(ds)
    elif model == "clipped":
        vs = P.clipped_vocos_state()
    elif model == "wide":
        vs = P.wide_phase_vocos_state()
    mel64 = P.dvae_f64(inp, P.widen(ds), has_vq)
    wav64 = P.vocos_f64(mel64, P.widen(vs))
    mel = O.dvae_decode(inp if has_vq else inp.float(), ds, has_vq=has_vq)
    d = P.distances(mel, mel64, O.vocos_decode(mel, vs), wav64)
    print(model, d)
    assert d["mel"] < 1.5e-6
    if model == "wide":   # the phase (~1e2) carries fp32's absolute rounding: its own bar, as on the GPU
        assert d["wav_rms"] < 3e-5 and d["wav_rms"] < P.WIDE_BARS["fma"]["wav_rms"] / 3
    else:
        assert d["wav_rms"] < 1.5e-6 and d["wav_max"] < 2e-6


def test_variants_reach_their_branches():
    b = base()
    mag, _ = P.vocos_head(b["mel"], P.widen(P.clipped_vocos_state()))
    assert float((mag > torch.log(torch.tensor(100.0, dtype=torch.float64))).double().mean()) > 0.8
    _, phase = P.vocos_head(b["mel"], P.widen(P.wide_phase_vocos_state()))
    assert float(phase.abs().max()) > 80
    loud = P.dvae_f64(b["x"], P.widen(P.loud_dvae_state(b["ds"])), False)
    assert float(loud.abs().max()) > 2 * float(b["mel"].abs().max())


@pytest.mark.parametrize("gemm,backends", [("idft_basis", ("wgmma", "fma")), ("dvae_pw2_0", ("fma",)),
                                            ("dvae_pw2_11", ("fma",))])
def test_one_gemm_without_w_lo_lands_above_the_gpu_bars(gemm, backends):
    """A GEMM that drops A_hi * W_lo computes with tf32(W): the iDFT basis, or one ConvNeXt pw2 of the DVAE.  The
    pw2 loss (~4e-5) is about twice the wgmma back end's own distance from float64, so only the FMA twin's bar sees it."""
    b = base()
    ds, vs, basis = b["ds"], P.widen(b["vs"]), P.gpu_basis(b["vs"]).double()
    if gemm == "idft_basis":
        basis = P.tf32(P.gpu_basis(b["vs"])).double()
    else:
        k = f"decoder.decoder_block.{gemm.rsplit('_', 1)[1]}.pwconv2.weight"
        ds = {**ds, k: P.tf32(ds[k])}
    mel = P.dvae_f64(b["x"], P.widen(ds), False)
    d = P.distances(mel, b["mel"], P.vocos_f64(mel, vs, basis=basis), b["wav"])
    print(gemm, d)
    for backend in backends:
        assert d["wav_rms"] > 1.3 * P.BARS[backend]["wav_rms"], (backend, d)
