"""Hot path 2 in float64: DVAE decoder (hidden states or codes) -> Vocos backbone -> ISTFT head, the reference the GPU
decode is held to.

``oracle/dvae_oracle.py`` is dtype-generic: on float64 states and inputs its ``dvae_decode`` (``gfsq_embed`` included)
is the float64 evaluation of the fp32 model.  ``vocos_f64`` is ``dvae_oracle.vocos_decode`` split at the head, so that a
test can see the head's log-magnitudes and phases, and so that the inverse STFT can be swapped for ``istft_gemm``: the
GPU's formulation (a GEMM of the interleaved spectrum against the windowed inverse-rDFT basis, then overlap-add and the
window-square envelope).  With the basis the GPU uses and no rounding, ``istft_gemm`` equals ``torch.istft`` to ~1e-7
of the signal (the basis is stored in fp32).

Model variants that take the kernels where the synthetic weights do not:
* ``clipped_vocos_state``: the magnitude half of the head bias at +5.5 (exp ~ 245), so most bins hit ``clip(., 100)``;
* ``wide_phase_vocos_state``: the phase rows of ``head.out`` x 40, so |phase| reaches ~1e2 (``sincosf``'s large
  argument reduction);
* ``loud_dvae_state``: the DVAE layer scales x 4, so the residual stream grows through the 12 blocks.

``tf32`` rounds a tensor like ``cvt.rna.tf32.f32``: a GEMM that loses the ``W_lo`` term of its 3xTF32 split computes
with ``tf32(W)``.  ``tests/test_f64_path2_cpu.py`` checks where such a one-GEMM loss lands against the bars below.

Distances (``distances``) are relative to the reference signal: the mel's max-abs error over the mel's max-abs, the
waveform's RMS error over its RMS, and the waveform's max-abs error over its max-abs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from chattts_b200.config import Config
from chattts_b200.decoder import idft_basis
from chattts_b200.synth import synth_dvae_state, synth_vocos_state
from oracle import dvae_oracle as O

CFG = Config()
N_FFT, HOP = CFG.vocos.n_fft, CFG.vocos.hop_length
NBIN = N_FFT // 2 + 1

# Bars of tests/test_gpu_path2_f64.py per GEMM back end (relative distances, see the module docstring), ~3.5x the
# largest distance observed on one H100 80 GB HBM3 (132 SMs; in brackets), over every case of that file.  A tf32-only
# iDFT basis lands above the waveform RMS bar of both back ends, one DVAE pw2 without W_lo above the FMA twin's only:
# the wgmma back end is itself about half that far from float64 (DESIGN.md, path 2 against float64).
BARS = {
    "wgmma": dict(mel=1e-4, wav_rms=7.5e-5, wav_max=8.5e-5),  # [2.9e-5, 2.1e-5, 2.4e-5]
    "fma": dict(mel=8e-6, wav_rms=6e-6, wav_max=8e-6),        # [2.3e-6, 1.6e-6, 2.2e-6]
}
# the wide-phase head: a phase of ~1e2 carries the head GEMM's rounding (~1e-5 rad in fp32) into every bin
WIDE_BARS = {
    "wgmma": dict(wav_rms=1e-3, wav_max=1e-3),                # [2.9e-4, 3.0e-4]
    "fma": dict(wav_rms=1e-4, wav_max=1e-4),                  # [2.8e-5, 2.7e-5]
}


def widen(state, dtype=torch.float64, device="cpu"):
    return {k: v.to(device, dtype) for k, v in state.items()}


def hidden_state(seed: int = 2):
    """The use_decoder=True model (hidden states [B, 768, T] in)."""
    return synth_dvae_state(seed, CFG.decoder, CFG.decoder.idim)


def code_state(seed: int = 3):
    """The use_decoder=False model (codes [B, 4, T] in)."""
    return synth_dvae_state(seed, CFG.dvae.decoder, CFG.dvae.decoder.idim, CFG.dvae.vq)


def loud_dvae_state(s, scale: float = 4.0):
    out = dict(s)
    for i in range(CFG.decoder.n_layer):
        k = f"decoder.decoder_block.{i}.weight"   # the ConvNeXt layer scale (dvae.py:59-63)
        out[k] = s[k] * scale
    return out


def clipped_vocos_state(seed: int = 5, mag_shift: float = 5.5):
    return synth_vocos_state(seed, CFG.vocos, mag_shift=mag_shift)


def wide_phase_vocos_state(seed: int = 5, scale: float = 40.0):
    s = synth_vocos_state(seed, CFG.vocos)
    s["head.out.weight"] = s["head.out.weight"].clone()
    s["head.out.bias"] = s["head.out.bias"].clone()
    s["head.out.weight"][NBIN:] *= scale
    s["head.out.bias"][NBIN:] *= scale
    return s


def tf32(t: torch.Tensor) -> torch.Tensor:
    """Round fp32 values to tf32 (10 mantissa bits, nearest, ties away from zero: ``cvt.rna.tf32.f32``)."""
    i = t.to(torch.float32).contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype)


def all_codes(B: int, T: int, seed: int) -> torch.Tensor:
    """Codes [B, 4, T] in [0, 625); with B * 4 * T >= 625 every value appears (0 and 624 included)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 625, (B, 4, T), generator=g)
    flat = ids.view(-1)
    n = min(625, flat.numel())
    pos = torch.randperm(flat.numel(), generator=g)[:n]
    flat[pos] = torch.randperm(625, generator=g)[:n]
    return ids


def dvae_f64(inp: torch.Tensor, s64, has_vq: bool) -> torch.Tensor:
    """Hidden states [B, 768, T] (channels-first) or codes [B, 4, T] -> mel [B, 100, 2T] in float64."""
    dev = next(iter(s64.values())).device
    x = inp.to(dev) if has_vq else inp.to(dev, torch.float64)
    return O.dvae_decode(x, s64, has_vq=has_vq)


def vocos_head(mel: torch.Tensor, s):
    """Backbone + head.out of ``dvae_oracle.vocos_decode``: mel [B, 100, F] -> (log-magnitude, phase), each [B, 513, F]."""
    x = F.conv1d(mel, s["backbone.embed.weight"], s["backbone.embed.bias"], padding=3)
    C = x.shape[1]
    x = F.layer_norm(x.transpose(1, 2), (C,), s["backbone.norm.weight"], s["backbone.norm.bias"], eps=1e-6).transpose(1, 2)
    for i in range(CFG.vocos.num_layers):
        x = O.convnext_block(x, s, f"backbone.convnext.{i}.", 1, "gamma")
    x = F.layer_norm(x.transpose(1, 2), (C,), s["backbone.final_layer_norm.weight"],
                     s["backbone.final_layer_norm.bias"], eps=1e-6)
    x = F.linear(x, s["head.out.weight"], s["head.out.bias"]).transpose(1, 2)
    return x.chunk(2, dim=1)


def istft_gemm(spec: torch.Tensor, window: torch.Tensor, basis: torch.Tensor) -> torch.Tensor:
    """``torch.istft(spec, N_FFT, HOP, N_FFT, window, center=True)`` as the GPU forms it: frames = interleaved
    (re, im) spectrum @ basis^T ([N_FFT, >= 2 NBIN] windowed inverse rDFT), overlap-add, / window-square envelope."""
    B, _, Fr = spec.shape
    ri = torch.stack([spec.real, spec.imag], dim=-1).transpose(1, 2).reshape(B, Fr, 2 * NBIN)
    frames = ri @ basis[:, : 2 * NBIN].to(ri).T                          # [B, F, N_FFT]
    L = N_FFT + HOP * (Fr - 1)
    fold = lambda v: F.fold(v, (1, L), (1, N_FFT), stride=(1, HOP))[:, 0, 0]  # noqa: E731  [B, N, F] -> [B, L]
    y = fold(frames.transpose(1, 2))
    w2 = (window.to(ri) ** 2)[None, :, None].expand(1, N_FFT, Fr)
    env = fold(w2.contiguous())
    a = N_FFT // 2
    return y[:, a: a + HOP * (Fr - 1)] / env[:, a: a + HOP * (Fr - 1)]


def vocos_f64(mel: torch.Tensor, s, basis: torch.Tensor | None = None) -> torch.Tensor:
    """``dvae_oracle.vocos_decode`` in the dtype of ``s``; with ``basis`` the inverse STFT is ``istft_gemm``."""
    mag, p = vocos_head(mel.to(s["head.out.weight"]), s)
    mag = torch.clip(torch.exp(mag), max=1e2)
    spec = mag * (torch.cos(p) + 1j * torch.sin(p))
    if basis is None:
        return torch.istft(spec, N_FFT, HOP, N_FFT, s["head.istft.window"], center=True)
    return istft_gemm(spec, s["head.istft.window"], basis)


def gpu_basis(s) -> torch.Tensor:
    """The fp32 inverse-rDFT basis the GPU multiplies by (``decoder.pack_vocos``)."""
    spec_k = (N_FFT + 2 + 31) // 32 * 32
    return idft_basis(N_FFT, s["head.istft.window"].float().cpu(), spec_k)


def distances(mel, mel_ref, wav, wav_ref) -> dict:
    """Relative distances of (mel, wav) from the reference; either pair may be None."""
    d = {}
    if mel is not None:
        mel, mel_ref = mel.double().cpu(), mel_ref.double().cpu()
        d["mel"] = float((mel - mel_ref).abs().max() / mel_ref.abs().max())
    if wav is not None:
        wav, wav_ref = wav.double().cpu(), wav_ref.double().cpu()
        e = wav - wav_ref
        d["wav_rms"] = float(e.pow(2).mean().sqrt() / wav_ref.pow(2).mean().sqrt())
        d["wav_max"] = float(e.abs().max() / wav_ref.abs().max())
    return d
