"""CPU (torch fp32) restatement of hot path 2: tokens / hidden states -> mel -> waveform.

TEST INFRASTRUCTURE (see oracle/__init__.py).

Pinned against the reference itself: ``dvae_decode`` without VQ (reference ``DVAE.forward``
decode branch, dvae.py:276-297, ``DVAEDecoder`` :131-172, ``ConvNeXtBlock`` :14-66).
**Parity unpinned** (third-party code absent from /root/reference, restated from call sites):
  * ``gfsq_embed``  - vector_quantize_pytorch ``GroupedResidualFSQ.get_output_from_indices``
    (requirements.txt:6 unpinned; call sites dvae.py:75-80,96).
  * ``fsq_quantize`` - vector_quantize_pytorch ``GroupedResidualFSQ.forward`` (same package; call site dvae.py:106);
    the rest of ``dvae_encode`` IS pinned: ``mel_features`` against torchaudio's ``MelSpectrogram`` through the reference's
    ``MelSpectrogramFeatures`` (dvae.py:175-206), the downsample convs and the encoder stack against the reference modules.
  * ``vocos_decode`` - vocos ``VocosBackbone`` + ``ISTFTHead`` (requirements.txt:8 unpinned; call
    sites core.py:298-317,505-510; head math restated in-tree at examples/onnx/exporter.py:391-405;
    hyper-parameters config/config.py:74-121).
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

State = Dict[str, torch.Tensor]


def convnext_block(x: torch.Tensor, s: State, p: str, dilation: int, scale_name: str) -> torch.Tensor:
    """dvae.py:46-66 (x is [B, C, T]); the Vocos block is the same with dilation 1 / 'gamma'."""
    C = x.shape[1]
    y = F.conv1d(x, s[p + "dwconv.weight"], s[p + "dwconv.bias"], padding=dilation * 3, dilation=dilation, groups=C)
    y = y.transpose(1, 2)
    y = F.layer_norm(y, (C,), s[p + "norm.weight"], s[p + "norm.bias"], eps=1e-6)
    y = F.linear(y, s[p + "pwconv1.weight"], s[p + "pwconv1.bias"])
    y = F.gelu(y)
    y = F.linear(y, s[p + "pwconv2.weight"], s[p + "pwconv2.bias"])
    y = y * s[p + scale_name]
    return y.transpose(1, 2) + x


def gfsq_embed(ids: torch.Tensor, s: State, G: int = 2, R: int = 2, levels=(5, 5, 5, 5), scale_base: int = 4
               ) -> torch.Tensor:
    """[3p] GFSQ._embed (dvae.py:87-97) -> GroupedResidualFSQ.get_output_from_indices.
    ids [B, G*R, T] -> feat [B, dim, T].  Codebook c = g*R + r; residual r is scaled by
    ``scale_base ** -r`` (``levels - 1`` = 4 in the releases ChatTTS was built against).
    The codes are evaluated in the dtype of the ``project_out`` weights, on the device of ``ids``."""
    B, _, T = ids.shape
    dt = s["vq_layer.quantizer.rvqs.0.project_out.weight"].dtype
    x = ids.transpose(1, 2).reshape(B, T, G, R).permute(2, 0, 1, 3)  # [G, B, T, R]
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1])), 0).to(ids.device)
    lv = torch.tensor(levels).to(ids.device)
    outs = []
    for g in range(G):
        z = 0
        for r in range(R):
            li = (x[g, :, :, r, None] // basis) % lv        # [B, T, 4] level indices
            code = (li.to(dt) - (lv // 2).to(dt)) / (lv // 2).to(dt)
            z = z + code * (float(scale_base) ** -r)
        outs.append(F.linear(z, s[f"vq_layer.quantizer.rvqs.{g}.project_out.weight"],
                             s[f"vq_layer.quantizer.rvqs.{g}.project_out.bias"]))
    return torch.cat(outs, dim=-1).transpose(1, 2)


def dvae_decode(inp: torch.Tensor, s: State, *, n_layer: int = 12, has_vq: bool = False, dilation: int = 2,
                scale_base: int = 4) -> torch.Tensor:
    """DVAE.forward(mode='decode') (dvae.py:276-297): [B, C, T] (or ids [B,4,T]) -> mel [B, 100, 2T]."""
    x = gfsq_embed(inp, s, scale_base=scale_base) if has_vq else inp
    B, C, T = x.shape
    x = x.view(B, 2, C // 2, T).permute(0, 2, 3, 1).flatten(2)  # frame doubling, dvae.py:281-287
    y = F.conv1d(x, s["decoder.conv_in.0.weight"], s["decoder.conv_in.0.bias"], padding=1)
    y = F.gelu(y)
    y = F.conv1d(y, s["decoder.conv_in.2.weight"], s["decoder.conv_in.2.bias"], padding=1)
    for i in range(n_layer):
        y = convnext_block(y, s, f"decoder.decoder_block.{i}.", dilation, "weight")
    y = F.conv1d(y, s["decoder.conv_out.weight"])
    y = F.conv1d(y, s["out_conv.weight"], padding=1)
    return y * s["coef"]


def vocos_decode(mel: torch.Tensor, s: State, *, num_layers: int = 8, n_fft: int = 1024, hop: int = 256
                 ) -> torch.Tensor:
    """[3p] Vocos.decode = ISTFTHead(VocosBackbone(mel)): mel [B,100,F] -> wav [B, hop*(F-1)]."""
    x = F.conv1d(mel, s["backbone.embed.weight"], s["backbone.embed.bias"], padding=3)
    C = x.shape[1]
    x = F.layer_norm(x.transpose(1, 2), (C,), s["backbone.norm.weight"], s["backbone.norm.bias"], eps=1e-6).transpose(1, 2)
    for i in range(num_layers):
        x = convnext_block(x, s, f"backbone.convnext.{i}.", 1, "gamma")
    x = F.layer_norm(x.transpose(1, 2), (C,), s["backbone.final_layer_norm.weight"],
                     s["backbone.final_layer_norm.bias"], eps=1e-6)
    x = F.linear(x, s["head.out.weight"], s["head.out.bias"]).transpose(1, 2)
    mag, p = x.chunk(2, dim=1)
    mag = torch.clip(torch.exp(mag), max=1e2)  # examples/onnx/exporter.py:395-398
    spec = mag * (torch.cos(p) + 1j * torch.sin(p))
    return torch.istft(spec, n_fft, hop, n_fft, s["head.istft.window"], center=True)


def decode_to_wavs(results, use_decoder: bool, dec_state: State, vocos_state: State) -> torch.Tensor:
    """core.py:512-539: zero-pad ragged per-utterance results to [B, C, maxT], decode, vocode."""
    maxT = max(int(r.shape[0]) for r in results)
    batch = torch.zeros(len(results), results[0].shape[1], maxT, dtype=results[0].dtype)
    for i, r in enumerate(results):
        batch[i, :, : r.shape[0]] = r.permute(1, 0)
    mel = dvae_decode(batch, dec_state, has_vq=not use_decoder)
    return vocos_decode(mel, vocos_state)


# ---------------------------------------------------------------------------------------------------------------------
# encode branch (speaker enrolment): DVAE.forward(mode="encode"), dvae.py:265-274


def mel_features(wav: torch.Tensor, n_fft: int = 1024, hop: int = 256, n_mels: int = 100, sr: int = 24000,
                 precise_stft: bool = False) -> torch.Tensor:
    """MelSpectrogramFeatures.forward (dvae.py:199-206) = log(clip(MelSpectrogram(power=1, center)(wav), 1e-5)).
    [3p] torchaudio: |stft| with a periodic Hann window and reflect padding, then the HTK triangular filterbank
    (norm=None, f_min 0, f_max sr/2).  wav [L] -> [n_mels, L // hop + 1].
    ``precise_stft`` evaluates the same |STFT| (fp32 samples, fp32 window) in float64 and rounds the magnitude to fp32:
    the value the reference's fp32 FFT approximates.  The log amplifies the FFT's rounding error in bins far below the
    frame's peak, so two correct fp32 implementations disagree there; the precise form is what the GPU path is held to."""
    win = torch.hann_window(n_fft)
    if precise_stft:
        spec = torch.stft(wav.double(), n_fft, hop, n_fft, win.double(), center=True, pad_mode="reflect", normalized=False,
                          onesided=True, return_complex=True).abs().float()
    else:
        spec = torch.stft(wav, n_fft, hop, n_fft, win, center=True, pad_mode="reflect", normalized=False,
                          onesided=True, return_complex=True).abs()
    n_freqs = n_fft // 2 + 1
    all_freqs = torch.linspace(0, sr // 2, n_freqs)
    m_pts = torch.linspace(0.0, 2595.0 * math.log10(1.0 + (sr / 2.0) / 700.0), n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    fb = torch.clamp(torch.min(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]), min=0.0)   # [n_freqs, n_mels]
    mel = torch.matmul(spec.transpose(-1, -2), fb).transpose(-1, -2)
    return torch.log(torch.clip(mel, min=1e-5))


def fsq_bound(z: torch.Tensor, levels: torch.Tensor, eps: float = 1e-3) -> torch.Tensor:
    """[3p] FSQ.bound: tanh squashing onto (levels - 1) * (1 + eps) / 2, shifted by half a step for even level counts."""
    half_l = (levels - 1).float() * (1 + eps) / 2
    offset = torch.where(levels % 2 == 0, 0.5, 0.0)
    shift = torch.atanh(offset / half_l)
    return torch.tanh(z + shift) * half_l - offset


def fsq_quantize(x: torch.Tensor, s: State, G: int = 2, R: int = 2, levels=(5, 5, 5, 5), scale_base: int = 4,
                 bound_input: bool = True, return_quantized: bool = False):
    """[3p] GFSQ.forward (dvae.py:102-128) -> GroupedResidualFSQ.forward: x [B, T, dim] -> (ids [B, G*R, T], margin).
    Per group: project_in, then R stages of ``q = round(bound(res / s_r))``, ``res -= q / (levels // 2) * s_r`` with
    ``s_r = scale_base ** -r``; index = sum_k (q_k + levels_k // 2) * prod(levels[:k]).  ``bound_input`` applies bound()
    to the projected vector before the first stage (current releases; older ones did not).  ``margin`` is the distance of
    the closest pre-rounding value to a rounding edge - the decision margin of each index."""
    B, T, D = x.shape
    lv = torch.tensor(levels)
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1])), 0)
    half_w = (lv // 2).float()
    ids, margins, zq = [], [], []
    for g, xg in enumerate(x.chunk(G, dim=-1)):
        z = F.linear(xg, s[f"vq_layer.quantizer.rvqs.{g}.project_in.weight"], s[f"vq_layer.quantizer.rvqs.{g}.project_in.bias"])
        res = fsq_bound(z, lv) if bound_input else z
        acc = torch.zeros_like(res)
        for r in range(R):
            sc = float(scale_base) ** -r
            bz = fsq_bound(res / sc, lv)
            q = torch.round(bz)
            margins.append((0.5 - (bz - q).abs()).amin(dim=-1))
            res = res - (q / half_w) * sc
            acc = acc + (q / half_w) * sc
            ids.append(((q + half_w).long() * basis).sum(-1))
        zq.append(acc)
    if return_quantized:
        return torch.stack(ids, dim=1), torch.stack(margins, dim=1), zq
    return torch.stack(ids, dim=1), torch.stack(margins, dim=1)


def dvae_encode(wav: torch.Tensor, s: State, *, n_layer: int = 12, dilation: int = 2, scale_base: int = 4,
                bound_input: bool = True, return_parts: bool = False, precise_stft: bool = False):
    """DVAE.forward(mode='encode') (dvae.py:265-274): wav [L] -> ids [1, G*R, T]."""
    mel = mel_features(wav, precise_stft=precise_stft) / s["coef"].view(100, 1)
    x = F.gelu(F.conv1d(mel[None], s["downsample_conv.0.weight"], s["downsample_conv.0.bias"], padding=1))
    x = F.gelu(F.conv1d(x, s["downsample_conv.2.weight"], s["downsample_conv.2.bias"], stride=2, padding=1))
    y = F.gelu(F.conv1d(x, s["encoder.conv_in.0.weight"], s["encoder.conv_in.0.bias"], padding=1))
    y = F.conv1d(y, s["encoder.conv_in.2.weight"], s["encoder.conv_in.2.bias"], padding=1)
    for i in range(n_layer):
        y = convnext_block(y, s, f"encoder.decoder_block.{i}.", dilation, "weight")
    y = F.conv1d(y, s["encoder.conv_out.weight"])
    ids, margin = fsq_quantize(y.transpose(1, 2), s, scale_base=scale_base, bound_input=bound_input)
    return (ids, margin, mel, y) if return_parts else ids
