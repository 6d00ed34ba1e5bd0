"""Host side of hot path 2: drop-ins for the reference's ``DVAE`` (decode branch,
ChatTTS/model/dvae.py:209-297), the third-party ``Vocos.decode`` (core.py:505-510) and
``Chat._decode_to_wavs`` (core.py:512-539), all running through ``ctb_dvae_decode`` /
``ctb_vocos_decode`` (include/chattts_b200.h).
"""
from __future__ import annotations

import ctypes as C
import math
import threading
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib
from .config import Config, ConvStackConfig, VocosConfig, VQConfig

State = Dict[str, torch.Tensor]
MEL, MEL_PAD = 100, 128


class _Packer:
    """Appends tensors in the order of decoder_api.cu's layout functions (each padded to 4 floats)."""

    def __init__(self):
        self.parts: List[torch.Tensor] = []
        self.n = 0

    def add(self, t: torch.Tensor):
        t = t.detach().to("cpu", torch.float32).contiguous().view(-1)
        pad = (-t.numel()) % 4
        if pad:
            t = torch.cat([t, torch.zeros(pad)])
        self.parts.append(t)
        self.n += t.numel()

    def blob(self) -> torch.Tensor:
        return torch.cat(self.parts)


def _tap_major(w: torch.Tensor, cin_pad: Optional[int] = None) -> torch.Tensor:
    """Conv1d weight [Cout, Cin, k] -> GEMM weight [Cout, k * Cin_pad] with kk = tap * Cin + c."""
    cout, cin, k = w.shape
    w = w.permute(0, 2, 1)
    if cin_pad and cin_pad != cin:
        w = torch.cat([w, torch.zeros(cout, k, cin_pad - cin)], dim=2)
    return w.reshape(cout, -1)


def _pack_block(pk: _Packer, s: State, p: str, scale_name: str):
    pk.add(s[p + "dwconv.weight"][:, 0, :].t())  # [7][C]
    pk.add(s[p + "dwconv.bias"])
    pk.add(s[p + "norm.weight"])
    pk.add(s[p + "norm.bias"])
    pk.add(s[p + "pwconv1.weight"])
    pk.add(s[p + "pwconv1.bias"])
    pk.add(s[p + "pwconv2.weight"])
    pk.add(s[p + "pwconv2.bias"])
    pk.add(s[p + scale_name])


def pack_dvae(s: State, stack: ConvStackConfig, dim: int, vq: Optional[VQConfig]) -> torch.Tensor:
    pk = _Packer()
    pk.add(_tap_major(s["decoder.conv_in.0.weight"]))
    pk.add(s["decoder.conv_in.0.bias"])
    pk.add(_tap_major(s["decoder.conv_in.2.weight"]))
    pk.add(s["decoder.conv_in.2.bias"])
    for i in range(stack.n_layer):
        _pack_block(pk, s, f"decoder.decoder_block.{i}.", "weight")
    pk.add(s["decoder.conv_out.weight"][:, :, 0])
    oc = _tap_major(s["out_conv.weight"])
    pk.add(torch.cat([oc, torch.zeros(MEL_PAD - MEL, oc.shape[1])], 0))
    pk.add(torch.cat([s["coef"].reshape(-1), torch.zeros(MEL_PAD - MEL)]))
    if vq is not None:
        pk.add(torch.stack([s[f"vq_layer.quantizer.rvqs.{g}.project_out.weight"] for g in range(vq.G)]))
        pk.add(torch.stack([s[f"vq_layer.quantizer.rvqs.{g}.project_out.bias"] for g in range(vq.G)]))
    return pk.blob()


def idft_basis(n_fft: int, window: torch.Tensor, spec_k: int) -> torch.Tensor:
    """Windowed inverse real DFT as a [n_fft, spec_k] matrix over interleaved (re_k, im_k) columns:
    y[n] = w[n]/N * (Re S_0 + (-1)^n Re S_{N/2} + 2 sum_{0<k<N/2} (Re S_k cos(2 pi k n/N) - Im S_k sin(2 pi k n/N)))
    i.e. ``torch.fft.irfft(S, n_fft) * window`` (what torch.istft folds)."""
    n = torch.arange(n_fft, dtype=torch.float64)[:, None]
    k = torch.arange(n_fft // 2 + 1, dtype=torch.float64)[None, :]
    ang = 2 * math.pi * ((n * k) % n_fft) / n_fft
    scale = torch.full((1, n_fft // 2 + 1), 2.0, dtype=torch.float64)
    scale[0, 0] = scale[0, -1] = 1.0
    re = torch.cos(ang) * scale
    im = -torch.sin(ang) * scale
    im[:, 0] = 0.0
    im[:, -1] = 0.0
    w = window.double()[:, None] / n_fft
    basis = torch.zeros(n_fft, spec_k, dtype=torch.float64)
    basis[:, 0: 2 * (n_fft // 2 + 1): 2] = re * w
    basis[:, 1: 2 * (n_fft // 2 + 1): 2] = im * w
    return basis.float()


def pack_vocos(s: State, cfg: VocosConfig) -> torch.Tensor:
    pk = _Packer()
    nbin = cfg.n_fft // 2 + 1
    spec_k = (cfg.n_fft + 2 + 31) // 32 * 32
    pk.add(_tap_major(s["backbone.embed.weight"], MEL_PAD))
    pk.add(s["backbone.embed.bias"])
    pk.add(s["backbone.norm.weight"])
    pk.add(s["backbone.norm.bias"])
    for i in range(cfg.num_layers):
        _pack_block(pk, s, f"backbone.convnext.{i}.", "gamma")
    pk.add(s["backbone.final_layer_norm.weight"])
    pk.add(s["backbone.final_layer_norm.bias"])
    hw, hb = s["head.out.weight"], s["head.out.bias"]
    w2 = torch.zeros(spec_k, cfg.dim)
    b2 = torch.zeros(spec_k)
    w2[0: 2 * nbin: 2], w2[1: 2 * nbin: 2] = hw[:nbin], hw[nbin:]
    b2[0: 2 * nbin: 2], b2[1: 2 * nbin: 2] = hb[:nbin], hb[nbin:]
    pk.add(w2)
    pk.add(b2)
    window = s.get("head.istft.window", torch.hann_window(cfg.n_fft))
    pk.add(idft_basis(cfg.n_fft, window, spec_k))
    pk.add(window)
    return pk.blob()


def _stack_cfg(stack: ConvStackConfig, dim: int, vq: Optional[VQConfig], scale_base: int = 4) -> "_lib.ConvStackConfig":
    levels = 0
    if vq is not None:
        assert len(set(vq.levels)) == 1 and len(vq.levels) == 4, "FSQ with 4 equal levels"
        levels = int(vq.levels[0]) | (int(scale_base) << 8)
    return _lib.ConvStackConfig(stack.idim, stack.odim, stack.hidden, stack.n_layer, stack.bn_dim, stack.kernel,
                                stack.dilation, dim, vq.dim if vq else 0, vq.G if vq else 0, vq.R if vq else 0, levels)


def _vocos_cfg(c: VocosConfig) -> "_lib.VocosConfig":
    return _lib.VocosConfig(c.input_channels, c.dim, c.intermediate_dim, c.num_layers, c.n_fft, c.hop_length)


class TokenDecoder:
    """One ``ctb_decoder`` handle = one DVAE stack (+ optional VQ) + the Vocos vocoder."""

    def __init__(self, stack: ConvStackConfig, dim: int, vq: Optional[VQConfig], vocos_cfg: VocosConfig,
                 dvae_blob: Optional[torch.Tensor], vocos_blob: Optional[torch.Tensor], device, max_batch: int = 8,
                 max_tokens: int = 2048, fsq_scale_base: int = 4):
        _lib.require_cuda()
        lib = _lib.load()
        self.device = torch.device(device)
        self.stack, self.dim, self.vq, self.vocos_cfg = stack, dim, vq, vocos_cfg
        self.max_batch, self.max_tokens = max_batch, max_tokens
        self._dc, self._vc = _stack_cfg(stack, dim, vq, fsq_scale_base), _vocos_cfg(vocos_cfg)
        if dvae_blob is not None:
            assert dvae_blob.numel() == lib.ctb_dvae_blob_floats(C.byref(self._dc)), "dvae blob layout mismatch"
        if vocos_blob is not None:
            assert vocos_blob.numel() == lib.ctb_vocos_blob_floats(C.byref(self._vc)), "vocos blob layout mismatch"
        self._dvae_blob = dvae_blob.to(self.device, torch.float32).contiguous() if dvae_blob is not None else None
        self._vocos_blob = vocos_blob.to(self.device, torch.float32).contiguous() if vocos_blob is not None else None
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.ctb_decoder_create(
                C.byref(self._dc), C.c_void_p(self._dvae_blob.data_ptr()) if dvae_blob is not None else None,
                C.byref(self._vc), C.c_void_p(self._vocos_blob.data_ptr()) if vocos_blob is not None else None,
                max_batch, max_tokens, C.byref(self._handle)))

    def __del__(self):
        try:
            if self._handle:
                _lib.load().ctb_decoder_destroy(self._handle)
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def dvae_decode(self, inp: torch.Tensor, layout: int, want_mel: bool = True) -> Optional[torch.Tensor]:
        """layout 0: [B,C,T] fp32; 1: [B,T,C] fp32; 2: ids [B,num_vq,T] -> mel [B,100,2T] (or None)."""
        lib = _lib.load()
        if layout == 2:
            inp = inp.to(self.device, torch.int32).contiguous()
            B, _, T = inp.shape
        else:
            inp = inp.to(self.device, torch.float32).contiguous()
            B, T = (inp.shape[0], inp.shape[2]) if layout == 0 else (inp.shape[0], inp.shape[1])
        mel = torch.empty(B, MEL, 2 * T, dtype=torch.float32, device=self.device) if want_mel else None
        with torch.cuda.device(self.device):
            _lib.check(lib.ctb_dvae_decode(self._handle, C.c_void_p(inp.data_ptr()), layout, B, T,
                                           C.c_void_p(mel.data_ptr()) if want_mel else None, self._stream()))
        self._last = (B, 2 * T)
        return mel

    def vocos_decode(self, mel: Optional[torch.Tensor]) -> torch.Tensor:
        lib = _lib.load()
        if mel is not None:
            mel = mel.to(self.device, torch.float32).contiguous()
            B, _, F = mel.shape
        else:
            B, F = self._last
        wav = torch.empty(B, self.vocos_cfg.hop_length * (F - 1), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.ctb_vocos_decode(self._handle, C.c_void_p(mel.data_ptr()) if mel is not None else None,
                                            B, F, C.c_void_p(wav.data_ptr()), self._stream()))
        return wav

    def tokens_to_wav(self, inp: torch.Tensor, layout: int) -> torch.Tensor:
        """Fused path: the mel never leaves the handle (no channels-first round trip)."""
        self.dvae_decode(inp, layout, want_mel=False)
        return self.vocos_decode(None)

    def decode_rows(self, rows: Sequence[torch.Tensor], kind: int) -> List[torch.Tensor]:
        """Independent token sequences -> waveforms through ``ctb_decode_rows``; row k comes out bit-identical to
        ``tokens_to_wav`` of that row alone.  kind 1: rows of [n_k, 2*idim] fp32 hidden states; kind 2: rows of
        [n_k, num_vq] int32 codes, both token-major on the device (slices of the GPT engine's output buffers work as
        they are).  Returns one [hop * (2 n_k - 1)] tensor per row (views into one buffer per call).  A batch larger
        than the handle's max_batch * 2 * max_tokens frames is split into several calls."""
        if kind not in (1, 2):
            raise ValueError("kind: 1 = hidden states, 2 = codes")
        dtype = torch.float32 if kind == 1 else torch.int32
        rows = [r if r.dtype == dtype and r.is_contiguous() and r.device == self.device
                else r.to(self.device, dtype).contiguous() for r in rows]
        if any(r.dim() != 2 or r.shape[0] < 1 for r in rows):
            raise ValueError("decode_rows: every row must be [n, C] with n >= 1")
        lib = _lib.load()
        hop, cap = self.vocos_cfg.hop_length, self.max_batch * 2 * self.max_tokens
        out: List[torch.Tensor] = []
        lo = 0
        while lo < len(rows):
            hi, W = lo, 0
            while hi < len(rows) and (hi - lo + 1) * 2 * max(W, int(rows[hi].shape[0])) <= cap:
                W = max(W, int(rows[hi].shape[0]))
                hi += 1
            if hi == lo:
                raise ValueError(f"a row of {int(rows[lo].shape[0])} tokens exceeds this handle "
                                 f"(max_tokens={self.max_tokens})")
            part = rows[lo:hi]
            ld = hop * (2 * W - 1)
            wav = torch.empty(len(part), ld, dtype=torch.float32, device=self.device)
            ptrs = (C.c_void_p * len(part))(*[r.data_ptr() for r in part])
            ns = (C.c_int32 * len(part))(*[int(r.shape[0]) for r in part])
            with torch.cuda.device(self.device):
                _lib.check(lib.ctb_decode_rows(self._handle, kind, len(part), ptrs, ns, C.c_void_p(wav.data_ptr()), ld,
                                               self._stream()))
            out += [wav[k, : hop * (2 * int(r.shape[0]) - 1)] for k, r in enumerate(part)]
            lo = hi
        return out



# ---------------------------------------------------------------------------------------------------------------------
# DVAE encode branch (speaker enrolment; SURVEY.md 8f N3): wav -> codes.  dvae.py:175-206,231-236,265-274,102-128.
ENC_NFFT, ENC_HOP, ENC_SR = 1024, 256, 24000   # MelSpectrogramFeatures defaults (dvae.py:176-181)


def mel_filterbank(n_freqs: int = ENC_NFFT // 2 + 1, n_mels: int = MEL, sample_rate: int = ENC_SR) -> torch.Tensor:
    """[3p] torchaudio ``melscale_fbanks(n_freqs, 0, sr/2, n_mels, sr, norm=None, mel_scale="htk")`` -> [n_freqs, n_mels]:
    triangles between HTK-mel-equidistant points (what ``torchaudio.transforms.MelSpectrogram`` builds, dvae.py:188-195)."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_max = 2595.0 * math.log10(1.0 + (sample_rate / 2.0) / 700.0)
    m_pts = torch.linspace(0.0, m_max, n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.clamp(torch.min(down, up), min=0.0)


def pack_dvae_encoder(s: State, stack: ConvStackConfig, dim: int, vq: VQConfig) -> torch.Tensor:
    """Blob of ``ctb_dvae_encoder_create`` (order of decoder_api.cu::enc_layout)."""
    assert stack.idim == dim and stack.odim == vq.dim, "encoder stack must map DVAE dim -> vq dim"
    pk = _Packer()
    # a real checkpoint carries torchaudio's buffers (window, filterbank); the synthetic states do not
    window = s.get("preprocessor_mel.mel_spec.spectrogram.window")
    pk.add(torch.hann_window(ENC_NFFT) if window is None else window)
    fb = s.get("preprocessor_mel.mel_spec.mel_scale.fb")
    fb = mel_filterbank() if fb is None else fb.detach().float().cpu()
    pk.add(torch.cat([fb, torch.zeros(fb.shape[0], MEL_PAD - MEL)], 1))
    pk.add(torch.cat([s["coef"].reshape(-1), torch.ones(MEL_PAD - MEL)]))
    pk.add(_tap_major(s["downsample_conv.0.weight"], MEL_PAD))
    pk.add(s["downsample_conv.0.bias"])
    w = s["downsample_conv.2.weight"]                       # [dim, dim, 4], stride 2, padding 1
    z = torch.zeros(dim, dim)
    # out[t] = W0 x[2t-1] + W1 x[2t] + W2 x[2t+1] + W3 x[2t+2] over pair rows r_t = (x[2t] | x[2t+1])
    pairs = torch.stack([torch.cat([z, w[:, :, 0]], 1), torch.cat([w[:, :, 1], w[:, :, 2]], 1),
                         torch.cat([w[:, :, 3], z], 1)], dim=1)   # [dim, 3 taps, 2*dim]
    pk.add(pairs.reshape(dim, -1))
    pk.add(s["downsample_conv.2.bias"])
    pk.add(_tap_major(s["encoder.conv_in.0.weight"]))
    pk.add(s["encoder.conv_in.0.bias"])
    pk.add(_tap_major(s["encoder.conv_in.2.weight"]))
    pk.add(s["encoder.conv_in.2.bias"])
    for i in range(stack.n_layer):
        _pack_block(pk, s, f"encoder.decoder_block.{i}.", "weight")
    pk.add(s["encoder.conv_out.weight"][:, :, 0])
    pk.add(torch.stack([s[f"vq_layer.quantizer.rvqs.{g}.project_in.weight"] for g in range(vq.G)]))
    pk.add(torch.stack([s[f"vq_layer.quantizer.rvqs.{g}.project_in.bias"] for g in range(vq.G)]))
    return pk.blob()


class AudioEncoder:
    """One ``ctb_encoder`` handle: ``DVAE.forward(mode="encode")`` on the GPU (wav [L] -> ids [G*R, T])."""

    def __init__(self, stack: ConvStackConfig, dim: int, vq: VQConfig, blob: torch.Tensor, device,
                 max_samples: int = 30 * ENC_SR, fsq_scale_base: int = 4, fsq_bound_input: bool = True):
        _lib.require_cuda()
        lib = _lib.load()
        self.device = torch.device(device)
        self.vq, self.max_samples = vq, max_samples
        self._cfg = _stack_cfg(stack, dim, vq, fsq_scale_base)
        if not fsq_bound_input:
            self._cfg.vq_levels |= 1 << 16
        assert blob.numel() == lib.ctb_dvae_encoder_blob_floats(C.byref(self._cfg)), "encoder blob layout mismatch"
        self._blob = blob.to(self.device, torch.float32).contiguous()
        # the handle is not re-entrant: an open engine's worker and Chat.sample_audio_speaker may share it
        self._lock = threading.Lock()
        self._done: Optional[torch.cuda.Event] = None
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.ctb_dvae_encoder_create(C.byref(self._cfg), C.c_void_p(self._blob.data_ptr()), max_samples,
                                                   C.byref(self._handle)))

    def __del__(self):
        try:
            if self._handle:
                _lib.load().ctb_dvae_encoder_destroy(self._handle)
        except Exception:
            pass

    def encode(self, wav: torch.Tensor, want_mel: bool = False, want_margin: bool = False):
        with self._lock, torch.cuda.device(self.device):
            self._after_last_call()
            out = self._encode(wav, want_mel, want_margin)
            self._record_call()
            return out

    def _after_last_call(self):
        """Callers on different CUDA streams share the handle's scratch: order this call after the previous one."""
        if self._done is not None:
            torch.cuda.current_stream().wait_event(self._done)

    def _record_call(self):
        self._done = torch.cuda.Event()
        self._done.record(torch.cuda.current_stream())

    def encode_rows(self, wavs: Sequence[torch.Tensor], want_margin: bool = False):
        """Independent waveforms -> codes in one ``ctb_dvae_encode_rows`` call: a list of ``[G*R, T_k]`` int32 (views
        into one buffer), row k bit-identical to ``encode(wavs[k])``; with ``want_margin`` a list of ``(ids, margin)``.
        Rows already on the device as contiguous fp32 (e.g. ``TokenDecoder.decode_rows`` outputs) are read in place."""
        wavs = [w.view(-1) if w.dtype == torch.float32 and w.is_contiguous() and w.device == self.device
                else w.to(self.device, torch.float32).contiguous().view(-1) for w in wavs]
        if not wavs:
            return []
        lib = _lib.load()
        rows, B = self.vq.G * self.vq.R, len(wavs)
        ld = max(1, max((w.numel() // ENC_HOP + 1) // 2 for w in wavs))
        ids = torch.empty(B, rows, ld, dtype=torch.int32, device=self.device)
        margin = torch.empty(B, rows, ld, dtype=torch.float32, device=self.device) if want_margin else None
        ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
        ns = (C.c_int64 * B)(*[w.numel() for w in wavs])
        n_tok = (C.c_int32 * B)()
        with self._lock, torch.cuda.device(self.device):
            self._after_last_call()
            _lib.check(lib.ctb_dvae_encode_rows(self._handle, B, ptrs, ns, C.c_void_p(ids.data_ptr()), ld, n_tok,
                                                C.c_void_p(margin.data_ptr()) if want_margin else None,
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            self._record_call()
        if want_margin:
            return [(ids[k, :, : n_tok[k]], margin[k, :, : n_tok[k]]) for k in range(B)]
        return [ids[k, :, : n_tok[k]] for k in range(B)]

    def _encode(self, wav: torch.Tensor, want_mel: bool, want_margin: bool):
        lib = _lib.load()
        wav = wav.to(self.device, torch.float32).contiguous().view(-1)
        n = wav.numel()
        frames = n // ENC_HOP + 1
        cap = max(frames // 2, 1)
        rows = self.vq.G * self.vq.R
        ids = torch.empty(rows, cap, dtype=torch.int32, device=self.device)
        mel = torch.empty(MEL, frames, dtype=torch.float32, device=self.device) if want_mel else None
        margin = torch.empty(rows, cap, dtype=torch.float32, device=self.device) if want_margin else None
        n_tok = C.c_int32(0)
        with torch.cuda.device(self.device):
            _lib.check(lib.ctb_dvae_encode(self._handle, C.c_void_p(wav.data_ptr()), n, C.c_void_p(ids.data_ptr()), cap,
                                           C.byref(n_tok), C.c_void_p(mel.data_ptr()) if want_mel else None,
                                           C.c_void_p(margin.data_ptr()) if want_margin else None,
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        assert n_tok.value == cap
        out = (ids,)
        if want_mel:
            out += (mel,)
        if want_margin:
            out += (margin,)
        return out if len(out) > 1 else ids


def _decode_coef(coef) -> torch.Tensor:
    """``DVAE(coef=...)`` of the reference takes a base16384 string of 100 float32 (dvae.py:220-226)."""
    if coef is None:
        return torch.rand(100)
    if isinstance(coef, str):
        from . import b14

        return torch.from_numpy(np.frombuffer(b14.decode_from_string(coef), dtype=np.float32).copy())
    return torch.as_tensor(coef, dtype=torch.float32).reshape(-1)


class DVAE:
    """Drop-in for the reference ``DVAE`` (dvae.py:209-303): ``dvae(inp)`` / ``dvae(inp, mode="decode")`` -> mel
    [B, 100, 2T]; ``dvae(wav, mode="encode")`` -> ids [1, G*R, T] and ``sample_audio(wav)`` -> [G*R, T] (speaker
    enrolment, dvae.py:265-274,299-303) when the model was built with an ``encoder_config`` and a ``vq_config``."""

    def __init__(self, decoder_config: Union[dict, ConvStackConfig], encoder_config=None,
                 vq_config: Union[dict, VQConfig, None] = None, dim: int = 512, coef: Optional[torch.Tensor] = None,
                 device=torch.device("cuda"), vocos: Optional["Vocos"] = None, max_batch: int = 8,
                 max_tokens: int = 2048):
        if isinstance(decoder_config, dict):
            decoder_config = ConvStackConfig(**{k: v for k, v in decoder_config.items()
                                                if k in ConvStackConfig.__dataclass_fields__})
        if isinstance(vq_config, dict):
            vq_config = VQConfig(**vq_config)
        if isinstance(encoder_config, dict):
            encoder_config = ConvStackConfig(**{k: v for k, v in encoder_config.items()
                                                if k in ConvStackConfig.__dataclass_fields__})
        self.enc_stack: Optional[ConvStackConfig] = encoder_config
        self.audio_encoder: Optional[AudioEncoder] = None
        self.stack, self.vq, self.dim = decoder_config, vq_config, dim
        self.device = torch.device(device)
        self.coef = coef
        self.vocos = vocos
        self.max_batch, self.max_tokens = max_batch, max_tokens
        self.state: State = {}
        self.engine: Optional[TokenDecoder] = None

    def load_pretrained(self, filename: str, device):
        from safetensors.torch import load_file

        self.device = torch.device(device)
        return self.load_state_dict(load_file(filename))

    def load_state_dict(self, state: State):
        self.state = {k: v.detach().float() for k, v in state.items()}
        # dvae.py:220-226: the constructor's `coef` (a base16384 string in the reference, a tensor here as well) only
        # initialises the persistent buffer; a checkpoint that carries `coef` overrides it in load_state_dict, and a
        # model with neither gets torch.rand(100)
        if "coef" not in self.state:
            self.state["coef"] = _decode_coef(self.coef).reshape(1, -1, 1)
        blob = pack_dvae(self.state, self.stack, self.dim, self.vq)
        vb = pack_vocos(self.vocos.state, self.vocos.cfg) if self.vocos is not None else None
        self.engine = TokenDecoder(self.stack, self.dim, self.vq, self.vocos.cfg if self.vocos else VocosConfig(),
                                   blob, vb, self.device, self.max_batch, self.max_tokens)
        self.audio_encoder = None
        if self.enc_stack is not None and self.vq is not None and "encoder.conv_in.0.weight" in self.state:
            self.audio_encoder = AudioEncoder(self.enc_stack, self.dim, self.vq,
                                              pack_dvae_encoder(self.state, self.enc_stack, self.dim, self.vq), self.device,
                                              max_samples=max(512 * self.max_tokens, 30 * ENC_SR))
        return self

    def eval(self):
        return self

    def __repr__(self) -> str:
        """dvae.py:250-253: the base16384 form of ``coef``."""
        from . import b14

        return b14.encode_to_string(self.state["coef"].cpu().numpy().astype(np.float32).tobytes())

    @torch.inference_mode()
    def __call__(self, inp: torch.Tensor, mode: str = "decode") -> torch.Tensor:
        if self.engine is None:
            raise _lib.CtbError("DVAE weights not loaded")
        # dvae.py:265: the encode branch is taken only when the model has an encoder AND a VQ layer; anything else
        # falls through to decode, like the reference
        if mode == "encode" and self.audio_encoder is not None:
            return self.audio_encoder.encode(inp).unsqueeze(0)
        return self.engine.dvae_decode(inp, 2 if self.vq is not None else 0)

    @torch.inference_mode()
    def sample_audio(self, wav: Union[np.ndarray, torch.Tensor]) -> torch.Tensor:
        """dvae.py:299-303: wav [L] -> codes [G*R, T]."""
        if isinstance(wav, np.ndarray):
            wav = torch.from_numpy(wav)
        return self(wav, "encode").squeeze_(0)


class Vocos:
    """Drop-in for ``vocos.Vocos`` as used by the reference (core.py:298-317,505-510): ``decode(mel)``."""

    def __init__(self, cfg: VocosConfig = VocosConfig(), device=torch.device("cuda"), max_batch: int = 8,
                 max_tokens: int = 2048):
        self.cfg, self.device = cfg, torch.device(device)
        self.max_batch, self.max_tokens = max_batch, max_tokens
        self.state: State = {}
        self.engine: Optional[TokenDecoder] = None

    def load_state_dict(self, state: State):
        self.state = {k: v.detach().float() for k, v in state.items()}
        stack = Config().decoder
        self.engine = TokenDecoder(stack, stack.idim, None, self.cfg, None, pack_vocos(self.state, self.cfg),
                                   self.device, self.max_batch, self.max_tokens)
        return self

    def to(self, device):
        return self

    def eval(self):
        return self

    @torch.inference_mode()
    def decode(self, mel: torch.Tensor) -> torch.Tensor:
        return self.engine.vocos_decode(mel)


@torch.inference_mode()
def decode_to_wavs(result_list: Sequence[torch.Tensor], use_decoder: bool, decoder: DVAE, dvae: DVAE) -> np.ndarray:
    """core.py:512-539: ragged per-utterance results ([T_b, 768] hiddens or [T_b, 4] ids) are zero-padded to
    the batch max length (quirk Q23: padding influences the tail, keep it), decoded and vocoded; returns
    ``np.ndarray [B, 512*maxT - 256]`` like ``Chat._decode_to_wavs``."""
    if len(result_list) == 0:
        return np.array([], dtype=np.float32)
    model = decoder if use_decoder else dvae
    eng = model.engine
    max_len = max(int(r.size(0)) for r in result_list)
    dev = eng.device
    if use_decoder:
        # token-major [B, T, 768]: the frame doubling is a re-interpretation inside the kernel path
        batch = torch.zeros(len(result_list), max_len, result_list[0].size(1), dtype=torch.float32, device=dev)
        for i, r in enumerate(result_list):
            batch[i, : r.size(0)] = r.to(dev)
        wav = eng.tokens_to_wav(batch, 1)
    else:
        batch = torch.zeros(len(result_list), result_list[0].size(1), max_len, dtype=torch.int32, device=dev)
        for i, r in enumerate(result_list):
            batch[i, :, : r.size(0)] = r.to(dev).permute(1, 0)
        wav = eng.tokens_to_wav(batch, 2)
    return wav.cpu().numpy()


#: tokens of context each side of a decoded window: DVAE decoder +-75 mel frames (conv_in 2 x k3, 12 ConvNeXt k7
#: dilation 2, out_conv k3), Vocos +-27 (embed k7, 8 ConvNeXt k7), iSTFT +-2 frames => +-104 frames = +-52 tokens
STREAM_HALO_TOKENS = 56


def stream_window(n_tokens: int, a: int, b: int, halo: int = STREAM_HALO_TOKENS):
    """``(a, b, t0, t1)``: samples [a, b) of the decode of an `n_tokens` sequence, clamped to its 512 n - 256 samples,
    and the tokens [t0, t1) they depend on (`halo` each side, clamped to the sequence, where the clamp reproduces the
    true boundary).  Samples [a, b) are samples [a - 512 t0, b - 512 t0) of the decode of tokens [t0, t1) alone."""
    total = 512 * n_tokens - 256
    a, b = max(0, a), min(b, total)
    t0 = max(0, a // 512 - halo)
    t1 = min(n_tokens, (b + 511) // 512 + halo + 1)
    if t1 - t0 < 2:  # a one-token window has a single frame pair: widen (the iSTFT needs >= 2 frames)
        t0, t1 = max(0, t1 - 2), max(t1, min(n_tokens, t0 + 2))
    return a, b, t0, t1


def _pad_batch(result_list: Sequence[torch.Tensor], use_decoder: bool, dev, t0: int, t1: int):
    """Columns [t0, t1) of the zero-padded batch `decode_to_wavs` builds (quirk Q23 padding included)."""
    n = len(result_list)
    if use_decoder:
        batch = torch.zeros(n, t1 - t0, result_list[0].size(1), dtype=torch.float32, device=dev)
        for i, r in enumerate(result_list):
            hi = min(int(r.size(0)), t1)
            if hi > t0:
                batch[i, : hi - t0] = r[t0:hi].to(dev)
        return batch, 1
    batch = torch.zeros(n, result_list[0].size(1), t1 - t0, dtype=torch.int32, device=dev)
    for i, r in enumerate(result_list):
        hi = min(int(r.size(0)), t1)
        if hi > t0:
            batch[i, :, : hi - t0] = r[t0:hi].to(dev).permute(1, 0)
    return batch, 2


@torch.inference_mode()
def decode_to_wavs_window(result_list: Sequence[torch.Tensor], use_decoder: bool, decoder: DVAE, dvae: DVAE, a: int,
                          b: int, halo: int = STREAM_HALO_TOKENS) -> np.ndarray:
    """Samples [a, b) of ``decode_to_wavs(result_list, ...)`` without decoding the whole sequence.

    Every layer of path 2 is local in time, so those samples depend only on the tokens within `halo` of the range: the
    window [a // 512 - halo, ceil(b / 512) + halo] is decoded (clamped to the sequence, where the clamp reproduces the
    true boundary) and the range is cut out of it.  This is SURVEY.md 8f N2: the reference re-decodes the cumulative
    sequence at every streaming yield (core.py:455-503, O(n^2)); here a yield costs O(stream_batch + 2 halo) tokens."""
    if len(result_list) == 0 or b <= a:
        return np.zeros((len(result_list), 0), dtype=np.float32)
    model = decoder if use_decoder else dvae
    eng = model.engine
    max_len = max(int(r.size(0)) for r in result_list)
    a, b, t0, t1 = stream_window(max_len, a, b, halo)
    batch, layout = _pad_batch(result_list, use_decoder, eng.device, t0, t1)
    wav = eng.tokens_to_wav(batch, layout)
    return wav[:, a - 512 * t0: b - 512 * t0].cpu().numpy()
