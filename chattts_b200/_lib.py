"""ctypes binding of ``libchattts_b200.so`` (the C ABI in include/chattts_b200.h).

There is deliberately no fallback: if the library is missing or no CUDA device is present
the product path raises (north_star: "no CPU fallback").
"""
from __future__ import annotations

import ctypes as C
import os
import threading

from . import build as _build

_lock = threading.Lock()
_lib = None


class GptConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "hidden_size", "intermediate_size", "num_layers", "num_heads", "num_kv_heads", "head_dim", "num_vq",
        "num_audio_tokens", "num_text_tokens", "max_positions")] + [
        ("rms_eps", C.c_float), ("max_batch", C.c_int32), ("max_context", C.c_int32)]


class GptLayout(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        "layer0", "layer_stride", "wqkv", "wo", "wgate_up", "wdown", "ln1", "ln2", "final_norm", "head_code",
        "head_text", "emb_code", "emb_text", "rope_cos", "rope_sin", "total")]


class SamplerConfig(C.Structure):
    _fields_ = [
        ("temperature", C.c_float * 8), ("top_p", C.c_float), ("top_k", C.c_int32),
        ("min_tokens_to_keep", C.c_int32), ("penalty_on", C.c_int32), ("penalty_lut", C.c_float * 32),
        ("past_window", C.c_int32), ("penalty_max_ids", C.c_int32), ("greedy", C.c_int32),
        ("eos_token", C.c_int32), ("min_new_token", C.c_int32), ("top_p_removed_max", C.c_float),
        ("has_removed_max", C.c_int32), ("philox_seed", C.c_uint64)]


class GptStatus(C.Structure):
    _fields_ = [("steps_done", C.c_int32), ("all_finished", C.c_int32),
                ("any_finished_first_step", C.c_int32), ("reserved", C.c_int32)]


#: precision flags of ctb_gpt_engine_begin_ex (CTB_ENGINE_FP16_* in the header)
ENGINE_FP16_WEIGHTS, ENGINE_FP16_KV = 1, 2


def engine_flags(dtype) -> int:
    """The ctb_gpt_engine_begin_ex flags of a slot engine's ``dtype``: torch.float32 (0) or torch.float16 (fp16 layer
    weights and KV cache).  Anything else raises ValueError; nothing touches the device."""
    import torch

    if dtype is None or dtype == torch.float32:
        return 0
    if dtype == torch.float16:
        return ENGINE_FP16_WEIGHTS | ENGINE_FP16_KV
    raise ValueError(f"slot engine dtype must be torch.float32 or torch.float16, not {dtype!r}")


#: ctb_gpt_engine_prefill_chunk: a chunk's first column, and every chunk but a prompt's last, are multiples of this
PREFILL_CHUNK_ALIGN = 128


#: CTB_ABI_VERSION of include/chattts_b200.h this binding is written for
ABI_VERSION = 4

#: the decode steps ctb_gpt_step_kind reports (CTB_STEP_* in the header)
STEP_FLOW_INK, STEP_FLOW, STEP_MEGA, STEP_FMA, STEP_WGMMA = 1, 2, 3, 4, 5
STEP_NAMES = {STEP_FLOW_INK: "k_flow+ink", STEP_FLOW: "k_flow", STEP_MEGA: "k_step", STEP_FMA: "fma", STEP_WGMMA: "wgmma"}


def step_kind(handle, B: int, infer_text: bool = False) -> int:
    """ctb_gpt_step_kind: which decode step serves a static batch of ``B`` rows on ``handle`` (a STEP_* value)."""
    kind = load().ctb_gpt_step_kind(handle, int(B), int(bool(infer_text)))
    check(min(kind, 0))
    return kind


#: slot states reported by ctb_gpt_engine_status (CTB_SLOT_* in the header)
SLOT_IDLE, SLOT_RUNNING, SLOT_FINISHED = 0, 1, 2

#: ctb_gpt_engine_reserve: the KV pool's free pages cannot cover the call (CTB_ERR_POOL)
ERR_POOL = -5
#: tokens per KV page
PAGE_TOKENS = 16


class SlotImage(C.Structure):
    """The header of a suspended slot's image (ctb_slot_image)."""
    _fields_ = [("magic", C.c_uint32)] + [(n, C.c_int32) for n in (
        "prec", "seq_len", "pos", "end_idx", "finish", "n_gen", "npages", "page_bytes", "num_vq", "hidden_size",
        "noise_floats", "has_hidden")] + [
        ("row", C.c_int32 * 8), ("reserved", C.c_int32 * 3), ("sampler", SamplerConfig)] + [
        (n, C.c_uint64) for n in ("off_noise", "off_ids", "off_hiddens", "off_kv", "bytes")]


class ConvStackConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "idim", "odim", "hidden", "n_layer", "bn_dim", "kernel", "dilation", "out_dim", "vq_dim", "vq_groups",
        "vq_residual", "vq_levels")]


class VocosConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("input_channels", "dim", "intermediate_dim", "num_layers", "n_fft",
                                         "hop_length")]


#: every symbol include/chattts_b200.h declares (checked by tests/test_abi.py)
EXPORTS = (
    "ctb_abi_version", "ctb_last_error", "ctb_launch_count", "ctb_gpt_layout_query", "ctb_gpt_create",
    "ctb_gpt_destroy", "ctb_gpt_step_kind", "ctb_gpt_begin", "ctb_gpt_decode", "ctb_gpt_status_query", "ctb_gpt_attention_maps", "ctb_gpt_score", "ctb_gpt_profile_kernel", "ctb_gpt_debug_trace", "ctb_gpt_embed_prompt", "ctb_sample",
    "ctb_gpt_engine_begin", "ctb_gpt_engine_admit", "ctb_gpt_engine_admit_text", "ctb_gpt_engine_status",
    "ctb_gpt_engine_cancel", "ctb_gpt_engine_begin_ex", "ctb_gpt_engine_prefill_chunk",
    "ctb_gpt_engine_begin_paged", "ctb_gpt_engine_reserve", "ctb_gpt_engine_release", "ctb_gpt_engine_pages",
    "ctb_gpt_engine_suspend_bytes",
    "ctb_gpt_engine_suspend", "ctb_gpt_engine_resume", "ctb_gpt_engine_share_prompt", "ctb_gpt_engine_logprobs",
    "ctb_token_logprobs", "ctb_gpt_engine_top_logprobs", "ctb_token_top_logprobs", "ctb_gpt_score_ex",
    "ctb_dvae_blob_floats", "ctb_vocos_blob_floats", "ctb_decoder_create", "ctb_decoder_destroy",
    "ctb_dvae_decode", "ctb_vocos_decode", "ctb_decode_rows",
    "ctb_dvae_encoder_blob_floats", "ctb_dvae_encoder_create", "ctb_dvae_encoder_destroy", "ctb_dvae_encode",
    "ctb_dvae_encode_rows",
)


class CtbError(RuntimeError):
    pass


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True):
    """Load (building in-tree first if needed) and type the C ABI."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = lib_path()
        if build_if_missing:
            # build() is a no-op when the digest of csrc/ + include/ matches the stamp beside the library, so an
            # edited kernel is never silently ignored; a box without nvcc keeps using the library that travelled
            try:
                _build.build()
            except Exception:
                if not os.path.exists(path):
                    raise
        if not os.path.exists(path):
            raise CtbError(f"{path} missing: run `python -m chattts_b200.build`")
        lib = C.CDLL(path)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
        lib.ctb_abi_version.restype = C.c_int
        lib.ctb_last_error.restype = C.c_char_p
        lib.ctb_launch_count.restype = C.c_uint64
        lib.ctb_gpt_layout_query.argtypes = [C.POINTER(GptConfig), C.POINTER(GptLayout)]
        lib.ctb_gpt_create.argtypes = [C.POINTER(GptConfig), vp, C.POINTER(vp)]
        lib.ctb_gpt_destroy.argtypes = [vp]
        lib.ctb_gpt_step_kind.argtypes = [vp, i32, i32]
        lib.ctb_gpt_begin.argtypes = [vp, i32, i32, vp, vp, C.POINTER(SamplerConfig), vp, i32, i32, vp, vp, vp]
        lib.ctb_gpt_decode.argtypes = [vp, i32, vp]
        lib.ctb_gpt_status_query.argtypes = [vp, C.POINTER(GptStatus), vp, vp, vp]
        lib.ctb_gpt_profile_kernel.argtypes = [vp, i32, vp]
        lib.ctb_gpt_debug_trace.argtypes = [vp, vp, i32]
        lib.ctb_gpt_embed_prompt.argtypes = [vp, vp, vp, i32, i32, vp, vp]
        lib.ctb_gpt_attention_maps.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, vp]
        lib.ctb_gpt_score.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32, vp, vp]
        lib.ctb_gpt_engine_begin.argtypes = [vp, i32, i32, vp, vp, vp]
        lib.ctb_gpt_engine_begin_ex.argtypes = [vp, i32, i32, i32, vp, vp, vp]
        lib.ctb_gpt_engine_admit.argtypes = [vp, i32, vp, i32, vp, vp, C.POINTER(SamplerConfig), vp, vp, vp]
        lib.ctb_gpt_engine_admit_text.argtypes = lib.ctb_gpt_engine_admit.argtypes
        lib.ctb_gpt_engine_status.argtypes = [vp, C.POINTER(GptStatus), vp, vp, vp, vp]
        lib.ctb_gpt_engine_cancel.argtypes = [vp, i32, vp, vp]
        lib.ctb_gpt_engine_prefill_chunk.argtypes = [vp, i32, i32, i32, i32, vp, i32, C.POINTER(SamplerConfig), vp, i32,
                                                     vp]
        lib.ctb_gpt_engine_begin_paged.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp]
        lib.ctb_gpt_engine_reserve.argtypes = [vp, i32, vp, vp, vp]
        lib.ctb_gpt_engine_release.argtypes = [vp, i32, vp, vp]
        lib.ctb_gpt_engine_pages.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
        lib.ctb_gpt_engine_suspend_bytes.argtypes = [vp, i32, C.POINTER(C.c_uint64), vp]
        lib.ctb_gpt_engine_suspend.argtypes = [vp, i32, vp, C.c_uint64, vp]
        lib.ctb_gpt_engine_resume.argtypes = [vp, i32, vp, C.c_uint64, vp]
        lib.ctb_gpt_engine_share_prompt.argtypes = [vp, i32, i32, i32, i32, vp]
        lib.ctb_gpt_engine_logprobs.argtypes = [vp, vp, vp]
        lib.ctb_token_logprobs.argtypes = [vp, i32, i32, vp, vp, vp]
        lib.ctb_gpt_engine_top_logprobs.argtypes = [vp, i32, vp, vp, vp]
        lib.ctb_token_top_logprobs.argtypes = [vp, i32, i32, i32, vp, vp, vp]
        lib.ctb_gpt_score_ex.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32, vp, i32, vp, vp, vp]
        lib.ctb_sample.argtypes = [vp, i32, i32, i32, C.POINTER(SamplerConfig), vp, vp, i32, i32, i32, vp, vp]
        lib.ctb_dvae_blob_floats.argtypes = [C.POINTER(ConvStackConfig)]
        lib.ctb_dvae_blob_floats.restype = i64
        lib.ctb_vocos_blob_floats.argtypes = [C.POINTER(VocosConfig)]
        lib.ctb_vocos_blob_floats.restype = i64
        lib.ctb_decoder_create.argtypes = [C.POINTER(ConvStackConfig), vp, C.POINTER(VocosConfig), vp, i32, i32,
                                           C.POINTER(vp)]
        lib.ctb_decoder_destroy.argtypes = [vp]
        lib.ctb_dvae_decode.argtypes = [vp, vp, i32, i32, i32, vp, vp]
        lib.ctb_vocos_decode.argtypes = [vp, vp, i32, i32, vp, vp]
        lib.ctb_decode_rows.argtypes = [vp, i32, i32, C.POINTER(vp), C.POINTER(i32), vp, i64, vp]
        lib.ctb_dvae_encoder_blob_floats.argtypes = [C.POINTER(ConvStackConfig)]
        lib.ctb_dvae_encoder_blob_floats.restype = i64
        lib.ctb_dvae_encoder_create.argtypes = [C.POINTER(ConvStackConfig), vp, i64, C.POINTER(vp)]
        lib.ctb_dvae_encoder_destroy.argtypes = [vp]
        lib.ctb_dvae_encode.argtypes = [vp, vp, i64, vp, i32, C.POINTER(i32), vp, vp, vp]
        lib.ctb_dvae_encode_rows.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(i64), vp, i32, C.POINTER(i32), vp, vp]
        if lib.ctb_abi_version() != ABI_VERSION:
            raise CtbError("ABI version mismatch")
        _lib = lib
        return lib


def check(rc: int) -> None:
    if rc != 0:
        raise CtbError(f"chattts_b200 error {rc}: {load().ctb_last_error().decode()}")


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise CtbError("chattts_b200 needs a CUDA device (sm_90a); there is no CPU path")
