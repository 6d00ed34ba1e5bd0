"""The half-precision slot engine's definition on the CPU: the fp16 oracle's transforms, its reduction to the fp32
oracle, the dtype argument's checks and the C ABI symbol."""
import ctypes
import os

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from fp16_oracle import GPTOracleFp16, fp16_layer_state
from oracle.gpt_oracle import GPTOracle, SamplerParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _small_state(seed=0):
    """A two-layer cut of the synthetic model (the oracle's cost is per layer)."""
    gs = synth_gpt_state(seed)
    return {k: v for k, v in gs.items() if not k.startswith("layers.") or int(k.split(".")[1]) < 2}


def test_layer_transform_is_the_definition():
    gs = _small_state()
    for l in range(2):
        p = f"layers.{l}."
        gs[p + "input_layernorm.weight"] = 1 + 0.1 * torch.randn(768)
        gs[p + "post_attention_layernorm.weight"] = 1 + 0.1 * torch.randn(768)
    s = fp16_layer_state(gs)
    for l in range(2):
        p = f"layers.{l}."
        for m, norm in (("self_attn.q_proj", "input_layernorm"), ("self_attn.k_proj", "input_layernorm"),
                        ("self_attn.v_proj", "input_layernorm"), ("mlp.gate_proj", "post_attention_layernorm"),
                        ("mlp.up_proj", "post_attention_layernorm")):
            W, ln = gs[p + m + ".weight"], gs[p + norm + ".weight"]
            assert torch.equal(s[p + m + ".weight"], (W * ln).half().float()), (l, m)
        for m in ("self_attn.o_proj", "mlp.down_proj"):
            assert torch.equal(s[p + m + ".weight"], gs[p + m + ".weight"].half().float()), (l, m)
        assert torch.equal(s[p + "input_layernorm.weight"], torch.ones(768))
        assert torch.equal(s[p + "post_attention_layernorm.weight"], torch.ones(768))
    for k in ("norm.weight",):
        assert torch.equal(s[k], gs[k])


def _run(orc, n=6, length=9):
    ids, mask, tmask = synth_prompt_batch([length], seed=4)
    return orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.7] * 4), 625, attention_mask=mask,
                        max_new_token=n, min_new_token=n, sampler=SamplerParams(), return_hidden=True, manual_seed=11,
                        trace=True)


def test_fp16_layers_reduce_to_fp32_on_representable_weights():
    """Unit norms and fp16-representable layer matrices: the fp16-layer oracle is the fp32 oracle, exactly."""
    gs = fp16_layer_state(_small_state())
    es = synth_embed_state(1)
    a = _run(GPTOracle(gs, es))
    b = _run(GPTOracleFp16(gs, es, fp16_layers=True, fp16_kv=False))
    assert torch.equal(a.ids[0], b.ids[0])
    assert torch.equal(a.hiddens[0], b.hiddens[0])


def test_fp16_kv_rounds_the_cache():
    gs, es = _small_state(), synth_embed_state(1)
    orc = GPTOracleFp16(gs, es, fp16_layers=True, fp16_kv=True)
    seen = []
    base = orc.forward

    def spy(x, positions, key_mask, past):
        out, new_past = base(x, positions, key_mask, past)
        seen.append(new_past)
        return out, new_past

    orc.forward = spy
    out = _run(orc, n=3)
    assert out.ids[0].shape[0] == 3 and len(seen) == 3
    for new_past in seen:
        for k, v in new_past:
            assert torch.equal(k, k.half().float()) and torch.equal(v, v.half().float())
    # and the rounding changes the cache of the fp32 model (the test is not vacuous)
    k32 = GPTOracleFp16(gs, es, fp16_layers=True, fp16_kv=False)
    ids, mask, tmask = synth_prompt_batch([9], seed=4)
    _, past = k32.forward(k32.embed_prompt(ids, tmask), torch.arange(9.0)[None], torch.ones(1, 9, dtype=torch.bool),
                          None)
    assert not torch.equal(past[0][0], past[0][0].half().float())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float64, torch.int8, "float16"])
def test_engine_dtype_rejected_before_any_device_call(dtype, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device touched")

    monkeypatch.setattr(_lib, "load", no_device)
    monkeypatch.setattr(_lib, "require_cuda", no_device)
    with pytest.raises(ValueError, match="float32 or torch.float16"):
        _lib.engine_flags(dtype)
    from chattts_b200.core import Chat
    from chattts_b200.gpt import GPT

    g = GPT.__new__(GPT)  # no handle: any device work would fail differently
    with pytest.raises(ValueError):
        next(g.generate_continuous([object()], dtype=dtype))
    with pytest.raises(ValueError):
        next(g.generate_continuous_stream([object()], dtype=dtype))
    with pytest.raises(ValueError):
        g.open_engine(2, 16, dtype=dtype)
    c = Chat.__new__(Chat)
    with pytest.raises(ValueError):
        c.infer_continuous(["x"], dtype=dtype)
    with pytest.raises(ValueError):
        c.infer_continuous_stream(["x"], dtype=dtype)
    with pytest.raises(ValueError):
        next(c.refine_continuous(["x"], dtype=dtype))
    with pytest.raises(ValueError):
        c.open_engine(dtype=dtype)


def test_engine_flags():
    assert _lib.engine_flags(torch.float32) == 0
    assert _lib.engine_flags(torch.float16) == _lib.ENGINE_FP16_WEIGHTS | _lib.ENGINE_FP16_KV == 3


def test_library_exports_begin_ex():
    from chattts_b200 import build

    build.build()
    lib = ctypes.CDLL(build.LIB_PATH)
    assert hasattr(lib, "ctb_gpt_engine_begin_ex")
    assert "ctb_gpt_engine_begin_ex" in _lib.EXPORTS
    header = open(os.path.join(ROOT, "include", "chattts_b200.h")).read()
    assert "#define CTB_ENGINE_FP16_WEIGHTS 1" in header and "#define CTB_ENGINE_FP16_KV 2" in header
