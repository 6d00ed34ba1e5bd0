"""Decode attention (k_attn, fp32 and fp16 caches) and the prompt kernels at long contexts, against float64.

``k_attn`` is the attention of every slot engine and of static batches of 5 or more.  Its grid is
min(ceil(2 * 132 / (12 * S)), ceil(max_context / 128)) split CTAs per (row, head) - 11 at S = 2, 2 at S = 12, 1 at
S = 24 - and a CTA walks chunks split, split + grid.x, ... of 128 keys with a running softmax, then the last CTA merges
the partials.  The requests here take rows to 300 .. 2048 keys (up to 128 KV pages of 16 tokens), so every one of
chunk wrap (S = 12 past 256 keys, S = 24 past 128), the merge of up to 11 partials (S = 2) and long page walks runs;
prompts of 8 .. 1024 tokens run the batched prefill (k_prefill_rope_kv, k_prefill_attn) at its full admitted range.

Every request is compared with the float64 reference of tests/f64_oracle.py, teacher-forced along the GPU's ids (one
causal pass per request, run on the GPU in float64 by torch).  Ids: each step's must be the reference's sampled id
unless its decision margin (argmax, top-p cut, top-k cut) is below MARGIN.  Hidden states, every step of every request:
* fp32 engine: step 0 (the prefill's token, through its 3xTF32 GEMMs) within 2e-4, later steps within 6e-5;
* fp16 engine: every step within 1.2e-3, and the root mean square of a request's errors within 4e-5.  The mean square
  is what sees a biased fp16 rounding of the appended K/V: the synthetic model's near-uniform attention averages V over
  hundreds of keys, so a one-ulp bias moves no single step far, but it moves every step.

A. fp32 engine at S = 2, 12, 24.  B. the same workload on the half-precision engine (fp16 weights + cache, and the
fp16 cache alone on fp32 weights) against the fp16 model's float64 reference.  C. peaked attention: q_proj and k_proj
x 4, so scores have std ~5 and a query's scores spread over ~30 across 1000 keys (tests/test_f64_oracle_cpu.py checks
these numbers on the CPU, and that the largest |K| the fp16 cache holds, ~12, is far below fp16's 65504).  Peaked
softmax amplifies rounding differences: on the fp16 engine the bars are 4x the distance of an fp32 evaluation of the
same model (the reference's code in float32, K/V rounded to fp16) from the float64 reference - that distance is ~5e-3
here, and the engine's about the same.  On the fp32 engine the bar is 1e-3 on every step: the engine is at ~3e-4, its
prompt K/V coming from the prefill's 3xTF32 GEMMs (operands kept to ~22 bits, against fp32's 24), while the float32
evaluation, whose GEMMs are plain fp32, stays at ~2e-5, so a multiple of it does not measure the engine's arithmetic.
D. static batches of 6 (PDL FMA chain) and 12 (wgmma step) on k_attn: ragged prompts to 512 tokens, 800 steps.
E. slot reuse: a 1500-key request, then a short one and a 1000-key one in the same slot give, bit for bit, what they
give in a fresh engine (no K/V of an earlier occupant and no split counter leaks).

Runs in ~2 minutes on one H100, the float64 references included.
"""
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.engine import EngineDevice, Request, schedule
from chattts_b200.gpt import GPT
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from f64_oracle import F64Oracle, peaked_state, sample_trace
from gpu_util import release_on_teardown
from oracle.gpt_oracle import SamplerParams, exp_noise

pytestmark = pytest.mark.gpu

W16, KV16 = _lib.ENGINE_FP16_WEIGHTS, _lib.ENGINE_FP16_KV
FP16 = W16 | KV16
EOS = 625
MAX_CONTEXT = 2048
CAP = 1024  # the engines' max_new capacity
MARGIN = 1e-3
# Bars (module docstring); in brackets the largest distance observed on one H100 80 GB HBM3 (132 SMs)
FP32_ATOL = 2e-4  # step 0, the prefill's token [8.9e-5]: the bar of test_gpu_gpt.py::test_long_context_vs_oracle
FP32_DECODE_ATOL = 6e-5  # steps 1.. [1.6e-5]
FP16_ATOL = 1.2e-3  # every step [3.4e-4]
FP16_RMS = 4e-5  # root mean square over a request's steps and dims [1.3e-5]
PEAKED_FP32_ATOL = 1e-3  # peaked model, fp32 engine, every step [3.3e-4]
PEAK_FACTOR = 4.0  # peaked model, fp16 engine: this multiple of the fp32 evaluation's distance [~1x]

# (prompt tokens, max_new = min_new): rows end at ~300, 700, 1100, 1500 keys, and one at exactly max_context
WORKLOAD = [(8, 292), (40, 660), (300, 800), (512, 988), (1024, 476), (1024, 1024)]
PARAMS = [(0.7, 20, 1.05), (None, 20, 1.0), (0.5, None, 1.05), (0.7, 20, 1.0), (0.95, 3, 1.2), (None, None, 1.05)]
TEMPS = [[0.3, 0.5, 0.7, 1.0], [0.7] * 4, [1.0, 0.3, 0.3, 0.5], [0.5] * 4, [0.3] * 4, [1.0] * 4]

_models, _oracles, _refs = {}, {}, {}
_release = release_on_teardown(_models, _oracles, _refs)  # two 32 x 2048 engines, float64 oracles


def _model(kind):
    """'plain': the synthetic model; 'peaked': its q_proj and k_proj x 4.  One handle each, 32 rows x 2048 tokens."""
    if kind not in _models:
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        if kind == "peaked":
            gs = peaked_state(gs)
        cfg = Config()
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=32, max_context=MAX_CONTEXT)
        gpt.load_state(gs)
        _models[kind] = (gpt, embed, gs, es)
    return _models[kind]


def _oracle(kind, flags, dtype=torch.float64):
    key = (kind, bool(flags & W16), bool(flags & KV16), dtype)
    if key not in _oracles:
        _, _, gs, es = _model(kind)
        _oracles[key] = F64Oracle(gs, es, fp16_layers=key[1], fp16_kv=key[2], dtype=dtype, device="cuda")
    return _oracles[key]


def _specs(workload=WORKLOAD, base=0):
    return [dict(key=("engine", base, i), prompt=synth_prompt_batch([L], seed=400 + base + i)[0][0], max_new=n,
                 seed=2000 + base + 13 * i, params=PARAMS[i % len(PARAMS)], temp=TEMPS[i % len(TEMPS)])
            for i, (L, n) in enumerate(workload)]


def _request(embed, s):
    L = s["prompt"].shape[0]
    tp, tk, rp = s["params"]
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    return Request(emb=embed(s["prompt"][None], torch.ones(1, L, dtype=torch.bool))[0], temperature=s["temp"],
                   eos_token=EOS, max_new_token=s["max_new"], min_new_token=s["max_new"],
                   logits_processors=(*proc, *warp), manual_seed=s["seed"])


def _engine(gpt, reqs, slots, flags, chunk=64):
    """Every request through one engine of ``slots`` slots -> {index: (ids, hiddens)} (host copies)."""
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, CAP, True, flags)
        for i, slot, n in schedule(reqs, dev, chunk):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
            o.destroy()
    return got


def _reference(kind, flags, s, ids, noise, dtype=torch.float64):
    """(hidden states, sampled ids, decision margins) of the model teacher-forced along ``ids``; cached per content,
    so runs that produced the same ids share one reference."""
    key = (kind, flags & FP16, dtype, s["key"], noise[1], ids.numpy().tobytes())
    if key not in _refs:
        orc = _oracle(kind, flags, dtype)
        hid, lg = orc.teacher_forced(orc.embed_prompt(s["prompt"]), ids)
        tp, tk, rp = s["params"]
        sp = SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp)
        sampled, margins = (None, None) if dtype != torch.float64 else sample_trace(
            lg, ids, torch.tensor(s["temp"]), sp, noise[0], EOS, s["max_new"])
        _refs[key] = (hid.cpu(), sampled, margins)
    return _refs[key]


def _check(tag, kind, flags, specs, got, noise_of=None):
    """Ids and hidden states of every request against the float64 reference (module docstring for the bars)."""
    worst0 = worst = worst_rms = worst32 = 0.0
    accepted = total = 0
    for i, s in enumerate(specs):
        ids, hid = got[i]
        assert ids.shape[0] == s["max_new"], (tag, i, ids.shape)
        noise = noise_of(i) if noise_of else (exp_noise(4, EOS + 1, s["seed"]), (1, 0))
        ref, sampled, margins = _reference(kind, flags, s, ids, noise)
        for t in range(ids.shape[0]):
            total += 1
            if not torch.equal(sampled[t], ids[t].long()):
                assert margins[t] < MARGIN, (tag, i, t, ids[t].tolist(), sampled[t].tolist(), float(margins[t]))
                accepted += 1
        e = (hid.double() - ref).abs()
        e0, ed, rms = float(e[0].max()), float(e[1:].max()), float(e.pow(2).mean().sqrt())
        bar0, bar, rms_bar = (FP16_ATOL, FP16_ATOL, FP16_RMS) if flags else (FP32_ATOL, FP32_DECODE_ATOL, None)
        if kind == "peaked":
            e32 = (_reference(kind, flags, s, ids, noise, torch.float32)[0].double() - ref).abs()
            worst32 = max(worst32, float(e32.max()))
            if flags:
                bar0 = bar = max(FP16_ATOL, PEAK_FACTOR * float(e32.max()))
                rms_bar = max(FP16_RMS, PEAK_FACTOR * float(e32.pow(2).mean().sqrt()))
            else:
                bar0 = bar = PEAKED_FP32_ATOL
        worst0, worst, worst_rms = max(worst0, e0), max(worst, ed), max(worst_rms, rms)
        L = s["prompt"].shape[0]
        assert e0 < bar0, (tag, i, L, s["max_new"], "step 0", e0, bar0)
        assert ed < bar, (tag, i, L, s["max_new"], "steps 1..", ed, bar)
        if rms_bar is not None:
            assert rms < rms_bar, (tag, i, L, s["max_new"], "rms", rms, rms_bar)
    extra = f"; fp32 evaluation's own max distance {worst32:.3e}" if kind == "peaked" else ""
    print(f"\n{tag}: max |hidden - f64| at step 0 {worst0:.3e}, at steps 1.. {worst:.3e}, largest per-request rms "
          f"{worst_rms:.3e}{extra}; margin-accepted steps {accepted} of {total}")


# ---------------------------------------------------------------------------------------------------- A, B
@pytest.mark.parametrize("slots", [2, 12, 24])
def test_a_fp32_engine_long_contexts(slots):
    gpt, embed, _, _ = _model("plain")
    specs = _specs()
    got = _engine(gpt, [_request(embed, s) for s in specs], slots, 0)
    _check(f"A S={slots}", "plain", 0, specs, got)


@pytest.mark.parametrize("slots,flags", [(2, FP16), (12, FP16), (24, FP16), (2, KV16)])
def test_b_fp16_engine_long_contexts(slots, flags):
    gpt, embed, _, _ = _model("plain")
    specs = _specs()
    got = _engine(gpt, [_request(embed, s) for s in specs], slots, flags)
    _check(f"B S={slots} flags={flags}", "plain", flags, specs, got)


# ---------------------------------------------------------------------------------------------------- C
@pytest.mark.parametrize("slots,flags", [(2, 0), (24, 0), (2, FP16), (24, FP16)])
def test_c_peaked_attention(slots, flags):
    gpt, embed, _, _ = _model("peaked")
    specs = _specs(base=50)
    got = _engine(gpt, [_request(embed, s) for s in specs], slots, flags)
    _check(f"C S={slots} flags={flags}", "peaked", flags, specs, got)


# ---------------------------------------------------------------------------------------------------- D
STATIC = {6: [512, 37, 300, 8, 129, 256], 12: [512, 8, 300, 40, 130, 450, 17, 256, 511, 77, 200, 390]}


@pytest.mark.parametrize("B", [6, 12])
def test_d_static_batches_on_k_attn(B):
    gpt, embed, _, _ = _model("plain")
    lengths, steps, seed = STATIC[B], 800, 90 + B
    ids, mask, tmask = synth_prompt_batch(lengths, seed=70 + B)
    temp = [0.3, 0.5, 0.7, 1.0]
    warp, proc = gen_logits(num_code=EOS, top_P=0.7, top_K=20, repetition_penalty=1.05)
    out = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor(temp), eos_token=EOS,
                            attention_mask=mask, max_new_token=steps, min_new_token=steps,
                            logits_processors=(*proc, *warp), return_hidden=True, show_tqdm=False,
                            manual_seed=seed))[-1]
    q = exp_noise(4 * B, EOS + 1, seed)  # row b samples with rows 4b .. 4b + 3 of the batch's noise
    specs = [dict(key=("static", B, b), prompt=ids[b, -L:], max_new=steps, seed=seed, params=(0.7, 20, 1.05), temp=temp)
             for b, L in enumerate(lengths)]
    got = {b: (out.ids[b].cpu(), out.hiddens[b].cpu()) for b in range(B)}
    _check(f"D B={B}", "plain", 0, specs, got, lambda b: (q[4 * b: 4 * b + 4], (B, b)))


# ---------------------------------------------------------------------------------------------------- E
def _in_slot_zero(gpt, reqs, flags, order):
    """Requests ``order`` one after another in slot 0 of one engine of 2 slots -> [(ids, hiddens)]."""
    outs = []
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 2, CAP, True, flags)
        for i in order:
            dev.admit([(0, i)])
            while True:
                st = dev.status()
                if st.state[0] == _lib.SLOT_FINISHED:
                    break
                dev.decode(64)
            o = dev.harvest(0, st.end_idx[0])
            outs.append((o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone()))
            o.destroy()
    return outs


@pytest.mark.parametrize("flags", [0, FP16])
def test_e_slot_reuse_leaks_nothing(flags):
    gpt, embed, _, _ = _model("plain")
    specs = _specs([(512, 988), (8, 40), (40, 960)], base=80)
    reqs = [_request(embed, s) for s in specs]
    reused = _in_slot_zero(gpt, reqs, flags, [0, 1, 2])
    for k in (1, 2):
        fresh = _in_slot_zero(gpt, reqs, flags, [k])[0]
        assert reused[k][0].shape[0] == specs[k]["max_new"]
        assert torch.equal(reused[k][0], fresh[0]), (flags, k)
        assert torch.equal(reused[k][1], fresh[1]), (flags, k, float((reused[k][1] - fresh[1]).abs().max()))
