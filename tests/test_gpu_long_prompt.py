"""Prompts of 1,025 .. max_context - 1 tokens on the slot engine: the tiled causal prefill attention
(k_prefill_attn_tiled, chosen when an admission's padded width T0 exceeds 1,024) against float64.

A prompt over 1,024 tokens is not bit-equal to a static ``GPT.generate`` of it: a static batch walks such a prompt's
columns through the decode kernels, the engine prefills it with token-parallel GEMMs and the tiled kernel.  The contract
is the float64 reference of tests/f64_oracle.py, teacher-forced along the engine's ids: each step's id must be the
reference's sampled id unless its decision margin (argmax, top-p cut, top-k cut) is below MARGIN, and hidden states
meet the bars of test_gpu_long_attention.py:
* fp32 engine: step 0 (the prefill's token) within 2e-4, later steps within 6e-5;
* fp16 engine (FP16, and KV16 alone): every step within 1.2e-3, a request's root mean square within 4e-5;
* peaked model (q_proj, k_proj x 4), fp32 engine: every step within 1e-3.
The longer prefill needed no wider bar.  Largest distances seen on one H100 80 GB HBM3 (each test prints its own):
fp32 step 0 9.1e-5, later steps 1.0e-5; fp16 1.0e-4 per step, 5.3e-6 RMS; peaked 3.8e-4; no step needed the margin
rule.

A. fp32 engine at S = 2 and 12: prompts of 1,025, 1,536, 2,047, 3,000 and 4,000 tokens, forced lengths, the last row
ending exactly at max_context (4,000 + 96).  B. the same on the half-precision engines.  C. the peaked model at 2,048 and
4,000 tokens.  D. left padding through the C ABI: one ctb_gpt_engine_admit of a 1,100- and a 3,000-token prompt padded
to 3,000 columns gives, bit for bit, what each gives admitted alone.  E. a 3,000-token prompt and 15 short ones at one
poll: the short ones are one prefill, bit-equal to the same engine without the long one, and the long one is prefilled
alone.  F. slot reuse after a 4,000-token request.  G. a 1,500-token prompt against static ``generate`` at B = 1.
H. ``Chat`` with a speaker sample of 1,100 codes, and a split-text paragraph whose sentence 0 has 1,100 codes.
I. the limits.

Runs in about 35 s on one H100, the float64 references included.
"""
import ctypes as C

import numpy as np
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
MAX_CONTEXT = 4096
CAP = 320  # the engines' max_new capacity
MARGIN = 1e-3
FP32_ATOL = 2e-4
FP32_DECODE_ATOL = 6e-5
FP16_ATOL = 1.2e-3
FP16_RMS = 4e-5
PEAKED_FP32_ATOL = 1e-3
ERR_ARG = -1  # CTB_ERR_ARG

WORKLOAD = [(1025, 200), (1536, 300), (2047, 150), (3000, 120), (4000, 96)]  # 4000 + 96 = max_context
PARAMS = [(0.7, 20, 1.05), (None, 20, 1.0), (0.5, None, 1.05), (0.7, 20, 1.0), (0.95, 3, 1.2)]
TEMPS = [[0.3, 0.5, 0.7, 1.0], [0.7] * 4, [1.0, 0.3, 0.3, 0.5], [0.5] * 4, [0.3] * 4]

_models, _oracles, _refs = {}, {}, {}
_release = release_on_teardown(_models, _oracles, _refs)


def _model(kind):
    """'plain': the synthetic model; 'peaked': its q_proj and k_proj x 4.  One handle each, 16 rows x 4096 tokens."""
    if kind not in _models:
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        if kind == "peaked":
            gs = peaked_state(gs)
        cfg = Config()
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=16, max_context=MAX_CONTEXT)
        gpt.load_state(gs)
        _models[kind] = (gpt, embed, gs, es)
    return _models[kind]


def _oracle(kind, flags):
    key = (kind, bool(flags & W16), bool(flags & KV16))
    if key not in _oracles:
        _, _, gs, es = _model(kind)
        _oracles[key] = F64Oracle(gs, es, fp16_layers=key[1], fp16_kv=key[2], device="cuda")
    return _oracles[key]


def _specs(workload=WORKLOAD, base=0):
    return [dict(key=(base, i), prompt=synth_prompt_batch([L], seed=500 + base + i)[0][0], max_new=n,
                 seed=3000 + base + 13 * i, params=PARAMS[i % len(PARAMS)], temp=TEMPS[i % len(TEMPS)])
            for i, (L, n) in enumerate(workload)]


def _request(embed, s):
    L = s["prompt"].shape[0]
    tp, tk, rp = s["params"]
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    return Request(emb=embed(s["prompt"][None], torch.ones(1, L, dtype=torch.bool))[0], temperature=s["temp"],
                   eos_token=EOS, max_new_token=s["max_new"], min_new_token=s["max_new"],
                   logits_processors=(*proc, *warp), manual_seed=s["seed"])


def _engine(gpt, reqs, slots, flags, chunk=64, spy=None):
    """Every request through one engine of ``slots`` slots -> {index: (ids, hiddens)} (host copies).  ``spy``: a list
    that receives the request indices of every prefill."""
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, CAP, True, flags)
        if spy is not None:
            admit_one = dev._admit
            dev._admit = lambda group, *a: (spy.append([i for _, i in group]), admit_one(group, *a))
        for i, slot, n in schedule(reqs, dev, chunk):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
            o.destroy()
    return got


def _reference(kind, flags, s, ids):
    key = (kind, flags & FP16, s["key"], ids.numpy().tobytes())
    if key not in _refs:
        orc = _oracle(kind, flags)
        hid, lg = orc.teacher_forced(orc.embed_prompt(s["prompt"]), ids)
        tp, tk, rp = s["params"]
        sp = SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp)
        sampled, margins = sample_trace(lg, ids, torch.tensor(s["temp"]), sp, exp_noise(4, EOS + 1, s["seed"]), EOS,
                                        s["max_new"])
        _refs[key] = (hid.cpu(), sampled, margins)
    return _refs[key]


def _check(tag, kind, flags, specs, got):
    """Ids and hidden states of every request against the float64 reference (module docstring for the bars)."""
    worst0 = worst = worst_rms = 0.0
    accepted = total = 0
    for i, s in enumerate(specs):
        ids, hid = got[i]
        assert ids.shape[0] == s["max_new"], (tag, i, ids.shape)
        ref, sampled, margins = _reference(kind, flags, s, ids)
        for t in range(ids.shape[0]):
            total += 1
            if not torch.equal(sampled[t], ids[t].long()):
                assert margins[t] < MARGIN, (tag, i, t, ids[t].tolist(), sampled[t].tolist(), float(margins[t]))
                accepted += 1
        e = (hid.double() - ref).abs()
        e0, rms = float(e[0].max()), float(e.pow(2).mean().sqrt())
        ed = float(e[1:].max()) if e.shape[0] > 1 else 0.0
        bar0, bar, rms_bar = (FP16_ATOL, FP16_ATOL, FP16_RMS) if flags else (FP32_ATOL, FP32_DECODE_ATOL, None)
        if kind == "peaked":
            bar0 = bar = PEAKED_FP32_ATOL
        worst0, worst, worst_rms = max(worst0, e0), max(worst, ed), max(worst_rms, rms)
        L = s["prompt"].shape[0]
        assert e0 < bar0, (tag, i, L, "step 0", e0, bar0)
        assert ed < bar, (tag, i, L, "steps 1..", ed, bar)
        if rms_bar is not None:
            assert rms < rms_bar, (tag, i, L, "rms", rms, rms_bar)
    print(f"\n{tag}: max |hidden - f64| at step 0 {worst0:.3e}, at steps 1.. {worst:.3e}, largest per-request rms "
          f"{worst_rms:.3e}; margin-accepted steps {accepted} of {total}")


def _run_alone(gpt, reqs, flags, groups, slots=2):
    """Each entry of ``groups`` (request indices) admitted by ONE ``EngineDevice._admit`` call (one
    ctb_gpt_engine_admit, left padded to the group's widest prompt) into slots 0.., then run to the end
    -> {index: (ids, hiddens)}."""
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, CAP, True, flags)
        for g in groups:
            pairs = list(enumerate(g))
            dev._admit(pairs, True, False, {})
            while True:
                st = dev.status()
                if all(st.state[s] == _lib.SLOT_FINISHED for s, _ in pairs):
                    break
                dev.decode(64)
            for s, i in pairs:
                o = dev.harvest(s, st.end_idx[s])
                got[i] = (o.ids[0].cpu().clone(), o.hiddens[0].cpu().clone())
                o.destroy()
    return got


# ---------------------------------------------------------------------------------------------------- A, B, C
@pytest.mark.parametrize("slots", [2, 12])
def test_a_fp32_engine_long_prompts(slots):
    gpt, embed, _, _ = _model("plain")
    specs = _specs()
    _check(f"A S={slots}", "plain", 0, specs, _engine(gpt, [_request(embed, s) for s in specs], slots, 0))


@pytest.mark.parametrize("slots,flags", [(2, FP16), (12, FP16), (2, KV16)])
def test_b_fp16_engine_long_prompts(slots, flags):
    gpt, embed, _, _ = _model("plain")
    specs = _specs()
    _check(f"B S={slots} flags={flags}", "plain", flags, specs,
           _engine(gpt, [_request(embed, s) for s in specs], slots, flags))


def test_c_peaked_attention_long_prompts():
    gpt, embed, _, _ = _model("peaked")
    specs = _specs([(2048, 200), (4000, 96)], base=50)
    _check("C peaked", "peaked", 0, specs, _engine(gpt, [_request(embed, s) for s in specs], 2, 0))


# ---------------------------------------------------------------------------------------------------- D, E, F
@pytest.mark.parametrize("flags", [0, KV16])
def test_d_left_padded_admission_equals_lone_admissions(flags):
    gpt, embed, _, _ = _model("plain")
    specs = _specs([(1100, 64), (3000, 64)], base=60)
    reqs = [_request(embed, s) for s in specs]
    both = _run_alone(gpt, reqs, flags, [[0, 1]])  # one call, padded to 3,000 columns: prompt 0 has c0 = 1,900
    alone = _run_alone(gpt, reqs, flags, [[0], [1]])
    for i in (0, 1):
        assert torch.equal(both[i][0], alone[i][0]), (flags, i)
        assert torch.equal(both[i][1], alone[i][1]), (flags, i, float((both[i][1] - alone[i][1]).abs().max()))
    if not flags:
        _check("D", "plain", 0, specs, both)


def test_e_mixed_admission_prefills_the_long_prompt_alone():
    gpt, embed, _, _ = _model("plain")
    short = [(8, 40), (40, 60), (1024, 50), (300, 70), (17, 40), (512, 64), (129, 48), (77, 40),
             (1000, 56), (256, 40), (33, 44), (640, 40), (9, 52), (450, 40), (200, 60)]
    specs = _specs([(3000, 80)] + short, base=70)
    reqs = [_request(embed, s) for s in specs]
    prefills = []
    mixed = _engine(gpt, reqs, 16, 0, spy=prefills)
    assert prefills == [list(range(1, 16)), [0]], prefills
    without = _engine(gpt, reqs[1:], 16, 0)
    for k in range(15):
        assert torch.equal(mixed[k + 1][0], without[k][0]), k
        assert torch.equal(mixed[k + 1][1], without[k][1]), k
    _check("E long", "plain", 0, specs[:1], {0: mixed[0]})


@pytest.mark.parametrize("flags", [0, FP16])
def test_f_slot_reuse_after_a_long_prompt(flags):
    gpt, embed, _, _ = _model("plain")
    specs = _specs([(4000, 96), (1100, 120)], base=80)
    reqs = [_request(embed, s) for s in specs]
    reused = _run_alone(gpt, reqs, flags, [[0], [1]])
    fresh = _run_alone(gpt, reqs, flags, [[1]])
    assert reused[1][0].shape[0] == specs[1]["max_new"]
    assert torch.equal(reused[1][0], fresh[1][0]), flags
    assert torch.equal(reused[1][1], fresh[1][1]), (flags, float((reused[1][1] - fresh[1][1]).abs().max()))


# ---------------------------------------------------------------------------------------------------- G
def test_g_against_static_generate():
    """What "equal to GPT.generate" means above 1,024 tokens: the engine (token-parallel prefill, tiled attention) and
    a static batch of one (the prompt's columns walked through the decode kernels) give the same ids except at steps
    whose float64 decision margin is below MARGIN, and both meet the step bars against float64."""
    gpt, embed, _, _ = _model("plain")
    (s,) = _specs([(1500, 160)], base=90)
    eng = _engine(gpt, [_request(embed, s)], 2, 0)[0]
    L = s["prompt"].shape[0]
    tp, tk, rp = s["params"]
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    ids = s["prompt"][None]
    out = list(gpt.generate(embed(ids, torch.ones(1, L, dtype=torch.bool)), ids, temperature=torch.tensor(s["temp"]),
                            eos_token=EOS, max_new_token=s["max_new"], min_new_token=s["max_new"],
                            logits_processors=(*proc, *warp), return_hidden=True, show_tqdm=False,
                            manual_seed=s["seed"]))[-1]
    static = (out.ids[0].cpu(), out.hiddens[0].cpu())
    out.destroy()
    _check("G engine", "plain", 0, [s], {0: eng})
    _check("G static", "plain", 0, [s], {0: static})
    _, _, margins = _reference("plain", 0, s, eng[0])
    differ = [t for t in range(s["max_new"]) if not torch.equal(eng[0][t], static[0][t])]
    if differ:  # the first step where the two differ must be a near-tie; later steps follow different histories
        assert margins[differ[0]] < MARGIN, (differ[0], float(margins[differ[0]]))
    else:
        assert (eng[1] - static[1]).abs().max() < FP32_DECODE_ATOL + FP32_ATOL
    print(f"\nG: engine and static ids differ at {len(differ)} of {s['max_new']} steps; max |engine - static| "
          f"hidden {float((eng[1] - static[1]).abs().max()):.3e}")


# ---------------------------------------------------------------------------------------------------- H
def _chat(max_batch=4):
    if "chat" not in _models:
        from chattts_b200 import Chat
        from chattts_b200.synth import synth_all
        from stubs import StubSpeaker, StubTokenizer

        c = Chat()
        assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                             max_batch=max_batch, max_context=MAX_CONTEXT)
        _models["chat"] = c
    return _models["chat"]


def _spy_prompt_widths(monkeypatch):
    """Record the padded width of every engine prefill."""
    widths = []
    admit_one = EngineDevice._admit

    def spy(self, group, *a):
        widths.append(max(int(self.requests[i].emb.shape[0]) for _, i in group))
        return admit_one(self, group, *a)

    monkeypatch.setattr(EngineDevice, "_admit", spy)
    return widths


def test_h_chat_speaker_sample_of_1100_codes(monkeypatch):
    from chattts_b200.speaker import Speaker

    c = _chat()
    g = torch.Generator().manual_seed(5)
    spk_smp = Speaker.encode_prompt(torch.randint(0, 625, (4, 1100), generator=g))
    p = c.InferCodeParams(manual_seed=7, max_new_token=64, min_new_token=64, show_tqdm=False, spk_smp=spk_smp,
                          txt_smp="a sample")
    widths = _spy_prompt_widths(monkeypatch)
    got = dict(c.infer_continuous(["speak with the sampled voice", "and a second text"], params_infer_code=p))
    assert sorted(got) == [0, 1] and all(w.size > 0 and np.isfinite(w).all() for w in got.values())
    assert widths and min(widths) > 1024, widths


def test_h_split_text_paragraph_with_a_long_first_sentence(monkeypatch):
    """Sentence 0 is forced to 1,100 codes, so the speaker sample every later sentence is prompted with is about as
    long, and sentence 1's prompt is over 1,024 tokens (at the parent commit the job failed with ValueError)."""
    c = _chat()
    p = c.InferCodeParams(manual_seed=11, max_new_token=1100, min_new_token=1100, show_tqdm=False)
    widths = _spy_prompt_widths(monkeypatch)
    with c.open_engine(slots=4, max_new_cap=1100) as eng:
        job = eng.submit("The first sentence is long. The second one follows.", params_infer_code=p,
                         split_text=True)
        wav = job.result(timeout=600)
    assert wav.size > 0 and np.isfinite(wav).all()
    assert max(widths) > 1024, widths


# ---------------------------------------------------------------------------------------------------- I
def test_i_limits():
    gpt, embed, _, _ = _model("plain")
    specs = _specs([(MAX_CONTEXT - 1, 1)], base=95)
    got = _engine(gpt, [_request(embed, s) for s in specs], 2, 0)
    _check("I max_context - 1", "plain", 0, specs, got)
    (s,) = _specs([(3000, 1097)], base=96)
    with pytest.raises(ValueError, match="max_context"):
        next(gpt.generate_continuous([_request(embed, s)], slots=2, max_new_cap=1100))
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, [_request(embed, specs[0])], 2, 8, True)
        emb = torch.zeros(1, MAX_CONTEXT, 768, device="cuda")
        mask = torch.ones(1, MAX_CONTEXT, dtype=torch.uint8, device="cuda")
        cfgs = (_lib.SamplerConfig * 1)()
        rc = dev.lib.ctb_gpt_engine_admit(gpt._handle, 1, (C.c_int32 * 1)(0), MAX_CONTEXT, C.c_void_p(emb.data_ptr()),
                                          C.c_void_p(mask.data_ptr()), cfgs, None, (C.c_int32 * 1)(1), dev.stream)
        assert rc == ERR_ARG
