"""Slot engines of 33..64 slots on the 64-row wgmma decode step (k_tc_dec<..., NPAD = 64, ...>), fp32 and half precision.

W1: fp32 engines of 40 and 64 slots follow the CPU oracle run of each request alone (B = 1) bit for bit, text requests
included.  W2: the fp16 engine (and the fp16 KV cache alone) follows the fp16 oracle, teacher-forced.  W3: a request's
results do not depend on its slot (0 or 63) or its neighbours, and the 64-wide step agrees with the 32-wide one.  W4: on
fp16-representable weights with unit norms, fp16 weights alone equal fp32 bit for bit at S = 64.  W5: the limits on a
handle of 72 rows.  W6: ``Chat.infer_continuous`` with 64 slots.  W7: one admission of 64 prompts of 1,024 tokens."""
import gc

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.engine import ADMIT_MAX_ROWS, EngineDevice, ScheduleStats, schedule
from chattts_b200.gpt import GPT
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from fp16_oracle import GPTOracleFp16, fp16_layer_state
from gpu_util import release_on_teardown
from oracle.gpt_oracle import GPTOracle, SamplerParams, apply_temperature, repetition_penalty, top_p_filter
from test_gpu_fp16_engine import EOS_TEXT, HIDDEN_ATOL, KV16, MARGIN, MIXED, W16, _engine, _request, _teacher_forced

pytestmark = pytest.mark.gpu

FP16 = W16 | KV16
CONTEXT = 640  # 64 slots x 640 tokens: 5.0 GB of fp32 KV
_handles = {}
_refs = {}
_release = release_on_teardown(_handles, _refs)


def _model(kind, max_batch=64, max_context=CONTEXT):
    """'plain': the synthetic model; 'rep': its fp16-representable, unit-norm form (W4)."""
    key = (kind, max_batch, max_context)
    if key not in _handles:
        cfg = Config()
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        if kind == "rep":
            gs = fp16_layer_state(gs)
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
        gpt.load_state(gs)
        _handles[key] = (gpt, embed, gs, es)
    return _handles[key]


def _drop(*keys):
    """Destroy the handles ``keys`` (every handle of this module when none is named) and return their device memory,
    so that the tests after them do not depend on what ran before."""
    for k in keys or list(_handles):
        _handles.pop(k, None)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _spec(i, max_new=(16, 48), seed_base=3000):
    """Seeded code request i: prompt 3..40 tokens, max_new in the given range; even ones forced to max_new."""
    lo, hi = max_new
    forced = i % 2 == 0
    mn = lo + (i * 7) % (hi - lo + 1)
    return dict(length=3 + (i * 13) % 38, prompt_seed=900 + i, seed=seed_base + 7 * i, max_new=mn,
                min_new=mn if forced else 2, temp=[0.3, 0.5, 0.7, 1.0] if forced else [1.5] * 4,
                params=MIXED[i % len(MIXED)], text=False)


def _text_spec(i):
    return dict(length=12 + i, prompt_seed=700 + i, seed=50 + i, max_new=24, min_new=4, temp=[0.7], text=True,
                params=(0.7, 20, 1.0))


def _oracle(orc, s):
    """GPTOracle.generate of request s alone (B = 1), cached per spec."""
    key = (id(orc), repr(sorted(s.items())))
    if key not in _refs:
        ids, mask, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
        tp, tk, rp = s["params"]
        _refs[key] = orc.generate(
            orc.embed_prompt(ids, tmask), ids, torch.tensor(s["temp"]), EOS_TEXT if s["text"] else 625,
            attention_mask=mask, max_new_token=s["max_new"], min_new_token=s["min_new"],
            sampler=SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp,
                                  **({"penalty_max_ids": 21178} if s["text"] else {})),
            infer_text=s["text"], return_hidden=not s["text"], manual_seed=s["seed"])
    return _refs[key]


def _orc(gs, es):
    if "orc" not in _refs:
        _refs["orc"] = GPTOracle(gs, es)
    return _refs["orc"]


def _check_oracle(got, ref, s, tag):
    ids, hid, _ = got
    if not ref.ids:  # first-step EOS: the B = 1 reference ends without output
        assert ids.shape[0] == 0, tag
        return
    assert torch.equal(ids, ref.ids[0]), (tag, ids.shape, ref.ids[0].shape)
    if not s["text"]:
        assert (hid - ref.hiddens[0]).abs().max() < 1e-4, tag


# ---------------------------------------------------------------------------------------------------- W1
@pytest.mark.parametrize("slots", [40, 64])
def test_w1_fp32_wide_engine_matches_b1_oracle(slots):
    """80 code requests with mixed sampling parameters and 4 text requests: admissions mid-decode and slot reuse."""
    gpt, embed, gs, es = _model("plain")
    orc = _orc(gs, es)
    specs = [_spec(i) for i in range(80)]
    specs[10:10] = [_text_spec(0), _text_spec(1)]
    specs[70:70] = [_text_spec(2), _text_spec(3)]
    reqs = [_request(embed, s) for s in specs]
    got = _engine(gpt, reqs, slots, 0, chunk=16, cap=48)
    assert sorted(got) == list(range(len(reqs)))
    used = {g[2] for g in got.values() if g[2] is not None}
    assert max(used) == slots - 1
    if slots == 64:
        assert len([u for u in used if u >= 48]) == 16
    for i, s in enumerate(specs):
        _check_oracle(got[i], _oracle(orc, s), s, (slots, i))


# ---------------------------------------------------------------------------------------------------- W2
def _top_k_margin(logits, ids, t, s):
    """Relative gap between the k-th and (k+1)-th largest scores at top-K's cut, minimised over the rows of step t:
    how close the set top-K keeps is to changing (the oracle's decision margins cover the arg-max and top-P's cut)."""
    tp, tk, rp = s["params"]
    if tk is None:
        return float("inf")
    sp = SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp, penalty_max_ids=21178 if s["text"] else 625)
    gen = ids[:t].long()
    gen_rows = gen[None] if s["text"] else gen.t()
    x = apply_temperature(logits, torch.tensor(s["temp"]))
    if rp != 1:
        x = repetition_penalty(gen_rows, x, rp, sp.penalty_max_ids, sp.penalty_window)
    if tp is not None:
        x = top_p_filter(x, tp, sp.min_keep)
    k = min(max(tk, sp.min_keep), x.shape[-1] - 1)
    v = torch.topk(x, k + 1).values
    return float(((v[:, k - 1] - v[:, k]) / v[:, k - 1].abs().clamp_min(1e-30)).min())


@pytest.mark.parametrize("slots,flags", [(40, FP16), (64, FP16), (64, KV16)])
def test_w2_fp16_wide_engine_follows_the_fp16_oracle(slots, flags):
    gpt, embed, gs, es = _model("plain")
    orc = GPTOracleFp16(gs, es, fp16_layers=bool(flags & W16), fp16_kv=bool(flags & KV16))
    specs = [_spec(i, max_new=(16, 24), seed_base=5000) for i in range(66)] + [_text_spec(4), _text_spec(5)]
    reqs = [_request(embed, s) for s in specs]
    got = _engine(gpt, reqs, slots, flags, cap=24)
    assert max(g[2] for g in got.values() if g[2] is not None) == slots - 1
    worst, accepted, total = 0.0, 0, 0
    for i, s in enumerate(specs):
        ids, hid, _ = got[i]
        out = _teacher_forced(orc, s, ids)
        tr = out.trace
        eos = EOS_TEXT if s["text"] else 625
        for t, sampled in enumerate(tr["sampled"]):
            total += 1
            eng = ids[t].long() if t < ids.shape[0] else None
            if eng is None:  # the engine ended here: it sampled EOS
                ok = bool((sampled == eos).any())
            else:
                ok = torch.equal(sampled[0].view(-1), eng.view(-1)[: sampled.shape[1]])
            if not ok:
                margin = min(tr["argmax_margin"][t], tr["top_p_margin"][t], _top_k_margin(tr["logits"][t], ids, t, s))
                assert margin < MARGIN, (slots, i, t, margin)
                accepted += 1
        n = min(hid.shape[0], len(tr["sampled"]))
        ref = out.hiddens[0][:n] if out.hiddens else torch.zeros(0, 768)
        n = min(n, ref.shape[0])
        if n:
            err = float((hid[:n] - ref[:n]).abs().max())
            worst = max(worst, err)
            assert err < HIDDEN_ATOL, (slots, i, err)
    print(f"\nW2 S={slots} flags={flags}: max |hidden - oracle| = {worst:.3e}, "
          f"margin-accepted steps {accepted} of {total}")


# ---------------------------------------------------------------------------------------------------- W3
@pytest.mark.parametrize("flags", [0, FP16])
def test_w3_slot_0_and_slot_63_give_the_same_results(flags):
    """The same request first (slot 0) among 63 neighbours, then last (slot 63) among 63 others."""
    gpt, embed, _, _ = _model("plain")
    target = dict(_spec(0, max_new=(40, 40)), prompt_seed=4242, seed=4243)
    na = [_spec(i, seed_base=6000) for i in range(1, 64)]
    nb = [dict(_spec(i, seed_base=7000), prompt_seed=1900 + i) for i in range(1, 64)]
    a = _engine(gpt, [_request(embed, s) for s in [target] + na], 64, flags, cap=48)
    b = _engine(gpt, [_request(embed, s) for s in nb + [target]], 64, flags, cap=48)
    assert a[0][2] == 0 and b[63][2] == 63
    assert a[0][0].shape[0] == 40
    assert torch.equal(a[0][0], b[63][0])
    assert torch.equal(a[0][1], b[63][1])


@pytest.mark.parametrize("flags", [0, FP16])
def test_w3_64_wide_step_agrees_with_32_wide_step(flags):
    gpt, embed, _, _ = _model("plain")
    specs = [_spec(i, seed_base=8000) for i in range(24)]
    reqs = [_request(embed, s) for s in specs]
    w32 = _engine(gpt, reqs, 32, flags, cap=48)
    w64 = _engine(gpt, reqs, 64, flags, cap=48)
    same = 0
    for i in range(len(specs)):
        assert torch.equal(w32[i][0], w64[i][0]), (flags, i)
        assert (w32[i][1] - w64[i][1]).abs().max() < 1e-4, (flags, i)
        same += torch.equal(w32[i][1], w64[i][1])
    print(f"\nW3 flags={flags}: NPAD 32 and NPAD 64 engines agree bit for bit on {same} of {len(specs)} requests")


# ---------------------------------------------------------------------------------------------------- W4
def test_w4_fp16_weights_equal_fp32_on_representable_weights_at_64_slots():
    gpt, embed, _, _ = _model("rep")
    specs = [_spec(i, seed_base=9000) for i in range(66)] + [_text_spec(6), _text_spec(7)]
    reqs = [_request(embed, s) for s in specs]
    a = _engine(gpt, reqs, 64, 0, cap=48)
    b = _engine(gpt, reqs, 64, W16, cap=48)
    assert sorted(a) == sorted(b) == list(range(len(reqs)))
    for i in range(len(specs)):
        assert torch.equal(a[i][0], b[i][0]), i
        assert torch.equal(a[i][1], b[i][1]), (i, (a[i][1] - b[i][1]).abs().max())
    _drop(("rep", 64, CONTEXT))


# ---------------------------------------------------------------------------------------------------- W5
def test_w5_limits_on_a_72_row_handle():
    gpt, embed, gs, es = _model("plain", max_batch=72)
    specs = [_spec(i, seed_base=9500) for i in range(4)]
    reqs = [_request(embed, s) for s in specs]
    with pytest.raises(_lib.CtbError, match="64"):
        _engine(gpt, reqs, 65, FP16, cap=48)
    got = _engine(gpt, reqs, 64, FP16, cap=48)
    ref, ref_embed, _, _ = _model("plain")
    want = _engine(ref, [_request(ref_embed, s) for s in specs], 64, FP16, cap=48)
    for i in range(len(specs)):
        assert torch.equal(got[i][0], want[i][0]) and torch.equal(got[i][1], want[i][1]), i
    # fp32 at 65 slots: the PDL chain
    orc = _orc(gs, es)
    chain = _engine(gpt, reqs[:2], 65, 0, cap=48)
    for i in range(2):
        _check_oracle(chain[i], _oracle(orc, specs[i]), specs[i], ("S=65", i))
    _drop(("plain", 72, CONTEXT))


# ---------------------------------------------------------------------------------------------------- W6
def test_w6_chat_infer_continuous_with_64_slots_equals_infer_per_text():
    from chattts_b200 import Chat
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=64, max_context=256)
    texts = [f"text number {i} " + "abc" * (i % 5) for i in range(66)]
    params = [c.InferCodeParams(manual_seed=3 + i, max_new_token=16 + (i * 5) % 24, min_new_token=16 + (i * 5) % 24,
                                temperature=0.3 + 0.01 * i, show_tqdm=False) for i in range(len(texts))]
    got = dict(c.infer_continuous(texts, params_infer_code=params, slots=64))
    assert sorted(got) == list(range(len(texts)))
    for i in (5, 57, 65):  # slot 5, slot 57 and a text admitted mid-decode
        ref = c.infer([texts[i]], split_text=False, skip_refine_text=True, params_infer_code=params[i])[0]
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        assert float(np.sqrt(np.mean((got[i] - ref) ** 2))) < 1e-4, i
    c.unload()


# ---------------------------------------------------------------------------------------------------- W7
def test_w7_admission_of_64_prompts_of_1024_tokens():
    """64 prompts of 1,024 tokens admitted at one poll: the host runs them as two prefills of 32 x 1,024 rows
    (ADMIT_MAX_ROWS), so the prefill's scratch stays at 1.9 GB, and every request still equals the B = 1 oracle."""
    _drop()
    free = torch.cuda.mem_get_info()[0]
    gpt, embed, gs, es = _model("plain", max_context=1040)
    orc = GPTOracle(gs, es)
    specs = [dict(length=1024, prompt_seed=11000 + i, seed=12000 + i, max_new=8, min_new=8,
                  temp=[0.5] * 4, params=MIXED[i % len(MIXED)], text=False) for i in range(64)]
    reqs = [_request(embed, s) for s in specs]
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 64, 8, True)
        prefills = []
        admit_one = dev._admit
        dev._admit = lambda group, *a: (prefills.append([i for _, i in group]), admit_one(group, *a))
        stats, got = ScheduleStats(), {}
        for i, slot, n in schedule(reqs, dev, 8, stats=stats):
            o = dev.harvest(slot, n)
            got[i] = (o.ids[0].cpu(), o.hiddens[0].cpu(), slot)
    used = free - torch.cuda.mem_get_info()[0]
    print(f"\nW7: {free / 1e9:.1f} GB free before the handle, {used / 1e9:.1f} GB used by it after the run")
    assert sorted(got) == list(range(64)) and stats.admissions == 1
    assert prefills == [list(range(32)), list(range(32, 64))] and 32 * 1024 <= ADMIT_MAX_ROWS
    for i in (0, 31, 32, 63):  # both ends of both prefills
        _check_oracle(got[i], _oracle(orc, specs[i]), specs[i], ("T0=1024", i))
    _drop()
