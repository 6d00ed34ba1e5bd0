"""Continuous batching on the GPU (chattts_b200.engine): whatever else is in flight and whichever slot a request lands
in, its token ids equal the live CPU oracle's run of that request alone (B = 1) bit for bit, hidden states within
1e-4."""
import numpy as np
import pytest
import torch

from chattts_b200.engine import EngineDevice, Request, schedule
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from oracle.gpt_oracle import GPTOracle, SamplerParams

pytestmark = pytest.mark.gpu

_oracle_cache = {}

# prompt lengths 3..40 (four below the prefill's 8 columns), max_new 20..90; even requests are forced to max_new,
# odd ones run hot and may end at EOS
LENGTHS = [3, 17, 40, 5, 9, 26, 7, 33, 12, 4, 21, 38]
MAX_NEW = [20, 45, 90, 33, 60, 25, 81, 40, 55, 70, 28, 64]
DEFAULT = (0.7, 20, 1.05)
MIXED = [(0.7, 20, 1.05), (None, 20, 1.0), (0.5, None, 1.05), (None, None, 1.0), (0.95, 3, 1.2), (0.7, 20, 1.0)]


def _spec(i, params):
    forced = i % 2 == 0
    temp = [0.3, 0.5, 0.7, 1.0] if forced else [1.5] * 4
    return dict(length=LENGTHS[i], prompt_seed=300 + i, seed=1000 + 7 * i, max_new=MAX_NEW[i],
                min_new=MAX_NEW[i] if forced else 2, temp=temp, params=params)


def _request(embed, s):
    ids, _, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
    tp, tk, rp = s["params"]
    warp, proc = gen_logits(num_code=625, top_P=tp, top_K=tk, repetition_penalty=rp)
    return Request(emb=embed(ids, tmask)[0], temperature=s["temp"], eos_token=625, max_new_token=s["max_new"],
                   min_new_token=s["min_new"], logits_processors=(*proc, *warp), manual_seed=s["seed"])


def _oracle(orc, s):
    key = tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in s.items()))
    if key not in _oracle_cache:
        ids, mask, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
        tp, tk, rp = s["params"]
        _oracle_cache[key] = orc.generate(
            orc.embed_prompt(ids, tmask), ids, torch.tensor(s["temp"]), 625, attention_mask=mask,
            max_new_token=s["max_new"], min_new_token=s["min_new"],
            sampler=SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp), return_hidden=True,
            manual_seed=s["seed"])
    return _oracle_cache[key]


def _check(out, ref, tag):
    if not ref.ids:  # first-step EOS: the B = 1 reference ends without output (gpt.py:527)
        assert out.ids[0].shape[0] == 0, tag
        return
    assert torch.equal(out.ids[0].cpu(), ref.ids[0]), (tag, out.ids[0].shape, ref.ids[0].shape)
    assert (out.hiddens[0].cpu() - ref.hiddens[0]).abs().max() < 1e-4, tag


@pytest.mark.parametrize("slots,chunk", [(3, 8), (6, 32), (12, 16)])
def test_continuous_matches_b1_oracle(slots, chunk):
    """12 requests through 3 / 6 slots (FMA chain; admissions mid-decode, several at once, slot reuse) and 12 slots
    (wgmma step)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [_spec(i, DEFAULT) for i in range(len(LENGTHS))]
    reqs = [_request(embed, s) for s in specs]
    got = dict(gpt.generate_continuous(reqs, slots=slots, chunk=chunk))
    assert sorted(got) == list(range(len(reqs)))
    stats = gpt.last_schedule_stats
    if slots < len(reqs):
        assert stats.admissions > 1
    for i, s in enumerate(specs):
        _check(got[i], _oracle(orc, s), (slots, i))


def test_continuous_mixed_sampling_parameters():
    """Repetition penalty on / off and top-P / top-K on / off side by side in one engine."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [_spec(i, MIXED[i % len(MIXED)]) for i in range(len(MIXED) + 2)]
    reqs = [_request(embed, s) for s in specs]
    got = dict(gpt.generate_continuous(reqs, slots=4, chunk=16))
    for i, s in enumerate(specs):
        _check(got[i], _oracle(orc, s), i)


def test_idle_slots_stay_untouched():
    """An engine with more slots than requests: the idle slots' outputs and state never change."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [_spec(i, DEFAULT) for i in (0, 3, 4)]
    reqs = [_request(embed, s) for s in specs]
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, 8, max(s["max_new"] for s in specs))
        dev.ids_out[3:] = -7
        dev.hid_out[3:] = 0.5
        got = {}
        for i, slot, n in schedule(reqs, dev, 16):
            got[i] = dev.harvest(slot, n) if slot is not None else dev.empty()
        st = dev.status()
    assert st.state[3:] == [0] * 5 and st.end_idx[3:] == [0] * 5
    assert bool((dev.ids_out[3:] == -7).all()) and bool((dev.hid_out[3:] == 0.5).all())
    for i, s in enumerate(specs):
        _check(got[i], _oracle(orc, s), i)


def test_chat_infer_continuous_equals_infer_per_text():
    from chattts_b200 import Chat
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=4, max_context=256)
    texts = ["hello there", "hi", "a somewhat longer sentence to speak", "ok", "fifth text"]
    params = [c.InferCodeParams(manual_seed=3 + i, max_new_token=24 + 9 * i, min_new_token=24 + 9 * i,
                                temperature=0.3 + 0.1 * i, top_P=[0.7, None, 0.9, 0.7, 0.5][i],
                                top_K=[20, 20, None, 5, 20][i], repetition_penalty=[1.05, 1.0, 1.05, 1.2, 1.0][i],
                                show_tqdm=False) for i in range(len(texts))]
    got = dict(c.infer_continuous(texts, params_infer_code=params, slots=3))
    assert sorted(got) == list(range(len(texts)))
    for i, t in enumerate(texts):
        ref = c.infer([t], split_text=False, skip_refine_text=True, params_infer_code=params[i])[0]
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        assert float(np.sqrt(np.mean((got[i] - ref) ** 2))) < 1e-4, i
