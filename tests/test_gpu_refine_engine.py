"""Text generation on the slot engine (Request.infer_text) and text refinement as engine requests: every text request's
ids equal the live CPU oracle's run of that request alone (B = 1, GPTOracle.generate(infer_text=True)) bit for bit,
whatever else is in flight - code requests included, which keep their own B = 1 parity - and the Chat entry points that
refine on the engine equal ``Chat.infer`` per text."""
import numpy as np
import pytest
import torch

from chattts_b200.engine import EngineDevice, Request, schedule
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from oracle.gpt_oracle import GPTOracle, SamplerParams
from test_gpu_continuous import DEFAULT, MIXED, _check, _oracle, _request, _spec

pytestmark = pytest.mark.gpu

EOS_TEXT = 21001
_text_cache = {}

# prompt lengths 3..40, max_new 6..40; even requests are forced to max_new, odd ones run hot and may end at EOS
T_LENGTHS = [6, 21, 3, 38, 11, 27, 9, 4, 33, 15, 8, 24]
T_MAX_NEW = [12, 30, 7, 40, 18, 25, 6, 34, 21, 16, 28, 10]


def _tspec(i, params):
    forced = i % 2 == 0
    return dict(length=T_LENGTHS[i], prompt_seed=500 + i, seed=2000 + 11 * i, max_new=T_MAX_NEW[i],
                min_new=T_MAX_NEW[i] if forced else 1, temp=0.7 if forced else 1.3, params=params)


def _trequest(embed, s):
    ids, _, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
    tp, tk, rp = s["params"]
    warp, proc = gen_logits(num_code=21178, top_P=tp, top_K=tk, repetition_penalty=rp)
    return Request(emb=embed(ids, tmask)[0], temperature=[s["temp"]], eos_token=EOS_TEXT, max_new_token=s["max_new"],
                   min_new_token=s["min_new"], logits_processors=(*proc, *warp), manual_seed=s["seed"], infer_text=True)


def _toracle(orc, s):
    key = tuple(sorted(s.items()))
    if key not in _text_cache:
        ids, mask, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
        tp, tk, rp = s["params"]
        _text_cache[key] = orc.generate(
            orc.embed_prompt(ids, tmask), ids, torch.tensor([s["temp"]]), EOS_TEXT, attention_mask=mask,
            max_new_token=s["max_new"], min_new_token=s["min_new"],
            sampler=SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp, penalty_max_ids=21178),
            infer_text=True, manual_seed=s["seed"])
    return _text_cache[key]


def _tcheck(out, ref, tag):
    assert out.hiddens == [], tag
    if not ref.ids:  # first-step EOS: the B = 1 reference ends without output
        assert out.ids[0].shape == (0,), tag
        return
    assert out.ids[0].dim() == 1 and out.ids[0].dtype == torch.int64, tag
    assert torch.equal(out.ids[0].cpu(), ref.ids[0]), (tag, out.ids[0].shape, ref.ids[0].shape)


@pytest.mark.parametrize("slots,chunk", [(3, 8), (6, 32), (12, 16)])
def test_text_requests_match_b1_oracle(slots, chunk):
    """12 text requests with mixed top-P / top-K / penalty through 3 / 6 slots (PDL chain) and 12 slots (wgmma)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [_tspec(i, MIXED[i % len(MIXED)]) for i in range(len(T_LENGTHS))]
    reqs = [_trequest(embed, s) for s in specs]
    got = dict(gpt.generate_continuous(reqs, slots=slots, chunk=chunk))
    assert sorted(got) == list(range(len(reqs)))
    for i, s in enumerate(specs):
        _tcheck(got[i], _toracle(orc, s), (slots, i))


@pytest.mark.parametrize("slots", [4, 10])
def test_text_and_code_requests_in_one_engine(slots):
    """Text and code requests decode in the same steps and take each other's slots as they free up."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    kinds, specs = [], []
    for i in range(12):
        text = i % 3 != 1
        kinds.append(text)
        specs.append(_tspec(i, MIXED[i % len(MIXED)]) if text else _spec(i, DEFAULT))
    reqs = [_trequest(embed, s) if t else _request(embed, s) for t, s in zip(kinds, specs)]
    got = dict(gpt.generate_continuous(reqs, slots=slots, chunk=8))
    assert sorted(got) == list(range(len(reqs)))
    for i, (t, s) in enumerate(zip(kinds, specs)):
        if t:
            _tcheck(got[i], _toracle(orc, s), (slots, i))
        else:
            _check(got[i], _oracle(orc, s), (slots, i))


@pytest.mark.parametrize("slots", [8, 12])
def test_idle_slots_stay_untouched_with_text_rows(slots):
    """More slots than requests, text and code mixed: the idle slots' outputs and state never change."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    specs = [(True, _tspec(0, DEFAULT)), (False, _spec(3, DEFAULT)), (True, _tspec(5, MIXED[4])),
             (False, _spec(4, DEFAULT))]
    reqs = [_trequest(embed, s) if t else _request(embed, s) for t, s in specs]
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, max(s["max_new"] for _, s in specs))
        dev.ids_out[4:] = -7
        dev.hid_out[4:] = 0.5
        got = {}
        for i, slot, n in schedule(reqs, dev, 16):
            got[i] = dev.harvest(slot, n) if slot is not None else dev.empty(i)
        st = dev.status()
    assert st.state[4:] == [0] * (slots - 4) and st.end_idx[4:] == [0] * (slots - 4)
    assert bool((dev.ids_out[4:] == -7).all()) and bool((dev.hid_out[4:] == 0.5).all())
    for i, (t, s) in enumerate(specs):
        if t:
            _tcheck(got[i], _toracle(orc, s), i)
        else:
            _check(got[i], _oracle(orc, s), i)


def test_follow_up_of_a_text_request_runs_after_it():
    """A text request's follow-up (a code request) is admitted when the text ends and matches its own B = 1 run."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    t, c = _tspec(2, DEFAULT), _spec(6, DEFAULT)
    seen = []

    def then(out):
        seen.append(out.ids[0].clone())
        return _request(embed, c)

    parent = _trequest(embed, t)
    parent.then = then
    reqs = [parent] + [_request(embed, _spec(i, DEFAULT)) for i in (0, 1)]
    got = dict(gpt.generate_continuous(reqs, slots=2, chunk=4, max_new_cap=max(c["max_new"], 90)))
    assert gpt.last_schedule_stats.children == {0: 3} and sorted(got) == [0, 1, 2, 3]
    _tcheck(got[0], _toracle(orc, t), "text")
    assert torch.equal(seen[0].cpu(), got[0].ids[0].cpu())
    _check(got[3], _oracle(orc, c), "follow-up")
    with pytest.raises(ValueError):  # a follow-up over the declared cap is refused like an up-front request
        p2 = _trequest(embed, t)
        p2.then = lambda out: _request(embed, _spec(2, DEFAULT))  # max_new 90
        list(gpt.generate_continuous([p2, _request(embed, _spec(0, DEFAULT))], slots=2, max_new_cap=40))


# ---------------------------------------------------------------------------------------------------- Chat
_c = {}


def chat():
    if not _c:
        from chattts_b200 import Chat
        from chattts_b200.synth import synth_all
        from stubs import StubSpeaker, StubTokenizer

        c = Chat()
        assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                             max_batch=4, max_context=256)
        _c["chat"] = c
    return _c["chat"]


TEXTS = ["hello there", "hi", "a somewhat longer sentence to speak", "ok", "fifth text"]


def _refine_params(c):
    n = [12, 20, 9, 16, 14]
    return [c.RefineTextParams(manual_seed=40 + i, max_new_token=n[i], min_new_token=n[i] if i % 2 == 0 else 0,
                               temperature=[0.7, 0.9, 0.5, 0.7, 1.1][i], top_P=[0.7, None, 0.9, 0.7, 0.5][i],
                               top_K=[20, 20, None, 5, 20][i], repetition_penalty=[1.0, 1.05, 1.0, 1.2, 1.0][i],
                               show_tqdm=False) for i in range(len(TEXTS))]


def _code_params(c):
    n = [48, 72, 61, 100, 37]
    return [c.InferCodeParams(manual_seed=3 + i, max_new_token=n[i], min_new_token=n[i], temperature=0.3 + 0.1 * i,
                              stream_batch=[16, 24, 16, 24, 16][i], stream_speed=[6000, 6000, 12000, 12000, 6000][i],
                              pass_first_n_batches=[0, 2, 0, 2, 2][i], show_tqdm=False)
            for i in range(len(TEXTS))]


def test_refine_continuous_equals_refine_text_only_per_text():
    c = chat()
    refine = _refine_params(c)
    got = dict(c.refine_continuous(TEXTS, params_refine_text=refine, slots=3))
    assert sorted(got) == list(range(len(TEXTS)))
    for i, t in enumerate(TEXTS):
        ref = c.infer([t], refine_text_only=True, split_text=False, params_refine_text=refine[i])[0]
        assert isinstance(got[i], str) and got[i] == ref, (i, got[i], ref)


@pytest.mark.parametrize("use_decoder", [False, True])
def test_infer_continuous_refine_on_engine_equals_infer_per_text(use_decoder):
    c = chat()
    refine, params = _refine_params(c), _code_params(c)
    got = dict(c.infer_continuous(TEXTS, params_infer_code=params, params_refine_text=refine, slots=3,
                                  use_decoder=use_decoder, skip_refine_text=False, refine_on_engine=True))
    assert sorted(got) == list(range(len(TEXTS)))
    for i, t in enumerate(TEXTS):
        ref = c.infer([t], split_text=False, skip_refine_text=False, use_decoder=use_decoder,
                      params_refine_text=refine[i], params_infer_code=params[i])[0]
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        if use_decoder:
            assert float(np.sqrt(np.mean((got[i] - ref) ** 2))) < 1e-4, i
        else:
            assert np.array_equal(got[i], ref), i


@pytest.mark.parametrize("use_decoder", [False, True])
def test_infer_continuous_batched_refinement_equals_infer_of_the_refined_texts(use_decoder):
    """The default mode: the texts are refined in static batches, as ``infer(refine_text_only=True)`` refines them,
    and each refined text is then spoken as ``infer`` speaks it."""
    c = chat()
    refine, params = _refine_params(c)[0], _code_params(c)
    refined = c.infer(TEXTS, refine_text_only=True, split_text=False, params_refine_text=refine)
    got = dict(c.infer_continuous(TEXTS, params_infer_code=params, params_refine_text=refine, slots=3,
                                  use_decoder=use_decoder, skip_refine_text=False))
    assert sorted(got) == list(range(len(TEXTS)))
    for i, t in enumerate(refined):
        ref = c.infer([t], split_text=False, skip_refine_text=True, use_decoder=use_decoder,
                      params_infer_code=params[i])[0]
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        if use_decoder:
            assert float(np.sqrt(np.mean((got[i] - ref) ** 2))) < 1e-4, i
        else:
            assert np.array_equal(got[i], ref), i


@pytest.mark.parametrize("use_decoder", [True, False])
def test_infer_continuous_stream_refine_on_engine_equals_static_stream(use_decoder):
    c = chat()
    refine, params = _refine_params(c), _code_params(c)
    got = {i: [] for i in range(len(TEXTS))}
    for i, chunk, last in c.infer_continuous_stream(TEXTS, params_infer_code=params, params_refine_text=refine,
                                                    slots=3, use_decoder=use_decoder, skip_refine_text=False,
                                                    refine_on_engine=True):
        got[i].append((chunk, last))
    for i, t in enumerate(TEXTS):
        ref = list(c.infer([t], stream=True, split_text=False, skip_refine_text=False, use_decoder=use_decoder,
                           params_refine_text=refine[i], params_infer_code=params[i]))
        assert len(got[i]) == len(ref), (i, len(got[i]), len(ref))
        assert [last for _, last in got[i]] == [False] * (len(ref) - 1) + [True]
        for (x, _), y in zip(got[i], ref):
            if not use_decoder:
                assert np.array_equal(x, y), i
        for (x, _), y in zip(got[i][:-1], ref[:-1]):
            assert x.shape == y.shape, (i, x.shape, y.shape)
            if x.size:
                assert float(np.sqrt(np.mean((x - y) ** 2))) < 1e-4, i
        assert abs(got[i][-1][0].shape[1] - ref[-1].shape[1]) <= 2
