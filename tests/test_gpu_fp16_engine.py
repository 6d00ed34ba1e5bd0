"""The half-precision slot engine on the GPU (ctb_gpt_engine_begin_ex).

G1: with fp16-representable layer matrices and unit layer norms, CTB_ENGINE_FP16_WEIGHTS alone gives the fp32 engine's
ids and hidden states bit for bit.  G2: the full fp16 engine follows the fp16 oracle (tests/fp16_oracle.py),
teacher-forced along its own ids.  G3: a request's results do not depend on its neighbours or its slot.  G4: an
out-of-range weight refuses the engine and leaves the handle as it was.  G5: the dtype option through ``Chat``."""
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
from fp16_oracle import GPTOracleFp16, fp16_layer_state
from gpu_util import release_on_teardown
from oracle.gpt_oracle import SamplerParams

pytestmark = pytest.mark.gpu

W16, KV16 = _lib.ENGINE_FP16_WEIGHTS, _lib.ENGINE_FP16_KV
FP16 = W16 | KV16
EOS_TEXT = 21001
# G2 bars.  Observed on one H100 (DESIGN.md §4): hidden states within 5.6e-4 of the fp16 oracle at S = 3 / 12 / 24,
# and every id the oracle's sampled id (0 of 529 steps needed the margin rule); 2e-3 leaves 3.5x headroom.
MARGIN = 1e-3
HIDDEN_ATOL = 2e-3

LENGTHS = [3, 17, 40, 5, 9, 26, 7, 33, 12, 4, 21, 38]
MAX_NEW = [20, 45, 90, 33, 60, 25, 81, 40, 55, 70, 28, 64]
MIXED = [(0.7, 20, 1.05), (None, 20, 1.0), (0.5, None, 1.05), (None, None, 1.0), (0.95, 3, 1.2), (0.7, 20, 1.0)]
_handles = {}
_release = release_on_teardown(_handles)


def _build(state, max_batch=32, max_context=640):
    cfg = Config()
    gs, es = state
    embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                  cfg.embed.num_vq).load_state_dict(es).to("cuda")
    gpt = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch, max_context=max_context)
    gpt.load_state(gs)
    return gpt, embed


def _model(kind):
    """'plain': the synthetic model; 'rep': its fp16-representable, unit-norm form (G1)."""
    if kind not in _handles:
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        if kind == "rep":
            gs = fp16_layer_state(gs)
        _handles[kind] = (*_build((gs, es)), gs, es)
    return _handles[kind]


def _spec(i, params, seeded=True):
    forced = i % 2 == 0
    return dict(length=LENGTHS[i % 12], prompt_seed=300 + i, seed=(1000 + 7 * i) if seeded else None,
                max_new=MAX_NEW[i % 12], min_new=MAX_NEW[i % 12] if forced else 2,
                temp=[0.3, 0.5, 0.7, 1.0] if forced else [1.5] * 4, params=params, text=False)


def _text_spec(i):
    return dict(length=12 + i, prompt_seed=700 + i, seed=50 + i, max_new=24, min_new=4, temp=[0.7], text=True,
                params=(0.7, 20, 1.0))


def _request(embed, s):
    ids, _, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
    tp, tk, rp = s["params"]
    V = 21178 if s["text"] else 625
    warp, proc = gen_logits(num_code=V, top_P=tp, top_K=tk, repetition_penalty=rp)
    return Request(emb=embed(ids, tmask)[0], temperature=s["temp"], eos_token=EOS_TEXT if s["text"] else 625,
                   max_new_token=s["max_new"], min_new_token=s["min_new"], logits_processors=(*proc, *warp),
                   manual_seed=s["seed"], infer_text=s["text"])


def _mix():
    specs = [_spec(i, MIXED[i % len(MIXED)], seeded=i % 5 != 4) for i in range(12)]
    return specs + [_text_spec(0), _text_spec(1)]


def _engine(gpt, reqs, slots, flags, chunk=16, cap=90):
    """Every request through one engine of ``slots`` slots -> {index: (ids, hiddens, slot)} (copies)."""
    got = {}
    with torch.cuda.device(gpt.device_gpt):
        dev = EngineDevice(gpt, reqs, slots, cap, True, flags)
        for i, slot, n in schedule(reqs, dev, chunk):
            if slot is None:
                got[i] = (torch.zeros(0, 4, dtype=torch.int32), torch.zeros(0, 768), None)
            else:
                o = dev.harvest(slot, n)
                hid = o.hiddens[0].cpu().clone() if o.hiddens else torch.zeros(0, 768)  # text requests have none
                got[i] = (o.ids[0].cpu().clone(), hid, slot)
                o.destroy()
    return got


# ---------------------------------------------------------------------------------------------------- G1
@pytest.mark.parametrize("slots", [12, 24])
def test_g1_fp16_weights_equal_fp32_on_representable_weights(slots):
    gpt, embed, _, _ = _model("rep")
    specs = _mix()
    reqs = [_request(embed, s) for s in specs]
    a = _engine(gpt, reqs, slots, 0)
    b = _engine(gpt, reqs, slots, W16)
    assert sorted(a) == sorted(b) == list(range(len(reqs)))
    for i, s in enumerate(specs):
        if s["seed"] is None:  # device Philox draws a fresh seed per engine: nothing to compare bit for bit
            continue
        assert torch.equal(a[i][0], b[i][0]), (slots, i)
        assert torch.equal(a[i][1], b[i][1]), (slots, i, (a[i][1] - b[i][1]).abs().max())


# ---------------------------------------------------------------------------------------------------- G2
def _teacher_forced(orc, s, ids):
    """The fp16 oracle teacher-forced along the engine's ids, one step past them when the engine ended at EOS."""
    pids, mask, tmask = synth_prompt_batch([s["length"]], seed=s["prompt_seed"])
    tp, tk, rp = s["params"]
    n = int(ids.shape[0])
    steps = min(n + 1, s["max_new"])
    forced = torch.zeros(1, steps, 4, dtype=torch.long)
    forced[0, :n] = ids.long()[:, None].expand(-1, 4) if s["text"] else ids.long()
    out = orc.generate(orc.embed_prompt(pids, tmask), pids, torch.tensor(s["temp"]), EOS_TEXT if s["text"] else 625,
                       attention_mask=mask, max_new_token=steps, min_new_token=s["min_new"],
                       sampler=SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp,
                                             penalty_max_ids=21178 if s["text"] else 625),
                       infer_text=s["text"], return_hidden=True, manual_seed=s["seed"], trace=True,
                       forced_ids=forced)
    return out


@pytest.mark.parametrize("slots,flags", [(3, FP16), (12, FP16), (24, FP16), (12, KV16)])
def test_g2_fp16_engine_follows_the_fp16_oracle(slots, flags):
    """The full fp16 engine, and (S = 12) the fp16 KV cache alone on fp32 weights."""
    gpt, embed, gs, es = _model("plain")
    orc = GPTOracleFp16(gs, es, fp16_layers=bool(flags & W16), fp16_kv=bool(flags & KV16))
    specs = [s for s in _mix() if s["seed"] is not None]  # the oracle covers the seeded path
    reqs = [_request(embed, s) for s in specs]
    got = _engine(gpt, reqs, slots, flags)
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
                assert min(tr["argmax_margin"][t], tr["top_p_margin"][t]) < MARGIN, (slots, i, t)
                accepted += 1
        # hidden states of every step the oracle ran on the engine's ids (it may stop earlier on a flipped EOS)
        n = min(hid.shape[0], len(tr["sampled"]))
        ref = out.hiddens[0][:n] if out.hiddens else torch.zeros(0, 768)
        n = min(n, ref.shape[0])
        if n:
            err = float((hid[:n] - ref[:n]).abs().max())
            worst = max(worst, err)
            assert err < HIDDEN_ATOL, (slots, i, err)
    print(f"\nG2 S={slots} flags={flags}: max |hidden - oracle| = {worst:.3e}, margin-accepted steps {accepted} of {total}")


# ---------------------------------------------------------------------------------------------------- G3
def test_g3_results_do_not_depend_on_neighbours_or_slot():
    gpt, embed, _, _ = _model("plain")
    specs = _mix()
    reqs = [_request(embed, s) for s in specs]
    seeded = [i for i, s in enumerate(specs) if s["seed"] is not None]
    for lo_slots, hi_slots in ((3, 12), (17, 24)):  # one engine width each: NPAD 16, then NPAD 32
        a = _engine(gpt, reqs, lo_slots, FP16, chunk=8)
        b = _engine(gpt, list(reversed(reqs)), hi_slots, FP16, chunk=16)
        n = len(reqs)
        for i in seeded:
            x, y = a[i], b[n - 1 - i]
            assert torch.equal(x[0], y[0]), (lo_slots, hi_slots, i)
            assert torch.equal(x[1], y[1]), (lo_slots, hi_slots, i)
    w16 = _engine(gpt, reqs, 12, FP16)
    w32 = _engine(gpt, reqs, 24, FP16)
    same = sum(torch.equal(w16[i][0], w32[i][0]) and torch.equal(w16[i][1], w32[i][1]) for i in seeded)
    print(f"\nG3: NPAD 16 and NPAD 32 engines agree bit for bit on {same} of {len(seeded)} seeded requests")


# ---------------------------------------------------------------------------------------------------- G4
def _static(gpt, embed, B, seed=5):
    ids, mask, tmask = synth_prompt_batch([9 + 3 * b for b in range(B)], seed=seed)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    out = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([0.5] * 4), eos_token=625,
                            attention_mask=mask, max_new_token=24, min_new_token=24,
                            logits_processors=(*proc, *warp), return_hidden=True, show_tqdm=False,
                            manual_seed=77))[-1]
    return [(i.cpu().clone(), h.cpu().clone()) for i, h in zip(out.ids, out.hiddens)]


def test_g4_out_of_range_weight_refuses_and_leaves_the_handle_intact():
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    gs = dict(gs)
    gs["layers.3.input_layernorm.weight"] = gs["layers.3.input_layernorm.weight"].clone()
    gs["layers.3.input_layernorm.weight"][17] = 1e7  # folded into Wqkv: |w * ln| > 65504
    gpt, embed = _build((gs, es))
    reqs = [_request(embed, s) for s in [_spec(i, MIXED[0]) for i in range(4)]]
    with pytest.raises(_lib.CtbError, match=r"layer 3 self_attn\.qkv"):
        _engine(gpt, reqs, 12, FP16)
    with pytest.raises(_lib.CtbError, match="layer 3"):
        _engine(gpt, reqs, 4, FP16)  # and again (nothing was kept)
    got = _engine(gpt, reqs, 12, 0)
    s1, s12 = _static(gpt, embed, 1), _static(gpt, embed, 12)
    fresh, fembed = _build((gs, es))
    ref = _engine(fresh, [_request(fembed, s) for s in [_spec(i, MIXED[0]) for i in range(4)]], 12, 0)
    r1, r12 = _static(fresh, fembed, 1), _static(fresh, fembed, 12)
    for i in range(4):
        torch.testing.assert_close(got[i][0], ref[i][0], rtol=0, atol=0, equal_nan=True)
        torch.testing.assert_close(got[i][1], ref[i][1], rtol=0, atol=0, equal_nan=True)
    for x, y in zip(s1 + s12, r1 + r12):
        torch.testing.assert_close(x[0], y[0], rtol=0, atol=0)
        torch.testing.assert_close(x[1], y[1], rtol=0, atol=0, equal_nan=True)


def test_g4_kv_pool_is_shared_across_precisions():
    """fp16 engine -> fp32 engine -> static generate -> fp16 engine on one handle (the pool is sized in bytes)."""
    gpt, embed, _, _ = _model("plain")
    reqs = [_request(embed, s) for s in [_spec(i, MIXED[0]) for i in range(6)]]
    a16 = _engine(gpt, reqs, 6, FP16)
    a32 = _engine(gpt, reqs, 6, 0)
    s12 = _static(gpt, embed, 12)
    b16 = _engine(gpt, reqs, 6, FP16)
    b32 = _engine(gpt, reqs, 6, 0)
    assert all(torch.equal(a16[i][0], b16[i][0]) and torch.equal(a16[i][1], b16[i][1]) for i in range(6))
    assert all(torch.equal(a32[i][0], b32[i][0]) and torch.equal(a32[i][1], b32[i][1]) for i in range(6))
    assert all(torch.equal(x[0], y[0]) for x, y in zip(s12, _static(gpt, embed, 12)))


def test_g4_small_handle_runs_the_fp16_engine():
    """max_batch 4: no tensor-core state until the first fp16 engine builds it; S = 3 there, S = 2 after."""
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    small, sembed = _build((gs, es), max_batch=4)
    big, bembed, _, _ = _model("plain")
    specs = [_spec(i, MIXED[0]) for i in range(5)]
    a = _engine(small, [_request(sembed, s) for s in specs], 3, FP16)
    b = _engine(big, [_request(bembed, s) for s in specs], 3, FP16)
    for i in range(5):
        assert torch.equal(a[i][0], b[i][0]) and torch.equal(a[i][1], b[i][1]), i
    with pytest.raises(_lib.CtbError, match="flags"):
        with torch.cuda.device(small.device_gpt):
            EngineDevice(small, [], 2, 16, True, 4)


# ---------------------------------------------------------------------------------------------------- G5
def _chat():
    from chattts_b200 import Chat
    from chattts_b200.synth import synth_all
    from stubs import StubSpeaker, StubTokenizer

    c = Chat()
    assert c.load_states(synth_all(0), tokenizer=StubTokenizer(), speaker=StubSpeaker(), device="cuda",
                         max_batch=4, max_context=256)
    return c


def test_g5_chat_fp16_infer_continuous_equals_open_engine():
    c = _chat()
    texts = ["hello there", "hi", "a somewhat longer sentence to speak", "ok"]
    params = [c.InferCodeParams(manual_seed=3 + i, max_new_token=24 + 9 * i, min_new_token=24 + 9 * i,
                                temperature=0.3 + 0.1 * i, show_tqdm=False) for i in range(len(texts))]
    got = dict(c.infer_continuous(texts, params_infer_code=params, slots=3, dtype=torch.float16))
    assert sorted(got) == list(range(len(texts)))
    with c.open_engine(slots=3, max_new_cap=60, dtype=torch.float16) as eng:
        jobs = [eng.submit(t, params_infer_code=p) for t, p in zip(texts, params)]
        wavs = [j.result(timeout=300) for j in jobs]
    for i in range(len(texts)):
        assert got[i].shape == wavs[i].shape, i
        assert float(np.sqrt(np.mean((got[i] - wavs[i]) ** 2))) < 1e-4, i
    fp32 = dict(c.infer_continuous(texts[:1], params_infer_code=params[:1], slots=3))
    assert fp32[0].size > 0 and got[0].size > 0


def test_g5_chat_fp16_stream_cancel_and_paragraph():
    import concurrent.futures

    c = _chat()
    p = c.InferCodeParams(manual_seed=5, max_new_token=120, min_new_token=120, stream_batch=16, stream_speed=6000,
                          pass_first_n_batches=0, show_tqdm=False)
    long = c.InferCodeParams(manual_seed=6, max_new_token=200, min_new_token=200, show_tqdm=False)
    with c.open_engine(slots=3, max_new_cap=200, use_decoder=False, dtype=torch.float16) as eng:
        s = eng.submit("one", params_infer_code=p, stream=True)
        a = eng.submit("two", params_infer_code=long)
        para = eng.submit("First sentence here. And a second one!", params_infer_code=c.InferCodeParams(
            manual_seed=8, max_new_token=40, show_tqdm=False), split_text=True)
        it = iter(s)
        first = next(it)  # 16 of 120 tokens streamed: "two" (200 tokens) is still decoding
        a.cancel()
        chunks = [first] + list(it)
        assert chunks[-1][1] is True and not any(last for _, last in chunks[:-1])
        with pytest.raises(concurrent.futures.CancelledError):
            a.result(timeout=120)
        wav = para.result(timeout=300)
        assert wav.ndim == 1 and wav.size > 0
