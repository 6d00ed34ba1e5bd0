"""The static-batch decode steps of 1 to 8 rows - k_flow (csrc/flow.cuh) and k_step (csrc/mega.cuh) - against float64,
and k_flow's in-kernel sampler against k_sample.

A. In-kernel sampler = k_sample, bit for bit.  At B <= 2 on audio rows k_flow samples inside the kernel, up to 64 steps
   per launch (fl_sample_row); CTB_FLOW_NO_INK=1 at ctb_gpt_create makes the same handle launch k_flow one step at a
   time and sample with k_sample / k_finalize.  Two handles over one weight blob, both CTB_FLOW_MAX_BATCH=2, run the
   same calls at B = 1 and 2 and must give identical ids, end_idx and hidden states: the six (top_p, top_k, penalty)
   rows of test_gpu_gpt.py::test_sampler_kernel_vs_oracle, greedy with and without the EOS column, per-codebook
   temperatures, a penalty window of 31 (the largest), device Philox noise, a streamed call whose windows are not
   multiples of 64, a temperature-1.5 batch in which one row meets EOS, and min_new_token bans that end at steps 1, 63,
   64, 65 and 130 - inside a launch, on its last step and on the next launch's first (the whole call is one
   ctb_gpt_decode, so launches cover steps 1..64, 65..128, ...).  For those the EOS id is a token k_sample draws at
   exactly step min_new_token, so the row must end there.  Both handles must report their step (ctb_gpt_step_kind), and
   the launch counter must show <= ceil(steps / 64) + 2 decode launches on the first and >= 2 per step on the second.
B. k_flow against float64: B = 1 rows decoded to the full default context of 2,560 keys from prompts of 16, 64 and
   1,100 tokens (the last walked column by column through the decode kernels); B = 2, 3, 4 with ragged left-padded
   prompts, whose longest row ends exactly at max_context, running S = min(6, SMs / (12 B)) attention splits (6, 5, 3,
   2 on 132 SMs); text rows at B = 1 through the 21,178-wide head.
C. k_step against float64: the same audio workloads under CTB_NO_FLOW=1 at B = 1, 2 (64-key chunks), 3, 4 (128-key
   chunks) and B = 8 (CTB_MEGA_MAX_BATCH=8), S = min(40, SMs / (12 B)) splits (11, 5, 3, 2, 1 on 132 SMs).

B and C run on the synthetic model and on its peaked variant (q_proj and k_proj x 4, score std ~5): with near-uniform
scores every split's running max is about the same, so only the peaked model makes a wrong rescale of a split's
partial visible.  Each row is compared with tests/f64_oracle.py teacher-forced along the GPU's ids (checks as in
test_gpu_long_attention.py): each step's ids must be the float64-sampled ids unless the decision margin is below
MARGIN, and every step's hidden state must be within the bars below.  References are cached by ids content, so k_step
runs that produce k_flow's ids reuse its references.

Runs in ~3.5 minutes on one H100 (700 W), the float64 references (sampled on the CPU) included.
"""
import math
import os

import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.config import Config
from chattts_b200.embed import Embed
from chattts_b200.gpt import GPT
from chattts_b200.processors import (ArgmaxOnly, CustomRepetitionPenaltyLogitsProcessorRepeat, TopPLogitsWarper,
                                     gen_logits)
from chattts_b200.prompts import synth_prompt_batch
from chattts_b200.synth import synth_embed_state, synth_gpt_state
from f64_oracle import F64Oracle, peaked_state, sample_trace
from gpu_util import expect_step, release_on_teardown
from oracle.gpt_oracle import SamplerParams, exp_noise

pytestmark = pytest.mark.gpu

EOS, TEXT_EOS, TEXT_V = 625, 21001, 21178
MAX_CONTEXT = 2560  # GPT's default
MARGIN = 1e-3
# Bars; in brackets the largest distance observed on one H100 80 GB HBM3 (132 SMs, 700 W)
# step 0: the prefill's token (3xTF32 GEMMs), or the last column of a prompt walked by the step
FP32_ATOL = 2e-4  # [8.9e-5]
FP32_DECODE_ATOL = 6e-5  # steps 1.. [1.5e-5]
PEAKED_ATOL = 1e-3  # peaked model, every step [3.9e-4]

PARAMS = [(0.7, 20, 1.05), (None, 20, 1.0), (0.5, None, 1.05), (0.7, 20, 1.0), (0.95, 3, 1.2), (None, None, 1.05)]
TEMPS = [[0.3, 0.5, 0.7, 1.0], [0.7] * 4, [1.0, 0.3, 0.3, 0.5], [0.5] * 4, [0.3] * 4, [1.0] * 4]
# prompt lengths of the static batches; the longest row of each ends at max_context (B = 8: at 1,560 keys)
BATCHES = {1: [[16], [64], [1100]], 2: [[1000, 37]], 3: [[1200, 650, 8]], 4: [[1024, 512, 77, 300]],
           8: [[1024, 8, 300, 40, 129, 256, 640, 77]]}
MAX_NEW_B8 = 536

FLOW_ENV = {"CTB_FLOW_MAX_BATCH": "4"}
STEP_ENV = {"CTB_NO_FLOW": "1", "CTB_MEGA_MAX_BATCH": "8"}
INK_ENV = {"CTB_FLOW_MAX_BATCH": "2"}
EXT_ENV = {"CTB_FLOW_MAX_BATCH": "2", "CTB_FLOW_NO_INK": "1"}

_weights, _handles, _oracles, _refs = {}, {}, {}, {}
_release = release_on_teardown(_handles, _weights, _oracles, _refs)


def _model(kind):
    """(gpt_state, embed, packed device blob) of 'plain' (the synthetic model) or 'peaked'."""
    if kind not in _weights:
        gs, es = synth_gpt_state(0), synth_embed_state(1)
        if kind == "peaked":
            gs = peaked_state(gs)
        cfg = Config()
        embed = Embed(cfg.embed.hidden_size, cfg.embed.num_audio_tokens, cfg.embed.num_text_tokens,
                      cfg.embed.num_vq).load_state_dict(es).to("cuda")
        packer = GPT(cfg.gpt, embed, device="cuda", device_gpt="cuda", max_batch=1, max_context=MAX_CONTEXT)
        _, lay = packer.query_layout()
        _weights[kind] = (gs, es, embed, packer.pack_weights(gs, lay).cuda())
    return _weights[kind]


def _gpt(kind, env, max_batch, max_context=MAX_CONTEXT):
    """A handle over ``kind``'s blob, created with ``env`` added to the environment -> (gpt, embed)."""
    key = (kind, tuple(sorted(env.items())), max_batch, max_context)
    if key not in _handles:
        _, _, embed, blob = _model(kind)
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=max_batch,
                      max_context=max_context)
            gpt.load_state(None, weights_blob=blob)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        _handles[key] = gpt
    gpt = _handles[key]
    gpt.embed._gpt = gpt  # the embedding tables are every handle's; embed through this one
    return gpt, gpt.embed


def _generate(gpt, lengths, procs, temp, min_new, max_new, seed, *, pseed=5, eos=EOS, text=False, stream=False,
              stream_batch=24, philox=None):
    """gpt.generate over synth_prompt_batch(lengths, pseed) -> (every yield, prompt ids).  ``seed`` None: device Philox
    noise, with torch's generator seeded to ``philox`` first (it draws the Philox seed)."""
    ids, mask, tmask = synth_prompt_batch(lengths, seed=pseed)
    emb = gpt.embed(ids, tmask)
    if seed is None:
        torch.manual_seed(philox)
    outs = list(gpt.generate(emb, ids, temperature=torch.tensor(temp), eos_token=eos, attention_mask=mask,
                             max_new_token=max_new, min_new_token=min_new, logits_processors=procs, infer_text=text,
                             return_hidden=True, show_tqdm=False, manual_seed=seed, stream=stream,
                             stream_batch=stream_batch))
    return outs, ids


def _host(out):
    return [t.cpu().clone() for t in out.ids], [t.cpu().clone() for t in out.hiddens]


# ---------------------------------------------------------------------------------------------------- A
def _ab(B, max_context=640):
    """The in-kernel-sampling handle and the k_sample handle (same blob), each checked for its step at B rows."""
    ink, _ = _gpt("plain", INK_ENV, 2, max_context)
    ext, _ = _gpt("plain", EXT_ENV, 2, max_context)
    expect_step(ext, B, _lib.STEP_FLOW)
    expect_step(ink, B, _lib.STEP_FLOW_INK)
    return ink, ext


def _same(tag, a, b):
    """Two lists of generate() yields are identical: ids (so end_idx) and hidden states, yield by yield."""
    assert len(a) == len(b), (tag, len(a), len(b))
    for y, (oa, ob) in enumerate(zip(a, b)):
        (ia, ha), (ib, hb) = _host(oa), _host(ob)
        for r in range(len(ia)):
            assert ia[r].shape == ib[r].shape, (tag, y, r, "end_idx", ia[r].shape[0], ib[r].shape[0])
            if not torch.equal(ia[r], ib[r]):
                t = int((ia[r] != ib[r]).reshape(ia[r].shape[0], -1).any(1).float().argmax())
                raise AssertionError((tag, y, r, "first differing step", t, ia[r][t].tolist(), ib[r][t].tolist()))
            assert torch.equal(ha[r], hb[r]), (tag, y, r, float((ha[r] - hb[r]).abs().max()))


def _both(tag, B, monkeypatch, **kw):
    """The same call on both handles, the whole decode in one ctb_gpt_decode (64-step launches) -> the ink yields."""
    monkeypatch.setenv("CTB_DECODE_CHUNK", "4096")
    ink, ext = _ab(B)
    lengths = [16, 9][:B]
    a, _ = _generate(ink, lengths, **kw)
    b, _ = _generate(ext, lengths, **kw)
    _same(tag, a, b)
    return a


def _procs(params, window=16):
    tp, tk, rp = params
    warp, proc = gen_logits(num_code=EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    if window != 16:
        proc = [CustomRepetitionPenaltyLogitsProcessorRepeat(rp, EOS, window)]
    return (*proc, *warp)


# the (top_p, top_k, penalty) rows of test_gpu_gpt.py::test_sampler_kernel_vs_oracle
SAMPLER_ROWS = [(0.7, 20, 1.05), (0.95, 3, 1.2), (None, 20, 1.0), (0.5, None, 1.05), (None, None, 1.0), (0.05, 1, 1.5)]
# (tag, logits processors, temperatures, min_new, seed)
A_CASES = [(f"params{i}", _procs(p), t, 200, 31 + i) for i, (p, t) in enumerate(zip(SAMPLER_ROWS, TEMPS))] + [
    ("greedy", (*_procs((0.7, 20, 1.05)), ArgmaxOnly()), [0.3, 0.5, 0.7, 1.0], 0, 41),
    ("greedy_no_eos", (*_procs((0.7, 20, 1.05)), ArgmaxOnly(exclude_eos=True)), [0.3, 0.5, 0.7, 1.0], 200, 42),
    ("window31", _procs((0.7, 20, 1.2), window=31), [0.3, 0.5, 0.7, 1.0], 200, 43),
    ("top_p_alone", (TopPLogitsWarper(0.8, min_tokens_to_keep=3),), [1.0] * 4, 200, 44)]


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("case", A_CASES, ids=[c[0] for c in A_CASES])
def test_a_sampler_matrix(case, B, monkeypatch):
    tag, procs, temp, min_new, seed = case
    outs = _both(f"A {tag} B={B}", B, monkeypatch, procs=procs, temp=temp, min_new=min_new, max_new=200,
                 seed=seed)
    print(f"\nA {tag} B={B}: identical, rows end at {[int(t.shape[0]) for t in outs[-1].ids]} of 200")


@pytest.mark.parametrize("B", [1, 2])
def test_a_device_philox_noise(B, monkeypatch):
    for k in (3, 4):
        _both(f"A philox {k} B={B}", B, monkeypatch, procs=_procs((0.7, 20, 1.05)), temp=[0.8] * 4,
              min_new=150, max_new=150, seed=None, philox=k)


@pytest.mark.parametrize("B", [1, 2])
def test_a_stream_windows_not_multiples_of_64(B, monkeypatch):
    outs = _both(f"A stream B={B}", B, monkeypatch, procs=_procs((0.7, 20, 1.05)), temp=[0.3] * 4, min_new=250,
                 max_new=250, seed=7, stream=True, stream_batch=100)
    assert [int(o.ids[0].shape[0]) for o in outs] == [100, 200, 250]


def test_a_eos_inside_a_launch(monkeypatch):
    """Temperature 1.5, B = 2: a row meets EOS while the other decodes on, inside a 64-step launch."""
    outs = _both("A eos", 2, monkeypatch, procs=_procs((0.7, 20, 1.05)), temp=[1.5] * 4, min_new=2,
                 max_new=300, seed=7)
    n = sorted(int(t.shape[0]) for t in outs[-1].ids)
    print(f"\nA eos: rows end at {n} of 300")
    assert n[0] < n[1] and n[0] % 64 != 0, n


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("min_new", [1, 63, 64, 65, 130])
def test_a_min_new_token_ban_ends_at_a_launch_edge(min_new, B, monkeypatch):
    """The EOS id is a token k_sample draws at step min_new in a run where EOS (625) is banned throughout and that
    token never appears before: banning it before min_new changes no earlier step, so the row ends at exactly
    min_new.  Seeds are tried until the k_sample handle shows that; the in-kernel sampler must then agree."""
    monkeypatch.setenv("CTB_DECODE_CHUNK", "4096")
    ink, ext = _ab(B)
    lengths, procs, temp, max_new = [16, 9][:B], _procs((0.7, 20, 1.05)), [0.3, 0.5, 0.7, 1.0], 200
    for seed in range(100, 116):
        probe = _host(_generate(ext, lengths, procs, temp, max_new, max_new, seed)[0][-1])[0][0]
        before = set(probe[:min_new].flatten().tolist())
        cand = [int(t) for t in probe[min_new] if int(t) not in before and int(t) != EOS]
        if not cand:
            continue
        b, _ = _generate(ext, lengths, procs, temp, min_new, max_new, seed, eos=cand[0])
        if int(b[-1].ids[0].shape[0]) == min_new:
            break
    else:
        raise AssertionError(f"no seed gives a row that ends at step {min_new}")
    a, _ = _generate(ink, lengths, procs, temp, min_new, max_new, seed, eos=cand[0])
    _same(f"A min_new={min_new} B={B} eos={cand[0]} seed={seed}", a, b)


def test_a_launch_counts(monkeypatch):
    """The in-kernel sampler runs 64 steps per launch; the k_sample handle launches its step, sampler and finalize
    every step.  Launches of a call minus those of the same call stopped after its first step (the prefill)."""
    monkeypatch.setenv("CTB_DECODE_CHUNK", "4096")
    lib = _lib.load()
    steps = 300
    for B in (1, 2):
        ink, ext = _ab(B)
        got = {}
        for tag, gpt in (("ink", ink), ("ext", ext)):
            n = []
            for max_new in (1, steps):
                c0 = lib.ctb_launch_count()
                _generate(gpt, [16, 9][:B], _procs((0.7, 20, 1.05)), [0.3] * 4, max_new, max_new, 9)
                n.append(lib.ctb_launch_count() - c0)
            got[tag] = n[1] - n[0]
        print(f"\nA launches B={B}: in-kernel sampler {got['ink']}, k_sample {got['ext']} for {steps - 1} steps")
        assert got["ink"] <= math.ceil((steps - 1) / 64) + 2, got
        assert got["ext"] >= 2 * (steps - 1), got


# ---------------------------------------------------------------------------------------------------- B, C
def _oracle(kind):
    if kind not in _oracles:
        gs, es, _, _ = _model(kind)
        _oracles[kind] = F64Oracle(gs, es, device="cuda")
    return _oracles[kind]


def _reference(kind, prompt, ids, params, temp, q, qkey, text):
    """(hidden states, sampled ids [n, rows], margins) of the float64 model teacher-forced along ``ids``; cached by
    content, so runs that produced the same ids share one reference."""
    key = (kind, text, prompt.numpy().tobytes(), params, tuple(temp), qkey, ids.numpy().tobytes())
    if key not in _refs:
        orc = _oracle(kind)
        tp, tk, rp = params
        if text:
            hid, lg = orc.teacher_forced_text(orc.embed_prompt(prompt), ids)
            ids, eos, sp = ids[:, None], TEXT_EOS, SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp,
                                                                 penalty_max_ids=TEXT_V)
        else:
            hid, lg = orc.teacher_forced(orc.embed_prompt(prompt), ids)
            eos, sp = EOS, SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp)
        threads = torch.get_num_threads()
        torch.set_num_threads(1)  # [rows, V] operations: threads cost more than they give
        try:
            sampled, margins = sample_trace(lg, ids, torch.tensor(temp), sp, q, eos, ids.shape[0])
        finally:
            torch.set_num_threads(threads)
        _refs[key] = (hid.cpu(), sampled, margins)
    return _refs[key]


def _splits(step, B):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min(6 if step == "k_flow" else math.ceil(MAX_CONTEXT / 64), sms // (12 * B)))


def _run_and_check(tag, kind, gpt, lengths, case, text=False):
    """One static batch against float64; returns (worst step-0 distance, worst later distance, accepted, steps)."""
    params, temp = PARAMS[case % len(PARAMS)], ([0.7] if text else TEMPS[case % len(TEMPS)])
    max_new = MAX_NEW_B8 if len(lengths) == 8 else MAX_CONTEXT - max(lengths)
    seed = 500 + case
    tp, tk, rp = params
    warp, proc = gen_logits(num_code=TEXT_V if text else EOS, top_P=tp, top_K=tk, repetition_penalty=rp)
    outs, ids = _generate(gpt, lengths, (*proc, *warp), temp, max_new, max_new, seed, pseed=60 + case,
                          eos=TEXT_EOS if text else EOS, text=text)
    got_ids, got_hid = _host(outs[-1])
    B, rows = len(lengths), 1 if text else 4
    q = exp_noise(B * rows, TEXT_V if text else EOS + 1, seed)
    worst0 = worst = 0.0
    accepted = total = 0
    for b, L in enumerate(lengths):
        g, h = got_ids[b], got_hid[b]
        assert g.shape[0] == max_new and h.shape[0] == max_new, (tag, b, g.shape, h.shape)
        ref, sampled, margins = _reference(kind, ids[b, -L:], g, params, temp, q[rows * b: rows * (b + 1)],
                                           (seed, b), text)
        g2 = g[:, None] if text else g
        for t in range(max_new):
            total += 1
            if not torch.equal(sampled[t], g2[t].long()):
                assert margins[t] < MARGIN, (tag, b, L, t, g2[t].tolist(), sampled[t].tolist(), float(margins[t]))
                accepted += 1
        e = (h.double() - ref).abs()
        e0, ed = float(e[0].max()), float(e[1:].max())
        bar0, bar = (PEAKED_ATOL, PEAKED_ATOL) if kind == "peaked" else (FP32_ATOL, FP32_DECODE_ATOL)
        assert e0 < bar0, (tag, b, L, max_new, "step 0", e0, bar0)
        assert ed < bar, (tag, b, L, max_new, "steps 1..", ed, bar, "worst step", int(e.amax(1).argmax()))
        worst0, worst = max(worst0, e0), max(worst, ed)
    return worst0, worst, accepted, total


def _report(tag, res):
    w0 = max(r[0] for r in res)
    w = max(r[1] for r in res)
    print(f"\n{tag}: max |hidden - f64| at step 0 {w0:.3e}, at steps 1.. {w:.3e}; margin-accepted steps "
          f"{sum(r[2] for r in res)} of {sum(r[3] for r in res)}")


@pytest.mark.parametrize("kind", ["plain", "peaked"])
@pytest.mark.parametrize("B", [1, 2, 3, 4])
def test_b_flow_vs_float64(B, kind):
    gpt, _ = _gpt(kind, FLOW_ENV, 4)
    ink = B <= 2 and "CTB_FLOW_NO_INK" not in os.environ  # either way k_flow's attention and merge
    expect_step(gpt, B, _lib.STEP_FLOW_INK if ink else _lib.STEP_FLOW)
    res = [_run_and_check(f"B k_flow B={B} {kind}", kind, gpt, lengths, B + i) for i, lengths in enumerate(BATCHES[B])]
    _report(f"B k_flow B={B} S={_splits('k_flow', B)} {kind} rows {BATCHES[B]}", res)


@pytest.mark.parametrize("kind", ["plain", "peaked"])
def test_b_flow_text_rows_vs_float64(kind):
    gpt, _ = _gpt(kind, FLOW_ENV, 4)
    expect_step(gpt, 1, _lib.STEP_FLOW, infer_text=True)
    res = [_run_and_check(f"B k_flow text {kind}", kind, gpt, lengths, 20 + i, text=True)
           for i, lengths in enumerate([[1800], [2200]])]
    _report(f"B k_flow text B=1 S={_splits('k_flow', 1)} {kind}", res)


@pytest.mark.parametrize("kind", ["plain", "peaked"])
@pytest.mark.parametrize("B", [1, 2, 3, 4, 8])
def test_c_step_vs_float64(B, kind):
    gpt, _ = _gpt(kind, STEP_ENV, 8)
    expect_step(gpt, B, _lib.STEP_MEGA)
    res = [_run_and_check(f"C k_step B={B} {kind}", kind, gpt, lengths, B + i) for i, lengths in enumerate(BATCHES[B])]
    chunk = 128 if B >= 3 else 64
    _report(f"C k_step B={B} S={_splits('k_step', B)} ({chunk}-key chunks) {kind} rows {BATCHES[B]}", res)
