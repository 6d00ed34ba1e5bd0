"""GPU parity of hot path 1 (through the C ABI) against the committed reference fixtures and
the live CPU oracle.  Bit-exact for token ids; hidden states within 1e-4 abs (fp32 reorder)."""
import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200.processors import ArgmaxOnly, build_sampler_config, exp_noise, gen_logits
from chattts_b200.prompts import synth_prompt_batch
from oracle.gpt_oracle import GPTOracle, SamplerParams, sample_step

pytestmark = pytest.mark.gpu


def _run(gpt, embed, lengths, pseed, sseed, steps, *, text=False, top_P=0.7, top_K=20, rp=1.05, min_new=None,
         extra=(), temp=None, stream=False):
    ids, mask, tmask = synth_prompt_batch(lengths, seed=pseed)
    warp, proc = gen_logits(num_code=21178 if text else 625, top_P=top_P, top_K=top_K, repetition_penalty=rp)
    emb = embed(ids, tmask)
    gen = gpt.generate(emb, ids, temperature=torch.tensor(temp or ([0.7] if text else [0.3] * 4)),
                       eos_token=21001 if text else 625, attention_mask=mask, max_new_token=steps,
                       min_new_token=steps if min_new is None else min_new, logits_processors=(*proc, *warp, *extra),
                       infer_text=text, return_hidden=not text, show_tqdm=False, manual_seed=sseed, stream=stream)
    return list(gen)


@pytest.mark.parametrize("name", ["gpt_audio_b1", "gpt_audio_b3_ragged", "gpt_audio_b2_nopenalty_topk5"])
def test_generate_matches_reference_fixture(name):
    from gpu_util import build_gpt, load_gold

    gpt, embed, _, _ = build_gpt()
    g = load_gold(name)
    kw = dict(top_P=0.9, top_K=5, rp=1.0) if "nopenalty" in name else {}
    out = _run(gpt, embed, g["lengths"].tolist(), int(g["prompt_seed"]), int(g["sampler_seed"]), int(g["steps"]), **kw)[-1]
    for b in range(len(g["lengths"])):
        n = int(g["n"][b])
        assert np.array_equal(out.ids[b].cpu().numpy(), g["ids"][b, :n]), (b, out.ids[b][:4], g["ids"][b, :4])
        assert np.abs(out.hiddens[b].cpu().numpy() - g["hiddens"][b][:n]).max() < 1e-4


def test_text_generate_matches_reference_fixture():
    from gpu_util import build_gpt, load_gold

    gpt, embed, _, _ = build_gpt()
    g = load_gold("gpt_text_b2")
    out = _run(gpt, embed, g["lengths"].tolist(), int(g["prompt_seed"]), int(g["sampler_seed"]), int(g["steps"]),
               text=True, rp=1.0, min_new=0)[-1]
    for b in range(2):
        assert np.array_equal(out.ids[b].cpu().numpy(), g["ids"][b, : int(g["n"][b]), 0])


@pytest.mark.parametrize("lengths,steps,sseed", [([16], 48, 1234), ([3, 20, 11, 7, 16], 24, 5)])
def test_generate_matches_live_oracle(lengths, steps, sseed):
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch(lengths, seed=9)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=steps, min_new_token=4, sampler=SamplerParams(), return_hidden=True,
                       manual_seed=sseed)
    out = _run(gpt, embed, lengths, 9, sseed, steps, min_new=4)
    if not ref.ids:  # first-step EOS: the reference generator ends without yielding (gpt.py:527-570)
        assert out == []
        return
    out = out[-1]
    for b in range(len(lengths)):
        assert torch.equal(out.ids[b].cpu(), ref.ids[b]), b
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 1e-4


def test_greedy_processor_and_larger_weights():
    """std=0.05 weights make attention/MLP contributions O(1): structure errors cannot hide."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(seed=3, std=0.05)
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch([9, 14], seed=4)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=20, min_new_token=20, sampler=SamplerParams(greedy=True, greedy_exclude_eos=True), return_hidden=True,
                       manual_seed=1)
    out = _run(gpt, embed, [9, 14], 4, 1, 20, extra=(ArgmaxOnly(exclude_eos=True),))[-1]
    for b in range(2):
        assert torch.equal(out.ids[b].cpu(), ref.ids[b])
        # |hidden| reaches ~4 with these weights and reorder noise compounds over 20 layers: 1e-4 relative
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 5e-4


@pytest.mark.parametrize("V,rpi,rows", [(626, 4, 32), (626, 4, 8), (21178, 1, 6)])
@pytest.mark.parametrize("tp,tk,rp", [(0.7, 20, 1.05), (0.95, 3, 1.2), (None, 20, 1.0), (0.5, None, 1.05),
                                      (None, None, 1.0), (0.05, 1, 1.5)])
def test_sampler_kernel_vs_oracle(V, rpi, rows, tp, tk, rp):
    g = torch.Generator().manual_seed(V + rows)
    logits = torch.randn(rows, V, generator=g) * 1.5
    n_gen = 23
    gen = torch.randint(0, 30, (rows // rpi, n_gen, rpi), generator=g)
    temp = [0.3, 0.5, 0.7, 1.0][:rpi]
    q = exp_noise(rows, V, 77)
    eos = V - 1
    for step, min_new in ((0, 0), (3, 10)):
        sp = SamplerParams(top_p=tp, top_k=tk, repetition_penalty=rp, penalty_max_ids=V - 1)
        ref = sample_step(logits, gen.permute(0, 2, 1).reshape(rows, n_gen), torch.tensor(temp), sp, q, eos,
                          step < min_new)
        warp, proc = gen_logits(num_code=V - 1, top_P=tp, top_K=tk, repetition_penalty=rp)
        cfg = build_sampler_config((*proc, *warp), temp, eos, min_new)
        from chattts_b200.sampler import sample_rows

        out = sample_rows(logits.cuda(), cfg, rpi, q.cuda(), gen.cuda(), step=step)
        assert torch.equal(out.cpu().long(), ref), (out.cpu()[:8], ref[:8])


def test_sampler_reference_fixture():
    from gpu_util import load_gold
    from chattts_b200.sampler import sample_rows

    g = load_gold("sampler_rows")
    logits = torch.from_numpy(g["logits"]).cuda()
    gen = torch.from_numpy(g["gen_ids"])  # [rows, n_gen] per (b,q) row
    rows, n_gen = gen.shape
    gen3 = gen.view(rows // 4, 4, n_gen).permute(0, 2, 1).contiguous()
    q = exp_noise(rows, logits.shape[1], int(g["seed"])).cuda()
    for tag, (tp, tk, rp) in {"default": (0.7, 20, 1.05), "p95k3": (0.95, 3, 1.2), "nop": (None, 20, 1.0),
                              "nok": (0.5, None, 1.05)}.items():
        warp, proc = gen_logits(num_code=625, top_P=tp, top_K=tk, repetition_penalty=rp)
        cfg = build_sampler_config((*proc, *warp), g["temperature"].tolist(), 625, 0)
        out = sample_rows(logits, cfg, 4, q, gen3.cuda())
        assert np.array_equal(out.cpu().numpy(), g["idx_" + tag]), tag


def test_unknown_processor_raises_no_fallback():
    with pytest.raises(TypeError):
        build_sampler_config((lambda ids, s: s,), [0.3] * 4, 625, 0)


def test_streaming_yields_cumulative_chunks():
    from gpu_util import build_gpt

    gpt, embed, _, _ = build_gpt()
    outs = _run(gpt, embed, [16], 1, 1234, 60, stream=True)
    lens = [int(o.ids[0].shape[0]) for o in outs]
    assert lens == [24, 48, 60]
    full = _run(gpt, embed, [16], 1, 1234, 60)[-1]
    assert torch.equal(outs[-1].ids[0], full.ids[0]) and torch.equal(outs[0].ids[0], full.ids[0][:24])


def _back_end_run(lengths):
    """The 80-step run of test_every_decode_back_end_gives_the_same_ids on a handle created with the environment as it
    is: (the handle's GPT, its outputs)."""
    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.gpt import GPT
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    gs, es = synth_gpt_state(0), synth_embed_state(1)
    embed = Embed(768, 626, 21178, 4).load_state_dict(es).to("cuda")
    gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=len(lengths), max_context=128)
    gpt.load_state(gs)
    return gpt, _run(gpt, embed, lengths, 13, 21, 80)[-1]


# CTB_NO_PDL is read once per process (the launch helper of common.cuh), so its leg runs in a child process
_CHILD = """
import sys
import torch
sys.path[:0] = [{root!r}, {tests!r}]
from chattts_b200 import _lib
from test_gpu_gpt import _back_end_run
gpt, out = _back_end_run({lengths!r})
torch.save(dict(kind=_lib.step_kind(gpt._handle, {B}), ids=[t.cpu() for t in out.ids],
                hiddens=[t.cpu() for t in out.hiddens]), {path!r})
"""


def _back_end_run_in_child(env, lengths, tmp_path):
    import os
    import subprocess
    import sys

    tests = os.path.dirname(os.path.abspath(__file__))
    path = str(tmp_path / "child.pt")
    code = _CHILD.format(root=os.path.dirname(tests), tests=tests, lengths=list(lengths), B=len(lengths), path=path)
    flags = ["-s"] if sys.flags.no_user_site else []
    # run() kills the child if it outlives the timeout
    r = subprocess.run([sys.executable, *flags, "-c", code], env={**os.environ, **env}, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    got = torch.load(path)
    return got["kind"], got["ids"], got["hiddens"]


# (environment at ctb_gpt_create, prompt lengths, the decode step that must serve the batch)
BACK_ENDS = [
    ({"CTB_GPT_TC": "1"}, [5, 12, 9], _lib.STEP_WGMMA), ({"CTB_GPT_TC": "1"}, [16], _lib.STEP_WGMMA),
    ({"CTB_NO_FLOW": "1", "CTB_MEGA_MAX_BATCH": "8"}, [5, 12, 9], _lib.STEP_MEGA),
    ({"CTB_NO_FLOW": "1"}, [16], _lib.STEP_MEGA), ({"CTB_NO_FLOW": "1", "CTB_NO_MEGA": "1"}, [16], _lib.STEP_FMA),
    ({"CTB_NO_FLOW": "1", "CTB_NO_MEGA": "1", "CTB_NO_GRAPH": "1", "CTB_NO_PDL": "1"}, [7, 3], _lib.STEP_FMA),
    ({"CTB_FLOW_NO_INK": "1", "CTB_FLOW_MAX_BATCH": "4"}, [7, 3], _lib.STEP_FLOW),
    ({"CTB_FLOW_R": "4", "CTB_FLOW_MAX_BATCH": "4"}, [5, 12, 9, 3], _lib.STEP_FLOW),
    ({"CTB_FLOW_MAX_BATCH": "2"}, [7, 3], _lib.STEP_FLOW_INK)]


@pytest.mark.parametrize("env,lengths", [(e, n) for e, n, _ in BACK_ENDS])
def test_every_decode_back_end_gives_the_same_ids(env, lengths, tmp_path):
    """The step implementations - the dataflow step (flow.cuh, default for B = 1) with and without its in-kernel
    sampler, the grid-barrier one-kernel step (mega.cuh), the PDL-chained FMA kernels (and the same kernels launched
    plainly, CTB_NO_PDL) and the wgmma 3xTF32 GEMM step (tc_decode.cuh) - are selected by batch size; each is forced
    here on batches it would not get by default, the handle must report that it got it (ctb_gpt_step_kind), and it must
    reproduce the CPU oracle's ids exactly."""
    import os

    from chattts_b200.synth import synth_embed_state, synth_gpt_state
    from gpu_util import expect_step

    kind = next(k for e, n, k in BACK_ENDS if (e, n) == (env, lengths))
    gs, es = synth_gpt_state(0), synth_embed_state(1)
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch(lengths, seed=13)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=80, min_new_token=80, sampler=SamplerParams(), return_hidden=True, manual_seed=21)
    if "CTB_NO_PDL" in env:
        got, out_ids, out_hid = _back_end_run_in_child(env, lengths, tmp_path)
        assert got == kind, (env, _lib.STEP_NAMES.get(got, got))
    else:
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            gpt, out = _back_end_run(lengths)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        expect_step(gpt, len(lengths), kind)
        out_ids, out_hid = out.ids, out.hiddens
    for b in range(len(lengths)):
        assert torch.equal(out_ids[b].cpu(), ref.ids[b]), (env, b)
        assert (out_hid[b].cpu() - ref.hiddens[b]).abs().max() < 1e-4


def test_batch_larger_than_one_tile_matches_oracle():
    """B = 34 > 32: the FMA kernels re-stream the weights per 32-row batch tile (grid.y); rows must still be
    independent of the batch they are decoded in (compare rows 0, 31, 32, 33 with the oracle run on those rows)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(max_batch=34, max_context=64)
    orc = GPTOracle(gs, es)
    lengths = [6 + (i % 5) for i in range(34)]
    ids, mask, tmask = synth_prompt_batch(lengths, seed=17)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    out = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([0.3] * 4), eos_token=625,
                            attention_mask=mask, max_new_token=6, min_new_token=6, logits_processors=(*proc, *warp),
                            return_hidden=True, show_tqdm=False, manual_seed=3))[-1]
    rows = [0, 31, 32, 33]
    # the Exp(1) noise is indexed by the global row (prefix-stable), so the oracle runs the full batch on the CPU
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=6, min_new_token=6, sampler=SamplerParams(), return_hidden=True, manual_seed=3)
    for b in rows:
        assert torch.equal(out.ids[b].cpu(), ref.ids[b]), b
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 1e-4


def test_unseeded_generation_uses_device_philox_and_is_valid():
    from gpu_util import build_gpt

    gpt, embed, _, _ = build_gpt()
    ids, mask, tmask = synth_prompt_batch([9, 5], seed=2)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    outs = []
    for _ in range(2):
        o = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([0.8] * 4), eos_token=625,
                              attention_mask=mask, max_new_token=24, min_new_token=24, logits_processors=(*proc, *warp),
                              return_hidden=False, show_tqdm=False, manual_seed=None))[-1]
        assert all(t.shape == (24, 4) and int(t.min()) >= 0 and int(t.max()) < 626 for t in o.ids)
        outs.append(torch.stack(o.ids))
    assert not torch.equal(outs[0], outs[1])  # fresh Philox stream per call (no parity target, SURVEY.md 7)


def test_batched_prefill_long_ragged_prompts():
    """SURVEY.md 8f N1: prompts of 40..128 tokens, left padded, go through the token-parallel wgmma prefill
    (prefill.cuh); ids must equal the CPU oracle's and the column-by-column prefill's."""
    import os

    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.gpt import GPT
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    gs, es = synth_gpt_state(0), synth_embed_state(1)
    lengths = [40, 128, 77]
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch(lengths, seed=23)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=10, min_new_token=10, sampler=SamplerParams(), return_hidden=True, manual_seed=5)
    outs = {}
    for tag, env in (("batched", {}), ("columns", {"CTB_NO_BATCHED_PREFILL": "1"})):
        os.environ.update(env)
        try:
            embed = Embed(768, 626, 21178, 4).load_state_dict(es).to("cuda")
            gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=3, max_context=160)
            gpt.load_state(gs)
            outs[tag] = _run(gpt, embed, lengths, 23, 5, 10)[-1]
        finally:
            for k in env:
                os.environ.pop(k, None)
    for b in range(3):
        assert torch.equal(outs["batched"].ids[b].cpu(), ref.ids[b]), b
        assert torch.equal(outs["columns"].ids[b].cpu(), ref.ids[b]), b
        assert (outs["batched"].hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 1e-4


def test_full_batch_rows_are_independent_of_batch_and_back_end():
    """BASELINE configs[2] scale: 32 mixed-length prompts decoded greedily in one batch (wgmma GEMM back end +
    batched prefill) must give, row by row, the ids of the same prompt decoded alone (one-kernel back end):
    rows never interact (SURVEY.md 8e) and every back end computes the same function."""
    from gpu_util import build_gpt

    big, embed, _, _ = build_gpt(max_batch=32, max_context=256)
    solo, _, _, _ = build_gpt(max_batch=1, max_context=256)
    g = torch.Generator().manual_seed(31)
    lengths = torch.randint(8, 129, (32,), generator=g).tolist()
    steps = 48
    batch = _run(big, embed, lengths, 41, 1, steps, extra=(ArgmaxOnly(exclude_eos=True),))[-1]
    ids, mask, tmask = synth_prompt_batch(lengths, seed=41)
    warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
    for b in (0, 7, 13, 31):
        n = lengths[b]
        row_ids = ids[b: b + 1, ids.shape[1] - n:]
        row_mask = torch.ones(1, n, dtype=torch.bool)
        out = list(solo.generate(embed(row_ids, row_mask), row_ids, temperature=torch.tensor([0.3] * 4), eos_token=625,
                                 attention_mask=row_mask, max_new_token=steps, min_new_token=steps,
                                 logits_processors=(*proc, *warp, ArgmaxOnly(exclude_eos=True)), return_hidden=False,
                                 show_tqdm=False, manual_seed=1))[-1]
        assert torch.equal(out.ids[0].cpu(), batch.ids[b].cpu()), b


def test_embed_prompt_kernel_matches_reference_embed_semantics():
    """Embed.forward (embed.py:51-79) through ctb_gpt_embed_prompt vs the oracle restatement, with mixed text/code
    positions (audio-prompt splice, tokenizer.py:115-124)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt()
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch([6, 3, 9], seed=5)
    tmask[0, -2:] = False
    ids[0, -2:] = torch.randint(0, 626, (2, 4))
    got = embed(ids, tmask)
    assert got.is_cuda and torch.equal(got.cpu(), orc.embed_prompt(ids, tmask))


@pytest.mark.parametrize("B", [24, 32])
def test_tensor_core_back_end_full_batches_vs_oracle(B):
    """VERDICT r1 weak #3: the wgmma decode back end at batch sizes it is the default for (9..32; here NPAD = 32)
    against the CPU oracle itself: ragged 8..128-token prompts (batched prefill), top-p 0.7 / top-k 20 / penalty 1.05."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(max_batch=32, max_context=256)
    orc = GPTOracle(gs, es)
    g = torch.Generator().manual_seed(100 + B)
    lengths = torch.randint(8, 129, (B,), generator=g).tolist()
    steps = 48
    ids, mask, tmask = synth_prompt_batch(lengths, seed=50 + B)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=steps, min_new_token=steps, sampler=SamplerParams(), return_hidden=True, manual_seed=77)
    out = _run(gpt, embed, lengths, 50 + B, 77, steps)[-1]
    for b in range(B):
        assert torch.equal(out.ids[b].cpu(), ref.ids[b]), (B, b)
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 1e-4


@pytest.mark.parametrize("lengths,steps,greedy", [([16], 512, True), ([16], 1100, False), ([16, 9, 30, 5], 300, False)])
def test_long_context_vs_oracle(lengths, steps, greedy):
    """VERDICT r1 weak #4: BASELINE configs[1] exactly (16-token prompt + 512 forced greedy tokens), a 1100-step B=1 run
    (contexts > 768 keys: every attention split walks several chunks, many KV pages) and a 300-step B=4 run, ids
    bit-equal to the CPU oracle."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(max_batch=4, max_context=1280)
    orc = GPTOracle(gs, es)
    ids, mask, tmask = synth_prompt_batch(lengths, seed=61)
    sp = SamplerParams(greedy=True, greedy_exclude_eos=True) if greedy else SamplerParams()
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=steps, min_new_token=steps, sampler=sp, return_hidden=True, manual_seed=1234)
    out = _run(gpt, embed, lengths, 61, 1234, steps, extra=(ArgmaxOnly(exclude_eos=True),) if greedy else ())[-1]
    for b in range(len(lengths)):
        assert out.ids[b].shape[0] == steps
        same = out.ids[b].cpu() == ref.ids[b]
        first = int((~same.all(-1)).float().argmax()) if not bool(same.all()) else -1
        assert first == -1, (b, first, out.ids[b][first].tolist(), ref.ids[b][first].tolist())
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 2e-4


def test_multi_step_launch_matches_single_step_launches():
    """The dataflow step kernel runs up to 64 decode iterations per launch with the sampling tail inside (csrc/flow.cuh);
    CTB_FLOW_NO_INK=1 at ctb_gpt_create launches one step at a time with k_sample / k_finalize outside.  Same ids, same
    early stop.  tests/test_gpu_small_batch_decode.py part A runs the sampler matrix on both."""
    import os

    from chattts_b200.config import Config
    from chattts_b200.embed import Embed
    from chattts_b200.gpt import GPT
    from chattts_b200.synth import synth_embed_state, synth_gpt_state

    from gpu_util import expect_step

    gs, es = synth_gpt_state(0), synth_embed_state(1)
    outs, gpts = {}, {}
    for tag, env in (("ink", {"CTB_FLOW_MAX_BATCH": "2"}), ("ext", {"CTB_FLOW_NO_INK": "1", "CTB_FLOW_MAX_BATCH": "2"})):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            embed = Embed(768, 626, 21178, 4).load_state_dict(es).to("cuda")
            gpt = GPT(Config().gpt, embed, device="cuda", device_gpt="cuda", max_batch=2, max_context=400)
            gpt.load_state(gs)
            gpts[tag] = gpt
            ids, mask, tmask = synth_prompt_batch([16, 9], seed=3)
            warp, proc = gen_logits(num_code=625, top_P=0.7, top_K=20, repetition_penalty=1.05)
            outs[tag] = list(gpt.generate(embed(ids, tmask), ids, temperature=torch.tensor([1.5] * 4), eos_token=625,
                                          attention_mask=mask, max_new_token=200, min_new_token=2,
                                          logits_processors=(*proc, *warp), return_hidden=True, show_tqdm=False,
                                          manual_seed=7))[-1]
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    expect_step(gpts["ext"], 2, _lib.STEP_FLOW)
    expect_step(gpts["ink"], 2, _lib.STEP_FLOW_INK)
    for b in range(2):
        assert torch.equal(outs["ink"].ids[b], outs["ext"].ids[b])
        assert torch.equal(outs["ink"].hiddens[b], outs["ext"].hiddens[b])
    assert len(outs["ink"].ids[0]) < 200  # high temperature: this row stops at an EOS well before max_new_token


def test_batched_prefill_512_token_prompts():
    """VERDICT r1 #8 / SURVEY.md 8f N1: prompts as long as speaker-prompt prefixes (up to 512 tokens, ragged) through the
    query-parallel prefill attention; first tokens and hidden states against the CPU oracle."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(max_batch=4, max_context=640)
    orc = GPTOracle(gs, es)
    lengths = [512, 300, 40]
    ids, mask, tmask = synth_prompt_batch(lengths, seed=29)
    ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                       max_new_token=12, min_new_token=12, sampler=SamplerParams(), return_hidden=True, manual_seed=5)
    out = _run(gpt, embed, lengths, 29, 5, 12)[-1]
    for b in range(3):
        assert torch.equal(out.ids[b].cpu(), ref.ids[b]), b
        assert (out.hiddens[b].cpu() - ref.hiddens[b]).abs().max() < 2e-4


def test_kv_pool_and_handle_are_reused_across_calls_of_different_shapes():
    """The KV pool is sized per generate() call (kv_reserve): a short call, then a much longer / wider one, then the
    short one again on the SAME handle must all reproduce the oracle (pages re-assigned, pool grown once)."""
    from gpu_util import build_gpt

    gpt, embed, gs, es = build_gpt(max_batch=4, max_context=1280)
    orc = GPTOracle(gs, es)
    for lengths, steps in (([9], 12), ([33, 120, 7], 200), ([9], 12)):
        ids, mask, tmask = synth_prompt_batch(lengths, seed=71)
        ref = orc.generate(orc.embed_prompt(ids, tmask), ids, torch.tensor([0.3] * 4), 625, attention_mask=mask,
                           max_new_token=steps, min_new_token=steps, sampler=SamplerParams(), return_hidden=True, manual_seed=9)
        out = _run(gpt, embed, lengths, 71, 9, steps)[-1]
        for b in range(len(lengths)):
            assert torch.equal(out.ids[b].cpu(), ref.ids[b]), (lengths, b)
