"""Attention maps of ``GPT.generate(return_attn=True)`` (ctb_gpt_attention_maps, k_attn_probs) on one H100.

M1: ids and hidden states are bit-equal with and without the maps, stream and not, on every static decode back end
(B = 1 k_flow, 3 k_step, 8 the PDL chain, 24 the wgmma step) and a left-padded ragged batch.  M2: the maps against
the float64 teacher-forced oracle (tests/attn_oracle.py) on the GPU's own ids: code and text rows, left padding, rows
that end early, a prompt over 1,024 tokens (walked through the decode kernels, whose pages the maps read) and several
hundred steps, with the structure checks (rows sum to 1, padding and rows past the end exactly 0, padded prompt rows
uniform).  M3: the reference's own eager maps (tests/golden/gpt_attn.npz).  M4: two runs give the same bits, and the
streamed list is one object extended in place.  M5: an interrupt keeps the steps done; the ABI's refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from attn_oracle import oracle_maps, pack_maps, step_offsets
from chattts_b200 import _lib
from chattts_b200.processors import gen_logits
from chattts_b200.prompts import synth_prompt_batch
from f64_oracle import F64Oracle
from gpu_util import build_gpt, release_on_teardown

pytestmark = pytest.mark.gpu

# max |GPU - float64 oracle| (and - the reference's fp32 eager maps) over every map entry: about 3.5x the largest
# distance measured on one H100 80 GB HBM3 at 700 W, 7.1e-6 to 7.5e-6 (DESIGN §4, "Attention maps")
BAR = 2.6e-5
_oracles = {}
_release = release_on_teardown(_oracles)


def _run(gpt, embed, lengths, steps, *, pseed=1, sseed=5, text=False, stream=False, attn=True, eos=None, min_new=None,
         context=None, stream_batch=24, return_hidden=None):
    ids, mask, tmask = synth_prompt_batch(lengths, seed=pseed)
    warp, proc = gen_logits(num_code=21178 if text else 625, top_P=0.7, top_K=20, repetition_penalty=1.0 if text else 1.05)
    emb = embed(ids, tmask)
    kw = dict(context=context) if context is not None else {}
    gen = gpt.generate(emb, ids, temperature=torch.tensor([0.7] if text else [0.3] * 4),
                       eos_token=(21001 if text else 625) if eos is None else eos, attention_mask=mask,
                       max_new_token=steps, min_new_token=(0 if text else steps) if min_new is None else min_new,
                       logits_processors=(*proc, *warp), infer_text=text, return_attn=attn,
                       return_hidden=(not text) if return_hidden is None else return_hidden, show_tqdm=False,
                       manual_seed=sseed, stream=stream, stream_batch=stream_batch, **kw)
    return emb, mask, gen


def _oracle(gs, es):
    if "f64" not in _oracles:
        _oracles["f64"] = F64Oracle(gs, es, device="cuda")
    return _oracles["f64"]


def _structure(maps, mask, end, steps):
    """Rows sum to 1, padded columns and steps past a row's end exactly 0, padded prompt rows exactly 1 / T0."""
    B, T0 = mask.shape
    for b in range(B):
        pad = T0 - int(mask[b].sum())
        for i, (o, r, c) in enumerate(step_offsets(T0, steps)):
            blk = maps[:, b, :, o: o + r * c].reshape(maps.shape[0], -1, r, c)
            if i > int(end[b]):
                assert (blk == 0).all(), (b, i)
                continue
            valid = blk[:, :, pad:, :] if r > 1 else blk
            assert ((valid.double().sum(-1) - 1).abs().max() < 1e-5), (b, i)
            assert (valid[..., :pad] == 0).all(), (b, i)
            if r > 1:
                assert (blk[:, :, :pad, :] == 1.0 / T0).all()
                assert (torch.ones(r, c, device=blk.device).triu(1)[None, None, pad:] * valid != 0).sum() == 0


def _check_against_oracle(name, gpt, embed, gs, es, lengths, steps, *, text=False, eos=None, pseed=1, sseed=5):
    emb, mask, gen = _run(gpt, embed, lengths, steps, text=text, eos=eos, pseed=pseed, sseed=sseed,
                          min_new=0 if eos is not None else None)
    out = list(gen)[-1]
    assert len(out.attentions) >= 1
    n_steps = len(out.attentions)
    L, H, T0 = gpt.config.num_hidden_layers, gpt.config.num_attention_heads, emb.shape[1]
    for i, a in enumerate(out.attentions):
        assert len(a) == L and all(t.dtype == torch.float32 and t.is_cuda for t in a)
        assert tuple(a[0].shape) == ((len(lengths), H, T0, T0) if i == 0 else (len(lengths), H, 1, T0 + i))
    maps = pack_maps(out.attentions)
    end = [len(t) for t in out.ids]
    _structure(maps, mask.cuda(), end, n_steps)
    ref = oracle_maps(_oracle(gs, es), emb, mask, [t.cpu() for t in out.ids], end, n_steps, text)
    d = (maps.double() - ref).abs().max().item()
    assert d < BAR, (name, d)
    return out, end, n_steps


def test_a_short_maps_run_leaves_longer_prefills_working():
    # first in the module: the maps pass must not lower a launch limit the prefill kernels rely on (a short run's
    # pass once set k_prefill_attn's dynamic shared memory limit to its own 800 bytes, and a 300-column prefill failed)
    gpt, embed, _, _ = build_gpt(max_context=700)  # a handle no other test uses
    before = list(_run(gpt, embed, [300, 280], 12, attn=False)[2])[-1]
    out = list(_run(gpt, embed, [16], 10)[2])[-1]
    assert len(out.attentions) == 10
    after = list(_run(gpt, embed, [300, 280], 12, attn=False)[2])[-1]
    assert all(torch.equal(x, y) for x, y in zip(before.ids, after.ids))
    assert all(torch.equal(x, y) for x, y in zip(before.hiddens, after.hiddens))


@pytest.mark.parametrize("lengths", [[16], [12, 14, 16], [16] * 8, [16] * 24, [5, 23, 11, 17]])
@pytest.mark.parametrize("stream", [False, True])
def test_ids_and_hiddens_unchanged(lengths, stream):
    gpt, embed, _, _ = build_gpt()
    outs = {}
    for attn in (False, True):
        outs[attn] = [(list(o.ids), list(o.hiddens), len(o.attentions))
                      for o in _run(gpt, embed, lengths, 40, stream=stream, attn=attn, stream_batch=16)[2]]
    assert len(outs[False]) == len(outs[True])
    for (i0, h0, a0), (i1, h1, a1) in zip(outs[False], outs[True]):
        assert a0 == 0 and a1 > 0
        assert all(torch.equal(x, y) for x, y in zip(i0, i1))
        assert all(torch.equal(x, y) for x, y in zip(h0, h1))


def test_maps_left_padded_code_rows_match_f64():
    gpt, embed, gs, es = build_gpt()
    _check_against_oracle("code_ragged_b4", gpt, embed, gs, es, [5, 23, 11, 17], 60)


def test_maps_text_rows_match_f64():
    gpt, embed, gs, es = build_gpt()
    _check_against_oracle("text_b2", gpt, embed, gs, es, [7, 19], 40, text=True)


def test_maps_rows_that_end_early():
    gpt, embed, gs, es = build_gpt()
    # an EOS id that row 0 samples at some step after the first, and no row samples at step 0
    full = list(_run(gpt, embed, [9, 16, 13], 40, attn=False, min_new=0)[2])[-1].ids
    first = {int(v) for t in full for v in t[0]}
    eos = next(int(v) for k in range(8, len(full[0])) for v in full[0][k] if int(v) not in first)
    out, end, n_steps = _check_against_oracle("code_early_end_b3", gpt, embed, gs, es, [9, 16, 13], 40, eos=eos)
    assert min(end) < n_steps - 1  # some row's later steps are zeros


def test_maps_long_prompt_match_f64():
    gpt, embed, gs, es = build_gpt(max_context=1400)
    _check_against_oracle("long_prompt_1100", gpt, embed, gs, es, [1100], 40)


def test_maps_several_hundred_steps_match_f64():
    gpt, embed, gs, es = build_gpt()
    _check_against_oracle("code_b2_400_steps", gpt, embed, gs, es, [30, 21], 400)


@pytest.mark.parametrize("case,text", [("audio_b3", False), ("text_b2", True)])
def test_reference_fixture(case, text):
    from gpu_util import load_gold

    gpt, embed, _, _ = build_gpt()
    g = load_gold("gpt_attn")
    lengths, steps = g[f"{case}_lengths"].tolist(), int(g[f"{case}_steps"])
    out = list(_run(gpt, embed, lengths, steps, pseed=int(g[f"{case}_prompt_seed"]),
                    sseed=int(g[f"{case}_sampler_seed"]), text=text)[2])[-1]
    for b in range(len(lengths)):
        n = int(g[f"{case}_n"][b])
        want = g[f"{case}_ids"][b, :n]
        assert np.array_equal(out.ids[b].cpu().numpy(), want[:, 0] if text else want)
    d = (pack_maps(out.attentions).cpu().double() - torch.from_numpy(g[f"{case}_maps"]).double()).abs().max().item()
    assert d < BAR, (case, d)


def test_two_runs_give_the_same_bits_and_stream_extends_one_list():
    gpt, embed, _, _ = build_gpt()
    a = pack_maps(list(_run(gpt, embed, [5, 23, 11], 70)[2])[-1].attentions)
    b = pack_maps(list(_run(gpt, embed, [5, 23, 11], 70)[2])[-1].attentions)
    assert torch.equal(a, b)
    lists, lens = [], []
    for o in _run(gpt, embed, [5, 23, 11], 70, stream=True, stream_batch=16)[2]:
        lists.append(o.attentions)
        lens.append(len(o.attentions))
    assert all(x is lists[0] for x in lists)
    assert lens[:-1] == [16, 32, 48, 64] and lens[-1] == 70
    s = pack_maps(lists[0])
    d = (s - a).abs().max().item()
    assert d < BAR, d


def test_interrupt_keeps_the_steps_done():
    gpt, embed, _, _ = build_gpt()
    from chattts_b200.gpt import GPT

    ctx = GPT.Context()
    outs = []
    for o in _run(gpt, embed, [12, 16], 200, stream=True, stream_batch=16, context=ctx)[2]:
        outs.append(len(o.attentions))
        ctx.set(True)
    assert len(outs) == 2 and outs[0] == 16 and outs[1] == 16


def test_abi_refusals():
    gpt, embed, _, _ = build_gpt()
    lib = _lib.load()
    h = gpt._handle
    emb, mask, gen = _run(gpt, embed, [12, 16], 8, attn=False)
    list(gen)
    m = mask.cuda().to(torch.uint8).contiguous()
    T0 = emb.shape[1]
    buf = torch.empty(1 << 20, device="cuda")
    e = torch.empty(2, T0 + 8, 768, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda B, T, q0, n: lib.ctb_gpt_attention_maps(h, B, T, q0, n, C.c_void_p(e.data_ptr()),  # noqa: E731
                                                          C.c_void_p(m.data_ptr()), C.c_void_p(buf.data_ptr()), s)
    ERR_ARG, ERR_STATE = -1, -3  # include/chattts_b200.h
    assert call(2, T0, 0, T0 + 7) == 0
    assert call(2, T0, 0, T0 + 8) == ERR_ARG      # past the columns fed
    assert call(2, T0, 3, 4) == ERR_ARG           # part of the prompt
    assert call(2, T0, 0, T0 - 1) == ERR_ARG
    assert call(3, T0, 0, T0) == ERR_ARG          # not the batch in flight
    assert call(2, T0, T0 + 2, 3) == 0
    torch.cuda.synchronize()
    from chattts_b200.engine import EngineDevice

    dev = EngineDevice(gpt, [], 2, 8)  # a slot engine now owns the handle
    assert call(2, T0, 0, T0) == ERR_STATE
    del dev
