"""``GPT.generate(return_attn=True)``'s host loop without a GPU: a stand-in library plays the device (steps, finish,
ctb_gpt_attention_maps filling each step's block with the number of the attempt that made it), so the list's length,
its per-step tuples, in-place growth under ``stream=True``, the regenerate that discards a failed attempt's maps and
an interrupt's prefix are checked on the CPU."""
import contextlib
import ctypes as C
import types

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200 import gpt as gpt_mod
from chattts_b200.config import Config

L, H = 20, 12


class FakeLib:
    def __init__(self, finish_at, first_step_eos_attempts=0):
        self.finish_at, self.first_eos = finish_at, first_step_eos_attempts
        self.attempt, self.map_calls = 0, []

    def ctb_gpt_begin(self, h, B, T0, emb, mask, cfg, q, max_new, text, ids_out, hid_out, stream):
        self.attempt += 1
        self.B, self.T0, self.max_new, self.steps = B, T0, max_new, 1
        return 0

    def ctb_gpt_decode(self, h, n, stream):
        self.steps = min(self.steps + n, self.max_new, self.finish_at + 1)
        return 0

    def ctb_gpt_status_query(self, h, st_ref, end_ptr, fin_ptr, stream):
        st = st_ref._obj
        first = self.attempt <= self.first_eos
        st.steps_done, st.any_finished_first_step = self.steps, int(first)
        st.all_finished = int(first or self.steps > self.finish_at)
        end = np.ctypeslib.as_array((C.c_int32 * self.B).from_address(end_ptr.value))
        fin = np.ctypeslib.as_array((C.c_uint8 * self.B).from_address(fin_ptr.value))
        end[:] = 0 if first else min(self.steps, self.finish_at)
        fin[:] = st.all_finished
        return 0

    def ctb_gpt_embed_prompt(self, h, ids, tm, B, T, out, stream):
        return 0

    def ctb_gpt_attention_maps(self, h, B, T0, q0, n, emb, mask, out, stream):
        assert (B, T0) == (self.B, self.T0) and q0 + n <= T0 + self.steps - 1
        i0, i1 = (0 if q0 == 0 else q0 - T0 + 1), q0 + n - T0 + 1
        floats = L * B * H * sum(T0 * T0 if i == 0 else T0 + i for i in range(i0, i1))
        np.ctypeslib.as_array((C.c_float * floats).from_address(out.value))[:] = self.attempt
        self.map_calls.append((q0, n))
        return 0


@pytest.fixture
def fake(monkeypatch):
    def make(**kw):
        lib = FakeLib(**kw)
        monkeypatch.setattr(_lib, "load", lambda *a, **k: lib)
        monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
        monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
        g = gpt_mod.GPT(Config().gpt, embed=None, device="cpu", device_gpt="cpu")
        g._handle = C.c_void_p(1)
        made.append(g)
        return g, lib

    made = []
    yield make
    for g in made:
        g._handle = C.c_void_p()  # never handed to the real library


def _gen(g, T0=6, B=2, max_new=50, **kw):
    emb = torch.zeros(B, T0, 768)
    ids = torch.zeros(B, T0, 4, dtype=torch.long)
    mask = torch.ones(B, T0, dtype=torch.bool)
    mask[0, :2] = False
    return g.generate(emb, ids, torch.tensor([0.3] * 4), 625, attention_mask=mask, max_new_token=max_new,
                      show_tqdm=False, return_attn=True, **kw)


def test_one_entry_per_step_with_the_reference_shapes(fake):
    g, lib = fake(finish_at=30)
    outs = list(_gen(g, manual_seed=1))
    assert len(outs) == 1
    att = outs[0].attentions
    assert len(att) == 31 and len(lib.map_calls) == 1  # a non-stream run computes the whole sequence once
    assert all(isinstance(a, tuple) and len(a) == L for a in att)
    assert tuple(att[0][0].shape) == (2, H, 6, 6)
    assert [tuple(a[7].shape) for a in att[1:4]] == [(2, H, 1, 7), (2, H, 1, 8), (2, H, 1, 9)]


def test_stream_extends_one_list_in_place(fake):
    g, lib = fake(finish_at=200)
    seen, firsts = [], []
    for o in _gen(g, max_new=60, stream=True, stream_batch=16, manual_seed=1):
        seen.append((o.attentions, len(o.attentions)))
        firsts.append(o.attentions[0][0])
    assert all(a is seen[0][0] for a, _ in seen)
    assert [n for _, n in seen] == [16, 32, 48, 60]
    assert all(f is firsts[0] for f in firsts)  # earlier entries are kept, not recomputed
    assert lib.map_calls == [(0, 6 + 15), (6 + 15, 16), (6 + 31, 16), (6 + 47, 12)]


def test_regenerate_discards_the_failed_attempt(fake):
    g, lib = fake(finish_at=20, first_step_eos_attempts=1)
    outs = list(_gen(g))  # unseeded, ensure_non_empty: the first attempt ends at step 0 and runs again
    assert lib.attempt == 2 and len(outs) == 1
    att = outs[0].attentions
    assert len(att) == 21
    assert all(bool((t == 2).all()) for a in att for t in a)


def test_interrupt_keeps_the_steps_done(fake):
    g, lib = fake(finish_at=200)
    ctx = gpt_mod.GPT.Context()
    lens = []
    for o in _gen(g, max_new=100, stream=True, stream_batch=16, manual_seed=1, context=ctx):
        lens.append(len(o.attentions))
        ctx.set(True)
    assert lens == [16, 16]


def test_default_makes_no_map_call(fake):
    g, lib = fake(finish_at=10)
    emb, ids = torch.zeros(1, 6, 768), torch.zeros(1, 6, 4, dtype=torch.long)
    out = list(g.generate(emb, ids, torch.tensor([0.3] * 4), 625, max_new_token=20, show_tqdm=False, manual_seed=1))
    assert out[-1].attentions == [] and lib.map_calls == []
