"""``GPT.score``'s host side without a GPU: a stand-in library plays ``ctb_gpt_embed_prompt`` (each position's
embedding holds its first id + 1000) and ``ctb_gpt_score`` (records every call and writes each entry's target id + 0.5
as its log-probability), so the grouping of rows into calls, the columns and padding each call gets, the argument
refusals and the order and shapes of the outputs are checked on the CPU."""
import contextlib
import ctypes as C
import types

import numpy as np
import pytest
import torch

from chattts_b200 import _lib
from chattts_b200 import gpt as gpt_mod
from chattts_b200.config import Config
from chattts_b200.engine import ADMIT_MAX_ROWS, LONG_PROMPT_COLS, MIN_PROMPT_COLS

D, NVQ = 768, 4


class FakeLib:
    def __init__(self):
        self.calls = []

    def ctb_gpt_embed_prompt(self, h, ids, tm, B, T, out, stream):
        i = np.ctypeslib.as_array((C.c_int64 * (B * T * NVQ)).from_address(ids.value)).reshape(B, T, NVQ)
        o = np.ctypeslib.as_array((C.c_float * (B * T * D)).from_address(out.value)).reshape(B, T, D)
        o[:] = i[:, :, :1] + 1000
        return 0

    def ctb_gpt_score(self, h, B, T, emb, n_prompt, n_given, targets, text, out, stream):
        P, n = list(n_prompt), list(n_given)
        m, rpi = sum(n), 1 if text else NVQ
        e = np.ctypeslib.as_array((C.c_float * (B * T * D)).from_address(emb.value)).reshape(B, T, D).copy()
        t = np.ctypeslib.as_array((C.c_int32 * (m * rpi)).from_address(targets.value)).copy()
        np.ctypeslib.as_array((C.c_float * (m * rpi)).from_address(out.value))[:] = t + 0.5
        self.calls.append(dict(B=B, T=T, P=P, n=n, emb=e, text=text))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda *a, **k: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    g = gpt_mod.GPT(Config().gpt, embed=None, device="cpu", device_gpt="cpu", max_batch=8, max_context=2560)
    g._handle = C.c_void_p(1)
    yield g, lib
    g._handle = C.c_void_p()


def _prompt(P, tag):
    return torch.full((P, D), float(tag))


def _codes(n, seed):
    return torch.randint(0, 626, (n, NVQ), generator=torch.Generator().manual_seed(seed))


def test_groups_bound_pairs_rows_and_long_rows_alone():
    widths = [5, 300, 1024, 1025, 40, 3000] + [900] * 40
    groups = gpt_mod.score_groups(widths, max_batch=32)
    seen = sorted(i for g, _ in groups for i in g)
    assert seen == list(range(len(widths)))
    for rows, T in groups:
        assert len(rows) <= 32 and len(rows) * T <= ADMIT_MAX_ROWS or len(rows) == 1
        assert all(widths[i] <= T for i in rows)
        if any(widths[i] > LONG_PROMPT_COLS for i in rows):
            assert len(rows) == 1 and T == widths[rows[0]]
        else:
            assert T == max(MIN_PROMPT_COLS, max(w for w in widths if w <= LONG_PROMPT_COLS))
    assert [g for g, _ in groups[-2:]] == [[3], [5]]  # long rows last, in order
    assert gpt_mod.score_groups([3], 8) == [([0], MIN_PROMPT_COLS)]


def test_columns_padding_and_outputs(fake):
    g, lib = fake
    Ps, ns = [3, 20, 7, 1100], [4, 1, 9, 6]
    codes = [_codes(n, i) for i, n in enumerate(ns)]
    out = g.score([_prompt(P, 10 + i) for i, P in enumerate(Ps)], codes)
    assert [c["B"] for c in lib.calls] == [3, 1] and [c["T"] for c in lib.calls] == [20, 1105]
    assert lib.calls[0]["P"] == Ps[:3] and lib.calls[0]["n"] == ns[:3]
    rows = [(0, 0), (0, 1), (0, 2), (1, 0)]  # (call, row) of each input
    for i, (k, b) in enumerate(rows):
        e, T, w = lib.calls[k]["emb"][b], lib.calls[k]["T"], Ps[i] + ns[i] - 1
        c0 = T - w
        assert (e[:c0] == 0).all()
        assert (e[c0: c0 + Ps[i]] == 10 + i).all()
        assert np.array_equal(e[c0 + Ps[i]:, 0], codes[i][:-1, 0].numpy() + 1000)
        assert out[i].shape == (ns[i], NVQ) and out[i].dtype == torch.float32
        assert torch.equal(out[i], codes[i].float() + 0.5)


def test_text_rows_and_empty_rows(fake):
    g, lib = fake
    t = [torch.tensor([5, 9, 21177]), torch.zeros(0, dtype=torch.long), torch.tensor([7])]
    out = g.score([_prompt(4, 1), _prompt(6, 2), _prompt(9, 3)], t, infer_text=True)
    assert [tuple(o.shape) for o in out] == [(3,), (0,), (1,)]
    assert torch.equal(out[0], t[0].float() + 0.5) and torch.equal(out[2], t[2].float() + 0.5)
    (call,) = lib.calls
    assert call["text"] == 1 and call["P"] == [4, 9] and call["n"] == [3, 1]
    e = call["emb"][0]
    assert np.array_equal(e[-2:, 0], np.array([1005, 1009], np.float32))
    assert g.score([_prompt(4, 1)], [torch.zeros(0, NVQ, dtype=torch.long)])[0].shape == (0, NVQ)
    assert len(lib.calls) == 1  # no call for rows with nothing to score


def test_refusals(fake):
    g, lib = fake
    with pytest.raises(ValueError, match="outside"):
        g.score([_prompt(4, 0)], [torch.tensor([[0, 1, 2, 626]])])
    with pytest.raises(ValueError, match="outside"):
        g.score([_prompt(4, 0)], [torch.tensor([-1])], infer_text=True)
    with pytest.raises(ValueError, match="max_context"):
        g.score([_prompt(2000, 0)], [_codes(562, 0)])
    g.score([_prompt(2000, 0)], [_codes(561, 0)])  # 2000 + 561 - 1 = max_context
    with pytest.raises(ValueError, match="shape"):
        g.score([_prompt(4, 0)], [torch.tensor([1, 2])])
    with pytest.raises(ValueError, match="shape"):
        g.score([torch.zeros(0, D)], [_codes(1, 0)])
    with pytest.raises(ValueError, match="prompts"):
        g.score([_prompt(4, 0)], [])
    g._open = object()
    with pytest.raises(RuntimeError, match="open engine"):
        g.score([_prompt(4, 0)], [_codes(1, 0)])
    g._open = None
    assert len(lib.calls) == 1
