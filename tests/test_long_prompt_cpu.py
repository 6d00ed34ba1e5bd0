"""Prompts over 1,024 tokens on the slot engine, host side: how an admission is split into prefills
(``engine.admission_groups``), the prompt limit of ``GPT._engine_args`` and ``admission_chunks``."""
import ctypes as C
import random

import pytest
import torch

from chattts_b200.engine import (ADMIT_MAX_ROWS, LONG_PROMPT_COLS, MIN_PROMPT_COLS, Request, admission_chunks,
                                 admission_groups)
from chattts_b200.gpt import GPT


def _req(T, max_new=8):
    return Request(emb=torch.zeros(T, 4), temperature=[0.3], eos_token=625, max_new_token=max_new)


def _short_rule(group, requests, max_context):
    """How an admission of prompts of at most 1,024 tokens was split before long prompts were admitted."""
    T0 = max(MIN_PROMPT_COLS, max(int(requests[i].emb.shape[0]) for _, i in group))
    alone = [(s, i) for s, i in group if T0 + requests[i].max_new_token > max_context]
    rest = [p for p in group if p not in alone]
    return [c for part in ([rest] if rest else []) + [[p] for p in alone] for c in admission_chunks(part, T0)]


def _prefills(group, requests, max_context):
    return [c for part, T0 in admission_groups(group, requests, max_context) for c in admission_chunks(part, T0)]


def test_short_admissions_split_as_before():
    rnd = random.Random(3)
    for trial in range(200):
        n = rnd.randint(1, 64)
        reqs = [_req(rnd.choice([1, 8, 40, 300, 512, 1000, 1024]), rnd.choice([8, 100, 1000, 3000, 3072]))
                for _ in range(n)]
        group = [(s, i) for s, i in enumerate(rnd.sample(range(n), n))]
        assert _prefills(group, reqs, 4096) == _short_rule(group, reqs, 4096), trial


def test_long_prompts_are_prefilled_alone_after_the_short_ones():
    reqs = [_req(3000, 80)] + [_req(T, 40) for T in (8, 40, 1024, 300)] + [_req(1025, 8), _req(4000, 96)]
    group = [(s, i) for s, i in enumerate(range(len(reqs)))]
    got = admission_groups(group, reqs, 4096)
    assert got == [([(1, 1), (2, 2), (3, 3), (4, 4)], 1024), ([(0, 0)], 3000), ([(5, 5)], 1025), ([(6, 6)], 4000)]
    # without the long prompts the short ones are one prefill of the same width
    assert admission_groups(group[1:5], reqs, 4096) == [(group[1:5], 1024)]
    # only long prompts: one prefill each
    assert admission_groups([(0, 5), (1, 0)], reqs, 4096) == [([(0, 5)], 1025), ([(1, 0)], 3000)]
    assert LONG_PROMPT_COLS == 1024


def test_a_short_prompt_that_no_longer_fits_next_to_the_width_is_still_admitted_alone():
    reqs = [_req(1000, 8), _req(20, 3100), _req(1100, 8)]
    got = admission_groups([(0, 0), (1, 1), (2, 2)], reqs, 4096)
    assert got == [([(0, 0)], 1000), ([(1, 1)], 1000), ([(2, 2)], 1100)]


@pytest.fixture
def gpt():
    g = GPT({"hidden_size": 4}, embed=None, device_gpt=torch.device("cpu"), max_batch=4, max_context=4096)
    g._handle = C.c_void_p(1)  # never reaches the library
    yield g
    g._handle = C.c_void_p()  # nothing for the destructor to free


@pytest.mark.parametrize("T,max_new", [(1025, 8), (2000, 2000), (3000, 1096), (4095, 1), (1024, 3072)])
def test_engine_args_accept_prompts_up_to_max_context(gpt, T, max_new):
    *_, check = gpt._engine_args("t", [_req(T, max_new)], 2, False, False, None, None, None)
    check(_req(T, max_new))


@pytest.mark.parametrize("T,max_new", [(3000, 1097), (4096, 1), (4095, 2), (1024, 3073)])
def test_engine_args_reject_prompt_plus_max_new_over_max_context(gpt, T, max_new):
    with pytest.raises(ValueError, match=r"max_context=4096") as e:
        gpt._engine_args("t", [_req(T, max_new)], 2, False, False, None, None, None)
    assert "up to 1024" not in str(e.value)


def test_admission_chunks_unchanged():
    group = list(range(64))
    assert admission_chunks(group, 1024) == [group[:32], group[32:]]
    assert admission_chunks(group[:1], 4000) == [group[:1]]
    assert admission_chunks(group, 8) == [group]
    assert ADMIT_MAX_ROWS == 32 * 1024
