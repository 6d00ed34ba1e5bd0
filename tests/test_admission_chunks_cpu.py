"""Admissions larger than ``ADMIT_MAX_ROWS`` prompt rows run as consecutive prefills (``engine.admission_chunks``); an
admission a 32-slot engine can make (32 prompts of up to 1,024 tokens) stays one prefill."""
from chattts_b200.engine import ADMIT_MAX_ROWS, admission_chunks


def test_admission_of_32_slots_is_one_prefill():
    group = list(range(32))
    for T0 in (8, 40, 512, 1024):
        assert admission_chunks(group, T0) == [group]


def test_64_long_prompts_run_as_two_prefills_of_bounded_rows():
    group = [(s, 100 + s) for s in range(64)]
    chunks = admission_chunks(group, 1024)
    assert chunks == [group[:32], group[32:]]
    assert all(len(c) * 1024 <= ADMIT_MAX_ROWS for c in chunks)
    assert admission_chunks(group, 40) == [group]  # short prompts: 64 x 40 rows fit one prefill
    assert [len(c) for c in admission_chunks(group, 600)] == [54, 10]
