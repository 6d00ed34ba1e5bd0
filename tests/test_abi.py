"""CPU checks of the C-ABI boundary: the library builds for sm_90a, loads, and exports every
symbol include/chattts_b200.h declares (no compute calls - there is no GPU here)."""
import ctypes
import os
import re

import pytest

from chattts_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_loads_abi_version_4():
    """Version 4 added ctb_gpt_step_kind and reads CTB_FLOW_NO_INK per handle."""
    path = build.build()
    assert os.path.exists(path)
    lib = _lib.load()
    assert lib.ctb_abi_version() == _lib.ABI_VERSION == 4


def test_every_declared_symbol_is_exported():
    hdr = open(os.path.join(ROOT, "include", "chattts_b200.h")).read()
    declared = set(re.findall(r"\b(ctb_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    lib = ctypes.CDLL(build.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name


def test_layout_query_matches_parameter_count():
    lib = _lib.load()
    cc = _lib.GptConfig(768, 3072, 20, 12, 12, 64, 4, 626, 21178, 4096, 1e-6, 8, 512)
    lay = _lib.GptLayout()
    assert lib.ctb_gpt_layout_query(ctypes.byref(cc), ctypes.byref(lay)) == 0
    per_layer = 4 * 768 * 768 + 3 * 768 * 3072 + 2 * 768
    assert lay.layer_stride == per_layer
    # SURVEY.md §8d: W = 190,698,240 streamed weight elements per audio step (layers + norms + 4 heads)
    assert per_layer * 20 + 768 + 4 * 626 * 768 == 190_698_240
    assert lay.total == per_layer * 20 + 768 + 2 * (4 * 626 + 21178) * 768 + 2 * 4096 * 64


def test_sampler_config_struct_size_matches_header():
    # 8 floats + float + 3 ints + 1 int + 32 floats + 5 ints + float + int (ABI v2) + pad + u64
    assert ctypes.sizeof(_lib.SamplerConfig) == 8 * 4 + 4 + 4 + 4 + 4 + 32 * 4 + 4 * 5 + 4 + 4 + 4 + 8


def test_graft_entry_build_runs_on_cpu():
    """The driver calls __graft_entry__.build() in the build container every round: it must compile, load and agree with
    the header's ABI version (a hard-coded version there went stale once)."""
    import importlib
    import sys

    sys.path.insert(0, ROOT)
    entry = importlib.import_module("__graft_entry__")
    entry.build()


def test_step_kind_constants_match_header_and_bad_arguments_are_refused():
    """ctb_gpt_step_kind: the binding's STEP_* values are the header's CTB_STEP_*, and a null handle is CTB_ERR_ARG
    (no device call: this runs without a GPU)."""
    hdr = open(os.path.join(ROOT, "include", "chattts_b200.h")).read()
    declared = {m[0]: int(m[1]) for m in re.findall(r"#define\s+CTB_STEP_([A-Z_]+)\s+(\d+)", hdr)}
    assert declared == {"FLOW_INK": _lib.STEP_FLOW_INK, "FLOW": _lib.STEP_FLOW, "MEGA": _lib.STEP_MEGA,
                        "FMA": _lib.STEP_FMA, "WGMMA": _lib.STEP_WGMMA}
    assert set(_lib.STEP_NAMES) == set(declared.values()) and min(declared.values()) > 0
    lib = _lib.load()
    assert lib.ctb_gpt_step_kind(None, 1, 0) == -1
    assert b"null" in lib.ctb_last_error()
    with pytest.raises(_lib.CtbError):
        _lib.step_kind(None, 1)
