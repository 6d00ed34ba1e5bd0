"""CPU checks of the C-ABI boundary: the library builds for sm_90a, loads, and exports every
symbol include/chattts_b200.h declares (no compute calls - there is no GPU here)."""
import ctypes
import os
import re

from chattts_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_loads():
    path = build.build()
    assert os.path.exists(path)
    lib = _lib.load()
    assert lib.ctb_abi_version() == 3


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
