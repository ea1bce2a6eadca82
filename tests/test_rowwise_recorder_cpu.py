"""The argument maps of the production row-wise replay (tests/test_production_rowwise_gpu.py) against the C ABI: the
kinds against _lib._SIGS and the names against the declarations in include/pnx.h.  An entry point whose arguments
move, appear, disappear or trade places fails here, without a GPU."""
import ctypes
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_production_rowwise_gpu as R  # noqa: E402
from pillarnext_b200 import _lib  # noqa: E402

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pnx.h")
KINDS = {"P": ctypes.c_void_p, "I": ctypes.c_int, "L": ctypes.c_longlong, "F": ctypes.c_float, "D": ctypes.c_double}


@pytest.mark.parametrize("name", sorted(R.ARG_MAPS))
def test_argument_map_matches_the_abi(name):
    spec = R.arg_map(name)
    assert name in _lib._SIGS, name
    assert [KINDS[k] for _, k in spec] == _lib._SIGS[name], name
    names = [a for a, _ in spec]
    assert len(set(names)) == len(names) and names[-1] == "stream", names


def _declared_names(name):
    """Parameter names of `int name(...);` in include/pnx.h (comments removed)."""
    with open(HEADER) as f:
        text = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % re.escape(name), text)
    assert m, "%s is not declared in include/pnx.h" % name
    return [re.findall(r"\w+", p)[-1] for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", sorted(R.ARG_MAPS))
def test_argument_names_match_the_header(name):
    assert [a for a, _ in R.arg_map(name)] == _declared_names(name)


def test_covered_and_excluded_entry_points_exist():
    for name in set(R.GEMM_REPLAYED) | set(R.EXCLUDED):
        assert name in _lib._SIGS, name
    assert not (set(R.ARG_MAPS) & set(R.EXCLUDED)) and not (set(R.GEMM_REPLAYED) & set(R.EXCLUDED))


def test_recorder_keeps_scalars_and_null_flags_once_per_configuration():
    calls = []

    class FakeLib:
        def pnx_add_relu(self, *a):
            calls.append(a)
            return 0

        def pnx_pfn_mean(self, *a):
            return 0

    rec = R.Recorder(FakeLib())
    rec.source = "unit"
    lib = rec.proxy()
    for _ in range(3):
        assert lib.pnx_add_relu(1000, 64, 2000, 128, 77, 64, None, 64, 5) == 0
    lib.pnx_add_relu(1000, 64, 2000, 128, 78, 64, 3000, 64, 5)
    lib.pnx_pfn_mean(1, 2)
    assert len(calls) == 4 and rec.called == {"pnx_add_relu", "pnx_pfn_mean"}
    assert len(rec.configs) == 2
    c = rec.configs[0]
    assert (c["fn"], c["M"], c["C"], c["lda"], c["ldb"], c["ldy"], c["calls"], c["source"]) == \
        ("pnx_add_relu", 77, 64, 64, 128, 64, 3, "unit")
    assert c["a"] is True and c["y"] is False and "stream" not in c
    assert rec.configs[1]["y"] is True and rec.configs[1]["calls"] == 1
