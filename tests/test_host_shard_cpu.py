"""CPU-only checks of the placement surface: the C-ABI declares and exports the three placement entries with the
signatures the ctypes binding applies, the Python layers refuse an unknown placement before any call reaches the
library, and the public header still compiles as C99 with the new declarations in use."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from ddstore_b200 import _capi
from ddstore_b200.store import PyDDStore

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    return open(os.path.join(ROOT, "include", "ddstore_b200.h")).read()


def test_placement_constants_match_the_header():
    src = _header()
    assert re.search(r"#define DDS_PLACE_HBM 0\b", src) and re.search(r"#define DDS_PLACE_HOST 1\b", src)
    assert _capi.PLACEMENTS == {"hbm": _capi.PLACE_HBM, "host": _capi.PLACE_HOST}
    assert (_capi.PLACE_HBM, _capi.PLACE_HOST) == (0, 1)


@pytest.mark.parametrize("name,args", [
    ("dds_add_placed", [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]),
    ("dds_init_placed", [C.c_void_p, C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int]),
    ("dds_query_placement", [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]),
    ("dds_host_gather_ctas", []),
])
def test_capi_declares_the_placement_entries(name, args):
    res, got = _capi.SIGNATURES[name]
    assert res is C.c_int and got == args
    fn = getattr(_capi.lib(), name)  # exported by the library
    assert fn.restype is C.c_int
    # the header declares it with as many parameters as the binding passes
    src = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", src)
    assert m, name
    params = [p for p in m.group(1).split(",") if p.strip() and p.strip() != "void"]
    assert len(params) == len(args)


def test_varinfo_layout_is_unchanged():
    assert C.sizeof(_capi.VarInfo) == 4 * 4 + 8 * 2 + 8 * 64 + 8
    assert [f[0] for f in _capi.VarInfo._fields_] == ["itemsize", "disp", "nranks", "fence_active", "local_nrows",
                                                     "total_nrows", "lenlist", "local_base"]


class _Recorder:
    """stands in for the loaded library: records every call"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append(name)
            return 0
        return fn


@pytest.mark.parametrize("placement", ["HOST", "dram", "", None, 1])
def test_python_refuses_unknown_placement_before_any_call(placement):
    store = PyDDStore.__new__(PyDDStore)
    store._L, store._h = _Recorder(), C.c_void_p(1)
    with pytest.raises(ValueError, match="placement"):
        store.add("x", np.zeros((4, 3), np.float32), placement=placement)
    with pytest.raises(ValueError, match="placement"):
        store.init("x", 4, 3, 4, placement=placement)
    assert store._L.calls == []
    store._h = None  # (nothing to close)


def test_python_passes_known_placements_through():
    store = PyDDStore.__new__(PyDDStore)
    rec = _Recorder()
    seen = []
    rec.dds_add_placed = lambda *a: seen.append(("add", a[-1])) or 0
    rec.dds_init_placed = lambda *a: seen.append(("init", a[-1])) or 0
    store._L, store._h = rec, C.c_void_p(1)
    store.add("x", np.zeros((4, 3), np.float32))
    store.add("y", np.zeros((4, 3), np.float32), placement="host")
    store.init("z", 4, 3, 4, placement="host")
    store.init("w", 4, 3, 4)
    assert seen == [("add", 0), ("add", 1), ("init", 1), ("init", 0)]
    store._h = None


def test_public_header_with_placement_is_plain_c(tmp_path):
    src = tmp_path / "use_placement.c"
    src.write_text('#include "ddstore_b200.h"\n'
                   "int main(void) {\n"
                   "    int p = DDS_PLACE_HOST;\n"
                   "    int (*a)(dds_store_t *, const char *, const void *, int64_t, int, int, int, int) = dds_add_placed;\n"
                   "    int (*i)(dds_store_t *, const char *, int64_t, int, int, int) = dds_init_placed;\n"
                   "    int (*q)(dds_store_t *, const char *, int *) = dds_query_placement;\n"
                   "    (void)a; (void)i; (void)q;\n"
                   "    return p == DDS_PLACE_HBM ? 1 : DDS_OK;\n"
                   "}\n")
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                        str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
