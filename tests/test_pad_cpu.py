"""Padded batches without a GPU: the NumPy oracle against torch's padding, the layout of the padded gather replayed on
the host (tests/cpp/pad_layout_check.cpp), the encoding of pad_value, and the argument checks that run before the
store is touched."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import pad_oracle as po

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("max_rows", [0, 1, 5, 17, 40])
def test_oracle_matches_pad_sequence(max_rows):
    """slots of the oracle == torch's pad_sequence of the truncated requests, lengths == min(count, max_rows)"""
    rng = np.random.default_rng(max_rows)
    row = 3
    counts = rng.integers(0, 30, 50)
    counts[[0, 7]] = 0
    seqs = [rng.standard_normal((int(c), row)).astype(np.float32) for c in counts]
    packed = np.concatenate([s.reshape(-1) for s in seqs])
    got, lengths = po.pad_rows(packed, counts, row, max_rows, np.float32(-7.5))
    assert lengths.tolist() == np.minimum(counts, max_rows).tolist()
    trunc = [torch.from_numpy(s[:max_rows]) for s in seqs] + [torch.zeros(max_rows, row)]  # (fixes the padded length)
    exp = torch.nn.utils.rnn.pad_sequence(trunc, batch_first=True, padding_value=-7.5)[:-1]
    assert got.shape == (len(counts), max_rows, row)
    assert np.array_equal(got, exp.numpy())


def test_oracle_invalid_requests_and_bits():
    """an invalid request's slot is all padding with length 0; the pad element keeps its bits (a NaN payload)"""
    nan_bits = np.array([0x7FC01234], np.uint32).view(np.float32)[0]
    counts = np.array([2, 3, 1])
    valid = np.array([True, False, True])
    packed = np.arange(3 * 2, dtype=np.float32)  # requests 0 and 2 only: 2 + 1 rows of 2
    got, lengths = po.pad_rows(packed, counts, 2, 2, nan_bits, valid)
    assert lengths.tolist() == [2, 0, 1]
    bits = got.view(np.uint32)
    assert np.array_equal(got[0], [[0, 1], [2, 3]])
    assert (bits[1] == 0x7FC01234).all()
    assert np.array_equal(got[2, 0], [4, 5]) and (bits[2, 1] == 0x7FC01234).all()


def test_layout_check():
    """compile tests/cpp/pad_layout_check.cpp (which includes the kernels' layout functions) and run it: every output
    byte of many padded shapes -- one above 4 GiB -- is written exactly once"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "pad_layout_check")
        subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "ddstore_b200", "csrc"),
                        "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pad_layout_check.cpp"),
                        "-o", exe], check=True, capture_output=True, text=True)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "pad layout ok" in r.stdout


def test_pad_value_encoding():
    from ddstore_b200.store import _pad_bits
    assert _pad_bits(0, torch.float32) == 0
    assert _pad_bits(-100, torch.int32) == 0xFFFFFF9C
    assert _pad_bits(-1, torch.int64) == (1 << 64) - 1
    assert _pad_bits(255, torch.uint8) == 0xFF
    assert _pad_bits(float("-inf"), torch.bfloat16) == 0xFF80
    assert _pad_bits(1.0, torch.float16) == 0x3C00
    assert _pad_bits(-2.5, torch.float64) == int(np.array([-2.5]).view(np.uint64)[0])
    assert _pad_bits(True, torch.bool) == 1
    nan = torch.tensor([0x7FC01234], dtype=torch.int32).view(torch.float32)
    assert _pad_bits(nan, torch.float32) == 0x7FC01234  # a one-element tensor: its bits, verbatim
    assert _pad_bits(torch.tensor(-3, dtype=torch.int16), torch.int16) == 0xFFFD
    for value, dt in [(256, torch.uint8), (-1, torch.uint8), (2**31, torch.int32), (1.5, torch.int32),
                      (1e39, torch.float32), (70000.0, torch.float16), (1e39, torch.bfloat16), (2, torch.bool)]:
        with pytest.raises(ValueError):
            _pad_bits(value, dt)
    with pytest.raises(ValueError, match="one-element"):
        _pad_bits(torch.zeros(2), torch.float32)
    with pytest.raises(ValueError, match="one-element"):
        _pad_bits(torch.zeros(1, dtype=torch.float64), torch.float32)


def test_python_argument_errors():
    from ddstore_b200 import PyDDStore
    bare = object.__new__(PyDDStore)  # (the checks run before the store is touched)
    with pytest.raises(ValueError, match="needs counts"):
        bare.get_batch("x", [0], out=torch.empty(4), pad_rows=3)
    with pytest.raises(ValueError, match="neither"):
        bare.get_batch("x", [0], [1], out=torch.empty(4), pad_rows=3, count=2)
    with pytest.raises(ValueError, match="no `offsets`"):
        bare.get_samples("x", [0], torch.empty(4), offsets=torch.empty(2, dtype=torch.int64), pad_rows=3)


def test_c_entries_check_their_store_first():
    from ddstore_b200 import _capi
    L = _capi.lib()
    pad = _capi.Pad(4, 0, None)
    t, b = ctypes.c_int64(5), ctypes.c_int64(5)
    assert L.dds_get_batch_padded(None, b"x", None, None, 0, 4, None, ctypes.byref(pad), None, 0, 2, None,
                                  ctypes.byref(t), ctypes.byref(b)) == _capi.ERR_ARG
    assert (t.value, b.value) == (0, -1)
    assert L.dds_get_samples_padded(None, b"x", None, 0, 4, None, ctypes.byref(pad), None, 0, 2, None, None,
                                    None) == _capi.ERR_ARG


def test_pad_struct_matches_the_header():
    """the ctypes dds_pad_t has the header's fields, in order, and the padded entries are declared"""
    from ddstore_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "ddstore_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} dds_pad_t;", hdr).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*;", body)
    assert fields == [f for f, _ in _capi.Pad._fields_] == ["max_rows", "pad_bits", "lengths"]
    assert "dds_get_batch_padded" in _capi.SIGNATURES and "dds_get_samples_padded" in _capi.SIGNATURES
