"""Converting batches without a GPU: the NumPy oracle of the element rules against torch's CPU casts, the byte and
offset arithmetic of converted packing, the Python-side argument checks and the C-ABI's device-free error paths."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import convert_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f32_classes():
    """float32 bit patterns of every non-NaN class: zeros, subnormals, normals, bf16 / f16 rounding ties both ways,
    values that round up into the next binade, overflow to inf, inf, and random bits"""
    rng = np.random.default_rng(7)
    edge = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x3F800000, 0xBF800000,
            0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x3F808000, 0x3F818000, 0x3F80FFFF, 0x3F7FFFFF, 0x7F7F8000,
            0x7F7F7FFF, 0x477FF000, 0x477FEFFF, 0x47800000, 0x387FC000, 0x33800000, 0x33000000, 0x33000001, 0x38800000]
    # every tie and near-tie of the bf16 rounding in a few binades, and of the f16 rounding
    hi = rng.integers(0, 1 << 16, 4096, dtype=np.uint32) << 16
    ties = np.concatenate([hi | 0x8000, hi | 0x7FFF, hi | 0x8001, (hi & ~np.uint32(1 << 16)) | 0x8000])
    f16t = (rng.integers(0x33000000 >> 13, 0x47800000 >> 13, 4096, dtype=np.uint32) << 13) | 0x1000
    bits = np.concatenate([np.array(edge, np.uint32), ties.astype(np.uint32), f16t, rng.integers(0, 1 << 32, 1 << 16, dtype=np.uint32)])
    f = bits.view(np.float32)
    return bits[~np.isnan(f)]


def test_bf16_integer_rounding_matches_torch_cpu_cast():
    bits = _f32_classes()
    exp = torch.from_numpy(bits.view(np.float32).copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    got = co.f32_to_bf16_bits(bits)
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, f"{bad.size} mismatches, first {bits[bad[0]]:#010x}: {got[bad[0]]:#06x} != {exp[bad[0]]:#06x}"
    # and NaN stays NaN, quiet
    nan = co.f32_to_bf16_bits(np.array([0x7FC00000, 0x7F800001, 0xFFFFFFFF], np.uint32))
    assert all((b & 0x7F80) == 0x7F80 and (b & 0x7F) for b in nan)


def test_f16_rule_matches_torch_cpu_cast():
    bits = _f32_classes()
    exp = torch.from_numpy(bits.view(np.float32).copy()).to(torch.float16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(co.f32_to_f16_bits(bits), exp)
    f = co.f32_to_f16_bits(np.array([0x7F7FFFFF, 0x477FF000, 0x33800000], np.uint32))  # overflow, overflow, subnormal
    assert f.tolist() == [0x7C00, 0x7C00, 0x0001]


def test_f64_rule_matches_torch_cpu_cast():
    rng = np.random.default_rng(3)
    bits = np.concatenate([rng.integers(0, 1 << 63, 1 << 15, dtype=np.uint64) * 2 + rng.integers(0, 2, 1 << 15, dtype=np.uint64),
                           np.array([0, 1 << 63, 1, 0x36A0000000000000, 0x47EFFFFFF0000000, 0x47EFFFFFE0000000,
                                     0x3FF0000010000000, 0x3FF0000030000000, 0x7FF0000000000000], np.uint64)])
    bits = bits[~np.isnan(bits.view(np.float64))]
    exp = torch.from_numpy(bits.view(np.float64).copy()).to(torch.float32).numpy().view(np.uint32)
    assert np.array_equal(co.f64_to_f32_bits(bits), exp)


def test_f64_edge_patterns_match_torch_cpu_cast():
    """the f64 -> f32 rounding edges the converting sweep stores in its float64 variables: the oracle's rule is torch's
    CPU cast on every one, and the edges land where their names say"""
    bits = co.f64_edge_bits()
    f = bits.view(np.float64)
    got = co.f64_to_f32_bits(bits)
    nan = np.isnan(f)
    exp = torch.from_numpy(f.copy()).to(torch.float32).numpy().view(np.uint32)
    bad = np.flatnonzero(~nan & (got != exp))
    assert bad.size == 0, f"{bits[bad[0]]:#018x}: oracle {got[bad[0]]:#010x}, torch {exp[bad[0]]:#010x}"
    # NaN stays NaN, also when its payload lies only in the 29 bits the cast drops (a truncation would give inf)
    assert nan.sum() == 8 and (np.isnan(got[nan].view(np.float32))).all() and (np.isnan(exp[nan].view(np.float32))).all()
    want = {0x3FF0000010000000: 0x3F800000, 0x3FF0000030000000: 0x3F800002, 0x3FF000000FFFFFFF: 0x3F800000,
            0x3FF0000010000001: 0x3F800001, 0x4123456790000000: 0x491A2B3C, 0x4123456770000000: 0x491A2B3C,
            0x47EFFFFFEFFFFFFF: 0x7F7FFFFF, 0x47EFFFFFF0000000: 0x7F800000, 0x380FFFFFC0000000: 0x007FFFFF,
            0x380FFFFFE0000000: 0x00800000, 0x380FFFFFDFFFFFFF: 0x007FFFFF, 0x36A0000000000000: 0x00000001, 0x36A8000000000000: 0x00000002,
            0x3690000000000000: 0x00000000, 0x3690000000000001: 0x00000001, 0x36B4000000000000: 0x00000002,
            0x0000000000000001: 0x00000000, 0x800FFFFFFFFFFFFF: 0x80000000, 0xB690000000000000: 0x80000000,
            0xFFF0000000000000: 0xFF800000}
    lut = dict(zip(bits.tolist(), got.tolist()))
    assert {k: lut[k] for k in want} == want


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_table_rules(out_dtype):
    from ddstore_b200.store import _conversion
    src = np.arange(256, dtype=np.uint8)
    x = torch.from_numpy(src)
    norm = ((x.float() - 127.5) * (1 / 58.4)).to(out_dtype)  # any torch expression: the table is bit-exact with it
    for table in (None, norm):
        cv, host = _conversion(torch.uint8, out_dtype, table)
        code = co.CVT_U8_LUT32 if out_dtype == torch.float32 else co.CVT_U8_LUT16
        assert cv.code == code and cv.lut == host.ctypes.data
        want = (x.to(out_dtype) if table is None else norm).contiguous().view(torch.uint8).numpy()
        rng = np.random.default_rng(1)
        row = rng.integers(0, 256, 3000, dtype=np.uint8)
        got = co.convert_bytes(row, code, host)
        assert np.array_equal(got, want.reshape(256, -1)[row].reshape(-1))


def test_converted_packing_arithmetic():
    # request i sits at sum_{j<i} count_j * disp * out_itemsize; capacity is whole output elements
    rng = np.random.default_rng(5)
    for code, (i_sz, o_sz) in co.SIZES.items():
        disp = 7
        counts = rng.integers(0, 9, 50)
        src_offs = np.concatenate([[0], np.cumsum(counts * disp * i_sz)])
        _, out_offs = co.convert_packed(np.zeros(int(src_offs[-1]), np.uint8), src_offs, code,
                                        np.zeros(256 * 4, np.uint8))
        assert out_offs.tolist() == np.concatenate([[0], np.cumsum(counts * disp * o_sz)]).tolist()
        total = int(out_offs[-1])
        assert co.cap_to_src(total, code) == src_offs[-1]            # fits exactly
        assert co.cap_to_src(total - 1, code) < src_offs[-1]         # one byte short: does not fit
        assert co.cap_to_src(total + o_sz - 1, code) == src_offs[-1]  # a partial element adds nothing


def test_python_conversion_arguments():
    from ddstore_b200.store import _Buf, _conversion
    assert _conversion(torch.float32, torch.bfloat16, None)[0].code == co.CVT_F32_BF16
    assert _conversion(np.float32, torch.float16, None)[0].code == co.CVT_F32_F16
    assert _conversion("float64", torch.float32, None)[0].code == co.CVT_F64_F32
    for bad in [(torch.float32, torch.float64), (torch.int64, torch.int32), (torch.float16, torch.float32),
                (torch.uint8, torch.int32), (torch.float32, torch.float32)]:
        with pytest.raises(ValueError):
            _conversion(bad[0], bad[1], None)
    with pytest.raises(ValueError):  # a table only for uint8 sources
        _conversion(torch.float32, torch.bfloat16, torch.zeros(256, dtype=torch.bfloat16))
    with pytest.raises(ValueError):  # wrong table dtype / length
        _conversion(torch.uint8, torch.bfloat16, torch.zeros(256, dtype=torch.float32))
    with pytest.raises(ValueError):
        _conversion(torch.uint8, torch.float32, torch.zeros(255, dtype=torch.float32))
    # 2-byte float buffers only for converting calls
    with pytest.raises(NotImplementedError):
        _Buf(torch.zeros(4, dtype=torch.bfloat16))
    assert _Buf(torch.zeros(4, dtype=torch.float16), half_ok=True).nbytes == 8


def test_capi_convert_errors_without_a_device():
    from ddstore_b200 import _capi
    L = _capi.lib()
    tot, bad = C.c_int64(5), C.c_int64(5)
    cv = _capi.Convert(co.CVT_F32_BF16, None)
    rc = L.dds_get_batch_convert(None, b"x", None, None, 1, 0, None, 0, None, _capi.DST_ON_DEVICE, None, C.byref(cv),
                                 C.byref(tot), C.byref(bad))
    assert rc == _capi.ERR_ARG and tot.value == 0 and bad.value == -1
    rc = L.dds_get_samples_convert(None, b"x", None, 0, None, 0, None, _capi.DST_ON_DEVICE, None, C.byref(cv),
                                   C.byref(tot), C.byref(bad))
    assert rc == _capi.ERR_ARG
    rc = L.dds_get_samples_multi_convert(None, 1, None, None, 0, None, None, None, _capi.DST_ON_DEVICE, None, None, None,
                                         C.byref(bad))
    assert rc == _capi.ERR_ARG


def test_header_declares_the_converting_abi():
    h = open(os.path.join(ROOT, "include", "ddstore_b200.h")).read()
    for sym in ("dds_get_batch_convert", "dds_get_samples_convert", "dds_get_samples_multi_convert", "dds_convert_t"):
        assert sym in h
    for name, val in [("DDS_CVT_F32_BF16", 1), ("DDS_CVT_F32_F16", 2), ("DDS_CVT_F64_F32", 3), ("DDS_CVT_U8_LUT16", 4),
                      ("DDS_CVT_U8_LUT32", 5)]:
        assert f"#define {name} {val}" in h


def test_bench_convert_cli_help_and_no_gpu_failure():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_convert.py"), "--help"], capture_output=True, text=True,
                       timeout=120)
    assert r.returncode == 0 and "--steps" in r.stdout
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_convert.py"), "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode != 0 and "GPU" in (r.stdout + r.stderr)
