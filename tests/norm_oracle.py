"""tests/norm_oracle.py -- NumPy restatement of the normalising conversions (DDS_CVT_NORM_*).

Element rule of include/ddstore_b200.h: y = (decode(x) - mean[ch]) / std[ch] in float32 with one IEEE rounding after
the subtraction and one after the division, then encoded. NumPy's float32 ufuncs round each operation to nearest even
and keep subnormals, so `(x - m) / s` on float32 arrays is that rule. Encoding reuses tests/convert_oracle.py (bf16
rounding in integer arithmetic). The channel of element e of a variable's packed rows is (e mod (nchan * inner)) // inner:
every request starts at a row boundary, and nchan * inner divides the row. NaN results are only specified by class.
"""
import numpy as np

from tests import convert_oracle as co

CVT_NORM_F32_F32, CVT_NORM_F32_BF16, CVT_NORM_F32_F16, CVT_NORM_F64_F32 = 6, 7, 8, 9
CVT_NORM_U8_F32, CVT_NORM_U8_BF16, CVT_NORM_U8_F16 = 10, 11, 12
# code -> (source itemsize, output itemsize, source kind, output kind)
NORM = {CVT_NORM_F32_F32: (4, 4, "f32", "f32"), CVT_NORM_F32_BF16: (4, 2, "f32", "bf16"),
        CVT_NORM_F32_F16: (4, 2, "f32", "f16"), CVT_NORM_F64_F32: (8, 4, "f64", "f32"),
        CVT_NORM_U8_F32: (1, 4, "u8", "f32"), CVT_NORM_U8_BF16: (1, 2, "u8", "bf16"), CVT_NORM_U8_F16: (1, 2, "u8", "f16")}


def channels(n, nchan, inner, first=0):
    """channel of elements first .. first + n - 1 of a variable's packed rows"""
    e = np.arange(first, first + n, dtype=np.int64)
    return (e % (nchan * inner)) // inner


def decode(src, code, lut=None):
    """packed source bytes -> float32 values (lut: 256 float32 entries, uint8 codes)"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    kind = NORM[code][2]
    if kind == "f32":
        return src.view(np.float32).copy()
    if kind == "f64":
        return co.f64_to_f32_bits(src.view(np.uint64)).view(np.float32)
    return np.ascontiguousarray(lut, dtype=np.float32).reshape(-1)[:256][src]


def normalise(x, mean, std, nchan, inner):
    """float32 values of a variable's packed rows (from its base) -> (x - mean[ch]) / std[ch], float32"""
    ch = channels(x.size, nchan, inner)
    m = np.asarray(mean, np.float32)[ch]
    s = np.asarray(std, np.float32)[ch]
    with np.errstate(all="ignore"):
        return (np.asarray(x, np.float32) - m) / s


def encode(y, code):
    """float32 values -> output bytes of the code's output type"""
    bits = np.ascontiguousarray(y, np.float32).view(np.uint32)
    kind = NORM[code][3]
    if kind == "f32":
        return bits.view(np.uint8).copy()
    if kind == "bf16":
        return co.f32_to_bf16_bits(bits).view(np.uint8)
    return co.f32_to_f16_bits(bits).view(np.uint8)


def norm_bytes(src, code, mean, std, nchan, inner, lut=None):
    """a variable's packed source bytes (from a row boundary) -> its normalised output bytes"""
    return encode(normalise(decode(src, code, lut), mean, std, nchan, inner), code)


def out_bytes(src_bytes, code):
    i, o = NORM[code][:2]
    assert src_bytes % i == 0
    return src_bytes // i * o


def bad_elements(got, exp, code):
    """indices of output elements that differ, NaN compared by class"""
    kind = NORM[code][3]
    dt = np.uint32 if kind == "f32" else np.uint16
    g, e = np.asarray(got, np.uint8).view(dt), np.asarray(exp, np.uint8).view(dt)
    if kind == "f32":
        isnan = lambda b: ((b & 0x7F800000) == 0x7F800000) & ((b & 0x7FFFFF) != 0)  # noqa: E731
    elif kind == "bf16":
        isnan = lambda b: ((b & 0x7F80) == 0x7F80) & ((b & 0x7F) != 0)  # noqa: E731
    else:
        isnan = lambda b: ((b & 0x7C00) == 0x7C00) & ((b & 0x3FF) != 0)  # noqa: E731
    return np.flatnonzero(~((g == e) | (isnan(g) & isnan(e))))


# table values at the edges of the arithmetic: std = 0 (+-inf, NaN for 0/0), negative std, infinite and NaN mean,
# subnormal std (huge quotients), -0 mean, std = 1 (exact), and values whose quotients overflow f16 / bf16 or land in
# their subnormal ranges
TABLE_EDGE_MEAN = np.array([0.0, -0.0, 1.5, np.inf, -np.inf, np.nan, 3.0e38, 1e-40, 0.1, -7.25, 2.0, 0.5],
                           np.float32)
TABLE_EDGE_STD = np.array([1.0, 0.0, -0.0, -2.0, 1e-45, 1e-39, 3.0e-5, 1e30, 0.3, -1e-8, np.inf, 7.0e-6], np.float32)
