"""tests/convert_oracle.py -- NumPy restatement of the converting batches (dds_get_batch_convert & co.).

What a converting batch must deliver, written without the store: the element rules of include/ddstore_b200.h
(DDS_CVT_*) and the byte arithmetic of converted packing. bf16 rounding is done in integer arithmetic, so it does
not lean on any library's cast; f16 and f64 -> f32 use NumPy's casts, which round to nearest even with subnormals and
overflow to inf. NaN results are only specified by class (quiet NaN), so compare them with `same_bits_or_both_nan`.
"""
import numpy as np

CVT_NONE, CVT_F32_BF16, CVT_F32_F16, CVT_F64_F32, CVT_U8_LUT16, CVT_U8_LUT32 = 0, 1, 2, 3, 4, 5
# code -> (source itemsize, output itemsize)
SIZES = {CVT_NONE: (1, 1), CVT_F32_BF16: (4, 2), CVT_F32_F16: (4, 2), CVT_F64_F32: (8, 4), CVT_U8_LUT16: (1, 2),
         CVT_U8_LUT32: (1, 4)}


def f32_to_bf16_bits(bits):
    """float32 bit patterns (uint32) -> bf16 bit patterns (uint16), round to nearest even; NaN -> 0x7FFF (quiet)"""
    u = np.asarray(bits, dtype=np.uint32).astype(np.uint64)
    nan = ((u >> 23) & 0xFF) == 0xFF
    nan &= (u & 0x7FFFFF) != 0
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16  # carries into the exponent: overflow becomes inf, as it should
    return np.where(nan, 0x7FFF, r & 0xFFFF).astype(np.uint16)


def f32_to_f16_bits(bits):
    return np.asarray(bits, dtype=np.uint32).view(np.float32).astype(np.float16).view(np.uint16)


def f64_to_f32_bits(bits):
    return np.asarray(bits, dtype=np.uint64).view(np.float64).astype(np.float32).view(np.uint32)


def convert_bytes(src, code, lut=None):
    """packed source bytes (uint8, whole elements) -> packed output bytes of conversion `code`"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    if code == CVT_NONE:
        return src.copy()
    if code == CVT_F32_BF16:
        return f32_to_bf16_bits(src.view(np.uint32)).view(np.uint8)
    if code == CVT_F32_F16:
        return f32_to_f16_bits(src.view(np.uint32)).view(np.uint8)
    if code == CVT_F64_F32:
        return f64_to_f32_bits(src.view(np.uint64)).view(np.uint8)
    table = np.ascontiguousarray(lut).view(np.uint16 if code == CVT_U8_LUT16 else np.uint32)[:256]
    return table[src].view(np.uint8)


def out_bytes(src_bytes, code):
    """source byte count / offset (whole elements) -> output bytes"""
    i, o = SIZES[code]
    assert src_bytes % i == 0
    return src_bytes // i * o


def cap_to_src(cap_out, code):
    """an output capacity -> the source bytes it holds: whole output elements, scaled"""
    i, o = SIZES[code]
    return cap_out // o * i


def convert_packed(src_packed, src_offsets, code, lut=None):
    """a raw packed batch and its byte offsets -> the converted batch and its output byte offsets"""
    return convert_bytes(src_packed, code, lut), np.array([out_bytes(int(x), code) for x in src_offsets], np.int64)


def same_bits_or_both_nan(got, exp, code):
    """element-wise equality of two converted byte arrays, NaN compared by class; returns the bad element indices"""
    o = SIZES[code][1]
    dt = {2: np.uint16, 4: np.uint32}[o] if code != CVT_NONE else np.uint8
    g, e = np.asarray(got, np.uint8).view(dt), np.asarray(exp, np.uint8).view(dt)
    if code in (CVT_F32_BF16,):
        isnan = lambda b: ((b & 0x7F80) == 0x7F80) & ((b & 0x7F) != 0)  # noqa: E731
    elif code in (CVT_F32_F16,):
        isnan = lambda b: ((b & 0x7C00) == 0x7C00) & ((b & 0x3FF) != 0)  # noqa: E731
    elif code == CVT_F64_F32:
        isnan = lambda b: ((b & 0x7F800000) == 0x7F800000) & ((b & 0x7FFFFF) != 0)  # noqa: E731
    else:
        isnan = lambda b: np.zeros(b.shape, bool)  # noqa: E731
    ok = (g == e) | (isnan(g) & isnan(e))
    return np.flatnonzero(~ok)
