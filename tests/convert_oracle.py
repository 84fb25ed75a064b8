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


# float32 rounding edges for bf16 and f16: ties both ways, overflow, subnormals, -0, inf, NaN
F32_EDGE_BITS = (0x3F808000, 0x3F818000, 0x3F80FFFF, 0x7F7FFFFF, 0x477FF000, 0x477FEFFF, 0x33800000, 0x33000000,
                 0x33000001, 0x387FC000, 0x80000000, 0x00000001, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001,
                 0xFF7FFFFF, 0x00800000)


def f64_edge_bits():
    """float64 bit patterns at the edges of the f64 -> f32 rounding (round to nearest even), each with its sign flipped
    too: ties at the f32 half-ulp with an even and an odd last kept bit, one f64 ulp either side of them; the largest
    value that rounds to FLT_MAX and the smallest that rounds to inf; results in the f32 subnormal range, the smallest
    subnormal's half (a tie to 0) and 1.5 of it (a tie to 2 units), the largest subnormal's tie into the normal range;
    f64 subnormals, 0, inf; NaNs whose payload lies only in the 29 bits the cast drops (quiet NaN, not inf)"""
    pos = [0x3FF0000010000000, 0x3FF0000030000000,                          # 1 + 2^-24 (down to even), 1 + 3*2^-24 (up)
           0x3FF000000FFFFFFF, 0x3FF0000010000001, 0x3FF000002FFFFFFF, 0x3FF0000030000001,
           0x4123456790000000, 0x4123456770000000,                          # ties in another binade, even / odd kept bit
           0x47EFFFFFE0000000, 0x47EFFFFFEFFFFFFF,                          # FLT_MAX, the largest that rounds to it
           0x47EFFFFFF0000000, 0x47F0000000000000,                          # the smallest that rounds to inf, 2^128
           0x3810000000000000, 0x380FFFFFC0000000,                          # FLT_MIN, the largest f32 subnormal,
           0x380FFFFFE0000000, 0x380FFFFFDFFFFFFF,                          # its tie up to FLT_MIN, just below it
           0x37D0000000000000, 0x36A0000000000000, 0x36A8000000000000,      # 2^-130, 2^-149, 1.5 * 2^-149
           0x3690000000000000, 0x3690000000000001, 0x368FFFFFFFFFFFFF,      # 2^-150 (tie to 0) and either side
           0x36B4000000000000, 0x36B2000000000000,                          # 2.5 units (tie to 2), 2.25 units
           0x0000000000000001, 0x000FFFFFFFFFFFFF, 0x0000000000000000,      # f64 subnormals, 0
           0x7FF0000000000000, 0x7FF0000000000001, 0x7FF000001FFFFFFF,      # inf, NaNs with low payload only
           0x7FF0000010000000, 0x7FF8000000000000]
    pos = np.array(pos, np.uint64)
    return np.concatenate([pos, pos | np.uint64(1 << 63)])


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
