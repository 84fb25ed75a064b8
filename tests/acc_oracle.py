"""NumPy oracle of the batched accumulate (dds_accumulate_batch / dds_accumulate_samples): calls applied to a world of shards.

Requests, the layout of src, validation and errors are the put's (tests/put_oracle.py: requests, locate and
expected_error are reused): an invalid request keeps its bytes in the layout and changes nothing, every valid one is
applied, a layout larger than src applies nothing. Each element of a valid request's rows becomes the shard's element
plus src's, in the accumulate's type. The expectation is start + the sum of every contribution per element: integer
types wrap; floating types are only checked here on data whose sums are exact in the type (integer values with |sum|
below 2^24 for f32, 2^53 for f64, at most 2048 for f16 and 256 for bf16), where every order of roundings gives it.

Shards are 2-D arrays of the element type (bf16: uint16 arrays of its bits), one per rank.
"""
import numpy as np

from tests import put_oracle as po

ACC_F32, ACC_F64, ACC_I32, ACC_I64, ACC_F16, ACC_BF16 = 1, 2, 3, 4, 5, 6
# element type -> NumPy storage dtype (bf16 is kept as its bits)
STORAGE = {ACC_F32: np.float32, ACC_F64: np.float64, ACC_I32: np.int32, ACC_I64: np.int64, ACC_F16: np.float16,
           ACC_BF16: np.uint16}
NAMES = {ACC_F32: "float32", ACC_F64: "float64", ACC_I32: "int32", ACC_I64: "int64", ACC_F16: "float16",
         ACC_BF16: "bfloat16"}
# the largest |sum| whose every partial sum is exact in the type, for integer-valued data
EXACT = {ACC_F32: 2**24 - 1, ACC_F64: 2**53 - 1, ACC_F16: 2048, ACC_BF16: 256}


def bf16_to_f32(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16(x):
    """round-to-nearest-even bits of float32 values (exact for values bf16 holds)"""
    b = np.asarray(x, np.float32).view(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def values(a, t):
    """element values of storage array `a` as float64 (floats) or int64 (integers)"""
    if t == ACC_BF16:
        return bf16_to_f32(a).astype(np.float64)
    return np.asarray(a).astype(np.int64 if t in (ACC_I32, ACC_I64) else np.float64)


def encode(v, t):
    """values (float64 / int64) -> storage array of type t (integers wrap)"""
    if t == ACC_BF16:
        return f32_to_bf16(np.asarray(v, np.float64).astype(np.float32))
    return np.asarray(v).astype(STORAGE[t])


def add(a, b, t):
    """a + b element-wise in type t (a, b storage arrays of one shape)"""
    if t == ACC_I64:
        return (np.asarray(a, np.int64).view(np.uint64) + np.asarray(b, np.int64).view(np.uint64)).view(np.int64)
    return encode(values(a, t) + values(b, t), t)


def accumulate(shards, src, t, src_bytes=None, **req):
    """Apply one accumulate call of type t to `shards` (not modified). src: the packed source as bytes (uint8 array).
    Returns (new shards, per-request codes, first bad index or -1, layout total), as put_oracle.put."""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1]) if len(lenlist) else 0
    dt = np.dtype(STORAGE[t])
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    row_bytes = dt.itemsize * disp
    src = np.asarray(src, np.uint8).reshape(-1)
    src_bytes = src.size if src_bytes is None else src_bytes
    codes, plan, o = [], [], 0
    for start, count, id_ok in po.requests(**req):
        n = count * row_bytes if id_ok and 0 < count <= rows else 0
        code, r, off = (po.CODE_SAMPLE, 0, 0) if not id_ok else po.locate(lenlist, start, count)
        codes.append(code)
        plan.append((r, start - off, count, o, n))
        o += n
    total = o
    bad = next((i for i, c in enumerate(codes) if c), -1)
    new = [s.copy() for s in shards]
    if total <= src_bytes:
        for (r, local, count, off, n), code in zip(plan, codes):
            if code == 0 and n > 0:
                rows_r = new[r].reshape(new[r].shape[0], -1)
                rows_r[local:local + count] = add(rows_r[local:local + count],
                                                  src[off:off + n].view(dt).reshape(count, disp), t)
    return new, codes, bad, total


def accumulate_many(shards, calls, t):
    """Apply `calls` = [(src, src_bytes or None, request keywords)] (any ranks' calls of one epoch) -> (new shards,
    [(status code, bad index, layout total)] as each call reports them). On exact data the order does not matter."""
    out = []
    for src, src_bytes, req in calls:
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        shards, codes, bad, total = accumulate(shards, src, t, src_bytes=sb, **req)
        out.append(po.expected_error(codes, bad, total, sb) + (total,))
    return shards, out


def layout_src(rng, lenlist, disp, t, batch, lo=-3, hi=4):
    """a packed source for `batch`: random integer values in [lo, hi) for every element of the layout (an invalid
    request's bytes included, as the caller lays them out) -> uint8 array"""
    rows = int(lenlist[-1])
    n = sum(c * disp for _, c, ok in po.requests(**batch) if ok and 0 < c <= rows)
    v = rng.integers(lo, hi, size=n)
    return encode(v, t).view(np.uint8)


def mismatch(got, exp, rank, lenlist, R, what):
    """None when rank `rank`'s shard bytes `got` equal `exp`; else a message naming rank, global row and byte"""
    got = np.asarray(got).reshape(-1).view(np.uint8)
    exp = np.asarray(exp).reshape(-1).view(np.uint8)
    d = np.nonzero(got != exp)[0]
    if not d.size:
        return None
    b = int(d[0])
    row = b // R + (int(lenlist[rank - 1]) if rank else 0)
    return (f"{what}: rank {rank}: {d.size} bytes differ, first at local byte {b} (global row {row}, byte {b % R}): "
            f"got {int(got[b]):#04x}, expected {int(exp[b]):#04x}")
