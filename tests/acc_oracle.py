"""NumPy oracle of the batched accumulate (dds_accumulate_batch / dds_accumulate_samples): calls applied to a world of shards.

Requests, the layout of src, validation and errors are the put's (tests/put_oracle.py: requests, locate and
expected_error are reused): an invalid request keeps its bytes in the layout and changes nothing, every valid one is
applied, a layout larger than src applies nothing. Each element of a valid request's rows becomes the shard's element
plus src's, in the accumulate's type. The expectation of `accumulate` is start + the sum of every contribution per
element: integer types wrap; floating types are only checked that way on data whose sums are exact in the type (integer
values with |sum| below 2^24 for f32, 2^53 for f64, at most 2048 for f16 and 256 for bf16), where every order of
roundings gives it.

The arithmetic itself, on inexact data, is checked against the second half of this module: `add` (one correctly
rounded addition per type), the f32 flush model, `admissible` (every result the header allows for an element with a
few contributions, over every order) and `sum_bound` (for elements with many), `verdict` (names the first element
outside them), and `drain_path` (which of the kernel's three reductions an element of a one-piece call takes).

Shards are 2-D arrays of the element type (bf16: uint16 arrays of its bits), one per rank.
"""
import itertools
import math
from fractions import Fraction

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
    """round-to-nearest-even bits of float32 values (exact for values bf16 holds); a NaN stays a NaN: its top 16 bits
    with the quiet bit set (rounding would carry a low payload into the exponent: 0x7F800001 -> 0x7F80, +inf)"""
    b = np.asarray(x, np.float32).view(np.uint32)
    rne = ((b + np.uint32(0x7FFF) + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where((b & 0x7FFFFFFF) > 0x7F800000, ((b >> 16) | 0x0040).astype(np.uint16), rne)


def values(a, t):
    """element values of storage array `a` as float64 (floats) or int64 (integers)"""
    with np.errstate(invalid="ignore"):  # (signalling NaNs stay NaNs)
        if t == ACC_BF16:
            return bf16_to_f32(a).astype(np.float64)
        return np.asarray(a).astype(np.int64 if t in (ACC_I32, ACC_I64) else np.float64)


def encode(v, t):
    """values (float64 / int64) -> storage array of type t (integers wrap)"""
    with np.errstate(over="ignore", invalid="ignore"):
        if t == ACC_BF16:
            return f32_to_bf16(np.asarray(v, np.float64).astype(np.float32))
        return np.asarray(v).astype(STORAGE[t])


def add(a, b, t):
    """a + b element-wise in type t (a, b storage arrays of one shape): integers wrap; floats are ONE correctly rounded
    IEEE addition (to nearest, ties to even; overflow to inf, subnormals kept, NaN in -> NaN out). f64 is NumPy's own
    addition. f32 is the sum taken in f64 and rounded once to f32, f16 and bf16 the sum taken in f32 and rounded once
    to nearest-even: a sum taken with q >= 2p + 2 significand bits and rounded once to p bits is the correctly rounded
    p-bit sum, and 53 >= 2*24 + 2, 24 >= 2*11 + 2 >= 2*8 + 2."""
    if t == ACC_I64:
        return (np.asarray(a, np.int64).view(np.uint64) + np.asarray(b, np.int64).view(np.uint64)).view(np.int64)
    if t == ACC_I32:
        return (np.asarray(a, np.int32).view(np.uint32) + np.asarray(b, np.int32).view(np.uint32)).view(np.int32)
    with np.errstate(over="ignore", invalid="ignore"):
        if t == ACC_F64:
            return np.asarray(a, np.float64) + np.asarray(b, np.float64)
        if t == ACC_F32:
            return (np.asarray(a, np.float32).astype(np.float64) + np.asarray(b, np.float32)).astype(np.float32)
        if t == ACC_F16:
            return (np.asarray(a, np.float16).astype(np.float32) + np.asarray(b, np.float16)).astype(np.float16)
        return f32_to_bf16(bf16_to_f32(a) + bf16_to_f32(b))


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


# ------------------------------------------------------------------------------------------------ the arithmetic
FLOATS = (ACC_F32, ACC_F64, ACC_F16, ACC_BF16)
BITS = {ACC_F32: np.uint32, ACC_F64: np.uint64, ACC_I32: np.uint32, ACC_I64: np.uint64, ACC_F16: np.uint16,
        ACC_BF16: np.uint16}
PREC = {ACC_F32: 24, ACC_F64: 53, ACC_F16: 11, ACC_BF16: 8}         # significand bits p (unit roundoff 2^-p)
EMIN = {ACC_F32: -126, ACC_F64: -1022, ACC_F16: -14, ACC_BF16: -126}  # exponent of the smallest normal
NAN = -1  # the key of every NaN: NaNs compare by class


def bits(a, t):
    """the bit patterns of storage array `a` (unsigned)"""
    return np.ascontiguousarray(a, STORAGE[t]).view(BITS[t])


def from_bits(b, t):
    return np.ascontiguousarray(b, BITS[t]).view(STORAGE[t])


def is_nan(a, t):
    if t not in FLOATS:
        return np.zeros(np.shape(a), bool)
    return np.isnan(values(a, t))


def keys(a, t):
    """int64 comparison keys of storage array `a`: its bits, NAN for every NaN"""
    k = bits(a, t).astype(np.uint64).view(np.int64)
    return np.where(is_nan(a, t), NAN, k)


def min_normal(t):
    return 2.0 ** EMIN[t]


def flush32(a):
    """f32 subnormals -> zero of their sign"""
    a = np.asarray(a, np.float32)
    return np.where(np.abs(a) < np.float32(min_normal(ACC_F32)), np.copysign(np.float32(0), a), a)


def add_flushed(a, b):
    """the f32 flush model: subnormal inputs flushed to signed zero, the IEEE sum of those, a subnormal result then
    flushed to signed zero (what REDG.E.ADD.F32.FTZ.RN does).

    A sum of two f32 values is a multiple of the smallest subnormal, so a sum below the smallest normal is exact and
    representable: no sum rounds UP to the smallest normal, and "tiny before or after rounding" never differ. The
    min-normal boundary that remains is a result AT it made of subnormal inputs (max subnormal + min subnormal = min
    normal: IEEE gives min normal, the model +0) or just below it (min normal - min subnormal: IEEE gives the max
    subnormal, the model min normal); `admissible` admits both and the GPU module reports which the hardware gave."""
    return flush32(add(flush32(a), flush32(b), ACC_F32))


def admissible_all(start, contribs, t):
    """every result the header allows for elements with start value `start` and contributions `contribs` (k <= 3
    storage arrays of start's shape): one addition per contribution, correctly rounded, in any of the k! orders; for f32
    each addition independently IEEE or flushed (an element's contributions may take different paths). Returns the
    keys, shape [options, *start.shape]."""
    contribs = list(contribs)
    assert len(contribs) <= 3
    out = []
    for order in itertools.permutations(range(len(contribs))):
        for mask in range(1 << len(contribs)) if t == ACC_F32 else (0,):
            acc = np.asarray(start, STORAGE[t])
            for step, i in enumerate(order):
                acc = add_flushed(acc, contribs[i]) if mask >> step & 1 else add(acc, contribs[i], t)
            out.append(keys(acc, t))
    return np.stack(out)


def admissible(start, contributions, t):
    """the set of admissible result keys of ONE element (start and contributions: scalars of the storage type)"""
    a = admissible_all(np.array([start], STORAGE[t]), [np.array([c], STORAGE[t]) for c in contributions], t)
    return set(a[:, 0].tolist())


def exact_sum(xs):
    """the exact sum of float64 values, as a Fraction"""
    return sum((Fraction(float(x)) for x in xs), Fraction(0))


def gamma(m, t):
    u = 2.0 ** -PREC[t]
    return m * u / (1 - m * u)


def sum_bound(start, contribs, t):
    """(s, bound) per element for a start value and n - 1 contributions summed in any order with one rounding per
    addition: |got - s| <= gamma(n - 1) * sum |x_i| (Higham, recursive summation), s the exact sum. start: [N] storage
    array, contribs: [n - 1, N]. s is math.fsum (the exact sum rounded once in f64); the bound grows by half an f64
    ulp of s to cover that rounding. Valid for data in the normal range that does not overflow."""
    x = np.concatenate([values(np.asarray(start)[None], t), values(np.asarray(contribs), t)])
    s = np.array([math.fsum(x[:, j]) for j in range(x.shape[1])])
    mag = np.array([math.fsum(np.abs(x[:, j])) for j in range(x.shape[1])])
    return s, gamma(x.shape[0] - 1, t) * mag + np.abs(s) * 2.0 ** -53


# ------------------------------------------------------------------------------------------------ test data
def _finite_bits(rng, n, t):
    nb = np.dtype(BITS[t]).itemsize * 8
    b = rng.integers(0, 2**nb, size=n, dtype=np.uint64).astype(BITS[t])
    v = from_bits(b, t)
    bad = ~np.isfinite(values(v, t))
    b[bad] &= ~BITS[t](1 << (nb - 2))  # the exponent's top bit cleared: finite
    return b


def inexact(rng, shape, t, lo=-2, hi=2):
    """values of random sign with exponents in [lo, hi] and random full-precision significands (storage array)"""
    n = int(np.prod(shape))
    p = PREC[t]
    m = (1 << (p - 1)) + rng.integers(0, 1 << (p - 1), size=n, dtype=np.int64)
    e = rng.integers(lo, hi + 1, size=n)
    v = np.ldexp(m.astype(np.float64), e - (p - 1)) * rng.choice([-1.0, 1.0], size=n)
    return encode(v, t).reshape(shape)


def families(rng, t, n):
    """name -> (a, b) storage arrays of n pairs each: the value families one addition is checked on. Integers: wraps
    past the type's range and random bits. Floats: random finite bits, ties both ways, subnormal + subnormal,
    normals cancelling to a subnormal, the smallest normal, the overflow threshold, signed zeros, inf and NaN."""
    if t in (ACC_I32, ACC_I64):
        top = 2**(8 * np.dtype(STORAGE[t]).itemsize - 1)
        near = rng.integers(0, 1 << 20, size=n).tolist()
        big = rng.integers(1, 1 << 30, size=n).tolist()
        st = lambda v: np.array(v, np.int64).astype(STORAGE[t])  # noqa: E731
        # a within 2^20 of the range's end, b past it by up to 2^30: every sum wraps
        return {"wrap up": (st([top - 1 - x for x in near]), st([x + y + 1 for x, y in zip(near, big)])),
                "wrap down": (st([-top + x for x in near]), st([-(x + y + 1) for x, y in zip(near, big)])),
                "random": (from_bits(rng.integers(0, 2**63, size=n, dtype=np.uint64).astype(BITS[t]), t),
                           from_bits(rng.integers(0, 2**63, size=n, dtype=np.uint64).astype(BITS[t]) << 1, t))}
    p, emin = PREC[t], EMIN[t]
    sub_min = 2.0 ** (emin - p + 1)
    mn = 2.0 ** emin
    sign = lambda: rng.choice([-1.0, 1.0], size=n)  # noqa: E731
    ex = lambda v: encode(v, t)  # noqa: E731 (every value below is exact in the type)
    out = {"random": (from_bits(_finite_bits(rng, n, t), t), from_bits(_finite_bits(rng, n, t), t))}
    # a + b exactly halfway between two neighbours: a's last significand bit decides the direction
    a = np.abs(values(inexact(rng, n, t, -3, 3), t)) * sign()
    ulp = np.ldexp(1.0, np.frexp(a)[1] - p)
    out["ties"] = (ex(a), ex(np.where(rng.random(n) < 0.5, 0.5, 1.5) * ulp * sign()))
    sub = lambda: rng.integers(1, 1 << (p - 1), size=n) * sub_min * sign()  # noqa: E731
    out["subnormal"] = (ex(sub()), ex(sub()))
    a = values(ex(rng.integers(1 << (p - 1), 1 << (p + 1), size=n) * sub_min * sign()), t)  # normals in [mn, 4 mn)
    d = rng.integers(-8, 9, size=n) * sub_min * np.where(np.abs(a) < 2 * mn, 1, 2)  # a few of a's ulps
    out["cancel"] = (ex(a), ex(-(a + d)))
    edge = np.array([mn, mn - sub_min, sub_min, 2 * mn, mn + 2 * sub_min, mn / 2, 0.0])
    pairs = np.array([(mn - sub_min, sub_min), (mn, -sub_min), (mn / 2, mn / 2), (mn - sub_min, mn - sub_min),
                      (mn, -mn), (2 * mn, -(mn + sub_min))])
    k = rng.integers(0, len(pairs) + 3, size=n)
    a = np.where(k < len(pairs), pairs[np.minimum(k, len(pairs) - 1), 0], edge[rng.integers(0, len(edge), size=n)])
    b = np.where(k < len(pairs), pairs[np.minimum(k, len(pairs) - 1), 1], edge[rng.integers(0, len(edge), size=n)])
    s = sign()
    out["min normal"] = (ex(a * s), ex(b * s * np.where(rng.random(n) < 0.8, 1, -1)))
    mx = float(values(from_bits(np.array([_max_bits(t)], BITS[t]), t), t)[0])
    mu = 2.0 ** (math.frexp(mx)[1] - p)  # the ulp of the largest finite value; mx + mu / 2 is the overflow threshold
    frac = np.array([0.25, 0.5, 0.75, 1.0, 0.5 - 2.0 ** -(p - 1), 8.0])  # below, at and above the threshold
    s = sign()
    out["overflow"] = (ex(mx * s), ex(frac[rng.integers(0, len(frac), size=n)] * mu * s))
    z = rng.integers(0, 4, size=n)
    x = values(inexact(rng, n, t, -6, 6), t)
    za = np.where(z == 0, 0.0, np.where(z == 1, -0.0, np.where(z == 2, -0.0, x)))
    zb = np.where(z == 0, -0.0, np.where(z == 1, -0.0, np.where(z == 2, x, -x)))
    out["zeros"] = (ex(za), ex(zb))
    sp = np.array([np.inf, -np.inf, np.nan, 1.5, -0.0])
    sa, sb = ex(sp[rng.integers(0, 5, size=n)]), ex(sp[rng.integers(0, 4, size=n)])
    nb = bits(sa, t).copy()
    nanb = is_nan(sa, t)  # NaNs with other payloads and signs: quiet, signalling, low payload, negative
    pay = np.array([_nan_bits(t, q) for q in range(4)], BITS[t])
    nb[nanb] = pay[rng.integers(0, 4, size=int(nanb.sum()))]
    out["inf nan"] = (from_bits(nb, t), sb)
    return out


def _max_bits(t):
    return {ACC_F32: 0x7F7FFFFF, ACC_F64: 0x7FEFFFFFFFFFFFFF, ACC_F16: 0x7BFF, ACC_BF16: 0x7F7F}[t]


def _nan_bits(t, q):
    """0: the canonical quiet NaN, 1: a signalling NaN with payload 1, 2: a negative quiet NaN with a payload,
    3: a quiet NaN with a payload in the low bits"""
    nb = np.dtype(BITS[t]).itemsize * 8
    e = ((1 << (nb - 1)) - 1) & ~((1 << (PREC[t] - 1)) - 1)
    qb = 1 << (PREC[t] - 2)
    return [e | qb, e | 1, (1 << (nb - 1)) | e | qb | 5, e | qb | 3][q]


# ------------------------------------------------------------------------------------------------ paths and verdicts
def drain_path(dst_phase, src_phase, nbytes, k):
    """which reduction the kernel's drain (write_chunk<kActReduce>) uses for byte k of ONE staged piece of nbytes bytes whose
    destination starts dst_phase bytes and whose staged source starts src_phase bytes past a 16-byte boundary: the
    head before the destination's first 16-byte boundary and the tail after its last are element reductions; the body
    between is one bulk reduction when source and destination share the phase, re-phased vector reductions otherwise.
    k may be an array."""
    k = np.asarray(k)
    head = min((16 - dst_phase) % 16, nbytes)
    body = ((nbytes - head) >> 4) << 4
    inner = "bulk" if (src_phase + head) % 16 == 0 else "vector"
    return np.where((k < head) | (k >= head + body), "element", inner)


def verdict(got, start, contribs, t, opts=None, where=None, paths=None, what=""):
    """None when every element's result (got, storage array [N]) is admissible; else a message naming the first bad
    element -- `where(i)` -> (rank, global row, column) -- with its inputs, the bits it got, the admissible bits and,
    when given, its predicted drain path. `opts`: admissible_all's keys, when already computed."""
    opts = admissible_all(start, contribs, t) if opts is None else opts
    gk = keys(got, t)
    ok = (opts == gk[None]).any(0)
    if ok.all():
        return None
    i = int(np.argmin(ok))
    rank, row, col = where(i) if where else (0, i, 0)
    w = 2 * np.dtype(BITS[t]).itemsize
    fmt = lambda k: "NaN" if k == NAN else f"{int(k) & ((1 << 4 * w) - 1):#0{w + 2}x}"  # noqa: E731
    ins = ", ".join(f"{fmt(keys(np.asarray(c)[i:i + 1], t)[0])} ({values(np.asarray(c)[i:i + 1], t)[0]!r})"
                    for c in [start] + list(contribs))
    return (f"{what}: {int((~ok).sum())} of {ok.size} elements outside the admissible set; first: rank {rank}, global row "
            f"{row}, column {col}{'' if paths is None else f' (path {paths[i]})'}: start + contributions {ins}: got "
            f"{fmt(gk[i])} ({values(np.asarray(got)[i:i + 1], t)[0]!r}), admissible "
            f"{{{', '.join(sorted(set(fmt(k) for k in opts[:, i])))}}}")


# the GPU module's data for elements with two or three contributions: at least this fraction of them has more than one
# admissible result, so the check tells orders (and a rounding other than one per addition) apart
DISCRIMINATION = 0.25
# hot elements: contributions per element, few enough for f16 / bf16 that sum_bound stays below the smallest |value|
# (values of random sign in [1, 4): inexact(..., 0, 1))
HOT = {ACC_F32: 1024, ACC_F64: 65536, ACC_F16: 16, ACC_BF16: 6, ACC_I32: 4096, ACC_I64: 4096}
