"""NumPy oracle of the pooled batches (dds_get_batch_pooled / dds_get_samples_pooled): bags of a batch's rows folded into
one row each, over a world of shards.

Requests are located and validated by tests/put_oracle.py (the reference's two checks, sample ids against the index).
Bag k folds the rows of requests [bags[k], bags[k+1]) -- request order, then row order -- into output row k; an invalid
request contributes nothing; an empty bag, or one whose requests are all invalid, is +0. Per output element:
  sum   acc = acc + x (one IEEE rounding), with weights acc = fma(w, x, acc) (one rounding: computed exactly);
  mean  the sum divided once by the rows folded;
  then one round-to-nearest-even conversion to the element type, a NaN becoming the canonical NaN;
  max   in the element type: the first row's bits, then x's bits wherever x > acc (so NaNs after the first row are ignored
        and of -0 / +0 the earlier one stays).
acc is float32 for float32, float16 and bfloat16 rows and float64 for float64 rows. bfloat16 is kept as its bits
(uint16). A malformed bag (bags[k] < 0, bags[k+1] < bags[k] or bags[k+1] > nreq) is written as zeros and reported
before any invalid request.
"""
from fractions import Fraction

import numpy as np

from tests import put_oracle as po

ACC_F32, ACC_F64, ACC_F16, ACC_BF16 = 1, 2, 5, 6
POOL_SUM, POOL_MEAN, POOL_MAX = 1, 2, 3
CODE_BAG = 16
STORAGE = {ACC_F32: np.float32, ACC_F64: np.float64, ACC_F16: np.float16, ACC_BF16: np.uint16}
BITS = {ACC_F32: np.uint32, ACC_F64: np.uint64, ACC_F16: np.uint16, ACC_BF16: np.uint16}
CANONICAL_NAN = {ACC_F32: 0x7FFFFFFF, ACC_F64: 0x7FFFFFFFFFFFFFFF, ACC_F16: 0x7FFF, ACC_BF16: 0x7FFF}
# (significand bits, smallest normal exponent, largest exponent) of the accumulators
FORMAT = {np.float32: (24, -126, 127), np.float64: (53, -1022, 1023)}


def acc_dtype(t):
    return np.float64 if t == ACC_F64 else np.float32


def decode(a, t):
    """storage array -> accumulator values (exact: every element type is a subset of its accumulator)"""
    with np.errstate(invalid="ignore"):
        if t == ACC_BF16:
            return (np.asarray(a, np.uint16).astype(np.uint32) << 16).view(np.float32)
        return np.asarray(a, STORAGE[t]).astype(acc_dtype(t))


def encode(v, t):
    """accumulator values -> element bits: one round-to-nearest-even conversion, NaN -> the canonical NaN"""
    v = np.asarray(v, acc_dtype(t))
    nan = np.isnan(v)
    with np.errstate(over="ignore", invalid="ignore"):
        if t == ACC_BF16:
            b = v.view(np.uint32)
            out = ((b + np.uint32(0x7FFF) + ((b >> 16) & 1)) >> 16).astype(np.uint16)
        else:
            out = v.astype(STORAGE[t]).view(BITS[t])
    return np.where(nan, BITS[t](CANONICAL_NAN[t]), out).astype(BITS[t])


def round_fraction(q, dt):
    """the exact rational q rounded once to nearest-even in float dtype dt (subnormals kept, overflow to inf)"""
    p, emin, emax = FORMAT[dt]
    if q == 0:
        return dt(0.0)
    sign = -1 if q < 0 else 1
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()  # 2^e <= a < 2^(e+2)
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    quantum = Fraction(2) ** (max(e, emin) - (p - 1))
    n = a / quantum
    fl = n.numerator // n.denominator
    rem = n - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    r = fl * quantum
    if r >= Fraction(2) ** (emax + 1):
        return dt(sign * np.inf)
    return dt(sign * float(r)) if dt is np.float64 else np.float32(sign * float(r))  # (r is exact in both)


def fma(w, x, acc, dt):
    """fma(w, x, acc) element-wise in float dtype dt with ONE rounding: exact when the float64 two-sum of the (exact)
    float32 product and acc leaves no error, else through Fraction"""
    shape = np.broadcast(w, x, acc).shape
    w, x, acc = (np.atleast_1d(np.asarray(v, dt)) for v in np.broadcast_arrays(w, x, acc))
    with np.errstate(over="ignore", invalid="ignore"):
        if dt is np.float32:
            s = w.astype(np.float64) * x.astype(np.float64)  # 24 + 24 bits: exact
            a = acc.astype(np.float64)
            t = s + a
            bp = t - s
            err = (s - (t - bp)) + (a - bp)
            out = t.astype(np.float32)
            slow = np.isfinite(t) & (err != 0)
        else:
            out = w * x + acc  # (replaced below wherever the operands are finite)
            slow = np.isfinite(w) & np.isfinite(x) & np.isfinite(acc)
    out = np.array(out, dt)
    for idx in zip(*np.nonzero(slow)):
        out[idx] = round_fraction(Fraction(float(w[idx])) * Fraction(float(x[idx])) + Fraction(float(acc[idx])), dt)
    return out.reshape(shape)


def bag_bounds(bags, nbags, nreq):
    """[(b0, b1) or None for a malformed bag] of every bag"""
    if bags is None:
        return [(k, k + 1) for k in range(nreq)]
    b = [int(v) for v in np.asarray(bags, np.int64).tolist()]
    return [(b[k], b[k + 1]) if 0 <= b[k] <= b[k + 1] <= nreq else None for k in range(nbags)]


def pool(shards, t, mode, bags=None, weights=None, **req):
    """The pooled batch over `shards` (one 2-D storage array per rank; bf16 as uint16 bits) -> (out bits [nbags, disp],
    per-request codes, (expected code, bad index)). weights: one per request (storage values/bits of t), sum only."""
    lenlist = po.lenlist_of(shards)
    disp = shards[0].shape[1]
    allrows = np.concatenate([np.asarray(s).reshape(-1, disp) for s in shards]) if len(shards) else None
    reqs = po.requests(**req)
    nreq = len(reqs)
    nbags = nreq if bags is None else len(bags) - 1
    bounds = bag_bounds(bags, nbags, nreq)
    codes, where = [], []
    for start, count, id_ok in reqs:
        code, _, _ = (po.CODE_SAMPLE, 0, 0) if not id_ok else po.locate(lenlist, start, count)
        codes.append(code)
        where.append((start, count))
    dt = acc_dtype(t)
    wv = decode(np.asarray(weights, STORAGE[t]), t) if weights is not None else None
    out = np.zeros((nbags, disp), BITS[t])
    for k, bd in enumerate(bounds):
        if bd is None:
            continue
        acc = np.zeros(disp, dt)
        mx = np.zeros(disp, BITS[t])
        rows = 0
        for i in range(*bd):
            if codes[i]:
                continue
            start, count = where[i]
            for r in range(start, start + count):
                xb = np.asarray(allrows[r]).view(BITS[t]) if t != ACC_BF16 else np.asarray(allrows[r], np.uint16)
                x = decode(allrows[r], t)
                if mode == POOL_MAX:
                    mx = xb.copy() if rows == 0 else np.where(x > decode_bits(mx, t), xb, mx)
                elif wv is not None:
                    acc = fma(wv[i], x, acc, dt)
                else:
                    with np.errstate(over="ignore", invalid="ignore"):
                        acc = (acc + x).astype(dt)
                rows += 1
        if mode == POOL_MAX:
            out[k] = mx
        else:
            if mode == POOL_MEAN and rows > 0:
                with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                    acc = (acc / dt(rows)).astype(dt)
            out[k] = encode(acc, t)
    badbag = next((k for k, bd in enumerate(bounds) if bd is None), -1)
    if badbag >= 0:
        return out, codes, (CODE_BAG, badbag)
    covered = sorted(i for bd in bounds for i in range(*bd) if codes[i])
    return out, codes, ((codes[covered[0]], covered[0]) if covered else (0, -1))


def decode_bits(bits, t):
    """element bits -> accumulator values"""
    if t == ACC_BF16:
        return decode(bits, t)
    return decode(np.asarray(bits, BITS[t]).view(STORAGE[t]), t)
