"""CPU checks of the pooled batches' oracle (tests/pool_oracle.py) and of their declarations: the fold against a brute-force
per-element restatement in exact rational arithmetic, sums every order gives, the max rule's NaN and signed-zero cases,
empty and malformed bags, and the precedence of a malformed bag over an invalid request."""
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from ddstore_b200 import _capi
from tests import pool_oracle as pl
from tests import put_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = (pl.ACC_F32, pl.ACC_F64, pl.ACC_F16, pl.ACC_BF16)
# (significand bits, smallest normal exponent, largest exponent) of each element type, for the brute force
FMT = {pl.ACC_F32: (24, -126, 127), pl.ACC_F64: (53, -1022, 1023), pl.ACC_F16: (11, -14, 15), pl.ACC_BF16: (8, -126, 127)}


def rnd(q, fmt):
    """q rounded once to nearest-even in format fmt -> Fraction, or +-inf as a float"""
    p, emin, emax = fmt
    if q == 0:
        return Fraction(0)
    s, a = (-1 if q < 0 else 1), abs(q)
    e = 0
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    qu = Fraction(2) ** (max(e, emin) - (p - 1))
    n = a / qu
    fl = n.numerator // n.denominator
    if n - fl > Fraction(1, 2) or (n - fl == Fraction(1, 2) and fl % 2):
        fl += 1
    r = fl * qu
    return s * float("inf") if r >= Fraction(2) ** (emax + 1) else s * r


def to_bits(q, t):
    v = np.array([float(q)], np.float64)
    if t == pl.ACC_BF16:
        return int(pl.encode(v.astype(np.float32), t)[0])  # (exact: q is a bf16 value)
    return int(v.astype(pl.STORAGE[t]).view(pl.BITS[t])[0])


def brute(rows_per_bag, t, mode, wts=None):
    """per element, exact rationals rounded by hand: rows_per_bag[k] = [(row values as Fractions, weight)]"""
    acc_fmt = FMT[pl.ACC_F64] if t == pl.ACC_F64 else FMT[pl.ACC_F32]
    out = []
    for rows in rows_per_bag:
        disp = len(rows[0][0]) if rows else None
        out.append([])
        for e in range(disp or 0):
            acc = Fraction(0)
            for x, w in rows:
                acc = rnd(acc + (w * x[e] if w is not None else x[e]), acc_fmt)
            if mode == pl.POOL_MEAN:
                acc = rnd(acc / len(rows), acc_fmt)
            out[-1].append(to_bits(rnd(acc, FMT[t]), t))
    return out


def finite_values(rng, t, n, lo=-6, hi=6):
    """n finite values of type t with every bit of the significand used, over exponents lo..hi, some subnormal"""
    m = rng.uniform(1, 2, n) * rng.choice([-1.0, 1.0], n) * np.exp2(rng.integers(lo, hi, n))
    p, emin, _ = FMT[t]
    sub = rng.random(n) < 0.1
    m[sub] = rng.integers(1, 64, sub.sum()) * 2.0 ** (emin - p + 1)
    if t == pl.ACC_BF16:
        return pl.encode(m.astype(np.float32), t)
    return m.astype(pl.STORAGE[t])


def as_fractions(a, t):
    return [Fraction(float(v)) for v in pl.decode(a, t)]


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("mode", ["sum", "weighted", "mean"])
def test_oracle_matches_brute_force(t, mode):
    rng = np.random.default_rng(t * 10 + len(mode))
    disp, n = 3, 40
    shards = [finite_values(rng, t, 17 * disp).reshape(17, disp), finite_values(rng, t, 0).reshape(0, disp),
              finite_values(rng, t, 23 * disp).reshape(23, disp)]
    starts = rng.integers(0, 40, n)
    counts = rng.integers(0, 3, n)
    starts[5], counts[7] = 45, 30  # two invalid requests
    bags = np.sort(np.concatenate([[0, n], rng.integers(0, n, 12)]))
    w = finite_values(rng, t, n, -2, 2) if mode == "weighted" else None
    pm = pl.POOL_MEAN if mode == "mean" else pl.POOL_SUM
    out, codes, err = pl.pool(shards, t, pm, bags=bags, weights=w, starts=starts, counts=counts)
    assert err == (codes[5], 5) and codes[5] and codes[7]
    allrows = np.concatenate(shards)
    wv = as_fractions(w, t) if w is not None else None
    per_bag = []
    for k in range(len(bags) - 1):
        rows = []
        for i in range(bags[k], bags[k + 1]):
            if codes[i]:
                continue
            for r in range(starts[i], starts[i] + counts[i]):
                rows.append((as_fractions(allrows[r], t), wv[i] if wv else None))
        per_bag.append(rows)
    exp = brute(per_bag, t, pl.POOL_MEAN if mode == "mean" else pl.POOL_SUM)
    for k, row in enumerate(exp):
        got = out[k].astype(np.uint64).tolist() if row else [0] * disp
        assert got == (row or [0] * disp), (k, got, row)


@pytest.mark.parametrize("t", TYPES)
def test_exact_sums_any_order(t):
    """integer-valued rows whose every partial sum is exact in the accumulator: the fold equals the exact sum"""
    rng = np.random.default_rng(t)
    disp = 5
    vals = rng.integers(-8, 9, (300, disp)).astype(np.float64)
    shard = pl.encode(vals.astype(np.float32), t) if t == pl.ACC_BF16 else vals.astype(pl.STORAGE[t])
    ids = rng.integers(0, 300, 200)
    bags = np.array([0, 0, 1, 33, 200])
    out, _, err = pl.pool([shard], t, pl.POOL_SUM, bags=bags, starts=ids, fixed_count=1)
    assert err == (0, -1)
    for k in range(4):
        exact = vals[ids[bags[k]:bags[k + 1]]].sum(axis=0)
        assert np.array_equal(pl.decode_bits(out[k], t), exact.astype(pl.acc_dtype(t)))
    assert not out[0].any()  # an empty bag is +0


def bits_of(v, t):
    if t == pl.ACC_BF16:
        return pl.encode(np.asarray(v, np.float32), t)
    return np.asarray(v, pl.STORAGE[t]).view(pl.BITS[t])


@pytest.mark.parametrize("t", TYPES)
def test_max_nan_and_signed_zeros(t):
    nan = bits_of([np.nan], t)[0] | 1  # a NaN with a payload: the first row's bits are kept as they are
    rows = np.stack([bits_of([np.nan, -0.0, 1.0, 0.0], t), bits_of([5.0, 0.0, np.nan, -0.0], t),
                     bits_of([7.0, 3.0, 0.5, -1.0], t)])
    rows[0, 0] = nan
    shard = rows if t == pl.ACC_BF16 else rows.view(pl.STORAGE[t])
    out, _, _ = pl.pool([shard], t, pl.POOL_MAX, bags=[0, 3, 4, 4], starts=[0, 1, 2, 1], fixed_count=1)
    assert out[0].tolist() == [nan, bits_of([3.0], t)[0], bits_of([1.0], t)[0], bits_of([0.0], t)[0]]
    assert out[1].tolist() == rows[1].tolist()  # one row: as it is, NaN and -0 included
    assert out[2].tolist() == [0, 0, 0, 0]      # empty: +0
    out, _, _ = pl.pool([shard], t, pl.POOL_MAX, bags=[0, 2], starts=[1, 0], fixed_count=1)
    assert out[0, 1] == bits_of([0.0], t)[0] and out[0, 3] == bits_of([-0.0], t)[0]  # the earlier zero stays


@pytest.mark.parametrize("t", TYPES)
def test_nan_results_are_canonical(t):
    big = {pl.ACC_F32: 3e38, pl.ACC_F64: 1e308, pl.ACC_F16: 6e4, pl.ACC_BF16: 3e38}[t]
    shard = bits_of([[np.inf, np.nan, big], [-np.inf, 1.0, big]], t)
    shard = shard if t == pl.ACC_BF16 else shard.view(pl.STORAGE[t])
    for mode in (pl.POOL_SUM, pl.POOL_MEAN):
        out, _, _ = pl.pool([shard], t, mode, bags=[0, 2], starts=[0, 1], fixed_count=1)
        assert out[0, 0] == out[0, 1] == pl.CANONICAL_NAN[t]
        if mode == pl.POOL_SUM:
            assert pl.decode_bits(out[0, 2:], t)[0] == np.inf  # overflow rounds to inf


def test_empty_and_malformed_bags():
    shard = np.arange(12, dtype=np.float32).reshape(6, 2) + 1
    out, _, err = pl.pool([shard], pl.ACC_F32, pl.POOL_MEAN, bags=[0, 0, 2, 2], starts=[0, 1], fixed_count=1)
    assert err == (0, -1) and out.view(np.float32).tolist() == [[0, 0], [2, 3], [0, 0]]
    for bags, k in (([0, 1, 3], 1), ([1, 0, 2], 0), ([-1, 1, 2], 0), ([0, 2, 1, 2], 1)):
        out, _, err = pl.pool([shard], pl.ACC_F32, pl.POOL_SUM, bags=bags, starts=[0, 1], fixed_count=1)
        assert err == (pl.CODE_BAG, k), bags
        assert not out[k].any()  # a malformed bag's row is zeros


def test_bag_error_precedes_request_errors():
    shard = np.ones((4, 2), np.float64)
    starts = [0, 9, 1, 2]  # request 1 is invalid, in a well-formed bag before the malformed one
    out, codes, err = pl.pool([shard], pl.ACC_F64, pl.POOL_SUM, bags=[0, 2, 1, 4], starts=starts, fixed_count=1)
    assert codes[1] == po.CODE_COUNT and err == (pl.CODE_BAG, 1)
    assert out.view(np.float64).tolist() == [[1, 1], [0, 0], [2, 2]]  # the valid requests of every good bag count
    _, _, err = pl.pool([shard], pl.ACC_F64, pl.POOL_SUM, bags=[0, 2, 4], starts=starts, fixed_count=1)
    assert err == (po.CODE_COUNT, 1)
    # requests no bag covers are not validated
    _, _, err = pl.pool([shard], pl.ACC_F64, pl.POOL_SUM, bags=[2, 4], starts=starts, fixed_count=1)
    assert err == (0, -1)


def test_weighted_sum_rounds_once():
    """fma(w, x, acc) differs from the product rounded first: w * x = 1 + 2^-11 + 2^-24 is not a float32"""
    w = np.float32(1 + 2 ** -12)
    got = pl.fma(w, w, np.float32(-1), np.float32)
    assert float(got) == 2 ** -11 + 2 ** -24
    assert float(np.float32(np.float32(w * w) - 1)) == 2 ** -11
    assert float(pl.fma(np.float64(1 + 2 ** -27), np.float64(1 + 2 ** -27), np.float64(-1), np.float64)) == \
        2 ** -26 + 2 ** -54


def test_header_and_bindings_declare_the_entries():
    hdr = open(os.path.join(ROOT, "include", "ddstore_b200.h")).read()
    for name in ("dds_get_batch_pooled", "dds_get_samples_pooled"):
        assert re.search(rf"\bint {name}\(", hdr) and name in _capi.SIGNATURES
    assert [f for f, _ in _capi.Pool._fields_] == ["mode", "dtype", "bags", "nbags", "weights"]
    for k, v in (("SUM", 1), ("MEAN", 2), ("MAX", 3)):
        assert re.search(rf"#define DDS_POOL_{k} {v}\b", hdr)
    hpp = open(os.path.join(ROOT, "include", "ddstore_b200.hpp")).read()
    assert "get_batch_pooled" in hpp and "get_samples_pooled" in hpp
    pyx = open(os.path.join(ROOT, "ddstore_b200", "cython", "pyddstore.pyx")).read()
    assert "def get_batch_pooled" in pyx


def test_geometry_helper_reports_zeros_without_a_device():
    """dds_pool_geometry, as dds_gather_geometry: no usable device, no geometry"""
    import ctypes as C
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    vb, ctas = C.c_int(-1), C.c_int(-1)
    sl, ns, w = C.c_int64(-1), C.c_int64(-1), C.c_int64(-1)
    for adjoint in (0, 1):
        _capi.lib().dds_pool_geometry(adjoint, 512, pl.ACC_F32, 100, 1, 0, C.byref(vb), C.byref(sl), C.byref(ns),
                                      C.byref(w), C.byref(ctas))
        assert (vb.value, sl.value, ns.value, w.value, ctas.value) == (0, 0, 0, 0, 0)
