"""The batched accumulate's NumPy oracle (tests/acc_oracle.py) against the compiled reference and on seeded worlds, and
the Python-side checks of accumulate_batch / accumulate_samples that need no device."""
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests import acc_oracle as ao
from tests import put_oracle as po
from tests import put_world as pw
from tests.test_put_cpu import _edge_requests

ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)


def _shards(rng, nrows, disp, t, lo=-20, hi=20):
    return [ao.encode(rng.integers(lo, hi, size=(n, disp)), t) for n in nrows]


def _src(rng, lenlist, disp, t, batch):
    return ao.layout_src(rng, lenlist, disp, t, batch)


def _naive(shards, src, t, batch):
    """element by element, in Python integers / floats: the oracle's rule restated"""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    disp = shards[0].shape[1]
    vals = ao.values(np.asarray(src, np.uint8).view(ao.STORAGE[t]), t).tolist()
    world = [ao.values(s, t).reshape(-1).tolist() for s in shards]
    o = 0
    for s, c, ok in po.requests(**batch):
        n = c * disp if ok and 0 < c <= rows else 0
        code = po.CODE_SAMPLE if not ok else po.locate(lenlist, s, c)[0]
        if code == 0:
            r = po.sortedsearch(lenlist, s)
            first = int(lenlist[r - 1]) if r else 0
            for k in range(n):
                world[r][(s - first) * disp + k] += vals[o + k]
        o += n
    out = []
    for w, sh in zip(world, shards):
        if t == ao.ACC_I32:
            w = [((x + 2**31) % 2**32) - 2**31 for x in w]
        elif t == ao.ACC_I64:
            w = [((x + 2**63) % 2**64) - 2**63 for x in w]
        out.append(ao.encode(np.array(w, np.float64 if t not in (ao.ACC_I32, ao.ACC_I64) else object).astype(
            np.int64 if t in (ao.ACC_I32, ao.ACC_I64) else np.float64), t).reshape(sh.shape))
    return out


@pytest.mark.parametrize("t", ALL)
@pytest.mark.parametrize("seed", range(4))
def test_oracle_edge_worlds(seed, t):
    """empty ranks, straddlers, out-of-range starts and counts, duplicates: the oracle equals the element-wise rule,
    reports the put's codes, and a short src applies nothing"""
    rng = np.random.default_rng([seed, t])
    nrows = [int(x) for x in rng.integers(0, 30, size=int(rng.integers(2, 5)))]
    nrows[int(rng.integers(0, len(nrows)))] += 1
    nrows[0] = 0 if seed % 2 else nrows[0]  # an empty first rank
    nrows.insert(1, 0)                       # an empty middle rank
    disp = int(rng.integers(1, 5))
    shards = _shards(rng, nrows, disp, t)
    lenlist = po.lenlist_of(shards)
    starts, counts = _edge_requests(rng, lenlist, 30)
    batch = {"starts": starts, "counts": counts}
    src = _src(rng, lenlist, disp, t, batch)
    new, codes, bad, total = ao.accumulate(shards, src, t, **batch)
    _, pcodes, pbad, ptotal = po.put([s.view(np.uint8) for s in shards], src, **batch)  # the put's checks and layout
    assert (codes, bad, total) == (pcodes, pbad, ptotal) and total == src.size
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, _naive(shards, src, t, batch)))
    short, codes2, bad2, _ = ao.accumulate(shards, src, t, src_bytes=src.size - 1, **batch)
    assert codes2 == codes and bad2 == bad
    if total:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(short, shards))


@pytest.mark.parametrize("t", ALL)
def test_oracle_sample_ids_fixed_count_and_duplicates(t):
    rng = np.random.default_rng(40 + t)
    shards = _shards(rng, [5, 0, 7], 3, t)
    lenlist = po.lenlist_of(shards)
    rs = np.array([0, 4, 5, 11, 3, 12], np.int64)
    rc = np.array([2, 3, 4, 1, -1, 1], np.int64)
    ids = np.array([0, 6, 2, -1, 2, 1, 3, 4, 5, 0], np.int64)  # ids 2 and 0 twice: both contributions count
    batch = {"sample_ids": ids, "table": (rs, rc)}
    src = _src(rng, lenlist, 3, t, batch)
    new, codes, bad, total = ao.accumulate(shards, src, t, **batch)
    assert codes[:4] == [0, po.CODE_SAMPLE, 0, po.CODE_SAMPLE] and bad == 1
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, _naive(shards, src, t, batch)))
    fixed = {"starts": np.array([0, 3, 11, 0, 5], np.int64), "fixed_count": 2}
    src = _src(rng, lenlist, 3, t, fixed)
    new, codes, bad, total = ao.accumulate(shards, src, t, **fixed)
    assert codes == [0, 0, po.CODE_COUNT, 0, 0] and bad == 2 and total == 5 * 2 * 3 * np.dtype(ao.STORAGE[t]).itemsize
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, _naive(shards, src, t, fixed)))


def test_integers_wrap_and_floats_round_once():
    i32 = ao.add(np.array([2**31 - 1, -2**31], np.int32), np.array([1, -1], np.int32), ao.ACC_I32)
    assert i32.tolist() == [-2**31, 2**31 - 1]
    i64 = ao.add(np.array([2**63 - 1], np.int64), np.array([2], np.int64), ao.ACC_I64)
    assert i64.tolist() == [-2**63 + 1]
    assert ao.values(ao.add(ao.encode([255], ao.ACC_BF16), ao.encode([1], ao.ACC_BF16), ao.ACC_BF16), ao.ACC_BF16) == 256
    assert ao.add(np.array([2047], np.float16), np.array([1], np.float16), ao.ACC_F16).tolist() == [2048.0]


@pytest.mark.parametrize("t", ALL)
@pytest.mark.parametrize("seed", range(3))
def test_order_does_not_matter(seed, t):
    """several writers' calls on a world with empty ranks, every writer hitting every owner's edges: any order of the
    calls gives the same world (exact data), and each call reports the same triple"""
    rng = np.random.default_rng([7, seed, t])
    nrows = [0, 9, 1, 0, 14][: 3 + seed]
    disp = 3
    shards = _shards(rng, nrows, disp, t)
    lenlist = po.lenlist_of(shards)
    calls = []
    for w in range(3):
        st, ct, _ = pw.edge_requests(rng, lenlist, w, first_bad=None if w == 0 else 2, body=8)
        batch = {"starts": st, "counts": ct}
        calls.append((_src(rng, lenlist, disp, t, batch), None, batch))
        if w == 1:
            s2, c2 = pw.dense_cover(rng, int(lenlist[-1]), min(5, int(lenlist[-1])))
            b2 = {"starts": s2, "counts": c2}
            calls.append((_src(rng, lenlist, disp, t, b2), None, b2))
    ref, triples = ao.accumulate_many(shards, calls, t)
    for perm in (rng.permutation(len(calls)) for _ in range(3)):
        got, tr = ao.accumulate_many(shards, [calls[i] for i in perm], t)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref))
        assert [tr[k] for k in np.argsort(perm)] == triples


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("t", (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64))
@pytest.mark.parametrize("seed", range(2))
def test_oracle_vs_compiled_reference(seed, t):
    """each valid request run on the reference as the owner's get of its rows, the addition, and the owner's update;
    the world read back with the reference's get() equals the oracle's"""
    rng = np.random.default_rng([100, seed, t])
    nrows = [int(x) for x in rng.integers(0, 20, size=3)]
    nrows[1] += 1
    disp = int(rng.integers(1, 4))
    shards = _shards(rng, nrows, disp, t, -1000, 1000)
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    starts, counts = _edge_requests(rng, lenlist, 25)
    batch = {"starts": starts, "counts": counts}
    src = _src(rng, lenlist, disp, t, batch)
    new, codes, _, _ = ao.accumulate(shards, src, t, **batch)
    dt = np.dtype(ao.STORAGE[t])
    w = O.RefWorld(len(shards))
    try:
        w.add("x", shards)
        o = 0
        for (s, n, _), code in zip(po.requests(**batch), codes):
            nb = n * disp * dt.itemsize if 0 < n <= rows else 0
            if code == 0 and nb:
                r = w.sortedsearch(lenlist, s)
                first = int(lenlist[r - 1]) if r else 0
                cur = np.empty((n, disp), dt)
                w.get(r, "x", cur, s)
                w.update(r, "x", ao.add(cur, src[o:o + nb].view(dt).reshape(n, disp), t), s - first)
            o += nb
        for r, sh in enumerate(new):
            if sh.shape[0] == 0:
                continue
            got = np.empty_like(sh)
            w.get((r + 1) % len(shards), "x", got, int(lenlist[r - 1]) if r else 0)
            assert got.tobytes() == sh.tobytes(), f"rank {r}"
    finally:
        w.close()


def test_wrong_expectations_are_named():
    """an expectation made wrong on purpose -- a dropped request, a duplicate counted once, an element off by one -- is
    reported at the right rank and global row"""
    rng = np.random.default_rng(5)
    t, disp = ao.ACC_I32, 4
    shards = _shards(rng, [6, 0, 9, 4], disp, t)
    lenlist = po.lenlist_of(shards)
    R = disp * 4
    batch = {"starts": np.array([2, 7, 7, 15, 18], np.int64), "counts": np.array([1, 2, 2, 3, 1], np.int64)}
    src = ao.layout_src(rng, lenlist, disp, t, batch, 1, 5)  # every contribution non-zero
    good, _, _, _ = ao.accumulate(shards, src, t, **batch)
    for r, sh in enumerate(good):
        assert ao.mismatch(sh, sh, r, lenlist, R, "same") is None
    # request 3 (rows 15..17, rank 3's rows 0..2: 15 = 6 + 0 + 9) dropped
    drop = {k: np.delete(v, 3) for k, v in batch.items()}
    src_drop = np.concatenate([src[:(1 + 2 + 2) * R], src[(1 + 2 + 2 + 3) * R:]])
    wrong, _, _, _ = ao.accumulate(shards, src_drop, t, **drop)
    msg = ao.mismatch(good[3], wrong[3], 3, lenlist, R, "dropped")
    assert msg and "rank 3" in msg and "global row 15" in msg
    # the duplicate request 2 counted once: rank 2 (global rows 6..14), row 7
    once = {k: np.delete(v, 2) for k, v in batch.items()}
    src_once = np.concatenate([src[:3 * R], src[5 * R:]])
    wrong, _, _, _ = ao.accumulate(shards, src_once, t, **once)
    msg = ao.mismatch(good[2], wrong[2], 2, lenlist, R, "duplicate")
    assert msg and "rank 2" in msg and "global row 7" in msg
    # one element off by one: rank 0 row 2, element 1
    bent = good[0].copy()
    bent[2, 1] += 1
    msg = ao.mismatch(good[0], bent, 0, lenlist, R, "element")
    assert msg and "rank 0" in msg and "global row 2" in msg and "byte 4" in msg


def test_accumulate_rejects_other_dtypes_before_the_call():
    from ddstore_b200.store import PyDDStore
    torch = pytest.importorskip("torch")
    for dt in (torch.uint8, torch.int16, torch.bool, torch.complex64):
        with pytest.raises(ValueError, match="is not one of"):
            PyDDStore._acc_type("x", torch.zeros(2, dtype=dt))
    for dt, code in ((torch.float32, 1), (torch.float64, 2), (torch.int32, 3), (torch.int64, 4), (torch.float16, 5),
                     (torch.bfloat16, 6)):
        assert PyDDStore._acc_type("x", torch.zeros(2, dtype=dt)) == code


def test_cpp_header_compiles(tmp_path):
    """DDStore::accumulate_batch<T>, its explicit-code overload and the dtype check of include/ddstore_b200.hpp build
    against the library (the program itself runs in the GPU module)"""
    from tests.test_gpu_accumulate import build_cpp_check
    build_cpp_check(tmp_path)


# ------------------------------------------------------------------------------------------------ the arithmetic
FLOATS = (ao.ACC_F32, ao.ACC_F64, ao.ACC_F16, ao.ACC_BF16)


def _torch_add(a, b, t):
    """a + b by torch on the CPU, as storage bits"""
    torch = pytest.importorskip("torch")
    if t == ao.ACC_BF16:
        ta, tb = (torch.from_numpy(x.view(np.int16).copy()).view(torch.bfloat16) for x in (a, b))
        return (ta + tb).view(torch.int16).numpy().view(np.uint16)
    return (torch.from_numpy(a.copy()) + torch.from_numpy(b.copy())).numpy()


def _round(q, t):
    """the exact rational q rounded to nearest-even in type t (subnormals, overflow to inf): a restatement from scratch"""
    if q == 0:
        return 0.0
    p, emin = ao.PREC[t], ao.EMIN[t]
    mx = float(ao.values(ao.from_bits(np.array([ao._max_bits(t)], ao.BITS[t]), t), t)[0])
    e = abs(q).numerator.bit_length() - abs(q).denominator.bit_length()
    while Fraction(2) ** e > abs(q):  # (the bit lengths give it within one)
        e -= 1
    while Fraction(2) ** (e + 1) <= abs(q) and e >= emin:
        e += 1
    e = max(e, emin)
    ulp = Fraction(2) ** (e - p + 1)
    m = q / ulp
    r = round(m)  # Python rounds halves to even
    v = r * ulp
    if abs(v) > mx:
        return math.inf if q > 0 else -math.inf
    return float(v)


@pytest.mark.parametrize("t", FLOATS)
def test_one_addition_matches_torch(t):
    """`add` is torch's CPU addition bit for bit (NaN by class) on random bit pairs over the whole range and on every
    value family the GPU module uses"""
    rng = np.random.default_rng(11 + t)
    a = ao.from_bits(ao._finite_bits(rng, 50000, t), t)
    b = ao.from_bits(ao._finite_bits(rng, 50000, t), t)
    pairs = [("random bits", a, b)]
    # random bit pairs of nearby exponents, where the sum actually rounds
    b2 = ao.from_bits(ao.bits(a, t) ^ rng.integers(0, 1 << (ao.PREC[t] + 2), size=a.size).astype(ao.BITS[t]), t)
    pairs.append(("near exponents", a, b2))
    pairs += [(name, x, y) for name, (x, y) in ao.families(rng, t, 4000).items()]
    for name, x, y in pairs:
        got, exp = ao.keys(ao.add(x, y, t), t), ao.keys(_torch_add(x, y, t), t)
        d = np.nonzero(got != exp)[0]
        assert not d.size, f"{ao.NAMES[t]} {name}: {d.size} differ, first {ao.bits(x, t)[d[0]]:#x} + {ao.bits(y, t)[d[0]]:#x}"


@pytest.mark.parametrize("t", FLOATS)
def test_one_addition_matches_exact_fractions(t):
    """spot check: `add` of finite operands is the exact rational sum rounded once to nearest-even"""
    rng = np.random.default_rng(21 + t)
    fam = ao.families(rng, t, 300)
    a = np.concatenate([ao.from_bits(ao._finite_bits(rng, 300, t), t)] + [x for k, (x, _) in fam.items() if k != "inf nan"])
    b = np.concatenate([ao.from_bits(ao._finite_bits(rng, 300, t), t)] + [y for k, (_, y) in fam.items() if k != "inf nan"])
    r = ao.values(ao.add(a, b, t), t)
    va, vb = ao.values(a, t), ao.values(b, t)
    for i in range(a.size):
        q = Fraction(float(va[i])) + Fraction(float(vb[i]))
        e = _round(q, t)
        if q == 0:  # the sign of an exact zero sum: -0 only for (-0) + (-0)
            e = -0.0 if math.copysign(1, va[i]) < 0 and math.copysign(1, vb[i]) < 0 else 0.0
        assert r[i] == e and math.copysign(1, r[i]) == math.copysign(1, e), (ao.NAMES[t], va[i], vb[i], r[i], e)


def test_f32_flush_model():
    f = lambda *v: np.array(v, np.float32)  # noqa: E731
    mn, sub = np.float32(2.0 ** -126), np.float32(2.0 ** -149)
    assert ao.admissible(mn - sub, [sub], ao.ACC_F32) == {int(ao.keys(f(mn), 1)[0]), 0}  # max sub + min sub: min normal or +0
    assert ao.admissible(mn, [-sub], ao.ACC_F32) == {int(ao.keys(f(mn - sub), 1)[0]), int(ao.keys(f(mn), 1)[0])}
    assert ao.admissible(np.float32(-1e-40), [np.float32(-1e-40)], ao.ACC_F32) == {int(ao.keys(f(np.float32(-1e-40) * 2), 1)[0]),
                                                                               0x80000000}  # flushed: -0
    assert ao.admissible(np.float32(1.5), [np.float32(1e-45)], ao.ACC_F32) == {int(ao.keys(f(1.5), 1)[0])}
    # normals cancelling to a subnormal: the IEEE subnormal or +-0 of its sign
    x = np.float32(1.25 * 2.0 ** -126)
    r = ao.admissible(x, [-np.nextafter(x, np.float32(0))], ao.ACC_F32)
    assert r == {int(ao.keys(f(sub), 1)[0]), 0}
    # the model is the f32 path only: f16 / bf16 / f64 admit the IEEE result alone
    for t in (ao.ACC_F16, ao.ACC_BF16, ao.ACC_F64):
        s = ao.encode([2.0 ** (ao.EMIN[t] - 2)], t)
        assert len(ao.admissible(s[0], [s[0]], t)) == 1


@pytest.mark.parametrize("t", FLOATS)
def test_admissible_holds_every_order(t):
    """every sequential order of one-rounding additions is admissible; on the GPU module's data a stated fraction of
    elements with two or three contributions has more than one admissible result"""
    rng = np.random.default_rng(31 + t)
    n = 3000
    start = ao.inexact(rng, n, t)
    cs = [ao.inexact(rng, n, t) for _ in range(3)]
    for k in (2, 3):
        opts = ao.admissible_all(start, cs[:k], t)
        for order in itertools.permutations(range(k)):
            acc = start
            for i in order:
                acc = ao.add(acc, cs[i], t)
            assert (opts == ao.keys(acc, t)[None]).any(0).all(), (k, order)
        frac = float((opts != opts[0]).any(0).mean())
        assert frac > ao.DISCRIMINATION, (ao.NAMES[t], k, frac)
    if t == ao.ACC_F32:  # on subnormal data: the IEEE and the flushed sequential sums are both admissible
        fam = ao.families(rng, t, 2000)["subnormal"]
        opts = ao.admissible_all(fam[0], [fam[1], fam[0]], t)
        for fn in (lambda x, y: ao.add(x, y, t), ao.add_flushed):
            assert (opts == ao.keys(fn(fn(fam[0], fam[1]), fam[0]), t)[None]).any(0).all()


@pytest.mark.parametrize("t", FLOATS)
def test_sum_bound_is_below_one_contribution(t):
    """for the hot-element data (HOT contributions of random sign in [1, 4)), the bound is below the smallest
    contribution, so a lost contribution cannot hide inside it; every sequential sum meets it"""
    rng = np.random.default_rng(41 + t)
    n, disp = ao.HOT[t], 5 if t != ao.ACC_F64 else 2
    start = ao.inexact(rng, disp, t, 0, 1)
    cs = ao.inexact(rng, (n, disp), t, 0, 1)
    s, bound = ao.sum_bound(start, cs, t)
    assert (bound < np.abs(ao.values(cs, t)).min(0)).all(), (bound, ao.NAMES[t])
    for perm in (np.arange(n), rng.permutation(n)):
        acc = start
        for i in perm:
            acc = ao.add(acc, cs[i], t)
        assert (np.abs(ao.values(acc, t) - s) <= bound).all()
        dropped = ao.values(acc, t) - ao.values(cs[perm[0]], t)
        assert (np.abs(dropped - s) > bound).all()


def _where(D, row0=100, rank=2):
    return lambda i: (rank, row0 + i // D, i % D)


def _first_outside(got, start, contribs, t):
    """the index of the first element outside its admissible set, found element by element with `admissible`"""
    g = ao.keys(got, t)
    for i in range(g.size):
        if int(g[i]) not in ao.admissible(start[i], [c[i] for c in contribs], t):
            return i
    return None


@pytest.mark.parametrize("wrong", ["truncation", "flushed", "bf16 pair in f32", "dropped", "-0 as +0"])
def test_wrong_arithmetic_is_named(wrong):
    """a result made wrong on purpose is reported at the right rank, global row and column, with the element's inputs,
    the bits it got and the admissible bits"""
    rng = np.random.default_rng(51)
    D = 7
    if wrong == "truncation":  # round toward zero: the RNE result moved one ulp toward zero where it rounded away
        t = ao.ACC_F32
        start, c = ao.inexact(rng, 700, t), ao.inexact(rng, 700, t)
        r = ao.add(start, c, t)
        exact = ao.values(start, t) + ao.values(c, t)  # (exact in f64: exponents within a few binades)
        away = np.abs(ao.values(r, t)) > np.abs(exact)
        got = np.where(away, np.nextafter(r, np.float32(0)), r)
        contribs = [c]
    elif wrong == "flushed":  # f16 and bf16 subnormal inputs and results flushed to signed zero
        for t in (ao.ACC_F16, ao.ACC_BF16):
            a, b = ao.families(rng, t, 700)["subnormal"]
            v = ao.values(ao.add(a, b, t), t)
            got = ao.encode(np.where(np.abs(v) < ao.min_normal(t), np.copysign(0.0, v), v), t)
            i = _first_outside(got, a, [b], t)
            msg = ao.verdict(got, a, [b], t, where=_where(D), what=wrong)
            assert i is not None and msg and f"global row {100 + i // D}, column {i % D}" in msg, msg
        return
    elif wrong == "bf16 pair in f32":  # start + (c1 + c2) with the pair combined in f32, rounded once at the end
        t = ao.ACC_BF16
        start, c1, c2 = ao.inexact(rng, 700, t), ao.inexact(rng, 700, t), ao.inexact(rng, 700, t)
        got = ao.f32_to_bf16(ao.bf16_to_f32(start) + (ao.bf16_to_f32(c1) + ao.bf16_to_f32(c2)))
        contribs = [c1, c2]
    elif wrong == "dropped":
        t = ao.ACC_F64
        start, c1, c2 = ao.inexact(rng, 700, t), ao.inexact(rng, 700, t), ao.inexact(rng, 700, t)
        got = ao.add(start, c1, t)
        contribs = [c1, c2]
    else:
        t = ao.ACC_F16
        start, c = ao.families(rng, t, 700)["zeros"]
        r = ao.add(start, c, t)
        got = np.where(ao.bits(r, t) == 0x8000, np.float16(0), r)
        contribs = [c]
    i = _first_outside(got, start, contribs, t)
    assert i is not None, wrong
    msg = ao.verdict(got, start, contribs, t, where=_where(D), paths=np.array(["vector"] * start.size), what=wrong)
    assert msg and f"rank 2, global row {100 + i // D}, column {i % D} (path vector)" in msg, msg
    assert f"got {int(ao.keys(got[i:i + 1], t)[0]) & ((1 << 8 * np.dtype(ao.BITS[t]).itemsize) - 1):#0{2 + 2 * np.dtype(ao.BITS[t]).itemsize}x}" in msg, msg
    assert ao.verdict(ao.add(start, contribs[0], t) if len(contribs) == 1 else
                      ao.add(ao.add(start, contribs[0], t), contribs[1], t), start, contribs, t) is None


def test_bf16_nan_encoding():
    """NaNs stay NaNs, quieted, whatever their payload; inf, overflow and ordinary values round to nearest-even"""
    b = np.array([0x7F800001, 0xFF800001, 0x7FC00000, 0x7FFFFFFF, 0x7F80FFFF, 0xFFC12345, 0x7F800000, 0xFF800000,
                  0x7F7FFFFF, 0x3F808000, 0x3F818000, 0x00000001], np.uint32)
    got = ao.f32_to_bf16(b.view(np.float32)).tolist()
    assert got == [0x7FC0, 0xFFC0, 0x7FC0, 0x7FFF, 0x7FC0, 0xFFC1, 0x7F80, 0xFF80, 0x7F80, 0x3F80, 0x3F82, 0x0000]
    assert all(np.isnan(ao.bf16_to_f32(np.array(got[:6], np.uint16))))
    assert np.isnan(ao.values(ao.add(np.array([0x7F81], np.uint16), np.array([0x3F80], np.uint16), ao.ACC_BF16),
                              ao.ACC_BF16)).all()


def test_drain_path():
    """write_chunk<kActReduce>'s cases, element by element: head and tail elements, a same-phase body in bulk, a re-phased body
    in vectors"""
    lab = lambda dp, sp, n: "".join(x[0] for x in ao.drain_path(dp, sp, n, np.arange(0, n, 4)))  # noqa: E731
    assert lab(0, 0, 64) == "b" * 16
    assert lab(4, 4, 40) == "eee" + "bbbb" + "eee"
    assert lab(4, 0, 40) == "eee" + "vvvv" + "eee"
    assert lab(0, 8, 20) == "vvvv" + "e"
    assert lab(12, 0, 8) == "e" + "e"          # head then tail: no body
    assert lab(8, 8, 8) == "ee"                # the head takes the whole piece
