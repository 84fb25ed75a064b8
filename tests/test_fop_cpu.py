"""The batched fetch-op's NumPy oracle (tests/fop_oracle.py) against the compiled reference and on seeded worlds, its
chain checkers against results made wrong on purpose, and the Python-side checks of get_accumulate_batch that need no
device. The second half checks the arithmetic checkers the GPU numerics module relies on: that they accept every order
of fetch-adds simulated with one rounding per step (f32: IEEE or flushed) on every value family, that they name the
element of each kind of wrong result (an ulp off, rounded toward zero, a flushed subnormal, a changed NaN payload, a
quieted signalling NaN, a duplicated ticket), that the hot-element generators raise every sum, and fop_path."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests import acc_oracle as ao
from tests import fop_oracle as fo
from tests import put_oracle as po
from tests.test_put_cpu import _edge_requests

ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)
OPS = (fo.OP_SUM, fo.OP_REPLACE)


def _shards(rng, nrows, disp, t, lo=-20, hi=20):
    return [ao.encode(rng.integers(lo, hi, size=(n, disp)), t) for n in nrows]


def _naive(shards, src, result, t, op, batch):
    """element by element, in request order: the rule restated (new shards, new result)"""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    disp = shards[0].shape[1]
    dt = np.dtype(ao.STORAGE[t])
    x = np.asarray(src, np.uint8).view(dt)
    world = [s.reshape(-1).copy() for s in shards]
    res = np.array(result, np.uint8).view(dt).copy()
    o = 0
    for s, c, ok in po.requests(**batch):
        n = c * disp if ok and 0 < c <= rows else 0
        if (po.CODE_SAMPLE if not ok else po.locate(lenlist, s, c)[0]) == 0:
            r = po.sortedsearch(lenlist, s)
            first = int(lenlist[r - 1]) if r else 0
            for k in range(n):
                e = (s - first) * disp + k
                res[o + k] = world[r][e]
                world[r][e] = ao.add(world[r][e:e + 1], x[o + k:o + k + 1], t)[0] if op == fo.OP_SUM else x[o + k]
        o += n
    return [w.reshape(sh.shape) for w, sh in zip(world, shards)], res.view(np.uint8)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("t", ALL)
@pytest.mark.parametrize("seed", range(3))
def test_oracle_edge_worlds(seed, t, op):
    """empty ranks, straddlers, out-of-range starts and counts, duplicates: the oracle equals the element-wise rule,
    reports the put's codes and layout, leaves an invalid request's result bytes alone, and a short src applies
    nothing and writes no result"""
    rng = np.random.default_rng([seed, t, op])
    nrows = [int(x) for x in rng.integers(0, 30, size=int(rng.integers(2, 5)))]
    nrows[int(rng.integers(0, len(nrows)))] += 1
    nrows[0] = 0 if seed % 2 else nrows[0]  # an empty first rank
    nrows.insert(1, 0)                       # an empty middle rank
    disp = int(rng.integers(1, 5))
    shards = _shards(rng, nrows, disp, t)
    lenlist = po.lenlist_of(shards)
    starts, counts = _edge_requests(rng, lenlist, 30)
    batch = {"starts": starts, "counts": counts}
    src = ao.layout_src(rng, lenlist, disp, t, batch)
    result = rng.integers(0, 256, size=src.size + 16, dtype=np.uint8)  # a sentinel past the layout
    new, res, codes, bad, total = fo.fetch_op(shards, src, t, op, result, **batch)
    _, pcodes, pbad, ptotal = po.put([s.view(np.uint8) for s in shards], src, **batch)
    assert (codes, bad, total) == (pcodes, pbad, ptotal) and total == src.size
    nnew, nres = _naive(shards, src, result, t, op, batch)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, nnew)) and res.tobytes() == nres.tobytes()
    assert res[src.size:].tobytes() == result[src.size:].tobytes()
    _, pl, _, _, _ = fo.plan(shards, t, src.size, **batch)
    for (_r, _l, _c, off, n), code in zip(pl, codes):
        if code:
            assert res[off:off + n].tobytes() == result[off:off + n].tobytes()
    short, sres, codes2, bad2, _ = fo.fetch_op(shards, src, t, op, result, src_bytes=src.size - 1, **batch)
    assert codes2 == codes and bad2 == bad
    if total:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(short, shards)) and sres.tobytes() == result.tobytes()


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("t", ALL)
def test_oracle_sample_ids_fixed_count_and_duplicates(t, op):
    """bad sample ids keep 0 bytes; duplicate ids apply twice, the second seeing the first's value; a fixed count past
    the end is a count error"""
    rng = np.random.default_rng([40, t, op])
    shards = _shards(rng, [5, 0, 7], 3, t)
    lenlist = po.lenlist_of(shards)
    rs = np.array([0, 4, 5, 11, 3, 12], np.int64)
    rc = np.array([2, 3, 4, 1, -1, 1], np.int64)
    ids = np.array([0, 6, 2, -1, 2, 1, 3, 4, 5, 0], np.int64)
    batch = {"sample_ids": ids, "table": (rs, rc)}
    src = ao.layout_src(rng, lenlist, 3, t, batch, 1, 5)
    result = np.zeros(src.size, np.uint8)
    new, res, codes, bad, total = fo.fetch_op(shards, src, t, op, result, **batch)
    assert codes[:4] == [0, po.CODE_SAMPLE, 0, po.CODE_SAMPLE] and bad == 1
    nnew, nres = _naive(shards, src, result, t, op, batch)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, nnew)) and res.tobytes() == nres.tobytes()
    # the second request of id 2 got what the first left
    E = np.dtype(ao.STORAGE[t]).itemsize
    R = 3 * E
    first, second = 2 * R, (2 + 4) * R  # layout: id 0 (2 rows), id 6 (0), id 2 (4 rows), id -1 (0), id 2
    exp = ao.add(shards[2][0:4], src[first:first + 4 * R].view(ao.STORAGE[t]).reshape(4, 3), t) if op == fo.OP_SUM \
        else src[first:first + 4 * R].view(ao.STORAGE[t]).reshape(4, 3)
    assert res[second:second + 4 * R].tobytes() == exp.tobytes()
    fixed = {"starts": np.array([0, 3, 11, 0, 5], np.int64), "fixed_count": 2}
    src = ao.layout_src(rng, lenlist, 3, t, fixed)
    new, res, codes, bad, total = fo.fetch_op(shards, src, t, op, np.zeros(src.size, np.uint8), **fixed)
    assert codes == [0, 0, po.CODE_COUNT, 0, 0] and bad == 2 and total == 5 * 2 * R
    assert not res[2 * 2 * R:3 * 2 * R].any()


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("t", (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64))
@pytest.mark.parametrize("seed", range(2))
def test_oracle_vs_compiled_reference(seed, t, op):
    """each valid request run on the reference as the owner's get of its rows (the previous rows), the addition or the
    copy, and the owner's update; the previous rows and the world read back with get() equal the oracle's"""
    rng = np.random.default_rng([100, seed, t, op])
    nrows = [int(x) for x in rng.integers(0, 20, size=3)]
    nrows[1] += 1
    disp = int(rng.integers(1, 4))
    shards = _shards(rng, nrows, disp, t, -1000, 1000)
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    starts, counts = _edge_requests(rng, lenlist, 25)
    batch = {"starts": starts, "counts": counts}
    src = ao.layout_src(rng, lenlist, disp, t, batch)
    result = rng.integers(0, 256, size=src.size, dtype=np.uint8)
    new, res, codes, _, _ = fo.fetch_op(shards, src, t, op, result, **batch)
    dt = np.dtype(ao.STORAGE[t])
    ref_res = result.copy()
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
                ref_res[o:o + nb] = cur.reshape(-1).view(np.uint8)
                x = src[o:o + nb].view(dt).reshape(n, disp)
                w.update(r, "x", ao.add(cur, x, t) if op == fo.OP_SUM else x.copy(), s - first)
            o += nb
        assert ref_res.tobytes() == res.tobytes()
        for r, sh in enumerate(new):
            if sh.shape[0] == 0:
                continue
            got = np.empty_like(sh)
            w.get((r + 1) % len(shards), "x", got, int(lenlist[r - 1]) if r else 0)
            assert got.tobytes() == sh.tobytes(), f"rank {r}"
    finally:
        w.close()


# ------------------------------------------------------------------------------------------------ the checkers
def _hot_world(t, op, k=6):
    """two elements hit by k fetch-ops (one per call; positive or distinct operands), plus a once-touched row; the
    oracle's (sequential) outcome"""
    shards = [ao.encode(np.arange(8).reshape(4, 2) + 10, t), ao.encode(np.arange(6).reshape(3, 2) + 50, t)]
    calls = []
    for j in range(k):
        src = ao.encode(np.array([[j + 1, 2 * j + 1] if op == fo.OP_SUM else [100 + j, 120 + j]]), t).view(np.uint8).reshape(-1)
        calls.append((src, None, np.zeros(src.size, np.uint8), {"starts": [5], "counts": [1]}))
    src = ao.encode(np.array([[7, 8]]), t).view(np.uint8).reshape(-1)
    calls.append((src, None, np.zeros(src.size, np.uint8), {"starts": [1], "counts": [1]}))
    new, results, _ = fo.fetch_op_many(shards, calls, t, op)
    return shards, calls, new, results


def _elem(results, k, t, j):
    return results[k].view(ao.STORAGE[t])[j]


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("t", (ao.ACC_I32, ao.ACC_I64, ao.ACC_F32, ao.ACC_F64, ao.ACC_F16, ao.ACC_BF16))
def test_checker_accepts_every_order(t, op):
    """the oracle's own outcome, and the outcome of the hot element's fetch-ops in reverse order, both pass"""
    shards, calls, new, results = _hot_world(t, op)
    assert fo.check(shards, calls, t, op, new, results) is None
    rev = list(reversed(calls[:-1])) + calls[-1:]
    new2, results2, _ = fo.fetch_op_many(shards, rev, t, op)
    back = list(reversed(results2[:-1])) + results2[-1:]
    assert fo.check(shards, calls, t, op, new2, back) is None


@pytest.mark.parametrize("op", OPS)
def test_checker_names_a_duplicated_ticket_and_a_lost_contribution(op):
    t = ao.ACC_I64
    shards, calls, new, results = _hot_world(t, op)
    dup = [r.copy() for r in results]
    dup[2].view(np.int64)[0] = _elem(results, 1, t, 0)  # two fetch-ops got the same previous value
    msg = fo.check(shards, calls, t, op, new, dup)
    assert msg and "rank 1 global row 5 column 0" in msg and ("same value" in msg or "both got" in msg), msg
    lost = [s.copy() for s in new]
    lost[1][1, 0] = _elem(results, 5, t, 0)  # the last contribution lost: final = what the last fetch-op got
    msg = fo.check(shards, calls, t, op, lost, results)
    assert msg and "rank 1 global row 5" in msg and "final value" in msg, msg


@pytest.mark.parametrize("op", OPS)
def test_checker_names_a_value_outside_the_chain(op):
    t = ao.ACC_I32
    shards, calls, new, results = _hot_world(t, op)
    bent = [r.copy() for r in results]
    bent[3].view(np.int32)[0] = 999
    msg = fo.check(shards, calls, t, op, new, bent)
    assert msg and "rank 1 global row 5 column 0" in msg, msg
    # a once-touched element: the previous value and the new value are compared exactly
    bent = [r.copy() for r in results]
    bent[-1].view(np.int32)[1] += 1
    msg = fo.check(shards, calls, t, op, new, bent)
    assert msg and "previous value: rank 0 global row 1 column 1" in msg, msg
    wrong = [s.copy() for s in new]
    wrong[0][1, 0] += 1
    msg = fo.check(shards, calls, t, op, wrong, results)
    assert msg and "new value: rank 0 global row 1 column 0" in msg, msg
    wrong = [s.copy() for s in new]
    wrong[0][3, 1] += 1
    msg = fo.check(shards, calls, t, op, wrong, results)
    assert msg and "no request touches" in msg and "global row 3 column 1" in msg, msg


@pytest.mark.parametrize("op", OPS)
def test_checker_names_a_result_written_for_an_invalid_request(op):
    t = ao.ACC_F32
    rng = np.random.default_rng(9)
    shards = _shards(rng, [6, 0, 9], 2, t)
    batch = {"starts": np.array([1, 14, 3], np.int64), "counts": np.array([2, 2, 1], np.int64)}  # 14 + 2 > 15
    src = ao.layout_src(rng, po.lenlist_of(shards), 2, t, batch)
    result = np.full(src.size, 0xA5, np.uint8)
    calls = [(src, None, result, batch)]
    new, results, out = fo.fetch_op_many(shards, calls, t, op)
    assert out[0][:2] == (po.CODE_COUNT, 1)
    assert fo.check(shards, calls, t, op, new, results) is None
    bad = [results[0].copy()]
    bad[0][2 * 8 + 5] = 0  # inside request 1's bytes
    msg = fo.check(shards, calls, t, op, new, bad)
    assert msg and "request 1" in msg and "written outside" in msg, msg
    # a capacity error: nothing may be written at all
    calls = [(src, src.size - 1, result, batch)]
    new, results, _ = fo.fetch_op_many(shards, calls, t, op)
    assert results[0].tobytes() == result.tobytes()
    bad = [results[0].copy()]
    bad[0][0] = 0
    assert "written outside" in fo.check(shards, calls, t, op, new, bad)


def test_chain_checkers_directly():
    assert fo.sum_chain(5, [1, 1, 1], [6, 5, 7], 8) is None
    assert "same value" in fo.sum_chain(5, [1, 1, 1], [5, 5, 6], 8)
    assert "final value" in fo.sum_chain(5, [1, 1, 1], [6, 5, 7], 7)
    assert "chain expects" in fo.sum_chain(5, [2, 1], [5, 8], 8)
    assert fo.replace_chain(0, [10, 11, 12], [11, 0, 10], 12) is None
    assert "both got" in fo.replace_chain(0, [10, 11, 12], [0, 0, 10], 12)
    assert "no fetch-op got" in fo.replace_chain(0, [10, 11, 12], [11, 3, 10], 12)
    assert "final value" in fo.replace_chain(0, [10, 11, 12], [11, 0, 10], 11)


# ------------------------------------------------------------------------------------------------ bindings
def test_fetch_op_rejects_bad_arguments_before_the_call():
    from ddstore_b200.store import PyDDStore
    from ddstore_b200 import _capi
    torch = pytest.importorskip("torch")

    class _Src:
        nbytes = 64
    with pytest.raises(ValueError, match="is not one of"):
        PyDDStore._fop_args("x", "max", None, _Src())
    with pytest.raises(ValueError, match="CUDA tensor"):
        PyDDStore._fop_args("x", "sum", torch.zeros(16), _Src())
    assert (_capi.OP_SUM, _capi.OP_REPLACE) == (1, 2) and _capi.FOP_OPS == {"sum": 1, "replace": 2}


# ------------------------------------------------------------------------------------------------ the arithmetic
FLOATS = (ao.ACC_F32, ao.ACC_F64, ao.ACC_F16, ao.ACC_BF16)


def _simulate(rng, t, start, contribs):
    """each element's fetch-adds in a random order, each f32 step IEEE or flushed at random -> (previous values [k,
    N], final [N])"""
    k, n = len(contribs), start.size
    orders = np.argsort(rng.random((n, k)), axis=1)
    modes = rng.random((n, k)) < 0.5 if t == ao.ACC_F32 else np.zeros((n, k), bool)
    cur, prev = start.copy(), np.empty((k, n), start.dtype)
    X = np.stack(contribs)
    for step in range(k):
        i = orders[:, step]
        x = X[i, np.arange(n)]
        prev[i, np.arange(n)] = cur
        cur = np.where(modes[:, step], ao.add_flushed(cur, x) if t == ao.ACC_F32 else cur, ao.add(cur, x, t))
    return prev, cur


def _family_world(t, k, seed=0, n=64):
    """n elements per value family, k fetch-adds each (one call per fetch-add, one request of row 0): (names, family
    of each element, start, contribs, shards, calls) with the calls' results still to fill in"""
    rng = np.random.default_rng([seed, t, k])
    fams = ao.families(rng, t, n)
    names = list(fams)
    start = np.concatenate([fams[nm][0] for nm in names])
    contribs = [np.concatenate([ao.families(rng, t, n)[nm][1] for nm in names]) for _ in range(k)]
    fam = np.repeat(np.array(names), n)
    return rng, names, fam, start, contribs


def _check_world(t, start, contribs, prev, final, op=fo.OP_SUM):
    """check() of one row holding every element, one call per fetch-op"""
    shards = [start[None].copy()]
    calls = [(c.view(np.uint8), None, np.zeros(c.nbytes, np.uint8), {"starts": [0], "counts": [1]}) for c in contribs]
    return fo.check(shards, calls, t, op, [final[None]], [p.copy().view(np.uint8) for p in prev])


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("t", ALL)
def test_fetch_checkers_accept_every_simulated_order(t, k):
    """on every value family, fetch-adds applied in random orders with ao.add / add_flushed: admissible_fetch holds
    every outcome, and so does check() (the chain walk, and the search where the walk is not enough)"""
    rng, names, fam, start, contribs = _family_world(t, k)
    for seed in range(3):
        prev, final = _simulate(rng, t, start, contribs)
        opts = fo.admissible_fetch(start, contribs, t)
        assert fo.fetch_match(opts, prev, final, t).all()
        assert fo.fetch_verdict(prev, final, start, contribs, t, opts=opts) is None
        assert _check_world(t, start, contribs, prev, final) is None
    # one plain accumulate beside one fetch-add, in either order
    acc = contribs[1]
    for first in (True, False):
        cur = ao.add(start, acc, t) if first else start
        prev = cur[None].copy()
        cur = ao.add(cur, contribs[0], t)
        final = cur if first else ao.add(cur, acc, t)
        assert fo.fetch_match(fo.admissible_fetch(start, contribs[:1], t, acc), prev, final, t).all()


def _W(i):
    return 0, 0, i


def _where_in(msg, e):
    return msg is not None and f"global row 0, column {e}:" in msg


def _first(mask):
    assert mask.any()
    return int(np.argmax(mask))


@pytest.mark.parametrize("t", FLOATS)
def test_fetch_checkers_report_wrong_arithmetic(t):
    """a previous value one ulp off, a final value rounded toward zero, two equal tickets on strictly increasing data:
    each reported at the right element, by fetch_verdict and by check()"""
    rng, names, fam, start, contribs = _family_world(t, 2, seed=1)
    prev, final = _simulate(rng, t, start, contribs)
    opts = fo.admissible_fetch(start, contribs, t)
    fin = ~ao.is_nan(prev, t).any(0) & np.isfinite(ao.values(final, t))
    # a previous value one ulp off
    e = _first(fin & (fam == "random"))
    bad = prev.copy()
    bad[1].view(ao.BITS[t])[e] += 1
    assert _where_in(fo.fetch_verdict(bad, final, start, contribs, t, opts=opts, where=_W), e)
    assert f"chain: rank 0 global row 0 column {e}" in _check_world(t, start, contribs, bad, final)
    # a final value rounded toward zero (one fetch-add: a once-touched element)
    x = contribs[0]
    rn = ao.add(start, x, t)
    ties = np.flatnonzero(fam == "ties")
    sv, xv, rv = (ao.values(a[ties], t) for a in (start, x, rn))
    up = np.array([abs(Fraction(float(r))) > abs(Fraction(float(a)) + Fraction(float(b))) for a, b, r in zip(sv, xv, rv)])
    e = int(ties[_first(up & (rv != 0))])
    rz = rn.copy()
    rz.view(ao.BITS[t])[e] -= 1
    msg = fo.once_verdict(start, rz, start, x, t, fo.OP_SUM, where=_W)
    assert _where_in(msg, e) and "new value" in msg, msg
    msg = _check_world(t, start, [x], [start], rz)
    assert msg and f"new value: rank 0 global row 0 column {e}" in msg, msg
    # two tickets equal on strictly increasing data
    rng = np.random.default_rng(5)
    v0 = fo.hot_values(rng, t, (3,))
    xs = fo.hot_values(rng, t, (40, 3))
    got, cur = np.empty_like(xs), v0.copy()
    for j in range(40):
        got[j], cur = cur, ao.add(cur, xs[j], t)
    assert fo.increasing_chain(v0, xs, got, cur, t) is None
    dup = got.copy()
    dup[17, 2] = dup[16, 2]
    bad = fo.increasing_chain(v0, xs, dup, cur, t)
    assert bad is not None and bad[0] == 2 and "duplicated ticket" in bad[1], bad
    calls = [(xs[j:j + 1].view(np.uint8).reshape(-1), None, np.zeros(xs[j:j + 1].nbytes, np.uint8),
              {"starts": [0], "counts": [1]}) for j in range(40)]
    assert fo.check([v0[None]], calls, t, fo.OP_SUM, [cur[None]], [g.view(np.uint8) for g in got]) is None
    msg = fo.check([v0[None]], calls, t, fo.OP_SUM, [cur[None]], [g.view(np.uint8) for g in dup])
    assert msg and "chain: rank 0 global row 0 column 2" in msg and "duplicated ticket" in msg, msg


@pytest.mark.parametrize("t", FLOATS)
def test_fetch_checkers_report_flushed_and_changed_bits(t):
    """a subnormal flushed (f16 / bf16 new values; any type's previous values, f32 included), a NaN payload changed in
    a previous value or a swap, a signalling NaN quieted by a swap: each reported at the right element"""
    rng = np.random.default_rng([2, t])
    n = 64
    p = ao.PREC[t]
    sub = ao.encode(rng.integers(1, 1 << (p - 1), size=n) * 2.0 ** (ao.EMIN[t] - p + 1), t)
    zero = ao.encode(np.zeros(n), t)
    # the shard holds subnormals; a sum of +0 keeps them: previous and new value are the subnormal
    assert fo.once_verdict(sub, sub, sub, zero, t, fo.OP_SUM, where=_W) is None
    e = 17
    flushed = sub.copy()
    flushed[e] = zero[e]
    msg = fo.once_verdict(flushed, sub, sub, zero, t, fo.OP_SUM, where=_W)
    assert _where_in(msg, e) and "previous value 0x0" in msg, msg
    msg = _check_world(t, sub, [zero], [flushed], sub)
    assert msg and f"previous value: rank 0 global row 0 column {e}" in msg, msg
    if t != ao.ACC_F32:  # (f32 may flush a subnormal result; f16 and bf16 may not)
        msg = fo.once_verdict(sub, flushed, sub, zero, t, fo.OP_SUM, where=_W)
        assert _where_in(msg, e) and "new value 0x0" in msg, msg
    else:
        assert fo.once_verdict(sub, flushed, sub, zero, t, fo.OP_SUM, where=_W) is None
    # NaN payloads: a previous value must keep the shard's payload; a swap's new value must be the operand's bits
    snan = ao.from_bits(np.full(n, ao._nan_bits(t, 1), ao.BITS[t]), t)    # signalling, payload 1
    qnan = ao.from_bits(np.full(n, ao._nan_bits(t, 3), ao.BITS[t]), t)    # quiet, payload 3
    quieted = ao.from_bits(ao.bits(snan, t) | ao.BITS[t](1 << (p - 2)), t)
    x = ao.inexact(rng, n, t)
    assert fo.once_verdict(qnan, ao.add(qnan, x, t), qnan, x, t, fo.OP_SUM, where=_W) is None
    bad = qnan.copy()
    bad[e] = ao.from_bits(np.array([ao._nan_bits(t, 0)], ao.BITS[t]), t)[0]
    assert _where_in(fo.once_verdict(bad, ao.add(qnan, x, t), qnan, x, t, fo.OP_SUM, where=_W), e)
    for op in (fo.OP_SUM, fo.OP_REPLACE):
        msg = _check_world(t, qnan, [x], [bad], ao.add(qnan, x, t) if op == fo.OP_SUM else x, op)
        assert msg and f"previous value: rank 0 global row 0 column {e}" in msg, msg
    assert fo.once_verdict(x, snan, x, snan, t, fo.OP_REPLACE, where=_W) is None
    got = snan.copy()
    got[e] = quieted[e]
    msg = fo.once_verdict(x, got, x, snan, t, fo.OP_REPLACE, where=_W)
    assert _where_in(msg, e) and "new value" in msg, msg
    msg = _check_world(t, x, [snan], [x], got, fo.OP_REPLACE)
    assert msg and f"new value: rank 0 global row 0 column {e}" in msg, msg
    # a swap chain v0 -> sNaN -> s1: the second swap got the sNaN quieted
    s1 = ao.inexact(rng, n, t)
    prev = [x.copy(), snan.copy()]
    assert _check_world(t, x, [snan, s1], prev, s1, fo.OP_REPLACE) is None
    prev[1][e] = quieted[e]
    msg = _check_world(t, x, [snan, s1], prev, s1, fo.OP_REPLACE)
    assert msg and f"chain: rank 0 global row 0 column {e}" in msg, msg


def test_f32_subnormal_previous_value_returned_as_zero():
    """an f32 subnormal start touched by two fetch-adds of +0: the first must get the subnormal back bit for bit,
    although the sums may flush it"""
    t = ao.ACC_F32
    sub = ao.from_bits(np.array([1, 0x80000005, 0x007FFFFF], np.uint32), t)
    zero = np.zeros(3, np.float32)
    prev, final = [sub.copy(), ao.add_flushed(sub, zero)], ao.add_flushed(sub, zero)
    assert _check_world(t, sub, [zero, zero], prev, final) is None
    assert fo.fetch_match(fo.admissible_fetch(sub, [zero, zero], t), np.stack(prev), final, t).all()
    prev[0] = np.copysign(zero, sub)
    msg = _check_world(t, sub, [zero, zero], prev, final)
    assert msg and "chain: rank 0 global row 0 column 0" in msg, msg
    ok = fo.fetch_match(fo.admissible_fetch(sub, [zero, zero], t), np.stack(prev), final, t)
    assert not ok.any()


@pytest.mark.parametrize("t", ALL)
def test_hot_generators_raise_every_sum(t):
    """HOT_FETCH[t] fetch-adds of hot_values onto a hot_values start, in order: every addition raises the running sum,
    also when every operand is the largest or the smallest the generator makes"""
    rng = np.random.default_rng(t)
    n = fo.HOT_FETCH[t]
    D = 4
    if t in FLOATS:
        p = ao.PREC[t]
        lo, hi = ao.encode(np.full(1, 1 + 2.0 ** -(p - 1)), t), ao.encode(np.full(1, 2 - 2.0 ** -(p - 1)), t)
    else:
        lo, hi = np.ones(1, ao.STORAGE[t]), np.full(1, (1 << 18) - 1, ao.STORAGE[t])
    x = fo.hot_values(rng, t, (n, D))
    x[:, 0], x[:, 1] = lo[0], hi[0]
    assert (ao.values(x, t) > (1 if t in FLOATS else 0)).all() and (ao.values(x, t) < (2 if t in FLOATS else 1 << 18)).all()
    cur = fo.hot_values(rng, t, (D,))
    cur[1] = hi[0]
    for j in range(n):
        nxt = ao.add(cur, x[j], t)
        assert (ao.values(nxt, t) > ao.values(cur, t)).all(), (ao.NAMES[t], j, cur, x[j], nxt)
        cur = nxt


@pytest.mark.parametrize("E", [2, 4, 8])
def test_fop_path(E):
    """the head and tail are element atomics, the body takes the re-phase variant of its staged phase -- every variant
    reachable for the element size -- and the result is one bulk store only when result, size and staged bytes are
    16-byte aligned"""
    t = {2: ao.ACC_F16, 4: ao.ACC_F32, 8: ao.ACC_F64}[E]
    seen = set()
    for dp in range(0, 16, E):
        for sp in range(0, 16, E):
            p, rp = fo.fop_path(dp, sp, 160, np.arange(0, 160, E), res_phase=0)
            head = (16 - dp) % 16
            end = head + (160 - head) // 16 * 16
            assert (p[:head // E] == "element").all() and (p[end // E:] == "element").all()
            assert len(set(p[head // E:end // E])) == 1
            seen.add(p[head // E])
            assert rp == ("bulk" if sp == 0 else "drain_chunk")
    assert seen == set(fo.vector_paths(t)) and len(seen) == 16 // E
    assert fo.fop_path(0, 0, 150, [0], res_phase=0)[1] == "drain_chunk"
    assert fo.fop_path(0, 0, 160, [0], res_phase=E)[1] == "drain_chunk"
    assert (fo.fop_path(4, 0, 8, np.arange(0, 8, E))[0] == "element").all()
