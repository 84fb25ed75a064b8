"""The batched reductions' NumPy oracle (tests/red_oracle.py) against the compiled reference and an element-wise
restatement on seeded edge worlds, its checker against device outcomes made wrong on purpose (each reported at the
right element), and the Python-side op tables and checks that need no device."""
import math
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests import acc_oracle as ao
from tests import put_oracle as po
from tests import red_oracle as ro
from tests.test_put_cpu import _edge_requests

CELLS = [(op, t) for op in ro.OPS.values() for t in ao.STORAGE if ro.allowed(op, t)]


def _ids(c):
    return f"{ro.NAMES[c[0]]}-{ao.NAMES[c[1]]}"


def _f(bits, t):
    """one float element's value (Python float) from its bits"""
    if t == ao.ACC_F64:
        return struct.unpack("<d", struct.pack("<Q", bits))[0]
    if t == ao.ACC_F32:
        return struct.unpack("<f", struct.pack("<I", bits))[0]
    if t == ao.ACC_F16:
        return float(np.array([bits], np.uint16).view(np.float16)[0])
    return struct.unpack("<f", struct.pack("<I", bits << 16))[0]


def _naive1(a, b, t, op):
    """the rule for one element, restated on Python ints and floats (a, b: the element's and operand's bits)"""
    nb = np.dtype(ao.BITS[t]).itemsize * 8
    if t in ro.INTS:
        sa, sb = (a - (1 << nb) if a >> (nb - 1) else a), (b - (1 << nb) if b >> (nb - 1) else b)
        if op == ro.OP_MAX:
            return a if sa >= sb else b
        if op == ro.OP_MIN:
            return a if sa <= sb else b
        return {ro.OP_BAND: a & b, ro.OP_BOR: a | b, ro.OP_BXOR: a ^ b}[op]
    fa, fb = _f(a, t), _f(b, t)
    if math.isnan(fb):
        return a
    if math.isnan(fa):
        return b
    if fa == fb:  # equal values: only the zeros differ, by sign (-0 < +0)
        neg_a, neg_b = a >> (nb - 1), b >> (nb - 1)
        if op == ro.OP_MAX:
            return b if neg_a and not neg_b else a
        return b if neg_b and not neg_a else a
    return b if (fb > fa) == (op == ro.OP_MAX) else a


def _world(rng, nrows, disp, t):
    return [ro.families(rng, t, n * disp).reshape(n, disp) for n in nrows]


def _src(rng, shards, t, batch):
    _, _, _, total, _ = ro.fo.plan(shards, t, 1 << 62, **batch)
    return ro.families(rng, t, total // np.dtype(ao.STORAGE[t]).itemsize).view(np.uint8)


@pytest.mark.parametrize("cell", CELLS, ids=_ids)
@pytest.mark.parametrize("seed", range(2))
def test_oracle_edge_worlds(seed, cell):
    """empty ranks, straddlers, out-of-range starts and counts, duplicates, every value family: the oracle equals the
    element-wise rule in request order, reports the put's codes and layout, leaves an invalid request's result bytes
    alone, a short src touches nothing, and the checker accepts the oracle's own outcome, fetch and accumulate"""
    op, t = cell
    rng = np.random.default_rng([seed, op, t])
    nrows = [int(x) for x in rng.integers(0, 25, size=int(rng.integers(2, 5)))]
    nrows[int(rng.integers(0, len(nrows)))] += 1
    nrows.insert(1, 0)
    disp = int(rng.integers(1, 5))
    shards = _world(rng, nrows, disp, t)
    lenlist = po.lenlist_of(shards)
    starts, counts = _edge_requests(rng, lenlist, 30)
    batch = {"starts": starts, "counts": counts}
    src = _src(rng, shards, t, batch)
    result = rng.integers(0, 256, size=src.size + 16, dtype=np.uint8)
    new, res, codes, bad, total = ro.reduce(shards, src, t, op, result, **batch)
    _, pcodes, pbad, ptotal = po.put([np.ascontiguousarray(s).view(np.uint8) for s in shards], src, **batch)
    assert (codes, bad, total) == (pcodes, pbad, ptotal) and total == src.size
    # the element-wise restatement
    u = ao.BITS[t]
    world = [np.ascontiguousarray(s).view(u).reshape(-1).astype(object).tolist() for s in shards]
    x = src.view(u).astype(object).tolist()
    prev = np.array(result, np.uint8)[:src.size].view(u).astype(object).tolist()
    o = 0
    rows = int(lenlist[-1])
    for (s, n, _), code in zip(po.requests(**batch), codes):
        m = n * disp if 0 < n <= rows else 0
        if code == 0:
            r = po.sortedsearch(lenlist, s)
            first = int(lenlist[r - 1]) if r else 0
            for k in range(m):
                e = (s - first) * disp + k
                prev[o + k] = world[r][e]
                world[r][e] = _naive1(int(world[r][e]), int(x[o + k]), t, op)
        o += m
    for r, sh in enumerate(new):
        assert np.ascontiguousarray(sh).view(u).reshape(-1).tolist() == [int(v) for v in world[r]], f"rank {r}"
    assert res[:src.size].view(u).tolist() == [int(v) for v in prev]
    assert res[src.size:].tobytes() == result[src.size:].tobytes()
    assert ro.check(shards, [(src, None, result, batch)], t, op, new, [res]) is None
    new_acc, none, _, _, _ = ro.reduce(shards, src, t, op, None, **batch)
    assert none is None and all(a.tobytes() == b.tobytes() for a, b in zip(new_acc, new))
    assert ro.check(shards, [(src, None, None, batch)], t, op, new_acc, [None]) is None
    short, sres, codes2, bad2, _ = ro.reduce(shards, src, t, op, result, src_bytes=src.size - 1, **batch)
    assert codes2 == codes and bad2 == bad
    if total:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(short, shards)) and sres.tobytes() == result.tobytes()


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_MIN, ao.ACC_I32), (ro.OP_BXOR, ao.ACC_I64),
                                  (ro.OP_MAX, ao.ACC_F64), (ro.OP_BOR, ao.ACC_I32)], ids=_ids)
def test_oracle_vs_compiled_reference(cell):
    """each valid request run on the reference as the owner's get of its rows, the op applied by the element-wise rule,
    and the owner's update; the previous rows and the world read back with get() equal the oracle's"""
    op, t = cell
    rng = np.random.default_rng([103, op, t])
    nrows = [int(x) for x in rng.integers(0, 20, size=3)]
    nrows[1] += 1
    disp = int(rng.integers(1, 4))
    shards = _world(rng, nrows, disp, t)
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    starts, counts = _edge_requests(rng, lenlist, 25)
    batch = {"starts": starts, "counts": counts}
    src = _src(rng, shards, t, batch)
    result = rng.integers(0, 256, size=src.size, dtype=np.uint8)
    new, res, codes, _, _ = ro.reduce(shards, src, t, op, result, **batch)
    dt = np.dtype(ao.STORAGE[t])
    u = ao.BITS[t]
    E = dt.itemsize
    ref_res = result.copy()
    w = O.RefWorld(len(shards))
    try:
        w.add("x", shards)
        o = 0
        for (s, n, _), code in zip(po.requests(**batch), codes):
            nb = n * disp * E if 0 < n <= rows else 0
            if code == 0 and nb:
                r = w.sortedsearch(lenlist, s)
                first = int(lenlist[r - 1]) if r else 0
                cur = np.empty((n, disp), dt)
                w.get(r, "x", cur, s)
                ref_res[o:o + nb] = cur.reshape(-1).view(np.uint8)
                upd = [_naive1(int(a), int(b), t, op)
                       for a, b in zip(cur.reshape(-1).view(u).tolist(), src[o:o + nb].view(u).tolist())]
                w.update(r, "x", np.array(upd, np.uint64).astype(u).view(dt).reshape(n, disp), s - first)
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


# ------------------------------------------------------------------------------------------------ the checker
def _one(t, op, v0, xs, fetch=True):
    """calls that each reduce x into global row 1 column 0 (rank 1) of a 2-rank world, plus column 1 touched once;
    the oracle's sequential outcome"""
    dt = ao.STORAGE[t]
    shards = [np.zeros((1, 2), dt), np.array([[v0, v0]], dt)]
    calls = []
    for x in xs:
        src = np.array([[x, x]], dt).view(np.uint8).reshape(-1)
        calls.append((src, None, np.zeros(src.size, np.uint8) if fetch else None, {"starts": [1], "counts": [1]}))
    new, results, _ = ro.reduce_many(shards, calls, t, op)
    return shards, calls, new, results


def _bits(v, t):
    return int(np.asarray([v], ao.STORAGE[t]).view(ao.BITS[t])[0])


def _set(arr, bits, t, idx=0):
    """arr (a storage array) with flat element idx replaced by the given bits"""
    a = np.ascontiguousarray(arr).copy()
    a.reshape(-1).view(ao.BITS[t])[idx] = bits
    return a


@pytest.mark.parametrize("cell", CELLS, ids=_ids)
def test_checker_accepts_every_order(cell):
    """every order of four fetches on one element is accepted, with an accumulate beside them too"""
    op, t = cell
    rng = np.random.default_rng([7, op, t])
    xs = ro.families(rng, t, 4)
    shards, calls, _, _ = _one(t, op, ro.families(rng, t, 1)[0], xs)
    for prev, final in ro.permutations_ok(np.asarray(shards[1])[0, 0], xs, t, op):
        new = [shards[0], _set(shards[1], _bits(final, t), t)]
        new[1] = _set(new[1], _bits(ro.fold(shards[1][0, 1], xs, t, op), t), t, 1)
        results = []
        for j, (src, _, _, _) in enumerate(calls):
            r = np.zeros(src.size, np.uint8)
            r.view(ao.STORAGE[t])[0] = prev[j]
            r.view(ao.STORAGE[t])[1] = prev[j]  # (column 1: the same order)
            results.append(r)
        # column 1 took the same order: its previous values are the same
        assert ro.check(shards, calls, t, op, new, results) is None


def test_checker_names_an_unsigned_compare():
    """max(-1, 1) of int32 is 1; an unsigned compare gives -1 (0xffffffff)"""
    t, op = ao.ACC_I32, ro.OP_MAX
    shards, calls, new, results = _one(t, op, -1, [1], fetch=False)
    bad = [shards[0], _set(new[1], 0xFFFFFFFF, t)]
    msg = ro.check(shards, calls, t, op, bad, results)
    assert msg and msg.startswith("final value: rank 1 global row 1 column 0") and "0xffffffff" in msg


@pytest.mark.parametrize("t", ro.FLOATS)
def test_checker_names_a_nan_operand_that_overwrote(t):
    """a NaN operand is ignored: the element keeps 1.0"""
    op = ro.OP_MAX
    nan = ao._nan_bits(t, 0)
    shards, calls, new, results = _one(t, op, 1.0 if t != ao.ACC_BF16 else 0x3F80, [0.0 if t != ao.ACC_BF16 else 0])
    # operand: a quiet NaN in column 0
    src = calls[0][0].copy()
    src.view(ao.BITS[t])[0] = nan
    calls = [(src,) + calls[0][1:]]
    new, results, _ = ro.reduce_many(shards, calls, t, op)
    assert ao.bits(np.ascontiguousarray(new[1]).reshape(-1)[:1], t)[0] == _bits(shards[1][0, 0], t)
    bad = [shards[0], _set(new[1], nan, t)]
    msg = ro.check(shards, calls, t, op, bad, results)
    assert msg and msg.startswith("final value: rank 1 global row 1 column 0")


@pytest.mark.parametrize("t", ro.FLOATS)
@pytest.mark.parametrize("op", (ro.OP_MAX, ro.OP_MIN))
def test_checker_names_a_zero_blind_compare(t, op):
    """max(-0, +0) is +0 and min(+0, -0) is -0: a compare that takes them as equal keeps the element"""
    sign = 1 << (np.dtype(ao.BITS[t]).itemsize * 8 - 1)
    v0, x = (sign, 0) if op == ro.OP_MAX else (0, sign)
    dt = ao.STORAGE[t]
    shards = [np.zeros((1, 2), dt), _set(_set(np.zeros((1, 2), dt), v0, t), v0, t, 1)]
    src = np.ascontiguousarray(_set(_set(np.zeros((1, 2), dt), x, t), x, t, 1)).view(np.uint8).reshape(-1)
    calls = [(src, None, np.zeros(src.size, np.uint8), {"starts": [1], "counts": [1]})]
    new, results, _ = ro.reduce_many(shards, calls, t, op)
    assert ao.bits(np.ascontiguousarray(new[1]).reshape(-1), t).tolist() == [x, x]
    msg = ro.check(shards, calls, t, op, [shards[0], shards[1]], results)  # (the element kept)
    assert msg and msg.startswith("final value: rank 1 global row 1 column 0")


@pytest.mark.parametrize("t", (ao.ACC_F16, ao.ACC_BF16))
def test_checker_names_a_changed_neighbour_half_word(t):
    """a 16-bit element's loop changed the other half of its word: the untouched neighbour is named"""
    op = ro.OP_MAX
    dt = ao.STORAGE[t]
    shards = [np.zeros((1, 2), dt), np.zeros((2, 2), dt)]
    src = np.ascontiguousarray(_set(np.zeros((1, 2), dt), 0x3C00 if t == ao.ACC_F16 else 0x3F80, t)).view(np.uint8)
    src = src.reshape(-1)[:2]  # one element: disp 1 below
    shards = [s.reshape(-1, 1) for s in (np.zeros(2, dt), np.zeros(4, dt))]
    calls = [(src, None, np.zeros(2, np.uint8), {"starts": [2], "counts": [1]})]
    new, results, _ = ro.reduce_many(shards, calls, t, op)
    bad = [shards[0], _set(new[1], 0x0001, t, 1)]  # global row 3 shares the word of row 2
    msg = ro.check(shards, calls, t, op, bad, results)
    assert msg and msg.startswith("an element no request touches changed: rank 1 global row 3 column 0")


@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_BOR, ao.ACC_I64), (ro.OP_BXOR, ao.ACC_I32),
                                  (ro.OP_MIN, ao.ACC_BF16)], ids=_ids)
def test_checker_names_a_lost_contribution(cell):
    """one of several accumulates dropped: the final value is named"""
    op, t = cell
    rng = np.random.default_rng([11, op, t])
    xs = ro.distinct(rng, t, 12) if op != ro.OP_BOR else (np.int64(1) << np.arange(12)).astype(ao.STORAGE[t])
    k = ro.order_keys(xs, t)
    # a start every contribution can move: the smallest value for max, the largest for min, zero for or / xor
    start = {ro.OP_MAX: xs[np.argmin(k)], ro.OP_MIN: xs[np.argmax(k)]}.get(op, np.zeros(1, ao.STORAGE[t])[0])
    shards, calls, new, results = _one(t, op, start, xs[1:], fetch=False)
    lost = ro.fold(start, xs[1:], t, op)
    for drop in range(11):
        cand = ro.fold(start, np.delete(xs[1:], drop), t, op)
        if _bits(cand, t) != _bits(lost, t):
            break
    else:
        pytest.skip("no contribution changes the final value")
    bad = [shards[0], _set(new[1], _bits(cand, t), t)]
    msg = ro.check(shards, calls, t, op, bad, results)
    assert msg and msg.startswith("final value: rank 1 global row 1 column 0")


@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_I64), (ro.OP_BXOR, ao.ACC_I32), (ro.OP_MIN, ao.ACC_F16),
                                  (ro.OP_BOR, ao.ACC_I32)], ids=_ids)
@pytest.mark.parametrize("k", (3, 40))
def test_checker_names_two_fetches_with_one_previous_value(cell, k):
    """fetches of strictly increasing (max), decreasing (min), new-bit (or) or any (xor) operands each change the
    element, so no two of them can return the same previous value"""
    op, t = cell
    dt = ao.STORAGE[t]
    if op == ro.OP_MAX:
        v0, xs = 0, np.arange(1, k + 1).astype(dt)
    elif op == ro.OP_MIN:
        v0, xs = 1000.0, (1000 - np.arange(1, k + 1)).astype(dt)
    elif op == ro.OP_BOR:
        k = min(k, 31)
        v0, xs = 0, (np.int64(1) << np.arange(k)).astype(dt)
    else:
        v0, xs = 0, np.arange(1, k + 1).astype(dt)
    shards, calls, new, results = _one(t, op, v0, xs)
    assert ro.check(shards, calls, t, op, new, results) is None
    bad = [r.copy() for r in results]
    bad[2].view(dt)[0] = results[1].view(dt)[0]  # call 2 got call 1's previous value
    msg = ro.check(shards, calls, t, op, new, bad)
    assert msg and msg.startswith("fetch chain: rank 1 global row 1 column 0")


def test_checker_names_a_wrong_once_previous_value():
    t, op = ao.ACC_F32, ro.OP_MIN
    shards, calls, new, results = _one(t, op, 2.0, [1.0])
    bad = [r.copy() for r in results]
    bad[0].view(np.float32)[1] = 1.0
    msg = ro.check(shards, calls, t, op, new, bad)
    assert msg and msg.startswith("previous value: rank 1 global row 1 column 1")


def test_red_path_names_the_hardware():
    """bulk bodies of f32 / f64 max / min become vector CAS loops; f16 ends are CAS loops; integers keep the bulk"""
    assert ro.red_path(ao.ACC_F32, ro.OP_MAX, 0, 0, 64, 0) == "vector (CAS loop)"
    assert ro.red_path(ao.ACC_I32, ro.OP_MAX, 0, 0, 64, 0) == "bulk"
    assert ro.red_path(ao.ACC_F16, ro.OP_MIN, 2, 2, 64, 0) == "element (CAS loop)"
    assert ro.red_path(ao.ACC_BF16, ro.OP_MIN, 0, 0, 64, 0) == "bulk"


# ------------------------------------------------------------------------------------------------ Python side
def test_op_tables():
    from ddstore_b200 import _capi
    assert _capi.FOP_OPS == {"sum": 1, "replace": 2}
    assert _capi.RED_OPS == ro.OPS
    assert (_capi.OP_MAX, _capi.OP_MIN, _capi.OP_BAND, _capi.OP_BOR, _capi.OP_BXOR) == (4, 5, 6, 7, 8)


def test_unknown_op_names_raise_before_the_call():
    from ddstore_b200.store import PyDDStore
    assert PyDDStore._red_op("x", "sum") == 1 and PyDDStore._red_op("x", "amax") == 4
    for bad in ("max", "replace", "prod", None):
        with pytest.raises(ValueError, match="is not one of"):
            PyDDStore._red_op("x", bad)
