"""The batched compare-and-swap's NumPy oracle (tests/cas_oracle.py) against the compiled reference and an element-wise
restatement on seeded edge worlds, its checker against device outcomes made wrong on purpose (each reported at the right
element), and the Python-side checks of compare_and_swap_batch that need no device."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import cas_oracle as co
from tests import put_oracle as po
from tests.test_put_cpu import _edge_requests

DTYPES = (np.uint8, np.int16, np.int32, np.float32, np.int64, np.float64)


def _shards(rng, nrows, disp, dtype, lo=0, hi=4):
    """small values, so that about a third of the compares match"""
    return [rng.integers(lo, hi, size=(n, disp)).astype(dtype) for n in nrows]


def _operands(rng, shards, batch, lo=0, hi=4):
    """src and compare of a batch's layout, as bytes (values of the shards' range, so compares match and fail)"""
    _, _, _, total, _ = co.plan(shards, 1 << 62, **batch)
    dt = shards[0].dtype
    n = total // dt.itemsize
    src = rng.integers(lo, hi, size=n).astype(dt).view(np.uint8)
    cmp = rng.integers(lo, hi, size=n).astype(dt).view(np.uint8)
    return src, cmp


def _naive(shards, src, cmp, result, batch):
    """element by element, in request order: the rule restated on the elements' bits (new shards, new result)"""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    disp = shards[0].shape[1]
    u = co.UINT[shards[0].dtype.itemsize]
    x, c = src.view(u), cmp.view(u)
    world = [np.ascontiguousarray(s).view(u).reshape(-1).copy() for s in shards]
    res = np.array(result, np.uint8).view(u).copy()
    o = 0
    for s, n, ok in po.requests(**batch):
        m = n * disp if ok and 0 < n <= rows else 0
        if (po.CODE_SAMPLE if not ok else po.locate(lenlist, s, n)[0]) == 0:
            r = po.sortedsearch(lenlist, s)
            first = int(lenlist[r - 1]) if r else 0
            for k in range(m):
                e = (s - first) * disp + k
                res[o + k] = world[r][e]
                if world[r][e] == c[o + k]:
                    world[r][e] = x[o + k]
        o += m
    return [w.view(sh.dtype).reshape(sh.shape) for w, sh in zip(world, shards)], res.view(np.uint8)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("seed", range(3))
def test_oracle_edge_worlds(seed, dtype):
    """empty ranks, straddlers, out-of-range starts and counts, duplicates: the oracle equals the element-wise rule,
    reports the put's codes and layout, leaves an invalid request's result bytes alone, a short src touches nothing,
    and the checker accepts the oracle's own outcome"""
    rng = np.random.default_rng([seed, np.dtype(dtype).num])
    nrows = [int(x) for x in rng.integers(0, 30, size=int(rng.integers(2, 5)))]
    nrows[int(rng.integers(0, len(nrows)))] += 1
    nrows[0] = 0 if seed % 2 else nrows[0]
    nrows.insert(1, 0)
    disp = int(rng.integers(1, 5))
    shards = _shards(rng, nrows, disp, dtype)
    lenlist = po.lenlist_of(shards)
    starts, counts = _edge_requests(rng, lenlist, 30)
    batch = {"starts": starts, "counts": counts}
    src, cmp = _operands(rng, shards, batch)
    result = rng.integers(0, 256, size=src.size + 16, dtype=np.uint8)
    new, res, codes, bad, total = co.cas(shards, src, cmp, result, **batch)
    _, pcodes, pbad, ptotal = po.put([s.view(np.uint8) for s in shards], src, **batch)
    assert (codes, bad, total) == (pcodes, pbad, ptotal) and total == src.size
    nnew, nres = _naive(shards, src, cmp, result, batch)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, nnew)) and res.tobytes() == nres.tobytes()
    assert res[src.size:].tobytes() == result[src.size:].tobytes()
    _, pl, _, _, _ = co.plan(shards, src.size, **batch)
    for (_r, _l, _c, off, n), code in zip(pl, codes):
        if code:
            assert res[off:off + n].tobytes() == result[off:off + n].tobytes()
    calls = [(src, None, cmp, result, batch)]
    assert co.check(shards, calls, new, [res]) is None
    short, sres, codes2, bad2, _ = co.cas(shards, src, cmp, result, src_bytes=src.size - 1, **batch)
    assert codes2 == codes and bad2 == bad
    if total:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(short, shards)) and sres.tobytes() == result.tobytes()


@pytest.mark.parametrize("dtype", (np.uint8, np.int16, np.int32, np.int64))
def test_oracle_sample_ids_fixed_count_and_duplicates(dtype):
    """bad sample ids keep 0 bytes; a duplicate id sees what the first left; a fixed count past the end is a count
    error"""
    rng = np.random.default_rng([41, np.dtype(dtype).num])
    shards = _shards(rng, [5, 0, 7], 3, dtype)
    lenlist = po.lenlist_of(shards)
    rs = np.array([0, 4, 5, 11, 3, 12], np.int64)
    rc = np.array([2, 3, 4, 1, -1, 1], np.int64)
    ids = np.array([0, 6, 2, -1, 2, 1, 3, 4, 5, 0], np.int64)
    batch = {"sample_ids": ids, "table": (rs, rc)}
    src, cmp = _operands(rng, shards, batch)
    result = np.zeros(src.size, np.uint8)
    new, res, codes, bad, total = co.cas(shards, src, cmp, result, **batch)
    assert codes[:4] == [0, po.CODE_SAMPLE, 0, po.CODE_SAMPLE] and bad == 1
    nnew, nres = _naive(shards, src, cmp, result, batch)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new, nnew)) and res.tobytes() == nres.tobytes()
    R = 3 * np.dtype(dtype).itemsize
    first, second = 2 * R, (2 + 4) * R  # layout: id 0 (2 rows), id 6 (0), id 2 (4 rows), id -1 (0), id 2
    old = shards[2][0:4]
    exp = np.where(old == cmp[first:first + 4 * R].view(dtype).reshape(4, 3),
                   src[first:first + 4 * R].view(dtype).reshape(4, 3), old)
    assert res[second:second + 4 * R].tobytes() == exp.tobytes()
    fixed = {"starts": np.array([0, 3, 11, 0, 5], np.int64), "fixed_count": 2}
    src, cmp = _operands(rng, shards, fixed)
    new, res, codes, bad, total = co.cas(shards, src, cmp, np.zeros(src.size, np.uint8), **fixed)
    assert codes == [0, 0, po.CODE_COUNT, 0, 0] and bad == 2 and total == 5 * 2 * R
    assert not res[2 * 2 * R:3 * 2 * R].any()


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("dtype", (np.uint8, np.int32, np.float32, np.int64, np.float64))
@pytest.mark.parametrize("seed", range(2))
def test_oracle_vs_compiled_reference(seed, dtype):
    """each valid request run on the reference as the owner's get of its rows (the previous rows), a bytewise select
    and the owner's update; the previous rows and the world read back with get() equal the oracle's"""
    rng = np.random.default_rng([101, seed, np.dtype(dtype).num])
    nrows = [int(x) for x in rng.integers(0, 20, size=3)]
    nrows[1] += 1
    disp = int(rng.integers(1, 4))
    shards = _shards(rng, nrows, disp, dtype)
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1])
    starts, counts = _edge_requests(rng, lenlist, 25)
    batch = {"starts": starts, "counts": counts}
    src, cmp = _operands(rng, shards, batch)
    result = rng.integers(0, 256, size=src.size, dtype=np.uint8)
    new, res, codes, _, _ = co.cas(shards, src, cmp, result, **batch)
    dt = np.dtype(dtype)
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
                cb = cur.reshape(-1).view(np.uint8).reshape(-1, E)
                eq = (cb == cmp[o:o + nb].reshape(-1, E)).all(1, keepdims=True)
                upd = np.where(eq, src[o:o + nb].reshape(-1, E), cb)
                w.update(r, "x", np.ascontiguousarray(upd).reshape(-1).view(dt).reshape(n, disp), s - first)
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
def _claims(dtype, k=6, v0=7):
    """k calls that each claim global row 5 (rank 1) with compare v0 and src 100 + j, plus a once-touched row whose
    compare matches in column 0 only; the oracle's (sequential) outcome"""
    shards = [np.arange(8).reshape(4, 2).astype(dtype) + 10, np.full((3, 2), v0).astype(dtype)]
    calls = []
    for j in range(k):
        src = np.array([[100 + j, 120 + j]], dtype).view(np.uint8).reshape(-1)
        cmp = np.array([[v0, v0]], dtype).view(np.uint8).reshape(-1)
        calls.append((src, None, cmp, np.zeros(src.size, np.uint8), {"starts": [5], "counts": [1]}))
    src = np.array([[70, 80]], dtype).view(np.uint8).reshape(-1)
    cmp = np.array([[12, 0]], dtype).view(np.uint8).reshape(-1)
    calls.append((src, None, cmp, np.zeros(src.size, np.uint8), {"starts": [1], "counts": [1]}))
    new, results, _ = co.cas_many(shards, calls)
    return shards, calls, new, results


@pytest.mark.parametrize("dtype", DTYPES)
def test_checker_accepts_every_order(dtype):
    """the oracle's own outcome and that of the claims in reverse order (a different winner) both pass"""
    shards, calls, new, results = _claims(dtype)
    assert co.check(shards, calls, new, results) is None
    rev = list(reversed(calls[:-1])) + calls[-1:]
    new2, results2, _ = co.cas_many(shards, rev)
    back = list(reversed(results2[:-1])) + results2[-1:]
    assert co.check(shards, calls, new2, back) is None
    assert new2[1].tobytes() != new[1].tobytes()


@pytest.mark.parametrize("dtype", (np.uint8, np.int16, np.int32, np.int64))
def test_checker_names_two_winners_and_a_lost_win(dtype):
    shards, calls, new, results = _claims(dtype)
    two = [r.copy() for r in results]
    two[3].view(dtype)[0] = 7  # a second claim also got the start value: two winners
    msg = co.check(shards, calls, new, two)
    assert msg and "compare-and-swaps: rank 1 global row 5 column 0" in msg, msg
    lost = [s.copy() for s in new]
    lost[1][1, 1] = 7  # the winner's value never stored, yet the others saw it
    msg = co.check(shards, calls, lost, results)
    assert msg and "compare-and-swaps: rank 1 global row 5 column 1" in msg, msg


@pytest.mark.parametrize("dtype", DTYPES)
def test_checker_names_a_wrong_previous_value_and_a_wrong_new_value(dtype):
    shards, calls, new, results = _claims(dtype)
    bent = [r.copy() for r in results]
    bent[-1].view(dtype)[1] += 1  # the once-touched row's column 1: not the pre-value
    msg = co.check(shards, calls, new, bent)
    assert msg and "previous value: rank 0 global row 1 column 1" in msg, msg
    wrong = [s.copy() for s in new]
    wrong[0][1, 1] = 80  # column 1's compare failed: no swap
    msg = co.check(shards, calls, wrong, results)
    assert msg and "new value: rank 0 global row 1 column 1" in msg, msg
    wrong = [s.copy() for s in new]
    wrong[0][1, 0] = 12  # column 0's compare matched: the swap lost
    msg = co.check(shards, calls, wrong, results)
    assert msg and "new value: rank 0 global row 1 column 0" in msg, msg


@pytest.mark.parametrize("dtype", (np.uint8, np.int16))
def test_checker_names_a_changed_neighbour_in_the_word(dtype):
    """1- and 2-byte elements: a neighbour no request touches, in the same 32-bit word, must keep its bits"""
    shards, calls, new, results = _claims(dtype)
    wrong = [s.copy() for s in new]
    wrong[1][2, 0] ^= 1  # global row 6, next to the claimed row 5 in the same word
    msg = co.check(shards, calls, wrong, results)
    assert msg and "no request touches changed: rank 1 global row 6 column 0" in msg, msg


@pytest.mark.parametrize("dtype,neg,pos,nan_a,nan_b", [
    (np.float16, 0x8000, 0x0000, 0x7E01, 0x7E02),
    (np.float32, 0x80000000, 0, 0x7FC00001, 0x7FC00002),
    (np.float64, 1 << 63, 0, 0x7FF8000000000001, 0x7FF8000000000002)])
def test_checker_compares_floats_by_bits(dtype, neg, pos, nan_a, nan_b):
    """-0 against a +0 compare fails, a NaN against another payload fails, a NaN against its own bits succeeds; the
    checker names a device that treated -0 as +0, matched NaNs by class, or changed a payload"""
    u = co.UINT[np.dtype(dtype).itemsize]
    shards = [np.array([[neg, nan_a, nan_a, 5]], u).view(dtype)]
    src = np.array([7, 8, 9, 10], u).view(np.uint8)
    cmp = np.array([pos, nan_b, nan_a, 5], u).view(np.uint8)
    calls = [(src, None, cmp, np.zeros(src.size, np.uint8), {"starts": [0], "counts": [1]})]
    new, results, _ = co.cas_many(shards, calls)
    assert new[0].view(u).tolist() == [[neg, nan_a, 9, 10]]
    assert results[0].view(u).tolist() == [neg, nan_a, nan_a, 5]
    assert co.check(shards, calls, new, results) is None
    as_pos = [new[0].copy()]
    as_pos[0].view(u)[0, 0] = 7
    msg = co.check(shards, calls, as_pos, results)
    assert msg and "new value: rank 0 global row 0 column 0" in msg, msg
    by_class = [new[0].copy()]
    by_class[0].view(u)[0, 1] = 8
    msg = co.check(shards, calls, by_class, results)
    assert msg and "new value: rank 0 global row 0 column 1" in msg, msg
    payload = [results[0].copy()]
    payload[0].view(u)[2] = nan_b
    msg = co.check(shards, calls, new, payload)
    assert msg and "previous value: rank 0 global row 0 column 2" in msg, msg


def test_checker_names_a_result_written_for_an_invalid_request():
    rng = np.random.default_rng(9)
    shards = _shards(rng, [6, 0, 9], 2, np.int32)
    batch = {"starts": np.array([1, 14, 3], np.int64), "counts": np.array([2, 2, 1], np.int64)}  # 14 + 2 > 15
    src, cmp = _operands(rng, shards, batch)
    result = np.full(src.size, 0xA5, np.uint8)
    calls = [(src, None, cmp, result, batch)]
    new, results, out = co.cas_many(shards, calls)
    assert out[0][:2] == (po.CODE_COUNT, 1)
    assert co.check(shards, calls, new, results) is None
    bad = [results[0].copy()]
    bad[0][2 * 8 + 5] = 0  # inside request 1's bytes
    msg = co.check(shards, calls, new, bad)
    assert msg and "request 1" in msg and "written outside" in msg, msg
    calls = [(src, src.size - 1, cmp, result, batch)]  # a capacity error: nothing may be written at all
    new, results, _ = co.cas_many(shards, calls)
    assert results[0].tobytes() == result.tobytes()
    bad = [results[0].copy()]
    bad[0][0] = 0
    assert "written outside" in co.check(shards, calls, new, bad)


def test_order_directly():
    assert co.order(0, [(0, 5, 0), (0, 6, 5), (0, 7, 5)], 5) is None          # one winner, two losers
    assert co.order(0, [(0, 5, 0), (0, 6, 0)], 6) is not None                 # two winners
    assert co.order(0, [(0, 5, 0), (5, 6, 5), (6, 7, 6)], 7) is None          # a chain
    assert co.order(0, [(5, 6, 5), (0, 5, 0), (6, 7, 6)], 7) is None          # the same, listed out of order
    assert co.order(0, [(0, 5, 0), (5, 5, 5)], 5) is None                     # a swap that keeps the value
    assert co.order(0, [(0, 5, 0), (0, 5, 0)], 5) is not None                 # two winners, even with equal srcs
    assert co.order(0, [(0, 5, 0), (0, 6, 5)], 6) is not None                 # lost: the final value is not 5
    # a search: two claims that could each go first, only one order explains the results
    assert co.order(1, [(1, 2, 1), (1, 3, 1), (2, 1, 2)], 3) is None


# ------------------------------------------------------------------------------------------------ bindings
def test_compare_and_swap_rejects_bad_arguments_before_the_call():
    from ddstore_b200.store import PyDDStore
    torch = pytest.importorskip("torch")

    class _Src:
        nbytes, itemsize = 64, 4
    with pytest.raises(ValueError, match="compare must be a CUDA tensor"):
        PyDDStore._cas_args("x", torch.zeros(16), None, _Src())
    with pytest.raises(ValueError, match="compare must be a CUDA tensor"):
        PyDDStore._cas_args("x", None, None, _Src())
    with pytest.raises(ValueError, match="src must be device memory"):
        PyDDStore._put_src("x", np.zeros(4, np.int32))
