"""The batched accumulate's NumPy oracle (tests/acc_oracle.py) against the compiled reference and on seeded worlds, and
the Python-side checks of accumulate_batch / accumulate_samples that need no device."""
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
