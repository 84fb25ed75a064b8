"""The batched put's NumPy oracle (tests/put_oracle.py) against the compiled reference and on seeded random worlds, and
the Python-side argument checks of put_batch / put_samples that need no device."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import put_oracle as po


def _world(rng, nrows, disp, dtype):
    return [rng.integers(0, 2**31, size=(n, disp)).astype(dtype) for n in nrows]


def _edge_requests(rng, lenlist, n):
    """valid requests mixed with every edge: start below 0, at and past the end, straddling two owners, negative and
    overflowing counts, zero counts, duplicates"""
    rows = int(lenlist[-1])
    st, ct = [], []
    for _ in range(n):
        s = int(rng.integers(0, rows))
        t = po.sortedsearch(lenlist, s)
        hi = int(lenlist[t]) - s
        st.append(s)
        ct.append(int(rng.integers(0, hi + 1)))
    edges = [(-1, 1), (rows, 1), (rows - 1, 1), (rows + 5, 0), (0, -1), (0, 2**62), (0, rows + 1), (rows - 1, 2)]
    for b in lenlist[:-1]:  # straddling an owner boundary
        if 0 < b < rows:
            edges.append((int(b) - 1, 2))
    edges.append((st[0], ct[0]))  # a duplicate of the first request
    for s, c in edges:
        k = int(rng.integers(0, len(st) + 1))
        st.insert(k, s)
        ct.insert(k, c)
    return np.array(st, np.int64), np.array(ct, np.int64)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_codes_layout_and_writes(seed):
    rng = np.random.default_rng(seed)
    nrows = [int(x) for x in rng.integers(0, 40, size=int(rng.integers(1, 5)))]
    nrows[int(rng.integers(0, len(nrows)))] += 1  # at least one row
    nrows[0] = 0 if seed % 2 else nrows[0]         # an empty rank
    if sum(nrows) == 0:
        nrows[-1] = 5
    disp = int(rng.integers(1, 5))
    shards = _world(rng, nrows, disp, np.int32)
    lenlist = po.lenlist_of(shards)
    rows, R = int(lenlist[-1]), disp * 4
    starts, counts = _edge_requests(rng, lenlist, 30)
    req = po.requests(starts, counts)
    src = rng.integers(0, 256, size=sum(c * R for _, c, _ in req if 0 < c <= rows), dtype=np.uint8)
    new, codes, bad, total = po.put(shards, src, starts=starts, counts=counts)
    assert total == src.size
    c = O.COracle()
    for i, (s, n) in enumerate(zip(starts.tolist(), counts.tolist())):
        owner, offset, rc = c.locate(lenlist, s, n)
        assert codes[i] == rc, (i, s, n)
    assert bad == next((i for i, x in enumerate(codes) if x), -1)
    # every byte of the new world was written by the last valid request covering it, or is the old byte
    exp = [s.copy() for s in shards]
    o = 0
    for (s, n, _), code in zip(req, codes):
        nb = n * R if 0 < n <= rows else 0
        if code == 0 and nb:
            t = po.sortedsearch(lenlist, s)
            first = int(lenlist[t - 1]) if t else 0
            exp[t][s - first:s - first + n] = src[o:o + nb].view(np.int32).reshape(n, disp)
        o += nb
    for a, b in zip(new, exp):
        assert a.tobytes() == b.tobytes()
    # a layout larger than src writes nothing, whatever else is wrong
    small, codes2, bad2, total2 = po.put(shards, src, src_bytes=src.size - 1, starts=starts, counts=counts)
    assert total2 == total and codes2 == codes and bad2 == bad
    if total:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(small, shards))
        assert po.expected_error(codes2, bad2, total2, src.size - 1) == ((codes[bad], bad) if bad >= 0 else (12, -1))


def test_oracle_sample_ids_and_fixed_count():
    rng = np.random.default_rng(7)
    shards = _world(rng, [5, 0, 7], 3, np.int64)
    lenlist = po.lenlist_of(shards)
    rs = np.array([0, 4, 5, 11, 3, 12], np.int64)
    # sample 1 straddles ranks 0/2, sample 4 has a negative count, sample 5 starts past the end
    rc = np.array([2, 3, 4, 1, -1, 1], np.int64)
    ids = np.array([0, 6, 2, -1, 1, 3, 4, 5], np.int64)
    req = po.requests(sample_ids=ids, table=(rs, rc))
    nb = [c * 24 if ok and 0 < c <= 12 else 0 for _, c, ok in req]
    src = rng.integers(0, 256, size=sum(nb), dtype=np.uint8)
    new, codes, bad, total = po.put(shards, src, sample_ids=ids, table=(rs, rc))
    assert codes == [0, po.CODE_SAMPLE, 0, po.CODE_SAMPLE, po.CODE_COUNT, 0, po.CODE_COUNT, po.CODE_COUNT]
    assert bad == 1 and total == sum(nb) == (2 + 4 + 3 + 1 + 1) * 24
    # sample 2 (rows 5..8, rank 2 rows 0..3) comes after sample 0's 48 bytes, sample 1's 72 bytes stay in the layout
    assert new[2][0:4].tobytes() == src[48:48 + 96].tobytes()
    starts = np.array([0, 3, 11, 12, 5], np.int64)
    new, codes, bad, total = po.put(shards, rng.integers(0, 256, size=5 * 48, dtype=np.uint8), starts=starts,
                                    fixed_count=2)
    assert codes == [0, 0, po.CODE_COUNT, po.CODE_COUNT, 0] and bad == 2 and total == 5 * 48
    new, codes, bad, total = po.put(shards, np.zeros(0, np.uint8), starts=starts, fixed_count=13)  # above the rows
    assert total == 0 and all(c == po.CODE_COUNT for c in codes[:3])


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("seed", range(4))
def test_oracle_vs_compiled_reference(seed):
    """every valid request applied in order as the owner's update(owner, name, rows, start - lenlist[owner-1]), the
    state read back with the reference's own get()"""
    rng = np.random.default_rng(100 + seed)
    nrows = [int(x) for x in rng.integers(0, 30, size=3)]
    nrows[1] += 1
    disp = int(rng.integers(1, 4))
    shards = _world(rng, nrows, disp, np.float32 if seed % 2 else np.int64)
    lenlist = po.lenlist_of(shards)
    rows, R = int(lenlist[-1]), disp * shards[0].dtype.itemsize
    starts, counts = _edge_requests(rng, lenlist, 25)
    req = po.requests(starts, counts)
    src = rng.integers(0, 256, size=sum(c * R for _, c, _ in req if 0 < c <= rows), dtype=np.uint8)
    if seed % 2:  # keep float rows free of NaN payload questions: the reference copies bytes, so does the oracle
        src = src.view(np.float32).copy()
        src[~np.isfinite(src)] = 1.5
        src = src.view(np.uint8)
    new, codes, bad, total = po.put(shards, src, starts=starts, counts=counts)
    w = O.RefWorld(len(shards))
    try:
        w.add("x", shards)
        o = 0
        for (s, n, _), code in zip(req, codes):
            nb = n * R if 0 < n <= rows else 0
            if code == 0 and nb:
                t = w.sortedsearch(lenlist, s)
                first = int(lenlist[t - 1]) if t else 0
                w.update(t, "x", src[o:o + nb].view(shards[0].dtype).reshape(n, disp), s - first)
            o += nb
        for r, sh in enumerate(new):
            if sh.shape[0] == 0:
                continue
            got = np.empty_like(sh)
            w.get((r + 1) % len(shards), "x", got, int(lenlist[r - 1]) if r else 0)
            assert got.tobytes() == sh.tobytes(), f"rank {r}"
    finally:
        w.close()


def test_put_rejects_host_and_missing_src():
    from ddstore_b200.store import PyDDStore
    with pytest.raises(ValueError, match="device memory"):
        PyDDStore._put_src("x", np.zeros((4, 3), np.float32))
    with pytest.raises(ValueError, match="needs `src`"):
        PyDDStore._put_src("x", None)
    torch = pytest.importorskip("torch")
    with pytest.raises(ValueError, match="device memory"):
        PyDDStore._put_src("x", torch.zeros(4, 3, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="contiguous"):
        PyDDStore._put_src("x", torch.zeros(4, 3).t())
