"""NumPy oracle of the batched put (dds_put_batch / dds_put_samples): a batch applied to a world of shards.

Request i writes global rows [start_i, start_i + count_i) of a variable from src bytes [o_i, o_i + n_i), where n_i =
count_i * row_bytes when 0 < count_i <= the variable's total rows and 0 otherwise (0 for a sample id outside the index),
and o_i is the exclusive scan of the n_i -- an invalid request keeps its bytes in the layout. Requests are checked by the
reference's two checks (include/ddstore.hpp:205-214 over src/ddstore.cxx:5-17); an invalid one writes nothing, every
valid one is written in request order (of two writes to the same bytes the later one wins here; the device leaves one of
them), and a layout larger than src writes nothing at all.
"""
import numpy as np

CODE_START, CODE_COUNT, CODE_CAPACITY, CODE_SAMPLE = 2, 3, 12, 15


def lenlist_of(shards):
    return np.cumsum([s.shape[0] for s in shards]).astype(np.int64)


def sortedsearch(lenlist, num):
    """src/ddstore.cxx:5-17: first i >= 1 with lenlist[i-1] <= num < lenlist[i], else 0"""
    for i in range(1, len(lenlist)):
        if lenlist[i - 1] <= num < lenlist[i]:
            return i
    return 0


def locate(lenlist, start, count):
    """-> (code, owner, first global row of the owner); code 0, CODE_START or CODE_COUNT"""
    t = sortedsearch(lenlist, start)
    off = int(lenlist[t - 1]) if t > 0 else 0
    if start < off:
        return CODE_START, t, off
    if count < 0 or count > int(lenlist[t]) - start:
        return CODE_COUNT, t, off
    return 0, t, off


def requests(starts=None, counts=None, fixed_count=None, sample_ids=None, table=None):
    """(start, count, id_ok) per request of an explicit, fixed-count or by-sample-id batch"""
    if sample_ids is not None:
        rs, rc = table
        out = []
        for sid in np.asarray(sample_ids, np.int64).tolist():
            ok = 0 <= sid < len(rs)
            out.append((int(rs[sid]) if ok else 0, int(rc[sid]) if ok else 0, ok))
        return out
    starts = np.asarray(starts, np.int64).tolist()
    cts = [int(fixed_count)] * len(starts) if counts is None else np.asarray(counts, np.int64).tolist()
    return [(s, c, True) for s, c in zip(starts, cts)]


def put(shards, src, src_bytes=None, **req):
    """Apply a put batch to `shards` (list of 2-D arrays of one dtype, one per rank; not modified).
    src: the packed source rows as bytes (uint8 array). Returns (new shards, per-request codes, first bad index or -1,
    layout total)."""
    lenlist = lenlist_of(shards)
    rows = int(lenlist[-1]) if len(lenlist) else 0
    row_bytes = shards[0].dtype.itemsize * (shards[0].shape[1] if shards[0].ndim > 1 else 1)
    src = np.asarray(src, np.uint8).reshape(-1)
    src_bytes = src.size if src_bytes is None else src_bytes
    reqs = requests(**req)
    codes, plan, o = [], [], 0
    for start, count, id_ok in reqs:
        n = count * row_bytes if id_ok and 0 < count <= rows else 0
        if not id_ok:
            code, t, off = CODE_SAMPLE, 0, 0
        else:
            code, t, off = locate(lenlist, start, count)
        codes.append(code)
        plan.append((t, start - off, count, o, n))
        o += n
    total = o
    bad = next((i for i, c in enumerate(codes) if c), -1)
    new = [s.copy() for s in shards]
    if total <= src_bytes:
        for (t, local, count, off, n), code in zip(plan, codes):
            if code == 0 and n > 0:
                flat = new[t].reshape(new[t].shape[0], -1).view(np.uint8)
                flat[local:local + count] = src[off:off + n].reshape(count, row_bytes)
    return new, codes, bad, total


def put_many(shards, calls):
    """Apply `calls` = [(src, src_bytes or None, request keywords)] one after the other (any ranks' calls of one epoch:
    each is a put() of its own) -> (new shards, [(status code, bad index, layout total)] as each call reports them)"""
    out = []
    for src, src_bytes, req in calls:
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        shards, codes, bad, total = put(shards, src, src_bytes=sb, **req)
        out.append(expected_error(codes, bad, total, sb) + (total,))
    return shards, out


def expected_error(codes, bad, total, src_bytes):
    """(status code, bad index) the entry reports: the first invalid request's, else CODE_CAPACITY (-1) when the layout
    does not fit, else (0, -1)"""
    if bad >= 0:
        return codes[bad], bad
    if total > src_bytes:
        return CODE_CAPACITY, -1
    return 0, -1
