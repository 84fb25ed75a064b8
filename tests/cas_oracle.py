"""NumPy oracle of the batched compare-and-swaps (dds_compare_and_swap_batch / dds_compare_and_swap_samples): calls applied
to a world of shards, each returning the previous rows.

Requests, the layout of src, validation and errors are the put's (tests/put_oracle.py: requests, locate and
expected_error). Elements are the variable's itemsize E (1, 2, 4 or 8 bytes) and compared BIT FOR BIT: the oracle works on
the unsigned integers of width E, so -0 and +0 differ and a NaN equals only its own bits. For every element e of a valid
request's rows, in one atomic step, result[e] = shard[e], and shard[e] becomes src[e] if it equalled compare[e]. compare
and result have src's layout; an invalid request's result bytes, every byte past the layout and -- after a capacity
error -- the whole buffer are left as they were.

`cas` applies the calls' requests in order, one element after the other: that is one of the orders the device may take.
`check` compares a device outcome with the calls: an element touched once must return the shard's bits and hold the
one possible new value; an element touched several times must be explained by ONE order of its compare-and-swaps, each
getting the value left by the one before it, the last leaving the final value (a search over the orders). Every other shard element and result byte must be unchanged. It reports the first inconsistency by
rank, global row and column, or None.
"""
import itertools

import numpy as np

from tests import put_oracle as po

UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
SEARCH_STEPS = 1 << 16  # states searched per element before an order is given up
VECTOR = 5  # elements with at most this many compare-and-swaps are checked in every order at once


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(UINT[a.dtype.itemsize])


def plan(shards, src_bytes, **req):
    """the put's plan of one call -> (codes, [(rank, first local row, count, src byte offset, bytes)], bad, total,
    applied: the layout fits)"""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1]) if len(lenlist) else 0
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    row_bytes = shards[0].dtype.itemsize * disp
    codes, pl, o = [], [], 0
    for start, count, id_ok in po.requests(**req):
        n = count * row_bytes if id_ok and 0 < count <= rows else 0
        code, r, off = (po.CODE_SAMPLE, 0, 0) if not id_ok else po.locate(lenlist, start, count)
        codes.append(code)
        pl.append((r, start - off, count, o, n))
        o += n
    bad = next((i for i, c in enumerate(codes) if c), -1)
    return codes, pl, bad, o, o <= src_bytes


def cas(shards, src, compare, result, src_bytes=None, **req):
    """Apply one compare-and-swap call to `shards` (not modified), request by request. src, compare: the packed operands
    as bytes; result: the caller's result buffer before the call, as bytes (not modified). Returns (new shards, new
    result, per-request codes, first bad index or -1, layout total)."""
    E = shards[0].dtype.itemsize
    u = UINT[E]
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    src = np.asarray(src, np.uint8).reshape(-1)
    cmp = np.asarray(compare, np.uint8).reshape(-1)
    src_bytes = src.size if src_bytes is None else src_bytes
    codes, pl, bad, total, applied = plan(shards, src_bytes, **req)
    new = [s.copy() for s in shards]
    res = np.array(result, np.uint8).reshape(-1)
    if applied:
        for (r, local, count, off, n), code in zip(pl, codes):
            if code == 0 and n > 0:
                rows_r = _bits(new[r]).reshape(new[r].shape[0], -1)
                old = rows_r[local:local + count].copy()
                x = src[off:off + n].view(u).reshape(count, disp)
                c = cmp[off:off + n].view(u).reshape(count, disp)
                rows_r[local:local + count] = np.where(old == c, x, old)
                res[off:off + n] = old.reshape(-1).view(np.uint8)
    return new, res, codes, bad, total


def cas_many(shards, calls):
    """Apply `calls` = [(src, src_bytes or None, compare, result, request keywords)] in order -> (new shards, [new result
    per call], [(status code, bad index, layout total)] as each call reports them)"""
    results, out = [], []
    for src, src_bytes, compare, result, req in calls:
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        shards, res, codes, bad, total = cas(shards, src, compare, result, src_bytes=sb, **req)
        results.append(res)
        out.append(po.expected_error(codes, bad, total, sb) + (total,))
    return shards, results, out


def touches(shards, calls):
    """every element the calls' valid requests touch -> (rank, local element index, call, element index in the call's
    src) arrays, grouped by element, request order kept within a call"""
    E = shards[0].dtype.itemsize
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    parts = []
    for k, (src, src_bytes, _cmp, _result, req) in enumerate(calls):
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        codes, pl, _bad, _total, applied = plan(shards, sb, **req)
        if not applied:
            continue
        for (r, local, count, off, n), code in zip(pl, codes):
            if code == 0 and n > 0:
                m = count * disp
                parts.append(np.stack([np.full(m, r), local * disp + np.arange(m), np.full(m, k),
                                       off // E + np.arange(m)]))
    if not parts:
        return (np.zeros(0, np.int64),) * 4
    a = np.concatenate(parts, axis=1).astype(np.int64)
    o = np.lexsort((a[2], a[1], a[0]))
    return tuple(a[:, o])


def _elem(what, r, e, disp, lenlist):
    row = e // disp + (int(lenlist[r - 1]) if r else 0)
    return f"{what}: rank {r} global row {row} column {e % disp}"


def order(v0, ops, final):
    """None when the compare-and-swaps `ops` = [(compare, src, got)] (ints) on one element with start value v0 have an
    order in which each got the value left by the one before it and the last left `final`; else what is wrong. The
    walk takes every op that got the current value and leaves it as it is (a failed compare, or a swap with the same
    value) at once, and searches over the ones that change it, remembering the states that failed (at most SEARCH_STEPS
    states per element)."""
    dead, steps = set(), [0]

    def walk(cur, left):
        same = frozenset(i for i in left if ops[i][2] == cur and (ops[i][0] != cur or ops[i][1] == cur))
        left = left - same
        if not left:
            return cur == final
        if (cur, left) in dead or steps[0] > SEARCH_STEPS:
            return False
        steps[0] += 1
        for i in sorted(i for i in left if ops[i][2] == cur):
            if walk(ops[i][1], left - {i}):
                return True
        dead.add((cur, left))
        return False
    if walk(v0, frozenset(range(len(ops)))):
        return None
    got = [o[2] for o in ops]
    wins = [i for i, o in enumerate(ops) if o[2] == o[0]]
    return (f"no order explains it: start {v0:#x}, final {final:#x}, compare/src/got "
            f"{[(hex(c), hex(s), hex(g)) for c, s, g in ops[:12]]}{' ...' if len(ops) > 12 else ''} "
            f"({len(wins)} got their compare value; values got: {sorted(set(hex(g) for g in got))[:8]})")


def check(shards0, calls, got_shards, got_results):
    """Compare what the device left -- got_shards (one storage array per rank, rows only) and got_results (each call's
    result buffer, bytes) -- with the calls [(src, src_bytes or None, compare, result before the call, request keywords)]
    of one epoch. Returns None or the first inconsistency."""
    E = shards0[0].dtype.itemsize
    u = UINT[E]
    lenlist = po.lenlist_of(shards0)
    disp = shards0[0].shape[1] if shards0[0].ndim > 1 else 1
    flat0 = [_bits(s).reshape(-1) for s in shards0]
    flatg = [_bits(s).reshape(-1) for s in got_shards]
    srcs = [np.asarray(c[0], np.uint8).reshape(-1) for c in calls]
    cmps = [np.asarray(c[2], np.uint8).reshape(-1) for c in calls]
    # result bytes outside the applied valid requests: untouched
    for k, (_src, src_bytes, _cmp, result, req) in enumerate(calls):
        sb = srcs[k].size if src_bytes is None else src_bytes
        codes, pl, _bad, _total, applied = plan(shards0, sb, **req)
        mask = np.zeros(np.asarray(result).size, bool)
        if applied:
            for (_r, _l, _c, off, n), code in zip(pl, codes):
                if code == 0:
                    mask[off:off + n] = True
        g, r0 = np.asarray(got_results[k], np.uint8).reshape(-1), np.asarray(result, np.uint8).reshape(-1)
        d = np.nonzero((g != r0) & ~mask)[0]
        if d.size:
            i = next((i for i, (_r, _l, _c, off, n) in enumerate(pl) if off <= d[0] < off + n), None)
            return (f"call {k}: result byte {int(d[0])} written outside the valid requests' rows (request {i}, code "
                    f"{codes[i] if i is not None else None}): {int(r0[d[0]]):#04x} -> {int(g[d[0]]):#04x}")
    rk, el, call, si = touches(shards0, calls)
    # shard elements no request touches: unchanged (for 1- and 2-byte elements, the neighbours in a word)
    for r in range(len(shards0)):
        keep = np.ones(flat0[r].size, bool)
        keep[el[rk == r]] = False
        d = np.nonzero(keep & (flat0[r] != flatg[r]))[0]
        if d.size:
            return _elem("an element no request touches changed", r, int(d[0]), disp, lenlist) + \
                f": {int(flat0[r][d[0]]):#x} -> {int(flatg[r][d[0]]):#x}"
    if not rk.size:
        return None
    src_el = [s[:s.size // E * E].view(u) for s in srcs]
    cmp_el = [s[:s.size // E * E].view(u) for s in cmps]
    res_el = [np.asarray(g, np.uint8).reshape(-1) for g in got_results]
    res_el = [g[:g.size // E * E].view(u) for g in res_el]
    x, c, got = np.empty(rk.size, u), np.empty(rk.size, u), np.empty(rk.size, u)
    for k in np.unique(call).tolist():
        m = call == k
        x[m], c[m], got[m] = src_el[k][si[m]], cmp_el[k][si[m]], res_el[k][si[m]]
    v0, fin = np.empty(rk.size, u), np.empty(rk.size, u)
    for r in range(len(shards0)):
        m = rk == r
        v0[m], fin[m] = flat0[r][el[m]], flatg[r][el[m]]
    key = rk * (1 << 40) + el
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    ends = np.r_[starts[1:], key.size]
    once = starts[(ends - starts) == 1]
    # touched once: exact
    bad = once[got[once] != v0[once]]
    first = None
    if bad.size:
        j = int(bad[0])
        first = (j, _elem("previous value", int(rk[j]), int(el[j]), disp, lenlist) +
                 f" (call {int(call[j])}): got {int(got[j]):#x}, the shard held {int(v0[j]):#x}")
    want = np.where(v0[once] == c[once], x[once], v0[once])
    bad = once[fin[once] != want]
    if bad.size and (first is None or bad[0] < first[0]):
        j = int(bad[0])
        first = (j, _elem("new value", int(rk[j]), int(el[j]), disp, lenlist) +
                 f": {int(fin[j]):#x}, expected {int(want[np.searchsorted(once, j)]):#x} (held {int(v0[j]):#x}, "
                 f"compare {int(c[j]):#x}, src {int(x[j]):#x})")
    # touched several times: one order per element -- elements of up to VECTOR ops tried in every order at once, the
    # others (and any that fail) searched one by one
    sizes = ends - starts
    cand = [starts[sizes > VECTOR]]
    for k in range(2, VECTOR + 1):
        g = starts[sizes == k]
        if not g.size:
            continue
        ok = np.zeros(g.size, bool)
        for perm in itertools.permutations(range(k)):
            cur, fine = v0[g], np.ones(g.size, bool)
            for p in perm:
                i = g + p
                fine &= got[i] == cur
                cur = np.where(cur == c[i], x[i], cur)
            ok |= fine & (fin[g] == cur)
        cand.append(g[~ok])
    for b in np.sort(np.concatenate(cand)).tolist():
        if first is not None and b > first[0]:
            break
        e = b + int(sizes[np.searchsorted(starts, b)])
        ops = list(zip(c[b:e].tolist(), x[b:e].tolist(), got[b:e].tolist()))
        msg = order(int(v0[b]), ops, int(fin[b]))
        if msg is not None:
            first = (b, _elem("compare-and-swaps", int(rk[b]), int(el[b]), disp, lenlist) + f": {msg}")
            break
    return None if first is None else first[1]
