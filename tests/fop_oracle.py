"""NumPy oracle of the batched fetch-ops (dds_get_accumulate_batch / dds_get_accumulate_samples): calls applied to a
world of shards, each returning the previous rows.

Requests, the layout of src, validation and errors are the accumulate's (tests/put_oracle.py: requests, locate and
expected_error; tests/acc_oracle.py: add, one rounded addition per type). For every element e of a valid request's
rows, in one atomic step, result[e] = shard[e] and shard[e] becomes shard[e] + src[e] (OP_SUM) or src[e] (OP_REPLACE).
result has src's layout; an invalid request's result bytes, every byte past the layout and -- after a capacity error --
the whole buffer are left as they were.

`fetch_op` applies the calls' requests in order, one element after the other: that is one of the orders the device may
take, so its shards and results are exact for every element one epoch touches once. For elements touched by several
fetch-ops, `check` compares each with a chain instead: the previous values the fetch-ops got and the final value must
be explained by ONE order of the contributions --
  * OP_SUM (integer-valued, positive contributions): sorted by the value each got back, contribution k got v0 plus the
    k before it, and the final value is v0 plus all of them;
  * OP_REPLACE (distinct src values): v0 -> s_a -> s_b -> ... -> final, each value got back exactly once.
`check` reports the first inconsistency with its element and inputs, or None.
"""
import numpy as np

from tests import acc_oracle as ao
from tests import put_oracle as po

OP_SUM, OP_REPLACE = 1, 2
OPS = {"sum": OP_SUM, "replace": OP_REPLACE}


def plan(shards, t, src_bytes, **req):
    """the put's plan of one call -> (codes, [(rank, first local row, count, src byte offset, bytes)], bad, total,
    applied: the layout fits)"""
    lenlist = po.lenlist_of(shards)
    rows = int(lenlist[-1]) if len(lenlist) else 0
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    row_bytes = np.dtype(ao.STORAGE[t]).itemsize * disp
    codes, pl, o = [], [], 0
    for start, count, id_ok in po.requests(**req):
        n = count * row_bytes if id_ok and 0 < count <= rows else 0
        code, r, off = (po.CODE_SAMPLE, 0, 0) if not id_ok else po.locate(lenlist, start, count)
        codes.append(code)
        pl.append((r, start - off, count, o, n))
        o += n
    bad = next((i for i, c in enumerate(codes) if c), -1)
    return codes, pl, bad, o, o <= src_bytes


def fetch_op(shards, src, t, op, result, src_bytes=None, **req):
    """Apply one fetch-op call to `shards` (not modified), request by request. src: the packed operands as bytes;
    result: the caller's result buffer before the call, as bytes (not modified). Returns (new shards, new result,
    per-request codes, first bad index or -1, layout total)."""
    dt = np.dtype(ao.STORAGE[t])
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    src = np.asarray(src, np.uint8).reshape(-1)
    src_bytes = src.size if src_bytes is None else src_bytes
    codes, pl, bad, total, applied = plan(shards, t, src_bytes, **req)
    new = [s.copy() for s in shards]
    res = np.array(result, np.uint8).reshape(-1)
    if applied:
        for (r, local, count, off, n), code in zip(pl, codes):
            if code == 0 and n > 0:
                rows_r = new[r].reshape(new[r].shape[0], -1)
                old = rows_r[local:local + count].copy()
                x = src[off:off + n].view(dt).reshape(count, disp)
                rows_r[local:local + count] = ao.add(old, x, t) if op == OP_SUM else x
                res[off:off + n] = old.reshape(-1).view(np.uint8)
    return new, res, codes, bad, total


def fetch_op_many(shards, calls, t, op):
    """Apply `calls` = [(src, src_bytes or None, result, request keywords)] in order -> (new shards, [new result per call],
    [(status code, bad index, layout total)] as each call reports them)"""
    results, out = [], []
    for src, src_bytes, result, req in calls:
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        shards, res, codes, bad, total = fetch_op(shards, src, t, op, result, src_bytes=sb, **req)
        results.append(res)
        out.append(po.expected_error(codes, bad, total, sb) + (total,))
    return shards, results, out


def touches(shards, calls, t):
    """every element the calls' valid requests touch -> (rank, local element index, call, element index in the call's
    src) arrays, grouped by element (one epoch's view: calls of any rank, in any order)"""
    E = np.dtype(ao.STORAGE[t]).itemsize
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    parts = []
    for k, (src, src_bytes, _result, req) in enumerate(calls):
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        codes, pl, _bad, _total, applied = plan(shards, t, sb, **req)
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
    o = np.lexsort((a[2], a[0], a[1]))  # by element, then call (stable within a call: request order)
    a = a[:, o]
    o = np.lexsort((a[1], a[0]))
    return tuple(a[:, o])


def _elem(what, r, e, disp, lenlist):
    row = e // disp + (int(lenlist[r - 1]) if r else 0)
    return f"{what}: rank {r} global row {row} column {e % disp}"


def sum_chain(v0, contribs, got, final):
    """None when the previous values `got` of an integer-valued SUM chain and the final value are explained by one
    order of the (positive) contributions; else what is wrong"""
    order = sorted(range(len(got)), key=lambda i: got[i])
    acc = v0
    for k, i in enumerate(order):
        if k and got[i] == got[order[k - 1]]:
            return f"two fetch-ops got the same value {got[i]} (a duplicated ticket)"
        if got[i] != acc:
            return f"fetch-op {i} got {got[i]}, the chain expects {acc} (contributions {contribs}, got {got}, v0 {v0})"
        acc += contribs[i]
    if final != acc:
        return f"final value {final}, the chain expects {acc} (a lost or extra contribution; v0 {v0}, contributions " \
               f"{contribs}, got {got})"
    return None


def replace_chain(v0, srcs, got, final):
    """None when the previous values `got` of swaps with distinct `srcs` and the final value form one chain
    v0 -> s_a -> s_b -> ... -> final; else what is wrong"""
    by_got = {}
    for i, g in enumerate(got):
        if g in by_got:
            return f"fetch-ops {by_got[g]} and {i} both got {g}"
        by_got[g] = i
    cur = v0
    for _ in range(len(srcs)):
        i = by_got.pop(cur, None)
        if i is None:
            return f"no fetch-op got {cur}, the chain's next value (v0 {v0}, srcs {srcs}, got {got})"
        cur = srcs[i]
    if by_got:
        return f"value(s) {sorted(by_got)} outside the chain (v0 {v0}, srcs {srcs}, got {got})"
    if final != cur:
        return f"final value {final}, the chain ends at {cur} (v0 {v0}, srcs {srcs}, got {got})"
    return None


def check(shards0, calls, t, op, got_shards, got_results):
    """Compare what the device left -- got_shards (one storage array per rank, rows only) and got_results (each call's
    result buffer, bytes) -- with the calls [(src, src_bytes or None, result before the call, request keywords)] of one
    epoch: elements touched once exactly (previous value and new value, bit for bit), elements touched several times by
    their chain (integer-valued data), every other shard element and result byte unchanged. Returns None or the first
    inconsistency."""
    dt = np.dtype(ao.STORAGE[t])
    E = dt.itemsize
    lenlist = po.lenlist_of(shards0)
    disp = shards0[0].shape[1] if shards0[0].ndim > 1 else 1
    flat0 = [np.ascontiguousarray(s).reshape(-1) for s in shards0]
    flatg = [np.ascontiguousarray(s).reshape(-1) for s in got_shards]
    srcs = [np.asarray(c[0], np.uint8).reshape(-1) for c in calls]
    # result bytes outside the applied valid requests: untouched
    for k, (src, src_bytes, result, req) in enumerate(calls):
        sb = srcs[k].size if src_bytes is None else src_bytes
        codes, pl, _bad, _total, applied = plan(shards0, t, sb, **req)
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
    rk, el, call, si = touches(shards0, calls, t)
    # shard elements no request touches: unchanged
    for r in range(len(shards0)):
        keep = np.ones(flat0[r].size, bool)
        keep[el[rk == r]] = False
        d = np.nonzero(keep & (flat0[r].view(ao.BITS[t]) != flatg[r].view(ao.BITS[t])))[0]
        if d.size:
            return _elem("an element no request touches changed", r, int(d[0]), disp, lenlist)
    if not rk.size:
        return None
    src_el = [s[:s.size // E * E].view(dt) for s in srcs]
    res_el = [np.asarray(g, np.uint8).reshape(-1) for g in got_results]
    res_el = [g[:g.size // E * E].view(dt) for g in res_el]
    key = rk * (1 << 40) + el
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    ends = np.r_[starts[1:], key.size]
    once = starts[(ends - starts) == 1]
    # touched once: exact, bit for bit
    if once.size:
        for r in range(len(shards0)):
            sel = once[rk[once] == r]
            if not sel.size:
                continue
            v0 = flat0[r][el[sel]]
            x, got = np.empty(sel.size, dt), np.empty(sel.size, dt)
            for c in np.unique(call[sel]).tolist():
                m = call[sel] == c
                x[m], got[m] = src_el[c][si[sel][m]], res_el[c][si[sel][m]]
            exp_new = ao.add(v0, x, t) if op == OP_SUM else x
            b = ao.BITS[t]
            bad = np.nonzero(got.view(b) != v0.view(b))[0]
            if bad.size:
                j = bad[0]
                return (_elem("previous value", r, int(el[sel][j]), disp, lenlist) +
                        f" (call {int(call[sel][j])}): got {got[j]!r}, the shard held {v0[j]!r}")
            bad = np.nonzero(flatg[r][el[sel]].view(b) != exp_new.view(b))[0]
            if bad.size:
                j = bad[0]
                return (_elem("new value", r, int(el[sel][j]), disp, lenlist) +
                        f": {flatg[r][el[sel][j]]!r}, expected {exp_new[j]!r} (v0 {v0[j]!r}, src {x[j]!r})")
    # touched several times: one chain per element (values converted once, the chains walked in plain Python)
    multi = np.flatnonzero((ends - starts) > 1)
    if not multi.size:
        return None
    if op == OP_SUM:
        def conv(a):
            return ao.values(np.asarray(a, dt), t)
    else:
        def conv(a):
            return np.asarray(a, dt).view(ao.BITS[t]).astype(np.int64)
    members = np.flatnonzero(np.repeat((ends - starts) > 1, ends - starts))
    heads = starts[multi]
    v0, final = np.empty(multi.size, dt), np.empty(multi.size, dt)
    for r in range(len(shards0)):
        m = rk[heads] == r
        v0[m], final[m] = flat0[r][el[heads][m]], flatg[r][el[heads][m]]
    v0, final = conv(v0), conv(final)
    xs, gs = np.empty(members.size, dt), np.empty(members.size, dt)
    for c in np.unique(call[members]).tolist():
        m = call[members] == c
        xs[m], gs[m] = src_el[c][si[members][m]], res_el[c][si[members][m]]
    bad = _first_bad_chain(np.repeat(np.arange(multi.size), (ends - starts)[multi]), conv(xs), conv(gs), v0, final, op)
    if bad is None:
        return None
    g = int(multi[bad])
    b, e = starts[g], ends[g]
    xs_g = conv(np.array([src_el[c][i] for c, i in zip(call[b:e].tolist(), si[b:e].tolist())], dt))
    gs_g = conv(np.array([res_el[c][i] for c, i in zip(call[b:e].tolist(), si[b:e].tolist())], dt))
    msg = (sum_chain if op == OP_SUM else replace_chain)(v0[bad].item(), xs_g.tolist(), gs_g.tolist(), final[bad].item())
    return _elem("chain", int(rk[b]), int(el[b]), disp, lenlist) + f": {msg}"


def _first_bad_chain(gid, x, got, v0, final, op):
    """the first group whose chain fails (sum_chain / replace_chain, all groups at once), or None. gid: each member's
    group (sorted), x / got: its operand and previous value, v0 / final: per group (lists of numbers)"""
    x, got = np.asarray(x), np.asarray(got)
    v0, final = np.asarray(v0), np.asarray(final)
    G = v0.size
    n_g = np.bincount(gid, minlength=G)
    failed = np.zeros(G, bool)
    o = np.lexsort((got, gid))  # two members of a group with the same previous value
    same = (gid[o][1:] == gid[o][:-1]) & (got[o][1:] == got[o][:-1])
    failed[gid[o][1:][same]] = True
    uv = np.unique(got)
    key = gid.astype(np.int64) * uv.size + np.searchsorted(uv, got)
    ko = np.argsort(key, kind="stable")
    ks = key[ko]
    used = np.zeros(got.size, bool)
    cur = v0.copy()
    for step in range(int(n_g.max())):
        act = np.flatnonzero((step < n_g) & ~failed)
        if not act.size:
            break
        pos = np.minimum(np.searchsorted(uv, cur[act]), uv.size - 1)
        k = act.astype(np.int64) * uv.size + pos
        j = np.minimum(np.searchsorted(ks, k), ks.size - 1)
        hit = (uv[pos] == cur[act]) & (ks[j] == k)
        m = ko[j]
        hit &= ~used[m]
        failed[act[~hit]] = True
        act, m = act[hit], m[hit]
        used[m] = True
        cur[act] = cur[act] + x[m] if op == OP_SUM else x[m]
    failed |= cur != final
    bad = np.flatnonzero(failed)
    return int(bad[0]) if bad.size else None
