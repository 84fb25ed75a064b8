"""NumPy oracle of the batched fetch-ops (dds_get_accumulate_batch / dds_get_accumulate_samples): calls applied to a
world of shards, each returning the previous rows.

Requests, the layout of src, validation and errors are the accumulate's (tests/put_oracle.py: requests, locate and
expected_error; tests/acc_oracle.py: add, one rounded addition per type). For every element e of a valid request's
rows, in one atomic step, result[e] = shard[e] and shard[e] becomes shard[e] + src[e] (OP_SUM) or src[e] (OP_REPLACE).
result has src's layout; an invalid request's result bytes, every byte past the layout and -- after a capacity error --
the whole buffer are left as they were.

`fetch_op` applies the calls' requests in order, one element after the other: that is one of the orders the device may
take. `check` compares a device outcome with the calls:
  * an element touched once: its previous value is the shard's bits exactly (NaN payloads, -0 and f32 subnormals
    included); its new value is the operand's bits (OP_REPLACE) or one correctly rounded addition, compared by
    `acc_oracle.keys` (every NaN alike), for f32 IEEE or flushed (`acc_oracle.add_flushed`);
  * an element touched several times: the previous values the fetch-ops got and the final value must be explained by
    ONE order of the contributions --
      - OP_SUM: each step one addition of the type (`acc_oracle.add`, for f32 or `add_flushed`) onto the value the
        step got; the first step got v0 bit for bit, a later one the previous step's sum (a NaN by class), and the
        final value is the last sum (by keys). Repeated previous values are allowed (a NaN, a contribution absorbed
        by rounding) as long as one order explains them;
      - OP_REPLACE (distinct src values): v0 -> s_a -> s_b -> ... -> final, each value got back exactly once, by bits.
`check` reports the first inconsistency with its element and inputs, or None.

The second half checks the arithmetic at single elements: `admissible_fetch` (every admissible tuple of previous values
and final value of an element with a few fetch-adds, and optionally one plain accumulate), `fetch_verdict` (names the
first element outside it), `fop_path` (which atomic and which result write an element of a one-piece call takes), and
the value generators of the GPU module.
"""
import itertools

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


SEARCH = 8  # chains of at most this many fetch-adds are searched over every order when the first walk fails


def bits64(a, t):
    """the bit patterns of storage array `a` as int64"""
    return ao.bits(np.asarray(a, ao.STORAGE[t]), t).astype(np.uint64).view(np.int64)


def fmt(v, t):
    """one storage element as its bits and value"""
    a = np.asarray(v, ao.STORAGE[t]).reshape(1)
    w = 2 * np.dtype(ao.BITS[t]).itemsize
    return f"{int(ao.bits(a, t)[0]):#0{w + 2}x} ({ao.values(a, t)[0]!r})"


def _fmt_keys(ks, t):
    w = 2 * np.dtype(ao.BITS[t]).itemsize
    return "{" + ", ".join(sorted({"NaN" if k == ao.NAN else f"{int(k) & ((1 << 4 * w) - 1):#0{w + 2}x}"
                                   for k in np.asarray(ks).tolist()})) + "}"


def new_values(v0, x, t, op):
    """the admissible new values of elements touched once, [options, N]: sums by keys (IEEE, and for f32 flushed),
    swaps the operand's bits"""
    if op == OP_REPLACE:
        return bits64(x, t)[None]
    opts = [ao.keys(ao.add(v0, x, t), t)]
    if t == ao.ACC_F32:
        opts.append(ao.keys(ao.add_flushed(v0, x), t))
    return np.stack(opts)


def _sum_order(v0, x, got, final, t):
    """one order (member indices) that explains a SUM chain -- step 0 got v0 bit for bit, each later step the previous
    sum (bits; a NaN by class), each sum one addition of type t (f32: IEEE or flushed), the final value the last sum
    by keys -- or None. Searched depth first over every order; members with the same operand and value got are
    interchangeable, and (members used, current value) states are visited once."""
    n = x.size
    gb, gn = bits64(got, t), ao.is_nan(got, t)
    xb = bits64(x, t)
    fk = int(ao.keys(final, t)[0])
    seen = set()

    def walk(cur, used, step):
        if step == n:
            return [] if int(ao.keys(cur, t)[0]) == fk else None
        cb = int(bits64(cur, t)[0])
        if (used, cb) in seen:
            return None
        seen.add((used, cb))
        cnan = bool(ao.is_nan(cur, t)[0])
        tried = set()
        for i in range(n):
            if used >> i & 1 or (int(gb[i]), int(xb[i])) in tried:
                continue
            if not (gb[i] == cb or (step and cnan and gn[i])):
                continue
            tried.add((int(gb[i]), int(xb[i])))
            nxt = {int(bits64(s, t)[0]): s for s in
                   [ao.add(got[i:i + 1], x[i:i + 1], t)] + ([ao.add_flushed(got[i:i + 1], x[i:i + 1])]
                                                           if t == ao.ACC_F32 else [])}
            for s in nxt.values():
                rest = walk(s, used | 1 << i, step + 1)
                if rest is not None:
                    return [i] + rest
        return None
    return walk(np.asarray(v0, ao.STORAGE[t]).reshape(1), 0, 0)


def sum_chain(v0, contribs, got, final, t=ao.ACC_I64):
    """None when the previous values `got` of a SUM chain and the final value are explained by one order of the
    contributions (see the module's docstring; chains of at most SEARCH are searched over every order, longer ones
    walked: each step the first fetch-op that got the current value); else what is wrong. Values: storage arrays or
    numbers of type t (the default: int64)"""
    dt = ao.STORAGE[t]
    v0, final = np.asarray(v0, dt).reshape(1), np.asarray(final, dt).reshape(1)
    x, g = np.asarray(contribs, dt).reshape(-1), np.asarray(got, dt).reshape(-1)
    n = x.size
    if n <= SEARCH and _sum_order(v0, x, g, final, t) is not None:
        return None
    gb, gk = bits64(g, t), ao.keys(g, t)
    ctx = (f"(v0 {fmt(v0, t)}, contributions [{', '.join(fmt(a, t) for a in x)}], got "
           f"[{', '.join(fmt(a, t) for a in g)}])") if n <= 16 else f"(v0 {fmt(v0, t)}, {n} fetch-ops)"
    uvals, cnt = np.unique(gb, return_counts=True)
    dup = "" if cnt.max() == 1 else (f"; two fetch-ops got the same value "
                                     f"{fmt(g[np.flatnonzero(gb == uvals[cnt > 1][0])[0]], t)} (a duplicated ticket)")
    cur, used = v0, np.zeros(n, bool)
    for step in range(n):
        ck = int(ao.keys(cur, t)[0])
        hit = np.flatnonzero(~used & ((gb == bits64(cur, t)[0]) if step == 0 else (gk == ck)))
        if not hit.size:
            return f"no fetch-op got {fmt(cur, t)}: the chain expects it after {step} step(s){dup} {ctx}"
        i = hit[0]
        used[i] = True
        cur = ao.add(g[i:i + 1], x[i:i + 1], t)
    if ao.keys(final, t)[0] != ao.keys(cur, t)[0]:
        return f"final value {fmt(final, t)}, the chain expects {fmt(cur, t)} (a lost or extra contribution){dup} {ctx}"
    return f"no order of the contributions explains the values got and the final value, with one rounding per step{dup} {ctx}"


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
            b = ao.BITS[t]
            bad = np.nonzero(got.view(b) != v0.view(b))[0]
            if bad.size:
                j = bad[0]
                return (_elem("previous value", r, int(el[sel][j]), disp, lenlist) +
                        f" (call {int(call[sel][j])}): got {fmt(got[j], t)}, the shard held {fmt(v0[j], t)}")
            new = flatg[r][el[sel]]
            opts = new_values(v0, x, t, op)
            ok = (opts == (ao.keys(new, t) if op == OP_SUM else bits64(new, t))[None]).any(0)
            bad = np.nonzero(~ok)[0]
            if bad.size:
                j = bad[0]
                return (_elem("new value", r, int(el[sel][j]), disp, lenlist) +
                        f": {fmt(new[j], t)}, admissible {_fmt_keys(opts[:, j], t)} (v0 {fmt(v0[j], t)}, src "
                        f"{fmt(x[j], t)})")
    # touched several times: one chain per element (values converted once, the chains walked in plain Python)
    multi = np.flatnonzero((ends - starts) > 1)
    if not multi.size:
        return None
    members = np.flatnonzero(np.repeat((ends - starts) > 1, ends - starts))
    heads = starts[multi]
    v0, final = np.empty(multi.size, dt), np.empty(multi.size, dt)
    for r in range(len(shards0)):
        m = rk[heads] == r
        v0[m], final[m] = flat0[r][el[heads][m]], flatg[r][el[heads][m]]
    xs, gs = np.empty(members.size, dt), np.empty(members.size, dt)
    for c in np.unique(call[members]).tolist():
        m = call[members] == c
        xs[m], gs[m] = src_el[c][si[members][m]], res_el[c][si[members][m]]
    gid = np.repeat(np.arange(multi.size), (ends - starts)[multi])
    bad = _first_bad_chain(gid, xs, gs, v0, final, op, t)
    if bad is None:
        return None
    g = int(multi[bad])
    b = starts[g]
    m = gid == bad
    msg = (sum_chain(v0[bad], xs[m], gs[m], final[bad], t) if op == OP_SUM else
           replace_chain(int(bits64(v0[bad], t)[0]), bits64(xs[m], t).tolist(), bits64(gs[m], t).tolist(),
                         int(bits64(final[bad], t)[0])))
    return _elem("chain", int(rk[b]), int(el[b]), disp, lenlist) + f": {msg}"


def _first_bad_chain(gid, x, got, v0, final, op, t):
    """the first group whose chain fails, or None: all groups walked at once, each step taking the first unused member
    that got the chain's current value (sums: one IEEE addition per step); a group that fails that walk and has at
    most SEARCH members is then searched over every order and f32 mode (sum_chain). gid: each member's group (sorted),
    x / got: its operand and previous value, v0 / final: per group (storage arrays)"""
    G = v0.size
    n_g = np.bincount(gid, minlength=G)
    failed = np.zeros(G, bool)
    if op == OP_SUM:
        gk = ao.keys(got, t)  # (a NaN got matches a NaN sum by class; the first step is checked bit for bit below)
    else:
        gk = bits64(got, t)
        o = np.lexsort((gk, gid))  # distinct operands: each value is got once
        same = (gid[o][1:] == gid[o][:-1]) & (gk[o][1:] == gk[o][:-1])
        failed[gid[o][1:][same]] = True
    uv = np.unique(gk)
    key = gid.astype(np.int64) * uv.size + np.searchsorted(uv, gk)
    ko = np.argsort(key, kind="stable")
    ks = key[ko]
    used = np.zeros(got.size, bool)
    cur = v0.copy()
    for step in range(int(n_g.max())):
        act = np.flatnonzero((step < n_g) & ~failed)
        if not act.size:
            break
        ck = ao.keys(cur[act], t) if op == OP_SUM else bits64(cur[act], t)
        pos = np.minimum(np.searchsorted(uv, ck), uv.size - 1)
        k = act.astype(np.int64) * uv.size + pos
        j = np.minimum(np.searchsorted(ks, k), ks.size - 1)
        hit = (uv[pos] == ck) & (ks[j] == k)
        m = ko[j]
        hit &= ~used[m]
        if op == OP_SUM and step == 0:
            hit &= bits64(got[m], t) == bits64(cur[act], t)
        failed[act[~hit]] = True
        act, m = act[hit], m[hit]
        used[m] = True
        cur[act] = ao.add(got[m], x[m], t) if op == OP_SUM else x[m]
    failed |= (ao.keys(cur, t) != ao.keys(final, t)) if op == OP_SUM else (bits64(cur, t) != bits64(final, t))
    for g in np.flatnonzero(failed & (n_g <= SEARCH)) if op == OP_SUM else ():
        m = gid == g
        failed[g] = _sum_order(v0[g:g + 1], x[m], got[m], final[g:g + 1], t) is None
    bad = np.flatnonzero(failed)
    return int(bad[0]) if bad.size else None


# ------------------------------------------------------------------------------------------------ the arithmetic
def admissible_fetch(start, contribs, t, acc=None):
    """every (previous value of each fetch-add, final value) tuple the header allows for elements with start value
    `start` ([N] storage array) and k <= 3 fetch-adds `contribs` (k arrays of start's shape), plus, when given, one
    plain accumulate `acc` (no previous value): all orders, each f32 step IEEE or flushed. Returns (prev [options, k,
    N], final [options, N]): final values as acc_oracle.keys; previous values as bits (int64), except NAN where the
    value is a NaN some addition made (its payload is not specified), so that a previous value matches when its bits
    are equal or both are NaN there (`fetch_match`)."""
    contribs = list(contribs)
    assert len(contribs) <= 3
    items = list(range(len(contribs))) + ([-1] if acc is not None else [])
    prevs, finals = [], []
    for order in itertools.permutations(items):
        for mask in range(1 << len(items)) if t == ao.ACC_F32 else (0,):
            cur = np.asarray(start, ao.STORAGE[t])
            made = np.zeros(cur.shape, bool)  # cur is a NaN an addition made
            prev = [None] * len(contribs)
            for step, i in enumerate(order):
                if i >= 0:
                    prev[i] = np.where(made, ao.NAN, bits64(cur, t))
                x = acc if i < 0 else contribs[i]
                cur = ao.add_flushed(cur, x) if mask >> step & 1 else ao.add(cur, x, t)
                made = ao.is_nan(cur, t)
            prevs.append(np.stack(prev) if prev else np.zeros((0,) + cur.shape, np.int64))
            finals.append(ao.keys(cur, t))
    return np.stack(prevs), np.stack(finals)


def fetch_match(opts, got_prev, got_final, t):
    """[N] bool: the observed tuple -- got_prev [k, N], got_final [N] (storage arrays) -- is one of admissible_fetch's
    options `opts`"""
    prev, final = opts
    gb = bits64(got_prev, t)[None]
    gn = ao.is_nan(got_prev, t)[None]
    okp = ((prev == gb) | ((prev == ao.NAN) & gn)).all(1)
    return (okp & (final == ao.keys(got_final, t)[None])).any(0)


def discrimination(opts):
    """the fraction of elements with more than one distinct admissible tuple"""
    prev, final = opts
    differ = (prev != prev[:1]).any(1) | (final != final[:1])
    return float(differ.any(0).mean()) if final.shape[1] else 0.0


def fetch_verdict(got_prev, got_final, start, contribs, t, acc=None, opts=None, where=None, paths=None, what=""):
    """None when every element's observed tuple (got_prev [k, N], got_final [N]) is admissible; else a message naming
    the first bad element -- `where(i)` -> (rank, global row, column) -- with its inputs, the bits it got, the
    admissible tuples and, when given, its predicted path"""
    opts = admissible_fetch(start, contribs, t, acc) if opts is None else opts
    ok = fetch_match(opts, got_prev, got_final, t)
    if ok.all():
        return None
    i = int(np.argmin(ok))
    rank, row, col = where(i) if where else (0, i, 0)
    w = 2 * np.dtype(ao.BITS[t]).itemsize
    f = lambda k: "NaN" if k == ao.NAN else f"{int(k) & ((1 << 4 * w) - 1):#0{w + 2}x}"  # noqa: E731
    tuples = sorted({"(" + ", ".join(f(k) for k in list(opts[0][o, :, i]) + [opts[1][o, i]]) + ")"
                     for o in range(opts[1].shape[0])})
    ins = ", ".join(fmt(np.asarray(c)[i], t) for c in contribs)
    got = ", ".join(fmt(np.asarray(got_prev)[j, i], t) for j in range(len(contribs)))
    return (f"{what}: {int((~ok).sum())} of {ok.size} elements outside the admissible set; first: rank {rank}, global row "
            f"{row}, column {col}{'' if paths is None else f' (path {paths[i]})'}: start {fmt(np.asarray(start)[i], t)}, "
            f"fetch-adds [{ins}]{'' if acc is None else f', accumulate {fmt(np.asarray(acc)[i], t)}'}: got previous "
            f"values [{got}], final {fmt(np.asarray(got_final)[i], t)}; admissible (previous values..., final): "
            f"{', '.join(tuples[:12])}{' ...' if len(tuples) > 12 else ''}")


def once_verdict(got_prev, got_new, start, x, t, op, where=None, paths=None, what=""):
    """None when every once-touched element (all [N] storage arrays) got the shard's bits back and holds an admissible
    new value; else a message naming the first bad element with its inputs, the bits got, the admissible bits and,
    when given, its predicted path"""
    okp = bits64(got_prev, t) == bits64(start, t)
    opts = new_values(start, x, t, op)
    okn = (opts == (ao.keys(got_new, t) if op == OP_SUM else bits64(got_new, t))[None]).any(0)
    ok = okp & okn
    if ok.all():
        return None
    i = int(np.argmin(ok))
    rank, row, col = where(i) if where else (0, i, 0)
    return (f"{what}: {int((~okp).sum())} previous and {int((~okn).sum())} new values of {ok.size} wrong; first: rank "
            f"{rank}, global row {row}, column {col}{'' if paths is None else f' (path {paths[i]})'}: shard "
            f"{fmt(start[i], t)}, src {fmt(x[i], t)}: got previous value {fmt(got_prev[i], t)} (admissible: the shard's "
            f"bits), new value {fmt(got_new[i], t)} (admissible {_fmt_keys(opts[:, i], t)})")


# ------------------------------------------------------------------------------------------------ paths
def fop_path(dst_phase, src_phase, nbytes, k, res_phase=0):
    """which atomic the fetch drain (write_chunk<kActFetch>) applies to byte k of ONE staged piece of nbytes bytes whose shard
    bytes start dst_phase and whose staged operands start src_phase bytes past a 16-byte boundary: "element" (fetch1)
    for the head before the shard's first 16-byte boundary and the tail after its last; for the body between,
    "vector WS/B", write_loop<kActFetch, WS, BYTES> with the word shift WS and BYTES (0 / 1) of the staged phase
    (src_phase + head) % 16. k may be an array. Also returns how the previous values reach the result whose bytes start
    res_phase past a boundary: "bulk" (one bulk store) when result, size and staged phase are all 16-byte aligned,
    else "drain_chunk" (the raw drain's head / body / tail)."""
    k = np.asarray(k)
    head = min((16 - dst_phase) % 16, nbytes)
    body = ((nbytes - head) >> 4) << 4
    sh = (src_phase + head) % 16
    path = np.where((k < head) | (k >= head + body), "element", f"vector {sh >> 2}/{int(sh % 4 != 0)}")
    return path, "bulk" if (res_phase | nbytes | src_phase) % 16 == 0 else "drain_chunk"


def vector_paths(t):
    """the write_loop<kActFetch> variants elements of type t can take: 8 for 2-byte types, 4 for 4-byte, 2 for 8-byte"""
    E = np.dtype(ao.STORAGE[t]).itemsize
    return [f"vector {sh >> 2}/{int(sh % 4 != 0)}" for sh in range(0, 16, E)]


# ------------------------------------------------------------------------------------------------ test data
def swap_patterns(rng, t, n):
    """n bit patterns from the whole range of type t: signalling NaNs with payload 1, negative and low-payload NaNs,
    +-0, subnormals, +-inf, +-max and random bits (integers: random bits and the range's ends)"""
    nb = np.dtype(ao.BITS[t]).itemsize * 8
    rnd = rng.integers(0, 2**63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    rnd = rnd.astype(ao.BITS[t])
    if t not in ao.FLOATS:
        ends = np.array([0, 1, (1 << (nb - 1)) - 1, 1 << (nb - 1), (1 << nb) - 1], np.uint64).astype(ao.BITS[t])
        return ao.from_bits(np.where(rng.random(n) < 0.3, ends[rng.integers(0, ends.size, size=n)], rnd), t)
    p = ao.PREC[t]
    sign = np.uint64(1) << np.uint64(nb - 1)
    special = [ao._nan_bits(t, q) for q in range(4)] + [0, 1, (1 << (p - 1)) - 1, 1 << (p - 1), ao._max_bits(t),
                                                        ((1 << (nb - 1)) - 1) & ~((1 << (p - 1)) - 1)]
    special = np.array(special, np.uint64)
    sp = special[rng.integers(0, special.size, size=n)] | np.where(rng.random(n) < 0.5, sign, np.uint64(0))
    sub = rng.integers(1, 1 << (p - 1), size=n).astype(np.uint64) | np.where(rng.random(n) < 0.5, sign, np.uint64(0))
    k = rng.integers(0, 4, size=n)
    return ao.from_bits(np.where(k == 0, rnd, np.where(k == 1, sub, sp)).astype(ao.BITS[t]), t)


def distinct_patterns(rng, t, n, avoid=()):
    """n distinct bit patterns of type t, every NaN kind, +-0, subnormals, +-inf and max among them when n allows,
    none of them in `avoid` (bits)"""
    nb = np.dtype(ao.BITS[t]).itemsize * 8
    first = ao.bits(swap_patterns(rng, t, 4 * n + 64), t)
    if t in ao.FLOATS:
        p = ao.PREC[t]
        sign = 1 << (nb - 1)
        e = ((1 << (nb - 1)) - 1) & ~((1 << (p - 1)) - 1)
        first = np.concatenate([np.array([ao._nan_bits(t, q) | s for q in range(4) for s in (0, sign)] +
                                         [0, sign, 1, 1 | sign, e, e | sign, ao._max_bits(t)], np.uint64
                                         ).astype(ao.BITS[t]), first])
    _, idx = np.unique(first, return_index=True)
    out = first[np.sort(idx)]
    out = out[~np.isin(out, np.asarray(avoid, ao.BITS[t]))]
    assert out.size >= n, (t, n, out.size)
    sel = np.concatenate([np.arange(min(15, n)), 15 + rng.permutation(out.size - 15)[:max(n - 15, 0)]])
    return ao.from_bits(out[rng.permutation(sel)], t)


# hot elements: fetch-adds per element of positive operands in (1, 2) onto a start value in [1, 2). Below these counts
# every addition raises the running sum (the sum stays below 2^(p+1): an ulp of at most 2), so sorting the previous
# values gives the only order
HOT_FETCH = {ao.ACC_F32: 4096, ao.ACC_F64: 65536, ao.ACC_F16: 512, ao.ACC_BF16: 128, ao.ACC_I32: 4096, ao.ACC_I64: 4096}


def hot_values(rng, t, shape):
    """positive operands of type t: floats in (1, 2) with random full-precision significands, integers in [1, 2^18)"""
    if t not in ao.FLOATS:
        return rng.integers(1, 1 << 18, size=shape).astype(ao.STORAGE[t])
    p = ao.PREC[t]
    m = (1 << (p - 1)) + rng.integers(1, 1 << (p - 1), size=shape, dtype=np.int64)
    return ao.encode(np.ldexp(m.astype(np.float64), -(p - 1)), t)


def increasing_chain(v0, x, got, final, t):
    """the hot-element check of elements whose contributions all raise the running sum: per column of x / got
    ([n, D] storage arrays; v0, final [D]), the previous values sorted give the only order, so sorted[0] is v0 bit for
    bit, sorted[j + 1] = add(sorted[j], its contribution) bit for bit and final = add(last, its contribution). Returns
    None or (column, what is wrong)."""
    gv = ao.values(got, t)
    order = np.argsort(gv, axis=0, kind="stable")
    gs = np.take_along_axis(got, order, 0)
    xs = np.take_along_axis(x, order, 0)
    nxt = ao.add(gs, xs, t)
    b = lambda a: bits64(a, t)  # noqa: E731
    bad0 = b(gs[0]) != b(v0)
    if bad0.any():
        c = int(np.argmax(bad0))
        return c, f"the smallest previous value {fmt(gs[0, c], t)} is not the start {fmt(v0[c], t)}"
    badm = b(gs[1:]) != b(nxt[:-1])
    if badm.any():
        j, c = (int(v) for v in np.argwhere(badm)[0])
        eq = " (two fetch-ops got the same value: a duplicated ticket)" if b(gs[j + 1, c]) == b(gs[j, c]) else ""
        return c, (f"step {j + 1} of {got.shape[0]}: got {fmt(gs[j + 1, c], t)}, one rounded addition of "
                   f"{fmt(xs[j, c], t)} onto {fmt(gs[j, c], t)} gives {fmt(nxt[j, c], t)}{eq}")
    badf = b(final) != b(nxt[-1])
    if badf.any():
        c = int(np.argmax(badf))
        return c, f"final value {fmt(final[c], t)}, the chain ends at {fmt(nxt[-1, c], t)}"
    return None
