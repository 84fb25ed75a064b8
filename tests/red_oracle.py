"""NumPy oracle of the batched reductions beside the sum: dds_accumulate_op_batch / _samples and dds_get_accumulate_batch /
_samples with DDS_OP_MAX, DDS_OP_MIN, DDS_OP_BAND, DDS_OP_BOR or DDS_OP_BXOR, applied to a world of shards.

Requests, the layout of src, validation and errors are the put's and the fetch-op's (tests/put_oracle.py and
tests/fop_oracle.py: plan, touches and the error rules are reused). For every element e of a valid request's rows the
element becomes `combine(shard[e], src[e])` and, for a fetch, result[e] is the element's value right before. `combine`
is each op's rule for each type, bit for bit:
  - max / min of the integer types compare as SIGNED;
  - max / min of the float types are IEEE 754-2019 maximumNumber / minimumNumber on the bits' total order (-0 < +0,
    subnormals exact, nothing flushed): a NaN operand leaves the element, a NaN element takes the operand, NaN with NaN
    stays a NaN (its bits unspecified: compared by class);
  - and / or / xor work on the bits of the 4- and 8-byte integer types.

`reduce` applies calls request by request: one of the orders the device may take. `check` compares a device outcome
with the calls of one epoch (accumulates and fetches of ONE op and type, in any mix): every element's final value must
be the op folded over its start and every contribution (order-free: these ops commute); its fetch results must be
explained by one order of its contributions, each fetch getting the value left by the ones before it. That is decided
exactly -- as an Eulerian trail from the start value through the fetches' (previous -> combined) steps when every
contribution is a fetch, by a search over every order for up to SEARCH contributions otherwise -- and by necessary
conditions above that (each result is a fold of the start and a subset: for max / min / and / or the results lie
between the start and the final value along the op's order). Every other shard element and result byte must be
unchanged. It names the first bad element by rank, global row and column, with its inputs and the predicted path.
"""
import itertools

import numpy as np

from tests import acc_oracle as ao
from tests import fop_oracle as fo
from tests import put_oracle as po

OP_MAX, OP_MIN, OP_BAND, OP_BOR, OP_BXOR = 4, 5, 6, 7, 8
OPS = {"amax": OP_MAX, "amin": OP_MIN, "bitwise_and": OP_BAND, "bitwise_or": OP_BOR, "bitwise_xor": OP_BXOR}
NAMES = {v: k for k, v in OPS.items()}
INTS = (ao.ACC_I32, ao.ACC_I64)
FLOATS = (ao.ACC_F32, ao.ACC_F64, ao.ACC_F16, ao.ACC_BF16)
SEARCH = 8  # elements with at most this many contributions (not all fetches) are searched over every order


def allowed(op, t):
    """the (op, dtype) pairs the header accepts"""
    return op in (OP_MAX, OP_MIN) or (op in (OP_BAND, OP_BOR, OP_BXOR) and t in INTS)


def order_keys(a, t):
    """int64 keys of storage array `a` that order its values as max / min compare them: signed integers as themselves,
    floats by the total order of their bits (-inf < ... < -0 < +0 < ... < +inf; NaNs are handled apart)"""
    if t in INTS:
        return np.asarray(a, ao.STORAGE[t]).astype(np.int64)
    b = ao.bits(np.asarray(a, ao.STORAGE[t]), t).astype(np.uint64)
    nb = np.dtype(ao.BITS[t]).itemsize * 8
    sign = np.uint64(1) << np.uint64(nb - 1)
    mag = (b & (sign - np.uint64(1))).astype(np.int64)
    return np.where((b & sign) != 0, -1 - mag, mag)


def combine(a, b, t, op):
    """op(a, b) element-wise in type t, bit for bit (a: the elements, b: the operands; storage arrays of one shape)"""
    dt = ao.STORAGE[t]
    a, b = np.asarray(a, dt), np.asarray(b, dt)
    if op in (OP_BAND, OP_BOR, OP_BXOR):
        assert t in INTS, "bitwise ops take the integer types"
        return {OP_BAND: np.bitwise_and, OP_BOR: np.bitwise_or, OP_BXOR: np.bitwise_xor}[op](a, b).astype(dt)
    ka, kb = order_keys(a, t), order_keys(b, t)
    take = kb > ka if op == OP_MAX else kb < ka
    if t in FLOATS:
        na, nb_ = ao.is_nan(a, t), ao.is_nan(b, t)
        take = np.where(nb_, False, np.where(na, True, take))
    return np.where(take, b, a).astype(dt)


def fold(v0, xs, t, op):
    """v0 combined with every operand of xs in order (one element)"""
    cur = np.asarray(v0, ao.STORAGE[t]).reshape(1)
    for x in np.asarray(xs, ao.STORAGE[t]).reshape(-1):
        cur = combine(cur, np.asarray([x], ao.STORAGE[t]), t, op)
    return cur[0]


def reduce(shards, src, t, op, result=None, src_bytes=None, **req):
    """Apply one call (an accumulate when result is None, else a fetch) to `shards` (not modified), request by request.
    src: the packed operands as bytes; result: the caller's result buffer before the call, as bytes. Returns (new
    shards, new result or None, per-request codes, first bad index or -1, layout total)."""
    dt = np.dtype(ao.STORAGE[t])
    disp = shards[0].shape[1] if shards[0].ndim > 1 else 1
    src = np.asarray(src, np.uint8).reshape(-1)
    src_bytes = src.size if src_bytes is None else src_bytes
    codes, pl, bad, total, applied = fo.plan(shards, t, src_bytes, **req)
    new = [s.copy() for s in shards]
    res = None if result is None else np.array(result, np.uint8).reshape(-1)
    if applied:
        for (r, local, count, off, n), code in zip(pl, codes):
            if code == 0 and n > 0:
                rows_r = new[r].reshape(new[r].shape[0], -1)
                x = src[off:off + n].view(dt).reshape(count, disp)
                for i in range(count):  # (row by row: duplicate rows of one request never occur, requests may repeat)
                    old = rows_r[local + i].copy()
                    rows_r[local + i] = combine(old, x[i], t, op)
                    if res is not None:
                        res[off + i * disp * dt.itemsize:off + (i + 1) * disp * dt.itemsize] = old.view(np.uint8)
    return new, res, codes, bad, total


def reduce_many(shards, calls, t, op):
    """Apply `calls` = [(src, src_bytes or None, result or None, request keywords)] in order -> (new shards, [new result
    per call or None], [(status code, bad index, layout total)] as each call reports them)"""
    results, out = [], []
    for src, src_bytes, result, req in calls:
        sb = np.asarray(src).size if src_bytes is None else src_bytes
        shards, res, codes, bad, total = reduce(shards, src, t, op, result, src_bytes=sb, **req)
        results.append(res)
        out.append(po.expected_error(codes, bad, total, sb) + (total,))
    return shards, results, out


def red_path(t, op, dst_phase, src_phase, nbytes, k, fetch=False):
    """the drain path byte k of ONE staged piece takes (acc_oracle.drain_path / fop_oracle.fop_path), with the
    hardware each uses for (op, t): "element" and "vector" pieces of f32 / f64 max / min are compare-and-swap loops, as
    is the whole body when it would be a bulk reduction (there is none); f16 / bf16 head and tail elements are word
    compare-and-swap loops"""
    if fetch:
        path = fo.fop_path(dst_phase, src_phase, nbytes, k)[0]
    else:
        path = ao.drain_path(dst_phase, src_phase, nbytes, k)
        if t in (ao.ACC_F32, ao.ACC_F64) and op in (OP_MAX, OP_MIN):
            path = np.where(path == "bulk", "vector", path)
    path = np.asarray(path).astype(object)
    if op in (OP_MAX, OP_MIN) and t in FLOATS:
        cas = (path == "element") | (t in (ao.ACC_F32, ao.ACC_F64))
        path = np.where(cas, path + " (CAS loop)", path)
    return path


# ------------------------------------------------------------------------------------------------ checking
def _kc(a, t):
    """comparison keys: bits, one class for every NaN"""
    return ao.keys(np.asarray(a, ao.STORAGE[t]), t)


def _euler(v0, final, xs, gs, t, op):
    """None if ONE order of the fetches (operand xs[i], previous value gs[i]) leads from v0 to final, each fetch
    getting the value left by the one before it; else why not. Each fetch is the step gs[i] -> combine(gs[i], xs[i]);
    an order is an Eulerian trail of those steps from v0, ending at final."""
    src_k = _kc(gs, t).tolist()
    dst_k = _kc(combine(gs, xs, t, op), t).tolist()
    a, z = int(_kc(v0, t)[0]), int(_kc(final, t)[0])
    bal = {}
    for s, d in zip(src_k, dst_k):
        bal[s] = bal.get(s, 0) + 1
        bal[d] = bal.get(d, 0) - 1
    want = {a: 1}
    want[z] = want.get(z, 0) - 1
    for v in set(bal) | set(want):
        if bal.get(v, 0) != want.get(v, 0):
            return (f"no order explains the previous values: value key {v:#x} is returned {sum(s == v for s in src_k)} "
                    f"time(s) but reached {sum(d == v for d in dst_k) + (v == a)} time(s)")
    parent = {}

    def find(v):
        parent.setdefault(v, v)
        while parent[v] != v:
            parent[v] = parent[parent[v]]
            v = parent[v]
        return v
    for s, d in zip(src_k, dst_k):
        parent[find(s)] = find(d)
    if any(find(s) != find(a) for s in src_k):
        return "no order explains the previous values: some fetches got values no chain from the start reaches"
    return None


def _search(v0, final, xs, gs, isf, t, op):
    """None if one order of the contributions (fetches: isf) explains every previous value and the final value"""
    n = len(xs)
    kfinal = int(_kc(final, t)[0])
    seen = set()

    def walk(cur, used):
        if used == (1 << n) - 1:
            return int(_kc(cur, t)[0]) == kfinal
        st = (used, int(_kc(cur, t)[0]))
        if st in seen:
            return False
        seen.add(st)
        for i in range(n):
            if used >> i & 1:
                continue
            if isf[i] and int(_kc(gs[i], t)[0]) != st[1]:
                continue
            if walk(combine(np.asarray([cur]), np.asarray([xs[i]]), t, op)[0], used | 1 << i):
                return True
        return False
    return None if walk(np.asarray(v0, ao.STORAGE[t]), 0) else "no order of the contributions explains the previous values"


def _necessary(v0, final, gs, t, op):
    """None if every previous value could be a fold of v0 and some of the contributions (necessary conditions)"""
    if op == OP_BXOR:
        return None
    if op in (OP_MAX, OP_MIN):
        ks, k0, kf = order_keys(gs, t), int(order_keys(np.asarray([v0]), t)[0]), int(order_keys(np.asarray([final]), t)[0])
        nan = ao.is_nan(gs, t)
        v0nan = bool(ao.is_nan(np.asarray([v0]), t)[0])
        lo, hi = (k0, kf) if op == OP_MAX else (kf, k0)
        ok = nan if v0nan else np.zeros(len(gs), bool)
        ok = ok | (~nan & (((ks >= lo) & (ks <= hi)) | v0nan))
        if v0nan:  # a NaN start: results are that NaN until the first operand, then bounded by the final value
            ok = nan | ((ks <= kf) if op == OP_MAX else (ks >= kf))
    else:
        u = ao.BITS[t]
        g = np.asarray(gs, ao.STORAGE[t]).view(u)
        a, z = np.asarray([v0], ao.STORAGE[t]).view(u)[0], np.asarray([final], ao.STORAGE[t]).view(u)[0]
        ok = ((g & ~a) == 0) & ((z & ~g) == 0) if op == OP_BAND else ((a & ~g) == 0) & ((g & ~z) == 0)
    bad = np.flatnonzero(~ok)
    return None if not bad.size else f"previous value {fo.fmt(gs[bad[0]], t)} is no fold of the start and some operands"


def check(shards0, calls, t, op, got_shards, got_results, paths=None):
    """Compare what the device left -- got_shards (one storage array per rank) and got_results (each fetch call's result
    buffer as bytes, None for an accumulate) -- with the calls [(src, src_bytes or None, result before the call or None,
    request keywords)] of one epoch. paths: optional function (call, element index in its src) -> the predicted path,
    added to a report. Returns None or the first inconsistency."""
    dt = np.dtype(ao.STORAGE[t])
    E = dt.itemsize
    lenlist = po.lenlist_of(shards0)
    disp = shards0[0].shape[1] if shards0[0].ndim > 1 else 1
    flat0 = [np.ascontiguousarray(s).reshape(-1) for s in shards0]
    flatg = [np.ascontiguousarray(s).reshape(-1) for s in got_shards]
    srcs = [np.asarray(c[0], np.uint8).reshape(-1) for c in calls]
    for k, (src, src_bytes, result, req) in enumerate(calls):
        if result is None:
            continue
        sb = srcs[k].size if src_bytes is None else src_bytes
        codes, pl, _bad, _total, applied = fo.plan(shards0, t, sb, **req)
        mask = np.zeros(np.asarray(result).size, bool)
        if applied:
            for (_r, _l, _c, off, n), code in zip(pl, codes):
                if code == 0:
                    mask[off:off + n] = True
        g, r0 = np.asarray(got_results[k], np.uint8).reshape(-1), np.asarray(result, np.uint8).reshape(-1)
        d = np.nonzero((g != r0) & ~mask)[0]
        if d.size:
            return f"call {k}: result byte {int(d[0])} written outside the valid requests' rows"
    rk, el, call, si = fo.touches(shards0, calls, t)
    for r in range(len(shards0)):
        keep = np.ones(flat0[r].size, bool)
        keep[el[rk == r]] = False
        d = np.nonzero(keep & (flat0[r].view(ao.BITS[t]) != flatg[r].view(ao.BITS[t])))[0]
        if d.size:
            return fo._elem("an element no request touches changed", r, int(d[0]), disp, lenlist)
    if not rk.size:
        return None
    src_el = [s[:s.size // E * E].view(dt) for s in srcs]
    res_el = [None if g is None else np.asarray(g, np.uint8).reshape(-1) for g in got_results]
    res_el = [None if g is None else g[:g.size // E * E].view(dt) for g in res_el]
    key = rk * (1 << 40) + el
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    ends = np.r_[starts[1:], key.size]
    # final values, all elements at once: the fold of every contribution (order-free), by key
    v0 = np.empty(starts.size, dt)
    fin = np.empty(starts.size, dt)
    for r in range(len(shards0)):
        m = rk[starts] == r
        v0[m], fin[m] = flat0[r][el[starts][m]], flatg[r][el[starts][m]]
    xs = np.empty(key.size, dt)
    for c in np.unique(call).tolist():
        m = call == c
        xs[m] = src_el[c][si[m]]
    cur = v0.copy()
    depth = ends - starts
    for j in range(int(depth.max())):
        live = depth > j
        cur[live] = combine(cur[live], xs[starts[live] + j], t, op)
    bad = np.flatnonzero(_kc(cur, t) != _kc(fin, t))
    if bad.size:
        g = int(bad[0])
        b = starts[g]
        where = f" [{paths(int(call[b]), int(si[b]))}]" if paths else ""
        return (fo._elem("final value", int(rk[b]), int(el[b]), disp, lenlist) +
                f"{where}: got {fo.fmt(fin[g], t)}, expected {fo.fmt(cur[g], t)} (start {fo.fmt(v0[g], t)}, operands "
                f"{', '.join(fo.fmt(x, t) for x in xs[b:ends[g]][:8])}{' ...' if depth[g] > 8 else ''})")
    # previous values of the fetches
    isf = np.array([res_el[c] is not None for c in call.tolist()])
    if not isf.any():
        return None
    gs = np.empty(key.size, dt)
    for c in np.unique(call[isf]).tolist():
        m = call == c
        gs[m] = res_el[c][si[m]]
    once = (depth == 1) & isf[starts]
    ob = starts[once]
    if ob.size:
        bad = np.flatnonzero(ao.bits(gs[ob], t) != ao.bits(v0[once], t))
        if bad.size:
            b = int(ob[bad[0]])
            where = f" [{paths(int(call[b]), int(si[b]))}]" if paths else ""
            return (fo._elem("previous value", int(rk[b]), int(el[b]), disp, lenlist) +
                    f"{where}: got {fo.fmt(gs[b], t)}, the shard held {fo.fmt(v0[once][bad[0]], t)}")
    for g in np.flatnonzero((depth > 1) & np.add.reduceat(isf.astype(np.int64), starts).astype(bool)).tolist():
        b, e = int(starts[g]), int(ends[g])
        f = isf[b:e]
        if f.all():
            why = _euler(v0[g], fin[g], xs[b:e], gs[b:e], t, op)
        elif e - b <= SEARCH:
            why = _search(v0[g], fin[g], xs[b:e], gs[b:e], f, t, op)
        else:
            why = _necessary(v0[g], fin[g], gs[b:e][f], t, op)
        if why:
            where = f" [{paths(int(call[b]), int(si[b]))}]" if paths else ""
            return (fo._elem("fetch chain", int(rk[b]), int(el[b]), disp, lenlist) +
                    f"{where}: {why} (start {fo.fmt(v0[g], t)}, {e - b} contributions, final {fo.fmt(fin[g], t)})")
    return None


# ------------------------------------------------------------------------------------------------ test data
def families(rng, t, n):
    """n storage elements of type t drawn from the value families that separate the ops' rules: for floats +-0, quiet
    and signalling NaNs with payloads (both signs), +-inf, subnormals of both signs, the largest finite values, small
    integers; for integers INT_MIN, INT_MAX, -1, 0, 1, all-ones patterns and random bits"""
    if t in INTS:
        info = np.iinfo(ao.STORAGE[t])
        special = np.array([info.min, info.max, -1, 0, 1, -2, 2, info.min + 1, info.max - 1], ao.STORAGE[t])
        rnd = rng.integers(info.min, info.max, size=n, dtype=ao.STORAGE[t], endpoint=True)
        small = rng.integers(-4, 5, size=n).astype(ao.STORAGE[t])
        pick = rng.integers(0, 3, size=n)
        return np.where(pick == 0, special[rng.integers(0, special.size, size=n)], np.where(pick == 1, small, rnd))
    u = ao.BITS[t]
    nb = np.dtype(u).itemsize * 8
    sign = 1 << (nb - 1)
    special = [0, sign, ao._max_bits(t), sign | ao._max_bits(t), 1, sign | 1, 2, sign | 3]
    special += [ao._nan_bits(t, q) for q in range(4)] + [sign | ao._nan_bits(t, 1)]
    inf = {ao.ACC_F32: 0x7F800000, ao.ACC_F64: 0x7FF0000000000000, ao.ACC_F16: 0x7C00, ao.ACC_BF16: 0x7F80}[t]
    special += [inf, sign | inf]
    special = np.array(special, np.uint64).astype(u)
    small = ao.encode(rng.integers(-4, 5, size=n), t).view(u)
    rnd = rng.integers(0, 1 << min(nb, 63), size=n, dtype=np.uint64).astype(u)
    if nb == 64:
        rnd |= (rng.integers(0, 2, size=n).astype(np.uint64) << np.uint64(63)).astype(u)
    pick = rng.integers(0, 3, size=n)
    out = np.where(pick == 0, special[rng.integers(0, special.size, size=n)], np.where(pick == 1, small, rnd))
    return np.ascontiguousarray(out.astype(u)).view(ao.STORAGE[t])


def distinct(rng, t, n):
    """n pairwise distinct non-NaN storage elements (their keys differ), for hot elements whose fetch results must
    be told apart"""
    out = families(rng, t, 4 * n + 64)
    k = _kc(out, t)
    _, first = np.unique(k, return_index=True)
    keep = np.sort(first[~ao.is_nan(out[first], t)])
    rng.shuffle(keep)
    assert keep.size >= n, "not enough distinct values"
    return out[keep[:n]]


def permutations_ok(v0, xs, t, op):
    """every order's (previous values, final) of contributions xs on start v0 (for the CPU tests of the checker)"""
    for p in itertools.permutations(range(len(xs))):
        cur, prev = np.asarray([v0], ao.STORAGE[t]), np.empty(len(xs), ao.STORAGE[t])
        for i in p:
            prev[i] = cur[0]
            cur = combine(cur, np.asarray([xs[i]], ao.STORAGE[t]), t, op)
        yield prev, cur[0]
