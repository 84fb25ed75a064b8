"""The batched fetch-ops' arithmetic and returned values on the GPU against the correctly rounded oracle of
tests/fop_oracle.py (built on tests/acc_oracle.py): inexact floats, subnormals, the min-normal boundary, overflow,
signed zeros, inf and NaN payloads and integer wraparound, through each atomic of the fetch drain -- the element
atomics of the head and tail (fetch1: returning atom.add / exch, the 2-byte swap's CAS loop, the f16 / bf16 element adds
ptxas makes CAS loops) and the eight re-phased vector forms of the body (write_loop<kActFetch, WS, BYTES>, fetch16) -- and both writes of
the previous values to the result (one bulk store, or drain_chunk).

  (a) one fetch-op per element, every path: previous values bit for bit, new values by one rounded addition (f32 IEEE
      or flushed) or the operand's bits, every (type, op, path, value family) cell covered, then read back;
  (b) two or three fetch-adds per element (duplicates in one batch, queued batches, thread-ranks, one fetch-add beside
      one accumulate): the whole tuple of previous values and final value against `admissible_fetch`;
  (c) hot elements: thousands of fetch-adds that all raise the running sum, each step one rounded addition, and swap
      chains of distinct bit patterns;
  (d) 65543-element rows cut at chunk boundaries;
  (e) with -s, a per-(type, path) table of what f32 did with subnormals and whether previous values came back whole.

Which atomic an element takes depends only on where its shard bytes and its staged operand sit relative to 16-byte
boundaries. A one-request call of at most 2048 bytes (the smallest chunk any fetch geometry stages) is one staged
piece, so there `fop_oracle.fop_path` names the path of every element.
"""
import ctypes as C

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import fop_oracle as fo
from tests.gpu_helpers import run_world
from tests.test_gpu_acc_numerics import DISP, ENTRIES, chunk_bytes, read_shard
from tests.test_gpu_accumulate import add_var, raw_acc
from tests.test_gpu_get_accumulate import raw_fop

pytestmark = pytest.mark.gpu
ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)
OPS = (fo.OP_SUM, fo.OP_REPLACE)
OPN = {fo.OP_SUM: "sum", fo.OP_REPLACE: "replace"}
E = {t: np.dtype(ao.STORAGE[t]).itemsize for t in ALL}
PIECE = 2048  # the smallest chunk a fetch geometry stages: a one-request call up to this size is one piece
NCALLS = 300
MIN_CELL = 4  # the fewest elements of one value family a (type, op, path) cell may hold
NO_SYNC = 4


@pytest.fixture(scope="module")
def torch():
    import torch as t
    if not t.cuda.is_available():
        pytest.skip("no GPU")
    return t


@pytest.fixture()
def store(torch):
    from ddstore_b200 import PyDDStore
    s = PyDDStore(device=0)
    yield s
    s.free()
    s.close()


class Call:
    """one fetch-op call: operands (storage array) on the device src_off bytes past a 16-byte boundary, the result
    res_off bytes past one (or the operands' own bytes: in_place)"""

    def __init__(self, torch, store, name, t, op, src, src_off, entry="counts", dev=False, start=0, count=1, sample=None,
                 res_off=0, in_place=False, flags=0, stream=None, device="cuda:0", keep=None):
        data = np.ascontiguousarray(src).view(np.uint8).reshape(-1)
        src_off, res_off = int(src_off), int(res_off)
        self.n, self.t, self.device = data.size, t, device
        self.src = torch.empty(src_off + data.size + 16, dtype=torch.uint8, device=device)
        self.src[src_off:src_off + data.size].copy_(torch.from_numpy(data))
        sp = self.src.data_ptr() + src_off
        if in_place:
            self.res, self.lo, rp = self.src, src_off, sp
        else:
            self.res = torch.full((res_off + data.size + 16,), 0xA5, dtype=torch.uint8, device=device)
            self.lo, rp = res_off, self.res.data_ptr() + res_off
        torch.cuda.synchronize(device)
        if entry == "counts":
            req = dict(starts=np.atleast_1d(start), counts=np.atleast_1d(count))
        elif entry == "fixed":
            req = dict(starts=np.atleast_1d(start), fixed=int(np.atleast_1d(count)[0]))
        else:
            req = dict(ids=np.atleast_1d(sample))
        rc, total, bad = raw_fop(torch, store, name, op, t, sp, rp, data.size, dev=dev, flags=flags, stream=stream,
                                 device=device, keep=keep, **req)
        if flags & NO_SYNC:  # (queued: the outcome comes with the wait)
            assert rc == 0, (name, entry, rc, store._L.dds_last_error())
        else:
            assert (rc, total, bad) == (0, data.size, -1), (name, entry, rc, total, bad, store._L.dds_last_error())

    def result(self, torch):
        """the previous values (storage array)"""
        torch.cuda.synchronize(self.device)
        return self.res[self.lo:self.lo + self.n].cpu().numpy().view(ao.STORAGE[self.t])


def family_data(rng, t, op, n):
    """per element: a value family's name, the shard's value and the operand (storage arrays). Swaps also take
    'patterns': both from the whole range of bit patterns (signalling NaNs, negative NaNs, +-0, subnormals, inf, max)"""
    fam_pairs = ao.families(rng, t, n)
    if op == fo.OP_REPLACE:
        fam_pairs["patterns"] = (fo.swap_patterns(rng, t, n), fo.swap_patterns(rng, t, n))
    names = np.array(list(fam_pairs))
    fam = names[rng.integers(0, len(names), size=n)]
    a, b = np.empty(n, ao.STORAGE[t]), np.empty(n, ao.STORAGE[t])
    for nm in names:
        m = fam == nm
        a[m], b[m] = fam_pairs[nm][0][m], fam_pairs[nm][1][m]
    return names, fam, a, b


def outcome_table(t, op, start, x, got_prev, got_new, fam, paths):
    """per path: whether previous values that are subnormals came back whole, and (sums) what the elements whose IEEE
    and flushed results differ got -- 'kept' (IEEE), 'flushed' or a mix -- among the subnormal families and at the
    min-normal boundary"""
    rows = []
    sub = ao.is_nan(start, t) == 0
    v = np.abs(ao.values(start, t))
    sub &= (v > 0) & (v < ao.min_normal(t))
    if op == fo.OP_SUM:
        ieee = ao.keys(ao.add(start, x, t), t)
        if t == ao.ACC_F32:
            fl = ao.keys(ao.add_flushed(start, x), t)
        else:  # (what flushing the result would give: these types must keep it)
            s = ao.values(ao.add(start, x, t), t)
            fl = ao.keys(ao.encode(np.where(np.abs(s) < ao.min_normal(t), np.copysign(0.0, s), s), t), t)
        g = ao.keys(got_new, t)
    for p in ["element"] + fo.vector_paths(t):
        m = (paths == p) & sub
        whole = int((fo.bits64(got_prev[m], t) == fo.bits64(start[m], t)).sum())
        cells = [f"previous subnormals: {'-' if not m.any() else f'whole ({whole})' if whole == m.sum() else f'{whole} of {int(m.sum())} whole'}"]
        if op == fo.OP_SUM:
            for what, fams in (("subnormals", ("subnormal", "cancel")), ("min normal", ("min normal",))):
                m = (paths == p) & np.isin(fam, fams) & (ieee != fl)
                k, f = int((g[m] == ieee[m]).sum()), int((g[m] == fl[m]).sum())
                cells.append(f"{what}: " + ("-" if not m.any() else f"kept ({k})" if k == m.sum() else
                                            f"flushed ({f})" if f == m.sum() else
                                            f"mixed: {k} kept, {f} flushed of {int(m.sum())}"))
        rows.append(f"  {ao.NAMES[t]:9s} {OPN[op]:7s} {p:11s} " + "   ".join(f"{c:30s}" for c in cells))
    return rows


# ------------------------------------------------------------------------------------------------ (a), (e)
@pytest.mark.parametrize("op", OPS, ids=lambda o: OPN[o])
@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_one_fetch_op_every_path(torch, store, t, op):
    """every value family through the element atomics and every re-phased vector form: NCALLS one-request calls of at
    most 2048 bytes (the six entry forms in turn) at every start-row phase, each staged phase chosen so that the
    re-phase variants take turns, results written by one bulk store (result, size and staged bytes 16-byte aligned) or
    by drain_chunk, some in place; every previous value bit for bit, every new value by `once_verdict`, every (path,
    family) cell covered; then get_batch and get() read the same bits back"""
    rng = np.random.default_rng([7000 + t, op])
    D = DISP[E[t]]
    R = D * E[t]
    assert 13 * R <= PIECE <= chunk_bytes(store)
    vpaths = fo.vector_paths(t)
    shs = list(range(0, 16, E[t]))
    bulk_rows = 16 // np.gcd(R, 16)  # rows whose bytes are a multiple of 16
    plan, r = [], 0
    for k in range(NCALLS):
        r += int(rng.integers(0, 3))
        c = bulk_rows if k % 5 == 0 else int(rng.integers(1, 5))
        plan.append((r, c))
        r += c
    nrows = r + 1
    names, fam, a, b = family_data(rng, t, op, nrows * D)
    fam, a, b = fam.reshape(nrows, D), a.reshape(nrows, D), b.reshape(nrows, D)
    add_var(torch, store, "n", a.view(np.uint8).reshape(-1), nrows, D, E[t])
    store.set_sample_index("n", np.array([p[0] for p in plan], np.int64), np.array([p[1] for p in plan], np.int64))
    base = store.query("n")["local_base"]
    paths = np.full((nrows, D), "", dtype=object)
    prev = np.zeros((nrows, D), ao.STORAGE[t])
    result_paths, in_place = {"bulk": 0, "drain_chunk": 0}, 0
    for k, (r, c) in enumerate(plan):
        dp = (base + r * R) % 16
        head = (16 - dp) % 16
        if k % 5 == 0:  # result, size and staged bytes aligned: the bulk result write
            off, ro = 0, 0
        else:
            off = (shs[k % len(shs)] - head) % 16  # the staged body's phase: each re-phase variant in turn
            ro = int(rng.choice(range(0, 16, E[t])))
        ip = k % 7 == 3
        entry, dev = ENTRIES[k % len(ENTRIES)]
        cl = Call(torch, store, "n", t, op, b[r:r + c], off, entry, dev, r, c, sample=k, res_off=ro, in_place=ip)
        prev[r:r + c] = cl.result(torch).reshape(c, D)
        p, rp = fo.fop_path(dp, off, c * R, np.arange(c * D) * E[t], res_phase=off if ip else ro)
        paths[r:r + c] = p.reshape(c, D)
        result_paths[rp] += 1
        in_place += ip
    got = read_shard(torch, store, "n", t, nrows, D)
    cov = (paths != "").reshape(-1)
    assert ao.bits(got, t).reshape(-1)[~cov].tolist() == ao.bits(a, t).reshape(-1)[~cov].tolist(), \
        "an untouched row changed"
    idx = np.nonzero(cov)[0]
    flat = lambda x: x.reshape(-1)[idx]  # noqa: E731
    gp, gn, af, bf, pf, ff = flat(prev), flat(got), flat(a), flat(b), flat(paths), flat(fam)
    msg = fo.once_verdict(gp, gn, af, bf, t, op, where=lambda i: (0, int(idx[i]) // D, int(idx[i]) % D), paths=pf,
                          what=f"{ao.NAMES[t]} {OPN[op]}, one fetch-op per element")
    assert msg is None, msg
    for p in ["element"] + vpaths:
        for nm in names:
            n = int(((pf == p) & (ff == nm)).sum())
            assert n >= MIN_CELL, f"{ao.NAMES[t]} {OPN[op]}: only {n} elements of family {nm!r} took the {p} path"
    assert min(result_paths.values()) >= 20 and in_place >= 20, (result_paths, in_place)
    print(f"\n{ao.NAMES[t]} {OPN[op]}: one fetch-op per element, {idx.size} elements over {NCALLS} calls "
          f"(results: {result_paths['bulk']} bulk, {result_paths['drain_chunk']} drain_chunk, {in_place} in place)")
    if t in ao.FLOATS:
        print("\n".join(outcome_table(t, op, af, bf, gp, gn, ff, pf)))
    # read-back: get_batch and get() return the shard's bits
    out = torch.zeros(nrows * D * E[t], dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    store.get_batch("n", [0], [nrows], out=out)
    assert out.cpu().numpy().tobytes() == got.tobytes(), "get_batch differs from the shard"
    host = np.zeros((nrows, D), ao.STORAGE[t])
    assert store._L.dds_get(store._h, b"n", 0, nrows, E[t], host.ctypes.data, 0) == 0
    assert host.tobytes() == got.tobytes(), "get() differs from the shard"


# ------------------------------------------------------------------------------------------------ (b)
def _start_and(rng, t, shape, which):
    if t in ao.FLOATS:
        return ao.inexact(rng, shape, t)
    return ao.families(rng, t, int(np.prod(shape)))["random"][which].reshape(shape)


def _check_tuples(t, start, xs, gots, final, ncon, what, acc=None, where_rank=0):
    """every element with k = ncon fetch-adds (xs / gots: [3, ...] operands and previous values) against
    admissible_fetch; -> the fraction of elements with more than one admissible tuple"""
    D = start.shape[-1]
    differ, total = 0.0, 0
    for k in (1, 2, 3):
        m = ncon.reshape(-1) == k
        if not m.any():
            continue
        idx = np.nonzero(m)[0]
        s = start.reshape(-1)[m]
        cs = [xs[j].reshape(-1)[m] for j in range(k)]
        gp = np.stack([gots[j].reshape(-1)[m] for j in range(k)])
        ac = None if acc is None else acc.reshape(-1)[m]
        opts = fo.admissible_fetch(s, cs, t, ac)
        msg = fo.fetch_verdict(gp, final.reshape(-1)[m], s, cs, t, acc=ac, opts=opts,
                               where=lambda i: (where_rank, int(idx[i]) // D, int(idx[i]) % D),
                               what=f"{what}, {k} fetch-adds")
        assert msg is None, msg
        if k + (acc is not None) >= 2:
            differ += fo.discrimination(opts) * idx.size
            total += idx.size
    frac = differ / max(total, 1)
    print(f"\n{what}: {frac:.3f} of the elements have more than one admissible tuple (threshold {ao.DISCRIMINATION})")
    if t in ao.FLOATS:
        assert frac > ao.DISCRIMINATION, (what, frac)
    return frac


@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_duplicates_in_one_batch(torch, store, t):
    """two or three requests of one batch fetch-add into each element, at different staged phases and from different
    start rows: copies of one element meet as a head or tail (element atomics) and in a body (vector atomics)"""
    rng = np.random.default_rng(8000 + t)
    D = DISP[E[t]]
    G = 300
    nrows = 2 * G
    start = _start_and(rng, t, (nrows, D), 0)
    add_var(torch, store, "d", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    reqs = []
    for g in range(G):
        r = 2 * g
        reqs += [(r, 2), (r + 1, 1), (r, 1)] + ([(r, 2)] if rng.random() < 0.5 else [])
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    xs, gots = np.zeros((2, 3, nrows, D), ao.STORAGE[t])
    ncon = np.zeros((nrows, D), np.int64)
    src = [_start_and(rng, t, (c, D), 1) for _, c in reqs]
    off = int(rng.choice(range(0, 16, E[t])))
    cl = Call(torch, store, "d", t, fo.OP_SUM, np.concatenate(src), off, "counts", True,
              [r for r, _ in reqs], [c for _, c in reqs], res_off=(off + E[t]) % 16)
    res, pos = cl.result(torch).reshape(-1, D), 0
    for (r, c), v in zip(reqs, src):
        for j in range(c):
            xs[ncon[r + j, 0], r + j], gots[ncon[r + j, 0], r + j] = v[j], res[pos + j]
        ncon[r:r + c] += 1
        pos += c
    got = read_shard(torch, store, "d", t, nrows, D)
    _check_tuples(t, start, xs, gots, got, ncon, f"{ao.NAMES[t]} duplicates in one batch")


@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_queued_batches(torch, store, t):
    """two or three batches queued on one stream (device indices, no synchronisation between them), each fetch-adding
    once into every element from its own staged phase, result phase and entry"""
    rng = np.random.default_rng(9000 + t)
    D = DISP[E[t]]
    nrows = 500
    start = _start_and(rng, t, (nrows, D), 0)
    add_var(torch, store, "q", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    xs, gots = np.zeros((2, 3, nrows, D), ao.STORAGE[t])
    ncon = np.zeros((nrows, D), np.int64)
    h = torch.cuda.Stream().cuda_stream
    keep, calls = [], []
    k_of = rng.integers(2, 4, size=nrows)
    store.epoch_begin()
    for j in range(3):
        rows = rng.permutation(np.nonzero(k_of > j)[0])
        v = _start_and(rng, t, (rows.size, D), 1)
        xs[j, rows] = v
        ncon[rows] += 1
        calls.append((rows, Call(torch, store, "q", t, fo.OP_SUM, v, (j * 6) % 16 // E[t] * E[t],
                                 "fixed" if j != 1 else "counts", True, rows, np.ones(rows.size, np.int64),
                                 res_off=(j * 2 * E[t]) % 16, flags=NO_SYNC, stream=h, keep=keep)))
    store.epoch_end()
    total, bad = C.c_int64(0), C.c_int64(-1)
    assert store._L.dds_batch_wait(store._h, C.byref(total), C.byref(bad)) == 0
    for j, (rows, cl) in enumerate(calls):
        gots[j, rows] = cl.result(torch).reshape(-1, D)
    got = read_shard(torch, store, "q", t, nrows, D)
    _check_tuples(t, start, xs, gots, got, ncon, f"{ao.NAMES[t]} queued batches")


@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_ranks_in_one_epoch(torch, t):
    """three thread-ranks fetch-add into rank 1's rows in one epoch, one fetch-add each per element (rank 0 from a
    re-phased source, rank 1 aligned, rank 2 by sample id), each rank's results at its own phase"""
    rng = np.random.default_rng(10000 + t)
    P, D = 3, DISP[E[t]]
    nrows = [5, 400, 0]
    first = nrows[0]
    start = _start_and(rng, t, (nrows[1], D), 0)
    contribs = [_start_and(rng, t, (nrows[1], D), 1) for _ in range(P)]
    perms = [rng.permutation(nrows[1]) for _ in range(P)]

    def body(st, r):
        import torch as tt
        dev = f"cuda:{tt.cuda.current_device()}"
        mine = start if r == 1 else np.zeros((nrows[r], D), ao.STORAGE[t])
        data = np.ascontiguousarray(mine).view(np.uint8).reshape(-1)
        assert st._L.dds_add(st._h, b"w", data.ctypes.data if data.size else None, nrows[r], D, E[t], 0) == 0
        st.set_sample_index("w", np.arange(first, first + nrows[1], dtype=np.int64), np.ones(nrows[1], np.int64))
        st.epoch_begin()
        p = perms[r]
        v = contribs[r][p]
        if r == 2:
            cl = Call(tt, st, "w", t, fo.OP_SUM, v, 0, "samples", True, sample=p, res_off=E[t], device=dev)
        else:
            cl = Call(tt, st, "w", t, fo.OP_SUM, v, E[t] if r == 0 else 0, "counts", r == 0, first + p,
                      np.ones(p.size, np.int64), res_off=16 - E[t] if r == 0 else 0, device=dev)
        st.epoch_end()
        res = np.empty_like(v)
        res[...] = cl.result(tt).reshape(-1, D)
        back = np.empty_like(res)
        back[p] = res
        return back, (read_shard(tt, st, "w", t, nrows[r], D, dev) if r == 1 else None)
    out = run_world(P, body)
    gots = np.stack([o[0] for o in out])
    _check_tuples(t, start, np.stack(contribs), gots, out[1][1], np.full((nrows[1], D), P),
                  f"{ao.NAMES[t]} {P} ranks", where_rank=1)


@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_fetch_add_beside_an_accumulate(torch, store, t):
    """one fetch-add and one accumulate_batch into every element, queued in one epoch in either order on two rows
    halves: the accumulate of whole aligned rows takes the bulk reduction (which keeps f32 subnormals), the fetch-add
    vector and element atomics; the fetch-add's previous value and the final value against admissible_fetch with the
    accumulate as its one plain contribution"""
    rng = np.random.default_rng(11000 + t)
    D = DISP[E[t]]
    nrows = 400
    start = _start_and(rng, t, (nrows, D), 0)
    add_var(torch, store, "m", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    base = store.query("m")["local_base"]
    x, y = _start_and(rng, t, (nrows, D), 1), _start_and(rng, t, (nrows, D), 1)
    h = torch.cuda.Stream().cuda_stream
    keep = []
    ybuf = torch.empty(16 + y.nbytes, dtype=torch.uint8, device="cuda:0")
    ybuf[base % 16:base % 16 + y.nbytes].copy_(torch.from_numpy(y.view(np.uint8).reshape(-1)))
    torch.cuda.synchronize()
    store.epoch_begin()
    half = nrows // 2
    rows = rng.permutation(nrows)
    acc = lambda: raw_acc(torch, store, "m", t, ybuf.data_ptr() + base % 16, y.nbytes, starts=[0],  # noqa: E731
                          counts=[nrows], dev=True, flags=NO_SYNC, stream=h, keep=keep)
    c1 = Call(torch, store, "m", t, fo.OP_SUM, x[rows[:half]], E[t], "fixed", True, rows[:half], [1], res_off=0,
              flags=NO_SYNC, stream=h, keep=keep)
    assert acc()[0] == 0
    c2 = Call(torch, store, "m", t, fo.OP_SUM, x[rows[half:]], 0, "counts", True, rows[half:],
              np.ones(nrows - half, np.int64), res_off=E[t], flags=NO_SYNC, stream=h, keep=keep)
    store.epoch_end()
    total, bad = C.c_int64(0), C.c_int64(-1)
    assert store._L.dds_batch_wait(store._h, C.byref(total), C.byref(bad)) == 0
    gots = np.zeros((1, nrows, D), ao.STORAGE[t])
    gots[0, rows[:half]] = c1.result(torch).reshape(-1, D)
    gots[0, rows[half:]] = c2.result(torch).reshape(-1, D)
    got = read_shard(torch, store, "m", t, nrows, D)
    _check_tuples(t, start, x[None], gots, got, np.ones((nrows, D), np.int64),
                  f"{ao.NAMES[t]} a fetch-add beside an accumulate", acc=y)


# ------------------------------------------------------------------------------------------------ (c)
@pytest.mark.parametrize("path", ["vector", "element"])
@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_hot_fetch_adds(torch, store, t, path):
    """HOT_FETCH[t] fetch-adds (4096 f32 and integers, 65536 f64, 512 f16, 128 bf16) of operands in (1, 2) into every
    element of a few hot rows, in one batch: 64-byte rows at 16-byte aligned shard addresses (a vector atomic per 16
    bytes, the staged operands re-phased by the source's phase) or one-element rows (element atomics). Every addition
    raises the running sum, so sorting an element's previous values gives the only order: each step one correctly
    rounded addition, bit for bit, and the final value the last; every other row unchanged"""
    rng = np.random.default_rng([12000 + t, path == "vector"])
    D = 64 // E[t] if path == "vector" else 1
    R = D * E[t]
    nrows, hot = 16, np.array([3, 8, 13])
    n = fo.HOT_FETCH[t]
    start = fo.hot_values(rng, t, (nrows, D))
    add_var(torch, store, "h", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    base = store.query("h")["local_base"]
    if path == "vector":
        assert base % 16 == 0 and R % 16 == 0
    rows = rng.permutation(np.repeat(hot, n))
    x = fo.hot_values(rng, t, (rows.size, D))
    off = int(rng.choice(range(E[t], 16, E[t]))) if path == "vector" else 0
    cl = Call(torch, store, "h", t, fo.OP_SUM, x, off, "fixed", True, rows, [1], res_off=(16 - off) % 16)
    res = cl.result(torch).reshape(-1, D)
    got = read_shard(torch, store, "h", t, nrows, D)
    cold = ~np.isin(np.arange(nrows), hot)
    assert got[cold].tobytes() == start[cold].tobytes(), "a row without fetch-adds changed"
    for h in hot:
        m = rows == h
        if t in ao.FLOATS:
            v = np.sort(ao.values(res[m], t), axis=0)
            assert (v[1:] > v[:-1]).all(), f"{ao.NAMES[t]} {path}: row {h}: two fetch-ops got the same value"
        bad = fo.increasing_chain(start[h], x[m], res[m], got[h], t)
        assert bad is None, (f"{ao.NAMES[t]} {path} ({m.sum()} fetch-adds per element): rank 0, global row {h}, column "
                             f"{bad[0]}: {bad[1]}")
    print(f"\n{ao.NAMES[t]} {path}: {n} fetch-adds per element of {hot.size} hot rows, each step one rounded addition")


@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_swap_chains(torch, store, t):
    """256 swaps per element of a few hot rows, operands distinct bit patterns (every NaN kind, +-0, subnormals, inf
    and max among them), by element atomics (the 2-byte swap's CAS loop) and re-phased vector exchanges: one chain
    v0 -> s_a -> ... -> final per element, bit for bit"""
    rng = np.random.default_rng(13000 + t)
    D = DISP[E[t]]
    nrows, hot, n = 12, np.array([2, 5, 9]), 256
    start = fo.swap_patterns(rng, t, nrows * D).reshape(nrows, D)
    add_var(torch, store, "s", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    rows = rng.permutation(np.repeat(hot, n))
    x = np.empty((rows.size, D), ao.STORAGE[t])
    for h in hot:
        for c in range(D):
            x[rows == h, c] = fo.distinct_patterns(rng, t, n, avoid=ao.bits(start[h, c:c + 1], t))
    off = int(rng.choice(range(0, 16, E[t])))
    res0 = np.full(x.nbytes, 0xA5, np.uint8)
    cl = Call(torch, store, "s", t, fo.OP_REPLACE, x, off, "counts", True, rows, np.ones(rows.size, np.int64),
              res_off=E[t])
    res = cl.result(torch)
    got = read_shard(torch, store, "s", t, nrows, D)
    call = (x.view(np.uint8).reshape(-1), None, res0, {"starts": rows, "counts": np.ones(rows.size, np.int64)})
    msg = fo.check([start], [call], t, fo.OP_REPLACE, [got], [res.view(np.uint8)])
    assert msg is None, f"{ao.NAMES[t]} swap chains: {msg}"


# ------------------------------------------------------------------------------------------------ (d)
@pytest.mark.parametrize("op", OPS, ids=lambda o: OPN[o])
@pytest.mark.parametrize("t", ALL, ids=lambda t: ao.NAMES[t])
def test_long_rows(torch, store, t, op):
    """65543-element rows, which the walk cuts at chunk boundaries: every value family, each staged phase and result
    phase 0, one element and 16 bytes less one element, by every entry; every element once, previous and new value"""
    rng = np.random.default_rng([14000 + t, op])
    D, nrows = 65543, 7
    _, _, a, b = family_data(rng, t, op, nrows * D)
    a, b = a.reshape(nrows, D), b.reshape(nrows, D)
    add_var(torch, store, "l", a.view(np.uint8).reshape(-1), nrows, D, E[t])
    store.set_sample_index("l", np.array([5, 6], np.int64), np.array([1, 1], np.int64))
    prev = np.empty_like(a)
    for rws, off, ro, entry, dev, kw in (([0, 2, 3], 0, E[t], "counts", False, dict(start=[0, 2], count=[1, 2])),
                                         ([1, 4], E[t], 0, "fixed", True, dict(start=[1, 4], count=[1, 1])),
                                         ([5], 16 - E[t], 16 - E[t], "samples", False, dict(sample=0)),
                                         ([6], 8 % 16, 0, "samples", True, dict(sample=1))):
        cl = Call(torch, store, "l", t, op, b[rws], off, entry, dev, res_off=ro, in_place=rws == [6], **kw)
        prev[rws] = cl.result(torch).reshape(-1, D)
    got = read_shard(torch, store, "l", t, nrows, D)
    msg = fo.once_verdict(prev.reshape(-1), got.reshape(-1), a.reshape(-1), b.reshape(-1), t, op,
                          where=lambda i: (0, i // D, i % D), what=f"{ao.NAMES[t]} {OPN[op]} 65543-element rows")
    assert msg is None, msg
