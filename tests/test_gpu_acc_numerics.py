"""The batched accumulate's arithmetic on the GPU against the correctly rounded oracle of tests/acc_oracle.py: inexact
floats, subnormals, the min-normal boundary, overflow, signed zeros, inf / NaN and integer wraparound, through each of
the drain's three reductions (bulk, re-phased vector, element), with one contribution per element (compared bit for
bit: `admissible`), two or three (every order admitted, nothing else) and many (`sum_bound`), then read back.

Which reduction an element takes depends only on where its destination and its staged source bytes sit relative to
16-byte boundaries (write_chunk<kActReduce>). A one-request call whose rows fit in one chunk is one staged piece, so there
`acc_oracle.drain_path` names the path of every element; the coverage of every (type, path, value family) cell is
asserted. The verdict on an element does not depend on its path, except that f32 may flush subnormals.
"""
import ctypes as C

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests.gpu_helpers import run_world
from tests.test_gpu_accumulate import add_var, raw_acc
from tests.test_gpu_put import shard_state, to_device

pytestmark = pytest.mark.gpu
ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)
FLOATS = (ao.ACC_F32, ao.ACC_F64, ao.ACC_F16, ao.ACC_BF16)
E = {t: np.dtype(ao.STORAGE[t]).itemsize for t in ALL}
DISP = {2: 75, 4: 37, 8: 19}  # odd elements per row, rows of 150, 148 and 152 bytes: every destination phase occurs
PATHS = ("bulk", "vector", "element")
ENTRIES = [(e, dev) for e in ("counts", "fixed", "samples") for dev in (False, True)]
NCALLS = 240
MIN_CELL = 4  # the fewest elements of one value family a (type, path) cell may hold
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


def chunk_bytes(store):
    vals = [C.c_int(0) for _ in range(5)]
    store._L.dds_gather_geometry(*[C.byref(v) for v in vals])
    return vals[3].value


def read_shard(torch, store, name, t, nrows, disp, device="cuda:0"):
    got, slack = shard_state(torch, store, name, nrows * disp * E[t], device)
    assert not got[nrows * disp * E[t]:].any(), f"{name}: the shard's slack was written"
    return got[:nrows * disp * E[t]].view(ao.STORAGE[t]).reshape(nrows, disp)


def call(torch, store, name, t, src, off, entry, dev, start, count, sample=None, **kw):
    """one accumulate of `src` (storage array) from `off` bytes past a 16-byte boundary, by `entry`; -> its bytes"""
    data = np.ascontiguousarray(src).view(np.uint8).reshape(-1)
    buf, ptr = to_device(torch, data, off)
    if entry == "counts":
        req = dict(starts=np.atleast_1d(start), counts=np.atleast_1d(count))
    elif entry == "fixed":
        req = dict(starts=np.atleast_1d(start), fixed=int(np.atleast_1d(count)[0]))
    else:
        req = dict(ids=np.atleast_1d(sample))
    rc, total, bad = raw_acc(torch, store, name, t, ptr, data.size, dev=dev, **req, **kw)
    if kw.get("flags", 0) & NO_SYNC:  # (queued: the outcome comes with the wait)
        assert rc == 0, (name, entry, rc, store._L.dds_last_error())
    else:
        assert (rc, total, bad) == (0, data.size, -1), (name, entry, rc, total, bad, store._L.dds_last_error())
    return buf


def outcome_table(t, got, a, b, fam, paths):
    """per path: what the elements whose IEEE and flushed results differ got -- 'kept' (IEEE), 'flushed' or a mix --
    among the subnormal families and at the min-normal boundary"""
    ieee = ao.keys(ao.add(a, b, t), t)
    if t == ao.ACC_F32:
        fl = ao.keys(ao.add_flushed(a, b), t)
    else:  # (what flushing the result would give: these types must keep it)
        v = ao.values(ao.add(a, b, t), t)
        fl = ao.keys(ao.encode(np.where(np.abs(v) < ao.min_normal(t), np.copysign(0.0, v), v), t), t)
    g = ao.keys(got, t)
    rows = []
    for p in PATHS:
        cells = []
        for what, fams in (("subnormals", ("subnormal", "cancel")), ("min normal", ("min normal",))):
            m = (paths == p) & np.isin(fam, fams) & (ieee != fl)
            k, f = int((g[m] == ieee[m]).sum()), int((g[m] == fl[m]).sum())
            cells.append("-" if not m.any() else f"kept ({k})" if k == m.sum() else f"flushed ({f})" if f == m.sum()
                         else f"mixed: {k} kept, {f} flushed of {int(m.sum())}")
        rows.append(f"  {ao.NAMES[t]:9s} {p:8s} subnormals: {cells[0]:28s} min-normal boundary: {cells[1]}")
    return rows


# ------------------------------------------------------------------------------------------------ (a), (b), (e)
@pytest.mark.parametrize("t", ALL)
def test_one_contribution_every_path(torch, store, t):
    """every value family through the bulk, vector and element reductions: NCALLS one-request calls (the six entry
    forms in turn) at every start-row phase, each source at the destination's phase (bulk body) or another one
    (re-phased body), with heads and tails; every element bit for bit against `admissible` (f32: IEEE or flushed), every
    (path, family) cell covered; then get_batch and get() read the same bits back (-0, subnormals, NaN payloads)"""
    rng = np.random.default_rng(1000 + t)
    D = DISP[E[t]]
    R = D * E[t]
    assert 3 * R <= chunk_bytes(store)
    plan, r = [], 0
    for k in range(NCALLS):
        r += int(rng.integers(0, 3))
        c = int(rng.integers(1, 4))
        plan.append((r, c))
        r += c
    nrows = r + 1
    fam_pairs = ao.families(rng, t, nrows * D)
    names = np.array(list(fam_pairs))
    fam = names[rng.integers(0, len(names), size=nrows * D)]
    a = np.empty(nrows * D, ao.STORAGE[t])
    b = np.empty(nrows * D, ao.STORAGE[t])
    for nm in names:
        m = fam == nm
        a[m], b[m] = fam_pairs[nm][0][m], fam_pairs[nm][1][m]
    a, b = a.reshape(nrows, D), b.reshape(nrows, D)
    add_var(torch, store, "n", a.view(np.uint8).reshape(-1), nrows, D, E[t])
    store.set_sample_index("n", np.array([p[0] for p in plan], np.int64), np.array([p[1] for p in plan], np.int64))
    base = store.query("n")["local_base"]
    paths = np.full((nrows, D), "", dtype=object)
    for k, (r, c) in enumerate(plan):
        dp = (base + r * R) % 16
        off = dp if k % 3 == 0 else int(rng.choice([o for o in range(0, 16, E[t]) if o != dp]))
        entry, dev = ENTRIES[k % len(ENTRIES)]
        call(torch, store, "n", t, b[r:r + c], off, entry, dev, r, c, sample=k)
        paths[r:r + c] = ao.drain_path(dp, off, c * R, np.arange(c * D) * E[t]).reshape(c, D)
    got = read_shard(torch, store, "n", t, nrows, D)
    cov = (paths != "").reshape(-1)
    assert ao.keys(got, t).reshape(-1)[~cov].tolist() == ao.keys(a, t).reshape(-1)[~cov].tolist(), "an untouched row changed"
    idx = np.nonzero(cov)[0]
    gf, af, bf, pf, ff = got.reshape(-1)[idx], a.reshape(-1)[idx], b.reshape(-1)[idx], paths.reshape(-1)[idx], fam[idx]
    opts = ao.admissible_all(af, [bf], t)
    first = int(np.argmin((opts == ao.keys(gf, t)[None]).any(0)))
    msg = ao.verdict(gf, af, [bf], t, opts=opts, where=lambda i: (0, int(idx[i]) // D, int(idx[i]) % D), paths=pf,
                     what=f"{ao.NAMES[t]} one contribution (first bad: family {ff[first]!r})")
    assert msg is None, msg
    for p in PATHS:
        for nm in names:
            n = int(((pf == p) & (ff == nm)).sum())
            assert n >= MIN_CELL, f"{ao.NAMES[t]}: only {n} elements of family {nm!r} took the {p} path"
    if t in FLOATS:
        print(f"\n{ao.NAMES[t]}: one contribution, {idx.size} elements over {NCALLS} calls; per path:")
        print("\n".join(outcome_table(t, gf, af, bf, ff, pf)))
    # (e) read-back: get_batch and get() return the shard's bits
    out = torch.zeros(nrows * D * E[t], dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    store.get_batch("n", [0], [nrows], out=out)  # (the element size is the variable's; out holds its bytes)
    assert out.cpu().numpy().tobytes() == got.tobytes(), "get_batch differs from the shard"
    host = np.zeros((nrows, D), ao.STORAGE[t])
    assert store._L.dds_get(store._h, b"n", 0, nrows, E[t], host.ctypes.data, 0) == 0
    assert host.tobytes() == got.tobytes(), "get() differs from the shard"
    one = np.zeros((1, D), ao.STORAGE[t])
    for g in (plan[0][0], plan[-1][0], plan[NCALLS // 2][0]):
        assert store._L.dds_get(store._h, b"n", g, 1, E[t], one.ctypes.data, 0) == 0
        assert one.tobytes() == got[g:g + 1].tobytes(), f"get() of row {g}"


@pytest.mark.parametrize("t", ALL)
def test_one_contribution_long_rows(torch, store, t):
    """65543-element rows, which the walk cuts at chunk boundaries: every value family, each source offset 0, one
    element and 16 bytes less one element, by every entry"""
    rng = np.random.default_rng(2000 + t)
    D, nrows = 65543, 7
    fam_pairs = ao.families(rng, t, nrows * D)
    names = list(fam_pairs)
    pick = rng.integers(0, len(names), size=nrows * D)
    a = np.choose(pick, [fam_pairs[n][0] for n in names]).astype(ao.STORAGE[t]).reshape(nrows, D)
    b = np.choose(pick, [fam_pairs[n][1] for n in names]).astype(ao.STORAGE[t]).reshape(nrows, D)
    add_var(torch, store, "l", a.view(np.uint8).reshape(-1), nrows, D, E[t])
    store.set_sample_index("l", np.array([5, 6], np.int64), np.array([1, 1], np.int64))
    call(torch, store, "l", t, b[[0, 2, 3]], 0, "counts", False, [0, 2], [1, 2])
    call(torch, store, "l", t, b[[1, 4]], E[t], "fixed", True, [1, 4], [1, 1])
    call(torch, store, "l", t, b[5], 16 - E[t], "samples", False, 0, 0, sample=0)
    call(torch, store, "l", t, b[6], 8 % 16, "samples", True, 0, 0, sample=1)
    got = read_shard(torch, store, "l", t, nrows, D)
    msg = ao.verdict(got.reshape(-1), a.reshape(-1), [b.reshape(-1)], t, where=lambda i: (0, i // D, i % D),
                     what=f"{ao.NAMES[t]} 65543-element rows")
    assert msg is None, msg


# ------------------------------------------------------------------------------------------------ (c)
def _track(nrows, D, t):
    return np.zeros((3, nrows, D), ao.STORAGE[t]), np.zeros((nrows, D), np.int64)


def _check_multi(t, got, start, contribs, ncon, what, where_rank=0):
    """every element against admissible_all over its own contributions; -> the fraction of elements with two or
    more contributions whose admissible set has more than one member"""
    many, multi = 0, 0
    for k in range(4):
        m = ncon.reshape(-1) == k
        if not m.any():
            continue
        s = start.reshape(-1)[m]
        cs = [contribs[j].reshape(-1)[m] for j in range(k)]
        opts = ao.admissible_all(s, cs, t)
        idx = np.nonzero(m)[0]
        D = start.shape[1]
        msg = ao.verdict(got.reshape(-1)[m], s, cs, t, opts=opts,
                         where=lambda i: (where_rank, int(idx[i]) // D, int(idx[i]) % D), what=f"{what}, {k} contributions")
        assert msg is None, msg
        if k >= 2:
            many += int(m.sum())
            multi += int((opts != opts[0]).any(0).sum())
    return multi / max(many, 1)


def _report(t, what, frac):
    print(f"\n{ao.NAMES[t]} {what}: {frac:.3f} of the elements with 2-3 contributions have more than one admissible "
          f"result (threshold {ao.DISCRIMINATION})")
    if t in FLOATS:
        assert frac > ao.DISCRIMINATION, (what, frac)


@pytest.mark.parametrize("t", ALL)
def test_duplicates_in_one_batch(torch, store, t):
    """two or three requests of one batch add into each element, at different source phases and from different start
    rows: copies of one element meet as a head (element reduction; the f16 / bf16 CAS) and as a body (bulk or
    vector) of another request"""
    rng = np.random.default_rng(3000 + t)
    D = DISP[E[t]]
    R = D * E[t]
    G = 400
    nrows = 2 * G
    start = ao.inexact(rng, (nrows, D), t) if t in FLOATS else ao.families(rng, t, nrows * D)["random"][0].reshape(nrows, D)
    add_var(torch, store, "d", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    base = store.query("d")["local_base"]
    reqs = []
    for g in range(G):
        r = 2 * g
        reqs += [(r, 2), (r + 1, 1), (r, 1)] + ([(r, 2)] if rng.random() < 0.5 else [])
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    contribs, ncon = _track(nrows, D, t)
    head_meets_body = np.zeros((nrows, D), np.int64)  # bit 0: an element reduction, bit 1: a bulk or vector one
    off = int(rng.choice(range(0, 16, E[t])))
    ch = chunk_bytes(store)
    src, pos = [], off
    for r, c in reqs:
        v = ao.inexact(rng, (c, D), t) if t in FLOATS else ao.families(rng, t, c * D)["random"][1].reshape(c, D)
        src.append(v)
        for j in range(c):
            contribs[ncon[r + j, 0], r + j] = v[j]
        ncon[r:r + c] += 1
        if (pos - off) // ch == (pos - off + c * R - 1) // ch:  # (one piece unless a chunk boundary of the layout cuts it)
            p = ao.drain_path((base + r * R) % 16, pos % 16, c * R, np.arange(c * D) * E[t]).reshape(c, D)
            head_meets_body[r:r + c] |= np.where(p == "element", 1, 2)
        pos += c * R
    call(torch, store, "d", t, np.concatenate(src), off, "counts", True, [r for r, _ in reqs], [c for _, c in reqs])
    got = read_shard(torch, store, "d", t, nrows, D)
    frac = _check_multi(t, got, start, contribs, ncon, f"{ao.NAMES[t]} duplicates in one batch")
    meets = int((head_meets_body == 3).sum())
    print(f"\n{ao.NAMES[t]}: {meets} elements took an element reduction and a bulk or vector one")
    assert meets >= 200, meets
    _report(t, "duplicates in one batch", frac)


@pytest.mark.parametrize("t", ALL)
def test_queued_batches(torch, store, t):
    """two or three batches queued on one stream (device indices, no synchronisation between them), each adding
    once into every element from its own source phase and entry"""
    rng = np.random.default_rng(4000 + t)
    D = DISP[E[t]]
    nrows = 600
    start = ao.inexact(rng, (nrows, D), t) if t in FLOATS else ao.families(rng, t, nrows * D)["random"][0].reshape(nrows, D)
    add_var(torch, store, "q", start.view(np.uint8).reshape(-1), nrows, D, E[t])
    contribs, ncon = _track(nrows, D, t)
    h = torch.cuda.Stream().cuda_stream
    keep = []
    k_of = rng.integers(2, 4, size=nrows)  # 2 or 3 contributions per row
    for j in range(3):
        rows = rng.permutation(np.nonzero(k_of > j)[0])
        v = ao.inexact(rng, (rows.size, D), t) if t in FLOATS else ao.families(rng, t, rows.size * D)["random"][1].reshape(-1, D)
        contribs[j, rows] = v
        ncon[rows] += 1
        keep.append(call(torch, store, "q", t, v, (j * 6) % 16 // E[t] * E[t], "fixed" if j != 1 else "counts", True,
                         rows, np.ones(rows.size, np.int64), flags=NO_SYNC, stream=h, keep=keep))
    total, bad = C.c_int64(0), C.c_int64(-1)
    assert store._L.dds_batch_wait(store._h, C.byref(total), C.byref(bad)) == 0
    got = read_shard(torch, store, "q", t, nrows, D)
    _report(t, "queued batches", _check_multi(t, got, start, contribs, ncon, f"{ao.NAMES[t]} queued batches"))


@pytest.mark.parametrize("t", ALL)
def test_ranks_in_one_epoch(torch, t):
    """three thread-ranks add into rank 1's rows in one epoch, one contribution each per element (rank 0 from a
    re-phased source, rank 1 aligned, rank 2 by sample id)"""
    rng = np.random.default_rng(5000 + t)
    P, D = 3, DISP[E[t]]
    nrows = [5, 500, 0]
    first = nrows[0]
    start = ao.inexact(rng, (nrows[1], D), t) if t in FLOATS else ao.families(rng, t, nrows[1] * D)["random"][0].reshape(-1, D)
    contribs = [ao.inexact(rng, (nrows[1], D), t) if t in FLOATS else
                ao.families(rng, t, nrows[1] * D)["random"][1].reshape(-1, D) for _ in range(P)]
    perms = [rng.permutation(nrows[1]) for _ in range(P)]

    def body(st, r):
        import torch as tt
        mine = start if r == 1 else np.zeros((nrows[r], D), ao.STORAGE[t])
        data = np.ascontiguousarray(mine).view(np.uint8).reshape(-1)
        assert st._L.dds_add(st._h, b"w", data.ctypes.data if data.size else None, nrows[r], D, E[t], 0) == 0
        st.set_sample_index("w", np.arange(first, first + nrows[1], dtype=np.int64), np.ones(nrows[1], np.int64))
        st.epoch_begin()
        p = perms[r]
        v = contribs[r][p]
        if r == 2:
            call(tt, st, "w", t, v, 0, "samples", True, None, None, sample=p, device=f"cuda:{tt.cuda.current_device()}")
        else:
            call(tt, st, "w", t, v, E[t] if r == 0 else 0, "counts", r == 0, first + p, np.ones(p.size, np.int64),
                 device=f"cuda:{tt.cuda.current_device()}")
        st.epoch_end()
        return read_shard(tt, st, "w", t, nrows[r], D, f"cuda:{tt.cuda.current_device()}") if r == 1 else None
    got = run_world(P, body)[1]
    frac = _check_multi(t, got, start, np.stack(contribs), np.full((nrows[1], D), P), f"{ao.NAMES[t]} {P} ranks",
                        where_rank=1)
    _report(t, f"{P} ranks in one epoch", frac)


# ------------------------------------------------------------------------------------------------ (d)
@pytest.mark.parametrize("how", ["one batch", "four ranks"])
@pytest.mark.parametrize("t", ALL)
def test_hot_elements(torch, t, how):
    """HOT[t] contributions into every element of one row (1024 f32, 65536 f64, 16 f16, 6 bf16, 4096 integers) from
    one batch or from four thread-ranks in one epoch: floats within sum_bound of the exact sum (the bound is below
    one contribution), integers the exact wrapped sum; every other row unchanged"""
    rng = np.random.default_rng([6000 + t, how == "one batch"])
    D, per, hot = 67, 6, 3
    P = 1 if how == "one batch" else 4
    n = ao.HOT[t]
    total_rows = per * P
    hot_g = per * (P - 1) + hot  # on the last rank
    if t in FLOATS:
        start = ao.inexact(rng, (total_rows, D), t, 0, 1)
        cs = ao.inexact(rng, (n, D), t, 0, 1)
    else:
        start = ao.families(rng, t, total_rows * D)["random"][0].reshape(total_rows, D)
        cs = ao.families(rng, t, n * D)["random"][1].reshape(n, D)
    share = np.array_split(np.arange(n), P)

    def body(st, r):
        import torch as tt
        dev = f"cuda:{tt.cuda.current_device()}"
        mine = np.ascontiguousarray(start[r * per:(r + 1) * per]).view(np.uint8).reshape(-1)
        assert st._L.dds_add(st._h, b"h", mine.ctypes.data, per, D, E[t], 0) == 0
        st.epoch_begin()
        k = share[r]
        call(tt, st, "h", t, cs[k], (E[t] * (r + 1)) % 16, "fixed", True, np.full(k.size, hot_g), [1], device=dev)
        st.epoch_end()
        return read_shard(tt, st, "h", t, per, D, dev)
    got = np.concatenate(run_world(P, body))
    others = np.arange(total_rows) != hot_g
    assert got[others].tobytes() == start[others].tobytes(), "a row without contributions changed"
    g = got[hot_g]
    if t in FLOATS:
        s, bound = ao.sum_bound(start[hot_g], cs, t)
        assert (bound < np.abs(ao.values(cs, t)).min(0)).all()
        err = np.abs(ao.values(g, t) - s)
        bad = np.nonzero(~(err <= bound))[0]
        assert not bad.size, (f"{ao.NAMES[t]} {how}: rank {P - 1}, global row {hot_g}, column {bad[0]}: got "
                              f"{ao.values(g, t)[bad[0]]!r}, exact sum {s[bad[0]]!r}, |error| {err[bad[0]]:.3g} > "
                              f"bound {bound[bad[0]]:.3g} ({n} contributions)")
        print(f"\n{ao.NAMES[t]} {how}: {n} contributions per element, max |error| / bound = {(err / bound).max():.3f}")
    else:
        u = np.uint64 if t == ao.ACC_I64 else np.uint32
        exp = (start[hot_g].view(u).astype(np.uint64) + cs.view(u).astype(np.uint64).sum(0, dtype=np.uint64)).astype(u)
        assert g.view(u).tolist() == exp.tolist(), f"{ao.NAMES[t]} {how}: the wrapped sum differs"
