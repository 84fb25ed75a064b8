"""Batched reductions beside the sum -- accumulate_batch / accumulate_samples with op="amax", "amin", "bitwise_and",
"bitwise_or" or "bitwise_xor", and get_accumulate_batch / _samples with the same ops -- on the GPU against the NumPy
oracle of tests/red_oracle.py.

Every check compares the whole local shard (rows and zero slack) and every result buffer with the oracle: final values
by bits (a NaN by class), fetch results by one order of the contributions that explains them all. Data are drawn from
the value families that separate the rules (+-0, quiet and signalling NaNs with payloads on both sides, +-inf,
subnormals, INT_MIN / INT_MAX, -1 against 1, all-ones). The requests are single rows whose shard and operand phases
vary, so each (op, dtype) cell goes through the bulk, re-phased vector and element drains, and the module asserts that
it did. With -s, test_semantics_table prints what each path gave on the float edge pairs.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import red_oracle as ro
from tests.gpu_helpers import run_world
from tests.test_gpu_accumulate import add_var
from tests.test_gpu_put import dev_bytes, shard_state

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CELLS = [(op, t) for op in ro.OPS.values() for t in ao.STORAGE if ro.allowed(op, t)]
E = {t: np.dtype(ao.STORAGE[t]).itemsize for t in ao.STORAGE}
TORCH = {ao.ACC_F32: "float32", ao.ACC_F64: "float64", ao.ACC_I32: "int32", ao.ACC_I64: "int64",
         ao.ACC_F16: "float16", ao.ACC_BF16: "bfloat16"}


def _ids(c):
    return f"{ro.NAMES[c[0]]}-{ao.NAMES[c[1]]}"


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


# ------------------------------------------------------------------------------------------------ helpers
def to_dev(torch, a, t, off=0, device="cuda:0"):
    """a CUDA tensor of type t holding storage array `a` (flat), starting `off` elements past a 16-byte boundary"""
    a = np.ascontiguousarray(a, ao.STORAGE[t]).reshape(-1)
    buf = torch.zeros(a.size + off + 16, dtype=getattr(torch, TORCH[t]), device=device)
    v = buf[off:off + a.size]
    if a.size:
        raw = torch.from_numpy(a.view(np.uint8).copy()).to(device)
        v.view(torch.uint8).copy_(raw)
    torch.cuda.synchronize(device)
    return v


def host(x, t):
    """a CUDA tensor's elements as a storage array of type t"""
    import torch
    return x.contiguous().view(-1).view(torch.uint8).cpu().numpy().view(ao.STORAGE[t])


def add_world(store, name, shard):
    """the variable `name` with this rank's rows `shard` (any element type: added by its bytes and itemsize)"""
    import torch
    a = np.ascontiguousarray(shard)
    add_var(torch, store, name, a.reshape(-1).view(np.uint8), a.shape[0], a.shape[1], a.dtype.itemsize)


def read_shard(torch, store, name, shard0):
    """(rows as a storage array of shard0's shape, slack bytes all zero)"""
    payload = shard0.nbytes
    raw, slack = shard_state(torch, store, name, payload)
    return raw[:payload].view(shard0.dtype).reshape(shard0.shape), not raw[payload:].any()


def run_call(torch, store, name, t, op, fetch, src, out, starts=None, ids=None, stream=None, wait=True):
    opn = ro.NAMES[op]
    if ids is not None:
        if fetch:
            return store.get_accumulate_samples(name, ids, src, out, op=opn, stream=stream, wait=wait)
        return store.accumulate_samples(name, ids, src, stream=stream, wait=wait, op=opn)
    if fetch:
        return store.get_accumulate_batch(name, starts, src=src, out=out, op=opn, count=1, stream=stream, wait=wait)
    return store.accumulate_batch(name, starts, src=src, count=1, stream=stream, wait=wait, op=opn)


def single_rows(torch, store, op, t, fetch, dev, seed, disp=37, nrows=600, by_id=False, dups=True):
    """one call of single-row requests (every row; with dups, some twice or more) with operands a random number of
    elements past a 16-byte boundary; returns the oracle's verdict and the paths the elements took"""
    rng = np.random.default_rng([seed, op, t, fetch, dev, by_id])
    shard0 = ro.families(rng, t, nrows * disp).reshape(nrows, disp)
    add_world(store, "c", shard0)
    rows = np.concatenate([rng.permutation(nrows)] + ([rng.integers(0, nrows, size=nrows // 4),
                                                      np.repeat(rng.integers(0, nrows, size=8), 2)] if dups else []))
    rows = rows.astype(np.int64)
    rng.shuffle(rows)
    x = ro.families(rng, t, rows.size * disp)
    off = int(rng.integers(0, 16 // E[t]))
    src = to_dev(torch, x, t, off)
    out = to_dev(torch, np.zeros(x.size, ao.STORAGE[t]), t, int(rng.integers(0, 16 // E[t]))) if fetch else None
    res0 = host(out, t).view(np.uint8).copy() if fetch else None
    if by_id:
        perm = rng.permutation(nrows).astype(np.int64)
        store.set_sample_index("c", perm, np.ones(nrows, np.int64))
        inv = np.argsort(perm)
        ids = inv[rows]
        idx = torch.from_numpy(ids).cuda() if dev else ids
        req = {"sample_ids": ids, "table": (perm, np.ones(nrows, np.int64))}
        total = run_call(torch, store, "c", t, op, fetch, src, out, ids=idx)
    else:
        idx = torch.from_numpy(rows).cuda() if dev else rows
        req = {"starts": rows, "fixed_count": 1}
        total = run_call(torch, store, "c", t, op, fetch, src, out, starts=idx)
    assert total == x.nbytes
    got, slack_ok = read_shard(torch, store, "c", shard0)
    assert slack_ok, "the shard's slack changed"
    res = host(out, t).view(np.uint8) if fetch else None
    R = disp * E[t]
    base = store.query("c")["local_base"]
    sp = src.data_ptr()

    def path(call, k):
        i = k // disp
        return ro.red_path(t, op, (base + int(rows[i]) * R) % 16, (sp + i * R) % 16, R, (k % disp) * E[t], fetch)
    why = ro.check([shard0], [(x.view(np.uint8), None, res0, req)], t, op, [got], [res], paths=path)
    paths = set()
    for i in range(rows.size):
        paths |= set(ro.red_path(t, op, (base + int(rows[i]) * R) % 16, (sp + i * R) % 16, R,
                                 np.arange(disp) * E[t], fetch).tolist())
    store.free()
    return why, paths


@pytest.mark.parametrize("dev", [False, True], ids=["host-idx", "dev-idx"])
@pytest.mark.parametrize("fetch", [False, True], ids=["acc", "fetch"])
@pytest.mark.parametrize("cell", CELLS, ids=_ids)
def test_cells(torch, store, cell, fetch, dev):
    """every (op, dtype) cell, both entry families, host and device indices: whole shard and results against the
    oracle, and the cell went through every drain path it has"""
    op, t = cell
    why, paths = single_rows(torch, store, op, t, fetch, dev, seed=1)
    assert why is None, why
    kinds = {p.split(" ")[0] for p in paths}
    assert {"element", "vector"} <= kinds, paths
    if not fetch and ro.red_path(t, op, 0, 0, 32, 0) == "bulk":
        assert "bulk" in kinds, paths
    if fetch:  # every re-phased vector variant the element size allows
        from tests import fop_oracle as fo
        assert set(fo.vector_paths(t)) <= {p.replace(" (CAS loop)", "") for p in paths}, paths


@pytest.mark.parametrize("fetch", [False, True], ids=["acc", "fetch"])
@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_MIN, ao.ACC_BF16), (ro.OP_BXOR, ao.ACC_I64),
                                  (ro.OP_BAND, ao.ACC_I32)], ids=_ids)
def test_by_sample_id(torch, store, cell, fetch):
    op, t = cell
    why, _ = single_rows(torch, store, op, t, fetch, True, seed=2, by_id=True)
    assert why is None, why


@pytest.mark.parametrize("fetch", [False, True], ids=["acc", "fetch"])
@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_MIN, ao.ACC_F16), (ro.OP_BOR, ao.ACC_I64),
                                  (ro.OP_MAX, ao.ACC_F64)], ids=_ids)
def test_65543_element_rows(torch, store, cell, fetch):
    """rows of 65543 elements: pieces cut at every chunk, each with head, body and tail"""
    op, t = cell
    why, _ = single_rows(torch, store, op, t, fetch, True, seed=3, disp=65543, nrows=6, dups=False)
    assert why is None, why


PAIRS = ["NaN,1", "1,NaN", "NaNa,NaNb", "-0,+0", "+0,-0", "sub,-sub", "sNaN,1", "-inf,NaN"]


def _pairs(t):
    nb = np.dtype(ao.BITS[t]).itemsize * 8
    s = 1 << (nb - 1)
    one = int(ao.bits(ao.encode([1.0], t), t)[0])
    q, sn, qa, qb = ao._nan_bits(t, 0), ao._nan_bits(t, 1), ao._nan_bits(t, 3), ao._nan_bits(t, 2)
    inf = int(ao.bits(ao.encode([np.inf], t), t)[0])
    v = [(q, one), (one, q), (qa, qb), (s, 0), (0, s), (1, s | 1), (sn, one), (s | inf, q)]
    u = ao.BITS[t]
    return (np.array([a for a, _ in v], np.uint64).astype(u).view(ao.STORAGE[t]),
            np.array([b for _, b in v], np.uint64).astype(u).view(ao.STORAGE[t]))


def test_semantics_table(torch, store, capsys):
    """the float edge pairs through each path of each entry family: bulk (same phase), vector (re-phased) and element
    (sub-16-byte requests). Every result meets the header's maximumNumber / minimumNumber rule; with -s the table of
    what each path returned is printed."""
    lines = []
    for t in ro.FLOATS:
        a, b = _pairs(t)
        per = 32 // E[t]
        n = -(-a.size // per) * per
        shard_w = np.zeros(n, ao.STORAGE[t])
        shard_w[:a.size] = a
        xs = np.zeros(n, ao.STORAGE[t])
        xs[:b.size] = b
        for op in (ro.OP_MAX, ro.OP_MIN):
            for fetch in (False, True):
                for pathname in ("bulk/vector0", "vector", "element"):
                    if pathname == "element":
                        shard0 = shard_w.reshape(-1, 1)
                        add_world(store, "s", shard0)
                        starts = np.arange(n, dtype=np.int64)
                        src = to_dev(torch, xs, t, 0)
                    else:
                        shard0 = shard_w.reshape(-1, per)
                        add_world(store, "s", shard0)
                        starts = np.zeros(1, np.int64)
                        src = to_dev(torch, xs, t, 0 if pathname != "vector" else 1)
                    out = to_dev(torch, np.zeros(n, ao.STORAGE[t]), t) if fetch else None
                    opn = ro.NAMES[op]
                    cnt = 1 if pathname == "element" else shard0.shape[0]
                    if fetch:
                        store.get_accumulate_batch("s", starts, src=src, out=out, op=opn, count=cnt)
                    else:
                        store.accumulate_batch("s", starts, src=src, count=cnt, op=opn)
                    got, _ = read_shard(torch, store, "s", shard0)
                    got = got.reshape(-1)
                    exp = ro.combine(a, b, t, op)
                    gk, ek = ro._kc(got[:a.size], t), ro._kc(exp, t)
                    assert (gk == ek).all(), (ao.NAMES[t], opn, fetch, pathname, got[:a.size], exp)
                    if fetch:
                        assert (ao.bits(host(out, t)[:a.size], t) == ao.bits(a, t)).all()
                    store.free()
                    w = 2 * E[t]
                    kind = ("fetch " if fetch else "acc ") + pathname
                    lines.append(f"{ao.NAMES[t]:9s} {opn:5s} {kind:20s} " + " ".join(
                        f"[{p}]={int(g):0{w}x}" for p, g in zip(PAIRS, ao.bits(got[:a.size], t).tolist())))
    with capsys.disabled():
        print("\nper-path semantics (shard, operand) -> result bits:\n" + "\n".join(lines))


# ------------------------------------------------------------------------------------------------ contention
HOT = [(ro.OP_MAX, ao.ACC_I32), (ro.OP_MIN, ao.ACC_F32), (ro.OP_BXOR, ao.ACC_I64), (ro.OP_BOR, ao.ACC_I32),
       (ro.OP_MAX, ao.ACC_F16), (ro.OP_MAX, ao.ACC_F64), (ro.OP_MIN, ao.ACC_BF16), (ro.OP_BAND, ao.ACC_I64)]


@pytest.mark.parametrize("cell", HOT, ids=_ids)
def test_65536_fetches_on_one_element(torch, store, cell):
    """65536 fetches of one element in one batch: the final value is the fold of them all, and one order of the
    65536 explains every returned previous value (an Eulerian trail through the fetches' steps)"""
    op, t = cell
    rng = np.random.default_rng([5, op, t])
    n = 65536
    shard0 = ro.families(rng, t, 64).reshape(64, 1)
    if op == ro.OP_BOR:
        x = (np.int64(1) << rng.integers(0, 31, size=n)).astype(ao.STORAGE[t])
    elif op == ro.OP_BAND:
        x = ~(np.int64(1) << rng.integers(0, 63, size=n)).astype(ao.STORAGE[t])
        shard0[:] = -1
    else:
        x = ro.families(rng, t, n)
    add_world(store, "h", shard0)
    starts = np.full(n, 5, np.int64)
    src = to_dev(torch, x, t)
    out = to_dev(torch, np.zeros(n, ao.STORAGE[t]), t)
    res0 = host(out, t).view(np.uint8).copy()
    store.get_accumulate_batch("h", torch.from_numpy(starts).cuda(), src=src, out=out, op=ro.NAMES[op], count=1)
    got, _ = read_shard(torch, store, "h", shard0)
    why = ro.check([shard0], [(x.view(np.uint8), None, res0, {"starts": starts, "fixed_count": 1})], t, op, [got],
                   [host(out, t).view(np.uint8)])
    assert why is None, why


@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_BXOR, ao.ACC_I32), (ro.OP_MIN, ao.ACC_F16)],
                         ids=_ids)
def test_fetch_beside_accumulate_and_queued_batches(torch, store, cell):
    """queued batches on two streams in one epoch -- accumulates and fetches of one op, with duplicate rows -- on a
    small hot set of 4 KiB rows: final values fold every contribution, fetch results obey the necessary conditions"""
    op, t = cell
    rng = np.random.default_rng([6, op, t])
    disp = 4096 // E[t]
    nrows = 16
    shard0 = ro.families(rng, t, nrows * disp).reshape(nrows, disp)
    add_world(store, "q", shard0)
    streams = [torch.cuda.Stream().cuda_stream for _ in range(2)]
    calls, outs, keep = [], [], []
    for k in range(6):
        rows = rng.integers(0, nrows, size=48).astype(np.int64)
        x = ro.families(rng, t, rows.size * disp)
        src = to_dev(torch, x, t, int(rng.integers(0, 16 // E[t])))
        fetch = k % 2 == 1
        out = to_dev(torch, np.zeros(x.size, ao.STORAGE[t]), t) if fetch else None
        res0 = host(out, t).view(np.uint8).copy() if fetch else None
        ix = torch.from_numpy(rows).cuda()
        torch.cuda.synchronize()
        run_call(torch, store, "q", t, op, fetch, src, out, starts=ix, stream=streams[k % 2], wait=False)
        keep.append((src, ix))
        calls.append((x.view(np.uint8), None, res0, {"starts": rows, "fixed_count": 1}))
        outs.append(out)
    assert store.wait() == 48 * 4096
    got, _ = read_shard(torch, store, "q", shard0)
    res = [None if o is None else host(o, t).view(np.uint8) for o in outs]
    why = ro.check([shard0], calls, t, op, [got], res)
    assert why is None, why


# ------------------------------------------------------------------------------------------------ ranks
def reduce_world(P, op, t, seed, disp=5):
    """P thread-ranks, each with its own shard; every rank queues an accumulate and a fetch of one op into rows of the
    whole world (duplicates included) in one epoch; after the closing fence the world and every result are checked"""
    rng = np.random.default_rng([seed, P, op, t])
    nrows = [int(n) for n in rng.integers(1, 30, size=P)]
    shards0 = [ro.families(rng, t, n * disp).reshape(n, disp) for n in nrows]
    total = sum(nrows)
    plans = []
    for r in range(P):
        mine = []
        for k in range(2):
            rows = rng.integers(0, total, size=40).astype(np.int64)
            mine.append((rows, ro.families(rng, t, rows.size * disp), k == 1))
        plans.append(mine)

    def body(store, r):
        import torch as tt
        add_world(store, "w", shards0[r])
        store.epoch_begin()
        st = tt.cuda.Stream().cuda_stream
        outs, keep = [], []
        for rows, x, fetch in plans[r]:
            src = to_dev(tt, x, t)
            out = to_dev(tt, np.zeros(x.size, ao.STORAGE[t]), t) if fetch else None
            ix = tt.from_numpy(rows).cuda()
            tt.cuda.synchronize()
            run_call(tt, store, "w", t, op, fetch, src, out, starts=ix, stream=st, wait=False)
            outs.append(out)
            keep.append((src, ix))
        store.wait()
        store.epoch_end()
        got = dev_bytes(tt, store.query("w")["local_base"], shards0[r].nbytes).view(ao.STORAGE[t])
        return got.reshape(shards0[r].shape), [None if o is None else host(o, t).view(np.uint8) for o in outs]
    res = run_world(P, body)
    calls, results = [], []
    for r in range(P):
        for (rows, x, fetch), got in zip(plans[r], res[r][1]):
            calls.append((x.view(np.uint8), None, np.zeros(x.nbytes, np.uint8) if fetch else None,
                          {"starts": rows, "fixed_count": 1}))
            results.append(got)
    return ro.check(shards0, calls, t, op, [res[r][0] for r in range(P)], results)


@pytest.mark.parametrize("P", [2, 3, 4])
@pytest.mark.parametrize("cell", [(ro.OP_MAX, ao.ACC_F32), (ro.OP_BOR, ao.ACC_I64), (ro.OP_MIN, ao.ACC_BF16)],
                         ids=_ids)
def test_rank_worlds(torch, P, cell):
    why = reduce_world(P, *cell, seed=7)
    assert why is None, why


def test_sixty_four_ranks(torch):
    why = reduce_world(64, ro.OP_MAX, ao.ACC_I32, seed=8, disp=2)
    assert why is None, why


# ------------------------------------------------------------------------------------------------ errors, queues
def test_errors(torch, store):
    from ddstore_b200 import _capi
    store.add("e", np.zeros((10, 4), np.float32))
    store.add("i", np.zeros((10, 4), np.int32))
    src = torch.ones(2, 4, device="cuda:0")
    isrc = torch.ones(2, 4, dtype=torch.int32, device="cuda:0")
    out = torch.zeros(2, 4, device="cuda:0")
    for bad in ("max", "replace", "prod"):
        with pytest.raises(ValueError, match="is not one of"):
            store.accumulate_batch("e", [0, 1], src=src, op=bad)
    with pytest.raises(ValueError, match="is not one of"):
        store.get_accumulate_batch("e", [0, 1], src=src, out=out, op="max")
    with pytest.raises(ValueError, match="bitwise"):
        store.accumulate_batch("e", [0, 1], src=src, op="bitwise_or")
    with pytest.raises(ValueError, match="bitwise"):
        store.get_accumulate_batch("e", [0, 1], src=src, out=out, op="bitwise_xor")
    with pytest.raises(ValueError, match="Invalid data type"):
        store.accumulate_batch("e", [0, 1], src=src.double(), op="amax")
    with pytest.raises(ValueError, match="no sample index"):
        store.accumulate_samples("e", [0], src, op="amin")
    total, bad = C.c_int64(0), C.c_int64(0)
    sa = np.zeros(1, np.int64)

    def call(name, op, dtype, ptr, flags=_capi.SRC_ON_DEVICE):
        return store._L.dds_accumulate_op_batch(store._h, name, sa.ctypes.data, None, 1, 1, op, dtype, ptr, 16, flags,
                                                None, C.byref(total), C.byref(bad))
    p, ip = src.data_ptr(), isrc.data_ptr()
    for op in (0, 2, 3, 9, -1):
        assert call(b"e", op, _capi.ACC_F32, p) == _capi.ERR_ARG, op
    for op in (6, 7, 8):
        assert call(b"e", op, _capi.ACC_F32, p) == _capi.ERR_ARG and "bitwise" in _capi.last_error()
    assert call(b"e", 99, 99, p) == _capi.ERR_ARG and "dtype" in _capi.last_error()  # dtype before op
    assert call(b"e", 4, _capi.ACC_F64, p) == _capi.ERR_DTYPE                          # itemsize before op
    assert call(b"e", 4, _capi.ACC_F32, p + 2) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(b"e", 4, _capi.ACC_F32, p, flags=0) == _capi.ERR_ARG
    assert call(b"nope", 4, _capi.ACC_F32, p) == _capi.ERR_UNKNOWN_VAR
    res = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    assert store._L.dds_get_accumulate_batch(store._h, b"i", sa.ctypes.data, None, 1, 1, 3, _capi.ACC_I32, ip,
                                             res.data_ptr(), 16, _capi.SRC_ON_DEVICE, None, C.byref(total),
                                             C.byref(bad)) == _capi.ERR_ARG  # (3 stays unassigned)
    sh = dev_bytes(torch, store.query("e")["local_base"], 160)
    assert not sh.any(), "a refused call changed the shard"
    assert call(b"i", 7, _capi.ACC_I32, ip) == 0 and call(b"i", 8, _capi.ACC_I32, ip) == 0
    assert call(b"i", 4, _capi.ACC_I32, ip) == 0
    assert (dev_bytes(torch, store.query("i")["local_base"], 16).view(np.int32) == 1).all()
    assert call(b"e", 1, _capi.ACC_F32, p) == 0   # DDS_OP_SUM: the accumulate itself
    assert (dev_bytes(torch, store.query("e")["local_base"], 16).view(np.float32) == 1).all()


def test_queue_endings_and_stream_order(torch, store):
    """queued amax batches between overlapped get runs on one stream: each get sees exactly what was queued before it;
    a bad request of a queued reduction is reported once by wait(), the valid ones applied"""
    nrows, disp = 2048, 256
    store.add("o", np.zeros((nrows, disp), np.float32))
    h = torch.cuda.Stream().cuda_stream
    starts = torch.arange(0, nrows, 2, device="cuda:0")
    zero = torch.zeros(starts.numel(), disp, device="cuda:0")
    a, b = zero + 3.0, zero - 7.0
    outs = [torch.zeros_like(a) for _ in range(9)]
    prev = torch.full_like(a, -1)
    torch.cuda.synchronize()
    for k in range(3):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.accumulate_batch("o", starts, src=a, count=1, stream=h, wait=False, op="amax")
    for k in range(3, 6):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.get_accumulate_batch("o", starts, src=b, out=prev, count=1, stream=h, wait=False, op="amin")
    for k in range(6, 9):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.wait()
    for k in range(9):
        assert outs[k].eq(0.0 if k < 3 else 3.0 if k < 6 else -7.0).all(), k
    assert prev.eq(3.0).all()
    badi = starts.clone()
    badi[7] = nrows + 1
    store.accumulate_batch("o", badi, src=a + 10, count=1, stream=h, wait=False, op="amax")
    with pytest.raises(ValueError, match="Invalid count on target"):
        store.wait()
    assert store.last_bad_index == 7
    sh = dev_bytes(torch, store.query("o")["local_base"], nrows * disp * 4).view(np.float32).reshape(nrows, disp)
    assert (sh[0:14:2] == 13.0).all() and (sh[16::2] == 13.0).all() and (sh[14] == -7.0).all()
    assert store.wait() == 0


# ------------------------------------------------------------------------------------------------ bindings
def test_cython_and_cpp_bindings(torch, tmp_path):
    """accumulate_batch(op=...) and get_accumulate_batch(op=...) through the Cython binding, and
    DDStore::accumulate_op_batch<T> / the explicit-dtype overload / accumulate_op_samples through the C++ header"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    s = pyd.PyDDStore(None, device=0)
    s.add("c", np.full((8, 3), 2, np.int32))
    src = torch.tensor([[1, 5, -3], [4, 4, 9]], dtype=torch.int32, device="cuda:0")
    out = torch.zeros(2, 3, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    assert s.accumulate_batch("c", np.array([1, 2], np.int64), src=src, count=1, op="amax") == 24
    got = np.zeros((2, 3), np.int32)
    s.get("c", got, 1)
    assert got.tolist() == [[2, 5, 2], [4, 4, 9]]
    assert s.get_accumulate_batch("c", np.array([1, 1], np.int64), src=src, out=out, op="bitwise_xor", count=1) == 24
    s.get("c", got, 1)
    x, o, v = src.cpu().numpy(), out.cpu().numpy(), np.array([2, 5, 2], np.int32)
    assert got[0].tolist() == (v ^ x[0] ^ x[1]).tolist()
    for c in range(3):  # one of the two orders per element
        assert (o[0, c], o[1, c]) in ((v[c], v[c] ^ x[0, c]), (v[c] ^ x[1, c], v[c])), c
    with pytest.raises(ValueError, match="is not one of"):
        s.accumulate_batch("c", np.array([1], np.int64), src=src[:1], op="max")
    s.free()
    exe = build_cpp_check(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cpp accumulate_op ok" in r.stdout, r.stdout + r.stderr


CPP_CHECK = r"""
#include <cuda_runtime.h>
#include <cstdio>
#include "ddstore_b200.hpp"
int main() {
    DDStore s;
    std::vector<int64_t> k(4, 10);
    std::vector<float> f(4, 1.0f);
    s.add("k", k.data(), 4, 1);
    s.add("f", f.data(), 4, 1);
    const long starts[3] = {2, 2, 2};
    int64_t *dk; float *df; long *ds;
    cudaMalloc(&dk, 24); cudaMalloc(&df, 12); cudaMalloc(&ds, 24);
    int64_t hk[3] = {1, 2, 4};
    float hf[3] = {-2.0f, 0.5f, 3.0f};
    cudaMemcpy(dk, hk, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(df, hf, 12, cudaMemcpyHostToDevice);
    cudaMemcpy(ds, starts, 24, cudaMemcpyHostToDevice);
    if (s.accumulate_op_batch<int64_t>("k", ds, nullptr, 1, 3, DDS_OP_BOR, dk, 24) != 24) return 2;
    if (s.accumulate_op_batch("f", starts, nullptr, 1, 3, DDS_OP_MIN, DDS_ACC_F32, df, 12, false) != 12) return 3;
    try { s.accumulate_op_samples<float>("f", ds, 1, DDS_OP_MAX, df, 4); return 4; }  // (no sample index)
    catch (std::exception &) {}
    try { s.accumulate_op_batch<float>("f", starts, nullptr, 1, 1, DDS_OP_BAND, df, 4, false); return 5; }
    catch (std::exception &) {}
    s.get("k", 2, 1, k.data());
    s.get("f", 2, 1, f.data());
    if (k[0] != (10 | 1 | 2 | 4) || f[0] != -2.0f) return 6;
    s.free();
    printf("cpp accumulate_op ok\n");
    return 0;
}
"""


def build_cpp_check(tmp_path):
    src = tmp_path / "red_check.cpp"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "red_check")
    lib = os.path.join(ROOT, "ddstore_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
           "-L", lib, "-lddstore_b200", f"-Wl,-rpath,{lib}", "-L", "/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe
