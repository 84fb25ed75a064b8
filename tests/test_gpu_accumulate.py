"""Batched accumulates (dds_accumulate_batch / dds_accumulate_samples) on the GPU against the NumPy oracle of
tests/acc_oracle.py.

Every check compares the WHOLE local shard -- every row, and the zero slack past the last row -- with the oracle's. Data
are small integers, so every sum is exact in every type and the expectation does not depend on the order in which the
device applies the contributions. The sweep runs in subprocesses, one per configuration (plan placement, segment size,
PDL), as the put's does.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import put_oracle as po
from tests import put_world as pw
from tests.gpu_helpers import padded_requests, run_world, sweep_requests
from tests.put_world import dense_cover
from tests.test_gpu_put import CONFIGS, ERR, inject_invalid, shard_state, to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)
E = {t: np.dtype(ao.STORAGE[t]).itemsize for t in ALL}


# ------------------------------------------------------------------------------------------------ helpers
def _index(torch, x, dev, device="cuda:0"):
    """(keepalive, pointer, length, IDX_ON_DEVICE or 0): device int64 tensors when `dev`, else host int64 arrays"""
    from ddstore_b200 import _capi
    a = np.ascontiguousarray(x, np.int64)
    if dev:
        t = torch.from_numpy(a).to(device)
        torch.cuda.synchronize(device)
        return t, t.data_ptr(), t.numel(), _capi.IDX_ON_DEVICE
    return a, a.ctypes.data, a.size, 0


def raw_acc(torch, store, name, t, src_ptr, src_bytes, starts=None, counts=None, fixed=1, ids=None, dev=False, flags=0,
            stream=None, device="cuda:0", keep=None):
    """the C-ABI entry itself -> (rc, total, bad); `keep` (a list): receives the index arrays, which a queued call
    needs alive until it has run"""
    from ddstore_b200 import _capi
    L, total, bad = store._L, C.c_int64(0), C.c_int64(-1)
    fl = _capi.SRC_ON_DEVICE | flags
    if ids is not None:
        keep_i, ip, n, d = _index(torch, ids, dev, device)
        rc = L.dds_accumulate_samples(store._h, name.encode(), ip, n, t, src_ptr, src_bytes, fl | d, stream,
                                      C.byref(total), C.byref(bad))
        held = (keep_i,)
    else:
        keep_i, sp, n, d = _index(torch, starts, dev, device)
        keep2, cp = (None, None) if counts is None else _index(torch, counts, dev, device)[:2]
        rc = L.dds_accumulate_batch(store._h, name.encode(), sp, cp, fixed, n, t, src_ptr, src_bytes, fl | d, stream,
                                    C.byref(total), C.byref(bad))
        held = (keep_i, keep2)
    if keep is not None:
        keep.append(held)
    return rc, total.value, bad.value


def add_var(torch, store, name, shard_bytes, nrows, disp, itemsize, device="cuda:0"):
    buf = torch.from_numpy(np.ascontiguousarray(shard_bytes)).to(device) if shard_bytes.size else None
    torch.cuda.synchronize(device)
    rc = store._L.dds_add(store._h, name.encode(), buf.data_ptr() if buf is not None else None, nrows, disp, itemsize, 1)
    assert rc == 0, store._L.dds_last_error()


class World:
    """one rank on cuda:0 with variable `name` of element type t: small random integers, a sample index"""

    def __init__(self, torch, store, name, t, disp, nrows, seed, table=None):
        self.rng = np.random.default_rng(seed)
        self.t, self.disp, self.rows, self.name = t, disp, nrows, name
        self.R = E[t] * disp
        self.payload = nrows * self.R
        self.shard = ao.encode(self.rng.integers(-8, 8, size=(nrows, disp)), t)
        add_var(torch, store, name, self.shard.view(np.uint8).reshape(-1), nrows, disp, E[t])
        self.table = table
        if table is not None:
            store.set_sample_index(name, table[0], table[1])

    def reset(self, torch, store):
        """the original rows back, by a put of the whole shard"""
        from ddstore_b200 import _capi
        buf, ptr = to_device(torch, self.shard.view(np.uint8).reshape(-1), 0)
        total, bad = C.c_int64(0), C.c_int64(-1)
        sa = np.zeros(1, np.int64)
        rc = store._L.dds_put_batch(store._h, self.name.encode(), sa.ctypes.data, None, self.rows, 1, E[self.t], ptr,
                                    self.payload, _capi.SRC_ON_DEVICE, None, C.byref(total), C.byref(bad))
        assert rc == 0 and total.value == self.payload, (rc, total.value, self.payload, store._L.dds_last_error())

    def check(self, torch, store, what, src_off=0, src_bytes=None, dev=False, **req):
        """accumulate `req` from a source `src_off` bytes past a 16-byte boundary; compare status, total and the whole
        shard with the oracle; restore the shard"""
        assert src_off % E[self.t] == 0
        ll = po.lenlist_of([self.shard])
        src = ao.layout_src(self.rng, ll, self.disp, self.t, req)
        sb = src.size if src_bytes is None else src_bytes
        buf, ptr = to_device(torch, src, src_off)
        kw = dict(req)
        if "table" in kw:
            kw.pop("table")
            kw["ids"] = kw.pop("sample_ids")
        if "fixed_count" in kw:
            kw["fixed"] = kw.pop("fixed_count")
        rc, total, bad = raw_acc(torch, store, self.name, self.t, ptr if src.size else None, sb, dev=dev, **kw)
        new, codes, ebad, etotal = ao.accumulate([self.shard], src, self.t, src_bytes=sb, **req)
        ecode, ebad2 = po.expected_error(codes, ebad, etotal, sb)
        assert (rc, bad) == (ERR[ecode], ebad2), f"{what}: rc {rc} bad {bad}, oracle {ERR[ecode]} {ebad2}"
        assert total == etotal, f"{what}: total {total}, oracle {etotal}"
        got, slack = shard_state(torch, store, self.name, self.payload)
        msg = ao.mismatch(got[:self.payload], new[0], 0, ll, self.R, what)
        assert msg is None, msg
        assert not got[self.payload:].any(), f"{what}: the shard's slack was written"
        self.reset(torch, store)
        return codes


# ------------------------------------------------------------------------------------------------ the sweep
# (disp, rows) per element type: ragged rows of a few elements (one element for the integer types) over ~13 MiB
SHAPES = {ao.ACC_F32: (5, (13 << 20) // 20), ao.ACC_F64: (3, (13 << 20) // 24), ao.ACC_I32: (1, (13 << 20) // 4),
          ao.ACC_I64: (1, (13 << 20) // 8), ao.ACC_F16: (3, (13 << 20) // 6), ao.ACC_BF16: (7, (13 << 20) // 14)}
BIG_DISP = 65543  # the largest rows: 65543 elements
DENSE_ROWS = 16400


def acc_sweep_main():
    import torch
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    cfg = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("DDS_")) or "default"
    for t in ALL:
        rng = np.random.default_rng(t)
        disp, nrows = SHAPES[t]
        tn = ao.NAMES[t]
        starts, counts = sweep_requests(rng, nrows, E[t] * disp, (4096, 3072))
        table = (starts.copy(), counts.copy())
        w = World(torch, store, f"v{t}", t, disp, nrows, t, table)
        # every element-aligned source offset of a 16-byte block: direct, same-phase and re-phased pieces
        for k, off in enumerate(range(0, 16, E[t])):
            w.check(torch, store, f"[{cfg}] {tn} counts, src +{off}", src_off=off, dev=k % 2 == 1, starts=starts, counts=counts)
        ids = np.concatenate([np.arange(len(starts)), rng.integers(0, len(starts), size=64)])  # 64 duplicates
        ids = rng.permutation(ids).astype(np.int64)
        for dev in (False, True):
            w.check(torch, store, f"[{cfg}] {tn} sample ids dev={dev}", src_off=(8 if dev else 0) % 16, dev=dev,
                    sample_ids=ids, table=table)
        fs = rng.integers(0, nrows - 40, size=300)
        for cnt in (1, 3, 40):
            w.check(torch, store, f"[{cfg}] {tn} fixed {cnt}", src_off=(E[t] * cnt) % 16, dev=cnt != 3, starts=fs,
                    fixed_count=cnt)
        for n in (1024, 1025, 4096, 4097, 8192, 8193):  # both sides of the shared-memory plan's thresholds
            s2, c2 = padded_requests(rng, nrows, starts, counts, n)
            w.check(torch, store, f"[{cfg}] {tn} n={n}", src_off=(E[t] * n) % 16, dev=n % 2 == 0, starts=s2, counts=c2)
        # invalid requests at the walk's lane edges, the plan tiles' edges and at 1 % density; capacity errors
        s2, c2 = padded_requests(rng, nrows, starts, counts, 2100)
        for where in ([0, 31, 32, 63, 1023, 1024, 2047, 2048], sorted(rng.choice(2100, size=21, replace=False).tolist())):
            si, ci = inject_invalid(rng, s2, c2, nrows, where)
            codes = w.check(torch, store, f"[{cfg}] {tn} invalid {where[:4]}", src_off=E[t], starts=si, counts=ci)
            assert codes[where[0]] != 0
            total = sum(c * w.R if 0 < c <= nrows else 0 for c in ci.tolist())
            w.check(torch, store, f"[{cfg}] {tn} capacity + invalid", src_bytes=total - 1, starts=si, counts=ci)
            w.check(torch, store, f"[{cfg}] {tn} invalid ids", dev=True,
                    sample_ids=np.where(np.isin(np.arange(ids.size), where), -5, ids), table=table)
        w.check(torch, store, f"[{cfg}] {tn} capacity", src_bytes=int(counts.sum()) * w.R - 1, starts=starts, counts=counts)
        w.check(torch, store, f"[{cfg}] {tn} fixed capacity", src_bytes=300 * 3 * w.R - 1, dev=True, starts=fs, fixed_count=3)
        # every row of a small variable exactly once per batch: every piece's neighbours are reduced by other warps
        ds, dc = dense_cover(rng, DENSE_ROWS, 4097)
        d = World(torch, store, f"d{t}", t, disp, DENSE_ROWS, 100 + t, (ds.copy(), dc.copy()))
        d.check(torch, store, f"[{cfg}] {tn} dense sample ids", src_off=E[t] * 3 % 16, dev=True,
                sample_ids=rng.permutation(4097), table=d.table)
        for n in (1025, 4097, 8193):
            ds, dc = dense_cover(rng, DENSE_ROWS, n)
            d.check(torch, store, f"[{cfg}] {tn} dense n={n}", src_off=(E[t] * n) % 16, starts=ds, counts=dc)
        d.check(torch, store, f"[{cfg}] {tn} dense fixed 1", src_off=E[t], dev=True, starts=rng.permutation(DENSE_ROWS),
                fixed_count=1)
        # rows of 65543 elements
        b = World(torch, store, f"b{t}", t, BIG_DISP, 24, 200 + t)
        bs = np.array([0, 23, 5, 5, 11, 0], np.int64)
        bc = np.array([2, 1, 1, 3, 13, 0], np.int64)
        for off in (0, E[t], 16 - E[t]):
            b.check(torch, store, f"[{cfg}] {tn} 65543-element rows, src +{off}", src_off=off, dev=off > 0, starts=bs, counts=bc)
        b.check(torch, store, f"[{cfg}] {tn} 65543-element rows fixed", src_off=8 % 16, starts=[3, 20, 3], fixed_count=2)
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_accumulate import acc_sweep_main
acc_sweep_main()
print("acc-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_accumulate_sweep(tmp_path, config):
    """every element type over the variant sweep's request sizes, src at every element-aligned offset of a 16-byte block,
    every entry with host and device indices, batch sizes around the plan thresholds, invalid requests, capacity
    errors, dense batches and 65543-element rows, in the environment of `config`"""
    script = tmp_path / "acc_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "acc-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]


# ------------------------------------------------------------------------------------------------ in-process checks
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


def _shard(torch, store, name, nrows, disp, dtype):
    base = store.query(name)["local_base"]
    from ddstore_b200.store import _DevMem
    n = nrows * disp * torch.tensor([], dtype=dtype).element_size()
    return torch.as_tensor(_DevMem(base, n), device="cuda:0").view(dtype).view(nrows, disp)


@pytest.mark.parametrize("src_off", [0, 4])
@pytest.mark.parametrize("dtype", ["float32", "int32"])
def test_hot_row_one_batch(torch, store, dtype, src_off):
    """65536 requests of ONE 4 KiB row in one batch (sample ids and fixed counts): the exact count shows every bulk
    (src_off 0) or vector (src_off 4: re-phased) reduction combined atomically across SMs"""
    dt = getattr(torch, dtype)
    nrows, disp, n = 64, 1024, 65536
    store.add("h", np.zeros((nrows, disp), np.float32 if dtype == "float32" else np.int32))
    store.set_sample_index("h", np.arange(nrows, dtype=np.int64), np.ones(nrows, np.int64))
    buf = torch.ones(n * disp + 4, dtype=dt, device="cuda:0")
    src = buf[src_off // 4:src_off // 4 + n * disp]
    idx = torch.full((n,), 17, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    assert store.accumulate_batch("h", idx, src=src) == n * disp * 4
    assert store.accumulate_samples("h", idx, src) == n * disp * 4
    sh = _shard(torch, store, "h", nrows, disp, dt)
    assert sh[17].eq(2 * n).all(), sh[17].unique()
    sh[17] = 0
    assert not sh.any()


@pytest.mark.parametrize("dtype", ["float32", "int64", "int32"])
def test_hot_row_four_ranks(torch, dtype):
    """every thread-rank of a 4-rank world adds into the same row in the same epoch, 4096 times each, and each rank
    also adds 1 to every row of the world once: after the fence every element holds the exact count"""
    P, N, disp, n = 4, 33, 1000, 4096
    dt = getattr(torch, dtype)

    def body(store, r):
        import torch as t
        dev = t.device("cuda", t.cuda.current_device())
        store._L.dds_init(store._h, b"c", N, disp, t.tensor([], dtype=dt).element_size())
        store.epoch_begin()
        hot = t.full((n,), N + 5, dtype=t.int64, device=dev)  # rank 1's row 5
        one = t.ones(n * disp, dtype=dt, device=dev)
        allrows = t.arange(P * N, dtype=t.int64, device=dev)[t.randperm(P * N, device=dev)]
        t.cuda.synchronize(dev)
        store.accumulate_batch("c", hot, src=one)
        store.accumulate_batch("c", allrows, src=one[:P * N * disp], wait=False)
        store.epoch_end()
        mine = _shard(t, store, "c", N, disp, dt).float()
        exp = t.full((N, disp), float(P), device=dev)
        if r == 1:
            exp[5] += P * n
        return bool(t.equal(mine, exp))
    assert all(run_world(P, body))


def test_queue_endings(torch, store):
    """queued accumulates completed by wait(), by a synchronous call, by epoch_begin and by epoch_end: every queued
    contribution is in place, the first failure is reported once, with its index"""
    nrows, disp = 1000, 16
    store.add("q", np.zeros((nrows, disp), np.int32))
    h = torch.cuda.Stream().cuda_stream
    good = torch.arange(0, 500, device="cuda:0")
    bad = good.clone()
    bad[7] = nrows + 1
    src = torch.ones(500, disp, dtype=torch.int32, device="cuda:0")
    sh = _shard(torch, store, "q", nrows, disp, torch.int32)
    torch.cuda.synchronize()
    store.accumulate_batch("q", good, src=src, stream=h, wait=False)
    store.accumulate_batch("q", bad, src=src * 2, stream=h, wait=False)
    with pytest.raises(ValueError, match="Invalid count on target"):
        store.wait()
    assert store.last_bad_index == 7
    assert sh[:500].sum(1).tolist() == [3 * disp] * 7 + [disp] + [3 * disp] * 492 and not sh[500:].any()
    expect = 3
    for ending in ("wait", "sync", "epoch_begin", "epoch_end"):
        if ending == "epoch_end":
            store.epoch_begin()
        store.accumulate_batch("q", bad, src=src, stream=h, wait=False)
        store.accumulate_batch("q", good, src=src, stream=h, wait=False)
        expect += 2
        if ending == "wait":
            with pytest.raises(ValueError, match="Invalid count on target"):
                store.wait()
        elif ending == "sync":
            assert store.accumulate_batch("q", good[:10], src=src[:10]) == 10 * disp * 4  # its own outcome: ok
        else:
            getattr(store, ending)()
        row = sh[20].clone()  # (nothing else synchronised the queue)
        assert row.eq(expect).all(), (ending, row)
        if ending != "wait":
            with pytest.raises(ValueError, match="Invalid count on target"):
                store.wait()
        assert store.last_bad_index == 7
        if ending == "epoch_begin":
            store.epoch_end()
    assert store.wait() == 0


def test_stream_ordering_with_overlapped_gets(torch, store):
    """an overlapped get run, an accumulate, a put, an overlapped get run on one stream: each get sees exactly what
    was queued before it"""
    nrows, disp = 2048, 256
    store.add("o", np.zeros((nrows, disp), np.float32))
    h = torch.cuda.Stream().cuda_stream
    starts = torch.arange(0, nrows, 2, device="cuda:0")
    a = torch.full((starts.numel(), disp), 3.0, device="cuda:0")
    b = torch.ones_like(a)
    outs = [torch.zeros_like(a) for _ in range(9)]
    torch.cuda.synchronize()
    for k in range(3):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.accumulate_batch("o", starts, src=a, stream=h, wait=False)
    for k in range(3, 6):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.put_batch("o", starts, src=b, stream=h, wait=False)
    store.accumulate_batch("o", starts, src=a, stream=h, wait=False)
    for k in range(6, 9):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.wait()
    for k in range(9):
        assert outs[k].eq(0.0 if k < 3 else 3.0 if k < 6 else 4.0).all(), k


def test_round_trips(torch, store):
    """after accumulates, get_batch, get_samples and get() (doorbell on and off) read the sums"""
    rng = np.random.default_rng(3)
    nrows, disp = 4000, 37
    base = rng.integers(-5, 5, size=(nrows, disp)).astype(np.float32)
    store.add("x", base)
    rs = np.sort(rng.choice(nrows - 20, size=300, replace=False)).astype(np.int64)
    rc = np.minimum(rng.integers(1, 20, size=300), np.append(np.diff(rs), 20)).astype(np.int64)
    store.set_sample_index("x", rs, rc)
    ids = rng.permutation(np.concatenate([np.arange(300), np.arange(0, 300, 7)])).astype(np.int64)  # duplicates
    rows = np.concatenate([np.arange(rs[i], rs[i] + rc[i]) for i in ids])
    vals = torch.from_numpy(rng.integers(-3, 4, size=(rows.size, disp)).astype(np.float32)).cuda()
    torch.cuda.synchronize()
    assert store.accumulate_samples("x", torch.from_numpy(ids).cuda(), vals) == vals.numel() * 4
    exp = base.copy()
    np.add.at(exp, rows, vals.cpu().numpy())
    out = torch.empty(nrows, disp, device="cuda:0")
    store.get_batch("x", [0], [nrows], out=out)
    assert np.array_equal(out.cpu().numpy(), exp)
    got = torch.empty(int(rc.sum()), disp, device="cuda:0")
    store.get_samples("x", np.arange(300), got)
    assert np.array_equal(got.cpu().numpy(), np.concatenate([exp[rs[i]:rs[i] + rc[i]] for i in range(300)]))
    one = np.zeros((2, disp), np.float32)
    for g in (int(rows[0]), int(rows[-1]) - 1):
        store.get("x", one, g)
        assert one.tobytes() == exp[g:g + 2].tobytes()


def test_errors(torch, store):
    from ddstore_b200 import _capi
    store.add("e", np.zeros((10, 4), np.float32))
    src = torch.zeros(2, 4, device="cuda:0")
    with pytest.raises(KeyError):
        store.accumulate_batch("nope", [0, 1], src=src)
    with pytest.raises(ValueError, match="device memory"):
        store.accumulate_batch("e", [0, 1], src=np.zeros((2, 4), np.float32))
    with pytest.raises(ValueError, match="Invalid data type"):
        store.accumulate_batch("e", [0, 1], src=src.double())
    with pytest.raises(ValueError, match="is not one of"):
        store.accumulate_batch("e", [0, 1], src=src.view(torch.uint8))
    with pytest.raises(ValueError, match="no sample index"):
        store.accumulate_samples("e", [0], src=src)
    assert store.accumulate_batch("e", np.zeros(0, np.int64), src=src) == 0
    total, bad = C.c_int64(0), C.c_int64(0)
    sa = np.zeros(1, np.int64)

    def call(t, ptr, flags=_capi.SRC_ON_DEVICE, nreq=1):
        return store._L.dds_accumulate_batch(store._h, b"e", sa.ctypes.data, None, 1, nreq, t, ptr, 32, flags, None,
                                             C.byref(total), C.byref(bad))
    p = src.data_ptr()
    assert call(0, p) == _capi.ERR_ARG and call(7, p) == _capi.ERR_ARG       # unknown dtype
    assert call(_capi.ACC_I64, p) == _capi.ERR_DTYPE                          # 8-byte type, 4-byte variable
    assert call(_capi.ACC_I32, p) == 0                                        # same size: the sum is taken as int32
    assert call(_capi.ACC_F32, p + 2) == _capi.ERR_ARG and "aligned" in _capi.last_error()  # misaligned src
    assert call(_capi.ACC_F32, p, flags=0) == _capi.ERR_ARG                   # host src
    assert call(_capi.ACC_F32, None) == _capi.ERR_ARG                         # null src
    assert call(_capi.ACC_F32, p, nreq=-1) == _capi.ERR_ARG
    assert call(_capi.ACC_F32, p, flags=_capi.SRC_ON_DEVICE | _capi.NO_SYNC) == _capi.ERR_ARG  # async, host indices
    assert not _shard(torch, store, "e", 10, 4, torch.float32).any()  # (the int32 sum of zero bits is zero bits)


def test_cython_and_cpp_bindings(torch, tmp_path):
    """accumulate_batch through the Cython binding, and DDStore::accumulate_batch<T> / the explicit-code overload /
    accumulate_samples through the C++ header"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    s = pyd.PyDDStore(None, device=0)
    s.add("c", np.ones((8, 3), np.float32))
    src = torch.arange(6, dtype=torch.float32, device="cuda:0").reshape(2, 3)
    torch.cuda.synchronize()
    assert s.accumulate_batch("c", np.array([1, 1], np.int64), src=src) == 24
    got = np.zeros((1, 3), np.float32)
    s.get("c", got, 1)
    assert got.tolist() == [[1 + 0 + 3, 1 + 1 + 4, 1 + 2 + 5]]
    with pytest.raises(ValueError, match="Invalid start on target"):
        s.accumulate_batch("c", np.array([-1], np.int64), src=src[:1])
    s.free()
    exe = build_cpp_check(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cpp accumulate ok" in r.stdout, r.stdout + r.stderr


CPP_CHECK = r"""
#include <cuda_runtime.h>
#include <cstdio>
#include "ddstore_b200.hpp"
int main() {
    DDStore s;
    std::vector<float> f(4 * 3, 1.0f);
    std::vector<int32_t> i(4 * 3, 5);
    std::vector<uint16_t> h(4 * 3, 0x3f80);  // bf16 1.0
    s.add("f", f.data(), 4, 3);
    s.add("i", i.data(), 4, 3);
    s.add("h", h.data(), 4, 3);
    const long starts[2] = {2, 2};
    float *df; int32_t *di; uint16_t *dh; long *ds;
    cudaMalloc(&df, 24); cudaMalloc(&di, 12); cudaMalloc(&dh, 12); cudaMalloc(&ds, 16);
    float hf[6] = {1, 2, 3, 4, 5, 6};
    int32_t hi[3] = {-5, 7, 1 << 30};
    uint16_t hh[6] = {0x3f80, 0x3f80, 0x4000, 0x3f80, 0x3f80, 0x4000};  // 1, 1, 2
    cudaMemcpy(df, hf, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(di, hi, 12, cudaMemcpyHostToDevice);
    cudaMemcpy(dh, hh, 12, cudaMemcpyHostToDevice);
    cudaMemcpy(ds, starts, 16, cudaMemcpyHostToDevice);
    if (s.accumulate_batch<float>("f", ds, nullptr, 1, 2, df, 24) != 24) return 2;
    if (s.accumulate_batch("h", starts, nullptr, 1, 2, DDS_ACC_BF16, dh, 12, false) != 12) return 3;
    if (s.accumulate_batch<int32_t>("i", starts, nullptr, 1, 1, di, 12, false) != 12) return 4;
    try { s.accumulate_batch<double>("f", starts, nullptr, 1, 1, (const double *)df, 24, false); return 5; }
    catch (std::invalid_argument &e) { if (std::string(e.what()) != "Invalid data type") return 6; }
    s.get("f", 2, 1, f.data());
    s.get("i", 2, 1, i.data());
    s.get("h", 2, 1, h.data());
    if (f[0] != 1 + 1 + 4 || f[1] != 1 + 2 + 5 || f[2] != 1 + 3 + 6) return 7;
    if (i[0] != 0 || i[1] != 12 || i[2] != (1 << 30) + 5) return 8;
    if (h[0] != 0x4040 || h[1] != 0x4040 || h[2] != 0x40a0) return 9;  // 3, 3, 5
    s.free();
    printf("cpp accumulate ok\n");
    return 0;
}
"""


def build_cpp_check(tmp_path):
    src = tmp_path / "acc_check.cpp"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "acc_check")
    lib = os.path.join(ROOT, "ddstore_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
           "-L", lib, "-lddstore_b200", f"-Wl,-rpath,{lib}", "-L", "/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


# ------------------------------------------------------------------------------------------------ other ranks
ROWS = {2: [1, 23], 3: [19, 0, 8], 4: [0, 26, 1, 9]}


def acc_world(torch, P, nrows, t, disp, seed, readers=False, devices=None, queued=False):
    """P thread-ranks; every rank accumulates into every other rank's rows (owner edges, straddlers and the invalid
    family, a by-sample-id form, a dense cover of the world, one call per rank short of source); after the closing fence
    every rank compares its whole shard and its own calls' (status, bad index, total) with the oracle"""
    rng = np.random.default_rng([seed, P, t])
    ll = pw.lenlist_of(nrows)
    R = E[t] * disp
    shards = [ao.encode(rng.integers(-8, 8, size=(n, disp)), t) for n in nrows]
    total = int(ll[-1])
    tables = []
    calls = []  # calls[r] = [(src bytes, src_bytes or None, batch, src offset)]
    cover = pw.interleaved_cover(rng, ll, P, R, big=R <= 64)
    for r in range(P):
        others = [o[0] for o in pw.owners(ll) if o[0] != r] or None
        st, ct, cls = pw.edge_requests(rng, ll, r, first_bad=None if r == 0 else int(rng.integers(0, 6)), body=12,
                                       only=others)
        mine = []
        b = {"starts": st, "counts": ct}
        mine.append((ao.layout_src(rng, ll, disp, t, b), None, b, E[t] * (r % (16 // E[t]))))
        sb, _ = pw.as_samples(rng, st, ct, cls, first_bad=None if r % 2 == 0 else 1)
        tables.append(sb["table"])
        mine.append((ao.layout_src(rng, ll, disp, t, sb), None, sb, 0))
        cb = {"starts": cover[r][0], "counts": cover[r][1]}
        mine.append((ao.layout_src(rng, ll, disp, t, cb), None, cb, E[t]))
        if r == P - 1 and total:
            fb = {"starts": np.array([0, total - 1], np.int64), "fixed_count": 1}
            full = ao.layout_src(rng, ll, disp, t, fb)
            mine.append((full, full.size - 1, fb, 0))  # capacity: nothing applied
        calls.append(mine)
    flat = [(c[0], c[1], c[2]) for mine in calls for c in mine]
    exp, triples = ao.accumulate_many(shards, flat, t)
    it = iter(triples)
    exp_status = [[next(it) for _ in mine] for mine in calls]

    def body(store, r):
        import torch as tt
        dev = tt.device("cuda", tt.cuda.current_device())
        problems = []
        mine = np.ascontiguousarray(shards[r]).view(np.uint8).reshape(-1)
        assert store._L.dds_add(store._h, b"w", mine.ctypes.data if mine.size else None, nrows[r], disp, E[t], 0) == 0
        store.set_sample_index("w", *tables[r])
        stream = tt.cuda.Stream(device=dev).cuda_stream if queued else None
        keep = []
        store.epoch_begin()
        for k, (src, sbytes, batch, off) in enumerate(calls[r]):
            buf, ptr = to_device(tt, src, off, dev)
            keep.append(buf)
            sb = src.size if sbytes is None else sbytes
            kw = {"ids": batch["sample_ids"]} if "sample_ids" in batch else \
                {"starts": batch["starts"], "counts": batch.get("counts"), "fixed": batch.get("fixed_count", 1)}
            got = raw_acc(tt, store, "w", t, ptr if src.size else None, sb, dev=queued or k % 2 == 1,
                          flags=(4 if queued else 0), stream=stream, device=dev, keep=keep, **kw)
            code, bad, etotal = exp_status[r][k]
            if queued:
                if got[0] != 0:
                    problems.append(f"rank {r} call {k}: queueing returned {got}")
            elif got != (ERR[code], etotal, bad):
                problems.append(f"rank {r} call {k}: (rc, total, bad) = {got}, oracle {(ERR[code], etotal, bad)}")
        store.epoch_end()
        if queued:
            total_, bad_ = C.c_int64(0), C.c_int64(-1)
            rc = store._L.dds_batch_wait(store._h, C.byref(total_), C.byref(bad_))
            first = next(((c, b) for c, b, _ in exp_status[r] if c), (0, -1))
            if (rc, bad_.value) != (ERR[first[0]], first[1]):
                problems.append(f"rank {r}: wait() -> {(rc, bad_.value)}, oracle {(ERR[first[0]], first[1])}")
        payload = nrows[r] * R
        got, slack = shard_state(tt, store, "w", payload, dev)
        m = ao.mismatch(got[:payload], exp[r], r, ll, R, f"P={P} {ao.NAMES[t]}")
        if m:
            problems.append(m)
        if got[payload:].any():
            problems.append(f"rank {r}: slack written")
        if readers and total:
            world = np.concatenate([e.view(np.uint8).reshape(-1) for e in exp])
            out = tt.zeros(total, disp, dtype=getattr(tt, ao.NAMES[t]), device=dev)
            tt.cuda.synchronize(dev)
            store.get_batch("w", np.arange(total), out=out)  # (one row per request: a request never spans owners)
            if not np.array_equal(out.cpu().numpy().view(np.uint8).reshape(-1), world):
                problems.append(f"rank {r}: get_batch of the world differs")
            one = np.zeros(R, np.uint8)
            for g in (0, total - 1, int(ll[r]) - 1 if nrows[r] else 0):
                store._L.dds_get(store._h, b"w", g, 1, E[t], one.ctypes.data, 0)
                if one.tobytes() != world[g * R:(g + 1) * R].tobytes():
                    problems.append(f"rank {r}: get() of row {g} differs")
        return problems
    res = run_world(P, body, devices=devices)
    problems = [p for r in res for p in r]
    assert not problems, "\n".join(problems[:12])


@pytest.mark.parametrize("P", [2, 3, 4])
@pytest.mark.parametrize("t", [ao.ACC_I32, ao.ACC_F32, ao.ACC_BF16, ao.ACC_F64])
def test_multi_owner_worlds(torch, P, t):
    acc_world(torch, P, [n * 20 if n > 1 else n for n in ROWS[P]], t, {ao.ACC_I32: 3, ao.ACC_F32: 5, ao.ACC_BF16: 7,
                                                                      ao.ACC_F64: 2}[t], seed=1)


@pytest.mark.parametrize("doorbell", [True, False])
def test_three_owner_world_readers_queued(torch, monkeypatch, doorbell):
    """queued accumulates completed by the fence, the world read back through get_batch and get() (doorbell kernel,
    and DDS_DOORBELL=0)"""
    monkeypatch.setenv("DDS_DOORBELL", "1" if doorbell else "0")
    monkeypatch.setenv("DDS_DOORBELL_IDLE_US", "5000000")
    acc_world(torch, 3, [380, 0, 160], ao.ACC_I64, 3, seed=2, readers=True, queued=True)


def test_sixty_four_owners(torch):
    rng = np.random.default_rng(64)
    nrows = [0 if k % 3 == 0 else int(rng.integers(1, 6)) for k in range(64)]
    acc_world(torch, 64, nrows, ao.ACC_I32, 5, seed=3)


def test_one_gpu_per_rank(torch):
    """the same across GPUs: bulk and element reductions into peer HBM over NVLink"""
    P = torch.cuda.device_count()
    if P < 2:
        pytest.skip("needs two or more GPUs")
    acc_world(torch, P, [37 * (k + 1) for k in range(P)], ao.ACC_F32, 1024, seed=4, devices=list(range(P)))
