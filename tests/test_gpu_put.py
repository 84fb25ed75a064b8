"""Batched puts (dds_put_batch / dds_put_samples) on the GPU against the NumPy oracle of tests/put_oracle.py.

Every check compares the WHOLE local shard -- every row, and the zero slack past the last row -- with the oracle's, not
only the rows that were put. Requests may overlap: the rows a batch writes are a fixed pattern of the destination byte
(`pattern`), so two writes of the same bytes write the same values and the result is exact (the duplicates test covers
writes of different values). The sweep runs in subprocesses, one per configuration (plan placement, segment size, PDL).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import put_oracle as po
from tests.gpu_helpers import padded_requests, run_world, sweep_requests
from tests.put_world import dense_cover

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR = {0: 0, po.CODE_START: 2, po.CODE_COUNT: 3, po.CODE_CAPACITY: 12, po.CODE_SAMPLE: 11}  # oracle code -> DDS_ERR_*
SRC_OFFSETS = (0, 1, 4, 8, 13)
CONFIGS = {"default": {},
           "smem8192": {"DDS_SMEM_PLAN_MAX": "8192"},  # 4097..8192 requests on the 12 x 3 x 3072 shared-memory plan
           "plankernels": {"DDS_SMEM_PLAN": "0"},       # every variable-count put planned by dds_plan_kernel<true>
           "minseg1": {"DDS_VAR_MINSEG": "1", "DDS_S_MINSEG": "1"},
           "nopdl": {"DDS_PDL": "0"}}


# ------------------------------------------------------------------------------------------------ helpers
def dev_bytes(torch, ptr, n, device="cuda:0"):
    """n bytes of device memory at ptr, copied to the host"""
    from ddstore_b200.store import _DevMem
    torch.cuda.synchronize(device)
    return torch.as_tensor(_DevMem(ptr, n), device=device).cpu().numpy().copy() if n else np.zeros(0, np.uint8)


def shard_state(torch, store, name, payload, device="cuda:0"):
    """the local shard's rows and its slack (the 16 bytes every shard keeps past its rows, up to the 256-byte
    allocation granule)"""
    slack = ((payload + 16 + 255) // 256) * 256 - payload
    return dev_bytes(torch, store.query(name)["local_base"], payload + slack, device), slack


def to_device(torch, data, off, device="cuda:0"):
    """a device copy of the bytes `data` starting `off` bytes past a 16-byte boundary; returns (keepalive, pointer)"""
    buf = torch.empty(off + data.size + 16, dtype=torch.uint8, device=device)
    if data.size:
        buf[off:off + data.size].copy_(torch.from_numpy(data))
    torch.cuda.synchronize(device)
    return buf, buf.data_ptr() + off


def _index(x):
    """(keepalive, pointer, length, IDX_ON_DEVICE or 0) of an index array: a CUDA int64 tensor as it is, anything else as
    a host int64 array"""
    from ddstore_b200 import _capi
    if hasattr(x, "data_ptr"):
        return x, x.data_ptr(), x.numel(), _capi.IDX_ON_DEVICE
    a = np.ascontiguousarray(x, np.int64)
    return a, a.ctypes.data, a.size, 0


def raw_put(store, name, itemsize, src_ptr, src_bytes, starts=None, counts=None, fixed=1, ids=None, flags=0,
            stream=None):
    """the C-ABI entry itself (any itemsize; src at any byte address; host index arrays, or CUDA int64 tensors)
    -> (rc, total, bad)"""
    from ddstore_b200 import _capi
    L, total, bad = store._L, C.c_int64(0), C.c_int64(-1)
    fl = _capi.SRC_ON_DEVICE | flags
    if ids is not None:
        keep, ip, n, dev = _index(ids)
        rc = L.dds_put_samples(store._h, name.encode(), ip, n, itemsize, src_ptr, src_bytes, fl | dev, stream,
                               C.byref(total), C.byref(bad))
    else:
        keep, sp, n, dev = _index(starts)
        keep2, cp = (None, None) if counts is None else _index(counts)[:2]
        rc = L.dds_put_batch(store._h, name.encode(), sp, cp, fixed, n, itemsize, src_ptr, src_bytes, fl | dev, stream,
                             C.byref(total), C.byref(bad))
    return rc, total.value, bad.value


def layout_src(pattern, R, rows, req):
    """the caller's src for requests `req`: request i's rows are the pattern's bytes at its destination (its slot is
    kept, zero-filled, when the request is invalid; 0 bytes when its count is out of range)"""
    parts = []
    for s, c, ok in req:
        n = c * R if ok and 0 < c <= rows else 0
        if n and 0 <= s and s + c <= rows:
            parts.append(pattern[s * R:s * R + n])
        elif n:
            parts.append(np.zeros(n, np.uint8))
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


class World:
    """one rank on cuda:0 with variable `name`: random rows, a sample index, the pattern batches write"""

    def __init__(self, torch, store, name, itemsize, disp, nrows, seed, table=None):
        rng = np.random.default_rng(seed)
        self.R, self.rows, self.name, self.itemsize = itemsize * disp, nrows, name, itemsize
        self.payload = nrows * self.R
        self.shard = rng.integers(0, 256, size=self.payload, dtype=np.uint8)
        self.pattern = rng.integers(0, 256, size=self.payload, dtype=np.uint8)
        # (through the C-ABI: any itemsize, rows given as bytes)
        t = torch.from_numpy(self.shard).cuda()
        torch.cuda.synchronize()
        assert store._L.dds_add(store._h, name.encode(), t.data_ptr(), nrows, disp, itemsize, 1) == 0, store._L.dds_last_error()
        self.table = table
        if table is not None:
            store.set_sample_index(name, table[0], table[1])

    def reset(self, torch, store):
        """put the original rows back (so every check starts from the same shard)"""
        buf, ptr = to_device(torch, self.shard, 0)
        rc, total, bad = raw_put(store, self.name, self.itemsize, ptr, self.shard.size, starts=[0], fixed=self.rows)
        assert rc == 0 and total == self.shard.size

    def check(self, torch, store, what, src_off=0, src_bytes=None, **req):
        reqs = po.requests(**req)
        src = layout_src(self.pattern, self.R, self.rows, reqs)
        sb = src.size if src_bytes is None else src_bytes
        buf, ptr = to_device(torch, src, src_off)
        kw = dict(req)
        if "table" in kw:
            kw.pop("table")
            kw["ids"] = kw.pop("sample_ids")
        if "fixed_count" in kw:
            kw["fixed"] = kw.pop("fixed_count")
        rc, total, bad = raw_put(store, self.name, self.itemsize, ptr if src.size else None, sb, **kw)
        shard = np.ascontiguousarray(self.shard.reshape(self.rows, -1))
        new, codes, ebad, etotal = po.put([shard], src, src_bytes=sb, **req)
        ecode, ebad2 = po.expected_error(codes, ebad, etotal, sb)
        assert (rc, bad) == (ERR[ecode], ebad2), f"{what}: rc {rc} bad {bad}, oracle {ERR[ecode]} {ebad2}"
        assert total == etotal, f"{what}: total {total}, oracle {etotal}"
        got, slack = shard_state(torch, store, self.name, self.payload)
        exp = new[0].reshape(-1).view(np.uint8)
        d = np.nonzero(got[:self.payload] != exp)[0]
        assert d.size == 0, (f"{what}: {d.size} shard bytes differ, first at byte {int(d[0])} (row {int(d[0]) // self.R}): "
                             f"got {int(got[d[0]])}, expected {int(exp[d[0]])}")
        assert not got[self.payload:].any(), f"{what}: the shard's slack was written"
        self.reset(torch, store)
        return codes


def inject_invalid(rng, starts, counts, rows, where):
    """invalid requests at the given indices: in turn a start past the end and a count straddling the end (both keep
    their bytes in the layout), and a negative count (0 bytes)"""
    st, ct = starts.copy(), counts.copy()
    for k, i in enumerate(where):
        if i >= len(st):
            continue
        if k % 3 == 0:
            st[i] = rows + 3
        elif k % 3 == 1:
            st[i], ct[i] = rows - 1, 2
        else:
            ct[i] = -1
    return st, ct


# ------------------------------------------------------------------------------------------------ the sweep
SHAPES = {1: (1, 13 << 20), 2: (3, (13 << 20) // 6), 4: (5, (13 << 20) // 20), 8: (3, (13 << 20) // 24)}
DENSE_ROWS = 16400  # rows of the small second variable that the dense batches write completely


def put_sweep_main():
    import torch
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    cfg = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("DDS_")) or "default"
    for itemsize, (disp, nrows) in SHAPES.items():
        rng = np.random.default_rng(itemsize)
        R = itemsize * disp
        starts, counts = sweep_requests(rng, nrows, R, (4096, 3072))
        table = (starts.copy(), counts.copy())
        w = World(torch, store, f"v{itemsize}", itemsize, disp, nrows, itemsize, table)
        for off in SRC_OFFSETS:
            w.check(torch, store, f"[{cfg}] itemsize {itemsize} counts, src +{off}", src_off=off, starts=starts, counts=counts)
        ids = np.concatenate([np.arange(len(starts)), rng.integers(0, len(starts), size=64)])
        ids = rng.permutation(ids).astype(np.int64)
        w.check(torch, store, f"[{cfg}] itemsize {itemsize} sample ids", src_off=5, sample_ids=ids, table=table)
        fs = rng.integers(0, nrows - 40, size=300)
        for cnt in (1, 3, 40):
            w.check(torch, store, f"[{cfg}] itemsize {itemsize} fixed {cnt}", src_off=3 * cnt % 16, starts=fs, fixed_count=cnt)
        # batch sizes on both sides of the shared-memory plan's thresholds (1024 by default, 4096, 8192)
        for n in (1024, 1025, 4096, 4097, 8192, 8193):
            s2, c2 = padded_requests(rng, nrows, starts, counts, n)
            w.check(torch, store, f"[{cfg}] itemsize {itemsize} n={n}", src_off=7, starts=s2, counts=c2)
        # invalid requests at the walk's lane edges, at the plan tiles' edges and at 1 % density; capacity errors
        s2, c2 = padded_requests(rng, nrows, starts, counts, 2100)
        edges = [0, 31, 32, 63, 1023, 1024, 2047, 2048]
        for where in (edges, sorted(rng.choice(2100, size=21, replace=False).tolist())):
            si, ci = inject_invalid(rng, s2, c2, nrows, where)
            codes = w.check(torch, store, f"[{cfg}] itemsize {itemsize} invalid {where[:4]}", src_off=1, starts=si, counts=ci)
            assert codes[where[0]] != 0
            total = sum(c * R if 0 < c <= nrows else 0 for c in ci.tolist())
            w.check(torch, store, f"[{cfg}] itemsize {itemsize} capacity + invalid", src_bytes=total - 1, starts=si, counts=ci)
            w.check(torch, store, f"[{cfg}] itemsize {itemsize} invalid ids", sample_ids=np.where(np.isin(np.arange(ids.size), where), -5, ids), table=table)
        w.check(torch, store, f"[{cfg}] itemsize {itemsize} capacity", src_bytes=int(counts.sum()) * R - 1, starts=starts, counts=counts)
        w.check(torch, store, f"[{cfg}] itemsize {itemsize} fixed capacity", src_bytes=300 * 3 * R - 1, starts=fs, fixed_count=3)
        # the dense form: each batch writes EVERY row of a small second variable exactly once, so every piece's
        # neighbours are written by other warps and CTAs of the same launch and a write wider than its piece is seen.
        # Batch sizes on both sides of the plan thresholds again: the placement decides who computes the shard addresses
        ds, dc = dense_cover(rng, DENSE_ROWS, 4097)
        d = World(torch, store, f"d{itemsize}", itemsize, disp, DENSE_ROWS, 100 + itemsize, (ds.copy(), dc.copy()))
        d.check(torch, store, f"[{cfg}] itemsize {itemsize} dense sample ids", src_off=9, sample_ids=rng.permutation(4097), table=d.table)
        for n in (1024, 1025, 4096, 4097, 8192, 8193):
            ds, dc = dense_cover(rng, DENSE_ROWS, n)
            d.check(torch, store, f"[{cfg}] itemsize {itemsize} dense n={n}", src_off=n % 16, starts=ds, counts=dc)
        for cnt in (1, 4):
            d.check(torch, store, f"[{cfg}] itemsize {itemsize} dense fixed {cnt}", src_off=5 * cnt,
                    starts=rng.permutation(DENSE_ROWS // cnt) * cnt, fixed_count=cnt)
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_put import put_sweep_main
put_sweep_main()
print("put-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_put_sweep(tmp_path, config):
    """raw itemsizes 1/2/4/8 over the variant sweep's request sizes, src at base offsets 0/1/4/8/13, every entry,
    batch sizes around the plan thresholds, invalid requests and capacity errors, and batches that write every row of
    a small variable exactly once, in the environment of `config`"""
    script = tmp_path / "put_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "put-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]


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


def test_put_above_4gib(torch, store):
    """layouts above 4 GiB (fixed and variable counts): the plan kernels' 64-bit offsets, rows repeated many times"""
    disp, nrows, cnt = 1024, 16384, 256  # 4 KiB rows, 1 MiB requests
    rng = np.random.default_rng(11)
    store.add("big", np.zeros((nrows, disp), np.float32))
    pat = torch.randint(-2**31, 2**31 - 1, (nrows, disp), dtype=torch.int32, device="cuda:0").view(torch.float32)
    n = (4 << 30) // (cnt * disp * 4) + 5
    starts = torch.from_numpy(rng.integers(0, nrows - cnt, size=n)).cuda()
    rows = (starts[:, None] + torch.arange(cnt, device="cuda:0")[None, :]).reshape(-1)
    src = pat[rows]
    torch.cuda.synchronize()
    covered = torch.zeros(nrows, dtype=torch.bool, device="cuda:0")
    covered[rows] = True
    for counts in (None, torch.full((n,), cnt, dtype=torch.int64, device="cuda:0")):
        torch.cuda.synchronize()
        total = store.put_batch("big", starts, counts, src=src, count=cnt)
        assert total == src.numel() * 4 > (4 << 30)
        shard = torch.as_tensor(_devmem(store.query("big")["local_base"], nrows * disp * 4), device="cuda:0")
        shard = shard.view(torch.float32).view(nrows, disp)
        assert torch.equal(shard[covered].view(torch.int32), pat[covered].view(torch.int32))
        assert not shard[~covered].view(torch.int32).any()
        shard[covered] = 0
        torch.cuda.synchronize()
    del src


def _devmem(ptr, n):
    from ddstore_b200.store import _DevMem
    return _DevMem(ptr, n)


def test_round_trip_through_every_get(torch, store):
    """after a put, get_batch, get_samples, a padded get_samples and a converting get of the same rows return it"""
    rng = np.random.default_rng(3)
    nrows, disp = 4000, 37
    store.add("x", np.zeros((nrows, disp), np.float32))
    rs = np.sort(rng.choice(nrows - 20, size=300, replace=False)).astype(np.int64)
    rc = rng.integers(1, 20, size=300).astype(np.int64)
    rc = np.minimum(rc, np.append(np.diff(rs), 20))  # disjoint samples
    store.set_sample_index("x", rs, rc)
    ids = rng.permutation(300).astype(np.int64)
    rows = np.concatenate([np.arange(rs[i], rs[i] + rc[i]) for i in ids])
    vals, ids_dev = torch.randn(rows.size, disp, device="cuda:0"), torch.from_numpy(ids).cuda()
    torch.cuda.synchronize()
    assert store.put_samples("x", ids_dev, vals) == vals.numel() * 4
    out = torch.empty_like(vals)
    store.get_batch("x", rs[ids], rc[ids], out=out)
    assert torch.equal(out, vals)
    out.zero_()
    store.get_samples("x", ids, out)
    assert torch.equal(out, vals)
    M = int(rc.max())
    pad = torch.empty(300, M, disp, device="cuda:0")
    lengths = torch.empty(300, dtype=torch.int64, device="cuda:0")
    store.get_samples("x", ids, pad, pad_rows=M, pad_value=-7.0, lengths=lengths)
    exp = torch.full((300, M, disp), -7.0, device="cuda:0")
    o = 0
    for j, i in enumerate(ids.tolist()):
        exp[j, :rc[i]] = vals[o:o + rc[i]]
        o += int(rc[i])
    assert torch.equal(pad, exp) and lengths.cpu().numpy().tolist() == rc[ids].tolist()
    bf = torch.empty(rows.size, disp, dtype=torch.bfloat16, device="cuda:0")
    store.get_batch("x", rs[ids], rc[ids], out=bf, src_dtype="float32")
    assert torch.equal(bf, vals.to(torch.bfloat16))


def test_ordering_in_one_stream(torch, store):
    """put -> get -> put queued on one stream: the get sees the first put, not the second; an overlapped get run, a
    put, an overlapped get run: every batch right, the get after the put sees it"""
    nrows, disp = 2048, 256
    store.add("o", np.zeros((nrows, disp), np.float32))
    st = torch.cuda.Stream()
    starts = torch.arange(0, nrows, 2, device="cuda:0")
    a = torch.full((starts.numel(), disp), 1.0, device="cuda:0")
    b = torch.full((starts.numel(), disp), 2.0, device="cuda:0")
    got = torch.zeros_like(a)
    torch.cuda.synchronize()
    h = st.cuda_stream
    store.put_batch("o", starts, src=a, stream=h, wait=False)
    store.get_batch("o", starts, out=got, stream=h, wait=False)
    store.put_batch("o", starts, src=b, stream=h, wait=False)
    assert store.wait() == b.numel() * 4
    assert torch.equal(got, a)
    outs = [torch.zeros_like(a) for _ in range(6)]
    torch.cuda.synchronize()
    for k in range(3):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.put_batch("o", starts, src=a, stream=h, wait=False)
    for k in range(3, 6):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.wait()
    for k in range(6):
        assert torch.equal(outs[k], b if k < 3 else a), k


def test_queue_endings_and_epoch_begin(torch, store):
    """wait() reports the first failing put with its index; a synchronous call, epoch_end and free complete a pending
    put queue and keep its error; epoch_begin completes a pending put queue and leaves a queue of gets as it is"""
    nrows, disp = 1000, 16
    store.add("q", np.zeros((nrows, disp), np.int32))
    st = torch.cuda.Stream()
    h = st.cuda_stream
    good = torch.arange(0, 500, device="cuda:0")
    bad = good.clone()
    bad[7] = nrows + 1
    src = torch.ones(500, disp, dtype=torch.int32, device="cuda:0")
    src3, src5, src9 = src * 3, src[:10] * 5, src * 9
    torch.cuda.synchronize()
    store.put_batch("q", good, src=src, stream=h, wait=False)
    store.put_batch("q", bad, src=src, stream=h, wait=False)
    with pytest.raises(ValueError, match="Invalid count on target"):
        store.wait()
    assert store.last_bad_index == 7
    for ending in ("sync", "epoch_end", "epoch_begin"):
        if ending == "epoch_end":
            store.epoch_begin()
        store.put_batch("q", bad, src=src3, stream=h, wait=False)
        if ending == "sync":
            store.put_batch("q", good[:10], src=src5)  # its own outcome: ok
        else:
            getattr(store, ending)()
        # the queue was completed: its rows are in place before anything else synchronises
        row = torch.as_tensor(_devmem(store.query("q")["local_base"] + 20 * disp * 4, disp * 4), device="cuda:0")
        assert row.view(torch.int32).eq(3).all(), ending
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.wait()
        assert store.last_bad_index == 7
        if ending == "epoch_begin":
            store.epoch_end()
    # a queue of gets at epoch_begin: reported by wait() as before
    out = torch.zeros(500, disp, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    store.get_batch("q", bad, out=out, stream=h, wait=False)
    store.epoch_begin()
    with pytest.raises(ValueError, match="Invalid count on target"):
        store.wait()
    assert store.last_bad_index == 7
    store.epoch_end()
    # free() completes a pending put queue (and drops nothing it has not reported: checked by the next wait)
    store.put_batch("q", good, src=src9, stream=h, wait=False)
    store.free()
    assert store.wait() == src.numel() * 4


def test_duplicates_leave_one_writers_bytes(torch, store):
    nrows, disp = 64, 1000
    store.add("d", np.zeros((nrows, disp), np.uint8))
    a = torch.randint(0, 256, (2, disp), dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    store.put_batch("d", [5, 5], src=a)
    got = torch.as_tensor(_devmem(store.query("d")["local_base"] + 5 * disp, disp), device="cuda:0")
    assert ((got == a[0]) | (got == a[1])).all()


def test_errors(torch, store):
    store.add("e", np.zeros((10, 4), np.float32))
    src = torch.zeros(2, 4, device="cuda:0")
    with pytest.raises(KeyError):
        store.put_batch("nope", [0, 1], src=src)
    with pytest.raises(ValueError, match="device memory"):
        store.put_batch("e", [0, 1], src=np.zeros((2, 4), np.float32))
    with pytest.raises(ValueError, match="Invalid data type"):
        store.put_batch("e", [0, 1], src=src.double())
    with pytest.raises(ValueError, match="no sample index"):
        store.put_samples("e", [0], src=src)
    assert store.put_batch("e", np.zeros(0, np.int64), src=src) == 0
    # the C-ABI's own argument checks
    rc, _, _ = raw_put(store, "e", 4, src.data_ptr(), 32, starts=[0], flags=0)  # (raw_put always sets SRC_ON_DEVICE)
    assert rc == 0
    from ddstore_b200 import _capi
    total, bad = C.c_int64(0), C.c_int64(0)
    sa = np.zeros(1, np.int64)
    assert store._L.dds_put_batch(store._h, b"e", sa.ctypes.data, None, 1, 1, 4, src.data_ptr(), 32, 0, None,
                                  C.byref(total), C.byref(bad)) == _capi.ERR_ARG  # host src
    assert store._L.dds_put_batch(store._h, b"e", sa.ctypes.data, None, 1, 1, 4, None, 32, _capi.SRC_ON_DEVICE, None,
                                  C.byref(total), C.byref(bad)) == _capi.ERR_ARG  # null src
    assert store._L.dds_put_batch(store._h, b"e", sa.ctypes.data, None, 1, -1, 4, src.data_ptr(), 32,
                                  _capi.SRC_ON_DEVICE, None, C.byref(total), C.byref(bad)) == _capi.ERR_ARG


def test_cython_binding(torch):
    """the C++ class (include/ddstore_b200.hpp) through the Cython binding: one put, one error"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    s = pyd.PyDDStore(None, device=0)
    s.add("c", np.zeros((8, 3), np.float32))
    src = torch.arange(6, dtype=torch.float32, device="cuda:0").reshape(2, 3)
    torch.cuda.synchronize()
    assert s.put_batch("c", np.array([1, 6], np.int64), src=src) == 24
    got = np.zeros((2, 3), np.float32)
    s.get("c", got, 6)
    assert got[0].tobytes() == src[1].cpu().numpy().tobytes() and not got[1].any()
    with pytest.raises(ValueError, match="Invalid start on target"):
        s.put_batch("c", np.array([-1], np.int64), src=src[:1])
    s.free()


# ------------------------------------------------------------------------------------------------ other ranks
def _ranks_body(torch, P, N, disp, doorbell_first):
    def body(store, r):
        import torch as t
        dev = t.device("cuda", t.cuda.current_device())
        base = np.arange(P * N * disp, dtype=np.float32).reshape(P * N, disp)
        store.add("w", base[r * N:(r + 1) * N].copy())
        # global row g of rank t's rows (local i) is written by rank (t + 1 + i % 2) % P -- never by its owner
        mine = np.array([g for g in range(P * N) if g // N != r and ((g // N) + 1 + (g % N) % 2) % P == r], np.int64)
        final = -base
        old = np.zeros((1, disp), np.float32)
        if doorbell_first:  # a resident doorbell CTA reads a row another rank writes later (a stale L1 line would show)
            store.get("w", old, int(((r + 1) % P) * N))
            assert old.tobytes() == base[((r + 1) % P) * N:((r + 1) % P) * N + 1].tobytes()
        store.epoch_begin()
        src, idx = t.from_numpy(final[mine]).to(dev), t.from_numpy(mine).to(dev)
        t.cuda.synchronize(dev)
        assert store.put_batch("w", idx, src=src) == src.numel() * 4
        store.epoch_end()
        exp = base.copy()
        for g in range(P * N):
            if ((g // N) + 1 + (g % N) % 2) % P != g // N:
                exp[g] = final[g]
        out = t.zeros(P * N, disp, device=dev)
        t.cuda.synchronize(dev)
        store.get_batch("w", np.arange(P * N), out=out)
        assert np.array_equal(out.cpu().numpy(), exp)
        store.set_sample_index("w", np.arange(P * N, dtype=np.int64), np.ones(P * N, np.int64))
        out.zero_()
        t.cuda.synchronize(dev)
        store.get_samples("w", np.arange(P * N)[::-1].copy(), out)
        assert np.array_equal(out.cpu().numpy(), exp[::-1])
        one = np.zeros((1, disp), np.float32)
        for g in (((r + 1) % P) * N, ((r + 2) % P) * N + 1, r * N):
            store.get("w", one, g)
            assert one.tobytes() == exp[g:g + 1].tobytes(), g
        return True
    return body


@pytest.mark.parametrize("doorbell", [True, False])
def test_three_owner_world(torch, monkeypatch, doorbell):
    """three thread-ranks on device 0: every rank puts into the others' rows, crosses a fence, reads them back through
    get_batch, get_samples and get() (doorbell kernel, and DDS_DOORBELL=0)"""
    monkeypatch.setenv("DDS_DOORBELL", "1" if doorbell else "0")
    monkeypatch.setenv("DDS_DOORBELL_IDLE_US", "5000000")  # the doorbell CTA stays resident across the fence
    assert all(run_world(3, _ranks_body(torch, 3, 40, 33, doorbell)))


def test_one_gpu_per_rank(torch):
    """the same across GPUs (peer-mapped shards over NVLink), one thread-rank per GPU"""
    P = torch.cuda.device_count()
    if P < 2:
        pytest.skip("needs two or more GPUs")
    assert all(run_world(P, _ranks_body(torch, P, 64, 257, True), devices=list(range(P))))
