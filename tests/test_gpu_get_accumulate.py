"""Batched fetch-ops (dds_get_accumulate_batch / dds_get_accumulate_samples) on the GPU against the NumPy oracle of
tests/fop_oracle.py.

Every check compares the WHOLE local shard -- every row, and the zero slack past the last row -- and the whole result
buffer, inside sentinel guard bands, with the oracle: elements one call touches once exactly, elements several
fetch-ops touch by their chain. Data are small integers (positive for sums that meet duplicates, distinct for swaps
that do), so every sum is exact in every type. The sweep runs in subprocesses, one per configuration (plan placement,
segment size, PDL), as the put's and the accumulate's do.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import fop_oracle as fo
from tests import put_oracle as po
from tests import put_world as pw
from tests.gpu_helpers import padded_requests, run_world, sweep_requests
from tests.put_world import dense_cover
from tests.test_gpu_accumulate import _index, _shard, add_var
from tests.test_gpu_put import CONFIGS, ERR, inject_invalid, shard_state

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = (ao.ACC_F32, ao.ACC_F64, ao.ACC_I32, ao.ACC_I64, ao.ACC_F16, ao.ACC_BF16)
E = {t: np.dtype(ao.STORAGE[t]).itemsize for t in ALL}
GUARD = 64  # sentinel bytes on either side of a result buffer


# ------------------------------------------------------------------------------------------------ helpers
def raw_fop(torch, store, name, op, t, src_ptr, res_ptr, src_bytes, starts=None, counts=None, fixed=1, ids=None,
            dev=False, flags=0, stream=None, device="cuda:0", keep=None):
    """the C-ABI entry itself -> (rc, total, bad); `keep` (a list) receives the index arrays"""
    from ddstore_b200 import _capi
    L, total, bad = store._L, C.c_int64(0), C.c_int64(-1)
    fl = _capi.SRC_ON_DEVICE | flags
    if ids is not None:
        keep_i, ip, n, d = _index(torch, ids, dev, device)
        rc = L.dds_get_accumulate_samples(store._h, name.encode(), ip, n, op, t, src_ptr, res_ptr, src_bytes, fl | d,
                                          stream, C.byref(total), C.byref(bad))
        held = (keep_i,)
    else:
        keep_i, sp, n, d = _index(torch, starts, dev, device)
        keep2, cp = (None, None) if counts is None else _index(torch, counts, dev, device)[:2]
        rc = L.dds_get_accumulate_batch(store._h, name.encode(), sp, cp, fixed, n, op, t, src_ptr, res_ptr, src_bytes,
                                        fl | d, stream, C.byref(total), C.byref(bad))
        held = (keep_i, keep2)
    if keep is not None:
        keep.append(held)
    return rc, total.value, bad.value


class Buffers:
    """device src and result buffers: src `src_off` bytes past a 16-byte boundary, result `res_off` bytes past one
    inside GUARD sentinel bytes (or the src itself: in_place)"""

    def __init__(self, torch, rng, src, src_off, res_off, in_place=False, device="cuda:0", before=None):
        self.n = src.size
        self.src_dev = torch.empty(src_off + src.size + 16, dtype=torch.uint8, device=device)
        if src.size:
            self.src_dev[src_off:src_off + src.size].copy_(torch.from_numpy(src))
        self.src_ptr = self.src_dev.data_ptr() + src_off
        self.in_place = in_place
        if in_place:
            self.before = src.copy()
            self.res_ptr, self.whole_off = self.src_ptr, src_off
        else:
            self.before = result_sentinel(rng, src.size, res_off) if before is None else before
            self.res_dev = torch.from_numpy(self.before).to(device)
            self.res_ptr = self.res_dev.data_ptr() + GUARD + res_off
            self.lo = GUARD + res_off
            self.before_res = self.before[self.lo:self.lo + src.size]
        torch.cuda.synchronize(device)

    def result0(self):
        return self.before if self.in_place else self.before_res

    def read(self, torch, device="cuda:0"):
        """(result bytes, None or a message about the guard bands)"""
        torch.cuda.synchronize(device)
        if self.in_place:
            whole = self.src_dev.cpu().numpy()
            return whole[self.whole_off:self.whole_off + self.n], None
        whole = self.res_dev.cpu().numpy()
        g = np.concatenate([whole[:self.lo], whole[self.lo + self.n:]])
        e = np.concatenate([self.before[:self.lo], self.before[self.lo + self.n:]])
        return whole[self.lo:self.lo + self.n], (None if np.array_equal(g, e) else "a guard band around result changed")


def result_sentinel(rng, n, res_off):
    """the bytes of a result buffer before the call: random, GUARD + res_off + n + GUARD of them"""
    return rng.integers(0, 256, size=GUARD + res_off + n + GUARD, dtype=np.uint8)


def operands(rng, t, op, n, base=0):
    """n operands: for sums small positive integers (chains need them); for swaps distinct bit patterns (base + k),
    none of them a shard's starting value (integers in [-8, 8)): 16-bit types take patterns 1 .. 15000, all below 1.0,
    the others the integers 1000 + base + k"""
    if op == fo.OP_SUM:
        return ao.encode(rng.integers(1, 4, size=n), t)
    if E[t] == 2:
        return ao.from_bits(1 + (base + np.arange(n)) % 15000, t)
    return ao.encode(1000 + base + np.arange(n), t)


def layout_src(rng, lenlist, disp, t, op, batch, base=0):
    """operands for every element of `batch`'s layout -> uint8 array"""
    rows = int(lenlist[-1])
    n = sum(c * disp for _, c, ok in po.requests(**batch) if ok and 0 < c <= rows)
    return operands(rng, t, op, n, base).view(np.uint8)


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
        buf = torch.from_numpy(self.shard.view(np.uint8).reshape(-1).copy()).cuda()
        torch.cuda.synchronize()
        total, bad = C.c_int64(0), C.c_int64(-1)
        sa = np.zeros(1, np.int64)
        rc = store._L.dds_put_batch(store._h, self.name.encode(), sa.ctypes.data, None, self.rows, 1, E[self.t],
                                    buf.data_ptr(), self.payload, _capi.SRC_ON_DEVICE, None, C.byref(total), C.byref(bad))
        assert rc == 0 and total.value == self.payload

    def check(self, torch, store, what, op, src_off=0, res_off=0, in_place=False, src_bytes=None, dev=False, **req):
        """one fetch-op of `req`; compare status, total, the whole shard and the whole result with the oracle; restore
        the shard"""
        t = self.t
        ll = po.lenlist_of([self.shard])
        src = layout_src(self.rng, ll, self.disp, t, op, req)
        sb = src.size if src_bytes is None else src_bytes
        b = Buffers(torch, self.rng, src, src_off, res_off, in_place)
        kw = dict(req)
        if "table" in kw:
            kw.pop("table")
            kw["ids"] = kw.pop("sample_ids")
        if "fixed_count" in kw:
            kw["fixed"] = kw.pop("fixed_count")
        rc, total, bad = raw_fop(torch, store, self.name, op, t, b.src_ptr if src.size else None,
                                 b.res_ptr if src.size else None, sb, dev=dev, **kw)
        _, _, codes, ebad, etotal = fo.fetch_op([self.shard], src, t, op, b.result0(), src_bytes=sb, **req)
        ecode, ebad2 = po.expected_error(codes, ebad, etotal, sb)
        assert (rc, bad) == (ERR[ecode], ebad2), f"{what}: rc {rc} bad {bad}, oracle {ERR[ecode]} {ebad2}"
        assert total == etotal, f"{what}: total {total}, oracle {etotal}"
        got, slack = shard_state(torch, store, self.name, self.payload)
        res, guard = b.read(torch)
        assert guard is None, f"{what}: {guard}"
        assert not got[self.payload:].any(), f"{what}: the shard's slack was written"
        gs = got[:self.payload].copy().view(ao.STORAGE[t]).reshape(self.rows, self.disp)
        msg = fo.check([self.shard], [(src, sb, b.result0(), req)], t, op, [gs], [res])
        assert msg is None, f"{what}: {msg}"
        self.reset(torch, store)
        return codes


# ------------------------------------------------------------------------------------------------ the sweep
from tests.test_gpu_accumulate import SHAPES  # noqa: E402  (the accumulate sweep's shapes: ~13 MiB per type)
BIG_DISP = 65543  # the largest rows: 65543 elements
DENSE_ROWS = 16400


def fop_sweep_main():
    import torch
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    cfg = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("DDS_")) or "default"
    full = cfg == "default"  # (the other configurations change the walk and the plan only: one op per type)
    for t in ALL:
        for op in (fo.OP_SUM, fo.OP_REPLACE) if full else ((fo.OP_SUM, fo.OP_REPLACE)[t % 2],):
            rng = np.random.default_rng([t, op])
            disp, nrows = SHAPES[t]
            tn = f"{ao.NAMES[t]} {'sum' if op == fo.OP_SUM else 'replace'}"
            starts, counts = sweep_requests(rng, nrows, E[t] * disp, (4096, 3072))
            # (the requests of 3 and 5 MiB go: every size up to the largest segment, 1 MiB + 1, stays)
            small = counts * E[t] * disp <= (1 << 20) + E[t] * disp
            starts, counts = starts[small], counts[small]
            table = (starts.copy(), counts.copy())
            w = World(torch, store, f"v{t}{op}", t, disp, nrows, t, table)
            # src and result at element-aligned phases of a 16-byte block (same, different), and in place
            offs = [(0, 0), (E[t], 16 - E[t]), (16 - E[t], 0)] if full else [(E[t], 16 - E[t])]
            for k, (so, ro) in enumerate(offs):
                w.check(torch, store, f"[{cfg}] {tn} counts, src +{so} result +{ro}", op, src_off=so, res_off=ro,
                        dev=k % 2 == 1, starts=starts, counts=counts)
            if full:
                w.check(torch, store, f"[{cfg}] {tn} in place", op, src_off=E[t], in_place=True, dev=True,
                        starts=starts, counts=counts)
            # sample ids with duplicates: sums form chains; swaps too, with distinct operands
            ids = np.concatenate([np.arange(len(starts)), rng.integers(0, len(starts), size=64)])
            ids = rng.permutation(ids).astype(np.int64)
            for dev in (False, True) if full else (True,):
                w.check(torch, store, f"[{cfg}] {tn} sample ids dev={dev}", op, src_off=(8 if dev else 0) % 16,
                        res_off=E[t] if dev else 0, dev=dev, sample_ids=ids, table=table)
            fs = rng.integers(0, nrows - 40, size=300)
            for cnt in (1, 3, 40):
                w.check(torch, store, f"[{cfg}] {tn} fixed {cnt}", op, src_off=(E[t] * cnt) % 16, dev=cnt != 3,
                        starts=fs, fixed_count=cnt)
            for n in (1024, 1025, 4096, 4097, 8192, 8193):  # both sides of the plan thresholds
                s2, c2 = padded_requests(rng, nrows, starts, counts, n)
                w.check(torch, store, f"[{cfg}] {tn} n={n}", op, src_off=(E[t] * n) % 16, res_off=(E[t] * 3) % 16,
                        dev=n % 2 == 0, starts=s2, counts=c2)
            # invalid requests at lane and tile edges and at 1 % density; capacity errors
            s2, c2 = padded_requests(rng, nrows, starts, counts, 2100)
            for where in ([0, 31, 32, 63, 1023, 1024, 2047, 2048], sorted(rng.choice(2100, size=21, replace=False).tolist())):
                si, ci = inject_invalid(rng, s2, c2, nrows, where)
                codes = w.check(torch, store, f"[{cfg}] {tn} invalid {where[:4]}", op, src_off=E[t], res_off=E[t],
                                starts=si, counts=ci)
                assert codes[where[0]] != 0
                total = sum(c * w.R if 0 < c <= nrows else 0 for c in ci.tolist())
                w.check(torch, store, f"[{cfg}] {tn} capacity + invalid", op, src_bytes=total - 1, starts=si, counts=ci)
                w.check(torch, store, f"[{cfg}] {tn} invalid ids", op, dev=True,
                        sample_ids=np.where(np.isin(np.arange(ids.size), where), -5, ids), table=table)
            w.check(torch, store, f"[{cfg}] {tn} capacity", op, src_bytes=int(counts.sum()) * w.R - 1, starts=starts,
                    counts=counts)
            # every row of a small variable once per batch: each piece's neighbours (for 2-byte elements: the other
            # half of a 32-bit word) belong to other warps' requests
            ds, dc = dense_cover(rng, DENSE_ROWS, 4097)
            d = World(torch, store, f"d{t}{op}", t, disp, DENSE_ROWS, 100 + t, (ds.copy(), dc.copy()))
            d.check(torch, store, f"[{cfg}] {tn} dense sample ids", op, src_off=E[t] * 3 % 16, dev=True,
                    sample_ids=rng.permutation(4097), table=d.table)
            for n in (1025, 8193):
                ds, dc = dense_cover(rng, DENSE_ROWS, n)
                d.check(torch, store, f"[{cfg}] {tn} dense n={n}", op, src_off=(E[t] * n) % 16, starts=ds, counts=dc)
            d.check(torch, store, f"[{cfg}] {tn} dense fixed 1", op, src_off=E[t], res_off=16 - E[t], dev=True,
                    starts=rng.permutation(DENSE_ROWS), fixed_count=1)
            if full:  # rows of 65543 elements, cut at chunk boundaries
                b = World(torch, store, f"b{t}{op}", t, BIG_DISP, 24, 200 + t)
                bs = np.array([0, 23, 5, 11, 0], np.int64)
                bc = np.array([2, 1, 3, 13, 0], np.int64)
                for so, ro in ((0, 0), (E[t], 0), (16 - E[t], E[t])):
                    b.check(torch, store, f"[{cfg}] {tn} 65543-element rows, src +{so} result +{ro}", op, src_off=so,
                            res_off=ro, dev=so > 0, starts=bs, counts=bc)
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_get_accumulate import fop_sweep_main
fop_sweep_main()
print("fop-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_get_accumulate_sweep(tmp_path, config):
    """both ops and every element type over the variant sweep's request sizes; src, result and in-place at different
    16-byte phases; both entries with host and device indices; batch sizes around the plan thresholds; duplicates;
    invalid requests; capacity errors; dense batches and 65543-element rows, in the environment of `config`"""
    script = tmp_path / "fop_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "fop-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]


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


@pytest.mark.parametrize("src_off", [0, 4])
@pytest.mark.parametrize("dtype", ["int32", "int64"])
def test_tickets_one_batch(torch, store, dtype, src_off):
    """65536 +1 fetch-adds of ONE element in one batch, by start row and by sample id: the tickets are exactly
    v0 .. v0 + 65535, each once"""
    dt = getattr(torch, dtype)
    n = 65536
    store.add("k", np.full((64, 1), 7, np.int32 if dtype == "int32" else np.int64))
    store.set_sample_index("k", np.arange(64, dtype=np.int64), np.ones(64, np.int64))
    es = torch.tensor([], dtype=dt).element_size()
    buf = torch.ones(n + 4, dtype=dt, device="cuda:0")
    src = buf[src_off // es:src_off // es + n] if src_off % es == 0 else buf[:n]
    out = torch.zeros(n, dtype=dt, device="cuda:0")
    idx = torch.full((n,), 17, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    assert store.get_accumulate_batch("k", idx, src=src, out=out) == n * es
    assert torch.equal(out.sort().values, torch.arange(7, 7 + n, dtype=dt, device="cuda:0"))
    assert store.get_accumulate_samples("k", idx, src, out) == n * es
    assert torch.equal(out.sort().values, torch.arange(7 + n, 7 + 2 * n, dtype=dt, device="cuda:0"))
    sh = _shard(torch, store, "k", 64, 1, dt)
    assert sh[17].item() == 7 + 2 * n and sh[:17].eq(7).all() and sh[18:].eq(7).all()


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_float_chains_one_row(torch, store, dtype):
    """4096 fetch-adds of integer-valued rows into ONE 1024-element row (vector atomics, src re-phased or not): every
    element's chain is exact"""
    dt = getattr(torch, dtype)
    n, disp = 4096, 1024
    store.add("f", np.zeros((8, disp), np.float32 if dtype == "float32" else np.float64))
    rng = np.random.default_rng(1)
    for src_off in (0, 1):
        vals = torch.from_numpy(rng.integers(1, 4, size=(n, disp)).astype(np.float64)).to(dt).cuda()
        buf = torch.zeros(n * disp + 1, dtype=dt, device="cuda:0")
        buf[src_off:src_off + n * disp] = vals.reshape(-1)
        out = torch.zeros(n, disp, dtype=dt, device="cuda:0")
        v0 = _shard(torch, store, "f", 8, disp, dt)[3].clone()
        torch.cuda.synchronize()
        store.get_accumulate_batch("f", torch.full((n,), 3, dtype=torch.int64, device="cuda:0"),
                                   src=buf[src_off:src_off + n * disp], out=out)
        final = _shard(torch, store, "f", 8, disp, dt)[3]
        # per column: sorted by what each got, the running sums of the contributions from v0
        got, order = out.double().sort(dim=0)
        contrib = vals.double().gather(0, order)
        exp = v0.double() + torch.cumsum(contrib, 0) - contrib
        assert torch.equal(got, exp), src_off
        assert torch.equal(final.double(), v0.double() + vals.double().sum(0))


@pytest.mark.parametrize("t", [ao.ACC_F16, ao.ACC_BF16, ao.ACC_I32])
def test_neighbours_and_swap_chains_two_ranks(torch, t):
    """two thread-ranks in one epoch: rank 0 swaps every even row of the world, rank 1 fetch-adds into every odd row
    (for 2-byte elements the two halves of every 32-bit word: a compare-and-swap loop beside a returning add), and both
    swap 100 distinct values each into the hot rows 5 and 6 (one word). Every element ends exact, neighbours bit for
    bit, and each hot row's swaps form one chain"""
    P, N = 2, 2048
    tn = ao.NAMES[t]
    rng = np.random.default_rng(t)
    ev = np.arange(8, P * N, 2, dtype=np.int64)
    od = np.arange(9, P * N, 2, dtype=np.int64)
    x_ev = ao.encode(rng.integers(-8, 8, size=ev.size), t)
    x_od = ao.encode(rng.integers(1, 4, size=od.size), t)
    hot = [np.repeat(np.array([5, 6], np.int64), 100) for _ in range(P)]
    for hr in hot:
        rng.shuffle(hr)
    x_hot = [operands(rng, t, fo.OP_REPLACE, 200, 200 * r) for r in range(P)]

    def body(store, r):
        import torch as tt
        dev = tt.device("cuda", tt.cuda.current_device())
        dt = getattr(tt, tn)
        store._L.dds_init(store._h, b"n", N, 1, E[t])
        store.epoch_begin()
        keep = []  # (the operands of queued calls stay allocated until the fence has completed them)

        def go(idx, x, op):
            sd = tt.from_numpy(x.view(np.uint8).copy()).to(dev).view(dt)
            keep.append(sd)
            out = tt.full_like(sd.view({2: tt.int16, 4: tt.int32}[E[t]]), -1).view(dt)  # (no operand's bits)
            tt.cuda.synchronize(dev)
            keep.append(tt.from_numpy(idx).to(dev))
            store.get_accumulate_batch("n", keep[-1], src=sd, out=out, op=op, wait=False)
            return out
        outs = [go(hot[r], x_hot[r], "replace")]
        outs.append(go(ev, x_ev, "replace") if r == 0 else go(od, x_od, "sum"))
        store.epoch_end()
        def host(x):
            return x.cpu().view({2: tt.int16, 4: tt.int32}[E[t]]).numpy().view(ao.STORAGE[t]).reshape(-1)
        return [host(o) for o in outs], host(_shard(tt, store, "n", N, 1, dt))
    res = run_world(P, body)
    world = np.concatenate([res[0][1], res[1][1]])
    bits = lambda a: np.asarray(a).view(ao.BITS[t])  # noqa: E731
    zero = ao.encode(np.zeros(1), t)
    assert np.array_equal(bits(world[ev]), bits(x_ev)), f"{tn}: even rows"
    assert np.array_equal(bits(world[od]), bits(x_od)), f"{tn}: odd rows"
    assert (bits(res[0][0][1]) == bits(zero)[0]).all() and (bits(res[1][0][1]) == bits(zero)[0]).all()
    assert (bits(world[:5]) == bits(zero)[0]).all() and (bits(world[7]) == bits(zero)[0]).all()
    for row in (5, 6):
        srcs = [int(v) for r in range(P) for v in bits(x_hot[r][hot[r] == row])]
        got = [int(v) for r in range(P) for v in bits(res[r][0][0][hot[r] == row])]
        msg = fo.replace_chain(int(bits(zero)[0]), srcs, got, int(bits(world[row:row + 1])[0]))
        who = [(r, int(i)) for r in range(P) for i in np.flatnonzero(hot[r] == row)]
        assert msg is None, f"{tn} row {row}: {msg}; (rank, request) of each: {who}"


def test_fetch_adds_mixed_with_accumulates(torch, store):
    """+1 fetch-adds and +1 accumulates on the same elements in one epoch, queued on two streams: the final count is
    exact and the fetch-adds' tickets are distinct"""
    n, disp = 8192, 4
    store.add("m", np.zeros((16, disp), np.int64))
    idx = torch.full((n,), 9, dtype=torch.int64, device="cuda:0")
    one = torch.ones(n, disp, dtype=torch.int64, device="cuda:0")
    out = torch.zeros(2, n, disp, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    store.epoch_begin()
    store.accumulate_batch("m", idx, src=one, wait=False)
    store.get_accumulate_batch("m", idx, src=one, out=out[0], wait=False)
    store.accumulate_batch("m", idx, src=one, wait=False)
    store.get_accumulate_batch("m", idx, src=one, out=out[1], wait=False)
    store.epoch_end()
    sh = _shard(torch, store, "m", 16, disp, torch.int64)
    assert sh[9].eq(4 * n).all() and sh[:9].eq(0).all() and sh[10:].eq(0).all()
    t = out.permute(2, 0, 1).reshape(disp, -1).sort(dim=1).values
    assert (t[:, 1:] > t[:, :-1]).all() and t.min() >= 0 and t.max() < 4 * n


def test_hot_elements_four_ranks(torch):
    """every thread-rank of a 4-rank world fetch-adds +1 into the same element 8192 times in one epoch, and swaps a
    distinct value into another: 32768 distinct tickets v0 .. v0 + 32767, and one swap chain"""
    P, N, n = 4, 33, 8192

    def body(store, r):
        import torch as t
        dev = t.device("cuda", t.cuda.current_device())
        store._L.dds_init(store._h, b"c", N, 1, 8)
        store.epoch_begin()
        hot = t.full((n,), N + 5, dtype=t.int64, device=dev)       # rank 1's row 5
        swap = t.full((n,), 2 * N + 1, dtype=t.int64, device=dev)  # rank 2's row 1
        one = t.ones(n, dtype=t.int64, device=dev)
        mine = t.arange(n, dtype=t.int64, device=dev) + 1 + r * n   # distinct over the world
        out = t.zeros(n, dtype=t.int64, device=dev)
        out2 = t.zeros(n, dtype=t.int64, device=dev)
        t.cuda.synchronize(dev)
        store.get_accumulate_batch("c", hot, src=one, out=out)
        store.get_accumulate_batch("c", swap, src=mine, out=out2, op="replace", wait=False)
        store.epoch_end()
        sh = _shard(t, store, "c", N, 1, t.int64).cpu().numpy().reshape(-1)
        return out.cpu().numpy(), mine.cpu().numpy(), out2.cpu().numpy(), sh
    res = run_world(P, body)
    tickets = np.sort(np.concatenate([x[0] for x in res]))
    assert np.array_equal(tickets, np.arange(P * n))
    assert res[1][3][5] == P * n
    srcs = np.concatenate([x[1] for x in res]).tolist()
    got = np.concatenate([x[2] for x in res]).tolist()
    assert fo.replace_chain(0, srcs, got, int(res[2][3][1])) is None


def test_queue_endings(torch, store):
    """queued fetch-ops completed by wait(), a synchronous call, epoch_begin, epoch_end and free: every queued
    contribution is in place, each result holds what its batch saw, the first failure is reported once with its
    index"""
    nrows, disp = 1000, 16
    h = torch.cuda.Stream().cuda_stream
    good = torch.arange(0, 500, device="cuda:0")
    bad = good.clone()
    bad[7] = nrows + 1
    src = torch.ones(500, disp, dtype=torch.int32, device="cuda:0")
    for ending in ("wait", "sync", "epoch_begin", "epoch_end", "free"):
        store.add("q", np.zeros((nrows, disp), np.int32))
        sh = _shard(torch, store, "q", nrows, disp, torch.int32)
        outs = [torch.full((500, disp), -1, dtype=torch.int32, device="cuda:0") for _ in range(2)]
        torch.cuda.synchronize()
        if ending == "epoch_end":
            store.epoch_begin()
        store.get_accumulate_batch("q", bad, src=src, out=outs[0], stream=h, wait=False)
        store.get_accumulate_batch("q", good, src=src, out=outs[1], stream=h, wait=False)
        if ending == "wait":
            with pytest.raises(ValueError, match="Invalid count on target"):
                store.wait()
        elif ending == "sync":  # its own outcome: ok
            sync_out = torch.zeros(10, disp, dtype=torch.int32, device="cuda:0")
            assert store.get_accumulate_batch("q", good[:10], src=src[:10], out=sync_out) == 10 * disp * 4
            assert sync_out[7].eq(1).all() and sync_out[:7].eq(2).all() and sync_out[8:].eq(2).all()
        else:
            getattr(store, ending)()
        if ending != "free":
            rows = sh.clone()  # (nothing else synchronised the queue)
            assert rows[20].eq(2).all() and rows[7].eq(1 + (ending == "sync")).all() and not rows[500:].any(), ending
        o0, o1 = outs[0].cpu().numpy(), outs[1].cpu().numpy()
        assert (o0[7] == -1).all() and not o0[:7].any() and not o0[8:].any(), ending
        assert (o1[7] == 0).all() and (o1[:7] == 1).all() and (o1[8:] == 1).all(), ending
        if ending != "wait":
            with pytest.raises(ValueError, match="Invalid count on target"):
                store.wait()
        assert store.last_bad_index == 7
        if ending == "epoch_begin":
            store.epoch_end()
        if ending != "free":
            store.free()
    assert store.wait() == 0


def test_stream_ordering_with_overlapped_gets(torch, store):
    """an overlapped get run, a fetch-op, an overlapped get run, a swap, a get run on one stream: each get and each
    fetch-op sees exactly what was queued before it"""
    nrows, disp = 2048, 256
    store.add("o", np.zeros((nrows, disp), np.float32))
    h = torch.cuda.Stream().cuda_stream
    starts = torch.arange(0, nrows, 2, device="cuda:0")
    a = torch.full((starts.numel(), disp), 3.0, device="cuda:0")
    b = torch.full_like(a, 7.0)
    outs = [torch.zeros_like(a) for _ in range(9)]
    r1, r2 = torch.full_like(a, -1), torch.full_like(a, -1)
    torch.cuda.synchronize()
    for k in range(3):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.get_accumulate_batch("o", starts, src=a, out=r1, stream=h, wait=False)
    for k in range(3, 6):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.get_accumulate_batch("o", starts, src=b, out=r2, op="replace", stream=h, wait=False)
    for k in range(6, 9):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.wait()
    for k in range(9):
        assert outs[k].eq(0.0 if k < 3 else 3.0 if k < 6 else 7.0).all(), k
    assert r1.eq(0.0).all() and r2.eq(3.0).all()


def test_errors(torch, store):
    from ddstore_b200 import _capi
    store.add("e", np.zeros((10, 4), np.float32))
    src = torch.ones(2, 4, device="cuda:0")
    out = torch.zeros(2, 4, device="cuda:0")
    with pytest.raises(KeyError):
        store.get_accumulate_batch("nope", [0, 1], src=src, out=out)
    with pytest.raises(ValueError, match="Invalid data type"):
        store.get_accumulate_batch("e", [0, 1], src=src.double(), out=out.double())
    with pytest.raises(ValueError, match="is not one of"):
        store.get_accumulate_batch("e", [0, 1], src=src, out=out, op="max")
    with pytest.raises(ValueError, match="out holds"):
        store.get_accumulate_batch("e", [0, 1], src=src, out=out[:1])
    with pytest.raises(ValueError, match="no sample index"):
        store.get_accumulate_samples("e", [0], src, out)
    assert store.get_accumulate_batch("e", np.zeros(0, np.int64), src=src, out=out) == 0
    total, bad = C.c_int64(0), C.c_int64(0)
    sa = np.zeros(1, np.int64)

    def call(op, t, ptr, res, flags=_capi.SRC_ON_DEVICE, nreq=1):
        return store._L.dds_get_accumulate_batch(store._h, b"e", sa.ctypes.data, None, 1, nreq, op, t, ptr, res, 16,
                                                 flags, None, C.byref(total), C.byref(bad))
    p, q = src.data_ptr(), out.data_ptr()
    assert call(0, _capi.ACC_F32, p, q) == _capi.ERR_ARG and "fetch-op" in _capi.last_error()  # unknown op
    assert call(3, _capi.ACC_F32, p, q) == _capi.ERR_ARG
    assert call(1, 7, p, q) == _capi.ERR_ARG                                   # unknown dtype
    assert call(1, _capi.ACC_I64, p, q) == _capi.ERR_DTYPE                     # 8-byte type, 4-byte variable
    assert call(1, _capi.ACC_F32, p, None) == _capi.ERR_ARG and "null result" in _capi.last_error()
    assert call(1, _capi.ACC_F32, p, q + 2) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(1, _capi.ACC_F32, p + 2, q) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(1, _capi.ACC_F32, p, q, flags=0) == _capi.ERR_ARG              # host src
    assert call(1, _capi.ACC_F32, None, q) == _capi.ERR_ARG                    # null src
    assert call(1, _capi.ACC_F32, p, q, nreq=-1) == _capi.ERR_ARG
    assert call(1, _capi.ACC_F32, p, q, flags=_capi.SRC_ON_DEVICE | _capi.NO_SYNC) == _capi.ERR_ARG  # host indices
    assert not _shard(torch, store, "e", 10, 4, torch.float32).any() and not out.any()
    assert call(_capi.OP_SUM, _capi.ACC_I32, p, q) == 0  # the int32 sum of 1.0f's bits into zero bits
    assert out.view(torch.int32).eq(0).all() and _shard(torch, store, "e", 10, 4, torch.int32)[0].eq(0x3F800000).all()


def test_cython_and_cpp_bindings(torch, tmp_path):
    """get_accumulate_batch through the Cython binding, and DDStore::get_accumulate_batch<T> / the explicit-code
    overload / get_accumulate_samples through the C++ header"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    s = pyd.PyDDStore(None, device=0)
    s.add("c", np.ones((8, 3), np.float32))
    src = torch.arange(6, dtype=torch.float32, device="cuda:0").reshape(2, 3)
    out = torch.zeros(2, 3, device="cuda:0")
    torch.cuda.synchronize()
    assert s.get_accumulate_batch("c", np.array([1, 1], np.int64), src=src, out=out) == 24
    assert sorted(out[:, 0].tolist()) in ([1.0, 1.0], [1.0, 4.0])  # (the second fetch-op sees the first's sum)
    got = np.zeros((1, 3), np.float32)
    s.get("c", got, 1)
    assert got.tolist() == [[1 + 0 + 3, 1 + 1 + 4, 1 + 2 + 5]]
    assert s.get_accumulate_batch("c", np.array([4], np.int64), src=src[:1], out=out[:1], op="replace") == 12
    assert out[0].tolist() == [1.0, 1.0, 1.0]
    with pytest.raises(ValueError, match="Invalid start on target"):
        s.get_accumulate_batch("c", np.array([-1], np.int64), src=src[:1], out=out[:1])
    s.free()
    exe = build_cpp_check(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cpp get_accumulate ok" in r.stdout, r.stdout + r.stderr


CPP_CHECK = r"""
#include <cuda_runtime.h>
#include <cstdio>
#include "ddstore_b200.hpp"
int main() {
    DDStore s;
    std::vector<int64_t> k(4, 10);
    std::vector<uint16_t> h(4 * 2, 0x3f80);  // bf16 1.0
    s.add("k", k.data(), 4, 1);
    s.add("h", h.data(), 4, 2);
    const long starts[3] = {2, 2, 2};
    int64_t *dk, *rk; uint16_t *dh, *rh; long *ds;
    cudaMalloc(&dk, 24); cudaMalloc(&rk, 24); cudaMalloc(&dh, 4); cudaMalloc(&rh, 4); cudaMalloc(&ds, 24);
    int64_t hk[3] = {1, 1, 1};
    uint16_t hh[2] = {0x4000, 0x4040};  // 2, 3
    cudaMemcpy(dk, hk, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(dh, hh, 4, cudaMemcpyHostToDevice);
    cudaMemcpy(ds, starts, 24, cudaMemcpyHostToDevice);
    if (s.get_accumulate_batch<int64_t>("k", ds, nullptr, 1, 3, DDS_OP_SUM, dk, rk, 24) != 24) return 2;
    int64_t got[3];
    cudaMemcpy(got, rk, 24, cudaMemcpyDeviceToHost);
    if (got[0] + got[1] + got[2] != 10 + 11 + 12 || got[0] == got[1] || got[1] == got[2] || got[0] == got[2]) return 3;
    if (s.get_accumulate_batch("h", starts, nullptr, 1, 1, DDS_OP_REPLACE, DDS_ACC_BF16, dh, rh, 4, false) != 4) return 4;
    uint16_t gh[2];
    cudaMemcpy(gh, rh, 4, cudaMemcpyDeviceToHost);
    if (gh[0] != 0x3f80 || gh[1] != 0x3f80) return 5;
    if (s.get_accumulate_batch<int64_t>("k", ds, nullptr, 1, 1, DDS_OP_REPLACE, dk, rk, 8) != 8) return 6;
    cudaMemcpy(got, rk, 8, cudaMemcpyDeviceToHost);
    if (got[0] != 13) return 7;
    try { s.get_accumulate_batch<double>("h", starts, nullptr, 1, 1, DDS_OP_SUM, (const double *)dk, (double *)rk, 8, false); return 8; }
    catch (std::invalid_argument &e) { if (std::string(e.what()) != "Invalid data type") return 9; }
    s.get("k", 2, 1, k.data());
    s.get("h", 2, 1, h.data());
    if (k[0] != 1 || h[0] != 0x4000 || h[1] != 0x4040) return 10;
    s.free();
    printf("cpp get_accumulate ok\n");
    return 0;
}
"""


def build_cpp_check(tmp_path):
    src = tmp_path / "fop_check.cpp"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "fop_check")
    lib = os.path.join(ROOT, "ddstore_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
           "-L", lib, "-lddstore_b200", f"-Wl,-rpath,{lib}", "-L", "/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


# ------------------------------------------------------------------------------------------------ other ranks
ROWS = {2: [1, 23], 3: [19, 0, 8], 4: [0, 26, 1, 9]}


def fop_world(torch, P, nrows, t, op, disp, seed, devices=None, queued=False):
    """P thread-ranks; every rank fetch-ops into every other rank's rows (owner edges, straddlers and the invalid
    family, a by-sample-id form, a dense cover of the world, one call per rank short of source) in one epoch; after the
    closing fence every rank returns its shard and its calls' results and statuses, checked against the oracle's
    chains (every element is touched by several ranks)"""
    rng = np.random.default_rng([seed, P, t, op])
    ll = pw.lenlist_of(nrows)
    R = E[t] * disp
    shards = [ao.encode(rng.integers(-8, 8, size=(n, disp)), t) for n in nrows]
    total = int(ll[-1])
    tables, calls = [], []  # calls[r] = [(src bytes, src_bytes or None, batch, src offset)]
    cover = pw.interleaved_cover(rng, ll, P, R, big=R <= 64)
    ctr = [0]

    def world_src(batch):  # (swap operands distinct over the whole world)
        x = layout_src(rng, ll, disp, t, op, batch, ctr[0])
        ctr[0] += x.size // E[t]
        return x
    for r in range(P):
        others = [o[0] for o in pw.owners(ll) if o[0] != r] or None
        st, ct, cls = pw.edge_requests(rng, ll, r, first_bad=None if r == 0 else int(rng.integers(0, 6)), body=12,
                                       only=others)
        mine = []
        b = {"starts": st, "counts": ct}
        mine.append((world_src(b), None, b, E[t] * (r % (16 // E[t]))))
        sb, _ = pw.as_samples(rng, st, ct, cls, first_bad=None if r % 2 == 0 else 1)
        tables.append(sb["table"])
        mine.append((world_src(sb), None, sb, 0))
        cb = {"starts": cover[r][0], "counts": cover[r][1]}
        mine.append((world_src(cb), None, cb, E[t]))
        if r == P - 1 and total:
            fb = {"starts": np.array([0, total - 1], np.int64), "fixed_count": 1}
            full = world_src(fb)
            mine.append((full, full.size - 1, fb, 0))  # capacity: nothing applied
        calls.append(mine)
    exp_status = [[po.expected_error(*_codes_bad(shards, t, c), c[0].size if c[1] is None else c[1])
                   for c in mine] for mine in calls]
    res_off = [[(c[3] + E[t]) % 16 for c in mine] for mine in calls]
    befores = [[result_sentinel(rng, c[0].size, o) for c, o in zip(mine, offs)] for mine, offs in zip(calls, res_off)]

    def body(store, r):
        import torch as tt
        dev = tt.device("cuda", tt.cuda.current_device())
        problems = []
        mine = np.ascontiguousarray(shards[r]).view(np.uint8).reshape(-1)
        assert store._L.dds_add(store._h, b"w", mine.ctypes.data if mine.size else None, nrows[r], disp, E[t], 0) == 0
        store.set_sample_index("w", *tables[r])
        stream = tt.cuda.Stream(device=dev).cuda_stream if queued else None
        keep, bufs = [], []
        store.epoch_begin()
        for k, (src, sbytes, batch, off) in enumerate(calls[r]):
            b = Buffers(tt, None, src, off, res_off[r][k], device=dev, before=befores[r][k])
            bufs.append(b)
            sb = src.size if sbytes is None else sbytes
            kw = {"ids": batch["sample_ids"]} if "sample_ids" in batch else \
                {"starts": batch["starts"], "counts": batch.get("counts"), "fixed": batch.get("fixed_count", 1)}
            got = raw_fop(tt, store, "w", op, t, b.src_ptr if src.size else None, b.res_ptr if src.size else None, sb,
                          dev=queued or k % 2 == 1, flags=(4 if queued else 0), stream=stream, device=dev, keep=keep,
                          **kw)
            code, bad = exp_status[r][k]
            if queued:
                if got[0] != 0:
                    problems.append(f"rank {r} call {k}: queueing returned {got}")
            elif (got[0], got[2]) != (ERR[code], bad):
                problems.append(f"rank {r} call {k}: (rc, total, bad) = {got}, oracle {(ERR[code], bad)}")
        store.epoch_end()
        if queued:
            total_, bad_ = C.c_int64(0), C.c_int64(-1)
            rc = store._L.dds_batch_wait(store._h, C.byref(total_), C.byref(bad_))
            first = next(((c, b) for c, b in exp_status[r] if c), (0, -1))
            if (rc, bad_.value) != (ERR[first[0]], first[1]):
                problems.append(f"rank {r}: wait() -> {(rc, bad_.value)}, oracle {(ERR[first[0]], first[1])}")
        payload = nrows[r] * R
        got, slack = shard_state(tt, store, "w", payload, dev)
        if got[payload:].any():
            problems.append(f"rank {r}: slack written")
        results = []
        for b in bufs:
            res, guard = b.read(tt, dev)
            if guard:
                problems.append(f"rank {r}: {guard}")
            results.append(res.copy())
        return problems, got[:payload].copy(), results
    out = run_world(P, body, devices=devices)
    problems = [p for o in out for p in o[0]]
    assert not problems, "\n".join(problems[:12])
    got_shards = [o[1].view(ao.STORAGE[t]).reshape(n, disp) for o, n in zip(out, nrows)]
    flat = [(c[0], c[1], bf[GUARD + o:GUARD + o + c[0].size], c[2])
            for mine, offs, bfs in zip(calls, res_off, befores) for c, o, bf in zip(mine, offs, bfs)]
    got_res = [res for o in out for res in o[2]]
    msg = fo.check(shards, flat, t, op, got_shards, got_res)
    assert msg is None, f"P={P} {ao.NAMES[t]} op {op}: {msg}"


def _codes_bad(shards, t, c):
    codes, _pl, bad, total, _applied = fo.plan(shards, t, c[0].size if c[1] is None else c[1], **c[2])
    return codes, bad, total


@pytest.mark.parametrize("P", [2, 3, 4])
@pytest.mark.parametrize("t, op", [(ao.ACC_I32, fo.OP_SUM), (ao.ACC_F64, fo.OP_SUM), (ao.ACC_BF16, fo.OP_SUM),
                                   (ao.ACC_I32, fo.OP_REPLACE), (ao.ACC_F64, fo.OP_REPLACE)])
def test_multi_owner_worlds(torch, P, t, op):
    fop_world(torch, P, [n * 20 if n > 1 else n for n in ROWS[P]], t, op, {ao.ACC_I32: 3, ao.ACC_BF16: 7,
                                                                           ao.ACC_F64: 2}[t], seed=1)


def test_three_owner_world_queued(torch):
    fop_world(torch, 3, [380, 0, 160], ao.ACC_I64, fo.OP_SUM, 3, seed=2, queued=True)


def test_sixty_four_owners(torch):
    rng = np.random.default_rng(64)
    nrows = [0 if k % 3 == 0 else int(rng.integers(1, 6)) for k in range(64)]
    fop_world(torch, 64, nrows, ao.ACC_I32, fo.OP_REPLACE, 5, seed=3)


def test_one_gpu_per_rank(torch):
    """the same across GPUs: returning atomics into peer HBM over NVLink"""
    P = torch.cuda.device_count()
    if P < 2:
        pytest.skip("needs two or more GPUs")
    fop_world(torch, P, [37 * (k + 1) for k in range(P)], ao.ACC_F32, fo.OP_SUM, 1024, seed=4,
              devices=list(range(P)))
