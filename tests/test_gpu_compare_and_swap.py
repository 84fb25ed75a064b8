"""Batched compare-and-swaps (dds_compare_and_swap_batch / dds_compare_and_swap_samples) on the GPU against the NumPy
oracle of tests/cas_oracle.py.

Every check compares the WHOLE local shard -- every row, and the zero slack past the last row -- and the whole result
buffer, inside sentinel guard bands, with the oracle: elements one call touches once exactly, elements several
compare-and-swaps touch by one order that explains every result and the final value. Data are random bit patterns;
about half of the compare operands are the shard's own elements, so half the compares succeed. The sweep runs in
subprocesses, one per configuration (plan placement, segment size, PDL), as the put's and the fetch-op's do.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import cas_oracle as co
from tests import put_oracle as po
from tests import put_world as pw
from tests.gpu_helpers import padded_requests, run_world, sweep_requests
from tests.put_world import dense_cover
from tests.test_gpu_accumulate import _index, _shard, add_var
from tests.test_gpu_put import CONFIGS, ERR, SHAPES, inject_invalid, shard_state

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = (1, 2, 4, 8)
U = co.UINT
GUARD = 64  # sentinel bytes on either side of a result buffer


# ------------------------------------------------------------------------------------------------ helpers
def raw_cas(store, name, E, src_ptr, cmp_ptr, res_ptr, src_bytes, torch=None, starts=None, counts=None, fixed=1,
            ids=None, dev=False, flags=0, stream=None, device="cuda:0", keep=None):
    """the C-ABI entry itself -> (rc, total, bad); `keep` (a list) receives the index arrays"""
    from ddstore_b200 import _capi
    L, total, bad = store._L, C.c_int64(0), C.c_int64(-1)
    fl = _capi.SRC_ON_DEVICE | flags
    if ids is not None:
        keep_i, ip, n, d = _index(torch, ids, dev, device)
        rc = L.dds_compare_and_swap_samples(store._h, name.encode(), ip, n, E, src_ptr, cmp_ptr, res_ptr, src_bytes,
                                            fl | d, stream, C.byref(total), C.byref(bad))
        held = (keep_i,)
    else:
        keep_i, sp, n, d = _index(torch, starts, dev, device)
        keep2, cp = (None, None) if counts is None else _index(torch, counts, dev, device)[:2]
        rc = L.dds_compare_and_swap_batch(store._h, name.encode(), sp, cp, fixed, n, E, src_ptr, cmp_ptr, res_ptr,
                                          src_bytes, fl | d, stream, C.byref(total), C.byref(bad))
        held = (keep_i, keep2)
    if keep is not None:
        keep.append(held)
    return rc, total.value, bad.value


class Buffers:
    """device src, compare and result: src `src_off` bytes past a 16-byte boundary, compare `cmp_off`, result `res_off`
    past one inside GUARD sentinel bytes -- or result in place of src (alias "src") or of compare (alias "compare")"""

    def __init__(self, torch, rng, src, cmp, src_off, cmp_off, res_off, alias=None, device="cuda:0", before=None):
        self.n = src.size
        self.alias = alias

        def place(data, off):
            buf = torch.empty(off + data.size + 16, dtype=torch.uint8, device=device)
            if data.size:
                buf[off:off + data.size].copy_(torch.from_numpy(data))
            return buf, buf.data_ptr() + off
        self.src_dev, self.src_ptr = place(src, src_off)
        self.cmp_dev, self.cmp_ptr = place(cmp, cmp_off)
        if alias:
            self.before = (src if alias == "src" else cmp).copy()
            self.whole, self.off = (self.src_dev, src_off) if alias == "src" else (self.cmp_dev, cmp_off)
            self.res_ptr = self.whole.data_ptr() + self.off
        else:
            self.sent = rng.integers(0, 256, size=GUARD + res_off + src.size + GUARD, dtype=np.uint8) \
                if before is None else before
            self.res_dev = torch.from_numpy(self.sent).to(device)
            self.lo = GUARD + res_off
            self.res_ptr = self.res_dev.data_ptr() + self.lo
            self.before = self.sent[self.lo:self.lo + src.size]
        torch.cuda.synchronize(device)

    def read(self, torch, device="cuda:0"):
        """(result bytes, None or a message about the guard bands)"""
        torch.cuda.synchronize(device)
        if self.alias:
            return self.whole.cpu().numpy()[self.off:self.off + self.n], None
        whole = self.res_dev.cpu().numpy()
        g = np.concatenate([whole[:self.lo], whole[self.lo + self.n:]])
        e = np.concatenate([self.sent[:self.lo], self.sent[self.lo + self.n:]])
        return whole[self.lo:self.lo + self.n], (None if np.array_equal(g, e) else "a guard band around result changed")


def operands(rng, shard, lenlist, batch):
    """src and compare of `batch`'s layout (uint8 arrays): src random bits; compare, element by element, the shard's
    value at that element or (half the time) random bits"""
    u = U[shard.dtype.itemsize]
    flat = np.ascontiguousarray(shard).view(u).reshape(-1)
    disp = shard.shape[1]
    rows = int(lenlist[-1])
    parts = []
    for s, c, ok in po.requests(**batch):
        if not (ok and 0 < c <= rows):
            continue
        valid = 0 <= s and s + c <= rows
        parts.append(flat[s * disp:(s + c) * disp] if valid else np.zeros(c * disp, u))
    held = np.concatenate(parts) if parts else np.zeros(0, u)
    rand = lambda n: rng.integers(0, 1 << (8 * u().itemsize), size=n, dtype=u)  # noqa: E731
    src = rand(held.size)
    cmp = np.where(rng.random(held.size) < 0.5, held, rand(held.size))
    return src.view(np.uint8), cmp.astype(u).view(np.uint8)


class World:
    """one rank on cuda:0 with variable `name` of E-byte elements (random bits), optionally a sample index"""

    def __init__(self, torch, store, name, E, disp, nrows, seed, table=None):
        self.rng = np.random.default_rng(seed)
        self.E, self.disp, self.rows, self.name = E, disp, nrows, name
        self.R = E * disp
        self.payload = nrows * self.R
        self.shard = self.rng.integers(0, 1 << (8 * E), size=(nrows, disp), dtype=U[E])
        add_var(torch, store, name, self.shard.view(np.uint8).reshape(-1), nrows, disp, E)
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
        rc = store._L.dds_put_batch(store._h, self.name.encode(), sa.ctypes.data, None, self.rows, 1, self.E,
                                    buf.data_ptr(), self.payload, _capi.SRC_ON_DEVICE, None, C.byref(total), C.byref(bad))
        assert rc == 0 and total.value == self.payload

    def check(self, torch, store, what, src_off=0, cmp_off=0, res_off=0, alias=None, src_bytes=None, dev=False,
              **req):
        """one compare-and-swap of `req`; compare status, total, the whole shard and the whole result with the oracle;
        restore the shard"""
        ll = po.lenlist_of([self.shard])
        src, cmp = operands(self.rng, self.shard, ll, req)
        sb = src.size if src_bytes is None else src_bytes
        b = Buffers(torch, self.rng, src, cmp, src_off, cmp_off, res_off, alias)
        kw = dict(req)
        if "table" in kw:
            kw.pop("table")
            kw["ids"] = kw.pop("sample_ids")
        if "fixed_count" in kw:
            kw["fixed"] = kw.pop("fixed_count")
        nz = src.size > 0
        rc, total, bad = raw_cas(store, self.name, self.E, b.src_ptr if nz else None, b.cmp_ptr if nz else None,
                                 b.res_ptr if nz else None, sb, torch=torch, dev=dev, **kw)
        _, _, codes, ebad, etotal = co.cas([self.shard], src, cmp, b.before, src_bytes=sb, **req)
        ecode, ebad2 = po.expected_error(codes, ebad, etotal, sb)
        assert (rc, bad) == (ERR[ecode], ebad2), f"{what}: rc {rc} bad {bad}, oracle {ERR[ecode]} {ebad2}"
        assert total == etotal, f"{what}: total {total}, oracle {etotal}"
        got, _ = shard_state(torch, store, self.name, self.payload)
        res, guard = b.read(torch)
        assert guard is None, f"{what}: {guard}"
        assert not got[self.payload:].any(), f"{what}: the shard's slack was written"
        gs = got[:self.payload].copy().view(U[self.E]).reshape(self.rows, self.disp)
        msg = co.check([self.shard], [(src, sb, cmp, b.before, req)], [gs], [res])
        assert msg is None, f"{what}: {msg}"
        self.reset(torch, store)
        return codes


# ------------------------------------------------------------------------------------------------ the sweep
BIG_DISP = 65543  # the largest rows: 65543 elements
DENSE_ROWS = 16400


def cas_sweep_main():
    import torch
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    cfg = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("DDS_")) or "default"
    full = cfg == "default"  # (the other configurations change the walk and the plan only)
    for E in WIDTHS:
        rng = np.random.default_rng([E, 7])
        disp, nrows = SHAPES[E]
        tn = f"{E}-byte"
        starts, counts = sweep_requests(rng, nrows, E * disp, (4096, 3072))
        small = counts * E * disp <= (1 << 20) + E * disp
        starts, counts = starts[small], counts[small]
        table = (starts.copy(), counts.copy())
        w = World(torch, store, f"v{E}", E, disp, nrows, E, table)
        # src, compare and result at element-aligned phases of a 16-byte block, and result in place of either
        offs = [(0, 0, 0), (E, 16 - E, 0), (16 - E, E, E), (0, E, 16 - E)] if full else [(E, 16 - E, 0)]
        for k, (so, qo, ro) in enumerate(offs):
            w.check(torch, store, f"[{cfg}] {tn} counts, src +{so} compare +{qo} result +{ro}", src_off=so,
                    cmp_off=qo, res_off=ro, dev=k % 2 == 1, starts=starts, counts=counts)
        if full:
            w.check(torch, store, f"[{cfg}] {tn} result == src", src_off=E, cmp_off=0, alias="src", dev=True,
                    starts=starts, counts=counts)
            w.check(torch, store, f"[{cfg}] {tn} result == compare", src_off=0, cmp_off=16 - E, alias="compare",
                    starts=starts, counts=counts)
        # sample ids with duplicates
        ids = np.concatenate([np.arange(len(starts)), rng.integers(0, len(starts), size=64)])
        ids = rng.permutation(ids).astype(np.int64)
        for dev in (False, True) if full else (True,):
            w.check(torch, store, f"[{cfg}] {tn} sample ids dev={dev}", src_off=(8 if dev else 0) % 16,
                    cmp_off=E if dev else 0, res_off=(3 * E) % 16, dev=dev, sample_ids=ids, table=table)
        fs = rng.integers(0, nrows - 40, size=300)
        for cnt in (1, 3, 40):
            w.check(torch, store, f"[{cfg}] {tn} fixed {cnt}", src_off=(E * cnt) % 16, cmp_off=(E * 5) % 16,
                    dev=cnt != 3, starts=fs, fixed_count=cnt)
        for n in (1024, 1025, 4096, 4097, 8192, 8193):  # both sides of the plan thresholds
            s2, c2 = padded_requests(rng, nrows, starts, counts, n)
            w.check(torch, store, f"[{cfg}] {tn} n={n}", src_off=(E * n) % 16, cmp_off=(E * 7) % 16,
                    res_off=(E * 3) % 16, dev=n % 2 == 0, starts=s2, counts=c2)
        # invalid requests at lane and tile edges and at 1 % density; capacity errors
        s2, c2 = padded_requests(rng, nrows, starts, counts, 2100)
        for where in ([0, 31, 32, 63, 1023, 1024, 2047, 2048], sorted(rng.choice(2100, size=21, replace=False).tolist())):
            si, ci = inject_invalid(rng, s2, c2, nrows, where)
            codes = w.check(torch, store, f"[{cfg}] {tn} invalid {where[:4]}", src_off=E, cmp_off=16 - E, res_off=E,
                            starts=si, counts=ci)
            assert codes[where[0]] != 0
            total = sum(c * w.R if 0 < c <= nrows else 0 for c in ci.tolist())
            w.check(torch, store, f"[{cfg}] {tn} capacity + invalid", src_bytes=total - 1, starts=si, counts=ci)
            w.check(torch, store, f"[{cfg}] {tn} invalid ids", dev=True,
                    sample_ids=np.where(np.isin(np.arange(ids.size), where), -5, ids), table=table)
        w.check(torch, store, f"[{cfg}] {tn} capacity", src_bytes=int(counts.sum()) * w.R - 1, starts=starts,
                counts=counts)
        # every row of a small variable once per batch: each piece's neighbours (for 1- and 2-byte elements: the
        # rest of a 32-bit word) belong to other warps' requests
        ds, dc = dense_cover(rng, DENSE_ROWS, 4097)
        d = World(torch, store, f"d{E}", E, disp, DENSE_ROWS, 100 + E, (ds.copy(), dc.copy()))
        d.check(torch, store, f"[{cfg}] {tn} dense sample ids", src_off=E * 3 % 16, cmp_off=E, dev=True,
                sample_ids=rng.permutation(4097), table=d.table)
        for n in (1025, 8193):
            ds, dc = dense_cover(rng, DENSE_ROWS, n)
            d.check(torch, store, f"[{cfg}] {tn} dense n={n}", src_off=(E * n) % 16, cmp_off=(E * 3) % 16,
                    starts=ds, counts=dc)
        d.check(torch, store, f"[{cfg}] {tn} dense fixed 1", src_off=E, cmp_off=0, res_off=16 - E, dev=True,
                starts=rng.permutation(DENSE_ROWS), fixed_count=1)
        if full:  # rows of 65543 elements, cut at chunk boundaries
            b = World(torch, store, f"b{E}", E, BIG_DISP, 24, 200 + E)
            bs = np.array([0, 23, 5, 11, 0], np.int64)
            bc = np.array([2, 1, 3, 13, 0], np.int64)
            for so, qo, ro in ((0, 0, 0), (E, 0, 16 - E), (16 - E, E, E)):
                b.check(torch, store, f"[{cfg}] {tn} 65543-element rows, src +{so} compare +{qo} result +{ro}",
                        src_off=so, cmp_off=qo, res_off=ro, dev=so > 0, starts=bs, counts=bc)
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_compare_and_swap import cas_sweep_main
cas_sweep_main()
print("cas-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_compare_and_swap_sweep(tmp_path, config):
    """all four widths over the variant sweep's request sizes and 65543-element rows; src, compare and result at
    different 16-byte phases, result == src and result == compare; both entries with host and device indices; batch
    sizes around the plan thresholds; duplicates; invalid requests; capacity errors; dense batches, in the environment
    of `config`"""
    script = tmp_path / "cas_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "cas-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]


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


SPECIALS = {  # bit patterns per float width: +-0, NaNs with different payloads, a signalling NaN, subnormals, +-inf, 1
    2: [0x0000, 0x8000, 0x7E00, 0x7E01, 0x7C01, 0xFE02, 0x0001, 0x8001, 0x03FF, 0x7C00, 0xFC00, 0x3C00,
        0x7FC0, 0x7FC1, 0x7F81, 0x0040, 0x7F80, 0xFF80, 0x3F80],  # (f16 and bf16 patterns alike)
    4: [0x00000000, 0x80000000, 0x7FC00000, 0x7FC00001, 0x7F800001, 0xFFC00002, 0x00000001, 0x80000001, 0x007FFFFF,
        0x7F800000, 0xFF800000, 0x3F800000],
    8: [0, 1 << 63, 0x7FF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0xFFF8000000000002, 1, (1 << 63) | 1,
        0x000FFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x3FF0000000000000]}


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "float32", "float64"])
def test_bitwise_semantics(torch, store, dtype):
    """every special pattern against every other as the compare value, through float tensors: an element is swapped
    exactly when its bits equal the compare's (-0 != +0, NaN payloads and the signalling bit count, subnormals are not
    flushed), and every result holds the previous bits"""
    dt = getattr(torch, dtype)
    E = torch.tensor([], dtype=dt).element_size()
    u = U[E]
    pats = np.array(SPECIALS[E], u)
    n = pats.size
    shard = np.repeat(pats[:, None], n, 1)                  # row i: pattern i everywhere
    cmp = np.repeat(pats[None, :], n, 0)                    # column j: compare against pattern j
    src = np.arange(n * n, dtype=u).reshape(n, n) + 0x11    # (no special pattern among them)
    add_var(torch, store, "f", shard.view(np.uint8).reshape(-1), n, n, E)
    tv = lambda a: torch.from_numpy(a.view({2: np.int16, 4: np.int32, 8: np.int64}[E])).cuda().view(dt)  # noqa: E731
    s_t, c_t = tv(src), tv(cmp)
    out = torch.zeros_like(s_t)
    assert store.compare_and_swap_batch("f", np.arange(n), src=s_t, compare=c_t, out=out) == n * n * E
    got = _shard(torch, store, "f", n, n, {2: torch.int16, 4: torch.int32, 8: torch.int64}[E]).cpu().numpy().view(u)
    exp = np.where(shard == cmp, src, shard)
    assert np.array_equal(got, exp), f"{dtype}: shard differs at {np.argwhere(got != exp)[:4].tolist()}"
    res = out.cpu().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[E]).numpy().view(u)
    assert np.array_equal(res, shard), f"{dtype}: results differ at {np.argwhere(res != shard)[:4].tolist()}"
    assert np.array_equal(res == cmp, np.eye(n, dtype=bool))


@pytest.mark.parametrize("E", WIDTHS)
def test_one_winner_of_65536_claims(torch, store, E):
    """65536 claims of ONE element in one batch (row ids and sample ids), all expecting its value: exactly one wins,
    every other result is the winner's value, and the element holds it"""
    n = 65536
    dt = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[E]
    add_var(torch, store, "c", np.full(64, 0x5A, U[E]).view(np.uint8), 64, 1, E)
    store.set_sample_index("c", np.arange(64), np.ones(64, np.int64))
    for by_id in (False, True):
        base = _shard(torch, store, "c", 64, 1, dt)
        base[9].fill_(0x5A)
        src = (torch.arange(n, device="cuda:0") % (1 << min(8 * E - 1, 62)) + 0x100).to(dt) if E > 1 else \
            (torch.arange(n, device="cuda:0") % 160 + 0x5B).to(dt)
        cmp = torch.full((n,), 0x5A, dtype=dt, device="cuda:0")
        out = torch.zeros_like(src)
        idx = torch.full((n,), 9, dtype=torch.int64, device="cuda:0")
        if by_id:
            store.compare_and_swap_samples("c", idx, src, cmp, out)
        else:
            store.compare_and_swap_batch("c", idx, src=src, compare=cmp, out=out)
        res = out.cpu().numpy()
        wins = np.flatnonzero(res == 0x5A)
        assert wins.size == 1, f"{E}-byte by_id={by_id}: {wins.size} winners"
        final = int(_shard(torch, store, "c", 64, 1, dt)[9, 0])
        w = int(src[int(wins[0])])
        assert final == w and (np.delete(res, wins) == w).all(), f"{E}-byte by_id={by_id}"
        assert not _shard(torch, store, "c", 64, 1, dt)[10:].ne(0x5A).any()


@pytest.mark.parametrize("E", [1, 2])
def test_adjacent_elements_of_one_word(torch, store, E):
    """claims on the 4 / E adjacent elements of each 32-bit word from one batch (200 duplicate claims each, in shuffled
    order): every element has one winner, and every byte ends as its own element's winner left it"""
    dt = {1: torch.uint8, 2: torch.int16}[E]
    rows = 64
    add_var(torch, store, "a", np.zeros(rows * E, np.uint8), rows, 1, E)
    rng = np.random.default_rng(E)
    idx = rng.permutation(np.repeat(np.arange(rows), 200)).astype(np.int64)
    src = torch.from_numpy((np.arange(idx.size) % 250 + 1).astype({1: np.uint8, 2: np.int16}[E])).cuda()
    cmp = torch.zeros_like(src)
    out = torch.full_like(src, -1 if E == 2 else 255)
    store.compare_and_swap_batch("a", torch.from_numpy(idx).cuda(), src=src, compare=cmp, out=out)
    final = _shard(torch, store, "a", rows, 1, dt).cpu().numpy().reshape(-1)
    res, s = out.cpu().numpy(), src.cpu().numpy()
    for r in range(rows):
        m = idx == r
        wins = np.flatnonzero(m & (res == 0))
        assert wins.size == 1 and final[r] == s[wins[0]], f"row {r}: {wins.size} winners"
        assert (res[m & (res != 0)] == final[r]).all(), f"row {r}"


@pytest.mark.parametrize("E", [1, 2])
def test_adjacent_elements_two_ranks(torch, E):
    """two thread-ranks at once, in one epoch: rank 0 claims the even elements of a world, rank 1 the odd ones (every
    32-bit word is shared), both 50 times each, and both claim the hot elements 5 and 6 (one word): every element has
    exactly one winner across the ranks and every byte ends as its winner left it"""
    P, N = 2, 2048
    npdt = {1: np.uint8, 2: np.int16}[E]
    rng = np.random.default_rng(10 + E)
    mine = [np.arange(8 + r, P * N, 2, dtype=np.int64) for r in range(P)]
    idx = [rng.permutation(np.concatenate([np.repeat(m[:64], 50), m, np.repeat([5, 6], 100)])).astype(np.int64)
           for m in mine]
    srcs = [(rng.integers(1, 120, size=i.size) + 120 * r).astype(npdt) for r, i in enumerate(idx)]

    def body(store, r):
        import torch as tt
        dt = {1: tt.uint8, 2: tt.int16}[E]
        store._L.dds_init(store._h, b"n", N, 1, E)
        store.epoch_begin()
        s = tt.from_numpy(srcs[r]).cuda()
        c = tt.zeros_like(s)
        o = tt.full_like(s, 127)
        ix = tt.from_numpy(idx[r]).cuda()
        tt.cuda.synchronize()
        store.compare_and_swap_batch("n", ix, src=s, compare=c, out=o, wait=False)
        store.epoch_end()
        return o.cpu().numpy(), _shard(tt, store, "n", N, 1, dt).cpu().numpy().reshape(-1)
    res = run_world(P, body)
    world = np.concatenate([res[0][1], res[1][1]])
    for e in range(P * N):
        who = [(r, np.flatnonzero(idx[r] == e)) for r in range(P)]
        wins = [(r, int(k)) for r, ks in who for k in ks if res[r][0][k] == 0]
        if sum(ks.size for _, ks in who) == 0:
            assert world[e] == 0, f"element {e} untouched but changed"
            continue
        assert len(wins) == 1, f"element {e}: winners {wins}"
        r, k = wins[0]
        assert world[e] == srcs[r][k], f"element {e}"
        for r2, ks in who:
            assert (res[r2][0][ks][res[r2][0][ks] != 0] == world[e]).all(), f"element {e} rank {r2}"


def test_four_ranks_claim_a_shared_id_set(torch):
    """four thread-ranks claim the same 3000 ids (each in its own order, by sample id) for themselves: every id is
    owned exactly once, and each rank's wins are exactly the ids that hold its rank"""
    P, N, K = 4, 1000, 3000
    rng = np.random.default_rng(4)
    orders = [rng.permutation(K).astype(np.int64) for _ in range(P)]

    def body(store, r):
        import torch as tt
        own = np.full((N, 1), -1, np.int32)
        store.add("owner", own)
        store.set_sample_index("owner", np.arange(K, dtype=np.int64) % (P * N), np.ones(K, np.int64))
        store.epoch_begin()
        ids = tt.from_numpy(orders[r]).cuda()
        s = tt.full((K,), r, dtype=tt.int32, device="cuda")
        c = tt.full((K,), -1, dtype=tt.int32, device="cuda")
        o = tt.zeros_like(s)
        tt.cuda.synchronize()
        store.compare_and_swap_samples("owner", ids, s, c, o)
        store.epoch_end()
        return o.cpu().numpy(), _shard(tt, store, "owner", N, 1, tt.int32).cpu().numpy().reshape(-1)
    res = run_world(P, body)
    world = np.concatenate([res[r][1] for r in range(P)])
    assert ((world[:K] >= 0) & (world[:K] < P)).all() and (world[K:] == -1).all()
    for r in range(P):
        won = orders[r][res[r][0] == -1]
        assert np.array_equal(np.sort(won), np.flatnonzero(world[:K] == r)), f"rank {r}"
        lost = res[r][0] != -1
        assert (res[r][0][lost] == world[orders[r][lost]]).all(), f"rank {r}: a loser's result is not the owner"
    assert sum((res[r][0] == -1).sum() for r in range(P)) == K


def test_queue_endings(torch, store):
    """queued compare-and-swaps completed by wait(), a synchronous call, epoch_begin, epoch_end and free: every queued
    swap is in place, each result holds what its batch saw, the first failure is reported once with its index"""
    nrows, disp = 1000, 16
    h = torch.cuda.Stream().cuda_stream
    good = torch.arange(0, 500, device="cuda:0")
    bad = good.clone()
    bad[7] = nrows + 1
    one = torch.ones(500, disp, dtype=torch.int32, device="cuda:0")
    two = one + 1
    zero = torch.zeros_like(one)
    for ending in ("wait", "sync", "epoch_begin", "epoch_end", "free"):
        store.add("q", np.zeros((nrows, disp), np.int32))
        sh = _shard(torch, store, "q", nrows, disp, torch.int32)
        outs = [torch.full((500, disp), -1, dtype=torch.int32, device="cuda:0") for _ in range(2)]
        torch.cuda.synchronize()
        if ending == "epoch_end":
            store.epoch_begin()
        store.compare_and_swap_batch("q", bad, src=one, compare=zero, out=outs[0], stream=h, wait=False)
        store.compare_and_swap_batch("q", good, src=two, compare=one, out=outs[1], stream=h, wait=False)
        if ending == "wait":
            with pytest.raises(ValueError, match="Invalid count on target"):
                store.wait()
        elif ending == "sync":  # its own outcome: ok
            sync_out = torch.zeros(10, disp, dtype=torch.int32, device="cuda:0")
            assert store.compare_and_swap_batch("q", good[:10], src=one[:10], compare=two[:10], out=sync_out) == \
                10 * disp * 4
            assert sync_out[7].eq(0).all() and sync_out[:7].eq(2).all() and sync_out[8:].eq(2).all()
        else:
            getattr(store, ending)()
        if ending != "free":
            rows = sh.clone()
            assert rows[20].eq(2).all() and rows[5].eq(1 if ending == "sync" else 2).all() and rows[7].eq(0).all() \
                and not rows[500:].any(), ending
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
    """an overlapped get run, a compare-and-swap, an overlapped get run, another, a get run on one stream: each get and
    each compare-and-swap sees exactly what was queued before it"""
    nrows, disp = 2048, 256
    store.add("o", np.zeros((nrows, disp), np.float32))
    h = torch.cuda.Stream().cuda_stream
    starts = torch.arange(0, nrows, 2, device="cuda:0")
    zero = torch.zeros(starts.numel(), disp, device="cuda:0")
    a, b = zero + 3.0, zero + 7.0
    outs = [torch.zeros_like(a) for _ in range(9)]
    r1, r2 = torch.full_like(a, -1), torch.full_like(a, -1)
    torch.cuda.synchronize()
    for k in range(3):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.compare_and_swap_batch("o", starts, src=a, compare=zero, out=r1, stream=h, wait=False)
    for k in range(3, 6):
        store.get_batch("o", starts, out=outs[k], stream=h, wait=False, overlap=True)
    store.compare_and_swap_batch("o", starts, src=b, compare=a, out=r2, stream=h, wait=False)
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
    cmp = torch.zeros(2, 4, device="cuda:0")
    out = torch.zeros(2, 4, device="cuda:0")
    with pytest.raises(KeyError):
        store.compare_and_swap_batch("nope", [0, 1], src=src, compare=cmp, out=out)
    with pytest.raises(ValueError, match="Invalid data type"):
        store.compare_and_swap_batch("e", [0, 1], src=src.double(), compare=cmp.double(), out=out.double())
    with pytest.raises(ValueError, match="elements"):
        store.compare_and_swap_batch("e", [0, 1], src=src, compare=cmp.double(), out=out)
    with pytest.raises(ValueError, match="out holds"):
        store.compare_and_swap_batch("e", [0, 1], src=src, compare=cmp, out=out[:1])
    with pytest.raises(ValueError, match="no sample index"):
        store.compare_and_swap_samples("e", [0], src, cmp, out)
    assert store.compare_and_swap_batch("e", np.zeros(0, np.int64), src=src, compare=cmp, out=out) == 0
    # any dtype of the variable's element size: int32 bits against float32 data
    assert store.compare_and_swap_batch("e", [3], src=src.view(torch.int32)[:1], compare=cmp.view(torch.int32)[:1],
                                        out=out.view(torch.int32)[:1]) == 16
    assert _shard(torch, store, "e", 10, 4, torch.float32)[3].eq(1.0).all()
    total, bad = C.c_int64(0), C.c_int64(0)
    sa = np.zeros(1, np.int64)

    def call(E, ptr, q, res, flags=_capi.SRC_ON_DEVICE, nreq=1):
        return store._L.dds_compare_and_swap_batch(store._h, b"e", sa.ctypes.data, None, 1, nreq, E, ptr, q, res, 16,
                                                   flags, None, C.byref(total), C.byref(bad))
    p, q, o = src.data_ptr(), cmp.data_ptr(), out.data_ptr()
    before = out.clone()
    assert call(3, p, q, o) == _capi.ERR_ARG and "1, 2, 4 or 8" in _capi.last_error()
    assert call(16, p, q, o) == _capi.ERR_ARG
    assert call(8, p, q, o) == _capi.ERR_DTYPE                                   # 8-byte elements, 4-byte variable
    assert call(4, p, None, o) == _capi.ERR_ARG and "null compare" in _capi.last_error()
    assert call(4, p, q, None) == _capi.ERR_ARG and "null result" in _capi.last_error()
    assert call(4, p, q, o + 2) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(4, p, q + 2, o) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(4, p + 2, q, o) == _capi.ERR_ARG and "aligned" in _capi.last_error()
    assert call(4, p, q, o, flags=0) == _capi.ERR_ARG                            # host src
    assert call(4, None, q, o) == _capi.ERR_ARG                                  # null src
    assert call(4, p, q, o, nreq=-1) == _capi.ERR_ARG
    assert call(4, p, q, o, flags=_capi.SRC_ON_DEVICE | _capi.NO_SYNC) == _capi.ERR_ARG  # host indices
    assert not _shard(torch, store, "e", 10, 4, torch.float32)[:3].any() and torch.equal(out, before)
    assert call(4, p, q, o) == 0 and out[0].eq(0).all()
    assert _shard(torch, store, "e", 10, 4, torch.float32)[0].eq(1.0).all()


def test_cython_and_cpp_bindings(torch, tmp_path):
    """compare_and_swap_batch through the Cython binding, and DDStore::compare_and_swap_batch<T> / the explicit-size
    overload / compare_and_swap_samples through the C++ header"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    s = pyd.PyDDStore(None, device=0)
    s.add("c", np.ones((8, 3), np.float32))
    src = torch.arange(6, dtype=torch.float32, device="cuda:0").reshape(2, 3)
    cmp = torch.ones(2, 3, device="cuda:0")
    cmp[0, 1] = 2.0
    out = torch.zeros(2, 3, device="cuda:0")
    torch.cuda.synchronize()
    assert s.compare_and_swap_batch("c", np.array([1, 2], np.int64), src=src, compare=cmp, out=out) == 24
    got = np.zeros((2, 3), np.float32)
    s.get("c", got, 1)
    assert got.tolist() == [[0.0, 1.0, 2.0], [3.0, 4.0, 5.0]] and out.eq(1.0).all()  # (row 1 column 1: compare 2)
    with pytest.raises(ValueError, match="Invalid start on target"):
        s.compare_and_swap_batch("c", np.array([-1], np.int64), src=src[:1], compare=cmp[:1], out=out[:1])
    s.free()
    exe = build_cpp_check(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cpp compare_and_swap ok" in r.stdout, r.stdout + r.stderr


CPP_CHECK = r"""
#include <cuda_runtime.h>
#include <cstdio>
#include "ddstore_b200.hpp"
int main() {
    DDStore s;
    std::vector<int64_t> k(4, 10);
    std::vector<uint8_t> f(8, 0);
    s.add("k", k.data(), 4, 1);
    s.add("f", f.data(), 4, 2);
    const long starts[3] = {2, 2, 2};
    int64_t *dk, *ck, *rk; uint8_t *df, *cf, *rf; long *ds;
    cudaMalloc(&dk, 24); cudaMalloc(&ck, 24); cudaMalloc(&rk, 24); cudaMalloc(&df, 2); cudaMalloc(&cf, 2);
    cudaMalloc(&rf, 2); cudaMalloc(&ds, 24);
    int64_t hk[3] = {21, 22, 23}, hc[3] = {10, 10, 10};
    uint8_t hf[2] = {1, 1}, hcf[2] = {0, 1};
    cudaMemcpy(dk, hk, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(ck, hc, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(df, hf, 2, cudaMemcpyHostToDevice);
    cudaMemcpy(cf, hcf, 2, cudaMemcpyHostToDevice);
    cudaMemcpy(ds, starts, 24, cudaMemcpyHostToDevice);
    if (s.compare_and_swap_batch<int64_t>("k", ds, nullptr, 1, 3, dk, ck, rk, 24) != 24) return 2;
    int64_t got[3];
    cudaMemcpy(got, rk, 24, cudaMemcpyDeviceToHost);
    int wins = 0;
    for (int i = 0; i < 3; i++) wins += got[i] == 10;
    if (wins != 1) return 3;
    if (s.compare_and_swap_batch("f", starts, nullptr, 1, 1, 1, df, cf, rf, 2, false) != 2) return 4;
    uint8_t gf[2];
    cudaMemcpy(gf, rf, 2, cudaMemcpyDeviceToHost);
    if (gf[0] != 0 || gf[1] != 0) return 5;
    try { s.compare_and_swap_samples<uint8_t>("f", ds, 1, df, cf, rf, 2); return 6; }  // (no sample index)
    catch (std::exception &) {}
    try { s.compare_and_swap_batch<double>("f", starts, nullptr, 1, 1, (const double *)dk, (const double *)ck, (double *)rk, 8, false); return 8; }
    catch (std::invalid_argument &e) { if (std::string(e.what()) != "Invalid data type") return 9; }
    s.get("k", 2, 1, k.data());
    s.get("f", 2, 1, f.data());
    if (k[0] < 21 || k[0] > 23 || k[0] != hk[0] + (got[1] == 10) + 2 * (got[2] == 10) || f[0] != 1 || f[1] != 0) return 10;
    s.free();
    printf("cpp compare_and_swap ok\n");
    return 0;
}
"""


def build_cpp_check(tmp_path):
    src = tmp_path / "cas_check.cpp"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "cas_check")
    lib = os.path.join(ROOT, "ddstore_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
           "-L", lib, "-lddstore_b200", f"-Wl,-rpath,{lib}", "-L", "/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


# ------------------------------------------------------------------------------------------------ other ranks
ROWS = {2: [1, 23], 3: [19, 0, 8], 4: [0, 26, 1, 9]}


def cas_world(torch, P, nrows, E, disp, seed, devices=None, queued=False):
    """P thread-ranks; every rank compare-and-swaps into every other rank's rows (owner edges, straddlers and the
    invalid family, a by-sample-id form, a dense cover of the world, one call per rank short of source) in one epoch;
    after the closing fence every rank returns its shard and its calls' results and statuses, checked against the
    oracle (every element is touched by several ranks)"""
    rng = np.random.default_rng([seed, P, E])
    ll = pw.lenlist_of(nrows)
    R = E * disp
    shards = [rng.integers(0, 1 << (8 * E), size=(n, disp), dtype=U[E]) for n in nrows]
    world = np.concatenate(shards) if sum(nrows) else np.zeros((0, disp), U[E])
    total = int(ll[-1])
    tables, calls = [], []  # calls[r] = [(src, src_bytes or None, compare, batch, src offset)]
    cover = pw.interleaved_cover(rng, ll, P, R, big=R <= 64)
    for r in range(P):
        others = [o[0] for o in pw.owners(ll) if o[0] != r] or None
        st, ct, cls = pw.edge_requests(rng, ll, r, first_bad=None if r == 0 else int(rng.integers(0, 6)), body=12,
                                       only=others)
        mine = []
        batches = [{"starts": st, "counts": ct}]
        sb, _ = pw.as_samples(rng, st, ct, cls, first_bad=None if r % 2 == 0 else 1)
        tables.append(sb["table"])
        batches += [sb, {"starts": cover[r][0], "counts": cover[r][1]}]
        for k, b in enumerate(batches):
            s, c = operands(rng, world, ll, b)
            mine.append((s, None, c, b, E * ((r + k) % (16 // E))))
        if r == P - 1 and total:
            fb = {"starts": np.array([0, total - 1], np.int64), "fixed_count": 1}
            s, c = operands(rng, world, ll, fb)
            mine.append((s, s.size - 1, c, fb, 0))  # capacity: nothing applied
        calls.append(mine)

    def status(c):
        codes, _pl, bad, tot, _ = co.plan(shards, c[0].size if c[1] is None else c[1], **c[3])
        return po.expected_error(codes, bad, tot, c[0].size if c[1] is None else c[1])
    exp_status = [[status(c) for c in mine] for mine in calls]
    res_off = [[(c[4] + E) % 16 for c in mine] for mine in calls]
    befores = [[rng.integers(0, 256, size=GUARD + o + c[0].size + GUARD, dtype=np.uint8) for c, o in zip(mine, offs)]
               for mine, offs in zip(calls, res_off)]

    def body(store, r):
        import torch as tt
        dev = tt.device("cuda", tt.cuda.current_device())
        problems = []
        mine = np.ascontiguousarray(shards[r]).view(np.uint8).reshape(-1)
        assert store._L.dds_add(store._h, b"w", mine.ctypes.data if mine.size else None, nrows[r], disp, E, 0) == 0
        store.set_sample_index("w", *tables[r])
        stream = tt.cuda.Stream(device=dev).cuda_stream if queued else None
        keep, bufs = [], []
        store.epoch_begin()
        for k, (src, sbytes, cmp, batch, off) in enumerate(calls[r]):
            b = Buffers(tt, None, src, cmp, off, (off + 2 * E) % 16, res_off[r][k], device=dev, before=befores[r][k])
            bufs.append(b)
            sb = src.size if sbytes is None else sbytes
            kw = {"ids": batch["sample_ids"]} if "sample_ids" in batch else \
                {"starts": batch["starts"], "counts": batch.get("counts"), "fixed": batch.get("fixed_count", 1)}
            nz = src.size > 0
            got = raw_cas(store, "w", E, b.src_ptr if nz else None, b.cmp_ptr if nz else None,
                          b.res_ptr if nz else None, sb, torch=tt, dev=queued or k % 2 == 1,
                          flags=(4 if queued else 0), stream=stream, device=dev, keep=keep, **kw)
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
        got, _ = shard_state(tt, store, "w", payload, dev)
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
    got_shards = [o[1].view(U[E]).reshape(n, disp) for o, n in zip(out, nrows)]
    flat = [(c[0], c[1], c[2], bf[GUARD + o:GUARD + o + c[0].size], c[3])
            for mine, offs, bfs in zip(calls, res_off, befores) for c, o, bf in zip(mine, offs, bfs)]
    got_res = [res for o in out for res in o[2]]
    msg = co.check(shards, flat, got_shards, got_res)
    assert msg is None, f"P={P} {E}-byte: {msg}"


@pytest.mark.parametrize("P", [2, 3, 4])
@pytest.mark.parametrize("E", WIDTHS)
def test_multi_owner_worlds(torch, P, E):
    cas_world(torch, P, [n * 20 if n > 1 else n for n in ROWS[P]], E, {1: 7, 2: 5, 4: 3, 8: 2}[E], seed=1)


@pytest.mark.parametrize("E", [1, 4])
def test_three_owner_world_queued(torch, E):
    cas_world(torch, 3, [380, 0, 160], E, 3, seed=2, queued=True)


def test_sixty_four_owners(torch):
    rng = np.random.default_rng(64)
    nrows = [0 if k % 3 == 0 else int(rng.integers(1, 6)) for k in range(64)]
    cas_world(torch, 64, nrows, 2, 5, seed=3)


def test_one_gpu_per_rank(torch):
    """the same across GPUs: compare-and-swaps into peer HBM over NVLink"""
    P = torch.cuda.device_count()
    if P < 2:
        pytest.skip("needs two or more GPUs")
    cas_world(torch, P, [37 * (k + 1) for k in range(P)], 4, 1024, seed=4, devices=list(range(P)))
