"""Pooled batches on the GPU (dds_get_batch_pooled / dds_get_samples_pooled, PyDDStore.get_batch_pooled /
get_samples_pooled) against tests/pool_oracle.py, bit for bit: every element type and mode over row sizes from one
element to 16 KiB, bags of 0 to 20000 rows, every request form with host and device indices, inexact floats,
subnormals, NaNs and signed zeros, thread-rank worlds with an empty shard, invalid requests, malformed bags, every
argument error, queues, HOST placement -- and torch's CUDA embedding_bag on a local copy of the table."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests import pool_oracle as pl
from tests import put_oracle as po
from tests.gpu_helpers import run_world

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TYPES = (pl.ACC_F32, pl.ACC_F64, pl.ACC_F16, pl.ACC_BF16)
TORCH_DT = {pl.ACC_F32: torch.float32, pl.ACC_F64: torch.float64, pl.ACC_F16: torch.float16,
            pl.ACC_BF16: torch.bfloat16}
INT_VIEW = {2: torch.int16, 4: torch.int32, 8: torch.int64}
SIZE = {pl.ACC_F32: 4, pl.ACC_F64: 8, pl.ACC_F16: 2, pl.ACC_BF16: 2}
MODES = {"sum": pl.POOL_SUM, "weighted": pl.POOL_SUM, "mean": pl.POOL_MEAN, "max": pl.POOL_MAX}


def data_bits(rng, t, n, special=True):
    """n elements of type t (storage array; bf16 as bits): inexact values over a wide range, subnormals, signed zeros
    and -- special=True -- a few NaNs (with payloads) and infinities"""
    v = rng.uniform(-4, 4, n) * np.exp2(rng.integers(-8, 8, n)) / 3
    a = pl.encode(v.astype(np.float32), t) if t == pl.ACC_BF16 else v.astype(pl.STORAGE[t])
    b = a.view(pl.BITS[t]) if t != pl.ACC_BF16 else a
    w = {2: 16, 4: 32, 8: 64}[SIZE[t]]
    mant = {pl.ACC_F32: 23, pl.ACC_F64: 52, pl.ACC_F16: 10, pl.ACC_BF16: 7}[t]
    u = rng.random(n)
    sub = u < 0.05
    b[sub] = (rng.integers(1, 1 << min(mant, 20), sub.sum()).astype(np.uint64) |
              (rng.integers(0, 2, sub.sum()).astype(np.uint64) << (w - 1))).astype(b.dtype)
    zero = (u >= 0.05) & (u < 0.09)
    b[zero] = (rng.integers(0, 2, zero.sum()).astype(np.uint64) << (w - 1)).astype(b.dtype)
    if special:
        exp_all = ((1 << (w - 1)) - 1) ^ ((1 << mant) - 1)
        nan = (u >= 0.09) & (u < 0.093)
        b[nan] = (exp_all | rng.integers(1, 1 << min(mant, 20), nan.sum()) | (1 << (mant - 1))).astype(b.dtype)
        inf = (u >= 0.093) & (u < 0.095)
        b[inf] = (exp_all | (rng.integers(0, 2, inf.sum()) << (w - 1))).astype(b.dtype)
    return a if t == pl.ACC_BF16 else b.view(pl.STORAGE[t])


def add_var(store, name, shard, t, placement=0):
    shard = np.ascontiguousarray(shard)
    nrows, disp = shard.shape
    rc = store._L.dds_add_placed(store._h, name.encode(), shard.ctypes.data if shard.size else None, nrows, disp,
                                 SIZE[t], 0, placement)
    assert rc == 0, store._L.dds_last_error()


def bits_of(out, t):
    return out.view(INT_VIEW[SIZE[t]]).cpu().numpy().view(pl.BITS[t])


def to_torch(a, t):
    """a storage array of type t (bf16 as bits) -> a CPU tensor of the torch dtype, bit for bit"""
    ints = np.ascontiguousarray(a).view(pl.BITS[t]).view({2: np.int16, 4: np.int32, 8: np.int64}[SIZE[t]])
    return torch.from_numpy(ints.copy()).view(TORCH_DT[t])


def bag_offsets(rng, sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def check(got, exp, what):
    if not np.array_equal(got, exp):
        k, e = (int(x[0]) for x in np.nonzero(got != exp))
        raise AssertionError(f"{what}: {int((got != exp).sum())} elements differ; first at bag {k}, element {e}: "
                             f"got {int(got[k, e]):#x}, oracle {int(exp[k, e]):#x}")


def run_pool(store, name, t, mode, form, dev, rng, nrows, bag_sizes, weighted=False, ids=None, out=None):
    """one pooled call on variable `name` (nrows global rows) with bags of bag_sizes requests; returns (got, exp, err)"""
    nreq = int(sum(bag_sizes))
    bags = bag_offsets(rng, bag_sizes)
    req = {}
    if form == "samples":
        req = {"sample_ids": ids[0][rng.integers(0, len(ids[0]), nreq)], "table": ids[1]}
    elif form == "counts":
        counts = rng.integers(0, 4, nreq)
        req = {"starts": rng.integers(0, max(1, nrows - 3), nreq), "counts": counts}
    else:
        c = 1 if form == "fixed1" else 2
        req = {"starts": rng.integers(0, max(1, nrows - c + 1), nreq), "fixed_count": c}
    w = data_bits(rng, t, nreq, special=False) if weighted else None
    return call(store, name, t, mode, dev, req, bags, w, out=out)


def call(store, name, t, mode, dev, req, bags, w, out=None):
    nbags = len(bags) - 1 if bags is not None else len(req.get("starts", req.get("sample_ids")))
    disp = store.query(name)["disp"]
    if out is None:
        out = torch.full((nbags, disp), 7, dtype=TORCH_DT[t], device="cuda")
    wt = None if w is None else to_torch(w, t)

    def idx(a):
        return torch.from_numpy(np.asarray(a, np.int64)).cuda() if dev else np.asarray(a, np.int64)
    b = None if bags is None else idx(bags)
    wv = None if wt is None else (wt.cuda() if dev else wt)
    pm = "max" if mode == pl.POOL_MAX else "mean" if mode == pl.POOL_MEAN else "sum"
    err = None
    try:
        if "sample_ids" in req:
            store.get_samples_pooled(name, idx(req["sample_ids"]), out, bags=b, mode=pm, weights=wv)
        else:
            store.get_batch_pooled(name, idx(req["starts"]), idx(req["counts"]) if "counts" in req else None,
                                   count=req.get("fixed_count"), out=out, bags=b, mode=pm, weights=wv)
    except ValueError as e:
        err = (str(e), store.last_bad_index)
    return out, req, w, err


def oracle(shards, t, mode, req, bags, w):
    return pl.pool(shards, t, mode, bags=bags, weights=w, **req)


# ----------------------------------------------------------------------------------------- types, modes, row sizes
@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("row_bytes", [None, 3, 64, 128, 1000, 16384])
def test_types_modes_rows(t, mode, row_bytes):
    from ddstore_b200 import PyDDStore
    disp = 1 if row_bytes is None else (row_bytes // SIZE[t] if row_bytes == 16384 else row_bytes)
    rng = np.random.default_rng(t * 100003 + list(MODES).index(mode) * 1009 + disp)
    nrows = 3000
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    sizes = [0, 1, 31, 32, 33, 5, 0, 2] if disp * SIZE[t] <= 4096 else [0, 1, 31, 33, 2]
    if mode == "weighted" and t == pl.ACC_F64 and disp > 64:
        sizes = [0, 1, 3, 2]  # (the oracle's exact fma is slow in float64)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        for off in (0, 1):  # out 16-byte aligned (vector path where rows allow), then one element past it
            buf = torch.full((len(sizes) * disp + 16 // SIZE[t],), 7, dtype=TORCH_DT[t], device="cuda")
            out = buf[off:off + len(sizes) * disp].view(len(sizes), disp)
            assert (out.data_ptr() % 16 == 0) == (off == 0)
            out, req, w, err = run_pool(store, "x", t, MODES[mode], "counts", True, rng, nrows, sizes, mode == "weighted",
                                        out=out)
            assert err is None, err
            exp, _, eerr = oracle([shard], t, MODES[mode], req, bag_offsets(rng, sizes), w)
            assert eerr == (0, -1)
            check(bits_of(out, t), exp, f"type {t} {mode} disp {disp} off {off}")
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- request forms, index residency
@pytest.mark.parametrize("form", ["fixed1", "fixed2", "counts", "samples"])
@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("t,mode", [(pl.ACC_F32, "weighted"), (pl.ACC_BF16, "mean"), (pl.ACC_F16, "max")])
def test_request_forms(form, dev, t, mode):
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(len(form) * 7 + dev + t)
    nrows, disp = 2000, 40
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        rs = rng.integers(0, nrows - 5, 300)
        rc = rng.integers(0, 5, 300)
        store.set_sample_index("x", rs, rc)
        sizes = rng.integers(0, 40, 30)
        sizes[3] = 0
        out, req, w, err = run_pool(store, "x", t, MODES[mode], form, dev, rng, nrows, sizes, mode == "weighted",
                                    ids=(np.arange(300), (rs, rc)))
        assert err is None, err
        exp, _, _ = oracle([shard], t, MODES[mode], req, bag_offsets(rng, sizes), w)
        check(bits_of(out, t), exp, f"{form} dev={dev}")
        # bags=None: one bag per request
        out2, req2, w2, err = call(store, "x", t, MODES[mode], dev, req, None, w)
        exp2, _, _ = oracle([shard], t, MODES[mode], req2, None, w2)
        check(bits_of(out2, t), exp2, f"{form} dev={dev}, a bag per request")
    finally:
        store.free()
        store.close()


def test_long_bag_among_short_ones():
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(5)
    for t, mode, disp in ((pl.ACC_F32, pl.POOL_SUM, 128), (pl.ACC_BF16, pl.POOL_MEAN, 256), (pl.ACC_F64, pl.POOL_MAX, 9)):
        nrows = 50000
        shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
        store = PyDDStore(device=0)
        try:
            add_var(store, "x", shard, t)
            sizes = [3, 1, 20000, 0, 7, 2]
            out, req, w, err = run_pool(store, "x", t, mode, "fixed1", True, rng, nrows, sizes)
            assert err is None, err
            exp, _, _ = oracle([shard], t, mode, req, bag_offsets(rng, sizes), w)
            check(bits_of(out, t), exp, f"a bag of 20000 rows, type {t}")
        finally:
            store.free()
            store.close()


# ----------------------------------------------------------------------------------------- worlds
@pytest.mark.parametrize("multi_gpu", [False, True])
def test_world_with_an_empty_shard(multi_gpu):
    P = 3
    if multi_gpu and torch.cuda.device_count() < P:
        pytest.skip("needs one GPU per rank")
    t, disp = pl.ACC_F32, 24
    rng = np.random.default_rng(11)
    nrows = [700, 0, 500]
    shards = [data_bits(rng, t, n * disp).reshape(n, disp) for n in nrows]
    total = sum(nrows)

    def body(store, r):
        dev = torch.device(f"cuda:{r if multi_gpu else 0}")
        torch.cuda.set_device(dev)
        add_var(store, "x", shards[r], t)
        store.epoch_begin()
        res = []
        for mode in (pl.POOL_SUM, pl.POOL_MEAN, pl.POOL_MAX):
            g = np.random.default_rng(100 * r + mode)
            sizes = g.integers(0, 50, 20)
            req = {"starts": g.integers(0, total - 3, int(sizes.sum())), "counts": g.integers(0, 4, int(sizes.sum()))}
            bags = bag_offsets(g, sizes)
            out = torch.zeros((len(sizes), disp), dtype=torch.float32, device=dev)
            pm = {pl.POOL_SUM: "sum", pl.POOL_MEAN: "mean", pl.POOL_MAX: "max"}[mode]
            err = (0, -1)
            try:  # (requests that cross a shard boundary are invalid: they are reported, the rest are pooled)
                store.get_batch_pooled("x", torch.from_numpy(req["starts"]).to(dev),
                                       torch.from_numpy(req["counts"]).to(dev), out=out,
                                       bags=torch.from_numpy(bags).to(dev), mode=pm)
            except ValueError as e:
                err = (str(e), store.last_bad_index)
            res.append((mode, req, bags, bits_of(out, t), err))
        store.epoch_end()
        return res

    for r, res in enumerate(run_world(P, body, devices=list(range(P)) if multi_gpu else None)):
        for mode, req, bags, got, err in res:
            exp, _, eerr = oracle(shards, t, mode, req, bags, None)
            check(got, exp, f"rank {r} mode {mode}")
            assert err[1] == eerr[1], (err, eerr)
            if eerr[1] >= 0:
                assert {po.CODE_START: "Invalid start on target", po.CODE_COUNT: "Invalid count on target"}[eerr[0]] \
                    in err[0]


# ----------------------------------------------------------------------------------------- invalid input
@pytest.mark.parametrize("form", ["counts", "samples"])
def test_invalid_requests_first_reported_valid_applied(form):
    from ddstore_b200 import PyDDStore
    t, disp, nrows = pl.ACC_F32, 16, 500
    rng = np.random.default_rng(3)
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        rs, rcnt = rng.integers(0, nrows - 4, 50), rng.integers(0, 4, 50)
        store.set_sample_index("x", rs, rcnt)
        sizes = [4, 6, 0, 5, 9]
        n = sum(sizes)
        if form == "counts":
            starts, counts = rng.integers(0, nrows - 4, n), rng.integers(0, 4, n)
            starts[7], counts[12], counts[20] = nrows + 3, -1, nrows  # start, negative count, count too large
            req = {"starts": starts, "counts": counts}
        else:
            ids = rng.integers(0, 50, n)
            ids[8], ids[15] = 50, -2
            req = {"sample_ids": ids, "table": (rs, rcnt)}
        bags = bag_offsets(rng, sizes)
        exp, codes, eerr = oracle([shard], t, pl.POOL_SUM, req, bags, None)
        for dev in (False, True):
            out, _, _, err = call(store, "x", t, pl.POOL_SUM, dev, req, bags, None)
            assert err is not None and err[1] == eerr[1], (err, eerr)
            text = "sample id" if eerr[0] == po.CODE_SAMPLE else {po.CODE_START: "Invalid start on target",
                                                                    po.CODE_COUNT: "Invalid count on target"}[eerr[0]]
            assert text in err[0]
            check(bits_of(out, t), exp, f"{form}, dev={dev}: every valid request applied")
    finally:
        store.free()
        store.close()


def test_malformed_bags():
    from ddstore_b200 import PyDDStore
    t, disp, nrows = pl.ACC_F64, 5, 100
    rng = np.random.default_rng(4)
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        starts = rng.integers(0, nrows, 10)
        starts[1] = nrows + 5  # an invalid request in a well-formed bag: the malformed bag still wins
        req = {"starts": starts, "fixed_count": 1}
        for bags, k in (([0, 3, 2, 10], 1), ([0, 4, 11], 1), ([-1, 2, 10], 0), ([0, 2, 5, 4, 10], 2)):
            bags = np.array(bags, np.int64)
            exp, _, eerr = oracle([shard], t, pl.POOL_SUM, req, bags, None)
            assert eerr == (pl.CODE_BAG, k)
            # device bags: checked by the kernel; the malformed bag's row is zeros, the others are pooled
            out, _, _, err = call(store, "x", t, pl.POOL_SUM, True, req, bags, None)
            assert err is not None and "malformed bag offsets" in err[0] and err[1] == k, err
            check(bits_of(out, t), exp, f"device bags {bags.tolist()}")
            # host bags: checked before anything is enqueued; nothing is written
            out, _, _, err = call(store, "x", t, pl.POOL_SUM, False, req, bags, None)
            assert err is not None and "malformed bag offsets" in err[0] and err[1] == k, err
            assert bool((out == 7).all()), "a call refused on the host wrote its destination"
    finally:
        store.free()
        store.close()


def test_argument_errors_write_nothing():
    from ddstore_b200 import PyDDStore, _capi
    store = PyDDStore(device=0)
    try:
        shard = np.ones((64, 8), np.float32)
        add_var(store, "x", shard, pl.ACC_F32)
        add_var(store, "y", np.ones((64, 8), np.float64), pl.ACC_F64)
        L, h = store._L, store._h
        starts = torch.arange(8, dtype=torch.int64, device="cuda")
        bags = torch.tensor([0, 4, 8], dtype=torch.int64, device="cuda")
        whole = torch.full((4096,), 0x5A, dtype=torch.uint8, device="cuda")
        dst = whole[64:]
        wts = torch.ones(16, dtype=torch.float32, device="cuda")
        D = _capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE

        def pool(mode=1, dtype=1, b=bags.data_ptr(), nb=2, w=None):
            return _capi.Pool(mode, dtype, b, nb, w)

        def go(p, name=b"x", d=dst.data_ptr(), cap=1024, flags=D, nreq=8, samples=False):
            tot, bad = C.c_int64(0), C.c_int64(-1)
            if samples:
                return L.dds_get_samples_pooled(h, name, starts.data_ptr(), nreq, C.byref(p), d, cap, flags, None,
                                                C.byref(tot), C.byref(bad))
            return L.dds_get_batch_pooled(h, name, starts.data_ptr(), None, 1, nreq, C.byref(p), d, cap, flags, None,
                                          C.byref(tot), C.byref(bad))
        cases = {
            "unknown mode": (pool(mode=4), {}),
            "mode 0": (pool(mode=0), {}),
            "integer dtype": (pool(dtype=_capi.ACC_I32), {}),
            "unknown dtype": (pool(dtype=9), {}),
            "weights with mean": (pool(mode=2, w=wts.data_ptr()), {}),
            "weights with max": (pool(mode=3, w=wts.data_ptr()), {}),
            "host destination": (pool(), {"flags": _capi.IDX_ON_DEVICE}),
            "negative nbags": (pool(nb=-1), {}),
            "no bags, nbags != nreq": (pool(b=None, nb=3), {}),
            "capacity": (pool(), {"cap": 2 * 32 - 1}),
            "overflow": (pool(nb=1 << 61), {"cap": 1 << 62}),
            "misaligned dst": (pool(), {"d": dst.data_ptr() + 2}),
            "misaligned weights": (pool(w=wts.data_ptr() + 2), {}),
            "no sample index": (pool(), {"samples": True}),
        }
        for what, (p, kw) in cases.items():
            assert go(p, **kw) == _capi.ERR_ARG, what
            torch.cuda.synchronize()
            assert bool((whole == 0x5A).all()), f"{what}: the destination was written"
        assert go(pool(dtype=_capi.ACC_F16)) == _capi.ERR_DTYPE
        assert go(pool(dtype=_capi.ACC_F32), name=b"y") == _capi.ERR_DTYPE
        torch.cuda.synchronize()
        assert bool((whole == 0x5A).all())
        assert go(pool()) == 0  # (the same call, well-formed, runs)
        with pytest.raises(ValueError):
            store.get_batch_pooled("x", starts, out=torch.zeros(8, 8, device="cuda"), mode="median")
        with pytest.raises(ValueError):
            store.get_batch_pooled("x", starts, out=torch.zeros(8, 8, dtype=torch.int32, device="cuda"))
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- queues
def test_queued_with_gets_and_puts():
    from ddstore_b200 import PyDDStore
    t, disp, nrows = pl.ACC_F32, 32, 1000
    rng = np.random.default_rng(9)
    shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        dev = torch.device("cuda")
        cur = shard.copy()
        outs, exps = [], []
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for q in range(6):
                starts = torch.from_numpy(rng.integers(0, nrows, 64)).to(dev)
                bags = torch.from_numpy(bag_offsets(rng, rng.integers(0, 16, 8)) * 0 + np.array(
                    [0, 3, 10, 10, 20, 33, 40, 50, 64])).to(dev)
                if q == 4:
                    starts[5] = nrows + 1  # the first failing batch of the queue: the 5th
                if q == 5:
                    starts[0] = -1
                out = torch.zeros((8, disp), dtype=torch.float32, device=dev)
                store.get_batch_pooled("x", starts, out=out, bags=bags, mode="sum", stream=s.cuda_stream, wait=False)
                exp, _, _ = oracle([cur], t, pl.POOL_SUM, {"starts": starts.cpu().numpy(), "fixed_count": 1},
                                   bags.cpu().numpy(), None)
                outs.append(out)
                exps.append(exp)
                if q == 1:  # a queued put between pooled batches: the next ones see its rows
                    rows = torch.from_numpy(data_bits(rng, t, 4 * disp, special=False).reshape(4, disp)).to(dev)
                    pst = torch.tensor([10, 11, 12, 13], dtype=torch.int64, device=dev)
                    store.put_batch("x", pst, src=rows, stream=s.cuda_stream, wait=False)
                    cur[10:14] = rows.cpu().numpy()
                if q == 2:  # and a queued get
                    g = torch.empty((8, disp), dtype=torch.float32, device=dev)
                    store.get_batch("x", torch.arange(8, device=dev), out=g, count=1, stream=s.cuda_stream, wait=False)
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.wait()
        assert store.last_bad_index == 5
        assert store.wait() == 0
        for q, (o, e) in enumerate(zip(outs, exps)):
            check(bits_of(o, t), e, f"queued batch {q}")
        assert np.array_equal(g.cpu().numpy(), cur[:8])
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- HOST placement
@pytest.mark.parametrize("t", [pl.ACC_F32, pl.ACC_BF16])
def test_host_placement_matches_hbm(t):
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(12)
    nrows, disp = 3000, 77
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "h", shard, t, placement=1)
        add_var(store, "m", shard, t, placement=0)
        assert store.query("h")["placement"] == "host"
        sizes = rng.integers(0, 60, 40)
        bags = bag_offsets(rng, sizes)
        req = {"starts": rng.integers(0, nrows - 3, int(sizes.sum())), "counts": rng.integers(0, 4, int(sizes.sum()))}
        for mode in (pl.POOL_SUM, pl.POOL_MEAN, pl.POOL_MAX):
            a, _, _, e1 = call(store, "h", t, mode, True, req, bags, None)
            b, _, _, e2 = call(store, "m", t, mode, True, req, bags, None)
            assert e1 is None and e2 is None
            exp, _, _ = oracle([shard], t, mode, req, bags, None)
            check(bits_of(a, t), exp, f"HOST mode {mode}")
            check(bits_of(b, t), exp, f"HBM mode {mode}")
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- torch's embedding_bag
@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("mode", list(MODES))
def test_matches_torch_embedding_bag(t, mode):
    """count=1 requests over a 3-rank world against F.embedding_bag on a CUDA copy of the concatenated shards"""
    import torch.nn.functional as F
    rng = np.random.default_rng(t * 4 + len(mode))
    disp, nrows = 64, [4000, 0, 3000]
    shards = [data_bits(rng, t, n * disp, special=False).reshape(n, disp) for n in nrows]
    allrows = np.concatenate(shards)
    table = to_torch(allrows, t).cuda()
    sizes = rng.integers(0, 40, 500)
    sizes[:4] = [0, 1, 32, 33]
    bags = bag_offsets(rng, sizes)
    ids = rng.integers(0, sum(nrows), int(bags[-1]))
    w = to_torch(data_bits(rng, t, ids.size, special=False), t).cuda() if mode == "weighted" else None
    pm = "sum" if mode == "weighted" else mode
    ref = F.embedding_bag(torch.from_numpy(ids).cuda(), table, torch.from_numpy(bags).cuda(), mode=pm,
                          per_sample_weights=w, include_last_offset=True)

    def body(store, r):
        add_var(store, "x", shards[r], t)
        store.epoch_begin()
        out = torch.empty((len(sizes), disp), dtype=TORCH_DT[t], device="cuda")
        store.get_batch_pooled("x", torch.from_numpy(ids).cuda(), out=out, bags=torch.from_numpy(bags).cuda(), mode=pm,
                               weights=w)
        store.epoch_end()
        return bits_of(out, t)

    got = run_world(3, body)
    check(got[0], bits_of(ref, t), f"type {t} {mode} against torch.nn.functional.embedding_bag")
    check(got[2], got[0], "ranks agree")


# ----------------------------------------------------------------------------------------- the Cython binding
@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("t,mode", [(pl.ACC_F32, "weighted"), (pl.ACC_F64, "mean")])
def test_cython_binding(dev, t, mode):
    """pyddstore.PyDDStore.get_batch_pooled: a weighted sum and a mean over bags, host and device indices"""
    cydir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    rng = np.random.default_rng(17 + dev + t)
    nrows, disp = 600, 24
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    sizes = rng.integers(0, 20, 12)
    sizes[2] = 0
    nreq = int(sizes.sum())
    bags = bag_offsets(rng, sizes)
    starts = rng.integers(0, nrows - 3, nreq).astype(np.int64)
    counts = rng.integers(0, 4, nreq).astype(np.int64)
    w = data_bits(rng, t, nreq, special=False) if mode == "weighted" else None
    wt = None if w is None else (to_torch(w, t).cuda() if dev else to_torch(w, t))
    out = torch.full((len(sizes), disp), 7, dtype=TORCH_DT[t], device="cuda")

    def idx(a):
        return torch.from_numpy(a).cuda() if dev else a
    s = pyd.PyDDStore(None, device=0)
    try:
        s.add("x", shard)
        total = s.get_batch_pooled("x", idx(starts), idx(counts), out=out, bags=idx(bags),
                                   mode="sum" if mode == "weighted" else mode, weights=wt)
        assert total == out.numel() * out.element_size()
        exp, _, eerr = oracle([shard], t, MODES[mode], {"starts": starts, "counts": counts}, bags, w)
        assert eerr == (0, -1)
        check(bits_of(out, t), exp, f"cython {mode} dev={dev}")
    finally:
        s.free()
