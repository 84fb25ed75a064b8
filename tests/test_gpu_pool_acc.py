"""Pooled accumulates on the GPU (dds_accumulate_batch_pooled / dds_accumulate_samples_pooled,
PyDDStore.accumulate_batch_pooled / accumulate_samples_pooled) against tests/pool_acc_oracle.py: every element type and
mode over row sizes from one element to 16 KiB, aligned and unaligned grad and weights, bags of 0 to 20000 requests,
every request form with host and device indices, duplicates and hot rows in one batch and across thread-ranks,
invalid requests, malformed bags and argument errors, queues mixed with the other batched calls, K SGD steps of a
sharded EmbeddingBag against torch's, and the Cython and C++ bindings.

Where every row is touched at most once, each element's result is one addition of its contribution to its start:
checked against acc_oracle's admissible results (IEEE, or f32's flush model), the contributions against torch's CUDA
expression on the expanded tensors bit for bit, and the shard against accumulate_batch of those expanded contributions
(bit for bit but where the f32 flush model admits two results)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import pool_acc_oracle as pao
from tests import pool_oracle as pl
from tests import put_oracle as po
from tests.gpu_helpers import run_world
from tests.test_gpu_pool import INT_VIEW, SIZE, TORCH_DT, add_var, bag_offsets, data_bits, to_torch

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = (pl.ACC_F32, pl.ACC_F64, pl.ACC_F16, pl.ACC_BF16)
MODES = {"sum": pl.POOL_SUM, "weighted": pl.POOL_SUM, "mean": pl.POOL_MEAN}


def shard_bits(store, name, nrows, disp, t, device="cuda:0"):
    """the local shard's elements as a storage array of t (bf16 as bits)"""
    from ddstore_b200.store import _DevMem
    n = nrows * disp * SIZE[t]
    if n == 0:
        return np.zeros((0, disp), ao.STORAGE[t])
    torch.cuda.synchronize(device)
    raw = torch.as_tensor(_DevMem(store.query(name)["local_base"], n), device=device).view(INT_VIEW[SIZE[t]])
    return raw.cpu().numpy().view(ao.STORAGE[t]).reshape(nrows, disp).copy()


def disjoint(rng, nrows, nreq, maxc, fixed=None):
    """nreq requests of 0..maxc rows (maxc 0: exactly one row each; `fixed`: that many each) over distinct rows ->
    (starts, counts)"""
    w = max(maxc, 1)
    slots = rng.permutation(nrows // w)[:nreq]
    assert len(slots) == nreq
    counts = np.full(nreq, fixed) if fixed else rng.integers(0, maxc + 1, nreq) if maxc else np.ones(nreq, np.int64)
    offs = rng.integers(0, w - counts + 1)
    return (slots * w + offs).astype(np.int64), counts.astype(np.int64)


def grad_tensor(g, t, off=0):
    """grad [nbags, disp] on the device, starting `off` elements past a 16-byte boundary"""
    flat = to_torch(g.reshape(-1), t).cuda()
    buf = torch.zeros(flat.numel() + off + 16 // SIZE[t], dtype=TORCH_DT[t], device="cuda")
    buf[off:off + flat.numel()].copy_(flat)
    return buf[off:off + flat.numel()].view(g.shape)


def call(store, name, t, mode, dev, req, bags, w, grad, alpha=1.0, woff=0, wait=True, stream=None):
    """one pooled accumulate -> (total, None) or (None, (message, last_bad_index))"""
    def idx(a):
        return torch.from_numpy(np.asarray(a, np.int64)).cuda() if dev else np.asarray(a, np.int64)
    b = None if bags is None else idx(bags)
    wv = None
    if w is not None:
        wv = to_torch(w, t)
        if dev:
            wv = grad_tensor(w, t, woff)
    pm = "mean" if mode == pl.POOL_MEAN else "sum"
    try:
        if "sample_ids" in req:
            n = store.accumulate_samples_pooled(name, idx(req["sample_ids"]), grad, bags=b, mode=pm, weights=wv,
                                                alpha=alpha, stream=stream, wait=wait)
        else:
            n = store.accumulate_batch_pooled(name, idx(req["starts"]), idx(req["counts"]) if "counts" in req else None,
                                              count=req.get("fixed_count"), grad=grad, bags=b, mode=pm, weights=wv,
                                              alpha=alpha, stream=stream, wait=wait)
        return n, None
    except ValueError as e:
        return None, (str(e), store.last_bad_index)


def check_touched_once(got, start, writes, t, what):
    """every row touched at most once: touched elements admissible for start + contribution, the others unchanged"""
    rows = pao.per_row(writes)
    assert all(len(c) == 1 for c in rows.values()), "rows touched more than once"
    keys = sorted(rows)
    untouched = np.ones(start.shape[0], bool)
    for r, row in keys:
        untouched[row] = False
    assert np.array_equal(ao.keys(got[untouched], t), ao.keys(start[untouched], t)), f"{what}: untouched rows changed"
    if keys:
        sel = [row for _, row in keys]
        c = np.stack([rows[k][0] for k in keys])
        v = ao.verdict(got[sel].reshape(-1), start[sel].reshape(-1), [c.reshape(-1)], t, what=what)
        assert v is None, v


def torch_contributions(g, t, mode, req, bags, w, alpha, nrows_total):
    """torch's CUDA expression on the expanded tensors: ((g.float()[bag] * w) / n * alpha).to(dtype), one row per
    (valid) request row, in the oracle's write order (every request here is valid)"""
    up = torch.float64 if t == pl.ACC_F64 else torch.float32
    counts = np.asarray(req["counts"]) if "counts" in req else np.full(len(req["starts"]), req.get("fixed_count", 1))
    nreq = len(counts)
    bb = bag_offsets(None, [1] * nreq) if bags is None else np.asarray(bags)
    bag_of_req = np.repeat(np.arange(len(bb) - 1), np.diff(bb))
    rows_req = np.repeat(np.arange(nreq), counts)
    gt = to_torch(g, t).cuda().to(up)
    x = gt[torch.from_numpy(bag_of_req[rows_req]).cuda()]
    if w is not None:
        x = x * to_torch(w, t).cuda().to(up)[torch.from_numpy(rows_req).cuda()][:, None]
    if mode == pl.POOL_MEAN:
        n = np.add.reduceat(counts, bb[:-1]) if nreq else np.zeros(0, np.int64)
        n = np.where(np.diff(bb) > 0, n, 1)
        x = x / torch.from_numpy(n[bag_of_req[rows_req]].astype(np.float64)).cuda().to(up)[:, None]
    return (x * alpha).to(TORCH_DT[t])


def bits(x, t):
    return x.contiguous().view(INT_VIEW[SIZE[t]]).cpu().numpy().view(pl.BITS[t])


def same_class(a, b, t):
    """element bits equal, NaNs compared by class"""
    na, nb = np.isnan(pl.decode_bits(a, t)), np.isnan(pl.decode_bits(b, t))
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a), np.where(nb, 0, b))


# ----------------------------------------------------------------------------------------- types, modes, row sizes
@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("row_bytes", [None, 6, 64, 1000, 16384])
def test_types_modes_rows(t, mode, row_bytes):
    """rows each touched once: the oracle's contribution added once, torch's expression on the expanded tensors and
    accumulate_batch of them give the same shard"""
    from ddstore_b200 import PyDDStore
    disp = 1 if row_bytes is None else max(1, row_bytes // SIZE[t])
    if row_bytes == 6:
        disp = 3  # (odd)
    rng = np.random.default_rng(t * 7919 + list(MODES).index(mode) * 101 + disp)
    nrows = 4000 if disp * SIZE[t] <= 1000 else 600
    shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
    sizes = [0, 1, 31, 32, 33, 5, 0, 2] if nrows > 1000 else [0, 1, 3, 33, 2]
    nreq = int(sum(sizes))
    starts, counts = disjoint(rng, nrows, nreq, 3)
    bags = bag_offsets(rng, sizes)
    g = data_bits(rng, t, len(sizes) * disp).reshape(len(sizes), disp)
    w = data_bits(rng, t, nreq, special=False) if mode == "weighted" else None
    alpha = -0.0375
    req = {"starts": starts, "counts": counts}
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        add_var(store, "y", shard, t)
        for off in (0, 1):  # 16-byte aligned grad (vector path where rows allow), then one element past it
            before = shard_bits(store, "x", nrows, disp, t)
            gt = grad_tensor(g, t, off)
            g_before = bits(gt, t).copy()
            n, err = call(store, "x", t, MODES[mode], True, req, bags, w, gt, alpha, woff=off)
            assert err is None, err
            assert n == len(sizes) * disp * SIZE[t]
            writes, _, eerr = pao.contributions([before], t, MODES[mode], g, bags=bags, weights=w, alpha=alpha, **req)
            assert eerr == (0, -1)
            got = shard_bits(store, "x", nrows, disp, t)
            check_touched_once(got, before, writes, t, f"type {t} {mode} disp {disp} off {off}")
            assert np.array_equal(bits(gt, t), g_before), "grad changed"
            ref = torch_contributions(g, t, MODES[mode], req, bags, w, alpha, nrows)
            exp = np.stack([c for _, _, c in writes]).reshape(-1, disp) if writes else np.zeros((0, disp))
            assert same_class(bits(ref, t).reshape(-1, disp), np.asarray(exp).view(pl.BITS[t]), t), "torch differs"
            # accumulate_batch of the expanded contributions on a twin variable
            ybefore = shard_bits(store, "y", nrows, disp, t)
            if len(ref):
                store.accumulate_batch("y", torch.from_numpy(np.repeat(starts, counts) +
                                                             np.concatenate([np.arange(c) for c in counts])).cuda(),
                                       src=ref.contiguous())
            ygot = shard_bits(store, "y", nrows, disp, t)
            same = ao.keys(ygot, t) == ao.keys(got, t)
            if t == pl.ACC_F32:  # (the flush model admits two results near the subnormal range)
                tiny = (np.abs(ybefore) < 2.0 ** -126) | (np.abs(ygot) < 2.0 ** -125) | (np.abs(got) < 2.0 ** -125)
                same |= tiny
            assert same.all(), f"accumulate_batch of the expanded contributions differs ({int((~same).sum())})"
            ints = np.ascontiguousarray(got).view({2: np.int16, 4: np.int32, 8: np.int64}[SIZE[t]])
            store.put_batch("y", np.arange(nrows), src=torch.from_numpy(ints).cuda())  # (y = x again)
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- request forms, index residency
@pytest.mark.parametrize("form", ["fixed1", "fixed2", "counts", "samples"])
@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("t,mode", [(pl.ACC_F32, "weighted"), (pl.ACC_BF16, "mean"), (pl.ACC_F64, "sum")])
def test_request_forms(form, dev, t, mode):
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(len(form) * 7 + dev + t)
    nrows, disp = 6000, 40
    shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
    sizes = rng.integers(0, 40, 30)
    sizes[3] = 0
    nreq = int(sizes.sum())
    maxc = {"fixed1": 0, "fixed2": 2, "counts": 4, "samples": 4}[form]
    starts, counts = disjoint(rng, nrows, nreq, maxc, 2 if form == "fixed2" else None)
    if form == "samples":
        perm = rng.permutation(nreq)
        table = (starts[perm], counts[perm])
        req = {"sample_ids": np.argsort(perm), "table": table}
    elif form == "counts":
        req = {"starts": starts, "counts": counts}
    else:
        req = {"starts": starts, "fixed_count": 1 if form == "fixed1" else 2}
    g = data_bits(rng, t, len(sizes) * disp).reshape(len(sizes), disp)
    w = data_bits(rng, t, nreq, special=False) if mode == "weighted" else None
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        if form == "samples":
            store.set_sample_index("x", table[0], table[1])
        for bags in (bag_offsets(rng, sizes), None):
            gg = g if bags is not None else data_bits(rng, t, nreq * disp).reshape(nreq, disp)
            before = shard_bits(store, "x", nrows, disp, t)
            n, err = call(store, "x", t, MODES[mode], dev, req, bags, w, grad_tensor(gg, t), 0.5)
            assert err is None, err
            writes, _, _ = pao.contributions([before], t, MODES[mode], gg, bags=bags, weights=w, alpha=0.5, **req)
            check_touched_once(shard_bits(store, "x", nrows, disp, t), before, writes, t, f"{form} dev={dev}")
    finally:
        store.free()
        store.close()


def test_long_bags_among_short_ones():
    """a bag of 20000 requests among short ones (sum, mean), and long mean-pooled samples (row windows of one request)"""
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(5)
    for t, mode, disp in ((pl.ACC_F32, pl.POOL_SUM, 128), (pl.ACC_BF16, pl.POOL_MEAN, 256),
                          (pl.ACC_F64, pl.POOL_MEAN, 9)):
        nrows = 30000
        shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
        store = PyDDStore(device=0)
        try:
            add_var(store, "x", shard, t)
            sizes = [3, 1, 20000, 0, 7, 2]
            nreq = sum(sizes)
            starts, _ = disjoint(rng, nrows, nreq, 0)
            req = {"starts": starts, "fixed_count": 1}
            g = data_bits(rng, t, len(sizes) * disp, special=False).reshape(len(sizes), disp)
            bags = bag_offsets(rng, sizes)
            n, err = call(store, "x", t, mode, True, req, bags, None, grad_tensor(g, t), -1.0)
            assert err is None, err
            writes, ns, _ = pao.contributions([shard], t, mode, g, bags=bags, alpha=-1.0, **req)
            assert ns[2] == 20000
            check_touched_once(shard_bits(store, "x", nrows, disp, t), shard, writes, t, f"long bag, type {t}")
            # samples of 1000 to 3000 rows, one bag each (the frames shape)
            lens = rng.integers(1000, 3000, 8)
            st = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
            store.set_sample_index("x", st, lens)
            before = shard_bits(store, "x", nrows, disp, t)
            g2 = data_bits(rng, t, 8 * disp, special=False).reshape(8, disp)
            n, err = call(store, "x", t, mode, True, {"sample_ids": np.arange(8), "table": (st, lens)}, None, None,
                          grad_tensor(g2, t), 0.25)
            assert err is None, err
            writes, _, _ = pao.contributions([before], t, mode, g2, alpha=0.25, sample_ids=np.arange(8),
                                             table=(st, lens))
            check_touched_once(shard_bits(store, "x", nrows, disp, t), before, writes, t, f"samples, type {t}")
        finally:
            store.free()
            store.close()


# ----------------------------------------------------------------------------------------- duplicates and hot rows
@pytest.mark.parametrize("t", TYPES)
def test_duplicates_and_hot_rows_one_batch(t):
    """exact data (integers, power-of-two alpha): the exact sum, however the atomics are ordered; inexact data with two
    or three contributions per element: acc_oracle's admissible results"""
    from ddstore_b200 import PyDDStore
    rng = np.random.default_rng(40 + t)
    nrows, disp = 64, 24
    lim = {pl.ACC_F32: 8, pl.ACC_F64: 8, pl.ACC_F16: 2, pl.ACC_BF16: 1}[t]
    shard = ao.encode(rng.integers(-lim, lim + 1, (nrows, disp)), t)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        hot = 100 if t in (pl.ACC_F16, pl.ACC_BF16) else 4000
        starts = np.concatenate([rng.integers(0, nrows, 300), np.full(hot, 7)]).astype(np.int64)
        rng.shuffle(starts)
        sizes = np.diff(np.unique(np.concatenate([[0, len(starts)], rng.integers(0, len(starts), 40)])))
        bags = bag_offsets(rng, sizes)
        g = ao.encode(rng.integers(-1, 2, (len(sizes), disp)), t)
        w = ao.encode(rng.integers(-1, 2, len(starts)), t)
        req = {"starts": starts, "fixed_count": 1}
        n, err = call(store, "x", t, pl.POOL_SUM, True, req, bags, w, grad_tensor(g, t), 0.5)
        assert err is None, err
        writes, _, _ = pao.contributions([shard], t, pl.POOL_SUM, g, bags=bags, weights=w, alpha=0.5, **req)
        exp = pao.apply([shard], writes, t)[0]
        got = shard_bits(store, "x", nrows, disp, t)
        assert np.array_equal(ao.keys(got, t), ao.keys(exp, t)), "exact duplicates"
        # inexact: each of 60 rows touched by two or three requests
        before = got
        k = rng.integers(2, 4, 60)
        starts = np.repeat(np.arange(60), k).astype(np.int64)
        rng.shuffle(starts)
        nb = len(starts)
        g = data_bits(rng, t, nb * disp, special=False).reshape(nb, disp)
        req = {"starts": starts, "fixed_count": 1}
        n, err = call(store, "x", t, pl.POOL_SUM, False, req, None, None, grad_tensor(g, t), -0.3)
        assert err is None, err
        writes, _, _ = pao.contributions([before], t, pl.POOL_SUM, g, alpha=-0.3, **req)
        got = shard_bits(store, "x", nrows, disp, t)
        rows = pao.per_row(writes)
        for m in (2, 3):
            sel = sorted(row for (_, row), c in rows.items() if len(c) == m)
            cs = [np.stack([rows[(0, row)][i] for row in sel]).reshape(-1) for i in range(m)]
            v = ao.verdict(got[sel].reshape(-1), before[sel].reshape(-1), cs, t, what=f"{m} contributions")
            assert v is None, v
    finally:
        store.free()
        store.close()


@pytest.mark.parametrize("multi_gpu", [False, True])
def test_four_ranks_into_shared_rows(multi_gpu):
    """four thread-ranks scatter into shared rows of a world with an empty shard (exact data: integer rows and grads,
    power-of-two bags and alpha), each queued with wait=False on a caller stream held busy before it: the next
    epoch_begin completes the queue -- the stream is idle when it returns -- and after its barrier every rank's shard
    is bit for bit the start plus every rank's contributions"""
    P = 4
    if multi_gpu and torch.cuda.device_count() < P:
        pytest.skip("needs one GPU per rank")
    t, disp = pl.ACC_F32, 40
    nrows = [300, 0, 200, 100]
    total = sum(nrows)
    rng = np.random.default_rng(77)
    shards = [ao.encode(rng.integers(-4, 5, (n, disp)), t) for n in nrows]
    plans = []
    for r in range(P):
        g = np.random.default_rng(1000 + r)
        sizes = g.choice([0, 1, 2, 4, 8, 16, 32, 64], 40)
        nreq = int(sizes.sum())
        starts = np.concatenate([g.integers(0, total, nreq - 50), np.full(50, 301)]).astype(np.int64)
        plans.append((bag_offsets(g, sizes), starts, ao.encode(g.integers(-2, 3, (len(sizes), disp)), t),
                      "mean" if r % 2 else "sum"))

    def body(store, r):
        dev = torch.device(f"cuda:{r if multi_gpu else 0}")
        torch.cuda.set_device(dev)
        add_var(store, "x", shards[r], t)
        bags, starts, g, mode = plans[r]
        gt = to_torch(g.reshape(-1), t).to(dev).view(g.shape)
        st, bg = torch.from_numpy(starts).to(dev), torch.from_numpy(bags).to(dev)
        s = torch.cuda.Stream(dev)
        torch.cuda.synchronize(dev)
        with torch.cuda.stream(s):
            torch.cuda._sleep(1_000_000_000)  # (about half a second: the queued launch runs only after it)
        store.accumulate_batch_pooled("x", st, grad=gt, bags=bg, mode=mode, alpha=0.5, stream=s.cuda_stream,
                                      wait=False)
        store.epoch_begin()
        done = s.query()
        got = shard_bits(store, "x", nrows[r], disp, t, device=dev)
        store.epoch_end()
        return done, got

    res = run_world(P, body, devices=list(range(P)) if multi_gpu else None)
    exp = shards
    for bags, starts, g, mode in plans:
        writes, ns, err = pao.contributions(exp, t, MODES[mode], g, bags=bags, alpha=0.5, starts=starts, fixed_count=1)
        assert err == (0, -1)
        exp = pao.apply(exp, writes, t)
    for r in range(P):
        assert res[r][0], f"rank {r}: epoch_begin returned with the queued pooled accumulate still in flight"
        assert np.array_equal(res[r][1], exp[r]), f"rank {r}"


# ----------------------------------------------------------------------------------------- errors
def test_invalid_requests_left_out_of_the_mean():
    from ddstore_b200 import PyDDStore
    t, disp, nrows = pl.ACC_F32, 8, 500
    rng = np.random.default_rng(3)
    shard = ao.encode(rng.integers(-4, 5, (nrows, disp)), t)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        starts, counts = disjoint(rng, nrows, 40, 3)
        starts[[5, 17, 30]] = [nrows + 3, -1, nrows - 1]
        counts[30] = 3  # runs past the end
        bags = np.array([0, 10, 25, 40], np.int64)
        g = ao.encode(rng.integers(-8, 9, (3, disp)) * 6, t)
        for dev in (False, True):
            before = shard_bits(store, "x", nrows, disp, t)
            n, err = call(store, "x", t, pl.POOL_MEAN, dev, {"starts": starts, "counts": counts}, bags, None,
                          grad_tensor(g, t))
            writes, ns, eerr = pao.contributions([before], t, pl.POOL_MEAN, g, bags=bags, starts=starts, counts=counts)
            assert eerr == (po.CODE_COUNT, 5)  # (a start past the world's end is the reference's count error)
            assert err is not None and err[1] == 5 and "Invalid count on target" in err[0], err
            check_touched_once(shard_bits(store, "x", nrows, disp, t), before, writes, t, f"invalid dev={dev}")
    finally:
        store.free()
        store.close()


def test_malformed_bag_writes_nothing_else_applied():
    from ddstore_b200 import PyDDStore
    t, disp, nrows = pl.ACC_F32, 8, 500
    rng = np.random.default_rng(4)
    shard = ao.encode(rng.integers(-4, 5, (nrows, disp)), t)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        starts, _ = disjoint(rng, nrows, 30, 0)
        starts[2] = -5  # an invalid request too: the bag is reported first
        bags = np.array([0, 10, 40, 20, 30], np.int64)  # bags 1 and 2 malformed, requests 10-19 in no bag
        g = ao.encode(rng.integers(-8, 9, (4, disp)), t)
        req = {"starts": starts, "fixed_count": 1}
        # host bags: refused before anything is enqueued
        n, err = call(store, "x", t, pl.POOL_SUM, False, req, bags, None, grad_tensor(g, t))
        assert err is not None and "malformed bag offsets" in err[0] and err[1] == 1, err
        assert np.array_equal(shard_bits(store, "x", nrows, disp, t), shard)
        # device bags: the kernel reports bag 1, applies bags 0 and 2
        n, err = call(store, "x", t, pl.POOL_SUM, True, req, bags, None, grad_tensor(g, t))
        assert err is not None and "malformed bag offsets" in err[0] and err[1] == 1, err
        writes, _, eerr = pao.contributions([shard], t, pl.POOL_SUM, g, bags=bags, **req)
        assert eerr == (pl.CODE_BAG, 1)
        check_touched_once(shard_bits(store, "x", nrows, disp, t), shard, writes, t, "malformed bag")
    finally:
        store.free()
        store.close()


def test_argument_errors_change_nothing():
    from ddstore_b200 import PyDDStore, _capi
    t, disp, nrows = pl.ACC_F32, 6, 100
    shard = ao.encode(np.arange(nrows * disp).reshape(nrows, disp) % 7, t)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        add_var(store, "h", shard, t, placement=1)  # DDS_PLACE_HOST
        add_var(store, "d", ao.encode(np.zeros((nrows, disp)), pl.ACC_F64), pl.ACC_F64)
        starts = torch.arange(4, dtype=torch.int64, device="cuda")
        bags = torch.tensor([0, 2, 4], dtype=torch.int64, device="cuda")
        gbuf = torch.ones(2 * disp + 2, dtype=torch.float32, device="cuda")
        g = gbuf[:2 * disp].view(2, disp)
        L, h = store._L, store._h

        def raw(name=b"x", mode=pl.POOL_SUM, dtype=pl.ACC_F32, alpha=1.0, grad=None, nbytes=2 * disp * 4, flags=None,
                weights=None, nbags=2):
            pool = _capi.Pool(mode, dtype, bags.data_ptr(), nbags, weights)
            total, bad = C.c_int64(0), C.c_int64(-1)
            fl = _capi.SRC_ON_DEVICE | _capi.IDX_ON_DEVICE if flags is None else flags
            rc = L.dds_accumulate_batch_pooled(h, name, starts.data_ptr(), None, 1, 4, C.byref(pool), alpha,
                                               g.data_ptr() if grad is None else grad, nbytes, fl, None,
                                               C.byref(total), C.byref(bad))
            torch.cuda.synchronize()
            return rc, L.dds_last_error().decode() if rc else ""

        cases = {
            "max": dict(mode=pl.POOL_MAX), "mode": dict(mode=9), "dtype": dict(dtype=ao.ACC_I32),
            "itemsize": dict(dtype=pl.ACC_F64), "nan alpha": dict(alpha=float("nan")),
            "inf alpha": dict(alpha=float("inf")), "host src": dict(flags=_capi.IDX_ON_DEVICE),
            "short grad": dict(nbytes=2 * disp * 4 - 1), "null grad": dict(grad=0),
            "unaligned grad": dict(grad=g.data_ptr() + 2, nbytes=2 * disp * 4),
            "unaligned weights": dict(weights=gbuf.data_ptr() + 1), "host": dict(name=b"h"),
            "nbags": dict(nbags=-1), "weights with mean": dict(mode=pl.POOL_MEAN, weights=gbuf.data_ptr()),
        }
        g_before = g.clone()
        for what, kw in cases.items():
            rc, msg = raw(**kw)
            assert rc != 0, what
            if what == "host":
                assert "DDS_PLACE_HOST" in msg, msg
            if what == "max":
                assert "argmax" in msg, msg
            assert np.array_equal(shard_bits(store, "x", nrows, disp, t), shard), what
            assert torch.equal(g, g_before), what
        assert raw()[0] == 0
        assert not np.array_equal(shard_bits(store, "x", nrows, disp, t), shard)
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- queues
def test_queued_with_other_batches():
    """wait=False pooled accumulates interleaved with accumulate_batch, get_batch and get_batch_pooled on one stream:
    wait() reports the queue's total, and a later pooled forward sees every update (exact data)"""
    from ddstore_b200 import PyDDStore
    t, disp, nrows, B, L = pl.ACC_F32, 32, 2000, 64, 8
    rng = np.random.default_rng(9)
    shard = ao.encode(rng.integers(-4, 5, (nrows, disp)), t)
    store = PyDDStore(device=0)
    s = torch.cuda.Stream()
    try:
        add_var(store, "x", shard, t)
        exp = [shard]
        keep = []
        with torch.cuda.stream(s):
            for step in range(4):
                ids = torch.from_numpy(rng.integers(0, nrows, B * L)).cuda()
                bags = torch.arange(0, B * L + 1, L, device="cuda")
                g = torch.from_numpy(rng.integers(-4, 5, (B, disp)).astype(np.float32)).cuda()
                src = torch.from_numpy(rng.integers(-2, 3, (B * L, disp)).astype(np.float32)).cuda()
                packed = torch.empty(B * L * disp * 4, dtype=torch.uint8, device="cuda")
                pooled = torch.empty(B, disp, device="cuda")
                s.synchronize()
                store.get_batch_pooled("x", ids, out=pooled, bags=bags, stream=s.cuda_stream, wait=False)
                store.get_batch("x", ids, out=packed, count=1, stream=s.cuda_stream, wait=False)
                store.accumulate_batch("x", ids, src=src, stream=s.cuda_stream, wait=False)
                store.accumulate_batch_pooled("x", ids, grad=g, bags=bags, mode="mean" if step % 2 else "sum",
                                              alpha=0.25, stream=s.cuda_stream, wait=False)
                keep.append((ids, bags, g, src, packed, pooled))
                ids_np = ids.cpu().numpy()
                e = exp[0].copy()
                np.add.at(e, ids_np, src.cpu().numpy())
                writes, _, _ = pao.contributions([e], t, pl.POOL_MEAN if step % 2 else pl.POOL_SUM, g.cpu().numpy(),
                                                 bags=bags.cpu().numpy(), alpha=0.25, starts=ids_np, fixed_count=1)
                exp = pao.apply([e], writes, t)
        assert store.wait() == B * disp * 4  # (the last batch queued: the pooled accumulate's nbags * R)
        got = shard_bits(store, "x", nrows, disp, t)
        assert np.array_equal(got, exp[0]), "queued updates"
        out = torch.empty(nrows, disp, device="cuda")
        store.get_batch_pooled("x", torch.arange(nrows, device="cuda"), out=out)
        assert np.array_equal(out.cpu().numpy(), got), "a later pooled forward sees the updates"
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- end to end: SGD steps
@pytest.mark.parametrize("mode", ["sum", "weighted", "mean"])
@pytest.mark.parametrize("exact", [True, False])
def test_sgd_steps_match_torch_embedding_bag(mode, exact):
    """K steps of a sharded EmbeddingBag (get_batch_pooled forward, accumulate_batch_pooled(alpha=-lr) backward)
    against nn.EmbeddingBag + torch.optim.SGD: exact on exact data (integer tables and grads, power-of-two lr and bag
    sizes; each step reads rows no earlier step wrote, so no value needs more bits than f32 has), else within 1e-5"""
    from ddstore_b200 import PyDDStore
    torch.manual_seed(1 + exact)
    nrows, disp, B, L, K, lr = 5000, 64, 128, 8, 5, 0.125
    table = torch.randint(-8, 9, (nrows, disp)).float() if exact else torch.randn(nrows, disp)
    ref = torch.nn.EmbeddingBag(nrows, disp, mode="sum" if mode == "weighted" else mode, include_last_offset=True).cuda()
    with torch.no_grad():
        ref.weight.copy_(table)
    opt = torch.optim.SGD(ref.parameters(), lr=lr)
    store = PyDDStore(device=0)
    try:
        add_var(store, "emb", table.numpy(), pl.ACC_F32)
        for step in range(K):
            ids = torch.randint(step * 1000, (step + 1) * 1000, (B * L,), device="cuda") if exact else torch.randint(
                0, nrows, (B * L,), device="cuda")
            bags = torch.arange(0, B * L + 1, L, device="cuda")
            w = (torch.randint(1, 3, (B * L,), device="cuda").float() if exact else
                 torch.rand(B * L, device="cuda") + 0.5) if mode == "weighted" else None
            target = torch.randint(-2, 3, (B, disp), device="cuda").float() if exact else torch.randn(B, disp,
                                                                                                    device="cuda")
            out = torch.empty(B, disp, device="cuda")
            store.get_batch_pooled("emb", ids, out=out, bags=bags, mode="mean" if mode == "mean" else "sum", weights=w)
            grad = out - target  # d/d out of 0.5 * |out - target|^2
            store.accumulate_batch_pooled("emb", ids, grad=grad.contiguous(), bags=bags,
                                          mode="mean" if mode == "mean" else "sum", weights=w, alpha=-lr)
            opt.zero_grad()
            r = ref(ids, bags, per_sample_weights=w)
            ((r - target) ** 2 / 2).sum().backward()
            opt.step()
        got = torch.from_numpy(shard_bits(store, "emb", nrows, disp, pl.ACC_F32)).cuda()
        if exact:
            assert torch.equal(got, ref.weight.detach()), "exact data"
        else:
            assert torch.allclose(got, ref.weight.detach(), rtol=1e-5, atol=1e-5)
    finally:
        store.free()
        store.close()


# ----------------------------------------------------------------------------------------- bindings
def test_cython_binding():
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    t, disp, nrows = pl.ACC_F64, 12, 300
    rng = np.random.default_rng(21)
    shard = ao.encode(rng.integers(-4, 5, (nrows, disp)), t)
    starts, _ = disjoint(rng, nrows, 40, 0)
    bags = np.array([0, 3, 3, 40], np.int64)
    g = ao.encode(rng.integers(-8, 9, (3, disp)), t)
    w = ao.encode(rng.integers(-2, 3, 40), t)
    s = pyd.PyDDStore(None, device=0)
    try:
        s.add("x", shard)
        for dev in (False, True):
            before = np.zeros_like(shard)
            s.get("x", before, 0)
            idx = (lambda a: torch.from_numpy(a).cuda()) if dev else (lambda a: a)
            n = s.accumulate_batch_pooled("x", idx(starts), count=1, grad=grad_tensor(g, t), bags=idx(bags), mode="sum",
                                          weights=to_torch(w, t).cuda() if dev else to_torch(w, t), alpha=0.5)
            assert n == 3 * disp * 8
            got = np.zeros_like(shard)
            s.get("x", got, 0)
            writes, _, _ = pao.contributions([before], t, pl.POOL_SUM, g, bags=bags, weights=w, alpha=0.5,
                                             starts=starts, fixed_count=1)
            assert np.array_equal(got, pao.apply([before], writes, t)[0]), f"cython dev={dev}"
        with pytest.raises(ValueError, match="max"):
            s.accumulate_batch_pooled("x", starts, count=1, grad=grad_tensor(g, t), bags=bags, mode="max")
    finally:
        s.free()


CPP_CHECK = r"""
#include <cuda_runtime.h>
#include <cstdio>
#include <stdexcept>
#include <string>
#include "ddstore_b200.hpp"
int main() {
    DDStore s;
    std::vector<float> f(6 * 3, 1.0f);
    s.add("f", f.data(), 6, 3);
    const long ids[4] = {1, 2, 4, 5}, bags[3] = {0, 3, 4};
    const float g[6] = {3, 6, 9, -2, -4, -8};
    float *dg; long *dids, *dbags;
    cudaMalloc(&dg, 24); cudaMalloc(&dids, 32); cudaMalloc(&dbags, 24);
    cudaMemcpy(dg, g, 24, cudaMemcpyHostToDevice);
    cudaMemcpy(dids, ids, 32, cudaMemcpyHostToDevice);
    cudaMemcpy(dbags, bags, 24, cudaMemcpyHostToDevice);
    // mean: bag 0 (rows 1, 2, 4) gets g[0] / 3 * 2, bag 1 (row 5) g[1] * 2
    if (s.accumulate_batch_pooled("f", dids, nullptr, 1, 4, DDS_POOL_MEAN, DDS_ACC_F32, dbags, 2, nullptr, 2.0, dg, 24)
        != 24) return 2;
    // host indices, one request of two rows, a bag per request: rows 0 and 1 get g[0] (sum, alpha 1)
    const long st[1] = {0}, ct[1] = {2};
    if (s.accumulate_batch_pooled("f", st, ct, 0, 1, DDS_POOL_SUM, DDS_ACC_F32, nullptr, 1, nullptr, 1.0, dg, 12, false)
        != 12) return 3;
    try { s.accumulate_batch_pooled("f", dids, nullptr, 1, 4, DDS_POOL_MAX, DDS_ACC_F32, dbags, 2, nullptr, 1.0, dg, 24);
          return 4; }
    catch (std::exception &e) { if (std::string(e.what()).find("argmax") == std::string::npos) return 6; }
    std::vector<float> got(6 * 3);
    s.get("f", 0, 6, got.data());
    const float exp[18] = {4, 7, 10, 6, 11, 16, 3, 5, 7, 1, 1, 1, 3, 5, 7, -3, -7, -15};
    for (int i = 0; i < 18; i++) if (got[i] != exp[i]) { printf("element %d: %g\n", i, got[i]); return 5; }
    s.free();
    printf("cpp pooled accumulate ok\n");
    return 0;
}
"""


def test_cpp_binding(tmp_path):
    src = tmp_path / "pool_acc_check.cpp"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "pool_acc_check")
    lib = os.path.join(ROOT, "ddstore_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
           "-L", lib, "-lddstore_b200", f"-Wl,-rpath,{lib}", "-L", "/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "cpp pooled accumulate ok" in r.stdout, r.stdout + r.stderr
