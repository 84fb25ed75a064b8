"""The first-invalid-request contract (-m gpu) on every fetch path and destination: a batch with invalid requests raises
the reference's error for the FIRST (lowest-index) one with its index in last_bad_index, and leaves exactly what the
serial get() loop that stops at the exception leaves -- the requests before it delivered, nothing else of the
destination touched (a device destination may also receive later VALID requests, each at the offset the store packs it
to). A capacity error touches nothing, and an invalid request wins over it. The next valid call on the same store and
destination works. Requests are classified by the NumPy oracle (np_locate, with the documented divergences: negative
and overflowing counts are "Invalid count on target")."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from tests.gpu_helpers import CODE_SAMPLE, INT64_MAX, Dest, Expected, check_dest, classify, expect_raise, run_world

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one world: 4 owners, owner 1 empty (a request can straddle across it), 24-byte rows (6 x float32)
NROWS = [40_000, 0, 50_000, 10_000]
LL = np.cumsum(NROWS)
TOTAL = int(LL[-1])
DISP, ROW = 6, 24
SENT = 0xA5


def _world(seed=7):
    rng = np.random.default_rng(seed)
    shards = [rng.integers(0, 2**32, size=(n, DISP), dtype=np.uint32).view(np.float32) for n in NROWS]
    allrows = np.concatenate([s.reshape(-1).view(np.uint8) for s in shards])
    return shards, allrows


def _torch():
    import torch
    return torch


def run_rank0(P, body, **kw):
    """run_world where rank 0 does the work and the other ranks only serve their shards until it is done (the
    collective free() waits for rank 0, so no barrier times out while it checks)"""
    done = threading.Event()

    def wrapped(store, r):
        try:
            return body(store, r)
        finally:
            if r == 0:
                done.set()
            else:
                done.wait(600)

    return run_world(P, wrapped, **kw)


# ------------------------------------------------------------------------------- the invalid-request generator
# (start, count) of each kind in the world above; `None` count: the batch's fixed count
def invalid_request(kind, rng, count=None):
    c = count if count is not None else 1
    if kind == "start_neg":
        return -int(rng.integers(1, 1000)), c
    if kind == "start_total":  # owner-0 fall-back: a count error, not a start error
        return TOTAL, c
    if kind == "start_past":
        return TOTAL + int(rng.integers(1, 1000)), c
    if kind == "straddle":  # owner 2 into owner 3
        return int(LL[2]) - 1, max(c, 2)
    if kind == "straddle_empty":  # owner 0 across the empty owner 1 into owner 2
        return int(LL[0]) - 1, max(c, 2)
    if kind == "past_end":
        return TOTAL - 1, max(c, 2)
    if kind == "zero_at_total":  # invalid when P > 1
        return TOTAL, 0
    if kind == "neg_count":
        return int(rng.integers(0, TOTAL)), -int(rng.integers(1, 5))
    if kind == "overflow":  # start + count overflows int64
        s = int(rng.integers(1, TOTAL))
        return s, INT64_MAX - s + int(rng.integers(1, 3))
    if kind == "overflow_max":
        return int(rng.integers(0, TOTAL)), INT64_MAX
    raise ValueError(kind)


FIXED_KINDS = ["start_neg", "start_total", "start_past", "straddle", "straddle_empty", "past_end"]
VAR_KINDS = FIXED_KINDS + ["zero_at_total", "neg_count", "overflow", "overflow_max"]


def valid_requests(rng, B, max_count):
    """B requests within one owner each (owners 0, 2, 3), counts 0..max_count"""
    own = rng.choice([0, 2, 3], size=B)
    lo = np.where(own == 0, 0, LL[np.maximum(own - 1, 0)])
    hi = LL[own]
    c = rng.integers(0, max_count + 1, size=B)
    s = lo + (rng.random(B) * (hi - lo - c + 1)).astype(np.int64)
    return s.astype(np.int64), c.astype(np.int64)


def placements(B, rng):
    """positions of invalid requests: lanes 0, 31 and 32 of a walk window, the first and the last request, and (large
    batches) ~1 % density in the second half, whose lowest one lands in a late-claimed segment"""
    base = 64 if B > 96 else 0
    out = {"lane0": [base], "lane31": [base + 31] if base + 31 < B else [B - 1],
           "lane32": [base + 32] if base + 32 < B else [B - 1], "first": [0], "last": [B - 1],
           "first_and_last": [0, B - 1], "lane32_then_lane0": [base + 32, base + 96] if base + 96 < B else [B - 1]}
    if B >= 4096:
        out["density"] = sorted(rng.choice(np.arange(B // 2, B), size=B // 100, replace=False).tolist())
    return out


def _call_get_batch(store, dest, starts, counts, fixed_count, idx_dev, offsets=None):
    torch = _torch()
    if idx_dev:
        s = torch.from_numpy(np.ascontiguousarray(starts)).cuda()
        c = None if counts is None else torch.from_numpy(np.ascontiguousarray(counts)).cuda()
        torch.cuda.synchronize()
    else:
        s, c = starts, counts
    return lambda: store.get_batch("v", s, c, out=dest.view, count=fixed_count, offsets=offsets)


def _repair(starts, counts, codes, fixed_count=None):
    """the same batch with every invalid request replaced by a valid one"""
    s, c = starts.copy(), None if counts is None else counts.copy()
    bad = np.nonzero(codes)[0]
    s[bad] = 1000 + bad % 1000
    if c is not None:
        c[bad] = 1
    return s, c


def _run_case(store, shards, allrows, dest, starts, counts, fixed_count, idx_dev, what, with_offsets=False):
    """one erroneous call, its checks, then the repaired batch through the same destination"""
    torch = _torch()
    cnt = np.full(len(starts), fixed_count, np.int64) if counts is None else counts
    exp = Expected(allrows, ROW, LL, starts, cnt, counts is None, shards=shards)
    over = exp.T > dest.nbytes
    offs = None
    if with_offsets:
        offs = (torch.full((len(starts) + 1,), -7, dtype=torch.int64, device="cuda") if dest.kind == "device"
                else np.full(len(starts) + 1, -7, np.int64))
    dest.reset()
    expect_raise(store, _call_get_batch(store, dest, starts, counts, fixed_count, idx_dev, offs), exp, over, what)
    check_dest(dest, exp, over, what, offsets=None if over else offs)
    # the next valid call on the same store, placement and destination
    s2, c2 = _repair(starts, counts, exp.codes)
    cnt2 = np.full(len(s2), fixed_count, np.int64) if c2 is None else c2
    exp2 = Expected(allrows, ROW, LL, s2, cnt2, c2 is None)
    if exp2.T > dest.nbytes or exp2.bad >= 0:
        return exp
    dest.reset()
    expect_raise(store, _call_get_batch(store, dest, s2, c2, fixed_count, idx_dev), exp2, False, what + " / next valid call")
    check_dest(dest, exp2, False, what + " / next valid call")
    return exp


# ------------------------------------------------------------------------------- fixed-count batches
# (B, destination kind, device indices): host destinations of <= 64 KiB use the pinned bounce buffer, larger pinned ones
# the HBM staging buffer + one D2H copy, pageable ones of >= 4 MiB the pipelined pageable copy
FIXED_CASES = [(3, "device", False), (3, "pinned", False), (3, "pageable", True), (9, "device", True), (9, "pinned", False),
               (9, "pageable", True), (4096, "device", True), (4096, "pinned", False), (4096, "pinned", True),
               (4096, "pageable", False), (200_000, "device", True), (200_000, "pageable", False),
               (200_000, "pinned", True)]


def test_fixed_count_first_invalid_request():
    """fixed count 2 (so requests can straddle), B = 3, 9 (one past the zero-copy index limit), 4096 and 200 000, errors
    of every start kind at lanes 0 / 31 / 32 of a walk window, first, last, and ~1 % density"""
    torch = _torch()
    shards, allrows = _world()

    def body(store, r):
        store.add("v", shards[r])
        if r:
            return True
        rng = np.random.default_rng(11)
        for B, kind, idx_dev in FIXED_CASES:
            dest = Dest(torch, kind, B * 2 * ROW, SENT, off=B % 5)
            base, _ = valid_requests(rng, B, 2)
            base = np.where(np.isin(base, LL - 1), base - 1, base)  # (a count of 2 must fit in the owner)
            for k, (pname, pos) in enumerate(placements(B, rng).items()):
                if B == 200_000 and pname not in ("lane32", "last", "density"):
                    continue
                starts = base.copy()
                for j, i in enumerate(pos):
                    starts[i] = invalid_request(FIXED_KINDS[(k + j) % len(FIXED_KINDS)], rng, 2)[0]
                _run_case(store, shards, allrows, dest, starts, None, 2, idx_dev,
                          f"fixed B={B} {kind} idx_dev={idx_dev} {pname}", with_offsets=(k % 2 == 0))
        return True

    assert all(run_rank0(4, body))


def test_fixed_count_with_nothing_to_walk():
    """the fixed entry's check pass (count 0, a negative or an overflowing count, a destination too small): the first
    invalid request is still the error, an invalid request wins over the capacity error, nothing is written"""
    torch = _torch()
    shards, allrows = _world()

    def body(store, r):
        store.add("v", shards[r])
        if r:
            return True
        rng = np.random.default_rng(12)
        for B in (5, 3000):
            base, _ = valid_requests(rng, B, 1)
            base = np.where(np.isin(base, LL - 1), base - 1, base)
            with_bad = base.copy()
            with_bad[B // 2] = TOTAL + 3
            with_bad[B - 1] = -4
            for kind in ("device", "pinned", "pageable"):
                for starts, tag in ((base, "valid"), (with_bad, "invalid")):
                    for count, cap in ((0, B * ROW), (-1, B * ROW), (-INT64_MAX, B * ROW), (INT64_MAX, B * ROW),
                                       (INT64_MAX // ROW + 1, B * ROW), (TOTAL + 1, B * ROW), (2, 2 * B * ROW - 1)):
                        dest = Dest(torch, kind, cap, SENT, off=3)
                        _run_case(store, shards, allrows, dest, starts, None, count, kind != "pageable",
                                  f"fixed nothing-to-walk B={B} count={count} cap={cap} {kind} {tag}")
        return True

    assert all(run_rank0(4, body))


# ------------------------------------------------------------------------------- variable counts
def _var_batch(rng, B, max_count, pos, kinds):
    s, c = valid_requests(rng, B, max_count)
    for j, i in enumerate(pos):
        s[i], c[i] = invalid_request(kinds[j % len(kinds)], rng, int(rng.integers(1, 4)))
    return s, c


def var_scenario(store, shards, allrows, sizes, seed):
    """variable-count batches of the given sizes with errors at the plan's edges, into every destination kind"""
    torch = _torch()
    rng = np.random.default_rng(seed)
    for B in sizes:
        edges = {"first": [0], "last": [B - 1], "lane31": [min(31, B - 1)], "lane32": [min(32, B - 1)]}
        if B > 1024:
            edges["tile_edge"] = [1023, 1024]
            edges["tile1_only"] = [1024, B - 1]
        if B > 34 * 1024:
            edges["tiles33_34"] = [33 * 1024 + 7, 34 * 1024 + 3]
            edges["tile34_only"] = [34 * 1024, 34 * 1024 + 1]  # the look-back passes a whole 32-tile window
        if B >= 4096:
            edges["density"] = sorted(rng.choice(np.arange(B // 2, B), size=B // 100, replace=False).tolist())
        for k, (pname, pos) in enumerate(edges.items()):
            j0 = (3 * k + B) % len(VAR_KINDS)  # (so that small batches meet every kind too)
            kinds = VAR_KINDS[j0:] + VAR_KINDS[:j0]
            starts, counts = _var_batch(rng, B, 12 if B > 30_000 else 3, pos, kinds)
            cap = int(np.clip(counts, 0, TOTAL).sum()) * ROW + 8
            for kind, idx_dev in (("device", k % 2 == 0), ("pinned", False), ("pageable", True), ("pinned", True)):
                dest = Dest(torch, kind, cap, SENT, off=(B + k) % 7)
                _run_case(store, shards, allrows, dest, starts, counts, None, idx_dev,
                          f"var B={B} {kind} idx_dev={idx_dev} {pname}", with_offsets=(k % 2 == 1))
            # too small by one byte for the valid requests: the invalid one still wins, nothing is written
            exp = Expected(allrows, ROW, LL, starts, counts, False)
            dest = Dest(torch, "device", max(exp.T - 1, 0), SENT, off=1)
            _run_case(store, shards, allrows, dest, starts, counts, None, True, f"var B={B} capacity-1 {pname}")


def test_variable_count_first_invalid_request():
    """shared-memory plan (<= 1024 requests) and plan kernel (1025, 8193 and 33 x 1024 + 5 requests: the look-back
    crosses a 32-tile window) with errors at 1023 / 1024 and in tiles 33 / 34, every invalid kind, every destination"""
    shards, allrows = _world()

    def body(store, r):
        store.add("v", shards[r])
        if r:
            return True
        var_scenario(store, shards, allrows, (5, 700, 1024, 1025, 8193, 33 * 1024 + 5), 21)
        return True

    assert all(run_rank0(4, body))


def test_zero_count_at_the_end_is_valid_on_one_owner_only():
    """(total, 0) is valid when there is one owner (no fall-back) and a count error with more than one"""
    torch = _torch()
    shard = np.arange(100 * DISP, dtype=np.float32).reshape(100, DISP)

    def body(store, r):
        store.add("v", shard)
        for kind in ("device", "pinned"):
            d = Dest(torch, kind, 3 * ROW, SENT)
            assert store.get_batch("v", [3, 100, 98], [1, 0, 2], out=d.view) == 3 * ROW
            got = d.host()[64:64 + 3 * ROW]
            assert got.tobytes() == shard[[3, 98, 99]].tobytes()
        return True

    assert all(run_world(1, body))


# ------------------------------------------------------------------------------- sample ids
def test_sample_ids_first_invalid_request():
    """get_samples with ids below 0 / at or above nsamples, and valid ids whose table entry is invalid (straddling,
    past the end, negative start, negative or overflowing count); the table registered from the host and from the
    device (then a host destination learns the packed size from the device)"""
    torch = _torch()
    shards, allrows = _world()
    rng = np.random.default_rng(31)
    nsamp = 6000
    tst, tct = valid_requests(rng, nsamp, 4)
    poison = {6000 - 1: (int(LL[0]) - 1, 2), 6000 - 2: (TOTAL - 1, 3), 6000 - 3: (-5, 1), 6000 - 4: (10, -2),
              6000 - 5: (10, INT64_MAX), 6000 - 6: (int(LL[2]) - 2, 3), 6000 - 7: (TOTAL, 0)}
    for i, (s, c) in poison.items():
        tst[i], tct[i] = s, c

    def body(store, r):
        store.add("v", shards[r])
        if r:
            return True
        for table_dev in (False, True):
            if table_dev:
                store.set_sample_index("v", torch.from_numpy(tst).cuda(), torch.from_numpy(tct).cuda())
            else:
                store.set_sample_index("v", tst, tct)
            for B in (6, 700, 9000):
                edges = {"first": [0], "lane32": [min(32, B - 1)], "last": [B - 1]}
                if B > 1024:
                    edges["tile_edge"] = [1023, 1024]
                for k, (pname, pos) in enumerate(edges.items()):
                    ids = rng.integers(0, nsamp - 10, size=B).astype(np.int64)
                    bad_ids = [-1, nsamp, nsamp + 7, -INT64_MAX] + sorted(poison)
                    for j, i in enumerate(pos):
                        ids[i] = bad_ids[(k + j) % len(bad_ids)]
                    inside = (ids >= 0) & (ids < nsamp)
                    st = np.where(inside, tst[np.clip(ids, 0, nsamp - 1)], 0)
                    ct = np.where(inside, tct[np.clip(ids, 0, nsamp - 1)], 0)
                    codes = np.where(inside, classify(LL, st, ct), CODE_SAMPLE)
                    exp = Expected(allrows, ROW, LL, st, ct, False, codes=codes)
                    good = np.where(codes != 0, 5, ids)  # the next valid call
                    exp2 = Expected(allrows, ROW, LL, tst[good], tct[good], False)
                    cap = max(int(np.clip(ct, 0, TOTAL).sum()) * ROW, exp2.T) + 4
                    for kind, idx_dev in (("device", True), ("pinned", False), ("pageable", False), ("pageable", True)):
                        what = f"samples table_dev={table_dev} B={B} {kind} idx_dev={idx_dev} {pname}"
                        dest = Dest(torch, kind, cap, SENT, off=k % 3)
                        offs = None
                        if k % 2:
                            offs = (torch.full((B + 1,), -7, dtype=torch.int64, device="cuda") if kind == "device"
                                    else np.full(B + 1, -7, np.int64))
                        d_ids = torch.from_numpy(ids).cuda() if idx_dev else ids
                        torch.cuda.synchronize()
                        expect_raise(store, lambda: store.get_samples("v", d_ids, dest.view, offsets=offs), exp, False, what)
                        check_dest(dest, exp, False, what, offsets=offs)
                        dest.reset()
                        assert store.get_samples("v", good, dest.view) == exp2.T
                        check_dest(dest, exp2, False, what + " / next valid call")
        return True

    assert all(run_rank0(4, body))


def test_multi_array_first_invalid_request():
    """get_samples_multi: the reported request is the first invalid one in variable order, then sample order (the
    lowest variable with an invalid entry, the lowest sample position in it); last_bad_index is its position in the id
    list. Variables before it are delivered whole, it up to that sample; later bytes are the sentinel or valid rows."""
    torch = _torch()
    rng = np.random.default_rng(41)
    nsamp = 3000
    rows = (1, 3, 2)  # rows per sample unit of the three variables
    worlds = []
    for v, rp in enumerate(rows):
        n = [int(x) * rp for x in NROWS]
        ll = np.cumsum(n)
        sh = [rng.integers(0, 2**32, size=(k, DISP), dtype=np.uint32).view(np.float32) for k in n]
        st = np.sort(rng.integers(0, int(ll[-1]) - 8, size=nsamp))
        st = np.where(np.isin(st + 3, ll) | np.isin(st + 2, ll) | np.isin(st + 1, ll), st - 4, st)
        ct = rng.integers(0, 4, size=nsamp)
        # sample nsamp - 1 - v is invalid in variable v only
        st[nsamp - 1 - v], ct[nsamp - 1 - v] = int(ll[0]) - 1, 3
        worlds.append((sh, np.concatenate([s.reshape(-1).view(np.uint8) for s in sh]), ll, st, ct))

    def body(store, r):
        names = [f"m{v}" for v in range(3)]
        for v in range(3):
            store.add(names[v], worlds[v][0][r])
            store.set_sample_index(names[v], worlds[v][3], worlds[v][4])
        if r:
            return True
        cases = [({0: nsamp - 1}, "var 0"), ({5: nsamp - 2}, "var 1"), ({7: nsamp - 3}, "var 2"),
                 ({3: nsamp - 3, 50: nsamp - 1}, "var 2 first, var 0 later"),
                 ({2: nsamp - 2, 9: nsamp - 1, 1: nsamp - 3}, "all three"), ({4: nsamp + 2}, "id out of range")]
        for B in (37, 5000):
            for placement, name in cases:
                ids = rng.integers(0, nsamp - 10, size=B).astype(np.int64)
                for j, sid in placement.items():
                    ids[j if B > 37 else j % B] = sid
                exps, codes = [], []
                for v in range(3):
                    sh, allr, ll, st, ct = worlds[v]
                    inside = (ids >= 0) & (ids < nsamp)
                    s_ = np.where(inside, st[np.clip(ids, 0, nsamp - 1)], 0)
                    c_ = np.where(inside, ct[np.clip(ids, 0, nsamp - 1)], 0)
                    cv = np.where(inside, classify(ll, s_, c_), CODE_SAMPLE)
                    codes.append(cv)
                    exps.append(Expected(allr, ROW, ll, s_, c_, False, codes=cv))
                flat = np.concatenate(codes)
                fb = np.nonzero(flat)[0]
                vbad, jbad = divmod(int(fb[0]), B)
                good = np.where(np.any(np.stack(codes), axis=0), 5, ids)  # the next valid call
                goods = [Expected(w[1], ROW, w[2], w[3][good], w[4][good], False) for w in worlds]
                dests = [Dest(torch, "device", max(e.T, g.T) + 5, SENT, off=v) for v, (e, g) in enumerate(zip(exps, goods))]
                offs = [torch.full((B + 1,), -7, dtype=torch.int64, device="cuda") for _ in range(3)]
                what = f"multi B={B} {name}"
                try:
                    store.get_samples_multi(names, ids, [d.view for d in dests], offsets=offs)
                    got = None
                except ValueError as ex:
                    got = str(ex)
                want = "sample id" if flat[fb[0]] == CODE_SAMPLE else {2: "Invalid start on target", 3: "Invalid count on target"}[int(flat[fb[0]])]
                assert got is not None and want in got, f"{what}: raised {got!r}, oracle {want!r}"
                assert store.last_bad_index == jbad, f"{what}: last_bad_index {store.last_bad_index}, oracle {jbad} (variable {vbad})"
                for v in range(3):
                    e = exps[v]
                    # the variable-major serial loop: variables before vbad whole, vbad up to jbad, later ones nothing
                    e.bad = -1 if v < vbad else (jbad if v == vbad else 0)
                    e.prefix = e.T if v < vbad else int(e.offs[e.bad])
                    check_dest(dests[v], e, False, f"{what} variable {v}", offsets=offs[v])
                for d in dests:
                    d.reset()
                totals = store.get_samples_multi(names, good, [d.view for d in dests])
                for v, e in enumerate(goods):
                    assert totals[v] == e.T
                    check_dest(dests[v], e, False, f"{what} variable {v} / next valid call")
        return True

    assert all(run_rank0(4, body))


# ------------------------------------------------------------------------------- queues
def test_queue_reports_the_first_failing_batch():
    """queued fixed and variable batches, plain and overlapped: wait() reports the earliest failing batch in queue order
    with that batch's first invalid index -- also when a later batch fails at a lower index, and when the earlier
    failure is a capacity error; every batch's destination holds what it may; the queue then runs on"""
    torch = _torch()
    shards, allrows = _world()

    def body(store, r):
        store.add("v", shards[r])
        if r:
            return True
        rng = np.random.default_rng(51)
        side = torch.cuda.Stream()
        st = side.cuda_stream
        B = 3000
        for fixed in (True, False):
            for overlap in (False, True):
                clean = []
                for k in range(5):
                    s, c = valid_requests(rng, B, 2 if fixed else 3)
                    if fixed:
                        s = np.where(np.isin(s, LL - 1), s - 1, s)
                        c = np.full(B, 2, np.int64)
                    clean.append((s, c))
                for first_fail in ("invalid", "capacity"):
                    batches = [(s.copy(), c.copy()) for s, c in clean]
                    # batch 1 fails at 500 (or is one byte too small), batch 2 at 7 -- a lower index --, batch 3 at 100
                    for k, i, kind in ((1, 500, "start_past"), (2, 7, "straddle"), (3, 100, "start_neg")):
                        if k == 1 and first_fail == "capacity":
                            continue
                        batches[k][0][i], cc = invalid_request(kind, rng, 2)
                        if not fixed:
                            batches[k][1][i] = cc
                    exps = [Expected(allrows, ROW, LL, s, c, fixed) for s, c in batches]
                    caps = [e.T + 16 for e in exps]
                    if first_fail == "capacity":  # batch 1 too small by one byte
                        caps[1] = exps[1].T - 1
                    dests = [Dest(torch, "device", caps[k], SENT, off=k) for k in range(5)]
                    d_s = [torch.from_numpy(s).cuda() for s, _ in batches]
                    d_c = [torch.from_numpy(c).cuda() for _, c in batches]
                    torch.cuda.synchronize()
                    for k in range(5):
                        if fixed:
                            store.get_batch("v", d_s[k], out=dests[k].view, count=2, stream=st, wait=False, overlap=overlap)
                        else:
                            store.get_batch("v", d_s[k], d_c[k], out=dests[k].view, stream=st, wait=False, overlap=overlap)
                    what = f"queue fixed={fixed} overlap={overlap} first failure {first_fail}"
                    with pytest.raises(ValueError) as ei:
                        store.wait()
                    if first_fail == "invalid":
                        assert str(ei.value) == "Invalid count on target", f"{what}: {ei.value} (batch 1 fails at 500)"
                        assert store.last_bad_index == 500, f"{what}: last_bad_index {store.last_bad_index}, batch 1 fails at 500"
                    else:
                        assert "too small" in str(ei.value), f"{what}: {ei.value}"
                        assert store.last_bad_index == -1, what
                    side.synchronize()
                    for k in range(5):
                        check_dest(dests[k], exps[k], caps[k] < exps[k].T, f"{what}: batch {k}")
                    # the queue runs on: a valid queue through the same destinations
                    for k in (0, 4, 0, 4):
                        if fixed:
                            store.get_batch("v", d_s[k], out=dests[k].view, count=2, stream=st, wait=False, overlap=overlap)
                        else:
                            store.get_batch("v", d_s[k], d_c[k], out=dests[k].view, stream=st, wait=False, overlap=overlap)
                    assert store.wait() == exps[4].T
                    for k in (0, 4):
                        check_dest(dests[k], exps[k], False, f"{what}: batch {k} after the failing queue")
        return True

    assert all(run_rank0(4, body))


# ------------------------------------------------------------------------------- single requests
def single_scenario(store, torch, names, what_prefix):
    """get() of every invalid kind on the single-request path (host and device destinations, the store's resident
    kernel or dds_small_get_kernel), each followed by a valid get(); an invalid request with a too small destination
    still reports the request"""
    from ddstore_b200 import _capi
    rng = np.random.default_rng(61)
    _, allrows = _world()
    for name in names:
        for kind in ("start_neg", "start_total", "start_past", "straddle", "straddle_empty", "past_end", "zero_at_total",
                     "neg_count", "overflow", "overflow_max"):
            s, c = invalid_request(kind, rng, 2)
            code = int(classify_one(s, c))
            assert code, (kind, s, c)
            for dk in ("pinned", "pageable", "device"):
                dest = Dest(torch, dk, 4 * ROW, SENT, off=1)
                what = f"{what_prefix} get({name}) {kind} {dk}"
                ptr = dest.view.data_ptr() if dk == "device" else dest.view.ctypes.data
                rc = store._L.dds_get(store._h, name.encode(), s, c, 4, ptr, 1 if dk == "device" else 0)
                want = {2: _capi.ERR_START, 3: _capi.ERR_COUNT}[code]
                assert rc == want, f"{what}: rc {rc}, oracle {want}"
                w = dest.host()
                hit = np.nonzero(w != SENT)[0]
                assert hit.size == 0, f"{what}: byte {int(hit[0]) - 65} written"
                # the next valid call: the request right before it, with the same destination
                g = int(rng.integers(0, int(LL[0]) - 4))
                arr = dest.view[:3 * ROW] if dk != "device" else dest.view[:3 * ROW]
                rc = store._L.dds_get(store._h, name.encode(), g, 3, 4, arr.data_ptr() if dk == "device" else arr.ctypes.data,
                                      1 if dk == "device" else 0)
                assert rc == 0, f"{what} / next valid call: rc {rc}"
                got = dest.host()[65:65 + 3 * ROW]
                assert got.tobytes() == allrows[g * ROW:(g + 3) * ROW].tobytes(), f"{what} / next valid call"
        # one request, too small a destination: the invalid request wins; a valid one is a capacity error, nothing written
        for s, c, want in ((TOTAL + 1, 3, "Invalid count on target"), (-1, 3, "Invalid start on target"), (4, 3, "too small")):
            dest = Dest(torch, "pinned", 2 * ROW, SENT)
            with pytest.raises(ValueError) as ei:
                store.get_batch(name, [s], out=dest.view, count=c)
            assert want in str(ei.value), f"{what_prefix} {name} ({s}, {c}) into {2 * ROW} B: {ei.value}"
            assert store.last_bad_index == (-1 if want == "too small" else 0)
            assert not np.any(dest.host() != SENT), f"{what_prefix} {name} ({s}, {c}): destination written"


def classify_one(s, c):
    return classify(LL, [s], [c])[0]


def test_single_request_errors_through_the_resident_kernel_and_the_1cta_kernel():
    """the doorbell kernel (the default), and dds_small_get_kernel for a variable past the 256th of a store (the
    resident kernel's table has 256 slots)"""
    torch = _torch()
    shards, _ = _world()

    def body(store, r):
        store.add("v", shards[r])
        for k in range(256):
            store.add(f"pad{k}", np.zeros((1, 1), np.uint8))
        store.add("late", shards[r])  # no doorbell slot left
        if r:
            return True
        single_scenario(store, torch, ["v", "late"], "in-process")
        return True

    assert all(run_rank0(4, body))


ENV_SCRIPT = r"""
import sys, threading
sys.path.insert(0, {root!r})
import numpy as np, torch
from tests import test_gpu_errors as T
from tests.gpu_helpers import run_world
shards, allrows = T._world()
def body(store, r):
    store.add("v", shards[r])
    if r == 0:
        {call}
    return True
assert all(T.run_rank0(4, body))
print("env-ok")
"""

ENV_CASES = {
    "no_doorbell": ({"DDS_DOORBELL": "0"}, "T.single_scenario(store, torch, ['v'], 'DDS_DOORBELL=0')"),
    "smem_plan_8192": ({"DDS_SMEM_PLAN_MAX": "8192"}, "T.var_scenario(store, shards, allrows, (4096, 8192), 22)"),
}


@pytest.mark.parametrize("case", sorted(ENV_CASES))
def test_environment_variants(tmp_path, case):
    """DDS_DOORBELL=0 (every get() launches dds_small_get_kernel) and DDS_SMEM_PLAN_MAX=8192 (4096- and 8192-request
    batches plan in shared memory)"""
    env, call = ENV_CASES[case]
    script = tmp_path / "errors_env.py"
    script.write_text(ENV_SCRIPT.format(root=ROOT, call=call))
    r = subprocess.run([sys.executable, str(script)], env=dict(os.environ, **env), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and "env-ok" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
