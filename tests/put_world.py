"""Batched puts on a whole world of shards: workloads, source layouts and the expectation (NumPy only, no GPU).

Everything is a pure function of its arguments, so the thread-ranks of a GPU test and the process that checks them see
the same batches and the same expected world. The bytes a put of epoch e writes are a fixed function of the DESTINATION
byte (`pattern_world`): overlapping and duplicate writes, from one batch or from several ranks, write equal values, so
the expectation is exact whatever order the device applies them in.

A batch is the keyword form tests/put_oracle.py takes: {"starts", "counts"}, {"starts", "fixed_count"} or
{"sample_ids", "table"}. A `Put` is one call of one writer: a batch, the pattern its valid rows carry, and optionally a
src_bytes smaller than its layout (a capacity error).
"""
from collections import namedtuple

import numpy as np

from tests import put_oracle as po

Put = namedtuple("Put", "batch pattern src_bytes", defaults=(None,))
FILL_OUTSIDE = 0xA5  # source filler of an invalid request's bytes that map to no row of the world
EDGE_CLASSES = {"first", "last", "tail", "whole", "zero", "zero_at_total", "body"}
PAIR_CLASSES = {"sides", "straddle"}  # need two non-empty owners
INVALID_CLASSES = {"start_at_total", "start_past_total", "start_negative", "count_negative", "count_over"}
SAMPLE_CLASSES = {"id_negative", "id_nsamples"}


def lenlist_of(nrows):
    return np.cumsum(np.asarray(nrows, np.int64))


def owners(lenlist):
    """(rank, first global row, end row) of every rank that owns rows"""
    lo = np.concatenate([[0], lenlist[:-1]])
    return [(t, int(a), int(b)) for t, (a, b) in enumerate(zip(lo, lenlist)) if b > a]


def pattern_world(seed, lenlist, R, epoch):
    """the world's bytes in global row order: epoch 0 is what the shards hold at first, epoch e >= 1 what every put of
    that epoch writes. Any two epochs differ in EVERY byte, so a byte left from the wrong epoch is always seen."""
    assert 0 <= epoch <= 6
    base = np.random.default_rng([seed, 0x7075]).integers(0, 256, size=int(lenlist[-1]) * R, dtype=np.uint8)
    return base + np.uint8((61 * epoch + (1 if epoch else 0)) % 256)  # (wraps)


def split_world(world, lenlist, R):
    """the world's bytes as one [nrows, R] uint8 shard per rank"""
    lo = np.concatenate([[0], lenlist[:-1]])
    return [world[int(a) * R:int(b) * R].reshape(int(b - a), R).copy() for a, b in zip(lo, lenlist)]


def layout_src(pattern, lenlist, R, batch):
    """the caller's packed source of `batch`: a valid request's rows are the pattern's bytes at its destination. An
    invalid request that keeps bytes gets filler that differs, at every position it would have hit, from the pattern of
    every epoch (pattern + 128; FILL_OUTSIDE where it maps to no row), so a put that wrongly writes it is seen."""
    rows, parts = int(lenlist[-1]), []
    for s, c, ok in po.requests(**batch):
        n = c * R if ok and 0 < c <= rows else 0
        if not n:
            continue
        if po.locate(lenlist, s, c)[0] == 0:
            parts.append(pattern[s * R:s * R + n])
            continue
        fill = np.full(n, FILL_OUTSIDE, np.uint8)
        a, b = max(s, 0), min(s + c, rows)  # the rows of the world it overlaps
        if a < b:
            fill[(a - s) * R:(b - s) * R] = pattern[a * R:b * R] + np.uint8(128)
        parts.append(fill)
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


def layout_total(lenlist, R, batch):
    """bytes of the caller's layout of `batch`"""
    rows = int(lenlist[-1])
    return sum(c * R for _, c, ok in po.requests(**batch) if ok and 0 < c <= rows)


def expected_world(shards, puts, lenlist=None):
    """Apply every writer's puts (puts[w]: list of Put) to `shards` with the oracle -> (new shards, per writer the list
    of (code, bad index, layout total) its calls report). The result does not depend on the order of the writers."""
    lenlist = po.lenlist_of(shards) if lenlist is None else lenlist
    R = shards[0].shape[1] * shards[0].dtype.itemsize
    flat, status = [], []
    for calls in puts:
        for p in calls:
            short = p.src_bytes is not None and p.src_bytes < layout_total(lenlist, R, p.batch)  # nothing is read
            flat.append((np.zeros(0, np.uint8) if short else layout_src(p.pattern, lenlist, R, p.batch), p.src_bytes, p.batch))
    new, triples = po.put_many(shards, flat)
    it = iter(triples)
    for calls in puts:
        status.append([next(it) for _ in calls])
    return new, status


# ------------------------------------------------------------------------------------------------ workloads
def edge_requests(rng, lenlist, writer, first_bad=None, body=24, only=None):
    """One writer's variable-count batch over every owner's edges -> (starts, counts, classes), classes[i] naming what
    request i is. Per owner with rows: its first row, its last row, its last k rows (ending exactly on the boundary),
    the whole shard, zero-count requests at both boundaries; per neighbouring pair of owners one row each side of the
    boundary as two requests ("sides") and, with first_bad, one request straddling it (invalid, keeps 2 rows of
    bytes); a zero-count request at `total`; `body` random valid requests. first_bad=None: only requests the oracle
    accepts. Otherwise the invalid family (start at / past total, start -1, negative count, count above the world's
    rows, the straddlers) is mixed in, the first of them at index `first_bad` exactly. only: the ranks to write to
    (default: every owner)."""
    total = int(lenlist[-1])
    own = [o for o in owners(lenlist) if only is None or o[0] in only]
    good, bad = [], []
    for j, (t, lo, hi) in enumerate(own):
        k = 1 + (writer + j) % min(hi - lo, 5)
        good += [(lo, 1, "first"), (hi - 1, 1, "last"), (hi - k, k, "tail"), (lo, hi - lo, "whole"), (lo, 0, "zero")]
        (good if hi < total else bad).append((hi, 0, "zero" if hi < total else "zero_at_total"))
    for (_, _, hi0), (_, lo1, _) in zip(own, own[1:]):
        if hi0 != lo1:  # (not neighbours)
            continue
        good += [(hi0 - 1, 1, "sides"), (lo1, 1, "sides")]
        bad.append((hi0 - 1, 2, "straddle"))
    for _ in range(body):
        t, lo, hi = own[int(rng.integers(0, len(own)))]
        s = int(rng.integers(lo, hi))
        good.append((s, int(rng.integers(1, min(hi - s, 4) + 1)), "body"))
    bad += [(total, 1, "start_at_total"), (total + 7, 2, "start_past_total"), (-1, 1, "start_negative"),
            (own[0][1], -1, "count_negative"), (0, total + 1, "count_over")]
    # (a zero-count request at `total` is the reference's quirk: valid only when rank 0 owns every row)
    ok = [r for r in good + bad if po.locate(lenlist, r[0], r[1])[0] == 0]
    rej = [r for r in good + bad if po.locate(lenlist, r[0], r[1])[0] != 0]
    reqs = [ok[i] for i in rng.permutation(len(ok))]
    if first_bad is not None:
        assert first_bad <= len(reqs)
        rej = [rej[i] for i in rng.permutation(len(rej))]
        reqs.insert(first_bad, rej[0])
        for r in rej[1:]:
            reqs.insert(int(rng.integers(first_bad + 1, len(reqs) + 1)), r)
    st, ct = np.array([r[:2] for r in reqs], np.int64).T
    return np.ascontiguousarray(st), np.ascontiguousarray(ct), [r[2] for r in reqs]


def as_samples(rng, starts, counts, classes, first_bad=None):
    """the same requests as a by-sample-id batch -> ({"sample_ids", "table"}, classes): the table holds the requests
    in shuffled order plus one sample nobody asks for; with first_bad, ids -1 and nsamples (0 bytes each) go in at
    first_bad and behind it."""
    n = len(starts)
    perm = rng.permutation(n)
    table = (np.append(starts[perm], 0), np.append(counts[perm], 1))
    ids = np.empty(n, np.int64)
    ids[perm] = np.arange(n)
    ids, classes = ids.tolist(), list(classes)
    if first_bad is not None:
        for k, (sid, cls) in enumerate([(-1, "id_negative"), (n + 1, "id_nsamples")]):
            at = first_bad if k == 0 else int(rng.integers(first_bad + 1, len(ids) + 1))
            ids.insert(at, sid)
            classes.insert(at, cls)
    return {"sample_ids": np.array(ids, np.int64), "table": table}, classes


def edge_fixed(rng, lenlist, cnt, first_bad=None, body=24):
    """A fixed-count batch of `cnt` rows per request -> (starts, classes): per owner with >= cnt rows its first and
    its last cnt rows; random valid starts; with first_bad also starts straddling every owner's end (when cnt > 1), at
    `total` and at -1, each keeping cnt rows of bytes, the first at index first_bad."""
    total, good = int(lenlist[-1]), []
    bad = [(total, "start_at_total"), (-1, "start_negative")]
    for t, lo, hi in owners(lenlist):
        if hi - lo >= cnt:
            good += [(lo, "first"), (hi - cnt, "tail")]
            good += [(int(s), "body") for s in rng.integers(lo, hi - cnt + 1, size=max(1, body // len(lenlist)))]
        if cnt > 1:
            bad.append((hi - 1, "straddle"))
    reqs = [good[i] for i in rng.permutation(len(good))]
    if first_bad is not None:
        first_bad = min(first_bad, len(reqs))
        bad = [bad[i] for i in rng.permutation(len(bad))]
        reqs.insert(first_bad, bad[0])
        for r in bad[1:]:
            reqs.insert(int(rng.integers(first_bad + 1, len(reqs) + 1)), r)
    return np.array([r[0] for r in reqs], np.int64), [r[1] for r in reqs]


def interleaved_cover(rng, lenlist, P, R, big=True):
    """A partition of EVERY row of the world into requests of 1..3 rows (with `big`, also one request of a chunk and
    one above 1 MiB per owner that has the rows), dealt round-robin to P writers in row order -- neighbouring requests
    have different writers -- and shuffled inside each writer's batch. -> [(starts, counts)] per writer. Every byte of
    every shard is written exactly once."""
    reqs = []
    for t, lo, hi in owners(lenlist):
        s, small, bigs = lo, 0, ([-(-4096 // R) + 1, -(-(1 << 20) // R) + 1] if big else [])
        while s < hi:
            c, small = int(rng.integers(1, 4)), small + 1
            fit = [b for b in bigs if hi - s >= b + 3]
            if fit and small > 3:  # (small requests on both sides of a big one)
                c, small = fit[-1], 0
                bigs.remove(c)
            c = min(c, hi - s)
            reqs.append((s, c))
            s += c
    out = []
    for w in range(P):
        mine = np.array(reqs[w::P], np.int64).reshape(-1, 2)
        mine = mine[rng.permutation(len(mine))]
        out.append((np.ascontiguousarray(mine[:, 0]), np.ascontiguousarray(mine[:, 1])))
    return out


def dense_cover(rng, nrows, n):
    """exactly n shuffled requests that partition rows [0, nrows) of one shard (n <= nrows): every row written once"""
    cuts = np.sort(rng.choice(np.arange(1, nrows), size=n - 1, replace=False))
    st = np.concatenate([[0], cuts]).astype(np.int64)
    ct = np.diff(np.concatenate([st, [nrows]])).astype(np.int64)
    p = rng.permutation(n)
    return st[p], ct[p]


# ------------------------------------------------------------------------------------------------ comparing a shard
def covering(lenlist, puts, row):
    """the requests whose rows include global row `row`, as "writer w call k request i (start, count)" strings"""
    out = []
    for w, calls in enumerate(puts):
        for k, p in enumerate(calls):
            for i, (s, c, ok) in enumerate(po.requests(**p.batch)):
                if ok and c > 0 and s <= row < s + c:
                    out.append(f"writer {w} call {k} request {i} ({s}, {c})"
                               + ("" if po.locate(lenlist, s, c)[0] == 0 else " [invalid]"))
    return out


def shard_mismatch(got, slack, exp, rank, lenlist, R, puts, what):
    """None when rank `rank`'s raw shard `got` (rows then `slack` bytes) holds exactly the expected rows `exp` and zero
    slack; else a message naming rank, row, byte and the request(s) covering the row"""
    exp = np.asarray(exp).reshape(-1).view(np.uint8)
    payload = exp.size
    assert got.size == payload + slack, (got.size, payload, slack)
    d = np.nonzero(got[:payload] != exp)[0]
    if d.size:
        b = int(d[0])
        row = b // R + (int(lenlist[rank - 1]) if rank else 0)
        cov = covering(lenlist, puts, row)
        return (f"{what}: rank {rank}: {d.size} shard bytes differ, first at local byte {b} (global row {row}, byte {b % R} "
                f"of it): got {int(got[b]):#04x}, expected {int(exp[b]):#04x}; covered by "
                + ("; ".join(cov[:6]) if cov else "no request"))
    z = np.nonzero(got[payload:])[0]
    if z.size:
        return f"{what}: rank {rank}: slack byte {int(z[0])} past the shard's {payload} bytes was written ({int(got[payload + z[0]]):#04x})"
    return None
