"""Batched puts across owners and on densely written shards, against the expectation of tests/put_world.py.

Every case runs thread-ranks (`run_world`), lets every rank put into the others' shards in one epoch and, after the
closing fence, has EVERY rank read its own shard raw -- rows and slack -- and compare it byte for byte with the
expected shard; every rank also checks the (status, bad index, total) of each of its own calls. The expectation is
computed once, before the ranks start. A rank never raises between two fences (the other ranks would wait for it at
the next one): it collects what it found and the test asserts after the world has finished.
"""
from collections import namedtuple

import numpy as np
import pytest

from tests import put_oracle as po
from tests import put_world as pw
from tests.gpu_helpers import error_text, run_world
from tests.test_gpu_put import ERR, SRC_OFFSETS, raw_put, shard_state, to_device
from tests.test_put_world_cpu import sixty_four_rows

pytestmark = pytest.mark.gpu
DT = {1: "uint8", 2: "int16", 4: "int32", 8: "int64"}
# one call of one rank: the put, the entry it goes through -- "host" / "dev": the C-ABI with host / device indices (src
# at any byte offset); "api": put_batch / put_samples with device indices, which raise; "queued": the same with
# wait=False on the rank's own stream, completed by the fence -- and the source's offset past a 16-byte boundary
Call = namedtuple("Call", "put entry off", defaults=("host", 0))
SHAPES = [(1, 1), (1, 3), (2, 3), (4, 5), (8, 3), (4, 37), (8, 512), (1, 65543)]  # (itemsize, disp): 1 .. 65543-byte rows
ROWS = {2: [1, 23], 3: [19, 0, 8], 4: [0, 26, 1, 9]}  # uneven, empty and one-row shards


@pytest.fixture(scope="module")
def torch():
    import torch as t
    if not t.cuda.is_available():
        pytest.skip("no GPU")
    return t


def devices_or_skip(torch, P, per_rank):
    if not per_rank:
        return None
    if torch.cuda.device_count() < P:
        pytest.skip(f"one GPU per rank needs {P} GPUs, this machine has {torch.cuda.device_count()}")
    return list(range(P))


def scaled(nrows, R):
    """small rows: enough of them that a shard is many 16-byte vectors (a one-row shard stays one row)"""
    return [n * 40 if n > 1 and R <= 24 else n for n in nrows]


def do_call(torch, store, dev, stream, name, itemsize, ll, R, call, exp, what):
    """one put through its entry -> (problems, keepalive); exp = the oracle's (code, bad, total) of this call"""
    p, (code, bad, total) = call.put, exp
    short = p.src_bytes is not None and p.src_bytes < pw.layout_total(ll, R, p.batch)
    src = np.full(p.src_bytes, pw.FILL_OUTSIDE, np.uint8) if short else pw.layout_src(p.pattern, ll, R, p.batch)
    sb = src.size if p.src_bytes is None else p.src_bytes
    buf, ptr = to_device(torch, src, call.off, dev)
    on_dev = call.entry != "host"
    idx = {k: (torch.from_numpy(np.ascontiguousarray(v, np.int64)).to(dev) if on_dev else v)
           for k, v in p.batch.items() if k in ("starts", "counts", "sample_ids")}
    torch.cuda.synchronize(dev)
    if call.entry in ("host", "dev"):
        kw = {"ids": idx["sample_ids"]} if "sample_ids" in idx else \
            {"starts": idx["starts"], "counts": idx.get("counts"), "fixed": p.batch.get("fixed_count", 1)}
        rc, gtotal, gbad = raw_put(store, name, itemsize, ptr if src.size else None, sb, **kw)
        got, want = (rc, gbad, gtotal), (ERR[code], bad, total)
        return ([] if got == want else [f"{what}: (rc, bad, total) = {got}, oracle {want}"]), (buf, idx)
    assert call.off == 0 and not short
    src_t = buf[:src.size].view(getattr(torch, DT[itemsize]))
    wait = call.entry == "api"
    raised = gtotal = None
    try:
        if "sample_ids" in idx:
            gtotal = store.put_samples(name, idx["sample_ids"], src_t, stream=stream, wait=wait)
        else:
            gtotal = store.put_batch(name, idx["starts"], idx.get("counts"), src=src_t, count=p.batch.get("fixed_count"),
                                     stream=stream, wait=wait)
    except ValueError as e:
        raised = str(e)
    if not wait:
        return ([f"{what}: queueing raised {raised!r}"] if raised else []), (buf, idx)
    return outcome_problems(what, raised, store.last_bad_index, gtotal, code, bad, total), (buf, idx)


def outcome_problems(what, raised, gbad, gtotal, code, bad, total):
    """the Python entry's outcome against the oracle's: the error text of `code` with last_bad_index = bad, or the total"""
    if code == 0:
        return [] if raised is None and gtotal == total else [f"{what}: raised {raised!r} / total {gtotal}, oracle: no error, total {total}"]
    want = "too small" if code == po.CODE_CAPACITY else error_text(code)
    if raised is None or want not in raised or gbad != bad:
        return [f"{what}: raised {raised!r} with last_bad_index {gbad}, oracle: {want!r} at request {bad}"]
    return []


def put_epochs(torch, P, nrows, itemsize, disp, seed, epochs, devices=None, tables=None, readers=None, updates=None):
    """Run `epochs` (epochs[e][rank] = [Call]) on P thread-ranks over shards of nrows[rank] rows. After every closing
    fence each rank compares its whole raw shard with the expectation, then runs `readers`. updates[e] (optional):
    {rank: (local row, rows)} rewritten by a local update() with epoch-6 bytes before epoch e. Returns nothing: asserts."""
    R, ll = itemsize * disp, pw.lenlist_of(nrows)
    state = pw.split_world(pw.pattern_world(seed, ll, R, 0), ll, R)
    fresh = pw.split_world(pw.pattern_world(seed, ll, R, 6), ll, R)
    initial, exp_shards, exp_status = state, [], []
    for e, epoch in enumerate(epochs):
        for r, (row, n) in (updates or {}).get(e, {}).items():
            state = [s.copy() for s in state]
            state[r][row:row + n] = fresh[r][row:row + n]
        state, status = pw.expected_world(state, [[c.put for c in calls] for calls in epoch], ll)
        exp_shards.append(state)
        exp_status.append(status)

    def body(store, r):
        import torch as t
        dev = t.device("cuda", t.cuda.current_device())
        stream = t.cuda.Stream(device=dev)
        problems, mine = [], np.ascontiguousarray(initial[r])
        assert store._L.dds_add(store._h, b"w", mine.ctypes.data if mine.size else None, nrows[r], disp, itemsize, 0) == 0, \
            store._L.dds_last_error()
        if tables:
            store.set_sample_index("w", *tables[r])
        for e, epoch in enumerate(epochs):
            if updates and e in updates:  # (inside a fence pair of its own: nobody reads these rows meanwhile)
                store.epoch_begin()
                if r in updates[e]:
                    row, n = updates[e][r]
                    store.update("w", np.ascontiguousarray(fresh[r][row:row + n]).view(DT[itemsize]).reshape(n, disp), row)
                store.epoch_end()
            store.epoch_begin()
            keep, queued = [], False
            for k, call in enumerate(epoch[r]):
                what = f"epoch {e} rank {r} call {k} ({call.entry}, src +{call.off})"
                try:
                    pr, ka = do_call(t, store, dev, stream.cuda_stream, "w", itemsize, ll, R, call, exp_status[e][r][k], what)
                    problems += pr
                    keep.append(ka)
                    queued |= call.entry == "queued"
                except Exception as ex:  # noqa: BLE001 -- the fence below must still be reached
                    problems.append(f"{what}: {type(ex).__name__}: {ex}")
            store.epoch_end()
            got, slack = shard_state(t, store, "w", nrows[r] * R, dev)
            msg = pw.shard_mismatch(got, slack, exp_shards[e][r], r, ll, R, [[c.put for c in calls] for calls in epoch],
                                    f"epoch {e}")
            if msg:
                problems.append(msg)
            if queued:  # the fence completed the queue and kept its outcome for wait(): this rank's own first error
                st = exp_status[e][r]
                first = next((s for s in st if s[0]), (0, -1, st[-1][2]))
                raised = gtotal = None
                try:
                    gtotal = store.wait()
                except ValueError as ex:
                    raised = str(ex)
                problems += outcome_problems(f"epoch {e} rank {r} wait()", raised, store.last_bad_index, gtotal,
                                             first[0], first[1], st[-1][2])
            if readers:
                try:
                    problems += readers(t, store, r, e, dev, np.concatenate([s.reshape(-1) for s in exp_shards[e]]))
                except Exception as ex:  # noqa: BLE001
                    problems.append(f"epoch {e} rank {r} readers: {type(ex).__name__}: {ex}")
            del keep
        return problems

    res = run_world(P, body, devices=devices)
    flat = [p for r in res for p in r]
    assert not flat, "\n".join(flat[:12])


# ------------------------------------------------------------------------------------------------ 1. owner edges
def edge_epochs(P, nrows, R, seed):
    """six epochs: variable counts twice, sample ids, fixed counts 1 / 3 / 40; host and device indices alternate over
    ranks and epochs, the source offset rotates. -> (epochs, tables, classes seen)"""
    ll = pw.lenlist_of(nrows)
    epochs, tables, seen = [], [None] * P, set()
    for e in range(6):
        pat, epoch = pw.pattern_world(7, ll, R, 1 + e), []
        for r in range(P):
            rng = np.random.default_rng([11, e, r])
            clean = (r + e) % P == 0  # one rank per epoch has no invalid request
            first_bad = None if clean else 2 + 3 * r + e
            off = SRC_OFFSETS[(r + e) % 5]
            entry = "dev" if (r + e) % 2 else "host"
            if e < 3:
                st, ct, cls = pw.edge_requests(rng, ll, r, first_bad=first_bad)
                batch = {"starts": st, "counts": ct}
                if e == 2:  # (the table holds the invalid requests too: a straddling sample keeps its bytes)
                    batch, cls = pw.as_samples(rng, st, ct, cls, first_bad=first_bad)
                    tables[r] = batch["table"]
                epoch.append([Call(pw.Put(batch, pat), entry, off)])
            else:
                cnt = (1, 3, 40)[e - 3]
                fs, cls = pw.edge_fixed(rng, ll, cnt, first_bad=first_bad)
                epoch.append([Call(pw.Put({"starts": fs, "fixed_count": cnt}, pat), entry, off)])
            seen |= set(cls)
        epochs.append(epoch)
    return epochs, tables, seen


EDGE_WORLDS = [(2 + i % 3, s) for i, s in enumerate(SHAPES)] + [(4, (1, 1)), (3, (8, 512))]


@pytest.mark.parametrize("per_rank", [False, True], ids=["one-gpu", "gpu-per-rank"])
@pytest.mark.parametrize("P,shape", EDGE_WORLDS, ids=[f"P{p}-{i}x{d}" for p, (i, d) in EDGE_WORLDS])
def test_owner_edges(torch, P, shape, per_rank):
    """every owner's first / last rows, whole shards, boundary neighbours, straddlers and the invalid family, through
    every entry, every rank with its own first invalid request (one rank per epoch has none)"""
    if per_rank and shape not in ((1, 3), (8, 512)):
        pytest.skip("the cross-GPU run takes one small-row and one 4 KiB world")
    devices = devices_or_skip(torch, P, per_rank)
    itemsize, disp = shape
    nrows = scaled(ROWS[P], itemsize * disp)
    epochs, tables, seen = edge_epochs(P, nrows, itemsize * disp, 7)
    assert seen >= pw.EDGE_CLASSES | pw.PAIR_CLASSES | pw.INVALID_CLASSES | pw.SAMPLE_CLASSES, seen
    put_epochs(torch, P, nrows, itemsize, disp, 7, epochs, devices=devices, tables=tables)


def test_some_ranks_raise_and_all_reach_the_fence(torch):
    """put_batch / put_samples themselves: the ranks with an invalid request raise the reference's error with their own
    index, the clean rank returns its total, and every rank reaches the fence (run_world fails a rank that hangs)"""
    P, itemsize, disp = 3, 4, 5
    nrows = scaled(ROWS[P], 20)
    ll, epochs, tables = pw.lenlist_of(nrows), [], [None] * P
    for e in range(2):
        pat, epoch = pw.pattern_world(3, ll, 20, 1 + e), []
        for r in range(P):
            rng = np.random.default_rng([13, e, r])
            first_bad = None if r == e else 4 + r
            st, ct, cls = pw.edge_requests(rng, ll, r, first_bad=None if e else first_bad)
            batch = {"starts": st, "counts": ct}
            if e:
                batch, cls = pw.as_samples(rng, st, ct, cls, first_bad=first_bad)
                tables[r] = batch["table"]
            epoch.append([Call(pw.Put(batch, pat), "api", 0)])
        epochs.append(epoch)
    put_epochs(torch, P, nrows, itemsize, disp, 3, epochs, tables=tables)


# ------------------------------------------------------------------------------------------------ 2. interleaved writers
@pytest.mark.parametrize("per_rank", [False, True], ids=["one-gpu", "gpu-per-rank"])
@pytest.mark.parametrize("P", [3, 4])
@pytest.mark.parametrize("shape", SHAPES[:5] + [(8, 512)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_interleaved_writers(torch, P, shape, per_rank):
    """a partition of every row of the world into 1..3-row requests (and a chunk-sized and a > 1 MiB one where they
    fit), neighbours dealt to different writers: rows of different ranks, CTAs and warps share 16-byte vectors. Every
    byte of every shard changes, the slack stays zero. P = 3: thousands of requests per writer (the plan kernels);
    P = 4: a few hundred (the shared-memory plan)."""
    if per_rank and (P != 3 or shape not in ((1, 3), (8, 512))):
        pytest.skip("the cross-GPU run takes one small-row and one 4 KiB world")
    devices = devices_or_skip(torch, P, per_rank)
    itemsize, disp = shape
    R = itemsize * disp
    nrows = [0, 300, 1, 600][4 - P:] if R == 4096 else ([9000, 1, 14000] if P == 3 else [0, 900, 1, 1400])
    ll = pw.lenlist_of(nrows)
    epochs = []
    for e in range(2):  # (the second epoch: other writers for the same rows)
        cover = pw.interleaved_cover(np.random.default_rng([17, e, R]), ll, P, R)
        pat = pw.pattern_world(5, ll, R, 1 + e)
        epochs.append([[Call(pw.Put({"starts": s, "counts": c}, pat), "dev" if (w + e) % 2 else "host",
                             SRC_OFFSETS[(w + 2 * e) % 5])] for w, (s, c) in enumerate(cover)])
    put_epochs(torch, P, nrows, itemsize, disp, 5, epochs, devices=devices)


# ------------------------------------------------------------------------------------------------ 3. capacity
def test_capacity_on_one_rank_only(torch):
    """one rank's source is a byte short of its layout: DDS_ERR_CAPACITY, bad index -1, nothing of it written, while the
    other ranks' batches of the same epoch land; with an invalid request as well, the invalid request is reported"""
    P, itemsize, disp = 3, 4, 5
    nrows, R = [500, 1, 300], 20
    ll, epochs = pw.lenlist_of(nrows), []
    for e, short_rank in enumerate((1, 2)):
        pat, epoch = pw.pattern_world(19, ll, R, 1 + e), []
        for r in range(P):
            rng = np.random.default_rng([19, e, r])
            st, ct, _ = pw.edge_requests(rng, ll, r, first_bad=(5 if e and r == short_rank else None), body=200)
            batch = {"starts": st, "counts": ct}
            sb = pw.layout_total(ll, R, batch) - 1 if r == short_rank else None
            epoch.append([Call(pw.Put(batch, pat, sb), "dev" if r % 2 else "host", SRC_OFFSETS[r])])
        epochs.append(epoch)
    status = pw.expected_world(pw.split_world(pw.pattern_world(19, ll, R, 0), ll, R), [[c.put for c in x] for x in epochs[0]])[1]
    assert status[1][0][:2] == (po.CODE_CAPACITY, -1) and status[0][0][0] == 0
    put_epochs(torch, P, nrows, itemsize, disp, 19, epochs)


def test_layout_above_4gib_only_from_invalid_requests(torch):
    """300 requests that straddle two owners keep ~16 MiB each in the caller's layout: 4.9 GiB, on the shared-memory
    plan, against a 64 KiB source. The layout total is carried in 64 bits (plan_in_smem sums int64 and compares it with
    the capacity before anything is walked), so: the first invalid request is reported, no byte of any shard is written,
    and the other rank's batch of the same epoch lands."""
    P, itemsize, disp = 2, 8, 512
    nrows = [2000, 2100]
    ll = pw.lenlist_of(nrows)
    pat = pw.pattern_world(23, ll, 4096, 1)
    st = np.concatenate([[0, 5], np.full(300, 1)]).astype(np.int64)
    ct = np.concatenate([[2, 1], np.full(300, 4098)]).astype(np.int64)
    big = pw.Put({"starts": st, "counts": ct}, pat, src_bytes=1 << 16)
    assert pw.layout_total(ll, 4096, big.batch) > 1 << 32
    s1, c1, _ = pw.edge_requests(np.random.default_rng(23), ll, 1)
    epochs = [[[Call(big, "host", 0), Call(big, "dev", 8)], [Call(pw.Put({"starts": s1, "counts": c1}, pat), "dev", 4)]]]
    put_epochs(torch, P, nrows, itemsize, disp, 23, epochs)


# ------------------------------------------------------------------------------------------------ 4. queued puts
def test_queued_puts_complete_at_the_fence(torch):
    """every rank queues three puts (wait=False, device indices, its own stream), the middle one with an invalid request
    on ranks 1 and 2, and crosses the fence without wait(): every shard is complete on every rank; the wait() that
    follows raises that rank's own error with its index, and returns cleanly on rank 0"""
    P, itemsize, disp = 3, 2, 3
    nrows = scaled(ROWS[P], 6)
    ll = pw.lenlist_of(nrows)
    pat, epoch = pw.pattern_world(29, ll, 6, 1), []
    for r in range(P):
        calls = []
        for k in range(3):
            rng = np.random.default_rng([29, r, k])
            st, ct, _ = pw.edge_requests(rng, ll, r, first_bad=(3 + r if k == 1 and r else None), body=300)
            calls.append(Call(pw.Put({"starts": st, "counts": ct}, pat), "queued", 0))
        epoch.append(calls)
    put_epochs(torch, P, nrows, itemsize, disp, 29, [epoch])


# ------------------------------------------------------------------------------------------------ 5. two epochs, every reader
def world_readers(nrows, itemsize, disp):
    """after a fence: the whole world through get_batch, get_samples, a padded get_samples, a converting get_batch and
    get() on every owner's boundary rows, against the expected world's bytes"""
    ll, R = pw.lenlist_of(nrows), itemsize * disp
    own = pw.owners(ll)
    total = int(ll[-1])
    rs = np.arange(0, total, 3, dtype=np.int64)  # samples of 3 rows that do not cross an owner's end
    rs = np.array([s for s in rs if po.locate(ll, int(s), min(3, total - int(s)))[0] == 0], np.int64)
    rc = np.minimum(3, total - rs)

    def readers(t, store, r, e, dev, world):
        dt, out_problems = getattr(t, DT[itemsize]), []
        exp = t.from_numpy(world.copy()).to(dev)

        def same(what, got, want):
            if not t.equal(got.reshape(-1).view(t.uint8), want.reshape(-1).view(t.uint8)):
                d = int((got.reshape(-1).view(t.uint8) != want.reshape(-1).view(t.uint8)).nonzero()[0])
                out_problems.append(f"epoch {e} rank {r} {what}: byte {d} differs (global row {d // R})")

        out = t.zeros(total * disp, dtype=dt, device=dev)
        t.cuda.synchronize(dev)
        store.get_batch("w", [o[1] for o in own], [o[2] - o[1] for o in own], out=out)
        same("get_batch", out, exp)
        if e == 0:
            store.set_sample_index("w", rs, rc)
        rows = np.concatenate([np.arange(s, s + c) for s, c in zip(rs, rc)])
        want = exp.view(total, R)[t.from_numpy(rows).to(dev)]
        out = t.zeros(rows.size * disp, dtype=dt, device=dev)
        t.cuda.synchronize(dev)
        store.get_samples("w", np.arange(len(rs)), out)
        same("get_samples", out, want)
        pad = t.zeros(len(rs), 3, disp, dtype=dt, device=dev)
        lengths = t.zeros(len(rs), dtype=t.int64, device=dev)
        t.cuda.synchronize(dev)
        store.get_samples("w", np.arange(len(rs)), pad, pad_rows=3, pad_value=0, lengths=lengths)
        wantp = t.zeros(len(rs), 3, R, dtype=t.uint8, device=dev)
        for j, (s, c) in enumerate(zip(rs.tolist(), rc.tolist())):
            wantp[j, :c] = exp.view(total, R)[s:s + c]
        same("padded get_samples", pad, wantp)
        if lengths.cpu().tolist() != rc.tolist():
            out_problems.append(f"epoch {e} rank {r}: padded lengths differ")
        if itemsize == 4:  # float32 -> bfloat16 inside the gather (finite values: NaN payloads are not the put's business)
            f = exp.view(t.float32)
            bf = t.zeros(total * disp, dtype=t.bfloat16, device=dev)
            t.cuda.synchronize(dev)
            store.get_batch("w", [o[1] for o in own], [o[2] - o[1] for o in own], out=bf, src_dtype="float32")
            ok = t.isfinite(f)
            if not t.equal(bf[ok].view(t.int16), f.to(t.bfloat16)[ok].view(t.int16)):
                out_problems.append(f"epoch {e} rank {r} converting get_batch differs")
        one = np.zeros((1, disp), DT[itemsize])
        for _, lo, hi in own:
            for g in (lo, hi - 1):
                store.get("w", one, g)
                if one.tobytes() != world[g * R:(g + 1) * R].tobytes():
                    out_problems.append(f"epoch {e} rank {r} get(): global row {g} differs")
        return out_problems

    return readers


@pytest.mark.parametrize("per_rank", [False, True], ids=["one-gpu", "gpu-per-rank"])
@pytest.mark.parametrize("doorbell", [True, False])
def test_two_epochs_every_reader(torch, monkeypatch, doorbell, per_rank):
    """epoch 1 writes every row of the world from interleaved writers; some rows are then rewritten by their owners'
    update(); epoch 2 rotates the writers and writes the rows again, except those next to the updated ones. After each
    fence every rank reads the whole world through every get path (doorbell kernel resident across the fences, and
    DDS_DOORBELL=0)."""
    P, itemsize, disp = 3, 4, 5
    devices = devices_or_skip(torch, P, per_rank)
    monkeypatch.setenv("DDS_DOORBELL", "1" if doorbell else "0")
    monkeypatch.setenv("DDS_DOORBELL_IDLE_US", "5000000")
    nrows, R = [700, 1, 401], 20
    ll = pw.lenlist_of(nrows)
    updates = {1: {0: (100, 7), 2: (0, 3)}}  # local rows rewritten between the epochs
    upd_rows = set(range(100, 107)) | set(range(701, 704))
    epochs = []
    for e in range(2):
        cover = pw.interleaved_cover(np.random.default_rng([31, e]), ll, P, R, big=False)
        pat, epoch = pw.pattern_world(31, ll, R, 1 + e), []
        for w in range(P):
            s, c = cover[(w + e) % P]
            if e:  # the second epoch leaves the updated rows alone: the put must not bring back what they held before
                m = np.array([not (upd_rows & set(range(a, a + b))) for a, b in zip(s.tolist(), c.tolist())])
                s, c = s[m], c[m]
            epoch.append([Call(pw.Put({"starts": s, "counts": c}, pat), "dev" if w % 2 else "host", SRC_OFFSETS[w + e])])
        epochs.append(epoch)
    put_epochs(torch, P, nrows, itemsize, disp, 31, epochs, devices=devices, updates=updates,
               readers=world_readers(nrows, itemsize, disp))


# ------------------------------------------------------------------------------------------------ 6. sixty-four owners
def test_sixty_four_owners(torch):
    """64 thread-ranks, a third of them empty (first and last rank, runs of empty ones, one-row owners): every non-empty
    rank puts the edge requests of the next two non-empty ranks, with its own first invalid request; every rank, the
    empty ones too, compares its raw shard"""
    P, itemsize, disp = 64, 1, 5
    nrows = sixty_four_rows()
    ll = pw.lenlist_of(nrows)
    own = [o[0] for o in pw.owners(ll)]
    pat, epoch, seen = pw.pattern_world(37, ll, 5, 1), [], set()
    for r in range(P):
        if not nrows[r]:
            epoch.append([])
            continue
        j = own.index(r)
        only = {own[(j + 1) % len(own)], own[(j + 2) % len(own)]}
        st, ct, cls = pw.edge_requests(np.random.default_rng([37, r]), ll, r, first_bad=r % 7, body=6, only=only)
        seen |= set(cls)
        epoch.append([Call(pw.Put({"starts": st, "counts": ct}, pat), "dev" if r % 2 else "host", SRC_OFFSETS[r % 5])])
    assert seen >= pw.EDGE_CLASSES | pw.PAIR_CLASSES | pw.INVALID_CLASSES
    put_epochs(torch, P, nrows, itemsize, disp, 37, [epoch])
