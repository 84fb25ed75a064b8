"""How a queue of DDS_NO_SYNC batches ends (-m gpu). The outcome of queued batches is reported by wait() and only by
it, exactly once: any other call that meets a pending queue completes it first, keeps its first failure (unless an
earlier one is kept already) and the total of its last batch, then does its own work and reports only its own outcome.
The next wait() raises the kept failure with its index, the one after that is clean.

Every queue kind (fixed count, explicit counts planned in shared memory and in global memory, get_samples, a
two-variable get_samples_multi, a converting f32 -> bf16 batch), plain and overlapped, with no failure, with two
invalid batches and with a capacity error before an invalid batch, meets every ending: wait(), synchronous calls on the
queue's stream, on the store's stream and into every host destination path, get() through both single-request
kernels, synchronous get_samples / get_samples_multi, a second queue on another stream, set_sample_index and
set_normalization, and the collective epoch_end and free. Also: a loader abandoned mid-epoch, a queue longer than the
16-bit ordinal of the status word, and the wrap of the plan kernels' 22-bit tag counter. Every delivered byte, offset
and total is compared with the oracle of tests/gpu_helpers.py, between sentinel guard bands."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.convert_oracle import CVT_F32_BF16, convert_bytes
from tests.gpu_helpers import CODE_SAMPLE, GUARD, Dest, Expected, check_dest, classify, error_text, expect_raise, \
    guarded_buffer, run_world
from tests.test_gpu_errors import DISP, LL, NROWS, ROW, SENT, TOTAL, _world, invalid_request, run_rank0, valid_requests

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NSAMP = 6000
KINDS = ("fixed", "var_smem", "var_global", "samples", "multi", "convert")
SIZES = {"fixed": 3000, "var_smem": 1000, "var_global": 3000, "samples": 3000, "multi": 1000, "convert": 3000}
OUTCOMES = ("clean", "invalid", "capacity")
OWN_BAD = 123  # where an ending's own invalid request sits (the queue's are at 500 and 7)


def _torch():
    import torch
    return torch


class Data:
    """the world's variables, host side: v and w (random bits, NaNs included), f (finite float32, for the f32 -> bf16
    conversion), all 4 owners with owner 1 empty and 24-byte rows; sample tables of v and w"""

    def __init__(self):
        self.shards, self.allrows = _world(7)
        self.shards_w, self.allrows_w = _world(8)
        rng = np.random.default_rng(9)
        self.shards_f = [rng.standard_normal((n, DISP)).astype(np.float32) for n in NROWS]
        self.allrows_f = np.concatenate([s.reshape(-1).view(np.uint8) for s in self.shards_f])
        self.allrows_fb = convert_bytes(self.allrows_f, CVT_F32_BF16)
        self.tab = {"v": valid_requests(rng, NSAMP, 3), "w": valid_requests(rng, NSAMP, 3)}

    def add(self, store, r):
        store.add("v", self.shards[r])
        store.add("w", self.shards_w[r])
        store.add("f", self.shards_f[r])
        for name in ("v", "w"):
            store.set_sample_index(name, *self.tab[name])

    def sample_exp(self, name, ids):
        tst, tct = self.tab[name]
        allrows = self.allrows if name == "v" else self.allrows_w
        inside = (ids >= 0) & (ids < NSAMP)
        st = np.where(inside, tst[np.clip(ids, 0, NSAMP - 1)], 0)
        ct = np.where(inside, tct[np.clip(ids, 0, NSAMP - 1)], 0)
        codes = np.where(inside, classify(LL, st, ct), CODE_SAMPLE)
        return Expected(allrows, ROW, LL, st, ct, False, codes=codes)


def _fixed_ok(s):
    """starts of valid_requests made valid for a fixed count of 2 (a zero-count draw may start at the total)"""
    return np.where(np.isin(s, LL - 1), s - 1, np.minimum(s, TOTAL - 2))


def make_batch(D, kind, rng, bad=None, B=None):
    """(host index arrays, [Expected per variable]) of one batch of B requests (default SIZES[kind]); bad = (position,
    0 or 1): an invalid request there, of a count-error kind (0) or a start-error kind (1); a sample id past or below
    the index for the sample kinds"""
    B = B or SIZES[kind]
    if kind in ("fixed", "convert"):
        s = _fixed_ok(valid_requests(rng, B, 2)[0])
        if bad:
            s[bad[0]] = invalid_request(("start_past", "start_neg")[bad[1]], rng, 2)[0]
        allrows, row = (D.allrows, ROW) if kind == "fixed" else (D.allrows_fb, ROW // 2)
        exp = Expected(allrows, row, LL, s, np.full(B, 2, np.int64), True)
        assert bad or exp.bad < 0
        return (s,), [exp]
    if kind in ("var_smem", "var_global"):
        s, c = valid_requests(rng, B, 3)
        if bad:
            s[bad[0]], c[bad[0]] = invalid_request(("past_end", "start_neg")[bad[1]], rng, 2)
        return (s, c), [Expected(D.allrows, ROW, LL, s, c, False)]
    ids = rng.integers(0, NSAMP, size=B).astype(np.int64)
    if bad:
        ids[bad[0]] = (NSAMP + 7, -1)[bad[1]]
    exps = [D.sample_exp("v", ids)] + ([D.sample_exp("w", ids)] if kind == "multi" else [])
    if len(exps) > 1 and exps[0].bad >= 0:  # the loop over variables stops in variable 0: nothing of variable 1 is due
        exps[1].prefix = 0
    assert bad or all(e.bad < 0 for e in exps)
    return (ids,), exps


def queue_var(kind):
    return "f" if kind == "convert" else "v"


def other_var(kind):
    return "f" if kind == "multi" else "w"


class Queued:
    """one batch of a queue: device indices, guarded destinations (and offsets), what they must hold"""

    def __init__(self, torch, kind, idx, exps, caps, k):
        self.kind, self.exps = kind, exps
        self.idx = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in idx]
        off = 2 * k + 2 if kind == "convert" else 2 * k + 1  # (a bf16 destination must be 2-byte aligned)
        self.dests = [Dest(torch, "device", c, SENT, off=off) for c in caps]
        self.nreq = len(idx[0])
        self.offs = [torch.full((self.nreq + 1,), -7, dtype=torch.int64, device="cuda") for _ in caps]
        self.over = [c < e.T for c, e in zip(caps, exps)]

    def outs(self):
        torch = _torch()
        return [d.view.view(torch.bfloat16) if self.kind == "convert" else d.view for d in self.dests]

    def launch(self, store, stream, wait, overlap=False):
        kw = dict(stream=stream, wait=wait, overlap=overlap)
        outs = self.outs()
        if self.kind == "fixed":
            return store.get_batch("v", self.idx[0], out=outs[0], count=2, offsets=self.offs[0], **kw)
        if self.kind == "convert":
            return store.get_batch("f", self.idx[0], out=outs[0], count=2, offsets=self.offs[0], src_dtype="float32", **kw)
        if self.kind in ("var_smem", "var_global"):
            return store.get_batch("v", self.idx[0], self.idx[1], out=outs[0], offsets=self.offs[0], **kw)
        if self.kind == "samples":
            return store.get_samples("v", self.idx[0], outs[0], offsets=self.offs[0], **kw)
        return store.get_samples_multi(["v", "w"], self.idx[0], outs, offsets=self.offs, **kw)

    def total(self):
        return sum(e.T for e in self.exps)

    def check(self, what):
        _torch().cuda.synchronize()
        over = any(self.over)  # (a multi-array batch that does not fit writes nothing in any variable)
        for v, (d, e, f) in enumerate(zip(self.dests, self.exps, self.offs)):
            check_dest(d, e, over, f"{what} variable {v}", offsets=None if over else f)

    def reset(self):
        for d in self.dests:
            d.reset()
        for f in self.offs:
            f.fill_(-7)
        _torch().cuda.synchronize()


class Queue:
    """five batches of one kind and outcome: 'clean'; 'invalid' -- batch 1 invalid at request 500, batch 3 at 7 (a
    lower index, later in queue order); 'capacity' -- batch 1 one byte (one bf16 element) too small, batch 3 invalid.
    `fresh` holds the same batches without failures, through the same destinations, for the valid queue that follows."""

    def __init__(self, torch, D, kind, outcome, seed):
        rng = np.random.default_rng(seed)
        self.kind, self.outcome = kind, outcome
        bads = {1: (500, 0), 3: (7, 1)} if outcome == "invalid" else {3: (7, 1)} if outcome == "capacity" else {}
        self.batches, self.fresh = [], []
        for k in range(5):
            state = rng.bit_generator.state
            idx, exps = make_batch(D, kind, rng, bads.get(k))
            rng2 = np.random.default_rng()
            rng2.bit_generator.state = state
            cidx, cexps = make_batch(D, kind, rng2)  # the same batch without its invalid request
            caps = [max(e.T, c.T) + 16 for e, c in zip(exps, cexps)]
            if outcome == "capacity" and k == 1:
                caps[0] = exps[0].T - (2 if kind == "convert" else 1)
            self.batches.append(Queued(torch, kind, idx, exps, caps, k))
            fq = Queued.__new__(Queued)
            fq.__dict__.update(self.batches[-1].__dict__)
            fq.idx = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in cidx]
            fq.exps = cexps
            fq.over = [c < e.T for c, e in zip(caps, cexps)]
            self.fresh.append(fq)
        # what wait() must report: the first failing batch in queue order
        self.fail = None
        for q in self.batches:
            if any(q.over) and not any(e.bad >= 0 for e in q.exps):
                self.fail = ("too small", -1)
                break
            bad = [e for e in q.exps if e.bad >= 0]
            if bad:
                self.fail = (error_text(bad[0].code), bad[0].bad)
                break

    def launch(self, store, stream, overlap):
        for q in self.batches:
            q.reset()
        for q in self.batches:
            assert q.launch(store, stream, False, overlap) in (0, None)

    def check(self, what):
        for k, q in enumerate(self.batches):
            q.check(f"{what}: batch {k}")

    def run_fresh(self, store, stream, overlap, what):
        """a valid queue through the same destinations (those it fits): it delivers, wait() returns its total"""
        qs = [q for q in self.fresh if not any(q.over)]
        for q in qs:
            q.reset()
        for q in qs:
            q.launch(store, stream, False, overlap)
        total = store.wait()
        assert total == qs[-1].total(), f"{what}: fresh queue: wait() returned {total}, the last batch packs {qs[-1].total()}"
        assert store.last_bad_index == -1, f"{what}: fresh queue: last_bad_index {store.last_bad_index}"
        for k, q in enumerate(qs):
            q.check(f"{what}: fresh queue batch {k}")


def expect_wait(store, fail, total, what):
    """the next wait() reports `fail` ((text, index) or None: returns `total`), the one after it is clean"""
    try:
        got = store.wait()
        err = None
    except ValueError as e:
        got, err = None, str(e)
    if fail is None:
        assert err is None, f"{what}: wait() raised {err!r}, nothing failed"
        assert got == total, f"{what}: wait() returned {got}, the last queued batch packs {total}"
        assert store.last_bad_index == -1, f"{what}: last_bad_index {store.last_bad_index} after a clean wait()"
    else:
        text, index = fail
        assert err is not None and text in err, f"{what}: wait() raised {err!r}, the queue's first failure is {text!r}"
        assert store.last_bad_index == index, f"{what}: wait() reported index {store.last_bad_index}, the queue's is {index}"
    assert store.wait() == 0, f"{what}: the wait() after the report"
    assert store.last_bad_index == -1, f"{what}: the wait() after the report: last_bad_index {store.last_bad_index}"


# ------------------------------------------------------------------------------- the endings of rank 0
class Endings:
    """the calls that end a pending queue on rank 0 without being wait(); each checks its own outcome, and returns a
    second queue's batch when it queued one (its failure and total then count for the next wait())"""

    def __init__(self, torch, D, side, side2):
        self.torch, self.D, self.side, self.side2 = torch, D, side, side2
        rng = np.random.default_rng(77)

        def fixed(B, bad):
            s = _fixed_ok(valid_requests(rng, B, 2)[0])
            if bad:
                s[OWN_BAD] = invalid_request("start_neg", rng, 2)[0]
            exp = Expected(D.allrows, ROW, LL, s, np.full(B, 2, np.int64), True)
            assert exp.bad == (OWN_BAD if bad else -1)
            return s, exp

        # (B, destination kind, stream): bounce buffer, staging buffer, pipelined pageable copy
        self.sync = {"sync_side": (200, "device", side.cuda_stream), "sync_store": (200, "device", None),
                     "pinned_small": (600, "pinned", None), "pinned_large": (3000, "pinned", None),
                     "pageable": (100_000, "pageable", None)}
        self.batches = {(name, bad): fixed(B, bad) for name, (B, _, _) in self.sync.items() for bad in (False, True)}
        self.q2 = {bad: fixed(200, bad) for bad in (False, True)}
        ids = rng.integers(0, NSAMP, size=500).astype(np.int64)
        bad_ids = ids.copy()
        bad_ids[OWN_BAD] = -1
        self.ids = {False: ids, True: bad_ids}

    names = ("wait", "sync_side", "sync_store", "pinned_small", "pinned_large", "pageable", "get_doorbell", "get_1cta",
             "samples_sync", "multi_sync", "q2_clean", "q2_fail", "setidx_queued", "setidx_other", "setnorm_queued",
             "setnorm_other")

    @staticmethod
    def has_own_bad(name):
        return name not in ("wait", "q2_clean", "q2_fail", "setidx_queued", "setidx_other")

    def run(self, store, name, kind, bad, what):
        torch, D = self.torch, self.D
        if name == "wait":
            return None
        if name in self.sync:
            B, dk, st = self.sync[name]
            s, exp = self.batches[(name, bad)]
            dest = Dest(torch, dk, exp.T, SENT, off=3)
            offs = torch.full((B + 1,), -7, dtype=torch.int64, device="cuda") if dk == "device" else np.full(B + 1, -7, np.int64)
            torch.cuda.synchronize()  # (the store's own stream is not ordered with torch's)
            got = []
            expect_raise(store, lambda: got.append(store.get_batch("v", s, out=dest.view, count=2, offsets=offs, stream=st)),
                         exp, False, what)
            if not bad:
                assert got == [exp.T], f"{what}: returned {got}, oracle {exp.T}"
                assert store.last_bad_index == -1, f"{what}: last_bad_index {store.last_bad_index} on a valid call"
            check_dest(dest, exp, False, what, offsets=offs)
            return None
        if name in ("get_doorbell", "get_1cta"):
            var = "v" if name == "get_doorbell" else "late"
            arr = np.full((3, DISP), -1.0, np.float32)
            if bad:  # (a start error: the queues fail with count errors first)
                with pytest.raises(ValueError) as ei:
                    store.get(var, arr, -5)
                assert str(ei.value) == "Invalid start on target", f"{what}: {ei.value}"
                assert np.all(arr == -1.0), f"{what}: the destination was written"
            else:
                store.get(var, arr, 1234)
                assert arr.tobytes() == D.allrows[1234 * ROW:1237 * ROW].tobytes(), what
            return None
        if name == "samples_sync":
            ids = self.ids[bad]
            exp = D.sample_exp("v", ids)
            dest = Dest(torch, "device", exp.T + 8, SENT, off=5)
            offs = torch.full((len(ids) + 1,), -7, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            got = []
            expect_raise(store, lambda: got.append(store.get_samples("v", ids, dest.view, offsets=offs)), exp, False, what)
            if not bad:
                assert got == [exp.T] and store.last_bad_index == -1, f"{what}: returned {got}, oracle {exp.T}"
            check_dest(dest, exp, False, what, offsets=offs)
            return None
        if name == "multi_sync":
            ids = self.ids[bad]
            exps = [D.sample_exp("v", ids), D.sample_exp("w", ids)]
            if bad:
                exps[1].prefix = 0
            dests = [Dest(torch, "device", e.T + 8, SENT, off=1 + v) for v, e in enumerate(exps)]
            offs = [torch.full((len(ids) + 1,), -7, dtype=torch.int64, device="cuda") for _ in exps]
            torch.cuda.synchronize()
            got = []
            expect_raise(store, lambda: got.append(store.get_samples_multi(["v", "w"], ids, [d.view for d in dests],
                                                                           offsets=offs)), exps[0], False, what)
            if not bad:
                assert got == [[e.T for e in exps]] and store.last_bad_index == -1, f"{what}: returned {got}"
            for v, (d, e, f) in enumerate(zip(dests, exps, offs)):
                check_dest(d, e, False, f"{what} variable {v}", offsets=f)
            return None
        if name in ("q2_clean", "q2_fail"):
            s, exp = self.q2[name == "q2_fail"]
            q = Queued.__new__(Queued)
            q.kind, q.exps, q.nreq, q.over = "fixed", [exp], len(s), [False]
            q.idx = [torch.from_numpy(s).cuda()]
            q.dests = [Dest(torch, "device", exp.T, SENT, off=7)]
            q.offs = [torch.full((len(s) + 1,), -7, dtype=torch.int64, device="cuda")]
            torch.cuda.synchronize()
            assert q.launch(store, self.side2.cuda_stream, False) == 0, what
            assert store.last_bad_index == -1, what
            return q
        var = {"setidx_queued": queue_var(kind), "setidx_other": other_var(kind),
               "setnorm_queued": queue_var(kind), "setnorm_other": other_var(kind)}[name]
        if name.startswith("setidx"):
            tab = D.tab[var if var in D.tab else "v"]
            store.set_sample_index(var, *tab)
        else:
            mean = np.full(4 if bad else 1, 0.5, np.float32)
            std = np.full(4 if bad else 1, 2.0, np.float32)
            if bad:  # 4 channels do not divide a row of 6 elements: an argument error before anything else
                with pytest.raises(ValueError) as ei:
                    store.set_normalization(var, mean, std)
                assert "Invalid argument" in str(ei.value), f"{what}: {ei.value}"
            else:
                store.set_normalization(var, mean, std)
        return None


def _late_world(D):
    """the world plus 256 one-byte variables and `late`, a copy of v past the resident kernel's 256 slots"""
    def add(store, r):
        D.add(store, r)
        for k in range(256):
            store.add(f"pad{k}", np.zeros((1, 1), np.uint8))
        store.add("late", D.shards[r])
    return add


@pytest.mark.parametrize("kind", KINDS)
def test_every_ending_of_every_queue(kind):
    """wait() and every rank-0 ending, each once per queue: plain and overlapped, no failure, two invalid batches, a
    capacity error before an invalid batch; each ending also once with an invalid request of its own"""
    torch = _torch()
    D = Data()
    add = _late_world(D)

    def body(store, r):
        add(store, r)
        if r:
            return True
        side, side2 = torch.cuda.Stream(), torch.cuda.Stream()
        ends = Endings(torch, D, side, side2)
        queues = {oc: Queue(torch, D, kind, oc, 100 + i) for i, oc in enumerate(OUTCOMES)}
        failed = {}  # (ending, outcome, own invalid request) -> its first failure: every combination runs
        for overlap in (False, True):
            for name in ends.names:
                runs = [(oc, False) for oc in OUTCOMES] + ([("invalid", True)] if ends.has_own_bad(name) else [])
                for oc, bad in runs:
                    Q = queues[oc]
                    what = f"{kind} overlap={overlap} {oc} queue, ended by {name}{' with an invalid request' if bad else ''}"
                    try:
                        Q.launch(store, side.cuda_stream, overlap)
                        q2 = ends.run(store, name, kind, bad, what)
                        fail, total = Q.fail, Q.batches[-1].total()
                        if q2 is not None:
                            if fail is None and q2.exps[0].bad >= 0:
                                fail = (error_text(q2.exps[0].code), q2.exps[0].bad)
                            total = q2.total()
                        expect_wait(store, fail, total, what)
                        Q.check(what)
                        if q2 is not None:
                            q2.check(f"{what}: the second queue")
                        if not bad:
                            Q.run_fresh(store, side.cuda_stream, overlap, what)
                    except (AssertionError, ValueError) as ex:
                        failed.setdefault((name, oc, bad), f"{type(ex).__name__}: {str(ex).splitlines()[0][:300]}")
                        try:  # (leave nothing pending for the next run)
                            store.wait()
                        except ValueError:
                            pass
                        torch.cuda.synchronize()
        assert not failed, f"{len(failed)} combinations failed:\n" + "\n".join(failed.values())
        return True

    assert all(run_rank0(4, body, timeout=900))


@pytest.mark.parametrize("ending", ("epoch_end", "free"))
def test_collective_endings(ending):
    """epoch_begin ... queue ... epoch_end, and free(), on all 4 ranks with only rank 0's queue failing: every rank
    returns (run_world's timeout names a hung one), rank 0's next wait() reports its queue, the others' their totals"""
    torch = _torch()
    D = Data()

    def body(store, r):
        D.add(store, r)
        side = torch.cuda.Stream()
        rng = np.random.default_rng(300 + r)
        s = _fixed_ok(valid_requests(rng, 500, 2)[0])
        mine = Queued(torch, "fixed", (s,), [Expected(D.allrows, ROW, LL, s, np.full(500, 2, np.int64), True)], [500 * 48], 0)
        for kind in KINDS:
            queues = {oc: Queue(torch, D, kind, oc, 400 + i) for i, oc in enumerate(OUTCOMES)} if r == 0 else None
            for overlap in (False, True):
                for oc in OUTCOMES:
                    what = f"rank {r}: {kind} overlap={overlap} {oc} queue, ended by {ending}"
                    if ending == "epoch_end":
                        store.epoch_begin()
                    if r == 0:
                        queues[oc].launch(store, side.cuda_stream, overlap)
                    else:
                        mine.reset()
                        mine.launch(store, side.cuda_stream, False, overlap)
                    if ending == "epoch_end":
                        store.epoch_end()
                    else:
                        store.free()
                    if r == 0:
                        expect_wait(store, queues[oc].fail, queues[oc].batches[-1].total(), what)
                        queues[oc].check(what)
                    else:
                        expect_wait(store, None, mine.total(), what)
                        mine.check(what)
                    if ending == "free":
                        D.add(store, r)
                    if r == 0:
                        queues[oc].run_fresh(store, side.cuda_stream, overlap, what)
        return True

    assert all(run_world(4, body, timeout=900))


# ------------------------------------------------------------------------------- a loader left mid-epoch
def test_prefetch_loader_abandoned_mid_epoch():
    """the 2nd batch of the sampler holds an out-of-range id; with depth 2 its fetch is queued when the first batch is
    yielded. The consumer takes that batch and stops. __getitems__ of valid ids returns the right rows; wait() then
    raises the loader's error with its index"""
    torch = _torch()
    from ddstore_b200.dataset import DistDataset, PrefetchLoader
    rng = np.random.default_rng(5)
    N, BS = 2000, 64
    imgs = rng.standard_normal((N, 3, 4)).astype(np.float32)
    ds = DistDataset([(imgs[i], i % 10) for i in range(N)], "img")
    try:
        order = rng.permutation(N)[:6 * BS].tolist()
        order[BS + 17] = N + 3  # batch 1, position 17: "Invalid count on target" (owner-0 fall-back)
        it = iter(PrefetchLoader(ds, order, BS))
        vals, labs = next(it)
        assert vals.cpu().numpy().tobytes() == imgs[order[:BS]].tobytes()
        del it  # the consumer stops: the loader's queue stays pending
        ids = [5, 1999, 0, 77]
        v, lab = ds.__getitems__(ids)
        assert ds.ddstore.last_bad_index == -1
        torch.cuda.synchronize()
        assert v.cpu().numpy().tobytes() == imgs[ids].tobytes() and lab.cpu().tolist() == [i % 10 for i in ids]
        with pytest.raises(ValueError) as ei:
            ds.ddstore.wait()
        assert str(ei.value) == "Invalid count on target" and ds.ddstore.last_bad_index == 17, \
            f"{ei.value} at {ds.ddstore.last_bad_index}, the loader's batch 1 fails at 17"
        assert ds.ddstore.wait() == 0 and ds.ddstore.last_bad_index == -1
    finally:
        ds.free()
        ds.ddstore.close()


def test_ragged_prefetch_loader_abandoned_mid_epoch():
    """the same for RaggedPrefetchLoader with a sample id below the index (-1: the loader sizes it from the host table,
    the gather rejects it)"""
    torch = _torch()
    from ddstore_b200.dataset import RaggedDataset, RaggedPrefetchLoader
    rng = np.random.default_rng(6)
    n = 500
    cnt = rng.integers(1, 6, size=n)
    ecnt = rng.integers(0, 4, size=n)
    x = rng.standard_normal((int(cnt.sum()), 5)).astype(np.float32)
    e = rng.integers(0, 1000, size=(int(ecnt.sum()), 2)).astype(np.int64)
    xs, es = np.concatenate([[0], np.cumsum(cnt)]), np.concatenate([[0], np.cumsum(ecnt)])
    ds = RaggedDataset({"x": x, "e": e}, {"x": cnt, "e": ecnt})
    try:
        BS = 32
        order = rng.permutation(n)[:5 * BS].tolist()
        order[BS + 9] = -1
        it = iter(RaggedPrefetchLoader(ds, order, BS))
        first = next(it)
        want = np.concatenate([x[xs[i]:xs[i + 1]] for i in order[:BS]])
        assert first["x"][0].cpu().numpy().tobytes() == want.tobytes()
        del it
        ids = [3, 499, 0]
        got = ds.__getitems__(ids)
        assert ds.ddstore.last_bad_index == -1
        torch.cuda.synchronize()
        assert got["x"][0].cpu().numpy().tobytes() == np.concatenate([x[xs[i]:xs[i + 1]] for i in ids]).tobytes()
        assert got["e"][0].cpu().numpy().tobytes() == np.concatenate([e[es[i]:es[i + 1]] for i in ids]).tobytes()
        with pytest.raises(ValueError) as ei:
            ds.ddstore.wait()
        assert "sample id" in str(ei.value) and ds.ddstore.last_bad_index == 9, \
            f"{ei.value} at {ds.ddstore.last_bad_index}, the loader's batch 1 fails at 9"
        assert ds.ddstore.wait() == 0 and ds.ddstore.last_bad_index == -1
    finally:
        ds.free()
        ds.ddstore.close()


# ------------------------------------------------------------------------------- a queue longer than the ordinal
LONG = 65_540
ORD_CAP = 65_535  # the first launch whose 16-bit ordinal would saturate


@pytest.mark.parametrize("overlap", (False, True))
@pytest.mark.parametrize("control", (False, True))
def test_queue_longer_than_the_ordinal(overlap, control):
    """65 540 fixed-count batches of 4 one-row requests, each into its own slice of one buffer. Launch 65 535 fails at
    request 3 ("Invalid start on target"), launch 65 536 at request 1 ("Invalid count on target"): wait() reports
    launch 65 535. The control adds a failure at launch 65 534, request 2, which wins over both."""
    torch = _torch()
    D = Data()

    def body(store, r):
        store.add("v", D.shards[r])
        if r:
            return True
        rng = np.random.default_rng(17)
        pool = [_fixed_ok(valid_requests(rng, 4, 1)[0]) for _ in range(7)]
        fails = {ORD_CAP: (3, "start_neg"), ORD_CAP + 1: (1, "start_past")}
        if control:
            fails[ORD_CAP - 1] = (2, "start_past")
        special = {}
        for k, (i, kind) in fails.items():
            s = pool[k % 7].copy()
            s[i] = invalid_request(kind, rng, 1)[0]
            special[k] = s
        d_pool = [torch.from_numpy(s).cuda() for s in pool]
        d_special = {k: torch.from_numpy(s).cuda() for k, s in special.items()}
        nb = 4 * ROW
        whole, view = guarded_buffer(torch, LONG * nb, 1, SENT)
        side = torch.cuda.Stream()
        for k in range(LONG):
            idx = d_special.get(k, d_pool[k % 7])
            store.get_batch("v", idx, out=view[k * nb:(k + 1) * nb], count=1, stream=side.cuda_stream, wait=False,
                            overlap=overlap)
        first = min(fails)
        want_i, want_kind = fails[first]
        want = {"start_neg": "Invalid start on target", "start_past": "Invalid count on target"}[want_kind]
        what = f"{LONG}-launch queue overlap={overlap} control={control}"
        with pytest.raises(ValueError) as ei:
            store.wait()
        assert str(ei.value) == want and store.last_bad_index == want_i, \
            f"{what}: wait() reported {ei.value!r} at {store.last_bad_index}; launch {first} fails with {want!r} at {want_i}"
        assert store.wait() == 0 and store.last_bad_index == -1
        torch.cuda.synchronize()
        w = whole.cpu().numpy()
        base = GUARD + 1
        assert np.all(w[:base] == SENT) and np.all(w[base + LONG * nb:] == SENT), f"{what}: a guard byte was written"
        got = w[base:base + LONG * nb].reshape(LONG, 4, ROW)
        rows = D.allrows.reshape(-1, ROW)
        exp = rows[np.clip(np.stack([special.get(k, pool[k % 7]) for k in range(LONG)]), 0, TOTAL - 1)]
        ok = np.ones(LONG, bool)
        ok[list(special)] = False
        bad = np.nonzero(np.any((got != exp).reshape(LONG, -1), axis=1) & ok)[0]
        assert bad.size == 0, f"{what}: batch {int(bad[0])} differs from the oracle"
        for k, s in special.items():  # the device-destination prefix rule: requests before the invalid one delivered,
            i = fails[k][0]             # the invalid one's slot untouched, later valid ones delivered or untouched
            assert np.array_equal(got[k, :i], exp[k, :i]), f"{what}: batch {k} before its invalid request {i}"
            assert np.all(got[k, i] == SENT), f"{what}: batch {k}: the slot of invalid request {i} was written"
            for j in range(i + 1, 4):
                assert np.all(got[k, j] == SENT) or np.array_equal(got[k, j], exp[k, j]), f"{what}: batch {k} request {j}"
        return True

    assert all(run_rank0(4, body, timeout=900))


# ------------------------------------------------------------------------------- the plan-tag wrap
TAG_START = 0x3FFFF0 - 20  # the 21st launch planned in global memory renews the tags (renew_plan_tags)


def plan_tag_wrap_scenario(store, torch, D):
    """40 batches planned in global memory across the wrap: explicit counts, get_samples and get_samples_multi; ten
    synchronous, twenty in one overlapped queue (the renewal falls in its middle), ten synchronous. Batch 25 (queued)
    and batch 36 (synchronous) fail after the wrap."""
    rng = np.random.default_rng(23)
    side = torch.cuda.Stream()
    kinds = ("var_global", "samples", "multi")
    bads = {25: (61, 0), 36: (5, 1)}
    queued = []
    for k in range(40):
        kind = kinds[k % 3]
        idx, exps = make_batch(D, kind, rng, bads.get(k), B=3000)
        q = Queued(torch, kind, idx, exps, [e.T + 16 for e in exps], k % 5)
        what = f"plan-tag wrap batch {k} ({kind})"
        if 10 <= k < 30:
            q.launch(store, side.cuda_stream, False, True)
            queued.append((k, q))
            continue
        got = []
        expect_raise(store, lambda: got.append(q.launch(store, None, True)), exps[0], False, what)
        if not bads.get(k):
            assert (got[0] if kind != "multi" else sum(got[0])) == q.total(), f"{what}: returned {got}"
        q.check(what)
    with pytest.raises(ValueError) as ei:
        store.wait()
    e25 = queued[15][1].exps[0]
    assert error_text(e25.code) in str(ei.value) and store.last_bad_index == e25.bad, \
        f"plan-tag wrap queue: wait() reported {ei.value!r} at {store.last_bad_index}, batch 25 fails at {e25.bad}"
    for k, q in queued:
        q.check(f"plan-tag wrap batch {k} (queued)")
    # a clean overlapped queue after the wrap, and its total
    qs = []
    for k in range(6):
        idx, exps = make_batch(D, kinds[k % 3], rng, B=3000)
        qs.append(Queued(torch, kinds[k % 3], idx, exps, [e.T + 16 for e in exps], k))
        qs[-1].launch(store, side.cuda_stream, False, True)
    assert store.wait() == qs[-1].total()
    for k, q in enumerate(qs):
        q.check(f"plan-tag wrap: clean queue batch {k}")


WRAP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
import torch
from tests import test_gpu_queue_end as T
D = T.Data()
def body(store, r):
    D.add(store, r)
    if r == 0:
        T.plan_tag_wrap_scenario(store, torch, D)
    return True
assert all(T.run_rank0(4, body))
print("wrap-ok")
"""


def test_plan_tag_wrap(tmp_path):
    """DDS_PLAN_TAG_START starts the 22-bit counter 20 launches below the renewal threshold"""
    script = tmp_path / "wrap.py"
    script.write_text(WRAP_SCRIPT.format(root=ROOT))
    r = subprocess.run([sys.executable, str(script)], env=dict(os.environ, DDS_PLAN_TAG_START=hex(TAG_START)),
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "wrap-ok" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
