"""helpers for the -m gpu parity tests: thread-rank worlds over one or more GPUs (test infrastructure)"""
import threading
import uuid

import numpy as np


def run_world(P, body, devices=None, timeout=300):
    """Run `body(store, rank)` on P thread-ranks (ShmComm across threads). devices[r] = CUDA ordinal of
    rank r (default: all on device 0 -- owner lookup and peer-table logic are exercised even on one GPU;
    with >= P GPUs pass range(P) for real NVLink peer loads)."""
    from ddstore_b200 import PyDDStore, ShmComm
    key = "g" + uuid.uuid4().hex[:12]
    res, errs = [None] * P, []

    def run(r):
        comm = store = None
        try:
            comm = ShmComm(key, r, P)
            store = PyDDStore(comm, device=(devices[r] if devices else 0))
            res[r] = body(store, r)
            store.free()
        except BaseException as e:  # noqa: BLE001
            import traceback
            errs.append((r, traceback.format_exc()))
        finally:
            if store is not None:
                store.close()
            if comm is not None:
                comm.close()

    th = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(P)]
    [t.start() for t in th]
    [t.join(timeout) for t in th]
    hung = [r for r, t in enumerate(th) if t.is_alive()]
    assert not hung, f"ranks {hung} did not finish within {timeout} s"
    assert not errs, "\n".join(f"rank {r}: {tb}" for r, tb in errs)
    return res


def packed_nbytes(counts, row):
    return int(np.clip(np.asarray(counts, np.int64), 0, None).sum()) * row


# ------------------------------------------------------------------------------- guarded destinations
GUARD = 64                     # sentinel bytes kept on each side of a destination
DST_OFFSETS = (0, 1, 4, 8, 13)  # destination base offsets (bytes past a 16-byte-aligned allocation)


def guarded_buffer(torch, nbytes, off, sentinel, device="cuda:0"):
    """A device buffer [GUARD + off sentinel bytes | nbytes | GUARD] filled with `sentinel`; returns (whole, view of the
    nbytes in the middle). The view starts `off` bytes past a 16-byte boundary. The fill has completed on return (the
    store's own stream is not ordered with torch's)."""
    whole = torch.full((2 * GUARD + off + nbytes,), sentinel, dtype=torch.uint8, device=device)
    torch.cuda.synchronize(device)
    return whole, whole[GUARD + off:GUARD + off + nbytes]


def mismatch_report(got, exp, exp_offs, starts, counts, what):
    """None when got == exp (uint8 arrays), else a message naming the first bad byte, its request and the request's
    (start, count, packed offset)"""
    if got.size == exp.size and np.array_equal(got, exp):
        return None
    if got.size != exp.size:
        return f"{what}: {got.size} bytes delivered, oracle {exp.size}"
    bad = np.nonzero(got != exp)[0]
    pos = int(bad[0])
    req = int(np.searchsorted(exp_offs, pos, side="right") - 1)
    return (f"{what}: {bad.size} bytes differ; first at packed byte {pos}, in request {req} (start={int(starts[req])}, "
            f"count={int(counts[req])}, packed offset={int(exp_offs[req])}, byte {pos - int(exp_offs[req])} of it): "
            f"got {int(got[pos]):#04x}, expected {int(exp[pos]):#04x}")


def check_guarded(whole, off, exp, exp_offs, starts, counts, sentinel, what, total=None, got_offs=None, slack_written=False):
    """Check a delivery into guarded_buffer(): the packed bytes equal the oracle's `exp`, the returned total and byte
    offsets equal the oracle's, and every byte before the base and after the packed end still holds the sentinel
    (slack_written: an earlier, larger batch used the same buffer, so only the GUARD bytes past its end are checked)."""
    w = whole.cpu().numpy() if hasattr(whole, "cpu") else whole
    base, n = GUARD + off, exp.size
    if total is not None:
        assert total == n, f"{what}: returned total {total}, oracle {n}"
    if got_offs is not None:
        go = got_offs.cpu().numpy() if hasattr(got_offs, "cpu") else np.asarray(got_offs)
        go = go[:len(exp_offs)]
        if not np.array_equal(go, exp_offs):
            i = int(np.nonzero(go != exp_offs)[0][0])
            raise AssertionError(f"{what}: offsets[{i}] = {int(go[i])}, oracle {int(exp_offs[i])}"
                                 + (f" (request start={int(starts[i])}, count={int(counts[i])})" if i < len(starts) else ""))
    pre = np.nonzero(w[:base] != sentinel)[0]
    assert pre.size == 0, f"{what}: byte {int(pre[-1]) - base} (before the destination base) was written"
    msg = mismatch_report(w[base:base + n], exp, exp_offs, starts, counts, what)
    assert msg is None, msg
    tail0 = w.size - GUARD if slack_written else base + n
    post = np.nonzero(w[tail0:] != sentinel)[0]
    assert post.size == 0, f"{what}: byte {int(post[0]) + tail0 - base} past the packed end ({n}) was written"


# ------------------------------------------------------------------------------- the variant sweep's workload
def sweep_sizes(chunks):
    """request byte sizes around the walk's thresholds for chunk sizes `chunks` (stage = chunk + 32)"""
    sizes = set(range(1, 34))
    for ch in chunks:
        st = ch + 32
        sizes |= {ch // 2 - 1, ch // 2, ch // 2 + 1, ch - 1, ch, ch + 1, ch + 15, ch + 16, ch + 17, st - 1, st + 1,
                  2 * ch - 1, 2 * ch + 1}
    # the plan's segment grain (16 KiB), the largest segment (1 MiB), and multi-MiB requests
    sizes |= {16383, 16385, (1 << 20) - 1, (1 << 20) + 1, 3 << 20, (5 << 20) + 7}
    return sorted(sizes)


def sweep_requests(rng, nrows, row, chunks):
    """(starts, counts) of one variable-count workload over a single shard of `nrows` rows of `row` bytes: every size of
    sweep_sizes() at rotating source phases, every source x destination phase (1-byte rows), a run of > 32 tiny
    requests, runs of small requests whose padded sizes overflow a stage mid-group, zero-count requests first, last and
    in between. Requests are valid by construction."""
    def rows_for(nbytes):
        return max(1, -(-nbytes // row))

    def start_for(cnt, phase=None):
        hi = nrows - max(cnt, 1)
        assert hi >= 0, (nrows, cnt)
        if phase is None or row != 1:
            return int(rng.integers(0, hi + 1))
        return int(rng.integers(0, (hi - phase) // 16 + 1)) * 16 + phase

    blk = [(rows_for(s), i % 16) for i, s in enumerate(sweep_sizes(chunks))]
    blk = [blk[i] for i in rng.permutation(len(blk))]
    reqs = [(start_for(c, ph), c) for c, ph in blk]
    if row == 1:  # 49-byte requests: the destination phase moves by one per request, the source phase by one per 16
        reqs += [(start_for(49, i // 16), 49) for i in range(256)]
    reqs += [(start_for(1), 1) for _ in range(40)]  # longer than the walk's 32-request window
    reqs += [(start_for(c), c) for c in rng.integers(1, 4, size=45).tolist()]
    for ch in chunks:  # ~ch/5-byte requests: a stage fills up after four or five of them, in the middle of a group
        c = rows_for(ch // 5 + 3)
        reqs += [(start_for(c, k % 16), c) for k in range(8)]
    for _ in range(len(reqs) // 20):
        reqs.insert(int(rng.integers(1, len(reqs))), (start_for(0), 0))
    reqs = [(start_for(0), 0)] + reqs + [(start_for(0), 0)]
    st, ct = np.array(reqs, np.int64).T
    return np.ascontiguousarray(st), np.ascontiguousarray(ct)


def padded_requests(rng, nrows, starts, counts, n, max_count=2):
    """the same requests with tiny (0..max_count-row) ones inserted at random places, n in all (first and last stay
    put)"""
    k = n - len(starts)
    pos = rng.integers(1, len(starts), size=k)
    return (np.insert(starts, pos, rng.integers(0, nrows - max_count, size=k)).astype(np.int64),
            np.insert(counts, pos, rng.integers(0, max_count + 1, size=k)).astype(np.int64))


def sample_ids(rng, nbytes, n):
    """n sample ids over samples of `nbytes` bytes each: every sample once, the rest drawn from the small (<= 4 KiB)
    ones, shuffled -- a long id list that does not repeat the multi-MiB samples thousands of times"""
    small = np.nonzero(np.asarray(nbytes) <= 4096)[0]
    ids = np.concatenate([np.arange(len(nbytes)), rng.choice(small, size=max(0, n - len(nbytes)))])
    return rng.permutation(ids)[:n].astype(np.int64)


# ------------------------------------------------------------------------------- invalid requests and their expected result
INT64_MAX = (1 << 63) - 1
CODE_SAMPLE = 15  # a sample id outside the variable's sample index (no counterpart in the reference)


def classify(lenlist, starts, counts):
    """per-request result of the serial get() loop: 0, 2 ("Invalid start on target") or 3 ("Invalid count on target"),
    with the documented divergences (negative and overflowing counts are count errors). Vectorised restatement of
    oracle.np_locate, checked against it on every invalid request and on a sample of the valid ones."""
    from oracle import oracle as O
    ll = np.asarray(lenlist, np.int64)
    s = np.asarray(starts, np.int64)
    c = np.asarray(counts, np.int64)
    k = np.searchsorted(ll, s, side="right")  # ll[k-1] <= s < ll[k]: the owner (src/ddstore.cxx:5-17), else owner 0
    t = np.where((k >= 1) & (k < len(ll)), k, 0)
    off = np.where(t > 0, ll[np.maximum(t - 1, 0)], 0)
    with np.errstate(over="ignore"):
        room = ll[t] - s  # (only used where s >= off >= 0: no wrap there)
    codes = np.where(s < off, 2, np.where((c < 0) | (c > room), 3, 0)).astype(np.int64)
    check = np.nonzero(codes)[0].tolist()[:3000] + list(range(0, len(s), max(1, len(s) // 500)))
    for i in check:
        assert O.np_locate(ll, int(s[i]), int(c[i]))[2] == codes[i], (int(s[i]), int(c[i]))
    return codes


class Expected:
    """What a batch must leave behind. codes: per-request oracle result; nbytes: bytes of every request in the store's
    packed layout (fixed counts keep a slot of count * row bytes for every request, variable counts pack an invalid
    request as zero bytes); offs: its exclusive scan; lay: the layout with every VALID request's rows in place and
    `valid` marking those bytes; bad: the first invalid request (-1: none); prefix: bytes the serial loop delivers."""

    def __init__(self, allrows, row, lenlist, starts, counts, fixed, codes=None, shards=None):
        starts = np.asarray(starts, np.int64)
        counts = np.asarray(counts, np.int64)
        total = int(lenlist[-1])
        self.codes = classify(lenlist, starts, counts) if codes is None else np.asarray(codes, np.int64)
        ok = self.codes == 0
        bad = np.nonzero(~ok)[0]
        self.bad = int(bad[0]) if bad.size else -1
        self.code = int(self.codes[self.bad]) if bad.size else 0
        sane = (counts > 0) & (counts <= total)  # (a larger count is invalid for every start, and packs nothing)
        self.nbytes = np.where(sane & (ok | fixed), counts, 0) * row
        self.offs = np.concatenate([[0], np.cumsum(self.nbytes)]).astype(np.int64)
        self.T = int(self.offs[-1])
        self.prefix = int(self.offs[self.bad]) if self.bad >= 0 else self.T
        self.lay = np.zeros(self.T, np.uint8)
        self.valid = np.zeros(self.T, bool)
        v = np.nonzero(ok & (counts > 0))[0]
        if v.size:
            nb = counts[v] * row
            dst = np.repeat(self.offs[v] - np.concatenate([[0], np.cumsum(nb)[:-1]]), nb) + np.arange(int(nb.sum()))
            src = np.repeat(starts[v] * row - np.concatenate([[0], np.cumsum(nb)[:-1]]), nb) + np.arange(int(nb.sum()))
            self.lay[dst] = allrows[src]
            self.valid[dst] = True
        n = self.bad if self.bad >= 0 else len(starts)
        if shards is not None and n <= 20_000:  # the prefix is the oracle's serial loop, byte for byte
            from oracle import oracle as O
            pre, pre_offs, pbad, _ = O.np_get_batch(shards, starts[:n], counts[:n])
            assert pbad == -1 and pre.size == self.prefix and np.array_equal(pre, self.lay[:self.prefix])
            assert np.array_equal(pre_offs, self.offs[:n + 1])

    def request_of(self, pos):
        return int(np.searchsorted(self.offs, pos, side="right") - 1)


def error_text(code):
    from oracle import oracle as O
    return "sample id" if code == CODE_SAMPLE else O.ERR_TEXT[code]


def expect_raise(store, call, exp, over, what):
    """run `call`; it must raise exactly the oracle's first error (an invalid request wins over a capacity error) with
    last_bad_index = its index, or succeed when there is none"""
    try:
        call()
        got = None
    except ValueError as e:
        got = str(e)
    if exp.bad >= 0:
        want = error_text(exp.code)
        assert got is not None and (want in got if exp.code == CODE_SAMPLE else got == want), \
            f"{what}: raised {got!r}, oracle: {want!r} at request {exp.bad}"
        assert store.last_bad_index == exp.bad, f"{what}: last_bad_index {store.last_bad_index}, oracle {exp.bad}"
    elif over:
        assert got is not None and "too small" in got, f"{what}: raised {got!r}, expected a capacity error"
        assert store.last_bad_index == -1, f"{what}: last_bad_index {store.last_bad_index} on a capacity error"
    else:
        assert got is None, f"{what}: raised {got!r} on a valid batch"


class Dest:
    """A destination of `nbytes` between GUARD-byte sentinel bands: kind 'device' (guarded_buffer), 'pinned' or
    'pageable' (a numpy view into a larger sentinel-filled host array)"""

    def __init__(self, torch, kind, nbytes, sentinel, off=0):
        self.torch, self.kind, self.nbytes, self.sentinel, self.off = torch, kind, int(nbytes), sentinel, off
        n = 2 * GUARD + off + self.nbytes
        if kind == "device":
            self.whole, self.view = guarded_buffer(torch, self.nbytes, off, sentinel)
        else:
            self.whole = torch.full((n,), sentinel, dtype=torch.uint8).pin_memory().numpy() if kind == "pinned" else \
                np.full(n, sentinel, np.uint8)
            self.view = self.whole[GUARD + off:GUARD + off + self.nbytes]

    def reset(self):
        if self.kind == "device":
            self.whole.fill_(self.sentinel)
            self.torch.cuda.synchronize()
        else:
            self.whole[:] = self.sentinel

    def host(self):
        return self.whole.cpu().numpy() if self.kind == "device" else self.whole.copy()


def check_dest(dest, exp, over, what, offsets=None):
    """The destination after a call (see expect_raise): no guard byte written; a capacity error leaves every byte
    untouched; else bytes [0, prefix) are the oracle's and every later byte is the sentinel -- host destinations, the
    serial loop's result exactly -- or, on the device, also may be a byte of a VALID request at the offset the store
    packs it to. offsets (when requested) equal the oracle's up to the first invalid request."""
    w = dest.host()
    base, n, s = GUARD + dest.off, dest.nbytes, dest.sentinel
    pre = np.nonzero(w[:base] != s)[0]
    assert pre.size == 0, f"{what}: guard byte {int(pre[-1]) - base} (before the destination) was written"
    post = np.nonzero(w[base + n:] != s)[0]
    assert post.size == 0, f"{what}: guard byte {int(post[0])} past the destination's end was written"
    d = w[base:base + n]
    if over:
        hit = np.nonzero(d != s)[0]
        assert hit.size == 0, f"{what}: capacity error, yet byte {int(hit[0])} of the destination was written"
        return
    p = exp.prefix
    diff = np.nonzero(d[:p] != exp.lay[:p])[0]
    if diff.size:
        i = int(diff[0])
        r = exp.request_of(i)
        raise AssertionError(f"{what}: byte {i} of the delivered prefix (request {r}, packed offset {int(exp.offs[r])}) is "
                             f"{int(d[i]):#04x}, oracle {int(exp.lay[i]):#04x}")
    rest = d[p:]
    lay = np.full(rest.size, s, np.uint8)
    ok_mask = np.zeros(rest.size, bool)
    m = min(exp.T, n) - p
    if dest.kind == "device" and m > 0:
        ok_mask[:m] = exp.valid[p:p + m]
        lay[:m] = exp.lay[p:p + m]
    bad = np.nonzero((rest != s) & ~(ok_mask & (rest == lay)))[0]
    if bad.size:
        i = p + int(bad[0])
        r = exp.request_of(i) if i < exp.T else None
        where = (f"request {r} (code {int(exp.codes[r])}, packed offset {int(exp.offs[r])})" if r is not None
                 else "past the packed end")
        raise AssertionError(f"{what}: byte {i} after the first invalid request ({exp.bad}) was written "
                             f"({int(rest[bad[0]]):#04x}); it lies in {where}")
    if offsets is not None:
        go = offsets.cpu().numpy() if hasattr(offsets, "cpu") else np.asarray(offsets)
        k = (exp.bad if exp.bad >= 0 else len(exp.offs) - 1) + 1
        diff = np.nonzero(go[:k] != exp.offs[:k])[0]
        assert diff.size == 0, f"{what}: offsets[{int(diff[0])}] = {int(go[diff[0]])}, oracle {int(exp.offs[diff[0]])}"
