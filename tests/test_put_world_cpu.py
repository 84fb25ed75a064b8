"""tests/put_world.py without a GPU: the generators produce the edges they claim, the expectation of a whole epoch does
not depend on the order of its writers, equals the compiled reference, and a wrong shard is reported with the rank, the
row and the requests that cover it."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import put_oracle as po
from tests import put_world as pw

SIXTY_FOUR_EMPTY = {0, 1, 2, 9, 10, 17, 23, 24, 25, 26, 31, 32, 40, 47, 48, 55, 58, 59, 60, 61, 63}


def sixty_four_rows():
    rng = np.random.default_rng(64)
    nrows = [0 if r in SIXTY_FOUR_EMPTY else int(rng.integers(2, 40)) for r in range(64)]
    nrows[3] = nrows[62] = 1
    return nrows


WORLDS = {"empty-first-last-middle": [0, 5, 0, 1, 7, 0], "empty-run": [3, 0, 0, 4], "one-row-ranks": [1, 1, 1],
          "one-owner": [0, 9, 0], "uneven": [40, 1, 13], "sixty-four": sixty_four_rows()}


@pytest.mark.parametrize("world", list(WORLDS))
def test_edge_generators_produce_every_class(world):
    nrows = WORLDS[world]
    ll = pw.lenlist_of(nrows)
    pairs = len(pw.owners(ll)) > 1
    for writer in range(3):
        rng = np.random.default_rng([5, writer])
        first_bad = 3 + 2 * writer
        st, ct, cls = pw.edge_requests(rng, ll, writer, first_bad=first_bad)
        want = pw.EDGE_CLASSES | pw.INVALID_CLASSES | (pw.PAIR_CLASSES if pairs else set())
        assert set(cls) == want, (want - set(cls), set(cls) - want)
        codes = [po.locate(ll, int(s), int(c))[0] for s, c in zip(st, ct)]
        assert next(i for i, c in enumerate(codes) if c) == first_bad  # the first invalid request is where it was put
        for s, c, k, code in zip(st.tolist(), ct.tolist(), cls, codes):
            if k in pw.INVALID_CLASSES or k == "straddle":
                assert code, (s, c, k)
            if k == "tail":  # ends exactly on its owner's last row
                assert code == 0 and s + c in ll.tolist()
            if k == "whole":
                t = po.sortedsearch(ll, s)
                assert code == 0 and c == nrows[t] and s + c == ll[t]
        # only requests the oracle accepts without first_bad, and none of the valid classes is lost
        st2, ct2, cls2 = pw.edge_requests(np.random.default_rng([5, writer]), ll, writer)
        assert all(po.locate(ll, int(s), int(c))[0] == 0 for s, c in zip(st2, ct2))
        assert set(cls2) >= (pw.EDGE_CLASSES - {"zero_at_total"}) | (pw.PAIR_CLASSES - {"straddle"} if pairs else set())
        # the sample-id form: ids -1 and nsamples keep no bytes and are the first error
        batch, cls3 = pw.as_samples(rng, st2, ct2, cls2, first_bad=2)
        assert set(cls3) >= pw.SAMPLE_CLASSES
        shards = [np.zeros((n, 3), np.uint8) for n in nrows]
        src = pw.layout_src(pw.pattern_world(1, ll, 3, 1), ll, 3, batch)
        new, codes, bad, total = po.put(shards, src, **batch)
        assert bad == 2 and codes[2] == po.CODE_SAMPLE and total == src.size == int(ct2.sum()) * 3
        for cnt in (1, 3):
            fs, fcls = pw.edge_fixed(rng, ll, cnt, first_bad=1)
            assert {"start_at_total", "start_negative"} <= set(fcls)
            if any(n >= cnt for n in nrows):
                assert {"first", "tail"} <= set(fcls)
            if cnt > 1:
                assert "straddle" in fcls
            codes = [po.locate(ll, int(s), cnt)[0] for s in fs]
            assert [bool(c) for c in codes] == [k in ("straddle", "start_at_total", "start_negative") for k in fcls]


def _epoch(seed, nrows, R, P, epoch=1):
    ll = pw.lenlist_of(nrows)
    pat = pw.pattern_world(seed, ll, R, epoch)
    puts = []
    for w in range(P):
        st, ct, _ = pw.edge_requests(np.random.default_rng([seed, w]), ll, w, first_bad=2 + w)
        puts.append([pw.Put({"starts": st, "counts": ct}, pat)])
    return ll, pat, pw.split_world(pw.pattern_world(seed, ll, R, 0), ll, R), puts


def test_patterns_and_filler_differ_everywhere():
    ll = pw.lenlist_of([4, 0, 9])
    e = [pw.pattern_world(3, ll, 6, k) for k in range(7)]
    for i in range(7):
        for j in range(7):
            assert i == j or (e[i] != e[j]).all()
            assert ((e[i] + np.uint8(128)) != e[j]).all()  # an invalid request's filler is no epoch's byte
    # an invalid request keeps its bytes in the layout, as filler; the requests behind it are read where they lie
    batch = {"starts": np.array([3, 2, 12, 4], np.int64), "counts": np.array([2, 1, 3, 2], np.int64)}
    src = pw.layout_src(e[1], ll, 6, batch)
    assert src.size == 8 * 6
    assert (src[:6] == e[1][18:24] + np.uint8(128)).all() and (src[6:12] == e[1][24:30] + np.uint8(128)).all()
    assert (src[12:18] == e[1][12:18]).all()
    assert (src[18:24] == e[1][72:78] + np.uint8(128)).all() and (src[24:36] == pw.FILL_OUTSIDE).all()
    assert (src[36:] == e[1][24:36]).all()


@pytest.mark.parametrize("world", ["empty-first-last-middle", "uneven", "sixty-four"])
def test_expected_world_is_independent_of_writer_order(world):
    nrows, R, P = WORLDS[world], 6, 4
    ll, pat, shards, puts = _epoch(9, nrows, R, P)
    new, status = pw.expected_world(shards, puts)
    for order in ([3, 2, 1, 0], [1, 3, 0, 2]):
        new2, status2 = pw.expected_world(shards, [puts[w] for w in order])
        assert all(a.tobytes() == b.tobytes() for a, b in zip(new, new2))
        assert [status[w] for w in order] == status2
    for w in range(P):  # every writer has its own first invalid request
        assert status[w][0][1] == 2 + w and status[w][0][0] in (po.CODE_START, po.CODE_COUNT)
    # a short source on one writer: that call writes nothing and reports its invalid request, the others land
    short = [list(c) for c in puts]
    short[1] = [pw.Put(puts[1][0].batch, pat, src_bytes=5)]
    new3, status3 = pw.expected_world(shards, short)
    assert status3[1][0] == status[1][0]
    without, _ = pw.expected_world(shards, [puts[0], puts[2], puts[3]])
    assert all(a.tobytes() == b.tobytes() for a, b in zip(new3, without))


@pytest.mark.parametrize("R,P", [(1, 3), (3, 4), (20, 3), (4096, 4)])
def test_interleaved_cover_writes_every_byte_once(R, P):
    nrows = [0, 700, 1, 0, 1300, 260] if R < 4096 else [0, 300, 1, 600]
    ll = pw.lenlist_of(nrows)
    rng = np.random.default_rng(R)
    cover = pw.interleaved_cover(rng, ll, P, R)
    hits = np.zeros(int(ll[-1]), np.int64)
    writer_of = np.full(int(ll[-1]), -1)
    for w, (st, ct) in enumerate(cover):
        assert all(po.locate(ll, int(s), int(c))[0] == 0 and c > 0 for s, c in zip(st, ct))
        for s, c in zip(st.tolist(), ct.tolist()):
            hits[s:s + c] += 1
            writer_of[s:s + c] = w
    assert (hits == 1).all()
    cuts = np.nonzero(np.diff(writer_of))[0].size  # neighbouring requests have different writers
    assert cuts >= sum(len(st) for st, _ in cover) - len(pw.owners(ll)) - P
    if R == 4096:
        assert max(int(ct.max()) for _, ct in cover) * R > 1 << 20
    pat = pw.pattern_world(2, ll, R, 1)
    shards = pw.split_world(pw.pattern_world(2, ll, R, 0), ll, R)
    new, status = pw.expected_world(shards, [[pw.Put({"starts": s, "counts": c}, pat)] for s, c in cover])
    assert np.concatenate([x.reshape(-1) for x in new]).tobytes() == pat.tobytes()
    assert all(s[0][:2] == (0, -1) for s in status)
    for n in (1, 1024, 1025, 2260):
        st, ct = pw.dense_cover(rng, 2260, n)
        assert len(st) == n and ct.min() >= 1 and np.array_equal(np.sort(np.concatenate(
            [np.arange(s, s + c) for s, c in zip(st, ct)])), np.arange(2260))


def test_a_wrong_shard_is_reported_with_rank_row_and_requests():
    """the comparison the GPU tests use, against expectations that are wrong on purpose"""
    nrows, R = [0, 5, 0, 1, 7, 0], 6
    ll, pat, shards, puts = _epoch(4, nrows, R, 3)
    good, status = pw.expected_world(shards, puts)
    raw = lambda sh: np.concatenate([sh.reshape(-1), np.zeros(16, np.uint8)])  # noqa: E731
    for r in range(len(nrows)):
        assert pw.shard_mismatch(raw(good[r]), 16, good[r], r, ll, R, puts, "ok") is None
    # one request dropped from a writer's batch in the expectation (a cover: every row has exactly one request)
    cover = pw.interleaved_cover(np.random.default_rng(1), ll, 3, R, big=False)
    cputs = [[pw.Put({"starts": s, "counts": c}, pat)] for s, c in cover]
    full, _ = pw.expected_world(shards, cputs)
    st, ct = cover[1]
    j, row = 2, int(st[2])
    rank = po.sortedsearch(ll, row)
    dropped = list(cputs)
    dropped[1] = [pw.Put({"starts": np.delete(st, j), "counts": np.delete(ct, j)}, pat)]
    wrong, _ = pw.expected_world(shards, dropped)
    msg = pw.shard_mismatch(raw(full[rank]), 16, wrong[rank], rank, ll, R, cputs, "dropped")
    assert msg and f"rank {rank}:" in msg and f"global row {row}," in msg, msg
    assert f"writer 1 call 0 request {j} ({row}, {int(ct[j])})" in msg, msg
    # one pattern byte flipped: rank 4, global row 8, byte 2
    flipped = [g.copy() for g in good]
    flipped[4][2, 2] ^= 1
    msg = pw.shard_mismatch(raw(good[4]), 16, flipped[4], 4, ll, R, puts, "flipped")
    assert msg and "rank 4" in msg and "global row 8, byte 2" in msg and "writer" in msg, msg
    # a boundary request moved by one row: (lo, whole shard of rank 1) shifted up leaves row 0 of rank 1 unwritten
    solo = [[pw.Put({"starts": np.array([0]), "counts": np.array([5])}, pat)]]
    moved = [[pw.Put({"starts": np.array([1]), "counts": np.array([4])}, pat)]]
    a, _ = pw.expected_world(shards, solo)
    bsh, _ = pw.expected_world(shards, moved)
    msg = pw.shard_mismatch(raw(a[1]), 16, bsh[1], 1, ll, R, solo, "moved")
    assert msg and "rank 1" in msg and "global row 0, byte 0" in msg and "request 0 (0, 5)" in msg, msg
    # a written slack byte
    bad = raw(good[1])
    bad[-3] = 7
    assert "slack byte 13" in pw.shard_mismatch(bad, 16, good[1], 1, ll, R, puts, "slack")
    # the status triple: the second invalid request is not the first
    b = puts[1][0].batch
    codes = [po.locate(ll, int(s), int(c))[0] for s, c in zip(b["starts"], b["counts"])]
    second = [i for i, c in enumerate(codes) if c][1]
    assert status[1][0][1] != second and status[1][0][1] == 3


@pytest.mark.skipif(not O.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("world", ["empty-first-last-middle", "empty-run", "one-row-ranks", "uneven"])
def test_expected_world_vs_compiled_reference(world):
    """every writer's valid requests applied as the owner's update(owner, name, rows, start - lenlist[owner-1]) of the
    unmodified reference, the state read back with its own get(): the expectation of the epoch"""
    nrows, disp, P = WORLDS[world], 2, 3
    R = disp * 4
    ll, pat, shards8, puts = _epoch(21, nrows, R, P)
    cover = pw.interleaved_cover(np.random.default_rng(8), ll, P, R, big=False)
    for w, (s, c) in enumerate(cover):
        puts[w].append(pw.Put({"starts": s, "counts": c}, pat))
    new, _ = pw.expected_world(shards8, puts)
    w = O.RefWorld(len(nrows))
    try:
        w.add("x", [s.view(np.int32) for s in shards8])
        for k in range(2):  # (the calls of one writer are ordered; the writers are not)
            for calls in puts:
                p = calls[k]
                src = pw.layout_src(p.pattern, ll, R, p.batch)
                o = 0
                for s, n, _ in po.requests(**p.batch):
                    nb = n * R if 0 < n <= int(ll[-1]) else 0
                    if nb and po.locate(ll, s, n)[0] == 0:
                        t = w.sortedsearch(ll, s)
                        w.update(t, "x", src[o:o + nb].view(np.int32).reshape(n, disp), s - (int(ll[t - 1]) if t else 0))
                    o += nb
        for r, sh in enumerate(new):
            if sh.shape[0]:
                got = np.empty((sh.shape[0], disp), np.int32)
                w.get((r + 1) % len(nrows), "x", got, int(ll[r - 1]) if r else 0)
                assert got.tobytes() == sh.tobytes(), f"rank {r}"
    finally:
        w.close()
