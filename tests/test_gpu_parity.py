"""Parity tests proper (-m gpu): the CUDA path, called through the C-ABI (ddstore_b200._capi via PyDDStore),
against the oracle and the committed golden vectors. Bit-exact: every comparison is on raw bytes."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.gpu_helpers import packed_nbytes, run_world
from tests.helpers import golden_world_shards, load_golden, random_valid_requests, random_world, sha

pytestmark = pytest.mark.gpu
G = load_golden()


def _torch():
    import torch
    return torch


# ------------------------------------------------------------------------------- golden vectors
@pytest.mark.parametrize("w", G["worlds"], ids=[w["name"] for w in G["worlds"]])
def test_golden_worlds(w):
    P = len(w["nrows"])
    shards = golden_world_shards(w)
    dtype = np.dtype(w["dtype"])
    row = w["disp"] * dtype.itemsize

    def body(store, r):
        store.add("v", shards[r])
        q = store.query("v")
        assert q["lenlist"] == w["lenlist"] and q["disp"] == w["disp"] and q["itemsize"] == w["itemsize"]
        if r != w["rank"]:
            return None
        good = []
        for req in w["requests"]:
            buf = np.zeros((req["count"], w["disp"]), dtype)
            if "error" in req:
                with pytest.raises(ValueError) as ei:
                    store.get("v", buf, req["start"])
                assert str(ei.value) == req["error"]
            else:
                store.get("v", buf, req["start"])
                assert sha(buf.tobytes()) == req["sha256"]
                if "hex" in req:
                    assert buf.tobytes().hex() == req["hex"]
                good.append((req["start"], req["count"]))
        st, ct = [g[0] for g in good], [g[1] for g in good]
        out = np.zeros(w["batch_nbytes"], np.uint8)
        offs = np.zeros(len(st) + 1, np.int64)
        n = store.get_batch("v", st, ct, out=out, offsets=offs)
        assert n == w["batch_nbytes"] and sha(out.tobytes()) == w["batch_sha256"]
        assert offs.tolist() == np.concatenate([[0], np.cumsum(np.array(ct) * row)]).tolist()
        # the whole request list incl. the invalid ones: first bad index + the reference's text
        st = [r_["start"] for r_ in w["requests"]]
        ct = [r_["count"] for r_ in w["requests"]]
        first_bad = next((i for i, r_ in enumerate(w["requests"]) if "error" in r_), None)
        if first_bad is not None:
            out2 = np.zeros(max(packed_nbytes(ct, row), 16), np.uint8)
            with pytest.raises(ValueError) as ei:
                store.get_batch("v", st, ct, out=out2)
            assert str(ei.value) == w["requests"][first_bad]["error"] and store.last_bad_index == first_bad
            # requests before the first bad one were delivered, like the serial loop
            pre = packed_nbytes(ct[:first_bad], row)
            exp, _, _, _ = O.np_get_batch(shards, st[:first_bad], ct[:first_bad])
            assert out2[:pre].tobytes() == exp.tobytes()
        return True

    res = run_world(P, body)
    assert res[w["rank"]] is True


def test_demo_cxx_known_answer():
    # test/demo.cxx:20-37 at P=2
    def body(store, r):
        buffer = np.array([1, 2, 3, 4], np.float64).reshape(2, 2) + 10 * r
        store.add("var", buffer)
        getbuf = np.zeros((1, 2), np.float64)
        start = (2 * (r + 1)) % (2 * 2) + 1
        store.get("var", getbuf, start)
        return getbuf.reshape(-1).tolist()

    assert run_world(2, body) == [[13.0, 14.0], [3.0, 4.0]]
    assert [d["got"] for d in G["demo_cxx"]] == [[13.0, 14.0], [3.0, 4.0]]


@pytest.mark.parametrize("dt", ["float64", "float32"])
def test_demo_py_mean_property(dt):
    # test/demo.py:35-56 / test/test.py:144-159: shard r is all (r+1); mean(row idx) == idx//num + 1
    rec = G["demo_py"][dt]
    num, dim = rec["num"], rec["dim"]

    def body(store, r):
        store.add("var", np.ones((num, dim), dt) * (r + 1))
        means = []
        for idx in rec["idx"]:
            buff = np.zeros((1, dim), dt)
            store.epoch_begin()
            store.get("var", buff, idx)
            store.epoch_end()
            means.append(float(np.mean(buff)))
        return means

    for means in run_world(rec["P"], body):
        assert means == rec["means"] == [i // num + 1 for i in rec["idx"]]


# ------------------------------------------------------------------------------- random worlds vs the oracle
CASES = [(np.float32, 1, 4), (np.float32, 16, 8), (np.int64, 2, 3), (np.uint8, 7, 2), (np.float64, 5, 1),
         (np.int32, 3, 5), (np.bool_, 3, 2), (np.uint8, 1, 4), (np.float32, 1024, 2)]


@pytest.mark.parametrize("dtype,disp,P", CASES)
def test_random_worlds_vs_oracle(coracle, dtype, disp, P):
    torch = _torch()
    rng = np.random.default_rng(4242 + disp * 7 + P)
    nrows, shards = random_world(rng, P, dtype, disp, max_rows=400)
    ll = O.np_lenlist(nrows)
    row = disp * np.dtype(dtype).itemsize
    starts, counts = random_valid_requests(rng, ll, 777, max_count=64)
    exp, exp_offs, bad, rc = coracle.get_batch(shards, starts, counts)
    assert bad == -1
    fixed_starts = starts[counts >= 3][:300]
    exp_fixed3 = None
    ok3 = [s for s in fixed_starts.tolist() if coracle.locate(ll, s, 3)[2] == 0]
    if ok3:
        exp_fixed3, _, bad, _ = coracle.get_batch(shards, ok3, [3] * len(ok3))
        assert bad == -1

    def body(store, r):
        store.add("v", shards[r])
        # (a) variable counts, host indices -> host buffer, with offsets
        out = np.zeros(max(exp.size, 1), np.uint8)
        offs = np.zeros(len(starts) + 1, np.int64)
        n = store.get_batch("v", starts, counts, out=out, offsets=offs)
        assert n == exp.size and out[:n].tobytes() == exp.tobytes() and offs.tolist() == exp_offs.tolist()
        # (b) device indices -> device buffer (bytes never leave HBM), device offsets
        dev = torch.device("cuda", 0)
        d_out = torch.zeros(max(exp.size, 16) + 64, dtype=torch.uint8, device=dev)
        d_offs = torch.zeros(len(starts) + 1, dtype=torch.int64, device=dev)
        n = store.get_batch("v", torch.from_numpy(starts).to(dev), torch.from_numpy(counts).to(dev), out=d_out,
                            offsets=d_offs)
        assert n == exp.size and d_out[:n].cpu().numpy().tobytes() == exp.tobytes()
        assert d_offs.cpu().numpy().tolist() == exp_offs.tolist()
        assert int(d_out[n:].sum()) == 0  # nothing written past the packed end
        # (c) fixed count (the single-launch path), host and device destinations
        if ok3:
            out3 = np.zeros(exp_fixed3.size, np.uint8)
            n3 = store.get_batch("v", ok3, out=out3, count=3)
            assert n3 == exp_fixed3.size and out3.tobytes() == exp_fixed3.tobytes()
            d3 = torch.zeros(exp_fixed3.size, dtype=torch.uint8, device=dev)
            store.get_batch("v", ok3, out=d3, count=3)
            assert d3.cpu().numpy().tobytes() == exp_fixed3.tobytes()
        # (d) per-request get() == the reference's per-sample loop
        for s, c in list(zip(starts.tolist(), counts.tolist()))[:40]:
            buf = np.zeros((c, disp), dtype)
            store.get("v", buf, s)
            e, _, _, _ = coracle.get_batch(shards, [s], [c])
            assert buf.tobytes() == e.tobytes()
        return True

    assert all(run_world(P, body))


def test_every_alignment_phase(coracle):
    """uint8 rows of odd width: source and destination 16-byte phases sweep all 16 x 16 combinations, and
    request sizes straddle the head/body/tail cases of the drain (1..70 bytes and a few multi-chunk ones)."""
    rng = np.random.default_rng(99)
    disp = 1
    shard = rng.integers(0, 256, size=(300000, disp), dtype=np.uint8)
    starts, counts = [], []
    for src_phase in range(16):
        for n in list(range(1, 40)) + [63, 64, 65, 70, 4095, 4096, 4097, 9000]:
            starts.append(1024 + src_phase + 16 * int(rng.integers(0, 1000)))
            counts.append(n)
    perm = rng.permutation(len(starts))
    starts, counts = np.array(starts, np.int64)[perm], np.array(counts, np.int64)[perm]
    exp, exp_offs, bad, _ = coracle.get_batch([shard], starts, counts)
    assert bad == -1

    def body(store, r):
        store.add("b", shard)
        out = np.zeros(exp.size, np.uint8)
        n = store.get_batch("b", starts, counts, out=out)
        assert n == exp.size
        if out.tobytes() != exp.tobytes():
            badpos = int(np.nonzero(out != exp)[0][0])
            req = int(np.searchsorted(exp_offs, badpos, side="right") - 1)
            raise AssertionError(f"first mismatch at byte {badpos} (request {req}: start={starts[req]} count={counts[req]} "
                                 f"dst_off={exp_offs[req]})")
        return True

    assert all(run_world(1, body))


def test_variable_length_cfg3_shape(coracle):
    """config 3 at reduced size: disp=1 float32 samples of 100..10000 elements, 4 ranks."""
    rng = np.random.default_rng(42)
    P, nsamp = 4, 2000
    L = rng.integers(100, 10001, size=nsamp)
    sample_start = np.concatenate([[0], np.cumsum(L)])
    per = nsamp // P
    shards = []
    for r in range(P):
        n = int(sample_start[(r + 1) * per] - sample_start[r * per])
        shards.append(rng.integers(0, 2**32, size=(n, 1), dtype=np.uint32).view(np.float32))
    pick = rng.integers(0, nsamp, size=1500)
    starts, counts = sample_start[pick], L[pick]
    exp, exp_offs, bad, _ = coracle.get_batch(shards, starts, counts)
    assert bad == -1

    def body(store, r):
        store.add("x", shards[r])
        out = np.zeros(exp.size, np.uint8)
        assert store.get_batch("x", starts, counts, out=out) == exp.size
        assert out.tobytes() == exp.tobytes()
        return True

    assert all(run_world(P, body))


def test_multi_array_cfg4_shape(coracle):
    """config 4 at reduced size: node_feat float32 [n_i,16] + edge_index int64 [8 n_i, 2], 2 ranks."""
    rng = np.random.default_rng(4)
    P, nsamp = 2, 600
    n = rng.integers(8, 513, size=nsamp)
    e = 8 * n
    ns, es = np.concatenate([[0], np.cumsum(n)]), np.concatenate([[0], np.cumsum(e)])
    per = nsamp // P
    feat = [rng.integers(0, 2**32, size=(int(ns[(r + 1) * per] - ns[r * per]), 16), dtype=np.uint32).view(np.float32)
            for r in range(P)]
    edge = [rng.integers(-2**40, 2**40, size=(int(es[(r + 1) * per] - es[r * per]), 2), dtype=np.int64) for r in range(P)]
    pick = rng.integers(0, nsamp, size=500)
    ef, _, b1, _ = coracle.get_batch(feat, ns[pick], n[pick])
    ee, _, b2, _ = coracle.get_batch(edge, es[pick], e[pick])
    assert b1 == b2 == -1

    def body(store, r):
        store.add("node_feat", feat[r])
        store.add("edge_index", edge[r])
        of, oe = np.zeros(ef.size, np.uint8), np.zeros(ee.size, np.uint8)
        store.get_batch("node_feat", ns[pick], n[pick], out=of)
        store.get_batch("edge_index", es[pick], e[pick], out=oe)
        assert of.tobytes() == ef.tobytes() and oe.tobytes() == ee.tobytes()
        return True

    assert all(run_world(P, body))


def test_large_requests_multi_chunk_and_segments(coracle):
    """a few multi-megabyte requests (config 5 shape) so one request spans many chunks and segments"""
    rng = np.random.default_rng(11)
    disp = 256 * 1024  # 1 MiB rows of float32
    shards = [rng.integers(0, 2**32, size=(6, disp), dtype=np.uint32).view(np.float32) for _ in range(2)]
    starts = np.array([7, 0, 11, 3, 6, 5], np.int64)
    counts = np.array([1, 3, 1, 2, 4, 1], np.int64)
    exp, _, bad, _ = coracle.get_batch(shards, starts, counts)
    assert bad == -1

    def body(store, r):
        store.add("big", shards[r])
        out = np.zeros(exp.size, np.uint8)
        assert store.get_batch("big", starts, counts, out=out) == exp.size
        assert out.tobytes() == exp.tobytes()
        return True

    assert all(run_world(2, body))


# ------------------------------------------------------------------------------- init / update / fences / errors
def test_init_update_and_fence_state_machine():
    def body(store, r):
        nrows = [4, 0, 6][r]
        store.init("z", nrows, 3, 4)  # include/ddstore.hpp:110-179
        if r == 0:
            store.update("z", np.arange(6, dtype=np.float32).reshape(2, 3), 1)  # :181-195
            with pytest.raises(ValueError, match="Invalid data type"):
                store.update("z", np.zeros((1, 3), np.float64), 0)
        store.epoch_begin()
        with pytest.raises(RuntimeError, match="Fence already activated"):  # src/ddstore.cxx:57-58
            store.epoch_begin()
        got = np.full((4, 3), -1, np.float32)
        store.get("z", got, 0)
        store.epoch_end()
        with pytest.raises(RuntimeError, match="Fence is not activated"):  # src/ddstore.cxx:71-72
            store.epoch_end()
        exp = np.zeros((4, 3), np.float32)
        exp[1:3] = np.arange(6, dtype=np.float32).reshape(2, 3)
        assert got.tobytes() == exp.tobytes()
        with pytest.raises(ValueError, match="Invalid data type"):  # include/ddstore.hpp:202-203
            store.get("z", np.zeros((1, 3), np.float64), 0)
        with pytest.raises(KeyError):
            store.get("nope", np.zeros((1, 3), np.float32), 0)
        with pytest.raises(NotImplementedError):  # src/pyddstore.pyx:100-101
            store.get("z", np.zeros((1, 3), np.float16), 0)
        return True

    assert all(run_world(3, body))


def test_invalid_disp_on_the_differing_rank():
    def body(store, r):
        arr = np.zeros((2, 4 if r != 1 else 3), np.float32)
        if r == 1:
            with pytest.raises(ValueError, match="Invalid disp"):  # include/ddstore.hpp:81-82
                store.add("bad", arr)
        else:
            store.add("bad", arr)
        return True

    assert all(run_world(3, body))


def test_capacity_is_enforced_without_overrun():
    torch = _torch()

    def body(store, r):
        store.add("v", np.arange(64 * 8, dtype=np.float32).reshape(64, 8))
        d = torch.full((100,), 7, dtype=torch.uint8, device="cuda:0")
        with pytest.raises(ValueError, match="too small"):
            store.get_batch("v", [0, 1, 2, 3], out=d[:96], count=1)  # needs 128 bytes
        assert int((d != 7).sum()) == 0
        return True

    assert all(run_world(1, body))


# ------------------------------------------------------------------------------- synthetic payload + full size
def test_synth_fill_matches_oracle_generator(coracle):
    def body(store, r):
        for name, dt, disp, seed in (("f", np.float32, 33, 0xDD5), ("i", np.int64, 2, 0xDD6), ("b", np.uint8, 5, 0xDD7)):
            nrows = 1000 + 13 * r
            store.init(name, nrows, disp, np.dtype(dt).itemsize)
            store.synth_fill(name, seed)
            ll = store.query(name)["lenlist"]
            first = ll[r - 1] if r else 0
            got = np.zeros((nrows, disp), dt)
            store.get(name, got, first)
            assert got.tobytes() == coracle.synth_rows(seed, first, nrows, disp, dt).tobytes()
        return True

    assert all(run_world(2, body))


def test_full_size_config2_spot_check(coracle):
    """BASELINE config 2 at FULL size on one GPU: 10M x 1024 float32 (40.96 GB), uniform-random batch of
    65536 rows. Expected bytes are recomputed from the generator for the sampled rows (size-independent
    property: every fetched row equals synth(row index))."""
    torch = _torch()
    free, total = torch.cuda.mem_get_info(0)
    nrows, disp = 10_000_000, 1024
    if free < nrows * disp * 4 + (2 << 30):
        pytest.skip("not enough free HBM for the full-size shard")
    B = 65536

    def body(store, r):
        store.init("x", nrows, disp, 4)
        store.synth_fill("x", 0xDD5)
        rng = np.random.default_rng(1234)
        idx = rng.integers(0, nrows, size=B)
        d_out = torch.empty(B * disp, dtype=torch.float32, device="cuda:0")
        n = store.get_batch("x", idx, out=d_out, count=1)
        assert n == B * disp * 4
        got = d_out.cpu().numpy().reshape(B, disp)
        sample = rng.choice(B, size=2048, replace=False)
        for j in sample.tolist() + [0, B - 1]:
            exp = O.np_synth_rows(0xDD5, int(idx[j]), 1, disp, np.float32)
            assert got[j].tobytes() == exp.tobytes(), f"row {j} (sample {idx[j]})"
        # checksum-of-checksums over the whole batch against a vectorised recomputation
        blk = 8192
        for b0 in range(0, B, blk):
            g = (idx[b0:b0 + blk].astype(np.uint64)[:, None] * np.uint64(disp) + np.arange(disp, dtype=np.uint64)[None, :])
            x = (g ^ np.uint64(0xDD5)) + np.uint64(0x9E3779B97F4A7C15)
            x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            x = (x ^ (x >> np.uint64(31))).astype(np.uint32)
            assert np.array_equal(x, got[b0:b0 + blk].view(np.uint32))
        return True

    assert all(run_world(1, body, timeout=900))


def test_sample_index_lookup_fused_in_the_launch(coracle):
    """SURVEY.md 8f rank 2: get_samples(ids) == get_batch(starts[ids], counts[ids]), small (1-CTA plan) and large
    (2-kernel plan) batches, host and device ids, plus out-of-range ids."""
    torch = _torch()
    rng = np.random.default_rng(21)
    P, nsamp = 3, 9000
    L = rng.integers(0, 40, size=nsamp)  # some empty samples
    sstart = np.concatenate([[0], np.cumsum(L)])
    per = nsamp // P
    shards = []
    for r in range(P):
        n = int(sstart[(r + 1) * per] - sstart[r * per])
        shards.append(rng.integers(0, 256, size=(n, 5), dtype=np.uint8))

    def body(store, r):
        store.add("x", shards[r])
        store.set_sample_index("x", sstart[:-1], L)
        for B in (300, 20000):
            ids = rng.integers(0, nsamp, size=B)
            exp, exp_offs, bad, _ = coracle.get_batch(shards, sstart[ids], L[ids])
            assert bad == -1
            out = np.zeros(max(exp.size, 1), np.uint8)
            offs = np.zeros(B + 1, np.int64)
            assert store.get_samples("x", ids, out, offsets=offs) == exp.size
            assert out[:exp.size].tobytes() == exp.tobytes() and offs.tolist() == exp_offs.tolist()
            d_out = torch.zeros(max(exp.size, 16), dtype=torch.uint8, device="cuda:0")
            assert store.get_samples("x", torch.from_numpy(ids).cuda(), d_out) == exp.size
            assert d_out[:exp.size].cpu().numpy().tobytes() == exp.tobytes()
        ids = np.array([5, 6, nsamp, 7])
        with pytest.raises(ValueError, match="sample id"):
            store.get_samples("x", ids, np.zeros(4096, np.uint8))
        assert store.last_bad_index == 2
        with pytest.raises(ValueError, match="sample id"):
            store.get_samples("x", [-1], np.zeros(16, np.uint8))
        return True

    assert all(run_world(P, body))


PLAN_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
import numpy as np
from ddstore_b200 import PyDDStore
from oracle.oracle import COracle
from tests.helpers import random_valid_requests
rng = np.random.default_rng(77)
shard = rng.integers(0, 256, size=(60000, 3), dtype=np.uint8)
store = PyDDStore(device=0)
store.add("b", shard)
for B in (300, 4096, 5000, 8192, 9000, 70000):
    starts, counts = random_valid_requests(rng, [60000], B, max_count=30)
    exp, exp_offs, bad, _ = COracle().get_batch([shard], starts, counts)
    out = np.zeros(max(exp.size, 1), np.uint8)
    offs = np.zeros(B + 1, np.int64)
    assert store.get_batch("b", starts, counts, out=out, offsets=offs) == exp.size
    assert out[:exp.size].tobytes() == exp.tobytes() and offs.tolist() == exp_offs.tolist(), B
    starts[B // 2], counts[B // 2] = 60000, 1  # first bad request in the middle
    try:
        store.get_batch("b", starts, counts, out=out)
        raise SystemExit("no error raised")
    except ValueError as e:
        assert str(e) == "Invalid count on target" and store.last_bad_index == B // 2
store.free(); store.close()
print("plan-ok")
"""


@pytest.mark.parametrize("mode", ["0", "1"])
def test_plan_variants_agree(tmp_path, mode):
    """DDS_SMEM_PLAN=0 (plan kernels + segment table at every size) and =1 (every CTA plans <= 8192 requests in its
    own shared memory) against the oracle"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "plan_variant.py"
    script.write_text(PLAN_SCRIPT.format(root=root))
    # (mode 1 also raises the shared-memory plan's limit to its maximum, so both of its kernel variants -- 4096 and 8192
    # requests -- are exercised; by default only batches of <= 1024 requests plan in shared memory)
    r = subprocess.run([sys.executable, str(script)], env=dict(os.environ, DDS_SMEM_PLAN=mode, DDS_SMEM_PLAN_MAX="8192"), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "plan-ok" in r.stdout, r.stdout + r.stderr


def test_edge_cases_of_the_batch_entry(coracle):
    """empty batches, zero counts, a million tiny requests (scratch growth), sticky-status re-arm after an error,
    queued async batches reporting through wait()"""
    torch = _torch()
    rng = np.random.default_rng(31)
    shards = [rng.integers(0, 256, size=(n, 6), dtype=np.uint8) for n in (500, 0, 700)]
    ll = O.np_lenlist([500, 0, 700])

    def body(store, r):
        store.add("v", shards[r])
        dev = torch.device("cuda", 0)
        # nreq == 0
        out = np.zeros(16, np.uint8)
        offs = np.full(1, -1, np.int64)
        assert store.get_batch("v", np.zeros(0, np.int64), np.zeros(0, np.int64), out=out, offsets=offs) == 0
        assert offs[0] == 0
        # every count zero (nothing to copy, but the range checks still run: start 1200 is out of range)
        assert store.get_batch("v", [0, 499, 500, 1199], [0, 0, 0, 0], out=out) == 0
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get_batch("v", [0, 1200], out=out, count=0)
        assert store.last_bad_index == 1
        # ... and the sticky status word is re-armed: the next valid call succeeds
        exp, _, _, _ = coracle.get_batch(shards, [3, 600], [2, 2])
        o2 = np.zeros(exp.size, np.uint8)
        assert store.get_batch("v", [3, 600], out=o2, count=2) == exp.size and o2.tobytes() == exp.tobytes()
        # fixed count > 1 with device offsets
        st = np.array([0, 10, 498, 500, 1190], np.int64)
        exp, exp_offs, bad, _ = coracle.get_batch(shards, st, [2] * 5)
        d_out = torch.zeros(exp.size, dtype=torch.uint8, device=dev)
        d_offs = torch.zeros(6, dtype=torch.int64, device=dev)
        store.get_batch("v", torch.from_numpy(st).to(dev), out=d_out, count=2, offsets=d_offs)
        assert d_out.cpu().numpy().tobytes() == exp.tobytes() and d_offs.cpu().tolist() == exp_offs.tolist()
        # a million one-row requests (plan scratch grows, > 8192 -> separate plan kernels)
        B = 1_000_000
        starts, counts = random_valid_requests(rng, ll, B, max_count=1)
        exp, exp_offs, bad, _ = coracle.get_batch(shards, starts, counts)
        big = np.zeros(exp.size, np.uint8)
        assert store.get_batch("v", starts, counts, out=big) == exp.size and big.tobytes() == exp.tobytes()
        # queued async batches: the first error of the queue surfaces in wait(), then the store is usable again
        ds, dc = torch.from_numpy(starts[:4096]).to(dev), torch.from_numpy(counts[:4096]).to(dev)
        bad_s = ds.clone()
        bad_s[77] = -5
        dbuf = torch.zeros(4096 * 6, dtype=torch.uint8, device=dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        store.get_batch("v", ds, dc, out=dbuf, stream=side.cuda_stream, wait=False)
        store.get_batch("v", bad_s, dc, out=dbuf, stream=side.cuda_stream, wait=False)
        store.get_batch("v", ds, dc, out=dbuf, stream=side.cuda_stream, wait=False)
        with pytest.raises(ValueError, match="Invalid start on target"):
            store.wait()
        assert store.last_bad_index == 77
        store.get_batch("v", ds, dc, out=dbuf, stream=side.cuda_stream, wait=False)
        n = store.wait()
        e4, _, _, _ = coracle.get_batch(shards, starts[:4096], counts[:4096])
        assert n == e4.size and dbuf[:n].cpu().numpy().tobytes() == e4.tobytes()
        return True

    assert all(run_world(3, body))


def test_overlapped_queue_of_independent_batches(coracle):
    """DDS_OVERLAP: a double-buffered queue of fixed-count batches whose launches overlap (no grid wait, static
    segment striding), mixed with ordinary ticketed launches; every buffer must hold exactly its last batch."""
    torch = _torch()
    rng = np.random.default_rng(91)
    shard = rng.integers(0, 2**32, size=(200_000, 256), dtype=np.uint32).view(np.float32)  # 1 KiB rows, 205 MB

    def body(store, r):
        store.add("x", shard)
        dev = torch.device("cuda", 0)
        B = 40_000
        side = torch.cuda.Stream(device=dev)
        bufs = [torch.zeros((B, 256), dtype=torch.float32, device=dev) for _ in range(2)]
        batches = [rng.integers(0, 200_000, size=B) for _ in range(9)]
        d_idx = [torch.from_numpy(b).to(dev) for b in batches]
        torch.cuda.synchronize()
        for k, ids in enumerate(d_idx):
            # batches 0-3 overlapped, 4 ordinary (ticketed, waits), 5-8 overlapped again
            store.get_batch("x", ids, out=bufs[k & 1], count=1, stream=side.cuda_stream, wait=False, overlap=(k != 4))
        store.wait()
        for slot, k in ((0, 8), (1, 7)):
            assert bufs[slot].cpu().numpy().tobytes() == shard[batches[k]].tobytes(), f"buffer {slot} != batch {k}"
        # an invalid request inside an overlapped queue is still reported, with its index
        bad = d_idx[0].clone()
        bad[123] = 200_000
        store.get_batch("x", d_idx[1], out=bufs[0], count=1, stream=side.cuda_stream, wait=False, overlap=True)
        store.get_batch("x", bad, out=bufs[1], count=1, stream=side.cuda_stream, wait=False, overlap=True)
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.wait()
        assert store.last_bad_index == 123
        return True

    assert all(run_world(1, body))


def test_multi_array_batch_in_one_launch(coracle):
    """dds_get_samples_multi: node_feat + edge_index (+ a third, byte-wide variable) of the same samples in one launch,
    fused plan (small batch) and separate plan kernels (large batch), against per-variable oracle results."""
    torch = _torch()
    rng = np.random.default_rng(17)
    P, per = 2, 400
    world = []
    for r in range(P):
        n = rng.integers(0, 60, size=per)  # some empty samples
        feat = rng.integers(0, 2**32, size=(int(n.sum()), 16), dtype=np.uint32).view(np.float32)
        edge = rng.integers(-2**40, 2**40, size=(int(8 * n.sum()), 2), dtype=np.int64)
        tags = rng.integers(0, 256, size=(int(3 * n.sum()), 5), dtype=np.uint8)
        world.append((n, feat, edge, tags))
    n_all = np.concatenate([w[0] for w in world])
    tabs = {"node_feat": (n_all, 1), "edge_index": (n_all, 8), "tags": (n_all, 3)}
    shards = {"node_feat": [w[1] for w in world], "edge_index": [w[2] for w in world], "tags": [w[3] for w in world]}

    def body(store, r):
        names = ["node_feat", "edge_index", "tags"]
        for nm in names:
            store.add(nm, shards[nm][r])
            cnt = tabs[nm][0] * tabs[nm][1]
            store.set_sample_index(nm, np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
        for B in (37, 5000):
            ids = rng.integers(0, P * per, size=B)
            exp = {}
            for nm in names:
                cnt = tabs[nm][0] * tabs[nm][1]
                st = np.concatenate([[0], np.cumsum(cnt)[:-1]])
                exp[nm] = coracle.get_batch(shards[nm], st[ids], cnt[ids])
            outs = [torch.zeros(max(exp[nm][0].size, 16) + 32, dtype=torch.uint8, device="cuda:0") for nm in names]
            offs = [torch.zeros(B + 1, dtype=torch.int64, device="cuda:0") for _ in names]
            totals = store.get_samples_multi(names, ids, outs, offsets=offs)
            for nm, o, f, t in zip(names, outs, offs, totals):
                e, eo, bad, _ = exp[nm]
                assert bad == -1 and t == e.size, (nm, t, e.size)
                assert o[:t].cpu().numpy().tobytes() == e.tobytes(), nm
                assert int(o[t:].sum()) == 0 and f.cpu().tolist() == eo.tolist()
        # an out-of-range sample id is reported with its position in the id list
        ids = np.array([1, 2, P * per + 3, 4])
        with pytest.raises(ValueError, match="sample id"):
            store.get_samples_multi(names, ids, outs)
        assert store.last_bad_index == 2
        # capacity of ONE variable too small
        ids = rng.integers(0, P * per, size=64)
        small = [outs[0], outs[1][:8], outs[2]]
        with pytest.raises(ValueError, match="too small"):
            store.get_samples_multi(names, ids, small)
        return True

    assert all(run_world(P, body))


def test_overlapped_queue_of_variable_count_batches(coracle):
    """DDS_OVERLAP on variable-count batches: every launch plans in its own scratch slot (ring of 4, monotonic counters,
    slot-reuse guard); explicit and by-sample requests, small and large batches, 11 launches deep."""
    torch = _torch()
    rng = np.random.default_rng(55)
    nsamp = 30_000
    L = rng.integers(0, 200, size=nsamp)
    sstart = np.concatenate([[0], np.cumsum(L)])
    shard = rng.integers(0, 2**32, size=(int(sstart[-1]), 3), dtype=np.uint32).view(np.float32)  # 12 B rows: re-phase path

    def body(store, r):
        store.add("x", shard)
        store.set_sample_index("x", sstart[:-1], L)
        dev = torch.device("cuda", 0)
        side = torch.cuda.Stream(device=dev)
        sizes = [300, 9000, 5000, 20000, 700, 9000, 9000, 300, 20000, 5000, 1234]
        batches = [rng.integers(0, nsamp, size=B) for B in sizes]
        exps = [coracle.get_batch([shard], sstart[b], L[b]) for b in batches]
        cap = max(e[0].size for e in exps) + 64
        bufs = [torch.zeros(cap, dtype=torch.uint8, device=dev) for _ in range(2)]
        offs = [torch.zeros(max(sizes) + 1, dtype=torch.int64, device=dev) for _ in range(2)]
        d_ids = [torch.from_numpy(b).to(dev) for b in batches]
        d_st = [torch.from_numpy(sstart[b]).to(dev) for b in batches]
        d_ct = [torch.from_numpy(L[b]).to(dev) for b in batches]
        torch.cuda.synchronize()
        for k in range(len(batches)):
            o, f = bufs[k & 1], offs[k & 1][:sizes[k] + 1]
            if k % 3 == 0:
                store.get_samples("x", d_ids[k], o, offsets=f, stream=side.cuda_stream, wait=False, overlap=True)
            elif k == 4:  # an ordinary queued launch in the middle of the run
                store.get_batch("x", d_st[k], d_ct[k], out=o, offsets=f, stream=side.cuda_stream, wait=False)
            else:
                store.get_batch("x", d_st[k], d_ct[k], out=o, offsets=f, stream=side.cuda_stream, wait=False, overlap=True)
        total = store.wait()
        assert total == exps[-1][0].size
        for slot, k in ((0, 10), (1, 9)):
            e, eo, bad, _ = exps[k]
            assert bad == -1 and bufs[slot][:e.size].cpu().numpy().tobytes() == e.tobytes(), f"buffer {slot} != batch {k}"
            assert offs[slot][:sizes[k] + 1].cpu().tolist() == eo.tolist()
        return True

    assert all(run_world(1, body))


OVERLAP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
import ctypes
import numpy as np, torch
from ddstore_b200 import PyDDStore, _capi
rng = np.random.default_rng(77)
shard = rng.integers(0, 2**32, size=(150_000, 256), dtype=np.uint32).view(np.float32)   # 1 KiB rows
L = rng.integers(1, 40, size=20_000)
sstart = np.concatenate([[0], np.cumsum(L)])
vshard = rng.integers(0, 2**32, size=(int(sstart[-1]), 5), dtype=np.uint32).view(np.float32)  # 20 B rows: re-phase path
store = PyDDStore(device=0)
store.add("x", shard)
store.add("v", vshard)
store.set_sample_index("v", sstart[:-1], L)
dev = torch.device("cuda", 0)
side, other = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
B = 30_000
bufs = [torch.zeros((B, 256), dtype=torch.float32, device=dev) for _ in range(2)]
vcap = int(L.max()) * 20 * 4096 + 64
vbufs = [torch.zeros(vcap, dtype=torch.uint8, device=dev) for _ in range(2)]
lib = _capi.lib()
for rnd in range(8):
    nb = 5 + rnd % 3
    batches = [rng.integers(0, 150_000, size=B) for _ in range(nb)]
    d_idx = [torch.from_numpy(b).to(dev) for b in batches]
    vids = [rng.integers(0, 20_000, size=4096) for _ in range(nb)]
    d_vid = [torch.from_numpy(b).to(dev) for b in vids]
    torch.cuda.synchronize()
    # a "training kernel" on another stream takes about half of the SMs away for the whole queue
    _capi.raise_for(lib.dds_test_occupy(0, 70 + rnd, 200 * 1024, 3_000_000, ctypes.c_void_p(other.cuda_stream)))
    for k in range(nb):
        store.get_batch("x", d_idx[k], out=bufs[k & 1], count=1, stream=side.cuda_stream, wait=False, overlap=True)
    store.wait()
    for slot, k in (((nb - 1) & 1, nb - 1), ((nb - 2) & 1, nb - 2)):
        assert bufs[slot].cpu().numpy().tobytes() == shard[batches[k]].tobytes(), ("fixed", rnd, slot, k)
    _capi.raise_for(lib.dds_test_occupy(0, 70 + rnd, 200 * 1024, 2_000_000, ctypes.c_void_p(other.cuda_stream)))
    for k in range(nb):
        store.get_samples("v", d_vid[k], vbufs[k & 1], stream=side.cuda_stream, wait=False, overlap=True)
    store.wait()
    for slot, k in (((nb - 1) & 1, nb - 1), ((nb - 2) & 1, nb - 2)):
        exp = np.concatenate([vshard[sstart[i]:sstart[i] + L[i]].reshape(-1) for i in vids[k]]).view(np.uint8)
        assert vbufs[slot][:exp.size].cpu().numpy().tobytes() == exp.tobytes(), ("var", rnd, slot, k)
    torch.cuda.synchronize()
store.free(); store.close()
print("overlap-ok")
"""


@pytest.mark.parametrize("ctas_per_sm", ["1", "2"])
def test_overlap_contract_holds_when_the_gpu_is_shared(tmp_path, ctas_per_sm):
    """DDS_OVERLAP is a contract the kernel enforces (generation words), not a capacity assumption: a double-buffered
    overlapped queue stays correct while another kernel holds half of the SMs, and with 2 gather CTAs per SM."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "overlap_contract.py"
    script.write_text(OVERLAP_SCRIPT.format(root=root))
    env = dict(os.environ, DDS_GATHER_CTAS_PER_SM=ctas_per_sm)
    if ctas_per_sm == "2":
        env["DDS_GATHER_GEOM"] = "5"  # 4 warps x 6 stages: two CTAs fit on an SM
        env["DDS_GATHER_GEOM_S"] = "4"
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "overlap-ok" in r.stdout, r.stdout + r.stderr


def test_negative_and_zero_fixed_count(coracle):
    """a negative fixed count is the reference's 'Invalid count on target' on request 0 -- unless request 0's start is
    invalid, which is checked first (ddstore.hpp:210-214); count 0 copies nothing and succeeds"""
    torch = _torch()
    shards = [np.arange(40, dtype=np.int64).reshape(10, 4), np.arange(40, 80, dtype=np.int64).reshape(10, 4)]

    def body(store, r):
        store.add("x", shards[r])
        out = np.zeros((8, 4), np.int64)
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get_batch("x", [3, 4, 5], out=out, count=-1)
        assert store.last_bad_index == 0
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get_batch("x", torch.tensor([3, 4, 5]).cuda(), out=torch.zeros(64, dtype=torch.int64).cuda(), count=-2)
        assert store.last_bad_index == 0
        assert store.get_batch("x", [3, 4, 5], out=out, count=0) == 0 and not out.any()
        from ddstore_b200 import _capi
        with pytest.raises(ValueError, match="Invalid count on target"):  # the single-request entry (1-CTA kernel)
            _capi.raise_for(store._L.dds_get(store._h, b"x", 3, -1, 8, out.ctypes.data, 0))
        return True

    assert all(run_world(2, body))


def test_single_request_kernel_alignments_and_errors(coracle):
    """dds_get's 1-CTA kernel: every source/destination alignment class (16 / 4 / 1 byte), host and device
    destinations, remote owners, zero rows, and the reference's two errors"""
    torch = _torch()
    rng = np.random.default_rng(5)
    shards = [rng.integers(0, 256, size=(n, 3), dtype=np.uint8) for n in (301, 0, 407)]
    f32 = [rng.integers(0, 2**32, size=(n, 5), dtype=np.uint32).view(np.float32) for n in (64, 64, 64)]
    allb = np.concatenate(shards)
    allf = np.concatenate(f32)

    def body(store, r):
        store.add("b", shards[r])
        store.add("f", f32[r])
        for start, cnt in ((0, 1), (299, 2), (301, 7), (500, 208), (707, 1), (3, 0)):
            if start + cnt > 708 or (start < 301 < start + cnt):
                continue
            out = np.zeros((cnt, 3), np.uint8)
            store.get("b", out, start)
            assert out.tobytes() == allb[start:start + cnt].tobytes(), (start, cnt)
            dout = torch.zeros((cnt + 1, 3), dtype=torch.uint8, device="cuda")[1:].contiguous() if cnt else torch.zeros((0, 3), dtype=torch.uint8, device="cuda")
            store.get("b", dout, start)
            assert dout.cpu().numpy().tobytes() == allb[start:start + cnt].tobytes()
        for start, cnt in ((0, 4), (63, 1), (64, 64), (130, 31)):
            out = np.zeros((cnt, 5), np.float32)
            store.get("f", out, start)
            assert out.tobytes() == allf[start:start + cnt].tobytes()
            big = torch.zeros(cnt * 5 + 3, dtype=torch.float32, device="cuda")
            view = big[3:].view(cnt, 5)  # 12-byte phase relative to the allocation
            store.get("f", view, start)
            assert view.cpu().numpy().tobytes() == allf[start:start + cnt].tobytes()
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get("b", np.zeros((5, 3), np.uint8), 299)  # straddles ranks 0 -> 2
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get("b", np.zeros((2, 3), np.uint8), 707)
        out = np.zeros((1, 3), np.uint8)
        store.get("b", out, 300)  # the call after an error works (no sticky state)
        assert out.tobytes() == allb[300:301].tobytes()
        return True

    assert all(run_world(3, body))


def test_large_pageable_destination_and_ingest(coracle):
    """host copies that run through the worker-thread pool: a packed batch of tens of MB into a PAGEABLE ndarray (the
    reference's np.zeros contract: copy engine -> pinned staging buffers -> worker threads), and dds_ingest of pageable
    chunks into a pre-init'd shard (bounds and dtype checked like update)"""
    torch = _torch()
    rng = np.random.default_rng(21)
    rows, disp = 120_000, 96  # 384 B rows, 46 MB shard
    src = rng.integers(0, 2**32, size=(rows, disp), dtype=np.uint32).view(np.float32)

    def body(store, r):
        store.init("x", rows, disp, 4)
        store.ingest("x", src[:70_001], 0)          # 26.9 MB: two staging buffers, ragged tail
        store.ingest("x", src[70_001:], 70_001)
        store.ingest_wait()
        with pytest.raises(ValueError):
            store.ingest("x", src[:10], rows - 5)   # outside the shard
        with pytest.raises(ValueError, match="Invalid data type"):
            store.ingest("x", src[:10].view(np.uint8).reshape(10, -1), 0)
        ids = rng.integers(0, rows, size=90_000)    # 34.6 MB packed: the pipelined pageable path (>= 4 MB)
        out = np.zeros((len(ids), disp), np.float32)
        assert store.get_batch("x", ids, out=out, count=1) == out.nbytes
        assert out.tobytes() == src[ids].tobytes()
        pinned = torch.zeros((len(ids), disp), dtype=torch.float32).pin_memory().numpy()
        store.get_batch("x", ids, out=pinned, count=1)
        assert pinned.tobytes() == out.tobytes()
        # an ingest right after a pageable fetch reuses the same staging buffers
        store.ingest("x", src[:5000][::-1].copy(), 0)
        store.ingest_wait()
        chk = np.zeros((5000, disp), np.float32)
        store.get_batch("x", np.arange(5000), out=chk, count=1)
        assert chk.tobytes() == src[:5000][::-1].tobytes()
        return True

    assert all(run_world(1, body))


def test_doorbell_kernel_lifecycle():
    """the resident CTA behind get(): it leaves by itself when idle and a later get() starts a fresh one without losing
    or repeating a request; a device-wide synchronize, an async batch and a free() in between all work. (Without the
    resident kernel -- DDS_DOORBELL=0, or a store's variables past the 256th -- every get() launches
    dds_small_get_kernel: tests/test_gpu_errors.py runs both.)"""
    import time
    torch = _torch()
    rng = np.random.default_rng(9)
    shard = rng.integers(0, 2**32, size=(5000, 33), dtype=np.uint32).view(np.float32)

    def body(store, r):
        store.add("x", shard)
        store.add("b", shard.view(np.uint8).reshape(5000, -1)[:, :7].copy())
        out = np.zeros((1, 33), np.float32)
        dout = torch.zeros((2, 33), dtype=torch.float32, device="cuda")
        for k in range(300):
            i = int(rng.integers(0, 4998))
            if k % 3 == 0:
                store.get("x", dout, i)
                assert dout.cpu().numpy().tobytes() == shard[i:i + 2].tobytes()
            else:
                store.get("x", out, i)
                assert out.tobytes() == shard[i:i + 1].tobytes()
            if k % 50 == 10:
                time.sleep(0.003)            # longer than the idle timeout: the kernel has left, the next get restarts it
            if k % 50 == 20:
                torch.cuda.synchronize()     # must not hang on the resident kernel
            if k % 50 == 30:                 # an async batch in between (the store parks the doorbell when it must sync)
                ids = torch.from_numpy(rng.integers(0, 5000, size=64)).cuda()
                big = torch.zeros((64, 33), dtype=torch.float32, device="cuda")
                store.get_batch("x", ids, out=big, count=1, wait=False)
                assert store.wait() == big.numel() * 4 and big.cpu().numpy().tobytes() == shard[ids.cpu().numpy()].tobytes()
            if k % 50 == 40:
                with pytest.raises(ValueError, match="Invalid count on target"):
                    store.get("x", np.zeros((3, 33), np.float32), 4998)
        b = np.zeros((4, 7), np.uint8)
        store.get("b", b, 100)               # another variable, byte-granular rows
        assert b.tobytes() == shard.view(np.uint8).reshape(5000, -1)[100:104, :7].tobytes()
        return True

    assert all(run_world(1, body))


def test_overlapped_variable_queue_edge_cases(coracle):
    """the memory-chained plan/gather protocol on the awkward batches of an overlapped run: all-zero counts (nothing to
    walk), a single request, a batch that does not fit its buffer (capacity error, nothing written), a bad sample id,
    more requests than the scratch slots hold (they grow mid-run) -- each followed by ordinary batches that must be
    delivered intact, with the error reported by wait() as the first of the queue"""
    torch = _torch()
    rng = np.random.default_rng(2718)
    nsamp = 20_000
    L = rng.integers(0, 60, size=nsamp)
    sstart = np.concatenate([[0], np.cumsum(L)])
    shard = rng.integers(0, 2**32, size=(int(sstart[-1]), 5), dtype=np.uint32).view(np.float32)  # 20 B rows

    def body(store, r):
        store.add("x", shard)
        store.set_sample_index("x", sstart[:-1], L)
        dev = torch.device("cuda", 0)
        side = torch.cuda.Stream(device=dev)
        st = side.cuda_stream
        good = [rng.integers(0, nsamp, size=n) for n in (9000, 12000, 9500, 30000, 9000, 9100)]
        exps = [coracle.get_batch([shard], sstart[g], L[g]) for g in good]
        cap = max(e[0].size for e in exps) + 64
        bufs = [torch.zeros(cap, dtype=torch.uint8, device=dev) for _ in range(2)]
        offs = [torch.zeros(30001, dtype=torch.int64, device=dev) for _ in range(2)]
        d_good = [torch.from_numpy(g).to(dev) for g in good]
        torch.cuda.synchronize()

        def check(slot, k):
            e, eo, bad, _ = exps[k]
            assert bad == -1 and bufs[slot][:e.size].cpu().numpy().tobytes() == e.tobytes(), (slot, k)
            assert offs[slot][:len(good[k]) + 1].cpu().tolist() == eo.tolist()

        def q(ids, slot, n=None):
            n = len(ids) if n is None else n
            store.get_samples("x", ids, bufs[slot], offsets=offs[slot][:n + 1], stream=st, wait=False, overlap=True)

        # 1. zero-length batch (explicit counts all 0) and a single request inside a run
        zeros = torch.zeros(9000, dtype=torch.int64, device=dev)
        q(d_good[0], 0)
        store.get_batch("x", d_good[0].clamp(max=100), zeros, out=bufs[1], offsets=offs[1][:9001], stream=st, wait=False, overlap=True)
        q(d_good[1], 0)
        one = torch.tensor([int(good[2][0])], device=dev)
        q(one, 1)
        q(d_good[2], 0)
        assert store.wait() == exps[2][0].size
        check(0, 2)
        e1 = coracle.get_batch([shard], sstart[good[2][:1]], L[good[2][:1]])[0]
        assert bufs[1][:e1.size].cpu().numpy().tobytes() == e1.tobytes() and offs[1][:2].cpu().tolist() == [0, e1.size]
        # 2. the scratch slots grow in the middle of a run (30000 requests after 9000-12000), results stay right
        q(d_good[0], 0); q(d_good[1], 1); q(d_good[3], 0); q(d_good[4], 1); q(d_good[5], 0)
        assert store.wait() == exps[5][0].size
        check(0, 5); check(1, 4)
        # 3. a batch that does not fit (capacity) in the middle: reported, its buffer untouched, neighbours intact
        small = torch.full((4096,), 7, dtype=torch.uint8, device=dev)
        q(d_good[0], 0)
        store.get_samples("x", d_good[1], small, stream=st, wait=False, overlap=True)
        q(d_good[2], 1)
        with pytest.raises(ValueError, match="too small"):
            store.wait()
        assert int(small.min()) == 7 and int(small.max()) == 7
        check(0, 0); check(1, 2)
        # 4. a bad sample id in the middle: first error of the queue, with its index; the run after it works
        bad = d_good[4].clone()
        bad[4321] = nsamp + 5
        q(d_good[0], 0); q(bad, 1); q(d_good[2], 0)
        with pytest.raises(ValueError, match="sample id"):
            store.wait()
        assert store.last_bad_index == 4321
        check(0, 2)
        q(d_good[4], 1); q(d_good[5], 0)
        assert store.wait() == exps[5][0].size
        check(1, 4); check(0, 5)
        return True

    assert all(run_world(1, body))
