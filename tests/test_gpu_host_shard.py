"""Variables placed in pinned host memory (placement="host", DDS_PLACE_HOST) on an H100 (-m gpu).

Every read entry must deliver, byte for byte, what the same rows of an HBM variable deliver -- the same synthetic payload
(synth_fill) goes into one variable of each placement -- errors included. Every batched write and the push fetch refuse a
HOST variable without launching anything; update / ingest write it; a rewritten row is never served stale; two rank
processes read each other's host shards; the shard takes no HBM, and free() leaves no descriptor behind."""
import ctypes as C
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest

from oracle.oracle import np_synth_rows

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from ddstore_b200 import PyDDStore, _capi  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
SEED = 0x5EED


def launches():
    return _capi.lib().dds_kernel_launches()


@pytest.fixture
def store():
    s = PyDDStore(device=0)
    yield s
    s.free()
    s.close()


def make_pair(store, nrows, disp, itemsize, name="v", seed=SEED):
    """the same synthetic rows in an HBM variable and a HOST variable: returns (hbm name, host name)"""
    for nm, pl in ((name + "_hbm", "hbm"), (name + "_host", "host")):
        store.init(nm, nrows, disp, itemsize, placement=pl)
        store.synth_fill(nm, seed)
    assert store.query(name + "_hbm")["placement"] == "hbm" and store.query(name + "_host")["placement"] == "host"
    return name + "_hbm", name + "_host"


def both(pair, fn):
    """fn(name) for each variable of the pair; asserts identical bytes, returns the HBM result"""
    a, b = fn(pair[0]), fn(pair[1])
    ab = a.cpu().numpy().tobytes() if hasattr(a, "cpu") else np.asarray(a).tobytes()
    bb = b.cpu().numpy().tobytes() if hasattr(b, "cpu") else np.asarray(b).tobytes()
    assert ab == bb
    return a


DTYPES = {1: (np.uint8, torch.uint8), 4: (np.float32, torch.float32)}
# (itemsize, disp, nrows): 1 B, 12 B (unaligned), 4 KiB, 64 KiB and 1 MiB rows
ROWS = [(1, 1, 1 << 16), (4, 3, 20000), (4, 1024, 8192), (4, 16384, 512), (4, 262144, 48)]


@pytest.mark.parametrize("itemsize,disp,nrows", ROWS)
def test_batches_match_hbm(store, itemsize, disp, nrows):
    pair = make_pair(store, nrows, disp, itemsize)
    row = disp * itemsize
    rng = np.random.default_rng(row)
    B = max(8, min(4096, (64 << 20) // row // 4))
    npdt, tdt = DTYPES[itemsize]
    # fixed count, host indices -> device
    starts = rng.integers(0, nrows - 2, size=B)
    exp = both(pair, lambda n: (lambda o: (store.get_batch(n, starts, out=o, count=2), o)[1])(
        torch.zeros(B * 2 * row, dtype=torch.uint8, device=DEV)))
    first = np_synth_rows(SEED, int(starts[0]), 2, disp, npdt).tobytes()
    assert exp[:2 * row].cpu().numpy().tobytes() == first
    # variable counts with zero-count requests, device indices, device out + offsets
    counts = rng.integers(0, 4, size=B)
    counts[::7] = 0
    sv = rng.integers(0, nrows - 4, size=B)
    ds, dc = torch.from_numpy(sv).to(DEV), torch.from_numpy(counts).to(DEV)
    tot = int(counts.sum()) * row

    def var(n):
        o = torch.zeros(tot + 64, dtype=torch.uint8, device=DEV)
        off = torch.zeros(B + 1, dtype=torch.int64, device=DEV)
        assert store.get_batch(n, ds, dc, out=o, offsets=off) == tot
        return torch.cat([o, off.view(torch.uint8)])
    both(pair, var)
    # host destinations: pageable and pinned
    for pin in (False, True):
        def host(n):
            o = torch.zeros(tot, dtype=torch.uint8, pin_memory=pin)
            assert store.get_batch(n, sv, counts, out=o) == tot
            return o
        both(pair, host)
    # sample ids
    ns = 1000
    rs = rng.integers(0, nrows - 8, size=ns)
    rc = rng.integers(0, 8, size=ns)
    for n in pair:
        store.set_sample_index(n, rs, rc)
    ids = rng.integers(0, ns, size=B)
    tot_s = int(rc[ids].sum()) * row

    def samples(n):
        o = torch.zeros(tot_s + 16, dtype=torch.uint8, device=DEV)
        assert store.get_samples(n, torch.from_numpy(ids).to(DEV), o) == tot_s
        return o
    both(pair, samples)
    # single-row get() (the doorbell / 1-CTA kernel path), host and device
    if row <= (64 << 10):
        for r in (0, nrows // 3, nrows - 1):
            both(pair, lambda n: (lambda a: (store.get(n, a, r), a)[1])(np.zeros((1, disp), npdt)))
    both(pair, lambda n: (lambda a: (store.get(n, a, 1), a)[1])(torch.zeros((1, disp), dtype=tdt, device=DEV)))


def test_conversions_padding_and_multi_match_hbm(store):
    rng = np.random.default_rng(3)
    nrows = 30000
    f32 = make_pair(store, nrows, 96, 4, "f")
    u8 = make_pair(store, nrows, 48, 1, "u")
    B = 3000
    starts = torch.from_numpy(rng.integers(0, nrows - 6, size=B)).to(DEV)
    counts = torch.from_numpy(rng.integers(0, 6, size=B)).to(DEV)
    tot = int(counts.sum())

    def bf16(n):
        o = torch.zeros(tot * 96, dtype=torch.bfloat16, device=DEV)
        store.get_batch(n, starts, counts, out=o, src_dtype=torch.float32)
        return o.view(torch.uint8)
    both(f32, bf16)
    mean = np.linspace(10, 200, 48).astype(np.float32)
    std = np.linspace(1, 70, 48).astype(np.float32)
    for n in u8:
        store.set_normalization(n, mean, std)

    def norm(n):
        o = torch.zeros(tot * 48, dtype=torch.float32, device=DEV)
        store.get_batch(n, starts, counts, out=o, src_dtype=torch.uint8, normalize=True)
        return o.view(torch.uint8)
    both(u8, norm)

    def padded(n):  # counts up to 5, three rows per slot: truncation and padding
        o = torch.zeros(B * 3 * 96, dtype=torch.float32, device=DEV)
        ln = torch.zeros(B, dtype=torch.int64, device=DEV)
        store.get_batch(n, starts, counts, out=o, pad_rows=3, pad_value=-1.5, lengths=ln)
        return torch.cat([o.view(torch.uint8), ln.view(torch.uint8)])
    both(f32, padded)

    def padded_bf16(n):
        o = torch.zeros(B * 3 * 96, dtype=torch.bfloat16, device=DEV)
        store.get_batch(n, starts, counts, out=o, pad_rows=3, src_dtype=torch.float32)
        return o.view(torch.uint8)
    both(f32, padded_bf16)
    # a two-variable multi launch: the HBM pair against the HOST pair
    ns = 2000
    rs, rc = rng.integers(0, nrows - 4, size=ns), rng.integers(0, 4, size=ns)
    for n in f32 + u8:
        store.set_sample_index(n, rs, rc)
    ids = torch.from_numpy(rng.integers(0, ns, size=B)).to(DEV)
    tr = int(rc[ids.cpu().numpy()].sum())

    def multi(pl):
        names = [f"f_{pl}", f"u_{pl}"]
        outs = [torch.zeros(tr * 96 * 4, dtype=torch.uint8, device=DEV), torch.zeros(tr * 48, dtype=torch.uint8, device=DEV)]
        offs = [torch.zeros(B + 1, dtype=torch.int64, device=DEV) for _ in names]
        assert store.get_samples_multi(names, ids, outs, offsets=offs) == [tr * 384, tr * 48]
        conv = [torch.zeros(tr * 96, dtype=torch.bfloat16, device=DEV), torch.zeros(tr * 48, dtype=torch.float32, device=DEV)]
        store.get_samples_multi(names, ids, conv, src_dtypes=[torch.float32, torch.uint8], normalize=[False, True])
        return torch.cat([o.view(torch.uint8) for o in outs + offs + conv])
    assert torch.equal(multi("hbm"), multi("host"))


def test_async_queue_with_overlap_matches_hbm(store):
    """a queue of wait=False batches with overlap=True (ignored for the HOST variable): every batch of it delivers what a
    synchronous batch from the HBM variable delivers"""
    pair = make_pair(store, 50000, 1024, 4, "q")
    st = torch.cuda.Stream()
    for n in pair:
        rng = np.random.default_rng(5)
        queued = []
        for k in range(6):
            ids = torch.from_numpy(rng.integers(0, 50000, size=2048)).to(DEV)
            cn = torch.from_numpy(rng.integers(0, 3, size=2048)).to(DEV)
            o = torch.zeros(2048 * 2 * 4096, dtype=torch.uint8, device=DEV)
            off = torch.zeros(2049, dtype=torch.int64, device=DEV)
            torch.cuda.synchronize()
            if k % 2:
                store.get_batch(n, ids, out=o, count=2, stream=st.cuda_stream, wait=False, overlap=True)
            else:
                store.get_batch(n, ids, cn, out=o, offsets=off, stream=st.cuda_stream, wait=False, overlap=True)
            queued.append((ids, cn, o, off))
        assert store.wait() == 2048 * 2 * 4096
        for k, (ids, cn, o, off) in enumerate(queued):
            ref, roff = torch.zeros_like(o), torch.zeros_like(off)
            if k % 2:
                store.get_batch(pair[0], ids, out=ref, count=2)
            else:
                store.get_batch(pair[0], ids, cn, out=ref, offsets=roff)
            bad = (ref != o).nonzero().flatten()
            assert bad.numel() == 0, (n, k, bad.numel(), bad[:4].tolist())
            assert torch.equal(roff, off), (n, k)


def test_errors_match_hbm(store):
    pair = make_pair(store, 4000, 37, 4, "e")
    rng = np.random.default_rng(9)
    starts = rng.integers(0, 3990, size=600)
    counts = rng.integers(1, 5, size=600)
    starts[211] = 4000   # invalid start
    starts[400] = -3

    def run(n, dev_out, fixed):
        o = torch.full((600 * 4 * 148,), 0xAB, dtype=torch.uint8, device=DEV if dev_out else "cpu")
        with pytest.raises(ValueError) as ei:
            if fixed:
                store.get_batch(n, starts, out=o, count=2)
            else:
                store.get_batch(n, starts, counts, out=o)
        return str(ei.value), store.last_bad_index, o.cpu().numpy().tobytes()
    for dev_out in (False, True):
        for fixed in (False, True):
            assert run(pair[0], dev_out, fixed) == run(pair[1], dev_out, fixed)
    # capacity: nothing written, same code
    small = [torch.zeros(10, dtype=torch.uint8, device=DEV) for _ in pair]
    errs = []
    for n, o in zip(pair, small):
        with pytest.raises(ValueError) as ei:
            store.get_batch(n, np.arange(10), out=o, count=1)
        errs.append((str(ei.value), store.last_bad_index))
    assert errs[0] == errs[1] and torch.equal(small[0], small[1])


def test_batched_writes_and_push_are_refused(store):
    nrows, disp = 1000, 16
    h, hb = "w_host", "w_hbm"
    store.init(h, nrows, disp, 4, placement="host")
    store.synth_fill(h, SEED)
    store.init(hb, nrows, disp, 4)
    for n in (h, hb):
        store.set_sample_index(n, np.arange(nrows), np.ones(nrows, np.int64))
    store.push_setup(64, 64 * disp * 4)

    def shard():
        o = torch.zeros(nrows * disp * 4, dtype=torch.uint8, device=DEV)
        store.get_batch(h, np.arange(nrows), out=o, count=1)
        return o
    before = shard()
    ids = torch.arange(8, dtype=torch.int64, device=DEV)
    src = torch.ones(8 * disp, dtype=torch.float32, device=DEV)
    isrc = torch.ones(8 * disp, dtype=torch.int32, device=DEV)
    res = torch.zeros_like(src)
    calls = {
        "put_batch": lambda: store.put_batch(h, ids, src=src, count=1),
        "put_samples": lambda: store.put_samples(h, ids, src),
        "accumulate_batch": lambda: store.accumulate_batch(h, ids, src=src, count=1),
        "accumulate_batch max": lambda: store.accumulate_batch(h, ids, src=src, count=1, op="amax"),
        "accumulate_samples": lambda: store.accumulate_samples(h, ids, src),
        "accumulate_samples bor": lambda: store.accumulate_samples(h, ids, isrc, op="bitwise_or"),
        "get_accumulate_batch": lambda: store.get_accumulate_batch(h, ids, src=src, out=res, count=1),
        "get_accumulate_samples": lambda: store.get_accumulate_samples(h, ids, src, res, op="replace"),
        "compare_and_swap_batch": lambda: store.compare_and_swap_batch(h, ids, src=src, compare=src, out=res, count=1),
        "compare_and_swap_samples": lambda: store.compare_and_swap_samples(h, ids, src, src, res),
        "get_batch_push": lambda: store.get_batch_push(h, ids, count=1),
        "multi mixing placements": lambda: store.get_samples_multi(
            [hb, h], ids, [torch.zeros(8 * disp * 4, dtype=torch.uint8, device=DEV)] * 2),
    }
    for what, call in calls.items():
        torch.cuda.synchronize()
        n0 = launches()
        with pytest.raises(ValueError, match="DDS_PLACE_HOST|placement"):
            call()
        assert launches() == n0, what
        assert torch.equal(res, torch.zeros_like(res)), what
    assert torch.equal(shard(), before)
    # the raw C entries give DDS_ERR_ARG
    L = store._L
    tot, bad = C.c_int64(0), C.c_int64(0)
    rc = L.dds_put_batch(store._h, h.encode(), ids.data_ptr(), None, 1, 8, 4, src.data_ptr(), src.numel() * 4,
                         _capi.IDX_ON_DEVICE | _capi.SRC_ON_DEVICE, None, C.byref(tot), C.byref(bad))
    assert rc == _capi.ERR_ARG
    # an argument error that comes before the placement check keeps its code: an unknown variable
    rc = L.dds_put_batch(store._h, b"nope", ids.data_ptr(), None, 1, 8, 4, src.data_ptr(), src.numel() * 4,
                         _capi.IDX_ON_DEVICE | _capi.SRC_ON_DEVICE, None, C.byref(tot), C.byref(bad))
    assert rc == _capi.ERR_UNKNOWN_VAR


def test_update_and_ingest_into_host(store):
    nrows, disp = 5000, 256
    store.init("u", nrows, disp, 4, placement="host")
    rng = np.random.default_rng(1)
    a = rng.standard_normal((100, disp)).astype(np.float32)
    store.update("u", a, 10)
    b = torch.from_numpy(rng.standard_normal((200, disp)).astype(np.float32)).pin_memory()
    st = torch.cuda.Stream()
    store.update("u", b, 1000, stream=st.cuda_stream, wait=False)
    c = rng.standard_normal((2900, disp)).astype(np.float32)  # pageable: the staged ingest
    store.ingest("u", c, 2000)
    d = torch.from_numpy(rng.standard_normal((100, disp)).astype(np.float32)).to(DEV)
    store.update("u", d, 4900)
    store.epoch_begin()
    store.epoch_end()
    out = torch.zeros(nrows * disp, dtype=torch.float32, device=DEV)
    store.get_batch("u", np.arange(nrows), out=out, count=1)
    got = out.view(nrows, disp).cpu().numpy()
    assert got[10:110].tobytes() == a.tobytes()
    assert got[1000:1200].tobytes() == b.numpy().tobytes()
    assert got[2000:4900].tobytes() == c.tobytes()
    assert got[4900:].tobytes() == d.cpu().numpy().tobytes()
    assert not got[:10].any() and not got[110:1000].any()


def test_rewritten_rows_are_not_served_stale(store):
    nrows, disp = 2048, 64
    store.init("s", nrows, disp, 4, placement="host")
    store.synth_fill("s", SEED)
    one = np.zeros((1, disp), np.float32)
    seen = {}
    for r in (5, 700, 2047):
        store.get("s", one, r)  # served by the resident doorbell CTA
        seen[r] = one.copy()
        assert seen[r].tobytes() == np_synth_rows(SEED, r, 1, disp, np.float32).tobytes()
    for k in range(3):
        for r in seen:
            new = np.full((1, disp), 1000 * k + r, np.float32)
            store.update("s", new, r)
            store.get("s", one, r)
            assert one.tobytes() == new.tobytes(), (k, r)
        store.epoch_begin()
        out = torch.zeros(3 * disp, dtype=torch.float32, device=DEV)
        store.get_batch("s", list(seen), out=out, count=1)
        store.epoch_end()
        exp = np.concatenate([np.full(disp, 1000 * k + r, np.float32) for r in seen])
        assert out.cpu().numpy().tobytes() == exp.tobytes()


def test_host_variable_takes_no_hbm(store):
    store.init("warm", 16, 16, 4, placement="host")  # store scratch and the host-shard path are set up
    store.get_batch("warm", [0, 1], out=torch.zeros(128, dtype=torch.uint8, device=DEV), count=1)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    store.init("big", 1 << 18, 1024, 4, placement="host")  # 1 GiB
    store.synth_fill("big", SEED)
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 < (64 << 20), (free0 - free1)
    out = torch.zeros(4 * 4096, dtype=torch.uint8, device=DEV)
    store.get_batch("big", [0, 1000, 200000, (1 << 18) - 1], out=out, count=1)
    exp = np.concatenate([np_synth_rows(SEED, r, 1, 1024, np.float32) for r in (0, 1000, 200000, (1 << 18) - 1)])
    assert out.cpu().numpy().tobytes() == exp.tobytes()
    assert 1 <= _capi.lib().dds_host_gather_ctas() <= 16


def test_free_and_readd_leaks_no_descriptors():
    def nfd():
        return len(os.listdir("/proc/self/fd"))
    s = PyDDStore(device=0)
    try:
        s.init("t", 64, 8, 4, placement="host")  # the store's own one-time setup
        s.get("t", np.zeros((2, 8), np.float32), 7)
        s.free()
        n0 = nfd()
        for k in range(4):
            s.add("t", np.full((300, 8), k, np.float32), placement="host")
            s.init("t2", 100, 8, 4, placement="host")
            o = np.zeros((2, 8), np.float32)
            s.get("t", o, 7)
            assert (o == k).all()
            with pytest.raises(ValueError, match="placement"):
                s.init("t3", 10, 8, 4, placement="nvme")
            s.free()
        assert nfd() == n0
    finally:
        s.close()


TWO_RANKS = r"""
import sys
sys.path.insert(0, {root!r})
import numpy as np, torch
from ddstore_b200 import PyDDStore, ShmComm
from oracle.oracle import np_synth_rows
rank, P, key = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
dev = rank % torch.cuda.device_count()
torch.cuda.set_device(dev)
comm = ShmComm(key, rank, P)
store = PyDDStore(comm, device=dev)
disp = 1024
store.init("h", 3000 + 101 * rank, disp, 4, placement="host")
store.synth_fill("h", 0xAB)
store.epoch_begin()
ll = store.query("h")["lenlist"]
lo = ll[rank - 1] if rank else 0
other = (rank + 1) % P
olo = ll[other - 1] if other else 0
ids = np.random.default_rng(rank).integers(olo, ll[other], size=500)
out = torch.zeros(500 * disp, dtype=torch.float32, device=f"cuda:{{dev}}")
store.get_batch("h", ids, out=out, count=1)
exp = np.concatenate([np_synth_rows(0xAB, int(i), 1, disp, np.float32) for i in ids])
assert out.cpu().numpy().tobytes() == exp.tobytes()
one = np.zeros((1, disp), np.float32)
store.get("h", one, int(ids[0]))
assert one.tobytes() == exp[0].tobytes()
store.epoch_end()
try:
    store.init("d", 100, 4, 4, placement="host" if rank == 0 else "hbm")
    raise SystemExit("placement disagreement was not refused")
except ValueError as e:
    assert "disagree on the placement" in str(e), e
store.init("d", 100, 4, 4, placement="host")
store.update("d", np.full((100, 4), rank, np.float32), 0)
store.epoch_begin()
got = np.zeros((1, 4), np.float32)
store.get("d", got, 100 * other)
assert (got == other).all()
store.epoch_end()
store.free(); store.close(); comm.close()
print("host-ok", rank)
"""


def test_two_rank_processes_read_each_others_host_shards(tmp_path):
    script = tmp_path / "two_ranks.py"
    script.write_text(TWO_RANKS.format(root=ROOT))
    key = "hs" + uuid.uuid4().hex[:10]
    procs = [subprocess.Popen([sys.executable, str(script), str(r), "2", key], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"host-ok {r}" in o, f"rank {r}:\n{o[-3000:]}"
