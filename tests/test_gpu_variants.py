"""Every raw gather geometry, and the limits the code handles explicitly, against the oracle (-m gpu).

A. one adversarial workload through every entry, into destinations at every base phase, with sentinel guard bands
   around them: it reaches every raw geometry of dds_gather_kernel the launcher selects (small and large rows, both
   shared-memory plans, the plan kernels); in a subprocess each by default, with 1-chunk segments and with PDL off;
B. packed results beyond 4 GiB (fixed count, variable count, by sample id, multi-array, capacity error, pageable host);
C. the on-device verifier the benchmark trusts (dds_synth_verify) reports the corruptions it must;
D. a world of DDSK_MAX_RANKS = 64 owners, a third of them empty, and the refusal of a 65th rank."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests.gpu_helpers import (DST_OFFSETS, GUARD, check_guarded, guarded_buffer, padded_requests, run_world,
                               sample_ids, sweep_requests)

# Every device buffer or index array a test prepares on torch's stream is complete (torch.cuda.synchronize) before a
# store call that has no `stream` argument reads or writes it: the store's own stream is not ordered with torch's.

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch():
    import torch
    return torch


# ------------------------------------------------------------------------------- A. variant sweep
# (warps, stages, chunk, plan capacity) of the raw gets' geometries in kernels.cu. The sweep reaches each of them:
#   large rows  fixed-count requests of 2 KiB and more (one row of f4096 / f4100, every variable's requests just over
#               a chunk), and every variable-count batch that plans in global memory (9000 requests: "var-big",
#               get_samples and get_samples_multi);
#   small rows  fixed-count requests under 2 KiB (one row of b1 ... i20);
#   plan 4K     variable-count batches of up to 4096 requests (the "var" base workload, get_samples with 500 ids);
#   plan 8K     4097 to 8192 requests ("var-mid", 6000 requests, under DDS_SMEM_PLAN_MAX=8192).
LARGE_ROWS, SMALL_ROWS = (12, 4, 4096, 0), (16, 3, 4096, 0)
PLAN_4K, PLAN_8K = (12, 3, 4096, 4096), (12, 3, 3072, 8192)
CHUNKS = sorted({g[2] for g in (LARGE_ROWS, SMALL_ROWS, PLAN_4K, PLAN_8K)})  # (3072, 4096: the walk's cuts)

CONFIGS = {"default": {}, "minseg1": {"DDS_VAR_MINSEG": "1", "DDS_S_MINSEG": "1"}, "nopdl": {"DDS_PDL": "0"}}

# name -> (dtype, disp, rows): 1-byte rows for the phase sweep, then 3, 4, 12, 20, 4096 and 4100-byte rows
SWEEP_VARS = {"b1": (np.uint8, 1, 8 << 20), "b3": (np.uint8, 3, 3 << 20), "f4": (np.float32, 1, 5 << 19),
              "f12": (np.float32, 3, 1 << 20), "i20": (np.int32, 5, 600_000), "f4096": (np.float32, 1024, 2000),
              "f4100": (np.float32, 1025, 2000)}
MID, BIG = 6000, 9000  # request counts: shared plan with 8192 entries, plan kernels (DDS_SMEM_PLAN_MAX=8192)


def sweep_main():
    """One variant-sweep configuration (taken from the environment) end to end; raises on the first discrepancy."""
    import torch
    from ddstore_b200 import PyDDStore, _capi
    from oracle.oracle import COracle
    env = os.environ
    cfg = " ".join(f"{k}={v}" for k, v in sorted(env.items()) if k.startswith("DDS_") and k != "DDS_COMM_TIMEOUT_S")
    coracle = COracle()
    rng = np.random.default_rng(20260)
    store = PyDDStore(device=0)

    # the geometry the store reports is the large-rows one, one CTA per SM
    vals = [C.c_int() for _ in range(5)]
    _capi.lib().dds_gather_geometry(*[C.byref(v) for v in vals])
    ctas, nw, stages, ch, _ = [v.value for v in vals]
    assert (nw, stages, ch) == LARGE_ROWS[:3], (cfg, (nw, stages, ch), LARGE_ROWS)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert ctas == sms, (cfg, ctas, sms)

    shards, base = {}, {}
    for name, (dt, disp, n) in SWEEP_VARS.items():
        shards[name] = rng.integers(0, 256, size=n * disp * np.dtype(dt).itemsize, dtype=np.uint8).view(dt).reshape(n, disp)
        store.add(name, shards[name])
        base[name] = sweep_requests(rng, n, disp * np.dtype(dt).itemsize, CHUNKS)
        store.set_sample_index(name, *base[name])

    ncall = [0]

    def oracle(name, st, ct):
        exp, exp_offs, bad, _ = coracle.get_batch([shards[name]], st, ct)
        assert bad == -1, (name, bad)
        return exp, exp_offs

    def run(what, exp, exp_offs, st, ct, call):
        """call(out_view, offsets_tensor, idx_on_device) -> returned total; every index residency x base offset"""
        for idx_dev in (False, True):
            for off in (DST_OFFSETS if idx_dev else (0, 13)):
                sent = (0xA5, 0x3C)[ncall[0] & 1]
                ncall[0] += 1
                d_offs = torch.full((len(st) + 1,), -7, dtype=torch.int64, device="cuda:0")
                whole, view = guarded_buffer(torch, exp.size + GUARD, off, sent)  # (synchronizes)
                total = call(view, d_offs, idx_dev)
                check_guarded(whole, off, exp, exp_offs, st, ct, sent, f"[{cfg}] {what} idx_dev={idx_dev} dst+{off}",
                              total=total, got_offs=d_offs)

    def idx(a, dev):
        """host array, or its device copy complete before the store's stream reads it"""
        if not dev:
            return a
        t = torch.from_numpy(np.ascontiguousarray(a, np.int64)).cuda()
        torch.cuda.synchronize()
        return t

    for name, (dt, disp, n) in SWEEP_VARS.items():
        row = disp * np.dtype(dt).itemsize
        # fixed count: one row, and requests just over a chunk
        for cnt, nreq in ((1, 3000), (max(1, -(-(ch + 17) // row)), 200)):
            st = rng.integers(0, n - cnt + 1, size=nreq).astype(np.int64)
            ct = np.full(nreq, cnt, np.int64)
            exp, eo = oracle(name, st, ct)
            run(f"{name} get_batch count={cnt}", exp, eo, st, ct,
                lambda v, o, d: store.get_batch(name, idx(st, d), out=v, count=cnt, offsets=o))
        # explicit counts: shared-memory plan (<= 4096 and 4097..8192 requests), plan kernels (> 8192)
        mc = 2 if row < 1024 else 1
        for label, (st, ct) in (("var", base[name]), ("var-mid", padded_requests(rng, n, *base[name], MID, mc)),
                                ("var-big", padded_requests(rng, n, *base[name], BIG, mc))):
            exp, eo = oracle(name, st, ct)
            run(f"{name} get_batch {label} ({len(st)} requests)", exp, eo, st, ct,
                lambda v, o, d: store.get_batch(name, idx(st, d), idx(ct, d), out=v, offsets=o))
        # by sample id (the base workload is the sample index)
        bst, bct = base[name]
        for nid in (500, BIG):
            ids = sample_ids(rng, bct * row, nid)
            exp, eo = oracle(name, bst[ids], bct[ids])
            run(f"{name} get_samples ({nid} ids)", exp, eo, bst[ids], bct[ids],
                lambda v, o, d: store.get_samples(name, idx(ids, d), v, offsets=o))

    # multi-array: three variables (1, 12 and 4100-byte rows), each at its own base offset
    names = ["b1", "f12", "f4100"]
    ns = min(len(base[nm][0]) for nm in names)
    worst = np.max([base[nm][1][:ns] * SWEEP_VARS[nm][1] * np.dtype(SWEEP_VARS[nm][0]).itemsize for nm in names], axis=0)
    for nid in (300, MID // 3, BIG // 3):
        ids = sample_ids(rng, worst, nid)
        exps = {nm: oracle(nm, base[nm][0][ids], base[nm][1][ids]) for nm in names}
        for idx_dev in (False, True):
            for k in range(len(DST_OFFSETS)):
                offs = [DST_OFFSETS[(k + j) % len(DST_OFFSETS)] for j in range(len(names))]
                sent = (0xA5, 0x3C)[k & 1]
                d_offs = [torch.full((nid + 1,), -7, dtype=torch.int64, device="cuda:0") for _ in names]
                bufs = [guarded_buffer(torch, exps[nm][0].size + GUARD, o, sent) for nm, o in zip(names, offs)]
                totals = store.get_samples_multi(names, idx(ids, idx_dev), [b[1] for b in bufs], offsets=d_offs)
                for nm, (whole, _), o, f, t in zip(names, bufs, offs, d_offs, totals):
                    exp, eo = exps[nm]
                    check_guarded(whole, o, exp, eo, base[nm][0][ids], base[nm][1][ids], sent,
                                  f"[{cfg}] get_samples_multi {nid} ids, {nm} idx_dev={idx_dev} dst+{o}", total=t, got_offs=f)

    # overlapped, double-buffered queues: 6 fixed-count and 6 variable-count batches
    name = "f12"
    n = SWEEP_VARS[name][2]
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    for kind in ("fixed", "var"):
        batches = []
        for k in range(6):
            if kind == "fixed":
                st = rng.integers(0, n, size=3000).astype(np.int64)
                ct = np.ones(3000, np.int64)
            else:
                st, ct = padded_requests(rng, n, *base[name], (len(base[name][0]) + 1, BIG, MID)[k % 3])
                p = rng.permutation(len(st))
                st, ct = st[p], ct[p]
            batches.append((st, ct) + oracle(name, st, ct))
        cap = max(b[2].size for b in batches) + GUARD
        slots = [guarded_buffer(torch, cap, o, 0xA5) for o in (1, 13)]
        offs = [torch.full((BIG + 1,), -7, dtype=torch.int64, device=dev) for _ in slots]
        d_b = [(torch.from_numpy(st).to(dev), torch.from_numpy(ct).to(dev)) for st, ct, _, _ in batches]
        torch.cuda.synchronize()
        for k, (ds, dc) in enumerate(d_b):
            o, f = slots[k & 1][1], offs[k & 1][:len(batches[k][0]) + 1]
            if kind == "fixed":
                store.get_batch(name, ds, out=o, count=1, offsets=f, stream=side.cuda_stream, wait=False, overlap=True)
            else:
                store.get_batch(name, ds, dc, out=o, offsets=f, stream=side.cuda_stream, wait=False, overlap=True)
        total = store.wait()
        assert total == batches[-1][2].size, (cfg, kind, total)
        for k in (len(batches) - 1, len(batches) - 2):
            st, ct, exp, eo = batches[k]
            check_guarded(slots[k & 1][0], (1, 13)[k & 1], exp, eo, st, ct, 0xA5,
                          f"[{cfg}] overlapped {kind} queue, batch {k}", got_offs=offs[k & 1][:len(st) + 1],
                          slack_written=True)
    torch.cuda.synchronize()
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_variants import sweep_main
sweep_main()
print("sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_gather_variant_sweep(tmp_path, config):
    """every raw kernel instantiation (small and large rows, both shared-memory plans, the plan kernels) on the same
    adversarial workload: bytes, offsets, totals and guard bands against the oracle"""
    script = tmp_path / "variant_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config], DDS_SMEM_PLAN_MAX="8192")
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]


# ------------------------------------------------------------------------------- B. beyond 4 GiB
GIB4 = 1 << 32


def _free_hbm():
    torch = _torch()
    return torch.cuda.mem_get_info(0)[0]


def _need_hbm(nbytes):
    if _free_hbm() < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of free HBM, {_free_hbm() / 2**30:.1f} GiB free")


def _sentinel_untouched(whole, sentinel, chunk=1 << 28):
    """number of bytes of a (large) device buffer that differ from the sentinel, in chunks (no full-size temporary)"""
    bad = 0
    for i in range(0, whole.numel(), chunk):
        bad += int((whole[i:i + chunk] != sentinel).sum())
    return bad


def _spot_check(whole, base, offs, starts, counts, disp, dtype, seed, what):
    """byte-exact host comparison of the requests covering packed bytes 2^31 and 2^32, and of the last request"""
    T = int(offs[-1])
    picks = {int(np.searchsorted(offs, p, side="right") - 1) for p in (1 << 31, 1 << 32) if p < T} | {len(starts) - 1}
    for i in sorted(picks):
        a, b = int(offs[i]), int(offs[i + 1])
        got = whole[base + a:base + b].cpu().numpy()
        exp = O.np_synth_rows(seed, int(starts[i]), int(counts[i]), disp, dtype).view(np.uint8).reshape(-1)
        assert np.array_equal(got, exp), f"{what}: request {i} (start={starts[i]}, count={counts[i]}, offset {a}) differs"


def test_fixed_count_beyond_4gib():
    """~1.1 M rows of 4100 bytes (4.5 GB) into a device buffer whose base is 4 bytes past a 16-byte boundary: 2^32 falls
    inside a row; then the same batch one byte too large for its buffer (capacity error, nothing written)"""
    torch = _torch()
    disp, shard_rows, B, off, seed = 1025, 50_000, 1_100_000, 4, 0xB16
    row = disp * 4
    T = B * row
    assert T > GIB4
    # peak: shard 205 MB + destination T + 2 x 8.8 MB of starts / offsets + store scratch
    _need_hbm(shard_rows * row + T + 2 * 8 * (B + 1) + (512 << 20))

    def body(store, r):
        store.init("x", shard_rows, disp, 4)
        store.synth_fill("x", seed)
        rng = np.random.default_rng(3)
        st = rng.integers(0, shard_rows, size=B).astype(np.int64)
        d_st = torch.from_numpy(st).cuda()
        d_offs = torch.full((B + 1,), -1, dtype=torch.int64, device="cuda:0")
        whole, view = guarded_buffer(torch, T, off, 0x5A)
        assert store.get_batch("x", d_st, out=view, count=1, offsets=d_offs) == T
        offs = d_offs.cpu().numpy()
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum(np.full(B, row, np.int64))]))
        bad, rows, hist = store.synth_verify("x", view, d_st, count=1, seed=seed)
        assert (bad, rows, hist) == (0, B, [B])
        _spot_check(whole, GUARD + off, offs, st, np.ones(B, np.int64), disp, np.float32, seed, "fixed > 4 GiB")
        assert _sentinel_untouched(whole[:GUARD + off], 0x5A) == 0
        assert _sentinel_untouched(whole[GUARD + off + T:], 0x5A) == 0
        # one byte short: "too small", and the whole buffer keeps its sentinel
        whole.fill_(0x77)
        torch.cuda.synchronize()
        short = whole[GUARD + off:GUARD + off + T - 1]
        with pytest.raises(ValueError, match="too small"):
            store.get_batch("x", d_st, out=short, count=1)
        assert _sentinel_untouched(whole, 0x77) == 0
        return True

    assert all(run_world(1, body, timeout=900))


def _var_world(store, rng, seed, nreq, per_req):
    """float32 x 3 (12-byte rows) synth shard; nreq requests of ~per_req bytes each"""
    disp, rows = 3, 1_000_000
    store.init("v", rows, disp, 4)
    store.synth_fill("v", seed)
    cnt = rng.integers(per_req // 12 // 2, per_req // 12 * 3 // 2, size=nreq).astype(np.int64)
    cnt[rng.integers(0, nreq, size=nreq // 50)] = 0  # some zero-count requests
    st = (rng.integers(0, rows - cnt.max(), size=nreq)).astype(np.int64)
    return disp, st, cnt


def test_variable_count_and_samples_beyond_4gib():
    """~700 explicit (start, count) requests packing to > 4 GiB: by request count this batch would plan in shared memory
    (32-bit offsets), the capacity alone must move it to the plan kernels; the same through get_samples; and the batch
    one byte too large for its buffer"""
    torch = _torch()
    nreq, per_req, off, seed = 700, 6_600_000, 4, 0xB17
    rng = np.random.default_rng(4)
    # peak: shard 12 MB + destination (<= 1.5 x per_req x nreq = 6.9 GB) + store scratch
    _need_hbm(12_000_000 + per_req * 3 // 2 * nreq + (512 << 20))

    def body(store, r):
        disp, st, ct = _var_world(store, rng, seed, nreq, per_req)
        row = disp * 4
        exp_offs = np.concatenate([[0], np.cumsum(ct * row)]).astype(np.int64)
        T = int(exp_offs[-1])
        assert T > GIB4
        d_st, d_ct = torch.from_numpy(st).cuda(), torch.from_numpy(ct).cuda()
        store.set_sample_index("v", st, ct)
        d_ids = torch.arange(nreq, dtype=torch.int64, device="cuda:0")
        whole, view = guarded_buffer(torch, T, off, 0x5A)
        for what, call in (("get_batch", lambda o: store.get_batch("v", d_st, d_ct, out=view, offsets=o)),
                           ("get_batch host idx", lambda o: store.get_batch("v", st, ct, out=view, offsets=o)),
                           ("get_samples", lambda o: store.get_samples("v", d_ids, view, offsets=o))):
            whole.fill_(0x5A)
            d_offs = torch.full((nreq + 1,), -1, dtype=torch.int64, device="cuda:0")
            torch.cuda.synchronize()
            assert call(d_offs) == T, what
            assert np.array_equal(d_offs.cpu().numpy(), exp_offs), what
            bad, rows, hist = store.synth_verify("v", view, d_st, d_ct, offsets=d_offs, seed=seed)
            assert (bad, rows, hist) == (0, int(ct.sum()), [int((ct > 0).sum())]), what
            _spot_check(whole, GUARD + off, exp_offs, st, ct, disp, np.float32, seed, what)
            assert _sentinel_untouched(whole[:GUARD + off], 0x5A) == 0, what
            assert _sentinel_untouched(whole[GUARD + off + T:], 0x5A) == 0, what
        whole.fill_(0x77)
        torch.cuda.synchronize()
        with pytest.raises(ValueError, match="too small"):
            store.get_batch("v", d_st, d_ct, out=whole[GUARD + off:GUARD + off + T - 1])
        assert _sentinel_untouched(whole, 0x77) == 0
        return True

    assert all(run_world(1, body, timeout=900))


def test_multi_array_beyond_4gib_in_total():
    """two variables whose packed results are each below 4 GiB but together above it, in one multi-array launch:
    per-variable offsets exact, payload verified on the device"""
    torch = _torch()
    rng = np.random.default_rng(5)
    nsamp, nid = 2000, 800
    # variable a: float32 x 1025 (4100-byte rows), variable b: int64 x 3 (24-byte rows); ~2.2 GB packed each
    spec = {"a": (1025, 4, 0xA1, 2_000, 900), "b": (3, 8, 0xB2, 300_000, 160_000)}
    # peak: shards 8.2 + 7.2 MB, destinations <= 2 x 2^32 - 1, store scratch
    _need_hbm(2 * GIB4 + (512 << 20))

    def body(store, r):
        tabs, outs, offs = {}, [], []
        ids = rng.integers(0, nsamp, size=nid).astype(np.int64)
        for nm, (disp, isz, seed, rows, maxc) in spec.items():
            store.init(nm, rows, disp, isz)
            store.synth_fill(nm, seed)
            ct = rng.integers(maxc // 2, maxc, size=nsamp).astype(np.int64)
            st = rng.integers(0, rows - ct).astype(np.int64)
            store.set_sample_index(nm, st, ct)
            tabs[nm] = (st, ct)
        tot = {nm: int((tabs[nm][1][ids] * spec[nm][0] * spec[nm][1]).sum()) for nm in spec}
        assert all(t < GIB4 for t in tot.values()) and sum(tot.values()) >= GIB4, tot
        for nm in spec:
            outs.append(torch.empty(tot[nm] + 16, dtype=torch.uint8, device="cuda:0"))
            offs.append(torch.full((nid + 1,), -1, dtype=torch.int64, device="cuda:0"))
        d_ids = torch.from_numpy(ids).cuda()
        torch.cuda.synchronize()
        totals = store.get_samples_multi(list(spec), d_ids, outs, offsets=offs)
        assert totals == [tot[nm] for nm in spec]
        for nm, o, f in zip(spec, outs, offs):
            disp, isz, seed, _, _ = spec[nm]
            st, ct = tabs[nm][0][ids], tabs[nm][1][ids]
            eo = np.concatenate([[0], np.cumsum(ct * disp * isz)]).astype(np.int64)
            assert np.array_equal(f.cpu().numpy(), eo), nm
            d_st, d_ct = torch.from_numpy(st).cuda(), torch.from_numpy(ct).cuda()
            torch.cuda.synchronize()
            bad, rows, _ = store.synth_verify(nm, o, d_st, d_ct, offsets=f, seed=seed)
            assert (bad, rows) == (0, int(ct.sum())), nm
            _spot_check(o, 0, eo, st, ct, disp, np.float32 if isz == 4 else np.int64, seed, f"multi {nm}")
        return True

    assert all(run_world(1, body, timeout=900))


def _host_available():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def test_pageable_host_destination_beyond_4gib():
    """a fixed-count batch of 4.5 GB into a pageable ndarray (staged through HBM and the pinned worker pool)"""
    torch = _torch()
    disp, shard_rows, B, seed = 1025, 50_000, 1_100_000, 0xB18
    row = disp * 4
    T = B * row
    # HBM: shard + the store's staging buffer (T) + the result copied back for the device verifier (T)
    _need_hbm(shard_rows * row + 2 * T + (512 << 20))
    if _host_available() < T + (4 << 30):
        pytest.skip(f"needs {(T + (4 << 30)) / 2**30:.1f} GiB of available host RAM for a {T / 2**30:.1f} GiB pageable "
                    f"destination, {_host_available() / 2**30:.1f} GiB available")

    def body(store, r):
        store.init("x", shard_rows, disp, 4)
        store.synth_fill("x", seed)
        st = np.random.default_rng(6).integers(0, shard_rows, size=B).astype(np.int64)
        host = np.full(T + 64, 0x5A, np.uint8)
        view = host[:T].view(np.float32).reshape(B, disp)
        assert store.get_batch("x", st, out=view, count=1) == T
        assert (host[T:] == 0x5A).all()
        offs = np.arange(B + 1, dtype=np.int64) * row
        _spot_check(torch.from_numpy(host), 0, offs, st, np.ones(B, np.int64), disp, np.float32, seed, "pageable > 4 GiB")
        back, d_st = torch.from_numpy(host[:T]).cuda(), torch.from_numpy(st).cuda()
        torch.cuda.synchronize()
        bad, rows, _ = store.synth_verify("x", back, d_st, count=1, seed=seed)
        assert (bad, rows) == (0, B)
        return True

    assert all(run_world(1, body, timeout=900))


# ------------------------------------------------------------------------------- C. the verifier can fail
def test_synth_verify_reports_corruptions():
    """dds_synth_verify (the bench's correctness gate) on a correct batch and on known corruptions of it: one flipped bit
    = exactly one mismatch wherever it is, a zeroed request = its nonzero elements, and the per-owner histogram over a
    world with empty ranks"""
    torch = _torch()
    nrows = [300, 0, 0, 257, 0, 411]
    P = len(nrows)
    ll = np.cumsum(nrows)
    VARS = (("v1", 1, 7, np.uint8, 0xC1), ("v4", 4, 5, np.uint32, 0xC4), ("v8", 8, 3, np.uint64, 0xC8))

    def body(store, r):
        for name, isz, disp, _, seed in VARS:
            store.init(name, nrows[r], disp, isz)
            store.synth_fill(name, seed)
        if r != 0:
            return True
        from tests.helpers import random_valid_requests
        rng = np.random.default_rng(7)
        for name, isz, disp, dt, seed in VARS:
            row = disp * isz
            st, ct = random_valid_requests(rng, ll, 300, max_count=5)
            ct[:3] = [0, 3, 2]  # a zero-count request first, then two multi-row ones back to back
            st[1:3] = [10, 20]
            ct[-1] = 0
            for mode in ("explicit", "fixed"):
                if mode == "fixed":
                    st = np.array([s for s in st.tolist() if O.np_locate(ll, s, 2)[2] == 0], np.int64)
                    ct = np.full(len(st), 2, np.int64)
                eo = np.concatenate([[0], np.cumsum(ct * row)]).astype(np.int64)
                T = int(eo[-1])
                d_st, d_ct = torch.from_numpy(st).cuda(), torch.from_numpy(ct).cuda()
                out = torch.zeros(T, dtype=torch.uint8, device="cuda:0")
                d_offs = torch.zeros(len(st) + 1, dtype=torch.int64, device="cuda:0")
                torch.cuda.synchronize()
                if mode == "fixed":
                    assert store.get_batch(name, d_st, out=out, count=2) == T

                    def verify():
                        torch.cuda.synchronize()  # (the corruption below is written on torch's stream)
                        return store.synth_verify(name, out, d_st, count=2, seed=seed)
                else:
                    assert store.get_batch(name, d_st, d_ct, out=out, offsets=d_offs) == T

                    def verify():
                        torch.cuda.synchronize()
                        return store.synth_verify(name, out, d_st, d_ct, offsets=d_offs, seed=seed)
                hist = np.bincount(np.searchsorted(ll, st[ct > 0], side="right"), minlength=P).tolist()
                assert verify() == (0, int(ct.sum()), hist), (name, mode)
                # one flipped bit: first element, last, one inside a multi-row request, both sides of a request boundary
                nz = np.nonzero(ct > 1)[0]
                k = int(nz[0])
                nxt = int(np.nonzero(ct[k + 1:] > 0)[0][0]) + k + 1
                elems = [0, T // isz - 1, int(eo[k]) // isz + disp + 1, int(eo[nxt]) // isz - 1, int(eo[nxt]) // isz]
                for e in elems:
                    b = e * isz + e % isz
                    orig = int(out[b])
                    out[b] = orig ^ (1 << (e % 8))
                    got = verify()
                    out[b] = orig
                    assert got[:2] == (1, int(ct.sum())), (name, mode, "element", e, got[:2])
                # a whole request zeroed: every element of it whose expected value is nonzero
                for q in (k, nxt, int(np.nonzero(ct > 0)[0][-1])):
                    saved = out[eo[q]:eo[q + 1]].clone()
                    out[eo[q]:eo[q + 1]] = 0
                    got = verify()
                    out[eo[q]:eo[q + 1]] = saved
                    nonzero = int(np.count_nonzero(O.np_synth_rows(seed, int(st[q]), int(ct[q]), disp, dt)))
                    assert got[0] == nonzero, (name, mode, "request", q, got[0], nonzero)
                assert verify()[0] == 0
        return True

    assert all(run_world(P, body))


# ------------------------------------------------------------------------------- D. 64 owners
def test_sixty_four_owners(coracle):
    """DDSK_MAX_RANKS thread-ranks on one GPU, a third of them empty (first and last rank, runs of empty ones): the first
    and last row of every owner, counts ending exactly at an owner's end and one row past it, through get, get_batch
    (fixed and variable counts) and get_samples"""
    torch = _torch()
    P = 64
    rng = np.random.default_rng(64)
    empty = {0, 1, 2, 9, 10, 17, 23, 24, 25, 26, 31, 32, 40, 47, 48, 55, 58, 59, 60, 61, 63}
    nrows = [0 if r in empty else int(rng.integers(2, 40)) for r in range(P)]
    nrows[3] = nrows[62] = 1  # one-row owners: first row == last row
    shards = [rng.integers(0, 256, size=(n, 5), dtype=np.uint8) for n in nrows]
    ll = O.np_lenlist(nrows)
    owners = [(int(ll[r] - nrows[r]), int(ll[r])) for r in range(P) if nrows[r]]
    good, bad = [], []
    for lo, hi in owners:
        good += [(lo, 1), (hi - 1, 1), (lo, hi - lo), (hi - 1, 0)]
        if hi - lo > 1:
            good.append((lo + 1, hi - lo - 1))
        bad += [(lo, hi - lo + 1), (hi - 1, 2)]
    for s, c in good:
        assert coracle.locate(ll, s, c)[2] == 0
    for s, c in bad:
        assert coracle.locate(ll, s, c)[2] == 3  # the reference's "Invalid count on target"
    gst, gct = np.array(good, np.int64).T.copy()
    exp, exp_offs, b, _ = coracle.get_batch(shards, gst, gct)
    assert b == -1
    CHECK = 63  # an empty rank does the checking: everything it fetches is remote

    def body(store, r):
        store.add("v", shards[r])
        assert store.query("v")["lenlist"] == ll.tolist()
        if r != CHECK:
            return True
        for s, c in good:
            buf = np.zeros((c, 5), np.uint8)
            store.get("v", buf, s)
            e, _, _, _ = coracle.get_batch(shards, [s], [c])
            assert buf.tobytes() == e.tobytes(), (s, c)
        for s, c in bad:
            with pytest.raises(ValueError) as ei:
                store.get("v", np.zeros((c, 5), np.uint8), s)
            assert str(ei.value) == "Invalid count on target", (s, c)
        # variable counts: host indices -> host buffer, device indices -> device buffer at an odd base
        out = np.zeros(exp.size, np.uint8)
        offs = np.zeros(len(gst) + 1, np.int64)
        assert store.get_batch("v", gst, gct, out=out, offsets=offs) == exp.size
        assert out.tobytes() == exp.tobytes() and offs.tolist() == exp_offs.tolist()
        d_offs = torch.zeros(len(gst) + 1, dtype=torch.int64, device="cuda:0")
        d_st, d_ct = torch.from_numpy(gst).cuda(), torch.from_numpy(gct).cuda()
        whole, view = guarded_buffer(torch, exp.size + GUARD, 13, 0xA5)  # (synchronizes)
        n = store.get_batch("v", d_st, d_ct, out=view, offsets=d_offs)
        check_guarded(whole, 13, exp, exp_offs, gst, gct, 0xA5, "64 owners, variable counts", total=n, got_offs=d_offs)
        # an invalid request in the middle: the reference's error, at its index
        k = len(good) // 2
        st2 = np.insert(gst, k, bad[len(bad) // 2][0])
        ct2 = np.insert(gct, k, bad[len(bad) // 2][1])
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get_batch("v", st2, ct2, out=np.zeros(exp.size + 1024, np.uint8))
        assert store.last_bad_index == k
        # fixed count 1: first and last row of every owner; fixed count 2 ending one row past an owner
        fst = np.array([x for lo, hi in owners for x in (lo, hi - 1)], np.int64)
        e1, eo1, b1, _ = coracle.get_batch(shards, fst, np.ones(len(fst), np.int64))
        assert b1 == -1
        d_offs = torch.zeros(len(fst) + 1, dtype=torch.int64, device="cuda:0")
        d_fst = torch.from_numpy(fst).cuda()
        whole, view = guarded_buffer(torch, e1.size, 1, 0x3C)
        n = store.get_batch("v", d_fst, out=view, count=1, offsets=d_offs)
        check_guarded(whole, 1, e1, eo1, fst, np.ones(len(fst)), 0x3C, "64 owners, fixed count", total=n, got_offs=d_offs)
        two = np.array([lo for lo, hi in owners if hi - lo >= 2] + [owners[5][1] - 1], np.int64)
        assert coracle.locate(ll, int(two[-1]), 2)[2] == 3
        with pytest.raises(ValueError, match="Invalid count on target"):
            store.get_batch("v", two, out=np.zeros(len(two) * 10, np.uint8), count=2)
        assert store.last_bad_index == len(two) - 1
        # by sample id: the good requests are the samples
        store.set_sample_index("v", gst, gct)
        ids = rng.permutation(len(gst)).astype(np.int64)
        e2, eo2, _, _ = coracle.get_batch(shards, gst[ids], gct[ids])
        d_offs = torch.zeros(len(ids) + 1, dtype=torch.int64, device="cuda:0")
        d_ids = torch.from_numpy(ids).cuda()
        whole, view = guarded_buffer(torch, e2.size + GUARD, 8, 0xA5)
        n = store.get_samples("v", d_ids, view, offsets=d_offs)
        check_guarded(whole, 8, e2, eo2, gst[ids], gct[ids], 0xA5, "64 owners, get_samples", total=n, got_offs=d_offs)
        return True

    assert all(run_world(P, body, timeout=600))


def test_sixty_five_ranks_are_refused():
    """a communicator larger than DDSK_MAX_RANKS: every rank gets the store's error from add(), nobody hangs"""
    def body(store, r):
        with pytest.raises(ValueError) as ei:
            store.add("v", np.zeros((2, 3), np.uint8))
        assert "DDSK_MAX_RANKS" in str(ei.value)
        return True

    assert run_world(65, body, timeout=300) == [True] * 65
