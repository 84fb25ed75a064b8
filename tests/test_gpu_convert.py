"""Converting batches on the GPU (dds_get_batch_convert, dds_get_samples_convert, dds_get_samples_multi_convert and
the loaders built on them).

Every converted batch is checked three ways: its bytes equal torch's CUDA `.to()` of the raw gather of the same
requests bitwise, and the NumPy oracle of tests/convert_oracle.py (NaN by class); its offsets and total are the raw
ones in output bytes; the sentinel guard bands around the destination are untouched. Payload comes from synth_fill
(its bits include NaN, +-inf, subnormals and -0) plus explicit rounding-edge rows. Each conversion goes through the
fixed-count entry, explicit counts at <= 1024, 4097..8192 and > 8192 requests (and, in a subprocess with
DDS_SMEM_PLAN_MAX=8192, the 8192-request shared-memory plan), get_samples, and get_samples_multi with mixed codes
including raw bytes; with host and device indices, into destinations at several aligned base offsets.

On an H100 80GB HBM3 (400 W power limit) the module takes about 30 s, the 4 GiB case and the subprocess included.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import convert_oracle as co

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD, SENT = 64, 0xA5
DEV = torch.device("cuda", 0)

# variable -> (numpy dtype, disp); odd disps make most rows start off a 16-byte boundary
VARS = {"f32": (np.float32, 37), "f64": (np.float64, 29), "u8": (np.uint8, 51)}
NROWS = 30_000
NSAMP = 12_000
_x = torch.arange(256, dtype=torch.float32)
# (name, variable, source dtype, output dtype, table, code)
CASES = [("f32_bf16", "f32", torch.float32, torch.bfloat16, None, co.CVT_F32_BF16),
         ("f32_f16", "f32", torch.float32, torch.float16, None, co.CVT_F32_F16),
         ("f64_f32", "f64", torch.float64, torch.float32, None, co.CVT_F64_F32),
         ("u8_lut16_bf16", "u8", torch.uint8, torch.bfloat16, ((_x - 127.5) / 60.1).to(torch.bfloat16), co.CVT_U8_LUT16),
         ("u8_lut16_f16_default", "u8", torch.uint8, torch.float16, None, co.CVT_U8_LUT16),
         ("u8_lut32", "u8", torch.uint8, torch.float32, _x / 255, co.CVT_U8_LUT32)]
CASE_IDS = [c[0] for c in CASES]


def _edge_rows(disp):
    """float32 rounding edges for bf16 and f16: ties both ways, overflow, subnormals, -0, inf, NaN"""
    vals = np.array(co.F32_EDGE_BITS, np.uint32)
    n = (len(vals) * 4 + disp - 1) // disp
    return np.resize(vals, n * disp).reshape(n, disp).view(np.float32)


@pytest.fixture(scope="module")
def env():
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    rng = np.random.default_rng(11)
    L = rng.integers(0, 5, NSAMP)  # (about 2 rows per sample: the samples fit the rows)
    L[:: 97] = 0
    sstart = np.concatenate([[0], np.cumsum(L)])
    assert sstart[-1] <= NROWS
    for name, (dt, disp) in VARS.items():
        store.init(name, NROWS, disp, np.dtype(dt).itemsize)
        store.synth_fill(name, 99)
        store.set_sample_index(name, sstart[:-1].copy(), L)
    edge = _edge_rows(VARS["f32"][1])
    store.update("f32", edge, 5)
    store.update("f64", edge.astype(np.float64)[:, :VARS["f64"][1]].copy(), 9)
    yield {"store": store, "L": L, "sstart": sstart, "rng": rng}
    store.free()
    store.close()


def _raw(store, var, kind, a, b=None, count=None):
    """the raw gather of the same requests: (bytes as a uint8 CUDA tensor, offsets)"""
    dt, disp = VARS[var]
    row = disp * np.dtype(dt).itemsize
    n = len(a)
    nb = n * count * row if kind == "fixed" else int(np.clip(b, 0, None).sum()) * row
    buf = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    offs = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    if kind == "fixed":
        t = store.get_batch(var, a, out=buf, count=count, offsets=offs)
    else:
        t = store.get_batch(var, a, b, out=buf, offsets=offs)
    return buf[:t], offs.cpu().numpy()


def _raw_samples(store, var, ids, L):
    dt, disp = VARS[var]
    nb = int(L[ids].sum()) * disp * np.dtype(dt).itemsize
    buf = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    offs = torch.empty(len(ids) + 1, dtype=torch.int64, device=DEV)
    t = store.get_samples(var, ids, buf, offsets=offs)
    return buf[:t], offs.cpu().numpy()


def _torch_cast(raw_u8, case):
    _, var, sdt, odt, lut, code = case
    if code in (co.CVT_U8_LUT16, co.CVT_U8_LUT32):
        table = (torch.arange(256).to(odt) if lut is None else lut).to(DEV)
        return table[raw_u8.long()].view(torch.uint8).reshape(-1)
    return raw_u8.view(sdt).to(odt).view(torch.uint8).reshape(-1)


def _table_bytes(case):
    _, _, _, odt, lut, code = case
    if code not in (co.CVT_U8_LUT16, co.CVT_U8_LUT32):
        return None
    t = torch.arange(256).to(odt) if lut is None else lut
    return t.contiguous().view(torch.uint8).numpy()


def _dest(nbytes, off):
    whole = torch.full((2 * GUARD + off + nbytes,), SENT, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    return whole, whole[GUARD + off:GUARD + off + nbytes]


def _check(case, whole, off, got_total, got_offs, raw_u8, raw_offs, what):
    code = case[5]
    exp_dev = _torch_cast(raw_u8, case)
    nb = exp_dev.numel()
    assert got_total == nb, f"{what}: total {got_total} != {nb}"
    body = whole[GUARD + off:GUARD + off + nb]
    eq = torch.equal(body, exp_dev)
    if not eq:
        bad = torch.nonzero(body != exp_dev)[:4].flatten().tolist()
        raise AssertionError(f"{what}: bytes differ from torch's cast at {bad}")
    h = whole.cpu().numpy()
    assert (h[:GUARD + off] == SENT).all() and (h[GUARD + off + nb:] == SENT).all(), f"{what}: guard band written"
    exp_np = co.convert_bytes(raw_u8.cpu().numpy(), code, _table_bytes(case))
    bad = co.same_bits_or_both_nan(h[GUARD + off:GUARD + off + nb], exp_np, code)
    assert bad.size == 0, f"{what}: {bad.size} elements differ from the NumPy oracle, first {bad[0]}"
    if got_offs is not None:
        assert got_offs.tolist() == [co.out_bytes(int(x), code) for x in raw_offs], f"{what}: offsets"


def _offsets_for(case):
    o = co.SIZES[case[5]][1]
    return [x for x in (0, 2, 4, 12) if x % o == 0]


def _requests(rng, var, n, max_count):
    starts = rng.integers(0, NROWS - max_count, n)
    counts = rng.integers(0, max_count + 1, n)
    starts[: min(n, 4)] = [5, 6, 9, 0][: min(n, 4)]  # the rounding-edge rows
    return starts.astype(np.int64), counts.astype(np.int64)


def _idx(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if dev else a


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_fixed_count(env, case):
    store, rng = env["store"], env["rng"]
    var, sdt, odt, lut = case[1], case[2], case[3], case[4]
    starts = rng.integers(0, NROWS - 3, 3000)
    starts[:3] = [5, 6, 9]
    raw, roffs = _raw(store, var, "fixed", starts, count=3)
    nb = co.out_bytes(raw.numel(), case[5])
    for dev in (False, True):
        for off in _offsets_for(case):
            whole, view = _dest(nb, off)
            offs = torch.full((len(starts) + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_batch(var, _idx(starts, dev), out=view.view(odt), count=3, offsets=offs, src_dtype=sdt, lut=lut)
            _check(case, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} fixed dev={dev} off={off}")


@pytest.mark.parametrize("nreq", [700, 5000, 9000])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_explicit_counts(env, case, nreq):
    store, rng = env["store"], env["rng"]
    var, sdt, odt, lut = case[1], case[2], case[3], case[4]
    starts, counts = _requests(rng, var, nreq, 6)
    raw, roffs = _raw(store, var, "var", starts, counts)
    nb = co.out_bytes(raw.numel(), case[5])
    for dev in (False, True):
        for off in _offsets_for(case)[:2]:
            whole, view = _dest(nb, off)
            offs = torch.full((nreq + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_batch(var, _idx(starts, dev), _idx(counts, dev), out=view.view(odt), offsets=offs, src_dtype=sdt,
                                lut=lut)
            _check(case, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} var n={nreq} dev={dev} off={off}")


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_samples(env, case):
    store, rng, L = env["store"], env["rng"], env["L"]
    var, sdt, odt, lut = case[1], case[2], case[3], case[4]
    for n in (900, 10_000):
        ids = rng.integers(0, NSAMP, n)
        raw, roffs = _raw_samples(store, var, ids, L)
        nb = co.out_bytes(raw.numel(), case[5])
        for dev in (False, True):
            off = _offsets_for(case)[-1]
            whole, view = _dest(nb, off)
            offs = torch.full((n + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_samples(var, _idx(ids, dev), view.view(odt), offsets=offs, src_dtype=sdt, lut=lut)
            _check(case, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} samples n={n} dev={dev}")


@pytest.mark.parametrize("n", [300, 3000])
def test_multi_mixed_codes(env, n):
    store, rng, L = env["store"], env["rng"], env["L"]
    combos = [[("f32", CASES[0]), ("f64", None), ("u8", CASES[5])], [("f64", CASES[2]), ("u8", CASES[3]), ("f32", CASES[1])],
              [("u8", None), ("f32", None), ("f64", CASES[2])], [("u8", CASES[4]), ("f32", CASES[0])]]
    for pairs in combos:
        names, combo = [p[0] for p in pairs], [p[1] for p in pairs]
        for dev in (False, True):
            ids = rng.integers(0, NSAMP, n)
            ids[0] = NSAMP - 1
            raws = [_raw_samples(store, nm, ids, L) for nm in names]
            wholes, outs, offs = [], [], []
            for c, nm, (raw, _) in zip(combo, names, raws):
                code = c[5] if c else co.CVT_NONE
                nb = co.out_bytes(raw.numel(), code)
                off = 4
                whole, view = _dest(nb, off)
                wholes.append(whole)
                outs.append(view.view(c[3]) if c else view)
                offs.append(torch.full((n + 1,), -7, dtype=torch.int64, device=DEV))
            tots = store.get_samples_multi(names, _idx(ids, dev), outs, offsets=offs,
                                           src_dtypes=[c[2] if c else None for c in combo],
                                           luts=[c[4] if c else None for c in combo])
            for c, nm, (raw, roffs), whole, of, t in zip(combo, names, raws, wholes, offs, tots):
                what = f"multi {names} var {nm} dev={dev}"
                if c is None:
                    assert t == raw.numel() and torch.equal(whole[GUARD + 4:GUARD + 4 + t], raw), what
                    assert of.cpu().numpy().tolist() == roffs.tolist(), what
                else:
                    _check(c, whole, 4, t, of.cpu().numpy(), raw, roffs, what)


def test_argument_errors(env):
    store = env["store"]
    out = torch.empty(64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(ValueError, match="Invalid data type"):  # itemsize of the variable vs the code's source
        store.get_batch("f64", [1, 2], out=out, src_dtype=torch.float32)
    with pytest.raises(ValueError):  # host destination
        store.get_batch("f32", [1, 2], out=np.zeros(200, np.float32), src_dtype=np.float64)
    with pytest.raises(ValueError):  # destination not aligned to the output itemsize
        _misaligned(store, torch.empty(1000, dtype=torch.uint8, device=DEV))
    with pytest.raises(NotImplementedError):  # a bf16 out without a conversion
        store.get_batch("f32", [1, 2], out=out)
    from ddstore_b200 import _capi
    L = _capi.lib()
    tot, bad = ctypes.c_int64(0), ctypes.c_int64(0)
    for cv in (_capi.Convert(9, None), _capi.Convert(0, None), _capi.Convert(co.CVT_U8_LUT32, None)):
        st = np.array([1], np.int64)
        rc = L.dds_get_batch_convert(store._h, b"u8" if cv.code == co.CVT_U8_LUT32 else b"f32", st.ctypes.data, None, 1, 1,
                                     out.data_ptr(), 128, None, _capi.DST_ON_DEVICE, None, ctypes.byref(cv),
                                     ctypes.byref(tot), ctypes.byref(bad))
        assert rc == _capi.ERR_ARG, cv.code


def _misaligned(store, raw):
    from ddstore_b200 import _capi
    L = _capi.lib()
    tot, bad = ctypes.c_int64(0), ctypes.c_int64(0)
    cv = _capi.Convert(co.CVT_F32_BF16, None)
    st = np.array([1], np.int64)
    rc = L.dds_get_batch_convert(store._h, b"f32", st.ctypes.data, None, 1, 1, raw.data_ptr() + 1, 500, None,
                                 _capi.DST_ON_DEVICE, None, ctypes.byref(cv), ctypes.byref(tot), ctypes.byref(bad))
    _capi.raise_for(rc)


@pytest.mark.parametrize("entry", ["fixed", "var", "samples", "multi"])
def test_first_invalid_request(env, entry):
    """the first invalid request raises with its index; the requests before it are delivered converted; later bytes are
    sentinel or the converted value of a valid request at its converted offset; capacity one element short writes
    nothing"""
    store, rng, L = env["store"], env["rng"], env["L"]
    case = CASES[0]
    n = 2000
    for bad_at, kind in ((0, "start"), (31, "count"), (1023, "start"), (n - 1, "start")):
        starts, counts = _requests(rng, "f32", n, 3)
        counts[counts == 0] = 1
        ids = rng.integers(0, NSAMP, n)
        if entry == "fixed":
            counts[:] = 2
        good_s, good_c, good_i = starts.copy(), counts.copy(), ids.copy()
        if entry in ("samples", "multi"):
            ids[bad_at] = NSAMP + 5
            good_i[bad_at] = 0
            kind = "sample"
        elif kind == "start":
            starts[bad_at] = NROWS + 3
            good_c[bad_at] = 0 if entry == "var" else good_c[bad_at]
        else:
            counts[bad_at] = NROWS * 4 if entry == "var" else counts[bad_at]
            if entry == "fixed":
                starts[bad_at] = NROWS - 1
            good_c[bad_at] = 0 if entry == "var" else good_c[bad_at]
        if entry == "fixed":
            raw, roffs = _raw(store, "f32", "fixed", good_s, count=2)
        elif entry == "var":
            raw, roffs = _raw(store, "f32", "var", good_s, good_c)
        else:
            Lg = L.copy()
            raw, roffs = _raw_samples(store, "f32", good_i, Lg)
        exp = _torch_cast(raw, case).cpu().numpy()
        eoffs = [co.out_bytes(int(x), case[5]) for x in roffs]
        cap = len(exp) + 64
        whole, view = _dest(cap, 0)
        with pytest.raises(ValueError) as ei:
            if entry == "fixed":
                store.get_batch("f32", starts, out=view.view(torch.bfloat16), count=2, src_dtype=torch.float32)
            elif entry == "var":
                store.get_batch("f32", starts, counts, out=view.view(torch.bfloat16), src_dtype=torch.float32)
            elif entry == "samples":
                store.get_samples("f32", ids, view.view(torch.bfloat16), src_dtype=torch.float32)
            else:  # (a raw second variable: the invalid sample is first met in variable 0)
                spare = torch.empty(int(L[good_i].sum()) * VARS["u8"][1] + 64, dtype=torch.uint8, device=DEV)
                store.get_samples_multi(["f32", "u8"], ids, [view.view(torch.bfloat16), spare],
                                        src_dtypes=[torch.float32, None])
        assert store.last_bad_index == bad_at, (entry, kind, store.last_bad_index)
        h = whole.cpu().numpy()[GUARD:GUARD + cap]
        p = eoffs[bad_at]
        assert np.array_equal(h[:p], exp[:p]), f"{entry}: prefix before request {bad_at}"
        rest = h[p:len(exp)]
        ok = (rest == SENT) | (rest == exp[p:])
        if entry == "fixed":  # the invalid request keeps its slot, untouched
            slot = np.zeros(len(rest), bool)
            slot[: eoffs[bad_at + 1] - p] = True
            ok |= slot & (rest == SENT)
        assert ok.all(), f"{entry}: a byte past the prefix is neither untouched nor the converted request's"
        assert (whole.cpu().numpy()[GUARD + len(exp):] == SENT).all()
        assert "nvalid" in str(ei.value) or "sample" in str(ei.value)
    # capacity one element short: nothing written; then the next valid call on the same destination works
    starts, counts = _requests(rng, "f32", 600, 3)
    raw, roffs = _raw(store, "f32", "var", starts, counts)
    nb = co.out_bytes(raw.numel(), case[5])
    whole, view = _dest(nb, 0)
    with pytest.raises(ValueError):
        store.get_batch("f32", starts, counts, out=view[:nb - 2].view(torch.bfloat16), src_dtype=torch.float32)
    assert (whole.cpu().numpy() == SENT).all(), "a capacity error wrote bytes"
    t = store.get_batch("f32", starts, counts, out=view.view(torch.bfloat16), src_dtype=torch.float32)
    _check(case, whole, 0, t, None, raw, roffs, "after the capacity error")


@pytest.mark.parametrize("contention", [False, True])
def test_overlapped_queues(env, contention):
    """converted only, and converted alternating with raw batches, DDS_NO_SYNC | DDS_OVERLAP, double-buffered; optionally
    with a kernel holding most SMs' shared memory on another stream"""
    from ddstore_b200 import _capi
    store, rng, L = env["store"], env["rng"], env["L"]
    side, other = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
    nb = 8
    for mode in ("converted", "alternating"):
        reqs = [rng.integers(0, NROWS - 4, 5000) for _ in range(nb)]
        sids = [rng.integers(0, NSAMP, 700) for _ in range(nb)]
        exp, bufs = [], []
        for k in range(nb):
            conv = mode == "converted" or k % 2 == 0
            if k % 3 == 2:  # a by-sample-id batch (variable counts, plan in shared memory)
                raw, _ = _raw_samples(store, "f32", sids[k], L)
            else:
                raw, _ = _raw(store, "f32", "fixed", reqs[k], count=4)
            exp.append(_torch_cast(raw, CASES[0]) if conv else raw)
            bufs.append(torch.zeros(exp[-1].numel() + 64, dtype=torch.uint8, device=DEV))
        d_req = [torch.from_numpy(r).to(DEV) for r in reqs]
        d_sid = [torch.from_numpy(s).to(DEV) for s in sids]
        torch.cuda.synchronize()
        if contention:
            _capi.raise_for(_capi.lib().dds_test_occupy(0, 100, 200 * 1024, 2_000_000, ctypes.c_void_p(other.cuda_stream)))
        for k in range(nb):
            conv = mode == "converted" or k % 2 == 0
            kw = dict(src_dtype=torch.float32) if conv else {}
            o = bufs[k].view(torch.bfloat16) if conv else bufs[k]
            if k % 3 == 2:
                store.get_samples("f32", d_sid[k], o, stream=side.cuda_stream, wait=False, overlap=True, **kw)
            else:
                store.get_batch("f32", d_req[k], out=o, count=4, stream=side.cuda_stream, wait=False, overlap=True, **kw)
        store.wait()
        torch.cuda.synchronize()
        for k in range(nb):
            assert torch.equal(bufs[k][:exp[k].numel()], exp[k]), f"{mode} contention={contention}: batch {k}"


def test_wait_total_after_a_converting_multi_array_batch_in_an_overlapped_queue():
    """regression: wait() reports the total of the LAST queued batch. A converting multi-array batch writes its total
    at the end of its walk, a batch planned in shared memory at its start; while an overlapped run shared one total
    word, the multi-array batch, still running, overwrote the total of the small batch queued behind it"""
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    try:
        rows, disp = 8192, 1024
        for nm in ("a", "b"):
            store.init(nm, rows, disp, 4)
            store.synth_fill(nm, 3)
            store.set_sample_index(nm, np.arange(0, rows, 8, dtype=np.int64), np.full(rows // 8, 8, np.int64))
        rng = np.random.default_rng(5)
        ids = torch.from_numpy(rng.integers(0, rows // 8, 2000)).to(DEV)  # 4000 requests: the plan kernels
        starts = torch.from_numpy(rng.integers(0, rows, 100)).to(DEV)     # 100 requests: the shared-memory plan
        counts = torch.ones(100, dtype=torch.int64, device=DEV)
        big = [torch.empty(2000 * 8 * disp, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
        small = torch.empty(100 * disp, dtype=torch.bfloat16, device=DEV)
        side = torch.cuda.Stream(device=DEV)
        torch.cuda.synchronize()
        store.get_samples_multi(["a", "b"], ids, big, stream=side.cuda_stream, wait=False, overlap=True,
                                src_dtypes=[torch.float32, torch.float32])
        store.get_batch("a", starts, counts, out=small, stream=side.cuda_stream, wait=False, overlap=True,
                        src_dtype=torch.float32)
        assert store.wait() == small.numel() * 2
        torch.cuda.synchronize()
    finally:
        store.free()
        store.close()


def test_u8_to_f32_beyond_4gib(env):
    """a uint8 source below 4 GiB whose float32 output is above it: fixed count and explicit counts"""
    from ddstore_b200 import PyDDStore
    D, rows = 4096, 300_000
    src_bytes = 280_000 * D
    need = rows * D + 2 * src_bytes + 4 * src_bytes + (1 << 30)  # store + raw copy + output + slack (computed, not measured)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs ~{need / 1e9:.1f} GB of free HBM")
    store = PyDDStore(device=0)
    try:
        store.init("big", rows, D, 1)
        store.synth_fill("big", 5)
        table = (torch.arange(256, dtype=torch.float32) * 0.5 - 3).to(DEV)
        rng = np.random.default_rng(2)
        starts = rng.integers(0, rows, 280_000)
        raw = torch.empty(src_bytes, dtype=torch.uint8, device=DEV)
        out = torch.empty(src_bytes, dtype=torch.float32, device=DEV)
        for kind in ("fixed", "var"):
            if kind == "fixed":
                d = torch.from_numpy(starts).to(DEV)
                store.get_batch("big", d, out=raw, count=1)
                t = store.get_batch("big", d, out=out, count=1, src_dtype=torch.uint8, lut=table)
            else:  # 700 requests of 400 rows: few enough for the shared-memory plan (its source offsets are < 4 GiB)
                s = (np.arange(700) * 400).astype(np.int64)
                c = np.full(700, 400, np.int64)
                store.get_batch("big", s, c, out=raw)
                offs = torch.empty(701, dtype=torch.int64, device=DEV)
                t = store.get_batch("big", s, c, out=out, offsets=offs, src_dtype=torch.uint8, lut=table)
                assert offs[-1].item() == 4 * src_bytes and offs[350].item() == 350 * 400 * D * 4
            assert t == 4 * src_bytes > (1 << 32)
            for c0 in range(0, src_bytes, 1 << 28):  # chunked comparison on the device
                c1 = min(src_bytes, c0 + (1 << 28))
                assert torch.equal(out[c0:c1].view(torch.int32), table[raw[c0:c1].long()].view(torch.int32)), (kind, c0)
    finally:
        store.free()
        store.close()


def _multi_owner_world(P, devices=None):
    from tests.gpu_helpers import run_world
    per, disp = 5000, 24

    def body(store, r):
        DEV = torch.device("cuda", devices[r] if devices else 0)
        rng = np.random.default_rng(r)
        shard = rng.integers(0, 2 ** 32, size=(per + 100 * r, disp), dtype=np.uint32).view(np.float32)
        store.add("w", shard)
        total = store.query("w")["total_nrows"]
        starts = np.random.default_rng(7).integers(0, total - 2, 4000)
        starts[:3] = [per - 2, per, total - 2]  # the last rows of owner 0, the first of owner 1, the last overall
        starts = starts[~np.isin(starts + 1, store.query("w")["lenlist"])]  # (no request straddles two owners)
        n = len(starts)
        raw = torch.empty(n * 2 * disp, dtype=torch.float32, device=DEV)
        store.get_batch("w", starts, out=raw, count=2)
        o = torch.empty(n * 2 * disp, dtype=torch.float16, device=DEV)
        store.get_batch("w", torch.from_numpy(starts).to(DEV), out=o, count=2, src_dtype=torch.float32)
        assert torch.equal(o.view(torch.int16), raw.to(torch.float16).view(torch.int16)), f"rank {r}"
        return True

    assert all(run_world(P, body, devices=devices))


def test_multi_owner_world():
    _multi_owner_world(3)


def test_multi_owner_world_peer_devices():
    """every rank on its own GPU: converting batches read the other owners' HBM through the peer mappings"""
    P = min(3, torch.cuda.device_count())
    if P < 2:
        pytest.skip("needs two or more GPUs")
    _multi_owner_world(P, devices=list(range(P)))


def test_loaders(env):
    from ddstore_b200.dataset import DistDataset, PrefetchLoader, RaggedDataset, RaggedPrefetchLoader
    rng = np.random.default_rng(3)
    data = [(rng.integers(0, 2 ** 32, 48, dtype=np.uint32).view(np.float32).reshape(6, 8), i % 7) for i in range(500)]
    raw_ds = DistDataset(data, "raw")
    cv_ds = DistDataset(data, "cv", out_dtype=torch.bfloat16)
    idx = list(rng.integers(0, 500, 64))
    (rv, rl), (cv, cl) = raw_ds.__getitems__(idx), cv_ds.__getitems__(idx)
    assert cv.dtype == torch.bfloat16 and torch.equal(rl, cl)
    assert torch.equal(cv.view(torch.int16), rv.to(torch.bfloat16).view(torch.int16))
    order = list(rng.permutation(500))
    for (a, la), (b, lb) in zip(PrefetchLoader(raw_ds, order, 64), PrefetchLoader(cv_ds, order, 64)):
        assert torch.equal(b.view(torch.int16), a.to(torch.bfloat16).view(torch.int16)) and torch.equal(la, lb)
    imgs = [(rng.integers(0, 256, 12, dtype=np.uint8), 0) for _ in range(300)]
    # (the table is built by the expression it replaces, on the device that expression runs on: bit-exact with it)
    u8 = DistDataset(imgs, "img", out_dtype=torch.float32, lut=torch.arange(256, dtype=torch.uint8, device=DEV).float() / 255)
    u8raw = DistDataset(imgs, "imgraw")
    a, _ = u8raw.__getitems__([i % 300 for i in idx])
    b, _ = u8.__getitems__([i % 300 for i in idx])
    assert torch.equal(b, a.float() / 255)
    for ds in (raw_ds, cv_ds, u8, u8raw):
        ds.free()
    # ragged: node features converted, edge index raw
    n = 400
    cnt = rng.integers(1, 20, n).astype(np.int64)
    ecnt = 2 * cnt
    feats = rng.integers(0, 2 ** 32, (int(cnt.sum()), 5), dtype=np.uint32).view(np.float32)
    edges = rng.integers(0, 1000, (int(ecnt.sum()), 2)).astype(np.int64)
    rr = RaggedDataset({"x": feats, "e": edges}, {"x": cnt, "e": ecnt})
    rc = RaggedDataset({"x": feats, "e": edges}, {"x": cnt, "e": ecnt}, out_dtypes={"x": torch.float16})
    ids = list(rng.integers(0, n, 50))
    A, Bc = rr.__getitems__(ids), rc.__getitems__(ids)
    assert torch.equal(Bc["x"][0].view(torch.int16), A["x"][0].to(torch.float16).view(torch.int16))
    assert torch.equal(Bc["x"][1], A["x"][1]) and torch.equal(Bc["e"][0], A["e"][0]) and torch.equal(Bc["e"][1], A["e"][1])
    order = list(rng.permutation(n))
    for ba, bb in zip(RaggedPrefetchLoader(rr, order, 32), RaggedPrefetchLoader(rc, order, 32)):
        assert torch.equal(bb["x"][0].view(torch.int16), ba["x"][0].to(torch.float16).view(torch.int16))
        assert torch.equal(bb["x"][1], ba["x"][1]) and torch.equal(bb["e"][0], ba["e"][0])
    rr.free()
    rc.free()


def test_plan_in_shared_memory_up_to_8192_requests():
    """DDS_SMEM_PLAN_MAX=8192 puts 4097..8192-request batches on the 8192-request shared-memory plan (set before the
    library reads it: a subprocess)"""
    env = dict(os.environ, DDS_SMEM_PLAN_MAX="8192")
    code = ("import sys; sys.path.insert(0, %r); import pytest; "
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', 'explicit_counts or samples or multi']))"
            % (ROOT, os.path.join(ROOT, "tests", "test_gpu_convert.py")))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_cython_binding(case):
    """pyddstore.PyDDStore.get_batch converting without padding: fixed and explicit counts, host and device indices,
    with offsets"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    _, var, sdt, odt, lut, code = case
    dt, disp = VARS[var]
    rng = np.random.default_rng(CASE_IDS.index(case[0]))
    nrows, n = 500, 300
    if dt is np.uint8:
        rows = rng.integers(0, 256, (nrows, disp)).astype(dt)
    else:
        rows = (rng.standard_normal((nrows, disp)) * np.exp2(rng.integers(-20, 20, (nrows, disp)))).astype(dt)
    row = disp * np.dtype(dt).itemsize
    starts = rng.integers(0, nrows - 3, n).astype(np.int64)
    store = pyd.PyDDStore(None, device=0)
    try:
        store.add(var, rows)
        for counts in (None, rng.integers(0, 4, n).astype(np.int64)):
            c = np.full(n, 3) if counts is None else counts
            packed = np.concatenate([rows[a:a + k].reshape(-1) for a, k in zip(starts, c)])
            raw = torch.from_numpy(packed.view(np.uint8).copy()).to(DEV)
            raw_offs = np.concatenate([[0], np.cumsum(c * row)])
            nb = co.out_bytes(raw.numel(), code)
            for dev in (False, True):
                whole, view = _dest(nb, 0)
                offs = torch.full((n + 1,), -7, dtype=torch.int64, device=DEV)
                t = store.get_batch(var, _idx(starts, dev), None if counts is None else _idx(counts, dev),
                                    out=view.view(odt), count=3 if counts is None else None, offsets=offs,
                                    src_dtype=sdt, lut=lut)
                _check(case, whole, 0, t, offs.cpu().numpy(), raw, raw_offs,
                       f"cython {case[0]} counts={counts is not None} dev={dev}")
    finally:
        store.free()
