"""Normalising batches on the GPU (the DDS_CVT_NORM_* codes through dds_get_batch_convert, dds_get_samples_convert,
dds_get_samples_multi_convert, and the loaders built on them).

Every batch is checked four ways: bitwise against torch's CUDA expression ((x.to(float32) - mean_t) / std_t).to(dtype)
applied to the raw gather of the same requests, with mean_t / std_t CUDA float32 tensors laid out by the channel rule;
against the NumPy oracle of tests/norm_oracle.py (NaN by class); its offsets and total against the plain conversion
with the same itemsizes; and the sentinel guard bands around the destination untouched. Layouts (nchan, inner): a
scalar (1, 1), channels-last (3, 1), CHW (3, 1024), per feature with odd rows of 37 and 1025 elements, and (2, 3) in
rows of 12. The tables of the 37-feature variable hold std = 0, negative and subnormal std, infinite and NaN means.

Entries: fixed counts at every destination base offset the output itemsize allows, explicit counts at <= 4096,
4097..8192 and > 8192 requests, get_samples, multi-array batches mixing normalised, plainly converted and raw variables
(a normalised one starting at an odd offset behind a uint8 variable), rows longer than a staged chunk and requests of a
few MiB; host and device indices. Then the first-invalid-request contract, a capacity one element short, overlapped
queues mixing normalised, plain and raw batches with their wait() totals (once under SM contention), re-registration
between batches, every registration and argument error, a three-owner world and the loaders. Subprocesses repeat the
batch tests with DDS_SMEM_PLAN_MAX=8192, with 1-chunk segments and with programmatic dependent launch off.

On an H100 80GB HBM3 (700 W power limit) the module takes about 195 s, 140 s of it in the three subprocesses.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import norm_oracle as no
from tests.gpu_helpers import GUARD, guarded_buffer

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENT = 0x5A
DEV = torch.device("cuda", 0)
NROWS, NSAMP = 12_000, 5_000

# variable -> (numpy dtype, disp, nchan, inner)
VARS = {"pf37": (np.float32, 37, 37, 1), "pf1025": (np.float32, 1025, 1025, 1), "div12": (np.float32, 12, 2, 3),
        "f64": (np.float64, 29, 1, 1), "hwc": (np.uint8, 51, 3, 1), "chw": (np.uint8, 3072, 3, 1024)}
_U8_LUT = torch.arange(256, dtype=torch.float32).div(255)  # ToTensor()'s scaling, as a decode table
# (name, variable, source dtype, output dtype, decode table, code)
CASES = [("f32_f32_pf37", "pf37", torch.float32, torch.float32, None, no.CVT_NORM_F32_F32),
         ("f32_bf16_pf1025", "pf1025", torch.float32, torch.bfloat16, None, no.CVT_NORM_F32_BF16),
         ("f32_f16_div12", "div12", torch.float32, torch.float16, None, no.CVT_NORM_F32_F16),
         ("f64_f32_scalar", "f64", torch.float64, torch.float32, None, no.CVT_NORM_F64_F32),
         ("u8_f32_hwc", "hwc", torch.uint8, torch.float32, _U8_LUT, no.CVT_NORM_U8_F32),
         ("u8_bf16_chw", "chw", torch.uint8, torch.bfloat16, _U8_LUT, no.CVT_NORM_U8_BF16),
         ("u8_f16_hwc_default", "hwc", torch.uint8, torch.float16, None, no.CVT_NORM_U8_F16)]
CASE_IDS = [c[0] for c in CASES]


def _tables(var, seed=0):
    _, _, nchan, _ = VARS[var]
    if var == "pf37":  # the arithmetic's edges: std = 0, negative / subnormal std, infinite and NaN means
        return np.resize(no.TABLE_EDGE_MEAN, nchan), np.resize(no.TABLE_EDGE_STD, nchan)
    rng = np.random.default_rng(len(var) + seed)
    mean = rng.standard_normal(nchan).astype(np.float32) * 0.5
    std = (rng.random(nchan).astype(np.float32) + 0.1) * 0.3
    return mean, std


@pytest.fixture(scope="module")
def env():
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    rng = np.random.default_rng(17)
    L = rng.integers(0, 5, NSAMP)
    L[::89] = 0
    sstart = np.concatenate([[0], np.cumsum(L)])
    assert sstart[-1] <= NROWS
    tabs = {}
    for name, (dt, disp, nchan, inner) in VARS.items():
        store.init(name, NROWS, disp, np.dtype(dt).itemsize)
        store.synth_fill(name, 7)
        store.set_sample_index(name, sstart[:-1].copy(), L)
        tabs[name] = _tables(name)
        m, s = tabs[name]
        # host tables for some variables, CUDA tensors for the others
        if dt == np.uint8:
            m, s = torch.from_numpy(m).to(DEV), torch.from_numpy(s).to(DEV)
        store.set_normalization(name, m, s, inner)
    yield {"store": store, "L": L, "rng": rng, "tabs": tabs}
    store.free()
    store.close()


def _row(var):
    dt, disp = VARS[var][:2]
    return disp * np.dtype(dt).itemsize


def _raw(store, var, kind, a, b=None, count=None, ids_L=None):
    """the raw gather of the same requests: (bytes as a uint8 CUDA tensor, offsets)"""
    n = len(a)
    if kind == "fixed":
        nb = n * count * _row(var)
    elif kind == "var":
        nb = int(np.clip(b, 0, None).sum()) * _row(var)
    else:
        nb = int(ids_L[a].sum()) * _row(var)
    buf = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    offs = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    if kind == "fixed":
        t = store.get_batch(var, a, out=buf, count=count, offsets=offs)
    elif kind == "var":
        t = store.get_batch(var, a, b, out=buf, offsets=offs)
    else:
        t = store.get_samples(var, a, buf, offsets=offs)
    return buf[:t], offs.cpu().numpy()


def _decode_table(case):
    return (torch.arange(256, dtype=torch.float32) if case[4] is None else case[4]).to(DEV)


def _torch_ref(raw_u8, case, tabs):
    """torch's CUDA expression on the raw gather: mean / std as CUDA float32 tensors laid out per row by the channel
    rule (division by a CUDA tensor, never by a scalar)"""
    _, var, sdt, odt, _, code = case
    _, disp, nchan, inner = VARS[var]
    ch = torch.from_numpy(no.channels(disp, nchan, inner)).to(DEV)
    m = torch.from_numpy(tabs[var][0]).to(DEV)[ch]
    s = torch.from_numpy(tabs[var][1]).to(DEV)[ch]
    x = _decode_table(case)[raw_u8.long()] if sdt == torch.uint8 else raw_u8.view(sdt).to(torch.float32)
    return ((x.view(-1, disp) - m) / s).to(odt).view(torch.uint8).reshape(-1)


# the plain conversion (or raw gather) with the same itemsizes: its offsets and totals are the normalised batch's
_PLAIN = {no.CVT_NORM_F32_BF16: (torch.float32, torch.bfloat16), no.CVT_NORM_F32_F16: (torch.float32, torch.float16),
          no.CVT_NORM_F64_F32: (torch.float64, torch.float32), no.CVT_NORM_U8_F32: (torch.uint8, torch.float32),
          no.CVT_NORM_U8_BF16: (torch.uint8, torch.bfloat16), no.CVT_NORM_U8_F16: (torch.uint8, torch.float16)}


def _check(case, tabs, whole, off, got_total, got_offs, raw_u8, raw_offs, what):
    code = case[5]
    exp_dev = _torch_ref(raw_u8, case, tabs)
    nb = exp_dev.numel()
    assert got_total == nb, f"{what}: total {got_total} != {nb}"
    body = whole[GUARD + off:GUARD + off + nb]
    if not torch.equal(body, exp_dev):
        bad = torch.nonzero(body != exp_dev)[:4].flatten().tolist()
        raise AssertionError(f"{what}: bytes differ from torch's CUDA expression at {bad}")
    h = whole.cpu().numpy()
    assert (h[:GUARD + off] == SENT).all() and (h[GUARD + off + nb:] == SENT).all(), f"{what}: guard band written"
    _, var, _, _, _, _ = case
    exp_np = no.norm_bytes(raw_u8.cpu().numpy(), code, tabs[var][0], tabs[var][1], VARS[var][2], VARS[var][3],
                           _decode_table(case).cpu().numpy())
    bad = no.bad_elements(h[GUARD + off:GUARD + off + nb], exp_np, code)
    assert bad.size == 0, f"{what}: {bad.size} elements differ from the NumPy oracle, first {bad[0]}"
    if got_offs is not None:
        assert got_offs.tolist() == [no.out_bytes(int(x), code) for x in raw_offs], f"{what}: offsets"


def _offsets_for(case, every=False):
    o = no.NORM[case[5]][1]
    return list(range(0, 16, o)) if every else [x for x in (0, 4, 12) if x % o == 0]


def _dest(nb, off):
    return guarded_buffer(torch, nb, off, SENT, device=DEV)


def _idx(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if dev else a


def _requests(rng, n, max_count):
    starts = rng.integers(0, NROWS - max_count, n).astype(np.int64)
    counts = rng.integers(0, max_count + 1, n).astype(np.int64)
    return starts, counts


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_fixed_count(env, case):
    store, rng, tabs = env["store"], env["rng"], env["tabs"]
    var, sdt, odt, lut = case[1:5]
    starts = rng.integers(0, NROWS - 3, 1500)
    raw, roffs = _raw(store, var, "fixed", starts, count=3)
    nb = no.out_bytes(raw.numel(), case[5])
    for dev in (False, True):
        for off in _offsets_for(case, every=dev):
            whole, view = _dest(nb, off)
            offs = torch.full((len(starts) + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_batch(var, _idx(starts, dev), out=view.view(odt), count=3, offsets=offs, src_dtype=sdt, lut=lut,
                                normalize=True)
            _check(case, tabs, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} fixed dev={dev} off={off}")


@pytest.mark.parametrize("nreq", [700, 5000, 9000])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_explicit_counts(env, case, nreq):
    store, rng, tabs = env["store"], env["rng"], env["tabs"]
    var, sdt, odt, lut, code = case[1:6]
    starts, counts = _requests(rng, nreq, 5)
    raw, roffs = _raw(store, var, "var", starts, counts)
    nb = no.out_bytes(raw.numel(), code)
    for dev in (False, True):
        off = _offsets_for(case)[1 if dev else 0]
        whole, view = _dest(nb, off)
        offs = torch.full((nreq + 1,), -7, dtype=torch.int64, device=DEV)
        t = store.get_batch(var, _idx(starts, dev), _idx(counts, dev), out=view.view(odt), offsets=offs, src_dtype=sdt,
                            lut=lut, normalize=True)
        _check(case, tabs, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} var n={nreq} dev={dev} off={off}")
    # offsets and total of the plain conversion with the same itemsizes (or of the raw gather: f32 -> f32)
    pl = torch.empty(nb + 16, dtype=torch.uint8, device=DEV)
    poffs = torch.empty(nreq + 1, dtype=torch.int64, device=DEV)
    if code in _PLAIN:
        psrc, pout = _PLAIN[code]
        tp = store.get_batch(var, starts, counts, out=pl[:nb].view(pout), offsets=poffs, src_dtype=psrc)
    else:
        tp = store.get_batch(var, starts, counts, out=pl[:nb], offsets=poffs)
    assert tp == t and torch.equal(poffs, offs), f"{case[0]}: offsets / total differ from the plain conversion's"


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_samples(env, case):
    store, rng, L, tabs = env["store"], env["rng"], env["L"], env["tabs"]
    var, sdt, odt, lut = case[1:5]
    for n in (900, 9000):
        ids = rng.integers(0, NSAMP, n)
        raw, roffs = _raw(store, var, "samples", ids, ids_L=L)
        nb = no.out_bytes(raw.numel(), case[5])
        for dev in (False, True):
            off = _offsets_for(case)[-1]
            whole, view = _dest(nb, off)
            offs = torch.full((n + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_samples(var, _idx(ids, dev), view.view(odt), offsets=offs, src_dtype=sdt, lut=lut, normalize=True)
            _check(case, tabs, whole, off, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} samples n={n} dev={dev}")


@pytest.mark.parametrize("case", [CASES[1], CASES[5]], ids=[CASE_IDS[1], CASE_IDS[5]])
def test_long_rows_and_large_requests(env, case):
    """rows longer than a staged chunk (4100 and 3072 bytes) and requests up to a few MiB: a row spans pieces, a request
    spans segments"""
    store, rng, tabs = env["store"], env["rng"], env["tabs"]
    var, sdt, odt, lut, code = case[1:6]
    counts = np.array([1, 1000, 0, 700, 1, 2, 513, 257, 3, 999], np.int64)
    starts = rng.integers(0, NROWS - 1000, counts.size).astype(np.int64)
    raw, roffs = _raw(store, var, "var", starts, counts)
    assert raw.numel() > (2 << 20)
    nb = no.out_bytes(raw.numel(), code)
    for dev in (False, True):
        whole, view = _dest(nb, 2)
        offs = torch.full((counts.size + 1,), -7, dtype=torch.int64, device=DEV)
        t = store.get_batch(var, _idx(starts, dev), _idx(counts, dev), out=view.view(odt), offsets=offs, src_dtype=sdt,
                            lut=lut, normalize=True)
        _check(case, tabs, whole, 2, t, offs.cpu().numpy(), raw, roffs, f"{case[0]} long dev={dev}")
    whole, view = _dest(no.out_bytes(3 * 600 * _row(var), code), 0)  # fixed count of 600 rows a request
    st3 = starts[:3] % (NROWS - 600)
    raw3, roffs3 = _raw(store, var, "fixed", st3, count=600)
    t = store.get_batch(var, st3, out=view.view(odt), count=600, src_dtype=sdt, lut=lut, normalize=True)
    _check(case, tabs, whole, 0, t, None, raw3, roffs3, f"{case[0]} long fixed")


@pytest.mark.parametrize("n", [300, 3000])
def test_multi_mixed(env, n):
    """normalised, plainly converted and raw variables in one launch; a normalised variable behind an odd-sized uint8
    variable starts at an odd offset of the concatenated walk"""
    store, rng, L, tabs = env["store"], env["rng"], env["L"], env["tabs"]
    plain_bf16 = ("plain", "pf37", torch.float32, torch.bfloat16, None, 1)
    combos = [[("hwc", None), ("pf37", CASES[0]), ("f64", CASES[3])],
              [("hwc", CASES[6]), ("div12", CASES[2]), ("pf37", plain_bf16), ("chw", CASES[5])],
              [("chw", None), ("pf1025", CASES[1])],
              [("f64", None), ("hwc", CASES[4]), ("div12", None)]]
    for pairs in combos:
        names, combo = [p[0] for p in pairs], [p[1] for p in pairs]
        for dev in (False, True):
            ids = rng.integers(0, NSAMP, n)
            ids[0] = NSAMP - 1
            if L[ids].sum() % 2 == 0:  # an odd number of rows: variable 1 starts at an odd offset behind 51-byte rows
                ids[1] = np.flatnonzero(L % 2 != L[ids[1]] % 2)[0]
            assert L[ids].sum() % 2 == 1
            raws = [_raw(store, nm, "samples", ids, ids_L=L) for nm in names]
            wholes, outs, offs = [], [], []
            for c, (raw, _) in zip(combo, raws):
                nb = raw.numel() if c is None else (raw.numel() // 4 * 2 if c[0] == "plain" else no.out_bytes(raw.numel(), c[5]))
                whole, view = _dest(nb, 4)
                wholes.append(whole)
                outs.append(view if c is None else view.view(c[3]))
                offs.append(torch.full((n + 1,), -7, dtype=torch.int64, device=DEV))
            tots = store.get_samples_multi(names, _idx(ids, dev), outs, offsets=offs,
                                           src_dtypes=[c[2] if c else None for c in combo],
                                           luts=[c[4] if c else None for c in combo],
                                           normalize=[c is not None and c[0] != "plain" for c in combo])
            for c, nm, (raw, roffs), whole, of, t in zip(combo, names, raws, wholes, offs, tots):
                what = f"multi {names} var {nm} dev={dev}"
                if c is None:
                    assert t == raw.numel() and torch.equal(whole[GUARD + 4:GUARD + 4 + t], raw), what
                    assert of.cpu().numpy().tolist() == roffs.tolist(), what
                elif c[0] == "plain":
                    exp = raw.view(torch.float32).to(torch.bfloat16).view(torch.uint8)
                    assert t == exp.numel() and torch.equal(whole[GUARD + 4:GUARD + 4 + t], exp), what
                else:
                    _check(c, tabs, whole, 4, t, of.cpu().numpy(), raw, roffs, what)


@pytest.mark.parametrize("entry", ["fixed", "var", "samples", "multi"])
def test_first_invalid_request(env, entry):
    """the first invalid request raises with its index; the requests before it are delivered normalised; later bytes are
    sentinel or the normalised value of a valid request at its offset; capacity one element short writes nothing"""
    store, rng, L, tabs = env["store"], env["rng"], env["L"], env["tabs"]
    case = CASES[1]
    var = case[1]
    n = 1500
    for bad_at in (0, 31, 1023, n - 1):
        starts, counts = _requests(rng, n, 2)
        counts[counts == 0] = 1
        ids = rng.integers(0, NSAMP, n)
        if entry == "fixed":
            counts[:] = 2
        good_s, good_c, good_i = starts.copy(), counts.copy(), ids.copy()
        if entry in ("samples", "multi"):
            ids[bad_at] = NSAMP + 5
            good_i[bad_at] = 0  # (sample 0 owns no rows)
        else:
            starts[bad_at] = NROWS + 3
            if entry == "var":
                good_c[bad_at] = 0
        if entry == "fixed":
            raw, roffs = _raw(store, var, "fixed", good_s, count=2)
        elif entry == "var":
            raw, roffs = _raw(store, var, "var", good_s, good_c)
        else:
            raw, roffs = _raw(store, var, "samples", good_i, ids_L=L)
        exp = _torch_ref(raw, case, tabs).cpu().numpy()
        eoffs = [no.out_bytes(int(x), case[5]) for x in roffs]
        cap = len(exp) + 64
        whole, view = _dest(cap, 0)
        with pytest.raises(ValueError) as ei:
            kw = dict(src_dtype=torch.float32, normalize=True)
            if entry == "fixed":
                store.get_batch(var, starts, out=view.view(torch.bfloat16), count=2, **kw)
            elif entry == "var":
                store.get_batch(var, starts, counts, out=view.view(torch.bfloat16), **kw)
            elif entry == "samples":
                store.get_samples(var, ids, view.view(torch.bfloat16), **kw)
            else:
                spare = torch.empty(int(L[good_i].sum()) * VARS["hwc"][1] + 64, dtype=torch.uint8, device=DEV)
                store.get_samples_multi([var, "hwc"], ids, [view.view(torch.bfloat16), spare],
                                        src_dtypes=[torch.float32, None], normalize=[True, False])
        assert store.last_bad_index == bad_at, (entry, store.last_bad_index)
        assert "nvalid" in str(ei.value) or "sample" in str(ei.value)
        h = whole.cpu().numpy()[GUARD:GUARD + cap]
        p = eoffs[bad_at]
        assert np.array_equal(h[:p], exp[:p]), f"{entry}: prefix before request {bad_at}"
        rest = h[p:len(exp)]
        assert ((rest == SENT) | (rest == exp[p:])).all(), f"{entry}: a byte past the prefix is neither untouched nor ours"
        assert (whole.cpu().numpy()[GUARD + len(exp):] == SENT).all()
    # capacity one element short: nothing written; the next valid call on the same destination works
    starts, counts = _requests(rng, 600, 3)
    raw, roffs = _raw(store, var, "var", starts, counts)
    nb = no.out_bytes(raw.numel(), case[5])
    whole, view = _dest(nb, 0)
    with pytest.raises(ValueError):
        store.get_batch(var, starts, counts, out=view[:nb - 2].view(torch.bfloat16), src_dtype=torch.float32, normalize=True)
    assert (whole.cpu().numpy() == SENT).all(), "a capacity error wrote bytes"
    t = store.get_batch(var, starts, counts, out=view.view(torch.bfloat16), src_dtype=torch.float32, normalize=True)
    _check(case, tabs, whole, 0, t, None, raw, roffs, "after the capacity error")


@pytest.mark.parametrize("contention", [False, True])
def test_overlapped_queues(env, contention):
    """normalised, plainly converted and raw batches queued with DDS_NO_SYNC | DDS_OVERLAP, double-buffered; fixed
    counts, shared-memory plans and plan kernels; every wait() total is the last batch's output bytes"""
    from ddstore_b200 import _capi
    store, rng, L, tabs = env["store"], env["rng"], env["L"], env["tabs"]
    side, other = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
    case = CASES[1]
    var = case[1]
    nb = 9
    kinds = ["norm", "plain", "raw"]
    for run in range(2):
        reqs = [rng.integers(0, NROWS - 4, 900) for _ in range(nb)]
        sids = [rng.integers(0, NSAMP, 700 if k % 2 else 5000) for k in range(nb)]  # shared-memory plan / plan kernels
        exp, bufs, mode = [], [], []
        for k in range(nb):
            m = kinds[(k + run) % 3]
            mode.append(m)
            raw, _ = _raw(store, var, "samples", sids[k], ids_L=L) if k % 3 == 2 else _raw(store, var, "fixed", reqs[k],
                                                                                               count=2)
            exp.append(_torch_ref(raw, case, tabs) if m == "norm" else
                       raw.view(torch.float32).to(torch.bfloat16).view(torch.uint8) if m == "plain" else raw)
            bufs.append(torch.zeros(exp[-1].numel() + 64, dtype=torch.uint8, device=DEV))
        d_req = [torch.from_numpy(r).to(DEV) for r in reqs]
        d_sid = [torch.from_numpy(s).to(DEV) for s in sids]
        torch.cuda.synchronize()
        if contention:
            _capi.raise_for(_capi.lib().dds_test_occupy(0, 100, 200 * 1024, 2_000_000, ctypes.c_void_p(other.cuda_stream)))
        for k in range(nb):
            kw = {"norm": dict(src_dtype=torch.float32, normalize=True), "plain": dict(src_dtype=torch.float32),
                  "raw": {}}[mode[k]]
            o = bufs[k] if mode[k] == "raw" else bufs[k].view(torch.bfloat16)
            if k % 3 == 2:
                store.get_samples(var, d_sid[k], o, stream=side.cuda_stream, wait=False, overlap=True, **kw)
            else:
                store.get_batch(var, d_req[k], out=o, count=2, stream=side.cuda_stream, wait=False, overlap=True, **kw)
        assert store.wait() == exp[-1].numel(), f"run {run}: wait() total"
        torch.cuda.synchronize()
        for k in range(nb):
            assert torch.equal(bufs[k][:exp[k].numel()], exp[k]), f"run {run} contention={contention}: batch {k} ({mode[k]})"
    # a queue that ends on a normalised multi-array batch reports that batch's total (the sum over its variables)
    ids = torch.from_numpy(rng.integers(0, NSAMP, 3000)).to(DEV)
    outs = [torch.empty(int(L[ids.cpu().numpy()].sum()) * VARS[v][1] * 4 + 64, dtype=torch.float32, device=DEV)
            for v in ("hwc", "f64")]
    plain = torch.empty(len(reqs[0]) * 2 * VARS[var][1], dtype=torch.bfloat16, device=DEV)
    store.get_batch(var, d_req[0], out=plain, count=2, stream=side.cuda_stream, wait=False, overlap=True,
                    src_dtype=torch.float32)
    store.get_samples_multi(["hwc", "f64"], ids, outs, stream=side.cuda_stream, wait=False, overlap=True,
                            src_dtypes=[torch.uint8, torch.float64], luts=[_U8_LUT, None], normalize=[True, True])
    exp_total = int(L[ids.cpu().numpy()].sum()) * (VARS["hwc"][1] + VARS["f64"][1]) * 4
    assert store.wait() == exp_total


def test_reregistration_takes_effect_on_the_next_batch(env):
    store, rng, tabs = env["store"], env["rng"], env["tabs"]
    case = CASES[3]
    var = case[1]
    starts = rng.integers(0, NROWS - 2, 2000)
    raw, roffs = _raw(store, var, "fixed", starts, count=2)
    nb = no.out_bytes(raw.numel(), case[5])
    try:
        for k, (m, s) in enumerate([(np.array([3.0], np.float32), np.array([-0.5], np.float32)),
                                    (np.array([-1.0], np.float32), np.array([7.0], np.float32))]):
            store.set_normalization(var, torch.from_numpy(m).to(DEV) if k else m, torch.from_numpy(s).to(DEV) if k else s)
            t2 = dict(tabs, **{var: (m, s)})
            whole, view = _dest(nb, 0)
            t = store.get_batch(var, starts, out=view.view(torch.float32), count=2, src_dtype=torch.float64, normalize=True)
            _check(case, t2, whole, 0, t, None, raw, roffs, f"registration {k}")
        # removal: normalising batches are refused, plain ones are not
        store.set_normalization(var, np.zeros(0, np.float32), np.zeros(0, np.float32))
        out = torch.empty(nb // 4, dtype=torch.float32, device=DEV)
        with pytest.raises(ValueError, match="no normalization"):
            store.get_batch(var, starts, out=out, count=2, src_dtype=torch.float64, normalize=True)
        store.get_batch(var, starts, out=out, count=2, src_dtype=torch.float64)
    finally:
        store.set_normalization(var, *tabs[var], VARS[var][3])


def test_registration_and_argument_errors(env):
    from ddstore_b200 import _capi
    store = env["store"]
    L = _capi.lib()
    m = np.zeros(8, np.float32)
    for nchan, inner in ((3, 0), (-1, 1), (2, 7), (37, 2), (38, 1), (1, 38)):  # pf37: disp 37
        assert L.dds_set_normalization(store._h, b"pf37", m.ctypes.data, m.ctypes.data, nchan, inner, 0) == _capi.ERR_ARG
    assert L.dds_set_normalization(store._h, b"pf37", None, m.ctypes.data, 1, 1, 0) == _capi.ERR_ARG
    assert L.dds_set_normalization(store._h, b"pf37", m.ctypes.data, None, 1, 1, 0) == _capi.ERR_ARG
    assert L.dds_set_normalization(store._h, b"nope", m.ctypes.data, m.ctypes.data, 1, 1, 0) == _capi.ERR_UNKNOWN_VAR
    with pytest.raises(ValueError, match="divide"):
        store.set_normalization("div12", np.zeros(5, np.float32), np.ones(5, np.float32))
    with pytest.raises(ValueError):
        store.set_normalization("div12", np.zeros(2, np.float32), np.ones(3, np.float32))
    # the failed calls left the registered tables in place
    case = CASES[2]
    starts = np.arange(50, dtype=np.int64)
    raw, roffs = _raw(store, "div12", "fixed", starts, count=1)
    whole, view = _dest(no.out_bytes(raw.numel(), case[5]), 0)
    t = store.get_batch("div12", starts, out=view.view(torch.float16), count=1, src_dtype=torch.float32, normalize=True)
    _check(case, env["tabs"], whole, 0, t, None, raw, roffs, "after failed registrations")
    out = torch.empty(4096, dtype=torch.float32, device=DEV)
    with pytest.raises(ValueError, match="Invalid data type"):  # the variable's itemsize vs the code's source
        store.get_batch("f64", [1, 2], out=out, src_dtype=torch.float32, normalize=True)
    with pytest.raises(ValueError):  # host destination
        store.get_batch("pf37", [1, 2], out=np.zeros(200, np.float32), src_dtype=torch.float32, normalize=True)
    tot, bad = ctypes.c_int64(0), ctypes.c_int64(0)
    st = np.array([1], np.int64)
    for name, code, lut, dst, rc_exp in ((b"pf37", no.CVT_NORM_F32_F32, None, out.data_ptr() + 2, _capi.ERR_ARG),
                                         (b"chw", no.CVT_NORM_U8_BF16, None, out.data_ptr(), _capi.ERR_ARG),  # no table
                                         (b"chw", 13, None, out.data_ptr(), _capi.ERR_ARG),
                                         (b"pf37", no.CVT_NORM_U8_F32, None, out.data_ptr(), _capi.ERR_DTYPE)):
        cv = _capi.Convert(code, lut)
        rc = L.dds_get_batch_convert(store._h, name, st.ctypes.data, None, 1, 1, dst, 4000, None, _capi.DST_ON_DEVICE, None,
                                     ctypes.byref(cv), ctypes.byref(tot), ctypes.byref(bad))
        assert rc == rc_exp, (name, code)
    with pytest.raises(ValueError):  # the plain rules are unchanged: f32 -> f32 is no conversion
        store.get_batch("pf37", [1, 2], out=out, src_dtype=torch.float32)


def test_unregistered_variable(env):
    from ddstore_b200 import PyDDStore
    s2 = PyDDStore(device=0)
    try:
        s2.init("v", 100, 8, 4)
        s2.set_sample_index("v", np.arange(100, dtype=np.int64), np.ones(100, np.int64))
        out = torch.empty(800, dtype=torch.bfloat16, device=DEV)
        for call in (lambda: s2.get_batch("v", [1, 2], out=out, src_dtype=torch.float32, normalize=True),
                     lambda: s2.get_samples("v", [1, 2], out, src_dtype=torch.float32, normalize=True),
                     lambda: s2.get_samples_multi(["v"], [1, 2], [out], src_dtypes=[torch.float32], normalize=[True])):
            with pytest.raises(ValueError, match="variable has no normalization"):
                call()
    finally:
        s2.free()
        s2.close()


def test_multi_owner_world():
    """three owners; every rank registers its own tables (the call is local) and normalises what it fetches"""
    from tests.gpu_helpers import run_world
    per, disp = 3000, 24

    def body(store, r):
        rng = np.random.default_rng(r)
        store.add("w", rng.standard_normal((per + 50 * r, disp)).astype(np.float32))
        mean = np.arange(6, dtype=np.float32) * (r + 1)
        std = np.full(6, 0.5 + r, np.float32)
        store.set_normalization("w", mean, std, 2)  # (6 channels of 2 elements, twice a row)
        total = store.query("w")["total_nrows"]
        starts = np.random.default_rng(9).integers(0, total - 2, 3000)
        starts = starts[~np.isin(starts + 1, store.query("w")["lenlist"])]
        n = len(starts)
        raw = torch.empty(n * 2 * disp, dtype=torch.float32, device=DEV)
        store.get_batch("w", starts, out=raw, count=2)
        o = torch.empty(n * 2 * disp, dtype=torch.bfloat16, device=DEV)
        store.get_batch("w", torch.from_numpy(starts).to(DEV), out=o, count=2, src_dtype=torch.float32, normalize=True)
        ch = torch.from_numpy(no.channels(disp, 6, 2)).to(DEV)
        m, s = torch.from_numpy(mean).to(DEV)[ch], torch.from_numpy(std).to(DEV)[ch]
        exp = ((raw.view(-1, disp) - m) / s).to(torch.bfloat16).reshape(-1)
        assert torch.equal(o.view(torch.int16), exp.view(torch.int16)), f"rank {r}"
        return True

    assert all(run_world(3, body))


def test_loaders(env):
    from ddstore_b200.dataset import DistDataset, PrefetchLoader, RaggedDataset, RaggedPrefetchLoader
    rng = np.random.default_rng(4)
    # images: uint8 CHW 3 x 4 x 5, ToTensor() + Normalize(mean, std) in one gather
    C, H, W = 3, 4, 5
    imgs = [(rng.integers(0, 256, (C, H, W), dtype=np.uint8), i % 5) for i in range(400)]
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    lut = torch.arange(256, dtype=torch.float32, device=DEV).div(255)
    ds = DistDataset(imgs, "img", out_dtype=torch.bfloat16, lut=lut, normalize=(mean, std, H * W))
    raw = DistDataset(imgs, "imgraw")
    mt = torch.tensor(mean, dtype=torch.float32, device=DEV).view(1, C, 1, 1)
    st = torch.tensor(std, dtype=torch.float32, device=DEV).view(1, C, 1, 1)

    def ref(x):  # torchvision's ToTensor() then Normalize() on the batch, then the cast
        return ((x.float().div(255) - mt) / st).to(torch.bfloat16)

    idx = list(rng.integers(0, 400, 64))
    (a, la), (b, lb) = raw.__getitems__(idx), ds.__getitems__(idx)
    assert b.dtype == torch.bfloat16 and b.shape == (64, C, H, W) and torch.equal(la, lb)
    assert torch.equal(b.view(torch.int16), ref(a).view(torch.int16))
    order = list(rng.permutation(400))
    for (a, la), (b, lb) in zip(PrefetchLoader(raw, order, 50), PrefetchLoader(ds, order, 50)):
        assert torch.equal(b.view(torch.int16), ref(a).view(torch.int16)) and torch.equal(la, lb)
    # per-feature standardisation of float32 samples, output defaults to float32
    feats = [(rng.standard_normal(9).astype(np.float32), 0) for _ in range(300)]
    fm, fs = rng.standard_normal(9).astype(np.float32), rng.random(9).astype(np.float32) + 0.5
    fds = DistDataset(feats, "feat", normalize=(fm, fs))
    fraw = DistDataset(feats, "featraw")
    b, _ = fds.__getitems__([i % 300 for i in idx[:40]])
    a, _ = fraw.__getitems__([i % 300 for i in idx[:40]])
    assert b.dtype == torch.float32
    assert torch.equal(b, (a - torch.from_numpy(fm).to(DEV)) / torch.from_numpy(fs).to(DEV))
    for d in (ds, raw, fds, fraw):
        d.free()
    # ragged: node features normalised per feature into f16, edge index raw
    n = 300
    cnt = rng.integers(1, 15, n).astype(np.int64)
    ecnt = 2 * cnt
    x = rng.standard_normal((int(cnt.sum()), 5)).astype(np.float32)
    e = rng.integers(0, 1000, (int(ecnt.sum()), 2)).astype(np.int64)
    xm, xs = rng.standard_normal(5).astype(np.float32), rng.random(5).astype(np.float32) + 0.2
    rr = RaggedDataset({"x": x, "e": e}, {"x": cnt, "e": ecnt})
    rn = RaggedDataset({"x": x, "e": e}, {"x": cnt, "e": ecnt}, out_dtypes={"x": torch.float16}, normalize={"x": (xm, xs)})
    xm_t, xs_t = torch.from_numpy(xm).to(DEV), torch.from_numpy(xs).to(DEV)
    ids = list(rng.integers(0, n, 40))
    A, B = rr.__getitems__(ids), rn.__getitems__(ids)
    assert torch.equal(B["x"][0].view(torch.int16), ((A["x"][0] - xm_t) / xs_t).to(torch.float16).view(torch.int16))
    assert torch.equal(B["x"][1], A["x"][1]) and torch.equal(B["e"][0], A["e"][0])
    order = list(rng.permutation(n))
    for ba, bb in zip(RaggedPrefetchLoader(rr, order, 32), RaggedPrefetchLoader(rn, order, 32)):
        assert torch.equal(bb["x"][0].view(torch.int16), ((ba["x"][0] - xm_t) / xs_t).to(torch.float16).view(torch.int16))
        assert torch.equal(bb["x"][1], ba["x"][1]) and torch.equal(bb["e"][0], ba["e"][0])
    rr.free()
    rn.free()


@pytest.mark.parametrize("config", ["smem8192", "minseg1", "nopdl"])
def test_configurations(config):
    """the batch tests again with DDS_SMEM_PLAN_MAX=8192 (4097..8192 requests on the 8192-request shared-memory plan),
    with 1-chunk segments, and with programmatic dependent launch off (set before the library reads them: a subprocess)"""
    extra = {"smem8192": {"DDS_SMEM_PLAN_MAX": "8192"}, "minseg1": {"DDS_VAR_MINSEG": "1", "DDS_S_MINSEG": "1"},
             "nopdl": {"DDS_PDL": "0"}}[config]
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(extra)
    code = ("import sys; sys.path.insert(0, %r); import pytest; "
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', "
            "'explicit_counts or samples or multi_mixed or long_rows or overlapped']))"
            % (ROOT, os.path.join(ROOT, "tests", "test_gpu_normalize.py")))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_cython_binding(case):
    """pyddstore.PyDDStore.set_normalization (host and CUDA tables) and get_batch(normalize=True), fixed and explicit
    counts, host and device indices"""
    cydir = os.path.join(ROOT, "ddstore_b200", "cython")
    if cydir not in sys.path:
        sys.path.insert(0, cydir)
    pyd = pytest.importorskip("pyddstore", reason="Cython binding not built")
    _, var, sdt, odt, lut, code = case
    dt, disp, nchan, inner = VARS[var]
    rng = np.random.default_rng(CASE_IDS.index(case[0]))
    nrows, n = 300, 200
    if dt is np.uint8:
        rows = rng.integers(0, 256, (nrows, disp)).astype(dt)
    else:
        rows = (rng.standard_normal((nrows, disp)) * 4).astype(dt)
    mean, std = _tables(var)
    tabs = {var: (mean, std)}
    row = disp * np.dtype(dt).itemsize
    starts = rng.integers(0, nrows - 3, n).astype(np.int64)
    store = pyd.PyDDStore(None, device=0)
    try:
        store.add(var, rows)
        for counts, dev in ((None, False), (rng.integers(0, 4, n).astype(np.int64), True)):
            if dev:
                store.set_normalization(var, torch.from_numpy(mean).to(DEV), torch.from_numpy(std).to(DEV), inner)
            else:
                store.set_normalization(var, mean, std, inner)
            c = np.full(n, 3) if counts is None else counts
            packed = np.concatenate([rows[a:a + k].reshape(-1) for a, k in zip(starts, c)])
            raw = torch.from_numpy(packed.view(np.uint8).copy()).to(DEV)
            raw_offs = np.concatenate([[0], np.cumsum(c * row)])
            nb = no.out_bytes(raw.numel(), code)
            whole, view = _dest(nb, 0)
            offs = torch.full((n + 1,), -7, dtype=torch.int64, device=DEV)
            t = store.get_batch(var, _idx(starts, dev), None if counts is None else _idx(counts, dev),
                                out=view.view(odt), count=3 if counts is None else None, offsets=offs, src_dtype=sdt,
                                lut=lut, normalize=True)
            _check(case, tabs, whole, 0, t, offs.cpu().numpy(), raw, raw_offs,
                   f"cython {case[0]} counts={counts is not None} dev={dev}")
    finally:
        store.free()
