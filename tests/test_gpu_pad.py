"""Padded batches on the GPU (dds_get_batch_padded, dds_get_samples_padded).

Every padded batch is compared with the NumPy oracle of tests/pad_oracle.py applied to the raw packed gather of the
same valid requests (converted by torch's CUDA expression when the batch converts): the slots bit for bit, the lengths,
the returned total, and the sentinel guard bands around the destination. Covered: raw itemsizes 1/2/4/8 with row bytes
1, 3, 12, 37, 40 and 4097; max_rows 0, 1, below / at / above the lengths; zero-length requests; nreq 0, 1, 31-33,
1023-1025 and 65536; slots under 16 bytes, around the 4 KiB chunk and of several MiB; every destination base offset the
output itemsize allows; explicit counts and sample ids, host and device indices; a three-owner world; every DDS_CVT_*
code with pad bits that must come out verbatim; every kind of invalid request at window lanes 0, 31, 32 and at the end;
every argument error; overlapped queues mixing padded, packed and converting batches, also under SM contention; one
batch whose padded output passes 4 GiB; RaggedDataset(pad=...) and RaggedPrefetchLoader over two epochs; the Cython
binding; the wait() total after an empty batch queued behind a padded one, through every entry. A subprocess
repeats the batch and loader tests with DDS_PDL=0.

On an H100 80GB HBM3 (700 W power limit) the module takes about 30 s, the subprocess included.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import pad_oracle as po
from tests.gpu_helpers import GUARD, classify, run_world

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENT = 0xA5
DEV = torch.device("cuda", 0)
NROWS = 20_000
# variable -> (itemsize, disp, torch dtype of a raw padded output, numpy dtype of its bits)
VARS = {"b1": (1, 1, torch.uint8, np.uint8), "b3": (1, 3, torch.uint8, np.uint8), "b37": (1, 37, torch.uint8, np.uint8),
        "b4097": (1, 4097, torch.uint8, np.uint8), "h6": (2, 6, torch.float16, np.uint16),
        "f3": (4, 3, torch.int32, np.int32), "f80": (4, 80, torch.float32, np.uint32),
        "d5": (8, 5, torch.float64, np.uint64)}
NSAMP = 6000


@pytest.fixture(scope="module")
def env():
    from ddstore_b200 import PyDDStore
    store = PyDDStore(device=0)
    rng = np.random.default_rng(5)
    L = rng.integers(0, 7, NSAMP)
    L[::53] = 0
    sstart = np.concatenate([[0], np.cumsum(L)])
    for name, (isz, disp, _, _) in VARS.items():
        store.init(name, NROWS, disp, isz)
        store.synth_fill(name, 7)
        store.set_sample_index(name, sstart[:-1].copy(), L)
    yield {"store": store, "rng": rng, "L": L, "sstart": sstart}
    store.free()
    store.close()


def _guarded(nbytes, off):
    whole = torch.full((2 * GUARD + off + nbytes,), SENT, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    return whole, whole[GUARD + off:GUARD + off + nbytes]


def _raw_packed(store, var, starts, counts, valid):
    """the raw packed gather of the valid requests, as host bytes"""
    isz, disp = VARS[var][:2]
    n = int(np.asarray(counts)[valid].sum()) * isz * disp
    buf = torch.empty(max(n, 1), dtype=torch.uint8, device=DEV)
    if valid.any():
        store.get_batch(var, np.asarray(starts)[valid], np.asarray(counts)[valid], out=buf[:n])
    return buf[:n].cpu().numpy()


def _expect(store, var, starts, counts, max_rows, pad_bits, bits_dtype):
    q = store.query(var)
    codes = classify(q["lenlist"], starts, counts)
    valid = codes == 0
    packed = _raw_packed(store, var, starts, counts, valid).view(bits_dtype)
    slots, lengths = po.pad_rows(packed, np.where(valid, counts, 0), VARS[var][1], max_rows,
                                 np.array([pad_bits]).astype(np.uint64).astype(bits_dtype)[0], valid)
    bad = int(np.nonzero(~valid)[0][0]) if (~valid).any() else -1
    return slots, lengths, bad, (codes[bad] if bad >= 0 else 0)


def _run_padded(store, var, starts, counts, max_rows, pad_value, off=0, dev_idx=True, out_dtype=None, bits=None,
                by_sample=False, **kw):
    """one padded batch into a guarded buffer -> (host bytes of the slots, lengths, total, error or None, whole)"""
    isz, disp, tdt, _ = VARS[var]
    tdt = out_dtype or tdt
    el = torch.empty(0, dtype=tdt).element_size()
    n = len(starts)
    nbytes = n * max_rows * disp * el
    whole, view = _guarded(nbytes, off)
    out = view.view(tdt)
    lengths = torch.full((max(n, 1),), -5, dtype=torch.int64, device=DEV)
    err = None
    try:
        if by_sample:
            ids = torch.as_tensor(np.asarray(starts, np.int64), device=DEV) if dev_idx else np.asarray(starts, np.int64)
            total = store.get_samples(var, ids, out, pad_rows=max_rows, pad_value=pad_value, lengths=lengths[:n], **kw)
        else:
            s = np.asarray(starts, np.int64)
            c = np.asarray(counts, np.int64)
            if dev_idx:
                s, c = torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV)
            total = store.get_batch(var, s, c, out=out, pad_rows=max_rows, pad_value=pad_value, lengths=lengths[:n], **kw)
    except ValueError as e:
        err, total = e, None
    torch.cuda.synchronize()
    h = whole.cpu().numpy()
    assert (h[:GUARD + off] == SENT).all() and (h[GUARD + off + nbytes:] == SENT).all(), "guard band written"
    return h[GUARD + off:GUARD + off + nbytes], lengths[:n].cpu().numpy(), total, err, nbytes


def _check(store, var, starts, counts, max_rows, pad_value=0, off=0, dev_idx=True, by_sample=False, tab=None):
    isz, disp, tdt, bdt = VARS[var]
    from ddstore_b200.store import _pad_bits
    pbits = _pad_bits(pad_value, tdt)
    if by_sample:
        env_tab = tab  # (sample table: row starts, row counts)
        ids = np.asarray(starts, np.int64)
        ok = (ids >= 0) & (ids < NSAMP)
        s = np.where(ok, env_tab[0][np.clip(ids, 0, NSAMP - 1)], 0)
        c = np.where(ok, env_tab[1][np.clip(ids, 0, NSAMP - 1)], 0)
        slots, lengths, bad, code = _expect(store, var, s, c, max_rows, pbits, bdt)
        if (~ok).any():
            lengths[~ok] = 0
            slots[~ok] = np.array([pbits]).astype(np.uint64).astype(bdt)[0]
            first = int(np.nonzero(~ok)[0][0])
            if bad < 0 or first < bad:
                bad = first
    else:
        slots, lengths, bad, code = _expect(store, var, starts, counts, max_rows, pbits, bdt)
    got, glen, total, err, nbytes = _run_padded(store, var, starts, counts, max_rows, pad_value, off, dev_idx,
                                                by_sample=by_sample)
    what = f"{var} n={len(starts)} max_rows={max_rows} off={off} dev={dev_idx} by_sample={by_sample}"
    assert got.tobytes() == slots.tobytes(), what
    assert glen.tolist() == lengths.tolist(), what
    if bad >= 0:
        assert err is not None and store.last_bad_index == bad, (what, err, store.last_bad_index, bad)
    else:
        assert err is None and total == nbytes, (what, err, total)


def _t(v):
    """a one-element float32 CUDA tensor (a CPU scalar divisor would make torch multiply by its reciprocal)"""
    return torch.tensor([v], dtype=torch.float32, device=DEV)


def _requests(rng, n, max_count):
    counts = rng.integers(0, max_count + 1, n)
    if n > 2:
        counts[[0, n // 2]] = 0
    starts = rng.integers(0, NROWS - max_count - 1, n)
    return starts, counts


@pytest.mark.parametrize("var", list(VARS))
def test_shapes_raw(env, var):
    store, rng = env["store"], env["rng"]
    isz, disp = VARS[var][:2]
    mc = 6 if disp < 4000 else 3
    for n in (0, 1, 31, 32, 33, 1023, 1024, 1025):
        s, c = _requests(rng, n, mc)
        for mr in (0, 1, 3, mc, mc + 5):
            _check(store, var, s, c, mr, pad_value=3, dev_idx=(n % 2 == 0))
    s, c = _requests(rng, 65536 if disp < 100 else 2048, mc)
    _check(store, var, s, c, 4, pad_value=1)


@pytest.mark.parametrize("var", ["b3", "h6", "f3", "d5"])
def test_destination_offsets(env, var):
    store, rng = env["store"], env["rng"]
    isz = VARS[var][0]
    s, c = _requests(rng, 77, 6)
    for off in range(0, 16, isz):
        _check(store, var, s, c, 4, pad_value=2, off=off)


def test_slot_sizes(env):
    """slots under 16 bytes, around the 4 KiB chunk and of several MiB"""
    store, rng = env["store"], env["rng"]
    s, c = _requests(rng, 40, 5)
    _check(store, "b3", s, c, 2, pad_value=9)         # 6-byte slots
    for mr in (1023, 1024, 1025):                      # f3: 12-byte rows; b1: 1-byte rows around 4096
        s, c = _requests(rng, 33, 1100)
        _check(store, "b1", s, c, mr * 4, pad_value=7)
        _check(store, "f3", s, c, mr // 3, pad_value=-1)
    s = rng.integers(0, NROWS - 5000, 9)
    c = rng.integers(0, 5000, 9)
    _check(store, "f80", s, c, 3000 * 4, pad_value=0)  # 3.84 MB slots


def test_sample_ids(env):
    store, rng = env["store"], env["rng"]
    tab = (env["sstart"][:-1], env["L"])
    for n in (1, 33, 1025, 5000):
        ids = rng.integers(0, NSAMP, n)
        for var in ("b37", "f80", "d5"):
            for mr in (0, 2, 6):
                _check(store, var, ids, None, mr, pad_value=4, by_sample=True, dev_idx=(n != 33), tab=tab)
    ids = rng.integers(0, NSAMP, 64)
    for bad in (0, 31, 32, 63):
        x = ids.copy()
        x[bad] = NSAMP + 3 if bad % 2 else -1
        _check(store, "f80", x, None, 4, pad_value=4, by_sample=True, tab=tab)


def test_invalid_requests(env):
    """every kind of invalid request at lanes 0 / 31 / 32 / end: the packed entry's error and index; every valid slot
    delivered, invalid slots all padding with length 0"""
    store, rng = env["store"], env["rng"]
    kinds = [(-1, 1), (NROWS, 1), (NROWS - 2, 5), (3, -1), (3, (1 << 62)), (5, NROWS + 1)]
    for st, ct in kinds:
        for at in (0, 31, 32, 99):
            s, c = _requests(rng, 100, 5)
            s[at], c[at] = st, ct
            s[at + 1 if at < 99 else 1], c[at + 1 if at < 99 else 1] = -7, 2  # a second one behind it
            _check(store, "f3", s, c, 4, pad_value=-3)
            # the same code and index as the packed entry
            try:
                store.get_batch("f3", s, c, out=torch.empty(10**6, dtype=torch.uint8, device=DEV))
                raise AssertionError("packed batch did not raise")
            except ValueError as e:
                packed_err, packed_bad = str(e), store.last_bad_index
            try:
                store.get_batch("f3", s, c, out=torch.empty(100 * 4 * 3, dtype=torch.int32, device=DEV), pad_rows=4)
                raise AssertionError("padded batch did not raise")
            except ValueError as e:
                assert str(e) == packed_err and store.last_bad_index == packed_bad


def test_conversions(env):
    """every DDS_CVT_* code: bitwise torch's CUDA expression on the raw packed gather, padded by the oracle; pad bits
    verbatim (bf16 -inf, a NaN payload)"""
    store, rng = env["store"], env["rng"]
    mean = torch.linspace(-1, 1, 80)
    std = torch.linspace(0.5, 2, 80)
    store.set_normalization("f80", mean, std)
    store.set_normalization("d5", torch.tensor([0.25]), torch.tensor([3.0]))
    lut32 = torch.arange(256, dtype=torch.float32) / 255
    store.set_normalization("b37", torch.tensor([0.5]), torch.tensor([0.25]))
    nan_f32 = torch.tensor([0x7FC01234], dtype=torch.int32).view(torch.float32)
    nan_f16 = torch.tensor([0x7E55], dtype=torch.int16).view(torch.float16)
    cases = [  # var, src dtype, out dtype, normalize, lut, pad_value, torch expression of the raw rows
        ("f80", torch.float32, torch.bfloat16, False, None, float("-inf"), lambda x: x.to(torch.bfloat16)),
        ("f80", torch.float32, torch.float16, False, None, nan_f16, lambda x: x.to(torch.float16)),
        ("d5", torch.float64, torch.float32, False, None, nan_f32, lambda x: x.to(torch.float32)),
        ("b37", torch.uint8, torch.bfloat16, False, None, -1.0, lambda x: x.to(torch.bfloat16)),
        ("b37", torch.uint8, torch.float32, False, lut32, nan_f32, lambda x: lut32.to(DEV)[x.long()]),
        ("f80", torch.float32, torch.float32, True, None, nan_f32,
         lambda x: (x.view(-1, 80) - mean.to(DEV)) / std.to(DEV)),
        ("f80", torch.float32, torch.bfloat16, True, None, float("-inf"),
         lambda x: ((x.view(-1, 80) - mean.to(DEV)) / std.to(DEV)).to(torch.bfloat16)),
        ("f80", torch.float32, torch.float16, True, None, 0.0,
         lambda x: ((x.view(-1, 80) - mean.to(DEV)) / std.to(DEV)).to(torch.float16)),
        ("d5", torch.float64, torch.float32, True, None, 2.0, lambda x: (x.to(torch.float32) - _t(0.25)) / _t(3.0)),
        ("b37", torch.uint8, torch.float32, True, None, nan_f32, lambda x: (x.to(torch.float32) - _t(0.5)) / _t(0.25)),
        ("b37", torch.uint8, torch.bfloat16, True, None, float("-inf"),
         lambda x: ((x.to(torch.float32) - _t(0.5)) / _t(0.25)).to(torch.bfloat16)),
        ("b37", torch.uint8, torch.float16, True, lut32, 1.0,
         lambda x: ((lut32.to(DEV)[x.long()] - _t(0.5)) / _t(0.25)).to(torch.float16)),
    ]
    from ddstore_b200.store import _pad_bits
    for var, sdt, odt, nz, lut, pv, expr in cases:
        disp = VARS[var][1]
        for n, mr, off_el in ((1, 3, 0), (33, 4, 1), (1025, 6, 3)):
            s, c = _requests(rng, n, 6)
            if n == 33:
                s[5], c[5] = NROWS - 1, 4  # an invalid request: all padding
            codes = classify(store.query(var)["lenlist"], s, c)
            valid = codes == 0
            el = torch.empty(0, dtype=odt).element_size()
            raw_np = _raw_packed(store, var, s, c, valid)
            packed = torch.from_numpy(raw_np.copy()).to(DEV).view(sdt) if raw_np.size else torch.empty(0, dtype=sdt, device=DEV)
            conv = expr(packed).reshape(-1).contiguous()
            bits_np = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[el]
            conv_bits = conv.view({2: torch.int16, 4: torch.int32}[el]).cpu().numpy().view(bits_np)
            pbits = _pad_bits(pv, odt)
            slots, lengths = po.pad_rows(conv_bits, np.where(valid, c, 0), disp, mr,
                                         np.array([pbits]).astype(np.uint64).astype(bits_np)[0], valid)
            off = off_el * el
            nbytes = n * mr * disp * el
            whole, view = _guarded(nbytes, off)
            lens = torch.full((n,), -5, dtype=torch.int64, device=DEV)
            try:
                total = store.get_batch(var, s, c, out=view.view(odt), src_dtype=sdt, lut=lut, normalize=nz, pad_rows=mr,
                                        pad_value=pv, lengths=lens)
                assert valid.all() and total == nbytes
            except ValueError:
                assert not valid.all() and store.last_bad_index == int(np.nonzero(~valid)[0][0])
            h = whole.cpu().numpy()
            what = (var, sdt, odt, nz, n)
            assert (h[:GUARD + off] == SENT).all() and (h[GUARD + off + nbytes:] == SENT).all(), what
            assert h[GUARD + off:GUARD + off + nbytes].tobytes() == slots.tobytes(), what
            assert lens.cpu().numpy().tolist() == lengths.tolist(), what
    for v in ("f80", "d5", "b37"):
        store.set_normalization(v, np.zeros(0, np.float32), np.zeros(0, np.float32))


def test_int32_pad_id(env):
    """token ids: an int32 variable padded with -100"""
    store, rng = env["store"], env["rng"]
    s, c = _requests(rng, 500, 6)
    _check(store, "f3", s, c, 3, pad_value=-100)


def test_argument_errors(env):
    """each argument error: ValueError, destination, lengths and guards untouched"""
    import ctypes

    from ddstore_b200 import _capi
    store = env["store"]
    L, h = store._L, store._h
    n, mr, disp = 8, 4, 3
    s = torch.arange(n, dtype=torch.int64, device=DEV)
    c = torch.full((n,), 2, dtype=torch.int64, device=DEV)
    nbytes = n * mr * disp * 4
    whole, view = _guarded(nbytes + 16, 0)
    lens = torch.full((n + 1,), -5, dtype=torch.int64, device=DEV)
    before = whole.cpu().numpy().copy()
    t, b = ctypes.c_int64(0), ctypes.c_int64(0)

    def call(starts=s.data_ptr(), counts=c.data_ptr(), itemsize=4, max_rows=mr, dst=view.data_ptr(), cap=nbytes,
             flags=_capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE, lengths=lens.data_ptr(), nreq=n):
        pad = _capi.Pad(max_rows, 0x12345678, lengths)
        return L.dds_get_batch_padded(h, b"f3", starts, counts, nreq, itemsize, None, ctypes.byref(pad), dst, cap, flags,
                                      None, ctypes.byref(t), ctypes.byref(b))

    assert call(counts=None) == _capi.ERR_ARG
    assert call(flags=_capi.IDX_ON_DEVICE) == _capi.ERR_ARG            # host destination
    assert call(dst=view.data_ptr() + 2) == _capi.ERR_ARG              # not aligned to the itemsize
    assert call(lengths=lens.data_ptr() + 4) == _capi.ERR_ARG          # lengths not aligned to 8
    assert call(max_rows=-1) == _capi.ERR_ARG
    assert call(max_rows=1 << 60) == _capi.ERR_ARG                     # nreq * S overflows
    assert call(cap=nbytes - mr * disp * 4) == _capi.ERR_ARG           # one slot short
    assert call(itemsize=8) == _capi.ERR_DTYPE
    pad = _capi.Pad(mr, 0, None)
    assert L.dds_get_samples_padded(h, b"nope", s.data_ptr(), n, 4, None, ctypes.byref(pad), view.data_ptr(), nbytes,
                                    _capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE, None, None, None) == _capi.ERR_UNKNOWN_VAR
    # uint8 -> bf16 with no table for the normalising code: the converting entries' rules
    cv = _capi.Convert(_capi.CVT_NORM_U8_BF16, None)
    assert L.dds_get_batch_padded(h, b"b3", s.data_ptr(), c.data_ptr(), n, 1, ctypes.byref(cv), ctypes.byref(pad),
                                  view.data_ptr(), nbytes, _capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE, None, None,
                                  None) == _capi.ERR_ARG
    cv = _capi.Convert(_capi.CVT_F32_BF16, None)
    assert L.dds_get_batch_padded(h, b"b3", s.data_ptr(), c.data_ptr(), n, 1, ctypes.byref(cv), ctypes.byref(pad),
                                  view.data_ptr(), nbytes, _capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE, None, None,
                                  None) == _capi.ERR_DTYPE
    torch.cuda.synchronize()
    assert np.array_equal(whole.cpu().numpy(), before)
    assert (lens.cpu().numpy() == -5).all()
    # raw variable whose itemsize is not 1, 2, 4 or 8
    store.init("odd", 100, 2, 3)
    pad = _capi.Pad(2, 0, None)
    assert L.dds_get_batch_padded(h, b"odd", s.data_ptr(), c.data_ptr(), n, 3, None, ctypes.byref(pad),
                                  view.data_ptr(), nbytes, _capi.IDX_ON_DEVICE | _capi.DST_ON_DEVICE, None, None,
                                  None) == _capi.ERR_ARG
    # Python: pad_value the dtype cannot hold
    with pytest.raises(ValueError):
        store.get_batch("f3", s, c, out=view[:nbytes].view(torch.int32), pad_rows=mr, pad_value=2**40)
    with pytest.raises(ValueError):
        store.get_batch("f3", s, c, out=view[:nbytes].view(torch.uint8), pad_rows=mr)  # wrong element size


def test_queue(env):
    """padded, packed and converting batches interleaved in an overlapped double-buffered queue, wait() totals; once
    under SM contention; an invalid padded batch reported by wait() with its index, also across an implicit drain"""
    from ddstore_b200 import _capi
    store, rng = env["store"], env["rng"]
    mr, disp = 5, 80
    batches = []
    for k in range(12):
        s, c = _requests(rng, 700, 6)
        batches.append((torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV), s, c))
    from ddstore_b200.store import _pad_bits
    nan_bits = _pad_bits(float("nan"), torch.float32)
    exp = [_expect(store, "f80", b[2], b[3], mr, nan_bits, np.uint32)[:2] for b in batches]
    pk = [np.asarray(b[3]).sum() * disp * 4 for b in batches]
    st = torch.cuda.Stream()
    for contention in (False, True):
        outs = [torch.empty(700 * mr * disp, dtype=torch.float32, device=DEV) for _ in range(2)]
        lens = [torch.empty(700, dtype=torch.int64, device=DEV) for _ in range(2)]
        packed = [torch.empty(int(max(pk)), dtype=torch.uint8, device=DEV) for _ in range(2)]
        conv = [torch.empty(int(max(pk)) // 2, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
        torch.cuda.synchronize()
        if contention:
            _capi.lib().dds_test_occupy(0, 66, 200 * 1024, 30_000_000, st.cuda_stream)
        for k, (s, c, _, _) in enumerate(batches):
            j = k % 2
            if k % 3 == 0:
                store.get_batch("f80", s, c, out=outs[j], pad_rows=mr, pad_value=float("nan"), lengths=lens[j],
                                wait=False, overlap=True, stream=st.cuda_stream)
                assert store.wait() == 700 * mr * disp * 4
                st.synchronize()
                got = outs[j].cpu().numpy().view(np.uint32)
                assert np.array_equal(got, exp[k][0].reshape(-1)), k
                assert lens[j].cpu().numpy().tolist() == exp[k][1].tolist()
            elif k % 3 == 1:
                store.get_batch("f80", s, c, out=packed[j], wait=False, overlap=True, stream=st.cuda_stream)
                store.get_batch("f80", s, c, out=outs[j], pad_rows=mr, pad_value=float("nan"), lengths=lens[j],
                                wait=False, overlap=True, stream=st.cuda_stream)
                assert store.wait() == 700 * mr * disp * 4
                got = outs[j].cpu().numpy().view(np.uint32)
                assert np.array_equal(got, exp[k][0].reshape(-1)), k
            else:
                store.get_batch("f80", s, c, out=conv[j], src_dtype=torch.float32, wait=False, overlap=True,
                                stream=st.cuda_stream)
                store.get_batch("f80", s, c, out=outs[j], pad_rows=mr, pad_value=float("nan"), lengths=lens[j],
                                wait=False, overlap=True, stream=st.cuda_stream)
                store.get_batch("f80", s, c, out=packed[j], wait=False, overlap=True, stream=st.cuda_stream)
                assert store.wait() == pk[k]
                got = outs[j].cpu().numpy().view(np.uint32)
                assert np.array_equal(got, exp[k][0].reshape(-1)), k
                assert np.array_equal(packed[j][:pk[k]].cpu().numpy(), _raw_packed(store, "f80", batches[k][2],
                                                                                   batches[k][3], np.ones(700, bool)))
    # an invalid padded batch inside a queue: reported by wait() with its index, kept across an implicit drain
    s, c = batches[0][2].copy(), batches[0][3].copy()
    s[40] = -1
    sd, cd = torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV)
    out = torch.empty(700 * mr * disp, dtype=torch.float32, device=DEV)
    store.get_batch("f80", batches[1][0], batches[1][1], out=packed[0], wait=False, overlap=True, stream=st.cuda_stream)
    store.get_batch("f80", sd, cd, out=out, pad_rows=mr, wait=False, overlap=True, stream=st.cuda_stream)
    store.get_batch("f80", batches[2][0], batches[2][1], out=packed[1], wait=False, overlap=True, stream=st.cuda_stream)
    with pytest.raises(ValueError):
        store.wait()
    assert store.last_bad_index == 40
    assert store.wait() == 0
    store.get_batch("f80", sd, cd, out=out, pad_rows=mr, wait=False, stream=st.cuda_stream)
    store.get_batch("f80", batches[2][2], batches[2][3], out=packed[1])  # synchronous: drains the queue, clean itself
    with pytest.raises(ValueError):
        store.wait()
    assert store.last_bad_index == 40


def test_empty_batch_wait_total(env):
    """an empty (nreq = 0) DDS_NO_SYNC batch queued behind a padded batch on the same stream is the last batch queued:
    wait() reports its total, 0 -- through the padded, packed, converting and multi-array entries alike"""
    store, rng = env["store"], env["rng"]
    st = torch.cuda.Stream()
    s, c = _requests(rng, 300, 6)
    ds, dc = torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV)
    out = torch.empty(300 * 4 * 80, dtype=torch.float32, device=DEV)
    e = torch.empty(0, dtype=torch.int64, device=DEV)
    small = torch.empty(16, dtype=torch.uint8, device=DEV)
    sb = torch.empty(16, dtype=torch.bfloat16, device=DEV)
    tab = (env["sstart"][:-1], env["L"])
    empties = {"padded": lambda: store.get_batch("f80", e, e, out=out, pad_rows=4, wait=False, stream=st.cuda_stream),
               "padded by sample": lambda: store.get_samples("f80", e, out, pad_rows=4, wait=False, stream=st.cuda_stream),
               "packed": lambda: store.get_batch("f80", e, e, out=small, wait=False, stream=st.cuda_stream),
               "converting": lambda: store.get_batch("f80", e, e, out=sb, src_dtype=torch.float32, wait=False,
                                                     stream=st.cuda_stream),
               "multi-array": lambda: store.get_samples_multi(["f80", "d5"], e, [small, small], wait=False,
                                                              stream=st.cuda_stream)}
    assert tab[0].size == NSAMP
    for kind, empty in empties.items():
        full = store.get_batch("f80", ds, dc, out=out, pad_rows=4, wait=False, stream=st.cuda_stream)
        assert full == 300 * 4 * 80 * 4
        empty()
        assert store.wait() == 0, kind
        store.get_batch("f80", ds, dc, out=out, pad_rows=4, wait=False, stream=st.cuda_stream)
        assert store.wait() == 300 * 4 * 80 * 4, kind  # (and a non-empty last batch still reports its own)


def test_over_4gib(env):
    """one batch whose padded output passes 4 GiB: the last slot and the guard band after it"""
    store, rng = env["store"], env["rng"]
    n, mr = 65536, 22000  # 3-byte rows: 4.33 GB
    var, disp = "b3", 3
    nbytes = n * mr * disp
    assert nbytes > 1 << 32
    s, c = _requests(rng, n, 6)
    c[-1] = 6
    whole, view = _guarded(nbytes, 0)
    lens = torch.empty(n, dtype=torch.int64, device=DEV)
    total = store.get_batch(var, torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV), out=view, pad_rows=mr,
                            pad_value=0x5A, lengths=lens)
    assert total == nbytes
    slots, lengths = po.pad_rows(_raw_packed(store, var, s[-3:], c[-3:], np.ones(3, bool)), c[-3:], disp, mr, np.uint8(0x5A))
    torch.cuda.synchronize()
    tail = whole[GUARD + nbytes - 3 * mr * disp:].cpu().numpy()
    assert tail[:3 * mr * disp].tobytes() == slots.tobytes()
    assert (tail[3 * mr * disp:] == SENT).all()
    assert lens[-3:].cpu().numpy().tolist() == lengths.tolist()
    head = whole[:GUARD + 2 * mr * disp].cpu().numpy()
    assert (head[:GUARD] == SENT).all()
    exp0, _ = po.pad_rows(_raw_packed(store, var, s[:2], c[:2], np.ones(2, bool)), c[:2], disp, mr, np.uint8(0x5A))
    assert head[GUARD:].tobytes() == exp0.tobytes()
    del whole, view
    torch.cuda.empty_cache()


def test_world():
    """three owners: every slot gathered across the owners' shards"""
    def body(store, r):
        disp = 4
        rows = np.arange(300 * disp, dtype=np.float32).reshape(300, disp) + 10000 * r
        store.add("w", rows)
        rng = np.random.default_rng(r)
        s = rng.integers(0, 890, 200)
        c = rng.integers(0, 8, 200)
        ll = store.query("w")["lenlist"]
        codes = classify(ll, s, c)
        allrows = np.concatenate([np.arange(300 * disp, dtype=np.float32).reshape(300, disp) + 10000 * k for k in range(3)])
        packed = np.concatenate([allrows[a:a + b].reshape(-1) for a, b, v in zip(s, c, codes == 0) if v] or
                                [np.zeros(0, np.float32)])
        exp, lens = po.pad_rows(packed, np.where(codes == 0, c, 0), disp, 5, np.float32(-1), codes == 0)
        out = torch.empty(200 * 5 * disp, dtype=torch.float32, device=DEV)
        ln = torch.empty(200, dtype=torch.int64, device=DEV)
        try:
            store.get_batch("w", s, c, out=out, pad_rows=5, pad_value=-1, lengths=ln)
            assert (codes == 0).all()
        except ValueError:
            assert store.last_bad_index == int(np.nonzero(codes)[0][0])
        assert np.array_equal(out.cpu().numpy(), exp.reshape(-1))
        assert ln.cpu().numpy().tolist() == lens.tolist()
        return True
    assert run_world(3, body) == [True] * 3


@pytest.mark.skipif(os.environ.get("DDS_PAD_SUBPROCESS") == "1", reason="already in the subprocess")
def test_subprocess_pdl_off():
    env = dict(os.environ, DDS_PDL="0", DDS_PAD_SUBPROCESS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", __file__, "-k",
                        "shapes_raw or offsets or sample_ids or invalid or conversions or queue or loaders"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]


def test_loaders():
    """RaggedDataset(pad=...) and RaggedPrefetchLoader over two epochs: the padded variables equal the unpadded
    dataset's packed batches padded by the oracle (one raw, one normalised into bf16); the packed variable is unchanged"""
    from ddstore_b200.dataset import RaggedDataset, RaggedPrefetchLoader
    from ddstore_b200.store import _pad_bits
    rng = np.random.default_rng(21)
    n = 300
    cnt = rng.integers(0, 12, n)
    tcnt = rng.integers(0, 40, n)
    ecnt = rng.integers(0, 6, n)
    x = rng.standard_normal((int(cnt.sum()), 5)).astype(np.float32)
    t = rng.integers(0, 30000, (int(tcnt.sum()), 1)).astype(np.int32)
    e = rng.integers(0, 1000, (int(ecnt.sum()), 2)).astype(np.int64)
    xm, xs = rng.standard_normal(5).astype(np.float32), rng.random(5).astype(np.float32) + 0.2
    arrays, counts = {"x": x, "t": t, "e": e}, {"x": cnt, "t": tcnt, "e": ecnt}
    rr = RaggedDataset(arrays, counts)
    rp = RaggedDataset(arrays, counts, out_dtypes={"x": torch.bfloat16}, normalize={"x": (xm, xs)},
                       pad={"x": (8, float("-inf")), "t": (24, -100)})
    xm_t, xs_t = torch.from_numpy(xm).to(DEV), torch.from_numpy(xs).to(DEV)
    ninf = _pad_bits(float("-inf"), torch.bfloat16)

    def expect(a, ids):
        px, ox = a["x"]
        xn = ((px - xm_t) / xs_t).to(torch.bfloat16).view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
        sx, lx = po.pad_rows(xn, cnt[ids], 5, 8, np.uint16(ninf))
        st_, lt = po.pad_rows(a["t"][0].cpu().numpy().reshape(-1), tcnt[ids], 1, 24, np.int32(-100))
        return sx, lx, st_, lt

    def check(a, b, ids):
        sx, lx, st_, lt = expect(a, ids)
        bx, blx = b["x"]
        assert tuple(bx.shape) == (len(ids), 8, 5) and bx.dtype == torch.bfloat16
        assert bx.view(torch.int16).cpu().numpy().view(np.uint16).tobytes() == sx.tobytes()
        assert blx.cpu().numpy().tolist() == lx.tolist()
        bt, blt = b["t"]
        assert tuple(bt.shape) == (len(ids), 24, 1) and bt.dtype == torch.int32
        assert bt.cpu().numpy().tobytes() == st_.tobytes() and blt.cpu().numpy().tolist() == lt.tolist()
        assert torch.equal(b["e"][0], a["e"][0]) and torch.equal(b["e"][1], a["e"][1])

    ids = list(rng.integers(0, n, 40))
    check(rr.__getitems__(ids), rp.__getitems__(ids), ids)
    for epoch in range(2):
        order = list(np.random.default_rng(epoch).permutation(n))
        batches = [order[i:i + 32] for i in range(0, n, 32)]
        for k, (ba, bb) in enumerate(zip(RaggedPrefetchLoader(rr, order, 32), RaggedPrefetchLoader(rp, order, 32))):
            check(ba, bb, batches[k])
        assert k == len(batches) - 1
    only = RaggedDataset({"t": t}, {"t": tcnt}, pad={"t": 24})  # every variable padded: no packed launch at all
    got = only.__getitems__(ids)
    assert list(got) == ["t"]
    assert got["t"][1].cpu().numpy().tolist() == np.minimum(tcnt[ids], 24).tolist()
    for bb in RaggedPrefetchLoader(only, list(range(n)), 64):
        assert tuple(bb["t"][0].shape)[1:] == (24, 1)
    with pytest.raises(ValueError):
        RaggedDataset({"t": t}, {"t": tcnt}, pad={"t": (4, 2**40)})
    rr.free()
    rp.free()
    only.free()


def test_cython_binding(env):
    """pyddstore.PyDDStore.get_batch with pad_rows / pad_value / lengths, raw and converting"""
    sys.path.insert(0, os.path.join(ROOT, "ddstore_b200", "cython"))
    import pyddstore
    from ddstore_b200.store import _pad_bits
    store = pyddstore.PyDDStore(device=0)
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((500, 4)).astype(np.float32)
    store.add("c", rows)
    s = rng.integers(0, 480, 50)
    c = rng.integers(0, 9, 50)
    packed = np.concatenate([rows[a:a + b].reshape(-1) for a, b in zip(s, c)])
    out = torch.empty(50 * 6 * 4, dtype=torch.float32, device=DEV)
    lens = torch.empty(50, dtype=torch.int64, device=DEV)
    total = store.get_batch("c", torch.as_tensor(s, device=DEV), torch.as_tensor(c, device=DEV), out=out, pad_rows=6,
                            pad_value=-2.0, lengths=lens)
    exp, el = po.pad_rows(packed, c, 4, 6, np.float32(-2.0))
    assert total == out.numel() * 4 and np.array_equal(out.cpu().numpy(), exp.reshape(-1))
    assert lens.cpu().numpy().tolist() == el.tolist()
    outb = torch.empty(50 * 6 * 4, dtype=torch.bfloat16, device=DEV)
    store.get_batch("c", s, c, out=outb, src_dtype=torch.float32, pad_rows=6, pad_value=float("-inf"))
    conv = torch.from_numpy(packed).to(DEV).to(torch.bfloat16).view(torch.int16).cpu().numpy().view(np.uint16)
    expb, _ = po.pad_rows(conv, c, 4, 6, np.uint16(_pad_bits(float("-inf"), torch.bfloat16)))
    assert outb.view(torch.int16).cpu().numpy().view(np.uint16).tobytes() == expb.tobytes()
    s2 = s.copy()
    s2[7] = -1
    with pytest.raises(ValueError):
        store.get_batch("c", s2, c, out=out, pad_rows=6)
    store.free()
