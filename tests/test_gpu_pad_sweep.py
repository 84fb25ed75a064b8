"""The padded gather (dds_get_batch_padded / dds_get_samples_padded) swept against a host reference (-m gpu).

Reference, independent of the store: every variable is added from NumPy rows kept on the host. A batch's expected
output is the NumPy slices of its valid requests (truncated to max_rows), converted by tests/convert_oracle.py or
normalised by tests/norm_oracle.py, then padded by tests/pad_oracle.pad_rows. Payload elements compare by NaN class;
for float sources they must also equal, bit for bit, torch's CUDA expression of the same host rows (`.to(dtype)`, or
((x.to(f32) - mean) / std).to(dtype) with the tables laid out by the channel rule). Padding elements compare bit for
bit. Payload is random bits (NaN, +-inf, subnormals, -0 all occur); the first rows of the float variables hold
convert_oracle.F32_EDGE_BITS / f64_edge_bits(), and the first batch of every variable covers them. Each batch is
checked on every slot, `lengths`, the returned total, the first invalid request's error and last_bad_index, and
64-byte sentinel bands on both sides of the destination and of `lengths`; a mismatch names the slot, its request, the
row and element, and whether the element is payload or padding.

The workload is tests/pad_sweep.workload() for the warp count of this GPU (12 warps per SM; the padded launch runs one
CTA per SM). The module asserts that it hits every category
of pad_sweep.REQUIRED: whole-slot and whole-chunk segments, segments of more than 32 and 64 slots, segment and chunk
cuts mid-row, at a row boundary, at the payload end and (segments) in padding, padding runs shorter than, equal to and
one element either side of a multiple of 16 bytes at every 16-byte phase, and invalid requests at window lanes 0, 31,
32, 63 and at a segment's first and last slot. Padding runs longer than 1 MiB of output need segments above 256 KiB,
i.e. a uint8 -> float32 batch of more than 13 GB at 132 SMs; they are out of reach here.

Also covered: get_samples with every conversion code and out-of-range ids; lengths=None; max_rows = 0 with requests
(lengths 0, total 0, errors reported); nreq = 0; normalising codes with scalar, per-feature (std = 0 and negative std
included), channels-last (C = 3), CHW rows longer than a chunk (uint8 3x40x40, float32 3x32x33) and a pattern that
repeats inside the row (4 channels of 5 on 40); overlapped double-buffered queues on one stream mixing padded raw,
converting, normalising, max_rows = 0 and all-invalid batches with packed fixed-count, variable-count (shared-memory
and plan-kernel plans) and converting multi-array batches, plain and under dds_test_occupy contention, checking every
buffer, wait() totals after queues ending in each kind and the first failing batch's request index; three 4 GiB cases
(uint8 -> normalised float32 with the output above 4 GiB, float32 -> bf16 and float64 -> normalised float32 with the
source space above 4 GiB); a three-owner world with thread-ranks on device 0, and one GPU per rank when three exist.

Each configuration runs in a subprocess of its own: default, DDS_PDL=0, DDS_SMEM_PLAN=0 and DDS_VAR_MINSEG=1
DDS_S_MINSEG=1. The last two change only the packed variable-count neighbours in the queues; the padded launch has no
plan and a fixed smallest segment.

On an H100 80GB HBM3 (700 W power limit, 132 SMs) the module takes about 120 s: 26 to 33 s per configuration.
"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import convert_oracle as co
from tests import norm_oracle as no
from tests import pad_oracle as po
from tests import pad_sweep as ps
from tests.gpu_helpers import GUARD, classify, error_text, run_world

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = {"default": {}, "nopdl": {"DDS_PDL": "0"}, "plankernels": {"DDS_SMEM_PLAN": "0"},
           "minseg1": {"DDS_VAR_MINSEG": "1", "DDS_S_MINSEG": "1"}}
SENT = 0xA5
LSENT = -5
NAN_F32, NAN_F16, NAN_F64 = 0x7FC01234, 0x7E55, 0x7FF80000DEADBEEF


class Ctx:
    """the store, the host rows of every variable, and the conversions as torch sees them"""

    def __init__(self, torch, store, rng):
        self.torch, self.store, self.rng = torch, store, rng
        self.dev = torch.device("cuda", 0)
        self.rows, self.norm = {}, {}
        x = torch.arange(256, dtype=torch.float32)
        self.lut16 = ((x - 127.5) / 60.1).to(torch.bfloat16)
        self.lut32 = x / 255 - 0.25
        self.dec = (x - 100.0) * 0.37  # uint8 decode table of the normalising codes
        t = torch
        # code -> (torch source dtype, output dtype, normalize, table, pad value: a one-element tensor of the output dtype)
        self.cv = {1: (t.float32, t.bfloat16, False, None, self.bits(0xFF80, t.bfloat16)),
                   2: (t.float32, t.float16, False, None, self.bits(NAN_F16, t.float16)),
                   3: (t.float64, t.float32, False, None, self.bits(NAN_F32, t.float32)),
                   4: (t.uint8, t.bfloat16, False, self.lut16, self.bits(0xFF80, t.bfloat16)),
                   5: (t.uint8, t.float32, False, self.lut32, self.bits(NAN_F32, t.float32)),
                   6: (t.float32, t.float32, True, None, self.bits(NAN_F32, t.float32)),
                   7: (t.float32, t.bfloat16, True, None, self.bits(0xFF80, t.bfloat16)),
                   8: (t.float32, t.float16, True, None, self.bits(NAN_F16, t.float16)),
                   9: (t.float64, t.float32, True, None, self.bits(NAN_F32, t.float32)),
                   10: (t.uint8, t.float32, True, self.dec, self.bits(NAN_F32, t.float32)),
                   11: (t.uint8, t.bfloat16, True, self.dec, self.bits(0xFF80, t.bfloat16)),
                   12: (t.uint8, t.float16, True, self.dec, self.bits(NAN_F16, t.float16))}

    def bits(self, b, dt):
        t = self.torch
        ib = {t.float16: t.int16, t.bfloat16: t.int16, t.float32: t.int32, t.float64: t.int64, t.int16: t.int16,
              t.int32: t.int32, t.uint8: t.uint8}[dt]
        nb = {t.int16: 16, t.int32: 32, t.int64: 64, t.uint8: 8}[ib]
        v = b - (1 << nb) if ib != t.uint8 and b >= 1 << (nb - 1) else b
        return t.tensor([v], dtype=ib).view(dt)

    def raw_conv(self, var):
        """raw output dtype and pad value of a variable"""
        t = self.torch
        dt = ps.VARS[var][0]
        if dt == "uint8":
            return t.uint8, self.bits(0x5A, t.uint8)
        if dt == "int16":
            return t.float16, self.bits(0xFFFD, t.float16)  # (a 2-byte padded output is a half tensor)
        if dt == "int32":
            return t.int32, self.bits(0xFFFFFF9C, t.int32)  # -100, a token id's padding
        if dt == "float32":
            return t.float32, self.bits(NAN_F32, t.float32)
        return t.float64, self.bits(NAN_F64, t.float64)

    def add(self, var):
        dt, disp, nrows = ps.VARS[var]
        h = self.rng.integers(0, 256, size=nrows * disp * np.dtype(dt).itemsize, dtype=np.uint8).view(dt).reshape(nrows, disp)
        edge = co.F32_EDGE_BITS if dt == "float32" else co.f64_edge_bits() if dt == "float64" else None
        if edge is not None:
            e = np.resize(np.asarray(edge, np.uint32 if dt == "float32" else np.uint64), min(nrows, 64) * disp)
            h.reshape(-1)[:e.size] = e.view(dt)
        self.rows[var] = h
        if dt == "int16":  # (PyDDStore.add takes no 2-byte arrays; the C entry does)
            from ddstore_b200 import _capi
            _capi.raise_for(self.store._L.dds_add(self.store._h, var.encode(), h.ctypes.data, nrows, disp, 2, 0))
        else:
            self.store.add(var, h)

    def set_norm(self, var, mean, std, inner=1):
        mean, std = np.asarray(mean, np.float32), np.asarray(std, np.float32)
        self.store.set_normalization(var, mean, std, inner=inner)
        self.norm[var] = (mean, std, mean.size, inner)


# ------------------------------------------------------------------------------------------------ the reference
def expected(ctx, var, code, starts, counts, max_rows, valid):
    """-> (expected output elements [nreq, max_rows, disp] as unsigned ints, lengths, payload mask, torch payload bits or
    None, out dtype, pad tensor)"""
    torch = ctx.torch
    dt, disp, _ = ps.VARS[var]
    rows = ctx.rows[var]
    take = np.where(valid, np.minimum(np.clip(counts, 0, None), max_rows), 0).astype(np.int64)
    parts = [rows[s:s + n] for s, n in zip(np.asarray(starts).tolist(), take.tolist()) if n > 0]
    src = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0, disp), dt)).view(np.uint8).reshape(-1)
    if code == 0:
        odt, pad = ctx.raw_conv(var)
        out_el = np.dtype(dt).itemsize
        ob, tb = src, None
    else:
        sdt, odt, nz, lut, pad = ctx.cv[code]
        out_el = ps.CVT_IO[code][1]
        if nz:
            mean, std, nch, inner = ctx.norm[var]
            ob = no.norm_bytes(src, code, mean, std, nch, inner, None if lut is None else lut.numpy())
        else:
            ob = co.convert_bytes(src, code, None if lut is None else lut.contiguous().view(torch.uint8).numpy())
        tb = None
        if sdt in (torch.float32, torch.float64) and src.size:
            x = torch.from_numpy(src.copy()).to(ctx.dev).view(sdt)
            if nz:
                ch = no.channels(disp, nch, inner)
                m = torch.from_numpy(mean[ch]).to(ctx.dev)
                s = torch.from_numpy(std[ch]).to(ctx.dev)
                y = ((x.to(torch.float32).view(-1, disp) - m) / s).to(odt)
            else:
                y = x.to(odt)
            tb = y.reshape(-1).view(torch.uint8).cpu().numpy()
    udt = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[out_el]
    pad_u = pad.view(torch.uint8).numpy().view(udt)[0]
    slots, lengths = po.pad_rows(np.ascontiguousarray(ob).view(udt), take, disp, max_rows, pad_u, valid)
    tslots = None
    if tb is not None:
        tslots, _ = po.pad_rows(tb.view(udt), take, disp, max_rows, pad_u, valid)
    mask = np.arange(max_rows)[None, :] < lengths[:, None]
    return slots, lengths, mask, tslots, odt, pad, out_el, code


def nan_class(u, out_el, kind):
    if kind == "raw":
        return np.zeros(u.shape, bool)
    if kind == "bf16":
        return ((u & 0x7F80) == 0x7F80) & ((u & 0x7F) != 0)
    if kind == "f16":
        return ((u & 0x7C00) == 0x7C00) & ((u & 0x3FF) != 0)
    if out_el == 4:
        return ((u & 0x7F800000) == 0x7F800000) & ((u & 0x7FFFFF) != 0)
    return np.zeros(u.shape, bool)


def out_kind(torch, odt):
    return {torch.bfloat16: "bf16", torch.float16: "f16"}.get(odt, "other")


def compare(ctx, got, exp, what, starts, counts, valid, max_rows, disp):
    """got: host bytes of the slots. Raises naming the first bad element's slot, request, row, element, part."""
    slots, lengths, mask, tslots, odt, _, out_el, code = exp
    udt = slots.dtype
    g = np.ascontiguousarray(got).view(udt).reshape(slots.shape)
    kind = out_kind(ctx.torch, odt) if code else "raw"
    pm = np.repeat(mask[:, :, None], disp, axis=2)
    bad = (g != slots) & ~(pm & nan_class(g, out_el, kind) & nan_class(slots, out_el, kind))
    if tslots is not None:
        tb = (tslots != slots) & ~(pm & nan_class(tslots, out_el, kind) & nan_class(slots, out_el, kind))
        assert not tb.any(), f"{what}: torch's CUDA expression and the NumPy oracle differ at {np.argwhere(tb)[0]}"
        bad |= pm & (g != tslots)
    if bad.any():
        i, r, e = (int(x) for x in np.argwhere(bad)[0])
        part = "payload" if pm[i, r, e] else "padding"
        raise AssertionError(
            f"{what}: {int(bad.sum())} elements differ; first in slot {i} (request start={int(starts[i])}, "
            f"count={int(counts[i])}, valid={bool(valid[i])}, length {int(lengths[i])}), row {r}, element {e} "
            f"({part}): got {int(g[i, r, e]):#x}, expected {int(slots[i, r, e]):#x}")


def first_bad(ctx, var, starts, counts, by_sample_ok=None):
    nrows = ps.VARS[var][2]
    valid = ps.row_valid(nrows, starts, counts)
    if by_sample_ok is not None:
        valid &= by_sample_ok
    bad = np.nonzero(~valid)[0]
    return valid, (int(bad[0]) if bad.size else -1)


def run_batch(ctx, var, code, starts, counts, max_rows, off=0, dev_idx=True, with_lengths=True, ids=None,
              sample_tab=None, what=""):
    """one padded batch between guard bands, checked against the reference"""
    torch, store = ctx.torch, ctx.store
    dev = ctx.dev
    dt, disp, nrows = ps.VARS[var]
    ok = None
    if ids is not None:
        ok = (ids >= 0) & (ids < len(sample_tab[0]))
        cl = np.clip(ids, 0, len(sample_tab[0]) - 1)
        starts, counts = np.where(ok, sample_tab[0][cl], 0), np.where(ok, sample_tab[1][cl], 0)
    valid, bad = first_bad(ctx, var, starts, counts, ok)
    exp = expected(ctx, var, code, starts, counts, max_rows, valid)
    odt, pad, out_el = exp[4], exp[5], exp[6]
    n = len(starts)
    nbytes = n * max_rows * disp * out_el
    whole = torch.full((2 * GUARD + off + nbytes,), SENT, dtype=torch.uint8, device=dev)
    lwhole = torch.full((2 * (GUARD // 8) + n,), LSENT, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    out = whole[GUARD + off:GUARD + off + nbytes].view(odt)
    lens = lwhole[GUARD // 8:GUARD // 8 + n] if with_lengths else None
    kw = {}
    if code:
        sdt, _, nz, lut, _ = ctx.cv[code]
        kw = dict(src_dtype=sdt, lut=lut, normalize=nz)
    err, total = None, None
    try:
        if ids is not None:
            x = torch.as_tensor(ids, device=dev) if dev_idx else ids
            total = store.get_samples(var, x, out, pad_rows=max_rows, pad_value=pad, lengths=lens, **kw)
        else:
            s, c = np.asarray(starts, np.int64), np.asarray(counts, np.int64)
            if dev_idx:
                s, c = torch.as_tensor(s, device=dev), torch.as_tensor(c, device=dev)
            total = store.get_batch(var, s, c, out=out, pad_rows=max_rows, pad_value=pad, lengths=lens, **kw)
    except ValueError as e:
        err = str(e)
    torch.cuda.synchronize()
    what = f"{what} {var} code={code} max_rows={max_rows} nreq={n} dst+{off} dev_idx={dev_idx} ids={ids is not None}"
    w = whole.cpu().numpy()
    pre, post = np.nonzero(w[:GUARD + off] != SENT)[0], np.nonzero(w[GUARD + off + nbytes:] != SENT)[0]
    assert pre.size == 0, f"{what}: guard byte {int(pre[-1]) - GUARD - off} before the destination was written"
    assert post.size == 0, f"{what}: guard byte {int(post[0])} past the destination's end was written"
    compare(ctx, w[GUARD + off:GUARD + off + nbytes], exp, what, starts, counts, valid, max_rows, disp)
    lw = lwhole.cpu().numpy()
    g8 = GUARD // 8
    assert (lw[:g8] == LSENT).all() and (lw[g8 + n:] == LSENT).all(), f"{what}: guard of lengths written"
    if with_lengths:
        d = np.nonzero(lw[g8:g8 + n] != exp[1])[0]
        assert d.size == 0, f"{what}: lengths[{int(d[0])}] = {int(lw[g8 + d[0]])}, expected {int(exp[1][d[0]])}"
    else:
        assert (lw == LSENT).all(), f"{what}: lengths=None, yet the lengths buffer was written"
    if bad >= 0:
        assert err is not None and store.last_bad_index == bad, (what, err, store.last_bad_index, bad)
        want = "sample id" if ids is not None and not ok[bad] else \
            error_text(int(classify([nrows], starts[bad:bad + 1], counts[bad:bad + 1])[0]))
        assert want in err, f"{what}: raised {err!r}, expected {want!r} for request {bad}"
    else:
        assert err is None and total == nbytes, f"{what}: raised {err!r} / total {total}, expected {nbytes}"
    return exp


# ------------------------------------------------------------------------------------------------ the parts
NORM_LAYOUTS = {  # variable -> [(label, mean, std, inner)]
    "f32x3": [("channels-last", [0.5, -1.0, 2.0], [0.25, 3.0, -0.5], 1), ("scalar", [0.125], [0.0], 1)],
    "f32x40": [("4 channels of 5, repeating", [0.1, -0.2, 3.0, 1e-3], [2.0, -1.5, 0.0, 7.0], 5),
               ("per-feature", np.resize(no.TABLE_EDGE_MEAN, 40), np.resize(no.TABLE_EDGE_STD, 40), 1)],
    "f32img": [("CHW 3x32x33", [0.485, 0.456, 0.406], [0.229, -0.224, 0.0], 32 * 33)],
    "u8img": [("CHW 3x40x40", [123.7, 116.3, 103.5], [58.4, 57.1, -57.4], 1600)],
    "u8x3": [("channels-last", [10.0, 20.0, 30.0], [2.0, 0.0, -4.0], 1)],
    "f64x3": [("channels-last", [0.5, 0.25, -3.0], [1.5, -2.0, 0.0], 1)],
    "f32x1025": [("per-feature", np.linspace(-1, 1, 1025), np.linspace(0.5, 2, 1025), 1)],
}


def default_norm(ctx, var):
    disp = ps.VARS[var][1]
    if var in NORM_LAYOUTS:
        lab, m, s, inner = NORM_LAYOUTS[var][0]
        ctx.set_norm(var, m, s, inner)
    else:
        ctx.set_norm(var, [0.75] if disp % 2 else np.linspace(-2, 2, disp), [1.25] if disp % 2 else np.linspace(0.5, -3, disp))


def part_sweep(ctx, nwarps, phase):
    batches = ps.workload(nwarps)
    hit = ps.workload_coverage(batches, nwarps)
    missing = ps.REQUIRED - hit
    assert not missing, f"the sweep's workload misses {sorted(missing)} at {nwarps} warps"
    for b in batches:
        run_batch(ctx, b.var, b.code, b.starts, b.counts, b.max_rows, b.off, b.dev_idx, b.with_lengths, what="sweep")
    phase(f"sweep of {len(batches)} batches")
    # every normalisation layout on its variable, through the normalising codes of its source type
    for var, layouts in NORM_LAYOUTS.items():
        dt, disp, nrows = ps.VARS[var]
        codes = [c for c in ps.CODES[dt] if c >= 6]
        rb = disp * np.dtype(dt).itemsize
        for lab, m, s, inner in layouts:
            ctx.set_norm(var, m, s, inner)
            for k, code in enumerate(codes):
                mr = max(1, (3 * ps.CH) // rb)  # rows long enough for chunk cuts to land mid-channel
                n = 40 if rb > 1000 else 300
                counts = ctx.rng.integers(0, mr + 2, n)
                starts = ctx.rng.integers(0, nrows - mr - 2, n)
                starts[0], counts[0] = 0, mr
                run_batch(ctx, var, code, starts, counts, mr, off=(4 * k) % 16 // ps.CVT_IO[code][1] * ps.CVT_IO[code][1],
                          what=f"norm {lab}")
        default_norm(ctx, var)
    phase("normalisation layouts")


def part_entries(ctx, tabs):
    """get_samples raw and with every code (out-of-range ids), lengths=None, max_rows 0, nreq 0"""
    rng = ctx.rng
    for var in ("u8x3", "f32x5", "f64x3", "tok"):
        dt = ps.VARS[var][0]
        st, ct = tabs[var]
        for k, code in enumerate(ps.CODES[dt]):
            ids = rng.integers(0, len(st), 900)
            ids[[0, 31, 500]] = [len(st) + 3, -1, len(st)] if k % 2 else [5, 6, 7]
            run_batch(ctx, var, code, None, None, 5, off=0, dev_idx=k % 2 == 0, with_lengths=k % 3 != 1, ids=ids,
                      sample_tab=(st, ct), what="get_samples")
    # max_rows = 0: nothing walked, lengths all 0, total 0, the first invalid request still reported
    for var, code in (("f32x5", 0), ("f32x5", 7), ("u8x3", 10)):
        nrows = ps.VARS[var][2]
        s, c = rng.integers(0, nrows - 9, 200), rng.integers(0, 9, 200)
        run_batch(ctx, var, code, s, c, 0, what="max_rows 0")
        s[77], c[77] = nrows, 1
        s[150], c[150] = 3, -1
        run_batch(ctx, var, code, s, c, 0, what="max_rows 0 invalid")
    # nreq = 0
    for var, code in (("f32x5", 0), ("f32x5", 8)):
        e = np.zeros(0, np.int64)
        run_batch(ctx, var, code, e, e, 4, dev_idx=True, what="nreq 0")
        run_batch(ctx, var, code, e, e, 4, dev_idx=False, what="nreq 0")


def part_queues(ctx, tabs):
    """overlapped double-buffered queues on one stream"""
    import torch
    from ddstore_b200 import _capi
    store, rng, dev = ctx.store, ctx.rng, ctx.dev
    side, other = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    CAP = 8 << 20
    bufs = [torch.full((2 * GUARD + CAP,), SENT, dtype=torch.uint8, device=dev) for _ in range(2)]
    lbufs = [torch.full((2 * (GUARD // 8) + 4096,), LSENT, dtype=torch.int64, device=dev) for _ in range(2)]
    mbufs = [torch.full((2 * GUARD + CAP,), SENT, dtype=torch.uint8, device=dev) for _ in range(2)]  # multi's 2nd var

    def dev_i64(a):
        return torch.as_tensor(np.ascontiguousarray(a, np.int64), device=dev)

    def padded(var, code, mr, n, invalid_all=False, bad_at=None):
        def make(j):
            dt, disp, nrows = ps.VARS[var]
            s, c = rng.integers(0, nrows - mr - 3, n), rng.integers(0, mr + 3, n)
            if invalid_all:
                s[:] = nrows
            if bad_at is not None:
                s[bad_at], c[bad_at] = -1, 1
            valid, bad = first_bad(ctx, var, s, c)
            exp = expected(ctx, var, code, s, c, mr, valid)
            odt, pad, out_el = exp[4], exp[5], exp[6]
            nbytes = n * mr * disp * out_el
            out = bufs[j][GUARD:GUARD + nbytes].view(odt)
            lens = lbufs[j][GUARD // 8:GUARD // 8 + n]
            kw = {}
            if code:
                sdt, _, nz, lut, _ = ctx.cv[code]
                kw = dict(src_dtype=sdt, lut=lut, normalize=nz)
            ds, dc = dev_i64(s), dev_i64(c)

            def launch(st):
                store.get_batch(var, ds, dc, out=out, pad_rows=mr, pad_value=pad, lengths=lens, wait=False, overlap=True,
                                stream=st, **kw)

            def check(what):
                w = bufs[j].cpu().numpy()
                compare(ctx, w[GUARD:GUARD + nbytes], exp, what, s, c, valid, mr, disp)
                lw = lbufs[j].cpu().numpy()[GUARD // 8:GUARD // 8 + n]
                assert np.array_equal(lw, exp[1]), f"{what}: lengths differ"
            return launch, check, nbytes, bad
        return make

    def packed_fixed(var, cnt, n):
        def make(j):
            dt, disp, nrows = ps.VARS[var]
            s = rng.integers(0, nrows - cnt, n)
            rows = ctx.rows[var]
            exp = np.concatenate([rows[a:a + cnt].reshape(-1).view(np.uint8) for a in s])
            ds = dev_i64(s)

            def launch(st):
                store.get_batch(var, ds, out=bufs[j][GUARD:GUARD + exp.size], count=cnt, wait=False, overlap=True,
                                stream=st)

            def check(what):
                assert np.array_equal(bufs[j][GUARD:GUARD + exp.size].cpu().numpy(), exp), f"{what}: packed bytes differ"
            return launch, check, exp.size, -1
        return make

    def packed_var(var, n):
        def make(j):
            dt, disp, nrows = ps.VARS[var]
            s, c = rng.integers(0, nrows - 9, n), rng.integers(0, 9, n)
            rows = ctx.rows[var]
            exp = np.concatenate([rows[a:a + b].reshape(-1).view(np.uint8) for a, b in zip(s, c)])
            ds, dc = dev_i64(s), dev_i64(c)

            def launch(st):
                store.get_batch(var, ds, dc, out=bufs[j][GUARD:GUARD + exp.size], wait=False, overlap=True, stream=st)

            def check(what):
                assert np.array_equal(bufs[j][GUARD:GUARD + exp.size].cpu().numpy(), exp), f"{what}: packed bytes differ"
            return launch, check, exp.size, -1
        return make

    def multi(n):
        """f32x3 -> bf16 and u8x3 raw by sample id, one converting launch"""
        def make(j):
            ids = rng.integers(0, len(tabs["f32x3"][0]), n)
            exps = []
            for var in ("f32x3", "u8x3"):
                st, ct = tabs[var]
                rows = ctx.rows[var]
                exps.append(np.concatenate([rows[st[i]:st[i] + ct[i]].reshape(-1) for i in ids]))
            e0 = exps[0].view(np.uint8)
            b0 = torch.from_numpy(e0.copy()).to(dev).view(torch.float32).to(torch.bfloat16).view(torch.uint8).cpu().numpy()
            e1 = exps[1].view(np.uint8)
            o0 = bufs[j][GUARD:GUARD + b0.size].view(torch.bfloat16)
            o1 = mbufs[j][GUARD:GUARD + e1.size]
            d_ids = dev_i64(ids)

            def launch(st):
                store.get_samples_multi(["f32x3", "u8x3"], d_ids, [o0, o1], stream=st, wait=False, overlap=True,
                                        src_dtypes=[torch.float32, None])

            def check(what):
                assert np.array_equal(bufs[j][GUARD:GUARD + b0.size].cpu().numpy(), b0), f"{what}: multi f32x3 differs"
                assert np.array_equal(mbufs[j][GUARD:GUARD + e1.size].cpu().numpy(), e1), f"{what}: multi u8x3 differs"
            return launch, check, b0.size + e1.size, -1
        return make

    kinds = {"padded raw": padded("f32x40", 0, 6, 700), "padded converting": padded("f32x3", 1, 9, 900),
             "padded normalising": padded("u8img", 11, 2, 40), "padded max_rows 0": padded("f32x5", 0, 0, 300),
             "padded all-invalid": padded("tok", 0, 5, 64, invalid_all=True),
             "packed fixed": packed_fixed("u8x3", 2, 3000), "var shared-memory plan": packed_var("f32x5", 600),
             "var plan kernels": packed_var("f64x3", 3000), "multi converting": multi(500)}
    for contention in (False, True):
        orders = []
        for last in kinds:  # every kind last once; the all-invalid batch only there (it fails its queue)
            head = [k for k in kinds if k not in (last, "padded all-invalid")]
            rng.shuffle(head)
            orders.append(head + [last])
        if contention:
            orders = orders[:3]
        for order in orders:
            made = [kinds[k](q % 2) for q, k in enumerate(order)]
            torch.cuda.synchronize()
            if contention:
                _capi.raise_for(_capi.lib().dds_test_occupy(0, 100, 200 * 1024, 2_000_000, C.c_void_p(other.cuda_stream)))
            for launch, _, _, _ in made:
                launch(side.cuda_stream)
            what = f"queue {order} contention={contention}"
            fails = [(q, m[3]) for q, m in enumerate(made) if m[3] >= 0]
            if fails:
                with pytest.raises(ValueError):
                    store.wait()
                assert store.last_bad_index == fails[0][1], (what, store.last_bad_index, fails)
                assert store.wait() == 0
            else:
                assert store.wait() == made[-1][2], f"{what}: wait() total"
            torch.cuda.synchronize()
            for q in (len(made) - 2, len(made) - 1):  # the last user of each double buffer
                made[q][1](f"{what}, batch {q} ({order[q]})")
            for b in bufs + mbufs:
                assert (b[:GUARD] == SENT).all() and (b[-GUARD:] == SENT).all(), f"{what}: guard written"
            for lb in lbufs:
                assert (lb[:GUARD // 8] == LSENT).all() and (lb[-(GUARD // 8):] == LSENT).all(), what
    # a failing padded batch (request 7) ahead of an all-invalid one: wait() reports the first
    made = [kinds["padded raw"](0), padded("f32x3", 6, 4, 300, bad_at=7)(1), kinds["padded all-invalid"](0),
            kinds["multi converting"](1)]
    for launch, _, _, _ in made:
        launch(side.cuda_stream)
    with pytest.raises(ValueError):
        store.wait()
    assert store.last_bad_index == 7
    made[2][1]("failing queue, batch 2")  # (the last users of the two buffers)
    made[3][1]("failing queue, batch 3")


def part_4gib(ctx):
    """three batches past 4 GiB: first and last slots, slots on both sides of output and source byte 2^32, lengths and
    the trailing guard; the memory is freed after each"""
    import torch
    store, rng, dev = ctx.store, ctx.rng, ctx.dev
    cases = [("u8x4097", 10, 300, 900), ("f32x1025", 1, 1000, 1100), ("f64x513", 9, 1000, 1100)]
    for var, code, mr, n in cases:
        dt, disp, nrows = ps.VARS[var]
        rb = disp * np.dtype(dt).itemsize
        i_el, o_el = ps.CVT_IO[code]
        s_src, s_out = mr * rb, mr * disp * o_el
        s, c = rng.integers(0, nrows - 1, n), rng.integers(0, mr + 2, n)
        c = np.minimum(c, nrows - s)
        c[0], c[-1] = 0, min(mr, nrows - s[-1])
        nbytes = n * s_out
        assert nbytes > 1 << 32 or n * s_src > 1 << 32
        sdt, odt, nz, lut, pad = ctx.cv[code]
        whole = torch.full((nbytes + 2 * GUARD,), SENT, dtype=torch.uint8, device=dev)
        lens = torch.full((n,), LSENT, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        total = store.get_batch(var, torch.as_tensor(s, device=dev), torch.as_tensor(c, device=dev),
                                out=whole[GUARD:GUARD + nbytes].view(odt), src_dtype=sdt, lut=lut, normalize=nz,
                                pad_rows=mr, pad_value=pad, lengths=lens)
        torch.cuda.synchronize()
        what = f"4 GiB {var} code={code} ({n} slots of {s_out} output / {s_src} source bytes)"
        assert total == nbytes, what
        valid = np.ones(n, bool)
        assert lens.cpu().numpy().tolist() == np.minimum(c, mr).tolist(), f"{what}: lengths"
        pick = {0, 1, n - 2, n - 1}
        for x, sz in ((1 << 32, s_out), (1 << 32, s_src)):
            j = x // sz
            pick |= {k for k in (j - 1, j, j + 1) if 0 <= k < n}
        for j in sorted(pick):
            exp = expected(ctx, var, code, s[j:j + 1], c[j:j + 1], mr, valid[j:j + 1])
            got = whole[GUARD + j * s_out:GUARD + (j + 1) * s_out].cpu().numpy()
            compare(ctx, got, exp, f"{what}, slot {j}", s[j:j + 1], c[j:j + 1], valid[j:j + 1], mr, disp)
        assert (whole[:GUARD] == SENT).all() and (whole[GUARD + nbytes:] == SENT).all(), f"{what}: guard written"
        del whole, lens
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def world_body(store, r, peer=False):
    """three owners of a float32 variable (6 columns, 300 rows each): converting and normalising padded batches"""
    import torch
    disp, per = 6, 300
    g = np.random.default_rng(100)
    allrows = g.integers(0, 256, size=3 * per * disp * 4, dtype=np.uint8).view(np.float32).reshape(3 * per, disp)
    store.add("w", allrows[r * per:(r + 1) * per].copy())
    mean, std = np.array([0.5, -1.0, 2.0], np.float32), np.array([0.25, 0.0, -3.0], np.float32)
    store.set_normalization("w", mean, std, inner=2)
    dev = torch.device("cuda", r if peer else 0)
    rng = np.random.default_rng(r)
    mr = 7
    s, c = rng.integers(0, 3 * per - 8, 400), rng.integers(0, 9, 400)
    s[:4] = [per - 5, per, 2 * per - 1, 2 * per]  # ending on an owner's last row, starting on the next's first
    c[:4] = [5, 7, 1, 3]
    s[4], c[4] = per - 2, 5                                   # crossing owners: all padding, length 0, an error
    ll = np.array(store.query("w")["lenlist"])
    owner = np.searchsorted(ll, s, side="right")
    valid = (c >= 0) & (s + c <= ll[np.minimum(owner, 2)])
    assert not valid[4] and valid[:4].all()
    take = np.where(valid, np.minimum(c, mr), 0)
    packed = np.concatenate([allrows[a:a + n].reshape(-1) for a, n in zip(s, take) if n > 0])
    x = torch.from_numpy(packed).to(dev)
    ch = no.channels(disp, 3, 2)
    exprs = {(torch.bfloat16, False): lambda t: t.to(torch.bfloat16),
             (torch.float16, True): lambda t: ((t.view(-1, disp) - torch.from_numpy(mean[ch]).to(dev))
                                               / torch.from_numpy(std[ch]).to(dev)).to(torch.float16)}
    for (odt, nz), f in exprs.items():
        ob = f(x).reshape(-1).view(torch.int16).cpu().numpy().view(np.uint16)
        exp, lens = po.pad_rows(ob, take, disp, mr, np.uint16(0xFF80 if odt == torch.bfloat16 else NAN_F16), valid)
        out = torch.full((400 * mr * disp,), 0, dtype=odt, device=dev)
        ln = torch.full((400,), LSENT, dtype=torch.int64, device=dev)
        pv = torch.tensor([-128 if odt == torch.bfloat16 else NAN_F16], dtype=torch.int16).view(odt)
        with pytest.raises(ValueError):
            store.get_batch("w", s, c, out=out, src_dtype=torch.float32, normalize=nz, pad_rows=mr, pad_value=pv, lengths=ln)
        assert store.last_bad_index == 4
        got = out.view(torch.int16).cpu().numpy().view(np.uint16).reshape(exp.shape)
        d = np.argwhere(got != exp)
        assert d.size == 0, f"rank {r} {odt}: slot {d[0][0]} row {d[0][1]} element {d[0][2]} differs"
        assert ln.cpu().numpy().tolist() == lens.tolist()
    return True


def sweep_main(parts=("sweep", "entries", "queues", "4gib", "world")):
    import torch
    from ddstore_b200 import PyDDStore
    env = os.environ
    cfg = " ".join(f"{k}={v}" for k, v in sorted(env.items()) if k.startswith("DDS_") and k != "DDS_COMM_TIMEOUT_S") or "default"
    t0 = time.time()

    def phase(what):
        print(f"[{cfg}] {what} done at {time.time() - t0:.1f} s", flush=True)

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nwarps = ps.WARPS_PER_SM * sms
    rng = np.random.default_rng(2026)
    store = PyDDStore(device=0)
    ctx = Ctx(torch, store, rng)
    tabs = {}
    for var in ps.VARS:
        ctx.add(var)
        default_norm(ctx, var)
    for var in ("u8x3", "f32x3", "f32x5", "f64x3", "tok"):  # sample tables (one length for the multi-array pair)
        nrows = ps.VARS[var][2]
        c = rng.integers(0, 12, 2000)
        s = rng.integers(0, nrows - 12, 2000)
        tabs[var] = (s.astype(np.int64), c.astype(np.int64))
        store.set_sample_index(var, tabs[var][0], tabs[var][1])
    phase("setup")
    if "sweep" in parts:
        part_sweep(ctx, nwarps, phase)
    if "entries" in parts:
        part_entries(ctx, tabs)
        phase("entries")
    if "queues" in parts:
        part_queues(ctx, tabs)
        phase("queues")
    if "4gib" in parts:
        part_4gib(ctx)
        phase("4 GiB")
    torch.cuda.synchronize()
    store.free()
    store.close()
    if "world" in parts:
        assert run_world(3, world_body) == [True] * 3
        if torch.cuda.device_count() >= 3:
            assert run_world(3, lambda st, r: world_body(st, r, peer=True), devices=[0, 1, 2]) == [True] * 3
        phase("world")


SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_pad_sweep import sweep_main
sweep_main()
print("pad-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_pad_sweep(tmp_path, config):
    """the padded sweep with the environment of `config`: slots, lengths, totals, errors and guard bands against the
    host reference"""
    script = tmp_path / "pad_sweep.py"
    script.write_text(SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "pad-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]
