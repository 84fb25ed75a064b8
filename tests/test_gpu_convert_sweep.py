"""The converting gather (dds_get_batch_convert & co.) on the variant sweep's adversarial workload (-m gpu).

tests/test_gpu_convert.py checks every conversion on one small odd row shape per source type. This module runs the
converted drain where it can go wrong: requests from 1 byte to 5 MiB (tests/gpu_helpers.sweep_requests for the chunk
sizes 4096 and 3072 of the four converting instantiations), so pieces are cut at the chunk, at fixed-count segments
inside a request and at variable-count segment boundaries; rows smaller than one 16-byte output vector (1, 3 and 5
elements), rows whose output is a multiple of 16 bytes (1024 f32, 512 f64) and rows next to them (1025 f32, 513 f64,
4097 u8), into destinations at
every base offset the output itemsize allows within 0..15, so every head length of the drain occurs; multi-array
batches whose converted variables start at odd offsets behind a raw uint8 variable (the VALIGN segment walk-back)
and that mix 2- and 4-byte tables; and overlapped queues that mix converted and raw batches of every plan placement,
each batch in its own guarded buffer, with the wait() total checked after queue orders that end in every hand-over
of the total word. Each configuration runs in a subprocess of its own with the environment it names.

Reference: the oracle's packed raw bytes -> tests/convert_oracle.convert_bytes, compared by NaN class; for float
sources also bitwise torch's CUDA `.to()` of the same raw bytes. Offsets are the oracle's in output bytes, the total is
the packed output size, and the 64-byte sentinel bands on both sides of every destination stay untouched. Payload is
random bits (NaN, +-inf, subnormals, -0 all occur); the first rows of every float32 variable hold
convert_oracle.F32_EDGE_BITS and of every float64 variable convert_oracle.f64_edge_bits(), and one request of every
workload covers them.

On an H100 80GB HBM3 (700 W power limit) the module takes about 150 s: about 30 s per configuration.
"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import convert_oracle as co
from tests.gpu_helpers import GUARD, guarded_buffer, padded_requests, sample_ids, sweep_requests

# Every device buffer or index array a test prepares on torch's stream is complete (torch.cuda.synchronize) before a
# store call that has no `stream` argument reads or writes it: the store's own stream is not ordered with torch's.

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = {"default": {},
           "smem8192": {"DDS_SMEM_PLAN_MAX": "8192"},  # 4097..8192 requests on the 12 x 3 x 3072 shared-memory plan
           "plankernels": {"DDS_SMEM_PLAN": "0"},       # every variable-count batch planned by dds_plan_kernel
           "minseg1": {"DDS_VAR_MINSEG": "1", "DDS_S_MINSEG": "1"},
           "nopdl": {"DDS_PDL": "0"}}
CHUNKS = (4096, 3072)  # chunk sizes of the converting instantiations (the 8192-request shared plan uses 3072)

# name -> (numpy dtype, disp, rows): every shard holds the 5 MiB requests of sweep_requests
VARS = {"u8x1": (np.uint8, 1, 6 << 20), "u8x3": (np.uint8, 3, 2 << 20), "u8x4097": (np.uint8, 4097, 1600),
        "f32x1": (np.float32, 1, 3 << 19), "f32x3": (np.float32, 3, 1 << 19), "f32x5": (np.float32, 5, 300_000),
        "f32x1024": (np.float32, 1024, 1600), "f32x1025": (np.float32, 1025, 1600),
        "f64x1": (np.float64, 1, 3 << 18), "f64x3": (np.float64, 3, 1 << 18), "f64x512": (np.float64, 512, 1600),
        "f64x513": (np.float64, 513, 1600)}
MID, BIG = 6000, 9000

# multi-array combinations: (variable, conversion label or None for raw bytes)
MULTI = [[("u8x1", None), ("f32x3", "bf16"), ("f64x3", "f32"), ("u8x4097", "lut32")],   # odd raw u8 first
         [("u8x3", None), ("f64x513", "f32"), ("f32x1025", "f16"), ("u8x1", "lut16-bf16")],
         [("u8x3", "lut16-f16-default"), ("u8x4097", "lut32"), ("f32x1", "bf16")],    # 2- and 4-byte tables
         [("f32x1024", "f16"), ("f64x512", "f32"), ("u8x1", "lut32")]]


def _conversions(torch):
    """numpy source dtype -> [(label, torch source dtype, output dtype, table or None, code)]"""
    x = torch.arange(256, dtype=torch.float32)
    return {np.uint8: [("lut16-bf16", torch.uint8, torch.bfloat16, ((x - 127.5) / 60.1).to(torch.bfloat16), co.CVT_U8_LUT16),
                       ("lut16-f16-default", torch.uint8, torch.float16, None, co.CVT_U8_LUT16),
                       ("lut32", torch.uint8, torch.float32, x / 255 - 0.25, co.CVT_U8_LUT32)],
            np.float32: [("bf16", torch.float32, torch.bfloat16, None, co.CVT_F32_BF16),
                         ("f16", torch.float32, torch.float16, None, co.CVT_F32_F16)],
            np.float64: [("f32", torch.float64, torch.float32, None, co.CVT_F64_F32)]}


def dst_offsets(code):
    """every destination base offset within 0..15 the output itemsize allows (raw bytes: a spread of odd and even)"""
    return [1, 13, 0, 6] if code == co.CVT_NONE else [o for o in range(0, 16, co.SIZES[code][1])]


def edge_rows(dt, disp):
    """the rounding-edge rows stored at the start of a float variable (None for uint8)"""
    if dt == np.float32:
        vals = np.array(co.F32_EDGE_BITS, np.uint32)
    elif dt == np.float64:
        vals = co.f64_edge_bits()
    else:
        return None
    n = -(-len(vals) // disp)
    return np.resize(vals, n * disp).reshape(n, disp).view(dt)


class Ref:
    """What a converted (or raw: conv None) delivery of packed raw bytes `raw` with byte offsets `eo` must be: `dev`, the
    expected output bytes on the device; `eo` / `d_eo`, the expected output byte offsets on the host / device"""

    def __init__(self, torch, raw, eo, conv, starts, counts):
        self.starts, self.counts = starts, counts
        raw = np.ascontiguousarray(raw, np.uint8)
        dev = torch.device("cuda", 0)
        if conv is None:
            self.code, self.odt = co.CVT_NONE, torch.uint8
            self.dev = torch.from_numpy(raw).to(dev)
        else:
            label, sdt, odt, lut, code = conv
            self.code, self.odt = code, odt
            table = None
            if code in (co.CVT_U8_LUT16, co.CVT_U8_LUT32):
                table = (torch.arange(256).to(odt) if lut is None else lut).contiguous().view(torch.uint8).numpy()
            exp_np = co.convert_bytes(raw, code, table)
            if table is not None or raw.size == 0:
                self.dev = torch.from_numpy(exp_np).to(dev)
            else:  # torch's CUDA cast of the raw bytes, which must also be the oracle's up to NaN payloads
                self.dev = torch.from_numpy(raw).to(dev).view(sdt).to(odt).view(torch.uint8).reshape(-1)
                bad = co.same_bits_or_both_nan(self.dev.cpu().numpy(), exp_np, code)
                assert bad.size == 0, f"torch's cast and the NumPy oracle differ at element {int(bad[0])} ({label})"
        i, o = co.SIZES[self.code]
        self.osz = o
        self.eo = (np.asarray(eo, np.int64) // i) * o
        self.d_eo = torch.from_numpy(self.eo).to(dev)
        self.n = self.dev.numel()


def report(ref, whole, off, sent, what, total, d_offs):
    """the first discrepancy of a delivery, named by request (start, count), element inside it and destination phase"""
    w = whole.cpu().numpy()
    base, n = GUARD + off, ref.n
    msgs = []
    if total is not None and total != n:
        msgs.append(f"returned total {total}, expected {n}")
    if d_offs is not None:
        go = d_offs.cpu().numpy()[:len(ref.eo)]
        d = np.nonzero(go != ref.eo)[0]
        if d.size:
            i = int(d[0])
            req = f" (request start={int(ref.starts[i])}, count={int(ref.counts[i])})" if i < len(ref.starts) else ""
            msgs.append(f"{d.size} offsets differ; offsets[{i}] = {int(go[i])}, expected {int(ref.eo[i])}{req}")
    pre = np.nonzero(w[:base] != sent)[0]
    if pre.size:
        msgs.append(f"byte {int(pre[-1]) - base} (before the destination base) was written")
    post = np.nonzero(w[base + n:] != sent)[0]
    if post.size:
        msgs.append(f"byte {n + int(post[0])} (past the packed end, {n}) was written")
    dt = {1: np.uint8, 2: np.uint16, 4: np.uint32}[ref.osz]
    got, exp = w[base:base + n].view(dt), ref.dev.cpu().numpy().view(dt)
    bad = np.flatnonzero(got != exp)
    if bad.size:
        e = int(bad[0])
        pos = e * ref.osz
        r = int(np.searchsorted(ref.eo, pos, side="right") - 1)
        reqs = np.unique(np.searchsorted(ref.eo, bad * ref.osz, side="right") - 1)
        msgs.append(f"{bad.size} elements in {reqs.size} requests differ; first: element {(pos - int(ref.eo[r])) // ref.osz} "
                    f"of request {r} (start={int(ref.starts[r])}, count={int(ref.counts[r])}, output offset "
                    f"{int(ref.eo[r])}, {int(ref.eo[r + 1] - ref.eo[r]) // ref.osz} elements; destination phase "
                    f"{(off + pos) % 16}): got {int(got[e]):#x}, expected {int(exp[e]):#x}")
    return f"{what}: " + ("; ".join(msgs) if msgs else "mismatch (not found on the host)")


def check(torch, ref, whole, off, sent, what, total=None, d_offs=None):
    base = GUARD + off
    ok = (total is None or total == ref.n) and torch.equal(whole[base:base + ref.n], ref.dev)
    ok = ok and bool((whole[:base] == sent).all()) and bool((whole[base + ref.n:] == sent).all())
    ok = ok and (d_offs is None or torch.equal(d_offs[:ref.d_eo.numel()], ref.d_eo))
    if not ok:
        raise AssertionError(report(ref, whole, off, sent, what, total, d_offs))


def convert_sweep_main(parts=("single", "multi", "queues")):
    """One configuration (taken from the environment) end to end, or only some `parts` of it; raises on the first
    discrepancy."""
    import torch
    from ddstore_b200 import PyDDStore, _capi
    from oracle.oracle import COracle
    env = os.environ
    cfg = " ".join(f"{k}={v}" for k, v in sorted(env.items()) if k.startswith("DDS_") and k != "DDS_COMM_TIMEOUT_S") or "default"
    dev = torch.device("cuda", 0)
    coracle = COracle()
    rng = np.random.default_rng(20261)
    store = PyDDStore(device=0)
    convs = _conversions(torch)
    conv_by = {(dt, c[0]): c for dt, cs in convs.items() for c in cs}
    t0 = time.time()

    def phase(what):
        print(f"[{cfg}] {what} done at {time.time() - t0:.1f} s", flush=True)

    shards, base = {}, {}
    for name, (dt, disp, n) in VARS.items():
        isz = np.dtype(dt).itemsize
        sh = rng.integers(0, 256, size=n * disp * isz, dtype=np.uint8).view(dt).reshape(n, disp)
        edge = edge_rows(dt, disp)
        st, ct = sweep_requests(rng, n, disp * isz, CHUNKS)
        if edge is not None:
            sh[:len(edge)] = edge
            st, ct = np.insert(st, 1, 0), np.insert(ct, 1, len(edge))  # one request covers the edge rows
        shards[name] = sh
        store.add(name, sh)
        base[name] = (st, ct)
        store.set_sample_index(name, st, ct)

    def oracle(name, st, ct):
        exp, exp_offs, bad, _ = coracle.get_batch([shards[name]], st, ct)
        assert bad == -1, (name, bad)
        return exp, exp_offs

    ncall = [0]

    def sentinel():
        ncall[0] += 1
        return (0xA5, 0x3C)[ncall[0] & 1]

    def idx(a, on_dev):
        if not on_dev:
            return a
        t = torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(dev)
        torch.cuda.synchronize()
        return t

    def run(ref, what, call):
        """call(out_view, offsets_tensor, idx_on_device) -> returned total; device indices into every allowed base
        offset, host indices into the first and the last"""
        offs = dst_offsets(ref.code)
        for idx_dev in (False, True):
            for off in (offs if idx_dev else (offs[0], offs[-1])):
                sent = sentinel()
                d_offs = torch.full((len(ref.starts) + 1,), -7, dtype=torch.int64, device=dev)
                whole, view = guarded_buffer(torch, ref.n + GUARD, off, sent)  # (synchronizes)
                total = call(view.view(ref.odt), d_offs, idx_dev)
                check(torch, ref, whole, off, sent, f"[{cfg}] {what} idx_dev={idx_dev} dst+{off}", total=total, d_offs=d_offs)

    # ---- single-variable entries
    for name, (dt, disp, n) in (VARS.items() if "single" in parts else ()):
        row = disp * np.dtype(dt).itemsize
        work = []
        for cnt, nreq in ((1, 3000), (4096 // row + 1, 200)):  # one row; the count that first exceeds one chunk
            st = rng.integers(0, n - cnt + 1, size=nreq).astype(np.int64)
            st[0] = 0
            work.append((f"get_batch count={cnt}", st, np.full(nreq, cnt, np.int64), cnt))
        mc = 2 if row < 1024 else 1
        bst, bct = base[name]
        for label, (st, ct) in (("var", base[name]), ("var-mid", padded_requests(rng, n, bst, bct, MID, mc)),
                                ("var-big", padded_requests(rng, n, bst, bct, BIG, mc))):
            work.append((f"get_batch {label}", st, ct, None))
        for nid in (500, BIG):
            ids = sample_ids(rng, bct * row, nid)
            work.append(("get_samples", bst[ids], bct[ids], ids))
        for what, st, ct, extra in work:
            raw, eo = oracle(name, st, ct)
            for conv in convs[dt]:
                ref = Ref(torch, raw, eo, conv, st, ct)
                kw = dict(src_dtype=conv[1], lut=conv[3])
                w = f"{name} -> {conv[0]} {what} ({len(st)} requests)"
                if what.startswith("get_batch count"):
                    run(ref, w, lambda v, o, d: store.get_batch(name, idx(st, d), out=v, count=extra, offsets=o, **kw))
                elif what.startswith("get_batch"):
                    run(ref, w, lambda v, o, d: store.get_batch(name, idx(st, d), idx(ct, d), out=v, offsets=o, **kw))
                else:
                    run(ref, w, lambda v, o, d: store.get_samples(name, idx(extra, d), v, offsets=o, **kw))
        phase(name)
        # nothing to deliver: a fixed count of 0, and explicit counts that are all 0 -- total 0, nothing written
        st = rng.integers(0, n, size=50).astype(np.int64)
        zero = np.zeros(50, np.int64)
        for conv in convs[dt]:
            ref = Ref(torch, np.zeros(0, np.uint8), np.zeros(51, np.int64), conv, st, zero)
            kw = dict(src_dtype=conv[1], lut=conv[3])
            run(ref, f"{name} -> {conv[0]} get_batch count=0",
                lambda v, o, d: store.get_batch(name, idx(st, d), out=v, count=0, offsets=o, **kw))
            run(ref, f"{name} -> {conv[0]} get_batch all-zero counts",
                lambda v, o, d: store.get_batch(name, idx(st, d), idx(zero, d), out=v, offsets=o, **kw))

    # ---- multi-array batches
    def multi_ids(names, nid, odd_first):
        ns = min(len(base[nm][0]) for nm in names)
        worst = np.max([base[nm][1][:ns] * VARS[nm][1] * np.dtype(VARS[nm][0]).itemsize for nm in names], axis=0)
        ids = sample_ids(rng, worst, nid)
        if odd_first:  # the first (raw uint8) variable packs an odd number of bytes: the next ones start at odd offsets
            c0 = base[names[0]][1][:ns] * VARS[names[0]][1]
            if int(c0[ids].sum()) % 2 == 0:
                j = int(np.nonzero(c0[ids] % 2 == 0)[0][0])
                ids[j] = int(np.nonzero(c0 % 2 == 1)[0][0])
            assert int(c0[ids].sum()) % 2 == 1
        return ids

    def multi_refs(combo, ids):
        refs = []
        for nm, lab in combo:
            st, ct = base[nm][0][ids], base[nm][1][ids]
            raw, eo = oracle(nm, st, ct)
            refs.append(Ref(torch, raw, eo, None if lab is None else conv_by[(VARS[nm][0], lab)], st, ct))
        return refs

    def multi_kw(combo):
        cs = [None if lab is None else conv_by[(VARS[nm][0], lab)] for nm, lab in combo]
        return dict(src_dtypes=[c and c[1] for c in cs], luts=[c and c[3] for c in cs])

    for combo in (MULTI if "multi" in parts else ()):
        names = [nm for nm, _ in combo]
        for nid in (300, 2000, 3000):
            ids = multi_ids(names, nid, combo[0][1] is None and VARS[names[0]][0] == np.uint8)
            refs = multi_refs(combo, ids)
            for idx_dev in (False, True):
                for k in (range(8) if idx_dev else (0, 7)):
                    offs = [dst_offsets(r.code)[(k + v) % len(dst_offsets(r.code))] for v, r in enumerate(refs)]
                    sent = sentinel()
                    d_offs = [torch.full((nid + 1,), -7, dtype=torch.int64, device=dev) for _ in refs]
                    bufs = [guarded_buffer(torch, r.n + GUARD, o, sent) for r, o in zip(refs, offs)]
                    totals = store.get_samples_multi(names, idx(ids, idx_dev), [b[1].view(r.odt) for b, r in zip(bufs, refs)],
                                                     offsets=d_offs, **multi_kw(combo))
                    for (nm, lab), (whole, _), r, o, f, t in zip(combo, bufs, refs, offs, d_offs, totals):
                        check(torch, r, whole, o, sent, f"[{cfg}] get_samples_multi {combo} {nid} ids, {nm} -> {lab} "
                              f"idx_dev={idx_dev} dst+{o}", total=t, d_offs=f)

    phase("multi-array batches")

    # ---- overlapped queues (DDS_NO_SYNC | DDS_OVERLAP) on a side stream, every batch in a guarded buffer of its own
    side, other = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)

    def single(kind, name, lab, nreq):
        """one queued batch of variable `name` (lab: conversion label, None: raw) -> (launch(stream), checks, total)"""
        dt, disp, n = VARS[name]
        conv = None if lab is None else conv_by[(dt, lab)]
        bst, bct = base[name]
        if kind == "fixed":
            st = rng.integers(0, n - 2, size=nreq).astype(np.int64)
            ct = np.full(nreq, 2, np.int64)
        elif kind == "var":
            st, ct = padded_requests(rng, n, bst, bct, nreq, 2) if nreq > len(bst) else (bst[:nreq], bct[:nreq])
        else:
            ids = sample_ids(rng, bct * disp * np.dtype(dt).itemsize, nreq)
            st, ct = bst[ids], bct[ids]
            d_ids = idx(ids, True)
        raw, eo = oracle(name, st, ct)
        ref = Ref(torch, raw, eo, conv, st, ct)
        off = dst_offsets(ref.code)[-1]
        sent = sentinel()
        whole, view = guarded_buffer(torch, ref.n + GUARD, off, sent)
        d_offs = torch.full((len(st) + 1,), -7, dtype=torch.int64, device=dev)
        d_st, d_ct = idx(st, True), idx(ct, True)
        o = view.view(ref.odt)
        kw = dict(offsets=d_offs, wait=False, overlap=True)
        if conv is not None:
            kw.update(src_dtype=conv[1], lut=conv[3])
        what = f"{name} -> {lab} {kind} ({nreq} requests)"
        if kind == "fixed":
            launch = lambda s: store.get_batch(name, d_st, out=o, count=2, stream=s, **kw)  # noqa: E731
        elif kind == "var":
            launch = lambda s: store.get_batch(name, d_st, d_ct, out=o, stream=s, **kw)  # noqa: E731
        else:
            launch = lambda s: store.get_samples(name, d_ids, o, stream=s, **kw)  # noqa: E731
        return launch, [(ref, whole, off, sent, d_offs, what)], ref.n

    def multi(ci, nid):
        combo = MULTI[ci]
        names = [nm for nm, _ in combo]
        ids = multi_ids(names, nid, combo[0][1] is None)
        refs = multi_refs(combo, ids)
        sent = sentinel()
        offs = [dst_offsets(r.code)[-1] for r in refs]
        bufs = [guarded_buffer(torch, r.n + GUARD, o, sent) for r, o in zip(refs, offs)]
        d_offs = [torch.full((nid + 1,), -7, dtype=torch.int64, device=dev) for _ in refs]
        d_ids = idx(ids, True)
        outs = [b[1].view(r.odt) for b, r in zip(bufs, refs)]
        kw = multi_kw(combo)
        launch = lambda s: store.get_samples_multi(names, d_ids, outs, offsets=d_offs, stream=s, wait=False,  # noqa: E731
                                                   overlap=True, **kw)
        checks = [(r, b[0], o, sent, f, f"multi {combo} ({nid} ids), {nm}")
                  for r, b, o, f, nm in zip(refs, bufs, offs, d_offs, names)]
        return launch, checks, sum(r.n for r in refs)

    Fc = lambda: single("fixed", "f32x3", "bf16", 4000)                       # noqa: E731  converted, fixed count
    Fr = lambda: single("fixed", "f32x3", None, 4000)                         # noqa: E731  raw, fixed count
    Vbig = lambda: single("var", "f64x3", "f32", BIG)                         # noqa: E731  plan kernels in a slot
    Vsmall_c = lambda: single("var", "f32x5", "f16", 800)                     # noqa: E731  shared-memory plan
    Vsmall_r = lambda: single("var", "f32x5", None, 800)                      # noqa: E731
    Sc = lambda: single("samples", "u8x3", "lut16-bf16", 700)                 # noqa: E731
    Sr = lambda: single("samples", "u8x3", None, 700)                         # noqa: E731
    Mbig = lambda: multi(0, 3000)                                             # noqa: E731  plan kernels, VALIGN walk-back
    Msmall = lambda: multi(0, 200)                                            # noqa: E731  shared-memory plan
    queues = {"large multi, then a small converted shared-plan batch": [Fc, Fr, Vbig, Sc, Mbig, Vsmall_c],
              "large multi, then a small raw shared-plan batch": [Vbig, Fr, Mbig, Vsmall_r],
              "two converted multi-array batches": [Sc, Vbig, Mbig, Msmall],
              "raw, then converted": [Mbig, Fc, Vbig, Fr, Sr, Vsmall_c],
              "converted, then raw": [Fr, Sc, Mbig, Vsmall_c, Vbig, Sr]}
    for contention in ((False, True) if "queues" in parts else ()):
        for qname, makers in queues.items():
            if contention and not qname.startswith("large multi, then a small converted"):
                continue
            batches = [mk() for mk in makers]
            torch.cuda.synchronize()
            if contention:  # a kernel holding most SMs' shared memory on another stream
                _capi.raise_for(_capi.lib().dds_test_occupy(0, 100, 200 * 1024, 2_000_000, C.c_void_p(other.cuda_stream)))
            for launch, _, _ in batches:
                launch(side.cuda_stream)
            total = store.wait()
            torch.cuda.synchronize()
            what = f"[{cfg}] overlapped queue '{qname}' contention={contention}"
            assert total == batches[-1][2], f"{what}: wait() returned {total}, the last batch packs {batches[-1][2]}"
            for k, (_, checks, _) in enumerate(batches):
                for ref, whole, off, sent, d_offs, w in checks:
                    check(torch, ref, whole, off, sent, f"{what}, batch {k}: {w}", d_offs=d_offs)
    phase("overlapped queues")
    torch.cuda.synchronize()
    store.free()
    store.close()


SWEEP_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r})
from tests.test_gpu_convert_sweep import convert_sweep_main
convert_sweep_main()
print("convert-sweep-ok")
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_convert_sweep(tmp_path, config):
    """every conversion through every entry on the sweep workload, multi-array batches and overlapped queues, with the
    environment of `config`: elements, offsets, totals and guard bands against the oracle"""
    script = tmp_path / "convert_sweep.py"
    script.write_text(SWEEP_SCRIPT.format(root=ROOT))
    env = {k: v for k, v in os.environ.items() if not k.startswith("DDS_") or k == "DDS_COMM_TIMEOUT_S"}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "convert-sweep-ok" in r.stdout, (r.stdout + r.stderr)[-6000:]
