"""The pooled get (dds_pool_kernel) and its adjoint (dds_pool_acc_kernel) in every launch geometry their launchers
select, against tests/pool_oracle.py and tests/pool_acc_oracle.py.

The launchers pick, per call, the lane vector (16 bytes or one element), the column slice (32 vectors, which the get
halves down to 128 bytes while its units leave resident warps idle), the adjoint's row windows W per bag (1 to 32) and
the grid, which warps stride over when it is smaller than the units. CLASSES names one geometry class per row. For each
row, the test asks dds_pool_geometry -- the launchers' own rule -- for the smallest number of bags that lands in the
class on this device. It asserts the class before it launches. A class the launchers can no longer reach fails by name.
So the module holds on any SM count and after any retuning of the kPool* constants.

Forward classes are checked bit for bit against the oracle: every type; sum, weighted sum, mean and max; inexact values
with NaNs, infinities, subnormals and signed zeros; outputs 16-byte aligned or one element past that; mixed bag sizes
(0, 1, 31, 32, 33 and 300 requests) or one bag per request for the many-bag classes; invalid requests in strided units;
HOST shards against an HBM twin, and on one CTA (DDS_HOST_CTAS=1, in a child process). Adjoint classes are checked where
every row is touched at most once, against acc_oracle's admissible results (the f32 flush model included), for W = 1, 2,
8, 31 and 32, with bags whose row totals are W - 1, W, W + 1 and one bag spanning several 32-request chunks whose totals
are not multiples of W; exact data with duplicate rows is checked at W = 1 and W > 1. The benchmarked shapes are here at
test scale: emb32 (128 x f32, bags of 32 one-row requests, strided forward sum, W = 1 adjoint) and frames (80 x f32, one
long sample per bag, mean).

Every class is reachable whatever the SM count but one: W = 31 takes a unit count in [4 r / 31, 4 r / 30) for r resident
warps (16 per SM), a range 64 * SMs / 930 wide, which is sure to hold an integer from 15 SMs up (132-SM H100 SXM: 273 to
281 units; 114-SM H100 PCIe: 236 to 243).
"""
import os
import subprocess
import sys

import ctypes as C
import numpy as np
import pytest

from tests import acc_oracle as ao
from tests import pool_acc_oracle as pao
from tests import pool_oracle as pl
from tests.test_gpu_pool import SIZE, TORCH_DT, add_var, bits_of, check, data_bits
from tests.test_gpu_pool import call as pool_call
from tests.test_gpu_pool_acc import call as acc_call
from tests.test_gpu_pool_acc import check_touched_once, grad_tensor, shard_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64, F16, BF16 = pl.ACC_F32, pl.ACC_F64, pl.ACC_F16, pl.ACC_BF16
MODES = {"sum": pl.POOL_SUM, "weighted": pl.POOL_SUM, "mean": pl.POOL_MEAN, "max": pl.POOL_MAX}
WARPS_PER_CTA = 8  # (256-thread CTAs)
MIXED = [0, 1, 31, 32, 33, 300]  # requests per bag of the few-bag forward classes
NBAGS_MAX = 40000


# ----------------------------------------------------------------------------------------- the launchers' geometry
def geometry(adjoint, row_bytes, t, nbags, aligned, host=False):
    """dds_pool_geometry -> (vb, slice, nslices, windows, ctas)"""
    from ddstore_b200 import _capi
    vb, ctas = C.c_int(), C.c_int()
    sl, ns, w = C.c_int64(), C.c_int64(), C.c_int64()
    _capi.lib().dds_pool_geometry(int(adjoint), row_bytes, t, nbags, int(aligned), int(host), C.byref(vb), C.byref(sl),
                                  C.byref(ns), C.byref(w), C.byref(ctas))
    return vb.value, sl.value, ns.value, w.value, ctas.value


def classify(row_bytes, nbags, g):
    vb, sl, ns, w, ctas = g
    units, warps = nbags * ns * w, ctas * WARPS_PER_CTA
    return {"vb": 16 if vb == 16 else "elem", "slice": "full" if sl == 32 * vb else "narrowed",
            "partial": ns > 1 and row_bytes % sl != 0, "stride": units > warps, "per_warp": units // warps,
            "W": w, "nslices": ns}


def matches(cls, want):
    for k, v in want.items():
        if k == "per_warp" and cls[k] < v:
            return False
        if k == "nslices" and cls[k] < v:
            return False
        if k not in ("per_warp", "nslices") and cls[k] != v:
            return False
    return True


def shape_of(c):
    """(nbags, geometry, class) of class row c: the fewest bags (from c's floor) that land in its class"""
    R = c["disp"] * SIZE[c["t"]]
    lo, hi = c.get("nbags", (1, NBAGS_MAX))
    for n in range(lo, hi + 1):
        g = geometry(c["adjoint"], R, c["t"], n, c["off"] == 0, c.get("host", False))
        assert g[0] > 0, "dds_pool_geometry reports no device"
        cls = classify(R, n, g)
        if matches(cls, c["want"]):
            return n, g, cls
    pytest.fail(f"geometry class {c['id']} ({c['want']}) is not reachable with {lo}..{hi} bags of {R}-byte rows "
                f"on this device: the launchers' rule changed")


def F(id, t, disp, want, kind, off=0, modes=("sum", "weighted", "mean", "max"), host=False, nbags=None, **kw):
    c = dict(id=id, adjoint=False, t=t, disp=disp, want=want, kind=kind, off=off, modes=modes, host=host, **kw)
    if nbags is not None:
        c["nbags"] = nbags
    return c


def A(id, t, disp, want, kind, off=0, modes=("sum", "weighted", "mean"), nbags=None, **kw):
    c = dict(id=id, adjoint=True, t=t, disp=disp, want=want, kind=kind, off=off, modes=modes, **kw)
    if nbags is not None:
        c["nbags"] = nbags
    return c


N6 = (len(MIXED), len(MIXED))
# One row per geometry class. want: vb (16 / "elem"), slice ("full" = 32 vectors / "narrowed"), partial (the last slice
# has idle lanes), stride (units > the grid's warps), per_warp (units per warp, at least), nslices (at least), W.
# (A narrowed get never has twice as many units as the grid has warps: the slices stop halving once the units reach the
# resident warps. Its strided classes stride only their last units; the full-slice ones stride every warp at least
# once.)
CLASSES = [
    # forward, few bags: narrowed slices
    F("fwd-f32-v16-narrowed", F32, 128, dict(vb=16, slice="narrowed", partial=False, stride=False, nslices=2), "mixed",
      nbags=N6),
    F("fwd-bf16-v16-narrowed-partial", BF16, 72, dict(vb=16, slice="narrowed", partial=True, stride=False), "mixed",
      nbags=N6),
    F("fwd-f64-elem-narrowed-partial", F64, 33, dict(vb="elem", slice="narrowed", partial=True, stride=False), "mixed",
      nbags=N6),
    F("fwd-f16-elem-offset-full-partial", F16, 200, dict(vb="elem", slice="full", partial=True, stride=False), "mixed",
      off=1, nbags=N6),
    F("fwd-f32-elem-offset-full", F32, 128, dict(vb="elem", slice="full", partial=False, stride=False, nslices=4),
      "mixed", off=1, nbags=N6),
    # forward, many bags (one per request)
    F("fwd-f32-v16-full-nostride", F32, 2048, dict(vb=16, slice="full", stride=False, nslices=2), "one"),
    F("fwd-f16-v16-narrowed-stride", F16, 512, dict(vb=16, slice="narrowed", stride=True, nslices=2), "one"),
    F("fwd-bf16-elem-full-partial-stride", BF16, 37, dict(vb="elem", slice="full", partial=True, per_warp=2), "one"),
    F("fwd-f64-elem-offset-full-stride", F64, 12, dict(vb="elem", slice="full", per_warp=2), "one", off=1,
      modes=("sum", "mean", "max"), invalid=True),
    # HOST shards: a 4-CTA grid strides over many units
    F("host-f32-v16-narrowed-stride", F32, 64, dict(vb=16, slice="narrowed", stride=True, per_warp=16), "one",
      host=True),
    F("host-bf16-v16-narrowed-partial-stride", BF16, 80, dict(vb=16, slice="narrowed", partial=True, stride=True,
                                                               per_warp=8), "one", host=True),
    # the benchmarked shapes at test scale
    F("fwd-emb32-f32-v16-full-stride", F32, 128, dict(vb=16, slice="full", stride=True, per_warp=2), "emb",
      modes=("sum",)),
    F("fwd-frames-f32-v16-narrowed-partial", F32, 80, dict(vb=16, slice="narrowed", partial=True, stride=False),
      "frames", modes=("mean",), nbags=(8, 8)),
    # adjoint: every W class, 16-byte and element vectors (grad aligned / one element past it)
    *[A(f"acc-W{W}-{name}-{'v16' if off == 0 else 'elem'}", t, disp,
        dict(vb=16 if off == 0 else "elem", W=W, **({"stride": stride} if stride is not None else {})), "W", off=off,
        Wt=W, **({"nbags": N6} if W == 32 and stride is False else {}))
      for W, name, t, disp, stride in ((1, "f32", F32, 16, None), (2, "bf16", BF16, 40, None), (8, "f64", F64, 6, None),
                                       (31, "f16", F16, 24, None), (32, "f64", F64, 34, False),
                                       (32, "f32", F32, 8, True))
      for off in (0, 1)],
    # adjoint, exact data with duplicate rows
    A("acc-emb32-W1-exact-duplicates", F32, 128, dict(vb=16, slice="full", W=1, stride=True), "emb-exact"),
    A("acc-W8-exact-duplicates", F32, 24, dict(vb=16, W=8, stride=True), "dup-exact", modes=("sum",)),
    A("acc-frames-f32-v16-W32", F32, 80, dict(vb=16, slice="full", W=32, stride=False), "frames", modes=("mean",),
      nbags=(8, 8)),
]
IDS = [c["id"] for c in CLASSES]
assert len(set(IDS)) == len(IDS)


def test_table_spans_every_geometry_dimension():
    """the table's classes, as the launchers place them on this device, cover every dimension of the geometry"""
    seen = [(c, shape_of(c)[2]) for c in CLASSES]
    fwd = [cls for c, cls in seen if not c["adjoint"]]
    acc = [cls for c, cls in seen if c["adjoint"]]
    assert {c["t"] for c in CLASSES if not c["adjoint"]} == {F32, F64, F16, BF16}
    assert {c["t"] for c in CLASSES if c["adjoint"]} == {F32, F64, F16, BF16}
    for cl in (fwd, acc):
        assert {x["vb"] for x in cl} == {16, "elem"}
        assert {x["stride"] for x in cl} == {True, False}
        assert any(x["partial"] for x in cl)
    assert {x["slice"] for x in fwd} == {"full", "narrowed"}
    assert {(x["slice"], x["vb"]) for x in fwd if x["slice"] == "narrowed"} == {("narrowed", 16), ("narrowed", "elem")}
    assert any(x["slice"] == "narrowed" and x["stride"] for x in fwd)
    assert {x["W"] for x in acc} >= {1, 2, 8, 31, 32}
    assert any(c.get("host") for c in CLASSES)


def test_geometry_helper():
    """the helper reports nothing for calls no pooled launch takes, and the HOST grid is the HOST gather's"""
    from ddstore_b200 import _capi
    assert geometry(False, 64, F32, 0, True) == (0, 0, 0, 0, 0)
    assert geometry(True, 0, F32, 5, True) == (0, 0, 0, 0, 0)
    assert geometry(False, 64, ao.ACC_I32, 5, True) == (0, 0, 0, 0, 0)
    host = _capi.lib().dds_host_gather_ctas()
    assert geometry(False, 64, F32, 100000, True, host=True)[4] == host
    vb, sl, ns, w, ctas = geometry(False, 4096, F32, 100000, True)
    assert (vb, sl, ns, w) == (16, 512, 8, 1) and ctas > host
    assert geometry(False, 4096, F32, 100000, False)[:3] == (4, 128, 32)  # (a destination not 16-byte aligned)
    assert geometry(False, 4100, F32, 100000, True)[0] == 4  # (rows not a multiple of 16 bytes)


# ----------------------------------------------------------------------------------------- inputs
def offset_out(nbags, disp, t, off):
    """a [nbags, disp] output of t filled with 7s, starting `off` elements past a 16-byte boundary"""
    buf = torch.full((nbags * disp + 16 // SIZE[t],), 7, dtype=TORCH_DT[t], device="cuda")
    out = buf[off:off + nbags * disp].view(nbags, disp)
    assert (out.data_ptr() % 16 == 0) == (off == 0)
    return out


def counts_for_total(rng, total):
    """request row counts (0..3 each) that add up to `total` (two empty requests for 0)"""
    if total == 0:
        return [0, 0]
    out, s = [], 0
    while s < total:
        c = min(int(rng.integers(0, 4)), total - s)
        out.append(c)
        s += c
    return out


def long_bag(rng, W, nreq=101):
    """a bag of nreq requests (several 32-request chunks) whose first chunk's and whole row totals are not multiples of
    W (for W > 1): window starts carried across chunks matter"""
    c = [int(x) for x in rng.integers(0, 4, nreq)]
    if W > 1:
        while sum(c[:32]) % W == 0:
            c[0] = (c[0] + 1) % 4
        while sum(c) % W == 0:  # (the last request is not in the first chunk)
            c[-1] = (c[-1] + 1) % 4
    return c


def w_bags(rng, W, nbags):
    """requests per bag and their row counts for a W class: row totals 0 (an empty bag and one of empty requests),
    W - 1, W, W + 1, a long bag, then one-request bags to nbags"""
    designed = [[], [0, 0]] + [counts_for_total(rng, T) for T in ([W - 1] if W > 1 else []) + [W, W + 1]]
    designed.append(long_bag(rng, W))
    designed = designed[:nbags]  # (the W = 32 no-stride class: its six bags are these)
    bags = designed + [[int(rng.integers(0, 4))] for _ in range(nbags - len(designed))]
    order = rng.permutation(len(bags))
    bags = [bags[i] for i in order]
    sizes = [len(b) for b in bags]
    counts = np.array([x for b in bags for x in b], np.int64)
    return sizes, counts


def disjoint_starts(rng, counts, width=3):
    """starts for requests of counts (<= width rows each) over distinct rows -> (starts, rows needed)"""
    n = len(counts)
    slots = rng.permutation(n)
    starts = slots * width + rng.integers(0, width - counts + 1)
    return starts.astype(np.int64), n * width


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


# ----------------------------------------------------------------------------------------- forward
def forward_inputs(c, n, rng):
    """(shard, req, bags, nbags) of forward class c with n bags"""
    t, disp = c["t"], c["disp"]
    kind = c["kind"]
    if kind == "frames":
        lens = rng.integers(1000, 3000, n)
        st = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        nrows = int(lens.sum())
        shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
        return shard, {"sample_ids": np.arange(n), "table": (st, lens)}, None, n
    nrows = 3000 if kind != "emb" else 50000
    shard = data_bits(rng, t, nrows * disp).reshape(nrows, disp)
    if kind == "mixed":
        nreq = sum(MIXED)
        req = {"starts": rng.integers(0, nrows - 3, nreq), "counts": rng.integers(0, 4, nreq)}
        return shard, req, offsets(MIXED), len(MIXED)
    if kind == "emb":
        return shard, {"starts": rng.integers(0, nrows, 32 * n), "fixed_count": 1}, np.arange(0, 32 * n + 1, 32), n
    req = {"starts": rng.integers(0, nrows - 3, n), "counts": rng.integers(0, 4, n)}
    return shard, req, None, n


@pytest.mark.parametrize("c", [c for c in CLASSES if not c["adjoint"]],
                         ids=[c["id"] for c in CLASSES if not c["adjoint"]])
def test_forward(c):
    from ddstore_b200 import PyDDStore
    n, g, cls = shape_of(c)
    t, disp = c["t"], c["disp"]
    rng = np.random.default_rng(IDS.index(c["id"]) * 7919 + 1)
    shard, req, bags, nbags = forward_inputs(c, n, rng)
    assert nbags == n
    warps = g[4] * WARPS_PER_CTA
    bad = []
    if c.get("invalid"):  # invalid requests in bags only strided warps reach: the first one is reported
        first = -(-warps // g[2])
        assert n - first >= 40
        bad = sorted(rng.choice(np.arange(first, n), 3, replace=False).tolist())
        req["starts"][bad[0]] = len(shard) + 5
        req["counts"][bad[1]] = -1
        req["counts"][bad[2]] = len(shard)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t, placement=1 if c["host"] else 0)
        if c["host"]:
            add_var(store, "m", shard, t)
        if "sample_ids" in req:
            store.set_sample_index("x", *req["table"])
        for mode in c["modes"]:
            w = data_bits(rng, t, len(req.get("starts", req.get("sample_ids"))), special=False) \
                if mode == "weighted" else None
            exp, _, eerr = pl.pool([shard], t, MODES[mode], bags=bags, weights=w, **req)
            if bad:
                assert eerr[1] == bad[0]
            else:
                assert eerr == (0, -1)
            what = f"{c['id']} ({n} bags, geometry {g}) {mode}"
            for name in ("x", "m") if c["host"] else ("x",):
                out = offset_out(nbags, disp, t, c["off"])
                out, _, _, err = pool_call(store, name, t, MODES[mode], True, req, bags, w, out=out)
                if bad:
                    assert err is not None and err[1] == bad[0], (what, err)
                else:
                    assert err is None, (what, err)
                check(bits_of(out, t), exp, f"{what} on {name}")
    finally:
        store.free()
        store.close()


HOST_CTAS_ONE = r"""
import sys
sys.path.insert(0, {root!r})
import numpy as np, torch
from tests import pool_oracle as pl
from tests.test_gpu_pool import add_var, bits_of, call, check, data_bits
from tests.test_gpu_pool_geometry import geometry
from ddstore_b200 import PyDDStore, _capi
assert _capi.lib().dds_host_gather_ctas() == 1
t, disp, n = pl.ACC_F32, 64, 700
assert geometry(False, disp * 4, t, n, True, host=True)[4] == 1
rng = np.random.default_rng(3)
shard = data_bits(rng, t, 2000 * disp).reshape(2000, disp)
req = {{"starts": rng.integers(0, 1997, n), "counts": rng.integers(0, 4, n)}}
s = PyDDStore(device=0)
add_var(s, "h", shard, t, placement=1)
for mode in (pl.POOL_SUM, pl.POOL_MAX):
    out, _, _, err = call(s, "h", t, mode, True, req, None, None)
    assert err is None, err
    check(bits_of(out, t), pl.pool([shard], t, mode, **req)[0], f"one HOST CTA, mode {{mode}}")
s.free()
s.close()
print("one-cta-ok")
"""


def test_host_forward_on_one_cta(tmp_path):
    """DDS_HOST_CTAS=1 (a child process): one CTA's eight warps stride over every unit of a HOST variable"""
    script = tmp_path / "host_one_cta.py"
    script.write_text(HOST_CTAS_ONE.format(root=ROOT))
    env = dict(os.environ, DDS_HOST_CTAS="1")
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "one-cta-ok" in r.stdout, r.stdout + r.stderr


# ----------------------------------------------------------------------------------------- adjoint
@pytest.mark.parametrize("c", [c for c in CLASSES if c["adjoint"] and c["kind"] in ("W", "frames")],
                         ids=[c["id"] for c in CLASSES if c["adjoint"] and c["kind"] in ("W", "frames")])
def test_adjoint(c):
    """rows touched at most once: each element start + its contribution, one admissible addition"""
    from ddstore_b200 import PyDDStore
    n, g, cls = shape_of(c)
    t, disp, off = c["t"], c["disp"], c["off"]
    rng = np.random.default_rng(IDS.index(c["id"]) * 7919 + 2)
    if c["kind"] == "frames":
        lens = rng.integers(1000, 3000, n)
        st = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        nrows = int(lens.sum())
        req, bags = {"sample_ids": rng.permutation(n), "table": (st, lens)}, None
        nreq = n
    else:
        sizes, counts = w_bags(rng, c["Wt"], n)
        starts, nrows = disjoint_starts(rng, counts)
        req, bags = {"starts": starts, "counts": counts}, offsets(sizes)
        nreq = len(counts)
        assert len(sizes) == n
    shard = data_bits(rng, t, nrows * disp, special=False).reshape(nrows, disp)
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        if "sample_ids" in req:
            store.set_sample_index("x", *req["table"])
        for mode in c["modes"]:
            g_ = data_bits(rng, t, n * disp).reshape(n, disp)
            w = data_bits(rng, t, nreq, special=False) if mode == "weighted" else None
            before = shard_bits(store, "x", nrows, disp, t)
            what = f"{c['id']} ({n} bags, geometry {g}) {mode}"
            gt = grad_tensor(g_, t, off)
            assert (gt.data_ptr() % 16 == 0) == (off == 0)
            total, err = acc_call(store, "x", t, MODES[mode], True, req, bags, w, gt, -0.375, woff=off)
            assert err is None, (what, err)
            writes, ns, eerr = pao.contributions([before], t, MODES[mode], g_, bags=bags, weights=w, alpha=-0.375,
                                                 **req)
            assert eerr == (0, -1)
            if c["kind"] == "W":  # the designed totals are there
                assert {c["Wt"], c["Wt"] + 1} <= set(ns) and any(x % c["Wt"] for x in ns if x > 32) | (c["Wt"] == 1)
            check_touched_once(shard_bits(store, "x", nrows, disp, t), before, writes, t, what)
    finally:
        store.free()
        store.close()


@pytest.mark.parametrize("c", [c for c in CLASSES if c["kind"] in ("emb-exact", "dup-exact")],
                         ids=[c["id"] for c in CLASSES if c["kind"] in ("emb-exact", "dup-exact")])
def test_adjoint_exact_duplicates(c):
    """exact data (integers, power-of-two alpha and bag sizes) with rows hit by many requests: the exact sum however the
    atomics are ordered -- for emb32 (bags of 32 one-row requests at W = 1) the start plus every contribution summed in
    float64, else pao.apply"""
    from ddstore_b200 import PyDDStore
    n, g, cls = shape_of(c)
    t, disp = c["t"], c["disp"]
    rng = np.random.default_rng(IDS.index(c["id"]) * 7919 + 3)
    if c["kind"] == "emb-exact":
        nrows, per = 20000, 32
        sizes = [per] * n
    else:
        nrows = 64
        sizes = rng.integers(0, 5, n)
    bags = offsets(sizes)
    nreq = int(bags[-1])
    starts = rng.integers(0, nrows, nreq).astype(np.int64)
    if c["kind"] == "dup-exact":
        starts[rng.random(nreq) < 0.3] = 7  # a hot row
    shard = ao.encode(rng.integers(-8, 9, (nrows, disp)), t)
    req = {"starts": starts, "fixed_count": 1}
    store = PyDDStore(device=0)
    try:
        add_var(store, "x", shard, t)
        for mode in c["modes"]:
            before = shard_bits(store, "x", nrows, disp, t)
            gr = ao.encode(rng.integers(-4, 5, (n, disp)), t)
            w = ao.encode(rng.integers(-1, 3, nreq), t) if mode == "weighted" else None
            total, err = acc_call(store, "x", t, MODES[mode], True, req, bags, w, grad_tensor(gr, t), 0.5)
            assert err is None, err
            what = f"{c['id']} ({n} bags, geometry {g}) {mode}"
            got = shard_bits(store, "x", nrows, disp, t)
            if c["kind"] == "dup-exact":
                writes, _, _ = pao.contributions([before], t, MODES[mode], gr, bags=bags, weights=w, alpha=0.5, **req)
                exp = pao.apply([before], writes, t)[0]
            else:  # contributions per request (the oracle's rule, vectorized), summed exactly
                bag_of = np.repeat(np.arange(n), sizes)
                wv = None if w is None else pl.decode(w, t)[:, None]
                contrib = pao.contribution(gr[bag_of], t, wv, per if mode == "mean" else 0, 0.5)
                exp = pl.decode(before, t).astype(np.float64)
                np.add.at(exp, starts, pl.decode_bits(contrib, t).astype(np.float64))
                exp = exp.astype(pl.STORAGE[t])
            assert np.array_equal(ao.keys(got, t), ao.keys(exp, t)), what
    finally:
        store.free()
        store.close()
