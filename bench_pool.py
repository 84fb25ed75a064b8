"""bench_pool.py -- the pooled batches (PyDDStore.get_batch_pooled / get_samples_pooled) against the unfused route on one
GPU, and against torch's embedding_bag on a local copy of the table.

Workloads (one H100's worth; --quick shrinks every table 16x for a smoke run):
  emb32   16M x 128 float32 table, 65536 bags of 32 random ids, sum            fused: get_batch_pooled
  emb16   16M x 256 bfloat16 table, the same bags, weighted sum                fused: get_batch_pooled
  frames  80-wide float32 frames, U{50..1500} rows per sample, 4096 samples,
          mean by sample id                                                    fused: get_samples_pooled
Baselines on the same stream: the packed gather (get_batch / get_samples) plus the fastest torch reduction tried, and
F.embedding_bag on a local torch copy of the table (embedding workloads). Every route is timed like bench_convert.py: K
batches after W warm-up ones, each between CUDA events, p10 / p50 / p90. The last batch of every route is checked against
the fused result: bitwise for embedding_bag (the same order), to a stated tolerance where torch reorders the sum.
Modelled HBM traffic, as a fraction of the H100 SXM data sheet's 3.35 TB/s: fused = rows read + output written + index
and weight bytes; unfused = the same plus the packed buffer written and read again.
Prints one JSON line with the card name and its power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ddstore_b200 import PyDDStore, _capi  # noqa: E402

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def timed(fn, steps, warmup, stream):
    """per-batch milliseconds of fn() on `stream`: warm-up, then `steps` batches each between two events"""
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in ev:
            a.record(stream)
            fn()
            b.record(stream)
    stream.synchronize()
    t = np.array([a.elapsed_time(b) for a, b in ev])
    return {"p10": float(np.percentile(t, 10)), "p50": float(np.percentile(t, 50)), "p90": float(np.percentile(t, 90))}


def add_device(store, name, t):
    """variable `name` from the 2-D CUDA tensor t (any dtype: only its element size matters)"""
    t = t.contiguous()
    torch.cuda.synchronize()  # (the store copies on its own stream: torch's kernels that made t must have finished)
    rc = store._L.dds_add(store._h, name.encode(), C.c_void_p(t.data_ptr()), t.shape[0], t.shape[1], t.element_size(), 1)
    _capi.raise_for(rc)


def fastest(routes, steps, warmup, stream):
    """the fastest of several equivalent routes: (name, timing)"""
    res = {k: timed(f, steps, warmup, stream) for k, f in routes.items()}
    k = min(res, key=lambda x: res[x]["p50"])
    return k, res[k]


def emb_workload(name, store, dtype, nrows, disp, B, L, weighted, steps, warmup, stream):
    g = torch.Generator(device="cuda").manual_seed(1)
    table = (torch.randn(nrows, disp, device="cuda", generator=g) / 4).to(dtype)
    add_device(store, name, table)
    ids = torch.randint(0, nrows, (B * L,), device="cuda", generator=g)
    bags = torch.arange(0, B * L + 1, L, device="cuda", dtype=torch.int64)
    w = (torch.rand(B * L, device="cuda", generator=g) + 0.5).to(dtype) if weighted else None
    out = torch.empty(B, disp, dtype=dtype, device="cuda")
    packed = torch.empty(B * L, disp, dtype=dtype, device="cuda")
    packed_bytes = packed.view(torch.uint8).view(-1)
    sh = stream.cuda_stream

    def fused():
        store.get_batch_pooled(name, ids, out=out, bags=bags, mode="sum", weights=w, stream=sh, wait=False)

    def gather():
        store.get_batch(name, ids, out=packed_bytes, count=1, stream=sh, wait=False)

    reductions = {"view_sum": lambda: packed.view(B, L, disp).sum(1)} if w is None else {
        "mul_sum": lambda: (packed.view(B, L, disp) * w.view(B, L, 1)).sum(1),
        "bmm": lambda: torch.bmm(w.view(B, 1, L), packed.view(B, L, disp)).view(B, disp)}
    unfused = {k: (lambda r=r: (gather(), r())[1]) for k, r in reductions.items()}

    def ebag():
        return F.embedding_bag(ids, table, bags, mode="sum", per_sample_weights=w, include_last_offset=True)

    t_fused = timed(fused, steps, warmup, stream)
    store.wait()
    red_name, t_unfused = fastest(unfused, steps, warmup, stream)
    store.wait()
    t_ebag = timed(ebag, steps, warmup, stream)
    # checks of the last batch of every route against the fused result
    with torch.cuda.stream(stream):
        fused()
        store.wait()
        ref = ebag()
        gather()
        store.wait()
        unf = unfused[red_name]()
    stream.synchronize()
    iv = torch.int16 if dtype != torch.float32 else torch.int32
    differ = int((out.view(iv) != ref.view(iv)).sum())
    max_diff = float((out.float() - ref.float()).abs().max())
    tol = 3e-2 if dtype == torch.bfloat16 else 1e-4
    unf_ok = bool(torch.allclose(unf.float(), out.float(), rtol=tol, atol=tol))
    R = disp * table.element_size()
    fused_bytes = B * L * R + B * R + B * L * 8 + (B + 1) * 8 + (B * L * table.element_size() if weighted else 0)
    unfused_bytes = fused_bytes + 2 * B * L * R
    del table, packed
    return {
        "fused_ms": t_fused, "unfused_ms": t_unfused, "unfused_reduction": red_name, "embedding_bag_ms": t_ebag,
        "speedup_vs_unfused": t_unfused["p50"] / t_fused["p50"], "speedup_vs_embedding_bag": t_ebag["p50"] / t_fused["p50"],
        "fused_hbm_fraction": fused_bytes / (t_fused["p50"] * 1e-3) / HBM_PEAK,
        "unfused_hbm_fraction": unfused_bytes / (t_unfused["p50"] * 1e-3) / HBM_PEAK,
        "embedding_bag_elements_differing": differ, "embedding_bag_max_abs_diff": max_diff,
        "unfused_within_tolerance": unf_ok, "unfused_rtol": tol,
    }


def frames_workload(store, nsamples, B, steps, warmup, stream):
    disp = 80
    rng = np.random.default_rng(2)
    lens = rng.integers(50, 1501, nsamples)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    nrows = int(lens.sum())
    g = torch.Generator(device="cuda").manual_seed(3)
    frames = torch.randn(nrows, disp, device="cuda", generator=g)
    add_device(store, "frames", frames)
    del frames
    store.set_sample_index("frames", starts, lens.astype(np.int64))
    sel = rng.choice(nsamples, B, replace=False)
    ids = torch.from_numpy(sel.astype(np.int64)).cuda()
    sel_lens = torch.from_numpy(lens[sel].astype(np.int64)).cuda()
    tot_rows = int(lens[sel].sum())
    out = torch.empty(B, disp, device="cuda")
    packed = torch.empty(tot_rows, disp, device="cuda")
    offs = torch.empty(B + 1, dtype=torch.int64, device="cuda")
    seg = torch.repeat_interleave(torch.arange(B, device="cuda"), sel_lens)
    sh = stream.cuda_stream

    def fused():
        store.get_samples_pooled("frames", ids, out, mode="mean", stream=sh, wait=False)

    def gather():
        store.get_samples("frames", ids, out=packed.view(torch.uint8).view(-1), offsets=offs, stream=sh, wait=False)

    def seg_reduce():
        return torch.segment_reduce(packed, "mean", lengths=sel_lens, axis=0)

    def index_add():
        return torch.zeros(B, disp, device="cuda").index_add_(0, seg, packed) / sel_lens.view(B, 1)

    unfused = {"segment_reduce": lambda: (gather(), seg_reduce())[1], "index_add": lambda: (gather(), index_add())[1]}
    t_fused = timed(fused, steps, warmup, stream)
    store.wait()
    red_name, t_unfused = fastest(unfused, steps, warmup, stream)
    store.wait()
    with torch.cuda.stream(stream):
        fused()
        store.wait()
        unf = unfused[red_name]()
        store.wait()
    stream.synchronize()
    unf_ok = bool(torch.allclose(unf, out, rtol=1e-4, atol=1e-5))
    R = disp * 4
    fused_bytes = tot_rows * R + B * R + B * 8 + B * 16
    unfused_bytes = fused_bytes + 2 * tot_rows * R
    return {"fused_ms": t_fused, "unfused_ms": t_unfused, "unfused_reduction": red_name,
            "speedup_vs_unfused": t_unfused["p50"] / t_fused["p50"],
            "fused_hbm_fraction": fused_bytes / (t_fused["p50"] * 1e-3) / HBM_PEAK,
            "unfused_hbm_fraction": unfused_bytes / (t_unfused["p50"] * 1e-3) / HBM_PEAK,
            "unfused_within_tolerance": unf_ok, "unfused_rtol": 1e-4}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workloads", default="emb32,emb16,frames")
    ap.add_argument("--quick", action="store_true", help="tables 16x smaller (a smoke run, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pool.py needs a GPU")
    torch.cuda.set_device(0)
    div = 16 if args.quick else 1
    stream = torch.cuda.Stream()
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps,
           "warmup": args.warmup, "quick": args.quick, "workloads": {}}
    for wl in args.workloads.split(","):
        store = PyDDStore(device=0)
        try:
            if wl == "emb32":
                r = emb_workload("emb32", store, torch.float32, (16 << 20) // div, 128, 65536, 32, False, args.steps,
                                 args.warmup, stream)
            elif wl == "emb16":
                r = emb_workload("emb16", store, torch.bfloat16, (16 << 20) // div, 256, 65536, 32, True, args.steps,
                                 args.warmup, stream)
            elif wl == "frames":
                r = frames_workload(store, 16384 // div, 4096 // div, args.steps, args.warmup, stream)
            else:
                raise SystemExit(f"unknown workload {wl}")
        finally:
            store.free()
            store.close()
            torch.cuda.empty_cache()
        res["workloads"][wl] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
