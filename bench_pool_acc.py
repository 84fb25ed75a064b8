"""bench_pool_acc.py -- the pooled accumulates (PyDDStore.accumulate_batch_pooled / accumulate_samples_pooled: each bag's
gradient scattered into its rows, the SGD step of a sharded EmbeddingBag) against the unfused route on one GPU, and
against index_add_ on a local copy of the table.

Workloads (one H100's worth; --quick shrinks every table 16x for a smoke run; --bags sets B of the embedding ones):
  emb32   16M x 128 float32 table, 65536 bags of 32 uniform ids, sum                fused: accumulate_batch_pooled
  emb16   16M x 256 bfloat16 table, the same bags, weighted sum                     fused: accumulate_batch_pooled
  zipf32  emb32 with Zipf(1.1) ids (hot rows: the atomics contend)                  fused: accumulate_batch_pooled
  frames  80-wide float32 frames, U{50..1500} rows per sample, 4096 samples,
          mean by sample id                                                         fused: accumulate_samples_pooled
Routes on the same stream, alpha = -lr:
  unfused  the fastest of repeat_interleave / index_select expanding the gradient to one row per table row (with the
           weight or 1/n scaling and alpha), then accumulate_batch / accumulate_samples of the expanded rows;
  local    table.index_add_(0, ids, expanded) on a torch copy of the table (embedding workloads).
Timing as bench_pool.py: K batches after W warm-up ones, each between CUDA events, p10 / p50 / p90; --alternate
times fused and unfused in turns, twice. Correctness: on exact data (integer tables and grads, power-of-two lr and bag
sizes) one batch of every route leaves the same table as the fused route.
Modelled HBM traffic (bytes_model), as a fraction of the H100 SXM data sheet's 3.35 TB/s: fused = grad B*R + 2*B*L*R of
read-modify-write at the owner + indices (+ weights); unfused additionally writes and rereads the B*L*R expanded rows.
Prints one JSON line with the card name and its power limit.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_pool import HBM_PEAK, add_device, fastest, power_limit, timed  # noqa: E402
from ddstore_b200 import PyDDStore  # noqa: E402

LR = 0.125


def bytes_model(B, L, R, idx_bytes, w_bytes=0):
    """(fused, unfused) modelled HBM bytes of one batch of B bags of L rows of R bytes"""
    fused = B * R + 2 * B * L * R + idx_bytes + w_bytes
    return fused, fused + 2 * B * L * R


def zipf_ids(g, n, nrows, a=1.1):
    """n ids in [0, nrows) with P(rank k) ~ k^-a, the ranks scattered over the table by a fixed permutation"""
    cdf = torch.arange(1, nrows + 1, device="cuda", dtype=torch.float64).pow(-a).cumsum(0)
    u = torch.rand(n, device="cuda", dtype=torch.float64, generator=g) * cdf[-1]
    r = torch.searchsorted(cdf, u).clamp_(max=nrows - 1)
    perm = torch.randperm(nrows, device="cuda", generator=g)
    return perm[r]


def emb_workload(name, store, dtype, nrows, disp, B, L, weighted, zipf, steps, warmup, alternate, stream):
    g = torch.Generator(device="cuda").manual_seed(1)
    table = torch.randint(-4, 5, (nrows, disp), device="cuda", generator=g).to(dtype)  # (sums stay exact in bf16)
    add_device(store, name, table)
    ids = zipf_ids(g, B * L, nrows) if zipf else torch.randint(0, nrows, (B * L,), device="cuda", generator=g)
    bags = torch.arange(0, B * L + 1, L, device="cuda", dtype=torch.int64)
    w = torch.randint(1, 3, (B * L,), device="cuda", generator=g).to(dtype) if weighted else None
    grad = torch.randint(-4, 5, (B, disp), device="cuda", generator=g).to(dtype)
    expanded = torch.empty(B * L, disp, dtype=dtype, device="cuda")
    sh = stream.cuda_stream
    bag_of_row = torch.arange(B, device="cuda").repeat_interleave(L)
    up = torch.float32

    def fused():
        store.accumulate_batch_pooled(name, ids, grad=grad, bags=bags, mode="sum", weights=w, alpha=-LR, stream=sh,
                                      wait=False)

    def expand_ri():
        x = grad.to(up).repeat_interleave(L, 0)
        if w is not None:
            x = x * w.to(up)[:, None]
        expanded.copy_(x * -LR)

    def expand_is():
        x = grad.to(up).index_select(0, bag_of_row)
        if w is not None:
            x = x * w.to(up)[:, None]
        torch.mul(x, -LR, out=x)
        expanded.copy_(x)

    def acc():
        store.accumulate_batch(name, ids, src=expanded, stream=sh, wait=False)

    unfused = {"repeat_interleave": lambda: (expand_ri(), acc()), "index_select": lambda: (expand_is(), acc())}
    local = table.clone()

    def local_route():
        expand_ri()
        local.index_add_(0, ids, expanded)

    res = {}
    runs = 2 if alternate else 1
    tf, tu = [], []
    red_name = None
    for _ in range(runs):
        tf.append(timed(fused, steps, warmup, stream))
        store.wait()
        red_name, t = fastest(unfused, steps, warmup, stream)
        store.wait()
        tu.append(t)
    t_local = timed(local_route, steps, warmup, stream)
    # correctness on exact data: one batch of each route from the same table
    R = disp * table.element_size()
    with torch.cuda.stream(stream):
        store.put_batch(name, torch.arange(nrows, device="cuda"), src=table, stream=sh)
        fused()
        store.wait()
    stream.synchronize()
    fused_tab = read_table(store, name, nrows, disp, dtype, stream)
    with torch.cuda.stream(stream):
        store.put_batch(name, torch.arange(nrows, device="cuda"), src=table, stream=sh)
        unfused[red_name]()
        store.wait()
    stream.synchronize()
    unf_tab = read_table(store, name, nrows, disp, dtype, stream)
    with torch.cuda.stream(stream):
        local.copy_(table)
        local_route()
    stream.synchronize()
    fb, ub = bytes_model(B, L, R, B * L * 8 + (B + 1) * 8, B * L * table.element_size() if weighted else 0)
    res.update({
        "fused_ms": tf, "unfused_ms": tu, "unfused_route": red_name, "local_index_add_ms": t_local,
        "speedup_vs_unfused": [u["p50"] / f["p50"] for f, u in zip(tf, tu)],
        "speedup_vs_local": t_local["p50"] / tf[-1]["p50"],
        "fused_hbm_fraction": fb / (tf[-1]["p50"] * 1e-3) / HBM_PEAK,
        "unfused_hbm_fraction": ub / (tu[-1]["p50"] * 1e-3) / HBM_PEAK,
        "unfused_equal": bool(torch.equal(unf_tab, fused_tab)), "local_equal": bool(torch.equal(local, fused_tab)),
        "bytes_model": {"fused": fb, "unfused": ub},
    })
    del table, local, expanded
    return res


def read_table(store, name, nrows, disp, dtype, stream):
    out = torch.empty(nrows * disp * torch.tensor([], dtype=dtype).element_size(), dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(stream):
        store.get_batch(name, torch.arange(nrows, device="cuda"), out=out, count=1, stream=stream.cuda_stream)
    stream.synchronize()
    return out.view(dtype).view(nrows, disp)


def frames_workload(store, nsamples, B, steps, warmup, alternate, stream):
    disp = 80
    rng = np.random.default_rng(2)
    lens = rng.integers(50, 1501, nsamples)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    nrows = int(lens.sum())
    g = torch.Generator(device="cuda").manual_seed(3)
    frames = torch.randint(-4, 5, (nrows, disp), device="cuda", generator=g).float()
    add_device(store, "frames", frames)
    store.set_sample_index("frames", starts, lens.astype(np.int64))
    sel = rng.choice(nsamples, B, replace=False)
    ids = torch.from_numpy(sel.astype(np.int64)).cuda()
    sel_lens = torch.from_numpy(lens[sel].astype(np.int64)).cuda()
    tot_rows = int(lens[sel].sum())
    grad = torch.randint(-4, 5, (B, disp), device="cuda", generator=g).float()
    expanded = torch.empty(tot_rows, disp, device="cuda")
    seg = torch.repeat_interleave(torch.arange(B, device="cuda"), sel_lens)
    sh = stream.cuda_stream

    def fused():
        store.accumulate_samples_pooled("frames", ids, grad, mode="mean", alpha=-LR, stream=sh, wait=False)

    def expand_ri():
        expanded.copy_((grad / sel_lens.view(B, 1)).repeat_interleave(sel_lens, 0, output_size=tot_rows) * -LR)

    def expand_is():
        expanded.copy_((grad / sel_lens.view(B, 1)).index_select(0, seg) * -LR)

    def acc():
        store.accumulate_samples("frames", ids, src=expanded, stream=sh, wait=False)

    unfused = {"repeat_interleave": lambda: (expand_ri(), acc()), "index_select": lambda: (expand_is(), acc())}
    tf, tu, red_name = [], [], None
    for _ in range(2 if alternate else 1):
        tf.append(timed(fused, steps, warmup, stream))
        store.wait()
        red_name, t = fastest(unfused, steps, warmup, stream)
        store.wait()
        tu.append(t)
    R = disp * 4
    with torch.cuda.stream(stream):
        store.put_batch("frames", torch.arange(nrows, device="cuda"), src=frames, stream=sh)
        fused()
        store.wait()
    fused_tab = read_table(store, "frames", nrows, disp, torch.float32, stream).clone()
    with torch.cuda.stream(stream):
        store.put_batch("frames", torch.arange(nrows, device="cuda"), src=frames, stream=sh)
        unfused[red_name]()
        store.wait()
    unf_tab = read_table(store, "frames", nrows, disp, torch.float32, stream)
    # (lens are not powers of two: the mean's 1/n is inexact, but both routes round grad / n once, then * alpha)
    fb = B * R + 2 * tot_rows * R + B * 8 + B * 16
    ub = fb + 2 * tot_rows * R
    del frames
    return {"fused_ms": tf, "unfused_ms": tu, "unfused_route": red_name,
            "speedup_vs_unfused": [u["p50"] / f["p50"] for f, u in zip(tf, tu)],
            "fused_hbm_fraction": fb / (tf[-1]["p50"] * 1e-3) / HBM_PEAK,
            "unfused_hbm_fraction": ub / (tu[-1]["p50"] * 1e-3) / HBM_PEAK,
            "unfused_equal": bool(torch.equal(unf_tab, fused_tab)), "bytes_model": {"fused": fb, "unfused": ub}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workloads", default="emb32,emb16,zipf32,frames")
    ap.add_argument("--alternate", action="store_true", help="time fused and unfused in turns, twice")
    ap.add_argument("--bags", type=int, default=65536, help="bags per batch of the embedding workloads")
    ap.add_argument("--quick", action="store_true", help="tables 16x smaller (a smoke run, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pool_acc.py needs a GPU")
    torch.cuda.set_device(0)
    div = 16 if args.quick else 1
    stream = torch.cuda.Stream()
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps, "bags": args.bags,
           "warmup": args.warmup, "quick": args.quick, "workloads": {}}
    for wl in args.workloads.split(","):
        store = PyDDStore(device=0)
        try:
            if wl in ("emb32", "zipf32"):
                r = emb_workload(wl, store, torch.float32, (16 << 20) // div, 128, args.bags, 32, False, wl == "zipf32",
                                 args.steps, args.warmup, args.alternate, stream)
            elif wl == "emb16":
                r = emb_workload(wl, store, torch.bfloat16, (16 << 20) // div, 256, args.bags, 32, True, False,
                                 args.steps, args.warmup, args.alternate, stream)
            elif wl == "frames":
                r = frames_workload(store, 16384 // div, 4096 // div, args.steps, args.warmup, args.alternate, stream)
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
