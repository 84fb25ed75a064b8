"""bench_put.py -- batched puts (put_batch / put_samples: rows written into the owners' shards from the GPU) against the
torch baseline and against get_batch of the same rows, on one GPU. Prints ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90; every result is checked bitwise before it is reported):
  cfg2   B = 65536 distinct uniform-random 4 KiB rows (float32, disp 1024) put into a 10M-row shard (--rows for a smaller
         one): synchronous calls, a queued run (wait=False), torch's index_copy_ into a tensor view of the local shard
         with the same rows, and get_batch of the same rows (same bytes) for scale
  cfg3   float32 samples of U{100..10000} elements (disp 1) by sample id, B = 16384 distinct ids: put_samples against a
         flat index_put_ with a precomputed element index (building that index is not timed)
  multi  the same put across GPUs: measured only when the box has two or more GPUs, else reported as not measured
Reported: ms/batch, payload GB/s and the modelled HBM traffic (payload read + payload written + index bytes) over the
time as a fraction of the H100 SXM data-sheet 3.35 TB/s. Without a GPU the script fails: there is no fallback.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_convert import HBM_BPS, card_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000, help="rows of the cfg2 shard (4 KiB each)")
    ap.add_argument("--workloads", default="cfg2,cfg3,multi")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_put.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    from ddstore_b200.store import _DevMem
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    rng = np.random.default_rng(0)
    store = PyDDStore(device=0)
    results = []
    wl = set(args.workloads.split(","))

    def row(name, ms, pct, payload, nidx, **extra):
        traffic = 2 * payload + 8 * nidx
        results.append({"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pct,
                        "payload_GBps": payload / (ms * 1e-3) / 1e9, "modelled_hbm_bytes": traffic,
                        "modelled_hbm_fraction_of_3p35TBps": traffic / (ms * 1e-3) / HBM_BPS, **extra})

    def shard_view(name, nbytes):
        return torch.as_tensor(_DevMem(store.query(name)["local_base"], nbytes), device=dev)

    if "cfg2" in wl:
        rows, disp, B = args.rows, 1024, 65536
        store.init("x", rows, disp, 4)
        shard = shard_view("x", rows * disp * 4).view(torch.float32).view(rows, disp)
        starts = torch.as_tensor(rng.choice(rows, B, replace=False), device=dev)
        srcs = [torch.randn(B, disp, device=dev) for _ in range(2)]
        out = torch.empty(B, disp, device=dev)
        torch.cuda.synchronize()
        payload = B * disp * 4

        def sync_put(i):
            store.put_batch("x", starts, src=srcs[i % 2], stream=sh)

        def queued_put(i):
            store.put_batch("x", starts, src=srcs[i % 2], stream=sh, wait=False)

        def torch_put(i):
            shard.index_copy_(0, starts, srcs[i % 2])

        def get(i):
            store.get_batch("x", starts, out=out, stream=sh)

        for tag, fn in (("put_sync", sync_put), ("put_queued", queued_put), ("torch_index_copy", torch_put),
                        ("get_batch_same_rows", get)):
            shard[starts] = 0
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            if tag == "put_queued":
                store.wait()
            torch.cuda.synchronize()
            last = srcs[(W + K - 1) % 2]
            if tag == "get_batch_same_rows":
                ok = bool(torch.equal(out.view(torch.int32), shard[starts].view(torch.int32)))
            else:
                ok = bool(torch.equal(shard[starts].view(torch.int32), last.view(torch.int32)))
            assert ok, f"cfg2/{tag}: result differs"
            row(f"cfg2_B{B}/{tag}", ms, pct, payload, B, bitwise_checked=ok)
        results.append({"name": "cfg2/shard", "rows": rows, "row_bytes": disp * 4, "default_rows": rows == 10_000_000})
        del shard, srcs, out
        torch.cuda.empty_cache()

    if "cfg3" in wl:
        nsamp, B = 40_000, 16384
        lens = rng.integers(100, 10001, nsamp).astype(np.int64)
        first = np.concatenate([[0], np.cumsum(lens)])[:-1]
        total_rows = int(lens.sum())
        store.init("s", total_rows, 1, 4)
        store.set_sample_index("s", first, lens)
        flat = shard_view("s", total_rows * 4).view(torch.float32)
        ids_np = rng.choice(nsamp, B, replace=False).astype(np.int64)
        ids = torch.as_tensor(ids_np, device=dev)
        n = int(lens[ids_np].sum())
        srcs = [torch.randn(n, device=dev) for _ in range(2)]
        # the baseline's element index (not timed): rows of sample ids[i], back to back
        elem = torch.repeat_interleave(torch.as_tensor(first[ids_np], device=dev), torch.as_tensor(lens[ids_np], device=dev))
        elem += torch.arange(n, device=dev) - torch.repeat_interleave(
            torch.as_tensor(np.concatenate([[0], np.cumsum(lens[ids_np])])[:-1], device=dev),
            torch.as_tensor(lens[ids_np], device=dev))
        torch.cuda.synchronize()
        payload = n * 4

        def put(i):
            store.put_samples("s", ids, srcs[i % 2], stream=sh)

        def torch_put(i):
            flat.index_put_((elem,), srcs[i % 2])

        for tag, fn in (("put_samples_sync", put), ("torch_index_put", torch_put)):
            flat.zero_()
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = bool(torch.equal(flat[elem].view(torch.int32), srcs[(W + K - 1) % 2].view(torch.int32)))
            assert ok, f"cfg3/{tag}: result differs"
            extra = {"note": "building the element index is not timed"} if tag.startswith("torch") else {}
            row(f"cfg3_B{B}/{tag}", ms, pct, payload, B, bitwise_checked=ok, **extra)
        del flat, srcs, elem
        torch.cuda.empty_cache()

    if "multi" in wl:
        n = torch.cuda.device_count()
        results.append({"name": "multi_gpu_put", "gpus": n,
                        "result": "not measured" + (" (one GPU on this box)" if n < 2 else " (no multi-GPU workload here)")})
    store.free()
    store.close()
    print(json.dumps({"bench": "put", "card": card_info(dev), "steps": K, "warmup": W, "results": results}))


if __name__ == "__main__":
    main()
