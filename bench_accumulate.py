"""bench_accumulate.py -- batched accumulates (accumulate_batch / accumulate_samples: rows ADDED into the owners' shards
from the GPU) against torch's index_add_ and against put_batch of the same rows, on one GPU. Prints ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90). Sources hold small integers, so every sum is exact and every result is checked bitwise against the
expected sums (float64 on the host side of the check) before it is reported:
  cfg2    B = 65536 distinct uniform-random 4 KiB rows (float32, disp 1024) added into a 10M-row shard (--rows for a
          smaller one): synchronous calls, a queued run (wait=False), torch's index_add_ into a tensor view of the local
          shard, and put_batch of the same rows
  cfg3    float32 samples of U{100..10000} elements (disp 1) by sample id, B = 16384 distinct ids: accumulate_samples
          against a flat index_add_ with a precomputed element index (building that index is not timed)
  embed   embedding-like rows: 1M x 64 float32, B = 65536 row ids drawn Zipf(1.1) -- many duplicates, the contended case
          -- accumulate_batch against index_add_
  multi   across GPUs: measured only when the box has two or more GPUs, else reported as not measured
Reported: ms/batch, payload GB/s and the modelled HBM traffic (src read + the shard element read and written by the
reduction = 3 x payload, plus 8 bytes of index per request) over the time as a fraction of the H100 SXM data-sheet
3.35 TB/s. Without a GPU the script fails: there is no fallback.
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
    ap.add_argument("--workloads", default="cfg2,cfg3,embed,multi")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_accumulate.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    from ddstore_b200.store import _DevMem
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    n_even, n_odd = (W + K + 1) // 2, (W + K) // 2  # calls with src[0] / src[1]
    rng = np.random.default_rng(0)
    store = PyDDStore(device=0)
    results = []
    wl = set(args.workloads.split(","))

    def row(name, ms, pct, payload, nidx, **extra):
        traffic = 3 * payload + 8 * nidx
        results.append({"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pct,
                        "payload_GBps": payload / (ms * 1e-3) / 1e9, "modelled_hbm_bytes": traffic,
                        "modelled_hbm_fraction_of_3p35TBps": traffic / (ms * 1e-3) / HBM_BPS, **extra})

    def shard_view(name, nbytes):
        return torch.as_tensor(_DevMem(store.query(name)["local_base"], nbytes), device=dev)

    def int_src(*shape):
        return torch.randint(-2, 3, shape, device=dev).float()

    def bitwise(got, exp64):
        """got (float32) equals the exact sums exp64 (float64, all representable) bit for bit"""
        return bool(torch.equal(got.contiguous().view(torch.int32), exp64.float().contiguous().view(torch.int32)))

    if "cfg2" in wl:
        rows, disp, B = args.rows, 1024, 65536
        store.init("x", rows, disp, 4)
        shard = shard_view("x", rows * disp * 4).view(torch.float32).view(rows, disp)
        starts = torch.as_tensor(rng.choice(rows, B, replace=False), device=dev)
        srcs = [int_src(B, disp) for _ in range(2)]
        exp_sum = n_even * srcs[0].double() + n_odd * srcs[1].double()
        torch.cuda.synchronize()
        payload = B * disp * 4

        def sync_acc(i):
            store.accumulate_batch("x", starts, src=srcs[i % 2], stream=sh)

        def queued_acc(i):
            store.accumulate_batch("x", starts, src=srcs[i % 2], stream=sh, wait=False)

        def torch_acc(i):
            shard.index_add_(0, starts, srcs[i % 2])

        def put(i):
            store.put_batch("x", starts, src=srcs[i % 2], stream=sh)

        for tag, fn in (("accumulate_sync", sync_acc), ("accumulate_queued", queued_acc),
                        ("torch_index_add", torch_acc), ("put_batch_same_rows", put)):
            shard[starts] = 0
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            if tag == "accumulate_queued":
                store.wait()
            torch.cuda.synchronize()
            exp = srcs[(W + K - 1) % 2].double() if tag.startswith("put") else exp_sum
            ok = bitwise(shard[starts], exp)
            assert ok, f"cfg2/{tag}: result differs"
            extra = {"note": "a put moves 2 x payload; the traffic model counts 3"} if tag.startswith("put") else {}
            row(f"cfg2_B{B}/{tag}", ms, pct, payload, B, bitwise_checked=ok, **extra)
        results.append({"name": "cfg2/shard", "rows": rows, "row_bytes": disp * 4, "default_rows": rows == 10_000_000})
        del shard, srcs, exp_sum
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
        srcs = [int_src(n) for _ in range(2)]
        exp_sum = n_even * srcs[0].double() + n_odd * srcs[1].double()
        # the baseline's element index (not timed): rows of sample ids[i], back to back
        elem = torch.repeat_interleave(torch.as_tensor(first[ids_np], device=dev), torch.as_tensor(lens[ids_np], device=dev))
        elem += torch.arange(n, device=dev) - torch.repeat_interleave(
            torch.as_tensor(np.concatenate([[0], np.cumsum(lens[ids_np])])[:-1], device=dev),
            torch.as_tensor(lens[ids_np], device=dev))
        torch.cuda.synchronize()
        payload = n * 4

        def acc(i):
            store.accumulate_samples("s", ids, srcs[i % 2], stream=sh)

        def torch_acc(i):
            flat.index_add_(0, elem, srcs[i % 2])

        for tag, fn in (("accumulate_samples_sync", acc), ("torch_index_add", torch_acc)):
            flat.zero_()
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = bitwise(flat[elem], exp_sum)
            assert ok, f"cfg3/{tag}: result differs"
            extra = {"note": "building the element index is not timed"} if tag.startswith("torch") else {}
            row(f"cfg3_B{B}/{tag}", ms, pct, payload, B, bitwise_checked=ok, **extra)
        del flat, srcs, elem, exp_sum
        torch.cuda.empty_cache()

    if "embed" in wl:
        rows, disp, B = 1_000_000, 64, 65536
        store.init("e", rows, disp, 4)
        table = shard_view("e", rows * disp * 4).view(torch.float32).view(rows, disp)
        ids_np = ((rng.zipf(1.1, B) - 1) % rows).astype(np.int64)
        ids = torch.as_tensor(ids_np, device=dev)
        srcs = [int_src(B, disp) for _ in range(2)]
        exp = torch.zeros(rows, disp, dtype=torch.float64, device=dev)
        exp.index_add_(0, ids, n_even * srcs[0].double() + n_odd * srcs[1].double())
        torch.cuda.synchronize()
        payload = B * disp * 4
        uniq = int(np.unique(ids_np).size)

        def acc(i):
            store.accumulate_batch("e", ids, src=srcs[i % 2], stream=sh)

        def torch_acc(i):
            table.index_add_(0, ids, srcs[i % 2])

        for tag, fn in (("accumulate_sync", acc), ("torch_index_add", torch_acc)):
            table.zero_()
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = bitwise(table, exp)
            assert ok, f"embed/{tag}: result differs"
            row(f"embed_zipf1.1_B{B}/{tag}", ms, pct, payload, B, bitwise_checked=ok, distinct_rows=uniq,
                most_hits_on_one_row=int(np.bincount(ids_np).max()))
        del table, srcs, exp
        torch.cuda.empty_cache()

    if "multi" in wl:
        n = torch.cuda.device_count()
        results.append({"name": "multi_gpu_accumulate", "gpus": n,
                        "result": "not measured" + (" (one GPU on this box)" if n < 2 else " (no multi-GPU workload here)")})
    store.free()
    store.close()
    print(json.dumps({"bench": "accumulate", "card": card_info(dev), "steps": K, "warmup": W, "results": results}))


if __name__ == "__main__":
    main()
