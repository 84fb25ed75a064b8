"""bench_get_accumulate.py -- batched fetch-ops (get_accumulate_batch / get_accumulate_samples: rows added into or
swapped with the owners' shards from the GPU, the previous rows returned) against the two-launch sequence they replace
and against torch, on one GPU. Prints ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90). Operands are small integers, so every sum is exact; every result -- the shard and the last call's
previous rows -- is checked bitwise before it is reported:
  cfg2    B = 65536 distinct uniform-random 4 KiB rows (float32, disp 1024) of a 10M-row shard (--rows for a smaller
          one), op sum and replace: synchronous and queued (wait=False) fetch-ops; get_batch + accumulate_batch /
          put_batch (two launches, not atomic); torch index_select + index_add_ / index_copy_ on a view of the shard
  cfg3    float32 samples of U{100..10000} elements (disp 1) by sample id, B = 16384 distinct ids, sum and replace:
          get_accumulate_samples against get_samples + accumulate_samples / put_samples and torch on a precomputed
          element index (building it is not timed)
  ticket  an int64 counter per row, 1M rows x 1, B = 65536 ids drawn Zipf(1.1) (many duplicates, the contended case):
          +1 fetch-adds, whose tickets must be distinct, against the same ids through accumulate_batch
Reported: ms/batch, payload GB/s and the modelled HBM traffic (src read + the shard element read and written + the
result written = 4 x payload, plus 8 bytes of index per request) over the time as a fraction of the H100 SXM data-sheet
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
    ap.add_argument("--workloads", default="cfg2,cfg3,ticket")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_get_accumulate.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    from ddstore_b200.store import _DevMem
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    N = W + K
    n_even, n_odd = (N + 1) // 2, N // 2  # calls with src[0] / src[1]
    rng = np.random.default_rng(0)
    store = PyDDStore(device=0)
    results = []
    wl = set(args.workloads.split(","))

    def row(name, ms, pct, payload, nidx, **extra):
        traffic = 4 * payload + 8 * nidx
        results.append({"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pct,
                        "payload_GBps": payload / (ms * 1e-3) / 1e9, "modelled_hbm_bytes": traffic,
                        "modelled_hbm_fraction_of_3p35TBps": traffic / (ms * 1e-3) / HBM_BPS, **extra})

    def shard_view(name, nbytes):
        return torch.as_tensor(_DevMem(store.query(name)["local_base"], nbytes), device=dev)

    def int_src(*shape):
        return torch.randint(1, 4, shape, device=dev).float()

    def same(a, b):
        return bool(torch.equal(a.contiguous().view(torch.int32), b.float().contiguous().view(torch.int32)))

    def expectation(op, srcs):
        """(final rows, previous rows of the last call) after N calls alternating srcs[0], srcs[1] from zero"""
        last, prev = srcs[(N - 1) % 2].double(), srcs[(N - 2) % 2].double()
        if op == "sum":
            final = n_even * srcs[0].double() + n_odd * srcs[1].double()
            return final, final - last
        return last, prev

    def run_set(tag0, B, payload, variants, reset, read_shard, srcs, outs):
        for op in ("sum", "replace"):
            final, prev = expectation(op, srcs)
            for tag, fn in variants(op):
                reset()
                for o in outs:
                    o.fill_(-1)
                torch.cuda.synchronize()
                ms, pct = timed(fn, K, W, st)
                if "queued" in tag:
                    store.wait()
                torch.cuda.synchronize()
                ok = same(read_shard(), final) and same(outs[(N - 1) % 2], prev)
                assert ok, f"{tag0}/{op}/{tag}: result differs"
                row(f"{tag0}/{op}/{tag}", ms, pct, payload, B, bitwise_checked=ok)

    if "cfg2" in wl:
        rows, disp, B = args.rows, 1024, 65536
        store.init("x", rows, disp, 4)
        shard = shard_view("x", rows * disp * 4).view(torch.float32).view(rows, disp)
        starts = torch.as_tensor(rng.choice(rows, B, replace=False), device=dev)
        srcs = [int_src(B, disp) for _ in range(2)]
        outs = [torch.empty(B, disp, device=dev) for _ in range(2)]
        payload = B * disp * 4

        def variants(op):
            second = store.accumulate_batch if op == "sum" else store.put_batch

            def fop(i):
                store.get_accumulate_batch("x", starts, src=srcs[i % 2], out=outs[i % 2], op=op, stream=sh)

            def fop_q(i):
                store.get_accumulate_batch("x", starts, src=srcs[i % 2], out=outs[i % 2], op=op, stream=sh, wait=False)

            def two(i):
                store.get_batch("x", starts, out=outs[i % 2], stream=sh)
                second("x", starts, src=srcs[i % 2], stream=sh)

            def tor(i):
                torch.index_select(shard, 0, starts, out=outs[i % 2])
                (shard.index_add_ if op == "sum" else shard.index_copy_)(0, starts, srcs[i % 2])
            return (("get_accumulate_sync", fop), ("get_accumulate_queued", fop_q),
                    ("get_batch_then_" + ("accumulate_batch" if op == "sum" else "put_batch"), two),
                    ("torch_index_select_then_" + ("index_add" if op == "sum" else "index_copy"), tor))

        def reset():
            shard[starts] = 0
        run_set(f"cfg2_B{B}", B, payload, variants, reset, lambda: shard[starts], srcs, outs)
        results.append({"name": "cfg2/shard", "rows": rows, "row_bytes": disp * 4, "default_rows": rows == 10_000_000})
        del shard, srcs, outs
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
        outs = [torch.empty(n, device=dev) for _ in range(2)]
        # torch's element index (not timed): rows of sample ids[i], back to back
        elem = torch.repeat_interleave(torch.as_tensor(first[ids_np], device=dev), torch.as_tensor(lens[ids_np], device=dev))
        elem += torch.arange(n, device=dev) - torch.repeat_interleave(
            torch.as_tensor(np.concatenate([[0], np.cumsum(lens[ids_np])])[:-1], device=dev),
            torch.as_tensor(lens[ids_np], device=dev))
        payload = n * 4

        def variants(op):
            second = store.accumulate_samples if op == "sum" else store.put_samples

            def fop(i):
                store.get_accumulate_samples("s", ids, srcs[i % 2], outs[i % 2], op=op, stream=sh)

            def two(i):
                store.get_samples("s", ids, outs[i % 2], stream=sh)
                second("s", ids, srcs[i % 2], stream=sh)

            def tor(i):
                torch.index_select(flat, 0, elem, out=outs[i % 2])
                (flat.index_add_ if op == "sum" else flat.index_copy_)(0, elem, srcs[i % 2])
            return (("get_accumulate_samples_sync", fop),
                    ("get_samples_then_" + ("accumulate_samples" if op == "sum" else "put_samples"), two),
                    ("torch_index_select_then_" + ("index_add" if op == "sum" else "index_copy"), tor))
        run_set(f"cfg3_B{B}", B, payload, variants, flat.zero_, lambda: flat[elem], srcs, outs)
        del flat, srcs, outs, elem
        torch.cuda.empty_cache()

    if "ticket" in wl:
        rows, B = 1_000_000, 65536
        store.init("t", rows, 1, 8)
        ctr = shard_view("t", rows * 8).view(torch.int64)
        ids_np = ((rng.zipf(1.1, B) - 1) % rows).astype(np.int64)
        ids = torch.as_tensor(ids_np, device=dev)
        one = torch.ones(B, dtype=torch.int64, device=dev)
        out = torch.empty(B, dtype=torch.int64, device=dev)
        counts = np.bincount(ids_np, minlength=rows)
        # the last call's tickets, sorted by row and then by ticket: (N - 1) * c_r .. N * c_r - 1 for row r
        ids_sorted = np.sort(ids_np)
        exp_tickets = (N - 1) * counts[ids_sorted] + np.arange(B) - np.searchsorted(ids_sorted, ids_sorted)

        def fadd(i):
            store.get_accumulate_batch("t", ids, src=one, out=out, stream=sh)

        def acc(i):
            store.accumulate_batch("t", ids, src=one, stream=sh)
        for tag, fn in (("get_accumulate_sync", fadd), ("accumulate_batch_same_ids", acc)):
            ctr.zero_()
            out.fill_(-1)
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = bool(np.array_equal(ctr.cpu().numpy(), N * counts))
            if tag.startswith("get"):
                got = out.cpu().numpy()
                ok = ok and bool(np.array_equal(got[np.lexsort((got, ids_np))], exp_tickets))
            assert ok, f"ticket/{tag}: result differs"
            row(f"ticket_zipf1.1_B{B}/{tag}", ms, pct, B * 8, B, bitwise_checked=ok,
                distinct_rows=int(np.unique(ids_np).size), most_hits_on_one_row=int(counts.max()))
        del ctr, out
        torch.cuda.empty_cache()

    store.free()
    store.close()
    print(json.dumps({"bench": "get_accumulate", "card": card_info(dev), "steps": K, "warmup": W, "results": results}))


if __name__ == "__main__":
    main()
