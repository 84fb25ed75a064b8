"""bench_compare_and_swap.py -- batched compare-and-swaps (compare_and_swap_batch: elements of the owners' shards
replaced where they hold the expected value, the previous rows returned) on one GPU, beside the unconditional
operations a caller would otherwise use. Prints ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90). Every shard and result is checked bitwise before its time is reported:
  claim       int32 owner slots, 1M rows x 1 per batch, B = 65536 ids drawn Zipf(1.1) (many duplicates): compare -1,
              src = the request's index. Each batch claims a fresh 1M-row block of the shard, so every batch is a real
              claim; exactly one winner per distinct id, and every loser gets the winner's index
  cfg2        B = 65536 distinct uniform-random 4 KiB rows (int32, disp 1024) of a 2M-row shard. Half the elements
              match (the even columns), half do not; batches alternate two (src, compare) pairs, so the even columns
              flip between 0 and 1 and every batch does the same work. For comparison: get_batch + put_batch (two
              launches, not atomic) and get_accumulate_batch(op="replace") (atomic but unconditional), same rows
  flags       1-byte elements, the 32-bit compare-and-swap word loop: flags_ids, uint8 flags of 16M rows x 1 with
              B = 65536 distinct ids; flags_rows, the cfg2 shape on uint8 rows of 4 KiB. Every compare matches
Reported: ms/batch, payload GB/s and the modelled HBM traffic (src and compare read, the shard element read and
written, the result written = 5 x payload, plus 8 bytes of index per request) over the time as a fraction of the H100
SXM data-sheet 3.35 TB/s. Without a GPU the script fails: there is no fallback.
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
    ap.add_argument("--workloads", default="claim,cfg2,flags")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_compare_and_swap.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    from ddstore_b200.store import _DevMem
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    N = W + K
    rng = np.random.default_rng(0)
    store = PyDDStore(device=0)
    results = []
    wl = set(args.workloads.split(","))

    def row(name, ms, pct, payload, nidx, traffic_x=5, **extra):
        traffic = traffic_x * payload + 8 * nidx
        results.append({"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pct,
                        "payload_GBps": payload / (ms * 1e-3) / 1e9, "modelled_hbm_bytes": traffic,
                        "modelled_hbm_fraction_of_3p35TBps": traffic / (ms * 1e-3) / HBM_BPS, **extra})

    def shard_view(name, nbytes):
        return torch.as_tensor(_DevMem(store.query(name)["local_base"], nbytes), device=dev)

    if "claim" in wl:
        rows, B = 1_000_000, 65536
        store.init("own", rows * N, 1, 4)
        own = shard_view("own", rows * N * 4).view(torch.int32).view(N, rows)
        ids_np = ((rng.zipf(1.1, B) - 1) % rows).astype(np.int64)
        ids = [torch.as_tensor(ids_np + i * rows, device=dev) for i in range(N)]
        src = torch.arange(B, dtype=torch.int32, device=dev)
        cmp = torch.full((B,), -1, dtype=torch.int32, device=dev)
        outs = torch.empty(N, B, dtype=torch.int32, device=dev)
        own.fill_(-1)
        torch.cuda.synchronize()

        def claim(i):
            store.compare_and_swap_batch("own", ids[i], src=src, compare=cmp, out=outs[i], stream=sh)
        ms, pct = timed(claim, K, W, st)
        torch.cuda.synchronize()
        distinct = np.unique(ids_np)
        ok = True
        for i in (0, N // 2, N - 1):
            res, blk = outs[i].cpu().numpy(), own[i].cpu().numpy()
            win = res == -1
            ok &= bool(np.array_equal(np.sort(ids_np[win]), distinct))          # one winner per distinct id
            ok &= bool(np.array_equal(blk[ids_np[win]], np.flatnonzero(win)))  # ... whose index the slot holds
            ok &= bool((res[~win] == blk[ids_np[~win]]).all())                 # every loser got it back
            ok &= int((blk != -1).sum()) == distinct.size
        assert ok, "claim: result differs"
        row(f"claim_zipf1.1_B{B}/compare_and_swap_sync", ms, pct, B * 4, B, bitwise_checked=ok,
            distinct_ids=int(distinct.size), most_claims_on_one_id=int(np.bincount(ids_np).max()))
        del own, outs
        store.free()
        torch.cuda.empty_cache()

    def alternating(tag0, name, rows, disp, dt, B, idx, extra_variants):
        """every batch on the same B rows: (src, compare) pairs alternate, the even columns flip 0 -> 1 -> 0 and the
        odd columns keep 0 against a compare of 7 (cfg2), or every column flips (disp 1)"""
        E = torch.tensor([], dtype=dt).element_size()
        store.init(name, rows, disp, E)
        shard = shard_view(name, rows * disp * E).view(dt).view(rows, disp)
        shape = (idx.numel(), disp)
        even = torch.zeros(disp, dtype=torch.bool, device=dev)
        even[0::2] = True
        if disp == 1:
            even[:] = True
        one, zero = torch.ones(shape, dtype=dt, device=dev), torch.zeros(shape, dtype=dt, device=dev)
        seven = torch.full(shape, 7, dtype=dt, device=dev)
        srcs = [one, zero]
        cmps = [torch.where(even, zero, seven), torch.where(even, one, seven)]
        outs = [torch.empty(shape, dtype=dt, device=dev) for _ in range(2)]
        payload = idx.numel() * disp * E
        states = [torch.where(even, zero, zero), torch.where(even, one, zero)]  # shard rows after an even / odd count

        def cas(i):
            store.compare_and_swap_batch(name, idx, src=srcs[i % 2], compare=cmps[i % 2], out=outs[i % 2], stream=sh)
        for tag, fn, final, prev in (("compare_and_swap_sync", cas, states[N % 2], states[(N - 1) % 2]),) + \
                extra_variants(name, idx, srcs, outs):
            shard.zero_()
            for o in outs:
                o.fill_(-1)
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = bool(torch.equal(shard[idx], final)) and bool(torch.equal(outs[(N - 1) % 2], prev))
            ok = ok and int(shard.ne(0).sum()) == int(final.ne(0).sum())
            assert ok, f"{tag0}/{tag}: result differs"
            row(f"{tag0}/{tag}", ms, pct, payload, idx.numel(), traffic_x=5 if "compare" in tag else 4,
                bitwise_checked=ok)
        del shard, srcs, cmps, outs
        store.free()
        torch.cuda.empty_cache()

    def unconditional(name, idx, srcs, outs):
        """get_batch + put_batch and the fetch-op swap on the same rows: the shard ends as the last src, every result
        as the src before it"""
        def two(i):
            store.get_batch(name, idx, out=outs[i % 2], stream=sh)
            store.put_batch(name, idx, src=srcs[i % 2], stream=sh)

        def swap(i):
            store.get_accumulate_batch(name, idx, src=srcs[i % 2], out=outs[i % 2], op="replace", stream=sh)
        return (("get_batch_then_put_batch", two, srcs[(N - 1) % 2], srcs[(N - 2) % 2]),
                ("get_accumulate_replace", swap, srcs[(N - 1) % 2], srcs[(N - 2) % 2]))

    if "cfg2" in wl:
        rows, B = 2_000_000, 65536
        idx = torch.as_tensor(rng.choice(rows, B, replace=False), device=dev)
        alternating(f"cfg2_B{B}", "x", rows, 1024, torch.int32, B, idx, unconditional)

    if "flags" in wl:
        B = 65536
        idx = torch.as_tensor(rng.choice(16_000_000, B, replace=False), device=dev)
        alternating(f"flags_ids_B{B}", "f", 16_000_000, 1, torch.uint8, B, idx, lambda *a: ())
        idx = torch.as_tensor(rng.choice(200_000, B, replace=False), device=dev)
        alternating(f"flags_rows_B{B}", "g", 200_000, 4096, torch.uint8, B, idx, lambda *a: ())

    store.close()
    print(json.dumps({"bench": "compare_and_swap", "card": card_info(dev), "steps": K, "warmup": W,
                      "results": results}))


if __name__ == "__main__":
    main()
