"""bench_reduce.py -- batched reductions beside the sum (accumulate_batch / get_accumulate_batch with op="amax",
"amin", "bitwise_and", "bitwise_or", "bitwise_xor") on one GPU, beside the sum and torch's local index_reduce_. Prints
ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90). Every shard and result is checked bitwise before its time is reported:
  cfg2_f32    B = 65536 distinct 4 KiB float32 rows (disp 1024) of a 2M-row shard, amax of random values into a
              zeroed shard. Batch i takes its own block of rows, so every batch changes every element it touches.
              f32 max has no atomic: the compare-and-swap loops. For comparison: accumulate_batch (sum) of the same
              rows, and torch's index_reduce_(0, idx, src, "amax") on a local view of the shard
  cfg2_bf16   the same shape in bfloat16 (2048 elements a row): the bulk max reduction
  stamps      int64 "last seen at step" stamps, 1M rows x 1: B = 65536 ids drawn Zipf(1.1) (many duplicates), batch
              i writes amax(stamp, i + 1): the contended case
  flags       int32 flags, 1M rows x 1, the same Zipf ids, batch i sets bit i % 31 with bitwise_or
  fetch       the cfg2_f32 shape through get_accumulate_batch(op="amax"): the previous rows (all zero) returned
Reported: ms/batch, payload GB/s, and the card's name and power limit. Without a GPU the script fails: there is no
fallback.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_convert import card_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2_f32,cfg2_bf16,stamps,flags,fetch")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_reduce.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
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
    B = 65536

    def row(name, ms, pct, payload, **extra):
        results.append({"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pct,
                        "payload_GBps": payload / (ms * 1e-3) / 1e9, **extra})

    def shard_view(name, nbytes):
        return torch.as_tensor(_DevMem(store.query(name)["local_base"], nbytes), device=dev)

    def cfg2(dt, tag, fetch_only=False):
        """N blocks of B distinct rows of 4 KiB; batch i reduces into block i"""
        E = torch.tensor([], dtype=dt).element_size()
        disp, rows = 4096 // E, 2_000_000
        assert N * B <= rows, "--steps + --warmup too large for the 2M-row shard"
        store.init("x", rows, disp, E)
        shard = shard_view("x", rows * disp * E).view(dt).view(rows, disp)
        perm = torch.as_tensor(rng.permutation(rows)[:N * B], device=dev).view(N, B)
        src = torch.randn(B, disp, device=dev).to(dt)
        exp = torch.clamp(src, min=0)  # amax with a zeroed shard: +0 where src < 0 or -0
        exp = torch.where(src == 0, torch.zeros_like(src), exp)  # (max(+0, -0) is +0)
        payload = B * 4096
        out = torch.empty(B, disp, dtype=dt, device=dev)
        variants = []
        if fetch_only:
            variants.append(("get_accumulate_amax", lambda i: store.get_accumulate_batch(
                "x", perm[i], src=src, out=out, op="amax", count=1, stream=sh), exp))
        else:
            variants.append(("accumulate_amax", lambda i: store.accumulate_batch(
                "x", perm[i], src=src, count=1, stream=sh, op="amax"), exp))
            if dt == torch.float32:
                variants.append(("accumulate_sum", lambda i: store.accumulate_batch(
                    "x", perm[i], src=src, count=1, stream=sh), src))
                variants.append(("torch_index_reduce_amax_local", lambda i: shard.index_reduce_(
                    0, perm[i], src, "amax"), exp))
        for vname, fn, want in variants:
            shard.zero_()
            out.fill_(1)
            torch.cuda.synchronize()
            ms, pct = timed(fn, K, W, st)
            torch.cuda.synchronize()
            ok = True
            for i in (0, N // 2, N - 1):
                ok &= bool(torch.equal(shard[perm[i]].view(torch.int16 if E == 2 else torch.int32),
                                       want.view(torch.int16 if E == 2 else torch.int32)))
            ok &= int(shard.ne(0).sum()) == N * int(want.ne(0).sum())
            if fetch_only:
                ok &= bool(out.eq(0).all()) and not bool(torch.signbit(out).any())
            assert ok, f"{tag}/{vname}: result differs"
            row(f"{tag}_B{B}/{vname}", ms, pct, payload, bitwise_checked=ok)
        del shard, perm, src, exp, out
        store.free()
        torch.cuda.empty_cache()

    if "cfg2_f32" in wl:
        cfg2(torch.float32, "cfg2_f32")
    if "cfg2_bf16" in wl:
        cfg2(torch.bfloat16, "cfg2_bf16")
    if "fetch" in wl:
        cfg2(torch.float32, "cfg2_f32", fetch_only=True)

    ids_np = ((rng.zipf(1.1, B) - 1) % 1_000_000).astype(np.int64)
    ids = torch.as_tensor(ids_np, device=dev)
    touched = np.unique(ids_np)
    for tag, dt, opn in (("stamps", torch.int64, "amax"), ("flags", torch.int32, "bitwise_or")):
        if tag not in wl:
            continue
        E = torch.tensor([], dtype=dt).element_size()
        store.init(tag, 1_000_000, 1, E)
        shard = shard_view(tag, 1_000_000 * E).view(dt)
        if opn == "amax":
            srcs = [torch.full((B,), i + 1, dtype=dt, device=dev) for i in range(N)]
            want = N
        else:
            srcs = [torch.full((B,), 1 << (i % 31), dtype=dt, device=dev) for i in range(N)]
            want = int(np.bitwise_or.reduce([1 << (i % 31) for i in range(N)]))
        shard.zero_()
        torch.cuda.synchronize()
        ms, pct = timed(lambda i: store.accumulate_batch(tag, ids, src=srcs[i], count=1, stream=sh, op=opn), K, W, st)
        torch.cuda.synchronize()
        got = shard.cpu().numpy()
        ok = bool((got[touched] == want).all()) and int(np.count_nonzero(got)) == touched.size
        assert ok, f"{tag}: result differs"
        row(f"{tag}_zipf1.1_B{B}/accumulate_{opn}", ms, pct, B * E, bitwise_checked=ok, distinct_ids=int(touched.size),
            most_requests_on_one_id=int(np.bincount(ids_np).max()))
        del shard, srcs
        store.free()
        torch.cuda.empty_cache()

    store.close()
    print(json.dumps({"bench": "reduce", "card": card_info(dev), "steps": K, "warmup": W, "results": results}))


if __name__ == "__main__":
    main()
