"""bench_pad.py -- padded batches ([B, max_rows, ...] slots + lengths from one gather launch) against the raw packed
gather followed by padding in torch, on one GPU. Prints ONE JSON line.

Workloads (timed as bench_convert.py times them: K batches between CUDA events after W warm-up batches, in blocks for
p10/p50/p90; the last batch of every route is compared bitwise with the fused result):
  cfg3     float32 samples of U{100..10000} elements (disp 1) by sample id, padded to 10000 rows, B = 4096 and 16384,
           synchronous and as an overlapped double-buffered queue
  tokens   int32 token documents of U{16..4096} by sample id, padded to 1024 with the pad id -100 (most are truncated)
  frames   80-wide float32 frames, U{50..1500} rows per sample, padded to 1500 and normalised per feature into bfloat16
Baseline of each: the raw packed gather (get_samples with offsets, plus the per-sample counts) and the fastest torch
padding route found, on the same stream: "scatter" (full() + one masked index_put of the kept rows) or, when nothing is
truncated, "nested" (nested_tensor_from_jagged(...).to_padded_tensor). Reported: ms/batch, samples/s and the modelled HBM
traffic (payload read + slots written for the fused fetch) over the time as a fraction of the H100 SXM data-sheet
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
    ap.add_argument("--workloads", default="cfg3,tokens,frames")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_pad.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    rng = np.random.default_rng(0)
    store = PyDDStore(device=0)
    results = []
    made = set()

    def workload(tag, name, lens, disp, np_dt, max_rows, B, pad_value, norm=None, queue=False):
        lens = np.asarray(lens, np.int64)
        nsamp = lens.size
        starts = np.concatenate([[0], np.cumsum(lens)])[:-1]
        rows = int(lens.sum())
        isz = np.dtype(np_dt).itemsize
        if name not in made:
            made.add(name)
            store.init(name, rows, disp, isz)
            store.synth_fill(name, 5)
            store.set_sample_index(name, starts, lens)
        tdt = {np.float32: torch.float32, np.int32: torch.int32}[np_dt]
        odt = torch.bfloat16 if norm is not None else tdt
        if norm is not None:
            store.set_normalization(name, norm[0], norm[1])
        lens_d = torch.as_tensor(lens, device=dev)
        ids = [torch.as_tensor(rng.integers(0, nsamp, B), device=dev) for _ in range(4)]
        out_el = torch.empty(0, dtype=odt).element_size()
        slot_bytes = max_rows * disp * out_el
        outs = [torch.empty(B * max_rows * disp, dtype=odt, device=dev) for _ in range(2)]
        lengths = [torch.empty(B, dtype=torch.int64, device=dev) for _ in range(2)]
        cvt = dict(src_dtype=tdt, normalize=True) if norm is not None else {}

        def fused(i):
            j = i % 2
            store.get_samples(name, ids[i % 4], outs[j], pad_rows=max_rows, pad_value=pad_value, lengths=lengths[j],
                              stream=sh, wait=not queue, overlap=queue, **cvt)

        # baseline: raw packed gather, then torch padding
        cap = int(lens.max()) * disp * isz * B
        packed = torch.empty(cap // isz, dtype=tdt, device=dev)
        offs = torch.empty(B + 1, dtype=torch.int64, device=dev)
        base_out = torch.empty(B * max_rows * disp, dtype=odt, device=dev)
        mean_t = std_t = None
        if norm is not None:
            mean_t = torch.as_tensor(norm[0], device=dev)
            std_t = torch.as_tensor(norm[1], device=dev)
        truncates = int(lens.max()) > max_rows

        def raw(i):
            store.get_samples(name, ids[i % 4], packed, offsets=offs, stream=sh)
            return lens_d[ids[i % 4]]

        def finish(x):
            if norm is None:
                return x
            return ((x.view(-1, disp) - mean_t) / std_t).to(odt).view(-1)

        def scatter(i):
            cnt = raw(i)
            total = int(offs[-1].item()) // isz // disp  # rows in the packed batch
            req = torch.repeat_interleave(torch.arange(B, device=dev), cnt, output_size=total)
            r = torch.arange(total, device=dev) - torch.repeat_interleave(offs[:-1] // (isz * disp), cnt, output_size=total)
            keep = r < max_rows
            v = finish(packed[:total * disp]).view(total, disp)
            o = base_out.view(B, max_rows, disp)
            o.fill_(pad_value)
            o[req[keep], r[keep]] = v[keep]

        def nested(i):
            cnt = raw(i)
            total = int(offs[-1].item()) // isz
            v = finish(packed[:total]).view(-1, disp)
            nt = torch.nested.nested_tensor_from_jagged(v, offsets=offs // (isz * disp))
            base_out.view(B, max_rows, disp).copy_(nt.to_padded_tensor(float(pad_value), output_size=(B, max_rows, disp)))

        ms, pct = timed(fused, K, W, st)
        if queue:
            store.wait()
        torch.cuda.synchronize()
        fused_last = outs[(W + K - 1) % 2].clone()
        last_i = W + K - 1
        routes = {"scatter": scatter}
        if not truncates:
            routes["nested"] = nested
        best = None
        for rname, fn in routes.items():
            try:
                bms, bpct = timed(fn, K, W, st)
            except Exception as e:  # noqa: BLE001  (a route torch cannot run here is skipped and named)
                results.append({"name": f"{tag}/{rname}", "error": str(e)[:200]})
                continue
            fn(last_i)
            torch.cuda.synchronize()
            ib = {2: torch.int16, 4: torch.int32}[out_el]
            same = bool(torch.equal(base_out.view(ib), fused_last.view(ib)))
            results.append({"name": f"{tag}/baseline_{rname}", "ms_per_batch": bms, "ms_per_batch_p10_p50_p90": bpct,
                            "samples_per_s": B / (bms * 1e-3), "bitwise_equal_to_fused": same})
            if best is None or bms < best[1]:
                best = (rname, bms)
        payload = float(np.minimum(lens, max_rows).mean()) * disp * isz * B  # (expected bytes read per batch)
        traffic = payload + B * slot_bytes
        results.append({"name": f"{tag}/fused" + ("_overlapped_queue" if queue else ""), "ms_per_batch": ms,
                        "ms_per_batch_p10_p50_p90": pct, "samples_per_s": B / (ms * 1e-3),
                        "modelled_hbm_bytes": traffic, "modelled_hbm_fraction_of_3p35TBps": traffic / (ms * 1e-3) / HBM_BPS,
                        "fastest_baseline": best[0] if best else None,
                        "speedup_vs_fastest_baseline": (best[1] / ms) if best else None})
        del outs, packed, base_out
        torch.cuda.empty_cache()

    wl = set(args.workloads.split(","))
    if "cfg3" in wl:
        lens = rng.integers(100, 10001, 40_000)
        for B in (4096, 16384):
            for q in (False, True):
                workload(f"cfg3_B{B}", "cfg3", lens, 1, np.float32, 10000, B, 0.0, queue=q)
    if "tokens" in wl:
        workload("tokens_B8192", "tok", rng.integers(16, 4097, 60_000), 1, np.int32, 1024, 8192, -100)
    if "frames" in wl:
        mean = np.linspace(-1, 1, 80).astype(np.float32)
        std = np.linspace(0.5, 2, 80).astype(np.float32)
        workload("frames_B512", "frames", rng.integers(50, 1501, 8000), 80, np.float32, 1500, 512, 0.0, norm=(mean, std))
    store.free()
    store.close()
    print(json.dumps({"bench": "pad", "card": card_info(dev), "steps": K, "warmup": W, "results": results}))


if __name__ == "__main__":
    main()
