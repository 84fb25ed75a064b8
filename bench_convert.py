"""bench_convert.py -- the converting gather against the raw gather (+ a torch cast) on one GPU. Prints ONE JSON line.

Workloads (every one timed as in bench.py: K launches between CUDA events after W warm-up launches, the K launches
split into blocks for p10/p50/p90, and verified: the whole last batch is compared ON THE DEVICE with torch's cast of the
raw gather of the same indices, bitwise, NaN also by class):
  cfg2   10M x 1024 float32 rows, B = 65536, fixed count: raw f32 gather; raw gather + .to(bfloat16) on the same stream;
         fused f32->bf16 and f32->f16, also as overlapped queues (DDS_OVERLAP, double-buffered)
  u8     4M x 3072 uint8 images, B = 65536: raw u8 gather + .float().div(255); fused LUT32 / LUT16 with the tables of
         that expression
  cfg3   variable-length float32 samples of 100..10000 elements by sample id, B = 16384, overlapped: raw vs f32->bf16
  f64    4 KiB float64 rows (disp 512), B = 65536: raw vs f64->f32
  norm   the cfg2 shape normalised per feature (1024 channels), (x - mean) / std into bfloat16: fused, also as an
         overlapped queue, against raw gather + (x - m) / s + .to(bfloat16) on the same stream (and the plain fused
         f32->bf16 of cfg2)
  u8norm the u8 images viewed as 3 x 32 x 32 CHW (3 channels of 1024), ToTensor() + Normalize() into bfloat16: fused
         with the div(255) decode table, against raw gather + .float().div(255).sub(m).div(s).to(bfloat16)
Reported per workload: ms/batch, samples/s, and the modelled HBM traffic (payload read + output written, and every
byte a torch cast reads and writes, computed from the shapes here; index reads are left out) over the time, as a
fraction of the H100 SXM data-sheet 3.35 TB/s. Without a GPU the script fails: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12  # H100 SXM data sheet
SEED = 1234


def card_info(dev):
    import torch
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:  # (a read-only query)
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:  # noqa: BLE001
        info["power_limit_error"] = str(e)[:200]
    return info


def timed(step, K, W, stream, blocks=5):
    """ms per step: W warm-up steps, then K steps in `blocks` blocks between CUDA events on `stream`"""
    import torch
    for i in range(W):
        step(i)
    per = [K // blocks + (1 if b < K % blocks else 0) for b in range(blocks)]
    per = [p for p in per if p > 0]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(per) + 1)]
    i = W
    ev[0].record(stream)
    for b, n in enumerate(per):
        for _ in range(n):
            step(i)
            i += 1
        ev[b + 1].record(stream)
    ev[-1].synchronize()
    ms_blocks = [ev[b].elapsed_time(ev[b + 1]) / per[b] for b in range(len(per))]
    total = ev[0].elapsed_time(ev[-1]) / sum(per)
    return total, [float(x) for x in np.percentile(ms_blocks, [10, 50, 90])]


def compare(got, ref):
    """-> (bitwise equal, mismatching elements with NaN compared by class); both tensors of the same float dtype"""
    import torch
    ib = {2: torch.int16, 4: torch.int32}[got.element_size()]
    g, r = got.reshape(-1), ref.reshape(-1)
    neq = g.view(ib) != r.view(ib)
    bitwise = not bool(neq.any())
    bad = int((neq & ~(torch.isnan(g) & torch.isnan(r))).sum().item())
    return bitwise, bad


def entry(name, ms, pcts, B, traffic_bytes, ver, extra=None):
    e = {"name": name, "ms_per_batch": ms, "ms_per_batch_p10_p50_p90": pcts, "samples_per_s": B / (ms * 1e-3),
         "modelled_hbm_bytes": traffic_bytes, "modelled_hbm_fraction_of_3p35TBps": traffic_bytes / (ms * 1e-3) / HBM_BPS,
         "verified_bitwise": ver[0], "mismatches_nan_by_class": ver[1]}
    if extra:
        e.update(extra)
    return e


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50, help="timed launches of every workload")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--scale", type=float, default=1.0, help="shrink every store (tests)")
    ap.add_argument("--workloads", default="cfg2,norm,u8,u8norm,cfg3,f64")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_convert.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W, B = args.steps, args.warmup, args.batch
    rng = np.random.default_rng(0)
    names = set(args.workloads.split(","))
    res = {"card": card_info(dev), "steps": K, "warmup": W, "workloads": []}
    out = res["workloads"]

    # ---- config-2 shape: 10M x 1024 float32, B rows per batch
    if "cfg2" in names or "norm" in names:
        N, D = int(10_000_000 * args.scale), 1024
        store = PyDDStore(device=0)
        store.init("x", N, D, 4)
        store.synth_fill("x", SEED)
        idx = [torch.from_numpy(rng.integers(0, N, B)).to(dev) for _ in range(2)]
        raw = [torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(2)]
        half = {dt: [torch.empty((B, D), dtype=dt, device=dev) for _ in range(2)] for dt in (torch.bfloat16, torch.float16)}
        rb = B * D * 4
    if "norm" in names:
        g = np.random.default_rng(SEED)
        mean = torch.from_numpy(g.standard_normal(D).astype(np.float32)).to(dev)
        std = torch.from_numpy((g.random(D) + 0.1).astype(np.float32)).to(dev)
        store.set_normalization("x", mean, std)
        tmp = torch.empty((B, D), dtype=torch.float32, device=dev)
        nrm = [torch.empty((B, D), dtype=torch.bfloat16, device=dev) for _ in range(2)]

        def gather_norm_cast(i):  # (division by a CUDA tensor: the expression the fused gather is bit-exact with)
            store.get_batch("x", idx[i & 1], out=raw[i & 1], stream=sh)
            torch.sub(raw[i & 1], mean, out=tmp)
            torch.div(tmp, std, out=tmp)
            nrm[i & 1].copy_(tmp)
        ms, p = timed(gather_norm_cast, K, W, st)
        out.append(entry("norm_raw_f32_then_torch_sub_div_bf16", ms, p, B, 2 * rb + 2 * rb + 2 * rb + rb + rb // 2, (None, 0)))
        for ovl in (False, True):
            kw = dict(wait=False, overlap=True) if ovl else {}
            ms, p = timed(lambda i: store.get_batch("x", idx[i & 1], out=nrm[i & 1], stream=sh, src_dtype=torch.float32,
                                                    normalize=True, **kw), K, W, st)  # noqa: B023
            if ovl:
                store.wait()
            last = (W + K - 1) & 1
            store.get_batch("x", idx[last], out=raw[0], stream=sh)
            ver = compare(nrm[last], ((raw[0] - mean) / std).to(torch.bfloat16))
            out.append(entry("norm_fused_f32_bf16_per_feature" + ("_overlapped" if ovl else ""), ms, p, B, rb + rb // 2, ver))
        del tmp, nrm
    if "cfg2" in names:
        ms, p = timed(lambda i: store.get_batch("x", idx[i & 1], out=raw[i & 1], stream=sh), K, W, st)
        out.append(entry("cfg2_raw_f32", ms, p, B, 2 * rb, (None, 0)))
        casted = [torch.empty((B, D), dtype=torch.bfloat16, device=dev) for _ in range(2)]

        def gather_cast(i):
            store.get_batch("x", idx[i & 1], out=raw[i & 1], stream=sh)
            casted[i & 1].copy_(raw[i & 1])
        ms, p = timed(gather_cast, K, W, st)
        out.append(entry("cfg2_raw_f32_then_torch_bf16", ms, p, B, 2 * rb + rb + rb // 2, (None, 0)))
        for dt, tag in ((torch.bfloat16, "bf16"), (torch.float16, "f16")):
            bufs = half[dt]
            for ovl in (False, True):
                if ovl:
                    fn = lambda i: store.get_batch("x", idx[i & 1], out=bufs[i & 1], stream=sh, wait=False, overlap=True, src_dtype=torch.float32)  # noqa: E731
                else:
                    fn = lambda i: store.get_batch("x", idx[i & 1], out=bufs[i & 1], stream=sh, src_dtype=torch.float32)  # noqa: E731
                ms, p = timed(fn, K, W, st)
                if ovl:
                    store.wait()
                last = (W + K - 1) & 1
                store.get_batch("x", idx[last], out=raw[0], stream=sh)
                ver = compare(bufs[last], raw[0].to(dt))
                out.append(entry(f"cfg2_fused_f32_{tag}" + ("_overlapped" if ovl else ""), ms, p, B, rb + rb // 2, ver))
        del casted
    if "cfg2" in names or "norm" in names:
        store.free()
        store.close()
        del raw, half
        torch.cuda.empty_cache()

    # ---- uint8 images: 4M x 3072, normalised to float
    if "u8" in names or "u8norm" in names:
        N, D = int(4_000_000 * args.scale), 3072
        store = PyDDStore(device=0)
        store.init("img", N, D, 1)
        store.synth_fill("img", SEED)
        idx = [torch.from_numpy(rng.integers(0, N, B)).to(dev) for _ in range(2)]
        raw = torch.empty((B, D), dtype=torch.uint8, device=dev)
        flt = torch.empty((B, D), dtype=torch.float32, device=dev)
        rb = B * D
    if "u8norm" in names:  # 3 x 32 x 32 CHW images, torchvision's ImageNet mean / std
        C, HW = 3, D // 3
        mean = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32, device=dev)
        std = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32, device=dev)
        store.set_normalization("img", mean, std, HW)
        m3, s3 = mean.view(1, C, 1), std.view(1, C, 1)
        table = torch.arange(256, device=dev, dtype=torch.uint8).float().div(255)  # ToTensor()'s expression
        bf = torch.empty((B, D), dtype=torch.bfloat16, device=dev)

        def gather_totensor_normalize(i):
            store.get_batch("img", idx[i & 1], out=raw, stream=sh)
            torch.div(raw.float(), 255, out=flt)
            v = flt.view(B, C, HW)
            torch.sub(v, m3, out=v)
            torch.div(v, s3, out=v)
            bf.copy_(flt)
        ms, p = timed(gather_totensor_normalize, K, W, st)
        out.append(entry("u8norm_raw_then_torch_float_div255_sub_div_bf16", ms, p, B,
                         2 * rb + (rb + 4 * rb) + 3 * (2 * 4 * rb) + (4 * rb + 2 * rb), (None, 0)))
        o = torch.empty((B, D), dtype=torch.bfloat16, device=dev)
        ms, p = timed(lambda i: store.get_batch("img", idx[i & 1], out=o, stream=sh, src_dtype=torch.uint8, lut=table,
                                                normalize=True), K, W, st)
        last = (W + K - 1) & 1
        store.get_batch("img", idx[last], out=raw, stream=sh)
        ver = compare(o, ((raw.view(B, C, HW).float().div(255) - m3) / s3).to(torch.bfloat16))
        out.append(entry("u8norm_fused_chw_bf16", ms, p, B, rb + 2 * rb, ver))
        del o, bf
    if "u8" in names:

        def gather_norm(i):
            store.get_batch("img", idx[i & 1], out=raw, stream=sh)
            torch.div(raw.float(), 255, out=flt)
        ms, p = timed(gather_norm, K, W, st)
        out.append(entry("u8_raw_then_torch_float_div255", ms, p, B, 2 * rb + (rb + 4 * rb) + 2 * 4 * rb, (None, 0)))
        x = torch.arange(256, device=dev, dtype=torch.uint8)
        for dt, tag in ((torch.float32, "lut32_f32"), (torch.bfloat16, "lut16_bf16")):
            table = x.float().div(255).to(dt)  # the same expression, so the fused result is bit-exact with it
            o = torch.empty((B, D), dtype=dt, device=dev)
            ms, p = timed(lambda i: store.get_batch("img", idx[i & 1], out=o, stream=sh, src_dtype=torch.uint8, lut=table), K, W, st)
            last = (W + K - 1) & 1
            store.get_batch("img", idx[last], out=raw, stream=sh)
            ver = compare(o, raw.float().div(255).to(dt))
            out.append(entry(f"u8_fused_{tag}", ms, p, B, rb + rb * o.element_size(), ver))
            del o
    if "u8" in names or "u8norm" in names:
        store.free()
        store.close()
        del raw, flt
        torch.cuda.empty_cache()

    # ---- config-3 shape by sample id, overlapped queue
    if "cfg3" in names:
        B3 = 16384
        nsamp = max(64, int(500_000 * args.scale))
        L = np.random.default_rng(42).integers(100, 10001, size=nsamp)
        sstart = np.concatenate([[0], np.cumsum(L)])
        store = PyDDStore(device=0)
        store.init("x", int(sstart[-1]), 1, 4)
        store.synth_fill("x", SEED)
        store.set_sample_index("x", torch.from_numpy(sstart[:-1].copy()).to(dev), torch.from_numpy(L).to(dev))
        NS = 4
        ids = [torch.from_numpy(rng.integers(0, nsamp, size=B3)).to(dev) for _ in range(NS)]
        rows = [int(L[i.cpu().numpy()].sum()) for i in ids]
        rmax = max(rows)
        offs = [torch.empty(B3 + 1, dtype=torch.int64, device=dev) for _ in range(2)]
        raw = [torch.empty(rmax, dtype=torch.float32, device=dev) for _ in range(2)]
        bf = [torch.empty(rmax, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        nb = float(np.mean(rows)) * 4
        ms, p = timed(lambda i: store.get_samples("x", ids[i % NS], raw[i & 1], offsets=offs[i & 1], stream=sh, wait=False,
                                                  overlap=True), K, W, st)
        store.wait()
        out.append(entry("cfg3_by_sample_id_raw_f32_overlapped", ms, p, B3, 2 * nb, (None, 0)))
        ms, p = timed(lambda i: store.get_samples("x", ids[i % NS], bf[i & 1], offsets=offs[i & 1], stream=sh, wait=False,
                                                  overlap=True, src_dtype=torch.float32), K, W, st)
        store.wait()
        li = W + K - 1
        r = rows[li % NS]
        store.get_samples("x", ids[li % NS], raw[0], stream=sh)
        ver = compare(bf[li & 1][:r], raw[0][:r].to(torch.bfloat16))
        out.append(entry("cfg3_by_sample_id_fused_f32_bf16_overlapped", ms, p, B3, nb + nb / 2, ver))
        store.free()
        store.close()
        del raw, bf
        torch.cuda.empty_cache()

    # ---- float64 rows of 4 KiB
    if "f64" in names:
        N, D = int(4_000_000 * args.scale), 512
        store = PyDDStore(device=0)
        store.init("d", N, D, 8)
        store.synth_fill("d", SEED)
        idx = [torch.from_numpy(rng.integers(0, N, B)).to(dev) for _ in range(2)]
        raw = torch.empty((B, D), dtype=torch.float64, device=dev)
        o = torch.empty((B, D), dtype=torch.float32, device=dev)
        rb = B * D * 8
        ms, p = timed(lambda i: store.get_batch("d", idx[i & 1], out=raw, stream=sh), K, W, st)
        out.append(entry("f64_raw", ms, p, B, 2 * rb, (None, 0)))
        ms, p = timed(lambda i: store.get_batch("d", idx[i & 1], out=o, stream=sh, src_dtype=torch.float64), K, W, st)
        last = (W + K - 1) & 1
        store.get_batch("d", idx[last], out=raw, stream=sh)
        out.append(entry("f64_fused_f32", ms, p, B, rb + rb // 2, compare(o, raw.to(torch.float32))))
        store.free()
        store.close()

    by = {e["name"]: e for e in out}
    if "cfg2_raw_f32" in by and "cfg2_fused_f32_bf16" in by:
        res["cfg2_fused_bf16_speedup_vs_raw_f32"] = by["cfg2_fused_f32_bf16"]["samples_per_s"] / by["cfg2_raw_f32"]["samples_per_s"]
        res["cfg2_fused_bf16_speedup_vs_gather_then_cast"] = (by["cfg2_fused_f32_bf16"]["samples_per_s"] /
                                                              by["cfg2_raw_f32_then_torch_bf16"]["samples_per_s"])
    if "norm_fused_f32_bf16_per_feature" in by:
        nf = by["norm_fused_f32_bf16_per_feature"]["samples_per_s"]
        res["norm_fused_speedup_vs_gather_then_sub_div_cast"] = nf / by["norm_raw_f32_then_torch_sub_div_bf16"]["samples_per_s"]
        if "cfg2_fused_f32_bf16" in by:
            res["norm_fused_vs_plain_fused_bf16"] = nf / by["cfg2_fused_f32_bf16"]["samples_per_s"]
    if "u8norm_fused_chw_bf16" in by:
        res["u8norm_fused_speedup_vs_unfused"] = (by["u8norm_fused_chw_bf16"]["samples_per_s"] /
                                                  by["u8norm_raw_then_torch_float_div255_sub_div_bf16"]["samples_per_s"])
    res["all_verified"] = all(e["mismatches_nan_by_class"] == 0 for e in out)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
