"""bench_host.py -- batches gathered from a variable placed in pinned host memory (placement="host") on one GPU, beside
the PCIe ceiling and the same batches from HBM. Prints ONE JSON line.

Workloads (every batch is checked on the device with synth_verify; each batch is timed alone between CUDA events, so
the checks are not in the time):
  cfg2        B = 65536 random 4 KiB rows (float32, disp 1024, count 1) of a HOST variable of --gib GiB
  cfg2_hbm    the same batches from an HBM variable holding the same rows
  h2d         one pinned-to-HBM cudaMemcpy of the cfg2 batch's byte count: the PCIe ceiling of this box
  cfg3        config-3-shaped batches by sample id: samples of U{100..10000} float32 elements (disp 1), B = 4096
  bf16        the cfg2 batches delivered as bfloat16 (converted in the gather)
  matmul      a bf16 8192^3 matmul alone, and while cfg2 batches from the HOST variable are queued on a side stream
Also reported: the CTA count of HOST launches, the card's name and power limit. --sweep-ctas runs cfg2 again in one child
process per CTA count (DDS_HOST_CTAS). Without a GPU the script fails: there is no fallback.
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

from bench_convert import card_info, compare  # noqa: E402

SEED = 0xB0057


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--gib", type=float, default=8.0, help="size of the HOST variable (and of its HBM twin)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2,cfg2_hbm,h2d,cfg3,bf16,matmul")
    ap.add_argument("--sweep-ctas", default="", help="comma-separated CTA counts to rerun cfg2 with, one process each")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print("bench_host.py needs a CUDA GPU (there is no CPU fallback)", file=sys.stderr)
        sys.exit(2)
    from ddstore_b200 import PyDDStore, _capi
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev)
    sh = st.cuda_stream
    K, W = args.steps, args.warmup
    wl = set(args.workloads.split(","))
    store = PyDDStore(device=0)
    rng = np.random.default_rng(0)
    out = {"card": card_info(dev), "gib": args.gib, "steps": K, "warmup": W,
           "host_ctas": _capi.lib().dds_host_gather_ctas()}
    B, disp = 65536, 1024
    row = disp * 4
    nrows = int(args.gib * (1 << 30)) // row
    batch_bytes = B * row

    def per_batch(step, check, n):
        """ms per batch: W + n calls of step(i) (enqueued on st), each between its own pair of events, then check(i)"""
        times = []
        for i in range(W + n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            step(i)
            e1.record(st)
            e1.synchronize()
            if i >= W:
                times.append(e0.elapsed_time(e1))
            check(i)
        return float(np.mean(times)), [float(x) for x in np.percentile(times, [10, 50, 90])]

    def verified(name, packed, starts, counts=None, count=1, offsets=None):
        bad, rows, _ = store.synth_verify(name, packed, starts, counts=counts, count=count, offsets=offsets, seed=SEED,
                                          stream=sh)
        assert bad == 0 and rows > 0, f"{name}: {bad} mismatching elements"

    need_cfg2 = wl & {"cfg2", "cfg2_hbm", "bf16", "matmul"}
    if need_cfg2:
        store.init("h", nrows, disp, 4, placement="host")
        store.synth_fill("h", SEED)
        ids = [torch.from_numpy(rng.integers(0, nrows, size=B)).to(dev) for _ in range(4)]
        buf = torch.empty(batch_bytes, dtype=torch.uint8, device=dev)

        def cfg2_on(name):
            return per_batch(lambda i: store.get_batch(name, ids[i % 4], out=buf, count=1, stream=sh),
                             lambda i: verified(name, buf.view(torch.float32), ids[i % 4]), K)

        if "cfg2" in wl:
            ms, pct = cfg2_on("h")
            out["cfg2"] = {"ms_per_batch": ms, "p10_p50_p90": pct, "payload_GBps": batch_bytes / ms / 1e6}
        if "cfg2_hbm" in wl:
            store.init("m", nrows, disp, 4)
            store.synth_fill("m", SEED)
            ms, pct = cfg2_on("m")
            out["cfg2_hbm"] = {"ms_per_batch": ms, "p10_p50_p90": pct, "payload_GBps": batch_bytes / ms / 1e6}
            store.free()  # (the HBM twin is not needed any more; re-create the HOST variable)
            store.init("h", nrows, disp, 4, placement="host")
            store.synth_fill("h", SEED)
        if "bf16" in wl:
            bo = torch.empty(B * disp, dtype=torch.bfloat16, device=dev)

            def check_bf16(i):
                ref = torch.empty(B * disp, dtype=torch.float32, device=dev)
                store.get_batch("h", ids[i % 4][:1024], out=ref[:1024 * disp], count=1, stream=sh)
                _, bad = compare(bo[:1024 * disp], ref[:1024 * disp].to(torch.bfloat16))  # (NaNs by class)
                assert bad == 0, f"bf16 batch differs in {bad} elements"
                verified("h", ref[:1024 * disp], ids[i % 4][:1024])
            ms, pct = per_batch(lambda i: store.get_batch("h", ids[i % 4], out=bo, count=1, stream=sh,
                                                          src_dtype=torch.float32), check_bf16, K)
            out["bf16"] = {"ms_per_batch": ms, "p10_p50_p90": pct, "payload_GBps": batch_bytes / ms / 1e6}
        if "matmul" in wl:
            a = torch.randn(8192, 8192, dtype=torch.bfloat16, device=dev)
            b = torch.randn(8192, 8192, dtype=torch.bfloat16, device=dev)
            c = torch.empty(8192, 8192, dtype=torch.bfloat16, device=dev)
            side = torch.cuda.Stream(dev)
            nmm = 40

            def mm_run():
                for _ in range(3):
                    torch.matmul(a, b, out=c)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(nmm):
                    torch.matmul(a, b, out=c)
                e1.record(st)
                e1.synchronize()
                return e0.elapsed_time(e1) / nmm
            alone = mm_run()
            torch.cuda.synchronize()
            outs = [torch.empty(batch_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
            nq = 24
            for k in range(nq):  # queued on the side stream, running under the matmuls
                store.get_batch("h", ids[k % 4], out=outs[k % 2], count=1, stream=side.cuda_stream, wait=False)
            beside = mm_run()
            t = store.wait()
            assert t == batch_bytes
            verified("h", outs[(nq - 1) % 2].view(torch.float32), ids[(nq - 1) % 4])
            out["matmul"] = {"ms_alone": alone, "ms_beside_host_batches": beside,
                             "host_batches_queued": nq, "slowdown": beside / alone}
        store.free()

    if "h2d" in wl:
        src = torch.empty(batch_bytes, dtype=torch.uint8).pin_memory()
        dst = torch.empty(batch_bytes, dtype=torch.uint8, device=dev)
        src.random_(0, 256)
        ms, pct = per_batch(lambda i: dst.copy_(src, non_blocking=True), lambda i: None, K)
        assert torch.equal(dst[:4096].cpu(), src[:4096])
        out["h2d"] = {"ms_per_copy": ms, "p10_p50_p90": pct, "GBps": batch_bytes / ms / 1e6}
        del src, dst

    if "cfg3" in wl:
        sys.path.insert(0, ROOT)
        from bench import cfg3_tables
        nsamp = 50000  # (about 1 GiB of rows)
        sstart, L = cfg3_tables(nsamp)
        total = int(sstart[-1] + L[-1])
        store.init("r", total, 1, 4, placement="host")
        store.synth_fill("r", SEED)
        store.set_sample_index("r", sstart, L)
        Bs = 4096
        sids = [torch.from_numpy(rng.integers(0, nsamp, size=Bs)).to(dev) for _ in range(4)]
        cap = int(L.max()) * Bs * 4
        rbuf = torch.empty(cap, dtype=torch.uint8, device=dev)
        offs = torch.empty(Bs + 1, dtype=torch.int64, device=dev)
        st_t = torch.from_numpy(np.asarray(sstart, np.int64)).to(dev)
        l_t = torch.from_numpy(np.asarray(L, np.int64)).to(dev)
        got = {}

        def step3(i):
            got[i] = store.get_samples("r", sids[i % 4], rbuf, offsets=offs, stream=sh)

        def check3(i):
            s = sids[i % 4]
            verified("r", rbuf.view(torch.float32), st_t[s], counts=l_t[s], offsets=offs)
        ms, pct = per_batch(step3, check3, K)
        nb = float(np.mean([v for v in got.values()]))
        out["cfg3_B4096"] = {"ms_per_batch": ms, "p10_p50_p90": pct, "payload_GBps": nb / ms / 1e6}
        store.free()

    if "cfg2" in out and "h2d" in out:
        out["cfg2_over_h2d"] = out["cfg2"]["payload_GBps"] / out["h2d"]["GBps"]
    store.close()

    if args.sweep_ctas:
        sweep = {}
        for n in args.sweep_ctas.split(","):
            env = dict(os.environ, DDS_HOST_CTAS=n)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--gib", str(args.gib), "--steps", str(K),
                                "--warmup", str(W), "--workloads", "cfg2"], env=env, capture_output=True, text=True)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            if r.returncode or not line:
                sweep[n] = {"error": (r.stderr or r.stdout)[-500:]}
                continue
            child = json.loads(line[-1])
            sweep[n] = {"host_ctas": child["host_ctas"], **child["cfg2"]}
        out["cfg2_ctas_sweep"] = sweep
    print(json.dumps(out))


if __name__ == "__main__":
    main()
