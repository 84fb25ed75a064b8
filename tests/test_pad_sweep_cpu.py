"""The padded sweep's host side, without a GPU: tests/pad_sweep.py's restatement of the walk against the C++ layout
functions of ddstore_b200/csrc/kernels.h, the sweep workload's coverage claim for H100 SXM (132 SMs) and H100 PCIe
(114 SMs), and the sweep's reference (NumPy slices of host rows, padded by tests/pad_oracle.py) against torch's
pad_sequence."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import pad_oracle as po
from tests import pad_sweep as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CPP = r"""
#include <stdio.h>
#include "kernels.h"
int main() {
    long long T, nb, nw, i, payload, slot, lo, hi;
    int il, ol;
    char kind;
    while (scanf(" %c", &kind) == 1) {
        if (kind == 's') {
            if (scanf("%lld %lld %lld", &T, &nb, &nw) != 3) return 2;
            printf("%lld\n", (long long)ddsk_fixed_seg_bytes(T, nb, nw, 1, 4096));
        } else {
            if (scanf("%lld %lld %lld %lld %lld %d %d", &i, &payload, &slot, &lo, &hi, &il, &ol) != 7) return 2;
            ddsk_pad_cut_t c = ddsk_pad_cut(i, payload, slot, lo, hi, il, ol);
            printf("%lld %lld %lld %lld %lld\n", (long long)c.pay_src, (long long)c.pay_len, (long long)c.pay_dst,
                   (long long)c.pad_dst, (long long)c.pad_len);
        }
    }
    return 0;
}
"""


def _shapes():
    """(T, slot, nwarps) and pad_cut arguments of the sweep's batches at 132 and 114 SMs, plus the 4 GiB cases"""
    segs, cuts = set(), []
    rng = np.random.default_rng(1)
    for sms in (132, 114):
        nw = ps.WARPS_PER_SM * sms
        for b in ps.workload(nw):
            T = b.starts.size * b.slot
            segs.add((T, b.slot, nw))
            if T == 0:
                continue
            seg, sg = ps.segments(T, b.slot, nw)
            pay = b.payload()
            il, ol = ps.log2(b.in_el), ps.log2(b.out_el)
            for k in rng.choice(len(sg), size=min(len(sg), 6), replace=False):
                sp, se = sg[k]
                for i in range(sp // b.slot, min(b.starts.size, -(-se // b.slot))):
                    cuts.append((i, int(pay[i]), b.slot, max(sp - i * b.slot, 0), min(se - i * b.slot, b.slot), il, ol))
        for rb, mr, n in ((4097, 300, 900), (4100, 1000, 1100), (4104, 1000, 1100)):  # the 4 GiB cases
            segs.add((n * mr * rb, mr * rb, nw))
    return sorted(segs), cuts[::7]


def test_restatement_matches_kernels_h(tmp_path):
    """fixed_seg_bytes and pad_cut agree with ddsk_fixed_seg_bytes and ddsk_pad_cut on the sweep's shapes"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = tmp_path / "restate.cpp"
    src.write_text(CPP)
    exe = str(tmp_path / "restate")
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "ddstore_b200", "csrc"),
                    str(src), "-o", exe], check=True, capture_output=True, text=True)
    segs, cuts = _shapes()
    lines = [f"s {T} {nb} {nw}" for T, nb, nw in segs] + ["c " + " ".join(map(str, c)) for c in cuts]
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = r.stdout.split("\n")
    for k, (T, nb, nw) in enumerate(segs):
        assert int(out[k]) == ps.fixed_seg_bytes(T, nb, nw), (T, nb, nw, out[k])
    for k, c in enumerate(cuts):
        got = tuple(int(x) for x in out[len(segs) + k].split())
        assert got == ps.pad_cut(*c), (c, got)
    assert len(segs) > 100 and len(cuts) > 1000


@pytest.mark.parametrize("sms", [132, 114])
def test_workload_hits_every_category(sms):
    """the sweep's workload hits every coverage category on an H100 SXM (132 SMs) and an H100 PCIe (114 SMs)"""
    nw = ps.WARPS_PER_SM * sms
    hit = ps.workload_coverage(ps.workload(nw), nw)
    assert not ps.REQUIRED - hit, sorted(ps.REQUIRED - hit)


def test_coverage_names_the_cuts():
    """coverage() on hand-made batches: a chunk-segment batch whose first cut lands mid-row, one at the payload end,
    one in padding; whole-slot segments of > 64 slots with an invalid request at lane 32"""
    nw = 12
    slot = 3 * 4097  # 3 rows of 4097 bytes; T = 10 slots < 8 * 12 * 4096: segments of one chunk
    pay = np.full(10, slot)
    valid = np.ones(10, bool)
    assert ps.fixed_seg_bytes(10 * slot, slot, nw) == 4096
    assert "segcut:mid-row" in ps.coverage(pay, valid, slot, 4097, nw, 1, 1, 0)
    assert "segcut:padding" in ps.coverage(np.r_[0, pay[1:]], valid, slot, 4097, nw, 1, 1, 0)
    pay2 = np.full(10, 4096)
    assert "segcut:payload-end" in ps.coverage(pay2, valid, 4096 * 2, 1024, nw, 4, 4, 0)
    v = np.ones(500, bool)
    v[32] = False
    hit = ps.coverage(np.where(v, 12, 0), v, 12, 12, nw, 4, 4, 0)
    assert {"seg:>64 slots", "invalid:lane32", "seg:whole-slots"} <= hit


@pytest.mark.parametrize("max_rows", [0, 1, 4, 9])
def test_host_reference_matches_pad_sequence(max_rows):
    """the sweep's reference -- NumPy slices of host rows truncated to max_rows, then pad_oracle.pad_rows -- equals
    torch's pad_sequence of the same rows; invalid requests give slots of padding and length 0"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(max_rows)
    rows = rng.integers(0, 2**32, size=(500, 3), dtype=np.uint32)
    starts, counts = rng.integers(0, 480, 60), rng.integers(0, 15, 60)
    starts[[3, 40]] = [-1, 600]
    valid = ps.row_valid(500, starts, counts)
    take = np.where(valid, np.minimum(counts, max_rows), 0)
    parts = [rows[s:s + n] for s, n in zip(starts, take) if n > 0]
    packed = np.concatenate(parts).reshape(-1) if parts else np.zeros(0, np.uint32)
    got, lengths = po.pad_rows(packed, take, 3, max_rows, np.uint32(0xDEADBEEF), valid)
    seqs = [torch.from_numpy(rows[s:s + n].astype(np.int64)) if v else torch.zeros((0, 3), dtype=torch.int64)
            for s, n, v in zip(starts, take, valid)] + [torch.zeros((max_rows, 3), dtype=torch.int64)]
    exp = torch.nn.utils.rnn.pad_sequence(seqs, batch_first=True, padding_value=0xDEADBEEF)[:-1]
    assert got.shape == tuple(exp.shape)
    assert np.array_equal(got.astype(np.int64), exp.numpy())
    assert lengths.tolist() == [int(n) for n in take]
    assert lengths[3] == 0 and lengths[40] == 0
