"""tests/pad_sweep.py -- the padded gather's walk restated in Python, and the padded sweep's workload built on it.

The padded gather (dds_get_batch_padded / dds_get_samples_padded) walks the padded SOURCE space [0, nreq * slot) of a
batch (slot = max_rows * row_bytes) in segments of fixed_seg_bytes(T, slot, nwarps) bytes, nwarps = 12 per SM (the
padded launch always runs one 12-warp CTA per SM). Inside a segment it copies each slot's payload in pieces of at most
CH source bytes, starting at max(slot start, segment start), and fills the slot's padding clipped to the segment
(pad_cut). fixed_seg_bytes and pad_cut restate ddsk_fixed_seg_bytes and ddsk_pad_cut of ddstore_b200/csrc/kernels.h;
tests/test_pad_sweep_cpu.py checks them against the C++ functions.

coverage() names every place a batch's cuts land (segment and chunk cuts mid-row, at a row boundary, at the payload
end, in padding; padding runs by output length and 16-byte phase; segments by slot count; invalid requests by their
position in a segment) and workload() builds the sweep's batches so that together they hit every category of
REQUIRED. Both take the warp count, so the claim is checked for the GPU the tests run on and for other SM counts.
Pure NumPy: no store, no GPU.
"""
import numpy as np

CH = 4096                # chunk of the padded gather's geometry (12 warps x 4 stages x 4096 bytes)
WARPS_PER_SM = 12
SEG_MAX = 1 << 20
CVT_IO = {0: None, 1: (4, 2), 2: (4, 2), 3: (8, 4), 4: (1, 2), 5: (1, 4), 6: (4, 4), 7: (4, 2), 8: (4, 2), 9: (8, 4),
          10: (1, 4), 11: (1, 2), 12: (1, 2)}  # DDS_CVT_* code -> (source, output) itemsize (None: raw)

# variable -> (numpy dtype name, disp, rows). Raw itemsizes 1/2/4/8, the convert sweep's row shapes, an int32 token
# variable, and the row shapes of the normalisation layouts (channels-last, CHW longer than a chunk, a pattern that
# repeats inside the row).
VARS = {"u8x1": ("uint8", 1, 3 << 20), "u8x3": ("uint8", 3, 1 << 20), "u8x4097": ("uint8", 4097, 900),
        "i16x7": ("int16", 7, 40_000), "tok": ("int32", 1, 400_000),
        "f32x1": ("float32", 1, 1 << 20), "f32x3": ("float32", 3, 300_000), "f32x5": ("float32", 5, 200_000),
        "f32x1024": ("float32", 1024, 900), "f32x1025": ("float32", 1025, 900), "f32x40": ("float32", 40, 30_000),
        "f64x1": ("float64", 1, 600_000), "f64x3": ("float64", 3, 200_000), "f64x512": ("float64", 512, 900),
        "f64x513": ("float64", 513, 900), "u8img": ("uint8", 4800, 900), "f32img": ("float32", 3168, 400)}
# conversion codes by source dtype (0: raw)
CODES = {"uint8": [0, 4, 5, 10, 11, 12], "float32": [0, 1, 2, 6, 7, 8], "float64": [0, 3, 9], "int16": [0],
         "int32": [0]}

SEG_CUTS = ("mid-row", "row-boundary", "payload-end", "padding")
REQUIRED = ({"seg:whole-slots", "seg:chunks", "seg:>32 slots", "seg:>64 slots"}
            | {f"segcut:{k}" for k in SEG_CUTS} | {"chunkcut:mid-row", "chunkcut:row-boundary", "chunkcut:payload-end"}
            | {"padlen:<16", "padlen:16", "padlen:16k+el", "padlen:16k-el"}
            | {f"padphase:{el}:{p}" for el in (1, 2, 4, 8) for p in range(0, 16, el)}
            | {f"invalid:lane{k}" for k in (0, 31, 32, 63)} | {"invalid:first-of-segment", "invalid:last-of-segment"})


def fixed_seg_bytes(T, nb, nwarps, min_chunks=1, ch=CH):
    """ddsk_fixed_seg_bytes: ~8 segments per warp, at most 1 MiB, whole requests when one fits, else whole chunks"""
    target = T // (nwarps * 8)
    target = min(target, SEG_MAX)
    target = max(target, min_chunks * ch, ch)
    return (target // nb) * nb if 0 < nb <= target else (target // ch) * ch


def pad_cut(i, payload, slot, lo, hi, in_log2, out_log2):
    """ddsk_pad_cut -> (pay_src, pay_len, pay_dst, pad_dst, pad_len)"""
    base = i * slot
    pe = min(payload, hi)
    ps = min(lo, pe)
    qs = max(lo, payload)
    pad_len = ((hi - qs) >> in_log2) << out_log2 if qs < hi else 0
    return base + ps, pe - ps, ((base + ps) >> in_log2) << out_log2, ((base + qs) >> in_log2) << out_log2, pad_len


def log2(n):
    return int(n).bit_length() - 1


def row_valid(nrows, starts, counts):
    """a single-owner variable of nrows rows: the requests dds_get_batch accepts"""
    s, c = np.asarray(starts, np.int64), np.asarray(counts, np.int64)
    with np.errstate(over="ignore"):
        return (s >= 0) & (s < nrows) & (c >= 0) & (c <= nrows - s)


def segments(T, slot, nwarps):
    seg = fixed_seg_bytes(T, slot, nwarps)
    return seg, [(p, min(T, p + seg)) for p in range(0, T, seg)]


def coverage(payload, valid, slot, row_bytes, nwarps, in_el, out_el, base_off):
    """the categories one batch hits. payload: source payload bytes per slot (min(count, max_rows) * row_bytes, 0 when
    invalid); valid: per slot; in_el / out_el: source / output element bytes; base_off: the destination's phase."""
    payload = np.asarray(payload, np.int64)
    nreq = payload.size
    T = nreq * slot
    hit = set()
    if T == 0:
        return hit
    il, ol = log2(in_el), log2(out_el)
    seg, segs = segments(T, slot, nwarps)
    hit.add("seg:whole-slots" if seg % slot == 0 else "seg:chunks")
    for sp, se in segs:
        i0, i_end = sp // slot, min(nreq, (se + slot - 1) // slot)
        if i_end - i0 > 32:
            hit.add("seg:>32 slots")
        if i_end - i0 > 64:
            hit.add("seg:>64 slots")
        if sp > 0 and sp % slot:
            o = sp % slot
            p = int(payload[sp // slot])
            hit.add("segcut:" + ("padding" if o > p else "payload-end" if o == p else
                                 "mid-row" if o % row_bytes else "row-boundary"))
        bad = np.nonzero(~valid[i0:i_end])[0]
        for k in bad.tolist():
            if k in (0, 31, 32, 63):
                hit.add(f"invalid:lane{k}")
            if k == 0:
                hit.add("invalid:first-of-segment")
            if i0 + k == i_end - 1 and se % slot == 0:
                hit.add("invalid:last-of-segment")
        for i in range(i0, i_end):
            ps, pl, _, pd, plen = pad_cut(i, int(payload[i]), slot, max(sp - i * slot, 0), min(se - i * slot, slot), il, ol)
            for c in range(ps + CH, ps + pl, CH):
                hit.add("chunkcut:" + ("mid-row" if (c - i * slot) % row_bytes else "row-boundary"))
            if pl >= CH and pl % CH == 0 and ps + pl == i * slot + payload[i] and payload[i] < slot:
                hit.add("chunkcut:payload-end")
            if plen > 0:
                if plen < 16:
                    hit.add("padlen:<16")
                elif plen == 16:
                    hit.add("padlen:16")
                elif plen % 16 == out_el:
                    hit.add("padlen:16k+el")
                if plen > 16 and plen % 16 == 16 - out_el:
                    hit.add("padlen:16k-el")
                if plen > SEG_MAX:
                    hit.add("padlen:>1MiB")
                hit.add(f"padphase:{out_el}:{(base_off + pd) % 16}")
    return hit


def slot_rows(row_bytes, el):
    """max_rows so that the source slot falls under 16 B; just below, at and just above CH; at 2 CH -+ one element;
    around the 1 MiB segment cap"""
    want = (15, CH - el, CH, CH + el, 2 * CH - el, 2 * CH + el, SEG_MAX - row_bytes, SEG_MAX + row_bytes)
    out = []
    for t in want:
        mr = max(1, t // row_bytes) if t < SEG_MAX else max(1, -(-t // row_bytes))
        if mr not in out:
            out.append(mr)
    return out


class Batch:
    """one padded batch of the sweep: variable, conversion code, max_rows, requests, destination phase, entry"""

    def __init__(self, var, code, max_rows, starts, counts, off, dev_idx=True, with_lengths=True):
        self.var, self.code, self.max_rows, self.off = var, code, int(max_rows), int(off)
        self.starts, self.counts = np.asarray(starts, np.int64), np.asarray(counts, np.int64)
        self.dev_idx, self.with_lengths = dev_idx, with_lengths
        dt, disp, nrows = VARS[var]
        isz = np.dtype(dt).itemsize
        self.row_bytes = disp * isz
        self.in_el, self.out_el = (isz, isz) if code == 0 else CVT_IO[code]
        self.valid = row_valid(nrows, self.starts, self.counts)
        self.slot = self.max_rows * self.row_bytes

    def payload(self):
        return np.where(self.valid, np.minimum(np.clip(self.counts, 0, None), self.max_rows), 0) * self.row_bytes

    def coverage(self, nwarps):
        return coverage(self.payload(), self.valid, self.slot, self.row_bytes, nwarps, self.in_el, self.out_el, self.off)

    def __repr__(self):
        return (f"Batch({self.var}, code={self.code}, max_rows={self.max_rows}, nreq={self.starts.size}, "
                f"dst+{self.off})")


INVALID_KINDS = lambda nrows: [(-1, 1), (nrows, 1), (nrows - 2, 5), (3, -1), (3, 1 << 62), (5, nrows + 1)]  # noqa: E731


def _counts_for_cuts(rng, counts, slot, row_bytes, max_rows, nreq, nwarps):
    """set the counts of the slots that segment cuts fall into, so the cuts land mid-row, at a row boundary, at the
    payload end and in padding in turn"""
    T = nreq * slot
    if T == 0:
        return
    _, segs = segments(T, slot, nwarps)
    done, turn = set(), 0
    for sp, _ in segs[1:]:
        i, o = sp // slot, sp % slot
        if o == 0 or i in done:
            continue
        done.add(i)
        want = SEG_CUTS[turn % 4]
        turn += 1
        on_row = o % row_bytes == 0
        if want == "padding" or (want == "payload-end" and not on_row):
            counts[i] = rng.integers(0, (o - 1) // row_bytes + 1)
        elif want == "payload-end":
            counts[i] = o // row_bytes
        else:  # mid-row or a row boundary, whichever the cut's offset gives: payload past it
            counts[i] = rng.integers(o // row_bytes + 1, max_rows + 2)


def workload(nwarps, seed=7):
    """the sweep's batches for a GPU of nwarps / 12 SMs: every variable at every slot shape of slot_rows, its
    conversions and destination phases in turn, counts of 0, 1, max_rows -+ 1, max_rows and several MiB, segment cuts
    steered into every kind of place, invalid requests at window lanes 0 / 31 / 32 / 63 and at a segment's end; then
    every destination phase of every output itemsize, and an all-invalid batch"""
    rng = np.random.default_rng(seed)
    out, phase = [], {1: 0, 2: 0, 4: 0, 8: 0}
    for var, (dt, disp, nrows) in VARS.items():
        isz = np.dtype(dt).itemsize
        rb = disp * isz
        codes = CODES[dt]
        for k, mr in enumerate(slot_rows(rb, isz)):
            slot = mr * rb
            code = codes[k % len(codes)]
            if slot >= SEG_MAX // 2 and dt == "uint8":
                code = (5, 10)[k % 2]  # padding of a near-1 MiB source slot comes out as > 1 MiB of float32
            out_el = isz if code == 0 else CVT_IO[code][1]
            nreq = int(min(3000, max(16, (4 << 20) // max(slot, 1))))
            big = max(1, min(nrows - 1, (6 << 20) // rb))  # a valid count several MiB long (truncated)
            choice = np.array([0, 1, max(mr - 1, 0), mr, mr + 1, big], np.int64)
            counts = choice[rng.integers(0, len(choice), nreq)]
            counts = np.where(rng.random(nreq) < 0.05, big, np.minimum(counts, nrows))
            _counts_for_cuts(rng, counts, slot, rb, mr, nreq, nwarps)
            counts = np.minimum(counts, nrows)
            starts = rng.integers(0, np.maximum(nrows - counts, 0) + 1).astype(np.int64)
            if k == 0:
                starts[0], counts[0] = 0, min(nrows, 64)  # the rounding-edge rows at the variable's start
            _, segs = segments(nreq * slot, slot, nwarps)
            if k == 0 and len(segs) > 1:  # invalid requests around a segment's first window and at its end
                sp, se = segs[1] if len(segs) > 2 else segs[0]
                i0, i_end = sp // slot, min(nreq, -(-se // slot))
                kinds = INVALID_KINDS(nrows)
                for j, lane in enumerate((0, 31, 32, 63, i_end - 1 - i0)):
                    if i0 + lane < i_end:
                        starts[i0 + lane], counts[i0 + lane] = kinds[j % len(kinds)]
                starts[-1], counts[-1] = kinds[5]
            off = phase[out_el] * out_el % 16
            phase[out_el] += 1
            out.append(Batch(var, code, mr, starts, counts, off, dev_idx=k % 2 == 0, with_lengths=k % 3 != 2))
    # Segments longer than one chunk need T > 16 * CH * nwarps: two batches of about 2.5 times that, so that chunk cuts
    # fall inside segments -- of whole chunks cutting 4100-byte rows mid-row, and of whole 8 KiB slots at a row boundary
    # and at the end of a one-row payload
    for var, mr, code in (("f32x1025", 4, 7), ("f32x1024", 2, 0)):
        dt, disp, nrows = VARS[var]
        slot = mr * disp * 4
        nreq = -(-5 * CH * nwarps * 4 // slot)
        counts = rng.integers(0, mr + 2, nreq)
        out.append(Batch(var, code, mr, rng.integers(0, nrows - mr - 2, nreq), counts, 2 * (len(out) % 8)))
    # every destination phase of every output itemsize (short batches of mixed counts)
    for var, el in (("u8x3", 1), ("i16x7", 2), ("f32x5", 4), ("f64x3", 8)):
        nrows = VARS[var][2]
        for off in range(0, 16, el):
            counts = rng.integers(0, 9, 77)
            out.append(Batch(var, 0, 6, rng.integers(0, nrows - 10, 77), counts, off, dev_idx=off % 2 == 1))
    nrows = VARS["tok"][2]
    kinds = INVALID_KINDS(nrows)
    bad = np.array([kinds[j % 6] for j in range(40)], np.int64)
    out.append(Batch("tok", 0, 5, bad[:, 0], bad[:, 1], 4))  # every request invalid
    return out


def workload_coverage(batches, nwarps):
    hit = set()
    for b in batches:
        hit |= b.coverage(nwarps)
    return hit
