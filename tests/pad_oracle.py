"""NumPy oracle of a padded batch (dds_get_batch_padded / dds_get_samples_padded), written without the store.

Request i owns slot i of an [nreq, max_rows, row] array: its first min(count_i, max_rows) rows, then `pad` elements up to
the slot's end. An invalid request's slot is all padding and its length is 0. The rows come from the packed rows of the
same requests (the raw gather, already converted when the batch converts) and their per-request row counts.
"""
import numpy as np


def pad_rows(packed, counts, row, max_rows, pad, valid=None):
    """packed: 1-D array of the VALID requests' rows back to back (`row` elements each), in request order; counts: the
    requests' row counts; valid: per-request bool (default: all). pad: one element of packed.dtype (an array scalar
    keeps its bits, e.g. a NaN payload). -> (slots [nreq, max_rows, row] of packed.dtype, lengths int64 [nreq])"""
    counts = np.asarray(counts, np.int64)
    nreq = counts.size
    valid = np.ones(nreq, bool) if valid is None else np.asarray(valid, bool)
    packed = np.asarray(packed).reshape(-1)
    pad_el = np.asarray(pad, dtype=packed.dtype).reshape(1)
    out = np.empty((nreq, max_rows, row), packed.dtype)
    out.reshape(-1).view(np.uint8).reshape(-1, packed.dtype.itemsize)[:] = pad_el.view(np.uint8)  # bit for bit
    lengths = np.where(valid, np.minimum(counts, max_rows), 0).astype(np.int64)
    at = 0
    for i in range(nreq):
        if not valid[i]:
            continue
        c = int(counts[i])
        rows = packed[at:at + c * row].reshape(c, row)
        out[i, :lengths[i]] = rows[:lengths[i]]
        at += c * row
    assert at == packed.size, "packed rows and counts disagree"
    return out, lengths
