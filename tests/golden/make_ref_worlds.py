"""Generates tests/golden/ref_worlds.json: what the UNMODIFIED reference (oracle/_ref/libddstore_ref.so) returns on the
seeded random worlds of tests/test_oracle.py::test_c_oracle_vs_compiled_reference, so that test also runs where the
reference is not built. Per case: the variable's query (itemsize, disp, lenlist), the sha256 of the packed batch of
300 valid requests, and for the 400 arbitrary (start, count) gets the reference's error code (0 = served) plus one
sha256 over the bytes of every served get, in order. Needs oracle/_ref; run from the repository root:
    python tests/golden/make_ref_worlds.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402
from tests.helpers import random_valid_requests, random_world, sha  # noqa: E402

CASES = [(np.float32, 1, 4), (np.float32, 16, 8), (np.int64, 2, 3), (np.uint8, 7, 2), (np.float64, 5, 1), (np.int32, 3, 5),
         (np.bool_, 3, 2)]
CODE = {text: code for code, text in O.ERR_TEXT.items()}


def key(dtype, disp, P):
    return f"{np.dtype(dtype).name}-{disp}-{P}"


def record(dtype, disp, P):
    # the same draws, in the same order, as the test
    rng = np.random.default_rng(1000 + disp * 31 + P)
    nrows, shards = random_world(rng, P, dtype, disp)
    w = O.RefWorld(P)
    try:
        w.add("v", shards)
        it, dp, ll = w.query(0, "v")
        starts, counts = random_valid_requests(rng, ll, 300)
        ref_out, bad, _, _ = w.get_batch(P - 1, "v", starts, counts)
        total = int(ll[-1])
        codes, served = [], []
        for _ in range(400):
            s = int(rng.integers(-5, total + 5))
            c = int(rng.integers(0, 60))
            buf = np.zeros((c, disp), dtype)
            try:
                w.get(0, "v", buf, s)
                codes.append(0)
                served.append(buf.tobytes())
            except ValueError as e:
                codes.append(CODE[str(e)])
        return {"itemsize": it, "disp": dp, "lenlist": ll.tolist(), "bad": bad, "batch_sha256": sha(ref_out.tobytes()),
                "codes": codes, "served_sha256": sha(b"".join(served))}
    finally:
        w.close()


if __name__ == "__main__":
    if not O.have_ref():
        raise SystemExit("oracle/_ref is not built")
    out = {key(*c): record(*c) for c in CASES}
    with open(os.path.join(ROOT, "tests", "golden", "ref_worlds.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
