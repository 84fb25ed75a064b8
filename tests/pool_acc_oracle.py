"""NumPy oracle of the pooled accumulates (dds_accumulate_batch_pooled / dds_accumulate_samples_pooled): the adjoint of
the pooled batches (tests/pool_oracle.py) over a world of shards.

Requests and bags are located and validated as in the pooled get. Every element of every row of every valid request i
in bag k gets one contribution, computed in the accumulator type A (float32 for f32, f16 and bf16 rows, float64 for
f64), each step one IEEE round-to-nearest operation:
  c = grad[k];  c = c * w_i (weights);  c = c / n_k (mean);  c = c * A(alpha);  then c rounded once to the element type,
  a NaN becoming the canonical NaN.
n_k is the number of rows the pooled get folds for bag k: the rows of its valid requests. The contributions are added
into the shards by the accumulate's rule (tests/acc_oracle.py): `contributions` lists them per shard row, `apply` adds
them with acc_oracle's correctly rounded `add` (on exact data every order gives that result), and `per_row` groups each
row's contributions for acc_oracle's `admissible_all` / `verdict` / `sum_bound` on inexact data. A malformed bag adds
nothing and is reported before any invalid request.
"""
import numpy as np

from tests import acc_oracle as ao
from tests import pool_oracle as pl
from tests import put_oracle as po


def contribution(g, t, w=None, n=0, alpha=1.0):
    """the contribution bits of grad values g (storage array of t; bf16 as its bits): times the weight w (a value of
    the accumulator type) when given, over n when n > 0 (mean), times alpha -- each step rounded once -- then encoded"""
    dt = pl.acc_dtype(t)
    c = pl.decode(g, t)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        if w is not None:
            c = (c * dt(w)).astype(dt)
        if n > 0:
            c = (c / dt(n)).astype(dt)
        c = (c * dt(alpha)).astype(dt)
    return pl.encode(c, t)


def contributions(shards, t, mode, grad, bags=None, weights=None, alpha=1.0, **req):
    """The pooled accumulate over `shards` -> (writes, n per bag, (expected code, bad index)). writes: [(rank, local row,
    contribution storage array [disp])] in request order, one per row of every valid request of every well-formed bag.
    grad: [nbags, disp] storage array of t; weights: one per request (storage values / bits of t), sum only."""
    lenlist = po.lenlist_of(shards)
    reqs = po.requests(**req)
    nreq = len(reqs)
    nbags = nreq if bags is None else len(bags) - 1
    bounds = pl.bag_bounds(bags, nbags, nreq)
    codes, locs = [], []
    for start, count, id_ok in reqs:
        code, r, off = (po.CODE_SAMPLE, 0, 0) if not id_ok else po.locate(lenlist, start, count)
        codes.append(code)
        locs.append((r, start - off, count))
    wv = pl.decode(np.asarray(weights, pl.STORAGE[t]), t) if weights is not None else None
    grad = np.asarray(grad).reshape(nbags, -1)
    writes, ns = [], []
    for k, bd in enumerate(bounds):
        if bd is None:
            ns.append(0)
            continue
        valid = [i for i in range(*bd) if not codes[i]]
        n = sum(locs[i][2] for i in valid)
        ns.append(n)
        for i in valid:
            c = contribution(grad[k], t, None if wv is None else wv[i], n if mode == pl.POOL_MEAN else 0, alpha)
            c = c.view(ao.STORAGE[t])
            r, local, count = locs[i]
            writes.extend((r, row, c) for row in range(local, local + count))
    badbag = next((k for k, bd in enumerate(bounds) if bd is None), -1)
    if badbag >= 0:
        return writes, ns, (pl.CODE_BAG, badbag)
    covered = sorted(i for bd in bounds for i in range(*bd) if codes[i])
    return writes, ns, ((codes[covered[0]], covered[0]) if covered else (0, -1))


def apply(shards, writes, t):
    """shards (not modified) with every contribution added, one correctly rounded addition each, in list order"""
    new = [np.array(s, copy=True) for s in shards]
    for r, row, c in writes:
        new[r][row] = ao.add(new[r][row], c, t)
    return new


def per_row(writes):
    """{(rank, local row): [contribution arrays]}"""
    out = {}
    for r, row, c in writes:
        out.setdefault((r, row), []).append(c)
    return out
