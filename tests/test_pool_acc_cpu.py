"""CPU checks of the pooled accumulates' oracle (tests/pool_acc_oracle.py), of their C declarations, and of the Python
argument checks of PyDDStore.accumulate_batch_pooled / accumulate_samples_pooled against a recording library (the
pattern of tests/test_binding_calls_cpu.py): accepted calls reach the right symbol with the right ABI arguments,
refused ones reach no call."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from ddstore_b200 import _capi
from ddstore_b200.store import PyDDStore
from tests import pool_acc_oracle as pao
from tests import pool_oracle as pl
from tests.test_binding_calls_cpu import _BYREF, H, SRC, TOTAL, _Lib

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = [pl.ACC_F32, pl.ACC_F64, pl.ACC_F16, pl.ACC_BF16]
TORCH = {pl.ACC_F32: torch.float32, pl.ACC_F64: torch.float64, pl.ACC_F16: torch.float16, pl.ACC_BF16: torch.bfloat16}


def _storage(v, t):
    """float values -> storage array of t (bf16: bits)"""
    v = np.asarray(v, np.float64)
    return pl.encode(v.astype(pl.acc_dtype(t)), t) if t == pl.ACC_BF16 else v.astype(pl.STORAGE[t])


def _rand(rng, n, t, spread=8):
    return _storage(rng.standard_normal(n) * 2.0 ** rng.integers(-spread, spread, n), t)


# ------------------------------------------------------------------------------------------------ the contribution rule
@pytest.mark.parametrize("t", TYPES)
def test_contribution_is_each_step_rounded_once(t):
    """against exact rationals: every step (weight, mean, alpha) is one round-to-nearest of the exact result"""
    rng = np.random.default_rng(t)
    dt = pl.acc_dtype(t)
    g, w = _rand(rng, 200, t), _rand(rng, 200, t, 2)
    for weighted, n, alpha in ((True, 0, -0.01), (False, 7, 0.3), (False, 0, 1.0), (True, 0, 1e-3)):
        for j in range(len(g)):
            got = pao.contribution(g[j:j + 1], t, pl.decode(w[j:j + 1], t)[0] if weighted else None, n, alpha)
            c = pl.decode(g[j:j + 1], t)[0]
            if weighted:
                c = pl.round_fraction(Fraction(float(c)) * Fraction(float(pl.decode(w[j:j + 1], t)[0])), dt)
            if n:
                c = pl.round_fraction(Fraction(float(c)) / n, dt)
            c = pl.round_fraction(Fraction(float(c)) * Fraction(float(dt(alpha))), dt)
            assert got.tolist() == pl.encode(np.array([c], dt), t).tolist(), (t, j, weighted, n, alpha)


@pytest.mark.parametrize("t", TYPES)
def test_contribution_matches_torch_cpu(t):
    """against torch's CPU expression ((g.float()[bag] * w) / n * alpha).to(dtype), element for element"""
    rng = np.random.default_rng(10 + t)
    g = _rand(rng, 4096, t)
    w = _rand(rng, 4096, t, 2)
    up = torch.float64 if t == pl.ACC_F64 else torch.float32
    tg = torch.from_numpy(g.view(np.int16) if t == pl.ACC_BF16 else g)
    tw = torch.from_numpy(w.view(np.int16) if t == pl.ACC_BF16 else w)
    if t == pl.ACC_BF16:
        tg, tw = tg.view(torch.bfloat16), tw.view(torch.bfloat16)
    bits = (lambda x: x.view(torch.int16).numpy().view(np.uint16)) if t == pl.ACC_BF16 else (
        lambda x: x.numpy().view(pl.BITS[t]))
    alpha = -0.0375
    wv = pl.decode(w, t)
    got = np.concatenate([pao.contribution(g[j:j + 1], t, wv[j], 0, alpha) for j in range(len(g))])
    ref = ((tg.to(up) * tw.to(up)) * alpha).to(TORCH[t])
    assert (got == bits(ref)).all()
    got = pao.contribution(g, t, None, 13, alpha)
    ref = ((tg.to(up) / 13) * alpha).to(TORCH[t])
    assert (got == bits(ref)).all()


def test_contribution_nan_is_canonical():
    for t in TYPES:
        g = _storage([np.inf, 1.0], t)
        got = pao.contribution(g, t, None, 0, 0.0)  # inf * 0
        assert got[0] == pl.CANONICAL_NAN[t] and pl.decode_bits(got[1:], t)[0] == 0


# ------------------------------------------------------------------------------------------------ bags and errors
def _world():
    return [np.zeros((6, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((5, 3), np.float32)]


def test_mean_counts_only_valid_rows():
    """n_k is the rows the forward folds: an invalid request is left out, and the first one is reported"""
    shards = _world()
    grad = np.array([[6.0, 12.0, -3.0], [8.0, 8.0, 8.0]], np.float32)
    starts, counts = [0, 20, 7, 9], [2, 1, 1, 2]  # request 1 is out of range; bag 0 = requests 0-2, bag 1 = request 3
    writes, ns, err = pao.contributions(shards, pl.ACC_F32, pl.POOL_MEAN, grad, bags=[0, 3, 4], starts=starts,
                                        counts=counts)
    assert ns == [3, 2] and err[1] == 1
    new = pao.apply(shards, writes, pl.ACC_F32)
    assert new[0][:2].tolist() == [[2.0, 4.0, -1.0]] * 2 and new[2][1].tolist() == [2.0, 4.0, -1.0]
    assert new[2][3:5].tolist() == [[4.0, 4.0, 4.0]] * 2 and not new[0][2:].any() and not new[2][0].any()
    pooled, _, _ = pl.pool([s + 1 for s in shards], pl.ACC_F32, pl.POOL_MEAN, bags=[0, 3, 4], starts=starts,
                           counts=counts)
    assert pooled.view(np.float32)[:, 0].tolist() == [1.0, 1.0]  # (the forward folds the same 3 and 2 rows)


def test_malformed_bag_writes_nothing_and_comes_first():
    shards = _world()
    grad = np.ones((3, 3), np.float32)
    writes, ns, err = pao.contributions(shards, pl.ACC_F32, pl.POOL_SUM, grad, bags=[0, 2, 1, 3], starts=[0, 30, 2],
                                        counts=[1, 1, 1])
    assert err == (pl.CODE_BAG, 1)  # bag 1 ([2, 1)) beats request 1 (out of range)
    assert [(r, row) for r, row, _ in writes] == [(0, 0), (0, 2)]


def test_uncovered_requests_are_not_validated():
    writes, ns, err = pao.contributions(_world(), pl.ACC_F32, pl.POOL_SUM, np.ones((1, 3), np.float32), bags=[0, 1],
                                        starts=[3, 99], counts=[1, 1])
    assert err == (0, -1) and len(writes) == 1


def test_weighted_duplicates_sum_exactly():
    shards = _world()
    grad = np.array([[1.0, 2.0, 3.0]], np.float32)
    writes, _, _ = pao.contributions(shards, pl.ACC_F32, pl.POOL_SUM, grad, bags=[0, 3],
                                     weights=np.array([2, -1, 4], np.float32), alpha=0.5, starts=[4, 4, 7],
                                     counts=[1, 1, 1])
    new = pao.apply(shards, writes, pl.ACC_F32)
    assert new[0][4].tolist() == [0.5, 1.0, 1.5] and new[2][1].tolist() == [2.0, 4.0, 6.0]
    assert len(pao.per_row(writes)[(0, 4)]) == 2


# ------------------------------------------------------------------------------------------------ declarations
def test_declarations_are_plain_c(tmp_path):
    src = tmp_path / "use_pool_acc.c"
    src.write_text('#include "ddstore_b200.h"\n'
                   'int main(void) { dds_pool_t p = {DDS_POOL_MEAN, DDS_ACC_F32, 0, 0, 0}; int64_t t, b;\n'
                   '  return dds_accumulate_batch_pooled(0, "x", 0, 0, 1, 0, &p, -0.5, 0, 0, DDS_SRC_ON_DEVICE, 0, &t, &b)\n'
                   '       + dds_accumulate_samples_pooled(0, "x", 0, 0, &p, 1.0, 0, 0, 0, 0, &t, &b); }\n')
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I",
                        os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ------------------------------------------------------------------------------------------------ Python argument checks
class _FakeCuda(torch.Tensor):
    """a host tensor the bindings take for a CUDA one (its address is only recorded, never read)"""

    @property
    def is_cuda(self):
        return True


def _grad(n, dtype=torch.float32, contiguous=True):
    t = torch.zeros(n, 2 * 3, dtype=dtype)[:, :3] if not contiguous else torch.zeros(n, 3, dtype=dtype)
    return torch.Tensor._make_subclass(_FakeCuda, t)


@pytest.fixture
def store():
    s = PyDDStore.__new__(PyDDStore)
    s._L, s._h = _Lib(), C.c_void_p(H)
    s._itemsize, s._cname, s._rowbytes = {}, {}, {}
    s.rank, s.size, s.last_bad_index = 0, 1, -1
    yield s
    s._h = None


def _pool_fields(p):
    return (p.mode, p.dtype, p.nbags, bool(p.bags), bool(p.weights))


class _RawLib(_Lib):
    """_Lib recording each call's raw arguments (the pooled entries pass their dds_pool_t by reference)"""

    def __getattr__(self, sym):
        if not sym.startswith("dds_"):
            raise AttributeError(sym)

        def fn(*args):
            self.calls.append((sym, args))
            outs = [a._obj for a in args if isinstance(a, _BYREF) and isinstance(a._obj, C.c_int64)]
            outs[0].value, outs[1].value = TOTAL, self.bad
            return 0
        return fn


def test_accumulate_pooled_abi(store):
    store._L = _RawLib()
    g = _grad(2)
    assert store.accumulate_batch_pooled("emb", [1, 2, 3], grad=g, bags=[0, 2, 3], mode="mean", alpha=-0.25) == TOTAL
    sym, args = store._L.calls.pop()
    assert sym == "dds_accumulate_batch_pooled" and args[1] == b"emb" and args[4] == 1 and args[5] == 3
    assert _pool_fields(args[6]._obj) == (_capi.POOL_MEAN, _capi.ACC_TYPES["float32"], 2, True, False)
    assert args[7] == -0.25 and args[8] == g.data_ptr() and args[9] == 2 * 3 * 4
    assert args[10] == SRC  # host indices, synchronous
    g = _grad(2, torch.float64)
    assert store.accumulate_samples_pooled("emb", [4, 5], g, weights=[1.0, 2.0], stream=7, wait=True) == TOTAL
    sym, args = store._L.calls.pop()
    assert sym == "dds_accumulate_samples_pooled" and args[3] == 2
    assert _pool_fields(args[4]._obj) == (_capi.POOL_SUM, _capi.ACC_TYPES["float64"], 2, False, True)
    assert args[5] == 1.0 and args[6] == g.data_ptr() and args[7] == 2 * 3 * 8 and args[8] == SRC


@pytest.mark.parametrize("kw, msg", [
    (dict(mode="max"), "mode 'max' has no adjoint"),
    (dict(mode="median"), "mode 'median' is not one of"),
    (dict(alpha=float("nan")), "alpha must be finite"),
    (dict(alpha=float("-inf")), "alpha must be finite"),
    (dict(alpha=None), "alpha must be finite"),  # (never taken for a pooled get)
    (dict(grad=torch.zeros(2, 3)), "grad must be a C-contiguous CUDA tensor"),
    (dict(grad=None), "grad must be a C-contiguous CUDA tensor"),
    (dict(grad=_grad(2, contiguous=False)), "grad must be a C-contiguous CUDA tensor"),
    (dict(grad=_grad(2, torch.int32)), "grad dtype int32 is not float32"),
])
def test_refused_before_any_call(store, kw, msg):
    args = dict(grad=_grad(2), bags=[0, 1, 2], mode="sum", alpha=1.0)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        store.accumulate_batch_pooled("emb", [0, 1], **args)
    with pytest.raises(ValueError, match=msg):
        store.accumulate_samples_pooled("emb", [0, 1], **args)
    assert store._L.calls == []


def test_max_is_refused_before_alpha_and_grad(store):
    with pytest.raises(ValueError, match="max"):
        store.accumulate_batch_pooled("emb", [0], grad=None, mode="max", alpha=float("nan"))
    assert store._L.calls == []
