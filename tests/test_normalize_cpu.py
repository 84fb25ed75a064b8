"""The normalising conversions without a GPU: the NumPy oracle of tests/norm_oracle.py against torch's CPU expression
((x.float() - mean) / std).to(dtype) bitwise (NaN by class), over the float32 rounding edges in the values and in the
tables; the channel rule against reshape-based torch expressions for every layout; and the argument checks that need
no device."""
import ctypes

import numpy as np
import pytest

from tests import convert_oracle as co
from tests import norm_oracle as no

torch = pytest.importorskip("torch")

OUT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
SRC = {"f32": torch.float32, "f64": torch.float64, "u8": torch.uint8}


def _torch_ref(x, code, mean, std, nchan, inner, lut=None):
    """torch's CPU expression on the values of a packed variable: mean / std broadcast by the channel rule"""
    n = x.numel()
    ch = torch.from_numpy(no.channels(n, nchan, inner))
    m, s = torch.from_numpy(np.asarray(mean, np.float32))[ch], torch.from_numpy(np.asarray(std, np.float32))[ch]
    xf = lut[x.long()] if no.NORM[code][2] == "u8" else x.to(torch.float32)
    return ((xf - m) / s).to(OUT[no.NORM[code][3]]).view(torch.uint8).numpy().reshape(-1)


def _values(kind, rng, n):
    if kind == "u8":
        return rng.integers(0, 256, n).astype(np.uint8)
    edges = np.array(co.F32_EDGE_BITS, np.uint32).view(np.float32)
    v = np.concatenate([edges, -edges, rng.standard_normal(n).astype(np.float32) * 3,
                        rng.integers(0, 2 ** 32, n, dtype=np.uint32).view(np.float32)])
    if kind == "f64":
        return np.concatenate([co.f64_edge_bits().view(np.float64), v.astype(np.float64)])
    return v


@pytest.mark.parametrize("code", sorted(no.NORM))
@pytest.mark.parametrize("tables", ["edges", "random"])
def test_oracle_matches_torch_cpu(code, tables):
    rng = np.random.default_rng(code)
    x = _values(no.NORM[code][2], rng, 3000)
    if tables == "edges":
        mean, std = no.TABLE_EDGE_MEAN, no.TABLE_EDGE_STD
    else:
        mean = rng.standard_normal(7).astype(np.float32)
        std = (rng.random(7).astype(np.float32) + 0.05) * rng.choice([-1, 1], 7).astype(np.float32)
    nchan = len(mean)
    x = x[: x.size - x.size % nchan]  # whole rows of disp = nchan
    lut = torch.arange(256, dtype=torch.float32).div(255) if no.NORM[code][2] == "u8" else None
    got = no.norm_bytes(x.view(np.uint8), code, mean, std, nchan, 1, None if lut is None else lut.numpy())
    exp = _torch_ref(torch.from_numpy(x), code, mean, std, nchan, 1, lut)
    bad = no.bad_elements(got, exp, code)
    assert bad.size == 0, f"{bad.size} elements differ, first {bad[0]}"


def test_edges_reach_the_interesting_results():
    """the edge tables produce what they are there for: +-inf and NaN from std = 0, f16 / bf16 overflow and subnormal
    results, -0"""
    x = np.array(co.F32_EDGE_BITS, np.uint32).view(np.float32)
    x = np.resize(x, 12 * 40)
    y = no.normalise(x, no.TABLE_EDGE_MEAN, no.TABLE_EDGE_STD, 12, 1)
    assert np.isinf(y).any() and np.isnan(y).any()
    h = y.astype(np.float16)
    assert np.isinf(h[np.isfinite(y)]).any(), "no f16 overflow"
    sub = (np.abs(y) < 6.1e-5) & (y != 0)
    assert sub.any(), "no f16 subnormal range result"
    assert (np.signbit(y) & (y == 0)).any(), "no -0"


@pytest.mark.parametrize("layout", ["scalar", "per_feature", "hwc", "chw", "divisor"])
def test_channel_rule_matches_reshape(layout):
    """(e mod (nchan * inner)) // inner against the way a user writes each layout in torch"""
    rng = np.random.default_rng(1)
    C, H, W, B = 3, 4, 5, 6
    disp, nchan, inner = {"scalar": (37, 1, 1), "per_feature": (37, 37, 1), "hwc": (H * W * C, C, 1),
                          "chw": (C * H * W, C, H * W), "divisor": (12, 2, 3)}[layout]
    x = torch.from_numpy(rng.standard_normal((B, disp)).astype(np.float32))
    mean = torch.from_numpy(rng.standard_normal(nchan).astype(np.float32))
    std = torch.from_numpy(rng.random(nchan).astype(np.float32) + 0.5)
    if layout == "scalar":
        ref = (x - mean) / std
    elif layout == "per_feature":
        ref = (x - mean.view(1, -1)) / std.view(1, -1)
    elif layout == "hwc":
        ref = ((x.view(B, H, W, C) - mean.view(1, 1, 1, C)) / std.view(1, 1, 1, C)).reshape(B, disp)
    elif layout == "chw":  # torchvision's Normalize on a CHW image
        ref = ((x.view(B, C, H, W) - mean.view(1, C, 1, 1)) / std.view(1, C, 1, 1)).reshape(B, disp)
    else:  # rows of 12 = 2 repetitions of (2 channels x 3 elements)
        ref = ((x.view(B, 2, nchan, inner) - mean.view(1, 1, nchan, 1)) / std.view(1, 1, nchan, 1)).reshape(B, disp)
    got = no.normalise(x.numpy().reshape(-1), mean.numpy(), std.numpy(), nchan, inner).reshape(B, disp)
    assert np.array_equal(got.view(np.uint32), ref.numpy().view(np.uint32))
    # a request starting at any row keeps the pattern (every request starts at a row boundary)
    assert np.array_equal(no.channels(disp, nchan, inner, first=5 * disp), no.channels(disp, nchan, inner))


def test_python_argument_checks():
    from ddstore_b200 import _capi
    from ddstore_b200.dataset import _norm_spec
    from ddstore_b200.store import PyDDStore, _conversion, _norm_tables
    pairs = {("float32", "float32"): 6, ("float32", "bfloat16"): 7, ("float32", "float16"): 8, ("float64", "float32"): 9,
             ("uint8", "float32"): 10, ("uint8", "bfloat16"): 11, ("uint8", "float16"): 12}
    for (s, o), code in pairs.items():
        cv, keep = _conversion(getattr(torch, s), getattr(torch, o), None, normalize=True)
        assert cv.code == code
        if s == "uint8":  # the default decode table: the plain value, as 256 float32 entries
            assert keep.dtype == np.int32 and np.array_equal(keep.view(np.float32), np.arange(256, dtype=np.float32))
    for s, o in (("float64", "bfloat16"), ("int32", "float32"), ("float32", "float64"), ("uint8", "uint8")):
        with pytest.raises(ValueError, match="normalising"):
            _conversion(getattr(torch, s), getattr(torch, o), None, normalize=True)
    with pytest.raises(ValueError):  # without normalize, f32 -> f32 is still no conversion
        _conversion(torch.float32, torch.float32, None)
    with pytest.raises(ValueError):  # the uint8 decode table of a normalising batch is float32
        _conversion(torch.uint8, torch.bfloat16, torch.arange(256).to(torch.bfloat16), normalize=True)
    with pytest.raises(ValueError):
        _conversion(torch.float32, torch.bfloat16, torch.zeros(256), normalize=True)
    _, keep = _conversion(torch.uint8, torch.float16, torch.arange(256, dtype=torch.float32) / 255, normalize=True)
    assert np.array_equal(keep.view(np.float32), (torch.arange(256, dtype=torch.float32) / 255).numpy())
    m, s, n, dev = _norm_tables(np.zeros(3, np.float32), torch.ones(3))
    assert n == 3 and dev == 0
    for mean, std in ((np.zeros(3), np.ones(3, np.float32)), (np.zeros(3, np.float32), np.ones(4, np.float32)),
                      (np.zeros((3, 1), np.float32), np.ones((3, 1), np.float32)), (torch.zeros(3, dtype=torch.int32),
                                                                                    torch.ones(3))):
        with pytest.raises(ValueError):
            _norm_tables(mean, std)
    with pytest.raises(TypeError):
        _norm_tables([0.0], [1.0])
    assert _norm_spec(([0.5, 0.25], [2, 4]))[2] == 1 and _norm_spec(([0.5], [2], 1024))[2] == 1024
    assert _norm_spec(([0.5, 0.25], [2, 4]))[0].dtype == np.float32
    with pytest.raises(ValueError):
        _norm_spec(([0.5],))
    bare = object.__new__(PyDDStore)  # (the checks run before the store is touched)
    with pytest.raises(ValueError, match="needs src_dtype"):
        bare.get_batch("x", [0], out=torch.empty(4), normalize=True)
    with pytest.raises(ValueError, match="needs src_dtype"):
        bare.get_samples("x", [0], torch.empty(4), normalize=True)
    with pytest.raises(ValueError, match="one entry per variable"):
        bare.get_samples_multi(["x", "y"], [0], [torch.empty(4)] * 2, src_dtypes=[torch.float32] * 2, normalize=[True])
    with pytest.raises(ValueError, match="src_dtypes entry"):
        bare.get_samples_multi(["x", "y"], [0], [torch.empty(4)] * 2, src_dtypes=[None, torch.float32],
                               normalize=[True, False])
    # the C entry checks its store first
    assert _capi.lib().dds_set_normalization(None, b"x", None, None, 1, 1, 0) == _capi.ERR_ARG
    L = _capi.lib()
    assert L.dds_set_normalization.argtypes[4] is ctypes.c_int64


def test_header_codes_match_the_bindings():
    """the DDS_CVT_NORM_* values and DDS_VERSION of the header are the ones the bindings and the oracle use"""
    import os
    import re
    from ddstore_b200 import _capi
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "ddstore_b200.h")).read()
    defs = {k: int(v) for k, v in re.findall(r"#define (DDS_CVT_NORM_\w+) (\d+)", hdr)}
    assert len(defs) == 7
    for k, v in defs.items():
        assert getattr(_capi, k[len("DDS_"):]) == v == getattr(no, k[len("DDS_"):])
    assert re.search(r"#define DDS_VERSION 111\b", hdr)
