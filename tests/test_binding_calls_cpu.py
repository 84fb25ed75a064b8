"""CPU-only checks of what the ctypes binding hands the C-ABI: every public batched method of PyDDStore (the pooled pair
aside, which needs real CUDA tensors) is driven against a recording stand-in for the library, and each call's symbol
and every ABI argument are compared with the expected ones. Host index arrays are recorded as the int64 values they
hold during the call, `byref` structs by their fields, and every other pointer by the address it converts to. Refused
inputs are checked to reach no library call, and to raise the message of the argument checked first."""
import ctypes as C

import numpy as np
import pytest

from ddstore_b200 import _capi
from ddstore_b200.store import PyDDStore

torch = pytest.importorskip("torch")

H = 0x5000          # the store handle
TOTAL = 4242        # what the stand-in reports as the call's total
IDX, DST, SRC, NOSYNC, OVL = _capi.IDX_ON_DEVICE, _capi.DST_ON_DEVICE, _capi.SRC_ON_DEVICE, _capi.NO_SYNC, _capi.OVERLAP
OUT = "out"         # a byref int64 the library writes

# symbol -> (positions of the index arrays, position of their length, position of the flags word)
_INDEX_ARGS = {
    "dds_get_batch": ((2, 3), 5, 10),
    "dds_get_batch_convert": ((2, 3), 5, 9),
    "dds_get_batch_padded": ((2, 3), 4, 10),
    "dds_get_samples": ((2,), 3, 8),
    "dds_get_samples_convert": ((2,), 3, 7),
    "dds_get_samples_padded": ((2,), 3, 9),
    "dds_get_samples_multi": ((3,), 4, 8),
    "dds_get_samples_multi_convert": ((3,), 4, 8),
    "dds_put_batch": ((2, 3), 5, 9),
    "dds_put_samples": ((2,), 3, 7),
    "dds_accumulate_op_batch": ((2, 3), 5, 10),
    "dds_accumulate_op_samples": ((2,), 3, 8),
    "dds_get_accumulate_batch": ((2, 3), 5, 11),
    "dds_get_accumulate_samples": ((2,), 3, 9),
    "dds_compare_and_swap_batch": ((2, 3), 5, 11),
    "dds_compare_and_swap_samples": ((2,), 3, 9),
    "dds_set_sample_index": ((2, 3), 4, 5),
}
_LUT_BYTES = {_capi.CVT_U8_LUT16: 512, _capi.CVT_U8_LUT32: 1024, _capi.CVT_NORM_U8_F32: 1024,
              _capi.CVT_NORM_U8_BF16: 1024, _capi.CVT_NORM_U8_F16: 1024}
_BYREF = type(C.byref(C.c_int()))


def _addr(a):
    if a is None:
        return 0
    if isinstance(a, C.c_void_p):
        return a.value or 0
    return int(a)


def _cvt(c):
    lut = C.string_at(c.lut, _LUT_BYTES[c.code]) if c.lut else 0
    return ("cvt", c.code, lut)


def _norm(a):
    if isinstance(a, bytes):
        return a
    if isinstance(a, _BYREF):
        o = a._obj
        if isinstance(o, C.c_int64):
            return OUT
        if isinstance(o, _capi.Convert):
            return _cvt(o)
        if isinstance(o, _capi.Pad):
            return ("pad", o.max_rows, o.pad_bits, o.lengths or 0)
        raise AssertionError(f"unexpected byref {type(o).__name__}")
    if isinstance(a, C.Array):
        if a._type_ is _capi.Convert:
            return [_cvt(c) for c in a]
        if a._type_ is C.c_char_p:
            return list(a)
        return [_addr(v) for v in a]
    return _addr(a)


class _Lib:
    """stands in for the loaded library: records every call with its arguments normalised, answers the variable
    queries (itemsize 4, 3 elements per row) and reports TOTAL bytes and `bad` as the first invalid request"""

    def __init__(self):
        self.calls = []
        self.bad = -1

    def dds_query(self, h, name, vi):
        vi._obj.itemsize, vi._obj.disp = 4, 3
        return 0

    def dds_query_placement(self, h, name, pl):
        pl._obj.value = 0
        return 0

    def __getattr__(self, sym):
        if not sym.startswith("dds_"):
            raise AttributeError(sym)

        def fn(*args):
            rec = [_norm(a) for a in args]
            if sym in _INDEX_ARGS:
                pos, npos, fpos = _INDEX_ARGS[sym]
                n, on_dev = int(args[npos]), int(args[fpos]) & IDX
                for p in pos:
                    a = _addr(args[p])
                    rec[p] = None if not a else a if on_dev else list(np.ctypeslib.as_array((C.c_int64 * n).from_address(a)))
            self.calls.append((sym, tuple(rec)))
            if "multi" in sym:
                for v in range(int(args[1])):
                    args[-2][v] = 100 + v
            outs = [a._obj for a in args if isinstance(a, _BYREF) and isinstance(a._obj, C.c_int64)]
            if len(outs) == 2:
                outs[0].value = TOTAL
            if outs:
                outs[-1].value = self.bad
            return 0
        return fn


class Dev:
    """a C-contiguous CUDA tensor as the bindings see it: a device address, a size and a torch dtype"""
    is_cuda = True

    def __init__(self, ptr, n, dtype=torch.float32, contiguous=True):
        self.ptr, self.n, self.dtype, self._contig = ptr, n, dtype, contiguous
        self.shape = (n,)

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n

    def element_size(self):
        return torch.empty(0, dtype=self.dtype).element_size()

    def is_contiguous(self):
        return self._contig

    def contiguous(self):
        return self

    def dim(self):
        return 1


@pytest.fixture
def store():
    s = PyDDStore.__new__(PyDDStore)
    s._L, s._h = _Lib(), C.c_void_p(H)
    s._itemsize, s._cname, s._rowbytes = {}, {}, {}
    s.rank, s.size, s.last_bad_index = 0, 1, -1
    yield s
    s._h = None  # (nothing to close)


def _one(store):
    calls = [c for c in store._L.calls]
    store._L.calls.clear()
    assert len(calls) == 1, calls
    return calls[0]


def _lut(t):
    t = t.reshape(-1).contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).numpy().tobytes()


# ------------------------------------------------------------------------------------------------ get_batch
def test_get_batch_raw(store):
    out = Dev(0xA000, 96)
    assert store.get_batch("x", [3, 1, 4], [1, 5, 9], out=out) == TOTAL
    assert _one(store) == ("dds_get_batch", (H, b"x", [3, 1, 4], [1, 5, 9], 1, 3, 4, 0xA000, 384, 0, DST, 0, OUT, OUT))
    host = np.zeros(10, np.float32)
    assert store.get_batch("x", np.array([7, 8], np.int32), out=host, count=2) == TOTAL
    assert _one(store) == ("dds_get_batch", (H, b"x", [7, 8], None, 2, 2, 4, host.ctypes.data, 40, 0, 0, 0, OUT, OUT))
    s, c, offs = Dev(0xB000, 3, torch.int64), Dev(0xC000, 3, torch.int64), Dev(0xD000, 4, torch.int64)
    store.get_batch("x", s, c, out=out, offsets=offs, stream=0, wait=False, overlap=True)
    assert _one(store) == ("dds_get_batch", (H, b"x", 0xB000, 0xC000, 1, 3, 4, 0xA000, 384, 0xD000,
                                             IDX | DST | NOSYNC | OVL, 1, OUT, OUT))
    store.get_batch("x", s, out=out, count=5, stream=0x1234, wait=False)
    assert _one(store) == ("dds_get_batch", (H, b"x", 0xB000, None, 5, 3, 4, 0xA000, 384, 0, IDX | DST | NOSYNC,
                                             0x1234, OUT, OUT))
    store.get_batch("x", s, out=out, overlap=True, stream=None)  # (overlap only applies to queued batches)
    assert _one(store) == ("dds_get_batch", (H, b"x", 0xB000, None, 1, 3, 4, 0xA000, 384, 0, IDX | DST, 0, OUT, OUT))


def test_get_batch_reports_the_first_invalid_request(store):
    store._L.bad = 2
    store.get_batch("x", [0, 1, 2], out=Dev(0xA000, 9))
    assert store.last_bad_index == 2
    _one(store)


def test_get_batch_converting(store):
    out = Dev(0xA000, 64, torch.bfloat16)
    store.get_batch("x", [1, 2], [3, 4], out=out, src_dtype=torch.float32)
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", [1, 2], [3, 4], 1, 2, 0xA000, 128, 0, DST, 0,
                                                     ("cvt", _capi.CVT_F32_BF16, 0), OUT, OUT))
    lut = torch.arange(256).flip(0).to(torch.bfloat16)
    s, offs = Dev(0xB000, 2, torch.int64), Dev(0xD000, 3, torch.int64)
    store.get_batch("x", s, out=out, count=3, offsets=offs, src_dtype=np.uint8, lut=lut, stream=7, wait=False)
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", 0xB000, None, 3, 2, 0xA000, 128, 0xD000,
                                                     IDX | DST | NOSYNC, 7, ("cvt", _capi.CVT_U8_LUT16, _lut(lut)),
                                                     OUT, OUT))
    out32 = Dev(0xA000, 64, torch.float32)
    store.get_batch("x", [5], out=out32, src_dtype="uint8")
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", [5], None, 1, 1, 0xA000, 256, 0, DST, 0,
                                                     ("cvt", _capi.CVT_U8_LUT32, _lut(torch.arange(256).float())),
                                                     OUT, OUT))


def test_get_batch_normalising(store):
    out = Dev(0xA000, 64, torch.float32)
    store.get_batch("x", [1], out=out, src_dtype=torch.float32, normalize=True)
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", [1], None, 1, 1, 0xA000, 256, 0, DST, 0,
                                                     ("cvt", _capi.CVT_NORM_F32_F32, 0), OUT, OUT))
    outb = Dev(0xA000, 64, torch.bfloat16)
    store.get_batch("x", [1], [2], out=outb, src_dtype=torch.uint8, normalize=True)
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", [1], [2], 1, 1, 0xA000, 128, 0, DST, 0,
                                                     ("cvt", _capi.CVT_NORM_U8_BF16, _lut(torch.arange(256).float())),
                                                     OUT, OUT))
    lut = torch.linspace(-1, 1, 256)
    store.get_batch("x", [1], out=outb, src_dtype=torch.uint8, normalize=True, lut=lut)
    assert _one(store) == ("dds_get_batch_convert", (H, b"x", [1], None, 1, 1, 0xA000, 128, 0, DST, 0,
                                                     ("cvt", _capi.CVT_NORM_U8_BF16, _lut(lut)), OUT, OUT))


def test_get_batch_padded(store):
    out, lens = Dev(0xA000, 72), Dev(0xE000, 3, torch.int64)
    bits = int(torch.tensor([-2.0]).view(torch.int32).item()) & 0xFFFFFFFF
    assert store.get_batch("x", [0, 4, 8], [1, 2, 3], out=out, pad_rows=2, pad_value=-2.0, lengths=lens) == TOTAL
    assert _one(store) == ("dds_get_batch_padded", (H, b"x", [0, 4, 8], [1, 2, 3], 3, 4, 0, ("pad", 2, bits, 0xE000),
                                                    0xA000, 288, DST, 0, OUT, OUT))
    s, c = Dev(0xB000, 3, torch.int64), Dev(0xC000, 3, torch.int64)
    outh = Dev(0xA000, 72, torch.float16)
    nan = torch.tensor([float("nan")], dtype=torch.float16)
    store.get_batch("x", s, c, out=outh, src_dtype=torch.float32, pad_rows=4, pad_value=nan, wait=False, overlap=True,
                    stream=0)
    assert _one(store) == ("dds_get_batch_padded", (H, b"x", 0xB000, 0xC000, 3, 4, ("cvt", _capi.CVT_F32_F16, 0),
                                                    ("pad", 4, int(nan.view(torch.int16).item()) & 0xFFFF, 0),
                                                    0xA000, 144, IDX | DST | NOSYNC | OVL, 1, OUT, OUT))
    outi = Dev(0xA000, 72, torch.int32)
    store.get_batch("x", [1], [1], out=outi, pad_rows=0, pad_value=-1)
    assert _one(store) == ("dds_get_batch_padded", (H, b"x", [1], [1], 1, 4, 0, ("pad", 0, 0xFFFFFFFF, 0), 0xA000,
                                                    288, DST, 0, OUT, OUT))


# ------------------------------------------------------------------------------------------------ get_samples
def test_get_samples(store):
    out = Dev(0xA000, 96)
    assert store.get_samples("x", [9, 2], out) == TOTAL
    assert _one(store) == ("dds_get_samples", (H, b"x", [9, 2], 2, 4, 0xA000, 384, 0, DST, 0, OUT, OUT))
    host, hoffs = np.zeros(12, np.int32), np.zeros(3, np.int64)
    store.get_samples("x", np.array([1, 0]), host, offsets=hoffs)
    assert _one(store) == ("dds_get_samples", (H, b"x", [1, 0], 2, 4, host.ctypes.data, 48, hoffs.ctypes.data, 0, 0,
                                               OUT, OUT))
    ids, offs = Dev(0xB000, 5, torch.int64), Dev(0xD000, 6, torch.int64)
    store.get_samples("x", ids, out, offsets=offs, stream=0x99, wait=False, overlap=True)
    assert _one(store) == ("dds_get_samples", (H, b"x", 0xB000, 5, 4, 0xA000, 384, 0xD000, IDX | DST | NOSYNC | OVL,
                                               0x99, OUT, OUT))


def test_get_samples_converting_and_padded(store):
    out = Dev(0xA000, 96, torch.bfloat16)
    ids = Dev(0xB000, 5, torch.int64)
    store.get_samples("x", ids, out, src_dtype=torch.float32, stream=0)
    assert _one(store) == ("dds_get_samples_convert", (H, b"x", 0xB000, 5, 0xA000, 192, 0, IDX | DST, 1,
                                                       ("cvt", _capi.CVT_F32_BF16, 0), OUT, OUT))
    store.get_samples("x", [3], out, src_dtype=torch.uint8, normalize=True, wait=False)
    assert _one(store) == ("dds_get_samples_convert", (H, b"x", [3], 1, 0xA000, 192, 0, DST | NOSYNC,
                                                       0, ("cvt", _capi.CVT_NORM_U8_BF16,
                                                           _lut(torch.arange(256).float())), OUT, OUT))
    out32, lens = Dev(0xA000, 96), Dev(0xE000, 2, torch.int64)
    store.get_samples("x", [3, 4], out32, pad_rows=3, pad_value=7, lengths=lens)
    assert _one(store) == ("dds_get_samples_padded", (H, b"x", [3, 4], 2, 4, 0, ("pad", 3, 0x40E00000, 0xE000),
                                                      0xA000, 384, DST, 0, OUT, OUT))
    store.get_samples("x", ids, out, src_dtype=torch.float32, normalize=True, pad_rows=1, stream=5, wait=False)
    assert _one(store) == ("dds_get_samples_padded", (H, b"x", 0xB000, 5, 4, ("cvt", _capi.CVT_NORM_F32_BF16, 0),
                                                      ("pad", 1, 0, 0), 0xA000, 192, IDX | DST | NOSYNC, 5, OUT, OUT))


# ------------------------------------------------------------------------------------------------ get_samples_multi
def test_get_samples_multi(store):
    o1, o2 = Dev(0xA000, 16), Dev(0xA800, 8, torch.int64)
    assert store.get_samples_multi(["x", "y"], [4, 5, 6], [o1, o2]) == [100, 101]
    assert _one(store) == ("dds_get_samples_multi", (H, 2, [b"x", b"y"], [4, 5, 6], 3, [0xA000, 0xA800], [64, 64], 0,
                                                     DST, 0, [0, 0], OUT))
    ids, f1, f2 = Dev(0xB000, 3, torch.int64), Dev(0xD000, 4, torch.int64), Dev(0xD800, 4, torch.int64)
    assert store.get_samples_multi(["x", "y"], ids, [o1, o2], offsets=[f1, f2], stream=0, wait=False,
                                   overlap=True) is None
    assert _one(store) == ("dds_get_samples_multi", (H, 2, [b"x", b"y"], 0xB000, 3, [0xA000, 0xA800], [64, 64],
                                                     [0xD000, 0xD800], IDX | DST | NOSYNC | OVL, 1, [0, 0], OUT))
    store.get_samples_multi(["x"], ids, [o1], overlap=True, stream=0x42)
    assert _one(store) == ("dds_get_samples_multi", (H, 1, [b"x"], 0xB000, 3, [0xA000], [64], 0, IDX | DST, 0x42,
                                                     [0], OUT))


def test_get_samples_multi_converting(store):
    o1, o2, o3 = Dev(0xA000, 16, torch.bfloat16), Dev(0xA800, 8, torch.int64), Dev(0xB800, 8, torch.float16)
    lut = torch.arange(256).to(torch.float16)
    assert store.get_samples_multi(["x", "y", "z"], [1], [o1, o2, o3], src_dtypes=[torch.float32, None, torch.uint8],
                                   luts=[None, None, lut], normalize=[True, False, False]) == [100, 101, 102]
    assert _one(store) == ("dds_get_samples_multi_convert", (
        H, 3, [b"x", b"y", b"z"], [1], 1, [0xA000, 0xA800, 0xB800], [32, 64, 16], 0, DST, 0,
        [("cvt", _capi.CVT_NORM_F32_BF16, 0), ("cvt", _capi.CVT_NONE, 0), ("cvt", _capi.CVT_U8_LUT16, _lut(lut))],
        [0, 0, 0], OUT))
    ids = Dev(0xB000, 2, torch.int64)
    store.get_samples_multi(["x", "y"], ids, [o1, o2], src_dtypes=["float32", None], wait=False, stream=3)
    assert _one(store) == ("dds_get_samples_multi_convert", (
        H, 2, [b"x", b"y"], 0xB000, 2, [0xA000, 0xA800], [32, 64], 0, IDX | DST | NOSYNC, 3,
        [("cvt", _capi.CVT_F32_BF16, 0), ("cvt", _capi.CVT_NONE, 0)], [0, 0], OUT))


# ------------------------------------------------------------------------------------------------ writes
def test_put(store):
    src = Dev(0xF000, 12)
    assert store.put_batch("x", [2, 5], [1, 3], src=src) == TOTAL
    assert _one(store) == ("dds_put_batch", (H, b"x", [2, 5], [1, 3], 1, 2, 4, 0xF000, 48, SRC, 0, OUT, OUT))
    s, c = Dev(0xB000, 2, torch.int64), Dev(0xC000, 2, torch.int64)
    store.put_batch("x", s, c, src=src, stream=0, wait=False)
    assert _one(store) == ("dds_put_batch", (H, b"x", 0xB000, 0xC000, 1, 2, 4, 0xF000, 48, SRC | IDX | NOSYNC, 1,
                                             OUT, OUT))
    store.put_batch("x", s, src=Dev(0xF000, 24, torch.float16), count=4, stream=0x77)
    assert _one(store) == ("dds_put_batch", (H, b"x", 0xB000, None, 4, 2, 2, 0xF000, 48, SRC | IDX, 0x77, OUT, OUT))
    assert store.put_samples("x", [6], src) == TOTAL
    assert _one(store) == ("dds_put_samples", (H, b"x", [6], 1, 4, 0xF000, 48, SRC, 0, OUT, OUT))
    store.put_samples("x", s, src, stream=9, wait=False)
    assert _one(store) == ("dds_put_samples", (H, b"x", 0xB000, 2, 4, 0xF000, 48, SRC | IDX | NOSYNC, 9, OUT, OUT))


def test_accumulate(store):
    src = Dev(0xF000, 12)
    assert store.accumulate_batch("x", [2, 5], [1, 3], src=src) == TOTAL
    assert _one(store) == ("dds_accumulate_op_batch", (H, b"x", [2, 5], [1, 3], 1, 2, _capi.OP_SUM, _capi.ACC_F32,
                                                       0xF000, 48, SRC, 0, OUT, OUT))
    s = Dev(0xB000, 2, torch.int64)
    store.accumulate_batch("x", s, src=Dev(0xF000, 6, torch.int64), count=3, op="bitwise_or", stream=0, wait=False)
    assert _one(store) == ("dds_accumulate_op_batch", (H, b"x", 0xB000, None, 3, 2, _capi.OP_BOR, _capi.ACC_I64,
                                                       0xF000, 48, SRC | IDX | NOSYNC, 1, OUT, OUT))
    assert store.accumulate_samples("x", [1, 1], Dev(0xF000, 24, torch.bfloat16), op="amin") == TOTAL
    assert _one(store) == ("dds_accumulate_op_samples", (H, b"x", [1, 1], 2, _capi.OP_MIN, _capi.ACC_BF16, 0xF000,
                                                         48, SRC, 0, OUT, OUT))
    store.accumulate_samples("x", s, src, stream=0x10, wait=False)
    assert _one(store) == ("dds_accumulate_op_samples", (H, b"x", 0xB000, 2, _capi.OP_SUM, _capi.ACC_F32, 0xF000,
                                                         48, SRC | IDX | NOSYNC, 0x10, OUT, OUT))


def test_get_accumulate(store):
    src, out = Dev(0xF000, 12), Dev(0x9000, 16)
    assert store.get_accumulate_batch("x", [2, 5], [1, 3], src=src, out=out) == TOTAL
    assert _one(store) == ("dds_get_accumulate_batch", (H, b"x", [2, 5], [1, 3], 1, 2, _capi.OP_SUM, _capi.ACC_F32,
                                                        0xF000, 0x9000, 48, SRC, 0, OUT, OUT))
    s = Dev(0xB000, 2, torch.int64)
    store.get_accumulate_batch("x", s, src=src, out=src, op="replace", count=2, stream=0, wait=False)
    assert _one(store) == ("dds_get_accumulate_batch", (H, b"x", 0xB000, None, 2, 2, _capi.OP_REPLACE, _capi.ACC_F32,
                                                        0xF000, 0xF000, 48, SRC | IDX | NOSYNC, 1, OUT, OUT))
    assert store.get_accumulate_samples("x", [0], Dev(0xF000, 3, torch.int32), out, op="amax") == TOTAL
    assert _one(store) == ("dds_get_accumulate_samples", (H, b"x", [0], 1, _capi.OP_MAX, _capi.ACC_I32, 0xF000,
                                                          0x9000, 12, SRC, 0, OUT, OUT))
    store.get_accumulate_samples("x", s, src, out, op="bitwise_xor", stream=0x21, wait=False)
    assert _one(store) == ("dds_get_accumulate_samples", (H, b"x", 0xB000, 2, _capi.OP_BXOR, _capi.ACC_F32, 0xF000,
                                                          0x9000, 48, SRC | IDX | NOSYNC, 0x21, OUT, OUT))


def test_compare_and_swap(store):
    src, cmp, out = Dev(0xF000, 12), Dev(0x8000, 12, torch.int32), Dev(0x9000, 16)
    assert store.compare_and_swap_batch("x", [2, 5], [1, 3], src=src, compare=cmp, out=out) == TOTAL
    assert _one(store) == ("dds_compare_and_swap_batch", (H, b"x", [2, 5], [1, 3], 1, 2, 4, 0xF000, 0x8000, 0x9000,
                                                          48, SRC, 0, OUT, OUT))
    s = Dev(0xB000, 2, torch.int64)
    store.compare_and_swap_batch("x", s, src=src, compare=cmp, out=cmp, count=6, stream=0, wait=False)
    assert _one(store) == ("dds_compare_and_swap_batch", (H, b"x", 0xB000, None, 6, 2, 4, 0xF000, 0x8000, 0x8000,
                                                          48, SRC | IDX | NOSYNC, 1, OUT, OUT))
    b = Dev(0xF000, 8, torch.uint8)
    assert store.compare_and_swap_samples("x", [3], b, b, Dev(0x9000, 8, torch.bool)) == TOTAL
    assert _one(store) == ("dds_compare_and_swap_samples", (H, b"x", [3], 1, 1, 0xF000, 0xF000, 0x9000, 8, SRC, 0,
                                                            OUT, OUT))
    store.compare_and_swap_samples("x", s, src, cmp, out, stream=0x31, wait=False)
    assert _one(store) == ("dds_compare_and_swap_samples", (H, b"x", 0xB000, 2, 4, 0xF000, 0x8000, 0x9000, 48,
                                                            SRC | IDX | NOSYNC, 0x31, OUT, OUT))


# ------------------------------------------------------------------------------------------------ tables and wait
def test_set_sample_index_set_normalization_and_wait(store):
    store.set_sample_index("x", [0, 3, 7], np.array([3, 4, 1], np.int32))
    assert _one(store) == ("dds_set_sample_index", (H, b"x", [0, 3, 7], [3, 4, 1], 3, 0))
    store.set_sample_index("x", Dev(0xB000, 4, torch.int64), Dev(0xC000, 4, torch.int64))
    assert _one(store) == ("dds_set_sample_index", (H, b"x", 0xB000, 0xC000, 4, 1))
    m, s = np.array([1, 2], np.float32), np.array([3, 4], np.float32)
    store.set_normalization("x", m, s, inner=5)
    assert _one(store) == ("dds_set_normalization", (H, b"x", m.ctypes.data, s.ctypes.data, 2, 5, 0))
    store.set_normalization("x", Dev(0xB000, 3), Dev(0xC000, 3))
    assert _one(store) == ("dds_set_normalization", (H, b"x", 0xB000, 0xC000, 3, 1, 1))
    store.set_normalization("x", np.zeros(0, np.float32), np.zeros(0, np.float32))
    assert _one(store) == ("dds_set_normalization", (H, b"x", 0, 0, 0, 1, 0))
    store._L.bad = 5
    assert store.wait() == TOTAL and store.last_bad_index == 5
    assert _one(store) == ("dds_batch_wait", (H, OUT, OUT))


# ------------------------------------------------------------------------------------------------ refusals
def _refused(store, match, fn, *a, **kw):
    with pytest.raises(ValueError, match=match):
        fn(*a, **kw)
    assert store._L.calls == []


def test_writes_refuse_before_any_call(store):
    src, out, cmp = Dev(0xF000, 12), Dev(0x9000, 12), Dev(0x8000, 12)
    host = np.zeros(12, np.float32)
    bent = Dev(0xF000, 12, contiguous=False)
    i8 = Dev(0xF000, 12, torch.int8)
    for put in (store.put_batch, lambda n, i, src: store.put_samples(n, i, src)):
        _refused(store, "a put needs `src` rows", put, "x", [0], src=None)
        _refused(store, r"put into 'x': src must be device memory", put, "x", [0], src=host)
        _refused(store, "src must be C-contiguous", put, "x", [0], src=bent)
    for acc in (store.accumulate_batch, lambda n, i, src, op="sum": store.accumulate_samples(n, i, src, op=op)):
        _refused(store, "a put needs `src` rows", acc, "x", [0], src=None, op="nope")
        _refused(store, "src must be device memory", acc, "x", [0], src=host, op="nope")
        _refused(store, "src dtype int8 is not one of float32", acc, "x", [0], src=i8, op="nope")
        _refused(store, "src dtype Cai is not one of", acc, "x", [0], src=type("Cai", (), {"__cuda_array_interface__": {
            "shape": (4,), "typestr": "<f4", "data": (0xF000, False), "version": 2}})())
        _refused(store, r"accumulate into 'x': op 'max' is not one of sum, amax", acc, "x", [0], src=src, op="max")
    for fop in (store.get_accumulate_batch,
                lambda n, i, src, out, op="sum": store.get_accumulate_samples(n, i, src, out, op=op)):
        _refused(store, "src must be device memory", fop, "x", [0], src=host, out=None, op="nope")
        _refused(store, "src dtype int8", fop, "x", [0], src=i8, out=None, op="nope")
        _refused(store, r"fetch-op on 'x': op 'nope' is not one of sum, replace, amax", fop, "x", [0], src=src,
                 out=None, op="nope")
        _refused(store, "fetch-op on 'x': out must be a CUDA tensor", fop, "x", [0], src=src, out=host)
        _refused(store, "out must be C-contiguous", fop, "x", [0], src=src, out=Dev(0x9000, 12, contiguous=False))
        _refused(store, "fetch-op on 'x': out holds 44 bytes, src 48", fop, "x", [0], src=src, out=Dev(0x9000, 11))
    for cas in (store.compare_and_swap_batch,
                lambda n, i, src, compare, out: store.compare_and_swap_samples(n, i, src, compare, out)):
        _refused(store, "a put needs `src` rows", cas, "x", [0], src=None, compare=None, out=None)
        _refused(store, "src must be device memory", cas, "x", [0], src=host, compare=None, out=None)
        _refused(store, "compare-and-swap on 'x': compare must be a CUDA tensor", cas, "x", [0], src=src,
                 compare=host, out=None)
        _refused(store, "compare must be C-contiguous", cas, "x", [0], src=src, compare=bent, out=None)
        _refused(store, "compare-and-swap on 'x': out has 8-byte elements, src 4-byte ones", cas, "x", [0], src=src,
                 compare=cmp, out=Dev(0x9000, 12, torch.float64))
        _refused(store, "compare-and-swap on 'x': compare holds 44 bytes, src 48", cas, "x", [0], src=src,
                 compare=Dev(0x8000, 11), out=Dev(0x9000, 11))
        _refused(store, "compare-and-swap on 'x': out must be a CUDA tensor", cas, "x", [0], src=src, compare=cmp,
                 out=None)


def test_get_batch_refuses_before_any_call(store):
    out, lens = Dev(0xA000, 64), Dev(0xE000, 2, torch.int64)
    g = store.get_batch
    _refused(store, "needs an `out` buffer", g, "x", [0], out=None, pad_rows=2, normalize=True)
    _refused(store, "pad_rows needs counts", g, "x", [0], out=out, pad_rows=2, count=2, normalize=True)
    _refused(store, "takes neither `count` nor `offsets`", g, "x", [0], [1], out=out, pad_rows=2, count=2,
             normalize=True)
    _refused(store, "takes neither `count` nor `offsets`", g, "x", [0], [1], out=out, pad_rows=2,
             offsets=Dev(0xD000, 2, torch.int64))
    _refused(store, "normalize=True needs src_dtype", g, "x", [0], out=out, normalize=True, lut=[0])
    _refused(store, "unsupported conversion float64 -> bfloat16", g, "x", [0], out=Dev(0xA000, 4, torch.bfloat16),
             src_dtype=torch.float64, lut=[0])
    _refused(store, "unsupported normalising conversion uint8 -> int32", g, "x", [0], out=Dev(0xA000, 4, torch.int32),
             src_dtype=torch.uint8, normalize=True)
    _refused(store, "a table", g, "x", [0], out=Dev(0xA000, 4, torch.bfloat16), src_dtype=torch.float32, lut=[0])
    _refused(store, "lut must hold 256 entries of torch.bfloat16", g, "x", [0], out=Dev(0xA000, 4, torch.bfloat16),
             src_dtype=torch.uint8, lut=torch.zeros(256))
    _refused(store, "offsets must be int64", g, "x", [0, 1], out=out, offsets=np.zeros(3, np.int64))
    _refused(store, "offsets must be int64", g, "x", [0, 1], out=out, offsets=Dev(0xD000, 2, torch.int64))
    _refused(store, "offsets must be int64", g, "x", [0, 1], out=out, offsets=Dev(0xD000, 6, torch.int32))
    _refused(store, "pad_rows must be >= 0", g, "x", [0], [1], out=np.zeros(4, np.float32), pad_rows=-1)
    _refused(store, "a padded batch delivers into a CUDA tensor", g, "x", [0], [1], out=np.zeros(4, np.float32),
             pad_rows=1, pad_value=float("nan"))
    _refused(store, "does not have the variable's itemsize", g, "x", [0], [1], out=Dev(0xA000, 4, torch.float64),
             pad_rows=1, pad_value=1e300, lengths=np.zeros(1, np.int64))
    _refused(store, "pad_value 1e\\+300 overflows", g, "x", [0], [1], out=out, pad_rows=1, pad_value=1e300,
             lengths=np.zeros(1, np.int64))
    _refused(store, "lengths must be an int64 CUDA tensor", g, "x", [0], [1], out=out, pad_rows=1,
             lengths=np.zeros(1, np.int64))
    _refused(store, "lengths must be an int64 CUDA tensor", g, "x", [0, 1, 2], [1, 1, 1], out=out, pad_rows=1,
             lengths=lens)
    with pytest.raises(TypeError, match="unsupported array type list"):
        g("x", [0], out=[0.0])
    assert store._L.calls == []
