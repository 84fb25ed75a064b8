"""ddstore_b200/store.py -- `PyDDStore`: the reference's Python surface over the C-ABI.

Mirrors /root/reference/src/pyddstore.pyx:58-131 method for method (same names, argument order and
meaning, same exception types/texts): add / get / epoch_begin / epoch_end / free / init / update, plus
`get_batch`, the batched form of get() that is this package's hot path. Arrays may be NumPy arrays
(host) or CUDA tensors / __cuda_array_interface__ objects (device; fetched bytes then never leave HBM).
"""
import ctypes as C
import math

import numpy as np

from . import _capi
from .comm import as_dds_comm

# dtypes the reference's if-chains accept (src/pyddstore.pyx:69-80, 88-99, 118-129)
_NP_OK = {np.dtype(np.int32), np.dtype(np.int64), np.dtype(np.uint8), np.dtype(np.float32),
          np.dtype(np.float64), np.dtype(np.bool_)}
_TORCH_OK = {"torch.int32", "torch.int64", "torch.uint8", "torch.float32", "torch.float64", "torch.bool"}
# output dtypes only a converting batch delivers (the store keeps no 2-byte floats)
_TORCH_HALF = {"torch.bfloat16", "torch.float16"}

# converting batches: (source dtype, output dtype) -> DDS_CVT_* code
_CVT_CODES = {("float32", "bfloat16"): _capi.CVT_F32_BF16, ("float32", "float16"): _capi.CVT_F32_F16,
              ("float64", "float32"): _capi.CVT_F64_F32, ("uint8", "bfloat16"): _capi.CVT_U8_LUT16,
              ("uint8", "float16"): _capi.CVT_U8_LUT16, ("uint8", "float32"): _capi.CVT_U8_LUT32}
# normalising batches ((x - mean[ch]) / std[ch] in float32, then the output dtype): (source, output) -> DDS_CVT_NORM_*
_NORM_CODES = {("float32", "float32"): _capi.CVT_NORM_F32_F32, ("float32", "bfloat16"): _capi.CVT_NORM_F32_BF16,
               ("float32", "float16"): _capi.CVT_NORM_F32_F16, ("float64", "float32"): _capi.CVT_NORM_F64_F32,
               ("uint8", "float32"): _capi.CVT_NORM_U8_F32, ("uint8", "bfloat16"): _capi.CVT_NORM_U8_BF16,
               ("uint8", "float16"): _capi.CVT_NORM_U8_F16}
_U8_NORM = (_capi.CVT_NORM_U8_F32, _capi.CVT_NORM_U8_BF16, _capi.CVT_NORM_U8_F16)
_default_luts = {}  # output dtype name -> host table of the plain value cast, torch.arange(256).to(dtype)


def _dtype_name(dt):
    """'float32', 'bfloat16', ... of a torch dtype, a NumPy dtype or a name"""
    s = str(dt)
    if s.startswith("torch."):
        return s[len("torch."):]
    if s in ("bfloat16", "float16"):
        return s
    return str(np.dtype(dt))


def _conversion(src_dtype, out_dtype, lut, normalize=False):
    """-> (dds_convert_t, keepalive) of a converting batch from `src_dtype` rows into an `out_dtype` buffer. A uint8 source
    takes `lut` (256 entries of the output dtype; default: the plain value cast torch.arange(256).to(out_dtype)).
    normalize=True: the normalising conversion ((x - mean) / std per channel, see set_normalization); a uint8 source then
    decodes through 256 float32 entries (default torch.arange(256).float())."""
    import torch
    key = (_dtype_name(src_dtype), _dtype_name(out_dtype))
    code = (_NORM_CODES if normalize else _CVT_CODES).get(key)
    if code is None:
        raise ValueError(f"unsupported {'normalising ' if normalize else ''}conversion {key[0]} -> {key[1]}")
    if code not in (_capi.CVT_U8_LUT16, _capi.CVT_U8_LUT32) + _U8_NORM:
        if lut is not None:
            raise ValueError("a table (lut) applies to uint8 sources only")
        return _capi.Convert(code, None), None
    tdt = torch.float32 if normalize else getattr(torch, key[1])
    key = (key[0], "float32") if normalize else key
    if lut is None:
        host = _default_luts.get(key[1])
        if host is None:
            host = _default_luts[key[1]] = _lut_bits(torch.arange(256).to(tdt))
    else:
        t = torch.as_tensor(lut)
        if t.dtype != tdt or t.numel() != 256:
            raise ValueError(f"lut must hold 256 entries of {tdt}")
        host = _lut_bits(t)
    return _capi.Convert(code, host.ctypes.data), host


def _norm_tables(mean, std):
    """(mean, std) of set_normalization -> (mean, std, nchan, on_device), both 1-D float32 of one length and residency"""
    def info(t, what):
        if isinstance(t, np.ndarray):
            if t.dtype != np.float32 or t.ndim != 1:
                raise ValueError(f"{what} must be a 1-D float32 array")
            return np.ascontiguousarray(t), t.size, 0
        if hasattr(t, "data_ptr") and hasattr(t, "element_size"):
            if str(t.dtype) != "torch.float32" or t.dim() != 1:
                raise ValueError(f"{what} must be a 1-D float32 tensor")
            return t.contiguous(), t.numel(), 1 if t.is_cuda else 0
        raise TypeError(f"{what}: unsupported array type {type(t).__name__}")
    m, nm, dm = info(mean, "mean")
    s, ns, ds = info(std, "std")
    if nm != ns:
        raise ValueError(f"mean and std differ in length ({nm} != {ns})")
    if dm != ds:
        raise ValueError("mean and std must both be on the host or both on the device")
    return m, s, nm, dm


_PLACEMENT_NAMES = {v: k for k, v in _capi.PLACEMENTS.items()}


def _placement(placement):
    if placement not in _capi.PLACEMENTS:
        raise ValueError(f"unknown placement {placement!r} (expected 'hbm' or 'host')")
    return _capi.PLACEMENTS[placement]


def _ptr(t):
    return t.ctypes.data if isinstance(t, np.ndarray) else t.data_ptr()


_INT_VIEW = {1: "uint8", 2: "int16", 4: "int32", 8: "int64"}


def _pad_bits(value, dtype):
    """the bits of one `dtype` element holding `value` (a number, or a one-element tensor of `dtype` whose bits are used
    verbatim, e.g. a NaN with a payload). ValueError for a value `dtype` cannot represent."""
    import math

    import torch
    if isinstance(value, torch.Tensor):
        if value.numel() != 1 or value.dtype != dtype:
            raise ValueError(f"pad_value must be a number or a one-element {dtype} tensor")
        t = value.detach().reshape(1).cpu()
    elif dtype == torch.bool:
        if value not in (0, 1):
            raise ValueError(f"pad_value {value!r} is not a bool")
        t = torch.tensor([bool(value)])
    elif dtype.is_floating_point:
        v = float(value)
        t = torch.tensor([v], dtype=dtype)
        if math.isfinite(v) and not bool(torch.isfinite(t).all()):
            raise ValueError(f"pad_value {value!r} overflows {dtype}")
    else:
        if isinstance(value, float) and not value.is_integer():
            raise ValueError(f"pad_value {value!r} is not an integer ({dtype})")
        iv, info = int(value), torch.iinfo(dtype)
        if not info.min <= iv <= info.max:
            raise ValueError(f"pad_value {value!r} is outside the range of {dtype}")
        t = torch.tensor([iv], dtype=dtype)
    n = t.element_size()
    return int(t.view(getattr(torch, _INT_VIEW[n])).item()) & ((1 << (8 * n)) - 1)


def _lut_bits(t):
    """a 256-entry torch table as a host int16 / int32 array of its bits"""
    import torch
    t = t.detach().reshape(-1).cpu().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).numpy().copy()


class _Buf:
    """pointer / shape / itemsize / residency of an ndarray, a CUDA tensor or a CAI object"""

    def __init__(self, arr, writable=False, half_ok=False):  # `writable` documents intent at the call sites; nothing is
        self.keep = arr                                          # copied. half_ok: bf16/f16 tensors (converting batches)
        if isinstance(arr, np.ndarray):
            assert arr.flags.c_contiguous  # src/pyddstore.pyx:66,85,116
            if arr.dtype not in _NP_OK:
                raise NotImplementedError
            self.ptr, self.on_device = arr.ctypes.data, 0
            self.shape, self.itemsize, self.size = arr.shape, arr.dtype.itemsize, arr.size
        elif hasattr(arr, "data_ptr") and hasattr(arr, "element_size"):  # torch.Tensor
            assert arr.is_contiguous()
            if str(arr.dtype) not in _TORCH_OK and not (half_ok and str(arr.dtype) in _TORCH_HALF):
                raise NotImplementedError
            self.ptr, self.on_device = arr.data_ptr(), 1 if arr.is_cuda else 0
            self.shape, self.itemsize, self.size = tuple(arr.shape), arr.element_size(), arr.numel()
        elif hasattr(arr, "__cuda_array_interface__"):
            cai = arr.__cuda_array_interface__
            if cai.get("strides") is not None:
                raise ValueError("device array must be C-contiguous")
            dt = np.dtype(cai["typestr"])
            if dt not in _NP_OK:
                raise NotImplementedError
            self.ptr, self.on_device = cai["data"][0], 1
            self.shape, self.itemsize = tuple(cai["shape"]), dt.itemsize
            self.size = int(np.prod(self.shape, dtype=np.int64))
        else:
            raise TypeError(f"unsupported array type {type(arr).__name__}")
        self.nbytes = self.size * self.itemsize


class _DevMem:
    """a raw device range as a __cuda_array_interface__ object (uint8)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


def _i64(x):
    """host int64 contiguous ndarray view of an index list/array"""
    return np.ascontiguousarray(x, dtype=np.int64)


def _requests(starts, counts=None):
    """-> (nreq, starts_ptr, counts_ptr, on_device, keep) of a batch's index arrays: CUDA tensors are passed as they
    are, anything else as host int64 arrays (counts None: a null counts pointer). `keep` holds what the pointers
    point into; the caller keeps it until the call has returned."""
    if hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False):
        return starts.numel(), starts.data_ptr(), counts.data_ptr() if counts is not None else None, True, \
            (starts, counts)
    sa = _i64(starts)
    ca = _i64(counts) if counts is not None else None
    return sa.size, sa.ctypes.data, ca.ctypes.data if ca is not None else None, False, (sa, ca)


def _stream_handle(stream):
    """the raw cudaStream_t of a `stream` argument: None -> 0, the store's own stream; otherwise the handle (e.g.
    torch.cuda.current_stream().cuda_stream). Handle 0 is CUDA's legacy default stream, which the C-ABI spells
    cudaStreamLegacy (0x1) because NULL there means "the store's stream"."""
    if stream is None:
        return 0
    h = int(stream)
    return h if h != 0 else 1


# ---------------------------------------------------------------- argument checks of the batched gets
def _get_args(by_sample, counts, count, out, offsets, src_dtype, lut, normalize, pad_rows):
    """the argument rules of get_batch / get_samples (by_sample) that precede the `out` buffer's -> (dds_convert_t,
    keepalive) of a converting batch, (None, None) of a raw one"""
    if by_sample:
        if pad_rows is not None and offsets is not None:
            raise ValueError("a padded batch takes no `offsets`")
    else:
        if out is None:
            raise ValueError("get_batch needs an `out` buffer (like get(), it never allocates)")
        if pad_rows is not None:
            if counts is None:
                raise ValueError("pad_rows needs counts (there is no fixed-count padded batch)")
            if count is not None or offsets is not None:
                raise ValueError("a padded batch takes neither `count` nor `offsets`")
    if normalize and src_dtype is None:
        raise ValueError("normalize=True needs src_dtype")
    if src_dtype is None:
        return None, None
    return _conversion(src_dtype, getattr(out, "dtype", None), lut, normalize)


def _offsets(offsets, ob, nreq, by_sample):
    """the address of a batch's `offsets` (None: no offsets); ValueError unless it is int64[nreq + 1] on out's side"""
    if offsets is None:
        return None
    fb = _Buf(offsets, writable=True)
    if fb.on_device != ob.on_device or fb.itemsize != 8 or fb.size < nreq + 1:
        raise ValueError(f"offsets must be int64[len({'sample_ids' if by_sample else 'starts'})+1] with the same "
                         f"residency as out")
    return fb.ptr


def _pad_rows(pad_rows, out, ob):
    """pad_rows of a padded batch into `out` (ob: its _Buf) as an int; ValueError unless it is >= 0 and out is a CUDA
    tensor"""
    pad_rows = int(pad_rows)
    if pad_rows < 0:
        raise ValueError("pad_rows must be >= 0")
    if not (ob.on_device and hasattr(out, "dtype") and str(out.dtype).startswith("torch.")):
        raise ValueError("a padded batch delivers into a CUDA tensor")
    return pad_rows


def _pad(pad_rows, pad_value, lengths, out, nreq):
    """the dds_pad_t of a padded batch of nreq requests into `out`"""
    pad = _capi.Pad(pad_rows, _pad_bits(pad_value, out.dtype), None)
    if lengths is not None:
        lb = _Buf(lengths, writable=True)
        if not lb.on_device or lb.itemsize != 8 or lb.size < nreq:
            raise ValueError("lengths must be an int64 CUDA tensor of len(starts)")
        pad.lengths = lb.ptr
    return pad


# ---------------------------------------------------------------- argument checks of the batched writes and pools
def _put_src(name, src):
    """the _Buf of a put's source rows (a CUDA tensor or CAI object; ValueError for host memory)"""
    if src is None:
        raise ValueError("a put needs `src` rows")
    if hasattr(src, "data_ptr") and hasattr(src, "element_size"):  # any torch dtype: only its element size matters
        if not src.is_contiguous():
            raise ValueError("src must be C-contiguous")
        sb = _Buf.__new__(_Buf)
        sb.ptr, sb.on_device, sb.itemsize = src.data_ptr(), 1 if src.is_cuda else 0, src.element_size()
        sb.nbytes = src.numel() * sb.itemsize
    else:
        sb = _Buf(src)
    if not sb.on_device:
        raise ValueError(f"put into {name!r}: src must be device memory (copy host rows to the device first)")
    return sb


def _acc_type(name, src):
    """the DDS_ACC_* element type of an accumulate's src, from its dtype (ValueError for any other)"""
    dt = str(getattr(src, "dtype", "")).replace("torch.", "")
    if dt not in _capi.ACC_TYPES:
        raise ValueError(f"accumulate into {name!r}: src dtype {dt or type(src).__name__} is not one of "
                         f"{', '.join(_capi.ACC_TYPES)}")
    return _capi.ACC_TYPES[dt]


def _red_op(name, op):
    """the DDS_OP_* code of an accumulate's reduction (ValueError for an unknown one)"""
    ops = {"sum": _capi.OP_SUM, **_capi.RED_OPS}
    if op not in ops:
        raise ValueError(f"accumulate into {name!r}: op {op!r} is not one of {', '.join(ops)}")
    return ops[op]


def _fop_args(name, op, out, sb):
    """the DDS_OP_* code of a fetch-op and the address of its `out` tensor (ValueError for an unknown op, or an out
    that is not a contiguous CUDA tensor of at least src's bytes)"""
    ops = {**_capi.FOP_OPS, **_capi.RED_OPS}
    if op not in ops:
        raise ValueError(f"fetch-op on {name!r}: op {op!r} is not one of {', '.join(ops)}")
    if not (hasattr(out, "data_ptr") and getattr(out, "is_cuda", False)):
        raise ValueError(f"fetch-op on {name!r}: out must be a CUDA tensor")
    if not out.is_contiguous():
        raise ValueError("out must be C-contiguous")
    if out.numel() * out.element_size() < sb.nbytes:
        raise ValueError(f"fetch-op on {name!r}: out holds {out.numel() * out.element_size()} bytes, src "
                         f"{sb.nbytes}")
    return ops[op], out.data_ptr()


def _cas_args(name, compare, out, sb):
    """the addresses of a compare-and-swap's `compare` and `out` tensors (ValueError unless each is a C-contiguous
    CUDA tensor of src's element size and at least src's bytes)"""
    ptrs = []
    for what, t in (("compare", compare), ("out", out)):
        if not (hasattr(t, "data_ptr") and getattr(t, "is_cuda", False)):
            raise ValueError(f"compare-and-swap on {name!r}: {what} must be a CUDA tensor")
        if not t.is_contiguous():
            raise ValueError(f"{what} must be C-contiguous")
        if t.element_size() != sb.itemsize:
            raise ValueError(f"compare-and-swap on {name!r}: {what} has {t.element_size()}-byte elements, src "
                             f"{sb.itemsize}-byte ones")
        if t.numel() * t.element_size() < sb.nbytes:
            raise ValueError(f"compare-and-swap on {name!r}: {what} holds {t.numel() * t.element_size()} bytes, "
                             f"src {sb.nbytes}")
        ptrs.append(t.data_ptr())
    return ptrs[0], ptrs[1]


def _pool_args(name, mode, t, what="out"):
    """the DDS_POOL_* mode and the DDS_ACC_* element type of a pooled batch's tensor t, its `out` or its `grad` (ValueError
    for an unknown mode, or a t that is not a C-contiguous CUDA float32, float64, float16 or bfloat16 tensor)"""
    import torch
    if mode not in _capi.POOL_MODES:
        raise ValueError(f"pooled batch of {name!r}: mode {mode!r} is not one of {', '.join(_capi.POOL_MODES)}")
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.is_contiguous()):
        raise ValueError(f"{what} must be a C-contiguous CUDA tensor")
    dt = _dtype_name(t.dtype)
    if dt not in ("float32", "float64", "float16", "bfloat16"):
        raise ValueError(f"pooled batch of {name!r}: {what} dtype {dt} is not float32, float64, float16 or bfloat16")
    return _capi.POOL_MODES[mode], _capi.ACC_TYPES[dt]


def _pool_acc_args(name, mode, alpha, grad):
    """_pool_args of a pooled accumulate's `grad`, refusing first mode "max" (its adjoint needs the forward's argmax)
    and a non-finite alpha (one NaN step would poison the whole table)"""
    if mode == "max":
        raise ValueError(f"pooled accumulate into {name!r}: mode 'max' has no adjoint here (use 'sum' or 'mean')")
    if alpha is None or not math.isfinite(alpha):
        raise ValueError(f"pooled accumulate into {name!r}: alpha must be finite, not {alpha!r}")
    return _pool_args(name, mode, grad, "grad")


def _pool_requests(starts, counts, bags, weights, out, wait):
    """-> (sa, ca, ba, wa, on_device) of a pooled batch: int64 starts, counts and bags and weights of out.dtype as
    contiguous tensors (None where not given) on the side starts lives. Unlike _requests this converts dtypes, so a
    queued batch (wait=False) must not be handed a converted copy the queued launch could outlive."""
    import torch
    if isinstance(starts, torch.Tensor) and starts.is_cuda:
        sa = starts.to(torch.int64).contiguous()
        ca = counts.to(torch.int64).contiguous() if counts is not None else None
        ba = torch.as_tensor(bags, dtype=torch.int64, device=out.device).contiguous() if bags is not None else None
        wa = torch.as_tensor(weights, dtype=out.dtype, device=out.device).contiguous() if weights is not None else None
        if not wait and any(t is not None and t is not u for t, u in ((sa, starts), (ca, counts), (ba, bags),
                                                                      (wa, weights))):
            raise ValueError("wait=False takes contiguous CUDA tensors: int64 starts, counts and bags, weights of "
                             "out.dtype (a converted copy could be freed before the queued launch reads it)")
        return sa, ca, ba, wa, True
    sa = torch.as_tensor(_i64(starts))
    ca = torch.as_tensor(_i64(counts)) if counts is not None else None
    ba = torch.as_tensor(_i64(bags)) if bags is not None else None
    wa = torch.as_tensor(weights, dtype=out.dtype, device="cpu").contiguous() if weights is not None else None
    return sa, ca, ba, wa, False


class PyDDStore:
    # the argument checks of the batched writes, also reachable from the class (the Cython binding calls the
    # module-level functions)
    _put_src = staticmethod(_put_src)
    _acc_type = staticmethod(_acc_type)
    _red_op = staticmethod(_red_op)
    _fop_args = staticmethod(_fop_args)
    _cas_args = staticmethod(_cas_args)

    def __init__(self, comm=None, method=0, device=None):
        # src/pyddstore.pyx:61-63. `comm`: see ddstore_b200.comm.as_dds_comm; `device`: CUDA ordinal
        # for this rank's shards (default: the current device).
        self._L = _capi.lib()
        self._comm = as_dds_comm(comm)
        self._h = self._L.dds_create(self._comm.handle, -1 if device is None else int(device), int(method))
        if not self._h:
            raise RuntimeError(_capi.last_error())
        self.rank, self.size = self._L.dds_rank(self._h), self._L.dds_size(self._h)
        self._itemsize = {}  # per-variable itemsize, cached for the hot path
        self._cname = {}     # name -> bytes, cached for the per-sample get() loop
        self._rowbytes = {}
        self.last_bad_index = -1

    # ---------------------------------------------------------------- reference surface
    def add(self, name, arr, placement="hbm"):
        # src/pyddstore.pyx:65-82. placement="host": the shards live in pinned host memory every rank of the box maps
        # (a dataset larger than free HBM); the gathers still run on the GPU. Batched writes refuse such variables.
        pl = _placement(placement)
        b = _Buf(arr)
        nrows = b.shape[0]
        disp = b.size // b.shape[0] if b.shape[0] else int(np.prod(b.shape[1:], dtype=np.int64))
        _capi.raise_for(self._L.dds_add_placed(self._h, name.encode(), b.ptr, nrows, disp, b.itemsize, b.on_device, pl))

    def get(self, name, arr, start=0):
        # src/pyddstore.pyx:84-101: count = arr.shape[0]; fills arr in place
        cn = self._cname.get(name)
        if cn is None:
            cn = self._cname[name] = name.encode()
        if type(arr) is np.ndarray:  # the legacy per-sample loop: keep the Python side of the call short
            assert arr.flags.c_contiguous
            if arr.dtype not in _NP_OK:
                raise NotImplementedError
            rc = self._L.dds_get(self._h, cn, int(start), arr.shape[0], arr.dtype.itemsize, arr.ctypes.data, 0)
        else:
            b = _Buf(arr, writable=True)
            rc = self._L.dds_get(self._h, cn, int(start), b.shape[0], b.itemsize, b.ptr, b.on_device)
        if rc:
            _capi.raise_for(rc)

    def epoch_begin(self):
        _capi.raise_for(self._L.dds_epoch_begin(self._h))  # src/pyddstore.pyx:103-104

    def epoch_end(self):
        _capi.raise_for(self._L.dds_epoch_end(self._h))  # src/pyddstore.pyx:106-107

    def free(self):
        if self._h:
            self._itemsize.clear()
            _capi.raise_for(self._L.dds_free(self._h))  # src/pyddstore.pyx:109-110

    def init(self, name, nrows, disp, itemsize=1, placement="hbm"):
        pl = _placement(placement)
        _capi.raise_for(self._L.dds_init_placed(self._h, name.encode(), int(nrows), int(disp), int(itemsize), pl))  # :112-113

    def update(self, name, arr, offset, stream=None, wait=True):
        # src/pyddstore.pyx:115-131. wait=False: enqueue the copy on `stream` and return (streaming ingest; the
        # source must stay valid -- pinned -- until the stream reaches it).
        b = _Buf(arr)
        if wait:
            rc = self._L.dds_update(self._h, name.encode(), b.ptr, b.shape[0], int(offset), b.itemsize, b.on_device)
        else:
            rc = self._L.dds_update_async(self._h, name.encode(), b.ptr, b.shape[0], int(offset), b.itemsize,
                                          b.on_device, _stream_handle(stream))
        _capi.raise_for(rc)

    def ingest(self, name, arr, offset):
        """update() for a chunk of pageable host rows, pipelined inside the library (parallel staging copy + async H2D).
        Returns when `arr` has been consumed; call ingest_wait() (or an epoch fence) before reading the rows back."""
        b = _Buf(arr)
        if b.on_device:
            raise ValueError("ingest takes host arrays (use update for device arrays)")
        _capi.raise_for(self._L.dds_ingest(self._h, name.encode(), b.ptr, b.shape[0], int(offset), b.itemsize))

    def ingest_wait(self):
        _capi.raise_for(self._L.dds_ingest_wait(self._h))

    # ---------------------------------------------------------------- the batched hot path
    def get_batch(self, name, starts, counts=None, out=None, count=None, offsets=None, stream=None, wait=True,
                  overlap=False, src_dtype=None, lut=None, normalize=False, pad_rows=None, pad_value=0, lengths=None):
        """Fetch len(starts) requests in ONE kernel launch, packed back to back in request order.

        starts/counts: int64 index arrays (host ndarray/list, or CUDA int64 tensors). counts=None means
        every request fetches `count` rows (default 1): the fixed-stride fast path.
        out: destination (host ndarray or CUDA tensor) of at least the packed size; row layout is the
        caller's business exactly as with get() (src/pyddstore.pyx:84-87 never checks it either).
        offsets: optional int64 array of len(starts)+1 receiving the byte offset of every request
        (same residency as `out`). Returns the number of packed bytes.
        wait=False (device indices + device out only): enqueue on `stream` and return at once; call
        `wait()` later for the status. Several such batches may be queued on one stream.
        overlap=True (with wait=False): this batch is independent of the one queued just before it (different `out`
        and `offsets`, indices not written by it) and may overlap with its tail -- double-buffered prefetch.
        stream: the cudaStream_t handle everything of this call is enqueued on (index copy, kernels, result copy).
        stream=None means the STORE'S OWN stream, which is not ordered with anything the caller has queued elsewhere:
        device tensors passed in (indices, out, offsets) must then be complete / free to overwrite before the call --
        e.g. produced by a synchronous copy. When they were produced or are consumed on torch's current stream, pass
        stream=torch.cuda.current_stream().cuda_stream.
        Raises the reference's ValueError for the first invalid request (requests before it are delivered).
        src_dtype (with a CUDA `out`): deliver the rows converted from `src_dtype` (the variable's element type) to
        out.dtype inside the gather: float32 -> bfloat16 / float16, float64 -> float32, uint8 -> bfloat16 / float16 /
        float32 through `lut` (256 entries of out.dtype; default torch.arange(256).to(out.dtype)). The capacity, the
        offsets and the returned size are then in bytes of `out`.
        normalize=True (with src_dtype): deliver (x - mean[ch]) / std[ch], computed in float32 with the tables registered
        by set_normalization, as out.dtype: float32 -> float32 / bfloat16 / float16, float64 -> float32, uint8 -> float32 /
        bfloat16 / float16 (decoded through `lut`, 256 float32 entries, default torch.arange(256).float()).
        pad_rows=M (with counts and a CUDA `out`): a padded batch. Request i fills slot i of `out`, viewed as
        [len(starts), M, row]: its first min(counts[i], M) rows (raw, or converted / normalised as above), then
        `pad_value` encoded in out.dtype (or a one-element out.dtype tensor, used bit for bit) up to the slot's end.
        out.dtype must have the delivered element size. An invalid request leaves a slot of padding and length 0, and
        every valid slot is still delivered; then the reference's ValueError is raised for the first invalid one.
        lengths (optional int64 CUDA tensor of len(starts)) receives the delivered row counts. Returns out's padded
        size in bytes, len(starts) * M * row elements * out.element_size().
        """
        return self._get(name, False, starts, counts, count, out, offsets, stream, wait, overlap, src_dtype, lut,
                         normalize, pad_rows, pad_value, lengths)

    # ---------------------------------------------------------------- batched puts (update<T> from any rank)
    def put_batch(self, name, starts, counts=None, src=None, count=None, stream=None, wait=True):
        """Write len(starts) requests into the owners' shards in ONE kernel launch -- update() from any rank, the dual
        of get_batch (MPI_Put between fences). Request i writes global rows [starts[i], starts[i] + counts[i]) (or
        `count` rows, default 1, when counts is None) from `src`, a C-contiguous CUDA tensor of any shape whose element
        size is the variable's itemsize. src holds the requests' rows back to back in request order; an invalid
        request keeps its counts[i] rows' worth of bytes in that layout (0 when counts[i] <= 0 or above the variable's
        rows), so the requests after it are read where the caller put them. Returns the layout's size in bytes.
        Raises the reference's ValueError for the first invalid request (last_bad_index: its index); every VALID
        request is still written, an invalid one writes nothing. A layout larger than src writes nothing at all.
        A host `src` raises ValueError (copy it to the device first). wait=False (device indices only): enqueue on
        `stream` and return; wait() reports the outcome. Other ranks see the rows after the next epoch fence both
        sides have passed (epoch_begin / epoch_end complete queued puts); later work on the same stream sees them at
        once. Two writes to the same bytes in one epoch leave one writer's byte; reading rows being put in the same
        epoch is undefined."""
        return self._write("put", name, False, starts, counts, count, src, stream, wait)

    def put_samples(self, name, sample_ids, src, stream=None, wait=True):
        """put_batch by SAMPLE ID: request i writes the rows of sample sample_ids[i] in the index registered with
        set_sample_index. Same layout, error behaviour (every valid request is still written), ordering and
        visibility as put_batch; a sample id outside the index keeps 0 bytes of the layout."""
        return self._write("put", name, True, sample_ids, None, None, src, stream, wait)

    # ---------------------------------------------------------------- batched accumulates (MPI_Accumulate)
    def accumulate_batch(self, name, starts, counts=None, src=None, count=None, stream=None, wait=True, op="sum"):
        """ADD len(starts) requests into the owners' shards in ONE kernel launch: every element e of request i's rows
        becomes shard[e] + src[e]. Requests, the layout of `src`, errors (every valid request is still applied, an
        invalid one changes nothing), wait=False, ordering and visibility are put_batch's. The sum is taken in
        src.dtype -- float32, float64, int32, int64, float16 or bfloat16, whose size must be the variable's itemsize
        (another dtype raises ValueError before the call). Accumulates into the same element in one epoch combine
        atomically, from any batch, rank or duplicate request: integers exactly (wrapping), floats with one rounding per
        addition in an unspecified order (float32 may flush subnormals to zero). Mixing puts and accumulates on the same
        rows in one epoch, or reading rows being accumulated, is undefined. Returns the layout's size in bytes.
        op="amax" / "amin" makes each element max(shard[e], src[e]) / min(...) instead -- signed for the integer types,
        IEEE maximumNumber / minimumNumber for floats (a NaN operand is ignored, -0 < +0, nothing flushes) -- and
        "bitwise_and" / "bitwise_or" / "bitwise_xor" (int32 and int64 src only) its bitwise combination with src[e].
        Reductions with the same op and dtype on one element in one epoch combine atomically, also with
        get_accumulate_batch's; mixing different ops on one element in one epoch is undefined."""
        return self._write("accumulate_op", name, False, starts, counts, count, src, stream, wait, op=op)

    def accumulate_samples(self, name, sample_ids, src, stream=None, wait=True, op="sum"):
        """accumulate_batch by SAMPLE ID: request i adds into (or reduces by op into) the rows of sample sample_ids[i]
        in the index registered with set_sample_index. Layout and errors as put_samples, ops as accumulate_batch."""
        return self._write("accumulate_op", name, True, sample_ids, None, None, src, stream, wait, op=op)

    # ---------------------------------------------------------------- batched fetch-ops (MPI_Get_accumulate)
    def get_accumulate_batch(self, name, starts, counts=None, src=None, out=None, op="sum", count=None, stream=None,
                             wait=True):
        """ADD (op="sum") or SWAP (op="replace") len(starts) requests into the owners' shards in ONE kernel launch and
        get the previous rows back: for every element e of request i's rows, in one atomic step, out[e] = shard[e]
        and shard[e] becomes shard[e] + src[e] (sum) or src[e] (replace). Requests, the layout of `src`, dtypes,
        errors (every valid request is still applied, an invalid one changes nothing), wait=False, ordering and
        visibility are accumulate_batch's. `out` is a C-contiguous CUDA tensor of at least src's bytes -- it may be src
        itself -- that receives the previous rows in src's layout; the bytes of invalid requests and every byte beyond
        the layout are left as they were. Fetch-ops on one element in one epoch are linearisable, from any batch, rank
        or duplicate request: each gets the value right before its own contribution (duplicate +1 requests of one batch
        get distinct tickets). Sums also combine atomically with accumulate_batch; mixing "replace" with sums, puts or
        accumulates on one element in one epoch is undefined. op may also be one of accumulate_batch's reductions
        ("amax", "amin", "bitwise_and", "bitwise_or", "bitwise_xor"), which combine atomically with accumulate_batch's
        of the same op. Returns the layout's size in bytes."""
        return self._write("get_accumulate", name, False, starts, counts, count, src, stream, wait, op=op, out=out)

    def get_accumulate_samples(self, name, sample_ids, src, out, op="sum", stream=None, wait=True):
        """get_accumulate_batch by SAMPLE ID: request i adds into (or swaps) the rows of sample sample_ids[i] in the
        index registered with set_sample_index. Layout and errors as put_samples, ops as get_accumulate_batch."""
        return self._write("get_accumulate", name, True, sample_ids, None, None, src, stream, wait, op=op, out=out)

    # ---------------------------------------------------------------- batched compare-and-swaps (MPI_Compare_and_swap)
    def compare_and_swap_batch(self, name, starts, counts=None, src=None, compare=None, out=None, count=None,
                               stream=None, wait=True):
        """COMPARE-AND-SWAP len(starts) requests against the owners' shards in ONE kernel launch: for every element e of
        request i's rows, in one atomic step, out[e] = shard[e], and shard[e] becomes src[e] if it equalled compare[e]
        BIT FOR BIT (on float data -0 != +0 and a NaN equals only its own bits). out always receives the previous
        value, so element e was swapped exactly when out[e] == compare[e] bitwise. Requests, the layout of `src`, errors
        (every valid request is still applied, an invalid one changes nothing and writes no out bytes), wait=False,
        ordering and visibility are get_accumulate_batch's. src, compare and out may be of any dtype whose element size
        is the variable's itemsize (1, 2, 4 or 8), the same for all three; compare and out are C-contiguous CUDA tensors
        of at least src's bytes in src's layout, and out may be src or compare. Compare-and-swaps on one element in one
        epoch are linearisable, from any batch, rank or duplicate request: of N that expect the same value exactly one
        wins. Mixing them with puts, accumulates or fetch-ops on one element in one epoch is undefined. Returns the
        layout's size in bytes."""
        return self._write("compare_and_swap", name, False, starts, counts, count, src, stream, wait,
                           compare=compare, out=out)

    def compare_and_swap_samples(self, name, sample_ids, src, compare, out, stream=None, wait=True):
        """compare_and_swap_batch by SAMPLE ID: request i compares and swaps the rows of sample sample_ids[i] in the
        index registered with set_sample_index. Layout and errors as put_samples, semantics as
        compare_and_swap_batch."""
        return self._write("compare_and_swap", name, True, sample_ids, None, None, src, stream, wait,
                           compare=compare, out=out)

    def _write(self, entry, name, by_sample, starts, counts, count, src, stream, wait, op="sum", compare=None,
               out=None):
        """the batched writes: `entry` ("put", "accumulate_op", "get_accumulate" or "compare_and_swap") names the
        C entries dds_<entry>_batch / dds_<entry>_samples; every argument is checked before the requests are staged"""
        sb = _put_src(name, src)
        if entry == "put":
            operands = (sb.itemsize, sb.ptr)
        elif entry == "compare_and_swap":
            operands = (sb.itemsize, sb.ptr, *_cas_args(name, compare, out, sb))
        else:
            code = _acc_type(name, src)
            if entry == "accumulate_op":
                operands = (_red_op(name, op), code, sb.ptr)
            else:
                opc, res = _fop_args(name, op, out, sb)
                operands = (opc, code, sb.ptr, res)
        nreq, sp, cp, s_dev, keep = _requests(starts, counts)
        flags = _capi.SRC_ON_DEVICE | (_capi.IDX_ON_DEVICE if s_dev else 0) | (0 if wait else _capi.NO_SYNC)
        if by_sample:
            return self._call(getattr(self._L, f"dds_{entry}_samples"), self._h, name.encode(), sp, nreq, *operands,
                              sb.nbytes, flags, _stream_handle(stream))
        return self._call(getattr(self._L, f"dds_{entry}_batch"), self._h, name.encode(), sp, cp,
                          1 if count is None else int(count), nreq, *operands, sb.nbytes, flags, _stream_handle(stream))

    # ---------------------------------------------------------------- pooled batches (embedding_bag)
    def get_batch_pooled(self, name, starts, counts=None, count=None, out=None, bags=None, mode="sum", weights=None,
                         stream=None, wait=True):
        """Fold bags of requests into one row each, in ONE kernel launch: torch's embedding_bag over a sharded variable.
        Bag k is requests [bags[k], bags[k+1]) (torch's include_last_offset offsets, nbags + 1 of them; None: one bag
        per request) and goes to out row k -- out (a CUDA float32, float64, float16 or bfloat16 tensor of the variable's
        itemsize) holds nbags rows of disp elements. mode "sum", "mean" or "max"; weights (mode "sum" only): one per
        request, torch's per_sample_weights. Requests are located and validated as in get_batch: an invalid one
        contributes nothing, every valid one is applied, the first invalid one raises with last_bad_index its index; a
        malformed bag raises ValueError("malformed bag offsets") with last_bad_index the bag, before any request error.
        Each element is the sequential fold of its bag's rows in float32 (float64 for float64 rows) -- a weighted sum
        with one fma per row, a mean divided once at the end -- rounded once to out.dtype; max keeps the first row and
        replaces it by any later row that compares greater. bags and weights live where starts lives (a CUDA tensor:
        device; else they are staged from the host). Returns the bytes written (None with wait=False)."""
        return self._pooled(name, False, starts, counts, count, out, bags, mode, weights, stream, wait)

    def get_samples_pooled(self, name, sample_ids, out, bags=None, mode="sum", weights=None, stream=None, wait=True):
        """get_batch_pooled by SAMPLE ID: request i = the rows of sample sample_ids[i] in the index registered with
        set_sample_index (e.g. a variable-length sample mean-pooled to one vector)."""
        return self._pooled(name, True, sample_ids, None, None, out, bags, mode, weights, stream, wait)

    # ---------------------------------------------------------------- pooled accumulates (embedding_bag backward)
    def accumulate_batch_pooled(self, name, starts, counts=None, count=None, grad=None, bags=None, mode="sum",
                                weights=None, alpha=1.0, stream=None, wait=True):
        """Scatter each bag's gradient into its rows, in ONE kernel launch: the adjoint of get_batch_pooled with the same
        requests, bags, mode ("sum" or "mean") and weights -- torch's embedding_bag backward fused with the SGD step
        p.add_(g, alpha=alpha) over a sharded variable. grad (a C-contiguous CUDA float32, float64, float16 or bfloat16
        tensor of the variable's itemsize) holds nbags rows of disp elements. Every row of every valid request i of bag
        k gets grad[k] * weights[i] (weighted sum), / n_k (mean: n_k the rows the pooled get folds for bag k), * alpha,
        each step rounded once in float32 (float64 for float64 rows), then rounded to grad.dtype and added atomically
        into the shard as accumulate_batch adds (atomic across ranks and duplicate ids, in no fixed order). Requests,
        bags, errors and wait=False are get_batch_pooled's: an invalid request adds nothing and is left out of n_k, a
        malformed bag adds nothing and raises before any request error. alpha must be finite. The rows are visible at
        the next fence. Returns nbags * R bytes (None with wait=False)."""
        return self._pooled(name, False, starts, counts, count, grad, bags, mode, weights, stream, wait, True, alpha)

    def accumulate_samples_pooled(self, name, sample_ids, grad, bags=None, mode="sum", weights=None, alpha=1.0,
                                  stream=None, wait=True):
        """accumulate_batch_pooled by SAMPLE ID: request i = the rows of sample sample_ids[i] in the index registered
        with set_sample_index (the backward of get_samples_pooled)."""
        return self._pooled(name, True, sample_ids, None, None, grad, bags, mode, weights, stream, wait, True, alpha)

    def _pooled(self, name, by_sample, starts, counts, count, buf, bags, mode, weights, stream, wait, acc=False,
                alpha=1.0):
        """the pooled batches into `buf` = out, or (acc) the pooled accumulates from `buf` = grad"""
        modec, dtc = _pool_acc_args(name, mode, alpha, buf) if acc else _pool_args(name, mode, buf)
        sa, ca, ba, wa, s_dev = _pool_requests(starts, counts, bags, weights, buf, wait)
        nreq = sa.numel()
        nbags = ba.numel() - 1 if ba is not None else nreq
        pool = _capi.Pool(modec, dtc, ba.data_ptr() if ba is not None else None, nbags,
                          wa.data_ptr() if wa is not None else None)
        flags = ((_capi.SRC_ON_DEVICE if acc else _capi.DST_ON_DEVICE) | (_capi.IDX_ON_DEVICE if s_dev else 0)
                 | (0 if wait else _capi.NO_SYNC))
        operands = (C.byref(pool), *((float(alpha),) if acc else ()), buf.data_ptr(), buf.numel() * buf.element_size())
        entry = f"dds_{'accumulate' if acc else 'get'}_{'samples' if by_sample else 'batch'}_pooled"
        if by_sample:
            total = self._call(getattr(self._L, entry), self._h, name.encode(), sa.data_ptr(), nreq, *operands, flags,
                               _stream_handle(stream))
        else:
            total = self._call(getattr(self._L, entry), self._h, name.encode(), sa.data_ptr(),
                               ca.data_ptr() if ca is not None else None, 1 if count is None else int(count), nreq,
                               *operands, flags, _stream_handle(stream))
        return total if wait else None

    # ---------------------------------------------------------------- collective owner-push fetch
    def push_setup(self, max_requests, max_bytes):
        """COLLECTIVE: allocate and peer-map the windows of the push fetch (see dds_push_setup)."""
        _capi.raise_for(self._L.dds_push_setup(self._h, int(max_requests), int(max_bytes)))

    def get_batch_push(self, name, starts, count=1, stream=None):
        """COLLECTIVE fetch of len(starts) requests (CUDA int64 tensor) of `count` rows each, by owner-push. Returns a
        uint8 CUDA tensor VIEW of the packed rows inside this rank's window (valid until the next-but-one push step);
        the step is enqueued on `stream`, wait() reports errors."""
        import torch
        itemsize = self._var_itemsize(name)
        if not (hasattr(starts, "data_ptr") and starts.is_cuda):
            raise ValueError("get_batch_push takes a CUDA int64 tensor of start rows")
        out = C.c_void_p()
        _capi.raise_for(self._L.dds_get_batch_push(self._h, name.encode(), starts.data_ptr(), int(count), starts.numel(), itemsize,
                                                   C.byref(out), _stream_handle(stream)))
        rb = self._rowbytes.get(name)
        if rb is None:
            rb = self._rowbytes[name] = self.query(name)["disp"] * itemsize
        nbytes = starts.numel() * int(count) * rb
        return torch.as_tensor(_DevMem(out.value or 0, nbytes), device=starts.device)

    # ---------------------------------------------------------------- per-sample index (variable-length datasets)
    def set_sample_index(self, name, row_start, row_count):
        """Register, for variable `name`, which GLOBAL rows every sample owns: sample i = rows
        [row_start[i], row_start[i] + row_count[i]). Tables: int64 host arrays or CUDA tensors; copied once."""
        n, sp, cp, dev, keep = _requests(row_start, row_count)
        _capi.raise_for(self._L.dds_set_sample_index(self._h, name.encode(), sp, cp, n, 1 if dev else 0))
        del keep

    def set_normalization(self, name, mean, std, inner=1):
        """Register the per-channel normalisation of variable `name` for batches fetched with normalize=True: element e
        of a row is in channel (e // inner) % len(mean) and becomes (x - mean[ch]) / std[ch]. mean / std: 1-D float32
        arrays of one length (ndarray or tensor, host or CUDA), copied. One value: a scalar; disp values with inner=1:
        per feature; C values with inner=H*W: a CHW image. Empty tables remove the normalisation. Local to this rank."""
        m, s, n, dev = _norm_tables(mean, std)
        _capi.raise_for(self._L.dds_set_normalization(self._h, name.encode(), _ptr(m) if n else None,
                                                      _ptr(s) if n else None, n, int(inner), dev))
        del m, s

    def get_samples(self, name, sample_ids, out, offsets=None, stream=None, wait=True, overlap=False, src_dtype=None,
                    lut=None, normalize=False, pad_rows=None, pad_value=0, lengths=None):
        """get_batch by SAMPLE ID: the id -> (start, count) lookup runs inside the launch, against the index
        registered with set_sample_index. Same packing / offsets / error behaviour, conversions and padding (pad_rows,
        pad_value, lengths) as get_batch."""
        return self._get(name, True, sample_ids, None, None, out, offsets, stream, wait, overlap, src_dtype, lut,
                         normalize, pad_rows, pad_value, lengths)

    def _get(self, name, by_sample, starts, counts, count, out, offsets, stream, wait, overlap, src_dtype, lut,
             normalize, pad_rows, pad_value, lengths):
        """get_batch, and get_samples (by_sample: starts are sample ids, counts and count are None)"""
        cv, lut_keep = _get_args(by_sample, counts, count, out, offsets, src_dtype, lut, normalize, pad_rows)
        if cv is None:
            itemsize = self._var_itemsize(name)
        ob = _Buf(out, writable=True, half_ok=cv is not None or pad_rows is not None)
        nreq, sp, cp, s_dev, keep = _requests(starts, counts)
        flags = (_capi.IDX_ON_DEVICE if s_dev else 0) | (_capi.DST_ON_DEVICE if ob.on_device else 0)
        if not wait:
            flags |= _capi.NO_SYNC | (_capi.OVERLAP if overlap else 0)
        if pad_rows is not None:
            return self._padded(name, by_sample, sp, cp, nreq, out, ob, cv, pad_rows, pad_value, lengths, flags, stream)
        op = _offsets(offsets, ob, nreq, by_sample)
        reqs = (sp, nreq) if by_sample else (sp, cp, 1 if count is None else int(count), nreq)
        if cv is None:
            fn = self._L.dds_get_samples if by_sample else self._L.dds_get_batch
            return self._call(fn, self._h, name.encode(), *reqs, itemsize, ob.ptr, ob.nbytes, op, flags,
                              _stream_handle(stream))
        fn = self._L.dds_get_samples_convert if by_sample else self._L.dds_get_batch_convert
        return self._call(fn, self._h, name.encode(), *reqs, ob.ptr, ob.nbytes, op, flags, _stream_handle(stream),
                          C.byref(cv))

    def _padded(self, name, by_sample, sp, cp, nreq, out, ob, cv, pad_rows, pad_value, lengths, flags, stream):
        """the padded form of get_batch / get_samples (arguments already converted by _get)"""
        pad_rows = _pad_rows(pad_rows, out, ob)
        itemsize = self._var_itemsize(name)
        if cv is None and ob.itemsize != itemsize:
            raise ValueError(f"out.dtype {out.dtype} does not have the variable's itemsize ({itemsize})")
        pad = _pad(pad_rows, pad_value, lengths, out, nreq)
        reqs = (sp, nreq) if by_sample else (sp, cp, nreq)
        fn = self._L.dds_get_samples_padded if by_sample else self._L.dds_get_batch_padded
        return self._call(fn, self._h, name.encode(), *reqs, itemsize, C.byref(cv) if cv is not None else None,
                          C.byref(pad), ob.ptr, ob.nbytes, flags, _stream_handle(stream))

    def get_samples_multi(self, names, sample_ids, outs, offsets=None, stream=None, wait=True, overlap=False,
                          src_dtypes=None, luts=None, normalize=None):
        """The rows of the same samples in several variables (<= 4, each with a sample index) in ONE launch:
        outs[v] (CUDA tensors) receive variable names[v]'s packed rows, offsets[v] (optional int64 CUDA tensors of
        len(ids)+1) the per-sample byte offsets. Returns the list of packed sizes (None when wait=False).
        src_dtypes[v] / luts[v]: variable v delivered converted to outs[v].dtype, as in get_batch (None: raw bytes);
        its offsets and size are then in bytes of outs[v]. normalize[v] (with src_dtypes[v]): variable v normalised, as
        in get_batch."""
        nv = len(names)
        cvs = None
        if normalize is not None:
            normalize = [bool(x) for x in normalize]
            if len(normalize) != nv:
                raise ValueError("normalize needs one entry per variable")
            if any(nz and (src_dtypes is None or src_dtypes[v] is None) for v, nz in enumerate(normalize)):
                raise ValueError("a normalised variable needs its src_dtypes entry")
        else:
            normalize = [False] * nv
        if src_dtypes is not None:
            luts = [None] * nv if luts is None else list(luts)
            if len(src_dtypes) != nv or len(luts) != nv:
                raise ValueError("src_dtypes / luts need one entry per variable")
            pairs = [(_capi.Convert(_capi.CVT_NONE, None), None) if sd is None else _conversion(sd, getattr(o, "dtype", None), lt, nz)
                     for sd, o, lt, nz in zip(src_dtypes, outs, luts, normalize)]
            cvs = (_capi.Convert * nv)(*[c for c, _ in pairs])
            lut_keep = [k for _, k in pairs]
        obs = [_Buf(o, writable=True, half_ok=cvs is not None and src_dtypes[v] is not None) for v, o in enumerate(outs)]
        if not all(o.on_device for o in obs):
            raise ValueError("get_samples_multi delivers into device buffers")
        nreq, sp, _, s_dev, keep = _requests(sample_ids)
        flags = (_capi.IDX_ON_DEVICE if s_dev else 0) | _capi.DST_ON_DEVICE | (0 if wait else _capi.NO_SYNC)
        if overlap and not wait:
            flags |= _capi.OVERLAP
        c_names = (C.c_char_p * nv)(*[n.encode() for n in names])
        c_dsts = (C.c_void_p * nv)(*[o.ptr for o in obs])
        c_caps = (C.c_int64 * nv)(*[o.nbytes for o in obs])
        c_offs = None
        if offsets is not None:
            fbs = [_Buf(f, writable=True) for f in offsets]
            c_offs = (C.c_void_p * nv)(*[f.ptr for f in fbs])
        totals = (C.c_int64 * nv)()
        if cvs is None:
            self._call(self._L.dds_get_samples_multi, self._h, nv, c_names, sp, nreq, c_dsts, c_caps, c_offs, flags,
                       _stream_handle(stream), totals=totals)
        else:
            self._call(self._L.dds_get_samples_multi_convert, self._h, nv, c_names, sp, nreq, c_dsts, c_caps, c_offs,
                       flags, _stream_handle(stream), cvs, totals=totals)
        return [totals[v] for v in range(nv)] if wait else None

    def wait(self):
        """Complete the batches queued with wait=False; raises like get_batch for the earliest failing batch in queue
        order (last_bad_index: its first invalid request); returns the packed bytes of the last batch queued since the
        previous wait() (0 if none).
        wait() alone reports the outcome of queued batches, exactly once. Any other call that meets a pending queue
        (a synchronous get_batch / get / get_samples / get_samples_multi / put_batch / put_samples / accumulate_batch /
        accumulate_samples / get_accumulate_batch / get_accumulate_samples / compare_and_swap_batch /
        compare_and_swap_samples, a batch on another stream, set_sample_index, set_normalization, epoch_end,
        epoch_begin when the queue holds a put, an accumulate, a fetch-op or a compare-and-swap, free) completes it, keeps its first failure for the next wait(), and raises only
        for its own requests. A failure kept from earlier wins over later ones; after wait() has raised it, the next
        wait() is clean. close() drops an outcome no wait() has reported."""
        return self._call(self._L.dds_batch_wait, self._h)

    def _call(self, fn, *args, totals=None):
        """fn(*args, &total, &bad) -- a batched C entry, or totals (an int64 array) in place of &total -> total. Sets
        last_bad_index and raises the reference's exception for a failed call."""
        total, bad = C.c_int64(0), C.c_int64(-1)
        rc = fn(*args, C.byref(total) if totals is None else totals, C.byref(bad))
        self.last_bad_index = bad.value
        if rc:
            _capi.raise_for(rc)
        return total.value

    def _var_itemsize(self, name):
        itemsize = self._itemsize.get(name)
        if itemsize is None:
            itemsize = self._itemsize[name] = self.query(name)["itemsize"]
        return itemsize

    # ---------------------------------------------------------------- extras
    def query(self, name):
        vi = _capi.VarInfo()
        _capi.raise_for(self._L.dds_query(self._h, name.encode(), C.byref(vi)))
        pl = C.c_int(0)
        _capi.raise_for(self._L.dds_query_placement(self._h, name.encode(), C.byref(pl)))
        return {"placement": _PLACEMENT_NAMES[pl.value],"itemsize": vi.itemsize, "disp": vi.disp, "nranks": vi.nranks, "fence_active": bool(vi.fence_active),
                "local_nrows": vi.local_nrows, "total_nrows": vi.total_nrows,
                "lenlist": [vi.lenlist[i] for i in range(vi.nranks)], "local_base": vi.local_base}

    def synth_fill(self, name, seed):
        _capi.raise_for(self._L.dds_synth_fill(self._h, name.encode(), int(seed)))

    def synth_verify(self, name, packed, starts, counts=None, count=1, offsets=None, seed=0, stream=None):
        """Check a packed batch (CUDA tensors) of variable `name` -- filled by synth_fill(name, seed) -- against the
        generator on the device. Returns (mismatching elements, rows checked, requests per owner rank)."""
        res = (C.c_uint64 * 66)()
        _capi.raise_for(self._L.dds_synth_verify(
            self._h, name.encode(), packed.data_ptr(), starts.data_ptr(), counts.data_ptr() if counts is not None else None,
            int(count), offsets.data_ptr() if offsets is not None else None, starts.numel(), int(seed),
            _stream_handle(stream), res))
        return int(res[0]), int(res[1]), [int(res[2 + r]) for r in range(self.size)]

    def close(self):
        """non-collective teardown of this rank's handle (the collective one is free())"""
        if self._h:
            self._L.dds_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass
