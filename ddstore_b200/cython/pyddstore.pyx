# distutils: language=c++
# cython: language_level=3
"""pyddstore -- Cython binding with the reference module's name and Python surface
(/root/reference/src/pyddstore.pyx:58-131: PyDDStore(comm, method=0) with add / get / epoch_begin /
epoch_end / free / init / update), bound to the C++ class in include/ddstore_b200.hpp, which is a thin
wrapper over the C-ABI (include/ddstore_b200.h) of libddstore_b200.so.

Differences from the reference binding, all at the edges:
  * `comm` is anything ddstore_b200.comm.as_dds_comm accepts (an mpi4py-style communicator, a
    torch.distributed adapter, ShmComm, None) -- MPI is not required;
  * arrays may also be CUDA tensors / __cuda_array_interface__ objects (then nothing touches the host);
  * `get_batch` fetches a whole batch in one kernel launch.
"""
from libcpp.string cimport string
from libcpp cimport bool as cbool
from libc.stdint cimport uint64_t

import numpy as np

from ddstore_b200.comm import as_dds_comm
from ddstore_b200.store import _Buf, _conversion, _dtype_name, _i64, _norm_tables, _pad_bits, _ptr

cdef extern from *:
    """
    #include <stdexcept>
    #include <Python.h>
    static void dds_translate_exception() {
        try { throw; }
        catch (const std::invalid_argument &e) { PyErr_SetString(PyExc_ValueError, e.what()); }
        catch (const std::out_of_range &e) { PyErr_SetString(PyExc_KeyError, e.what()); }
        catch (const std::exception &e) { PyErr_SetString(PyExc_RuntimeError, e.what()); }
    }
    """
    void dds_translate_exception()

cdef extern from "ddstore_b200.h":
    ctypedef struct dds_comm_t:
        pass

cdef extern from "ddstore_b200.hpp" nogil:
    cdef cppclass DDStore:
        DDStore(int method, dds_comm_t* comm, int device) except +dds_translate_exception
        void add[T](string name, T* buffer, long nrows, int disp, int placement) except +dds_translate_exception
        void add_device[T](string name, const T* buffer, long nrows, int disp, int placement) except +dds_translate_exception
        void get[T](string name, long start, long count, T* buffer) except +dds_translate_exception
        void get_device[T](string name, long start, long count, T* buffer) except +dds_translate_exception
        long get_batch[T](string name, const long* starts, const long* counts, long fixed_count, long nreq, T* dst,
                          long cap, long* offsets, cbool on_device, void* stream) except +dds_translate_exception
        long get_batch_convert(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                               void* dst, long cap, int code, const void* lut, long* offsets, cbool idx_on_device,
                               void* stream) except +dds_translate_exception
        long get_batch_padded_convert(string name, const long* starts, const long* counts, long nreq, int itemsize,
                                      int code, const void* lut, long max_rows, uint64_t pad_bits, void* dst, long cap,
                                      long* lengths, cbool idx_on_device, void* stream) except +dds_translate_exception
        void set_normalization(string name, const float* mean, const float* std, long nchan, long inner,
                               cbool tables_on_device) except +dds_translate_exception
        long put_batch[T](string name, const long* starts, const long* counts, long fixed_count, long nreq, const T* src,
                          long src_bytes, cbool idx_on_device, void* stream) except +dds_translate_exception
        long accumulate_batch(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                              int dtype, const void* src, long src_bytes, cbool idx_on_device,
                              void* stream) except +dds_translate_exception
        long accumulate_op_batch(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                                 int op, int dtype, const void* src, long src_bytes, cbool idx_on_device,
                                 void* stream) except +dds_translate_exception
        long get_accumulate_batch(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                                  int op, int dtype, const void* src, void* result, long src_bytes, cbool idx_on_device,
                                  void* stream) except +dds_translate_exception
        long get_batch_pooled(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                              int mode, int dtype, const long* bags, long nbags, const void* weights, void* dst,
                              long dst_capacity_bytes, cbool idx_on_device, void* stream) except +dds_translate_exception
        long compare_and_swap_batch(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                                    int itemsize, const void* src, const void* compare, void* result, long src_bytes,
                                    cbool idx_on_device, void* stream) except +dds_translate_exception
        void epoch_begin() except +dds_translate_exception
        void epoch_end() except +dds_translate_exception
        void free() except +dds_translate_exception
        void init(string name, long nrows, int disp, int itemsize, int placement) except +dds_translate_exception
        int placement(string name) except +dds_translate_exception
        void update[T](string name, T* buffer, long nrows, long offset) except +dds_translate_exception
        int rank()
        int size()


# where a variable's shards live (DDS_PLACE_*), by name
PLACEMENTS = {"hbm": 0, "host": 1}
PLACEMENT_NAMES = {v: k for k, v in PLACEMENTS.items()}


def _placement(str placement):
    if placement not in PLACEMENTS:
        raise ValueError(f"unknown placement {placement!r} (expected 'hbm' or 'host')")
    return PLACEMENTS[placement]


# element types of accumulate_batch (DDS_ACC_*), by dtype name
_ACC_TYPES = {"float32": 1, "float64": 2, "int32": 3, "int64": 4, "float16": 5, "bfloat16": 6}
# ops of get_accumulate_batch (DDS_OP_*), by name
_FOP_OPS = {"sum": 1, "replace": 2}
# reductions of accumulate_batch and get_accumulate_batch beside the sum (DDS_OP_MAX..), by torch's names
_RED_OPS = {"amax": 4, "amin": 5, "bitwise_and": 6, "bitwise_or": 7, "bitwise_xor": 8}
# pooling modes of get_batch_pooled (DDS_POOL_*), by torch's embedding_bag names
_POOL_MODES = {"sum": 1, "mean": 2, "max": 3}

cdef class PyDDStore:
    cdef DDStore* c_ddstore
    cdef object _comm

    def __cinit__(self, comm=None, int method=0, device=None):
        self._comm = as_dds_comm(comm)
        cdef size_t h = <size_t> self._comm.handle
        cdef int dev = -1 if device is None else int(device)
        # every call below may block on the other ranks (collectives) or on the GPU: never hold the GIL across it,
        # so thread-ranks of one interpreter cannot deadlock each other
        with nogil:
            self.c_ddstore = new DDStore(method, <dds_comm_t*> h, dev)

    def __dealloc__(self):
        if self.c_ddstore != NULL:
            del self.c_ddstore
            self.c_ddstore = NULL

    @property
    def rank(self):
        return self.c_ddstore.rank()

    @property
    def size(self):
        return self.c_ddstore.size()

    def add(self, str name, arr, str placement="hbm"):
        cdef int pl = _placement(placement)
        b = _Buf(arr)
        cdef long nrows = b.shape[0]
        cdef int disp = (b.size // b.shape[0]) if b.shape[0] else int(np.prod(b.shape[1:], dtype=np.int64))
        cdef size_t p = b.ptr
        cdef string nm = name.encode()
        cdef int w = b.itemsize
        if b.on_device:
            with nogil:
                if w == 1: self.c_ddstore.add_device[char](nm, <const char*> p, nrows, disp, pl)
                elif w == 4: self.c_ddstore.add_device[int](nm, <const int*> p, nrows, disp, pl)
                else: self.c_ddstore.add_device[long](nm, <const long*> p, nrows, disp, pl)
        else:
            with nogil:
                if w == 1: self.c_ddstore.add[char](nm, <char*> p, nrows, disp, pl)
                elif w == 4: self.c_ddstore.add[int](nm, <int*> p, nrows, disp, pl)
                else: self.c_ddstore.add[long](nm, <long*> p, nrows, disp, pl)

    def get(self, str name, arr, long start=0):
        b = _Buf(arr, writable=True)
        cdef long count = b.shape[0]
        cdef size_t p = b.ptr
        cdef string nm = name.encode()
        cdef int w = b.itemsize
        if b.on_device:
            with nogil:
                if w == 1: self.c_ddstore.get_device[char](nm, start, count, <char*> p)
                elif w == 4: self.c_ddstore.get_device[int](nm, start, count, <int*> p)
                else: self.c_ddstore.get_device[long](nm, start, count, <long*> p)
        else:
            with nogil:
                if w == 1: self.c_ddstore.get[char](nm, start, count, <char*> p)
                elif w == 4: self.c_ddstore.get[int](nm, start, count, <int*> p)
                else: self.c_ddstore.get[long](nm, start, count, <long*> p)

    def get_batch(self, str name, starts, counts=None, out=None, count=None, offsets=None, stream=None, src_dtype=None,
                  lut=None, normalize=False, pad_rows=None, pad_value=0, lengths=None):
        """one kernel launch for len(starts) requests, packed in request order into `out`; see
        ddstore_b200.store.PyDDStore.get_batch. `out` decides the element width checked against the variable.
        src_dtype / lut: deliver the rows converted to out.dtype (a CUDA tensor), as in ddstore_b200's get_batch;
        normalize=True: normalised with the tables of set_normalization, as there.
        pad_rows / pad_value / lengths (with counts and a CUDA tensor `out`): a padded batch, as there."""
        if out is None:
            raise ValueError("get_batch needs an `out` buffer")
        cv = lut_keep = None
        if normalize and src_dtype is None:
            raise ValueError("normalize=True needs src_dtype")
        if pad_rows is not None and (counts is None or count is not None or offsets is not None):
            raise ValueError("pad_rows needs counts, and takes neither `count` nor `offsets`")
        if src_dtype is not None:
            cv, lut_keep = _conversion(src_dtype, getattr(out, "dtype", None), lut, normalize)
        ob = _Buf(out, writable=True, half_ok=cv is not None or pad_rows is not None)
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        if pad_rows is not None:
            return self._get_batch_padded(name, starts, counts, out, ob, stream, src_dtype, cv, lut_keep, bool(s_dev),
                                          pad_rows, pad_value, lengths)
        if cv is not None:
            return self._get_batch_convert(name, starts, counts, ob, count, offsets, stream, cv, lut_keep, bool(s_dev))
        if bool(s_dev) != bool(ob.on_device):
            raise ValueError("the Cython get_batch wants indices and out on the same side (both host or both device)")
        cdef size_t sp, cp = 0, op = 0, dp = ob.ptr
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        if offsets is not None:
            fb = _Buf(offsets, writable=True)
            op = fb.ptr
        cdef long fixed = 1 if count is None else int(count)
        cdef long cap = ob.nbytes
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef int w = ob.itemsize
        cdef cbool dev = bool(ob.on_device)
        cdef long total
        with nogil:
          if w == 1:
            total = self.c_ddstore.get_batch[char](nm, <const long*> sp, <const long*> cp, fixed, nreq, <char*> dp, cap, <long*> op, dev, <void*> st)
          elif w == 4:
            total = self.c_ddstore.get_batch[int](nm, <const long*> sp, <const long*> cp, fixed, nreq, <int*> dp, cap, <long*> op, dev, <void*> st)
          else:
            total = self.c_ddstore.get_batch[long](nm, <const long*> sp, <const long*> cp, fixed, nreq, <long*> dp, cap, <long*> op, dev, <void*> st)
        del keep
        return total

    def _get_batch_convert(self, str name, starts, counts, ob, count, offsets, stream, cv, lut_keep, s_dev):
        cdef size_t sp, cp = 0, op = 0, dp = ob.ptr, lp = cv.lut or 0
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        if offsets is not None:
            op = _Buf(offsets, writable=True).ptr
        cdef long fixed = 1 if count is None else int(count)
        cdef long cap = ob.nbytes
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef int code = cv.code
        cdef cbool idx_dev = s_dev
        cdef long total
        if not ob.on_device:
            raise ValueError("converting batches deliver into device memory")
        with nogil:
            total = self.c_ddstore.get_batch_convert(nm, <const long*> sp, <const long*> cp, fixed, nreq, <void*> dp, cap,
                                                     code, <const void*> lp, <long*> op, idx_dev, <void*> st)
        del keep, lut_keep
        return total

    def _get_batch_padded(self, str name, starts, counts, out, ob, stream, src_dtype, cv, lut_keep, s_dev, pad_rows,
                          pad_value, lengths):
        if not (ob.on_device and str(getattr(out, "dtype", "")).startswith("torch.")):
            raise ValueError("a padded batch delivers into a CUDA tensor")
        cdef size_t sp, cp, dp = ob.ptr, lp = (cv.lut or 0) if cv is not None else 0, lnp = 0
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr(); cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts); cp = ca.ctypes.data
            keep = (sa, ca)
        if lengths is not None:
            lb = _Buf(lengths, writable=True)
            if not lb.on_device or lb.itemsize != 8 or lb.size < nreq:
                raise ValueError("lengths must be an int64 CUDA tensor of len(starts)")
            lnp = lb.ptr
        cdef int itemsize = ob.itemsize if cv is None else np.dtype(_dtype_name(src_dtype)).itemsize
        cdef int code = 0 if cv is None else cv.code
        cdef long max_rows = int(pad_rows)
        if max_rows < 0:
            raise ValueError("pad_rows must be >= 0")
        cdef uint64_t bits = _pad_bits(pad_value, out.dtype)
        cdef long cap = ob.nbytes
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
        cdef long total
        with nogil:
            total = self.c_ddstore.get_batch_padded_convert(nm, <const long*> sp, <const long*> cp, nreq, itemsize, code,
                                                            <const void*> lp, max_rows, bits, <void*> dp, cap,
                                                            <long*> lnp, idx_dev, <void*> st)
        del keep, lut_keep
        return total

    def put_batch(self, str name, starts, counts=None, src=None, count=None, stream=None):
        """one kernel launch writing len(starts) requests from the CUDA tensor `src` into the owners' shards; see
        ddstore_b200.store.PyDDStore.put_batch (this binding's put is synchronous). Returns the layout's bytes."""
        if src is None:
            raise ValueError("a put needs `src` rows")
        if not (hasattr(src, "data_ptr") and getattr(src, "is_cuda", False)):
            raise ValueError(f"put into {name!r}: src must be a CUDA tensor (copy host rows to the device first)")
        if not src.is_contiguous():
            raise ValueError("src must be C-contiguous")
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        cdef size_t sp, cp = 0, dp = src.data_ptr()
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        cdef long fixed = 1 if count is None else int(count)
        cdef int w = src.element_size()
        cdef long nbytes = src.numel() * w
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = bool(s_dev)
        cdef long total
        with nogil:
            if w == 1: total = self.c_ddstore.put_batch[char](nm, <const long*> sp, <const long*> cp, fixed, nreq, <const char*> dp, nbytes, idx_dev, <void*> st)
            elif w == 2: total = self.c_ddstore.put_batch[short](nm, <const long*> sp, <const long*> cp, fixed, nreq, <const short*> dp, nbytes, idx_dev, <void*> st)
            elif w == 4: total = self.c_ddstore.put_batch[int](nm, <const long*> sp, <const long*> cp, fixed, nreq, <const int*> dp, nbytes, idx_dev, <void*> st)
            else: total = self.c_ddstore.put_batch[long](nm, <const long*> sp, <const long*> cp, fixed, nreq, <const long*> dp, nbytes, idx_dev, <void*> st)
        del keep
        return total

    def accumulate_batch(self, str name, starts, counts=None, src=None, count=None, stream=None, op="sum"):
        """one kernel launch ADDING (or reducing by op: "amax", "amin", "bitwise_and", "bitwise_or", "bitwise_xor")
        len(starts) requests of the CUDA tensor `src` into the owners' shards, in src's dtype (float32, float64, int32,
        int64, float16 or bfloat16); see ddstore_b200.store.PyDDStore.accumulate_batch (this binding's accumulate is
        synchronous). Returns the layout's bytes."""
        if src is None:
            raise ValueError("an accumulate needs `src` rows")
        if not (hasattr(src, "data_ptr") and getattr(src, "is_cuda", False)):
            raise ValueError(f"accumulate into {name!r}: src must be a CUDA tensor (copy host rows to the device first)")
        if not src.is_contiguous():
            raise ValueError("src must be C-contiguous")
        dt = str(src.dtype).replace("torch.", "")
        if dt not in _ACC_TYPES:
            raise ValueError(f"accumulate into {name!r}: src dtype {dt} is not one of {', '.join(_ACC_TYPES)}")
        ops = {"sum": 1, **_RED_OPS}
        if op not in ops:
            raise ValueError(f"accumulate into {name!r}: op {op!r} is not one of {', '.join(ops)}")
        cdef int code = _ACC_TYPES[dt], opc = ops[op]
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        cdef size_t sp, cp = 0, dp = src.data_ptr()
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        cdef long fixed = 1 if count is None else int(count)
        cdef long nbytes = src.numel() * src.element_size()
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = bool(s_dev)
        cdef long total
        with nogil:
            total = self.c_ddstore.accumulate_op_batch(nm, <const long*> sp, <const long*> cp, fixed, nreq, opc, code,
                                                       <const void*> dp, nbytes, idx_dev, <void*> st)
        del keep
        return total

    def get_batch_pooled(self, str name, starts, counts=None, count=None, out=None, bags=None, mode="sum",
                         weights=None, stream=None):
        """one kernel launch folding bags of requests into the rows of the CUDA tensor `out` (float32, float64, float16
        or bfloat16); see ddstore_b200.store.PyDDStore.get_batch_pooled (this binding's call is synchronous). bags and
        weights are converted to where starts lives. Returns the bytes written."""
        import torch
        if mode not in _POOL_MODES:
            raise ValueError(f"pooled batch of {name!r}: mode {mode!r} is not one of {', '.join(_POOL_MODES)}")
        if not (hasattr(out, "data_ptr") and getattr(out, "is_cuda", False)) or not out.is_contiguous():
            raise ValueError("out must be a C-contiguous CUDA tensor")
        dt = str(out.dtype).replace("torch.", "")
        if dt not in ("float32", "float64", "float16", "bfloat16"):
            raise ValueError(f"pooled batch of {name!r}: out dtype {dt} is not float32, float64, float16 or bfloat16")
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        dev = out.device if s_dev else "cpu"
        sa = torch.as_tensor(_i64(starts) if not s_dev else starts, dtype=torch.int64, device=dev).contiguous()
        ca = torch.as_tensor(_i64(counts) if not s_dev else counts, dtype=torch.int64, device=dev).contiguous() \
            if counts is not None else None
        ba = torch.as_tensor(_i64(bags) if not s_dev else bags, dtype=torch.int64, device=dev).contiguous() \
            if bags is not None else None
        wa = torch.as_tensor(weights, dtype=out.dtype, device=dev).contiguous() if weights is not None else None
        cdef long nreq = sa.numel()
        cdef long nbags = ba.numel() - 1 if ba is not None else nreq
        cdef size_t sp = sa.data_ptr(), cp = ca.data_ptr() if ca is not None else 0
        cdef size_t bp = ba.data_ptr() if ba is not None else 0, wp = wa.data_ptr() if wa is not None else 0
        cdef size_t dp = out.data_ptr()
        cdef long cap = out.numel() * out.element_size()
        cdef long fixed = 1 if count is None else int(count)
        cdef int modec = _POOL_MODES[mode], code = _ACC_TYPES[dt]
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = bool(s_dev)
        cdef long total
        with nogil:
            total = self.c_ddstore.get_batch_pooled(nm, <const long*> sp, <const long*> cp, fixed, nreq, modec, code,
                                                    <const long*> bp, nbags, <const void*> wp, <void*> dp, cap, idx_dev,
                                                    <void*> st)
        del sa, ca, ba, wa
        return total

    def get_accumulate_batch(self, str name, starts, counts=None, src=None, out=None, op="sum", count=None,
                             stream=None):
        """one kernel launch ADDING (op="sum"), SWAPPING (op="replace") or reducing (accumulate_batch's ops) len(starts)
        requests of the CUDA tensor `src` into the owners' shards and writing the previous rows to the CUDA tensor `out` (src's layout, at least its
        bytes; it may be src); see ddstore_b200.store.PyDDStore.get_accumulate_batch (this binding's fetch-op is
        synchronous). Returns the layout's bytes."""
        if src is None:
            raise ValueError("a fetch-op needs `src` rows")
        if not (hasattr(src, "data_ptr") and getattr(src, "is_cuda", False)):
            raise ValueError(f"fetch-op on {name!r}: src must be a CUDA tensor (copy host rows to the device first)")
        if not (hasattr(out, "data_ptr") and getattr(out, "is_cuda", False)):
            raise ValueError(f"fetch-op on {name!r}: out must be a CUDA tensor")
        if not src.is_contiguous() or not out.is_contiguous():
            raise ValueError("src and out must be C-contiguous")
        dt = str(src.dtype).replace("torch.", "")
        if dt not in _ACC_TYPES:
            raise ValueError(f"fetch-op on {name!r}: src dtype {dt} is not one of {', '.join(_ACC_TYPES)}")
        ops = {**_FOP_OPS, **_RED_OPS}
        if op not in ops:
            raise ValueError(f"fetch-op on {name!r}: op {op!r} is not one of {', '.join(ops)}")
        cdef long nbytes = src.numel() * src.element_size()
        if out.numel() * out.element_size() < nbytes:
            raise ValueError(f"fetch-op on {name!r}: out holds {out.numel() * out.element_size()} bytes, src {nbytes}")
        cdef int code = _ACC_TYPES[dt], opc = ops[op]
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        cdef size_t sp, cp = 0, dp = src.data_ptr(), rp = out.data_ptr()
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        cdef long fixed = 1 if count is None else int(count)
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = bool(s_dev)
        cdef long total
        with nogil:
            total = self.c_ddstore.get_accumulate_batch(nm, <const long*> sp, <const long*> cp, fixed, nreq, opc, code,
                                                        <const void*> dp, <void*> rp, nbytes, idx_dev, <void*> st)
        del keep
        return total

    def compare_and_swap_batch(self, str name, starts, counts=None, src=None, compare=None, out=None, count=None,
                               stream=None):
        """one kernel launch COMPARE-AND-SWAPPING len(starts) requests: each element of the rows becomes src's where it
        equals compare's bit for bit, and its previous value goes to `out` either way (compare and out: CUDA tensors of
        src's element size and at least its bytes, src's layout; out may be src or compare); see
        ddstore_b200.store.PyDDStore.compare_and_swap_batch (this binding's compare-and-swap is synchronous). Returns the
        layout's bytes."""
        if src is None:
            raise ValueError("a compare-and-swap needs `src` rows")
        for what, t in (("src", src), ("compare", compare), ("out", out)):
            if not (hasattr(t, "data_ptr") and getattr(t, "is_cuda", False)):
                raise ValueError(f"compare-and-swap on {name!r}: {what} must be a CUDA tensor")
            if not t.is_contiguous():
                raise ValueError(f"{what} must be C-contiguous")
            if t.element_size() != src.element_size():
                raise ValueError(f"compare-and-swap on {name!r}: {what} has {t.element_size()}-byte elements, src "
                                 f"{src.element_size()}-byte ones")
        cdef long nbytes = src.numel() * src.element_size()
        for what, t in (("compare", compare), ("out", out)):
            if t.numel() * t.element_size() < nbytes:
                raise ValueError(f"compare-and-swap on {name!r}: {what} holds {t.numel() * t.element_size()} bytes, "
                                 f"src {nbytes}")
        cdef int itemsize = src.element_size()
        s_dev = hasattr(starts, "data_ptr") and getattr(starts, "is_cuda", False)
        cdef size_t sp, cp = 0, dp = src.data_ptr(), qp = compare.data_ptr(), rp = out.data_ptr()
        cdef long nreq
        if s_dev:
            nreq = starts.numel(); sp = starts.data_ptr()
            if counts is not None: cp = counts.data_ptr()
            keep = (starts, counts)
        else:
            sa = _i64(starts); nreq = sa.size; sp = sa.ctypes.data
            ca = _i64(counts) if counts is not None else None
            if ca is not None: cp = ca.ctypes.data
            keep = (sa, ca)
        cdef long fixed = 1 if count is None else int(count)
        cdef size_t st = 0
        if stream is not None:
            st = int(stream) if int(stream) != 0 else 1
        cdef string nm = name.encode()
        cdef cbool idx_dev = bool(s_dev)
        cdef long total
        with nogil:
            total = self.c_ddstore.compare_and_swap_batch(nm, <const long*> sp, <const long*> cp, fixed, nreq, itemsize,
                                                          <const void*> dp, <const void*> qp, <void*> rp, nbytes,
                                                          idx_dev, <void*> st)
        del keep
        return total

    def set_normalization(self, str name, mean, std, long inner=1):
        """per-channel normalisation of `name` for normalize=True batches; see ddstore_b200.store.PyDDStore.set_normalization"""
        m, s, n, dev = _norm_tables(mean, std)
        cdef size_t mp = _ptr(m) if n else 0, sp = _ptr(s) if n else 0
        cdef long nchan = n
        cdef cbool on_dev = bool(dev)
        cdef string nm = name.encode()
        with nogil:
            self.c_ddstore.set_normalization(nm, <const float*> mp, <const float*> sp, nchan, inner, on_dev)
        del m, s

    def epoch_begin(self):
        with nogil:
            self.c_ddstore.epoch_begin()

    def epoch_end(self):
        with nogil:
            self.c_ddstore.epoch_end()

    def free(self):
        with nogil:
            self.c_ddstore.free()

    def init(self, str name, long nrows, int disp, int itemsize=1, str placement="hbm"):
        cdef int pl = _placement(placement)
        cdef string nm = name.encode()
        with nogil:
            self.c_ddstore.init(nm, nrows, disp, itemsize, pl)

    def placement(self, str name):
        cdef string nm = name.encode()
        return PLACEMENT_NAMES[self.c_ddstore.placement(nm)]

    def update(self, str name, arr, long offset):
        b = _Buf(arr)
        if b.on_device:
            raise NotImplementedError("update() from a device array: use ddstore_b200.PyDDStore")
        cdef long nrows = b.shape[0]
        cdef size_t p = b.ptr
        cdef string nm = name.encode()
        cdef int w = b.itemsize
        with nogil:
            if w == 1: self.c_ddstore.update[char](nm, <char*> p, nrows, offset)
            elif w == 4: self.c_ddstore.update[int](nm, <int*> p, nrows, offset)
            else: self.c_ddstore.update[long](nm, <long*> p, nrows, offset)
