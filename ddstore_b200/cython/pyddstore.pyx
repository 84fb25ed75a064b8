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

from ddstore_b200._capi import PLACEMENTS
from ddstore_b200.comm import as_dds_comm
from ddstore_b200.store import (_PLACEMENT_NAMES as PLACEMENT_NAMES, _Buf, _acc_type, _cas_args, _dtype_name, _fop_args,
                                _get_args, _norm_tables, _offsets, _pad, _pad_rows, _placement, _pool_acc_args, _pool_args,
                                _pool_requests, _ptr, _put_src, _red_op, _requests, _stream_handle)

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
        long accumulate_batch_pooled(string name, const long* starts, const long* counts, long fixed_count, long nreq,
                                     int mode, int dtype, const long* bags, long nbags, const void* weights,
                                     double alpha, const void* grad, long grad_bytes, cbool idx_on_device,
                                     void* stream) except +dds_translate_exception
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
        cv, lut_keep = _get_args(False, counts, count, out, offsets, src_dtype, lut, normalize, pad_rows)
        ob = _Buf(out, writable=True, half_ok=cv is not None or pad_rows is not None)
        py_nreq, py_sp, py_cp, s_dev, keep = _requests(starts, counts)
        if pad_rows is not None:
            return self._get_batch_padded(name, py_sp, py_cp, py_nreq, s_dev, out, ob, stream, src_dtype, cv, pad_rows,
                                          pad_value, lengths)
        if cv is None and s_dev != bool(ob.on_device):
            raise ValueError("the Cython get_batch wants indices and out on the same side (both host or both device)")
        if cv is not None and not ob.on_device:
            raise ValueError("converting batches deliver into device memory")
        cdef size_t op = _offsets(offsets, ob, py_nreq, False) or 0
        cdef size_t sp = py_sp, cp = py_cp or 0, dp = ob.ptr, lp = (cv.lut or 0) if cv is not None else 0
        cdef long nreq = py_nreq, fixed = 1 if count is None else int(count), cap = ob.nbytes
        cdef size_t st = _stream_handle(stream)
        cdef string nm = name.encode()
        cdef int w = ob.itemsize, code = cv.code if cv is not None else 0
        cdef cbool dev = s_dev
        cdef long total
        with nogil:
          if code:
            total = self.c_ddstore.get_batch_convert(nm, <const long*> sp, <const long*> cp, fixed, nreq, <void*> dp, cap,
                                                     code, <const void*> lp, <long*> op, dev, <void*> st)
          elif w == 1:
            total = self.c_ddstore.get_batch[char](nm, <const long*> sp, <const long*> cp, fixed, nreq, <char*> dp, cap, <long*> op, dev, <void*> st)
          elif w == 4:
            total = self.c_ddstore.get_batch[int](nm, <const long*> sp, <const long*> cp, fixed, nreq, <int*> dp, cap, <long*> op, dev, <void*> st)
          else:
            total = self.c_ddstore.get_batch[long](nm, <const long*> sp, <const long*> cp, fixed, nreq, <long*> dp, cap, <long*> op, dev, <void*> st)
        del keep, lut_keep
        return total

    def _get_batch_padded(self, str name, py_sp, py_cp, py_nreq, s_dev, out, ob, stream, src_dtype, cv, pad_rows,
                          pad_value, lengths):
        cdef long max_rows = _pad_rows(pad_rows, out, ob)
        pad = _pad(max_rows, pad_value, lengths, out, py_nreq)
        cdef size_t sp = py_sp, cp = py_cp, dp = ob.ptr, lp = (cv.lut or 0) if cv is not None else 0
        cdef size_t lnp = pad.lengths or 0
        cdef int itemsize = ob.itemsize if cv is None else np.dtype(_dtype_name(src_dtype)).itemsize
        cdef int code = 0 if cv is None else cv.code
        cdef uint64_t bits = pad.pad_bits
        cdef long nreq = py_nreq, cap = ob.nbytes
        cdef size_t st = _stream_handle(stream)
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
        cdef long total
        with nogil:
            total = self.c_ddstore.get_batch_padded_convert(nm, <const long*> sp, <const long*> cp, nreq, itemsize, code,
                                                            <const void*> lp, max_rows, bits, <void*> dp, cap,
                                                            <long*> lnp, idx_dev, <void*> st)
        return total

    def put_batch(self, str name, starts, counts=None, src=None, count=None, stream=None):
        """one kernel launch writing len(starts) requests from the CUDA tensor `src` into the owners' shards; see
        ddstore_b200.store.PyDDStore.put_batch (this binding's put is synchronous). Returns the layout's bytes."""
        sb = _put_src(name, src)
        py_nreq, py_sp, py_cp, s_dev, keep = _requests(starts, counts)
        cdef size_t sp = py_sp, cp = py_cp or 0, dp = sb.ptr, st = _stream_handle(stream)
        cdef long nreq = py_nreq, fixed = 1 if count is None else int(count), nbytes = sb.nbytes
        cdef int w = sb.itemsize
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
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
        sb = _put_src(name, src)
        cdef int code = _acc_type(name, src), opc = _red_op(name, op)
        py_nreq, py_sp, py_cp, s_dev, keep = _requests(starts, counts)
        cdef size_t sp = py_sp, cp = py_cp or 0, dp = sb.ptr, st = _stream_handle(stream)
        cdef long nreq = py_nreq, fixed = 1 if count is None else int(count), nbytes = sb.nbytes
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
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
        modes_types = _pool_args(name, mode, out)
        cdef int modec = modes_types[0], code = modes_types[1]
        sa, ca, ba, wa, s_dev = _pool_requests(starts, counts, bags, weights, out, True)
        cdef long nreq = sa.numel()
        cdef long nbags = ba.numel() - 1 if ba is not None else nreq
        cdef size_t sp = sa.data_ptr(), cp = ca.data_ptr() if ca is not None else 0
        cdef size_t bp = ba.data_ptr() if ba is not None else 0, wp = wa.data_ptr() if wa is not None else 0
        cdef size_t dp = out.data_ptr(), st = _stream_handle(stream)
        cdef long cap = out.numel() * out.element_size(), fixed = 1 if count is None else int(count)
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
        cdef long total
        with nogil:
            total = self.c_ddstore.get_batch_pooled(nm, <const long*> sp, <const long*> cp, fixed, nreq, modec, code,
                                                    <const long*> bp, nbags, <const void*> wp, <void*> dp, cap, idx_dev,
                                                    <void*> st)
        del sa, ca, ba, wa
        return total

    def accumulate_batch_pooled(self, str name, starts, counts=None, count=None, grad=None, bags=None, mode="sum",
                                weights=None, alpha=1.0, stream=None):
        """one kernel launch scattering each bag's row of the CUDA tensor `grad` (float32, float64, float16 or bfloat16)
        into the rows of its requests, the adjoint of get_batch_pooled; see
        ddstore_b200.store.PyDDStore.accumulate_batch_pooled (this binding's call is synchronous). Returns nbags * R."""
        modes_types = _pool_acc_args(name, mode, alpha, grad)
        cdef int modec = modes_types[0], code = modes_types[1]
        sa, ca, ba, wa, s_dev = _pool_requests(starts, counts, bags, weights, grad, True)
        cdef long nreq = sa.numel()
        cdef long nbags = ba.numel() - 1 if ba is not None else nreq
        cdef size_t sp = sa.data_ptr(), cp = ca.data_ptr() if ca is not None else 0
        cdef size_t bp = ba.data_ptr() if ba is not None else 0, wp = wa.data_ptr() if wa is not None else 0
        cdef size_t gp = grad.data_ptr(), st = _stream_handle(stream)
        cdef long nbytes = grad.numel() * grad.element_size(), fixed = 1 if count is None else int(count)
        cdef double a = alpha
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
        cdef long total
        with nogil:
            total = self.c_ddstore.accumulate_batch_pooled(nm, <const long*> sp, <const long*> cp, fixed, nreq, modec,
                                                           code, <const long*> bp, nbags, <const void*> wp, a,
                                                           <const void*> gp, nbytes, idx_dev, <void*> st)
        del sa, ca, ba, wa
        return total

    def get_accumulate_batch(self, str name, starts, counts=None, src=None, out=None, op="sum", count=None,
                             stream=None):
        """one kernel launch ADDING (op="sum"), SWAPPING (op="replace") or reducing (accumulate_batch's ops) len(starts)
        requests of the CUDA tensor `src` into the owners' shards and writing the previous rows to the CUDA tensor `out` (src's layout, at least its
        bytes; it may be src); see ddstore_b200.store.PyDDStore.get_accumulate_batch (this binding's fetch-op is
        synchronous). Returns the layout's bytes."""
        sb = _put_src(name, src)
        cdef int code = _acc_type(name, src)
        opc_res = _fop_args(name, op, out, sb)
        cdef int opc = opc_res[0]
        py_nreq, py_sp, py_cp, s_dev, keep = _requests(starts, counts)
        cdef size_t sp = py_sp, cp = py_cp or 0, dp = sb.ptr, rp = opc_res[1], st = _stream_handle(stream)
        cdef long nreq = py_nreq, fixed = 1 if count is None else int(count), nbytes = sb.nbytes
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
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
        sb = _put_src(name, src)
        cmp_res = _cas_args(name, compare, out, sb)
        py_nreq, py_sp, py_cp, s_dev, keep = _requests(starts, counts)
        cdef size_t sp = py_sp, cp = py_cp or 0, dp = sb.ptr, qp = cmp_res[0], rp = cmp_res[1]
        cdef size_t st = _stream_handle(stream)
        cdef long nreq = py_nreq, fixed = 1 if count is None else int(count), nbytes = sb.nbytes
        cdef int itemsize = sb.itemsize
        cdef string nm = name.encode()
        cdef cbool idx_dev = s_dev
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
