"""ddstore_b200/_capi.py -- ctypes binding of the C-ABI in include/ddstore_b200.h.

Loads ddstore_b200/libddstore_b200.so (built in-tree by __graft_entry__.build() /
ddstore_b200/csrc/Makefile). If the library is missing this raises -- there is no Python or CPU
stand-in for the data path.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libddstore_b200.so")

DDS_OK = 0
ERR_DTYPE, ERR_START, ERR_COUNT, ERR_DISP, ERR_FENCE_ACTIVE, ERR_FENCE_INACTIVE = 1, 2, 3, 4, 5, 6
ERR_UNKNOWN_VAR, ERR_EXISTS, ERR_CUDA, ERR_COMM, ERR_ARG, ERR_CAPACITY, ERR_NO_DEVICE, ERR_WATCHDOG = \
    7, 8, 9, 10, 11, 12, 13, 14
IDX_ON_DEVICE, DST_ON_DEVICE, NO_SYNC, OVERLAP = 1, 2, 4, 8
SRC_ON_DEVICE = 2  # dds_put_*: the packed source rows are device memory (same bit as DST_ON_DEVICE)
# element types of the batched accumulates (DDS_ACC_*), by dtype name
ACC_F32, ACC_F64, ACC_I32, ACC_I64, ACC_F16, ACC_BF16 = 1, 2, 3, 4, 5, 6
ACC_TYPES = {"float32": ACC_F32, "float64": ACC_F64, "int32": ACC_I32, "int64": ACC_I64, "float16": ACC_F16,
             "bfloat16": ACC_BF16}
# ops of the batched fetch-ops (DDS_OP_*), by name
OP_SUM, OP_REPLACE = 1, 2
FOP_OPS = {"sum": OP_SUM, "replace": OP_REPLACE}
# reductions beside the sum (DDS_OP_MAX..), by torch's names: the batched reductions and the fetch-ops take them
OP_MAX, OP_MIN, OP_BAND, OP_BOR, OP_BXOR = 4, 5, 6, 7, 8
RED_OPS = {"amax": OP_MAX, "amin": OP_MIN, "bitwise_and": OP_BAND, "bitwise_or": OP_BOR, "bitwise_xor": OP_BXOR}

# where a variable's shards live (DDS_PLACE_*), by name
PLACE_HBM, PLACE_HOST = 0, 1
PLACEMENTS = {"hbm": PLACE_HBM, "host": PLACE_HOST}

ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t)
BARRIER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)


class VarInfo(C.Structure):
    _fields_ = [("itemsize", C.c_int32), ("disp", C.c_int32), ("nranks", C.c_int32), ("fence_active", C.c_int32),
                ("local_nrows", C.c_int64), ("total_nrows", C.c_int64), ("lenlist", C.c_int64 * 64),
                ("local_base", C.c_void_p)]


# conversions of the converting batch entries (DDS_CVT_*)
CVT_NONE, CVT_F32_BF16, CVT_F32_F16, CVT_F64_F32, CVT_U8_LUT16, CVT_U8_LUT32 = 0, 1, 2, 3, 4, 5
# normalising conversions ((x - mean[ch]) / std[ch] in f32; dds_set_normalization registers the tables)
CVT_NORM_F32_F32, CVT_NORM_F32_BF16, CVT_NORM_F32_F16, CVT_NORM_F64_F32 = 6, 7, 8, 9
CVT_NORM_U8_F32, CVT_NORM_U8_BF16, CVT_NORM_U8_F16 = 10, 11, 12


class Convert(C.Structure):  # dds_convert_t
    _fields_ = [("code", C.c_int32), ("lut", C.c_void_p)]


class Pad(C.Structure):  # dds_pad_t
    _fields_ = [("max_rows", C.c_int64), ("pad_bits", C.c_uint64), ("lengths", C.c_void_p)]


# pooling modes of the pooled batches (DDS_POOL_*), by torch's embedding_bag names
POOL_SUM, POOL_MEAN, POOL_MAX = 1, 2, 3
POOL_MODES = {"sum": POOL_SUM, "mean": POOL_MEAN, "max": POOL_MAX}


class Pool(C.Structure):  # dds_pool_t
    _fields_ = [("mode", C.c_int32), ("dtype", C.c_int32), ("bags", C.c_void_p), ("nbags", C.c_int64),
                ("weights", C.c_void_p)]


# every symbol include/ddstore_b200.h declares: name -> (restype, argtypes)
I64P = C.POINTER(C.c_int64)
SIGNATURES = {
    "dds_last_error": (C.c_char_p, []),
    "dds_strerror": (C.c_char_p, [C.c_int]),
    "dds_comm_self": (C.c_void_p, []),
    "dds_comm_shm": (C.c_void_p, [C.c_char_p, C.c_int, C.c_int]),
    "dds_comm_callbacks": (C.c_void_p, [C.c_int, C.c_int, ALLGATHER_FN, BARRIER_FN, C.c_void_p]),
    "dds_comm_rank": (C.c_int, [C.c_void_p]),
    "dds_comm_size": (C.c_int, [C.c_void_p]),
    "dds_comm_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dds_comm_barrier": (C.c_int, [C.c_void_p]),
    "dds_comm_free": (None, [C.c_void_p]),
    "dds_sortedsearch": (C.c_int, [I64P, C.c_int, C.c_int64]),
    "dds_locate": (C.c_int, [I64P, C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_int), I64P]),
    "dds_exchange_lenlist": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, I64P]),
    "dds_create": (C.c_void_p, [C.c_void_p, C.c_int, C.c_int]),
    "dds_destroy": (None, [C.c_void_p]),
    "dds_rank": (C.c_int, [C.c_void_p]),
    "dds_size": (C.c_int, [C.c_void_p]),
    "dds_add": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int]),
    "dds_init": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, C.c_int, C.c_int]),
    "dds_add_placed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]),
    "dds_init_placed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int]),
    "dds_query_placement": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]),
    "dds_update": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int]),
    "dds_update_async": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                   C.c_void_p]),
    "dds_get": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int]),
    "dds_get_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                C.c_void_p, C.c_int64, C.c_void_p, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_get_samples_multi": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.c_void_p, C.c_int64,
                                        C.POINTER(C.c_void_p), I64P, C.POINTER(C.c_void_p), C.c_uint, C.c_void_p, I64P,
                                        I64P]),
    "dds_get_batch_convert": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                        C.c_void_p, C.c_int64, C.c_void_p, C.c_uint, C.c_void_p, C.POINTER(Convert),
                                        I64P, I64P]),
    "dds_get_samples_convert": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_uint, C.c_void_p, C.POINTER(Convert), I64P, I64P]),
    "dds_get_samples_multi_convert": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.c_void_p, C.c_int64,
                                                C.POINTER(C.c_void_p), I64P, C.POINTER(C.c_void_p), C.c_uint,
                                                C.c_void_p, C.POINTER(Convert), I64P, I64P]),
    "dds_get_batch_padded": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                       C.POINTER(Convert), C.POINTER(Pad), C.c_void_p, C.c_int64, C.c_uint, C.c_void_p,
                                       I64P, I64P]),
    "dds_get_samples_padded": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(Convert),
                                         C.POINTER(Pad), C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_put_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_put_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                  C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_accumulate_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                       C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_accumulate_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                         C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_accumulate_op_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                          C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_accumulate_op_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                            C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_get_accumulate_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p,
                                           I64P, I64P]),
    "dds_get_accumulate_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_compare_and_swap_batch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                             C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_uint,
                                             C.c_void_p, I64P, I64P]),
    "dds_compare_and_swap_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_get_batch_pooled": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                       C.POINTER(Pool), C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_get_samples_pooled": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(Pool), C.c_void_p,
                                         C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_accumulate_batch_pooled": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                              C.POINTER(Pool), C.c_double, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p,
                                              I64P, I64P]),
    "dds_accumulate_samples_pooled": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(Pool),
                                                C.c_double, C.c_void_p, C.c_int64, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_batch_wait": (C.c_int, [C.c_void_p, I64P, I64P]),
    "dds_set_sample_index": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int]),
    "dds_set_normalization": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                        C.c_int]),
    "dds_get_samples": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                  C.c_void_p, C.c_uint, C.c_void_p, I64P, I64P]),
    "dds_query": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(VarInfo)]),
    "dds_epoch_begin": (C.c_int, [C.c_void_p]),
    "dds_epoch_end": (C.c_int, [C.c_void_p]),
    "dds_free": (C.c_int, [C.c_void_p]),
    "dds_synth_fill": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64]),
    "dds_push_setup": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64]),
    "dds_get_batch_push": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.POINTER(C.c_void_p),
                                    C.c_void_p]),
    "dds_ingest": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int]),
    "dds_ingest_wait": (C.c_int, [C.c_void_p]),
    "dds_synth_verify": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                  C.c_int64, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]),
    "dds_test_occupy": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p]),
    "dds_kernel_launches": (C.c_ulonglong, []),
    "dds_gather_geometry": (None, [C.POINTER(C.c_int)] * 5),
    "dds_pool_geometry": (None, [C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int), I64P, I64P,
                                 I64P, C.POINTER(C.c_int)]),
    "dds_host_gather_ctas": (C.c_int, []),
}

_lib = None


def lib():
    """The loaded shared library, with signatures applied. Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(ddstore_b200 has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the header and the library ever diverge
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    return lib().dds_last_error().decode()


class DDSError(Exception):
    def __init__(self, code, text):
        super().__init__(text)
        self.code = code


def raise_for(code):
    """Map a status code to the exception type the reference's binding surfaces.

    Codes 1-4 are std::invalid_argument in the reference (ValueError through Cython's `except +`,
    src/pyddstore.pyx:44-50); 5-6 are std::logic_error (ddstore.cxx:58,72)."""
    if code == DDS_OK:
        return
    text = last_error() or lib().dds_strerror(code).decode()
    if code in (ERR_DTYPE, ERR_START, ERR_COUNT, ERR_DISP, ERR_ARG, ERR_CAPACITY):
        raise ValueError(text)
    if code in (ERR_UNKNOWN_VAR,):
        raise KeyError(text)
    raise RuntimeError(text)
