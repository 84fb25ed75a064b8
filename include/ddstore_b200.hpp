// include/ddstore_b200.hpp -- `class DDStore` with the reference's public shape
// (/root/reference/include/ddstore.hpp:26-258), implemented as a thin header-only wrapper over the C-ABI in
// ddstore_b200.h. A C++ caller of the reference switches by including this header, linking
// libddstore_b200.so, and passing a dds_comm_t* where it used to pass an MPI_Comm (INTEGRATION.md).
//
// Same member names, argument order and meaning; the same exception types and texts:
//   std::invalid_argument("Invalid data type" | "Invalid start on target" | "Invalid count on target" |
//                         "Invalid disp")                      ddstore.hpp:82,153,190,203,211,214
//   std::logic_error("Fence already activated" | "Fence is not activated")   ddstore.cxx:58,72
// Everything the reference leaves undefined throws with the C-ABI's message instead: std::out_of_range for an
// unknown variable (the reference default-inserts one, UB), std::runtime_error otherwise (no device, CUDA, comm).
#ifndef DDSTORE_B200_HPP
#define DDSTORE_B200_HPP

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "ddstore_b200.h"

struct VarInfo { // ddstore.hpp:10-22 (window/base/fabric_state replaced by what exists here)
    std::string name;
    int itemsize;
    int disp;
    std::vector<long> lenlist;
    bool active;
    bool fence_active;
    void *base; // device pointer of the local shard
};
typedef struct VarInfo VarInfo_t;

inline int sortedsearch(std::vector<long> &vec, long num) { // src/ddstore.cxx:5-17
    std::vector<int64_t> v(vec.begin(), vec.end());
    return dds_sortedsearch(v.data(), (int)v.size(), (int64_t)num);
}

class DDStore {
  public:
    // DDStore() -- MPI_COMM_SELF, ddstore.cxx:19-24
    DDStore() : own_comm_(dds_comm_self()), comm_(own_comm_), store_(nullptr) { open(0, -1); }
    // DDStore(MPI_Comm comm), ddstore.cxx:26-31
    explicit DDStore(dds_comm_t *comm, int device = -1) : own_comm_(nullptr), comm_(comm), store_(nullptr) {
        open(0, device);
    }
    // DDStore(int method, MPI_Comm comm), ddstore.cxx:33-39
    DDStore(int method, dds_comm_t *comm, int device = -1) : own_comm_(nullptr), comm_(comm), store_(nullptr) {
        open(method, device);
    }
    ~DDStore() { // ddstore.cxx:41-44 (local teardown; the collective one is free())
        if (store_) dds_destroy(store_);
        if (own_comm_) dds_comm_free(own_comm_);
    }
    DDStore(const DDStore &) = delete;
    DDStore &operator=(const DDStore &) = delete;

    void query(std::string name, VarInfo_t &varinfo) { // ddstore.cxx:46-49
        dds_varinfo_t vi;
        check(dds_query(store_, name.c_str(), &vi));
        varinfo.name = name;
        varinfo.itemsize = vi.itemsize;
        varinfo.disp = vi.disp;
        varinfo.lenlist.assign(vi.lenlist, vi.lenlist + vi.nranks);
        varinfo.active = true;
        varinfo.fence_active = vi.fence_active != 0;
        varinfo.base = vi.local_base;
    }
    void epoch_begin() { check(dds_epoch_begin(store_)); } // ddstore.cxx:51-63
    void epoch_end() { check(dds_epoch_end(store_)); }     // ddstore.cxx:65-77
    void free() { check(dds_free(store_)); }               // ddstore.cxx:79-96

    // (placement: DDS_PLACE_HBM, the reference's behaviour, or DDS_PLACE_HOST -- see include/ddstore_b200.h)
    template <typename T>
    void add(std::string name, T *buffer, long nrows, int disp, int placement = DDS_PLACE_HBM) { // ddstore.hpp:39-108
        check(dds_add_placed(store_, name.c_str(), buffer, nrows, disp, (int)sizeof(T), 0, placement));
    }
    void init(std::string name, long nrows, int disp, int itemsize, int placement = DDS_PLACE_HBM) { // ddstore.hpp:110-179
        check(dds_init_placed(store_, name.c_str(), nrows, disp, itemsize, placement));
    }
    int placement(std::string name) {
        int p = DDS_PLACE_HBM;
        check(dds_query_placement(store_, name.c_str(), &p));
        return p;
    }
    template <typename T>
    void update(std::string name, T *buffer, long nrows, long offset = 0) { // ddstore.hpp:181-195
        check(dds_update(store_, name.c_str(), buffer, nrows, offset, (int)sizeof(T), 0));
    }
    template <typename T>
    void get(std::string name, long start, long count, T *buffer) { // ddstore.hpp:197-248
        check(dds_get(store_, name.c_str(), start, count, (int)sizeof(T), buffer, 0));
    }

    // ---- beyond the reference: the batched get() (one kernel launch for the whole batch) -----------------
    // Packs request i = (starts[i], counts[i]) at byte offset sum_{j<i} counts[j]*disp*sizeof(T) of dst.
    // counts == nullptr: every request fetches fixed_count rows. Returns the packed bytes.
    template <typename T>
    long get_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq, T *dst,
                   long dst_capacity_bytes, long *dst_offsets = nullptr, bool on_device = false,
                   void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        unsigned flags = on_device ? (DDS_IDX_ON_DEVICE | DDS_DST_ON_DEVICE) : 0u;
        check(dds_get_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count, nreq,
                            (int)sizeof(T), dst, dst_capacity_bytes, (int64_t *)dst_offsets, flags, cuda_stream, &total,
                            &bad));
        return (long)total;
    }
    // The same requests delivered padded (dds_get_batch_padded): request i fills the max_rows * disp * sizeof(T) bytes of
    // slot i of dst with its first min(counts[i], max_rows) rows, then pad elements. dst (and lengths, nullable: the
    // delivered row counts) are device memory. Returns the padded bytes, nreq * slot.
    template <typename T>
    long get_batch_padded(std::string name, const long *starts, const long *counts, long nreq, long max_rows, T pad, T *dst,
                          long dst_capacity_bytes, long *lengths = nullptr, bool idx_on_device = true,
                          void *cuda_stream = nullptr) {
        static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "element of 1, 2, 4 or 8 bytes");
        uint64_t bits = 0;
        memcpy(&bits, &pad, sizeof(T));
        return get_batch_padded_convert(name, starts, counts, nreq, (int)sizeof(T), DDS_CVT_NONE, nullptr, max_rows, bits,
                                        dst, dst_capacity_bytes, lengths, idx_on_device, cuda_stream);
    }
    // The general form: `itemsize` is the variable's, `code` a DDS_CVT_* code (DDS_CVT_NONE: raw rows; `lut` as for
    // get_batch_convert), pad_bits one OUTPUT element's bits in its low bytes.
    long get_batch_padded_convert(std::string name, const long *starts, const long *counts, long nreq, int itemsize, int code,
                                  const void *lut, long max_rows, uint64_t pad_bits, void *dst, long dst_capacity_bytes,
                                  long *lengths = nullptr, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        dds_pad_t p;
        p.max_rows = max_rows;
        p.pad_bits = pad_bits;
        p.lengths = (int64_t *)lengths;
        const dds_convert_t cvt = {code, lut};
        const unsigned flags = DDS_DST_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_batch_padded(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, nreq, itemsize,
                                   code == DDS_CVT_NONE ? nullptr : &cvt, &p, dst, dst_capacity_bytes, flags, cuda_stream,
                                   &total, &bad));
        return (long)total;
    }
    // The per-channel normalisation of variable `name` for the DDS_CVT_NORM_* codes (dds_set_normalization): nchan
    // means and standard deviations, element e of a row in channel (e / inner) % nchan. nchan = 0 removes it.
    void set_normalization(std::string name, const float *mean, const float *std, long nchan, long inner = 1,
                           bool tables_on_device = false) {
        check(dds_set_normalization(store_, name.c_str(), mean, std, nchan, inner, tables_on_device ? 1 : 0));
    }
    // The same batch delivered converted (dds_get_batch_convert): `code` is a DDS_CVT_* code, `lut` a host table of 256
    // entries for the LUT codes (copied by the call). dst / dst_offsets are device memory; the capacity, the offsets and
    // the result are in OUTPUT bytes. idx_on_device: starts / counts are device pointers.
    long get_batch_convert(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                           void *dst, long dst_capacity_bytes, int code, const void *lut = nullptr,
                           long *dst_offsets = nullptr, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const dds_convert_t cvt = {code, lut};
        const unsigned flags = DDS_DST_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_batch_convert(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count,
                                    nreq, dst, dst_capacity_bytes, (int64_t *)dst_offsets, flags, cuda_stream, &cvt,
                                    &total, &bad));
        return (long)total;
    }
    // Batched put (dds_put_batch): request i writes global rows [starts[i], starts[i] + counts[i]) (counts == nullptr:
    // fixed_count rows) into the owner's shard, from src (device memory), which holds the requests' rows back to back in
    // request order -- an invalid request keeps its rows' bytes in that layout. Every valid request is written; the
    // first invalid one throws like get_batch. Other ranks see the rows after the next epoch fence. Returns the layout's
    // bytes. idx_on_device: starts / counts are device pointers.
    template <typename T>
    long put_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq, const T *src,
                   long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_put_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count, nreq,
                            (int)sizeof(T), src, src_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    // The same by sample id (dds_put_samples): request i = the rows of sample sample_ids[i] in the sample index.
    template <typename T>
    long put_samples(std::string name, const long *sample_ids, long nreq, const T *src, long src_bytes,
                     bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_put_samples(store_, name.c_str(), (const int64_t *)sample_ids, nreq, (int)sizeof(T), src, src_bytes, flags,
                              cuda_stream, &total, &bad));
        return (long)total;
    }
    // Batched accumulate (dds_accumulate_batch): put_batch's requests and layout, each element of the rows becoming
    // shard + src, atomically across requests, batches and ranks. T = float, double, int32_t or int64_t; the overload
    // with an explicit DDS_ACC_* code takes any element type (DDS_ACC_F16 / DDS_ACC_BF16 for 2-byte floats).
    long accumulate_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                          int dtype, const void *src, long src_bytes, bool idx_on_device = true,
                          void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count,
                                   nreq, dtype, src, src_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long accumulate_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                          const T *src, long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        return accumulate_batch(name, starts, counts, fixed_count, nreq, acc_type<T>(), src, src_bytes, idx_on_device,
                                cuda_stream);
    }
    // The same by sample id (dds_accumulate_samples).
    long accumulate_samples(std::string name, const long *sample_ids, long nreq, int dtype, const void *src,
                            long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_samples(store_, name.c_str(), (const int64_t *)sample_ids, nreq, dtype, src, src_bytes,
                                     flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long accumulate_samples(std::string name, const long *sample_ids, long nreq, const T *src, long src_bytes,
                            bool idx_on_device = true, void *cuda_stream = nullptr) {
        return accumulate_samples(name, sample_ids, nreq, acc_type<T>(), src, src_bytes, idx_on_device, cuda_stream);
    }
    // Pooled batch (dds_get_batch_pooled): bag k = requests [bags[k], bags[k+1]) (bags NULL: one bag per request) folded
    // into row k of dst by `mode` (DDS_POOL_*) in `dtype` (DDS_ACC_F32, F64, F16 or BF16); weights nullable, one per
    // request, DDS_POOL_SUM only. dst is device memory; bags and weights live where the indices do. Returns nbags * R.
    long get_batch_pooled(std::string name, const long *starts, const long *counts, long fixed_count, long nreq, int mode,
                          int dtype, const long *bags, long nbags, const void *weights, void *dst, long dst_capacity_bytes,
                          bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        dds_pool_t p{mode, dtype, (const int64_t *)bags, nbags, weights};
        const unsigned flags = DDS_DST_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_batch_pooled(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count, nreq,
                                   &p, dst, dst_capacity_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    // The same by sample id (dds_get_samples_pooled).
    long get_samples_pooled(std::string name, const long *sample_ids, long nreq, int mode, int dtype, const long *bags,
                            long nbags, const void *weights, void *dst, long dst_capacity_bytes, bool idx_on_device = true,
                            void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        dds_pool_t p{mode, dtype, (const int64_t *)bags, nbags, weights};
        const unsigned flags = DDS_DST_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_samples_pooled(store_, name.c_str(), (const int64_t *)sample_ids, nreq, &p, dst, dst_capacity_bytes,
                                     flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    // Pooled accumulate (dds_accumulate_batch_pooled), the adjoint of get_batch_pooled: grad row k (nbags rows of R bytes
    // in `dtype`, device memory) times the request's weight, over the bag's rows for DDS_POOL_MEAN, times alpha, added into
    // every row of bag k. mode is DDS_POOL_SUM or DDS_POOL_MEAN. Returns nbags * R.
    long accumulate_batch_pooled(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                                 int mode, int dtype, const long *bags, long nbags, const void *weights, double alpha,
                                 const void *grad, long grad_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        dds_pool_t p{mode, dtype, (const int64_t *)bags, nbags, weights};
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_batch_pooled(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts,
                                          fixed_count, nreq, &p, alpha, grad, grad_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    // The same by sample id (dds_accumulate_samples_pooled).
    long accumulate_samples_pooled(std::string name, const long *sample_ids, long nreq, int mode, int dtype,
                                   const long *bags, long nbags, const void *weights, double alpha, const void *grad,
                                   long grad_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        dds_pool_t p{mode, dtype, (const int64_t *)bags, nbags, weights};
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_samples_pooled(store_, name.c_str(), (const int64_t *)sample_ids, nreq, &p, alpha, grad,
                                            grad_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    // Batched reduction (dds_accumulate_op_batch): accumulate_batch with each element becoming op(shard, src), op one of
    // DDS_OP_SUM, DDS_OP_MAX, DDS_OP_MIN, DDS_OP_BAND, DDS_OP_BOR, DDS_OP_BXOR (the bitwise ops on integer types only).
    long accumulate_op_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq, int op,
                             int dtype, const void *src, long src_bytes, bool idx_on_device = true,
                             void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_op_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts, fixed_count,
                                      nreq, op, dtype, src, src_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long accumulate_op_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq, int op,
                             const T *src, long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        return accumulate_op_batch(name, starts, counts, fixed_count, nreq, op, acc_type<T>(), src, src_bytes,
                                   idx_on_device, cuda_stream);
    }
    // The same by sample id (dds_accumulate_op_samples).
    long accumulate_op_samples(std::string name, const long *sample_ids, long nreq, int op, int dtype, const void *src,
                               long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_accumulate_op_samples(store_, name.c_str(), (const int64_t *)sample_ids, nreq, op, dtype, src, src_bytes,
                                        flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long accumulate_op_samples(std::string name, const long *sample_ids, long nreq, int op, const T *src, long src_bytes,
                               bool idx_on_device = true, void *cuda_stream = nullptr) {
        return accumulate_op_samples(name, sample_ids, nreq, op, acc_type<T>(), src, src_bytes, idx_on_device,
                                     cuda_stream);
    }
    // Batched fetch-op (dds_get_accumulate_batch): accumulate_batch's requests and layout, each element of the rows
    // added to (op = DDS_OP_SUM) or swapped with (DDS_OP_REPLACE) src atomically, its previous value written to `result`
    // (device memory of at least src_bytes, the layout of src; it may be src). T and the explicit-code overload as for
    // accumulate_batch.
    long get_accumulate_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                              int op, int dtype, const void *src, void *result, long src_bytes, bool idx_on_device = true,
                              void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_accumulate_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts,
                                       fixed_count, nreq, op, dtype, src, result, src_bytes, flags, cuda_stream, &total,
                                       &bad));
        return (long)total;
    }
    template <typename T>
    long get_accumulate_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                              int op, const T *src, T *result, long src_bytes, bool idx_on_device = true,
                              void *cuda_stream = nullptr) {
        return get_accumulate_batch(name, starts, counts, fixed_count, nreq, op, acc_type<T>(), src, result, src_bytes,
                                    idx_on_device, cuda_stream);
    }
    // The same by sample id (dds_get_accumulate_samples).
    long get_accumulate_samples(std::string name, const long *sample_ids, long nreq, int op, int dtype, const void *src,
                                void *result, long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_get_accumulate_samples(store_, name.c_str(), (const int64_t *)sample_ids, nreq, op, dtype, src, result,
                                         src_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long get_accumulate_samples(std::string name, const long *sample_ids, long nreq, int op, const T *src, T *result,
                                long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        return get_accumulate_samples(name, sample_ids, nreq, op, acc_type<T>(), src, result, src_bytes, idx_on_device,
                                      cuda_stream);
    }
    // Batched compare-and-swap (dds_compare_and_swap_batch): accumulate_batch's requests and layout, each element of the
    // rows replaced by src's where it equals compare's bit for bit, atomically, its previous value written to `result`
    // either way (compare and result: device memory of at least src_bytes, the layout of src; result may be src or
    // compare). Elements are itemsize bytes (1, 2, 4 or 8, the variable's); T gives it as sizeof(T).
    long compare_and_swap_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                                int itemsize, const void *src, const void *compare, void *result, long src_bytes,
                                bool idx_on_device = true, void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_compare_and_swap_batch(store_, name.c_str(), (const int64_t *)starts, (const int64_t *)counts,
                                         fixed_count, nreq, itemsize, src, compare, result, src_bytes, flags, cuda_stream,
                                         &total, &bad));
        return (long)total;
    }
    template <typename T>
    long compare_and_swap_batch(std::string name, const long *starts, const long *counts, long fixed_count, long nreq,
                                const T *src, const T *compare, T *result, long src_bytes, bool idx_on_device = true,
                                void *cuda_stream = nullptr) {
        return compare_and_swap_batch(name, starts, counts, fixed_count, nreq, (int)sizeof(T), src, compare, result,
                                      src_bytes, idx_on_device, cuda_stream);
    }
    // The same by sample id (dds_compare_and_swap_samples).
    long compare_and_swap_samples(std::string name, const long *sample_ids, long nreq, int itemsize, const void *src,
                                  const void *compare, void *result, long src_bytes, bool idx_on_device = true,
                                  void *cuda_stream = nullptr) {
        int64_t total = 0, bad = -1;
        const unsigned flags = DDS_SRC_ON_DEVICE | (idx_on_device ? DDS_IDX_ON_DEVICE : 0u);
        check(dds_compare_and_swap_samples(store_, name.c_str(), (const int64_t *)sample_ids, nreq, itemsize, src, compare,
                                           result, src_bytes, flags, cuda_stream, &total, &bad));
        return (long)total;
    }
    template <typename T>
    long compare_and_swap_samples(std::string name, const long *sample_ids, long nreq, const T *src, const T *compare,
                                  T *result, long src_bytes, bool idx_on_device = true, void *cuda_stream = nullptr) {
        return compare_and_swap_samples(name, sample_ids, nreq, (int)sizeof(T), src, compare, result, src_bytes,
                                        idx_on_device, cuda_stream);
    }
    // the DDS_ACC_* code of an element type
    template <typename T>
    static constexpr int acc_type() {
        static_assert(std::is_same<T, float>::value || std::is_same<T, double>::value ||
                          std::is_same<T, int32_t>::value || std::is_same<T, int64_t>::value,
                      "accumulate_batch<T>: T is float, double, int32_t or int64_t (2-byte floats: pass DDS_ACC_F16 / "
                      "DDS_ACC_BF16)");
        return std::is_same<T, float>::value ? DDS_ACC_F32 : std::is_same<T, double>::value ? DDS_ACC_F64
               : std::is_same<T, int32_t>::value ? DDS_ACC_I32 : DDS_ACC_I64;
    }
    // device-pointer variants of add/get for callers that already hold the data in HBM
    template <typename T>
    void add_device(std::string name, const T *dev_buffer, long nrows, int disp, int placement = DDS_PLACE_HBM) {
        check(dds_add_placed(store_, name.c_str(), dev_buffer, nrows, disp, (int)sizeof(T), 1, placement));
    }
    template <typename T>
    void get_device(std::string name, long start, long count, T *dev_buffer) {
        check(dds_get(store_, name.c_str(), start, count, (int)sizeof(T), dev_buffer, 1));
    }

    int rank() const { return dds_rank(store_); }
    int size() const { return dds_size(store_); }
    dds_store_t *handle() { return store_; }

  private:
    void open(int method, int device) {
        store_ = dds_create(comm_, device, method);
        if (!store_) throw std::runtime_error(dds_last_error());
    }
    static void check(int rc) {
        switch (rc) {
        case DDS_OK: return;
        case DDS_ERR_DTYPE:
        case DDS_ERR_START:
        case DDS_ERR_COUNT:
        case DDS_ERR_DISP: throw std::invalid_argument(dds_last_error());
        case DDS_ERR_FENCE_ACTIVE:
        case DDS_ERR_FENCE_INACTIVE: throw std::logic_error(dds_last_error());
        case DDS_ERR_UNKNOWN_VAR: throw std::out_of_range(dds_last_error());
        default: throw std::runtime_error(dds_last_error());
        }
    }
    dds_comm_t *own_comm_;
    dds_comm_t *comm_;
    dds_store_t *store_;
};

#endif
