/* include/ddstore_b200.h -- the drop-in boundary: a C-ABI over an H100-native distributed sample
 * store with the behaviour of ORNL/DDStore's `DDStore` class.
 *
 * The reference's FFI for this path is Cython binding the C++ class (src/pyddstore.pyx:34-50 ->
 * include/ddstore.hpp:26-258). Every entry point below replaces one member of that class (cited),
 * flattened to `extern "C"`, plain pointers and sizes, int status codes and a thread-local message.
 * include/ddstore_b200.hpp wraps this header back into a C++ class of the reference's shape;
 * ddstore_b200/pyddstore.pyx wraps that class with the reference's Python surface.
 *
 * Data plane: each rank's shard lives in its GPU's HBM (cudaMalloc); peers map it through CUDA IPC
 * (the analogue of MPI_Win_create, ddstore.hpp:56-61); get() is a batched-gather sm_90a kernel
 * reading the owner's HBM directly (local or over NVLink/NVSwitch). There is NO CPU data path:
 * without a CUDA device every data-plane call fails with DDS_ERR_NO_DEVICE.
 */
#ifndef DDSTORE_B200_H
#define DDSTORE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDS_VERSION 111 /* 110: converting batches (dds_get_batch_convert & co.); 111: normalising conversions.
                           The padded batches (dds_get_batch_padded, dds_get_samples_padded) add entries only: callers
                           that built against 111 are unaffected, and a caller finds them by symbol. So do the batched
                           puts (dds_put_batch, dds_put_samples, DDS_SRC_ON_DEVICE), the batched accumulates
                           (dds_accumulate_batch, dds_accumulate_samples, DDS_ACC_*), the batched fetch-ops
                           (dds_get_accumulate_batch, dds_get_accumulate_samples, DDS_OP_*), the batched
                           compare-and-swaps (dds_compare_and_swap_batch, dds_compare_and_swap_samples), the batched
                           reductions (dds_accumulate_op_batch, dds_accumulate_op_samples, DDS_OP_MAX & co.), the
                           placed variables (dds_add_placed, dds_init_placed, dds_query_placement, DDS_PLACE_*) and the
                           pooled batches (dds_get_batch_pooled, dds_get_samples_pooled, DDS_POOL_*) and the pooled
                           accumulates (dds_accumulate_batch_pooled, dds_accumulate_samples_pooled). */

/* ---- status codes. 1-6 carry the reference's exception texts verbatim ------------------------- */
#define DDS_OK 0
#define DDS_ERR_DTYPE 1          /* "Invalid data type"        std::invalid_argument, ddstore.hpp:189-190,202-203 */
#define DDS_ERR_START 2          /* "Invalid start on target"  std::invalid_argument, ddstore.hpp:210-211 */
#define DDS_ERR_COUNT 3          /* "Invalid count on target"  std::invalid_argument, ddstore.hpp:213-214 */
#define DDS_ERR_DISP 4           /* "Invalid disp"             std::invalid_argument, ddstore.hpp:81-82,152-153 */
#define DDS_ERR_FENCE_ACTIVE 5   /* "Fence already activated"  std::logic_error, ddstore.cxx:57-58 */
#define DDS_ERR_FENCE_INACTIVE 6 /* "Fence is not activated"   std::logic_error, ddstore.cxx:71-72 */
/* the rest have no counterpart in the reference (it has UB / exit(1) / a hang there) */
#define DDS_ERR_UNKNOWN_VAR 7    /* reference: map operator[] default-inserts, UB (ddstore.hpp:200) */
#define DDS_ERR_EXISTS 8         /* reference: map::insert silently keeps the old entry (ddstore.hpp:107) */
#define DDS_ERR_CUDA 9
#define DDS_ERR_COMM 10
#define DDS_ERR_ARG 11
#define DDS_ERR_CAPACITY 12      /* packed batch does not fit the destination buffer */
#define DDS_ERR_NO_DEVICE 13     /* no usable CUDA device: there is no CPU fallback */
#define DDS_ERR_WATCHDOG 14

/* Text for the calling thread's most recent failure ("" if none). For codes 1-6 this is exactly the
 * reference's exception text. */
const char *dds_last_error(void);
/* The fixed text of a status code (the reference's what() for 1-6). */
const char *dds_strerror(int code);

/* ---- communicator: replaces MPI_Comm in DDStore(int method, MPI_Comm comm), ddstore.hpp:29-31 ----
 * Only two collectives are ever needed (bootstrap all-gather of a few hundred bytes, and a barrier for
 * the epoch fences), so a communicator is {rank, size, allgather, barrier}. */
typedef struct dds_comm dds_comm_t;
typedef int (*dds_allgather_fn)(void *ctx, const void *send, void *recv, size_t bytes_per_rank);
typedef int (*dds_barrier_fn)(void *ctx);

dds_comm_t *dds_comm_self(void); /* MPI_COMM_SELF, ddstore.cxx:19-24 */
/* Ranks on ONE box (processes or threads) rendezvous through a POSIX shared-memory segment named after
 * `key` (all ranks pass the same key; unique per job). No MPI, no sockets. */
dds_comm_t *dds_comm_shm(const char *key, int rank, int size);
/* Any other runtime (mpi4py, torch.distributed, ...) through two callbacks. */
dds_comm_t *dds_comm_callbacks(int rank, int size, dds_allgather_fn allgather, dds_barrier_fn barrier, void *ctx);
int dds_comm_rank(const dds_comm_t *c);
int dds_comm_size(const dds_comm_t *c);
int dds_comm_allgather(dds_comm_t *c, const void *send, void *recv, size_t bytes_per_rank);
int dds_comm_barrier(dds_comm_t *c);
void dds_comm_free(dds_comm_t *c);

/* ---- host-side index math (pure functions; what the kernels also compute per request) -------- */
/* int sortedsearch(std::vector<long>&, long), src/ddstore.cxx:5-17 */
int dds_sortedsearch(const int64_t *lenlist, int nranks, int64_t num);
/* ddstore.hpp:205-214: owner, first global row of the owner, DDS_OK / DDS_ERR_START / DDS_ERR_COUNT */
int dds_locate(const int64_t *lenlist, int nranks, int64_t start, int64_t count, int *owner, int64_t *offset);
/* ddstore.hpp:75-89: COLLECTIVE. All-gathers (nrows, disp), checks disp uniformity (DDS_ERR_DISP on the
 * ranks that differ from the maximum), writes the inclusive running sum to lenlist[size]. */
int dds_exchange_lenlist(dds_comm_t *c, int64_t nrows, int disp, int64_t *lenlist);

/* ---- the store: class DDStore, ddstore.hpp:26-258 --------------------------------------------- */
typedef struct dds_store dds_store_t;

typedef struct dds_varinfo { /* VarInfo_t, ddstore.hpp:10-22 (win/base replaced by what a caller can use) */
    int32_t itemsize;
    int32_t disp;
    int32_t nranks;
    int32_t fence_active;
    int64_t local_nrows;
    int64_t total_nrows;
    int64_t lenlist[64]; /* inclusive cumulative rows, first nranks entries valid */
    void *local_base;    /* device pointer of this rank's shard */
} dds_varinfo_t;

/* DDStore(int method, MPI_Comm comm), ddstore.cxx:33-39. `device` = CUDA ordinal for this rank's shard
 * (-1: current device). `method` is accepted for signature compatibility (0 and 1 both select the one
 * NVLink transport; there is no multi-backend dispatch). The store borrows `comm` (caller frees it after
 * dds_destroy). Fails with DDS_ERR_NO_DEVICE when no GPU is usable. */
dds_store_t *dds_create(dds_comm_t *comm, int device, int method);
void dds_destroy(dds_store_t *s); /* ~DDStore, ddstore.cxx:41-44 */
int dds_rank(const dds_store_t *s);
int dds_size(const dds_store_t *s);

/* template<T> void add(string name, T* buffer, long nrows, int disp), ddstore.hpp:39-108. COLLECTIVE.
 * Copies nrows*disp*itemsize bytes from `buffer` (host, or device when buffer_on_device) into a fresh HBM
 * shard, exchanges row counts and IPC handles, maps every peer's shard. */
int dds_add(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int disp, int itemsize,
            int buffer_on_device);
/* void init(string name, long nrows, int disp, int itemsize), ddstore.hpp:110-179. COLLECTIVE, zero-filled. */
int dds_init(dds_store_t *s, const char *name, int64_t nrows, int disp, int itemsize);

/* ---- placement: where a variable's shards live, chosen when it is created -----------------------------------------
 * DDS_PLACE_HBM (dds_add / dds_init): each shard in its GPU's HBM. DDS_PLACE_HOST: each shard in pinned host memory that
 * every rank of the box maps (the reference's host-RAM shards), so a dataset may be larger than the HBM a model leaves
 * free. The gathers still run on the GPU and read a HOST shard over PCIe, into HBM or a host buffer as usual.
 * On a HOST variable these work exactly as on an HBM one, byte for byte, errors included: dds_get, dds_get_batch,
 * dds_get_samples, the converting, normalising and padded entries, dds_get_samples_multi(_convert) when every variable
 * of the batch is HOST, dds_update(_async), dds_ingest, dds_synth_fill and dds_synth_verify. DDS_OVERLAP is ignored for
 * HOST batches (a HOST batch ends an overlap run, like a put).
 * Refused with DDS_ERR_ARG, nothing enqueued, right after the unknown-variable check: every batched write (put,
 * accumulate, accumulate_op, get_accumulate, compare_and_swap, batch and samples forms), dds_get_batch_push, and a
 * multi-array batch that mixes placements. Device atomics on mapped host memory are not atomic across GPUs over PCIe,
 * and one rule is simpler than two: a HOST variable is written only by its owner's update / ingest. Per-sample state
 * that training writes back belongs in HBM variables.
 * dds_add_placed / dds_init_placed are dds_add / dds_init with a placement (COLLECTIVE): an unknown placement is
 * DDS_ERR_ARG, and so is a placement the ranks disagree on (on every rank; nothing is registered). */
#define DDS_PLACE_HBM 0
#define DDS_PLACE_HOST 1
int dds_add_placed(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int disp, int itemsize,
                   int buffer_on_device, int placement);
int dds_init_placed(dds_store_t *s, const char *name, int64_t nrows, int disp, int itemsize, int placement);
int dds_query_placement(dds_store_t *s, const char *name, int *placement);
/* template<T> void update(string name, T* buffer, long nrows, long offset), ddstore.hpp:181-195. Local copy
 * into rows [offset, offset+nrows) of this rank's shard. (The reference does not bounds-check; this does:
 * DDS_ERR_ARG.) */
int dds_update(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int64_t offset, int itemsize,
               int buffer_on_device);
/* dds_update without the trailing synchronise, on `cuda_stream` (NULL: the store's stream): for streaming ingest of a
 * pre-init'd shard from pinned chunks (the copy of chunk k overlaps the host producing chunk k+1). */
int dds_update_async(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int64_t offset, int itemsize,
                     int buffer_on_device, void *cuda_stream);
/* dds_update for a chunk of PAGEABLE host rows, pipelined inside the library: a few worker threads copy slices of the
 * chunk into pinned staging buffers while the copy engine moves the previous buffer into the shard (streaming ingest of
 * a pre-init'd shard, the reference's init + update-in-chunks pattern). Returns once the source has been consumed; the
 * tail of the copies completes at the next epoch fence, dds_ingest_wait or dds_free. DDS_INGEST_THREADS (default 6). */
int dds_ingest(dds_store_t *s, const char *name, const void *host_rows, int64_t nrows, int64_t offset, int itemsize);
int dds_ingest_wait(dds_store_t *s);
/* template<T> void get(string name, long start, long count, T* buffer), ddstore.hpp:197-248. Fetches
 * count rows starting at GLOBAL row `start` (must lie within one owner) into `buffer` (host, or device).
 * Results up to 64 KiB (host) / 1 MiB (device) take a 1-CTA kernel whose completion the host spins on in mapped
 * pinned memory: one launch, no stream synchronize (the legacy one-get-per-sample loader loop). */
int dds_get(dds_store_t *s, const char *name, int64_t start, int64_t count, int itemsize, void *buffer,
            int buffer_on_device);

/* The batched form of get(): nreq requests (starts[i], counts[i]) on one variable, results packed back to
 * back in request order into dst -- byte for byte what nreq successive get() calls would have written
 * (the loader loop, examples/vae/distdataset.py:79-89). counts == NULL means every request fetches
 * `fixed_count` rows. dst_offsets (nullable) receives nreq+1 byte offsets (exclusive scan).
 * On the first (lowest-index) invalid request returns its DDS_ERR_START/COUNT and its index in
 * *bad_index; requests before it are delivered, like the serial loop that stops at the exception. A host dst
 * receives exactly those bytes and nothing else; a device dst may also receive later VALID requests, each at the
 * offset the batch packs it to (an invalid request packs as zero bytes; with a fixed count it keeps its slot),
 * never anything else. A negative count, and a count for which start + count overflows, are "Invalid count on
 * target". If the packed batch does not fit dst_capacity, nothing is written: DDS_ERR_CAPACITY (*bad_index = -1),
 * unless a request is invalid -- then that request's error wins, as in the loop that raises before it runs out of
 * room. */
/* cuda_stream: a cudaStream_t to enqueue on; NULL selects the store's own stream (pass cudaStreamLegacy,
 * (void*)0x1, for CUDA's legacy default stream). */
#define DDS_IDX_ON_DEVICE 1u /* starts / counts are device pointers */
#define DDS_DST_ON_DEVICE 2u /* dst / dst_offsets are device pointers */
#define DDS_NO_SYNC 4u       /* needs both flags above: enqueue on cuda_stream and return; dds_batch_wait() reports,
                              * and only it: see dds_batch_wait for how a queue of such batches ends */
#define DDS_OVERLAP 8u       /* with DDS_NO_SYNC: this batch is INDEPENDENT of the ONE batch queued just before it on the
                              * same stream (different destination / offsets buffers; indices not produced by it), so the
                              * two may overlap: the head of this one fills the SMs the tail of the previous one vacates
                              * (double-buffered prefetch). The contract is enforced by the kernel, not assumed: batch q
                              * writes nothing before batch q-2 has retired (so reusing the buffers of batch q-2 is safe
                              * whatever else shares the GPU), and batches retire in order (whatever follows batch q on
                              * the stream sees all earlier ones complete). Honoured for fixed-count batches and for
                              * variable-count batches of <= 8192 requests into < 4 GiB; ignored otherwise. */
int dds_get_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                  int64_t fixed_count, int64_t nreq, int itemsize, void *dst, int64_t dst_capacity,
                  int64_t *dst_offsets, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                  int64_t *bad_index);

/* Per-sample index of a variable (variable-length / multi-array datasets): sample i owns global rows
 * [row_start[i], row_start[i] + row_count[i]) -- the (start, count) pairs a HydraGNN-style loader passes to
 * get(name, arr, start) with count = arr.shape[0] (src/pyddstore.pyx:84-87). The tables are copied to the device
 * once; dds_get_samples then needs only the sample ids: the id -> (start, count) lookup is fused into the launch. */
int dds_set_sample_index(dds_store_t *s, const char *name, const int64_t *row_start, const int64_t *row_count,
                         int64_t nsamples, int tables_on_device);
/* dds_get_batch with request i = the rows of sample sample_ids[i]. Same flags, packing, offsets and error rules. */
int dds_get_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize, void *dst,
                    int64_t dst_capacity, int64_t *dst_offsets, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                    int64_t *bad_index);

/* Multi-array samples (BASELINE config 4: node_feat + edge_index per graph): the rows of the SAME nreq samples in
 * nvars (1..4) variables that each have a sample index, in ONE launch. dsts[v] (device) receives variable v's packed
 * rows, dst_offsets[v] (nullable, device, nreq+1 entries) its per-sample byte offsets, total_bytes[v] its packed size.
 * Needs DDS_DST_ON_DEVICE. The reported request is the first invalid one in variable order, then sample order: the
 * lowest variable with an invalid request, and in it the lowest one (the loop over variables of a loop over samples);
 * *bad_index is its position in sample_ids. Variables before it are delivered whole, that variable up to the sample. */
int dds_get_samples_multi(dds_store_t *s, int nvars, const char *const *names, const int64_t *sample_ids, int64_t nreq,
                          void *const *dsts, const int64_t *dst_capacities, int64_t *const *dst_offsets, unsigned flags,
                          void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);

/* ---- converting batches: rows delivered in the training dtype, converted inside the gather ----------------------
 * The store only knows a variable's itemsize; the code names the source type. Element rules:
 *   DDS_CVT_F32_BF16  4 -> 2 bytes  round to nearest even (cvt.rn.bf16.f32)
 *   DDS_CVT_F32_F16   4 -> 2 bytes  round to nearest even, overflow to +-inf, f16 subnormals kept (cvt.rn.f16.f32)
 *   DDS_CVT_F64_F32   8 -> 4 bytes  cvt.rn.f32.f64
 *   DDS_CVT_U8_LUT16  1 -> 2 bytes  out = lut[in], 256 two-byte entries (bf16 or f16 bits)
 *   DDS_CVT_U8_LUT32  1 -> 4 bytes  out = lut[in], 256 four-byte entries (f32 bits)
 * NaN inputs of the float rules give the quiet NaN of cvt.rn, which is what torch's CUDA .to(dtype) gives. A table makes
 * a uint8 normalisation bit-exact with whatever expression built it. `lut` is a host pointer, copied when the call is
 * made (the caller may free it on return; every queued batch keeps its own tables).
 * Request i is located, validated and ordered exactly as in the raw entry, then written converted: it sits at output
 * byte sum_{j<i} count_j * disp * out_itemsize. The capacity, dst_offsets and the reported totals are all in OUTPUT
 * bytes, and the error rules are those of dds_get_batch with sizes in output bytes. The entries take the raw entries'
 * arguments and flags minus `itemsize`, and require DDS_DST_ON_DEVICE (host indices are fine). Argument errors: the
 * variable's itemsize is not the code's source itemsize -> DDS_ERR_DTYPE; an unknown code, a LUT code without a table,
 * a host destination, or dst / dst_offsets not aligned to the output itemsize / 8 bytes -> DDS_ERR_ARG. */
#define DDS_CVT_NONE 0 /* raw bytes: valid only for a variable of dds_get_samples_multi_convert */
#define DDS_CVT_F32_BF16 1
#define DDS_CVT_F32_F16 2
#define DDS_CVT_F64_F32 3
#define DDS_CVT_U8_LUT16 4
#define DDS_CVT_U8_LUT32 5
/* Normalising conversions: every element x of a delivered row becomes
 *   y   = __fdiv_rn(__fsub_rn(decode(x), mean[ch]), std[ch])   (f32, two IEEE roundings, no contraction)
 *   out = encode(y)                                              (f32 as is, cvt.rn.bf16.f32 or cvt.rn.f16.f32)
 * with mean / std / the channel rule registered for the variable by dds_set_normalization. decode: f32 as is, f64 by
 * cvt.rn.f32.f64, uint8 through `lut`, 256 FLOAT32 entries (required; {0, 1, ..., 255} is the plain value, {k / 255.f}
 * that of ToTensor()). The result is bit-exact with torch's ((x.to(float32) - mean_t) / std_t).to(out_dtype) on CUDA
 * for CUDA float32 tensors mean_t / std_t laid out by the channel rule. Capacity, offsets, totals and every error rule
 * are those of the plain conversions with the same itemsizes, plus DDS_ERR_ARG for a variable without a registered
 * normalisation (checked before the itemsize). They may be mixed with plain and raw variables in dds_get_samples_multi_convert.
 *   code                     source -> output   table */
#define DDS_CVT_NORM_F32_F32 6  /* 4 -> 4 */
#define DDS_CVT_NORM_F32_BF16 7 /* 4 -> 2 */
#define DDS_CVT_NORM_F32_F16 8  /* 4 -> 2 */
#define DDS_CVT_NORM_F64_F32 9  /* 8 -> 4 */
#define DDS_CVT_NORM_U8_F32 10  /* 1 -> 4   256 f32 */
#define DDS_CVT_NORM_U8_BF16 11 /* 1 -> 2   256 f32 */
#define DDS_CVT_NORM_U8_F16 12  /* 1 -> 2   256 f32 */
typedef struct {
    int32_t code;    /* DDS_CVT_* */
    const void *lut; /* host pointer to 256 table entries (LUT and uint8 normalising codes only) */
} dds_convert_t;
/* The per-channel normalisation of a variable, for the DDS_CVT_NORM_* codes: nchan means and standard deviations
 * (float32, host or device pointers), copied into device memory the store owns. Element e in [0, disp) of a row is in
 * channel (e / inner) % nchan: nchan = 1 is one scalar, nchan = disp per feature, (C, 1) channels-last, (C, H*W) CHW.
 * Local (not collective): the normalisation is applied on the requesting rank. nchan = 0 removes it. Like
 * dds_set_sample_index it first completes pending batches and synchronises, so no queued batch reads replaced tables.
 * DDS_ERR_ARG: inner < 1, nchan < 0, nchan * inner not dividing disp, or a null table. */
int dds_set_normalization(dds_store_t *s, const char *name, const float *mean, const float *std, int64_t nchan,
                          int64_t inner, int tables_on_device);
int dds_get_batch_convert(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                          int64_t fixed_count, int64_t nreq, void *dst, int64_t dst_capacity, int64_t *dst_offsets,
                          unsigned flags, void *cuda_stream, const dds_convert_t *cvt, int64_t *total_bytes,
                          int64_t *bad_index);
int dds_get_samples_convert(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, void *dst,
                            int64_t dst_capacity, int64_t *dst_offsets, unsigned flags, void *cuda_stream,
                            const dds_convert_t *cvt, int64_t *total_bytes, int64_t *bad_index);
/* cvts[v]: variable v's conversion; DDS_CVT_NONE delivers that variable's bytes unchanged in the same launch. */
int dds_get_samples_multi_convert(dds_store_t *s, int nvars, const char *const *names, const int64_t *sample_ids,
                                  int64_t nreq, void *const *dsts, const int64_t *dst_capacities,
                                  int64_t *const *dst_offsets, unsigned flags, void *cuda_stream,
                                  const dds_convert_t *cvts, int64_t *total_bytes, int64_t *bad_index);

/* ---- padded batches: variable-length requests delivered as [nreq, max_rows, disp] slots plus lengths --------------
 * Let S = max_rows * disp * out_itemsize (out_itemsize: the variable's itemsize for a raw batch, the code's output
 * itemsize with a conversion). Request i owns bytes [i * S, (i + 1) * S) of dst: its first min(count_i, max_rows) rows,
 * raw or converted / normalised exactly as by the *_convert entries (cvt NULL: raw), then pad_bits, one output element
 * at a time, written verbatim (padding is never converted). lengths[i] (nullable, device) receives the delivered row
 * count; *total_bytes = nreq * S.
 * Requests are validated on their FULL (start, count), by the rules of dds_get_batch: a valid request longer than
 * max_rows is truncated (not an error); an invalid one gets a slot of padding only and length 0, and the first invalid
 * request's code and index are returned as dds_get_batch returns them. Unlike the packed entries, every valid request's
 * slot is delivered even when some are invalid.
 * DDS_ERR_ARG, with nothing enqueued or written: counts == NULL (padding needs counts; dds_get_samples_padded takes them
 * from the sample index), a host destination (DDS_DST_ON_DEVICE is required), dst not aligned to out_itemsize or lengths
 * not aligned to 8, max_rows < 0, nreq * S overflowing, a raw variable whose itemsize is not 1, 2, 4 or 8, and
 * dst_capacity < nreq * S (checked on the host: the padded size does not depend on the requests). DDS_ERR_DTYPE as for
 * the raw and the converting entries. DDS_NO_SYNC and DDS_OVERLAP work as for fixed-count batches (overlap is honoured
 * at every size); a queued padded batch's total is nreq * S. */
typedef struct {
    int64_t max_rows;  /* rows per slot, >= 0 */
    uint64_t pad_bits; /* one OUTPUT element's bits, in the low out_itemsize bytes (e.g. a bf16 -inf, an int32 pad id) */
    int64_t *lengths;  /* device, nullable: nreq delivered row counts */
} dds_pad_t;
int dds_get_batch_padded(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts, int64_t nreq,
                         int itemsize, const dds_convert_t *cvt, const dds_pad_t *pad, void *dst, int64_t dst_capacity,
                         unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);
int dds_get_samples_padded(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                           const dds_convert_t *cvt, const dds_pad_t *pad, void *dst, int64_t dst_capacity, unsigned flags,
                           void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);

/* ---- batched puts: rows written into ANY rank's shard from this GPU (update<T> from any rank / MPI_Put between fences)
 * The dual of dds_get_batch / dds_get_samples. Request i writes global rows [start_i, start_i + count_i) of `name` (count_i
 * = counts[i], or fixed_count when counts == NULL); for dds_put_samples it is sample sample_ids[i]'s (row_start,
 * row_count) from the sample index. The rows are raw, in the variable's dtype.
 * Layout of src: request i's rows are src bytes [o_i, o_i + n_i), where n_i = count_i * disp * itemsize when
 * 0 < count_i <= the variable's total rows and 0 otherwise (0 for a sample id outside the index), and o_i is the
 * exclusive scan of the n_i. Unlike the packed get, an INVALID request keeps its bytes in the layout: the caller built
 * src from its own counts, so the requests after it find their rows where the caller put them. *total_bytes = the layout
 * total sum n_i. src may have any byte alignment.
 * Validation: requests are checked by dds_get_batch's rules, with its codes, texts and documented divergences (a negative
 * count, or one for which start + count overflows, is "Invalid count on target"); a sample id outside the index is
 * DDS_ERR_ARG, "sample id outside the variable's sample index", as in dds_get_samples. An invalid request writes nothing;
 * EVERY valid request is written, as in the padded entries; the first (lowest-index) invalid request's code and index are
 * returned. If the layout total exceeds src_bytes, nothing at all is written: DDS_ERR_CAPACITY (*bad_index = -1), unless
 * a request is invalid -- then that request's error is reported, as in dds_get_batch.
 * Argument errors, DDS_ERR_ARG with nothing enqueued: flags without DDS_SRC_ON_DEVICE (a host src: copy it to the device
 * first), nreq < 0, src_bytes < 0, src == NULL with src_bytes > 0 or with a layout the host knows to be non-empty (fixed
 * count, or host indices; with device indices an empty src is the kernel's DDS_ERR_CAPACITY), DDS_NO_SYNC with host
 * indices, and dds_put_samples on a variable without a sample index. An itemsize other than the variable's is
 * DDS_ERR_DTYPE ("Invalid data type", ddstore.hpp:189-190, as update reports it). nreq = 0 writes nothing and returns
 * DDS_OK with *total_bytes = 0.
 * Flags: DDS_IDX_ON_DEVICE as in the get entries (host indices are staged the same way). DDS_NO_SYNC queues the put on
 * cuda_stream; dds_batch_wait reports it like a queued get, *total_bytes being its layout total. DDS_OVERLAP is ignored:
 * a put is never overlapped with the launch before it or after it. It ends an overlap run, so the next DDS_OVERLAP batch
 * starts a new run, whose first launch waits for the grid before it.
 * Ordering and visibility: later work on the same stream sees the rows; a synchronous put returns after its rows are
 * written; other ranks see them after the next fence (dds_epoch_begin or dds_epoch_end) that both sides have passed.
 * Both fences complete a pending queue that holds a put (dds_epoch_begin leaves a queue of gets alone).
 * Conflicts are undefined, as for conflicting MPI_Puts: two writes to the same bytes in one epoch -- from one batch or
 * from several ranks -- leave each byte equal to that byte of one of the writers; a read of rows that are being put in
 * the same epoch returns undefined bytes; a src that overlaps a shard gives undefined rows. */
#define DDS_SRC_ON_DEVICE 2u /* dds_put_*: the packed source rows are device memory (same bit as DDS_DST_ON_DEVICE); required */
int dds_put_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts, int64_t fixed_count,
                  int64_t nreq, int itemsize, const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream,
                  int64_t *total_bytes, int64_t *bad_index);
int dds_put_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                    const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                    int64_t *bad_index);

/* ---- batched accumulates: rows ADDED into any rank's shard from this GPU (MPI_Accumulate with MPI_SUM between fences)
 * Every element e of request i's rows becomes shard[e] + src[e], the sum taken in `dtype` (DDS_ACC_*). Requests, the
 * layout of src, validation, error reporting (every valid request is applied, an invalid one changes nothing, the
 * first invalid one is reported; a layout total above src_bytes applies nothing, DDS_ERR_CAPACITY), flags, queueing and
 * fences are dds_put_batch's / dds_put_samples's, word for word. In addition, with DDS_ERR_ARG and nothing enqueued:
 * an unknown dtype, and a src not aligned to the element size. A dtype whose size is not the variable's itemsize is
 * DDS_ERR_DTYPE ("Invalid data type").
 * Concurrency -- this replaces the put's conflict rule: accumulates into the same element in one epoch, from any batch,
 * any rank, or duplicate requests of one batch, combine atomically. The element ends at its starting value plus every
 * contribution: exactly for the integer types (two's complement, wrapping), with one rounding per addition in an
 * unspecified order for the floating types. f32 may flush subnormal inputs and results to (sign-preserving) zero, as
 * atomicAdd(float *) does; f16 and bf16 do not flush; f64 is IEEE. Mixing puts and accumulates on the same bytes in one
 * epoch, or reading rows while they are being accumulated, is undefined (as in MPI). */
#define DDS_ACC_F32 1 /* element types of an accumulate: the sum is taken in this type */
#define DDS_ACC_F64 2
#define DDS_ACC_I32 3 /* two's-complement, wraps */
#define DDS_ACC_I64 4
#define DDS_ACC_F16 5
#define DDS_ACC_BF16 6
int dds_accumulate_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                         int64_t fixed_count, int64_t nreq, int dtype, const void *src, int64_t src_bytes, unsigned flags,
                         void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);
int dds_accumulate_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int dtype,
                           const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                           int64_t *bad_index);

/* ---- batched fetch-ops: rows added into or swapped with any rank's shard, the previous rows returned (MPI_Get_accumulate
 * with MPI_SUM or MPI_REPLACE between fences). For every element e of request i's rows, in one atomic step:
 *   DDS_OP_SUM:     result[e] = shard[e]; shard[e] = shard[e] + src[e]   (the sum taken in dtype)
 *   DDS_OP_REPLACE: result[e] = shard[e]; shard[e] = src[e]              (a swap)
 * Requests, the layout of src, validation, error reporting (every valid request is applied, an invalid one changes
 * nothing, the first invalid one is reported; a layout total above src_bytes applies nothing, DDS_ERR_CAPACITY), dtype
 * (a DDS_ACC_* code; a size other than the variable's itemsize is DDS_ERR_DTYPE), flags, DDS_NO_SYNC queueing, fences
 * and the ignored DDS_OVERLAP (a fetch-op ends an overlap run) are dds_accumulate_batch's / dds_accumulate_samples's,
 * word for word.
 * result has the layout of src: request i's previous rows go to result bytes [o_i, o_i + n_i), the offsets its src rows
 * occupy. It is device memory of at least src_bytes bytes. An invalid request's result bytes, and every byte outside
 * the valid requests' ranges, are left untouched; a capacity error writes nothing to the shards or to result. result ==
 * src is allowed (an in-place exchange); any other overlap of result with src, or of either with a shard, is undefined.
 * Atomicity is per element, as in MPI: fetch-ops on one element in one epoch -- from any batch, any rank, or duplicate
 * requests of one batch -- are linearisable, and each one's result is the element's value immediately before its own
 * contribution. DDS_OP_SUM fetch-ops also combine atomically with dds_accumulate_* of the same dtype on the same element.
 * Mixing DDS_OP_REPLACE with sums, accumulates or puts on one element in one epoch is undefined (MPI allows only the
 * same op or MPI_NO_OP). Rows are not atomic as a whole. Float sums round once per addition, f32 may flush subnormal
 * inputs and results to zero as the accumulate's may; f16 and bf16 do not flush; f64 is IEEE; integers wrap.
 * In addition to the accumulate's argument errors, with DDS_ERR_ARG and nothing enqueued: an unknown op, result == NULL
 * while the layout is non-empty, and a result not aligned to the element size. */
#define DDS_OP_SUM 1     /* result[e] = shard[e]; shard[e] = shard[e] + src[e]   (MPI_SUM, in dtype) */
#define DDS_OP_REPLACE 2 /* result[e] = shard[e]; shard[e] = src[e]              (MPI_REPLACE: swap) */
int dds_get_accumulate_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                             int64_t fixed_count, int64_t nreq, int op, int dtype, const void *src, void *result,
                             int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                             int64_t *bad_index);
int dds_get_accumulate_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int op,
                               int dtype, const void *src, void *result, int64_t src_bytes, unsigned flags,
                               void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);

/* ---- batched reductions: max, min and bitwise ops into any rank's shard (the rest of MPI_Accumulate's predefined ops,
 * MPI_MAX, MPI_MIN, MPI_BAND, MPI_BOR and MPI_BXOR, between fences). dds_accumulate_op_batch / dds_accumulate_op_samples
 * take dds_accumulate_batch's / dds_accumulate_samples's arguments plus `op`, and every element e of request i's rows
 * becomes op(shard[e], src[e]). They accept DDS_OP_SUM (exactly dds_accumulate_batch / _samples) and ops 4-8 below.
 * dds_get_accumulate_batch / dds_get_accumulate_samples accept ops 4-8 too: result[e] = shard[e] in the same atomic step.
 * Requests, the layout of src, validation, error reporting, flags, DDS_NO_SYNC queueing, fences, the result rules and the
 * ignored DDS_OVERLAP are dds_accumulate_batch's / dds_get_accumulate_batch's, word for word.
 * Allowed (op, dtype) pairs:
 *   DDS_OP_MAX, DDS_OP_MIN: every DDS_ACC_* type. DDS_ACC_I32 / I64 compare as signed. Floats follow IEEE 754-2019
 *     maximumNumber / minimumNumber with -0 < +0: a NaN operand is ignored, a NaN in the shard is replaced by a non-NaN
 *     operand, NaN with NaN gives a NaN whose bits are unspecified. Nothing flushes: every result is the bits of one of
 *     its inputs (or that NaN).
 *   DDS_OP_BAND, DDS_OP_BOR, DDS_OP_BXOR: DDS_ACC_I32 and DDS_ACC_I64 only (on the bits of any 4- or 8-byte variable).
 * Argument errors, with DDS_ERR_ARG and nothing enqueued, checked after the dtype's: an unknown op, DDS_OP_REPLACE given
 * to dds_accumulate_op_* (a put writes rows), and a bitwise op with a float dtype.
 * Concurrency: reductions on one element in one epoch with the same op and dtype combine atomically -- from any batch,
 * any rank, or duplicate requests of one batch, through either entry family. The element ends at the op folded over its
 * starting value and every contribution; these ops are commutative and associative, so that does not depend on the
 * order (but for the bits of a NaN-with-NaN result). The fetch forms are linearisable per element, each result the value
 * immediately before its own contribution. Mixing different ops, or reductions with puts or compare-and-swaps, on one
 * element in one epoch is undefined, as in MPI. Rows are not atomic as a whole. */
#define DDS_OP_MAX 4  /* shard[e] = max(shard[e], src[e])   (MPI_MAX) */
#define DDS_OP_MIN 5  /* shard[e] = min(shard[e], src[e])   (MPI_MIN) */
#define DDS_OP_BAND 6 /* shard[e] = shard[e] & src[e]       (MPI_BAND) */
#define DDS_OP_BOR 7  /* shard[e] = shard[e] | src[e]       (MPI_BOR) */
#define DDS_OP_BXOR 8 /* shard[e] = shard[e] ^ src[e]       (MPI_BXOR) */
int dds_accumulate_op_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                            int64_t fixed_count, int64_t nreq, int op, int dtype, const void *src, int64_t src_bytes,
                            unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);
int dds_accumulate_op_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int op,
                              int dtype, const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream,
                              int64_t *total_bytes, int64_t *bad_index);

/* ---- batched compare-and-swaps: elements of any rank's shard replaced where they hold an expected value, the previous
 * rows returned (MPI_Compare_and_swap between fences, batched). For every element e of request i's rows, in one atomic
 * step:
 *   result[e] = shard[e]; if (shard[e] == compare[e]) shard[e] = src[e]
 * Elements are itemsize bytes, which must be the variable's itemsize and 1, 2, 4 or 8. The comparison is BITWISE, as
 * MPI_Compare_and_swap restricts itself to integer and byte types: on float data -0 and +0 differ, a NaN equals only the
 * same bit pattern (payload and signalling bit included), and subnormals compare by their bits.
 * Requests, the layout of src, validation, error reporting (every valid request is applied, an invalid one changes
 * nothing and writes no result bytes, the first invalid one is reported; a layout total above src_bytes touches nothing,
 * DDS_ERR_CAPACITY), flags, DDS_NO_SYNC queueing, fences and the ignored DDS_OVERLAP (a compare-and-swap ends an overlap
 * run) are dds_get_accumulate_batch's / dds_get_accumulate_samples's, word for word.
 * compare and result have the layout of src and are device memory of at least src_bytes bytes. result always receives
 * the previous value, for failed compares too: element e was swapped exactly when result[e] == compare[e]. An invalid
 * request's result bytes, and every byte outside the valid requests' ranges, are left untouched, and no compare byte
 * outside them is read. result == src and result == compare are allowed; any other overlap of src, compare and result
 * with each other or with a shard is undefined.
 * Atomicity is per element: compare-and-swaps on one element in one epoch -- from any batch, any rank, or duplicate
 * requests of one batch -- are linearisable. So of N requests that all compare against the element's value, exactly one
 * succeeds and the others get its value back. 1- and 2-byte elements are swapped by a compare-and-swap loop on their
 * aligned 32-bit word, which leaves every other byte of the word as it finds it, also while other requests or ranks
 * change those bytes. Mixing compare-and-swaps with puts, accumulates or fetch-ops on one element in one epoch is
 * undefined. Rows are not atomic as a whole.
 * Argument errors, with DDS_ERR_ARG and nothing enqueued: the put's, an itemsize other than 1, 2, 4 or 8, compare or
 * result == NULL while the layout is non-empty, and src, compare or result not aligned to the itemsize. An itemsize other
 * than the variable's is DDS_ERR_DTYPE. */
int dds_compare_and_swap_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                               int64_t fixed_count, int64_t nreq, int itemsize, const void *src, const void *compare,
                               void *result, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                               int64_t *bad_index);
int dds_compare_and_swap_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                                 const void *src, const void *compare, void *result, int64_t src_bytes, unsigned flags,
                                 void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);

/* ---- pooled batches: bags of rows from any rank's shard reduced to one row each (torch's embedding_bag over a sharded
 * variable, in one launch)
 * Requests are located and validated exactly as in dds_get_batch / dds_get_samples, with the same codes, texts and
 * divergences; a sample id outside the index is DDS_ERR_ARG, "sample id outside the variable's sample index".
 * Bag k folds the rows of requests [bags[k], bags[k+1]) -- in request order, within a request in row order -- into output
 * row k: dst bytes [k * R, (k + 1) * R), R = disp * itemsize, in `dtype`. *total_bytes = nbags * R. bags == NULL: bag i is
 * request i (nbags must equal nreq). Requests no bag covers are neither read nor validated.
 * An invalid request contributes nothing and every valid request is still applied (the padded entries' rule); the first
 * (lowest-index) invalid request is reported.
 * Numerics, per output element -- the sequential fold torch's CUDA embedding_bag forward computes:
 *   acc is f32 for f32, f16 and bf16 rows and f64 for f64 rows, starting at +0;
 *   DDS_POOL_SUM   acc = acc + x, or with weights acc = fma(w, x, acc) (one rounding);
 *   DDS_POOL_MEAN  acc = acc + x, then acc / (rows folded) (IEEE division; a bag with no rows stays 0);
 *   then one round-to-nearest conversion to dtype;
 *   DDS_POOL_MAX   in dtype: the bag's first row as it is, then acc = (x > acc) ? x : acc -- so a leading NaN stays,
 *                  later NaNs are ignored, and of -0 and +0 the earlier one is kept.
 * An empty bag, or one whose requests are all invalid, is +0 in every mode. Nothing flushes subnormals. NaN results of the
 * arithmetic are the canonical NaN. The result is bitwise deterministic: it does not depend on the grid, the ranks, the
 * stream or the queue.
 * Argument errors, DDS_ERR_ARG with nothing enqueued: an unknown mode; a dtype that is not DDS_ACC_F32, F64, F16 or BF16;
 * weights with a mode other than DDS_POOL_SUM; flags without DDS_DST_ON_DEVICE; nbags < 0; bags == NULL with nbags !=
 * nreq; dst_capacity < nbags * R or nbags * R overflowing; dst or weights not aligned to the element size;
 * dds_get_samples_pooled on a variable without a sample index; DDS_NO_SYNC with host indices. A dtype whose size is not
 * the variable's itemsize is DDS_ERR_DTYPE.
 * Malformed bags: bag k is malformed when bags[k] < 0, bags[k + 1] < bags[k] or bags[k + 1] > nreq. Host bags are checked
 * before anything is enqueued; device bags by the kernel, which writes a malformed bag's row as zeros. Either way the call
 * returns DDS_ERR_ARG, "malformed bag offsets", with *bad_index = the lowest such k; a malformed bag takes precedence over
 * any invalid request.
 * Flags: DDS_IDX_ON_DEVICE covers starts, counts, sample ids, bags and weights alike; host ones are staged as in the get
 * entries. DDS_NO_SYNC queues the call (dds_batch_wait reports it like a queued get, its total nbags * R). DDS_OVERLAP is
 * ignored: a pooled launch ends an overlap run, like a put. DDS_PLACE_HOST variables are read over PCIe on the host
 * gather's small grid, with the same results. */
#define DDS_POOL_SUM 1
#define DDS_POOL_MEAN 2
#define DDS_POOL_MAX 3
typedef struct {
    int32_t mode;        /* DDS_POOL_* */
    int32_t dtype;       /* DDS_ACC_F32, DDS_ACC_F64, DDS_ACC_F16 or DDS_ACC_BF16: element type of rows and output */
    const int64_t *bags; /* nbags + 1 request offsets (torch's include_last_offset form); NULL: bag i = request i */
    int64_t nbags;
    const void *weights; /* nullable, one per REQUEST, in `dtype`; DDS_POOL_SUM only (torch's per_sample_weights) */
} dds_pool_t;
int dds_get_batch_pooled(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                         int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, void *dst, int64_t dst_capacity,
                         unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);
int dds_get_samples_pooled(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq,
                           const dds_pool_t *pool, void *dst, int64_t dst_capacity, unsigned flags, void *cuda_stream,
                           int64_t *total_bytes, int64_t *bad_index);

/* ---- pooled accumulates: each bag's gradient scattered into its rows of any rank's shard (the backward of the pooled
 * batches: torch's embedding_bag backward plus the SGD step over a sharded variable, in one launch)
 * The exact adjoint of dds_get_batch_pooled / dds_get_samples_pooled with the same requests and dds_pool_t (bags,
 * weights, DDS_POOL_SUM or DDS_POOL_MEAN). grad holds nbags rows of R = disp * itemsize bytes in pool->dtype. Every
 * element e of every row of every valid request i in bag k gets one contribution c, computed in the forward's
 * accumulator type A (f32 for f32, f16 and bf16; f64 for f64), each step one round-to-nearest operation, none contracted:
 *   c = grad[k][e];  c = c * w_i (weights);  c = c / n_k (DDS_POOL_MEAN);  c = c * (A)alpha;
 * n_k = the rows the pooled get folds for bag k (the rows of its valid requests). c is then rounded once to dtype (a NaN
 * becomes the canonical NaN) and added into the shard by dds_accumulate_batch's rule: atomic across batches, ranks and
 * duplicate ids, one rounding per addition in an unspecified order; f32 may flush subnormals (atomicAdd's rule), f16 and
 * bf16 do not, f64 is IEEE. It combines atomically with dds_accumulate_* and DDS_OP_SUM fetch-ops of the same dtype on the
 * same elements. alpha is torch's alpha in p.add_(g, alpha=-lr); 1.0 gives the plain adjoint. *total_bytes = nbags * R.
 * Errors follow the pooled get's rules: an invalid request contributes nothing and is left out of n_k, every valid one is
 * still applied and the first invalid one is reported; a malformed bag writes nothing and is reported as DDS_ERR_ARG,
 * "malformed bag offsets", with *bad_index = the bag, ahead of any invalid request (host bags are checked before anything
 * is enqueued); requests no bag covers are neither read nor validated.
 * Argument errors, DDS_ERR_ARG with nothing enqueued: any of the pooled get's; DDS_POOL_MAX (its adjoint needs the
 * forward's argmax); flags without DDS_SRC_ON_DEVICE; grad_bytes < nbags * R, or grad == NULL with nbags * R > 0; grad or
 * weights not aligned to the element size; a non-finite alpha. DDS_PLACE_HOST variables are refused as by every batched
 * write. A dtype whose size is not the variable's itemsize is DDS_ERR_DTYPE.
 * Flags: DDS_IDX_ON_DEVICE covers indices, bags and weights alike (host ones are staged). DDS_NO_SYNC queues the call
 * (dds_batch_wait reports it with total nbags * R). DDS_OVERLAP is ignored: the call ends an overlap run, like a put. The
 * rows are visible at the next fence, as for dds_accumulate_batch. */
int dds_accumulate_batch_pooled(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                                int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, double alpha,
                                const void *grad, int64_t grad_bytes, unsigned flags, void *cuda_stream,
                                int64_t *total_bytes, int64_t *bad_index);
int dds_accumulate_samples_pooled(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq,
                                  const dds_pool_t *pool, double alpha, const void *grad, int64_t grad_bytes,
                                  unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index);

/* COLLECTIVE fetch by owner-PUSH (every rank calls, every rank on a GPU of its own; fixed-count batches). A one-sided
 * get() pulls: every NVLink direction then carries payload + response headers + the read requests of the opposite
 * flow. When all ranks fetch in the same
 * step anyway -- a DDP loader -- the owners can push instead (posted writes, less link overhead per payload byte): each rank
 * publishes its start rows in its WINDOW, every owner sends the rows it owns straight into the requesters' windows and
 * signals arrival; the call's kernel ends when this rank's batch is complete. dds_push_setup allocates and maps the
 * windows (room for max_requests start rows and max_bytes of packed rows, twice: results alternate between two
 * buffers, so the buffer returned for step t stays valid until step t + 2). dds_get_batch_push enqueues one step on
 * cuda_stream and returns the device address the packed rows will be at; dds_batch_wait reports errors (same texts
 * and first-bad index as dds_get_batch). */
int dds_push_setup(dds_store_t *s, int64_t max_requests, int64_t max_bytes);
int dds_get_batch_push(dds_store_t *s, const char *name, const int64_t *starts_dev, int64_t fixed_count, int64_t nreq,
                       int itemsize, void **dst_out, void *cuda_stream);

/* Completes the batches issued with DDS_NO_SYNC (stream sync + status decode). Of a queue of several, the earliest
 * failing batch in queue order is reported, with that batch's first invalid request in *bad_index.
 * The outcome of queued batches is reported here and only here, exactly once. Any other call that meets a pending
 * queue (a synchronous batch or get(), a batch on another stream, dds_set_sample_index, dds_set_normalization,
 * dds_epoch_end, dds_epoch_begin when the queue holds a put, an accumulate, a fetch-op or a compare-and-swap, dds_free, a push step on another stream) completes it first and keeps its first failing status; it
 * then does its own work and reports only its own outcome (its error and *bad_index describe its own requests). The
 * next dds_batch_wait reports the kept failure, with its index and text, after completing any queue still pending; a
 * failure kept from earlier wins over any failure queued after it, since it is earlier in queue order. After it has
 * been reported, the next call returns DDS_OK. *total_bytes is the packed size of the last batch queued since the
 * previous dds_batch_wait (an empty one, nreq = 0, counts with size 0), 0 if there was none. A queue reaching 65535
 * launches is completed the same way before its next launch (the status word's queue ordinal has 16 bits), so its
 * failures are still reported in queue order.
 * dds_destroy drops a kept outcome that no dds_batch_wait has reported. */
int dds_batch_wait(dds_store_t *s, int64_t *total_bytes, int64_t *bad_index);

/* void query(string name, VarInfo_t&), ddstore.cxx:46-49 */
int dds_query(dds_store_t *s, const char *name, dds_varinfo_t *out);
/* void epoch_begin() / epoch_end(), ddstore.cxx:51-77: COLLECTIVE fence = stream sync + barrier, with the
 * reference's begin/end state machine. */
int dds_epoch_begin(dds_store_t *s);
int dds_epoch_end(dds_store_t *s);
/* void free(), ddstore.cxx:79-96: COLLECTIVE. Unmaps peers, barriers, releases the shards. */
int dds_free(dds_store_t *s);

/* ---- bench / test helpers (not part of the reference surface) --------------------------------- */
/* Fill this rank's shard of `name` with the synthetic payload of SURVEY.md 8d, on device:
 * element (global_row g, col c) = low itemsize bytes of splitmix64(seed ^ (g*disp + c)). */
int dds_synth_fill(dds_store_t *s, const char *name, uint64_t seed);
/* Check a packed batch against that generator ON THE DEVICE: request i = rows [starts[i], + counts[i] or fixed_count) of
 * `name`, its bytes at packed + (offsets ? offsets[i] : i * fixed_count * disp * itemsize); all pointers device memory
 * (counts / offsets nullable). result[0] = mismatching elements, result[1] = rows checked, result[2 + r] = requests
 * owned by rank r (66 words, host memory). Synchronous. */
int dds_synth_verify(dds_store_t *s, const char *name, const void *packed_dev, const int64_t *starts_dev,
                     const int64_t *counts_dev, int64_t fixed_count, const int64_t *offsets_dev, int64_t nreq, uint64_t seed,
                     void *cuda_stream, uint64_t *result);
/* Test helper: occupy `ctas` SMs' worth of shared memory (`smem_bytes` per CTA) for `nanoseconds` on `cuda_stream` --
 * a stand-in for a training kernel sharing the GPU with a prefetch queue. */
int dds_test_occupy(int device, int ctas, int smem_bytes, uint64_t nanoseconds, void *cuda_stream);
/* kernels launched by this library since load, and the gather launch geometry in use */
unsigned long long dds_kernel_launches(void);
void dds_gather_geometry(int *ctas, int *warps_per_cta, int *stages, int *chunk_bytes, int *smem_bytes);
/* Test helper: the launch geometry a pooled get (adjoint 0) or pooled accumulate (adjoint 1) of `nbags` bags over rows of
 * `row_bytes` of element type `dtype` (DDS_ACC_F32 / F64 / F16 / BF16) is launched with, its destination / grad
 * 16-byte aligned or not, on a DDS_PLACE_HOST variable or not: bytes per lane vector (16 or one element), bytes per column
 * slice, slices per row, row windows per bag (1 for a get) and CTAs of 256 threads. All zeros without a usable device,
 * for nbags or row_bytes <= 0, or for another dtype. */
void dds_pool_geometry(int adjoint, int64_t row_bytes, int dtype, int64_t nbags, int aligned16, int host, int *vb,
                       int64_t *slice, int64_t *nslices, int64_t *windows, int *ctas);
/* CTAs of a gather launch that reads DDS_PLACE_HOST shards (at most 16; 0 without a usable device) */
int dds_host_gather_ctas(void);

#ifdef __cplusplus
}
#endif
#endif
