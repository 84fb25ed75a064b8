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

#define DDS_VERSION 100

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
#define DDS_NO_SYNC 4u       /* needs both flags above: enqueue on cuda_stream and return; dds_batch_wait() reports */
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
 * failing batch in queue order is reported, with that batch's first invalid request in *bad_index. */
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

#ifdef __cplusplus
}
#endif
#endif
