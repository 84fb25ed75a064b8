// ddstore_b200/csrc/kernels.cu -- the get() hot path as hand-written sm_90a CUDA.
//
// What the reference does per sample (include/ddstore.hpp:197-238 + src/ddstore.cxx:5-17):
//   owner = sortedsearch(lenlist, start); offset = lenlist[owner-1] (or 0); two range checks;
//   MPI_Get of count*disp*itemsize bytes from the owner's window at row (start-offset).
// What this file does per BATCH, in one persistent kernel (dds_gather_kernel):
//   the same lookup + checks for every request, then a gather of all payloads from the owners'
//   HBM shards (local, or peer-mapped over NVLink/NVSwitch -- CUDA VMM blocks shared by file
//   descriptor, see vmm.cpp) packed back to back into one contiguous device buffer.
//
// Kernel design (bandwidth-bound byte mover, no tensor cores):
//   * The packed destination byte range [0, T) is cut into segments that warps claim dynamically
//     (one atomic per segment, requested one segment ahead; fixed-count DDS_OVERLAP launches stride
//     statically), so load balance is by
//     BYTES, not by request count (lengths differ 100x in the variable-length configs) and not by
//     owner (remote rows are slower than local).
//   * Every warp is an autonomous pipeline with a private ring of S shared-memory stages. A stage
//     carries a GROUP of up to 32 pieces, one per lane (consecutive small requests, or one <= CH-byte
//     piece of a large one); every lane issues the 1-D TMA bulk load of its own piece
//     (cp.async.bulk global->shared, mbarrier complete_tx), S-1 stages ahead, on the
//     16-byte-aligned superset of the source range, so arbitrary element alignment (4-byte
//     floats, single bytes) is legal for TMA.
//   * Drain, per piece:
//       - staged bytes, destination, size all 16-byte aligned -> the piece's own lane issues one
//         TMA bulk store shared->global, all lanes at once;
//       - same 16-byte phase, ragged ends -> lane 0 bulk-stores the body, byte stores for head/tail;
//       - different phase -> all lanes read two aligned 16-byte vectors from shared memory,
//         funnel-shift (or word-select) them into place and issue aligned 128-bit stores.
//   * Request offsets in the packed buffer are an exclusive prefix sum of request sizes: arithmetic
//     in the fixed-count entry. For variable counts the PLAN (lookup + checks + scan) is
//       - one single-pass kernel (dds_plan_kernel: decoupled look-back over 1024-request tiles), which
//         also fills a segment table (request covering every 16 KiB boundary) so that a segment claim
//         of the gather is one load; in an overlapped queue it runs UNDER the previous batch's gather,
//         in a scratch slot of its own, chained to its gather through a memory word instead of the grid
//         dependency; or
//       - for small batches, computed by EVERY CTA redundantly into its own shared memory (no
//         inter-CTA dependency, one launch per batch).
//     The (start, count) of a request may come from a device-resident per-sample index (sample ids in;
//     the table is kept in the persisting part of L2).
//   * Launches carry the programmatic-dependent-launch attribute; independent batches
//     (DDS_OVERLAP) skip the grid wait and overlap head-to-tail, under a contract the kernel
//     enforces itself with per-launch generation words (see the overlap protocol at GatherArgs).
//
// Also here: the single-request kernels of the legacy one-get()-per-sample loop (dds_doorbell_kernel: a
// resident CTA polling a mailbox in pinned memory, no launch per call; dds_small_get_kernel), the
// collective owner-push variant of the fetch (the push section of dds_gather_kernel), and the
// bench / test helpers (payload generator, on-device verifier, SM occupier).
//
// Nothing here calls a library kernel; everything is launched from the ddsk_* functions at the end.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>

#include "kernels.h"

namespace {

thread_local char g_cuda_err[512] = "";
std::atomic<unsigned long long> g_launches{0};

#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            snprintf(g_cuda_err, sizeof(g_cuda_err), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                     __FILE__, __LINE__);                                                                \
            return (int)e__ ? (int)e__ : -1;                                                             \
        }                                                                                                \
    } while (0)

// ------------------------------------------------------------------------------------------------
// PTX helpers (sm_90a): mbarrier, 1-D TMA bulk copies, shared-memory vector access
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok;
}
// global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
                 "l"(src_gmem), "r"(bytes), "r"(bar)
                 : "memory");
}
// shared -> global, tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_1d(void *dst_gmem, uint32_t src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(src_smem), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void stg128(void *p, uint4 v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------------------------------------
// owner lookup + range checks, exactly the reference's arithmetic
// ------------------------------------------------------------------------------------------------
// src/ddstore.cxx:5-17: first i>=1 with vec[i-1] <= num < vec[i]; else 0 (also when out of range).
__device__ __forceinline__ int dev_sortedsearch(const ddsk_var_t &v, int64_t num) {
    int rtn = 0;
    for (int i = 1; i < v.nranks; i++) {
        if (v.lenlist[i - 1] <= num && num < v.lenlist[i]) {
            rtn = i;
            break;
        }
    }
    return rtn;
}

// include/ddstore.hpp:205-214. Returns 0 or DDSK_CODE_*; *src = address of the first payload byte.
__device__ __forceinline__ int dev_locate(const ddsk_var_t &v, int64_t start, int64_t count, uint64_t *src) {
    int t = dev_sortedsearch(v, start);
    int64_t off = t > 0 ? v.lenlist[t - 1] : 0;
    if (start < off) return DDSK_CODE_START;
    // (count < 0 is UB in the reference; start + count could wrap: start >= off >= 0 here, so the difference cannot)
    if (count < 0 || count > v.lenlist[t] - start) return DDSK_CODE_COUNT;
    *src = (uint64_t)v.bases[t] + (uint64_t)(start - off) * (uint64_t)v.row_bytes; /* ddstore.hpp:229-236 */
    return 0;
}

// same, also returning the owner rank (the collective push fetch lets only the owner act on a request)
__device__ __forceinline__ int dev_locate_owner(const ddsk_var_t &v, int64_t start, int64_t count, uint64_t *src, int *owner) {
    int t = dev_sortedsearch(v, start);
    *owner = t;
    int64_t off = t > 0 ? v.lenlist[t - 1] : 0;
    if (start < off) return DDSK_CODE_START;
    if (count < 0 || count > v.lenlist[t] - start) return DDSK_CODE_COUNT;
    *src = (uint64_t)v.bases[t] + (uint64_t)(start - off) * (uint64_t)v.row_bytes;
    return 0;
}

// Status word: (launch ordinal in its queue << 48) | (request << 8) | code; the lowest report wins. `tag` is the ordinal
// part (DDSK_STATUS_ORD_SHIFT), so an error of an earlier batch of a queue beats any error of a later one.
__device__ __forceinline__ void report(unsigned long long *status, unsigned long long tag, int64_t req, int code) {
    atomicMin(status, tag | ((unsigned long long)req << 8) | (unsigned long long)code);
}

// a few more PTX helpers used below
template <int N>
__device__ __forceinline__ void bulk_wait_all() { // full completion (global writes performed), not just the smem reads
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint64_t lds64(uint32_t addr) {
    uint64_t v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t addr, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// system scope: words other GPUs poll / write over NVLink (collective push fetch)
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ int64_t ld_relaxed_sys_s64(const int64_t *p) {
    int64_t v;
    asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int *p, unsigned int v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------------
// gather kernel
// ------------------------------------------------------------------------------------------------
// where request i's (start row, row count) comes from: explicit arrays, or a per-sample table indexed by ids[i]
struct PlanSrc {
    const int64_t *starts, *counts; // explicit (ids == nullptr)
    const int64_t *ids;             // sample ids (SURVEY.md 8f rank 2: device-resident sample index)
    const longlong2 *tab;           // [nsamples] {row_start, row_count} of every sample of this variable: ONE 16-byte load
    int64_t nsamples;
    // multi-array batches (config 4: node_feat + edge_index of the same samples in ONE launch): request i belongs to
    // variable i / per_var and to sample ids[i % per_var]; every variable has its own window and sample index
    int nvars;               // 0/1: single variable
    int64_t per_var;         // requests per variable (= number of sample ids)
    const ddsk_var_t *mvars; // [nvars] windows, device memory
    const longlong2 *mtab[DDSK_MAX_MULTI];
    int64_t mnsamples[DDSK_MAX_MULTI];
};

__device__ __forceinline__ longlong2 ldg_pair(const longlong2 *p) { return __ldg(p); }

// Lookup + checks of K requests per thread -> (source address or 0, byte size). Written as unrolled passes
// (ids, then table rows, then arithmetic) so that the K independent -- and for the sample index, dependent
// two-level -- global loads of a thread are all in flight together instead of one DRAM latency after another.
// `limit`: requests idx >= limit are not this thread's business (dead lanes).
template <int K>
__device__ __forceinline__ void plan_many(const ddsk_var_t &var, const PlanSrc &p, const int64_t (&idx)[K], int64_t limit,
                                          unsigned long long *status, unsigned long long tag, uint64_t (&src)[K],
                                          int64_t (&nbytes)[K]) {
    int64_t start[K], count[K];
    bool live[K], badid[K];
    const ddsk_var_t *vp[K];
    if (p.nvars > 1) {
        int64_t id[K];
        int v[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            live[k] = idx[k] < limit;
            v[k] = live[k] ? (int)(idx[k] / p.per_var) : 0;
            id[k] = live[k] ? p.ids[idx[k] - (int64_t)v[k] * p.per_var] : 0;
            vp[k] = &p.mvars[v[k]];
        }
#pragma unroll
        for (int k = 0; k < K; k++) {
            badid[k] = live[k] && (id[k] < 0 || id[k] >= p.mnsamples[v[k]]);
            const bool ok = live[k] && !badid[k];
            const longlong2 e = ok ? ldg_pair(&p.mtab[v[k]][id[k]]) : make_longlong2(0, 0);
            start[k] = e.x;
            count[k] = e.y;
        }
    } else if (p.ids) {
        int64_t id[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            live[k] = idx[k] < limit;
            id[k] = live[k] ? p.ids[idx[k]] : 0;
            vp[k] = &var;
        }
#pragma unroll
        for (int k = 0; k < K; k++) {
            badid[k] = live[k] && (id[k] < 0 || id[k] >= p.nsamples);
            const bool ok = live[k] && !badid[k];
            const longlong2 e = ok ? ldg_pair(&p.tab[id[k]]) : make_longlong2(0, 0);
            start[k] = e.x;
            count[k] = e.y;
        }
    } else {
#pragma unroll
        for (int k = 0; k < K; k++) {
            live[k] = idx[k] < limit;
            badid[k] = false;
            start[k] = live[k] ? p.starts[idx[k]] : 0;
            count[k] = live[k] ? p.counts[idx[k]] : 0;
            vp[k] = &var;
        }
    }
#pragma unroll
    for (int k = 0; k < K; k++) {
        src[k] = 0;
        nbytes[k] = 0;
        if (!live[k]) continue;
        if (badid[k]) {
            report(status, tag, idx[k], DDSK_CODE_SAMPLE);
            continue;
        }
        uint64_t s = 0;
        const int code = dev_locate(*vp[k], start[k], count[k], &s);
        if (code) {
            report(status, tag, idx[k], code);
            continue;
        }
        src[k] = s;
        nbytes[k] = count[k] * vp[k]->row_bytes;
    }
}

__device__ __forceinline__ int64_t warp_incl_scan(int64_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int64_t o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += o;
    }
    return v;
}
__device__ __forceinline__ int64_t warp_sum(int64_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

struct GatherArgs {
    ddsk_var_t var;
    const int64_t *starts; // FIXED: start row per request
    int64_t count;         // FIXED: rows per request
    // VAR, plan in global scratch (large batches; written by the two plan kernels before this launch)
    const uint64_t *req_src;  // planned source address (0 = skip)
    const int64_t *req_dst;   // [nreq+1] exclusive scan; req_dst[nreq] = total bytes
    const uint32_t *seg_tab;  // [T / SEG_GRAIN + 1] request covering byte k * SEG_GRAIN of the packed buffer
    // VAR, plan in shared memory (<= PCAP requests): where (start, count) of request i comes from
    PlanSrc plan;
    int64_t *total_out; // VAR + shared plan: CTA 0 publishes the packed total here (one device word)
    int64_t nreq;
    char *dst;
    int64_t dst_cap;
    int64_t *offsets_out; // optional [nreq+1]
    unsigned long long *status;
    unsigned long long status_tag; // this launch's ordinal in its queue, as OR-ed into every status report
    unsigned int *counters; // [0] segment ticket, [1] finished warps -- self-resetting, ticketed launches only
    // multi-array batches (plan.nvars > 1): the packed result of variable v goes to mdst[v]
    char *mdst[DDSK_MAX_MULTI];
    int64_t mcap[DDSK_MAX_MULTI];
    int64_t *moffsets[DDSK_MAX_MULTI]; // optional per-variable [per_var + 1] byte offsets
    int min_seg_chunks;                // smallest segment, in chunks (claims cost more when the plan is in global memory)
    // ---- overlap protocol (DDS_OVERLAP: a batch declared independent of the ONE batch queued right before it)
    //   * fixed-count launches stride their segments statically; variable-count launches (whose CTAs may start late,
    //     behind the plan kernel) claim them by ticket from a word of their own slot, armed once the gate below is open;
    //   * launch q of a run may start while q-1 is still running (skip_wait: no griddepcontrol.wait), but
    //     - it does not write a byte of caller-visible memory before launch q-2 has RETIRED (gate on done[q-2]):
    //       a double-buffered queue that reuses the buffers of batch q-2 is safe whatever else occupies the GPU;
    //     - its last warp publishes done[q] only after done[q-1] is published: launches retire in order, so whatever
    //       the stream runs after launch q sees every earlier batch complete.
    //   Every CTA of q-2 and q-1 has started before the first CTA of q can (programmatic launch order), so the waits
    //   are on warps that are already running: no co-residency assumption, no deadlock.
    //   * a variable-count launch planned by the plan kernels owns scratch slot q & 3. griddepcontrol.wait waits for
    //     EVERY earlier grid of the stream (measured: with it, nothing of batch q moved before gather q-1 had finished),
    //     so inside a run the two kernels of a batch are chained through memory instead: every tile of the plan kernel
    //     adds (1 << 40 | its bytes) to the slot's plan word when its outputs are written, and the gather spins until
    //     the word reads (tiles << 40 | packed total). The PLAN of batch q thus runs under the gather of batch q-1. The lookup kernel first checks that
    //     launch q-4, the slot's previous user, has retired. A kernel only ever spins on kernels launched before it.
    int overlap, skip_wait;
    int wait1_valid, wait2_valid; // q-1 / q-2 belong to the same run
    unsigned int seq;             // q (per-store counter of overlap launches, wraps)
    unsigned int *ovl;            // per slot (q & 3): [0..3] finished-warp counters, [4..7] done words, [8..11] segment
                                  // tickets
    int wait_plan;                // the plan kernels of this launch signal through plan_word[slot] (no grid dependency)
    unsigned long long *plan_word; // [4] per slot: (finished plan tiles << 40) | packed total so far (see dds_plan_kernel)
    int64_t plan_tiles;            // tiles of this launch's plan
    unsigned int *tickets;        // the segment ticket word of this launch (counters[0], or ovl[8 + slot]); NULL: static striding
    unsigned long long *host_mirror; // zero-copy pinned host words: [0] status, [1] packed total (written at kernel end)
    unsigned long long *dbg;         // DDS_DEBUG_TIMING: per CTA [entry, plan done, first data, last warp done] (globaltimer ns)
    // ---- collective owner-push fetch (FIXED only; see the protocol at dds_gather_kernel's push section)
    const ddsk_push_t *push; // device copy of the windows' table; NULL: ordinary (pull) batch
    int64_t push_nreq;           // length of this rank's index list for the step (the list is already in its window)
    unsigned long long push_step;
};

// the walk's granularity for segment tables: segment sizes of variable-count launches are multiples of this
constexpr int64_t SEG_GRAIN = 16384;

// One pipeline stage carries a GROUP of up to 32 pieces (one per lane): consecutive requests of the walk, or one
// <= CH-byte piece of a large request. Small requests therefore still put ~CH bytes in flight per stage.
struct Piece {
    uint64_t src;  // first payload byte (0: nothing to copy)
    int64_t dpos;  // byte position in the packed buffer
    uint32_t n;    // payload bytes (0: lane idle)
    uint32_t off;  // byte offset of this piece's aligned superset inside the stage
};

// The plan as the walk sees it: request i's source address and packed offset.
//   PCAP > 0: the CTA's own copy in shared memory (uint32 offsets: this path requires dst_cap < 4 GiB)
//   PCAP = 0: global scratch written by the plan kernels
template <int PCAP>
struct PlanView {
    uint32_t src_s, dst_s; // shared addresses of u64 src[PCAP], u32 dst[PCAP + 1]
    __device__ __forceinline__ uint64_t s(int64_t i) const { return lds64(src_s + (uint32_t)i * 8u); }
    __device__ __forceinline__ int64_t d(int64_t i) const { return (int64_t)lds32(dst_s + (uint32_t)i * 4u); }
};
template <>
struct PlanView<0> {
    const uint64_t *src;
    const int64_t *dst;
    const uint32_t *seg_tab;
    // (L2 loads: inside an overlap run the plan was written by kernels that ran concurrently with this one)
    __device__ __forceinline__ uint64_t s(int64_t i) const { return __ldcg(&src[i]); }
    __device__ __forceinline__ int64_t d(int64_t i) const { return __ldcg(&dst[i]); }
};

template <bool FIXED, int CH, int PCAP>
struct ChunkWalker {
    // warp-uniform state
    int64_t seg_pos = 0, seg_end = 0, T = 0, seg_bytes = 0, nseg = 0, nb = 0;
    int64_t gwarp = 0, nwarps = 1; // this warp's global index / warps in the grid (first segment = gwarp)
    bool first_claim = true, static_claims = false;
    int64_t cur_seg = 0;
    unsigned int pend = 0; // lane 0: ticket claimed ahead of need (the atomic's latency hides behind the current segment)
    bool armed = false;    // a ticket has been requested and not yet consumed
    bool gate_ok = true;   // the ticket word may be touched (overlap launches: only once launch q-2 has retired)
    int64_t r = 0, win_base = -64;
    int64_t nreq = 0; // requests of the walk (a.nreq; the sum over all requesters in a collective push fetch)
    // collective push fetch: the walk runs over the concatenation of every requester's list
    int push_n = 0, push_me = 0, push_par = 0;
    const int64_t *push_rbase = nullptr;  // shared memory: [push_n + 1] first virtual request of requester p
    const uint64_t *push_win = nullptr;   // shared memory: [push_n] window of requester p
    int64_t push_idx_off = 0;
    PlanView<PCAP> pv;
    // per-lane window of 32 request descriptors
    uint64_t w_src = 0;
    int64_t w_dst = 0, w_n = 0;

    __device__ __forceinline__ void load_window(const GatherArgs &a, int lane) {
        win_base = r;
        int64_t idx = r + lane;
        w_src = 0;
        w_dst = 0;
        w_n = 0;
        if (idx < nreq) {
            if (FIXED && push_n > 0) {
                // which requester's list does virtual request idx belong to, and which entry of it?
                int p = 0;
                for (int k = 1; k < push_n; k++)
                    if (idx >= push_rbase[k]) p = k;
                const int64_t i = idx - push_rbase[p];
                const int64_t start = ld_relaxed_sys_s64((const int64_t *)(push_win[p] + push_idx_off) + i);
                uint64_t s = 0;
                int owner = 0;
                const int code = dev_locate_owner(a.var, start, a.count, &s, &owner);
                // only the owner acts on a request: it pushes the rows, or tells the requester what is wrong with it
                if (code && owner == push_me) {
                    unsigned long long *st = (unsigned long long *)push_win[p] + 3;
                    asm volatile("red.relaxed.sys.global.min.u64 [%0], %1;" ::"l"(st), "l"(((unsigned long long)i << 8) | (unsigned long long)code) : "memory");
                }
                w_src = (code || owner != push_me) ? 0 : s;
                w_dst = idx * nb;
                w_n = nb;
            } else if (FIXED) {
                uint64_t s = 0;
                int code = dev_locate(a.var, a.starts[idx], a.count, &s);
                // the reference's two checks; every request with bytes to fetch passes through some warp's window at least once
                if (code) report(a.status, a.status_tag, idx, code);
                w_src = code ? 0 : s; // invalid request: keep its slot in the packed layout, copy nothing
                w_dst = idx * nb;
                w_n = nb;
            } else {
                w_src = pv.s(idx);
                w_dst = pv.d(idx);
                w_n = pv.d(idx + 1) - w_dst;
            }
        }
    }

    // largest r in [0, nreq) with dst[r] <= pos
    __device__ __forceinline__ int64_t locate_var(const GatherArgs &a, int64_t pos, int lane) {
        if (PCAP == 0) {
            // plan in global memory: the plan kernels left the answer for every SEG_GRAIN boundary (one load)
            int64_t r0 = (int64_t)__ldcg(&a.seg_tab[pos / SEG_GRAIN]);
            // zero-length requests right after it share its end offset only if pos is their start too; the table holds
            // the request whose bytes cover pos, which is the largest index with dst <= pos
            return r0;
        }
        int64_t lo = 0, hi = nreq; // 32-ary search across the lanes, shared-memory reads
        while (hi - lo > 1) {
            int64_t step = (hi - lo + 31) / 32;
            int64_t idx = lo + (int64_t)(lane + 1) * step;
            bool le = (idx < hi) && (pv.d(idx) <= pos);
            int k = __popc(__ballot_sync(0xffffffffu, le));
            lo = lo + (int64_t)k * step;
            hi = min(hi, lo + step);
        }
        return lo;
    }

    // Next group of the walk. Returns the bytes to expect in the stage (0: no more work); `pc` is this lane's piece.
    __device__ __forceinline__ void arm(const GatherArgs &a, int lane) { // request the ticket of the NEXT segment
        if (lane == 0) pend = atomicAdd(a.tickets, 1u);
        armed = true;
    }

    template <int STAGE, typename Gate>
    __device__ __forceinline__ uint32_t next_group(const GatherArgs &a, int lane, Piece &pc, Gate &&gate) {
        while (true) {
            if (seg_pos >= seg_end) {
                // the first segment of warp g is segment g (no ticket: spares ~1800 same-address atomics at the
                // start of every launch); later ones come from the ticket counter, offset by the warp count. The
                // ticket for the segment AFTER this one is requested ahead of need and read at the next claim. In an
                // overlap launch the ticket word belongs to the launch's slot and may only be touched once the gate
                // is open (its previous user has retired): normally that happens at this warp's first drain.
                int64_t seg;
                if (first_claim) {
                    first_claim = false;
                    seg = gwarp;
                    if (!static_claims && seg < nseg && gate_ok) arm(a, lane);
                } else if (static_claims) {
                    seg = cur_seg + nwarps; // no ticket word at all: plain striding
                } else {
                    if (!armed) { // (first segment exhausted before the first drain: open the gate here)
                        gate();
                        gate_ok = true;
                        arm(a, lane);
                    }
                    seg = nwarps + (int64_t)__shfl_sync(0xffffffffu, pend, 0);
                    armed = false;
                    if (seg < nseg) arm(a, lane);
                }
                cur_seg = seg;
                if (seg >= nseg) return 0;
                seg_pos = seg * seg_bytes;
                seg_end = min(T, seg_pos + seg_bytes);
                r = FIXED ? seg_pos / nb : locate_var(a, seg_pos, lane);
            }
            if (r >= nreq) { // defensive: cannot happen while seg_pos < T
                seg_pos = seg_end;
                continue;
            }
            if (r < win_base || r >= win_base + 32) load_window(a, lane);
            {   // fast path: the current request alone (nearly) fills a stage, or is cut by CH / the segment end
                const int wl = (int)(r - win_base);
                const uint64_t s0 = __shfl_sync(0xffffffffu, w_src, wl);
                const int64_t d0 = __shfl_sync(0xffffffffu, w_dst, wl);
                const int64_t e0 = d0 + __shfl_sync(0xffffffffu, w_n, wl);
                const int64_t p0 = max(d0, seg_pos);
                const int64_t len = min(min(e0, seg_end) - p0, (int64_t)CH);
                if (len >= CH / 2 || p0 + len < e0) {
                    seg_pos = p0 + len;
                    if (seg_pos >= e0) r++;
                    if (s0 == 0) continue; // rejected request (FIXED): its slot stays untouched
                    const uint64_t src = s0 + (uint64_t)(p0 - d0);
                    pc.src = lane == 0 ? src : 0;
                    pc.dpos = p0;
                    pc.n = lane == 0 ? (uint32_t)len : 0u;
                    pc.off = 0;
                    return ((uint32_t)(src & 15u) + (uint32_t)len + 15u) & ~15u;
                }
            }
            // group path: lane j looks at request r + j (as long as the 32-entry window covers it)
            const int srcl = (int)(r - win_base) + lane;
            const uint64_t q_src = __shfl_sync(0xffffffffu, w_src, srcl & 31);
            const int64_t q_d0 = __shfl_sync(0xffffffffu, w_dst, srcl & 31);
            const int64_t q_n = __shfl_sync(0xffffffffu, w_n, srcl & 31);
            const int64_t q_end = q_d0 + q_n;
            const bool valid = srcl < 32 && r + lane < nreq && q_d0 < seg_end;
            const int64_t p0 = max(q_d0, seg_pos);
            int64_t len = min(q_end, seg_end) - p0;
            len = max(len, (int64_t)0);
            len = min(len, (int64_t)CH);
            const bool complete = p0 + len >= q_end; // this piece finishes its request
            const bool copy = valid && len > 0 && q_src != 0;
            const uint64_t src = q_src + (uint64_t)(p0 - q_d0);
            const uint32_t sz = copy ? (((uint32_t)(src & 15u) + (uint32_t)len + 15u) & ~15u) : 0u;
            uint32_t end = sz; // inclusive scan of the padded sizes -> stage offsets
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                uint32_t o = __shfl_up_sync(0xffffffffu, end, d);
                if (lane >= d) end += o;
            }
            const unsigned ok = __ballot_sync(0xffffffffu, valid && end <= (uint32_t)STAGE);
            const unsigned part = __ballot_sync(0xffffffffu, valid && !complete);
            int m = ok == 0xffffffffu ? 32 : __ffs(~ok) - 1;   // leading lanes that are valid and fit
            if (part) m = min(m, __ffs(part));                  // ... up to and including the first partial piece
            // lane 0 is always valid and fits (STAGE >= CH + 30), so m >= 1
            const bool active = lane < m;
            const int64_t new_pos = __shfl_sync(0xffffffffu, p0 + len, m - 1);
            const uint32_t total = __shfl_sync(0xffffffffu, end, m - 1);
            r += __popc(__ballot_sync(0xffffffffu, active && complete));
            seg_pos = max(seg_pos, new_pos);
            if (total == 0) continue; // only empty / rejected requests in this run
            pc.src = (active && copy) ? src : 0;
            pc.dpos = p0;
            pc.n = (active && copy) ? (uint32_t)len : 0u;
            pc.off = end - sz;
            return total;
        }
    }
};

// Re-phase loop: output vector j = staged bytes [q16 + 16j + 4*WS + bs, +16). Specialised on the word shift WS
// (and on whether a sub-word byte shift is needed at all) so the loop body is branch-free: two aligned 128-bit
// shared loads, at most four funnel shifts, one aligned 128-bit global store.
template <int WS, bool BYTES>
__device__ __forceinline__ void rephase_loop(uint32_t sbase, char *dv, uint32_t nv, uint32_t bs8, int lane) {
#pragma unroll 4
    for (uint32_t j = (uint32_t)lane; j < nv; j += 32) {
        const uint4 lo = lds128(sbase + (j << 4));
        const uint4 hi = lds128(sbase + (j << 4) + 16);
        const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        uint4 out;
        if (BYTES) {
            out.x = __funnelshift_r(w[WS + 0], w[WS + 1], bs8);
            out.y = __funnelshift_r(w[WS + 1], w[WS + 2], bs8);
            out.z = __funnelshift_r(w[WS + 2], w[WS + 3], bs8);
            out.w = __funnelshift_r(w[WS + 3], w[WS + 4], bs8);
        } else { // 4-byte-aligned shift (float32 / int32 / int64 rows): pure word selection
            out.x = w[WS + 0];
            out.y = w[WS + 1];
            out.z = w[WS + 2];
            out.w = w[WS + 3];
        }
        stg128(dv + ((size_t)j << 4), out);
    }
}

// Drain one staged piece: payload byte k lives at shared address sb + a + k and goes to d[k].
template <int CH>
__device__ __forceinline__ void drain_chunk(uint32_t sb, uint32_t a, char *d, uint32_t n, int lane) {
    uint32_t head = (16u - (uint32_t)((uint64_t)d & 15u)) & 15u;
    if (head > n) head = n;
    uint32_t nv = (n - head) >> 4;
    uint32_t tail = n - head - (nv << 4);
    uint32_t s = a + head; // shared offset of the first body byte, 0..30
    uint32_t sh = s & 15u;
    if (nv) {
        if (sh == 0) {
            // source and destination share the 16-byte phase: one bulk store moves the whole body
            if (lane == 0) {
                fence_proxy_async();
                tma_store_1d(d + head, sb + s, nv << 4);
            }
        } else {
            const uint32_t sbase = sb + (s & ~15u);
            const uint32_t bs8 = (sh & 3u) * 8u;
            char *dv = d + head;
            switch ((sh >> 2) * 2u + (bs8 ? 1u : 0u)) { // warp-uniform
            case 0: rephase_loop<0, false>(sbase, dv, nv, bs8, lane); break; // unreachable (sh == 0), kept for the table
            case 1: rephase_loop<0, true>(sbase, dv, nv, bs8, lane); break;
            case 2: rephase_loop<1, false>(sbase, dv, nv, bs8, lane); break;
            case 3: rephase_loop<1, true>(sbase, dv, nv, bs8, lane); break;
            case 4: rephase_loop<2, false>(sbase, dv, nv, bs8, lane); break;
            case 5: rephase_loop<2, true>(sbase, dv, nv, bs8, lane); break;
            case 6: rephase_loop<3, false>(sbase, dv, nv, bs8, lane); break;
            default: rephase_loop<3, true>(sbase, dv, nv, bs8, lane); break;
            }
        }
    }
    if ((uint32_t)lane < head) d[lane] = (char)lds8(sb + a + (uint32_t)lane);
    if ((uint32_t)lane < tail) {
        uint32_t k = head + (nv << 4) + (uint32_t)lane;
        d[k] = (char)lds8(sb + a + k);
    }
}

// ------------------------------------------------------------------------------------------------
// Plan in shared memory (variable counts, <= PCAP requests): EVERY CTA computes the whole plan -- lookup + checks +
// exclusive scan of the request sizes -- for itself. The index arrays are a few tens of KB that stay in L2 after
// the first CTA touched them, so the redundancy is cheap, and it removes every inter-CTA dependency the plan
// used to have (tile tickets, look-back, a grid-wide "all tiles written" wait) as well as the L2 round trips of the
// walk's searches and descriptor loads. Warp w owns a contiguous run of requests; loads are coalesced (lane-strided).
// Returns the packed total T (exact, int64); the shared copy keeps 32-bit offsets (the launcher uses this path only
// when the destination capacity is below 4 GiB, so T > 2^32 is a capacity error and nothing is copied).
// ------------------------------------------------------------------------------------------------
template <int NW, int PCAP>
__device__ __forceinline__ int64_t plan_in_smem(const GatherArgs &a, const PlanView<PCAP> &pv, int64_t *wtot, int warp,
                                                int lane, bool writer) {
    const int64_t nreq = a.nreq;
    const int64_t per_warp = ((nreq + NW * 128 - 1) / (NW * 128)) * 128;
    const int64_t w0 = min(nreq, (int64_t)warp * per_warp), w1 = min(nreq, w0 + per_warp);
    int64_t lane_sum = 0;
    for (int64_t b = w0; b < w1; b += 128) {
        int64_t idx[4], nb[4];
        uint64_t sv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) idx[k] = b + k * 32 + lane;
        plan_many<4>(a.var, a.plan, idx, w1, a.status, a.status_tag, sv, nb);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (idx[k] < w1) {
                sts64(pv.src_s + (uint32_t)idx[k] * 8u, sv[k]);
                sts32(pv.dst_s + (uint32_t)idx[k] * 4u, (uint32_t)min(nb[k], (int64_t)0xFFFFFFFFll)); // size, for pass 2
                lane_sum += nb[k];
            }
        }
    }
    const int64_t wsum = warp_sum(lane_sum);
    if (lane == 0) wtot[warp] = wsum;
    __syncthreads();
    int64_t mine = lane < NW ? wtot[lane] : 0;
    const int64_t T = warp_sum(mine);
    const int64_t base = warp_sum(lane < warp ? mine : 0);
    // pass 2: exclusive scan of this warp's run, in place
    int64_t run = base;
    for (int64_t b = w0; b < w1; b += 32) {
        const int64_t i = b + lane;
        const int64_t v = i < w1 ? (int64_t)lds32(pv.dst_s + (uint32_t)i * 4u) : 0;
        const int64_t incl = warp_incl_scan(v, lane);
        if (i < w1) {
            sts32(pv.dst_s + (uint32_t)i * 4u, (uint32_t)(run + incl - v));
            if (writer && a.offsets_out) a.offsets_out[i] = run + incl - v;
        }
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (warp == 0 && lane == 0) {
        sts32(pv.dst_s + (uint32_t)nreq * 4u, (uint32_t)min(T, (int64_t)0xFFFFFFFFll));
        if (writer) {
            if (a.offsets_out) a.offsets_out[nreq] = T;
            if (a.total_out) *a.total_out = T;
        }
    }
    __syncthreads();
    return T;
}

struct PieceDesc {
    int64_t dpos;
    uint32_t n, pack; // pack = stage offset | (source misalignment << 16)
};

// wait until overlap launch q has retired (its done word carries a sequence number >= q)
__device__ __forceinline__ void spin_until_done(const unsigned int *ovl, unsigned int q, unsigned long long *status,
                                                unsigned long long tag, int64_t nreq) {
    const uint64_t t0 = globaltimer_ns();
    while ((int)(ld_acquire_u32(&ovl[4 + (q & 3u)]) - q) < 0) {
        __nanosleep(100);
        if (globaltimer_ns() - t0 > 4000000000ull) { // never expected; do not hang the box
            report(status, tag, nreq, DDSK_CODE_WATCHDOG);
            __trap();
        }
    }
}

template <bool FIXED, int NW, int S, int CH, int PCAP>
__global__ void __launch_bounds__(NW * 32, 1) dds_gather_kernel(const __grid_constant__ GatherArgs a) {
    constexpr int STAGE = CH + 32; // room for the aligned superset of a misaligned CH-byte range
    extern __shared__ __align__(128) unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t full_bar[NW][S];
    __shared__ __align__(16) PieceDesc desc[NW][S][32];
    __shared__ int64_t wtot[PCAP > 0 ? NW : 1];
    __shared__ int64_t push_rbase[FIXED ? DDSK_MAX_RANKS + 1 : 1];
    __shared__ uint64_t push_win[FIXED ? DDSK_MAX_RANKS : 1];

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t gwarp = (int64_t)blockIdx.x * NW + warp;
    const int64_t nwarps = (int64_t)gridDim.x * NW;

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < S; s++) mbar_init(smem_u32(&full_bar[warp][s]), 1);
        fence_mbar_init();
    }
    if (a.dbg && threadIdx.x == 0) a.dbg[blockIdx.x * 4 + 0] = globaltimer_ns();
    // Programmatic dependent launch: let the NEXT kernel of the stream start launching early (its CTAs take over each
    // SM as ours retire), and do not touch global memory before the PREVIOUS kernel (which may have produced our
    // indices / plan, and resets the ticket counters) has completed and flushed.
    // The first launch of an overlap run triggers only AFTER its own wait: its successor skips the wait, and must not
    // be able to start while anything older than this launch is still in flight.
    if (a.overlap && !a.wait1_valid) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    } else {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        if (!a.skip_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    // gate of the overlap protocol: no caller-visible byte is written before launch q-2 has retired
    bool gate_open = !(a.overlap && a.wait2_valid);
    auto pass_gate = [&]() {
        if (!gate_open) {
            if (lane == 0) spin_until_done(a.ovl, a.seq - 2u, a.status, a.status_tag, a.nreq);
            __syncwarp();
            gate_open = true;
        }
    };

    // ---- the plan (variable counts) ------------------------------------------------------------
    ChunkWalker<FIXED, CH, PCAP> w;
    if (!FIXED) {
        if constexpr (PCAP > 0) {
            w.pv.src_s = smem_u32(smem_dyn) + (uint32_t)(NW * S * STAGE);
            w.pv.dst_s = w.pv.src_s + (uint32_t)PCAP * 8u;
            const bool writer = blockIdx.x == 0;
            if (writer) pass_gate(); // CTA 0 writes the offsets / the total for the caller
            w.T = plan_in_smem<NW, PCAP>(a, w.pv, wtot, warp, lane, writer);
        } else {
            w.pv.src = a.req_src;
            w.pv.dst = a.req_dst;
            w.pv.seg_tab = a.seg_tab;
            if (a.wait_plan) {
                // This batch's plan kernels publish through memory (they may still be running): one word carries
                // "ready" and the packed total. Lane 1 checks the overlap gate (launch q-2 retired) in the same round
                // trip, so a CTA that arrives in a running queue pays one L2 latency for both.
                const bool need_gate = !gate_open;
                unsigned long long pw = 0;
                const uint64_t t0 = globaltimer_ns();
                while (true) {
                    bool ok = true;
                    if (lane == 0) {
                        pw = ld_acquire_u64(&a.plan_word[a.seq & 3u]);
                        ok = (pw >> 40) == (unsigned long long)a.plan_tiles; // every tile of the plan has added its share
                    } else if (lane == 1 && need_gate) {
                        ok = (int)(ld_acquire_u32(&a.ovl[4 + ((a.seq - 2u) & 3u)]) - (a.seq - 2u)) >= 0;
                    }
                    if (__all_sync(0xffffffffu, ok)) break;
                    __nanosleep(100);
                    if (globaltimer_ns() - t0 > 4000000000ull) {
                        report(a.status, a.status_tag, a.nreq, DDSK_CODE_WATCHDOG);
                        __trap();
                    }
                }
                gate_open = true;
                w.T = (int64_t)(__shfl_sync(0xffffffffu, pw, 0) & 0xFFFFFFFFFFull);
            } else {
                w.T = __ldcg(&a.req_dst[a.nreq]);
            }
        }
    }

    // ---- collective owner-push fetch: publish my list, wait for everybody's, build the requester table -------------
    // Protocol (one launch per rank per step t, every rank on its own GPU):
    //   1. this rank's index list is copied into its window (list [t & 1]) by a memcpy queued in front of the launch;
    //      CTA 0 publishes ready = t;
    //   2. every warp waits until every rank's ready >= t (words polled over NVLink, system scope);
    //   3. the walk below runs over the CONCATENATION of all lists; a request is acted on only by its owner, which
    //      TMA-loads the rows from its own HBM and TMA-stores them into the requester's window (posted NVLink writes);
    //   4. the last warp of the grid tells every requester "owner `me`: rows of step t have landed" (after its stores
    //      were performed and fenced at system scope) and then waits for the same word from every owner in its own
    //      window, so the kernel ends only when this rank's batch is complete.
    // A window's list / buffer [t & 1] is reused at step t + 2: this rank's kernel t + 2 starts after its kernel t
    // ended, i.e. after every owner finished reading list t (they signalled arrival after their last read).
    // CTA 0 never waits for another CTA of its own grid, and CTAs are dispatched in index order, so the only waits are
    // on other GPUs' kernels -- which every rank launches (the call is collective).
    const bool push = FIXED && a.push != nullptr;
    if (FIXED && push) {
        const ddsk_push_t *ps = a.push;
        const int P = ps->nranks, me = ps->me, par = (int)(a.push_step & 1ull);
        if (blockIdx.x == 0 && threadIdx.x == 0) { // (the list itself was copied into the window by a stream-ordered
                                                    // memcpy in front of this launch: ddsk_gather_push)
            unsigned long long *hdr = (unsigned long long *)ps->win[me];
            *(volatile unsigned long long *)&hdr[1 + par] = (unsigned long long)a.push_nreq;
            __threadfence_system();
            st_release_sys_u64(&hdr[0], a.push_step);
        }
        const uint64_t t0 = globaltimer_ns();
        for (int r0 = 0; r0 < P; r0 += 32) {
            const int r = r0 + lane;
            while (r < P && ld_acquire_sys_u64((const unsigned long long *)ps->win[r]) < a.push_step) {
                __nanosleep(200);
                if (globaltimer_ns() - t0 > 30000000000ull) { // 30 s: a rank that never launched must not hang the box
                    report(a.status, a.status_tag, a.nreq, DDSK_CODE_WATCHDOG);
                    __trap();
                }
            }
        }
        __syncwarp();
        if (warp == 0) {
            int64_t n = 0;
            for (int r0 = 0; r0 < P; r0 += 32) { // (P <= 64: at most two rounds)
                const int r = r0 + lane;
                int64_t mine_n = 0;
                if (r < P) {
                    push_win[r] = (uint64_t)ps->win[r];
                    mine_n = ld_relaxed_sys_s64((const int64_t *)ps->win[r] + 1 + par);
                }
                const int64_t incl = warp_incl_scan(mine_n, lane);
                if (r < P) push_rbase[r] = n + incl - mine_n;
                n += __shfl_sync(0xffffffffu, incl, 31);
            }
            if (lane == 0) push_rbase[P] = n;
        }
        __syncthreads();
        w.push_n = P;
        w.push_me = me;
        w.push_par = par;
        w.push_rbase = push_rbase;
        w.push_win = push_win;
        w.push_idx_off = ps->idx_off[par];
    }
    if (a.dbg && threadIdx.x == 0) a.dbg[blockIdx.x * 4 + 1] = globaltimer_ns();
    bool dbg_first = a.dbg != nullptr && warp == 0;
    // ---- total bytes, segment geometry -------------------------------------------------------
    w.gwarp = gwarp;
    w.nwarps = nwarps;
    w.static_claims = a.tickets == nullptr;
    w.gate_ok = gate_open; // (variable-count overlap launches opened it together with the plan word)
    // (a fixed count above the variable's row total is invalid for every request, and count * row_bytes need not even
    //  fit in 64 bits: nothing to walk, the check pass below reports the first request)
    w.nb = (FIXED && a.count <= a.var.lenlist[a.var.nranks - 1]) ? a.count * a.var.row_bytes : 0;
    w.nreq = (FIXED && push) ? push_rbase[w.push_n] : a.nreq;
    if (FIXED) w.T = w.nb * w.nreq;
    bool over = w.T > a.dst_cap;
    const int64_t push_dst_off = (FIXED && push) ? a.push->dst_off[w.push_par] : 0;
    // multi-array batch: the walk runs over the concatenation of the variables' packed results; vbase[v] is where
    // variable v starts in that virtual space (unused slots are +inf so dst_of() never selects them)
    const bool multi = !FIXED && a.plan.nvars > 1;
    int64_t vbase[DDSK_MAX_MULTI + 1];
#pragma unroll
    for (int v = 0; v <= DDSK_MAX_MULTI; v++) vbase[v] = INT64_MAX;
    if (multi) {
        over = false;
#pragma unroll
        for (int v = 0; v < DDSK_MAX_MULTI; v++)
            if (v < a.plan.nvars) vbase[v] = w.pv.d((int64_t)v * a.plan.per_var);
#pragma unroll
        for (int v = 0; v < DDSK_MAX_MULTI; v++)
            if (v < a.plan.nvars) {
                const int64_t endv = v + 1 < a.plan.nvars ? vbase[v + 1] : w.T;
                over |= endv - vbase[v] > a.mcap[v];
            }
        if (PCAP > 0) over |= w.T > 0xFFFFFFFFll; // 32-bit shared offsets
    }
    auto dst_of = [&](int64_t dpos) -> char * {
        if (FIXED && push) { // the requester's window, found from the position in the concatenated packed space
            int p = 0;
            for (int k = 1; k < w.push_n; k++)
                if (dpos >= push_rbase[k] * w.nb) p = k;
            return (char *)push_win[p] + push_dst_off + (dpos - push_rbase[p] * w.nb);
        }
        if (!multi) return a.dst + dpos;
        int64_t b = vbase[0]; // static indices only: the tables stay in registers / the constant bank
        char *d = a.mdst[0];
#pragma unroll
        for (int k = 1; k < DDSK_MAX_MULTI; k++)
            if (dpos >= vbase[k]) {
                b = vbase[k];
                d = a.mdst[k];
            }
        return d + (dpos - b);
    };
    {
        // A claim is one atomic (requested ahead of need) + a division (FIXED), a shared-memory search (VAR, plan in
        // shared memory) or one global load (VAR, plan in global scratch). Small segments (8 per warp) keep the tail
        // short; variable-count segments are multiples of SEG_GRAIN when the segment table is in use.
        // (push fetch: finer segments were slower, because every claim costs a window of index reads from the
        // requester's list over NVLink)
        int64_t target = w.T / (nwarps * 8);
        const int64_t unit = (!FIXED && PCAP == 0) ? SEG_GRAIN : (int64_t)CH;
        target = max((int64_t)a.min_seg_chunks * CH, min(target, (int64_t)1 << 20));
        target = max(target, unit);
        if (FIXED && w.nb > 0 && w.nb <= target)
            w.seg_bytes = (target / w.nb) * w.nb; // whole requests per segment
        else
            w.seg_bytes = (target / unit) * unit;
        w.nseg = w.T > 0 ? (w.T + w.seg_bytes - 1) / w.seg_bytes : 0;
    }
    if (over) {
        if (gwarp == 0 && lane == 0) report(a.status, a.status_tag, a.nreq, DDSK_CODE_CAPACITY);
        w.nseg = 0;
    }

    // ---- FIXED with nothing to walk (count <= 0, or the batch does not fit): run the reference's two checks here,
    //      so an invalid request is still the error that gets reported
    if (FIXED && !push && (w.nb <= 0 || over)) {
        for (int64_t i = gwarp * 32 + lane; i < a.nreq; i += nwarps * 32) {
            uint64_t s;
            int code = dev_locate(a.var, a.starts[i], a.count, &s);
            if (code) report(a.status, a.status_tag, i, code);
        }
    }

    // ---- per-warp pipeline -------------------------------------------------------------------
    const uint32_t ring = smem_u32(smem_dyn) + (uint32_t)warp * (uint32_t)(S * STAGE);

    uint32_t issued = 0, consumed = 0;
    bool more = w.nseg > 0;
    while (true) {
        // issue up to S-1 groups ahead
        while (more && issued - consumed < (uint32_t)(S - 1)) {
            Piece pc;
            const uint32_t total = w.template next_group<STAGE>(a, lane, pc, pass_gate);
            if (total == 0) {
                more = false;
                break;
            }
            const uint32_t st = issued % S;
            const uint32_t bar = smem_u32(&full_bar[warp][st]);
            // the stage's previous tenant was drained >= 2 drains ago; the bulk stores a lane issued for it (if any)
            // are at most that lane's second most recent bulk group
            bulk_wait_read<1>();
            if (lane == 0) mbar_expect_tx(bar, total);
            __syncwarp();
            const uint32_t al = (uint32_t)(pc.src & 15u);
            desc[warp][st][lane].dpos = pc.dpos;
            desc[warp][st][lane].n = pc.n;
            desc[warp][st][lane].pack = pc.off | (al << 16);
            if (pc.n) // every lane issues its own piece's TMA load; all complete on the stage's mbarrier
                tma_load_1d(ring + st * STAGE + pc.off, (const void *)(pc.src - al), (al + pc.n + 15u) & ~15u, bar);
            issued++;
        }
        if (consumed == issued) break;
        // drain the oldest group
        const uint32_t st = consumed % S;
        const uint32_t parity = (consumed / S) & 1u;
        const uint32_t bar = smem_u32(&full_bar[warp][st]);
        if (!mbar_try_wait(bar, parity)) {
            const uint64_t t0 = globaltimer_ns();
            while (!mbar_try_wait(bar, parity)) {
                if (globaltimer_ns() - t0 > 4000000000ull) { // 4 s: a lost TMA completion must not hang the box
                    report(a.status, a.status_tag, a.nreq, DDSK_CODE_WATCHDOG);
                    __trap();
                }
            }
        }
        __syncwarp();
        if (dbg_first) {
            dbg_first = false;
            if (lane == 0) a.dbg[blockIdx.x * 4 + 2] = globaltimer_ns();
        }
        pass_gate(); // overlap protocol: the loads above were harmless, the stores below are not
        if (!w.static_claims && !w.gate_ok) { // ... and now the slot's ticket word is this launch's to use
            w.gate_ok = true;
            if (!w.armed) w.arm(a, lane);
        }
        const int64_t my_dpos = desc[warp][st][lane].dpos;
        const uint32_t my_n = desc[warp][st][lane].n;
        const uint32_t my_pack = desc[warp][st][lane].pack;
        // Pieces whose staged bytes, destination and size are all 16-byte aligned (every piece of an aligned
        // fixed-stride batch) are stored by their own lane, all lanes at once: one TMA bulk store each, no loop.
        char *const my_dst = dst_of(my_dpos);
        const bool direct = my_n != 0 && (((uint32_t)(uint64_t)my_dst | my_n | (my_pack >> 16)) & 15u) == 0;
        if (direct) tma_store_1d(my_dst, ring + st * STAGE + (my_pack & 0xffffu), my_n);
        // the rest (re-phase, or <16-byte heads/tails) is drained cooperatively, piece by piece
        unsigned todo = __ballot_sync(0xffffffffu, my_n != 0 && !direct);
        while (todo) {
            const int j = __ffs(todo) - 1;
            todo &= todo - 1;
            const int64_t dpos = __shfl_sync(0xffffffffu, my_dpos, j);
            const uint32_t n = __shfl_sync(0xffffffffu, my_n, j);
            const uint32_t pk = __shfl_sync(0xffffffffu, my_pack, j);
            drain_chunk<CH>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, dst_of(dpos), n, lane);
        }
        bulk_commit(); // every lane: one (possibly empty) bulk group per drained stage
        __syncwarp();  // all lanes are done reading the stage before it is refilled
        consumed++;
    }
    if (a.overlap || (FIXED && push)) {
        bulk_wait_all<0>(); // every lane: its bulk stores have been performed (the done / arrive word below promises that)
        fence_proxy_async_global();
    } else {
        bulk_wait_read<0>(); // every lane: its stages have been read out; the global writes complete with the grid
    }
    __syncwarp();
    pass_gate();
    if (multi) { // per-variable byte offsets = plan offsets rebased to the variable's start
        for (int64_t i = gwarp * 32 + lane; i < a.nreq + a.plan.nvars; i += nwarps * 32) {
            // entry (v, j) for j in [0, per_var]: i enumerates nvars * (per_var + 1) slots
            const int v = (int)(i / (a.plan.per_var + 1));
            const int64_t j = i - (int64_t)v * (a.plan.per_var + 1);
            if (v < a.plan.nvars && a.moffsets[v]) {
                const int64_t basev = w.pv.d((int64_t)v * a.plan.per_var); // == vbase[v]; re-read so that vbase[] is
                int64_t e = (v * a.plan.per_var + j == a.nreq) ? w.T : w.pv.d((int64_t)v * a.plan.per_var + j);
                a.moffsets[v][j] = e - basev;                                // never indexed dynamically
            }
        }
    }
    if (FIXED && a.offsets_out && !push) { // arithmetic offsets, written off the critical path
        for (int64_t i = gwarp * 32 + lane; i <= a.nreq; i += nwarps * 32) a.offsets_out[i] = i * w.nb;
    }

    if (a.dbg && lane == 0) atomicMax(&a.dbg[blockIdx.x * 4 + 3], (unsigned long long)globaltimer_ns());
    if (a.overlap) {
        // ---- overlap protocol: retire in order
        if (lane == 0) {
            __threadfence();
            const unsigned int slot = a.seq & 3u;
            const unsigned int done = atomicAdd(&a.ovl[slot], 1u);
            if (done == (unsigned int)(nwarps - 1)) {
                a.ovl[slot] = 0;
                a.ovl[8 + slot] = 0;
                if (a.wait_plan) a.plan_word[slot] = 0; // (every CTA has read the total long ago)
                if (a.wait1_valid) spin_until_done(a.ovl, a.seq - 1u, a.status, a.status_tag, a.nreq);
                __threadfence();
                st_release_u32(&a.ovl[4 + slot], a.seq);
            }
        }
    } else if (lane == 0) {
        // ---- self-resetting ticket counters
        if (FIXED && push) __threadfence_system(); else __threadfence();
        unsigned int done = atomicAdd(&a.counters[1], 1u);
        if (done == (unsigned int)(nwarps - 1)) {
            a.counters[0] = 0;
            a.counters[1] = 0;
            __threadfence();
            if (FIXED && push) {
                // every warp of this rank has pushed and fenced: tell the requesters, then wait for my own owners
                const ddsk_push_t *ps = a.push;
                for (int r = 0; r < ps->nranks; r++)
                    st_release_sys_u64((unsigned long long *)ps->win[r] + 8 + ps->me, a.push_step);
                const unsigned long long *hdr = (const unsigned long long *)ps->win[ps->me];
                const uint64_t t0 = globaltimer_ns();
                for (int r = 0; r < ps->nranks; r++)
                    while (ld_acquire_sys_u64(&hdr[8 + r]) < a.push_step) {
                        __nanosleep(200);
                        if (globaltimer_ns() - t0 > 30000000000ull) {
                            report(a.status, a.status_tag, a.nreq, DDSK_CODE_WATCHDOG);
                            __trap();
                        }
                    }
                // errors the owners found in MY requests sit in my window's status word
                const unsigned long long st = *(volatile const unsigned long long *)&hdr[3];
                if (st != DDSK_STATUS_OK) atomicMin(a.status, st | a.status_tag);
            }
            if (a.host_mirror) { // the last warp publishes status + total straight into pinned host memory: the host
                                 // reads them after the stream sync, no D2H copy in the call
                a.host_mirror[0] = *(volatile unsigned long long *)a.status;
                a.host_mirror[1] = (unsigned long long)w.T;
                __threadfence_system();
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// dds_small_get_kernel: ONE request, ONE CTA -- the legacy one-get()-per-sample loop (include/ddstore.hpp:197-238
// driven by examples/vae/distdataset.py:79-92). A one-CTA-per-SM persistent launch costs more in ramp/retire than a few KB are worth;
// this one is a plain copy loop that also does the reference's checks, writes the payload (device memory, or pinned
// host memory zero-copy) and then a completion word the host spins on -- no stream synchronize in the call.
// flag[0] = status word ((bad << 8) | code, or DDSK_STATUS_OK), flag[1] = bytes, flag[2] = ticket (written last).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dds_small_get_kernel(const __grid_constant__ ddsk_var_t var, int64_t start, int64_t count,
                                                            char *__restrict__ dst, int64_t dst_cap,
                                                            volatile unsigned long long *flag, unsigned long long ticket) {
    uint64_t src = 0;
    const int code = dev_locate(var, start, count, &src);
    const int64_t n = code ? 0 : count * var.row_bytes;
    unsigned long long st = DDSK_STATUS_OK;
    if (code) st = (unsigned long long)code;                   // request 0
    else if (n > dst_cap) st = ((unsigned long long)1 << 8) | DDSK_CODE_CAPACITY; // index 1 = nreq, like the batch kernel
    if (st == DDSK_STATUS_OK && n > 0) {
        const char *s = (const char *)src;
        if ((((uint64_t)s | (uint64_t)dst | (uint64_t)n) & 15u) == 0) {
            const uint4 *s4 = (const uint4 *)s;
            uint4 *d4 = (uint4 *)dst;
            for (int64_t i = threadIdx.x; i < (n >> 4); i += blockDim.x) d4[i] = s4[i];
        } else if ((((uint64_t)s | (uint64_t)dst | (uint64_t)n) & 3u) == 0) {
            const uint32_t *s1 = (const uint32_t *)s;
            uint32_t *d1 = (uint32_t *)dst;
            for (int64_t i = threadIdx.x; i < (n >> 2); i += blockDim.x) d1[i] = s1[i];
        } else {
            for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = s[i];
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        flag[0] = st;
        flag[1] = (unsigned long long)n;
        __threadfence_system();
        flag[2] = ticket;
    }
}

// ------------------------------------------------------------------------------------------------
// plan kernels (variable counts, batches too large for the shared-memory plan): lookup + checks + exclusive scan of
// request bytes into global scratch, plus the segment table the walk's claims read
// ------------------------------------------------------------------------------------------------
constexpr int PLAN_THREADS = 256;
constexpr int PLAN_ITEMS = 4;
constexpr int PLAN_TILE = PLAN_THREADS * PLAN_ITEMS;

struct PlanProto { // overlap protocol as the plan kernel sees it (all zero: ordinary launch)
    unsigned long long *dbg; // DDS_DEBUG_TIMING
    unsigned int *ovl;
    unsigned long long *plan_word;
    unsigned int seq;
    int skip_wait, wait2_valid, wait4_valid;
};

// The plan kernel: ONE pass. Every CTA takes a tile of PLAN_TILE requests (thread t: 4 consecutive ones), looks them up,
// scans their sizes on chip, publishes the tile's byte count, resolves its offset by a decoupled look-back over the
// tiles before it (words tagged with a per-launch tag, so no memset), and writes source addresses, packed offsets and
// the segment table (which request covers every SEG_GRAIN boundary of the packed buffer -- a segment claim of the
// gather is then one load instead of a search). The chain of DEPENDENT memory round trips is what this kernel costs
// when it runs under the previous batch's gather (each one takes microseconds in a saturated memory system), so
// there are as few as possible: index loads (+ the sample-table gather) and the
// slot / gate polls in parallel, one look-back, one finish count.
// tile_state word: [63:42] tag (22 bits) | [41:40] flag (1 = tile aggregate, 2 = inclusive prefix) | [39:0] bytes
__device__ __forceinline__ unsigned long long tile_pack(unsigned int tag, unsigned int flag, int64_t v) {
    return ((unsigned long long)(tag & 0x3FFFFFu) << 42) | ((unsigned long long)flag << 40) |
           ((unsigned long long)v & 0xFFFFFFFFFFull);
}

__global__ void __launch_bounds__(PLAN_THREADS) dds_plan_kernel(const __grid_constant__ ddsk_var_t var,
                                                                const __grid_constant__ PlanSrc p, int64_t nreq,
                                                                uint64_t *__restrict__ req_src, int64_t *__restrict__ req_dst,
                                                                unsigned long long *tile_state, unsigned int tag,
                                                                int64_t *__restrict__ offsets_out, uint32_t *__restrict__ seg_tab,
                                                                int64_t seg_cap, unsigned long long *status,
                                                                unsigned long long status_tag, PlanProto pr) {
    __shared__ int64_t warp_tot[PLAN_THREADS / 32];
    __shared__ int64_t tile_excl_s;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (pr.dbg && threadIdx.x == 0) atomicMax(&pr.dbg[4096 + 0], (unsigned long long)globaltimer_ns());
    if (!pr.skip_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    // tiles are taken in launch order (blockIdx); a tile only ever waits for lower-numbered tiles
    const int64_t tile = blockIdx.x;
    const int64_t base = tile * PLAN_TILE + (int64_t)threadIdx.x * PLAN_ITEMS;
    int64_t idx[PLAN_ITEMS], nb[PLAN_ITEMS];
    uint64_t sv[PLAN_ITEMS];
#pragma unroll
    for (int k = 0; k < PLAN_ITEMS; k++) idx[k] = base + k;
    plan_many<PLAN_ITEMS>(var, p, idx, nreq, status, status_tag, sv, nb); // (only reads: may run before the slot is known to be free)
    int64_t mine = 0;
#pragma unroll
    for (int k = 0; k < PLAN_ITEMS; k++) mine += nb[k];
    const int64_t incl = warp_incl_scan(mine, lane);
    if (lane == 31) warp_tot[wid] = incl;
    // the scratch slot's previous user (launch seq-4) must have retired before anything is written to the slot; the
    // offsets are caller-visible, so launch seq-2 must have retired too (it implies seq-4): one poll, issued with the
    // index loads above in flight
    if (threadIdx.x == 0) {
        if (pr.wait2_valid && offsets_out) spin_until_done(pr.ovl, pr.seq - 2u, status, status_tag, nreq);
        else if (pr.wait4_valid) spin_until_done(pr.ovl, pr.seq - 4u, status, status_tag, nreq);
    }
    __syncthreads();
    int64_t wbase = 0, agg = 0;
#pragma unroll
    for (int k = 0; k < PLAN_THREADS / 32; k++) {
        const int64_t t = warp_tot[k];
        if (k < wid) wbase += t;
        agg += t;
    }
    // ---- publish the aggregate, look back
    if (wid == 0) {
        if (lane == 0) st_release_u64(&tile_state[tile], tile_pack(tag, tile == 0 ? 2u : 1u, agg));
        int64_t excl = 0;
        if (tile > 0) {
            int64_t win = tile - 1;
            const uint64_t t0 = globaltimer_ns();
            while (true) {
                const int64_t t = win - lane; // lane 0 polls the nearest predecessor
                unsigned long long wv = tile_pack(tag, 2u, 0);
                if (t >= 0) {
                    do {
                        wv = ld_acquire_u64(&tile_state[t]);
                        if (globaltimer_ns() - t0 > 4000000000ull) { // never expected; do not hang the box
                            report(status, status_tag, nreq, DDSK_CODE_WATCHDOG);
                            __trap();
                        }
                    } while ((unsigned int)(wv >> 42) != (tag & 0x3FFFFFu) || ((wv >> 40) & 3u) == 0);
                }
                const unsigned int flag = (unsigned int)((wv >> 40) & 3u);
                const int64_t val = (int64_t)(wv & 0xFFFFFFFFFFull);
                const unsigned inc = __ballot_sync(0xffffffffu, flag == 2u);
                const int stop = inc ? __ffs(inc) - 1 : 31; // nearest tile that already knows its inclusive prefix
                excl += warp_sum(lane <= stop ? val : 0);
                if (inc) break;
                win -= 32;
            }
            if (lane == 0) st_release_u64(&tile_state[tile], tile_pack(tag, 2u, excl + agg));
        }
        if (lane == 0) tile_excl_s = excl;
    }
    __syncthreads();
    int64_t run = tile_excl_s + wbase + incl - mine;
#pragma unroll
    for (int k = 0; k < PLAN_ITEMS; k++) {
        if (idx[k] < nreq) {
            const int64_t d0 = run, d1 = run + nb[k];
            req_src[idx[k]] = sv[k];
            req_dst[idx[k]] = d0;
            if (offsets_out) offsets_out[idx[k]] = d0;
            for (int64_t g = (d0 + SEG_GRAIN - 1) / SEG_GRAIN; g * SEG_GRAIN < d1 && g < seg_cap; g++) seg_tab[g] = (uint32_t)idx[k];
            run = d1;
        }
    }
    const bool last_tile = tile == (int64_t)gridDim.x - 1;
    const int64_t T = tile_excl_s + agg;
    if (last_tile && threadIdx.x == 0) {
        req_dst[nreq] = T;
        if (offsets_out) offsets_out[nreq] = T;
    }
    if (pr.dbg && threadIdx.x == 0) atomicMax(&pr.dbg[4096 + 1], (unsigned long long)globaltimer_ns());
    if (pr.ovl) {
        // overlap run: the gather of this batch spins on the slot's plan word instead of waiting for the grid. Every tile
        // adds (1 << 40 | its bytes) with ONE fire-and-forget release-add once its outputs are written (the barrier makes
        // the other threads' stores part of what thread 0 releases): the word reads (tiles << 40 | packed total) exactly
        // when the plan is complete. The gather's retiring warp clears it for the slot's next user.
        __syncthreads();
        if (threadIdx.x == 0)
            asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(&pr.plan_word[pr.seq & 3u]),
                         "l"((1ull << 40) | ((unsigned long long)agg & 0xFFFFFFFFFFull))
                         : "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// synthetic payload generator + its on-device verifier (bench / test helpers)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

template <typename T>
__global__ void dds_synth_kernel(T *__restrict__ base, uint64_t first_elem, uint64_t nelem, uint64_t seed) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nelem; i += (uint64_t)gridDim.x * blockDim.x)
        base[i] = (T)splitmix64(seed ^ (first_elem + i));
}

// Check a packed batch against the generator: request i = rows [starts[i], starts[i] + count_i) of a variable filled by
// dds_synth_kernel with `seed`; its bytes sit at packed + (offsets ? offsets[i] : i * fixed_count * disp * itemsize).
// out[0] += mismatching elements, out[1] += rows checked, out[2 + owner] += requests served by that owner.
template <typename T>
__global__ void dds_verify_kernel(const __grid_constant__ ddsk_var_t var, const unsigned char *__restrict__ packed,
                                  const int64_t *__restrict__ starts, const int64_t *__restrict__ counts, int64_t fixed_count,
                                  const int64_t *__restrict__ offsets, int64_t nreq, int64_t disp, uint64_t seed,
                                  unsigned long long *out) {
    const int lane = threadIdx.x & 31;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long bad = 0, rows = 0;
    for (int64_t i = gw; i < nreq; i += nw) {
        const int64_t start = starts[i], cnt = counts ? counts[i] : fixed_count;
        if (cnt <= 0) continue;
        const int64_t off = offsets ? offsets[i] : i * fixed_count * disp * (int64_t)sizeof(T);
        const T *p = (const T *)(packed + off);
        const uint64_t e0 = (uint64_t)start * (uint64_t)disp, ne = (uint64_t)cnt * (uint64_t)disp;
        for (uint64_t e = lane; e < ne; e += 32) bad += p[e] != (T)splitmix64(seed ^ (e0 + e));
        if (lane == 0) {
            rows += (unsigned long long)cnt;
            atomicAdd(&out[2 + dev_sortedsearch(var, start)], 1ull);
        }
    }
    for (int d = 16; d > 0; d >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, d);
    if (lane == 0) {
        if (bad) atomicAdd(&out[0], bad);
        if (rows) atomicAdd(&out[1], rows);
    }
}

// ------------------------------------------------------------------------------------------------
// dds_doorbell_kernel: the same single request WITHOUT a kernel launch. One CTA stays resident for as long as get()
// calls keep coming (it leaves by itself after `idle_ns` without one, so a device-wide synchronize never waits longer
// than that) and polls a mailbox in mapped pinned host memory: the host writes the request fields, then a sequence
// number; the kernel does the reference's checks, copies the rows (to device memory, or zero-copy to a pinned bounce
// buffer) and answers with ONE word, (sequence << 8) | code. A mailbox round trip is a fraction of the cost of a
// kernel launch + completion.
// Exit protocol: the kernel's last action is to write its generation number to mb->exit_gen; it never touches the
// mailbox afterwards. A host that finds exit_gen == the generation it believes alive while its request is still
// unanswered launches a fresh kernel (which starts by looking for an unserved request), so no request is lost or
// served twice.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dds_doorbell_kernel(const ddsk_var_t *__restrict__ vars, ddsk_mailbox_t *mb,
                                                           unsigned long long served, unsigned long long gen,
                                                           unsigned long long idle_ns) {
    // the request of the current round: [0] seq_head [1] start [2] count [3] dst [4] dst_cap [5] var | stop << 32 [7] seq_tail
    __shared__ unsigned long long req[8];
    __shared__ int sh_state; // 0: serve req[], 1: leave (idle), 2: leave (asked to)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    while (true) {
        if (warp == 0) {
            // Only this warp polls; the other warps sleep in the barrier below. One poll = ONE coalesced 64-byte read of
            // the request line over PCIe (lanes 0..7, 8 bytes each). The host writes the fields, then seq_tail, then
            // seq_head; a request counts as posted when BOTH equal a new sequence number, which makes the snapshot
            // consistent whatever order the line's pieces are fetched in.
            const uint64_t t0 = globaltimer_ns();
            int state = -1;
            while (state < 0) {
                unsigned long long w = 0;
                if (lane < 8) w = ((volatile unsigned long long *)mb)[lane];
                const unsigned long long head = __shfl_sync(0xffffffffu, w, 0), tail = __shfl_sync(0xffffffffu, w, 7);
                if (head != served && head == tail) {
                    if (lane < 8) req[lane] = w;
                    state = (int)((__shfl_sync(0xffffffffu, w, 5) >> 32) & 1ull) ? 2 : 0;
                } else if (globaltimer_ns() - t0 > idle_ns) {
                    state = 1;
                }
            }
            if (lane == 0) sh_state = state;
        }
        __syncthreads();
        const int state = sh_state;
        const unsigned long long q = req[0];
        if (state != 0) { // idle for too long, or asked to leave (that request IS the stop: answer it, then go)
            if (threadIdx.x == 0) {
                if (state == 2) {
                    *(volatile unsigned long long *)&mb->resp = (q << 8);
                    __threadfence_system();
                }
                *(volatile unsigned long long *)&mb->exit_gen = gen;
                __threadfence_system();
            }
            return;
        }
        const int64_t start = (int64_t)req[1], count = (int64_t)req[2], cap = (int64_t)req[4];
        char *dp = (char *)req[3];
        const ddsk_var_t &var = vars[(int)(req[5] & 0xFFFFFFFFull)];
        uint64_t src = 0;
        const int code = dev_locate(var, start, count, &src);
        const int64_t n = code ? 0 : count * var.row_bytes;
        unsigned long long st = 0; // 0 = ok in the mailbox encoding
        if (code) st = (unsigned long long)code;
        else if (n > cap) st = DDSK_CODE_CAPACITY;
        if (st == 0 && n > 0) {
            const char *sp = (const char *)src;
            if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 15u) == 0) {
                for (int64_t i = threadIdx.x; i < (n >> 4); i += blockDim.x) ((uint4 *)dp)[i] = ((const uint4 *)sp)[i];
            } else if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 3u) == 0) {
                for (int64_t i = threadIdx.x; i < (n >> 2); i += blockDim.x) ((uint32_t *)dp)[i] = ((const uint32_t *)sp)[i];
            } else {
                for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dp[i] = sp[i];
            }
            __threadfence_system(); // the payload is visible (host memory or HBM) before the answer is
        }
        __syncthreads();
        if (threadIdx.x == 0) *(volatile unsigned long long *)&mb->resp = (q << 8) | st;
        served = q;
        // (the next poll overwrites req[]: every thread has read it before the barrier above)
    }
}

// Read a range once (launched with a persisting access-policy window: pulls a per-sample table into the part of L2 the
// gather's streaming traffic cannot evict).
__global__ void dds_touch_kernel(const uint4 *__restrict__ p, size_t n, unsigned int *sink) {
    unsigned int acc = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = p[i];
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x9E3779B9u && sink) *sink = acc; // (keeps the loads alive)
}

// Test helper: hold `gridDim.x` SMs' worth of shared memory busy for `ns` nanoseconds (a stand-in for a training kernel
// that shares the GPU with a prefetch queue; tests/test_gpu_parity.py uses it to attack the overlap protocol).
__global__ void dds_occupy_kernel(unsigned long long ns, int smem_bytes) {
    extern __shared__ unsigned char occ_smem[];
    if ((int)threadIdx.x < smem_bytes) occ_smem[threadIdx.x] = (unsigned char)threadIdx.x;
    const uint64_t t0 = globaltimer_ns();
    while (globaltimer_ns() - t0 < ns) __nanosleep(1000);
    if ((int)threadIdx.x < smem_bytes && occ_smem[threadIdx.x] == 255 && ns == 0) printf("");
}

// ------------------------------------------------------------------------------------------------
// launch geometry
// ------------------------------------------------------------------------------------------------
struct Geometry {
    int nw, stages, ch, pcap;
};
// plan-in-global variants (fixed-count entry, and variable-count batches above 8192 requests)
constexpr Geometry kGeoms[] = {{8, 4, 4096, 0}, {8, 6, 4096, 0}, {16, 3, 4096, 0}, {4, 4, 8192, 0}, {12, 4, 4096, 0}, {4, 6, 4096, 0},
                               {6, 4, 4096, 0},   // (5-6: half-size CTAs, two per SM with DDS_GATHER_CTAS_PER_SM=2)
                               {12, 3, 4096, 0}}; // (7: less in flight per SM -> shorter memory queues)
constexpr int kNumGeoms = (int)(sizeof(kGeoms) / sizeof(kGeoms[0]));
// plan-in-shared-memory variants (variable-count entry): the plan's 12 B per request come out of the stage budget
constexpr Geometry kGeomsS[] = {{12, 3, 4096, 4096}, {12, 3, 3072, 8192}, {16, 3, 2048, 8192}, {16, 3, 3072, 4096}, {8, 4, 4096, 4096}};
constexpr int kNumGeomsS = (int)(sizeof(kGeomsS) / sizeof(kGeomsS[0]));
constexpr int64_t kPlanSmemMax = 8192;
// The redundant plan grows with the batch (every SM reads the same index lines), while the plan kernels cost ~0 when
// they run under the previous batch's gather -- so by default only small batches, where one launch beats three, plan
// in shared memory.
int64_t g_plan_smem_default = 1024; // DDS_SMEM_PLAN_MAX

// On an H100 SXM (400 W limit) config 2 (4 KiB rows) is HBM-bound with every fixed-count variant: 0-4 and 7 are within
// 0.3 % of each other, so 12 warps x 4 stages (also used for the instruction-heavier variable / re-phase path) stays
// the default; rows under 2 KiB take more warps (16 x 3) to keep more small copies in flight.
constexpr int kGeomLarge = 4, kGeomSmall = 2, kGeomVar = 4;

int g_geom_fixed_env = -1; // DDS_GATHER_GEOM      (tuning: force one variant for the fixed-count entry)
int g_geom_var_env = -1;   // DDS_GATHER_GEOM_VAR  (... for the variable-count entry, plan in global; defaults to the former)
int g_geom_s_env = -1;     // DDS_GATHER_GEOM_S    (... for the variable-count entry, plan in shared memory)
int g_min_seg_var = 4, g_min_seg_s = 2; // DDS_VAR_MINSEG / DDS_S_MINSEG: smallest segment in chunks
bool g_geom_init = false;
int g_sms = 0;
int g_ctas_per_sm = 1;
int g_pdl = 1;
// DDS_DEBUG_TIMING=1: device buffer of globaltimer stamps, two regions (overlap launches alternate by sequence parity):
// [cta * 4 + {entry, plan known, first data, last warp done}] for cta < 1024, then [4096 + {lookup last CTA start, lookup
// last CTA end, scan last CTA start, scan last CTA end}]. Never reset (every stamp only grows).
unsigned long long *g_dbg = nullptr;
constexpr size_t kDbgRegion = 4096 + 8;
int g_l2_persist = 1;    // DDS_L2_PERSIST: keep per-sample tables in the persisting part of L2 (A/B switch)
int g_smem_plan = 1; // DDS_SMEM_PLAN: 1 = plan in shared memory when it fits (default), 0 = always the plan kernels (A/B switch)

int pick_geometry() {
    if (g_geom_init) return 0;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev));
    if (const char *e = getenv("DDS_GATHER_GEOM")) g_geom_fixed_env = atoi(e);
    if (g_geom_fixed_env >= kNumGeoms) g_geom_fixed_env = -1;
    g_geom_var_env = g_geom_fixed_env;
    if (const char *e = getenv("DDS_GATHER_GEOM_VAR")) g_geom_var_env = atoi(e);
    if (g_geom_var_env >= kNumGeoms) g_geom_var_env = -1;
    if (const char *e = getenv("DDS_GATHER_GEOM_S")) g_geom_s_env = atoi(e);
    if (g_geom_s_env >= kNumGeomsS) g_geom_s_env = -1;
    if (const char *e = getenv("DDS_VAR_MINSEG")) g_min_seg_var = atoi(e) > 0 ? atoi(e) : 4;
    if (const char *e = getenv("DDS_S_MINSEG")) g_min_seg_s = atoi(e) > 0 ? atoi(e) : 2;
    if (const char *e = getenv("DDS_GATHER_CTAS_PER_SM")) g_ctas_per_sm = atoi(e) > 0 ? atoi(e) : 1;
    if (const char *e = getenv("DDS_PDL")) g_pdl = atoi(e) != 0;
    if (const char *e = getenv("DDS_SMEM_PLAN")) g_smem_plan = atoi(e);
    if (const char *e = getenv("DDS_SMEM_PLAN_MAX")) g_plan_smem_default = atoll(e);
    if (const char *e = getenv("DDS_L2_PERSIST")) g_l2_persist = atoi(e);
    if (const char *e = getenv("DDS_DEBUG_TIMING"))
        if (atoi(e)) {
            CUDA_TRY(cudaMalloc((void **)&g_dbg, 2 * kDbgRegion * 8));
            CUDA_TRY(cudaMemset(g_dbg, 0, 2 * kDbgRegion * 8));
        }
    g_geom_init = true;
    return 0;
}

int geometry_for(bool fixed, int64_t request_bytes) {
    if (fixed) {
        if (g_geom_fixed_env >= 0) return g_geom_fixed_env;
        return request_bytes < 2048 ? kGeomSmall : kGeomLarge;
    }
    return g_geom_var_env >= 0 ? g_geom_var_env : kGeomVar;
}
// shared-memory-plan variant for a batch of nreq requests (-1: does not fit)
int geometry_s_for(int64_t nreq) {
    if (nreq > kPlanSmemMax || nreq > g_plan_smem_default) return -1;
    if (g_geom_s_env >= 0 && kGeomsS[g_geom_s_env].pcap >= nreq) return g_geom_s_env;
    return nreq <= 4096 ? 0 : 1;
}

constexpr int smem_bytes_of(int nw, int s, int ch, int pcap) { return nw * s * (ch + 32) + (pcap ? pcap * 12 + 16 : 0); }
int static_smem_of(int nw, int s) { return nw * s * (8 + 32 * 16) + 16 * 8 + 64; }
int ctas_per_sm_for(int nw, int s, int ch, int pcap) {
    int per_sm = g_ctas_per_sm;
    while (per_sm > 1 && per_sm * (smem_bytes_of(nw, s, ch, pcap) + static_smem_of(nw, s) + 1024) > 227 * 1024) per_sm--;
    return per_sm;
}

template <bool FIXED, int NW, int S, int CH, int PCAP>
int launch_gather_t(const GatherArgs &args_in, cudaStream_t stream) {
    constexpr int smem = smem_bytes_of(NW, S, CH, PCAP);
    static std::atomic<unsigned long long> configured{0}; // bit d: attribute set on device d (it is per device)
    auto kern = dds_gather_kernel<FIXED, NW, S, CH, PCAP>;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    if (dev >= 64 || !(configured.load() & (1ull << dev))) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        if (dev < 64) configured.fetch_or(1ull << dev);
    }
    const int per_sm = ctas_per_sm_for(NW, S, CH, PCAP);
    GatherArgs args = args_in;
    args.dbg = g_dbg ? g_dbg + (size_t)(args.overlap ? (args.seq & 1u) : 0u) * kDbgRegion : nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(g_sms * per_sm));
    cfg.blockDim = dim3(NW * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args));
    g_launches++;
    return 0;
}

// launch with the programmatic-dependent-launch attribute (the kernels call griddepcontrol.wait themselves)
// optional L2 persistence window of the next launch_pdl call (the per-sample table of a by-sample-id plan)
thread_local const void *g_l2_base = nullptr;
thread_local size_t g_l2_bytes = 0;

template <typename... KArgs, typename... Args>
int launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (g_l2_base && g_l2_bytes && g_l2_persist) {
        // the random 16-byte table reads of a by-sample-id plan should hit L2 while the previous gather saturates HBM
        attr[1].id = cudaLaunchAttributeAccessPolicyWindow;
        attr[1].val.accessPolicyWindow.base_ptr = const_cast<void *>(g_l2_base);
        attr[1].val.accessPolicyWindow.num_bytes = g_l2_bytes;
        attr[1].val.accessPolicyWindow.hitRatio = 1.0f;
        attr[1].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr[1].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cfg.numAttrs = 2;
    }
    g_l2_base = nullptr;
    g_l2_bytes = 0;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args...));
    g_launches++;
    return 0;
}

template <bool FIXED>
int launch_gather(const GatherArgs &args, cudaStream_t stream) {
    // (the request size only picks a variant: a count too large to multiply safely counts as large)
    const int64_t request_bytes = args.count < ((int64_t)1 << 20) ? args.count * args.var.row_bytes : INT64_MAX;
    switch (geometry_for(FIXED, FIXED ? request_bytes : 0)) {
    case 1: return launch_gather_t<FIXED, 8, 6, 4096, 0>(args, stream);
    case 2: return launch_gather_t<FIXED, 16, 3, 4096, 0>(args, stream);
    case 3: return launch_gather_t<FIXED, 4, 4, 8192, 0>(args, stream);
    case 4: return launch_gather_t<FIXED, 12, 4, 4096, 0>(args, stream);
    case 5: return launch_gather_t<FIXED, 4, 6, 4096, 0>(args, stream);
    case 6: return launch_gather_t<FIXED, 6, 4, 4096, 0>(args, stream);
    case 7: return launch_gather_t<FIXED, 12, 3, 4096, 0>(args, stream);
    default: return launch_gather_t<FIXED, 8, 4, 4096, 0>(args, stream);
    }
}
int launch_gather_s(int g, const GatherArgs &args, cudaStream_t stream) {
    switch (g) {
    case 1: return launch_gather_t<false, 12, 3, 3072, 8192>(args, stream);
    case 2: return launch_gather_t<false, 16, 3, 2048, 8192>(args, stream);
    case 3: return launch_gather_t<false, 16, 3, 3072, 4096>(args, stream);
    case 4: return launch_gather_t<false, 8, 4, 4096, 4096>(args, stream);
    default: return launch_gather_t<false, 12, 3, 4096, 4096>(args, stream);
    }
}

void fill_overlap(GatherArgs &a, const ddsk_scratch_t *scr, int flags) {
    a.overlap = (flags & DDSK_F_OVERLAP) ? 1 : 0;
    a.skip_wait = (flags & DDSK_F_SKIP_WAIT) ? 1 : 0;
    a.wait1_valid = (flags & DDSK_F_PREV1) ? 1 : 0;
    a.wait2_valid = (flags & DDSK_F_PREV2) ? 1 : 0;
    a.seq = scr->ovl_seq;
    a.ovl = scr->ovl;
    // segment tickets: the store's word for ordinary launches. Overlap launches: none for the fixed-count entry (plain
    // striding -- slot tickets put every warp's claims on one word per launch and did not help a queue that shares the
    // GPU either); the variable-count entries set the slot's own word below (their CTAs
    // may start late, behind the plan kernel, and must not keep a fixed share of the work).
    a.tickets = a.overlap ? nullptr : scr->counters;
}

} // namespace

// ------------------------------------------------------------------------------------------------
// the thin C-ABI the host C++ calls
// ------------------------------------------------------------------------------------------------
extern "C" {

const char *ddsk_last_cuda_error(void) { return g_cuda_err; }
unsigned long long ddsk_launch_count(void) { return g_launches.load(); }
int64_t ddsk_plan_smem_max(void) { return kPlanSmemMax; }
int ddsk_debug_timing(unsigned long long *host_out, int max_words) { // both regions, 2 * (4096 + 8) words
    if (!g_dbg) return 0;
    const size_t n = (size_t)max_words < 2 * kDbgRegion ? (size_t)max_words : 2 * kDbgRegion;
    if (cudaMemcpy(host_out, g_dbg, n * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return (int)n;
}

void ddsk_gather_geometry(int *ctas, int *warps_per_cta, int *stages, int *chunk_bytes, int *smem_bytes) {
    if (pick_geometry()) {
        *ctas = *warps_per_cta = *stages = *chunk_bytes = *smem_bytes = 0;
        return;
    }
    const Geometry &g = kGeoms[geometry_for(true, 4096)];
    *ctas = g_sms * ctas_per_sm_for(g.nw, g.stages, g.ch, 0);
    *warps_per_cta = g.nw;
    *stages = g.stages;
    *chunk_bytes = g.ch;
    *smem_bytes = smem_bytes_of(g.nw, g.stages, g.ch, 0);
}

int ddsk_gather_fixed(const ddsk_var_t *var, const int64_t *starts_dev, int64_t count, int64_t nreq, void *dst_dev,
                      int64_t dst_capacity, int64_t *offsets_dev_or_null, const ddsk_scratch_t *scr, int flags,
                      void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (flags & DDSK_F_RESET) CUDA_TRY(cudaMemsetAsync(scr->status, 0xFF, sizeof(unsigned long long), st));
    if (nreq <= 0) return 0;
    if (int rc = pick_geometry()) return rc;
    GatherArgs a;
    memset(&a, 0, sizeof(a));
    a.var = *var;
    a.starts = starts_dev;
    a.count = count;
    a.nreq = nreq;
    a.dst = (char *)dst_dev;
    a.dst_cap = dst_capacity;
    a.offsets_out = offsets_dev_or_null;
    a.status = scr->status;
    a.status_tag = scr->status_tag;
    a.counters = scr->counters;
    a.min_seg_chunks = 1;
    fill_overlap(a, scr, flags);
    a.host_mirror = (flags & DDSK_F_MIRROR) ? scr->host_mirror : nullptr;
    return launch_gather<true>(a, st);
}

int ddsk_gather_push(const ddsk_var_t *var, const ddsk_push_t *push_host, const ddsk_push_t *push_dev,
                     const int64_t *starts_dev, int64_t count, int64_t nreq, unsigned long long step,
                     const ddsk_scratch_t *scr, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = pick_geometry()) return rc;
    GatherArgs a;
    memset(&a, 0, sizeof(a));
    a.var = *var;
    a.count = count;
    a.nreq = nreq; // (this rank's own requests; the walk covers every rank's)
    a.dst = nullptr;
    a.dst_cap = INT64_MAX;
    a.status = scr->status;
    a.status_tag = scr->status_tag;
    a.counters = scr->counters;
    a.tickets = scr->counters;
    a.min_seg_chunks = 1;
    a.push = push_dev;
    if (nreq > 0) // this rank's list into its window, stream-ordered before the kernel that publishes it
        CUDA_TRY(cudaMemcpyAsync(push_host->win[push_host->me] + push_host->idx_off[step & 1ull], starts_dev, (size_t)nreq * 8,
                                 cudaMemcpyDeviceToDevice, st));
    a.push_nreq = nreq;
    a.push_step = step;
    return launch_gather<true>(a, st);
}

// shared by ddsk_gather_var / ddsk_gather_multi: plan (in the launch, or by the two plan kernels) + gather
static int plan_and_gather(const ddsk_var_t *var, const PlanSrc &p, int64_t nreq, int64_t cap_total, GatherArgs &a,
                           int64_t *offsets_dev_or_null, ddsk_scratch_t *scr, int flags, cudaStream_t st) {
    a.nreq = nreq;
    a.status = scr->status;
    a.status_tag = scr->status_tag;
    a.counters = scr->counters;
    a.host_mirror = (flags & DDSK_F_MIRROR) ? scr->host_mirror : nullptr;
    a.plan = p; // the gather needs nvars / per_var even when the plan ran in its own kernels
    a.total_out = scr->total;
    const int gs = (g_smem_plan && cap_total < ((int64_t)1 << 32)) ? geometry_s_for(nreq) : -1;
    if (gs >= 0) {
        a.offsets_out = offsets_dev_or_null;
        a.min_seg_chunks = g_min_seg_s;
        fill_overlap(a, scr, flags); // no scratch is shared between launches: independent batches may overlap
        if (a.overlap) a.tickets = scr->ovl + 8 + (a.seq & 3u);
        return launch_gather_s(gs, a, st);
    }
    if (nreq > scr->cap_req || cap_total / SEG_GRAIN + 2 > scr->seg_cap) {
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_gather_var: scratch too small (%lld requests > %lld, or %lld segments > %lld)",
                 (long long)nreq, (long long)scr->cap_req, (long long)(cap_total / SEG_GRAIN + 2), (long long)scr->seg_cap);
        return -2;
    }
    // DDS_OVERLAP here means: `scr` carries a scratch slot of this launch's own (slot = ovl_seq & 3), so the plan kernels
    // may run while the previous batch's gather is still going, and the gather overlaps with its tail.
    PlanProto pr;
    memset(&pr, 0, sizeof(pr));
    if (flags & DDSK_F_OVERLAP) {
        pr.dbg = g_dbg ? g_dbg + (size_t)(scr->ovl_seq & 1u) * kDbgRegion : nullptr;
        pr.ovl = scr->ovl;
        pr.plan_word = scr->plan_word;
        pr.seq = scr->ovl_seq;
        pr.skip_wait = (flags & DDSK_F_SKIP_WAIT) ? 1 : 0;
        pr.wait2_valid = (flags & DDSK_F_PREV2) ? 1 : 0;
        pr.wait4_valid = (flags & DDSK_F_PREV4) ? 1 : 0;
    }
    const int tiles = (int)((nreq + PLAN_TILE - 1) / PLAN_TILE);
    // tags the look-back words of this launch (they are never cleared; the caller clears every scratch area it owns
    // when the 22-bit tag is about to wrap and restarts it at 0)
    scr->plan_tag = (scr->plan_tag + 1) & 0x3FFFFFu;
    if (p.ids && (p.tab || p.mtab[0])) { // (multi-array batches: the first variable's table)
        g_l2_base = p.tab ? (const void *)p.tab : (const void *)p.mtab[0];
        g_l2_bytes = (size_t)(p.tab ? p.nsamples : p.mnsamples[0]) * 16;
    }
    if (int rc = launch_pdl(dds_plan_kernel, dim3(tiles), dim3(PLAN_THREADS), st, *var, p, nreq, scr->req_src, scr->req_dst,
                            (unsigned long long *)scr->tile_sums, scr->plan_tag, offsets_dev_or_null, scr->seg_tab, scr->seg_cap,
                            scr->status, scr->status_tag, pr))
        return rc;
    a.req_src = scr->req_src;
    a.req_dst = scr->req_dst;
    a.seg_tab = scr->seg_tab;
    a.total_out = nullptr;
    a.min_seg_chunks = g_min_seg_var;
    fill_overlap(a, scr, flags);
    if (a.overlap) {
        a.tickets = scr->ovl + 8 + (a.seq & 3u);
        a.wait_plan = 1; // (a.skip_wait: inside a run the gather skips the grid wait and spins on the plan-ready word)
        a.plan_word = scr->plan_word;
        a.plan_tiles = tiles;
    }
    return launch_gather<false>(a, st);
}

int ddsk_var_uses_scratch(int64_t nreq, int64_t dst_capacity) {
    if (pick_geometry()) return 1;
    return !(g_smem_plan && dst_capacity < ((int64_t)1 << 32) && geometry_s_for(nreq) >= 0);
}

int ddsk_gather_var(const ddsk_var_t *var, const ddsk_index_t *index, int64_t nreq, void *dst_dev, int64_t dst_capacity,
                    int64_t *offsets_dev_or_null, ddsk_scratch_t *scr, int flags, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (flags & DDSK_F_RESET) CUDA_TRY(cudaMemsetAsync(scr->status, 0xFF, sizeof(unsigned long long), st));
    if (nreq <= 0) return 0;
    if (int rc = pick_geometry()) return rc;
    PlanSrc p;
    memset(&p, 0, sizeof(p));
    p.starts = index->starts;
    p.counts = index->counts;
    p.ids = index->sample_ids;
    p.tab = (const longlong2 *)index->table;
    p.nsamples = index->nsamples;
    GatherArgs a;
    memset(&a, 0, sizeof(a));
    a.var = *var;
    a.dst = (char *)dst_dev;
    a.dst_cap = dst_capacity;
    return plan_and_gather(var, p, nreq, dst_capacity, a, offsets_dev_or_null, scr, flags, st);
}

int ddsk_gather_multi(const ddsk_multi_t *m, const int64_t *sample_ids_dev, int64_t nreq, ddsk_scratch_t *scr, int flags,
                      void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (flags & DDSK_F_RESET) CUDA_TRY(cudaMemsetAsync(scr->status, 0xFF, sizeof(unsigned long long), st));
    if (nreq <= 0 || m->nvars <= 0) return 0;
    if (m->nvars > DDSK_MAX_MULTI) {
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_gather_multi: more than %d variables", DDSK_MAX_MULTI);
        return -2;
    }
    if (int rc = pick_geometry()) return rc;
    PlanSrc p;
    memset(&p, 0, sizeof(p));
    p.ids = sample_ids_dev;
    p.nvars = m->nvars;
    p.per_var = nreq;
    p.mvars = m->vars_dev;
    int64_t cap_total = 0;
    for (int v = 0; v < m->nvars; v++) {
        p.mtab[v] = (const longlong2 *)m->table[v];
        p.mnsamples[v] = m->nsamples[v];
        cap_total += m->cap[v]; // (saturation is irrelevant: anything >= 4 GiB selects the plan kernels)
        if (cap_total < 0 || m->cap[v] < 0) cap_total = INT64_MAX / 2;
    }
    ddsk_var_t dummy;
    memset(&dummy, 0, sizeof(dummy));
    GatherArgs a;
    memset(&a, 0, sizeof(a));
    a.dst = nullptr;
    a.dst_cap = INT64_MAX;
    for (int v = 0; v < m->nvars; v++) {
        a.mdst[v] = (char *)m->dst[v];
        a.mcap[v] = m->cap[v];
        a.moffsets[v] = m->offsets[v];
    }
    return plan_and_gather(&dummy, p, nreq * m->nvars, cap_total, a, nullptr, scr, flags, st);
}

int ddsk_small_get(const ddsk_var_t *var, int64_t start, int64_t count, void *dst, int64_t dst_capacity,
                   unsigned long long *flag_dev, unsigned long long ticket, void *stream) {
    dds_small_get_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(*var, start, count, (char *)dst, dst_capacity, flag_dev, ticket);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int ddsk_doorbell_launch(const ddsk_var_t *vars_dev, ddsk_mailbox_t *mailbox_dev, unsigned long long served,
                         unsigned long long gen, unsigned long long idle_ns, void *stream) {
    dds_doorbell_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(vars_dev, mailbox_dev, served, gen, idle_ns);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int ddsk_l2_warm(const void *base_dev, size_t bytes, void *stream) {
    if (int rc = pick_geometry()) return rc;
    if (!g_l2_persist || !base_dev || bytes < 16) return 0;
    g_l2_base = base_dev;
    g_l2_bytes = bytes;
    const size_t n = bytes / 16;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)g_sms * 8);
    return launch_pdl(dds_touch_kernel, dim3(blocks), dim3(256), (cudaStream_t)stream, (const uint4 *)base_dev, n, (unsigned int *)nullptr);
}

int ddsk_occupy(int ctas, int smem_bytes, unsigned long long ns, void *stream) {
    if (ctas <= 0) return 0;
    CUDA_TRY(cudaFuncSetAttribute(dds_occupy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    dds_occupy_kernel<<<ctas, 128, smem_bytes, (cudaStream_t)stream>>>(ns, smem_bytes);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int ddsk_synth_fill(void *base_dev, int64_t first_global_row, int64_t nrows, int64_t disp, int itemsize, uint64_t seed,
                    void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t nelem = (uint64_t)nrows * (uint64_t)disp;
    uint64_t first = (uint64_t)first_global_row * (uint64_t)disp;
    if (nelem == 0) return 0;
    if (int rc = pick_geometry()) return rc;
    int blocks = (int)std::min<uint64_t>((nelem + 255) / 256, (uint64_t)g_sms * 16);
    switch (itemsize) {
    case 1: dds_synth_kernel<uint8_t><<<blocks, 256, 0, st>>>((uint8_t *)base_dev, first, nelem, seed); break;
    case 2: dds_synth_kernel<uint16_t><<<blocks, 256, 0, st>>>((uint16_t *)base_dev, first, nelem, seed); break;
    case 4: dds_synth_kernel<uint32_t><<<blocks, 256, 0, st>>>((uint32_t *)base_dev, first, nelem, seed); break;
    case 8: dds_synth_kernel<uint64_t><<<blocks, 256, 0, st>>>((uint64_t *)base_dev, first, nelem, seed); break;
    default:
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_synth_fill: unsupported itemsize %d", itemsize);
        return -2;
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int ddsk_synth_verify(const ddsk_var_t *var, const void *packed_dev, const int64_t *starts_dev, const int64_t *counts_dev_or_null,
                      int64_t fixed_count, const int64_t *offsets_dev_or_null, int64_t nreq, int64_t disp, int itemsize,
                      uint64_t seed, unsigned long long *out_dev, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (nreq <= 0) return 0;
    if (int rc = pick_geometry()) return rc;
    const int blocks = g_sms * 8;
    const unsigned char *pk = (const unsigned char *)packed_dev;
    switch (itemsize) {
    case 1: dds_verify_kernel<uint8_t><<<blocks, 256, 0, st>>>(*var, pk, starts_dev, counts_dev_or_null, fixed_count, offsets_dev_or_null, nreq, disp, seed, out_dev); break;
    case 2: dds_verify_kernel<uint16_t><<<blocks, 256, 0, st>>>(*var, pk, starts_dev, counts_dev_or_null, fixed_count, offsets_dev_or_null, nreq, disp, seed, out_dev); break;
    case 4: dds_verify_kernel<uint32_t><<<blocks, 256, 0, st>>>(*var, pk, starts_dev, counts_dev_or_null, fixed_count, offsets_dev_or_null, nreq, disp, seed, out_dev); break;
    case 8: dds_verify_kernel<uint64_t><<<blocks, 256, 0, st>>>(*var, pk, starts_dev, counts_dev_or_null, fixed_count, offsets_dev_or_null, nreq, disp, seed, out_dev); break;
    default:
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_synth_verify: unsupported itemsize %d", itemsize);
        return -2;
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

} // extern "C"
