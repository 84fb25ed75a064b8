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
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <type_traits>

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
// global -> shared, 16 bytes, through L2 only (SASS: LDGSTS): the producer for sources in mapped host memory
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, uint64_t src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src_gmem) : "memory");
}
// one arrival on `bar` once every cp.async this thread issued so far has landed (the barrier counts it: .noinc)
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
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
__device__ __forceinline__ unsigned short lds16h(uint32_t addr) { // (into a 16-bit register, for f16 / bf16 operands)
    unsigned short v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}

// Fetch-ops (fetch1 / fetch16 below): atomics that return the element's previous value, at .sys scope for the
// accumulate's reason. Adds round and flush exactly as the accumulate's element and
// vector reductions do (f32 flushes, f16 / bf16 are .noftz, f64 is IEEE, integers wrap).
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts16(uint32_t addr, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"((unsigned short)v) : "memory"); }
__device__ __forceinline__ uint32_t atom_add_u32(char *d, uint32_t v) {
    uint32_t o;
    asm volatile("atom.relaxed.sys.global.add.u32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory");
    return o;
}
__device__ __forceinline__ uint64_t atom_add_u64(char *d, uint64_t v) {
    uint64_t o;
    asm volatile("atom.relaxed.sys.global.add.u64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory");
    return o;
}
__device__ __forceinline__ uint64_t atom_add_f64(char *d, uint64_t v) {
    double o;
    asm volatile("atom.relaxed.sys.global.add.f64 %0, [%1], %2;" : "=d"(o) : "l"(d), "d"(__longlong_as_double((long long)v)) : "memory");
    return (uint64_t)__double_as_longlong(o);
}
__device__ __forceinline__ uint32_t atom_exch_b32(char *d, uint32_t v) {
    uint32_t o;
    asm volatile("atom.relaxed.sys.global.exch.b32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory");
    return o;
}
__device__ __forceinline__ uint64_t atom_exch_b64(char *d, uint64_t v) {
    uint64_t o;
    asm volatile("atom.relaxed.sys.global.exch.b64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory");
    return o;
}
// 16-bit swap (there is no 16-bit exchange): a compare-and-swap loop on the aligned 32-bit word that holds the element,
// which replaces the element's 16 bits and leaves the other 16 exactly as it finds them
__device__ __forceinline__ uint32_t atom_exch_b16(char *d, uint32_t v) {
    unsigned int *w = (unsigned int *)((uint64_t)d & ~(uint64_t)3);
    const uint32_t sh = ((uint32_t)(uint64_t)d & 2u) * 8u, mask = 0xFFFFu << sh;
    uint32_t cur;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(cur) : "l"(w) : "memory");
    while (true) {
        const uint32_t want = (cur & ~mask) | ((v & 0xFFFFu) << sh);
        uint32_t seen;
        asm volatile("atom.relaxed.sys.global.cas.b32 %0, [%1], %2, %3;" : "=r"(seen) : "l"(w), "r"(cur), "r"(want) : "memory");
        if (seen == cur) break;
        cur = seen;
    }
    return (cur >> sh) & 0xFFFFu;
}

// Compare-and-swap (a fetch-op of op DDSK_OP_CAS), element size 1 << el (warp-uniform): the element becomes the operand where it
// equals the compare operand bit for bit, and its previous value comes back either way. 4- and 8-byte elements take one
// atom.cas each (no atom.cas.b128: its behaviour towards a peer over NVLink is not established); 1- and 2-byte elements
// a compare-and-swap loop on the aligned 32-bit word that holds them (cas_word). .sys scope, as the other fetch-ops.
__device__ __forceinline__ uint32_t atom_cas_b32(char *d, uint32_t c, uint32_t v) {
    uint32_t o;
    asm volatile("atom.relaxed.sys.global.cas.b32 %0, [%1], %2, %3;" : "=r"(o) : "l"(d), "r"(c), "r"(v) : "memory");
    return o;
}
__device__ __forceinline__ uint64_t atom_cas_b64(char *d, uint64_t c, uint64_t v) {
    uint64_t o;
    asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(o) : "l"(d), "l"(c), "l"(v) : "memory");
    return o;
}
// The elements of the bytes m of the aligned word w (1 << el bytes each, el 0 or 1): each becomes v's where it equals c's;
// every byte outside m is left exactly as it is found, whoever changes it meanwhile. Returns the word the step found.
// When no element changes, the load was the atomic step (a failed compare is a read).
__device__ __forceinline__ uint32_t cas_word(char *w, uint32_t c, uint32_t v, uint32_t m, uint32_t el) {
    uint32_t cur;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(cur) : "l"(w) : "memory");
    while (true) {
        const uint32_t eq = (el ? __vcmpeq2(cur, c) : __vcmpeq4(cur, c)) & m;
        const uint32_t want = (cur & ~eq) | (v & eq);
        if (want == cur) return cur;
        const uint32_t seen = atom_cas_b32(w, cur, want);
        if (seen == cur) return cur;
        cur = seen;
    }
}
// Compare operands are read with plain global loads of exactly their own bytes (the compare buffer may end where the
// layout does, and may be the result buffer)
__device__ __forceinline__ uint32_t ldg8(const char *p) {
    uint32_t v;
    asm volatile("ld.global.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ldg16(const char *p) {
    uint32_t v;
    asm volatile("ld.global.u16 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ldg32(const char *p) {
    uint32_t v;
    asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint64_t ldg64(const char *p) {
    uint64_t v;
    asm volatile("ld.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
// 16 bytes at p, in p's own 16-byte phase: the widest loads its alignment allows
__device__ __forceinline__ uint4 ldg16_any(const char *p) {
    const uint32_t ph = (uint32_t)(uint64_t)p & 15u;
    uint4 r;
    if (ph == 0) {
        asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    } else if ((ph & 7u) == 0) {
        const uint64_t a = ldg64(p), b = ldg64(p + 8);
        r = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
    } else if ((ph & 3u) == 0) {
        r = make_uint4(ldg32(p), ldg32(p + 4), ldg32(p + 8), ldg32(p + 12));
    } else if ((ph & 1u) == 0) {
        r = make_uint4(ldg16(p) | ldg16(p + 2) << 16, ldg16(p + 4) | ldg16(p + 6) << 16, ldg16(p + 8) | ldg16(p + 10) << 16,
                       ldg16(p + 12) | ldg16(p + 14) << 16);
    } else {
        uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int i = 0; i < 16; i++) w[i >> 2] |= ldg8(p + i) << ((i & 3) * 8);
        r = make_uint4(w[0], w[1], w[2], w[3]);
    }
    return r;
}
__device__ __forceinline__ void sts8(uint32_t addr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
// 16 bytes o to shared address p of any phase, touching exactly them
__device__ __forceinline__ void sts16_any(uint32_t p, uint4 o) {
    switch (p & 3u) {
    case 0:
        sts32(p, o.x);
        sts32(p + 4, o.y);
        sts32(p + 8, o.z);
        sts32(p + 12, o.w);
        break;
    case 1:
        sts8(p, o.x);
        sts16(p + 1, o.x >> 8);
        sts32(p + 3, __funnelshift_r(o.x, o.y, 24));
        sts32(p + 7, __funnelshift_r(o.y, o.z, 24));
        sts32(p + 11, __funnelshift_r(o.z, o.w, 24));
        sts8(p + 15, o.w >> 24);
        break;
    case 2:
        sts16(p, o.x);
        sts32(p + 2, __funnelshift_r(o.x, o.y, 16));
        sts32(p + 6, __funnelshift_r(o.y, o.z, 16));
        sts32(p + 10, __funnelshift_r(o.z, o.w, 16));
        sts16(p + 14, o.w >> 16);
        break;
    default:
        sts8(p, o.x);
        sts32(p + 1, __funnelshift_r(o.x, o.y, 8));
        sts32(p + 5, __funnelshift_r(o.y, o.z, 8));
        sts32(p + 9, __funnelshift_r(o.z, o.w, 8));
        sts16(p + 13, o.w >> 8);
        sts8(p + 15, o.w >> 24);
        break;
    }
}
// one element at d: the operand staged at shared address s, compared with the element at c, is replaced by the
// element's previous value (all three aligned to the element size)
__device__ __forceinline__ void cas1(char *d, uint32_t s, const char *c, uint32_t el) {
    switch (el) {
    case 3: sts64(s, atom_cas_b64(d, ldg64(c), lds64(s))); break;
    case 2: sts32(s, atom_cas_b32(d, ldg32(c), lds32(s))); break;
    default: {
        const uint32_t sh = ((uint32_t)(uint64_t)d & 3u) * 8u, m = (el ? 0xFFFFu : 0xFFu) << sh;
        const uint32_t o = cas_word((char *)((uint64_t)d & ~(uint64_t)3), (el ? ldg16(c) : ldg8(c)) << sh,
                                    (el ? (uint32_t)lds16h(s) : lds8(s)) << sh, m, el) >> sh;
        if (el) sts16(s, o);
        else sts8(s, o);
        break;
    }
    }
}
// 16 bytes at a 16-byte aligned d: the operands v, compared with c, element-wise; returns the previous 16 bytes
__device__ __forceinline__ uint4 cas16(char *d, uint4 v, uint4 c, uint32_t el) {
    if (el == 3) {
        const uint64_t a = atom_cas_b64(d, (uint64_t)c.y << 32 | c.x, (uint64_t)v.y << 32 | v.x);
        const uint64_t b = atom_cas_b64(d + 8, (uint64_t)c.w << 32 | c.z, (uint64_t)v.w << 32 | v.z);
        return make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
    }
    if (el == 2) return make_uint4(atom_cas_b32(d, c.x, v.x), atom_cas_b32(d + 4, c.y, v.y), atom_cas_b32(d + 8, c.z, v.z),
                                   atom_cas_b32(d + 12, c.w, v.w));
    return make_uint4(cas_word(d, c.x, v.x, ~0u, el), cas_word(d + 4, c.y, v.y, ~0u, el), cas_word(d + 8, c.z, v.z, ~0u, el),
                      cas_word(d + 12, c.w, v.w, ~0u, el));
}

// The reductions and fetch-ops of the batched writes: op = DDSK_OP_* and element type t = DDSK_ACC_*, both warp-uniform.
// Every one is atomic per element: the element ops at .sys scope (a peer's ops on the same shard must combine with the
// owner's), the bulk reductions at the scope the ISA gives them.
// Sums: the f32 element and vector reductions flush subnormal inputs and results to zero (atomicAdd's rule; the f32 bulk
// reduction kept them on H100, see DESIGN.md 3.8); f16 / bf16 are .noftz; f64 is exact IEEE; the integer types wrap.
// Max / min / bitwise: integers take the hardware's signed min / max and bitwise reductions and atomics. f16 / bf16 take the bulk, vector and vector-atomic
// max / min, whose maximumNumber / minimumNumber semantics (NaN ignored, -0 < +0, nothing flushed) were measured on H100
// (DESIGN.md 3.11); there is no scalar 16-bit max / min, so their ragged ends take a compare-and-swap loop on the aligned
// word. f32 and f64 have no max / min atomic in any form: every element takes a compare-and-swap loop, and the bulk
// reduction's pieces fall back to the cooperative drain (red_bulk).
__device__ __forceinline__ bool red_bulk(int t, int op) { return op == DDSK_OP_SUM || (t != DDSK_ACC_F32 && t != DDSK_ACC_F64); }
// maximumNumber (mx) / minimumNumber of the element bits c and operand bits o of a W-bit float (inf: its +inf bits):
// a NaN operand leaves c, a NaN c takes o, else the larger / smaller by the total order of the bits (so -0 < +0, and
// subnormals compare exactly whatever the ftz mode). The result is always the bits of c or of o.
template <typename U, int W>
__device__ __forceinline__ U fpick(U c, U o, U inf, bool mx) {
    constexpr U S = (U)1 << (W - 1), M = S - 1;
    if ((o & M) > inf) return c;
    if ((c & M) > inf) return o;
    const U kc = (c & S) ? (~c & (S | M)) : (c | S), ko = (o & S) ? (~o & (S | M)) : (o | S); // order-preserving keys
    return (mx ? ko > kc : ko < kc) ? o : c;
}
// f32 / f64 max / min of one element: a compare-and-swap loop that leaves without one when the element stays (the load
// was the atomic step). Returns the previous value.
__device__ __forceinline__ uint32_t fmm32(char *d, uint32_t o, bool mx) {
    uint32_t cur;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(cur) : "l"(d) : "memory");
    while (true) {
        const uint32_t want = fpick<uint32_t, 32>(cur, o, 0x7f800000u, mx);
        if (want == cur) return cur;
        const uint32_t seen = atom_cas_b32(d, cur, want);
        if (seen == cur) return cur;
        cur = seen;
    }
}
__device__ __forceinline__ uint64_t fmm64(char *d, uint64_t o, bool mx) {
    uint64_t cur;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(cur) : "l"(d) : "memory");
    while (true) {
        const uint64_t want = fpick<uint64_t, 64>(cur, o, 0x7ff0000000000000ull, mx);
        if (want == cur) return cur;
        const uint64_t seen = atom_cas_b64(d, cur, want);
        if (seen == cur) return cur;
        cur = seen;
    }
}
// f16 / bf16 max / min of the 16-bit elements of the aligned word w that mask m selects (low half, high half or both),
// with the operands at the same positions of o: cas_word's loop, which leaves the other half exactly as it finds it.
// Returns the word the step found.
__device__ __forceinline__ uint32_t fmm_word(char *w, uint32_t o, uint32_t m, bool bf, bool mx) {
    const uint32_t inf = bf ? 0x7f80u : 0x7c00u;
    uint32_t cur;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(cur) : "l"(w) : "memory");
    while (true) {
        uint32_t want = cur;
        if (m & 0xFFFFu) want = (want & 0xFFFF0000u) | fpick<uint32_t, 16>(cur & 0xFFFFu, o & 0xFFFFu, inf, mx);
        if (m >> 16) want = (want & 0xFFFFu) | fpick<uint32_t, 16>(cur >> 16, o >> 16, inf, mx) << 16;
        if (want == cur) return cur;
        const uint32_t seen = atom_cas_b32(w, cur, want);
        if (seen == cur) return cur;
        cur = seen;
    }
}
// integer reductions, without (red) and with (atom) the previous value
__device__ __forceinline__ void red_i32(char *d, uint32_t v, int op) {
    switch (op) {
    case DDSK_OP_MAX: asm volatile("red.relaxed.sys.global.max.s32 [%0], %1;" ::"l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_MIN: asm volatile("red.relaxed.sys.global.min.s32 [%0], %1;" ::"l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_BAND: asm volatile("red.relaxed.sys.global.and.b32 [%0], %1;" ::"l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_BOR: asm volatile("red.relaxed.sys.global.or.b32 [%0], %1;" ::"l"(d), "r"(v) : "memory"); break;
    default: asm volatile("red.relaxed.sys.global.xor.b32 [%0], %1;" ::"l"(d), "r"(v) : "memory"); break;
    }
}
__device__ __forceinline__ void red_i64(char *d, uint64_t v, int op) {
    switch (op) {
    case DDSK_OP_MAX: asm volatile("red.relaxed.sys.global.max.s64 [%0], %1;" ::"l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_MIN: asm volatile("red.relaxed.sys.global.min.s64 [%0], %1;" ::"l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_BAND: asm volatile("red.relaxed.sys.global.and.b64 [%0], %1;" ::"l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_BOR: asm volatile("red.relaxed.sys.global.or.b64 [%0], %1;" ::"l"(d), "l"(v) : "memory"); break;
    default: asm volatile("red.relaxed.sys.global.xor.b64 [%0], %1;" ::"l"(d), "l"(v) : "memory"); break;
    }
}
__device__ __forceinline__ uint32_t atom_i32(char *d, uint32_t v, int op) {
    uint32_t o;
    switch (op) {
    case DDSK_OP_MAX: asm volatile("atom.relaxed.sys.global.max.s32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_MIN: asm volatile("atom.relaxed.sys.global.min.s32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_BAND: asm volatile("atom.relaxed.sys.global.and.b32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory"); break;
    case DDSK_OP_BOR: asm volatile("atom.relaxed.sys.global.or.b32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory"); break;
    default: asm volatile("atom.relaxed.sys.global.xor.b32 %0, [%1], %2;" : "=r"(o) : "l"(d), "r"(v) : "memory"); break;
    }
    return o;
}
__device__ __forceinline__ uint64_t atom_i64(char *d, uint64_t v, int op) {
    uint64_t o;
    switch (op) {
    case DDSK_OP_MAX: asm volatile("atom.relaxed.sys.global.max.s64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_MIN: asm volatile("atom.relaxed.sys.global.min.s64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_BAND: asm volatile("atom.relaxed.sys.global.and.b64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory"); break;
    case DDSK_OP_BOR: asm volatile("atom.relaxed.sys.global.or.b64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory"); break;
    default: asm volatile("atom.relaxed.sys.global.xor.b64 %0, [%1], %2;" : "=l"(o) : "l"(d), "l"(v) : "memory"); break;
    }
    return o;
}
// shared -> global bulk reduction of op, dst[e] = op(dst[e], staged[e]): tma_store_1d's rules (16-byte aligned addresses
// and size) and bulk async-group (SASS: UBLKRED); red_bulk(t, op) holds
__device__ __forceinline__ void tma_red_1d(void *dst_gmem, uint32_t src_smem, uint32_t bytes, int t, int op) {
#define DDSK_BULK_RED(OPT)                                                                                                     \
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group." OPT " [%0], [%1], %2;" ::"l"(dst_gmem), "r"(src_smem), \
                 "r"(bytes)                                                                                                    \
                 : "memory")
    const bool w64 = t == DDSK_ACC_I64;
    switch (op) {
    case DDSK_OP_SUM:
        switch (t) {
        case DDSK_ACC_F32: DDSK_BULK_RED("add.f32"); break;
        case DDSK_ACC_F64: DDSK_BULK_RED("add.f64"); break;
        case DDSK_ACC_I32: DDSK_BULK_RED("add.u32"); break;
        case DDSK_ACC_I64: DDSK_BULK_RED("add.u64"); break;
        case DDSK_ACC_F16: DDSK_BULK_RED("add.noftz.f16"); break;
        default: DDSK_BULK_RED("add.noftz.bf16"); break;
        }
        break;
    case DDSK_OP_MAX:
        if (t == DDSK_ACC_I32) DDSK_BULK_RED("max.s32");
        else if (t == DDSK_ACC_I64) DDSK_BULK_RED("max.s64");
        else if (t == DDSK_ACC_F16) DDSK_BULK_RED("max.f16");
        else DDSK_BULK_RED("max.bf16");
        break;
    case DDSK_OP_MIN:
        if (t == DDSK_ACC_I32) DDSK_BULK_RED("min.s32");
        else if (t == DDSK_ACC_I64) DDSK_BULK_RED("min.s64");
        else if (t == DDSK_ACC_F16) DDSK_BULK_RED("min.f16");
        else DDSK_BULK_RED("min.bf16");
        break;
    case DDSK_OP_BAND:
        if (w64) DDSK_BULK_RED("and.b64");
        else DDSK_BULK_RED("and.b32");
        break;
    case DDSK_OP_BOR:
        if (w64) DDSK_BULK_RED("or.b64");
        else DDSK_BULK_RED("or.b32");
        break;
    default:
        if (w64) DDSK_BULK_RED("xor.b64");
        else DDSK_BULK_RED("xor.b32");
        break;
    }
#undef DDSK_BULK_RED
}
// The operand of red1v: the element staged at a shared address (red1), or its bits held in a register (Held). Each
// accessor reads it at one width (16, 32, 64 bits), at the point the reduction takes it.
struct Staged {
    uint32_t s;
    __device__ __forceinline__ unsigned short h() const { return lds16h(s); }
    __device__ __forceinline__ uint32_t w() const { return lds32(s); }
    __device__ __forceinline__ uint64_t l() const { return lds64(s); }
};
struct Held {
    uint64_t v;
    __device__ __forceinline__ unsigned short h() const { return (unsigned short)v; }
    __device__ __forceinline__ uint32_t w() const { return (uint32_t)v; }
    __device__ __forceinline__ uint64_t l() const { return v; }
};
// one element at d: *d = op(*d, o) (d aligned to the element size)
template <typename O>
__device__ __forceinline__ void red1v(char *d, O o, int t, int op) {
    if (op == DDSK_OP_SUM) {
        switch (t) {
        case DDSK_ACC_F32:
            asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(d), "f"(__uint_as_float(o.w())) : "memory");
            break;
        case DDSK_ACC_F64:
            asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(d), "d"(__longlong_as_double((long long)o.l())) : "memory");
            break;
        case DDSK_ACC_I32: asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(d), "r"(o.w()) : "memory"); break;
        case DDSK_ACC_I64: asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(d), "l"(o.l()) : "memory"); break;
        case DDSK_ACC_F16: asm volatile("red.relaxed.sys.global.add.noftz.f16 [%0], %1;" ::"l"(d), "h"(o.h()) : "memory"); break;
        default: asm volatile("red.relaxed.sys.global.add.noftz.bf16 [%0], %1;" ::"l"(d), "h"(o.h()) : "memory"); break;
        }
        return;
    }
    const bool mx = op == DDSK_OP_MAX;
    switch (t) {
    case DDSK_ACC_I32: red_i32(d, o.w(), op); break;
    case DDSK_ACC_I64: red_i64(d, o.l(), op); break;
    case DDSK_ACC_F32: fmm32(d, o.w(), mx); break;
    case DDSK_ACC_F64: fmm64(d, o.l(), mx); break;
    default: {
        const uint32_t sh = ((uint32_t)(uint64_t)d & 2u) * 8u;
        fmm_word((char *)((uint64_t)d & ~(uint64_t)3), (uint32_t)o.h() << sh, 0xFFFFu << sh, t == DDSK_ACC_BF16, mx);
        break;
    }
    }
}
// one element at d: *d = op(*d, the element staged at shared address s) (both aligned to the element size)
__device__ __forceinline__ void red1(char *d, uint32_t s, int t, int op) { red1v(d, Staged{s}, t, op); }
// 16 bytes at a 16-byte aligned d, element-wise: *d = op(*d, v)
__device__ __forceinline__ void red16(char *d, uint4 v, int t, int op) {
    if (op == DDSK_OP_SUM) {
        switch (t) {
        case DDSK_ACC_F32:
            asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(d), "f"(__uint_as_float(v.x)),
                         "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
            break;
        case DDSK_ACC_F64:
            asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(d), "d"(__hiloint2double((int)v.y, (int)v.x)) : "memory");
            asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(d + 8), "d"(__hiloint2double((int)v.w, (int)v.z)) : "memory");
            break;
        case DDSK_ACC_I32:
            asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(d), "r"(v.x) : "memory");
            asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(d + 4), "r"(v.y) : "memory");
            asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(d + 8), "r"(v.z) : "memory");
            asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(d + 12), "r"(v.w) : "memory");
            break;
        case DDSK_ACC_I64:
            asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(d), "l"((uint64_t)v.y << 32 | v.x) : "memory");
            asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(d + 8), "l"((uint64_t)v.w << 32 | v.z) : "memory");
            break;
        case DDSK_ACC_F16:
            asm volatile("red.relaxed.sys.global.add.noftz.v4.f16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z),
                         "r"(v.w) : "memory");
            break;
        default:
            asm volatile("red.relaxed.sys.global.add.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z),
                         "r"(v.w) : "memory");
            break;
        }
        return;
    }
    const bool mx = op == DDSK_OP_MAX;
    switch (t) {
    case DDSK_ACC_I32:
        red_i32(d, v.x, op);
        red_i32(d + 4, v.y, op);
        red_i32(d + 8, v.z, op);
        red_i32(d + 12, v.w, op);
        break;
    case DDSK_ACC_I64:
        red_i64(d, (uint64_t)v.y << 32 | v.x, op);
        red_i64(d + 8, (uint64_t)v.w << 32 | v.z, op);
        break;
    case DDSK_ACC_F32:
        fmm32(d, v.x, mx);
        fmm32(d + 4, v.y, mx);
        fmm32(d + 8, v.z, mx);
        fmm32(d + 12, v.w, mx);
        break;
    case DDSK_ACC_F64:
        fmm64(d, (uint64_t)v.y << 32 | v.x, mx);
        fmm64(d + 8, (uint64_t)v.w << 32 | v.z, mx);
        break;
    case DDSK_ACC_F16:
        if (mx) asm volatile("red.relaxed.sys.global.max.noftz.v4.f16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        else asm volatile("red.relaxed.sys.global.min.noftz.v4.f16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        break;
    default:
        if (mx) asm volatile("red.relaxed.sys.global.max.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        else asm volatile("red.relaxed.sys.global.min.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        break;
    }
}
// The fetch forms of red1 and red16, and the swap (DDSK_OP_REPLACE: shard = operand, on elements of 1 << el bytes).
// One element at d: the operand staged at shared address s is replaced by the element's previous value (both aligned to
// the element size).
__device__ __forceinline__ void fetch1(char *d, uint32_t s, int t, int op, uint32_t el) {
    if (op == DDSK_OP_REPLACE) {
        switch (el) {
        case 3: sts64(s, atom_exch_b64(d, lds64(s))); break;
        case 2: sts32(s, atom_exch_b32(d, lds32(s))); break;
        default: sts16(s, atom_exch_b16(d, lds16h(s))); break;
        }
        return;
    }
    if (op == DDSK_OP_SUM) {
        switch (t) {
        case DDSK_ACC_F32: {
            float o;
            asm volatile("atom.relaxed.sys.global.add.f32 %0, [%1], %2;" : "=f"(o) : "l"(d), "f"(__uint_as_float(lds32(s))) : "memory");
            sts32(s, __float_as_uint(o));
            break;
        }
        case DDSK_ACC_F64: sts64(s, atom_add_f64(d, lds64(s))); break;
        case DDSK_ACC_I32: sts32(s, atom_add_u32(d, lds32(s))); break;
        case DDSK_ACC_I64: sts64(s, atom_add_u64(d, lds64(s))); break;
        case DDSK_ACC_F16: {
            unsigned short o;
            asm volatile("atom.relaxed.sys.global.add.noftz.f16 %0, [%1], %2;" : "=h"(o) : "l"(d), "h"(lds16h(s)) : "memory");
            sts16(s, o);
            break;
        }
        default: {
            unsigned short o;
            asm volatile("atom.relaxed.sys.global.add.noftz.bf16 %0, [%1], %2;" : "=h"(o) : "l"(d), "h"(lds16h(s)) : "memory");
            sts16(s, o);
            break;
        }
        }
        return;
    }
    const bool mx = op == DDSK_OP_MAX;
    switch (t) {
    case DDSK_ACC_I32: sts32(s, atom_i32(d, lds32(s), op)); break;
    case DDSK_ACC_I64: sts64(s, atom_i64(d, lds64(s), op)); break;
    case DDSK_ACC_F32: sts32(s, fmm32(d, lds32(s), mx)); break;
    case DDSK_ACC_F64: sts64(s, fmm64(d, lds64(s), mx)); break;
    default: {
        const uint32_t sh = ((uint32_t)(uint64_t)d & 2u) * 8u;
        sts16(s, fmm_word((char *)((uint64_t)d & ~(uint64_t)3), (uint32_t)lds16h(s) << sh, 0xFFFFu << sh, t == DDSK_ACC_BF16,
                          mx) >> sh);
        break;
    }
    }
}
// 16 bytes at a 16-byte aligned d: the operands v, element-wise; returns the previous 16 bytes
__device__ __forceinline__ uint4 fetch16(char *d, uint4 v, int t, int op, uint32_t el) {
    uint4 o;
    if (op == DDSK_OP_REPLACE) {
        if (el == 3) {
            const uint64_t a = atom_exch_b64(d, (uint64_t)v.y << 32 | v.x), b = atom_exch_b64(d + 8, (uint64_t)v.w << 32 | v.z);
            o = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
        } else { // (a 32-bit exchange is atomic for each 16-bit element it holds)
            o = make_uint4(atom_exch_b32(d, v.x), atom_exch_b32(d + 4, v.y), atom_exch_b32(d + 8, v.z), atom_exch_b32(d + 12, v.w));
        }
        return o;
    }
    if (op == DDSK_OP_SUM) {
        switch (t) {
        case DDSK_ACC_F32:
            asm volatile("atom.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                         : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
            break;
        case DDSK_ACC_F64: {
            const uint64_t a = atom_add_f64(d, (uint64_t)v.y << 32 | v.x), b = atom_add_f64(d + 8, (uint64_t)v.w << 32 | v.z);
            o = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
            break;
        }
        case DDSK_ACC_I32:
            o = make_uint4(atom_add_u32(d, v.x), atom_add_u32(d + 4, v.y), atom_add_u32(d + 8, v.z), atom_add_u32(d + 12, v.w));
            break;
        case DDSK_ACC_I64: {
            const uint64_t a = atom_add_u64(d, (uint64_t)v.y << 32 | v.x), b = atom_add_u64(d + 8, (uint64_t)v.w << 32 | v.z);
            o = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
            break;
        }
        case DDSK_ACC_F16:
            asm volatile("atom.relaxed.sys.global.add.noftz.v4.f16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                         : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
            break;
        default:
            asm volatile("atom.relaxed.sys.global.add.noftz.v4.bf16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                         : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
            break;
        }
        return o;
    }
    const bool mx = op == DDSK_OP_MAX;
    switch (t) {
    case DDSK_ACC_I32:
        o = make_uint4(atom_i32(d, v.x, op), atom_i32(d + 4, v.y, op), atom_i32(d + 8, v.z, op), atom_i32(d + 12, v.w, op));
        break;
    case DDSK_ACC_I64: {
        const uint64_t a = atom_i64(d, (uint64_t)v.y << 32 | v.x, op), b = atom_i64(d + 8, (uint64_t)v.w << 32 | v.z, op);
        o = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
        break;
    }
    case DDSK_ACC_F32: o = make_uint4(fmm32(d, v.x, mx), fmm32(d + 4, v.y, mx), fmm32(d + 8, v.z, mx), fmm32(d + 12, v.w, mx)); break;
    case DDSK_ACC_F64: {
        const uint64_t a = fmm64(d, (uint64_t)v.y << 32 | v.x, mx), b = fmm64(d + 8, (uint64_t)v.w << 32 | v.z, mx);
        o = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
        break;
    }
    case DDSK_ACC_F16:
        if (mx)
            asm volatile("atom.relaxed.sys.global.max.noftz.v4.f16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w) : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        else
            asm volatile("atom.relaxed.sys.global.min.noftz.v4.f16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w) : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        break;
    default:
        if (mx)
            asm volatile("atom.relaxed.sys.global.max.noftz.v4.bf16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w) : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        else
            asm volatile("atom.relaxed.sys.global.min.noftz.v4.bf16x2 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                         : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w) : "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        break;
    }
    return o;
}
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
// PUT (a batched put): an invalid request keeps its bytes in the caller's layout -- count * row_bytes when 0 < count <=
// the variable's rows, 0 otherwise and for a sample id outside the index -- with source address 0 (nothing is written).
template <int K, bool PUT = false>
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
            if constexpr (PUT) {
                const int64_t rows = vp[k]->lenlist[vp[k]->nranks - 1];
                nbytes[k] = count[k] > 0 && count[k] <= rows ? count[k] * vp[k]->row_bytes : 0;
            }
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

// What a gather launch does with its pieces (dds_gather_kernel's WR): a get, or a batched write (GatherArgs::wr) that
// stores them (a put), reduces them into the shard (an accumulate) or applies a returning atomic (a fetch-op, the
// compare-and-swap included)
constexpr int kWrNone = 0, kWrPut = 1, kWrReduce = 2, kWrFetch = 3;

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
    char *dst;            // the packed buffer (a put: the caller's packed SOURCE rows, only read)
    int64_t dst_cap;      // its size in bytes
    int64_t *offsets_out; // optional [nreq+1]
    unsigned long long *status;
    unsigned long long status_tag; // this launch's ordinal in its queue, as OR-ed into every status report
    unsigned int *counters; // [0] segment ticket, [1] finished warps -- self-resetting, ticketed launches only
    union { // (a launch is never both: the union keeps the parameter block, and the conversion behind it, where they were)
        struct { // multi-array batches (plan.nvars > 1): the packed result of variable v goes to mdst[v]
            char *mdst[DDSK_MAX_MULTI];
            int64_t mcap[DDSK_MAX_MULTI];
            int64_t *moffsets[DDSK_MAX_MULTI]; // optional per-variable [per_var + 1] byte offsets
        };
        struct { // padded batches (PAD). Request i = the plan's (start, count) of index i; its slot is pad_slot source
                 // bytes (count = max_rows). See ddsk_pad_cut in kernels.h.
            int64_t pad_slot;
            uint64_t pad_bits;
            int pad_log2, pad_in_log2, pad_out_log2; // output element size; source -> output position shifts
            int64_t *pad_lengths;                    // optional [nreq] delivered row counts
        };
        ddsk_write_t wr; // batched writes (WR != kWrNone): neither padded nor multi-array. op and type are warp-uniform.
    };
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

// ---- padded batches: request lookup and padding fill
// (start, count) of request idx through the plan's index (explicit arrays or the sample table), validated on the FULL
// count (errors reported); -> source address (0: invalid) and payload bytes min(count, max_rows) * row_bytes
__device__ __forceinline__ void pad_lookup(const GatherArgs &a, int64_t idx, uint64_t &src, int64_t &payload) {
    const int64_t ix[1] = {idx};
    uint64_t s[1];
    int64_t nbytes[1];
    plan_many<1>(a.var, a.plan, ix, a.nreq, a.status, a.status_tag, s, nbytes);
    src = s[0];
    payload = min(nbytes[0], a.pad_slot);
}

// the 16-byte pattern of a padding element of 1 << el bytes (dst positions are aligned to the element, so every aligned
// 16-byte vector of padding holds this pattern)
__device__ __forceinline__ uint4 pad_pattern(uint64_t bits, int el) {
    uint32_t lo, hi;
    if (el == 0) lo = hi = (uint32_t)(bits & 0xFFu) * 0x01010101u;
    else if (el == 1) lo = hi = (uint32_t)(bits & 0xFFFFu) * 0x00010001u;
    else if (el == 2) lo = hi = (uint32_t)bits;
    else {
        lo = (uint32_t)bits;
        hi = (uint32_t)(bits >> 32);
    }
    return make_uint4(lo, hi, lo, hi);
}
__device__ __forceinline__ void pad_store1(char *d, uint64_t bits, int el) {
    if (el == 0) *(uint8_t *)d = (uint8_t)bits;
    else if (el == 1) *(uint16_t *)d = (uint16_t)bits;
    else if (el == 2) *(uint32_t *)d = (uint32_t)bits;
    else *(uint64_t *)d = bits;
}
// the whole warp writes n bytes (whole elements) of padding at d: element-wise head up to the first 16-byte boundary,
// aligned 128-bit stores, element-wise tail
__device__ __forceinline__ void pad_fill(char *d, int64_t n, uint64_t bits, int el, int lane) {
    int64_t head = (16 - (int64_t)((uint64_t)d & 15u)) & 15;
    if (head > n) head = n;
    const int64_t nv = (n - head) >> 4;
    const int64_t tail = n - head - (nv << 4);
    if ((int64_t)lane < (head >> el)) pad_store1(d + ((int64_t)lane << el), bits, el);
    const uint4 v = pad_pattern(bits, el);
    char *dv = d + head;
    for (int64_t j = lane; j < nv; j += 32) stg128(dv + (j << 4), v);
    if ((int64_t)lane < (tail >> el)) pad_store1(dv + (nv << 4) + ((int64_t)lane << el), bits, el);
}

// VALIGN (converting multi-array launches): segment boundaries are aligned down to 8 bytes relative to the variable
// they fall in (vb[]: the variables' starts in the concatenated packed space), so that no segment cuts a source element
// of a variable that starts at an odd offset
// PAD (padded batches, with FIXED): slot i of the walk holds request i's payload followed by padding; the walk copies the
// payload and each warp fills the padding of the segments it claims
// PUT (batched puts): the same walk with the roles of the two addresses swapped: a piece's src is its packed position in
// a.dst (the caller's rows, where the TMA load reads, so the stage offsets follow that address's 16-byte phase) and its
// dpos the shard address its drain writes
template <bool FIXED, int CH, int PCAP, bool VALIGN = false, bool PAD = false, bool PUT = false>
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
    bool valign = false;
    int64_t vb[VALIGN ? DDSK_MAX_MULTI : 1];
    // per-lane window of 32 request descriptors
    uint64_t w_src = 0;
    int64_t w_dst = 0, w_n = 0;
    uint64_t w_shard; // PUT: the request's shard address (w_src is then its packed position in the caller's buffer)

    __device__ __forceinline__ void load_window(const GatherArgs &a, int lane) {
        win_base = r;
        int64_t idx = r + lane;
        w_src = 0;
        w_dst = 0;
        w_n = 0;
        if (idx < nreq) {
            if constexpr (PAD) {
                int64_t payload;
                pad_lookup(a, idx, w_src, payload);
                w_dst = idx * nb; // the slot's start in the padded source space
                w_n = payload;    // (the rest of the slot is padding: no piece covers it)
            } else if (FIXED && push_n > 0) {
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
            if constexpr (PUT) { // the pieces load from the caller's rows and are written to the shard
                w_shard = w_src;
                w_src = w_src ? (uint64_t)a.dst + (uint64_t)w_dst : 0;
            }
        }
    }

    __device__ __forceinline__ int64_t align_to_var(int64_t pos) const {
        int64_t b = vb[0];
#pragma unroll
        for (int k = 1; k < (VALIGN ? DDSK_MAX_MULTI : 1); k++)
            if (pos >= vb[k]) b = vb[k];
        return b + ((pos - b) & ~(int64_t)7);
    }

    // largest r in [0, nreq) with dst[r] <= pos
    __device__ __forceinline__ int64_t locate_var(const GatherArgs &a, int64_t pos, int lane) {
        if constexpr (VALIGN && PCAP == 0) {
            if (valign) { // pos lies at most 7 bytes below a SEG_GRAIN boundary (that of the segment's nominal start)
                int64_t r0 = (int64_t)__ldcg(&a.seg_tab[(pos + 7) / SEG_GRAIN]);
                while (r0 > 0 && pv.d(r0) > pos) r0--;
                return r0;
            }
        }
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

    // PAD: write the padding of every slot the new segment [seg_pos, seg_end) covers, clipped to it, 32 slots at a time
    // (one lookup per lane), each region by the whole warp. Padding is caller-visible: the overlap gate opens first.
    template <typename Gate>
    __device__ __forceinline__ void fill_pads(const GatherArgs &a, int lane, Gate &&gate) {
        const int64_t i_end = min(nreq, (seg_end + nb - 1) / nb);
        for (int64_t i0 = seg_pos / nb; i0 < i_end; i0 += 32) {
            const int64_t i = i0 + lane;
            int64_t pad_dst = 0, pad_len = 0;
            if (i < i_end) {
                uint64_t src;
                int64_t payload;
                pad_lookup(a, i, src, payload);
                const ddsk_pad_cut_t c = ddsk_pad_cut(i, payload, nb, max(seg_pos - i * nb, (int64_t)0),
                                                      min(seg_end - i * nb, nb), a.pad_in_log2, a.pad_out_log2);
                pad_dst = c.pad_dst;
                pad_len = c.pad_len;
            }
            unsigned todo = __ballot_sync(0xffffffffu, pad_len > 0);
            if (todo) gate();
            while (todo) {
                const int j = __ffs(todo) - 1;
                todo &= todo - 1;
                pad_fill(a.dst + __shfl_sync(0xffffffffu, pad_dst, j), __shfl_sync(0xffffffffu, pad_len, j), a.pad_bits,
                         a.pad_log2, lane);
            }
        }
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
                if constexpr (VALIGN) {
                    if (valign) {
                        seg_pos = align_to_var(seg_pos);
                        if (seg_end < T) seg_end = align_to_var(seg_end);
                        if (seg_pos >= seg_end) continue; // (an empty segment)
                    }
                }
                r = FIXED ? seg_pos / nb : locate_var(a, seg_pos, lane);
                if constexpr (PAD) fill_pads(a, lane, gate);
            }
            // (PAD: the rest of the segment, if any, is the padding fill_pads wrote)
            if (r >= nreq || (PAD && r * nb >= seg_end)) { // defensive without PAD: cannot happen while seg_pos < T
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
                    if constexpr (PUT) pc.dpos = (int64_t)(__shfl_sync(0xffffffffu, w_shard, wl) + (uint64_t)(p0 - d0));
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
            if constexpr (PUT) pc.dpos = (int64_t)(__shfl_sync(0xffffffffu, w_shard, srcl & 31) + (uint64_t)(p0 - q_d0));
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

// The batched writes' drain: what write_chunk does to each element and each re-phased 16-byte vector of a piece.
// kActReduce: combine it with the shard's (red1 / red16; tma_red_1d for a same-phase body). kActFetch: combine it by a
// returning atomic (fetch1 / fetch16) and put the previous value back in the stage, over the operand. kActCas: the same
// with cas1 / cas16 and the piece's compare operands.
constexpr int kActReduce = 0, kActFetch = 1, kActCas = 2;

// Operand vector j of a piece's body: rephase_loop's shift of the staged bytes. (rephase_loop keeps its own copy: the
// get instantiations' register allocation changed when a loop was shared with the writes.)
template <int WS, bool BYTES>
__device__ __forceinline__ uint4 rephased(uint32_t sbase, uint32_t j, uint32_t bs8) {
    const uint4 lo = lds128(sbase + (j << 4));
    const uint4 hi = lds128(sbase + (j << 4) + 16);
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    uint4 v;
    if (BYTES) {
        v.x = __funnelshift_r(w[WS + 0], w[WS + 1], bs8);
        v.y = __funnelshift_r(w[WS + 1], w[WS + 2], bs8);
        v.z = __funnelshift_r(w[WS + 2], w[WS + 3], bs8);
        v.w = __funnelshift_r(w[WS + 3], w[WS + 4], bs8);
    } else {
        v = make_uint4(w[WS + 0], w[WS + 1], w[WS + 2], w[WS + 3]);
    }
    return v;
}

// ACT applied to operand vector j, for j = lane, lane + 32, .. < nv: the shard's 16 bytes at dv + 16j. The fetch forms
// write the previous 16 bytes back over the operand's staged bytes at s + 16j with stores that touch exactly them (the
// neighbouring vectors are other lanes'): a fetch-op's elements are 2, 4 or 8 bytes (s is then 0 or 2 mod 4), a
// compare-and-swap's may be single bytes (any phase). A compare-and-swap reads compare vector j at cv + 16j, in the
// compare buffer's own phase.
template <int ACT, int WS, bool BYTES>
__device__ __forceinline__ void write_loop(uint32_t sbase, uint32_t s, char *dv, const char *cv, uint32_t nv, uint32_t bs8,
                                           int lane, int t, int op, uint32_t el) {
#pragma unroll(ACT == kActCas ? 2 : 4)
    for (uint32_t j = (uint32_t)lane; j < nv; j += 32) {
        const uint4 v = rephased<WS, BYTES>(sbase, j, bs8);
        char *const d = dv + ((size_t)j << 4);
        const uint32_t p = s + (j << 4);
        if constexpr (ACT == kActReduce) {
            red16(d, v, t, op);
        } else if constexpr (ACT == kActFetch) {
            const uint4 o = fetch16(d, v, t, op, el);
            if (!BYTES && WS == 0) {
                sts128(p, o);
            } else if (!BYTES) {
                sts32(p, o.x);
                sts32(p + 4, o.y);
                sts32(p + 8, o.z);
                sts32(p + 12, o.w);
            } else {
                sts16(p, o.x);
                sts32(p + 2, __funnelshift_r(o.x, o.y, 16));
                sts32(p + 6, __funnelshift_r(o.y, o.z, 16));
                sts32(p + 10, __funnelshift_r(o.z, o.w, 16));
                sts16(p + 14, o.w >> 16);
            }
        } else {
            const uint4 o = cas16(d, v, ldg16_any(cv + ((size_t)j << 4)), el);
            if (!BYTES && WS == 0) sts128(p, o);
            else sts16_any(p, o);
        }
    }
}

// ACT applied to the element of 1 << el bytes at d + k, its operand staged at shared address s + k (and its compare
// operand at c + k)
template <int ACT>
__device__ __forceinline__ void write1(char *d, uint32_t s, const char *c, uint32_t k, int t, int op, uint32_t el) {
    if constexpr (ACT == kActReduce) red1(d + k, s + k, t, op);
    else if constexpr (ACT == kActFetch) fetch1(d + k, s + k, t, op, el);
    else cas1(d + k, s + k, c + k, el);
}

// A batched write's drain of one staged piece (payload byte k at shared address sb + a + k, shard byte d[k], compare
// operand c[k] for kActCas), drain_chunk's cut in the shard's 16-byte phase: the head and tail, below 16 bytes, element
// by element on the first lanes (write1), the body as 16-byte vectors re-phased from the stage (write_loop). A reduction
// whose body shares the stage's phase, and whose op has a bulk form for t (red_bulk), bulk-reduces it from lane 0
// instead; no bulk form returns the old values. A piece never cuts an element and the caller's rows are element-aligned
// (see cvt_in_log2), so head, body and tail are whole, aligned elements. After a fetch form the caller drains the stage,
// now the previous values, to the result with the raw drain.
template <int ACT>
__device__ __forceinline__ void write_chunk(uint32_t sb, uint32_t a, char *d, const char *c, uint32_t n, int lane, int t,
                                            int op, uint32_t el) {
    uint32_t head = (16u - (uint32_t)((uint64_t)d & 15u)) & 15u;
    if (head > n) head = n;
    const uint32_t nv = (n - head) >> 4;
    const uint32_t tail = n - head - (nv << 4);
    const uint32_t s = a + head;
    const uint32_t sh = s & 15u;
    if (nv) {
        if (ACT == kActReduce && sh == 0 && red_bulk(t, op)) {
            if (lane == 0) {
                fence_proxy_async();
                tma_red_1d(d + head, sb + s, nv << 4, t, op);
            }
        } else {
            const uint32_t sbase = sb + (s & ~15u);
            const uint32_t bs8 = (sh & 3u) * 8u;
            char *dv = d + head;
            const char *cv = ACT == kActCas ? c + head : nullptr;
            switch ((sh >> 2) * 2u + (bs8 ? 1u : 0u)) { // warp-uniform (2-byte elements: bs8 is 0 or 16)
            case 0: write_loop<ACT, 0, false>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 1: write_loop<ACT, 0, true>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 2: write_loop<ACT, 1, false>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 3: write_loop<ACT, 1, true>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 4: write_loop<ACT, 2, false>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 5: write_loop<ACT, 2, true>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            case 6: write_loop<ACT, 3, false>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            default: write_loop<ACT, 3, true>(sbase, sb + s, dv, cv, nv, bs8, lane, t, op, el); break;
            }
        }
    }
    if ((uint32_t)lane < (head >> el)) {
        write1<ACT>(d, sb + a, c, (uint32_t)lane << el, t, op, el);
    }
    if ((uint32_t)lane < (tail >> el)) {
        write1<ACT>(d, sb + a, c, head + (nv << 4) + ((uint32_t)lane << el), t, op, el);
    }
}

// ------------------------------------------------------------------------------------------------
// Converting drain (DDSK_CVT_*): the load side of the walk is unchanged, the staged SOURCE elements are converted on the
// way out of shared memory. Source byte p of a variable's packed rows goes to output byte (p >> IL) << OL; the ratio is
// a power of two, so every position is a shift.
// Invariant relied on here: a staged piece never cuts a source element. The walk cuts only at request boundaries
// (multiples of the row size, itself a multiple of the itemsize), at segment boundaries (multiples of CH, SEG_GRAIN or
// of a whole fixed-count request) and at CH bytes -- CH and SEG_GRAIN are multiples of 8, and itemsizes are 1, 4 or 8.
// Source elements are therefore also aligned to their size in shared memory (stage offsets are 16-byte aligned and
// source rows start at itemsize-aligned addresses).
// ------------------------------------------------------------------------------------------------
// (NORM: the codes may include the normalising ones; launches without them evaluate the tables of codes 0..5 only)
template <bool NORM = false>
__host__ __device__ constexpr int cvt_in_log2(int code) {
    if constexpr (NORM) return DDSK_CVT_IN_LOG2(code);
    else return DDSK_CVT_PLAIN_IN_LOG2(code);
}
template <bool NORM = false>
__host__ __device__ constexpr int cvt_out_log2(int code) {
    if constexpr (NORM) return DDSK_CVT_OUT_LOG2(code);
    else return DDSK_CVT_PLAIN_OUT_LOG2(code);
}
template <bool NORM = false>
__device__ __forceinline__ int64_t cvt_scale(int64_t p, int code) { return (p >> cvt_in_log2<NORM>(code)) << cvt_out_log2<NORM>(code); }

__device__ __forceinline__ uint32_t cvt2_bf16(float lo, float hi) { // packs (lo, hi) -> [15:0] lo, [31:16] hi
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ uint32_t cvt2_f16(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ uint32_t cvt_f32_of_f64(uint64_t bits) {
    float f;
    asm("cvt.rn.f32.f64 %0, %1;" : "=f"(f) : "d"(__longlong_as_double((long long)bits)));
    return __float_as_uint(f);
}
__device__ __forceinline__ uint32_t lds16(uint32_t addr) {
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lut16(uint32_t lut, uint32_t b) { return lds16(lut + (b << 1)); }
__device__ __forceinline__ uint32_t lut32(uint32_t lut, uint32_t b) { return lds32(lut + (b << 2)); }

// one element: source at shared address s, output at d
template <int CODE>
__device__ __forceinline__ void cvt_one(uint32_t s, char *d, uint32_t lut) {
    if constexpr (CODE == DDSK_CVT_F32_BF16 || CODE == DDSK_CVT_F32_F16) {
        const float f = __uint_as_float(lds32(s));
        const uint32_t w = CODE == DDSK_CVT_F32_BF16 ? cvt2_bf16(f, 0.0f) : cvt2_f16(f, 0.0f);
        *(uint16_t *)d = (uint16_t)(w & 0xFFFFu);
    } else if constexpr (CODE == DDSK_CVT_F64_F32) {
        *(uint32_t *)d = cvt_f32_of_f64(lds64(s));
    } else if constexpr (CODE == DDSK_CVT_U8_LUT16) {
        *(uint16_t *)d = (uint16_t)lut16(lut, lds8(s));
    } else {
        *(uint32_t *)d = lut32(lut, lds8(s));
    }
}

// one 16-byte output vector from the source elements at shared address s (VEC: s is aligned for vector loads)
template <int CODE, bool VEC>
__device__ __forceinline__ uint4 cvt_vec(uint32_t s, uint32_t lut) {
    uint4 o;
    if constexpr (CODE == DDSK_CVT_F32_BF16 || CODE == DDSK_CVT_F32_F16) { // 8 floats (32 B) -> 8 halves
        uint32_t w[8];
        if (VEC) {
            const uint4 a = lds128(s), b = lds128(s + 16);
            w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) w[k] = lds32(s + 4u * k);
        }
        uint32_t r[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
            r[k] = CODE == DDSK_CVT_F32_BF16 ? cvt2_bf16(__uint_as_float(w[2 * k]), __uint_as_float(w[2 * k + 1]))
                                             : cvt2_f16(__uint_as_float(w[2 * k]), __uint_as_float(w[2 * k + 1]));
        o = make_uint4(r[0], r[1], r[2], r[3]);
    } else if constexpr (CODE == DDSK_CVT_F64_F32) { // 4 doubles (32 B) -> 4 floats
        uint64_t q[4];
        if (VEC) {
            const uint4 a = lds128(s), b = lds128(s + 16);
            q[0] = (uint64_t)a.y << 32 | a.x; q[1] = (uint64_t)a.w << 32 | a.z;
            q[2] = (uint64_t)b.y << 32 | b.x; q[3] = (uint64_t)b.w << 32 | b.z;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = lds64(s + 8u * k);
        }
        o = make_uint4(cvt_f32_of_f64(q[0]), cvt_f32_of_f64(q[1]), cvt_f32_of_f64(q[2]), cvt_f32_of_f64(q[3]));
    } else if constexpr (CODE == DDSK_CVT_U8_LUT16) { // 8 bytes -> 8 table entries of 2 bytes
        uint32_t b[8];
        if (VEC) {
            const uint64_t v = lds64(s);
#pragma unroll
            for (int k = 0; k < 8; k++) b[k] = (uint32_t)(v >> (8 * k)) & 0xFFu;
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) b[k] = lds8(s + k);
        }
        uint32_t r[4];
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = lut16(lut, b[2 * k]) | (lut16(lut, b[2 * k + 1]) << 16);
        o = make_uint4(r[0], r[1], r[2], r[3]);
    } else { // LUT32: 4 bytes -> 4 table entries of 4 bytes
        uint32_t b[4];
        if (VEC) {
            const uint32_t v = lds32(s);
#pragma unroll
            for (int k = 0; k < 4; k++) b[k] = (v >> (8 * k)) & 0xFFu;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) b[k] = lds8(s + k);
        }
        o = make_uint4(lut32(lut, b[0]), lut32(lut, b[1]), lut32(lut, b[2]), lut32(lut, b[3]));
    }
    return o;
}

// Drain one staged piece converted: n source bytes at shared address s0 (whole elements) go to d (aligned to the output
// itemsize). Element-wise head up to the first 16-byte boundary of d, aligned 128-bit stores, element-wise tail.
template <int CODE>
__device__ __forceinline__ void cvt_drain(uint32_t s0, char *d, uint32_t n, uint32_t lut, int lane) {
    constexpr int IL = cvt_in_log2(CODE), OL = cvt_out_log2(CODE);
    constexpr uint32_t E = 16u >> OL;                              // elements per output vector
    constexpr uint32_t VA = (E << IL) < 16u ? (E << IL) : 16u;     // source alignment of the vector loads
    const uint32_t ne = n >> IL;
    uint32_t head = ((16u - (uint32_t)((uint64_t)d & 15u)) & 15u) >> OL;
    if (head > ne) head = ne;
    const uint32_t nv = (ne - head) / E;
    const uint32_t tail = ne - head - nv * E;
    const uint32_t sb = s0 + (head << IL);
    char *dv = d + (head << OL);
    if ((sb & (VA - 1u)) == 0) { // warp-uniform
#pragma unroll 2
        for (uint32_t j = (uint32_t)lane; j < nv; j += 32) stg128(dv + ((size_t)j << 4), cvt_vec<CODE, true>(sb + j * (E << IL), lut));
    } else {
#pragma unroll 2
        for (uint32_t j = (uint32_t)lane; j < nv; j += 32) stg128(dv + ((size_t)j << 4), cvt_vec<CODE, false>(sb + j * (E << IL), lut));
    }
    if ((uint32_t)lane < head) cvt_one<CODE>(s0 + ((uint32_t)lane << IL), d + ((uint32_t)lane << OL), lut);
    if ((uint32_t)lane < tail) {
        const uint32_t k = head + nv * E + (uint32_t)lane;
        cvt_one<CODE>(s0 + (k << IL), d + ((size_t)k << OL), lut);
    }
}

// ------------------------------------------------------------------------------------------------
// Normalising drain (DDSK_CVT_NORM_*): y = __fdiv_rn(__fsub_rn(decode(x), mean[ch]), std[ch]), then encoded -- explicit
// IEEE roundings, so the result does not depend on contraction flags. Channel of element e of a variable's packed rows:
// (e mod (nchan * inner)) / inner -- every request starts at a row boundary and nchan * inner divides the row. It is
// found once per piece (one 64-bit remainder) and per lane (32-bit), then advanced incrementally element by element.
// The {mean, std} pairs are read with ld.global.nc: nchan * 8 bytes that stay in L1 / L2.
// ------------------------------------------------------------------------------------------------
// source (0 f32, 1 f64, 2 uint8 through the f32 table) and output (0 f32, 1 bf16, 2 f16) of a normalising code
__host__ __device__ constexpr int norm_src(int code) { return code == DDSK_CVT_NORM_F64_F32 ? 1 : code >= DDSK_CVT_NORM_U8_F32 ? 2 : 0; }
__host__ __device__ constexpr int norm_out(int code) {
    return (code == DDSK_CVT_NORM_F32_BF16 || code == DDSK_CVT_NORM_U8_BF16) ? 1
         : (code == DDSK_CVT_NORM_F32_F16 || code == DDSK_CVT_NORM_U8_F16)  ? 2 : 0;
}

// position inside the channel pattern: channel ch, element in of its run of `inner`
struct ChanPos {
    uint32_t ch, in;
    __device__ __forceinline__ void step(uint32_t nchan, uint32_t inner) {
        if (++in == inner) {
            in = 0;
            if (++ch == nchan) ch = 0;
        }
    }
    // forward by dq * inner + dr elements (dq < nchan, dr < inner)
    __device__ __forceinline__ void advance(uint32_t dq, uint32_t dr, uint32_t nchan, uint32_t inner) {
        uint32_t c = ch + dq;
        in += dr;
        if (in >= inner) {
            in -= inner;
            c++;
        }
        ch = c >= nchan ? c - nchan : c;
    }
};
// the position r elements into the pattern (r < nchan * inner)
__device__ __forceinline__ ChanPos chan_at(uint32_t r, uint32_t inner) {
    const uint32_t ch = r / inner;
    return ChanPos{ch, r - ch * inner};
}

template <int CODE>
__device__ __forceinline__ float norm_decode1(uint32_t s, uint32_t lut) {
    if constexpr (norm_src(CODE) == 0) return __uint_as_float(lds32(s));
    else if constexpr (norm_src(CODE) == 1) return __uint_as_float(cvt_f32_of_f64(lds64(s)));
    else return __uint_as_float(lut32(lut, lds8(s)));
}
__device__ __forceinline__ float norm_apply(float x, const float *tab, uint32_t ch) {
    const float2 ms = __ldg((const float2 *)tab + ch);
    return __fdiv_rn(__fsub_rn(x, ms.x), ms.y);
}

// one element: source at shared address s, output at d, channel ch
template <int CODE>
__device__ __forceinline__ void norm_one(uint32_t s, char *d, uint32_t lut, const float *tab, uint32_t ch) {
    const float y = norm_apply(norm_decode1<CODE>(s, lut), tab, ch);
    if constexpr (norm_out(CODE) == 0) *(uint32_t *)d = __float_as_uint(y);
    else *(uint16_t *)d = (uint16_t)((norm_out(CODE) == 1 ? cvt2_bf16(y, 0.0f) : cvt2_f16(y, 0.0f)) & 0xFFFFu);
}

// one 16-byte output vector (E elements) from the source elements at shared address s; p = channel of the first
template <int CODE, bool VEC>
__device__ __forceinline__ uint4 norm_vec(uint32_t s, uint32_t lut, const float *tab, ChanPos p, uint32_t nchan, uint32_t inner) {
    constexpr int E = norm_out(CODE) == 0 ? 4 : 8;
    float x[E];
    if constexpr (norm_src(CODE) == 0) { // 4 or 8 floats
        if (VEC) {
#pragma unroll
            for (int k = 0; k < E; k += 4) {
                const uint4 a = lds128(s + 4u * k);
                x[k] = __uint_as_float(a.x); x[k + 1] = __uint_as_float(a.y); x[k + 2] = __uint_as_float(a.z); x[k + 3] = __uint_as_float(a.w);
            }
        } else {
#pragma unroll
            for (int k = 0; k < E; k++) x[k] = __uint_as_float(lds32(s + 4u * k));
        }
    } else if constexpr (norm_src(CODE) == 1) { // 4 doubles
        uint64_t q[4];
        if (VEC) {
            const uint4 a = lds128(s), b = lds128(s + 16);
            q[0] = (uint64_t)a.y << 32 | a.x; q[1] = (uint64_t)a.w << 32 | a.z;
            q[2] = (uint64_t)b.y << 32 | b.x; q[3] = (uint64_t)b.w << 32 | b.z;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = lds64(s + 8u * k);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) x[k] = __uint_as_float(cvt_f32_of_f64(q[k]));
    } else { // 4 or 8 bytes through the decode table
        uint32_t b[E];
        if (VEC) {
            const uint64_t v = E == 8 ? lds64(s) : (uint64_t)lds32(s);
#pragma unroll
            for (int k = 0; k < E; k++) b[k] = (uint32_t)(v >> (8 * k)) & 0xFFu;
        } else {
#pragma unroll
            for (int k = 0; k < E; k++) b[k] = lds8(s + k);
        }
#pragma unroll
        for (int k = 0; k < E; k++) x[k] = __uint_as_float(lut32(lut, b[k]));
    }
#pragma unroll
    for (int k = 0; k < E; k++) {
        x[k] = norm_apply(x[k], tab, p.ch);
        p.step(nchan, inner);
    }
    if constexpr (norm_out(CODE) == 0) {
        return make_uint4(__float_as_uint(x[0]), __float_as_uint(x[1]), __float_as_uint(x[2]), __float_as_uint(x[3]));
    } else {
        uint32_t r[4];
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = norm_out(CODE) == 1 ? cvt2_bf16(x[2 * k], x[2 * k + 1]) : cvt2_f16(x[2 * k], x[2 * k + 1]);
        return make_uint4(r[0], r[1], r[2], r[3]);
    }
}

// Drain one staged piece normalised: as cvt_drain; `rel` = the piece's first source byte relative to its variable's
// packed base, tab / nchan / inner = that variable's normalisation.
template <int CODE>
__device__ __forceinline__ void norm_drain(uint32_t s0, char *d, uint32_t n, uint32_t lut, int lane, const float *tab,
                                           int64_t rel, uint32_t nchan, uint32_t inner) {
    constexpr int IL = cvt_in_log2<true>(CODE), OL = cvt_out_log2<true>(CODE);
    constexpr uint32_t E = 16u >> OL;                          // elements per output vector
    constexpr uint32_t VA = (E << IL) < 16u ? (E << IL) : 16u; // source alignment of the vector loads
    const uint32_t ne = n >> IL;
    uint32_t head = ((16u - (uint32_t)((uint64_t)d & 15u)) & 15u) >> OL;
    if (head > ne) head = ne;
    const uint32_t nv = (ne - head) / E;
    const uint32_t tail = ne - head - nv * E;
    const uint32_t sb = s0 + (head << IL);
    char *dv = d + (head << OL);
    const uint32_t period = nchan * inner;
    const uint32_t r0 = (uint32_t)((rel >> IL) % (int64_t)period); // pattern position of the piece's first element
    // (r0 + k < 2^32: the pattern is below 2^31 elements, a piece below 2^16)
    ChanPos p = chan_at((r0 + head + (uint32_t)lane * E) % period, inner);
    const uint32_t dq = ((32u * E) / inner) % nchan, dr = (32u * E) % inner; // one round of the warp: 32 vectors
    if ((sb & (VA - 1u)) == 0) { // warp-uniform
#pragma unroll 2
        for (uint32_t j = (uint32_t)lane; j < nv; j += 32) {
            stg128(dv + ((size_t)j << 4), norm_vec<CODE, true>(sb + j * (E << IL), lut, tab, p, nchan, inner));
            p.advance(dq, dr, nchan, inner);
        }
    } else {
#pragma unroll 2
        for (uint32_t j = (uint32_t)lane; j < nv; j += 32) {
            stg128(dv + ((size_t)j << 4), norm_vec<CODE, false>(sb + j * (E << IL), lut, tab, p, nchan, inner));
            p.advance(dq, dr, nchan, inner);
        }
    }
    if ((uint32_t)lane < head) {
        const uint32_t k = (uint32_t)lane;
        norm_one<CODE>(s0 + (k << IL), d + (k << OL), lut, tab, chan_at((r0 + k) % period, inner).ch);
    }
    if ((uint32_t)lane < tail) {
        const uint32_t k = head + nv * E + (uint32_t)lane;
        norm_one<CODE>(s0 + (k << IL), d + ((size_t)k << OL), lut, tab, chan_at((r0 + k) % period, inner).ch);
    }
}

// a normalising launch drains one piece of a variable with a normalising code (its position relative to the variable's
// packed base gives the channels; vbase: the variables' starts in a multi-array launch)
__device__ __forceinline__ void norm_piece(const ddsk_cvt_t &c, bool multi, const int64_t (&vbase)[DDSK_MAX_MULTI + 1],
                                           int64_t dpos, int code, uint32_t lut, char *d, uint32_t s, uint32_t n, int lane) {
    int64_t b = 0;
    const float *tab = c.norm[0];
    uint32_t nc = (uint32_t)c.nchan[0], inr = (uint32_t)c.inner[0];
    if (multi) {
        b = vbase[0];
#pragma unroll
        for (int k = 1; k < DDSK_MAX_MULTI; k++)
            if (dpos >= vbase[k]) {
                b = vbase[k];
                tab = c.norm[k];
                nc = (uint32_t)c.nchan[k];
                inr = (uint32_t)c.inner[k];
            }
    }
    const int64_t rel = dpos - b;
    switch (code) { // warp-uniform
    case DDSK_CVT_NORM_F32_F32: norm_drain<DDSK_CVT_NORM_F32_F32>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    case DDSK_CVT_NORM_F32_BF16: norm_drain<DDSK_CVT_NORM_F32_BF16>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    case DDSK_CVT_NORM_F32_F16: norm_drain<DDSK_CVT_NORM_F32_F16>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    case DDSK_CVT_NORM_F64_F32: norm_drain<DDSK_CVT_NORM_F64_F32>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    case DDSK_CVT_NORM_U8_F32: norm_drain<DDSK_CVT_NORM_U8_F32>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    case DDSK_CVT_NORM_U8_BF16: norm_drain<DDSK_CVT_NORM_U8_BF16>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    default: norm_drain<DDSK_CVT_NORM_U8_F16>(s, d, n, lut, lane, tab, rel, nc, inr); break;
    }
}

// the kernel parameter carrying a launch's conversion: ddsk_cvt_t, or nothing at all for raw launches
struct NoCvt {
    int32_t unused_;
};
template <bool CVT>
using CvtParam = typename std::conditional<CVT, ddsk_cvt_t, NoCvt>::type;

// ------------------------------------------------------------------------------------------------
// Plan in shared memory (variable counts, <= PCAP requests): EVERY CTA computes the whole plan -- lookup + checks +
// exclusive scan of the request sizes -- for itself. The index arrays are a few tens of KB that stay in L2 after
// the first CTA touched them, so the redundancy is cheap, and it removes every inter-CTA dependency the plan
// used to have (tile tickets, look-back, a grid-wide "all tiles written" wait) as well as the L2 round trips of the
// walk's searches and descriptor loads. Warp w owns a contiguous run of requests; loads are coalesced (lane-strided).
// Returns the packed total T (exact, int64); the shared copy keeps 32-bit offsets (the launcher uses this path only
// when the destination capacity is below 4 GiB, so T > 2^32 is a capacity error and nothing is copied).
// ------------------------------------------------------------------------------------------------
// (CVT: the offsets the caller sees are in output bytes of conversion `code`; the plan itself stays in source bytes)
// (PUT: the put form of the lookup, plan_many<4, true>)
template <int NW, int PCAP, bool CVT = false, bool NORM = false, bool PUT = false>
__device__ __forceinline__ int64_t plan_in_smem(const GatherArgs &a, const PlanView<PCAP> &pv, int64_t *wtot, int warp,
                                                int lane, bool writer, int code = 0) {
    auto out = [&](int64_t x) -> int64_t {
        if constexpr (CVT) return cvt_scale<NORM>(x, code);
        else return x;
    };
    const int64_t nreq = a.nreq;
    const int64_t per_warp = ((nreq + NW * 128 - 1) / (NW * 128)) * 128;
    const int64_t w0 = min(nreq, (int64_t)warp * per_warp), w1 = min(nreq, w0 + per_warp);
    int64_t lane_sum = 0;
    for (int64_t b = w0; b < w1; b += 128) {
        int64_t idx[4], nb[4];
        uint64_t sv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) idx[k] = b + k * 32 + lane;
        plan_many<4, PUT>(a.var, a.plan, idx, w1, a.status, a.status_tag, sv, nb);
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
            if (writer && a.offsets_out) a.offsets_out[i] = out(run + incl - v);
        }
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (warp == 0 && lane == 0) {
        sts32(pv.dst_s + (uint32_t)nreq * 4u, (uint32_t)min(T, (int64_t)0xFFFFFFFFll));
        if (writer) {
            if (a.offsets_out) a.offsets_out[nreq] = out(T);
            if (a.total_out) *a.total_out = T; // (source bytes: the host scales the total it reports)
        }
    }
    __syncthreads();
    return T;
}

struct PieceDesc {
    int64_t dpos;
    uint32_t n, pack; // pack = stage offset | (source misalignment << 16)
};
// kWrFetch: the shared address of a piece's result address, [NW][S][32] in dynamic shared memory behind the rings and the
// plan. (A function: a constant of the kernel itself changed the other instantiations' register allocation.)
template <int NW, int S, int STAGE, int PCAP>
__device__ __forceinline__ uint32_t fop_rdst(const unsigned char *smem_dyn, int warp, uint32_t st, int lane) {
    return smem_u32(smem_dyn) + (uint32_t)(NW * S * STAGE + (PCAP ? PCAP * 12 + 16 : 0)) +
           (uint32_t)((warp * S + (int)st) * 32 + lane) * 8u;
}

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

// CVT: the converting form (DDSK_CVT_*, `c` carries the codes and tables). Everything on the load side -- walk over the
// packed SOURCE byte space, rings, plan, checks, overlap protocol -- is the raw kernel's; only the drain and the
// caller-visible offsets differ. Converting launches have no push fetch.
// NORM (with CVT): the form of launches that carry a normalising code (DDSK_CVT_NORM_*); its drain handles every code,
// since a multi-array launch may mix normalised, plainly converted and raw variables.
// PAD (with FIXED): a padded batch -- a fixed-stride walk over slots of a.pad_slot source bytes (see ChunkWalker), the
// padding filled by the warps that claim it, the lengths written after the walk. No plan, no offsets, no push fetch.
// WR: a get (kWrNone) or a batched write (a.wr). kWrPut, a batched put (DDSK_OP_PUT) -- the raw walk with every copy
// reversed. Lookup, checks, plan, segment claims and
// status reports are the gather's; a piece's TMA load reads its packed position in a.dst (the caller's rows, a.dst_cap
// bytes) and the drain writes its shard address, through the same drain paths, which store exactly the piece's bytes
// (plain byte / 16-byte stores and bulk stores, never a read-modify-write of a neighbouring byte: other warps and other
// ranks may be writing the adjacent rows). Nothing is written outside the requests' rows, so a shard's zero slack stays
// zero. The load reads the 16-byte-aligned superset of the piece's range in the caller's buffer: up to 15 bytes on
// either side that belong to no request, in the same 16-byte block (which never crosses a page), whose values are
// discarded. Never overlapped, no offsets, no conversion, no push.
// kWrReduce: a batched accumulate -- the put whose drain reduces by a.wr.op (the sum or another) instead of storing, in
// the element type a.wr.type: bulk reductions where the put bulk-stores (and the op has a bulk form), element reductions
// for the ragged ends, vector reductions of the re-phased body (write_chunk). Each is atomic per element, so requests of
// any batch or rank that hit the same element combine.
// kWrFetch: a batched fetch-op -- the put whose drain applies a returning atomic (a.wr.op, in the element type a.wr.type;
// a compare-and-swap on 1 << a.wr.el_log2 bytes) to every element and sends the previous values to a.wr.result, at the
// operands' positions. Every piece is drained cooperatively in two passes: write_chunk replaces the staged operands by
// the previous values, then the raw drain (bulk stores where the phases allow) writes the stage to the result. The result
// address of each piece is kept beside its descriptor, in dynamic shared memory behind the rings and the plan.
template <bool FIXED, int NW, int S, int CH, int PCAP, bool CVT = false, bool NORM = false, bool PAD = false,
          int WR = kWrNone, bool HOST = false>
__global__ void __launch_bounds__(NW * 32, 1) dds_gather_kernel(const __grid_constant__ GatherArgs a,
                                                                const __grid_constant__ CvtParam<CVT> c) {
    static_assert(CVT || !NORM, "a normalising launch is a converting one");
    static_assert(FIXED || !PAD, "a padded batch is a fixed-stride walk");
    static_assert(WR == kWrNone || (!CVT && !PAD), "a write writes raw rows");
    static_assert(!HOST || WR == kWrNone, "HOST shards take no batched writes");
    constexpr int STAGE = CH + 32; // room for the aligned superset of a misaligned CH-byte range
    constexpr bool PUSH = FIXED && !CVT && !PAD && WR == kWrNone;
    extern __shared__ __align__(128) unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t full_bar[NW][S];
    __shared__ __align__(16) PieceDesc desc[NW][S][32];
    __shared__ int64_t wtot[PCAP > 0 ? NW : 1];
    __shared__ int64_t push_rbase[PUSH ? DDSK_MAX_RANKS + 1 : 1];
    __shared__ uint64_t push_win[PUSH ? DDSK_MAX_RANKS : 1];

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t gwarp = (int64_t)blockIdx.x * NW + warp;
    const int64_t nwarps = (int64_t)gridDim.x * NW;

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < S; s++) mbar_init(smem_u32(&full_bar[warp][s]), HOST ? 32 : 1); // (HOST: one per lane)
        fence_mbar_init();
    }
    // the launch's tables, copied from the parameter into shared memory behind the rings and the plan
    uint32_t lut_s = 0;
    if constexpr (CVT) {
        lut_s = smem_u32(smem_dyn) + (uint32_t)(NW * S * STAGE + (PCAP ? PCAP * 12 + 16 : 0));
        for (int i = threadIdx.x; i < c.lut_bytes / 4; i += NW * 32) sts32(lut_s + 4u * (uint32_t)i, c.lut[i]);
        __syncthreads();
    }
    int code0 = 0; // the conversion of a single-variable launch
    if constexpr (CVT) code0 = c.code[0];
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
    ChunkWalker<FIXED, CH, PCAP, CVT, PAD, WR != kWrNone> w; // (every write walks, plans and checks as a put)
    if (!FIXED) {
        if constexpr (PCAP > 0) {
            w.pv.src_s = smem_u32(smem_dyn) + (uint32_t)(NW * S * STAGE);
            w.pv.dst_s = w.pv.src_s + (uint32_t)PCAP * 8u;
            const bool writer = blockIdx.x == 0;
            if (writer) pass_gate(); // CTA 0 writes the offsets / the total for the caller
            w.T = plan_in_smem<NW, PCAP, CVT, NORM, WR != kWrNone>(a, w.pv, wtot, warp, lane, writer, code0);
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
    const bool push = PUSH && a.push != nullptr;
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
    if constexpr (PAD) w.nb = a.pad_slot; // (max_rows * row_bytes, checked by the host: nreq * slot fits)
    else w.nb = (FIXED && a.count <= a.var.lenlist[a.var.nranks - 1]) ? a.count * a.var.row_bytes : 0;
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
        if constexpr (CVT) {
            w.valign = true;
#pragma unroll
            for (int v = 0; v < DDSK_MAX_MULTI; v++) w.vb[v] = vbase[v];
        }
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
    // converting launches: the OUTPUT address of packed source position dpos, the conversion of its variable and the
    // shared address of that variable's table
    auto out_of = [&](int64_t dpos, int &code, uint32_t &lut) -> char * {
        if constexpr (CVT) {
            if (!multi) {
                code = code0;
                lut = lut_s + (uint32_t)c.lut_off[0];
                return a.dst + cvt_scale<NORM>(dpos, code0);
            }
            int64_t b = vbase[0];
            char *d = a.mdst[0];
            int cd = c.code[0], lo = c.lut_off[0];
#pragma unroll
            for (int k = 1; k < DDSK_MAX_MULTI; k++)
                if (dpos >= vbase[k]) {
                    b = vbase[k];
                    d = a.mdst[k];
                    cd = c.code[k];
                    lo = c.lut_off[k];
                }
            code = cd;
            lut = lut_s + (uint32_t)lo;
            return d + cvt_scale<NORM>(dpos - b, cd);
        } else {
            return nullptr; // (never called)
        }
    };
    {
        // A claim is one atomic (requested ahead of need) + a division (FIXED), a shared-memory search (VAR, plan in
        // shared memory) or one global load (VAR, plan in global scratch). Small segments (8 per warp) keep the tail
        // short; variable-count segments are multiples of SEG_GRAIN when the segment table is in use.
        // (push fetch: finer segments were slower, because every claim costs a window of index reads from the
        // requester's list over NVLink)
        if constexpr (PAD) {
            w.seg_bytes = ddsk_fixed_seg_bytes(w.T, w.nb, nwarps, a.min_seg_chunks, CH);
        } else {
        int64_t target = w.T / (nwarps * 8);
        const int64_t unit = (!FIXED && PCAP == 0) ? SEG_GRAIN : (int64_t)CH;
        target = max((int64_t)a.min_seg_chunks * CH, min(target, (int64_t)1 << 20));
        target = max(target, unit);
        if (FIXED && w.nb > 0 && w.nb <= target)
            w.seg_bytes = (target / w.nb) * w.nb; // whole requests per segment
        else
            w.seg_bytes = (target / unit) * unit;
        }
        w.nseg = w.T > 0 ? (w.T + w.seg_bytes - 1) / w.seg_bytes : 0;
    }
    if (over) {
        if (gwarp == 0 && lane == 0) report(a.status, a.status_tag, a.nreq, DDSK_CODE_CAPACITY);
        w.nseg = 0;
    }

    // ---- FIXED with nothing to walk (count <= 0, or the batch does not fit): run the reference's two checks here,
    //      so an invalid request is still the error that gets reported
    if (FIXED && !PAD && !push && (w.nb <= 0 || over)) {
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
            if (!HOST && lane == 0) mbar_expect_tx(bar, total);
            __syncwarp();
            const uint32_t al = (uint32_t)(pc.src & 15u);
            desc[warp][st][lane].dpos = pc.dpos;
            desc[warp][st][lane].n = pc.n;
            desc[warp][st][lane].pack = pc.off | (al << 16);
            if constexpr (WR == kWrFetch) // the piece's result address: its source position, in the result buffer
                sts64(fop_rdst<NW, S, STAGE, PCAP>(smem_dyn, warp, st, lane),
                      pc.n ? (uint64_t)a.wr.result + (pc.src - (uint64_t)a.dst) : 0);
            if constexpr (HOST) {
                // A source in mapped host memory never goes to the TMA unit. The lanes copy each piece's 16-byte-aligned
                // superset window together, 16 bytes per cp.async, and every lane's arrival completes the stage.
                const uint64_t my_src = pc.src - al;
                const uint32_t my_dst = ring + st * STAGE + pc.off, my_len = pc.n ? (al + pc.n + 15u) & ~15u : 0u;
                for (unsigned todo = __ballot_sync(0xffffffffu, pc.n != 0); todo; todo &= todo - 1) {
                    const int j = __ffs(todo) - 1;
                    const uint64_t sj = __shfl_sync(0xffffffffu, my_src, j);
                    const uint32_t dj = __shfl_sync(0xffffffffu, my_dst, j), lj = __shfl_sync(0xffffffffu, my_len, j);
                    for (uint32_t o = (uint32_t)lane * 16u; o < lj; o += 512u) cp_async_16(dj + o, sj + o);
                }
                cp_async_mbar_arrive(bar);
            } else if (pc.n) { // every lane issues its own piece's TMA load; all complete on the stage's mbarrier
                tma_load_1d(ring + st * STAGE + pc.off, (const void *)(pc.src - al), (al + pc.n + 15u) & ~15u, bar);
            }
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
        if constexpr (HOST) fence_proxy_async(); // the cp.async writes, before this lane's bulk stores read the stage
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
        if constexpr (WR == kWrFetch) {
            // fetch-op: pass 1, the atomics, every piece cooperatively; pass 2, the previous values to the result. A
            // compare-and-swap finds a piece's compare operands at its result address's position in a.wr.compare; pass 1
            // has read them all before pass 2 writes a result byte (result == compare is allowed).
            char *const my_res = (char *)lds64(fop_rdst<NW, S, STAGE, PCAP>(smem_dyn, warp, st, lane));
            unsigned todo = __ballot_sync(0xffffffffu, my_n != 0);
            for (unsigned rest = todo; rest; rest &= rest - 1) {
                const int j = __ffs(rest) - 1;
                const int64_t dpos = __shfl_sync(0xffffffffu, my_dpos, j);
                const uint32_t n = __shfl_sync(0xffffffffu, my_n, j);
                const uint32_t pk = __shfl_sync(0xffffffffu, my_pack, j);
                if (a.wr.op == DDSK_OP_CAS) {
                    const uint64_t r = __shfl_sync(0xffffffffu, (uint64_t)my_res, j);
                    write_chunk<kActCas>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, (char *)dpos,
                                         (const char *)a.wr.compare + (r - (uint64_t)a.wr.result), n, lane, a.wr.type,
                                         a.wr.op, (uint32_t)a.wr.el_log2);
                } else {
                    write_chunk<kActFetch>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, (char *)dpos, nullptr, n, lane,
                                           a.wr.type, a.wr.op, (uint32_t)a.wr.el_log2);
                }
            }
            fence_proxy_async(); // (every lane: its stage writes, before any lane's bulk store reads them)
            __syncwarp();
            const bool direct = my_n != 0 && (((uint32_t)(uint64_t)my_res | my_n | (my_pack >> 16)) & 15u) == 0;
            if (direct) tma_store_1d(my_res, ring + st * STAGE + (my_pack & 0xffffu), my_n);
            todo = __ballot_sync(0xffffffffu, my_n != 0 && !direct);
            while (todo) {
                const int j = __ffs(todo) - 1;
                todo &= todo - 1;
                char *const d = (char *)__shfl_sync(0xffffffffu, (uint64_t)my_res, j);
                const uint32_t n = __shfl_sync(0xffffffffu, my_n, j);
                const uint32_t pk = __shfl_sync(0xffffffffu, my_pack, j);
                drain_chunk<CH>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, d, n, lane);
            }
        } else if constexpr (WR != kWrNone) {
            // put: the raw drain (the last branch) into the shard address the descriptor carries -- a branch of its own,
            // so that the raw instantiations compile exactly as they did
            char *const my_dst = (char *)my_dpos;
            bool direct = my_n != 0 && (((uint32_t)(uint64_t)my_dst | my_n | (my_pack >> 16)) & 15u) == 0;
            if constexpr (WR == kWrReduce) {
                direct = direct && red_bulk(a.wr.type, a.wr.op);
                if (direct) tma_red_1d(my_dst, ring + st * STAGE + (my_pack & 0xffffu), my_n, a.wr.type, a.wr.op);
            } else {
                if (direct) tma_store_1d(my_dst, ring + st * STAGE + (my_pack & 0xffffu), my_n);
            }
            unsigned todo = __ballot_sync(0xffffffffu, my_n != 0 && !direct);
            while (todo) {
                const int j = __ffs(todo) - 1;
                todo &= todo - 1;
                const int64_t dpos = __shfl_sync(0xffffffffu, my_dpos, j);
                const uint32_t n = __shfl_sync(0xffffffffu, my_n, j);
                const uint32_t pk = __shfl_sync(0xffffffffu, my_pack, j);
                if constexpr (WR == kWrReduce) // (the element size from the type: read from the record, it cost the
                                                // fixed-count form two registers)
                    write_chunk<kActReduce>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, (char *)dpos, nullptr, n, lane,
                                            a.wr.type, a.wr.op, (uint32_t)DDSK_ACC_LOG2(a.wr.type));
                else drain_chunk<CH>(ring + st * STAGE + (pk & 0xffffu), pk >> 16, (char *)dpos, n, lane);
            }
        } else if constexpr (CVT) {
            // converting launch: a converted piece is always drained cooperatively; the raw variables of a multi-array
            // batch (code 0) keep the raw paths below
            int my_code;
            uint32_t my_lut;
            char *const my_dst = out_of(my_dpos, my_code, my_lut);
            const bool direct = my_code == 0 && my_n != 0 && (((uint32_t)(uint64_t)my_dst | my_n | (my_pack >> 16)) & 15u) == 0;
            if (direct) tma_store_1d(my_dst, ring + st * STAGE + (my_pack & 0xffffu), my_n);
            unsigned todo = __ballot_sync(0xffffffffu, my_n != 0 && !direct);
            while (todo) {
                const int j = __ffs(todo) - 1;
                todo &= todo - 1;
                const int64_t dpos = __shfl_sync(0xffffffffu, my_dpos, j);
                const uint32_t n = __shfl_sync(0xffffffffu, my_n, j);
                const uint32_t pk = __shfl_sync(0xffffffffu, my_pack, j);
                int code;
                uint32_t lut;
                char *const d = out_of(dpos, code, lut);
                const uint32_t s0 = ring + st * STAGE + (pk & 0xffffu); // + source misalignment = first payload byte
                if constexpr (NORM) {
                    if (DDSK_CVT_IS_NORM(code)) {
                        norm_piece(c, multi, vbase, dpos, code, lut, d, s0 + (pk >> 16), n, lane);
                        continue;
                    }
                }
                switch (code) { // warp-uniform
                case DDSK_CVT_F32_BF16: cvt_drain<DDSK_CVT_F32_BF16>(s0 + (pk >> 16), d, n, lut, lane); break;
                case DDSK_CVT_F32_F16: cvt_drain<DDSK_CVT_F32_F16>(s0 + (pk >> 16), d, n, lut, lane); break;
                case DDSK_CVT_F64_F32: cvt_drain<DDSK_CVT_F64_F32>(s0 + (pk >> 16), d, n, lut, lane); break;
                case DDSK_CVT_U8_LUT16: cvt_drain<DDSK_CVT_U8_LUT16>(s0 + (pk >> 16), d, n, lut, lane); break;
                case DDSK_CVT_U8_LUT32: cvt_drain<DDSK_CVT_U8_LUT32>(s0 + (pk >> 16), d, n, lut, lane); break;
                default: drain_chunk<CH>(s0, pk >> 16, d, n, lane); break;
                }
            }
        } else {
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
        } // (raw drain: the same code as before converting launches existed)
        bulk_commit(); // every lane: one (possibly empty) bulk group per drained stage
        __syncwarp();  // all lanes are done reading the stage before it is refilled
        consumed++;
    }
    if (WR != kWrNone || a.overlap || (FIXED && push)) {
        // every lane: its bulk stores have been performed (the done / arrive word below promises that; a put's rows are
        // complete when its last warp finishes)
        bulk_wait_all<0>();
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
                if constexpr (CVT) a.moffsets[v][j] = cvt_scale<NORM>(e - basev, c.code[v]); // (output bytes)
                else a.moffsets[v][j] = e - basev;                                     // never indexed dynamically
            }
        }
        if constexpr (CVT) { // the batch's total in output bytes (the sum over the variables' conversions)
            if (gwarp == 0 && lane == 0 && a.total_out) {
                int64_t t = 0;
#pragma unroll
                for (int v = 0; v < DDSK_MAX_MULTI; v++)
                    if (v < a.plan.nvars) t += cvt_scale<NORM>((v + 1 < a.plan.nvars ? vbase[v + 1] : w.T) - vbase[v], c.code[v]);
                *a.total_out = t;
            }
        }
    }
    if constexpr (PAD) { // delivered row counts; with max_rows = 0 nothing was walked, and this pass runs the checks
        if (a.pad_lengths || w.nb == 0) {
            for (int64_t i = gwarp * 32 + lane; i < a.nreq; i += nwarps * 32) {
                uint64_t src;
                int64_t payload;
                pad_lookup(a, i, src, payload);
                if (a.pad_lengths) a.pad_lengths[i] = payload / a.var.row_bytes;
            }
        }
    }
    if (FIXED && a.offsets_out && !push) { // arithmetic offsets, written off the critical path
        if constexpr (CVT) {
            for (int64_t i = gwarp * 32 + lane; i <= a.nreq; i += nwarps * 32) a.offsets_out[i] = cvt_scale<NORM>(i * w.nb, code0);
        } else {
            for (int64_t i = gwarp * 32 + lane; i <= a.nreq; i += nwarps * 32) a.offsets_out[i] = i * w.nb;
        }
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

// PUT: the plan of a batched put (plan_many's put form: an invalid request keeps its layout bytes, source address 0)
template <bool PUT = false>
__global__ void __launch_bounds__(PLAN_THREADS) dds_plan_kernel(const __grid_constant__ ddsk_var_t var,
                                                                const __grid_constant__ PlanSrc p, int64_t nreq,
                                                                uint64_t *__restrict__ req_src, int64_t *__restrict__ req_dst,
                                                                unsigned long long *tile_state, unsigned int tag,
                                                                int64_t *__restrict__ offsets_out, uint32_t *__restrict__ seg_tab,
                                                                int64_t seg_cap, unsigned long long *status,
                                                                unsigned long long status_tag, PlanProto pr,
                                                                int cvt_code) { // offsets_out in output bytes of this conversion
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
    plan_many<PLAN_ITEMS, PUT>(var, p, idx, nreq, status, status_tag, sv, nb); // (only reads: may run before the slot is known to be free)
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
            if (offsets_out) offsets_out[idx[k]] = cvt_scale<true>(d0, cvt_code);
            for (int64_t g = (d0 + SEG_GRAIN - 1) / SEG_GRAIN; g * SEG_GRAIN < d1 && g < seg_cap; g++) seg_tab[g] = (uint32_t)idx[k];
            run = d1;
        }
    }
    const bool last_tile = tile == (int64_t)gridDim.x - 1;
    const int64_t T = tile_excl_s + agg;
    if (last_tile && threadIdx.x == 0) {
        req_dst[nreq] = T;
        if (offsets_out) offsets_out[nreq] = cvt_scale<true>(T, cvt_code);
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
            // The row loads bypass L1 (ld.global.cg): this CTA stays resident across calls, and its SM's L1 is not
            // coherent with writes from other SMs or GPUs -- a batched put by any rank -- so a cached line could
            // return a row as it was before a put the caller has fenced since.
            // A HOST shard is read with ld.global.cv: the owner's update rewrites host memory behind the GPU's back, and
            // .cv drops a matching L2 line of system memory and fetches it again on every load.
            const char *sp = (const char *)src;
            if (var.host) {
                if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 15u) == 0) {
                    for (int64_t i = threadIdx.x; i < (n >> 4); i += blockDim.x) ((uint4 *)dp)[i] = __ldcv((const uint4 *)sp + i);
                } else if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 3u) == 0) {
                    for (int64_t i = threadIdx.x; i < (n >> 2); i += blockDim.x)
                        ((uint32_t *)dp)[i] = __ldcv((const unsigned int *)sp + i);
                } else {
                    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dp[i] = __ldcv(sp + i);
                }
            } else if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 15u) == 0) {
                for (int64_t i = threadIdx.x; i < (n >> 4); i += blockDim.x) ((uint4 *)dp)[i] = __ldcg((const uint4 *)sp + i);
            } else if ((((uint64_t)sp | (uint64_t)dp | (uint64_t)n) & 3u) == 0) {
                for (int64_t i = threadIdx.x; i < (n >> 2); i += blockDim.x) ((uint32_t *)dp)[i] = __ldcg((const unsigned int *)sp + i);
            } else {
                for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dp[i] = __ldcg(sp + i);
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
// pooled batches (dds_get_batch_pooled / dds_get_samples_pooled): each bag of requests folded into one output row
// ------------------------------------------------------------------------------------------------
// One warp per (bag, column slice), grid-striding over them. A lane owns one VB-byte vector of the slice (VB = 16, or one
// element when the row or the destination is not 16-byte aligned) and folds it over the bag's rows in request order, then
// row order: every output element is the sequential fold the contract defines, whatever the grid or the slicing. A bag's
// requests are read 32 at a time (one coalesced load of starts / counts / ids / weights, located lane-parallel); the rows
// of that window are then walked kPoolRows at a time, their loads in flight together before any of them is folded.
// Slices need no synchronisation with each other; the launcher narrows them (down to kPoolMinSlice bytes) until a few long
// bags still give every SM warps.
constexpr int kPoolThreads = 256;
constexpr int kPoolMinBlocks = 2; // CTAs per SM the registers must allow (__launch_bounds__)
constexpr int kPoolRows = 4;      // rows in flight per warp
constexpr int64_t kPoolMinSlice = 128;

struct PoolArgs {
    ddsk_var_t var;
    const int64_t *starts, *counts; // explicit requests (counts NULL: `count` rows each), or
    int64_t count;
    const int64_t *ids;             // sample ids looked up in the variable's sample index
    const longlong2 *tab;
    int64_t nsamples;
    const int64_t *bags; // [nbags + 1] request offsets, NULL: bag k = request k
    int64_t nbags, nreq;
    const void *weights; // [nreq] in the element type, NULL: unweighted
    int mode;            // DDSK_POOL_*
    char *dst;
    int64_t slice, nslices; // bytes per column slice (a multiple of VB, at most 32 * VB) and slices per row
    unsigned long long *status;
    unsigned long long status_tag;
};

// element bits (U) and accumulator (A) of each element type
template <int DT>
struct PoolType {
    using U = uint32_t;
    using A = float;
};
template <>
struct PoolType<DDSK_ACC_F64> {
    using U = uint64_t;
    using A = double;
};
template <>
struct PoolType<DDSK_ACC_F16> {
    using U = uint16_t;
    using A = float;
};
template <>
struct PoolType<DDSK_ACC_BF16> {
    using U = uint16_t;
    using A = float;
};

template <int DT>
__device__ __forceinline__ typename PoolType<DT>::A pool_dec(typename PoolType<DT>::U b) {
    if constexpr (DT == DDSK_ACC_F64) return __longlong_as_double((long long)b);
    else if constexpr (DT == DDSK_ACC_F16) return __half2float(__ushort_as_half(b));
    else if constexpr (DT == DDSK_ACC_BF16) return __bfloat162float(__ushort_as_bfloat16(b));
    else return __uint_as_float(b);
}
// one round-to-nearest conversion; a NaN becomes the type's canonical NaN (all ones but the sign)
template <int DT>
__device__ __forceinline__ typename PoolType<DT>::U pool_enc(typename PoolType<DT>::A v) {
    if constexpr (DT == DDSK_ACC_F64) return v != v ? 0x7FFFFFFFFFFFFFFFull : (uint64_t)__double_as_longlong(v);
    else if constexpr (DT == DDSK_ACC_F16) return v != v ? (uint16_t)0x7FFF : __half_as_ushort(__float2half_rn(v));
    else if constexpr (DT == DDSK_ACC_BF16) return v != v ? (uint16_t)0x7FFF : __bfloat16_as_ushort(__float2bfloat16_rn(v));
    else return v != v ? 0x7FFFFFFFu : __float_as_uint(v);
}
// IEEE round-to-nearest arithmetic, never contracted
__device__ __forceinline__ float pool_add(float a, float x) { return __fadd_rn(a, x); }
__device__ __forceinline__ double pool_add(double a, double x) { return __dadd_rn(a, x); }
__device__ __forceinline__ float pool_fma(float w, float x, float a) { return __fmaf_rn(w, x, a); }
__device__ __forceinline__ double pool_fma(double w, double x, double a) { return __fma_rn(w, x, a); }
__device__ __forceinline__ float pool_div(float a, int64_t n) { return __fdiv_rn(a, (float)n); }
__device__ __forceinline__ double pool_div(double a, int64_t n) { return __ddiv_rn(a, (double)n); }

// element e of a lane's vector RW (uint4, or one element)
template <typename U, typename RW>
__device__ __forceinline__ U pool_elem(const RW &r, int e) {
    if constexpr (std::is_same<RW, uint4>::value) {
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
        if constexpr (sizeof(U) == 2) return (U)(w[e >> 1] >> ((e & 1) * 16));
        else if constexpr (sizeof(U) == 4) return (U)w[e];
        else return (U)w[2 * e] | ((U)w[2 * e + 1] << 32);
    } else {
        return r;
    }
}
template <typename RW>
__device__ __forceinline__ RW pool_load(uint64_t p) {
    if constexpr (std::is_same<RW, uint4>::value) return __ldcg((const uint4 *)p);
    else if constexpr (sizeof(RW) == 2) return (RW)__ldcg((const unsigned short *)p);
    else if constexpr (sizeof(RW) == 4) return (RW)__ldcg((const unsigned int *)p);
    else return (RW)__ldcg((const unsigned long long *)p);
}
// the 16 bytes of E elements
template <typename U, int E>
__device__ __forceinline__ uint4 pool_pack(const U (&o)[E]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        if constexpr (sizeof(U) == 2) w[i] = (uint32_t)o[2 * i] | ((uint32_t)o[2 * i + 1] << 16);
        else if constexpr (sizeof(U) == 4) w[i] = (uint32_t)o[i];
        else w[i] = (uint32_t)(o[i >> 1] >> ((i & 1) * 32));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
template <typename U, int E>
__device__ __forceinline__ void pool_store(char *p, const U (&o)[E]) {
    if constexpr (E * sizeof(U) == 16) stg128(p, pool_pack<U, E>(o));
    else *(U *)p = o[0];
}
// Request i of a pooled batch: its first row's address in *src and its row count in *n; an invalid request leaves *n and
// is reported when `rep` (ordered after every bag report)
__device__ __forceinline__ void pool_req(const PoolArgs &a, int64_t i, uint64_t *src, int64_t *n, bool rep) {
    int64_t start = 0, count = 0;
    int code = 0;
    if (a.ids) {
        const int64_t id = a.ids[i];
        if (id < 0 || id >= a.nsamples) {
            code = DDSK_CODE_SAMPLE;
        } else {
            const longlong2 e = ldg_pair(&a.tab[id]);
            start = e.x;
            count = e.y;
        }
    } else {
        start = a.starts[i];
        count = a.counts ? a.counts[i] : a.count;
    }
    if (!code) code = dev_locate(a.var, start, count, src);
    if (code) {
        if (rep) report(a.status, a.status_tag, (int64_t)(DDSK_STATUS_LATE | (uint64_t)i), code);
    } else {
        *n = count;
    }
}

template <int DT, int VB>
__global__ void __launch_bounds__(kPoolThreads, kPoolMinBlocks) dds_pool_kernel(const __grid_constant__ PoolArgs a) {
    using U = typename PoolType<DT>::U;
    using A = typename PoolType<DT>::A;
    using RW = typename std::conditional<VB == 16, uint4, U>::type;
    constexpr int E = VB / (int)sizeof(U);
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (kPoolThreads / 32);
    const int64_t row_bytes = a.var.row_bytes;
    for (int64_t w = (int64_t)blockIdx.x * (kPoolThreads / 32) + (threadIdx.x >> 5); w < a.nbags * a.nslices; w += nwarps) {
        const int64_t k = w / a.nslices, sl = w - k * a.nslices;
        const int64_t col = sl * a.slice + (int64_t)lane * VB;
        const bool mine = (int64_t)lane * VB < a.slice && col < row_bytes; // (everything below is warp-uniform but the loads)
        int64_t b0 = k, b1 = k + 1;
        if (a.bags) {
            b0 = a.bags[k];
            b1 = a.bags[k + 1];
        }
        if (b0 < 0 || b1 < b0 || b1 > a.nreq) { // malformed: the row is written as zeros
            if (lane == 0 && sl == 0) report(a.status, a.status_tag, k, DDSK_CODE_BAG);
            b0 = b1 = 0;
        }
        A acc[E];
        U mx[E];
#pragma unroll
        for (int e = 0; e < E; e++) {
            acc[e] = A(0);
            mx[e] = U(0);
        }
        int64_t rows = 0; // rows folded so far
        for (int64_t base = b0; base < b1; base += 32) {
            const int64_t i = base + lane;
            uint64_t src = 0;
            int64_t n = 0;
            A wt = A(1);
            if (i < b1) { // (pool_req's locate, kept inline here: calling it changes this kernel's register allocation)
                int64_t start = 0, count = 0;
                int code = 0;
                if (a.ids) {
                    const int64_t id = a.ids[i];
                    if (id < 0 || id >= a.nsamples) {
                        code = DDSK_CODE_SAMPLE;
                    } else {
                        const longlong2 e = ldg_pair(&a.tab[id]);
                        start = e.x;
                        count = e.y;
                    }
                } else {
                    start = a.starts[i];
                    count = a.counts ? a.counts[i] : a.count;
                }
                if (!code) code = dev_locate(a.var, start, count, &src);
                if (code) report(a.status, a.status_tag, (int64_t)(DDSK_STATUS_LATE | (uint64_t)i), code);
                else n = count;
                if (a.weights) wt = pool_dec<DT>(((const U *)a.weights)[i]);
            }
            // the window's rows, in order: row r belongs to the request whose inclusive row scan first exceeds r
            const int64_t incl = warp_incl_scan(n, lane), excl = incl - n;
            const int64_t total = __shfl_sync(0xffffffffu, incl, 31);
            for (int64_t g = 0; g < total; g += kPoolRows) {
                RW x[kPoolRows];
                A wr[kPoolRows];
#pragma unroll
                for (int u = 0; u < kPoolRows; u++) {
                    const int64_t r = g + u;
                    const int j = __popc(__ballot_sync(0xffffffffu, incl <= r)) & 31;
                    const uint64_t s = __shfl_sync(0xffffffffu, src, j);
                    const int64_t e0 = __shfl_sync(0xffffffffu, excl, j);
                    wr[u] = __shfl_sync(0xffffffffu, wt, j);
                    x[u] = RW{};
                    if (mine && r < total) x[u] = pool_load<RW>(s + (uint64_t)(r - e0) * (uint64_t)row_bytes + (uint64_t)col);
                }
#pragma unroll
                for (int u = 0; u < kPoolRows; u++) {
                    if (g + u >= total) break;
#pragma unroll
                    for (int e = 0; e < E; e++) {
                        const U xb = pool_elem<U>(x[u], e);
                        if (a.mode == DDSK_POOL_MAX) {
                            if (rows + g + u == 0 || pool_dec<DT>(xb) > pool_dec<DT>(mx[e])) mx[e] = xb;
                        } else if (a.weights) {
                            acc[e] = pool_fma(wr[u], pool_dec<DT>(xb), acc[e]);
                        } else {
                            acc[e] = pool_add(acc[e], pool_dec<DT>(xb));
                        }
                    }
                }
            }
            rows += total;
        }
        if (mine) {
            U o[E];
#pragma unroll
            for (int e = 0; e < E; e++) {
                if (a.mode == DDSK_POOL_MAX) {
                    o[e] = mx[e];
                } else {
                    const A v = a.mode == DDSK_POOL_MEAN && rows > 0 ? pool_div(acc[e], rows) : acc[e];
                    o[e] = pool_enc<DT>(v);
                }
            }
            pool_store<U, E>(a.dst + k * row_bytes + col, o);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// pooled accumulates (dds_accumulate_batch_pooled / dds_accumulate_samples_pooled): the pooled batch's adjoint
// ------------------------------------------------------------------------------------------------
// One warp per (bag, row window, column slice). A lane loads its vector of grad[k] once; every row of the bag's valid
// requests then takes one atomic of the contribution (grad, times the request's weight, over the bag's row count for a
// mean, times alpha; each step rounded once, then rounded to the element type): red16 per 16-byte vector, else one red1v
// per element. The contributions are independent atomics, so there is no order to keep: window j of a bag's `windows`
// takes the bag's valid rows j, j + windows, ... The requests are read and located 32 at a time as in the pooled get, and
// every window walks all of them (it needs each row's place in the bag). A mean needs the bag's row count before its first
// atomic: for bags of at most 32 requests it is the first window of requests' row total, longer bags count in a first pass.
// An unweighted bag's contribution is the same for every row and is computed once.
struct PoolAccArgs {
    PoolArgs p;       // requests, bags, weights, mode and slices as in the pooled get (p.dst unused)
    const char *grad; // [nbags] rows of row_bytes in the element type
    double alpha;
    int64_t windows; // row windows per bag
};
constexpr int64_t kPoolAccFill = 4;        // warps per resident warp the launcher aims for
constexpr int64_t kPoolAccMaxWindows = 32; // row windows per bag at most

__device__ __forceinline__ float pool_mul(float a, float x) { return __fmul_rn(a, x); }
__device__ __forceinline__ double pool_mul(double a, double x) { return __dmul_rn(a, x); }
template <typename RW>
__device__ __forceinline__ RW pool_ldg(const char *p) {
    if constexpr (std::is_same<RW, uint4>::value) return __ldg((const uint4 *)p);
    else if constexpr (sizeof(RW) == 2) return (RW)__ldg((const unsigned short *)p);
    else if constexpr (sizeof(RW) == 4) return (RW)__ldg((const unsigned int *)p);
    else return (RW)__ldg((const unsigned long long *)p);
}
// a lane's contribution vector: g (weighted by w), over n (mean, n > 0), times alpha, each step rounded; then encoded
template <int DT, int E>
__device__ __forceinline__ void pool_contrib(typename PoolType<DT>::U (&c)[E], const typename PoolType<DT>::A (&g)[E],
                                             bool weighted, typename PoolType<DT>::A w, int64_t n,
                                             typename PoolType<DT>::A alpha) {
#pragma unroll
    for (int e = 0; e < E; e++) {
        typename PoolType<DT>::A v = g[e];
        if (weighted) v = pool_mul(v, w);
        if (n > 0) v = pool_div(v, n);
        c[e] = pool_enc<DT>(pool_mul(v, alpha));
    }
}
template <int DT, int E>
__device__ __forceinline__ void pool_red(char *d, const typename PoolType<DT>::U (&c)[E]) {
    if constexpr (E * sizeof(typename PoolType<DT>::U) == 16) red16(d, pool_pack(c), DT, DDSK_OP_SUM);
    else red1v(d, Held{(uint64_t)c[0]}, DT, DDSK_OP_SUM);
}

template <int DT, int VB>
__global__ void __launch_bounds__(kPoolThreads, kPoolMinBlocks) dds_pool_acc_kernel(const __grid_constant__ PoolAccArgs aa) {
    using U = typename PoolType<DT>::U;
    using A = typename PoolType<DT>::A;
    using RW = typename std::conditional<VB == 16, uint4, U>::type;
    constexpr int E = VB / (int)sizeof(U);
    const PoolArgs &a = aa.p;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (kPoolThreads / 32);
    const int64_t row_bytes = a.var.row_bytes, W = aa.windows, per_bag = a.nslices * W;
    const bool mean = a.mode == DDSK_POOL_MEAN, weighted = a.weights != nullptr;
    const A alpha = (A)aa.alpha;
    for (int64_t w = (int64_t)blockIdx.x * (kPoolThreads / 32) + (threadIdx.x >> 5); w < a.nbags * per_bag; w += nwarps) {
        const int64_t k = w / per_bag, rem = w - k * per_bag, j = rem / a.nslices, sl = rem - j * a.nslices;
        const int64_t col = sl * a.slice + (int64_t)lane * VB;
        const bool mine = (int64_t)lane * VB < a.slice && col < row_bytes; // (everything below is warp-uniform but the loads)
        int64_t b0 = k, b1 = k + 1;
        if (a.bags) {
            b0 = a.bags[k];
            b1 = a.bags[k + 1];
        }
        if (b0 < 0 || b1 < b0 || b1 > a.nreq) { // malformed: nothing is written
            if (lane == 0 && sl == 0 && j == 0) report(a.status, a.status_tag, k, DDSK_CODE_BAG);
            continue;
        }
        A g[E];
        {
            const RW x = mine ? pool_ldg<RW>(aa.grad + k * row_bytes + col) : RW{};
#pragma unroll
            for (int e = 0; e < E; e++) g[e] = pool_dec<DT>(pool_elem<U>(x, e));
        }
        int64_t nk = 0; // a mean bag's rows (0: no division)
        if (mean && b1 - b0 > 32)
            for (int64_t base = b0; base < b1; base += 32) {
                uint64_t src;
                int64_t n = 0;
                if (base + lane < b1) pool_req(a, base + lane, &src, &n, false);
                nk += warp_sum(n);
            }
        U cu[E]; // the unweighted contribution, once the bag's row count is known
        int64_t rows = 0; // the bag's valid rows before this window of requests
        for (int64_t base = b0; base < b1; base += 32) {
            const int64_t i = base + lane;
            uint64_t src = 0;
            int64_t n = 0;
            A wt = A(1);
            if (i < b1) {
                pool_req(a, i, &src, &n, j == 0);
                if (weighted) wt = pool_dec<DT>(((const U *)a.weights)[i]);
            }
            const int64_t incl = warp_incl_scan(n, lane), excl = incl - n;
            const int64_t total = __shfl_sync(0xffffffffu, incl, 31);
            if (base == b0 && !weighted) {
                if (mean && b1 - b0 <= 32) nk = total;
                pool_contrib<DT, E>(cu, g, false, A(1), nk, alpha);
            }
            // this window's rows r of the requests: (rows + r) % W == j
            for (int64_t r = ((j - rows) % W + W) % W; r < total; r += W) {
                const int q = __popc(__ballot_sync(0xffffffffu, incl <= r)) & 31;
                const uint64_t s = __shfl_sync(0xffffffffu, src, q);
                const int64_t e0 = __shfl_sync(0xffffffffu, excl, q);
                char *d = (char *)(s + (uint64_t)(r - e0) * (uint64_t)row_bytes + (uint64_t)col);
                if (weighted) {
                    const A wr = __shfl_sync(0xffffffffu, wt, q);
                    U c[E];
                    pool_contrib<DT, E>(c, g, true, wr, 0, alpha);
                    if (mine) pool_red<DT, E>(d, c);
                } else if (mine) {
                    pool_red<DT, E>(d, cu);
                }
            }
            rows += total;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// launch geometry
// ------------------------------------------------------------------------------------------------
// Every geometry dds_gather_kernel is launched with: warps per CTA, ring stages per warp, chunk bytes, and the capacity of
// a plan held in shared memory (0: the plan, if any, is in global memory). Each is named here once; every launch, fit
// check and plan threshold below reads it from these constants. Every geometry runs one CTA per SM.
struct Geometry {
    int nw, stages, ch, pcap;
};
// On an H100 SXM (400 W limit) config 2 (4 KiB rows) is HBM-bound with every fixed-count geometry tried: they measured
// within 0.3 % of each other, so large rows keep 12 warps x 4 stages (also used for the instruction-heavier variable /
// re-phase path); rows under 2 KiB take more warps to keep more small copies in flight.
constexpr Geometry kLargeRows = {12, 4, 4096, 0}; // every plan-in-global launch but the two below
constexpr Geometry kSmallRows = {16, 3, 4096, 0}; // fixed-count raw gets of requests under 2 KiB
constexpr Geometry kFetch = {12, 3, 4096, 0};     // fetch-ops: one stage fewer leaves room for their result addresses
// plan in shared memory (variable-count entries): the plan's 12 B per request come out of the stage budget
constexpr Geometry kPlan4K = {12, 3, 4096, 4096};
constexpr Geometry kPlan8K = {12, 3, 3072, 8192};
constexpr Geometry kPlan8KFetch = {12, 3, 2048, 8192}; // (with their result addresses too, fetch-ops fit 2 KiB chunks only)
constexpr int64_t kPlanSmemMax = kPlan8K.pcap;
// Launches that read DDS_PLACE_HOST shards: kLargeRows with the cp.async producer on a grid of kHostCtas CTAs. Their
// bytes cross PCIe at a small fraction of the HBM rate, so a full-machine grid would hold every SM for the whole transfer
// (DESIGN.md 3.12 has the sweep this count comes from). They always plan in the plan kernels.
constexpr int kHostCtas = 4;
int g_host_ctas = kHostCtas; // DDS_HOST_CTAS (1..16): measurement switch of the sweep
// The redundant plan grows with the batch (every SM reads the same index lines), while the plan kernels cost ~0 when
// they run under the previous batch's gather -- so by default only small batches, where one launch beats three, plan
// in shared memory.
int64_t g_plan_smem_default = 1024; // DDS_SMEM_PLAN_MAX

int g_min_seg_var = 4, g_min_seg_s = 2; // DDS_VAR_MINSEG / DDS_S_MINSEG: smallest segment in chunks
bool g_geom_init = false;
int g_sms = 0;
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
    if (const char *e = getenv("DDS_VAR_MINSEG")) g_min_seg_var = atoi(e) > 0 ? atoi(e) : 4;
    if (const char *e = getenv("DDS_S_MINSEG")) g_min_seg_s = atoi(e) > 0 ? atoi(e) : 2;
    if (const char *e = getenv("DDS_PDL")) g_pdl = atoi(e) != 0;
    if (const char *e = getenv("DDS_SMEM_PLAN")) g_smem_plan = atoi(e);
    if (const char *e = getenv("DDS_SMEM_PLAN_MAX")) g_plan_smem_default = atoll(e);
    if (const char *e = getenv("DDS_L2_PERSIST")) g_l2_persist = atoi(e);
    if (const char *e = getenv("DDS_HOST_CTAS")) g_host_ctas = std::max(1, std::min(16, atoi(e)));
    if (const char *e = getenv("DDS_DEBUG_TIMING"))
        if (atoi(e)) {
            CUDA_TRY(cudaMalloc((void **)&g_dbg, 2 * kDbgRegion * 8));
            CUDA_TRY(cudaMemset(g_dbg, 0, 2 * kDbgRegion * 8));
        }
    g_geom_init = true;
    return 0;
}

constexpr int smem_bytes_of(const Geometry &g) { return g.nw * g.stages * (g.ch + 32) + (g.pcap ? g.pcap * 12 + 16 : 0); }

// does a converting launch carry a normalising code? (then it takes the NORM form of the kernel; unused slots are 0)
bool cvt_has_norm(const ddsk_cvt_t *cvt) {
    for (int v = 0; v < DDSK_MAX_MULTI; v++)
        if (DDSK_CVT_IS_NORM(cvt->code[v])) return true;
    return false;
}

template <bool FIXED, const Geometry &G, bool CVT = false, bool NORM = false, bool PAD = false, int WR = kWrNone,
          bool HOST = false>
int launch_gather_t(const GatherArgs &args_in, cudaStream_t stream, const ddsk_cvt_t *cvt = nullptr) {
    // (a converting launch also holds its tables in dynamic shared memory, behind the rings and the plan; a fetch-op its
    //  pieces' result addresses)
    const int smem = smem_bytes_of(G) + (CVT ? cvt->lut_bytes : 0) + (WR == kWrFetch ? G.nw * G.stages * 32 * 8 : 0);
    static std::atomic<unsigned long long> configured{0}; // bit d: attribute set on device d (it is per device)
    auto kern = dds_gather_kernel<FIXED, G.nw, G.stages, G.ch, G.pcap, CVT, NORM, PAD, WR, HOST>;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    if (CVT) { // the most a converting launch can ask for: every table at its widest
        if (dev >= 64 || !(configured.load() & (1ull << dev))) {
            cudaFuncAttributes fa;
            int optin = 0;
            CUDA_TRY(cudaFuncGetAttributes(&fa, kern));
            CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
            const int most = std::min(smem_bytes_of(G) + DDSK_MAX_MULTI * 1024, optin - (int)fa.sharedSizeBytes);
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
            if (dev < 64) configured.fetch_or(1ull << dev);
        }
    } else if (dev >= 64 || !(configured.load() & (1ull << dev))) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        if (dev < 64) configured.fetch_or(1ull << dev);
    }
    GatherArgs args = args_in;
    args.dbg = g_dbg ? g_dbg + (size_t)(args.overlap ? (args.seq & 1u) : 0u) * kDbgRegion : nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(HOST ? std::min(g_sms, g_host_ctas) : g_sms));
    cfg.blockDim = dim3(G.nw * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if constexpr (CVT) {
        CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args, *cvt));
    } else {
        CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args, NoCvt{0}));
    }
    g_launches++;
    return 0;
}

// Does a converting launch of shared-memory-plan geometry G with `lut_bytes` of tables fit in shared memory? (With four
// 1 KiB tables the 8192-request plan does not: such batches plan in global memory instead.)
template <const Geometry &G>
bool cvt_s_fits_t(int lut_bytes) {
    cudaFuncAttributes fa;
    int dev = 0, optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, dds_gather_kernel<false, G.nw, G.stages, G.ch, G.pcap, true>) != cudaSuccess ||
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    return smem_bytes_of(G) + lut_bytes + (int)fa.sharedSizeBytes <= optin;
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

// One launch of the kind asked for (wr: kWr*; cvt): a fetch-op at geometry GF, every other kind (accumulate, put,
// normalising, converting, raw) at G.
template <bool FIXED, const Geometry &G, const Geometry &GF>
int launch_kind(const GatherArgs &args, cudaStream_t stream, const ddsk_cvt_t *cvt, int wr) {
    if (wr == kWrFetch) return launch_gather_t<FIXED, GF, false, false, false, kWrFetch>(args, stream);
    if (wr == kWrReduce) return launch_gather_t<FIXED, G, false, false, false, kWrReduce>(args, stream);
    if (wr == kWrPut) return launch_gather_t<FIXED, G, false, false, false, kWrPut>(args, stream);
    if (cvt) return cvt_has_norm(cvt) ? launch_gather_t<FIXED, G, true, true>(args, stream, cvt)
                                      : launch_gather_t<FIXED, G, true>(args, stream, cvt);
    return launch_gather_t<FIXED, G>(args, stream);
}

// a read of HOST shards (never a write: the store refuses those), raw, converting or normalising
template <bool FIXED, bool PAD = false>
int launch_host(const GatherArgs &args, cudaStream_t stream, const ddsk_cvt_t *cvt) {
    if (!cvt) return launch_gather_t<FIXED, kLargeRows, false, false, PAD, kWrNone, true>(args, stream);
    return cvt_has_norm(cvt) ? launch_gather_t<FIXED, kLargeRows, true, true, PAD, kWrNone, true>(args, stream, cvt)
                             : launch_gather_t<FIXED, kLargeRows, true, false, PAD, kWrNone, true>(args, stream, cvt);
}

// plan in global memory (or none): small rows for fixed-count raw gets of requests under 2 KiB, large rows otherwise
template <bool FIXED>
int launch_gather(const GatherArgs &args, cudaStream_t stream, const ddsk_cvt_t *cvt, int wr = kWrNone) {
    if (args.var.host) return launch_host<FIXED>(args, stream, cvt);
    if constexpr (FIXED) {
        // (a count too large to multiply safely counts as large)
        const int64_t request_bytes = args.count < ((int64_t)1 << 20) ? args.count * args.var.row_bytes : INT64_MAX;
        if (wr == kWrNone && !cvt && request_bytes < 2048) return launch_gather_t<true, kSmallRows>(args, stream);
    }
    return launch_kind<FIXED, kLargeRows, kFetch>(args, stream, cvt, wr);
}

// The shared-memory plan for a batch of nreq requests into cap bytes: 0 = kPlan4K, 1 = kPlan8K (-1: the plan kernels).
// A converting launch also needs room for its tables.
int select_s(int64_t nreq, int64_t cap, const ddsk_cvt_t *cvt, bool host) {
    if (host || !g_smem_plan || cap >= ((int64_t)1 << 32) || nreq > kPlanSmemMax || nreq > g_plan_smem_default) return -1;
    if (nreq <= kPlan4K.pcap) return !cvt || cvt_s_fits_t<kPlan4K>(cvt->lut_bytes) ? 0 : -1;
    return !cvt || cvt_s_fits_t<kPlan8K>(cvt->lut_bytes) ? 1 : -1;
}

// The fields every gather launch shares: the variable's window, status reporting, the host mirror (DDSK_F_MIRROR), the
// overlap protocol and segment tickets, and the default smallest segment. Picks the geometry on first use.
int gather_args(GatherArgs &a, const ddsk_var_t *var, const ddsk_scratch_t *scr, int flags) {
    if (int rc = pick_geometry()) return rc;
    memset(&a, 0, sizeof(a));
    a.var = *var;
    a.status = scr->status;
    a.status_tag = scr->status_tag;
    a.counters = scr->counters;
    a.host_mirror = (flags & DDSK_F_MIRROR) ? scr->host_mirror : nullptr;
    a.min_seg_chunks = 1;
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
    return 0;
}

// The kernel form of a launch that carries the write record wr (NULL for a get), which then goes into a.wr: op 0 is a
// put, a record without a result a reduction, one with a result a fetch-op
int write_form(GatherArgs &a, const ddsk_write_t *wr) {
    if (!wr) return kWrNone;
    a.wr = *wr;
    return wr->op == DDSK_OP_PUT ? kWrPut : wr->result ? kWrFetch : kWrReduce;
}

template <int DT>
int launch_pool_t(const PoolArgs &a, int vb, int blocks, cudaStream_t st) {
    if (vb == 16) dds_pool_kernel<DT, 16><<<blocks, kPoolThreads, 0, st>>>(a);
    else dds_pool_kernel<DT, (int)sizeof(typename PoolType<DT>::U)><<<blocks, kPoolThreads, 0, st>>>(a);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}
template <int DT>
int launch_pool_acc_t(const PoolAccArgs &a, int vb, int blocks, cudaStream_t st) {
    if (vb == 16) dds_pool_acc_kernel<DT, 16><<<blocks, kPoolThreads, 0, st>>>(a);
    else dds_pool_acc_kernel<DT, (int)sizeof(typename PoolType<DT>::U)><<<blocks, kPoolThreads, 0, st>>>(a);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// A pooled launch's arguments but its slices and output
void pool_args(PoolArgs &a, const ddsk_var_t *var, const ddsk_index_t *index, int64_t fixed_count, int64_t nreq,
               const ddsk_pool_t *pool, const ddsk_scratch_t *scr) {
    memset(&a, 0, sizeof(a));
    a.var = *var;
    a.starts = index->starts;
    a.counts = index->counts;
    a.count = fixed_count;
    a.ids = index->sample_ids;
    a.tab = (const longlong2 *)index->table;
    a.nsamples = index->nsamples;
    a.bags = pool->bags;
    a.nbags = pool->nbags;
    a.nreq = nreq;
    a.weights = pool->weights;
    a.mode = pool->mode;
    a.status = scr->status;
    a.status_tag = scr->status_tag;
}

// The launch geometry of a pooled get (adjoint false) or of its adjoint, the one place its rule is written: rows of
// row_bytes of element type `type`, nbags bags (both > 0), a destination / grad that is 16-byte aligned or not, HOST
// shards or not. pick_geometry() must have succeeded.
struct PoolGeometry {
    int vb;                          // bytes per lane vector: 16, or one element
    int64_t slice, nslices, windows; // bytes per column slice and slices per row; row windows per bag (1 for the get)
    int blocks;                      // CTAs of kPoolThreads
};
PoolGeometry pool_geometry(bool adjoint, int64_t row_bytes, int type, int64_t nbags, bool aligned16, bool host) {
    PoolGeometry g;
    g.vb = (row_bytes % 16 == 0 && aligned16) ? 16 : 1 << DDSK_ACC_LOG2(type);
    const int64_t resident = (int64_t)g_sms * kPoolMinBlocks * (kPoolThreads / 32), per_cta = kPoolThreads / 32;
    g.slice = 32 * g.vb;
    g.nslices = (row_bytes + g.slice - 1) / g.slice;
    g.windows = 1;
    if (!adjoint) {
        // get: slices halved while the bags leave resident warps idle (a few long bags then still spread)
        while (g.slice / 2 >= kPoolMinSlice && nbags * g.nslices < resident) {
            g.slice /= 2;
            g.nslices = (row_bytes + g.slice - 1) / g.slice;
        }
    } else {
        // adjoint: whole-warp slices; then each bag's rows are dealt to row windows until there are kPoolAccFill warps
        // per resident one (a few long bags, such as mean-pooled frames, then still spread over the machine)
        const int64_t units = nbags * g.nslices;
        g.windows = std::max<int64_t>(1, std::min<int64_t>(kPoolAccMaxWindows, (kPoolAccFill * resident + units - 1) / units));
    }
    const int64_t most = host ? std::min(g_sms, g_host_ctas) : (int64_t)g_sms * kPoolMinBlocks;
    g.blocks = (int)std::min((nbags * g.nslices * g.windows + per_cta - 1) / per_cta, most);
    return g;
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

int ddsk_host_gather_ctas(void) { return pick_geometry() ? 0 : std::min(g_sms, g_host_ctas); }

void ddsk_gather_geometry(int *ctas, int *warps_per_cta, int *stages, int *chunk_bytes, int *smem_bytes) {
    if (pick_geometry()) {
        *ctas = *warps_per_cta = *stages = *chunk_bytes = *smem_bytes = 0;
        return;
    }
    *ctas = g_sms;
    *warps_per_cta = kLargeRows.nw;
    *stages = kLargeRows.stages;
    *chunk_bytes = kLargeRows.ch;
    *smem_bytes = smem_bytes_of(kLargeRows);
}

void ddsk_pool_geometry(int adjoint, int64_t row_bytes, int type, int64_t nbags, int aligned16, int host, int *vb,
                        int64_t *slice, int64_t *nslices, int64_t *windows, int *blocks) {
    const bool ok = type == DDSK_ACC_F32 || type == DDSK_ACC_F64 || type == DDSK_ACC_F16 || type == DDSK_ACC_BF16;
    if (!ok || nbags <= 0 || row_bytes <= 0 || pick_geometry()) {
        *vb = *blocks = 0;
        *slice = *nslices = *windows = 0;
        return;
    }
    const PoolGeometry g = pool_geometry(adjoint != 0, row_bytes, type, nbags, aligned16 != 0, host != 0);
    *vb = g.vb;
    *slice = g.slice;
    *nslices = g.nslices;
    *windows = g.windows;
    *blocks = g.blocks;
}

int ddsk_gather_fixed(const ddsk_var_t *var, const int64_t *starts_dev, int64_t count, int64_t nreq, void *dst_dev,
                      int64_t dst_capacity, int64_t *offsets_dev_or_null, const ddsk_scratch_t *scr, int flags,
                      const ddsk_cvt_t *cvt, const ddsk_write_t *wr, void *stream) {
    if (nreq <= 0) return 0;
    GatherArgs a;
    if (int rc = gather_args(a, var, scr, flags)) return rc;
    const int form = write_form(a, wr);
    a.starts = starts_dev;
    a.count = count;
    a.nreq = nreq;
    a.dst = (char *)dst_dev;
    a.dst_cap = dst_capacity;
    a.offsets_out = offsets_dev_or_null;
    return launch_gather<true>(a, (cudaStream_t)stream, cvt, form);
}

int ddsk_gather_push(const ddsk_var_t *var, const ddsk_push_t *push_host, const ddsk_push_t *push_dev,
                     const int64_t *starts_dev, int64_t count, int64_t nreq, unsigned long long step,
                     const ddsk_scratch_t *scr, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GatherArgs a;
    if (int rc = gather_args(a, var, scr, 0)) return rc;
    a.count = count;
    a.nreq = nreq; // (this rank's own requests; the walk covers every rank's)
    a.dst_cap = INT64_MAX;
    a.push = push_dev;
    if (nreq > 0) // this rank's list into its window, stream-ordered before the kernel that publishes it
        CUDA_TRY(cudaMemcpyAsync(push_host->win[push_host->me] + push_host->idx_off[step & 1ull], starts_dev, (size_t)nreq * 8,
                                 cudaMemcpyDeviceToDevice, st));
    a.push_nreq = nreq;
    a.push_step = step;
    return launch_gather<true>(a, st, nullptr);
}

int ddsk_gather_padded(const ddsk_var_t *var, const ddsk_index_t *index, int64_t nreq, int64_t max_rows, uint64_t pad_bits,
                       int pad_log2, int64_t *lengths, void *dst_dev, const ddsk_scratch_t *scr, int flags,
                       const ddsk_cvt_t *cvt, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (nreq <= 0) return 0;
    GatherArgs a;
    if (int rc = gather_args(a, var, scr, flags)) return rc;
    a.plan.starts = index->starts;
    a.plan.counts = index->counts;
    a.plan.ids = index->sample_ids;
    a.plan.tab = (const longlong2 *)index->table;
    a.plan.nsamples = index->nsamples;
    a.count = max_rows;
    a.nreq = nreq;
    a.dst = (char *)dst_dev;
    a.pad_slot = max_rows * var->row_bytes;
    a.dst_cap = nreq * a.pad_slot; // (the host checked the padded size against the caller's capacity)
    a.pad_bits = pad_bits;
    a.pad_log2 = pad_log2;
    a.pad_in_log2 = cvt ? cvt_in_log2<true>(cvt->code[0]) : 0;
    a.pad_out_log2 = cvt ? cvt_out_log2<true>(cvt->code[0]) : 0;
    a.pad_lengths = lengths;
    if (var->host) return launch_host<true, true>(a, st, cvt);
    if (!cvt) return launch_gather_t<true, kLargeRows, false, false, true>(a, st);
    return cvt_has_norm(cvt) ? launch_gather_t<true, kLargeRows, true, true, true>(a, st, cvt)
                             : launch_gather_t<true, kLargeRows, true, false, true>(a, st, cvt);
}

// shared by ddsk_gather_var / ddsk_gather_multi: plan (in the launch, or by the two plan kernels) + gather. `a` comes
// from gather_args; form is write_form's.
static int plan_and_gather(const ddsk_var_t *var, const PlanSrc &p, int64_t nreq, int64_t cap_total, GatherArgs &a,
                           int64_t *offsets_dev_or_null, ddsk_scratch_t *scr, int flags, const ddsk_cvt_t *cvt, int form,
                           cudaStream_t st) {
    a.nreq = nreq;
    a.plan = p; // the gather needs nvars / per_var even when the plan ran in its own kernels
    a.total_out = scr->total;
    const int gs = select_s(nreq, cap_total, cvt, a.var.host != 0);
    if (gs >= 0) {
        a.offsets_out = offsets_dev_or_null;
        a.min_seg_chunks = g_min_seg_s;
        // (no scratch is shared between launches: independent batches may overlap)
        if (a.overlap) a.tickets = scr->ovl + 8 + (a.seq & 3u);
        return gs ? launch_kind<false, kPlan8K, kPlan8KFetch>(a, st, cvt, form)
                  : launch_kind<false, kPlan4K, kPlan4K>(a, st, cvt, form);
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
    if (int rc = launch_pdl(form != kWrNone ? dds_plan_kernel<true> : dds_plan_kernel<false>, dim3(tiles), dim3(PLAN_THREADS), st, *var, p, nreq, scr->req_src, scr->req_dst,
                            (unsigned long long *)scr->tile_sums, scr->plan_tag, offsets_dev_or_null, scr->seg_tab, scr->seg_cap,
                            scr->status, scr->status_tag, pr, cvt && p.nvars <= 1 ? (int)cvt->code[0] : 0))
        return rc;
    a.req_src = scr->req_src;
    a.req_dst = scr->req_dst;
    a.seg_tab = scr->seg_tab;
    // (a converting multi-array batch has no single source total: its gather writes the output total here)
    a.total_out = (cvt && p.nvars > 1) ? scr->total : nullptr;
    a.min_seg_chunks = g_min_seg_var;
    if (a.overlap) {
        a.tickets = scr->ovl + 8 + (a.seq & 3u);
        a.wait_plan = 1; // (a.skip_wait: inside a run the gather skips the grid wait and spins on the plan-ready word)
        a.plan_word = scr->plan_word;
        a.plan_tiles = tiles;
    }
    return launch_gather<false>(a, st, cvt, form);
}

int ddsk_var_uses_scratch(int64_t nreq, int64_t dst_capacity, const ddsk_cvt_t *cvt, int host) {
    if (pick_geometry()) return 1;
    return select_s(nreq, dst_capacity, cvt, host != 0) < 0;
}

int ddsk_gather_var(const ddsk_var_t *var, const ddsk_index_t *index, int64_t nreq, void *dst_dev, int64_t dst_capacity,
                    int64_t *offsets_dev_or_null, ddsk_scratch_t *scr, int flags, const ddsk_cvt_t *cvt,
                    const ddsk_write_t *wr, void *stream) {
    if (nreq <= 0) return 0;
    GatherArgs a;
    if (int rc = gather_args(a, var, scr, flags)) return rc;
    const int form = write_form(a, wr);
    PlanSrc p;
    memset(&p, 0, sizeof(p));
    p.starts = index->starts;
    p.counts = index->counts;
    p.ids = index->sample_ids;
    p.tab = (const longlong2 *)index->table;
    p.nsamples = index->nsamples;
    a.dst = (char *)dst_dev;
    a.dst_cap = dst_capacity;
    return plan_and_gather(var, p, nreq, dst_capacity, a, offsets_dev_or_null, scr, flags, cvt, form, (cudaStream_t)stream);
}

int ddsk_gather_multi(const ddsk_multi_t *m, const int64_t *sample_ids_dev, int64_t nreq, ddsk_scratch_t *scr, int flags,
                      const ddsk_cvt_t *cvt, void *stream) {
    if (nreq <= 0 || m->nvars <= 0) return 0;
    if (m->nvars > DDSK_MAX_MULTI) {
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_gather_multi: more than %d variables", DDSK_MAX_MULTI);
        return -2;
    }
    ddsk_var_t dummy; // (each variable's window is read from m->vars_dev)
    memset(&dummy, 0, sizeof(dummy));
    dummy.host = m->host;
    GatherArgs a;
    if (int rc = gather_args(a, &dummy, scr, flags)) return rc;
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
    a.dst_cap = INT64_MAX;
    for (int v = 0; v < m->nvars; v++) {
        a.mdst[v] = (char *)m->dst[v];
        a.mcap[v] = m->cap[v];
        a.moffsets[v] = m->offsets[v];
    }
    return plan_and_gather(&dummy, p, nreq * m->nvars, cap_total, a, nullptr, scr, flags, cvt, kWrNone, (cudaStream_t)stream);
}

int ddsk_pool(const ddsk_var_t *var, const ddsk_index_t *index, int64_t fixed_count, int64_t nreq, const ddsk_pool_t *pool,
              void *dst, const ddsk_scratch_t *scr, int flags, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (pool->nbags <= 0 || var->row_bytes <= 0) return 0;
    if (int rc = pick_geometry()) return rc;
    PoolArgs a;
    pool_args(a, var, index, fixed_count, nreq, pool, scr);
    a.dst = (char *)dst;
    const PoolGeometry g = pool_geometry(false, var->row_bytes, pool->type, pool->nbags, (uint64_t)dst % 16 == 0, var->host);
    a.slice = g.slice;
    a.nslices = g.nslices;
    int rc = 0;
    switch (pool->type) {
    case DDSK_ACC_F32: rc = launch_pool_t<DDSK_ACC_F32>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_F64: rc = launch_pool_t<DDSK_ACC_F64>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_F16: rc = launch_pool_t<DDSK_ACC_F16>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_BF16: rc = launch_pool_t<DDSK_ACC_BF16>(a, g.vb, g.blocks, st); break;
    default:
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_pool: unsupported element type %d", (int)pool->type);
        return -2;
    }
    if (rc) return rc;
    if (flags & DDSK_F_MIRROR) // (a synchronous call reads the status from the pinned mirror word)
        CUDA_TRY(cudaMemcpyAsync(scr->host_mirror, scr->status, 8, cudaMemcpyDefault, st));
    return 0;
}

int ddsk_pool_acc(const ddsk_var_t *var, const ddsk_index_t *index, int64_t fixed_count, int64_t nreq,
                  const ddsk_pool_t *pool, double alpha, const void *grad, const ddsk_scratch_t *scr, int flags,
                  void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (pool->nbags <= 0 || var->row_bytes <= 0) return 0;
    if (int rc = pick_geometry()) return rc;
    PoolAccArgs a;
    pool_args(a.p, var, index, fixed_count, nreq, pool, scr);
    a.grad = (const char *)grad;
    a.alpha = alpha;
    // (the store refuses DDS_PLACE_HOST variables for every batched write: var->host is false here)
    const PoolGeometry g = pool_geometry(true, var->row_bytes, pool->type, pool->nbags, (uint64_t)grad % 16 == 0, var->host);
    a.p.slice = g.slice;
    a.p.nslices = g.nslices;
    a.windows = g.windows;
    int rc = 0;
    switch (pool->type) {
    case DDSK_ACC_F32: rc = launch_pool_acc_t<DDSK_ACC_F32>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_F64: rc = launch_pool_acc_t<DDSK_ACC_F64>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_F16: rc = launch_pool_acc_t<DDSK_ACC_F16>(a, g.vb, g.blocks, st); break;
    case DDSK_ACC_BF16: rc = launch_pool_acc_t<DDSK_ACC_BF16>(a, g.vb, g.blocks, st); break;
    default:
        snprintf(g_cuda_err, sizeof(g_cuda_err), "ddsk_pool_acc: unsupported element type %d", (int)pool->type);
        return -2;
    }
    if (rc) return rc;
    if (flags & DDSK_F_MIRROR) // (a synchronous call reads the status from the pinned mirror word)
        CUDA_TRY(cudaMemcpyAsync(scr->host_mirror, scr->status, 8, cudaMemcpyDefault, st));
    return 0;
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
