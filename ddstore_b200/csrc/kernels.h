/* ddstore_b200/csrc/kernels.h -- the thin C-ABI between the host C++ store (store.cpp) and the
 * CUDA side (kernels.cu). Plain pointers, sizes and a cudaStream_t passed as void*. Nothing here
 * is public; the public boundary is include/ddstore_b200.h. */
#ifndef DDSK_KERNELS_H
#define DDSK_KERNELS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDSK_MAX_RANKS 64
#define DDSK_MAX_MULTI 4 /* variables per multi-array launch */

/* Device-visible description of one variable: what the reference keeps in VarInfo
 * (/root/reference/include/ddstore.hpp:10-22) minus the MPI window, plus the peer-mapped shard base
 * of every owner (the "window"). Passed BY VALUE as a kernel parameter (constant bank). */
typedef struct ddsk_var {
    const void *bases[DDSK_MAX_RANKS]; /* shard base of rank r as mapped into THIS process (IPC / peer) */
    int64_t lenlist[DDSK_MAX_RANKS];   /* inclusive cumulative row counts, ddstore.hpp:84-89 */
    int64_t row_bytes;                 /* disp * itemsize, the window's disp_unit, ddstore.hpp:58 */
    int32_t nranks;
    int32_t pad_;
} ddsk_var_t;

/* status word written by the kernels: 0xFFFF... = ok, else (ordinal << 48) | (first_bad_request << 8) | code, where
 * ordinal is the launch's position in its queue of DDS_NO_SYNC batches (0 for a synchronous call; saturates at 0xFFFF).
 * Kernels only atomicMin into it, so the word holds the first error in queue order, and inside that batch the
 * lowest-index one. Request indices stay below 2^40. */
#define DDSK_STATUS_OK 0xFFFFFFFFFFFFFFFFull
#define DDSK_STATUS_ORD_SHIFT 48
#define DDSK_STATUS_REQ_MASK 0xFFFFFFFFFFull /* (word >> 8) & this = request index */
#define DDSK_CODE_START 2
#define DDSK_CODE_COUNT 3
#define DDSK_CODE_CAPACITY 12
#define DDSK_CODE_WATCHDOG 14
#define DDSK_CODE_SAMPLE 15

/* scratch a store owns for the batched path (all device memory) */
typedef struct ddsk_scratch {
    unsigned long long *status; /* 1 word, sticky (kernels only atomicMin into it) */
    int64_t *total;             /* 1 word: packed total of the last variable-count launch planned in shared memory */
    unsigned int *counters;     /* 2 words: [0] segment ticket, [1] finished warps -- self-resetting */
    unsigned int *ovl;          /* 24 words of the overlap protocol, one of each kind per slot (sequence number & 3):
                                   finished-warp counters, done words, segment tickets, lookup tiles done, scan tiles
                                   done, plan-ready words */
    unsigned long long *plan_word; /* 8 words: [0..3] per slot (sequence number & 0xFFFFFF) << 40 | packed total ("plan
                                      ready"), [4..7] per slot the packed total parked by the plan kernel's last tile */
    unsigned int ovl_seq;       /* sequence number the NEXT overlap launch carries (host side, set by the caller) */
    unsigned long long status_tag; /* ordinal << DDSK_STATUS_ORD_SHIFT of the NEXT launch (host side, set by the caller) */
    /* plan in global memory (variable-count batches above ddsk_plan_smem_max() requests, or >= 4 GiB destinations) */
    uint64_t *req_src;          /* [cap_req]   planned source address per request (0 = skip) */
    int64_t *req_dst;           /* [cap_req+1] exclusive scan of request bytes */
    int64_t *tile_sums;         /* [cap_req/1024 + 2] look-back words of the plan kernel (tagged per launch, never cleared) */
    unsigned int plan_tag;      /* host-side launch counter tagging them (22 bits; 0 = never used) */
    int64_t cap_req;
    uint32_t *seg_tab;          /* [seg_cap] request covering byte k * 16384 of the packed buffer */
    int64_t seg_cap;
    unsigned long long *host_mirror; /* device alias of pinned host words: [0] status, [1] packed total (written by the
                                        last warp of a gather launch that asks for it), [2] ticket of dds_small_get */
} ddsk_scratch_t;

/* `flags` of the launchers */
#define DDSK_F_RESET 1      /* reset the status word first */
#define DDSK_F_MIRROR 2     /* the kernel's last warp mirrors status + total into scr->host_mirror (synchronous calls;
                               costs time at the kernel's end, so async queues skip it) */
#define DDSK_F_OVERLAP 4    /* independent batch: static segment striding, overlap protocol (see kernels.cu) */
#define DDSK_F_SKIP_WAIT 16 /* ... and the launch right before it in the stream was one too: skip griddepcontrol.wait */
#define DDSK_F_PREV1 32     /* overlap launch ovl_seq-1 belongs to the same run (retire after it) */
#define DDSK_F_PREV2 64     /* overlap launch ovl_seq-2 belongs to the same run (do not write before it retired) */
#define DDSK_F_PREV4 128    /* overlap launch ovl_seq-4 belongs to the same run (it used the same plan scratch slot) */

/* Fixed-count batch: every request fetches `count` rows; offsets are i*count*row_bytes.
 * One launch: validate + owner lookup + gather + pack. */
int ddsk_gather_fixed(const ddsk_var_t *var, const int64_t *starts_dev, int64_t count, int64_t nreq, void *dst_dev,
                      int64_t dst_capacity, int64_t *offsets_dev_or_null, const ddsk_scratch_t *scr, int flags,
                      void *stream);

/* Where the (start row, row count) of request i comes from (all device pointers): explicit arrays, or -- when
 * sample_ids is set -- the per-sample table of the variable: {start, count} = table[sample_ids[i]] (int64 pairs). */
typedef struct ddsk_index {
    const int64_t *starts, *counts;
    const int64_t *sample_ids;
    const int64_t *table; /* [nsamples][2] */
    int64_t nsamples;
} ddsk_index_t;

/* Variable-count batch: plan (lookup + validate + exclusive scan) then gather + pack. The plan runs inside the gather
 * launch (every CTA for itself, in shared memory) for small batches into < 4 GiB; else in two plan kernels writing the
 * scratch arrays of `scr` (ddsk_var_uses_scratch tells which). With DDSK_F_OVERLAP the scratch arrays must be a slot
 * of the launch's own (slot = ovl_seq & 3): the plan then runs under the previous batch's gather. */
int ddsk_gather_var(const ddsk_var_t *var, const ddsk_index_t *index, int64_t nreq, void *dst_dev,
                    int64_t dst_capacity, int64_t *offsets_dev_or_null, ddsk_scratch_t *scr, int flags,
                    void *stream);
int ddsk_var_uses_scratch(int64_t nreq, int64_t dst_capacity);
int64_t ddsk_plan_smem_max(void);

/* Multi-array batch: the rows of the SAME nreq sample ids in nvars (<= DDSK_MAX_MULTI) variables, one launch. vars_dev =
 * device array of the variables' windows; table[v] = sample index of variable v; dst[v]/cap[v]/offsets[v] per variable
 * (offsets[v] nullable, nreq+1 entries). */
typedef struct ddsk_multi {
    int nvars;
    const ddsk_var_t *vars_dev;
    const int64_t *table[DDSK_MAX_MULTI]; /* [nsamples[v]][2] */
    int64_t nsamples[DDSK_MAX_MULTI];
    void *dst[DDSK_MAX_MULTI];
    int64_t cap[DDSK_MAX_MULTI];
    int64_t *offsets[DDSK_MAX_MULTI];
} ddsk_multi_t;
int ddsk_gather_multi(const ddsk_multi_t *m, const int64_t *sample_ids_dev, int64_t nreq, ddsk_scratch_t *scr, int flags,
                      void *stream);

/* Collective owner-push fetch (fixed-count batches, every rank on its own GPU). Each rank owns a WINDOW -- a peer-mapped
 * block of the store -- holding a header, two index lists and two destination buffers (alternating by step parity).
 * Header, as 64-bit words: [0] ready (the step whose index list is published), [1 + parity] number of requests,
 * [3] sticky status (atomicMin, written by the owners), [8 + r] arrive (the step for which owner r's rows have landed). */
#define DDSK_PUSH_HDR_BYTES 4096
typedef struct ddsk_push {
    int32_t nranks, me;
    unsigned char *win[DDSK_MAX_RANKS]; /* rank r's window as mapped into this process */
    int64_t idx_off[2], dst_off[2];     /* byte offsets inside a window */
    int64_t max_requests, max_bytes;
} ddsk_push_t;
/* One step of the collective fetch: publish this rank's `nreq` start rows (device array), wait for every rank's list,
 * push the rows THIS rank owns into the requesters' windows, wait until every owner's rows have landed here.
 * push_host / push_dev: the table above and its device copy. Result: window dst buffer [step & 1]. */
int ddsk_gather_push(const ddsk_var_t *var, const ddsk_push_t *push_host, const ddsk_push_t *push_dev,
                     const int64_t *starts_dev, int64_t count, int64_t nreq, unsigned long long step,
                     const ddsk_scratch_t *scr, void *stream);

/* One request in a 1-CTA kernel (the legacy per-sample get()): checks + copy into `dst` (device memory or mapped pinned
 * host memory), then flag[0] = status word, flag[1] = bytes, flag[2] = ticket (flag = mapped pinned host words). */
int ddsk_small_get(const ddsk_var_t *var, int64_t start, int64_t count, void *dst, int64_t dst_capacity,
                   unsigned long long *flag_dev, unsigned long long ticket, void *stream);

/* Synthetic payload (SURVEY.md 8d): element (global_row g, col c) = low itemsize bytes of
 * splitmix64(seed ^ (g*disp + c)). Bench / test helper, fills a local shard in place. */
int ddsk_synth_fill(void *base_dev, int64_t first_global_row, int64_t nrows, int64_t disp, int itemsize, uint64_t seed,
                    void *stream);

/* Mailbox of the doorbell kernel (mapped pinned host memory; request line written by the host, answer line by the
 * device). resp = (req_seq << 8) | code, code 0 = ok, else DDSK_CODE_*; exit_gen = generation of the kernel that left. */
typedef struct ddsk_mailbox {
    /* request line (64 bytes, read by the device in one piece): the host writes the fields, then seq_tail, then seq_head */
    unsigned long long seq_head;
    int64_t start, count;
    uint64_t dst;
    int64_t dst_cap;
    uint64_t var_stop; /* low 32 bits: index into the device table of windows; bit 32: this request asks the kernel to leave */
    unsigned long long pad0_;
    unsigned long long seq_tail;
    unsigned long long pad_[8];
    /* answer line (written by the device) */
    unsigned long long resp;
    unsigned long long exit_gen;
    unsigned long long pad2_[14];
} ddsk_mailbox_t;
/* One resident CTA serving single-row requests from the mailbox until idle for idle_ns; `served` = last sequence number
 * already answered, `gen` = this kernel's generation (written to exit_gen when it leaves). */
int ddsk_doorbell_launch(const ddsk_var_t *vars_dev, ddsk_mailbox_t *mailbox_dev, unsigned long long served,
                         unsigned long long gen, unsigned long long idle_ns, void *stream);

/* Check a packed batch against the generator on the device: request i = rows [starts[i], +counts[i] or fixed_count) at
 * byte offset offsets[i] (or i * fixed_count * disp * itemsize). out_dev: 2 + DDSK_MAX_RANKS words, accumulated into:
 * [0] mismatching elements, [1] rows checked, [2 + r] requests owned by rank r. */
int ddsk_synth_verify(const ddsk_var_t *var, const void *packed_dev, const int64_t *starts_dev,
                      const int64_t *counts_dev_or_null, int64_t fixed_count, const int64_t *offsets_dev_or_null,
                      int64_t nreq, int64_t disp, int itemsize, uint64_t seed, unsigned long long *out_dev, void *stream);

/* pull [base, base + bytes) into the persisting part of L2 (no-op with DDS_L2_PERSIST=0) */
int ddsk_l2_warm(const void *base_dev, size_t bytes, void *stream);

/* test helper: `ctas` CTAs holding `smem_bytes` of shared memory each for `ns` nanoseconds on `stream` */
int ddsk_occupy(int ctas, int smem_bytes, unsigned long long ns, void *stream);

/* DDS_DEBUG_TIMING=1: per-CTA globaltimer stamps [entry, plan done, first data, last warp done] of the last gather launch */
int ddsk_debug_timing(unsigned long long *host_out, int max_ctas);

/* launch geometry actually used (for bench reporting / DESIGN.md) */
void ddsk_gather_geometry(int *ctas, int *warps_per_cta, int *stages, int *chunk_bytes, int *smem_bytes);

/* number of kernels launched by this library since load (bench.py's gpu_launches) */
unsigned long long ddsk_launch_count(void);

const char *ddsk_last_cuda_error(void);

#ifdef __cplusplus
}
#endif
#endif
