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
    int32_t host;                      /* 1: every shard is mapped host memory (DDS_PLACE_HOST), read over PCIe */
} ddsk_var_t;

/* status word written by the kernels: 0xFFFF... = ok, else (ordinal << 48) | (first_bad_request << 8) | code, where
 * ordinal is the launch's position in its queue of DDS_NO_SYNC batches (0 for a synchronous call; saturates at 0xFFFF).
 * Kernels only atomicMin into it, so the word holds the first error in queue order, and inside that batch the
 * lowest-index one. Request indices stay below 2^39: a pooled launch sets bit 39 of the index field (DDSK_STATUS_LATE) in
 * its request reports, so that its malformed-bag reports (DDSK_CODE_BAG, index = the bag) come first. */
#define DDSK_STATUS_OK 0xFFFFFFFFFFFFFFFFull
#define DDSK_STATUS_ORD_SHIFT 48
#define DDSK_STATUS_REQ_MASK 0x7FFFFFFFFFull /* (word >> 8) & this = request index */
#define DDSK_STATUS_LATE (1ull << 39)        /* in the index field: a report ordered after every bag report */
#define DDSK_CODE_START 2
#define DDSK_CODE_COUNT 3
#define DDSK_CODE_CAPACITY 12
#define DDSK_CODE_WATCHDOG 14
#define DDSK_CODE_SAMPLE 15
#define DDSK_CODE_BAG 16 /* a pooled launch's malformed bag offsets (index = the bag) */

/* scratch a store owns for the batched path (all device memory) */
typedef struct ddsk_scratch {
    unsigned long long *status; /* 1 word, sticky (kernels only atomicMin into it) */
    int64_t *total;             /* 1 word: packed total of the last variable-count launch planned in shared memory (and of
                                   a converting multi-array launch); an overlap launch gets the word of its slot */
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
#define DDSK_F_MIRROR 2     /* the kernel's last warp mirrors status + total into scr->host_mirror (synchronous calls;
                               costs time at the kernel's end, so async queues skip it) */
#define DDSK_F_OVERLAP 4    /* independent batch: static segment striding, overlap protocol (see kernels.cu) */
#define DDSK_F_SKIP_WAIT 16 /* ... and the launch right before it in the stream was one too: skip griddepcontrol.wait */
#define DDSK_F_PREV1 32     /* overlap launch ovl_seq-1 belongs to the same run (retire after it) */
#define DDSK_F_PREV2 64     /* overlap launch ovl_seq-2 belongs to the same run (do not write before it retired) */
#define DDSK_F_PREV4 128    /* overlap launch ovl_seq-4 belongs to the same run (it used the same plan scratch slot) */

/* ops of a batched write (same values as DDS_OP_* in include/ddstore_b200.h; DDSK_OP_PUT and DDSK_OP_CAS have no public
 * op code). Max and min compare integers as signed and floats by IEEE 754-2019 maximumNumber / minimumNumber with
 * -0 < +0; the bitwise ops take the integer types only. */
#define DDSK_OP_PUT 0     /* shard = src */
#define DDSK_OP_SUM 1     /* shard = shard + src */
#define DDSK_OP_REPLACE 2 /* shard = src (a fetch-op only: the swap) */
#define DDSK_OP_CAS 3     /* shard = src where shard == compare, bit for bit (a fetch-op only) */
#define DDSK_OP_MAX 4
#define DDSK_OP_MIN 5
#define DDSK_OP_BAND 6
#define DDSK_OP_BOR 7
#define DDSK_OP_BXOR 8

/* A batched write (ddsk_gather_fixed / ddsk_gather_var, raw, never with DDSK_F_OVERLAP): the get's walk with every copy
 * reversed. dst_dev is the caller's packed SOURCE rows and dst_capacity its size; request i's bytes are taken from its
 * packed position and written to its rows in the owner's shard, by `op`. The layout keeps an invalid request's bytes
 * (count * row_bytes when 0 < count <= the variable's rows, else 0; 0 for a sample id outside the index); it writes
 * nothing, like a layout above dst_capacity. No offsets.
 * - a put (DDSK_OP_PUT) stores the bytes;
 * - a reduction (any other op, result NULL: an accumulate) combines every element with the shard's atomically;
 * - a fetch-op (result set) applies an atomic that returns each element's previous value and writes that value to the
 *   same position of result as the operand's in the caller's rows. DDSK_OP_CAS is a fetch-op whose operands are compared
 *   with the compare operands at the same position of `compare`.
 * The caller's rows, result and compare are aligned to the element size. */
typedef struct ddsk_write {
    int32_t op;          /* DDSK_OP_* */
    int32_t type;        /* the element type (DDSK_ACC_*) of a sum or reduction (a fetch-op's too), else 0 */
    int32_t el_log2;     /* log2 of the element size (the type's, or the variable's itemsize) */
    void *result;        /* a fetch-op's previous values (device memory, the layout of the source rows), else NULL */
    const void *compare; /* DDSK_OP_CAS: the compare operands (device memory, the layout of the source rows), else NULL */
} ddsk_write_t;

/* element types of an accumulate (same values as DDS_ACC_* in include/ddstore_b200.h) */
#define DDSK_ACC_F32 1
#define DDSK_ACC_F64 2
#define DDSK_ACC_I32 3
#define DDSK_ACC_I64 4
#define DDSK_ACC_F16 5
#define DDSK_ACC_BF16 6
#define DDSK_ACC_LOG2(t) ((t) == DDSK_ACC_F64 || (t) == DDSK_ACC_I64 ? 3 : (t) >= DDSK_ACC_F16 ? 1 : 2)

/* Element conversion inside the gather (same values as DDS_CVT_* in include/ddstore_b200.h). Source byte p of a
 * variable's packed rows goes to output byte (p >> in_log2) << out_log2. */
#define DDSK_CVT_NONE 0      /* raw bytes (a variable of a multi-array batch that is not converted) */
#define DDSK_CVT_F32_BF16 1  /* 4 -> 2 bytes, cvt.rn.bf16.f32 */
#define DDSK_CVT_F32_F16 2   /* 4 -> 2 bytes, cvt.rn.f16.f32 */
#define DDSK_CVT_F64_F32 3   /* 8 -> 4 bytes, cvt.rn.f32.f64 */
#define DDSK_CVT_U8_LUT16 4  /* 1 -> 2 bytes, out = lut[in] */
#define DDSK_CVT_U8_LUT32 5  /* 1 -> 4 bytes, out = lut[in] */
/* normalising conversions: y = (decode(x) - mean[ch]) / std[ch] in f32 (two IEEE roundings), then encoded */
#define DDSK_CVT_NORM_F32_F32 6  /* 4 -> 4 bytes */
#define DDSK_CVT_NORM_F32_BF16 7 /* 4 -> 2 bytes */
#define DDSK_CVT_NORM_F32_F16 8  /* 4 -> 2 bytes */
#define DDSK_CVT_NORM_F64_F32 9  /* 8 -> 4 bytes, decode = cvt.rn.f32.f64 */
#define DDSK_CVT_NORM_U8_F32 10  /* 1 -> 4 bytes, decode = 256-entry f32 table */
#define DDSK_CVT_NORM_U8_BF16 11 /* 1 -> 2 bytes, decode = 256-entry f32 table */
#define DDSK_CVT_NORM_U8_F16 12  /* 1 -> 2 bytes, decode = 256-entry f32 table */
#define DDSK_CVT_MAX 12
#define DDSK_CVT_IS_NORM(c) ((c) >= DDSK_CVT_NORM_F32_F32)
/* source / output itemsize of a code, as log2: the one table the host and the kernels share. The _PLAIN forms cover codes
 * 0..5 only (the launches that carry no normalising code evaluate those). */
#define DDSK_CVT_PLAIN_IN_LOG2(c) ((c) == DDSK_CVT_F64_F32 ? 3 : ((c) == DDSK_CVT_F32_BF16 || (c) == DDSK_CVT_F32_F16) ? 2 : 0)
#define DDSK_CVT_PLAIN_OUT_LOG2(c) ((c) == DDSK_CVT_NONE ? 0 : ((c) == DDSK_CVT_F64_F32 || (c) == DDSK_CVT_U8_LUT32) ? 2 : 1)
#define DDSK_CVT_IN_LOG2(c) \
    (DDSK_CVT_IS_NORM(c) ? ((c) == DDSK_CVT_NORM_F64_F32 ? 3 : (c) >= DDSK_CVT_NORM_U8_F32 ? 0 : 2) : DDSK_CVT_PLAIN_IN_LOG2(c))
#define DDSK_CVT_OUT_LOG2(c)                                                                                              \
    (DDSK_CVT_IS_NORM(c) ? (((c) == DDSK_CVT_NORM_F32_F32 || (c) == DDSK_CVT_NORM_F64_F32 || (c) == DDSK_CVT_NORM_U8_F32) ? 2 : 1) \
                         : DDSK_CVT_PLAIN_OUT_LOG2(c))
/* The conversion of one launch, passed BY VALUE as a kernel parameter (so every queued launch carries its own tables).
 * code[v] is variable v's conversion; the tables of the variables with a LUT code (and the f32 decode tables of the
 * uint8 normalising codes) are packed into lut[] (lut_off[v] bytes in, 256 entries of the output itemsize -- 4 bytes for
 * the normalising codes) and copied to shared memory by every CTA. A variable with a normalising code also has norm[v]:
 * nchan {mean, std} f32 pairs in device memory the store owns (read through the non-coherent cache, never copied), and
 * element e of a row belongs to channel (e / inner) % nchan. */
typedef struct ddsk_cvt {
    int32_t code[DDSK_MAX_MULTI];
    int32_t lut_off[DDSK_MAX_MULTI];
    int32_t lut_bytes; /* bytes of lut[] in use (0..4096) */
    int32_t pad_;
    uint32_t lut[DDSK_MAX_MULTI * 256];
    const float *norm[DDSK_MAX_MULTI]; /* [nchan][2] = {mean, std} */
    int32_t nchan[DDSK_MAX_MULTI];     /* nchan * inner divides the variable's disp (< 2^31) */
    int32_t inner[DDSK_MAX_MULTI];
} ddsk_cvt_t;

/* Fixed-count batch: every request fetches `count` rows; offsets are i*count*row_bytes.
 * One launch: validate + owner lookup + gather + pack.
 * cvt (nullable): convert the elements on the way; dst_capacity is then in SOURCE bytes (the caller's output capacity
 * rounded down to whole elements, scaled), while offsets_dev_or_null receives OUTPUT byte offsets. The same holds for
 * ddsk_gather_var and ddsk_gather_multi (per variable).
 * wr (nullable): a batched write (see ddsk_write_t) instead of a get, here and in ddsk_gather_var; cvt is then NULL. */
int ddsk_gather_fixed(const ddsk_var_t *var, const int64_t *starts_dev, int64_t count, int64_t nreq, void *dst_dev,
                      int64_t dst_capacity, int64_t *offsets_dev_or_null, const ddsk_scratch_t *scr, int flags,
                      const ddsk_cvt_t *cvt, const ddsk_write_t *wr, void *stream);

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
                    const ddsk_cvt_t *cvt, const ddsk_write_t *wr, void *stream);
/* (cvt: the conversion the launch will carry, or NULL; its tables take shared memory from the in-launch plan. host: the
 * variable's ddsk_var_t.host -- HOST launches always plan in the plan kernels) */
int ddsk_var_uses_scratch(int64_t nreq, int64_t dst_capacity, const ddsk_cvt_t *cvt, int host);
int64_t ddsk_plan_smem_max(void);

/* Padded batch: request i owns a slot of max_rows rows. The walk runs over the padded SOURCE byte space [0, nreq * slot)
 * (slot = max_rows * row_bytes) exactly like a fixed-count batch whose requests are all `slot` bytes long; the first
 * `payload` = min(count_i, max_rows) * row_bytes bytes of slot i are rows (0 for an invalid request), the rest padding.
 * Source position p goes to output byte (p >> in_log2) << out_log2 (0 / 0 for raw batches, the conversion's otherwise),
 * and every padding element of the output is `pad_bits` (its low 1 << pad_log2 bytes), written verbatim. index: explicit
 * starts AND counts, or sample ids. lengths (nullable, device): nreq delivered row counts. cvt: NULL for raw bytes. */
int ddsk_gather_padded(const ddsk_var_t *var, const ddsk_index_t *index, int64_t nreq, int64_t max_rows, uint64_t pad_bits,
                       int pad_log2, int64_t *lengths, void *dst_dev, const ddsk_scratch_t *scr, int flags,
                       const ddsk_cvt_t *cvt, void *stream);

#if defined(__CUDACC__)
#define DDSK_HD __host__ __device__
#else
#define DDSK_HD
#endif

/* Segment size of a fixed-stride walk over T bytes of `nb`-byte requests by `nwarps` warps (chunk: CH; min_chunks: the
 * smallest segment in chunks): about 8 segments per warp, at most 1 MiB, whole requests when one fits, else whole chunks.
 * Every cut is therefore a request boundary or a multiple of CH. The padded gather uses it (tests/cpp/pad_layout_check.cpp
 * replays it). */
static inline DDSK_HD int64_t ddsk_fixed_seg_bytes(int64_t T, int64_t nb, int64_t nwarps, int64_t min_chunks, int64_t ch) {
    int64_t target = T / (nwarps * 8);
    if (target > ((int64_t)1 << 20)) target = (int64_t)1 << 20;
    if (target < min_chunks * ch) target = min_chunks * ch;
    if (target < ch) target = ch;
    return (nb > 0 && nb <= target) ? (target / nb) * nb : (target / ch) * ch;
}

/* The layout of a padded batch, for a source range [lo, hi) of slot i (0 <= lo <= hi <= slot) whose first `payload`
 * bytes are rows: which of those bytes are payload and where they go, and which OUTPUT bytes are padding. Source and
 * output positions are absolute (from the batch's start); lengths are in source bytes for the payload, output bytes for
 * the padding. Every cut the walk makes (slot boundaries, multiples of CH, row boundaries) is element-aligned, so the
 * shifts are exact. */
typedef struct ddsk_pad_cut {
    int64_t pay_src, pay_len; /* source range [pay_src, pay_src + pay_len) of rows */
    int64_t pay_dst;          /* its output position */
    int64_t pad_dst, pad_len; /* output range of padding */
} ddsk_pad_cut_t;
static inline DDSK_HD ddsk_pad_cut_t ddsk_pad_cut(int64_t i, int64_t payload, int64_t slot, int64_t lo, int64_t hi,
                                                  int in_log2, int out_log2) {
    ddsk_pad_cut_t c;
    const int64_t base = i * slot;
    const int64_t pe = payload < hi ? payload : hi;
    const int64_t ps = lo < pe ? lo : pe;
    const int64_t qs = lo > payload ? lo : payload;
    c.pay_src = base + ps;
    c.pay_len = pe - ps;
    c.pay_dst = ((base + ps) >> in_log2) << out_log2;
    c.pad_dst = ((base + qs) >> in_log2) << out_log2;
    c.pad_len = qs < hi ? ((hi - qs) >> in_log2) << out_log2 : 0;
    return c;
}

/* Pooled batch (dds_get_batch_pooled): bag k folds the rows of requests [bags[k], bags[k+1]) (bags NULL: request k) into
 * output row k of dst, by `mode` in element type `type` (the public DDS_POOL_* / DDS_ACC_* codes). index: explicit starts
 * (counts NULL: fixed_count rows each) or sample ids. bags and weights are device memory; the kernel checks the bags and
 * reports a malformed one as DDSK_CODE_BAG. The host has checked everything else (dst holds nbags rows, alignment). */
#define DDSK_POOL_SUM 1
#define DDSK_POOL_MEAN 2
#define DDSK_POOL_MAX 3
typedef struct ddsk_pool {
    int32_t mode, type;
    const int64_t *bags;
    int64_t nbags;
    const void *weights;
} ddsk_pool_t;
int ddsk_pool(const ddsk_var_t *var, const ddsk_index_t *index, int64_t fixed_count, int64_t nreq, const ddsk_pool_t *pool,
              void *dst, const ddsk_scratch_t *scr, int flags, void *stream);
/* Pooled accumulate (dds_accumulate_batch_pooled), the adjoint of ddsk_pool with the same requests and pool (mode SUM or
 * MEAN): every row of bag k's valid requests gets grad row k (times the request's weight, over the bag's valid rows for
 * a mean, times alpha) added atomically. grad is device memory holding nbags rows, aligned to the element size. */
int ddsk_pool_acc(const ddsk_var_t *var, const ddsk_index_t *index, int64_t fixed_count, int64_t nreq,
                  const ddsk_pool_t *pool, double alpha, const void *grad, const ddsk_scratch_t *scr, int flags,
                  void *stream);

/* Multi-array batch: the rows of the SAME nreq sample ids in nvars (<= DDSK_MAX_MULTI) variables, one launch. vars_dev =
 * device array of the variables' windows; table[v] = sample index of variable v; dst[v]/cap[v]/offsets[v] per variable
 * (offsets[v] nullable, nreq+1 entries). */
typedef struct ddsk_multi {
    int nvars;
    int host; /* every variable is HOST (a batch never mixes placements) */
    const ddsk_var_t *vars_dev;
    const int64_t *table[DDSK_MAX_MULTI]; /* [nsamples[v]][2] */
    int64_t nsamples[DDSK_MAX_MULTI];
    void *dst[DDSK_MAX_MULTI];
    int64_t cap[DDSK_MAX_MULTI];
    int64_t *offsets[DDSK_MAX_MULTI];
} ddsk_multi_t;
int ddsk_gather_multi(const ddsk_multi_t *m, const int64_t *sample_ids_dev, int64_t nreq, ddsk_scratch_t *scr, int flags,
                      const ddsk_cvt_t *cvt, void *stream);

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

/* launch geometry of a pooled get (adjoint 0) or pooled accumulate (adjoint 1); all zeros without a usable device or for
 * arguments no pooled launch takes */
void ddsk_pool_geometry(int adjoint, int64_t row_bytes, int type, int64_t nbags, int aligned16, int host, int *vb,
                        int64_t *slice, int64_t *nslices, int64_t *windows, int *blocks);

/* CTAs of a gather launch that reads DDS_PLACE_HOST shards */
int ddsk_host_gather_ctas(void);

/* number of kernels launched by this library since load (bench.py's gpu_launches) */
unsigned long long ddsk_launch_count(void);

const char *ddsk_last_cuda_error(void);

#ifdef __cplusplus
}
#endif
#endif
