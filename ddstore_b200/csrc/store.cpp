// ddstore_b200/csrc/store.cpp -- host side of the store: the reference's `class DDStore`
// (/root/reference/include/ddstore.hpp:26-258, src/ddstore.cxx:19-96) re-built for H100:
//   * a variable's shard is a CUDA VMM block of this rank's HBM (reference: MPI_Alloc_mem + memcpy,
//     ddstore.hpp:44-49);
//   * the "window" is the table of every rank's shard base mapped into this process (VMM handle passed as a file
//     descriptor; reference: MPI_Win_create, ddstore.hpp:56-61) -- NVSwitch makes every peer equally near;
//   * lenlist / disp bookkeeping is the reference's (ddstore.hpp:75-89);
//   * get() of a batch is a launch of the batched-gather kernel in kernels.cu (reference: MPI_Win_lock / MPI_Get /
//     MPI_Win_unlock per sample, ddstore.hpp:222-237); a single get() is a mailbox round trip to a resident CTA;
//   * epoch_begin/epoch_end are stream-sync + barrier with the reference's state machine
//     (MPI_Win_fence, ddstore.cxx:51-77).
// Also here: the bookkeeping of overlap runs (sequence numbers, scratch slots), the doorbell kernel's lifecycle, the
// worker-thread pool of the pipelined host copies (ingest, pageable destinations), the windows of the collective
// push fetch. All CUDA work goes through the CUDA runtime C API and the ddsk_* launchers (kernels.h).
// There is no CPU data path: if no device is usable, dds_create fails with DDS_ERR_NO_DEVICE.
#include <cuda_runtime_api.h>
#include <sched.h>
#include <sys/random.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "ddstore_b200.h"
#include "internal.h"
#include "kernels.h"
#include "vmm.h"


namespace {

constexpr int64_t kSmallIdx = 8;          // requests whose host indices are read zero-copy (more go through an H2D copy)
constexpr int64_t kSmallOut = 64 * 1024;  // host destinations up to this size are written zero-copy

thread_local std::string g_err;

const char *code_text(int code) {
    switch (code) {
    case DDS_OK: return "";
    case DDS_ERR_DTYPE: return "Invalid data type";
    case DDS_ERR_START: return "Invalid start on target";
    case DDS_ERR_COUNT: return "Invalid count on target";
    case DDS_ERR_DISP: return "Invalid disp";
    case DDS_ERR_FENCE_ACTIVE: return "Fence already activated";
    case DDS_ERR_FENCE_INACTIVE: return "Fence is not activated";
    case DDS_ERR_UNKNOWN_VAR: return "Unknown variable";
    case DDS_ERR_EXISTS: return "Variable already exists";
    case DDS_ERR_CUDA: return "CUDA error";
    case DDS_ERR_COMM: return "Communicator error";
    case DDS_ERR_ARG: return "Invalid argument";
    case DDS_ERR_CAPACITY: return "Destination buffer too small for the packed batch";
    case DDS_ERR_NO_DEVICE: return "No usable CUDA device (ddstore_b200 has no CPU fallback)";
    case DDS_ERR_WATCHDOG: return "Gather kernel watchdog fired";
    default: return "Unknown error";
    }
}

} // namespace

namespace dds_internal {
int fail(int code, const std::string &detail) {
    // codes 1-6 keep the reference's exception text EXACTLY; the others append detail
    g_err = code_text(code);
    if (code > DDS_ERR_FENCE_INACTIVE && !detail.empty()) g_err += ": " + detail;
    return code;
}
void clear_error() { g_err.clear(); }
} // namespace dds_internal

using dds_internal::clear_error;
using dds_internal::fail;

namespace {

int cuda_fail(cudaError_t e, const char *what) {
    char buf[384];
    snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInitializationError)
        return fail(DDS_ERR_NO_DEVICE, buf);
    return fail(DDS_ERR_CUDA, buf);
}
#define CU(expr)                                     \
    do {                                             \
        cudaError_t e__ = (expr);                    \
        if (e__ != cudaSuccess) return cuda_fail(e__, #expr); \
    } while (0)

struct PeerRec { // what every rank publishes in add()/init(): the reference's Allgather(nrows) + Allreduce(disp)
                 // + Win_create rolled into one exchange
    int64_t nrows;
    int32_t disp;
    int32_t itemsize;
    int32_t pid;
    int32_t device;
    uint64_t raw_ptr;
    uint64_t host_tag;
    uint64_t alloc_bytes; // mapped size of the shard block
    int32_t vmm;          // 1: CUDA VMM block shared by POSIX fd; 0: cudaMalloc + legacy cudaIpc handle
    int32_t ok;           // 0: this rank failed locally (bad argument, allocation, fill): every rank fails the call
    int32_t placement;    // DDS_PLACE_*: every rank must pass the same
    int32_t pad_;
    cudaIpcMemHandle_t handle;
};

struct Var {
    std::string name;
    int itemsize = 0;
    int disp = 0;
    int64_t nrows = 0; // local
    std::vector<int64_t> lenlist;
    void *base = nullptr; // local shard (device)
    size_t bytes = 0;
    bool vmm = false;               // shard is a CUDA VMM block (else cudaMalloc)
    bool host = false;              // DDS_PLACE_HOST: shard is a mapped host block, shared by memfd (never vmm)
    dds_vmm::Block block;           // valid when vmm or host
    std::vector<void *> peer_base;  // as mapped here
    std::vector<char> peer_opened;  // 1 = cudaIpcOpenMemHandle'd (must be closed), 2 = VMM import (peer_block)
    bool unprotected_peers = false; // a peer reads this shard through a raw pointer / legacy IPC mapping: the memory
                                    // must not go away before that peer is done (VMM imports hold their own reference)
    std::vector<dds_vmm::Block> peer_block;
    bool fence_active = false;
    ddsk_var_t kv;
    int id = -1; // slot of kv in the store's device table of windows (doorbell kernel); -1: not there
    // per-sample index (SURVEY.md 8f rank 2): sample i owns rows [tab_start[i], tab_start[i] + tab_count[i])
    int64_t *d_tab = nullptr; // [nsamples][2] = {row_start, row_count}: one 16-byte load per sample id
    int64_t nsamples = 0;
    std::vector<int64_t> h_tab_count;
    // per-channel normalisation (dds_set_normalization): element e of a row is in channel (e / norm_inner) % norm_nchan
    float *d_norm = nullptr; // [norm_nchan][2] = {mean, std}: one 8-byte load per element
    int64_t norm_nchan = 0, norm_inner = 1;
};

} // namespace

// Streaming ingest (SURVEY.md 8f rank 3): a few worker threads copy slices of a pageable source chunk into a pinned
// staging buffer in parallel (one thread's memcpy cannot keep a PCIe Gen5 x16 link busy), while
// the copy engine moves the previous staging buffer into the shard.
struct IngestPool {
    static constexpr size_t kStage = 16u << 20; // bytes per staging buffer
    char *pin[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    bool ev_pending[2] = {false, false};
    cudaStream_t stream = nullptr;
    int next = 0;
    // fork-join pool
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_go, cv_done;
    unsigned long long gen = 0;
    int remaining = 0;
    bool quit = false;
    const char *src = nullptr;
    char *dst = nullptr;
    size_t bytes = 0;

    void worker(int idx, int n) {
        unsigned long long seen = 0;
        while (true) {
            std::unique_lock<std::mutex> lk(mu);
            cv_go.wait(lk, [&] { return quit || gen != seen; });
            if (quit) return;
            seen = gen;
            const char *sp = src;
            char *dp = dst;
            const size_t total = bytes;
            lk.unlock();
            const size_t per = ((total + n - 1) / n + 4095) & ~(size_t)4095;
            const size_t lo = std::min(total, per * (size_t)idx), hi = std::min(total, lo + per);
            if (hi > lo) memcpy(dp + lo, sp + lo, hi - lo);
            lk.lock();
            if (--remaining == 0) cv_done.notify_one();
        }
    }
    void start(int n) {
        for (int i = 0; i < n; i++) workers.emplace_back([this, i, n] { worker(i, n); });
    }
    void copy(char *d, const char *sp, size_t n) { // all workers copy their slice of [sp, sp + n) to d; returns when done
        std::unique_lock<std::mutex> lk(mu);
        src = sp;
        dst = d;
        bytes = n;
        remaining = (int)workers.size();
        gen++;
        cv_go.notify_all();
        cv_done.wait(lk, [&] { return remaining == 0; });
    }
    void stop() {
        {
            std::lock_guard<std::mutex> lk(mu);
            quit = true;
        }
        cv_go.notify_all();
        for (auto &t : workers) t.join();
        workers.clear();
    }
};

struct dds_store {
    dds_comm_t *comm = nullptr;
    int rank = 0, size = 1, device = 0, method = 0;
    cudaStream_t stream = nullptr;
    std::map<std::string, Var> vars;
    std::vector<void *> zombies; // shards of failed add()s, kept until free so no peer mapping dangles
    std::vector<dds_vmm::Block> zombie_blocks;
    unsigned long long token = 0; // job-unique tag for the descriptor-passing sockets
    unsigned long long reg_seq = 0;
    // scratch for the batched path
    ddsk_scratch_t scr;
    int64_t *d_starts = nullptr, *d_counts = nullptr;
    int64_t idx_cap = 0;
    void *d_out = nullptr;
    int64_t out_cap = 0;
    unsigned long long *h_status = nullptr; // pinned: [0] status, [1] total bytes
    // small-call fast path (the legacy one-get-per-sample loader): zero-copy pinned bounce buffers the kernel reads
    // indices from / writes the payload to directly, so a small host-to-host call is one launch + one sync
    char *h_small = nullptr, *d_small = nullptr; // kSmallIdx*16 bytes of indices + kSmallOut bytes of payload
    // The queue of DDS_NO_SYNC batches and the overlap run it may hold. Only the queue functions touch it (begin_call,
    // launch_flags, end_launch, note_empty_async, break_run, drain_pending, dds_batch_wait).
    struct Queue {
        bool pending = false; // launches are queued and not drained yet
        cudaStream_t pending_stream = nullptr;
        int64_t pending_fixed_total = -1;           // total of the last queued batch as the host knows it (-1: below)
        const int64_t *pending_total_ptr = nullptr; // device word holding the packed total of the last queued launch
        int pending_cvt = 0;                        // that word is in source bytes of this conversion (DDSK_CVT_*)
        bool pending_put = false;                   // the pending queue holds a batched put (dds_epoch_begin completes it)
        unsigned int queue_len = 0; // launches in the current queue (< kQueueMax, see launch_flags)
        // overlap protocol (DDS_OVERLAP): sequence number of the next overlap launch, and how many overlap launches in
        // a row were chained on the pending stream right before it (0: the next one starts a new run)
        unsigned int ovl_seq = 1;
        int run_len = 0;
        // outcome of queues completed by calls other than dds_batch_wait (drain_pending), reported by the next
        // dds_batch_wait: the first failing status word in queue order, and the total of the last batch queued
        unsigned long long kept_status = DDSK_STATUS_OK;
        int64_t kept_total = 0;
    } q;
    ddsk_var_t *d_multi_vars = nullptr; // device copy of the windows of the last multi-array combination
    std::string multi_key;
    // plan scratch slots of overlapped variable-count batches: launch q plans into slot q & 3, so its plan kernels can
    // run while the gather of launch q-1 is still reading slot (q-1) & 3
    struct Slot {
        uint64_t *req_src = nullptr;
        int64_t *req_dst = nullptr, *tile_sums = nullptr;
        uint32_t *seg_tab = nullptr;
        int64_t cap_req = 0, seg_cap = 0;
    } slots[4];
    int64_t *d_offs = nullptr; // device staging of byte offsets (host destinations, multi-array totals)
    int64_t offs_cap = 0;
    unsigned long long small_ticket = 0; // ticket of the last dds_small_get launch
    // doorbell (launch-free single-request path): a mailbox in mapped pinned memory and one resident CTA polling it
    static constexpr int kMaxDbVars = 256;
    ddsk_mailbox_t *h_mb = nullptr, *d_mb = nullptr;
    cudaStream_t db_stream = nullptr;
    ddsk_var_t *d_vars = nullptr;
    int next_var_id = 0;
    unsigned long long db_seq = 0, db_gen = 0, db_idle_ns = 200000;
    bool db_alive = false, db_enabled = true;
    std::set<cudaStream_t> update_streams; // caller streams that carried dds_update_async copies since the last fence
    IngestPool *ingest = nullptr;
    // collective owner-push fetch: the windows are an internal byte variable of the store (so the ordinary shard
    // machinery allocates, exports and maps them on every rank)
    struct Push {
        bool ready = false;
        ddsk_push_t table;
        ddsk_push_t *d_table = nullptr;
        unsigned long long step = 0;
    } push;
};

namespace {

uint64_t host_tag() {
    char buf[256] = {0};
    gethostname(buf, sizeof(buf) - 1);
    uint64_t h = 1469598103934665603ull;
    for (char *p = buf; *p; p++) h = (h ^ (unsigned char)*p) * 1099511628211ull;
    return h;
}

// ---- doorbell kernel lifecycle
// ask the resident CTA (if any) to leave and wait until it has: needed before anything that synchronises the device
int db_stop(dds_store *s) {
    if (!s->db_alive) return DDS_OK;
    volatile ddsk_mailbox_t *mb = s->h_mb;
    if (mb->exit_gen != s->db_gen) {
        mb->var_stop = 1ull << 32;
        std::atomic_thread_fence(std::memory_order_release);
        const unsigned long long q = ++s->db_seq;
        mb->seq_tail = q;
        std::atomic_thread_fence(std::memory_order_release);
        mb->seq_head = q;
        for (unsigned spins = 0; mb->exit_gen != s->db_gen; spins++) {
            if ((spins & 0xFFFF) == 0xFFFF && cudaStreamQuery(s->db_stream) != cudaErrorNotReady) break;
#if defined(__x86_64__)
            __builtin_ia32_pause();
#endif
        }
    }
    s->db_alive = false;
    cudaError_t e = cudaStreamSynchronize(s->db_stream);
    if (e != cudaSuccess) return cuda_fail(e, "doorbell kernel");
    return DDS_OK;
}

cudaError_t device_sync(dds_store *s) {
    db_stop(s);
    return cudaDeviceSynchronize();
}

// The next overlap launch starts a new run: it waits for the grid before it rather than overlapping with its tail.
void break_run(dds_store *s) { s->q.run_len = 0; }

// scratch of the plan kernels (variable-count batches the shared-memory plan does not take)
int ensure_scratch(dds_store *s, int64_t nreq, int64_t cap_bytes) {
    if (nreq > s->scr.cap_req) {
        int64_t cap = std::max<int64_t>(16384, s->scr.cap_req);
        while (cap < nreq) cap *= 2;
        CU(device_sync(s)); // nothing queued may still be reading the old arrays
        if (s->scr.req_src) cudaFree(s->scr.req_src);
        if (s->scr.req_dst) cudaFree(s->scr.req_dst);
        if (s->scr.tile_sums) cudaFree(s->scr.tile_sums);
        s->scr.req_src = nullptr;
        s->scr.req_dst = nullptr;
        s->scr.tile_sums = nullptr;
        s->scr.cap_req = 0;
        CU(cudaMalloc((void **)&s->scr.req_src, (size_t)cap * 8));
        CU(cudaMalloc((void **)&s->scr.req_dst, (size_t)(cap + 1) * 8));
        CU(cudaMalloc((void **)&s->scr.tile_sums, (size_t)(cap / 1024 + 2) * 8));
        CU(cudaMemset(s->scr.tile_sums, 0, (size_t)(cap / 1024 + 2) * 8));
        s->scr.cap_req = cap;
    }
    const int64_t need = cap_bytes / 16384 + 2; // one entry per SEG_GRAIN of the packed buffer
    if (need > s->scr.seg_cap) {
        int64_t cap = std::max<int64_t>(1 << 16, s->scr.seg_cap);
        while (cap < need) cap *= 2;
        CU(device_sync(s));
        if (s->scr.seg_tab) cudaFree(s->scr.seg_tab);
        s->scr.seg_tab = nullptr;
        s->scr.seg_cap = 0;
        CU(cudaMalloc((void **)&s->scr.seg_tab, (size_t)cap * 4));
        s->scr.seg_cap = cap;
    }
    return DDS_OK;
}

int ensure_slots(dds_store *s, int64_t nreq, int64_t cap_bytes) {
    const int64_t need_seg = cap_bytes / 16384 + 2;
    if (nreq <= s->slots[0].cap_req && need_seg <= s->slots[0].seg_cap) return DDS_OK;
    int64_t cap = std::max<int64_t>(16384, s->slots[0].cap_req), scap = std::max<int64_t>(1 << 16, s->slots[0].seg_cap);
    while (cap < nreq) cap *= 2;
    while (scap < need_seg) scap *= 2;
    CU(device_sync(s)); // nothing queued may still be using the old slots
    break_run(s);
    for (auto &sl : s->slots) {
        if (sl.req_src) cudaFree(sl.req_src);
        if (sl.req_dst) cudaFree(sl.req_dst);
        if (sl.tile_sums) cudaFree(sl.tile_sums);
        if (sl.seg_tab) cudaFree(sl.seg_tab);
        sl = dds_store::Slot();
        CU(cudaMalloc((void **)&sl.req_src, (size_t)cap * 8));
        CU(cudaMalloc((void **)&sl.req_dst, (size_t)(cap + 1) * 8));
        CU(cudaMalloc((void **)&sl.tile_sums, (size_t)(cap / 1024 + 2) * 8));
        CU(cudaMemset(sl.tile_sums, 0, (size_t)(cap / 1024 + 2) * 8));
        CU(cudaMalloc((void **)&sl.seg_tab, (size_t)scap * 4));
        sl.cap_req = cap;
        sl.seg_cap = scap;
    }
    return DDS_OK;
}

// The plan kernel tags its look-back words with a 22-bit launch counter instead of clearing them; shortly before the
// counter wraps, clear every scratch area once and start over.
int renew_plan_tags(dds_store *s) {
    if (s->scr.plan_tag < 0x3FFFF0u) return DDS_OK;
    CU(device_sync(s));
    break_run(s);
    if (s->scr.tile_sums) CU(cudaMemset(s->scr.tile_sums, 0, (size_t)(s->scr.cap_req / 1024 + 2) * 8));
    for (auto &sl : s->slots)
        if (sl.tile_sums) CU(cudaMemset(sl.tile_sums, 0, (size_t)(sl.cap_req / 1024 + 2) * 8));
    s->scr.plan_tag = 0;
    return DDS_OK;
}

// Whether a variable-count launch of nreq requests into cap (source) bytes is planned by the plan kernels rather than
// in shared memory, and if so their scratch made ready: an overlapped launch plans into a slot of its own.
int plan_scratch(dds_store *s, int64_t nreq, int64_t cap, const ddsk_cvt_t *cvt, bool ovl, bool host, bool *uses_scratch) {
    *uses_scratch = ddsk_var_uses_scratch(nreq, cap, cvt, host);
    if (!*uses_scratch) return DDS_OK;
    if (int rc = renew_plan_tags(s)) return rc;
    return ovl ? ensure_slots(s, nreq, cap) : ensure_scratch(s, nreq, cap);
}

// The scratch a launch works in: the store's own arrays, or -- for an overlap launch planned by the plan kernels
// (`slot`) -- slot (sequence number & 3).
// An overlap launch (`ovl`) reports its packed total in a device word of its slot, behind the plan words. The store's
// single total word cannot serve an overlapped run: a launch planned in shared memory writes it at its start, a
// converting multi-array launch at the end of its walk, and launch q may start before launch q-1 has retired, so q-1
// could overwrite q's total. Slot q & 3 is next written by launch q+4, which writes nothing before launch q+2 -- and
// so q -- has retired.
ddsk_scratch_t scratch_view(dds_store *s, bool ovl, bool slot) {
    ddsk_scratch_t v = s->scr;
    const unsigned int q = s->scr.ovl_seq & 3u;
    if (slot) {
        const dds_store::Slot &sl = s->slots[q];
        v.req_src = sl.req_src;
        v.req_dst = sl.req_dst;
        v.tile_sums = sl.tile_sums;
        v.seg_tab = sl.seg_tab;
        v.cap_req = sl.cap_req;
        v.seg_cap = sl.seg_cap;
    }
    if (ovl) v.total = (int64_t *)(s->scr.counters + 48) + q;
    return v;
}

int ensure_offs(dds_store *s, int64_t n) {
    if (n <= s->offs_cap) return DDS_OK;
    int64_t cap = std::max<int64_t>(4096, s->offs_cap);
    while (cap < n) cap *= 2;
    CU(device_sync(s));
    if (s->d_offs) cudaFree(s->d_offs);
    s->d_offs = nullptr;
    s->offs_cap = 0;
    CU(cudaMalloc((void **)&s->d_offs, (size_t)cap * 8));
    s->offs_cap = cap;
    return DDS_OK;
}

int ensure_idx(dds_store *s, int64_t nreq) {
    if (nreq <= s->idx_cap) return DDS_OK;
    int64_t cap = std::max<int64_t>(4096, s->idx_cap);
    while (cap < nreq) cap *= 2;
    if (s->d_starts) cudaFree(s->d_starts);
    if (s->d_counts) cudaFree(s->d_counts);
    s->d_starts = s->d_counts = nullptr;
    s->idx_cap = 0;
    CU(cudaMalloc((void **)&s->d_starts, (size_t)cap * 8));
    CU(cudaMalloc((void **)&s->d_counts, (size_t)cap * 8));
    s->idx_cap = cap;
    return DDS_OK;
}

int ensure_out(dds_store *s, int64_t bytes) {
    if (bytes <= s->out_cap) return DDS_OK;
    int64_t cap = std::max<int64_t>(1 << 20, s->out_cap);
    while (cap < bytes) cap *= 2;
    if (s->d_out) cudaFree(s->d_out);
    s->d_out = nullptr;
    s->out_cap = 0;
    CU(cudaMalloc(&s->d_out, (size_t)cap));
    s->out_cap = cap;
    return DDS_OK;
}

Var *find_var(dds_store *s, const char *name) {
    if (!name) return nullptr;
    auto it = s->vars.find(name);
    return it == s->vars.end() ? nullptr : &it->second;
}

// What the entries do first: clear the error, reset the outputs, resolve the store and the variable, and check
// the variable's itemsize when the entry takes one (ddstore.hpp:189-190, 202-203; NULL: none, or checked per conversion).
// `host_refused` (non-null): the entry does not take DDS_PLACE_HOST variables; the text of its DDS_ERR_ARG.
int entry_var(dds_store *s, const char *name, const int *itemsize, int64_t *total_bytes, int64_t *bad_index, Var **v,
              const char *host_refused = nullptr) {
    clear_error();
    if (bad_index) *bad_index = -1;
    if (total_bytes) *total_bytes = 0;
    if (!s) return fail(DDS_ERR_ARG, "null store");
    *v = find_var(s, name);
    if (!*v) return fail(DDS_ERR_UNKNOWN_VAR, name ? name : "(null)");
    if (host_refused && (*v)->host) return fail(DDS_ERR_ARG, host_refused);
    if (itemsize && (*v)->itemsize != *itemsize) return fail(DDS_ERR_DTYPE);
    return DDS_OK;
}

void release_var(Var &v, int rank) {
    for (size_t r = 0; r < v.peer_base.size(); r++) {
        if ((int)r == rank || !v.peer_base[r]) continue;
        if (v.peer_opened[r] == 1) cudaIpcCloseMemHandle(v.peer_base[r]);
        if (v.peer_opened[r] == 2) dds_vmm::release(&v.peer_block[r]);
    }
    v.peer_base.clear();
    v.peer_opened.clear();
    v.peer_block.clear();
}

void free_shard(Var &v) {
    if (v.d_tab) cudaFree(v.d_tab);
    v.d_tab = nullptr;
    if (v.d_norm) cudaFree(v.d_norm);
    v.d_norm = nullptr;
    v.norm_nchan = 0;
    if (v.vmm || v.host)
        dds_vmm::release(&v.block);
    else if (v.base)
        cudaFree(v.base);
    v.base = nullptr;
}

// add() and init() share everything but the fill (ddstore.hpp:39-108 vs :110-179).
// COLLECTIVE: every rank always runs the all-gather, the descriptor exchange (when any is due) and the barrier, in the
// same order, whatever failed locally -- a local failure (bad argument, out of memory, a failed copy) travels in the
// all-gathered record (PeerRec.ok) and makes EVERY rank fail consistently afterwards, instead of leaving the peers
// stuck in a collective the failing rank never entered.
int register_var(dds_store *s, const char *name, const void *buffer, int64_t nrows, int disp, int itemsize,
                 int buffer_on_device, bool zero_fill, int placement) {
    if (!s || !name) return fail(DDS_ERR_ARG, "null store or name");
    int local_rc = DDS_OK;
    std::string local_err;
    auto note = [&](int rc) {
        if (rc && !local_rc) {
            local_rc = rc;
            local_err = dds_last_error();
        }
    };
    auto note_cuda = [&](cudaError_t e, const char *what) {
        if (e != cudaSuccess) note(cuda_fail(e, what));
    };
    if (nrows < 0 || disp < 0 || itemsize <= 0) note(fail(DDS_ERR_ARG, "negative nrows/disp or itemsize <= 0"));
    if (s->size > DDSK_MAX_RANKS) note(fail(DDS_ERR_ARG, "communicator larger than DDSK_MAX_RANKS"));
    if (!zero_fill && !buffer && nrows * (int64_t)disp > 0) note(fail(DDS_ERR_ARG, "null buffer"));
    if (placement != DDS_PLACE_HBM && placement != DDS_PLACE_HOST) note(fail(DDS_ERR_ARG, "unknown placement"));
    note_cuda(cudaSetDevice(s->device), "cudaSetDevice");
    const bool exists = s->vars.count(name) != 0;
    const unsigned long long seq = s->reg_seq++;

    // shard: payload + 16 bytes of slack so the kernel's 16-byte-aligned superset loads never leave it
    const size_t payload = local_rc ? 0 : (size_t)nrows * (size_t)disp * (size_t)itemsize;
    size_t alloc = ((payload + 16 + 255) / 256) * 256;
    Var v;
    v.host = placement == DDS_PLACE_HOST;
    v.vmm = !v.host && dds_vmm::available(s->device);
    void *base = nullptr;
    if (!local_rc) {
        if (v.host) { // (a fresh memfd reads as zeros: no fill for zero_fill or the slack)
            note(dds_vmm::host_alloc(alloc, &v.block));
            if (!local_rc) {
                base = v.block.ptr;
                alloc = v.block.size;
            }
        } else if (v.vmm) {
            note(dds_vmm::alloc(s->device, alloc, &v.block));
            if (!local_rc) {
                base = v.block.ptr;
                alloc = v.block.size;
            }
        } else {
            note_cuda(cudaMalloc(&base, alloc), "cudaMalloc (shard)");
            if (local_rc) base = nullptr;
        }
    }
    v.base = base;
    v.bytes = alloc;
    if (base && v.host) {
        if (!zero_fill && payload > 0)
            note_cuda(cudaMemcpyAsync(v.block.host, buffer, payload, cudaMemcpyDefault, s->stream), "cudaMemcpyAsync (shard fill)");
        note_cuda(cudaStreamSynchronize(s->stream), "cudaStreamSynchronize (shard fill)");
    } else if (base) {
        if (zero_fill || payload == 0) {
            note_cuda(cudaMemsetAsync(base, 0, alloc, s->stream), "cudaMemsetAsync (shard)");
        } else {
            note_cuda(cudaMemsetAsync((char *)base + payload, 0, alloc - payload, s->stream), "cudaMemsetAsync (slack)");
            note_cuda(cudaMemcpyAsync(base, buffer, payload,
                                      buffer_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s->stream),
                      "cudaMemcpyAsync (shard fill)");
        }
        note_cuda(cudaStreamSynchronize(s->stream), "cudaStreamSynchronize (shard fill)");
    }

    PeerRec mine;
    memset(&mine, 0, sizeof(mine));
    mine.nrows = local_rc ? 0 : nrows;
    mine.disp = disp;
    mine.itemsize = itemsize;
    mine.pid = (int32_t)getpid();
    mine.device = s->device;
    mine.raw_ptr = (uint64_t)base;
    mine.host_tag = host_tag();
    mine.alloc_bytes = alloc;
    mine.vmm = v.vmm ? 1 : 0;
    mine.placement = placement;
    if (s->size > 1 && !v.vmm && !v.host && base) note_cuda(cudaIpcGetMemHandle(&mine.handle, base), "cudaIpcGetMemHandle");
    mine.ok = local_rc ? 0 : 1;
    std::vector<PeerRec> all((size_t)s->size);
    if (int rc = dds_comm_allgather(s->comm, &mine, all.data(), sizeof(PeerRec))) {
        free_shard(v); // the communicator itself is broken: nothing collective can follow
        return rc;
    }

    // ddstore.hpp:78-82: every rank must pass the same disp; the ranks that differ from the max throw
    int max_disp = 0;
    bool bad_item = false, mixed = false, other_host = false, other_proc = false, peer_failed = false, bad_place = false;
    for (auto &p : all) {
        max_disp = std::max(max_disp, (int)p.disp);
        bad_place |= p.placement != placement;
        bad_item |= p.itemsize != itemsize;
        mixed |= p.vmm != mine.vmm;
        other_host |= p.host_tag != mine.host_tag;
        other_proc |= p.pid != mine.pid;
        peer_failed |= !p.ok;
    }
    const bool bad_disp = max_disp != disp;
    int map_rc = DDS_OK;
    if (peer_failed) {
        if (local_rc) {
            g_err = local_err;
            map_rc = local_rc;
        } else {
            map_rc = fail(DDS_ERR_COMM, "a peer rank failed to allocate or fill its shard");
        }
    }
    if (!map_rc && bad_place) map_rc = fail(DDS_ERR_ARG, "ranks disagree on the placement of a variable");
    if (!map_rc && mixed)
        map_rc = fail(DDS_ERR_CUDA, "ranks disagree on the shard allocation mode (set DDS_SHARD_ALLOC on all ranks)");
    if (!map_rc && other_host)
        map_rc = fail(DDS_ERR_COMM, "ranks on different hosts: the store spans one NVSwitch box (use one store per box)");

    // ---- build the "window": every rank's shard mapped here. Done on ALL ranks whatever their own verdict on
    // disp / itemsize, so the collective steps stay in lock-step (a rank that will fail below still serves its shard to
    // the others, like the reference's ranks that pass the disp check keep a window containing every rank's buffer).
    // Whether the descriptor exchange runs depends only on all-gathered facts, so every rank decides the same.
    v.name = name;
    v.itemsize = itemsize;
    v.disp = disp;
    v.nrows = nrows;
    v.lenlist.resize((size_t)s->size);
    int64_t sum = 0; // ddstore.hpp:84-89 inclusive running sum
    for (int r = 0; r < s->size; r++) {
        sum += all[(size_t)r].nrows;
        v.lenlist[(size_t)r] = sum;
    }
    v.peer_base.assign((size_t)s->size, nullptr);
    v.peer_opened.assign((size_t)s->size, 0);
    v.peer_block.resize((size_t)s->size);
    std::vector<int> fds;
    if (!map_rc && (v.vmm || v.host) && other_proc) {
        std::vector<char> want((size_t)s->size, 0);
        std::vector<int> pids((size_t)s->size, 0);
        for (int r = 0; r < s->size; r++) {
            want[(size_t)r] = all[(size_t)r].pid != mine.pid;
            pids[(size_t)r] = all[(size_t)r].pid;
        }
        map_rc = dds_vmm::export_fd(&v.block);
        char tag[96];
        snprintf(tag, sizeof(tag), "dds-b200-%016llx-%llu", s->token, seq);
        // collective even if the export failed: the message then says "no descriptor"
        int xrc = dds_vmm::exchange_fds(s->comm, tag, v.block.fd, want, pids, &fds);
        if (!map_rc) map_rc = xrc;
        if (v.block.fd >= 0) { // every peer holds its own duplicate now; one descriptor per variable would add up
            close(v.block.fd);
            v.block.fd = -1;
        }
    }
    for (int r = 0; r < s->size && !map_rc; r++) {
        const PeerRec &p = all[(size_t)r];
        if (r == s->rank) {
            v.peer_base[(size_t)r] = base;
        } else if (p.pid == mine.pid) {
            // thread-ranks of one process: the raw pointer is already valid here
            v.unprotected_peers = true;
            if (p.device != s->device && !v.vmm && !v.host) { // (a host block is portable: valid on every device)
                int can = 0;
                cudaError_t e = cudaDeviceCanAccessPeer(&can, s->device, p.device);
                if (e != cudaSuccess) {
                    map_rc = cuda_fail(e, "cudaDeviceCanAccessPeer");
                    break;
                }
                if (!can) {
                    map_rc = fail(DDS_ERR_CUDA, "peer GPUs of one process cannot access each other");
                    break;
                }
                e = cudaDeviceEnablePeerAccess(p.device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                    map_rc = cuda_fail(e, "cudaDeviceEnablePeerAccess");
                    break;
                }
                (void)cudaGetLastError();
            }
            v.peer_base[(size_t)r] = (void *)p.raw_ptr;
        } else if (v.vmm || v.host) {
            int fd = fds.size() > (size_t)r ? fds[(size_t)r] : -1;
            if (fd < 0) {
                map_rc = fail(DDS_ERR_COMM, "no descriptor received from a peer rank");
                break;
            }
            map_rc = v.host ? dds_vmm::host_import(fd, (size_t)p.alloc_bytes, &v.peer_block[(size_t)r])
                            : dds_vmm::import_fd(s->device, fd, (size_t)p.alloc_bytes, &v.peer_block[(size_t)r]);
            close(fd);
            fds[(size_t)r] = -1;
            if (map_rc) break;
            v.peer_base[(size_t)r] = v.peer_block[(size_t)r].ptr;
            v.peer_opened[(size_t)r] = 2;
        } else {
            v.unprotected_peers = true;
            void *mapped = nullptr;
            cudaError_t e = cudaIpcOpenMemHandle(&mapped, p.handle, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                map_rc = cuda_fail(e, "cudaIpcOpenMemHandle");
                break;
            }
            v.peer_base[(size_t)r] = mapped;
            v.peer_opened[(size_t)r] = 1;
        }
    }
    for (int fd : fds)
        if (fd >= 0) close(fd);
    // VMM blocks are not covered by cudaDeviceEnablePeerAccess: grant the other devices of THIS process access
    if (!map_rc && v.vmm) {
        for (int r = 0; r < s->size && !map_rc; r++) {
            const PeerRec &p = all[(size_t)r];
            if (r != s->rank && p.pid == mine.pid && p.device != s->device) map_rc = dds_vmm::grant(&v.block, p.device);
        }
    }
    const std::string keep_err = dds_last_error(); // (the text of whatever set map_rc)
    int brc = dds_comm_barrier(s->comm); // every shard is filled, mapped and granted before anyone may read it

    if (map_rc || bad_disp || bad_item || exists) {
        release_var(v, s->rank);
        if (base) {
            if (v.vmm || v.host)
                s->zombie_blocks.push_back(v.block); // peers may have mapped it; released in dds_free
            else
                s->zombies.push_back(base);
        }
        if (local_rc) {
            g_err = local_err;
            return local_rc;
        }
        if (map_rc) {
            g_err = keep_err;
            return map_rc;
        }
        if (bad_disp) return fail(DDS_ERR_DISP);
        if (bad_item) return fail(DDS_ERR_DTYPE);
        return fail(DDS_ERR_EXISTS, name);
    }
    memset(&v.kv, 0, sizeof(v.kv));
    for (int r = 0; r < s->size; r++) {
        v.kv.bases[r] = v.peer_base[(size_t)r];
        v.kv.lenlist[r] = v.lenlist[(size_t)r];
    }
    v.kv.row_bytes = (int64_t)disp * (int64_t)itemsize;
    v.kv.nranks = s->size;
    v.kv.host = v.host ? 1 : 0;
    if (s->db_enabled && s->d_vars && s->next_var_id < dds_store::kMaxDbVars) { // window into the doorbell kernel's table
        if (cudaMemcpy(&s->d_vars[s->next_var_id], &v.kv, sizeof(ddsk_var_t), cudaMemcpyHostToDevice) == cudaSuccess)
            v.id = s->next_var_id++;
        (void)cudaGetLastError();
    }
    s->vars.emplace(v.name, std::move(v));
    return brc;
}

// nonnegative a * b and a + b, INT64_MAX when the exact result does not fit
int64_t sat_mul(int64_t a, int64_t b) {
    int64_t r;
    return __builtin_mul_overflow(a, b, &r) ? INT64_MAX : r;
}
int64_t sat_add(int64_t a, int64_t b) {
    int64_t r;
    return __builtin_add_overflow(a, b, &r) ? INT64_MAX : r;
}

// ---- converting batches: source itemsize / output itemsize of a DDSK_CVT_* code, as log2
int cvt_in_log2(int code) { return DDSK_CVT_IN_LOG2(code); }
int cvt_out_log2(int code) { return DDSK_CVT_OUT_LOG2(code); }
// source bytes (whole elements) -> output bytes; saturates
int64_t cvt_to_out(int64_t p, int code) {
    if (p == INT64_MAX) return p;
    return sat_mul(p >> cvt_in_log2(code), (int64_t)1 << cvt_out_log2(code));
}
// output capacity -> the source bytes it holds: whole output elements, scaled (exact, since every packed total is a whole
// number of elements); saturates
int64_t cvt_cap_to_src(int64_t cap, int code) { return sat_mul(cap >> cvt_out_log2(code), (int64_t)1 << cvt_in_log2(code)); }

// The device status word is sticky (kernels only atomicMin into it): re-arm it after an error was read.
void rearm_status(dds_store *s, cudaStream_t stream) {
    if (s->push.ready) // the owners report errors of a pushed batch into this rank's window
        cudaMemsetAsync(s->push.table.win[s->push.table.me] + 24, 0xFF, 8, stream);
    cudaMemsetAsync(s->scr.status, 0xFF, 8, stream);
    cudaStreamSynchronize(stream);
}

int decode_status_word(unsigned long long st, int64_t *bad_index) {
    if (st == DDSK_STATUS_OK) {
        if (bad_index) *bad_index = -1;
        return DDS_OK;
    }
    int code = (int)(st & 0xFFull);
    if (bad_index) *bad_index = (int64_t)((st >> 8) & DDSK_STATUS_REQ_MASK);
    switch (code) {
    case DDSK_CODE_START: return fail(DDS_ERR_START);
    case DDSK_CODE_COUNT: return fail(DDS_ERR_COUNT);
    case DDSK_CODE_CAPACITY:
        if (bad_index) *bad_index = -1;
        return fail(DDS_ERR_CAPACITY);
    case DDSK_CODE_SAMPLE: return fail(DDS_ERR_ARG, "sample id outside the variable's sample index");
    case DDSK_CODE_BAG: return fail(DDS_ERR_ARG, "malformed bag offsets");
    default: return fail(DDS_ERR_WATCHDOG);
    }
}

int decode_status(dds_store *s, cudaStream_t stream, unsigned long long st, int64_t *bad_index) {
    if (st != DDSK_STATUS_OK) rearm_status(s, stream);
    return decode_status_word(st, bad_index);
}

// ---- the queue of DDS_NO_SYNC batches: every batched call goes begin_call -> launch_flags -> launch -> end_launch
// Async batches may queue up behind each other on ONE stream (the status word is then sticky, and every launch tags its
// reports with its position in the queue: dds_batch_wait reports the first failing batch of the queue, with that
// batch's first invalid request). Anything else drains the queue first.

// Complete the pending queue without reporting its outcome: dds_batch_wait alone reports it, once. The queue's first
// failure is kept unless an earlier one already is (that one is earlier in queue order), and so is the total of its
// last batch. Every call that must complete a queue before its own work comes through here, and then reports only its
// own outcome. `puts_only`: only a queue that holds a put. Returns nothing but a CUDA error of the drain itself.
int drain_pending(dds_store *s, bool puts_only = false) {
    dds_store::Queue &q = s->q;
    if (!q.pending || (puts_only && !q.pending_put)) return DDS_OK;
    q.pending = false;
    q.pending_put = false;
    break_run(s);
    cudaStream_t st = q.pending_stream;
    // queued launches skip the host mirror (it costs time at the end of every kernel): read the words back here
    CU(cudaMemcpyAsync(&s->h_status[0], s->scr.status, 8, cudaMemcpyDeviceToHost, st));
    if (q.pending_fixed_total < 0 && q.pending_total_ptr)
        CU(cudaMemcpyAsync(&s->h_status[1], q.pending_total_ptr, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    q.kept_total = q.pending_fixed_total >= 0 ? q.pending_fixed_total : cvt_to_out((int64_t)s->h_status[1], q.pending_cvt);
    const unsigned long long stw = s->h_status[0];
    if (stw != DDSK_STATUS_OK) {
        if (q.kept_status == DDSK_STATUS_OK) q.kept_status = stw;
        rearm_status(s, st);
    }
    return DDS_OK;
}

// A batched call's stream, and whether it goes behind batches still pending on that stream (`chain`)
struct Call {
    cudaStream_t st;
    bool no_sync, chain;
};

// Begin a batched call on the caller's stream (NULL: the store's). A DDS_NO_SYNC call chains onto a queue pending on
// the same stream; anything else drains the queue first. (The push fetch passes no_sync: it is always queued.)
int begin_call(dds_store *s, void *cuda_stream, bool no_sync, Call *c) {
    CU(cudaSetDevice(s->device));
    c->st = cuda_stream ? (cudaStream_t)cuda_stream : s->stream;
    c->no_sync = no_sync;
    c->chain = s->q.pending && no_sync && c->st == s->q.pending_stream;
    if (s->q.pending && !c->chain) return drain_pending(s);
    return DDS_OK;
}

// An empty DDS_NO_SYNC batch launches nothing, yet it is the last batch queued: the next dds_batch_wait reports its
// total, 0. Chained onto a pending queue, that queue's drain keeps the 0; otherwise nothing is pending any more.
void note_empty_async(dds_store *s, const Call &c) {
    if (!c.no_sync) return;
    if (s->q.pending) {
        s->q.pending_fixed_total = 0;
        s->q.pending_cvt = DDSK_CVT_NONE;
    } else {
        s->q.kept_total = 0;
    }
}

// The kernel flags of a launch and the scratch it works in (scratch_view; `plan_slot`: the plan kernels plan it).
// The kernels tag every status report with the launch's position in its queue (0 for a synchronous call or the first
// of a queue), so the sticky word ends up holding the first failing batch in queue order. The tag has 16 bits: a launch
// that would be the kQueueMax-th of its queue first drains the queue and starts a new one (one stream synchronise per
// kQueueMax launches), so no two launches of a queue share a tag.
// A synchronous launch mirrors status + total into pinned host words (DDSK_F_MIRROR). An overlap launch (`ovl`:
// DDS_OVERLAP, declared independent of the batch queued right before it) joins the run of overlap launches chained
// right before it or starts one; any other launch -- a put and a push included -- ends the run.
constexpr unsigned int kQueueMax = 0xFFFF;
int launch_flags(dds_store *s, const Call &c, bool ovl, bool plan_slot, int *kflags, ddsk_scratch_t *scr) {
    dds_store::Queue &q = s->q;
    bool chain = c.chain;
    if (chain && q.queue_len >= kQueueMax) {
        if (int rc = drain_pending(s)) return rc;
        chain = false;
    }
    const unsigned int ord = chain ? q.queue_len : 0u;
    q.queue_len = ord + 1u;
    s->scr.status_tag = (unsigned long long)ord << DDSK_STATUS_ORD_SHIFT;
    int f = c.no_sync ? 0 : DDSK_F_MIRROR;
    if (!ovl || !chain) break_run(s);
    if (ovl) {
        f |= DDSK_F_OVERLAP;
        if (q.run_len >= 1) f |= DDSK_F_SKIP_WAIT | DDSK_F_PREV1;
        if (q.run_len >= 2) f |= DDSK_F_PREV2;
        if (q.run_len >= 4) f |= DDSK_F_PREV4;
        s->scr.ovl_seq = q.ovl_seq++;
        q.run_len++;
    }
    *kflags = f;
    *scr = scratch_view(s, ovl, plan_slot && ovl);
    return DDS_OK;
}

// The outcome of a launch (its total: `fixed_total` when the host knows it, else the device word `total_ptr` in source
// bytes of conversion `cvt`). Queued: it is the pending queue's last batch now (`put`: a batched put). Synchronous:
// wait for it -- status and total arrive in the pinned mirror words with the end of the kernel -- and report both.
int end_launch(dds_store *s, const Call &c, int64_t fixed_total, const int64_t *total_ptr, int cvt, bool put,
               int64_t *total_bytes, int64_t *bad_index) {
    if (c.no_sync) { // nothing but the kernel(s) goes on the stream; the status word is read back by drain_pending
        dds_store::Queue &q = s->q;
        q.pending = true;
        q.pending_put |= put;
        q.pending_stream = c.st;
        q.pending_fixed_total = fixed_total;
        q.pending_total_ptr = total_ptr;
        q.pending_cvt = cvt;
        return DDS_OK;
    }
    CU(cudaStreamSynchronize(c.st));
    if (total_bytes) *total_bytes = fixed_total >= 0 ? fixed_total : cvt_to_out((int64_t)s->h_status[1], cvt);
    return decode_status(s, c.st, s->h_status[0], bad_index);
}

} // namespace

extern "C" {

const char *dds_last_error(void) { return g_err.c_str(); }
const char *dds_strerror(int code) { return code_text(code); }

// ---------------------------------------------------------------- host-side index math
int dds_sortedsearch(const int64_t *lenlist, int nranks, int64_t num) {
    // src/ddstore.cxx:5-17
    int rtn = 0;
    for (int i = 1; i < nranks; i++)
        if (lenlist[i - 1] <= num && num < lenlist[i]) {
            rtn = i;
            break;
        }
    return rtn;
}

int dds_locate(const int64_t *lenlist, int nranks, int64_t start, int64_t count, int *owner, int64_t *offset) {
    // include/ddstore.hpp:205-214
    int t = dds_sortedsearch(lenlist, nranks, start);
    int64_t off = t > 0 ? lenlist[t - 1] : 0;
    if (owner) *owner = t;
    if (offset) *offset = off;
    if (start < off) return fail(DDS_ERR_START);
    // (start >= off >= 0 here: lenlist[t] - start cannot wrap, where start + count could)
    if (count < 0 || count > lenlist[t] - start) return fail(DDS_ERR_COUNT);
    return DDS_OK;
}

int dds_exchange_lenlist(dds_comm_t *c, int64_t nrows, int disp, int64_t *lenlist) {
    // include/ddstore.hpp:75-89
    if (!c || !lenlist) return fail(DDS_ERR_ARG, "null communicator or lenlist");
    const int n = dds_comm_size(c);
    int64_t mine[2] = {nrows, (int64_t)disp};
    std::vector<int64_t> all((size_t)n * 2);
    if (int rc = dds_comm_allgather(c, mine, all.data(), sizeof(mine))) return rc;
    int64_t max_disp = 0, sum = 0;
    for (int r = 0; r < n; r++) max_disp = std::max(max_disp, all[(size_t)r * 2 + 1]);
    for (int r = 0; r < n; r++) {
        sum += all[(size_t)r * 2];
        lenlist[r] = sum;
    }
    if (max_disp != disp) return fail(DDS_ERR_DISP);
    return DDS_OK;
}

// ---------------------------------------------------------------- lifecycle
dds_store_t *dds_create(dds_comm_t *comm, int device, int method) {
    clear_error();
    if (!comm) {
        fail(DDS_ERR_ARG, "null communicator");
        return nullptr;
    }
    if (method != 0 && method != 1) {
        fail(DDS_ERR_ARG, "method must be 0 or 1 (both select the NVLink transport)");
        return nullptr;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        (void)cudaGetLastError();
        fail(DDS_ERR_NO_DEVICE, e != cudaSuccess ? cudaGetErrorString(e) : "cudaGetDeviceCount returned 0");
        return nullptr;
    }
    if (device < 0) {
        if (cudaGetDevice(&device) != cudaSuccess) device = 0;
    }
    if (device >= ndev) {
        fail(DDS_ERR_ARG, "device ordinal out of range");
        return nullptr;
    }
    dds_store *s = new dds_store;
    memset(&s->scr, 0, sizeof(s->scr));
    s->comm = comm;
    s->rank = dds_comm_rank(comm);
    s->size = dds_comm_size(comm);
    s->device = device;
    s->method = method;
    bool ok = cudaSetDevice(device) == cudaSuccess &&
              cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc((void **)&s->scr.status, 16) == cudaSuccess && // [0] sticky status, [1] packed total
              cudaMalloc((void **)&s->scr.counters, 256) == cudaSuccess && // 2 ticket words (+pad), 24 protocol words, 8 plan
                                                                           // words, 4 total words (scratch_view)
              cudaMemset(s->scr.counters, 0, 256) == cudaSuccess &&
              cudaMemset(s->scr.status, 0xFF, 8) == cudaSuccess &&
              cudaHostAlloc((void **)&s->h_status, 32, cudaHostAllocMapped) == cudaSuccess &&
              cudaHostGetDevicePointer((void **)&s->scr.host_mirror, s->h_status, 0) == cudaSuccess &&
              cudaHostAlloc((void **)&s->h_small, (size_t)(kSmallIdx * 16 + kSmallOut), cudaHostAllocMapped) == cudaSuccess &&
              cudaHostGetDevicePointer((void **)&s->d_small, s->h_small, 0) == cudaSuccess;
    if (const char *e = getenv("DDS_DOORBELL")) s->db_enabled = atoi(e) != 0;
    if (const char *e = getenv("DDS_DOORBELL_IDLE_US")) s->db_idle_ns = (unsigned long long)std::max(1, atoi(e)) * 1000ull;
    // test hook: where the 22-bit plan-tag counter starts, so a test can reach its wrap (renew_plan_tags) in a few launches
    if (const char *e = getenv("DDS_PLAN_TAG_START")) s->scr.plan_tag = (unsigned int)strtoul(e, nullptr, 0) & 0x3FFFFFu;
    if (ok && s->db_enabled) {
        ok = cudaHostAlloc((void **)&s->h_mb, sizeof(ddsk_mailbox_t), cudaHostAllocMapped) == cudaSuccess &&
             cudaHostGetDevicePointer((void **)&s->d_mb, s->h_mb, 0) == cudaSuccess &&
             cudaStreamCreateWithFlags(&s->db_stream, cudaStreamNonBlocking) == cudaSuccess &&
             cudaMalloc((void **)&s->d_vars, sizeof(ddsk_var_t) * dds_store::kMaxDbVars) == cudaSuccess;
        if (ok) memset(s->h_mb, 0, sizeof(ddsk_mailbox_t));
    }
    if (ok) {
        s->scr.total = (int64_t *)(s->scr.status + 1);
        s->scr.ovl = s->scr.counters + 8;
        s->scr.plan_word = (unsigned long long *)(s->scr.counters + 32);
        memset(s->h_status, 0, 32);
    }
    if (!ok) {
        cuda_fail(cudaGetLastError(), "dds_create: device setup");
        delete s;
        return nullptr;
    }
    // job-unique token (rank 0's) naming the descriptor-passing sockets of this store
    {
        unsigned long long mine = 0; // unguessable: it names the abstract sockets the shard descriptors travel over
        if (getrandom(&mine, sizeof(mine), 0) != (ssize_t)sizeof(mine))
            mine = ((unsigned long long)getpid() << 32) ^ (unsigned long long)(uintptr_t)s ^
                   (unsigned long long)time(nullptr) * 0x9E3779B97F4A7C15ull;
        std::vector<unsigned long long> all((size_t)s->size);
        if (dds_comm_allgather(comm, &mine, all.data(), sizeof(mine)) != DDS_OK) {
            dds_destroy(s);
            return nullptr;
        }
        s->token = all[0];
    }
    return s;
}

int dds_rank(const dds_store_t *s) { return s ? s->rank : -1; }
int dds_size(const dds_store_t *s) { return s ? s->size : -1; }

int dds_add(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int disp, int itemsize,
            int buffer_on_device) {
    return dds_add_placed(s, name, buffer, nrows, disp, itemsize, buffer_on_device, DDS_PLACE_HBM);
}

int dds_init(dds_store_t *s, const char *name, int64_t nrows, int disp, int itemsize) {
    return dds_init_placed(s, name, nrows, disp, itemsize, DDS_PLACE_HBM);
}

int dds_add_placed(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int disp, int itemsize,
                   int buffer_on_device, int placement) {
    clear_error();
    return register_var(s, name, buffer, nrows, disp, itemsize, buffer_on_device, false, placement);
}

int dds_init_placed(dds_store_t *s, const char *name, int64_t nrows, int disp, int itemsize, int placement) {
    clear_error();
    return register_var(s, name, nullptr, nrows, disp, itemsize, 0, true, placement);
}

int dds_query_placement(dds_store_t *s, const char *name, int *placement) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    if (!placement) return fail(DDS_ERR_ARG, "null placement");
    *placement = v->host ? DDS_PLACE_HOST : DDS_PLACE_HBM;
    return DDS_OK;
}

static int update_impl(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int64_t offset, int itemsize,
                       int buffer_on_device, cudaStream_t st, bool sync) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, nullptr, nullptr, &v)) return rc;
    if (nrows < 0 || offset < 0 || offset + nrows > v->nrows)
        return fail(DDS_ERR_ARG, "update outside the local shard (unchecked memcpy in the reference)");
    CU(cudaSetDevice(s->device));
    const size_t row = (size_t)v->disp * (size_t)v->itemsize;
    if (nrows * (int64_t)row > 0) {
        if (v->host)
            CU(cudaMemcpyAsync((char *)v->block.host + (size_t)offset * row, buffer, (size_t)nrows * row, cudaMemcpyDefault, st));
        else
            CU(cudaMemcpyAsync((char *)v->base + (size_t)offset * row, buffer, (size_t)nrows * row,
                               buffer_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        if (sync) CU(cudaStreamSynchronize(st));
        else if (st != s->stream) s->update_streams.insert(st); // the next fence / free waits for it
    }
    return DDS_OK;
}

int dds_update(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int64_t offset, int itemsize,
               int buffer_on_device) {
    return update_impl(s, name, buffer, nrows, offset, itemsize, buffer_on_device, s ? s->stream : nullptr, true);
}

int dds_update_async(dds_store_t *s, const char *name, const void *buffer, int64_t nrows, int64_t offset, int itemsize,
                     int buffer_on_device, void *cuda_stream) {
    return update_impl(s, name, buffer, nrows, offset, itemsize, buffer_on_device,
                       cuda_stream ? (cudaStream_t)cuda_stream : (s ? s->stream : nullptr), false);
}

// the staging pool shared by dds_ingest (pageable -> shard) and large pageable destinations (staging buffer -> pageable)
static int ensure_pool(dds_store_t *s) {
    if (s->ingest) return DDS_OK;
    IngestPool *p = new IngestPool;
    bool ok = cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) == cudaSuccess;
    for (int k = 0; k < 2 && ok; k++)
        ok = cudaHostAlloc((void **)&p->pin[k], IngestPool::kStage, cudaHostAllocDefault) == cudaSuccess &&
             cudaEventCreateWithFlags(&p->ev[k], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
        cudaError_t e = cudaGetLastError();
        for (int k = 0; k < 2; k++) {
            if (p->pin[k]) cudaFreeHost(p->pin[k]);
            if (p->ev[k]) cudaEventDestroy(p->ev[k]);
        }
        if (p->stream) cudaStreamDestroy(p->stream);
        delete p;
        return cuda_fail(e, "staging pool setup");
    }
    int nt = 6;
    if (const char *e = getenv("DDS_INGEST_THREADS")) nt = std::max(1, std::min(64, atoi(e)));
    cpu_set_t cs;
    if (sched_getaffinity(0, sizeof(cs), &cs) == 0) nt = std::max(1, std::min(nt, CPU_COUNT(&cs)));
    p->start(nt);
    s->ingest = p;
    return DDS_OK;
}

int dds_ingest(dds_store_t *s, const char *name, const void *host_rows, int64_t nrows, int64_t offset, int itemsize) {
    // update<T> (ddstore.hpp:181-195) for a chunk of PAGEABLE host rows, pipelined: parallel CPU copy into pinned staging
    // buffers + async H2D. Returns once the source has been consumed (the caller may reuse it); the last copies complete
    // at the next fence, dds_ingest_wait, or free.
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, nullptr, nullptr, &v)) return rc;
    if (nrows < 0 || offset < 0 || offset + nrows > v->nrows)
        return fail(DDS_ERR_ARG, "update outside the local shard (unchecked memcpy in the reference)");
    const size_t row = (size_t)v->disp * (size_t)v->itemsize;
    size_t total = (size_t)nrows * row;
    if (total == 0) return DDS_OK;
    if (!host_rows) return fail(DDS_ERR_ARG, "null buffer");
    CU(cudaSetDevice(s->device));
    if (int rc = ensure_pool(s)) return rc;
    IngestPool *p = s->ingest;
    const char *src = (const char *)host_rows;
    char *dst = (char *)(v->host ? v->block.host : v->base) + (size_t)offset * row;
    while (total) {
        const size_t n = std::min(total, IngestPool::kStage);
        const int k = p->next;
        if (p->ev_pending[k]) { // the H2D copy that last used this staging buffer
            CU(cudaEventSynchronize(p->ev[k]));
            p->ev_pending[k] = false;
        }
        p->copy(p->pin[k], src, n);
        CU(cudaMemcpyAsync(dst, p->pin[k], n, v->host ? cudaMemcpyDefault : cudaMemcpyHostToDevice, p->stream));
        CU(cudaEventRecord(p->ev[k], p->stream));
        p->ev_pending[k] = true;
        p->next ^= 1;
        src += n;
        dst += n;
        total -= n;
    }
    s->update_streams.insert(p->stream); // the next fence / free waits for the tail
    return DDS_OK;
}

// A packed batch from the store's HBM staging buffer into a PAGEABLE host destination (the reference's np.zeros
// contract, examples/vae/distdataset.py:80-85): cudaMemcpyAsync into pageable memory is staged by the driver through
// one thread; here the copy engine fills the pool's pinned buffers chunk by chunk while the
// worker threads copy the previous chunk out. `st` has the gather queued; synchronous.
static int d2h_pageable(dds_store_t *s, void *dst, const void *d_src, size_t bytes, cudaStream_t st) {
    if (int rc = ensure_pool(s)) return rc;
    IngestPool *p = s->ingest;
    for (int k = 0; k < 2; k++)
        if (p->ev_pending[k]) { // an ingest still owns the staging buffers
            CU(cudaEventSynchronize(p->ev[k]));
            p->ev_pending[k] = false;
        }
    const size_t step = IngestPool::kStage;
    const size_t nchunks = (bytes + step - 1) / step;
    auto issue = [&](size_t c) -> cudaError_t {
        const size_t off = c * step, n = std::min(step, bytes - off);
        cudaError_t e = cudaMemcpyAsync(p->pin[c & 1], (const char *)d_src + off, n, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaEventRecord(p->ev[c & 1], st);
        return e;
    };
    CU(issue(0));
    for (size_t c = 0; c < nchunks; c++) {
        if (c + 1 < nchunks) CU(issue(c + 1)); // (its buffer was emptied by the CPU copy of chunk c - 1, below)
        CU(cudaEventSynchronize(p->ev[c & 1]));
        const size_t off = c * step, n = std::min(step, bytes - off);
        p->copy((char *)dst + off, p->pin[c & 1], n);
    }
    return DDS_OK;
}

static bool is_pageable(const void *ptr) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
        (void)cudaGetLastError();
        return true;
    }
    return a.type == cudaMemoryTypeUnregistered;
}

int dds_ingest_wait(dds_store_t *s) {
    clear_error();
    if (!s) return fail(DDS_ERR_ARG, "null store");
    if (!s->ingest) return DDS_OK;
    CU(cudaSetDevice(s->device));
    CU(cudaStreamSynchronize(s->ingest->stream));
    s->ingest->ev_pending[0] = s->ingest->ev_pending[1] = false;
    return DDS_OK;
}

// every copy queued by dds_update_async on a caller's stream has landed (the fences promise the shard is complete)
static int drain_update_streams(dds_store_t *s) {
    for (cudaStream_t st : s->update_streams) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            s->update_streams.clear();
            return cuda_fail(e, "cudaStreamSynchronize (update stream)");
        }
    }
    s->update_streams.clear();
    return DDS_OK;
}

// One request through the 1-CTA kernel: the legacy one-get()-per-sample call. One launch, no stream synchronize: the
// kernel's last store is a ticket in mapped pinned memory the host spins on.
static int doorbell_launch(dds_store_t *s, unsigned long long served) {
    s->db_gen++;
    if (ddsk_doorbell_launch(s->d_vars, s->d_mb, served, s->db_gen, s->db_idle_ns, s->db_stream))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    s->db_alive = true;
    return DDS_OK;
}

// The launch-free form of small_get: post the request in the mailbox of the resident doorbell CTA (starting one if none
// is alive) and spin on its one-word answer.
static int doorbell_get(dds_store_t *s, Var *v, int64_t start, int64_t count, void *dst, int64_t cap, bool dst_dev,
                        int64_t *total_bytes, int64_t *bad_index) {
    volatile ddsk_mailbox_t *mb = s->h_mb;
    if (s->db_alive && mb->exit_gen == s->db_gen) s->db_alive = false; // it left on its own (idle)
    if (!s->db_alive) {
        if (int rc = doorbell_launch(s, s->db_seq)) return rc;
    }
    mb->start = start;
    mb->count = count;
    mb->dst = (uint64_t)(dst_dev ? dst : (void *)(s->d_small + kSmallIdx * 16));
    mb->dst_cap = cap;
    mb->var_stop = (uint64_t)(uint32_t)v->id;
    std::atomic_thread_fence(std::memory_order_release);
    const unsigned long long seq = ++s->db_seq;
    mb->seq_tail = seq;
    std::atomic_thread_fence(std::memory_order_release);
    mb->seq_head = seq;
    unsigned long long r = 0;
    for (unsigned spins = 0;; spins++) {
        r = mb->resp;
        if ((r >> 8) == seq) break;
        if (mb->exit_gen == s->db_gen) { // the kernel left; unless it answered first, a fresh one takes the request
            r = mb->resp;
            if ((r >> 8) == seq) break;
            cudaError_t e = cudaStreamSynchronize(s->db_stream);
            if (e != cudaSuccess) {
                s->db_alive = false;
                return cuda_fail(e, "doorbell kernel");
            }
            if (int rc = doorbell_launch(s, seq - 1)) return rc;
        }
        if ((spins & 0xFFFF) == 0xFFFF) {
            cudaError_t q = cudaStreamQuery(s->db_stream);
            if (q != cudaErrorNotReady && q != cudaSuccess) {
                s->db_alive = false;
                return cuda_fail(q, "doorbell kernel");
            }
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    const int code = (int)(r & 0xFFu);
    const int64_t n = code ? 0 : (count > 0 ? count * v->kv.row_bytes : 0);
    if (!dst_dev && n > 0) memcpy(dst, s->h_small + kSmallIdx * 16, (size_t)n);
    if (total_bytes) *total_bytes = n;
    if (!code) {
        if (bad_index) *bad_index = -1;
        return DDS_OK;
    }
    return decode_status_word(code == DDSK_CODE_CAPACITY ? (((unsigned long long)1 << 8) | DDSK_CODE_CAPACITY)
                                                          : (unsigned long long)code, bad_index);
}

static int small_get(dds_store_t *s, Var *v, int64_t start, int64_t count, void *dst, int64_t cap, bool dst_dev,
                     int64_t *total_bytes, int64_t *bad_index) {
    if (s->db_enabled && v->id >= 0) return doorbell_get(s, v, start, count, dst, cap, dst_dev, total_bytes, bad_index);
    cudaStream_t st = s->stream;
    volatile unsigned long long *flag = s->h_status;
    const unsigned long long ticket = ++s->small_ticket;
    void *d_dst = dst_dev ? dst : (void *)(s->d_small + kSmallIdx * 16);
    if (ddsk_small_get(&v->kv, start, count, d_dst, cap, s->scr.host_mirror, ticket, st))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    // spin on the ticket (a few microseconds); fall back to a stream synchronize if the kernel died
    for (unsigned spins = 0; flag[2] != ticket; spins++) {
        if ((spins & 0x3FFF) == 0x3FFF) {
            cudaError_t q = cudaStreamQuery(st);
            if (q != cudaErrorNotReady) {
                if (q != cudaSuccess) return cuda_fail(q, "dds_small_get_kernel");
                if (flag[2] != ticket) return fail(DDS_ERR_CUDA, "small get: the kernel finished without publishing its ticket");
            }
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    const unsigned long long stw = flag[0];
    const int64_t n = (int64_t)flag[1];
    if (!dst_dev && stw == DDSK_STATUS_OK && n > 0) memcpy(dst, s->h_small + kSmallIdx * 16, (size_t)n);
    if (total_bytes) *total_bytes = n;
    return decode_status_word(stw, bad_index);
}

// The requests of a batch as the kernels read them: explicit starts (and counts; NULL for a fixed count), or -- by_sample
// -- sample ids looked up in v's per-sample table. Host indices: few requests are read by the kernel straight from
// pinned host memory (no H2D copy to wait for), more are copied on `st` into the store's index arrays.
static int stage_indices(dds_store_t *s, Var *v, bool by_sample, const int64_t *starts, const int64_t *counts, int64_t nreq,
                         bool idx_dev, cudaStream_t st, ddsk_index_t *ix) {
    if (by_sample) counts = nullptr;
    if (!idx_dev && nreq <= kSmallIdx) {
        int64_t *hs = (int64_t *)s->h_small, *hc = hs + kSmallIdx;
        memcpy(hs, starts, (size_t)nreq * 8);
        if (counts) memcpy(hc, counts, (size_t)nreq * 8);
        starts = (const int64_t *)s->d_small;
        if (counts) counts = (const int64_t *)s->d_small + kSmallIdx;
    } else if (!idx_dev) {
        if (int rc = ensure_idx(s, nreq)) return rc;
        CU(cudaMemcpyAsync(s->d_starts, starts, (size_t)nreq * 8, cudaMemcpyHostToDevice, st));
        if (counts) CU(cudaMemcpyAsync(s->d_counts, counts, (size_t)nreq * 8, cudaMemcpyHostToDevice, st));
        starts = s->d_starts;
        if (counts) counts = s->d_counts;
    }
    memset(ix, 0, sizeof(*ix));
    if (by_sample) {
        ix->sample_ids = starts;
        ix->table = v->d_tab;
        ix->nsamples = v->nsamples;
    } else {
        ix->starts = starts;
        ix->counts = counts;
    }
    return DDS_OK;
}

// The bytes a request of c rows packs. A count above the variable's row total cannot be valid for any start (and
// c * row_bytes may not fit in 64 bits): such requests pack nothing, so every product is bounded by the variable's size.
static int64_t req_bytes(const Var *v, int64_t c) {
    const int64_t rows = v->lenlist.empty() ? 0 : v->lenlist.back();
    return c > 0 && c <= rows ? c * v->kv.row_bytes : 0;
}

// The packed bytes of a batch as far as the host can know them (-1: only the kernel knows): exact for a fixed count,
// else an upper bound -- the total when every request is valid -- from host counts, or from host sample ids and the
// host copy of the variable's sample table. Sums saturate.
static int64_t host_layout(const Var *v, bool by_sample, const int64_t *starts, const int64_t *counts, int64_t fixed_count,
                           int64_t nreq, bool idx_dev) {
    if (!by_sample && !counts) return sat_mul(nreq, req_bytes(v, fixed_count));
    if (idx_dev || (by_sample && v->h_tab_count.empty())) return -1;
    int64_t n = 0;
    for (int64_t i = 0; i < nreq; i++) {
        if (!by_sample)
            n = sat_add(n, req_bytes(v, counts[i]));
        else if (starts[i] >= 0 && starts[i] < v->nsamples)
            n = sat_add(n, req_bytes(v, v->h_tab_count[(size_t)starts[i]]));
    }
    return n;
}

// The one batched path behind dds_get_batch / dds_get_samples / dds_get.
//   by_sample == false: request i = (starts[i], counts ? counts[i] : fixed_count)
//   by_sample == true : request i = the rows of sample starts[i] (= sample id) in v's per-sample index
//   cvt != NULL: a converting batch (checked by the caller: device destination); dst_capacity, dst_offsets and the
//   totals are in output bytes, the kernels get the capacity in source bytes
static int batch_impl(dds_store_t *s, Var *v, bool by_sample, const int64_t *starts, const int64_t *counts,
                      int64_t fixed_count, int64_t nreq, void *dst, int64_t dst_capacity, int64_t *dst_offsets,
                      unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index,
                      const ddsk_cvt_t *cvt = nullptr) {
    if (nreq < 0 || dst_capacity < 0) return fail(DDS_ERR_ARG, "negative nreq or capacity");
    if (nreq > 0 && !starts) return fail(DDS_ERR_ARG, "null starts / sample ids");
    const bool idx_dev = flags & DDS_IDX_ON_DEVICE, dst_dev = flags & DDS_DST_ON_DEVICE;
    const bool no_sync = flags & DDS_NO_SYNC;
    if (no_sync && !(idx_dev && dst_dev)) return fail(DDS_ERR_ARG, "async batches need device indices and a device destination");
    Call c;
    if (int rc = begin_call(s, cuda_stream, no_sync, &c)) return rc;
    const bool fixed = !by_sample && counts == nullptr;
    const int64_t nb_fixed = fixed ? req_bytes(v, fixed_count) : 0;

    if (nreq == 0) {
        if (dst_offsets) {
            int64_t z = 0;
            if (dst_dev) CU(cudaMemcpyAsync(dst_offsets, &z, 8, cudaMemcpyHostToDevice, c.st));
            else dst_offsets[0] = 0;
            if (dst_dev) CU(cudaStreamSynchronize(c.st));
        }
        note_empty_async(s, c);
        return DDS_OK;
    }

    // ---- the legacy per-sample call: one request, host indices, synchronous, small result -> 1-CTA kernel
    if (fixed && nreq == 1 && !idx_dev && !no_sync && !cuda_stream && !dst_offsets && !cvt) {
        const int64_t need = nb_fixed;
        if (need <= (dst_dev ? (int64_t)(1 << 20) : kSmallOut) && (dst || need == 0))
            return small_get(s, v, starts[0], fixed_count, dst, dst_dev ? dst_capacity : std::min(dst_capacity, kSmallOut), dst_dev,
                             total_bytes, bad_index);
    }

    // ---- indices to the device (8-16 B per request)
    ddsk_index_t ix;
    if (int rc = stage_indices(s, v, by_sample, starts, counts, nreq, idx_dev, c.st, &ix)) return rc;
    const int64_t upper = host_layout(v, by_sample, starts, counts, fixed_count, nreq, idx_dev);

    // ---- destination: the caller's device buffer, or the store's staging buffer for a host destination
    void *d_dst = dst;
    int64_t cap = dst_capacity;
    // (Large pinned destinations still go through an HBM staging buffer + one D2H copy: letting the kernel's bulk
    // stores write over PCIe directly was slower.)
    bool small_out = false;
    if (!dst_dev) {
        int64_t need = upper >= 0 ? std::min(upper, dst_capacity) : dst_capacity;
        if (need <= kSmallOut) { // small result: the kernel writes it straight into pinned host memory
            small_out = true;
            d_dst = s->d_small + kSmallIdx * 16;
        } else {
            if (int rc = ensure_out(s, std::max<int64_t>(need, 16))) return rc;
            d_dst = s->d_out;
        }
        cap = need;
    }
    const int code = cvt ? cvt->code[0] : DDSK_CVT_NONE;
    if (cvt) cap = cvt_cap_to_src(dst_capacity, code);
    if (!d_dst && cap > 0) return fail(DDS_ERR_ARG, "null destination");
    const bool ovl = no_sync && (flags & DDS_OVERLAP) && !v->host; // (a HOST launch ends an overlap run)
    bool uses_scratch = false;
    if (!fixed)
        if (int rc = plan_scratch(s, nreq, cap, cvt, ovl, v->host, &uses_scratch)) return rc;

    // ---- launch
    int64_t *d_offsets = dst_dev ? dst_offsets : nullptr;
    if (!dst_dev && !fixed) { // byte offsets for a host destination: staged on the device (the caller's, and the length of
                              // the prefix to copy back on an error), copied back below
        if (int rc = ensure_offs(s, nreq + 1)) return rc;
        d_offsets = s->d_offs;
    }
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, ovl, uses_scratch, &kflags, &scr)) return rc;
    const int krc = fixed ? ddsk_gather_fixed(&v->kv, ix.starts, fixed_count, nreq, d_dst, cap, d_offsets, &scr, kflags, cvt,
                                              nullptr, c.st)
                          : ddsk_gather_var(&v->kv, &ix, nreq, d_dst, cap, d_offsets, &scr, kflags, cvt, nullptr, c.st);
    s->scr.plan_tag = scr.plan_tag;
    if (krc) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());

    // ---- results back to a host destination: exactly what the serial get() loop would have left there. The status
    // comes first: after an invalid request only the requests before it are copied, after a capacity error nothing --
    // the rest of the staging buffer holds whatever an earlier batch left in it.
    if (!dst_dev) {
        CU(cudaStreamSynchronize(c.st));
        const unsigned long long stw = s->h_status[0];
        const int64_t total = fixed ? upper : (int64_t)s->h_status[1];
        int64_t n = total; // bytes the caller receives
        if (stw != DDSK_STATUS_OK) {
            const int code = (int)(stw & 0xFFull);
            const int64_t bad = (int64_t)((stw >> 8) & DDSK_STATUS_REQ_MASK);
            const bool invalid = code == DDSK_CODE_START || code == DDSK_CODE_COUNT || code == DDSK_CODE_SAMPLE;
            if (total > cap || !invalid || bad >= nreq)
                n = 0; // the batch did not fit (whatever else was wrong): nothing was packed
            else if (fixed)
                n = bad * nb_fixed;
            else { // the packed offset of the first invalid request
                CU(cudaMemcpyAsync(&n, d_offsets + bad, 8, cudaMemcpyDeviceToHost, c.st));
                CU(cudaStreamSynchronize(c.st));
            }
        }
        if (n > 0) {
            if (small_out) {
                memcpy(dst, s->h_small + kSmallIdx * 16, (size_t)n); // pinned bounce -> the caller's buffer
            } else if (n >= (int64_t)(4u << 20) && is_pageable(dst)) {
                if (int rc = d2h_pageable(s, dst, d_dst, (size_t)n, c.st)) return rc;
            } else {
                CU(cudaMemcpyAsync(dst, d_dst, (size_t)n, cudaMemcpyDeviceToHost, c.st));
            }
        }
        if (dst_offsets && !fixed)
            CU(cudaMemcpyAsync(dst_offsets, d_offsets, (size_t)(nreq + 1) * 8, cudaMemcpyDeviceToHost, c.st));
        if (dst_offsets && fixed)
            for (int64_t i = 0; i <= nreq; i++) dst_offsets[i] = i * nb_fixed;
    }
    // (the device word of a variable-count total is in source bytes)
    return end_launch(s, c, fixed ? cvt_to_out(upper, code) : -1, uses_scratch ? &scr.req_dst[nreq] : scr.total, code, false,
                      total_bytes, bad_index);
}

// Validate the conversions of a converting call (one per variable) and pack them, tables included, into the launch's
// parameter. `none_ok`: DDS_CVT_NONE is allowed (a raw variable of a multi-array batch).
static int make_cvt(Var *const *vars, const dds_convert_t *cv, int nvars, bool none_ok, ddsk_cvt_t *out) {
    memset(out, 0, sizeof(*out));
    if (!cv) return fail(DDS_ERR_ARG, "null conversion");
    int off = 0;
    for (int v = 0; v < nvars; v++) {
        const int code = cv[v].code;
        if (code < (none_ok ? DDS_CVT_NONE : DDS_CVT_F32_BF16) || code > DDSK_CVT_MAX)
            return fail(DDS_ERR_ARG, "unknown conversion code " + std::to_string(code));
        // (a normalising code needs the variable's tables before anything else: without them it names no conversion)
        if (DDSK_CVT_IS_NORM(code) && vars[v]->norm_nchan <= 0) // checked at call time: they may have been removed since
            return fail(DDS_ERR_ARG, "variable has no normalization (call dds_set_normalization first)");
        if (code != DDS_CVT_NONE && vars[v]->itemsize != (1 << cvt_in_log2(code))) return fail(DDS_ERR_DTYPE);
        out->code[v] = code;
        const bool u8_norm = code == DDS_CVT_NORM_U8_F32 || code == DDS_CVT_NORM_U8_BF16 || code == DDS_CVT_NORM_U8_F16;
        if (code == DDS_CVT_U8_LUT16 || code == DDS_CVT_U8_LUT32 || u8_norm) {
            if (!cv[v].lut) return fail(DDS_ERR_ARG, "a LUT conversion needs a table");
            const int bytes = u8_norm ? 256 * 4 : 256 << cvt_out_log2(code); // (a normalising code decodes through f32)
            memcpy((char *)out->lut + off, cv[v].lut, (size_t)bytes); // copied now: the caller may free it on return
            out->lut_off[v] = off;
            off += bytes;
        }
        if (DDSK_CVT_IS_NORM(code)) {
            out->norm[v] = vars[v]->d_norm;
            out->nchan[v] = (int32_t)vars[v]->norm_nchan;
            out->inner[v] = (int32_t)vars[v]->norm_inner;
        }
    }
    out->lut_bytes = off;
    return DDS_OK;
}

int dds_set_normalization(dds_store_t *s, const char *name, const float *mean, const float *std, int64_t nchan,
                          int64_t inner, int tables_on_device) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    if (nchan < 0 || inner < 1) return fail(DDS_ERR_ARG, "bad normalization layout (nchan >= 0, inner >= 1)");
    if (nchan > 0 && (!mean || !std)) return fail(DDS_ERR_ARG, "null normalization table");
    // (both factors are bounded by disp before they are multiplied: no overflow, and the pattern stays below 2^31)
    if (nchan > 0 && (nchan > v->disp || inner > v->disp || v->disp % (nchan * inner) != 0))
        return fail(DDS_ERR_ARG, "nchan * inner must divide the row's element count (disp " + std::to_string(v->disp) + ")");
    CU(cudaSetDevice(s->device));
    if (int rc = drain_pending(s)) return rc;
    CU(device_sync(s)); // no queued launch may still be reading the old tables
    if (v->d_norm) cudaFree(v->d_norm);
    v->d_norm = nullptr;
    v->norm_nchan = 0;
    v->norm_inner = 1;
    if (nchan == 0) return DDS_OK;
    // mean and std are interleaved into {mean, std} pairs: an element's channel is ONE 8-byte load
    CU(cudaMalloc((void **)&v->d_norm, (size_t)nchan * 8));
    const cudaMemcpyKind kind = tables_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    CU(cudaMemcpy2DAsync(v->d_norm, 8, mean, 4, 4, (size_t)nchan, kind, s->stream));
    CU(cudaMemcpy2DAsync(v->d_norm + 1, 8, std, 4, 4, (size_t)nchan, kind, s->stream));
    CU(cudaStreamSynchronize(s->stream));
    v->norm_nchan = nchan;
    v->norm_inner = inner;
    return DDS_OK;
}

// the argument checks the converting single-variable entries share
static int convert_args(Var *v, const dds_convert_t *cvt, void *dst, const int64_t *dst_offsets, unsigned flags,
                        ddsk_cvt_t *kc) {
    if (int rc = make_cvt(&v, cvt, 1, false, kc)) return rc;
    if (!(flags & DDS_DST_ON_DEVICE)) return fail(DDS_ERR_ARG, "converting batches deliver into device memory");
    if ((uint64_t)dst % (uint64_t)(1 << cvt_out_log2(kc->code[0])) || (uint64_t)dst_offsets % 8u)
        return fail(DDS_ERR_ARG, "destination not aligned to the output itemsize (or offsets to 8 bytes)");
    return DDS_OK;
}

int dds_get_batch_convert(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                          int64_t fixed_count, int64_t nreq, void *dst, int64_t dst_capacity, int64_t *dst_offsets,
                          unsigned flags, void *cuda_stream, const dds_convert_t *cvt, int64_t *total_bytes,
                          int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, &v)) return rc;
    ddsk_cvt_t kc;
    if (int rc = convert_args(v, cvt, dst, dst_offsets, flags, &kc)) return rc;
    return batch_impl(s, v, false, starts, counts, fixed_count, nreq, dst, dst_capacity, dst_offsets, flags, cuda_stream,
                      total_bytes, bad_index, &kc);
}

int dds_get_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                  int64_t fixed_count, int64_t nreq, int itemsize, void *dst, int64_t dst_capacity,
                  int64_t *dst_offsets, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                  int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v)) return rc;
    return batch_impl(s, v, false, starts, counts, fixed_count, nreq, dst, dst_capacity, dst_offsets, flags, cuda_stream,
                      total_bytes, bad_index);
}

int dds_set_sample_index(dds_store_t *s, const char *name, const int64_t *row_start, const int64_t *row_count,
                         int64_t nsamples, int tables_on_device) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    if (nsamples < 0 || (nsamples > 0 && (!row_start || !row_count))) return fail(DDS_ERR_ARG, "bad sample index");
    CU(cudaSetDevice(s->device));
    if (int rc = drain_pending(s)) return rc;
    CU(device_sync(s)); // no queued launch may still be reading the old table
    if (v->d_tab) cudaFree(v->d_tab);
    v->d_tab = nullptr;
    v->h_tab_count.clear();
    v->nsamples = 0;
    if (nsamples == 0) return DDS_OK;
    // the two arrays are interleaved into {start, count} pairs: the lookup of a sample id is ONE 16-byte load
    CU(cudaMalloc((void **)&v->d_tab, (size_t)nsamples * 16));
    const cudaMemcpyKind kind = tables_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    CU(cudaMemcpy2DAsync(v->d_tab, 16, row_start, 8, 8, (size_t)nsamples, kind, s->stream));
    CU(cudaMemcpy2DAsync(v->d_tab + 1, 16, row_count, 8, 8, (size_t)nsamples, kind, s->stream));
    CU(cudaStreamSynchronize(s->stream));
    if (!tables_on_device) v->h_tab_count.assign(row_count, row_count + nsamples); // sizes a host destination needs
    v->nsamples = nsamples;
    // room in the persisting part of L2 for the tables (the plan kernel asks for it with an access-policy window): the
    // gather streams hundreds of MB per batch through L2 and would otherwise evict them between batches
    {
        size_t want = 0;
        for (auto &x : s->vars) want += (size_t)x.second.nsamples * 16;
        int maxp = 0;
        if (cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, s->device) != cudaSuccess) maxp = 0;
        // (at most 12 MiB -- a quarter of the H100's 50 MB L2 -- is set aside: the rest of the process shares this cache)
        maxp = (int)std::min<size_t>((size_t)std::max(maxp, 0), (size_t)12 << 20);
        if (maxp > 0) (void)cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, std::min(want, (size_t)maxp));
        (void)cudaGetLastError();
        if (maxp > 0 && (size_t)nsamples * 16 <= (size_t)maxp) { // warm it now: every later lookup hits L2
            (void)ddsk_l2_warm(v->d_tab, (size_t)nsamples * 16, s->stream);
            (void)cudaStreamSynchronize(s->stream);
            (void)cudaGetLastError();
        }
    }
    return DDS_OK;
}

int dds_get_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize, void *dst,
                    int64_t dst_capacity, int64_t *dst_offsets, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                    int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v)) return rc;
    if (!v->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");
    return batch_impl(s, v, true, sample_ids, nullptr, 0, nreq, dst, dst_capacity, dst_offsets, flags, cuda_stream,
                      total_bytes, bad_index);
}

int dds_get_samples_convert(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, void *dst,
                            int64_t dst_capacity, int64_t *dst_offsets, unsigned flags, void *cuda_stream,
                            const dds_convert_t *cvt, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, &v)) return rc;
    ddsk_cvt_t kc;
    if (int rc = convert_args(v, cvt, dst, dst_offsets, flags, &kc)) return rc;
    if (!v->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");
    return batch_impl(s, v, true, sample_ids, nullptr, 0, nreq, dst, dst_capacity, dst_offsets, flags, cuda_stream,
                      total_bytes, bad_index, &kc);
}

// The padded path behind dds_get_batch_padded / dds_get_samples_padded (by_sample: starts = sample ids, counts unused;
// cvt: the checked conversion, or NULL for raw bytes). Every argument is checked before anything is enqueued.
static int padded_impl(dds_store_t *s, Var *v, bool by_sample, const int64_t *starts, const int64_t *counts, int64_t nreq,
                       const ddsk_cvt_t *cvt, const dds_pad_t *pad, void *dst, int64_t dst_capacity, unsigned flags,
                       void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    if (!pad) return fail(DDS_ERR_ARG, "null padding");
    if (nreq < 0 || dst_capacity < 0) return fail(DDS_ERR_ARG, "negative nreq or capacity");
    if (nreq > 0 && !starts) return fail(DDS_ERR_ARG, "null starts / sample ids");
    if (!by_sample && nreq > 0 && !counts)
        return fail(DDS_ERR_ARG, "padded batches need counts (there is no fixed-count form)");
    if (!(flags & DDS_DST_ON_DEVICE)) return fail(DDS_ERR_ARG, "padded batches deliver into device memory");
    const bool idx_dev = flags & DDS_IDX_ON_DEVICE, no_sync = flags & DDS_NO_SYNC;
    if (no_sync && !idx_dev) return fail(DDS_ERR_ARG, "async batches need device indices and a device destination");
    int out_log2 = cvt ? cvt_out_log2(cvt->code[0]) : -1;
    if (!cvt)
        for (int l = 0; l <= 3; l++)
            if (v->itemsize == 1 << l) out_log2 = l;
    if (out_log2 < 0) return fail(DDS_ERR_ARG, "padded batches need an itemsize of 1, 2, 4 or 8");
    if ((uint64_t)dst % (uint64_t)(1 << out_log2) || (uint64_t)pad->lengths % 8u)
        return fail(DDS_ERR_ARG, "destination not aligned to the output itemsize (or lengths to 8 bytes)");
    if (pad->max_rows < 0) return fail(DDS_ERR_ARG, "max_rows < 0");
    // slot sizes in source and output bytes, and the batch in both: the walk runs over nreq * src_slot
    int64_t slot = 0, src_slot = 0, total = 0, src_total = 0;
    if (__builtin_mul_overflow(pad->max_rows, (int64_t)v->disp << out_log2, &slot) ||
        __builtin_mul_overflow(pad->max_rows, v->kv.row_bytes, &src_slot) || __builtin_mul_overflow(nreq, slot, &total) ||
        __builtin_mul_overflow(nreq, src_slot, &src_total))
        return fail(DDS_ERR_ARG, "the padded batch's size overflows");
    if (dst_capacity < total)
        return fail(DDS_ERR_ARG, "destination holds " + std::to_string(dst_capacity) + " bytes, the padded batch " +
                                     std::to_string(total));
    if (total > 0 && !dst) return fail(DDS_ERR_ARG, "null destination");
    if (by_sample && !v->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");

    Call c;
    if (int rc = begin_call(s, cuda_stream, no_sync, &c)) return rc;
    if (nreq == 0) {
        note_empty_async(s, c);
        return DDS_OK;
    }
    ddsk_index_t ix;
    if (int rc = stage_indices(s, v, by_sample, starts, counts, nreq, idx_dev, c.st, &ix)) return rc;
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, no_sync && (flags & DDS_OVERLAP) && !v->host, false, &kflags, &scr)) return rc;
    if (ddsk_gather_padded(&v->kv, &ix, nreq, pad->max_rows, pad->pad_bits, out_log2, pad->lengths, dst, &scr, kflags, cvt, c.st))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    if (total_bytes) *total_bytes = total; // (the padded size, whatever the status says)
    return end_launch(s, c, total, nullptr, DDSK_CVT_NONE, false, nullptr, bad_index);
}

int dds_get_batch_padded(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts, int64_t nreq,
                         int itemsize, const dds_convert_t *cvt, const dds_pad_t *pad, void *dst, int64_t dst_capacity,
                         unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v)) return rc;
    ddsk_cvt_t kc;
    if (cvt)
        if (int rc = make_cvt(&v, cvt, 1, false, &kc)) return rc;
    return padded_impl(s, v, false, starts, counts, nreq, cvt ? &kc : nullptr, pad, dst, dst_capacity, flags, cuda_stream,
                       total_bytes, bad_index);
}

int dds_get_samples_padded(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                           const dds_convert_t *cvt, const dds_pad_t *pad, void *dst, int64_t dst_capacity, unsigned flags,
                           void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v)) return rc;
    ddsk_cvt_t kc;
    if (cvt)
        if (int rc = make_cvt(&v, cvt, 1, false, &kc)) return rc;
    return padded_impl(s, v, true, sample_ids, nullptr, nreq, cvt ? &kc : nullptr, pad, dst, dst_capacity, flags,
                       cuda_stream, total_bytes, bad_index);
}

// The batched writes behind dds_put_*, dds_accumulate_*, dds_get_accumulate_* and dds_compare_and_swap_* (by_sample:
// starts = sample ids): the gather's launch with every copy reversed, whose drain does what the write record `w` (see
// ddsk_write_t) says. Request i's rows come from src bytes [o_i, o_i + n_i), n_i = req_bytes(count_i) even for an
// invalid request, o_i the exclusive scan. Like batch_impl, the host knows the layout of a fixed count or of host indices
// and leaves capacity and validation to the kernel. A write is never overlapped and never takes the single-request
// kernels.
// w.type is set for a sum or reduction (an accumulate or a fetch-op): src must be aligned to that element type. fetch:
// the entry returns the previous rows in w.result (a fetch-op or a compare-and-swap), which must be aligned to the
// element size too; it may be NULL only when there is nothing to write, and the launch then writes nothing either way.
// A compare-and-swap (DDSK_OP_CAS) takes src and compare aligned to the variable's itemsize.
// Device atomics on mapped host memory are not atomic across GPUs over PCIe, so HOST variables take no batched write
// at all: they are written only by their owner's update / ingest.
static const char *const kHostWrite = "batched writes do not take DDS_PLACE_HOST variables (write them with update / ingest)";
static int put_impl(dds_store_t *s, Var *v, bool by_sample, const int64_t *starts, const int64_t *counts,
                    int64_t fixed_count, int64_t nreq, const void *src, int64_t src_bytes, unsigned flags,
                    void *cuda_stream, int64_t *total_bytes, int64_t *bad_index, const ddsk_write_t &w, bool fetch = false) {
    if (!(flags & DDS_SRC_ON_DEVICE)) return fail(DDS_ERR_ARG, "puts take their rows from device memory (DDS_SRC_ON_DEVICE)");
    if (nreq < 0 || src_bytes < 0) return fail(DDS_ERR_ARG, "negative nreq or src_bytes");
    if (nreq > 0 && !starts) return fail(DDS_ERR_ARG, "null starts / sample ids");
    if (by_sample && !v->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");
    const bool idx_dev = flags & DDS_IDX_ON_DEVICE, no_sync = flags & DDS_NO_SYNC;
    if (no_sync && !idx_dev) return fail(DDS_ERR_ARG, "async puts need device indices");
    const bool fixed = !by_sample && counts == nullptr;
    const int64_t layout = host_layout(v, by_sample, starts, counts, fixed_count, nreq, idx_dev);
    if (!src && (src_bytes > 0 || layout > 0)) return fail(DDS_ERR_ARG, "null src");
    if (w.type && (uintptr_t)src % (uintptr_t)v->itemsize)
        return fail(DDS_ERR_ARG, "accumulates take src aligned to the element size");
    if (fetch && !w.result && (src_bytes > 0 || layout > 0)) return fail(DDS_ERR_ARG, "null result");
    if (fetch && (uintptr_t)w.result % (uintptr_t)v->itemsize)
        return fail(DDS_ERR_ARG, "fetch-ops take result aligned to the element size");
    if (w.op == DDSK_OP_CAS && !w.compare && (src_bytes > 0 || layout > 0)) return fail(DDS_ERR_ARG, "null compare");
    if (w.op == DDSK_OP_CAS && ((uintptr_t)src % (uintptr_t)v->itemsize || (uintptr_t)w.compare % (uintptr_t)v->itemsize))
        return fail(DDS_ERR_ARG, "compare-and-swaps take src and compare aligned to the element size");

    Call c;
    if (int rc = begin_call(s, cuda_stream, no_sync, &c)) return rc;
    if (nreq == 0) {
        note_empty_async(s, c);
        return DDS_OK;
    }
    ddsk_index_t ix;
    if (int rc = stage_indices(s, v, by_sample, starts, counts, nreq, idx_dev, c.st, &ix)) return rc;
    bool uses_scratch = false;
    if (!fixed)
        if (int rc = plan_scratch(s, nreq, src_bytes, nullptr, false, false, &uses_scratch)) return rc;
    // (never overlapped: a put ends any overlap run, and the next overlapped batch starts a new one and waits for the grid)
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, false, false, &kflags, &scr)) return rc;
    void *d_src = const_cast<void *>(src);
    const int krc = fixed ? ddsk_gather_fixed(&v->kv, ix.starts, fixed_count, nreq, d_src, src_bytes, nullptr, &scr, kflags,
                                              nullptr, &w, c.st)
                          : ddsk_gather_var(&v->kv, &ix, nreq, d_src, src_bytes, nullptr, &scr, kflags, nullptr, &w, c.st);
    s->scr.plan_tag = scr.plan_tag;
    if (krc) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    return end_launch(s, c, fixed ? layout : -1, uses_scratch ? &scr.req_dst[nreq] : scr.total, DDSK_CVT_NONE, true,
                      total_bytes, bad_index);
}

// The write record of op on variable v: type the element type of a sum or reduction (0 for a put or a compare-and-swap),
// result and compare the fetch forms' buffers. Every element is the variable's itemsize (an accumulate's type has it).
static ddsk_write_t write_rec(const Var *v, int op, int type = 0, void *result = nullptr, const void *compare = nullptr) {
    const int el = v->itemsize == 8 ? 3 : v->itemsize == 4 ? 2 : v->itemsize == 2 ? 1 : 0;
    return ddsk_write_t{op, type, el, result, compare};
}

int dds_put_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts, int64_t fixed_count,
                  int64_t nreq, int itemsize, const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream,
                  int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v, kHostWrite)) return rc;
    return put_impl(s, v, false, starts, counts, fixed_count, nreq, src, src_bytes, flags, cuda_stream, total_bytes,
                    bad_index, write_rec(v, DDSK_OP_PUT));
}

int dds_put_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                    const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                    int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, total_bytes, bad_index, &v, kHostWrite)) return rc;
    return put_impl(s, v, true, sample_ids, nullptr, 0, nreq, src, src_bytes, flags, cuda_stream, total_bytes, bad_index,
                    write_rec(v, DDSK_OP_PUT));
}

static_assert(DDS_ACC_F32 == DDSK_ACC_F32 && DDS_ACC_F64 == DDSK_ACC_F64 && DDS_ACC_I32 == DDSK_ACC_I32 &&
                  DDS_ACC_I64 == DDSK_ACC_I64 && DDS_ACC_F16 == DDSK_ACC_F16 && DDS_ACC_BF16 == DDSK_ACC_BF16,
              "the kernels' accumulate types are the public ones");

// The accumulates' prologue: entry_var with the dtype in place of the itemsize (an unknown type is an argument error, a
// size other than the variable's itemsize the reference's "Invalid data type")
static int acc_entry(dds_store_t *s, const char *name, int dtype, int64_t *total_bytes, int64_t *bad_index, Var **v) {
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, v, kHostWrite)) return rc;
    if (dtype < DDS_ACC_F32 || dtype > DDS_ACC_BF16) return fail(DDS_ERR_ARG, "unknown accumulate dtype");
    if ((*v)->itemsize != 1 << DDSK_ACC_LOG2(dtype)) return fail(DDS_ERR_DTYPE);
    return DDS_OK;
}

static_assert(DDS_OP_SUM == DDSK_OP_SUM && DDS_OP_REPLACE == DDSK_OP_REPLACE && DDS_OP_MAX == DDSK_OP_MAX &&
                  DDS_OP_MIN == DDSK_OP_MIN && DDS_OP_BAND == DDSK_OP_BAND && DDS_OP_BOR == DDSK_OP_BOR &&
                  DDS_OP_BXOR == DDSK_OP_BXOR,
              "the kernels' ops are the public ones");

// The reductions' and fetch-ops' prologue: the accumulates', then an unknown op (fetch: DDS_OP_REPLACE is an op; not
// fetch: it is not, a put writes rows), then a bitwise op on a float dtype.
static int fop_entry(dds_store_t *s, const char *name, int op, int dtype, int64_t *total_bytes, int64_t *bad_index,
                     Var **v, bool fetch = true) {
    if (int rc = acc_entry(s, name, dtype, total_bytes, bad_index, v)) return rc;
    if (!(op == DDS_OP_SUM || (fetch && op == DDS_OP_REPLACE) || (op >= DDS_OP_MAX && op <= DDS_OP_BXOR)))
        return fail(DDS_ERR_ARG, fetch ? "unknown fetch-op" : "unknown accumulate op");
    if (op >= DDS_OP_BAND && dtype != DDS_ACC_I32 && dtype != DDS_ACC_I64)
        return fail(DDS_ERR_ARG, "bitwise ops take DDS_ACC_I32 or DDS_ACC_I64");
    return DDS_OK;
}

int dds_accumulate_op_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                            int64_t fixed_count, int64_t nreq, int op, int dtype, const void *src, int64_t src_bytes,
                            unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = fop_entry(s, name, op, dtype, total_bytes, bad_index, &v, false)) return rc;
    return put_impl(s, v, false, starts, counts, fixed_count, nreq, src, src_bytes, flags, cuda_stream, total_bytes,
                    bad_index, write_rec(v, op, dtype));
}

int dds_accumulate_op_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int op,
                              int dtype, const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream,
                              int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = fop_entry(s, name, op, dtype, total_bytes, bad_index, &v, false)) return rc;
    return put_impl(s, v, true, sample_ids, nullptr, 0, nreq, src, src_bytes, flags, cuda_stream, total_bytes, bad_index,
                    write_rec(v, op, dtype));
}

int dds_accumulate_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                         int64_t fixed_count, int64_t nreq, int dtype, const void *src, int64_t src_bytes, unsigned flags,
                         void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    return dds_accumulate_op_batch(s, name, starts, counts, fixed_count, nreq, DDS_OP_SUM, dtype, src, src_bytes, flags,
                                   cuda_stream, total_bytes, bad_index);
}

int dds_accumulate_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int dtype,
                           const void *src, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                           int64_t *bad_index) {
    return dds_accumulate_op_samples(s, name, sample_ids, nreq, DDS_OP_SUM, dtype, src, src_bytes, flags, cuda_stream,
                                     total_bytes, bad_index);
}

int dds_get_accumulate_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                             int64_t fixed_count, int64_t nreq, int op, int dtype, const void *src, void *result,
                             int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                             int64_t *bad_index) {
    Var *v;
    if (int rc = fop_entry(s, name, op, dtype, total_bytes, bad_index, &v)) return rc;
    return put_impl(s, v, false, starts, counts, fixed_count, nreq, src, src_bytes, flags, cuda_stream, total_bytes,
                    bad_index, write_rec(v, op, dtype, result), true);
}

int dds_get_accumulate_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int op,
                               int dtype, const void *src, void *result, int64_t src_bytes, unsigned flags,
                               void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = fop_entry(s, name, op, dtype, total_bytes, bad_index, &v)) return rc;
    return put_impl(s, v, true, sample_ids, nullptr, 0, nreq, src, src_bytes, flags, cuda_stream, total_bytes, bad_index,
                    write_rec(v, op, dtype, result), true);
}

// The compare-and-swaps' prologue: entry_var, an itemsize outside {1, 2, 4, 8} (an argument error) and then one other
// than the variable's (the reference's "Invalid data type")
static int cas_entry(dds_store_t *s, const char *name, int itemsize, int64_t *total_bytes, int64_t *bad_index, Var **v) {
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, v, kHostWrite)) return rc;
    if (itemsize != 1 && itemsize != 2 && itemsize != 4 && itemsize != 8)
        return fail(DDS_ERR_ARG, "compare-and-swaps take elements of 1, 2, 4 or 8 bytes");
    if ((*v)->itemsize != itemsize) return fail(DDS_ERR_DTYPE);
    return DDS_OK;
}

int dds_compare_and_swap_batch(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                               int64_t fixed_count, int64_t nreq, int itemsize, const void *src, const void *compare,
                               void *result, int64_t src_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes,
                               int64_t *bad_index) {
    Var *v;
    if (int rc = cas_entry(s, name, itemsize, total_bytes, bad_index, &v)) return rc;
    return put_impl(s, v, false, starts, counts, fixed_count, nreq, src, src_bytes, flags, cuda_stream, total_bytes,
                    bad_index, write_rec(v, DDSK_OP_CAS, 0, result, compare), true);
}

int dds_compare_and_swap_samples(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq, int itemsize,
                                 const void *src, const void *compare, void *result, int64_t src_bytes, unsigned flags,
                                 void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = cas_entry(s, name, itemsize, total_bytes, bad_index, &v)) return rc;
    return put_impl(s, v, true, sample_ids, nullptr, 0, nreq, src, src_bytes, flags, cuda_stream, total_bytes, bad_index,
                    write_rec(v, DDSK_OP_CAS, 0, result, compare), true);
}

static_assert(DDS_POOL_SUM == DDSK_POOL_SUM && DDS_POOL_MEAN == DDSK_POOL_MEAN && DDS_POOL_MAX == DDSK_POOL_MAX,
              "the kernels' pooling modes are the public ones");
// The argument checks of both pooled paths, in one order. buf is the get's destination (`acc` false) or the
// accumulate's grad (`acc`: no max mode, a device source, "grad" in the texts), holding buf_bytes; it must hold
// *total = nbags * R. Host bags are checked last, before anything is enqueued.
static int pool_check(Var *v, bool by_sample, const int64_t *starts, int64_t nreq, const dds_pool_t *pool, const void *buf,
                      int64_t buf_bytes, bool acc, unsigned flags, int64_t *bad_index, int64_t *total) {
    if (!pool) return fail(DDS_ERR_ARG, "null pooling");
    if (pool->mode < DDS_POOL_SUM || pool->mode > DDS_POOL_MAX) return fail(DDS_ERR_ARG, "unknown pooling mode");
    if (acc && pool->mode == DDS_POOL_MAX)
        return fail(DDS_ERR_ARG, "pooled accumulates take DDS_POOL_SUM or DDS_POOL_MEAN (max has no adjoint without its argmax)");
    const int dt = pool->dtype;
    if (dt != DDS_ACC_F32 && dt != DDS_ACC_F64 && dt != DDS_ACC_F16 && dt != DDS_ACC_BF16)
        return fail(DDS_ERR_ARG, "pooled batches take DDS_ACC_F32, F64, F16 or BF16");
    const int64_t el = (int64_t)1 << DDSK_ACC_LOG2(dt);
    if (v->itemsize != el) return fail(DDS_ERR_DTYPE);
    if (pool->weights && pool->mode != DDS_POOL_SUM) return fail(DDS_ERR_ARG, "weights apply to DDS_POOL_SUM only");
    if (!acc && !(flags & DDS_DST_ON_DEVICE)) return fail(DDS_ERR_ARG, "pooled batches deliver into device memory");
    if (acc && !(flags & DDS_SRC_ON_DEVICE))
        return fail(DDS_ERR_ARG, "pooled accumulates take grad from device memory (DDS_SRC_ON_DEVICE)");
    if (nreq < 0 || buf_bytes < 0) return fail(DDS_ERR_ARG, acc ? "negative nreq or grad_bytes" : "negative nreq or capacity");
    if (pool->nbags < 0) return fail(DDS_ERR_ARG, "nbags < 0");
    if (!pool->bags && pool->nbags != nreq) return fail(DDS_ERR_ARG, "without bag offsets, nbags must equal nreq");
    if (__builtin_mul_overflow(pool->nbags, v->kv.row_bytes, total)) return fail(DDS_ERR_ARG, "the pooled batch's size overflows");
    const char *what = acc ? "grad" : "destination";
    if (buf_bytes < *total)
        return fail(DDS_ERR_ARG, std::string(what) + " holds " + std::to_string(buf_bytes) + " bytes, the pooled batch " +
                                     std::to_string(*total));
    if ((uint64_t)buf % (uint64_t)el || (uint64_t)pool->weights % (uint64_t)el)
        return fail(DDS_ERR_ARG, std::string(what) + " or weights not aligned to the element size");
    if (*total > 0 && !buf) return fail(DDS_ERR_ARG, std::string("null ") + what);
    if (nreq > 0 && !starts) return fail(DDS_ERR_ARG, "null starts / sample ids");
    if (by_sample && !v->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");
    const bool idx_dev = flags & DDS_IDX_ON_DEVICE;
    if ((flags & DDS_NO_SYNC) && !idx_dev)
        return fail(DDS_ERR_ARG, acc ? "async pooled accumulates need device indices, bags and weights"
                                     : "async batches need device indices and a device destination");
    if (pool->bags && !idx_dev) // host bags: checked here, before anything is enqueued
        for (int64_t k = 0; k < pool->nbags; k++)
            if (pool->bags[k] < 0 || pool->bags[k + 1] < pool->bags[k] || pool->bags[k + 1] > nreq) {
                if (bad_index) *bad_index = k;
                return fail(DDS_ERR_ARG, "malformed bag offsets");
            }
    return DDS_OK;
}

// A pooled call's requests, bags and weights on the device: host ones are staged (bags and weights in the store's
// offsets buffer, behind each other)
static int pool_stage(dds_store_t *s, Var *v, bool by_sample, const int64_t *starts, const int64_t *counts, int64_t nreq,
                      const dds_pool_t *pool, bool idx_dev, cudaStream_t st, ddsk_index_t *ix, ddsk_pool_t *kp) {
    if (int rc = stage_indices(s, v, by_sample, starts, counts, nreq, idx_dev, st, ix)) return rc;
    *kp = ddsk_pool_t{pool->mode, pool->dtype, pool->bags, pool->nbags, pool->weights};
    if (!idx_dev && (pool->bags || pool->weights)) {
        const int64_t nb = pool->bags ? pool->nbags + 1 : 0;
        if (int rc = ensure_offs(s, nb + nreq)) return rc;
        if (pool->bags) CU(cudaMemcpyAsync(s->d_offs, pool->bags, (size_t)nb * 8, cudaMemcpyHostToDevice, st));
        if (pool->weights && nreq > 0)
            CU(cudaMemcpyAsync(s->d_offs + nb, pool->weights, (size_t)(nreq * v->itemsize), cudaMemcpyHostToDevice, st));
        kp->bags = pool->bags ? s->d_offs : nullptr;
        kp->weights = pool->weights ? (const void *)(s->d_offs + nb) : nullptr;
    }
    return DDS_OK;
}

// The pooled path behind dds_get_batch_pooled / dds_get_samples_pooled (by_sample: starts = sample ids, counts unused).
// Every argument, and host bags, are checked before anything is enqueued; device bags are checked by the kernel. A pooled
// launch is never overlapped.
static int pool_impl(dds_store_t *s, const char *name, bool by_sample, const int64_t *starts, const int64_t *counts,
                     int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, void *dst, int64_t dst_capacity,
                     unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, &v)) return rc;
    int64_t total = 0;
    if (int rc = pool_check(v, by_sample, starts, nreq, pool, dst, dst_capacity, false, flags, bad_index, &total)) return rc;

    Call c;
    if (int rc = begin_call(s, cuda_stream, flags & DDS_NO_SYNC, &c)) return rc;
    if (pool->nbags == 0) {
        note_empty_async(s, c);
        return DDS_OK;
    }
    ddsk_index_t ix;
    ddsk_pool_t kp;
    if (int rc = pool_stage(s, v, by_sample, starts, counts, nreq, pool, flags & DDS_IDX_ON_DEVICE, c.st, &ix, &kp)) return rc;
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, false, false, &kflags, &scr)) return rc;
    if (ddsk_pool(&v->kv, &ix, fixed_count, nreq, &kp, dst, &scr, kflags, c.st)) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    if (total_bytes) *total_bytes = total;
    return end_launch(s, c, total, nullptr, DDSK_CVT_NONE, false, nullptr, bad_index);
}

// The pooled accumulates behind dds_accumulate_batch_pooled / dds_accumulate_samples_pooled: the pooled get's checks
// and staging, with grad in place of the destination, then the same lifecycle (a write: it ends any overlap run).
static int pool_acc_impl(dds_store_t *s, const char *name, bool by_sample, const int64_t *starts, const int64_t *counts,
                         int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, double alpha, const void *grad,
                         int64_t grad_bytes, unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, total_bytes, bad_index, &v, kHostWrite)) return rc;
    int64_t total = 0;
    if (int rc = pool_check(v, by_sample, starts, nreq, pool, grad, grad_bytes, true, flags, bad_index, &total)) return rc;
    if (!std::isfinite(alpha)) return fail(DDS_ERR_ARG, "alpha must be finite");

    Call c;
    if (int rc = begin_call(s, cuda_stream, flags & DDS_NO_SYNC, &c)) return rc;
    if (pool->nbags == 0) {
        note_empty_async(s, c);
        return DDS_OK;
    }
    ddsk_index_t ix;
    ddsk_pool_t kp;
    if (int rc = pool_stage(s, v, by_sample, starts, counts, nreq, pool, flags & DDS_IDX_ON_DEVICE, c.st, &ix, &kp)) return rc;
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, false, false, &kflags, &scr)) return rc;
    if (ddsk_pool_acc(&v->kv, &ix, fixed_count, nreq, &kp, alpha, grad, &scr, kflags, c.st))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    if (total_bytes) *total_bytes = total;
    // (a write: queued, it is completed by the next dds_epoch_begin, as every batched write is)
    return end_launch(s, c, total, nullptr, DDSK_CVT_NONE, true, nullptr, bad_index);
}

int dds_get_batch_pooled(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                         int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, void *dst, int64_t dst_capacity,
                         unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    return pool_impl(s, name, false, starts, counts, fixed_count, nreq, pool, dst, dst_capacity, flags, cuda_stream,
                     total_bytes, bad_index);
}

int dds_get_samples_pooled(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq,
                           const dds_pool_t *pool, void *dst, int64_t dst_capacity, unsigned flags, void *cuda_stream,
                           int64_t *total_bytes, int64_t *bad_index) {
    return pool_impl(s, name, true, sample_ids, nullptr, 0, nreq, pool, dst, dst_capacity, flags, cuda_stream, total_bytes,
                     bad_index);
}

int dds_accumulate_batch_pooled(dds_store_t *s, const char *name, const int64_t *starts, const int64_t *counts,
                                int64_t fixed_count, int64_t nreq, const dds_pool_t *pool, double alpha,
                                const void *grad, int64_t grad_bytes, unsigned flags, void *cuda_stream,
                                int64_t *total_bytes, int64_t *bad_index) {
    return pool_acc_impl(s, name, false, starts, counts, fixed_count, nreq, pool, alpha, grad, grad_bytes, flags,
                         cuda_stream, total_bytes, bad_index);
}

int dds_accumulate_samples_pooled(dds_store_t *s, const char *name, const int64_t *sample_ids, int64_t nreq,
                                  const dds_pool_t *pool, double alpha, const void *grad, int64_t grad_bytes,
                                  unsigned flags, void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    return pool_acc_impl(s, name, true, sample_ids, nullptr, 0, nreq, pool, alpha, grad, grad_bytes, flags, cuda_stream,
                         total_bytes, bad_index);
}

// The multi-array path behind dds_get_samples_multi / dds_get_samples_multi_convert (cvts: one conversion per variable,
// or NULL for raw bytes)
static int multi_impl(dds_store_t *s, int nvars, const char *const *names, const int64_t *sample_ids, int64_t nreq,
                      void *const *dsts, const int64_t *dst_capacities, int64_t *const *dst_offsets, unsigned flags,
                      void *cuda_stream, int64_t *total_bytes, int64_t *bad_index, const dds_convert_t *cvts) {
    clear_error();
    if (bad_index) *bad_index = -1;
    if (!s || !names || !dsts || !dst_capacities) return fail(DDS_ERR_ARG, "null argument");
    if (nvars < 1 || nvars > DDSK_MAX_MULTI) return fail(DDS_ERR_ARG, "1..4 variables per multi-array batch");
    if (!(flags & DDS_DST_ON_DEVICE)) return fail(DDS_ERR_ARG, "multi-array batches deliver into device buffers");
    if (nreq < 0 || (nreq > 0 && !sample_ids)) return fail(DDS_ERR_ARG, "bad sample ids");
    Var *vv[DDSK_MAX_MULTI];
    std::string key;
    int64_t cap_total = 0;
    for (int v = 0; v < nvars; v++) {
        vv[v] = find_var(s, names[v]);
        if (!vv[v]) return fail(DDS_ERR_UNKNOWN_VAR, names[v] ? names[v] : "(null)");
        if (vv[v]->host != vv[0]->host) return fail(DDS_ERR_ARG, "a multi-array batch takes variables of one placement");
        if (!vv[v]->d_tab) return fail(DDS_ERR_ARG, "variable has no sample index (call dds_set_sample_index first)");
        if (dst_capacities[v] < 0) return fail(DDS_ERR_ARG, "negative capacity");
        key += vv[v]->name;
        key += '\n';
    }
    ddsk_cvt_t kc;
    const ddsk_cvt_t *kcp = nullptr;
    int64_t cap_src[DDSK_MAX_MULTI]; // the kernels check capacities in source bytes
    if (cvts) {
        if (int rc = make_cvt(vv, cvts, nvars, true, &kc)) return rc;
        for (int v = 0; v < nvars; v++)
            if ((uint64_t)dsts[v] % (uint64_t)(1 << cvt_out_log2(kc.code[v])) || (dst_offsets && (uint64_t)dst_offsets[v] % 8u))
                return fail(DDS_ERR_ARG, "destination not aligned to the output itemsize (or offsets to 8 bytes)");
        kcp = &kc;
    }
    for (int v = 0; v < nvars; v++) {
        cap_src[v] = kcp ? cvt_cap_to_src(dst_capacities[v], kc.code[v]) : dst_capacities[v];
        cap_total += cap_src[v];
    }
    const bool idx_dev = flags & DDS_IDX_ON_DEVICE, no_sync = flags & DDS_NO_SYNC;
    if (no_sync && !idx_dev) return fail(DDS_ERR_ARG, "async batches need device indices and a device destination");
    Call c;
    if (int rc = begin_call(s, cuda_stream, no_sync, &c)) return rc;
    if (total_bytes)
        for (int v = 0; v < nvars; v++) total_bytes[v] = 0;
    if (nreq == 0) {
        note_empty_async(s, c);
        return DDS_OK;
    }
    if (key != s->multi_key) { // (re)build the device array of windows for this combination of variables
        if (!s->d_multi_vars) CU(cudaMalloc((void **)&s->d_multi_vars, sizeof(ddsk_var_t) * DDSK_MAX_MULTI));
        CU(cudaStreamSynchronize(c.st)); // nothing in flight may still read the previous combination
        for (int v = 0; v < nvars; v++)
            CU(cudaMemcpy(&s->d_multi_vars[v], &vv[v]->kv, sizeof(ddsk_var_t), cudaMemcpyHostToDevice));
        s->multi_key = key;
    }
    const int64_t *d_ids = sample_ids;
    if (!idx_dev) {
        if (int rc = ensure_idx(s, nreq)) return rc;
        CU(cudaMemcpyAsync(s->d_starts, sample_ids, (size_t)nreq * 8, cudaMemcpyHostToDevice, c.st));
        d_ids = s->d_starts;
    }
    const bool host = vv[0]->host;
    const bool ovl = no_sync && (flags & DDS_OVERLAP) && !host;
    bool uses_scratch;
    if (int rc = plan_scratch(s, nreq * nvars, cap_total, kcp, ovl, host, &uses_scratch)) return rc;
    // a synchronous caller wants the per-variable totals: they are the last entries of the per-variable offsets, which
    // go to the caller's arrays or to a staging array of the store
    const bool stage_offs = !no_sync && total_bytes != nullptr;
    if (stage_offs) {
        if (int rc = ensure_offs(s, (int64_t)nvars * (nreq + 1))) return rc;
    }
    ddsk_multi_t m;
    memset(&m, 0, sizeof(m));
    m.nvars = nvars;
    m.host = host ? 1 : 0;
    m.vars_dev = s->d_multi_vars;
    for (int v = 0; v < nvars; v++) {
        m.table[v] = vv[v]->d_tab;
        m.nsamples[v] = vv[v]->nsamples;
        m.dst[v] = dsts[v];
        m.cap[v] = cap_src[v];
        m.offsets[v] = dst_offsets && dst_offsets[v] ? dst_offsets[v] : (stage_offs ? s->d_offs + (int64_t)v * (nreq + 1) : nullptr);
    }
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, ovl, uses_scratch, &kflags, &scr)) return rc;
    const int mrc = ddsk_gather_multi(&m, d_ids, nreq, &scr, kflags, kcp, c.st);
    s->scr.plan_tag = scr.plan_tag;
    if (mrc) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    // (a converting launch writes its total in output bytes to the total word, whichever plan it used)
    if (no_sync)
        return end_launch(s, c, -1, (uses_scratch && !kcp) ? &scr.req_dst[nreq * nvars] : scr.total, DDSK_CVT_NONE, false,
                          nullptr, nullptr);
    int64_t *hb = (int64_t *)s->h_small;
    if (total_bytes)
        for (int v = 0; v < nvars; v++) CU(cudaMemcpyAsync(&hb[v], m.offsets[v] + nreq, 8, cudaMemcpyDeviceToHost, c.st));
    CU(cudaStreamSynchronize(c.st));
    int rc = decode_status(s, c.st, s->h_status[0], bad_index);
    if (total_bytes)
        for (int v = 0; v < nvars; v++) total_bytes[v] = rc == DDS_ERR_CAPACITY ? 0 : hb[v];
    if (bad_index && *bad_index >= 0) *bad_index %= nreq; // index of the sample in the id list
    return rc;
}

int dds_get_samples_multi(dds_store_t *s, int nvars, const char *const *names, const int64_t *sample_ids, int64_t nreq,
                          void *const *dsts, const int64_t *dst_capacities, int64_t *const *dst_offsets, unsigned flags,
                          void *cuda_stream, int64_t *total_bytes, int64_t *bad_index) {
    return multi_impl(s, nvars, names, sample_ids, nreq, dsts, dst_capacities, dst_offsets, flags, cuda_stream, total_bytes,
                      bad_index, nullptr);
}

int dds_get_samples_multi_convert(dds_store_t *s, int nvars, const char *const *names, const int64_t *sample_ids,
                                  int64_t nreq, void *const *dsts, const int64_t *dst_capacities,
                                  int64_t *const *dst_offsets, unsigned flags, void *cuda_stream,
                                  const dds_convert_t *cvts, int64_t *total_bytes, int64_t *bad_index) {
    if (!cvts) {
        clear_error();
        if (bad_index) *bad_index = -1;
        return fail(DDS_ERR_ARG, "null conversion");
    }
    return multi_impl(s, nvars, names, sample_ids, nreq, dsts, dst_capacities, dst_offsets, flags, cuda_stream, total_bytes,
                      bad_index, cvts);
}

// completes the batches issued with DDS_NO_SYNC, and reports what every queue completed since the last call left
int dds_batch_wait(dds_store_t *s, int64_t *total_bytes, int64_t *bad_index) {
    if (!s) return fail(DDS_ERR_ARG, "null store");
    dds_store::Queue &q = s->q;
    if (q.pending) {
        CU(cudaSetDevice(s->device));
        if (int rc = drain_pending(s)) return rc;
    }
    const unsigned long long st = q.kept_status;
    if (total_bytes) *total_bytes = q.kept_total;
    q.kept_status = DDSK_STATUS_OK;
    q.kept_total = 0;
    return decode_status_word(st, bad_index);
}

int dds_get(dds_store_t *s, const char *name, int64_t start, int64_t count, int itemsize, void *buffer,
            int buffer_on_device) {
    // one request through the batch entry: same checks (ddstore.hpp:197-238); small results take the 1-CTA kernel
    if (!s) return fail(DDS_ERR_ARG, "null store");
    Var *v = find_var(s, name);
    if (!v) {
        clear_error();
        return fail(DDS_ERR_UNKNOWN_VAR, name ? name : "(null)");
    }
    // (a count above the variable's row total is invalid whatever the start: no room is needed for it)
    const int64_t cap = req_bytes(v, count);
    return dds_get_batch(s, name, &start, nullptr, count, 1, itemsize, buffer, cap, nullptr,
                         buffer_on_device ? DDS_DST_ON_DEVICE : 0u, nullptr, nullptr, nullptr);
}

static const char *kPushWindow = "\001dds-push-window";

int dds_push_setup(dds_store_t *s, int64_t max_requests, int64_t max_bytes) {
    clear_error();
    if (!s) return fail(DDS_ERR_ARG, "null store");
    if (s->push.ready) return fail(DDS_ERR_EXISTS, "push windows");
    int rc_local = DDS_OK;
    if (max_requests <= 0 || max_bytes <= 0) rc_local = fail(DDS_ERR_ARG, "push windows need positive sizes");
    // every rank must sit on a GPU of its own: a rank's kernel waits for the other ranks' kernels to run
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), s->device) != cudaSuccess) bus[0] = 0;
    (void)cudaGetLastError();
    struct Rec {
        char bus[32];
        int64_t max_requests, max_bytes;
        int32_t ok, pad_;
    } mine;
    memset(&mine, 0, sizeof(mine));
    memcpy(mine.bus, bus, sizeof(bus));
    mine.max_requests = max_requests;
    mine.max_bytes = max_bytes;
    mine.ok = rc_local == DDS_OK;
    std::vector<Rec> all((size_t)s->size);
    if (int rc = dds_comm_allgather(s->comm, &mine, all.data(), sizeof(Rec))) return rc;
    bool bad = false, shared = false, differ = false;
    for (int a = 0; a < s->size; a++) {
        bad |= !all[(size_t)a].ok;
        differ |= all[(size_t)a].max_requests != max_requests || all[(size_t)a].max_bytes != max_bytes;
        for (int b = a + 1; b < s->size; b++) shared |= memcmp(all[(size_t)a].bus, all[(size_t)b].bus, sizeof(mine.bus)) == 0;
    }
    if (bad) return rc_local ? rc_local : fail(DDS_ERR_ARG, "a peer rank passed bad push window sizes");
    if (differ) return fail(DDS_ERR_ARG, "every rank must pass the same push window sizes");
    if (shared) return fail(DDS_ERR_ARG, "the collective push fetch needs every rank on a GPU of its own");
    auto up = [](int64_t v) { return (v + 4095) / 4096 * 4096; };
    ddsk_push_t &t = s->push.table;
    memset(&t, 0, sizeof(t));
    t.nranks = s->size;
    t.me = s->rank;
    t.max_requests = max_requests;
    t.max_bytes = max_bytes;
    t.idx_off[0] = DDSK_PUSH_HDR_BYTES;
    t.idx_off[1] = t.idx_off[0] + up(max_requests * 8);
    t.dst_off[0] = t.idx_off[1] + up(max_requests * 8);
    t.dst_off[1] = t.dst_off[0] + up(max_bytes);
    const int64_t bytes = t.dst_off[1] + up(max_bytes);
    if (int rc = register_var(s, kPushWindow, nullptr, bytes, 1, 1, 0, true, DDS_PLACE_HBM)) return rc; // collective, zero-filled, mapped
    Var *w = find_var(s, kPushWindow);
    for (int r = 0; r < s->size; r++) t.win[r] = (unsigned char *)w->kv.bases[r];
    CU(cudaMemset(t.win[t.me] + 24, 0xFF, 8)); // the window's status word starts as "ok"
    CU(cudaMalloc((void **)&s->push.d_table, sizeof(ddsk_push_t)));
    CU(cudaMemcpy(s->push.d_table, &t, sizeof(t), cudaMemcpyHostToDevice));
    s->push.step = 0;
    if (int rc = dds_comm_barrier(s->comm)) return rc; // every window is armed before anyone pushes
    s->push.ready = true;
    return DDS_OK;
}

int dds_get_batch_push(dds_store_t *s, const char *name, const int64_t *starts_dev, int64_t fixed_count, int64_t nreq,
                       int itemsize, void **dst_out, void *cuda_stream) {
    if (!s || !dst_out) return fail(DDS_ERR_ARG, "null store or dst_out");
    if (!s->push.ready) return fail(DDS_ERR_ARG, "no push windows (call dds_push_setup on every rank first)");
    Var *v;
    if (int rc = entry_var(s, name, &itemsize, nullptr, nullptr, &v, "the push fetch does not serve DDS_PLACE_HOST variables"))
        return rc;
    const int64_t nb = fixed_count * v->kv.row_bytes;
    if (fixed_count <= 0 || nreq < 0 || (nreq > 0 && !starts_dev)) return fail(DDS_ERR_ARG, "push batches fetch count >= 1 rows per request");
    if (nreq > s->push.table.max_requests || nreq * nb > s->push.table.max_bytes)
        return fail(DDS_ERR_CAPACITY, "batch larger than the push window");
    // always queued: dds_batch_wait reports what the owners found wrong with this rank's requests. Never overlapped: a
    // push ends any overlap run.
    Call c;
    if (int rc = begin_call(s, cuda_stream, true, &c)) return rc;
    int kflags;
    ddsk_scratch_t scr;
    if (int rc = launch_flags(s, c, false, false, &kflags, &scr)) return rc;
    const unsigned long long step = ++s->push.step;
    if (ddsk_gather_push(&v->kv, &s->push.table, s->push.d_table, starts_dev, fixed_count, nreq, step, &scr, c.st))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    *dst_out = s->push.table.win[s->push.table.me] + s->push.table.dst_off[step & 1ull];
    return end_launch(s, c, nreq * nb, nullptr, DDSK_CVT_NONE, false, nullptr, nullptr);
}

int dds_query(dds_store_t *s, const char *name, dds_varinfo_t *out) {
    if (!s || !out) return fail(DDS_ERR_ARG, "null store or out");
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    memset(out, 0, sizeof(*out));
    out->itemsize = v->itemsize;
    out->disp = v->disp;
    out->nranks = s->size;
    out->fence_active = v->fence_active;
    out->local_nrows = v->nrows;
    out->total_nrows = v->lenlist.empty() ? 0 : v->lenlist.back();
    for (int r = 0; r < s->size && r < 64; r++) out->lenlist[r] = v->lenlist[(size_t)r];
    out->local_base = v->base;
    return DDS_OK;
}

int dds_epoch_begin(dds_store_t *s) {
    // src/ddstore.cxx:51-63
    clear_error();
    if (!s) return fail(DDS_ERR_ARG, "null store");
    for (auto &x : s->vars)
        if (x.second.fence_active) return fail(DDS_ERR_FENCE_ACTIVE);
    CU(cudaSetDevice(s->device));
    // queued puts are part of the epoch that ends here (a queue of gets is left to dds_batch_wait)
    if (int rc = drain_pending(s, true)) return rc;
    CU(cudaStreamSynchronize(s->stream));
    if (int rc = drain_update_streams(s)) return rc; // dds_update_async copies on caller streams are part of the epoch
    if (int rc = dds_comm_barrier(s->comm)) return rc;
    for (auto &x : s->vars) x.second.fence_active = true;
    return DDS_OK;
}

int dds_epoch_end(dds_store_t *s) {
    // src/ddstore.cxx:65-77
    clear_error();
    if (!s) return fail(DDS_ERR_ARG, "null store");
    for (auto &x : s->vars)
        if (!x.second.fence_active) return fail(DDS_ERR_FENCE_INACTIVE);
    CU(cudaSetDevice(s->device));
    if (int rc = drain_pending(s)) return rc;
    CU(cudaStreamSynchronize(s->stream));
    if (int rc = drain_update_streams(s)) return rc;
    if (int rc = dds_comm_barrier(s->comm)) return rc;
    for (auto &x : s->vars) x.second.fence_active = false;
    return DDS_OK;
}

static void local_release(dds_store *s) {
    for (auto &x : s->vars) release_var(x.second, s->rank);
}

int dds_free(dds_store_t *s) {
    // src/ddstore.cxx:79-96 (MPI_Win_free is collective; so is this)
    clear_error();
    if (!s) return fail(DDS_ERR_ARG, "null store");
    if (s->vars.empty() && s->zombies.empty() && s->zombie_blocks.empty()) return DDS_OK;
    CU(cudaSetDevice(s->device));
    if (int rc = drain_pending(s)) return rc;
    s->update_streams.clear();
    CU(device_sync(s));
    int rc = dds_comm_barrier(s->comm); // nobody is reading any more
    local_release(s);
    int rc2 = dds_comm_barrier(s->comm); // every mapping is closed before the memory goes away
    for (auto &x : s->vars) free_shard(x.second);
    for (void *z : s->zombies) cudaFree(z);
    for (auto &b : s->zombie_blocks) dds_vmm::release(&b);
    s->vars.clear();
    s->zombies.clear();
    s->zombie_blocks.clear();
    s->multi_key.clear();
    if (s->push.d_table) cudaFree(s->push.d_table);
    s->push = dds_store::Push();
    return rc ? rc : rc2;
}

void dds_destroy(dds_store_t *s) {
    if (!s) return;
    // Teardown of this rank's handle. The reference's destructor runs the collective free() (ddstore.cxx:41-44); here
    // peers that imported a shard as a VMM handle hold their own reference to the memory, so a local release is safe
    // for them. Shards that peers read through a raw pointer (thread-ranks) or a legacy IPC mapping have no such
    // protection: if any is still registered, go through the collective dds_free first so that no peer can fault on
    // memory this rank is about to release (the communicator's own timeout bounds the wait if a peer is gone).
    bool unprotected = false;
    for (auto &x : s->vars) unprotected |= x.second.unprotected_peers;
    if (unprotected && s->size > 1) (void)dds_free(s);
    if (cudaSetDevice(s->device) == cudaSuccess) {
        device_sync(s);
        local_release(s);
        for (auto &x : s->vars) free_shard(x.second);
        for (void *z : s->zombies) cudaFree(z);
        for (auto &b : s->zombie_blocks) dds_vmm::release(&b);
        if (s->scr.status) cudaFree(s->scr.status);
        if (s->scr.counters) cudaFree(s->scr.counters);
        if (s->scr.req_src) cudaFree(s->scr.req_src);
        if (s->scr.req_dst) cudaFree(s->scr.req_dst);
        if (s->scr.tile_sums) cudaFree(s->scr.tile_sums);
        if (s->scr.seg_tab) cudaFree(s->scr.seg_tab);
        for (auto &sl : s->slots) {
            if (sl.req_src) cudaFree(sl.req_src);
            if (sl.req_dst) cudaFree(sl.req_dst);
            if (sl.tile_sums) cudaFree(sl.tile_sums);
            if (sl.seg_tab) cudaFree(sl.seg_tab);
        }
        if (s->d_starts) cudaFree(s->d_starts);
        if (s->d_counts) cudaFree(s->d_counts);
        if (s->d_out) cudaFree(s->d_out);
        if (s->d_offs) cudaFree(s->d_offs);
        if (s->h_status) cudaFreeHost(s->h_status);
        if (s->h_small) cudaFreeHost(s->h_small);
        if (s->ingest) {
            s->ingest->stop();
            cudaStreamSynchronize(s->ingest->stream);
            for (int k = 0; k < 2; k++) {
                cudaFreeHost(s->ingest->pin[k]);
                cudaEventDestroy(s->ingest->ev[k]);
            }
            cudaStreamDestroy(s->ingest->stream);
            delete s->ingest;
            s->ingest = nullptr;
        }
        if (s->h_mb) cudaFreeHost(s->h_mb);
        if (s->d_vars) cudaFree(s->d_vars);
        if (s->db_stream) cudaStreamDestroy(s->db_stream);
        if (s->d_multi_vars) cudaFree(s->d_multi_vars);
        if (s->push.d_table) cudaFree(s->push.d_table);
            if (s->stream) cudaStreamDestroy(s->stream);
    }
    (void)cudaGetLastError();
    delete s;
}

int dds_synth_fill(dds_store_t *s, const char *name, uint64_t seed) {
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    CU(cudaSetDevice(s->device));
    int64_t first = s->rank > 0 ? v->lenlist[(size_t)s->rank - 1] : 0;
    if (ddsk_synth_fill(v->base, first, v->nrows, v->disp, v->itemsize, seed, s->stream))
        return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    CU(cudaStreamSynchronize(s->stream));
    return DDS_OK;
}

int dds_synth_verify(dds_store_t *s, const char *name, const void *packed_dev, const int64_t *starts_dev,
                     const int64_t *counts_dev, int64_t fixed_count, const int64_t *offsets_dev, int64_t nreq, uint64_t seed,
                     void *cuda_stream, uint64_t *result) {
    if (!s || !result) return fail(DDS_ERR_ARG, "null store or result");
    Var *v;
    if (int rc = entry_var(s, name, nullptr, nullptr, nullptr, &v)) return rc;
    CU(cudaSetDevice(s->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : s->stream;
    const size_t words = 2 + DDSK_MAX_RANKS;
    unsigned long long *d_out = nullptr;
    CU(cudaMalloc((void **)&d_out, words * 8));
    cudaError_t e = cudaMemsetAsync(d_out, 0, words * 8, st);
    int krc = 0;
    if (e == cudaSuccess)
        krc = ddsk_synth_verify(&v->kv, packed_dev, starts_dev, counts_dev, fixed_count, offsets_dev, nreq, v->disp, v->itemsize,
                                seed, d_out, st);
    if (e == cudaSuccess && !krc) e = cudaMemcpyAsync(result, d_out, words * 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && !krc) e = cudaStreamSynchronize(st);
    cudaFree(d_out);
    if (krc) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    if (e != cudaSuccess) return cuda_fail(e, "dds_synth_verify");
    return DDS_OK;
}

int dds_test_occupy(int device, int ctas, int smem_bytes, uint64_t nanoseconds, void *cuda_stream) {
    clear_error();
    CU(cudaSetDevice(device));
    if (ddsk_occupy(ctas, smem_bytes, nanoseconds, cuda_stream)) return fail(DDS_ERR_CUDA, ddsk_last_cuda_error());
    return DDS_OK;
}

unsigned long long dds_kernel_launches(void) { return ddsk_launch_count(); }
int dds_host_gather_ctas(void) { return ddsk_host_gather_ctas(); }
void dds_gather_geometry(int *ctas, int *warps_per_cta, int *stages, int *chunk_bytes, int *smem_bytes) {
    ddsk_gather_geometry(ctas, warps_per_cta, stages, chunk_bytes, smem_bytes);
}
void dds_pool_geometry(int adjoint, int64_t row_bytes, int dtype, int64_t nbags, int aligned16, int host, int *vb,
                       int64_t *slice, int64_t *nslices, int64_t *windows, int *ctas) {
    ddsk_pool_geometry(adjoint, row_bytes, dtype, nbags, aligned16, host, vb, slice, nslices, windows, ctas);
}

} // extern "C"
