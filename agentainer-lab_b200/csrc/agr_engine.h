// agr_engine.h — what the host-side sources of the engine share (agr_engine.cu: the core; agr_front.cu, agr_snapshot.cu,
// agr_exchange.cu).  Private to the library.  Functions live in agr_impl, whose symbols are hidden: the library exports none
// of them.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>      // types only: every NCCL symbol is resolved with dlopen/dlsym at run time
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>
#include "../../include/agentainer_gpu.h"
#include "agr_agents.hpp"
#include "agr_kernels.cuh"
#include "agr_svc.h"

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(AGR_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_));              \
    } while (0)

// One exchange over a batch: K4's launch parameters, the per-peer send / receive counts, and their offsets.  Send offsets are
// owner-major (in-place mode: the peers' segments only), receive offsets source-major.
struct exchange_plan {
    agr_k4_params p{};
    uint32_t G = 1, me = 0, scnt[32], rcnt[32], soff[33], roff[33], n_local = 0, n_recv = 0;
    uint32_t recv_res_base = 0;      // index of the first received item's result in the result array
};

// Rows [first, first + n) whose records lie back to back.  On a variable-length engine a row that agr_reserve_rows (or the
// exchange) hands out owns a 512-byte slot of the byte ring: the record of row first + i is at physical byte vbase + 512 i.
struct slot_run {
    uint64_t first = 0;
    uint32_t n = 0;
    uint64_t vbase = 0;          // (variable-length engines only)
};
// a reservation of agr_reserve_rows that K1 has not decided yet: rows [first, end), slots from vbase (variable-length engines)
struct resv_run {
    uint64_t first, end, vbase;
};

// grow-only scratch: a buffer and the element count it was allocated with (regrow sets both)
template <typename T>
struct scratch {
    T* p = nullptr;
    size_t cap = 0;
};

// the header of a full snapshot file (agr_snapshot); a delta file carries the one of its cut
struct snap_header {
    char magic[8];                 // "AGRSNAP3"
    uint32_t flags, n_agents, shard, gen;
    uint64_t rows_used, vused, log_len[2], id_secret, scan_lo, resp_used, expired_total, tail, released_total, slab_rows, vtail, vcap, resp_tail, resp_cap;
};
// AGR_CFG_DELTA_SNAPSHOT: what the next snapshot builds on — the files since the last full one (absolute paths, oldest
// first), the full file's size and the deltas' total, the last cut's header, its ingested bound and its digest
struct snap_chain {
    std::vector<std::string> paths;
    uint64_t full_bytes = 0, delta_bytes = 0;
    snap_header base{};
    uint64_t base_bound = 0;
    unsigned long long digest[2] = {0, 0};
};

struct svc_host {
    // ---- read-mostly (every caller reads these on every call; nothing here is written while callers run)
    svc_desc* desc = nullptr; uint8_t* payload = nullptr; svc_res* res = nullptr; svc_ctl* ctl = nullptr;   // pinned, device-mapped
    std::atomic<uint32_t>* ready = nullptr;             // [SVC_SLOTS] (lap + 1) << 2 | SVC_OP_* once the slot's payload is complete
    uint32_t spin_cpus = 1;                             // how many waiters may spin (CPU allowance minus dispatcher and driver threads)
    std::atomic<bool> shutdown{false}, sleeping{false}; // (sleeping flips only when the ring has been empty for 2 ms)
    std::atomic<int> fatal{0};                          // a CUDA error in the dispatcher: every later call fails with it
    // ---- the words the callers / the dispatcher keep writing: a cache line each
    alignas(64) std::atomic<uint64_t> head{0};          // next ring slot to hand out (absolute number)
    alignas(64) std::atomic<uint32_t> waiters{0};       // callers blocked in svc_wait right now
    alignas(64) std::atomic<uint64_t> scanned{0};       // dispatcher: first slot whose ready word it has not consumed yet (>= taken)
    std::atomic<uint64_t> rows_out{0};                  // = the handle's rows_used (sync_window): callers rebuild a row's high bits from it (svc_try)
    // ---- the dispatcher's own
    alignas(64) uint64_t taken = 0;                     // first slot not yet put into a batch
    uint64_t seq = 0;                                   // last batch number published
    bool running = false;                               // service kernel resident (changed under the handle mutex only)
    std::chrono::steady_clock::time_point started;      // when it was launched
    agr_k2_scratch k2{};                                // K2 scratch of the service kernel (SVC_MAX_OPS ops)
    uint32_t* d_dupfix = nullptr;
    unsigned long long *d_boff = nullptr, *d_bdst = nullptr; uint32_t* d_bhlen = nullptr;   // per-outcome byte places (svc_dev)
    std::atomic<uint64_t> batches{0}, ops{0};
    // diagnostics (AGR_SVC_DEBUG=1 prints them when the handle is destroyed)
    uint64_t starts = 0, stops = 0, sleeps = 0, flow_waits = 0;
    double cyc[4] = {0, 0, 0, 0}; uint64_t polls = 0;
    std::thread thr;
    alignas(64) std::mutex smu; std::condition_variable scv;   // the dispatcher sleeps here when the ring has been empty for a while
};

struct agr_handle {
    std::mutex mu;
    agr_config cfg{};
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;        // H2D of chunk k+1 overlaps K1 of chunk k (agr_ingest pipeline)
    std::vector<cudaEvent_t> chunk_ev;
    cudaStream_t d2h_stream = nullptr;         // verdicts / ids of chunk k go back while chunk k+1 comes in (PCIe is full duplex)
    std::vector<cudaEvent_t> out_ev;
    agr_verdict* d_verdicts = nullptr;         // [max_batch], written by k1_post
    agr_verdict* h_verdicts = nullptr;         // pinned [max_batch]
    uint8_t* d_ids = nullptr;                  // [max_batch][16] Request.ID per record (agr_ingest_ex)
    uint8_t* h_ids = nullptr;                  // pinned
    agr_dev d{};
    uint64_t rows_used = 0;   // LOGICAL rows handed out so far (ring: includes the rows skipped at a wrap)
    uint64_t tail = 0;        // ring: first logical row that has not been released
    uint32_t* d_log_scratch = nullptr; uint32_t* d_lc_chunks = nullptr;   // ring: log compaction
    uint64_t released_total = 0;
    uint32_t* d_reclaim_scratch = nullptr;                        // k_first_live: {offset found, ticket}
    uint8_t* d_reclaim = nullptr; uint8_t* h_reclaim = nullptr;   // agr_reclaim's scan result (device scratch / pinned copy)
    cudaEvent_t reclaim_ev = nullptr; bool reclaim_pending = false; uint64_t reclaim_bound = 0;
    uint32_t* dupfix_base = nullptr; uint32_t batch_phase = 0;   // two sets of per-batch words, used alternately
    uint64_t scan_lo = 0;     // every row below has left its pending list for good
    uint64_t sweep_clean = 0; // append-only slab: rows below were ingested when agr_expire last ran (their chunks' time bounds are exact)
    // host agent map + mirror
    std::unordered_map<std::string, uint32_t> slot_of;
    std::vector<std::string> agent_names;
    std::vector<uint8_t> agent_status;
    std::vector<agr_agent_key> akeys_host;
    std::vector<uint32_t> akey_index;          // slot -> index of its entry in the open-addressing key table (agr_agents.hpp)
    // slot reuse once every slot has been handed out (set_agent_state_locked): the removed slots no live row carried at the last
    // held-slot scan, highest first (taken from the back), and the generations of the events that can free a slot (agr_drop_agent,
    // a release of rows, a restore) now and at that scan
    std::vector<uint32_t> free_slots;
    uint64_t agent_gen = 0, free_gen = ~0ull;
    uint32_t *d_slot_cand = nullptr, *d_slot_held = nullptr;   // the scan's bitmaps, max_agents bits each (allocated on first use)
    // staging
    uint8_t* bounce[2] = {nullptr, nullptr};   // pinned, for pageable caller buffers
    cudaEvent_t bounce_ev[2] = {nullptr, nullptr};
    size_t bounce_bytes = 0;
    agr_dop* h_ops = nullptr;                  // pinned [16] (single-key lookups)
    agr_outcome* h_outs = nullptr;             // pinned [max_batch]
    agr_outcome* d_outs = nullptr;             // [max_batch]
    int32_t* h_results = nullptr;              // pinned [max_batch]
    agr_k2_scratch k2{};
    uint32_t* d_hrid = nullptr;                // rows found by the single-key resolve (k_resolve)
    uint32_t* h_k2flag = nullptr;              // pinned: k2_append's overflow flag of the last batch
    agr_dop* d_ops = nullptr;
    std::vector<resv_run> resv;                // rows handed out by agr_reserve_rows and not ingested yet, in row order
    // K3
    scratch<uint32_t> d_matrix, d_cta_matrix;
    scratch<uint32_t> d_selmask;               // one selection bit per scanned item (k3_mark -> k3_place)
    uint32_t* d_gtotal = nullptr; uint32_t* d_goff = nullptr;
    scratch<uint32_t> d_out_rid, d_out_slot;
    uint32_t* d_min_inq = nullptr;
    scratch<uint8_t> d_gather, h_gather;       // (h_gather pinned)
    uint32_t* h_small = nullptr;               // pinned scratch (>= 64 words)
    scratch<unsigned long long> d_cdf;
    // launch accounting
    uint64_t k1_launches = 0, k2_launches = 0, k3_launches = 0, k4_launches = 0;
    uint64_t replay_scans = 0, replay_dispatched = 0;
    std::vector<void*> dev_allocs, host_allocs;
    alignas(64) unsigned char tmap[128];       // CUtensorMap of the slab for the fixed-stride TMA K1
    // stored responses: byte slab + per-row (offset, length), written off the hot path
    uint8_t* d_resp = nullptr; uint64_t resp_used = 0, resp_cap = 0;   // bytes appended so far (ring: logical, pads included) / capacity
    uint64_t resp_tail = 0;                    // ring: logical offset of the oldest byte a live row still refers to
    unsigned long long* d_resp_off = nullptr; uint32_t* d_resp_len = nullptr;
    uint32_t* d_resp_hlen = nullptr;           // leading bytes of the stored response that are its flattened headers
    unsigned long long* d_err_off = nullptr; uint32_t* d_err_len = nullptr;   // Request.Error text, same byte slab
    // agr_complete_ex staging, allocated on first use: per-op offsets / slab places / header lengths, and the batch's bytes
    unsigned long long *h_boff = nullptr, *d_boff = nullptr, *h_bdst = nullptr, *d_bdst = nullptr;
    uint32_t *h_bhlen = nullptr, *d_bhlen = nullptr;
    scratch<uint8_t> h_bsrc, d_bsrc;           // (h_bsrc pinned)
    // K5 (JSON wire form) scratch
    scratch<uint32_t> d_jlen; scratch<unsigned long long> d_joff, d_jchunk;
    scratch<uint8_t> d_json;
    uint64_t k5_launches = 0;
    uint64_t expired_total = 0;                // records dropped by agr_expire so far
    // single-request front end (AGR_CFG_COMBINE): pinned op ring + dispatcher thread + resident service kernel (agr_svc.h)
    struct svc_host* svc = nullptr;
    // variable-length mode
    uint64_t vused = 0, vcap = 0;               // bytes appended so far (ring: logical, pads included) / capacity
    uint64_t vtail = 0;                        // ring: logical offset of the first byte that has not been released
    uint32_t* d_voffsets = nullptr; uint32_t* d_tile_first = nullptr;   // per-batch offsets [max_batch+1], tile index
    uint32_t* h_voffsets = nullptr;
    uint32_t* d_slot_off = nullptr;            // 512 i for i = 0 .. slot_off_max: the offsets of a run of 512-byte slots (K1v)
    uint32_t slot_off_max = 0;
    scratch<uint32_t> d_lens; scratch<unsigned long long> d_goffs;      // gather scratch
    // long records (stored length over AGR_VAR_MAX_RECORD, up to cfg.max_record_bytes): the batch's list for K1v's checksum
    // pass (agr_launch_k1v_long: batch indices, then first pieces) and, on the device, the list followed by two sums per record
    std::vector<uint32_t> long_list;
    scratch<uint32_t> d_long;
    // multi-GPU exchange (K4)
    ncclComm_t comm = nullptr; int rank = 0, world = 1;
    uint8_t* d_stage = nullptr;                // incoming batch before binning [max_batch * 512]
    uint8_t* d_send = nullptr;                 // owner-major send buffer [max_batch * 512]
    uint8_t* d_owner = nullptr; uint32_t* d_perm = nullptr;
    uint32_t* d_k4matrix = nullptr; uint32_t k4_nwarps = 0;
    uint32_t* d_k4cnt = nullptr;               // [4][32]: gtotal, goff(33 → second row pair), recv counts
    agr_verdict* d_xverd = nullptr;            // verdicts of local + received rows [2 * max_batch]
    agr_verdict* d_vback = nullptr;            // verdicts returned by owners, owner-major [max_batch]
    agr_verdict* d_vout = nullptr;             // caller-order verdicts [max_batch]
    exchange_plan xdbg{}; uint64_t xdbg_first = 0; uint32_t xdbg_n = 0; bool xdbg_open = false;   // agr_debug_exchange_begin -> _end
    // AGR_CFG_TIMING: CUDA-event pairs around the dominant K1 kernel, on the launching stream
    std::vector<cudaEvent_t> tev; uint64_t tev_next = 0, tev_read = 0, timing_calls = 0;
    cudaEvent_t op_ev[10] = {};                // [0,1] last K2 group, [2,3] last K3 select group, [4,5] last K5 encode, [6,7] last snapshot cut, [8,9] the relocation of the restore that made the engine
    bool op_timed[5] = {false, false, false, false, false};
    // AGR_CFG_ONLINE_SNAPSHOT: the cut's device shadow of the sections rewritten in place (the two log lengths at offset 0, then
    // every such section at shadow_off), the writer's own stream, its two pinned buffers, and the pins (agr_snapshot)
    uint8_t* d_shadow = nullptr; size_t shadow_off[17] = {};
    cudaStream_t snap_stream = nullptr;
    cudaEvent_t snap_ev[3] = {nullptr, nullptr, nullptr};   // [0] the cut, [1 + b] the last copy into snap_buf[b]
    uint8_t* snap_buf[2] = {nullptr, nullptr}; size_t snap_buf_bytes = 0;
    int snap_cur = 0; size_t snap_pend = 0;                 // buffer of the next chunk; bytes of the chunk waiting in the other one
    std::mutex snap_mu;                                      // one online snapshot at a time: there is one shadow
    bool pinned = false; uint64_t pin_tail = 0, pin_vtail = 0, pin_resp_tail = 0;   // (h->mu) the cut's ring tails while it is written
    // AGR_CFG_DELTA_SNAPSHOT (and a restore that applies deltas): the compare cut's dirty bits (word blocks, then the completed
    // and failed logs' blocks at snap_bit_off[1], [2]) and digest, the pinned copy the writer reads them from (the digest at
    // offset 16, the bits at 32), the device block list and the staging buffer of the block gather / scatter
    uint32_t* d_snap_bits = nullptr; unsigned long long* d_snap_digest = nullptr; uint8_t* h_snap_bits = nullptr;
    size_t snap_bit_off[3] = {}, snap_bit_words = 0;
    uint32_t* d_snap_list = nullptr; uint8_t* d_snap_stage = nullptr; size_t snap_stage_bytes = 0;
    snap_chain chain;                                        // (snap_mu) empty: the next snapshot is a full file
};
#define AGR_TIMING_RING 1024

namespace agr_impl __attribute__((visibility("hidden"))) {
extern thread_local std::string g_err;   // agr_last_error
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
template <typename T>
static int dev_alloc(agr_handle* h, T** p, size_t count, bool zero) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T));
    if (e != cudaSuccess) return fail(AGR_ENOMEM, std::string("cudaMalloc ") + std::to_string(count * sizeof(T)) + " B: " + cudaGetErrorString(e));
    if (zero) { e = cudaMemsetAsync(q, 0, count * sizeof(T), h->stream); if (e != cudaSuccess) return fail(AGR_ECUDA, cudaGetErrorString(e)); }
    h->dev_allocs.push_back(q);
    *p = (T*)q;
    return 0;
}
template <typename T>
static int host_alloc(agr_handle* h, T** p, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaHostAlloc(&q, count * sizeof(T), cudaHostAllocDefault);
    if (e != cudaSuccess) return fail(AGR_ENOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
    h->host_allocs.push_back(q);
    *p = (T*)q;
    return 0;
}
#define TRY(x) do { int r_ = (x); if (r_ < 0) return r_; } while (0)
// replaces s by a buffer of count elements (device memory, or pinned host memory) and releases the old one (every user of
// the old buffer has been synchronised by then: the callers hold the handle mutex and the previous operation ended with a
// stream sync)
template <typename T>
static int regrow(agr_handle* h, scratch<T>& s, size_t count, bool pinned = false) {
    T* old = s.p;
    TRY(pinned ? host_alloc(h, &s.p, count) : dev_alloc(h, &s.p, count, false));
    s.cap = count;
    if (old) {
        cudaStreamSynchronize(h->stream);
        std::vector<void*>& allocs = pinned ? h->host_allocs : h->dev_allocs;
        auto it = std::find(allocs.begin(), allocs.end(), (void*)old);
        if (it != allocs.end()) allocs.erase(it);
        if (pinned) cudaFreeHost(old); else cudaFree(old);
    }
    return 0;
}

// ---- logical rows (arrival numbers, what the API speaks) vs physical rows (where the record lives; see agr_dev)
static inline bool is_ring(const agr_handle* h) { return (h->cfg.flags & AGR_CFG_RING) != 0; }
static inline uint64_t phys_row(const agr_handle* h, uint64_t l) { return is_ring(h) ? l % h->cfg.slab_rows : l; }
static inline uint64_t rows_span(const agr_handle* h) {       // physical rows that have ever been handed out
    return is_ring(h) ? std::min<uint64_t>(h->rows_used, h->cfg.slab_rows) : h->rows_used;
}
// (called under the handle mutex by every change of rows_used: reserve_rows_locked stores the new value before the dispatcher
// publishes the batch whose answers name the rows)
static inline void sync_svc_rows(agr_handle* h) {
    if (h->svc) h->svc->rows_out.store(h->rows_used, std::memory_order_release);
}
static inline void sync_window(agr_handle* h) {               // the live window the kernels check decoded ids against
    h->d.tail = h->tail; h->d.head_l = h->rows_used;
    h->d.ring_rows = is_ring(h) ? (uint32_t)h->cfg.slab_rows : 0u;
    h->d.tail_phys = is_ring(h) ? (uint32_t)(h->tail % h->cfg.slab_rows) : 0u;
    sync_svc_rows(h);
}

int svc_stop_locked(agr_handle* h);
// the handle lock every entry point other than the single-request path takes: the resident kernel owns the handle's stream
// while it runs, so it is stopped first (it finishes the batches already published) and started again by the dispatcher
struct HLock {
    agr_handle* h;
    explicit HLock(agr_handle* h_) : h(h_) {
        h->mu.lock();
        if (h->svc && h->svc->running) { cudaSetDevice(h->device); svc_stop_locked(h); }
    }
    ~HLock() { h->mu.unlock(); }
    HLock(const HLock&) = delete; HLock& operator=(const HLock&) = delete;
};

// agr_engine.cu
int k2_scratch_alloc(agr_handle* h, size_t n);
bool is_pinned(const void* p);
int d2h_staged(agr_handle* h, void* dst, const void* dsrc, size_t bytes, void* stage);
int upload_rows(agr_handle* h, uint8_t* dst, const uint8_t* src, size_t bytes, bool src_pinned, int& bk);
int read_log_lens(agr_handle* h, unsigned long long lens[2]);
int grow_events(std::vector<cudaEvent_t>& ev, size_t k);
int chunk_bounds_unknown(agr_handle* h);
int ring_reindex_locked(agr_handle* h);
int push_agent_status(agr_handle* h, uint32_t slot, uint8_t status);
int set_agent_state_locked(agr_handle* h, const char* agent_id, uint8_t status, bool upload);
int agent_forget_locked(agr_handle* h, uint32_t slot, bool upload);
int agent_bind_locked(agr_handle* h, uint32_t slot, const char* agent_id, uint8_t status, bool upload);
uint64_t ingested_bound(const agr_handle* h);
void resv_remove(agr_handle* h, uint64_t first, uint64_t end);
int reserve_rows_locked(agr_handle* h, uint32_t n, uint64_t* first);
int vbytes_fit(const agr_handle* h, uint64_t bytes, uint64_t* vpad);
uint64_t vbytes_take(agr_handle* h, uint64_t bytes, uint64_t vpad);
int reserve_run_locked(agr_handle* h, uint32_t n, bool listed, slot_run* run);
int row_runs(agr_handle* h, uint64_t first, uint32_t n, std::vector<slot_run>& out);
int op_time_begin(agr_handle* h, int g);
int op_time_end(agr_handle* h, int g);
int launch_k1_locked(agr_handle* h, uint64_t first, uint32_t n, agr_verdict* d_out, uint8_t* d_ids = nullptr);
int decide_run_locked(agr_handle* h, const slot_run& r, agr_verdict* d_out);
static inline uint8_t* run_ptr(const agr_handle* h, const slot_run& r) {   // where the run's first record lies
    return (h->cfg.flags & AGR_CFG_VARLEN) ? h->d.slab + r.vbase : h->d.slab + phys_row(h, r.first) * AGR_REC;
}
int resp_reserve_locked(agr_handle* h, uint64_t need, uint64_t len, unsigned long long* off);
int check_segments(const agr_outcome* outs, uint32_t n, const uint64_t* offsets, const uint32_t* hdr_lens, uint64_t* total,
                   uint64_t* max_len);
// agr_last_error of an agr_complete / agr_complete_ex whose pushes did not all fit the completed / failed log (batch and ring)
constexpr const char* K2_LOG_FULL =
    "completed / failed log full: entries of this batch were dropped (raise agr_config.log_entries, or agr_reclaim)";
// agr_front.cu
int svc_create(agr_handle* h);
void svc_destroy(agr_handle* h);
int svc_ingest(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid);
int svc_ingest_var(agr_handle* h, const uint8_t* blob, const uint32_t* offsets, uint32_t n, agr_verdict* out, uint8_t (*ids)[16],
                   uint64_t* first_rid);
int svc_complete(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results);
int svc_complete_ex(agr_handle* h, const agr_outcome* outs, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                    const uint32_t* hdr_lens, int32_t* results);
// agr_snapshot.cu
int snap_online_create(agr_handle* h);
// agr_exchange.cu
void comm_destroy(agr_handle* h);
}  // namespace agr_impl
using namespace agr_impl;                // (the sources call these from their extern "C" entry points)
