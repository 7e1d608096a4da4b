// agr_exchange.cu — the multi-GPU exchange: NCCL loaded at run time, agr_comm_*, K4 around K1 / K2, agr_*_sharded and its test-only stages.
#include <dlfcn.h>
#include "agr_engine.h"

// ------------------------------------------------------------------------------------------ K4 exchange
struct nccl_api {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static nccl_api g_nccl;
static int nccl_load() {
    if (g_nccl.lib) return 0;
    void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return fail(AGR_ECOMM, std::string("dlopen libnccl.so.2: ") + dlerror());
#define SYM(field, name) *(void**)(&g_nccl.field) = dlsym(lib, name); if (!g_nccl.field) return fail(AGR_ECOMM, "libnccl.so.2 lacks " name)
    SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommDestroy, "ncclCommDestroy");
    SYM(Send, "ncclSend"); SYM(Recv, "ncclRecv"); SYM(GroupStart, "ncclGroupStart"); SYM(GroupEnd, "ncclGroupEnd");
    SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
    g_nccl.lib = lib;
    return 0;
}
#define NK(call) do { ncclResult_t r_ = (call); if (r_ != ncclSuccess) return fail(AGR_ECOMM, std::string(#call) + ": " + g_nccl.GetErrorString(r_)); } while (0)

namespace agr_impl __attribute__((visibility("hidden"))) {
void comm_destroy(agr_handle* h) { if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm); }   // (agr_destroy)
}  // namespace agr_impl
extern "C" {
int agr_comm_unique_id(uint8_t out[128]) {
    if (!out) return fail(AGR_EINVAL, "NULL argument");
    TRY(nccl_load());
    ncclUniqueId id;
    NK(g_nccl.GetUniqueId(&id));
    memcpy(out, id.internal, 128);
    return 0;
}

// Everything agr_comm_init does besides the communicator: this shard's rank (minted ids carry it) and the exchange's scratch
static int exchange_setup(agr_handle* h, int rank, int world) {
    h->rank = rank; h->world = world;
    h->d.shard_id = (uint32_t)rank;
    if (h->d_k4cnt) return 0;                      // scratch of an earlier call (agr_debug_world may run more than once)
    const size_t mb = h->cfg.max_batch;
    TRY(dev_alloc(h, &h->d_stage, mb * sizeof(agr_outcome), false));   // outcomes before binning (records are binned in their slab rows)
    TRY(dev_alloc(h, &h->d_send, mb * AGR_REC, false));
    TRY(dev_alloc(h, &h->d_owner, mb, false));
    h->d.xowner = h->d_owner;                      // K1 tells the rows K4 shipped away by it (AGR_CFGI_HOLES)
    TRY(dev_alloc(h, &h->d_perm, mb, false));
    h->k4_nwarps = (uint32_t)std::min<size_t>((size_t)h->sm_count * 32, std::max<size_t>(1, (mb + 1023) / 1024));
    TRY(dev_alloc(h, &h->d_k4matrix, (size_t)h->k4_nwarps * 32, false));
    TRY(dev_alloc(h, &h->d_k4cnt, (size_t)4 * 40, true));
    TRY(dev_alloc(h, &h->d_xverd, 2 * mb, false));
    TRY(dev_alloc(h, &h->d_vback, mb, false));
    TRY(dev_alloc(h, &h->d_vout, mb, false));
    // K2 over local + received outcomes: scratch for 2 * max_batch ops
    TRY(dev_alloc(h, &h->d_outs, 2 * mb, false));
    TRY(k2_scratch_alloc(h, 2 * mb));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

int agr_comm_init(agr_handle* h, const uint8_t id[128], int rank, int world) {
    if (!h || !id) return fail(AGR_EINVAL, "NULL argument");
    if (world < 1 || world > 32 || rank < 0 || rank >= world) return fail(AGR_EINVAL, "bad rank / world (1..32 shards)");
    TRY(nccl_load());
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    ncclUniqueId uid; memcpy(uid.internal, id, 128);
    NK(g_nccl.CommInitRank(&h->comm, world, uid, rank));
    return exchange_setup(h, rank, world);
}

// The first half of the exchanges, in three stages: find every item's owner (K4 count + scan: exchange_count), swap the per-peer
// counts with one grouped send/recv (exchange_swap_counts), and lay out the owner-major send offsets and the source-major receive
// offsets (exchange_layout).  `d_items` are the items on the device: the staging buffer (outcomes), or the slab rows the batch was
// DMA'd into (records, in-place mode).
static uint32_t* k4_gtotal(agr_handle* h) { return h->d_k4cnt; }
static uint32_t* k4_goff(agr_handle* h) { return h->d_k4cnt + 40; }
static uint32_t* k4_rcnt(agr_handle* h) { return h->d_k4cnt + 80; }
static int exchange_count(agr_handle* h, uint8_t* d_items, uint32_t item_bytes, uint32_t agent_off, uint32_t n, bool inplace, exchange_plan& x) {
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    x.G = (uint32_t)h->world; x.me = (uint32_t)h->rank;
    agr_k4_params& p = x.p;
    p.items = d_items; p.inplace = inplace ? 1u : 0u;
    p.item_bytes = item_bytes; p.agent_off = agent_off; p.n = n; p.G = x.G; p.me = x.me;
    // every warp takes a run of per_warp items (a multiple of 32); at most k4_nwarps warps (32 per SM)
    uint32_t per = (n + h->k4_nwarps - 1) / std::max<uint32_t>(1, h->k4_nwarps);
    per = std::max<uint32_t>(32, (per + 31) & ~31u);
    p.per_warp = per; p.nwarps = std::max<uint32_t>(1, (n + per - 1) / per);
    p.matrix = h->d_k4matrix; p.gtotal = k4_gtotal(h); p.goff = k4_goff(h); p.owner = h->d_owner; p.perm = h->d_perm;
    agr_launch_k4_count(p, h->stream);
    h->k4_launches += 2;
    CK(cudaGetLastError());
    return 0;
}
static int exchange_swap_counts(agr_handle* h, const exchange_plan& x) {
    NK(g_nccl.GroupStart());
    for (uint32_t q = 0; q < x.G; ++q) {
        NK(g_nccl.Send(k4_gtotal(h) + q, 1, ncclUint32, (int)q, h->comm, h->stream));
        NK(g_nccl.Recv(k4_rcnt(h) + q, 1, ncclUint32, (int)q, h->comm, h->stream));
    }
    NK(g_nccl.GroupEnd());
    return 0;
}
static int exchange_layout(agr_handle* h, exchange_plan& x) {
    const bool inplace = x.p.inplace != 0u;
    const uint32_t n = x.p.n;
    cudaStream_t st = h->stream;
    // the one host round trip of the exchange: ncclSend / ncclRecv take their element counts from the host, and the rows for
    // the records that arrive have to be reserved
    uint32_t* hc = h->h_small;                       // [0..31] send counts, [32..63] receive counts
    CK(cudaMemcpyAsync(hc, k4_gtotal(h), x.G * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hc + 32, k4_rcnt(h), x.G * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    x.soff[0] = 0; x.roff[0] = 0;
    for (uint32_t q = 0; q < x.G; ++q) {
        x.scnt[q] = hc[q]; x.rcnt[q] = (q == x.me) ? 0 : hc[32 + q];
        // in-place mode: the send buffer holds the peers' segments only
        x.soff[q + 1] = x.soff[q] + ((inplace && q == x.me) ? 0u : x.scnt[q]); x.roff[q + 1] = x.roff[q] + x.rcnt[q];
    }
    x.n_local = x.scnt[x.me]; x.n_recv = x.roff[x.G];
    x.recv_res_base = inplace ? n : x.n_local;
    if ((inplace ? n : x.n_local) + x.n_recv > 2 * h->cfg.max_batch) return fail(AGR_ENOSPC, "received more items than 2 * max_batch");
    return 0;
}
static int exchange_begin(agr_handle* h, uint8_t* d_items, uint32_t item_bytes, uint32_t agent_off, uint32_t n, bool inplace, exchange_plan& x) {
    if (!h->comm) return fail(AGR_ECOMM, "agr_comm_init has not been called on this handle");
    TRY(exchange_count(h, d_items, item_bytes, agent_off, n, inplace, x));
    TRY(exchange_swap_counts(h, x));
    return exchange_layout(h, x);
}
// the all-to-all itself: peer segments of `send` to their owners, landing at recv_base in source-rank order
static int exchange_payload(agr_handle* h, const exchange_plan& x, const uint8_t* send, uint8_t* recv_base, size_t item_bytes) {
    NK(g_nccl.GroupStart());
    for (uint32_t q = 0; q < x.G; ++q) {
        if (q == x.me) continue;
        if (x.scnt[q]) NK(g_nccl.Send(send + (size_t)x.soff[q] * item_bytes, (size_t)x.scnt[q] * item_bytes, ncclUint8, (int)q, h->comm, h->stream));
        if (x.rcnt[q]) NK(g_nccl.Recv(recv_base + (size_t)x.roff[q] * item_bytes, (size_t)x.rcnt[q] * item_bytes, ncclUint8, (int)q, h->comm, h->stream));
    }
    NK(g_nccl.GroupEnd());
    return 0;
}
static int exchange_unpermute(agr_handle* h, const exchange_plan& x, const uint8_t* res_all, const uint8_t* back, uint8_t* out_dev, uint32_t res_bytes) {
    if (x.p.n) {
        agr_launch_k4_unpermute(x.p, res_all, back, out_dev, res_bytes, h->stream);
        h->k4_launches += 1;
        CK(cudaGetLastError());
    }
    return 0;
}
// results of the received items back to where they came from (owner-major at the reporter), then the caller's order
static int exchange_results(agr_handle* h, const exchange_plan& x, const uint8_t* res_all /*own items first, then received*/, uint8_t* back,
                            uint8_t* out_dev, uint32_t res_bytes) {
    NK(g_nccl.GroupStart());
    for (uint32_t q = 0; q < x.G; ++q) {
        if (q == x.me) continue;
        if (x.rcnt[q]) NK(g_nccl.Send(res_all + (size_t)(x.recv_res_base + x.roff[q]) * res_bytes, (size_t)x.rcnt[q] * res_bytes, ncclUint8, (int)q, h->comm, h->stream));
        if (x.scnt[q]) NK(g_nccl.Recv(back + (size_t)x.soff[q] * res_bytes, (size_t)x.scnt[q] * res_bytes, ncclUint8, (int)q, h->comm, h->stream));
    }
    NK(g_nccl.GroupEnd());
    return exchange_unpermute(h, x, res_all, back, out_dev, res_bytes);
}
static void exchange_fill_info(const exchange_plan& x, uint32_t n, uint64_t first, uint64_t recv_first, agr_exchange_info* info) {
    if (!info) return;
    memset(info, 0, sizeof *info);
    info->world = x.G; info->rank = x.me; info->n_local = x.n_local; info->n_sent = n - x.n_local; info->n_received = x.n_recv;
    info->first_rid = first; info->recv_first_rid = recv_first;
    for (uint32_t q = 0; q < x.G; ++q) { info->sent_to[q] = (q == x.me) ? 0 : x.scnt[q]; info->received_from[q] = x.rcnt[q]; }
}

// The exchange over a batch that already lies in slab rows [first, first + n) (DMA'd there by agr_ingest_sharded, or filled on
// the device).  Records of this shard's agents never move: K4 only copies the records owned by a PEER into the send buffer and
// K1 skips their rows; received records land in rows reserved behind the batch, straight from the all-to-all.
// Its stages: K4 count + scan over the rows, then (after the counts are known) sharded_rows_local, the all-to-all of the records,
// K1 over the received rows, the all-to-all of their verdicts, and sharded_rows_finish.  agr_debug_exchange_begin / _end run the
// same stages with the test in place of the two all-to-alls.
// Variable-length engines: the batch's rows own 512-byte slots of the byte ring, and records cross shards in that fixed form (a
// cross-shard record is a replay re-injection: only its header decides it).  K4 bins the slots exactly as it bins slab rows, and
// K1v decides them (decide_run_locked).  The batch's slots must lie back to back: a row range across a skip of the byte ring is
// refused.
static int exchange_run(agr_handle* h, uint64_t first, uint32_t n, slot_run* run) {
    *run = slot_run{first, n, 0};
    if (!(h->cfg.flags & AGR_CFG_VARLEN) || n == 0) return 0;
    std::vector<slot_run> runs;
    TRY(row_runs(h, first, n, runs));
    if (runs.size() != 1)
        return fail(AGR_EINVAL, "the rows' 512-byte slots are not back to back (the byte ring skipped to its start between two "
                                "reservations): exchange each reservation on its own");
    *run = runs[0];
    return 0;
}
// rows for the records that arrive, the peers' records packed for shipping, K1 over the batch's own rows (the rows of the records
// K4 packed are holes: K1 skips them by K4's owner array, AGR_CFGI_HOLES) — runs while the all-to-all moves the peers' records
static int sharded_rows_local(agr_handle* h, const slot_run& own, exchange_plan& x, slot_run* recv) {
    const uint32_t n = x.p.n;
    *recv = slot_run{h->rows_used, 0, 0};
    if (x.n_recv) TRY(reserve_run_locked(h, x.n_recv, false, recv));
    const uint32_t n_remote = n - x.n_local;
    x.p.local_dst = nullptr; x.p.send_dst = h->d_send;
    if (n_remote) { agr_launch_k4_scatter(x.p, h->stream); h->k4_launches += 1; CK(cudaGetLastError()); }
    if (n) {
        const uint32_t keep = h->d.cfg_flags;
        if (n_remote) h->d.cfg_flags |= AGR_CFGI_HOLES;
        const int rc = decide_run_locked(h, own, h->d_xverd);
        h->d.cfg_flags = keep;
        TRY(rc);
    }
    return 0;
}
// the verdicts in the caller's order (d_vout, after exchange_unpermute) to the host
static int sharded_rows_finish(agr_handle* h, const exchange_plan& x, uint64_t first, uint64_t first2, agr_verdict* out, agr_exchange_info* info) {
    const uint32_t n = x.p.n;
    if (n && out) TRY(d2h_staged(h, out, h->d_vout, (size_t)n * sizeof(agr_verdict), h->h_verdicts));
    else CK(cudaStreamSynchronize(h->stream));
    exchange_fill_info(x, n, first, first2, info);
    return 0;
}
static int sharded_rows_locked(agr_handle* h, const slot_run& own, agr_verdict* out, agr_exchange_info* info) {
    const uint32_t n = own.n;
    exchange_plan x;
    TRY(exchange_begin(h, run_ptr(h, own), AGR_REC, AGR_OFF_AGENT_ID, n, true, x));
    slot_run recv;
    TRY(sharded_rows_local(h, own, x, &recv));
    // the all-to-all: every peer segment to its owner, landing directly in the owner's slab rows (slots)
    TRY(exchange_payload(h, x, h->d_send, run_ptr(h, recv), AGR_REC));
    // K1 at the owner over the received rows (own host's records first, then peers by rank: the merge order)
    if (x.n_recv) TRY(decide_run_locked(h, recv, h->d_xverd + n));
    // verdicts back to where the records came from, restored to the caller's order
    TRY(exchange_results(h, x, (const uint8_t*)h->d_xverd, (uint8_t*)h->d_vback, (uint8_t*)h->d_vout, sizeof(agr_verdict)));
    return sharded_rows_finish(h, x, own.first, recv.first, out, info);
}

int agr_ingest_sharded(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, agr_exchange_info* info) {
    if (!h || (n && !recs)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->comm) return fail(AGR_ECOMM, "agr_comm_init has not been called on this handle");
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    slot_run own{h->rows_used, 0, 0};
    if (n) {
        TRY(reserve_run_locked(h, n, false, &own));
        // the batch goes STRAIGHT into its slab rows (slots), on the copy stream
        TRY(grow_events(h->chunk_ev, 2));
        CK(cudaEventRecord(h->chunk_ev[0], h->stream));
        CK(cudaStreamWaitEvent(h->copy_stream, h->chunk_ev[0], 0));
        int bk = 0;
        TRY(upload_rows(h, run_ptr(h, own), (const uint8_t*)recs, (size_t)n * AGR_REC, is_pinned(recs), bk));
        CK(cudaEventRecord(h->chunk_ev[1], h->copy_stream));
        CK(cudaStreamWaitEvent(h->stream, h->chunk_ev[1], 0));
    }
    return sharded_rows_locked(h, own, out, info);
}
// The same over rows the caller reserved (agr_reserve_rows) and filled on the device: the exchange with the batch resident in HBM.
int agr_ingest_sharded_rows(agr_handle* h, uint64_t first_rid, uint32_t n, agr_verdict* out, agr_exchange_info* info) {
    if (!h) return fail(AGR_EINVAL, "NULL handle");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->comm) return fail(AGR_ECOMM, "agr_comm_init has not been called on this handle");
    if (first_rid + n > h->rows_used) return fail(AGR_EINVAL, "rows not reserved");
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    slot_run own;
    TRY(exchange_run(h, first_rid, n, &own));
    if (!h->resv.empty()) resv_remove(h, first_rid, first_rid + n);
    return sharded_rows_locked(h, own, out, info);
}

int agr_complete_sharded(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results, agr_exchange_info* info) {
    if (!h || (n && !outs)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    exchange_plan x;
    if (!h->comm) return fail(AGR_ECOMM, "agr_comm_init has not been called on this handle");
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    if (n) CK(cudaMemcpyAsync(h->d_stage, outs, (size_t)n * sizeof(agr_outcome), cudaMemcpyHostToDevice, h->stream));
    TRY(exchange_begin(h, h->d_stage, sizeof(agr_outcome), 16, n, false, x));
    const uint32_t total = x.n_local + x.n_recv;
    // pack: own outcomes straight into the K2 input array, peer segments into the send buffer
    x.p.local_dst = (uint8_t*)h->d_outs; x.p.send_dst = h->d_send;
    if (n) { agr_launch_k4_scatter(x.p, h->stream); h->k4_launches += 1; CK(cudaGetLastError()); }
    TRY(exchange_payload(h, x, h->d_send, (uint8_t*)(h->d_outs + x.n_local), sizeof(agr_outcome)));
    // K2 at the owner over local + received outcomes (own host first, then peers by rank)
    if (total) {
        sync_window(h);
        agr_launch_k2(h->d, h->d_outs, h->k2, total, h->stream);
        h->k2_launches += 3;
        CK(cudaGetLastError());
    }
    TRY(exchange_results(h, x, (const uint8_t*)h->k2.results, (uint8_t*)h->d_vback, (uint8_t*)h->d_vout, 4));
    if (n && results) TRY(d2h_staged(h, results, h->d_vout, (size_t)n * 4, h->h_results));
    else CK(cudaStreamSynchronize(h->stream));
    exchange_fill_info(x, n, 0, 0, info);
    return 0;
}

// ------------------------------------------------------------------ test-only stages of the exchange (no communicator)
int agr_debug_world(agr_handle* h, int rank, int world) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    if (world < 1 || world > 32 || rank < 0 || rank >= world) return fail(AGR_EINVAL, "bad rank / world (1..32 shards)");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (h->comm) return fail(AGR_EINVAL, "the handle has a communicator (agr_comm_init)");
    if (h->xdbg_open) return fail(AGR_EINVAL, "an agr_debug_exchange_begin is waiting for its agr_debug_exchange_end");
    return exchange_setup(h, rank, world);
}

namespace {
struct dbg_dev_buf {                     // device scratch of one agr_debug_k4 call
    void* p = nullptr;
    ~dbg_dev_buf() { if (p) cudaFree(p); }
};
}
int agr_debug_k4(agr_handle* h, const void* items, uint32_t n, uint32_t item_bytes, uint32_t agent_off, int inplace,
                 const void* local_res, const void* remote_res, uint32_t res_bytes, uint8_t* owner, uint32_t* perm, uint32_t* gtotal,
                 uint32_t* goff, void* send_out, void* local_out, void* items_out, void* res_out) {
    if (!h || (n && (!items || !local_res || !remote_res || !owner || !perm || !send_out || !local_out || !items_out || !res_out)) || !gtotal || !goff)
        return fail(AGR_EINVAL, "NULL argument");
    if (item_bytes < 48 || item_bytes > AGR_REC || item_bytes % 16 || agent_off % 16 || agent_off + 32 > item_bytes)
        return fail(AGR_EINVAL, "items are 48..512 B, a multiple of 16, with the 32 B agent id 16 B aligned inside");
    if (res_bytes != 4 && res_bytes != 8) return fail(AGR_EINVAL, "results are 4 or 8 B");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->d_k4cnt) return fail(AGR_ECOMM, "neither agr_comm_init nor agr_debug_world has been called on this handle");
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    const size_t ib = (size_t)std::max<uint32_t>(n, 1) * item_bytes, rb = (size_t)std::max<uint32_t>(n, 1) * res_bytes;
    dbg_dev_buf d_items, d_local, d_lres, d_rres, d_out;
    CK(cudaMalloc(&d_items.p, ib)); CK(cudaMalloc(&d_local.p, ib));
    CK(cudaMalloc(&d_lres.p, rb)); CK(cudaMalloc(&d_rres.p, rb)); CK(cudaMalloc(&d_out.p, rb));
    cudaStream_t st = h->stream;
    CK(cudaMemsetAsync(d_local.p, 0, ib, st));
    CK(cudaMemsetAsync(h->d_send, 0, ib, st));
    CK(cudaMemsetAsync(d_out.p, 0, rb, st));
    if (n) {
        CK(cudaMemcpyAsync(d_items.p, items, (size_t)n * item_bytes, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_lres.p, local_res, (size_t)n * res_bytes, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_rres.p, remote_res, (size_t)n * res_bytes, cudaMemcpyHostToDevice, st));
    }
    exchange_plan x;
    TRY(exchange_count(h, (uint8_t*)d_items.p, item_bytes, agent_off, n, inplace != 0, x));
    CK(cudaMemsetAsync(k4_rcnt(h), 0, 32 * sizeof(uint32_t), st));        // nothing received
    TRY(exchange_layout(h, x));
    x.p.local_dst = (uint8_t*)d_local.p; x.p.send_dst = h->d_send;
    agr_launch_k4_scatter(x.p, st); h->k4_launches += 1;
    CK(cudaGetLastError());
    TRY(exchange_unpermute(h, x, (const uint8_t*)d_lres.p, (const uint8_t*)d_rres.p, (uint8_t*)d_out.p, res_bytes));
    CK(cudaMemcpyAsync(gtotal, k4_gtotal(h), x.G * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(goff, k4_goff(h), (x.G + 1) * 4, cudaMemcpyDeviceToHost, st));
    if (n) {
        CK(cudaMemcpyAsync(owner, h->d_owner, n, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(perm, h->d_perm, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(send_out, h->d_send, (size_t)n * item_bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(local_out, d_local.p, (size_t)n * item_bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(items_out, d_items.p, (size_t)n * item_bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(res_out, d_out.p, (size_t)n * res_bytes, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    return 0;
}

int agr_debug_exchange_begin(agr_handle* h, uint64_t first_rid, uint32_t n, agr_record* send_out, agr_exchange_info* info) {
    if (!h || (n && !send_out)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->d_k4cnt || h->comm) return fail(AGR_EINVAL, "agr_debug_world has not been called on this handle");
    if (h->xdbg_open) return fail(AGR_EINVAL, "an agr_debug_exchange_begin is waiting for its agr_debug_exchange_end");
    if (first_rid + n > h->rows_used) return fail(AGR_EINVAL, "rows not reserved");
    slot_run own;
    TRY(exchange_run(h, first_rid, n, &own));
    if (!h->resv.empty()) resv_remove(h, first_rid, first_rid + n);
    exchange_plan& x = h->xdbg;
    x = exchange_plan{};
    TRY(exchange_count(h, run_ptr(h, own), AGR_REC, AGR_OFF_AGENT_ID, n, true, x));
    CK(cudaMemsetAsync(k4_rcnt(h), 0, 32 * sizeof(uint32_t), h->stream));   // the peers' records arrive through agr_ingest_rows instead
    TRY(exchange_layout(h, x));
    slot_run recv;
    TRY(sharded_rows_local(h, own, x, &recv));
    const uint32_t n_sent = n - x.n_local;
    if (n_sent) CK(cudaMemcpyAsync(send_out, h->d_send, (size_t)n_sent * AGR_REC, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    exchange_fill_info(x, n, first_rid, recv.first, info);
    h->xdbg_first = first_rid; h->xdbg_n = n; h->xdbg_open = true;
    return 0;
}

int agr_debug_exchange_end(agr_handle* h, const agr_verdict* back, agr_verdict* out) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->xdbg_open) return fail(AGR_EINVAL, "no agr_debug_exchange_begin to end");
    const exchange_plan& x = h->xdbg;
    const uint32_t n = h->xdbg_n, n_sent = n - x.n_local;
    if ((n_sent && !back) || (n && !out)) return fail(AGR_EINVAL, "NULL argument");
    h->xdbg_open = false;
    if (n_sent) CK(cudaMemcpyAsync(h->d_vback, back, (size_t)n_sent * sizeof(agr_verdict), cudaMemcpyHostToDevice, h->stream));
    TRY(exchange_unpermute(h, x, (const uint8_t*)h->d_xverd, (const uint8_t*)h->d_vback, (uint8_t*)h->d_vout, sizeof(agr_verdict)));
    return sharded_rows_finish(h, x, h->xdbg_first, h->rows_used, out, nullptr);
}
}  // extern "C"
