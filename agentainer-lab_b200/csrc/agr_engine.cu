// agr_engine.cu — host side of the engine and the C-ABI of include/agentainer_gpu.h: the core (the other parts: agr_engine.h).
//
// One agr_handle == one GPU shard: HBM slab + SoA state + dedupe index + logs + agent-table mirror, one stream.
// Calls are linearised by the handle mutex; the order in which calls take it is the event order the state
// machine sees (the reference's serialisation point is the single-threaded Redis server).
// There is NO CPU fallback: every state transition happens in the kernels of agr_kernels.cu.
#include <sys/random.h>
#include "agr_engine.h"

static_assert(sizeof(agr_record) == 512, "agr_record must be 512 B");
static_assert(sizeof(agr_outcome) == 64, "agr_outcome must be 64 B");
static_assert(sizeof(agr_dispatch) == 32, "agr_dispatch must be 32 B");
static_assert(sizeof(agr_verdict) == 8, "agr_verdict must be 8 B");
static_assert(sizeof(agr_slot) == 32, "agr_slot must be 32 B");
static_assert(sizeof(agr_agent_key) == 48, "agr_agent_key must be 48 B");
static_assert(sizeof(agr_dop) == 32, "agr_dop must be 32 B");
static_assert(sizeof(agr_k2op) == 16, "agr_k2op must be 16 B");

namespace agr_impl __attribute__((visibility("hidden"))) {
thread_local std::string g_err;
// K2 scratch for up to n outcomes per batch
int k2_scratch_alloc(agr_handle* h, size_t n) {
    TRY(dev_alloc(h, &h->k2.ops, n, false));
    TRY(dev_alloc(h, &h->k2.nxt, n, false));
    TRY(dev_alloc(h, &h->k2.eff, n + 8, false));
    TRY(dev_alloc(h, &h->k2.results, n, false));
    // word 0 = {ticket, overflow}, then one look-back word per tile: agr_launch_k2 clears the prefix a batch uses
    unsigned long long* words = nullptr;
    TRY(dev_alloc(h, &words, (size_t)agr_k2_tiles((uint32_t)n) + 2, true));
    h->k2.ticket = (uint32_t*)words;
    h->k2.overflow = h->k2.ticket + 1;
    h->k2.tiles = words + 1;
    return 0;
}

// pageable -> pinned staging copy.  One core moves ~13 GB/s, a quarter of what the link takes; big pieces are split over a
// few short-lived threads (the pinned path, agr_host_alloc, needs none of this).
static void par_memcpy(void* dst, const void* src, size_t bytes) {
    const size_t min_slice = (size_t)4 << 20;
    unsigned nt = (unsigned)std::min<size_t>(4, bytes / min_slice);
    if (nt <= 1) { memcpy(dst, src, bytes); return; }
    const size_t slice = ((bytes / nt) + 63) & ~(size_t)63;
    std::vector<std::thread> th;
    for (unsigned t = 1; t < nt; ++t) {
        const size_t o = (size_t)t * slice;
        if (o >= bytes) break;
        th.emplace_back([=] { memcpy((uint8_t*)dst + o, (const uint8_t*)src + o, std::min(slice, bytes - o)); });
    }
    memcpy(dst, src, std::min(slice, bytes));
    for (auto& x : th) x.join();
}
bool is_pinned(const void* p) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) == cudaSuccess) return attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    return false;
}
// host -> device on the compute stream: pinned caller memory is copied in place, pageable memory through the pinned stage
static int h2d_staged(agr_handle* h, void* dst, const void* src, size_t bytes, void* stage) {
    if (!is_pinned(src)) { memcpy(stage, src, bytes); src = stage; }
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
    return 0;
}
// device -> host on the compute stream through the pinned stage, then into dst (NULL: the bytes stay in the stage)
int d2h_staged(agr_handle* h, void* dst, const void* dsrc, size_t bytes, void* stage) {
    CK(cudaMemcpyAsync(stage, dsrc, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (dst) memcpy(dst, stage, bytes);
    return 0;
}
// caller records -> slab rows on the copy stream: pinned (or registered) memory is DMA'd in place, pageable memory goes
// through the two pinned bounce buffers; bk is the bounce buffer to use next, carried from one call to the next
int upload_rows(agr_handle* h, uint8_t* dst, const uint8_t* src, size_t bytes, bool src_pinned, int& bk) {
    if (src_pinned) {
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->copy_stream));
        return 0;
    }
    for (size_t o = 0; o < bytes;) {
        const size_t piece = std::min(h->bounce_bytes, bytes - o);
        CK(cudaEventSynchronize(h->bounce_ev[bk]));
        par_memcpy(h->bounce[bk], src + o, piece);
        CK(cudaMemcpyAsync(dst + o, h->bounce[bk], piece, cudaMemcpyHostToDevice, h->copy_stream));
        CK(cudaEventRecord(h->bounce_ev[bk], h->copy_stream));
        o += piece; bk ^= 1;
    }
    return 0;
}
// the lengths of the completed and failed logs
int read_log_lens(agr_handle* h, unsigned long long lens[2]) {
    CK(cudaMemcpyAsync(lens, h->d.log_len, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
// the last counter slot, used as an 8-byte scratch count by the maintenance kernels: zeroed before the launch, read after
static unsigned long long* count_slot(agr_handle* h) { return (unsigned long long*)(h->d.ctr + C_NCTR - 1); }
static int read_count(agr_handle* h, unsigned long long* v) {
    CK(cudaMemcpyAsync(v, count_slot(h), 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
// grows an event pool to k events (without timing); the ones it has are kept
int grow_events(std::vector<cudaEvent_t>& ev, size_t k) {
    while (ev.size() < k) { cudaEvent_t e; CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); ev.push_back(e); }
    return 0;
}
// every chunk's time bounds "unknown" (after a restore, or a jump of the arrival counter): the next agr_expire recomputes them
int chunk_bounds_unknown(agr_handle* h) {
    CK(cudaMemsetAsync(h->d.cmin, 0, (size_t)(h->cfg.slab_rows / AGR_CHUNK_ROWS + 2) * 8, h->stream));
    return 0;
}

static uint64_t next_pow2(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

// Hash-id ring: the dedupe index rebuilt from the window's rows that still hold a record (ST_STORED in the state word), over
// the window's one or two physical runs.  Open addressing has no cheap delete, so a release rebuilds the index instead of
// taking the released rows' ids out; a restore of a ring rebuilds it the same way, so that the restored index is the one a
// release leaves (an expired row's id is in neither).
int ring_reindex_locked(agr_handle* h) {
    CK(cudaMemsetAsync(h->d.table, 0, (size_t)(h->d.table_mask + 1) * sizeof(agr_slot), h->stream));
    h->d.idx_base = h->tail;                                              // row words of the rebuilt index are relative to the tail
    const uint64_t R = h->cfg.slab_rows, live = h->rows_used - h->tail, p0 = h->tail % R;
    const uint64_t n0 = std::min<uint64_t>(live, R - p0);
    agr_launch_reindex_range(h->d, (uint32_t)p0, (uint32_t)n0, h->stream);
    if (live > n0) agr_launch_reindex_range(h->d, 0, (uint32_t)(live - n0), h->stream);
    CK(cudaGetLastError());
    h->k1_launches += 2;
    return 0;
}
}  // namespace agr_impl

extern "C" {

uint32_t agr_abi_version(void) { return AGR_ABI_VERSION; }
const char* agr_last_error(void) { return g_err.c_str(); }
const char* agr_strerror(int code) {
    switch (code) {
        case AGR_OK: return "ok";
        case AGR_EINVAL: return "invalid argument";
        case AGR_ENODEV: return "no usable CUDA device";
        case AGR_ENOMEM: return "out of memory";
        case AGR_ENOSPC: return "capacity exhausted";
        case AGR_ENOTFOUND: return "not found";
        case AGR_ECUDA: return "CUDA error";
        case AGR_ECAP: return "output array too small";
        case AGR_ECOMM: return "multi-GPU exchange error";
        default: return "unknown error";
    }
}

void* agr_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { g_err = "cudaHostAlloc failed"; return nullptr; }
    return p;
}
void agr_host_free(void* p) { if (p) cudaFreeHost(p); }

static int create_impl(const agr_config* cfg_in, agr_handle* h) {
    agr_config c{};
    if (cfg_in) c = *cfg_in;
    if (c.flags == 0) c.flags = AGR_CFG_PERSISTENCE;
    if (c.slab_rows == 0) c.slab_rows = 1ull << 20;
    if (c.slab_rows >= 0x7fffffffull) return fail(AGR_EINVAL, "slab_rows must be < 2^31");
    if ((c.flags & AGR_CFG_DELTA_SNAPSHOT) && !(c.flags & AGR_CFG_ONLINE_SNAPSHOT))
        return fail(AGR_EINVAL, "AGR_CFG_DELTA_SNAPSHOT needs AGR_CFG_ONLINE_SNAPSHOT (the delta is taken by the online cut)");
    const bool mint = (c.flags & AGR_CFG_MINT_IDS) != 0;
    if (mint) c.table_slots = 64;                               // no dedupe index in this mode (a stub keeps pointers valid)
    if (c.table_slots == 0) c.table_slots = next_pow2(c.slab_rows * 2);
    if (c.table_slots & (c.table_slots - 1)) return fail(AGR_EINVAL, "table_slots must be a power of two");
    if (!mint && c.table_slots < c.slab_rows + c.slab_rows / 4) return fail(AGR_EINVAL, "table_slots must be >= 1.25 * slab_rows");
    if (c.table_slots > (1ull << 32)) return fail(AGR_EINVAL, "table_slots must be <= 2^32");
    if (c.max_agents == 0) c.max_agents = 4096;
    if (c.max_agents >= RT_SLOT_NONE) return fail(AGR_EINVAL, "max_agents must be < 2^23 - 1");
    if (c.max_batch == 0) c.max_batch = 1u << 20;
    if (c.flags & AGR_CFG_RING) {
        if (c.max_batch > c.slab_rows / 2) c.max_batch = (uint32_t)(c.slab_rows / 2);
        if (c.max_batch == 0) return fail(AGR_EINVAL, "AGR_CFG_RING: slab_rows too small");
    }
    if (c.log_entries == 0) c.log_entries = c.slab_rows * 3;   // a replayed request pushes twice (Q7), plus once per earlier retry
    if (c.k1_variant & ~(0x20u | 0xff0000u))
        return fail(AGR_EINVAL, "k1_variant: only bit 0x20 (K1v form) and bits 16..23 (timing stride) are defined; the A/B alternates of the fixed-stride K1 were retired");
    if ((c.flags & AGR_CFG_VARLEN) && c.vslab_bytes == 0) c.vslab_bytes = 1024ull * c.slab_rows;
    if (c.max_record_bytes != 0) {
        if (!(c.flags & AGR_CFG_VARLEN)) return fail(AGR_EINVAL, "max_record_bytes needs AGR_CFG_VARLEN (fixed-stride records are 512 B)");
        if ((c.max_record_bytes & 15u) || c.max_record_bytes < AGR_VAR_MAX_RECORD || c.max_record_bytes > AGR_VAR_MAX_RECORD_LIMIT)
            return fail(AGR_EINVAL, "max_record_bytes must be a multiple of 16 in [8192, 2^26], or 0 for 8192");
        if (c.max_record_bytes > c.vslab_bytes / 2)
            return fail(AGR_EINVAL, "max_record_bytes must be at most vslab_bytes / 2 (" + std::to_string(c.vslab_bytes / 2) + "): a batch never takes more than half the byte slab");
    }
    if (c.max_record_bytes == 0) c.max_record_bytes = AGR_VAR_MAX_RECORD;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(AGR_ENODEV, "no CUDA device visible (this library has no CPU fallback)"); }
    int dev = c.device;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) return fail(AGR_ENODEV, "cudaGetDevice failed"); }
    if (dev >= ndev) return fail(AGR_ENODEV, "device ordinal out of range");
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    // arch-specific sm_90a code loads on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0) return fail(AGR_ENODEV, std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major * 10 + prop.minor) + "; this library is built for sm_90a only");
    CK(cudaSetDevice(dev));
    h->device = dev;
    h->sm_count = prop.multiProcessorCount;
    h->cfg = c;
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->d2h_stream, cudaStreamNonBlocking));
    agr_dev& d = h->d;
    const bool varlen = (c.flags & AGR_CFG_VARLEN) != 0;
    if (varlen) {
        h->vcap = c.vslab_bytes;
        TRY(dev_alloc(h, &d.slab, (size_t)c.vslab_bytes + AGR_VT_MAXREC, false));
        TRY(dev_alloc(h, &d.voff, c.slab_rows, true));
        TRY(dev_alloc(h, &d.vlen, c.slab_rows, true));
        TRY(dev_alloc(h, &h->d_voffsets, (size_t)c.max_batch + 1, false));
        TRY(host_alloc(h, &h->h_voffsets, (size_t)c.max_batch + 1));
        // (a blob holds at most max_batch records and, with long records, at most vslab_bytes)
        const size_t tile_bytes = (size_t)c.max_batch * AGR_VT_MAXREC + (c.max_record_bytes > AGR_VAR_MAX_RECORD ? c.vslab_bytes : 0);
        TRY(dev_alloc(h, &h->d_tile_first, tile_bytes / AGR_VT_TILE + 8, false));
        // runs of 512-byte slots: up to 2 x max_batch (the exchange decides own + received rows), offsets below 2^32
        h->slot_off_max = (uint32_t)std::min<uint64_t>(2ull * c.max_batch, (0xffffffffull / AGR_REC) - 1);
        TRY(dev_alloc(h, &h->d_slot_off, (size_t)h->slot_off_max + 1, false));
        agr_launch_slot_offsets(h->d_slot_off, h->slot_off_max, h->stream);
        CK(cudaGetLastError());
    } else {
        TRY(dev_alloc(h, &d.slab, (size_t)c.slab_rows * AGR_REC, false));
    }
    TRY(dev_alloc(h, &d.state, c.slab_rows + 4, true));        // (+4: k3_mark reads these two four rows at a time)
    TRY(dev_alloc(h, &d.route, c.slab_rows + 4, true));
    TRY(dev_alloc(h, &d.aux, c.slab_rows, true));
    TRY(dev_alloc(h, &d.cksum, c.slab_rows, true));
    TRY(dev_alloc(h, &d.table, c.table_slots, true));
    d.table_mask = c.table_slots - 1;
    uint32_t acap = (uint32_t)next_pow2((uint64_t)c.max_agents * 2);
    TRY(dev_alloc(h, &d.akeys, acap, true));
    d.amask = acap - 1;
    h->akeys_host.assign(acap, agr_agent_key{});
    TRY(dev_alloc(h, &d.astatus, c.max_agents, true));
    TRY(dev_alloc(h, &d.ctr, (size_t)C_NCTR, true));
    TRY(dev_alloc(h, &d.completed_log, c.log_entries, false));
    TRY(dev_alloc(h, &d.failed_log, c.log_entries, false));
    TRY(dev_alloc(h, &d.log_len, (size_t)2, true));
    d.log_cap = c.log_entries;
    TRY(dev_alloc(h, &d.marks, (size_t)(2 * (size_t)c.max_batch / 32 + 8), true));   // (2 x max_batch: the exchange runs K1 over own + received rows)
    TRY(dev_alloc(h, &d.dupfix, (size_t)8, true));
    h->dupfix_base = d.dupfix; d.dupfix_next = d.dupfix + 4;
    if (c.flags & AGR_CFG_RING) {
        TRY(dev_alloc(h, &h->d_log_scratch, c.log_entries, false));
        TRY(dev_alloc(h, &h->d_lc_chunks, (size_t)(c.log_entries / 1024 + 4), false));
    }
    if (c.resp_bytes == 0) c.resp_bytes = 64ull * c.slab_rows;
    h->cfg.resp_bytes = c.resp_bytes; h->resp_cap = c.resp_bytes;
    TRY(dev_alloc(h, &h->d_resp, (size_t)c.resp_bytes, false));
    TRY(dev_alloc(h, &h->d_resp_off, c.slab_rows, true));
    TRY(dev_alloc(h, &h->d_resp_len, c.slab_rows, true));
    TRY(dev_alloc(h, &h->d_resp_hlen, c.slab_rows, true));
    TRY(dev_alloc(h, &h->d_err_off, c.slab_rows, true));
    TRY(dev_alloc(h, &h->d_err_len, c.slab_rows, true));
    TRY(dev_alloc(h, &d.ptime, c.slab_rows, true));
    TRY(dev_alloc(h, &d.mtime, c.slab_rows, true));
    TRY(dev_alloc(h, &d.head, c.slab_rows, true));
    TRY(dev_alloc(h, &d.cmin, (size_t)(c.slab_rows / AGR_CHUNK_ROWS + 2), false));
    CK(cudaMemsetAsync(d.cmin, 0xff, (size_t)(c.slab_rows / AGR_CHUNK_ROWS + 2) * 8, h->stream));   // ~0: no stored row in any chunk yet
    // the key of the id permutation: drawn from the OS CSPRNG unless the caller brings one (a restore passes the snapshot's),
    // so that ids of one engine instance never resolve in another and cannot be guessed (the reference mints uuid.New())
    d.id_secret = c.id_secret;
    while (d.id_secret == 0) {
        if (getrandom(&d.id_secret, sizeof d.id_secret, 0) != (ssize_t)sizeof d.id_secret) return fail(AGR_EINVAL, "getrandom failed: pass agr_config.id_secret");
    }
    h->cfg.id_secret = d.id_secret;
    d.shard_id = 0; d.id_gen = 1; d.tail = 0; d.head_l = 0; d.ring_rows = 0; d.tail_phys = 0; d.idx_base = 0;
    if (!varlen && agr_k1_tma_make_map(d.slab, c.slab_rows, h->tmap) != 0)
        return fail(AGR_ECUDA, "cuTensorMapEncodeTiled failed for the slab");
    d.cfg_flags = c.flags & 0xffffu;
    // staging
    h->bounce_bytes = std::min<size_t>((size_t)c.max_batch * AGR_REC, (size_t)32 << 20);
    for (int k = 0; k < 2; ++k) {
        TRY(host_alloc(h, &h->bounce[k], h->bounce_bytes));
        CK(cudaEventCreateWithFlags(&h->bounce_ev[k], cudaEventDisableTiming));
    }
    TRY(host_alloc(h, &h->h_verdicts, c.max_batch));
    TRY(dev_alloc(h, &h->d_verdicts, c.max_batch, false));
    TRY(dev_alloc(h, &h->d_ids, (size_t)c.max_batch * 16, false));
    TRY(host_alloc(h, &h->h_ids, (size_t)c.max_batch * 16));
    TRY(host_alloc(h, &h->h_ops, (size_t)16));
    TRY(host_alloc(h, &h->h_outs, c.max_batch));
    TRY(dev_alloc(h, &h->d_outs, c.max_batch, false));
    TRY(host_alloc(h, &h->h_results, c.max_batch));
    TRY(host_alloc(h, &h->h_small, (size_t)64));
    TRY(dev_alloc(h, &h->d_reclaim, (size_t)64, true));
    TRY(dev_alloc(h, &h->d_reclaim_scratch, (size_t)2, false));
    { const uint32_t init[2] = {0xffffffffu, 0u}; CK(cudaMemcpyAsync(h->d_reclaim_scratch, init, 8, cudaMemcpyHostToDevice, h->stream)); CK(cudaStreamSynchronize(h->stream)); }
    TRY(host_alloc(h, &h->h_reclaim, (size_t)64));
    TRY(dev_alloc(h, &h->d_ops, (size_t)16, false));
    TRY(dev_alloc(h, &h->d_hrid, (size_t)16, false));
    TRY(host_alloc(h, &h->h_k2flag, (size_t)4));
    TRY(k2_scratch_alloc(h, c.max_batch));
    TRY(dev_alloc(h, &h->d_gtotal, ((size_t)c.max_agents + 8) * 66, false));   // gtotal + 64 segment partials per group
    TRY(dev_alloc(h, &h->d_goff, (size_t)c.max_agents + 2, false));
    TRY(dev_alloc(h, &h->d_min_inq, (size_t)1, false));
    if (c.flags & AGR_CFG_ONLINE_SNAPSHOT) TRY(snap_online_create(h));
    CK(cudaStreamSynchronize(h->stream));
    if (c.flags & AGR_CFG_COMBINE) TRY(svc_create(h));
    return 0;
}

int agr_create(const agr_config* cfg, agr_handle** out) {
    if (!out) return fail(AGR_EINVAL, "out is NULL");
    *out = nullptr;
    agr_handle* h = new agr_handle();
    int r = create_impl(cfg, h);
    if (r < 0) { std::string keep = g_err; agr_destroy(h); g_err = keep; return r; }
    *out = h;
    return 0;
}

void agr_destroy(agr_handle* h) {
    if (!h) return;
    svc_destroy(h);
    if (h->stream) { cudaSetDevice(h->device); cudaStreamSynchronize(h->stream); }
    for (void* p : h->dev_allocs) cudaFree(p);
    for (void* p : h->host_allocs) cudaFreeHost(p);
    for (int k = 0; k < 2; ++k) if (h->bounce_ev[k]) cudaEventDestroy(h->bounce_ev[k]);
    for (auto e : h->tev) cudaEventDestroy(e);
    for (auto e : h->op_ev) if (e) cudaEventDestroy(e);
    for (auto e : h->snap_ev) if (e) cudaEventDestroy(e);
    if (h->snap_stream) cudaStreamDestroy(h->snap_stream);
    for (auto e : h->chunk_ev) cudaEventDestroy(e);
    if (h->reclaim_ev) cudaEventDestroy(h->reclaim_ev);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->d2h_stream) cudaStreamDestroy(h->d2h_stream);
    for (auto e : h->out_ev) cudaEventDestroy(e);
    comm_destroy(h);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

}  // extern "C"
namespace agr_impl __attribute__((visibility("hidden"))) {
// ------------------------------------------------------------------------------------------ agent table
static int agent_find(agr_handle* h, const char* id) {
    auto it = h->slot_of.find(std::string(id));
    return it == h->slot_of.end() ? -1 : (int)it->second;
}

// status lives in two places on the device: astatus[slot] (K3 reads it by slot) and the key entry (K1 reads it with
// the key in one access); both copies are stream-ordered before the next kernel
int push_agent_status(agr_handle* h, uint32_t slot, uint8_t status) {
    const uint32_t idx = h->akey_index[slot];
    h->akeys_host[idx].status = status;
    CK(cudaMemcpyAsync(h->d.astatus + slot, &status, 1, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(&h->d.akeys[idx].status, &h->akeys_host[idx].status, 4, cudaMemcpyHostToDevice, h->stream));
    return 0;
}

// ---- slot reuse.  A slot is held while a row of the live window [tail, rows_used) records a decision for it (verdict code != 0 and
// the route word's slot): AGR_V_NOT_FOUND rows (RT_SLOT_NONE), exchange holes, rows skipped at the end of a lap, released rows and
// reserved rows not decided yet hold nothing.  Once every slot has been handed out, a new agent id takes the lowest removed slot
// that is not held.  The table changes only under the handle lock, between calls, and a slot changes hands only when no live row
// carries it, so within a call agent ids and slots stay one to one (K1's in-batch replay rule relies on it; DESIGN.md section 4).

// the held-slot scan: removed slots up (one bit each), k_slot_refs over the window's physical ranges, held slots back
static int scan_held_locked(agr_handle* h, std::vector<uint32_t>& held) {
    const uint32_t nslots = (uint32_t)h->agent_names.size(), words = (nslots + 31) / 32;
    std::vector<uint32_t> cand(words, 0u);
    bool any = false;
    for (uint32_t s = 0; s < nslots; ++s)
        if (h->agent_status[s] == AG_STATUS_REMOVED) { cand[s >> 5] |= 1u << (s & 31); any = true; }
    held.assign(words, 0u);
    if (!any) return 0;
    if (!h->d_slot_cand) {
        const size_t cap = ((size_t)h->cfg.max_agents + 31) / 32;
        TRY(dev_alloc(h, &h->d_slot_cand, cap, false));
        TRY(dev_alloc(h, &h->d_slot_held, cap, false));
    }
    CK(cudaMemcpyAsync(h->d_slot_cand, cand.data(), (size_t)words * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->d_slot_held, 0, (size_t)words * 4, h->stream));
    const uint64_t live = h->rows_used - h->tail, p0 = phys_row(h, h->tail);
    const uint64_t n0 = is_ring(h) ? std::min<uint64_t>(live, h->cfg.slab_rows - p0) : live;   // a ring's window wraps at most once
    agr_launch_slot_refs(h->d.route, p0, n0, h->d_slot_cand, nslots, h->d_slot_held, h->sm_count, h->stream);
    if (live > n0) agr_launch_slot_refs(h->d.route, 0, live - n0, h->d_slot_cand, nslots, h->d_slot_held, h->sm_count, h->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(held.data(), h->d_slot_held, (size_t)words * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

// The slot for an agent id the table does not hold: the next never-used one, else the lowest removed slot that is not held, else
// AGR_ENOSPC.  One scan lists every removed, unheld slot (lowest last).  Each entry stays removed and unheld (a removed agent gets
// no new rows, and a revived one leaves the list), so the lowest entry is the answer unless a lower slot has been freed since the
// scan: that takes an event that can free a slot (agent_gen: a drop, a release of rows, a restore) and a removed slot below that
// entry.  Only then is the window scanned again, so a table full of live agents refuses without a scan and a run of
// registrations after one release shares one scan.
static int take_slot_locked(agr_handle* h, uint32_t* slot) {
    if (h->agent_names.size() < h->cfg.max_agents) { *slot = (uint32_t)h->agent_names.size(); return 0; }
    if (h->free_gen != h->agent_gen) {
        const uint32_t head = h->free_slots.empty() ? (uint32_t)h->agent_names.size() : h->free_slots.back();
        bool lower = false;
        for (uint32_t s = 0; s < head && !lower; ++s) lower = h->agent_status[s] == AG_STATUS_REMOVED;
        if (lower) {
            std::vector<uint32_t> held;
            TRY(scan_held_locked(h, held));
            h->free_gen = h->agent_gen;
            h->free_slots.clear();
            for (uint32_t s = (uint32_t)h->agent_names.size(); s-- > 0;)
                if (h->agent_status[s] == AG_STATUS_REMOVED && !((held[s >> 5] >> (s & 31)) & 1u)) h->free_slots.push_back(s);
        }
    }
    if (!h->free_slots.empty()) {
        *slot = h->free_slots.back();
        h->free_slots.pop_back();
        return 0;
    }
    // (every removed slot is held now: the list is empty, and a slot removed since the last scan would have caused one)
    const size_t held = std::count(h->agent_status.begin(), h->agent_status.end(), (uint8_t)AG_STATUS_REMOVED);
    return fail(AGR_ENOSPC, "agent table full (" + std::to_string(held) +
                                " removed agents' slots are still held by live rows: agr_expire + agr_reclaim release them)");
}

// puts the key of slot (its name and status set) into the key table; upload: status first, then the key that makes the slot
// reachable, both stream-ordered before the next kernel
static int insert_key_locked(agr_handle* h, uint32_t slot, bool upload) {
    agr_agent_key key{};
    agt_pack(h->agent_names[slot].c_str(), key.w);
    key.slot = slot;
    key.status = h->agent_status[slot];
    const uint32_t idx = agt_insert(h->akeys_host.data(), h->d.amask, key);
    h->akey_index[slot] = idx;
    if (upload) {
        CK(cudaMemcpyAsync(h->d.astatus + slot, &h->agent_status[slot], 1, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d.akeys + idx, &h->akeys_host[idx], sizeof key, cudaMemcpyHostToDevice, h->stream));
    }
    return 0;
}

// Forgets the agent of a handed-out slot: its name leaves the map and its key leaves the key table by backward shift (the entries
// of the probe cluster that moved go up with it).  The slot stays handed out; agent_bind_locked gives it its next agent.
int agent_forget_locked(agr_handle* h, uint32_t slot, bool upload) {
    const uint32_t idx = h->akey_index[slot], mask = h->d.amask;
    auto it = h->slot_of.find(h->agent_names[slot]);
    if (it != h->slot_of.end() && it->second == slot) h->slot_of.erase(it);
    const uint32_t count = agt_delete(h->akeys_host.data(), mask, idx);
    for (uint32_t k = 0; k < count; ++k) {
        const uint32_t j = (idx + k) & mask;
        if (!agt_empty(h->akeys_host[j])) h->akey_index[h->akeys_host[j].slot] = j;
    }
    if (upload) {
        const uint32_t n0 = std::min(count, mask + 1 - idx);
        CK(cudaMemcpyAsync(h->d.akeys + idx, &h->akeys_host[idx], (size_t)n0 * sizeof(agr_agent_key), cudaMemcpyHostToDevice, h->stream));
        if (count > n0) CK(cudaMemcpyAsync(h->d.akeys, &h->akeys_host[0], (size_t)(count - n0) * sizeof(agr_agent_key), cudaMemcpyHostToDevice, h->stream));
    }
    return 0;
}
// registers agent_id (not in the table) on a handed-out slot whose agent was forgotten
int agent_bind_locked(agr_handle* h, uint32_t slot, const char* agent_id, uint8_t status, bool upload) {
    h->agent_names[slot] = agent_id;
    h->agent_status[slot] = status;
    h->slot_of[std::string(agent_id)] = slot;
    return insert_key_locked(h, slot, upload);
}

// core of agr_set_agent_state; `upload` = push the change to the device now (the bulk call uploads the tables once instead)
int set_agent_state_locked(agr_handle* h, const char* agent_id, uint8_t status, bool upload) {
    size_t len = strnlen(agent_id, AGR_AGENT_ID_BYTES);
    if (len == 0 || len >= AGR_AGENT_ID_BYTES) return fail(AGR_EINVAL, "agent id must be 1..31 bytes");
    if (status > AGR_AGENT_FAILED) return fail(AGR_EINVAL, "bad agent status");
    int slot = agent_find(h, agent_id);
    if (slot < 0) {
        uint32_t s = 0;
        TRY(take_slot_locked(h, &s));
        if (s < h->agent_names.size()) {
            TRY(agent_forget_locked(h, s, upload));
            TRY(agent_bind_locked(h, s, agent_id, status, upload));
            return (int)s;
        }
        h->agent_names.emplace_back(agent_id);
        h->agent_status.push_back(status);
        h->akey_index.push_back(0);
        h->slot_of.emplace(std::string(agent_id), s);
        TRY(insert_key_locked(h, s, upload));
        return (int)s;
    }
    if (h->agent_status[slot] == AG_STATUS_REMOVED) {
        // revived on its slot: off the free list, which a later drop does not put it back on (its rows from now on may hold it)
        auto it = std::find(h->free_slots.begin(), h->free_slots.end(), (uint32_t)slot);
        if (it != h->free_slots.end()) h->free_slots.erase(it);
    }
    h->agent_status[slot] = status;
    if (upload) TRY(push_agent_status(h, (uint32_t)slot, status));
    else h->akeys_host[h->akey_index[slot]].status = status;
    return slot;
}
}  // namespace agr_impl
extern "C" {
int agr_set_agent_state(agr_handle* h, const char* agent_id, uint8_t status) {
    if (!h || !agent_id) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return set_agent_state_locked(h, agent_id, status, true);
}
int agr_set_agent_states(agr_handle* h, const char (*agent_ids)[AGR_AGENT_ID_BYTES], const uint8_t* statuses, uint32_t n, int32_t* slots) {
    if (!h || (n && (!agent_ids || !statuses))) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    const bool bulk = n > 16;                       // many writes: update the host mirror, upload both tables once
    int rc = 0;
    for (uint32_t i = 0; i < n; ++i) {
        char id[AGR_AGENT_ID_BYTES];
        memcpy(id, agent_ids[i], AGR_AGENT_ID_BYTES); id[AGR_AGENT_ID_BYTES - 1] = 0;
        const int s = set_agent_state_locked(h, id, statuses[i], !bulk);
        if (slots) slots[i] = s;
        if (s < 0 && rc == 0) rc = s;               // keep going: one bad entry must not hide the other status writes
    }
    if (bulk && !h->agent_status.empty()) {
        CK(cudaMemcpyAsync(h->d.astatus, h->agent_status.data(), h->agent_status.size(), cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d.akeys, h->akeys_host.data(), h->akeys_host.size() * sizeof(agr_agent_key), cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));       // the host vectors may be reallocated by the next call
    }
    return rc;
}

int agr_agent_slot(agr_handle* h, const char* agent_id) {
    if (!h || !agent_id) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    int s = agent_find(h, agent_id);
    if (s < 0 || h->agent_status[s] == AG_STATUS_REMOVED) return fail(AGR_ENOTFOUND, "agent not found");
    return s;
}

int agr_drop_agent(agr_handle* h, const char* agent_id) {
    if (!h || !agent_id) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    int slot = agent_find(h, agent_id);
    if (slot < 0) return fail(AGR_ENOTFOUND, "agent not found");
    h->agent_status[slot] = AG_STATUS_REMOVED;
    TRY(push_agent_status(h, (uint32_t)slot, AG_STATUS_REMOVED));                          // DEL agent:{id} (agent.go:344)
    h->agent_gen++;                                                                        // the slot may be free once its rows are gone
    unsigned long long lens[2];
    TRY(read_log_lens(h, lens));
    agr_launch_drop_agent(h->d, (uint32_t)slot, rows_span(h), std::max(lens[0], lens[1]), h->stream);
    h->k3_launches += 2;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

}  // extern "C"
namespace agr_impl __attribute__((visibility("hidden"))) {
// Rows handed out by agr_reserve_rows hold no record until agr_ingest_rows has run over them.  The replay scan, the pending
// views and agr_reclaim stop at the first such row: otherwise a scan that finds "nothing pending" above its low-water mark
// would move the mark past rows that K1 fills in later, and those requests would never be replayed.
uint64_t ingested_bound(const agr_handle* h) {
    uint64_t b = h->rows_used;
    for (const auto& r : h->resv) b = std::min(b, r.first);
    return b;
}
void resv_remove(agr_handle* h, uint64_t first, uint64_t end) {
    std::vector<resv_run> keep;
    for (const auto& r : h->resv) {
        if (r.end <= first || r.first >= end) { keep.push_back(r); continue; }
        if (r.first < first) keep.push_back(resv_run{r.first, first, r.vbase});
        if (r.end > end) keep.push_back(resv_run{end, r.end, r.vbase + (end - r.first) * AGR_REC});
    }
    h->resv.swap(keep);
}
// b continues a: the rows follow on (logically and physically: K1 numbers a run's rows from its first physical row) and so do
// the slots (variable-length engines; a slot run never wraps the byte ring)
static bool runs_adjoin(const agr_handle* h, uint64_t a_first, uint64_t a_end, uint64_t a_vbase, uint64_t b_first, uint64_t b_vbase) {
    if (a_end != b_first) return false;
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) return true;
    return phys_row(h, a_first) + (a_end - a_first) == phys_row(h, b_first) && a_vbase + (a_end - a_first) * AGR_REC == b_vbase;
}
// Variable-length engines: rows [first, first + n) as the runs whose slots lie back to back, in row order.  Every row must be
// reserved and not decided yet (the resv list keeps the slots of those rows only).  Fixed-stride engines: the range itself.
int row_runs(agr_handle* h, uint64_t first, uint32_t n, std::vector<slot_run>& out) {
    out.clear();
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) {
        if (n) out.push_back(slot_run{first, n, 0});
        return 0;
    }
    for (uint64_t at = first, end = first + n; at < end;) {
        const resv_run* r = nullptr;
        for (const auto& q : h->resv) if (q.first <= at && at < q.end) { r = &q; break; }
        if (!r) return fail(AGR_EINVAL, "variable-length engine: row " + std::to_string(at) + " is not a reserved row that awaits its record "
                                        "(agr_reserve_rows hands out rows with 512-byte slots; a decided row has none)");
        const uint64_t k = std::min(end, r->end) - at;
        const slot_run s{at, (uint32_t)k, r->vbase + (at - r->first) * AGR_REC};
        slot_run* b = out.empty() ? nullptr : &out.back();
        if (b && runs_adjoin(h, b->first, b->first + b->n, b->vbase, s.first, s.vbase)) b->n += s.n;
        else out.push_back(s);
        at += k;
    }
    return 0;
}
// The cursor rule of the three rings (slab rows, variable-length record bytes, response bytes), in logical units: a piece of
// `need` units never wraps — if it does not fit before the end of the lap, the rest of the lap is skipped (*pad units) — and
// it fits when everything from the tail to the end of the piece stays within one lap of `cap`.
static bool ring_fits(uint64_t used, uint64_t tail, uint64_t cap, uint64_t need, uint64_t* pad) {
    const uint64_t at = used % cap;
    *pad = (at + need > cap) ? cap - at : 0;
    return used + *pad + need - tail <= cap;
}
// While an online snapshot is being written, its file streams the rows and bytes of the cut's window from where they lie, so
// a reservation may not lap into that window even once agr_reclaim has released it: the ring's tail is min(tail, pin).
static const char* const PINNED_FULL = "ring full up to the window of the snapshot being written (agr_snapshot with AGR_CFG_ONLINE_SNAPSHOT): "
                                       "its rows and bytes are reused once the file is written";
static inline bool ring_fits_pinned(const agr_handle* h, uint64_t used, uint64_t tail, uint64_t pin, uint64_t cap, uint64_t need) {
    uint64_t pad = 0;
    return !h->pinned || ring_fits(used, std::min(tail, pin), cap, need, &pad);
}

// ------------------------------------------------------------------------------------------ K1
int reserve_rows_locked(agr_handle* h, uint32_t n, uint64_t* first) {
    if (!is_ring(h)) {
        if (h->rows_used + n > h->cfg.slab_rows) return fail(AGR_ENOSPC, "slab full");
        *first = h->rows_used;
        h->rows_used += n;
        sync_window(h);
        return 0;
    }
    // ring: rows skipped at the end of a lap stay "no record" (released rows are zeroed), at most max_batch rows per lap
    uint64_t pad = 0;
    if (!ring_fits(h->rows_used, h->tail, h->cfg.slab_rows, n, &pad)) return fail(AGR_ENOSPC, "slab full: agr_expire + agr_reclaim release rows at the tail");
    if (!ring_fits_pinned(h, h->rows_used, h->tail, h->pin_tail, h->cfg.slab_rows, n)) return fail(AGR_ENOSPC, std::string("slab ") + PINNED_FULL);
    if (h->rows_used + pad + n > AGR_ROW_LIMIT) return fail(AGR_ENOSPC, "row ids exhausted: a shard hands out 2^52 rows (minted ids stay unique that long)");
    h->rows_used += pad;
    *first = h->rows_used;
    h->rows_used += n;
    sync_window(h);
    return 0;
}

// The byte ring of a variable-length engine takes `bytes` as one piece (a blob of agr_ingest_var, or the slots of one row
// reservation): vbytes_fit checks (*vpad = the bytes skipped at the end of the lap), vbytes_take hands the piece out and
// returns its physical offset.  The rows are reserved in between, so that a refused call leaves both rings as they were.
int vbytes_fit(const agr_handle* h, uint64_t bytes, uint64_t* vpad) {
    *vpad = 0;
    if (!is_ring(h)) {
        if (h->vused + bytes > h->vcap) return fail(AGR_ENOSPC, "byte slab full");
        return 0;
    }
    if (bytes > h->vcap / 2) return fail(AGR_EINVAL, "batch larger than half the byte slab");
    if (!ring_fits(h->vused, h->vtail, h->vcap, bytes, vpad)) return fail(AGR_ENOSPC, "byte slab full: agr_expire + agr_reclaim release bytes at the tail");
    if (!ring_fits_pinned(h, h->vused, h->vtail, h->pin_vtail, h->vcap, bytes)) return fail(AGR_ENOSPC, std::string("byte slab ") + PINNED_FULL);
    return 0;
}
uint64_t vbytes_take(agr_handle* h, uint64_t bytes, uint64_t vpad) {
    h->vused += vpad;
    const uint64_t base = is_ring(h) ? h->vused % h->vcap : h->vused;
    h->vused += bytes;
    return base;
}

// n rows and, on a variable-length engine, their n consecutive 512-byte slots.  listed: the rows wait for agr_fill_rows /
// agr_ingest_rows (agr_reserve_rows), so they go on the resv list; the exchange's own reservations are decided in the same
// call and are not listed.
int reserve_run_locked(agr_handle* h, uint32_t n, bool listed, slot_run* run) {
    const bool varlen = (h->cfg.flags & AGR_CFG_VARLEN) != 0 && n;
    uint64_t vpad = 0;
    if (varlen) TRY(vbytes_fit(h, (uint64_t)n * AGR_REC, &vpad));
    TRY(reserve_rows_locked(h, n, &run->first));
    run->n = n;
    run->vbase = varlen ? vbytes_take(h, (uint64_t)n * AGR_REC, vpad) : 0;
    if (listed && n) {
        resv_run* b = h->resv.empty() ? nullptr : &h->resv.back();
        if (b && runs_adjoin(h, b->first, b->end, b->vbase, run->first, run->vbase)) b->end += n;   // back-to-back reservations merge
        else h->resv.push_back(resv_run{run->first, run->first + n, run->vbase});
    }
    return 0;
}

// every K1 batch gets a zeroed set of per-batch words; the set it does not use is cleared by its k1_post for the next one
static inline void flip_batch_words(agr_handle* h) {
    h->batch_phase ^= 1u;
    h->d.dupfix = h->dupfix_base + 4u * h->batch_phase;
    h->d.dupfix_next = h->dupfix_base + 4u * (h->batch_phase ^ 1u);
}

// AGR_CFG_TIMING: the next event pair of the ring agr_kernel_time reads (one pair per timed K1 launch)
static int claim_k1_events(agr_handle* h, cudaEvent_t* e0, cudaEvent_t* e1) {
    if (h->tev.empty()) {
        h->tev.resize(2 * AGR_TIMING_RING);
        for (auto& e : h->tev) CK(cudaEventCreate(&e));
    }
    const uint64_t k = h->tev_next++ % AGR_TIMING_RING;
    *e0 = h->tev[2 * k]; *e1 = h->tev[2 * k + 1];
    return 0;
}
// AGR_CFG_TIMING: events around the last launch group g (0 = K2, 1 = K3 select, 2 = K5 encode, 3 = snapshot cut, 4 = the
// relocation of a restore) that agr_op_time reads
int op_time_begin(agr_handle* h, int g) {
    if (!(h->cfg.flags & AGR_CFG_TIMING)) return 0;
    for (auto& e : h->op_ev) if (!e) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(h->op_ev[2 * g], h->stream));
    return 0;
}
int op_time_end(agr_handle* h, int g) {
    if (!(h->cfg.flags & AGR_CFG_TIMING)) return 0;
    CK(cudaEventRecord(h->op_ev[2 * g + 1], h->stream));
    h->op_timed[g] = true;
    return 0;
}

int launch_k1_locked(agr_handle* h, uint64_t first, uint32_t n, agr_verdict* d_out, uint8_t* d_ids) {
    sync_window(h);
    flip_batch_words(h);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    // AGR_CFG_TIMING: events around the K1 kernel of every launch, or of every k-th one (k1_variant bits 16..23): an event record
    // is a stream operation of its own between two kernels, and two of them per step cost a back-to-back loop a few microseconds
    const uint32_t tstride = std::max<uint32_t>(1u, (h->cfg.k1_variant >> 16) & 0xffu);
    if ((h->cfg.flags & AGR_CFG_TIMING) && (h->timing_calls++ % tstride) == 0) TRY(claim_k1_events(h, &e0, &e1));
    h->k1_launches += agr_launch_k1(h->d, (uint32_t)phys_row(h, first), first, n, h->tmap, h->sm_count, h->stream, e0, e1, d_out, d_ids);
    CK(cudaGetLastError());
    return 0;
}

// K1v and its post pass over rows [first, first + n) of a variable-length engine, whose records lie at physical byte `base` of
// the byte slab, record i at d_off[i] .. d_off[i + 1] from there (`bytes` in all)
// (nlong: the batch's long records, listed in h->long_list as agr_launch_k1v_long takes it)
static int launch_k1v_locked(agr_handle* h, uint64_t first, uint32_t n, uint64_t base, const uint32_t* d_off, uint64_t bytes,
                             agr_verdict* d_out, uint8_t* d_ids, uint32_t nlong = 0) {
    cudaStream_t st = h->stream;
    sync_window(h);
    flip_batch_words(h);
    const size_t words = 2 * (size_t)nlong + 1;                   // long records: the list, then two sums per record
    if (nlong) {
        if (words + 2 * (size_t)nlong > h->d_long.cap) TRY(regrow(h, h->d_long, std::max<size_t>(words + 2 * (size_t)nlong, 1024)));
        CK(cudaMemcpyAsync(h->d_long.p, h->long_list.data(), words * 4, cudaMemcpyHostToDevice, st));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (h->cfg.flags & AGR_CFG_TIMING) {
        TRY(claim_k1_events(h, &e0, &e1));
        CK(cudaEventRecord(e0, st));
    }
    CK(agr_launch_k1_var(h->d, h->d.slab + base, d_off, n, bytes, h->d_tile_first, (uint32_t)phys_row(h, first), base, h->sm_count, st, h->cfg.k1_variant));
    if (nlong) {
        CK(agr_launch_k1v_long(h->d, h->d.slab + base, d_off, h->d_long.p, nlong, h->long_list[2 * nlong], h->d_long.p + words,
                               (uint32_t)phys_row(h, first), st));
        h->k1_launches += 2;
    }
    if (e1) CK(cudaEventRecord(e1, st));
    agr_launch_k1_post(h->d, (uint32_t)phys_row(h, first), n, h->sm_count, st, d_out, d_ids);
    h->k1_launches += 3;
    CK(cudaGetLastError());
    return 0;
}

// K1 over one run: the fixed-stride kernel, or K1v reading the run's 512-byte slots as a blob with offsets 512 i
int decide_run_locked(agr_handle* h, const slot_run& r, agr_verdict* d_out) {
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) return launch_k1_locked(h, r.first, r.n, d_out);
    if (r.n == 0) return 0;
    if (r.n > h->slot_off_max) return fail(AGR_EINVAL, "more slots in one run than K1v's offsets reach");
    return launch_k1v_locked(h, r.first, r.n, r.vbase, h->d_slot_off, (uint64_t)r.n * AGR_REC, d_out, nullptr);
}
}  // namespace agr_impl
extern "C" {

static int ingest_rows_locked(agr_handle* h, uint64_t first, uint32_t n, agr_verdict* out, bool sync) {
    if (first + n > h->rows_used) return fail(AGR_EINVAL, "rows not reserved");
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    if (n == 0) return 0;
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) {
        TRY(launch_k1_locked(h, first, n, out ? h->d_verdicts : nullptr));
    } else {
        // one K1v per run of back-to-back slots: a range across a skip of the byte ring is decided as the reservations on either
        // side of the skip would be on their own
        std::vector<slot_run> runs;
        TRY(row_runs(h, first, n, runs));
        uint32_t done = 0;
        for (const slot_run& r : runs) {
            TRY(decide_run_locked(h, r, out ? h->d_verdicts + done : nullptr));
            done += r.n;
        }
    }
    if (!h->resv.empty()) resv_remove(h, first, first + n);
    if (out) {
        TRY(d2h_staged(h, out, h->d_verdicts, (size_t)n * sizeof(agr_verdict), h->h_verdicts));
    } else if (sync) {
        CK(cudaStreamSynchronize(h->stream));
    }
    return 0;
}

int agr_mint_ids(agr_handle* h, uint64_t first_rid, uint32_t n, uint8_t (*ids)[16]) {
    if (!h || (n && !ids)) return fail(AGR_EINVAL, "NULL argument");
    if (!(h->cfg.flags & AGR_CFG_MINT_IDS)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_MINT_IDS");
    for (uint32_t i = 0; i < n; ++i) {
        unsigned long long lo, hi;
        agr_mint_id(first_rid + i, h->d.shard_id, h->d.id_gen, h->d.id_secret, lo, hi);
        memcpy(ids[i], &lo, 8); memcpy(ids[i] + 8, &hi, 8);
    }
    return 0;
}

int agr_reserve_rows(agr_handle* h, uint32_t n, uint64_t* first_rid) {
    if (!h || !first_rid) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    slot_run r;
    TRY(reserve_run_locked(h, n, true, &r));
    *first_rid = r.first;
    return 0;
}
int agr_fill_rows(agr_handle* h, uint64_t first_rid, const agr_record* recs, uint32_t n) {
    if (!h || (n && !recs)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (first_rid + n > h->rows_used || first_rid < h->tail) return fail(AGR_EINVAL, "rows not reserved");
    if (h->cfg.flags & AGR_CFG_VARLEN) {                         // into the rows' slots of the byte ring
        std::vector<slot_run> runs;
        TRY(row_runs(h, first_rid, n, runs));
        uint32_t done = 0;
        for (const slot_run& r : runs) {
            CK(cudaMemcpyAsync(run_ptr(h, r), recs + done, (size_t)r.n * AGR_REC, cudaMemcpyHostToDevice, h->stream));
            done += r.n;
        }
        CK(cudaStreamSynchronize(h->stream));
        return 0;
    }
    if (n == 0) return 0;
    if (phys_row(h, first_rid) + n > h->cfg.slab_rows) return fail(AGR_EINVAL, "row range wraps");
    CK(cudaMemcpyAsync(h->d.slab + phys_row(h, first_rid) * AGR_REC, recs, (size_t)n * AGR_REC, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
int agr_ingest_rows(agr_handle* h, uint64_t first_rid, uint32_t n, agr_verdict* out) {
    if (!h) return fail(AGR_EINVAL, "NULL handle");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return ingest_rows_locked(h, first_rid, n, out, true);
}
int agr_ingest_rows_async(agr_handle* h, uint64_t first_rid, uint32_t n) {
    if (!h) return fail(AGR_EINVAL, "NULL handle");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return ingest_rows_locked(h, first_rid, n, nullptr, false);
}
int agr_sync(agr_handle* h) {
    if (!h) return fail(AGR_EINVAL, "NULL handle");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
void* agr_stream(agr_handle* h) { return h ? (void*)h->stream : nullptr; }
void* agr_slab_ptr(agr_handle* h, uint64_t rid) {
    if (!h || rid >= h->rows_used || rid < h->tail) return nullptr;
    if (h->cfg.flags & AGR_CFG_VARLEN) {                         // a reserved row that awaits its record: its 512-byte slot
        HLock lk(h);
        for (const auto& r : h->resv)
            if (r.first <= rid && rid < r.end) return (void*)(h->d.slab + r.vbase + (rid - r.first) * AGR_REC);
    }
    return (void*)(h->d.slab + phys_row(h, rid) * AGR_REC);
}

// host -> slab rows -> K1 -> verdicts, pipelined in chunks: the H2D copy of chunk k+1 (copy stream) overlaps K1 and the
// verdict D2H of chunk k (compute stream).  Chunks are consecutive sub-batches in arrival order, so the result is
// identical to one big batch (tests/test_parity_gpu.py::test_result_does_not_depend_on_batching).
// Pinned (or registered) caller memory is DMA'd in place; pageable memory goes through two pinned bounce buffers.
#define AGR_INGEST_CHUNK (1u << 17)   // 128 Ki records = 64 MiB per H2D chunk
int agr_ingest(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint64_t* first_rid) {
    return agr_ingest_ex(h, recs, n, out, nullptr, first_rid);
}

static int ingest_ex_locked(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid);

int agr_ingest_ex(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid) {
    if (!h || (n && !recs)) return fail(AGR_EINVAL, "NULL argument");
    if (h->cfg.flags & AGR_CFG_VARLEN) return fail(AGR_EINVAL, "variable-length engine: use agr_ingest_var");
    if (h->svc && n >= 1 && n <= SVC_MAX_CALL) return svc_ingest(h, recs, n, out, ids, first_rid);
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return ingest_ex_locked(h, recs, n, out, ids, first_rid);
}

static int ingest_ex_locked(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid) {
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    uint64_t first = 0;
    TRY(reserve_rows_locked(h, n, &first));
    if (first_rid) *first_rid = first;
    if (n == 0) return 0;
    const bool src_pinned = is_pinned(recs);
    const bool out_pinned = out && is_pinned(out);
    const bool ids_pinned = ids && is_pinned(ids);
    const uint32_t nchunks = (n + AGR_INGEST_CHUNK - 1) / AGR_INGEST_CHUNK;
    TRY(grow_events(h->chunk_ev, nchunks + 1));
    // the copy stream must not overwrite rows before earlier work on the compute stream is done with the slab
    CK(cudaEventRecord(h->chunk_ev[nchunks], h->stream));
    CK(cudaStreamWaitEvent(h->copy_stream, h->chunk_ev[nchunks], 0));
    int bk = 0;
    for (uint32_t c = 0; c < nchunks; ++c) {
        const uint32_t off = c * AGR_INGEST_CHUNK, cn = std::min(AGR_INGEST_CHUNK, n - off);
        TRY(upload_rows(h, h->d.slab + (phys_row(h, first) + off) * AGR_REC, (const uint8_t*)(recs + off), (size_t)cn * AGR_REC, src_pinned, bk));
        CK(cudaEventRecord(h->chunk_ev[c], h->copy_stream));
        CK(cudaStreamWaitEvent(h->stream, h->chunk_ev[c], 0));
        TRY(launch_k1_locked(h, first + off, cn, out ? h->d_verdicts + off : nullptr, ids ? h->d_ids + (size_t)off * 16 : nullptr));
        if (out || ids) {
            // the chunk's read-backs (8 + 16 B per record) leave on their own stream as soon as its K1 is done
            TRY(grow_events(h->out_ev, c + 1));
            CK(cudaEventRecord(h->out_ev[c], h->stream));
            CK(cudaStreamWaitEvent(h->d2h_stream, h->out_ev[c], 0));
            if (out) CK(cudaMemcpyAsync((out_pinned ? out : h->h_verdicts) + off, h->d_verdicts + off, (size_t)cn * sizeof(agr_verdict), cudaMemcpyDeviceToHost, h->d2h_stream));
            if (ids) CK(cudaMemcpyAsync((ids_pinned ? (uint8_t*)ids : h->h_ids) + (size_t)off * 16, h->d_ids + (size_t)off * 16, (size_t)cn * 16, cudaMemcpyDeviceToHost, h->d2h_stream));
        }
    }
    CK(cudaStreamSynchronize(h->stream));
    if (out || ids) CK(cudaStreamSynchronize(h->d2h_stream));
    if (out && !out_pinned) memcpy(out, h->h_verdicts, (size_t)n * sizeof(agr_verdict));
    if (ids && !ids_pinned) memcpy(ids, h->h_ids, (size_t)n * 16);
    return 0;
}

// ------------------------------------------------------------------------------------------ K2
static int complete_locked(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results, const agr_k2_bytes* bytes = nullptr,
                           bool bytes_dropped = false);
static int complete_ex_locked(agr_handle* h, const agr_outcome* outs, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                              const uint32_t* hdr_lens, int32_t* results);

int agr_complete(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results) {
    if (!h || (n && !outs)) return fail(AGR_EINVAL, "NULL argument");
    if (h->svc && n >= 1 && n <= SVC_MAX_CALL) return svc_complete(h, outs, n, results);
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return complete_locked(h, outs, n, results);
}

int agr_complete_ex(agr_handle* h, const agr_outcome* outs, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                    const uint32_t* hdr_lens, int32_t* results) {
    if (!h || (n && (!outs || !offsets))) return fail(AGR_EINVAL, "NULL argument");
    if (h->svc && n >= 1 && n <= SVC_MAX_CALL) {
        bool fits = true;
        for (uint32_t i = 0; i < n && fits; ++i) fits = offsets[i + 1] >= offsets[i] && offsets[i + 1] - offsets[i] <= AGR_OUT_INLINE_BYTES;
        if (fits) return svc_complete_ex(h, outs, n, bytes, offsets, hdr_lens, results);
    }
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return complete_ex_locked(h, outs, n, bytes, offsets, hdr_lens, results);
}

// bytes (agr_complete_ex): the batch's bytes are staged on the device and have a region of the byte slab; bytes_dropped: they
// have none (the transitions are applied all the same, and the call fails with AGR_ENOSPC)
static int complete_locked(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results, const agr_k2_bytes* bytes,
                           bool bytes_dropped) {
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    if (n == 0) return 0;
    // outcomes go to the device as they are; k2_prepare resolves the agent ids in the device agent table
    TRY(h2d_staged(h, h->d_outs, outs, (size_t)n * sizeof(agr_outcome), h->h_outs));
    sync_window(h);
    TRY(op_time_begin(h, 0));
    agr_launch_k2(h->d, h->d_outs, h->k2, n, h->stream, bytes);
    h->k2_launches += bytes ? 4 : 3;
    CK(cudaGetLastError());
    TRY(op_time_end(h, 0));
    CK(cudaMemcpyAsync(h->h_k2flag, h->k2.overflow, 4, cudaMemcpyDeviceToHost, h->stream));
    if (results) {
        TRY(d2h_staged(h, results, h->k2.results, (size_t)n * 4, h->h_results));
    } else {
        CK(cudaStreamSynchronize(h->stream));
    }
    // the state transitions were applied; list entries beyond the log capacity were dropped (agr_config.log_entries)
    if (bytes_dropped)
        return fail(AGR_ENOSPC, std::string("response byte slab full: the batch's outcomes were applied, none of its response / error bytes "
                                            "were stored (raise agr_config.resp_bytes, or agr_reclaim with AGR_CFG_RING)") +
                                    (*h->h_k2flag ? std::string("; also ") + K2_LOG_FULL : std::string()));
    if (*h->h_k2flag) return fail(AGR_ENOSPC, K2_LOG_FULL);
    return 0;
}

}  // extern "C"
namespace agr_impl __attribute__((visibility("hidden"))) {
// ------------------------------------------------------------------------------------------ K2 with bytes (agr_complete_ex)
// Places need bytes (a multiple of 16) in the response byte slab as one piece; len is the unrounded size the append-only check
// uses.  With the ring a piece never wraps: the rest of the lap is skipped, and agr_reclaim moves resp_tail.
int resp_reserve_locked(agr_handle* h, uint64_t need, uint64_t len, unsigned long long* off) {
    if (!is_ring(h)) {
        if (h->resp_used + len > h->resp_cap) return fail(AGR_ENOSPC, "response slab full");
        *off = h->resp_used;
        h->resp_used += need;
        return 0;
    }
    if (need > h->resp_cap / 2) return fail(AGR_ENOSPC, "response larger than half the response slab");
    uint64_t pad = 0;
    if (!ring_fits(h->resp_used, h->resp_tail, h->resp_cap, need, &pad))
        return fail(AGR_ENOSPC, "response slab full: agr_reclaim releases the bytes of released rows");
    if (!ring_fits_pinned(h, h->resp_used, h->resp_tail, h->pin_resp_tail, h->resp_cap, need)) return fail(AGR_ENOSPC, std::string("response slab ") + PINNED_FULL);
    h->resp_used += pad;
    *off = h->resp_used % h->resp_cap;                           // the rows keep PHYSICAL offsets
    h->resp_used += need;
    return 0;
}

// Checks what agr_complete_ex got; *total = the size of the batch's region (every segment rounded up to 16 B), *max_len = the
// longest segment.
int check_segments(const agr_outcome* outs, uint32_t n, const uint64_t* offsets, const uint32_t* hdr_lens, uint64_t* total,
                   uint64_t* max_len) {
    uint64_t t = 0, m = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (offsets[i + 1] < offsets[i]) return fail(AGR_EINVAL, "offsets must not decrease");
        const uint64_t len = offsets[i + 1] - offsets[i];
        if (len > 0xffffffffull) return fail(AGR_EINVAL, "a segment is longer than 4 GiB");
        if (outs[i].kind == AGR_OUT_RESPONSE) {
            if (hdr_lens && hdr_lens[i] > len) return fail(AGR_EINVAL, "hdr_lens[i] is longer than segment i");
        } else if (outs[i].kind != AGR_OUT_ERROR && len) {
            return fail(AGR_EINVAL, "only AGR_OUT_RESPONSE and AGR_OUT_ERROR outcomes carry bytes");
        }
        t += (len + 15u) & ~15ull;
        m = std::max(m, len);
    }
    *total = t; *max_len = m;
    return 0;
}
}  // namespace agr_impl
extern "C" {

static int complete_ex_locked(agr_handle* h, const agr_outcome* outs, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                              const uint32_t* hdr_lens, int32_t* results) {
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    if (n == 0) return 0;
    uint64_t total = 0, max_len = 0;
    TRY(check_segments(outs, n, offsets, hdr_lens, &total, &max_len));
    const uint64_t nbytes = offsets[n] - offsets[0];
    if (nbytes && !bytes) return fail(AGR_EINVAL, "NULL bytes");
    if (!h->d_boff) {
        const size_t mb = h->cfg.max_batch;
        TRY(host_alloc(h, &h->h_boff, mb + 1)); TRY(dev_alloc(h, &h->d_boff, mb + 1, false));
        TRY(host_alloc(h, &h->h_bdst, mb)); TRY(dev_alloc(h, &h->d_bdst, mb, false));
        TRY(host_alloc(h, &h->h_bhlen, mb)); TRY(dev_alloc(h, &h->d_bhlen, mb, false));
    }
    // the batch's region: all or nothing
    unsigned long long base = 0;
    if (resp_reserve_locked(h, total, total, &base) < 0) return complete_locked(h, outs, n, results, nullptr, true);
    // each segment's place in it, in array order (the host has the offsets: no device round trip)
    uint64_t run = 0;
    for (uint32_t i = 0; i < n; ++i) { h->h_bdst[i] = run; run += (offsets[i + 1] - offsets[i] + 15u) & ~15ull; }
    CK(cudaMemcpyAsync(h->d_bdst, h->h_bdst, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    TRY(h2d_staged(h, h->d_boff, offsets, ((size_t)n + 1) * 8, h->h_boff));
    if (hdr_lens) TRY(h2d_staged(h, h->d_bhlen, hdr_lens, (size_t)n * 4, h->h_bhlen));
    if (nbytes) {
        // (+ 16: warp_copy16 reads whole aligned 16-byte blocks around a segment)
        if (nbytes + 16 > h->d_bsrc.cap) TRY(regrow(h, h->d_bsrc, (size_t)(nbytes + nbytes / 4 + 16)));
        const uint8_t* src = bytes + offsets[0];
        if (!is_pinned(src)) {
            if (nbytes > h->h_bsrc.cap) TRY(regrow(h, h->h_bsrc, (size_t)(nbytes + nbytes / 4), true));
            par_memcpy(h->h_bsrc.p, src, nbytes);
            src = h->h_bsrc.p;
        }
        CK(cudaMemcpyAsync(h->d_bsrc.p, src, nbytes, cudaMemcpyHostToDevice, h->stream));
    }
    agr_k2_bytes b{};
    b.src = h->d_bsrc.p; b.src_off = h->d_boff; b.dst = h->d_bdst; b.hlen = hdr_lens ? h->d_bhlen : nullptr; b.base = base;
    b.slab = h->d_resp; b.resp_off = h->d_resp_off; b.resp_len = h->d_resp_len; b.resp_hlen = h->d_resp_hlen;
    b.err_off = h->d_err_off; b.err_len = h->d_err_len;
    return complete_locked(h, outs, n, results, &b, false);
}

// ------------------------------------------------------------------------------------------ K3
// (each buffer of a group is checked against its own capacity: after a failed regrow of one of them the others keep theirs)
static int ensure_out(agr_handle* h, uint32_t cap) {
    uint32_t ncap = std::max<uint32_t>(cap, 1024);
    if (cap > h->d_out_rid.cap) TRY(regrow(h, h->d_out_rid, ncap));
    if (cap > h->d_out_slot.cap) TRY(regrow(h, h->d_out_slot, ncap));
    return 0;
}
static int ensure_gather(agr_handle* h, size_t bytes) {
    if (bytes > h->d_gather.cap) TRY(regrow(h, h->d_gather, bytes));
    if (bytes > h->h_gather.cap) TRY(regrow(h, h->h_gather, bytes, true));
    return 0;
}
// copies out what the K3 gather makes of rows d_rids[0..n): dispatch entries, records and / or request ids (each skipped when
// NULL), through one device buffer laid out in that order and one device -> host copy
static int gather_rows_locked(agr_handle* h, const uint32_t* d_rids, uint32_t n, agr_dispatch* disp, agr_record* recs, uint8_t (*ids)[16]) {
    const size_t disp_bytes = disp ? (size_t)n * 32 : 0, rec_bytes = recs ? (size_t)n * AGR_REC : 0, id_bytes = ids ? (size_t)n * 16 : 0;
    const size_t bytes = disp_bytes + rec_bytes + id_bytes;
    TRY(ensure_gather(h, bytes));
    uint8_t* g = h->d_gather.p;
    agr_launch_k3_gather(h->d, d_rids, nullptr, n, recs ? g + disp_bytes : nullptr, disp ? g : nullptr, ids ? g + disp_bytes + rec_bytes : nullptr,
                         h->stream);
    h->k3_launches += 1;
    CK(cudaGetLastError());
    TRY(d2h_staged(h, nullptr, g, bytes, h->h_gather.p));
    if (disp) memcpy(disp, h->h_gather.p, disp_bytes);
    if (recs) memcpy(recs, h->h_gather.p + disp_bytes, rec_bytes);
    if (ids) memcpy(ids, h->h_gather.p + disp_bytes + rec_bytes, id_bytes);
    return 0;
}

// runs the stable partition; returns the number selected in *total (may exceed cap: then only counts are valid)
static int select_locked(agr_handle* h, int mode, uint32_t slot, const uint32_t* log, uint64_t lo, uint64_t hi,
                         uint32_t cap, uint32_t* total) {
    *total = 0;
    if (hi <= lo) return 0;
    agr_k3_params p{};
    p.mode = mode; p.slot = slot; p.log = log; p.lo = lo; p.hi = hi; p.lo_real = lo;
    if (mode != K3_LOG_AGENT) p.lo = lo & ~3ull;               // k3_mark reads the row words four rows per lane (16-byte loads)
    p.groups = (mode == K3_TICK) ? std::max<uint32_t>(1, (uint32_t)h->agent_names.size()) : 1;
    uint64_t items = hi - p.lo;
    uint64_t max_warps = std::max<uint64_t>(1, (4u << 20) / p.groups);
    uint64_t want = std::min<uint64_t>((uint64_t)h->sm_count * 128, (items + 1023) / 1024);  // several waves of 8-warp CTAs; the column scan runs over per-CTA rows
    p.nwarps = (uint32_t)std::max<uint64_t>(1, std::min(want, max_warps));
    uint64_t per = (items + p.nwarps - 1) / p.nwarps;
    per = (per + 255) & ~255ull;
    p.per_warp = (uint32_t)per;
    p.nwarps = (uint32_t)((items + per - 1) / per);
    size_t need = (size_t)p.nwarps * p.groups;
    if (need > h->d_matrix.cap) TRY(regrow(h, h->d_matrix, need));
    const size_t need_cta = (size_t)((p.nwarps + 7) / 8) * p.groups;
    if (need_cta > h->d_cta_matrix.cap) TRY(regrow(h, h->d_cta_matrix, need_cta));
    p.cta_matrix = h->d_cta_matrix.p;
    const size_t mask_words = (size_t)p.nwarps * (p.per_warp >> 5);
    if (mask_words > h->d_selmask.cap) TRY(regrow(h, h->d_selmask, mask_words));
    p.selmask = h->d_selmask.p;
    TRY(ensure_out(h, cap));
    p.matrix = h->d_matrix.p; p.gtotal = h->d_gtotal; p.goff = h->d_goff;
    p.out_rid = h->d_out_rid.p; p.out_slot = h->d_out_slot.p; p.cap = cap;
    p.min_inq = (mode == K3_TICK) ? h->d_min_inq : nullptr;
    if (mode == K3_TICK) CK(cudaMemsetAsync(h->d_min_inq, 0xff, 4, h->stream));
    TRY(op_time_begin(h, 1));
    agr_launch_k3_select(h->d, p, h->sm_count, h->stream);
    h->k3_launches += 4;
    CK(cudaGetLastError());
    TRY(op_time_end(h, 1));
    CK(cudaMemcpyAsync(h->h_small, h->d_goff + p.groups, 4, cudaMemcpyDeviceToHost, h->stream));
    if (mode == K3_TICK) CK(cudaMemcpyAsync(h->h_small + 1, h->d_min_inq, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *total = h->h_small[0];
    if (mode == K3_TICK) {
        uint32_t m = h->h_small[1];
        h->scan_lo = (m == AGR_RID_NONE) ? hi : std::max<uint64_t>(h->scan_lo, p.lo + m);
    }
    return 0;
}

int agr_replay_scan(agr_handle* h, agr_dispatch* out, agr_record* recs, uint32_t cap, uint32_t* n) {
    if (!h || !n) return fail(AGR_EINVAL, "NULL argument");
    if ((h->cfg.flags & AGR_CFG_VARLEN) && recs) return fail(AGR_EINVAL, "variable-length engine: use agr_replay_scan_var to gather records");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    *n = 0;
    h->replay_scans++;
    uint32_t total = 0;
    TRY(select_locked(h, K3_TICK, 0, nullptr, h->scan_lo, ingested_bound(h), cap, &total));
    *n = total;
    if (total > cap) return fail(AGR_ECAP, "dispatch array too small");
    h->replay_dispatched += total;
    if (total == 0 || !out) return 0;
    return gather_rows_locked(h, h->d_out_rid.p, total, out, recs, nullptr);
}

int agr_pending(agr_handle* h, const char* agent_id, agr_record* out, uint32_t cap, uint32_t* n) {
    if (!h || !agent_id || !n) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    *n = 0;
    int slot = agent_find(h, agent_id);
    if (slot < 0) return 0;     // LRANGE on a missing key is an empty list
    uint32_t total = 0;
    TRY(select_locked(h, K3_AGENT_PENDING, (uint32_t)slot, nullptr, h->scan_lo, ingested_bound(h), cap, &total));
    *n = total;
    if (total > cap) return fail(AGR_ECAP, "output array too small");
    if (total == 0 || !out) return 0;
    return gather_rows_locked(h, h->d_out_rid.p, total, nullptr, out, nullptr);
}

int agr_list(agr_handle* h, const char* agent_id, int which, uint8_t (*ids)[16], uint32_t cap, uint32_t* n) {
    if (!h || !agent_id || !n) return fail(AGR_EINVAL, "NULL argument");
    if (which < AGR_LIST_PENDING || which > AGR_LIST_FAILED) return fail(AGR_EINVAL, "bad list selector");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    *n = 0;
    int slot = agent_find(h, agent_id);
    if (slot < 0) return 0;
    uint32_t total = 0;
    if (which == AGR_LIST_PENDING) {
        // LRANGE: ids of expired records are still in the list; they lie below the scan's low-water mark
        TRY(select_locked(h, K3_AGENT_PENDING_IDS, (uint32_t)slot, nullptr, h->expired_total ? h->tail : h->scan_lo, ingested_bound(h), cap, &total));
    } else {
        unsigned long long lens[2];
        TRY(read_log_lens(h, lens));
        const uint32_t* log = (which == AGR_LIST_COMPLETED) ? h->d.completed_log : h->d.failed_log;
        uint64_t len = (which == AGR_LIST_COMPLETED) ? lens[0] : lens[1];
        TRY(select_locked(h, K3_LOG_AGENT, (uint32_t)slot, log, 0, len, cap, &total));
    }
    *n = total;
    if (total > cap) return fail(AGR_ECAP, "output array too small");
    if (total == 0 || !ids) return 0;
    return gather_rows_locked(h, h->d_out_rid.p, total, nullptr, nullptr, ids);
}

// The read-only resolve of one request id in the dedupe index: its physical row is left in d_hrid[0] (and in *rid, unless
// rid is NULL).  count_launch:
// the resolve launch counts in k3_launches (agr_get_record_var's does not).
static int resolve_one_locked(agr_handle* h, const char* agent_id, const uint8_t request_id[16], uint32_t* rid, bool count_launch) {
    int slot = agent_find(h, agent_id);
    if (slot < 0) return fail(AGR_ENOTFOUND, "request not found");
    agr_dop& op = h->h_ops[0];
    memcpy(&op.id_lo, request_id, 8); memcpy(&op.id_hi, request_id + 8, 8);
    op.slot = (uint32_t)slot; op.http = 0; op.kind = 0; op.pad = 0; op.seq = 0;
    CK(cudaMemcpyAsync(h->d_ops, h->h_ops, sizeof(agr_dop), cudaMemcpyHostToDevice, h->stream));
    sync_window(h);
    agr_launch_resolve(h->d, h->d_ops, h->d_hrid, 1, h->stream);
    if (count_launch) h->k3_launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h->h_small, h->d_hrid, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (h->h_small[0] == AGR_RID_NONE) return fail(AGR_ENOTFOUND, "request not found");
    if (rid) *rid = h->h_small[0];
    return 0;
}

// storage.Get("agent:{a}:requests:{r}") (server.go:661-662): read-only resolve in the dedupe index, then a 1-row gather
int agr_get_record(agr_handle* h, const char* agent_id, const uint8_t request_id[16], agr_record* out) {
    if (!h || !agent_id || !request_id || !out) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    TRY(resolve_one_locked(h, agent_id, request_id, nullptr, true));
    return gather_rows_locked(h, h->d_hrid, 1, nullptr, out, nullptr);
}

// ------------------------------------------------------------------------------------------ variable-length records
int agr_ingest_var(agr_handle* h, const uint8_t* blob, const uint32_t* offsets, uint32_t n, agr_verdict* out, uint8_t (*ids)[16],
                   uint64_t* first_rid) {
    if (!h || (n && (!blob || !offsets))) return fail(AGR_EINVAL, "NULL argument");
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_VARLEN");
    if (h->svc && n >= 1 && n <= SVC_MAX_CALL && offsets[0] == 0) {
        // single-request front end when every record is in the compact form (its length is the one its header gives): such a
        // record is a record span of the ring (agr_svc.h); any other blob is one locked batch
        bool compact = true;
        for (uint32_t i = 0; i < n && compact; ++i) compact = offsets[i + 1] >= offsets[i] + AGR_HEADER_BYTES;
        for (uint32_t i = 0; i < n && compact; ++i) compact = offsets[i + 1] - offsets[i] == svc_rec_len_at(blob + offsets[i]);
        if (compact) return svc_ingest_var(h, blob, offsets, n, out, ids, first_rid);
    }
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (n > h->cfg.max_batch) return fail(AGR_EINVAL, "n exceeds max_batch");
    uint64_t first = 0;
    if (n == 0) { if (first_rid) *first_rid = h->rows_used; return 0; }
    const uint64_t bytes = offsets[n];
    if (offsets[0] != 0) return fail(AGR_EINVAL, "offsets[0] must be 0");
    const uint32_t maxrec = h->cfg.max_record_bytes;
    h->long_list.clear();
    for (uint32_t i = 0; i < n; ++i) {                           // host-side shape check (lengths are part of the wire format)
        const uint32_t len = offsets[i + 1] - offsets[i];
        if (offsets[i + 1] < offsets[i] || (len & 15u) || len < AGR_HEADER_BYTES || len > maxrec)
            return fail(AGR_EINVAL, "record " + std::to_string(i) + ": length must be a multiple of 16 in [96, " + std::to_string(maxrec) + "]");
        if (len > AGR_VAR_MAX_RECORD) h->long_list.push_back(i);
    }
    const uint32_t nlong = (uint32_t)h->long_list.size();
    if (nlong) {                                                 // then each long record's first 8 KiB piece, and the total
        uint32_t pieces = 0;
        for (uint32_t k = 0; k < nlong; ++k) {
            const uint32_t i = h->long_list[k];
            h->long_list.push_back(pieces);
            pieces += (offsets[i + 1] - offsets[i] + AGR_VT_TILE - 1) / AGR_VT_TILE;
        }
        h->long_list.push_back(pieces);
    }
    uint64_t vpad = 0;
    TRY(vbytes_fit(h, bytes, &vpad));                             // (byte ring: a blob never wraps either)
    TRY(reserve_rows_locked(h, n, &first));
    if (first_rid) *first_rid = first;
    const uint64_t base = vbytes_take(h, bytes, vpad);            // physical byte offset of the blob
    cudaStream_t st = h->stream;
    CK(cudaMemcpyAsync(h->d.slab + base, blob, bytes, cudaMemcpyHostToDevice, st));
    TRY(h2d_staged(h, h->d_voffsets, offsets, ((size_t)n + 1) * 4, h->h_voffsets));
    TRY(launch_k1v_locked(h, first, n, base, h->d_voffsets, bytes, out ? h->d_verdicts : nullptr, ids ? h->d_ids : nullptr, nlong));
    if (out) CK(cudaMemcpyAsync(h->h_verdicts, h->d_verdicts, (size_t)n * sizeof(agr_verdict), cudaMemcpyDeviceToHost, st));
    if (ids) CK(cudaMemcpyAsync(h->h_ids, h->d_ids, (size_t)n * 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (out) memcpy(out, h->h_verdicts, (size_t)n * sizeof(agr_verdict));
    if (ids) memcpy(ids, h->h_ids, (size_t)n * 16);
    return 0;
}

// packs the variable-length records of rows d_out_rid[0..total) into the caller's blob
static int gather_var_locked(agr_handle* h, uint32_t total, uint8_t* blob, uint64_t blob_cap, uint64_t* offsets, uint64_t* blob_bytes) {
    const uint32_t ncap = std::max<uint32_t>(total, 1024);
    if (total > h->d_lens.cap) TRY(regrow(h, h->d_lens, ncap));
    if ((size_t)total + 1 > h->d_goffs.cap) TRY(regrow(h, h->d_goffs, (size_t)ncap + 1));
    agr_launch_var_lens(h->d, h->d_out_rid.p, total, h->d_lens.p, h->stream);
    std::vector<uint32_t> lens(total);
    CK(cudaMemcpyAsync(lens.data(), h->d_lens.p, (size_t)total * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    std::vector<unsigned long long> offs((size_t)total + 1);
    offs[0] = 0;
    for (uint32_t j = 0; j < total; ++j) offs[j + 1] = offs[j] + lens[j];
    *blob_bytes = offs[total];
    if (offsets) for (uint32_t j = 0; j <= total; ++j) offsets[j] = offs[j];
    if (!blob) return 0;
    if (offs[total] > blob_cap) return fail(AGR_ECAP, "blob too small");
    TRY(ensure_gather(h, (size_t)offs[total] + 16));
    CK(cudaMemcpyAsync(h->d_goffs.p, offs.data(), ((size_t)total + 1) * 8, cudaMemcpyHostToDevice, h->stream));
    agr_launch_var_copy(h->d, h->d_out_rid.p, total, h->d_goffs.p, h->d_gather.p, h->stream);
    h->k3_launches += 2;
    CK(cudaGetLastError());
    TRY(d2h_staged(h, blob, h->d_gather.p, (size_t)offs[total], h->h_gather.p));
    return 0;
}

int agr_replay_scan_var(agr_handle* h, agr_dispatch* out, uint8_t* blob, uint64_t blob_cap, uint64_t* offsets, uint32_t cap,
                        uint32_t* n, uint64_t* blob_bytes) {
    if (!h || !n || !blob_bytes) return fail(AGR_EINVAL, "NULL argument");
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_VARLEN");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    *n = 0; *blob_bytes = 0;
    h->replay_scans++;
    uint32_t total = 0;
    TRY(select_locked(h, K3_TICK, 0, nullptr, h->scan_lo, ingested_bound(h), cap, &total));
    *n = total;
    if (total > cap) return fail(AGR_ECAP, "dispatch array too small");
    h->replay_dispatched += total;
    if (total == 0) return 0;
    if (out) TRY(gather_rows_locked(h, h->d_out_rid.p, total, out, nullptr, nullptr));
    return gather_var_locked(h, total, blob, blob_cap, offsets, blob_bytes);
}

int agr_get_record_var(agr_handle* h, const char* agent_id, const uint8_t request_id[16], uint8_t* out, uint32_t cap, uint32_t* len) {
    if (!h || !agent_id || !request_id || !len) return fail(AGR_EINVAL, "NULL argument");
    if (!(h->cfg.flags & AGR_CFG_VARLEN)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_VARLEN");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    TRY(resolve_one_locked(h, agent_id, request_id, nullptr, false));
    TRY(ensure_out(h, 1));
    CK(cudaMemcpyAsync(h->d_out_rid.p, h->d_hrid, 4, cudaMemcpyDeviceToDevice, h->stream));
    uint64_t bytes = 0;
    uint64_t offs[2];
    TRY(gather_var_locked(h, 1, nullptr, 0, offs, &bytes));      // the record's length, then the record itself
    *len = (uint32_t)bytes;
    if (bytes > cap || !out) return out ? fail(AGR_ECAP, "output buffer too small") : 0;
    return gather_var_locked(h, 1, out, cap, offs, &bytes);
}

// ------------------------------------------------------------------------------------------ stored responses
// which: 0 = response (hdr_len leading bytes are its flattened headers), 1 = error text
static int store_bytes_locked(agr_handle* h, const char* agent_id, const uint8_t request_id[16], int which, const uint8_t* a, uint32_t alen,
                              const uint8_t* b, uint32_t blen) {
    uint32_t rid = 0;
    TRY(resolve_one_locked(h, agent_id, request_id, &rid, true));
    const uint32_t len = alen + blen;
    const uint64_t need = ((uint64_t)len + 15u) & ~15ull;
    unsigned long long off;
    TRY(resp_reserve_locked(h, need, len, &off));
    if (alen) CK(cudaMemcpyAsync(h->d_resp + off, a, alen, cudaMemcpyHostToDevice, h->stream));
    if (blen) CK(cudaMemcpyAsync(h->d_resp + off + alen, b, blen, cudaMemcpyHostToDevice, h->stream));
    if (which == 0) {
        CK(cudaMemcpyAsync(h->d_resp_off + rid, &off, 8, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_resp_len + rid, &len, 4, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_resp_hlen + rid, &alen, 4, cudaMemcpyHostToDevice, h->stream));
    } else {
        CK(cudaMemcpyAsync(h->d_err_off + rid, &off, 8, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_err_len + rid, &len, 4, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
int agr_store_response(agr_handle* h, const char* agent_id, const uint8_t request_id[16], const uint8_t* headers, uint32_t hdr_len,
                       const uint8_t* body, uint32_t body_len) {
    if (!h || !agent_id || !request_id || (hdr_len && !headers) || (body_len && !body)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return store_bytes_locked(h, agent_id, request_id, 0, headers, hdr_len, body, body_len);
}
int agr_store_response_body(agr_handle* h, const char* agent_id, const uint8_t request_id[16], const uint8_t* bytes, uint32_t len) {
    return agr_store_response(h, agent_id, request_id, nullptr, 0, bytes, len);
}
int agr_store_error_text(agr_handle* h, const char* agent_id, const uint8_t request_id[16], const char* text, uint32_t len) {
    if (!h || !agent_id || !request_id || (len && !text)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    return store_bytes_locked(h, agent_id, request_id, 1, (const uint8_t*)text, len, nullptr, 0);
}

int agr_get_response_body(agr_handle* h, const char* agent_id, const uint8_t request_id[16], uint8_t* out, uint32_t cap, uint32_t* len) {
    if (!h || !agent_id || !request_id || !len) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    uint32_t rid = 0;
    TRY(resolve_one_locked(h, agent_id, request_id, &rid, true));
    unsigned long long off = 0; uint32_t l = 0;
    CK(cudaMemcpyAsync(&off, h->d_resp_off + rid, 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&l, h->d_resp_len + rid, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *len = l;
    if (l > cap || !out) return (out && l > cap) ? fail(AGR_ECAP, "output buffer too small") : 0;
    if (l) { CK(cudaMemcpyAsync(out, h->d_resp + off, l, cudaMemcpyDeviceToHost, h->stream)); CK(cudaStreamSynchronize(h->stream)); }
    return 0;
}

// ------------------------------------------------------------------------------------------ K5: JSON wire form
// Encodes n records (rows d_rids[0..n) or first_rid + [0..n)) into h->d_json; *total = bytes.  Offsets stay in h->d_joff.
static int json_encode_locked(agr_handle* h, const uint32_t* d_rids, uint64_t first_rid, uint32_t n, bool array, uint64_t* total, bool roundtrip = false) {
    *total = 0;
    if (n == 0) return 0;
    const uint32_t cap = std::max<uint32_t>(n, 1024);
    if (n > h->d_jlen.cap) TRY(regrow(h, h->d_jlen, cap));
    if ((size_t)n + 1 > h->d_joff.cap) TRY(regrow(h, h->d_joff, (size_t)cap + 1));
    if ((size_t)agr_k5_chunks(n) + 1 > h->d_jchunk.cap) TRY(regrow(h, h->d_jchunk, (size_t)agr_k5_chunks(cap) + 1));
    agr_k5_params p{};
    p.rids = d_rids; p.first_l = first_rid; p.n = n; p.array = array ? 1u : 0u; p.roundtrip = roundtrip ? 1u : 0u;
    sync_window(h);
    p.len = h->d_jlen.p; p.off = h->d_joff.p; p.chunk_sum = h->d_jchunk.p; p.out = nullptr;
    p.bytes = h->d_resp; p.resp_off = h->d_resp_off; p.resp_len = h->d_resp_len; p.resp_hlen = h->d_resp_hlen;
    p.err_off = h->d_err_off; p.err_len = h->d_err_len; p.ptime = h->d.ptime;
    TRY(op_time_begin(h, 2));
    agr_launch_k5_measure(h->d, p, h->stream);
    CK(cudaGetLastError());
    unsigned long long tot = 0;
    CK(cudaMemcpyAsync(&tot, h->d_jchunk.p + agr_k5_chunks(n), 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (tot + 16 > h->d_json.cap) TRY(regrow(h, h->d_json, (size_t)std::max<uint64_t>(tot + tot / 4 + 16, 1 << 16)));
    p.out = h->d_json.p;
    agr_launch_k5_emit(h->d, p, h->stream);
    CK(cudaGetLastError());
    TRY(op_time_end(h, 2));
    h->k5_launches += 3;
    *total = tot;
    return 0;
}
static int json_copy_out(agr_handle* h, uint64_t total, uint8_t* out, uint64_t cap, uint64_t* len) {
    *len = total;
    if (!out) { CK(cudaStreamSynchronize(h->stream)); return 0; }
    if (total > cap) return fail(AGR_ECAP, "output buffer too small");
    if (total) CK(cudaMemcpyAsync(out, h->d_json.p, (size_t)total, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

int agr_rows_json(agr_handle* h, uint64_t first_rid, uint32_t n, int as_array, uint8_t* out, uint64_t cap, uint64_t* len, uint64_t* offsets) {
    if (!h || !len) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (first_rid + n > h->rows_used || first_rid < h->tail) return fail(AGR_EINVAL, "row range outside the rows in use");
    uint64_t total = 0;
    TRY(json_encode_locked(h, nullptr, first_rid, n, (as_array & 1) != 0, &total, (as_array & 2) != 0));
    if (n == 0 && (as_array & 1)) {                              // json.Marshal of a nil slice
        *len = 4;
        if (out) { if (cap < 4) return fail(AGR_ECAP, "output buffer too small"); memcpy(out, "null", 4); }
        if (offsets) offsets[0] = 0;
        return 0;
    }
    if (offsets && n) CK(cudaMemcpyAsync(offsets, h->d_joff.p, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, h->stream));
    else if (offsets) offsets[0] = 0;
    return json_copy_out(h, total, out, cap, len);
}

int agr_pending_json(agr_handle* h, const char* agent_id, uint8_t* out, uint64_t cap, uint64_t* len, uint32_t* count) {
    if (!h || !agent_id || !len) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (count) *count = 0;
    uint32_t total_rows = 0;
    int slot = agent_find(h, agent_id);
    if (slot >= 0) {
        const uint32_t cap0 = std::max<uint32_t>((uint32_t)h->d_out_rid.cap, 1024);
        TRY(select_locked(h, K3_AGENT_PENDING, (uint32_t)slot, nullptr, h->scan_lo, ingested_bound(h), cap0, &total_rows));
        if (total_rows > cap0)                                   // counts only: run again with room for all of it
            TRY(select_locked(h, K3_AGENT_PENDING, (uint32_t)slot, nullptr, h->scan_lo, ingested_bound(h), total_rows, &total_rows));
    }
    if (count) *count = total_rows;
    if (total_rows == 0) {                                       // var requests []*Request stays nil (requests.go:204): "null"
        *len = 4;
        if (out) { if (cap < 4) return fail(AGR_ECAP, "output buffer too small"); memcpy(out, "null", 4); }
        return 0;
    }
    uint64_t total = 0;
    TRY(json_encode_locked(h, h->d_out_rid.p, 0, total_rows, true, &total, true));   // GetPendingRequests unmarshals every record
    return json_copy_out(h, total, out, cap, len);
}

int agr_get_record_json(agr_handle* h, const char* agent_id, const uint8_t request_id[16], uint8_t* out, uint32_t cap, uint32_t* len) {
    if (!h || !agent_id || !request_id || !len) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    TRY(resolve_one_locked(h, agent_id, request_id, nullptr, true));
    uint64_t total = 0, l = 0;
    TRY(json_encode_locked(h, h->d_hrid, 0, 1, false, &total));   // k2.hrid[0] = the physical row resolve_one_locked found
    int rc = json_copy_out(h, total, out, cap, &l);
    *len = (uint32_t)l;
    return rc;
}

int agr_expire(agr_handle* h, uint64_t now, uint64_t ttl, uint64_t* expired) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    unsigned long long* d_cnt = expired ? count_slot(h) : nullptr;
    if (d_cnt) CK(cudaMemsetAsync(d_cnt, 0, 8, h->stream));
    sync_window(h);
    if ((!is_ring(h) || (h->cfg.flags & AGR_CFG_VARLEN)) && h->rows_used > h->sweep_clean) {
        // append-only slabs and variable-length engines: K1 does not keep the chunks' time bounds (k1_note_time); the chunks that
        // received rows since the last sweep are marked "unknown" here and get their exact bound back from this sweep
        const uint64_t R = h->cfg.slab_rows, lo = std::max(h->sweep_clean, h->tail), hi = h->rows_used;
        if (is_ring(h) && hi - lo >= R) CK(cudaMemsetAsync(h->d.cmin, 0, (size_t)(R / AGR_CHUNK_ROWS + 1) * 8, h->stream));
        else if (hi > lo) {
            const uint64_t p0 = phys_row(h, lo), p1 = phys_row(h, hi - 1);
            auto zero = [&](uint64_t a, uint64_t b) { return cudaMemsetAsync(h->d.cmin + a / AGR_CHUNK_ROWS, 0, (size_t)(b / AGR_CHUNK_ROWS - a / AGR_CHUNK_ROWS + 1) * 8, h->stream); };
            if (p0 <= p1) CK(zero(p0, p1)); else { CK(zero(p0, R - 1)); CK(zero(0, p1)); }
        }
        h->sweep_clean = ingested_bound(h);
    }
    agr_launch_expire(h->d, rows_span(h), now, ttl, d_cnt, h->stream);
    h->k3_launches += 1;
    CK(cudaGetLastError());
    if (!expired) {                       // no count wanted: stay asynchronous (the sweep is stream-ordered before whatever follows)
        h->expired_total = std::max<uint64_t>(h->expired_total, 1);   // "records may have expired": the list views widen their scan
        return 0;
    }
    unsigned long long v = 0;
    TRY(read_count(h, &v));
    h->expired_total += v;
    *expired = v;
    return 0;
}

// what one scan of the ring's tail reports back (device -> pinned host, one 32-byte copy)
struct reclaim_result { uint32_t off, pad; unsigned long long lens[2]; unsigned long long voff; };

// enqueues the scan: first stored row behind the tail (k_first_live), the log lengths and — variable-length mode — the byte
// offset of that row's record, packed by the scan's last CTA straight into pinned memory; nothing waits here
static int reclaim_scan_launch(agr_handle* h, uint64_t bound) {
    sync_window(h);
    // (the scan's two scratch words re-arm themselves, and its last CTA writes the result into the pinned buffer: one launch)
    agr_launch_first_live(h->d, bound - h->tail, is_ring(h) && !(h->cfg.flags & AGR_CFG_VARLEN), h->d_reclaim_scratch, h->h_reclaim, h->stream);
    CK(cudaGetLastError());
    if (!h->reclaim_ev) CK(cudaEventCreateWithFlags(&h->reclaim_ev, cudaEventDisableTiming));
    CK(cudaEventRecord(h->reclaim_ev, h->stream));
    h->reclaim_bound = bound;
    h->reclaim_pending = true;
    h->k3_launches += 2;
    return 0;
}

// releases what a finished scan found: rows [tail, tail + count) go back to the ring
static int reclaim_apply(agr_handle* h, uint64_t* released) {
    h->reclaim_pending = false;
    const reclaim_result r = *reinterpret_cast<const reclaim_result*>(h->h_reclaim);
    const uint64_t bound = h->reclaim_bound;
    const uint64_t count = (r.off == 0xffffffffu) ? bound - h->tail : r.off;
    if (count == 0) return 0;
    sync_window(h);
    agr_launch_release_rows(h->d, (uint32_t)count, h->d_resp_len, h->d_resp_hlen, h->d_err_len, h->stream);
    h->k3_launches += 1;
    for (int k = 0; k < 2; ++k) {                                              // completed, failed
        if (!r.lens[k]) continue;
        uint32_t*& log = k == 0 ? h->d.completed_log : h->d.failed_log;
        agr_launch_log_compact(h->d, log, r.lens[k], (uint32_t)count, h->d_log_scratch, h->d_lc_chunks, h->d.log_len + k, h->stream);
        CK(cudaGetLastError());
        std::swap(log, h->d_log_scratch);                                      // the compacted copy becomes the log
        h->k3_launches += 3;
    }
    h->tail += count;
    h->released_total += count;
    h->agent_gen++;                                            // released rows may have held removed agents' slots
    if (h->scan_lo < h->tail) h->scan_lo = h->tail;
    sync_window(h);
    // hash-id mode: the released rows' ids must leave the dedupe index before their rows are reused
    if (!(h->cfg.flags & AGR_CFG_MINT_IDS)) TRY(ring_reindex_locked(h));
    if (h->resp_used != h->resp_tail) {   // the response / error byte ring: its tail follows the oldest blob a live row still refers to
        CK(cudaMemsetAsync(count_slot(h), 0, 8, h->stream));
        agr_launch_bytes_span(h->d, h->resp_used % h->resp_cap, h->resp_cap, h->d_resp_off, h->d_resp_len, h->d_err_off, h->d_err_len, count_slot(h), h->stream);
        CK(cudaGetLastError());
        unsigned long long span = 0;
        TRY(read_count(h, &span));
        h->resp_tail = h->resp_used - span;
        h->k3_launches += 1;
    }
    // The byte ring's tail follows: first byte of the first live record.  It never passes the slot of a reserved row that K1 has
    // not decided yet: the scan stops at `bound` (ingested_bound: the first such row), bytes are handed out in row order under the
    // handle mutex (reserve_run_locked, agr_ingest_var), so the live record found below the bound lies before every such slot,
    // and with none found the tail moves to vused only when no row is reserved at all.
    if (h->cfg.flags & AGR_CFG_VARLEN) {
        if (r.off == 0xffffffffu) h->vtail = (bound == h->rows_used) ? h->vused : h->vtail;
        else {
            uint64_t used = (h->vused % h->vcap + h->vcap - r.voff) % h->vcap;
            if (used == 0) used = h->vcap;                         // head == tail with live records: the ring is exactly full
            h->vtail = h->vused - used;
        }
    }
    if (released) *released = count;
    return 0;
}

// AGR_CFG_RING: hand the rows at the tail that hold no record any more (expired or never stored) back to the ring, up to
// the first row that still does, and drop their entries from the completed / failed logs.
int agr_reclaim(agr_handle* h, uint64_t* released) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (released) *released = 0;
    if (!is_ring(h)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_RING");
    uint64_t got = 0;
    if (h->reclaim_pending) { CK(cudaEventSynchronize(h->reclaim_ev)); TRY(reclaim_apply(h, &got)); }   // a scan agr_reclaim_async left behind
    const uint64_t bound = ingested_bound(h);                                  // reserved rows that K1 has not filled yet are not "dead"
    if (bound > h->tail) {
        TRY(reclaim_scan_launch(h, bound));
        CK(cudaStreamSynchronize(h->stream));                                  // the only host round trip
        uint64_t more = 0;
        TRY(reclaim_apply(h, &more));
        got += more;
    }
    if (released) *released = got;
    return 0;
}
// The same without the host round trip in the caller's way: releases what the scan started by the PREVIOUS call found (it has
// long finished) and starts the next scan.  A ring that is maintained every step lags one step behind and never waits.
int agr_reclaim_async(agr_handle* h, uint64_t* released) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (released) *released = 0;
    if (!is_ring(h)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_RING");
    if (h->reclaim_pending) { CK(cudaEventSynchronize(h->reclaim_ev)); TRY(reclaim_apply(h, released)); }
    const uint64_t bound = ingested_bound(h);
    if (bound > h->tail) TRY(reclaim_scan_launch(h, bound));
    return 0;
}

// The sweep covers the physical rows [0, rows_span) except those of reservations that agr_ingest_rows has not decided yet:
// such a row may hold bytes (agr_fill_rows) but no checksum until K1 takes one.  One launch per range between them.
int agr_verify(agr_handle* h, uint64_t* rows_checked, uint64_t* bad) {
    if (!h || !bad) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    CK(cudaMemsetAsync(count_slot(h), 0, 8, h->stream));
    sync_window(h);
    const uint64_t span = rows_span(h);
    std::vector<std::pair<uint64_t, uint64_t>> skip;          // physical [first, end) of the undecided rows, a ring's split where it wraps
    for (const auto& r : h->resv) {
        const uint64_t p = phys_row(h, r.first), n = r.end - r.first;
        const uint64_t n0 = is_ring(h) ? std::min<uint64_t>(n, h->cfg.slab_rows - p) : n;
        skip.emplace_back(p, p + n0);
        if (n > n0) skip.emplace_back(0, n - n0);
    }
    std::sort(skip.begin(), skip.end());
    uint64_t at = 0, checked = 0;
    skip.emplace_back(span, span);
    for (const auto& s : skip) {
        const uint64_t end = std::min(s.first, span);
        if (end > at) {
            agr_launch_verify(h->d, at, end - at, count_slot(h), h->stream);
            h->k3_launches += 1;
            checked += end - at;
        }
        at = std::max(at, std::min(s.second, span));
    }
    CK(cudaGetLastError());
    unsigned long long v = 0;
    TRY(read_count(h, &v));
    *bad = v;
    if (rows_checked) *rows_checked = checked;
    return 0;
}

// ------------------------------------------------------------------------------------------ stats
int agr_stats_get(agr_handle* h, agr_stats* out) {
    if (!h || !out) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    unsigned long long c[C_NCTR], lens[2];
    CK(cudaMemcpyAsync(c, h->d.ctr, sizeof c, cudaMemcpyDeviceToHost, h->stream));
    TRY(read_log_lens(h, lens));
    memset(out, 0, sizeof *out);
    out->rows_used = h->rows_used; out->rows_cap = h->cfg.slab_rows;
    out->ingested = c[C_INGESTED]; out->stored = c[C_STORED]; out->replay_flagged = c[C_REPLAY];
    out->dedupe_hits = c[C_DEDUPE_HITS]; out->forwarded = c[C_FORWARDED]; out->queued = c[C_QUEUED];
    out->unavailable = c[C_UNAVAILABLE]; out->not_found = c[C_NOT_FOUND]; out->dup_ids = c[C_DUP_IDS];
    out->completions = c[C_COMPLETIONS]; out->completion_misses = c[C_COMPLETION_MISSES];
    out->failures = c[C_FAILURES]; out->dead_lettered = c[C_DEAD_LETTERED]; out->dial_errors = c[C_DIAL_ERRORS];
    out->replay_scans = h->replay_scans; out->replay_dispatched = h->replay_dispatched;
    out->completed_log_len = lens[0]; out->failed_log_len = lens[1];
    out->k1_launches = h->k1_launches; out->k2_launches = h->k2_launches;
    out->k3_launches = h->k3_launches; out->k4_launches = h->k4_launches; out->k5_launches = h->k5_launches; out->rows_tail = h->tail;
    out->malformed = c[C_BAD_LEN]; out->log_overflow = c[C_LOG_OVERFLOW];
    if (h->svc) { out->svc_batches = h->svc->batches.load(); out->svc_ops = h->svc->ops.load(); }
    out->agents = (uint32_t)h->agent_names.size(); out->device = (uint32_t)h->device;
    return 0;
}

int agr_debug_read(agr_handle* h, int which, uint64_t first_rid, uint32_t n, void* out) {
    if (!h || (n && !out)) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (which == AGR_DBG_CMIN) {                              // per physical chunk, not per row
        const uint64_t chunks = h->cfg.slab_rows / AGR_CHUNK_ROWS + 1;
        if (first_rid > chunks || n > chunks - first_rid) return fail(AGR_EINVAL, "chunk range out of bounds");
        if (n) CK(cudaMemcpyAsync(out, h->d.cmin + first_rid, (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return 0;
    }
    if (which == AGR_DBG_INDEX_USED) {                        // one count over the whole dedupe index
        if (first_rid != 0 || n != 1) return fail(AGR_EINVAL, "AGR_DBG_INDEX_USED reads one value (first_rid 0, n 1)");
        std::vector<agr_slot> t(h->d.table_mask + 1);
        CK(cudaMemcpyAsync(t.data(), h->d.table, t.size() * sizeof(agr_slot), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        uint64_t used = 0;
        for (const agr_slot& s : t) used += (s.key_lo | s.key_hi) != 0ULL;
        memcpy(out, &used, 8);
        return 0;
    }
    if (!is_ring(h) && first_rid + n > h->cfg.slab_rows) return fail(AGR_EINVAL, "row range out of bounds");
    if (is_ring(h) && (first_rid + n > h->rows_used || n > h->cfg.slab_rows)) return fail(AGR_EINVAL, "row range out of bounds");
    const uint8_t* base = nullptr; size_t w = 4;
    const bool verdict = which == AGR_DBG_VERDICT;            // route words, turned into agr_verdict on the host
    std::vector<uint32_t> words(verdict ? n : 0);
    void* dst = verdict ? (void*)words.data() : out;
    switch (which) {
        case AGR_DBG_STATE: base = (const uint8_t*)h->d.state; break;
        case AGR_DBG_ROUTE: case AGR_DBG_VERDICT: base = (const uint8_t*)h->d.route; break;
        case AGR_DBG_AUX: base = (const uint8_t*)h->d.aux; break;
        case AGR_DBG_CKSUM: base = (const uint8_t*)h->d.cksum; w = 8; break;
        case AGR_DBG_MTIME: base = (const uint8_t*)h->d.mtime; w = 8; break;
        case AGR_DBG_VOFF: base = (const uint8_t*)h->d.voff; w = 8; break;
        case AGR_DBG_VLEN: base = (const uint8_t*)h->d.vlen; break;
        case AGR_DBG_RESP_OFF: base = (const uint8_t*)h->d_resp_off; w = 8; break;
        case AGR_DBG_RESP_LEN: base = (const uint8_t*)h->d_resp_len; break;
        case AGR_DBG_ERR_OFF: base = (const uint8_t*)h->d_err_off; w = 8; break;
        case AGR_DBG_ERR_LEN: base = (const uint8_t*)h->d_err_len; break;
        default: return fail(AGR_EINVAL, "bad array selector");
    }
    if (!base) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_VARLEN");
    const uint64_t p0 = phys_row(h, first_rid);
    const uint64_t n0 = is_ring(h) ? std::min<uint64_t>(n, h->cfg.slab_rows - p0) : n;          // a logical range may wrap once
    if (n0) CK(cudaMemcpyAsync(dst, base + p0 * w, (size_t)n0 * w, cudaMemcpyDeviceToHost, h->stream));
    if (n > n0) CK(cudaMemcpyAsync((uint8_t*)dst + n0 * w, base, (size_t)(n - n0) * w, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    for (uint32_t i = 0; verdict && i < n; ++i) {
        const unsigned long long v = rt_verdict(words[i]);
        memcpy((uint8_t*)out + (size_t)i * sizeof(agr_verdict), &v, sizeof v);
    }
    return 0;
}

// Test-only: a ring engine whose window is empty moves its arrival counter forward by n, as if n records had arrived and been
// expired and released.  Every logical cursor moves together; the chunks' time bounds become "unknown" as after a restore.
int agr_debug_skip_arrivals(agr_handle* h, uint64_t n) {
    if (!h) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!is_ring(h)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_RING");
    if (n > AGR_ROW_LIMIT - h->rows_used) return fail(AGR_EINVAL, "skip would pass the row id bound (2^52)");
    if (h->tail != h->rows_used || !h->resv.empty() || h->reclaim_pending) return fail(AGR_EINVAL, "window not empty: expire and reclaim every row first");
    unsigned long long lens[2];
    TRY(read_log_lens(h, lens));
    if (lens[0] || lens[1]) return fail(AGR_EINVAL, "window not empty: the completed / failed logs hold entries");
    if (n == 0) return 0;
    h->rows_used += n; h->tail += n; h->released_total += n;
    h->scan_lo = h->tail; h->sweep_clean = h->rows_used; h->reclaim_bound = h->tail;
    h->d.idx_base = h->tail;
    sync_window(h);                                          // agr_dev's window, and rows_out for the single-request callers
    TRY(chunk_bounds_unknown(h));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

int agr_op_time(agr_handle* h, int which, double* ms) {
    if (!h || !ms || which < 0 || which > 4) return fail(AGR_EINVAL, "bad argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (!h->op_timed[which]) return fail(AGR_ENOTFOUND, "no timed launch of that group yet (needs AGR_CFG_TIMING)");
    CK(cudaStreamSynchronize(h->stream));
    float f = 0;
    CK(cudaEventElapsedTime(&f, h->op_ev[2 * which], h->op_ev[2 * which + 1]));
    *ms = f;
    return 0;
}

int agr_kernel_time(agr_handle* h, double* sum_ms, uint64_t* launches) {
    if (!h || !sum_ms || !launches) return fail(AGR_EINVAL, "NULL argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    *sum_ms = 0; *launches = 0;
    uint64_t from = h->tev_read;
    if (h->tev_next - from > AGR_TIMING_RING) from = h->tev_next - AGR_TIMING_RING;
    for (uint64_t i = from; i < h->tev_next; ++i) {
        float ms = 0;
        const uint64_t k = i % AGR_TIMING_RING;
        CK(cudaEventElapsedTime(&ms, h->tev[2 * k], h->tev[2 * k + 1]));
        *sum_ms += ms; (*launches)++;
    }
    h->tev_read = h->tev_next;
    h->timing_calls = 0;                       // the next launch is a timed one again (stride, k1_variant bits 16..23)
    return 0;
}

// ------------------------------------------------------------------------------------------ synthetic stream
int agr_synth_bind_mint(agr_handle* h, agr_synth* s, uint64_t base_rid) {
    if (!h || !s) return fail(AGR_EINVAL, "NULL argument");
    if (!(h->cfg.flags & AGR_CFG_MINT_IDS)) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_MINT_IDS");
    s->mint = 1; s->mint_base_rid = base_rid; s->mint_secret = h->d.id_secret; s->mint_shard = h->d.shard_id; s->mint_gen = h->d.id_gen;
    return 0;
}

static agr_synth_dev synth_params(const agr_synth* s, const unsigned long long* cdf) {
    agr_synth_dev p;
    p.mint = s->mint; p.mint_shard = s->mint_shard; p.mint_gen = s->mint_gen; p.pad = 0;
    p.mint_base_rid = s->mint_base_rid; p.mint_secret = s->mint_secret;
    p.seed = s->seed; p.n_agents = s->n_agents; p.dup_permille = s->dup_permille;
    p.agent_nanos0 = s->agent_nanos0 ? s->agent_nanos0 : 1700000000000000000ULL;
    p.cdf = cdf;
    return p;
}
// Zipf(s = zipf_milli / 1000) cumulative thresholds in pure integer arithmetic, so the table (and therefore the
// stream) is bit-identical on every host: weight_k = 2^40 * 2^-(s * log2(k+1)), log2 in 32.32 fixed point by
// repeated squaring, 2^-f as a product of the constants 2^-(2^-(b+1)) obtained from an integer square-root chain.
typedef unsigned __int128 u128_t;
static unsigned long long fx_log2(unsigned long long x) {        // integer x >= 1 -> log2(x) in 32.32
    unsigned long long ip = 0;
    for (unsigned long long v = x; v >= 2; v >>= 1) ip++;
    u128_t m = (u128_t)x << (63 - ip);                           // mantissa in [1,2) as Q1.63
    unsigned long long frac = 0;
    for (int b = 31; b >= 0; --b) {
        m = (m * m) >> 63;                                       // square: value in [1,4)
        if (m >> 64) { m >>= 1; frac |= (1ULL << b); }           // >= 2: emit a one bit, renormalise
    }
    return (ip << 32) | frac;
}
static unsigned long long isqrt128(u128_t v) {
    u128_t lo = 0, hi = (u128_t)1 << 64;
    while (lo + 1 < hi) { u128_t mid = (lo + hi) >> 1; if (mid * mid <= v) lo = mid; else hi = mid; }
    return (unsigned long long)lo;
}
static void zipf_cdf(uint32_t n, uint32_t zipf_milli, std::vector<unsigned long long>& cdf) {
    unsigned long long r[32];                                    // r[b] = 2^-(2^-(b+1)) in Q0.64
    r[0] = isqrt128((u128_t)1 << 127);
    for (int k = 1; k < 32; ++k) r[k] = isqrt128((u128_t)r[k - 1] << 64);
    std::vector<unsigned long long> w(n);
    u128_t total = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const unsigned long long y = (unsigned long long)(((u128_t)fx_log2((unsigned long long)k + 1) * zipf_milli) / 1000);
        const unsigned long long ip = y >> 32, fr = y & 0xffffffffULL;
        u128_t a = (u128_t)1 << 64;                              // 1.0 in Q1.64
        for (int b = 0; b < 32; ++b)
            if (fr & (1ULL << (31 - b))) a = (a * r[b]) >> 64;
        unsigned long long wk = ip >= 40 ? 0 : (unsigned long long)(a >> 24) >> ip;   // 2^40 * 2^-y
        w[k] = wk ? wk : 1;
        total += w[k];
    }
    cdf.resize(n);
    u128_t run = 0;
    for (uint32_t k = 0; k < n; ++k) {
        run += w[k];
        u128_t t = (run << 64) / total;
        cdf[k] = (k + 1 == n || (t >> 64)) ? ~0ULL : (unsigned long long)t;
    }
}

int agr_synth_agent_id(const agr_synth* s, uint32_t k, char out[AGR_AGENT_ID_BYTES]) {
    if (!s || !out) return fail(AGR_EINVAL, "NULL argument");
    unsigned long long n0 = s->agent_nanos0 ? s->agent_nanos0 : 1700000000000000000ULL;
    agr_synth_agent_name(n0 + (unsigned long long)k * 1000003ULL, out);
    return 0;
}
int agr_synth_fill_host(const agr_synth* s, uint64_t first_index, uint32_t n, agr_record* out) {
    if (!s || (n && !out) || s->n_agents == 0) return fail(AGR_EINVAL, "bad argument");
    std::vector<unsigned long long> cdf;
    if (s->zipf_milli) zipf_cdf(s->n_agents, s->zipf_milli, cdf);
    agr_synth_dev p = synth_params(s, s->zipf_milli ? cdf.data() : nullptr);
    for (uint32_t i = 0; i < n; ++i) agr_synth_record(p, first_index + i, (unsigned char*)&out[i]);
    return 0;
}
int agr_synth_fill_rows(agr_handle* h, const agr_synth* s, uint64_t first_index, uint64_t first_rid, uint32_t n) {
    if (!h || !s || s->n_agents == 0) return fail(AGR_EINVAL, "bad argument");
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    if (first_rid + n > h->rows_used) return fail(AGR_EINVAL, "rows not reserved");
    std::vector<slot_run> runs;                                  // (variable-length engines: the rows' slots)
    TRY(row_runs(h, first_rid, n, runs));
    const unsigned long long* dcdf = nullptr;
    if (s->zipf_milli) {
        std::vector<unsigned long long> cdf;
        zipf_cdf(s->n_agents, s->zipf_milli, cdf);
        if (h->d_cdf.cap < s->n_agents) TRY(regrow(h, h->d_cdf, s->n_agents));
        CK(cudaMemcpyAsync(h->d_cdf.p, cdf.data(), (size_t)s->n_agents * 8, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        dcdf = h->d_cdf.p;
    }
    uint32_t done = 0;
    for (const slot_run& r : runs) {
        agr_launch_synth(run_ptr(h, r), synth_params(s, dcdf), first_index + done, r.n, h->stream);
        done += r.n;
    }
    CK(cudaGetLastError());                                      // (stream-ordered before whatever reads the rows: no wait here)
    return 0;
}

uint64_t agr_agent_hash(const char* agent_id) { return agent_id ? agr_fnv1a64(agent_id, AGR_AGENT_ID_BYTES) : 0; }
uint32_t agr_agent_shard(const char* agent_id, uint32_t n_shards) {
    return n_shards ? (uint32_t)(agr_agent_hash(agent_id) % n_shards) : 0;
}

}  // extern "C"
