// agr_front.cu — the single-request front end (AGR_CFG_COMBINE): dispatcher thread, blocking calls through the ring, tickets.
#include "agr_engine.h"
#include "agr_ring.hpp"

// ------------------------------------------------------------------------------------------ single-request front end
// Host side of agr_svc.h.  Lock-free for the callers: one fetch_add claims ring slots, the payload is written into pinned
// device-mapped memory, a release store publishes it, and the caller waits on a word the GPU writes.  One dispatcher thread
// per handle turns the published prefix of the ring into batch descriptors; the resident service kernel (k_svc) does the rest.
cudaError_t agr_launch_svc(const agr_dev& d, const svc_dev& v, const agr_k2_scratch& k2, unsigned long long next_seq, bool var, cudaStream_t st);
unsigned long long agr_svc_desc_check(const svc_desc* dsc);

namespace agr_impl __attribute__((visibility("hidden"))) {
// answers every op of [from, to) from the host side (slab full, CUDA error): the callers see rc.  conts: the batch's
// continuation bits (relative to from), answered as already collected (nobody waits for them)
static void svc_fail_ops(svc_host* s, uint64_t from, uint64_t to, int rc, bool records_only, const uint32_t* conts) {
    for (uint64_t a = from; a < to; ++a) {
        const uint32_t slot = (uint32_t)(a & (SVC_SLOTS - 1u));
        const uint32_t rw = s->ready[slot].load(std::memory_order_relaxed), kd = rw & 3u;
        const bool rec = kd == SVC_OP_RECORD, cont = (conts[(a - from) >> 5] >> ((a - from) & 31u)) & 1u;
        // (a skipped slot has no waiter and keeps its old answer; it may even have been published again for the NEXT lap already)
        if ((rw >> 2) != (uint32_t)(a / SVC_SLOTS) + 1u || kd == SVC_OP_SKIP || (records_only && !rec)) continue;
        svc_res* r = s->res + slot;
        r->w[0] = rec ? 0u : cont ? 0u : (uint32_t)rc; r->w[1] = rec ? (uint32_t)rc : 0u; r->w[2] = 0;
        std::atomic_thread_fence(std::memory_order_release);
        r->w[3] = (svc_tag(a) | (cont ? SVC_COLLECTED : 0u)) << 16;
    }
}

// stops the resident kernel; the caller holds h->mu, so no new batch can be published meanwhile
int svc_stop_locked(agr_handle* h) {
    svc_host* s = h->svc;
    if (!s || !s->running) return 0;
    s->ctl->stop = 1;
    std::atomic_thread_fence(std::memory_order_seq_cst);
    cudaError_t e = cudaStreamSynchronize(h->stream);
    s->ctl->stop = 0;
    s->running = false;
    s->stops++;
    s->cyc[0] += (double)s->ctl->cyc_wait; s->cyc[1] += (double)s->ctl->cyc_load; s->cyc[2] += (double)s->ctl->cyc_work; s->cyc[3] += (double)s->ctl->cyc_publish;
    s->polls += s->ctl->heartbeat;
    if (e != cudaSuccess) { s->fatal = AGR_ECUDA; return fail(AGR_ECUDA, std::string("service kernel: ") + cudaGetErrorString(e)); }
    if (s->ctl->done_seq != s->seq) {
        // (cannot happen while the dispatcher runs: it stops the kernel after 2 ms without traffic, the kernel's own idle exit is 2 s)
        // whoever waits for an operation of those batches gets an error instead of waiting for ever
        for (uint64_t q = s->ctl->done_seq + 1; q <= s->seq; ++q) {
            const svc_desc* dsc = s->desc + (q % SVC_DESCS);
            if (dsc->seq == q) svc_fail_ops(s, dsc->from, dsc->from + dsc->count, AGR_ECUDA, false, dsc->cont);
        }
        s->fatal = AGR_ECUDA;
        return fail(AGR_ECUDA, "service kernel left with batches unprocessed");
    }
    return 0;
}
static int svc_start_locked(agr_handle* h) {
    svc_host* s = h->svc;
    if (s->running) return 0;
    svc_dev v{};
    v.desc = s->desc; v.payload = s->payload; v.res = s->res; v.ctl = s->ctl; v.dupfix = s->d_dupfix;
    v.resp = h->d_resp; v.resp_off = h->d_resp_off; v.resp_len = h->d_resp_len; v.resp_hlen = h->d_resp_hlen;
    v.err_off = h->d_err_off; v.err_len = h->d_err_len; v.b_off = s->d_boff; v.b_dst = s->d_bdst; v.b_hlen = s->d_bhlen;
    v.idle_ns = 2000000000ULL;                                   // safety only: the dispatcher stops the kernel long before
    s->ctl->state = 1; s->ctl->stop = 0;
    std::atomic_thread_fence(std::memory_order_seq_cst);
    sync_window(h);
    // resume at the first batch the previous incarnation did not run (normally none is pending; a batch published right
    // before this launch is)
    cudaError_t e = agr_launch_svc(h->d, v, s->k2, s->ctl->done_seq + 1, (h->cfg.flags & AGR_CFG_VARLEN) != 0, h->stream);
    if (e != cudaSuccess) { s->fatal = AGR_ECUDA; return fail(AGR_ECUDA, std::string("service kernel launch: ") + cudaGetErrorString(e)); }
    s->running = true;
    s->starts++;
    s->ctl->cyc_wait = 0; s->ctl->cyc_load = 0; s->ctl->cyc_work = 0; s->ctl->cyc_publish = 0; s->ctl->heartbeat = 0;
    s->started = std::chrono::steady_clock::now();
    return 0;
}

static void svc_dispatcher(agr_handle* h) {
    svc_host* s = h->svc;
    cudaSetDevice(h->device);
    auto last_work = std::chrono::steady_clock::now();
    uint32_t spins = 0;
    // the contiguous published prefix [taken, to), grown INCREMENTALLY: a slot is looked at until it is published and never again
    // (re-reading the callers' ready words every iteration keeps pulling their cache lines away from the cores that write them)
    uint64_t to = s->taken;
    uint32_t nstaged = 0;                                        // records + outcomes with bytes: one 512 B stage slot of k_svc each
    uint32_t kinds[SVC_MAX_OPS / 16] = {0}, conts[SVC_MAX_OPS / 32] = {0};
    // variable-length engines: records are record spans, and a batch's record bytes (one piece of the byte ring) stay within what
    // vbytes_fit takes in one piece
    const bool var = (h->cfg.flags & AGR_CFG_VARLEN) != 0;
    const uint64_t rec_bytes_max = is_ring(h) ? h->vcap / 2 : ~0ULL;
    uint64_t rec_bytes = 0;
    while (!s->shutdown.load(std::memory_order_acquire)) {
        // (csrc/agr_ring.hpp: shared with the CPU simulations of the ring)
        svc_scan(s, s->taken, &to, &nstaged, kinds, 128u, conts, var ? &rec_bytes : nullptr, rec_bytes_max);
        const auto now = std::chrono::steady_clock::now();
        if (to == s->taken) {
            const auto idle = std::chrono::duration_cast<std::chrono::microseconds>(now - last_work).count();
            if (idle > 2000) {
                // nothing for 2 ms: give the GPU (and this core) back; the next caller wakes us up
                { std::lock_guard<std::mutex> hl(h->mu); if (s->running) svc_stop_locked(h); }
                std::unique_lock<std::mutex> lk(s->smu);
                s->sleeping.store(true, std::memory_order_seq_cst);
                s->sleeps++;
                const uint32_t slot = (uint32_t)(s->taken & (SVC_SLOTS - 1u));
                if ((s->ready[slot].load(std::memory_order_seq_cst) >> 2) != (uint32_t)(s->taken / SVC_SLOTS) + 1u && !s->shutdown.load())
                    s->scv.wait_for(lk, std::chrono::milliseconds(50));
                s->sleeping.store(false, std::memory_order_seq_cst);
                last_work = std::chrono::steady_clock::now();
            } else {
                cpu_relax(spins);
            }
            continue;
        }
        last_work = now;
        // Batching window = the kernel's own pace: at most two batches are outstanding (one being decided, one being pulled by
        // the kernel's loader warps); while both are, keep collecting — whatever arrives meanwhile joins the next batch instead
        // of queueing behind a train of one-request batches.
        if (s->running && s->seq - s->ctl->done_seq >= 2 && to - s->taken < SVC_MAX_OPS) {
            s->flow_waits++;
            for (int k = 0; k < 8; ++k) _mm_pause();
            continue;
        }
        spins = 0;
        std::lock_guard<std::mutex> hl(h->mu);
        if (s->fatal.load()) {
            svc_fail_ops(s, s->taken, to, s->fatal.load(), false, conts);
            s->taken = to; nstaged = 0; rec_bytes = 0; memset(kinds, 0, sizeof kinds); memset(conts, 0, sizeof conts);
            continue;
        }
        if (s->running && s->ctl->state != 1u) {                // it left on its own (safety timeout): note it and start another
            cudaStreamSynchronize(h->stream);
            s->running = false;
        }
        // a resident kernel blocks device-wide synchronisations of other threads (cudaFree ...): let it go every 20 ms
        if (s->running && std::chrono::duration_cast<std::chrono::milliseconds>(now - s->started).count() > 20) svc_stop_locked(h);
        // records, and the outcomes with bytes with their segments' region (16 B-rounded, in ring order; a span's length is
        // clamped to the slots the batch holds of it, as the kernel does)
        const uint32_t count = (uint32_t)(to - s->taken);
        uint32_t nrec = 0, rec_slots = 0, nbytes = 0, ncont = 0;  // records (rows), their ring slots (record spans' continuations too)
        uint64_t byte_total = 0;
        for (uint32_t k = 0; k < count; ++k) {
            const uint32_t kd = (kinds[k >> 4] >> ((k & 15u) * 2u)) & 3u;
            if (kd == SVC_OP_RECORD) rec_slots++;
            if ((conts[k >> 5] >> (k & 31u)) & 1u) { ncont++; continue; }
            if (kd == SVC_OP_RECORD) nrec++;
            if (kd == SVC_OP_OUTCOME_BYTES) {                    // (the slot's payload is visible: its ready word was acquired)
                uint32_t len;
                memcpy(&len, s->payload + (size_t)((s->taken + k) & (SVC_SLOTS - 1u)) * SVC_PAYLOAD + SVC_BYTES_HDR + 4, 4);
                byte_total += (svc_span_len(len, svc_conts_after(conts, k, count)) + 15u) & ~15u;
                nbytes++;
            }
        }
        uint64_t first = 0;
        bool have_rows = true;
        svc_desc dsc{};
        if (nrec) {
            // rows, and on a variable-length engine the records' bytes, as one piece in agr_ingest_var's order: a refusal leaves
            // both rings as they were (the scan kept the bytes within vbytes_fit's limit unless one record alone exceeds it)
            uint64_t vpad = 0;
            int rc = var ? vbytes_fit(h, rec_bytes, &vpad) : 0;
            if (rc == 0) rc = reserve_rows_locked(h, nrec, &first) < 0 ? AGR_ENOSPC : 0;
            if (rc == 0 && var) dsc.vbase = vbytes_take(h, rec_bytes, vpad);
            if (rc < 0) { svc_fail_ops(s, s->taken, to, rc, true, conts); have_rows = false; }
        }
        for (uint32_t k = 0; k < (uint32_t)(to - s->taken); ++k) {
            uint32_t kd = (kinds[k >> 4] >> ((k & 15u) * 2u)) & 3u;
            if (kd == SVC_OP_RECORD && !have_rows) kd = SVC_OP_SKIP;
            dsc.kinds[k >> 4] |= kd << ((k & 15u) * 2u);
        }
        memcpy(dsc.cont, conts, sizeof conts);
        dsc.resp_base = SVC_NO_BYTES;
        if (nbytes) {
            unsigned long long off;
            if (resp_reserve_locked(h, byte_total, byte_total, &off) == 0) dsc.resp_base = off;
        }
        dsc.from = s->taken; dsc.count = count; dsc.n_records = have_rows ? nrec : 0u; dsc.rec_slots = have_rows ? rec_slots : 0u;
        dsc.first_l = first; dsc.first_p = (uint32_t)phys_row(h, first);
        dsc.tail = h->tail; dsc.head_l = h->rows_used; dsc.tail_phys = is_ring(h) ? (uint32_t)(h->tail % h->cfg.slab_rows) : 0u;
        dsc.idx_base = h->d.idx_base;
        dsc.seq = s->seq + 1;
        dsc.check = agr_svc_desc_check(&dsc);
        svc_desc* slot = s->desc + (dsc.seq % SVC_DESCS);
        // the batch number goes last; the kernel also verifies the check word, so a torn read is never accepted
        const uint64_t* src = reinterpret_cast<const uint64_t*>(&dsc);
        volatile uint64_t* dst = reinterpret_cast<volatile uint64_t*>(slot);
        for (int i = 0; i < 31; ++i) dst[i] = src[i];
        std::atomic_thread_fence(std::memory_order_release);
        dst[31] = src[31];
        std::atomic_thread_fence(std::memory_order_seq_cst);
        s->seq = dsc.seq;
        s->taken = to;
        s->batches.fetch_add(1, std::memory_order_relaxed);
        s->ops.fetch_add(dsc.count - ncont, std::memory_order_relaxed);     // operations: a span counts once
        h->k1_launches += nrec ? 1 : 0;                         // accounting: batches with records / with outcomes served by k_svc
        h->k2_launches += (dsc.count > nrec) ? 1 : 0;
        nstaged = 0; rec_bytes = 0; memset(kinds, 0, sizeof kinds); memset(conts, 0, sizeof conts);
        if (!s->running && svc_start_locked(h) < 0) {
            // could not launch: nothing will ever process this batch — fail it from here
            svc_fail_ops(s, dsc.from, to, AGR_ECUDA, false, dsc.cont);
        }
    }
    std::lock_guard<std::mutex> hl(h->mu);
    cudaSetDevice(h->device);
    svc_stop_locked(h);
}

// CPUs this process may keep busy: the cgroup CPU quota if there is one, else the online CPUs
static uint32_t cpu_allowance() {
    uint32_t n = std::max(1u, std::thread::hardware_concurrency());
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char a[64]; unsigned long long period = 0;
        if (fscanf(f, "%63s %llu", a, &period) == 2 && strcmp(a, "max") != 0 && period) {
            const unsigned long long q = strtoull(a, nullptr, 10);
            if (q) n = std::min<uint32_t>(n, (uint32_t)std::max<unsigned long long>(1, q / period));
        }
        fclose(f);
    }
    return n;
}

int svc_create(agr_handle* h) {
    svc_host* s = new svc_host();
    h->svc = s;
    auto pin = [&](void** p, size_t bytes) -> int {
        cudaError_t e = cudaHostAlloc(p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
        if (e != cudaSuccess) return fail(AGR_ENOMEM, std::string("cudaHostAlloc (request ring): ") + cudaGetErrorString(e));
        memset(*p, 0, bytes);
        h->host_allocs.push_back(*p);
        return 0;
    };
    TRY(pin((void**)&s->desc, sizeof(svc_desc) * SVC_DESCS));
    TRY(pin((void**)&s->payload, (size_t)SVC_SLOTS * SVC_PAYLOAD));
    TRY(pin((void**)&s->res, sizeof(svc_res) * SVC_SLOTS));
    TRY(pin((void**)&s->ctl, sizeof(svc_ctl)));
    s->ready = new std::atomic<uint32_t>[SVC_SLOTS];
    for (uint32_t i = 0; i < SVC_SLOTS; ++i) s->ready[i].store(0);
    TRY(dev_alloc(h, &s->k2.ops, (size_t)SVC_MAX_OPS, false));
    TRY(dev_alloc(h, &s->k2.nxt, (size_t)SVC_MAX_OPS, false));
    TRY(dev_alloc(h, &s->k2.eff, (size_t)SVC_MAX_OPS + 8, false));
    TRY(dev_alloc(h, &s->k2.results, (size_t)SVC_MAX_OPS, false));
    TRY(dev_alloc(h, &s->d_dupfix, (size_t)4, true));
    TRY(dev_alloc(h, &s->d_boff, (size_t)SVC_MAX_OPS + 1, false));
    TRY(dev_alloc(h, &s->d_bdst, (size_t)SVC_MAX_OPS, false));
    TRY(dev_alloc(h, &s->d_bhlen, (size_t)SVC_MAX_OPS, false));
    CK(cudaStreamSynchronize(h->stream));
    const uint32_t cpus = cpu_allowance();
    s->spin_cpus = cpus > 6 ? cpus - 6 : 1;             // leave room for the dispatcher, the driver's threads and the nappers' wake-ups
    s->thr = std::thread(svc_dispatcher, h);
    return 0;
}
void svc_destroy(agr_handle* h) {
    svc_host* s = h->svc;
    if (!s) return;
    if (s->thr.joinable()) {
        s->shutdown.store(true, std::memory_order_release);
        { std::lock_guard<std::mutex> lk(s->smu); s->scv.notify_all(); }
        s->thr.join();
    }
    if (getenv("AGR_SVC_DEBUG")) {
        const double mhz = 1965.0, tot = s->cyc[0] + s->cyc[1] + s->cyc[2] + s->cyc[3];
        const double nb = (double)std::max<uint64_t>(1, s->batches.load());
        fprintf(stderr, "[agr svc] batches %llu ops %llu (%.1f/batch) | kernel starts %llu stops %llu, dispatcher sleeps %llu, flow waits %llu | "
                        "per batch: wait %.2f us, load %.2f us, work %.2f us, publish %.2f us (kernel alive %.1f ms), polls %llu\n",
                (unsigned long long)s->batches.load(), (unsigned long long)s->ops.load(), (double)s->ops.load() / nb,
                (unsigned long long)s->starts, (unsigned long long)s->stops, (unsigned long long)s->sleeps, (unsigned long long)s->flow_waits,
                s->cyc[0] / mhz / nb, s->cyc[1] / mhz / nb, s->cyc[2] / mhz / nb, s->cyc[3] / mhz / nb, tot / mhz / 1000.0, (unsigned long long)s->polls);
    }
    delete[] s->ready;
    h->svc = nullptr;
    delete s;
}

// (the callers' side of the ring — svc_submit_one, svc_try, svc_wait, svc_release — is csrc/agr_ring.hpp: the same code runs against a
// stand-in for the dispatcher and the GPU in tests/ring_sim.cpp, on the CPU)
// Request.ID of the record in ring slot a: minted from its row, or the caller's own (still in the slot's payload)
static inline void svc_request_id(agr_handle* h, uint64_t a, uint64_t rid, uint8_t id[16]) {
    if (h->cfg.flags & AGR_CFG_MINT_IDS) {
        unsigned long long lo, hi;
        agr_mint_id(rid, h->d.shard_id, h->d.id_gen, h->d.id_secret, lo, hi);
        memcpy(id, &lo, 8); memcpy(id + 8, &hi, 8);
    } else memcpy(id, h->svc->payload + (size_t)(a & (SVC_SLOTS - 1u)) * SVC_PAYLOAD, 16);
}

// collects the answers of the records a blocking call handed over (ring slots pos[0..n), in call order)
static int svc_collect_records(agr_handle* h, const uint64_t* pos, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid) {
    svc_host* s = h->svc;
    int rc = 0;
    for (uint32_t i = 0; i < n; ++i) {
        svc_answer r; svc_wait(s, pos[i], &r);
        if ((r.w0 & 0xffu) == 0u) rc = (int)r.w1;
        else {
            if (out) { memcpy(&out[i], &r.w0, 4); memcpy((uint8_t*)&out[i] + 4, &r.w1, 4); }
            const uint64_t row = svc_row(s, r);
            if (ids) svc_request_id(h, pos[i], row, ids[i]);
            if (i == 0 && first_rid) *first_rid = row;
        }
        svc_release(s, pos[i]);
    }
    if (rc == AGR_EINVAL) return fail(rc, "record larger than half the byte slab");
    if (rc < 0) return fail(rc, rc == AGR_ENOSPC ? "slab full" : "single-request front end: CUDA error");
    return 0;
}
int svc_ingest(agr_handle* h, const agr_record* recs, uint32_t n, agr_verdict* out, uint8_t (*ids)[16], uint64_t* first_rid) {
    uint64_t pos[SVC_MAX_CALL];
    for (uint32_t i = 0; i < n; ++i) while (!svc_submit_one(h->svc, SVC_OP_RECORD, &recs[i], sizeof(agr_record), &pos[i])) {}   // in call order
    return svc_collect_records(h, pos, n, out, ids, first_rid);
}
// agr_ingest_var through the ring: record i is the svc_rec_len bytes at blob + offsets[i] (the caller checked that they are)
int svc_ingest_var(agr_handle* h, const uint8_t* blob, const uint32_t* offsets, uint32_t n, agr_verdict* out, uint8_t (*ids)[16],
                   uint64_t* first_rid) {
    uint64_t pos[SVC_MAX_CALL];
    for (uint32_t i = 0; i < n; ++i) while (!svc_submit_record(h->svc, blob + offsets[i], &pos[i])) {}
    return svc_collect_records(h, pos, n, out, ids, first_rid);
}
int svc_complete(agr_handle* h, const agr_outcome* outs, uint32_t n, int32_t* results) {
    svc_host* s = h->svc;
    uint64_t pos[SVC_MAX_CALL];
    for (uint32_t i = 0; i < n; ++i) while (!svc_submit_one(s, SVC_OP_OUTCOME, &outs[i], sizeof(agr_outcome), &pos[i])) {}
    int rc = 0;
    bool log_full = false;
    for (uint32_t i = 0; i < n; ++i) {
        svc_answer r; svc_wait(s, pos[i], &r);
        const int32_t res = (int32_t)r.w0;
        if (res < 0 && res != AGR_ENOTFOUND) rc = res;
        log_full |= (r.w1 & SVC_OUT_LOG_FULL) != 0u;
        if (results) results[i] = res;
        svc_release(s, pos[i]);
    }
    if (rc < 0) return fail(rc, "single-request front end: CUDA error");
    if (log_full) return fail(AGR_ENOSPC, K2_LOG_FULL);       // as the batch path: applied, the push dropped
    return 0;
}

// agr_complete_ex through the single-request ring: every outcome goes as SVC_OP_OUTCOME_BYTES with its segment inline
int svc_complete_ex(agr_handle* h, const agr_outcome* outs, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                    const uint32_t* hdr_lens, int32_t* results) {
    uint64_t total = 0, max_len = 0;
    TRY(check_segments(outs, n, offsets, hdr_lens, &total, &max_len));
    if (total && !bytes) return fail(AGR_EINVAL, "NULL bytes");
    svc_host* s = h->svc;
    uint64_t pos[SVC_MAX_CALL];
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t len = (uint32_t)(offsets[i + 1] - offsets[i]);
        const uint32_t hl = (hdr_lens && outs[i].kind == AGR_OUT_RESPONSE) ? hdr_lens[i] : 0u;
        while (!svc_submit_outcome_bytes(s, &outs[i], hl, len ? bytes + offsets[i] : nullptr, len, nullptr, 0u, &pos[i])) {}
    }
    int rc = 0;
    bool log_full = false;
    for (uint32_t i = 0; i < n; ++i) {
        svc_answer r; svc_wait(s, pos[i], &r);
        int32_t res = (int32_t)r.w0;
        if (res == AGR_ENOSPC) { res = 0; if (rc == 0) rc = AGR_ENOSPC; }
        else if (res < 0 && res != AGR_ENOTFOUND) rc = res;
        log_full |= (r.w1 & SVC_OUT_LOG_FULL) != 0u;
        if (results) results[i] = res;
        svc_release(s, pos[i]);
    }
    if (rc == AGR_ENOSPC)
        return fail(rc, std::string("response byte slab full: the outcomes were applied, their response / error bytes were not stored "
                                    "(raise agr_config.resp_bytes, or agr_reclaim with AGR_CFG_RING)") +
                            (log_full ? std::string("; also ") + K2_LOG_FULL : std::string()));
    if (rc < 0) return fail(rc, "single-request front end: CUDA error");
    if (log_full) return fail(AGR_ENOSPC, K2_LOG_FULL);
    return 0;
}

}  // namespace agr_impl

extern "C" {
// ------------------------------------------------------------------------------------------ tickets (submit / collect)
uint32_t agr_ring_capacity(void) { return SVC_SLOTS; }
#define TICKET_OUTCOME (1ULL << 63)                               // a ticket = ring slot number | kind
static int submit_one(agr_handle* h, uint32_t kind, const void* item, size_t bytes, agr_ticket* ticket) {
    if (!h || !item || !ticket) return fail(AGR_EINVAL, "NULL argument");
    svc_host* s = h->svc;
    if (!s) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_COMBINE");
    uint64_t a = 0;
    if (!svc_submit_one(s, kind, item, bytes, &a)) return AGR_EAGAIN;   // collect outstanding tickets (agr_poll) and come again
    *ticket = a | (kind == SVC_OP_OUTCOME ? TICKET_OUTCOME : 0ULL);
    return 0;
}
int agr_submit_ingest(agr_handle* h, const agr_record* rec, agr_ticket* ticket) {
    if (!h || !rec || !ticket || !h->svc || !(h->cfg.flags & AGR_CFG_VARLEN)) return submit_one(h, SVC_OP_RECORD, rec, sizeof(agr_record), ticket);
    if (h->cfg.max_record_bytes > AGR_VAR_MAX_RECORD) {         // a long record would be stored whole by agr_ingest_var: refuse, do not cut it
        uint32_t w[2];
        memcpy(w, reinterpret_cast<const uint8_t*>(rec) + 76, 8);   // path_len, hdr_len | body_len (as svc_rec_len_at)
        if ((uint64_t)(w[0] & 0xffffu) + (w[0] >> 16) + w[1] > AGR_VAR_MAX_RECORD - AGR_HEADER_BYTES)
            return fail(AGR_EINVAL, "record longer than AGR_VAR_MAX_RECORD: a ticket carries at most 8192 B, agr_ingest_var takes longer records");
    }
    uint64_t a = 0;                                              // a variable-length record: a record span of its stored length
    if (!svc_submit_record(h->svc, reinterpret_cast<const uint8_t*>(rec), &a)) return AGR_EAGAIN;
    *ticket = a;
    return 0;
}
int agr_submit_complete(agr_handle* h, const agr_outcome* outcome, agr_ticket* ticket) { return submit_one(h, SVC_OP_OUTCOME, outcome, sizeof(agr_outcome), ticket); }
static int collect(agr_handle* h, agr_ticket ticket, const svc_answer& r, agr_result* out) {
    svc_host* s = h->svc;
    const bool rec = !(ticket & TICKET_OUTCOME);
    const uint64_t t = ticket & ~TICKET_OUTCOME;
    if (out) {
        memset(out, 0, sizeof *out);
        out->is_outcome = rec ? 0u : 1u;
        if (rec) {
            if ((r.w0 & 0xffu) == 0u) out->result = (int32_t)r.w1;
            else { memcpy(&out->verdict, &r.w0, 4); memcpy((uint8_t*)&out->verdict + 4, &r.w1, 4); out->rid = svc_row(s, r); svc_request_id(h, t, out->rid, out->request_id); }
        } else out->result = (r.w1 & SVC_OUT_LOG_FULL) ? AGR_ENOSPC : (int32_t)r.w0;   // applied, its log push dropped
    }
    svc_release(s, t);
    return 0;
}
int agr_poll(agr_handle* h, agr_ticket ticket, agr_result* out) {
    if (!h || !h->svc) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_COMBINE");
    svc_answer r;
    if (!svc_try(h->svc, ticket & ~TICKET_OUTCOME, &r)) return AGR_EAGAIN;
    return collect(h, ticket, r, out);
}
int agr_wait(agr_handle* h, agr_ticket ticket, agr_result* out) {
    if (!h || !h->svc) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_COMBINE");
    svc_answer r;
    svc_wait(h->svc, ticket & ~TICKET_OUTCOME, &r);
    return collect(h, ticket, r, out);
}

// one outcome with its bytes in one ticket, hdr_len + body_len <= max_len (agr_submit_complete_ex: one slot;
// agr_submit_complete_large: a span of slots above AGR_OUT_INLINE_BYTES)
static int submit_outcome_bytes(agr_handle* h, const agr_outcome* outcome, const uint8_t* headers, uint32_t hdr_len, const uint8_t* body,
                                uint32_t body_len, agr_ticket* ticket, uint32_t max_len, const char* too_long) {
    if (!h || !outcome || !ticket || (hdr_len && !headers) || (body_len && !body)) return fail(AGR_EINVAL, "NULL argument");
    if (!h->svc) return fail(AGR_EINVAL, "engine was not created with AGR_CFG_COMBINE");
    if ((uint64_t)hdr_len + body_len > max_len) return fail(AGR_EINVAL, too_long);
    if (outcome->kind != AGR_OUT_RESPONSE && outcome->kind != AGR_OUT_ERROR && hdr_len + body_len)
        return fail(AGR_EINVAL, "only AGR_OUT_RESPONSE and AGR_OUT_ERROR outcomes carry bytes");
    uint64_t a = 0;
    if (!svc_submit_outcome_span(h->svc, outcome, outcome->kind == AGR_OUT_RESPONSE ? hdr_len : 0u, headers, hdr_len, body, body_len, &a))
        return AGR_EAGAIN;                                       // collect outstanding tickets (agr_poll) and come again
    *ticket = a | TICKET_OUTCOME;
    return 0;
}
int agr_submit_complete_ex(agr_handle* h, const agr_outcome* outcome, const uint8_t* headers, uint32_t hdr_len,
                           const uint8_t* body, uint32_t body_len, agr_ticket* ticket) {
    return submit_outcome_bytes(h, outcome, headers, hdr_len, body, body_len, ticket, AGR_OUT_INLINE_BYTES,
                                "headers + body exceed AGR_OUT_INLINE_BYTES: use agr_submit_complete_large or agr_complete_ex(n = 1)");
}
int agr_submit_complete_large(agr_handle* h, const agr_outcome* outcome, const uint8_t* headers, uint32_t hdr_len,
                              const uint8_t* body, uint32_t body_len, agr_ticket* ticket) {
    return submit_outcome_bytes(h, outcome, headers, hdr_len, body, body_len, ticket, AGR_OUT_TICKET_MAX_BYTES,
                                "headers + body exceed AGR_OUT_TICKET_MAX_BYTES: use agr_complete_ex(n = 1)");
}
}  // extern "C"
