// agr_ring.hpp — the CALLERS' side of the single-request ring (AGR_CFG_COMBINE; layout and protocol: agr_svc.h).
//
// Everything a calling thread does to hand one operation over and to collect its answer, as templates over the host-side ring
// object H (agr_engine.h's svc_host; the stand-ins of tests/ring_sim.cpp, tests/ring_sim_bytes.cpp, tests/ring_sim_span.cpp and
// tests/ring_sim_var.cpp).
// H provides:
//   svc_res* res; uint8_t* payload; std::atomic<uint32_t>* ready;          pinned, device-mapped in the engine
//   std::atomic<uint64_t> head, scanned; std::atomic<uint32_t> waiters; uint32_t spin_cpus;
//   std::atomic<uint64_t> rows_out                                          only where svc_row is used (callers that collect records)
//   std::atomic<bool> sleeping; std::mutex smu; std::condition_variable scv;   the dispatcher's sleep / wake-up
// The dispatcher (engine) or its stand-in (simulation) consumes ready words in slot order, keeps `scanned` = first slot whose
// ready word it has not consumed, and sees to it that every consumed operation other than SVC_OP_SKIP gets its 16-byte answer.
#pragma once
#include <stdint.h>
#include <string.h>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <immintrin.h>
#include <sched.h>
#include <time.h>
#include <sys/prctl.h>
#include "agr_svc.h"

// The answer cells are written by the GPU (one 16-byte PCIe store) and by host threads (svc_release, svc_fail_ops); their tag word
// is the synchronising one.  Acquire / release accesses through the compiler's atomic builtins: plain MOVs on x86-64, and a form
// ThreadSanitizer understands when this header runs against the CPU stand-in (tests/ring_sim.cpp).
static inline uint32_t svc_tag_word(const svc_res* r) { return __atomic_load_n(&r->w[3], __ATOMIC_ACQUIRE); }
static inline uint32_t svc_word(const svc_res* r, int k) { return __atomic_load_n(&r->w[k], __ATOMIC_RELAXED); }

static inline void cpu_relax(uint32_t& spins) {
    if (++spins < 4096u) _mm_pause();
    else { sched_yield(); }
}

// Slot reuse.  A caller that draws slot number a (lap = a / SVC_SLOTS of the ring) may overwrite the slot's payload and ready
// word only when the op one lap earlier is completely over: the dispatcher has consumed its ready word, the GPU has answered it
// and its caller has collected the answer (svc_release puts SVC_COLLECTED into the answer's tag).  The first two depend on
// the dispatcher and the GPU alone and are waited for.  The third depends on ANOTHER CALLER — the holder of that ticket, who may
// itself be inside a submit, waiting for one of our uncollected tickets — so it is never waited for beyond a short spin:
// the slot is published as a no-op instead (the ring moves on, the uncollected answer stays intact) and the caller is told to
// collect and come again (AGR_EAGAIN from agr_submit_*; the blocking calls, which hold no tickets, simply take the next slot).
template <class H>
static bool svc_slot_free(H* s, uint64_t a, uint32_t slot, uint32_t lap) {
    if (!lap) return true;
    const uint32_t prev = svc_tag(a - SVC_SLOTS);
    // usual case: the previous lap's op was a real one and is over (its tag in the cell says all three at once — and the ready
    // word, which sits in the dispatcher's cache, need not be read)
    if ((svc_tag_word(&s->res[slot]) >> 16) == (prev | SVC_COLLECTED)) return true;
    uint32_t w = 0;
    while (s->scanned.load(std::memory_order_acquire) <= a - SVC_SLOTS) cpu_relax(w);     // its ready word has been consumed
    const uint32_t rw = s->ready[slot].load(std::memory_order_acquire);
    if ((rw & 3u) != SVC_OP_SKIP) {
        w = 0;
        while (((svc_tag_word(&s->res[slot]) >> 16) & 0x7fffu) != prev) cpu_relax(w);                // answered (GPU, or svc_fail_ops)
    }
    // the previous lap was a no-op: the cell holds an older answer (or none at all)
    for (uint32_t k = 0; k < 2000u; ++k) {                                                   // ~0.1 ms of patience
        const uint32_t t = svc_tag_word(&s->res[slot]) >> 16;
        if (t == 0u || (t & SVC_COLLECTED)) return true;
        _mm_pause();
    }
    return false;
}
// hands ONE operation over.  true: *abs is its slot (ticket); false: the slot it drew was not free (see above).
template <class H>
static bool svc_submit_one(H* s, uint32_t kind, const void* item, size_t item_bytes, uint64_t* abs) {
    const uint64_t a = s->head.fetch_add(1, std::memory_order_relaxed);
    const uint32_t slot = (uint32_t)(a & (SVC_SLOTS - 1u)), lap = (uint32_t)(a / SVC_SLOTS);
    const bool ok = svc_slot_free(s, a, slot, lap);
    if (ok) {
        // streaming stores: the slot's lines were last written by another core a lap ago and are read next by the GPU (DMA),
        // so pulling them into this core's cache first (read-for-ownership) would only cost a miss per line
        __m128i* dst = reinterpret_cast<__m128i*>(s->payload + (size_t)slot * SVC_PAYLOAD);
        const __m128i* src = reinterpret_cast<const __m128i*>(item);
        for (size_t k = 0; k < item_bytes / 16; ++k) _mm_stream_si128(dst + k, _mm_loadu_si128(src + k));
        _mm_sfence();
    }
    s->ready[slot].store(((lap + 1u) << 2) | (ok ? kind : (uint32_t)SVC_OP_SKIP), std::memory_order_release);
    if (s->sleeping.load(std::memory_order_seq_cst)) { std::lock_guard<std::mutex> lk(s->smu); s->scv.notify_one(); }
    *abs = a;
    return ok;
}
// hands over ONE outcome with its bytes (SVC_OP_OUTCOME_BYTES): the 64 B outcome, hdr_len, the segment's length and the segment
// a | b; only the 16 B-rounded part of the slot that is used is written.  a_len + b_len <= SVC_BYTES_MAX (the caller checks).
template <class H>
static bool svc_submit_outcome_bytes(H* s, const void* outcome, uint32_t hdr_len, const uint8_t* a, uint32_t a_len, const uint8_t* b,
                                     uint32_t b_len, uint64_t* abs) {
    alignas(16) uint8_t item[SVC_PAYLOAD];
    const uint32_t len = a_len + b_len, used = (SVC_BYTES_DATA + len + 15u) & ~15u;
    memcpy(item, outcome, SVC_BYTES_HDR);
    memcpy(item + SVC_BYTES_HDR, &hdr_len, 4);
    memcpy(item + SVC_BYTES_HDR + 4, &len, 4);
    if (a_len) memcpy(item + SVC_BYTES_DATA, a, a_len);
    if (b_len) memcpy(item + SVC_BYTES_DATA + a_len, b, b_len);
    memset(item + SVC_BYTES_DATA + len, 0, used - SVC_BYTES_DATA - len);
    return svc_submit_one(s, SVC_OP_OUTCOME_BYTES, item, used, abs);
}
// item_bytes (a multiple of 16) into a slot's payload, with streaming stores as in svc_submit_one
template <class H>
static inline void svc_stream_slot(H* s, uint32_t slot, const void* item, size_t item_bytes) {
    __m128i* dst = reinterpret_cast<__m128i*>(s->payload + (size_t)slot * SVC_PAYLOAD);
    const __m128i* src = reinterpret_cast<const __m128i*>(item);
    for (size_t k = 0; k < item_bytes / 16; ++k) _mm_stream_si128(dst + k, _mm_loadu_si128(src + k));
}
// bytes [off, off + n) of the segment a | b
static inline void svc_copy_seg(uint8_t* dst, const uint8_t* a, uint32_t a_len, const uint8_t* b, uint32_t off, uint32_t n) {
    if (off < a_len) {
        const uint32_t m = a_len - off < n ? a_len - off : n;
        memcpy(dst, a + off, m);
        dst += m; off += m; n -= m;
    }
    if (n) memcpy(dst, b + (off - a_len), n);
}
// hands over ONE operation that takes n consecutive slots (a SPAN, agr_svc.h), claimed with one fetch_add (slot numbers wrap past
// the ring's end like any other); write(j, slot) streams the bytes of its j-th slot.  It is handed over only if every slot of
// it is free; otherwise all of them go out as no-ops and the result is false, as for svc_submit_one.
template <class H, class W>
static bool svc_submit_span(H* s, uint32_t kind, uint32_t n, W&& write, uint64_t* abs) {
    const uint64_t a0 = s->head.fetch_add(n, std::memory_order_relaxed);
    // every slot is looked at, also after one that is not free: a slot's ready word may be written again only once the
    // dispatcher has consumed its previous lap (svc_slot_free waits for that before it answers false)
    bool ok = true;
    for (uint32_t j = 0; j < n; ++j) {
        const uint64_t x = a0 + j;
        ok = svc_slot_free(s, x, (uint32_t)(x & (SVC_SLOTS - 1u)), (uint32_t)(x / SVC_SLOTS)) && ok;
    }
    if (ok) {
        for (uint32_t j = 0; j < n; ++j) write(j, (uint32_t)((a0 + j) & (SVC_SLOTS - 1u)));
        _mm_sfence();
    }
    // the continuations first, the head last: the dispatcher, which consumes slots in order, finds a published head complete
    if (!ok) kind = SVC_OP_SKIP;
    for (uint32_t j = n; j-- > 0;) {
        const uint64_t x = a0 + j;
        s->ready[x & (SVC_SLOTS - 1u)].store(((uint32_t)(x / SVC_SLOTS) + 1u) << 2 | kind, std::memory_order_release);
    }
    if (s->sleeping.load(std::memory_order_seq_cst)) { std::lock_guard<std::mutex> lk(s->smu); s->scv.notify_one(); }
    *abs = a0;
    return ok;
}
// hands over ONE outcome whose segment a | b may be longer than a slot holds (agr_submit_complete_large).  Up to SVC_BYTES_MAX
// bytes it is svc_submit_outcome_bytes; above that a span of 1 + svc_span_conts(len) slots.  a_len + b_len <=
// AGR_OUT_TICKET_MAX_BYTES (the caller checks).
template <class H>
static bool svc_submit_outcome_span(H* s, const void* outcome, uint32_t hdr_len, const uint8_t* a, uint32_t a_len, const uint8_t* b,
                                    uint32_t b_len, uint64_t* abs) {
    const uint32_t len = a_len + b_len;
    if (len <= SVC_BYTES_MAX) return svc_submit_outcome_bytes(s, outcome, hdr_len, a, a_len, b, b_len, abs);
    return svc_submit_span(s, SVC_OP_OUTCOME_BYTES, 1u + svc_span_conts(len), [&](uint32_t j, uint32_t slot) {
        alignas(16) uint8_t item[SVC_PAYLOAD];
        if (j == 0) {                                                 // head: outcome, hdr_len, len, the first SVC_BYTES_MAX bytes
            memcpy(item, outcome, SVC_BYTES_HDR);
            memcpy(item + SVC_BYTES_HDR, &hdr_len, 4);
            memcpy(item + SVC_BYTES_HDR + 4, &len, 4);
            svc_copy_seg(item + SVC_BYTES_DATA, a, a_len, b, 0u, SVC_BYTES_MAX);
            svc_stream_slot(s, slot, item, SVC_PAYLOAD);
            return;
        }
        // continuations: SVC_PAYLOAD bytes each, the last one 16 B-rounded
        const uint32_t off = SVC_BYTES_MAX + (j - 1u) * SVC_PAYLOAD, m = len - off < SVC_PAYLOAD ? len - off : SVC_PAYLOAD;
        const uint32_t used = (m + 15u) & ~15u;
        svc_copy_seg(item, a, a_len, b, off, m);
        memset(item + m, 0, used - m);
        svc_stream_slot(s, slot, item, used);
    }, abs);
}
// hands over ONE variable-length record (agr_svc.h: record span): the svc_rec_len_at(rec) bytes at rec, 512 per slot, the last
// slot holding the 16 B-rounded rest.  Only for a ring whose dispatcher scans with record spans (svc_scan's rec_bytes).
template <class H>
static bool svc_submit_record(H* s, const uint8_t* rec, uint64_t* abs) {
    const uint32_t len = svc_rec_len_at(rec);
    return svc_submit_span(s, SVC_OP_RECORD, svc_rec_slots(len), [&](uint32_t j, uint32_t slot) {
        const uint32_t off = j * SVC_PAYLOAD;
        svc_stream_slot(s, slot, rec + off, len - off < SVC_PAYLOAD ? len - off : SVC_PAYLOAD);
    }, abs);
}
// A record's answer carries the low 48 bits of its row (arrival number): svc_answer.rid.  svc_row rebuilds the full row from H's
// rows_out (rows handed out so far, stored with release by the dispatcher before it publishes the batch that names the row).
// Read after the answer's tag was acquired (svc_try / svc_wait), rows_out is above the row and less than 2^48 rows above it, so
// the row is the one below rows_out with those low bits.  Only callers that collect records need rows_out in H.
static inline uint64_t svc_full_row(uint64_t low48, uint64_t rows_out) {
    const uint64_t top = rows_out - 1u;
    return top - ((top - low48) & ((1ULL << 48) - 1u));
}
struct svc_answer { uint32_t w0, w1; uint64_t rid; };   // rid: low 48 bits of a record's row (svc_row gives all of it)
template <class H>
static inline bool svc_try(H* s, uint64_t a, svc_answer* out) {
    const svc_res* r = s->res + (a & (SVC_SLOTS - 1u));
    const uint32_t w3 = svc_tag_word(r);
    if ((w3 >> 16) != svc_tag(a)) return false;
    out->w0 = svc_word(r, 0); out->w1 = svc_word(r, 1); out->rid = (uint64_t)svc_word(r, 2) | ((uint64_t)(w3 & 0xffffu) << 32);
    return true;
}
// the full row of a collected record's answer (call after svc_try / svc_wait returned it, before svc_release)
template <class H>
static inline uint64_t svc_row(H* s, const svc_answer& r) {
    return svc_full_row(r.rid, s->rows_out.load(std::memory_order_acquire));
}
// Blocking wait.  The first spin_cpus waiters spin (the answer is ~20 us away); waiters beyond that many would only burn the
// process's CPU allowance against each other (a container with a CPU quota throttles ALL its threads once it is spent), so they
// sleep in short naps instead.
template <class H>
static inline void svc_wait(H* s, uint64_t a, svc_answer* out) {
    if (svc_try(s, a, out)) return;
    const uint32_t me = s->waiters.fetch_add(1, std::memory_order_relaxed);
    if (me < s->spin_cpus) {
        uint32_t w = 0;
        while (!svc_try(s, a, out)) cpu_relax(w);
    } else {
        static thread_local bool slack_set = false;
        if (!slack_set) { prctl(PR_SET_TIMERSLACK, 1000UL, 0, 0, 0); slack_set = true; }   // naps of tens of us, not the default +50 us
        struct timespec ts = {0, 25000};
        while (!svc_try(s, a, out)) nanosleep(&ts, nullptr);
    }
    s->waiters.fetch_sub(1, std::memory_order_relaxed);
}
template <class H>
static inline void svc_release(H* s, uint64_t a) {       // everything of the answer (and of the payload) has been read
    __atomic_store_n(&s->res[a & (SVC_SLOTS - 1u)].w[3], (svc_tag(a) | SVC_COLLECTED) << 16, __ATOMIC_RELEASE);
}

// ---- the dispatcher's side of the ready words
// Grows the contiguous published prefix [taken, *to) by whatever has been published since: at most SVC_MAX_OPS operations and
// max_staged records plus outcomes with bytes per batch (*nstaged counts those: each takes a whole 512 B slot of the kernel's
// stage; the dispatcher tells the two apart by kinds[]).  A slot is looked at until it is published and never again (re-reading
// the callers' ready words every iteration keeps pulling their cache lines away from the cores that write them), and an
// operation's kind is noted in kinds[] (2 bits each, the batch descriptor's form) AT THAT MOMENT: a no-op slot may be published
// again, for the next lap, as soon as `scanned` has passed it.  Publishes the new scan position.
// A span (agr_svc.h) is taken whole or not at all: its head's len word (visible: the head's ready word was acquired, and the
// continuations were published before it) says how many continuation slots follow; they count against both budgets, take the
// head's kind in kinds[] and are marked in conts[] (1 bit per op, svc_desc.cont).  Callers that never hand over spans may pass
// no conts.
// rec_bytes (rings of a variable-length engine only): records are record spans too, and *rec_bytes sums their svc_rec_len; a record
// that would take the sum above max_rec_bytes ends the batch unless it is the batch's first (the byte ring takes a batch's
// records as one piece, and a piece above half a ring is refused outright — a lone record still gets its answer from there).
template <class H>
static inline void svc_scan(H* s, const uint64_t taken, uint64_t* to, uint32_t* nstaged, uint32_t* kinds, const uint32_t max_staged,
                            uint32_t* conts = nullptr, uint64_t* rec_bytes = nullptr, const uint64_t max_rec_bytes = 0) {
    while (*to - taken < SVC_MAX_OPS) {
        const uint32_t slot = (uint32_t)(*to & (SVC_SLOTS - 1u));
        const uint32_t rw = s->ready[slot].load(std::memory_order_acquire), kind = rw & 3u;
        if ((rw >> 2) != (uint32_t)(*to / SVC_SLOTS) + 1u) break;
        uint32_t n = 1u, rlen = 0u;                                       // slots the op takes, a record's stored length
        if (kind == SVC_OP_OUTCOME_BYTES) {
            uint32_t len;
            memcpy(&len, s->payload + (size_t)slot * SVC_PAYLOAD + SVC_BYTES_HDR + 4, 4);
            n += svc_span_conts(len);
        } else if (kind == SVC_OP_RECORD && rec_bytes) {
            rlen = svc_rec_len_at(s->payload + (size_t)slot * SVC_PAYLOAD);
            n = svc_rec_slots(rlen);
        }
        if (n > 1u) {
            if (*to - taken + n > SVC_MAX_OPS) break;
            bool all = true;
            for (uint32_t j = 1; j < n && all; ++j)
                all = (s->ready[(slot + j) & (SVC_SLOTS - 1u)].load(std::memory_order_acquire) >> 2) == (uint32_t)((*to + j) / SVC_SLOTS) + 1u;
            if (!all) break;
        }
        const bool staged = kind == SVC_OP_RECORD || kind == SVC_OP_OUTCOME_BYTES;
        if (staged && *nstaged + n > max_staged) break;
        if (rlen && *rec_bytes && *rec_bytes + rlen > max_rec_bytes) break;
        if (staged) *nstaged += n;
        if (rlen) *rec_bytes += rlen;
        for (uint32_t j = 0; j < n; ++j, ++*to) {
            kinds[(*to - taken) >> 4] |= kind << (((*to - taken) & 15u) * 2u);
            if (j) conts[(*to - taken) >> 5] |= 1u << ((*to - taken) & 31u);
        }
    }
    if (*to != s->scanned.load(std::memory_order_relaxed)) s->scanned.store(*to, std::memory_order_release);
}
