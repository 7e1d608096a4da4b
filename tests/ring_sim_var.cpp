// ring_sim_var.cpp — the callers' side of the single-request ring (csrc/agr_ring.hpp: the code the library ships) on a ring that
// serves a variable-length engine: records are RECORD SPANS (svc_submit_record: agr_submit_ingest / agr_ingest_var through the
// ring) of 1 .. 16 slots, mixed with outcome spans (svc_submit_outcome_span) and plain outcomes, against a stand-in for the
// dispatcher and the service kernel on the CPU (the companion of tests/ring_sim_span.cpp).  The stand-in scans with record spans
// and a record-byte budget (svc_scan's rec_bytes), pulls a batch's staged slots into its own stage, reassembles every record from
// its span's stage slots, answers the continuations as collected, then answers every operation from the stage.  Checks:
//   * every operation handed over is answered exactly once, with the answer computed from ITS OWN bytes — for a record from a
//     checksum of all svc_rec_len bytes read across its span (a continuation rewritten before it was pulled, a span split
//     across batches or a record written short shows up as a wrong answer);
//   * the record bytes svc_scan sums for a batch equal the sum of its records' lengths, and stay within the budget unless the
//     batch's first record alone exceeds it; a batch never stages more than 128 slots;
//   * record lengths 96 .. 8192 with every slot count and the slot edges among them, and headers whose lengths exceed 8 KiB
//     (stored at the cap); spans cross the ring's end;
//   * blocking callers and ticket callers, also with more tickets held than the ring has slots (AGR_EAGAIN + no-op slots).
// usage: ring_sim_var <blocking threads> <ticket threads> <tickets in flight per ticket thread> <operations per thread>
//        [service delay us] [record-byte budget per batch]
// prints one JSON line; exit code 0 = every check passed.  Test infrastructure (tests/test_ring_sim_var.py), no CUDA.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <chrono>
#include <thread>
#include <vector>
#include "../agentainer-lab_b200/csrc/agr_ring.hpp"

struct sim_host {
    svc_res* res = nullptr; uint8_t* payload = nullptr;
    std::atomic<uint32_t>* ready = nullptr;
    uint32_t spin_cpus = 2;
    std::atomic<bool> sleeping{false};
    alignas(64) std::atomic<uint64_t> head{0};
    alignas(64) std::atomic<uint32_t> waiters{0};
    alignas(64) std::atomic<uint64_t> scanned{0};
    std::mutex smu; std::condition_variable scv;
};

static inline uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; return x ^ (x >> 33); }
static inline uint64_t fnv(const uint8_t* p, uint32_t n, uint64_t h) { for (uint32_t i = 0; i < n; ++i) h = (h ^ p[i]) * 0x100000001b3ULL; return h; }
static inline uint64_t bytes_key(uint32_t hdr_len, uint32_t len, const uint8_t* seg) { return fnv(seg, len, 0xcbf29ce484222325ULL ^ ((uint64_t)hdr_len << 32 | len)); }
static inline void fill(uint8_t* p, uint32_t len, uint64_t token) {
    uint64_t x = token | 1u;
    for (uint32_t k = 0; k < len; k += 8) {
        x ^= x << 13; x ^= x >> 7; x ^= x << 17;
        memcpy(p + k, &x, len - k < 8 ? len - k : 8);
    }
}

// a record: a stored length with every slot count 1 .. 16 and the slot edges among them, or a header whose lengths exceed
// 8 KiB; its header's path / headers / body lengths add up to anything that rounds to that length
static const uint32_t kLens[] = {96, 112, 496, 512, 528, 1008, 1024, 1040, 4192, 8176, 8192};
static uint32_t make_record(uint8_t* rec, uint64_t token) {
    uint32_t want;
    if ((token & 3u) == 0u) want = kLens[(token >> 8) % (sizeof kLens / sizeof kLens[0])];
    else if ((token & 3u) == 1u) want = 96u + 16u * (uint32_t)((token >> 8) % ((8192u - 96u) / 16u + 1u));
    else want = 512u * (1u + (uint32_t)((token >> 8) % 16u)) - 16u * (uint32_t)((token >> 20) % 3u);   // each slot count
    if (want < 96u) want = 96u;
    const uint32_t p = want - 96u;
    uint32_t body = p ? p - (uint32_t)((token >> 24) % 16u) : 0u, path = 0u, hdr = 0u;
    if (body > 40u) { path = (uint32_t)((token >> 32) % 20u); hdr = (uint32_t)((token >> 40) % 20u); body -= path + hdr; }
    if ((token >> 48) % 17u == 0u) body = 9000u + (uint32_t)(token >> 56);                   // lengths beyond 8 KiB
    fill(rec, 8192u, token);
    memcpy(rec, &token, 8);
    const uint32_t lens = path | (hdr << 16);
    memcpy(rec + 76, &lens, 4); memcpy(rec + 80, &body, 4);
    const uint32_t len = svc_rec_len(lens, body);
    if (len != ((body >= 9000u) ? 8192u : want)) return 0u;                                  // the length rule itself
    return len;
}

int main(int argc, char** argv) {
    const int nb = argc > 1 ? atoi(argv[1]) : 2, nt = argc > 2 ? atoi(argv[2]) : 4;
    const uint32_t inflight = argc > 3 ? (uint32_t)atoi(argv[3]) : 512u;
    const uint64_t per_thread = argc > 4 ? strtoull(argv[4], nullptr, 10) : 20000ULL;
    const int delay_us = argc > 5 ? atoi(argv[5]) : 0;
    const uint64_t budget = argc > 6 ? strtoull(argv[6], nullptr, 10) : ~0ULL;
    sim_host S;
    S.res = (svc_res*)aligned_alloc(64, sizeof(svc_res) * SVC_SLOTS); memset((void*)S.res, 0, sizeof(svc_res) * SVC_SLOTS);
    S.payload = (uint8_t*)aligned_alloc(64, (size_t)SVC_SLOTS * SVC_PAYLOAD); memset(S.payload, 0, (size_t)SVC_SLOTS * SVC_PAYLOAD);
    S.ready = new std::atomic<uint32_t>[SVC_SLOTS];
    for (uint32_t i = 0; i < SVC_SLOTS; ++i) S.ready[i].store(0);
    std::atomic<bool> quit{false};
    std::atomic<uint64_t> served{0}, skipped{0}, bad{0}, eagain{0}, done_ops{0}, rec_spans{0}, span_slots{0}, wrapped{0}, max_staged{0},
        max_rec_slots{0}, over_budget{0}, max_batch_bytes{0}, bad_len{0};

    // dispatcher + service kernel in one thread: the dispatcher's own scan (agr_ring.hpp), then what k_svc_var does with a batch
    std::thread service([&] {
        std::vector<uint8_t> stage((size_t)128 * SVC_PAYLOAD);
        uint64_t to = 0;
        while (!quit.load(std::memory_order_acquire)) {
            const uint64_t from = to;
            uint32_t nstaged = 0, kinds[SVC_MAX_OPS / 16] = {0}, conts[SVC_MAX_OPS / 32] = {0};
            uint64_t rec_bytes = 0;
            svc_scan(&S, from, &to, &nstaged, kinds, 128u, conts, &rec_bytes, budget);
            if (to == from) { std::this_thread::yield(); continue; }
            if (delay_us) std::this_thread::sleep_for(std::chrono::microseconds(delay_us));     // the batch is "on the GPU"
            const uint32_t count = (uint32_t)(to - from);
            auto kind_of = [&](uint32_t i) { return (kinds[i >> 4] >> ((i & 15u) * 2u)) & 3u; };
            auto is_cont = [&](uint32_t i) { return ((conts[i >> 5] >> (i & 31u)) & 1u) != 0u; };
            // pull: every record and outcome with bytes slot takes one stage slot, a span's slots next to each other
            uint32_t staged = 0;
            std::vector<int> stage_of(count, -1);
            for (uint32_t i = 0; i < count; ++i) {
                const uint32_t kind = kind_of(i);
                if (kind != SVC_OP_RECORD && kind != SVC_OP_OUTCOME_BYTES) continue;
                if (staged == 128u) { bad++; break; }
                memcpy(stage.data() + (size_t)staged * SVC_PAYLOAD, S.payload + (size_t)((from + i) & (SVC_SLOTS - 1u)) * SVC_PAYLOAD, SVC_PAYLOAD);
                stage_of[i] = (int)staged++;
            }
            if (staged != nstaged) bad++;
            if (staged > max_staged.load()) max_staged.store(staged);
            // the continuations' bytes are in the stage: answered as collected
            for (uint32_t i = 0; i < count; ++i) {
                if (!is_cont(i)) continue;
                if (i == 0 || kind_of(i) != kind_of(i - 1)) bad++;                      // never at a batch's start, the head's kind
                const uint64_t a = from + i;
                svc_res* r = S.res + (a & (SVC_SLOTS - 1u));
                __atomic_store_n(&r->w[0], 0u, __ATOMIC_RELAXED); __atomic_store_n(&r->w[1], 0u, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[2], 0u, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[3], (svc_tag(a) | SVC_COLLECTED) << 16, __ATOMIC_RELEASE);
                span_slots++;
            }
            // the operations, from the stage (outcomes without bytes: their own first 8 bytes, read from the ring)
            uint64_t batch_bytes = 0, first_len = 0;
            uint32_t nrec = 0;
            for (uint32_t i = 0; i < count; ++i) {
                const uint32_t kind = kind_of(i);
                const uint64_t a = from + i;
                if (kind == SVC_OP_SKIP) { skipped++; continue; }
                if (is_cont(i)) continue;
                const uint8_t* p = stage_of[i] >= 0 ? stage.data() + (size_t)stage_of[i] * SVC_PAYLOAD
                                                    : S.payload + (size_t)(a & (SVC_SLOTS - 1u)) * SVC_PAYLOAD;
                uint64_t token; memcpy(&token, p, 8);
                const uint32_t k = svc_conts_after(conts, i, count);
                if (kind == SVC_OP_RECORD) {
                    const uint32_t len = svc_rec_len_at(p);
                    if (k + 1u != svc_rec_slots(len)) { bad++; continue; }                // split or short span
                    if (len == 8192u) { uint32_t b; memcpy(&b, p + 80, 4); if (b >= 9000u) bad_len++; }
                    if (!nrec++) first_len = len;
                    batch_bytes += len;
                    if (k) {
                        rec_spans++;
                        if ((a & (SVC_SLOTS - 1u)) + k >= SVC_SLOTS) wrapped++;
                        if (k + 1u > max_rec_slots.load()) max_rec_slots.store(k + 1u);
                    }
                    token = fnv(p, len, token);                                          // contiguous across the span's stage slots
                } else if (kind == SVC_OP_OUTCOME_BYTES) {
                    uint32_t hl, len; memcpy(&hl, p + SVC_BYTES_HDR, 4); memcpy(&len, p + SVC_BYTES_HDR + 4, 4);
                    const uint32_t have = svc_span_len(len, k);
                    if (have != len || k != svc_span_conts(len) || hl > len) { bad++; len = have; hl = 0; }
                    token ^= bytes_key(hl, len, p + SVC_BYTES_DATA);
                }
                const uint64_t ans = mix(token ^ a);                                   // depends on the bytes AND the slot number
                svc_res* r = S.res + (a & (SVC_SLOTS - 1u));
                __atomic_store_n(&r->w[0], (uint32_t)ans | 1u, __ATOMIC_RELAXED); __atomic_store_n(&r->w[1], (uint32_t)(ans >> 32), __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[2], (uint32_t)kind, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[3], svc_tag(a) << 16, __ATOMIC_RELEASE);
                served++;
            }
            if (batch_bytes != rec_bytes) bad++;                                         // the scan's sum is the records' sum
            if (batch_bytes > budget) { if (nrec > 1u || first_len <= budget) bad++; else over_budget++; }
            if (batch_bytes > max_batch_bytes.load()) max_batch_bytes.store(batch_bytes);
        }
    });

    auto check = [&](uint64_t a, uint64_t token, const svc_answer& r) {
        const uint64_t ans = mix(token ^ a);
        if (r.w0 != ((uint32_t)ans | 1u) || r.w1 != (uint32_t)(ans >> 32)) bad++;
    };
    // one operation: a record (half of them), an outcome span or an inline outcome, a plain outcome.  *token = the answer's key
    auto submit = [&](uint64_t token, uint8_t* rec, uint8_t* seg, uint64_t* a, uint64_t* key) -> bool {
        const uint32_t pick = (uint32_t)(token >> 60) & 3u;
        alignas(16) uint8_t item[64];
        memset(item, 0, sizeof item); memcpy(item, &token, 8);
        *key = token;
        if (pick <= 1u) {
            const uint32_t len = make_record(rec, token);
            if (!len) { bad++; return true; }
            *key = fnv(rec, len, token);
            return svc_submit_record(&S, rec, a);
        }
        if (pick == 2u) {
            const uint32_t len = (uint32_t)((token >> 16) % 5000u), hl = (uint32_t)((token >> 24) % (len + 1u));
            fill(seg, len, token);
            *key = token ^ bytes_key(hl, len, seg);
            return svc_submit_outcome_span(&S, item, hl, seg, hl, seg + hl, len - hl, a);
        }
        return svc_submit_one(&S, SVC_OP_OUTCOME, item, sizeof item, a);
    };
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> ths;
    for (int t = 0; t < nb; ++t) ths.emplace_back([&, t] {                              // blocking callers: submit, wait, release
        std::vector<uint8_t> rec(8192), seg(8192);
        for (uint64_t i = 0; i < per_thread; ++i) {
            const uint64_t token = mix(((uint64_t)t << 40) | i);
            uint64_t a, key;
            while (!submit(token, rec.data(), seg.data(), &a, &key)) {}
            svc_answer r; svc_wait(&S, a, &r);
            check(a, key, r);
            svc_release(&S, a);
            done_ops++;
        }
    });
    for (int t = 0; t < nt; ++t) ths.emplace_back([&, t] {                              // ticket callers: a FIFO of parked operations
        struct fl { uint64_t a, key; };
        std::vector<fl> q(inflight);
        size_t head = 0, count = 0;
        std::vector<uint8_t> rec(8192), seg(8192);
        uint64_t issued = 0;
        while (issued < per_thread || count) {
            while (issued < per_thread && count < q.size()) {
                const uint64_t token = mix(((uint64_t)(t + 1000) << 40) | issued);
                uint64_t a, key;
                if (!submit(token, rec.data(), seg.data(), &a, &key)) { eagain++; break; }   // AGR_EAGAIN: collect, come again
                q[(head + count) % q.size()] = fl{a, key}; count++; issued++;
            }
            uint32_t reaped = 0;
            while (count && reaped < 64) {
                svc_answer r;
                if (!svc_try(&S, q[head].a, &r)) break;
                check(q[head].a, q[head].key, r);
                svc_release(&S, q[head].a);
                head = (head + 1) % q.size(); count--; reaped++; done_ops++;
            }
            if (!reaped) _mm_pause();
        }
    });
    for (auto& th : ths) th.join();
    const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    quit.store(true, std::memory_order_release);
    service.join();
    const uint64_t want = (uint64_t)(nb + nt) * per_thread;
    const bool ok = bad.load() == 0 && done_ops.load() == want && served.load() == want && max_staged.load() <= 128u;
    printf("{\"blocking_threads\": %d, \"ticket_threads\": %d, \"inflight\": %u, \"operations\": %llu, \"served\": %llu, \"record_spans\": %llu, "
           "\"span_slots\": %llu, \"wrapped_spans\": %llu, \"max_staged\": %llu, \"max_record_slots\": %llu, \"max_batch_bytes\": %llu, "
           "\"lone_over_budget\": %llu, \"capped_headers\": %llu, \"skipped_slots\": %llu, \"eagain\": %llu, \"wrong_answers\": %llu, "
           "\"seconds\": %.3f, \"ok\": %s}\n",
           nb, nt, inflight, (unsigned long long)done_ops.load(), (unsigned long long)served.load(), (unsigned long long)rec_spans.load(),
           (unsigned long long)span_slots.load(), (unsigned long long)wrapped.load(), (unsigned long long)max_staged.load(),
           (unsigned long long)max_rec_slots.load(), (unsigned long long)max_batch_bytes.load(), (unsigned long long)over_budget.load(),
           (unsigned long long)bad_len.load(), (unsigned long long)skipped.load(), (unsigned long long)eagain.load(),
           (unsigned long long)bad.load(), secs, ok ? "true" : "false");
    return ok ? 0 : 1;
}
