// ring_sim_span.cpp — the callers' side of the single-request ring (csrc/agr_ring.hpp: the code the library ships) with outcomes
// whose segment spans consecutive slots (svc_submit_outcome_span: agr_submit_complete_large), against a stand-in for the
// dispatcher and the service kernel that follows the span rules of agr_svc.h, on the CPU (the companion of
// tests/ring_sim_bytes.cpp).  The stand-in pulls a batch's staged slots into its own stage first, then answers the spans'
// continuation slots as collected (so callers may take them for the next lap at once), then answers every operation from the
// stage.  Checks:
//   * every operation handed over is answered exactly once, with the answer computed from ITS OWN payload — for an outcome with
//     bytes from a checksum of its hdr_len and len words and the WHOLE segment read across its span (a continuation rewritten
//     before it was pulled, a span split across batches or a segment written short shows up as a wrong answer);
//   * a batch never stages more than 128 slots (records, outcomes with bytes and continuation slots: one 512 B stage slot each);
//   * spans cross the ring's end; segment lengths 0 .. AGR_OUT_TICKET_MAX_BYTES with 440, 441, 952, 953 and 16384 among them,
//     mixed with records and plain and inline outcomes;
//   * blocking callers and ticket callers, also with more tickets held than the ring has slots (AGR_EAGAIN + no-op slots).
// usage: ring_sim_span <blocking threads> <ticket threads> <tickets in flight per ticket thread> <operations per thread>
//        [service delay us]
// prints one JSON line; exit code 0 = every check passed.  Test infrastructure (tests/test_ring_sim_span.py), no CUDA.
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

// a segment length: the edges of the slot layout often, anything up to the limit otherwise
static const uint32_t kEdges[] = {0, 1, 100, 440, 441, 951, 952, 953, 1464, 1465, 4096, 16383, 16384};
static inline uint32_t seg_len(uint64_t token) {
    if (token & 1u) return kEdges[(token >> 8) % (sizeof kEdges / sizeof kEdges[0])];
    return (uint32_t)((token >> 16) % (AGR_OUT_TICKET_MAX_BYTES + 1u));
}
static inline void fill(uint8_t* seg, uint32_t len, uint64_t token) {
    uint64_t x = token | 1u;
    for (uint32_t k = 0; k < len; k += 8) {
        x ^= x << 13; x ^= x >> 7; x ^= x << 17;
        memcpy(seg + k, &x, len - k < 8 ? len - k : 8);
    }
}

int main(int argc, char** argv) {
    const int nb = argc > 1 ? atoi(argv[1]) : 2, nt = argc > 2 ? atoi(argv[2]) : 4;
    const uint32_t inflight = argc > 3 ? (uint32_t)atoi(argv[3]) : 512u;
    const uint64_t per_thread = argc > 4 ? strtoull(argv[4], nullptr, 10) : 20000ULL;
    const int delay_us = argc > 5 ? atoi(argv[5]) : 0;
    sim_host S;
    S.res = (svc_res*)aligned_alloc(64, sizeof(svc_res) * SVC_SLOTS); memset((void*)S.res, 0, sizeof(svc_res) * SVC_SLOTS);
    S.payload = (uint8_t*)aligned_alloc(64, (size_t)SVC_SLOTS * SVC_PAYLOAD); memset(S.payload, 0, (size_t)SVC_SLOTS * SVC_PAYLOAD);
    S.ready = new std::atomic<uint32_t>[SVC_SLOTS];
    for (uint32_t i = 0; i < SVC_SLOTS; ++i) S.ready[i].store(0);
    std::atomic<bool> quit{false};
    std::atomic<uint64_t> served{0}, skipped{0}, bad{0}, eagain{0}, done_ops{0}, spans{0}, span_slots{0}, wrapped{0}, max_staged{0};

    // dispatcher + service kernel in one thread: the dispatcher's own scan (agr_ring.hpp), then what k_svc does with a batch
    std::thread service([&] {
        std::vector<uint8_t> stage((size_t)128 * SVC_PAYLOAD);
        std::vector<uint64_t> staged_op(128);
        uint64_t to = 0;
        while (!quit.load(std::memory_order_acquire)) {
            const uint64_t from = to;
            uint32_t nstaged = 0, kinds[SVC_MAX_OPS / 16] = {0}, conts[SVC_MAX_OPS / 32] = {0};
            svc_scan(&S, from, &to, &nstaged, kinds, 128u, conts);
            if (to == from) { std::this_thread::yield(); continue; }
            if (delay_us) std::this_thread::sleep_for(std::chrono::microseconds(delay_us));     // the batch is "on the GPU"
            const uint32_t count = (uint32_t)(to - from);
            auto kind_of = [&](uint32_t i) { return (kinds[i >> 4] >> ((i & 15u) * 2u)) & 3u; };
            auto is_cont = [&](uint32_t i) { return ((conts[i >> 5] >> (i & 31u)) & 1u) != 0u; };
            // pull: every record and outcome with bytes takes one stage slot, a span's slots next to each other
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
                if (i == 0 || kind_of(i) != SVC_OP_OUTCOME_BYTES) bad++;                  // never at a batch's start
                const uint64_t a = from + i;
                svc_res* r = S.res + (a & (SVC_SLOTS - 1u));
                __atomic_store_n(&r->w[0], 0u, __ATOMIC_RELAXED); __atomic_store_n(&r->w[1], 0u, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[2], 0u, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[3], (svc_tag(a) | SVC_COLLECTED) << 16, __ATOMIC_RELEASE);
                span_slots++;
            }
            // the operations, from the stage (outcomes without bytes: their own first 8 bytes, read from the ring)
            for (uint32_t i = 0; i < count; ++i) {
                const uint32_t kind = kind_of(i);
                const uint64_t a = from + i;
                if (kind == SVC_OP_SKIP) { skipped++; continue; }
                if (is_cont(i)) continue;
                const uint8_t* p = stage_of[i] >= 0 ? stage.data() + (size_t)stage_of[i] * SVC_PAYLOAD
                                                    : S.payload + (size_t)(a & (SVC_SLOTS - 1u)) * SVC_PAYLOAD;
                uint64_t token; memcpy(&token, p, 8);
                if (kind == SVC_OP_OUTCOME_BYTES) {
                    uint32_t hl, len; memcpy(&hl, p + SVC_BYTES_HDR, 4); memcpy(&len, p + SVC_BYTES_HDR + 4, 4);
                    const uint32_t k = svc_conts_after(conts, i, count), have = svc_span_len(len, k);
                    if (have != len || k != svc_span_conts(len) || hl > len) { bad++; len = have; hl = 0; }   // split or short span
                    if (k) {
                        spans++;
                        if ((a & (SVC_SLOTS - 1u)) + k >= SVC_SLOTS) wrapped++;
                    }
                    token ^= bytes_key(hl, len, p + SVC_BYTES_DATA);                    // contiguous across the span's stage slots
                }
                const uint64_t ans = mix(token ^ a);                                   // depends on the payload AND the slot number
                svc_res* r = S.res + (a & (SVC_SLOTS - 1u));
                __atomic_store_n(&r->w[0], (uint32_t)ans | 1u, __ATOMIC_RELAXED); __atomic_store_n(&r->w[1], (uint32_t)(ans >> 32), __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[2], (uint32_t)kind, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[3], svc_tag(a) << 16, __ATOMIC_RELEASE);
                served++;
            }
        }
    });

    auto check = [&](uint64_t a, uint64_t token, const svc_answer& r) {
        const uint64_t ans = mix(token ^ a);
        if (r.w0 != ((uint32_t)ans | 1u) || r.w1 != (uint32_t)(ans >> 32)) bad++;
    };
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> ths;
    for (int t = 0; t < nb; ++t) ths.emplace_back([&, t] {                              // blocking callers: submit, wait, release
        alignas(16) uint8_t item[64];
        std::vector<uint8_t> seg(AGR_OUT_TICKET_MAX_BYTES);
        for (uint64_t i = 0; i < per_thread; ++i) {
            uint64_t token = mix(((uint64_t)t << 40) | i);
            memset(item, 0, sizeof item); memcpy(item, &token, 8);
            uint64_t a;
            if ((i % 3u) != 0u) {                                         // headers + body, split anywhere
                const uint32_t len = seg_len(token), hl = (uint32_t)((token >> 24) % (len + 1u));
                fill(seg.data(), len, token);
                while (!svc_submit_outcome_span(&S, item, hl, seg.data(), hl, seg.data() + hl, len - hl, &a)) {}
                token ^= bytes_key(hl, len, seg.data());
            } else {
                while (!svc_submit_one(&S, SVC_OP_OUTCOME, item, sizeof item, &a)) {}
            }
            svc_answer r; svc_wait(&S, a, &r);
            check(a, token, r);
            svc_release(&S, a);
            done_ops++;
        }
    });
    for (int t = 0; t < nt; ++t) ths.emplace_back([&, t] {                              // ticket callers: a FIFO of parked operations
        struct fl { uint64_t a, token; };
        std::vector<fl> q(inflight);
        size_t head = 0, count = 0;
        alignas(16) uint8_t item[512];
        std::vector<uint8_t> seg(AGR_OUT_TICKET_MAX_BYTES);
        uint64_t issued = 0;
        while (issued < per_thread || count) {
            while (issued < per_thread && count < q.size()) {
                uint64_t token = mix(((uint64_t)(t + 1000) << 40) | issued);
                memset(item, 0, sizeof item); memcpy(item, &token, 8);
                uint64_t a;
                const uint32_t pick = (uint32_t)(issued % 4u);
                if (pick >= 2u) {                                         // outcomes with bytes: inline or a span
                    const uint32_t len = seg_len(token), hl = (uint32_t)((token >> 24) % (len + 1u));
                    fill(seg.data(), len, token);
                    // all in the first part, or split between headers and body
                    const uint32_t a_len = pick == 2u ? len : hl;
                    if (!svc_submit_outcome_span(&S, item, hl, seg.data(), a_len, seg.data() + a_len, len - a_len, &a)) { eagain++; break; }
                    token ^= bytes_key(hl, len, seg.data());
                } else if (!svc_submit_one(&S, pick == 0u ? SVC_OP_RECORD : SVC_OP_OUTCOME, item, pick == 0u ? sizeof item : 64u, &a)) {
                    eagain++; break;                                      // AGR_EAGAIN: collect, come again
                }
                q[(head + count) % q.size()] = fl{a, token}; count++; issued++;
            }
            uint32_t reaped = 0;
            while (count && reaped < 64) {
                svc_answer r;
                if (!svc_try(&S, q[head].a, &r)) break;
                check(q[head].a, q[head].token, r);
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
    printf("{\"blocking_threads\": %d, \"ticket_threads\": %d, \"inflight\": %u, \"operations\": %llu, \"served\": %llu, \"spans\": %llu, "
           "\"span_slots\": %llu, \"wrapped_spans\": %llu, \"max_staged\": %llu, \"skipped_slots\": %llu, \"eagain\": %llu, "
           "\"wrong_answers\": %llu, \"seconds\": %.3f, \"ok\": %s}\n",
           nb, nt, inflight, (unsigned long long)done_ops.load(), (unsigned long long)served.load(), (unsigned long long)spans.load(),
           (unsigned long long)span_slots.load(), (unsigned long long)wrapped.load(), (unsigned long long)max_staged.load(),
           (unsigned long long)skipped.load(), (unsigned long long)eagain.load(), (unsigned long long)bad.load(), secs, ok ? "true" : "false");
    return ok ? 0 : 1;
}
