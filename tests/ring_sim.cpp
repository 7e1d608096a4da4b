// ring_sim.cpp — the callers' side of the single-request ring (csrc/agr_ring.hpp: the code the library ships) against a
// stand-in for the dispatcher and the service kernel, on the CPU.  Checks the protocol, not the GPU:
//   * every operation handed over is answered exactly once, with the answer computed from ITS OWN payload (a slot reused
//     before its previous answer was collected, or a payload overwritten before it was consumed, shows up as a wrong token);
//   * ticket holders that together hold more tickets than the ring has slots make progress and finish (a submit never waits
//     for another caller's ticket: AGR_EAGAIN instead — the first version of the ring deadlocked here);
//   * blocking callers and ticket callers can share one ring;
//   * a record's answer names its full 64-bit row although the answer carries only the low 48 bits: the stand-in hands out
//     row base + slot number (base near 2^48 puts the rows across that edge) and every caller checks the row it gets.
// usage: ring_sim <blocking threads> <ticket threads> <tickets in flight per ticket thread> <operations per thread> [service delay us]
//        [row base]
// prints one JSON line; exit code 0 = every check passed.  Test infrastructure (tests/test_ring_sim.py), no CUDA.
#include <stdio.h>
#include <stdlib.h>
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
    std::atomic<uint64_t> rows_out{0};
    std::mutex smu; std::condition_variable scv;
};

static inline uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; return x ^ (x >> 33); }

int main(int argc, char** argv) {
    const int nb = argc > 1 ? atoi(argv[1]) : 4, nt = argc > 2 ? atoi(argv[2]) : 4;
    const uint32_t inflight = argc > 3 ? (uint32_t)atoi(argv[3]) : 512u;
    const uint64_t per_thread = argc > 4 ? strtoull(argv[4], nullptr, 10) : 200000ULL;
    const int delay_us = argc > 5 ? atoi(argv[5]) : 0;
    const uint64_t row_base = argc > 6 ? strtoull(argv[6], nullptr, 0) : 0ULL;
    sim_host S;
    S.rows_out.store(row_base);
    S.res = (svc_res*)aligned_alloc(64, sizeof(svc_res) * SVC_SLOTS); memset((void*)S.res, 0, sizeof(svc_res) * SVC_SLOTS);
    S.payload = (uint8_t*)aligned_alloc(64, (size_t)SVC_SLOTS * SVC_PAYLOAD); memset(S.payload, 0, (size_t)SVC_SLOTS * SVC_PAYLOAD);
    S.ready = new std::atomic<uint32_t>[SVC_SLOTS];
    for (uint32_t i = 0; i < SVC_SLOTS; ++i) S.ready[i].store(0);
    std::atomic<bool> quit{false};
    std::atomic<uint64_t> served{0}, skipped{0}, bad{0}, bad_rows{0}, eagain{0}, done_ops{0};

    // dispatcher + service kernel in one thread: consume the published prefix in slot order (like svc_dispatcher), in batches of
    // up to SVC_MAX_OPS, answer every real operation with ONE 16-byte result whose last word carries the lap tag (like k_svc)
    std::thread service([&] {
        uint64_t to = 0;
        while (!quit.load(std::memory_order_acquire)) {
            const uint64_t from = to;
            uint32_t nrec = 0, kinds[SVC_MAX_OPS / 16] = {0};
            svc_scan(&S, from, &to, &nrec, kinds, 128u);                               // the dispatcher's own scan (agr_ring.hpp)
            if (to == from) { std::this_thread::yield(); continue; }
            S.rows_out.store(row_base + to, std::memory_order_release);            // (the dispatcher: rows reserved, then the batch goes out)
            if (delay_us) std::this_thread::sleep_for(std::chrono::microseconds(delay_us));     // the batch is "on the GPU"
            for (uint64_t a = from; a < to; ++a) {
                const uint32_t slot = (uint32_t)(a & (SVC_SLOTS - 1u));
                const uint32_t kind = (kinds[(a - from) >> 4] >> (((a - from) & 15u) * 2u)) & 3u;
                if (kind == SVC_OP_SKIP) { skipped++; continue; }
                uint64_t token; memcpy(&token, S.payload + (size_t)slot * SVC_PAYLOAD, 8);
                const uint64_t ans = mix(token ^ a);                                   // depends on the payload AND the slot number
                svc_res* r = S.res + slot;
                __atomic_store_n(&r->w[0], (uint32_t)ans | 1u, __ATOMIC_RELAXED); __atomic_store_n(&r->w[1], (uint32_t)(ans >> 32), __ATOMIC_RELAXED);
                const uint64_t row = row_base + a;                                     // a record's row: its low 48 bits, as k_svc writes them
                const bool rec = kind == SVC_OP_RECORD;
                __atomic_store_n(&r->w[2], rec ? (uint32_t)row : (uint32_t)kind, __ATOMIC_RELAXED);
                __atomic_store_n(&r->w[3], (svc_tag(a) << 16) | (rec ? (uint32_t)((row >> 32) & 0xffffu) : 0u), __ATOMIC_RELEASE);   // (the kernel: one 16-byte store)
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
        for (uint64_t i = 0; i < per_thread; ++i) {
            const uint64_t token = mix(((uint64_t)t << 40) | i);
            memset(item, 0, sizeof item); memcpy(item, &token, 8);
            uint64_t a;
            while (!svc_submit_one(&S, t == 0 ? SVC_OP_RECORD : SVC_OP_OUTCOME, item, sizeof item, &a)) {}
            svc_answer r; svc_wait(&S, a, &r);
            check(a, token, r);
            if (t == 0 && svc_row(&S, r) != row_base + a) {                                      // (blocking thread 0 hands over records)
                if (bad_rows.fetch_add(1) < 4) fprintf(stderr, "slot %llu: row %llu, want %llu\n", (unsigned long long)a, (unsigned long long)svc_row(&S, r), (unsigned long long)(row_base + a));
            }
            svc_release(&S, a);
            done_ops++;
        }
    });
    for (int t = 0; t < nt; ++t) ths.emplace_back([&, t] {                              // ticket callers: a FIFO of parked operations
        struct fl { uint64_t a, token; };
        std::vector<fl> q(inflight);
        size_t head = 0, count = 0;
        alignas(16) uint8_t item[512];
        uint64_t issued = 0;
        while (issued < per_thread || count) {
            while (issued < per_thread && count < q.size()) {
                const uint64_t token = mix(((uint64_t)(t + 1000) << 40) | issued);
                memset(item, 0, sizeof item); memcpy(item, &token, 8);
                uint64_t a;
                if (!svc_submit_one(&S, SVC_OP_RECORD, item, sizeof item, &a)) { eagain++; break; }   // AGR_EAGAIN: collect, come again
                q[(head + count) % q.size()] = fl{a, token}; count++; issued++;
            }
            uint32_t reaped = 0;
            while (count && reaped < 64) {
                svc_answer r;
                if (!svc_try(&S, q[head].a, &r)) break;
                check(q[head].a, q[head].token, r);
                if (svc_row(&S, r) != row_base + q[head].a) bad_rows++;
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
    const bool ok = bad.load() == 0 && bad_rows.load() == 0 && done_ops.load() == want && served.load() == want;
    printf("{\"blocking_threads\": %d, \"ticket_threads\": %d, \"inflight\": %u, \"operations\": %llu, \"served\": %llu, \"skipped_slots\": %llu, "
           "\"eagain\": %llu, \"wrong_answers\": %llu, \"wrong_rows\": %llu, \"row_base\": %llu, \"last_row\": %llu, \"seconds\": %.3f, \"ok\": %s}\n",
           nb, nt, inflight, (unsigned long long)done_ops.load(), (unsigned long long)served.load(), (unsigned long long)skipped.load(),
           (unsigned long long)eagain.load(), (unsigned long long)bad.load(), (unsigned long long)bad_rows.load(),
           (unsigned long long)row_base, (unsigned long long)(S.rows_out.load() - 1), secs, ok ? "true" : "false");
    return ok ? 0 : 1;
}
