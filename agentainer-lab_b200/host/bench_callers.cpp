// bench_callers.cpp — the reference's real call pattern at the C-ABI: one OS thread per in-flight HTTP request
// (net/http's goroutine per connection -> proxyToAgentHandler, internal/api/server.go:493-573), every thread doing
//     agr_ingest_ex(n = 1)  ->  [forward]  ->  agr_complete(n = 1)
// i.e. StoreRequest + the routing decision, then StoreResponse (server.go:508-518, 588-594), through the single-request
// front end (AGR_CFG_COMBINE).  Prints ONE JSON object: round trips per second, p50 / p99 latency of a round trip.
// With <inflight> > 0 every thread keeps that many requests in flight through the ticket calls (agr_submit_ingest ->
// agr_poll -> agr_submit_complete -> agr_poll): the goroutine-per-request pattern of a Go host, where a request parks instead
// of pinning an OS thread (INTEGRATION.md).  Every request is still handed over one at a time.
// With <bytes> = store | fused every StoreResponse keeps a response of 64 B of flattened headers plus <body> bytes of body
// (requests.go:134-175): store = today's pattern, the completion (blocking call or ticket) and then agr_store_response;
// fused = the bytes travel with the completion, agr_submit_complete_ex (tickets) or agr_complete_ex(n = 1) (blocking), and a
// body above AGR_OUT_INLINE_BYTES falls back to the locked agr_complete_ex(n = 1); large = the same with
// agr_submit_complete_large (blocking threads: it and agr_wait), which carries up to AGR_OUT_TICKET_MAX_BYTES in one ticket.
// With mode `var` the engine holds VARIABLE-LENGTH records (AGR_CFG_VARLEN) with chat bodies of 128 B - 4 KiB, log-uniform and
// seeded per thread (BASELINE config 5): with <inflight> > 0 the ticket arm (AGR_CFG_COMBINE: agr_submit_ingest of the record ->
// agr_poll -> agr_submit_complete -> agr_poll), with 0 the locked arm a variable-length deployment has without the ring
// (agr_ingest_var(n = 1) -> agr_complete(n = 1), each taking the handle mutex and synchronising the stream).  A <body> given
// with `var` makes every body that long instead.
//   bench_callers <threads> <seconds> [device] [mint|hash] [agents] [inflight per thread, 0 = blocking calls] [none|store|fused|large|var] [body]
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <string>
#include <thread>
#include <vector>

#include "../../include/agentainer_gpu.h"

static uint64_t splitmix(uint64_t& x) {
    uint64_t z = (x += 0x9e3779b97f4a7c15ULL);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL; z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    return z ^ (z >> 31);
}

int main(int argc, char** argv) {
    const int threads = argc > 1 ? atoi(argv[1]) : 64;
    const double seconds = argc > 2 ? atof(argv[2]) : 2.0;
    const int device = argc > 3 ? atoi(argv[3]) : 0;
    const bool mint = !(argc > 4 && strcmp(argv[4], "hash") == 0);
    const int n_agents = argc > 5 ? atoi(argv[5]) : 256;
    const int inflight = argc > 6 ? atoi(argv[6]) : 0;
    const int bytes_mode = argc > 7 ? (strcmp(argv[7], "store") == 0 ? 1 : strcmp(argv[7], "fused") == 0 ? 2 : strcmp(argv[7], "large") == 0 ? 3 : 0) : 0;
    const uint32_t body_len = argc > 8 ? (uint32_t)atoi(argv[8]) : 256u;
    const bool var = argc > 7 && strcmp(argv[7], "var") == 0;
    const uint32_t var_body = var && argc > 8 ? (uint32_t)atoi(argv[8]) : 0u;   // var: every body this long (0: the log-uniform mix)
    static constexpr char kHdr[] = "Content-Type: application/json\nX-Trace-Id: 0123456789abcdef0123\n";
    static_assert(sizeof kHdr - 1 == 64, "64 B of headers");
    const std::string hdr = kHdr;
    const std::vector<uint8_t> body(body_len, (uint8_t)'x');
    std::string seg = hdr; seg.append(body.begin(), body.end());
    const uint64_t seg_off[2] = {0, seg.size()};
    const uint32_t seg_hlen = (uint32_t)hdr.size();
    const bool ticket_fits = seg.size() <= (bytes_mode == 3 ? AGR_OUT_TICKET_MAX_BYTES : AGR_OUT_INLINE_BYTES);
    agr_config cfg; memset(&cfg, 0, sizeof cfg);
    cfg.device = device;
    cfg.slab_rows = 1ull << 26;                         // 64 Mi rows = 32 GiB of slab (~43 GB with the per-row arrays)
    cfg.max_agents = 1024; cfg.max_batch = 1u << 16; cfg.log_entries = cfg.slab_rows;
    cfg.resp_bytes = bytes_mode ? 8ull << 30 : 1 << 20;               // append-only: room for a few seconds of stored responses
    if (bytes_mode == 3) {                              // bodies up to 16 KB arrive at GB/s: half the rows, four times the bytes
        cfg.slab_rows = 1ull << 25; cfg.log_entries = cfg.slab_rows; cfg.resp_bytes = 32ull << 30;
    }
    cfg.flags = AGR_CFG_PERSISTENCE | AGR_CFG_COMBINE | (mint ? AGR_CFG_MINT_IDS : 0u);
    if (var) {                                          // ~1.4 KiB per record on average: 16 Mi rows, 24 GiB of record bytes
        cfg.slab_rows = 1ull << 24; cfg.log_entries = cfg.slab_rows; cfg.vslab_bytes = 24ull << 30;
        cfg.flags = AGR_CFG_PERSISTENCE | AGR_CFG_VARLEN | (inflight > 0 ? AGR_CFG_COMBINE : 0u) | (mint ? AGR_CFG_MINT_IDS : 0u);
    }
    agr_handle* h = nullptr;
    if (agr_create(&cfg, &h) < 0) { fprintf(stderr, "agr_create: %s\n", agr_last_error()); return 2; }
    agr_synth sy; memset(&sy, 0, sizeof sy); sy.seed = 7; sy.n_agents = (uint32_t)n_agents;
    std::vector<std::string> names;
    for (int k = 0; k < n_agents; ++k) {
        char id[AGR_AGENT_ID_BYTES]; agr_synth_agent_id(&sy, (uint32_t)k, id);
        names.emplace_back(id);
        if (agr_set_agent_state(h, id, AGR_AGENT_RUNNING) < 0) { fprintf(stderr, "set_agent_state: %s\n", agr_last_error()); return 2; }
    }
    std::atomic<bool> go{false}, stop{false};
    std::atomic<uint64_t> total{0}, bad{0}, vbytes{0};
    std::vector<std::vector<uint32_t>> lat(threads);
    std::vector<std::thread> ths;
    for (int t = 0; t < threads; ++t) ths.emplace_back([&, t] {
        // every thread sends the synthetic stream's records (BASELINE's 512 B POST /agent/<id>/chat shape), one per call
        std::vector<agr_record> recs(64);
        agr_synth s2 = sy; s2.seed = 1000 + t;
        agr_synth_fill_host(&s2, 0, 64, recs.data());
        uint64_t x = 0x1234 + t, n = 0;
        auto& my = lat[t]; my.reserve(1 << 20);
        // var: the same records as variable-length ones, each with its own body (one 8 KiB cell per record)
        std::vector<uint8_t> vrec(var ? 64u * AGR_VAR_MAX_RECORD : 0u, (uint8_t)'x');
        std::vector<uint32_t> vlen(var ? 64u : 0u);
        for (uint32_t k = 0; var && k < 64u; ++k) {
            uint8_t* p = vrec.data() + (size_t)k * AGR_VAR_MAX_RECORD;
            const agr_record& r = recs[k];
            const uint32_t ph = (uint32_t)r.path_len + r.hdr_len;
            const double u = (double)(splitmix(x) >> 11) * (1.0 / 9007199254740992.0);
            uint32_t blen = var_body ? var_body : (uint32_t)(128.0 * std::exp(u * std::log(32.0)));   // or log-uniform in [128, 4096]
            blen = std::min<uint32_t>(blen, AGR_VAR_MAX_RECORD - AGR_HEADER_BYTES - ph);
            memcpy(p, &r, AGR_HEADER_BYTES);
            memcpy(p + AGR_HEADER_BYTES, r.payload, ph);
            memcpy(p + offsetof(agr_record, body_len), &blen, 4);
            vlen[k] = AGR_HEADER_BYTES + ((ph + blen + 15u) & ~15u);
            memset(p + AGR_HEADER_BYTES + ph + blen, 0, vlen[k] - AGR_HEADER_BYTES - ph - blen);
            vbytes += vlen[k];
        }
        while (!go.load(std::memory_order_acquire)) std::this_thread::yield();
        auto record_of = [&](uint32_t k) -> agr_record* {               // record k of this thread, with a fresh id and seq
            agr_record* r = var ? reinterpret_cast<agr_record*>(vrec.data() + (size_t)k * AGR_VAR_MAX_RECORD) : &recs[k];
            if (!mint) { uint64_t a = splitmix(x), b = splitmix(x) | 1; memcpy(r->request_id, &a, 8); memcpy(r->request_id + 8, &b, 8); }
            r->seq = n;
            return r;
        };
        if (inflight > 0) {
            // Tickets are answered in hand-over order (batch by batch), so the thread keeps its requests in a FIFO and polls only
            // the OLDEST one: a poll that says "not yet" means nothing younger is ready either.
            // stage 0: ingest ticket, 1: completion ticket, 2 (large): a completion waiting to be handed over again
            struct flight { int stage; agr_ticket t; std::chrono::steady_clock::time_point t0; uint32_t rec; uint8_t rid[16]; agr_outcome o; };
            std::vector<flight> q((size_t)inflight);
            size_t head = 0, count = 0;                                   // FIFO over q: [head, head + count)
            auto push = [&](const flight& f) { q[(head + count) % q.size()] = f; count++; };
            while (!stop.load(std::memory_order_relaxed)) {
                while (count < q.size()) {                                 // start requests: StoreRequest + routing decision
                    flight f; f.rec = (uint32_t)(n & 63); agr_record& r = *record_of(f.rec);
                    f.t0 = std::chrono::steady_clock::now();
                    const int rc = agr_submit_ingest(h, &r, &f.t);
                    if (rc == AGR_EAGAIN) break;
                    if (rc < 0) { bad++; stop.store(true); break; }
                    f.stage = 0; n++;
                    push(f);
                }
                uint32_t reaped = 0;
                while (count && reaped < 64) {
                    flight f = q[head];
                    if (f.stage == 2) {
                        head = (head + 1) % q.size(); count--;
                        const int rc2 = agr_submit_complete_large(h, &f.o, (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len, &f.t);
                        if (rc2 < 0) { bad++; stop.store(true); break; }
                        if (rc2 == AGR_EAGAIN) { push(f); break; }           // still no room: collect more first
                        f.stage = 1; push(f); reaped++;
                        continue;
                    }
                    agr_result res;
                    const int rc = agr_poll(h, f.t, &res);
                    if (rc == AGR_EAGAIN) break;
                    head = (head + 1) % q.size(); count--; reaped++;
                    if (rc < 0 || res.result != 0) { bad++; stop.store(true); break; }
                    if (f.stage == 0) {                                    // forwarded: the agent answered, StoreResponse
                        if (res.verdict.code != AGR_V_FORWARD) { bad++; stop.store(true); break; }
                        agr_outcome o; memset(&o, 0, sizeof o);
                        memcpy(o.request_id, res.request_id, 16); memcpy(o.agent_id, recs[f.rec].agent_id, AGR_AGENT_ID_BYTES);
                        o.kind = AGR_OUT_RESPONSE; o.http_status = 200; o.seq = n;
                        if (bytes_mode >= 2 && !ticket_fits) {                // too big for a ticket: the locked batch call, n = 1
                            int32_t r1 = -1;
                            if (agr_complete_ex(h, &o, 1, (const uint8_t*)seg.data(), seg_off, &seg_hlen, &r1) < 0 || r1 != 0) { bad++; stop.store(true); break; }
                            const auto t1 = std::chrono::steady_clock::now();
                            if (my.size() < my.capacity()) my.push_back((uint32_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - f.t0).count());
                            continue;
                        }
                        int rc2;
                        if (bytes_mode == 3) {
                            // a span needs up to 33 free slots in a row, and the thread's own uncollected tickets may be among
                            // them: on AGR_EAGAIN collect first, as the header asks, and hand it over again when it comes round
                            memcpy(&f.rid, o.request_id, 16); f.o = o;
                            rc2 = agr_submit_complete_large(h, &o, (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len, &f.t);
                            if (rc2 < 0) { bad++; stop.store(true); break; }
                            f.stage = rc2 == AGR_EAGAIN ? 2 : 1;
                            push(f);
                            continue;
                        }
                        // AGR_EAGAIN: the slot drawn still holds somebody's uncollected answer; the next draw is another slot
                        while ((rc2 = (bytes_mode == 2 ? agr_submit_complete_ex(h, &o, (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len, &f.t)
                                                       : agr_submit_complete(h, &o, &f.t))) == AGR_EAGAIN && !stop.load(std::memory_order_relaxed)) {}
                        if (rc2 == AGR_EAGAIN) break;                      // the run is over: this request stays forwarded-but-uncompleted
                        if (rc2 < 0) { bad++; stop.store(true); break; }
                        f.stage = 1;
                        memcpy(&f.rid, o.request_id, 16);
                        push(f);
                    } else {
                        if (bytes_mode == 1 && agr_store_response(h, recs[f.rec].agent_id, f.rid, (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len) < 0) {
                            bad++; stop.store(true); break;
                        }
                        const auto t1 = std::chrono::steady_clock::now();
                        if (my.size() < my.capacity()) my.push_back((uint32_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - f.t0).count());
                    }
                }
            }
            while (count) { agr_result res; if (q[head].stage != 2) agr_wait(h, q[head].t, &res); head = (head + 1) % q.size(); count--; }   // drain
            total += n;
            return;
        }
        while (!stop.load(std::memory_order_relaxed)) {
            agr_record& r = *record_of((uint32_t)(n & 63));
            agr_verdict v; uint8_t id[1][16]; uint64_t first;
            const auto t0 = std::chrono::steady_clock::now();
            if (var) {
                const uint32_t off[2] = {0u, vlen[n & 63]};
                if (agr_ingest_var(h, reinterpret_cast<const uint8_t*>(&r), off, 1, &v, id, &first) < 0 || v.code != AGR_V_FORWARD) { bad++; break; }
            } else if (agr_ingest_ex(h, &r, 1, &v, id, &first) < 0 || v.code != AGR_V_FORWARD) { bad++; break; }
            agr_outcome o; memset(&o, 0, sizeof o);
            memcpy(o.request_id, id[0], 16); memcpy(o.agent_id, r.agent_id, AGR_AGENT_ID_BYTES);
            o.kind = AGR_OUT_RESPONSE; o.http_status = 200; o.seq = n + 1;
            int32_t res = -1;
            if (bytes_mode == 3 && ticket_fits) {
                agr_ticket tk; agr_result rr; int rc2;
                while ((rc2 = agr_submit_complete_large(h, &o, (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len, &tk)) == AGR_EAGAIN) {}
                if (rc2 < 0 || agr_wait(h, tk, &rr) < 0 || rr.result != 0) { bad++; break; }
            } else if (bytes_mode >= 2) {
                if (agr_complete_ex(h, &o, 1, (const uint8_t*)seg.data(), seg_off, &seg_hlen, &res) < 0 || res != 0) { bad++; break; }
            } else {
                if (agr_complete(h, &o, 1, &res) < 0 || res != 0) { bad++; break; }
                if (bytes_mode == 1 && agr_store_response(h, r.agent_id, id[0], (const uint8_t*)hdr.data(), seg_hlen, body.data(), body_len) < 0) { bad++; break; }
            }
            const auto t1 = std::chrono::steady_clock::now();
            if (my.size() < my.capacity()) my.push_back((uint32_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count());
            n++;
        }
        total += n;
    });
    // warm-up: let the dispatcher and the resident kernel come up, then measure
    go.store(true, std::memory_order_release);
    std::this_thread::sleep_for(std::chrono::milliseconds(300));
    for (auto& v : lat) v.clear();                      // (racy by design: warm-up samples may survive; they are few)
    agr_stats s0; agr_stats_get(h, &s0);
    const auto t0 = std::chrono::steady_clock::now();
    std::this_thread::sleep_for(std::chrono::duration<double>(seconds));
    agr_stats s1; agr_stats_get(h, &s1);
    const auto t1 = std::chrono::steady_clock::now();
    stop.store(true);
    for (auto& th : ths) th.join();
    const double secs = std::chrono::duration<double>(t1 - t0).count();
    // every round trip is one stored request + one completion: count them on the ENGINE's side of the boundary
    const double rt = (double)(s1.completions - s0.completions);
    std::vector<uint32_t> all;
    for (auto& v : lat) all.insert(all.end(), v.begin(), v.end());
    std::sort(all.begin(), all.end());
    auto pct = [&](double p) { return all.empty() ? 0.0 : all[(size_t)std::min<double>(all.size() - 1, p * all.size())] / 1000.0; };
    agr_stats s2; agr_stats_get(h, &s2);
    if (!var)
    printf("{\"threads\": %d, \"seconds\": %.3f, \"round_trips\": %.0f, \"round_trips_per_s\": %.1f, \"ops_per_s\": %.1f, "
           "\"p50_us\": %.2f, \"p99_us\": %.2f, \"latency_samples\": %zu, \"svc_batches\": %llu, \"ops_per_batch\": %.1f, "
           "\"id_mode\": \"%s\", \"agents\": %d, \"inflight_per_thread\": %d, \"response_bytes\": \"%s\", \"hdr_bytes\": %u, \"body_bytes\": %u, \"errors\": %llu, \"stored\": %llu, \"completions\": %llu, \"host_cpus\": %u}\n",
           threads, secs, rt, rt / secs, 2.0 * rt / secs, pct(0.50), pct(0.99), all.size(),
           (unsigned long long)(s1.svc_batches - s0.svc_batches), (double)(s1.svc_ops - s0.svc_ops) / std::max<double>(1.0, (double)(s1.svc_batches - s0.svc_batches)),
           mint ? "mint" : "hash", n_agents, inflight, bytes_mode == 0 ? "none" : bytes_mode == 1 ? "store" : bytes_mode == 2 ? "fused" : "large",
           bytes_mode ? seg_hlen : 0u, bytes_mode ? body_len : 0u, (unsigned long long)bad.load(), (unsigned long long)s2.stored, (unsigned long long)s2.completions,
           std::thread::hardware_concurrency());
    if (var)
        printf("{\"threads\": %d, \"seconds\": %.3f, \"round_trips_per_s\": %.1f, \"p50_us\": %.2f, \"p99_us\": %.2f, \"latency_samples\": %zu, "
               "\"svc_batches\": %llu, \"arm\": \"%s\", \"id_mode\": \"%s\", \"inflight_per_thread\": %d, \"record_bytes_mean\": %.0f, "
               "\"errors\": %llu}\n",
               threads, secs, rt / secs, pct(0.50), pct(0.99), all.size(), (unsigned long long)(s1.svc_batches - s0.svc_batches),
               inflight > 0 ? "ticket" : "locked", mint ? "mint" : "hash", inflight, (double)vbytes.load() / (64.0 * threads),
               (unsigned long long)bad.load());
    agr_destroy(h);
    return bad.load() ? 1 : 0;
}
