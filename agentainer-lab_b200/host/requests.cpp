// requests.cpp — see requests.hpp.  Thin: every state change is a C-ABI call; nothing is decided on the host.
#include "requests.hpp"
#include <mutex>
#include <stdexcept>
#include <algorithm>

#include <chrono>
#include <cstring>
#include <random>

namespace agentainer {
namespace requests {

const char* StatusString(RequestStatus s) {
    switch (s) { case RequestStatus::Pending: return "pending"; case RequestStatus::Processing: return "processing";
                 case RequestStatus::Completed: return "completed"; default: return "failed"; }
}
std::string FormatUUID(const uint8_t id[16]) {
    static const char* hex = "0123456789abcdef";
    std::string s;
    for (int i = 0; i < 16; ++i) { if (i == 4 || i == 6 || i == 8 || i == 10) s.push_back('-'); s.push_back(hex[id[i] >> 4]); s.push_back(hex[id[i] & 15]); }
    return s;
}
bool ParseUUID(const std::string& s, uint8_t id[16]) {
    int n = 0, hi = -1;
    for (char c : s) {
        if (c == '-') continue;
        int v = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : (c >= 'A' && c <= 'F') ? c - 'A' + 10 : -1;
        if (v < 0 || n >= 16) return false;
        if (hi < 0) hi = v; else { id[n++] = (uint8_t)((hi << 4) | v); hi = -1; }
    }
    return n == 16 && hi < 0;
}
static void mint_uuid(uint8_t id[16]) {                      // uuid.New() (requests.go:87): random v4
    static thread_local std::mt19937_64 rng{std::random_device{}()};
    uint64_t a = rng(), b = rng();
    memcpy(id, &a, 8); memcpy(id + 8, &b, 8);
    id[6] = (uint8_t)((id[6] & 0x0f) | 0x40); id[8] = (uint8_t)((id[8] & 0x3f) | 0x80);
}
static uint32_t method_code(const std::string& m) {
    static const char* names[] = {"", "GET", "POST", "PUT", "DELETE", "PATCH", "HEAD", "OPTIONS"};
    for (uint32_t c = 1; c < 8; ++c) if (m == names[c]) return c;
    return 0;
}
static const char* method_name(uint32_t flags) {
    static const char* names[] = {"", "GET", "POST", "PUT", "DELETE", "PATCH", "HEAD", "OPTIONS"};
    uint32_t c = (flags & AGR_F_METHOD_MASK) >> AGR_F_METHOD_SHIFT;
    return c < 8 ? names[c] : "";
}

void Manager::ToRecord(const std::string& agentID, const HttpRequest& req, const uint8_t id[16], bool replay,
                       const uint8_t replay_of[16], uint64_t seq, agr_record* rec) {
    memset(rec, 0, sizeof *rec);
    memcpy(rec->request_id, id, 16);
    if (replay && replay_of) memcpy(rec->replay_of, replay_of, 16);
    strncpy(rec->agent_id, agentID.c_str(), AGR_AGENT_ID_BYTES - 1);
    rec->seq = seq;
    rec->flags = (replay ? AGR_F_REPLAY : 0u) | (method_code(req.Method) << AGR_F_METHOD_SHIFT);
    std::string hdrs;
    for (const auto& kv : req.Header) {                      // std::map iterates sorted by key, like encoding/json
        if (kv.first == "X-Agentainer-Replay" || kv.first == "X-Agentainer-Request-ID") continue;
        hdrs += kv.first + ": " + kv.second + "\n";
    }
    size_t room = AGR_PAYLOAD_BYTES, p = std::min(room, req.Path.size());
    memcpy(rec->payload, req.Path.data(), p); room -= p;
    size_t hl = std::min(room, hdrs.size());
    memcpy(rec->payload + p, hdrs.data(), hl); room -= hl;
    size_t bl = std::min(room, req.Body.size());             // fixed-stride build: longer bodies need the
    memcpy(rec->payload + p + hl, req.Body.data(), bl);      // variable-length slab (DESIGN.md section 7)
    rec->path_len = (uint16_t)p; rec->hdr_len = (uint16_t)hl; rec->body_len = (uint32_t)bl;
    rec->status = AGR_ST_PENDING; rec->max_retries = 3;      // requests.go:93-95
}
void Manager::FromRecord(const agr_record& r, Request* out) {
    out->ID = FormatUUID(r.request_id);
    out->AgentID.assign(r.agent_id, strnlen(r.agent_id, AGR_AGENT_ID_BYTES));
    out->Method = method_name(r.flags);
    out->Path.assign((const char*)r.payload, r.path_len);
    out->Headers.clear();
    const char* h = (const char*)r.payload + r.path_len; const char* e = h + r.hdr_len;
    while (h < e) {
        const char* nl = (const char*)memchr(h, '\n', (size_t)(e - h)); if (!nl) nl = e;
        const char* colon = (const char*)memchr(h, ':', (size_t)(nl - h));
        if (colon) { const char* v = colon + 1; if (v < nl && *v == ' ') ++v; out->Headers[std::string(h, colon)] = std::string(v, nl); }
        h = nl + 1;
    }
    out->Body.assign(r.payload + r.path_len + r.hdr_len, r.payload + r.path_len + r.hdr_len + r.body_len);
    out->Status = r.status == AGR_ST_COMPLETED ? RequestStatus::Completed : r.status == AGR_ST_FAILED ? RequestStatus::Failed
                  : r.status == AGR_ST_PROCESSING ? RequestStatus::Processing : RequestStatus::Pending;
    out->RetryCount = r.retry_count; out->MaxRetries = r.max_retries; out->CreatedAt = r.seq;
    out->ResponseStatus = r.resp_status;
    out->Error = r.error_code ? "transport error" : "";
}

// one shared handle per process (a14): the first Manager registers its handle, later ones must bring the same
static std::mutex g_handle_mu;
static agr_handle* g_process_handle = nullptr;
static int g_managers = 0;
Manager::Manager(agr_handle* h, bool engine_mints_ids) : h_(h), mint_(engine_mints_ids) {
    std::lock_guard<std::mutex> lk(g_handle_mu);
    if (g_managers > 0 && g_process_handle != h)
        throw std::logic_error("requests.Manager: a second engine handle in one process — the server's and the replay worker's "
                               "managers must share ONE handle (server.go:62, main.go:335)");
    g_process_handle = h;
    g_managers++;
}
Manager::~Manager() {
    std::lock_guard<std::mutex> lk(g_handle_mu);
    if (--g_managers == 0) g_process_handle = nullptr;
}
agr_handle* Manager::ProcessHandle() {
    std::lock_guard<std::mutex> lk(g_handle_mu);
    return g_process_handle;
}

Error Manager::Decide(const std::string& agentID, const HttpRequest& req, Verdict* out) {
    auto it = req.Header.find("X-Agentainer-Replay");
    const bool replay = it != req.Header.end() && it->second == "true";                  // server.go:506
    uint8_t id[16], of[16] = {0};
    mint_uuid(id);
    if (replay) { auto r = req.Header.find("X-Agentainer-Request-ID"); if (r != req.Header.end()) ParseUUID(r->second, of); }   // :519-522
    agr_record rec; agr_verdict v;
    ToRecord(agentID, req, id, replay, of, now(), &rec);
    uint8_t minted[1][16];
    int rc = agr_ingest_ex(h_, &rec, 1, &v, minted, nullptr);
    if (rc < 0) return std::string("failed to store request: ") + agr_last_error();
    if (mint_) memcpy(id, minted[0], 16);                                                // storedReq.ID (server.go:515)
    out->Code = v.code; out->HTTPStatus = v.http_status; out->Stored = (v.flags & AGR_VF_STORED) != 0;
    out->RequestID = !(v.flags & AGR_VF_TRACKED) ? "" : replay ? FormatUUID(of) : FormatUUID(id);
    return "";
}
Error Manager::StoreRequest(const std::string& agentID, const HttpRequest& req, Request* out) {
    HttpRequest fresh = req;
    fresh.Header.erase("X-Agentainer-Replay");
    Verdict v;
    Error e = Decide(agentID, fresh, &v);
    if (!e.empty()) return e;
    if (v.Code == AGR_V_NOT_FOUND) return "failed to store request: agent not found";
    if (!v.Stored) return "failed to store request: duplicate request id";
    uint8_t id[16]; ParseUUID(v.RequestID, id);
    agr_record rec;
    if (agr_get_record(h_, agentID.c_str(), id, &rec) < 0) return std::string("failed to store request: ") + agr_last_error();
    if (out) FromRecord(rec, out);
    return "";
}
Error Manager::complete(const std::string& agentID, const std::string& requestID, uint8_t kind, int http) {
    agr_outcome o; memset(&o, 0, sizeof o);
    if (!ParseUUID(requestID, o.request_id)) return "failed to get request: malformed id";
    strncpy(o.agent_id, agentID.c_str(), AGR_AGENT_ID_BYTES - 1);
    o.kind = kind; o.http_status = (uint16_t)http; o.seq = now();
    int32_t res = 0;
    int rc = agr_complete(h_, &o, 1, &res);
    if (rc < 0) return std::string("failed to update request: ") + agr_last_error();
    if (res == AGR_ENOTFOUND) return "failed to get request: redis: nil";                  // requests.go:153-156,232-235
    return "";
}
static std::string flatten(const std::map<std::string, std::string>& h) {      // sorted by key, "Key: Value\n"
    std::string out;
    for (const auto& kv : h) out += kv.first + ": " + kv.second + "\n";
    return out;
}
Error Manager::complete_ex(const std::string& agentID, const std::string& requestID, uint8_t kind, int http, const std::string& seg,
                           uint32_t hdr_len) {
    agr_outcome o; memset(&o, 0, sizeof o);
    if (!ParseUUID(requestID, o.request_id)) return "failed to get request: malformed id";
    strncpy(o.agent_id, agentID.c_str(), AGR_AGENT_ID_BYTES - 1);
    o.kind = kind; o.http_status = (uint16_t)http; o.seq = now();
    const uint64_t offs[2] = {0, seg.size()};
    int32_t res = 0;
    // one call: the transition and the bytes (through the single-request ring when they fit a ticket)
    const int rc = agr_complete_ex(h_, &o, 1, (const uint8_t*)seg.data(), offs, &hdr_len, &res);
    if (rc < 0 && rc != AGR_ENOSPC) return std::string("failed to update request: ") + agr_last_error();
    if (res == AGR_ENOTFOUND) return "failed to get request: redis: nil";                  // requests.go:153-156,232-235
    if (rc == AGR_ENOSPC) return std::string("failed to update request: ") + agr_last_error();
    return "";
}
Error Manager::StoreResponse(const std::string& agentID, const std::string& requestID, const Response& resp) {
    if (resp.Headers.empty() && resp.Body.empty()) return complete(agentID, requestID, AGR_OUT_RESPONSE, resp.StatusCode);   // only the status to keep
    std::string seg = flatten(resp.Headers);                                // requests.go:134-147
    const uint32_t hdr_len = (uint32_t)seg.size();
    seg.append(resp.Body.begin(), resp.Body.end());
    return complete_ex(agentID, requestID, AGR_OUT_RESPONSE, resp.StatusCode, seg, hdr_len);
}
Error Manager::MarkRequestFailed(const std::string& agentID, const std::string& requestID, const std::string& err) {
    return complete_ex(agentID, requestID, AGR_OUT_ERROR, 0, err, 0);       // request.Error = err.Error(), requests.go:244
}
Error Manager::GetRequestJSON(const std::string& agentID, const std::string& requestID, std::string* out) {
    uint8_t id[16];
    if (!ParseUUID(requestID, id)) return "redis: nil";
    uint32_t len = 0;
    out->resize(4096);
    int rc = agr_get_record_json(h_, agentID.c_str(), id, (uint8_t*)&(*out)[0], (uint32_t)out->size(), &len);
    if (rc == AGR_ECAP) { out->resize(len); rc = agr_get_record_json(h_, agentID.c_str(), id, (uint8_t*)&(*out)[0], len, &len); }
    if (rc < 0) { out->clear(); return "redis: nil"; }                      // storage.Get's miss (server.go:662-666)
    out->resize(len);
    return "";
}
Error Manager::GetPendingRequestsJSON(const std::string& agentID, std::string* out, size_t* count) {
    uint64_t len = 0; uint32_t n = 0;
    if (agr_pending_json(h_, agentID.c_str(), nullptr, 0, &len, &n) < 0) return std::string("failed to get pending queue: ") + agr_last_error();
    out->resize(len);
    if (agr_pending_json(h_, agentID.c_str(), (uint8_t*)&(*out)[0], len, &len, &n) < 0) return std::string("failed to get pending queue: ") + agr_last_error();
    out->resize(len);
    if (count) *count = n;
    return "";
}
Error Manager::Reclaim(uint64_t* released) {
    return agr_reclaim(h_, released) < 0 ? std::string("reclaim: ") + agr_last_error() : "";
}
Error Manager::Expire(uint64_t now_ns, uint64_t ttl, uint64_t* expired) {
    return agr_expire(h_, now_ns, ttl, expired) < 0 ? std::string("expire: ") + agr_last_error() : "";
}
Error Manager::RecordTransportError(const std::string& agentID, const std::string& requestID, const std::string& err) {
    // server.go:600-602: substring tests on err.Error()
    const bool dial = err.find("connection refused") != std::string::npos || err.find("no such host") != std::string::npos ||
                      err.find("dial tcp") != std::string::npos;
    return complete(agentID, requestID, dial ? AGR_OUT_DIAL_ERR : AGR_OUT_ERROR, 0);
}
Error Manager::GetPendingRequests(const std::string& agentID, std::vector<Request>* out) {
    uint32_t n = 0, cap = 256;
    std::vector<agr_record> recs;
    for (;;) {
        recs.resize(cap);
        int rc = agr_pending(h_, agentID.c_str(), recs.data(), cap, &n);
        if (rc == AGR_ECAP) { cap = n; continue; }
        if (rc < 0) return std::string("failed to get pending queue: ") + agr_last_error();
        break;
    }
    out->resize(n);
    for (uint32_t i = 0; i < n; ++i) FromRecord(recs[i], &(*out)[i]);
    return "";
}

void ReplayWorker::Start(unsigned interval_ms) {
    stop_ = false;
    th_ = std::thread([this, interval_ms] {
        while (!stop_) {
            for (unsigned t = 0; t < interval_ms && !stop_; t += 10) std::this_thread::sleep_for(std::chrono::milliseconds(10));
            if (!stop_) ProcessAgents();
        }
    });
}
void ReplayWorker::Stop() { stop_ = true; if (th_.joinable()) th_.join(); }

size_t ReplayWorker::ProcessAgents() {
    uint32_t n = 0, cap = 1024;
    std::vector<agr_dispatch> disp; std::vector<agr_record> recs;
    for (;;) {
        disp.resize(cap); recs.resize(cap);
        int rc = agr_replay_scan(m_->handle(), disp.data(), recs.data(), cap, &n);   // KEYS + isAgentRunning + LRANGE + skip rule
        if (rc == AGR_ECAP) { cap = n; continue; }
        if (rc < 0) return 0;
        break;
    }
    for (uint32_t i = 0; i < n; ++i) {                                                // replay_worker.go:99-116, sequential
        Request req; Manager::FromRecord(recs[i], &req);
        const int status = send_(req.AgentID, req);                                   // replayRequest's HTTP call (:151)
        if (status < 0) m_->MarkRequestFailed(req.AgentID, req.ID, "request failed"); // :109-112
        else { Response r; r.StatusCode = status; m_->StoreResponse(req.AgentID, req.ID, r); }   // :158 (second completion, Q7)
    }
    return n;
}

size_t ReplayWorker::ProcessAgentsConcurrent(unsigned workers) {
    uint32_t n = 0, cap = 1024;
    std::vector<agr_dispatch> disp; std::vector<agr_record> recs;
    for (;;) {
        disp.resize(cap); recs.resize(cap);
        int rc = agr_replay_scan(m_->handle(), disp.data(), recs.data(), cap, &n);
        if (rc == AGR_ECAP) { cap = n; continue; }
        if (rc < 0) return 0;
        break;
    }
    // the dispatch list is grouped by agent: cut it into runs
    std::vector<std::pair<uint32_t, uint32_t>> runs;                                  // [begin, end)
    for (uint32_t i = 0; i < n;) {
        uint32_t j = i + 1;
        while (j < n && disp[j].agent_slot == disp[i].agent_slot) ++j;
        runs.emplace_back(i, j);
        i = j;
    }
    std::atomic<size_t> next{0};
    auto work = [&] {
        for (size_t r; (r = next.fetch_add(1)) < runs.size();) {
            for (uint32_t i = runs[r].first; i < runs[r].second; ++i) {               // FIFO inside the agent
                Request req; Manager::FromRecord(recs[i], &req);
                const int status = send_(req.AgentID, req);
                if (status < 0) m_->MarkRequestFailed(req.AgentID, req.ID, "request failed");
                else { Response rr; rr.StatusCode = status; m_->StoreResponse(req.AgentID, req.ID, rr); }
            }
        }
    };
    std::vector<std::thread> ths;
    const unsigned nt = std::max(1u, std::min<unsigned>(workers, (unsigned)runs.size()));
    for (unsigned t = 1; t < nt; ++t) ths.emplace_back(work);
    work();
    for (auto& th : ths) th.join();
    return n;
}

}  // namespace requests
}  // namespace agentainer
