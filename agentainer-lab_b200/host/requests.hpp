// requests.hpp — C++ mirror of the reference's Go package internal/requests over the C-ABI.
//
// The reference toolchain (Go) is not available in the build image, so the host side above the C-ABI is written in
// C++ with the SAME names, argument meaning and error behaviour as the Go types it stands in for:
//   requests.Manager        internal/requests/requests.go:52-275
//   requests.ReplayWorker   internal/requests/replay_worker.go:16-199
//   proxy decision          internal/api/server.go:493-541  (Manager::Decide — the one call proxyToAgentHandler makes
//                           instead of GetAgent + StoreRequest + status gate)
// Errors follow the Go convention: methods return an Error (empty == nil) that callers log and ignore (Q20).
#pragma once
#include <atomic>
#include <cstdint>
#include <functional>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "../../include/agentainer_gpu.h"

namespace agentainer {
namespace requests {

using Error = std::string;   // "" == nil

enum class RequestStatus { Pending, Processing, Completed, Failed };   // requests.go:19-24
const char* StatusString(RequestStatus s);

struct Response {            // requests.go:44-49
    int StatusCode = 0;
    std::map<std::string, std::string> Headers;
    std::vector<uint8_t> Body;
    uint64_t ReceivedAt = 0;
};
struct Request {             // requests.go:27-41
    std::string ID, AgentID, Method, Path;
    std::map<std::string, std::string> Headers;
    std::vector<uint8_t> Body;
    RequestStatus Status = RequestStatus::Pending;
    int RetryCount = 0, MaxRetries = 3;
    uint64_t CreatedAt = 0;
    int ResponseStatus = 0;  // Response.StatusCode of the stored response (0: none)
    std::string Error;
};
struct HttpRequest {         // the parts of *http.Request StoreRequest reads (requests.go:66-97)
    std::string Method, Path;                               // URL.Path, still with the /agent/{id} prefix (Q3)
    std::map<std::string, std::string> Header;              // first value per key (Q5)
    std::vector<uint8_t> Body;
};
struct Verdict {             // what proxyToAgentHandler does next
    int Code = 0;            // AGR_V_*
    int HTTPStatus = 0;      // 0 forward, 202, 503, 404
    std::string RequestID;   // requestID variable of the handler ("" = untracked)
    bool Stored = false;
};

std::string FormatUUID(const uint8_t id[16]);
bool ParseUUID(const std::string& s, uint8_t id[16]);

class Manager {
  public:
    // NewManager (requests.go:57).  engine_mints_ids: the handle was created with AGR_CFG_MINT_IDS, so Request.ID is what
    // the engine minted (read back through agr_ingest_ex), exactly as StoreRequest returns storedReq.ID (server.go:515).
    // The reference builds TWO managers (api.NewServer, server.go:62, and runServer, main.go:335): harmless there, both are
    // stateless wrappers of one Redis.  Here the state lives behind the handle, so every Manager of a process MUST wrap the
    // same handle (SURVEY 8a row a14): the constructor throws std::logic_error when a second, different handle shows up.
    explicit Manager(agr_handle* h, bool engine_mints_ids = false);
    ~Manager();
    // proxyToAgentHandler's decision (server.go:493-541): agent lookup, replay-flag dedupe, StoreRequest, status gate.
    Error Decide(const std::string& agentID, const HttpRequest& req, Verdict* out);
    // StoreRequest (requests.go:64-117).  Persists and appends to the pending queue regardless of the agent's status.
    Error StoreRequest(const std::string& agentID, const HttpRequest& req, Request* out);
    // StoreResponse (requests.go:120-194): completed + LREM pending + RPUSH completed.  "failed to get request" on a miss.
    Error StoreResponse(const std::string& agentID, const std::string& requestID, const Response& resp);
    // GetPendingRequests (requests.go:197-225)
    Error GetPendingRequests(const std::string& agentID, std::vector<Request>* out);
    // MarkRequestFailed (requests.go:228-275)
    Error MarkRequestFailed(const std::string& agentID, const std::string& requestID, const std::string& err);
    // json.Marshal(record) as the reference keeps it in Redis (requests.go:101,170,265; read by server.go:661-669,687-695)
    Error GetRequestJSON(const std::string& agentID, const std::string& requestID, std::string* out);
    // json.Marshal(GetPendingRequests(agentID)) — the "pending" member of GET /agents/{id}/requests (server.go:646-650)
    Error GetPendingRequestsJSON(const std::string& agentID, std::string* out, size_t* count);
    // the 24 h TTL of the record keys (SET ... EX, requests.go:106,175,270): drop what was last SET ttl or more before now
    Error Expire(uint64_t now, uint64_t ttl, uint64_t* expired);
    // AGR_CFG_RING: release the rows at the tail that no longer hold a record
    Error Reclaim(uint64_t* released);
    // interceptTransport.RoundTrip's classification (server.go:597-611): dial errors leave the record pending
    Error RecordTransportError(const std::string& agentID, const std::string& requestID, const std::string& err);
    agr_handle* handle() const { return h_; }
    static agr_handle* ProcessHandle();          // the handle every live Manager of this process wraps (nullptr: none yet)
    static void ToRecord(const std::string& agentID, const HttpRequest& req, const uint8_t id[16], bool replay,
                         const uint8_t replay_of[16], uint64_t seq, agr_record* rec);
    static void FromRecord(const agr_record& rec, Request* out);

  private:
    Error complete(const std::string& agentID, const std::string& requestID, uint8_t kind, int http);
    // the same with the bytes the record keeps (agr_complete_ex): seg = flattened headers (hdr_len bytes) + body, or the error text
    Error complete_ex(const std::string& agentID, const std::string& requestID, uint8_t kind, int http, const std::string& seg,
                      uint32_t hdr_len);
    agr_handle* h_;
    bool mint_;
    std::atomic<uint64_t> seq_{0};

  public:
    // time.Now() of the mirror: a logical counter by default; SetClock makes it the caller's clock (Unix nanoseconds)
    void SetClock(std::function<uint64_t()> now) { now_ = std::move(now); }
  private:
    uint64_t now() { return now_ ? now_() : ++seq_; }
    std::function<uint64_t()> now_;
};

// ReplayWorker (replay_worker.go:16-55).  The HTTP re-injection (replayRequest, :120-163) stays host I/O: the caller
// supplies it as `send`, which returns the status the proxy answered (or < 0 for a client error, :152-154).
class ReplayWorker {
  public:
    using Sender = std::function<int(const std::string& agentID, const Request& req)>;
    ReplayWorker(Manager* m, Sender send) : m_(m), send_(std::move(send)) {}   // NewReplayWorker (:24)
    void Start(unsigned interval_ms = 5000);   // :36-50 (5 s ticker)
    void Stop();                               // :53-55
    size_t ProcessAgents();                    // :58-117 — one tick; returns the number of replays dispatched
    // The same tick with the agents replayed CONCURRENTLY by `workers` threads (SURVEY 8f-3).  The reference walks agents
    // and their requests strictly one after the other (Q14); nothing in its semantics orders two different agents, so the
    // per-agent runs of the dispatch list may proceed side by side while each run stays FIFO.  `send` is called from
    // several threads at once.
    size_t ProcessAgentsConcurrent(unsigned workers);
  private:
    Manager* m_;
    Sender send_;
    std::thread th_;
    std::atomic<bool> stop_{false};
};

}  // namespace requests
}  // namespace agentainer
