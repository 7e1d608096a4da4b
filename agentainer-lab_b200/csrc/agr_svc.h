// agr_svc.h — the single-request front end (AGR_CFG_COMBINE): shared layout of the pinned op ring between the calling
// threads, the dispatcher thread (agr_front.cu) and the service kernel (agr_svc.cu).
//
// The reference serves one goroutine per HTTP request (net/http accept loop -> proxyToAgentHandler, server.go:493-573), so
// the call pattern at the boundary is "many OS threads, ONE request per call": agr_ingest_ex(n = 1) then agr_complete(n = 1).
// A kernel launch per call would cap the engine near 10^5 requests/s.  Instead:
//   callers     claim ring slots with one fetch_add, write their record / outcome into PINNED, device-mapped host memory,
//               publish the slot, and spin (then yield) on the slot's result word;
//   dispatcher  one thread per handle: takes the contiguous published prefix of the ring (<= SVC_MAX_OPS), reserves slab rows
//               for its records under the handle mutex and publishes a 256 B batch descriptor;
//   service kernel  ONE resident CTA polls the descriptor ring over PCIe, pulls the batch's payloads straight out of host
//               memory, runs the K1 decision chain (records) and the K2 state machine (outcomes) of agr_device.cuh on them,
//               and writes verdict / id / row / result back into host memory.  No launch, no cudaMemcpy and no stream
//               synchronisation on the per-request path.
// Event order: batch by batch; inside a batch the records in ring order, then the outcomes in ring order.  All operations of
// one batch were in flight at the same time (none had returned), so this is a linearisation of the concurrent calls.
// Every other entry point stops the kernel first (it runs on the handle's stream), so the rest of the engine never sees it.
#pragma once
#include <stdint.h>
#include <string.h>
#include "../../include/agentainer_gpu.h"   // AGR_OUT_TICKET_MAX_BYTES, AGR_VAR_MAX_RECORD
#if defined(__CUDACC__)
#define SVC_HD __host__ __device__
#else
#define SVC_HD
#endif

#define SVC_SLOTS 16384u          // ring slots (power of two)
#define SVC_MAX_OPS 256u          // operations per batch (<= 128 of them records: what one shared-memory stage of the kernel holds)
#define SVC_MAX_CALL 32u          // records / outcomes per call that go through the ring
#define SVC_DESCS 64u             // descriptor ring entries
#define SVC_PAYLOAD 512u          // bytes per slot: an agr_record, or an agr_outcome in the first 64 B
// SVC_OP_OUTCOME_BYTES (agr_submit_complete_ex, agr_complete_ex): the 64 B outcome, then u32 hdr_len, u32 len, then the len
// bytes of its segment (response headers + body, or the error text); the caller writes only the 16 B-rounded part it uses
#define SVC_BYTES_HDR 64u         // offset of hdr_len (len follows)
#define SVC_BYTES_DATA 72u        // offset of the segment
#define SVC_BYTES_MAX (SVC_PAYLOAD - SVC_BYTES_DATA)   // 440 = AGR_OUT_INLINE_BYTES
#define SVC_NO_BYTES (~0ULL)      // svc_desc.resp_base when the batch's bytes found no room in the response byte slab

enum { SVC_OP_SKIP = 0, SVC_OP_RECORD = 1, SVC_OP_OUTCOME = 2, SVC_OP_OUTCOME_BYTES = 3 };

// A SPAN (agr_submit_complete_large): an SVC_OP_OUTCOME_BYTES op whose len word exceeds SVC_BYTES_MAX is the HEAD of
// svc_span_conts(len) CONTINUATION slots that follow it in ring order, each holding the next SVC_PAYLOAD bytes of the segment.
//   callers     claim the whole span with one fetch_add, publish the continuations (also as SVC_OP_OUTCOME_BYTES) and then the
//               head; if any slot of it is not free, all of them go out as SVC_OP_SKIP;
//   dispatcher  takes a span whole or not at all (svc_scan), marks its continuations in svc_desc.cont;
//   kernel      stages a span's slots next to each other, so the segment is contiguous in shared memory.
// A continuation is not an operation: nobody collects it, so whoever answers its batch (k_svc, svc_fail_ops) writes its answer
// with SVC_COLLECTED already set.  Until then its slot is not free, so it is never rewritten before its bytes were pulled.
#define SVC_SPAN_MAX (1u + (AGR_OUT_TICKET_MAX_BYTES - SVC_BYTES_MAX + SVC_PAYLOAD - 1u) / SVC_PAYLOAD)   // 33 slots
static_assert(SVC_SPAN_MAX <= 128u / 2u, "a span of the longest segment must fit a batch that already holds other ops");
// continuation slots of a head whose len word says len (a word beyond the longest segment counts as the longest)
SVC_HD static inline uint32_t svc_span_conts(uint32_t len) {
    if (len <= SVC_BYTES_MAX) return 0u;
    if (len > AGR_OUT_TICKET_MAX_BYTES) len = AGR_OUT_TICKET_MAX_BYTES;
    return (len - SVC_BYTES_MAX + SVC_PAYLOAD - 1u) / SVC_PAYLOAD;
}
// the segment length of an op with `conts` continuations staged: its len word clamped to what those slots hold.  The dispatcher
// reserves the batch's bytes and the kernel places them with this one function, so the two totals cannot differ.
SVC_HD static inline uint32_t svc_span_len(uint32_t len, uint32_t conts) {
    const uint32_t cap = SVC_BYTES_MAX + conts * SVC_PAYLOAD;
    return len < cap ? len : cap;
}
// A RECORD SPAN (variable-length engines: agr_submit_ingest, agr_ingest_var through the ring): a record of stored length L
// (svc_rec_len of its header) takes svc_rec_slots(L) consecutive slots, slot k holding bytes [512 k, 512 k + 512) of it — the
// head holds the 96-byte header and the first 416 payload bytes, which is what a fixed-stride engine receives.  Same rules as an
// outcome span: continuations published first and the head last, all slots or none, the continuations of kind SVC_OP_RECORD
// marked in svc_desc.cont.  On a fixed-stride engine a record is one slot, whatever its header says.
#define SVC_REC_SPAN_MAX (AGR_VAR_MAX_RECORD / SVC_PAYLOAD)   // 16 slots
static_assert(SVC_REC_SPAN_MAX <= 128u / 2u, "a record span of the longest record must fit a batch that already holds other ops");
// stored length of a variable-length record whose header holds lens (path_len | hdr_len << 16) and body_len: 96 + its 16 B-rounded
// payload, capped at AGR_VAR_MAX_RECORD (a header whose lengths exceed that is stored at the cap and decided AGR_VF_BAD_LEN).
// The submitting side, svc_scan, the dispatcher and the kernel all take a record's length from this one function.
SVC_HD static inline uint32_t svc_rec_len(uint32_t lens, uint32_t body_len) {
    const uint64_t p = (uint64_t)(lens & 0xffffu) + (lens >> 16) + body_len;
    return p > AGR_VAR_MAX_RECORD - AGR_HEADER_BYTES ? AGR_VAR_MAX_RECORD : AGR_HEADER_BYTES + (uint32_t)((p + 15u) & ~15ULL);
}
// the same, from a header in memory (any alignment)
SVC_HD static inline uint32_t svc_rec_len_at(const uint8_t* head) {
    uint32_t w[2];
    memcpy(w, head + 76, 8);                                  // path_len, hdr_len | body_len (agr_record)
    return svc_rec_len(w[0], w[1]);
}
SVC_HD static inline uint32_t svc_rec_slots(uint32_t rec_len) { return (rec_len + SVC_PAYLOAD - 1u) / SVC_PAYLOAD; }

// continuations that follow op in a batch of count ops (cont: svc_desc.cont, one bit per op)
SVC_HD static inline uint32_t svc_conts_after(const uint32_t* cont, uint32_t op, uint32_t count) {
    uint32_t k = 0;
    while (op + 1u + k < count && ((cont[(op + 1u + k) >> 5] >> ((op + 1u + k) & 31u)) & 1u)) ++k;
    return k;
}

// batch descriptor (256 B = 64 words), written by the dispatcher (host), polled by the kernel: sixteen lanes read 16 B each
// in ONE poll; the kernel accepts it when the batch number matches and the check word agrees with the other 62 words (a poll
// that raced the host's stores sees a mix of old and new words and fails the check), so no second PCIe round trip is needed
struct __attribute__((aligned(64))) svc_desc {
    uint32_t kinds[SVC_MAX_OPS / 16];     // words 0..15: 2 bits per op, SVC_OP_*
    uint64_t from;                        // absolute number of the batch's first ring slot
    uint32_t count;                       // ops in the batch
    uint32_t n_records;                   // SVC_OP_RECORD ops among them: rows first_p .. first_p + n_records
    uint64_t first_l;                     // logical (arrival) number of the first record's row
    uint32_t first_p;                     // its physical row
    uint32_t tail_phys;                   // live window of the slab after this batch's rows were reserved
    uint64_t tail, head_l;
    uint64_t idx_base;
    uint64_t resp_base;                   // SVC_OP_OUTCOME_BYTES ops: physical offset of the batch's region of the response byte
                                          // slab (their 16 B-rounded segments in ring order), or SVC_NO_BYTES
    uint32_t cont[SVC_MAX_OPS / 32];      // words 32..39: 1 bit per op, set for a span's continuation slots
    uint64_t vbase;                       // words 40..41, variable-length engines: physical byte offset in the byte slab of the
                                          // batch's records (back to back in ring order, each svc_rec_len long)
    uint32_t rec_slots;                   // word 42, variable-length engines: ring slots of the records, continuations included
    uint32_t pad0;
    uint64_t reserved[8];
    uint64_t check;                       // words 60..61: XOR of svc_mix_word over words 0..59 and 62..63
    uint64_t seq;                         // words 62..63: batch number; the kernel waits for desc[seq % SVC_DESCS].seq == seq
};

static_assert(sizeof(svc_desc) == 256, "svc_desc must be 256 B (sixteen 16 B lanes)");

// per-slot result: ONE 16-byte store from the kernel (a single PCIe write inside one cache line: the caller sees all of it or
// none of it, so no system-wide fence sits between "result" and "done"):
//   record   w0, w1 = agr_verdict (w0's low byte = AGR_V_*, never 0);  w2 | (w3 & 0xffff) << 32 = logical row
//            host-side failure (slab full / CUDA error, written by the dispatcher): w0 = 0, w1 = (uint32_t)error code
//   outcome  w0 = (uint32_t)result (0 / AGR_ENOTFOUND / error code);  w1 = SVC_OUT_LOG_FULL when its completed / failed
//            push landed past the log's capacity and was dropped (the transition was applied), else 0
//   w3 >> 16 = tag of the slot's lap (svc_tag): the caller spins on it, and sets SVC_COLLECTED in it once it has read the
//              answer — that line is in the collector's cache anyway, so freeing a slot costs no extra miss.
// Request.ID is not shipped: with engine-minted ids it is a function of the row (agr_mint_id, computed by the caller's
// thread), with caller-supplied ids the caller has it already.
struct __attribute__((aligned(16))) svc_res { volatile uint32_t w[4]; };
#define SVC_OUT_LOG_FULL 1u
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline uint32_t svc_tag(uint64_t slot_abs) { return (uint32_t)((slot_abs / SVC_SLOTS) & 0x3fffu) + 1u; }   // 1 .. 16384
#define SVC_COLLECTED 0x8000u     // or-ed into the tag by whoever collected the answer: the slot may be written for the next lap

// control block (host memory): how the host stops the kernel and how the kernel says where it stopped
struct __attribute__((aligned(64))) svc_ctl {
    volatile uint32_t stop;               // host -> kernel: leave once no published batch is left
    volatile uint32_t state;              // kernel -> host: 1 running, 0 exited, 2 exited on the safety timeout
    volatile uint64_t done_seq;           // kernel -> host: last batch completed
    volatile uint64_t heartbeat;          // kernel -> host: polls so far (diagnostics)
    volatile uint64_t cyc_wait, cyc_load, cyc_work, cyc_publish;   // kernel -> host: SM cycles spent waiting for a batch, pulling
                                          // payloads, deciding, publishing results (diagnostics, AGR_SVC_DEBUG)
};

static_assert(sizeof(svc_res) == 16, "svc_res must be 16 B");

struct svc_dev {                          // device-visible addresses of the pinned ring (UVA: host pointer == device pointer)
    const svc_desc* desc;
    const uint8_t* payload;               // [SVC_SLOTS][SVC_PAYLOAD]
    svc_res* res;                         // [SVC_SLOTS]
    svc_ctl* ctl;
    uint32_t* dupfix;                     // device word for in-batch duplicate ids (hash-id mode)
    unsigned long long idle_ns;           // safety: leave after this long without a batch even if nobody said stop
    // SVC_OP_OUTCOME_BYTES: the response byte slab and its per-row words, and per-outcome scratch [SVC_MAX_OPS (+ 1)]
    uint8_t* resp;
    unsigned long long *resp_off, *err_off;
    uint32_t *resp_len, *resp_hlen, *err_len;
    unsigned long long *b_off, *b_dst;    // running sums of the segments' lengths / of their 16 B-rounded lengths
    uint32_t* b_hlen;
};
