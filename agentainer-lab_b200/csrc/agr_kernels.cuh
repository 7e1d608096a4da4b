// agr_kernels.cuh — device-side view of the engine state and the launch entry points of the K1..K3 kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/agentainer_gpu.h"
#include "agr_common.h"
#include "agr_synth.h"

#define AGR_CHUNK_ROWS 4096u   // granularity of the TTL sweep's per-chunk time bounds (k_expire) and of k_first_live

// agr_verdict {u8 code, u8 flags, u16 http_status, u32 agent_slot} of a route word, as one little-endian 64-bit word
AGR_HD unsigned long long rt_verdict(uint32_t r) {
    const uint32_t code = rt_code(r);
    const uint32_t http = code == AGR_V_QUEUED ? 202u : code == AGR_V_UNAVAILABLE ? 503u : code == AGR_V_NOT_FOUND ? 404u : 0u;
    return (unsigned long long)(code | (rt_flags(r) << 8) | (http << 16)) | ((unsigned long long)rt_slot(r) << 32);
}

// global counters (device u64 array), mirrored into agr_stats
enum {
    C_INGESTED = 0, C_STORED, C_REPLAY, C_DEDUPE_HITS, C_FORWARDED, C_QUEUED, C_UNAVAILABLE, C_NOT_FOUND, C_DUP_IDS, C_BAD_LEN,
    C_COMPLETIONS, C_COMPLETION_MISSES, C_FAILURES, C_DEAD_LETTERED, C_DIAL_ERRORS,
    C_REPLAY_DISPATCHED, C_LOG_OVERFLOW, C_NCTR = 24
};

struct agr_dev {
    uint8_t* slab;
    uint32_t* state;
    uint32_t* route;
    uint32_t* aux;
    unsigned long long* cksum;
    agr_slot* table;
    unsigned long long table_mask;
    agr_agent_key* akeys;
    uint32_t amask;
    uint8_t* astatus;          // [max_agents]
    unsigned long long* ctr;   // C_NCTR
    uint32_t* completed_log;
    uint32_t* failed_log;
    unsigned long long* log_len;   // [0] completed, [1] failed
    unsigned long long log_cap;
    uint32_t* dupfix;          // per-batch words: [0] in-batch duplicate-id races (see k1_post), [1] spare, [2] replay-flagged records
    uint32_t* dupfix_next;     // the other copy of those words: the TMA K1 and k1_post clear it for the next batch (no memset between batches)
    uint32_t* marks;           // K1 (TMA kernel) -> k1_post: one bit per row of the batch that the post pass must visit; nullptr = visit all
    uint32_t* head;            // [rows] K2 per-batch chain head of a row (op index + 1, 0 when idle)
    unsigned long long* ptime; // [rows] time.Now() of the latest StoreResponse (requests.go:146,164), the outcome's seq
    unsigned long long* mtime; // [rows] time of the latest SET of the record by K2 (0: only StoreRequest's, = the record's seq)
    unsigned long long* cmin;  // [rows / AGR_CHUNK_ROWS + 2] TTL sweep: lower bound of the last-SET times in a chunk (0 unknown, ~0 empty)
    unsigned long long* voff;  // variable-length mode: byte offset of row's record in the slab (nullptr = fixed 512 B rows)
    uint32_t* vlen;            // variable-length mode: stored length of the record
    unsigned long long id_secret;   // AGR_CFG_MINT_IDS
    uint32_t shard_id, id_gen;
    // Rows are named two ways.  The LOGICAL row id counts arrivals (what the API calls first_rid, what a minted id encodes,
    // what FIFO order means); the PHYSICAL row is where the record lives: the same number in append-only mode, logical
    // mod ring_rows with AGR_CFG_RING.  Every per-row array is indexed by the physical row; [tail, head_l) is the live
    // logical window (tail = 0 without the ring).
    unsigned long long tail, head_l;
    unsigned long long idx_base;   // hash-id mode: arrival number the dedupe index's row words are relative to (idx_encode)
    uint32_t ring_rows;        // 0 = append-only slab
    uint32_t tail_phys;        // tail % ring_rows
    uint32_t cfg_flags;
    const uint8_t* xowner;     // exchange batch (AGR_CFGI_HOLES): K4's owner shard of each of its rows; rows owned by a peer are holes
};

// single-key lookup descriptor (agr_get_record & co.: the host resolves agent_id -> slot)
struct __attribute__((aligned(16))) agr_dop {
    unsigned long long id_lo, id_hi;
    uint32_t slot;
    uint16_t http;
    uint8_t kind;
    uint8_t pad;
    unsigned long long seq;
};

// K2 on-device op, 16 B: what is left of a 64 B agr_outcome once its ids are resolved
struct __attribute__((aligned(16))) agr_k2op {
    uint32_t rid;              // physical row, AGR_RID_NONE = nothing to apply
    uint32_t kh;               // kind | http_status << 16
    unsigned long long seq;    // the outcome's logical time (processed_at / received_at, and the TTL clock)
};

struct agr_k2_scratch {
    agr_k2op* ops;             // [n]
    uint32_t* nxt;             // [n] chain link (op index + 1, 0 = end)
    uint8_t* eff;              // [n] bit0 push completed, bit1 push failed (8-byte aligned)
    int32_t* results;          // [n] 0 / AGR_ENOTFOUND
    uint32_t* ticket;          // k2_append's tile ticket; one 8-byte word {ticket, overflow} directly in front of tiles[]
    uint32_t* overflow;        // = ticket + 1: set when the batch's pushes did not fit the logs
    unsigned long long* tiles; // [tiles] k2_append's look-back words
};

// agr_complete_ex: the bytes a batch's outcomes carry (StoreResponse's response, MarkRequestFailed's error text).  The chain
// root of a row writes the stored-response / error words of its last applied RESPONSE / ERROR op and marks that op's eff
// byte with K2_EFF_WIN; only marked ops' segments are copied into the byte slab.
#define K2_EFF_WIN 4u
#define K2_NO_BYTES (~0ULL)   // dst[j] of an op that carries no bytes (a plain outcome in a batch of the service kernel)
struct agr_k2_bytes {
    const uint8_t* src;                  // the batch's bytes on the device
    const unsigned long long* src_off;   // [n + 1] the caller's offsets: segment j = src + (src_off[j] - src_off[0]), src_off[j+1] - src_off[j] bytes
    const unsigned long long* dst;       // [n] where segment j goes, relative to base (16-byte rounded running sum of the lengths)
    const uint32_t* hlen;                // [n] leading bytes of a RESPONSE segment that are its flattened headers; nullptr = none
    unsigned long long base;             // physical offset of the batch's region in the byte slab (a multiple of 16)
    uint8_t* slab;                       // the byte slab
    unsigned long long* resp_off; uint32_t* resp_len; uint32_t* resp_hlen;   // per-row words of the stored response
    unsigned long long* err_off; uint32_t* err_len;                           // and of the stored error text
};

// K3 select modes
enum { K3_TICK = 0, K3_AGENT_PENDING = 1, K3_LOG_AGENT = 2, K3_AGENT_PENDING_IDS = 3 /* LRANGE: expired records' ids included */ };
struct agr_k3_params {
    int mode;
    uint32_t slot;             // agent for the single-agent modes
    const uint32_t* log;       // K3_LOG_AGENT: source log
    unsigned long long lo, hi; // item range [lo, hi): rids or log positions (row modes: lo rounded down to a multiple of 4)
    unsigned long long lo_real; // first item that counts (items in [lo, lo_real) are skipped)
    uint32_t groups;           // matrix columns: max agent slot + 1 (TICK) or 1
    uint32_t nwarps;           // matrix rows
    uint32_t per_warp;         // items per warp chunk (multiple of 32)
    uint32_t* matrix;          // [nwarps][groups]
    uint32_t* cta_matrix;      // [ceil(nwarps / 8)][groups] per-CTA sums of eight consecutive warp rows: what the column scan runs over
    uint32_t* gtotal;          // [groups]
    uint32_t* goff;            // [groups + 1]
    uint32_t* out_rid;         // [cap]
    uint32_t* out_slot;        // [cap]
    uint32_t cap;
    uint32_t* selmask;         // [nwarps * per_warp / 32] one selection bit per item, written by k3_mark, read by k3_place
    uint32_t* min_inq;         // TICK: lowest item (offset from lo) still in a pending list: low-water mark for the next scan
};

// K1 for variable-length records (agr_k1_var.cu) and the matching gathers
cudaError_t agr_launch_k1_var(const agr_dev& d, const uint8_t* blob, const uint32_t* off, uint32_t n, unsigned long long blob_bytes,
                              uint32_t* tile_first, uint32_t first_rid, unsigned long long blob_base, int sm_count, cudaStream_t st,
                              uint32_t variant = 0 /* k1_variant: bit 0x20 = LSU form */);
// The checksums of the batch's LONG records (stored length over AGR_VT_MAXREC), which K1v decides but does not sum: list[0..nl)
// = their batch indices, list[nl..2 nl] = the index of each one's first 8 KiB piece (list[2 nl] = all pieces); acc = 2 nl
// scratch words.  One warp per piece, the pieces' sums added per record, then packed into cksum[first_rid + index].
cudaError_t agr_launch_k1v_long(const agr_dev& d, const uint8_t* blob, const uint32_t* off, const uint32_t* list, uint32_t nl,
                                uint32_t npieces, uint32_t* acc, uint32_t first_rid, cudaStream_t st);
// off[i] = 512 i for i = 0 .. n: the offsets K1v reads a run of 512-byte slots by
void agr_launch_slot_offsets(uint32_t* off, uint32_t n, cudaStream_t st);
void agr_launch_var_lens(const agr_dev& d, const uint32_t* rids, uint32_t n, uint32_t* lens, cudaStream_t st);
void agr_launch_var_copy(const agr_dev& d, const uint32_t* rids, uint32_t n, const unsigned long long* out_off, uint8_t* out, cudaStream_t st);
#define AGR_VT_TILE 8192u   // lower bound of the tile size used by agr_k1_var.cu (sizes the tile index)
#define AGR_VT_MAXREC 8192u

// K5: JSON wire form of stored records (agr_k5_json.cu)
struct agr_k5_params {
    const uint32_t* rids;            // physical rows; nullable: record i is logical row first_l + i
    unsigned long long first_l;
    uint32_t n;
    uint32_t array;                  // 1: emit json.Marshal([]*Request) = [rec,rec,...]; 0: records back to back
    uint32_t roundtrip;              // 1: every string has been through json.Unmarshal (GetPendingRequests, requests.go:215-221)
    uint32_t* len;                   // [n] encoded length of record i (with its '[' / ',' / ']' in array mode)
    unsigned long long* off;         // [n + 1] byte offsets of the records in out
    unsigned long long* chunk_sum;   // [chunks + 1]; chunk_sum[chunks] = total bytes after agr_launch_k5_measure
    uint8_t* out;
    const uint8_t* bytes;            // byte slab of stored responses and error texts
    const unsigned long long* resp_off; const uint32_t* resp_len; const uint32_t* resp_hlen;
    const unsigned long long* err_off; const uint32_t* err_len;
    const unsigned long long* ptime;
};
uint32_t agr_k5_chunks(uint32_t n);
void agr_launch_k5_measure(const agr_dev& d, const agr_k5_params& p, cudaStream_t st);
void agr_launch_k5_emit(const agr_dev& d, const agr_k5_params& p, cudaStream_t st);

// K4: shard binning / stable pack for the multi-GPU exchange
struct agr_k4_params {
    const uint8_t* items;      // n items of item_bytes each (records: 512, outcome descriptors: 32)
    uint32_t item_bytes, agent_off, n, G, me;
    uint32_t nwarps, per_warp;
    uint32_t* matrix;          // [nwarps][G]
    uint32_t* gtotal;          // [G]   items per owner
    uint32_t* goff;            // [G+1] owner-major offsets
    uint8_t* owner;            // [n]
    uint32_t* perm;            // [n]   position of item i in owner-major order
    uint8_t* local_dst;        // where this shard's own items go (final slab rows / local op array)
    uint8_t* send_dst;         // owner-major send buffer (peer segments are shipped as they lie)
    uint32_t inplace;          // 1: items are slab rows already in their final place: own items are not moved, peers' items are
                               //    copied to the (peers-only) send buffer; their rows are left as they are (K1 skips them by owner)
};
void agr_launch_k4_count(const agr_k4_params& p, cudaStream_t st);
void agr_launch_k4_scatter(const agr_k4_params& p, cudaStream_t st);
void agr_launch_k4_unpermute(const agr_k4_params& p, const void* local_res, const void* remote_res, void* out, uint32_t res_bytes,
                             cudaStream_t st);

// first_log: arrival number of the batch's first row (= first_rid unless the slab is a ring); tmap: the slab's CUtensorMap (128 B,
// agr_k1_tma_make_map).  With engine-minted ids the TMA kernel decides every replay's dedupe hit itself, and k1_post is launched
// only to write verdicts or ids.  The optional events bracket the TMA kernel.  Returns the number of kernels launched (1 or 2).
int agr_launch_k1(const agr_dev& d, uint32_t first_rid, unsigned long long first_log, uint32_t n, const void* tmap,
                   int sm_count, cudaStream_t st, cudaEvent_t ev0 = nullptr, cudaEvent_t ev1 = nullptr,
                   void* verdicts = nullptr /* device agr_verdict[n], written by k1_post */,
                   void* ids = nullptr /* device u8[n][16]: Request.ID per record, written by k1_post */);
void agr_launch_expire(const agr_dev& d, unsigned long long rows, unsigned long long now, unsigned long long ttl,
                       unsigned long long* expired, cudaStream_t st);
// ring mode: first live (STORED) row at or after the tail, as an offset from it (0xffffffff: none), then release of
// `count` rows from the tail and stable compaction of a log (entries of released rows drop out)
void agr_launch_first_live(const agr_dev& d, unsigned long long live, bool use_cmin, uint32_t* scratch, void* out_host, cudaStream_t st);
void agr_launch_release_rows(const agr_dev& d, uint32_t count, uint32_t* resp_len, uint32_t* resp_hlen, uint32_t* err_len, cudaStream_t st);
void agr_launch_bytes_span(const agr_dev& d, unsigned long long head, unsigned long long cap, const unsigned long long* resp_off,
                           const uint32_t* resp_len, const unsigned long long* err_off, const uint32_t* err_len, unsigned long long* span,
                           cudaStream_t st);
void agr_launch_log_compact(const agr_dev& d, const uint32_t* log, unsigned long long len, uint32_t released, uint32_t* out,
                            uint32_t* chunk_cnt /* [chunks + 1] */, unsigned long long* new_len /* device: receives the kept count */,
                            cudaStream_t st);
// physical rows [first, first + rows)
void agr_launch_verify(const agr_dev& d, unsigned long long first, unsigned long long rows, unsigned long long* bad, cudaStream_t st);
void agr_launch_reindex(const agr_dev& d, uint32_t rows, cudaStream_t st);
void agr_launch_reindex_range(const agr_dev& d, uint32_t first, uint32_t n, cudaStream_t st);
void agr_launch_k1_post(const agr_dev& d, uint32_t first_rid, uint32_t n, int sm_count, cudaStream_t st, void* verdicts, void* ids,
                        const uint32_t* marks = nullptr);
int agr_k1_tma_make_map(void* slab, unsigned long long rows, void* out_map /*128 B, 64 B aligned*/);
uint32_t agr_k2_tiles(uint32_t n);
void agr_launch_k2(const agr_dev& d, const void* outs /*device agr_outcome[n]*/, const agr_k2_scratch& s, uint32_t n, cudaStream_t st,
                   const agr_k2_bytes* bytes = nullptr /* agr_complete_ex: apply with bytes, then copy the winners' segments */);
void agr_launch_resolve(const agr_dev& d, const agr_dop* ops, uint32_t* hrid, uint32_t n, cudaStream_t st);
void agr_launch_k3_select(const agr_dev& d, const agr_k3_params& p, int sm_count, cudaStream_t st);
void agr_launch_k3_gather(const agr_dev& d, const uint32_t* rids, const uint32_t* slots, uint32_t n,
                          uint8_t* out_recs /*nullable*/, uint8_t* out_dispatch /*nullable, 32 B each*/,
                          uint8_t* out_ids /*nullable, 16 B each*/, cudaStream_t st);
void agr_launch_drop_agent(const agr_dev& d, uint32_t slot, unsigned long long rows, unsigned long long max_log_len,
                           cudaStream_t st);
// The held-slot scan: sets bit s of held (cleared by the caller) for every candidate slot s (bit s of cand, nslots bits) that
// the route word of a decided row among physical rows [p0, p0 + n) carries.  route is the engine's route array (4 words of
// padding past its end).
void agr_launch_slot_refs(const uint32_t* route, unsigned long long p0, unsigned long long n, const uint32_t* cand, uint32_t nslots,
                          uint32_t* held, int sm_count, cudaStream_t st);
void agr_launch_synth(uint8_t* dst, agr_synth_dev s, unsigned long long first_index, uint32_t n, cudaStream_t st);

// Online snapshot (AGR_CFG_ONLINE_SNAPSHOT): the cut copies the sections that later calls rewrite in place (per-row words, the
// completed / failed logs) into a device shadow.  Every destination is 256 B-aligned; every source is the start of its array.
// Sections [0, nrow) have the byte counts given here; sections nrow and nrow + 1 are the completed and failed logs, whose
// lengths the kernel reads from d.log_len and stores as two u64 at the start of the shadow.  The cut reads src, dst_off,
// bytes[0, nrow), shadow and nrow of agr_snap_cmp below.
//
// Delta snapshots (AGR_CFG_DELTA_SNAPSHOT).  The compare cut is the cut above that also compares each 16 B piece with what the
// shadow held (the previous cut) before it overwrites it: a piece that differs sets the bit of its block (256 rows of a word
// section, 1024 entries of a log) in bits, and every piece, live or not, goes into a 128-bit keyed sum (digest[2], added to).
// Section s covers bytes[s] bytes (sections nrow and nrow + 1, the logs, as in the cut unless lens_from_host); its
// block of piece i is i >> pshift[s], its bit word bit_off[s] + block / 32.  The digest-only pass (compare = false) reads
// src alone: no shadow, no bits.  The sum does not depend on the grid: it adds one keyed hash per (section, piece).
#define AGR_SNAP_CUT_MAX 16
struct agr_snap_cmp {
    const uint8_t* src[AGR_SNAP_CUT_MAX];
    unsigned long long dst_off[AGR_SNAP_CUT_MAX];
    unsigned long long bytes[AGR_SNAP_CUT_MAX];
    uint32_t pshift[AGR_SNAP_CUT_MAX];
    uint32_t bit_off[AGR_SNAP_CUT_MAX];
    uint32_t sec_id[AGR_SNAP_CUT_MAX];     // the section's index in the file's table: part of each piece's key
    uint8_t* shadow;
    uint32_t* bits;
    unsigned long long* digest;
    unsigned long long key;
    uint32_t nrow;
    uint32_t lens_from_host;               // 1: the logs' byte counts are bytes[nrow], bytes[nrow + 1] (restore-time checks)
};
void agr_launch_snap_cut(const agr_dev& d, const agr_snap_cmp& c, int sm_count, cudaStream_t st);
void agr_launch_snap_cmp(const agr_dev& d, const agr_snap_cmp& c, bool compare, int sm_count, cudaStream_t st);
// Block gather / scatter: block list[j] of a section table (arr[s], width[s] bytes per row, rows rows in all, block_rows rows
// per block) is packed at stage + j * rec_bytes as each section's slice in table order; the last block of the table may be
// short.  gather: arrays -> stage (the writer packs dirty blocks from the shadow); scatter: stage -> arrays (restore).
struct agr_snap_blocks {
    uint8_t* arr[AGR_SNAP_CUT_MAX];
    uint32_t width[AGR_SNAP_CUT_MAX];
    uint32_t nsec, block_rows;
    unsigned long long rows, rec_bytes;
    const uint32_t* list;
    uint8_t* stage;
};
void agr_launch_snap_blocks(const agr_snap_blocks& g, uint32_t n, bool gather, cudaStream_t st);

// Relocation of a restore into other capacities (agr_relayout.cu).  Row ids [s.tail, s.tail + n) of the source engine s move
// to row id mod t.ring_rows of the target t with every per-row word; the record bytes (AGR_CFG_VARLEN) and the response / error
// bytes of the live rows (state != 0) are packed in row-id order from byte 0 of t's byte rings, each response and error
// segment on a 16 B boundary.  The record form is the target's (t.voff): a fixed-stride source's live rows go into a
// variable-length target as their compact records, a variable-length source's records into a fixed-stride target as 512 B
// rows padded with zeros.  count: per-tile sums, then their exclusive scan and the two totals (record bytes, response bytes)
// at totals[0..1], and (variable-length into fixed-stride) the count of records longer than 512 B and the least
// (k << 32 | vlen) of them at totals[2..3]; rows: the words, the 512 B rows and the segment lists; bytes: one byte ring from
// its segment list (destination offsets non-decreasing); log: one completed / failed log's physical rows.
struct agr_relayout_words {            // the per-row words of the stored responses, which agr_dev does not carry
    unsigned long long* resp_off; uint32_t* resp_len; uint32_t* resp_hlen;
    unsigned long long* err_off; uint32_t* err_len;
};
struct agr_relayout {
    agr_dev s, t;
    agr_relayout_words sw, tw;
    unsigned long long n;
    unsigned long long* tile_sum;      // [2 * agr_relayout_tiles(n)]
    unsigned long long* totals;        // [4]
    unsigned long long *vseg_dst, *vseg_src; uint32_t* vseg_len;   // [n]: row k's record (either side variable-length)
    unsigned long long *rseg_dst, *rseg_src; uint32_t* rseg_len;   // [2n]: row k's response, then its error text
};
uint32_t agr_relayout_tiles(unsigned long long n);
void agr_launch_relayout_count(const agr_relayout& p, cudaStream_t st);
void agr_launch_relayout_rows(const agr_relayout& p, cudaStream_t st);
void agr_launch_relayout_bytes(const uint8_t* src, uint8_t* dst, const unsigned long long* seg_dst, const unsigned long long* seg_src,
                               const uint32_t* seg_len, unsigned long long nseg, unsigned long long total, cudaStream_t st);
void agr_launch_relayout_log(const agr_dev& s, const agr_dev& t, const uint32_t* in, uint32_t* out, unsigned long long len, cudaStream_t st);
