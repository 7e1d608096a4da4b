// agr_common.h — layout constants, state-word encoding and hashes shared by host and device code.
//
// Data layout in HBM (see DESIGN.md section 3):
//   slab      : rows of 512 B (agr_record), row index = rid, rows are handed out in arrival order and never
//               move; the slab IS the arrival log, so "FIFO within an agent" == ascending rid.
//   state[rid]: u32  status | INQ | INFLIGHT | STORED | retry | max_retries      (K1 writes, K2 RMWs, K3 reads)
//   route[rid]: u32  agent slot(23) | verdict(3) | verdict flags(6)                       (K1 writes, K2/K3 read)
//   aux[rid]  : u32  response status | error kind                                (K2 writes)
//   cksum[rid]: u64  position-weighted checksum of the 512 B record              (K1 writes)
//   head[rid] : u32  K2 per-batch chain head of the row
//   ptime[rid]: u64  processed_at / received_at of the latest stored response        (K2 writes, K5 reads)
//   table     : hash-id mode only: open-addressing dedupe index, 32 B slots {id128, ~rid}, 128-bit CAS on the id
//               (absent with engine-minted ids, where the id is a keyed bijection of rid: agr_mint_id below)
//   logs      : completed / failed append-only logs of rid (per-agent lists are stable filters of them)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define AGR_HD __host__ __device__ __forceinline__
#else
#define AGR_HD static inline
#endif

// ---- record field offsets (agr_record in include/agentainer_gpu.h)
#define AGR_OFF_REQUEST_ID 0
#define AGR_OFF_REPLAY_OF 16
#define AGR_OFF_AGENT_ID 32
#define AGR_OFF_SEQ 64
#define AGR_OFF_FLAGS 72
#define AGR_OFF_PATH_LEN 76
#define AGR_OFF_HDR_LEN 78
#define AGR_OFF_BODY_LEN 80
#define AGR_OFF_STATUS 84
#define AGR_OFF_RETRY 85
#define AGR_OFF_MAX_RETRIES 86
#define AGR_OFF_ERROR_CODE 87
#define AGR_OFF_RESP_STATUS 88
#define AGR_OFF_PAYLOAD 96
#define AGR_REC 512u

// ---- state word
#define ST_STATUS_MASK 0x7u
#define ST_INQ 0x8u        // member of agent:{a}:requests:pending
#define ST_INFLIGHT 0x10u  // extension bookkeeping (never reference-visible): forward issued, no outcome yet
#define ST_STORED 0x20u    // row holds a record that StoreRequest persisted
#define ST_RESPONDED 0x40u // StoreResponse has run on it: Response / ProcessedAt are set (requests.go:165-167)
#define ST_RESP_RT 0x80u   // the stored Response has been through a later Unmarshal + Marshal (only the JSON form of
#define ST_ERR_RT 0x01000000u  // invalid UTF-8 depends on it: "\ufffd" when first written, EF BF BD afterwards); same for Error
#define ST_RETRY_SHIFT 8
#define ST_RETRY_MASK 0xff00u
#define ST_MAX_SHIFT 16
#define ST_MAX_MASK 0xff0000u
AGR_HD uint32_t st_status(uint32_t s) { return s & ST_STATUS_MASK; }
AGR_HD uint32_t st_retry(uint32_t s) { return (s & ST_RETRY_MASK) >> ST_RETRY_SHIFT; }
AGR_HD uint32_t st_max(uint32_t s) { return (s & ST_MAX_MASK) >> ST_MAX_SHIFT; }

// ---- route word
#define RT_SLOT_MASK 0x007fffffu
#define RT_SLOT_NONE 0x007fffffu
#define RT_CODE_SHIFT 23
#define RT_CODE_MASK 0x03800000u
#define RT_FLAG_SHIFT 26   // AGR_VF_* << 26 (six flag bits)
AGR_HD uint32_t rt_slot(uint32_t r) { return r & RT_SLOT_MASK; }
AGR_HD uint32_t rt_code(uint32_t r) { return (r & RT_CODE_MASK) >> RT_CODE_SHIFT; }
AGR_HD uint32_t rt_flags(uint32_t r) { return r >> RT_FLAG_SHIFT; }

// ---- aux word: response status (low 16) | error kind (bits 16..23)
#define AUX_ERR_SHIFT 16

#define AGR_RID_NONE 0xffffffffu
#define AGR_CFGI_HOLES 0x20000u         // internal cfg_flags bit (set per launch by the exchange path): rows of the batch that K4
                                        // shipped to their owner shard (agr_dev::xowner) are skipped

// ---- dedupe-index slot.  key == 0 means empty (a UUIDv4 is never all-zero); inv_rid = ~rid so that a zeroed
// slot is "no rid yet" and atomicMax keeps the LOWEST rid (arrival order wins among duplicate ids).
struct __attribute__((aligned(32))) agr_slot {
    unsigned long long key_lo, key_hi;
    uint32_t inv_rid;
    uint32_t pad[3];
};

// ---- agent table entry (device mirror of the host map): 48 B key+slot, open addressing
struct __attribute__((aligned(16))) agr_agent_key {
    unsigned long long w[4];  // 32 B id, NUL padded; all-zero = empty
    uint32_t slot;
    uint32_t status;          // AGR_AGENT_* or AG_STATUS_REMOVED (mirrors astatus[slot]; read together with the key)
    uint32_t pad[2];
};
#define AG_STATUS_REMOVED 0xffu

// ---- hashes (device-internal placement only: no observable result depends on them)
AGR_HD unsigned long long agr_fmix64(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return k;
}
AGR_HD unsigned long long agr_hash_id(unsigned long long lo, unsigned long long hi) {
    return agr_fmix64(lo ^ (hi * 0x9e3779b97f4a7c15ULL));
}
AGR_HD unsigned long long agr_hash_agent(unsigned long long w0, unsigned long long w1, unsigned long long w2,
                                         unsigned long long w3) {
    unsigned long long h = w0 * 0x9e3779b97f4a7c15ULL;
    h ^= (w1 + 0x165667b19e3779f9ULL) * 0xc2b2ae3d27d4eb4fULL;
    h ^= (w2 + 0x27d4eb2f165667c5ULL) * 0xff51afd7ed558ccdULL;
    h ^= (w3 + 0x85ebca77c2b2ae63ULL) * 0xc4ceb9fe1a85ec53ULL;
    return agr_fmix64(h);
}

// FNV-1a 64 over the id bytes (up to NUL): the SHARD hash, part of the ABI (Go: hash/fnv New64a).
AGR_HD unsigned long long agr_fnv1a64(const char* s, uint32_t maxlen) {
    unsigned long long h = 0xcbf29ce484222325ULL;
    for (uint32_t i = 0; i < maxlen && s[i]; ++i) { h ^= (unsigned char)s[i]; h *= 0x100000001b3ULL; }
    return h;
}

// ---- engine-minted request ids (AGR_CFG_MINT_IDS).  The reference mints uuid.New() INSIDE StoreRequest
// (internal/requests/requests.go:87); in this mode the engine does the same, and the id is an exact invertible
// function of where the record lives: lo = a keyed 60-bit permutation of x = (row mod 2^40 | shard << 40 |
// (generation ^ row >> 40) << 48) laid around the UUIDv4 version nibble, hi = a keyed hash of x with the RFC 4122 variant
// bits.  The row is the arrival number: a ring keeps counting past 2^40, and its 2^40-row periods are told apart by the
// 12-bit generation field, so ids are unique for AGR_ROW_LIMIT = 2^52 arrivals (rows below 2^40 keep the ids they always
// had).  A lookup decodes the row's low 40 bits from lo, places them in the live window (agr_unmint_in_window) and accepts
// only if mint(row) equals ALL 128 presented bits — an exact membership test with no table, no atomics and no random DRAM
// traffic on the ingest path.
#define AGR_MINT_M60 ((1ULL << 60) - 1)
#define AGR_MINT_ROW_M40 ((1ULL << 40) - 1)
#define AGR_ROW_LIMIT (1ULL << 52)      // rows (arrival numbers) an engine hands out: agr_reserve_rows stops there
#define AGR_MINT_C1 0x9e3779b97f4a7c15ULL
#define AGR_MINT_C2 0xbf58476d1ce4e5b9ULL
AGR_HD unsigned long long agr_inv_odd(unsigned long long c) {           // inverse mod 2^64 (Newton), masked by callers
    unsigned long long x = c;
    for (int k = 0; k < 6; ++k) x *= 2 - c * x;
    return x;
}
AGR_HD unsigned long long agr_perm60(unsigned long long x) {
    x &= AGR_MINT_M60;
    x = (x * AGR_MINT_C1) & AGR_MINT_M60; x ^= x >> 29;
    x = (x * AGR_MINT_C2) & AGR_MINT_M60; x ^= x >> 31;
    return x;
}
AGR_HD unsigned long long agr_perm60_inv(unsigned long long y) {
    y &= AGR_MINT_M60;
    y ^= y >> 31;                                                          // 2 * 31 >= 60: self-inverse
    y = (y * agr_inv_odd(AGR_MINT_C2)) & AGR_MINT_M60;
    y ^= y >> 29; y ^= y >> 58;                                            // inverse of y ^= y >> 29 on 60 bits
    y = (y * agr_inv_odd(AGR_MINT_C1)) & AGR_MINT_M60;
    return y;
}
AGR_HD void agr_mint_id(unsigned long long rid, uint32_t shard, uint32_t gen, unsigned long long secret,
                        unsigned long long& lo, unsigned long long& hi) {
    const unsigned long long x = (rid & AGR_MINT_ROW_M40) | ((unsigned long long)(shard & 0xffu) << 40) |
                                 (((unsigned long long)gen ^ (rid >> 40)) & 0xfffULL) << 48;
    const unsigned long long y = agr_perm60(x ^ (secret & AGR_MINT_M60));
    lo = (y & ((1ULL << 52) - 1)) | (0x4ULL << 52) | ((y >> 52) << 56);
    hi = agr_fmix64((x + 0x632be59bd9b4e019ULL) * 0x9e3779b97f4a7c15ULL ^ (secret >> 7));
    hi = (hi & ~0xc0ULL) | 0x80ULL;
}
// decodes x's fields from lo: the row's low 40 bits, the shard and the generation field (gen ^ row >> 40); returns false if
// lo cannot be a minted id.  Callers must still place the row (agr_unmint_in_window) and compare all 128 bits.
AGR_HD bool agr_unmint_id(unsigned long long lo, unsigned long long secret, unsigned long long& rid40, uint32_t& shard, uint32_t& genf) {
    if (((lo >> 52) & 0xfULL) != 0x4ULL) return false;
    const unsigned long long y = (lo & ((1ULL << 52) - 1)) | ((lo >> 56) << 52);
    const unsigned long long x = agr_perm60_inv(y) ^ (secret & AGR_MINT_M60);
    rid40 = x & AGR_MINT_ROW_M40; shard = (uint32_t)((x >> 40) & 0xffu); genf = (uint32_t)((x >> 48) & 0xfffu);
    return true;
}
// The row of the live window [tail, head_l) an id was minted for, or false.  The window is narrower than 2^40 rows (it never
// exceeds slab_rows), so at most one row in it has the decoded low 40 bits: row = tail + ((rid40 - tail) mod 2^40).  That row
// must lie below head_l, carry this shard and the generation field its period gives, and mint to all 128 presented bits.
AGR_HD bool agr_unmint_in_window(unsigned long long lo, unsigned long long hi, unsigned long long secret, uint32_t shard, uint32_t gen,
                                 unsigned long long tail, unsigned long long head_l, unsigned long long& row) {
    unsigned long long r40; uint32_t s, g;
    if (!agr_unmint_id(lo, secret, r40, s, g)) return false;
    const unsigned long long a = tail + ((r40 - tail) & AGR_MINT_ROW_M40);
    if (a >= head_l || s != shard || g != (uint32_t)((gen ^ (a >> 40)) & 0xfffULL)) return false;   // not a live row
    unsigned long long mlo, mhi;
    agr_mint_id(a, shard, gen, secret, mlo, mhi);
    if (mlo != lo || mhi != hi) return false;
    row = a;
    return true;
}

// ---- record checksum: c0 = sum w_k, c1 = sum (k+1) w_k over the 128 little-endian u32 words, mod 2^32
// (Fletcher-style).  It detects every single-word change (c0 moves by the change).  A swap of words a and b at distance d
// leaves c0 alone and moves c1 by d (b - a): it is missed exactly when d (b - a) = 0 mod 2^32, e.g. 0 and 0x80000000 two
// words apart; so is bit 31 flipped in two words an even distance apart.
AGR_HD unsigned long long agr_cksum_pack(uint32_t c0, uint32_t c1) {
    return ((unsigned long long)c1 << 32) | c0;
}
