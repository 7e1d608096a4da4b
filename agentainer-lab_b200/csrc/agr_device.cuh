// agr_device.cuh — device helpers shared by the K1 kernels and K2/K3: cache-hinted loads, the 128-bit CAS, the
// agent-table and dedupe-index probes, and the per-record decision of proxyToAgentHandler + StoreRequest.
#pragma once
#include "agr_kernels.cuh"
#include "../../include/agentainer_gpu.h"

#define FULL 0xffffffffu

// ------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint4 ldg_v4(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// 128-bit compare-and-swap on a dedupe-index slot's id.  The result stays an opaque 128-bit value (no unpacking
// at the issue point), so nothing depends on the atomic's return until the caller actually inspects it.
typedef unsigned __int128 u128;
__device__ __forceinline__ u128 make_u128(unsigned long long lo, unsigned long long hi) { return ((u128)hi << 64) | lo; }
__device__ __forceinline__ u128 cas128(void* addr, u128 cmp, u128 val) {
    u128 old;
    asm volatile("atom.relaxed.gpu.global.cas.b128 %0, [%1], %2, %3;" : "=q"(old) : "l"(addr), "q"(cmp), "q"(val) : "memory");
    return old;
}
__device__ __forceinline__ unsigned long long pack64(uint32_t lo, uint32_t hi) {
    return ((unsigned long long)hi << 32) | lo;
}

// dedupe-index lookup: returns slot index or ~0ULL
__device__ __forceinline__ unsigned long long table_find(const agr_dev& d, unsigned long long lo, unsigned long long hi) {
    unsigned long long idx = agr_hash_id(lo, hi) & d.table_mask;
    for (unsigned long long probe = 0; probe <= d.table_mask; ++probe) {
        const agr_slot* s = d.table + idx;
        const uint4 k = __ldcg(reinterpret_cast<const uint4*>(s));
        unsigned long long klo = pack64(k.x, k.y), khi = pack64(k.z, k.w);
        if ((klo | khi) == 0ULL) return ~0ULL;
        if (klo == lo && khi == hi) return idx;
        idx = (idx + 1) & d.table_mask;
    }
    return ~0ULL;
}

// logical <-> physical row (see agr_dev)
__device__ __forceinline__ unsigned long long row_logical(const agr_dev& d, uint32_t p) {
    if (!d.ring_rows) return p;
    return d.tail + (p >= d.tail_phys ? p - d.tail_phys : p + d.ring_rows - d.tail_phys);
}
__device__ __forceinline__ uint32_t row_physical(const agr_dev& d, unsigned long long l) {
    return d.ring_rows ? (uint32_t)(l % d.ring_rows) : (uint32_t)l;
}

// What the dedupe index stores for a row: ~(arrival number - idx_base).  "Lowest row wins" among duplicate ids is decided
// by RED.max on this word, so it must order rows by ARRIVAL, not by where they live: after the ring has wrapped a later
// arrival can sit at a lower physical row.  idx_base is the tail at the last index rebuild (every agr_reclaim rebuilds the
// index in this mode), so the offset always fits 31 bits; in append-only mode idx_base = 0 and this is ~row.
__device__ __forceinline__ uint32_t idx_encode(const agr_dev& d, uint32_t prow) {
    return ~(uint32_t)(row_logical(d, prow) - d.idx_base);
}
__device__ __forceinline__ uint32_t idx_decode(const agr_dev& d, uint32_t inv) {
    return row_physical(d, d.idx_base + (unsigned long long)(~inv));
}

// address of a row's record: fixed 512 B stride, or the byte offset kept per row in variable-length mode
__device__ __forceinline__ const uint8_t* rec_ptr(const agr_dev& d, uint32_t rid) {
    return d.voff ? d.slab + d.voff[rid] : d.slab + (size_t)rid * AGR_REC;
}

// (agent slot is checked by the callers) request id -> row holding the record stored under it, or AGR_RID_NONE.
// Hash mode: probe the dedupe index.  Mint mode: decode the row from the id relative to the live window and accept only an
// exact 128-bit match (agr_unmint_in_window).
__device__ __forceinline__ uint32_t lookup_rid(const agr_dev& d, unsigned long long lo, unsigned long long hi) {
    if ((lo | hi) == 0ULL) return AGR_RID_NONE;
    if (d.cfg_flags & AGR_CFG_MINT_IDS) {
        unsigned long long rid;
        return agr_unmint_in_window(lo, hi, d.id_secret, d.shard_id, d.id_gen, d.tail, d.head_l, rid) ? row_physical(d, rid) : AGR_RID_NONE;
    }
    const unsigned long long idx = table_find(d, lo, hi);
    if (idx == ~0ULL) return AGR_RID_NONE;
    const uint32_t inv = __ldcg(&d.table[idx].inv_rid);
    return inv ? idx_decode(d, inv) : AGR_RID_NONE;
}

// ------------------------------------------------------------------------------------------------ K1
#define K1_NLC 10  // counters C_INGESTED .. C_BAD_LEN are contiguous from 0; lc[K1_NLC] counts rows left to the post pass
// Decision + persistence for ONE record whose 96 B header is in registers: the sequential semantics of
// proxyToAgentHandler (server.go:498-541) with StoreRequest (requests.go:64-117) inlined, split in stages so a
// kernel can put independent work (the record checksum) between the long-latency global operations:
//   k1_agent_issue   -> loads of the first agent-table probe                      (GetAgent, server.go:498)
//   k1_begin         -> resolves the agent, classifies, issues the FIRST index CAS (StoreRequest's SET)
//   k1_finish        -> finishes probing, publishes the row id, forms verdict + state word
// The index insert is ONE returning atomic (CAS.128 on the id) plus a fire-and-forget RED.max of ~rid.  Who owns
// an id is therefore decided by the final value of inv_rid (lowest row wins = arrival order); a row that found its
// id already present is provisionally a duplicate and bumps dupfix, and only then does k1_post re-check owners.
struct k1_result { uint32_t state, route; };
struct ag_probe { uint4 a, b, t; uint32_t idx; };
struct k1_ctx {
    unsigned long long id_lo, id_hi, tidx;
    u128 old;
    uint32_t slot, astatus;
    bool replay, want_store, cas_issued, deferred, bad, hole;
    uint32_t known;            // replay-flagged + tracked: 0 n/a, 1 target row's words are in o_route / o_state, 2 resolve in the post pass,
    uint32_t o_route, o_state; //                           3 cannot be a dedupe hit (no live row, or not an earlier one),
                               //                           4 earlier row of the same batch: its header words are in t_*
    uint4 t_agent0, t_agent1, r_agent0, r_agent1;   // known == 4: the target's agent id and this row's
    uint32_t t_flags, t_lens, t_body;               //             the target's flags, path_len | hdr_len << 16, body_len
};

__device__ __forceinline__ ag_probe agent_probe_load(const agr_dev& d, uint32_t idx) {
    ag_probe p;
    const agr_agent_key* e = d.akeys + idx;
    p.a = ldg_v4(&e->w[0]); p.b = ldg_v4(&e->w[2]); p.t = ldg_v4(&e->slot); p.idx = idx;
    return p;
}
__device__ __forceinline__ ag_probe k1_agent_issue(const agr_dev& d, const uint4& h2, const uint4& h3) {
    return agent_probe_load(d, (uint32_t)agr_hash_agent(pack64(h2.x, h2.y), pack64(h2.z, h2.w), pack64(h3.x, h3.y), pack64(h3.z, h3.w)) & d.amask);
}
// resolves (slot, status) from the first probe, continuing the linear probe if needed
__device__ __forceinline__ void agent_resolve(const agr_dev& d, ag_probe p, const uint4& h2, const uint4& h3, uint32_t& slot, uint32_t& status) {
    slot = RT_SLOT_NONE; status = AG_STATUS_REMOVED;
    if ((h2.x | h2.y | h2.z | h2.w | h3.x | h3.y | h3.z | h3.w) == 0u) return;
    for (uint32_t probe = 0; probe <= d.amask; ++probe) {
        if ((p.a.x | p.a.y | p.a.z | p.a.w | p.b.x | p.b.y | p.b.z | p.b.w) == 0u) return;          // empty: miss
        if (p.a.x == h2.x && p.a.y == h2.y && p.a.z == h2.z && p.a.w == h2.w && p.b.x == h3.x && p.b.y == h3.y &&
            p.b.z == h3.z && p.b.w == h3.w) { slot = p.t.x; status = p.t.y & 0xffu; return; }
        p = agent_probe_load(d, (p.idx + 1) & d.amask);
    }
}

// body_len = the record's body_len field, payload_cap = the payload bytes the record form can hold (416 for the fixed
// stride, stored length - 96 for a variable-length record): a record whose lengths do not fit is never persisted.
// decide (fixed-stride batch kernels only): first_log is the arrival number of the batch's first row and my_log this row's.  With
// engine-minted ids the row a replay-flagged request names is a pure function of the id, so the dedupe hit (AGR_VF_KNOWN) is
// decided here and nothing is left to the post pass:
//   - a target that arrived BEFORE this batch: its route and state words are final (two 4-byte loads);
//   - an earlier target of the SAME batch: it is stored, with this row's slot, exactly when its agent id equals this row's (slots
//     are never reused, so equal slots mean equal ids), persistence is on and it is neither replay-flagged nor too long
//     for its row.  Its header bytes 32..83 are loaded instead of its words, which this launch may not have written yet;
//   - any other row (this one, a later one) is not a dedupe hit.
// (An earlier row of the same agent is owned by the same shard, so it is never a hole of an exchange batch.)
// The loads are issued here and consumed by k1_finish, one tile later.  Without `decide`, or with caller-supplied ids, every
// tracked replay is left to the post pass.
// bi: the row's index in its batch.  In an exchange batch (AGR_CFGI_HOLES) a row whose record K4 shipped to its owner shard
// (xowner[bi] != shard_id) is a hole: it is neither stored nor indexed here, and it gets no verdict.  The caller's flags word
// plays no part in that.
__device__ __forceinline__ bool k1_is_hole(const agr_dev& d, const uint32_t bi) {
    return (d.cfg_flags & AGR_CFGI_HOLES) && __ldg(d.xowner + bi) != d.shard_id;
}
__device__ __forceinline__ void k1_begin(const agr_dev& d, const ag_probe& ap, const uint4& h0, const uint4& h1, const uint4& h2, const uint4& h3,
                                         const uint4& h4, const uint32_t body_len, const uint32_t payload_cap, const bool decide,
                                         const unsigned long long first_log, const unsigned long long my_log, const uint32_t bi, k1_ctx& c) {
    c.id_lo = pack64(h0.x, h0.y); c.id_hi = pack64(h0.z, h0.w);
    c.replay = (h4.z & AGR_F_REPLAY) != 0;                                                // server.go:506
    c.hole = k1_is_hole(d, bi);                                                           // row emptied by the exchange (K4)
    agent_resolve(d, ap, h2, h3, c.slot, c.astatus);                                      // server.go:498
    const bool found = c.slot != RT_SLOT_NONE && c.astatus != AG_STATUS_REMOVED;
    c.want_store = found && (d.cfg_flags & AGR_CFG_PERSISTENCE) && !c.replay && !c.hole;  // server.go:508
    c.bad = c.want_store && ((unsigned long long)(h4.w & 0xffffu) + (h4.w >> 16) + body_len > payload_cap);
    // mint mode: the id is a function of the row, nothing to insert; the caller's request_id is ignored
    c.deferred = c.want_store && !c.bad && (d.cfg_flags & AGR_CFG_MINT_IDS);
    c.cas_issued = c.want_store && !c.bad && (c.id_lo | c.id_hi) != 0ULL && !c.deferred && !(d.cfg_flags & AGR_CFG_DIAG_NO_INDEX);
    c.old = 0;
    c.tidx = 0;
    c.known = 0u; c.o_route = 0u; c.o_state = 0u;
    if (c.replay && found && (h1.x | h1.y | h1.z | h1.w) != 0u) {
        c.known = 2u;
        if ((d.cfg_flags & AGR_CFG_MINT_IDS) && decide) {
            const uint32_t orid = lookup_rid(d, pack64(h1.x, h1.y), pack64(h1.z, h1.w));
            const unsigned long long olog = orid == AGR_RID_NONE ? ~0ULL : row_logical(d, orid);
            if (olog < first_log) { c.o_route = __ldcg(&d.route[orid]); c.o_state = __ldcg(&d.state[orid]); c.known = 1u; }
            else if (olog < my_log) {
                const uint8_t* t = rec_ptr(d, orid);
                c.t_agent0 = __ldcg(reinterpret_cast<const uint4*>(t + AGR_OFF_AGENT_ID));
                c.t_agent1 = __ldcg(reinterpret_cast<const uint4*>(t + AGR_OFF_AGENT_ID + 16));
                const uint2 fl = __ldcg(reinterpret_cast<const uint2*>(t + AGR_OFF_FLAGS));
                c.t_flags = fl.x; c.t_lens = fl.y;
                c.t_body = __ldcg(reinterpret_cast<const uint32_t*>(t + AGR_OFF_BODY_LEN));
                c.r_agent0 = h2; c.r_agent1 = h3;
                c.known = 4u;
            } else c.known = 3u;
        }
    }
    if (c.cas_issued) {
        c.tidx = agr_hash_id(c.id_lo, c.id_hi) & d.table_mask;
        c.old = cas128(&d.table[c.tidx], 0, make_u128(c.id_lo, c.id_hi));
    }
}

__device__ __forceinline__ k1_result k1_finish(const agr_dev& d, uint32_t rid, const uint4& h1, const uint4& h5, k1_ctx& c,
                                               uint32_t* lc /*local counters*/) {
    k1_result out{0u, 0u};
    if (c.hole) return out;                                                               // not a record of this shard
    lc[C_INGESTED]++;
    if (c.slot == RT_SLOT_NONE || c.astatus == AG_STATUS_REMOVED) {                       // server.go:499-502
        lc[C_NOT_FOUND]++;
        out.route = RT_SLOT_NONE | (AGR_V_NOT_FOUND << RT_CODE_SHIFT);
        return out;
    }
    uint32_t vflags = 0;
    bool tracked = false;
    if (c.want_store) {
        // StoreRequest: SET rec (the row itself, already in the slab) + index insert + RPUSH pending (INQ bit)
        bool ok = c.cas_issued || c.deferred;
        if (c.cas_issued) {
            const u128 key = make_u128(c.id_lo, c.id_hi);
            for (;;) {
                if (c.old == 0) break;                                                    // claimed an empty slot
                if (c.old == key) {                                                       // id already present
                    ok = false;
                    asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(d.dupfix) : "memory");
                    break;
                }
                c.tidx = (c.tidx + 1) & d.table_mask;
                c.old = cas128(&d.table[c.tidx], 0, key);
            }
            asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(&d.table[c.tidx].inv_rid), "r"(idx_encode(d, rid)) : "memory");
        }
        if (ok) {
            uint32_t maxr = (h5.y >> 16) & 0xffu;
            if (maxr == 0) maxr = 3;                                                      // requests.go:95
            out.state = AGR_ST_PENDING | ST_INQ | ST_STORED | (maxr << ST_MAX_SHIFT);     // requests.go:93-95,111
            vflags |= AGR_VF_STORED | AGR_VF_TRACKED;
            tracked = true;
            lc[C_STORED]++;
        } else if (c.bad) {
            vflags |= AGR_VF_BAD_LEN;                                                     // StoreRequest fails: server.go:511-514 path
            lc[C_BAD_LEN]++;
        } else {
            vflags |= AGR_VF_DUP_ID;                                                      // server.go:511-514 path
            lc[C_DUP_IDS]++;
        }
    } else if (c.replay) {                                                                // server.go:519-522
        vflags |= AGR_VF_REPLAY;
        lc[C_REPLAY]++;
        tracked = (h1.x | h1.y | h1.z | h1.w) != 0u;
        if (tracked) {
            vflags |= AGR_VF_TRACKED;
            if (c.known == 1u) {                                                          // dedupe hit decided here (see k1_begin)
                if (rt_slot(c.o_route) == c.slot && (c.o_state & ST_STORED)) { vflags |= AGR_VF_KNOWN; lc[C_DEDUPE_HITS]++; }
            } else if (c.known == 4u) {                                                   // the same-batch target's store condition
                const uint4 x0 = make_uint4(c.t_agent0.x ^ c.r_agent0.x, c.t_agent0.y ^ c.r_agent0.y, c.t_agent0.z ^ c.r_agent0.z, c.t_agent0.w ^ c.r_agent0.w);
                const uint4 x1 = make_uint4(c.t_agent1.x ^ c.r_agent1.x, c.t_agent1.y ^ c.r_agent1.y, c.t_agent1.z ^ c.r_agent1.z, c.t_agent1.w ^ c.r_agent1.w);
                const bool same_agent = (x0.x | x0.y | x0.z | x0.w | x1.x | x1.y | x1.z | x1.w) == 0u;
                const bool stored = (d.cfg_flags & AGR_CFG_PERSISTENCE) && !(c.t_flags & AGR_F_REPLAY) &&
                                    (unsigned long long)(c.t_lens & 0xffffu) + (c.t_lens >> 16) + c.t_body <= AGR_REC - AGR_OFF_PAYLOAD;
                if (same_agent && stored) { vflags |= AGR_VF_KNOWN; lc[C_DEDUPE_HITS]++; }
            } else if (c.known == 2u) {
                vflags |= AGR_VF_DUP_ID;                                                  // marker "resolve me in the post pass" (never
                lc[K1_NLC]++;                                                             // a real flag of a replay-flagged row)
            }
        }
    }
    uint32_t code;
    if (c.astatus != AGR_AGENT_RUNNING) {                                                 // server.go:525
        if ((d.cfg_flags & AGR_CFG_PERSISTENCE) && tracked) { code = AGR_V_QUEUED; lc[C_QUEUED]++; }   // :526-536
        else { code = AGR_V_UNAVAILABLE; lc[C_UNAVAILABLE]++; }                           // :539-540
    } else {
        code = AGR_V_FORWARD; lc[C_FORWARDED]++;                                          // :546-572
        if (out.state) out.state |= ST_INFLIGHT;
    }
    out.route = c.slot | (code << RT_CODE_SHIFT) | (vflags << RT_FLAG_SHIFT);
    return out;
}

// TTL bookkeeping of a K1 tile: `mine` = this lane's record created_at (~0 for a lane without a record); the warp's minimum
// lowers the time bound of the chunk(s) the tile's rows [first, first + count) lie in (k_expire reads them).  One or two
// atomics per 32 records.
__device__ __forceinline__ void k1_note_time(const agr_dev& d, const uint32_t first, const uint32_t count, const unsigned long long mine) {
    // a ring runs for ever and sweeps every step: K1 keeps the bounds.  An append-only slab is swept rarely: agr_expire resets
    // the bounds of the chunks filled since its last call instead (sweep_invalidate), and K1 spends nothing on it.
    if (!(d.cfg_flags & AGR_CFG_RING)) return;
    const uint32_t hi = (uint32_t)(mine >> 32), hmin = __reduce_min_sync(FULL, hi);
    const uint32_t lmin = __reduce_min_sync(FULL, hi == hmin ? (uint32_t)mine : 0xffffffffu);
    if ((threadIdx.x & 31) == 0 && count) {
        unsigned long long t = pack64(lmin, hmin);
        if (t == 0ULL) t = 1ULL;                                                          // 0 means "unknown"
        if (t == ~0ULL) t = ~0ULL - 1ULL;                                                 // ~0 means "no stored row"
        const uint32_t c0 = first / AGR_CHUNK_ROWS, c1 = (first + count - 1u) / AGR_CHUNK_ROWS;
        atomicMin(d.cmin + c0, t);
        if (c1 != c0) atomicMin(d.cmin + c1, t);
    }
}


__device__ __forceinline__ void k1_flush_counters(const agr_dev& d, uint32_t* lc, uint32_t* s_ctr) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int c = 0; c < K1_NLC; ++c) {
        uint32_t v = __reduce_add_sync(FULL, lc[c]);
        if (lane == 0 && v) atomicAdd(&s_ctr[c], v);
    }
    {   // per-batch note for k1_post: how many replay-flagged rows wait for its "stored earlier?" pass
        const uint32_t v = __reduce_add_sync(FULL, lc[K1_NLC]);
        if (lane == 0 && v) atomicAdd(d.dupfix + 2, v);
    }
    __syncthreads();
    if (threadIdx.x < K1_NLC && s_ctr[threadIdx.x]) atomicAdd(&d.ctr[threadIdx.x], (unsigned long long)s_ctr[threadIdx.x]);
}


// Post pass of ONE record of a batch, after ALL inserts of the batch (k1_post; the service kernel runs it behind a CTA barrier):
//   (a) replay-flagged row: resolve replay_of -> KNOWN (dedupe hit), compared by ARRIVAL so that "known" means "stored
//       earlier in arrival order" (also after the ring has wrapped);
//   (b) only if some row found its id already present (dupfix != 0 — never with minted UUIDs): owner of an id = the
//       EARLIEST row that carried it (final inv_rid).  A provisionally stored row that is not the owner is demoted to a
//       persistence failure (server.go:511-514); a provisional duplicate that IS the owner (it lost the CAS race to a
//       later row of the same batch) is promoted to stored.
// Returns the row's final route word; delta = {dedupe hits, stored, queued} corrections for the global counters.
// `marked`: the caller knows from K1's row marks that this row is a tracked replay, so the row's own route word and its
// replay_of are fetched together, and the target row's two words together: two dependent round trips instead of four.
// first_log: arrival number of the batch's first row.  (a) and (b) of different rows run in no particular order, so with
// dupfix != 0 a target of this batch may not have been promoted yet when (a) reads its state word.  The row the index names
// for an id is the id's owner, and a caller-id owner of this batch always ends up stored, so (a) takes that from its arrival.
__device__ __forceinline__ uint32_t k1_post_one(const agr_dev& d, const uint32_t rid, const uint32_t dupfix, int* delta, const bool marked = false,
                                                const unsigned long long first_log = ~0ULL) {
    uint4 t = make_uint4(0, 0, 0, 0);
    if (marked) t = __ldcg(reinterpret_cast<const uint4*>(rec_ptr(d, rid) + AGR_OFF_REPLAY_OF));
    uint32_t r = d.route[rid];
    uint32_t vf = rt_flags(r);
    if ((vf & AGR_VF_REPLAY) && (vf & AGR_VF_DUP_ID)) {              // a tracked replay K1 left for this pass (k1_finish's marker)
        if (!marked) t = __ldcg(reinterpret_cast<const uint4*>(rec_ptr(d, rid) + AGR_OFF_REPLAY_OF));
        const uint32_t orid = lookup_rid(d, pack64(t.x, t.y), pack64(t.z, t.w));
        vf &= ~AGR_VF_DUP_ID;
        uint32_t oroute = 0u, ostate = 0u;
        if (orid != AGR_RID_NONE) { oroute = __ldcg(&d.route[orid]); ostate = __ldcg(&d.state[orid]); }
        const unsigned long long olog = orid != AGR_RID_NONE ? row_logical(d, orid) : ~0ULL;
        const bool owner_here = dupfix != 0u && !(d.cfg_flags & AGR_CFG_MINT_IDS) && olog >= first_log;   // promoted, or about to be
        if (orid != AGR_RID_NONE && olog < row_logical(d, rid) && rt_slot(oroute) == rt_slot(r) && ((ostate & ST_STORED) || owner_here)) {
            vf |= AGR_VF_KNOWN;
            delta[0]++;
        }
        r = (r & ((1u << RT_FLAG_SHIFT) - 1u)) | (vf << RT_FLAG_SHIFT);
        d.route[rid] = r;
    }
    if (dupfix != 0u && (vf & (AGR_VF_STORED | AGR_VF_DUP_ID))) {
        const uint4 h0 = __ldcg(reinterpret_cast<const uint4*>(rec_ptr(d, rid)));
        const unsigned long long idx = table_find(d, pack64(h0.x, h0.y), pack64(h0.z, h0.w));
        const uint32_t owner = (idx == ~0ULL) ? AGR_RID_NONE : idx_decode(d, __ldcg(&d.table[idx].inv_rid));
        uint32_t code = rt_code(r);
        const bool running = d.astatus[rt_slot(r)] == AGR_AGENT_RUNNING;
        if ((vf & AGR_VF_STORED) && owner != rid) {                 // demote
            if (code == AGR_V_QUEUED) { code = AGR_V_UNAVAILABLE; delta[2]--; }
            vf = (vf & ~(AGR_VF_STORED | AGR_VF_TRACKED)) | AGR_VF_DUP_ID;
            d.state[rid] = 0;
            delta[1]--;
        } else if ((vf & AGR_VF_DUP_ID) && owner == rid && (pack64(h0.x, h0.y) | pack64(h0.z, h0.w)) != 0ULL) {   // promote
            const uint4 h5 = __ldcg(reinterpret_cast<const uint4*>(rec_ptr(d, rid) + 80));
            uint32_t maxr = (h5.y >> 16) & 0xffu;
            if (maxr == 0) maxr = 3;
            uint32_t st = AGR_ST_PENDING | ST_INQ | ST_STORED | (maxr << ST_MAX_SHIFT);
            if (running) st |= ST_INFLIGHT;
            else if (code == AGR_V_UNAVAILABLE) { code = AGR_V_QUEUED; delta[2]++; }
            vf = (vf & ~AGR_VF_DUP_ID) | AGR_VF_STORED | AGR_VF_TRACKED;
            d.state[rid] = st;
            delta[1]++;
        }
        r = rt_slot(r) | (code << RT_CODE_SHIFT) | (vf << RT_FLAG_SHIFT);
        d.route[rid] = r;
    }
    return r;
}
// agr_verdict {u8 code, u8 flags, u16 http_status, u32 agent_slot} as two words
__device__ __forceinline__ uint2 k1_verdict_word(const uint32_t r) {
    const unsigned long long v = rt_verdict(r);
    return make_uint2((uint32_t)v, (uint32_t)(v >> 32));
}
// Request.ID of a row as the engine knows it
__device__ __forceinline__ uint4 k1_request_id(const agr_dev& d, const uint32_t rid) {
    if (d.cfg_flags & AGR_CFG_MINT_IDS) {
        unsigned long long lo, hi;
        agr_mint_id(row_logical(d, rid), d.shard_id, d.id_gen, d.id_secret, lo, hi);
        return make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
    }
    return __ldcg(reinterpret_cast<const uint4*>(rec_ptr(d, rid)));
}
__device__ __forceinline__ void k1_post_apply(const agr_dev& d, const int* tot) {
    const int hits = tot[0], stored = tot[1], q = tot[2];
    {
        if (hits) atomicAdd(&d.ctr[C_DEDUPE_HITS], (unsigned long long)hits);
        if (stored) {
            atomicAdd(&d.ctr[C_STORED], (unsigned long long)(long long)stored);
            atomicAdd(&d.ctr[C_DUP_IDS], (unsigned long long)(long long)(-stored));
        }
        if (q) {
            atomicAdd(&d.ctr[C_QUEUED], (unsigned long long)(long long)q);
            atomicAdd(&d.ctr[C_UNAVAILABLE], (unsigned long long)(long long)(-q));
        }
    }
}
__device__ __forceinline__ void k1_post_flush(const agr_dev& d, int* delta, const int lane) {
    const int tot[3] = {__reduce_add_sync(FULL, delta[0]), __reduce_add_sync(FULL, delta[1]), __reduce_add_sync(FULL, delta[2])};
    if (lane == 0) k1_post_apply(d, tot);
}

// ------------------------------------------------------------------------------------------------ K2
// A warp copies len bytes from src (any alignment; global or shared memory) to the 16-byte aligned dst with 16-byte stores; the
// last store fills the tail of dst's 16-byte rounded space.  Lane l reads the aligned 16-byte blocks around its output block
// and funnel-shifts them into place; a block is read only if it holds a byte of the segment.
__device__ __forceinline__ void warp_copy16(uint4* dst, const uint8_t* src, const uint32_t len, const uint32_t lane) {
    const uint32_t sh = (uint32_t)reinterpret_cast<uintptr_t>(src) & 15u, q = sh >> 2, r = (sh & 3u) * 8u;
    const uint4* as = reinterpret_cast<const uint4*>(src - sh);
    const uint32_t chunks = (len + 15u) >> 4;
    for (uint32_t c = lane; c < chunks; c += 32u) {
        const uint4 lo = as[c];
        uint4 hi = make_uint4(0u, 0u, 0u, 0u);
        if (sh && sh + len > 16u * (c + 1u)) hi = as[c + 1u];
        uint32_t w0 = lo.x, w1 = lo.y, w2 = lo.z, w3 = lo.w, w4 = hi.x, w5 = hi.y, w6 = hi.z, w7 = hi.w;
        if (q & 2u) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; w5 = w7; }
        if (q & 1u) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
        dst[c] = make_uint4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
    }
}

// One outcome (64 B agr_outcome as four 16 B words: request id | agent id[0..15] | agent id[16..31] | kind,http,seq):
// resolve the agent in the device agent table (no per-outcome host work) and the request id to its row, write the 16 B op
// and thread it onto its row's chain (head[row] = index of the last op linked + 1).
__device__ __forceinline__ void k2_link_one(const agr_dev& d, const agr_k2_scratch& s, const uint32_t j, const uint4& id, const uint4& a0,
                                            const uint4& a1, const uint4& t) {
    uint32_t slot, status;
    agent_resolve(d, k1_agent_issue(d, a0, a1), a0, a1, slot, status);     // RT_SLOT_NONE for an unknown agent: the key cannot exist
    const unsigned long long id_lo = pack64(id.x, id.y), id_hi = pack64(id.z, id.w);
    const uint32_t kind = t.x & 0xffu;
    uint32_t rid = AGR_RID_NONE, nxt = 0u;
    int32_t res = 0;
    const bool ext = (d.cfg_flags & AGR_CFG_SKIP_INFLIGHT) != 0;
    if ((id_lo | id_hi) != 0ULL && (kind == AGR_OUT_RESPONSE || kind == AGR_OUT_ERROR || (kind == AGR_OUT_DIAL_ERR && ext))) {
        const uint32_t cand = lookup_rid(d, id_lo, id_hi);
        // the Redis key is agent:{a}:requests:{r}: the agent is part of the key (requests.go:150,229)
        if (cand != AGR_RID_NONE && (d.state[cand] & ST_STORED) && rt_slot(d.route[cand]) == slot) {
            rid = cand;
            nxt = atomicExch(&d.head[rid], j + 1u);
        }
        if (rid == AGR_RID_NONE && kind != AGR_OUT_DIAL_ERR) {
            res = AGR_ENOTFOUND;                                           // requests.go:153-156 / 232-235
            atomicAdd(&d.ctr[C_COMPLETION_MISSES], 1ULL);
        }
    }
    if (kind == AGR_OUT_DIAL_ERR) atomicAdd(&d.ctr[C_DIAL_ERRORS], 1ULL);  // server.go:600-605: stays pending
    agr_k2op op;
    op.rid = rid; op.kh = kind | (t.x & 0xffff0000u); op.seq = pack64(t.z, t.w);
    s.ops[j] = op;
    s.nxt[j] = nxt;
    s.eff[j] = 0;
    if (s.results) s.results[j] = res;
}

// the state transition of ONE outcome on a private copy of the row words; returns the list pushes (bit0 completed, bit1 failed)
struct k2_row { uint32_t st, aux; unsigned long long ptime, mtime; bool responded, written; };
__device__ __forceinline__ uint32_t k2_apply_op(k2_row& r, const uint32_t kh, const unsigned long long seq, uint32_t* cnt) {
    const uint32_t kind = kh & 0xffu;
    uint32_t eff = 0;
    uint32_t st = r.st;
    if (kind == AGR_OUT_RESPONSE) {                                        // StoreResponse, requests.go:163-191
        st = (st & ~(ST_STATUS_MASK | ST_INFLIGHT)) | AGR_ST_COMPLETED | ST_RESPONDED;   // :166
        r.ptime = seq; r.responded = true;                                 // :164,167 now / ProcessedAt
        r.mtime = seq; r.written = true;                                   // :175 SET ... EX 24h restarts the TTL (Q11)
        st &= ~ST_RESP_RT;                                                 // a fresh Response object
        if (st_retry(st)) st |= ST_ERR_RT;                                 // Error went through Unmarshal + Marshal
        r.aux = (r.aux & 0xffff0000u) | (kh >> 16);                        // :165 request.Response
        st &= ~ST_INQ;                                                     // :180-184 LREM pending 1 id
        eff |= 1u; cnt[0]++;                                               // :187-191 RPUSH completed
    } else if (kind == AGR_OUT_ERROR) {                                    // MarkRequestFailed, requests.go:243-262
        uint32_t retry = st_retry(st);
        if (retry < 255u) retry++;                                         // :245
        st = (st & ~(ST_RETRY_MASK | ST_STATUS_MASK | ST_INFLIGHT | ST_ERR_RT)) | (retry << ST_RETRY_SHIFT);
        if (st & ST_RESPONDED) st |= ST_RESP_RT;
        r.aux = (r.aux & 0xff00ffffu) | ((uint32_t)AGR_OUT_ERROR << AUX_ERR_SHIFT);   // :244 request.Error
        r.mtime = seq; r.written = true;                                   // :270 SET ... EX 24h
        cnt[1]++;
        if (retry < st_max(st)) {
            st |= AGR_ST_PENDING;                                          // :248-249, keeps queue position (Q11)
        } else {
            st |= AGR_ST_FAILED;                                           // :243
            eff |= 2u; cnt[2]++;                                           // :252-255 RPUSH failed
            st &= ~ST_INQ;                                                 // :258-261 LREM pending 1 id
        }
    } else {                                                               // dial error, extension bookkeeping only
        st &= ~ST_INFLIGHT;
    }
    r.st = st;
    return eff;
}

// Op j applies its row's chain if it is the chain ROOT (the last op linked onto the row).  One outcome per row and batch is
// the common case and takes no loop at all; short chains are sorted in registers (the walk order is the link order, which is
// arbitrary); longer ones fall back to repeated minimum selection over the chain.
// BYTES (agr_complete_ex): the ops carry bytes; the root also stores the segments of its row's last RESPONSE and last ERROR
// op (the latest StoreResponse / MarkRequestFailed SET wins) and marks those ops K2_EFF_WIN for the copy.
#define K2_SORT_MAX 8
template <bool BYTES>
__device__ __forceinline__ void k2_note_bytes(const agr_k2_bytes* b, const uint32_t o, const uint32_t kh, int& wr, int& we) {
    if (BYTES && b->dst[o] != K2_NO_BYTES) {                               // (plain outcomes of a service-kernel batch carry none)
        if ((kh & 0xffu) == AGR_OUT_RESPONSE) wr = (int)o;
        else if ((kh & 0xffu) == AGR_OUT_ERROR) we = (int)o;
    }
}
template <bool BYTES = false>
__device__ __forceinline__ void k2_apply_one(const agr_dev& d, const agr_k2_scratch& s, const uint32_t j, uint32_t* cnt,
                                             const agr_k2_bytes* b = nullptr) {
    const agr_k2op me = s.ops[j];
    const uint32_t rid = me.rid;
    if (rid == AGR_RID_NONE) return;
    if (__ldcg(&d.head[rid]) != j + 1u) return;
    k2_row r{d.state[rid], d.aux[rid], 0ULL, 0ULL, false, false};
    int wr = -1, we = -1;                                                  // BYTES: last RESPONSE / ERROR op of the row
    const uint32_t first = __ldcg(&s.nxt[j]);
    if (first == 0u) {
        s.eff[j] = (uint8_t)k2_apply_op(r, me.kh, me.seq, cnt);
        k2_note_bytes<BYTES>(b, j, me.kh, wr, we);
    } else {
        uint32_t idx[K2_SORT_MAX];
        uint32_t len = 0;
        for (uint32_t cur = j + 1u; cur != 0u; cur = __ldcg(&s.nxt[cur - 1u])) {
            if (len < K2_SORT_MAX) {
                // insertion into the ascending prefix (fully unrolled compare-exchange chain: idx stays in registers)
                uint32_t v = cur - 1u;
#pragma unroll
                for (int k = 0; k < K2_SORT_MAX; ++k) {
                    if ((uint32_t)k < len) { const uint32_t lo = min(idx[k], v), hi = max(idx[k], v); idx[k] = lo; v = hi; }
                    else if ((uint32_t)k == len) idx[k] = v;
                }
            }
            len++;
        }
        if (len <= K2_SORT_MAX) {
#pragma unroll
            for (int k = 0; k < K2_SORT_MAX; ++k) {
                if ((uint32_t)k < len) {
                    const agr_k2op op = s.ops[idx[k]];
                    s.eff[idx[k]] = (uint8_t)k2_apply_op(r, op.kh, op.seq, cnt);
                    k2_note_bytes<BYTES>(b, idx[k], op.kh, wr, we);
                }
            }
        } else {
            long long last = -1;
            for (;;) {                                                     // next op of this row in ascending op index
                uint32_t best = 0xffffffffu;
                for (uint32_t cur = j + 1u; cur != 0u; cur = __ldcg(&s.nxt[cur - 1u])) {
                    const uint32_t o = cur - 1u;
                    if ((long long)o > last && o < best) best = o;
                }
                if (best == 0xffffffffu) break;
                last = best;
                const agr_k2op op = s.ops[best];
                s.eff[best] = (uint8_t)k2_apply_op(r, op.kh, op.seq, cnt);
                k2_note_bytes<BYTES>(b, best, op.kh, wr, we);
            }
        }
    }
    if (BYTES) {
        if (wr >= 0) {
            b->resp_off[rid] = b->base + b->dst[wr];
            b->resp_len[rid] = (uint32_t)(b->src_off[wr + 1] - b->src_off[wr]);
            b->resp_hlen[rid] = b->hlen ? b->hlen[wr] : 0u;
            s.eff[wr] |= (uint8_t)K2_EFF_WIN;
        }
        if (we >= 0) {
            b->err_off[rid] = b->base + b->dst[we];
            b->err_len[rid] = (uint32_t)(b->src_off[we + 1] - b->src_off[we]);
            s.eff[we] |= (uint8_t)K2_EFF_WIN;
        }
    }
    d.state[rid] = r.st;
    d.aux[rid] = r.aux;
    if (r.responded) d.ptime[rid] = r.ptime;
    if (r.written) {
        // mtime 0 reads "K2 never SET this row" in the sweep (it then takes created_at): a SET at time 0 counts as one at 1 ns
        const unsigned long long t = r.mtime ? r.mtime : 1ULL;
        d.mtime[rid] = t;
        unsigned long long* cm = d.cmin + rid / AGR_CHUNK_ROWS;             // the TTL sweep's bound must stay a lower bound
        const unsigned long long cur = __ldcg(cm), b = t < ~0ULL ? t : ~0ULL - 1ULL;  // (~0 means "no stored row")
        if (cur != 0ULL && cur != ~0ULL && b < cur) atomicMin(cm, b);   // (0: unknown, ~0: never swept / empty — both are recomputed)
    }
    d.head[rid] = 0;
}
