// agr_kernels.cu — sm_90a kernels of the request path.
//
//   K1  k1_post, k1_index (the TMA kernel is in agr_k1_tma.cu, the variable-length one in agr_k1_var.cu)
//                                                                 (requests.go:64-117, server.go:493-557)
//   K2  k2_link / k2_apply / k2_append; with bytes (agr_complete_ex) k2_apply_bytes and k2_copy_bytes
//                                                                 (requests.go:120-194,228-275, server.go:583-615)
//   K3  k3_pass<count|scatter> / k3_scan_groups / k3_scan_total / k3_gather, k_resolve, k_verify, k_drop_*
//                                                                 (replay_worker.go:58-117, requests.go:197-225)
//
// All arithmetic is integer / byte work bounded by HBM bandwidth; there is no tensor-core work on this path.
#include "agr_device.cuh"


// Post pass over the batch's route words (4 B / record; the records themselves are re-read only for the rare rows
// that need it).  Runs after ALL inserts of the batch:
//   (a) replay-flagged rows: resolve replay_of in the dedupe index -> KNOWN (dedupe hit), compared by row id so that
//       "known" means "stored EARLIER in arrival order";
//   (b) only if some row found its id already present (dupfix != 0 — never with minted UUIDs): owner of an id = the
//       LOWEST row that carried it (final inv_rid).  A provisionally stored row that is not the owner is demoted to a
//       persistence failure (server.go:511-514); a provisional duplicate that IS the owner (it lost the CAS race to a
//       later row of the same batch) is promoted to stored.
__global__ void __launch_bounds__(256) k1_post(const agr_dev d, const uint32_t first_rid, const uint32_t n, uint2* __restrict__ verdicts,
                                               uint4* __restrict__ ids, const uint32_t* __restrict__ marks) {
    const uint32_t dupfix = __ldcg(d.dupfix);
    if (blockIdx.x == 0 && threadIdx.x < 4) d.dupfix_next[threadIdx.x] = 0;      // the previous batch is done with these words
    // nothing to do: no in-batch id races, no replay-flagged records to resolve, nobody asked for verdicts or ids
    if (dupfix == 0u && __ldcg(d.dupfix + 2) == 0u && verdicts == nullptr && ids == nullptr) return;
    const uint32_t stride = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    const unsigned long long first_log = row_logical(d, first_rid);
    int delta[3] = {0, 0, 0};                                                     // dedupe hits, stored, queued
    if (marks && dupfix == 0u && (d.cfg_flags & AGR_CFG_MINT_IDS) && verdicts == nullptr && ids == nullptr) {
        // minted ids: K1 has decided every replay that names a row of an earlier batch, so the few rows left are far apart.  One
        // thread per marks word (agr_launch_k1 sizes the grid for n / 32 threads) walks the word's set bits.
        for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < (n + 31u) / 32u; w += stride) {
            for (uint32_t m = __ldg(&marks[w]); m != 0u; m &= m - 1u) k1_post_one(d, first_rid + w * 32u + (uint32_t)(__ffs(m) - 1), 0u, delta, true);
        }
    } else {
        for (uint32_t i0 = blockIdx.x * blockDim.x; i0 < n; i0 += stride) {
            const uint32_t i = i0 + threadIdx.x;
            if (i >= n) continue;
            // with the K1 kernel's row marks and nothing else to do for unmarked rows, 4 B per 32 rows decide who stays
            const bool marked = marks && ((__ldg(&marks[i >> 5]) >> (i & 31u)) & 1u);
            if (marks && !marked && dupfix == 0u && verdicts == nullptr && ids == nullptr) continue;
            const uint32_t rid = first_rid + i;
            const uint32_t r = k1_post_one(d, rid, dupfix, delta, marked, first_log);
            if (verdicts) verdicts[i] = k1_verdict_word(r);
            if (ids) ids[i] = k1_request_id(d, rid);
        }
    }
    // counter corrections: one global atomic per CTA and counter (thousands of warps adding to the same three words would
    // serialise in L2 for longer than the pass itself takes)
    __shared__ int s_delta[3];
    if (threadIdx.x < 3) s_delta[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int v = __reduce_add_sync(FULL, delta[k]);
        if (lane == 0 && v) atomicAdd(&s_delta[k], v);
    }
    __syncthreads();
    if (threadIdx.x == 0) { int tot[3] = {s_delta[0], s_delta[1], s_delta[2]}; k1_post_apply(d, tot); }
}

// The dedupe-index insert of every stored row, one thread per row at full occupancy (agr_launch_reindex: rebuilds the index
// after the restore of an append-only engine, whose index holds every row K1 ever stored).  A row whose id is already present becomes a provisional duplicate (k1_post decides).
__global__ void __launch_bounds__(256) k1_index(const agr_dev d, const uint32_t first_rid, const uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int dups = 0, q2u = 0;
    if (i < n) {
        const uint32_t rid = first_rid + i;
        uint32_t r = d.route[rid];
        uint32_t vf = rt_flags(r);
        if (vf & AGR_VF_STORED) {
            const uint4 h0 = ldg_nc_v4(rec_ptr(d, rid));
            const u128 key = make_u128(pack64(h0.x, h0.y), pack64(h0.z, h0.w));
            unsigned long long idx = agr_hash_id(pack64(h0.x, h0.y), pack64(h0.z, h0.w)) & d.table_mask;
            bool dup = false;
            for (;;) {
                const u128 old = cas128(&d.table[idx], 0, key);
                if (old == 0) break;
                if (old == key) { dup = true; break; }
                idx = (idx + 1) & d.table_mask;
            }
            asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(&d.table[idx].inv_rid), "r"(idx_encode(d, rid)) : "memory");
            if (dup) {
                asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(d.dupfix) : "memory");
                uint32_t code = rt_code(r);
                if (code == AGR_V_QUEUED) { code = AGR_V_UNAVAILABLE; q2u = 1; }
                vf = (vf & ~(AGR_VF_STORED | AGR_VF_TRACKED)) | AGR_VF_DUP_ID;
                d.route[rid] = rt_slot(r) | (code << RT_CODE_SHIFT) | (vf << RT_FLAG_SHIFT);
                d.state[rid] = 0;
                dups = 1;
            }
        }
    }
    dups = __reduce_add_sync(FULL, dups);
    q2u = __reduce_add_sync(FULL, q2u);
    if (lane == 0 && dups) {
        atomicAdd(&d.ctr[C_STORED], (unsigned long long)(long long)(-dups));
        atomicAdd(&d.ctr[C_DUP_IDS], (unsigned long long)dups);
        if (q2u) {
            atomicAdd(&d.ctr[C_QUEUED], (unsigned long long)(long long)(-q2u));
            atomicAdd(&d.ctr[C_UNAVAILABLE], (unsigned long long)q2u);
        }
    }
}

// integrity sweep over physical rows [first, first + rows): warp per row, recompute the position-weighted checksum of the
// stored bytes and compare
__global__ void __launch_bounds__(256) k_verify(const agr_dev d, const unsigned long long first, const unsigned long long rows,
                                                unsigned long long* __restrict__ bad) {
    const unsigned long long w = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= rows) return;
    const uint32_t rid = (uint32_t)(first + w);
    if (d.ring_rows && !(d.state[rid] & ST_STORED)) return;    // ring: released / skipped rows hold no record
    const uint8_t* src = rec_ptr(d, rid);
    const uint32_t chunks = d.voff ? (d.vlen[rid] >> 4) : 32u;
    uint32_t c0 = 0, c1 = 0;
    for (uint32_t c = lane; c < chunks; c += 32) {
        const uint4 v = ldg_nc_v4(src + (size_t)c * 16);
        c0 += v.x + v.y + v.z + v.w;
        c1 += (4 * c + 1) * v.x + (4 * c + 2) * v.y + (4 * c + 3) * v.z + (4 * c + 4) * v.w;
    }
    c0 = __reduce_add_sync(FULL, c0);
    c1 = __reduce_add_sync(FULL, c1);
    if (lane == 0 && agr_cksum_pack(c0, c1) != d.cksum[rid]) atomicAdd(bad, 1ULL);
}
// TTL sweep: the reference stores every record with SET ... EX 24h (requests.go:106,175,270); a record whose last SET is
// ttl or more in the past is gone (GET misses), while its id stays in whatever lists hold it.
// One CTA per chunk of AGR_CHUNK_ROWS physical rows.  cmin[c] is a lower bound of the last-SET times of the chunk's stored
// rows (~0 = no stored row, 0 = unknown: after a restore): K1 lowers it to a tile's earliest created_at when it stores the
// tile (k1_note_time), K2 lowers it if an outcome carries an older time, and this sweep replaces it by the exact minimum of
// what it leaves behind.  A chunk whose bound says nothing can have expired costs one 8-byte load instead of a sweep, so
// a periodic call reads only the chunks that are due.
#define EXP_PER_THREAD (AGR_CHUNK_ROWS / 256u)
__global__ void __launch_bounds__(256) k_expire(const agr_dev d, const unsigned long long rows, const unsigned long long now,
                                                const unsigned long long ttl, unsigned long long* __restrict__ expired) {
    __shared__ unsigned long long s_min[8];
    __shared__ uint32_t s_cnt;
    const uint32_t c = blockIdx.x;
    const unsigned long long cm = d.cmin[c];
    if (cm == ~0ULL) return;
    if (cm != 0ULL && (now < cm || now - cm < ttl)) return;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const unsigned long long r0 = (unsigned long long)c * AGR_CHUNK_ROWS;
    // three rounds of independent loads (state words, then the K2 times, then created_at of the rows K2 never wrote) instead
    // of a dependent chain per row
    uint32_t st[EXP_PER_THREAD];
    unsigned long long t[EXP_PER_THREAD];
#pragma unroll
    for (uint32_t q = 0; q < EXP_PER_THREAD; ++q) {
        const unsigned long long rid = r0 + threadIdx.x + q * 256u;
        st[q] = rid < rows ? d.state[rid] : 0u;
    }
#pragma unroll
    for (uint32_t q = 0; q < EXP_PER_THREAD; ++q) {
        const unsigned long long rid = r0 + threadIdx.x + q * 256u;
        t[q] = (st[q] & ST_STORED) ? d.mtime[rid] : 1ULL;
    }
#pragma unroll
    for (uint32_t q = 0; q < EXP_PER_THREAD; ++q) {
        const unsigned long long rid = r0 + threadIdx.x + q * 256u;
        if ((st[q] & ST_STORED) && t[q] == 0ULL) t[q] = __ldcs(reinterpret_cast<const unsigned long long*>(rec_ptr(d, (uint32_t)rid) + AGR_OFF_SEQ));
    }
    // a SET at time 0 counts as one at 1 ns everywhere (0 is "never SET" in mtime and "unknown" in the bound), and a row kept
    // at time ~0 enters the bound as ~0 - 1 (~0 is "no stored row", which would let k_first_live skip the chunk)
    unsigned long long lmin = ~0ULL;
    uint32_t gone = 0;
#pragma unroll
    for (uint32_t q = 0; q < EXP_PER_THREAD; ++q) {
        if (!(st[q] & ST_STORED)) continue;
        const unsigned long long rid = r0 + threadIdx.x + q * 256u;
        const unsigned long long tq = t[q] ? t[q] : 1ULL;
        if (now >= tq && now - tq >= ttl) { d.state[rid] = st[q] & ~ST_STORED; gone++; }
        else lmin = min(lmin, min(tq, ~0ULL - 1ULL));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(FULL, lmin, o); if (y < lmin) lmin = y; }
    gone = __reduce_add_sync(FULL, gone);
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = lmin; if (gone) atomicAdd(&s_cnt, gone); }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 1; w < 8; ++w) if (s_min[w] < lmin) lmin = s_min[w];
        if (s_cnt && expired) atomicAdd(expired, (unsigned long long)s_cnt);
        d.cmin[c] = lmin;                                       // exact now (~0: the chunk holds no stored row any more)
    }
}
void agr_launch_expire(const agr_dev& d, unsigned long long rows, unsigned long long now, unsigned long long ttl,
                       unsigned long long* expired, cudaStream_t st) {
    if (rows) k_expire<<<(unsigned)((rows + AGR_CHUNK_ROWS - 1) / AGR_CHUNK_ROWS), 256, 0, st>>>(d, rows, now, ttl, expired);
}
// ---- ring mode (AGR_CFG_RING): releasing rows at the tail
// offset (from the tail) of the first row that still holds a stored record, among the `live` rows behind the tail.
// One CTA per PHYSICAL chunk of the ring (the chunks of the TTL sweep).  A chunk that lies behind an offset already found has
// nothing to add; with use_cmin (fixed-stride ring: K1 and K2 keep the chunk bounds current) a chunk whose bound says "no stored
// row" costs one 8-byte load — after a sweep that is every chunk up to the one the answer lies in.
// The last CTA to finish packs what agr_reclaim needs on the host into one 32-byte record — the offset found, both log lengths
// and (variable-length mode) the byte offset of the first live row's record — writes it straight into the pinned host buffer
// `out`, and re-arms the two scratch words (offset = "none", ticket = 0) for the next scan: no memset, no copy, one launch.
__global__ void __launch_bounds__(256) k_first_live(const agr_dev d, const unsigned long long live, const uint32_t use_cmin,
                                                    uint32_t* __restrict__ scratch /* [0] offset found, [1] ticket */,
                                                    unsigned long long* __restrict__ out) {
    __shared__ uint32_t s_last;
    uint32_t* out_off = scratch;
    const unsigned long long R = d.ring_rows, tp = d.tail_phys;
    const unsigned long long p0 = (unsigned long long)blockIdx.x * AGR_CHUNK_ROWS;
    const bool holds_tail = tp >= p0 && tp < p0 + AGR_CHUNK_ROWS;
    const unsigned long long kmin = holds_tail ? 0ULL : (p0 + R - tp) % R;      // smallest offset of a row of this chunk
    bool work = kmin < live && *reinterpret_cast<volatile uint32_t*>(out_off) >= kmin;
    if (work && use_cmin && d.cmin[blockIdx.x] == ~0ULL) work = false;
    if (work) {
        uint32_t st[EXP_PER_THREAD];
        unsigned long long kk[EXP_PER_THREAD];
#pragma unroll
        for (uint32_t q = 0; q < EXP_PER_THREAD; ++q) {
            const unsigned long long p = p0 + threadIdx.x + q * 256u;
            kk[q] = (p >= tp) ? p - tp : p + R - tp;
            st[q] = (p < R && kk[q] < live) ? d.state[p] : 0u;
        }
        uint32_t mine = 0xffffffffu;
#pragma unroll
        for (uint32_t q = 0; q < EXP_PER_THREAD; ++q)
            if ((st[q] & ST_STORED) && (uint32_t)kk[q] < mine) mine = (uint32_t)kk[q];
        mine = __reduce_min_sync(FULL, mine);
        if ((threadIdx.x & 31) == 0 && mine != 0xffffffffu) atomicMin(out_off, mine);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = (atomicAdd(scratch + 1, 1u) == gridDim.x - 1u) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
        __threadfence();
        const uint32_t o = *reinterpret_cast<volatile uint32_t*>(out_off);
        out[1] = d.log_len[0]; out[2] = d.log_len[1];
        out[3] = (d.voff && o != 0xffffffffu) ? d.voff[row_physical(d, d.tail + o)] : 0ULL;
        out[0] = o;
        scratch[0] = 0xffffffffu; scratch[1] = 0u;
    }
}
void agr_launch_first_live(const agr_dev& d, unsigned long long live, bool use_cmin, uint32_t* scratch, void* out, cudaStream_t st) {
    k_first_live<<<(unsigned)((d.ring_rows + AGR_CHUNK_ROWS - 1) / AGR_CHUNK_ROWS), 256, 0, st>>>(d, live, use_cmin ? 1u : 0u, scratch,
                                                                                                 (unsigned long long*)out);
}
// rows tail .. tail + count go back to the pool: every per-row word reads "no record"
__global__ void __launch_bounds__(256) k_release_rows(const agr_dev d, const uint32_t count, uint32_t* __restrict__ resp_len,
                                                      uint32_t* __restrict__ resp_hlen, uint32_t* __restrict__ err_len) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const uint32_t p = row_physical(d, d.tail + k);
    d.state[p] = 0; d.route[p] = 0; d.aux[p] = 0; d.head[p] = 0; d.ptime[p] = 0; d.mtime[p] = 0;
    resp_len[p] = 0; resp_hlen[p] = 0; err_len[p] = 0;      // (the chunk's time bound stays a valid lower bound of what is left)
}
void agr_launch_release_rows(const agr_dev& d, uint32_t count, uint32_t* resp_len, uint32_t* resp_hlen, uint32_t* err_len, cudaStream_t st) {
    if (count) k_release_rows<<<(count + 255u) / 256u, 256, 0, st>>>(d, count, resp_len, resp_hlen, err_len);
}
// how far back from the byte slab's head (physical offset `head`) the oldest blob lies that a live row still refers to
__global__ void __launch_bounds__(256) k_bytes_span(const agr_dev d, const unsigned long long head, const unsigned long long cap,
                                                    const unsigned long long* __restrict__ resp_off, const uint32_t* __restrict__ resp_len,
                                                    const unsigned long long* __restrict__ err_off, const uint32_t* __restrict__ err_len,
                                                    unsigned long long* __restrict__ span) {
    const unsigned long long live = d.head_l - d.tail;
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long mine = 0;
    if (k < live) {
        const uint32_t p = row_physical(d, d.tail + k);
        if (resp_len[p]) { unsigned long long dist = (head + cap - resp_off[p]) % cap; if (dist == 0) dist = cap; mine = dist; }
        if (err_len[p]) { unsigned long long dist = (head + cap - err_off[p]) % cap; if (dist == 0) dist = cap; if (dist > mine) mine = dist; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(FULL, mine, o); if (y > mine) mine = y; }
    if ((threadIdx.x & 31) == 0 && mine) atomicMax(span, mine);
}
void agr_launch_bytes_span(const agr_dev& d, unsigned long long head, unsigned long long cap, const unsigned long long* resp_off,
                           const uint32_t* resp_len, const unsigned long long* err_off, const uint32_t* err_len, unsigned long long* span,
                           cudaStream_t st) {
    const unsigned long long live = d.head_l - d.tail;
    if (live) k_bytes_span<<<(unsigned)((live + 255) / 256), 256, 0, st>>>(d, head, cap, resp_off, resp_len, err_off, err_len, span);
}
// stable compaction of a log: entries whose row is among the `released` rows at the tail drop out
#define LC_CHUNK 1024u
__device__ __forceinline__ bool log_keep(const agr_dev& d, uint32_t p, uint32_t released) {
    if (p == AGR_RID_NONE) return false;
    const uint32_t off = p >= d.tail_phys ? p - d.tail_phys : p + d.ring_rows - d.tail_phys;   // distance from the tail
    return off >= released;
}
__global__ void __launch_bounds__(256) k_log_count(const agr_dev d, const uint32_t* __restrict__ log, const unsigned long long len,
                                                   const uint32_t released, uint32_t* __restrict__ chunk_cnt) {
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const unsigned long long base = (unsigned long long)blockIdx.x * LC_CHUNK;
    uint32_t c = 0;
    for (uint32_t j = threadIdx.x; j < LC_CHUNK; j += 256) {
        const unsigned long long i = base + j;
        if (i < len && log_keep(d, log[i], released)) c++;
    }
    c = __reduce_add_sync(FULL, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) chunk_cnt[blockIdx.x] = s_cnt;
}
// exclusive scan of the chunk counts; the new length goes to *log_len.  Entries K2 pushed after the first `len` (agr_reclaim_async
// compacts what its scan saw one step later) name rows that were stored when they were pushed, never released ones: they are
// copied after the kept ones as they are.
__global__ void __launch_bounds__(1024) k_log_scan(uint32_t* chunk_cnt, const uint32_t nchunks, const uint32_t* __restrict__ log,
                                                   const unsigned long long len, uint32_t* __restrict__ out,
                                                   unsigned long long* log_len) {
    __shared__ uint32_t s_w[32];
    __shared__ uint32_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nchunks; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < nchunks ? chunk_cnt[i] : 0u;
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(FULL, x, o); if (lane >= o) x += y; }
        if (lane == 31) s_w[warp] = x;
        __syncthreads();
        uint32_t pre = s_carry;
        for (int k = 0; k < warp; ++k) pre += s_w[k];
        if (i < nchunks) chunk_cnt[i] = pre + x - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = pre + x;
        __syncthreads();
    }
    const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(log_len), kept = s_carry;
    for (unsigned long long i = len + threadIdx.x; i < cur; i += 1024) out[kept + (i - len)] = log[i];
    __syncthreads();
    if (threadIdx.x == 0) { chunk_cnt[nchunks] = s_carry; *log_len = kept + (cur - len); }
}
// one warp per chunk keeps the order: 32 entries per step, ballot + popc
__global__ void __launch_bounds__(32) k_log_scatter(const agr_dev d, const uint32_t* __restrict__ log, const unsigned long long len,
                                                    const uint32_t released, const uint32_t* __restrict__ chunk_off, uint32_t* __restrict__ out) {
    const int lane = threadIdx.x;
    const unsigned long long base = (unsigned long long)blockIdx.x * LC_CHUNK;
    uint32_t pos = chunk_off[blockIdx.x];
    for (uint32_t j = 0; j < LC_CHUNK; j += 32) {
        const unsigned long long i = base + j + lane;
        const uint32_t v = i < len ? log[i] : AGR_RID_NONE;
        const bool keep = i < len && log_keep(d, v, released);
        const uint32_t m = __ballot_sync(FULL, keep);
        if (keep) out[pos + __popc(m & ((1u << lane) - 1u))] = v;
        pos += __popc(m);
    }
}
void agr_launch_log_compact(const agr_dev& d, const uint32_t* log, unsigned long long len, uint32_t released, uint32_t* out,
                            uint32_t* chunk_cnt, unsigned long long* new_len, cudaStream_t st) {
    if (!len) return;
    const uint32_t nch = (uint32_t)((len + LC_CHUNK - 1) / LC_CHUNK);
    k_log_count<<<nch, 256, 0, st>>>(d, log, len, released, chunk_cnt);
    k_log_scan<<<1, 1024, 0, st>>>(chunk_cnt, nch, log, len, out, new_len);
    k_log_scatter<<<nch, 32, 0, st>>>(d, log, len, released, chunk_cnt, out);
}

void agr_launch_verify(const agr_dev& d, unsigned long long first, unsigned long long rows, unsigned long long* bad, cudaStream_t st) {
    if (rows) k_verify<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(d, first, rows, bad);
}
// hash-id ring: rebuild of the dedupe index over a range of physical rows — only rows that still hold a record go in (a release,
// a restore: ring_reindex_locked)
__global__ void __launch_bounds__(256) k_reindex_range(const agr_dev d, const uint32_t first, const uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t rid = first + i;
    if (!(d.state[rid] & ST_STORED)) return;
    const uint4 h0 = ldg_nc_v4(rec_ptr(d, rid));
    const u128 key = make_u128(pack64(h0.x, h0.y), pack64(h0.z, h0.w));
    unsigned long long idx = agr_hash_id(pack64(h0.x, h0.y), pack64(h0.z, h0.w)) & d.table_mask;
    for (;;) {
        const u128 old = cas128(&d.table[idx], 0, key);
        if (old == 0 || old == key) break;
        idx = (idx + 1) & d.table_mask;
    }
    asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(&d.table[idx].inv_rid), "r"(idx_encode(d, rid)) : "memory");
}
void agr_launch_reindex_range(const agr_dev& d, uint32_t first, uint32_t n, cudaStream_t st) {
    if (n) k_reindex_range<<<(n + 255u) / 256u, 256, 0, st>>>(d, first, n);
}
// rebuild of the dedupe index from restored rows (hash-id mode, append-only): k1_index over every row K1 stored
void agr_launch_reindex(const agr_dev& d, uint32_t rows, cudaStream_t st) {
    if (rows) k1_index<<<(rows + 255u) / 256u, 256, 0, st>>>(d, 0u, rows);
}

static uint32_t k1_post_blocks(uint32_t n, int sm_count) {
    uint32_t b = (n + 255u) / 256u, cap = (uint32_t)sm_count * 16u;
    return b < cap ? b : cap;
}

cudaError_t agr_launch_k1_tma(const void* map, const agr_dev& d, uint32_t first_rid, unsigned long long first_log, uint32_t n,
                              int sm_count, cudaStream_t st);

void agr_launch_k1_post(const agr_dev& d, uint32_t first_rid, uint32_t n, int sm_count, cudaStream_t st, void* verdicts, void* ids,
                        const uint32_t* marks) {
    if (n) k1_post<<<k1_post_blocks(n, sm_count), 256, 0, st>>>(d, first_rid, n, (uint2*)verdicts, (uint4*)ids, marks);
}

int agr_launch_k1(const agr_dev& d, uint32_t first_rid, unsigned long long first_log, uint32_t n, const void* tmap,
                  int sm_count, cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, void* verdicts, void* ids) {
    if (n == 0) return 0;
    if (ev0) cudaEventRecord(ev0, st);
    // minted ids never race for an id (dupfix stays 0) and the TMA kernel decides every replay's dedupe hit itself: without
    // verdicts or ids to write there is nothing left for k1_post, and the kernel neither marks rows nor needs the pass
    const bool post = !(d.cfg_flags & AGR_CFG_MINT_IDS) || verdicts != nullptr || ids != nullptr;
    agr_dev dk = d;
    if (!post) dk.marks = nullptr;
    agr_launch_k1_tma(tmap, dk, first_rid, first_log, n, sm_count, st);
    if (ev1) cudaEventRecord(ev1, st);
    if (!post) return 1;
    // minted ids never race for an id (dupfix stays 0): without verdicts or ids to write, k1_post visits the marked rows only
    const bool sparse = d.marks && (d.cfg_flags & AGR_CFG_MINT_IDS) && verdicts == nullptr && ids == nullptr;
    k1_post<<<k1_post_blocks(sparse ? (n + 31u) / 32u : n, sm_count), 256, 0, st>>>(d, first_rid, n, (uint2*)verdicts, (uint4*)ids, d.marks);
    return 2;
}

// ------------------------------------------------------------------------------------------------ K2
// Outcomes must be applied in array order per record (MarkRequestFailed then StoreResponse is not the same as the
// reverse, KAT-H).  Three launches (device functions in agr_device.cuh, shared with the service kernel of agr_svc.cu):
//   k2_link   reads the caller's 64 B outcome, resolves the agent id in the device agent table and the request id to its
//             row, writes a 16 B op {row, kind|http, seq} and threads the outcomes of one row onto a chain rooted in head[row];
//   k2_apply  the chain root replays its row's outcomes in ascending op index on a private copy of the state word (Q24's
//             lost updates cannot happen) and notes which ops push to the completed / failed lists;
//   k2_append one pass with decoupled look-back: the pushes are appended in op order (RPUSH order == call order, Q7) and
//             the last tile moves the log tails.
__global__ void __launch_bounds__(256) k2_link(const agr_dev d, const uint8_t* __restrict__ outs, const agr_k2_scratch s, const uint32_t n) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint8_t* o = outs + (size_t)j * 64;
    const uint4 id = ldg_nc_v4(o), a0 = ldg_nc_v4(o + 16), a1 = ldg_nc_v4(o + 32), t = ldg_nc_v4(o + 48);
    k2_link_one(d, s, j, id, a0, a1, t);
}

// read-only resolve of (agent slot, request id) -> rid, used by agr_get_record
__global__ void __launch_bounds__(256) k_resolve(const agr_dev d, const agr_dop* __restrict__ ops, uint32_t* __restrict__ hrid, const uint32_t n) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const agr_dop op = ops[j];
    uint32_t rid = AGR_RID_NONE;
    const uint32_t cand = lookup_rid(d, op.id_lo, op.id_hi);
    if (cand != AGR_RID_NONE && (d.state[cand] & ST_STORED) && rt_slot(d.route[cand]) == op.slot) rid = cand;
    hrid[j] = rid;
}
void agr_launch_resolve(const agr_dev& d, const agr_dop* ops, uint32_t* hrid, uint32_t n, cudaStream_t st) {
    if (n) k_resolve<<<(n + 255u) / 256u, 256, 0, st>>>(d, ops, hrid, n);
}

template <bool BYTES>
__device__ __forceinline__ void k2_apply_body(const agr_dev& d, const agr_k2_scratch& s, const uint32_t n, const agr_k2_bytes* b) {
    __shared__ uint32_t s_cnt[3];
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    uint32_t cnt[3] = {0u, 0u, 0u};                                  // completions, errors, dead-lettered
    if (j < n) k2_apply_one<BYTES>(d, s, j, cnt, b);
    // one global atomic per CTA and counter: a million outcomes are 32 K warps, and that many adds to one word serialise in L2
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint32_t v = __reduce_add_sync(FULL, cnt[k]);
        if (lane == 0 && v) atomicAdd(&s_cnt[k], v);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_cnt[0]) atomicAdd(&d.ctr[C_COMPLETIONS], (unsigned long long)s_cnt[0]);
        if (s_cnt[1]) atomicAdd(&d.ctr[C_FAILURES], (unsigned long long)s_cnt[1]);
        if (s_cnt[2]) atomicAdd(&d.ctr[C_DEAD_LETTERED], (unsigned long long)s_cnt[2]);
    }
}
__global__ void __launch_bounds__(256) k2_apply(const agr_dev d, const agr_k2_scratch s, const uint32_t n) {
    k2_apply_body<false>(d, s, n, nullptr);
}
__global__ void __launch_bounds__(256) k2_apply_bytes(const agr_dev d, const agr_k2_scratch s, const uint32_t n, const agr_k2_bytes b) {
    k2_apply_body<true>(d, s, n, &b);
}

// One warp per op: copies the segments of the ops k2_apply_bytes marked K2_EFF_WIN from the staged batch into their 16-byte
// aligned places in the byte slab (losers' places stay unused).
__global__ void __launch_bounds__(256) k2_copy_bytes(const agr_k2_scratch s, const agr_k2_bytes b, const uint32_t n) {
    const uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (j >= n || !(s.eff[j] & K2_EFF_WIN)) return;
    const unsigned long long o = b.src_off[j];
    warp_copy16(reinterpret_cast<uint4*>(b.slab + b.base + b.dst[j]), b.src + (o - b.src_off[0]), (uint32_t)(b.src_off[j + 1] - o), lane);
}

// Order-preserving append of the batch's completed / failed pushes.  Tiles of K2_TILE ops are claimed through a ticket (so a
// tile's predecessors are always running or done) and chained with decoupled look-back: a tile publishes its aggregate
// {completed, failed} count, then its inclusive prefix once the look-back over its predecessors has found one.
// tile word: flag(2) << 62 | completed(31) << 31 | failed(31);  flag 1 = aggregate, 2 = inclusive prefix.
#define K2_TILE 2048u
__global__ void __launch_bounds__(256) k2_append(const agr_dev d, const agr_k2_scratch s, const uint32_t n) {
    __shared__ uint32_t s_tile;
    __shared__ uint32_t s_wc[8], s_wf[8];
    __shared__ unsigned long long s_prefix;
    const unsigned long long base_c = d.log_len[0], base_f = d.log_len[1];   // read before this tile publishes anything
    if (threadIdx.x == 0) s_tile = atomicAdd(s.ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile, ntiles = (n + K2_TILE - 1u) / K2_TILE;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // thread t owns 8 consecutive ops of the tile: one 8-byte load of their effect bytes
    const uint32_t k0 = tile * K2_TILE + threadIdx.x * 8u;
    unsigned long long eff8 = 0;
    if (k0 + 8u <= n) eff8 = *reinterpret_cast<const unsigned long long*>(s.eff + k0);
    else for (uint32_t q = 0; k0 + q < n && q < 8u; ++q) eff8 |= (unsigned long long)s.eff[k0 + q] << (8u * q);
    const uint32_t mc = __popcll(eff8 & 0x0101010101010101ULL), mf = __popcll(eff8 & 0x0202020202020202ULL);
    uint32_t xc = mc, xf = mf;                                        // inclusive scan inside the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t yc = __shfl_up_sync(FULL, xc, o), yf = __shfl_up_sync(FULL, xf, o);
        if (lane >= o) { xc += yc; xf += yf; }
    }
    if (lane == 31) { s_wc[warp] = xc; s_wf[warp] = xf; }
    __syncthreads();
    uint32_t pc = 0, pf = 0, tc = 0, tf = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { if (w < warp) { pc += s_wc[w]; pf += s_wf[w]; } tc += s_wc[w]; tf += s_wf[w]; }
    if (warp == 0) {
        volatile unsigned long long* st = s.tiles;
        unsigned long long excl = 0;
        if (tile == 0) {
            if (lane == 0) { st[0] = (2ULL << 62) | ((unsigned long long)tc << 31) | tf; }
        } else {
            if (lane == 0) { st[tile] = (1ULL << 62) | ((unsigned long long)tc << 31) | tf; }
            __threadfence();
            // look back 32 tiles at a time: lane l looks at tile - 1 - l
            long long look = (long long)tile - 1;
            for (;;) {
                const long long mine = look - lane;
                unsigned long long v = 0;
                if (mine >= 0) { do { v = st[mine]; } while ((v >> 62) == 0ULL); }
                const uint32_t incl_mask = __ballot_sync(FULL, mine >= 0 && (v >> 62) == 2ULL);
                const int stop = incl_mask ? __ffs(incl_mask) - 1 : 32;          // nearest predecessor with an inclusive prefix
                unsigned long long add = (mine >= 0 && lane <= stop) ? (v & 0x3fffffffffffffffULL) : 0ULL;
#pragma unroll
                for (int o = 16; o; o >>= 1) add += __shfl_xor_sync(FULL, add, o);   // fields cannot carry into each other (sums <= n < 2^31)
                excl += add;
                if (incl_mask || look - 32 < 0) break;
                look -= 32;
            }
            if (lane == 0) {
                const unsigned long long incl = excl + (((unsigned long long)tc << 31) | tf);
                __threadfence();
                st[tile] = (2ULL << 62) | incl;
            }
        }
        if (lane == 0) s_prefix = excl;
    }
    __syncthreads();
    const unsigned long long ex = s_prefix;
    unsigned long long wc = base_c + (uint32_t)(ex >> 31) + pc + (xc - mc);
    unsigned long long wf = base_f + (uint32_t)(ex & 0x7fffffffULL) + pf + (xf - mf);
    if (eff8) {
#pragma unroll
        for (uint32_t q = 0; q < 8u; ++q) {
            const uint32_t f = (uint32_t)(eff8 >> (8u * q)) & 3u;
            if (f & 1u) { if (wc < d.log_cap) d.completed_log[wc] = s.ops[k0 + q].rid; wc++; }
            if (f & 2u) { if (wf < d.log_cap) d.failed_log[wf] = s.ops[k0 + q].rid; wf++; }
        }
    }
    if (tile == ntiles - 1u && threadIdx.x == 0) {                   // the last tile's inclusive prefix is the batch total
        unsigned long long nc = base_c + (uint32_t)(ex >> 31) + tc, nf = base_f + (uint32_t)(ex & 0x7fffffffULL) + tf;
        if (nc > d.log_cap || nf > d.log_cap) {
            atomicAdd(&d.ctr[C_LOG_OVERFLOW], 1ULL);
            *s.overflow = 1u;
            if (nc > d.log_cap) nc = d.log_cap;
            if (nf > d.log_cap) nf = d.log_cap;
        }
        d.log_len[0] = nc; d.log_len[1] = nf;
    }
}

uint32_t agr_k2_tiles(uint32_t n) { return (n + K2_TILE - 1u) / K2_TILE; }
void agr_launch_k2(const agr_dev& d, const void* outs, const agr_k2_scratch& s, uint32_t n, cudaStream_t st, const agr_k2_bytes* bytes) {
    if (n == 0) return;
    const uint32_t blocks = (n + 255u) / 256u, ntiles = agr_k2_tiles(n);
    cudaMemsetAsync(s.ticket, 0, (size_t)(ntiles + 1u) * 8u, st);   // {ticket, overflow}, then the batch's tile words
    k2_link<<<blocks, 256, 0, st>>>(d, (const uint8_t*)outs, s, n);
    if (bytes) k2_apply_bytes<<<blocks, 256, 0, st>>>(d, s, n, *bytes);
    else k2_apply<<<blocks, 256, 0, st>>>(d, s, n);
    k2_append<<<ntiles, 256, 0, st>>>(d, s, n);
    if (bytes) k2_copy_bytes<<<(n + 7u) / 8u, 256, 0, st>>>(s, *bytes, n);
}

// ------------------------------------------------------------------------------------------------ K3
// Stable agent-major partition of the selected items: output order = (agent slot ascending, item order ascending).
// Each warp owns a contiguous run of items; matrix[w][g] first holds the warp's per-group count, then (after the
// column scan) the position where warp w's first item of group g goes.  Inside a 32-item step match_any + popc
// give the stable rank — the warp-ballot agent-id partition.
struct k3_item { bool sel; uint32_t rid; uint32_t slot; bool inq; };

// q = pb + offset within a warp's run (< 2 * ring_rows + 2) back into the ring
__device__ __forceinline__ uint32_t k3_wrap(const agr_dev& d, uint32_t q) {
    if (d.ring_rows && q >= d.ring_rows) {
        q -= d.ring_rows;
        if (q >= d.ring_rows) q -= d.ring_rows;
    }
    return q;
}

// `st` = the row's state word (row modes; prefetched by the caller) — unused in log mode
// `prow` = the physical row of item `it` (row modes)
__device__ __forceinline__ k3_item k3_eval(const agr_dev& d, const agr_k3_params& p, unsigned long long it, uint32_t prow, uint32_t st, uint32_t rt) {
    k3_item o{false, AGR_RID_NONE, RT_SLOT_NONE, false};
    if (it >= p.hi) return o;
    if (p.mode == K3_LOG_AGENT) {
        const uint32_t rid = p.log[it];
        if (rid == AGR_RID_NONE) return o;
        o.rid = rid; o.slot = rt_slot(d.route[rid]);
        o.sel = (o.slot == p.slot);
        return o;
    }
    const uint32_t rid = prow;
    if (!(st & ST_INQ)) return o;                       // not in agent:{a}:requests:pending
    o.rid = rid; o.slot = rt_slot(rt);
    if (p.mode == K3_AGENT_PENDING_IDS) { o.sel = (o.slot == p.slot); return o; }   // LRANGE pending 0 -1
    // the record key has expired (agr_expire): its id stays in the list but GetPendingRequests skips it
    // (requests.go:210-213, Q10), so it is neither returned nor replayed, and it no longer holds the scan's low-water mark
    if (!(st & ST_STORED)) return o;
    o.inq = true;
    if (p.mode == K3_AGENT_PENDING) { o.sel = (o.slot == p.slot); return o; }   // GetPendingRequests, requests.go:197-225
    // K3_TICK: isAgentRunning (replay_worker.go:76-81,166-189) + the skip rule of :101
    if (d.astatus[o.slot] != AGR_AGENT_RUNNING) return o;
    if (st_status(st) == AGR_ST_PROCESSING || st_retry(st) >= st_max(st)) return o;
    if ((d.cfg_flags & AGR_CFG_SKIP_INFLIGHT) && (st & ST_INFLIGHT)) return o;  // extension, off in parity mode
    o.sel = true;
    return o;
}

// Two passes over a warp's contiguous run of items, but the row words are read ONCE:
//   k3_mark   reads state + route (or the log entry and its row's route), decides, leaves one selection bit per item in
//             selmask and the warp's per-group counts in its matrix row (shared-memory counters when groups <= K3_SMEM_GROUPS);
//   column scan (k3_colscan + k3_scan_total): matrix[w][g] = number of group-g items in warps < w, goff = group offsets;
//   k3_place  walks the selection bits (4 B per 32 items), fetches the agent slot of the SELECTED items only, and writes them
//             at goff[g] + matrix[w][g] + stable rank (match_any + popc: the warp-ballot agent-id partition).
#define K3_SMEM_GROUPS 512u
template <bool SMEM>
__global__ void __launch_bounds__(256) k3_mark(const agr_dev d, const agr_k3_params p) {
    extern __shared__ uint32_t s_rows[];
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const bool live = w < p.nwarps;                              // (a CTA's surplus warps only take part in its barrier)
    uint32_t* grow = p.matrix + (size_t)(live ? w : 0u) * p.groups;
    uint32_t* srow = s_rows + (size_t)(threadIdx.x >> 5) * p.groups;
    if (SMEM) {
        for (uint32_t g = lane; g < p.groups; g += 32) srow[g] = 0u;
        __syncwarp();
    }
    const unsigned long long b = p.lo + (unsigned long long)w * p.per_warp;
    unsigned long long e = live ? b + p.per_warp : b;
    if (e > p.hi) e = p.hi;
    if (!live) e = b;
    uint32_t mininq = AGR_RID_NONE;
    const bool rows = (p.mode != K3_LOG_AGENT);
    uint32_t* mask = p.selmask + (size_t)w * (p.per_warp >> 5);
    // physical row of item k: the warp's run is contiguous in the ring.  The window is [lo & ~3, hi) with hi - lo <= ring_rows,
    // so a run holds at most ring_rows + 3 items; one that starts at pb >= ring_rows - 2 (only when ring_rows % 4 != 0) wraps twice
    const uint32_t pb = rows ? row_physical(d, b) : 0u;
    auto prow_of = [&](unsigned long long k) -> uint32_t { return k3_wrap(d, pb + (uint32_t)(k - b)); };
    // Row modes, aligned run (the host rounds `lo` down to a multiple of 4; ring sizes that are not one take the scalar path): a lane
    // owns FOUR consecutive rows, so the row words arrive as two 16-byte loads per 128-row group instead of eight 4-byte ones;
    // the groups of 512 rows are in flight at once.  The selection bits are put together from the lanes' nibbles (three xor-shuffles).
    const bool vec = rows && ((pb | d.ring_rows | (uint32_t)p.per_warp) & 3u) == 0u;
    if (vec) {
        constexpr int NG = 4;
        uint4 st_v[NG], rt_v[NG]; uint32_t q_v[NG];
        for (unsigned long long k8 = b; k8 < e; k8 += 128u * NG) {
#pragma unroll
            for (int j = 0; j < NG; ++j) {
                const unsigned long long k = k8 + 128u * j + 4u * lane;
                q_v[j] = prow_of(k);
                const bool ok = k < e;                                // (e - b and hi need not be multiples of 4: k3_eval checks every row)
                st_v[j] = ok ? __ldcs(reinterpret_cast<const uint4*>(d.state + q_v[j])) : make_uint4(0u, 0u, 0u, 0u);
                rt_v[j] = ok ? __ldcs(reinterpret_cast<const uint4*>(d.route + q_v[j])) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int j = 0; j < NG; ++j) {
                const unsigned long long k0 = k8 + 128u * j;
                if (k0 >= e) break;
                const uint32_t st4[4] = {st_v[j].x, st_v[j].y, st_v[j].z, st_v[j].w}, rt4[4] = {rt_v[j].x, rt_v[j].y, rt_v[j].z, rt_v[j].w};
                uint32_t nib = 0u;
                if (__any_sync(FULL, ((st4[0] | st4[1] | st4[2] | st4[3]) & ST_INQ) != 0u)) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const unsigned long long kk = k0 + 4u * lane + i;
                        if (kk < p.lo_real || kk >= e) continue;
                        const k3_item it = k3_eval(d, p, kk, q_v[j] + i, st4[i], rt4[i]);
                        if (it.inq && (uint32_t)(kk - p.lo) < mininq) mininq = (uint32_t)(kk - p.lo);
                        if (it.sel) { atomicAdd((SMEM ? srow : grow) + ((p.groups == 1) ? 0u : it.slot), 1u); nib |= 1u << i; }
                    }
                }
                uint32_t v = nib << (4u * (lane & 7u));
                v |= __shfl_xor_sync(FULL, v, 1); v |= __shfl_xor_sync(FULL, v, 2); v |= __shfl_xor_sync(FULL, v, 4);
                if ((lane & 7) == 0) mask[((k0 - b) >> 5) + (lane >> 3)] = v;
            }
        }
    } else {
    // the row words of eight steps (256 rows) are in flight at once
    constexpr int NS = 8;
    uint32_t st_c[NS], rt_c[NS], pr_c[NS];
    for (unsigned long long k8 = b; k8 < e; k8 += 32u * NS) {
#pragma unroll
        for (int j = 0; j < NS; ++j) {
            const unsigned long long k = k8 + 32u * j + lane;
            pr_c[j] = prow_of(k);
            const bool ok = rows && k < e;
            st_c[j] = ok ? __ldcs(&d.state[pr_c[j]]) : 0u;
            rt_c[j] = ok ? __ldcs(&d.route[pr_c[j]]) : 0u;
        }
#pragma unroll
        for (int j = 0; j < NS; ++j) {
            const unsigned long long k0 = k8 + 32u * j;
            if (k0 >= e) break;
            const uint32_t st = st_c[j], rt = rt_c[j], pr = pr_c[j];
            uint32_t selbits = 0u;
            if (!rows || __any_sync(FULL, (st & ST_INQ) != 0u)) {                    // else: nothing pending in these 32 rows
                const bool in = k0 + lane >= p.lo_real;
                const k3_item it = in ? k3_eval(d, p, k0 + lane, pr, st, rt) : k3_item{false, AGR_RID_NONE, RT_SLOT_NONE, false};
                if (it.inq && (uint32_t)(k0 + lane - p.lo) < mininq) mininq = (uint32_t)(k0 + lane - p.lo);
                if (it.sel) atomicAdd((SMEM ? srow : grow) + ((p.groups == 1) ? 0u : it.slot), 1u);   // counting needs no order
                selbits = __ballot_sync(FULL, it.sel);
            }
            if (lane == 0) mask[(k0 - b) >> 5] = selbits;
        }
    }
    }
    if (SMEM) {
        __syncwarp();
        if (live) for (uint32_t g = lane; g < p.groups; g += 32) grow[g] = srow[g];
        // the CTA's eight warps own eight consecutive runs: their sum is the CTA's row of the (8x smaller) matrix the column scan
        // runs over; k3_place rebuilds a warp's offsets from the CTA's scanned row and the earlier warps' counts
        __syncthreads();
        for (uint32_t g = threadIdx.x; g < p.groups; g += 256) {
            uint32_t sum = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) sum += s_rows[(size_t)k * p.groups + g];
            p.cta_matrix[(size_t)blockIdx.x * p.groups + g] = sum;
        }
    }
    if (p.min_inq && p.mode == K3_TICK) {
        mininq = __reduce_min_sync(FULL, mininq);
        if (lane == 0 && mininq != AGR_RID_NONE) atomicMin(p.min_inq, mininq);
    }
}

template <bool SMEM>
__global__ void __launch_bounds__(256) k3_place(const agr_dev d, const agr_k3_params p) {
    extern __shared__ uint32_t s_rows[];
    __shared__ uint16_t s_list[8][1024];
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const bool live = w < p.nwarps;
    uint32_t* grow = p.matrix + (size_t)(live ? w : 0u) * p.groups;
    uint32_t* srow = s_rows + (size_t)(threadIdx.x >> 5) * p.groups;
    if (SMEM) {
        // cursors of this warp = the CTA's scanned row + the counts of the CTA's earlier warps (k3_mark left them in the matrix)
        for (uint32_t g = lane; g < p.groups; g += 32) srow[g] = live ? grow[g] : 0u;
        __syncthreads();
        uint32_t* cur = s_rows + (size_t)(8u + (threadIdx.x >> 5)) * p.groups;
        for (uint32_t g = lane; g < p.groups; g += 32) {
            uint32_t base = p.cta_matrix[(size_t)blockIdx.x * p.groups + g];
            for (uint32_t k = 0; k < (threadIdx.x >> 5); ++k) base += s_rows[(size_t)k * p.groups + g];
            cur[g] = base + p.goff[g];                               // absolute output position of the warp's next item of group g
        }
        __syncwarp();
        srow = cur;
    }
    if (!live) return;
    const unsigned long long b = p.lo + (unsigned long long)w * p.per_warp;
    unsigned long long e = b + p.per_warp;
    if (e > p.hi) e = p.hi;
    const bool rows = (p.mode != K3_LOG_AGENT);
    const uint32_t* mask = p.selmask + (size_t)w * (p.per_warp >> 5);
    const uint32_t pb = rows ? row_physical(d, b) : 0u;
    const uint32_t steps = (uint32_t)((e - b + 31u) >> 5);
    // A block = 32 selection words = 1024 items.  The set bits are first expanded into a dense list of item offsets (shared memory,
    // 2 KB per warp), so the rank / claim / store rounds below run on 32 SELECTED items each instead of on 32 items of which a
    // quarter are selected — and the route word of the next round is in flight while this one is placed.
    uint16_t* list = s_list[threadIdx.x >> 5];
    auto fetch = [&](const uint32_t blk_first, const uint32_t i, uint32_t& rid, uint32_t& rt) {
        const unsigned long long k = b + blk_first + list[i];
        if (rows) rid = k3_wrap(d, pb + (uint32_t)(k - b));
        else rid = p.log[k];
        rt = __ldg(&d.route[rid]);
    };
    for (uint32_t s0 = 0; s0 < steps; s0 += 32) {
        const uint32_t mine = (s0 + lane < steps) ? mask[s0 + lane] : 0u;          // 32 steps' selection words in one load
        if (!__any_sync(FULL, mine != 0u)) continue;
        const uint32_t c = (uint32_t)__popc(mine);
        uint32_t incl = c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, off); if (lane >= off) incl += v; }
        const uint32_t total = __shfl_sync(FULL, incl, 31);
        {
            uint32_t o = incl - c, m = mine;
            while (m) { const int bit = __ffs(m) - 1; m &= m - 1u; list[o++] = (uint16_t)(lane * 32 + bit); }
        }
        __syncwarp();
        uint32_t rid_n = AGR_RID_NONE, rt_n = 0u;
        if ((uint32_t)lane < total) fetch(s0 << 5, lane, rid_n, rt_n);
        for (uint32_t i0 = 0; i0 < total; i0 += 32) {
            const bool sel = i0 + lane < total;
            const uint32_t rid = rid_n, slot = rt_slot(rt_n);
            if (i0 + 32u + lane < total) fetch(s0 << 5, i0 + 32u + lane, rid_n, rt_n);
            const uint32_t g = (p.groups == 1) ? 0u : slot;
            const uint32_t key = sel ? g : (0x80000000u | (uint32_t)lane);
            const uint32_t peers = __match_any_sync(FULL, key);
            if (sel) {
                // the lowest lane of each group claims room for the whole group; stable rank inside the group = popc below
                const int leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd((SMEM ? srow : grow) + g, (uint32_t)__popc(peers));
                base = __shfl_sync(peers, base, leader);
                const uint32_t pos = (SMEM ? 0u : p.goff[g]) + base + __popc(peers & ((1u << lane) - 1u));
                if (pos < p.cap) p.out_rid[pos] = rid;              // (the agent slot is one load away for whoever needs it: route[rid])
            }
        }
        __syncwarp();                                                // the list is rewritten by the next block
    }
}

// Column scan of matrix[nwarps][groups] in ONE launch: a CTA owns 32 adjacent columns (coalesced 128 B rows); its 32 warps cut
// the rows into 32 segments: (1) every warp sums its segment per column, (2) an exclusive scan over the 32 segment sums in shared
// memory, (3) every warp rewrites its segment as exclusive prefixes.  gtotal[g] = the column total.
__global__ void __launch_bounds__(1024) k3_colscan(const agr_k3_params pp, uint32_t* __restrict__ matrix, const uint32_t nrows) {
    agr_k3_params p = pp; p.matrix = matrix; p.nwarps = nrows;          // the matrix to scan: per-CTA rows (or per-warp rows, flat mode)
    __shared__ uint32_t s_seg[32][33];
    const uint32_t g = blockIdx.x * 32u + (threadIdx.x & 31u), seg = threadIdx.x >> 5;
    const uint32_t per = (p.nwarps + 31u) / 32u, w0 = seg * per, w1 = min(p.nwarps, w0 + per);
    const bool ok = g < p.groups;
    uint32_t sum = 0;
    if (ok) {
#pragma unroll 8
        for (uint32_t w = w0; w < w1; ++w) sum += __ldcg(&p.matrix[(size_t)w * p.groups + g]);
    }
    s_seg[seg][threadIdx.x & 31u] = sum;
    __syncthreads();
    uint32_t run = 0, total = 0;
#pragma unroll
    for (int k = 0; k < 32; ++k) { const uint32_t v = s_seg[k][threadIdx.x & 31u]; if ((uint32_t)k < seg) run += v; total += v; }
    if (ok) {
        for (uint32_t wb = w0; wb < w1; wb += 8) {                   // eight independent loads, then the serial prefix
            uint32_t v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = (wb + k < w1) ? __ldcg(&p.matrix[(size_t)(wb + k) * p.groups + g]) : 0u;
#pragma unroll
            for (int k = 0; k < 8; ++k) if (wb + k < w1) { p.matrix[(size_t)(wb + k) * p.groups + g] = run; run += v[k]; }
        }
        if (seg == 0) p.gtotal[g] = total;
    }
}
// exclusive scan over groups (one CTA, loops for groups > 1024); goff[groups] = total
__global__ void __launch_bounds__(1024) k3_scan_total(const agr_k3_params p) {
    __shared__ uint32_t sh[1024];
    __shared__ uint32_t carry;
    const uint32_t t = threadIdx.x;
    if (t == 0) carry = 0;
    __syncthreads();
    for (uint32_t b = 0; b < p.groups; b += 1024) {
        uint32_t v = (b + t < p.groups) ? p.gtotal[b + t] : 0u;
        sh[t] = v;
        __syncthreads();
        for (uint32_t off = 1; off < 1024; off <<= 1) {
            uint32_t a = (t >= off) ? sh[t - off] : 0u;
            __syncthreads();
            sh[t] += a;
            __syncthreads();
        }
        if (b + t < p.groups) p.goff[b + t] = carry + sh[t] - v;
        __syncthreads();
        if (t == 1023) carry += sh[1023];
        __syncthreads();
    }
    if (t == 0) p.goff[p.groups] = carry;
}

void agr_launch_k3_select(const agr_dev& d, const agr_k3_params& p, int, cudaStream_t st) {
    const uint32_t blocks = (p.nwarps * 32u + 255u) / 256u;
    if (p.groups <= K3_SMEM_GROUPS) {
        const size_t smem = (size_t)8 * p.groups * sizeof(uint32_t);          // <= 16 KiB of counters (mark); twice that for place
        k3_mark<true><<<blocks, 256, smem, st>>>(d, p);
        k3_colscan<<<(p.groups + 31u) / 32u, 1024, 0, st>>>(p, p.cta_matrix, blocks);
        k3_scan_total<<<1, 1024, 0, st>>>(p);
        k3_place<true><<<blocks, 256, 2 * smem, st>>>(d, p);
    } else {
        cudaMemsetAsync(p.matrix, 0, (size_t)p.nwarps * p.groups * sizeof(uint32_t), st);
        k3_mark<false><<<blocks, 256, 0, st>>>(d, p);
        k3_colscan<<<(p.groups + 31u) / 32u, 1024, 0, st>>>(p, p.matrix, p.nwarps);
        k3_scan_total<<<1, 1024, 0, st>>>(p);
        k3_place<false><<<blocks, 256, 0, st>>>(d, p);
    }
}

// warp per selected row: copy the record out with the live state patched into the header, and/or emit the
// dispatch entry / the bare id
__global__ void __launch_bounds__(256) k3_gather(const agr_dev d, const uint32_t* rids, const uint32_t* slots, const uint32_t n,
                                                 uint8_t* out_recs, uint8_t* out_dispatch, uint8_t* out_ids) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n) return;
    const uint32_t rid = rids[w];
    const uint8_t* src = rec_ptr(d, rid);      // (variable-length rows: the first 512 B; use the *_var gathers for all of it)
    uint4 v = ldg_nc_v4(src + lane * 16);
    if (lane == 0 && (d.cfg_flags & AGR_CFG_MINT_IDS)) {          // Request.ID = what the engine minted for this row
        unsigned long long lo, hi;
        agr_mint_id(row_logical(d, rid), d.shard_id, d.id_gen, d.id_secret, lo, hi);
        v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
    }
    if (out_recs) {
        if (lane == 5) {   // bytes 80..95: body_len | status,retry,max,err | resp_status
            const uint32_t st = d.state[rid], aux = d.aux[rid];
            v.y = st_status(st) | (st_retry(st) << 8) | (st_max(st) << 16) | (((aux >> AUX_ERR_SHIFT) & 0xffu) << 24);
            v.z = (v.z & 0xffff0000u) | (aux & 0xffffu);
        }
        *reinterpret_cast<uint4*>(out_recs + (size_t)w * AGR_REC + lane * 16) = v;
    }
    uint4 id;
    id.x = __shfl_sync(FULL, v.x, 0); id.y = __shfl_sync(FULL, v.y, 0);
    id.z = __shfl_sync(FULL, v.z, 0); id.w = __shfl_sync(FULL, v.w, 0);
    if (out_dispatch && lane == 0) {
        const unsigned long long lrow = row_logical(d, rid);                  // agr_dispatch.rid: the row id the API speaks
        uint4 head = make_uint4((uint32_t)lrow, (uint32_t)(lrow >> 32), slots ? slots[w] : rt_slot(d.route[rid]), 0u);
        *reinterpret_cast<uint4*>(out_dispatch + (size_t)w * 32) = head;
        *reinterpret_cast<uint4*>(out_dispatch + (size_t)w * 32 + 16) = id;
    }
    if (out_ids && lane == 0) *reinterpret_cast<uint4*>(out_ids + (size_t)w * 16) = id;
}

void agr_launch_k3_gather(const agr_dev& d, const uint32_t* rids, const uint32_t* slots, uint32_t n, uint8_t* out_recs,
                          uint8_t* out_dispatch, uint8_t* out_ids, cudaStream_t st) {
    if (n == 0) return;
    k3_gather<<<(n * 32u + 255u) / 256u, 256, 0, st>>>(d, rids, slots, n, out_recs, out_dispatch, out_ids);
}

// agent.Manager.Remove queue cleanup (agent.go:349-359): DEL the three lists of one agent
__global__ void __launch_bounds__(256) k_drop_rows(const agr_dev d, const uint32_t slot, const unsigned long long rows) {
    const unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const uint32_t st = d.state[r];
    if ((st & ST_INQ) && rt_slot(d.route[r]) == slot) d.state[r] = st & ~ST_INQ;
}
__global__ void __launch_bounds__(256) k_drop_logs(const agr_dev d, const uint32_t slot) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < d.log_len[0]) { uint32_t rid = d.completed_log[k]; if (rid != AGR_RID_NONE && rt_slot(d.route[rid]) == slot) d.completed_log[k] = AGR_RID_NONE; }
    if (k < d.log_len[1]) { uint32_t rid = d.failed_log[k]; if (rid != AGR_RID_NONE && rt_slot(d.route[rid]) == slot) d.failed_log[k] = AGR_RID_NONE; }
}
void agr_launch_drop_agent(const agr_dev& d, uint32_t slot, unsigned long long rows, unsigned long long max_log_len,
                           cudaStream_t st) {
    if (rows) k_drop_rows<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(d, slot, rows);
    if (max_log_len) k_drop_logs<<<(unsigned)((max_log_len + 255) / 256), 256, 0, st>>>(d, slot);
}

// ------------------------------------------------------------------------------------------------ agent slot reuse
// Which candidate slots (removed agents) a decided row of physical rows [p0, p0 + n) still carries.  A lane reads four route words
// with one 16-byte load (from p0 rounded down to a multiple of 4; the rows outside the range are masked).  Only a decided row whose
// slot is a candidate issues an atomic, and the lanes of a warp that hit the same slot issue one between them (match_any), so a run
// of one agent's rows costs one atomicOr per warp step.  SMEM: the candidate bitmap is staged in shared memory (up to 2^18 slots),
// else it is read through L2.
template <bool SMEM>
__global__ void __launch_bounds__(256) k_slot_refs(const uint32_t* __restrict__ route, const unsigned long long p0, const unsigned long long n,
                                                   const uint32_t* __restrict__ cand, const uint32_t nslots, uint32_t* __restrict__ held) {
    extern __shared__ uint32_t s_cand[];
    if (SMEM) {
        for (uint32_t i = threadIdx.x; i < (nslots + 31u) >> 5; i += blockDim.x) s_cand[i] = cand[i];
        __syncthreads();
    }
    const uint32_t* cb = SMEM ? s_cand : cand;
    const int lane = threadIdx.x & 31;
    const unsigned long long e = p0 + n, stride = 4ull * gridDim.x * blockDim.x;
    for (unsigned long long q = (p0 & ~3ull) + 4ull * (blockIdx.x * blockDim.x + threadIdx.x);; q += stride) {
        const bool in = q < e;
        if (!__any_sync(FULL, in)) break;                                  // (the lanes of a warp cover 128 consecutive rows)
        const uint4 v = in ? __ldcs(reinterpret_cast<const uint4*>(route + q)) : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t s = rt_slot(w4[i]);
            const bool hit = q + i >= p0 && q + i < e && rt_code(w4[i]) != 0u && s < nslots && ((cb[s >> 5] >> (s & 31u)) & 1u);
            if (!__any_sync(FULL, hit)) continue;
            const uint32_t peers = __match_any_sync(FULL, hit ? s : 0xffffffffu);
            if (hit && lane == __ffs(peers) - 1) atomicOr(held + (s >> 5), 1u << (s & 31u));
        }
    }
}
#define SLOT_REFS_SMEM_WORDS 8192u   // 32 KiB: 2^18 slots
void agr_launch_slot_refs(const uint32_t* route, unsigned long long p0, unsigned long long n, const uint32_t* cand, uint32_t nslots,
                          uint32_t* held, int sm_count, cudaStream_t st) {
    if (!n || !nslots) return;
    const unsigned long long lanes = ((p0 & 3ull) + n + 3ull) / 4ull;
    const unsigned long long want = (lanes + 255ull) / 256ull, cap = (unsigned long long)sm_count * 8ull;
    const unsigned blocks = (unsigned)(want < cap ? want : cap);
    const uint32_t words = (nslots + 31u) >> 5;
    if (words <= SLOT_REFS_SMEM_WORDS) k_slot_refs<true><<<blocks, 256, words * 4u, st>>>(route, p0, n, cand, nslots, held);
    else k_slot_refs<false><<<blocks, 256, 0, st>>>(route, p0, n, cand, nslots, held);
}

// ------------------------------------------------------------------------------------------------ online snapshot cut
// blockIdx.y = section; the blocks of a section stride over it in 16 B pieces, four independent loads in flight per thread,
// and block 0 copies the tail (< 16 B).  The log lengths are read here, on the device, so the host never waits to learn them.
__global__ void __launch_bounds__(256) k_snap_cut(const agr_dev d, const agr_snap_cmp c) {
    const uint32_t s = blockIdx.y;
    unsigned long long bytes = c.bytes[s];
    if (s >= c.nrow) {
        const unsigned long long n = d.log_len[s - c.nrow];
        bytes = (n < d.log_cap ? n : d.log_cap) * 4ull;
        if (blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<unsigned long long*>(c.shadow)[s - c.nrow] = n;
    }
    const uint4* __restrict__ src = reinterpret_cast<const uint4*>(c.src[s]);
    uint4* __restrict__ dst = reinterpret_cast<uint4*>(c.shadow + c.dst_off[s]);
    const unsigned long long n16 = bytes >> 4, stride = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 a = src[i], b = src[i + stride], e = src[i + 2 * stride], f = src[i + 3 * stride];
        dst[i] = a; dst[i + stride] = b; dst[i + 2 * stride] = e; dst[i + 3 * stride] = f;
    }
    for (; i < n16; i += stride) dst[i] = src[i];
    if (blockIdx.x == 0 && threadIdx.x < (bytes & 15u)) {
        const unsigned long long t = (n16 << 4) + threadIdx.x;
        c.shadow[c.dst_off[s] + t] = c.src[s][t];
    }
}
void agr_launch_snap_cut(const agr_dev& d, const agr_snap_cmp& c, int sm_count, cudaStream_t st) {
    unsigned long long most = 0;                      // (the logs are at most log_cap entries)
    for (uint32_t s = 0; s < c.nrow; ++s) most = c.bytes[s] > most ? c.bytes[s] : most;
    if (d.log_cap * 4ull > most) most = d.log_cap * 4ull;
    const unsigned long long want = (most / 16 + 1023) / 1024;   // four pieces per thread
    const uint32_t bx = (uint32_t)(want < 1 ? 1 : want > (unsigned long long)sm_count * 2 ? (unsigned long long)sm_count * 2 : want);
    k_snap_cut<<<dim3(bx, c.nrow + 2), 256, 0, st>>>(d, c);
}

// ------------------------------------------------------------------------------------------------ delta snapshot cut
// The same grid as k_snap_cut.  Each warp takes 32 consecutive pieces, aligned to 32: 512 B, inside one block of any section
// (blocks are 1, 2 or 4 KiB), so a warp sets at most one bit, with one atomicOr, and only when a lane differs.  A piece at the
// end of a section (< 16 B) is read and written by words and zero-padded for the sum.
__device__ __forceinline__ uint4 snap_load_piece(const uint8_t* p, unsigned long long i, unsigned long long bytes) {
    if ((i + 1) * 16 <= bytes) return reinterpret_cast<const uint4*>(p)[i];
    uint32_t w[4] = {0, 0, 0, 0};
    for (unsigned k = 0; k < 4 && i * 16 + k * 4 < bytes; ++k) w[k] = reinterpret_cast<const uint32_t*>(p)[i * 4 + k];
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void snap_store_piece(uint8_t* p, unsigned long long i, unsigned long long bytes, uint4 v) {
    if ((i + 1) * 16 <= bytes) { reinterpret_cast<uint4*>(p)[i] = v; return; }
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    for (unsigned k = 0; k < 4 && i * 16 + k * 4 < bytes; ++k) reinterpret_cast<uint32_t*>(p)[i * 4 + k] = w[k];
}
template <bool COMPARE>
__global__ void __launch_bounds__(256) k_snap_cmp(const agr_dev d, const agr_snap_cmp c) {
    __shared__ unsigned long long part[2][8];
    const uint32_t s = blockIdx.y, lane = threadIdx.x & 31u;
    unsigned long long bytes = c.bytes[s];
    if (s >= c.nrow && !c.lens_from_host) {
        const unsigned long long n = d.log_len[s - c.nrow];
        bytes = (n < d.log_cap ? n : d.log_cap) * 4ull;
        if (COMPARE && blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<unsigned long long*>(c.shadow)[s - c.nrow] = n;
    }
    const uint8_t* __restrict__ src = c.src[s];
    uint8_t* __restrict__ dst = COMPARE ? c.shadow + c.dst_off[s] : nullptr;
    const unsigned long long np = (bytes + 15) >> 4, stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long skey = agr_fmix64(c.key ^ ((unsigned long long)(c.sec_id[s] + 1) << 56));
    unsigned long long h0 = 0, h1 = 0;
    for (unsigned long long i0 = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < np; i0 += stride) {
        const unsigned long long i = i0 + lane;
        bool differ = false;
        if (i < np) {
            const uint4 v = snap_load_piece(src, i, bytes);
            if (COMPARE) {
                const uint4 o = snap_load_piece(dst, i, bytes);
                differ = (v.x != o.x) | (v.y != o.y) | (v.z != o.z) | (v.w != o.w);
                if (differ) snap_store_piece(dst, i, bytes, v);
            }
            const unsigned long long a = ((unsigned long long)v.y << 32) | v.x, b = ((unsigned long long)v.w << 32) | v.z;
            const unsigned long long t = agr_fmix64(skey + i * 0x9e3779b97f4a7c15ULL);
            h0 += agr_fmix64(agr_fmix64(t ^ a) ^ b);
            h1 += agr_fmix64(agr_fmix64((t + 0x632be59bd9b4e019ULL) ^ b) ^ a);
        }
        if (COMPARE && __ballot_sync(0xffffffffu, differ) != 0u && lane == 0) {
            const unsigned long long blk = i0 >> c.pshift[s];
            atomicOr(c.bits + c.bit_off[s] + (blk >> 5), 1u << (blk & 31u));
        }
    }
    for (int o = 16; o > 0; o >>= 1) { h0 += __shfl_xor_sync(0xffffffffu, h0, o); h1 += __shfl_xor_sync(0xffffffffu, h1, o); }
    if (lane == 0) { part[0][threadIdx.x >> 5] = h0; part[1][threadIdx.x >> 5] = h1; }
    __syncthreads();
    if (threadIdx.x < 2) {
        unsigned long long sum = 0;
        for (int w = 0; w < 8; ++w) sum += part[threadIdx.x][w];
        atomicAdd(c.digest + threadIdx.x, sum);
    }
}
void agr_launch_snap_cmp(const agr_dev& d, const agr_snap_cmp& c, bool compare, int sm_count, cudaStream_t st) {
    unsigned long long most = 0;
    for (uint32_t s = 0; s < c.nrow + 2; ++s) most = c.bytes[s] > most ? c.bytes[s] : most;
    if (d.log_cap * 4ull > most) most = d.log_cap * 4ull;
    const unsigned long long want = (most / 16 + 1023) / 1024;
    const uint32_t bx = (uint32_t)(want < 1 ? 1 : want > (unsigned long long)sm_count * 2 ? (unsigned long long)sm_count * 2 : want);
    if (compare) k_snap_cmp<true><<<dim3(bx, c.nrow + 2), 256, 0, st>>>(d, c);
    else k_snap_cmp<false><<<dim3(bx, c.nrow + 2), 256, 0, st>>>(d, c);
}

// One CTA per listed block.  A full block's slices are whole multiples of 1 KiB: 16 B moves; the short last block by words.
template <bool GATHER>
__global__ void __launch_bounds__(256) k_snap_blocks(const agr_snap_blocks g) {
    const uint32_t b = g.list[blockIdx.x];
    const unsigned long long r0 = (unsigned long long)b * g.block_rows;
    const unsigned long long nr = g.rows - r0 < g.block_rows ? g.rows - r0 : g.block_rows;
    uint8_t* rec = g.stage + (unsigned long long)blockIdx.x * g.rec_bytes;
    unsigned long long at = 0;
    for (uint32_t s = 0; s < g.nsec; ++s) {
        const unsigned long long n = nr * g.width[s];
        uint8_t* a = g.arr[s] + r0 * g.width[s];
        uint8_t* st = rec + at;
        if (nr == g.block_rows) {
            for (unsigned long long k = threadIdx.x; k < n / 16; k += blockDim.x) {
                if (GATHER) reinterpret_cast<uint4*>(st)[k] = reinterpret_cast<const uint4*>(a)[k];
                else reinterpret_cast<uint4*>(a)[k] = reinterpret_cast<const uint4*>(st)[k];
            }
        } else {
            for (unsigned long long k = threadIdx.x; k < n / 4; k += blockDim.x) {
                if (GATHER) reinterpret_cast<uint32_t*>(st)[k] = reinterpret_cast<const uint32_t*>(a)[k];
                else reinterpret_cast<uint32_t*>(a)[k] = reinterpret_cast<const uint32_t*>(st)[k];
            }
        }
        at += n;
    }
}
void agr_launch_snap_blocks(const agr_snap_blocks& g, uint32_t n, bool gather, cudaStream_t st) {
    if (!n) return;
    if (gather) k_snap_blocks<true><<<n, 256, 0, st>>>(g);
    else k_snap_blocks<false><<<n, 256, 0, st>>>(g);
}

// ------------------------------------------------------------------------------------------------ synthetic stream
__global__ void __launch_bounds__(128) k_synth(uint8_t* dst, const agr_synth_dev s, const unsigned long long first_index, const uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    agr_synth_record(s, first_index + i, dst + (size_t)i * AGR_REC);
}
void agr_launch_synth(uint8_t* dst, agr_synth_dev s, unsigned long long first_index, uint32_t n, cudaStream_t st) {
    if (n == 0) return;
    k_synth<<<(n + 127u) / 128u, 128, 0, st>>>(dst, s, first_index, n);
}
