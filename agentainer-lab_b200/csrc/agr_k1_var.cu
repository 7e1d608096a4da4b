// agr_k1_var.cu — K1 for VARIABLE-LENGTH records (BASELINE config 5: 128 B - 4 KB bodies).
//
// A variable-length record = the same 96 B header as agr_record + its payload (path | headers | body) rounded up to
// 16 B; a batch is one contiguous blob plus an offsets array (n + 1 entries).  Work is balanced by BYTES, not by
// records: the blob is cut into 8 KiB tiles and a tile OWNS the records that START in it (k1v_tile_index), so a warp
// always moves about the same number of bytes whether they hold 60 small requests or two 4 KB ones, and no record is
// ever split between warps.  Per tile: one 1-D bulk TMA copy (UBLKCP) of the owned records into the warp's stage behind
// an mbarrier; a warp-cooperative, position-weighted checksum per record (lane = 16 B chunk, REDUX per record); then
// the decisions thread-per-record with the same staged functions as the fixed-stride kernel (agr_device.cuh).
// Algorithmic bytes per record: its stored length (96 + 16-rounded payload) + 8 (SURVEY 8d).
//
// A LONG record (stored length over VT_MAXREC, on an engine whose max_record_bytes allows it) is always the last record its
// tile owns, since nothing else can start before it ends.  K1v stages and decides only its 96-byte header; its checksum comes
// from k1v_long_sums below, 8 KiB per warp, so that one warp never streams a megabyte alone while the tiles inside the record
// own nothing.  Records up to VT_MAXREC take the same path as before.
#include "agr_device.cuh"

#define VT_TILE 8192u                 // bytes of blob per tile
#define VT_WARPS 16
#define VT_MAXREC 8192u               // longest record K1v sums itself (header + payload); longer ones are long records
#define VT_TAIL 4608u                 // stage room behind the tile for the last owned record (a 4 KB body fits); a record that
                                      // ends beyond the stage (> 4.5 KiB and badly placed: rare) is read from global memory
#define VT_STAGE (VT_TILE + VT_TAIL)  // 12800 B = 100 x 128
#define VT_MAXCNT (VT_TILE / 96u + 2u)   // at most this many records can start in one tile (87: three offsets per lane)

__device__ __forceinline__ uint32_t v_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint4 v_lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}

// TTL bookkeeping (k_expire): a stored record lowers its chunk's time bound to its created_at.  Arrival times hardly ever run
// backwards, so after a chunk's first records the bound is already low enough and the atomic is skipped.
__device__ __forceinline__ void k1v_note_time(const agr_dev& d, const uint32_t rid, const uint32_t state, const uint4& h4) {
    return;   // variable-length engines: agr_expire resets the bounds of the chunks filled since its last call instead (the
              // per-record read of the bound cost this issue-bound kernel 8 %); kept for reference
    if (!(state & ST_STORED) || !(d.cfg_flags & AGR_CFG_RING)) return;
    unsigned long long t = pack64(h4.x, h4.y);
    if (t == 0ULL) t = 1ULL;
    unsigned long long* cm = d.cmin + rid / AGR_CHUNK_ROWS;
    if (t < __ldcg(cm)) atomicMin(cm, t);
}

// tile_first[t] = index of the first record whose start offset is >= t * VT_TILE, for t = 0 .. ntiles (tile_first[ntiles]
// = n).  Record i is that record for every boundary t * VT_TILE in (start(i-1), start(i)]; the sentinel i == n takes the
// boundaries after the last start.  Tile t then owns records [tile_first[t], tile_first[t+1]).
__global__ void __launch_bounds__(256) k1v_tile_index(const uint32_t* __restrict__ off, const uint32_t n, uint32_t* __restrict__ tile_first,
                                                      const uint32_t ntiles) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    const uint32_t lo = (i == 0) ? 0u : off[i - 1] / VT_TILE + 1u;
    const uint32_t hi = (i == n) ? ntiles : off[i] / VT_TILE;
    for (uint32_t t = lo; t <= hi; ++t) tile_first[t] = i;
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
k1_ingest_var(const agr_dev d, const uint8_t* __restrict__ blob, const uint32_t* __restrict__ off, const uint32_t* __restrict__ tile_first,
              const uint32_t ntiles, const uint32_t first_rid, const unsigned long long blob_base /* byte offset of blob in the slab */) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t bars[WARPS];
    __shared__ uint32_t s_off[WARPS][2][VT_MAXCNT + 1];       // record offsets of the current / the next tile
    __shared__ unsigned long long s_ck[WARPS][VT_MAXCNT];
    __shared__ uint32_t s_ctr[K1_NLC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t smem_base = (v_smem_u32(smem_raw) + 127u) & ~127u;
    if (threadIdx.x < K1_NLC) s_ctr[threadIdx.x] = 0;
    if (threadIdx.x < WARPS) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(v_smem_u32(&bars[threadIdx.x])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t lc[K1_NLC + 1];
#pragma unroll
    for (int c = 0; c <= K1_NLC; ++c) lc[c] = 0;
    const uint32_t stage = smem_base + (uint32_t)warp * VT_STAGE;
    const uint32_t bar = v_smem_u32(&bars[warp]);
    const uint32_t tstride = gridDim.x * WARPS;

    // Tile metadata is software-pipelined two tiles deep so that no global-load latency sits on the warp's critical path:
    // while tile T is processed, the record offsets of T+1 are in flight into registers (their range [a1, b1) was read one
    // iteration earlier) and the range of T+2 is being read.  A tile inside one long record owns nothing (cnt == 0).
    // bytes staged for a tile: its records, of a long last record only the header
    auto stage_bytes = [](const uint32_t* so, uint32_t cnt) {
        const uint32_t end = (so[cnt] - so[cnt - 1] > VT_MAXREC) ? so[cnt - 1] + AGR_OFF_PAYLOAD : so[cnt];
        return min(end - so[0], VT_STAGE);
    };
    auto issue = [&](int buf, uint32_t cnt) {
        if (lane == 0) {
            const uint32_t start = s_off[warp][buf][0];
            const uint32_t bytes = stage_bytes(s_off[warp][buf], cnt);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(stage), "l"(blob + start), "r"(bytes), "r"(bar) : "memory");
        }
    };
    auto range_of = [&](uint32_t t, uint32_t& ra, uint32_t& rb) {
        ra = rb = 0;
        if (t < ntiles) { ra = __ldg(&tile_first[t]); rb = __ldg(&tile_first[t + 1]); }
    };

    int cur = 0;
    uint32_t phase = 0;
    uint32_t tile = blockIdx.x * WARPS + warp;
    uint32_t a, b1v, a1, b1;
    range_of(tile, a, b1v);
    uint32_t cnt = b1v - a;
    if (cnt) {
        for (uint32_t k = lane; k <= cnt; k += 32) s_off[warp][cur][k] = __ldg(&off[a + k]);
        __syncwarp();
        issue(cur, cnt);
    }
    range_of(tile + tstride, a1, b1);
    while (tile < ntiles) {
        // offsets of the next tile -> registers (at most 3 per lane), range of the one after it -> registers
        const uint32_t ncnt = b1 - a1;
        uint32_t o0 = 0, o1 = 0, o2 = 0, a2, b2;
        if (ncnt) {
            if ((uint32_t)lane <= ncnt) o0 = __ldg(&off[a1 + lane]);
            if ((uint32_t)lane + 32u <= ncnt) o1 = __ldg(&off[a1 + lane + 32u]);
            if ((uint32_t)lane + 64u <= ncnt) o2 = __ldg(&off[a1 + lane + 64u]);
        }
        range_of(tile + 2u * tstride, a2, b2);
        auto stage_next = [&]() {                                 // called once this tile's stage has been consumed
            if (ncnt) {
                uint32_t* nso = s_off[warp][cur ^ 1];
                if ((uint32_t)lane <= ncnt) nso[lane] = o0;
                if ((uint32_t)lane + 32u <= ncnt) nso[lane + 32u] = o1;
                if ((uint32_t)lane + 64u <= ncnt) nso[lane + 64u] = o2;
                __syncwarp();
                issue(cur ^ 1, ncnt);
            }
        };
        if (cnt == 0) {                                           // nothing starts in this tile
            stage_next();
            tile += tstride; a = a1; cnt = ncnt; a1 = a2; b1 = b2; cur ^= 1;
            continue;
        }
        const uint32_t* so = s_off[warp][cur];
        const uint32_t start = so[0], bytes = stage_bytes(so, cnt);
        asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}"
                     ::"r"(bar), "r"(phase) : "memory");
        phase ^= 1u;
        // ---- checksum: one record at a time, lanes sweep its 16 B chunks (conflict-free), REDUX per record
        for (uint32_t r = 0; r < cnt; ++r) {
            if (so[r + 1] - so[r] > VT_MAXREC) break;                           // a long last record: k1v_long_sums
            const uint32_t lo = so[r] - start, chunks = (so[r + 1] - so[r]) >> 4;
            const bool in_stage = (so[r + 1] - start) <= bytes;                    // warp-uniform
            const uint8_t* g = blob + so[r];
            uint32_t c0 = 0, c1 = 0;
            for (uint32_t c = lane; c < chunks; c += 32) {
                const uint4 v = in_stage ? v_lds128(stage + lo + (c << 4)) : ldg_nc_v4(g + ((size_t)c << 4));
                c0 += v.x + v.y + v.z + v.w;
                c1 += (4 * c + 1) * v.x + (4 * c + 2) * v.y + (4 * c + 3) * v.z + (4 * c + 4) * v.w;
            }
            c0 = __reduce_add_sync(FULL, c0);
            c1 = __reduce_add_sync(FULL, c1);
            if (lane == 0) s_ck[warp][r] = agr_cksum_pack(c0, c1);
        }
        __syncwarp();
        // ---- decisions, one record per lane.  Round 0 (records 0..31 of the tile) reads its headers, THEN the stage is
        // handed back to the TMA unit for the next tile, and only then does the long-latency decision chain run.
        auto load_header = [&](uint32_t r, uint4& h0, uint4& h1, uint4& h2, uint4& h3, uint4& h4, uint4& h5) {
            const uint32_t hb = stage + (so[r] - start);
            if ((so[r] - start) + 96u <= bytes) {
                h0 = v_lds128(hb); h1 = v_lds128(hb + 16); h2 = v_lds128(hb + 32); h3 = v_lds128(hb + 48); h4 = v_lds128(hb + 64); h5 = v_lds128(hb + 80);
            } else {
                const uint8_t* g = blob + so[r];
                h0 = ldg_nc_v4(g); h1 = ldg_nc_v4(g + 16); h2 = ldg_nc_v4(g + 32); h3 = ldg_nc_v4(g + 48); h4 = ldg_nc_v4(g + 64); h5 = ldg_nc_v4(g + 80);
            }
        };
        auto decide = [&](uint32_t r, const uint4& h0, const uint4& h1, const uint4& h2, const uint4& h3, const uint4& h4, const uint4& h5) {
            const uint32_t rid = first_rid + a + r;
            k1_ctx cx;
            k1_begin(d, k1_agent_issue(d, h2, h3), h0, h1, h2, h3, h4, h5.x, (so[r + 1] - so[r]) - AGR_OFF_PAYLOAD, false, 0ULL, 0ULL, a + r, cx);
            const k1_result res = k1_finish(d, rid, h1, h5, cx, lc);
            k1v_note_time(d, rid, res.state, h4);
            d.state[rid] = res.state;
            d.route[rid] = res.route;
            if (so[r + 1] - so[r] <= VT_MAXREC) d.cksum[rid] = s_ck[warp][r];
            d.voff[rid] = blob_base + so[r];
            d.vlen[rid] = so[r + 1] - so[r];
        };
        for (uint32_t r = 32 + lane; r < cnt; r += 32) {          // rounds 1.. (tiles of many small records) first
            uint4 h0, h1, h2, h3, h4, h5;
            load_header(r, h0, h1, h2, h3, h4, h5);
            decide(r, h0, h1, h2, h3, h4, h5);
        }
        uint4 h0 = make_uint4(0, 0, 0, 0), h1 = h0, h2 = h0, h3 = h0, h4 = h0, h5 = h0;
        const bool mine = (uint32_t)lane < cnt;
        if (mine) load_header(lane, h0, h1, h2, h3, h4, h5);
        __syncwarp();                                             // the stage has been consumed
        stage_next();
        if (mine) decide(lane, h0, h1, h2, h3, h4, h5);
        __syncwarp();
        tile += tstride; a = a1; cnt = ncnt; a1 = a2; b1 = b2; cur ^= 1;
    }
    k1_flush_counters(d, lc, s_ctr);
}

// ---- LSU form of the same kernel (k1_variant bit 0x20): no shared-memory stage and no TMA — the warp streams its tile
// straight from global memory with coalesced 16 B loads.  Without a 12.5 KiB stage per warp an SM holds 48 warps instead
// of 16, which is what the byte-tiled kernel above is short of (every warp there issues once per 8 cycles).  The
// checksums come from ONE linear sweep over the tile: the record checksum weights word k of the record by k + 1; with g =
// the word's index in the sweep that is (g + 1) - 4 lo (lo = the record's first chunk), so every lane accumulates
// s0 = sum w and s1 = sum (g + 1) w of the chunks it meets and a record's pair is (S0, S1 - 4 lo S0) over the chunks between
// two record starts.  A bitmap of record-start chunks tells each 32-chunk row where records begin: rows without a start
// cost a load and a dozen integer ops; a row with a start closes the running record with two REDUX; records that lie
// entirely inside one row are summed by a segmented shuffle reduction.  The sweep stops at the start of a long last record
// (k1v_long_sums sums it), so it never spans more than the tile and one record of at most VT_MAXREC.
#define VL_WARPS 8
#define VL_MAXCH ((VT_TILE + VT_MAXREC) / 16u)         // chunks a tile's sweep can span (1024)
#define VL_HWORDS (VL_MAXCH / 32u)
__global__ void __launch_bounds__(VL_WARPS * 32, 5)
k1_ingest_var_lsu(const agr_dev d, const uint8_t* __restrict__ blob, const uint32_t* __restrict__ off, const uint32_t* __restrict__ tile_first,
                  const uint32_t ntiles, const uint32_t first_rid, const unsigned long long blob_base) {
    __shared__ uint32_t s_off[VL_WARPS][VT_MAXCNT + 1];
    __shared__ unsigned long long s_ck[VL_WARPS][VT_MAXCNT];
    __shared__ uint32_t s_heads[VL_WARPS][VL_HWORDS];
    __shared__ uint32_t s_ctr[K1_NLC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < K1_NLC) s_ctr[threadIdx.x] = 0;
    __syncthreads();
    uint32_t lc[K1_NLC + 1];
#pragma unroll
    for (int c = 0; c <= K1_NLC; ++c) lc[c] = 0;
    const uint32_t tstride = gridDim.x * VL_WARPS;
    const uint32_t below = (1u << lane) - 1u;
    uint32_t* so = s_off[warp];
    uint32_t* hb = s_heads[warp];
    auto range_of = [&](uint32_t t, uint32_t& ra, uint32_t& rb) {
        ra = rb = 0;
        if (t < ntiles) { ra = __ldg(&tile_first[t]); rb = __ldg(&tile_first[t + 1]); }
    };
    uint32_t tile = blockIdx.x * VL_WARPS + warp;
    uint32_t a, b, a1, b1;
    range_of(tile, a, b);
    range_of(tile + tstride, a1, b1);
    for (; tile < ntiles; tile += tstride) {
        const uint32_t cnt = b - a;
        uint32_t a2, b2;
        range_of(tile + 2u * tstride, a2, b2);                    // two tiles ahead: in flight during this tile's sweep
        if (cnt) {
            for (uint32_t k = lane; k <= cnt; k += 32) so[k] = __ldg(&off[a + k]);
            if (lane < (int)VL_HWORDS) hb[lane] = 0;
            __syncwarp();
            const uint32_t swept = cnt - (so[cnt] - so[cnt - 1] > VT_MAXREC ? 1u : 0u);   // records the sweep sums
            const uint32_t start = so[0], nch = (so[swept] - start) >> 4;
            for (uint32_t r = lane; r < swept; r += 32) { const uint32_t c = (so[r] - start) >> 4; atomicOr(&hb[c >> 5], 1u << (c & 31u)); }
            __syncwarp();
            const uint8_t* base = blob + start;
            uint32_t a0 = 0, a1s = 0, base_r = 0, cur_r = 0xffffffffu, cur_lo = 0;
            const uint32_t nrows = (nch + 31u) >> 5;
            auto load_row = [&](uint32_t row) -> uint4 {
                const uint32_t g = (row << 5) + lane;
                return g < nch ? ldg_nc_v4(base + ((size_t)g << 4)) : make_uint4(0, 0, 0, 0);
            };
            auto do_row = [&](const uint4 v, const uint32_t row) {
                const uint32_t g = (row << 5) + lane;
                const uint32_t s0 = v.x + v.y + v.z + v.w;
                const uint32_t s1 = 4u * g * s0 + (v.x + 2u * v.y + 3u * v.z + 4u * v.w);
                const uint32_t word = hb[row];
                if (word == 0) { a0 += s0; a1s += s1; return; }
                const uint32_t first = __ffs(word) - 1u, last = 31u - __clz(word);
                if ((uint32_t)lane < first) { a0 += s0; a1s += s1; }
                if (cur_r != 0xffffffffu) {                                    // the running record ends at the first start
                    const uint32_t S0 = __reduce_add_sync(FULL, a0), S1 = __reduce_add_sync(FULL, a1s);
                    if (lane == 0) s_ck[warp][cur_r] = agr_cksum_pack(S0, S1 - 4u * cur_lo * S0);
                }
                if (word & (word - 1u)) {                                      // records that start AND end inside this row
                    const bool in = (uint32_t)lane >= first && (uint32_t)lane < last;
                    uint32_t x0 = in ? s0 : 0u, x1 = in ? s1 : 0u;
                    const uint32_t ahead = lane < 31 ? word >> (lane + 1) : 0u;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t y0 = __shfl_down_sync(FULL, x0, o), y1 = __shfl_down_sync(FULL, x1, o);
                        if (lane + o < 32 && (ahead & ((1u << o) - 1u)) == 0u) { x0 += y0; x1 += y1; }
                    }
                    if (((word >> lane) & 1u) && (uint32_t)lane != last)
                        s_ck[warp][base_r + __popc(word & below)] = agr_cksum_pack(x0, x1 - 4u * g * x0);
                }
                const bool tail = (uint32_t)lane >= last;
                a0 = tail ? s0 : 0u; a1s = tail ? s1 : 0u;
                base_r += __popc(word);
                cur_r = base_r - 1u; cur_lo = (row << 5) + last;
            };
            // four rows (2 KiB per warp) stay in flight: a slot is refilled as soon as it has been consumed
            uint4 q0 = load_row(0), q1 = load_row(1), q2 = load_row(2), q3 = load_row(3);
            for (uint32_t row = 0; row < nrows; row += 4) {
                do_row(q0, row);     q0 = load_row(row + 4);
                if (row + 1 < nrows) { do_row(q1, row + 1); q1 = load_row(row + 5); }
                if (row + 2 < nrows) { do_row(q2, row + 2); q2 = load_row(row + 6); }
                if (row + 3 < nrows) { do_row(q3, row + 3); q3 = load_row(row + 7); }
            }
            if (cur_r != 0xffffffffu) {
                const uint32_t S0 = __reduce_add_sync(FULL, a0), S1 = __reduce_add_sync(FULL, a1s);
                if (lane == 0) s_ck[warp][cur_r] = agr_cksum_pack(S0, S1 - 4u * cur_lo * S0);
            }
            __syncwarp();
            // ---- decisions, one record per lane; the headers were streamed a moment ago and come back from L2
            for (uint32_t r = lane; r < cnt; r += 32) {
                const uint8_t* gp = blob + so[r];
                const uint4 h0 = ldg_nc_v4(gp), h1 = ldg_nc_v4(gp + 16), h2 = ldg_nc_v4(gp + 32), h3 = ldg_nc_v4(gp + 48),
                            h4 = ldg_nc_v4(gp + 64), h5 = ldg_nc_v4(gp + 80);
                const uint32_t rid = first_rid + a + r;
                k1_ctx cx;
                k1_begin(d, k1_agent_issue(d, h2, h3), h0, h1, h2, h3, h4, h5.x, (so[r + 1] - so[r]) - AGR_OFF_PAYLOAD, false, 0ULL, 0ULL, a + r, cx);
                const k1_result res = k1_finish(d, rid, h1, h5, cx, lc);
                k1v_note_time(d, rid, res.state, h4);
                d.state[rid] = res.state;
                d.route[rid] = res.route;
                if (r < swept) d.cksum[rid] = s_ck[warp][r];
                d.voff[rid] = blob_base + so[r];
                d.vlen[rid] = so[r + 1] - so[r];
            }
            __syncwarp();
        }
        a = a1; b = b1; a1 = a2; b1 = b2;
    }
    k1_flush_counters(d, lc, s_ctr);
}

// ---- checksums of long records.  Piece p of a record covers its chunks [512 p, 512 p + 512): lanes on 16 B chunks, all
// sixteen loads of a lane issued before any is summed.  Word k of the record (k = 4 c + j in chunk c) weighs k + 1 as in K1v,
// so the pieces' (s0, s1) add up to the record's exactly (mod 2^32 in any order): two atomics per piece, then one pack.
#define VL_PIECE_CH (VT_TILE / 16u)                    // chunks per piece (512: 16 per lane)
#define VL_LONG_WARPS 8
__global__ void __launch_bounds__(VL_LONG_WARPS * 32) k1v_long_sums(const uint8_t* __restrict__ blob, const uint32_t* __restrict__ off,
                                                                    const uint32_t* __restrict__ list, const uint32_t nl,
                                                                    const uint32_t npieces, uint32_t* __restrict__ acc) {
    const uint32_t w = blockIdx.x * VL_LONG_WARPS + (threadIdx.x >> 5);
    const uint32_t lane = threadIdx.x & 31u;
    if (w >= npieces) return;
    const uint32_t* first = list + nl;                  // first[k] = first piece of long record k, first[nl] = npieces
    uint32_t lo = 0, hi = nl;                           // the k with first[k] <= w < first[k + 1]
    while (hi - lo > 1u) { const uint32_t m = (lo + hi) >> 1; if (__ldg(&first[m]) <= w) lo = m; else hi = m; }
    const uint32_t i = __ldg(&list[lo]);
    const uint32_t o = __ldg(&off[i]), chunks = (__ldg(&off[i + 1]) - o) >> 4;
    const uint32_t c0 = (w - __ldg(&first[lo])) * VL_PIECE_CH;
    const uint8_t* g = blob + o;
    uint4 v[VL_PIECE_CH / 32u];
#pragma unroll
    for (uint32_t j = 0; j < VL_PIECE_CH / 32u; ++j) {
        const uint32_t c = c0 + lane + 32u * j;
        v[j] = c < chunks ? ldg_nc_v4(g + ((size_t)c << 4)) : make_uint4(0, 0, 0, 0);
    }
    uint32_t s0 = 0, s1 = 0;
#pragma unroll
    for (uint32_t j = 0; j < VL_PIECE_CH / 32u; ++j) {
        const uint32_t c = c0 + lane + 32u * j;
        s0 += v[j].x + v[j].y + v[j].z + v[j].w;
        s1 += (4u * c + 1u) * v[j].x + (4u * c + 2u) * v[j].y + (4u * c + 3u) * v[j].z + (4u * c + 4u) * v[j].w;
    }
    s0 = __reduce_add_sync(FULL, s0);
    s1 = __reduce_add_sync(FULL, s1);
    if (lane == 0) { atomicAdd(&acc[2u * lo], s0); atomicAdd(&acc[2u * lo + 1u], s1); }
}
__global__ void __launch_bounds__(256) k1v_long_pack(const agr_dev d, const uint32_t* __restrict__ list, const uint32_t nl,
                                                     const uint32_t* __restrict__ acc, const uint32_t first_rid) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < nl) d.cksum[first_rid + list[k]] = agr_cksum_pack(acc[2u * k], acc[2u * k + 1u]);
}
cudaError_t agr_launch_k1v_long(const agr_dev& d, const uint8_t* blob, const uint32_t* off, const uint32_t* list, uint32_t nl,
                                uint32_t npieces, uint32_t* acc, uint32_t first_rid, cudaStream_t st) {
    if (nl == 0) return cudaSuccess;
    const cudaError_t e = cudaMemsetAsync(acc, 0, (size_t)nl * 2u * sizeof(uint32_t), st);
    if (e != cudaSuccess) return e;
    k1v_long_sums<<<(npieces + VL_LONG_WARPS - 1u) / VL_LONG_WARPS, VL_LONG_WARPS * 32, 0, st>>>(blob, off, list, nl, npieces, acc);
    k1v_long_pack<<<(nl + 255u) / 256u, 256, 0, st>>>(d, list, nl, acc, first_rid);
    return cudaGetLastError();
}

// gather of variable-length rows: lens pass, then copy pass (offsets are scanned on the host: a per-tick operation)
__global__ void __launch_bounds__(256) k_var_lens(const agr_dev d, const uint32_t* __restrict__ rids, const uint32_t n, uint32_t* __restrict__ lens) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) lens[j] = d.vlen[rids[j]];
}
__global__ void __launch_bounds__(256) k_var_copy(const agr_dev d, const uint32_t* __restrict__ rids, const uint32_t n,
                                                  const unsigned long long* __restrict__ out_off, uint8_t* __restrict__ out) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n) return;
    const uint32_t rid = rids[w];
    const uint8_t* src = d.slab + d.voff[rid];
    uint8_t* dst = out + out_off[w];
    const uint32_t chunks = d.vlen[rid] >> 4;
    for (uint32_t c = lane; c < chunks; c += 32) {
        uint4 v = ldg_nc_v4(src + (size_t)c * 16);
        if (c == 0 && (d.cfg_flags & AGR_CFG_MINT_IDS)) {
            unsigned long long lo, hi;
            agr_mint_id(row_logical(d, rid), d.shard_id, d.id_gen, d.id_secret, lo, hi);
            v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
        }
        if (c == 5) {   // bytes 80..95: body_len | status,retry,max,err | resp_status  (live state patched in)
            const uint32_t st = d.state[rid], aux = d.aux[rid];
            v.y = st_status(st) | (st_retry(st) << 8) | (st_max(st) << 16) | (((aux >> AUX_ERR_SHIFT) & 0xffu) << 24);
            v.z = (v.z & 0xffff0000u) | (aux & 0xffffu);
        }
        *reinterpret_cast<uint4*>(dst + (size_t)c * 16) = v;
    }
}

cudaError_t agr_launch_k1_var(const agr_dev& d, const uint8_t* blob, const uint32_t* off, uint32_t n, unsigned long long blob_bytes,
                              uint32_t* tile_first, uint32_t first_rid, unsigned long long blob_base, int sm_count, cudaStream_t st,
                              uint32_t variant) {
    if (variant & 0x20u) {                                       // LSU form
        const uint32_t ntiles = (uint32_t)((blob_bytes + VT_TILE - 1) / VT_TILE);
        k1v_tile_index<<<(n + 1 + 255u) / 256u, 256, 0, st>>>(off, n, tile_first, ntiles);
        uint32_t blocks = (uint32_t)sm_count * 5u;
        const uint32_t need = (ntiles + VL_WARPS - 1) / VL_WARPS;
        if (blocks > need) blocks = need;
        if (blocks == 0) blocks = 1;
        k1_ingest_var_lsu<<<blocks, VL_WARPS * 32, 0, st>>>(d, blob, off, tile_first, ntiles, first_rid, blob_base);
        return cudaGetLastError();
    }
    constexpr int WARPS = VT_WARPS;
    const size_t smem = (size_t)WARPS * VT_STAGE + 128;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(k1_ingest_var<WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr_done = true;
    }
    const uint32_t ntiles = (uint32_t)((blob_bytes + VT_TILE - 1) / VT_TILE);
    k1v_tile_index<<<(n + 1 + 255u) / 256u, 256, 0, st>>>(off, n, tile_first, ntiles);
    uint32_t blocks = (uint32_t)sm_count;
    const uint32_t need = (ntiles + WARPS - 1) / WARPS;
    if (blocks > need) blocks = need;
    if (blocks == 0) blocks = 1;
    k1_ingest_var<WARPS><<<blocks, WARPS * 32, smem, st>>>(d, blob, off, tile_first, ntiles, first_rid, blob_base);
    return cudaGetLastError();
}
// A run of rows reserved with agr_reserve_rows (or by the exchange) on a variable-length engine holds 512-byte records back to
// back: K1v reads it as a blob whose offsets are 512 i.
__global__ void __launch_bounds__(256) k1v_slot_offsets(uint32_t* __restrict__ off, const uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n) off[i] = i * (uint32_t)AGR_REC;
}
void agr_launch_slot_offsets(uint32_t* off, uint32_t n, cudaStream_t st) {
    k1v_slot_offsets<<<(n + 1 + 255u) / 256u, 256, 0, st>>>(off, n);
}
void agr_launch_var_lens(const agr_dev& d, const uint32_t* rids, uint32_t n, uint32_t* lens, cudaStream_t st) {
    if (n) k_var_lens<<<(n + 255u) / 256u, 256, 0, st>>>(d, rids, n, lens);
}
void agr_launch_var_copy(const agr_dev& d, const uint32_t* rids, uint32_t n, const unsigned long long* out_off, uint8_t* out, cudaStream_t st) {
    if (n) k_var_copy<<<(n * 32u + 255u) / 256u, 256, 0, st>>>(d, rids, n, out_off, out);
}
