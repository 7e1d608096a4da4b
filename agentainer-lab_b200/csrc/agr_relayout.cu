// agr_relayout.cu — the relocation of a restore into other capacities (agr_restore, DESIGN.md section 5): the live window
// of a source engine moves to row id mod the target's slab_rows, and the record / response bytes of its live rows are
// packed from byte 0 of the target's byte rings.  The target may hold records in the other form: 512 B rows become their
// compact variable-length records, and variable-length records become 512 B rows padded with zeros.  Everything here is
// bulk movement over HBM.
#include "agr_device.cuh"

#define RL_T 256u                       // threads per CTA of the row kernels
#define RL_PER 8u                       // rows per thread
#define RL_TILE (RL_T * RL_PER)         // rows per CTA (one entry of tile_sum)
#define RL_WORDS 4u                     // 16 B destination words per thread of the byte move
#define RL_CHUNK (RL_T * RL_WORDS * 16u)   // destination bytes per CTA of the byte move

__device__ __forceinline__ unsigned long long rl_r16(unsigned long long x) { return (x + 15ull) & ~15ull; }

// block-wide exclusive scan of two u64 per thread; returns the block's totals in ta, tb
__device__ __forceinline__ void rl_block_scan(unsigned long long& a, unsigned long long& b, unsigned long long& ta, unsigned long long& tb) {
    __shared__ unsigned long long s_w[2][RL_T / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned long long ia = a, ib = b;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const unsigned long long ya = __shfl_up_sync(FULL, ia, o), yb = __shfl_up_sync(FULL, ib, o);
        if (lane >= o) { ia += ya; ib += yb; }
    }
    if (lane == 31) { s_w[0][warp] = ia; s_w[1][warp] = ib; }
    __syncthreads();
    unsigned long long pa = 0, pb = 0;
    ta = 0; tb = 0;
#pragma unroll
    for (uint32_t w = 0; w < RL_T / 32; ++w) {
        if (w < warp) { pa += s_w[0][w]; pb += s_w[1][w]; }
        ta += s_w[0][w]; tb += s_w[1][w];
    }
    a = pa + ia - a; b = pb + ib - b;
    __syncthreads();                    // (s_w is reused by the next call)
}

// The compact length of a fixed-stride row's record, 96 + round16(path_len + hdr_len + body_len), from the lengths in its
// header (one sector); capped at the row's 512 B, which K1 never stores a longer record in.
__device__ __forceinline__ uint32_t rl_compact_len(const uint8_t* row) {
    const uint32_t ph = __ldg(reinterpret_cast<const uint32_t*>(row + offsetof(agr_record, path_len)));   // path_len | hdr_len << 16
    const uint32_t body = __ldg(reinterpret_cast<const uint32_t*>(row + offsetof(agr_record, body_len)));
    const unsigned long long n = AGR_HEADER_BYTES + rl_r16((unsigned long long)(ph & 0xffffu) + (ph >> 16) + body);
    return (uint32_t)(n < AGR_REC ? n : AGR_REC);
}

// What row k of the window takes: its record's length (the source's vlen, or with a fixed-stride source and a variable-length
// target the compact length of its row; 0 for fixed-stride to fixed-stride), and its 16 B-rounded response + error bytes
struct rl_row {
    uint32_t ps, st, vlen, rlen, elen;
};
__device__ __forceinline__ rl_row rl_read(const agr_relayout& p, unsigned long long k) {
    rl_row r;
    r.ps = row_physical(p.s, p.s.tail + k);
    r.st = p.s.state[r.ps];
    const bool live = r.st != 0u;
    r.vlen = !live ? 0u : p.s.voff ? p.s.vlen[r.ps] : p.t.voff ? rl_compact_len(p.s.slab + (size_t)r.ps * AGR_REC) : 0u;
    r.rlen = live ? p.sw.resp_len[r.ps] : 0u;
    r.elen = live ? p.sw.err_len[r.ps] : 0u;
    return r;
}

// per tile of RL_TILE rows: record bytes and response bytes of its live rows.  Into a fixed-stride target from a
// variable-length source, also the records longer than a 512 B row: their count at totals[2], and the least (k << 32 | vlen)
// at totals[3] (the caller sets them to 0 and ~0 first).
__global__ void __launch_bounds__(RL_T) k_rl_count(const agr_relayout p) {
    unsigned long long a = 0, b = 0, ta, tb;
    const unsigned long long k0 = (unsigned long long)blockIdx.x * RL_TILE;
    const bool to_rows = p.s.voff && !p.t.voff;
#pragma unroll
    for (uint32_t j = 0; j < RL_PER; ++j) {
        const unsigned long long k = k0 + j * RL_T + threadIdx.x;
        if (k >= p.n) break;
        const rl_row r = rl_read(p, k);
        a += r.vlen; b += rl_r16(r.rlen) + rl_r16(r.elen);
        if (to_rows && r.vlen > AGR_REC) {               // a refusal: the host reads the totals before anything moves
            atomicAdd(p.totals + 2, 1ull);
            atomicMin(p.totals + 3, k << 32 | r.vlen);
        }
    }
    rl_block_scan(a, b, ta, tb);
    if (threadIdx.x == 0) { p.tile_sum[2 * blockIdx.x] = ta; p.tile_sum[2 * blockIdx.x + 1] = tb; }
}
// one CTA: exclusive scan of the tile sums in place, the totals into p.totals
__global__ void __launch_bounds__(RL_T) k_rl_scan(const agr_relayout p, const uint32_t tiles) {
    unsigned long long ca = 0, cb = 0;
    for (uint32_t base = 0; base < tiles; base += RL_T) {
        const uint32_t i = base + threadIdx.x;
        unsigned long long a = i < tiles ? p.tile_sum[2 * i] : 0ull, b = i < tiles ? p.tile_sum[2 * i + 1] : 0ull, ta, tb;
        rl_block_scan(a, b, ta, tb);
        if (i < tiles) { p.tile_sum[2 * i] = ca + a; p.tile_sum[2 * i + 1] = cb + b; }
        ca += ta; cb += tb;
    }
    if (threadIdx.x == 0) { p.totals[0] = ca; p.totals[1] = cb; }
}

// Row move.  Thread t of tile T takes the RL_PER consecutive rows k = T * RL_TILE + t * RL_PER + j: their packed offsets are
// the tile's prefix plus a block scan, written with every other per-row word to the target row (row id mod the target's
// slab_rows), and the rows' byte segments go to the segment lists of the byte move (a variable-length target: from the
// source's record bytes, or from its 512 B rows, cut to their compact length).  Then (fixed-stride target) each warp writes
// RL_TILE / 8 of the tile's 512 B rows, one 16 B vector per lane: copied from the source's rows, or gathered from its record
// bytes and zero past vlen.
__device__ __forceinline__ uint4 rl_row16(const agr_relayout& p, unsigned long long k, uint32_t lane) {
    const uint32_t ps = row_physical(p.s, p.s.tail + k);
    if (!p.s.voff) return ldg_nc_v4(p.s.slab + (size_t)ps * AGR_REC + lane * 16u);
    const uint32_t vl = p.s.state[ps] ? p.s.vlen[ps] : 0u;
    return lane * 16u < vl ? ldg_nc_v4(p.s.slab + p.s.voff[ps] + lane * 16u) : make_uint4(0u, 0u, 0u, 0u);
}
__global__ void __launch_bounds__(RL_T) k_rl_rows(const agr_relayout p) {
    const unsigned long long k0 = (unsigned long long)blockIdx.x * RL_TILE + threadIdx.x * RL_PER;
    rl_row r[RL_PER];
    unsigned long long a = 0, b = 0, ta, tb;
#pragma unroll
    for (uint32_t j = 0; j < RL_PER; ++j) {
        r[j] = rl_row{0u, 0u, 0u, 0u, 0u};
        if (k0 + j < p.n) r[j] = rl_read(p, k0 + j);
        a += r[j].vlen; b += rl_r16(r[j].rlen) + rl_r16(r[j].elen);
    }
    rl_block_scan(a, b, ta, tb);
    a += p.tile_sum[2 * blockIdx.x]; b += p.tile_sum[2 * blockIdx.x + 1];
#pragma unroll
    for (uint32_t j = 0; j < RL_PER; ++j) {
        const unsigned long long k = k0 + j;
        if (k >= p.n) break;
        const uint32_t ps = r[j].ps, pt = row_physical(p.t, p.s.tail + k);
        const bool live = r[j].st != 0u;
        p.t.state[pt] = r[j].st;
        p.t.route[pt] = p.s.route[ps];
        p.t.aux[pt] = p.s.aux[ps];
        p.t.cksum[pt] = p.s.cksum[ps];
        p.t.ptime[pt] = p.s.ptime[ps];
        p.t.mtime[pt] = p.s.mtime[ps];
        if (p.t.voff) {
            p.t.vlen[pt] = p.s.voff ? p.s.vlen[ps] : r[j].vlen;
            p.t.voff[pt] = live ? a : 0ull;
            p.vseg_dst[k] = a; p.vseg_src[k] = !live ? 0ull : p.s.voff ? p.s.voff[ps] : (unsigned long long)ps * AGR_REC;
            p.vseg_len[k] = r[j].vlen;
            a += r[j].vlen;
        }
        const uint32_t rl = p.sw.resp_len[ps], el = p.sw.err_len[ps];
        const unsigned long long eo = b + rl_r16(r[j].rlen);
        p.tw.resp_len[pt] = rl; p.tw.resp_hlen[pt] = p.sw.resp_hlen[ps]; p.tw.err_len[pt] = el;
        p.tw.resp_off[pt] = (live && rl) ? b : 0ull;
        p.tw.err_off[pt] = (live && el) ? eo : 0ull;
        p.rseg_dst[2 * k] = b; p.rseg_src[2 * k] = r[j].rlen ? p.sw.resp_off[ps] : 0ull; p.rseg_len[2 * k] = r[j].rlen;
        p.rseg_dst[2 * k + 1] = eo; p.rseg_src[2 * k + 1] = r[j].elen ? p.sw.err_off[ps] : 0ull; p.rseg_len[2 * k + 1] = r[j].elen;
        b = eo + rl_r16(r[j].elen);
    }
    if (p.t.voff) return;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const unsigned long long w0 = (unsigned long long)blockIdx.x * RL_TILE + warp * (RL_TILE / 8u);
    for (uint32_t q = 0; q < RL_TILE / 8u; q += 4u) {
        uint4 v[4];
#pragma unroll
        for (uint32_t u = 0; u < 4u; ++u) {                 // four rows' loads in flight per lane
            const unsigned long long k = w0 + q + u;
            if (k < p.n) v[u] = rl_row16(p, k, lane);
        }
#pragma unroll
        for (uint32_t u = 0; u < 4u; ++u) {
            const unsigned long long k = w0 + q + u;
            if (k < p.n) *reinterpret_cast<uint4*>(p.t.slab + (size_t)row_physical(p.t, p.s.tail + k) * AGR_REC + lane * 16u) = v[u];
        }
    }
}

// 16 bytes from any address: two aligned 16 B loads and a funnel shift (the second load only when the bytes span it)
__device__ __forceinline__ uint4 rl_load16(const uint8_t* src) {
    const uint32_t sh = (uint32_t)reinterpret_cast<uintptr_t>(src) & 15u;
    const uint4* as = reinterpret_cast<const uint4*>(src - sh);
    const uint4 lo = __ldg(as);
    if (!sh) return lo;
    const uint4 hi = __ldg(as + 1);
    uint32_t w0 = lo.x, w1 = lo.y, w2 = lo.z, w3 = lo.w, w4 = hi.x, w5 = hi.y, w6 = hi.z, w7 = hi.w;
    const uint32_t q = sh >> 2, rs = (sh & 3u) * 8u;
    if (q & 2u) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; w5 = w7; }
    if (q & 1u) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
    return make_uint4(__funnelshift_r(w0, w1, rs), __funnelshift_r(w1, w2, rs), __funnelshift_r(w2, w3, rs), __funnelshift_r(w3, w4, rs));
}
// first index in [lo, hi) whose seg_dst is > x (seg_dst is non-decreasing)
__device__ __forceinline__ unsigned long long rl_upper(const unsigned long long* d, unsigned long long lo, unsigned long long hi, unsigned long long x) {
    while (lo < hi) {
        const unsigned long long m = lo + ((hi - lo) >> 1);
        if (__ldg(d + m) <= x) lo = m + 1; else hi = m;
    }
    return lo;
}
// Byte move, balanced by bytes: CTA c writes destination bytes [c * RL_CHUNK, (c + 1) * RL_CHUNK) in 16 B words, whatever rows
// they belong to.  A word inside one segment is one unaligned 16 B read; a word that spans segment ends (or 16 B padding, which
// is written as zero) is assembled byte by byte.
__global__ void __launch_bounds__(RL_T) k_rl_bytes(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                   const unsigned long long* __restrict__ seg_dst, const unsigned long long* __restrict__ seg_src,
                                                   const uint32_t* __restrict__ seg_len, const unsigned long long nseg, const unsigned long long total) {
    __shared__ unsigned long long s_lo, s_hi;
    const unsigned long long c0 = (unsigned long long)blockIdx.x * RL_CHUNK;
    if (threadIdx.x == 0) {
        s_lo = rl_upper(seg_dst, 0, nseg, c0) - 1;            // (seg_dst[0] = 0 <= c0)
        s_hi = rl_upper(seg_dst, s_lo, nseg, c0 + RL_CHUNK - 1);
    }
    __syncthreads();
    const unsigned long long jlo = s_lo, jhi = s_hi;
#pragma unroll 1
    for (uint32_t i = 0; i < RL_WORDS; ++i) {
        const unsigned long long x = c0 + 16ull * (threadIdx.x + i * RL_T);
        if (x >= total) break;
        unsigned long long j = rl_upper(seg_dst, jlo, jhi, x) - 1;
        unsigned long long d0 = seg_dst[j], n0 = seg_len[j];
        uint4 v;
        if (x + 16 <= d0 + n0) {
            v = rl_load16(src + seg_src[j] + (x - d0));
        } else {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            for (uint32_t q = 0; q < 16u; ++q) {
                const unsigned long long at = x + q;
                while (j + 1 < jhi && seg_dst[j + 1] <= at) { ++j; d0 = seg_dst[j]; n0 = seg_len[j]; }
                const uint32_t byte = at < d0 + n0 ? src[seg_src[j] + (at - d0)] : 0u;
                w[q >> 2] |= byte << (8u * (q & 3u));
            }
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        *reinterpret_cast<uint4*>(dst + x) = v;
    }
}

// log remap: a source physical row -> its row id in the source's window -> the target's physical row
__global__ void __launch_bounds__(256) k_rl_log(const agr_dev s, const agr_dev t, const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                const unsigned long long len) {
    const unsigned long long i = (unsigned long long)blockIdx.x * 256u + threadIdx.x;
    if (i >= len) return;
    const uint32_t e = in[i];
    out[i] = e == AGR_RID_NONE ? AGR_RID_NONE : row_physical(t, row_logical(s, e));
}

uint32_t agr_relayout_tiles(unsigned long long n) { return (uint32_t)((n + RL_TILE - 1) / RL_TILE); }
void agr_launch_relayout_count(const agr_relayout& p, cudaStream_t st) {
    const uint32_t tiles = agr_relayout_tiles(p.n);
    if (tiles) k_rl_count<<<tiles, RL_T, 0, st>>>(p);
    k_rl_scan<<<1, RL_T, 0, st>>>(p, tiles);
}
void agr_launch_relayout_rows(const agr_relayout& p, cudaStream_t st) {
    const uint32_t tiles = agr_relayout_tiles(p.n);
    if (tiles) k_rl_rows<<<tiles, RL_T, 0, st>>>(p);
}
void agr_launch_relayout_bytes(const uint8_t* src, uint8_t* dst, const unsigned long long* seg_dst, const unsigned long long* seg_src,
                               const uint32_t* seg_len, unsigned long long nseg, unsigned long long total, cudaStream_t st) {
    if (total) k_rl_bytes<<<(unsigned)((total + RL_CHUNK - 1) / RL_CHUNK), RL_T, 0, st>>>(src, dst, seg_dst, seg_src, seg_len, nseg, total);
}
void agr_launch_relayout_log(const agr_dev& s, const agr_dev& t, const uint32_t* in, uint32_t* out, unsigned long long len, cudaStream_t st) {
    if (len) k_rl_log<<<(unsigned)((len + 255) / 256), 256, 0, st>>>(s, t, in, out, len);
}
