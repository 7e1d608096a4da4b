// agr_k1_tma.cu — K1 (ingest + dedupe + route), TMA variant for sm_90a.
//
// The slab is described to the TMA unit as a 2-D u8 tensor [rows][512 B].  A tile is 32 records (16 KiB), fetched
// as four boxes of [32 rows x 128 B] with the 128 B hardware swizzle: 16 B chunk c of row r lands at chunk
// position c ^ (r & 7) of its 128 B line, so when lane r walks ITS OWN record chunk by chunk, the eight lanes of a
// quarter-warp hit eight different 16 B bank groups — thread-per-record parsing without bank conflicts and without
// a single LSU global load for the record stream (the SM's LSU only sees the index / state traffic).
// Every warp runs its own one-stage mbarrier pipeline over a static schedule of tiles; CTAs are persistent (one per SM,
// 14 warps each), so the grid is exactly the SM count.
#include <cuda.h>

#include "agr_device.cuh"

#define TILE_RECS 32u
#define TILE_BYTES (TILE_RECS * AGR_REC)   // 16384

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// MINT: the engine mints ids (AGR_CFG_MINT_IDS), so k1_begin decides every replay's dedupe hit; the hash-id instantiation carries
// none of that code (the index CAS loop is latency-bound, and the larger loop body cost it ~1.6 us a C2 step on H100).
template <int WARPS, bool MINT>
__global__ void __launch_bounds__(WARPS * 32, 1)
k1_ingest_tma(const __grid_constant__ CUtensorMap tmap, const agr_dev d, const uint32_t first_rid, const unsigned long long first_log,
              const uint32_t n) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t bars[WARPS];
    __shared__ uint32_t s_ctr[K1_NLC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // 128 B swizzle needs 1024 B aligned tiles
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    if (threadIdx.x < K1_NLC) s_ctr[threadIdx.x] = 0;
    if (threadIdx.x < WARPS) mbar_init(smem_u32(&bars[threadIdx.x]), 1);
    if (threadIdx.x == 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    // Programmatic dependent launch (launch_tma): nothing above touches global memory, and the wait returns once the previous
    // kernel of the stream has completed and its writes are visible (at once when the launch was not programmatic).
    asm volatile("griddepcontrol.wait;" ::: "memory");
    // the previous batch is done with the other set of per-batch words: zero it for the next one (k1_post, when it runs, does too)
    if (blockIdx.x == 0 && threadIdx.x < 4) d.dupfix_next[threadIdx.x] = 0;

    uint32_t lc[K1_NLC + 1];
#pragma unroll
    for (int c = 0; c <= K1_NLC; ++c) lc[c] = 0;
    const uint32_t tiles = (n + TILE_RECS - 1) / TILE_RECS;
    const uint32_t my_smem = smem_base + (uint32_t)warp * TILE_BYTES;
    const uint32_t bar = smem_u32(&bars[warp]);

    // static schedule: tile = warp's global index + k * total warps (no atomics on the refill path)
    uint32_t tile = blockIdx.x * WARPS + warp;
    // prologue: issue the first tile
    if (lane == 0 && tile < tiles) {
        mbar_expect_tx(bar, TILE_BYTES);
#pragma unroll
        for (int cb = 0; cb < 4; ++cb) tma_load_2d(my_smem + cb * 4096, &tmap, bar, cb * 128, (int32_t)(first_rid + tile * TILE_RECS));
    }
    // per-lane swizzled chunk offsets inside a [32][128 B] box: row * 128 + ((c ^ (row & 7)) << 4)
    const uint32_t rowoff = (uint32_t)lane * 128u;
    const uint32_t sw = ((uint32_t)lane & 7u) << 4;
    const uint32_t base = my_smem + rowoff;
    uint32_t phase = 0;
    // software pipeline across tiles: the index CAS of tile t is issued in the middle of tile t and consumed in the
    // middle of tile t+1 (k1_finish), so its whole round trip hides behind a tile of checksum work
    k1_ctx pcx; uint4 ph1 = make_uint4(0, 0, 0, 0); uint32_t ph5y = 0, prid = 0, ptile = 0; bool pvalid = false;
    for (uint32_t it = 0; tile < tiles; ++it) {
        mbar_wait(bar, phase);
        const uint32_t i = tile * TILE_RECS + lane;
        const bool valid = i < n;
        const uint32_t rid = first_rid + i;
        // header: chunks 0..5 of this lane's record
        const uint4 h0 = lds128(base + ((0u << 4) ^ sw)), h1 = lds128(base + ((1u << 4) ^ sw)), h2 = lds128(base + ((2u << 4) ^ sw));
        const uint4 h3 = lds128(base + ((3u << 4) ^ sw)), h4 = lds128(base + ((4u << 4) ^ sw)), h5 = lds128(base + ((5u << 4) ^ sw));
        // long-latency work first: agent-table probe, index-line prefetch, and the claim of the NEXT tile
        const ag_probe ap = k1_agent_issue(d, h2, h3);
        if (valid && !(h4.z & AGR_F_REPLAY) && !(d.cfg_flags & AGR_CFG_MINT_IDS))
            prefetch_l2(&d.table[agr_hash_id(pack64(h0.x, h0.y), pack64(h0.z, h0.w)) & d.table_mask]);
        const uint32_t next_tile = tile + gridDim.x * WARPS;
        // position-weighted checksum over the 32 chunks of the record (weights k+1 over the 128 words).  Only shared
        // memory is touched between the wait and the refill, so the stage is held for the checksum alone.
        uint32_t c0 = 0, c1 = 0;
        if (!(d.cfg_flags & AGR_CFG_DIAG_NO_CKSUM)) {
#pragma unroll
            for (int k = 0; k < 32; ++k) {
                const uint4 v = lds128(base + (uint32_t)(k >> 3) * 4096u + ((((uint32_t)k & 7u) << 4) ^ sw));
                c0 += v.x + v.y + v.z + v.w;
                c1 += (uint32_t)(4 * k + 1) * v.x + (uint32_t)(4 * k + 2) * v.y + (uint32_t)(4 * k + 3) * v.z + (uint32_t)(4 * k + 4) * v.w;
            }
        }
        __syncwarp();      // every lane has consumed the stage: refill it right away
        if (lane == 0 && next_tile < tiles) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads before async refill
            mbar_expect_tx(bar, TILE_BYTES);
#pragma unroll
            for (int cb = 0; cb < 4; ++cb) tma_load_2d(my_smem + cb * 4096, &tmap, bar, cb * 128, (int32_t)(first_rid + next_tile * TILE_RECS));
        }
        if (valid) {
            d.cksum[rid] = agr_cksum_pack(c0, c1);
            // a ring sweeps every step: the row's last-SET time (= created_at, requests.go:106) goes into the word the sweep streams,
            // so k_expire never has to fetch created_at out of the 512 B records (one 32 B sector per row)
            if (d.cfg_flags & AGR_CFG_RING) d.mtime[rid] = pack64(h4.x, h4.y);
        }
        k1_note_time(d, first_rid + tile * TILE_RECS, min(TILE_RECS, n - tile * TILE_RECS), valid ? pack64(h4.x, h4.y) : ~0ULL);
        // previous tile: its CAS has had a full tile to come back
        if (it) {                                                 // (warp-uniform: every lane has a previous tile or none has)
            k1_result r{0u, 0u};
            if (pvalid) {
                const uint4 qh5 = make_uint4(0, ph5y, 0, 0);
                r = k1_finish(d, prid, ph1, qh5, pcx, lc);
                d.state[prid] = r.state;
                d.route[prid] = r.route;
            }
            // one bit per row the post pass has to visit (tracked replays): it then reads 4 B per 32 rows instead of every route word
            if (d.marks) {
                const uint32_t mk = __ballot_sync(FULL, pvalid && (rt_flags(r.route) & (AGR_VF_REPLAY | AGR_VF_DUP_ID)) == (AGR_VF_REPLAY | AGR_VF_DUP_ID));
                if (lane == 0) d.marks[ptile] = mk;
            }
        }
        // this tile: agent loads have landed by now; classify and put the index CAS in flight.  pcx is dead here
        // (just consumed), so the CAS writes straight into the loop-carried registers.
        if (valid) k1_begin(d, ap, h0, h1, h2, h3, h4, h5.x, AGR_REC - AGR_OFF_PAYLOAD, MINT, first_log, first_log + i, i, pcx);
        ph1 = h1; ph5y = h5.y; prid = rid; pvalid = valid; ptile = tile;
        phase ^= 1u;
        tile = next_tile;
    }
    // The next K1 on the stream may start once every CTA of this one has streamed its tiles: its launch is processed during this
    // launch's drain, and its CTAs take each SM the moment this launch's CTA leaves it.  (Measured on H100: ~0.5 us a step
    // better than triggering at the start.)
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if ((blockIdx.x * WARPS + warp) < tiles) {                    // this warp had at least one tile: flush its last one
        k1_result r{0u, 0u};
        if (pvalid) {
            const uint4 qh5 = make_uint4(0, ph5y, 0, 0);
            r = k1_finish(d, prid, ph1, qh5, pcx, lc);
            d.state[prid] = r.state;
            d.route[prid] = r.route;
        }
        if (d.marks) {
            const uint32_t mk = __ballot_sync(FULL, pvalid && (rt_flags(r.route) & (AGR_VF_REPLAY | AGR_VF_DUP_ID)) == (AGR_VF_REPLAY | AGR_VF_DUP_ID));
            if (lane == 0) d.marks[ptile] = mk;
        }
    }
    k1_flush_counters(d, lc, s_ctr);
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int agr_k1_tma_make_map(void* slab, unsigned long long rows, void* out_map /*128 B*/) {
    static encode_tiled_fn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return -1;
        fn = (encode_tiled_fn)p;
    }
    const cuuint64_t dims[2] = {AGR_REC, rows};
    const cuuint64_t strides[1] = {AGR_REC};
    const cuuint32_t box[2] = {128, TILE_RECS};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = fn((CUtensorMap*)out_map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, slab, dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

template <bool MINT>
static cudaError_t launch_tma(const void* map, const agr_dev& d, uint32_t first_rid, unsigned long long first_log, uint32_t n,
                             int sm_count, cudaStream_t st) {
    constexpr int WARPS = 14;
    const size_t smem = (size_t)WARPS * TILE_BYTES + 1024;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(k1_ingest_tma<WARPS, MINT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr_done = true;
    }
    const uint32_t tiles = (n + TILE_RECS - 1) / TILE_RECS;
    uint32_t blocks = (uint32_t)sm_count;
    const uint32_t need = (tiles + WARPS - 1) / WARPS;
    if (blocks > need) blocks = need;
    // programmatic stream serialization: the launch may start during the tail of the kernel before it on the stream (the kernel
    // waits for that one to complete before it touches global memory)
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k1_ingest_tma<WARPS, MINT>, *(const CUtensorMap*)map, d, first_rid, first_log, n);
}

// one persistent CTA of 14 warps per SM, each warp with one 16 KiB stage
cudaError_t agr_launch_k1_tma(const void* map, const agr_dev& d, uint32_t first_rid, unsigned long long first_log, uint32_t n,
                              int sm_count, cudaStream_t st) {
    return (d.cfg_flags & AGR_CFG_MINT_IDS) ? launch_tma<true>(map, d, first_rid, first_log, n, sm_count, st)
                                            : launch_tma<false>(map, d, first_rid, first_log, n, sm_count, st);
}
