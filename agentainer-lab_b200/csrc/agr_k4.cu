// agr_k4.cu — K4: shard binning + stable pack for the multi-GPU exchange (SURVEY 8e).
//
// owner(agent_id) = FNV-1a64(id bytes) mod G  (the ABI's shard hash: Go's hash/fnv New64a computes the same).
// k4_count   : owner of every item + per-(warp chunk, owner) counts           (warp-ballot partition, as in K3)
// k4_scan    : column scan -> per-owner totals / offsets
// k4_scatter : stable scatter in owner-major order.  Items owned by this shard go STRAIGHT into their final slab rows;
//              items owned by a peer go to the send buffer at their owner-major position, which is exactly the
//              contiguous segment ncclSend ships — the pack is fused with the placement, nothing is copied twice.
// k4_unpermute: verdicts (or K2 results) that came back from the owners, restored to the caller's item order.
#include "agr_device.cuh"

__device__ __forceinline__ uint32_t k4_owner_of(const uint8_t* agent_id, uint32_t G) {
    // 32 B id as two 16 B loads; FNV-1a over the bytes up to the first NUL
    const uint4 a = ldg_nc_v4(agent_id), b = ldg_nc_v4(agent_id + 16);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    unsigned long long h = 0xcbf29ce484222325ULL;
    bool done = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
#pragma unroll
        for (int s = 0; s < 32; s += 8) {
            const uint32_t c = (w[k] >> s) & 0xffu;
            if (c == 0u) done = true;
            if (!done) { h ^= c; h *= 0x100000001b3ULL; }
        }
    }
    return (uint32_t)(h % G);
}

template <bool SCATTER>
__global__ void __launch_bounds__(256) k4_pass(const agr_k4_params p) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= p.nwarps) return;
    uint32_t* row = p.matrix + (size_t)w * p.G;
    const uint32_t b = w * p.per_warp;
    const uint32_t e = min(p.n, b + p.per_warp);
    for (uint32_t k0 = b; k0 < e; k0 += 32) {
        const uint32_t i = k0 + lane;
        const bool valid = i < e;
        uint32_t owner = 0;
        if (valid) {
            if (SCATTER) owner = p.owner[i];
            else { owner = k4_owner_of(p.items + (size_t)i * p.item_bytes + p.agent_off, p.G); p.owner[i] = (uint8_t)owner; }
        }
        const uint32_t key = valid ? owner : (0x80000000u | (uint32_t)lane);
        const uint32_t peers = __match_any_sync(FULL, key);
        uint32_t pos = 0;
        if (valid) {
            const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
            volatile uint32_t* cell = row + owner;
            const uint32_t base = *cell;
            pos = p.goff ? (SCATTER ? p.goff[owner] + base + rank : 0u) : 0u;
            __syncwarp(peers);
            if (rank == 0) *cell = base + __popc(peers);
        }
        __syncwarp();
        if (SCATTER) {
            // in-place mode (records that were DMA'd straight into their slab rows): own items stay where they are, and the
            // send buffer holds the peers' segments only — positions of owners behind this shard move up by its own count
            if (p.inplace && valid && owner > p.me) pos -= p.gtotal[p.me];
            if (valid) p.perm[i] = pos;
            // warp-cooperative move of the step's items (item_bytes is a multiple of 16)
            const uint32_t chunks = p.item_bytes >> 4;
            if (p.inplace && __all_sync(FULL, !valid || owner == p.me)) continue;     // nothing of this step leaves the shard
            for (int src = 0; src < 32; ++src) {
                const uint32_t si = k0 + src;
                if (si >= e) break;
                const uint32_t sowner = __shfl_sync(FULL, owner, src), spos = __shfl_sync(FULL, pos, src);
                if (p.inplace && sowner == p.me) continue;
                uint8_t* dst = (sowner == p.me) ? p.local_dst + (size_t)(spos - p.goff[p.me]) * p.item_bytes
                                                : p.send_dst + (size_t)spos * p.item_bytes;
                const uint8_t* s = p.items + (size_t)si * p.item_bytes;
                for (uint32_t c = lane; c < chunks; c += 32)
                    *reinterpret_cast<uint4*>(dst + c * 16) = __ldcg(reinterpret_cast<const uint4*>(s + c * 16));
            }
        }
    }
}

__global__ void __launch_bounds__(32) k4_scan(const agr_k4_params p) {
    // G <= 32 owners: one lane per owner walks the warp chunks, then a warp scan gives the owner-major offsets
    const int g = threadIdx.x;
    uint32_t run = 0;
    if ((uint32_t)g < p.G) {
        for (uint32_t w = 0; w < p.nwarps; ++w) {
            uint32_t* cell = p.matrix + (size_t)w * p.G + g;
            const uint32_t c = *cell; *cell = run; run += c;
        }
        p.gtotal[g] = run;
    }
    uint32_t incl = run;
    for (int off = 1; off < 32; off <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, off); if (g >= off) incl += v; }
    if ((uint32_t)g < p.G) p.goff[g] = incl - run;
    if ((uint32_t)g == p.G - 1) p.goff[p.G] = incl;
}

__global__ void __launch_bounds__(256) k4_unpermute(const agr_k4_params p, const uint8_t* __restrict__ local_res,
                                                    const uint8_t* __restrict__ remote_res, uint8_t* __restrict__ out, uint32_t res_bytes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint32_t owner = p.owner[i], pos = p.perm[i];
    const uint8_t* s = (owner == p.me) ? local_res + (size_t)(p.inplace ? i : pos - p.goff[p.me]) * res_bytes : remote_res + (size_t)pos * res_bytes;
    if (res_bytes == 8) *reinterpret_cast<uint2*>(out + (size_t)i * 8) = *reinterpret_cast<const uint2*>(s);
    else *reinterpret_cast<uint32_t*>(out + (size_t)i * 4) = *reinterpret_cast<const uint32_t*>(s);
}

void agr_launch_k4_count(const agr_k4_params& p, cudaStream_t st) {
    cudaMemsetAsync(p.matrix, 0, (size_t)p.nwarps * p.G * sizeof(uint32_t), st);
    agr_k4_params q = p; q.goff = nullptr;
    k4_pass<false><<<(p.nwarps * 32u + 255u) / 256u, 256, 0, st>>>(q);
    k4_scan<<<1, 32, 0, st>>>(p);
}
void agr_launch_k4_scatter(const agr_k4_params& p, cudaStream_t st) {
    k4_pass<true><<<(p.nwarps * 32u + 255u) / 256u, 256, 0, st>>>(p);
}
void agr_launch_k4_unpermute(const agr_k4_params& p, const void* local_res, const void* remote_res, void* out, uint32_t res_bytes,
                             cudaStream_t st) {
    if (p.n) k4_unpermute<<<(p.n + 255u) / 256u, 256, 0, st>>>(p, (const uint8_t*)local_res, (const uint8_t*)remote_res, (uint8_t*)out, res_bytes);
}
