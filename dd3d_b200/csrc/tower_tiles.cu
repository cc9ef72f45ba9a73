// Tile lists of the sparse box3d tower (TowerTilesParams, b3d_sparse.cuh).
//
// One CTA per (level, image).  Every final candidate of the decode's `fin` list lowers, by a shared-memory atomicMin (order
// free, so deterministic), the Chebyshev distance of the conv tiles around it: the distance from the candidate pixel to the
// part of the tile inside the map.  Tower layer i of `depth` is needed at the candidates dilated by depth - i pixels, so its
// list holds the tiles with distance <= depth - i, in row-major order, written to the (level, image) region of the staging
// area.  The last CTA to finish (atomic ticket, no waiting) concatenates the regions level-major, then image -- a fixed order,
// so the lists and the conv schedule do not depend on timing -- writes the counts and resets the ticket.
#include <cuda_runtime.h>
#include <stdint.h>

#include "b3d_sparse.cuh"
#include "conv_igemm.cuh"
#include "pdl.cuh"

namespace dd3d {

namespace {

constexpr int kThreads = 1024, kWarps = kThreads / 32;
constexpr int kCopyBatch = 8;  // list entries per lane in flight while concatenating

// Exclusive prefix of v over the block and the block total.  Every thread of the block calls it; s_warp: kWarps ints.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
        const int c = s_warp[w];
        before += w < warp ? c : 0;
        all += c;
    }
    __syncthreads();  // s_warp may be reused
    *total = all;
    return before + x - v;
}

__device__ __forceinline__ uint32_t tile_entry(int l, int b, int tile) {
    return (static_cast<uint32_t>(l) << 29) | (static_cast<uint32_t>(b) << 16) | static_cast<uint32_t>(tile);
}

__global__ void __launch_bounds__(kThreads) tower_tiles_kernel(const TowerTilesParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ int s_dist[];  // [max_tiles]
    __shared__ int s_warp[kWarps];
    __shared__ int s_at[kThreads], s_n[kThreads];
    __shared__ int s_pix;
    __shared__ unsigned long long s_pix_all;
    __shared__ bool s_last;
    const int nbl = static_cast<int>(gridDim.x);
    const int k = static_cast<int>(blockIdx.x), l = k / p.B, b = k - l * p.B;
    const TowerTilesLevel& L = p.lvl[l];
    const int T = L.tiles_x * L.tiles_y;
    const int D = p.depth;
    for (int t = threadIdx.x; t < T; t += kThreads) s_dist[t] = 1 << 30;
    __syncthreads();
    const int bl = b * kLevels + l;  // fin / cand_count order
    const int n = min(p.cand_count[bl], p.topk);
    for (int c = threadIdx.x; c < n; c += kThreads) {
        const int pix = static_cast<int>(p.fin[static_cast<size_t>(bl) * p.topk + c].y / static_cast<uint32_t>(p.C));
        const int py = pix / L.W, px = pix - py * L.W;
        const int ty0 = max(py - D, 0) / L.th, ty1 = min(py + D, L.H - 1) / L.th;
        const int tx0 = max(px - D, 0) / L.tw, tx1 = min(px + D, L.W - 1) / L.tw;
        for (int ty = ty0; ty <= ty1; ++ty) {
            const int y0 = ty * L.th, y1 = min(y0 + L.th, L.H) - 1;
            const int dy = py < y0 ? y0 - py : (py > y1 ? py - y1 : 0);
            for (int tx = tx0; tx <= tx1; ++tx) {
                const int x0 = tx * L.tw, x1 = min(x0 + L.tw, L.W) - 1;
                const int dx = px < x0 ? x0 - px : (px > x1 ? px - x1 : 0);
                atomicMin(&s_dist[ty * L.tiles_x + tx], max(dy, dx));
            }
        }
    }
    __syncthreads();

    uint32_t* stage = p.stage + L.stage_begin + static_cast<size_t>(b) * (T + (T & 1));
    for (int i = 0; i < D; ++i) {
        if (threadIdx.x == 0) s_pix = 0;
        int written = 0;
        for (int base = 0; base < T; base += kThreads) {
            const int t = base + threadIdx.x;
            const bool on = t < T && s_dist[t] <= D - i;
            int total;
            const int at = written + block_exclusive_scan(on ? 1 : 0, s_warp, &total);
            if (on) {
                stage[static_cast<size_t>(i) * p.cap + at] = tile_entry(l, b, t);
                const int ty = t / L.tiles_x, tx = t - ty * L.tiles_x;
                atomicAdd(&s_pix, min(L.th, L.H - ty * L.th) * min(L.tw, L.W - tx * L.tw));
            }
            written += total;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            // pair tile: an odd list gets the out-of-image tile T (tile row tiles_y), whose rows are never stored
            if (written & 1) stage[static_cast<size_t>(i) * p.cap + written++] = tile_entry(l, b, T);
            p.bl_count[i * nbl + k] = written;
            p.bl_pixels[i * nbl + k] = s_pix;
        }
        __syncthreads();
    }

    // ---- the last CTA concatenates every (level, image) list
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(p.ticket, 1u) == static_cast<unsigned>(nbl - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_pix_all = 0;
    for (int i = 0; i < D; ++i) {
        int written = 0;
        for (int k0 = 0; k0 < nbl; k0 += kThreads) {
            const int kk = k0 + threadIdx.x;
            const int c = kk < nbl ? __ldcg(p.bl_count + i * nbl + kk) : 0;
            int total;
            const int at = written + block_exclusive_scan(c, s_warp, &total);
            s_at[threadIdx.x] = at;
            s_n[threadIdx.x] = c;
            if (kk < nbl) atomicAdd(&s_pix_all, static_cast<unsigned long long>(__ldcg(p.bl_pixels + i * nbl + kk)));
            __syncthreads();
            for (int s = warp; s < min(kThreads, nbl - k0); s += kWarps) {
                const int k2 = k0 + s, l2 = k2 / p.B, b2 = k2 - l2 * p.B;
                const int T2 = p.lvl[l2].tiles_x * p.lvl[l2].tiles_y;
                const uint32_t* src = p.stage + static_cast<size_t>(i) * p.cap + p.lvl[l2].stage_begin +
                                      static_cast<size_t>(b2) * (T2 + (T2 & 1));
                uint32_t* dst = p.list + static_cast<size_t>(i) * p.cap + s_at[s];
                const int cnt = s_n[s];
                for (int j0 = 0; j0 < cnt; j0 += 32 * kCopyBatch) {
                    uint32_t v[kCopyBatch];
#pragma unroll
                    for (int u = 0; u < kCopyBatch; ++u) {
                        const int j = j0 + 32 * u + lane;
                        v[u] = j < cnt ? __ldcg(src + j) : 0u;
                    }
#pragma unroll
                    for (int u = 0; u < kCopyBatch; ++u) {
                        const int j = j0 + 32 * u + lane;
                        if (j < cnt) dst[j] = v[u];
                    }
                }
            }
            written += total;
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            p.count[i] = written;
            p.pixels[i] = static_cast<long long>(s_pix_all);
            s_pix_all = 0;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *p.ticket = 0u;
}

}  // namespace

size_t tower_tiles_smem_bytes(int max_tiles) { return static_cast<size_t>(max_tiles) * 4; }

cudaError_t launch_tower_tiles(const TowerTilesParams& p, cudaStream_t stream) {
    if (p.depth < 1 || p.B < 1 || p.B > kTileListMaxImages || p.topk < 1 || p.C < 1 || p.max_tiles >= kTileListMaxTiles ||
        tower_tiles_smem_bytes(p.max_tiles) > 48 * 1024)
        return cudaErrorInvalidValue;
    return launch_pdl(tower_tiles_kernel, dim3(kLevels * p.B), dim3(kThreads), tower_tiles_smem_bytes(p.max_tiles), stream, p);
}

}  // namespace dd3d
