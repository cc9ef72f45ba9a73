// Tile lists of the sparse box3d and box2d towers (TowerTilesParams, b3d_sparse.cuh).
//
// One CTA per (level, image).  Every seed pixel lowers, by an atomicMin (order free, so deterministic), the Chebyshev
// distance of the conv tiles around it: the distance from the seed pixel to the part of the tile inside the map.  The box3d
// tower's seeds are the final candidates of the decode's `fin` list, read by the CTA itself into shared memory; the box2d
// tower's are the pixels of P, marked by tower_mark_kernel (one thread per head pixel) in the global `dist` array, which the
// CTA copies and resets.  List i holds the tiles with distance <= reach - i, in row-major order, written to the (level,
// image) region of the staging area, padded to a multiple of 4 entries (the work unit of the list-mode pair tile) with the
// out-of-image tile; the box2d predictor's list (pred16) holds 16x8 tiles, unpadded.  The last CTA to finish (atomic ticket, no waiting) concatenates the regions
// level-major, then image -- a fixed order, so the lists and the conv schedule do not depend on timing -- writes the counts
// and resets the ticket.
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

// seed pixel (py, px): lower the distance of every tile within `reach` of it (dist: shared or global, [tiles_y][tiles_x])
__device__ __forceinline__ void seed_tiles(int* dist, const TowerTilesLevel& L, int py, int px, int reach) {
    const int ty0 = max(py - reach, 0) / L.th, ty1 = min(py + reach, L.H - 1) / L.th;
    const int tx0 = max(px - reach, 0) / L.tw, tx1 = min(px + reach, L.W - 1) / L.tw;
    for (int ty = ty0; ty <= ty1; ++ty) {
        const int y0 = ty * L.th, y1 = min(y0 + L.th, L.H) - 1;
        const int dy = py < y0 ? y0 - py : (py > y1 ? py - y1 : 0);
        for (int tx = tx0; tx <= tx1; ++tx) {
            const int x0 = tx * L.tw, x1 = min(x0 + L.tw, L.W) - 1;
            const int dx = px < x0 ? x0 - px : (px > x1 ? px - x1 : 0);
            atomicMin(&dist[ty * L.tiles_x + tx], max(dy, dx));
        }
    }
}

// (level, image) region of a layer's staging / list area, and of `dist`: the level's tiles per image rounded up to a
// multiple of 4
__device__ __forceinline__ int region_size(const TowerTilesLevel& L) { return (L.tiles_x * L.tiles_y + 3) & ~3; }
__device__ __forceinline__ size_t region(const TowerTilesLevel& L, int b) {
    return L.stage_begin + static_cast<size_t>(b) * region_size(L);
}

// One thread per head pixel, the grid of the decode's dense passes: the pixels of P seed the tiles around them.
constexpr int kMarkThreads = kTowerMarkThreads;
__global__ void __launch_bounds__(kMarkThreads) tower_mark_kernel(const __grid_constant__ TowerTilesParams p) {
    DD3D_PDL_PROLOGUE();
    int l = 0;
#pragma unroll
    for (int i = 1; i < kLevels; ++i)
        if (i < p.num_levels && static_cast<int>(blockIdx.x) >= p.lvl[i].mark_begin) l = i;
    const TowerTilesLevel& L = p.lvl[l];
    const int b = blockIdx.y;
    const int pix = (static_cast<int>(blockIdx.x) - L.mark_begin) * kMarkThreads + static_cast<int>(threadIdx.x);
    const int hw = L.H * L.W;
    if (pix >= hw || !class_passes(L.cls + (static_cast<size_t>(b) * hw + pix) * p.cls_pitch, p.C, p.thresh)) return;
    const int py = pix / L.W;
    seed_tiles(p.dist + region(L, b), L, py, pix - py * L.W, p.reach);
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
    if (p.fin != nullptr) {
        for (int t = threadIdx.x; t < T; t += kThreads) s_dist[t] = kTowerTileFar;
        __syncthreads();
        const int bl = b * p.num_levels + l;  // fin / cand_count order
        const int n = min(p.cand_count[bl], p.topk);
        for (int c = threadIdx.x; c < n; c += kThreads) {
            const int pix = static_cast<int>(p.fin[static_cast<size_t>(bl) * p.topk + c].y / static_cast<uint32_t>(p.C));
            const int py = pix / L.W;
            seed_tiles(s_dist, L, py, pix - py * L.W, p.reach);
        }
    } else {
        int* dist = p.dist + region(L, b);
        for (int t = threadIdx.x; t < T; t += kThreads) {
            s_dist[t] = __ldcg(dist + t);
            dist[t] = kTowerTileFar;  // ready for the next forward's mark pass
        }
    }
    __syncthreads();

    uint32_t* stage = p.stage + region(L, b);
    for (int i = 0; i < D; ++i) {
        if (threadIdx.x == 0) s_pix = 0;
        // the box2d predictor's list: 16x8 tiles, each the 8x8 tiles 2 ty and 2 ty + 1 of a tile column
        const bool pred = p.pred16 && i == D - 1;
        const int th = pred ? 2 * L.th : L.th, Ti = (pred ? (L.tiles_y + 1) / 2 : L.tiles_y) * L.tiles_x;
        int written = 0;
        for (int base = 0; base < Ti; base += kThreads) {
            const int t = base + threadIdx.x;
            const int ty = t / L.tiles_x, tx = t - ty * L.tiles_x;
            int d = kTowerTileFar;
            if (t < Ti) {
                d = s_dist[pred ? 2 * ty * L.tiles_x + tx : t];
                if (pred && 2 * ty + 1 < L.tiles_y) d = min(d, s_dist[(2 * ty + 1) * L.tiles_x + tx]);
            }
            const bool on = d <= p.reach - i;
            int total;
            const int at = written + block_exclusive_scan(on ? 1 : 0, s_warp, &total);
            if (on) {
                stage[static_cast<size_t>(i) * p.cap + at] = tile_entry(l, b, t);
                atomicAdd(&s_pix, min(th, L.H - ty * th) * min(L.tw, L.W - tx * L.tw));
            }
            written += total;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            // pair tile: the list is padded to whole units with the out-of-image tile T (tile row tiles_y), whose rows are
            // never stored
            while (!pred && (written & 3)) stage[static_cast<size_t>(i) * p.cap + written++] = tile_entry(l, b, T);
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
                const uint32_t* src = p.stage + static_cast<size_t>(i) * p.cap + region(p.lvl[l2], b2);
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

cudaError_t launch_tower_mark(const TowerTilesParams& p, cudaStream_t stream) {
    if (p.dist == nullptr || p.fin != nullptr || p.B < 1 || p.C < 1 || p.cls_pitch < p.C || p.cls_pitch % 4 ||
        p.mark_blocks < 1 || p.reach < 0 || p.num_levels < 1 || p.num_levels > kLevels)
        return cudaErrorInvalidValue;
    return launch_pdl(tower_mark_kernel, dim3(p.mark_blocks, p.B), dim3(kMarkThreads), 0, stream, p);
}

cudaError_t launch_tower_tiles(const TowerTilesParams& p, cudaStream_t stream) {
    if (p.depth < 1 || p.reach < p.depth - 1 || p.B < 1 || p.B > kTileListMaxImages || p.C < 1 ||
        (p.fin != nullptr ? p.topk < 1 : p.dist == nullptr) || p.max_tiles >= kTileListMaxTiles ||
        tower_tiles_smem_bytes(p.max_tiles) > 48 * 1024 || p.num_levels < 1 || p.num_levels > kLevels)
        return cudaErrorInvalidValue;
    return launch_pdl(tower_tiles_kernel, dim3(p.num_levels * p.B), dim3(kThreads), tower_tiles_smem_bytes(p.max_tiles), stream, p);
}

}  // namespace dd3d
