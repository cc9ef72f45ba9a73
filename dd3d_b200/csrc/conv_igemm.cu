// Implicit-GEMM convolution: host side (tensor maps, tiling policy, launch) and the taps-in-N kernel.  The main kernel and its
// design notes are in conv_igemm_kernel.cuh.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>

#include "conv_igemm_kernel.cuh"
#include "device_once.cuh"

namespace dd3d {

namespace {

// =========================================================================================== taps-in-N variant
// 3x3 stride-1 convolutions with <= 16 output channels (FCOS predictors cls / [box2d_reg | centerness], DLA level0).
// As nine N = 16 GEMMs per 64-channel block they sit at the tensor-core instruction floor.  Here the taps are GEMM COLUMNS:
//   P[pixel of the (16+2)x(8+2) halo patch][tap * 16 + co] = sum_c in[pixel][c] * W[co][tap][c]
// -- three M64 x N144 x K16 wgmmas per K step (one per consumer warpgroup: patch rows 0..63, 64..127, 128..191) over the
// SAME halo patch the halo variant stages -- and the output is the shifted sum
//   out[y][x][co] = sum_{r,s} P[(y + r) * 10 + (x + s)][(3 r + s) * 16 + co]
// taken from shared memory in a fixed order (deterministic).  9x fewer tensor cycles, no extra HBM traffic.
constexpr int kTapsThreads = 512;                 // warpgroup 0: TMA (warp 0); warpgroups 1..3: wgmma + epilogue
constexpr int kTapsStages = 2;
constexpr int kTapsBBytes = kTapsN * 128;         // 18 KiB weight tile per 64-channel block
constexpr int kTapsPStride = 148;                 // fp32 words per patch pixel in P (144 + 4: conflict-free 128-bit access)
constexpr int kTapsPRows = kHaloPW * kHaloPH;     // 180
constexpr int kTapsPBytes = (kTapsPRows * kTapsPStride * 4 + 1023) / 1024 * 1024;
constexpr int kTapsSmem = kTapsStages * (kHaloABytes + kTapsBBytes) + kTapsPBytes + kBarBytes + 1024;
constexpr int kTapsConsumerWarps = 12;

template <bool F16>
__global__ void __launch_bounds__(kTapsThreads, 1) conv_taps_kernel(const __grid_constant__ ConvParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    // [A patches x stages | B tiles x stages | P | barriers].  The third warpgroup reads patch rows 128..191; rows 180..191
    // lie past the patch (in the next slot / the B tiles): finite values that only reach accumulator rows never stored.
    uint8_t* a_base = smem;
    uint8_t* b_base = smem + kTapsStages * kHaloABytes;
    const uint32_t p_u32 = ptx::smem_u32(b_base + kTapsStages * kTapsBBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + kTapsStages * kTapsBBytes + kTapsPBytes);
    uint64_t* full_bar = bars;                   // [kTapsStages]
    uint64_t* empty_bar = bars + kTapsStages;    // [kTapsStages]

    const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&p.w_map);
        for (int s = 0; s < p.nseg; ++s) ptx::prefetch_tensormap(&p.seg[s].in_map[0]);
        for (int i = 0; i < kTapsStages; ++i) {
            ptx::mbar_init(&full_bar[i], 1);
            ptx::mbar_init(&empty_bar[i], kTapsConsumerWarps);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const int w_first = static_cast<int>(blockIdx.x), w_step = static_cast<int>(gridDim.x), w_total = p.total_work;
    if (warp == 0) {
        // ------------------------------------------------------------ TMA producer: halo patch + weight tile per 64-ch block
        int stage = 0;
        uint32_t phase = 0;
        for (int work = w_first; work < w_total; work += w_step) {
            const TileCoord t = decode_tile(p, work);
            const ConvSeg& g = p.seg[t.seg];
            for (int kc = 0; kc < p.kchunks; ++kc) {
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                if (elect_one()) {
                    ptx::mbar_expect_tx(&full_bar[stage], kHaloPW * kHaloPH * 128 + kTapsBBytes);
                    ptx::tma_load_4d(a_base + stage * kHaloABytes, &g.in_map[0], &full_bar[stage], kc * kBlockK, t.x0 - 1,
                                     t.y0 - 1, t.img);
                    ptx::tma_load_2d(b_base + stage * kTapsBBytes, &p.w_map, &full_bar[stage], kc * kBlockK, 0);
                }
                __syncwarp();
                if (++stage == kTapsStages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    } else if (warp >= 4) {
        // ------------------------------------------------------------ consumers: wgmma into registers, dump P, shifted sum
        const int slice = (warp >> 2) - 1;  // patch rows 64 * slice ..
        const int et = static_cast<int>(threadIdx.x) - 128;
        const int wl = (et >> 5) & 3;
        const uint64_t desc_hi = ptx::make_sw128_desc(0) & ~0x3FFFull;
        const uint32_t a_lo0 = (ptx::smem_u32(a_base) >> 4) + slice * (64 * 128 / 16);
        const uint32_t b_lo0 = ptx::smem_u32(b_base) >> 4;
        float acc[kTapsN / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int work = w_first; work < w_total; work += w_step) {
            const TileCoord t = decode_tile(p, work);
            const ConvSeg& g = p.seg[t.seg];
            for (int kc = 0; kc < p.kchunks; ++kc) {
                ptx::mbar_wait(&full_bar[stage], phase);
                const uint32_t a_lo = a_lo0 + static_cast<uint32_t>(stage) * (kHaloABytes >> 4);
                const uint32_t b_lo = b_lo0 + static_cast<uint32_t>(stage) * (kTapsBBytes >> 4);
                mma_kblock<kTapsN, F16>(acc, desc_hi | a_lo, desc_hi | b_lo, kc == 0);
                wg::wait<0>();
                if (lane == 0) ptx::mbar_arrive(&empty_bar[stage]);
                if (++stage == kTapsStages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wg::fence_regs(acc);
            // ---- 1. registers -> P (fp32 [180][148])
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int prow = 64 * slice + 16 * wl + (lane >> 2) + 8 * h;
                if (prow < kTapsPRows) {
                    const uint32_t dst = p_u32 + prow * (kTapsPStride * 4) + 2 * (lane & 3) * 4;
#pragma unroll
                    for (int j = 0; j < kTapsN / 8; ++j)
                        ptx::st_shared_f2(dst + 8 * j * 4, make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
                }
            }
            ptx::named_bar_sync(1, kTapsConsumerWarps * 32);  // P complete
            if (et < 128) {
                // ---- 2. out[y][x][:] = sum over the nine taps of the shifted partial sums (fixed order r, s)
                const int m = et;
                const int ly = m >> 3, lx = m & 7;
                const int oy = t.y0 + ly, ox = t.x0 + lx;
                float sum[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) sum[i] = 0.f;
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
                    const int r = tap / 3, s = tap - 3 * r;
                    const uint32_t src = p_u32 + ((ly + r) * kHaloPW + lx + s) * (kTapsPStride * 4) + tap * 64;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 f = ptx::ld_shared_f4(src + 16 * i);
                        sum[4 * i + 0] += f.x;
                        sum[4 * i + 1] += f.y;
                        sum[4 * i + 2] += f.z;
                        sum[4 * i + 3] += f.w;
                    }
                }
                if (oy < g.H && ox < g.W) {
                    float y[16];
#pragma unroll
                    for (int i = 0; i < 16; i += 4) {
                        const float4 sc = __ldg(reinterpret_cast<const float4*>(g.scale + i));
                        const float4 bi = __ldg(reinterpret_cast<const float4*>(g.bias + i));
                        y[i + 0] = fmaf(sum[i + 0], sc.x, bi.x);
                        y[i + 1] = fmaf(sum[i + 1], sc.y, bi.y);
                        y[i + 2] = fmaf(sum[i + 2], sc.z, bi.z);
                        y[i + 3] = fmaf(sum[i + 3], sc.w, bi.w);
                    }
                    if (p.relu) {
#pragma unroll
                        for (int i = 0; i < 16; ++i) y[i] = fmaxf(y[i], 0.f);
                    }
                    const size_t pix = static_cast<size_t>(t.img * g.H + oy) * g.W + ox;
                    if (p.out_mode == 1) {
                        float* dst = g.out_f32 + pix * g.out_pitch;
#pragma unroll
                        for (int i = 0; i < 16; i += 4) {
                            float4 o = make_float4(y[i], y[i + 1], y[i + 2], y[i + 3]);
                            if (g.lo != nullptr) {
                                const float4 lo = __ldg(reinterpret_cast<const float4*>(g.lo + i));
                                o.x = fmaxf(o.x, lo.x);
                                o.y = fmaxf(o.y, lo.y);
                                o.z = fmaxf(o.z, lo.z);
                                o.w = fmaxf(o.w, lo.w);
                            }
                            *reinterpret_cast<float4*>(dst + i) = o;
                        }
                    } else {
                        uint4 o0, o1;
                        o0.x = pack2_act(y[0], y[1], F16 ? 1 : 0);
                        o0.y = pack2_act(y[2], y[3], F16 ? 1 : 0);
                        o0.z = pack2_act(y[4], y[5], F16 ? 1 : 0);
                        o0.w = pack2_act(y[6], y[7], F16 ? 1 : 0);
                        o1.x = pack2_act(y[8], y[9], F16 ? 1 : 0);
                        o1.y = pack2_act(y[10], y[11], F16 ? 1 : 0);
                        o1.z = pack2_act(y[12], y[13], F16 ? 1 : 0);
                        o1.w = pack2_act(y[14], y[15], F16 ? 1 : 0);
                        uint4* dst = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(g.out16) + pix * g.out_pitch);
                        dst[0] = o0;
                        dst[1] = o1;
                    }
                }
            }
            ptx::named_bar_sync(1, kTapsConsumerWarps * 32);  // every thread is done with P before the next tile's dump
        }
    }
}

// ------------------------------------------------------------------------------------------- host side

thread_local std::string g_conv_error;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres);
        if (e != cudaSuccess || sym == nullptr) {
            g_conv_error = std::string("cuTensorMapEncodeTiled unavailable: ") + cudaGetErrorString(e);
            return nullptr;
        }
        fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

bool encode(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
            const cuuint32_t* box, CUtensorMapL2promotion promo, int fp16,
            CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn fn = get_encode_fn();
    if (fn == nullptr) return false;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swz, promo,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu,%llu]",
                 static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                 (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0));
        g_conv_error = buf;
        return false;
    }
    return true;
}

}  // namespace

const char* conv_last_error() { return g_conv_error.c_str(); }

// NHWC bf16 activation view: C logical channels of a buffer with `pitch` channels per pixel.
bool make_act_map(CUtensorMap* map, const void* base, int B, int H, int W, int C, int pitch, int th, int tw, int fp16) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)tw, (cuuint32_t)th, 1};
    return encode(map, base, 4, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, fp16);
}

// Parity-split view for stride-2 convs: element (b, 2*h2+hp, 2*w2+wp, c) -> coords {c, w2, hp, h2, b} of map[wp].
bool make_act_map_s2(CUtensorMap* map, const void* base, int wp, int B, int H, int W, int C, int pitch, int th,
                     int tw, int fp16) {
    const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(base) + (size_t)wp * pitch;
    cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)(W / 2), 2, (cuuint64_t)(H / 2), (cuuint64_t)B};
    cuuint64_t strides[4] = {(cuuint64_t)2 * pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)2 * W * pitch * 2,
                             (cuuint64_t)H * W * pitch * 2};
    cuuint32_t box[5] = {(cuuint32_t)kBlockK, (cuuint32_t)tw, 1, (cuuint32_t)th, 1};
    return encode(map, b, 5, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, fp16);
}

bool make_weight_map_taps(CUtensorMap* map, const void* base, int cin_pad, int fp16) {
    cuuint64_t dims[2] = {(cuuint64_t)cin_pad, (cuuint64_t)kTapsN};
    cuuint64_t strides[1] = {(cuuint64_t)cin_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)kTapsN};
    return encode(map, base, 2, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, fp16);
}

// taps-in-N needs the fixed 16x8 halo tiling (same rule as the halo variant) and a 16-wide output
static int g_taps_mode = -1;  // DD3D_CONV_TAPS=0 / dd3d_set_conv_policy("taps", 0) disables the variant (A/B, tests)

void conv_set_taps(int mode) { g_taps_mode = (mode == 0 || mode == 1) ? mode : -1; }

bool conv_taps_eligible(int taps, int stride, int cout_pad, int nseg, const int* Hs, const int* Ws) {
    if (g_taps_mode < 0) {
        const char* e = getenv("DD3D_CONV_TAPS");
        g_taps_mode = (e && atoi(e) == 0) ? 0 : 1;
    }
    const int mode = g_taps_mode;
    return mode && taps == 9 && stride == 1 && cout_pad == 16 && conv_prefer_halo(taps, stride, cout_pad, nseg, Hs, Ws);
}

int conv_halo_mode() { return 2; }  // one 128B-swizzled [18][10][64ch] box per 64-channel block

bool make_act_map_halo(CUtensorMap* map, const void* base, int B, int H, int W, int C, int pitch, int fp16) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)kHaloPW, (cuuint32_t)kHaloPH, 1};
    return encode(map, base, 4, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, fp16);
}

bool conv_prefer_halo(int taps, int stride, int block_n, int nseg, const int* Hs, const int* Ws) {
    if (taps != 9 || stride != 1) return false;
    (void)block_n;
    static int mode = -1;  // 0 auto, 1 generic, 2 halo
    if (mode < 0) {
        const char* e = getenv("DD3D_CONV_MODE");
        mode = (e && !strcmp(e, "generic")) ? 1 : (e && !strcmp(e, "halo")) ? 2 : 0;
    }
    if (mode == 1) return false;
    if (mode == 2) return true;
    long halo_tiles = 0, gen_tiles = 0;
    for (int s = 0; s < nseg; ++s) {
        int th, tw;
        choose_tile(Hs[s], Ws[s], &th, &tw);
        gen_tiles += (long)((Hs[s] + th - 1) / th) * ((Ws[s] + tw - 1) / tw);
        halo_tiles += (long)((Hs[s] + kHaloTh - 1) / kHaloTh) * ((Ws[s] + kHaloTw - 1) / kHaloTw);
    }
    return halo_tiles * 100 <= gen_tiles * 110;  // fixed 16x8 tiling may cost at most 10 % more tiles
}

bool make_weight_map(CUtensorMap* map, const void* base, int ktot, int cout_pad, int block_n, int fp16) {
    cuuint64_t dims[2] = {(cuuint64_t)ktot, (cuuint64_t)cout_pad};
    cuuint64_t strides[1] = {(cuuint64_t)ktot * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)block_n};
    return encode(map, base, 2, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, fp16);
}

// Pick the 128-pixel patch shape that wastes the fewest out-of-image pixels.
void choose_tile(int H, int W, int* th, int* tw) {
    static const int shapes[][2] = {{8, 16}, {4, 32}, {16, 8}, {2, 64}, {1, 128}, {32, 4}};
    long best = -1;
    for (auto& s : shapes) {
        long tiles = (long)((H + s[0] - 1) / s[0]) * ((W + s[1] - 1) / s[1]);
        if (best < 0 || tiles < best) {
            best = tiles;
            *th = s[0];
            *tw = s[1];
        }
    }
}

int conv_tiles_per_image(int H, int W) {
    int th, tw;
    choose_tile(H, W, &th, &tw);
    return ((H + th - 1) / th) * ((W + tw - 1) / tw);
}

// M units per image of a segment: tiles, or tile pairs with the pair tile
static int conv_units_per_image(const ConvParams& p, const ConvSeg& g) {
    const int tiles = ((g.W + g.tw - 1) / g.tw) * ((g.H + g.th - 1) / g.th);
    return p.pair ? (tiles + 1) / 2 : tiles;
}

// Dynamic shared memory of everything but the B ring: staging tiles, alignment slack, barriers, (scale, bias) vectors and
// the A patches (pair tile: two staging tiles per consumer warpgroup, two patches per A stage).
static int conv_fixed_smem(const ConvParams& p) {
    return (p.pair ? 4 : 2) * kStagingBytes + 1024 /*alignment slack*/ + kBarBytes + kSbBytes +
           p.a_stages * (p.pair ? 2 : 1) * kHaloABytes;
}

void conv_finalize_params(ConvParams* p) {
    int unit = 0;
    for (int s = 0; s < p->nseg; ++s) {
        ConvSeg& g = p->seg[s];
        g.tw_shift = 0;
        while ((1 << g.tw_shift) < g.tw) ++g.tw_shift;
        g.tiles_x = (g.W + g.tw - 1) / g.tw;
        g.tiles_y = (g.H + g.th - 1) / g.th;
        g.tile_begin = unit;
        const int per_img = conv_units_per_image(*p, g);
        g.inv_per_img = 1.0f / static_cast<float>(per_img);
        g.inv_tiles_x = 1.0f / static_cast<float>(g.tiles_x);
        unit += per_img * p->B;
    }
    p->inv_n_blocks = 1.0f / static_cast<float>(p->n_blocks);
    p->total_work = unit * p->n_blocks;
    const int stage_bytes = (p->halo ? 0 : kABytes) + p->block_n * 128;
    p->a_stages = p->pair ? kPairAStages : p->halo ? kHaloAStages : 0;
    p->wstat = 0;
    // Weight-stationary: a 3x3 layer whose whole weight tensor is a few k-blocks (64 -> 64: 9 x 8 KiB; DLA-34 level2, VoVNet
    // stem_2) would re-stream it through the B ring for every 128-pixel tile -- barely one tile of lookahead against a TMA
    // round trip.  The tensor stays resident instead and the freed barriers / shared memory go to deeper A-patch prefetch.
    // (Never with the pair tile: 128 output channels x 9 taps of even one k-block do not fit next to the patches.)
    if (p->halo && !p->taps_n && !p->pair && p->n_blocks == 1 && conv_wstat_enabled()) {
        const int resident = p->taps * p->kchunks * stage_bytes;
        for (int a = kMaxAStages; a >= kHaloAStages; --a) {
            p->a_stages = a;
            if (conv_fixed_smem(*p) + resident <= kSmemBudget) {
                p->wstat = 1;
                break;
            }
        }
        if (!p->wstat) p->a_stages = kHaloAStages;
    }
    int stages = (kSmemBudget - conv_fixed_smem(*p)) / stage_bytes;
    p->num_stages = p->wstat ? 2 : std::max(2, std::min(kMaxStages, stages));
}

static int g_n_split = -1;
static int g_wstat = -1;
static int g_pair = -1;

void conv_set_pair(int mode) { g_pair = (mode == 0 || mode == 1) ? mode : -1; }

int conv_block_n(int cout_pad) {
    if (cout_pad <= 256) return cout_pad;
    if (cout_pad % 256 == 0) return 256;
    for (int n = 192; n >= 64; n -= 64)
        if (cout_pad % n == 0) return n;
    return 0;
}

bool conv_select_pair(ConvParams* p, int cout_pad, int num_sms) {
    int mode = g_pair;
    if (mode < 0) {
        const char* e = getenv("DD3D_CONV_PAIR");
        mode = (e && atoi(e) == 0) ? 0 : -1;
    }
    if (mode == 0 || !p->halo || p->taps_n || p->out_mode != 0 || cout_pad % 128 != 0) return false;
    p->pair = 1;
    if (mode < 0) {
        // fill rule: below one work item per SM the 128-pixel tile (and the N-split) keeps more SMs busy
        long pairs = 0;
        for (int s = 0; s < p->nseg; ++s) pairs += static_cast<long>(p->B) * conv_units_per_image(*p, p->seg[s]);
        if (pairs * (cout_pad / 128) < num_sms) {
            p->pair = 0;
            return false;
        }
    }
    p->block_n = 128;
    p->n_blocks = cout_pad / 128;
    return true;
}

bool conv_wstat_enabled() {
    if (g_wstat < 0) {
        const char* e = getenv("DD3D_CONV_WSTAT");
        g_wstat = (e && atoi(e) == 0) ? 0 : 1;
    }
    return g_wstat != 0;
}
void conv_set_wstat(int mode) { g_wstat = (mode == 0 || mode == 1) ? mode : -1; }

bool conv_n_split_enabled() {
    if (g_n_split < 0) {
        const char* e = getenv("DD3D_CONV_NSPLIT");
        g_n_split = (e && atoi(e) == 0) ? 0 : 1;
    }
    return g_n_split != 0;
}
void conv_set_n_split(int mode) { g_n_split = (mode == 0 || mode == 1) ? mode : -1; }

cudaError_t launch_conv(const ConvParams& p, int num_sms, cudaStream_t stream) {
    const int stage_bytes = (p.halo ? 0 : kABytes) + p.block_n * 128;
    const int smem_bytes = (p.wstat ? p.taps * p.kchunks : p.num_stages) * stage_bytes + conv_fixed_smem(p);
    ConvKernel kernel = nullptr;
    if (p.tile_list != nullptr && (!p.pair || p.tile_count == nullptr)) return cudaErrorInvalidValue;  // list mode: pair tile only
    if (p.pair) {
        if (!p.halo || p.block_n != 128 || p.out_mode != 0) return cudaErrorInvalidValue;
        kernel = conv_kernel_pair(p.fp16 != 0, p.tile_list != nullptr);
    }
    for (auto group : {conv_kernel_n16_64, conv_kernel_n80_128, conv_kernel_n144_192, conv_kernel_n208_256}) {
        if (kernel == nullptr) kernel = group(p.halo != 0, p.fp16 != 0, p.block_n);
    }
    if (kernel == nullptr) return cudaErrorInvalidValue;  // block_n must be a multiple of 16 in [16, 256] (the wgmma N)
    static uint64_t attr_devices = 0;  // per-device opt-in to > 48 KB dynamic shared memory
    if (first_use_on_device(&attr_devices)) {
        cudaError_t e = cudaSuccess;
        for (bool halo : {false, true}) {
            for (bool fp16 : {false, true}) {
                for (int n = 16; n <= 256; n += 16) {
                    ConvKernel k = nullptr;
                    for (auto group : {conv_kernel_n16_64, conv_kernel_n80_128, conv_kernel_n144_192, conv_kernel_n208_256}) {
                        if (k == nullptr) k = group(halo, fp16, n);
                    }
                    if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget);
                }
            }
        }
        for (bool fp16 : {false, true}) {
            for (bool list : {false, true}) {
                if (e == cudaSuccess)
                    e = cudaFuncSetAttribute(conv_kernel_pair(fp16, list), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kSmemBudget);
            }
        }
        for (auto fn : {conv_taps_kernel<false>, conv_taps_kernel<true>}) {
            if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kTapsSmem);
        }
        if (e != cudaSuccess) return e;
    }
    if (p.total_work <= 0) return cudaSuccess;
    if (p.total_work >= (1 << 24)) return cudaErrorInvalidValue;  // fast_div range of the tile decode
    static int use_pdl = -1;
    if (use_pdl < 0) {
        const char* e = getenv("DD3D_NO_PDL");
        use_pdl = (e && atoi(e)) ? 0 : 1;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(std::min(p.total_work, num_sms));
    cfg.blockDim = dim3(p.taps_n ? kTapsThreads : kConvThreads);
    cfg.dynamicSmemBytes = p.taps_n ? kTapsSmem : smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl ? 1 : 0;
    if (p.taps_n)
        return p.fp16 ? cudaLaunchKernelEx(&cfg, conv_taps_kernel<true>, p) : cudaLaunchKernelEx(&cfg, conv_taps_kernel<false>, p);
    return cudaLaunchKernelEx(&cfg, kernel, p);
}

}  // namespace dd3d
