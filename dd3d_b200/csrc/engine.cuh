#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <array>
#include <map>
#include <string>
#include <vector>

#include "../../include/dd3d_b200.h"
#include "conv_igemm.cuh"
#include "b3d_sparse.cuh"
#include "detect.cuh"
#include "group_norm.cuh"
#include "resize.cuh"
#include "small_kernels.cuh"

namespace dd3d {

struct EngineError {
    int status;
    std::string msg;
    EngineError(int s, std::string m) : status(s), msg(std::move(m)) {}
};

struct HostTensor {
    std::vector<float> data;
    std::vector<int64_t> shape;
};

// NHWC bf16 activation view: C channels starting at ptr, `pitch` channels per pixel in the underlying buffer.
struct View {
    __nv_bfloat16* ptr = nullptr;
    int B = 0, H = 0, W = 0, C = 0, pitch = 0;
    int buf = -1;  // arena buffer this view (or channel slice) lives in: index into the plan's liveness table
};

// One activation buffer of the workspace arena: its size, the first / last engine op that touches it (liveness interval,
// inclusive) and the offset the planner gave it.  Buffers whose intervals do not intersect share memory.
struct ArenaBuf {
    size_t bytes = 0;
    int first = 1 << 30, last = -1;
    bool persistent = false;  // FPN outputs: kept for dd3d_get_tensor after the forward
    size_t offset = 0;
};

struct ConvLayer {
    int cin, cout, ksize, taps, kchunks, ktot, cout_pad, block_n, n_blocks;
    __nv_bfloat16* d_w;
    CUtensorMap w_map;
    __nv_bfloat16* d_w_taps = nullptr;  // taps-in-N layout [9 * 16][cin_pad64] (3x3 layers with cout_pad == 16 only)
    CUtensorMap w_map_taps;
};
struct Epilogue {
    float* d_scale;
    float* d_bias;
    float* d_lo;
};
struct StemLayer {
    __nv_bfloat16* d_w;
    int ksize, stride, cout;
    Epilogue epi;
    __nv_bfloat16* d_w_mma = nullptr;  // 3x3 stride-2 64-channel stem (VoVNet stem_1): [64][3][4][4] for stem_mma.cu
    float* d_sb_mma = nullptr;         // scale[64] | bias[64]
};
struct FrontLayer {  // DLA-34 base_layer + level0 + level1 packed for dla_front.cu
    __nv_bfloat16 *d_w0, *d_w1, *d_w2;
    float *d_sb0, *d_sb1, *d_sb2;
};
struct EseLayer {
    float* d_w;
    float* d_b;
    int C;
};
struct DwLayer {  // depthwise 3x3 weights, 16-bit [9][C]
    __nv_bfloat16* d_w;
    int C;
};

// One VoVNet variant (reference _STAGE_SPECS, vovnet.py:19-97); the table is in engine.cu
struct VovSpec {
    int arch;  // dd3d_arch
    int stem[3];
    int stage_ch[4];
    int out_ch[4];
    int layers;  // layer_per_block
    int blocks[4];
    bool dw;  // depthwise 3x3 layers (and stem_2 / stem_3) with 1x1 conv_reduction where in_ch != stage_ch
};
const VovSpec* vovnet_spec(int arch);  // nullptr: not a VoVNet arch

struct Op {
    enum Type { CONV, STEM, POOL, ESE, RELU, FRONT, DW, GN } type;
    ConvParams conv;
    GroupNormParams gn;  // GN: GroupNorm (or, without gamma, the FPN avg fuse) in place on outs[0..nouts)
    View in, out, identity;
    View outs[kMaxSeg];  // bf16 output views (CONV: one per segment; others: outs[0] == out), for dd3d_get_tensor "op<i>"
    int nouts = 0;
    bool has_identity = false;
    int ksize = 0, stride = 0;
    const StemLayer* stem = nullptr;
    const EseLayer* ese = nullptr;
    const FrontLayer* front = nullptr;  // FRONT: in = input, out = level1 output, identity = its 2x2 max-pool
    const DwLayer* dw = nullptr;        // DW: depthwise 3x3 of `in` into `out` with `stride`
    float* f0 = nullptr;
    float* f1 = nullptr;
    float* f2 = nullptr;
    double flops = 0.0;  // algorithmic FLOPs (2*MACs over the real, unpadded channels)
    double bytes = 0.0;  // algorithmic HBM bytes for the bandwidth-bound ops
};

struct Plan {
    bool valid = false;
    int B = 0, Hs = 0, Ws = 0, Hp = 0, Wp = 0;
    void* owned_workspace = nullptr;
    size_t owned_bytes = 0;
    size_t arena_bytes = 0;  // part of the workspace that holds the liveness-packed bf16 activations
    void* slot1 = nullptr;  // second set of host-path staging buffers (dd3d_submit_host slot 1), allocated on first use
    void* s1_images = nullptr;
    float* s1_K = nullptr;
    int32_t* s1_sizes = nullptr;
    Det* s1_out = nullptr;
    int32_t* s1_counts = nullptr;
    View input;
    View fpn[kLevels];
    float* cls_map[kLevels] = {};
    float* box_map[kLevels] = {};
    float* b3d_map[kLevels] = {};
    int lvl_h[kLevels] = {}, lvl_w[kLevels] = {};
    int cls_pitch = 0, b3d_pitch = 0;
    std::vector<Op> ops;
    void* detect_scratch = nullptr;
    void* nms_scratch = nullptr;
    float* d_K = nullptr;
    int32_t* d_sizes = nullptr;
    Det* d_out = nullptr;
    int32_t* d_counts = nullptr;
    void* d_images = nullptr;
    const float* d_canon = nullptr;
    DecodeParams decode;
    NmsParams nms;
    // sparse FCOS3D predictor (b3d_sparse.cu): the fused box3d conv runs only at the final 2-D candidates, between the two
    // halves of the decode; the dense fp32 maps b3d_map[] then do not exist
    bool sparse_b3d = false;
    float* b3d_rows = nullptr;  // [B][L][topk][b3d_pitch]
    B3dSparseParams b3d_sparse;
    // sparse box3d tower: ops [tower_begin, ops.size()) are the box3d tower convs.  They run after the threshold / top-k half
    // of the decode, in work-list mode on the tiles tower_tiles_kernel lists; every other pixel of their outputs keeps stale
    // workspace contents and is read by nothing.  -1: dense tower.
    int tower_begin = -1;
    TowerTilesParams tower_tiles;
    bool ran = false;  // a forward has run on this plan (the tile counts on the device are valid)
};

void fill_decode_params(DecodeParams* dp, const dd3d_model_desc& desc, int B, int cls_pitch, int b3d_pitch,
                        const float* d_canon);
void fill_nms_params(NmsParams* np, const dd3d_model_desc& desc, const DecodeParams& dp, int B);

class Engine {
   public:
    explicit Engine(const dd3d_model_desc& d);
    ~Engine();
    void load_weight(const char* name, const float* data, const int64_t* shape, int ndim);
    void finalize();
    int size_divisibility() const;
    size_t workspace_bytes(int B, int Hs, int Ws);
    void make_plan(int B, int Hs, int Ws, void* workspace, size_t bytes);
    void forward(const void* d_images, int img_dtype, const float* d_K, const int32_t* d_sizes, Det* d_out,
                 int32_t* d_counts, cudaStream_t stream);
    void forward_host(const void* h_images, int img_dtype, const float* h_K, const int32_t* h_sizes, Det* h_out,
                      int32_t* h_counts, cudaStream_t stream);
    // double-buffered host path: H2D of one slot on a private copy stream while the other slot computes
    void submit_host(int slot, const void* h_images, int img_dtype, const float* h_K, const int32_t* h_sizes, Det* h_out,
                     int32_t* h_counts, cudaStream_t stream);
    void wait_host(int slot);
    // raw dataset images: ResizeShortestEdge + intrinsics rescale (dataset_mapper.py:100-153) fused with the preprocess
    void forward_raw(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes, const float* h_K,
                     int min_size, int max_size, Det* d_out, int32_t* d_counts, float* h_K_out, int32_t* h_new_sizes,
                     cudaStream_t stream);
    // same with caller-chosen output shapes, optional horizontal flips, final intrinsics and (h, w, out_h, out_w) rows:
    // the augmented views of test-time augmentation (test_time_augmentation.py:24-87)
    void forward_resized(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes, const int32_t* h_new_sizes,
                         const int32_t* h_flip, const float* h_K, const int32_t* h_sizes4, Det* d_out, int32_t* d_counts,
                         cudaStream_t stream);
    void drop_plans();  // frees the active and the cached plans (an option that changes the op graph was flipped)
    int launches_per_forward() const;
    // categories: 0 preprocess, 1 stem and depthwise conv, 2 conv (wgmma), 3 pool, 4 eSE, 5 relu and GroupNorm, 6 decode, 7 nms
    void get_profile(double* ms, double* flops, double* bytes, int32_t* launches);
    int get_op_times(float* ms, int32_t* cats, double* flops, int max_ops);

    // layer factories (cached by key)
    const HostTensor& weight(const std::string& name) const;
    const ConvLayer& conv_layer(const std::string& key, const std::vector<std::string>& wnames, int cin, int ksize);
    void bn_fold(const std::string& bn_prefix, const std::string& conv_bias_name, int cout, std::vector<float>* scale,
                 std::vector<float>* bias) const;
    const Epilogue& epilogue(const std::string& key, const std::vector<float>& scale, const std::vector<float>& bias,
                             const std::vector<float>* lo);
    const Epilogue& bn_epilogue(const std::string& key, const std::string& bn_prefix, const std::string& conv_bias_name,
                                int cout);
    const StemLayer& stem_layer(const std::string& wname, const std::string& bn, int ksize, int stride);
    const EseLayer& ese_layer(const std::string& fc, int C);
    const FrontLayer& front_layer(const std::string& prefix);
    const DwLayer& dw_layer(const std::string& wname, int C);
    const Epilogue& gn_affine(const std::string& prefix);  // GroupNorm weight / bias as d_scale / d_bias
    void set_layout(const dd3d_layout_desc& l);

    dd3d_model_desc desc;
    // FPN / head layout (dd3d_set_layout); the default is the shipped one
    dd3d_layout_desc layout = {DD3D_NORM_BN_PER_LEVEL, DD3D_NORM_BN_PER_LEVEL, DD3D_NORM_BN_SHARED, 4, 4, 4, 0};
    int device = 0;
    int num_sms = 132;
    int fp16 = 0;  // desc.act_dtype == DD3D_ACT_FP16: 16-bit storage of activations / weights is fp16 instead of bf16
    bool finalized = false;
    int opt_do_postprocess = 1;
    int opt_profile = 0;
    int opt_workspace_reuse = 1;  // 0: bump allocation, every op output keeps its own memory (stage-level tests / debugging)
    int opt_ese_pool = 0;  // 1: a VoVNet stage's last eSE scale pass also writes the next stage's max-pooled input; 0 (default):
                           // separate pool kernel (the fused pass re-reads each pooling window's inputs 2.25 times)
    int opt_stem_mma = 1;  // 1: VoVNet stem_1 on the register-fragment kernel (stem_mma.cu); 0: wgmma im2col kernel (stem_tc.cu)
    int opt_sparse_box3d = 2;  // box3d predictor at the final candidates only (b3d_sparse.cu): 0 never (dense maps), 1 always, 2 auto (by head size)
    int opt_sparse_tower = 2;  // box3d tower on the tiles the sparse predictor reads (tower_tiles.cu): 0 never, 1 whenever the
                               // sparse predictor runs and the tower norm is not GN, 2 auto (as 1, for heads of >= 50 000 pixels)
    int opt_dla_front = 1;  // 1: DLA-34 base_layer + level0 + level1 (+ pool) as ONE kernel (dla_front.cu); 0: layer by layer
    int opt_workspace_fill = -1;  // >= 0: byte the whole arena is filled with at dd3d_plan (poison test)
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_cat;
    std::vector<int> prof_op;  // plan op that ends at event i, or -1
    size_t prof_used = 0;
    std::string err;
    std::map<std::string, HostTensor> weights;
    std::map<std::string, ConvLayer> convs;
    std::map<std::string, Epilogue> epis;
    std::map<std::string, StemLayer> stems;
    std::map<std::string, EseLayer> eses;
    std::map<std::string, FrontLayer> fronts;
    std::map<std::string, DwLayer> dws;
    std::vector<void*> device_allocs;
    float* d_canon = nullptr;
    Plan plan;
    // inactive engine-owned plans, keyed by (B, Hs, Ws): test-time augmentation cycles through one shape per scale
    // (test_time_augmentation.py:57-64); only small plans are kept (kPlanCacheBytes each, kPlanCacheMax entries)
    std::map<std::array<int, 3>, Plan> plan_cache;
    static constexpr size_t kPlanCacheBytes = size_t(4) << 30;
    static constexpr size_t kPlanCacheMax = 12;
    ResizeTables resize_tables;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t h2d_done[2] = {nullptr, nullptr}, all_done[2] = {nullptr, nullptr};
    bool slot_busy[2] = {false, false};
    struct RawArgs {
        const uint8_t* d_raw;
        int raw_h, raw_w;
        const int32_t* h_raw_sizes;
        const int32_t* h_new_sizes;
        const int32_t* h_flip;
    } raw_args{};
    bool raw_pending = false;  // set by forward_raw for the forward() call it makes

   private:
    void* dev_alloc(size_t bytes);
    float* upload_f32(const std::vector<float>& v);
    size_t build(Plan* P, int B, int Hs, int Ws, void* workspace, bool dry);
    void release_plan();
    static void free_plan(Plan* P);
    std::vector<double> op_flops();
};

}  // namespace dd3d
