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

constexpr int kFpnMaxOutputs = DD3D_FPN_MAX_OUTPUTS;  // FPN outputs (p<first> .. P6 / P7); the heads run at most kLevels

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
    int groups = 1;  // > 1: grouped 3x3 packed block-diagonally for ConvParams::grouped (Engine::grouped_conv_layer)
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
struct StemLayer {  // VoVNet stem_1 (3x3 / stride 2, 3 -> 64) packed for stem_mma.cu
    __nv_bfloat16* d_w;  // [64][3][4][4]
    float* d_sb;         // scale[64] | bias[64]
    bool relu = true;    // false: raw output (VoVNet stem_1 in front of its GroupNorm)
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

// One DLA network the engine builds (reference DLA_NAME_TO_BUILDER, dla.py:358-441); the table is in engine.cu
struct DlaSpec {
    int arch;  // dd3d_arch
    int levels[6];
    int channels[6];
    bool bottleneck_x;   // BottleneckX blocks (dla.py:104-143) instead of BasicBlock (dla.py:24-62)
    bool root_residual;  // Root adds its first child before the ReLU (dla.py:160-167)
    int cardinality;     // BottleneckX groups; its bottleneck width is planes * cardinality / 32
};
const DlaSpec* dla_spec(int arch);  // nullptr: not a DLA arch

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

// One step of the forward = one profile event (Engine::plan_steps).  The forward launches the steps in order; the launch
// count and the profile are sums over them.
struct Step {
    enum Kind {
        PREPROCESS,   // caller images or the raw-image resize -> padded input
        OP,           // plan op `op`
        BOX2D_TILES,  // sparse box2d tower: seeds (pixels passing the class-only threshold) + tile lists
        BOX3D_TILES,  // sparse box3d tower: decode threshold / top-k + tile lists around the final candidates
        DETECT,       // [decode threshold / top-k] [sparse or gathered box3d predictor] decode of the final candidates
        NMS,          // NMS [+ BEV NMS]
        AGGREGATE,    // NuscenesDD3D sample aggregation over the call's images (after detector_postprocess)
    } kind;
    int op = -1;        // OP: index into Plan::ops, else -1
    int cat = 0;        // profile category (Engine::get_profile)
    int launches = 0;   // kernels the step enqueues
    double bytes = 0.0;  // algorithmic HBM bytes of a non-op step (an op's are Op::bytes)
    bool select = false;  // DETECT: the threshold / top-k half runs here (no BOX3D_TILES step ran it)
    int b3d = 0;          // DETECT: box3d predictor at the final candidates: 0 none (dense maps), kB3dSparse, kB3dGathered
    int bev = 0;          // NMS: 0, or the bev_nms_path() of the BEV NMS that follows
    int agg = 0;          // AGGREGATE: the sample_aggregate_path() it runs
    static constexpr int kB3dSparse = 1, kB3dGathered = 2;
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
    float* s1_poses = nullptr;  // BEV NMS or sample aggregation on: slot 1's copy of the host poses
    int32_t* s1_group = nullptr;  // sample aggregation on: slot 1's copy of the host group indices
    float* s1_global = nullptr;   // and its pred_boxes3d_global rows [B][out_cap][10]
    View input;
    View fpn[kFpnMaxOutputs];  // by FPN output index; an output no head reads is not built (null ptr)
    int num_levels = kLevels;  // head positions; the per-level arrays below are by position
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
    // BEV NMS as the last op of the forward (dd3d_set_bev_nms): 0 off, else bev_nms_path() of the config at plan time
    int bev = 0;
    float* d_poses = nullptr;      // [B][7] staging of the host poses (host paths, slot 0)
    void* bev_scratch = nullptr;   // image_bev_nms_scratch_bytes(B, out_cap, num_classes) (multi-CTA path only)
    // sample aggregation as the last step (dd3d_set_sample_aggregate): 0 off, else sample_aggregate_path() at plan time
    int agg = 0;
    int32_t* d_group = nullptr;   // [B] staging of the host group indices (host paths, slot 0)
    float* d_global = nullptr;    // [B][out_cap][10] pred_boxes3d_global staging (host paths, slot 0)
    void* agg_scratch = nullptr;  // sample_aggregate_scratch_bytes / group_bev_nms_large_scratch_bytes of the path
    // sparse FCOS3D predictor (b3d_sparse.cu): the fused box3d conv runs only at the final 2-D candidates, between the two
    // halves of the decode; the dense fp32 maps b3d_map[] then do not exist
    bool sparse_b3d = false;
    float* b3d_rows = nullptr;  // [B][L][topk][b3d_pitch]
    B3dSparseParams b3d_sparse;
    // class-gathered sparse predictor (b3d_gather.cu), for class-specific heads whose 11 C outputs exceed kB3dSparseMaxN: rows
    // [B][L][topk][kB3dGatherPitch] in b3d_rows, same place in the forward as the sparse predictor (sparse_b3d is also set)
    bool gather_b3d = false;
    B3dGatherParams b3d_gather;
    void* b3d_gather_scratch = nullptr;  // b3d_gather_scratch_bytes(B, C, topk): the class grouping
    // sparse box3d tower: ops [tower_begin, ops.size()) are the box3d tower convs.  They run after the threshold / top-k half
    // of the decode, in work-list mode on the tiles tower_tiles_kernel lists; every other pixel of their outputs keeps stale
    // workspace contents and is read by nothing.  -1: dense tower.
    int tower_begin = -1;
    TowerTilesParams tower_tiles;
    // sparse box2d tower: ops [box2d_begin, box2d_begin + depth) are the box2d tower convs and its predictor (depth = tower
    // convs + 1), in work-list mode on the tiles the class-only threshold needs (box2d_tiles, seeded by tower_mark_kernel
    // right before them); the box map holds stale workspace contents outside those tiles.  -1: dense.
    int box2d_begin = -1;
    TowerTilesParams box2d_tiles;
    std::vector<Step> steps;  // what a forward of this plan launches, in order
    bool ran = false;  // a forward has run on this plan (the tile counts on the device are valid)
};

void fill_decode_params(DecodeParams* dp, const dd3d_model_desc& desc, int B, int cls_pitch, int b3d_pitch,
                        const float* d_canon, int num_levels = kLevels);
void fill_nms_params(NmsParams* np, const dd3d_model_desc& desc, const DecodeParams& dp, int B, void* scratch);

class Engine {
   public:
    explicit Engine(const dd3d_model_desc& d);
    ~Engine();
    void load_weight(const char* name, const float* data, const int64_t* shape, int ndim);
    void finalize();
    int size_divisibility() const;
    size_t workspace_bytes(int B, int Hs, int Ws);
    void make_plan(int B, int Hs, int Ws, void* workspace, size_t bytes);
    struct RawArgs {  // raw dataset images the preprocess resizes (forward_resized)
        const uint8_t* d_raw;
        int raw_h, raw_w;
        const int32_t* h_raw_sizes;
        const int32_t* h_new_sizes;
        const int32_t* h_flip;
    };
    // d_poses: [B][7] poses the BEV NMS reads (unused when it is off); the preprocess reads `raw` when given, else d_images
    // sample aggregation operands: [B] group indices of num_groups groups, [B][out_cap][10] pred_boxes3d_global rows
    struct AggArgs {
        const int32_t* d_group;
        int num_groups;
        float* d_global;
    };
    void forward(const void* d_images, int img_dtype, const float* d_K, const int32_t* d_sizes, Det* d_out,
                 int32_t* d_counts, const float* d_poses, const AggArgs& agg, cudaStream_t stream,
                 const RawArgs* raw = nullptr);
    // One forward of the current plan recorded by stream capture and instantiated (dd3d_graph_create): the launches of
    // forward() with the device poses / groups / global rows and the options as they are now
    struct CapturedForward {
        cudaGraphExec_t exec = nullptr;
        int kernel_nodes = 0;
        int programmatic_edges = 0;  // edges the PDL launch attribute became
    };
    CapturedForward capture_forward(const void* d_images, int img_dtype, const float* d_K, const int32_t* d_sizes,
                                    Det* d_out, int32_t* d_counts, cudaStream_t stream);
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
    void set_do_nms(int do_nms);  // DO_NMS at run time: the plans' NMS steps follow it
    int launches_per_forward() const;
    // BEV NMS (DO_BEV_NMS): on / off and its IoU threshold; the poses of dd3d_forward / dd3d_forward_raw (device) and of
    // the host paths (copied per slot)
    void set_bev_nms(int enable, float thr);
    int bev_mode() const;  // 0 off, else the bev_nms_path() the current options select
    void set_host_poses(int slot, const float* h_poses);
    // NuscenesDD3D sample aggregation (dd3d_set_sample_aggregate) as the last step of every forward; its group indices and
    // global rows: device (dd3d_set_groups / dd3d_set_global_out) and per host slot (dd3d_set_host_groups /
    // dd3d_set_host_global_out)
    void set_sample_aggregate(int enable, float thr, int max_dets);
    int agg_mode() const;  // 0 off, else the sample_aggregate_path() the current options select
    void set_host_groups(int slot, const int32_t* h_group, int num_groups);
    AggArgs device_agg_args() const { return {user_groups, user_num_groups, user_global}; }
    // categories: 0 preprocess, 1 stem and depthwise conv, 2 conv (wgmma), 3 pool, 4 eSE, 5 relu and GroupNorm, 6 decode, 7 nms
    void get_profile(double* ms, double* flops, double* bytes, int32_t* launches);
    int get_op_times(float* ms, int32_t* cats, double* flops, int32_t* ops, int max_ops);  // ops may be null

    // layer factories (cached by key)
    const HostTensor& weight(const std::string& name) const;
    const ConvLayer& conv_layer(const std::string& key, const std::vector<std::string>& wnames, int cin, int ksize);
    void bn_fold(const std::string& bn_prefix, const std::string& conv_bias_name, int cout, std::vector<float>* scale,
                 std::vector<float>* bias) const;
    const Epilogue& epilogue(const std::string& key, const std::vector<float>& scale, const std::vector<float>& bias,
                             const std::vector<float>* lo);
    const Epilogue& bn_epilogue(const std::string& key, const std::string& bn_prefix, const std::string& conv_bias_name,
                                int cout);
    const StemLayer& stem_layer(const std::string& wname, const std::string& bn, const std::string& conv_bias_name, bool relu);
    const EseLayer& ese_layer(const std::string& fc, int C);
    const FrontLayer& front_layer(const std::string& prefix);
    const DwLayer& dw_layer(const std::string& wname, int C);
    const ConvLayer& grouped_conv_layer(const std::string& wname, int C, int groups);  // (C, C / groups, 3, 3) weights
    const Epilogue& gn_affine(const std::string& prefix, int C = kGnChannels);  // GroupNorm weight / bias as d_scale / d_bias
    void set_layout(const dd3d_layout_desc& l);
    void set_backbone_norm(int norm);
    void set_fpn_channels(int C);
    void set_canonical_sizes(int num_classes, const float* sizes);
    void set_fpn_inputs(const int32_t* inputs, int n);
    void set_in_features(const int32_t* fpn_levels, int n);
    std::vector<int> fpn_input_list() const;  // FE.FPN.IN_FEATURES as dd3d_set_fpn_inputs numbers (the default when unset)
    int fpn_first_stage() const;  // log2 of the stride of FPN output 0
    int fpn_outputs() const;      // inputs + the top block's P6 (VoVNet) or P6 and P7 (DLA): 2 .. kFpnMaxOutputs
    int num_levels() const { return in_features.empty() ? fpn_outputs() : static_cast<int>(in_features.size()); }
    int head_level(int l) const { return in_features.empty() ? l : in_features[l]; }  // FPN output read at position l

    dd3d_model_desc desc;
    // FCOS3D.CANONICAL_BOX3D_SIZES rows 0..num_classes-1 (dd3d_set_canonical_sizes); empty: the desc's rows (num_classes <= 16)
    std::vector<float> canonical_sizes;
    // FE.FPN.IN_FEATURES (dd3d_set_fpn_inputs): backbone outputs feeding the FPN, stride-contiguous and ending at stride 32;
    // empty: the builder's default (DLA level3..5, VoVNet stage2..5)
    std::vector<int> fpn_inputs;
    // DD3D.IN_FEATURES (dd3d_set_in_features): the FPN output each head position reads, distinct; empty: every FPN output in
    // order.  Per-level BN, Scale / Offset and PER_LEVEL_PREDICTORS predictors are taken by position.
    std::vector<int> in_features;
    // FPN / head layout (dd3d_set_layout); the default is the shipped one
    dd3d_layout_desc layout = {DD3D_NORM_BN_PER_LEVEL, DD3D_NORM_BN_PER_LEVEL, DD3D_NORM_BN_SHARED, 4, 4, 4, 0};
    // FE.BACKBONE.NORM (dd3d_set_backbone_norm): BN folded into the conv epilogues (default), DD3D_NORM_NONE (DLA-34: conv bias)
    // or DD3D_NORM_GN (VoVNet: raw conv outputs, each normalised by a GroupNorm op)
    int backbone_norm = DD3D_NORM_BN_SHARED;
    // FE.FPN.OUT_CHANNELS (dd3d_set_fpn_channels): width of the FPN outputs, the head towers and the predictors' input; a
    // multiple of 64 in [64, 512]
    int fpn_channels = 256;
    int device = 0;
    int num_sms = 132;
    int fp16 = 0;  // desc.act_dtype == DD3D_ACT_FP16: 16-bit storage of activations / weights is fp16 instead of bf16
    bool finalized = false;
    // Bumped by every dd3d_plan, every plan drop and every dd3d_set_* call a forward reads (options, BEV NMS, poses, sample
    // aggregation, groups, global rows): a captured forward is current while the counter still has its capture-time value
    uint64_t generation = 0;
    int opt_do_postprocess = 1;
    int opt_profile = 0;
    int opt_workspace_reuse = 1;  // 0: bump allocation, every op output keeps its own memory (stage-level tests / debugging)
    int opt_sparse_box3d = 2;  // box3d predictor at the final candidates only (b3d_sparse.cu): 0 never (dense maps), 1 always, 2 auto (by head size)
    int opt_sparse_tower = 2;  // box3d tower on the tiles the sparse predictor reads (tower_tiles.cu): 0 never, 1 whenever the
                               // sparse predictor runs and the tower norm is not GN, 2 auto (as 1, for heads of >= 50 000 pixels)
    int opt_sparse_box2d_tower = 2;  // box2d tower + predictor on the tiles around the pixels whose class score passes the
                                     // threshold (tower_tiles.cu): 0 never, 1 whenever the tower norm is not GN and the tower
                                     // convs use the pair tile, 2 auto (as 1, with the sparse box3d predictor and heads of
                                     // >= 50 000 pixels)
    int opt_workspace_fill = -1;  // >= 0: byte the whole arena is filled with at dd3d_plan (poison test)
    int opt_bev_nms = 0;
    float bev_nms_thresh = 0.f;
    const float* user_poses = nullptr;   // dd3d_set_poses
    std::vector<float> host_poses[2];    // dd3d_set_host_poses, per slot
    int opt_sample_agg = 0;
    float agg_thresh = 0.f;
    int agg_max_dets = 0;                 // <= 0: no cap
    const int32_t* user_groups = nullptr;  // dd3d_set_groups
    int user_num_groups = 0;
    float* user_global = nullptr;          // dd3d_set_global_out
    std::vector<int32_t> host_groups[2];   // dd3d_set_host_groups, per slot
    int host_num_groups[2] = {0, 0};
    float* host_global[2] = {nullptr, nullptr};  // dd3d_set_host_global_out, per slot
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

   private:
    void launch_op(const Op& op, cudaStream_t stream);
    void* dev_alloc(size_t bytes);
    float* upload_f32(const std::vector<float>& v);
    size_t build(Plan* P, int B, int Hs, int Ws, void* workspace, bool dry);
    void plan_steps(Plan* P);  // the NMS params and the step list of a built plan
    void check_host_agg(int slot) const;
    void release_plan();
    static void free_plan(Plan* P);
    std::vector<double> op_flops();
};

}  // namespace dd3d
