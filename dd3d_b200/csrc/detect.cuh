// Detection post-processing: dense threshold + exact per-level top-k + fused 2-D/3-D box decode (decode.cu) and
// per-image class-aware NMS + top-k + rescale (nms.cu).  All fp32, sync-free, deterministic output order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dd3d {

constexpr int kLevels = 5;
constexpr int kNumAttributes = 3;  // MAX_NUM_ATTRIBUTES, tridet/data/datasets/nuscenes/build.py:77
constexpr int kHistBins = 2048;

// Dynamic shared memory of the NMS's one-CTA working set (nms_kernel, nms_finish_kernel; csrc/nms.cu) for `cap` =
// kLevels * PRE_NMS_TOPK candidates: 8192-entry sort keys and payloads + per-candidate box, lists, class and flag.
constexpr int kNmsSortCap = 8192;
constexpr size_t nms_smem_bytes(int cap) { return static_cast<size_t>(kNmsSortCap) * 10 + static_cast<size_t>(cap) * 26; }
// The largest PRE_NMS_TOPK whose working set fits the 227 KiB a block may opt into on sm_90, 1 KiB left for the kernels'
// static shared memory: 1150.  A larger value is refused (DD3D_ERR_INVALID) before any launch.
constexpr int max_pre_nms_topk() {
    int t = kNmsSortCap / kLevels;
    while (nms_smem_bytes(kLevels * t) + 1024 > 227 * 1024) --t;
    return t;
}
constexpr int kMaxPreNmsTopk = max_pre_nms_topk();
static_assert(kMaxPreNmsTopk == 1150, "PRE_NMS_TOPK limit (documented in include/dd3d_b200.h)");
constexpr int kBoundaryCap = 4096;  // candidates sharing the histogram bin of the k-th score (per image x level) that the
                                    // boundary buffer ranks; a fuller bin is ranked by re-reading the level (decode.cu)

// One decoded detection, 24 x 4 bytes.  Also the element type of the C-ABI output buffer (dd3d_det in the header).
struct Det {
    float box[4];      // x1, y1, x2, y2
    float score;       // sqrt(sigmoid(cls) * sigmoid(ctr))                    fcos2d.py:333
    float score3d;     // score * sigmoid(conf)                                fcos3d.py:375-376
    int32_t cls;
    int32_t level;
    float quat[4];     // egocentric, (w, x, y, z)
    float proj_ctr[2];
    float depth;
    float size[3];     // (W, L, H)
    float loc[2];      // feature location (x, y)
    int32_t index;     // pixel * num_classes + class at its level (deterministic tie-break key)
    int32_t attr;      // NuscenesDD3D: argmax of the attribute logits at the pixel (nuscenes_dd3d.py:296), else 0
    float speed;       // NuscenesDD3D: relu(speed conv) at the pixel (nuscenes_dd3d.py:297), else 0
    int32_t pad;
};
static_assert(sizeof(Det) == 96, "Det must be 24 words");

__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

// Axis-aligned IoU of (x1, y1, x2, y2) boxes exactly as torchvision computes it: the 2-D NMS kernels (nms.cu, tta_large.cu)
__device__ __forceinline__ float iou_tv(const float4 a, const float4 b) {
    const float area_a = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float area_b = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
    const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
    const float w = fmaxf(0.f, __fsub_rn(xx2, xx1)), h = fmaxf(0.f, __fsub_rn(yy2, yy1));
    const float inter = __fmul_rn(w, h);
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// The class-only threshold: some class column c < C of a pixel's logits (a 16-byte aligned cls map row) has
// sigmoid(logit) > thresh.  The decode reads a pixel's box2d map row only when this holds: with THRESH_WITH_CTR the
// thresholded score is RN(sigmoid(cls) * sigmoid(ctr)) <= sigmoid(cls), since sigmoid(ctr) <= 1 (or NaN) and rounding is
// monotone.  So the sparse box2d tower (tower_tiles.cu) seeds its tile lists with the pixels this returns true for.
__device__ __forceinline__ bool class_passes(const float* logits, int C, float thresh) {
    bool any = false;
    for (int c0 = 0; c0 < C; c0 += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(logits + c0));
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) any |= c0 + j < C && sigmoidf(vv[j]) > thresh;
    }
    return any;
}

struct DecodeLevel {
    const float* cls;  // [B][H*W][cls_pitch]   logits
    const float* box;  // [B][H*W][16]          0..3 = relu(scale*reg) (l,t,r,b), 4 = centerness logit
    const float* b3d;  // [B][H*W][b3d_pitch]   channel = comp*C + class; comps: quat 0-3, ctr 4-5, depth 6, size 7-9, conf 10
    int H, W, stride;
    int block_begin;   // first block (of the dense kernels' grid.x) that belongs to this level
};

struct DecodeParams {
    DecodeLevel lvl[kLevels];  // positions 0 .. num_levels - 1 (DD3D.IN_FEATURES order)
    int num_levels;            // head levels (1 .. kLevels): the per-(image, level) scratch and the grids follow it
    int B, C, cls_pitch, b3d_pitch;
    int attr_off;       // NuscenesDD3D: channel of the first attribute logit in the cls map (speed follows), else -1
    int num_attr;
    int topk;           // PRE_NMS_TOPK
    float thresh;       // PRE_NMS_THRESH
    int loc_offset_half;  // FEATURE_LOCATIONS_OFFSET == "half"
    int hist_shift;
    uint32_t thresh_bits;
    int total_blocks;
    // 3-D decode constants
    const float* K;       // [B][9] intrinsics (row-major)
    const float* canon;   // [C][3]
    float min_depth, max_depth, depth_factor;
    int scale_depth_by_focal, allocentric, predict_distance;
    int thresh_with_ctr;  // 1: threshold sigmoid(cls) * sigmoid(ctr); 0: threshold sigmoid(cls), rank by the product (fcos2d.py:280-290)
    int C3;               // classes of the 3-D maps: num_classes, or 1 when CLASS_AGNOSTIC_BOX3D (fcos3d.py:333-352)
    int box3d_on;         // 0: no 3-D head (MODEL.BOX3D_ON False): score_3d = score, 3-D fields zero
    // scratch (all per image x level)
    uint32_t* hist;       // [B][L][kHistBins]
    int32_t* sel;         // [B][L][4] : T, n_above, need, total
    int32_t* counters;    // [B][L][2] : sure, boundary
    uint2* sure;          // [B][L][topk]          (score bits, index)
    uint2* boundary;      // [B][L][kBoundaryCap]
    Det* cand;            // [B][L*topk]           decoded candidates (L = num_levels)
    int32_t* cand_count;  // [B][L]
    int32_t* flags;       // [1] overflow word (the decode sets no bit; NMS: bit1)
    uint2* fin;           // [B][L][topk] final candidates (score bits, index): slot order of `cand`
    // sparse 3-D head: the box3d predictor is evaluated only at the final candidates (b3d_sparse.cu); row of candidate `slot`
    // of (image b, level l) = b3d_rows + ((b * L + l) * topk + slot) * b3d_pitch, same channel layout as a dense map pixel
    const float* b3d_rows;  // nullptr: dense maps (lvl[].b3d)
    // 1: b3d_rows come from the class-gathered predictor (b3d_gather.cu): channel q of the candidate's own class at column q,
    // read as if C3 were 1
    int b3d_by_class;
};

struct NmsParams {
    const Det* cand;            // [B][L*topk]
    const int32_t* cand_count;  // [B][L]
    const int32_t* sizes;       // [B][4] : image h, w, output h, w
    Det* out;                   // [B][out_cap]
    int32_t* out_count;         // [B]
    int32_t* flags;             // bit1: output overflow
    int B, topk, out_cap;
    int num_levels;             // L of cand / cand_count: the DecodeParams' num_levels
    int do_nms, post_topk, do_postprocess;
    float nms_thresh;
    void* scratch;    // nms_scratch_bytes(B, topk, num_classes) bytes, or nullptr (single-CTA kernel only)
    int num_classes;
    // 1: the multi-CTA path (sort / IoU bit matrix on all SMs / one scan CTA per (class, image) / finish), 0: one CTA per
    // image does the whole NMS.  Chosen once with nms_class_parallel() by whoever fills the params.
    int class_parallel;
};

size_t decode_scratch_bytes(int B, int topk, int num_levels = kLevels);
void decode_bind_scratch(DecodeParams* p, void* scratch);
void decode_finalize_params(DecodeParams* p);
cudaError_t launch_decode(const DecodeParams& p, cudaStream_t stream);  // = select + final
// the two halves: threshold / top-k / final candidate list (fin, cand_count), then the per-candidate 2-D + 3-D decode;
// the sparse box3d predictor runs between them
constexpr int kDecodeSelectLaunches = 5;  // clear, dense pass, select, dense pass, final select
constexpr int kDecodeFinalLaunches = 1;
cudaError_t launch_decode_select(const DecodeParams& p, cudaStream_t stream);
cudaError_t launch_decode_final(const DecodeParams& p, cudaStream_t stream);
cudaError_t launch_nms(const NmsParams& p, cudaStream_t stream);  // the path p.class_parallel names
int nms_launches(const NmsParams& p);
size_t nms_scratch_bytes(int B, int topk, int num_classes, int num_levels = kLevels);
void nms_set_class_parallel(int mode);  // 0 single-CTA kernel, 1 multi-CTA path, -1 environment / default (1)
// The NMS path for params whose other fields are filled: the multi-CTA one when the policy above allows it, the params
// have its scratch, there is something to suppress (do_nms, nms_thresh > 0) and 1 <= num_classes <= 255.
int nms_class_parallel(const NmsParams& p);
// BEV rotated NMS of DD3D.forward (DO_BEV_NMS, core.py:137-151).  The one-CTA kernel (launch_bev_nms) holds kBevNmsMax
// boxes per image and relies on them arriving sorted by scores_3d: the output of the 2-D NMS with 0 < POST_NMS_TOPK <=
// kBevNmsMax.  Every other configuration -- DO_NMS off (all 5 * PRE_NMS_TOPK candidates, level-major) or POST_NMS_TOPK
// outside 1..kBevNmsMax (every 2-D NMS survivor) -- takes the multi-CTA path (launch_image_bev_nms), which sorts itself.
constexpr int kBevNmsMax = 256;
constexpr int kBevPathOneCta = 1, kBevPathMultiCta = 2;
inline int bev_nms_path(int do_nms, int post_nms_topk) {
    return (do_nms && post_nms_topk > 0 && post_nms_topk <= kBevNmsMax) ? kBevPathOneCta : kBevPathMultiCta;
}
// BEV rotated NMS on the (already 2-D-NMSed, score-sorted) detections, in place; poses: [B][7] (w,x,y,z, tx,ty,tz).
cudaError_t launch_bev_nms(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* sizes,
                           int32_t* flags, int B, int cap, float thr, int do_postprocess, cudaStream_t stream);
// out[i] = rotated IoU of rectangles a[i], b[i] ((cx, cy, w, h, angle_deg) rows), the function the BEV kernels threshold.
cudaError_t launch_rotated_iou(const float* a, const float* b, int n, float* out, cudaStream_t stream);

// Test-time-augmentation merge (tta.cu): the views' detections back to the original image + one merged NMS.
constexpr int kTtaMaxViews = 16;
constexpr int kTtaMergedMax = 1024;  // merged detections the single NMS pass holds (10 views x POST_NMS_TOPK 100 fit)
struct TtaView {       // one augmented view = ResizeShortestEdge scale (+ horizontal flip); mirrors dd3d_tta_view
    int32_t flip;      // HFlipTransform applied after the resize
    float view_w;      // width of the view (flip axis)
    float inv_sx[2];   // fp32 x factors of the inverse resizes, applied in this order: view -> input, input -> original
    float inv_sy[2];
    float K_view[9];   // intrinsics the view was run with
    float K_orig[9];   // inverse transforms applied to K_view = the original camera (re-projection of tvec)
};
int tta_merged_cap(int A, int cap);  // slots of the merged output buffer: min(A * cap, kTtaMergedMax)
size_t tta_scratch_bytes(int A, int cap);
cudaError_t launch_tta_merge(const Det* dets, const int32_t* counts, const TtaView* h_views, int A, int cap,
                             float nms_thresh, int do_nms, void* scratch, Det* out, int32_t* out_count, int32_t* flags,
                             cudaStream_t stream);

// The same merge for large sets (tta_large.cu): no kTtaMergedMax clamp, A * cap merged slots (cap <= kLevels *
// kMaxPreNmsTopk, so up to 92 000 per image), multi-CTA transform, blocked class-aware NMS with O(A * cap) scratch; -1 /
// 0 bytes / cudaErrorInvalidValue for arguments out of range.
int tta_merged_cap_large(int A, int cap);
size_t tta_large_scratch_bytes(int A, int cap);
cudaError_t launch_tta_merge_large(const Det* dets, const int32_t* counts, const TtaView* h_views, int A, int cap,
                                   float nms_thresh, int do_nms, void* scratch, Det* out, int32_t* out_count,
                                   int32_t* flags, cudaStream_t stream);

// NuscenesDD3D sample aggregation: BEV rotated NMS jointly over the images of each sample group, then the cap on the
// survivors of the call; in place; global: [B][cap][10] pred_boxes3d_global rows; cap <= 256.
size_t sample_aggregate_scratch_bytes(int B, int cap);
cudaError_t launch_sample_aggregate(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* group,
                                    int num_groups, float* global, void* scratch, int32_t* flags, int B, int cap,
                                    float thr, int max_dets, cudaStream_t stream);

// Grouped rotated BEV NMS for large sets (bev_nms_group.cu): B <= 256 images of cap <= 1024 slots, groups of
// <= max_group_images <= 16 images; view_K [B][num_views][9] indexed by Det::level; pose_mode 0: global (poses [B][7]),
// 1: camera (CAMERA_TO_VEHICLE_ROTATION); global (or nullptr): [B][cap][10]; max_dets <= 0: no cap.
// Image mode of the same kernels: the per-image BEV NMS of DD3D.forward on up to kLevels * kMaxPreNmsTopk unsorted boxes
// per image (each image its own group, its own K [B][9] and pose [B][7], no cap); then detector_postprocess when sizes
// ([B][4]) is not null.  Any B (chunks of 256 images share the scratch); flags bit 6 (64): a count above cap.  num_classes
// (1..128) sizes the per-group class table and the scan grid: 64 class segments up to 64 classes, 128 above.
// The grouped mode (launch_group_bev_nms) always has 128 class segments: class ids 0..127.
size_t image_bev_nms_scratch_bytes(int B, int cap, int num_classes);
cudaError_t launch_image_bev_nms(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* sizes,
                                 void* scratch, int32_t* flags, int B, int cap, float thr, int num_classes,
                                 cudaStream_t stream);
int image_bev_nms_launches(int B);
size_t group_bev_nms_scratch_bytes(int B, int cap, int max_group_images);
cudaError_t launch_group_bev_nms(Det* dets, int32_t* counts, const float* view_K, int num_views, const float* poses,
                                 int pose_mode, const int32_t* group, int num_groups, int max_group_images, float* global,
                                 void* scratch, int32_t* flags, int B, int cap, float thr, int max_dets,
                                 cudaStream_t stream);

// launch_group_bev_nms on the blocked NMS of tta_large.cu: the same arguments, outputs and flags for cap <= 92 000 slots
// per image, scratch O(B * cap) (0 bytes: arguments out of range).
size_t group_bev_nms_large_scratch_bytes(int B, int cap, int max_group_images);
cudaError_t launch_group_bev_nms_large(Det* dets, int32_t* counts, const float* view_K, int num_views, const float* poses,
                                       int pose_mode, const int32_t* group, int num_groups, int max_group_images,
                                       float* global, void* scratch, int32_t* flags, int B, int cap, float thr,
                                       int max_dets, cudaStream_t stream);
// Kernels launch_group_bev_nms_large enqueues for these arguments (the radix sort's pass count follows num_groups).
int group_bev_nms_large_launches(int num_groups);
constexpr int kGroupBevNmsLargeMaxB = 256;          // images per call of launch_group_bev_nms_large
constexpr int kGroupBevNmsLargeGroupImages = 16;    // images per group it holds

// NuscenesDD3D sample aggregation as a step of the forward (Engine::set_sample_aggregate).  The one-CTA pair of
// launch_sample_aggregate holds kSampleAggOneCtaTopk boxes of each of 6 cameras (its 768-box group) and out_cap <=
// kBevNmsMax slots: the 2-D NMS output with 0 < POST_NMS_TOPK <= 128.  Every other configuration -- DO_NMS off (all
// L * PRE_NMS_TOPK candidates per image) or a larger top-k -- runs the blocked kernels of launch_group_bev_nms_large in
// global pose mode, up to 6 * 5 * 1150 = 34 500 boxes per sample.
constexpr int kSampleAggOneCtaTopk = 128;
constexpr int kAggPathOneCta = 1, kAggPathBlocked = 2;
inline int sample_aggregate_path(int do_nms, int post_nms_topk, int out_cap) {
    return (do_nms && post_nms_topk > 0 && post_nms_topk <= kSampleAggOneCtaTopk && out_cap <= kBevNmsMax) ? kAggPathOneCta
                                                                                                       : kAggPathBlocked;
}
constexpr int kSampleAggOneCtaLaunches = 2;  // sample_nms_kernel + sample_compact_kernel

}  // namespace dd3d
