// Detection post-processing: dense threshold + exact per-level top-k + fused 2-D/3-D box decode (decode.cu) and
// per-image class-aware NMS + top-k + rescale (nms.cu).  All fp32, sync-free, deterministic output order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dd3d {

constexpr int kLevels = 5;
constexpr int kNumAttributes = 3;  // MAX_NUM_ATTRIBUTES, tridet/data/datasets/nuscenes/build.py:77
constexpr int kHistBins = 2048;
constexpr int kBoundaryCap = 4096;  // candidates sharing the histogram bin of the k-th score (per image x level)

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

struct DecodeLevel {
    const float* cls;  // [B][H*W][cls_pitch]   logits
    const float* box;  // [B][H*W][16]          0..3 = relu(scale*reg) (l,t,r,b), 4 = centerness logit
    const float* b3d;  // [B][H*W][b3d_pitch]   channel = comp*C + class; comps: quat 0-3, ctr 4-5, depth 6, size 7-9, conf 10
    int H, W, stride;
    int block_begin;   // first block (of the dense kernels' grid.x) that belongs to this level
};

struct DecodeParams {
    DecodeLevel lvl[kLevels];
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
    Det* cand;            // [B][L*topk]           decoded candidates
    int32_t* cand_count;  // [B][L]
    int32_t* flags;       // [1] bit0: boundary overflow
    uint2* fin;           // [B][L][topk] final candidates (score bits, index): slot order of `cand`
    // sparse 3-D head: the box3d predictor is evaluated only at the final candidates (b3d_sparse.cu); row of candidate `slot`
    // of (image b, level l) = b3d_rows + ((b * L + l) * topk + slot) * b3d_pitch, same channel layout as a dense map pixel
    const float* b3d_rows;  // nullptr: dense maps (lvl[].b3d)
};

struct NmsParams {
    const Det* cand;            // [B][L*topk]
    const int32_t* cand_count;  // [B][L]
    const int32_t* sizes;       // [B][4] : image h, w, output h, w
    Det* out;                   // [B][out_cap]
    int32_t* out_count;         // [B]
    int32_t* flags;             // bit1: output overflow
    int B, topk, out_cap;
    int do_nms, post_topk, do_postprocess;
    float nms_thresh;
    void* scratch;    // nms_scratch_bytes(B, topk, num_classes) bytes, or nullptr: single-CTA kernel (one CTA per image)
    int num_classes;  // with scratch: IoU bit matrix on all SMs + one scan CTA per (class, image)
};

size_t decode_scratch_bytes(int B, int topk);
void decode_bind_scratch(DecodeParams* p, void* scratch);
void decode_finalize_params(DecodeParams* p);
cudaError_t launch_decode(const DecodeParams& p, cudaStream_t stream);  // = select + final
// the two halves: threshold / top-k / final candidate list (fin, cand_count), then the per-candidate 2-D + 3-D decode;
// the sparse box3d predictor runs between them
cudaError_t launch_decode_select(const DecodeParams& p, cudaStream_t stream);
cudaError_t launch_decode_final(const DecodeParams& p, cudaStream_t stream);
cudaError_t launch_nms(const NmsParams& p, cudaStream_t stream);
size_t nms_scratch_bytes(int B, int topk, int num_classes);
void nms_set_class_parallel(int mode);  // 0 single-CTA kernel, 1 multi-CTA path (sort / IoU bit matrix / scan / finish), -1 environment / default (1)
// BEV rotated NMS on the (already 2-D-NMSed, score-sorted) detections, in place; poses: [B][7] (w,x,y,z, tx,ty,tz).
cudaError_t launch_bev_nms(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* sizes,
                           int32_t* flags, int B, int cap, float thr, int do_postprocess, cudaStream_t stream);

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

// NuscenesDD3D sample aggregation: BEV rotated NMS jointly over the images of each sample group, then the cap on the
// survivors of the call; in place; global: [B][cap][10] pred_boxes3d_global rows; cap <= 256.
size_t sample_aggregate_scratch_bytes(int B, int cap);
cudaError_t launch_sample_aggregate(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* group,
                                    int num_groups, float* global, void* scratch, int32_t* flags, int B, int cap,
                                    float thr, int max_dets, cudaStream_t stream);

// Grouped rotated BEV NMS for large sets (bev_nms_group.cu): B <= 256 images of cap <= 1024 slots, groups of
// <= max_group_images <= 16 images; view_K [B][num_views][9] indexed by Det::level; pose_mode 0: global (poses [B][7]),
// 1: camera (CAMERA_TO_VEHICLE_ROTATION); global (or nullptr): [B][cap][10]; max_dets <= 0: no cap.
size_t group_bev_nms_scratch_bytes(int B, int cap, int max_group_images);
cudaError_t launch_group_bev_nms(Det* dets, int32_t* counts, const float* view_K, int num_views, const float* poses,
                                 int pose_mode, const int32_t* group, int num_groups, int max_group_images, float* global,
                                 void* scratch, int32_t* flags, int B, int cap, float thr, int max_dets,
                                 cudaStream_t stream);

}  // namespace dd3d
