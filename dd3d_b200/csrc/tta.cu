// Test-time-augmentation merge on the device (SURVEY.md 8f row 4).
//
// Replaces DD3DWithTTA._get_augmented_instances step 2 and the merged NMS of _inference_one_image
// (tridet/modeling/dd3d/test_time_augmentation.py:190-239 and :160-171): for every augmented view (one ResizeShortestEdge
// scale, optionally followed by a horizontal flip) the detections are mapped back to the original image --
//   2-D boxes   TransformList.inverse().apply_box: un-flip (x -> W_aug - x), un-resize, un-resize of the mapper's own
//               resize; fp32 at every step like the numpy code;
//   3-D boxes   apply_hflip_box3d (tridet/data/augmentations/flip_transform.py:28-55) on (quat, tvec): quat ->
//               (z, -y, -x, w) of (w, x, y, z), tvec.x -> -tvec.x; resizes leave 3-D boxes alone;
//   intrinsics  the inverse transforms applied to the view's intrinsics give the original camera, through which
//               Boxes3D.from_vectors (tridet/structures/boxes3d.py:176-216) re-projects tvec to (proj_ctr, depth) --
// then concatenated in view order and reduced by ONE class-aware NMS on scores_3d (detectron2 batched_nms), output in
// descending scores_3d order (merged_instances[keep]).
#include "tta_view.cuh"

#include <string.h>

namespace dd3d {

namespace {

constexpr int kTtaThreads = 256;

struct TtaParams {
    const Det* dets;         // [A][cap] detections of the views (engine output, do_postprocess = 0)
    const int32_t* counts;   // [A]
    TtaView view[kTtaMaxViews];
    Det* cand;               // [>= A * cap] merged candidates (NMS input)
    int32_t* cand_count;     // [kLevels] : total, 0, 0, 0, 0
    int32_t* flags;          // bit 4: more merged detections than merged_cap
    int A, cap, merged_cap;
};

__global__ void __launch_bounds__(kTtaThreads) tta_merge_kernel(const TtaParams p) {
    __shared__ int s_off[kTtaMaxViews + 1];
    if (threadIdx.x == 0) {
        int off = 0;
        for (int a = 0; a < p.A; ++a) {
            s_off[a] = off;
            off += min(p.counts[a], p.cap);
            if (off > p.merged_cap) {
                atomicOr(p.flags, 16);
                off = p.merged_cap;
            }
        }
        s_off[p.A] = off;
        p.cand_count[0] = off;
        for (int l = 1; l < kLevels; ++l) p.cand_count[l] = 0;
    }
    __syncthreads();
    for (int a = 0; a < p.A; ++a) {
        const TtaView& V = p.view[a];
        const int n = s_off[a + 1] - s_off[a];
        float iK[9];
        tta_inv3(V.K_view, iK);
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            Det d = p.dets[static_cast<size_t>(a) * p.cap + i];
            tta_invert_det(d, V, iK, a);
            p.cand[s_off[a] + i] = d;
        }
    }
}

}  // namespace

int tta_merged_cap(int A, int cap) { return A * cap < kTtaMergedMax ? A * cap : kTtaMergedMax; }

size_t tta_scratch_bytes(int A, int cap) { return static_cast<size_t>(tta_merged_cap(A, cap)) * sizeof(Det) + 256; }

cudaError_t launch_tta_merge(const Det* dets, const int32_t* counts, const TtaView* h_views, int A, int cap,
                             float nms_thresh, int do_nms, void* scratch, Det* out, int32_t* out_count, int32_t* flags,
                             cudaStream_t stream) {
    if (A < 1 || A > kTtaMaxViews || cap < 1) return cudaErrorInvalidValue;
    const int total = tta_merged_cap(A, cap);
    TtaParams p;
    p.dets = dets;
    p.counts = counts;
    for (int a = 0; a < A; ++a) p.view[a] = h_views[a];
    p.cand = static_cast<Det*>(scratch);
    p.cand_count = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(scratch) + static_cast<size_t>(total) * sizeof(Det));
    p.flags = flags;
    p.A = A;
    p.cap = cap;
    p.merged_cap = total;
    tta_merge_kernel<<<1, kTtaThreads, 0, stream>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // one class-aware NMS over the merged set (all candidates sit in "level 0" of the NMS kernel's layout); no top-k,
    // no rescale: test_time_augmentation.py:163-171
    NmsParams np;
    memset(&np, 0, sizeof(np));  // scratch = nullptr: single-CTA kernel (one merged set)
    np.cand = p.cand;
    np.cand_count = p.cand_count;
    np.sizes = p.cand_count;  // read but unused without do_postprocess
    np.out = out;
    np.out_count = out_count;
    np.flags = flags;
    np.B = 1;
    np.num_levels = kLevels;
    np.topk = total;
    np.out_cap = total;
    np.do_nms = do_nms;
    np.post_topk = 0;
    np.do_postprocess = 0;
    np.nms_thresh = nms_thresh;
    return launch_nms(np, stream);
}

}  // namespace dd3d
