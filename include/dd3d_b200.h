/*
 * dd3d_b200 -- C ABI of the H100-native (sm_90a) DD3D inference path.
 *
 * Drop-in boundary for ONE reference call: the eval-mode DD3D.forward()
 *   /root/reference/tridet/modeling/dd3d/core.py:64-164
 * (backbone + FPN: feature_extractor/dla.py:346-355, vovnet.py:357-367, detectron2 FPN; heads: fcos2d.py:130-156,
 * fcos3d.py:160-188; decode: fcos2d.py:270-344, fcos3d.py:328-399; NMS/top-k: fcos2d.py:346-367; rescale:
 * detectron2 detector_postprocess, core.py:153-160).  The Python mirror of the meta-arch
 * (dd3d_b200/meta_arch.py::DD3DB200) binds these symbols with ctypes and keeps the reference's
 * forward(batched_inputs) -> [{"instances": Instances}] contract; see INTEGRATION.md.
 *
 * Conventions: every function returns 0 on success or a negative dd3d_status; dd3d_last_error() gives the text.
 * Pointers prefixed d_ are device pointers, h_ host pointers.  A handle is bound to the CUDA device that was
 * current at dd3d_create and is not thread-safe.  There is no CPU fallback: without a CUDA device every entry
 * point that needs one fails with DD3D_ERR_CUDA.
 */
#ifndef DD3D_B200_H_
#define DD3D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dd3d_engine* dd3d_handle;
typedef void* dd3d_stream; /* cudaStream_t */

enum dd3d_status {
    DD3D_OK = 0,
    DD3D_ERR_INVALID = -1,  /* bad argument / unknown weight name / shape mismatch */
    DD3D_ERR_STATE = -2,    /* call order (e.g. forward before finalize) */
    DD3D_ERR_CUDA = -3,     /* CUDA runtime / driver error */
    DD3D_ERR_MISSING = -4   /* a weight the architecture needs was never loaded */
};

/* FE.BUILDER build_fcos_dla_fpn_backbone_p67 with FE.BACKBONE.NAME "DLA-34", or build_fcos_vovnet_fpn_backbone_p6 with the
 * VoVNet named by FE.BACKBONE.NAME (vovnet.py:19-97): "V-99-eSE" (1), "V-19-slim-dw-eSE", "V-19-dw-eSE", "V-19-slim-eSE",
 * "V-19-eSE", "V-39-eSE", "V-57-eSE" (2..7).  Every VoVNet has FPN levels p2..p6 and a size divisibility of 64.  The DLA
 * builder also takes "DLA-X-46-C", "DLA-X-60-C", "DLA-X-60", "DLA-X-102", "DLA-X-102-64" (8..12); every DLA has FPN levels
 * p3..p7 and a size divisibility of 128. */
enum dd3d_arch {
    DD3D_ARCH_DLA34 = 0,
    DD3D_ARCH_V2_99 = 1,
    DD3D_ARCH_V2_19_SLIM_DW = 2,
    DD3D_ARCH_V2_19_DW = 3,
    DD3D_ARCH_V2_19_SLIM = 4,
    DD3D_ARCH_V2_19 = 5,
    DD3D_ARCH_V2_39 = 6,
    DD3D_ARCH_V2_57 = 7,
    /* DLA-X (ResNeXt-style BottleneckX blocks with a grouped 3x3; dla.py:104-143,370-415) */
    DD3D_ARCH_DLA_X_46_C = 8,
    DD3D_ARCH_DLA_X_60_C = 9,
    DD3D_ARCH_DLA_X_60 = 10,
    DD3D_ARCH_DLA_X_102 = 11,
    DD3D_ARCH_DLA_X_102_64 = 12
};
enum dd3d_image_dtype { DD3D_IMG_U8 = 0, DD3D_IMG_F32 = 1 };
/* 16-bit storage type of activations and conv weights (accumulation, BN affine, head maps, decode and NMS are fp32
 * either way).  bf16 is the default; fp16 is the reference's mixed-precision type (amp.autocast, scripts/train.py:121;
 * BASELINE.json configs[4]) -- 3 more mantissa bits, range +-65504. */
enum dd3d_act_dtype { DD3D_ACT_BF16 = 0, DD3D_ACT_FP16 = 1 };

#define DD3D_MAX_CLASSES 16      /* rows of dd3d_model_desc.canonical_box3d_sizes */
#define DD3D_MAX_NUM_CLASSES 128 /* largest DD3D.NUM_CLASSES: above DD3D_MAX_CLASSES the sizes come from dd3d_set_canonical_sizes */
#define DD3D_NUM_LEVELS 5      /* most head levels (DD3D.IN_FEATURES entries) one engine runs */
#define DD3D_FPN_MAX_OUTPUTS 6 /* most FPN outputs: DLA level2..5 give p2..p7 */
#define DD3D_FPN_IN_STEM 1     /* dd3d_set_fpn_inputs number of the VoVNet stem output */

/* Mirrors the cfg values DD3D.__init__ / FCOS2DInference / FCOS3DInference read
 * (core.py:20-55, fcos2d.py:242-249, fcos3d.py:302-313; defaults configs/models/dd3d.yaml). */
typedef struct dd3d_model_desc {
    int32_t arch;        /* dd3d_arch: FE.BUILDER + FE.BACKBONE.NAME */
    int32_t num_classes; /* DD3D.NUM_CLASSES, 1..DD3D_MAX_NUM_CLASSES */
    float pixel_mean[3]; /* MODEL.PIXEL_MEAN (BGR) */
    float pixel_std[3];  /* MODEL.PIXEL_STD */
    int32_t feature_locations_offset_half; /* DD3D.FEATURE_LOCATIONS_OFFSET == "half" */
    float pre_nms_thresh;   /* FCOS2D.INFERENCE.PRE_NMS_THRESH (applied to sigmoid(cls)*sigmoid(ctr)) */
    int32_t pre_nms_topk;   /* PRE_NMS_TOPK (<= 1150: 5 levels of candidates fit the NMS's shared memory) */
    int32_t post_nms_topk;  /* POST_NMS_TOPK */
    float nms_thresh;       /* NMS_THRESH (<= 0 disables suppression) */
    int32_t do_nms;         /* DD3D.INFERENCE.DO_NMS */
    float min_depth, max_depth;             /* FCOS3D.MIN_DEPTH / MAX_DEPTH */
    int32_t scale_depth_by_focal_lengths;   /* FCOS3D.SCALE_DEPTH_BY_FOCAL_LENGTHS */
    float scale_depth_by_focal_lengths_factor;
    int32_t predict_allocentric_rot;        /* FCOS3D.PREDICT_ALLOCENTRIC_ROT */
    int32_t predict_distance;               /* FCOS3D.PREDICT_DISTANCE */
    float canonical_box3d_sizes[DD3D_MAX_CLASSES * 3]; /* FCOS3D.CANONICAL_BOX3D_SIZES rows 0..num_classes-1 (W,L,H); rows
                                                        * 0..15 only: more classes pass theirs to dd3d_set_canonical_sizes */
    int32_t out_cap;        /* detection slots per image in the output buffer (>= post_nms_topk; ties may exceed it) */
    int32_t nuscenes_heads; /* MODEL.META_ARCHITECTURE == NuscenesDD3D: attr_logits (3) + speed (1, relu) predictor convs
                             * on the cls tower (nuscenes_dd3d.py:311-312,380-383) */
    int32_t act_dtype;      /* dd3d_act_dtype */
    /* head switches no shipped experiment changes, mirrored for completeness (defaults 1, 1, 1, 0, 0, 1): */
    int32_t thresh_with_ctr;      /* FCOS2D.INFERENCE.THRESH_WITH_CTR: 0 = threshold sigmoid(cls) alone, rank by cls * ctr
                                   * (fcos2d.py:280-290) */
    int32_t fcos2d_use_scale;     /* FCOS2D.USE_SCALE: per-level Scale on box2d_reg (fcos2d.py:100-108,145-152) */
    int32_t fcos3d_use_scale;     /* FCOS3D.USE_SCALE: per-level Scale / Offset on ctr, size, conf, depth; when 0 the depth
                                   * predictor has a bias instead (fcos3d.py:116,128-139,175-180) */
    int32_t class_agnostic_box3d; /* FCOS3D.CLASS_AGNOSTIC_BOX3D: 11 instead of 11 * num_classes 3-D channels (fcos3d.py:103) */
    int32_t per_level_predictors; /* FCOS3D.PER_LEVEL_PREDICTORS: box3d_{quat,ctr,depth,size,conf}.<level> (fcos3d.py:104,166) */
    int32_t box3d_on;             /* MODEL.BOX3D_ON: 0 = 2-D detector only (core.py:34-40; NMS keyed on `scores`, :117-125) */
} dd3d_model_desc;

/* Normalisation after a head-tower or FPN conv (get_norm in fcos2d.py:73-91, fcos3d.py:82-100, detectron2 FPN):
 * "BN" / "FrozenBN" in a head tower give one BN per FPN level (ModuleListDial, keys <conv>.norm.<level>); "SyncBN" gives one
 * BN shared by the levels (<conv>.norm); "GN" GroupNorm(32, C) at the FPN width C (<conv>.norm.weight / .bias); "" no norm,
 * the conv has a bias.  The FPN has no per-level case: its BN / FrozenBN / SyncBN is DD3D_NORM_BN_SHARED (DD3D_NORM_BN_PER_LEVEL is
 * accepted as the same). */
enum dd3d_norm { DD3D_NORM_BN_PER_LEVEL = 0, DD3D_NORM_BN_SHARED = 1, DD3D_NORM_GN = 2, DD3D_NORM_NONE = 3 };

/* Structural switches of the FPN and the FCOS heads (defaults = the shipped layout, in brackets).  A separate struct so
 * that dd3d_model_desc keeps its size: an engine that never receives one builds the default layout. */
typedef struct dd3d_layout_desc {
    int32_t fcos2d_norm;      /* dd3d_norm of the cls / box2d towers: DD3D.FCOS2D.NORM [BN per level] */
    int32_t fcos3d_norm;      /* dd3d_norm of the box3d tower: DD3D.FCOS3D.NORM [BN per level] */
    int32_t fpn_norm;         /* dd3d_norm of the FPN lateral / output convs: FE.FPN.NORM [BN shared] */
    int32_t num_cls_convs;    /* DD3D.FCOS2D.NUM_CLS_CONVS, 0..16 [4]; 0: the predictors read the FPN outputs */
    int32_t num_box2d_convs;  /* DD3D.FCOS2D.NUM_BOX_CONVS, 0..16 [4] */
    int32_t num_box3d_convs;  /* DD3D.FCOS3D.NUM_CONVS, 0..16 [4] */
    int32_t fpn_fuse_avg;     /* FE.FPN.FUSE_TYPE == "avg": (lateral + top-down) / 2 [0 = "sum"] */
} dd3d_layout_desc;

/* One detection = the fields the reference returns in Instances (fcos2d.py:331-335,263; fcos3d.py:398-399). */
typedef struct dd3d_det {
    float box[4];      /* pred_boxes (x1, y1, x2, y2) */
    float score;       /* scores */
    float score_3d;    /* scores_3d */
    int32_t cls;       /* pred_classes */
    int32_t level;     /* fpn_levels */
    float quat[4];     /* pred_boxes3d.quat (w, x, y, z), egocentric */
    float proj_ctr[2]; /* pred_boxes3d.proj_ctr */
    float depth;       /* pred_boxes3d.depth */
    float size[3];     /* pred_boxes3d.size (W, L, H) */
    float loc[2];      /* locations */
    int32_t index;     /* pixel * num_classes + class at its level */
    int32_t attr;      /* pred_attributes (NuscenesDD3D, nuscenes_dd3d.py:296); 0 otherwise */
    float speed;       /* pred_speeds (NuscenesDD3D, nuscenes_dd3d.py:297); 0 otherwise */
    int32_t pad;
} dd3d_det;

/* One augmented view of test-time augmentation (SURVEY.md 8f row 4): a ResizeShortestEdge scale optionally followed by a
 * horizontal flip, described by what DD3DWithTTA needs to map its detections back (test_time_augmentation.py:190-239). */
typedef struct dd3d_tta_view {
    int32_t flip;       /* HFlipTransform after the resize */
    float view_w;       /* width of the view (flip axis) */
    float inv_sx[2];    /* fp32 x factors of the inverse ResizeTransforms, in application order: view -> model input,
                         * model input -> original image (1 if the dataset mapper did not resize) */
    float inv_sy[2];
    float K_view[9];    /* intrinsics the view was run with (tfms.apply_intrinsics, :78-82) */
    float K_orig[9];    /* inv_tfm.apply_intrinsics(K_view) (:214): the original camera, used by Boxes3D.from_vectors */
} dd3d_tta_view;

/* ---- lifetime ------------------------------------------------------------------------------------------- */
int dd3d_create(const dd3d_model_desc* h_desc, dd3d_handle* out);
void dd3d_destroy(dd3d_handle h);
const char* dd3d_last_error(dd3d_handle h); /* h may be NULL: error of the last failed dd3d_create,
                                             * dd3d_create_from_file, dd3d_graph_create or dd3d_graph_launch */

/* ---- self-contained model file: a trained model without Python or the PyTorch checkpoint -----------------------------
 * dd3d_create_from_file reads a model file written by DD3DB200.save_model_file (dd3d_b200/meta_arch.py) and builds the
 * engine that model builds from its config and state_dict: dd3d_create, dd3d_set_layout, dd3d_set_backbone_norm,
 * dd3d_set_fpn_channels, then dd3d_set_fpn_inputs / dd3d_set_in_features / dd3d_set_canonical_sizes when the file holds
 * them, one dd3d_load_weight per tensor record, dd3d_finalize.  The whole file is read and validated on the host before
 * the first CUDA call; a defect returns DD3D_ERR_INVALID with dd3d_last_error(NULL) naming it (unreadable file, bad magic,
 * unknown version, struct size mismatch, truncation, checksum mismatch, a record overrunning the file, a name twice).  An
 * error of one of the calls above is returned unchanged, its text prefixed with the call.  No handle survives an error.
 *
 * Layout, little-endian, no padding:
 *   char[8] "DD3DB200" | u32 version (1) | u32 size of dd3d_model_desc | u32 size of dd3d_layout_desc |
 *   u32 tensor records | u64 file size in bytes, checksum included
 *   dd3d_model_desc: pixel_mean / pixel_std of the state_dict, do_nms and the out_cap of the model's forward
 *   dd3d_layout_desc | i32 backbone dd3d_norm | i32 FPN width
 *   u32 n + i32[n] FPN inputs (n = 0: not set) | u32 n + i32[n] head levels (n = 0: not set)
 *   u32 n + f32[n][3] canonical sizes (n = 0: not set, the desc's 16 rows apply)
 *   per record: u32 name length + name bytes (no terminator) | u32 ndim (0..8) + i64[ndim] shape | f32 data, row-major
 *   u64 checksum: BLAKE2b (RFC 7693) with an 8-byte digest of every byte before it
 * Records hold the reference state_dict's floating-point tensors as fp32, not packed device weights, so a file does not
 * depend on the kernels' weight layouts.
 * Run-time switches are not in the file: option "do_postprocess" (dd3d_set_option), dd3d_set_bev_nms,
 * dd3d_set_sample_aggregate, the poses and groups stay per-call settings of the handle, as for an engine built call by
 * call. */
int dd3d_create_from_file(const char* path, dd3d_handle* out);
/* Detection slots per image of the output buffers of the forwards: dd3d_model_desc.out_cap of the engine. */
int dd3d_out_cap(dd3d_handle h);
/* backbone.size_divisibility: 128 (DLA p67) / 64 (VoVNet p6).  Every FPN input list the engine builds ends at stride 32
 * (dd3d_set_fpn_inputs), so the FPN inputs never change it. */
int dd3d_size_divisibility(dd3d_handle h);
/* Sets the FPN / head layout (dd3d_layout_desc) before dd3d_finalize (DD3D_ERR_STATE afterwards).  An unknown dd3d_norm value,
 * a depth outside 0..16 or fpn_fuse_avg other than 0 / 1 returns DD3D_ERR_INVALID and leaves the layout unchanged. */
int dd3d_set_layout(dd3d_handle h, const dd3d_layout_desc* h_layout);
/* Sets the backbone's norm (FE.BACKBONE.NORM) before dd3d_finalize (DD3D_ERR_STATE afterwards), as a dd3d_norm:
 * DD3D_NORM_BN_SHARED or DD3D_NORM_BN_PER_LEVEL (the default, for "FrozenBN", "BN" and "SyncBN", which compute the same thing in
 * eval: the BN is folded into each conv) or DD3D_NORM_NONE (DLA-34 only: "", every backbone conv has a bias and no norm).
 * DD3D_NORM_GN and, for a VoVNet, DD3D_NORM_NONE return DD3D_ERR_INVALID and leave the backbone unchanged.  An engine that
 * never receives the call builds the BN backbone. */
int dd3d_set_backbone_norm(dd3d_handle h, int32_t dd3d_norm);
/* Sets the FPN width (FE.FPN.OUT_CHANNELS) before dd3d_finalize (DD3D_ERR_STATE afterwards): the channels of the FPN laterals,
 * outputs and P6 / P7, of every head-tower conv and of the predictors' input (the reference's heads take their width from the
 * backbone's output shape).  Every multiple of 64 from 64 to 512; anything else returns DD3D_ERR_INVALID and leaves the width
 * unchanged.  An engine that never receives the call builds 256.  The sparse box2d / box3d towers need the pair tile, which
 * only widths that 128 divides run: at 64, 192, 320 and 448 those towers are dense (the sparse box3d predictor still runs). */
int dd3d_set_fpn_channels(dd3d_handle h, int32_t channels);
/* Sets FCOS3D.CANONICAL_BOX3D_SIZES, h_sizes = [num_classes][3] (W, L, H), before dd3d_finalize (DD3D_ERR_STATE afterwards);
 * num_classes must equal the desc's (DD3D_ERR_INVALID otherwise).  Required when num_classes > DD3D_MAX_CLASSES and box3d_on
 * (dd3d_finalize fails with DD3D_ERR_STATE without it); at 16 classes or fewer the desc's rows are used unless this call
 * replaces them.  Class-specific heads above 16 classes run the box3d predictor at the final candidates only, 11 channels
 * each, on the class-gathered kernel (csrc/b3d_gather.cu) under the "sparse_box3d" rule of dd3d_set_option. */
int dd3d_set_canonical_sizes(dd3d_handle h, int32_t num_classes, const float* h_sizes);
/* Sets FE.FPN.IN_FEATURES before dd3d_finalize and before dd3d_set_in_features (DD3D_ERR_STATE otherwise): h_inputs[0 .. n)
 * are the backbone outputs the FPN reads, by number: DLA level<k> is k, VoVNet stage<k> is k and the VoVNet stem is
 * DD3D_FPN_IN_STEM.  Their strides (DLA 2^k; VoVNet stem and stage2 4, stage<k> 2^k) must double from one input to the next
 * and end at 32, where the top block reads p5, with the first stride at least 4: DLA level2..5 and VoVNet stem / stage2..5.
 * The FPN outputs are p<log2 first stride> .. p5, then P6 (and P7 for a DLA): 2 to DD3D_FPN_MAX_OUTPUTS outputs; lateral /
 * output convs are named fpn_lateral<log2 stride> / fpn_output<log2 stride>.  Any other list returns DD3D_ERR_INVALID and
 * leaves the inputs unchanged.  An engine that never receives the call builds DLA level3..5 / VoVNet stage2..5.  With more
 * than DD3D_NUM_LEVELS FPN outputs, dd3d_set_in_features must select at most DD3D_NUM_LEVELS of them (dd3d_finalize returns
 * DD3D_ERR_INVALID otherwise). */
int dd3d_set_fpn_inputs(dd3d_handle h, const int32_t* h_inputs, int n);
/* Sets DD3D.IN_FEATURES before dd3d_finalize (DD3D_ERR_STATE afterwards): h_fpn_levels[0 .. n) are the FPN outputs the heads
 * run on, in head order, as indices into the FPN's outputs (by default DLA: p3..p7, VoVNet: p2..p6; dd3d_set_fpn_inputs
 * changes them), 1 <= n <= DD3D_NUM_LEVELS, no index twice (DD3D_ERR_INVALID otherwise, leaving the selection unchanged).  Every per-level tensor is taken by position:
 * tower norm l, Scale l, Offset l and (PER_LEVEL_PREDICTORS) predictor l serve the head at position l, and dd3d_det.level is
 * the position.  FPN outputs no head reads are not computed (dd3d_get_tensor refuses their "p<i>"); the head maps
 * "cls<l>" / "box<l>" / "b3d<l>" are by position.  Without DO_NMS up to n * pre_nms_topk detections per image survive.  An
 * engine that never receives the call runs every FPN output in order. */
int dd3d_set_in_features(dd3d_handle h, const int32_t* h_fpn_levels, int n);

/* ---- weights: one call per tensor of the reference state_dict (Checkpointer.load, scripts/train.py:52) ----- */
/* h_data: host fp32, contiguous, `ndim` dims in h_shape.  Unknown names are ignored (return DD3D_OK, e.g.
 * num_batches_tracked); known names with a wrong shape return DD3D_ERR_INVALID. */
int dd3d_load_weight(dd3d_handle h, const char* h_name, const float* h_data, const int64_t* h_shape, int ndim);
/* Folds BN / Scale / Offset into per-channel epilogue vectors, repacks conv weights to bf16 [Cout][tap][Cin]
 * and uploads them.  DD3D_ERR_MISSING names the first absent tensor. */
int dd3d_finalize(dd3d_handle h);

/* ---- planning: buffers + TMA descriptors for one (batch, source height, source width) --------------------- */
/* Hs, Ws: height/width of the source batch tensor [B][3][Hs][Ws]; the padded size is rounded up to the size
 * divisibility.  Returns the workspace bytes the plan needs. */
int64_t dd3d_workspace_bytes(dd3d_handle h, int B, int Hs, int Ws);
/* d_workspace may be NULL: the engine then allocates (and owns) the workspace. */
int dd3d_plan(dd3d_handle h, int B, int Hs, int Ws, void* d_workspace, int64_t workspace_bytes);

/* ---- the hot path ---------------------------------------------------------------------------------------- */
/* d_images: [B][3][Hs][Ws] (dd3d_image_dtype), image b valid in its top-left (h_b, w_b) corner.
 * d_intrinsics: [B][9] fp32 row-major K.  d_sizes: [B][4] int32 = (h_b, w_b, out_h, out_w): valid image size and
 * the size boxes are rescaled to (input["height"/"width"], core.py:156-158).
 * d_out: [B][out_cap] dd3d_det, d_counts: [B] int32.  Enqueues on `stream`; no host sync, no allocation. */
int dd3d_forward(dd3d_handle h, const void* d_images, int img_dtype, const float* d_intrinsics,
                 const int32_t* d_sizes, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream);
/* ---- the forward as a CUDA graph: record once, replay every frame -------------------------------------------------
 * dd3d_graph_create records one dd3d_forward of the current plan with these device buffers (stream capture on `stream` in
 * cudaStreamCaptureModeThreadLocal; the legacy default stream NULL cannot be captured, so a private stream records it then)
 * and instantiates it.  Nothing runs at the call.  The graph holds the launches the forward would make now: the buffers
 * above, the poses / groups / global-row buffers of dd3d_set_poses / dd3d_set_groups / dd3d_set_global_out, the BEV NMS and
 * sample aggregation settings and options "do_postprocess" / "do_nms".  Per frame the caller writes the new images,
 * intrinsics and sizes into the same buffers and calls dd3d_graph_launch, which enqueues the whole forward on `stream` (any
 * stream of the handle's device) with one cudaGraphLaunch: the same kernels as dd3d_forward, bit-identical results, the
 * kernels' programmatic dependent launches kept as programmatic edges (needs CUDA 12.3 or later).  Device state one forward
 * leaves for the next is reset by the forward's own kernels, so replays may follow each other and dd3d_forward calls freely;
 * like two forwards of one handle, they must not run concurrently (they share the plan's workspace).
 * Staleness: dd3d_plan (any shape), a plan drop, and every dd3d_set_option / dd3d_set_bev_nms / dd3d_set_poses /
 * dd3d_set_sample_aggregate / dd3d_set_groups / dd3d_set_global_out call after the capture make the graph stale: its
 * dd3d_graph_launch returns DD3D_ERR_STATE and launches nothing; create a new graph.  dd3d_destroy makes every graph of the
 * handle stale the same way; dd3d_graph_destroy frees a graph before or after its handle.
 * dd3d_graph_create returns DD3D_ERR_STATE before dd3d_plan or with option "profile" on (its events are for dd3d_forward),
 * any status of dd3d_forward for its arguments, and DD3D_ERR_CUDA when the capture or the instantiation fails; a failed
 * capture is ended and discarded, `stream` is not left capturing and *out is NULL.  The text of a failed dd3d_graph_create
 * or dd3d_graph_launch is in dd3d_last_error(NULL), and in dd3d_last_error(h) while the handle lives. */
typedef struct dd3d_graph_t* dd3d_graph;
int dd3d_graph_create(dd3d_handle h, const void* d_images, int img_dtype, const float* d_intrinsics,
                      const int32_t* d_sizes, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream, dd3d_graph* out);
int dd3d_graph_launch(dd3d_graph g, dd3d_stream stream);
void dd3d_graph_destroy(dd3d_graph g); /* NULL: no-op */
/* Kernel nodes of the graph: dd3d_launches_per_forward of the plan it was captured from. */
int dd3d_graph_kernel_nodes(dd3d_graph g);
/* Programmatic (PDL) edges of the graph: one per launch made with the programmatic-serialization attribute. */
int dd3d_graph_programmatic_edges(dd3d_graph g);
/* dd3d_forward through HOST buffers (pinned recommended): copies inputs H2D, runs, copies detections and counts D2H,
 * then synchronises `stream`. */
int dd3d_forward_host(dd3d_handle h, const void* h_images, int img_dtype, const float* h_intrinsics,
                      const int32_t* h_sizes, dd3d_det* h_out, int32_t* h_counts, dd3d_stream stream);
/* Double-buffered host path for a serving / evaluation loop (the role of the reference dataloader's prefetch +
 * x["image"].to(device), core.py:65): dd3d_submit_host enqueues H2D (on an engine-owned copy stream) -> kernels -> D2H (on
 * `stream`) for slot 0 or 1 and returns at once; dd3d_wait_host blocks until that slot's detections are in h_out /
 * h_counts.  Submitting batch i+1 to the other slot before waiting for batch i overlaps its H2D with batch i's kernels.
 * Host buffers must be pinned and stay valid until the wait; a slot must be waited before it is submitted again. */
int dd3d_submit_host(dd3d_handle h, int slot, const void* h_images, int img_dtype, const float* h_intrinsics,
                     const int32_t* h_sizes, dd3d_det* h_out, int32_t* h_counts, dd3d_stream stream);
int dd3d_wait_host(dd3d_handle h, int slot);
/* bit 0: unused (the pre-NMS top-k is exact for every input and sets no bit); bit 1: more than out_cap detections
 * survived; with the BEV NMS on (dd3d_set_bev_nms), bit 2: more than 256 boxes reached the one-CTA BEV kernel of an
 * image, bit 6: a count above out_cap reached the multi-CTA one; with the sample aggregation on
 * (dd3d_set_sample_aggregate), bit 3 (one-CTA path) / bit 5 (blocked path): a sample group beyond the kernel's capacity.
 * Reads a device word (synchronises `stream`). */
int dd3d_overflow_flags(dd3d_handle h, dd3d_stream stream, int32_t* h_flags);
/* Runtime switches the reference's callers toggle on the meta-arch: "do_postprocess" (postprocess_in_inference,
 * scripts/train.py:206-209, test_time_augmentation.py:107), "do_nms" (core.py:134), "profile" (see
 * dd3d_get_profile), "sparse_box3d" (2 = auto, the default: the fused FCOS3D predictor conv is evaluated only at the pixels that survive the 2-D
 * threshold and per-level top-k, between the two halves of the decode, when the head maps of one image hold >= 50 000 pixels (a per-image rule: batch-independent results) -- the dense
 * "b3d<l>" maps of dd3d_get_tensor then do not exist; 1: always; 0: never (dense fp32 maps, for stage-level tests); changing
 * it drops the engine's plans), "sparse_tower" (2 = auto, the default: with the sparse predictor, a non-GN box3d tower on
 * pair-tile convs and >= 50 000 head pixels per image, the tower runs after the threshold / top-k on the conv tiles the
 * predictor's reads need -- bit-identical detections, the "op<i>" outputs of the tower hold stale values elsewhere; 1: whenever
 * the sparse predictor runs and the tower qualifies; 0: dense tower; changing it drops the engine's plans),
 * "sparse_box2d_tower" (2 = auto, the default: with the sparse box3d predictor, a non-GN FCOS2D head whose box2d tower runs
 * on pair-tile convs and >= 50 000 head pixels per image, the box2d tower and its [box2d_reg | centerness] predictor run
 * only on the conv tiles around the pixels where some class score passes PRE_NMS_THRESH -- bit-identical detections;
 * "box0".."box4" of dd3d_get_tensor then refuse (the map is stale elsewhere) and the "op<i>" outputs of that tower hold
 * stale values; 1: whenever the head qualifies; 0: dense; environment DD3D_SPARSE_BOX2D_TOWER; changing it drops the
 * engine's plans), "workspace_reuse" (default 1: activation buffers with disjoint lifetimes share workspace memory --
 * after a forward only "input", "p0".."p4" and the head maps of dd3d_get_tensor are intact; 0: every op output keeps its own
 * memory, for stage-level tests; applies to plans made afterwards), and "workspace_fill" (0..255: dd3d_plan fills the whole workspace with that byte first, -1 = off;
 * the poison test of tests/test_determinism_gpu.py: results must not depend on what the arena held). */
int dd3d_set_option(dd3d_handle h, const char* name, int value);

/* ---- BEV NMS (DD3D.INFERENCE.DO_BEV_NMS, core.py:137-151) as the last op of every forward ----------------------------
 * dd3d_set_bev_nms(h, 1, thr): every following dd3d_forward / dd3d_forward_host / dd3d_submit_host / dd3d_forward_raw
 * ends with the reference's per-image BEV NMS (boxes to the global frame through the image's pose, class-aware rotated
 * NMS on scores_3d with IoU threshold BEV_NMS_IOU_THRESH; survivors keep their order), and option "do_postprocess" then
 * applies detector_postprocess after it instead of inside the 2-D NMS (core.py:153-160).  Needs box3d_on.  The kernel is
 * chosen from the config (dd3d_bev_nms_path); turning the BEV NMS on or off, or a "do_nms" change that switches the
 * kernel, drops the engine's plans (call dd3d_plan again).  With it off the op list, the launches and the workspace are
 * those of an engine that never had it.
 * Poses: [B][7] sensor->global pose of each image (quaternion w, x, y, z + translation; input["pose"] /
 * input["extrinsics"]).  dd3d_set_poses: a DEVICE buffer read by every following dd3d_forward / dd3d_forward_raw (kept
 * until replaced; it must stay valid while those forwards run).  dd3d_set_host_poses: a HOST array of the current plan's
 * B images, copied at the call, for dd3d_forward_host (slot 0) and dd3d_submit_host (slot 0 / 1).  A forward with the BEV
 * NMS on and no poses returns DD3D_ERR_STATE. */
int dd3d_set_bev_nms(dd3d_handle h, int enable, float iou_thresh);
int dd3d_set_poses(dd3d_handle h, const float* d_poses);
int dd3d_set_host_poses(dd3d_handle h, int slot, const float* h_poses);
/* The BEV NMS kernel a config runs (no device needed): 1 = the one-CTA kernel of dd3d_op_bev_nms (do_nms and
 * 0 < post_nms_topk <= 256: at most 256 score-sorted boxes per image), 2 = the multi-CTA kernels of dd3d_op_bev_nms_large
 * (every other config: up to 5 * pre_nms_topk unsorted boxes per image). */
int dd3d_bev_nms_path(const dd3d_model_desc* h_desc);
/* ---- NuscenesDD3D sample aggregation (nuscenes_dd3d.py:449-463 -> postprocessing.py:58-108) as the last step of every
 * forward -------------------------------------------------------------------------------------------------------------
 * dd3d_set_sample_aggregate(h, 1, thr, max_dets): every following dd3d_forward / dd3d_forward_host / dd3d_submit_host /
 * dd3d_forward_raw ends, after the NMS (and BEV NMS) step with detector_postprocess applied, with the reference's
 * nuscenes_sample_aggregate on the detections of the call: boxes to the global frame through each image's pose, one
 * class-aware rotated BEV NMS on scores_3d (IoU threshold thr, BEV_NMS_IOU_THRESH) per sample group, then only the
 * max_dets best survivors OF THE CALL stay (keep[:MAX_NUM_DETS_PER_SAMPLE]; max_dets <= 0: no cap) -- per rank under
 * multi-GPU, as the reference's per-rank forward; survivors keep their order, and the pred_boxes3d_global rows (quat w, x,
 * y, z, tvec, size) of the survivors, compacted like the detections, go to the global-row buffer.  Same results as
 * dd3d_op_sample_aggregate after the forward.  A sample's images must all be in one call.  Needs box3d_on.  The kernel is
 * chosen from the config (dd3d_sample_aggregate_path); turning the step on or off, or a "do_nms" change that switches the
 * kernel, drops the engine's plans (call dd3d_plan again).  With it off the op list, the launches and the workspace are
 * those of an engine that never had it.  Overflow: flags bit 3 (one-CTA path: a group above 768 boxes or 16 images), bit 5
 * (blocked path: a count above out_cap or a group above 16 images / out of range).
 * Poses: dd3d_set_poses / dd3d_set_host_poses (the BEV NMS's).  Group indices: [B] int32, 0..num_groups-1 (get_group_idxs,
 * postprocessing.py:111-123), 1 <= num_groups <= B: dd3d_set_groups, a DEVICE buffer read by every following dd3d_forward /
 * dd3d_forward_raw (kept until replaced; NULL clears it); dd3d_set_host_groups, a HOST array copied at the call for the
 * host paths' slot 0 / 1 (needs a plan).  Global rows: dd3d_set_global_out, a DEVICE buffer [B][out_cap][10] fp32 the
 * device forwards write; dd3d_set_host_global_out, a HOST buffer (pinned) of the same shape per slot, filled by
 * dd3d_forward_host (slot 0) or by the time dd3d_wait_host(slot) returns.  A forward with the step on and no poses, groups
 * or global-row buffer returns DD3D_ERR_STATE. */
int dd3d_set_sample_aggregate(dd3d_handle h, int enable, float iou_thresh, int max_dets);
int dd3d_set_groups(dd3d_handle h, const int32_t* d_group, int num_groups);
int dd3d_set_host_groups(dd3d_handle h, int slot, const int32_t* h_group, int num_groups);
int dd3d_set_global_out(dd3d_handle h, float* d_global);
int dd3d_set_host_global_out(dd3d_handle h, int slot, float* h_global);
/* The sample aggregation kernels a config runs (no device needed): 1 = the one-CTA pair of dd3d_op_sample_aggregate (do_nms,
 * 0 < post_nms_topk <= 128 and out_cap <= 256: six cameras fit its 768-box group), 2 = the blocked kernels of
 * dd3d_op_group_bev_nms_large in global mode (every other config: up to 6 * 5 * 1150 = 34 500 boxes per sample, at most 256
 * images per call). */
int dd3d_sample_aggregate_path(const dd3d_model_desc* h_desc);
/* Process-wide kernel-selection policy for plans / operator calls made afterwards (tests, A/B measurements):
 * "op_fp16" = 1: the dd3d_op_* entry points below treat their 16-bit buffers as fp16 (default 0: bf16).
 * "nms_class_parallel" = 0: one CTA per image does the whole NMS instead of the multi-CTA path (rank sort, IoU bit matrix on
 * all SMs, one scan CTA per (class, image), finish; default 1; same kept set and order).  A plan also reads it again when
 * option "do_nms" changes.
 * "taps" = 0: 3x3 convs with <= 16 output channels use the per-tap kernels instead of the taps-in-N kernel (default 1).
 * "wstat" = 0: 3x3 layers whose whole weight tensor fits in shared memory next to the activation patches (64 -> 64 channels)
 * stream it per tile like every other layer instead of keeping it resident (default 1; bit-identical results either way).
 * "n_split" = 0: conv launches with fewer work items than half the SMs keep their N tile instead of splitting it (default 1;
 * bit-identical results either way).
 * "pair_tile": 3x3 stride-1 (halo) layers whose padded output channels are a multiple of 128 run a 256-pixel x 128-channel
 * tile (two 16x8 tiles share each weight tile: half the weight traffic per MAC).  -1 (default): when the launch has at least
 * one (tile pair, 128-channel block) per SM, otherwise the 128-pixel tile and the N-split keep the machine filled; 1: wherever
 * eligible; 0 (or environment DD3D_CONV_PAIR=0): never.  Bit-identical results either way. */
int dd3d_set_conv_policy(const char* name, int value);
/* Number of kernel launches one dd3d_forward of the current plan enqueues (for the bench's gpu_launches claim): the sum over
 * the steps the plan will launch (0 without a plan). */
int dd3d_launches_per_forward(dd3d_handle h);

/* Per-category device time of the LAST dd3d_forward issued with option "profile" = 1 (CUDA events recorded on the
 * launch stream around every op), with the algorithmic FLOPs / HBM bytes and launch counts of one forward.
 * Categories (arrays of 8): 0 preprocess, 1 special-purpose conv kernels (stem convs, the fused DLA-34 front end and the
 * depthwise 3x3 convs of the VoVNet -dw variants), 2 wgmma implicit-GEMM conv, 3 max-pool, 4 eSE, 5 relu and GroupNorm (the
 * elementwise passes over a map), 6 decode, 7 NMS (with the BEV NMS and the sample aggregation). */
int dd3d_get_profile(dd3d_handle h, double* h_ms, double* h_flops, double* h_bytes, int32_t* h_launches);
/* Same events, one entry per step in launch order: the preprocess, every engine op (with the sparse box2d / box3d towers,
 * their tile lists in front of them), the decode, the NMS, the sample aggregation when it is on.  Per entry: device ms, category, algorithmic FLOPs and, when
 * h_ops is not null, the engine op it timed (the index of dd3d_get_conv_info / dd3d_get_tensor "op<i>"), or -1 for the
 * preprocess, tile-list, decode and NMS entries.  Returns the number of entries written (<= max_ops). */
int dd3d_get_op_times(dd3d_handle h, float* h_ms, int32_t* h_cats, double* h_flops, int32_t* h_ops, int max_ops);
/* Kernel choice of every engine op of the current plan, in op order (dd3d_get_op_times names the op of each of its
 * entries): 8 int32 per op = {implicit-GEMM conv: 1 dense, 2 grouped block-diagonal mode; taps, stride, cin, padded cout,
 * halo variant, pair tile, block_n}, all 0 for other ops.  Returns the number of ops written (<= max_ops). */
int dd3d_get_conv_info(dd3d_handle h, int32_t* h_info, int max_ops);

/* ---- GPU input pipeline (SURVEY.md 8f row 3) ------------------------------------------------------------------
 * Replaces the per-image CPU work of DefaultDatasetMapper.__call__ at test time
 * (tridet/data/dataset_mappers/dataset_mapper.py:100-153 with augmentations = [ResizeShortestEdge],
 * tridet/data/augmentations/build.py:35-44): detectron2 ResizeShortestEdge.get_transform (output shape),
 * ResizeTransform.apply_image = PIL.Image.resize(BILINEAR) (bit-exact restatement of Pillow's 8-bit ImagingResample),
 * apply_imresize_intrinsics (tridet/data/augmentations/resize_transform.py:13-21), and the model's own preprocess. */
int dd3d_resize_shape(int h, int w, int min_size, int max_size, int32_t* new_h, int32_t* new_w);
/* d_raw: [B][raw_h][raw_w][3] uint8, cv2 layout (HWC, BGR); image b occupies the top-left h_raw_sizes[b] = (h, w) of its
 * slot.  h_intrinsics: [B][9] of the ORIGINAL images.  min_size / max_size: INPUT.RESIZE.MIN_SIZE_TEST / MAX_SIZE_TEST
 * (min_size 0: no resize).  The plan must cover the resized sizes (dd3d_resize_shape).  Detections are mapped back to
 * the original resolution when option do_postprocess is on (dataset dicts carry the file's height / width).
 * h_intrinsics_out [B][9] / h_new_sizes [B][2] (optional) receive the rescaled intrinsics and the resized (h, w). */
int dd3d_forward_raw(dd3d_handle h, const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                     const float* h_intrinsics, int min_size, int max_size, dd3d_det* d_out, int32_t* d_counts,
                     float* h_intrinsics_out, int32_t* h_new_sizes, dd3d_stream stream);

/* Same kernels with caller-chosen shapes: h_new_sizes [B][2] resized (h, w), h_flip [B] (or NULL) horizontal flip after
 * the resize, h_intrinsics [B][9] the intrinsics the views run with, h_sizes [B][4] (h, w, out_h, out_w) rows of
 * dd3d_forward.  These are the augmented views of DatasetMapperTTA (test_time_augmentation.py:24-87). */
int dd3d_forward_resized(dd3d_handle h, const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                         const int32_t* h_new_sizes, const int32_t* h_flip, const float* h_intrinsics,
                         const int32_t* h_sizes, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream);

/* ---- multi-GPU: ONE NCCL all-gather of the packed detections (SURVEY.md 8e) --------------------------------------
 * Batches shard over the GPUs with replicated weights and no collective inside dd3d_forward; for whole-batch evaluation
 * each rank contributes one fixed-stride buffer and receives everybody's -- the replacement of detectron2 comm.gather of
 * pickled prediction lists (kitti_3d_evaluator.py:152-164).  Packed layout (dd3d_packed_bytes(B, out_cap) bytes, 256-byte
 * padded):  dd3d_det[B][out_cap] | int32 counts[B] | int32 flags  -- allocate ONE device buffer, pass its two parts as
 * d_out / d_counts of dd3d_forward, fill the flags word with dd3d_copy_flags, then gather the whole buffer.
 * NCCL is resolved at run time (dlopen libnccl.so.2; env DD3D_NCCL_LIB overrides); without it these calls return
 * DD3D_ERR_CUDA and dd3d_comm_last_error() says why.  One process per GPU. */
typedef struct dd3d_comm_s* dd3d_comm;
int64_t dd3d_packed_bytes(int B, int out_cap);
/* Extended layout for NuscenesDD3D (dd3d_set_sample_aggregate): the three parts above at the same offsets, then
 * float global[B][out_cap][10] (the global-row buffer of the forward) at byte offset dd3d_packed_bytes(B, out_cap), padded to
 * 256 bytes -- detections, counts, flags and pred_boxes3d_global in ONE buffer for ONE all-gather. */
int64_t dd3d_packed_bytes_global(int B, int out_cap);
/* device word of the overflow flags of the last forward (bits as dd3d_overflow_flags) -> d_dst, on `stream`, no sync */
int dd3d_copy_flags(dd3d_handle h, int32_t* d_dst, dd3d_stream stream);
int dd3d_comm_unique_id(uint8_t* h_id128);          /* rank 0: ncclGetUniqueId; ship the 128 bytes to the other ranks */
int dd3d_comm_create(const uint8_t* h_id128, int rank, int world, dd3d_comm* out); /* ncclCommInitRank, current device */
int dd3d_comm_from_nccl(void* nccl_comm, int rank, int world, dd3d_comm* out);     /* adopt an existing ncclComm_t */
int dd3d_comm_world(dd3d_comm c);
void dd3d_comm_destroy(dd3d_comm c);
const char* dd3d_comm_last_error(void);
/* ncclAllGather of bytes_per_rank bytes: d_recv receives world x bytes_per_rank, rank-major.  Enqueued on `stream`. */
int dd3d_allgather(dd3d_comm c, const void* d_send, void* d_recv, int64_t bytes_per_rank, dd3d_stream stream);

/* ---- introspection for stage-level parity tests ---------------------------------------------------------- */
/* name: "p0".."p4" (FPN outputs, bf16 NHWC), "cls0".."cls4", "box0".."box4", "b3d0".."b3d4" (fp32 NHWC head maps),
 * "input" (bf16 [B][Hp][Wp][4]).  Returns the device pointer and fills dims = {B, H, W, C, pitch, elem_bytes}. */
int dd3d_get_tensor(dd3d_handle h, const char* name, void** d_ptr, int32_t dims[6]);
/* Also "op<i>" / "op<i>:<seg>": the bf16 NHWC output view of engine op i in launch order (segment seg of a multi-level
 * tower conv), 0 <= i < dd3d_num_ops; fp32 predictor outputs are the "cls"/"box"/"b3d" maps above. */
int dd3d_num_ops(dd3d_handle h);

/* ---- single operators (same kernels the engine launches; used by the kernel-level parity tests) ----------- */
/* The 16-bit element type of the operator entry points is process-wide: dd3d_set_conv_policy("op_fp16", 0 | 1). */
/* NHWC bf16 conv via the wgmma implicit-GEMM kernel.  d_w: bf16 [cout_pad][ksize*ksize][cin_pad64];
 * d_scale/d_bias: fp32 [cout_pad]; d_residual (optional) NHWC bf16 with res_pitch channels, res_up2: residual is
 * the 2x coarser map; out: bf16 (out_f32 == 0, pitch out_pitch) or fp32. */
int dd3d_op_conv2d(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout, int ksize,
                   int stride, const float* d_scale, const float* d_bias, int relu, const void* d_residual,
                   int res_pitch, int res_up2, void* d_out, int out_pitch, int out_f32, dd3d_stream stream);
/* dd3d_op_conv2d_grouped: grouped 3x3 conv (padding 1, C input = C output channels, `groups` groups of cpg = C / groups
 * channels; the BottleneckX conv2 of dla.py:113-124) -> scale / bias -> ReLU when relu -> 16-bit NHWC, on the block-diagonal
 * mode of the implicit-GEMM kernel: one launch, 64 output channels per n-block, each reading only its own 64 input channels.
 * Needs C a multiple of 64 and cpg dividing 64 (cpg 2..32 for groups 32 / 64).  d_in / d_out: first channel of the input /
 * output slice, pitches in channels (multiples of 8); stride 1 or 2 (even H, W).  d_w: 16-bit [C][9][64], tap = ky * 3 + kx:
 * row co holds w[co][i][ky][kx] at column (co / cpg) * cpg % 64 + i and zeros in every other column.  d_scale / d_bias:
 * fp32 [C].  Channels outside the output slice are not written. */
int dd3d_op_conv2d_grouped(const void* d_in, int B, int H, int W, int C, int in_pitch, const void* d_w, int groups,
                           int stride, const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch,
                           dd3d_stream stream);
/* dd3d_op_conv2d_tiles: dd3d_op_conv2d (3x3, stride 1, 16-bit output, cout a multiple of 128, no residual) on the pair-tile
 * kernel in work-list mode: only the 16x8 output tiles listed in d_tiles are computed, every other output pixel is left
 * untouched.  d_tiles: device uint32 entries (img << 16) | tile, tile = the row-major index of a 16x8 tile of one image (the
 * tile count of an image, ceil(H/16) * ceil(W/8), names the out-of-image tile, which writes nothing); consecutive entries
 * 2i, 2i + 1 form one work item and name one image.  d_count: device int32, the number of entries (even), read by the kernel.
 * dd3d_op_conv2d_tiles8x8: the same on 8x8 tiles (ceil(H/8) * ceil(W/8) per image), the form the engine runs the sparse
 * towers in: consecutive entries 4i .. 4i + 3 form one work item and name one image; the number of entries is a multiple
 * of 4. */
int dd3d_op_conv2d_tiles(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                         const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch, const uint32_t* d_tiles,
                         const int32_t* d_count, dd3d_stream stream);
int dd3d_op_conv2d_tiles8x8(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                            const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch,
                            const uint32_t* d_tiles, const int32_t* d_count, dd3d_stream stream);
/* dd3d_op_conv2d_taps_tiles: the 3x3 stride-1 conv of dd3d_op_conv2d with cout <= 16 on the taps-in-N kernel in work-list
 * mode, the form the engine runs the sparse box2d tower's predictor in: only the 16x8 output tiles listed in d_tiles are
 * computed (entries as in dd3d_op_conv2d_tiles, one work item each, the out-of-image tile writes nothing), every other output
 * pixel is left untouched.  d_scale / d_bias: fp32 [16]; out: fp32 (out_f32, out_pitch a multiple of 4) or 16-bit (a
 * multiple of 8), 16 channels written per pixel.  d_count: device int32, the number of entries, read by the kernel. */
int dd3d_op_conv2d_taps_tiles(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                              const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch, int out_f32,
                              const uint32_t* d_tiles, const int32_t* d_count, dd3d_stream stream);
/* dd3d_op_b3d_sparse: the sparse FCOS3D box3d predictor (csrc/b3d_sparse.cu) on caller buffers: for every (image b, level l)
 * and slot s < min(d_counts[b * 5 + l], topk), row (b * 5 + l) * topk + s of d_rows (fp32, out_pitch floats per row) receives
 * the 3x3 conv of level l's tower output at the candidate's pixel, channels 0 .. n_pad-1, times d_scale[l] plus d_bias[l]
 * (fp32).  Other rows are not written.  d_in[l]: 16-bit NHWC [B][H_l][W_l][h_pitch[l]] with 256 channels (h_level_hw = [5][2]
 * (H, W)); d_w[l]: 16-bit [n_pad][9][256] (dd3d_op_conv2d layout); d_fin: device [B][5][topk] uint32 pairs (any, pixel * C +
 * class); n_pad a multiple of 8, at most 112. */
int dd3d_op_b3d_sparse(const void* const* d_in /*[5]*/, const int32_t* h_level_hw, const int32_t* h_pitch /*[5]*/,
                       const void* const* d_w /*[5]*/, const float* const* d_scale /*[5]*/, const float* const* d_bias /*[5]*/,
                       const void* d_fin, const int32_t* d_counts, int B, int C, int topk, int n_pad, float* d_rows,
                       int out_pitch, dd3d_stream stream);
/* dd3d_op_b3d_sparse_c: dd3d_op_b3d_sparse with `cin` tower channels instead of 256 (FE.FPN.OUT_CHANNELS): d_in[l] has cin
 * channels (h_pitch[l] >= cin), d_w[l] is 16-bit [n_pad][9][cin].  cin a multiple of 64 from 64 to 512.  With cin = 256 it is
 * dd3d_op_b3d_sparse. */
int dd3d_op_b3d_sparse_c(const void* const* d_in /*[5]*/, const int32_t* h_level_hw, const int32_t* h_pitch /*[5]*/,
                         const void* const* d_w /*[5]*/, const float* const* d_scale /*[5]*/, const float* const* d_bias /*[5]*/,
                         const void* d_fin, const int32_t* d_counts, int B, int C, int topk, int n_pad, float* d_rows,
                         int out_pitch, int cin, dd3d_stream stream);
/* dd3d_op_b3d_gather: the class-gathered sparse box3d predictor (csrc/b3d_gather.cu) on caller buffers: for every (image b,
 * level l) and slot s < min(d_counts[b * 5 + l], topk) with class c = d_fin entry % C, row (b * 5 + l) * topk + s of d_rows
 * (fp32, 16 floats per row) receives at column q < 11 channel q * C + c of the 3x3 conv of level l's tower output at the
 * candidate's pixel, times d_scale[l][q * C + c] plus d_bias[l][q * C + c]: the values dd3d_op_b3d_sparse_c writes to those
 * columns, bit for bit.  Columns 11..15 and other rows are not written.  d_in / h_level_hw / h_pitch / d_fin / cin as for
 * dd3d_op_b3d_sparse_c; d_w[l]: 16-bit [>= 11 * C][9][cin]; C 1..128.  d_scratch: dd3d_op_b3d_gather_scratch_bytes(B, C, topk)
 * bytes, any content. */
int64_t dd3d_op_b3d_gather_scratch_bytes(int B, int C, int topk);
int dd3d_op_b3d_gather(const void* const* d_in /*[5]*/, const int32_t* h_level_hw, const int32_t* h_pitch /*[5]*/,
                       const void* const* d_w /*[5]*/, const float* const* d_scale /*[5]*/, const float* const* d_bias /*[5]*/,
                       const void* d_fin, const int32_t* d_counts, int B, int C, int topk, int cin, float* d_rows,
                       void* d_scratch, dd3d_stream stream);
/* dd3d_op_dla_front: the fused DLA-34 front end (csrc/dla_front.cu; reference dla.py:271-283,346-350 base_layer -> level0
 * -> level1, each conv + FrozenBN + ReLU, plus the 2x2 max-pool of level1's output, dla.py:235).  d_in4 = 16-bit
 * [B][H][W][4] (dd3d_op_preprocess output); d_w0 = 16-bit [16][7][8][4] (ky, kx padded to 8, c padded to 4), d_w1 = [16][9][16], d_w2 = [32][9][16]
 * (cout, tap, cin); d_sb* = fp32 scale[cout] | bias[cout]; d_out = [B][H/2][W/2][out_pitch], d_pool (may be NULL) =
 * [B][H/4][W/4][pool_pitch].  H, W multiples of 4. */
int dd3d_op_dla_front(const void* d_in4, const void* d_w0, const void* d_w1, const void* d_w2, const float* d_sb0,
                      const float* d_sb1, const float* d_sb2, void* d_out, int out_pitch, void* d_pool, int pool_pitch,
                      int B, int H, int W, dd3d_stream stream);
/* dd3d_op_stem_s2_mma: VoVNet stem_1 (3x3 stride 2, 3 -> 64, FrozenBN + ReLU; vovnet.py:302,357-359) on the register-fragment
 * kernel (csrc/stem_mma.cu), the kernel the engine runs for that layer.  d_in4 = 16-bit [B][H][W][4] (dd3d_op_preprocess
 * output), d_w = 16-bit [64][3][4][4] (cout, ky, kx, c; kx = 3 and c = 3 zero), d_sb = fp32 scale[64] | bias[64], d_out = [B][ceil(H/2)][ceil(W/2)][out_pitch]. */
int dd3d_op_stem_s2_mma(const void* d_in4, const void* d_w, const float* d_sb, void* d_out, int out_pitch, int B, int H, int W,
                        dd3d_stream stream);
/* dd3d_op_dwconv3x3: depthwise 3x3 conv (groups = C, padding 1, no bias; vovnet.py:100-121 dw_conv3x3) on the kernel the
 * engine runs for the VoVNet -dw variants (csrc/dwconv.cu).  d_in = [B][H][W][in_pitch], d_w = 16-bit [9][C] (tap = ky * 3
 * + kx), d_out = [B][(H-1)/stride+1][(W-1)/stride+1][out_pitch]; stride 1 or 2; C and both pitches multiples of 8, all three
 * pointers 16-byte aligned.  fp32 accumulation in tap order, one rounding to the 16-bit type at the store. */
int dd3d_op_dwconv3x3(const void* d_in, int B, int H, int W, int C, int in_pitch, const void* d_w, int stride, void* d_out,
                      int out_pitch, dd3d_stream stream);
/* dd3d_op_group_norm: GroupNorm(32, 256) on the kernels the engine runs for NORM "GN" (csrc/group_norm.cu): statistics over
 * each image's whole H x W map (biased variance, eps 1e-5, fp32 chunk statistics combined in a fixed order), then
 * y = x * gamma_c * rstd_g + (beta_c - mean_g * gamma_c * rstd_g), then + nearest-2x(d_residual) when d_residual is not NULL
 * (the coarser map [B][(H+1)/2 or H/2][(W+1)/2 or W/2][res_pitch]), then * 0.5 when avg, then ReLU when relu; one rounding to
 * the 16-bit type at the store.  d_in / d_out = [B][H][W][pitch] with 256 channels, d_out may equal d_in.  d_gamma == NULL
 * (d_beta too): add / scale only, no statistics.  d_scratch: dd3d_op_group_norm_scratch_bytes(B, H, W) bytes, any content.
 * Pitches multiples of 8 and >= 256, every pointer 16-byte aligned. */
int64_t dd3d_op_group_norm_scratch_bytes(int B, int H, int W);
int dd3d_op_group_norm(const void* d_in, int B, int H, int W, int in_pitch, const float* d_gamma, const float* d_beta, int relu,
                       const void* d_residual, int res_pitch, int avg, void* d_out, int out_pitch, void* d_scratch,
                       dd3d_stream stream);
/* dd3d_op_group_norm_c: GroupNorm(32, C) for C = 32 * cpg, cpg in {2, 4, 5, 6, 7, 8, 10, 12, 14, 16, 24, 32} (64 .. 1024
 * channels), same kernels and arithmetic as dd3d_op_group_norm (for C = 256 bit-identical to it), then ReLU when relu; one
 * rounding at the store.  Reads channels [in_c0, in_c0 + C) of d_in = [B][H][W][in_pitch] and writes channels [out_c0, out_c0 + C) of
 * d_out = [B][H][W][out_pitch]: channel slices of concat buffers; in place when d_out == d_in and out_c0 == in_c0.  d_gamma,
 * d_beta: fp32 [C].  d_scratch: dd3d_op_group_norm_scratch_bytes(B, H, W) bytes, any content.  Offsets and pitches multiples
 * of 8, d_in / d_out 16-byte aligned. */
int dd3d_op_group_norm_c(const void* d_in, int B, int H, int W, int C, int in_c0, int in_pitch, const float* d_gamma,
                         const float* d_beta, int relu, void* d_out, int out_c0, int out_pitch, void* d_scratch, dd3d_stream stream);
int dd3d_op_preprocess(const void* d_images, int img_dtype, const int32_t* d_sizes2, void* d_out4, int B, int Hs, int Ws,
                       int Hp, int Wp, const float* h_mean, const float* h_std, dd3d_stream stream);
int dd3d_op_maxpool(const void* d_in, void* d_out, int B, int H, int W, int C, int in_pitch, int out_pitch, int ksize,
                    dd3d_stream stream);
int dd3d_op_ese(const void* d_x, int x_pitch, const float* d_fc_w, const float* d_fc_b, const void* d_identity,
                int id_pitch, void* d_out, int out_pitch, float* d_scratch, int B, int HW, int C, dd3d_stream stream);
int64_t dd3d_op_ese_scratch_bytes(int B, int HW, int C);
/* Bird's-eye-view rotated NMS (reference DO_BEV_NMS branch, core.py:137-151 -> postprocessing.py:22-108 ->
 * tridet/layers/bev_nms.py:51-133 -> detectron2 batched_nms_rotated), in place on the detections a dd3d_forward run
 * with option "do_postprocess" = 0 produced: d_dets [B][cap], d_counts [B].  d_poses: [B][7] sensor->global pose of
 * each image (quaternion w,x,y,z + translation; input["pose"] / input["extrinsics"]).  Applies detector_postprocess
 * afterwards when do_postprocess != 0.  d_flags: one int32 word, bit 2 set if an image had more than 256 boxes.  The input
 * must be sorted by scores_3d (the 2-D NMS output); dd3d_op_bev_nms_large takes any order and size. */
int dd3d_op_bev_nms(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                    const int32_t* d_sizes, int32_t* d_flags, int B, int cap, float iou_thresh, int do_postprocess,
                    dd3d_stream stream);
/* dd3d_op_bev_nms_large: the same BEV NMS on the multi-CTA kernels of csrc/bev_nms_group.cu for up to 5 * 1150 boxes per
 * image in any order (cap <= 5750): per image a sort by (class, scores_3d descending, slot), the rotated-IoU bit matrix on
 * all SMs, one greedy scan per (image, class), then an order-preserving compaction (with detector_postprocess when
 * do_postprocess != 0).  d_scratch: dd3d_op_bev_nms_large_scratch_bytes(B, cap) bytes, any content (about
 * min(B, 256) * cap^2 / 8 bytes: the IoU bit matrix).  Class ids 0..127.  d_flags bit 6 (64): a count above cap. */
int64_t dd3d_op_bev_nms_large_scratch_bytes(int B, int cap);
int dd3d_op_bev_nms_large(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                          const int32_t* d_sizes, void* d_scratch, int32_t* d_flags, int B, int cap, float iou_thresh,
                          int do_postprocess, dd3d_stream stream);
/* d_out[i] = rotated IoU of the BEV rectangles d_a[i] and d_b[i] (rows of 5 floats: cx, cy, w, h, angle in degrees;
 * detectron2's single_box_iou_rotated), one thread per pair: the function the three BEV NMS kernels threshold, exposed
 * for tests. */
int dd3d_op_rotated_iou(const float* d_a, const float* d_b, int n, float* d_out, dd3d_stream stream);
/* resize (+ optional horizontal flip, h_flip [B] or NULL) + normalise + pad + NHWC4 bf16 of raw HWC uint8 images (the
 * first kernel of dd3d_forward_raw / dd3d_forward_resized). */
int dd3d_op_resize_preprocess(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                              const int32_t* h_new_sizes, const int32_t* h_flip, void* d_out4, int B, int Hp, int Wp,
                              const float* h_mean, const float* h_std, dd3d_stream stream);
/* Test-time-augmentation merge (DD3DWithTTA._get_augmented_instances + the merged NMS of _inference_one_image,
 * tridet/modeling/dd3d/test_time_augmentation.py:160-171,190-239) for ONE image: d_dets [num_views][cap] / d_counts
 * [num_views] are the views' detections (dd3d_forward* with do_postprocess = 0); 2-D boxes, 3-D boxes and the projected
 * centres are mapped back to the original image, concatenated in view order and reduced by one class-aware NMS on
 * scores_3d (do_nms = 0: the plain concatenation in view order).  d_out: dd3d_op_tta_merged_cap(num_views, cap) slots,
 * descending scores_3d after the NMS; field `level` = view index.  d_flags bit 4: more merged detections than slots. */
int dd3d_op_tta_merged_cap(int num_views, int cap);
int64_t dd3d_op_tta_merge_scratch_bytes(int num_views, int cap);
int dd3d_op_tta_merge(const dd3d_det* d_dets, const int32_t* d_counts, const dd3d_tta_view* h_views, int num_views, int cap,
                      float nms_thresh, int do_nms, void* d_scratch, dd3d_det* d_out, int32_t* d_out_count,
                      int32_t* d_flags, dd3d_stream stream);
/* dd3d_op_tta_merge for merged sets beyond its 1024 slots: the same arguments, transforms and output contract (descending
 * scores_3d after the class-aware NMS; do_nms = 0: the plain concatenation in view order; `level` = view index) with
 * dd3d_op_tta_merged_cap_large(num_views, cap) = num_views * cap slots in d_out, cap <= 5 * 1150 per view (so up to
 * 16 * 5750 = 92 000 per image).  Equal scores_3d are ordered by the detection's `index`, then by view order.  The NMS is
 * a blocked greedy pass per class on all SMs (csrc/tta_large.cu); d_scratch: dd3d_op_tta_merge_large_scratch_bytes bytes,
 * any content, linear in num_views * cap.  Arguments out of range return DD3D_ERR_INVALID before any launch; d_flags bit 4
 * (16): a view count above cap.  do_nms = 2 (this operator only): no NMS, the concatenation sorted by scores_3d descending
 * with ties in view order -- the order of bev_nms's keep when the merged BEV NMS follows without the 2-D NMS
 * (test_time_augmentation.py:172-181): dd3d_op_group_bev_nms(_large) keeps the order of its input. */
int dd3d_op_tta_merged_cap_large(int num_views, int cap);
int64_t dd3d_op_tta_merge_large_scratch_bytes(int num_views, int cap);
int dd3d_op_tta_merge_large(const dd3d_det* d_dets, const int32_t* d_counts, const dd3d_tta_view* h_views, int num_views,
                            int cap, float nms_thresh, int do_nms, void* d_scratch, dd3d_det* d_out, int32_t* d_out_count,
                            int32_t* d_flags, dd3d_stream stream);
/* NuscenesDD3D sample aggregation (nuscenes_dd3d.py:449-463 -> postprocessing.py:58-108 nuscenes_sample_aggregate with
 * get_group_idxs groups, :111-129): BEV rotated NMS (scores_3d order, class aware) jointly over the images that share a
 * sample group, then -- like the reference's keep[:max_num_dets_per_sample] on the concatenation of the whole call -- only
 * the max_dets best survivors of the call stay (max_dets <= 0: no cap).  In place on d_dets [B][cap] / d_counts [B]
 * (cap <= 256), survivors keep their order.  d_group: [B] group index (0..num_groups-1) of each image; d_poses: [B][7]
 * global camera poses (input["pose"]); d_global: [B][cap][10] receives pred_boxes3d_global (quat wxyz, tvec, size) of the
 * survivors, compacted like d_dets; d_scratch: dd3d_op_sample_aggregate_scratch_bytes(B, cap) bytes.  d_flags: bit 3 set
 * if a group exceeded 768 boxes or 16 images. */
int64_t dd3d_op_sample_aggregate_scratch_bytes(int B, int cap);
int dd3d_op_sample_aggregate(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                             const int32_t* d_group, int num_groups, float* d_global, void* d_scratch, int32_t* d_flags,
                             int B, int cap, float iou_thresh, int max_dets, dd3d_stream stream);
/* Grouped rotated BEV NMS for large detection sets (csrc/bev_nms_group.cu): the BEV steps of NuscenesDD3D test-time
 * augmentation (nuscenes_dd3d_tta.py), whose merged sets exceed the limits of the two entry points above.  In place on
 * d_dets [B][cap] / d_counts [B] (B <= 256, cap <= 1024): one class-aware rotated NMS (scores_3d descending, ties by image
 * then slot) per group of images (d_group [B], 0..num_groups-1, at most max_group_images <= 16 images per group), then --
 * max_dets > 0 -- only
 * the max_dets best survivors of the WHOLE call stay (keep[:max_num_dets_per_sample] of postprocessing.py:92-93); survivors
 * keep their order.  Each box's translation is inv(K) (proj_ctr, 1) * depth with K = d_view_K[b][level][9] (num_views = 1:
 * one K per image; the TTA merge stores the view index in `level`).  pose_mode DD3D_POSE_GLOBAL: boxes go to the global
 * frame through d_poses [B][7] (sample_bev_nms, postprocessing.py:22-55); DD3D_POSE_CAMERA: bev_nms with its default
 * pose_cam_global = CAMERA_TO_VEHICLE_ROTATION (tridet/layers/bev_nms.py:99-133), d_poses unused.  d_global (or NULL):
 * [B][cap][10] receives quat (w,x,y,z), tvec, size of every survivor in that frame, compacted like d_dets.  d_scratch:
 * dd3d_op_group_bev_nms_scratch_bytes(B, cap, max_group_images) bytes, any content (about
 * B * cap^2 * max_group_images / 8 bytes: the IoU bit matrix).  Arguments out of range return DD3D_ERR_INVALID before any
 * launch; d_flags bit 5 (32) is set when a count exceeds cap, a group holds more than max_group_images images, or a group
 * index, class (>= 128) or view index is out of range. */
enum dd3d_pose_mode { DD3D_POSE_GLOBAL = 0, DD3D_POSE_CAMERA = 1 };
int64_t dd3d_op_group_bev_nms_scratch_bytes(int B, int cap, int max_group_images);
int dd3d_op_group_bev_nms(dd3d_det* d_dets, int32_t* d_counts, const float* d_view_K, int num_views, const float* d_poses,
                          int pose_mode, const int32_t* d_group, int num_groups, int max_group_images, float* d_global,
                          void* d_scratch, int32_t* d_flags, int B, int cap, float iou_thresh, int max_dets,
                          dd3d_stream stream);
/* dd3d_op_group_bev_nms for merged sets beyond its limits: the same arguments, modes, survivors, order, d_global rows and
 * flags (bit 5, 32) for B <= 256 images of cap <= 92 000 slots and groups of up to max_group_images <= 16 images, on the
 * blocked NMS of csrc/tta_large.cu.  d_scratch: dd3d_op_group_bev_nms_large_scratch_bytes(B, cap, max_group_images)
 * bytes, any content, linear in B * cap (no IoU bit matrix).  Arguments out of range return DD3D_ERR_INVALID before any
 * launch. */
int64_t dd3d_op_group_bev_nms_large_scratch_bytes(int B, int cap, int max_group_images);
int dd3d_op_group_bev_nms_large(dd3d_det* d_dets, int32_t* d_counts, const float* d_view_K, int num_views,
                                const float* d_poses, int pose_mode, const int32_t* d_group, int num_groups,
                                int max_group_images, float* d_global, void* d_scratch, int32_t* d_flags, int B, int cap,
                                float iou_thresh, int max_dets, dd3d_stream stream);
/* decode + NMS on caller-provided head maps (layout documented in csrc/detect.cuh). */
/* dd3d_op_detect_scratch_bytes sizes the NMS scratch for DD3D_MAX_CLASSES classes (dd3d_op_detect / _flags take at most that
 * many); dd3d_op_detect_c takes up to DD3D_MAX_NUM_CLASSES with dd3d_op_detect_c_scratch_bytes(B, pre_nms_topk, num_classes). */
int64_t dd3d_op_detect_scratch_bytes(int B, int pre_nms_topk);
int dd3d_op_detect(const dd3d_model_desc* h_desc, int B, const int32_t* h_level_hw /*[5][2]*/,
                   const int32_t* h_strides /*[5]*/, const float* const* d_cls /*[5]*/, const float* const* d_box,
                   const float* const* d_b3d, int cls_pitch, int b3d_pitch, const float* d_intrinsics,
                   const int32_t* d_sizes, void* d_scratch, dd3d_det* d_pre_nms /* [B][5*topk] or NULL */,
                   int32_t* d_pre_counts /* [B][5] or NULL */, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream);
/* Same, and d_flags (or NULL) receives one int32 word on `stream`: the overflow flags of this call (bits as
 * dd3d_overflow_flags). */
int dd3d_op_detect_flags(const dd3d_model_desc* h_desc, int B, const int32_t* h_level_hw /*[5][2]*/,
                         const int32_t* h_strides /*[5]*/, const float* const* d_cls /*[5]*/, const float* const* d_box,
                         const float* const* d_b3d, int cls_pitch, int b3d_pitch, const float* d_intrinsics,
                         const int32_t* d_sizes, void* d_scratch, dd3d_det* d_pre_nms, int32_t* d_pre_counts,
                         dd3d_det* d_out, int32_t* d_counts, int32_t* d_flags /* or NULL */, dd3d_stream stream);
/* dd3d_op_detect_flags for h_desc->num_classes up to DD3D_MAX_NUM_CLASSES: h_canonical_sizes = [num_classes][3] host array of
 * FCOS3D.CANONICAL_BOX3D_SIZES (NULL: the desc's rows, num_classes <= DD3D_MAX_CLASSES); d_scratch:
 * dd3d_op_detect_c_scratch_bytes(B, pre_nms_topk, num_classes) bytes.  The head map layout is dd3d_op_detect's. */
int64_t dd3d_op_detect_c_scratch_bytes(int B, int pre_nms_topk, int num_classes);
int dd3d_op_detect_c(const dd3d_model_desc* h_desc, const float* h_canonical_sizes, int B, const int32_t* h_level_hw /*[5][2]*/,
                     const int32_t* h_strides /*[5]*/, const float* const* d_cls /*[5]*/, const float* const* d_box,
                     const float* const* d_b3d, int cls_pitch, int b3d_pitch, const float* d_intrinsics,
                     const int32_t* d_sizes, void* d_scratch, dd3d_det* d_pre_nms, int32_t* d_pre_counts,
                     dd3d_det* d_out, int32_t* d_counts, int32_t* d_flags /* or NULL */, dd3d_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* DD3D_B200_H_ */
