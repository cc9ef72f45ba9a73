// extern "C" boundary of libdd3d_b200.so (declared in include/dd3d_b200.h).  Plain pointers and sizes only.
#include <stdlib.h>
#include <string.h>

#include <set>
#include <string>

#include "engine.cuh"
#include "model_file.cuh"

using namespace dd3d;

struct dd3d_engine {
    Engine* eng = nullptr;
    std::string err;
    std::set<dd3d_graph_t*> graphs;  // live graphs of this handle: dd3d_destroy detaches them
};

// A captured forward; `h` is null once its handle is destroyed.
struct dd3d_graph_t {
    dd3d_engine* h = nullptr;
    Engine::CapturedForward cf;
    uint64_t generation = 0;  // Engine::generation at the capture
    int device = 0;
};

namespace {

thread_local std::string g_create_error;
int g_op_fp16 = 0;  // element type of the operator-level entry points (dd3d_set_conv_policy("op_fp16", v))

template <typename F>
int guarded(dd3d_handle h, F&& f) {
    try {
        if (h == nullptr || h->eng == nullptr) return DD3D_ERR_INVALID;
        cudaSetDevice(h->eng->device);
        f(*h->eng);
        return DD3D_OK;
    } catch (const EngineError& e) {
        h->err = e.msg;
        return e.status;
    } catch (const std::exception& e) {
        h->err = e.what();
        return DD3D_ERR_INVALID;
    }
}

int cuda_status(cudaError_t e, std::string* err) {
    if (e == cudaSuccess) return DD3D_OK;
    if (err) *err = cudaGetErrorString(e);
    return DD3D_ERR_CUDA;
}

int device_sms() {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

}  // namespace

extern "C" {

int dd3d_create(const dd3d_model_desc* h_desc, dd3d_handle* out) {
    if (h_desc == nullptr || out == nullptr) return DD3D_ERR_INVALID;
    *out = nullptr;
    try {
        dd3d_engine* h = new dd3d_engine();
        h->eng = new Engine(*h_desc);
        *out = h;
        return DD3D_OK;
    } catch (const EngineError& e) {
        g_create_error = e.msg;
        return e.status;
    } catch (const std::exception& e) {
        g_create_error = e.what();
        return DD3D_ERR_INVALID;
    }
}

void dd3d_destroy(dd3d_handle h) {
    if (h == nullptr) return;
    for (dd3d_graph_t* g : h->graphs) g->h = nullptr;  // stale from now on; dd3d_graph_destroy still frees them
    delete h->eng;
    delete h;
}

const char* dd3d_last_error(dd3d_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int dd3d_create_from_file(const char* path, dd3d_handle* out) {
    if (path == nullptr || out == nullptr) return DD3D_ERR_INVALID;
    *out = nullptr;
    ModelFile mf;
    try {
        if (!read_model_file(path, &mf, &g_create_error)) return DD3D_ERR_INVALID;
    } catch (const std::exception& e) {  // std::bad_alloc for a file larger than memory
        g_create_error = std::string("cannot read model file: ") + e.what();
        return DD3D_ERR_INVALID;
    }
    // the calls DD3DB200._engine() makes, in its order
    dd3d_handle h = nullptr;
    int st = dd3d_create(&mf.desc, &h);
    if (st != DD3D_OK) {
        g_create_error = "dd3d_create: " + g_create_error;
        return st;
    }
    std::string call;
    const auto step = [&](const std::string& name, auto&& f) {
        if (st != DD3D_OK) return;
        call = name;
        st = f();
    };
    step("dd3d_set_layout", [&] { return dd3d_set_layout(h, &mf.layout); });
    step("dd3d_set_backbone_norm", [&] { return dd3d_set_backbone_norm(h, mf.backbone_norm); });
    step("dd3d_set_fpn_channels", [&] { return dd3d_set_fpn_channels(h, mf.fpn_channels); });
    if (!mf.fpn_inputs.empty())
        step("dd3d_set_fpn_inputs", [&] { return dd3d_set_fpn_inputs(h, mf.fpn_inputs.data(), int(mf.fpn_inputs.size())); });
    if (!mf.in_features.empty())
        step("dd3d_set_in_features",
             [&] { return dd3d_set_in_features(h, mf.in_features.data(), int(mf.in_features.size())); });
    if (mf.canon_classes > 0)
        step("dd3d_set_canonical_sizes", [&] { return dd3d_set_canonical_sizes(h, mf.canon_classes, mf.canon.data()); });
    std::vector<float> data;  // a record's fp32 data need not be 4-byte aligned in the file
    for (const ModelFileTensor& t : mf.tensors) {
        step("dd3d_load_weight('" + t.name + "')", [&] {
            data.resize(std::max<size_t>(t.count, 1));
            memcpy(data.data(), mf.bytes.data() + t.data_offset, 4 * t.count);
            return dd3d_load_weight(h, t.name.c_str(), data.data(), t.shape.data(), int(t.shape.size()));
        });
    }
    step("dd3d_finalize", [&] { return dd3d_finalize(h); });
    if (st != DD3D_OK) {
        g_create_error = call + ": " + h->err;
        dd3d_destroy(h);
        return st;
    }
    *out = h;
    return DD3D_OK;
}

int dd3d_out_cap(dd3d_handle h) { return (h && h->eng) ? h->eng->desc.out_cap : DD3D_ERR_INVALID; }

int dd3d_size_divisibility(dd3d_handle h) { return (h && h->eng) ? h->eng->size_divisibility() : DD3D_ERR_INVALID; }

int dd3d_set_layout(dd3d_handle h, const dd3d_layout_desc* layout) {
    if (layout == nullptr) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_layout(*layout); });
}

int dd3d_set_backbone_norm(dd3d_handle h, int32_t norm) {
    return guarded(h, [&](Engine& e) { e.set_backbone_norm(norm); });
}

int dd3d_set_fpn_channels(dd3d_handle h, int32_t channels) {
    return guarded(h, [&](Engine& e) { e.set_fpn_channels(channels); });
}

int dd3d_set_fpn_inputs(dd3d_handle h, const int32_t* h_inputs, int n) {
    if (h_inputs == nullptr) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_fpn_inputs(h_inputs, n); });
}

int dd3d_set_in_features(dd3d_handle h, const int32_t* h_fpn_levels, int n) {
    if (h_fpn_levels == nullptr) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_in_features(h_fpn_levels, n); });
}

int dd3d_set_canonical_sizes(dd3d_handle h, int32_t num_classes, const float* h_sizes) {
    if (h_sizes == nullptr) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_canonical_sizes(num_classes, h_sizes); });
}

int dd3d_load_weight(dd3d_handle h, const char* name, const float* data, const int64_t* shape, int ndim) {
    if (name == nullptr || data == nullptr || (ndim > 0 && shape == nullptr) || ndim < 0 || ndim > 8)
        return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.load_weight(name, data, shape, ndim); });
}

int dd3d_finalize(dd3d_handle h) {
    return guarded(h, [&](Engine& e) { e.finalize(); });
}

int64_t dd3d_workspace_bytes(dd3d_handle h, int B, int Hs, int Ws) {
    int64_t bytes = 0;
    int st = guarded(h, [&](Engine& e) { bytes = static_cast<int64_t>(e.workspace_bytes(B, Hs, Ws)); });
    return st == DD3D_OK ? bytes : st;
}

int dd3d_plan(dd3d_handle h, int B, int Hs, int Ws, void* d_workspace, int64_t workspace_bytes) {
    return guarded(h, [&](Engine& e) { e.make_plan(B, Hs, Ws, d_workspace, static_cast<size_t>(workspace_bytes)); });
}

int dd3d_forward(dd3d_handle h, const void* d_images, int img_dtype, const float* d_intrinsics, const int32_t* d_sizes,
                 dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream) {
    if (!d_images || !d_intrinsics || !d_sizes || !d_out || !d_counts) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        e.forward(d_images, img_dtype, d_intrinsics, d_sizes, reinterpret_cast<Det*>(d_out), d_counts, e.user_poses,
                  e.device_agg_args(), static_cast<cudaStream_t>(stream));
    });
}

int dd3d_forward_host(dd3d_handle h, const void* h_images, int img_dtype, const float* h_intrinsics,
                      const int32_t* h_sizes, dd3d_det* h_out, int32_t* h_counts, dd3d_stream stream) {
    if (!h_images || !h_intrinsics || !h_sizes || !h_out || !h_counts) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        e.forward_host(h_images, img_dtype, h_intrinsics, h_sizes, reinterpret_cast<Det*>(h_out), h_counts,
                       static_cast<cudaStream_t>(stream));
    });
}

int dd3d_graph_create(dd3d_handle h, const void* d_images, int img_dtype, const float* d_intrinsics,
                      const int32_t* d_sizes, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream, dd3d_graph* out) {
    if (!out) return DD3D_ERR_INVALID;
    *out = nullptr;
    if (!d_images || !d_intrinsics || !d_sizes || !d_out || !d_counts) return DD3D_ERR_INVALID;
    dd3d_graph_t* g = nullptr;
    const int st = guarded(h, [&](Engine& e) {
        const Engine::CapturedForward cf = e.capture_forward(d_images, img_dtype, d_intrinsics, d_sizes,
                                                             reinterpret_cast<Det*>(d_out), d_counts,
                                                             static_cast<cudaStream_t>(stream));
        g = new dd3d_graph_t{h, cf, e.generation, e.device};
    });
    if (st != DD3D_OK) {
        if (h) g_create_error = h->err;
        return st;
    }
    h->graphs.insert(g);
    *out = g;
    return DD3D_OK;
}

int dd3d_graph_launch(dd3d_graph g, dd3d_stream stream) {
    if (g == nullptr) return DD3D_ERR_INVALID;
    const char* stale = g->h == nullptr                             ? "the handle was destroyed"
                        : g->h->eng->generation != g->generation ? "dd3d_plan or a dd3d_set_* call since the capture"
                                                                  : nullptr;
    std::string err;
    int st = DD3D_OK;
    if (stale) {
        err = std::string("stale graph: ") + stale + "; create a new one";
        st = DD3D_ERR_STATE;
    } else {
        cudaSetDevice(g->device);
        st = cuda_status(cudaGraphLaunch(g->cf.exec, static_cast<cudaStream_t>(stream)), &err);
    }
    if (st != DD3D_OK) {
        g_create_error = err;
        if (g->h) g->h->err = err;
    }
    return st;
}

void dd3d_graph_destroy(dd3d_graph g) {
    if (g == nullptr) return;
    if (g->h) g->h->graphs.erase(g);
    cudaSetDevice(g->device);
    cudaGraphExecDestroy(g->cf.exec);
    delete g;
}

int dd3d_graph_kernel_nodes(dd3d_graph g) { return g ? g->cf.kernel_nodes : DD3D_ERR_INVALID; }

int dd3d_graph_programmatic_edges(dd3d_graph g) { return g ? g->cf.programmatic_edges : DD3D_ERR_INVALID; }

int dd3d_set_conv_policy(const char* name, int value) {
    if (!name) return DD3D_ERR_INVALID;
    if (!strcmp(name, "nms_class_parallel")) {
        nms_set_class_parallel(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "taps")) {
        conv_set_taps(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "wstat")) {
        conv_set_wstat(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "n_split")) {
        conv_set_n_split(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "stagger")) {
        conv_set_stagger(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "pair_tile")) {
        conv_set_pair(value);
        return DD3D_OK;
    }
    if (!strcmp(name, "op_fp16")) {
        g_op_fp16 = value ? 1 : 0;
        return DD3D_OK;
    }
    return DD3D_ERR_INVALID;
}

int dd3d_resize_shape(int h, int w, int min_size, int max_size, int32_t* new_h, int32_t* new_w) {
    if (h < 1 || w < 1 || !new_h || !new_w) return DD3D_ERR_INVALID;
    int nh, nw;
    resize_shortest_edge_shape(h, w, min_size, max_size, &nh, &nw);
    *new_h = nh;
    *new_w = nw;
    return DD3D_OK;
}

int dd3d_forward_raw(dd3d_handle h, const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                     const float* h_intrinsics, int min_size, int max_size, dd3d_det* d_out, int32_t* d_counts,
                     float* h_intrinsics_out, int32_t* h_new_sizes, dd3d_stream stream) {
    if (!d_raw || !h_raw_sizes || !h_intrinsics || !d_out || !d_counts || raw_h < 1 || raw_w < 1) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        e.forward_raw(d_raw, raw_h, raw_w, h_raw_sizes, h_intrinsics, min_size, max_size, reinterpret_cast<Det*>(d_out),
                      d_counts, h_intrinsics_out, h_new_sizes, static_cast<cudaStream_t>(stream));
    });
}

int dd3d_submit_host(dd3d_handle h, int slot, const void* h_images, int img_dtype, const float* h_intrinsics,
                     const int32_t* h_sizes, dd3d_det* h_out, int32_t* h_counts, dd3d_stream stream) {
    if (!h_images || !h_intrinsics || !h_sizes || !h_out || !h_counts) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        e.submit_host(slot, h_images, img_dtype, h_intrinsics, h_sizes, reinterpret_cast<Det*>(h_out), h_counts,
                      static_cast<cudaStream_t>(stream));
    });
}

int dd3d_wait_host(dd3d_handle h, int slot) {
    return guarded(h, [&](Engine& e) { e.wait_host(slot); });
}

int dd3d_overflow_flags(dd3d_handle h, dd3d_stream stream, int32_t* h_flags) {
    return guarded(h, [&](Engine& e) {
        if (!e.plan.valid) throw EngineError(DD3D_ERR_STATE, "no plan");
        cudaError_t c = cudaMemcpyAsync(h_flags, e.plan.decode.flags, 4, cudaMemcpyDeviceToHost,
                                        static_cast<cudaStream_t>(stream));
        if (c == cudaSuccess) c = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
        if (c != cudaSuccess) throw EngineError(DD3D_ERR_CUDA, cudaGetErrorString(c));
    });
}

int dd3d_copy_flags(dd3d_handle h, int32_t* d_dst, dd3d_stream stream) {
    if (!d_dst) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        if (!e.plan.valid) throw EngineError(DD3D_ERR_STATE, "no plan");
        cudaError_t c = cudaMemcpyAsync(d_dst, e.plan.decode.flags, 4, cudaMemcpyDeviceToDevice,
                                        static_cast<cudaStream_t>(stream));
        if (c != cudaSuccess) throw EngineError(DD3D_ERR_CUDA, cudaGetErrorString(c));
    });
}

int dd3d_set_option(dd3d_handle h, const char* name, int value) {
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        const std::string n(name ? name : "");
        if (n == "do_postprocess") {
            e.opt_do_postprocess = value ? 1 : 0;
        } else if (n == "do_nms") {
            // without NMS up to L * PRE_NMS_TOPK detections per image survive (L head levels): refuse a buffer that would
            // truncate them
            const int L = e.num_levels();
            if (!value && e.desc.out_cap < L * e.desc.pre_nms_topk)
                throw EngineError(DD3D_ERR_INVALID, "do_nms = 0 needs out_cap >= " + std::to_string(L) + " * pre_nms_topk (" +
                                                        std::to_string(L * e.desc.pre_nms_topk) + "), engine has " +
                                                        std::to_string(e.desc.out_cap) + ": recreate the engine");
            e.set_do_nms(value ? 1 : 0);
        } else if (n == "profile") {
            e.opt_profile = value ? 1 : 0;
        } else if (n == "workspace_reuse") {  // applies to plans made afterwards
            e.opt_workspace_reuse = value ? 1 : 0;
        } else if (n == "sparse_box3d") {  // 2 (default): auto by head size; 1: always sparse; 0: dense fp32 maps
            const int v = value < 0 ? 0 : (value > 2 ? 2 : value);
            if (e.opt_sparse_box3d != v) e.drop_plans();
            e.opt_sparse_box3d = v;
        } else if (n == "sparse_tower") {  // 2 (default): auto by head size; 1: with every sparse predictor; 0: dense tower
            const int v = value < 0 ? 0 : (value > 2 ? 2 : value);
            if (e.opt_sparse_tower != v) e.drop_plans();
            e.opt_sparse_tower = v;
        } else if (n == "sparse_box2d_tower") {  // 2 (default): auto with the sparse predictor; 1: whenever eligible; 0: dense
            const int v = value < 0 ? 0 : (value > 2 ? 2 : value);
            if (e.opt_sparse_box2d_tower != v) e.drop_plans();
            e.opt_sparse_box2d_tower = v;
        } else if (n == "workspace_fill") {
            e.opt_workspace_fill = (value >= 0 && value <= 255) ? value : -1;
        } else {
            throw EngineError(DD3D_ERR_INVALID, "unknown option: " + n);
        }
    });
}

int dd3d_set_bev_nms(dd3d_handle h, int enable, float iou_thresh) {
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        e.set_bev_nms(enable, iou_thresh);
    });
}

int dd3d_set_poses(dd3d_handle h, const float* d_poses) {
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        e.user_poses = d_poses;
    });
}

int dd3d_set_host_poses(dd3d_handle h, int slot, const float* h_poses) {
    if (!h_poses) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_host_poses(slot, h_poses); });
}

int dd3d_bev_nms_path(const dd3d_model_desc* h_desc) {
    if (!h_desc) return DD3D_ERR_INVALID;
    return bev_nms_path(h_desc->do_nms, h_desc->post_nms_topk);
}

int dd3d_set_sample_aggregate(dd3d_handle h, int enable, float iou_thresh, int max_dets) {
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        e.set_sample_aggregate(enable, iou_thresh, max_dets);
    });
}

int dd3d_set_groups(dd3d_handle h, const int32_t* d_group, int num_groups) {
    if (d_group && num_groups < 1) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        e.user_groups = d_group;
        e.user_num_groups = d_group ? num_groups : 0;
    });
}

int dd3d_set_host_groups(dd3d_handle h, int slot, const int32_t* h_group, int num_groups) {
    if (!h_group) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.set_host_groups(slot, h_group, num_groups); });
}

int dd3d_set_global_out(dd3d_handle h, float* d_global) {
    return guarded(h, [&](Engine& e) {
        ++e.generation;
        e.user_global = d_global;
    });
}

int dd3d_set_host_global_out(dd3d_handle h, int slot, float* h_global) {
    return guarded(h, [&](Engine& e) {
        if (slot < 0 || slot > 1) throw EngineError(DD3D_ERR_INVALID, "slot must be 0 or 1");
        if (e.slot_busy[slot]) throw EngineError(DD3D_ERR_STATE, "slot has a pending dd3d_submit_host");
        e.host_global[slot] = h_global;
    });
}

int dd3d_sample_aggregate_path(const dd3d_model_desc* h_desc) {
    if (!h_desc) return DD3D_ERR_INVALID;
    return sample_aggregate_path(h_desc->do_nms, h_desc->post_nms_topk, h_desc->out_cap);
}

int dd3d_num_ops(dd3d_handle h) {
    int n = 0;
    int st = guarded(h, [&](Engine& e) {
        if (!e.plan.valid) throw EngineError(DD3D_ERR_STATE, "no plan");
        n = static_cast<int>(e.plan.ops.size());
    });
    return st == DD3D_OK ? n : st;
}

int dd3d_launches_per_forward(dd3d_handle h) {
    int n = 0;
    int st = guarded(h, [&](Engine& e) { n = e.launches_per_forward(); });
    return st == DD3D_OK ? n : st;
}

int dd3d_get_profile(dd3d_handle h, double* h_ms, double* h_flops, double* h_bytes, int32_t* h_launches) {
    if (!h_ms || !h_flops || !h_bytes || !h_launches) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) { e.get_profile(h_ms, h_flops, h_bytes, h_launches); });
}

int dd3d_get_op_times(dd3d_handle h, float* h_ms, int32_t* h_cats, double* h_flops, int32_t* h_ops, int max_ops) {
    if (!h_ms || !h_cats || !h_flops || max_ops < 1) return DD3D_ERR_INVALID;
    int n = 0;
    int st = guarded(h, [&](Engine& e) { n = e.get_op_times(h_ms, h_cats, h_flops, h_ops, max_ops); });
    return st == DD3D_OK ? n : st;
}

int dd3d_get_conv_info(dd3d_handle h, int32_t* h_info, int max_ops) {
    if (!h_info || max_ops < 1) return DD3D_ERR_INVALID;
    int n = 0;
    int st = guarded(h, [&](Engine& e) {
        if (!e.plan.valid) throw EngineError(DD3D_ERR_STATE, "no plan");
        for (const Op& op : e.plan.ops) {
            if (n == max_ops) break;
            int32_t* r = h_info + 8 * n++;
            for (int i = 0; i < 8; ++i) r[i] = 0;
            if (op.type != Op::CONV) continue;
            const ConvParams& p = op.conv;
            const int v[8] = {p.grouped ? 2 : 1, p.taps, p.stride, p.cin, p.block_n * p.n_blocks, p.halo ? 1 : 0, p.pair, p.block_n};
            for (int i = 0; i < 8; ++i) r[i] = v[i];
        }
    });
    return st == DD3D_OK ? n : st;
}

int dd3d_get_tensor(dd3d_handle h, const char* name, void** d_ptr, int32_t dims[6]) {
    return guarded(h, [&](Engine& e) {
        if (!e.plan.valid) throw EngineError(DD3D_ERR_STATE, "no plan");
        const Plan& P = e.plan;
        const std::string n(name ? name : "");
        auto level = [&](size_t prefix_len) {
            const int l = n.size() == prefix_len + 1 ? n[prefix_len] - '0' : -1;
            if (l < 0 || l >= kLevels) throw EngineError(DD3D_ERR_INVALID, "unknown tensor: " + n);
            return l;
        };
        auto position = [&](size_t prefix_len) {  // head maps: by DD3D.IN_FEATURES position
            const int l = level(prefix_len);
            if (l >= P.num_levels) throw EngineError(DD3D_ERR_INVALID, "unknown tensor: " + n + " (head levels: " +
                                                                            std::to_string(P.num_levels) + ")");
            return l;
        };
        if (n.rfind("op", 0) == 0) {  // "op<i>" / "op<i>:<seg>": bf16 output view of engine op i (launch order)
            const size_t colon = n.find(':');
            const int i = atoi(n.substr(2, colon == std::string::npos ? std::string::npos : colon - 2).c_str());
            const int sg = colon == std::string::npos ? 0 : atoi(n.substr(colon + 1).c_str());
            if (i < 0 || i >= static_cast<int>(P.ops.size()) || sg < 0 || sg >= P.ops[i].nouts)
                throw EngineError(DD3D_ERR_INVALID, "no such op output: " + n);
            const View& v = P.ops[i].outs[sg];
            *d_ptr = v.ptr;
            const int32_t d[6] = {v.B, v.H, v.W, v.C, v.pitch, 2};
            memcpy(dims, d, sizeof(d));
        } else if (n == "input") {
            *d_ptr = P.input.ptr;
            const int32_t d[6] = {P.B, P.Hp, P.Wp, 4, 4, 2};
            memcpy(dims, d, sizeof(d));
        } else if (n[0] == 'p') {  // "p<i>": FPN output i, i < the FPN's output count
            const int l = n.size() == 2 ? n[1] - '0' : -1;
            if (l < 0 || l >= e.fpn_outputs()) throw EngineError(DD3D_ERR_INVALID, "unknown tensor: " + n);
            const View& v = P.fpn[l];
            if (v.ptr == nullptr) throw EngineError(DD3D_ERR_INVALID, "FPN output " + n + " is not built: no head reads it");
            *d_ptr = v.ptr;
            const int32_t d[6] = {v.B, v.H, v.W, v.C, v.pitch, 2};
            memcpy(dims, d, sizeof(d));
        } else if (n.rfind("cls", 0) == 0) {
            const int l = position(3);
            *d_ptr = P.cls_map[l];
            const int32_t d[6] = {P.B, P.lvl_h[l], P.lvl_w[l], e.desc.num_classes, P.cls_pitch, 4};
            memcpy(dims, d, sizeof(d));
        } else if (n.rfind("box", 0) == 0) {
            const int l = position(3);
            if (P.box2d_begin >= 0)
                throw EngineError(DD3D_ERR_INVALID, "the box2d map is computed only around the pixels that pass the threshold "
                                                    "with option sparse_box2d_tower: " + n);
            *d_ptr = P.box_map[l];
            const int32_t d[6] = {P.B, P.lvl_h[l], P.lvl_w[l], 5, 16, 4};
            memcpy(dims, d, sizeof(d));
        } else if (n.rfind("b3d", 0) == 0) {
            const int l = position(3);
            if (P.b3d_map[l] == nullptr)
                throw EngineError(DD3D_ERR_INVALID, P.sparse_b3d ? "dense box3d maps are not computed with option sparse_box3d = 1: " + n
                                                                 : "no 3-D head (box3d_on = 0): " + n);
            *d_ptr = P.b3d_map[l];
            const int32_t d[6] = {P.B, P.lvl_h[l], P.lvl_w[l], 11 * (e.desc.class_agnostic_box3d ? 1 : e.desc.num_classes),
                                  P.b3d_pitch, 4};
            memcpy(dims, d, sizeof(d));
        } else {
            throw EngineError(DD3D_ERR_INVALID, "unknown tensor: " + n);
        }
    });
}

// ------------------------------------------------------------------------------------------------ operators

// Repacks the 3x3 weights [16][9][cin_pad] into the taps-in-N layout [9 * 16][cin_pad] in a new device buffer *d_w_taps
// (the caller frees it after the launch has run; operator entry points only, not a hot path) and encodes its tensor map.
static bool taps_weights(const void* d_w, int cin_pad, CUtensorMap* map, void** d_w_taps, cudaStream_t stream) {
    if (cudaMalloc(d_w_taps, static_cast<size_t>(kTapsN) * cin_pad * 2) != cudaSuccess) return false;
    for (int t = 0; t < 9; ++t)
        cudaMemcpy2DAsync(static_cast<uint8_t*>(*d_w_taps) + static_cast<size_t>(t) * 16 * cin_pad * 2, cin_pad * 2,
                          static_cast<const uint8_t*>(d_w) + static_cast<size_t>(t) * cin_pad * 2, 9 * cin_pad * 2,
                          cin_pad * 2, 16, cudaMemcpyDeviceToDevice, stream);
    if (!make_weight_map_taps(map, *d_w_taps, cin_pad, g_op_fp16)) {
        cudaStreamSynchronize(stream);
        cudaFree(*d_w_taps);
        return false;
    }
    return true;
}

int dd3d_op_conv2d(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout, int ksize,
                   int stride, const float* d_scale, const float* d_bias, int relu, const void* d_residual,
                   int res_pitch, int res_up2, void* d_out, int out_pitch, int out_f32, dd3d_stream stream) {
    if (!d_in || !d_w || !d_scale || !d_bias || !d_out) return DD3D_ERR_INVALID;
    if ((ksize != 1 && ksize != 3) || (stride != 1 && stride != 2) || (stride == 2 && ksize != 3)) return DD3D_ERR_INVALID;
    if (stride == 2 && ((H | W) & 1)) return DD3D_ERR_INVALID;
    ConvParams p;
    memset(&p, 0, sizeof(p));
    const int kchunks = (cin + kBlockK - 1) / kBlockK;
    const int taps = ksize * ksize;
    const int cout_pad = (cout + 15) / 16 * 16;
    const int block_n = conv_block_n(cout_pad);
    if (block_n == 0) return DD3D_ERR_INVALID;
    if (!out_f32 && cout % 16) return DD3D_ERR_INVALID;
    p.nseg = 1;
    p.B = B;
    p.taps = taps;
    p.stride = stride;
    p.kchunks = kchunks;
    p.cin = cin;
    p.n_blocks = cout_pad / block_n;
    p.block_n = block_n;
    p.relu = relu;
    p.out_mode = out_f32 ? 1 : 0;
    p.fp16 = g_op_fp16;
    ConvSeg& g = p.seg[0];
    const int Ho = H / stride, Wo = W / stride;
    g.H = Ho;
    g.W = Wo;
    choose_tile(Ho, Wo, &g.th, &g.tw);
    bool ok = true;
    p.halo = conv_prefer_halo(taps, stride, block_n, 1, &Ho, &Wo) ? 1 : 0;
    if (p.halo) {
        g.th = kHaloTh;
        g.tw = kHaloTw;
        ok = ok && make_act_map_halo(&g.in_map[0], d_in, B, H, W, cin, in_pitch, g_op_fp16);
    } else if (stride == 1) {
        ok = ok && make_act_map(&g.in_map[0], d_in, B, H, W, cin, in_pitch, g.th, g.tw, g_op_fp16);
    } else {
        ok = ok && make_act_map_s2(&g.in_map[0], d_in, 0, B, H, W, cin, in_pitch, g.th, g.tw, g_op_fp16) &&
             make_act_map_s2(&g.in_map[1], d_in, 1, B, H, W, cin, in_pitch, g.th, g.tw, g_op_fp16);
    }
    if (!out_f32) ok = ok && make_out_map(&g.out_map, d_out, B, Ho, Wo, cout, out_pitch, g.tw, g_op_fp16);
    if (!ok) {
        fprintf(stderr, "dd3d_op_conv2d: %s\n", conv_last_error());
        return DD3D_ERR_CUDA;
    }
    g.scale = d_scale;
    g.bias = d_bias;
    g.lo = nullptr;
    g.out_f32 = static_cast<float*>(out_f32 ? d_out : nullptr);
    g.out_pitch = out_pitch;
    if (d_residual) {
        g.residual = static_cast<const __nv_bfloat16*>(d_residual);
        g.res_pitch = res_pitch;
        g.res_up2 = res_up2;
        g.res_H = res_up2 ? Ho / 2 : Ho;
        g.res_W = res_up2 ? Wo / 2 : Wo;
    }
    p.taps_n = conv_taps_eligible(taps, stride, cout_pad, 1, &Ho, &Wo) ? 1 : 0;
    if (!out_f32) g.out16 = d_out;
    conv_select_pair(&p, cout_pad, device_sms());
    conv_finalize_params(&p);
    void* d_w_taps = nullptr;
    if (p.taps_n) {
        if (!taps_weights(d_w, kchunks * kBlockK, &p.w_map, &d_w_taps, static_cast<cudaStream_t>(stream))) return DD3D_ERR_CUDA;
    } else if (!make_weight_map(&p.w_map, d_w, taps * kchunks * kBlockK, cout_pad, p.block_n, g_op_fp16)) {
        fprintf(stderr, "dd3d_op_conv2d: %s\n", conv_last_error());
        return DD3D_ERR_CUDA;
    }
    const int st = cuda_status(launch_conv(p, device_sms(), static_cast<cudaStream_t>(stream)), nullptr);
    if (d_w_taps) {
        cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
        cudaFree(d_w_taps);
    }
    return st;
}

int dd3d_op_conv2d_grouped(const void* d_in, int B, int H, int W, int C, int in_pitch, const void* d_w, int groups,
                           int stride, const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch,
                           dd3d_stream stream) {
    if (!d_in || !d_w || !d_scale || !d_bias || !d_out) return DD3D_ERR_INVALID;
    if (B < 1 || H < 1 || W < 1 || C < kBlockK || C % kBlockK || groups < 1 || C % groups || kBlockK % (C / groups) ||
        in_pitch < C || out_pitch < C || (in_pitch | out_pitch) & 7)
        return DD3D_ERR_INVALID;
    if ((stride != 1 && stride != 2) || (stride == 2 && ((H | W) & 1))) return DD3D_ERR_INVALID;
    ConvParams p;
    memset(&p, 0, sizeof(p));
    p.nseg = 1;
    p.B = B;
    p.taps = 9;
    p.stride = stride;
    p.kchunks = 1;
    p.cin = C;
    p.block_n = kBlockK;
    p.n_blocks = C / kBlockK;
    p.relu = relu;
    p.fp16 = g_op_fp16;
    p.grouped = 1;
    ConvSeg& g = p.seg[0];
    const int Ho = H / stride, Wo = W / stride;
    g.H = Ho;
    g.W = Wo;
    choose_tile(Ho, Wo, &g.th, &g.tw);
    bool ok = true;
    p.halo = conv_prefer_halo(9, stride, kBlockK, 1, &Ho, &Wo) ? 1 : 0;
    if (p.halo) {
        g.th = kHaloTh;
        g.tw = kHaloTw;
        ok = make_act_map_halo(&g.in_map[0], d_in, B, H, W, C, in_pitch, g_op_fp16);
    } else if (stride == 1) {
        ok = make_act_map(&g.in_map[0], d_in, B, H, W, C, in_pitch, g.th, g.tw, g_op_fp16);
    } else {
        ok = make_act_map_s2(&g.in_map[0], d_in, 0, B, H, W, C, in_pitch, g.th, g.tw, g_op_fp16) &&
             make_act_map_s2(&g.in_map[1], d_in, 1, B, H, W, C, in_pitch, g.th, g.tw, g_op_fp16);
    }
    ok = ok && make_out_map(&g.out_map, d_out, B, Ho, Wo, C, out_pitch, g.tw, g_op_fp16) &&
         make_weight_map(&p.w_map, d_w, 9 * kBlockK, C, kBlockK, g_op_fp16);
    if (!ok) {
        fprintf(stderr, "dd3d_op_conv2d_grouped: %s\n", conv_last_error());
        return DD3D_ERR_CUDA;
    }
    g.scale = d_scale;
    g.bias = d_bias;
    g.out16 = d_out;
    g.out_pitch = out_pitch;
    conv_finalize_params(&p);
    return cuda_status(launch_conv(p, device_sms(), static_cast<cudaStream_t>(stream)), nullptr);
}

// the work-list pair tile on tiles th x 8 (th = 16: dd3d_op_conv2d_tiles, kListTile: dd3d_op_conv2d_tiles8x8)
static int conv2d_tiles(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                        const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch, const uint32_t* d_tiles,
                        const int32_t* d_count, dd3d_stream stream, int th) {
    if (!d_in || !d_w || !d_scale || !d_bias || !d_out || !d_tiles || !d_count) return DD3D_ERR_INVALID;
    if (B < 1 || B > kTileListMaxImages || H < 1 || W < 1 || cin < 1 || in_pitch < cin || cout < 128 || cout % 128 ||
        out_pitch < cout)
        return DD3D_ERR_INVALID;
    ConvParams p;
    memset(&p, 0, sizeof(p));
    const int kchunks = (cin + kBlockK - 1) / kBlockK;
    p.nseg = 1;
    p.B = B;
    p.taps = 9;
    p.stride = 1;
    p.kchunks = kchunks;
    p.cin = cin;
    p.relu = relu;
    p.fp16 = g_op_fp16;
    // the pair tile in work-list mode, whatever the pair / halo policies choose for dd3d_op_conv2d
    p.halo = 1;
    p.pair = 1;
    p.block_n = 128;
    p.n_blocks = cout / 128;
    p.tile_list = d_tiles;
    p.tile_count = d_count;
    ConvSeg& g = p.seg[0];
    g.H = H;
    g.W = W;
    g.th = th;
    g.tw = kListTile;
    if (((H + th - 1) / th) * ((W + kListTile - 1) / kListTile) >= kTileListMaxTiles) return DD3D_ERR_INVALID;
    if (!make_act_map(&g.in_map[0], d_in, B, H, W, cin, in_pitch, kListTile + 2, kListTile + 2, g_op_fp16) ||
        !make_out_map(&g.out_map, d_out, B, H, W, cout, out_pitch, g.tw, g_op_fp16) ||
        !make_weight_map(&p.w_map, d_w, 9 * kchunks * kBlockK, cout, p.block_n, g_op_fp16)) {
        fprintf(stderr, "dd3d_op_conv2d_tiles: %s\n", conv_last_error());
        return DD3D_ERR_CUDA;
    }
    g.scale = d_scale;
    g.bias = d_bias;
    g.out_pitch = out_pitch;
    conv_finalize_params(&p);
    const cudaError_t e = launch_conv(p, device_sms(), static_cast<cudaStream_t>(stream));
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int dd3d_op_conv2d_tiles(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                         const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch, const uint32_t* d_tiles,
                         const int32_t* d_count, dd3d_stream stream) {
    return conv2d_tiles(d_in, B, H, W, cin, in_pitch, d_w, cout, d_scale, d_bias, relu, d_out, out_pitch, d_tiles, d_count,
                        stream, 2 * kListTile);
}

int dd3d_op_conv2d_tiles8x8(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                            const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch,
                            const uint32_t* d_tiles, const int32_t* d_count, dd3d_stream stream) {
    return conv2d_tiles(d_in, B, H, W, cin, in_pitch, d_w, cout, d_scale, d_bias, relu, d_out, out_pitch, d_tiles, d_count,
                        stream, kListTile);
}

int dd3d_op_conv2d_taps_tiles(const void* d_in, int B, int H, int W, int cin, int in_pitch, const void* d_w, int cout,
                              const float* d_scale, const float* d_bias, int relu, void* d_out, int out_pitch, int out_f32,
                              const uint32_t* d_tiles, const int32_t* d_count, dd3d_stream stream) {
    if (!d_in || !d_w || !d_scale || !d_bias || !d_out || !d_tiles || !d_count) return DD3D_ERR_INVALID;
    if (B < 1 || B > kTileListMaxImages || H < 1 || W < 1 || cin < 1 || in_pitch < cin || cout < 1 || cout > 16 ||
        out_pitch < 16 || (out_f32 ? out_pitch % 4 : out_pitch % 8))
        return DD3D_ERR_INVALID;
    if (((H + kHaloTh - 1) / kHaloTh) * ((W + kHaloTw - 1) / kHaloTw) >= kTileListMaxTiles) return DD3D_ERR_INVALID;
    ConvParams p;
    memset(&p, 0, sizeof(p));
    const int kchunks = (cin + kBlockK - 1) / kBlockK;
    p.nseg = 1;
    p.B = B;
    p.taps = 9;
    p.stride = 1;
    p.kchunks = kchunks;
    p.cin = cin;
    p.n_blocks = 1;
    p.block_n = 16;
    p.relu = relu;
    p.out_mode = out_f32 ? 1 : 0;
    p.fp16 = g_op_fp16;
    // the taps-in-N kernel in work-list mode, whatever the taps / halo policies choose for dd3d_op_conv2d
    p.halo = 1;
    p.taps_n = 1;
    p.tile_list = d_tiles;
    p.tile_count = d_count;
    ConvSeg& g = p.seg[0];
    g.H = H;
    g.W = W;
    g.th = kHaloTh;
    g.tw = kHaloTw;
    if (!make_act_map_halo(&g.in_map[0], d_in, B, H, W, cin, in_pitch, g_op_fp16)) {
        fprintf(stderr, "dd3d_op_conv2d_taps_tiles: %s\n", conv_last_error());
        return DD3D_ERR_CUDA;
    }
    g.scale = d_scale;
    g.bias = d_bias;
    g.out_pitch = out_pitch;
    if (out_f32)
        g.out_f32 = static_cast<float*>(d_out);
    else
        g.out16 = d_out;
    conv_finalize_params(&p);
    void* d_w_taps = nullptr;
    if (!taps_weights(d_w, kchunks * kBlockK, &p.w_map, &d_w_taps, static_cast<cudaStream_t>(stream))) return DD3D_ERR_CUDA;
    const cudaError_t e = launch_conv(p, device_sms(), static_cast<cudaStream_t>(stream));
    cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
    cudaFree(d_w_taps);
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int dd3d_op_b3d_sparse_c(const void* const* d_in, const int32_t* h_level_hw, const int32_t* h_pitch, const void* const* d_w,
                         const float* const* d_scale, const float* const* d_bias, const void* d_fin, const int32_t* d_counts,
                         int B, int C, int topk, int n_pad, float* d_rows, int out_pitch, int cin, dd3d_stream stream) {
    if (!d_in || !h_level_hw || !h_pitch || !d_w || !d_scale || !d_bias || !d_fin || !d_counts || !d_rows) return DD3D_ERR_INVALID;
    if (B < 1 || C < 1 || topk < 1 || cin < 1) return DD3D_ERR_INVALID;
    B3dSparseParams p;
    memset(&p, 0, sizeof(p));
    for (int l = 0; l < kLevels; ++l) {
        B3dSparseLevel& v = p.lvl[l];
        v.in = static_cast<const __nv_bfloat16*>(d_in[l]);
        v.w = static_cast<const __nv_bfloat16*>(d_w[l]);
        v.scale = d_scale[l];
        v.bias = d_bias[l];
        v.H = h_level_hw[2 * l];
        v.W = h_level_hw[2 * l + 1];
        v.pitch = h_pitch[l];
        if (!v.scale || !v.bias || v.H < 1 || v.W < 1 || v.pitch < cin) return DD3D_ERR_INVALID;
    }
    p.fin = static_cast<const uint2*>(d_fin);
    p.cand_count = d_counts;
    p.rows = d_rows;
    p.num_levels = kLevels;
    p.B = B;
    p.C = C;
    p.topk = topk;
    p.n_pad = n_pad;
    p.out_pitch = out_pitch;
    p.fp16 = g_op_fp16;
    p.cin = cin;
    const cudaError_t e = launch_b3d_sparse(p, static_cast<cudaStream_t>(stream));
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int64_t dd3d_op_b3d_gather_scratch_bytes(int B, int C, int topk) {
    if (B < 1 || C < 1 || C > kB3dGatherMaxC || topk < 1) return DD3D_ERR_INVALID;
    return static_cast<int64_t>(b3d_gather_scratch_bytes(B, C, topk));
}

int dd3d_op_b3d_gather(const void* const* d_in, const int32_t* h_level_hw, const int32_t* h_pitch, const void* const* d_w,
                       const float* const* d_scale, const float* const* d_bias, const void* d_fin, const int32_t* d_counts,
                       int B, int C, int topk, int cin, float* d_rows, void* d_scratch, dd3d_stream stream) {
    if (!d_in || !h_level_hw || !h_pitch || !d_w || !d_scale || !d_bias || !d_fin || !d_counts || !d_rows || !d_scratch)
        return DD3D_ERR_INVALID;
    if (B < 1 || C < 1 || C > kB3dGatherMaxC || topk < 1 || cin < 1) return DD3D_ERR_INVALID;
    B3dGatherParams p;
    memset(&p, 0, sizeof(p));
    for (int l = 0; l < kLevels; ++l) {
        B3dSparseLevel& v = p.lvl[l];
        v.in = static_cast<const __nv_bfloat16*>(d_in[l]);
        v.w = static_cast<const __nv_bfloat16*>(d_w[l]);
        v.scale = d_scale[l];
        v.bias = d_bias[l];
        v.H = h_level_hw[2 * l];
        v.W = h_level_hw[2 * l + 1];
        v.pitch = h_pitch[l];
        if (!v.scale || !v.bias || v.H < 1 || v.W < 1 || v.pitch < cin) return DD3D_ERR_INVALID;
    }
    p.fin = static_cast<const uint2*>(d_fin);
    p.cand_count = d_counts;
    p.rows = d_rows;
    p.num_levels = kLevels;
    p.B = B;
    p.C = C;
    p.topk = topk;
    p.fp16 = g_op_fp16;
    p.cin = cin;
    b3d_gather_bind_scratch(&p, d_scratch);
    const cudaError_t e = launch_b3d_gather(p, static_cast<cudaStream_t>(stream));
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int dd3d_op_b3d_sparse(const void* const* d_in, const int32_t* h_level_hw, const int32_t* h_pitch, const void* const* d_w,
                       const float* const* d_scale, const float* const* d_bias, const void* d_fin, const int32_t* d_counts,
                       int B, int C, int topk, int n_pad, float* d_rows, int out_pitch, dd3d_stream stream) {
    return dd3d_op_b3d_sparse_c(d_in, h_level_hw, h_pitch, d_w, d_scale, d_bias, d_fin, d_counts, B, C, topk, n_pad, d_rows,
                                out_pitch, 256, stream);
}

int dd3d_op_dla_front(const void* d_in4, const void* d_w0, const void* d_w1, const void* d_w2, const float* d_sb0,
                      const float* d_sb1, const float* d_sb2, void* d_out, int out_pitch, void* d_pool, int pool_pitch,
                      int B, int H, int W, dd3d_stream stream) {
    using bf = __nv_bfloat16;
    return cuda_status(launch_dla_front(static_cast<const bf*>(d_in4), static_cast<const bf*>(d_w0), static_cast<const bf*>(d_w1),
                                        static_cast<const bf*>(d_w2), d_sb0, d_sb1, d_sb2, static_cast<bf*>(d_out), out_pitch,
                                        static_cast<bf*>(d_pool), pool_pitch, B, H, W, device_sms(),
                                        static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int dd3d_op_stem_s2_mma(const void* d_in4, const void* d_w, const float* d_sb, void* d_out, int out_pitch, int B, int H, int W,
                        dd3d_stream stream) {
    return cuda_status(launch_stem_s2_mma(static_cast<const __nv_bfloat16*>(d_in4), static_cast<const __nv_bfloat16*>(d_w), d_sb,
                                          static_cast<__nv_bfloat16*>(d_out), out_pitch, B, H, W, device_sms(),
                                          static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int dd3d_op_dwconv3x3(const void* d_in, int B, int H, int W, int C, int in_pitch, const void* d_w, int stride, void* d_out,
                      int out_pitch, dd3d_stream stream) {
    if (!d_in || !d_w || !d_out) return DD3D_ERR_INVALID;
    return cuda_status(launch_dwconv3x3(static_cast<const __nv_bfloat16*>(d_in), B, H, W, C, in_pitch,
                                        static_cast<const __nv_bfloat16*>(d_w), stride, static_cast<__nv_bfloat16*>(d_out),
                                        out_pitch, static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int64_t dd3d_op_group_norm_scratch_bytes(int B, int H, int W) {
    if (B < 1 || H < 1 || W < 1) return DD3D_ERR_INVALID;
    return static_cast<int64_t>(group_norm_scratch_bytes(B, H, W));
}

int dd3d_op_group_norm(const void* d_in, int B, int H, int W, int in_pitch, const float* d_gamma, const float* d_beta, int relu,
                       const void* d_residual, int res_pitch, int avg, void* d_out, int out_pitch, void* d_scratch,
                       dd3d_stream stream) {
    if (!d_in || !d_out || (d_gamma == nullptr) != (d_beta == nullptr) || (d_gamma && !d_scratch)) return DD3D_ERR_INVALID;
    if (B < 1 || H < 1 || W < 1) return DD3D_ERR_INVALID;
    GroupNormParams p;
    p.nseg = 1;
    p.B = B;
    p.gamma = d_gamma;
    p.beta = d_beta;
    p.relu = relu ? 1 : 0;
    p.avg = avg ? 1 : 0;
    p.fp16 = g_op_fp16;
    GroupNormSeg& g = p.seg[0];
    g.in = static_cast<const __nv_bfloat16*>(d_in);
    g.out = static_cast<__nv_bfloat16*>(d_out);
    g.H = H;
    g.W = W;
    g.in_pitch = in_pitch;
    g.out_pitch = out_pitch;
    if (d_residual) {
        g.res = static_cast<const __nv_bfloat16*>(d_residual);
        g.res_pitch = res_pitch;
        g.res_H = (H + 1) / 2;
        g.res_W = (W + 1) / 2;
    }
    g.part = static_cast<float2*>(d_scratch);
    const cudaError_t e = launch_group_norm(p, static_cast<cudaStream_t>(stream));
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int dd3d_op_group_norm_c(const void* d_in, int B, int H, int W, int C, int in_c0, int in_pitch, const float* d_gamma,
                         const float* d_beta, int relu, void* d_out, int out_c0, int out_pitch, void* d_scratch, dd3d_stream stream) {
    if (!d_in || !d_out || !d_gamma || !d_beta || !d_scratch) return DD3D_ERR_INVALID;
    if (B < 1 || H < 1 || W < 1 || in_c0 < 0 || out_c0 < 0 || in_c0 % 8 || out_c0 % 8) return DD3D_ERR_INVALID;
    if (in_c0 + C > in_pitch || out_c0 + C > out_pitch) return DD3D_ERR_INVALID;
    GroupNormParams p;
    p.nseg = 1;
    p.B = B;
    p.C = C;
    p.gamma = d_gamma;
    p.beta = d_beta;
    p.relu = relu ? 1 : 0;
    p.fp16 = g_op_fp16;
    GroupNormSeg& g = p.seg[0];
    g.in = static_cast<const __nv_bfloat16*>(d_in) + in_c0;
    g.out = static_cast<__nv_bfloat16*>(d_out) + out_c0;
    g.H = H;
    g.W = W;
    g.in_pitch = in_pitch;
    g.out_pitch = out_pitch;
    g.part = static_cast<float2*>(d_scratch);
    const cudaError_t e = launch_group_norm(p, static_cast<cudaStream_t>(stream));
    return e == cudaErrorInvalidValue ? DD3D_ERR_INVALID : cuda_status(e, nullptr);
}

int dd3d_op_preprocess(const void* d_images, int img_dtype, const int32_t* d_sizes2, void* d_out4, int B, int Hs, int Ws,
                       int Hp, int Wp, const float* h_mean, const float* h_std, dd3d_stream stream) {
    return cuda_status(launch_preprocess(d_images, img_dtype == DD3D_IMG_U8, d_sizes2, 2, static_cast<__nv_bfloat16*>(d_out4),
                                         B, Hs, Ws, Hp, Wp, h_mean, h_std, static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int dd3d_op_maxpool(const void* d_in, void* d_out, int B, int H, int W, int C, int in_pitch, int out_pitch, int ksize,
                    dd3d_stream stream) {
    if (C % 8 || (ksize != 2 && ksize != 3)) return DD3D_ERR_INVALID;
    const int Ho = ksize == 2 ? H / 2 : (H - 3 + 1) / 2 + 1;
    const int Wo = ksize == 2 ? W / 2 : (W - 3 + 1) / 2 + 1;
    return cuda_status(launch_maxpool(static_cast<const __nv_bfloat16*>(d_in), static_cast<__nv_bfloat16*>(d_out), B, H,
                                      W, C, in_pitch, Ho, Wo, out_pitch, ksize, device_sms(),
                                      static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int64_t dd3d_op_ese_scratch_bytes(int B, int HW, int C) {
    return static_cast<int64_t>(B) * (ese_nsplit(HW) + 1) * C * 4;
}

int dd3d_op_ese(const void* d_x, int x_pitch, const float* d_fc_w, const float* d_fc_b, const void* d_identity,
                int id_pitch, void* d_out, int out_pitch, float* d_scratch, int B, int HW, int C, dd3d_stream stream) {
    if (C % 8) return DD3D_ERR_INVALID;
    float* partial = d_scratch;
    float* gate = d_scratch + static_cast<size_t>(B) * ese_nsplit(HW) * C;
    return cuda_status(launch_ese(static_cast<const __nv_bfloat16*>(d_x), x_pitch, d_fc_w, d_fc_b,
                                  static_cast<const __nv_bfloat16*>(d_identity), id_pitch,
                                  static_cast<__nv_bfloat16*>(d_out), out_pitch, partial, gate, B, HW, C, device_sms(),
                                  static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int dd3d_op_bev_nms(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                    const int32_t* d_sizes, int32_t* d_flags, int B, int cap, float iou_thresh, int do_postprocess,
                    dd3d_stream stream) {
    if (!d_dets || !d_counts || !d_intrinsics || !d_poses || !d_sizes || !d_flags || B < 1 || cap < 1)
        return DD3D_ERR_INVALID;
    return cuda_status(launch_bev_nms(reinterpret_cast<Det*>(d_dets), d_counts, d_intrinsics, d_poses, d_sizes, d_flags, B,
                                      cap, iou_thresh, do_postprocess, static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int64_t dd3d_op_bev_nms_large_scratch_bytes(int B, int cap) {
    if (B < 1 || cap < 1 || cap > kLevels * kMaxPreNmsTopk) return DD3D_ERR_INVALID;
    return static_cast<int64_t>(image_bev_nms_scratch_bytes(B, cap, DD3D_MAX_NUM_CLASSES));
}

int dd3d_op_bev_nms_large(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                          const int32_t* d_sizes, void* d_scratch, int32_t* d_flags, int B, int cap, float iou_thresh,
                          int do_postprocess, dd3d_stream stream) {
    if (!d_dets || !d_counts || !d_intrinsics || !d_poses || (do_postprocess && !d_sizes) || !d_scratch || !d_flags ||
        B < 1 || cap < 1 || cap > kLevels * kMaxPreNmsTopk)
        return DD3D_ERR_INVALID;
    return cuda_status(launch_image_bev_nms(reinterpret_cast<Det*>(d_dets), d_counts, d_intrinsics, d_poses,
                                            do_postprocess ? d_sizes : nullptr, d_scratch, d_flags, B, cap, iou_thresh,
                                            DD3D_MAX_NUM_CLASSES, static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int dd3d_op_rotated_iou(const float* d_a, const float* d_b, int n, float* d_out, dd3d_stream stream) {
    if (!d_a || !d_b || !d_out || n < 0) return DD3D_ERR_INVALID;
    return cuda_status(launch_rotated_iou(d_a, d_b, n, d_out, static_cast<cudaStream_t>(stream)), nullptr);
}

static_assert(sizeof(dd3d_tta_view) == sizeof(TtaView), "dd3d_tta_view must mirror TtaView");

int dd3d_op_tta_merged_cap(int num_views, int cap) { return tta_merged_cap(num_views, cap); }

int64_t dd3d_op_tta_merge_scratch_bytes(int num_views, int cap) {
    return static_cast<int64_t>(tta_scratch_bytes(num_views, cap));
}

int dd3d_op_tta_merge(const dd3d_det* d_dets, const int32_t* d_counts, const dd3d_tta_view* h_views, int num_views, int cap,
                      float nms_thresh, int do_nms, void* d_scratch, dd3d_det* d_out, int32_t* d_out_count,
                      int32_t* d_flags, dd3d_stream stream) {
    if (!d_dets || !d_counts || !h_views || !d_scratch || !d_out || !d_out_count || !d_flags) return DD3D_ERR_INVALID;
    return cuda_status(launch_tta_merge(reinterpret_cast<const Det*>(d_dets), d_counts,
                                        reinterpret_cast<const TtaView*>(h_views), num_views, cap, nms_thresh, do_nms,
                                        d_scratch, reinterpret_cast<Det*>(d_out), d_out_count, d_flags,
                                        static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int dd3d_op_tta_merged_cap_large(int num_views, int cap) {
    const int n = tta_merged_cap_large(num_views, cap);
    return n < 0 ? DD3D_ERR_INVALID : n;
}

int64_t dd3d_op_tta_merge_large_scratch_bytes(int num_views, int cap) {
    const size_t bytes = tta_large_scratch_bytes(num_views, cap);
    return bytes ? static_cast<int64_t>(bytes) : DD3D_ERR_INVALID;
}

int dd3d_op_tta_merge_large(const dd3d_det* d_dets, const int32_t* d_counts, const dd3d_tta_view* h_views, int num_views,
                            int cap, float nms_thresh, int do_nms, void* d_scratch, dd3d_det* d_out, int32_t* d_out_count,
                            int32_t* d_flags, dd3d_stream stream) {
    if (!d_dets || !d_counts || !h_views || !d_scratch || !d_out || !d_out_count || !d_flags ||
        tta_merged_cap_large(num_views, cap) < 0)
        return DD3D_ERR_INVALID;
    return cuda_status(launch_tta_merge_large(reinterpret_cast<const Det*>(d_dets), d_counts,
                                              reinterpret_cast<const TtaView*>(h_views), num_views, cap, nms_thresh,
                                              do_nms, d_scratch, reinterpret_cast<Det*>(d_out), d_out_count, d_flags,
                                              static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int dd3d_forward_resized(dd3d_handle h, const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                         const int32_t* h_new_sizes, const int32_t* h_flip, const float* h_intrinsics,
                         const int32_t* h_sizes, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream) {
    if (!d_raw || !h_raw_sizes || !h_new_sizes || !h_intrinsics || !h_sizes || !d_out || !d_counts) return DD3D_ERR_INVALID;
    return guarded(h, [&](Engine& e) {
        e.forward_resized(d_raw, raw_h, raw_w, h_raw_sizes, h_new_sizes, h_flip, h_intrinsics, h_sizes,
                          reinterpret_cast<Det*>(d_out), d_counts, static_cast<cudaStream_t>(stream));
    });
}

int dd3d_op_resize_preprocess(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                              const int32_t* h_new_sizes, const int32_t* h_flip, void* d_out4, int B, int Hp, int Wp,
                              const float* h_mean, const float* h_std, dd3d_stream stream) {
    if (!d_raw || !h_raw_sizes || !h_new_sizes || !d_out4 || !h_mean || !h_std || B < 1) return DD3D_ERR_INVALID;
    static ResizeTables tables;  // operator-level entry point: one table cache per process (tests; not thread safe)
    return cuda_status(tables.launch(d_raw, raw_h, raw_w, h_raw_sizes, h_new_sizes, h_flip,
                                     static_cast<__nv_bfloat16*>(d_out4), B, Hp, Wp, h_mean, h_std,
                                     static_cast<cudaStream_t>(stream), g_op_fp16),
                       nullptr);
}

int64_t dd3d_op_sample_aggregate_scratch_bytes(int B, int cap) {
    return static_cast<int64_t>(sample_aggregate_scratch_bytes(B, cap));
}

int dd3d_op_sample_aggregate(dd3d_det* d_dets, int32_t* d_counts, const float* d_intrinsics, const float* d_poses,
                             const int32_t* d_group, int num_groups, float* d_global, void* d_scratch, int32_t* d_flags,
                             int B, int cap, float iou_thresh, int max_dets, dd3d_stream stream) {
    if (!d_dets || !d_counts || !d_intrinsics || !d_poses || !d_group || !d_global || !d_scratch || !d_flags || B < 1 ||
        cap < 1 || cap > 256 || num_groups < 1 || num_groups > B)
        return DD3D_ERR_INVALID;
    return cuda_status(launch_sample_aggregate(reinterpret_cast<Det*>(d_dets), d_counts, d_intrinsics, d_poses, d_group,
                                               num_groups, d_global, d_scratch, d_flags, B, cap, iou_thresh, max_dets,
                                               static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int64_t dd3d_op_group_bev_nms_scratch_bytes(int B, int cap, int max_group_images) {
    if (B < 1 || B > 256 || cap < 1 || cap > 1024 || max_group_images < 1 || max_group_images > 16) return DD3D_ERR_INVALID;
    return static_cast<int64_t>(group_bev_nms_scratch_bytes(B, cap, max_group_images));
}

int dd3d_op_group_bev_nms(dd3d_det* d_dets, int32_t* d_counts, const float* d_view_K, int num_views, const float* d_poses,
                          int pose_mode, const int32_t* d_group, int num_groups, int max_group_images, float* d_global,
                          void* d_scratch, int32_t* d_flags, int B, int cap, float iou_thresh, int max_dets,
                          dd3d_stream stream) {
    if (!d_dets || !d_counts || !d_view_K || !d_group || !d_scratch || !d_flags || num_views < 1 || B < 1 || B > 256 ||
        cap < 1 || cap > 1024 || num_groups < 1 || num_groups > B || max_group_images < 1 || max_group_images > 16 ||
        (pose_mode != DD3D_POSE_GLOBAL && pose_mode != DD3D_POSE_CAMERA) || (pose_mode == DD3D_POSE_GLOBAL && !d_poses))
        return DD3D_ERR_INVALID;
    return cuda_status(launch_group_bev_nms(reinterpret_cast<Det*>(d_dets), d_counts, d_view_K, num_views, d_poses,
                                            pose_mode, d_group, num_groups, max_group_images, d_global, d_scratch,
                                            d_flags, B, cap, iou_thresh, max_dets, static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int64_t dd3d_op_group_bev_nms_large_scratch_bytes(int B, int cap, int max_group_images) {
    const size_t bytes = group_bev_nms_large_scratch_bytes(B, cap, max_group_images);
    return bytes ? static_cast<int64_t>(bytes) : DD3D_ERR_INVALID;
}

int dd3d_op_group_bev_nms_large(dd3d_det* d_dets, int32_t* d_counts, const float* d_view_K, int num_views,
                                const float* d_poses, int pose_mode, const int32_t* d_group, int num_groups,
                                int max_group_images, float* d_global, void* d_scratch, int32_t* d_flags, int B, int cap,
                                float iou_thresh, int max_dets, dd3d_stream stream) {
    if (!d_dets || !d_counts || !d_view_K || !d_group || !d_scratch || !d_flags || num_views < 1 ||
        group_bev_nms_large_scratch_bytes(B, cap, max_group_images) == 0 || num_groups < 1 || num_groups > B ||
        (pose_mode != DD3D_POSE_GLOBAL && pose_mode != DD3D_POSE_CAMERA) || (pose_mode == DD3D_POSE_GLOBAL && !d_poses))
        return DD3D_ERR_INVALID;
    return cuda_status(launch_group_bev_nms_large(reinterpret_cast<Det*>(d_dets), d_counts, d_view_K, num_views, d_poses,
                                                  pose_mode, d_group, num_groups, max_group_images, d_global, d_scratch,
                                                  d_flags, B, cap, iou_thresh, max_dets,
                                                  static_cast<cudaStream_t>(stream)),
                       nullptr);
}

int64_t dd3d_op_detect_scratch_bytes(int B, int pre_nms_topk) {
    return static_cast<int64_t>(decode_scratch_bytes(B, pre_nms_topk)) + DD3D_MAX_CLASSES * 3 * 4 + 512 +
           static_cast<int64_t>(nms_scratch_bytes(B, pre_nms_topk, DD3D_MAX_CLASSES));
}

// scratch of dd3d_op_detect_c: decode | canonical sizes (256-byte aligned, [C][3] fp32) | NMS.  At C <= 16 this is the layout
// dd3d_op_detect_scratch_bytes has always sized: the sizes take one 256-byte block.
int64_t dd3d_op_detect_c_scratch_bytes(int B, int pre_nms_topk, int num_classes) {
    if (B < 1 || pre_nms_topk < 1 || num_classes < 1 || num_classes > DD3D_MAX_NUM_CLASSES) return DD3D_ERR_INVALID;
    const int64_t canon = (num_classes * 3 * 4 + 255) / 256 * 256;
    return static_cast<int64_t>(decode_scratch_bytes(B, pre_nms_topk)) + 255 + canon + 256 +
           static_cast<int64_t>(nms_scratch_bytes(B, pre_nms_topk, num_classes));
}

int dd3d_op_detect_c(const dd3d_model_desc* desc, const float* h_canon, int B, const int32_t* h_level_hw, const int32_t* h_strides,
                     const float* const* d_cls, const float* const* d_box, const float* const* d_b3d, int cls_pitch,
                     int b3d_pitch, const float* d_intrinsics, const int32_t* d_sizes, void* d_scratch,
                     dd3d_det* d_pre_nms, int32_t* d_pre_counts, dd3d_det* d_out, int32_t* d_counts, int32_t* d_flags,
                     dd3d_stream stream_) {
    if (!desc || !h_level_hw || !h_strides || !d_cls || !d_box || !d_b3d || !d_scratch || !d_out || !d_counts)
        return DD3D_ERR_INVALID;
    if (desc->pre_nms_topk < 1 || desc->pre_nms_topk > kMaxPreNmsTopk) return DD3D_ERR_INVALID;
    const int C = desc->num_classes;
    if (C < 1 || C > DD3D_MAX_NUM_CLASSES || (h_canon == nullptr && C > DD3D_MAX_CLASSES)) return DD3D_ERR_INVALID;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    DecodeParams dp;
    memset(&dp, 0, sizeof(dp));
    for (int l = 0; l < kLevels; ++l) {
        dp.lvl[l].cls = d_cls[l];
        dp.lvl[l].box = d_box[l];
        dp.lvl[l].b3d = d_b3d[l];
        dp.lvl[l].H = h_level_hw[2 * l];
        dp.lvl[l].W = h_level_hw[2 * l + 1];
        dp.lvl[l].stride = h_strides[l];
    }
    // canonical sizes live at the tail of the caller's scratch
    const size_t dec_bytes = decode_scratch_bytes(B, desc->pre_nms_topk);
    float* d_canon = reinterpret_cast<float*>(static_cast<uint8_t*>(d_scratch) + (dec_bytes + 255) / 256 * 256);
    cudaError_t c = h_canon ? cudaMemcpyAsync(d_canon, h_canon, static_cast<size_t>(C) * 3 * 4, cudaMemcpyHostToDevice, stream)
                            : cudaMemcpyAsync(d_canon, desc->canonical_box3d_sizes, DD3D_MAX_CLASSES * 3 * 4,
                                              cudaMemcpyHostToDevice, stream);
    if (c != cudaSuccess) return DD3D_ERR_CUDA;
    fill_decode_params(&dp, *desc, B, cls_pitch, b3d_pitch, d_canon);
    decode_bind_scratch(&dp, d_scratch);
    decode_finalize_params(&dp);
    dp.K = d_intrinsics;
    c = launch_decode(dp, stream);
    if (c != cudaSuccess) return cuda_status(c, nullptr);
    if (d_pre_nms && d_pre_counts) {
        cudaMemcpyAsync(d_pre_nms, dp.cand, static_cast<size_t>(B) * kLevels * desc->pre_nms_topk * sizeof(Det),
                        cudaMemcpyDeviceToDevice, stream);
        cudaMemcpyAsync(d_pre_counts, dp.cand_count, static_cast<size_t>(B) * kLevels * 4, cudaMemcpyDeviceToDevice,
                        stream);
    }
    NmsParams np;
    // scratch behind the canonical sizes at the tail of d_scratch (one 256-byte block at C <= 16)
    fill_nms_params(&np, *desc, dp, B, reinterpret_cast<uint8_t*>(d_canon) + (static_cast<size_t>(C) * 3 * 4 + 255) / 256 * 256);
    np.sizes = d_sizes;
    np.out = reinterpret_cast<Det*>(d_out);
    np.out_count = d_counts;
    c = launch_nms(np, stream);
    if (c == cudaSuccess && d_flags) c = cudaMemcpyAsync(d_flags, dp.flags, 4, cudaMemcpyDeviceToDevice, stream);
    return cuda_status(c, nullptr);
}

int dd3d_op_detect_flags(const dd3d_model_desc* desc, int B, const int32_t* h_level_hw, const int32_t* h_strides,
                         const float* const* d_cls, const float* const* d_box, const float* const* d_b3d, int cls_pitch,
                         int b3d_pitch, const float* d_intrinsics, const int32_t* d_sizes, void* d_scratch,
                         dd3d_det* d_pre_nms, int32_t* d_pre_counts, dd3d_det* d_out, int32_t* d_counts, int32_t* d_flags,
                         dd3d_stream stream) {
    // its scratch (dd3d_op_detect_scratch_bytes) holds the NMS of DD3D_MAX_CLASSES classes
    if (desc && desc->num_classes > DD3D_MAX_CLASSES) return DD3D_ERR_INVALID;
    return dd3d_op_detect_c(desc, nullptr, B, h_level_hw, h_strides, d_cls, d_box, d_b3d, cls_pitch, b3d_pitch, d_intrinsics,
                            d_sizes, d_scratch, d_pre_nms, d_pre_counts, d_out, d_counts, d_flags, stream);
}

int dd3d_op_detect(const dd3d_model_desc* desc, int B, const int32_t* h_level_hw, const int32_t* h_strides,
                   const float* const* d_cls, const float* const* d_box, const float* const* d_b3d, int cls_pitch,
                   int b3d_pitch, const float* d_intrinsics, const int32_t* d_sizes, void* d_scratch, dd3d_det* d_pre_nms,
                   int32_t* d_pre_counts, dd3d_det* d_out, int32_t* d_counts, dd3d_stream stream) {
    return dd3d_op_detect_flags(desc, B, h_level_hw, h_strides, d_cls, d_box, d_b3d, cls_pitch, b3d_pitch, d_intrinsics,
                                d_sizes, d_scratch, d_pre_nms, d_pre_counts, d_out, d_counts, nullptr, stream);
}

}  // extern "C"
