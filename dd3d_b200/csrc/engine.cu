// DD3D inference engine: weight folding/packing, static graph for DLA-34 and DLA-X / every VoVNetV2-eSE variant + FPN + FCOS2D/3D
// heads, workspace planning and the forward launch sequence.  Reference structure being reproduced:
//   DD3D.forward                      tridet/modeling/dd3d/core.py:64-164
//   DLA-34, DLA-X-{46-C,60-C,60,102,102-64}  tridet/modeling/feature_extractor/dla.py:24-62,104-247,250-441
//   VoVNetV2-{19-slim-dw,19-dw,19-slim,19,39,57,99}-eSE   tridet/modeling/feature_extractor/vovnet.py:19-143,173-273,276-367
//   FPN + LastLevelP6P7 / LastLevelP6 detectron2 (SURVEY.md Appendix A), dla.py:537-561, vovnet.py:411-454
//   FCOS2DHead / FCOS3DHead           fcos2d.py:30-156, fcos3d.py:55-188 (+ normalization.py Scale/Offset/ModuleListDial)
// Design notes (DESIGN.md): NHWC bf16 activations; BN folded to fp32 (scale, bias) applied in the conv epilogue;
// concats never materialised (producers write channel slices); predictors fused per tower.
#include "engine.cuh"

#include "act16.cuh"
#include "pdl.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <optional>
#include <stdexcept>

namespace dd3d {

namespace {

inline int round_up(int v, int a) { return (v + a - 1) / a * a; }
inline size_t round_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }
// Output channels a conv layer (and its epilogue vectors) is padded to: a multiple of 16, or of 64 when no N-block width of the
// conv kernel divides that (wide class-specific heads: 11 x 26 = 286 -> 320)
inline int cout_padded(int cout) {
    const int p = round_up(cout, 16);
    return conv_block_n(p) != 0 ? p : round_up(cout, 64);
}

[[noreturn]] void fail(int status, const std::string& msg) { throw EngineError(status, msg); }

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) fail(DD3D_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

}  // namespace

// ================================================================================================ Engine basics

Engine::Engine(const dd3d_model_desc& d) : desc(d) {
    if (dla_spec(d.arch) == nullptr && vovnet_spec(d.arch) == nullptr) fail(DD3D_ERR_INVALID, "unknown arch");
    if (d.num_classes < 1 || d.num_classes > DD3D_MAX_NUM_CLASSES) fail(DD3D_ERR_INVALID, "num_classes out of range");
    if (d.pre_nms_topk < 1 || d.pre_nms_topk > kMaxPreNmsTopk) fail(DD3D_ERR_INVALID, "pre_nms_topk out of range");
    if (d.out_cap < 1) fail(DD3D_ERR_INVALID, "out_cap must be positive");
    if (d.act_dtype != DD3D_ACT_BF16 && d.act_dtype != DD3D_ACT_FP16) fail(DD3D_ERR_INVALID, "unknown act_dtype");
    fp16 = d.act_dtype == DD3D_ACT_FP16 ? 1 : 0;
    cuda_check(cudaGetDevice(&device), "cudaGetDevice");
    cudaDeviceProp prop;
    cuda_check(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
    if (prop.major != 9) {
        fail(DD3D_ERR_CUDA, std::string("dd3d_b200 needs an sm_90 (H100) device, found ") + prop.name + " sm_" +
                                std::to_string(prop.major) + std::to_string(prop.minor));
    }
    num_sms = prop.multiProcessorCount;
    if (const char* e = getenv("DD3D_SPARSE_BOX3D")) opt_sparse_box3d = std::max(0, std::min(2, atoi(e)));
    if (const char* e = getenv("DD3D_SPARSE_TOWER")) opt_sparse_tower = std::max(0, std::min(2, atoi(e)));
    if (const char* e = getenv("DD3D_SPARSE_BOX2D_TOWER")) opt_sparse_box2d_tower = std::max(0, std::min(2, atoi(e)));
}

Engine::~Engine() {
    release_plan();
    for (auto& kv : plan_cache) free_plan(&kv.second);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    for (int i = 0; i < 2; ++i) {
        if (h2d_done[i]) cudaEventDestroy(h2d_done[i]);
        if (all_done[i]) cudaEventDestroy(all_done[i]);
    }
    for (void* p : device_allocs) cudaFree(p);
}

void* Engine::dev_alloc(size_t bytes) {
    void* p = nullptr;
    cuda_check(cudaMalloc(&p, std::max<size_t>(bytes, 16)), "cudaMalloc(weights)");
    device_allocs.push_back(p);
    return p;
}

float* Engine::upload_f32(const std::vector<float>& v) {
    float* d = static_cast<float*>(dev_alloc(v.size() * 4));
    cuda_check(cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice), "upload f32");
    return d;
}

const HostTensor& Engine::weight(const std::string& name) const {
    auto it = weights.find(name);
    if (it == weights.end()) fail(DD3D_ERR_MISSING, "missing weight: " + name);
    return it->second;
}

void Engine::load_weight(const char* name, const float* data, const int64_t* shape, int ndim) {
    if (finalized) fail(DD3D_ERR_STATE, "load_weight after finalize");
    HostTensor t;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) {
        t.shape.push_back(shape[i]);
        n *= static_cast<size_t>(shape[i]);
    }
    t.data.assign(data, data + n);
    weights[name] = std::move(t);
}

// ------------------------------------------------------------------------------------------------ layer builders

// Conv weights of one or more reference tensors stacked along Cout -> bf16 [cout_pad][taps][cin_pad64].
const ConvLayer& Engine::conv_layer(const std::string& key, const std::vector<std::string>& wnames, int cin,
                                    int ksize) {
    auto it = convs.find(key);
    if (it != convs.end()) return it->second;
    ConvLayer L;
    L.cin = cin;
    L.ksize = ksize;
    L.taps = ksize * ksize;
    L.kchunks = (cin + kBlockK - 1) / kBlockK;
    const int cin_pad = L.kchunks * kBlockK;
    L.ktot = L.taps * cin_pad;
    int cout = 0;
    for (auto& n : wnames) {
        const HostTensor& w = weight(n + ".weight");
        if (w.shape.size() != 4 || w.shape[1] != cin || w.shape[2] != ksize || w.shape[3] != ksize)
            fail(DD3D_ERR_INVALID, "bad conv weight shape: " + n);
        cout += static_cast<int>(w.shape[0]);
    }
    L.cout = cout;
    L.cout_pad = cout_padded(cout);
    L.block_n = conv_block_n(L.cout_pad);  // 384 (slim VoVNet stage 4) -> 192
    if (L.block_n == 0) fail(DD3D_ERR_INVALID, "cout > 256 needs a multiple of 64 <= 256 that divides it: " + key);
    L.n_blocks = L.cout_pad / L.block_n;
    std::vector<uint16_t> packed(static_cast<size_t>(L.cout_pad) * L.ktot, 0);
    int co0 = 0;
    for (auto& n : wnames) {
        const HostTensor& w = weight(n + ".weight");
        const int co_n = static_cast<int>(w.shape[0]);
        for (int co = 0; co < co_n; ++co)
            for (int ci = 0; ci < cin; ++ci)
                for (int t = 0; t < L.taps; ++t)
                    packed[(static_cast<size_t>(co0 + co) * L.taps + t) * cin_pad + ci] =
                        host_f32_to_act(w.data[(static_cast<size_t>(co) * cin + ci) * L.taps + t], fp16);
        co0 += co_n;
    }
    L.d_w = static_cast<__nv_bfloat16*>(dev_alloc(packed.size() * 2));
    cuda_check(cudaMemcpy(L.d_w, packed.data(), packed.size() * 2, cudaMemcpyHostToDevice), "upload conv weights");
    if (!make_weight_map(&L.w_map, L.d_w, L.ktot, L.cout_pad, L.block_n, fp16)) fail(DD3D_ERR_CUDA, conv_last_error());
    if (L.taps == 9 && L.cout_pad == 16) {
        // taps-in-N copy (conv_taps_kernel): row = tap * 16 + cout, K = channels
        std::vector<uint16_t> tp(static_cast<size_t>(kTapsN) * cin_pad, 0);
        for (int co = 0; co < L.cout_pad; ++co)
            for (int t = 0; t < 9; ++t)
                for (int ci = 0; ci < cin_pad; ++ci)
                    tp[(static_cast<size_t>(t) * 16 + co) * cin_pad + ci] = packed[(static_cast<size_t>(co) * L.taps + t) * cin_pad + ci];
        L.d_w_taps = static_cast<__nv_bfloat16*>(dev_alloc(tp.size() * 2));
        cuda_check(cudaMemcpy(L.d_w_taps, tp.data(), tp.size() * 2, cudaMemcpyHostToDevice), "upload taps-in-N weights");
        if (!make_weight_map_taps(&L.w_map_taps, L.d_w_taps, cin_pad, fp16)) fail(DD3D_ERR_CUDA, conv_last_error());
    }
    return convs.emplace(key, L).first->second;
}

// Depthwise 3x3 weights [C][1][3][3] -> 16-bit [9][C] (tap-major: one 16-byte load per 8 channels and tap, dwconv.cu).
const DwLayer& Engine::dw_layer(const std::string& wname, int C) {
    auto it = dws.find(wname);
    if (it != dws.end()) return it->second;
    const HostTensor& w = weight(wname + ".weight");
    if (w.shape.size() != 4 || w.shape[0] != C || w.shape[1] != 1 || w.shape[2] != 3 || w.shape[3] != 3 || C % 8)
        fail(DD3D_ERR_INVALID, "bad depthwise conv weight shape: " + wname);
    std::vector<uint16_t> packed(static_cast<size_t>(9) * C);
    for (int c = 0; c < C; ++c)
        for (int t = 0; t < 9; ++t) packed[static_cast<size_t>(t) * C + c] = host_f32_to_act(w.data[static_cast<size_t>(c) * 9 + t], fp16);
    DwLayer L;
    L.C = C;
    L.d_w = static_cast<__nv_bfloat16*>(dev_alloc(packed.size() * 2));
    cuda_check(cudaMemcpy(L.d_w, packed.data(), packed.size() * 2, cudaMemcpyHostToDevice), "upload depthwise weights");
    return dws.emplace(wname, L).first->second;
}

// Grouped 3x3 weights [C][C / groups][3][3] (groups dividing C, channels per group dividing 64) -> 16-bit [C][9][64] for the
// block-diagonal mode of the implicit-GEMM kernel: row co holds its group's input channels at their position inside the
// 64-channel block of co, zeros elsewhere.
const ConvLayer& Engine::grouped_conv_layer(const std::string& wname, int C, int groups) {
    auto it = convs.find(wname);
    if (it != convs.end()) return it->second;
    const HostTensor& w = weight(wname + ".weight");
    const int cpg = groups > 0 ? C / groups : 0;
    if (groups < 1 || C % groups || C % kBlockK || cpg < 1 || kBlockK % cpg || w.shape.size() != 4 || w.shape[0] != C ||
        w.shape[1] != cpg || w.shape[2] != 3 || w.shape[3] != 3)
        fail(DD3D_ERR_INVALID, "bad grouped conv weight shape: " + wname);
    ConvLayer L;
    L.cin = C;
    L.cout = C;
    L.cout_pad = C;
    L.ksize = 3;
    L.taps = 9;
    L.kchunks = 1;
    L.ktot = 9 * kBlockK;
    L.block_n = kBlockK;
    L.n_blocks = C / kBlockK;
    L.groups = groups;
    std::vector<uint16_t> packed(static_cast<size_t>(C) * L.ktot, 0);
    for (int co = 0; co < C; ++co) {
        const int ci0 = (co / cpg) * cpg % kBlockK;  // the group's first input channel inside co's 64-channel block
        for (int ci = 0; ci < cpg; ++ci)
            for (int t = 0; t < 9; ++t)
                packed[(static_cast<size_t>(co) * 9 + t) * kBlockK + ci0 + ci] =
                    host_f32_to_act(w.data[(static_cast<size_t>(co) * cpg + ci) * 9 + t], fp16);
    }
    L.d_w = static_cast<__nv_bfloat16*>(dev_alloc(packed.size() * 2));
    cuda_check(cudaMemcpy(L.d_w, packed.data(), packed.size() * 2, cudaMemcpyHostToDevice), "upload grouped conv weights");
    if (!make_weight_map(&L.w_map, L.d_w, L.ktot, L.cout_pad, L.block_n, fp16)) fail(DD3D_ERR_CUDA, conv_last_error());
    return convs.emplace(wname, L).first->second;
}

void Engine::set_layout(const dd3d_layout_desc& l) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_layout after finalize");
    for (int n : {l.fcos2d_norm, l.fcos3d_norm, l.fpn_norm})
        if (n < DD3D_NORM_BN_PER_LEVEL || n > DD3D_NORM_NONE) fail(DD3D_ERR_INVALID, "unknown dd3d_norm value");
    for (int d : {l.num_cls_convs, l.num_box2d_convs, l.num_box3d_convs})
        if (d < 0 || d > 16) fail(DD3D_ERR_INVALID, "tower depth outside 0..16");
    if (l.fpn_fuse_avg != 0 && l.fpn_fuse_avg != 1) fail(DD3D_ERR_INVALID, "fpn_fuse_avg must be 0 or 1");
    layout = l;
}

void Engine::set_backbone_norm(int norm) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_backbone_norm after finalize");
    if (norm < DD3D_NORM_BN_PER_LEVEL || norm > DD3D_NORM_NONE) fail(DD3D_ERR_INVALID, "unknown dd3d_norm value");
    const bool dla = dla_spec(desc.arch) != nullptr;
    // the 16-channel base_layer of every DLA cannot take GroupNorm(32, C); a VoVNet without a norm fails in the reference's forward
    if (dla && norm == DD3D_NORM_GN) fail(DD3D_ERR_INVALID, "a DLA has no GroupNorm backbone (16 channels)");
    if (!dla && norm == DD3D_NORM_NONE) fail(DD3D_ERR_INVALID, "a VoVNet backbone needs a norm");
    if (!dla && norm == DD3D_NORM_GN) {  // GroupNorm(32, C) of every stem, OSA, concat and reduction conv
        const VovSpec& S = *vovnet_spec(desc.arch);
        bool ok = true;
        for (int i = 0; i < 4; ++i) ok = ok && group_norm_channels_ok(S.stage_ch[i]) && group_norm_channels_ok(S.out_ch[i]);
        for (int i = 0; i < 3; ++i) ok = ok && group_norm_channels_ok(S.stem[i]);
        if (!ok) fail(DD3D_ERR_INVALID, "GroupNorm(32, C) needs channel counts 32 divides (slim VoVNets have 112)");
    }
    backbone_norm = norm;
}

void Engine::set_fpn_channels(int C) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_fpn_channels after finalize");
    if (C < 64 || C > 512 || C % 64) fail(DD3D_ERR_INVALID, "FPN width must be a multiple of 64 in [64, 512]");
    fpn_channels = C;
}

// VoVNet: the stem and stage2 share stride 4, so the stem stands in for stage 2 of the stride order
static int fpn_input_stage(int v) { return v == DD3D_FPN_IN_STEM ? 2 : v; }

std::vector<int> Engine::fpn_input_list() const {
    if (!fpn_inputs.empty()) return fpn_inputs;
    if (dla_spec(desc.arch) != nullptr) return {3, 4, 5};
    return {2, 3, 4, 5};
}

int Engine::fpn_first_stage() const { return fpn_input_stage(fpn_input_list()[0]); }

int Engine::fpn_outputs() const {
    return static_cast<int>(fpn_input_list().size()) + (dla_spec(desc.arch) != nullptr ? 2 : 1);
}

void Engine::set_fpn_inputs(const int32_t* inputs, int n) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_fpn_inputs after finalize");
    if (!in_features.empty()) fail(DD3D_ERR_STATE, "dd3d_set_fpn_inputs after dd3d_set_in_features");
    if (inputs == nullptr || n < 1 || n > 4) fail(DD3D_ERR_INVALID, "dd3d_set_fpn_inputs needs 1 to 4 backbone outputs");
    const bool dla = dla_spec(desc.arch) != nullptr;
    std::vector<int> v(inputs, inputs + n);
    for (int i = 0; i < n; ++i) {
        // DLA level2..5 (level0 / level1 are stride 1 / 2: the fused front end never stores them); VoVNet stem, stage2..5
        const bool known = dla ? (v[i] >= 2 && v[i] <= 5) : (v[i] == DD3D_FPN_IN_STEM || (v[i] >= 2 && v[i] <= 5));
        if (!known) fail(DD3D_ERR_INVALID, "backbone output " + std::to_string(v[i]) + " cannot feed the FPN");
        if (i > 0 && fpn_input_stage(v[i]) != fpn_input_stage(v[i - 1]) + 1)
            fail(DD3D_ERR_INVALID, "FPN input strides must double from one input to the next");
    }
    if (v.back() != 5) fail(DD3D_ERR_INVALID, "the FPN inputs must end at stride 32 (the top block reads p5)");
    fpn_inputs.clear();
    if (v != fpn_input_list()) fpn_inputs = v;  // the default list is the default graph
}

void Engine::set_in_features(const int32_t* fpn_levels, int n) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_in_features after finalize");
    if (fpn_levels == nullptr || n < 1 || n > kLevels) fail(DD3D_ERR_INVALID, "dd3d_set_in_features needs 1 to 5 FPN levels");
    const int outs = fpn_outputs();
    std::vector<int> v(fpn_levels, fpn_levels + n);
    for (int i = 0; i < n; ++i) {
        if (v[i] < 0 || v[i] >= outs)
            fail(DD3D_ERR_INVALID, "FPN level " + std::to_string(v[i]) + " outside 0.." + std::to_string(outs - 1));
        for (int j = 0; j < i; ++j)
            if (v[j] == v[i]) fail(DD3D_ERR_INVALID, "FPN level " + std::to_string(v[i]) + " repeated");
    }
    in_features = v;
    if (n == outs) {  // every FPN output in order is the default graph
        bool identity = true;
        for (int i = 0; i < n; ++i) identity = identity && v[i] == i;
        if (identity) in_features.clear();
    }
}

void Engine::set_canonical_sizes(int num_classes, const float* sizes) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_canonical_sizes after finalize");
    if (num_classes != desc.num_classes || sizes == nullptr)
        fail(DD3D_ERR_INVALID, "dd3d_set_canonical_sizes needs num_classes (" + std::to_string(desc.num_classes) + ") rows");
    canonical_sizes.assign(sizes, sizes + static_cast<size_t>(num_classes) * 3);
}

// GroupNorm(32, C) affine of `<prefix>.weight` / `<prefix>.bias`, uploaded as fp32 vectors (cached like the epilogues)
const Epilogue& Engine::gn_affine(const std::string& prefix, int C) {
    const std::string key = "gn|" + prefix;
    auto it = epis.find(key);
    if (it != epis.end()) return it->second;
    const HostTensor& g = weight(prefix + ".weight");
    const HostTensor& b = weight(prefix + ".bias");
    if (g.data.size() != static_cast<size_t>(C) || b.data.size() != static_cast<size_t>(C))
        fail(DD3D_ERR_INVALID, "bad GroupNorm shape: " + prefix);
    return epilogue(key, g.data, b.data, nullptr);
}

// (scale, bias) of `conv (+bias) -> BN` for channels [0, cout); identity on the padding channels.
void Engine::bn_fold(const std::string& bn_prefix, const std::string& conv_bias_name, int cout, std::vector<float>* scale,
                     std::vector<float>* bias) const {
    scale->assign(cout, 1.0f);
    bias->assign(cout, 0.0f);
    if (!conv_bias_name.empty()) {
        const HostTensor& b = weight(conv_bias_name);
        if (static_cast<int>(b.data.size()) != cout) fail(DD3D_ERR_INVALID, "bad bias shape: " + conv_bias_name);
        *bias = b.data;
    }
    if (!bn_prefix.empty()) {
        const HostTensor& g = weight(bn_prefix + ".weight");
        const HostTensor& be = weight(bn_prefix + ".bias");
        const HostTensor& mu = weight(bn_prefix + ".running_mean");
        const HostTensor& var = weight(bn_prefix + ".running_var");
        if (static_cast<int>(g.data.size()) != cout) fail(DD3D_ERR_INVALID, "bad BN shape: " + bn_prefix);
        for (int c = 0; c < cout; ++c) {
            // FrozenBatchNorm2d / eval BatchNorm2d, eps = 1e-5: s = gamma * rsqrt(var + eps); b = beta - mean * s
            const float s = g.data[c] * (1.0f / sqrtf(var.data[c] + 1e-5f));
            const float b = be.data[c] - mu.data[c] * s;
            (*bias)[c] = (*bias)[c] * s + b;
            (*scale)[c] = s;
        }
    }
}

const Epilogue& Engine::epilogue(const std::string& key, const std::vector<float>& scale, const std::vector<float>& bias,
                                 const std::vector<float>* lo) {
    auto it = epis.find(key);
    if (it != epis.end()) return it->second;
    const int n_pad = cout_padded(static_cast<int>(scale.size()));
    std::vector<float> s(n_pad, 1.0f), b(n_pad, 0.0f);
    std::copy(scale.begin(), scale.end(), s.begin());
    std::copy(bias.begin(), bias.end(), b.begin());
    Epilogue e;
    e.d_scale = upload_f32(s);
    e.d_bias = upload_f32(b);
    e.d_lo = nullptr;
    if (lo != nullptr) {
        std::vector<float> l(n_pad, -INFINITY);
        std::copy(lo->begin(), lo->end(), l.begin());
        e.d_lo = upload_f32(l);
    }
    return epis.emplace(key, e).first->second;
}

const Epilogue& Engine::bn_epilogue(const std::string& key, const std::string& bn_prefix,
                                    const std::string& conv_bias_name, int cout) {
    auto it = epis.find(key);
    if (it != epis.end()) return it->second;
    std::vector<float> s, b;
    bn_fold(bn_prefix, conv_bias_name, cout, &s, &b);
    return epilogue(key, s, b, nullptr);
}

// ================================================================================================ graph builder

// The reference's VoVNet _STAGE_SPECS (vovnet.py:19-97).  eSE is applied in every module whatever the "eSE" flag says
// (_OSA_module, vovnet.py:216,233), so the flag is not carried.  dd3d_b200/arch.py keeps the copy param_specs needs.
static const VovSpec kVovSpecs[] = {
    // arch                     stem            stage_conv_ch          stage_out_ch            layers blocks        dw
    {DD3D_ARCH_V2_19_SLIM_DW, {64, 64, 64}, {64, 80, 96, 112}, {112, 256, 384, 512}, 3, {1, 1, 1, 1}, true},
    {DD3D_ARCH_V2_19_DW, {64, 64, 64}, {128, 160, 192, 224}, {256, 512, 768, 1024}, 3, {1, 1, 1, 1}, true},
    {DD3D_ARCH_V2_19_SLIM, {64, 64, 128}, {64, 80, 96, 112}, {112, 256, 384, 512}, 3, {1, 1, 1, 1}, false},
    {DD3D_ARCH_V2_19, {64, 64, 128}, {128, 160, 192, 224}, {256, 512, 768, 1024}, 3, {1, 1, 1, 1}, false},
    {DD3D_ARCH_V2_39, {64, 64, 128}, {128, 160, 192, 224}, {256, 512, 768, 1024}, 5, {1, 1, 2, 2}, false},
    {DD3D_ARCH_V2_57, {64, 64, 128}, {128, 160, 192, 224}, {256, 512, 768, 1024}, 5, {1, 1, 4, 3}, false},
    {DD3D_ARCH_V2_99, {64, 64, 128}, {128, 160, 192, 224}, {256, 512, 768, 1024}, 5, {1, 3, 9, 3}, false},
};

const VovSpec* vovnet_spec(int arch) {
    for (const VovSpec& s : kVovSpecs)
        if (s.arch == arch) return &s;
    return nullptr;
}

// The DLA networks of the reference's DLA_NAME_TO_BUILDER (dla.py:358-441) that the engine builds.  DLA-X-102-64 is
// dla102x2, which sets BottleneckX.cardinality = 64 (dla.py:411).  dd3d_b200/arch.py keeps the copy param_specs needs.
static const DlaSpec kDlaSpecs[] = {
    // arch                    levels                channels                          bottleneck_x root_res  cardinality
    {DD3D_ARCH_DLA34, {1, 1, 1, 2, 2, 1}, {16, 32, 64, 128, 256, 512}, false, false, 0},
    {DD3D_ARCH_DLA_X_46_C, {1, 1, 1, 2, 2, 1}, {16, 32, 64, 64, 128, 256}, true, false, 32},
    {DD3D_ARCH_DLA_X_60_C, {1, 1, 1, 2, 3, 1}, {16, 32, 64, 64, 128, 256}, true, false, 32},
    {DD3D_ARCH_DLA_X_60, {1, 1, 1, 2, 3, 1}, {16, 32, 128, 256, 512, 1024}, true, false, 32},
    {DD3D_ARCH_DLA_X_102, {1, 1, 1, 3, 4, 1}, {16, 32, 128, 256, 512, 1024}, true, true, 32},
    {DD3D_ARCH_DLA_X_102_64, {1, 1, 1, 3, 4, 1}, {16, 32, 128, 256, 512, 1024}, true, true, 64},
};

const DlaSpec* dla_spec(int arch) {
    for (const DlaSpec& s : kDlaSpecs)
        if (s.arch == arch) return &s;
    return nullptr;
}

struct Builder {
    Engine* E;
    Plan* P;
    bool dry;       // true: only size the arena and create layers (no tensor maps, no ops)
    uint8_t* base;  // arena base (nullptr when dry)
    size_t off = 0;  // bump offset of the PERSISTENT region (input, fp32 maps, scratch); starts after the activation arena
    int B;
    // Activation arena with liveness reuse: a first (dry, tracing) walk of the graph records for every bf16 activation
    // buffer the first and last op that touches it; plan_arena() then packs buffers with disjoint lifetimes into the same
    // memory (48 GB -> ~15 GB for V2-99 at B = 32), and the real walk hands out those offsets in the same order.
    std::vector<ArenaBuf>* bufs = nullptr;
    bool tracing = false;
    int next_buf = 0, op_idx = 0;
    bool list_tiles = false;  // the halo convs emitted meanwhile are sparse tower layers: kListTile x kListTile tiles

    View alloc(int H, int W, int C) {
        View v;
        v.B = B; v.H = H; v.W = W; v.C = C; v.pitch = C;
        const size_t bytes = round_up_sz(static_cast<size_t>(B) * H * W * C * 2, 1024);
        v.buf = next_buf++;
        if (tracing) {
            ArenaBuf b;
            b.bytes = bytes;
            bufs->push_back(b);
        }
        v.ptr = dry ? nullptr : reinterpret_cast<__nv_bfloat16*>(base + (*bufs)[v.buf].offset);
        return v;
    }
    void touch(const View& v) {  // op `op_idx` reads or writes v
        if (!tracing || v.buf < 0) return;
        ArenaBuf& b = (*bufs)[v.buf];
        b.first = std::min(b.first, op_idx);
        b.last = std::max(b.last, op_idx);
    }
    void persist(const View& v) {
        if (tracing && v.buf >= 0) (*bufs)[v.buf].persistent = true;
    }
    float* alloc_f32(size_t n) {
        float* p = dry ? nullptr : reinterpret_cast<float*>(base + off);
        off += round_up_sz(n * 4, 1024);
        return p;
    }
    void* alloc_bytes(size_t n) {
        void* p = dry ? nullptr : static_cast<void*>(base + off);
        off += round_up_sz(n, 1024);
        return p;
    }
    static View slice(View v, int c0, int C) {
        if (v.ptr) v.ptr += c0;
        v.C = C;
        return v;
    }

    // ---- conv (one or several segments sharing the weights) ------------------------------------------------
    struct SegSpec {
        View in, out;
        const Epilogue* epi;
        View res;           // residual (ptr == nullptr: none)
        bool has_res = false;
        bool res_up2 = false;
        float* out_f32 = nullptr;
        int out_pitch = 0;
    };

    void conv(const ConvLayer& L, int stride, bool relu, std::vector<SegSpec>& segs, bool f32_out) {
        for (auto& sp : segs) {
            touch(sp.in);
            if (!f32_out) touch(sp.out);
            if (sp.has_res) touch(sp.res);
        }
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::CONV;
        ConvParams& p = op.conv;
        memset(&p, 0, sizeof(p));
        p.nseg = static_cast<int>(segs.size());
        p.B = B;
        p.taps = L.taps;
        p.stride = stride;
        p.kchunks = L.kchunks;
        p.cin = L.cin;
        p.n_blocks = L.n_blocks;
        p.block_n = L.block_n;
        p.relu = relu ? 1 : 0;
        p.out_mode = f32_out ? 1 : 0;
        p.fp16 = E->fp16;
        p.grouped = L.groups > 1 ? 1 : 0;
        {
            int hs[kMaxSeg], ws[kMaxSeg];
            for (int s = 0; s < p.nseg; ++s) {
                hs[s] = segs[s].in.H / stride;
                ws[s] = segs[s].in.W / stride;
            }
            p.halo = conv_prefer_halo(L.taps, stride, L.block_n, p.nseg, hs, ws) ? 1 : 0;
            p.taps_n = (L.d_w_taps != nullptr && conv_taps_eligible(L.taps, stride, L.cout_pad, p.nseg, hs, ws)) ? 1 : 0;
        }
        for (int s = 0; s < p.nseg; ++s) {
            SegSpec& sp = segs[s];
            ConvSeg& g = p.seg[s];
            if (sp.in.C != L.cin) fail(DD3D_ERR_INVALID, "conv input channel mismatch");
            int Ho = sp.in.H, Wo = sp.in.W;
            if (stride == 2) {
                if ((sp.in.H & 1) || (sp.in.W & 1)) fail(DD3D_ERR_INVALID, "stride-2 conv needs even input size");
                Ho = sp.in.H / 2;
                Wo = sp.in.W / 2;
            }
            g.H = Ho;
            g.W = Wo;
            choose_tile(Ho, Wo, &g.th, &g.tw);
            bool ok;
            if (p.halo && list_tiles) {  // the work-list pair tile: one [10][10] patch per 8x8 tile (use_tile_lists)
                g.th = g.tw = kListTile;
                ok = make_act_map(&g.in_map[0], sp.in.ptr, B, sp.in.H, sp.in.W, sp.in.C, sp.in.pitch, kListTile + 2,
                                  kListTile + 2, E->fp16);
            } else if (p.halo) {
                g.th = kHaloTh;
                g.tw = kHaloTw;
                ok = make_act_map_halo(&g.in_map[0], sp.in.ptr, B, sp.in.H, sp.in.W, sp.in.C, sp.in.pitch, E->fp16);
            } else if (stride == 1) {
                ok = make_act_map(&g.in_map[0], sp.in.ptr, B, sp.in.H, sp.in.W, sp.in.C, sp.in.pitch, g.th, g.tw, E->fp16);
            } else {
                ok = make_act_map_s2(&g.in_map[0], sp.in.ptr, 0, B, sp.in.H, sp.in.W, sp.in.C, sp.in.pitch, g.th, g.tw,
                                     E->fp16) &&
                     make_act_map_s2(&g.in_map[1], sp.in.ptr, 1, B, sp.in.H, sp.in.W, sp.in.C, sp.in.pitch, g.th, g.tw,
                                     E->fp16);
            }
            if (!ok) fail(DD3D_ERR_CUDA, conv_last_error());
            g.scale = sp.epi->d_scale;
            g.bias = sp.epi->d_bias;
            g.lo = sp.epi->d_lo;
            if (f32_out) {
                g.out_f32 = sp.out_f32;
                g.out_pitch = sp.out_pitch;
            } else {
                if (sp.out.H != Ho || sp.out.W != Wo || sp.out.C != L.cout)
                    fail(DD3D_ERR_INVALID, "conv output view mismatch");
                if (!make_out_map(&g.out_map, sp.out.ptr, B, Ho, Wo, sp.out.C, sp.out.pitch, g.tw, E->fp16))
                    fail(DD3D_ERR_CUDA, conv_last_error());
                g.out16 = sp.out.ptr;
                g.out_pitch = sp.out.pitch;
            }
            if (sp.has_res) {
                g.residual = sp.res.ptr;
                g.res_pitch = sp.res.pitch;
                g.res_up2 = sp.res_up2 ? 1 : 0;
                g.res_H = sp.res.H;
                g.res_W = sp.res.W;
            }
        }
        // Under-filled launches (DLA-34 level5 at B = 8: 30 M-tiles x 2 N-blocks on 132 SMs; p6 / p7): split N until the grid
        // covers the machine.  Each CTA's serial MMA chain shrinks with N while the
        // A tiles it re-reads are tiny; K order per output element is unchanged, so results are bit-identical.
        // Filled halo layers with 128-multiple widths (FCOS towers, FPN outputs, VoVNet stage 2) run the 256 x 128 pair tile:
        // half the weight traffic per MAC, same K order -> bit-identical.
        // Grouped layers (block-diagonal mode) keep block_n 64, one k-block per n-block: no pair tile, no N-split (the weight-
        // stationary variant still applies to a single n-block, conv_finalize_params)
        const bool pair = !p.grouped && conv_select_pair(&p, L.cout_pad, E->num_sms);
        bool n_split = false;
        if (!p.taps_n && !pair && !p.grouped && conv_n_split_enabled()) {
            int tiles = 0;
            for (int s = 0; s < p.nseg; ++s)
                tiles += B * ((p.seg[s].H + p.seg[s].th - 1) / p.seg[s].th) * ((p.seg[s].W + p.seg[s].tw - 1) / p.seg[s].tw);
            // halves must stay multiples of 64: the epilogue stores 64-channel TMA boxes, and a box that starts inside this
            // n-block but ends in the next one would overwrite the neighbour's channels (only the tensor edge is clipped)
            while (tiles * p.n_blocks * 2 <= E->num_sms && p.block_n % 128 == 0) {
                p.block_n /= 2;
                p.n_blocks *= 2;
                n_split = true;
            }
        }
        conv_finalize_params(&p);
        if (n_split || pair) {
            if (!make_weight_map(&p.w_map, L.d_w, L.ktot, L.cout_pad, p.block_n, E->fp16))
                fail(DD3D_ERR_CUDA, conv_last_error());
        } else {
            p.w_map = p.taps_n ? L.w_map_taps : L.w_map;
        }
        for (int s = 0; s < p.nseg; ++s)
            op.flops += 2.0 * B * p.seg[s].H * p.seg[s].W * static_cast<double>(L.cout) * (L.cin / L.groups) * L.taps;  // useful MACs
        if (!f32_out) {
            op.nouts = p.nseg;
            for (int s = 0; s < p.nseg; ++s) op.outs[s] = segs[s].out;
        }
        P->ops.push_back(op);
    }

    // single-segment convenience: conv -> (BN) -> (+res) -> (ReLU) into `out`
    void conv1(const std::string& wname, const std::string& bn_prefix, bool has_bias, View in, View out, int ksize,
               int stride, bool relu, const View* res = nullptr, bool res_up2 = false) {
        const ConvLayer& L = E->conv_layer(wname, {wname}, in.C, ksize);
        const Epilogue& e = E->bn_epilogue(wname + "|" + bn_prefix, bn_prefix, has_bias ? wname + ".bias" : "", L.cout);
        std::vector<SegSpec> segs(1);
        segs[0].in = in;
        segs[0].out = out;
        segs[0].epi = &e;
        if (res) {
            segs[0].res = *res;
            segs[0].has_res = true;
            segs[0].res_up2 = res_up2;
        }
        conv(L, stride, relu, segs, false);
    }

    // GroupNorm (affine != nullptr) or the add / scale alone, in place on every map of `x`: + nearest-2x(res[s]) when
    // res is given, * 0.5 when avg, ReLU when relu (group_norm.cu).  Statistics scratch in the persistent region.
    void group_norm(const std::vector<View>& x, const Epilogue* affine, bool relu, const View* res, bool avg) {
        std::vector<float*> part(x.size(), nullptr);
        for (size_t s = 0; s < x.size(); ++s) {
            touch(x[s]);
            if (res) touch(res[s]);
            if (affine) part[s] = alloc_f32(group_norm_scratch_bytes(B, x[s].H, x[s].W) / 4);
        }
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::GN;
        GroupNormParams& p = op.gn;
        p.nseg = static_cast<int>(x.size());
        p.B = B;
        p.gamma = affine ? affine->d_scale : nullptr;
        p.beta = affine ? affine->d_bias : nullptr;
        p.relu = relu ? 1 : 0;
        p.avg = avg ? 1 : 0;
        p.fp16 = E->fp16;
        p.C = x[0].C;
        for (size_t s = 0; s < x.size(); ++s) {
            if (x[s].C != p.C || !group_norm_channels_ok(p.C)) fail(DD3D_ERR_INVALID, "GroupNorm channel count");
            GroupNormSeg& g = p.seg[s];
            g.in = x[s].ptr;
            g.out = x[s].ptr;
            g.H = x[s].H;
            g.W = x[s].W;
            g.in_pitch = g.out_pitch = x[s].pitch;
            if (res) {
                g.res = res[s].ptr;
                g.res_pitch = res[s].pitch;
                g.res_H = res[s].H;
                g.res_W = res[s].W;
            }
            g.part = reinterpret_cast<float2*>(part[s]);
            op.outs[s] = x[s];
            const double px = static_cast<double>(B) * x[s].H * x[s].W * p.C * 2;
            op.bytes += px * (affine ? 3 : 2) + (res ? px / 4 : 0.0);  // stats read, apply read + write, residual read
        }
        op.nouts = p.nseg;
        P->ops.push_back(op);
    }

    void maxpool(View in, View out, int ksize) {
        touch(in);
        touch(out);
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::POOL;
        op.in = in;
        op.out = out;
        op.ksize = ksize;
        op.outs[0] = out;
        op.nouts = 1;
        op.bytes = (static_cast<double>(B) * in.H * in.W + static_cast<double>(B) * out.H * out.W) * in.C * 2;
        P->ops.push_back(op);
    }
    void relu(View in, View out) {
        touch(in);
        touch(out);
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::RELU;
        op.in = in;
        op.out = out;
        op.outs[0] = out;
        op.nouts = 1;
        op.bytes = static_cast<double>(B) * in.H * in.W * in.C * 4;
        P->ops.push_back(op);
    }

    // ---- DLA (DLA-34 and the DLA-X networks of kDlaSpecs) ---------------------------------------------------------
    // DLA conv -> norm: the folded BN, or with FE.BACKBONE.NORM "" the conv's own bias (Conv2d(bias=norm == ""), dla.py:33,44,
    // 154,230,277,337).  Returns the (BN prefix, bias name) pair bn_fold takes.
    std::pair<std::string, std::string> dla_norm(const std::string& conv) const {
        if (E->backbone_norm == DD3D_NORM_NONE) return {"", conv + ".bias"};
        return {conv + ".norm", ""};
    }
    void dla_conv(const std::string& name, View in, View out, int ksize, int stride, bool relu, const View* res = nullptr) {
        const auto nb = dla_norm(name);
        conv1(name, nb.first, !nb.second.empty(), in, out, ksize, stride, relu, res);
    }
    // BasicBlock (dla.py:24-62): conv1 -> BN -> ReLU -> conv2 -> BN -> (+residual) -> ReLU
    void dla_block(const std::string& p, View x, int stride, View residual, View dst) {
        const int Ho = x.H / stride, Wo = x.W / stride;
        View t = alloc(Ho, Wo, dst.C);
        dla_conv(p + ".conv1", x, t, 3, stride, true);
        dla_conv(p + ".conv2", t, dst, 3, 1, true, &residual);
    }
    // BottleneckX (dla.py:104-143): 1x1 -> BN -> ReLU -> grouped 3x3 (stride) -> BN -> ReLU -> 1x1 -> BN -> (+residual) -> ReLU;
    // bottleneck width planes * cardinality / 32
    void dla_block_x(const std::string& p, View x, int stride, View residual, View dst, int cardinality) {
        const int width = dst.C * cardinality / 32;
        View t1 = alloc(x.H, x.W, width);
        dla_conv(p + ".conv1", x, t1, 1, 1, true);
        View t2 = alloc(x.H / stride, x.W / stride, width);
        const auto nb = dla_norm(p + ".conv2");
        const ConvLayer& L = E->grouped_conv_layer(p + ".conv2", width, cardinality);
        const Epilogue& e = E->bn_epilogue(p + ".conv2|" + nb.first, nb.first, nb.second, width);
        std::vector<SegSpec> segs(1);
        segs[0].in = t1;
        segs[0].out = t2;
        segs[0].epi = &e;
        conv(L, stride, true, segs, false);
        dla_conv(p + ".conv3", t2, dst, 1, 1, true, &residual);
    }
    // Tree (dla.py:170-247) of `levels` levels, output into *dst (a new buffer when dst is null, allocated where DLA-34's
    // hand-written builder allocated it, so that its ops and workspace plan are unchanged).  `rc` is the Root concat of the
    // levels-1 tree at the end of this tree's tree2 chain, laid out [x2 | x1 | bottom (level_root) | x1 of each enclosing
    // tree, outermost first]; `child` is the channel of this tree's first child slot in it.  `pooled`: x max-pooled by
    // `stride` when the caller has it already (every nested tree1 pools the same tensor as its parent, dla.py:235).
    View dla_tree(const std::string& p, View x, int levels, int in_ch, int out_ch, int stride, bool level_root, View rc,
                  int child, const View* pooled, const View* dst) {
        const DlaSpec& S = *dla_spec(E->desc.arch);
        const int Ho = x.H / stride, Wo = x.W / stride;
        View bottom = x;
        if (level_root) {
            if (pooled != nullptr || stride != 2) fail(DD3D_ERR_INVALID, "DLA level_root tree without its own pool: " + p);
            bottom = slice(rc, child, in_ch);
            maxpool(x, bottom, 2);
            child += in_ch;
        } else if (stride > 1) {
            if (pooled != nullptr) {
                bottom = *pooled;
            } else {
                bottom = alloc(Ho, Wo, in_ch);
                maxpool(x, bottom, stride);
            }
        }
        if (levels > 1) {
            View t1 = slice(rc, child, out_ch);
            View rc1 = alloc(Ho, Wo, levels * out_ch);  // tree1's own chain: [x2 | x1 | one x1 per level below]
            dla_tree(p + ".tree1", x, levels - 1, in_ch, out_ch, stride, false, rc1, 2 * out_ch, stride > 1 ? &bottom : nullptr,
                     &t1);
            return dla_tree(p + ".tree2", t1, levels - 1, out_ch, out_ch, 1, false, rc, child + out_ch, nullptr, dst);
        }
        View out = dst != nullptr ? *dst : alloc(Ho, Wo, out_ch);
        View residual = bottom;
        if (in_ch != out_ch) {
            residual = alloc(bottom.H, bottom.W, out_ch);
            dla_conv(p + ".project", bottom, residual, 1, 1, false);
        }
        View x1 = slice(rc, out_ch, out_ch);
        View x2 = slice(rc, 0, out_ch);
        if (S.bottleneck_x) {
            dla_block_x(p + ".tree1", x, stride, residual, x1, S.cardinality);
            dla_block_x(p + ".tree2", x1, 1, x1, x2, S.cardinality);
        } else {
            dla_block(p + ".tree1", x, stride, residual, x1);
            dla_block(p + ".tree2", x1, 1, x1, x2);
        }
        // Root: cat -> 1x1 -> BN (-> + x2 with residual_root) -> ReLU; x2 is the concat's first slice
        dla_conv(p + ".root.conv", rc, out, 1, 1, true, S.root_residual ? &x2 : nullptr);
        return out;
    }
    // DLA level 2..5: Tree(levels, channels[l-1] -> channels[l], stride 2, level_root = l > 2) with its root concat
    View dla_level(const std::string& p, View x, int levels, int in_ch, int out_ch, bool level_root, const View* pooled) {
        View rc = alloc(x.H / 2, x.W / 2, (levels + 1) * out_ch + (level_root ? in_ch : 0));
        return dla_tree(p, x, levels, in_ch, out_ch, 2, level_root, rc, 2 * out_ch, pooled, nullptr);
    }

    void build_dla(View input, std::vector<View>* feats) {
        const DlaSpec& S = *dla_spec(E->desc.arch);
        const std::string p = "backbone.bottom_up";
        const int H = input.H, W = input.W;
        // base_layer -> level0 -> level1 -> 2x2 max-pool in one kernel (dla_front.cu); the two full-resolution 16-channel
        // maps never reach HBM.  base_layer / level0 / level1 have DLA-34's shapes in every variant (channels 16, 16, 32).
        if (H % 4 || W % 4) fail(DD3D_ERR_STATE, "internal: the DLA front end needs H and W divisible by 4");
        View a2 = alloc(H / 2, W / 2, 32);
        View bottom = alloc(H / 4, W / 4, 32);
        front(E->front_layer(p), input, a2, bottom);
        const int* ch = S.channels;
        // the FPN inputs (FE.FPN.IN_FEATURES): level<first> .. level5
        const int first = E->fpn_first_stage();
        View x = dla_level(p + ".level2", a2, S.levels[2], ch[1], ch[2], false, &bottom);
        feats->clear();
        if (first == 2) feats->push_back(x);
        for (int l = 3; l <= 5; ++l) {
            x = dla_level(p + ".level" + std::to_string(l), x, S.levels[l], ch[l - 1], ch[l], true, nullptr);
            if (l >= first) feats->push_back(x);
        }
    }

    void front(const FrontLayer& F, View in4, View out, View pooled) {
        touch(out);
        touch(pooled);
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::FRONT;
        op.in = in4;
        op.out = out;
        op.identity = pooled;
        op.front = &F;
        op.outs[0] = out;
        op.outs[1] = pooled;
        op.nouts = 2;
        const double px = static_cast<double>(B) * in4.H * in4.W;
        op.flops = 2.0 * px * (16.0 * 3 * 49 + 16.0 * 16 * 9 + 32.0 * 16 * 9 / 4);
        op.bytes = px * (8.0 + 64.0 / 4 + 64.0 / 16);
        P->ops.push_back(op);
    }

    // VoVNet stem_1: 3x3 / stride 2, 3 -> 64 channels (stem_mma.cu)
    void stem(const std::string& wname, const std::string& bn, const std::string& bias, View in4, View out, bool relu = true) {
        const StemLayer& S = E->stem_layer(wname, bn, bias, relu);
        touch(out);
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::STEM;
        op.in = in4;
        op.out = out;
        op.stem = &S;
        op.outs[0] = out;
        op.nouts = 1;
        const double in_px = static_cast<double>(B) * in4.H * in4.W, out_px = static_cast<double>(B) * out.H * out.W;
        op.flops = 2.0 * out_px * 64 * 3 * 9;
        op.bytes = in_px * 8 + out_px * 64 * 2;
        P->ops.push_back(op);
    }

    // ---- VoVNetV2-eSE (every entry of the reference's _STAGE_SPECS) ----------------------------------------------
    // depthwise 3x3 (groups = C, no bias / norm / activation)
    void dwconv(const std::string& wname, View in, View out, int stride) {
        const DwLayer& L = E->dw_layer(wname, in.C);
        touch(in);
        touch(out);
        ++op_idx;
        if (dry) return;
        if (out.C != in.C || out.H != dwconv3x3_out_size(in.H, stride) || out.W != dwconv3x3_out_size(in.W, stride))
            fail(DD3D_ERR_INVALID, "depthwise conv output view mismatch: " + wname);
        Op op;
        op.type = Op::DW;
        op.in = in;
        op.out = out;
        op.stride = stride;
        op.dw = &L;
        op.outs[0] = out;
        op.nouts = 1;
        const double out_px = static_cast<double>(B) * out.H * out.W, in_px = static_cast<double>(B) * in.H * in.W;
        op.flops = 2.0 * out_px * L.C * 9;
        op.bytes = (in_px + out_px) * L.C * 2;
        P->ops.push_back(op);
    }

    // 3x3 conv -> norm -> ReLU (conv3x3, vovnet.py:124-143), or for the -dw variants depthwise 3x3 -> pointwise 1x1 ->
    // pw_norm -> ReLU (dw_conv3x3, vovnet.py:100-121) through a depthwise output buffer
    void vov_conv3x3(const std::string& n, View in, View out, int stride, bool dw) {
        if (!dw) {
            vov_conv_norm(n + "/conv", n + "/norm", in, out, 3, stride);
            return;
        }
        View t = alloc(out.H, out.W, in.C);
        dwconv(n + "/dw_conv3x3", in, t, stride);
        vov_conv_norm(n + "/pw_conv1x1", n + "/pw_norm", t, out, 1, 1);
    }
    // VoVNet conv -> norm -> ReLU (get_norm(cfg.NORM), vovnet.py:119,139,159): the BN folded into the conv epilogue, or for GN
    // the raw conv output stored (a channel slice of the concat buffer for the OSA layers), then GroupNorm + ReLU in place on
    // it.  One GN op per conv: every VoVNet conv reads the previous one's normalised output, so none can share a launch.
    void vov_conv_norm(const std::string& conv, const std::string& norm, View in, View out, int ksize, int stride) {
        if (E->backbone_norm != DD3D_NORM_GN) {
            conv1(conv, norm, false, in, out, ksize, stride, true);
            return;
        }
        conv1(conv, "", false, in, out, ksize, stride, false);
        group_norm({out}, &E->gn_affine(norm, out.C), true, nullptr, false);
    }

    void build_vovnet(const VovSpec& S, View input, std::vector<View>* feats) {
        const std::string p = "backbone.bottom_up";
        const int H = input.H, W = input.W;
        const int* stage_ch = S.stage_ch;
        const int* out_ch = S.out_ch;
        const int* blocks = S.blocks;
        const int nl = S.layers;
        View s1 = alloc(H / 2, W / 2, S.stem[0]);
        if (E->backbone_norm == DD3D_NORM_GN) {
            stem(p + ".stem.stem_1/conv", "", "", input, s1, false);
            group_norm({s1}, &E->gn_affine(p + ".stem.stem_1/norm", s1.C), true, nullptr, false);
        } else {
            stem(p + ".stem.stem_1/conv", p + ".stem.stem_1/norm", "", input, s1);
        }
        View s2 = alloc(H / 2, W / 2, S.stem[1]);
        vov_conv3x3(p + ".stem.stem_2", s1, s2, 1, S.dw);
        int h = H / 4, w = W / 4;
        int in_ch = S.stem[2];
        View cat = alloc(h, w, in_ch + nl * stage_ch[0]);
        vov_conv3x3(p + ".stem.stem_3", s2, slice(cat, 0, in_ch), 2, S.dw);
        // the FPN inputs (FE.FPN.IN_FEATURES): the stem (a slice of stage 2's first concat buffer, which nothing overwrites)
        // and stage<first> .. stage5
        const std::vector<int> fpn_in = E->fpn_input_list();
        feats->clear();
        if (fpn_in[0] == DD3D_FPN_IN_STEM) feats->push_back(slice(cat, 0, in_ch));
        View stage_out;
        for (int si = 0; si < 4; ++si) {
            const int sc = stage_ch[si], oc = out_ch[si];
            if (si > 0) {
                const int hp = (h - 3 + 1) / 2 + 1, wp = (w - 3 + 1) / 2 + 1;  // 3x3 / s2, ceil_mode (vovnet.py:249)
                cat = alloc(hp, wp, in_ch + nl * sc);
                maxpool(stage_out, slice(cat, 0, in_ch), 3);
                h = hp;
                w = wp;
            }
            for (int b = 0; b < blocks[si]; ++b) {
                const std::string name = "OSA" + std::to_string(si + 2) + "_" + std::to_string(b + 1);
                const std::string q = p + ".stage" + std::to_string(si + 2) + "." + name;
                View x = slice(cat, 0, in_ch);
                int c0 = in_ch;
                View prev = x;
                if (S.dw && in_ch != sc) {
                    // conv_reduction (vovnet.py:200-205,221-222): feeds layer 0 only; the concat keeps the unreduced input
                    View r = alloc(h, w, sc);
                    const std::string rn = q + ".conv_reduction." + name + "_reduction_0";
                    vov_conv_norm(rn + "/conv", rn + "/norm", x, r, 1, 1);
                    prev = r;
                }
                for (int i = 0; i < nl; ++i) {
                    const std::string ln = q + ".layers." + std::to_string(i) + "." + name + "_" + std::to_string(i);
                    View o = slice(cat, c0, sc);
                    vov_conv3x3(ln, prev, o, 1, S.dw);
                    prev = o;
                    c0 += sc;
                }
                View xt = alloc(h, w, oc);
                vov_conv_norm(q + ".concat." + name + "_concat/conv", q + ".concat." + name + "_concat/norm", cat, xt, 1, 1);
                // eSE (always applied, vovnet.py:216,233) then identity add for non-first blocks (:235-236), after the norm
                View dst;
                View next_cat;
                const bool last = (b == blocks[si] - 1);
                if (last) {
                    dst = alloc(h, w, oc);
                } else {
                    next_cat = alloc(h, w, oc + nl * sc);
                    dst = slice(next_cat, 0, oc);
                }
                ese(q + ".ese.fc", xt, b > 0 ? &x : nullptr, dst);
                if (last) {
                    stage_out = dst;
                } else {
                    cat = next_cat;
                }
                in_ch = oc;
            }
            if (std::find(fpn_in.begin(), fpn_in.end(), si + 2) != fpn_in.end()) feats->push_back(stage_out);
        }
    }

    void ese(const std::string& fc, View xt, const View* identity, View dst) {
        const EseLayer& L = E->ese_layer(fc, xt.C);
        // The concat conv (the op just emitted) writes per-tile channel sums from its epilogue: [B][T][C], T = 4 * tiles.
        // Behind a GroupNorm the eSE pools the normalised map itself (launch_ese): [B][ese_nsplit(HW)][C] partial sums.
        const bool fused = E->backbone_norm != DD3D_NORM_GN;
        const int T = 4 * conv_tiles_per_image(xt.H, xt.W);
        float* tile_partial = fused ? alloc_f32(static_cast<size_t>(B) * T * xt.C) : nullptr;
        float* sums = alloc_f32(static_cast<size_t>(B) * (fused ? 1 : ese_nsplit(xt.H * xt.W)) * xt.C);
        float* gate = alloc_f32(static_cast<size_t>(B) * xt.C);
        touch(xt);
        if (identity) touch(*identity);
        touch(dst);
        ++op_idx;
        if (dry) return;
        if (fused) {
            Op& cv = P->ops.back();
            if (cv.type != Op::CONV || cv.conv.nseg != 1 || cv.conv.halo || cv.conv.out_mode != 0 ||
                4 * cv.conv.seg[0].tiles_x * cv.conv.seg[0].tiles_y != T)
                fail(DD3D_ERR_STATE, "internal: eSE must follow its concat conv");
            cv.conv.seg[0].pool_partial = tile_partial;
            cv.conv.seg[0].pool_pitch = xt.C;
        }
        Op op;
        op.type = Op::ESE;
        op.in = xt;
        op.out = dst;
        op.ese = &L;
        op.has_identity = identity != nullptr;
        if (identity) op.identity = *identity;
        op.f0 = sums;
        op.f1 = gate;
        op.f2 = tile_partial;
        op.ksize = T;
        op.outs[0] = dst;
        op.nouts = 1;
        // pooling is fused into the concat conv, or behind a GroupNorm one more pass over the map
        op.bytes = static_cast<double>(B) * xt.H * xt.W * xt.C * 2 * ((identity ? 3 : 2) + (fused ? 0 : 1));
        P->ops.push_back(op);
    }

    // ---- FPN (detectron2 FPN.forward + top block) -----------------------------------------------------------
    void build_fpn(const std::vector<View>& feats, int first_stage, std::vector<View>* outs) {
        const std::string p = "backbone";
        const int n = static_cast<int>(feats.size());
        // FE.FPN.NORM: BN (folded into the conv epilogue), "" (biased convs) or GN (identity epilogue, then a GN op);
        // FUSE_TYPE avg halves lateral + top-down.  The add follows the norm (detectron2 FPN.forward), so with GN or avg it
        // moves from the lateral conv's epilogue into the GN apply pass.
        const int norm = E->layout.fpn_norm;
        const bool gn = norm == DD3D_NORM_GN, bn = norm == DD3D_NORM_BN_SHARED || norm == DD3D_NORM_BN_PER_LEVEL;
        const bool avg = E->layout.fpn_fuse_avg != 0;
        const int width = E->fpn_channels;  // FE.FPN.OUT_CHANNELS: laterals, outputs, P6 / P7
        // outputs the heads read (DD3D.IN_FEATURES): stage outputs 0 .. n-1, then P6 (n) and P7 (n + 1).  P6 reads output
        // n - 1 and P7 reads P6; lateral i feeds output i and every lateral below it, so the laterals below the lowest output
        // read are skipped too.  The reference still computes them; nothing reads them.
        const bool dla = dla_spec(E->desc.arch) != nullptr;
        bool read[kFpnMaxOutputs + 1] = {};
        for (int l = 0; l < E->num_levels(); ++l) read[E->head_level(l)] = true;
        const bool want_p7 = dla && read[n + 1], want_p6 = read[n] || want_p7;
        std::vector<bool> need(n);
        int lowest = n;
        for (int i = n - 1; i >= 0; --i) {
            need[i] = read[i] || (i == n - 1 && want_p6);
            if (need[i]) lowest = i;
        }
        auto conv_norm = [&](const std::string& name, View in, View out, int ksize, const View* res) {
            conv1(name, bn ? name + ".norm" : "", norm == DD3D_NORM_NONE, in, out, ksize, 1, false, res, res != nullptr);
        };
        std::vector<View> res(n);
        View prev;
        for (int i = n - 1; i >= lowest; --i) {
            const std::string st = std::to_string(first_stage + i);
            const std::string lname = p + ".fpn_lateral" + st, oname = p + ".fpn_output" + st;
            const View& c = feats[i];
            View lat = alloc(c.H, c.W, width);
            if (i == n - 1 || gn || avg) {
                conv_norm(lname, c, lat, 1, nullptr);
                const bool add = i != n - 1;
                if (gn || add) group_norm({lat}, gn ? &E->gn_affine(lname + ".norm", width) : nullptr, false, add ? &prev : nullptr, add && avg);
            } else {
                // lateral + nearest-2x(prev): the un-smoothed `prev` is what propagates downwards
                conv_norm(lname, c, lat, 1, &prev);
            }
            prev = lat;
            if (!need[i]) continue;
            res[i] = alloc(c.H, c.W, width);
            persist(res[i]);
            conv_norm(oname, lat, res[i], 3, nullptr);
            if (gn) group_norm({res[i]}, &E->gn_affine(oname + ".norm", width), false, nullptr, false);
        }
        *outs = res;
        if (!want_p6) {
            outs->resize(E->fpn_outputs());
            return;
        }
        const View& p5 = res[n - 1];
        View p6 = alloc(p5.H / 2, p5.W / 2, width);
        persist(p6);
        conv1(p + ".top_block.p6", "", true, p5, p6, 3, 2, false);
        outs->push_back(p6);
        if (want_p7) {  // LastLevelP6P7
            View r6 = alloc(p6.H, p6.W, width);
            relu(p6, r6);
            View p7 = alloc(p6.H / 2, p6.W / 2, width);
            persist(p7);
            conv1(p + ".top_block.p7", "", true, r6, p7, 3, 2, false);
            outs->push_back(p7);
        }
        outs->resize(E->fpn_outputs());  // VoVNet: P6 is the last; a skipped output stays an empty view
    }

    // ---- heads ------------------------------------------------------------------------------------------------
    // `depth` x (3x3 conv -> norm -> ReLU) over every level in one launch per layer (fcos2d.py:55-91, fcos3d.py:81-112).
    // norm: per-level BN (ModuleListDial, folded per segment), shared BN (one folded epilogue), none (conv bias), or GN
    // (identity epilogue, then one GN op over the levels).  Depth 0: the FPN outputs themselves.  Every layer is as wide as the
    // FPN (FE.FPN.OUT_CHANNELS; the reference's heads take their width from the backbone's output shape).
    void tower(const std::string& tp, int depth, int norm, const std::vector<View>& feats, std::vector<View>* out) {
        const int width = E->fpn_channels;
        std::vector<View> cur = feats;
        std::vector<View> buf[2];
        for (int k = 0; k < std::min(depth, 2); ++k)
            for (auto& f : feats) buf[k].push_back(alloc(f.H, f.W, width));
        for (int i = 0; i < depth; ++i) {
            const std::string wn = tp + "." + std::to_string(i);
            const ConvLayer& L = E->conv_layer(wn, {wn}, width, 3);
            std::vector<SegSpec> segs(feats.size());
            for (size_t l = 0; l < feats.size(); ++l) {
                segs[l].in = cur[l];
                segs[l].out = buf[i & 1][l];
                if (norm == DD3D_NORM_BN_PER_LEVEL) {
                    const std::string bn = wn + ".norm." + std::to_string(l);  // ModuleListDial: level l -> norm l
                    segs[l].epi = &E->bn_epilogue(wn + "|" + bn, bn, "", width);
                } else if (norm == DD3D_NORM_BN_SHARED) {
                    segs[l].epi = &E->bn_epilogue(wn + "|" + wn + ".norm", wn + ".norm", "", width);
                } else {  // none: conv bias; GN: raw conv output, normalised by the GN op below
                    segs[l].epi = &E->bn_epilogue(wn + "|", "", norm == DD3D_NORM_NONE ? wn + ".bias" : "", width);
                }
            }
            const bool gn = norm == DD3D_NORM_GN;
            conv(L, 1, !gn, segs, false);
            if (gn) group_norm(buf[i & 1], &E->gn_affine(wn + ".norm", width), true, nullptr, false);
            cur = buf[i & 1];
        }
        *out = cur;
    }

    // Tile lists of a sparse tower (TowerTilesParams): `depth` lists, list i at distance <= reach - i, on 8x8 tiles (pred16:
    // the last one on the box2d predictor's 16x8 tiles), and the staging, list and count areas in the persistent region.
    // false: the shapes exceed the list entry fields or the layers would not run the pair tile, the tower stays dense.  The
    // pair tile needs a width that 128 divides, so at FPN widths 64, 192, 320 and 448 the sparse box2d / box3d towers always
    // fall back to the dense tower.
    bool tower_tile_lists(TowerTilesParams& tt, const std::vector<View>& feats, int depth, int reach, bool pred16) {
        memset(&tt, 0, sizeof(tt));
        const int L = static_cast<int>(feats.size());
        tt.num_levels = L;
        int hs[kMaxSeg] = {}, ws[kMaxSeg] = {};
        for (int l = 0; l < L; ++l) {
            hs[l] = feats[l].H;
            ws[l] = feats[l].W;
        }
        const int width = E->fpn_channels;
        const bool halo = conv_prefer_halo(9, 1, width, L, hs, ws);
        for (int l = 0; l < L; ++l) {
            TowerTilesLevel& v = tt.lvl[l];
            v.H = hs[l];
            v.W = ws[l];
            v.th = v.tw = kListTile;
            v.tiles_x = (v.W + v.tw - 1) / v.tw;
            v.tiles_y = (v.H + v.th - 1) / v.th;
            const int T = v.tiles_x * v.tiles_y;
            v.stage_begin = tt.cap;
            tt.cap += B * ((T + 3) & ~3);
            tt.max_tiles = std::max(tt.max_tiles, T);
        }
        if (B > kTileListMaxImages || tt.max_tiles >= kTileListMaxTiles || tower_tiles_smem_bytes(tt.max_tiles) > 48 * 1024)
            return false;
        // the work-list mode is built for the pair tile, which every filled halo layer of a 128-multiple width selects (conv());
        // the fill rule looks at the dense tower's 16x8 tiles
        ConvParams cp;
        memset(&cp, 0, sizeof(cp));
        cp.nseg = L;
        cp.B = B;
        cp.halo = halo ? 1 : 0;
        for (int l = 0; l < L; ++l) {
            cp.seg[l].H = hs[l];
            cp.seg[l].W = ws[l];
            cp.seg[l].th = kHaloTh;
            cp.seg[l].tw = kHaloTw;
        }
        if (!conv_select_pair(&cp, width, E->num_sms)) return false;
        tt.B = B;
        tt.depth = depth;
        tt.reach = reach;
        tt.pred16 = pred16 ? 1 : 0;
        const size_t list_bytes = static_cast<size_t>(depth) * tt.cap * 4, bl_bytes = static_cast<size_t>(depth) * L * B * 4;
        tt.stage = static_cast<uint32_t*>(alloc_bytes(list_bytes));
        tt.list = static_cast<uint32_t*>(alloc_bytes(list_bytes));
        tt.bl_count = static_cast<int32_t*>(alloc_bytes(bl_bytes));
        tt.bl_pixels = static_cast<int32_t*>(alloc_bytes(bl_bytes));
        tt.count = static_cast<int32_t*>(alloc_bytes(static_cast<size_t>(depth) * 4));
        tt.pixels = static_cast<long long*>(alloc_bytes(static_cast<size_t>(depth) * 8));
        tt.ticket = static_cast<uint32_t*>(alloc_bytes(4));
        return true;
    }

    // Points plan ops [begin, begin + tt.depth) -- tower convs on the pair tile (built with list_tiles), then (box2d) the
    // taps-in-N predictor -- at their tile lists.
    void use_tile_lists(int begin, const TowerTilesParams& tt, int L, const char* what) {
        for (int j = 0; j < tt.depth; ++j) {
            Op& op = P->ops[begin + j];
            ConvParams& c = op.conv;
            const bool pred = tt.pred16 && j == tt.depth - 1;
            if (op.type != Op::CONV || c.nseg != L || !(pred ? c.taps_n : c.pair))
                fail(DD3D_ERR_STATE, std::string("internal: sparse ") + what + " layout");
            for (int l = 0; l < L; ++l)
                if (c.seg[l].th != (pred ? 2 * tt.lvl[l].th : tt.lvl[l].th) || c.seg[l].tw != tt.lvl[l].tw)
                    fail(DD3D_ERR_STATE, std::string("internal: sparse ") + what + " tiling");
            c.tile_list = tt.list + static_cast<size_t>(j) * tt.cap;
            c.tile_count = tt.count + j;
            conv_finalize_params(&c);  // the list-mode pair tile lays out its shared memory differently
        }
    }

    void build_heads(const std::vector<View>& feats) {
        const int C = E->desc.num_classes;
        const int L = static_cast<int>(feats.size());
        const int width = E->fpn_channels;  // input channels of every predictor
        const bool nusc = E->desc.nuscenes_heads != 0;
        // head switches no shipped experiment changes (dd3d_model_desc): class-agnostic 3-D channels, per-level predictors,
        // no Scale / Offset layers, no 3-D head at all
        const bool use_scale2 = E->desc.fcos2d_use_scale != 0, use_scale3 = E->desc.fcos3d_use_scale != 0;
        const bool per_level = E->desc.per_level_predictors != 0, box3d_on = E->desc.box3d_on != 0;
        const int C3 = E->desc.class_agnostic_box3d ? 1 : C;
        const int cls_pitch = round_up(C + (nusc ? kNumAttributes + 1 : 0), 16), b3d_pitch = cout_padded(11 * C3);
        // sparse box3d predictor: forced (1), off (0) or auto (2, default).  The dense launch costs time in proportion to the
        // head pixels, the gathered one a near-constant latency-bound K loop, so large heads go sparse.  The rule looks at
        // the head pixels of ONE image, not of the batch, so that an image gives bit-identical detections whatever batch it
        // rides in (the two predictors differ in fp32 summation order): 900x1600 V2-99 = 127 875 pixels -> sparse at every
        // batch size, 384x1280 DLA-34 = 10 230 -> dense.
        size_t head_px = 0;
        for (int l = 0; l < L; ++l) head_px += static_cast<size_t>(feats[l].H) * feats[l].W;
        // Class-specific heads wider than the sparse kernel's registers (C3 > 10) take the class-gathered predictor
        // (b3d_gather.cu) under the same rule; C3 11..16 keep the dense predictor, as before that kernel existed.
        const bool gather3 = box3d_on && C3 > DD3D_MAX_CLASSES;
        const bool sparse3 = box3d_on && (b3d_pitch <= kB3dSparseMaxN || gather3) &&
                             (E->opt_sparse_box3d == 1 || (E->opt_sparse_box3d == 2 && head_px >= 50000));
        const int rows_pitch = gather3 ? kB3dGatherPitch : b3d_pitch;
        P->sparse_b3d = sparse3;
        P->gather_b3d = sparse3 && gather3;
        P->b3d_rows = sparse3 ? alloc_f32(static_cast<size_t>(B) * L * E->desc.pre_nms_topk * rows_pitch) : nullptr;
        P->b3d_gather_scratch =
            P->gather_b3d ? alloc_bytes(b3d_gather_scratch_bytes(B, C, E->desc.pre_nms_topk, L)) : nullptr;
        P->num_levels = L;
        P->cls_pitch = cls_pitch;
        P->b3d_pitch = b3d_pitch;
        // each tower is followed at once by its predictor, so that its ping-pong buffers die before the next tower starts
        // (arena reuse); the launch order differs from fcos2d.py:130-156 / fcos3d.py:160-188, the arithmetic does not
        std::vector<View> cls_t, box_t, b3d_t;
        for (int l = 0; l < L; ++l) {
            const size_t hw = static_cast<size_t>(B) * feats[l].H * feats[l].W;
            P->cls_map[l] = alloc_f32(hw * cls_pitch);
            P->box_map[l] = alloc_f32(hw * 16);
            P->b3d_map[l] = (box3d_on && !sparse3) ? alloc_f32(hw * b3d_pitch) : nullptr;
            P->lvl_h[l] = feats[l].H;
            P->lvl_w[l] = feats[l].W;
        }
        // cls_logits (fcos2d.py:96,142): bias only, shared across levels.  NuscenesDD3D adds attr_logits (3) and
        // relu(speed) (1) on the same tower output (nuscenes_dd3d.py:311-312,380-383): fused as extra GEMM columns
        // [cls C | attr 3 | speed 1] of the one predictor conv (still N = 16 for the 10 nuScenes classes).
        tower("fcos2d_head.cls_tower", E->layout.num_cls_convs, E->layout.fcos2d_norm, feats, &cls_t);
        {
            std::vector<std::string> names = {"fcos2d_head.cls_logits"};
            if (nusc) {
                names.push_back("attr_logits");
                names.push_back("speed");
            }
            const ConvLayer& Lc = E->conv_layer(nusc ? "fcos2d_head.cls_logits+attr+speed" : "fcos2d_head.cls_logits",
                                                names, width, 3);
            const std::string ekey = "fcos2d_head.cls_logits|";
            if (E->epis.find(ekey) == E->epis.end()) {
                std::vector<float> sc, bi, lo;
                for (auto& n : names) {
                    const HostTensor& b = E->weight(n + ".bias");
                    for (float v : b.data) {
                        sc.push_back(1.0f);
                        bi.push_back(v);
                        lo.push_back(n == "speed" ? 0.0f : -INFINITY);
                    }
                }
                if (static_cast<int>(sc.size()) != Lc.cout) fail(DD3D_ERR_INVALID, "bad cls predictor bias shapes");
                E->epilogue(ekey, sc, bi, nusc ? &lo : nullptr);
            }
            const Epilogue& e = E->epis.at(ekey);
            std::vector<SegSpec> segs(L);
            for (int l = 0; l < L; ++l) {
                segs[l].in = cls_t[l];
                segs[l].epi = &e;
                segs[l].out_f32 = P->cls_map[l];
                segs[l].out_pitch = cls_pitch;
            }
            conv(Lc, 1, false, segs, true);
        }
        // sparse box2d tower: the decode reads the box map only at the pixels where some class passes the threshold alone
        // (class_passes, detect.cuh), which the cls map above decides.  So the tower runs on the tiles within d2 - i of them
        // and the taps-in-N predictor on the tiles that meet them, listed right before the tower (GN needs whole-map
        // statistics).  Auto follows the sparse box3d predictor, which the stage-level tests switch off to read dense maps.
        const int d2 = E->layout.num_box2d_convs;
        int hs[kMaxSeg], ws[kMaxSeg];
        for (int l = 0; l < L; ++l) {
            hs[l] = feats[l].H;
            ws[l] = feats[l].W;
        }
        const bool sparse_box2d =
            d2 > 0 && E->layout.fcos2d_norm != DD3D_NORM_GN &&
            (E->opt_sparse_box2d_tower == 1 || (E->opt_sparse_box2d_tower == 2 && sparse3 && head_px >= 50000)) &&
            conv_taps_eligible(9, 1, 16, L, hs, ws) && tower_tile_lists(P->box2d_tiles, feats, d2 + 1, d2, true);
        P->box2d_begin = sparse_box2d ? static_cast<int>(P->ops.size()) : -1;
        if (sparse_box2d) {
            TowerTilesParams& tt = P->box2d_tiles;
            tt.dist = static_cast<int32_t*>(alloc_bytes(static_cast<size_t>(tt.cap) * 4));
            tt.cls_pitch = cls_pitch;
            for (int l = 0; l < L; ++l) {
                tt.lvl[l].cls = P->cls_map[l];
                tt.lvl[l].mark_begin = tt.mark_blocks;
                tt.mark_blocks += (feats[l].H * feats[l].W + kTowerMarkThreads - 1) / kTowerMarkThreads;
            }
        }
        // [box2d_reg (4) | centerness (1)] on the box2d tower: relu(scale_l * (conv + b)) / conv + b (fcos2d.py:143-152)
        list_tiles = sparse_box2d;
        tower("fcos2d_head.box2d_tower", d2, E->layout.fcos2d_norm, feats, &box_t);
        list_tiles = false;
        {
            const ConvLayer& Lb = E->conv_layer("fcos2d_head.box2d_reg+centerness",
                                                {"fcos2d_head.box2d_reg", "fcos2d_head.centerness"}, width, 3);
            std::vector<SegSpec> segs(L);
            for (int l = 0; l < L; ++l) {
                const std::string key = "fcos2d_head.box@" + std::to_string(l);
                if (E->epis.find(key) == E->epis.end()) {
                    const float s = use_scale2 ? E->weight("fcos2d_head.scales_box2d_reg." + std::to_string(l) + ".scale").data[0]
                                               : 1.0f;  // fcos2d.py:145-152
                    const HostTensor& br = E->weight("fcos2d_head.box2d_reg.bias");
                    const HostTensor& bc = E->weight("fcos2d_head.centerness.bias");
                    std::vector<float> sc(5), bi(5), lo(5);
                    for (int k = 0; k < 4; ++k) {
                        sc[k] = s;
                        bi[k] = br.data[k] * s;
                        lo[k] = 0.0f;
                    }
                    sc[4] = 1.0f;
                    bi[4] = bc.data[0];
                    lo[4] = -INFINITY;
                    E->epilogue(key, sc, bi, &lo);
                }
                segs[l].in = box_t[l];
                segs[l].epi = &E->epis.at(key);
                segs[l].out_f32 = P->box_map[l];
                segs[l].out_pitch = 16;
            }
            conv(Lb, 1, false, segs, true);
        }
        if (sparse_box2d && !dry) use_tile_lists(P->box2d_begin, P->box2d_tiles, L, "box2d tower");
        // [quat 4C | ctr 2C | depth C | size 3C | conf C] on the box3d tower with the per-level Scale/Offset folded
        // (fcos3d.py:166-180; PER_LEVEL_PREDICTORS False -> predictor index 0)
        if (!box3d_on) return;  // MODEL.BOX3D_ON = False (core.py:34-40): 2-D detector only
        // sparse box3d tower: the sparse predictor reads the tower output only around the final candidates, so the tower runs
        // after the threshold / top-k half of the decode on the tiles tower_tiles_kernel lists (GN needs whole-map statistics).
        // It is the last part of the op list, so its buffers keep the lifetimes of the dense order: the decode between the
        // two parts touches only the persistent region.
        const int d3 = E->layout.num_box3d_convs;
        const bool sparse_tower = sparse3 && d3 > 0 && E->layout.fcos3d_norm != DD3D_NORM_GN &&
                                  (E->opt_sparse_tower == 1 || (E->opt_sparse_tower == 2 && head_px >= 50000)) &&
                                  tower_tile_lists(P->tower_tiles, feats, d3, d3, false);
        P->tower_begin = sparse_tower ? static_cast<int>(P->ops.size()) : -1;
        list_tiles = sparse_tower;
        tower("fcos3d_head.box3d_tower", d3, E->layout.fcos3d_norm, feats, &b3d_t);
        list_tiles = false;
        if (sparse_tower && !dry) use_tile_lists(P->tower_begin, P->tower_tiles, L, "box3d tower");
        // [quat 4C | ctr 2C | depth C | size 3C | conf C] on the box3d tower with the per-level Scale/Offset folded
        // (fcos3d.py:166-180).  PER_LEVEL_PREDICTORS False (shipped): predictor index 0 for every level, one launch over the
        // five levels; True: level l uses predictor l, one launch per level.
        {
            auto layer_for = [&](int li) -> const ConvLayer& {
                const std::string i = std::to_string(li);
                return E->conv_layer("fcos3d_head.box3d_all." + i,
                                     {"fcos3d_head.box3d_quat." + i, "fcos3d_head.box3d_ctr." + i, "fcos3d_head.box3d_depth." + i,
                                      "fcos3d_head.box3d_size." + i, "fcos3d_head.box3d_conf." + i},
                                     width, 3);
            };
            std::vector<SegSpec> segs(L);
            for (int l = 0; l < L; ++l) {
                const std::string key = "fcos3d_head.b3d@" + std::to_string(l);
                if (E->epis.find(key) == E->epis.end()) {
                    const std::string ls = std::to_string(l), pi = std::to_string(per_level ? l : 0);
                    auto scalar = [&](const std::string& n, float dflt) { return use_scale3 ? E->weight(n).data[0] : dflt; };
                    const float s_ctr = scalar("fcos3d_head.scales_proj_ctr." + ls + ".scale", 1.0f);
                    const float s_size = scalar("fcos3d_head.scales_size." + ls + ".scale", 1.0f);
                    const float s_conf = scalar("fcos3d_head.scales_conf." + ls + ".scale", 1.0f);
                    const float s_depth = scalar("fcos3d_head.scales_depth." + ls + ".scale", 1.0f);
                    const float o_depth = scalar("fcos3d_head.offsets_depth." + ls + ".bias", 0.0f);
                    std::vector<float> sc(11 * C3), bi(11 * C3);
                    auto fill = [&](int c0, int n, float s, const std::string& bias_name, float add) {
                        const bool has = E->weights.find(bias_name) != E->weights.end();
                        for (int k = 0; k < n; ++k) {
                            sc[c0 + k] = s;
                            bi[c0 + k] = (has ? E->weight(bias_name).data[k] : 0.0f) * s + add;
                        }
                    };
                    fill(0, 4 * C3, 1.0f, "fcos3d_head.box3d_quat." + pi + ".bias", 0.f);
                    fill(4 * C3, 2 * C3, s_ctr, "fcos3d_head.box3d_ctr." + pi + ".bias", 0.f);
                    fill(6 * C3, C3, s_depth, "fcos3d_head.box3d_depth." + pi + ".bias", o_depth);  // bias only without USE_SCALE
                    fill(7 * C3, 3 * C3, s_size, "fcos3d_head.box3d_size." + pi + ".bias", 0.f);
                    fill(10 * C3, C3, s_conf, "fcos3d_head.box3d_conf." + pi + ".bias", 0.f);
                    E->epilogue(key, sc, bi, nullptr);
                }
                segs[l].in = b3d_t[l];
                segs[l].epi = &E->epis.at(key);
                segs[l].out_f32 = P->b3d_map[l];
                segs[l].out_pitch = b3d_pitch;
            }
            if (sparse3 && gather3) {
                // as below, on the class-gathered kernel: 11 channels per candidate, those of its own class
                B3dGatherParams& gp = P->b3d_gather;
                memset(&gp, 0, sizeof(gp));
                for (int l = 0; l < L; ++l) {
                    const ConvLayer& Lw = layer_for(per_level ? l : 0);
                    touch(b3d_t[l]);
                    gp.lvl[l].in = b3d_t[l].ptr;
                    gp.lvl[l].H = b3d_t[l].H;
                    gp.lvl[l].W = b3d_t[l].W;
                    gp.lvl[l].pitch = b3d_t[l].pitch;
                    gp.lvl[l].w = Lw.d_w;
                    gp.lvl[l].scale = segs[l].epi->d_scale;
                    gp.lvl[l].bias = segs[l].epi->d_bias;
                    if (Lw.cout < 11 * C || Lw.cin != width) fail(DD3D_ERR_INVALID, "box3d predictor shape");
                }
                ++op_idx;
                gp.rows = P->b3d_rows;
                gp.num_levels = L;
                gp.B = B;
                gp.C = C;
                gp.topk = E->desc.pre_nms_topk;
                gp.fp16 = E->fp16;
                gp.cin = width;
                if (!dry) b3d_gather_bind_scratch(&gp, P->b3d_gather_scratch);
            } else if (sparse3) {
                // no dense launch: the predictor runs on the final candidates, after the threshold / top-k half of the decode
                // (Engine::forward).  The tower outputs must outlive every op: a phantom op index keeps them in the arena.
                B3dSparseParams& sp = P->b3d_sparse;
                memset(&sp, 0, sizeof(sp));
                for (int l = 0; l < L; ++l) {
                    const ConvLayer& Lw = layer_for(per_level ? l : 0);
                    touch(b3d_t[l]);
                    sp.lvl[l].in = b3d_t[l].ptr;
                    sp.lvl[l].H = b3d_t[l].H;
                    sp.lvl[l].W = b3d_t[l].W;
                    sp.lvl[l].pitch = b3d_t[l].pitch;
                    sp.lvl[l].w = Lw.d_w;
                    sp.lvl[l].scale = segs[l].epi->d_scale;
                    sp.lvl[l].bias = segs[l].epi->d_bias;
                    if (Lw.cout_pad != b3d_pitch || Lw.cin != width) fail(DD3D_ERR_INVALID, "box3d predictor shape");
                }
                ++op_idx;
                sp.rows = P->b3d_rows;
                sp.num_levels = L;
                sp.B = B;
                sp.C = C;
                sp.topk = E->desc.pre_nms_topk;
                sp.n_pad = b3d_pitch;
                sp.out_pitch = b3d_pitch;
                sp.fp16 = E->fp16;
                sp.cin = width;
            } else if (!per_level) {
                conv(layer_for(0), 1, false, segs, true);
            } else {
                for (int l = 0; l < L; ++l) {
                    std::vector<SegSpec> one(1, segs[l]);
                    conv(layer_for(l), 1, false, one, true);
                }
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------ misc layers

// VoVNet stem_1 in the layout stem_mma.cu reads: [64][3][4][4] (cout, ky, kx, c; kernel column 3 and the 4th input channel
// are zero); folded BN as scale[64] | bias[64].
const StemLayer& Engine::stem_layer(const std::string& wname, const std::string& bn, const std::string& conv_bias_name,
                                    bool relu) {
    auto it = stems.find(wname);
    if (it != stems.end()) return it->second;
    const HostTensor& w = weight(wname + ".weight");
    if (w.shape.size() != 4 || w.shape[0] != 64 || w.shape[1] != 3 || w.shape[2] != 3 || w.shape[3] != 3)
        fail(DD3D_ERR_INVALID, "bad stem weight: " + wname);
    StemLayer S;
    S.relu = relu;
    std::vector<uint16_t> pm(64 * 3 * 4 * 4, 0);
    for (int co = 0; co < 64; ++co)
        for (int c = 0; c < 3; ++c)
            for (int ky = 0; ky < 3; ++ky)
                for (int kx = 0; kx < 3; ++kx)
                    pm[((co * 3 + ky) * 4 + kx) * 4 + c] = host_f32_to_act(w.data[((co * 3 + c) * 3 + ky) * 3 + kx], fp16);
    S.d_w = static_cast<__nv_bfloat16*>(dev_alloc(pm.size() * 2));
    cuda_check(cudaMemcpy(S.d_w, pm.data(), pm.size() * 2, cudaMemcpyHostToDevice), "upload stem weights");
    std::vector<float> sc, bi;
    bn_fold(bn, conv_bias_name, 64, &sc, &bi);
    sc.insert(sc.end(), bi.begin(), bi.end());
    S.d_sb = upload_f32(sc);
    return stems.emplace(wname, S).first->second;
}

// DLA-34 base_layer / level0 / level1 in the layouts dla_front.cu reads: base_layer [16][7][8][4] (kernel column 7 and
// the 4th input channel are zero), level0 [16][9][16], level1 [32][9][16]; folded BN as scale[cout] | bias[cout].
const FrontLayer& Engine::front_layer(const std::string& prefix) {
    auto it = fronts.find(prefix);
    if (it != fronts.end()) return it->second;
    const HostTensor& w0 = weight(prefix + ".base_layer.weight");
    const HostTensor& w1 = weight(prefix + ".level0.0.weight");
    const HostTensor& w2 = weight(prefix + ".level1.0.weight");
    auto is = [](const HostTensor& w, int64_t a, int64_t b, int64_t k) {
        return w.shape.size() == 4 && w.shape[0] == a && w.shape[1] == b && w.shape[2] == k && w.shape[3] == k;
    };
    if (!is(w0, 16, 3, 7) || !is(w1, 16, 16, 3) || !is(w2, 32, 16, 3)) fail(DD3D_ERR_INVALID, "bad DLA front weights: " + prefix);
    std::vector<uint16_t> p0(16 * 7 * 8 * 4, 0), p1(16 * 9 * 16, 0), p2(32 * 9 * 16, 0);
    for (int co = 0; co < 16; ++co)
        for (int c = 0; c < 3; ++c)
            for (int ky = 0; ky < 7; ++ky)
                for (int kx = 0; kx < 7; ++kx)
                    p0[((co * 7 + ky) * 8 + kx) * 4 + c] = host_f32_to_act(w0.data[((co * 3 + c) * 7 + ky) * 7 + kx], fp16);
    for (int co = 0; co < 16; ++co)
        for (int ci = 0; ci < 16; ++ci)
            for (int t = 0; t < 9; ++t) p1[(co * 9 + t) * 16 + ci] = host_f32_to_act(w1.data[(co * 16 + ci) * 9 + t], fp16);
    for (int co = 0; co < 32; ++co)
        for (int ci = 0; ci < 16; ++ci)
            for (int t = 0; t < 9; ++t) p2[(co * 9 + t) * 16 + ci] = host_f32_to_act(w2.data[(co * 16 + ci) * 9 + t], fp16);
    auto up16 = [&](const std::vector<uint16_t>& v) {
        __nv_bfloat16* d = static_cast<__nv_bfloat16*>(dev_alloc(v.size() * 2));
        cuda_check(cudaMemcpy(d, v.data(), v.size() * 2, cudaMemcpyHostToDevice), "upload DLA front weights");
        return d;
    };
    auto sb = [&](const std::string& conv, int cout) {  // folded BN, or the conv bias with FE.BACKBONE.NORM ""
        const bool none = backbone_norm == DD3D_NORM_NONE;
        std::vector<float> s, b;
        bn_fold(none ? "" : conv + ".norm", none ? conv + ".bias" : "", cout, &s, &b);
        s.insert(s.end(), b.begin(), b.end());
        return upload_f32(s);
    };
    FrontLayer F;
    F.d_w0 = up16(p0);
    F.d_w1 = up16(p1);
    F.d_w2 = up16(p2);
    F.d_sb0 = sb(prefix + ".base_layer", 16);
    F.d_sb1 = sb(prefix + ".level0.0", 16);
    F.d_sb2 = sb(prefix + ".level1.0", 32);
    return fronts.emplace(prefix, F).first->second;
}

const EseLayer& Engine::ese_layer(const std::string& fc, int C) {
    auto it = eses.find(fc);
    if (it != eses.end()) return it->second;
    const HostTensor& w = weight(fc + ".weight");
    const HostTensor& b = weight(fc + ".bias");
    if (static_cast<int>(w.data.size()) != C * C || static_cast<int>(b.data.size()) != C)
        fail(DD3D_ERR_INVALID, "bad eSE fc shape: " + fc);
    EseLayer L;
    L.C = C;
    L.d_w = upload_f32(w.data);
    L.d_b = upload_f32(b.data);
    return eses.emplace(fc, L).first->second;
}

// ================================================================================================ plan / forward

int Engine::size_divisibility() const { return dla_spec(desc.arch) != nullptr ? 128 : 64; }

// Offsets for the activation buffers: largest first, each at the lowest address where it does not collide (in address
// AND lifetime) with an already placed one -- the greedy interval packing of static memory planners.  Without reuse
// (opt_workspace_reuse = 0) buffers are simply laid out one after the other.  Returns the arena size.
static size_t plan_arena(std::vector<ArenaBuf>& bufs, bool reuse) {
    size_t total = 0;
    if (!reuse) {
        for (ArenaBuf& b : bufs) {
            b.offset = total;
            total += b.bytes;
        }
        return total;
    }
    const int last_op = 1 << 29;
    for (ArenaBuf& b : bufs) {
        if (b.last < 0) {  // never touched by an op (cannot happen for a well-formed graph): keep it alive throughout
            b.first = 0;
            b.last = last_op;
        }
        if (b.persistent) b.last = last_op;
    }
    std::vector<int> order(bufs.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = static_cast<int>(i);
    std::sort(order.begin(), order.end(), [&](int a, int b) {
        return bufs[a].bytes != bufs[b].bytes ? bufs[a].bytes > bufs[b].bytes : a < b;
    });
    std::vector<int> placed;
    for (int id : order) {
        ArenaBuf& b = bufs[id];
        std::vector<std::pair<size_t, size_t>> busy;  // address ranges of placed buffers alive at the same time
        for (int o : placed) {
            const ArenaBuf& q = bufs[o];
            if (q.first <= b.last && b.first <= q.last) busy.emplace_back(q.offset, q.offset + q.bytes);
        }
        std::sort(busy.begin(), busy.end());
        size_t at = 0;
        for (auto& r : busy) {
            if (at + b.bytes <= r.first) break;
            at = std::max(at, r.second);
        }
        b.offset = at;
        total = std::max(total, at + b.bytes);
        placed.push_back(id);
    }
    return total;
}

size_t Engine::build(Plan* P, int B, int Hs, int Ws, void* workspace, bool dry) {
    const int d = size_divisibility();
    const int Hp = round_up(Hs, d), Wp = round_up(Ws, d);
    std::vector<ArenaBuf> bufs;
    size_t arena_bytes = 0, total = 0;
    // pass 0: trace (liveness of every activation buffer, layer creation); pass 1: the real walk with the planned offsets
    for (int pass = 0; pass < (dry ? 1 : 2); ++pass) {
        const bool tracing = pass == 0;
        P->B = B; P->Hs = Hs; P->Ws = Ws; P->Hp = Hp; P->Wp = Wp;
        P->ops.clear();
        Builder bld;
        bld.E = this;
        bld.P = P;
        bld.dry = tracing;
        bld.tracing = tracing;
        bld.bufs = &bufs;
        bld.base = tracing ? nullptr : static_cast<uint8_t*>(workspace);
        bld.B = B;
        bld.off = arena_bytes;  // persistent region follows the activation arena (0 while tracing: sizes only)
        View input;
        input.B = B; input.H = Hp; input.W = Wp; input.C = 4; input.pitch = 4;
        input.ptr = tracing ? nullptr : reinterpret_cast<__nv_bfloat16*>(bld.base + bld.off);
        bld.off += round_up_sz(static_cast<size_t>(B) * Hp * Wp * 4 * 2, 1024);
        P->input = input;
        std::vector<View> feats, fpn;
        if (dla_spec(desc.arch) != nullptr)
            bld.build_dla(input, &feats);
        else
            bld.build_vovnet(*vovnet_spec(desc.arch), input, &feats);
        bld.build_fpn(feats, fpn_first_stage(), &fpn);
        if (static_cast<int>(fpn.size()) != fpn_outputs()) fail(DD3D_ERR_STATE, "internal: FPN output count");
        for (int l = 0; l < fpn_outputs(); ++l) P->fpn[l] = fpn[l];
        std::vector<View> heads(num_levels());  // the FPN outputs in DD3D.IN_FEATURES order
        for (int l = 0; l < num_levels(); ++l) heads[l] = fpn[head_level(l)];
        bld.build_heads(heads);
        // detection scratch + staging for the host-facing path
        P->detect_scratch = bld.alloc_bytes(decode_scratch_bytes(B, desc.pre_nms_topk, num_levels()));
        P->nms_scratch = bld.alloc_bytes(nms_scratch_bytes(B, desc.pre_nms_topk, desc.num_classes, num_levels()));
        P->d_K = static_cast<float*>(bld.alloc_bytes(static_cast<size_t>(B) * 9 * 4));
        P->d_sizes = static_cast<int32_t*>(bld.alloc_bytes(static_cast<size_t>(B) * 4 * 4));
        P->d_out = static_cast<Det*>(bld.alloc_bytes(static_cast<size_t>(B) * desc.out_cap * sizeof(Det)));
        P->d_counts = static_cast<int32_t*>(bld.alloc_bytes(static_cast<size_t>(B) * 4));
        P->d_images = bld.alloc_bytes(static_cast<size_t>(B) * 3 * Hs * Ws * 4);
        P->d_canon = nullptr;
        P->bev = bev_mode();
        P->agg = agg_mode();
        if (P->bev || P->agg) P->d_poses = static_cast<float*>(bld.alloc_bytes(static_cast<size_t>(B) * 7 * 4));
        if (P->bev == kBevPathMultiCta) P->bev_scratch = bld.alloc_bytes(image_bev_nms_scratch_bytes(B, desc.out_cap, desc.num_classes));
        if (P->agg) {
            if (P->agg == kAggPathBlocked && B > kGroupBevNmsLargeMaxB)
                fail(DD3D_ERR_INVALID, "the blocked sample aggregation holds at most " + std::to_string(kGroupBevNmsLargeMaxB) +
                                           " images per call, plan has " + std::to_string(B));
            P->d_group = static_cast<int32_t*>(bld.alloc_bytes(static_cast<size_t>(B) * 4));
            P->d_global = static_cast<float*>(bld.alloc_bytes(static_cast<size_t>(B) * desc.out_cap * 10 * 4));
            P->agg_scratch = bld.alloc_bytes(P->agg == kAggPathOneCta
                                                 ? sample_aggregate_scratch_bytes(B, desc.out_cap)
                                                 : group_bev_nms_large_scratch_bytes(B, desc.out_cap, kGroupBevNmsLargeGroupImages));
        }
        if (tracing) {
            arena_bytes = plan_arena(bufs, opt_workspace_reuse != 0);
            total = arena_bytes + bld.off;
        }
    }
    P->arena_bytes = arena_bytes;
    return total;
}

void Engine::finalize() {
    if (finalized) return;
    // dry graph walk with the smallest legal shape: creates (packs + uploads) every layer and names the first
    // missing tensor, without needing a workspace.
    Plan tmp;
    if (num_levels() > kLevels)
        fail(DD3D_ERR_INVALID, std::to_string(fpn_outputs()) + " FPN outputs need dd3d_set_in_features with at most " +
                                   std::to_string(kLevels) + " of them");
    if (canonical_sizes.empty() && desc.num_classes > DD3D_MAX_CLASSES && desc.box3d_on)
        fail(DD3D_ERR_STATE, "num_classes " + std::to_string(desc.num_classes) + " > " + std::to_string(DD3D_MAX_CLASSES) +
                                 " needs dd3d_set_canonical_sizes before dd3d_finalize");
    build(&tmp, 1, size_divisibility(), size_divisibility(), nullptr, true);
    std::vector<float> canon(desc.canonical_box3d_sizes, desc.canonical_box3d_sizes + DD3D_MAX_CLASSES * 3);
    if (!canonical_sizes.empty()) canon = canonical_sizes;
    d_canon = upload_f32(canon);
    finalized = true;
    weights.clear();  // host copies are no longer needed
}

size_t Engine::workspace_bytes(int B, int Hs, int Ws) {
    if (!finalized) fail(DD3D_ERR_STATE, "workspace_bytes before finalize");
    Plan tmp;
    return build(&tmp, B, Hs, Ws, nullptr, true);
}

void Engine::free_plan(Plan* P) {
    if (P->owned_workspace) cudaFree(P->owned_workspace);
    if (P->slot1) cudaFree(P->slot1);
    *P = Plan();
}

void Engine::release_plan() { free_plan(&plan); }

void Engine::drop_plans() {
    if (slot_busy[0] || slot_busy[1]) fail(DD3D_ERR_STATE, "plan change with a pending dd3d_submit_host");
    ++generation;
    release_plan();
    for (auto& kv : plan_cache) free_plan(&kv.second);
    plan_cache.clear();
}

void Engine::make_plan(int B, int Hs, int Ws, void* workspace, size_t bytes) {
    if (!finalized) fail(DD3D_ERR_STATE, "plan before finalize");
    if (B < 1 || Hs < 1 || Ws < 1) fail(DD3D_ERR_INVALID, "bad plan shape");
    if (slot_busy[0] || slot_busy[1]) fail(DD3D_ERR_STATE, "plan change with a pending dd3d_submit_host");
    ++generation;  // even a same-shape call: captured forwards of the old plan are stale
    cuda_check(cudaSetDevice(device), "cudaSetDevice");
    if (workspace == nullptr && plan.valid && plan.owned_workspace && plan.B == B && plan.Hs == Hs && plan.Ws == Ws &&
        opt_workspace_fill < 0)
        return;
    // park the active plan if it is engine-owned and small, else free it
    if (plan.valid && plan.owned_workspace && plan.owned_bytes <= kPlanCacheBytes) {
        if (plan_cache.size() >= kPlanCacheMax) {
            free_plan(&plan_cache.begin()->second);
            plan_cache.erase(plan_cache.begin());
        }
        plan_cache[{plan.B, plan.Hs, plan.Ws}] = std::move(plan);
        plan = Plan();
    } else {
        release_plan();
    }
    if (workspace == nullptr && opt_workspace_fill < 0) {
        auto it = plan_cache.find({B, Hs, Ws});
        if (it != plan_cache.end()) {
            plan = std::move(it->second);
            plan_cache.erase(it);
            return;
        }
    }
    const size_t need = workspace_bytes(B, Hs, Ws);
    if (workspace == nullptr) {
        cuda_check(cudaMalloc(&plan.owned_workspace, need), "cudaMalloc(workspace)");
        plan.owned_bytes = need;
        workspace = plan.owned_workspace;
    } else if (bytes < need) {
        fail(DD3D_ERR_INVALID, "workspace too small: need " + std::to_string(need) + " bytes");
    }
    if (reinterpret_cast<uintptr_t>(workspace) % 1024) fail(DD3D_ERR_INVALID, "workspace must be 1024-byte aligned");
    // Every byte a kernel reads is written earlier in the same forward, so the arena needs no clearing.  Option
    // "workspace_fill" (0..255; -1 = leave as is) proves it: tests plan once over 0x00 and once over 0xFF (= NaN in bf16
    // and fp32) and require bit-identical maps and detections (tests/test_determinism_gpu.py).
    if (opt_workspace_fill >= 0) {
        cuda_check(cudaMemset(workspace, opt_workspace_fill, need), "cudaMemset(workspace)");
        cuda_check(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    }
    build(&plan, B, Hs, Ws, workspace, false);
    plan.valid = true;
    // decode / NMS parameter blocks
    DecodeParams& dp = plan.decode;
    memset(&dp, 0, sizeof(dp));
    for (int l = 0; l < plan.num_levels; ++l) {  // compute_locations with the strides of the selected levels
        dp.lvl[l].cls = plan.cls_map[l];
        dp.lvl[l].box = plan.box_map[l];
        dp.lvl[l].b3d = plan.b3d_map[l];
        dp.lvl[l].H = plan.lvl_h[l];
        dp.lvl[l].W = plan.lvl_w[l];
        dp.lvl[l].stride = 1 << (fpn_first_stage() + head_level(l));  // FPN output i has stride 2^(first stage + i)
    }
    fill_decode_params(&dp, desc, B, plan.cls_pitch, plan.b3d_pitch, d_canon, plan.num_levels);
    decode_bind_scratch(&dp, plan.detect_scratch);
    decode_finalize_params(&dp);
    if (plan.gather_b3d) {
        dp.b3d_rows = plan.b3d_rows;
        dp.b3d_pitch = kB3dGatherPitch;
        dp.b3d_by_class = 1;
        plan.b3d_gather.fin = dp.fin;
        plan.b3d_gather.cand_count = dp.cand_count;
    } else if (plan.sparse_b3d) {
        dp.b3d_rows = plan.b3d_rows;
        plan.b3d_sparse.fin = dp.fin;
        plan.b3d_sparse.cand_count = dp.cand_count;
    }
    if (plan.tower_begin >= 0) {
        TowerTilesParams& tt = plan.tower_tiles;
        tt.fin = dp.fin;
        tt.cand_count = dp.cand_count;
        tt.C = desc.num_classes;
        tt.topk = desc.pre_nms_topk;
        // the kernel's completion ticket starts at zero; each launch leaves it at zero
        cuda_check(cudaMemset(tt.ticket, 0, 4), "cudaMemset(tower tile ticket)");
        cuda_check(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    }
    if (plan.box2d_begin >= 0) {
        TowerTilesParams& tt = plan.box2d_tiles;
        tt.C = desc.num_classes;
        tt.thresh = dp.thresh;  // the decode's own threshold value: class_passes must agree bit for bit
        // the ticket and the tile distances start as each launch leaves them
        cuda_check(cudaMemset(tt.ticket, 0, 4), "cudaMemset(box2d tile ticket)");
        cuda_check(cudaMemset(tt.dist, kTowerTileFar & 0xFF, static_cast<size_t>(tt.cap) * 4), "cudaMemset(box2d tile distances)");
        cuda_check(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    }
    plan_steps(&plan);
}

void Engine::plan_steps(Plan* P) {
    fill_nms_params(&P->nms, desc, P->decode, P->B, P->nms_scratch);
    std::vector<Step>& S = P->steps;
    S.clear();
    auto add = [&](Step::Kind kind, int cat, int launches) -> Step& {  // the reference lives until the next add
        S.push_back(Step{kind, -1, cat, launches});
        return S.back();
    };
    add(Step::PREPROCESS, 0, kOneLaunch).bytes =
        static_cast<double>(P->B) * 3 * P->Hs * P->Ws + static_cast<double>(P->B) * P->Hp * P->Wp * 8;
    for (int oi = 0; oi < static_cast<int>(P->ops.size()); ++oi) {
        if (oi == P->box2d_begin) add(Step::BOX2D_TILES, 6, kOneLaunch + kOneLaunch);  // seeds, tile lists
        if (oi == P->tower_begin) add(Step::BOX3D_TILES, 6, kDecodeSelectLaunches + kOneLaunch);
        const Op& op = P->ops[oi];
        // special-purpose conv kernels are counted with the stems, so category 2 stays wgmma-only
        const int cat = (op.type == Op::STEM || op.type == Op::FRONT || op.type == Op::DW) ? 1 : op.type == Op::CONV ? 2
                        : op.type == Op::POOL ? 3 : op.type == Op::ESE ? 4 : 5;
        add(Step::OP, cat, op.type == Op::ESE ? kEseLaunches : op.type == Op::GN ? group_norm_launches(op.gn) : kOneLaunch).op = oi;
    }
    Step& det = add(Step::DETECT, 6, kDecodeFinalLaunches);
    det.select = P->tower_begin < 0;
    det.b3d = P->gather_b3d ? Step::kB3dGathered : P->sparse_b3d ? Step::kB3dSparse : 0;
    det.launches += (det.select ? kDecodeSelectLaunches : 0) + (P->gather_b3d ? kB3dGatherLaunches : P->sparse_b3d ? kOneLaunch : 0);
    for (int l = 0; l < P->num_levels; ++l)  // two dense passes over the fp32 logits + centerness
        det.bytes += 2.0 * P->B * P->lvl_h[l] * P->lvl_w[l] * (static_cast<double>(desc.num_classes) + 1) * 4;
    add(Step::NMS, 7, nms_launches(P->nms) + (P->bev == kBevPathOneCta     ? kOneLaunch
                                              : P->bev == kBevPathMultiCta ? image_bev_nms_launches(P->B) : 0))
        .bev = P->bev;
    // the blocked kernels run with one group per image of the call (num_groups = B), so their launches follow the plan
    if (P->agg)
        add(Step::AGGREGATE, 7, P->agg == kAggPathOneCta ? kSampleAggOneCtaLaunches : group_bev_nms_large_launches(P->B)).agg =
            P->agg;
}

void fill_decode_params(DecodeParams* dp, const dd3d_model_desc& desc, int B, int cls_pitch, int b3d_pitch,
                        const float* d_canon, int num_levels) {
    dp->num_levels = num_levels;
    dp->B = B;
    dp->C = desc.num_classes;
    dp->cls_pitch = cls_pitch;
    dp->b3d_pitch = b3d_pitch;
    dp->attr_off = desc.nuscenes_heads ? desc.num_classes : -1;
    dp->num_attr = kNumAttributes;
    dp->topk = desc.pre_nms_topk;
    dp->thresh = desc.pre_nms_thresh;
    dp->loc_offset_half = desc.feature_locations_offset_half;
    dp->canon = d_canon;
    dp->min_depth = desc.min_depth;
    dp->max_depth = desc.max_depth;
    dp->depth_factor = desc.scale_depth_by_focal_lengths_factor;
    dp->scale_depth_by_focal = desc.scale_depth_by_focal_lengths;
    dp->allocentric = desc.predict_allocentric_rot;
    dp->predict_distance = desc.predict_distance;
    dp->thresh_with_ctr = desc.thresh_with_ctr;
    dp->C3 = desc.class_agnostic_box3d ? 1 : desc.num_classes;
    dp->box3d_on = desc.box3d_on;
}

void fill_nms_params(NmsParams* np, const dd3d_model_desc& desc, const DecodeParams& dp, int B, void* scratch) {
    memset(np, 0, sizeof(*np));
    np->scratch = scratch;
    np->cand = dp.cand;
    np->cand_count = dp.cand_count;
    np->flags = dp.flags;
    np->B = B;
    np->num_levels = dp.num_levels;
    np->topk = desc.pre_nms_topk;
    np->out_cap = desc.out_cap;
    np->do_nms = desc.do_nms;
    np->post_topk = desc.post_nms_topk;
    np->do_postprocess = 1;
    np->nms_thresh = desc.nms_thresh;
    np->num_classes = desc.num_classes;
    np->class_parallel = nms_class_parallel(*np);
}

int Engine::bev_mode() const { return opt_bev_nms ? bev_nms_path(desc.do_nms, desc.post_nms_topk) : 0; }

void Engine::set_do_nms(int do_nms) {
    if (do_nms == desc.do_nms) return;
    if (bev_mode() && bev_nms_path(do_nms, desc.post_nms_topk) != bev_mode()) drop_plans();  // BEV kernel changes
    if (agg_mode() && sample_aggregate_path(do_nms, desc.post_nms_topk, desc.out_cap) != agg_mode()) drop_plans();
    desc.do_nms = do_nms;
    if (plan.valid) plan_steps(&plan);
    for (auto& kv : plan_cache) plan_steps(&kv.second);
}

void Engine::set_bev_nms(int enable, float thr) {
    if (enable && !desc.box3d_on) fail(DD3D_ERR_INVALID, "the BEV NMS needs the 3-D head (box3d_on)");
    if (!(thr == thr)) fail(DD3D_ERR_INVALID, "BEV NMS IoU threshold is NaN");
    const int after = enable ? bev_nms_path(desc.do_nms, desc.post_nms_topk) : 0;
    // the op list and the workspace change: plans are rebuilt at the next dd3d_plan (throws, changing nothing, while a
    // dd3d_submit_host is pending)
    if (after != bev_mode()) drop_plans();
    opt_bev_nms = enable ? 1 : 0;
    bev_nms_thresh = thr;
}

int Engine::agg_mode() const {
    return opt_sample_agg ? sample_aggregate_path(desc.do_nms, desc.post_nms_topk, desc.out_cap) : 0;
}

void Engine::set_sample_aggregate(int enable, float thr, int max_dets) {
    if (enable && !desc.box3d_on) fail(DD3D_ERR_INVALID, "the sample aggregation needs the 3-D head (box3d_on)");
    if (!(thr == thr)) fail(DD3D_ERR_INVALID, "sample aggregation IoU threshold is NaN");
    const int after = enable ? sample_aggregate_path(desc.do_nms, desc.post_nms_topk, desc.out_cap) : 0;
    if (after != agg_mode()) drop_plans();  // the step list and the workspace change (as set_bev_nms)
    opt_sample_agg = enable ? 1 : 0;
    agg_thresh = thr;
    agg_max_dets = max_dets;
}

void Engine::set_host_groups(int slot, const int32_t* h_group, int num_groups) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "set_host_groups before plan");
    if (slot < 0 || slot > 1) fail(DD3D_ERR_INVALID, "slot must be 0 or 1");
    if (num_groups < 1 || num_groups > plan.B) fail(DD3D_ERR_INVALID, "num_groups must be in 1..B");
    host_groups[slot].assign(h_group, h_group + plan.B);
    host_num_groups[slot] = num_groups;
}

void Engine::set_host_poses(int slot, const float* h_poses) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "set_host_poses before plan");
    if (slot < 0 || slot > 1) fail(DD3D_ERR_INVALID, "slot must be 0 or 1");
    host_poses[slot].assign(h_poses, h_poses + static_cast<size_t>(plan.B) * 7);
}

int Engine::launches_per_forward() const {
    int n = 0;
    for (const Step& s : plan.steps) n += s.launches;
    return n;
}

void Engine::forward_raw(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes, const float* h_K,
                         int min_size, int max_size, Det* d_out, int32_t* d_counts, float* h_K_out, int32_t* h_new_sizes,
                         cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    std::vector<int32_t> new_sizes(2 * P.B), sizes(4 * P.B);
    std::vector<float> K(9 * P.B);
    for (int b = 0; b < P.B; ++b) {
        const int h0 = h_raw_sizes[2 * b], w0 = h_raw_sizes[2 * b + 1];
        int nh, nw;
        resize_shortest_edge_shape(h0, w0, min_size, max_size, &nh, &nw);
        if (nh > P.Hs || nw > P.Ws)
            fail(DD3D_ERR_INVALID, "resized image " + std::to_string(nh) + "x" + std::to_string(nw) + " exceeds the plan");
        new_sizes[2 * b] = nh;
        new_sizes[2 * b + 1] = nw;
        // detections are mapped back to the ORIGINAL resolution: dataset dicts carry the file's height / width
        // (core.py:154-157 input_per_image.get("height"))
        sizes[4 * b] = nh; sizes[4 * b + 1] = nw; sizes[4 * b + 2] = h0; sizes[4 * b + 3] = w0;
        // apply_imresize_intrinsics (resize_transform.py:13-21): float32 rows scaled by float32(new / old)
        const float fx = static_cast<float>(static_cast<double>(nw) / w0), fy = static_cast<float>(static_cast<double>(nh) / h0);
        for (int c = 0; c < 3; ++c) {
            K[9 * b + c] = h_K[9 * b + c] * fx;
            K[9 * b + 3 + c] = h_K[9 * b + 3 + c] * fy;
            K[9 * b + 6 + c] = h_K[9 * b + 6 + c] * 1.0f;
        }
    }
    if (h_K_out) memcpy(h_K_out, K.data(), K.size() * 4);
    if (h_new_sizes) memcpy(h_new_sizes, new_sizes.data(), new_sizes.size() * 4);
    forward_resized(d_raw, raw_h, raw_w, h_raw_sizes, new_sizes.data(), nullptr, K.data(), sizes.data(), d_out, d_counts,
                    stream);
}

void Engine::forward_resized(const uint8_t* d_raw, int raw_h, int raw_w, const int32_t* h_raw_sizes,
                             const int32_t* h_new_sizes, const int32_t* h_flip, const float* h_K, const int32_t* h_sizes4,
                             Det* d_out, int32_t* d_counts, cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    for (int b = 0; b < P.B; ++b)
        if (h_new_sizes[2 * b] > P.Hs || h_new_sizes[2 * b + 1] > P.Ws) fail(DD3D_ERR_INVALID, "resized image exceeds the plan");
    cuda_check(cudaMemcpyAsync(P.d_K, h_K, static_cast<size_t>(P.B) * 36, cudaMemcpyHostToDevice, stream), "H2D K");
    cuda_check(cudaMemcpyAsync(P.d_sizes, h_sizes4, static_cast<size_t>(P.B) * 16, cudaMemcpyHostToDevice, stream),
               "H2D sizes");
    const RawArgs raw = {d_raw, raw_h, raw_w, h_raw_sizes, h_new_sizes, h_flip};
    forward(nullptr, DD3D_IMG_U8, P.d_K, P.d_sizes, d_out, d_counts, user_poses, device_agg_args(), stream, &raw);
}

void Engine::forward(const void* d_images, int img_dtype, const float* d_K, const int32_t* d_sizes, Det* d_out,
                     int32_t* d_counts, const float* d_poses, const AggArgs& agg, cudaStream_t stream, const RawArgs* raw) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    if (P.bev && d_poses == nullptr)
        fail(DD3D_ERR_STATE, "BEV NMS is on: the forward needs the poses (dd3d_set_poses / dd3d_set_host_poses)");
    if (P.agg) {
        if (d_poses == nullptr || agg.d_group == nullptr || agg.d_global == nullptr)
            fail(DD3D_ERR_STATE, "sample aggregation is on: the forward needs the poses, the group indices and the global rows "
                                 "(dd3d_set_poses / dd3d_set_groups / dd3d_set_global_out or their host forms)");
        if (agg.num_groups < 1 || agg.num_groups > P.B) fail(DD3D_ERR_INVALID, "num_groups must be in 1..B");
    }
    size_t ev_i = 0;
    auto mark = [&](int cat, int op) {  // opt_profile: CUDA events on the launch stream around every step
        if (!opt_profile) return;
        if (ev_i >= prof_ev.size()) {
            cudaEvent_t e;
            cuda_check(cudaEventCreate(&e), "cudaEventCreate");
            prof_ev.push_back(e);
            prof_cat.push_back(cat);
            prof_op.push_back(op);
        }
        prof_cat[ev_i] = cat;
        prof_op[ev_i] = op;
        cuda_check(cudaEventRecord(prof_ev[ev_i++], stream), "cudaEventRecord");
    };
    plan.ran = true;
    mark(-1, -1);
    std::optional<PdlScope> pdl_scope;  // opened behind the preprocess: every later launch follows one of our kernels (pdl.cuh)
    DecodeParams dp = P.decode;
    dp.K = d_K;
    for (const Step& s : P.steps) {
        switch (s.kind) {
            case Step::PREPROCESS:
                // sizes (h, w, out_h, out_w) -> the (h, w) pairs the preprocess kernel reads are its first two columns
                if (raw)
                    cuda_check(resize_tables.launch(raw->d_raw, raw->raw_h, raw->raw_w, raw->h_raw_sizes, raw->h_new_sizes,
                                                    raw->h_flip, P.input.ptr, P.B, P.Hp, P.Wp, desc.pixel_mean,
                                                    desc.pixel_std, stream, fp16),
                               "resize + preprocess");
                else
                    cuda_check(launch_preprocess(d_images, img_dtype == DD3D_IMG_U8, d_sizes, 4, P.input.ptr, P.B, P.Hs, P.Ws,
                                                 P.Hp, P.Wp, desc.pixel_mean, desc.pixel_std, stream, fp16),
                               "preprocess");
                pdl_scope.emplace();
                break;
            case Step::OP:
                launch_op(P.ops[s.op], stream);
                break;
            case Step::BOX2D_TILES:  // the pixels of the cls maps that pass the threshold, then the tiles
                cuda_check(launch_tower_mark(P.box2d_tiles, stream), "box2d tower seeds");
                cuda_check(launch_tower_tiles(P.box2d_tiles, stream), "box2d tower tile lists");
                break;
            case Step::BOX3D_TILES:  // the final candidates first, then the tiles they need
                cuda_check(launch_decode_select(dp, stream), "decode (threshold + top-k)");
                cuda_check(launch_tower_tiles(P.tower_tiles, stream), "box3d tower tile lists");
                break;
            case Step::DETECT:
                if (s.select) cuda_check(launch_decode_select(dp, stream), "decode (threshold + top-k)");
                if (s.b3d == Step::kB3dGathered)
                    cuda_check(launch_b3d_gather(P.b3d_gather, stream), "class-gathered box3d predictor");
                else if (s.b3d == Step::kB3dSparse)
                    cuda_check(launch_b3d_sparse(P.b3d_sparse, stream), "sparse box3d predictor");
                cuda_check(launch_decode_final(dp, stream), "decode (boxes)");
                break;
            case Step::NMS: {
                NmsParams np = P.nms;
                np.do_postprocess = s.bev ? 0 : opt_do_postprocess;  // with BEV NMS detector_postprocess follows it (core.py:137-160)
                np.sizes = d_sizes;
                np.out = d_out;
                np.out_count = d_counts;
                cuda_check(launch_nms(np, stream), "nms");
                if (s.bev == kBevPathOneCta)
                    cuda_check(launch_bev_nms(d_out, d_counts, d_K, d_poses, d_sizes, P.decode.flags, P.B, desc.out_cap,
                                              bev_nms_thresh, opt_do_postprocess, stream),
                               "bev nms");
                else if (s.bev == kBevPathMultiCta)
                    cuda_check(launch_image_bev_nms(d_out, d_counts, d_K, d_poses, opt_do_postprocess ? d_sizes : nullptr,
                                                    P.bev_scratch, P.decode.flags, P.B, desc.out_cap, bev_nms_thresh,
                                                    desc.num_classes, stream),
                               "bev nms (multi-CTA)");
                break;
            }
            case Step::AGGREGATE:  // in place on the detector_postprocess'ed detections, like the reference's order
                if (s.agg == kAggPathOneCta)
                    cuda_check(launch_sample_aggregate(d_out, d_counts, d_K, d_poses, agg.d_group, agg.num_groups,
                                                       agg.d_global, P.agg_scratch, P.decode.flags, P.B, desc.out_cap,
                                                       agg_thresh, agg_max_dets, stream),
                               "sample aggregation");
                else
                    cuda_check(launch_group_bev_nms_large(d_out, d_counts, d_K, 1, d_poses, 0, agg.d_group, P.B,
                                                          kGroupBevNmsLargeGroupImages, agg.d_global, P.agg_scratch,
                                                          P.decode.flags, P.B, desc.out_cap, agg_thresh, agg_max_dets,
                                                          stream),
                               "sample aggregation (blocked)");
                break;
        }
        mark(s.cat, s.op);
    }
    if (opt_profile) prof_used = ev_i;
}

// The forward above, recorded once.  Nothing in it synchronises, allocates or reads a device value back while profiling is
// off, and the device state that outlives a forward (tile-list tickets, box2d tile distances, the flags word) is reset by
// its own kernels, so a replay does what a new call would.  launch_pdl's attribute becomes a programmatic edge.
Engine::CapturedForward Engine::capture_forward(const void* d_images, int img_dtype, const float* d_K,
                                                const int32_t* d_sizes, Det* d_out, int32_t* d_counts,
                                                cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "graph capture before dd3d_plan");
    if (opt_profile) fail(DD3D_ERR_STATE, "graph capture with option \"profile\" on: its per-step events are for dd3d_forward");
    // the legacy default stream cannot be captured; a private one records the same launches
    struct OwnStream {
        cudaStream_t s = nullptr;
        ~OwnStream() { if (s) cudaStreamDestroy(s); }
    } own;
    if (stream == nullptr || stream == cudaStreamLegacy) {
        cuda_check(cudaStreamCreateWithFlags(&own.s, cudaStreamNonBlocking), "cudaStreamCreate");
        stream = own.s;
    }
    cuda_check(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCapture");
    int status = DD3D_OK;
    std::string msg;
    try {
        forward(d_images, img_dtype, d_K, d_sizes, d_out, d_counts, user_poses, device_agg_args(), stream);
    } catch (const EngineError& e) {
        status = e.status;
        msg = e.msg;
    }
    struct OwnGraph {
        cudaGraph_t g = nullptr;
        ~OwnGraph() { if (g) cudaGraphDestroy(g); }
    } graph;
    const cudaError_t end = cudaStreamEndCapture(stream, &graph.g);  // ends the capture whatever happened inside it
    if (status != DD3D_OK || end != cudaSuccess) {
        cudaGetLastError();  // a failed capture leaves no sticky error
        if (status == DD3D_OK) status = DD3D_ERR_CUDA, msg = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(end);
        fail(status, "graph capture: " + msg);
    }
    CapturedForward cf;
    size_t n = 0;
    cuda_check(cudaGraphGetNodes(graph.g, nullptr, &n), "cudaGraphGetNodes");
    std::vector<cudaGraphNode_t> nodes(n);
    cuda_check(cudaGraphGetNodes(graph.g, nodes.data(), &n), "cudaGraphGetNodes");
    for (cudaGraphNode_t node : nodes) {
        cudaGraphNodeType t;
        cuda_check(cudaGraphNodeGetType(node, &t), "cudaGraphNodeGetType");
        cf.kernel_nodes += t == cudaGraphNodeTypeKernel;
    }
    size_t ne = 0;
    cuda_check(cudaGraphGetEdges_v2(graph.g, nullptr, nullptr, nullptr, &ne), "cudaGraphGetEdges");
    std::vector<cudaGraphNode_t> from(ne), to(ne);
    std::vector<cudaGraphEdgeData> edges(ne);
    cuda_check(cudaGraphGetEdges_v2(graph.g, from.data(), to.data(), edges.data(), &ne), "cudaGraphGetEdges");
    for (const cudaGraphEdgeData& e : edges) cf.programmatic_edges += e.type == cudaGraphDependencyTypeProgrammatic;
    cuda_check(cudaGraphInstantiate(&cf.exec, graph.g, 0), "cudaGraphInstantiate");
    return cf;
}

void Engine::launch_op(const Op& op, cudaStream_t stream) {
    switch (op.type) {
        case Op::CONV:
            cuda_check(launch_conv(op.conv, num_sms, stream), "conv");
            break;
        case Op::STEM:
            cuda_check(launch_stem_s2_mma(op.in.ptr, op.stem->d_w, op.stem->d_sb, op.out.ptr, op.out.pitch, plan.B, op.in.H,
                                          op.in.W, num_sms, stream, fp16, op.stem->relu ? 1 : 0),
                       "stem conv");
            break;
        case Op::POOL:
            cuda_check(launch_maxpool(op.in.ptr, op.out.ptr, plan.B, op.in.H, op.in.W, op.in.C, op.in.pitch, op.out.H,
                                      op.out.W, op.out.pitch, op.ksize, num_sms, stream, fp16),
                       "maxpool");
            break;
        case Op::ESE:
            if (op.f2 == nullptr) {  // behind a GroupNorm: pool pass over the normalised map -> fc -> scale
                cuda_check(launch_ese(op.in.ptr, op.in.pitch, op.ese->d_w, op.ese->d_b,
                                      op.has_identity ? op.identity.ptr : nullptr, op.has_identity ? op.identity.pitch : 0,
                                      op.out.ptr, op.out.pitch, op.f0, op.f1, plan.B, op.in.H * op.in.W, op.in.C, num_sms,
                                      stream, fp16),
                           "eSE");
                break;
            }
            cuda_check(launch_ese_fused(op.in.ptr, op.in.pitch, op.f2, op.ksize, op.ese->d_w, op.ese->d_b,
                                        op.has_identity ? op.identity.ptr : nullptr,
                                        op.has_identity ? op.identity.pitch : 0, op.out.ptr, op.out.pitch, op.f0, op.f1,
                                        plan.B, op.in.H * op.in.W, op.in.C, num_sms, stream, fp16),
                       "eSE");
            break;
        case Op::RELU:
            cuda_check(launch_relu(op.in.ptr, op.out.ptr, static_cast<size_t>(plan.B) * op.in.H * op.in.W * op.in.C,
                                   num_sms, stream),
                       "relu");
            break;
        case Op::FRONT:
            cuda_check(launch_dla_front(op.in.ptr, op.front->d_w0, op.front->d_w1, op.front->d_w2, op.front->d_sb0,
                                        op.front->d_sb1, op.front->d_sb2, op.out.ptr, op.out.pitch, op.identity.ptr,
                                        op.identity.pitch, plan.B, op.in.H, op.in.W, num_sms, stream, fp16),
                       "dla front");
            break;
        case Op::DW:
            cuda_check(launch_dwconv3x3(op.in.ptr, plan.B, op.in.H, op.in.W, op.in.C, op.in.pitch, op.dw->d_w, op.stride,
                                        op.out.ptr, op.out.pitch, stream, fp16),
                       "depthwise conv");
            break;
        case Op::GN:
            cuda_check(launch_group_norm(op.gn, stream), "group norm");
            break;
    }
}

// Algorithmic FLOPs per plan op.  The convs of the sparse towers count the in-map pixels of the tiles the last forward ran,
// read back from the device (call after that forward has completed).
std::vector<double> Engine::op_flops() {
    std::vector<double> f(plan.ops.size());
    for (size_t i = 0; i < f.size(); ++i) f[i] = plan.ops[i].flops;
    auto listed = [&](int begin, const TowerTilesParams& tt, const char* what) {
        if (begin < 0) return;
        const int d = tt.depth;
        std::vector<long long> px(d, 0);
        if (plan.ran && prof_used >= 2)  // the callers have synchronised the last profiled forward
            cuda_check(cudaMemcpy(px.data(), tt.pixels, d * sizeof(long long), cudaMemcpyDeviceToHost), what);
        for (int j = 0; j < d; ++j) {
            const ConvParams& c = plan.ops[begin + j].conv;
            double dense_px = 0.0;
            for (int s = 0; s < c.nseg; ++s) dense_px += static_cast<double>(c.B) * c.seg[s].H * c.seg[s].W;
            f[begin + j] *= static_cast<double>(px[j]) / dense_px;
        }
    };
    listed(plan.box2d_begin, plan.box2d_tiles, "D2H box2d tile pixels");
    listed(plan.tower_begin, plan.tower_tiles, "D2H tower tile pixels");
    return f;
}

// per-step device time of the last profiled forward (Plan::steps in order), with the plan op each step ran (or -1)
int Engine::get_op_times(float* ms, int32_t* cats, double* flops, int32_t* ops, int max_ops) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "no plan");
    if (prof_used < 2) return 0;
    cuda_check(cudaEventSynchronize(prof_ev[prof_used - 1]), "cudaEventSynchronize");
    const std::vector<double> f = op_flops();
    int n = 0;
    for (size_t i = 1; i < prof_used && n < max_ops; ++i, ++n) {
        cuda_check(cudaEventElapsedTime(&ms[n], prof_ev[i - 1], prof_ev[i]), "cudaEventElapsedTime");
        cats[n] = prof_cat[i];
        flops[n] = (prof_op[i] >= 0 && prof_op[i] < static_cast<int>(f.size())) ? f[prof_op[i]] : 0.0;
        if (ops) ops[n] = prof_op[i];
    }
    return n;
}

void Engine::get_profile(double* ms, double* flops, double* bytes, int32_t* launches) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "no plan");
    for (int c = 0; c < 8; ++c) ms[c] = flops[c] = bytes[c] = 0.0, launches[c] = 0;
    if (prof_used >= 2) {
        cuda_check(cudaEventSynchronize(prof_ev[prof_used - 1]), "cudaEventSynchronize");
        for (size_t i = 1; i < prof_used; ++i) {
            float t = 0.f;
            cuda_check(cudaEventElapsedTime(&t, prof_ev[i - 1], prof_ev[i]), "cudaEventElapsedTime");
            ms[prof_cat[i]] += t;
        }
    }
    const std::vector<double> f = op_flops();
    for (const Step& s : plan.steps) {
        launches[s.cat] += s.launches;
        flops[s.cat] += s.op >= 0 ? f[s.op] : 0.0;
        bytes[s.cat] += s.op >= 0 ? plan.ops[s.op].bytes : s.bytes;
    }
}

void Engine::forward_host(const void* h_images, int img_dtype, const float* h_K, const int32_t* h_sizes, Det* h_out,
                          int32_t* h_counts, cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    check_host_agg(0);
    const size_t img_bytes = static_cast<size_t>(P.B) * 3 * P.Hs * P.Ws * (img_dtype == DD3D_IMG_U8 ? 1 : 4);
    cuda_check(cudaMemcpyAsync(P.d_images, h_images, img_bytes, cudaMemcpyHostToDevice, stream), "H2D images");
    cuda_check(cudaMemcpyAsync(P.d_K, h_K, static_cast<size_t>(P.B) * 36, cudaMemcpyHostToDevice, stream), "H2D K");
    cuda_check(cudaMemcpyAsync(P.d_sizes, h_sizes, static_cast<size_t>(P.B) * 16, cudaMemcpyHostToDevice, stream),
               "H2D sizes");
    if (P.bev || P.agg) {
        if (host_poses[0].size() != static_cast<size_t>(P.B) * 7)
            fail(DD3D_ERR_STATE, std::string(P.bev ? "BEV NMS" : "sample aggregation") + " is on: dd3d_set_host_poses(0, ...) first");
        cuda_check(cudaMemcpyAsync(P.d_poses, host_poses[0].data(), host_poses[0].size() * 4, cudaMemcpyHostToDevice, stream),
                   "H2D poses");
    }
    if (P.agg)
        cuda_check(cudaMemcpyAsync(P.d_group, host_groups[0].data(), host_groups[0].size() * 4, cudaMemcpyHostToDevice, stream),
                   "H2D groups");
    forward(P.d_images, img_dtype, P.d_K, P.d_sizes, P.d_out, P.d_counts, P.d_poses, {P.d_group, host_num_groups[0], P.d_global},
            stream);
    cuda_check(cudaMemcpyAsync(h_out, P.d_out, static_cast<size_t>(P.B) * desc.out_cap * sizeof(Det),
                               cudaMemcpyDeviceToHost, stream),
               "D2H dets");
    if (P.agg)
        cuda_check(cudaMemcpyAsync(host_global[0], P.d_global, static_cast<size_t>(P.B) * desc.out_cap * 40,
                                   cudaMemcpyDeviceToHost, stream),
                   "D2H global rows");
    cuda_check(cudaMemcpyAsync(h_counts, P.d_counts, static_cast<size_t>(P.B) * 4, cudaMemcpyDeviceToHost, stream),
               "D2H counts");
    cuda_check(cudaStreamSynchronize(stream), "sync");
}

// Double-buffered host path.  Slot s owns one set of device staging buffers; its inputs travel on a private copy stream,
// so the H2D of the next batch overlaps the kernels of the current one (the copy engines and the SMs are independent),
// while kernels and the (small) D2H stay ordered on the caller's stream.
void Engine::submit_host(int slot, const void* h_images, int img_dtype, const float* h_K, const int32_t* h_sizes, Det* h_out,
                         int32_t* h_counts, cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "submit before plan");
    if (slot < 0 || slot > 1) fail(DD3D_ERR_INVALID, "slot must be 0 or 1");
    if (slot_busy[slot]) fail(DD3D_ERR_STATE, "slot resubmitted before dd3d_wait_host");
    Plan& P = plan;
    const size_t img_cap = static_cast<size_t>(P.B) * 3 * P.Hs * P.Ws * 4;
    const size_t out_bytes = static_cast<size_t>(P.B) * desc.out_cap * sizeof(Det);
    if (copy_stream == nullptr) {
        cuda_check(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking), "cudaStreamCreate");
        for (int i = 0; i < 2; ++i) {
            cuda_check(cudaEventCreateWithFlags(&h2d_done[i], cudaEventDisableTiming), "cudaEventCreate");
            cuda_check(cudaEventCreateWithFlags(&all_done[i], cudaEventDisableTiming), "cudaEventCreate");
        }
    }
    if (slot == 1 && P.slot1 == nullptr) {
        const size_t a = 1024;
        auto up = [&](size_t n) { return (n + a - 1) / a * a; };
        const size_t glob_bytes = static_cast<size_t>(P.B) * desc.out_cap * 40;
        const size_t total = up(img_cap) + up(P.B * 36) + up(P.B * 16) + up(out_bytes) + up(P.B * 4) +
                             (P.bev || P.agg ? up(P.B * 28) : 0) + (P.agg ? up(P.B * 4) + up(glob_bytes) : 0);
        cuda_check(cudaMalloc(&P.slot1, total), "cudaMalloc(slot 1 staging)");
        uint8_t* q = static_cast<uint8_t*>(P.slot1);
        P.s1_images = q; q += up(img_cap);
        P.s1_K = reinterpret_cast<float*>(q); q += up(P.B * 36);
        P.s1_sizes = reinterpret_cast<int32_t*>(q); q += up(P.B * 16);
        P.s1_out = reinterpret_cast<Det*>(q); q += up(out_bytes);
        P.s1_counts = reinterpret_cast<int32_t*>(q); q += up(P.B * 4);
        if (P.bev || P.agg) {
            P.s1_poses = reinterpret_cast<float*>(q); q += up(P.B * 28);
        }
        if (P.agg) {
            P.s1_group = reinterpret_cast<int32_t*>(q); q += up(P.B * 4);
            P.s1_global = reinterpret_cast<float*>(q);
        }
    }
    void* d_img = slot ? P.s1_images : P.d_images;
    float* d_K = slot ? P.s1_K : P.d_K;
    int32_t* d_sz = slot ? P.s1_sizes : P.d_sizes;
    Det* d_out = slot ? P.s1_out : P.d_out;
    int32_t* d_cnt = slot ? P.s1_counts : P.d_counts;
    float* d_poses = slot ? P.s1_poses : P.d_poses;
    int32_t* d_group = slot ? P.s1_group : P.d_group;
    float* d_global = slot ? P.s1_global : P.d_global;
    if ((P.bev || P.agg) && host_poses[slot].size() != static_cast<size_t>(P.B) * 7)
        fail(DD3D_ERR_STATE, std::string(P.bev ? "BEV NMS" : "sample aggregation") + " is on: dd3d_set_host_poses(slot, ...) first");
    check_host_agg(slot);
    const size_t img_bytes = static_cast<size_t>(P.B) * 3 * P.Hs * P.Ws * (img_dtype == DD3D_IMG_U8 ? 1 : 4);
    cuda_check(cudaMemcpyAsync(d_img, h_images, img_bytes, cudaMemcpyHostToDevice, copy_stream), "H2D images");
    cuda_check(cudaMemcpyAsync(d_K, h_K, static_cast<size_t>(P.B) * 36, cudaMemcpyHostToDevice, copy_stream), "H2D K");
    cuda_check(cudaMemcpyAsync(d_sz, h_sizes, static_cast<size_t>(P.B) * 16, cudaMemcpyHostToDevice, copy_stream), "H2D sizes");
    if (P.bev || P.agg)  // pageable source: staged before the call returns, so the next dd3d_set_host_poses may overwrite it
        cuda_check(cudaMemcpyAsync(d_poses, host_poses[slot].data(), host_poses[slot].size() * 4, cudaMemcpyHostToDevice,
                                   copy_stream),
                   "H2D poses");
    if (P.agg)  // pageable as well
        cuda_check(cudaMemcpyAsync(d_group, host_groups[slot].data(), host_groups[slot].size() * 4, cudaMemcpyHostToDevice,
                                   copy_stream),
                   "H2D groups");
    cuda_check(cudaEventRecord(h2d_done[slot], copy_stream), "cudaEventRecord");
    cuda_check(cudaStreamWaitEvent(stream, h2d_done[slot], 0), "cudaStreamWaitEvent");
    forward(d_img, img_dtype, d_K, d_sz, d_out, d_cnt, d_poses, {d_group, host_num_groups[slot], d_global}, stream);
    cuda_check(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, stream), "D2H dets");
    if (P.agg)
        cuda_check(cudaMemcpyAsync(host_global[slot], d_global, static_cast<size_t>(P.B) * desc.out_cap * 40,
                                   cudaMemcpyDeviceToHost, stream),
                   "D2H global rows");
    cuda_check(cudaMemcpyAsync(h_counts, d_cnt, static_cast<size_t>(P.B) * 4, cudaMemcpyDeviceToHost, stream), "D2H counts");
    cuda_check(cudaEventRecord(all_done[slot], stream), "cudaEventRecord");
    slot_busy[slot] = true;
}

// the host group indices and the global-row buffer of a host slot, before anything is enqueued
void Engine::check_host_agg(int slot) const {
    if (!plan.agg) return;
    if (host_groups[slot].size() != static_cast<size_t>(plan.B))
        fail(DD3D_ERR_STATE, "sample aggregation is on: dd3d_set_host_groups(" + std::to_string(slot) + ", ...) first");
    if (host_global[slot] == nullptr)
        fail(DD3D_ERR_STATE, "sample aggregation is on: dd3d_set_host_global_out(" + std::to_string(slot) + ", ...) first");
}

void Engine::wait_host(int slot) {
    if (slot < 0 || slot > 1) fail(DD3D_ERR_INVALID, "slot must be 0 or 1");
    if (!slot_busy[slot]) fail(DD3D_ERR_STATE, "dd3d_wait_host without dd3d_submit_host");
    cuda_check(cudaEventSynchronize(all_done[slot]), "cudaEventSynchronize");
    slot_busy[slot] = false;
}

}  // namespace dd3d
