// DD3D inference engine: weight folding/packing, static graph for DLA-34 / every VoVNetV2-eSE variant + FPN + FCOS2D/3D
// heads, workspace planning and the forward launch sequence.  Reference structure being reproduced:
//   DD3D.forward                      tridet/modeling/dd3d/core.py:64-164
//   DLA-34                            tridet/modeling/feature_extractor/dla.py:24-62,146-247,250-361
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
#include <stdexcept>

namespace dd3d {

namespace {

inline int round_up(int v, int a) { return (v + a - 1) / a * a; }
inline size_t round_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }

[[noreturn]] void fail(int status, const std::string& msg) { throw EngineError(status, msg); }

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) fail(DD3D_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

}  // namespace

// ================================================================================================ Engine basics

Engine::Engine(const dd3d_model_desc& d) : desc(d) {
    if (d.arch != DD3D_ARCH_DLA34 && vovnet_spec(d.arch) == nullptr) fail(DD3D_ERR_INVALID, "unknown arch");
    if (d.num_classes < 1 || d.num_classes > DD3D_MAX_CLASSES) fail(DD3D_ERR_INVALID, "num_classes out of range");
    if (d.pre_nms_topk < 1 || d.pre_nms_topk * kLevels > 8192) fail(DD3D_ERR_INVALID, "pre_nms_topk out of range");
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
    if (const char* e = getenv("DD3D_DLA_FRONT")) opt_dla_front = atoi(e) ? 1 : 0;  // A/B runs of bench.py; default 1
    if (const char* e = getenv("DD3D_SPARSE_BOX3D")) opt_sparse_box3d = std::max(0, std::min(2, atoi(e)));
    if (const char* e = getenv("DD3D_SPARSE_TOWER")) opt_sparse_tower = std::max(0, std::min(2, atoi(e)));
    if (const char* e = getenv("DD3D_STEM_MMA")) opt_stem_mma = atoi(e) ? 1 : 0;
    if (const char* e = getenv("DD3D_ESE_POOL")) opt_ese_pool = atoi(e) ? 1 : 0;
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
    L.cout_pad = round_up(cout, 16);
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

void Engine::set_layout(const dd3d_layout_desc& l) {
    if (finalized) fail(DD3D_ERR_STATE, "dd3d_set_layout after finalize");
    for (int n : {l.fcos2d_norm, l.fcos3d_norm, l.fpn_norm})
        if (n < DD3D_NORM_BN_PER_LEVEL || n > DD3D_NORM_NONE) fail(DD3D_ERR_INVALID, "unknown dd3d_norm value");
    for (int d : {l.num_cls_convs, l.num_box2d_convs, l.num_box3d_convs})
        if (d < 0 || d > 16) fail(DD3D_ERR_INVALID, "tower depth outside 0..16");
    if (l.fpn_fuse_avg != 0 && l.fpn_fuse_avg != 1) fail(DD3D_ERR_INVALID, "fpn_fuse_avg must be 0 or 1");
    layout = l;
}

// GroupNorm(32, C) affine of `<prefix>.weight` / `<prefix>.bias`, uploaded as fp32 vectors (cached like the epilogues)
const Epilogue& Engine::gn_affine(const std::string& prefix) {
    const std::string key = "gn|" + prefix;
    auto it = epis.find(key);
    if (it != epis.end()) return it->second;
    const HostTensor& g = weight(prefix + ".weight");
    const HostTensor& b = weight(prefix + ".bias");
    if (g.data.size() != static_cast<size_t>(kGnChannels) || b.data.size() != static_cast<size_t>(kGnChannels))
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
    const int n_pad = round_up(static_cast<int>(scale.size()), 16);
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
        {
            int hs[kMaxSeg], ws[kMaxSeg];
            for (int s = 0; s < p.nseg; ++s) {
                hs[s] = segs[s].in.H / stride;
                ws[s] = segs[s].in.W / stride;
            }
            p.halo = conv_prefer_halo(L.taps, stride, L.block_n, p.nseg, hs, ws) ? conv_halo_mode() : 0;
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
            if (p.halo) {
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
                if (!make_act_map(&g.out_map, sp.out.ptr, B, Ho, Wo, sp.out.C, sp.out.pitch, g.th, g.tw, E->fp16))
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
        const bool pair = conv_select_pair(&p, L.cout_pad, E->num_sms);
        bool n_split = false;
        if (!p.taps_n && !pair && conv_n_split_enabled()) {
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
            op.flops += 2.0 * B * p.seg[s].H * p.seg[s].W * static_cast<double>(L.cout) * L.cin * L.taps;
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
        for (size_t s = 0; s < x.size(); ++s) {
            if (x[s].C != kGnChannels) fail(DD3D_ERR_INVALID, "GroupNorm needs 256 channels");
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
            const double px = static_cast<double>(B) * x[s].H * x[s].W * kGnChannels * 2;
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
        P->ops.push_back(op);
    }

    // ---- DLA-34 -------------------------------------------------------------------------------------------
    // BasicBlock (dla.py:24-62): conv1 -> BN -> ReLU -> conv2 -> BN -> (+residual) -> ReLU
    void dla_block(const std::string& p, View x, int stride, View residual, View dst) {
        const int Ho = x.H / stride, Wo = x.W / stride;
        View t = alloc(Ho, Wo, dst.C);
        conv1(p + ".conv1", p + ".conv1.norm", false, x, t, 3, stride, true);
        conv1(p + ".conv2", p + ".conv2.norm", false, t, dst, 3, 1, true, &residual);
    }
    // Tree with levels == 1 (dla.py:170-247): `rc` is the Root's concat buffer, laid out [x2 | x1 | children...]
    // with the children already in place; `bottom` is the (pooled) input the optional `project` acts on.
    void dla_tree1(const std::string& p, View x, int in_ch, int out_ch, int stride, View rc, View bottom, View dst) {
        View residual = bottom;
        if (in_ch != out_ch) {
            residual = alloc(bottom.H, bottom.W, out_ch);
            conv1(p + ".project", p + ".project.norm", false, bottom, residual, 1, 1, false);
        }
        View x1 = slice(rc, out_ch, out_ch);
        View x2 = slice(rc, 0, out_ch);
        dla_block(p + ".tree1", x, stride, residual, x1);
        dla_block(p + ".tree2", x1, 1, x1, x2);
        conv1(p + ".root.conv", p + ".root.conv.norm", false, rc, dst, 1, 1, true);  // Root: cat -> 1x1 -> BN -> ReLU
    }
    // Tree with levels == 2 and level_root (level3 / level4, dla.py:309-314)
    View dla_tree2(const std::string& p, View x, int in_ch, int out_ch) {
        const int Ho = x.H / 2, Wo = x.W / 2;
        View rc2 = alloc(Ho, Wo, 3 * out_ch + in_ch);  // [x2 | x1 | bottom | tree1-out]   (dla.py:235-245)
        View bottom = slice(rc2, 2 * out_ch, in_ch);
        View t1_out = slice(rc2, 2 * out_ch + in_ch, out_ch);
        maxpool(x, bottom, 2);  // outer and inner Tree pool the same tensor (dla.py:235) -> computed once
        View rc1 = alloc(Ho, Wo, 2 * out_ch);
        dla_tree1(p + ".tree1", x, in_ch, out_ch, 2, rc1, bottom, t1_out);
        View out = alloc(Ho, Wo, out_ch);
        dla_tree1(p + ".tree2", t1_out, out_ch, out_ch, 1, rc2, t1_out, out);
        return out;
    }

    void build_dla34(View input, std::vector<View>* feats) {
        const std::string p = "backbone.bottom_up";
        const int H = input.H, W = input.W;
        // both forms of the front end are packed at finalize (host weights are dropped afterwards), so that the
        // "dla_front" option can be flipped on a finalized engine
        const FrontLayer& F = E->front_layer(p);
        E->stem_layer(p + ".base_layer", p + ".base_layer.norm", 7, 1);
        E->conv_layer(p + ".level0.0", {p + ".level0.0"}, 16, 3);
        E->bn_epilogue(p + ".level0.0|" + p + ".level0.0.norm", p + ".level0.0.norm", "", 16);
        E->conv_layer(p + ".level1.0", {p + ".level1.0"}, 16, 3);
        E->bn_epilogue(p + ".level1.0|" + p + ".level1.0.norm", p + ".level1.0.norm", "", 32);
        View a2, bottom;
        if (E->opt_dla_front && H % 4 == 0 && W % 4 == 0) {
            // base_layer -> level0 -> level1 -> 2x2 max-pool in one kernel (dla_front.cu); the two full-resolution
            // 16-channel maps never reach HBM
            a2 = alloc(H / 2, W / 2, 32);
            bottom = alloc(H / 4, W / 4, 32);
            front(F, input, a2, bottom);
        } else {
            View a0 = alloc(H, W, 16);
            stem(p + ".base_layer", p + ".base_layer.norm", input, a0, 7, 1);
            View a1 = alloc(H, W, 16);
            conv1(p + ".level0.0", p + ".level0.0.norm", false, a0, a1, 3, 1, true);
            a2 = alloc(H / 2, W / 2, 32);
            conv1(p + ".level1.0", p + ".level1.0.norm", false, a1, a2, 3, 2, true);
            bottom = alloc(H / 4, W / 4, 32);
            maxpool(a2, bottom, 2);
        }
        // level2: Tree(levels=1, 32->64, stride 2)
        View rc = alloc(H / 4, W / 4, 128);
        View l2 = alloc(H / 4, W / 4, 64);
        dla_tree1(p + ".level2", a2, 32, 64, 2, rc, bottom, l2);
        View l3 = dla_tree2(p + ".level3", l2, 64, 128);
        View l4 = dla_tree2(p + ".level4", l3, 128, 256);
        // level5: Tree(levels=1, 256->512, stride 2, level_root) -> root input [x2 | x1 | bottom]
        View rc5 = alloc(H / 32, W / 32, 1280);
        View bottom5 = slice(rc5, 1024, 256);
        maxpool(l4, bottom5, 2);
        View l5 = alloc(H / 32, W / 32, 512);
        dla_tree1(p + ".level5", l4, 256, 512, 2, rc5, bottom5, l5);
        feats->assign({l3, l4, l5});
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

    void stem(const std::string& wname, const std::string& bn, View in4, View out, int ksize, int stride) {
        const StemLayer& S = E->stem_layer(wname, bn, ksize, stride);
        touch(out);
        ++op_idx;
        if (dry) return;
        Op op;
        op.type = Op::STEM;
        op.in = in4;
        op.out = out;
        op.ksize = ksize;
        op.stride = stride;
        op.stem = &S;
        op.outs[0] = out;
        op.nouts = 1;
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
            conv1(n + "/conv", n + "/norm", false, in, out, 3, stride, true);
            return;
        }
        View t = alloc(out.H, out.W, in.C);
        dwconv(n + "/dw_conv3x3", in, t, stride);
        conv1(n + "/pw_conv1x1", n + "/pw_norm", false, t, out, 1, 1, true);
    }

    void build_vovnet(const VovSpec& S, View input, std::vector<View>* feats) {
        const std::string p = "backbone.bottom_up";
        const int H = input.H, W = input.W;
        const int* stage_ch = S.stage_ch;
        const int* out_ch = S.out_ch;
        const int* blocks = S.blocks;
        const int nl = S.layers;
        View s1 = alloc(H / 2, W / 2, S.stem[0]);
        stem(p + ".stem.stem_1/conv", p + ".stem.stem_1/norm", input, s1, 3, 2);
        View s2 = alloc(H / 2, W / 2, S.stem[1]);
        vov_conv3x3(p + ".stem.stem_2", s1, s2, 1, S.dw);
        int h = H / 4, w = W / 4;
        int in_ch = S.stem[2];
        View cat = alloc(h, w, in_ch + nl * stage_ch[0]);
        vov_conv3x3(p + ".stem.stem_3", s2, slice(cat, 0, in_ch), 2, S.dw);
        View stage_out;
        View pooled_cat;  // next stage's concat buffer when its pooled slice was produced by the previous stage's eSE pass
        for (int si = 0; si < 4; ++si) {
            const int sc = stage_ch[si], oc = out_ch[si];
            if (si > 0) {
                const int hp = (h - 3 + 1) / 2 + 1, wp = (w - 3 + 1) / 2 + 1;  // 3x3 / s2, ceil_mode (vovnet.py:249)
                if (pooled_cat.ptr != nullptr || pooled_cat.buf >= 0) {
                    cat = pooled_cat;  // the previous stage's last eSE pass already wrote the pooled map (ese_scale_pool_kernel)
                } else {
                    cat = alloc(hp, wp, in_ch + nl * sc);
                    maxpool(stage_out, slice(cat, 0, in_ch), 3);
                }
                h = hp;
                w = wp;
            }
            View pooled_next;  // stays empty unless this stage's last module fuses the next stage's pool
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
                    conv1(rn + "/conv", rn + "/norm", false, x, r, 1, 1, true);
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
                conv1(q + ".concat." + name + "_concat/conv", q + ".concat." + name + "_concat/norm", false, cat, xt, 1,
                      1, true);
                // eSE (always applied, vovnet.py:216,233) then identity add for non-first blocks (:235-236)
                View dst;
                View next_cat;
                const bool last = (b == blocks[si] - 1);
                View pooled;
                if (last) {
                    dst = alloc(h, w, oc);
                    if (si < 3 && E->opt_ese_pool && h >= 3 && w >= 3) {
                        // the eSE scale pass of a stage's last module also writes the next stage's 3x3 / s2 pooled input
                        pooled_next = alloc((h - 3 + 1) / 2 + 1, (w - 3 + 1) / 2 + 1, oc + nl * stage_ch[si + 1]);
                        pooled = slice(pooled_next, 0, oc);
                    }
                } else {
                    next_cat = alloc(h, w, oc + nl * sc);
                    dst = slice(next_cat, 0, oc);
                }
                ese(q + ".ese.fc", xt, b > 0 ? &x : nullptr, dst, pooled.buf >= 0 ? &pooled : nullptr);
                if (last) {
                    stage_out = dst;
                } else {
                    cat = next_cat;
                }
                in_ch = oc;
            }
            pooled_cat = pooled_next;
            feats->push_back(stage_out);
        }
    }

    void ese(const std::string& fc, View xt, const View* identity, View dst, const View* pooled = nullptr) {
        const EseLayer& L = E->ese_layer(fc, xt.C);
        // The concat conv (the op just emitted) writes per-tile channel sums from its epilogue: [B][T][C], T = 4 * tiles
        const int T = 4 * conv_tiles_per_image(xt.H, xt.W);
        float* tile_partial = alloc_f32(static_cast<size_t>(B) * T * xt.C);
        float* sums = alloc_f32(static_cast<size_t>(B) * xt.C);
        float* gate = alloc_f32(static_cast<size_t>(B) * xt.C);
        touch(xt);
        if (identity) touch(*identity);
        touch(dst);
        if (pooled) touch(*pooled);
        ++op_idx;
        if (dry) return;
        Op& cv = P->ops.back();
        if (cv.type != Op::CONV || cv.conv.nseg != 1 || cv.conv.halo || cv.conv.out_mode != 0 ||
            4 * cv.conv.seg[0].tiles_x * cv.conv.seg[0].tiles_y != T)
            fail(DD3D_ERR_STATE, "internal: eSE must follow its concat conv");
        cv.conv.seg[0].pool_partial = tile_partial;
        cv.conv.seg[0].pool_pitch = xt.C;
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
        if (pooled) {  // outs[1]: the 3x3 / s2 ceil-mode max-pool of dst, written by the same pass
            op.outs[1] = *pooled;
            op.nouts = 2;
        }
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
        auto conv_norm = [&](const std::string& name, View in, View out, int ksize, const View* res) {
            conv1(name, bn ? name + ".norm" : "", norm == DD3D_NORM_NONE, in, out, ksize, 1, false, res, res != nullptr);
        };
        std::vector<View> res(n);
        View prev;
        for (int i = n - 1; i >= 0; --i) {
            const std::string st = std::to_string(first_stage + i);
            const std::string lname = p + ".fpn_lateral" + st, oname = p + ".fpn_output" + st;
            const View& c = feats[i];
            View lat = alloc(c.H, c.W, 256);
            if (i == n - 1 || gn || avg) {
                conv_norm(lname, c, lat, 1, nullptr);
                const bool add = i != n - 1;
                if (gn || add) group_norm({lat}, gn ? &E->gn_affine(lname + ".norm") : nullptr, false, add ? &prev : nullptr, add && avg);
            } else {
                // lateral + nearest-2x(prev): the un-smoothed `prev` is what propagates downwards
                conv_norm(lname, c, lat, 1, &prev);
            }
            prev = lat;
            res[i] = alloc(c.H, c.W, 256);
            persist(res[i]);
            conv_norm(oname, lat, res[i], 3, nullptr);
            if (gn) group_norm({res[i]}, &E->gn_affine(oname + ".norm"), false, nullptr, false);
        }
        *outs = res;
        const View& p5 = res[n - 1];
        View p6 = alloc(p5.H / 2, p5.W / 2, 256);
        persist(p6);
        conv1(p + ".top_block.p6", "", true, p5, p6, 3, 2, false);
        outs->push_back(p6);
        if (E->desc.arch == DD3D_ARCH_DLA34) {
            View r6 = alloc(p6.H, p6.W, 256);
            relu(p6, r6);
            View p7 = alloc(p6.H / 2, p6.W / 2, 256);
            persist(p7);
            conv1(p + ".top_block.p7", "", true, r6, p7, 3, 2, false);
            outs->push_back(p7);
        }
    }

    // ---- heads ------------------------------------------------------------------------------------------------
    // `depth` x (3x3 conv -> norm -> ReLU) over every level in one launch per layer (fcos2d.py:55-91, fcos3d.py:81-112).
    // norm: per-level BN (ModuleListDial, folded per segment), shared BN (one folded epilogue), none (conv bias), or GN
    // (identity epilogue, then one GN op over the levels).  Depth 0: the FPN outputs themselves.
    void tower(const std::string& tp, int depth, int norm, const std::vector<View>& feats, std::vector<View>* out) {
        std::vector<View> cur = feats;
        std::vector<View> buf[2];
        for (int k = 0; k < std::min(depth, 2); ++k)
            for (auto& f : feats) buf[k].push_back(alloc(f.H, f.W, 256));
        for (int i = 0; i < depth; ++i) {
            const std::string wn = tp + "." + std::to_string(i);
            const ConvLayer& L = E->conv_layer(wn, {wn}, 256, 3);
            std::vector<SegSpec> segs(feats.size());
            for (size_t l = 0; l < feats.size(); ++l) {
                segs[l].in = cur[l];
                segs[l].out = buf[i & 1][l];
                if (norm == DD3D_NORM_BN_PER_LEVEL) {
                    const std::string bn = wn + ".norm." + std::to_string(l);  // ModuleListDial: level l -> norm l
                    segs[l].epi = &E->bn_epilogue(wn + "|" + bn, bn, "", 256);
                } else if (norm == DD3D_NORM_BN_SHARED) {
                    segs[l].epi = &E->bn_epilogue(wn + "|" + wn + ".norm", wn + ".norm", "", 256);
                } else {  // none: conv bias; GN: raw conv output, normalised by the GN op below
                    segs[l].epi = &E->bn_epilogue(wn + "|", "", norm == DD3D_NORM_NONE ? wn + ".bias" : "", 256);
                }
            }
            const bool gn = norm == DD3D_NORM_GN;
            conv(L, 1, !gn, segs, false);
            if (gn) group_norm(buf[i & 1], &E->gn_affine(wn + ".norm"), true, nullptr, false);
            cur = buf[i & 1];
        }
        *out = cur;
    }

    // Tile lists of the sparse box3d tower (TowerTilesParams): the tiling conv() gives the tower layers, and the staging, list
    // and count areas in the persistent region.  false: the shapes exceed the list entry fields, the tower stays dense.
    bool tower_tile_lists(const std::vector<View>& feats, int depth) {
        TowerTilesParams& tt = P->tower_tiles;
        memset(&tt, 0, sizeof(tt));
        const int L = static_cast<int>(feats.size());
        int hs[kMaxSeg], ws[kMaxSeg];
        for (int l = 0; l < L; ++l) {
            hs[l] = feats[l].H;
            ws[l] = feats[l].W;
        }
        const bool halo = conv_prefer_halo(9, 1, 256, L, hs, ws);
        for (int l = 0; l < L; ++l) {
            TowerTilesLevel& v = tt.lvl[l];
            v.H = hs[l];
            v.W = ws[l];
            if (halo) {
                v.th = kHaloTh;
                v.tw = kHaloTw;
            } else {
                choose_tile(v.H, v.W, &v.th, &v.tw);
            }
            v.tiles_x = (v.W + v.tw - 1) / v.tw;
            v.tiles_y = (v.H + v.th - 1) / v.th;
            const int T = v.tiles_x * v.tiles_y;
            v.stage_begin = tt.cap;
            tt.cap += B * (T + (T & 1));
            tt.max_tiles = std::max(tt.max_tiles, T);
        }
        if (B > kTileListMaxImages || tt.max_tiles >= kTileListMaxTiles || tower_tiles_smem_bytes(tt.max_tiles) > 48 * 1024)
            return false;
        // the work-list mode is built for the pair tile, which every filled 256-channel halo layer selects (conv() below)
        ConvParams cp;
        memset(&cp, 0, sizeof(cp));
        cp.nseg = L;
        cp.B = B;
        cp.halo = halo ? conv_halo_mode() : 0;
        for (int l = 0; l < L; ++l) {
            cp.seg[l].H = hs[l];
            cp.seg[l].W = ws[l];
            cp.seg[l].th = tt.lvl[l].th;
            cp.seg[l].tw = tt.lvl[l].tw;
        }
        if (!conv_select_pair(&cp, 256, E->num_sms)) return false;
        tt.B = B;
        tt.depth = depth;
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

    void build_heads(const std::vector<View>& feats) {
        const int C = E->desc.num_classes;
        const int L = static_cast<int>(feats.size());
        const bool nusc = E->desc.nuscenes_heads != 0;
        // head switches no shipped experiment changes (dd3d_model_desc): class-agnostic 3-D channels, per-level predictors,
        // no Scale / Offset layers, no 3-D head at all
        const bool use_scale2 = E->desc.fcos2d_use_scale != 0, use_scale3 = E->desc.fcos3d_use_scale != 0;
        const bool per_level = E->desc.per_level_predictors != 0, box3d_on = E->desc.box3d_on != 0;
        const int C3 = E->desc.class_agnostic_box3d ? 1 : C;
        const int cls_pitch = round_up(C + (nusc ? kNumAttributes + 1 : 0), 16), b3d_pitch = round_up(11 * C3, 16);
        // sparse box3d predictor: forced (1), off (0) or auto (2, default).  The dense launch costs time in proportion to the
        // head pixels, the gathered one a near-constant latency-bound K loop, so large heads go sparse.  The rule looks at
        // the head pixels of ONE image, not of the batch, so that an image gives bit-identical detections whatever batch it
        // rides in (the two predictors differ in fp32 summation order): 900x1600 V2-99 = 127 875 pixels -> sparse at every
        // batch size, 384x1280 DLA-34 = 10 230 -> dense.
        size_t head_px = 0;
        for (int l = 0; l < L; ++l) head_px += static_cast<size_t>(feats[l].H) * feats[l].W;
        const bool sparse3 = box3d_on && b3d_pitch <= kB3dSparseMaxN &&
                             (E->opt_sparse_box3d == 1 || (E->opt_sparse_box3d == 2 && head_px >= 50000));
        P->sparse_b3d = sparse3;
        P->b3d_rows = sparse3 ? alloc_f32(static_cast<size_t>(B) * kLevels * E->desc.pre_nms_topk * b3d_pitch) : nullptr;
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
                                                names, 256, 3);
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
        // [box2d_reg (4) | centerness (1)] on the box2d tower: relu(scale_l * (conv + b)) / conv + b (fcos2d.py:143-152)
        tower("fcos2d_head.box2d_tower", E->layout.num_box2d_convs, E->layout.fcos2d_norm, feats, &box_t);
        {
            const ConvLayer& Lb = E->conv_layer("fcos2d_head.box2d_reg+centerness",
                                                {"fcos2d_head.box2d_reg", "fcos2d_head.centerness"}, 256, 3);
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
                                  tower_tile_lists(feats, d3);
        P->tower_begin = sparse_tower ? static_cast<int>(P->ops.size()) : -1;
        tower("fcos3d_head.box3d_tower", d3, E->layout.fcos3d_norm, feats, &b3d_t);
        if (sparse_tower && !dry) {
            const TowerTilesParams& tt = P->tower_tiles;
            for (int j = 0; j < d3; ++j) {
                Op& op = P->ops[P->tower_begin + j];
                ConvParams& c = op.conv;
                if (op.type != Op::CONV || c.nseg != L || !c.pair) fail(DD3D_ERR_STATE, "internal: sparse box3d tower layout");
                for (int l = 0; l < L; ++l)
                    if (c.seg[l].th != tt.lvl[l].th || c.seg[l].tw != tt.lvl[l].tw)
                        fail(DD3D_ERR_STATE, "internal: sparse box3d tower tiling");
                c.tile_list = tt.list + static_cast<size_t>(j) * tt.cap;
                c.tile_count = tt.count + j;
            }
        }
        // [quat 4C | ctr 2C | depth C | size 3C | conf C] on the box3d tower with the per-level Scale/Offset folded
        // (fcos3d.py:166-180).  PER_LEVEL_PREDICTORS False (shipped): predictor index 0 for every level, one launch over the
        // five levels; True: level l uses predictor l, one launch per level.
        {
            auto layer_for = [&](int li) -> const ConvLayer& {
                const std::string i = std::to_string(li);
                return E->conv_layer("fcos3d_head.box3d_all." + i,
                                     {"fcos3d_head.box3d_quat." + i, "fcos3d_head.box3d_ctr." + i, "fcos3d_head.box3d_depth." + i,
                                      "fcos3d_head.box3d_size." + i, "fcos3d_head.box3d_conf." + i},
                                     256, 3);
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
            if (sparse3) {
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
                    if (Lw.cout_pad != b3d_pitch || Lw.cin != 256) fail(DD3D_ERR_INVALID, "box3d predictor shape");
                }
                ++op_idx;
                sp.rows = P->b3d_rows;
                sp.B = B;
                sp.C = C;
                sp.topk = E->desc.pre_nms_topk;
                sp.n_pad = b3d_pitch;
                sp.out_pitch = b3d_pitch;
                sp.fp16 = E->fp16;
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

const StemLayer& Engine::stem_layer(const std::string& wname, const std::string& bn, int ksize, int stride) {
    auto it = stems.find(wname);
    if (it != stems.end()) return it->second;
    const HostTensor& w = weight(wname + ".weight");
    if (w.shape.size() != 4 || w.shape[1] != 3 || w.shape[2] != ksize || w.shape[0] % 16)
        fail(DD3D_ERR_INVALID, "bad stem weight: " + wname);
    StemLayer S;
    S.ksize = ksize;
    S.stride = stride;
    S.cout = static_cast<int>(w.shape[0]);
    // tensor-core stem layout: bf16 [cout][kpad], k = (ky*ksize + kx)*4 + c, zero padded (4th channel and K tail)
    const int kpad = stem_tc_kpad(ksize);
    std::vector<uint16_t> packed(static_cast<size_t>(S.cout) * kpad, 0);
    for (int co = 0; co < S.cout; ++co)
        for (int c = 0; c < 3; ++c)
            for (int t = 0; t < ksize * ksize; ++t)
                packed[static_cast<size_t>(co) * kpad + t * 4 + c] =
                    host_f32_to_act(w.data[(static_cast<size_t>(co) * 3 + c) * ksize * ksize + t], fp16);
    S.d_w = static_cast<__nv_bfloat16*>(dev_alloc(packed.size() * 2));
    cuda_check(cudaMemcpy(S.d_w, packed.data(), packed.size() * 2, cudaMemcpyHostToDevice), "upload stem weights");
    S.epi = bn_epilogue(wname + "|" + bn, bn, "", S.cout);
    if (ksize == 3 && stride == 2 && S.cout == 64) {
        std::vector<uint16_t> pm(64 * 3 * 4 * 4, 0);
        for (int co = 0; co < 64; ++co)
            for (int c = 0; c < 3; ++c)
                for (int ky = 0; ky < 3; ++ky)
                    for (int kx = 0; kx < 3; ++kx)
                        pm[((co * 3 + ky) * 4 + kx) * 4 + c] = host_f32_to_act(w.data[((co * 3 + c) * 3 + ky) * 3 + kx], fp16);
        S.d_w_mma = static_cast<__nv_bfloat16*>(dev_alloc(pm.size() * 2));
        cuda_check(cudaMemcpy(S.d_w_mma, pm.data(), pm.size() * 2, cudaMemcpyHostToDevice), "upload stem weights (mma)");
        std::vector<float> sc, bi;
        bn_fold(bn, "", 64, &sc, &bi);
        sc.insert(sc.end(), bi.begin(), bi.end());
        S.d_sb_mma = upload_f32(sc);
    }
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
    auto sb = [&](const std::string& bn, int cout) {
        std::vector<float> s, b;
        bn_fold(bn, "", cout, &s, &b);
        s.insert(s.end(), b.begin(), b.end());
        return upload_f32(s);
    };
    FrontLayer F;
    F.d_w0 = up16(p0);
    F.d_w1 = up16(p1);
    F.d_w2 = up16(p2);
    F.d_sb0 = sb(prefix + ".base_layer.norm", 16);
    F.d_sb1 = sb(prefix + ".level0.0.norm", 16);
    F.d_sb2 = sb(prefix + ".level1.0.norm", 32);
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

int Engine::size_divisibility() const { return desc.arch == DD3D_ARCH_DLA34 ? 128 : 64; }

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
        if (desc.arch == DD3D_ARCH_DLA34) {
            bld.build_dla34(input, &feats);
            bld.build_fpn(feats, 3, &fpn);
        } else {
            bld.build_vovnet(*vovnet_spec(desc.arch), input, &feats);
            bld.build_fpn(feats, 2, &fpn);
        }
        if (static_cast<int>(fpn.size()) != kLevels) fail(DD3D_ERR_STATE, "internal: expected 5 FPN levels");
        for (int l = 0; l < kLevels; ++l) P->fpn[l] = fpn[l];
        bld.build_heads(fpn);
        // detection scratch + staging for the host-facing path
        P->detect_scratch = bld.alloc_bytes(decode_scratch_bytes(B, desc.pre_nms_topk));
        P->nms_scratch = bld.alloc_bytes(nms_scratch_bytes(B, desc.pre_nms_topk, desc.num_classes));
        P->d_K = static_cast<float*>(bld.alloc_bytes(static_cast<size_t>(B) * 9 * 4));
        P->d_sizes = static_cast<int32_t*>(bld.alloc_bytes(static_cast<size_t>(B) * 4 * 4));
        P->d_out = static_cast<Det*>(bld.alloc_bytes(static_cast<size_t>(B) * desc.out_cap * sizeof(Det)));
        P->d_counts = static_cast<int32_t*>(bld.alloc_bytes(static_cast<size_t>(B) * 4));
        P->d_images = bld.alloc_bytes(static_cast<size_t>(B) * 3 * Hs * Ws * 4);
        P->d_canon = nullptr;
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
    build(&tmp, 1, size_divisibility(), size_divisibility(), nullptr, true);
    std::vector<float> canon(desc.canonical_box3d_sizes, desc.canonical_box3d_sizes + DD3D_MAX_CLASSES * 3);
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
    release_plan();
    for (auto& kv : plan_cache) free_plan(&kv.second);
    plan_cache.clear();
}

void Engine::make_plan(int B, int Hs, int Ws, void* workspace, size_t bytes) {
    if (!finalized) fail(DD3D_ERR_STATE, "plan before finalize");
    if (B < 1 || Hs < 1 || Ws < 1) fail(DD3D_ERR_INVALID, "bad plan shape");
    if (slot_busy[0] || slot_busy[1]) fail(DD3D_ERR_STATE, "plan change with a pending dd3d_submit_host");
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
    static const int strides_dla[5] = {8, 16, 32, 64, 128};
    static const int strides_vov[5] = {4, 8, 16, 32, 64};
    const int* strides = desc.arch == DD3D_ARCH_DLA34 ? strides_dla : strides_vov;
    for (int l = 0; l < kLevels; ++l) {
        dp.lvl[l].cls = plan.cls_map[l];
        dp.lvl[l].box = plan.box_map[l];
        dp.lvl[l].b3d = plan.b3d_map[l];
        dp.lvl[l].H = plan.lvl_h[l];
        dp.lvl[l].W = plan.lvl_w[l];
        dp.lvl[l].stride = strides[l];
    }
    fill_decode_params(&dp, desc, B, plan.cls_pitch, plan.b3d_pitch, d_canon);
    decode_bind_scratch(&dp, plan.detect_scratch);
    decode_finalize_params(&dp);
    if (plan.sparse_b3d) {
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
    fill_nms_params(&plan.nms, desc, dp, B);
    plan.nms.scratch = plan.nms_scratch;
}

void fill_decode_params(DecodeParams* dp, const dd3d_model_desc& desc, int B, int cls_pitch, int b3d_pitch,
                        const float* d_canon) {
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

void fill_nms_params(NmsParams* np, const dd3d_model_desc& desc, const DecodeParams& dp, int B) {
    memset(np, 0, sizeof(*np));
    np->cand = dp.cand;
    np->cand_count = dp.cand_count;
    np->flags = dp.flags;
    np->B = B;
    np->topk = desc.pre_nms_topk;
    np->out_cap = desc.out_cap;
    np->do_nms = desc.do_nms;
    np->post_topk = desc.post_nms_topk;
    np->do_postprocess = 1;
    np->nms_thresh = desc.nms_thresh;
    np->num_classes = desc.num_classes;
}

int Engine::launches_per_forward() const {
    int n = 1 /*preprocess*/ + 6 /*decode: clear, 2 dense passes, 2 selects, final*/ + (plan.sparse_b3d ? 1 : 0) +
            (plan.tower_begin >= 0 ? 1 : 0) /*tower tile lists*/ + ((desc.do_nms && desc.nms_thresh > 0.f) ? 4 : 1) /*nms: sort, IoU bit matrix, scan, finish*/;
    for (const Op& op : plan.ops) n += (op.type == Op::ESE) ? 3 : (op.type == Op::GN && op.gn.gamma != nullptr) ? 2 : 1;
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
    raw_pending = true;
    raw_args = {d_raw, raw_h, raw_w, h_raw_sizes, h_new_sizes, h_flip};
    forward(nullptr, DD3D_IMG_U8, P.d_K, P.d_sizes, d_out, d_counts, stream);
}

void Engine::forward(const void* d_images, int img_dtype, const float* d_K, const int32_t* d_sizes, Det* d_out,
                     int32_t* d_counts, cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    const bool raw = raw_pending;
    raw_pending = false;
    size_t ev_i = 0;
    auto mark = [&](int cat, int op = -1) {  // opt_profile: CUDA events on the launch stream around every op
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
    mark(-1);
    // sizes (h, w, out_h, out_w) -> the (h, w) pairs the preprocess kernel reads are its first two columns
    if (raw) {
        cuda_check(resize_tables.launch(raw_args.d_raw, raw_args.raw_h, raw_args.raw_w, raw_args.h_raw_sizes,
                                        raw_args.h_new_sizes, raw_args.h_flip, P.input.ptr, P.B, P.Hp, P.Wp, desc.pixel_mean, desc.pixel_std,
                                        stream, fp16),
                   "resize + preprocess");
    } else {
        cuda_check(launch_preprocess(d_images, img_dtype == DD3D_IMG_U8, d_sizes, 4, P.input.ptr, P.B, P.Hs, P.Ws, P.Hp,
                                     P.Wp, desc.pixel_mean, desc.pixel_std, stream, fp16),
                   "preprocess");
    }
    mark(0);
    // from here on every launch follows one of our kernels: the small kernels may use programmatic dependent launch (pdl.cuh)
    PdlScope pdl_scope;
    DecodeParams dp = P.decode;
    dp.K = d_K;
    for (const Op& op : P.ops) {
        const int oi = static_cast<int>(&op - P.ops.data());
        if (oi == P.tower_begin) {  // sparse box3d tower: the final candidates first, then the tiles they need
            cuda_check(launch_decode_select(dp, stream), "decode (threshold + top-k)");
            cuda_check(launch_tower_tiles(P.tower_tiles, stream), "box3d tower tile lists");
            mark(6);
        }
        switch (op.type) {
            case Op::CONV:
                cuda_check(launch_conv(op.conv, num_sms, stream), "conv");
                break;
            case Op::STEM:
                if (op.stem->d_w_mma != nullptr && opt_stem_mma) {
                    cuda_check(launch_stem_s2_mma(op.in.ptr, op.stem->d_w_mma, op.stem->d_sb_mma, op.out.ptr, op.out.pitch, P.B,
                                                  op.in.H, op.in.W, num_sms, stream, fp16),
                               "stem conv (mma)");
                    break;
                }
                cuda_check(launch_stem_tc(op.in.ptr, op.stem->d_w, op.stem->epi.d_scale, op.stem->epi.d_bias, op.out.ptr,
                                          P.B, op.in.H, op.in.W, op.ksize, op.stride, op.stem->cout, op.out.pitch, num_sms,
                                          stream, fp16),
                           "stem conv");
                break;
            case Op::POOL:
                cuda_check(launch_maxpool(op.in.ptr, op.out.ptr, P.B, op.in.H, op.in.W, op.in.C, op.in.pitch, op.out.H,
                                          op.out.W, op.out.pitch, op.ksize, num_sms, stream, fp16),
                           "maxpool");
                break;
            case Op::ESE:
                cuda_check(launch_ese_fused(op.in.ptr, op.in.pitch, op.f2, op.ksize, op.ese->d_w, op.ese->d_b,
                                            op.has_identity ? op.identity.ptr : nullptr,
                                            op.has_identity ? op.identity.pitch : 0, op.out.ptr, op.out.pitch, op.f0, op.f1,
                                            P.B, op.in.H * op.in.W, op.in.C, num_sms, stream, fp16,
                                            op.nouts == 2 ? op.outs[1].ptr : nullptr, op.nouts == 2 ? op.outs[1].pitch : 0,
                                            op.in.H, op.in.W),
                           "eSE");
                break;
            case Op::RELU:
                cuda_check(launch_relu(op.in.ptr, op.out.ptr, static_cast<size_t>(P.B) * op.in.H * op.in.W * op.in.C,
                                       num_sms, stream),
                           "relu");
                break;
            case Op::FRONT:
                cuda_check(launch_dla_front(op.in.ptr, op.front->d_w0, op.front->d_w1, op.front->d_w2, op.front->d_sb0,
                                            op.front->d_sb1, op.front->d_sb2, op.out.ptr, op.out.pitch, op.identity.ptr,
                                            op.identity.pitch, P.B, op.in.H, op.in.W, num_sms, stream, fp16),
                           "dla front");
                break;
            case Op::DW:
                cuda_check(launch_dwconv3x3(op.in.ptr, P.B, op.in.H, op.in.W, op.in.C, op.in.pitch, op.dw->d_w, op.stride,
                                            op.out.ptr, op.out.pitch, stream, fp16),
                           "depthwise conv");
                break;
            case Op::GN:
                cuda_check(launch_group_norm(op.gn, stream), "group norm");
                break;
        }
        mark((op.type == Op::STEM || op.type == Op::FRONT || op.type == Op::DW) ? 1 : op.type == Op::CONV ? 2 : op.type == Op::POOL ? 3 : op.type == Op::ESE ? 4 : 5,
             oi);
    }
    if (P.sparse_b3d) {
        if (P.tower_begin < 0) cuda_check(launch_decode_select(dp, stream), "decode (threshold + top-k)");
        cuda_check(launch_b3d_sparse(P.b3d_sparse, stream), "sparse box3d predictor");
        cuda_check(launch_decode_final(dp, stream), "decode (boxes)");
    } else {
        cuda_check(launch_decode(dp, stream), "decode");
    }
    mark(6);
    NmsParams np = P.nms;
    np.do_postprocess = opt_do_postprocess;
    np.do_nms = desc.do_nms;
    np.sizes = d_sizes;
    np.out = d_out;
    np.out_count = d_counts;
    cuda_check(launch_nms(np, stream), "nms");
    mark(7);
    if (opt_profile) prof_used = ev_i;
}

// Algorithmic FLOPs per plan op.  The sparse box3d tower convs count the in-map pixels of the tiles the last forward ran,
// read back from the device (call after that forward has completed).
std::vector<double> Engine::op_flops() {
    std::vector<double> f(plan.ops.size());
    for (size_t i = 0; i < f.size(); ++i) f[i] = plan.ops[i].flops;
    if (plan.tower_begin >= 0) {
        const int d = plan.tower_tiles.depth;
        std::vector<long long> px(d, 0);
        if (plan.ran && prof_used >= 2)  // the callers have synchronised the last profiled forward
            cuda_check(cudaMemcpy(px.data(), plan.tower_tiles.pixels, d * sizeof(long long), cudaMemcpyDeviceToHost),
                       "D2H tower tile pixels");
        for (int j = 0; j < d; ++j) {
            const ConvParams& c = plan.ops[plan.tower_begin + j].conv;
            double dense_px = 0.0;
            for (int s = 0; s < c.nseg; ++s) dense_px += static_cast<double>(c.B) * c.seg[s].H * c.seg[s].W;
            f[plan.tower_begin + j] *= static_cast<double>(px[j]) / dense_px;
        }
    }
    return f;
}

// per-op device time of the last profiled forward: entry 0 = preprocess, then plan.ops in order (with the sparse box3d
// tower, the threshold / top-k and the tile lists before the tower convs), then decode, nms
int Engine::get_op_times(float* ms, int32_t* cats, double* flops, int max_ops) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "no plan");
    if (prof_used < 2) return 0;
    cuda_check(cudaEventSynchronize(prof_ev[prof_used - 1]), "cudaEventSynchronize");
    const std::vector<double> f = op_flops();
    int n = 0;
    for (size_t i = 1; i < prof_used && n < max_ops; ++i, ++n) {
        cuda_check(cudaEventElapsedTime(&ms[n], prof_ev[i - 1], prof_ev[i]), "cudaEventElapsedTime");
        cats[n] = prof_cat[i];
        flops[n] = (prof_op[i] >= 0 && prof_op[i] < static_cast<int>(f.size())) ? f[prof_op[i]] : 0.0;
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
    const Plan& P = plan;
    const double C = desc.num_classes;
    const std::vector<double> f = op_flops();
    launches[0] = 1;
    bytes[0] = static_cast<double>(P.B) * 3 * P.Hs * P.Ws + static_cast<double>(P.B) * P.Hp * P.Wp * 8;
    for (const Op& op : P.ops) {
        const double in_px = static_cast<double>(P.B) * op.in.H * op.in.W, out_px = static_cast<double>(P.B) * op.out.H * op.out.W;
        switch (op.type) {
            case Op::STEM:
                launches[1] += 1;
                flops[1] += 2.0 * out_px * op.stem->cout * 3 * op.ksize * op.ksize;
                bytes[1] += in_px * 8 + out_px * op.stem->cout * 2;
                break;
            case Op::CONV:
                launches[2] += 1;
                flops[2] += f[&op - P.ops.data()];
                break;
            case Op::POOL:
                launches[3] += 1;
                bytes[3] += (in_px + out_px) * op.in.C * 2;
                break;
            case Op::ESE:
                launches[4] += 3;
                bytes[4] += in_px * op.in.C * 2 * (op.has_identity ? 3 : 2);  // pooling is fused into the concat conv
                if (op.nouts == 2) bytes[4] += static_cast<double>(P.B) * op.outs[1].H * op.outs[1].W * op.in.C * 2;
                break;
            case Op::RELU:
                launches[5] += 1;
                bytes[5] += in_px * op.in.C * 4;
                break;
            case Op::GN:  // statistics + apply (one launch without the affine)
                launches[5] += op.gn.gamma != nullptr ? 2 : 1;
                bytes[5] += op.bytes;
                break;
            case Op::FRONT:
            case Op::DW:  // special-purpose conv kernels are counted with the stems, so category 2 stays wgmma-only
                launches[1] += 1;
                flops[1] += op.flops;
                bytes[1] += op.bytes;
                break;
        }
    }
    launches[6] = 6 + (P.sparse_b3d ? 1 : 0) + (P.tower_begin >= 0 ? 1 : 0);
    launches[7] = (desc.do_nms && desc.nms_thresh > 0.f) ? 4 : 1;
    for (int l = 0; l < kLevels; ++l)  // two dense passes over the fp32 logits + centerness
        bytes[6] += 2.0 * P.B * P.lvl_h[l] * P.lvl_w[l] * (C + 1) * 4;
}

void Engine::forward_host(const void* h_images, int img_dtype, const float* h_K, const int32_t* h_sizes, Det* h_out,
                          int32_t* h_counts, cudaStream_t stream) {
    if (!plan.valid) fail(DD3D_ERR_STATE, "forward before plan");
    const Plan& P = plan;
    const size_t img_bytes = static_cast<size_t>(P.B) * 3 * P.Hs * P.Ws * (img_dtype == DD3D_IMG_U8 ? 1 : 4);
    cuda_check(cudaMemcpyAsync(P.d_images, h_images, img_bytes, cudaMemcpyHostToDevice, stream), "H2D images");
    cuda_check(cudaMemcpyAsync(P.d_K, h_K, static_cast<size_t>(P.B) * 36, cudaMemcpyHostToDevice, stream), "H2D K");
    cuda_check(cudaMemcpyAsync(P.d_sizes, h_sizes, static_cast<size_t>(P.B) * 16, cudaMemcpyHostToDevice, stream),
               "H2D sizes");
    forward(P.d_images, img_dtype, P.d_K, P.d_sizes, P.d_out, P.d_counts, stream);
    cuda_check(cudaMemcpyAsync(h_out, P.d_out, static_cast<size_t>(P.B) * desc.out_cap * sizeof(Det),
                               cudaMemcpyDeviceToHost, stream),
               "D2H dets");
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
        const size_t total = up(img_cap) + up(P.B * 36) + up(P.B * 16) + up(out_bytes) + up(P.B * 4);
        cuda_check(cudaMalloc(&P.slot1, total), "cudaMalloc(slot 1 staging)");
        uint8_t* q = static_cast<uint8_t*>(P.slot1);
        P.s1_images = q; q += up(img_cap);
        P.s1_K = reinterpret_cast<float*>(q); q += up(P.B * 36);
        P.s1_sizes = reinterpret_cast<int32_t*>(q); q += up(P.B * 16);
        P.s1_out = reinterpret_cast<Det*>(q); q += up(out_bytes);
        P.s1_counts = reinterpret_cast<int32_t*>(q);
    }
    void* d_img = slot ? P.s1_images : P.d_images;
    float* d_K = slot ? P.s1_K : P.d_K;
    int32_t* d_sz = slot ? P.s1_sizes : P.d_sizes;
    Det* d_out = slot ? P.s1_out : P.d_out;
    int32_t* d_cnt = slot ? P.s1_counts : P.d_counts;
    const size_t img_bytes = static_cast<size_t>(P.B) * 3 * P.Hs * P.Ws * (img_dtype == DD3D_IMG_U8 ? 1 : 4);
    cuda_check(cudaMemcpyAsync(d_img, h_images, img_bytes, cudaMemcpyHostToDevice, copy_stream), "H2D images");
    cuda_check(cudaMemcpyAsync(d_K, h_K, static_cast<size_t>(P.B) * 36, cudaMemcpyHostToDevice, copy_stream), "H2D K");
    cuda_check(cudaMemcpyAsync(d_sz, h_sizes, static_cast<size_t>(P.B) * 16, cudaMemcpyHostToDevice, copy_stream), "H2D sizes");
    cuda_check(cudaEventRecord(h2d_done[slot], copy_stream), "cudaEventRecord");
    cuda_check(cudaStreamWaitEvent(stream, h2d_done[slot], 0), "cudaStreamWaitEvent");
    forward(d_img, img_dtype, d_K, d_sz, d_out, d_cnt, stream);
    cuda_check(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, stream), "D2H dets");
    cuda_check(cudaMemcpyAsync(h_counts, d_cnt, static_cast<size_t>(P.B) * 4, cudaMemcpyDeviceToHost, stream), "D2H counts");
    cuda_check(cudaEventRecord(all_done[slot], stream), "cudaEventRecord");
    slot_busy[slot] = true;
}

void Engine::wait_host(int slot) {
    if (slot < 0 || slot > 1) fail(DD3D_ERR_INVALID, "slot must be 0 or 1");
    if (!slot_busy[slot]) fail(DD3D_ERR_STATE, "dd3d_wait_host without dd3d_submit_host");
    cuda_check(cudaEventSynchronize(all_done[slot]), "cudaEventSynchronize");
    slot_busy[slot] = false;
}

}  // namespace dd3d
