// Programmatic dependent launch for the small kernels of the forward (pools, eSE, decode, NMS, sparse predictor): every one of
// them used to be a full serialisation point of the stream (drain, then launch latency: ~4 us x 51 kernels per V2-99 forward,
// x 14 per DLA-34 forward).  DD3D_PDL_PROLOGUE() is the FIRST statement of such a kernel: it waits until every earlier kernel of
// the stream has completed and its memory is visible (so nothing the kernel reads or overwrites can be in flight), then lets
// the next kernel's CTAs be scheduled as this grid's CTAs retire.
// RULE: the launch attribute is only used where the preceding operation of the stream is one of OUR KERNELS.  griddepcontrol.wait
// waits for the primary GRID; a kernel launched programmatically right behind an asynchronous memcpy (the caller's H2D of the
// images / sizes in front of the preprocess kernel) has no grid to wait for and can overtake the copy -- seen once as a
// preprocess output that depended on timing (tests/test_determinism_gpu.py).  So launch_pdl() sets the attribute only inside a
// PdlScope, which Engine::forward opens AFTER its first (normally launched) kernel; the operator-level entry points, which
// run behind arbitrary caller work, never open one.  DD3D_NO_PDL=1 turns the attribute off everywhere (the prologue is then a
// no-op): tests/test_determinism_gpu.py compares both modes bit for bit across processes.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <utility>

#define DD3D_PDL_PROLOGUE()                                   \
    do {                                                      \
        asm volatile("griddepcontrol.wait;" ::: "memory");    \
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); \
    } while (0)

namespace dd3d {

// Kernels a launch wrapper without a count of its own enqueues (launch_conv, the preprocess / stem / pool / relu / depthwise
// wrappers, the resize, the sparse predictor, the tile lists, the one-CTA BEV NMS).  Multi-kernel wrappers name their count
// next to their declaration (kDecodeSelectLaunches, kEseLaunches, kB3dGatherLaunches, nms_launches, ...).
constexpr int kOneLaunch = 1;

inline bool pdl_enabled() {
    static int on = -1;
    if (on < 0) {
        const char* e = getenv("DD3D_NO_PDL");
        on = (e && atoi(e)) ? 0 : 1;
    }
    return on != 0;
}

inline thread_local int g_pdl_scope_depth = 0;
struct PdlScope {
    PdlScope() { ++g_pdl_scope_depth; }
    ~PdlScope() { --g_pdl_scope_depth; }
    PdlScope(const PdlScope&) = delete;
    PdlScope& operator=(const PdlScope&) = delete;
};

template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (pdl_enabled() && g_pdl_scope_depth > 0) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace dd3d
