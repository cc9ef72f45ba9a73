// conv_igemm_kernel instantiations for block_n in {80, 96, 112, 128}, and the pair-tile halo kernel (dense and work-list mode; see conv_igemm_kernel.cuh).
#include "conv_igemm_kernel.cuh"

namespace dd3d {
DD3D_CONV_KERNEL_GROUP(conv_kernel_n80_128, 80, 96, 112, 128)
ConvKernel conv_kernel_pair(bool fp16, bool list) {
    if (list) return fp16 ? conv_igemm_kernel<true, true, 128, true, true> : conv_igemm_kernel<true, false, 128, true, true>;
    return fp16 ? conv_igemm_kernel<true, true, 128, true> : conv_igemm_kernel<true, false, 128, true>;
}
}  // namespace dd3d
