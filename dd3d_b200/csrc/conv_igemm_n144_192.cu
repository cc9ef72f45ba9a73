// conv_igemm_kernel instantiations for block_n in {144, 160, 176, 192} (see conv_igemm_kernel.cuh).
#include "conv_igemm_kernel.cuh"

namespace dd3d {
DD3D_CONV_KERNEL_GROUP(conv_kernel_n144_192, 144, 160, 176, 192)
}  // namespace dd3d
