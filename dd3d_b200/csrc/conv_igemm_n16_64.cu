// conv_igemm_kernel instantiations for block_n in {16, 32, 48, 64} (see conv_igemm_kernel.cuh).
#include "conv_igemm_kernel.cuh"

namespace dd3d {
DD3D_CONV_KERNEL_GROUP(conv_kernel_n16_64, 16, 32, 48, 64)
}  // namespace dd3d
