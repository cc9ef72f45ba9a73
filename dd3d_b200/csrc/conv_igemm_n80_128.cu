// conv_igemm_kernel instantiations for block_n in {80, 96, 112, 128} (see conv_igemm_kernel.cuh).
#include "conv_igemm_kernel.cuh"

namespace dd3d {
DD3D_CONV_KERNEL_GROUP(conv_kernel_n80_128, 80, 96, 112, 128)
}  // namespace dd3d
