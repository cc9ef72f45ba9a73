// conv_igemm_kernel instantiations for block_n in {208, 224, 240, 256} (see conv_igemm_kernel.cuh).
#include "conv_igemm_kernel.cuh"

namespace dd3d {
DD3D_CONV_KERNEL_GROUP(conv_kernel_n208_256, 208, 224, 240, 256)
}  // namespace dd3d
