// Translation unit: KD (kernels_dwse.cuh), the depthwise + squeeze-excite kernel of the late blocks (see inst_k1_bf16.cu).
#include "kernels_dwse.cuh"

namespace whenet {
namespace fused {
template int launch_dwse<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int);
template int launch_dwse_x<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int);
template int launch_dwse_spatial<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int);
}  // namespace fused
}  // namespace whenet
