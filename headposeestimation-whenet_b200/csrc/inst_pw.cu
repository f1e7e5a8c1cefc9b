// Translation unit: the tensor-core 1x1-convolution kernels (pw_tc2 in kernels_tc.cuh, K2 in kernels_k2.cuh) for both 16-bit
// storage types (see inst_k1_bf16.cu for why the kernel families live in their own units).
#include "kernels_simt.cuh"
#include "kernels_tc.cuh"
#include "kernels_k2.cuh"

namespace whenet {
namespace tc {
#define WHENET_INST_PW(T)                                                                                                    \
    template int launch_pw_tc2<T>(cudaStream_t, const T*, const void*, const float*, const float*, const T*, T*, long long, \
                                  int, int, int, bool, int, int, int, bool);                                                 \
    template int launch_k2<T>(cudaStream_t, const K2Params&, size_t, bool, bool, bool, int);                \
    template int launch_pw_tc3<T>(cudaStream_t, const T*, const void*, const float*, const float*, const T*, T*, long long, int, int, int);
WHENET_INST_PW(__nv_bfloat16)
WHENET_INST_PW(__half)
#undef WHENET_INST_PW
}  // namespace tc
}  // namespace whenet
