// Translation unit: K1 (kernels_fused.cuh) and its TMA-fed sibling K1X (kernels_k1x.cuh) for bf16 storage.  The fused kernels are by far the slowest part of the build
// (48 heavily unrolled instantiations); giving each storage type and the K1P/K1T variants their own unit lets nvcc
// processes run side by side and limits a rebuild to the unit whose header changed (build.py).
#include "kernels_fused.cuh"
#include "kernels_k1x.cuh"

namespace whenet {
namespace fused {
template int launch_k1<__nv_bfloat16>(cudaStream_t, K1Params, int, int, int, int, size_t, int);
template int launch_dw_only<__nv_bfloat16>(cudaStream_t, K1Params, size_t, int);
template int launch_k1x<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int, int, int, int);
}  // namespace fused
}  // namespace whenet
