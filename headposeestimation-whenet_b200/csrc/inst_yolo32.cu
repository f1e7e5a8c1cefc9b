// The detector's fp32 parity kernels (kernels_yolo32.cuh) and their launchers, in a unit of their own.
#define WHENET_YOLO_HOST_ONLY      // the bf16 kernels are inst_yolo.cu's
#include "kernels_yolo32.cuh"

namespace whenet {
namespace yolo {

template <int N>
int launch_conv0_32_t(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, const float* bias, float* out,
                      int n, int S_h, int S_w) {
    constexpr size_t smem = 128 * 128 + 2 * N * 128 + 256 * 4 + tc::acc_tile_bytes(N) + 1024;
    cudaError_t e = cudaFuncSetAttribute(yolo_conv0_32_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    const long long tiles = (long long)n * S_h * S_w / 128;           // S_h * S_w is a multiple of 1024
    yolo_conv0_32_kernel<N><<<(unsigned)tiles, 128, smem, s>>>(img, w_hi, w_lo, bias, out, S_h, S_w);
    return (int)cudaGetLastError();
}

int launch_conv0_32(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, const float* bias, float* out,
                    int n, int S_h, int S_w, int cout) {
    switch (cout) {
        case 16: return launch_conv0_32_t<16>(s, img, w_hi, w_lo, bias, out, n, S_h, S_w);
        case 32: return launch_conv0_32_t<32>(s, img, w_hi, w_lo, bias, out, n, S_h, S_w);
    }
    return (int)cudaErrorInvalidValue;
}

int launch_maxpool32(cudaStream_t s, const float* in, float* out, int n, int H, int W, int C, int stride) {
    const long long threads = (long long)n * ((H + stride - 1) / stride) * ((W + stride - 1) / stride) * (C / 4);
    yolo_maxpool32_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(in, out, n, H, W, C, stride);
    return (int)cudaGetLastError();
}

template <int MODE, int UN>
int launch_igemm32_t(cudaStream_t s, const Igemm32Params& p, size_t smem, int grid_n, int grid_m) {
    auto kfn = conv_igemm32_kernel<MODE, UN>;
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    kfn<<<dim3(grid_n, grid_m), 128, smem, s>>>(p);
    return (int)cudaGetLastError();
}

template <int MODE>
int launch_igemm32_m(cudaStream_t s, const Igemm32Params& p, int un, size_t smem, int grid_n, int grid_m) {
    switch (un) {
        case 32: return launch_igemm32_t<MODE, 32>(s, p, smem, grid_n, grid_m);
        case 64: return launch_igemm32_t<MODE, 64>(s, p, smem, grid_n, grid_m);
        case 128: return launch_igemm32_t<MODE, 128>(s, p, smem, grid_n, grid_m);
    }
    return (int)cudaErrorInvalidValue;
}

int launch_igemm32_mode(cudaStream_t s, const Igemm32Params& p, int mode, int un, size_t smem, int grid_n, int grid_m) {
    switch (mode) {
        case kLeaky: return launch_igemm32_m<kLeaky>(s, p, un, smem, grid_n, grid_m);
        case kLeakyRes: return launch_igemm32_m<kLeakyRes>(s, p, un, smem, grid_n, grid_m);
        case kLeakyCat: return launch_igemm32_m<kLeakyCat>(s, p, un, smem, grid_n, grid_m);
        case kLinearF32: return launch_igemm32_m<kLinearF32>(s, p, un, smem, grid_n, grid_m);
    }
    return (int)cudaErrorInvalidValue;
}

// launch_igemm's split into groups of whole frames past gridDim.y's limit; every tensor is fp32 here
int launch_igemm32(cudaStream_t s, const Igemm32Params& p, int mode, int un, size_t smem, int grid_n, int grid_m) {
    const long long hw = (long long)p.Ho * p.Wo;
    return for_each_frame_group((int)(p.M / hw), hw, [&](int f0, int nf) {
        if (nf * hw == p.M) return launch_igemm32_mode(s, p, mode, un, smem, grid_n, grid_m);
        Igemm32Params q = p;
        q.in = p.in + (size_t)f0 * p.Hi * p.Wi * (p.Cin - p.c_up);
        if (p.up) q.up = p.up + (size_t)f0 * (p.Hi / 2) * (p.Wi / 2) * p.c_up;
        if (p.resid) q.resid = p.resid + (size_t)f0 * hw * p.N;
        q.out = p.out + (size_t)f0 * hw * p.N;
        q.M = (int)(nf * hw);
        return launch_igemm32_mode(s, q, mode, un, smem, grid_n, (q.M + BM - 1) / BM);
    });
}

}  // namespace yolo
}  // namespace whenet
