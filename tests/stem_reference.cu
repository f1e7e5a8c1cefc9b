// Bit reference for the stem: the one-pixel-per-thread stem_tile_kernel the library ran before the register-blocked
// kernel replaced it, with the helpers it calls, copied verbatim into a namespace of their own so that this file
// depends on nothing in the library.  tests/test_gpu_stem.py compiles it into a shared library and compares the
// library's stem tap with stem_reference_launch's output bit for bit.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace stem_ref {

__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, const float (&v)[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    uint2 t; t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
}
__device__ __forceinline__ void st4(__half* p, const float (&v)[4]) {
    __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
    uint2 t; t.x = *reinterpret_cast<uint32_t*>(&a); t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
}
template <typename T> __device__ __forceinline__ void st8(T* p, const float (&v)[8]) {
    float a[4] = {v[0], v[1], v[2], v[3]}, b[4] = {v[4], v[5], v[6], v[7]};
    st4(p, a); st4(p + 4, b);
}
template <> __device__ __forceinline__ void st8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
    uint4 t; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
}
template <> __device__ __forceinline__ void st8<__half>(__half* p, const float (&v)[8]) {
    uint4 t; __half2* h = reinterpret_cast<__half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
}

__device__ __forceinline__ float swish_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float swish_fast(float x) {
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}

// ----------------------------------------------------------------------------- stem, tiled
// One CTA = two output rows of one crop (224 threads, one output pixel x 32 channels each).
// The 5 input rows are loaded with 16-byte vectors, normalised through the LUT once and staged as fp32 in
// shared memory (one extra zero pixel/row: TF-SAME puts its single pad row/column AFTER index 223).
// The 27x32 BN-folded weights + 32 shifts arrive as a __grid_constant__ kernel parameter, so every FFMA
// takes its weight straight from the constant bank (864 FFMA per thread, no weight loads at all).
struct StemParams { float w[27 * 32]; float b[32]; };

template <typename T, bool IN_U8, bool FAST>
__global__ void __launch_bounds__(224) stem_tile_kernel(const void* __restrict__ in_, T* __restrict__ out,
                                                        const __grid_constant__ StemParams sp,
                                                        const float* __restrict__ lut) {
    constexpr int ROWF = 225 * 3 + 1;              // floats per staged row (225 pixels incl. the zero pad pixel)
    __shared__ float s_in[5 * ROWF];
    __shared__ float s_lut[768];
    const int tid = threadIdx.x;
    const int n = blockIdx.y, oy0 = blockIdx.x * 2;
    if (IN_U8) {
        for (int i = tid; i < 768; i += 224) s_lut[i] = lut[i];
        __syncthreads();
    }
    // stage rows 2*oy0 .. 2*oy0+4 (row 224 does not exist -> zeros)
    if (IN_U8) {
        const uint8_t* src = reinterpret_cast<const uint8_t*>(in_) + (long long)n * 224 * 224 * 3;
        for (int v = tid; v < 5 * 42; v += 224) {           // 42 x 16 bytes per input row
            const int r = v / 42, q = v - r * 42;
            const int iy = 2 * oy0 + r;
            float* dst = &s_in[r * ROWF + q * 16];
            if (iy < 224) {
                const uint4 raw = *reinterpret_cast<const uint4*>(src + (long long)iy * 672 + q * 16);
                const uint8_t* b = reinterpret_cast<const uint8_t*>(&raw);
#pragma unroll
                for (int j = 0; j < 16; ++j) dst[j] = s_lut[((q * 16 + j) % 3) * 256 + b[j]];
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) dst[j] = 0.f;
            }
        }
    } else {
        const float* src = reinterpret_cast<const float*>(in_) + (long long)n * 224 * 224 * 3;
        for (int v = tid; v < 5 * 168; v += 224) {          // 168 x float4 per input row
            const int r = v / 168, q = v - r * 168;
            const int iy = 2 * oy0 + r;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (iy < 224) x = *reinterpret_cast<const float4*>(src + (long long)iy * 672 + q * 4);
            float* dst = &s_in[r * ROWF + q * 4];
            dst[0] = x.x; dst[1] = x.y; dst[2] = x.z; dst[3] = x.w;
        }
    }
    if (tid < 15) s_in[(tid / 3) * ROWF + 672 + tid % 3] = 0.f;   // pad pixel (column 224) of the 5 rows
    __syncthreads();
    const int oyl = tid / 112, ox = tid - oyl * 112;
    // 32 output channels as 16 pairs, weights from the constant bank, the scalar input broadcast
    float2 acc2[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc2[c] = make_float2(sp.b[2 * c], sp.b[2 * c + 1]);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const float* row = &s_in[(2 * oyl + ky) * ROWF + 6 * ox];
#pragma unroll
        for (int t = 0; t < 9; ++t) {                       // kx*3 + ci
            const float x = row[t];
            const float2 xx = make_float2(x, x);
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const float2 w2 = make_float2(sp.w[(ky * 9 + t) * 32 + 2 * c], sp.w[(ky * 9 + t) * 32 + 2 * c + 1]);
                acc2[c].x = fmaf(xx.x, w2.x, acc2[c].x);
                acc2[c].y = fmaf(xx.y, w2.y, acc2[c].y);
            }
        }
    }
    float acc[32];
#pragma unroll
    for (int c = 0; c < 16; ++c) { acc[2 * c] = acc2[c].x; acc[2 * c + 1] = acc2[c].y; }
    T* dst = out + (((long long)n * 112 + oy0 + oyl) * 112 + ox) * 32;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = FAST ? swish_fast(acc[g * 8 + j]) : swish_f(acc[g * 8 + j]);
        st8<T>(dst + g * 8, o);
    }
}

template <typename T, bool IN_U8, bool FAST>
static cudaError_t launch(const void* in, void* out, const StemParams& sp, const float* lut, int n) {
    stem_tile_kernel<T, IN_U8, FAST><<<dim3(56, n), 224>>>(in, reinterpret_cast<T*>(out), sp, lut);
    return cudaGetLastError();
}

}  // namespace stem_ref

// in: n x 224 x 224 x 3 uint8 (in_u8) or float32, device.  out: n x 112 x 112 x 32 device elements of the storage type
// out_type (0 = fp32, 1 = fp16 with the tanh swish, 2 = bf16 with the tanh swish).  w [27][32], b [32], host.
// lut [3][256], device (in_u8 only).  Synchronises and returns the CUDA error code.
extern "C" int stem_reference_launch(const void* in, void* out, int in_u8, int out_type, const float* w, const float* b,
                                     const float* lut, int n) {
    stem_ref::StemParams sp;
    for (int i = 0; i < 27 * 32; ++i) sp.w[i] = w[i];
    for (int i = 0; i < 32; ++i) sp.b[i] = b[i];
    cudaError_t e;
    if (out_type == 0) e = in_u8 ? stem_ref::launch<float, true, false>(in, out, sp, lut, n) : stem_ref::launch<float, false, false>(in, out, sp, lut, n);
    else if (out_type == 1) e = in_u8 ? stem_ref::launch<__half, true, true>(in, out, sp, lut, n) : stem_ref::launch<__half, false, true>(in, out, sp, lut, n);
    else if (out_type == 2) e = in_u8 ? stem_ref::launch<__nv_bfloat16, true, true>(in, out, sp, lut, n)
                                      : stem_ref::launch<__nv_bfloat16, false, true>(in, out, sp, lut, n);
    else return (int)cudaErrorInvalidValue;
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}
