// kernels_simt.cuh - CUDA-core (fp32 FMA) kernels of the WHENet forward.
//
// These are the parity-mode kernels (fp32 storage) and the fallback family for
// bf16/fp16 storage.  One kernel per logical op of SURVEY.md section 2.2:
//   stem_kernel        u8/f32 NHWC -> conv3x3 s2 SAME + BN + swish          (reference whenet.py:25-27 front)
//   pw_conv_kernel     1x1 conv as a tiled GEMM + BN bias (+swish) (+SE gate on A) (+residual)
//   dw_conv_kernel     depthwise kxk SAME + BN + swish + deterministic SE partial sums
//   se_gate_kernel     SE squeeze mean -> FC+swish -> FC+sigmoid
//   head_pool_fc_decode_kernel  GAP(7x7) -> 3 Dense -> softmax -> expectation  (whenet.py:10-13, 28-33; utils.py:7-11)
//
// Activations are NHWC in the storage type T (float, __nv_bfloat16, __half);
// all arithmetic is fp32.  BatchNorm is folded into the weights on the host
// (scale into the kernel, shift into `bias`).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

namespace whenet {

// ----------------------------------------------------------------------------- storage helpers
template <typename T> struct Store;
template <> struct Store<float> {
    static constexpr int VEC = 4;   // elements per 16-byte vector
    __device__ static __forceinline__ float ld(const float* p) { return *p; }
    __device__ static __forceinline__ void st(float* p, float v) { *p = v; }
    __device__ static __forceinline__ float rnd(float v) { return v; }
};
template <> struct Store<__nv_bfloat16> {
    static constexpr int VEC = 8;
    __device__ static __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
    __device__ static __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
    __device__ static __forceinline__ float rnd(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
};
template <> struct Store<__half> {
    static constexpr int VEC = 8;
    __device__ static __forceinline__ float ld(const __half* p) { return __half2float(*p); }
    __device__ static __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
    __device__ static __forceinline__ float rnd(float v) { return __half2float(__float2half_rn(v)); }
};

// load / store 4 consecutive elements as fp32
__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x), b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
    float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
__device__ __forceinline__ void ld4(const __half* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    __half2 a = *reinterpret_cast<__half2*>(&t.x), b = *reinterpret_cast<__half2*>(&t.y);
    float2 fa = __half22float2(a), fb = __half22float2(b);
    v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
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

// 8 consecutive elements (16 B for 16-bit types, 2x16 B for float)
template <typename T> __device__ __forceinline__ void ld8(const T* p, float (&v)[8]) {
    float a[4], b[4];
    ld4(p, a); ld4(p + 4, b);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[i] = a[i]; v[4 + i] = b[i]; }
}
template <> __device__ __forceinline__ void ld8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}
template <> __device__ __forceinline__ void ld8<__half>(const __half* p, float (&v)[8]) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
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

// x * sigmoid(x).  expf (not __expf): the parity mode has to stay within 1e-2 deg.
__device__ __forceinline__ float swish_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// x*sigmoid(x) = h + h*tanh(h), h = x/2  (MUFU.TANH: one SFU op instead of EX2 + RCP); 16-bit modes only
__device__ __forceinline__ float swish_fast(float x) {
    // x*sigmoid(x) = h + h*tanh(h), h = x/2  (MUFU.TANH: one SFU op instead of EX2 + RCP)
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}

// same, for an argument that is ALREADY x/2 (the producer folded the 1/2 into its weights and shift)
__device__ __forceinline__ float swish_from_half(float h) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}

// ----------------------------------------------------------------------------- stem
// out[n,oy,ox,co] = swish( bias[co] + sum_{ky,kx,ci} w[ky,kx,ci,co] * norm(in[n,2oy+ky,2ox+kx,ci]) )
// TF SAME for 224/k3/s2: pad_before 0, pad_after 1 -> the taps at index 224 read zero
// IN NORMALISED SPACE (SURVEY.md section 7, hard part 7), hence the explicit bounds test.
// 4 threads per output pixel, 8 output channels each -> 16 B (bf16) coalesced stores.
template <typename T, bool IN_U8>
__global__ void __launch_bounds__(256) stem_kernel(const void* __restrict__ in_, T* __restrict__ out,
                                                   const float* __restrict__ w,     // [27][32], BN-scale folded
                                                   const float* __restrict__ bias,  // [32]
                                                   const float* __restrict__ lut,   // [3][256] (IN_U8 only)
                                                   int n_img) {
    __shared__ float s_w[27 * 32];
    __shared__ float s_lut[3 * 256];
    for (int i = threadIdx.x; i < 27 * 32; i += 256) s_w[i] = w[i];
    if (IN_U8)
        for (int i = threadIdx.x; i < 768; i += 256) s_lut[i] = lut[i];
    __syncthreads();
    const long long total = (long long)n_img * 112 * 112 * 4;
    long long gid = (long long)blockIdx.x * 256 + threadIdx.x;
    if (gid >= total) return;
    const int cg = (int)(gid & 3);
    long long pix = gid >> 2;
    const int ox = (int)(pix % 112); pix /= 112;
    const int oy = (int)(pix % 112);
    const int n = (int)(pix / 112);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = bias[cg * 8 + i];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = 2 * oy + ky;
        if (iy >= 224) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int ix = 2 * ox + kx;
            if (ix >= 224) continue;
            const long long base = (((long long)n * 224 + iy) * 224 + ix) * 3;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                float x;
                if (IN_U8) x = s_lut[ci * 256 + reinterpret_cast<const uint8_t*>(in_)[base + ci]];
                else x = reinterpret_cast<const float*>(in_)[base + ci];
                const float* wr = &s_w[((ky * 3 + kx) * 3 + ci) * 32 + cg * 8];
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[i] = fmaf(x, wr[i], acc[i]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = swish_f(acc[i]);
    st8(out + (gid >> 2) * 32 + cg * 8, acc);
}

// ----------------------------------------------------------------------------- stem, register-blocked
// A tile = 8 output rows of one crop; a persistent CTA of 224 threads walks tiles blockIdx.x, + gridDim.x, ...  A thread
// computes 4 consecutive output pixels along x x 16 channels (64 fp32 accumulators), first for channels 0-15, then for
// 16-31: the channel half is a template argument, so every weight address is warp-uniform and an immediate.  The 27x32
// BN-folded weights sit in shared memory and are read as broadcast 16-byte loads; each weight feeds 4 FFMAs (one per
// pixel).  Each output is bias + fmaf over (ky, kx, ci) in that order, then swish: the padding taps are FMA'd with
// staged zeros (fmaf(0, w, acc) decides the sign of a zero).
//
// The tile's 17 input rows arrive raw by cp.async, issued while the previous tile computes, and are then converted once
// to fp32 (u8 through the LUT) in 9 planes per row, plane kx*3+ci holding x[2*ox + kx][ci] for ox = 0..111 (TF SAME
// puts its single pad row/column after index 223: row 224 and the last element of the kx = 2 planes are zeros).  A tap
// is then one conflict-free 16-byte load of the thread's 4 pixels.  Each half's outputs go through shared memory
// (XOR-swizzled 16-byte chunks) and leave as whole 32-byte sectors.
struct StemParams { float w[27 * 32]; float b[32]; };

constexpr int kStemRows = 8;                      // output rows per tile
constexpr int kStemTilesPerCrop = 112 / kStemRows;
constexpr int kStemThreads = kStemRows * 28;      // one thread per quad of output pixels
constexpr int kStemPlane = 112;                   // floats per plane (one per output column)
constexpr int kStemRowF = 9 * kStemPlane + 8;     // floats per staged input row; 8 mod 16 keeps a quarter-warp that spans
                                                  // two output rows (input rows 2 apart) on disjoint banks
constexpr int kStemInRows = 2 * kStemRows + 1;

// shared memory: planes | the stage of channels 0-15, which also holds the next tile's raw rows | LUT (u8) | weights.
// Channels 16-31 are staged over the planes.  16-bit storage, u8 input: 102 KB, two CTAs per SM.
template <typename T, bool IN_U8>
struct StemSmem {
    static constexpr size_t PLANES = (size_t)kStemInRows * kStemRowF * 4;
    static constexpr size_t RAW_ROW = 672 * (IN_U8 ? 1 : 4);                     // bytes of one input row
    static constexpr size_t STAGE = (size_t)kStemRows * 112 * 16 * sizeof(T);
    static constexpr size_t RAW = (size_t)kStemInRows * RAW_ROW;
    static constexpr size_t UNION = STAGE > RAW ? STAGE : RAW;
    static constexpr size_t LUT = PLANES + UNION, W = LUT + (IN_U8 ? 768 * 4 : 0);
    static constexpr size_t BYTES = W + 27 * 32 * 4;
};

// One channel half for pixel quad q (output row q / 28, columns 4 (q % 28) + 0..3): FMA, swish into `stage`, store.
// HALF 1 stages over the planes, hence its barrier before the stage writes.
template <int HALF, typename T, bool FAST>
__device__ __forceinline__ void stem_half(const float* s_in, const float* s_w, uint4* stage, T* out_run, int q, int tid,
                                          const StemParams& sp) {
    float acc[4][16];
#pragma unroll
    for (int c = 0; c < 16; ++c)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[p][c] = sp.b[HALF * 16 + c];
    const int oyl = q / 28;
    const float* x0 = s_in + 2 * oyl * kStemRowF + 4 * (q - oyl * 28);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int t = 0; t < 9; ++t) {                   // kx*3 + ci
            const float4 x = *reinterpret_cast<const float4*>(x0 + ky * kStemRowF + t * kStemPlane);
            const float xs[4] = {x.x, x.y, x.z, x.w};
            float ws[16];
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
                const float4 w4 = *reinterpret_cast<const float4*>(s_w + (ky * 9 + t) * 32 + HALF * 16 + 4 * c4);
                ws[4 * c4] = w4.x; ws[4 * c4 + 1] = w4.y; ws[4 * c4 + 2] = w4.z; ws[4 * c4 + 3] = w4.w;
            }
#pragma unroll
            for (int c = 0; c < 16; ++c)
#pragma unroll
                for (int p = 0; p < 4; ++p) acc[p][c] = fmaf(xs[p], ws[c], acc[p][c]);
        }
    if (HALF == 1) __syncthreads();
    // 16-byte chunk k of the half's stage (pixel k / CPH, chunk k % CPH of its 16 channels) is stored at
    // k ^ ((k >> SH) & 7): a quarter-warp's chunks (same pixel slot, consecutive quads) then fall on distinct banks, and
    // so do 8 consecutive chunks read back
    constexpr int CPH = (int)sizeof(T);                     // 16-byte chunks per pixel and half (16 channels)
    constexpr int SH = CPH == 2 ? 3 : 4;                    // log2(4 * CPH): k >> SH is the quad index
    constexpr int VPC = 16 / (int)sizeof(T);                // values per chunk
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int j = 0; j < CPH; ++j) {
            const int k = (q * 4 + p) * CPH + j;
            float o[VPC];
#pragma unroll
            for (int e = 0; e < VPC; ++e) o[e] = FAST ? swish_fast(acc[p][j * VPC + e]) : swish_f(acc[p][j * VPC + e]);
            T* dst = reinterpret_cast<T*>(stage + (k ^ ((k >> SH) & 7)));
            if constexpr (sizeof(T) == 2) st8<T>(dst, o);
            else st4(dst, o);
        }
    __syncthreads();
    uint4* g = reinterpret_cast<uint4*>(out_run + HALF * 16);
#pragma unroll
    for (int k = tid; k < kStemRows * 112 * CPH; k += kStemThreads)
        g[(k / CPH) * 2 * CPH + k % CPH] = stage[k ^ ((k >> SH) & 7)];
}

// cp.async the existing input rows 2*oy0 .. 2*oy0+16 of tile `tile` into `raw` (row 224 does not exist: never read)
template <bool IN_U8>
__device__ __forceinline__ void stem_fetch(const void* in_, char* raw, int tile, int tid) {
    constexpr int ROW = 672 * (IN_U8 ? 1 : 4), CPR = ROW / 16;
    const int n = tile / kStemTilesPerCrop, oy0 = (tile - n * kStemTilesPerCrop) * kStemRows;
    const int rows = min(kStemInRows, 224 - 2 * oy0);
    const char* src = reinterpret_cast<const char*>(in_) + ((long long)n * 224 + 2 * oy0) * ROW;
    for (int i = tid; i < rows * CPR; i += kStemThreads) {
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(raw + i * 16);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + (long long)i * 16) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

template <typename T, bool IN_U8, bool FAST>
__global__ void __launch_bounds__(kStemThreads, 2) stem_tile_kernel(const void* __restrict__ in_, T* __restrict__ out,
                                                                    const __grid_constant__ StemParams sp,
                                                                    const float* __restrict__ lut, int n_img) {
    using S = StemSmem<T, IN_U8>;
    extern __shared__ float4 stem_smem_v[];
    char* base = reinterpret_cast<char*>(stem_smem_v);
    float* s_in = reinterpret_cast<float*>(base);
    char* s_raw = base + S::PLANES;
    uint4* stage0 = reinterpret_cast<uint4*>(base + S::PLANES);
    float* s_lut = reinterpret_cast<float*>(base + S::LUT);
    float* s_w = reinterpret_cast<float*>(base + S::W);
    const int tid = threadIdx.x;
    const int tiles = n_img * kStemTilesPerCrop;
    int tile = blockIdx.x;
    if (tile < tiles) stem_fetch<IN_U8>(in_, s_raw, tile, tid);
    for (int i = tid; i < 27 * 32; i += kStemThreads) s_w[i] = sp.w[i];
    if (IN_U8)
        for (int i = tid; i < 768; i += kStemThreads) s_lut[i] = lut[i];
    for (; tile < tiles; tile += gridDim.x) {
        const int n = tile / kStemTilesPerCrop, oy0 = (tile - n * kStemTilesPerCrop) * kStemRows;
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                                    // raw rows in; the previous tile's output stage is drained
        // item (r, m) = input columns 2m, 2m+1 of input row 2*oy0 + r
        for (int i = tid; i < kStemInRows * 112; i += kStemThreads) {
            const int r = i / 112, m = i - r * 112;
            float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};    // row 224 (TF SAME's pad row) is staged as zeros
            if (2 * oy0 + r < 224) {
                const char* src = s_raw + r * S::RAW_ROW;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    if (IN_U8) {
                        const uint16_t u = reinterpret_cast<const uint16_t*>(src + 6 * m)[k];
                        v[2 * k] = s_lut[((2 * k) % 3) * 256 + (u & 0xff)];
                        v[2 * k + 1] = s_lut[((2 * k + 1) % 3) * 256 + (u >> 8)];
                    } else {
                        const float2 f = reinterpret_cast<const float2*>(src + 24 * m)[k];
                        v[2 * k] = f.x; v[2 * k + 1] = f.y;
                    }
                }
            }
            float* row = s_in + r * kStemRowF;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                row[ci * kStemPlane + m] = v[ci];                                  // kx = 0: column 2m
                row[(3 + ci) * kStemPlane + m] = v[3 + ci];                        // kx = 1: column 2m + 1
                if (m > 0) row[(6 + ci) * kStemPlane + m - 1] = v[ci];             // kx = 2: column 2(m - 1) + 2
                else row[(6 + ci) * kStemPlane + 111] = 0.f;                       // ... and the pad column 224
            }
        }
        __syncthreads();
        T* out_run = out + ((long long)n * 112 + oy0) * 112 * 32;   // the tile's 8 rows: one contiguous run of NHWC
        stem_half<0, T, FAST>(s_in, s_w, stage0, out_run, tid, tid, sp);
        __syncthreads();                                    // stage 0 drained: the next tile's rows may land there
        if (tile + (int)gridDim.x < tiles) stem_fetch<IN_U8>(in_, s_raw, tile + gridDim.x, tid);
        stem_half<1, T, FAST>(s_in, s_w, reinterpret_cast<uint4*>(base), out_run, tid, tid, sp);
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// `in` must be 16-byte aligned (cp.async of whole rows).  Grid: as many CTAs as fit on the device, at most one per tile.
template <typename T, bool IN_U8, bool FAST>
cudaError_t launch_stem_tile(cudaStream_t stream, const void* in, T* out, const StemParams& sp, const float* lut, int n) {
    auto kfn = stem_tile_kernel<T, IN_U8, FAST>;
    constexpr size_t smem = StemSmem<T, IN_U8>::BYTES;
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int dev = 0, sms = 0, per_sm = 0;
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, kStemThreads, smem);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) return cudaErrorInvalidConfiguration;
    const long long tiles = (long long)n * kStemTilesPerCrop;
    kfn<<<(unsigned)std::min(tiles, (long long)per_sm * sms), kStemThreads, smem, stream>>>(in, out, sp, lut, n);
    return cudaGetLastError();
}

// ----------------------------------------------------------------------------- 1x1 conv (CUDA-core GEMM)
// out[m, n] = act( bias[n] + sum_k A[m,k]*gate[m/hw, k] * W[k,n] ) (+ resid[m,n])
// 64x64 tile, BK=16, 256 threads, 4x4 outputs per thread.  K and N are multiples of 8.
template <typename T, bool SWISH, bool GATE, bool RESID>
__global__ void __launch_bounds__(256) pw_conv_kernel(const T* __restrict__ A, const float* __restrict__ W,
                                                      const float* __restrict__ bias, const float* __restrict__ gate,
                                                      const T* __restrict__ resid, T* __restrict__ out,
                                                      long long M, int K, int N, int hw) {
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const long long m0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int a_row = tid >> 2, a_k = (tid & 3) * 4;      // A tile: 64 rows x 16 k, 4 k per thread
    const int b_k = tid >> 4, b_n = (tid & 15) * 4;       // B tile: 16 k x 64 n, 4 n per thread
    const long long a_m = m0 + a_row;
    const bool a_ok = a_m < M;
    const float* gate_row = GATE ? gate + (a_ok ? (a_m / hw) : 0) * K : nullptr;

    for (int k0 = 0; k0 < K; k0 += BK) {
        float av[4] = {0.f, 0.f, 0.f, 0.f};
        if (a_ok && k0 + a_k < K) {
            ld4(A + a_m * K + k0 + a_k, av);
            if (GATE) {
                float g[4]; ld4(gate_row + k0 + a_k, g);
#pragma unroll
                for (int i = 0; i < 4; ++i) av[i] *= g[i];
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) As[a_k + i][a_row] = av[i];
        float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k0 + b_k < K && n0 + b_n < N) bv = *reinterpret_cast<const float4*>(W + (long long)(k0 + b_k) * N + n0 + b_n);
        *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = bv;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    const int n = n0 + tx * 4;
    if (n >= N) return;
    float bb[4]; ld4(bias + n, bb);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= M) break;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float x = acc[i][j] + bb[j];
            v[j] = SWISH ? swish_f(x) : x;
        }
        if (RESID) {
            float r[4]; ld4(resid + m * N + n, r);
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] += r[j];
        }
        st4(out + m * N + n, v);
    }
}

// ----------------------------------------------------------------------------- depthwise
// out[n,oy,ox,c] = swish( bias[c] + sum_{ky,kx} w[ky,kx,c] * in[n, oy*S+ky-pad, ox*S+kx-pad, c] )
// plus partial[n][tile][c] = sum over the tile's pixels of out (fp32, fixed order -> batch invariant).
// block = (C/8 channel vectors, PY pixel lanes); grid = (tiles, N); a tile is ROWS output rows.
template <typename T, int KS, int S>
__global__ void __launch_bounds__(256) dw_conv_kernel(const T* __restrict__ in, const float* __restrict__ w,  // [KS*KS][C]
                                                      const float* __restrict__ bias, T* __restrict__ out,
                                                      float* __restrict__ partial,  // [N][tiles][C]
                                                      int Hin, int Ho, int C, int pad, int rows) {
    extern __shared__ float s_red[];   // [PY][C]
    const int cv = threadIdx.x, py = threadIdx.y, PY = blockDim.y;
    const int c0 = cv * 8;
    const int n = blockIdx.y, tile = blockIdx.x;
    const int r0 = tile * rows;
    const int r1 = min(Ho, r0 + rows);
    const int npix = (r1 - r0) * Ho;
    const T* in_n = in + (long long)n * Hin * Hin * C;
    T* out_n = out + (long long)n * Ho * Ho * C;
    float bb[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) bb[i] = bias[c0 + i];
    float sum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sum[i] = 0.f;
    for (int p = py; p < npix; p += PY) {
        const int oy = r0 + p / Ho, ox = p % Ho;
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = bb[i];
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) {
            const int iy = oy * S + ky - pad;
            if (iy < 0 || iy >= Hin) continue;
#pragma unroll
            for (int kx = 0; kx < KS; ++kx) {
                const int ix = ox * S + kx - pad;
                if (ix < 0 || ix >= Hin) continue;
                float x[8], ww[8];
                ld8(in_n + ((long long)iy * Hin + ix) * C + c0, x);
                ld8(w + (ky * KS + kx) * C + c0, ww);
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[i] = fmaf(x[i], ww[i], acc[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) { acc[i] = swish_f(acc[i]); }
        st8(out_n + ((long long)oy * Ho + ox) * C + c0, acc);
        // the SE squeeze averages what the next layer will actually read: the stored (rounded) value
#pragma unroll
        for (int i = 0; i < 8; ++i) sum[i] += Store<T>::rnd(acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_red[py * C + c0 + i] = sum[i];
    __syncthreads();
    if (py == 0) {
        float tot[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) tot[i] = 0.f;
        for (int y = 0; y < PY; ++y)
#pragma unroll
            for (int i = 0; i < 8; ++i) tot[i] += s_red[y * C + c0 + i];
        float* dst = partial + ((long long)n * gridDim.x + tile) * C + c0;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = tot[i];
    }
}

// ----------------------------------------------------------------------------- depthwise, register-blocked
// Same contract as dw_conv_kernel, but every thread produces a strip of R consecutive output pixels of
// one row for its 8 channels: the (R-1)*S+KS input columns of each kernel row are loaded once and feed
// all the taps that touch them (KS*KS loads per output -> ((R-1)*S+KS)*KS/R), the KS weights of the
// current kernel row live in registers.  FAST selects the 1-MUFU swish (tanh.approx) of the 16-bit modes.

template <typename T, int KS, int S, int R, bool FAST>
__global__ void __launch_bounds__(256) dw_strip_kernel(const T* __restrict__ in, const float* __restrict__ w,  // [KS*KS][C]
                                                       const float* __restrict__ bias, T* __restrict__ out,
                                                       float* __restrict__ partial,  // [N][tiles][C]
                                                       int Hin, int Ho, int C, int pad, int rows) {
    extern __shared__ float s_red[];   // [PY][C]
    constexpr int NCOL = (R - 1) * S + KS;
    const int cv = threadIdx.x, py = threadIdx.y, PY = blockDim.y;
    const int c0 = cv * 8;
    const int n = blockIdx.y, tile = blockIdx.x;
    const int r0 = tile * rows;
    const int r1 = min(Ho, r0 + rows);
    const int spr = (Ho + R - 1) / R;              // strips per output row
    const int nstrips = (r1 - r0) * spr;
    const T* in_n = in + (long long)n * Hin * Hin * C;
    T* out_n = out + (long long)n * Ho * Ho * C;
    float bb[8];
    {
        const float4 b0 = *reinterpret_cast<const float4*>(bias + c0), b1 = *reinterpret_cast<const float4*>(bias + c0 + 4);
        bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w; bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
    }
    float sum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sum[i] = 0.f;
    for (int sidx = py; sidx < nstrips; sidx += PY) {
        const int oy = r0 + sidx / spr, ox0 = (sidx % spr) * R;
        float acc[R][8];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[r][i] = bb[i];
        const int ix0 = ox0 * S - pad;
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) {
            const int iy = oy * S + ky - pad;
            if (iy < 0 || iy >= Hin) continue;
            float wr[KS][8];
#pragma unroll
            for (int kx = 0; kx < KS; ++kx) {
                const float4 w0 = *reinterpret_cast<const float4*>(w + (ky * KS + kx) * C + c0);
                const float4 w1 = *reinterpret_cast<const float4*>(w + (ky * KS + kx) * C + c0 + 4);
                wr[kx][0] = w0.x; wr[kx][1] = w0.y; wr[kx][2] = w0.z; wr[kx][3] = w0.w;
                wr[kx][4] = w1.x; wr[kx][5] = w1.y; wr[kx][6] = w1.z; wr[kx][7] = w1.w;
            }
            const T* row = in_n + (long long)iy * Hin * C + c0;
#pragma unroll
            for (int col = 0; col < NCOL; ++col) {
                const int ix = ix0 + col;
                if (ix < 0 || ix >= Hin) continue;
                float x[8];
                ld8<T>(row + (long long)ix * C, x);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int kx = col - r * S;          // compile-time after unrolling
                    if (kx >= 0 && kx < KS) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) acc[r][i] = fmaf(x[i], wr[kx][i], acc[r][i]);
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int ox = ox0 + r;
            if (ox < Ho) {
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[r][i] = FAST ? swish_fast(acc[r][i]) : swish_f(acc[r][i]);
                st8<T>(out_n + ((long long)oy * Ho + ox) * C + c0, acc[r]);
#pragma unroll
                for (int i = 0; i < 8; ++i) sum[i] += Store<T>::rnd(acc[r][i]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_red[py * C + c0 + i] = sum[i];
    __syncthreads();
    if (py == 0) {
        float tot[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) tot[i] = 0.f;
        for (int y = 0; y < PY; ++y)
#pragma unroll
            for (int i = 0; i < 8; ++i) tot[i] += s_red[y * C + c0 + i];
        float* dst = partial + ((long long)n * gridDim.x + tile) * C + c0;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = tot[i];
    }
}

// ----------------------------------------------------------------------------- SE gate
// mean[c] = sum_tiles partial / (Ho*Ho); h = swish(W1^T mean + b1); gate = sigmoid(W2^T h + b2)
// Device function for ONE crop, executed by a whole 256-thread CTA: the stand-alone kernel below and the tail of
// K1 (the last CTA of a crop to finish) both call it.  `sm` = C + Cse floats of shared memory.
// `partial` is read with ld.global.cg: it may have been written by other CTAs of the same launch.
// the two FC layers of the gate, from the channel means in shared memory (`mean`: C floats, `hid`: Cse floats of scratch).
// The arithmetic and its order do not depend on NT or on who calls it (se_gate_kernel, the ticket tail of K1, the
// per-CTA tail of K1 for blocks whose tile is the whole image), so every route gives the same bits.
template <int NT>
__device__ __forceinline__ void se_gate_fc(const float* mean, float* hid, const float* __restrict__ w1t, const float* __restrict__ b1,
                                           const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ gate_n,
                                           int C, int Cse, float* gate_sm = nullptr) {
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    // FC1: lane L owns the channels 128 k + 4 L + {0..3} (one 16-byte load per k; every load of a row is in flight at once -
    // the serial chain of L2 round trips was the whole cost of the gate at C = 1152), FMAs in ascending channel order,
    // then the xor-shuffle tree.  This order is the definition every route shares (se_gate_kernel, se_gate_batch_kernel,
    // the tails of K1 / KD), so their gates agree bit for bit.
    for (int j = warp; j < Cse; j += NT / 32) {
        float s = 0.f;
        const float* wr = w1t + (long long)j * C;
        for (int c0 = lane * 4; c0 < C; c0 += 8 * 128) {
            float4 wv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (c0 + u * 128 < C) wv[u] = __ldg(reinterpret_cast<const float4*>(wr + c0 + u * 128));
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (c0 + u * 128 < C) {
                    const float4 mv = *reinterpret_cast<const float4*>(mean + c0 + u * 128);
                    s = fmaf(mv.x, wv[u].x, s); s = fmaf(mv.y, wv[u].y, s); s = fmaf(mv.z, wv[u].z, s); s = fmaf(mv.w, wv[u].w, s);
                }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) hid[j] = swish_f(s + b1[j]);
    }
    __syncthreads();
    for (int c = tid; c < C; c += NT) {
        float s = b2[c];
        const float* wc = w2 + c;
        int j = 0;
        for (; j + 7 < Cse; j += 8) {
            float wv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) wv[u] = wc[(long long)(j + u) * C];
#pragma unroll
            for (int u = 0; u < 8; ++u) s = fmaf(hid[j + u], wv[u], s);
        }
        for (; j < Cse; ++j) s = fmaf(hid[j], wc[(long long)j * C], s);
        const float g = sigmoid_f(s);
        gate_n[c] = g;
        if (gate_sm) gate_sm[c] = g;      // may alias `mean`: the means are dead after the barrier above
    }
}

template <bool COHERENT, int NT = 256>
__device__ __forceinline__ void se_gate_crop(const float* __restrict__ partial_n, int tiles, float inv_hw,
                                             const float* __restrict__ w1t, const float* __restrict__ b1,
                                             const float* __restrict__ w2, const float* __restrict__ b2,
                                             float* __restrict__ gate_n, int C, int Cse, float* sm) {
    float* mean = sm;
    float* hid = sm + C;
    const int tid = threadIdx.x;
    for (int c = tid; c < C; c += NT) {
        // four independent partial chains keep several loads in flight; the association order is fixed (t mod 4), so
        // the sum stays bitwise reproducible
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int t = 0;
        for (; t + 3 < tiles; t += 4) {
            const float* q = partial_n + (long long)t * C + c;
            if (COHERENT) { s0 += __ldcg(q); s1 += __ldcg(q + C); s2 += __ldcg(q + 2 * C); s3 += __ldcg(q + 3 * C); }
            else { s0 += q[0]; s1 += q[C]; s2 += q[2 * C]; s3 += q[3 * C]; }
        }
        for (; t < tiles; ++t) s0 += COHERENT ? __ldcg(partial_n + (long long)t * C + c) : partial_n[(long long)t * C + c];
        mean[c] = ((s0 + s1) + (s2 + s3)) * inv_hw;
    }
    __syncthreads();
    se_gate_fc<NT>(mean, hid, w1t, b1, w2, b2, gate_n, C, Cse);
}

template <int NT>
__global__ void __launch_bounds__(NT) se_gate_kernel(const float* __restrict__ partial, int tiles, float inv_hw,
                                                      const float* __restrict__ w1t,  // [Cse][C]
                                                      const float* __restrict__ b1,   // [Cse]
                                                      const float* __restrict__ w2,   // [Cse][C]
                                                      const float* __restrict__ b2,   // [C]
                                                      float* __restrict__ gate,       // [N][C]
                                                      int C, int Cse) {
    extern __shared__ float sm[];   // mean[C] | hid[Cse]
    const int n = blockIdx.x;
    se_gate_crop<false, NT>(partial + (long long)n * tiles * C, tiles, inv_hw, w1t, b1, w2, b2, gate + (long long)n * C, C, Cse, sm);
}

// The same gates for SEB crops per CTA: the two FC matrices (2 x Cse x C floats - 442 KB at C = 1152) are read once per
// SEB crops instead of once per crop, with 16-byte loads and every load of a row in flight together.  Every sum keeps the
// order of se_gate_crop / se_gate_fc (partials: four chains by tile index; FC1: lane L owns channels 128 k + 4 L + i,
// ascending, xor-shuffle tree; FC2: j ascending), so the gates are bit-identical to se_gate_kernel's and the routes can be
// mixed freely.  Shared-memory arrays are 16-byte aligned: C % 4 == 0 (every block of the network).
template <int SEB, int NT>
__global__ void __launch_bounds__(NT) se_gate_batch_kernel(const float* __restrict__ partial, int tiles, float inv_hw,
                                                            const float* __restrict__ w1t, const float* __restrict__ b1,
                                                            const float* __restrict__ w2, const float* __restrict__ b2,
                                                            float* __restrict__ gate, int C, int Cse, int N) {
    extern __shared__ __align__(16) float sm[];   // mean[SEB][C] | hid[SEB][Cse]
    float* mean = sm;
    float* hid = sm + SEB * C;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n0 = blockIdx.x * SEB;
    const int nb = min(SEB, N - n0);
    const int C4 = C >> 2;
    for (int idx = tid; idx < SEB * C4; idx += NT) {
        const int b = idx / C4, c = (idx - b * C4) * 4;
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b < nb) {
            const float* q0 = partial + (long long)(n0 + b) * tiles * C + c;
            float4 s0 = m, s1 = m, s2 = m, s3 = m;
            auto add = [](float4& a, const float4 v) { a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; };
            int t = 0;
            for (; t + 3 < tiles; t += 4) {
                const float* q = q0 + (long long)t * C;
                const float4 v0 = __ldg(reinterpret_cast<const float4*>(q)), v1 = __ldg(reinterpret_cast<const float4*>(q + C));
                const float4 v2 = __ldg(reinterpret_cast<const float4*>(q + 2 * C)), v3 = __ldg(reinterpret_cast<const float4*>(q + 3 * C));
                add(s0, v0); add(s1, v1); add(s2, v2); add(s3, v3);
            }
            for (; t < tiles; ++t) add(s0, __ldg(reinterpret_cast<const float4*>(q0 + (long long)t * C)));
            m.x = ((s0.x + s1.x) + (s2.x + s3.x)) * inv_hw; m.y = ((s0.y + s1.y) + (s2.y + s3.y)) * inv_hw;
            m.z = ((s0.z + s1.z) + (s2.z + s3.z)) * inv_hw; m.w = ((s0.w + s1.w) + (s2.w + s3.w)) * inv_hw;
        }
        *reinterpret_cast<float4*>(mean + b * C + c) = m;
    }
    __syncthreads();
    for (int j = warp; j < Cse; j += NT / 32) {
        float s[SEB];
#pragma unroll
        for (int b = 0; b < SEB; ++b) s[b] = 0.f;
        const float* wr = w1t + (long long)j * C;
        for (int c0 = lane * 4; c0 < C; c0 += 8 * 128) {
            float4 wv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (c0 + u * 128 < C) wv[u] = __ldg(reinterpret_cast<const float4*>(wr + c0 + u * 128));
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (c0 + u * 128 < C) {
#pragma unroll
                    for (int b = 0; b < SEB; ++b) {
                        const float4 mv = *reinterpret_cast<const float4*>(mean + b * C + c0 + u * 128);
                        s[b] = fmaf(mv.x, wv[u].x, s[b]); s[b] = fmaf(mv.y, wv[u].y, s[b]);
                        s[b] = fmaf(mv.z, wv[u].z, s[b]); s[b] = fmaf(mv.w, wv[u].w, s[b]);
                    }
                }
        }
#pragma unroll
        for (int b = 0; b < SEB; ++b) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[b] += __shfl_xor_sync(0xffffffffu, s[b], o);
        }
        if (lane == 0) {
            const float bj = b1[j];
#pragma unroll
            for (int b = 0; b < SEB; ++b) hid[b * Cse + j] = swish_f(s[b] + bj);
        }
    }
    __syncthreads();
    // FC2: one thread per four channels, sixteen weight rows in flight per step
    for (int c = tid * 4; c < C; c += NT * 4) {
        float4 s[SEB];
        const float4 bc = __ldg(reinterpret_cast<const float4*>(b2 + c));
#pragma unroll
        for (int b = 0; b < SEB; ++b) s[b] = bc;
        const float* wc = w2 + c;
        for (int j0 = 0; j0 < Cse; j0 += 16) {
            float4 wv[16];
#pragma unroll
            for (int u = 0; u < 16; ++u)
                if (j0 + u < Cse) wv[u] = __ldg(reinterpret_cast<const float4*>(wc + (long long)(j0 + u) * C));
#pragma unroll
            for (int u = 0; u < 16; ++u)
                if (j0 + u < Cse) {
#pragma unroll
                    for (int b = 0; b < SEB; ++b) {
                        const float h = hid[b * Cse + j0 + u];
                        s[b].x = fmaf(h, wv[u].x, s[b].x); s[b].y = fmaf(h, wv[u].y, s[b].y);
                        s[b].z = fmaf(h, wv[u].z, s[b].z); s[b].w = fmaf(h, wv[u].w, s[b].w);
                    }
                }
        }
#pragma unroll
        for (int b = 0; b < SEB; ++b)
            if (b < nb)
                *reinterpret_cast<float4*>(gate + (long long)(n0 + b) * C + c) =
                    make_float4(sigmoid_f(s[b].x), sigmoid_f(s[b].y), sigmoid_f(s[b].z), sigmoid_f(s[b].w));
    }
}

// softmax (reference utils.py:7-11: exp(x - max) / sum) and the bin-index expectation (reference whenet.py:31-33) of the
// three heads: warp w < 3 of the CTA decodes head w from the 252 logits in shared memory.
__device__ __forceinline__ void decode_heads(const float* logit, float* __restrict__ angles_n, int warp, int lane) {
    if (warp < 3) {
        const int off = warp == 0 ? 0 : (warp == 1 ? 120 : 186);
        const int cnt = warp == 0 ? 120 : 66;
        float mx = -INFINITY;
        for (int j = lane; j < cnt; j += 32) mx = fmaxf(mx, logit[off + j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float se = 0.f, sw = 0.f;
        for (int j = lane; j < cnt; j += 32) {
            const float e = expf(logit[off + j] - mx);
            se += e; sw = fmaf(e, (float)j, sw);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { se += __shfl_xor_sync(0xffffffffu, se, o); sw += __shfl_xor_sync(0xffffffffu, sw, o); }
        if (lane == 0) angles_n[warp] = (sw / se) * 3.0f - (warp == 0 ? 180.0f : 99.0f);
    }
}

// ----------------------------------------------------------------------------- head: GAP + 3 Dense + softmax + expectation
// feat: [N][49][1280] (post BN+swish head conv), or pooled sums when POOLED.
// One CTA per crop.  angles[n] = {yaw, pitch, roll}; logits optional [N][252].
template <typename T>
__global__ void __launch_bounds__(256) head_pool_fc_decode_kernel(const T* __restrict__ feat, const float* __restrict__ pooled_in,
                                                                 const float* __restrict__ wfc_t,  // [252][1280]
                                                                 const float* __restrict__ bfc,    // [252]
                                                                 float* __restrict__ angles, float* __restrict__ logits_out,
                                                                 float* __restrict__ pooled_out) {
    constexpr int C = 1280, NL = 252, HW = 49;
    __shared__ __align__(16) float pooled[C];
    __shared__ float logit[NL + 4];
    const int n = blockIdx.x, tid = threadIdx.x;
    if (pooled_in) {
        for (int c = tid; c < C; c += 256) pooled[c] = pooled_in[(long long)n * C + c];
    } else {
        const T* f = feat + (long long)n * HW * C;
        for (int c = tid; c < C; c += 256) {
            float s = 0.f;
#pragma unroll 7
            for (int p = 0; p < HW; ++p) s += Store<T>::ld(f + p * C + c);
            pooled[c] = s * (1.0f / 49.0f);
        }
    }
    __syncthreads();
    if (pooled_out)
        for (int c = tid; c < C; c += 256) pooled_out[(long long)n * C + c] = pooled[c];
    const int warp = tid >> 5, lane = tid & 31;
    // Dense rows: lane L owns the channels 128 k + 4 L + {0..3} (ten 16-byte weight loads, all in flight), FMAs in ascending
    // channel order, xor-shuffle tree - the order head_fc_decode_batch_kernel shares, so both give the same bits
    for (int j = warp; j < NL; j += 8) {
        const float* wr = wfc_t + (long long)j * C;
        float4 wv[C / 128];
#pragma unroll
        for (int u = 0; u < C / 128; ++u) wv[u] = __ldg(reinterpret_cast<const float4*>(wr + lane * 4 + u * 128));
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < C / 128; ++u) {
            const float4 pv = *reinterpret_cast<const float4*>(pooled + lane * 4 + u * 128);
            s = fmaf(pv.x, wv[u].x, s); s = fmaf(pv.y, wv[u].y, s); s = fmaf(pv.z, wv[u].z, s); s = fmaf(pv.w, wv[u].w, s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) logit[j] = s + bfc[j];
    }
    __syncthreads();
    if (logits_out)
        for (int j = tid; j < NL; j += 256) logits_out[(long long)n * NL + j] = logit[j];
    decode_heads(logit, angles + (long long)n * 3, warp, lane);
}

// Throughput batches: the head as two kernels.  (1) GAP: one thread per eight channels, 16-byte loads, the 49 pixels summed in
// ascending order exactly as above -> pooled [N][1280] fp32.  (2) Dense + decode for HB crops per CTA: every 16-byte load of the
// 1.3 MB Dense matrix serves HB crops (one CTA per crop re-read the whole matrix from L2 for each crop: 0.09 ms per 512 crops).
template <typename T>
__global__ void __launch_bounds__(160) head_pool_kernel(const T* __restrict__ feat, float* __restrict__ pooled) {
    constexpr int C = 1280, HW = 49;
    const int n = blockIdx.x, c0 = threadIdx.x * 8;
    const T* f = feat + (long long)n * HW * C + c0;
    float s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = 0.f;
#pragma unroll 7
    for (int p = 0; p < HW; ++p) {
        float v[8];
        ld8<T>(f + (long long)p * C, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += v[i];
    }
    float* dst = pooled + (long long)n * C + c0;
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = s[i] * (1.0f / 49.0f);
}

template <int HB>
__global__ void __launch_bounds__(512) head_fc_decode_batch_kernel(const float* __restrict__ pooled_in, const float* __restrict__ wfc_t,
                                                                   const float* __restrict__ bfc, float* __restrict__ angles,
                                                                   float* __restrict__ logits_out, int N) {
    constexpr int C = 1280, NL = 252, LP = 256;
    extern __shared__ __align__(16) float sm_head[];     // pooled[HB][C] | logit[HB][LP]
    float* pooled = sm_head;
    float* logit = sm_head + HB * C;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n0 = blockIdx.x * HB, nb = min(HB, N - n0);
    for (int i = tid; i < HB * C / 4; i += 512) {
        const int b = i / (C / 4);
        reinterpret_cast<float4*>(pooled)[i] = b < nb ? __ldg(reinterpret_cast<const float4*>(pooled_in + (long long)n0 * C) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    for (int j = warp; j < NL; j += 16) {
        const float* wr = wfc_t + (long long)j * C;
        float4 wv[C / 128];
#pragma unroll
        for (int u = 0; u < C / 128; ++u) wv[u] = __ldg(reinterpret_cast<const float4*>(wr + lane * 4 + u * 128));
        float s[HB];
#pragma unroll
        for (int b = 0; b < HB; ++b) s[b] = 0.f;
#pragma unroll
        for (int u = 0; u < C / 128; ++u)
#pragma unroll
            for (int b = 0; b < HB; ++b) {
                const float4 pv = *reinterpret_cast<const float4*>(pooled + b * C + lane * 4 + u * 128);
                s[b] = fmaf(pv.x, wv[u].x, s[b]); s[b] = fmaf(pv.y, wv[u].y, s[b]); s[b] = fmaf(pv.z, wv[u].z, s[b]); s[b] = fmaf(pv.w, wv[u].w, s[b]);
            }
#pragma unroll
        for (int b = 0; b < HB; ++b) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[b] += __shfl_xor_sync(0xffffffffu, s[b], o);
        }
        if (lane == 0) {
            const float bj = bfc[j];
#pragma unroll
            for (int b = 0; b < HB; ++b) logit[b * LP + j] = s[b] + bj;
        }
    }
    __syncthreads();
    if (logits_out)
        for (int i = tid; i < nb * NL; i += 512) {
            const int b = i / NL, j = i - b * NL;
            logits_out[(long long)(n0 + b) * NL + j] = logit[b * LP + j];
        }
    for (int q = warp; q < nb * 3; q += 16) {
        const int b = q / 3, h = q - b * 3;
        decode_heads(logit + b * LP, angles + (long long)(n0 + b) * 3, h, lane);
    }
}

// decode only (test hook whenet_debug_decode): logits [N][252] -> angles [N][3], the same device function as the head kernel
static __global__ void __launch_bounds__(96) decode_only_kernel(const float* __restrict__ logits, float* __restrict__ angles) {
    __shared__ float logit[252 + 4];
    const int n = blockIdx.x, tid = threadIdx.x;
    for (int j = tid; j < 252; j += 96) logit[j] = logits[(long long)n * 252 + j];
    __syncthreads();
    decode_heads(logit, angles + (long long)n * 3, tid >> 5, tid & 31);
}

// raises the context's timeout flag from the device (test hook: proves every synchronising path reports it)
static __global__ void raise_flag_kernel(int* flag) { *reinterpret_cast<volatile int*>(flag) = 1; }

// T -> float gather for debug taps: CTA row y copies crop map[y].x (relative to src) into tap row map[y].y
template <typename T>
__global__ void tap_gather_kernel(const T* __restrict__ src, float* __restrict__ dst, const int2* __restrict__ map, int base,
                                  long long per) {
    const int2 m = map[blockIdx.y];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < per) dst[(long long)m.y * per + i] = Store<T>::ld(src + (long long)(m.x - base) * per + i);
}

}  // namespace whenet
