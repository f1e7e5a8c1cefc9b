// kernels_tc32.cuh - the 1x1 convolutions of the fp32 PARITY mode on the tensor core (option "tensor_cores" = 1 in fp32):
//
//   out[m, n] = act( bias[n] + sum_k (A[m,k] * gate[m/hw, k]) * W[k,n] ) (+ resid[m,n])      A, out, resid: fp32 in HBM
//
// The tensor core has no fp32 x fp32 MMA; tf32 keeps 10 mantissa bits (0.034 deg on the Sample crops, SURVEY.md 8c - over the
// 0.01 deg target).  Here every fp32 operand is split into two bf16 terms, x = hi + lo with hi = bf16(x), lo = bf16(x - hi)
// (|x - hi - lo| <= 2^-18 |x|), and the product is three bf16 MMAs accumulated in fp32 registers:
//
//   A*W ~= Ahi*Whi + Ahi*Wlo + Alo*Whi          (the dropped Alo*Wlo term and the split residuals are ~2^-17 relative)
//
// The weights are split once at load time (two K-major [N][K] bf16 arrays); activations are split on the fly by the threads
// that stage them: global fp32 -> registers -> (x SE gate, in fp32) -> hi / lo -> two SWIZZLE_128B tiles in shared memory.
// One 128-thread CTA owns a 128-pixel x n_tile tile; K runs in blocks of 64 channels through a 2-stage ring whose stages are
// recycled once wgmma.wait_group reports the block that read them complete; the epilogue is fp32 throughout (precise expf swish, as the CUDA-core parity kernels).
#pragma once
#include "kernels_tc.cuh"

namespace whenet {
namespace tc {

// UN = pw_mma_width(n_tile): rows of the W stages, MMA width
template <bool SWISH, bool GATE, bool RESID, int UN>
__global__ void __launch_bounds__(128) pw_tc32_kernel(const float* __restrict__ A, const __nv_bfloat16* __restrict__ Whi,
                                                      const __nv_bfloat16* __restrict__ Wlo, const float* __restrict__ bias,
                                                      const float* __restrict__ gate, const float* __restrict__ resid,
                                                      float* __restrict__ out, int M, int K, int N, int hw,
                                                      int n_tile) {
    extern __shared__ uint8_t smem_raw[];

    const int tid = threadIdx.x;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr uint32_t w_bytes = (uint32_t)UN * 128;
    const uint32_t stage_bytes = 2 * A_STAGE_BYTES + 2 * w_bytes;      // A hi | A lo | W hi | W lo

    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * n_tile;
    const int rows_valid = min(BM, M - m0), n_valid = min(n_tile, N - n0);
    const int nkb = (K + BK - 1) / BK, kchunks = K >> 3;

    WgAcc<UN> acc;

    // this thread stages chunk c (8 channels) of rows r0 + 16 i: its gate row index per row is fixed for the whole K loop
    const int c = tid & 7, r0 = tid >> 3;
    const uint32_t swz = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));

    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb & 1;
        if (kb >= 2) {              // the MMAs of block kb-2 are done with this stage (in every thread): block kb-1's three groups may be pending
            wg_wait<3>();
            __syncthreads();
        }
        const uint32_t a_hi = smem0 + s * stage_bytes, a_lo = a_hi + A_STAGE_BYTES, w_hi = a_lo + A_STAGE_BYTES, w_lo = w_hi + w_bytes;
        const int kc = kb * 8 + c;                        // global 16-byte (8-channel) chunk of this thread
        const bool cvalid = kc < kchunks;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = r0 + 16 * i;
            uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
            if (cvalid && r < rows_valid) {
                const float* src = A + (long long)(m0 + r) * K + kc * 8;
                const float4 v0 = *reinterpret_cast<const float4*>(src), v1 = *reinterpret_cast<const float4*>(src + 4);
                float x[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                if (GATE) {
                    const float* g = gate + (long long)((m0 + r) / hw) * K + kc * 8;
                    const float4 g0 = __ldg(reinterpret_cast<const float4*>(g)), g1 = __ldg(reinterpret_cast<const float4*>(g + 4));
                    x[0] *= g0.x; x[1] *= g0.y; x[2] *= g0.z; x[3] *= g0.w; x[4] *= g1.x; x[5] *= g1.y; x[6] *= g1.z; x[7] *= g1.w;
                }
                split8(x, hi, lo);
            }
            sts128_(a_hi + swz + i * 2048, hi);
            sts128_(a_lo + swz + i * 2048, lo);
        }
#pragma unroll
        for (int i = 0; i < UN / 16; ++i) {
            const int r = r0 + 16 * i;
            uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
            if (cvalid && r < n_valid) {
                hi = __ldg(reinterpret_cast<const uint4*>(Whi + (long long)(n0 + r) * K + kc * 8));
                lo = __ldg(reinterpret_cast<const uint4*>(Wlo + (long long)(n0 + r) * K + kc * 8));
            }
            sts128_(w_hi + swz + i * 2048, hi);
            sts128_(w_lo + swz + i * 2048, lo);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        const int ksteps = (min(BK, K - kb * BK) + 15) >> 4;
        wg_mma_tile<true, UN>(acc, a_hi, w_hi, ksteps, kb ? 1u : 0u);      // one commit group each
        wg_mma_tile<true, UN>(acc, a_hi, w_lo, ksteps, 1u);
        wg_mma_tile<true, UN>(acc, a_lo, w_hi, ksteps, 1u);
    }
    wg_wait<0>();
    __syncthreads();
    // the operand stages are free: accumulators -> shared accumulator tile
    const uint32_t sAcc = smem0;
    wg_acc_store<UN>(acc, sAcc, tid);
    __syncthreads();

    // ---- epilogue, fp32: thread == pixel row; + shift, swish (precise), + residual; 16-byte stores
    const bool row_ok = tid < rows_valid;
    const long long m = (long long)m0 + tid;
    {
        for (int c0 = 0; c0 < n_valid; c0 += 16) {
            float v[16];
            acc_ld16(sAcc, tid, c0, v);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int n = n0 + c0 + q * 4;
                if (c0 + q * 4 >= n_valid) break;
                const float4 b = __ldg(reinterpret_cast<const float4*>(bias + n));
                float o[4] = {v[q * 4] + b.x, v[q * 4 + 1] + b.y, v[q * 4 + 2] + b.z, v[q * 4 + 3] + b.w};
                if (SWISH) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) o[j] = swish_f(o[j]);
                }
                if (row_ok) {
                    if (RESID) {
                        const float4 r = *reinterpret_cast<const float4*>(resid + m * N + n);
                        o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
                    }
                    *reinterpret_cast<float4*>(out + m * N + n) = make_float4(o[0], o[1], o[2], o[3]);
                }
            }
        }
    }
}

// 0 = launched, > 0 = shape unsupported (caller falls back to the CUDA-core kernel), < 0 = error
inline int launch_pw_tc32(cudaStream_t stream, const float* A, const void* Whi, const void* Wlo, const float* bias, const float* gate,
                          const float* resid, float* out, long long M, int K, int N, int hw, bool swish) {
    if ((K & 7) || (N & 7) || M > 0x7fffffffLL || !Whi || !Wlo) return 1;
    int n_tile = N;
    if (N > 128) {
        int parts = (N + 127) / 128;
        while (true) {
            n_tile = ((N + parts - 1) / parts + 15) & ~15;
            if (n_tile <= 128) break;
            ++parts;
        }
    }
    const int umma_n = pw_mma_width(n_tile);
    const size_t smem = std::max((size_t)2 * (2 * A_STAGE_BYTES + 2 * (size_t)umma_n * 128), (size_t)acc_tile_bytes(umma_n)) + 1024;
    dim3 grid((unsigned)((N + n_tile - 1) / n_tile), (unsigned)((M + BM - 1) / BM));
    const __nv_bfloat16 *wh = reinterpret_cast<const __nv_bfloat16*>(Whi), *wl = reinterpret_cast<const __nv_bfloat16*>(Wlo);
#define TC32(SW, GA, RE)                                                                                                   \
    return with_mma_width<128>(umma_n, [&](auto un) {                                                                      \
        auto kfn = pw_tc32_kernel<SW, GA, RE, decltype(un)::value>;                                                        \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) return -1;  \
        kfn<<<grid, 128, smem, stream>>>(A, wh, wl, bias, gate, resid, out, (int)M, K, N, hw, n_tile);                     \
        return 0;                                                                                                          \
    })
    if (swish && !gate && !resid) TC32(true, false, false);
    if (!swish && gate && !resid) TC32(false, true, false);
    if (!swish && gate && resid) TC32(false, true, true);
    if (!swish && !gate && !resid) TC32(false, false, false);
    if (!swish && !gate && resid) TC32(false, false, true);
#undef TC32
    return 1;
}

}  // namespace tc
}  // namespace whenet
