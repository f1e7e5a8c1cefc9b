// kernels_stem_tc.cuh - the stem (conv 3x3 stride 2, 3 -> 32 channels, TF-SAME, BN, swish; reference whenet.py:8 ->
// efficientnet stem) on the tensor core, for uint8 input and 16-bit output.
//
// The CUDA-core stem (stem_tile_kernel) is bound by its 27 x 32 FMAs per output pixel: 0.15 ms per 512 crops at 100 % of the
// FMA pipe, 0.34 ms measured.  As a GEMM the stem is [pixels x 27] x [27 x 32] - far too thin for the tensor core to notice,
// and the im2col operand can be BUILT in shared memory for less than the FMAs cost:
//
//   A row (one output pixel) = 27 taps (ky, kx, ci); each tap = one byte of the staged input rows -> a 256-entry table per
//   channel that holds float32(((v/255) - mean)/std) (reference whenet.py:25-26, evaluated in float64 like numpy) already split
//   into a bf16 high part and a bf16 low part (hi + lo carries 16 mantissa bits: the bf16 rounding of the INPUT alone would cost
//   0.24 deg, SURVEY.md 8c) -> K = 64: [hi(27) 0(5) | lo(27) 0(5)] against W = [w | 0 | w | 0] (bf16 weights).
//   One warpgroup MMA block (128 pixels x 32 channels x K 64, four K steps) per output row; fp32 accumulators in registers.
//
// CTA = 128 threads = one output row at a time (112 pixels + 16 idle rows of the M = 128 tile), ROWS rows per CTA.  Thread p
// builds A row p for output row r+1 (27 byte loads, 27 table loads, 28 PRMT, 8 swizzled 16-byte stores) while the MMA of row r
// runs, then drains row r through the shared accumulator tile: h = acc/2 + b/2 -> MUFU.TANH -> FMA -> 16-bit -> four 16-byte
// stores (32 channels).
#pragma once
#include "kernels_fused.cuh"

namespace whenet {

struct StemTcGeom {
    static constexpr int ROWS = 8;                  // output rows per CTA (112 = 14 x 8)
    static constexpr int IN_ROWS = 2 * ROWS + 1;    // input rows staged per CTA
    static constexpr int ROW_BYTES = 224 * 3;       // one input row
    static constexpr int ROW_PITCH = 688;           // staged pitch (16-byte multiple, >= 672 + 3 for the pad pixel's bytes)
};

template <typename TOUT>
__global__ void __launch_bounds__(128) stem_tc_kernel(const uint8_t* __restrict__ in, TOUT* __restrict__ out,
                                                      const __grid_constant__ StemParams sp, const float* __restrict__ lut) {
    using G = StemTcGeom;
    constexpr int A_BYTES = 128 * 128;              // one A tile: 128 rows x 64 bf16, SWIZZLE_128B
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem0 = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem0;                                  // 2 x A tile
    const uint32_t sW = sA + 2 * A_BYTES;                       // [32 rows n][128 B]  (4 KB)
    const uint32_t sL = sW + 32 * 128;                          // table [3][256] u32 = hi | lo << 16
    const uint32_t sI = sL + 3 * 256 * 4;                       // staged input rows [IN_ROWS][ROW_PITCH] bytes
    const uint32_t sB = sI + G::IN_ROWS * G::ROW_PITCH;         // 32 floats: b/2
    const uint32_t sAcc = sB + 128;                             // shared accumulator tile, 32 columns
    const int tid = threadIdx.x;
    const int n = blockIdx.y, oy0 = blockIdx.x * G::ROWS;

    // ---- table: float -> bf16 hi | bf16 lo
    for (int i = tid; i < 768; i += 128) {
        const float f = lut[i];
        const __nv_bfloat16 hi = __float2bfloat16_rn(f), lo = __float2bfloat16_rn(f - __bfloat162float(hi));
        const uint32_t w = (uint32_t)__bfloat16_as_ushort(hi) | ((uint32_t)__bfloat16_as_ushort(lo) << 16);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sL + (uint32_t)i * 4u), "r"(w) : "memory");
    }
    // ---- W: row n = [w(k = 0..26)[n] | 0 x 5 | the same | 0 x 5] bf16, K-major, SWIZZLE_128B
    for (int i = tid; i < 32 * 8; i += 128) {
        const int r = i >> 3, c = i & 7;                        // row n, 16-byte chunk
        uint32_t pk[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k0 = (c & 3) * 8 + 2 * j, k1 = k0 + 1;    // tap index inside the 32-wide half
            const float w0 = k0 < 27 ? sp.w[k0 * 32 + r] : 0.f, w1 = k1 < 27 ? sp.w[k1 * 32 + r] : 0.f;
            pk[j] = fused::pack2<__nv_bfloat16>(w0, w1);
        }
        fused::sts128(sW + (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4)), make_uint4(pk[0], pk[1], pk[2], pk[3]));
    }
    if (tid < 32) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sB + (uint32_t)tid * 4u), "f"(0.5f * sp.b[tid]) : "memory");
    // ---- input rows 2*oy0 .. 2*oy0 + 2*ROWS (row 224 does not exist: its taps are masked below)
    {
        const uint8_t* src = in + (long long)n * 224 * G::ROW_BYTES;
        for (int v = tid; v < G::IN_ROWS * 42; v += 128) {      // 42 x 16 bytes per row
            const int r = v / 42, q = v - r * 42;
            const int iy = 2 * oy0 + r;
            fused::cp_async16(sI + (uint32_t)(r * G::ROW_PITCH + q * 16), src + (long long)min(iy, 223) * G::ROW_BYTES + q * 16, iy < 224);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();

    const int ox = tid;                                         // pixel of the row = A row = accumulator row
    const bool px_ok = ox < 112;
    // one A row: 27 taps -> table -> hi chunks 0..3, lo chunks 4..7
    auto build = [&](int rl, int buf) {                          // rl = output row inside the CTA
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) { hi[j] = 0u; lo[j] = 0u; }
        if (px_ok) {
            const int oy = oy0 + rl;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const bool row_ok = 2 * oy + ky < 224;
                const uint32_t rb = sI + (uint32_t)((2 * rl + ky) * G::ROW_PITCH + 6 * ox);
#pragma unroll
                for (int t = 0; t < 9; ++t) {                   // kx * 3 + ci
                    const int k = ky * 9 + t;
                    uint32_t b, w = 0u;
                    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(b) : "r"(rb + (uint32_t)t));
                    const bool ok = row_ok && (t < 6 || ox < 111);                      // column 224 does not exist either
                    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(sL + (uint32_t)(((t % 3) * 256) * 4) + b * 4u));
                    w = ok ? w : 0u;
                    // even taps fill the low half-word of their pair, odd taps the high one
                    if ((k & 1) == 0) { hi[k >> 1] = w & 0xffffu; lo[k >> 1] = w >> 16; }
                    else { hi[k >> 1] |= w << 16; lo[k >> 1] |= w & 0xffff0000u; }
                }
            }
        }
        const uint32_t a0 = sA + buf * A_BYTES + (uint32_t)((ox >> 3) * 1024 + (ox & 7) * 128);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            fused::sts128(a0 + (uint32_t)(((c) ^ (ox & 7)) << 4), make_uint4(hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]));
            fused::sts128(a0 + (uint32_t)(((c + 4) ^ (ox & 7)) << 4), make_uint4(lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]));
        }
    };
    auto drain = [&](int rl) {
        TOUT* dst = out + (((long long)n * 112 + oy0 + rl) * 112 + ox) * 32;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            float v[16];
            tc::acc_ld16(sAcc, ox, u * 16, v);
            uint32_t pk[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 bq = fused::lds_f4(sB + (uint32_t)(u * 16 + j * 4) * 4u);
                const float h0 = swish_from_half(fmaf(v[4 * j], 0.5f, bq.x)), h1 = swish_from_half(fmaf(v[4 * j + 1], 0.5f, bq.y));
                const float h2 = swish_from_half(fmaf(v[4 * j + 2], 0.5f, bq.z)), h3 = swish_from_half(fmaf(v[4 * j + 3], 0.5f, bq.w));
                pk[2 * j] = fused::pack2<TOUT>(h0, h1);
                pk[2 * j + 1] = fused::pack2<TOUT>(h2, h3);
            }
            if (px_ok) {
                *reinterpret_cast<uint4*>(dst + u * 16) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                *reinterpret_cast<uint4*>(dst + u * 16 + 8) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            }
        }
    };

    tc::WgAcc<32> acc;
    build(0, 0);
    for (int rl = 0; rl < G::ROWS; ++rl) {
        const int buf = rl & 1;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();                            // A(rl) complete; row rl-1 drained out of the accumulator tile
        tc::wg_mma_tile<true, 32>(acc, sA + buf * A_BYTES, sW, 4, 0u);
        if (rl + 1 < G::ROWS) build(rl + 1, buf ^ 1);           // A[buf^1]: its MMA (row rl-1) completed last iteration
        tc::wg_wait<0>();
        tc::wg_acc_store<32>(acc, sAcc, tid);
        __syncthreads();
        drain(rl);
    }
}

constexpr size_t stem_tc_smem() {
    return (size_t)2 * 128 * 128 + 32 * 128 + 3 * 256 * 4 + (size_t)StemTcGeom::IN_ROWS * StemTcGeom::ROW_PITCH + 128 + tc::acc_tile_bytes(32) + 1024;
}

template <typename TOUT>
int launch_stem_tc(cudaStream_t stream, const uint8_t* in, TOUT* out, const StemParams& sp, const float* lut, int n_crops) {
    auto kfn = stem_tc_kernel<TOUT>;
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stem_tc_smem()) != cudaSuccess) return -1;
    kfn<<<dim3(112 / StemTcGeom::ROWS, n_crops), 128, stem_tc_smem(), stream>>>(in, out, sp, lut);
    return 0;
}

}  // namespace whenet
