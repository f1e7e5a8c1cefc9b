// kernels_yolo32.cuh - the YOLOv3 / tiny YOLOv3 detector's fp32 PARITY mode (whenet_det_create_ex(.., WHENET_PRECISION_FP32)).
//
//   yolo_conv0_32_kernel<N>                    first conv, fp32 output: the v/255 table's bf16 hi + lo parts as the A row
//                                              [hi | lo | hi] against the B row [w_hi | w_hi | w_lo] (K = 96)
//   conv_igemm32_kernel<MODE, UN>              every other conv: conv_igemm_kernel's tiling (128 pixels x UN columns per CTA, K
//                                              blocks of (tap, 64-channel chunk), zero-filled out-of-image taps, virtual concat)
//                                              on fp32 activations, split into bf16 hi + lo as they are staged, and three MMAs
//                                              per K block, Ahi*Whi + Ahi*Wlo + Alo*Whi, into one fp32 accumulator
//   yolo_maxpool32_kernel                      tiny YOLOv3's 2x2 max-pools on fp32 (exact)
//
// Activations fp32 in HBM, weights split once on the host (hi = bf16(w), lo = bf16(w - hi), two K-major [N][K] arrays), the
// epilogue fp32 throughout.  The split is pw_tc32_kernel's (tc::split8): each product loses at most about 3 * 2^-18 of its
// magnitude (two split residuals and the dropped Alo*Wlo term), below the fp32 accumulation error of a K ~ 1000 sum.
//
// The device code is left out under WHENET_YOLO32_HOST_ONLY (the host side); inst_yolo32.cu includes kernels_yolo.cuh for its
// declarations only (WHENET_YOLO_HOST_ONLY), since the bf16 kernels are compiled in inst_yolo.cu.
#pragma once
#include "kernels_yolo.cuh"

namespace whenet {
namespace yolo {

struct Igemm32Params {
    const float* in;             // [n][Hi][Wi][Cin - c_up]  (concat: the skip tensor)
    const float* up;             // concat: [n][Hi/2][Wi/2][c_up], read at (y >> 1, x >> 1)
    const __nv_bfloat16* w_hi;   // [N][K] bf16(w), K = k*k*Cin, k index = (ky*k + kx)*Cin + ci
    const __nv_bfloat16* w_lo;   // [N][K] bf16(w - hi)
    const float* bias;           // [N]
    const float* resid;          // [M][N]
    float* out;                  // [M][N]
    int M, Hi, Wi, Ho, Wo, Cin, c_up, N, k, stride, n_tile, n_stages;
};

constexpr size_t kSmemPerSm = 228 * 1024;   // shared memory of one H100 SM; 1 KB of it is reserved per resident CTA
constexpr size_t kSmemOptin = 227 * 1024;   // dynamic shared memory one CTA may opt in to

// Tile plan of one fp32 conv: plan_igemm's tile (so it too depends on the per-frame shape only, and a frame's results are the
// same bits in any batch).  A stage holds two A planes (hi, lo) and two W planes, twice the bf16 stage; the ring is as deep as
// fits (at most 4) two CTAs per SM, or one CTA per SM where two stages do not fit two CTAs (the 128-wide tiles).
struct Igemm32Plan { int n_tile, un, n_stages, ctas_per_sm; size_t smem; };
inline size_t igemm32_stage_bytes(int un) { return 2 * (size_t)tc::A_STAGE_BYTES + 2 * (size_t)un * BK * 2; }
inline Igemm32Plan plan_igemm32(int Ho, int Wo, int N, int Cin, int k, int sm_count) {
    const IgemmPlan b = plan_igemm(Ho, Wo, N, Cin, k, sm_count);
    Igemm32Plan pl{b.n_tile, b.un, 0, 0, 0};
    const int nkb = k * k * ((Cin + BK - 1) / BK);
    const size_t stage = igemm32_stage_bytes(pl.un);
    for (int ctas = 2; ctas >= 1; --ctas) {
        const size_t cap = std::min(kSmemOptin, kSmemPerSm / ctas - 1024) - 1024;     // - the 1 KB alignment slack
        const int st = (int)std::min<size_t>(4, cap / stage);
        if (st < 2) continue;
        pl.ctas_per_sm = ctas;
        pl.n_stages = nkb < st ? (nkb < 2 ? 2 : nkb) : st;
        break;
    }
    pl.smem = std::max((size_t)pl.n_stages * stage, (size_t)tc::acc_tile_bytes(pl.un)) + 1024;
    return pl;
}

// launchers (inst_yolo32.cu); each returns 0 or the CUDA error of the launch
int launch_conv0_32(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, const float* bias, float* out,
                    int n, int S_h, int S_w, int cout);
int launch_igemm32(cudaStream_t s, const Igemm32Params& p, int mode, int un, size_t smem, int grid_n, int grid_m);
int launch_maxpool32(cudaStream_t s, const float* in, float* out, int n, int H, int W, int C, int stride);

#ifndef WHENET_YOLO32_HOST_ONLY
__device__ __forceinline__ float leaky32(float x) { return x > 0.f ? x : 0.1f * x; }

// ----------------------------------------------------------------------------- first conv
// yolo_conv0_kernel's A tile (K 0..26 the taps' bf16 hi parts, K 32..58 their lo parts) once more against two B tiles: W0 = the
// bf16 kernel's [w_hi | 0 | w_hi | 0] rows (4 K steps: hi*w_hi + lo*w_hi), W1 = [w_lo | 0] (2 K steps over the hi half: hi*w_lo).
// Bias, LeakyReLU and the stores in fp32.
template <int N>
__global__ void __launch_bounds__(128) yolo_conv0_32_kernel(const uint8_t* __restrict__ img, const __nv_bfloat16* __restrict__ w_hi,
                                                            const __nv_bfloat16* __restrict__ w_lo, const float* __restrict__ bias,
                                                            float* __restrict__ out, int S_h, int S_w) {
    static_assert(N == 16 || N == 32, "first conv: 16 or 32 outputs");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem0;                      // 128 rows x 128 B
    const uint32_t sW = sA + 128 * 128;             // N rows x 128 B: [w_hi | w_hi]
    const uint32_t sWl = sW + N * 128;              // N rows x 128 B: [w_lo | 0]
    const uint32_t sL = sWl + N * 128;              // 256 x u32 (hi | lo << 16)
    const uint32_t sAcc = sL + 256 * 4;             // accumulator tile, N columns
    const int tid = threadIdx.x;
    for (int i = tid; i < 256; i += 128) {
        const float f = (float)i / 255.0f;          // float32(v / 255.), as np.array(.., 'float32') / 255. (yolo_postprocess.py:191-195)
        const __nv_bfloat16 hi = __float2bfloat16_rn(f), lo = __float2bfloat16_rn(f - __bfloat162float(hi));
        const uint32_t w = (uint32_t)__bfloat16_as_ushort(hi) | ((uint32_t)__bfloat16_as_ushort(lo) << 16);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sL + (uint32_t)i * 4u), "r"(w) : "memory");
    }
    for (int i = tid; i < N * 8; i += 128) {
        const int r = i >> 3, c = i & 7;
        const uint32_t off = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
        tc::sts128_(sW + off, *reinterpret_cast<const uint4*>(w_hi + r * 64 + c * 8));
        tc::sts128_(sWl + off, *reinterpret_cast<const uint4*>(w_lo + r * 64 + c * 8));
    }
    __syncthreads();
    const long long m = (long long)blockIdx.x * 128 + tid;
    const int hw = S_h * S_w;
    const int f = (int)(m / hw), p = (int)(m - (long long)f * hw);
    const int y = p / S_w, x = p - y * S_w;
    uint32_t hi[16], lo[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { hi[j] = 0u; lo[j] = 0u; }
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int iy = y + ky - 1, ix = x + kx - 1;
            const bool ok = iy >= 0 && iy < S_h && ix >= 0 && ix < S_w;
            const uint8_t* src = img + (((long long)f * S_h + (ok ? iy : 0)) * S_w + (ok ? ix : 0)) * 3;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                const int k = (ky * 3 + kx) * 3 + ci;
                uint32_t w;
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(sL + (uint32_t)src[ci] * 4u));
                w = ok ? w : 0u;
                if ((k & 1) == 0) { hi[k >> 1] = w & 0xffffu; lo[k >> 1] = w >> 16; }
                else { hi[k >> 1] |= w << 16; lo[k >> 1] |= w & 0xffff0000u; }
            }
        }
    const uint32_t a0 = sA + (uint32_t)((tid >> 3) * 1024 + (tid & 7) * 128);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        tc::sts128_(a0 + (uint32_t)((c ^ (tid & 7)) << 4), make_uint4(hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]));
        tc::sts128_(a0 + (uint32_t)(((c + 4) ^ (tid & 7)) << 4), make_uint4(lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tc::WgAcc<N> acc;
    tc::wg_mma_tile<true, N>(acc, sA, sW, 4, 0u);
    tc::wg_mma_tile<true, N>(acc, sA, sWl, 2, 1u);
    tc::wg_wait<0>();
    tc::wg_acc_store<N>(acc, sAcc, tid);
    __syncthreads();
    float* dst = out + m * N;
#pragma unroll
    for (int u = 0; u < N / 16; ++u) {
        float v[16];
        tc::acc_ld16(sAcc, tid, u * 16, v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float4 b = *reinterpret_cast<const float4*>(bias + u * 16 + q * 4);
            *reinterpret_cast<float4*>(dst + u * 16 + q * 4) =
                make_float4(leaky32(v[q * 4] + b.x), leaky32(v[q * 4 + 1] + b.y), leaky32(v[q * 4 + 2] + b.z), leaky32(v[q * 4 + 3] + b.w));
        }
    }
}

// ----------------------------------------------------------------------------- implicit-GEMM conv, fp32 in and out
// One 128-pixel x UN-column output tile per CTA; K blocks = (tap, 64-channel chunk) through an n_stages ring.  A stage is
// A hi | A lo | W hi | W lo.  The W planes arrive by cp.async; the A rows are loaded into registers, split into hi and lo and
// stored by the thread that loaded them.  Block kb + n_stages - 1 is staged while block kb's MMAs run, into the stage block
// kb - 1 read (its three commit groups are complete once wgmma.wait_group 3 returns).
template <int MODE, int UN>
__global__ void __launch_bounds__(128) conv_igemm32_kernel(const __grid_constant__ Igemm32Params p) {
    extern __shared__ uint8_t smem_raw[];
    const int tid = threadIdx.x;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr uint32_t w_plane = UN * BK * 2;
    constexpr uint32_t stage_bytes = 2 * tc::A_STAGE_BYTES + 2 * w_plane;
    const int m0 = blockIdx.y * BM;
    const int n0 = blockIdx.x * p.n_tile;
    const int n_valid = min(p.n_tile, p.N - n0);
    const int cchunks = (p.Cin + BK - 1) / BK;
    const int nkb = p.k * p.k * cchunks;
    const int K = p.k * p.k * p.Cin;
    const int pad = p.k >> 1;
    const int hw = p.Ho * p.Wo;

    // this thread's 8 A rows (r0 + 16 i) and its 8-channel chunk c: frame row base and top-left input coordinate
    const int c = tid & 7, r0 = tid >> 3;
    int rbase[8], iy0[8], ix0[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + r0 + 16 * i;
        if (m < p.M) {
            const int f = m / hw, q = m - f * hw;
            const int oy = q / p.Wo, ox = q - oy * p.Wo;
            rbase[i] = f * p.Hi;
            iy0[i] = oy * p.stride - pad;
            ix0[i] = ox * p.stride - pad;
        } else {
            rbase[i] = 0;
            iy0[i] = -(1 << 20);
            ix0[i] = 0;
        }
    }
    const uint32_t swz = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));

    auto fill = [&](int kb) {
        const int s = kb % p.n_stages;
        const uint32_t a_hi = smem0 + s * stage_bytes, a_lo = a_hi + tc::A_STAGE_BYTES;
        const uint32_t w_hi = a_lo + tc::A_STAGE_BYTES, w_lo = w_hi + w_plane;
        const int tap = kb / cchunks, cc = kb - tap * cchunks;
        const int ky = tap / p.k, kx = tap - ky * p.k;
        const int c0 = cc * BK;
        const bool cvalid = c0 + c * 8 < p.Cin;
        const __nv_bfloat16* wsrc_hi = p.w_hi + (long long)(n0 + r0) * K + tap * p.Cin + c0 + c * 8;
        const __nv_bfloat16* wsrc_lo = p.w_lo + (long long)(n0 + r0) * K + tap * p.Cin + c0 + c * 8;
#pragma unroll
        for (int i = 0; i < UN / 16; ++i) {
            const bool valid = cvalid && r0 + 16 * i < n_valid;
            cp_async16_z(w_hi + swz + i * 2048, valid ? wsrc_hi + (long long)i * 16 * K : p.w_hi, valid);
            cp_async16_z(w_lo + swz + i * 2048, valid ? wsrc_lo + (long long)i * 16 * K : p.w_lo, valid);
        }
        // source of this chunk: the skip tensor, or (concat, c0 < c_up) the low-resolution tensor at half the coordinates
        const bool from_up = MODE == kLeakyCat && c0 < p.c_up;
        const float* src = from_up ? p.up : p.in;
        const int cs = from_up ? p.c_up : p.Cin - p.c_up;
        const int sh = from_up ? 1 : 0;
        const int Ws = p.Wi >> sh;
        const int ch = (from_up ? c0 : c0 - p.c_up) + c * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int iy = iy0[i] + ky, ix = ix0[i] + kx;
            uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
            if (cvalid && iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi) {
                const float* a = src + ((long long)((rbase[i] + iy) >> sh) * Ws + (ix >> sh)) * cs + ch;
                const float4 v0 = __ldg(reinterpret_cast<const float4*>(a)), v1 = __ldg(reinterpret_cast<const float4*>(a + 4));
                const float x[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                tc::split8(x, hi, lo);
            }
            tc::sts128_(a_hi + swz + i * 2048, hi);
            tc::sts128_(a_lo + swz + i * 2048, lo);
        }
    };
    for (int j = 0; j + 1 < p.n_stages; ++j) {
        if (j < nkb) fill(j);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    tc::WgAcc<UN> acc;
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % p.n_stages;
        const uint32_t a_hi = smem0 + s * stage_bytes, a_lo = a_hi + tc::A_STAGE_BYTES;
        const uint32_t w_hi = a_lo + tc::A_STAGE_BYTES, w_lo = w_hi + w_plane;
        // block kb's W copies: n_stages - 1 + kb groups are committed, those of the n_stages - 2 blocks after kb may be pending
        if (p.n_stages >= 4) asm volatile("cp.async.wait_group 2;" ::: "memory");
        else if (p.n_stages == 3) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        {
            const int cc = kb % cchunks;
            const int ks = (min(BK, p.Cin - cc * BK) + 15) >> 4;
            tc::wg_mma_tile<true, UN>(acc, a_hi, w_hi, ks, kb ? 1u : 0u);      // one commit group each
            tc::wg_mma_tile<true, UN>(acc, a_hi, w_lo, ks, 1u);
            tc::wg_mma_tile<true, UN>(acc, a_lo, w_hi, ks, 1u);
        }
        if (kb + p.n_stages - 1 < nkb) {
            if (kb >= 1) {
                tc::wg_wait<3>();
                __syncthreads();
            }
            fill(kb + p.n_stages - 1);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    tc::wg_wait<0>();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const uint32_t sAcc = smem0;
    tc::wg_acc_store<UN>(acc, sAcc, tid);
    __syncthreads();

    const bool row_ok = tid < min(BM, p.M - m0);
    const long long m = (long long)m0 + tid;
    if (MODE == kLinearF32) {      // output convs: bias, no activation (any N)
        if (row_ok)
            for (int j = 0; j < n_valid; ++j) {
                float v;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(sAcc + (uint32_t)(j * tc::kAccPitch + tid) * 4u));
                p.out[m * p.N + n0 + j] = v + p.bias[n0 + j];
            }
        return;
    }
    if (!row_ok) return;
    for (int c0 = 0; c0 < n_valid; c0 += 16) {
        float v[16];
        tc::acc_ld16(sAcc, tid, c0, v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (c0 + q * 4 >= n_valid) break;
            const int n = n0 + c0 + q * 4;
            const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n));
            float o[4] = {leaky32(v[q * 4] + b.x), leaky32(v[q * 4 + 1] + b.y), leaky32(v[q * 4 + 2] + b.z), leaky32(v[q * 4 + 3] + b.w)};
            if (MODE == kLeakyRes) {
                const float4 r = *reinterpret_cast<const float4*>(p.resid + m * p.N + n);
                o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
            }
            *reinterpret_cast<float4*>(p.out + m * p.N + n) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
}

// ----------------------------------------------------------------------------- max-pool (tiny YOLOv3), fp32
// yolo_maxpool_kernel's TF SAME window on fp32: one thread per 4-channel chunk of an output pixel, C % 4 == 0.  A max is one of
// its inputs, so the pool is exact.
__global__ void __launch_bounds__(256) yolo_maxpool32_kernel(const float* __restrict__ in, float* __restrict__ out, int n, int H, int W,
                                                             int C, int stride) {
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride, cc = C >> 2;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n * Ho * Wo * cc) return;
    const int c = (int)(i % cc);
    const long long px = i / cc;
    const int ox = (int)(px % Wo);
    const long long fy = px / Wo;
    const int oy = (int)(fy % Ho), f = (int)(fy / Ho);
    const int y0 = oy * stride, x0 = ox * stride;
    const bool y1 = y0 + 1 < H, x1 = x0 + 1 < W;
    const float4* src = reinterpret_cast<const float4*>(in + (((long long)f * H + y0) * W + x0) * C) + c;
    const long long row = (long long)W * cc;            // float4s per input row
    float4 v = src[0];
    auto mx = [](float4& a, float4 b) { a.x = fmaxf(a.x, b.x); a.y = fmaxf(a.y, b.y); a.z = fmaxf(a.z, b.z); a.w = fmaxf(a.w, b.w); };
    if (x1) mx(v, src[cc]);
    if (y1) mx(v, src[row]);
    if (x1 && y1) mx(v, src[row + cc]);
    reinterpret_cast<float4*>(out)[i] = v;
}
#endif  // WHENET_YOLO32_HOST_ONLY

}  // namespace yolo
}  // namespace whenet
