// kernels_dwse.cuh - KD: depthwise KSxKS + BN shift + swish + squeeze + excite (+ gating of its own output) for the blocks
// whose feature map is small enough that ONE CTA holds a whole crop (14x14 and 7x7, blocks 7-16).
//
// Why a second route next to K1 for these blocks: K1 tiles the map, stages its expand operands with cp.async and pays for
// that with a chain of CTA-wide phases per channel chunk; here one CTA owns a whole crop and every thread runs identical
// depthwise work:
//
//   CTA = one crop; for each chunk of CC channels (two buffers):
//       E tile [PW][PW][CC] fp16 in shared memory, its out-of-image border zero = TF-SAME padding
//       thread = (strip of 7 output pixels of one row, 4 channels): HFMA2 running sums over the fp16 tile, fp16 weights / 4
//       -> fp32: sum * 4 + shift, swish, squeeze partial sums (fixed order), 16-bit store of D
//   tail: channel means -> FC + swish -> FC + sigmoid -> gate (same device function as se_gate_kernel, same bits);
//         the CTA then rescales its own D (still in L2) so that the project conv runs ungated.
//
// Two kernels fill the E tiles:
//   dwse_x_kernel (one CTA per crop with all its chunks: throughput batches) computes the expand conv itself.  The crop's
//       block input X [H*W][Cin] is loaded once by TMA (K-major SWIZZLE_128B, 64-channel K blocks); per chunk, the W slice
//       [CC][Cin] comes by TMA, wgmma runs over the resident X and the epilogue writes swish(acc + bias) as fp16 straight
//       from the fragments into the tile.  The MMAs of chunk i+1 run while the CUDA cores do chunk i's depthwise.  E never
//       leaves the SM: at 512 crops the late blocks' E tensors are 29..135 MB, far more than the H100's 50 MB L2, so
//       writing them out meant a round trip through HBM.
//   dwse_kernel (small batches, where a crop's chunks are spread over several CTAs to fill the GPU) reads E, written by the
//       expand GEMM (pw_tc2, fp16 output), one tile per chunk by ONE cp.async.bulk.tensor.4d whose box starts at
//       (-pad, -pad): the TMA unit zero-fills the border.
//
// Both compute an E element with the expand GEMM's arithmetic (same wgmma K steps, h = acc/2 + b/2, swish_from_half, fp16),
// so the two routes give the same bits.  The arithmetic of one depthwise output is exactly K1's (fp16 E, HFMA2 taps in the
// same order, fp32 epilogue), so KD and K1 agree to the rounding of the expand accumulators (K1 carries the BN shift through
// the tensor core as a bf16 hi/lo pair, the GEMM adds it in fp32).
#pragma once
#include <cuda.h>

#include "kernels_fused.cuh"

namespace whenet {
namespace fused {

struct alignas(64) DwSeParams {
    CUtensorMap tmE;        // E [N][HIN][HIN][C] fp16 (expand conv + BN + swish): dims (C, W, H, N), box (CC, PW, PW, 1), no swizzle
    CUtensorMap tmW;        // w16 [KS*KS][C] fp16 = 0.5 * BN-folded depthwise weights / kDwScale: dims (C, KS*KS), box (CC, KS*KS)
    CUtensorMap tmX;        // dwse_x: block input [N*H*W][Cin] bf16, box {64, XROWS}, SWIZZLE_128B
    CUtensorMap tmWx;       // dwse_x: expand weights [C][Cin] bf16 (K-major), box {64, CC}, SWIZZLE_128B
    const float* b_exp;     // dwse_x: [C] expand BN shift
    const float* b_dw;      // [C]         0.5 * BN shift
    int* tflag;             // the context's mbarrier-timeout flag
    void* out;              // T [N][Ho][Ho][C]
    float* partial;         // [N][1][C]   squeeze sums (tiles = 1)
    const float *w_se1t, *b_se1, *w_se2, *b_se2;
    float* gate;            // [N][C]
    int Cse;
    float inv_hw;
    int se_tail;            // 1: this CTA sees every channel of its crop -> computes the gate itself
    int scale_out;          // se_tail only: D *= gate in place
    int C, pad;             // channels, TF-SAME pad_before
    int n_chunks, chunks_per_cta;
    int N;
    int tiles_x, Ho_img;    // SPATIAL only: tiles per image row, output image size
};

template <int KS, int S, int HIN>
struct DwSeGeom {
    static constexpr int HO = (HIN + S - 1) / S;
    static constexpr int R = 7;                                // outputs per strip (HO is 14 or 7)
    static constexpr int SPR = HO / R;                         // strips per output row
    static constexpr int NSTRIPS = HO * SPR;
    static constexpr int PW = (HO - 1) * S + KS;               // padded tile width
    static constexpr int NCOL = (R - 1) * S + KS;
};

template <int KS, int S, int HIN, int CC>
struct DwSeThreads { static constexpr int value = ((DwSeGeom<KS, S, HIN>::NSTRIPS * (CC / 4)) + 31) / 32 * 32; };

template <int KS, int S, int HIN, int CC>
constexpr size_t dwse_smem(int C, int Cse) {
    using G = DwSeGeom<KS, S, HIN>;
    return (size_t)2 * ((G::PW * G::PW * CC * 2 + 127) / 128 * 128)                  // two tiles
           + (size_t)2 * ((CC * 4 + KS * KS * CC * 2 + 127) / 128 * 128)             // two constant sets
           + (size_t)2 * G::NSTRIPS * CC * 4                                          // two squeeze scratch sets
           + (size_t)(C + Cse + 32) * 4 + 256;
}

// Depthwise of one strip (7 outputs of one row, 4 channels) of one chunk: `erow` = top-left of the strip's input window in
// the E tile, `cst` = the chunk's constants (CC fp32 shifts | [KS*KS][CC] fp16 weights), `dst` = its first output in D (pixels
// C apart).  The strip's four squeeze partial sums go to shared memory at `red`.
template <typename T, int KS, int S, int HIN, int CC>
__device__ __forceinline__ void dw_strip(uint32_t erow, uint32_t cst, int cv, T* dst, int C, uint32_t red) {
    using G = DwSeGeom<KS, S, HIN>;
    constexpr int PITCH = CC * 2;
    const float4 bq = lds_f4(cst + (uint32_t)cv * 16);
    const uint32_t cst_h = cst + (uint32_t)(CC * 4 + cv * 8);
    __half2 hacc[G::R][2];
#pragma unroll
    for (int r = 0; r < G::R; ++r) { hacc[r][0] = __float2half2_rn(0.f); hacc[r][1] = __float2half2_rn(0.f); }
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
        __half2 wr[KS][2];
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
            uint32_t w0, w1;
            lds64(cst_h + (uint32_t)((ky * KS + kx) * CC) * 2, w0, w1);
            wr[kx][0] = *reinterpret_cast<__half2*>(&w0); wr[kx][1] = *reinterpret_cast<__half2*>(&w1);
        }
#pragma unroll
        for (int col = 0; col < G::NCOL; ++col) {
            uint32_t a, b;
            lds64(erow + (uint32_t)(col * PITCH), a, b);
            const __half2 x01 = *reinterpret_cast<__half2*>(&a), x23 = *reinterpret_cast<__half2*>(&b);
#pragma unroll
            for (int r = 0; r < G::R; ++r) {
                const int kx = col - r * S;          // compile-time after unrolling
                if (kx >= 0 && kx < KS) {
                    hacc[r][0] = __hfma2(x01, wr[kx][0], hacc[r][0]);
                    hacc[r][1] = __hfma2(x23, wr[kx][1], hacc[r][1]);
                }
            }
        }
        erow += G::PW * PITCH;
    }
    const float2 sc = make_float2(kDwScale, kDwScale);
    float sum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int r = 0; r < G::R; ++r) {
        float2 a0 = make_float2(bq.x, bq.y), a1 = make_float2(bq.z, bq.w);
        ffma2(a0, __half22float2(hacc[r][0]), sc);          // sum * kDwScale + shift, in fp32
        ffma2(a1, __half22float2(hacc[r][1]), sc);
        a0.x = swish_from_half(a0.x); a0.y = swish_from_half(a0.y);
        a1.x = swish_from_half(a1.x); a1.y = swish_from_half(a1.y);
        sum[0] += a0.x; sum[1] += a0.y; sum[2] += a1.x; sum[3] += a1.y;
        uint2 o;
        o.x = pack2<T>(a0.x, a0.y);
        o.y = pack2<T>(a1.x, a1.y);
        *reinterpret_cast<uint2*>(dst + (long long)r * C) = o;
    }
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(red), "f"(sum[0]), "f"(sum[1]), "f"(sum[2]), "f"(sum[3]) : "memory");
}

// Squeeze sums of a finished chunk (one warp): fixed order over the strips (four chains, as K1) -> reproducible bits.
// `red` = the chunk's scratch [NSTRIPS][CC] fp32; the CC totals go to dst[0..CC), and times inv_hw to means[0..CC) if given.
template <int NSTRIPS, int CC>
__device__ __forceinline__ void squeeze_sums(uint32_t red, float* dst, float* means, float inv_hw, int lane) {
    for (int cc = lane; cc < CC; cc += 32) {
        const uint32_t r0 = red + (uint32_t)(cc * 4);
        float s4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int y = 0; y < NSTRIPS; ++y) {
            float t;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t) : "r"(r0 + (uint32_t)(y * CC * 4)));
            s4[y & 3] += t;
        }
        const float tot = (s4[0] + s4[1]) + (s4[2] + s4[3]);
        dst[cc] = tot;
        if (means) means[cc] = tot * inv_hw;
    }
}

// SE excite + gating of one crop's depthwise output (the CTA wrote all of it; it is still in L2).  sM holds the C channel
// means and room for the Cse hidden units.
template <typename T, int NT, int HO>
__device__ __forceinline__ void se_tail_gate(const DwSeParams& p, int n, T* out_n, float* sM) {
    const int C = p.C;
    se_gate_fc<NT>(sM, sM + C, p.w_se1t, p.b_se1, p.w_se2, p.b_se2, p.gate + (long long)n * C, C, p.Cse, sM);
    __syncthreads();
    if (p.scale_out) {
        const int cv8 = C >> 3, total = HO * HO * cv8;
        const float inv_cv8 = 1.0f / (float)cv8;
        for (int v = threadIdx.x; v < total; v += NT) {
            const int c8 = (v - div_small(v, inv_cv8) * cv8) * 8;
            uint4* ptr = reinterpret_cast<uint4*>(out_n) + v;
            *ptr = tc::scale8s<T>(__ldcg(ptr), tc::smem_u32(sM + c8));
        }
    }
}

// SPATIAL: the map is larger than one CTA can hold and has exactly CC channels (block 1: 112x112x32): the loop runs over the
// HO x HO output tiles of the crop instead of over channel chunks - the same box, started at the tile's corner minus the
// padding, the same strip geometry, squeeze partials per (crop, tile).
template <typename T, int KS, int S, int HIN, int CC, bool SPATIAL = false>
__global__ void __launch_bounds__((DwSeThreads<KS, S, HIN, CC>::value)) dwse_kernel(const __grid_constant__ DwSeParams p) {
    using G = DwSeGeom<KS, S, HIN>;
    constexpr int NT = DwSeThreads<KS, S, HIN, CC>::value;
    constexpr int NW = NT / 32;
    constexpr int CV = CC / 4;                                 // 4-channel vectors per pixel
    constexpr int PITCH = CC * 2;                              // bytes per tile pixel
    constexpr int TILE_TX = G::PW * G::PW * PITCH;             // bytes one tile copy delivers (the zero-filled border counts)
    constexpr int TILE_BYTES = (TILE_TX + 127) / 128 * 128;
    constexpr int CST_TX = CC * 4 + KS * KS * CC * 2;
    constexpr int CST_BYTES = (CST_TX + 127) / 128 * 128;
    constexpr int RED_BYTES = G::NSTRIPS * CC * 4;
    extern __shared__ __align__(128) uint8_t smem_dw[];
    __shared__ __align__(8) uint64_t bars[4];                  // full[2] (TMA bytes), empty[2] (one arrival per warp)
    __shared__ int s_abort_mem;
    volatile int* s_abort = &s_abort_mem;
    const uint32_t s0 = (tc::smem_u32(smem_dw) + 127u) & ~127u;
    const uint32_t sT = s0, sC = sT + 2 * TILE_BYTES, sR = sC + 2 * CST_BYTES;
    float* const sM = reinterpret_cast<float*>(smem_dw + (sR + 2 * RED_BYTES - tc::smem_u32(smem_dw)));     // [C] means | [Cse] hidden
    const uint32_t b_full = tc::smem_u32(&bars[0]), b_empty = tc::smem_u32(&bars[2]);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n = blockIdx.x;
    const int C = p.C;
    const int ch_begin = blockIdx.y * p.chunks_per_cta;
    const int ch_end = min(p.n_chunks, ch_begin + p.chunks_per_cta);
    const int Ho_img = SPATIAL ? p.Ho_img : G::HO;
    T* const out_n = reinterpret_cast<T*>(p.out) + (long long)n * Ho_img * Ho_img * C;

    if (tid == 0) {
        tc::mbar_init(&bars[0], 1); tc::mbar_init(&bars[1], 1);
        tc::mbar_init(&bars[2], NW); tc::mbar_init(&bars[3], NW);
        s_abort_mem = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmE) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
    }
    __syncthreads();

    // the three async copies of one chunk, all completing on full[buf] (thread 0 only)
    auto issue = [&](int ch, int buf) {
        const int cbase = SPATIAL ? 0 : ch * CC;
        const uint32_t bar = b_full + 8 * buf;
        tc::mbar::arrive_expect_tx(bar, (uint32_t)(TILE_TX + CST_TX));
        if (SPATIAL) {
            const int ty = ch / p.tiles_x, tx = ch - ty * p.tiles_x;
            tc::mbar::tma_4d(sT + buf * TILE_BYTES, &p.tmE, 0, tx * G::HO * S - p.pad, ty * G::HO * S - p.pad, n, bar);
        } else
            tc::mbar::tma_4d(sT + buf * TILE_BYTES, &p.tmE, cbase, -p.pad, -p.pad, n, bar);
        tc::mbar::tma_2d(sC + buf * CST_BYTES + CC * 4, &p.tmW, cbase, 0, bar);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(sC + buf * CST_BYTES), "l"(p.b_dw + cbase), "r"((uint32_t)(CC * 4)), "r"(bar) : "memory");
    };

    const int strip = tid / CV, cv = tid - strip * CV;
    const bool active = strip < G::NSTRIPS;
    const int oy = strip / G::SPR, ox0 = (strip - oy * G::SPR) * G::R;
    const uint32_t win = (uint32_t)(((oy * S) * G::PW + ox0 * S) * PITCH + cv * 8);       // top-left of this strip's input window

    if (tid == 0) {
        issue(ch_begin, 0);
        if (ch_begin + 1 < ch_end) issue(ch_begin + 1, 1);
    }

    for (int ch = ch_begin; ch < ch_end; ++ch) {
        const int it = ch - ch_begin, buf = it & 1;
        const uint32_t par = (uint32_t)(it >> 1) & 1u;
        tc::mbar::wait(b_full + 8 * buf, par, s_abort, p.tflag);        // tile + constants of chunk ch have landed
        if (active && !*s_abort) {
            T* dst;
            if (SPATIAL) {
                const int ty = ch / p.tiles_x, tx = ch - ty * p.tiles_x;
                dst = out_n + ((long long)(ty * G::HO + oy) * Ho_img + tx * G::HO + ox0) * C + cv * 4;
            } else
                dst = out_n + ((long long)oy * G::HO + ox0) * C + ch * CC + cv * 4;
            dw_strip<T, KS, S, HIN, CC>(sT + buf * TILE_BYTES + win, sC + buf * CST_BYTES, cv, dst, C,
                                        sR + (uint32_t)(buf * RED_BYTES + (strip * CC + cv * 4) * 4));
        }
        // this warp is done with tile / constants / (its part of) the squeeze scratch of buffer `buf`
        tc::mbar::arrive_warp(b_empty + 8 * buf);
        if (warp == 0) {
            // warp 0 closes the chunk: once EVERY warp has released the buffer it reduces the squeeze scratch and only then
            // refills the buffer with chunk ch+2 - no warp can reach chunk ch+2 (and overwrite the scratch) before that copy lands
            tc::mbar::wait(b_empty + 8 * buf, par, s_abort, p.tflag);
            if (SPATIAL) squeeze_sums<G::NSTRIPS, CC>(sR + buf * RED_BYTES, p.partial + ((long long)n * p.n_chunks + ch) * C, nullptr, 0.f, lane);
            else squeeze_sums<G::NSTRIPS, CC>(sR + buf * RED_BYTES, p.partial + (long long)n * C + ch * CC, p.se_tail ? sM + ch * CC : nullptr, p.inv_hw, lane);
            __syncwarp();
            if (lane == 0 && ch + 2 < ch_end) issue(ch + 2, buf);
        }
    }
    __syncthreads();
    if (!SPATIAL && p.se_tail) se_tail_gate<T, NT, G::HO>(p, n, out_n, sM);
}

// Shapes of the kernel that computes the expand conv itself (dwse_x_kernel): CIN input channels, 256 threads = two
// warpgroups.  X rows per K block: the crop's H*W pixels rounded up to 8 (one swizzle atom); the wgmma reads whole 64-row
// halves, so the last half runs on past X into the next region (the next K block of X, or past the last one into W[0],
// which a TMA refill may be writing at that moment).  Rows of an MMA are independent and those accumulator rows are never
// stored, so whatever the bytes are at that moment cannot reach a result.
template <int KS, int S, int HIN, int CC, int CIN>
struct DwSeX {
    using G = DwSeGeom<KS, S, HIN>;
    static constexpr int NT = 256;
    static constexpr int NKB = (CIN + 63) / 64;                // 64-channel K blocks
    static constexpr int KSTEPS = (CIN + 15) / 16;             // K = 16 MMA steps (the expand GEMM's: channels >= CIN are zero)
    static constexpr int PIX = HIN * HIN;
    static constexpr int HALVES = (PIX + 63) / 64;             // 64-row MMA halves: 4 at 14x14, 1 at 7x7
    static constexpr int XROWS = (PIX + 7) / 8 * 8;
    static_assert(HALVES == 4 || HALVES == 1, "14x14 or 7x7 maps");
    // 14x14: warpgroup g takes halves 2g, 2g+1 over all CC columns; 7x7: the one half, columns [g CC/2, (g+1) CC/2)
    static constexpr int HPW = HALVES == 4 ? 2 : 1;
    static constexpr int NWG = HALVES == 4 ? CC : CC / 2;
    static_assert(NWG % 16 == 0 && NWG <= 128, "wgmma width");
    static_assert(G::NSTRIPS * (CC / 4) <= NT, "one depthwise strip per thread");
    static constexpr uint32_t X_KB = XROWS * 128, X_BYTES = NKB * X_KB;
    static constexpr uint32_t W_KB = CC * 128, W_BYTES = NKB * W_KB;
    static constexpr uint32_t TILE_BYTES = (G::PW * G::PW * CC * 2 + 127) / 128 * 128;
    static constexpr uint32_t CST_TX = CC * 4 + KS * KS * CC * 2;
    static constexpr uint32_t CST_BYTES = (CST_TX + 127) / 128 * 128;
    static constexpr uint32_t RED_BYTES = G::NSTRIPS * CC * 4;
    // offsets from the 1024-aligned base: X | W[2] | E tile[2] | constants[2] | squeeze scratch[2] | means + hidden
    static constexpr uint32_t OFF_W = X_BYTES, OFF_T = OFF_W + 2 * W_BYTES, OFF_C = OFF_T + 2 * TILE_BYTES;
    static constexpr uint32_t OFF_R = OFF_C + 2 * CST_BYTES, OFF_M = OFF_R + 2 * RED_BYTES;
    static_assert((X_KB | W_KB | OFF_W | OFF_T) % 1024 == 0, "SWIZZLE_128B operands sit on 1024-byte boundaries");
    static constexpr size_t smem(int C, int Cse) { return (size_t)OFF_M + (size_t)(C + Cse + 32) * 4 + 1024; }
    // CTAs per SM the instance is compiled for: two where two fit the SM's 228 KB (with <= 1024 SE floats and the 1 KB the
    // SM reserves per CTA) - blocks 7-8; __launch_bounds__ then caps the registers at 128 per thread so that the register
    // file holds both
    static constexpr int CTAS_PER_SM = 2 * ((size_t)OFF_M + 4096 + 1024 + 1024) <= 228 * 1024 ? 2 : 1;
};

template <int KS, int S, int HIN, int CC, int CIN>
__global__ void __launch_bounds__(256, (DwSeX<KS, S, HIN, CC, CIN>::CTAS_PER_SM)) dwse_x_kernel(const __grid_constant__ DwSeParams p) {
    using X = DwSeX<KS, S, HIN, CC, CIN>;
    using G = typename X::G;
    using T = __nv_bfloat16;
    constexpr int NT = X::NT;
    constexpr int CV = CC / 4;
    extern __shared__ uint8_t smem_dwx[];
    __shared__ __align__(8) uint64_t bars[5];                  // X, W[2], constants[2] (TMA bytes)
    __shared__ int s_abort_mem;
    volatile int* s_abort = &s_abort_mem;
    const uint32_t s0 = (tc::smem_u32(smem_dwx) + 1023u) & ~1023u;
    const uint32_t sX = s0, sW = s0 + X::OFF_W, sT = s0 + X::OFF_T, sC = s0 + X::OFF_C, sR = s0 + X::OFF_R;
    float* const sM = reinterpret_cast<float*>(smem_dwx + (s0 + X::OFF_M - tc::smem_u32(smem_dwx)));     // [C] means | [Cse] hidden
    const uint32_t b_x = tc::smem_u32(&bars[0]), b_w = b_x + 8, b_c = b_x + 24;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = tid >> 7, wq = warp & 3;
    const int n = blockIdx.x;
    const int C = p.C, n_chunks = p.n_chunks;
    T* const out_n = reinterpret_cast<T*>(p.out) + (long long)n * G::HO * G::HO * C;

    if (tid == 0) {
        for (int i = 0; i < 5; ++i) tc::mbar_init(&bars[i], 1);
        s_abort_mem = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmX) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmWx) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
    }
    // both E tiles start at zero: the epilogues only ever write the in-image pixels, so the border stays the TF-SAME padding
    for (uint32_t o = (uint32_t)tid * 16; o < 2 * X::TILE_BYTES; o += NT * 16) sts128(sT + o, make_uint4(0, 0, 0, 0));
    __syncthreads();

    // async copies (thread 0): the W slice of chunk j -> W[j & 1]; its depthwise weights + shifts -> constants[j & 1]
    auto issue_w = [&](int j) {
        const uint32_t bar = b_w + 8 * (j & 1);
        tc::mbar::arrive_expect_tx(bar, X::W_BYTES);
        for (int kb = 0; kb < X::NKB; ++kb) tc::mbar::tma_2d(sW + (j & 1) * X::W_BYTES + kb * X::W_KB, &p.tmWx, kb * 64, j * CC, bar);
    };
    auto issue_c = [&](int j) {
        const uint32_t bar = b_c + 8 * (j & 1), dst = sC + (j & 1) * X::CST_BYTES;
        tc::mbar::arrive_expect_tx(bar, X::CST_TX);
        tc::mbar::tma_2d(dst + CC * 4, &p.tmW, j * CC, 0, bar);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "l"(p.b_dw + j * CC), "r"((uint32_t)(CC * 4)), "r"(bar) : "memory");
    };
    if (tid == 0) {
        tc::mbar::arrive_expect_tx(b_x, X::X_BYTES);
        for (int kb = 0; kb < X::NKB; ++kb) tc::mbar::tma_2d(sX + kb * X::X_KB, &p.tmX, kb * 64, n * X::PIX, b_x);
        issue_w(0); issue_c(0);
        if (n_chunks > 1) { issue_w(1); issue_c(1); }
    }

    float acc[X::HPW][X::NWG / 2];
    // the expand MMAs of chunk j over the resident X (one commit group per K block; the caller waits)
    auto mma = [&](int j) {
        tc::mbar::wait(b_x, 0, s_abort, p.tflag);
        tc::mbar::wait(b_w + 8 * (j & 1), (uint32_t)(j >> 1) & 1u, s_abort, p.tflag);
        const uint32_t wb = sW + (j & 1) * X::W_BYTES;
#pragma unroll
        for (int h = 0; h < X::HPW; ++h) {
            if constexpr (X::HALVES == 4) tc::wg_mma_m64<true, X::NWG>(acc[h], sX + (uint32_t)(wg * X::HPW + h) * 64 * 128, X::X_KB, wb, X::W_KB, X::KSTEPS);
            else tc::wg_mma_m64<true, X::NWG>(acc[h], sX, X::X_KB, wb + (uint32_t)wg * X::NWG * 128, X::W_KB, X::KSTEPS);
        }
    };
    // fragments -> swish(acc + bias) as fp16 -> E tile of chunk j (the expand GEMM's epilogue: the bias is halved, h = acc/2 + b/2)
    // register 4i + 2e + q: pixel 16 wq + lane/4 + 8e of the half, column 8i + 2 (lane % 4) + q
    auto epilogue = [&](int j) {
        const uint32_t tile = sT + (j & 1) * X::TILE_BYTES;
        const int c0 = X::HALVES == 4 ? 0 : wg * X::NWG;
        float2 bias[X::NWG / 8];                               // b/2 of this thread's columns 8i + 2 (lane % 4) + {0, 1}
#pragma unroll
        for (int i = 0; i < X::NWG / 8; ++i) {
            const float* b = p.b_exp + j * CC + c0 + 8 * i + 2 * (lane & 3);
            bias[i] = make_float2(0.5f * __ldg(b), 0.5f * __ldg(b + 1));
        }
#pragma unroll
        for (int h = 0; h < X::HPW; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int pix = 64 * (X::HALVES == 4 ? wg * X::HPW + h : 0) + 16 * wq + (lane >> 2) + 8 * e;
                if (pix >= X::PIX) continue;
                const int y = pix / HIN, x = pix - y * HIN;
                const uint32_t prow = tile + (uint32_t)(((y + p.pad) * G::PW + x + p.pad) * CC + c0) * 2;
#pragma unroll
                for (int i = 0; i < X::NWG / 8; ++i) {
                    const int c = 8 * i + 2 * (lane & 3);
                    const float o0 = swish_from_half(fmaf(acc[h][4 * i + 2 * e], 0.5f, bias[i].x));
                    const float o1 = swish_from_half(fmaf(acc[h][4 * i + 2 * e + 1], 0.5f, bias[i].y));
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(prow + (uint32_t)c * 2), "r"(pack2<__half>(o0, o1)) : "memory");
                }
            }
    };

    const int strip = tid / CV, cv = tid - strip * CV;
    const bool active = strip < G::NSTRIPS;
    const int oy = strip / G::SPR, ox0 = (strip - oy * G::SPR) * G::R;
    const uint32_t win = (uint32_t)(((oy * S) * G::PW + ox0 * S) * CC * 2 + cv * 8);       // top-left of this strip's input window

    // depthwise of chunk j out of E tile j & 1
    auto depthwise = [&](int j) {
        tc::mbar::wait(b_c + 8 * (j & 1), (uint32_t)(j >> 1) & 1u, s_abort, p.tflag);
        if (active && !*s_abort)
            dw_strip<T, KS, S, HIN, CC>(sT + (j & 1) * X::TILE_BYTES + win, sC + (j & 1) * X::CST_BYTES, cv,
                                        out_n + ((long long)oy * G::HO + ox0) * C + j * CC + cv * 4, C,
                                        sR + (uint32_t)((j & 1) * X::RED_BYTES + (strip * CC + cv * 4) * 4));
    };
    // after the CTA barrier that ends chunk j: its squeeze sums (warp 0), refills of the buffers it freed (thread 0)
    auto close = [&](int j) {
        if (warp == 0)
            squeeze_sums<G::NSTRIPS, CC>(sR + (j & 1) * X::RED_BYTES, p.partial + (long long)n * C + j * CC,
                                         p.se_tail ? sM + j * CC : nullptr, p.inv_hw, lane);
        if (tid == 0) {
            if (j + 3 < n_chunks) issue_w(j + 3);
            if (j + 2 < n_chunks) issue_c(j + 2);
        }
    };

    mma(0);
    tc::wg_wait<0>();
    epilogue(0);
    __syncthreads();                                           // E tile 0 complete, W[0] free
    if (tid == 0 && 2 < n_chunks) issue_w(2);
    // the MMAs of chunk j+1 run on the tensor cores under chunk j's depthwise; the loop leaves the last chunk out so that
    // issue and wait are unconditional (a wgmma group that is only conditionally waited for makes ptxas wait right away)
    for (int j = 0; j + 1 < n_chunks; ++j) {
        mma(j + 1);
        depthwise(j);
        tc::wg_wait<0>();
        epilogue(j + 1);                                       // into the tile chunk j-1 used
        // chunk j's tile, constants and scratch are read; chunk j+1's MMAs are complete (W[(j+1) & 1] is free)
        __syncthreads();
        close(j);
    }
    depthwise(n_chunks - 1);
    __syncthreads();
    close(n_chunks - 1);
    __syncthreads();
    if (p.se_tail) se_tail_gate<T, NT, G::HO>(p, n, out_n, sM);
}

// which (kernel, stride, map size, channels) combinations have an instance, and with which chunk width
inline int dwse_chunk(int k, int s, int hin, int C) {
    if (hin == 14 && s == 1 && (k == 3 || k == 5) && C % 32 == 0) return 32;
    if (hin == 14 && s == 2 && k == 5 && C % 96 == 0) return 96;
    if (hin == 7 && s == 1 && (k == 3 || k == 5) && C % 128 == 0) return 128;
    return 0;
}

template <typename T>
int launch_dwse(cudaStream_t stream, DwSeParams p, int k, int s, int hin, int n_crops, int split) {
    const int CCr = dwse_chunk(k, s, hin, p.C);
    if (!CCr) return 1;
    p.N = n_crops;
    p.n_chunks = p.C / CCr;
    if (split < 1) split = 1;
    if (split > p.n_chunks) split = p.n_chunks;
    p.chunks_per_cta = (p.n_chunks + split - 1) / split;
    const int gy = (p.n_chunks + p.chunks_per_cta - 1) / p.chunks_per_cta;
    if (gy > 1) { p.se_tail = 0; p.scale_out = 0; }
#define DWSE(KS, S, HIN, CC)                                                                                              \
    do {                                                                                                                  \
        auto kfn = dwse_kernel<T, KS, S, HIN, CC>;                                                                        \
        const size_t smem = dwse_smem<KS, S, HIN, CC>(p.C, p.Cse);                                                        \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;  \
        kfn<<<dim3(n_crops, gy), DwSeThreads<KS, S, HIN, CC>::value, smem, stream>>>(p);                                    \
        return 0;                                                                                                         \
    } while (0)
    if (hin == 14 && s == 1 && k == 3) DWSE(3, 1, 14, 32);
    if (hin == 14 && s == 1 && k == 5) DWSE(5, 1, 14, 32);
    if (hin == 14 && s == 2 && k == 5) DWSE(5, 2, 14, 96);
    if (hin == 7 && s == 1 && k == 5) DWSE(5, 1, 7, 128);
    if (hin == 7 && s == 1 && k == 3) DWSE(3, 1, 7, 128);
#undef DWSE
    return 1;
}


// The crop's depthwise + SE with the expand conv computed on chip (dwse_x_kernel): one CTA per crop, every chunk.  `cin` = the
// block's input channels; the tensor maps tmX / tmWx and b_exp must be set.  1: no instance for this shape.
template <typename T>
int launch_dwse_x(cudaStream_t stream, DwSeParams p, int k, int s, int hin, int cin, int n_crops) {
    static_assert(std::is_same<T, __nv_bfloat16>::value, "the on-chip expand runs the bf16 wgmma");
    const int CCr = dwse_chunk(k, s, hin, p.C);
    if (!CCr) return 1;
    p.N = n_crops;
    p.n_chunks = p.C / CCr;
    p.chunks_per_cta = p.n_chunks;
#define DWSEX(KS, S, HIN, CC, CIN)                                                                                        \
    do {                                                                                                                  \
        auto kfn = dwse_x_kernel<KS, S, HIN, CC, CIN>;                                                                    \
        const size_t smem = DwSeX<KS, S, HIN, CC, CIN>::smem(p.C, p.Cse);                                                 \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;  \
        kfn<<<n_crops, DwSeX<KS, S, HIN, CC, CIN>::NT, smem, stream>>>(p);                                                \
        return 0;                                                                                                         \
    } while (0)
    if (CCr == 32 && hin == 14 && s == 1 && k == 3 && cin == 80) DWSEX(3, 1, 14, 32, 80);
    if (CCr == 32 && hin == 14 && s == 1 && k == 5 && cin == 80) DWSEX(5, 1, 14, 32, 80);
    if (CCr == 32 && hin == 14 && s == 1 && k == 5 && cin == 112) DWSEX(5, 1, 14, 32, 112);
    if (CCr == 96 && hin == 14 && s == 2 && k == 5 && cin == 112) DWSEX(5, 2, 14, 96, 112);
    if (CCr == 128 && hin == 7 && s == 1 && k == 5 && cin == 192) DWSEX(5, 1, 7, 128, 192);
    if (CCr == 128 && hin == 7 && s == 1 && k == 3 && cin == 192) DWSEX(3, 1, 7, 128, 192);
#undef DWSEX
    return 1;
}

// Block 1 (no expand conv): 3x3 stride-1 depthwise over the 112x112x32 stem output (fp16) in 14x14 output tiles.
template <typename T>
int launch_dwse_spatial(cudaStream_t stream, DwSeParams p, int H, int n_crops, int split) {
    if (p.C != 32 || H % 14) return 1;
    p.N = n_crops;
    p.tiles_x = H / 14; p.Ho_img = H;
    p.n_chunks = p.tiles_x * p.tiles_x;
    if (split < 1) split = 1;
    if (split > p.n_chunks) split = p.n_chunks;
    p.chunks_per_cta = (p.n_chunks + split - 1) / split;
    const int gy = (p.n_chunks + p.chunks_per_cta - 1) / p.chunks_per_cta;
    p.se_tail = 0; p.scale_out = 0;
    auto kfn = dwse_kernel<T, 3, 1, 14, 32, true>;
    const size_t smem = dwse_smem<3, 1, 14, 32>(0, 0);
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    kfn<<<dim3(n_crops, gy), DwSeThreads<3, 1, 14, 32>::value, smem, stream>>>(p);
    return 0;
}

}  // namespace fused
}  // namespace whenet
