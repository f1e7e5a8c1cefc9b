// kernels_dwse.cuh - KD: depthwise KSxKS + BN shift + swish + squeeze + excite (+ gating of its own output) for the blocks
// whose feature map is small enough that ONE CTA holds a whole crop (14x14 and 7x7, blocks 7-16).
//
// Why a second route next to K1 for these blocks: K1 keeps the expanded tensor on the SM, which saves HBM traffic the late
// blocks do not have (their expanded tensors - 29..135 MB per 256..512 crops - live in the 126 MB L2), and pays for it with
// a chain of CTA-wide phases (MMA wait -> TMEM epilogue -> barrier -> depthwise -> barrier -> reduce) at one CTA per SM;
// measured 13.9 k cycles per channel chunk at 7x7 for ~6.5 k warp instructions (profiles/README.md, round 2).  Here the
// expand conv runs as a plain tensor-core GEMM whose epilogue writes E as fp16 (pw_tc2, OUT_H) and this kernel does the rest
// with every thread busy on identical work:
//
//   CTA = one crop; for each chunk of CC channels (two buffers; thread 0 issues the TMA copies of chunk i+2 as soon as every
//   warp has released the buffer of chunk i, so the warps run up to one chunk apart instead of meeting at a CTA barrier):
//       E[crop][all pixels][CC] -> smem tile by ONE cp.async.bulk.tensor.4d whose box starts at (-pad, -pad): the TMA unit
//       zero-fills the out-of-image border = TF-SAME padding for free, no bounds tests and no address arithmetic in the
//       kernel; the chunk's depthwise weights [k*k][CC] come by a 2-D tensor copy, its BN shifts by a 1-D bulk copy
//       thread = (strip of 7 output pixels of one row, 4 channels): HFMA2 running sums over the fp16 tile, fp16 weights / 4
//       -> fp32: sum * 4 + shift, swish, squeeze partial sums (fixed order), 16-bit store of D
//   tail: channel means -> FC + swish -> FC + sigmoid -> gate (same device function as se_gate_kernel, same bits);
//         the CTA then rescales its own D (still in L2) so that the project conv runs ungated.
//
// The arithmetic of one output is exactly K1's (fp16 E, HFMA2 taps in the same order, fp32 epilogue), so both routes agree to
// the rounding of the expand accumulators (K1 carries the BN shift through the tensor core as a bf16 hi/lo pair, the GEMM
// route adds it in fp32).
#pragma once
#include <cuda.h>

#include "kernels_fused.cuh"

namespace whenet {
namespace fused {

struct alignas(64) DwSeParams {
    CUtensorMap tmE;        // E [N][HIN][HIN][C] fp16 (expand conv + BN + swish): dims (C, W, H, N), box (CC, PW, PW, 1), no swizzle
    CUtensorMap tmW;        // w16 [KS*KS][C] fp16 = 0.5 * BN-folded depthwise weights / kDwScale: dims (C, KS*KS), box (CC, KS*KS)
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
    // squeeze sums of a finished chunk (warp 0): fixed order over the strips (four chains, as K1) -> reproducible bits
    auto finish_sums = [&](int ch, int buf) {
        for (int cc = lane; cc < CC; cc += 32) {
            const uint32_t r0 = sR + (uint32_t)(buf * RED_BYTES + cc * 4);
            float s4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int y = 0; y < G::NSTRIPS; ++y) {
                float t;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t) : "r"(r0 + (uint32_t)(y * CC * 4)));
                s4[y & 3] += t;
            }
            const float tot = (s4[0] + s4[1]) + (s4[2] + s4[3]);
            if (SPATIAL) p.partial[((long long)n * p.n_chunks + ch) * C + cc] = tot;
            else {
                p.partial[(long long)n * C + ch * CC + cc] = tot;
                if (p.se_tail) sM[ch * CC + cc] = tot * p.inv_hw;
            }
        }
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
            const uint32_t cst = sC + buf * CST_BYTES;
            const float4 bq = lds_f4(cst + (uint32_t)cv * 16);
            const uint32_t cst_h = cst + (uint32_t)(CC * 4 + cv * 8);
            uint32_t erow = sT + buf * TILE_BYTES + win;
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
            T* dst;
            if (SPATIAL) {
                const int ty = ch / p.tiles_x, tx = ch - ty * p.tiles_x;
                dst = out_n + ((long long)(ty * G::HO + oy) * Ho_img + tx * G::HO + ox0) * C + cv * 4;
            } else
                dst = out_n + ((long long)oy * G::HO + ox0) * C + ch * CC + cv * 4;
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
            asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(sR + (uint32_t)(buf * RED_BYTES + (strip * CC + cv * 4) * 4)),
                         "f"(sum[0]), "f"(sum[1]), "f"(sum[2]), "f"(sum[3]) : "memory");
        }
        // this warp is done with tile / constants / (its part of) the squeeze scratch of buffer `buf`
        tc::mbar::arrive_warp(b_empty + 8 * buf);
        if (warp == 0) {
            // warp 0 closes the chunk: once EVERY warp has released the buffer it reduces the squeeze scratch and only then
            // refills the buffer with chunk ch+2 - no warp can reach chunk ch+2 (and overwrite the scratch) before that copy lands
            tc::mbar::wait(b_empty + 8 * buf, par, s_abort, p.tflag);
            finish_sums(ch, buf);
            __syncwarp();
            if (lane == 0 && ch + 2 < ch_end) issue(ch + 2, buf);
        }
    }
    __syncthreads();

    // ---- SE excite + gating of this crop's depthwise output (the CTA wrote all of it; it is still in L2)
    if (!SPATIAL && p.se_tail) {
        se_gate_fc<NT>(sM, sM + C, p.w_se1t, p.b_se1, p.w_se2, p.b_se2, p.gate + (long long)n * C, C, p.Cse, sM);
        __syncthreads();
        if (p.scale_out) {
            const int cv8 = C >> 3, total = G::HO * G::HO * cv8;
            const float inv_cv8 = 1.0f / (float)cv8;
            for (int v = tid; v < total; v += NT) {
                const int c8 = (v - div_small(v, inv_cv8) * cv8) * 8;
                uint4* ptr = reinterpret_cast<uint4*>(out_n) + v;
                *ptr = tc::scale8s<T>(__ldcg(ptr), tc::smem_u32(sM + c8));
            }
        }
    }
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
