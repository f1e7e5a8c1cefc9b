// kernels_k2.cuh - K2: persistent, TMA-fed, warp-specialised 1x1 convolution (project convs, head conv).
//
//   out[m, n] = act( bias[n] + sum_k (A[m,k] * gate[m/hw, k]) * Wt[n,k] ) (+ resid[m,n])
//
// Same contract as pw_tc2_kernel (kernels_tc.cuh); different machine mapping.  pw_tc2 gives one 128-thread CTA one
// 128-row tile: every tile pays barrier set-up, a cold cp.async ring and a serial fill -> MMA -> epilogue sequence.
// K2 keeps ONE CTA per SM for the whole launch:
//
//   warp 0            TMA producer   A[128 x 64] (+ W[n_tile x 64] when the weights are streamed) per K block -> ring
//   warps 4-7, 8-11   MMA + epilogue two warpgroups (group 0: this CTA's even tiles, group 1: the odd ones): wgmma over the ring
//                                    stages of the tile (full-width m64nNk16, one commit group per K block, two blocks in
//                                    flight; each stage handed back to the producer once its MMAs are complete;
//                                    the groups take the ring in turns, tile by tile, so that no group waits on a ring slot
//                                    more than one phase ahead of the producer - parity waits cannot tell phases two apart),
//                                    then registers -> +bias (-> swish) (+residual) -> 16-bit -> global, while the other group
//                                    runs the MMAs of its tile.  The bias row sits in shared memory (pre-halved for the swish
//                                    form h = acc/2 + b/2: one FFMA, then MUFU.TANH + FFMA)
//   warps 12-15       gate           (gated convs) rescale the freshly landed A stage in shared memory by the SE gate of
//                                    each row's crop, fence.proxy.async, hand the stage to the MMA warpgroup
//
// Tiles (128 rows x n_tile columns) are dealt round-robin; weights that fit (<= 64 KB: every project up to block 9) are
// loaded once per CTA and stay resident.  The producer runs several K blocks ahead, across tile boundaries.
#pragma once
#include <cuda.h>

#include "kernels_fused.cuh"

namespace whenet {
namespace tc {

struct alignas(64) K2Params {
    CUtensorMap tmA;       // activations [M][K] (dims: K, M), box {64, 128}, SWIZZLE_128B
    CUtensorMap tmW;       // weights [N][K] K-major (dims: K, N), box {64, n_tile}, SWIZZLE_128B
    const float* bias;     // [N]
    const float* gate;     // [crops][K] or NULL
    const void* resid;     // T [M][N] or NULL
    void* out;             // T [M][N]
    int* tflag;
    int M, K, N, hw;
    int n_tile, n_tiles;   // columns per tile (multiple of 16, <= kK2MaxN), tiles along N
    int m_tiles, tiles;    // tiles = m_tiles * n_tiles
    int nkb;               // 64-channel K blocks
    int ksteps_last;       // K = 16 MMA steps of the last K block
    int stages;            // ring depth
    int w_resident;        // 1: the whole [n_tile x K] weight slice of this CTA's n tile stays in shared memory
    uint32_t a_stage, w_stage;        // bytes per ring stage (w_stage = 0 when resident)
    uint32_t off_w, off_ring, off_g;  // shared-memory offsets from the 1024-aligned base: resident W | ring | gate rows
    uint32_t off_b;                   // ... | bias row [N] fp32
    uint32_t g_rows;                  // gate rows (crops) one tile can touch
};

constexpr int kK2Threads = 512;
constexpr int kK2MaxN = 64;       // accumulator registers per MMA thread = n_tile (128 rows x n_tile over one warpgroup)

// NT = p.n_tile (16, 32, 48 or 64): the MMA width
template <typename T, bool SWISH, bool GATE, bool RESID, int NT>
__global__ void __launch_bounds__(kK2Threads, 1) k2_kernel(const __grid_constant__ K2Params p) {
    using namespace whenet::fused;
    extern __shared__ uint8_t smem_raw[];
    // [0..7] full  [8..15] ready  [16..23] empty  [24] w  [25, 26] turn of MMA group 0 / 1
    __shared__ __align__(8) uint64_t bars[27];
    __shared__ int s_abort_mem;
    volatile int* s_abort = &s_abort_mem;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sW = smem0 + p.off_w, sRing = smem0 + p.off_ring, sG = smem0 + p.off_g, sB = smem0 + p.off_b;
    const uint32_t bar0 = smem_u32(&bars[0]);
    const uint32_t b_full = bar0, b_ready = bar0 + 64, b_empty = bar0 + 128, b_w = bar0 + 192, b_turn = bar0 + 200;
    const uint32_t stage_bytes = p.a_stage + p.w_stage;
    constexpr int kGateThreads = 128;

    if (tid == 0) {
        for (int i = 0; i < 8; ++i) {
            mbar_init(&bars[i], 1);
            mbar_init(&bars[8 + i], kGateThreads / 32);     // counts are WARPS (arrive_warp)
            mbar_init(&bars[16 + i], 1);
        }
        mbar_init(&bars[24], 1);
        mbar_init(&bars[25], 1);
        mbar_init(&bars[26], 1);
        s_abort_mem = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < p.N; i += kK2Threads) {
        const float b = __ldg(p.bias + i);
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(sB + (uint32_t)i * 4u), "f"(SWISH ? 0.5f * b : b) : "memory");
    }
    __syncthreads();

    // tile -> (m tile, n tile): the n tiles of one m tile are adjacent (A re-read from L2); with resident weights every
    // CTA keeps ONE n tile (n_tiles == 1 in that mode)
    const int first = blockIdx.x, step = gridDim.x;

    if (warp == 0) {
        // =========================================================================== TMA producer
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
            if (p.w_resident) {
                mbar::arrive_expect_tx(b_w, (uint32_t)p.nkb * p.n_tile * 128);
                for (int kb = 0; kb < p.nkb; ++kb) mbar::tma_2d(sW + (uint32_t)kb * p.n_tile * 128, &p.tmW, kb * 64, 0, b_w);
            }
            int g = 0;                                  // global K-block counter of this CTA: ring slot = g % stages
            for (int tile = first; tile < p.tiles; tile += step) {
                const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
                for (int kb = 0; kb < p.nkb; ++kb, ++g) {
                    const int s = g % p.stages;
                    const uint32_t par = (uint32_t)(g / p.stages) & 1u;
                    mbar::wait(b_empty + 8 * s, par ^ 1, s_abort, p.tflag);          // the MMAs that read this slot have completed
                    mbar::arrive_expect_tx(b_full + 8 * s, stage_bytes);
                    mbar::tma_2d(sRing + (uint32_t)s * stage_bytes, &p.tmA, kb * 64, mt * BM, b_full + 8 * s);
                    if (!p.w_resident) mbar::tma_2d(sRing + (uint32_t)s * stage_bytes + p.a_stage, &p.tmW, kb * 64, nt * p.n_tile, b_full + 8 * s);
                }
            }
        }
    } else if (warp >= 4 && warp < 12) {
        // =========================================================================== MMA + epilogue (group grp: tiles k = grp, grp + 2, ...)
        constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
        const int wq = warp & 3, grp = (warp - 4) >> 2;
        const int wt = tid & 127;
        const T* resid = reinterpret_cast<const T*>(p.resid);
        T* out = reinterpret_cast<T*>(p.out);
        if (p.w_resident) mbar::wait(b_w, 0, s_abort, p.tflag);
        for (int tile = first + grp * step, k = grp; tile < p.tiles; tile += 2 * step, k += 2) {
            const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
            WgAcc<NT> acc;
            if (k > 0) mbar::wait(b_turn + 8 * grp, (uint32_t)((k - 1) >> 1) & 1u, s_abort, p.tflag);    // the other group is done with tile k-1
            // one wgmma group per K block, up to two in flight: once block kb is issued, wait for block kb-1's group and hand
            // ITS slot back to the producer, so the MMAs of block kb-1 are still running while block kb is issued
            const int g0 = k * p.nkb;                            // ring slots are filled in tile order
            for (int kb = 0; kb < p.nkb; ++kb) {
                const int g = g0 + kb;
                const int s = g % p.stages;
                const uint32_t par = (uint32_t)(g / p.stages) & 1u;
                mbar::wait((GATE ? b_ready : b_full) + 8 * s, par, s_abort, p.tflag);
                const uint32_t a_st = sRing + (uint32_t)s * stage_bytes;
                const uint32_t w_st = p.w_resident ? sW + (uint32_t)kb * NT * 128 : a_st + p.a_stage;
                wg_mma_tile<BF16, NT>(acc, a_st, w_st, kb == p.nkb - 1 ? p.ksteps_last : 4, kb ? 1u : 0u);     // one commit group
                if (kb > 0) {
                    wg_wait<1>();
                    asm volatile("bar.sync %0, 128;" ::"r"(2 + grp) : "memory");  // the whole warpgroup's MMAs are done with slot g-1
                    if (wt == 0) mbar::arrive(b_empty + 8 * ((g - 1) % p.stages));
                }
            }
            wg_wait<0>();
            asm volatile("bar.sync %0, 128;" ::"r"(2 + grp) : "memory");
            if (wt == 0) {
                mbar::arrive(b_empty + 8 * ((g0 + p.nkb - 1) % p.stages));
                mbar::arrive(b_turn + 8 * (grp ^ 1));
            }
            if (*s_abort) continue;
            // fragment -> output: register 4i + e = row 16 wq + lane/4 (+8 for e >= 2) of row half h,
            // columns 8 i + 2 (lane % 4) + {0, 1}
            const int n0 = nt * NT;
            const int n_valid = min(NT, p.N - n0);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e2 = 0; e2 < 2; ++e2) {
                    const long long m = (long long)mt * BM + 64 * h + 16 * wq + (lane >> 2) + 8 * e2;
                    if (m >= p.M) continue;
#pragma unroll
                    for (int i = 0; i < NT / 8; ++i) {
                        const int c = 8 * i + 2 * (lane & 3);
                        if (c >= n_valid) continue;
                        const int n = n0 + c;
                        float2 b;
                        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(b.x), "=f"(b.y) : "r"(sB + (uint32_t)n * 4u));
                        const float a0 = acc.d[h][4 * i + 2 * e2], a1 = acc.d[h][4 * i + 2 * e2 + 1];
                        // swish: b holds b/2 -> h = acc/2 + b/2 == (acc + b)/2 bit for bit (the halving is exact)
                        float o0 = SWISH ? swish_from_half(fmaf(a0, 0.5f, b.x)) : a0 + b.x;
                        float o1 = SWISH ? swish_from_half(fmaf(a1, 0.5f, b.y)) : a1 + b.y;
                        if (RESID) {
                            float lo, hi;
                            unpack2<T>(*reinterpret_cast<const uint32_t*>(resid + m * p.N + n), lo, hi);
                            o0 += lo; o1 += hi;
                        }
                        *reinterpret_cast<uint32_t*>(out + m * p.N + n) = pack2<T>(o0, o1);
                    }
                }
        }
    } else if (GATE && warp >= 12) {
        // =========================================================================== gate: A stage <- A stage * gate[crop(row)]
        const int gtid = tid - 384;
        const int c = gtid & 7, r0 = gtid >> 3;                  // this thread: 16-byte chunk c of rows r0, r0 + 16, ..., r0 + 112
        const uint32_t swz = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));
        const int kchunks = p.K >> 3;
        int g = 0;
        int crop0_loaded = -1;
        for (int tile = first; tile < p.tiles; tile += step) {
            const int mt = tile / p.n_tiles;
            const int m0 = mt * BM;
            const int rows_valid = min(BM, p.M - m0);
            const int crop0 = m0 / p.hw;
            // gate rows of the crops this tile touches -> shared memory (skipped when the previous tile had the same first crop
            // and the tile stays inside the rows already loaded: tiles of one crop follow each other only with one n tile)
            const int ncrops = (m0 + rows_valid - 1) / p.hw - crop0 + 1;
            if (crop0 != crop0_loaded || ncrops > 1) {
                asm volatile("bar.sync 1, %0;" ::"n"(kGateThreads) : "memory");   // every gate thread is done with the previous rows
                const int q = p.K >> 2;
                for (int idx = gtid; idx < ncrops * q; idx += kGateThreads) {
                    const int cr = idx / q, j = idx - cr * q;
                    const float4 v = __ldg(reinterpret_cast<const float4*>(p.gate + (long long)(crop0 + cr) * p.K) + j);
                    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(sG + (uint32_t)(cr * p.K + j * 4) * 4), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
                }
                asm volatile("bar.sync 1, %0;" ::"n"(kGateThreads) : "memory");
                crop0_loaded = ncrops > 1 ? -1 : crop0;
            }
            // gate row of each of this thread's four tile rows: (m0 + r) / hw - crop0 without an integer division per row
            // (r + offset-in-crop < 128 + hw: the float reciprocal is exact for these small numbers)
            uint32_t g_row[8];
            {
                const int off = m0 - crop0 * p.hw;
                const float inv_hw = 1.0f / (float)p.hw;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = r0 + 16 * i;
                    g_row[i] = r < rows_valid ? (uint32_t)(div_small(r + off, inv_hw) * p.K) * 4u : 0u;
                }
            }
            for (int kb = 0; kb < p.nkb; ++kb, ++g) {
                const int s = g % p.stages;
                const uint32_t par = (uint32_t)(g / p.stages) & 1u;
                mbar::wait(b_full + 8 * s, par, s_abort, p.tflag);
                const uint32_t a0 = sRing + (uint32_t)s * stage_bytes + swz;
                if (kb * 8 + c < kchunks) {
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (r0 + 16 * i < rows_valid)
                            sts128_(a0 + i * 2048, scale8s<T>(lds128(a0 + i * 2048), sG + g_row[i] + (uint32_t)((kb * 8 + c) * 8) * 4));
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar::arrive_warp(b_ready + 8 * s);
            }
        }
    }
}

// Fills every field of K2Params except the tensor maps and the pointers.  false: shape not supported (caller falls back).
inline bool plan_k2(long long M, int K, int N, int hw, bool has_gate, bool is_bf16, K2Params* p, size_t* smem_out) {
    if ((K & 7) || (N & 7) || M < 1 || M > 0x7fffffffLL || K < 16) return false;
    p->M = (int)M; p->K = K; p->N = N; p->hw = hw;
    int n_tile = N;
    if (N > kK2MaxN) {
        int parts = (N + kK2MaxN - 1) / kK2MaxN;
        while (true) {
            n_tile = ((N + parts - 1) / parts + 15) & ~15;
            if (n_tile <= kK2MaxN) break;
            ++parts;
        }
    }
    n_tile = (n_tile + 15) & ~15;
    p->n_tile = n_tile;
    p->n_tiles = (N + n_tile - 1) / n_tile;
    p->m_tiles = (int)((M + BM - 1) / BM);
    p->tiles = p->m_tiles * p->n_tiles;
    p->nkb = (K + 63) / 64;
    p->ksteps_last = ((K - (p->nkb - 1) * 64) + 15) / 16;
    (void)is_bf16;
    p->a_stage = BM * 128;
    const size_t w_all = (size_t)p->nkb * n_tile * 128;
    p->g_rows = has_gate ? (uint32_t)std::min(4, (BM - 1) / hw + 2) : 0;
    const size_t g_bytes = (size_t)p->g_rows * K * 4;
    const size_t budget = 222 * 1024 - (size_t)N * 4;
    // weights stay resident when the whole [N x K] slice fits next to a ring of at least three A stages (every project up to
    // block 11: <= 154 KB); streaming them with every A stage doubled the L2 -> SM traffic of the K = 480 / 672 projects
    p->w_resident = (p->n_tiles == 1 && w_all + 3 * (size_t)p->a_stage + g_bytes <= budget) ? 1 : 0;
    p->w_stage = p->w_resident ? 0 : (uint32_t)n_tile * 128;
    int stages = 8;
    while (stages > 2 && (p->w_resident ? w_all : 0) + (size_t)stages * (p->a_stage + p->w_stage) + g_bytes > budget) --stages;
    if ((p->w_resident ? w_all : 0) + (size_t)stages * (p->a_stage + p->w_stage) + g_bytes > budget) return false;
    p->stages = stages;
    p->off_w = 0;
    p->off_ring = (uint32_t)((p->w_resident ? w_all : 0) + 1023) & ~1023u;
    p->off_g = p->off_ring + (uint32_t)stages * (p->a_stage + p->w_stage);
    p->off_b = p->off_g + (uint32_t)((g_bytes + 15) & ~(size_t)15);
    *smem_out = (size_t)p->off_b + (size_t)N * 4 + 1024;
    return true;
}

template <typename T>
int launch_k2(cudaStream_t stream, const K2Params& p, size_t smem, bool swish, bool gate, bool resid, int sm_count) {
    const int ctas = p.tiles < sm_count ? p.tiles : sm_count;
    if (ctas < 1) return 0;
#define K2_GO(SW, GA, RE)                                                                                                     \
    return with_mma_width<kK2MaxN>(p.n_tile, [&](auto nt) {                                                                 \
        auto kfn = k2_kernel<T, SW, GA, RE, decltype(nt)::value>;                                                           \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024) != cudaSuccess) return -1;   \
        kfn<<<ctas, kK2Threads, smem, stream>>>(p);                                                                         \
        return 0;                                                                                                           \
    })
    if (swish && !gate && !resid) K2_GO(true, false, false);
    if (!swish && !gate && !resid) K2_GO(false, false, false);
    if (!swish && !gate && resid) K2_GO(false, false, true);
    if (!swish && gate && !resid) K2_GO(false, true, false);
    if (!swish && gate && resid) K2_GO(false, true, true);
#undef K2_GO
    return 1;
}

}  // namespace tc
}  // namespace whenet
