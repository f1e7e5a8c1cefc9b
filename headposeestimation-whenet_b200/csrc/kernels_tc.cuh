// kernels_tc.cuh - Hopper warpgroup-MMA (wgmma) kernels for the 1x1 convolutions + the helpers every tensor-core kernel shares.
//
//   out[m, n] = act( bias[n] + sum_k (A[m,k] * gate[m/hw, k]) * Wt[n,k] ) (+ resid[m,n])
//
// A  : activations, NHWC == row-major [M = crops*H*W][K = Cin], 16-bit (bf16 / fp16)   -> "K-major"
// Wt : BN-folded weights transposed to [N = Cout][K], 16-bit                           -> "K-major"
// D  : fp32 accumulators in the registers of the issuing warpgroup (128 threads)
//
// Operands sit in shared memory in the canonical K-major SWIZZLE_128B layout (16-byte chunk c of row r lands at chunk
// c ^ (r & 7) of its 128-byte row; 8-row atoms of 1024 B).  A 128-row tile is two wgmma.m64nNk16 row halves, one
// instruction per half and K step for the full tile width N (a template parameter of the kernels).  After the last K step
// the warpgroup writes its fragments to a shared-memory accumulator tile ([column][kAccPitch] fp32), where the epilogues
// read one pixel row per thread.
//
// Every mbarrier wait is bounded: a wait that exceeds its budget raises the context's timeout flag (mapped pinned host
// memory) and the CTA bails out instead of hanging the GPU.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels_simt.cuh"

namespace whenet {
namespace tc {

// Timeout flag: ONE int per context in mapped pinned host memory (whenet_api.cu); every pipelined tensor-core kernel gets its
// device address as a parameter and raises it when a bounded mbarrier wait expires.  The host reads it straight from the
// pinned page after any stream synchronisation - no per-translation-unit device symbols, no extra copies.

constexpr int BM = 128;          // pixels per tile (two wgmma row halves of 64)
constexpr int BK = 64;           // channels per stage (one 128-byte swizzle row of 16-bit elements)
constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KB
constexpr int kAccPitch = 132;   // floats per column of the shared-memory accumulator tile (128 rows + 4: conflict-free both ways)
__host__ __device__ constexpr uint32_t acc_tile_bytes(int cols) { return (uint32_t)cols * kAccPitch * 4u; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// bounded parity wait; returns false on timeout
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* tflag) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t it = 0; it < (1u << 22); ++it) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return true;
    }
    *reinterpret_cast<volatile int*>(tflag) = 1;
    return false;
}

// Barriers by shared-memory address and the TMA copies that complete on them, for the warp-specialised kernels (K2, KD),
// whose roles share one abort flag per CTA.
namespace mbar {

// Bounded wait on a barrier given by its shared-memory address.  The loop body is try_wait + branch (ncu showed the
// re-poll loop of the first version at 16-22 % of all issued instructions, taken from the warps that had work); the abort
// flag is looked at every 64 polls only.  A protocol bug ends in the timeout flag instead of a hung GPU.
// No suspend-time hint: with one, ptxas emits NANOSLEEP.SYNCS and the wake-up after the arrive was measured to cost the
// waiting role far more than the polls it saves (K2: 1.9 us per 128-row tile of a K = 32 layer).
__device__ __forceinline__ void wait(uint32_t bar_addr, uint32_t parity, volatile int* abort_flag, int* tflag) {
    for (uint32_t outer = 0; outer < (1u << 18); ++outer) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
            "mov.u32 n, 64;\n"
            "MBAR_POLL_%=:\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "@p bra MBAR_DONE_%=;\n\t"
            "sub.u32 n, n, 1;\n\t"
            "setp.ne.u32 p, n, 0;\n\t"
            "@p bra MBAR_POLL_%=;\n\t"
            "setp.eq.u32 p, n, 1;\n"          // false: n == 0 here
            "MBAR_DONE_%=:\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar_addr), "r"(parity) : "memory");
        if (done) return;
        if (*abort_flag) return;
    }
    *abort_flag = 1;
    *reinterpret_cast<volatile int*>(tflag) = 1;
}
__device__ __forceinline__ void arrive(uint32_t bar_addr) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_addr) : "memory");
}
// One arrival per WARP: __syncwarp orders the lanes' shared-memory accesses before lane 0's (releasing) arrive.  Per-thread
// arrives are 32 serialised shared-memory atomics per warp on one word; with 20+ warps signalling 4-5 barriers per item they
// kept the LSU busy for more than a thousand cycles per item.
__device__ __forceinline__ void arrive_warp(uint32_t bar_addr) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) arrive(bar_addr);
}
__device__ __forceinline__ void arrive_expect_tx(uint32_t bar_addr, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_4d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, uint32_t bar_addr) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar_addr) : "memory");
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar_addr) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(bar_addr) : "memory");
}

}  // namespace mbar

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA descriptor):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 = 1 | [32,46) SBO >> 4 = 64 (8 rows x 128 B) | [62,64) layout = 1 (SWIZZLE_128B)
// A K step of 16 elements (32 bytes inside the swizzle row) advances the start address field by 2.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)64 << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// K-major SWIZZLE_64B descriptor: as make_desc with SBO >> 4 = 32 (8 rows x 64 B) and layout = 2 (SWIZZLE_64B).  The
// operand sits on 512-byte atoms; a K step of 16 elements still advances the start address field by 2.
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)32 << 32;
    d |= (uint64_t)2 << 62;
    return d;
}
// the descriptor of a K-major operand with ROWB-byte rows (128: SWIZZLE_128B, 64: SWIZZLE_64B)
template <int ROWB>
__device__ __forceinline__ uint64_t make_desc_rows(uint32_t saddr) {
    static_assert(ROWB == 64 || ROWB == 128, "rows of 64 or 128 bytes");
    if constexpr (ROWB == 64) return make_desc_sw64(saddr);
    else return make_desc(saddr);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Operand lists of wgmma.mma_async.m64nNk16 for N = 16 k (k = 1..8): the N / 2 fp32 accumulators are operands %0 .. %(8k - 1),
// the A and B descriptors and the scale-d flag follow them.  WG_REGS_k extends WG_REGS_(k-1) by one group of eight.
#define WG_D8(g) "+f"(d[8 * g]), "+f"(d[8 * g + 1]), "+f"(d[8 * g + 2]), "+f"(d[8 * g + 3]), \
                 "+f"(d[8 * g + 4]), "+f"(d[8 * g + 5]), "+f"(d[8 * g + 6]), "+f"(d[8 * g + 7])
#define WG_OPS_1 WG_D8(0)
#define WG_OPS_2 WG_OPS_1, WG_D8(1)
#define WG_OPS_3 WG_OPS_2, WG_D8(2)
#define WG_OPS_4 WG_OPS_3, WG_D8(3)
#define WG_OPS_5 WG_OPS_4, WG_D8(4)
#define WG_OPS_6 WG_OPS_5, WG_D8(5)
#define WG_OPS_7 WG_OPS_6, WG_D8(6)
#define WG_OPS_8 WG_OPS_7, WG_D8(7)
#define WG_REGS_1 "%0,%1,%2,%3,%4,%5,%6,%7"
#define WG_REGS_2 WG_REGS_1 ",%8,%9,%10,%11,%12,%13,%14,%15"
#define WG_REGS_3 WG_REGS_2 ",%16,%17,%18,%19,%20,%21,%22,%23"
#define WG_REGS_4 WG_REGS_3 ",%24,%25,%26,%27,%28,%29,%30,%31"
#define WG_REGS_5 WG_REGS_4 ",%32,%33,%34,%35,%36,%37,%38,%39"
#define WG_REGS_6 WG_REGS_5 ",%40,%41,%42,%43,%44,%45,%46,%47"
#define WG_REGS_7 WG_REGS_6 ",%48,%49,%50,%51,%52,%53,%54,%55"
#define WG_REGS_8 WG_REGS_7 ",%56,%57,%58,%59,%60,%61,%62,%63"
// N, then the operand numbers of (A descriptor, B descriptor) and of the scale-d flag
#define WG_TAIL_1 "16", "%8, %9", "%10"
#define WG_TAIL_2 "32", "%16, %17", "%18"
#define WG_TAIL_3 "48", "%24, %25", "%26"
#define WG_TAIL_4 "64", "%32, %33", "%34"
#define WG_TAIL_5 "80", "%40, %41", "%42"
#define WG_TAIL_6 "96", "%48, %49", "%50"
#define WG_TAIL_7 "112", "%56, %57", "%58"
#define WG_TAIL_8 "128", "%64, %65", "%66"
#define WG_ASM_(TY, REGS, NS, AB, SC, ...)                                                                              \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " SC ", 0;\n\t"                                                    \
                 "wgmma.mma_async.sync.aligned.m64n" NS "k16.f32." TY "." TY " {" REGS "}, " AB ", p, 1, 1, 0, 0;\n\t}" \
                 : __VA_ARGS__ : "l"(ad), "l"(bd), "r"(accumulate))
#define WG_ASM(TY, REGS, TAIL, OPS) WG_ASM_(TY, REGS, TAIL, OPS)     // (one more expansion: TAIL and OPS split into their commas)
#define WG_CASE(k)                                                                                                 \
    if constexpr (N == 16 * k) {                                                                                   \
        if constexpr (BF16) WG_ASM("bf16", WG_REGS_##k, WG_TAIL_##k, WG_OPS_##k);                                  \
        else WG_ASM("f16", WG_REGS_##k, WG_TAIL_##k, WG_OPS_##k);                                                  \
    }

// D(64 x N) (+)= A(64 x 16) * B(N x 16)^T, both operands K-major in shared memory; fp32 accumulators.  ONE instruction for
// the whole width: B's N rows are 8-row atoms of 1024 B from `bd` on.  The m64nN fragment is the m64n16 fragments laid end
// to end: register 8j + 4i + e holds what register 4i + e of 16-column piece j would.
template <bool BF16, int N>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t ad, uint64_t bd, uint32_t accumulate) {
    static_assert(N % 16 == 0 && N >= 16 && N <= 128, "wgmma: N = 16, 32, ..., 128");
    WG_CASE(1) WG_CASE(2) WG_CASE(3) WG_CASE(4) WG_CASE(5) WG_CASE(6) WG_CASE(7) WG_CASE(8)
}
#undef WG_CASE
#undef WG_ASM
#undef WG_ASM_

// Accumulators of one warpgroup for an N-column tile: row half h (rows 64h..64h+63), fragment register r
template <int N> struct WgAcc { float d[2][N / 2]; };

// KS K steps of one 64-channel K block for H row halves (A descriptors a0, a1), issued as ONE straight run between its own
// wgmma.fence and commit_group: with no branch and no other register traffic inside the run, ptxas has no reason to inject
// warpgroup arrives or to serialise the MMAs.  `accumulate` == 0 starts the sums at zero with the first step.
template <bool BF16, int N, int H, int KS>
__device__ __forceinline__ void wg_mma_run(float (&d)[H][N / 2], uint64_t a0, uint64_t a1, uint64_t b0, uint32_t accumulate) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const uint32_t sc = (accumulate | (uint32_t)k) ? 1u : 0u;
        wgmma<BF16, N>(d[0], a0 + (uint64_t)(k * 2), b0 + (uint64_t)(k * 2), sc);
        if constexpr (H == 2) wgmma<BF16, N>(d[1], a1 + (uint64_t)(k * 2), b0 + (uint64_t)(k * 2), sc);
    }
    wg_commit();
}
// the run for the block's K step count (1..4; a ragged last block has fewer than 4)
template <bool BF16, int N, int H>
__device__ __forceinline__ void wg_mma_block(float (&d)[H][N / 2], uint64_t a0, uint64_t a1, uint64_t b0, int ksteps, uint32_t accumulate) {
    if (ksteps >= 4) wg_mma_run<BF16, N, H, 4>(d, a0, a1, b0, accumulate);
    else if (ksteps == 3) wg_mma_run<BF16, N, H, 3>(d, a0, a1, b0, accumulate);
    else if (ksteps == 2) wg_mma_run<BF16, N, H, 2>(d, a0, a1, b0, accumulate);
    else wg_mma_run<BF16, N, H, 1>(d, a0, a1, b0, accumulate);
}

// One K block (ksteps = 1..4 K steps) of a 128 x N tile: a_st / b_st are the block's operand bases (8-row atoms of 1024 B),
// B = rows 0..N-1 of the weight tile (rows past the valid columns zero-filled; their columns are never stored).  Called by
// all 128 threads of a warpgroup: one wgmma per row half and K step, fenced and committed (one group) here; the caller waits.
template <bool BF16, int N>
__device__ __forceinline__ void wg_mma_tile(WgAcc<N>& acc, uint32_t a_st, uint32_t b_st, int ksteps, uint32_t accumulate) {
    wg_mma_block<BF16, N, 2>(acc.d, make_desc(a_st), make_desc(a_st + 64 * 128), make_desc(b_st), ksteps, accumulate);
}

// One 64-row half on its own (kernels whose warpgroups split the M tiles of a CTA between them): D(64 x N) = A * B^T over
// `ksteps` K steps, 4 per 64-channel K block (one commit group each); a_kb / b_kb = byte distance between consecutive K
// blocks of A / B.  The caller waits.
template <bool BF16, int N>
__device__ __forceinline__ void wg_mma_m64(float (&d)[N / 2], uint32_t a_st, uint32_t a_kb, uint32_t b_st, uint32_t b_kb, int ksteps) {
    float (&d1)[1][N / 2] = *reinterpret_cast<float(*)[1][N / 2]>(&d);
    for (int kb = 0; kb * 4 < ksteps; ++kb)
        wg_mma_block<BF16, N, 1>(d1, make_desc(a_st + (uint32_t)kb * a_kb), 0, make_desc(b_st + (uint32_t)kb * b_kb), ksteps - 4 * kb, kb ? 1u : 0u);
}

// Fragments -> shared accumulator tile [column][kAccPitch] (fp32), all N columns.  `wt` = thread index inside the warpgroup.
// m64nN fragment: register 4i + {0,1} -> row 16 w + l/4, columns 8 i + 2 (l%4) + {0,1}; 4i + {2,3} -> row + 8
template <int N>
__device__ __forceinline__ void wg_acc_store(const WgAcc<N>& acc, uint32_t dst, int wt) {
    const int w = wt >> 5, l = wt & 31;
    const int r = 16 * w + (l >> 2), cq = 2 * (l & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < N / 8; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = 64 * h + r + (e >> 1) * 8, col = 8 * i + cq + (e & 1);
                asm volatile("st.shared.f32 [%0], %1;" ::"r"(dst + (uint32_t)(col * kAccPitch + row) * 4u), "f"(acc.d[h][4 * i + e]) : "memory");
            }
}

// fp32 -> bf16 hi + lo, x = hi + lo with hi = bf16(x), lo = bf16(x - hi) (|x - hi - lo| <= 2^-18 |x|), for the MMAs of the fp32
// parity kernels (pw_tc32_kernel, conv_igemm32_kernel)
__device__ __forceinline__ void split8(const float (&x)[8], uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __nv_bfloat162 hh = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
        const float2 hf = __bfloat1622float2(hh);
        const __nv_bfloat162 ll = __floats2bfloat162_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
        h[i] = *reinterpret_cast<const uint32_t*>(&hh);
        l[i] = *reinterpret_cast<const uint32_t*>(&ll);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// MMA widths the 1x1 kernels are instantiated for; a tile of n columns runs at the smallest one >= n (the extra B rows are
// zero-filled, the extra columns never stored)
__host__ __device__ constexpr int pw_mma_width(int n) { return n <= 64 ? (n + 15) & ~15 : n <= 96 ? 96 : 128; }

// Host: f(std::integral_constant<int, w>{}) when w is one of those widths and <= MAXW (only those are instantiated); else 1
template <int W, int MAXW, typename F>
int call_with_width(F& f) {
    if constexpr (W <= MAXW) return f(std::integral_constant<int, W>{});
    else return 1;
}
template <int MAXW, typename F>
int with_mma_width(int w, F&& f) {
    switch (w) {
        case 16: return call_with_width<16, MAXW>(f);
        case 32: return call_with_width<32, MAXW>(f);
        case 48: return call_with_width<48, MAXW>(f);
        case 64: return call_with_width<64, MAXW>(f);
        case 96: return call_with_width<96, MAXW>(f);
        case 128: return call_with_width<128, MAXW>(f);
    }
    return 1;
}

// 16 consecutive columns of one accumulator row from the shared accumulator tile
__device__ __forceinline__ void acc_ld16(uint32_t base, int row, int c0, float (&v)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i)
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[i]) : "r"(base + (uint32_t)((c0 + i) * kAccPitch + row) * 4u));
}

template <typename T> __device__ __forceinline__ uint4 scale8(uint4 raw, const float* g);
template <> __device__ __forceinline__ uint4 scale8<__nv_bfloat16>(uint4 raw, const float* g) {
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&raw);
    const float4 g0 = *reinterpret_cast<const float4*>(g), g1 = *reinterpret_cast<const float4*>(g + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 f = __bfloat1622float2(h[i]);
        h[i] = __floats2bfloat162_rn(f.x * gg[2 * i], f.y * gg[2 * i + 1]);
    }
    return raw;
}
template <> __device__ __forceinline__ uint4 scale8<__half>(uint4 raw, const float* g) {
    __half2* h = reinterpret_cast<__half2*>(&raw);
    const float4 g0 = *reinterpret_cast<const float4*>(g), g1 = *reinterpret_cast<const float4*>(g + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 f = __half22float2(h[i]);
        h[i] = __floats2half2_rn(f.x * gg[2 * i], f.y * gg[2 * i + 1]);
    }
    return raw;
}

// ----------------------------------------------------------------------------- pw_tc2: cp.async ring
// pw_tc2_kernel: one 128-pixel x n_tile(<=256) output tile per CTA, K in blocks of 64 channels:
//   * operand K blocks travel global -> shared with cp.async (16 B, zero-fill for tails) through a ring of
//     n_stages stages, several blocks in flight, no register staging;
//   * the SE gate is applied IN shared memory by the thread that copied the chunk (so no extra barrier):
//       GATE == 1: on the A rows (tiles may span up to four crops; their gate rows sit in smem)
//       GATE == 2: on the W rows (per-crop tiling: a tile never leaves its crop, used while H*W >= 784)
//   * stage reuse waits for the wgmma group of the block that last read the stage.
// exact floor(x / d) for small non-negative ints (x < 2^17, d < 2^8) with inv = 1.0f / d: (x + 0.5) / d is at least 0.5 / d
// away from every integer, far more than the float rounding error - replaces the ~20-instruction integer division
__device__ __forceinline__ int fdiv_small(int x, float inv) { return __float2int_rz(((float)x + 0.5f) * inv); }
__device__ __forceinline__ void cp_async16_z(uint32_t dst, const void* src, bool valid) {
    const uint32_t sz = valid ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128_(uint32_t addr, const uint4& v) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
template <typename T> __device__ __forceinline__ uint4 scale8s(uint4 raw, uint32_t gaddr);   // gate values from smem
template <> __device__ __forceinline__ uint4 scale8s<__nv_bfloat16>(uint4 raw, uint32_t gaddr) {
    float4 g0, g1;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(g0.x), "=f"(g0.y), "=f"(g0.z), "=f"(g0.w) : "r"(gaddr));
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(g1.x), "=f"(g1.y), "=f"(g1.z), "=f"(g1.w) : "r"(gaddr + 16));
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&raw);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 f = __bfloat1622float2(h[i]);
        h[i] = __floats2bfloat162_rn(f.x * gg[2 * i], f.y * gg[2 * i + 1]);
    }
    return raw;
}
template <> __device__ __forceinline__ uint4 scale8s<__half>(uint4 raw, uint32_t gaddr) {
    float4 g0, g1;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(g0.x), "=f"(g0.y), "=f"(g0.z), "=f"(g0.w) : "r"(gaddr));
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(g1.x), "=f"(g1.y), "=f"(g1.z), "=f"(g1.w) : "r"(gaddr + 16));
    __half2* h = reinterpret_cast<__half2*>(&raw);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 f = __half22float2(h[i]);
        h[i] = __floats2half2_rn(f.x * gg[2 * i], f.y * gg[2 * i + 1]);
    }
    return raw;
}

// OUT_H: the result is written as fp16 whatever T is (the expand conv feeding the HFMA2 depthwise kernel KD)
// UN: MMA width (pw_mma_width(n_tile)): rows of the W stage, columns of the accumulator tile
template <typename T, bool SWISH, int GATE, bool RESID, bool OUT_H, int UN>
__global__ void __launch_bounds__(128) pw_tc2_kernel(const T* __restrict__ A, const T* __restrict__ Wt,
                                                     const float* __restrict__ bias, const float* __restrict__ gate,
                                                     const T* __restrict__ resid, T* __restrict__ out,
                                                     int M, int K, int N, int hw,
                                                     int n_tile, int n_stages,
                                                     int tiles_per_crop) {    // GATE == 2 only
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    extern __shared__ uint8_t smem_raw[];

    const int tid = threadIdx.x;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr int w_stage_bytes = UN * BK * 2;
    const uint32_t stage_bytes = A_STAGE_BYTES + w_stage_bytes;
    const uint32_t sG = smem0 + n_stages * stage_bytes;          // gate rows: [<=4 crops][K] fp32 (GATE only)

    // ---- tile -> rows
    int m0, rows_valid, crop0;
    if (GATE == 2) {
        const int crop = blockIdx.y / tiles_per_crop, t = blockIdx.y - crop * tiles_per_crop;
        m0 = crop * hw + t * BM;
        rows_valid = min(BM, hw - t * BM);
        crop0 = crop;
    } else {
        m0 = blockIdx.y * BM;
        rows_valid = min(BM, M - m0);
        crop0 = GATE ? m0 / hw : 0;
    }
    const int n0 = blockIdx.x * n_tile;
    const int n_valid = min(n_tile, N - n0);
    const int nkb = (K + BK - 1) / BK;
    const int kchunks = K >> 3;

    // gate rows of the crops this tile touches -> smem (joins the first cp.async group)
    if (GATE) {
        const int ncrops = GATE == 2 ? 1 : ((m0 + rows_valid - 1) / hw - crop0 + 1);
        const int q = K >> 2;
        for (int idx = tid; idx < ncrops * q; idx += 128) {
            const int cr = idx / q, j = idx - cr * q;
            cp_async16_z(sG + (uint32_t)(cr * K + j * 4) * 4, gate + (long long)(crop0 + cr) * K + j * 4, true);
        }
    }
    auto fill = [&](int kb) {
        const int s = kb % n_stages;
        const uint32_t a_st = smem0 + s * stage_bytes, w_st = a_st + A_STAGE_BYTES;
        const int kc0 = kb * 8;
        const int cb = min(8, kchunks - kc0), cbp = (cb + 1) & ~1;
        if (cbp == 8) {
            // full block: item idx = tid + i*128 -> row tid/8 + 16 i, chunk tid%8 (no divisions in the hot loop)
            const int c = tid & 7, r0 = tid >> 3;
            const bool cvalid = c < cb;
            const T* asrc = A + (long long)(m0 + r0) * K + (kc0 + c) * 8;
            const uint32_t swz = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const bool valid = cvalid && (r0 + 16 * i) < rows_valid;
                cp_async16_z(a_st + swz + i * 2048, valid ? asrc + (long long)i * 16 * K : A, valid);
            }
            const T* wsrc = Wt + (long long)(n0 + r0) * K + (kc0 + c) * 8;
#pragma unroll
            for (int i = 0; i < UN / 16; ++i) {
                const int r = r0 + 16 * i;
                const bool valid = cvalid && r < n_valid;
                cp_async16_z(w_st + swz + i * 2048, valid ? wsrc + (long long)i * 16 * K : Wt, valid);
            }
            return;
        }
        for (int idx = tid; idx < BM * cbp; idx += 128) {
            const int r = fdiv_small(idx, 1.0f / (float)cbp), c = idx - r * cbp;
            const bool valid = r < rows_valid && c < cb;
            cp_async16_z(a_st + (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4),
                         valid ? A + (long long)(m0 + r) * K + (kc0 + c) * 8 : A, valid);
        }
        for (int idx = tid; idx < UN * cbp; idx += 128) {
            const int r = fdiv_small(idx, 1.0f / (float)cbp), c = idx - r * cbp;
            const bool valid = r < n_valid && c < cb;
            cp_async16_z(w_st + (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4),
                         valid ? Wt + (long long)(n0 + r) * K + (kc0 + c) * 8 : Wt, valid);
        }
    };
    for (int j = 0; j < n_stages; ++j) {
        if (j < nkb) fill(j);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    WgAcc<UN> acc;

    // GATE == 1: byte offset of the gate row (crop) of each of the 8 rows this thread rescales, fixed for the whole K loop
    uint32_t g_row[8];
    if (GATE == 1) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = (tid >> 3) + 16 * i;
            g_row[i] = r < rows_valid ? (uint32_t)(((m0 + r) / hw - crop0) * K) * 4u : 0u;
        }
    }
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % n_stages;
        const uint32_t a_st = smem0 + s * stage_bytes, w_st = a_st + A_STAGE_BYTES;
        // groups committed so far: n_stages + kb ; block kb sits in group kb (kb < n_stages) or kb+1 -> allow n_stages-2 pending
        if (n_stages >= 4) asm volatile("cp.async.wait_group 2;" ::: "memory");
        else if (n_stages == 3) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        if (GATE) {
            // the gate rows in sG were copied by ALL threads (group 0): one CTA barrier before their first use.
            // The operand chunks themselves need none: each thread rescales exactly the chunks it copied itself.
            if (kb == 0) __syncthreads();
            const int kc0 = kb * 8;
            const int cb = min(8, kchunks - kc0), cbp = (cb + 1) & ~1;
            if (GATE == 1) {
                if (cbp == 8) {
                    const int c = tid & 7, r0 = tid >> 3;
                    if (c < cb) {
                        const uint32_t a0 = a_st + (r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4);
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            if (r0 + 16 * i < rows_valid)
                                sts128_(a0 + i * 2048, scale8s<T>(lds128(a0 + i * 2048), sG + g_row[i] + (uint32_t)((kc0 + c) * 8) * 4));
                        }
                    }
                } else {
                    for (int idx = tid; idx < BM * cbp; idx += 128) {
                        const int r = fdiv_small(idx, 1.0f / (float)cbp), c = idx - r * cbp;
                        if (r < rows_valid && c < cb) {
                            const uint32_t addr = a_st + (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4);
                            const int cr = (m0 + r) / hw - crop0;
                            sts128_(addr, scale8s<T>(lds128(addr), sG + (uint32_t)(cr * K + (kc0 + c) * 8) * 4));
                        }
                    }
                }
            } else {
                if (cbp == 8) {
                    const int c = tid & 7, r0 = tid >> 3;
                    if (c < cb)
                        for (int r = r0, i = 0; r < n_valid; r += 16, ++i) {
                            const uint32_t addr = w_st + (r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4) + i * 2048;
                            sts128_(addr, scale8s<T>(lds128(addr), sG + (uint32_t)((kc0 + c) * 8) * 4));
                        }
                } else {
                    for (int idx = tid; idx < UN * cbp; idx += 128) {
                        const int r = fdiv_small(idx, 1.0f / (float)cbp), c = idx - r * cbp;
                        if (r < n_valid && c < cb) {
                            const uint32_t addr = w_st + (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4);
                            sts128_(addr, scale8s<T>(lds128(addr), sG + (uint32_t)((kc0 + c) * 8) * 4));
                        }
                    }
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        {
            const int krem = min(BK, K - kb * BK);
            wg_mma_tile<BF16, UN>(acc, a_st, w_st, (krem + 15) >> 4, kb ? 1u : 0u);     // one commit group per K block
        }
        // refill the stage block kb-1 used with block kb-1+n_stages once its MMAs have completed (every thread's group)
        if (kb >= 1 && kb - 1 + n_stages < nkb) {
            wg_wait<1>();
            __syncthreads();
            fill(kb - 1 + n_stages);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    wg_wait<0>();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    // the operand ring is free: accumulators -> shared accumulator tile at smem0, the 16-bit output stage after it
    const uint32_t sAcc = smem0;
    wg_acc_store<UN>(acc, sAcc, tid);
    __syncthreads();

    // ---- epilogue: TMEM -> +shift, swish, +residual -> 16-bit -> stage -> coalesced stores
    const int nch = n_valid >> 3;
    const float inv_nch = 1.0f / (float)(nch > 0 ? nch : 1);
    const int pitch16 = nch | 1;
    uint4* stage = reinterpret_cast<uint4*>(smem_raw + (smem0 + acc_tile_bytes(UN) - smem_u32(smem_raw)));
    const bool row_ok = tid < rows_valid;
    const long long m = (long long)m0 + tid;
    {
        for (int c0 = 0; c0 < n_valid; c0 += 16) {
            float v[16];
            acc_ld16(sAcc, tid, c0, v);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + c0 + h * 8;
                if (c0 + h * 8 >= n_valid) break;
                float o[8];
                const float4 b0 = *reinterpret_cast<const float4*>(bias + n), b1 = *reinterpret_cast<const float4*>(bias + n + 4);
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float x = v[h * 8 + j] + bb[j];
                    o[j] = SWISH ? swish_fast(x) : x;
                }
                if (RESID && row_ok) {
                    float r[8];
                    ld8<T>(resid + m * N + n, r);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += r[j];
                }
                if (OUT_H) st8<__half>(reinterpret_cast<__half*>(stage + tid * pitch16 + ((c0 >> 3) + h)), o);
                else st8<T>(reinterpret_cast<T*>(stage + tid * pitch16 + ((c0 >> 3) + h)), o);
            }
        }
    }
    __syncthreads();
    for (int idx = tid; idx < rows_valid * nch; idx += 128) {
        const int r = fdiv_small(idx, inv_nch), j = idx - r * nch;
        *reinterpret_cast<uint4*>(out + ((long long)m0 + r) * N + n0 + j * 8) = stage[r * pitch16 + j];
    }
}

template <typename T>
int launch_pw_tc2(cudaStream_t stream, const T* A, const void* Wt16, const float* bias, const float* gate, const T* resid,
                  T* out, long long M, int K, int N, int hw, bool swish, int stage_cap = 0, int smem_budget_kb = 54, int min_ctas = 264,
                  bool out_half = false) {
    if (sizeof(T) != 2) return 1;
    if ((K & 7) || (N & 7) || M > 0x7fffffffLL) return 1;
    const bool per_crop = gate && hw >= 784;                 // gate on W, tiles stay inside a crop
    const int tpc = (hw + BM - 1) / BM;
    const long long m_tiles = per_crop ? (M / hw) * tpc : (M + BM - 1) / BM;
    // at most 128 columns per tile: the warpgroup holds the whole 128 x n_tile accumulator in registers (n_tile per thread)
    int n_tile = N;
    if (N > 128) {
        int parts = (N + 127) / 128;
        while (true) {
            n_tile = ((N + parts - 1) / parts + 15) & ~15;
            if (n_tile <= 128) break;
            ++parts;
        }
    }
    while (n_tile > 48 && m_tiles * ((N + n_tile - 1) / n_tile) < min_ctas) {
        const int parts = (N + n_tile - 1) / n_tile + 1;
        const int nt = ((N + parts - 1) / parts + 15) & ~15;
        if (nt >= n_tile) break;
        n_tile = nt;
    }
    const int umma_n = pw_mma_width(n_tile);
    const int nkb = (K + BK - 1) / BK;
    const size_t stage_bytes = A_STAGE_BYTES + (size_t)umma_n * BK * 2;
    const int gate_crops = per_crop ? 1 : std::min(4, (BM - 1) / hw + 2);      // crops one 128-row tile can touch
    const size_t gate_bytes = gate ? (size_t)gate_crops * K * 4 : 0;
    const size_t out_bytes = acc_tile_bytes(umma_n) + (size_t)BM * ((size_t)(n_tile >> 3) | 1) * 16;     // accumulator tile + output stage
    int n_stages = nkb < 4 ? nkb : 4;
    if (stage_cap > 0 && n_stages > stage_cap) n_stages = stage_cap;
    // a grid that does not even fill the SMs once (single-crop latency path) gains nothing from co-residency: deepest ring
    if (m_tiles * ((N + n_tile - 1) / n_tile) < 132) smem_budget_kb = 180;
    // ring depth vs co-residency: a shallower ring lets more CTAs share the SM (budget = smem per CTA)
    while (n_stages > 2 && n_stages * stage_bytes + gate_bytes > (size_t)smem_budget_kb * 1024) --n_stages;
    size_t smem = n_stages * stage_bytes + gate_bytes;
    if (smem < out_bytes) smem = out_bytes;
    smem += 1024;
    if (smem > 225 * 1024) return 1;
    dim3 grid((unsigned)((N + n_tile - 1) / n_tile), (unsigned)m_tiles);
    const T* W = reinterpret_cast<const T*>(Wt16);
#define TC2(SW, GA, RE, OH)                                                                                              \
    return with_mma_width<128>(umma_n, [&](auto un) {                                                                         \
        auto kfn = pw_tc2_kernel<T, SW, GA, RE, OH, decltype(un)::value>;                                                \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024) != cudaSuccess) return -1; \
        kfn<<<grid, 128, smem, stream>>>(A, W, bias, gate, resid, out, (int)M, K, N, hw, n_tile, n_stages, tpc);         \
        return 0;                                                                                                        \
    })
    if (out_half && !(swish && !gate && !resid)) return 1;
    if (swish && !gate && !resid) { if (out_half) TC2(true, 0, false, true); else TC2(true, 0, false, false); }
    else if (!swish && !gate && !resid) TC2(false, 0, false, false);
    else if (!swish && !gate && resid) TC2(false, 0, true, false);           // project conv whose input K1 has already gated
    else if (!swish && gate && !resid) { if (per_crop) TC2(false, 2, false, false); else TC2(false, 1, false, false); }
    else if (!swish && gate && resid) { if (per_crop) TC2(false, 2, true, false); else TC2(false, 1, true, false); }
#undef TC2
    return 1;
}


// ----------------------------------------------------------------------------- pw_tc3: gated projects of the large maps
// The gated project convs of blocks 1-5 are streams of tiny GEMMs (K = 32..144, N = 16..40, millions of rows): with one 128-row
// tile per CTA (pw_tc2) every tile pays the gate row, the W copy + its rescale and a cold load -> MMA -> epilogue chain.
// Here a CTA walks `tpc` consecutive tiles of ONE crop: gate row and W' = bf16(W * g) once per CTA (the same scale8s and the
// same wgmma sequence as pw_tc2's per-crop route, so the results are bit-identical); the cp.async of tile t+1 runs under the
// MMA and the epilogue of tile t.
// UN = the plan's umma_n (N rounded up to 16): rows of the resident W, MMA width
template <typename T, bool RESID, int UN>
__global__ void __launch_bounds__(128) pw_tc3_kernel(const T* __restrict__ A, const T* __restrict__ Wt, const float* __restrict__ bias,
                                                     const float* __restrict__ gate, const T* __restrict__ resid, T* __restrict__ out,
                                                     int K, int N, int hw, int tiles_per_crop, int tpc, int groups) {
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    constexpr int umma_n = UN;
    extern __shared__ uint8_t smem_raw[];
    const int tid = threadIdx.x;
    const int nkb = (K + BK - 1) / BK, kchunks = K >> 3;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_bytes = (uint32_t)nkb * umma_n * 128, a_bytes = (uint32_t)nkb * A_STAGE_BYTES;
    const uint32_t sW = smem0, sA = sW + ((w_bytes + 1023u) & ~1023u), sG = sA + 2 * a_bytes;
    const uint32_t sAcc = sG + (((uint32_t)K * 4 + 15u) & ~15u);
    const int nch = N >> 3, pitch16 = nch | 1;
    uint4* stage = reinterpret_cast<uint4*>(smem_raw + (sAcc + acc_tile_bytes(umma_n) - smem_u32(smem_raw)));
    const float inv_nch = 1.0f / (float)nch;

    const int crop = blockIdx.x / groups, g = blockIdx.x - crop * groups;
    const int t_begin = g * tpc, t_end = min(tiles_per_crop, t_begin + tpc);
    if (t_begin >= t_end) return;

    // one K block of an operand: 16-byte chunk c of rows r0, r0+16, ... (the mapping pw_tc2 uses; ragged last block: zero fill)
    auto fill_rows = [&](uint32_t dst, const T* src0, int rows, int kb) {
        const int kc0 = kb * 8;
        const int cb = min(8, kchunks - kc0);
        const int c = tid & 7, r0 = tid >> 3;
        const uint32_t swz = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));
        const T* src = src0 + (long long)r0 * K + (kc0 + c) * 8;
        for (int r = r0, i = 0; r < rows; r += 16, ++i)
            cp_async16_z(dst + swz + i * 2048, c < cb ? src + (long long)i * 16 * K : src0, c < cb);
    };
    auto fill_a = [&](int t, int buf) {
        const int rows_valid = min(BM, hw - t * BM);
        const T* a0 = A + ((long long)crop * hw + (long long)t * BM) * K;
        for (int kb = 0; kb < nkb; ++kb) {
            const int kc0 = kb * 8;
            const int cb = min(8, kchunks - kc0);
            const int c = tid & 7, r0 = tid >> 3;
            const uint32_t dst = sA + buf * a_bytes + kb * A_STAGE_BYTES + (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4));
            const T* src = a0 + (long long)r0 * K + (kc0 + c) * 8;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const bool valid = c < cb && (r0 + 16 * i) < rows_valid;
                cp_async16_z(dst + i * 2048, valid ? src + (long long)i * 16 * K : A, valid);
            }
        }
    };
    {   // gate row of this crop, the whole W, the first A tile
        const int q = K >> 2;
        for (int idx = tid; idx < q; idx += 128) cp_async16_z(sG + (uint32_t)idx * 16, gate + (long long)crop * K + idx * 4, true);
        for (int kb = 0; kb < nkb; ++kb) fill_rows(sW + (uint32_t)kb * umma_n * 128, Wt, umma_n <= N ? umma_n : N, kb);
        if (umma_n > N) {       // rows N..umma_n-1 of W (padding of the MMA's N): zeros
            const uint4 z = make_uint4(0u, 0u, 0u, 0u);
            for (int kb = 0; kb < nkb; ++kb)
                for (int idx = tid; idx < (umma_n - N) * 8; idx += 128) {
                    const int r = N + (idx >> 3), c = idx & 7;
                    sts128_(sW + (uint32_t)kb * umma_n * 128 + (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4)), z);
                }
        }
        fill_a(t_begin, 0);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                         // gate row (copied by all threads) visible
        // W' = 16-bit(W * g): each thread rescales exactly the chunks it copied
        for (int kb = 0; kb < nkb; ++kb) {
            const int kc0 = kb * 8;
            const int cb = min(8, kchunks - kc0);
            const int c = tid & 7, r0 = tid >> 3;
            if (c < cb)
                for (int r = r0, i = 0; r < N; r += 16, ++i) {
                    const uint32_t addr = sW + (uint32_t)kb * umma_n * 128 + (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((c ^ (r0 & 7)) << 4)) + i * 2048;
                    sts128_(addr, scale8s<T>(lds128(addr), sG + (uint32_t)((kc0 + c) * 8) * 4));
                }
        }
    }
    auto epilogue = [&](int t) {
        const int rows_valid = min(BM, hw - t * BM);
        const long long m0 = (long long)crop * hw + (long long)t * BM;
        const bool row_ok = tid < rows_valid;
        for (int c0 = 0; c0 < N; c0 += 16) {
            float v[16];
            acc_ld16(sAcc, tid, c0, v);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = c0 + h * 8;
                if (n >= N) break;
                float o[8];
                const float4 b0 = *reinterpret_cast<const float4*>(bias + n), b1 = *reinterpret_cast<const float4*>(bias + n + 4);
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = v[h * 8 + j] + bb[j];
                if (RESID && row_ok) {
                    float r[8];
                    ld8<T>(resid + (m0 + tid) * N + n, r);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += r[j];
                }
                st8<T>(reinterpret_cast<T*>(stage + tid * pitch16 + ((c0 >> 3) + h)), o);
            }
        }
        __syncthreads();
        for (int idx = tid; idx < rows_valid * nch; idx += 128) {
            const int r = fdiv_small(idx, inv_nch), j = idx - r * nch;
            *reinterpret_cast<uint4*>(out + (m0 + r) * N + j * 8) = stage[r * pitch16 + j];
        }
    };

    const int ntiles = t_end - t_begin;
    WgAcc<UN> acc;
    for (int it = 0; it < ntiles; ++it) {
        const int t = t_begin + it, buf = it & 1;
        asm volatile("cp.async.wait_group 0;" ::: "memory");            // A(t) has landed (this thread's part)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();                                                // ... everyone's; the store loop of tile t-1 is done with `stage`
        for (int kb = 0; kb < nkb; ++kb) {
            const int krem = min(BK, K - kb * BK);
            wg_mma_tile<BF16, UN>(acc, sA + buf * a_bytes + kb * A_STAGE_BYTES, sW + (uint32_t)kb * umma_n * 128, (krem + 15) >> 4, kb ? 1u : 0u);
        }
        // A buffer buf ^ 1 was read by the MMA of tile t-1, which has completed
        if (it + 1 < ntiles) fill_a(t + 1, buf ^ 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        wg_wait<0>();
        wg_acc_store<UN>(acc, sAcc, tid);
        __syncthreads();
        epilogue(t);
    }
}

// Which gated projects pw_tc3 takes and how it walks them (host-side, tested without a GPU by tests/test_route_plans.py).
struct Pw3Plan { int tiles_per_crop, tpc, groups, umma_n; size_t smem; };
inline bool plan_pw_tc3(long long M, int K, int N, int hw, bool has_gate, Pw3Plan* pl) {
    // K <= 64 (one K block): the larger K of blocks 2-4 need two or three A blocks per buffer and lose co-residency
    if (!has_gate || hw < 784 || (K & 7) || (N & 7) || K > 64 || N > 64 || M < 1 || M % hw) return false;
    const int crops = (int)(M / hw);
    pl->tiles_per_crop = (hw + BM - 1) / BM;
    int groups = (1536 + crops - 1) / crops;                      // enough CTAs for ~10 per SM
    if (groups > pl->tiles_per_crop) groups = pl->tiles_per_crop;
    if (groups < 1) groups = 1;
    pl->tpc = (pl->tiles_per_crop + groups - 1) / groups;
    pl->groups = (pl->tiles_per_crop + pl->tpc - 1) / pl->tpc;
    if (pl->tpc < 3) return false;                                // nothing to pipeline
    pl->umma_n = (N + 15) & ~15;
    const int nkb = (K + BK - 1) / BK;
    const size_t w_bytes = ((size_t)nkb * pl->umma_n * 128 + 1023) & ~(size_t)1023;
    pl->smem = w_bytes + 2 * (size_t)nkb * A_STAGE_BYTES + (((size_t)K * 4 + 15) & ~(size_t)15) + acc_tile_bytes(pl->umma_n) + (size_t)BM * ((size_t)(N >> 3) | 1) * 16 + 1024;
    return pl->smem <= 200 * 1024;
}

// 0 = launched; 1 = shape not covered (caller falls back to pw_tc2)
template <typename T>
int launch_pw_tc3(cudaStream_t stream, const T* A, const void* Wt16, const float* bias, const float* gate, const T* resid, T* out,
                  long long M, int K, int N, int hw) {
    Pw3Plan pl{};
    if (sizeof(T) != 2 || !plan_pw_tc3(M, K, N, hw, gate != nullptr, &pl)) return 1;
    const int crops = (int)(M / hw);
    const int tiles_per_crop = pl.tiles_per_crop, tpc = pl.tpc, groups = pl.groups;
    const size_t smem = pl.smem;
    const T* W = reinterpret_cast<const T*>(Wt16);
    // umma_n <= 64: a multiple of 16, so pw_mma_width(umma_n) == umma_n
    return with_mma_width<64>(pl.umma_n, [&](auto un) {
        auto kfn = resid ? pw_tc3_kernel<T, true, decltype(un)::value> : pw_tc3_kernel<T, false, decltype(un)::value>;
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) return -1;
        kfn<<<crops * groups, 128, smem, stream>>>(A, W, bias, gate, resid, out, K, N, hw, tiles_per_crop, tpc, groups);
        return 0;
    });
}

}  // namespace tc
}  // namespace whenet
