// kernels_k1w.cuh - K1W: weight-stationary, persistent, warp-specialised front half of an MBConv block.
//
//   expand 1x1 (warpgroup MMA, fp32 accumulators in registers) -> + BN shift -> swish -> 16-bit E tile in shared memory
//   -> depthwise KSxKS stride S, TF-SAME (HFMA2 on the E tile) -> + BN shift -> swish
//   -> D (global, 16-bit) + deterministic SE squeeze partial sums
//
// Same arithmetic as K1 (kernels_fused.cuh), different machine mapping.  K1 gives one CTA one tile and walks its phases
// behind CTA-wide barriers, which leaves the late blocks latency-bound (one 512-thread CTA per SM, 6-18 serial chunks per
// crop).  K1W instead:
//
//   * a CTA owns ONE chunk of CC expanded channels for the whole launch: its slice of the expand weights (TMA, once), its
//     BN shifts and its depthwise constants stay in shared memory ("weight stationary"), and it loops over ITEMS
//     = (crop [pair], output tile); grid = n_chunks x groups <= #SMs, items are dealt round-robin to the groups;
//   * the halo tile of the block INPUT of an item arrives by ONE TMA box per 64-channel K block
//     (cp.async.bulk.tensor.4d over the NHWC tensor, SWIZZLE_128B = the wgmma K-major operand layout, rows = halo
//     pixels in raster order).  Out-of-image halo pixels and channels past Cin are zero-filled by the TMA unit, so
//     TF-SAME padding and K padding cost no instructions;
//   * warp roles, connected by mbarriers (no CTA-wide barrier in the item loop):
//       warp 0            TMA producer   A ring (NA stages)
//       warps 2-3         reducer        fixed-order column sums of the depthwise lanes' squeeze partials -> global
//       last E warps      MMA + epilogue wgmma of (64-row half, 16 columns) pieces, round-robin over the epilogue warpgroups
//                                        -> +shift -> swish -> 16-bit -> E ring (2 deep); rows outside the image -> 0
//       remaining warps   depthwise      E -> k x k HFMA2 -> +shift, swish -> D; per-lane squeeze sums -> smem ring
//     Registers follow the roles (setmaxnreg): 48 for the control group, 72-80 for the epilogue, 88-96 for the depthwise
//     warps, which lets 12-16 of them run beside 4-8 epilogue warps in one 768-thread CTA.
//     so the MMA + SFU-bound epilogue of item i+1, the FMA-bound depthwise of item i and the TMA unit all run at the same time.
//
// E row index == GEMM row index == raster index of the halo pixel, so neither the epilogue nor the depthwise needs
// a division to find its data.  Every mbarrier wait is bounded (flag in mapped host memory + fast exit).
#pragma once
#include <cuda.h>

#include "kernels_fused.cuh"

namespace whenet {
namespace fused {

struct alignas(64) K1WParams {
    CUtensorMap tmA;       // block input  [N][Hin][Hin][Cin]  (dims innermost first: C, W, H, N), box {64, IW, IH, NB}, SWIZZLE_128B
    CUtensorMap tmW;       // 0.5 * BN-folded expand weights [Cexp][Cin] K-major, box {64, CC}, SWIZZLE_128B
    const float* shift;    // [Cexp]        0.5 * BN shift of the expand conv
    const void* w_dw16;    // half [KS*KS][Cexp] 0.5 * BN-folded depthwise weights / kDwScale (HFMA2 depthwise, see kernels_fused.cuh)
    const float* b_dw;     // [Cexp]        0.5 * BN shift of the depthwise conv
    void* out;             // T [N][Ho][Ho][Cexp]
    float* partial;        // [N][tiles][Cexp]
    int* tflag;            // mbarrier-timeout flag (mapped pinned host memory)
    long long* trace;      // NULL, or [grid][16] cycle counters: where each role of each CTA waited (tools/k1w_trace.py)
    int Hin, Ho, Cin, Cexp, pad;
    int TH, TW, IH, IW, tiles_x, tiles;
    int NB;                // crops per item (> 1 only when one tile is the whole image)
    int N, items;          // crops in this launch, items = ceil(N / NB) * tiles
    int CC, n_chunks, groups;
    int nkb;               // 64-channel K blocks of the input
    int ksteps;            // K = 16 MMA steps = ceil(Cin / 16)
    int mtiles;            // 128-row GEMM tiles of one item
    int rows;              // GEMM rows of one item = NB * IH * IW
    int rows_alloc;        // A rows per K block in shared memory (rows rounded up to 8)
    int pitchE;            // bytes per E row = CC * 2 + 16
    int e_rows;            // E rows per crop (IH * IW + slack for ragged strips)
    int NA;                // A ring depth (1 or 2)
    int n_epi;             // epilogue warps: 4 or 8 (one or two warpgroups)
    int n_dw;              // depthwise threads
    int PY, PYc;           // strip lanes (all crops of the item / per crop)
    int spr_log2;          // log2(strips per output row)
    uint32_t a_stage, a_tx, w_tx;               // bytes of one A stage, of its TMA transactions, of the W chunk
    uint32_t off_w, off_c, off_e, e_buf, off_r;  // shared-memory offsets from the 1024-aligned base (A is at 0)
};

namespace k1w {

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
            "K1W_POLL_%=:\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "@p bra K1W_DONE_%=;\n\t"
            "sub.u32 n, n, 1;\n\t"
            "setp.ne.u32 p, n, 0;\n\t"
            "@p bra K1W_POLL_%=;\n\t"
            "setp.eq.u32 p, n, 1;\n"          // false: n == 0 here
            "K1W_DONE_%=:\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar_addr), "r"(parity) : "memory");
        if (done) return;
        if (*abort_flag) return;
    }
    *abort_flag = 1;
    *reinterpret_cast<volatile int*>(tflag) = 1;
}
// the same with the cycles spent waiting added to `acc` (trace builds of the roles' lane 0)
__device__ __forceinline__ void wait_t(uint32_t bar_addr, uint32_t parity, volatile int* abort_flag, int* tflag, bool tr, long long& acc) {
    if (!tr) { wait(bar_addr, parity, abort_flag, tflag); return; }
    const long long t0 = clock64();
    wait(bar_addr, parity, abort_flag, tflag);
    acc += clock64() - t0;
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
// two fp32 adds on a channel pair
__device__ __forceinline__ float2 fadd2(const float2& a, const float2& b) { return make_float2(a.x + b.x, a.y + b.y); }
// swish of two values that are already x/2: h + h * tanh(h)
__device__ __forceinline__ float2 swish2_from_half(const float2& h) {
    float2 t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t.x) : "f"(h.x));
    asm("tanh.approx.f32 %0, %1;" : "=f"(t.y) : "f"(h.y));
    float2 d = h;
    ffma2(d, h, t);
    return d;
}

constexpr int kCtrlThreads = 128;      // warps 0-3: TMA producer, MMA issuer, two idle warps (the epilogue must start on a
                                       // warp whose index is a multiple of 4: TMEM lane quadrant = warp & 3)
}  // namespace k1w

// Items of one CTA: item = group + k * groups, decomposed into (crop block q, tile t) without a division per step.
struct ItemIter {
    int item, q, t, dq, dt, tiles, step;
    __device__ __forceinline__ void init(int group, int groups, int tiles_) {
        tiles = tiles_; step = groups; item = group;
        q = group / tiles_; t = group - q * tiles_;
        dq = groups / tiles_; dt = groups - dq * tiles_;
    }
    __device__ __forceinline__ void next() {
        item += step; q += dq; t += dt;
        if (t >= tiles) { t -= tiles; ++q; }
    }
};

constexpr int kK1WThreads = 768;       // six warpgroups: control | EPI_WG x epilogue | (5 - EPI_WG) x depthwise

template <typename T, int KS, int S, int R, int EPI_WG>
__global__ void __maxnreg__(80) k1w_kernel(const __grid_constant__ K1WParams p) {
    extern __shared__ uint8_t smem_raw[];
    // [0,1] a_full  [2,3] a_empty  [8,9] e_full  [10,11] e_empty  [12] w  [13,14] r_full  [15,16] r_empty
    __shared__ __align__(8) uint64_t bars[17];
    __shared__ int s_abort_mem;
    volatile int* s_abort = &s_abort_mem;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t smem0 = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem0, sW = smem0 + p.off_w, sC = smem0 + p.off_c, sE = smem0 + p.off_e, sR = smem0 + p.off_r;
    const uint32_t bar0 = tc::smem_u32(&bars[0]);
    const uint32_t b_a_full = bar0, b_a_empty = bar0 + 16, b_e_full = bar0 + 64,
                   b_e_empty = bar0 + 80, b_w = bar0 + 96, b_r_full = bar0 + 104, b_r_empty = bar0 + 120;
    const int CC = p.CC, pitchE = p.pitchE;
    const int chunk = blockIdx.x % p.n_chunks, group = blockIdx.x / p.n_chunks;
    const int cbase = chunk * CC;
    const int n_epi_threads = 32 * p.n_epi;
    const bool tr = p.trace != nullptr && lane == 0;
    long long tw0 = 0, tw1 = 0, tw2 = 0, tw3 = 0, tn = 0; // trace: cycles this thread spent in its waits / sub-steps
    const long long t_begin = tr ? clock64() : 0;

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) {
            tc::mbar_init(&bars[0 + i], 1);
            tc::mbar_init(&bars[2 + i], 1);
            tc::mbar_init(&bars[8 + i], p.n_epi);          // counts are WARPS (arrive_warp)
            tc::mbar_init(&bars[10 + i], p.n_dw >> 5);
            tc::mbar_init(&bars[13 + i], p.n_dw >> 5);
            tc::mbar_init(&bars[15 + i], 2);
        }
        tc::mbar_init(&bars[12], 1);
        s_abort_mem = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // registers follow the roles: the launch gives every thread 80; control and epilogue groups hand theirs back, the
    // depthwise groups (the only code with 28-56 accumulators + a kernel row of weights live) take them
    // (each setmaxnreg sits at the top of its role's branch: ptxas budgets the code it dominates)

    const float inv_tx = 1.0f / (float)p.tiles_x;
    ItemIter it;
    it.init(group, p.groups, p.tiles);

    if (warp < 4) {
      asm volatile("setmaxnreg.dec.sync.aligned.u32 48;");
      if (warp == 0) {
        // =========================================================================== TMA producer
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
            // this CTA's slice of the expand weights: resident for the whole launch
            k1w::arrive_expect_tx(b_w, p.w_tx);
            for (int kb = 0; kb < p.nkb; ++kb) k1w::tma_2d(sW + (uint32_t)kb * CC * 128, &p.tmW, kb * 64, cbase, b_w);
            for (int k = 0; it.item < p.items; it.next(), ++k) {
                const int tyi = div_small(it.t, inv_tx);
                const int iy0 = tyi * p.TH * S - p.pad, ix0 = (it.t - tyi * p.tiles_x) * p.TW * S - p.pad;
                const int st = p.NA == 2 ? (k & 1) : 0;
                const uint32_t par = p.NA == 2 ? ((k >> 1) & 1) : (k & 1);
                k1w::wait_t(b_a_empty + 8 * st, par ^ 1, s_abort, p.tflag, tr, tw0);         // the MMAs that read this stage have completed
                k1w::arrive_expect_tx(b_a_full + 8 * st, p.a_tx);
                for (int kb = 0; kb < p.nkb; ++kb)
                    k1w::tma_4d(sA + (uint32_t)st * p.a_stage + (uint32_t)kb * p.rows_alloc * 128, &p.tmA, kb * 64, ix0, iy0, it.q * p.NB, b_a_full + 8 * st);
            }
        }
      } else if (warp == 1) {
        // idle: the epilogue warpgroups issue their own MMAs
      } else {
        // =========================================================================== reducer: squeeze partial sums of an item
        // The depthwise lanes leave their per-lane sums in a 2-slot ring; these two warps add them up in a FIXED order
        // (four chains by lane mod 4, as K1 does) and write partial[crop][tile][channel].  The depthwise warps never wait
        // for each other, so they drift apart and their SFU / FMA phases interleave.
        const int rtid = tid - 64;
        for (int k = 0; it.item < p.items; it.next(), ++k) {
            const int buf = k & 1, n0 = it.q * p.NB;
            k1w::wait(b_r_full + 8 * buf, (k >> 1) & 1, s_abort, p.tflag);
            const uint32_t r_buf = sR + (uint32_t)(buf * p.PY * CC) * 4;
            for (int col = rtid; col < p.NB * CC; col += 64) {
                const int jj = col >= CC ? 1 : 0, cc = col - jj * CC;          // NB <= 2
                float s4[4] = {0.f, 0.f, 0.f, 0.f};
                const uint32_t r0 = r_buf + (uint32_t)(jj * p.PYc * CC + cc) * 4;
                int y = 0;
                for (; y + 3 < p.PYc; y += 4) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float t;
                        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t) : "r"(r0 + (uint32_t)((y + i) * CC) * 4));
                        s4[i] += t;
                    }
                }
                for (; y < p.PYc; ++y) {
                    float t;
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t) : "r"(r0 + (uint32_t)(y * CC) * 4));
                    s4[y & 3] += t;
                }
                if (n0 + jj < p.N)
                    p.partial[((long long)(n0 + jj) * p.tiles + it.t) * p.Cexp + cbase + cc] = (s4[0] + s4[1]) + (s4[2] + s4[3]);
            }
            k1w::arrive_warp(b_r_empty + 8 * buf);
        }
      }
    } else if (warp >= 24 - 4 * EPI_WG) {
        // register budget of the CTA: 768 x 80 = 61440 = 128 x 48 (control) + 128 x 80 + 512 x 88   (one epilogue group)
        //                                               = 128 x 48 (control) + 256 x 72 + 384 x 96   (two epilogue groups)
        if (EPI_WG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 72;");          // one group: keeps its 80
        // =========================================================================== MMA + epilogue: wgmma -> +shift -> swish -> E
        constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
        const int wq = warp & 3;
        const int e_first = kK1WThreads - n_epi_threads;     // first epilogue thread
        const int grp = (warp - (e_first >> 5)) >> 2, NG = p.n_epi >> 2;
        const int units = CC >> 4;
        const int npix = p.IH * p.IW;
        const float inv_IW = 1.0f / (float)p.IW, inv_npix = 1.0f / (float)npix;
        // BN shifts of this CTA's channels -> shared memory (read by this group only; published by a group barrier)
        {
            float* sh = reinterpret_cast<float*>(smem_raw + (sC - tc::smem_u32(smem_raw)));
            for (int c = tid - e_first; c < CC; c += n_epi_threads) sh[c] = p.shift[cbase + c];
            asm volatile("bar.sync 2, %0;" ::"r"(n_epi_threads) : "memory");
        }
        k1w::wait(b_w, 0, s_abort, p.tflag);
        const int halves = (p.rows + 63) >> 6;
        for (int k = 0; it.item < p.items; it.next(), ++k) {
            const int tyi = div_small(it.t, inv_tx);
            const int iy0 = tyi * p.TH * S - p.pad, ix0 = (it.t - tyi * p.tiles_x) * p.TW * S - p.pad, n0 = it.q * p.NB;
            const int buf = k & 1;
            const int st = p.NA == 2 ? (k & 1) : 0;
            const uint32_t par = p.NA == 2 ? ((k >> 1) & 1) : (k & 1);
            k1w::wait_t(b_a_full + 8 * st, par, s_abort, p.tflag, tr, tw0);
            k1w::wait_t(b_e_empty + 8 * buf, ((k >> 1) & 1) ^ 1, s_abort, p.tflag, tr, tw1);     // the depthwise of item k-2 is done with this E
            if (!*s_abort) {
                const uint32_t e0 = sE + (uint32_t)buf * p.e_buf;
                const uint32_t a0 = sA + (uint32_t)st * p.a_stage;
                // (64-row half, 16-column unit) pieces f = grp, grp + NG, ...
                for (int f = grp; f < halves * units; f += NG) {
                    const int hh = f / units, u = f - hh * units;
                    float d[8];
                    long long tq = tr ? clock64() : 0;
                    tc::wg_mma_m64<BF16, 16>(d, a0 + (uint32_t)hh * 64 * 128, (uint32_t)p.rows_alloc * 128, sW + (uint32_t)u * 2048, (uint32_t)CC * 128, p.ksteps);
                    tc::wg_wait<0>();
                    if (tr) tw2 += clock64() - tq;
                    tq = tr ? clock64() : 0;
                    // fragment: register 4i + e -> row 16 wq + lane/4 (+8 for e >= 2), column 8 i + 2 (lane % 4) + (e & 1)
#pragma unroll
                    for (int e2 = 0; e2 < 2; ++e2) {
                        const int r = hh * 64 + 16 * wq + (lane >> 2) + 8 * e2;
                        if (r >= p.rows) continue;
                        const int j = p.NB == 1 ? 0 : div_small(r, inv_npix);
                        const int q = r - j * npix;
                        const int ty = div_small(q, inv_IW), tx = q - ty * p.IW;
                        // halo pixels outside the image (or crops past the batch): the depthwise pads the EXPANDED tensor with zeros
                        const bool img = (unsigned)(iy0 + ty) < (unsigned)p.Hin && (unsigned)(ix0 + tx) < (unsigned)p.Hin && n0 + j < p.N;
                        const uint32_t dst = e0 + (uint32_t)(j * p.e_rows + q) * pitchE;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int c = u * 16 + 8 * i + 2 * (lane & 3);
                            float2 sh;
                            asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(sh.x), "=f"(sh.y) : "r"(sC + (uint32_t)c * 4u));
                            const float2 h = k1w::swish2_from_half(k1w::fadd2(make_float2(d[4 * i + 2 * e2], d[4 * i + 2 * e2 + 1]), sh));
                            const uint32_t v = img ? pack2<__half>(h.x, h.y) : 0u;
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst + (uint32_t)c * 2u), "r"(v) : "memory");
                        }
                    }
                    if (tr) { tw3 += clock64() - tq; ++tn; }
                }
            }
            // every epilogue warpgroup's MMAs are done with the A stage
            asm volatile("bar.sync 2, %0;" ::"r"(n_epi_threads) : "memory");
            if (tid == e_first) k1w::arrive(b_a_empty + 8 * st);
            k1w::arrive_warp(b_e_full + 8 * buf);
        }
    } else {
        if (EPI_WG == 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 88;");
        else asm volatile("setmaxnreg.inc.sync.aligned.u32 96;");
        // =========================================================================== depthwise on E
        const int dtid = tid - k1w::kCtrlThreads;
        const int CVc = CC >> 2;
        const int py = div_small(dtid, 1.0f / (float)CVc), cv = dtid - py * CVc;
        const int jc = p.NB == 1 ? 0 : div_small(py, 1.0f / (float)p.PYc), pl = py - jc * p.PYc;   // crop of this lane, lane within the crop
        const bool lane_ok = py < p.PY;
        const int nstrips = p.TH << p.spr_log2;
        const uint32_t e_rowstride = (uint32_t)p.IW * pitchE;
        constexpr int NCOL = (R - 1) * S + KS;
        // depthwise constants of this CTA's channels: { b_dw[CC] fp32 | w_dw16[KS*KS][CC] fp16 }, staged once by this group
        {
            float* cb = reinterpret_cast<float*>(smem_raw + (sC - tc::smem_u32(smem_raw))) + CC;
            __half* cw = reinterpret_cast<__half*>(cb + CC);
            const __half* w16 = reinterpret_cast<const __half*>(p.w_dw16);
            for (int i = dtid; i < CC; i += p.n_dw) cb[i] = p.b_dw[cbase + i];
            for (int i = dtid; i < KS * KS * CC; i += p.n_dw) {
                const int row = div_small(i, 1.0f / (float)CC), c = i - row * CC;
                cw[i] = w16[(long long)row * p.Cexp + cbase + c];
            }
            asm volatile("bar.sync 1, %0;" ::"r"(p.n_dw) : "memory");
        }
        const uint32_t cst = sC + (uint32_t)CC * 4 + (uint32_t)cv * 16;         // this thread's shift values
        const uint32_t cst_h = sC + (uint32_t)CC * 8 + (uint32_t)cv * 8;          // ... and its column of the fp16 weights
        const int c0 = cbase + cv * 4;
        T* const out = reinterpret_cast<T*>(p.out);
        const long long crop_elems = (long long)p.Ho * p.Ho * p.Cexp;
        for (int k = 0; it.item < p.items; it.next(), ++k) {
            const int tyi = div_small(it.t, inv_tx);
            const int ty0 = tyi * p.TH, tx0 = (it.t - tyi * p.tiles_x) * p.TW, n0 = it.q * p.NB;
            const int buf = k & 1;
            const bool dw_active = lane_ok && n0 + jc < p.N;
            T* const out_n = out + (long long)(n0 + jc) * crop_elems;
            k1w::wait_t(b_e_full + 8 * buf, (k >> 1) & 1, s_abort, p.tflag, tr, tw0);
            float2 sum01 = make_float2(0.f, 0.f), sum23 = make_float2(0.f, 0.f);
            if (dw_active) {
                const float4 bq = lds_f4(cst);
                const uint32_t e_cv = sE + (uint32_t)buf * p.e_buf + (uint32_t)(jc * p.e_rows) * pitchE + (uint32_t)cv * 8;
                for (int sidx = pl; sidx < nstrips; sidx += p.PYc) {
                    const int oyl = sidx >> p.spr_log2, oxl0 = (sidx - (oyl << p.spr_log2)) * R;
                    // fp16 E, fp16 weights, HFMA2 running sums (no unpack instructions); sum * kDwScale + shift in fp32
                    __half2 hacc[R][2];
#pragma unroll
                    for (int r = 0; r < R; ++r) { hacc[r][0] = __float2half2_rn(0.f); hacc[r][1] = __float2half2_rn(0.f); }
                    uint32_t erow = e_cv + (uint32_t)(oyl * S) * e_rowstride + (uint32_t)(oxl0 * S) * pitchE;
#pragma unroll
                    for (int ky = 0; ky < KS; ++ky) {
                        __half2 wr[KS][2];
#pragma unroll
                        for (int kx = 0; kx < KS; ++kx) {
                            uint32_t w0, w1;
                            lds64(cst_h + (uint32_t)((ky * KS + kx) * CC) * 2, w0, w1);
                            wr[kx][0] = *reinterpret_cast<__half2*>(&w0); wr[kx][1] = *reinterpret_cast<__half2*>(&w1);
                        }
                        uint32_t ea = erow;
#pragma unroll
                        for (int col = 0; col < NCOL; ++col) {
                            uint32_t a, b;
                            lds64(ea, a, b);
                            ea += pitchE;
                            const __half2 x01 = *reinterpret_cast<__half2*>(&a), x23 = *reinterpret_cast<__half2*>(&b);
#pragma unroll
                            for (int r = 0; r < R; ++r) {
                                const int kx = col - r * S;          // compile-time after unrolling
                                if (kx >= 0 && kx < KS) {
                                    hacc[r][0] = __hfma2(x01, wr[kx][0], hacc[r][0]);
                                    hacc[r][1] = __hfma2(x23, wr[kx][1], hacc[r][1]);
                                }
                            }
                        }
                        erow += e_rowstride;
                    }
                    float2 acc[R][2];
                    const float2 sc = make_float2(kDwScale, kDwScale);
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        acc[r][0] = make_float2(bq.x, bq.y); acc[r][1] = make_float2(bq.z, bq.w);
                        ffma2(acc[r][0], __half22float2(hacc[r][0]), sc);
                        ffma2(acc[r][1], __half22float2(hacc[r][1]), sc);
                    }
                    T* dst = out_n + ((long long)(ty0 + oyl) * p.Ho + tx0 + oxl0) * p.Cexp + c0;
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        if (oxl0 + r < p.TW) {
                            const float2 s01 = k1w::swish2_from_half(acc[r][0]), s23 = k1w::swish2_from_half(acc[r][1]);
                            sum01 = k1w::fadd2(sum01, s01); sum23 = k1w::fadd2(sum23, s23);
                            uint2 o;
                            o.x = pack2<T>(s01.x, s01.y);
                            o.y = pack2<T>(s23.x, s23.y);
                            *reinterpret_cast<uint2*>(dst + (long long)r * p.Cexp) = o;
                        }
                    }
                }
            }
            k1w::arrive_warp(b_e_empty + 8 * buf);            // this warp's reads of this E are done
            // squeeze partial sums of the item: this lane's sums -> ring slot; the reducer warps take it from there
            k1w::wait_t(b_r_empty + 8 * buf, ((k >> 1) & 1) ^ 1, s_abort, p.tflag, tr, tw1);
            if (lane_ok)
                asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(sR + (uint32_t)((buf * p.PY + py) * CC + cv * 4) * 4),
                             "f"(sum01.x), "f"(sum01.y), "f"(sum23.x), "f"(sum23.y) : "memory");
            k1w::arrive_warp(b_r_full + 8 * buf);
        }
    }
    if (tr && (warp == 0 || warp == 1 || warp == 4 || warp == 24 - 4 * EPI_WG)) {
        // trace row of this CTA: [0] total cycles, then per role (producer, idle warp 1, epilogue warp 0, depthwise warp 0): its waits
        long long* row = p.trace + (long long)blockIdx.x * 16;
        const int slot = warp == 0 ? 1 : (warp == 1 ? 4 : (warp == 4 ? 10 : 7));
        row[slot] = tw0; row[slot + 1] = tw1; row[slot + 2] = clock64() - t_begin;
        if (warp == 24 - 4 * EPI_WG) { row[13] = tw2; row[14] = tw3; row[15] = tn; }      // epilogue: in the MMAs, in the epilogue, pieces
        if (warp == 0) row[0] = clock64() - t_begin;
    }
}

// ----------------------------------------------------------------------------- planning (host)
// TH x TW output tile, R outputs per strip, CC channels per CTA, NB crops per item, n_epi epilogue warps, NT threads.
// Fills every field of K1WParams except the tensor maps and the pointers.  false = this plan cannot run.
inline bool plan_k1w_candidate(int Hin, int Ho, int Cin, int Cexp, int k, int s, int pad, bool is_bf16, int TH, int TW, int R, int CC, int NB,
                               int n_epi, int NT, K1WParams* p, size_t* smem_out) {
    if (Ho % TH || Ho % TW || Cexp % CC || (CC & 15) || CC > 256 || (n_epi != 4 && n_epi != 8) || NB < 1 || NB > 2) return false;
    p->Hin = Hin; p->Ho = Ho; p->Cin = Cin; p->Cexp = Cexp; p->pad = pad;
    p->TH = TH; p->TW = TW;
    p->IH = (TH - 1) * s + k; p->IW = (TW - 1) * s + k;
    p->tiles_x = Ho / TW; p->tiles = p->tiles_x * (Ho / TH);
    if (NB > 1 && p->tiles != 1) return false;
    if (p->IH > 256 || p->IW > 256) return false;
    p->NB = NB;
    p->CC = CC; p->n_chunks = Cexp / CC;
    p->nkb = (Cin + 63) / 64;
    p->ksteps = (Cin + 15) / 16;
    p->rows = NB * p->IH * p->IW;
    p->mtiles = (p->rows + BM - 1) / BM;
    if (p->mtiles > 3) return false;
    p->rows_alloc = (p->rows + 7) & ~7;
    (void)is_bf16;
    p->pitchE = CC * 2 + 16;
    p->e_rows = p->IH * p->IW + R * s + 16;          // a ragged strip still LOADS the columns of its discarded outputs
    p->n_epi = n_epi;
    if (NT != kK1WThreads) return false;
    p->n_dw = NT - k1w::kCtrlThreads - 32 * n_epi;
    if (p->n_dw < 64 || (p->n_dw & 31)) return false;
    const int CVc = CC / 4;
    p->PYc = p->n_dw / CVc / NB;
    p->PY = p->PYc * NB;
    if (p->PYc < 1 || NB * CC > p->n_dw) return false;
    const int spr = (TW + R - 1) / R;
    p->spr_log2 = spr == 1 ? 0 : spr == 2 ? 1 : spr == 4 ? 2 : -1;
    if (p->spr_log2 < 0) return false;
    p->a_stage = (uint32_t)p->nkb * p->rows_alloc * 128;                      // multiple of 1024
    p->a_tx = (uint32_t)p->nkb * p->rows * 128;                               // full boxes, zero fill included
    p->w_tx = (uint32_t)p->nkb * CC * 128;
    const uint32_t w_bytes = ((uint32_t)p->nkb * CC * 128 + 1023u) & ~1023u;
    const uint32_t c_bytes = (uint32_t)(2 * CC * 4 + k * k * CC * 2 + 15) & ~15u;    // shift[CC] | b_dw[CC] fp32 | w_dw16[k*k][CC] fp16
    p->e_buf = ((uint32_t)NB * p->e_rows * p->pitchE + 15u) & ~15u;
    const uint32_t r_bytes = 2u * p->PY * CC * 4;
    for (int na = 2; na >= 1; --na) {
        p->NA = na;
        p->off_w = (uint32_t)na * p->a_stage;
        p->off_c = p->off_w + w_bytes;
        p->off_e = p->off_c + c_bytes;
        p->off_r = p->off_e + 2 * p->e_buf;
        const size_t total = (size_t)p->off_r + r_bytes + 1024;
        // the UMMA of the last M tile reads 128 rows even when fewer were staged: that read has to stay inside the window
        const size_t over = (size_t)(na - 1) * p->a_stage + (size_t)(p->nkb - 1) * p->rows_alloc * 128 + (size_t)p->mtiles * BM * 128 + 1024;
        if (total <= K1_MAX_SMEM && over <= total) { *smem_out = total; return true; }
    }
    return false;
}

struct K1WChoice { int th, tw, r, cc, nb, n_epi, nt; };

// Per-block plan table (first guesses from the per-role instruction model in DESIGN.md; tools/tune_k1w.py re-measures them).
inline bool plan_k1w(int Hin, int Ho, int Cin, int Cexp, int k, int s, int pad, bool is_bf16, K1WParams* p, K1WChoice* choice, size_t* smem_out) {
    struct Tuned { int hin, k, s, cexp; K1WChoice c; };
    static const Tuned tuned[] = {
        {112, 3, 2, 96, {8, 8, 4, 48, 1, 8, 768}},      // block 2: 17x17 halo = 289 rows, SFU-bound -> 8 epilogue warps
        {56, 3, 1, 144, {14, 14, 7, 48, 1, 4, 768}},    // block 3: 16x16 = 256 rows
        {56, 5, 2, 144, {7, 7, 4, 48, 1, 8, 768}},      // block 4: 17x17
        {28, 5, 1, 240, {14, 14, 7, 80, 1, 4, 768}},    // block 5: 18x18 = 324 rows
        {28, 3, 2, 240, {7, 7, 4, 80, 1, 8, 768}},      // block 6: 15x15 = 225 rows
        {14, 3, 1, 480, {14, 14, 7, 96, 1, 4, 768}},    // blocks 7, 8: whole image, 16x16
        {14, 5, 1, 480, {14, 14, 7, 48, 1, 4, 768}},    // block 9: 18x18
        {14, 5, 1, 672, {14, 14, 7, 48, 1, 4, 768}},    // blocks 10, 11
        {14, 5, 2, 672, {7, 7, 4, 48, 1, 4, 768}},      // block 12: 17x17
        {7, 5, 1, 1152, {7, 7, 4, 64, 2, 4, 768}},      // blocks 13-15: two crops per item, 2 x 11x11 = 242 rows
        {7, 3, 1, 1152, {7, 7, 7, 96, 2, 4, 768}},      // block 16: 2 x 9x9 = 162 rows
    };
    for (const Tuned& t : tuned)
        if (t.hin == Hin && t.k == k && t.s == s && t.cexp == Cexp) {
            K1WParams q{};
            size_t smem = 0;
            if (plan_k1w_candidate(Hin, Ho, Cin, Cexp, k, s, pad, is_bf16, t.c.th, t.c.tw, t.c.r, t.c.cc, t.c.nb, t.c.n_epi, t.c.nt, &q, &smem)) {
                *p = q; *choice = t.c; *smem_out = smem;
                return true;
            }
        }
    return false;
}

inline bool k1w_has_instance(int k, int s, int R, int NT) {
    return (k == 3 || k == 5) && (s == 1 || s == 2) && (R == 4 || R == 7) && NT == kK1WThreads;
}

template <typename T>
int launch_k1w(cudaStream_t stream, K1WParams p, int k, int s, int R, int NT, size_t smem, int n_crops, int sm_count) {
    p.N = n_crops;
    p.items = ((n_crops + p.NB - 1) / p.NB) * p.tiles;
    int groups = sm_count / p.n_chunks;
    if (groups < 1) groups = 1;
    if (groups > p.items) groups = p.items;
    p.groups = groups;
    const int ctas = groups * p.n_chunks;
    if (ctas < 1) return 0;
#define K1W_GO(KS, S, RR, EW)                                                                                              \
    do {                                                                                                                   \
        auto kfn = k1w_kernel<T, KS, S, RR, EW>;                                                                           \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K1_MAX_SMEM) != cudaSuccess) return -1;  \
        kfn<<<ctas, kK1WThreads, smem, stream>>>(p);                                                                       \
        return 0;                                                                                                          \
    } while (0)
#define K1W(KS, S, RR)                                  \
    do {                                                \
        if (NT != kK1WThreads) return 1;                \
        if (p.n_epi == 4) K1W_GO(KS, S, RR, 1);         \
        if (p.n_epi == 8) K1W_GO(KS, S, RR, 2);         \
    } while (0)
    if (k == 3 && s == 2 && R == 4) K1W(3, 2, 4);
    if (k == 3 && s == 1 && R == 7) K1W(3, 1, 7);
    if (k == 5 && s == 1 && R == 7) K1W(5, 1, 7);
    if (k == 5 && s == 2 && R == 4) K1W(5, 2, 4);
    if (k == 3 && s == 2 && R == 7) K1W(3, 2, 7);
    if (k == 3 && s == 1 && R == 4) K1W(3, 1, 4);
    if (k == 5 && s == 1 && R == 4) K1W(5, 1, 4);
    if (k == 5 && s == 2 && R == 7) K1W(5, 2, 7);
#undef K1W
#undef K1W_GO
    return 1;
}

}  // namespace fused
}  // namespace whenet
