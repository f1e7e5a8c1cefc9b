// kernels_fused.cuh - K1: the fused front half of an MBConv block.
//
//   expand 1x1 (warpgroup MMA, fp32 accumulators in registers, BN shift folded in as two extra K columns)
//   -> swish -> shared memory (never HBM)
//   -> depthwise KSxKS stride S, TF-SAME (CUDA-core FMA on the smem tile) -> BN shift + swish
//   -> D (global, 16-bit) + deterministic SE squeeze partial sums
//
// One CTA owns a TH x TW tile of the depthwise OUTPUT of one crop (or, where one tile is the whole image, of NB
// crops).  The matching input halo tile is IH x IW = (TH-1)*S+KS square; only its pixels INSIDE the image become GEMM
// rows (raster order over the inside rectangle) - the depthwise pads the EXPANDED tensor with zeros, so halo pixels
// outside the image are plain zero rows of E that are written once and never touched by the tensor core.  The rows are
// staged once with cp.async in the UMMA K-major SWIZZLE_128B layout; the expanded channels are then produced and
// consumed CC at a time:
//
//   for each chunk of CC expanded channels (W chunk + depthwise constants of chunk i+1 prefetched with cp.async):
//       wgmma  D[u][64 x CC] = [A | 1 1] (64 x (Cin+8)) * [Wc | shift_hi shift_lo]^T   for every 64-row half u (the warp
//       groups of the CTA take the halves in turn) -> swish -> 16-bit -> E[halo pixel][CC] in smem
//       depthwise strips straight out of E (ld.shared.v2), the KS weights of one kernel row from smem
//       -> store D, accumulate the squeeze sums
//
// The expanded tensor (the largest activation of the network: 112*112*96 values per crop in block 2)
// never leaves the SM.  The BN shift of the expand conv rides on the tensor core: A gets two constant
// 1.0 columns, W gets the shift split into a bf16 high and low part (error 2^-17 relative), so the
// epilogue has no bias loads or adds.
#pragma once
#include <algorithm>

#include "kernels_tc.cuh"

namespace whenet {
namespace fused {

using tc::BK;
using tc::BM;

constexpr size_t K1_MAX_SMEM = 227 * 1024 - 256;
// fp16 depthwise: weights are stored / kDwScale so that the fp16 running sums stay far from 65504 (largest |folded sum| seen
// on real and synthetic crops: ~2 x 10^4 before the 1/2 pre-scaling -> ~2.5 x 10^3 here); the scale returns in the fp32 FMA that
// adds the BN shift, at no cost.
constexpr float kDwScale = 4.0f;     // opt-in limit per CTA minus the kernel's static shared memory

struct K1Params {
    const void* in;        // T [N][Hin][Hin][Cin]
    // every K1 constant is pre-multiplied by 1/2 (exact): swish(x) = h + h*tanh(h) with h = x/2 then needs no multiply
    const void* wt_aug;    // T [Cexp][Cin+8]   0.5 * BN-folded weights, K-major, columns Cin / Cin+1 = 0.5*shift hi / lo, rest 0
    const float* w_dw;     // [KS*KS][Cexp]     0.5 * BN-folded depthwise weights
    const void* w_dw16;    // half [KS*KS][Cexp] the same / kDwScale, fp16: the depthwise of the blocks with an expand conv runs on
                           // HFMA2 (the fp16 E tile needs no unpacking); NULL for block 1
    const float* b_dw;     // [Cexp]            0.5 * BN shift
    void* out;             // T [N][Ho][Ho][Cexp]
    float* partial;        // [N][tiles][Cexp]
    // SE excite, run by the last CTA of each crop to finish (se_counter == nullptr: left to se_gate_kernel)
    const float *w_se1t, *b_se1, *w_se2, *b_se2;
    float* gate;           // [N][Cexp]
    int* se_counter;       // [N], zero on entry, self-resetting
    int se_tail;           // 1: this CTA holds every pixel and channel of its crops (one tile per image, no chunk split): it
                           // keeps the channel means in shared memory and computes the gate itself - no ticket, no fence
    float inv_hw;          // 1 / (Ho*Ho), as the stand-alone SE kernel gets it
    int scale_out;         // se_tail only: multiply the depthwise output by the gate in place (16-bit rounding of d*g, exactly
                           // what the project conv's gate pass would feed the tensor core), so the project runs ungated
    int Cse;
    int Hin, Ho, Cin, Cexp, pad;
    int TH, TW, IH, IW;    // output tile, input halo tile
    int tiles_x, tiles_y;
    int CC, n_chunks;      // expanded channels per chunk (multiple of 16), number of chunks
    int mtiles;            // most 128-row GEMM tiles any CTA needs (<= 3)
    int rows_alloc;        // A rows per K block in smem: most GEMM rows any CTA has, rounded up to 8 (the last M tile's
                           // UMMA reads on past them into whatever follows - those accumulator rows are never used)
    int NB;                // crops per CTA (> 1 only when one tile is the whole image)
    int N;                 // crops in this launch
    int e_rows;            // E rows per crop (halo pixels + slack)
    int PYc;               // strip lanes per crop = PY / NB
    int cpr;               // 16-byte chunks per operand row incl. the ones/shift chunk, rounded up to even
    int nkb;               // ceil(cpr / 8)
    int pitchE;            // bytes per E row = CC*2 + 16
    int PY;                // strip lanes in the depthwise phase = threads / (CC/4), rounded down to a multiple of NB
    int spr_log2;          // log2(strips per output row)
    int smem_A, smem_W, smem_C, smem_E;   // region sizes in bytes (W and C are per buffer; both double-buffered)
    int* tflag;            // the context's mbarrier-timeout flag (mapped pinned host memory)
    int chunks_per_cta;    // grid.z CTAs share one tile, each takes this many consecutive chunks (small batches: more CTAs per crop)
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const uint32_t sz = valid ? 16u : 0u;     // src-size 0 -> 16 zero bytes
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void lds64(uint32_t addr, uint32_t& a, uint32_t& b) {
    asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "r"(addr));
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
// two IEEE fp32 FMAs on a channel pair: d.x = a.x*b.x + d.x, d.y = a.y*b.y + d.y
__device__ __forceinline__ void ffma2(float2& d, const float2& a, const float2& b) {
    d.x = fmaf(a.x, b.x, d.x);
    d.y = fmaf(a.y, b.y, d.y);
}
template <typename T> __device__ __forceinline__ void unpack2(uint32_t u, float& lo, float& hi);
template <> __device__ __forceinline__ void unpack2<__nv_bfloat16>(uint32_t u, float& lo, float& hi) {
    lo = __uint_as_float(u << 16);
    hi = __uint_as_float(u & 0xffff0000u);
}
template <> __device__ __forceinline__ void unpack2<__half>(uint32_t u, float& lo, float& hi) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
    lo = f.x; hi = f.y;
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}
template <typename T> __device__ __forceinline__ uint32_t ones2();
template <> __device__ __forceinline__ uint32_t ones2<__nv_bfloat16>() { return 0x3f803f80u; }
template <> __device__ __forceinline__ uint32_t ones2<__half>() { return 0x3c003c00u; }

// swizzled byte offset of 16-byte chunk c (0..7) of row r inside one K block ([rows][128 B], 8-row atoms of 1024 B)
__device__ __forceinline__ uint32_t sw128(int r, int c) {
    return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
}
// the same for 64-byte rows (SWIZZLE_64B): chunk c (0..3) of row r lands at chunk c ^ ((r >> 1) & 3); 8-row atoms of 512 B
__device__ __forceinline__ uint32_t sw64(int r, int c) {
    return (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4));
}

// exact floor(x / d) for the small non-negative ints of the tile arithmetic (x < 2^17, d < 2^8), with inv = 1.0f / d:
// (x + 0.5) / d is at least 0.5 / d away from every integer, far more than the float rounding error
__device__ __forceinline__ int div_small(int x, float inv) { return __float2int_rz(((float)x + 0.5f) * inv); }

// The arithmetic of one 16-bit-storage K1 tile that k1x_kernel (kernels_k1x.cuh) shares, so that the two kernels cannot drift
// apart by a bit.
//
// Expand epilogue of one fragment row: the NP 16-column pieces of accumulator row `hr` (0: row lane/4, 1: that + 8) of a
// m64nN fragment -> swish -> fp16 -> E row at `er` (cq = 2 (lane % 4)).  The BN shift is already in the accumulator.
// E is fp16 whatever the storage type: 3 more mantissa bits than bf16 and HFMA2-ready.
template <int NP>
__device__ __forceinline__ void expand_row_to_e(const float (&d)[8 * NP], int nch16, int hr, uint32_t er, int cq) {
#pragma unroll
    for (int jj = 0; jj < NP; ++jj) {
        if (jj < nch16) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const uint32_t v = pack2<__half>(swish_from_half(d[8 * jj + 4 * i + 2 * hr]), swish_from_half(d[8 * jj + 4 * i + 2 * hr + 1]));
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(er + (uint32_t)(16 * jj + 8 * i + cq) * 2u), "r"(v) : "memory");
            }
        }
    }
}

// HFMA2 depthwise of one strip (R outputs of one row, 4 channels): fp16 E, fp16 weights, fp16 running sums - the loaded
// words ARE the operands (no unpack instructions), one HFMA2 per channel pair and tap - then sum * kDwScale + shift in fp32.
// Measured against the float64 oracle this is MORE accurate than the bf16-E / fp32-FMA form it replaced (0.12 vs 0.19 deg
// on the golden crops): E keeps 11 mantissa bits.  `erow` = top-left of the strip's input window (rows e_rowstride, pixels
// pitchE bytes apart), `wts` = this thread's 4 channels of tap 0 (taps w_pitch bytes apart), bq = their BN shifts.
template <int KS, int S, int R>
__device__ __forceinline__ void dw_strip_hfma2(uint32_t erow, uint32_t e_rowstride, uint32_t pitchE, uint32_t wts, uint32_t w_pitch,
                                               const float4& bq, float2 (&acc)[R][2]) {
    constexpr int NCOL = (R - 1) * S + KS;
    __half2 hacc[R][2];
#pragma unroll
    for (int r = 0; r < R; ++r) { hacc[r][0] = __float2half2_rn(0.f); hacc[r][1] = __float2half2_rn(0.f); }
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
        __half2 wr[KS][2];
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
            uint32_t w0, w1;
            lds64(wts + (uint32_t)(ky * KS + kx) * w_pitch, w0, w1);
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
    const float2 sc = make_float2(kDwScale, kDwScale);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        acc[r][0] = make_float2(bq.x, bq.y); acc[r][1] = make_float2(bq.z, bq.w);
        ffma2(acc[r][0], __half22float2(hacc[r][0]), sc);          // sum * kDwScale + shift, in fp32
        ffma2(acc[r][1], __half22float2(hacc[r][1]), sc);
    }
}

// The strip's first `nvalid` outputs: swish, squeeze sums (in strip order), 16-bit store to dst (pixels Cexp apart).
template <typename T, int R>
__device__ __forceinline__ void dw_strip_finish(float2 (&acc)[R][2], int nvalid, T* dst, int Cexp, float (&sum)[4]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (r < nvalid) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                acc[r][i].x = swish_from_half(acc[r][i].x); acc[r][i].y = swish_from_half(acc[r][i].y);
                sum[2 * i] += acc[r][i].x; sum[2 * i + 1] += acc[r][i].y;
            }
            uint2 o;
            o.x = pack2<T>(acc[r][0].x, acc[r][0].y);
            o.y = pack2<T>(acc[r][1].x, acc[r][1].y);
            *reinterpret_cast<uint2*>(dst + (long long)r * Cexp) = o;
        }
    }
}

// NOEXP: the block has no expand conv (block 1): the halo tile of the block INPUT is copied straight into E and only the
// depthwise half of the kernel runs (single chunk, no tensor-core work).
// CCT != 0 bakes the chunk width (and with it the E row pitch and every constant-table offset) into the code: the
// depthwise inner loop then addresses shared memory with immediates instead of computed offsets.
// NT = threads per CTA: 256 (two CTAs share an SM) or 512 (one CTA per SM - the late blocks, whose operands do not
// leave room for two CTAs, get their 16 warps this way).
template <typename T, int KS, int S, int R, bool NOEXP = false, int CCT = 0, int NT = 256>
__global__ void __launch_bounds__(NT, NT == 256 ? 2 : 1) k1_expand_dw_kernel(const K1Params p) {
    const int CC = CCT ? CCT : p.CC;
    const int pitchE = CCT ? CCT * 2 + 16 : p.pitchE;
    // depthwise on HFMA2 (fp16 running sums over the fp16 E tile, fp16 weights): bf16 storage with an expand conv
    constexpr bool HDW = !NOEXP && std::is_same<T, __nv_bfloat16>::value;
    constexpr int NG = NT / 128;                                // warp groups (each issues the MMAs of its 64-row halves)
    extern __shared__ uint8_t smem_raw[];
    __shared__ int s_last;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t smem0 = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem0;                                  // [nkb][rows_alloc][128 B]        swizzled
    const uint32_t sW = sA + p.smem_A;                          // 2 x [nkb][CC rows][128 B]       swizzled
    const uint32_t sC = sW + 2 * p.smem_W;                      // 2 x { b_dw[CC], w_dw[KS*KS][CC] } fp32
    const uint32_t sE = sC + 2 * p.smem_C;                      // [NB][e_rows][pitchE]
    const uint32_t sR = sE + p.smem_E;                          // [PY][CC] fp32 squeeze partials
    float* const sM = reinterpret_cast<float*>(smem_raw + (sR + (uint32_t)(p.PY * CC) * 4u - tc::smem_u32(smem_raw)));
                                                                // [NB][Cexp] channel means, [Cse] hidden (se_tail only)

    const T* in = reinterpret_cast<const T*>(p.in);
    const T* wt = reinterpret_cast<const T*>(p.wt_aug);
    T* out = reinterpret_cast<T*>(p.out);

    const int n0 = blockIdx.y * p.NB, tile = blockIdx.x;
    const int nb_here = min(p.NB, p.N - n0);                                       // crops of this CTA
    const int tyi = div_small(tile, 1.0f / (float)p.tiles_x);
    const int ty0 = tyi * p.TH, tx0 = (tile - tyi * p.tiles_x) * p.TW;             // output-tile origin
    const int iy0 = ty0 * S - p.pad, ix0 = tx0 * S - p.pad;                       // input-tile origin (may be < 0)
    const int npix = p.IH * p.IW;
    // the part of the halo tile that lies inside the image: these pixels are the GEMM rows
    const int ty_lo = max(0, -iy0), tx_lo = max(0, -ix0);
    const int IHin = min(p.IH, p.Hin - iy0) - ty_lo, IWin = min(p.IW, p.Hin - ix0) - tx_lo;
    const int npix_in = IHin * IWin;
    const int rows_gemm = nb_here * npix_in;
    const float inv_IWin = 1.0f / (float)IWin, inv_npix = 1.0f / (float)npix_in;
    const int kchunks = p.Cin >> 3;                     // data chunks per row; chunk `kchunks` holds the ones / the shift
    const int Kaug = p.Cin + 8;
    const uint32_t a_kb_stride = (uint32_t)p.rows_alloc * 128u;
    const float inv_cpr = 1.0f / (float)p.cpr, inv_q = 4.0f / (float)CC;

    if (NOEXP) {
        // ---- E <- the input halo tile itself (Cin == Cexp == CC), zero outside the image (depthwise SAME padding)
        const T* in_n = in + (long long)n0 * p.Hin * p.Hin * p.Cin;
        const int cpp = CC >> 3;                                  // 16-byte chunks per pixel
        const float inv_cpp = 1.0f / (float)cpp, inv_IW = 1.0f / (float)p.IW;
        for (int idx = tid; idx < npix * cpp; idx += NT) {
            const int r = div_small(idx, inv_cpp), c = idx - r * cpp;
            const int ty = div_small(r, inv_IW), tx = r - ty * p.IW;
            const int iy = iy0 + ty, ix = ix0 + tx;
            const bool valid = iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Hin;
            cp_async16(sE + (uint32_t)r * pitchE + c * 16, valid ? in_n + ((long long)iy * p.Hin + ix) * p.Cin + c * 8 : in_n, valid);
        }
    }

    // ---- A: the inside pixels of the halo tile (cp.async), + the ones chunk, + an even-count pad chunk
    if (!NOEXP) {
        const float inv_kch = 1.0f / (float)kchunks;
        const T* in_t = in + ((long long)n0 * p.Hin * p.Hin + (long long)(iy0 + ty_lo) * p.Hin + (ix0 + tx_lo)) * p.Cin;
        const int items = rows_gemm * kchunks;
        for (int idx = tid; idx < items; idx += NT) {
            const int r = div_small(idx, inv_kch), c = idx - r * kchunks;
            const int j = div_small(r, inv_npix), q = r - j * npix_in;
            const int ty = div_small(q, inv_IWin), tx = q - ty * IWin;
            const T* src = in_t + ((long long)(j * p.Hin + ty) * p.Hin + tx) * p.Cin + c * 8;
            cp_async16(sA + (uint32_t)(c >> 3) * a_kb_stride + sw128(r, c & 7), src, true);
        }
        const uint4 ones = make_uint4(ones2<T>(), 0u, 0u, 0u), zero = make_uint4(0u, 0u, 0u, 0u);
        for (int rr = tid; rr < rows_gemm; rr += NT) {
            sts128(sA + (uint32_t)(kchunks >> 3) * a_kb_stride + sw128(rr, kchunks & 7), ones);
            if (p.cpr > kchunks + 1)
                sts128(sA + (uint32_t)((kchunks + 1) >> 3) * a_kb_stride + sw128(rr, (kchunks + 1) & 7), zero);
        }
        // halo pixels outside the image: zero rows of E for the whole kernel (epilogue 1 only writes inside rows)
        if (npix_in != npix) {
            const int pieces = (p.NB * p.e_rows * pitchE) >> 4;
            for (int i = tid; i < pieces; i += NT) sts128(sE + (uint32_t)i * 16u, zero);
        }
    }
    // ---- cp.async prefetch of a W chunk / of a chunk's depthwise constants into buffer `buf` (the caller commits)
    auto prefetch_w = [&](int ch, int buf) {
        const int cbase = ch * CC;
        const uint32_t w_dst = sW + buf * p.smem_W;
        const int per_row = p.cpr;                                 // data chunks + shift chunk (+ zero pad chunk)
        for (int idx = tid; idx < (NOEXP ? 0 : CC * per_row); idx += NT) {
            const int r = div_small(idx, inv_cpr), c = idx - r * per_row;
            const bool valid = c <= kchunks;
            cp_async16(w_dst + (uint32_t)(c >> 3) * CC * 128 + sw128(r, c & 7),
                       valid ? wt + (long long)(cbase + r) * Kaug + c * 8 : wt, valid);
        }
    };
    auto prefetch_c = [&](int ch, int buf) {
        const int cbase = ch * CC;
        const uint32_t c_dst = sC + buf * p.smem_C;
        const int q = CC >> 2;                                   // 16-byte pieces per fp32 constant row
        if (!HDW) {
            for (int idx = tid; idx < (KS * KS + 1) * q; idx += NT) {
                const int row = div_small(idx, inv_q), j = idx - row * q;
                const float* src = row == 0 ? p.b_dw + cbase + j * 4 : p.w_dw + (long long)(row - 1) * p.Cexp + cbase + j * 4;
                cp_async16(c_dst + (uint32_t)(row * CC + j * 4) * 4, src, true);
            }
        } else {
            // { b_dw[CC] fp32 | w_dw16[KS*KS][CC] fp16 }: q pieces of shift, then q/2 pieces per tap
            const int qh = CC >> 3;
            const __half* w16 = reinterpret_cast<const __half*>(p.w_dw16);
            for (int idx = tid; idx < q + KS * KS * qh; idx += NT) {
                if (idx < q) cp_async16(c_dst + (uint32_t)idx * 16, p.b_dw + cbase + idx * 4, true);
                else {
                    const int t = idx - q;
                    const int row = div_small(t, 2.0f * inv_q), j = t - row * qh;
                    cp_async16(c_dst + (uint32_t)(CC * 4 + row * CC * 2 + j * 16), w16 + (long long)row * p.Cexp + cbase + j * 8, true);
                }
            }
        }
    };
    const int ch_begin = blockIdx.z * p.chunks_per_cta;
    const int ch_end = min(p.n_chunks, ch_begin + p.chunks_per_cta);
    // W runs TWO chunks ahead (its buffer is free as soon as the MMA that read it has completed), the depthwise
    // constants one chunk ahead (their buffer is read until the end of the depthwise phase)
    prefetch_w(ch_begin, ch_begin & 1);
    prefetch_c(ch_begin, ch_begin & 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (ch_begin + 1 < ch_end) prefetch_w(ch_begin + 1, (ch_begin + 1) & 1);
    asm volatile("cp.async.commit_group;" ::: "memory");

    // ---- per-thread constants of the two compute phases
    // epilogue 1: fragment row of thread (warp w of its group, lane l) -> E row of that GEMM row (halo pixel)
    const int grp = warp >> 2, wq = warp & 3;
    auto e_row_of = [&](int r) -> uint32_t {
        const int j = div_small(r, inv_npix), q = r - j * npix_in;
        const int ty = div_small(q, inv_IWin), tx = q - ty * IWin;
        return sE + (uint32_t)(j * p.e_rows + (ty_lo + ty) * p.IW + tx_lo + tx) * pitchE;
    };
    // depthwise: thread = (4-channel vector cv, strip lane py); with NB crops per CTA the lanes split evenly between them
    const int CVc = CC >> 2;
    const int py = tid / CVc, cv = tid - py * CVc;
    const int jc = p.NB == 1 ? 0 : div_small(py, 1.0f / (float)p.PYc), pl = py - jc * p.PYc;   // crop of this lane, lane within the crop
    const bool dw_active = py < p.PY && jc < nb_here;
    const int nstrips = p.TH << p.spr_log2;
    const uint32_t e_rowstride = (uint32_t)p.IW * pitchE;
    constexpr int NCOL = (R - 1) * S + KS;
    T* const out_n = out + (long long)(n0 + jc) * p.Ho * p.Ho * p.Cexp;

    // A, W(ch_begin), constants(ch_begin) and W(ch_begin + 1) have landed
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    const int nch16 = CC >> 4;
    constexpr int kMaxPieces = CCT ? CCT / 16 : 8;        // 16-column pieces of the expand tile (at most 128 columns)

    for (int ch = ch_begin; ch < ch_end; ++ch) {
        const int buf = ch & 1;
        const int cbase = ch * CC;
        // ---- expand MMA + epilogue 1: swish -> E (fp16).  The BN shift is already in the accumulator.  The 64-row halves of
        //      the GEMM rows go round-robin over the warp groups; halves past the last GEMM row are skipped.
        if (!NOEXP) {
            for (int u = grp; u * 64 < rows_gemm; u += NG) {
                // fragment register 8 jj + 4 i + e: piece jj of the m64nCC fragment
                float d[8 * kMaxPieces];
                if constexpr (CCT != 0) {
                    tc::wg_mma_m64<BF16, CCT>(d, sA + (uint32_t)u * 64 * 128, a_kb_stride, sW + buf * p.smem_W, (uint32_t)CC * 128, p.cpr >> 1);
                } else {
                    // chunk width chosen at run time: one m64n16 sequence per 16-column piece
#pragma unroll
                    for (int jj = 0; jj < kMaxPieces; ++jj)
                        if (jj < nch16)
                            tc::wg_mma_m64<BF16, 16>(*reinterpret_cast<float(*)[8]>(d + 8 * jj), sA + (uint32_t)u * 64 * 128, a_kb_stride,
                                                     sW + buf * p.smem_W + (uint32_t)jj * 2048u, (uint32_t)CC * 128, p.cpr >> 1);
                }
                tc::wg_wait<0>();
                const int r_lo = u * 64 + 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = r_lo + 8 * hr;
                    if (r < rows_gemm) {
                        expand_row_to_e<kMaxPieces>(d, nch16, hr, e_row_of(r), cq);
                    }
                }
            }
        }
        // constants of chunk ch+1 into the buffer the depthwise of chunk ch-1 has finished with
        if (ch + 1 < ch_end) prefetch_c(ch + 1, buf ^ 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        // E(ch) is complete, every MMA of chunk ch is done with W[buf], W(ch+1) and constants(ch+1) have landed
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (ch + 2 < ch_end) prefetch_w(ch + 2, buf);
        asm volatile("cp.async.commit_group;" ::: "memory");

        // ---- depthwise on E: 8-byte ld.shared, fp32 FMA, weights of one kernel row from smem
        float sum[4] = {0.f, 0.f, 0.f, 0.f};
        if (dw_active) {
            const int c0 = cbase + cv * 4;
            const uint32_t cst = sC + buf * p.smem_C + (uint32_t)cv * 16;         // this thread's column of the constants
            const float4 bq = lds_f4(cst);
            const uint32_t e_cv = sE + (uint32_t)(jc * p.e_rows) * pitchE + (uint32_t)cv * 8;
            for (int sidx = pl; sidx < nstrips; sidx += p.PYc) {
                const int oyl = sidx >> p.spr_log2, oxl0 = (sidx - (oyl << p.spr_log2)) * R;
                float2 acc[R][2];      // (ch0,ch1), (ch2,ch3): one FFMA2 (fma.rn.f32x2) per pair - same IEEE FMAs, half the issue slots
                uint32_t erow = e_cv + (uint32_t)(oyl * S) * e_rowstride + (uint32_t)(oxl0 * S) * pitchE;
                // fp16 storage mode keeps the fp32 FFMA2 form (E is fp16 there as well): that mode exists for its accuracy
                // (0.02 deg), and fp16 running sums would double its error; bf16 storage gains accuracy AND speed from HFMA2
                using TE = typename std::conditional<NOEXP, T, __half>::type;       // element type of the E tile
                if constexpr (!HDW) {
#pragma unroll
                    for (int r = 0; r < R; ++r) { acc[r][0] = make_float2(bq.x, bq.y); acc[r][1] = make_float2(bq.z, bq.w); }
#pragma unroll
                    for (int ky = 0; ky < KS; ++ky) {
                        float2 wr[KS][2];
#pragma unroll
                        for (int kx = 0; kx < KS; ++kx) {
                            const float4 wq = lds_f4(cst + (uint32_t)((1 + ky * KS + kx) * CC) * 4);
                            wr[kx][0] = make_float2(wq.x, wq.y); wr[kx][1] = make_float2(wq.z, wq.w);
                        }
                        uint32_t ea = erow;
#pragma unroll
                        for (int col = 0; col < NCOL; ++col) {
                            uint32_t a, b;
                            lds64(ea, a, b);
                            ea += pitchE;
                            float2 x01, x23;
                            unpack2<TE>(a, x01.x, x01.y);
                            unpack2<TE>(b, x23.x, x23.y);
#pragma unroll
                            for (int r = 0; r < R; ++r) {
                                const int kx = col - r * S;          // compile-time after unrolling
                                if (kx >= 0 && kx < KS) {
                                    ffma2(acc[r][0], x01, wr[kx][0]);
                                    ffma2(acc[r][1], x23, wr[kx][1]);
                                }
                            }
                        }
                        erow += e_rowstride;
                    }
                } else {
                    dw_strip_hfma2<KS, S, R>(erow, e_rowstride, (uint32_t)pitchE, cst - (uint32_t)cv * 16 + (uint32_t)CC * 4 + (uint32_t)cv * 8,
                                             (uint32_t)CC * 2, bq, acc);
                }
                const int oy = ty0 + oyl;
                T* dst = out_n + ((long long)oy * p.Ho + tx0 + oxl0) * p.Cexp + c0;
                dw_strip_finish<T, R>(acc, oy < p.Ho ? min(p.TW - oxl0, p.Ho - tx0 - oxl0) : 0, dst, p.Cexp, sum);
            }
            asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(sR + (uint32_t)(py * CC + cv * 4) * 4),
                         "f"(sum[0]), "f"(sum[1]), "f"(sum[2]), "f"(sum[3]) : "memory");
        }
        __syncthreads();
        if (tid < p.NB * CC) {
            const int jj = tid >= CC ? 1 : 0, cc = tid - jj * CC;          // NB <= 2
            if (jj < nb_here) {
                // four independent chains (lane mod 4) keep this short: the two warps doing it are the ones every other warp
                // waits for at the next barrier.  Fixed association order -> reproducible bits.
                float s4[4] = {0.f, 0.f, 0.f, 0.f};
                const uint32_t r0 = sR + (uint32_t)(jj * p.PYc * CC + cc) * 4;
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
                const float tot = (s4[0] + s4[1]) + (s4[2] + s4[3]);
                p.partial[((long long)(n0 + jj) * gridDim.x + tile) * p.Cexp + cbase + cc] = tot;
                if (p.se_tail) sM[jj * p.Cexp + cbase + cc] = tot * p.inv_hw;      // == the mean se_gate_crop forms from one tile
            }
        }
        // E and the squeeze scratch are reused only after this barrier
        __syncthreads();
    }
    if (p.se_counter) __threadfence();     // fused SE only: this CTA's squeeze partials are visible device-wide before the ticket
                                           // (unconditional, the MEMBAR made every CTA wait out its own output stores)
    __syncthreads();

    // ---- SE excite for the crops of this CTA when it holds all of their pixels and channels
    if (p.se_tail) {
        for (int jj = 0; jj < nb_here; ++jj) {
            float* const g_sm = sM + jj * p.Cexp;           // means in, gate out
            se_gate_fc<NT>(g_sm, sM + p.NB * p.Cexp, p.w_se1t, p.b_se1, p.w_se2, p.b_se2,
                           p.gate + (long long)(n0 + jj) * p.Cexp, p.Cexp, p.Cse, g_sm);
            __syncthreads();
            if (p.scale_out) {
                // D of this crop was written by this CTA (visible after the barriers above) and is still in L2
                T* const d_n = out + (long long)(n0 + jj) * p.Ho * p.Ho * p.Cexp;
                const int cv8 = p.Cexp >> 3, total = p.Ho * p.Ho * cv8;
                const float inv_cv8 = 1.0f / (float)cv8;
                for (int v = tid; v < total; v += NT) {
                    const int c8 = (v - div_small(v, inv_cv8) * cv8) * 8;
                    uint4* ptr = reinterpret_cast<uint4*>(d_n) + v;
                    *ptr = tc::scale8s<T>(__ldcg(ptr), tc::smem_u32(g_sm + c8));
                }
            }
        }
    }
    // ---- SE excite by the last CTA of this crop (classic fence + ticket pattern; the sums stay in fixed order; NB == 1 only)
    if (p.se_counter) {
        if (tid == 0) {
            const int ticket = atomicAdd(p.se_counter + n0, 1);
            s_last = ticket == (int)(gridDim.x * gridDim.z) - 1;
            if (s_last) p.se_counter[n0] = 0;
        }
        __syncthreads();
        if (s_last) {
            __threadfence();
            float* sm = reinterpret_cast<float*>(smem_raw + (sE - tc::smem_u32(smem_raw)));    // E is free now
            se_gate_crop<true, NT>(p.partial + (long long)n0 * gridDim.x * p.Cexp, (int)gridDim.x, 1.0f / (float)(p.Ho * p.Ho),
                         p.w_se1t, p.b_se1, p.w_se2, p.b_se2, p.gate + (long long)n0 * p.Cexp, p.Cexp, p.Cse, sm);
        }
    }
}

// One tile plan: TH x TW output tile, R outputs per depthwise strip, CC expanded channels per chunk, NT threads per CTA,
// NB crops per CTA.  Returns false when K1 cannot run it (shape does not divide, shared memory exceeded).
inline bool plan_k1_candidate(int Hin, int Ho, int Cin, int Cexp, int k, int s, int pad, bool is_bf16, int TH, int TW, int R, int CC,
                              int NT, int NB, K1Params* p, size_t* smem_out) {
    if (Ho % TH || Ho % TW || Cexp % CC || (NT != 256 && NT != 512) || NB < 1) return false;
    p->Hin = Hin; p->Ho = Ho; p->Cin = Cin; p->Cexp = Cexp; p->pad = pad;
    p->TH = TH; p->TW = TW;
    p->IH = (TH - 1) * s + k; p->IW = (TW - 1) * s + k;
    p->tiles_x = Ho / TW; p->tiles_y = Ho / TH;
    if (NB > 1 && p->tiles_x * p->tiles_y != 1) return false;
    p->NB = NB;
    // GEMM rows of a CTA = halo pixels inside the image; the largest count over all tiles sizes the A buffer
    int max_in = 0;
    for (int ty = 0; ty < p->tiles_y; ++ty)
        for (int tx = 0; tx < p->tiles_x; ++tx) {
            const int iy0 = ty * TH * s - pad, ix0 = tx * TW * s - pad;
            const int ih = std::min(p->IH, Hin - iy0) - std::max(0, -iy0), iw = std::min(p->IW, Hin - ix0) - std::max(0, -ix0);
            max_in = std::max(max_in, ih * iw);
        }
    p->mtiles = (NB * max_in + BM - 1) / BM;
    if (p->mtiles > 3 || CC > 128) return false;
    p->rows_alloc = (NB * max_in + 7) & ~7;
    p->cpr = ((Cin >> 3) + 1 + 1) & ~1;
    p->nkb = (p->cpr + 7) / 8;
    p->CC = CC; p->n_chunks = Cexp / CC;
    p->chunks_per_cta = p->n_chunks;
    p->pitchE = CC * 2 + 16;
    p->PYc = NT / (CC / 4) / NB;
    p->PY = p->PYc * NB;
    if (p->PYc < 1 || NB * CC > NT) return false;
    const int spr = (TW + R - 1) / R;         // a ragged last strip computes (and discards) up to R-1 extra outputs
    p->spr_log2 = spr == 1 ? 0 : spr == 2 ? 1 : spr == 4 ? 2 : -1;
    if (p->spr_log2 < 0) return false;
    p->smem_A = p->nkb * p->rows_alloc * 128;           // multiple of 1024 (rows_alloc % 8 == 0)
    p->smem_W = p->nkb * CC * 128;                      // multiple of 2048 (CC % 16 == 0)
    p->smem_C = (k * k + 1) * CC * 4;
    // slack rows: a ragged strip still LOADS the columns of its discarded outputs
    p->e_rows = p->IH * p->IW + R * s + 16;
    p->smem_E = NB * p->e_rows * p->pitchE;
    const size_t se_tail_bytes = p->tiles_x * p->tiles_y == 1 ? (size_t)(NB * Cexp + 64) * 4 : 0;     // means + hidden layer
    *smem_out = (size_t)p->smem_A + 2 * p->smem_W + 2 * p->smem_C + p->smem_E + (size_t)p->PY * CC * 4 + se_tail_bytes + 1024;
    // the MMA of the last 64-row half reads 64 rows even when fewer are staged: that read must stay inside the CTA's window
    if ((size_t)(p->nkb - 1) * p->rows_alloc * 128 + (size_t)((p->rows_alloc + 63) / 64) * 64 * 128 + 1024 > *smem_out) return false;
    return *smem_out <= K1_MAX_SMEM;
}

// can two CTAs of this plan share an SM?  (228 KB per SM, 1 KB reserved per CTA)
inline bool k1_two_per_sm(const K1Params& p, size_t smem, int NT) { (void)p; return NT == 256 && smem <= 115000; }

struct K1Choice { int th, tw, r, cc, nt, nb; };

// Per-block plan.  The table holds the plans tools/tune_k1.py measured fastest; blocks without an entry
// (or whose entry does not fit) fall back to a small search ranked by a thread-instruction model.
inline bool plan_k1(int Hin, int Ho, int Cin, int Cexp, int k, int s, int pad, bool is_bf16, bool allow_nb, K1Params* p, K1Choice* choice,
                    size_t* smem_out) {
    struct Tuned { int hin, k, s, cexp; K1Choice c; };
    static const Tuned tuned[] = {
        {112, 3, 2, 96, {8, 8, 4, 48, 256, 1}},      // block 2
        {56, 3, 1, 144, {14, 14, 7, 48, 256, 1}},    // block 3
        {56, 5, 2, 144, {7, 7, 4, 48, 256, 1}},      // block 4
        {28, 5, 1, 240, {14, 14, 7, 48, 256, 1}},    // block 5
        {28, 3, 2, 240, {7, 7, 7, 80, 256, 1}},      // block 6
        {14, 3, 1, 480, {14, 14, 7, 96, 512, 1}},    // blocks 7, 8
        {14, 5, 1, 480, {14, 14, 7, 96, 512, 1}},    // block 9
        {14, 5, 1, 672, {14, 14, 7, 112, 512, 1}},   // blocks 10, 11
        {14, 5, 2, 672, {7, 7, 7, 112, 512, 1}},     // block 12
        {7, 5, 1, 1152, {7, 7, 7, 64, 512, 2}},      // blocks 13-15
        {7, 3, 1, 1152, {7, 7, 7, 96, 512, 2}},      // block 16
        {7, 5, 1, 1152, {7, 7, 4, 64, 256, 1}},      // blocks 13-15 when a CTA may hold one crop only (fused SE tail)
        {7, 3, 1, 1152, {7, 7, 7, 96, 256, 1}},      // block 16, ditto
    };
    for (const Tuned& t : tuned)
        if (t.hin == Hin && t.k == k && t.s == s && t.cexp == Cexp && (allow_nb || t.c.nb == 1)) {
            K1Params q{};
            size_t smem = 0;
            if (plan_k1_candidate(Hin, Ho, Cin, Cexp, k, s, pad, is_bf16, t.c.th, t.c.tw, t.c.r, t.c.cc, t.c.nt, t.c.nb, &q, &smem)) {
                *p = q; *choice = t.c; *smem_out = smem;
                return true;
            }
        }
    struct Cand { int th, tw, r; };
    const Cand s1[] = {{14, 14, 7}, {7, 14, 7}, {7, 7, 7}, {7, 7, 4}};
    const Cand s2k3[] = {{8, 8, 4}, {7, 7, 7}, {7, 7, 4}};
    const Cand s2[] = {{7, 7, 7}, {7, 7, 4}};
    const Cand* cands = s == 1 ? s1 : (k == 3 ? s2k3 : s2);
    const int ncand = s == 1 ? 4 : (k == 3 ? 3 : 2);
    bool found = false;
    double best = -1;
    for (int i = 0; i < ncand; ++i)
        for (int cc = 128; cc >= 16; cc -= 16) {
            K1Params q{};
            size_t smem = 0;
            if (!plan_k1_candidate(Hin, Ho, Cin, Cexp, k, s, pad, is_bf16, cands[i].th, cands[i].tw, cands[i].r, cc, 256, 1, &q, &smem)) continue;
            const bool two = k1_two_per_sm(q, smem, 256);
            // rough thread-instruction model of one CTA (constants from the ncu source view of round 1):
            //   A fill ~20 / (pixel, chunk); per chunk: epilogue-1 ~4 / E element, depthwise ~1.8 x FMA count over
            //   whole rounds of the 256 threads, ~400 / thread of barrier + prefetch overhead
            const int R = cands[i].r, th = cands[i].th, tw = cands[i].tw;
            const double items = (double)(th * ((tw + R - 1) / R)) * (cc / 4);
            const double lanes = (double)q.PY * (cc / 4);
            const double rounds = (double)(long long)((items + lanes - 1) / lanes);
            const double epi = (double)q.mtiles * BM * cc * 4.0;
            const double dw = rounds * 256.0 * R * k * k * 4 * 1.8;
            const double per_cta = (double)q.rows_alloc * (Cin / 8) * 20.0 + q.n_chunks * (epi + dw + 256.0 * 400.0);
            double cost = per_cta / ((double)th * tw * Cexp);
            if (!two) cost *= 1.4;
            if (best < 0 || cost < best) {
                best = cost; *p = q; *choice = K1Choice{th, tw, R, cc, 256, 1}; *smem_out = smem; found = true;
            }
        }
    return found;
}

// Block 1 (no expand conv): 14x14 output tiles, 3x3 stride 1, all 32 channels in one chunk.
inline bool plan_dw_only(int Hin, int C, int k, int s, int pad, K1Params* p, size_t* smem_out) {
    if (k != 3 || s != 1 || Hin % 14 || C % 16 || C > 128) return false;
    *p = K1Params{};
    p->Hin = Hin; p->Ho = Hin; p->Cin = C; p->Cexp = C; p->pad = pad;
    p->TH = 14; p->TW = 14; p->IH = 16; p->IW = 16;
    p->tiles_x = Hin / 14; p->tiles_y = Hin / 14;
    p->mtiles = 2; p->rows_alloc = 256; p->cpr = 2; p->nkb = 1; p->CC = C; p->n_chunks = 1;
    p->NB = 1;
    p->pitchE = C * 2 + 16;
    p->PY = 256 / (C / 4);
    p->PYc = p->PY;
    p->spr_log2 = 1;
    p->smem_A = 0; p->smem_W = 0; p->chunks_per_cta = 1;
    p->smem_C = (((k * k + 1) * C * 4) + 1023) & ~1023;
    p->e_rows = 16 * 16 + 7 + 16;
    p->smem_E = ((p->e_rows * p->pitchE) + 1023) & ~1023;
    *smem_out = (size_t)2 * p->smem_C + p->smem_E + (size_t)p->PY * C * 4 + 1024;
    return true;
}

template <typename T>
int launch_dw_only(cudaStream_t stream, K1Params p, size_t smem, int n_crops) {
    p.N = n_crops;
    dim3 grid(p.tiles_x * p.tiles_y, n_crops, 1);
    auto kfn = k1_expand_dw_kernel<T, 3, 1, 7, true>;
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K1_MAX_SMEM) != cudaSuccess) return -1;
    kfn<<<grid, 256, smem, stream>>>(p);
    return 0;
}

inline bool k1_has_instance(int k, int s, int R) { return (k == 3 || k == 5) && (s == 1 || s == 2) && (R == 4 || R == 7); }

template <typename T>
int launch_k1(cudaStream_t stream, K1Params p, int k, int s, int R, int NT, size_t smem, int n_crops) {
    p.N = n_crops;
    dim3 grid(p.tiles_x * p.tiles_y, (n_crops + p.NB - 1) / p.NB, (p.n_chunks + p.chunks_per_cta - 1) / p.chunks_per_cta);
#define K1_GO(KFN)                                                                                                         \
    do {                                                                                                                   \
        auto kfn = KFN;                                                                                                    \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K1_MAX_SMEM) != cudaSuccess) return -1;  \
        kfn<<<grid, NT, smem, stream>>>(p);                                                                                \
        return 0;                                                                                                          \
    } while (0)
#define K1(KS, S, RR)                                                                      \
    do {                                                                                   \
        if (NT == 512) K1_GO((k1_expand_dw_kernel<T, KS, S, RR, false, 0, 512>));          \
        if (p.CC == 48) K1_GO((k1_expand_dw_kernel<T, KS, S, RR, false, 48, 256>));        \
        K1_GO((k1_expand_dw_kernel<T, KS, S, RR, false, 0, 256>));                         \
    } while (0)
    if (k == 3 && s == 2 && R == 4) K1(3, 2, 4);
    if (k == 3 && s == 1 && R == 7) K1(3, 1, 7);
    if (k == 5 && s == 1 && R == 7) K1(5, 1, 7);
    if (k == 5 && s == 2 && R == 7) K1(5, 2, 7);
    if (k == 3 && s == 2 && R == 7) K1(3, 2, 7);
    if (k == 3 && s == 1 && R == 4) K1(3, 1, 4);
    if (k == 5 && s == 1 && R == 4) K1(5, 1, 4);
    if (k == 5 && s == 2 && R == 4) K1(5, 2, 4);
#undef K1
#undef K1_GO
    return 1;
}

}  // namespace fused
}  // namespace whenet
