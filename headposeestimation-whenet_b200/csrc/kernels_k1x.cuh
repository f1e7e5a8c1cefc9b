// kernels_k1x.cuh - K1X: K1 (kernels_fused.cuh) for bf16 storage at throughput batches, fed by TMA (blocks 2, 3, 4, 6).
//
// Same tiles, same chunks and - through the device functions it shares with K1 - the same arithmetic in the same order as
// k1_expand_dw_kernel, so the two give the same bits; what differs is how a CTA gets its operands and how often it stops:
//
//   - the input halo tile comes by ONE cp.async.bulk.tensor.4d over the block input [N][H][W][Cin]: box {ROWB / 2 channels,
//     IW, IW, 1} started at the tile's corner (which may be negative).  Channels >= Cin and pixels outside the image arrive
//     as zeros, and GEMM row r IS halo pixel r = E row r: none of K1's per-piece index arithmetic is left.
//   - A and W rows are 64 bytes (SWIZZLE_64B) where Cin + 8 <= 32 (blocks 2-4: K = 32, half of a 128-byte row would be zero
//     fill no MMA reads), else 128 bytes (SWIZZLE_128B).  The smaller footprint lets three CTAs share an SM instead of two.
//   - K1 folds the expand BN shift into the accumulator (a ones chunk in A against the shift columns of wt_aug).  Here the
//     threads write that ones chunk, after the copy has landed, for the rows INSIDE the image only.  A row outside is then
//     all zero, its accumulators are 0 and swish(0) = 0: the TF-SAME zero padding of E falls out of the epilogue unmasked.
//   - per chunk the W slice of wt_aug and the depthwise constants come by TMA / bulk copy on mbarriers, two buffers each.
//   - two CTA barriers per chunk (E complete, E consumed) instead of K1's three plus its cp.async drains; the squeeze sums
//     of a chunk are formed by one warp after the second barrier, off the other warps' path.
//   - the CTAs are persistent: each walks a fixed list of (tile, crop) items, pays its set-up once, and loads the next halo
//     under the depthwise of the current item's last chunk.
//
// One E tile per CTA: the overlap of a CTA's expand with its own depthwise is left to the other CTAs on the SM, as in K1.
#pragma once
#include "kernels_dwse.cuh"

namespace whenet {
namespace fused {

// Bytes per A / W row: K = CIN + 8 (the input channels, then the ones chunk) in one 64-byte SWIZZLE_64B row when it fits in
// 32 channels (blocks 2-4), else one 128-byte SWIZZLE_128B row.  The MMAs read K = 16 KSTEPS channels either way.
__host__ __device__ constexpr int k1x_row_bytes(int cin) { return cin + 8 <= 32 ? 64 : 128; }

// Geometry of one instance: KS x KS stride S depthwise over a HIN x HIN map, TH x TH output tiles, R outputs per strip, CC
// expanded channels per chunk, CIN input channels.  The tile plan (TH, R, CC) is K1's (plan_k1).
template <int KS, int S, int HIN, int TH, int R, int CC, int CIN>
struct K1X {
    static constexpr int NT = 256;
    static constexpr int HO = (HIN + S - 1) / S;
    static constexpr int PAD = ((HO - 1) * S + KS - HIN > 0 ? (HO - 1) * S + KS - HIN : 0) / 2;     // TF-SAME pad_before
    static constexpr int TILES_X = HO / TH, TILES = TILES_X * TILES_X;
    static constexpr int IW = (TH - 1) * S + KS;               // halo tile width
    static constexpr int NPIX = IW * IW;                       // halo pixels = GEMM rows = E rows
    static constexpr int HALVES = (NPIX + 63) / 64;            // 64-row MMA halves, taken in turn by the two warpgroups
    static constexpr int KCH = CIN / 8;                        // 16-byte chunk of an A row that holds the ones
    static constexpr int KSTEPS = ((KCH + 2) & ~1) >> 1;       // K = 16 MMA steps: K1's (cpr >> 1)
    static constexpr int ROWB = k1x_row_bytes(CIN);            // bytes per A / W row
    static constexpr uint32_t ATOM = 8 * ROWB;                 // swizzle atom: 8 rows
    static constexpr int CTAS_PER_SM = ROWB == 64 ? 3 : 2;
    static constexpr int SPR = (TH + R - 1) / R;               // strips per output row (a ragged last strip discards outputs)
    static constexpr int NSTRIPS = TH * SPR;
    static constexpr int CV = CC / 4;                          // 4-channel vectors per pixel
    static constexpr int PY = NT / CV;                         // strip lanes
    static constexpr uint32_t PITCHE = CC * 2 + 16;            // bytes per E row
    static constexpr int E_ROWS = NPIX + R * S + 16;           // slack: a ragged strip still LOADS the columns of its discarded outputs
    static_assert(HO % TH == 0 && CIN % 8 == 0 && KSTEPS * 32 <= ROWB && CC % 16 == 0 && CC <= 128, "tile plan");
    // A rows: the halo pixels rounded up to a swizzle atom.  The last half's MMA reads whole 64 rows, on past A into W (which
    // a TMA refill may be writing): MMA rows are independent and those accumulator rows are never stored.
    static constexpr uint32_t A_BYTES = (NPIX + 7) / 8 * ATOM;
    static constexpr uint32_t A_TX = NPIX * ROWB;
    static constexpr uint32_t W_BYTES = CC * ROWB;
    static constexpr uint32_t E_BYTES = (E_ROWS * PITCHE + 127) / 128 * 128;
    // constants of a chunk: fp16 depthwise weights [KS*KS][CC] (tensor copy: 128-byte aligned), then the CC fp32 shifts
    static constexpr uint32_t DWW_BYTES = KS * KS * CC * 2;
    static constexpr uint32_t CST_TX = DWW_BYTES + CC * 4;
    static constexpr uint32_t CST_BYTES = (CST_TX + 127) / 128 * 128;
    static constexpr uint32_t RED_BYTES = PY * CC * 4;
    // offsets from the 1024-aligned base: A | W[2] | E | constants[2] | squeeze scratch[2]
    static constexpr uint32_t OFF_W = A_BYTES, OFF_E = OFF_W + 2 * W_BYTES, OFF_C = OFF_E + E_BYTES, OFF_R = OFF_C + 2 * CST_BYTES;
    static constexpr size_t SMEM = (size_t)OFF_R + 2 * RED_BYTES + 1024;
    static_assert((A_BYTES | W_BYTES) % ATOM == 0 && OFF_E % 128 == 0 && DWW_BYTES % 16 == 0, "operand alignment");
    static_assert((size_t)HALVES * 64 * ROWB + 1024 <= SMEM, "the last half's MMA stays inside the CTA's window");
    // 228 KB per SM, 1 KB of it reserved per CTA, + the static barriers
    static_assert(CTAS_PER_SM * (SMEM + 1024 + 256) <= 228 * 1024, "CTAS_PER_SM CTAs per SM");
    __device__ static uint32_t sw(int r, int c) { return ROWB == 64 ? sw64(r, c) : sw128(r, c); }
};

// Persistent: the grid is at most one wave of resident CTAs, and CTA b takes the items (tiles x crops, in crop-major order)
// b, b + gridDim.x, b + 2 gridDim.x, ...  Barrier init and tensor-map prefetch happen once per CTA; the halo of the next item
// is loaded under the depthwise of the current item's last chunk, and the W / constants ring runs on across items, indexed
// by the CTA's chunk counter g (buffer g & 1, phase g >> 1).
template <int KS, int S, int HIN, int TH, int R, int CC, int CIN>
__global__ void __launch_bounds__(256, (K1X<KS, S, HIN, TH, R, CC, CIN>::CTAS_PER_SM)) k1x_kernel(const __grid_constant__ DwSeParams p) {
    using X = K1X<KS, S, HIN, TH, R, CC, CIN>;
    using T = __nv_bfloat16;
    extern __shared__ uint8_t smem_k1x[];
    __shared__ __align__(8) uint64_t bars[5];                  // A, W[2], constants[2] (TMA bytes)
    __shared__ int s_abort_mem;
    volatile int* s_abort = &s_abort_mem;
    const uint32_t s0 = (tc::smem_u32(smem_k1x) + 1023u) & ~1023u;
    const uint32_t sA = s0, sW = s0 + X::OFF_W, sE = s0 + X::OFF_E, sC = s0 + X::OFF_C, sR = s0 + X::OFF_R;
    const uint32_t b_a = tc::smem_u32(&bars[0]), b_w = b_a + 8, b_c = b_a + 24;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = tid >> 7, wq = warp & 3;
    const int C = p.C, n_chunks = p.n_chunks;
    const int items = p.N * X::TILES;
    const int n_items = (items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // this CTA's
    const int n_g = n_items * n_chunks;                                                     // ... and their chunks

    if (tid == 0) {
        for (int i = 0; i < 5; ++i) tc::mbar_init(&bars[i], 1);
        s_abort_mem = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmX) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmWx) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
    }
    __syncthreads();

    // async copies (one thread): the halo tile of an item -> A; the W slice of chunk j -> W[g & 1]; its depthwise weights +
    // shifts -> constants[g & 1]
    auto issue_a = [&](int item) {
        const int n = item / X::TILES, tile = item - n * X::TILES, tyi = tile / X::TILES_X;
        tc::mbar::arrive_expect_tx(b_a, X::A_TX);
        tc::mbar::tma_4d(sA, &p.tmX, 0, (tile - tyi * X::TILES_X) * TH * S - X::PAD, tyi * TH * S - X::PAD, n, b_a);
    };
    auto issue_w = [&](int g, int j) {
        const uint32_t bar = b_w + 8 * (g & 1);
        tc::mbar::arrive_expect_tx(bar, X::W_BYTES);
        tc::mbar::tma_2d(sW + (g & 1) * X::W_BYTES, &p.tmWx, 0, j * CC, bar);
    };
    auto issue_c = [&](int g, int j) {
        const uint32_t bar = b_c + 8 * (g & 1), dst = sC + (g & 1) * X::CST_BYTES;
        tc::mbar::arrive_expect_tx(bar, X::CST_TX);
        tc::mbar::tma_2d(dst, &p.tmW, j * CC, 0, bar);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst + X::DWW_BYTES), "l"(p.b_dw + j * CC), "r"((uint32_t)(CC * 4)), "r"(bar) : "memory");
    };
    if (tid == 0) {
        issue_a(blockIdx.x);
        issue_w(0, 0); issue_c(0, 0);
        if (n_g > 1) { issue_w(1, 1 % n_chunks); issue_c(1, 1 % n_chunks); }
    }

    // depthwise: thread = (4-channel vector cv, strip lane py)
    const int py = tid / X::CV, cv = tid - py * X::CV;
    const bool dw_active = py < X::PY;

    int g = 0;
    for (int k = 0, item = blockIdx.x; k < n_items; ++k, item += gridDim.x) {
        const int n = item / X::TILES, tile = item - n * X::TILES;
        const int tyi = tile / X::TILES_X;
        const int ty0 = tyi * TH, tx0 = (tile - tyi * X::TILES_X) * TH;        // output-tile origin
        const int iy0 = ty0 * S - X::PAD, ix0 = tx0 * S - X::PAD;              // halo-tile origin (may be < 0)
        T* const out_t = reinterpret_cast<T*>(p.out) + (((long long)n * X::HO + ty0) * X::HO + tx0) * C + cv * 4;

        // the ones chunk of the rows inside the image (generic-proxy writes over zeros the copy delivered), fenced against
        // the MMAs that read them and against the next item's copy that overwrites them
        tc::mbar::wait(b_a, (uint32_t)k & 1u, s_abort, p.tflag);
        for (int r = tid; r < X::NPIX; r += X::NT) {
            const int ty = r / X::IW, tx = r - ty * X::IW;
            const int iy = iy0 + ty, ix = ix0 + tx;
            if (iy >= 0 && iy < HIN && ix >= 0 && ix < HIN) sts128(sA + X::sw(r, X::KCH), make_uint4(ones2<T>(), 0u, 0u, 0u));
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        // a CTA that has timed out takes no further item (the OR gives every thread the same answer)
        if (__syncthreads_or(*s_abort)) return;

        for (int j = 0; j < n_chunks; ++j, ++g) {
            const int buf = g & 1;
            const uint32_t par = (uint32_t)(g >> 1) & 1u;
            // ---- expand MMA + epilogue: swish -> E (fp16), one 64-row half at a time
            tc::mbar::wait(b_w + 8 * buf, par, s_abort, p.tflag);
            for (int u = wg; u < X::HALVES; u += 2) {
                float d[CC / 2];
                tc::wg_mma_block<true, CC, 1>(*reinterpret_cast<float(*)[1][CC / 2]>(&d), tc::make_desc_rows<X::ROWB>(sA + (uint32_t)u * 64 * X::ROWB), 0,
                                              tc::make_desc_rows<X::ROWB>(sW + buf * X::W_BYTES), X::KSTEPS, 0u);
                tc::wg_wait<0>();
                const int r_lo = u * 64 + 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = r_lo + 8 * hr;
                    if (r < X::NPIX) expand_row_to_e<CC / 16>(d, CC / 16, hr, sE + (uint32_t)r * X::PITCHE, cq);
                }
            }
            // E(j) is complete and every MMA of chunk j is done with W[buf] - and, after the last chunk, with A
            __syncthreads();
            if (tid == 0) {
                if (j == n_chunks - 1 && k + 1 < n_items) issue_a(item + gridDim.x);
                if (g + 2 < n_g) issue_w(g + 2, (j + 2) % n_chunks);
            }

            // ---- depthwise on E
            tc::mbar::wait(b_c + 8 * buf, par, s_abort, p.tflag);
            if (dw_active && !*s_abort) {
                const uint32_t cst = sC + buf * X::CST_BYTES;
                const float4 bq = lds_f4(cst + X::DWW_BYTES + (uint32_t)cv * 16);
                float sum[4] = {0.f, 0.f, 0.f, 0.f};
                for (int sidx = py; sidx < X::NSTRIPS; sidx += X::PY) {
                    const int oyl = sidx / X::SPR, oxl0 = (sidx - oyl * X::SPR) * R;
                    float2 acc[R][2];
                    dw_strip_hfma2<KS, S, R>(sE + (uint32_t)((oyl * S * X::IW + oxl0 * S) * X::PITCHE + cv * 8), X::IW * X::PITCHE, X::PITCHE,
                                             cst + (uint32_t)cv * 8, CC * 2, bq, acc);
                    dw_strip_finish<T, R>(acc, TH - oxl0, out_t + ((long long)oyl * X::HO + oxl0) * C + j * CC, C, sum);
                }
                asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(sR + (uint32_t)(buf * X::RED_BYTES + (py * CC + cv * 4) * 4)),
                             "f"(sum[0]), "f"(sum[1]), "f"(sum[2]), "f"(sum[3]) : "memory");
            }
            // E, the constants and the squeeze scratch of chunk g are read / written
            __syncthreads();
            // the last warp closes the chunk while the others start the next one: squeeze sums in K1's order (strip lanes in
            // four chains), then the refill of the constants buffer.  Scratch[buf] is written again two barriers further on.
            if (warp == X::NT / 32 - 1) {
                squeeze_sums<X::PY, CC>(sR + buf * X::RED_BYTES, p.partial + ((long long)n * X::TILES + tile) * C + j * CC, nullptr, 0.f, lane);
                if (lane == 0 && g + 2 < n_g) issue_c(g + 2, (j + 2) % n_chunks);
            }
        }
    }
}

// the instances: (KS, S, HIN, TH, R, CC, CIN) of blocks 2, 3, 4 and 6 under plan_k1's tuned plans.  Block 5 (5x5 stride 1 over
// 28x28 in four tiles) has none: its instance measured 3 % SLOWER than K1 (DESIGN.md 5.2) and the block stays on K1.  A fifth
// of each of its 18x18 halo tiles lies outside the image; K1 leaves those pixels out of the GEMM (4 row halves), here they
// are rows like any other (6 halves).
#define WHENET_K1X_INSTANCES(F) F(3, 2, 112, 8, 4, 48, 16) F(3, 1, 56, 14, 7, 48, 24) F(5, 2, 56, 7, 4, 48, 24) F(3, 2, 28, 7, 7, 80, 40)

// is there an instance for this block shape under this K1 plan?
inline bool k1x_has_instance(int k, int s, int hin, int cin, int pad, const K1Params& pl, int R) {
#define K1X_MATCH(KS_, S_, HIN_, TH_, R_, CC_, CIN_)                                                                        \
    if (k == KS_ && s == S_ && hin == HIN_ && cin == CIN_ && pl.TH == TH_ && pl.TW == TH_ && R == R_ && pl.CC == CC_ && pl.NB == 1 && \
        pad == K1X<KS_, S_, HIN_, TH_, R_, CC_, CIN_>::PAD)                                                                  \
        return true;
    WHENET_K1X_INSTANCES(K1X_MATCH)
#undef K1X_MATCH
    return false;
}

// A persistent grid over the (tile, crop) items, each with all its chunks: min(items, resident CTAs per SM x SMs), both read
// from the device.  p: tmX = the block input (4-D, box {ROWB / 2, IW, IW, 1}, swizzled as the rows), tmWx = wt_aug (box
// {ROWB / 2, CC}), tmW = the fp16 depthwise weights (box {CC, KS*KS}); b_dw, out, partial, tflag, C.  1: no instance.
template <typename T>
int launch_k1x(cudaStream_t stream, DwSeParams p, int k, int s, int hin, int cin, int th, int r, int cc, int n_crops) {
    static_assert(std::is_same<T, __nv_bfloat16>::value, "K1X runs the bf16 wgmma and the HFMA2 depthwise");
    p.N = n_crops;
    p.n_chunks = p.C / cc;
    p.chunks_per_cta = p.n_chunks;
#define K1X_GO(KS, S, HIN, TH, RR, CC, CIN)                                                                                  \
    if (k == KS && s == S && hin == HIN && cin == CIN && th == TH && r == RR && cc == CC) {                                  \
        using X = K1X<KS, S, HIN, TH, RR, CC, CIN>;                                                                          \
        auto kfn = k1x_kernel<KS, S, HIN, TH, RR, CC, CIN>;                                                                  \
        if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)X::SMEM) != cudaSuccess) return -1;  \
        int dev = 0, sms = 0, per_sm = 0;                                                                                    \
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || \
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, X::NT, X::SMEM) != cudaSuccess || per_sm < 1)        \
            return -1;                                                                                                       \
        const long long items = (long long)X::TILES * n_crops;                                                               \
        kfn<<<(unsigned)std::min(items, (long long)per_sm * sms), X::NT, X::SMEM, stream>>>(p);                              \
        return 0;                                                                                                            \
    }
    WHENET_K1X_INSTANCES(K1X_GO)
#undef K1X_GO
    return 1;
}

}  // namespace fused
}  // namespace whenet
