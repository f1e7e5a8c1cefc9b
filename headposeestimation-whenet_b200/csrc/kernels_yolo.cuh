// kernels_yolo.cuh - the YOLOv3 head detector (reference yolo_v3/): letterbox, Darknet-53 + three heads (or tiny YOLOv3's
// 13 convs, six max-pools and two heads) on wgmma, decode + NMS.
//
//   letterbox_h_kernel / letterbox_v_kernel   Pillow's uint8 BICUBIC resample (two integer passes, 22-bit coefficients computed on
//                                             the host exactly as ImagingResample does) + the (128,128,128) canvas and the paste
//                                             (reference utils.py:23-34)
//   letterbox_{h,v}_ragged_kernel              the same two passes over frames of different sizes, one LetterboxFrame each
//   letterbox_h{,_ragged}_yuv_kernel<L>        the horizontal passes over NV12 / I420 / YUYV / UYVY frames, converting each pixel
//                                             as it is read
//   yolo_conv0_kernel<N>                       first conv (3 -> N = 32, tiny: 16, 3x3): im2col row built in shared memory from the
//                                             uint8 canvas through a v/255 table split into bf16 hi + lo parts, one K = 64 wgmma
//                                             block per row
//   conv_igemm_kernel<MODE, UN>                every other conv as an implicit GEMM (M = pixels, N = Cout, K = taps x Cin): the A
//                                             operand is gathered per (tap, 64-channel chunk) with cp.async, out-of-image taps are
//                                             zero-filled (= the padding); concat convs read [upsample(up), skip] virtually
//   yolo_maxpool_kernel                        tiny YOLOv3's 2x2 max-pools (stride 2, or stride 1 with TF SAME padding)
//   yolo_decode_nms_kernel                     one CTA per frame: decode every candidate, per-class score mask, greedy NMS
//   yolo_decode_kernel / yolo_nms_kernel /     the same past kNmsPer x kNmsThreads candidates (model inputs above 608): decode over
//   yolo_pack_kernel                           (candidate blocks x frames), NMS per (class, frame), pack per frame
//
// Storage bf16 NHWC, fp32 accumulation; the output convs write fp32.
#pragma once
#include <vector>

#include "kernels_tc.cuh"
#include "yuv.cuh"

namespace whenet {
namespace yolo {

using tc::BK;
using tc::BM;
using tc::cp_async16_z;
using tc::smem_u32;

// ----------------------------------------------------------------------------- host-visible parameters and plans
enum { kLeaky = 0, kLeakyRes = 1, kLeakyCat = 2, kLinearF32 = 3 };

struct IgemmParams {
    const __nv_bfloat16* in;     // [n][Hi][Wi][Cin - c_up]  (concat: the skip tensor)
    const __nv_bfloat16* up;     // concat: [n][Hi/2][Wi/2][c_up], read at (y >> 1, x >> 1)
    const __nv_bfloat16* wt;     // [N][K], K = k*k*Cin, k index = (ky*k + kx)*Cin + ci
    const float* bias;           // [N]
    const __nv_bfloat16* resid;  // [M][N]
    void* out;                   // [M][N] bf16, fp32 for kLinearF32
    int M, Hi, Wi, Ho, Wo, Cin, c_up, N, k, stride, n_tile, n_stages;
};

// Tile plan of one conv.  It depends on the per-frame shape only, never on the batch size, so a frame's results are the same bits
// whatever batch it runs in: the widest tile (<= 128 columns, what one warpgroup holds in registers) that still gives one frame
// at least one CTA per SM, down to 32 columns.  The ring is as deep as fits two CTAs per SM.
struct IgemmPlan { int n_tile, un, n_stages; size_t smem; };
inline IgemmPlan plan_igemm(int Ho, int Wo, int N, int Cin, int k, int sm_count) {
    IgemmPlan pl{};
    const long long m_tiles = ((long long)Ho * Wo + BM - 1) / BM;
    int n_tile = (N + 15) & ~15;
    if (n_tile > 128) {
        int parts = (N + 127) / 128;
        n_tile = (((N + parts - 1) / parts) + 15) & ~15;
    }
    while (n_tile > 32 && m_tiles * ((N + n_tile - 1) / n_tile) < sm_count) n_tile = ((n_tile / 2) + 15) & ~15;
    pl.n_tile = n_tile;
    pl.un = n_tile <= 32 ? 32 : n_tile <= 64 ? 64 : 128;
    const int nkb = k * k * ((Cin + BK - 1) / BK);
    const size_t stage_bytes = tc::A_STAGE_BYTES + (size_t)pl.un * BK * 2;
    int st = 4;
    while (st > 2 && st * stage_bytes > 100 * 1024) --st;
    pl.n_stages = nkb < st ? (nkb < 2 ? 2 : nkb) : st;
    const size_t out_bytes = tc::acc_tile_bytes(pl.un) + (size_t)BM * ((size_t)(n_tile >> 3) | 1) * 16;
    pl.smem = std::max((size_t)pl.n_stages * stage_bytes, out_bytes) + 1024;
    return pl;
}

// The 75 convolutions (tiny YOLOv3: 13) in Keras weight order; the python twin (and the documentation of every field) is
// yolo_arch.py.  pool: the conv's input is out[src] max-pooled 2x2 with this stride (0: no pool).
struct ConvCfg { int k, stride, cin, cout, src, res, up; bool bn; int head; int pool = 0; };

inline std::vector<ConvCfg> make_table() {
    std::vector<ConvCfg> v;
    auto add = [&](int k, int s, int cin, int cout, int src, bool bn = true, int res = -1, int up = -1, int head = -1) {
        v.push_back(ConvCfg{k, s, cin, cout, src, res, up, bn, head});
        return (int)v.size() - 1;
    };
    int x = add(3, 1, 3, 32, -1), c = 32;
    int skip256 = -1, skip512 = -1;
    const int nfs[5] = {64, 128, 256, 512, 1024}, nbs[5] = {1, 2, 8, 8, 4};
    for (int b = 0; b < 5; ++b) {
        x = add(3, 2, c, nfs[b], x);
        for (int i = 0; i < nbs[b]; ++i) {
            const int y = add(1, 1, nfs[b], nfs[b] / 2, x);
            x = add(3, 1, nfs[b] / 2, nfs[b], y, true, x);
        }
        c = nfs[b];
        if (c == 256) skip256 = x;
        if (c == 512) skip512 = x;
    }
    int last5[3];
    auto five = [&](int x, int cin, int nf, int up, int h) {
        x = add(1, 1, cin, nf, x, true, -1, up);
        for (int i = 0; i < 2; ++i) {
            x = add(3, 1, nf, 2 * nf, x);
            x = add(1, 1, 2 * nf, nf, x);
        }
        last5[h] = x;
        return x;
    };
    x = five(x, 1024, 512, -1, 0);
    int u = add(1, 1, 512, 256, x);
    x = five(skip512, 256 + 512, 256, u, 1);
    u = add(1, 1, 256, 128, x);
    five(skip256, 128 + 256, 128, u, 2);
    int y3[3];
    const int nf3[3] = {512, 256, 128};
    for (int h = 0; h < 3; ++h) y3[h] = add(3, 1, nf3[h], 2 * nf3[h], last5[h]);
    for (int h = 0; h < 3; ++h) add(1, 1, 2 * nf3[h], 0, y3[h], false, -1, -1, h);
    return v;
}

// The 13 convolutions of tiny YOLOv3 (reference model.py:92-122) in Keras weight order (yolo_arch.TINY_LAYERS)
inline std::vector<ConvCfg> make_tiny_table() {
    std::vector<ConvCfg> v;
    auto add = [&](int k, int cin, int cout, int src, int pool = 0, int up = -1, int head = -1) {
        ConvCfg c{k, 1, cin, cout, src, -1, up, head < 0, head};
        c.pool = pool;
        v.push_back(c);
    };
    add(3, 3, 16, -1);
    for (int i = 1; i <= 5; ++i) add(3, 8 << i, 16 << i, i - 1, 2);    // 16 -> 32 ... 256 -> 512, each after a stride-2 pool
    add(3, 512, 1024, 5, 1);                                          // after the stride-1 pool
    add(1, 1024, 256, 6);
    add(1, 256, 128, 7);                                              // upsampled into conv 10
    add(3, 256, 512, 7);
    add(3, 128 + 256, 256, 4, 0, 8);                                  // 3x3 concat conv: [upsample(out[8]), out[4]]
    add(1, 512, 0, 9, 0, -1, 0);
    add(1, 256, 0, 10, 0, -1, 1);
    return v;
}

// anchor_mask (model.py:199): the anchors of head l, anchor-in-layer a.  The host writes the anchors into (l, a) slots in
// this order, so the decode reads slot 3 * l + a for either network.
constexpr int kAnchorMask[3][3] = {{6, 7, 8}, {3, 4, 5}, {0, 1, 2}};
constexpr int kTinyAnchorMask[2][3] = {{3, 4, 5}, {1, 2, 3}};

// input size of a table conv from its source's output size (the pool of a tiny conv: TF SAME, ceil(h / stride))
inline int pooled(int h, int pool) { return pool ? (h + pool - 1) / pool : h; }

// conv_igemm_kernel's epilogue mode for a table conv
inline int igemm_mode(const ConvCfg& c) { return c.head >= 0 ? kLinearF32 : c.up >= 0 ? kLeakyCat : c.res >= 0 ? kLeakyRes : kLeaky; }

constexpr int kNmsThreads = 1024;
constexpr int kNmsPer = 24;             // candidates per thread: 24 x 1024 >= 22,743 (608 x 608)
constexpr int kMaxBoxes = 256;

// The decode + NMS route for more candidates than yolo_decode_nms_kernel holds (kNmsPer * kNmsThreads): one alive bit per
// candidate in shared memory, up to the 1,032,192 candidates of YOLOv3 at 4096 x 4096 (126 KB).
constexpr int kMaxSide = 4096;          // whenet_det_create_large's largest input side
constexpr int kMaxCandidates = 3 * (kMaxSide / 32) * (kMaxSide / 32) * 21;
constexpr int kLargeAliveBytes = kMaxCandidates / 32 * 4;
inline bool large_decode_route(int NC) { return NC > kNmsPer * kNmsThreads; }

// Conv launches put the M tiles on gridDim.y, which holds at most 65,535.  A call with more tiles runs as groups of whole frames,
// this many frames (of hw output pixels each) per group; one frame needs at most 32,768 tiles (conv 1 at 4096 x 4096).
constexpr int kMaxGridY = 65535;
inline int igemm_group_frames(long long hw) {
    const long long g = (long long)kMaxGridY * BM / hw;
    return g < 1 ? 1 : g > (1 << 30) ? (1 << 30) : (int)g;
}
// The launches of a conv over n frames of hw output pixels: fn(f0, nf) for each group of nf frames from frame f0 (one group of
// all n while their tiles fit gridDim.y); stops at and returns the first nonzero fn result.  launch_igemm, launch_igemm32 and
// tools/yolo_plan_dump.cu all go through it.
template <class Fn>
int for_each_frame_group(int n, long long hw, Fn&& fn) {
    const int g = ((long long)n * hw + BM - 1) / BM <= kMaxGridY ? n : igemm_group_frames(hw);
    for (int f0 = 0; f0 < n; f0 += g)
        if (int rc = fn(f0, n - f0 < g ? n - f0 : g)) return rc;
    return 0;
}

constexpr int kMaxFrames = 64;          // frames per detector call (whenet_det_create's max_frames)

// yolo_correct_boxes (model.py:159-161) of one frame, float32 on the host
struct FrameGeo {
    float img_h, img_w;                 // original image size
    float off_y, off_x, scale_y, scale_x;
};

struct DecodeParams {
    const float* head[3];               // [n][gh_l][gw_l][3 * (5 + C)] fp32 logits, l = 0, 1, 2 (13x13, 26x26, 52x52 at 416; tiny: 2 heads)
    float4* cand;                       // workspace [n][NC] boxes (y_min, x_min, y_max, x_max)
    float* cand_score;                  // workspace [n][C][NC]
    float* out_boxes;                   // [n][C * max_boxes][4]
    float* out_scores;                  // [n][C * max_boxes]
    int* out_classes;                   // [n][C * max_boxes]
    int* out_count;                     // [n]
    float anchors[18];                  // (w, h) of head l, anchor-in-layer a at slot 3 * l + a (kAnchorMask / kTinyAnchorMask)
    int gh0, gw0, C, NC, max_boxes;     // NC: candidates of all heads (the walk over the heads ends there)
    float in_h, in_w;                   // model input size
    float score, iou;
    FrameGeo geo[kMaxFrames];           // row f: frame f (a one-size batch repeats one row)
};

// launchers (inst_yolo.cu); each returns 0 or the CUDA error of the launch
struct LetterboxPlan {
    int H, W;                // source frame
    int nw, nh, ox, oy;      // resized size and paste offset on the S_h x S_w canvas
    int y0, rows;            // source rows the vertical pass reads (Pillow's ybox)
    int ksx, ksy;            // coefficients per output column / row
    const int2* xb;          // [nw] (xmin, count)
    const int* kx;           // [nw][ksx]
    const int2* yb;          // [nh] (first row relative to y0, count)
    const int* ky;           // [nh][ksy]
};
// One frame of a batch of differently sized frames: LetterboxPlan's geometry, where its tables sit in the batch's coefficient
// allocation and where its pixels and its horizontal-pass rows sit in the input and tmp buffers (byte offsets).
struct LetterboxFrame {
    long long src, tmp;
    int H, W, nw, nh, ox, oy, y0, rows, ksx, ksy;
    int xb, kx, yb, ky;
};
// yuv_layout 0: packed 8-bit frames (BGR when swap_rb); kYuvNV12 / kYuvI420 / kYuvYUYV / kYuvUYVY: YUV frames (yuv.cuh),
// swap_rb ignored
int launch_letterbox(cudaStream_t s, const LetterboxPlan& lp, const uint8_t* in, uint8_t* tmp, uint8_t* out, int n, int S_h, int S_w, int swap_rb,
                     int yuv_layout);
// plans: n device LetterboxFrame; max_hx: the largest rows * nw among them
int launch_letterbox_ragged(cudaStream_t s, const LetterboxFrame* plans, const char* coef, const uint8_t* in, uint8_t* tmp, uint8_t* out, int n,
                            long long max_hx, int S_h, int S_w, int swap_rb, int yuv_layout);
int launch_conv0(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w0, const float* bias, __nv_bfloat16* out, int n, int S_h, int S_w,
                 int cout);
int launch_igemm(cudaStream_t s, const IgemmParams& p, int mode, int un, size_t smem, int grid_n, int grid_m);
int launch_maxpool(cudaStream_t s, const __nv_bfloat16* in, __nv_bfloat16* out, int n, int H, int W, int C, int stride);
// The one-CTA kernel when NC <= kNmsPer * kNmsThreads, else (or with force_large) decode / NMS / pack.  The second route keeps
// each (frame, class)'s kept keys in keep ([n][C][kMaxBoxes]) and their count in keep_count ([n][C]); it needs both.
int launch_decode_nms(cudaStream_t s, const DecodeParams& p, int n, bool force_large, unsigned long long* keep, int* keep_count);

#ifndef WHENET_YOLO_HOST_ONLY
// ----------------------------------------------------------------------------- letterbox
constexpr int kPrecisionBits = 22;          // Pillow Resample.c PRECISION_BITS (32 - 8 - 2)

__device__ __forceinline__ uint8_t clip8(int v) {
    if (v >= (1 << kPrecisionBits << 8)) return 255;
    if (v <= 0) return 0;
    return (uint8_t)(v >> kPrecisionBits);
}

// Horizontal pass: rows [y0, y0 + rows) of every frame, W -> nw columns.  in: n x H x W x 3 (BGR when swap_rb), tmp: n x rows x nw x 3.
// xb = (xmin, count) per output column, kx = ksize int32 coefficients per output column.
__global__ void letterbox_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ tmp, int H, int W, int nw, int y0, int rows,
                                   const int2* __restrict__ xb, const int* __restrict__ kx, int ksize, int swap_rb) {
    const int f = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * nw) return;
    const int r = (int)(i / nw), x = (int)(i - (long long)r * nw);
    const int2 b = xb[x];
    const int* k = kx + (long long)x * ksize;
    const uint8_t* src = in + (((long long)f * H + y0 + r) * W + b.x) * 3;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < b.y; ++j) {
        const int w = k[j];
        s0 += src[3 * j] * w;
        s1 += src[3 * j + 1] * w;
        s2 += src[3 * j + 2] * w;
    }
    uint8_t* dst = tmp + (((long long)f * rows + r) * nw + x) * 3;
    dst[0] = clip8(swap_rb ? s2 : s0);
    dst[1] = clip8(s1);
    dst[2] = clip8(swap_rb ? s0 : s2);
}

// Vertical pass + canvas: every pixel of the S_h x S_w canvas; inside the pasted nw x nh image at (ox, oy) the vertical sum over tmp
// rows yb = (first row relative to tmp, count), elsewhere 128.
__global__ void letterbox_v_kernel(const uint8_t* __restrict__ tmp, uint8_t* __restrict__ out, int nw, int nh, int rows, int S_h, int S_w,
                                   int ox, int oy, const int2* __restrict__ yb, const int* __restrict__ ky, int ksize) {
    const int f = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S_h * S_w) return;
    const int y = i / S_w, x = i - y * S_w;
    uint8_t* dst = out + ((long long)f * S_h * S_w + i) * 3;
    const int yy = y - oy, xx = x - ox;
    if (yy < 0 || yy >= nh || xx < 0 || xx >= nw) {
        dst[0] = dst[1] = dst[2] = 128;
        return;
    }
    const int2 b = yb[yy];
    const int* k = ky + (long long)yy * ksize;
    const uint8_t* src = tmp + (((long long)f * rows + b.x) * nw + xx) * 3;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < b.y; ++j) {
        const int w = k[j];
        const uint8_t* p = src + (long long)j * nw * 3;
        s0 += p[0] * w;
        s1 += p[1] * w;
        s2 += p[2] * w;
    }
    dst[0] = clip8(s0);
    dst[1] = clip8(s1);
    dst[2] = clip8(s2);
}

// The two passes over n frames that each have their own size: frame blockIdx.y follows plans[blockIdx.y], with the arithmetic of
// letterbox_h_kernel / letterbox_v_kernel, so its canvas is the one those give it alone.  The x grid covers the largest frame.
__global__ void letterbox_h_ragged_kernel(const LetterboxFrame* __restrict__ plans, const char* __restrict__ coef, const uint8_t* __restrict__ in,
                                          uint8_t* __restrict__ tmp, int swap_rb) {
    const LetterboxFrame& P = plans[blockIdx.y];
    const int nw = P.nw, ksize = P.ksx;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)P.rows * nw) return;
    const int r = (int)(i / nw), x = (int)(i - (long long)r * nw);
    const int2 b = reinterpret_cast<const int2*>(coef + P.xb)[x];
    const int* k = reinterpret_cast<const int*>(coef + P.kx) + (long long)x * ksize;
    const uint8_t* src = in + P.src + ((long long)(P.y0 + r) * P.W + b.x) * 3;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < b.y; ++j) {
        const int w = k[j];
        s0 += src[3 * j] * w;
        s1 += src[3 * j + 1] * w;
        s2 += src[3 * j + 2] * w;
    }
    uint8_t* dst = tmp + P.tmp + ((long long)r * nw + x) * 3;
    dst[0] = clip8(swap_rb ? s2 : s0);
    dst[1] = clip8(s1);
    dst[2] = clip8(swap_rb ? s0 : s2);
}

// The horizontal pass over a YUV frame (yuv.cuh): every tap converts its source pixel to B, G, R and accumulates it as
// letterbox_h_kernel does, and the row goes to tmp in RGB order, so tmp holds the bits the BGR pass with swap_rb gives on
// cv2.cvtColor's output.  frame: the frame's Y plane; y: the source row; x0, count, k: the output column's taps.
template <int L>
__device__ __forceinline__ void letterbox_h_yuv_taps(const uint8_t* __restrict__ frame, int H, int W, int y, int x0, int count,
                                                     const int* __restrict__ k, uint8_t* __restrict__ dst) {
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < count; ++j) {
        const int w = k[j];
        int p[3];
        yuv_pixel<L>(frame, H, W, y, x0 + j, p);
        s0 += p[0] * w;
        s1 += p[1] * w;
        s2 += p[2] * w;
    }
    dst[0] = clip8(s2);
    dst[1] = clip8(s1);
    dst[2] = clip8(s0);
}

// letterbox_h_kernel on n YUV frames of one size, H * W * 3/2 (4:2:0) or H * W * 2 (4:2:2) bytes each
template <int L>
__global__ void letterbox_h_yuv_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ tmp, int H, int W, int nw, int y0, int rows,
                                       const int2* __restrict__ xb, const int* __restrict__ kx, int ksize) {
    const int f = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * nw) return;
    const int r = (int)(i / nw), x = (int)(i - (long long)r * nw);
    const int2 b = xb[x];
    letterbox_h_yuv_taps<L>(in + yuv_frame_offset<L>(f, H, W), H, W, y0 + r, b.x, b.y, kx + (long long)x * ksize,
                            tmp + (((long long)f * rows + r) * nw + x) * 3);
}

// letterbox_h_ragged_kernel on YUV frames of their own sizes
template <int L>
__global__ void letterbox_h_ragged_yuv_kernel(const LetterboxFrame* __restrict__ plans, const char* __restrict__ coef,
                                              const uint8_t* __restrict__ in, uint8_t* __restrict__ tmp) {
    const LetterboxFrame& P = plans[blockIdx.y];
    const int nw = P.nw;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)P.rows * nw) return;
    const int r = (int)(i / nw), x = (int)(i - (long long)r * nw);
    const int2 b = reinterpret_cast<const int2*>(coef + P.xb)[x];
    letterbox_h_yuv_taps<L>(in + P.src, P.H, P.W, P.y0 + r, b.x, b.y, reinterpret_cast<const int*>(coef + P.kx) + (long long)x * P.ksx,
                            tmp + P.tmp + ((long long)r * nw + x) * 3);
}

__global__ void letterbox_v_ragged_kernel(const LetterboxFrame* __restrict__ plans, const char* __restrict__ coef, const uint8_t* __restrict__ tmp,
                                          uint8_t* __restrict__ out, int S_h, int S_w) {
    const int f = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S_h * S_w) return;
    const LetterboxFrame& P = plans[f];
    const int y = i / S_w, x = i - y * S_w;
    uint8_t* dst = out + ((long long)f * S_h * S_w + i) * 3;
    const int nw = P.nw, yy = y - P.oy, xx = x - P.ox;
    if (yy < 0 || yy >= P.nh || xx < 0 || xx >= nw) {
        dst[0] = dst[1] = dst[2] = 128;
        return;
    }
    const int2 b = reinterpret_cast<const int2*>(coef + P.yb)[yy];
    const int* k = reinterpret_cast<const int*>(coef + P.ky) + (long long)yy * P.ksy;
    const uint8_t* src = tmp + P.tmp + ((long long)b.x * nw + xx) * 3;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < b.y; ++j) {
        const int w = k[j];
        const uint8_t* p = src + (long long)j * nw * 3;
        s0 += p[0] * w;
        s1 += p[1] * w;
        s2 += p[2] * w;
    }
    dst[0] = clip8(s0);
    dst[1] = clip8(s1);
    dst[2] = clip8(s2);
}

// ----------------------------------------------------------------------------- shared epilogue pieces
__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : 0.1f * x; }

// ----------------------------------------------------------------------------- first conv
// 128 consecutive output pixels per CTA (S_h * S_w is a multiple of 1024: a tile never straddles frames).  A row = 27 taps
// (ky, kx, ci) of v/255 as bf16 hi (K 0..26) and bf16 lo (K 32..58); B row n = [w | 0 | w | 0] (w0: N x 64 bf16, packed by the host).
// N = 32 output channels (YOLOv3) or 16 (tiny YOLOv3).
template <int N>
__global__ void __launch_bounds__(128) yolo_conv0_kernel(const uint8_t* __restrict__ img, const __nv_bfloat16* __restrict__ w0,
                                                         const float* __restrict__ bias, __nv_bfloat16* __restrict__ out, int S_h, int S_w) {
    static_assert(N == 16 || N == 32, "first conv: 16 or 32 outputs");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem0;                      // 128 rows x 128 B
    const uint32_t sW = sA + 128 * 128;             // N rows x 128 B
    const uint32_t sL = sW + N * 128;               // 256 x u32 (hi | lo << 16)
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
        tc::sts128_(sW + (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4)),
                    *reinterpret_cast<const uint4*>(w0 + r * 64 + c * 8));
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
    tc::wg_wait<0>();
    tc::wg_acc_store<N>(acc, sAcc, tid);
    __syncthreads();
    __nv_bfloat16* dst = out + m * N;
#pragma unroll
    for (int u = 0; u < N / 16; ++u) {
        float v[16];
        tc::acc_ld16(sAcc, tid, u * 16, v);
        float o[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) o[j] = leaky(v[j] + bias[u * 16 + j]);
        float a[8], b[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { a[j] = o[j]; b[j] = o[8 + j]; }
        st8<__nv_bfloat16>(dst + u * 16, a);
        st8<__nv_bfloat16>(dst + u * 16 + 8, b);
    }
}

// ----------------------------------------------------------------------------- implicit-GEMM conv
// one 128-pixel x UN-column output tile per CTA; K blocks = (tap, 64-channel chunk) through an n_stages cp.async ring, one wgmma
// commit group per block (the pw_tc2 pipeline)
template <int MODE, int UN>
__global__ void __launch_bounds__(128) conv_igemm_kernel(const __grid_constant__ IgemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    const int tid = threadIdx.x;
    const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr uint32_t w_stage_bytes = UN * BK * 2;
    constexpr uint32_t stage_bytes = tc::A_STAGE_BYTES + w_stage_bytes;
    const int m0 = blockIdx.y * BM;
    const int n0 = blockIdx.x * p.n_tile;
    const int n_valid = min(p.n_tile, p.N - n0);
    const int cchunks = (p.Cin + BK - 1) / BK;
    const int nkb = p.k * p.k * cchunks;
    const int K = p.k * p.k * p.Cin;
    const int pad = p.k >> 1;
    const int hw = p.Ho * p.Wo;

    // this thread's 8 A rows (r0 + 16 i) and its 16-byte chunk c: frame row base and top-left input coordinate
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
        const uint32_t a_st = smem0 + s * stage_bytes, w_st = a_st + tc::A_STAGE_BYTES;
        const int tap = kb / cchunks, cc = kb - tap * cchunks;
        const int ky = tap / p.k, kx = tap - ky * p.k;
        const int c0 = cc * BK;
        const bool cvalid = c0 + c * 8 < p.Cin;
        // source of this chunk: the skip tensor, or (concat, c0 < c_up) the low-resolution tensor at half the coordinates
        const bool from_up = MODE == kLeakyCat && c0 < p.c_up;
        const __nv_bfloat16* src = from_up ? p.up : p.in;
        const int cs = from_up ? p.c_up : p.Cin - p.c_up;
        const int sh = from_up ? 1 : 0;
        const int Ws = p.Wi >> sh;
        const int ch = (from_up ? c0 : c0 - p.c_up) + c * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int iy = iy0[i] + ky, ix = ix0[i] + kx;
            const bool valid = cvalid && iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi;
            const __nv_bfloat16* a = src + ((long long)((rbase[i] + iy) >> sh) * Ws + (ix >> sh)) * cs + ch;
            cp_async16_z(a_st + swz + i * 2048, valid ? a : p.in, valid);
        }
        const __nv_bfloat16* wsrc = p.wt + (long long)(n0 + r0) * K + tap * p.Cin + c0 + c * 8;
#pragma unroll
        for (int i = 0; i < UN / 16; ++i) {
            const bool valid = cvalid && r0 + 16 * i < n_valid;
            cp_async16_z(w_st + swz + i * 2048, valid ? wsrc + (long long)i * 16 * K : p.wt, valid);
        }
    };
    for (int j = 0; j < p.n_stages; ++j) {
        if (j < nkb) fill(j);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    tc::WgAcc<UN> acc;
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % p.n_stages;
        const uint32_t a_st = smem0 + s * stage_bytes, w_st = a_st + tc::A_STAGE_BYTES;
        if (p.n_stages >= 4) asm volatile("cp.async.wait_group 2;" ::: "memory");
        else if (p.n_stages == 3) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        {
            const int cc = kb % cchunks;
            const int krem = min(BK, p.Cin - cc * BK);
            tc::wg_mma_tile<true, UN>(acc, a_st, w_st, (krem + 15) >> 4, kb ? 1u : 0u);
        }
        // refill the stage block kb-1 used once its MMAs have completed
        if (kb >= 1 && kb - 1 + p.n_stages < nkb) {
            tc::wg_wait<1>();
            __syncthreads();
            fill(kb - 1 + p.n_stages);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    tc::wg_wait<0>();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const uint32_t sAcc = smem0;
    tc::wg_acc_store<UN>(acc, sAcc, tid);
    __syncthreads();

    const int rows_valid = min(BM, p.M - m0);
    const bool row_ok = tid < rows_valid;
    const long long m = (long long)m0 + tid;
    if (MODE == kLinearF32) {      // output convs: bias, no activation, fp32 (any N)
        float* out = reinterpret_cast<float*>(p.out);
        if (row_ok)
            for (int j = 0; j < n_valid; ++j) {
                float v;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(sAcc + (uint32_t)(j * tc::kAccPitch + tid) * 4u));
                out[m * p.N + n0 + j] = v + p.bias[n0 + j];
            }
        return;
    }
    const int nch = n_valid >> 3;
    const float inv_nch = 1.0f / (float)(nch > 0 ? nch : 1);
    const int pitch16 = nch | 1;
    uint4* stage = reinterpret_cast<uint4*>(smem_raw + (smem0 + tc::acc_tile_bytes(UN) - smem_u32(smem_raw)));
    for (int c0 = 0; c0 < n_valid; c0 += 16) {
        float v[16];
        tc::acc_ld16(sAcc, tid, c0, v);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = n0 + c0 + h * 8;
            if (c0 + h * 8 >= n_valid) break;
            float o[8];
            const float4 b0 = *reinterpret_cast<const float4*>(p.bias + n), b1 = *reinterpret_cast<const float4*>(p.bias + n + 4);
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = leaky(v[h * 8 + j] + bb[j]);
            if (MODE == kLeakyRes && row_ok) {
                float r[8];
                ld8<__nv_bfloat16>(p.resid + m * p.N + n, r);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] += r[j];
            }
            st8<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(stage + tid * pitch16 + ((c0 >> 3) + h)), o);
        }
    }
    __syncthreads();
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
    for (int idx = tid; idx < rows_valid * nch; idx += 128) {
        const int r = tc::fdiv_small(idx, inv_nch), j = idx - r * nch;
        *reinterpret_cast<uint4*>(out + ((long long)m0 + r) * p.N + n0 + j * 8) = stage[r * pitch16 + j];
    }
}

// ----------------------------------------------------------------------------- max-pool (tiny YOLOv3)
// MaxPooling2D(pool_size 2, padding 'same') with TF's SAME rule: Ho = ceil(H / stride), the window of output y is input rows
// y * stride and y * stride + 1, padding only at the bottom / right, and a padded cell never wins (it is left out).  bf16
// rounding is monotone, so the max of the bf16 inputs is exact.  One thread per 8-channel chunk of an output pixel; C % 8 == 0.
__global__ void __launch_bounds__(256) yolo_maxpool_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int n,
                                                           int H, int W, int C, int stride) {
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride, cc = C >> 3;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n * Ho * Wo * cc) return;
    const int c = (int)(i % cc);
    const long long px = i / cc;
    const int ox = (int)(px % Wo);
    const long long fy = px / Wo;
    const int oy = (int)(fy % Ho), f = (int)(fy / Ho);
    const int y0 = oy * stride, x0 = ox * stride;
    const bool y1 = y0 + 1 < H, x1 = x0 + 1 < W;
    const uint4* src = reinterpret_cast<const uint4*>(in + (((long long)f * H + y0) * W + x0) * C) + c;
    const long long row = (long long)W * cc;            // uint4s per input row
    uint4 v = src[0];
    auto mx = [](uint4& a, uint4 b) {
        __nv_bfloat162* pa = reinterpret_cast<__nv_bfloat162*>(&a);
        const __nv_bfloat162* pb = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) pa[j] = __hmax2(pa[j], pb[j]);
    };
    if (x1) mx(v, src[cc]);
    if (y1) mx(v, src[row]);
    if (x1 && y1) mx(v, src[row + cc]);
    reinterpret_cast<uint4*>(out)[i] = v;
}

// ----------------------------------------------------------------------------- decode + NMS
__device__ __forceinline__ float sigmoidf_(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// TF's IoU (non_max_suppression_op.cc): corners via min/max, 0 when either area <= 0
__device__ __forceinline__ float iou_tf(float4 a, float4 b) {
    const float aymin = fminf(a.x, a.z), aymax = fmaxf(a.x, a.z), axmin = fminf(a.y, a.w), axmax = fmaxf(a.y, a.w);
    const float bymin = fminf(b.x, b.z), bymax = fmaxf(b.x, b.z), bxmin = fminf(b.y, b.w), bxmax = fmaxf(b.y, b.w);
    const float area_a = __fmul_rn(__fsub_rn(aymax, aymin), __fsub_rn(axmax, axmin));
    const float area_b = __fmul_rn(__fsub_rn(bymax, bymin), __fsub_rn(bxmax, bxmin));
    if (area_a <= 0.f || area_b <= 0.f) return 0.f;
    const float iymin = fmaxf(aymin, bymin), ixmin = fmaxf(axmin, bxmin), iymax = fminf(aymax, bymax), ixmax = fminf(axmax, bxmax);
    const float inter = __fmul_rn(fmaxf(__fsub_rn(iymax, iymin), 0.f), fmaxf(__fsub_rn(ixmax, ixmin), 0.f));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// Decode candidate i of frame f (model.py:125-187; candidates ordered layer 0, 1 (, 2), then (y, x, anchor)) with the frame's
// yolo_correct_boxes row g: its box to cand[i], its class scores to cscore[c * NC + i].  yolo_decode_kernel's body; the loop of
// yolo_decode_nms_kernel does the same operations in the same order.
__device__ __forceinline__ void decode_candidate(const DecodeParams& p, const FrameGeo& g, int f, int i, float4* cand, float* cscore) {
    const int CH = 5 + p.C;
    int l = 0, rem = i;
    int gh = p.gh0, gw = p.gw0;
    while (rem >= 3 * gh * gw) { rem -= 3 * gh * gw; ++l; gh *= 2; gw *= 2; }
    const int cell = rem / 3, a = rem - cell * 3;
    const int y = cell / gw, x = cell - y * gw;
    const float* t = p.head[l] + (((long long)f * gh + y) * gw + x) * 3 * CH + a * CH;
    const int an = 3 * l + a;                                           // the host put anchor_mask[l][a] in this slot
    const float bx = __fdiv_rn(__fadd_rn(sigmoidf_(t[0]), (float)x), (float)gw);
    const float by = __fdiv_rn(__fadd_rn(sigmoidf_(t[1]), (float)y), (float)gh);
    const float bw = __fdiv_rn(__fmul_rn(expf(t[2]), p.anchors[2 * an]), p.in_w);
    const float bh = __fdiv_rn(__fmul_rn(expf(t[3]), p.anchors[2 * an + 1]), p.in_h);
    // yolo_correct_boxes (model.py:153-176)
    const float yc = __fmul_rn(__fsub_rn(by, g.off_y), g.scale_y), xc = __fmul_rn(__fsub_rn(bx, g.off_x), g.scale_x);
    const float hh = __fmul_rn(bh, g.scale_y), ww = __fmul_rn(bw, g.scale_x);
    const float hh2 = __fdiv_rn(hh, 2.0f), ww2 = __fdiv_rn(ww, 2.0f);
    cand[i] = make_float4(__fmul_rn(__fsub_rn(yc, hh2), g.img_h), __fmul_rn(__fsub_rn(xc, ww2), g.img_w),
                          __fmul_rn(__fadd_rn(yc, hh2), g.img_h), __fmul_rn(__fadd_rn(xc, ww2), g.img_w));
    const float conf = sigmoidf_(t[4]);
    for (int c = 0; c < p.C; ++c) cscore[(long long)c * p.NC + i] = __fmul_rn(conf, sigmoidf_(t[5 + c]));
}

__global__ void __launch_bounds__(kNmsThreads) yolo_decode_nms_kernel(const __grid_constant__ DecodeParams p) {
    const int f = blockIdx.x, tid = threadIdx.x;
    const int CH = 5 + p.C;
    // the frame's row through shared memory: read from the parameter bank by a register index, it costs the decode loop a
    // register it does not have at 32 per thread, and spills
    __shared__ FrameGeo g;
    if (tid == 0) g = p.geo[f];
    __syncthreads();
    float4* cand = p.cand + (long long)f * p.NC;
    float* cscore = p.cand_score + (long long)f * p.C * p.NC;
    // ---- decode (model.py:125-187): decode_candidate's operations, kept inline here because calling it changes this kernel's
    // register allocation
    for (int i = tid; i < p.NC; i += kNmsThreads) {
        int l = 0, rem = i;
        int gh = p.gh0, gw = p.gw0;
        while (rem >= 3 * gh * gw) { rem -= 3 * gh * gw; ++l; gh *= 2; gw *= 2; }
        const int cell = rem / 3, a = rem - cell * 3;
        const int y = cell / gw, x = cell - y * gw;
        const float* t = p.head[l] + (((long long)f * gh + y) * gw + x) * 3 * CH + a * CH;
        const int an = 3 * l + a;                                           // the host put anchor_mask[l][a] in this slot
        const float bx = __fdiv_rn(__fadd_rn(sigmoidf_(t[0]), (float)x), (float)gw);
        const float by = __fdiv_rn(__fadd_rn(sigmoidf_(t[1]), (float)y), (float)gh);
        const float bw = __fdiv_rn(__fmul_rn(expf(t[2]), p.anchors[2 * an]), p.in_w);
        const float bh = __fdiv_rn(__fmul_rn(expf(t[3]), p.anchors[2 * an + 1]), p.in_h);
        // yolo_correct_boxes (model.py:153-176)
        const float yc = __fmul_rn(__fsub_rn(by, g.off_y), g.scale_y), xc = __fmul_rn(__fsub_rn(bx, g.off_x), g.scale_x);
        const float hh = __fmul_rn(bh, g.scale_y), ww = __fmul_rn(bw, g.scale_x);
        const float hh2 = __fdiv_rn(hh, 2.0f), ww2 = __fdiv_rn(ww, 2.0f);
        cand[i] = make_float4(__fmul_rn(__fsub_rn(yc, hh2), g.img_h), __fmul_rn(__fsub_rn(xc, ww2), g.img_w),
                              __fmul_rn(__fadd_rn(yc, hh2), g.img_h), __fmul_rn(__fadd_rn(xc, ww2), g.img_w));
        const float conf = sigmoidf_(t[4]);
        for (int c = 0; c < p.C; ++c) cscore[(long long)c * p.NC + i] = __fmul_rn(conf, sigmoidf_(t[5 + c]));
    }
    __syncthreads();
    __shared__ unsigned long long s_red[kNmsThreads / 32];
    __shared__ unsigned long long s_best;
    int kept_total = 0;
    for (int c = 0; c < p.C; ++c) {
        const float* sc = cscore + (long long)c * p.NC;
        // alive bit j: candidate tid + j * 1024 passes the class mask (model.py:211: score >= threshold) and is not suppressed yet
        uint32_t alive = 0u;
#pragma unroll
        for (int j = 0; j < kNmsPer; ++j) {
            const int i = tid + j * kNmsThreads;
            if (i < p.NC && sc[i] >= p.score) alive |= 1u << j;
        }
        // greedy NMS (tf.image.non_max_suppression): the highest remaining score is never suppressed by an already kept box (those
        // were removed when each was kept), so it is the next box kept; equal scores: lower candidate index first
        int kept = 0;
        while (kept < p.max_boxes) {
            unsigned long long best = 0ull;
#pragma unroll
            for (int j = 0; j < kNmsPer; ++j)
                if (alive & (1u << j)) {
                    const int i = tid + j * kNmsThreads;
                    // scores are >= 0: their float bits order like the floats; ~i makes the lower index win a tie
                    const unsigned long long key = ((unsigned long long)__float_as_uint(sc[i]) << 32) | (unsigned)(~i);
                    best = key > best ? key : best;
                }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o);
                best = v > best ? v : best;
            }
            if ((tid & 31) == 0) s_red[tid >> 5] = best;
            __syncthreads();
            if (tid < 32) {
                unsigned long long v = s_red[tid];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
                    v = u > v ? u : v;
                }
                if (tid == 0) s_best = v;
            }
            __syncthreads();
            best = s_best;
            __syncthreads();                                        // s_red / s_best are rewritten by the next round
            if (best == 0ull) break;
            const int bi = (int)(~(unsigned)(best & 0xffffffffu));
            const float4 bb = cand[bi];
            if (tid == 0) {
                const long long o = (long long)f * p.C * p.max_boxes + kept_total + kept;
                reinterpret_cast<float4*>(p.out_boxes)[o] = bb;
                p.out_scores[o] = __uint_as_float((unsigned)(best >> 32));
                p.out_classes[o] = c;
            }
#pragma unroll
            for (int j = 0; j < kNmsPer; ++j)
                if (alive & (1u << j)) {
                    const int i = tid + j * kNmsThreads;
                    if (i == bi || iou_tf(cand[i], bb) > p.iou) alive &= ~(1u << j);
                }
            ++kept;
        }
        kept_total += kept;
    }
    if (tid == 0) p.out_count[f] = kept_total;
}

// ----------------------------------------------------------------------------- decode + NMS past kNmsPer * kNmsThreads candidates
// Three kernels with yolo_decode_nms_kernel's arithmetic, keys and order: the decode over (candidate blocks x frames), greedy NMS
// per (class, frame) with one alive bit per candidate in shared memory, and the pack into the outputs' class-by-class layout.
__global__ void __launch_bounds__(256) yolo_decode_kernel(const __grid_constant__ DecodeParams p) {
    const int f = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= p.NC) return;
    const FrameGeo g = p.geo[f];
    decode_candidate(p, g, f, i, p.cand + (long long)f * p.NC, p.cand_score + (long long)f * p.C * p.NC);
}

// The largest key of the CTA (kNmsThreads threads) to every thread
__device__ __forceinline__ unsigned long long block_max_key(unsigned long long v, unsigned long long* s_red, unsigned long long* s_best) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
        v = u > v ? u : v;
    }
    if ((tid & 31) == 0) s_red[tid >> 5] = v;
    __syncthreads();
    if (tid < 32) {
        v = s_red[tid];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
            v = u > v ? u : v;
        }
        if (tid == 0) *s_best = v;
    }
    __syncthreads();
    v = *s_best;
    __syncthreads();                                                // s_red / s_best are rewritten by the next call
    return v;
}

// Greedy NMS of class blockIdx.x of frame blockIdx.y.  Alive word w (dynamic shared memory) holds candidates 32w .. 32w + 31;
// thread t owns words t, t + kNmsThreads, ... and alone clears their bits.  Each round suppresses against the box just kept and
// finds the next largest key among the survivors in the same pass.  Kept keys go to keep[(f * C + c) * kMaxBoxes + k].
__global__ void __launch_bounds__(kNmsThreads) yolo_nms_kernel(const __grid_constant__ DecodeParams p, unsigned long long* __restrict__ keep,
                                                               int* __restrict__ keep_count) {
    extern __shared__ uint32_t s_alive[];
    __shared__ unsigned long long s_red[kNmsThreads / 32];
    __shared__ unsigned long long s_best;
    const int c = blockIdx.x, f = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
    const float4* cand = p.cand + (long long)f * p.NC;
    const float* sc = p.cand_score + ((long long)f * p.C + c) * p.NC;
    const int nw = (p.NC + 31) >> 5;
    // the class mask (model.py:211: score >= threshold), one coalesced ballot per word
    for (int w = tid >> 5; w < nw; w += kNmsThreads / 32) {
        const int i = w * 32 + lane;
        const uint32_t b = __ballot_sync(0xffffffffu, i < p.NC && sc[i] >= p.score);
        if (lane == 0) s_alive[w] = b;
    }
    __syncthreads();
    // scores are >= 0: their float bits order like the floats; ~i makes the lower index win a tie
    auto key = [&](int i) { return ((unsigned long long)__float_as_uint(sc[i]) << 32) | (unsigned)(~i); };
    unsigned long long best = 0ull;
    for (int w = tid; w < nw; w += kNmsThreads)
        for (uint32_t b = s_alive[w]; b; b &= b - 1u) {
            const unsigned long long k = key(w * 32 + __ffs(b) - 1);
            best = k > best ? k : best;
        }
    unsigned long long* out = keep + ((long long)f * p.C + c) * kMaxBoxes;
    int kept = 0;
    while (kept < p.max_boxes) {
        best = block_max_key(best, s_red, &s_best);
        if (best == 0ull) break;
        if (tid == 0) out[kept] = best;
        if (++kept == p.max_boxes) break;
        const int bi = (int)(~(unsigned)(best & 0xffffffffu));
        const float4 bb = cand[bi];
        best = 0ull;
        for (int w = tid; w < nw; w += kNmsThreads) {
            uint32_t a = s_alive[w];
            for (uint32_t b = a; b; b &= b - 1u) {
                const int j = __ffs(b) - 1, i = w * 32 + j;
                if (i == bi || iou_tf(cand[i], bb) > p.iou) {
                    a &= ~(1u << j);
                } else {
                    const unsigned long long k = key(i);
                    best = k > best ? k : best;
                }
            }
            s_alive[w] = a;
        }
    }
    if (tid == 0) keep_count[f * p.C + c] = kept;
}

// frame blockIdx.x: its classes' kept boxes in order, class by class, and its count
__global__ void __launch_bounds__(256) yolo_pack_kernel(const __grid_constant__ DecodeParams p, const unsigned long long* __restrict__ keep,
                                                        const int* __restrict__ keep_count) {
    const int f = blockIdx.x;
    const float4* cand = p.cand + (long long)f * p.NC;
    int base = 0;
    for (int c = 0; c < p.C; ++c) {
        const int k = keep_count[f * p.C + c];
        const unsigned long long* kk = keep + ((long long)f * p.C + c) * kMaxBoxes;
        for (int j = threadIdx.x; j < k; j += 256) {
            const unsigned long long key = kk[j];
            const long long o = (long long)f * p.C * p.max_boxes + base + j;
            reinterpret_cast<float4*>(p.out_boxes)[o] = cand[(int)(~(unsigned)(key & 0xffffffffu))];
            p.out_scores[o] = __uint_as_float((unsigned)(key >> 32));
            p.out_classes[o] = c;
        }
        base += k;
    }
    if (threadIdx.x == 0) p.out_count[f] = base;
}

#endif  // WHENET_YOLO_HOST_ONLY
}  // namespace yolo
}  // namespace whenet
