// yuv.cuh - YUV source pixels for the kernels that read video frames (the detector's letterbox horizontal pass and the crop
// kernel), converted to B, G, R as each pixel is read, and the kernel that converts whole frames to BGR.
//
// A 4:2:0 frame is cv2's contiguous (H * 3/2) x W layout, H and W even: the H x W Y plane, then
//   NV12: one (H/2) x W plane of interleaved (U, V) pairs, U first
//   I420: the (H/2) x (W/2) U plane, then the (H/2) x (W/2) V plane
// A packed 4:2:2 frame is H x W x 2 bytes, W even, any H: row y holds W/2 pixel pairs, pair p at byte 4p of the row as
//   YUYV: Y0 U Y1 V
//   UYVY: U Y0 V Y1
// where both pixels of the pair share its U and V.
// The conversion is cv2.cvtColor's COLOR_YUV2BGR_NV12 / _I420 / _YUYV / _UYVY: BT.601 limited range in 20-bit fixed point, so
// a kernel that converts each pixel as it reads it gives the bits of cvtColor followed by the BGR path (oracle/yuv_oracle.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace whenet {

enum { kYuvNV12 = 1, kYuvI420 = 2, kYuvYUYV = 3, kYuvUYVY = 4 };    // = WHENET_YUV_NV12 / _I420 / _YUYV / _UYVY

__host__ __device__ constexpr bool yuv422(int L) { return L == kYuvYUYV || L == kYuvUYVY; }

// u = U - 128, v = V - 128, c = max(0, Y - 16) * 1220542;  B = clip8((c + 2^19 + 2116026 u) >> 20),
// G = clip8((c + 2^19 - 409993 u - 852492 v) >> 20), R = clip8((c + 2^19 + 1673527 v) >> 20).  |sums| < 2^30: no overflow.
__device__ __forceinline__ void yuv_to_bgr(int Y, int U, int V, int bgr[3]) {
    const int u = U - 128, v = V - 128, c = max(0, Y - 16) * 1220542 + (1 << 19);
    bgr[0] = min(max((c + 2116026 * u) >> 20, 0), 255);
    bgr[1] = min(max((c - 409993 * u - 852492 * v) >> 20, 0), 255);
    bgr[2] = min(max((c + 1673527 * v) >> 20, 0), 255);
}

// B, G, R of pixel (y, x) of an H x W frame in layout L that starts at `frame`
template <int L>
__device__ __forceinline__ void yuv_pixel(const uint8_t* __restrict__ frame, int H, int W, int y, int x, int bgr[3]) {
    static_assert(L == kYuvNV12 || L == kYuvI420 || yuv422(L), "NV12, I420, YUYV or UYVY");
    if constexpr (yuv422(L)) {
        const uint8_t* p = frame + ((long long)y * W + (x & ~1)) * 2;       // the pixel's pair
        if constexpr (L == kYuvYUYV) yuv_to_bgr(p[(x & 1) * 2], p[1], p[3], bgr);
        else yuv_to_bgr(p[1 + (x & 1) * 2], p[0], p[2], bgr);
        return;
    } else {
        const uint8_t* uv = frame + (long long)H * W;
        int U, V;
        if constexpr (L == kYuvNV12) {
            const uint8_t* p = uv + (long long)(y >> 1) * W + (x & ~1);
            U = p[0];
            V = p[1];
        } else {
            const long long q = (long long)(y >> 1) * (W >> 1) + (x >> 1);
            U = uv[q];
            V = uv[q + (long long)(H >> 1) * (W >> 1)];
        }
        yuv_to_bgr(frame[(long long)y * W + x], U, V, bgr);
    }
}

// Byte offset of frame f of a batch of H x W frames in layout L, back to back
template <int L>
__device__ __forceinline__ long long yuv_frame_offset(long long f, int H, int W) {
    if constexpr (yuv422(L)) return f * H * W * 2;
    else return f * H * W / 2 * 3;
}

// ----------------------------------------------------------------------------- whole frames -> BGR (whenet_yuv_to_bgr_*)
constexpr int kMaxConvertFrames = 64;

// n <= kMaxConvertFrames frames: each converts src (layout L, H x W) into dst (H x W x 3 BGR, contiguous)
struct YuvConvertFrames {
    struct Frame { const uint8_t* src; uint8_t* dst; int H, W; } f[kMaxConvertFrames];
};

__device__ __forceinline__ void store_bgr(uint8_t* __restrict__ d, const int bgr[3]) {
    d[0] = (uint8_t)bgr[0];
    d[1] = (uint8_t)bgr[1];
    d[2] = (uint8_t)bgr[2];
}

// grid = (ceil(units of the largest frame / 256), n).  A thread owns one unit of frame blockIdx.y: a pixel pair (4:2:2), read
// as one 32-bit word, or a 2 x 2 block (4:2:0), its Y pairs and NV12's (U, V) pair read as 16-bit words.  Those loads are
// aligned whenever the frame's base is (W is even); a frame whose base is not reads the same bytes one by one.
template <int L>
__global__ void __launch_bounds__(256) yuv_to_bgr_kernel(const __grid_constant__ YuvConvertFrames frames) {
    const auto& fr = frames.f[blockIdx.y];
    const int H = fr.H, W = fr.W, hw = W >> 1;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    int a[3], b[3];
    if constexpr (yuv422(L)) {
        if (i >= (long long)H * hw) return;
        const uint8_t* p = fr.src + i * 4;                      // pair i of the frame: row i / hw, pixels 2 (i % hw) and + 1
        uint32_t w;
        if ((reinterpret_cast<uintptr_t>(fr.src) & 3) == 0) w = *reinterpret_cast<const uint32_t*>(p);
        else w = p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
        const int b0 = w & 255, b1 = (w >> 8) & 255, b2 = (w >> 16) & 255, b3 = w >> 24;
        if constexpr (L == kYuvYUYV) { yuv_to_bgr(b0, b1, b3, a); yuv_to_bgr(b2, b1, b3, b); }
        else { yuv_to_bgr(b1, b0, b2, a); yuv_to_bgr(b3, b0, b2, b); }
        uint8_t* d = fr.dst + i * 6;
        store_bgr(d, a);
        store_bgr(d + 3, b);
    } else {
        if (i >= (long long)(H >> 1) * hw) return;
        const long long by = i / hw, bx = i - by * hw;          // block (by, bx): rows 2 by and + 1, columns 2 bx and + 1
        const uint8_t* y0 = fr.src + 2 * by * W + 2 * bx;
        const uint8_t* uv = fr.src + (long long)H * W;
        const bool aligned = (reinterpret_cast<uintptr_t>(fr.src) & 1) == 0;
        int Y[4], U, V;
        if (aligned) {
            const uint16_t r0 = *reinterpret_cast<const uint16_t*>(y0), r1 = *reinterpret_cast<const uint16_t*>(y0 + W);
            Y[0] = r0 & 255; Y[1] = r0 >> 8; Y[2] = r1 & 255; Y[3] = r1 >> 8;
        } else {
            Y[0] = y0[0]; Y[1] = y0[1]; Y[2] = y0[W]; Y[3] = y0[W + 1];
        }
        if constexpr (L == kYuvNV12) {
            const uint8_t* p = uv + by * W + 2 * bx;
            if (aligned) {
                const uint16_t c = *reinterpret_cast<const uint16_t*>(p);
                U = c & 255; V = c >> 8;
            } else {
                U = p[0]; V = p[1];
            }
        } else {
            U = uv[i];
            V = uv[i + (long long)(H >> 1) * hw];
        }
        uint8_t* d = fr.dst + (2 * by * W + 2 * bx) * 3;
        yuv_to_bgr(Y[0], U, V, a); store_bgr(d, a);
        yuv_to_bgr(Y[1], U, V, b); store_bgr(d + 3, b);
        d += (long long)W * 3;
        yuv_to_bgr(Y[2], U, V, a); store_bgr(d, a);
        yuv_to_bgr(Y[3], U, V, b); store_bgr(d + 3, b);
    }
}

}  // namespace whenet
