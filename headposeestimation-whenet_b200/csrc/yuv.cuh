// yuv.cuh - planar YUV 4:2:0 source pixels for the kernels that read video frames (the detector's letterbox horizontal pass and
// the crop kernel), converted to B, G, R as each pixel is read.
//
// A frame is cv2's contiguous (H * 3/2) x W layout, H and W even: the H x W Y plane, then
//   NV12: one (H/2) x W plane of interleaved (U, V) pairs, U first
//   I420: the (H/2) x (W/2) U plane, then the (H/2) x (W/2) V plane
// The conversion is cv2.cvtColor's COLOR_YUV2BGR_NV12 / COLOR_YUV2BGR_I420: BT.601 limited range in 20-bit fixed point, so a
// kernel that converts each pixel as it reads it gives the bits of cvtColor followed by the BGR path (oracle/yuv_oracle.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace whenet {

enum { kYuvNV12 = 1, kYuvI420 = 2 };    // = WHENET_YUV_NV12 / WHENET_YUV_I420

// u = U - 128, v = V - 128, c = max(0, Y - 16) * 1220542;  B = clip8((c + 2^19 + 2116026 u) >> 20),
// G = clip8((c + 2^19 - 409993 u - 852492 v) >> 20), R = clip8((c + 2^19 + 1673527 v) >> 20).  |sums| < 2^30: no overflow.
__device__ __forceinline__ void yuv_to_bgr(int Y, int U, int V, int bgr[3]) {
    const int u = U - 128, v = V - 128, c = max(0, Y - 16) * 1220542 + (1 << 19);
    bgr[0] = min(max((c + 2116026 * u) >> 20, 0), 255);
    bgr[1] = min(max((c - 409993 * u - 852492 * v) >> 20, 0), 255);
    bgr[2] = min(max((c + 1673527 * v) >> 20, 0), 255);
}

// B, G, R of pixel (y, x) of an H x W frame in layout L whose Y plane starts at `frame`
template <int L>
__device__ __forceinline__ void yuv_pixel(const uint8_t* __restrict__ frame, int H, int W, int y, int x, int bgr[3]) {
    static_assert(L == kYuvNV12 || L == kYuvI420, "NV12 or I420");
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

}  // namespace whenet
