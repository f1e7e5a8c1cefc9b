// kernels_crop.cuh - crop front-end of the stream path (SURVEY.md section 8f-1).
//
// For every head box: slice [y0:y1, x0:x1] out of its BGR frame, swap to RGB and resize to
// 224x224 exactly as cv2.resize's 8-bit INTER_LINEAR kernel does (reference demo_video.py:21-23,
// demo.py:10-11): half-pixel centres, 11-bit weights rounded to nearest-even, int32 horizontal pass,
// ((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2 >> 2 vertical pass, 2x2 box for exact 2x down-scaling.
// All heads of one frame, of n frames of one size or of n frames of their own sizes come out as ONE uint8 NHWC batch that feeds the
// stem kernel directly - the reference crops, resizes and runs the network one head at a time
// (demo_video.py:13-23, 57-58).  crop_resize_yuv_kernel does the same on NV12 / I420 / YUYV / UYVY frames (yuv.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "yuv.cuh"

namespace whenet {

struct AxisTap { int s0, s1, w0, w1; };

// OpenCV resize(): left source index + the two 11-bit weights for destination index d.
// clamp_weights: x axis resets the fraction at the borders, y axis only clips the row indices.
__device__ __forceinline__ AxisTap axis_tap(int d, int src, bool clamp_weights) {
    const double scale = 1.0 / (224.0 / (double)src);
    float f = (float)(((double)d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    AxisTap t;
    if (clamp_weights) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
        t.s0 = s;
        t.s1 = min(s + 1, src - 1);
    } else {
        t.s0 = min(max(s, 0), src - 1);
        t.s1 = min(max(s + 1, 0), src - 1);
    }
    t.w1 = __float2int_rn(f * 2048.f);              // saturate_cast<short>(float): round half to even
    t.w0 = __float2int_rn((1.f - f) * 2048.f);
    return t;
}

constexpr int kMaxCropFrames = 64;

// n frames of one size H x W x 3, back to back
struct OneSizeFrames {
    const uint8_t* frames;
    int H, W;
};
// n <= kMaxCropFrames frames of their own sizes, each H x W x 3 at its own base (the host checked every rect against its H).
// H locates a YUV frame's chroma plane(s); the BGR kernel does not read it.
struct PerFrameSources {
    struct Frame { const uint8_t* base; int W, H; } f[kMaxCropFrames];
};

// grid = (ceil(224*224/256), M).  src: the frames; rects[m] = (y0, y1, x0, x1) slice bounds inside frame frame_of[m]
// (frame 0 for every crop when frame_of is NULL, OneSizeFrames only).  An empty rect (y1 <= y0 or x1 <= x0) marks an
// invalid crop: it reads nothing and is written as zeros.
template <class Frames>
__global__ void __launch_bounds__(256) crop_resize_kernel(const __grid_constant__ Frames src_frames,
                                                          const int4* __restrict__ rects, const int* __restrict__ frame_of,
                                                          uint8_t* __restrict__ out, int swap_rb) {
    const int m = blockIdx.y;
    const int pix = blockIdx.x * 256 + threadIdx.x;
    if (pix >= 224 * 224) return;
    const int dy = pix / 224, dx = pix - dy * 224;
    const int4 r = rects[m];
    const int y0 = r.x, h = r.y - r.x, x0 = r.z, w = r.w - r.z;
    uint8_t* dst = out + ((long long)m * 224 * 224 + pix) * 3;
    if (h <= 0 || w <= 0) { dst[0] = 0; dst[1] = 0; dst[2] = 0; return; }
    const uint8_t* frame;
    int W;
    if constexpr (std::is_same<Frames, OneSizeFrames>::value) {
        W = src_frames.W;
        const long long f = frame_of ? frame_of[m] : 0;
        frame = src_frames.frames + f * src_frames.H * ((long long)W * 3);
    } else {
        const auto& fr = src_frames.f[frame_of[m]];
        W = fr.W;
        frame = fr.base;
    }
    const long long pitch = (long long)W * 3;
    const uint8_t* src = frame + ((long long)y0 * W + x0) * 3;
    int v[3];
    if (h == 448 && w == 448) {                     // resize(): INTER_LINEAR with exact 2x down-scale -> 2x2 box
        const uint8_t* p = src + (long long)(2 * dy) * pitch + (2 * dx) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = (p[c] + p[3 + c] + p[pitch + c] + p[pitch + 3 + c] + 2) >> 2;
    } else {
        const AxisTap tx = axis_tap(dx, w, true), ty = axis_tap(dy, h, false);
        const uint8_t* r0 = src + (long long)ty.s0 * pitch;
        const uint8_t* r1 = src + (long long)ty.s1 * pitch;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int h0 = r0[tx.s0 * 3 + c] * tx.w0 + r0[tx.s1 * 3 + c] * tx.w1;
            const int h1 = r1[tx.s0 * 3 + c] * tx.w0 + r1[tx.s1 * 3 + c] * tx.w1;
            v[c] = (((ty.w0 * (h0 >> 4)) >> 16) + ((ty.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
        }
    }
    if (swap_rb) { dst[0] = (uint8_t)v[2]; dst[1] = (uint8_t)v[1]; dst[2] = (uint8_t)v[0]; }
    else { dst[0] = (uint8_t)v[0]; dst[1] = (uint8_t)v[1]; dst[2] = (uint8_t)v[2]; }
}

// crop_resize_kernel on YUV frames in layout L (yuv.cuh; OneSizeFrames: H * W * 3/2 bytes apart for 4:2:0, H * W * 2 for
// 4:2:2): each source pixel the
// resize reads is converted to B, G, R first, and the crop is written in RGB order, so it is the crop crop_resize_kernel
// gives with swap_rb on cv2.cvtColor's output.
template <class Frames, int L>
__global__ void __launch_bounds__(256) crop_resize_yuv_kernel(const __grid_constant__ Frames src_frames,
                                                              const int4* __restrict__ rects, const int* __restrict__ frame_of,
                                                              uint8_t* __restrict__ out) {
    const int m = blockIdx.y;
    const int pix = blockIdx.x * 256 + threadIdx.x;
    if (pix >= 224 * 224) return;
    const int dy = pix / 224, dx = pix - dy * 224;
    const int4 r = rects[m];
    const int y0 = r.x, h = r.y - r.x, x0 = r.z, w = r.w - r.z;
    uint8_t* dst = out + ((long long)m * 224 * 224 + pix) * 3;
    if (h <= 0 || w <= 0) { dst[0] = 0; dst[1] = 0; dst[2] = 0; return; }
    const uint8_t* frame;
    int H, W;
    if constexpr (std::is_same<Frames, OneSizeFrames>::value) {
        H = src_frames.H;
        W = src_frames.W;
        const long long f = frame_of ? frame_of[m] : 0;
        frame = src_frames.frames + yuv_frame_offset<L>(f, H, W);
    } else {
        const auto& fr = src_frames.f[frame_of[m]];
        H = fr.H;
        W = fr.W;
        frame = fr.base;
    }
    int v[3], a[3], b[3], c[3], d[3];
    if (h == 448 && w == 448) {                     // the 2x2 box of an exact 2x down-scale
        const int y = y0 + 2 * dy, x = x0 + 2 * dx;
        yuv_pixel<L>(frame, H, W, y, x, a);
        yuv_pixel<L>(frame, H, W, y, x + 1, b);
        yuv_pixel<L>(frame, H, W, y + 1, x, c);
        yuv_pixel<L>(frame, H, W, y + 1, x + 1, d);
#pragma unroll
        for (int k = 0; k < 3; ++k) v[k] = (a[k] + b[k] + c[k] + d[k] + 2) >> 2;
    } else {
        const AxisTap tx = axis_tap(dx, w, true), ty = axis_tap(dy, h, false);
        yuv_pixel<L>(frame, H, W, y0 + ty.s0, x0 + tx.s0, a);
        yuv_pixel<L>(frame, H, W, y0 + ty.s0, x0 + tx.s1, b);
        yuv_pixel<L>(frame, H, W, y0 + ty.s1, x0 + tx.s0, c);
        yuv_pixel<L>(frame, H, W, y0 + ty.s1, x0 + tx.s1, d);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int h0 = a[k] * tx.w0 + b[k] * tx.w1;
            const int h1 = c[k] * tx.w0 + d[k] * tx.w1;
            v[k] = (((ty.w0 * (h0 >> 4)) >> 16) + ((ty.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
        }
    }
    dst[0] = (uint8_t)v[2];
    dst[1] = (uint8_t)v[1];
    dst[2] = (uint8_t)v[0];
}

}  // namespace whenet
