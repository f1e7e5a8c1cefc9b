// Head overlay: thickness-2 LINE_8 segments (OpenCV's cv2.line(img, p0, p1, color, 2) bit for bit, oracle/draw_oracle.py)
// rasterised into BGR frames in place.  The host (frames_api.cu) clips each segment's end points against the frame grown by
// the thickness and computes its 16.16 quad; everything here is integer arithmetic except the outline clip, which is the
// same double multiply-then-divide OpenCV truncates (no add, so nothing to contract).
//
// One thread owns one row of one frame and walks that frame's segments in order, writing the pixels each covers on its row:
// later segments overwrite earlier ones with no atomics, and the result does not depend on how frames are batched.
#pragma once
#include <cstdint>

namespace whenet {

constexpr int kOverlayMaxFrames = 64;     // = kMaxCropFrames

struct OverlaySeg {
    long long vx[4], vy[4];   // quad vertices p0 + dp, p0 - dp, p1 - dp, p1 + dp (16.16); unused when !quad
    int q0x, q0y, q1x, q1y;   // clipped end points (caps)
    int y_lo, y_hi;           // rows the segment can cover, clipped to the frame
    int quad;                 // the clipped end points differ
    uint32_t bgr;             // b | g << 8 | r << 16
};

struct OverlayFrames {
    uint8_t* ptr[kOverlayMaxFrames];
    int H[kOverlayMaxFrames], W[kOverlayMaxFrames];
    int seg_begin[kOverlayMaxFrames + 1];   // frame f's segments: [seg_begin[f], seg_begin[f + 1])
};

__host__ __device__ inline long long ov_floor_div(long long a, long long b) {
    long long q = a / b;
    return (q * b != a && ((a < 0) != (b < 0))) ? q - 1 : q;
}
__host__ __device__ inline long long ov_ceil_div(long long a, long long b) { return -ov_floor_div(-a, b); }

__host__ __device__ inline void ov_put(uint8_t* row, int W, long long x, uint32_t bgr) {
    if (x < 0 || x >= W) return;
    uint8_t* p = row + 3 * x;
    p[0] = (uint8_t)bgr; p[1] = (uint8_t)(bgr >> 8); p[2] = (uint8_t)(bgr >> 16);
}

__host__ __device__ inline void ov_span(uint8_t* row, int W, long long a, long long b, uint32_t bgr) {
    if (a < 0) a = 0;
    if (b > W - 1) b = W - 1;
    for (long long x = a; x <= b; ++x) ov_put(row, W, x, bgr);
}

// OpenCV's clipLine (Cohen-Sutherland, one pass per axis) against [0, w-1] x [0, h-1]
__host__ __device__ inline bool ov_clip(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
    if (w <= 0 || h <= 0) return false;
    const long long right = w - 1, bottom = h - 1;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (long long)((double)(a - y1) * (double)(x2 - x1) / (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (long long)((double)(a - y2) * (double)(x2 - x1) / (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (long long)((double)(a - x1) * (double)(y2 - y1) / (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (long long)((double)(a - x2) * (double)(y2 - y1) / (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// The pixels of one outline edge (a 16.16 line stepped one pixel per major-axis step) on row y.  The stepper's k-th pixel is
// a closed form of k: its incremental adds are exact integer arithmetic.
__host__ __device__ inline void ov_outline_row(uint8_t* row, int H, int W, int y, long long x1, long long y1, long long x2, long long y2,
                                               uint32_t bgr) {
    if (!ov_clip((long long)W << 16, (long long)H << 16, x1, y1, x2, y2)) return;
    long long dx = x2 - x1, dy = y2 - y1;
    const bool xmajor = (dx < 0 ? -dx : dx) > (dy < 0 ? -dy : dy);
    if (xmajor ? dx < 0 : dy < 0) {
        long long t = x1; x1 = x2; x2 = t;
        t = y1; y1 = y2; y2 = t;
        dx = -dx; dy = -dy;
    }
    if (((y2 + 32768) >> 16) == y) ov_put(row, W, (x2 + 32768) >> 16, bgr);
    if (xmajor) {
        const long long step = (dy << 16) / (dx | 1), count = (x2 - x1) >> 16;
        const long long X = (x1 + 32768) >> 16, Y = y1 + 32768;
        const long long A = ((long long)y << 16) - Y, B = A + 65535;     // want A <= k * step <= B
        long long k0, k1;
        if (step == 0) {
            if (A > 0 || B < 0) return;
            k0 = 0; k1 = count;
        } else if (step > 0) {
            k0 = ov_ceil_div(A, step); k1 = ov_floor_div(B, step);
        } else {
            k0 = ov_ceil_div(B, step); k1 = ov_floor_div(A, step);
        }
        if (k0 < 0) k0 = 0;
        if (k1 > count) k1 = count;
        for (long long k = k0; k <= k1; ++k) ov_put(row, W, X + k, bgr);
    } else {
        const long long step = (dx << 16) / ((dy < 0 ? -dy : dy) | 1), count = (y2 - y1) >> 16;
        const long long k = y - ((y1 + 32768) >> 16);
        if (k >= 0 && k <= count) ov_put(row, W, (x1 + 32768 + k * step) >> 16, bgr);
    }
}

// The quad's scan conversion on row y: OpenCV's two edge chains from the top vertex, each edge picked up at the row its
// predecessor ends, x advanced by a rounded per-row increment.  Only the pick-ups are walked; x at row y is closed form.
__host__ __device__ inline void ov_fill_row(uint8_t* row, int H, int W, int y, const long long* vx, const long long* vy, uint32_t bgr) {
    int imin = 0;
    long long xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
    for (int i = 1; i < 4; ++i) {
        if (vy[i] < ymin) { ymin = vy[i]; imin = i; }
        ymax = vy[i] > ymax ? vy[i] : ymax;
        xmax = vx[i] > xmax ? vx[i] : xmax;
        xmin = vx[i] < xmin ? vx[i] : xmin;
    }
    xmin = (xmin + 32768) >> 16; xmax = (xmax + 32768) >> 16;
    ymin = (ymin + 32768) >> 16; ymax = (ymax + 32768) >> 16;
    if (xmax < 0 || ymax < 0 || xmin >= W || ymin >= H) return;
    if (ymax > H - 1) ymax = H - 1;
    if (y < ymin || y > ymax) return;
    int idx[2] = {imin, imin};
    const int di[2] = {1, 3};
    long long ex[2] = {-65536, -65536}, edx[2] = {0, 0}, ye[2] = {ymin, ymin}, ys[2] = {ymin, ymin};
    int edges = 4;
    long long yc = ymin;
    for (;;) {
        for (int i = 0; i < 2; ++i) {
            if (yc < ye[i]) continue;
            int i0 = idx[i], i1 = (i0 + di[i]) & 3;
            while (edges-- > 0) {
                const long long ty = (vy[i1] + 32768) >> 16;
                if (ty > yc) {
                    ye[i] = ty; ys[i] = yc; ex[i] = vx[i0];
                    edx[i] = ((vx[i1] - vx[i0]) * 2 + (ty - yc)) / (2 * (ty - yc));
                    idx[i] = i1;
                    break;
                }
                i0 = i1; i1 = (i1 + di[i]) & 3;
            }
        }
        if (edges < 0) return;                  // the fill stops before row yc <= y
        const long long next = ye[0] < ye[1] ? ye[0] : ye[1];
        if (next > y) break;
        yc = next;
    }
    const long long xa = ex[0] + edx[0] * (y - ys[0]), xb = ex[1] + edx[1] * (y - ys[1]);
    const long long lo = xa > xb ? xb : xa, hi = xa > xb ? xa : xb;
    const long long a = (lo + 32768) >> 16, b = (hi + 32768) >> 16;
    if (b >= 0 && a < W) ov_span(row, W, a, b, bgr);
}

__host__ __device__ inline void ov_cap_row(uint8_t* row, int W, int y, int cx, int cy, uint32_t bgr) {
    if (y == cy) ov_span(row, W, (long long)cx - 1, (long long)cx + 1, bgr);
    else if (y == cy - 1 || y == cy + 1) ov_put(row, W, cx, bgr);
}

// Everything segment s draws on row y of an H x W frame whose row y starts at `row`
__host__ __device__ inline void overlay_seg_row(const OverlaySeg& s, uint8_t* row, int H, int W, int y) {
    if (s.quad) {
        for (int k = 0; k < 4; ++k) {
            const int j = (k + 3) & 3;
            ov_outline_row(row, H, W, y, s.vx[j], s.vy[j], s.vx[k], s.vy[k], s.bgr);
        }
        ov_fill_row(row, H, W, y, s.vx, s.vy, s.bgr);
    }
    ov_cap_row(row, W, y, s.q0x, s.q0y, s.bgr);
    ov_cap_row(row, W, y, s.q1x, s.q1y, s.bgr);
}

// grid (ceil(max H / blockDim.x), n frames); thread = one row of one frame
__global__ void __launch_bounds__(128) overlay_draw_kernel(const __grid_constant__ OverlayFrames fr, const OverlaySeg* __restrict__ segs) {
    const int f = blockIdx.y;
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    const int H = fr.H[f], W = fr.W[f];
    if (y >= H) return;
    uint8_t* row = fr.ptr[f] + (size_t)y * W * 3;
    for (int i = fr.seg_begin[f]; i < fr.seg_begin[f + 1]; ++i) {
        if (y < __ldg(&segs[i].y_lo) || y > __ldg(&segs[i].y_hi)) continue;
        const OverlaySeg s = segs[i];
        overlay_seg_row(s, row, H, W, y);
    }
}

// ----------------------------------------------------------------------------- text (DESIGN.md section 8.8)
// A thickness-1 LINE_8 segment of cv2.putText (oracle/text_oracle.py draw_line1): the host rounds its 16.16 end points to
// pixels, clips them against the frame and orders them left end first; OpenCV's 8-connected LineIterator then puts pixel k
// of the major axis ceil((2Bk - A) / 2A) pixels along the minor one (A = major length, B = minor length).
struct OverlayThin {
    int x1, y1, x2, y2;       // clipped pixel end points, x1 <= x2
    int y_lo, y_hi;           // min / max of y1, y2
    uint32_t bgr;
    int pad;
};

constexpr int kOverlayBandRows = 32;      // one warp of rows shares one band's primitive list

__host__ __device__ inline void ov_thin_row(const OverlayThin& t, uint8_t* row, int W, int y) {
    const long long dx = t.x2 - t.x1, dy = t.y2 >= t.y1 ? t.y2 - t.y1 : t.y1 - t.y2;
    const long long k = t.y2 >= t.y1 ? y - t.y1 : t.y1 - y;         // steps from the left end point along y
    if (dy > dx) {                      // y-major: one pixel per row
        if (k < 0 || k > dy) return;
        const long long m = ov_ceil_div(2 * dx * k - dy, 2 * dy);
        ov_put(row, W, t.x1 + (m > 0 ? m : 0), t.bgr);
    } else {                            // x-major: the run of steps whose minor offset is k
        if (k < 0 || k > dy) return;
        long long lo = 0, hi = dx;
        if (dy > 0) {
            lo = ov_floor_div(2 * dx * k - dx, 2 * dy) + 1;
            hi = ov_floor_div(2 * dx * k + dx, 2 * dy);
            lo = lo < 0 ? 0 : lo;
            hi = hi > dx ? dx : hi;
        }
        ov_span(row, W, t.x1 + lo, t.x1 + hi, t.bgr);
    }
}

// grid (ceil(max H / blockDim.x), n frames); thread = one row of one frame.  fr.seg_begin[f] is frame f's first band;
// band b's primitives, in draw order, are items[band_begin[b] .. band_begin[b + 1]): i >= 0 is segs[i] (thickness 2),
// i < 0 is thin[~i] (thickness 1).
__global__ void __launch_bounds__(128) overlay_draw_banded_kernel(const __grid_constant__ OverlayFrames fr, const OverlaySeg* __restrict__ segs,
                                                                  const OverlayThin* __restrict__ thin, const int* __restrict__ band_begin,
                                                                  const int* __restrict__ items) {
    const int f = blockIdx.y;
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    const int H = fr.H[f], W = fr.W[f];
    if (y >= H) return;
    uint8_t* row = fr.ptr[f] + (size_t)y * W * 3;
    const int b = fr.seg_begin[f] + y / kOverlayBandRows;
    for (int j = __ldg(&band_begin[b]), e = __ldg(&band_begin[b + 1]); j < e; ++j) {
        const int i = __ldg(&items[j]);
        if (i >= 0) {
            if (y < __ldg(&segs[i].y_lo) || y > __ldg(&segs[i].y_hi)) continue;
            const OverlaySeg s = segs[i];
            overlay_seg_row(s, row, H, W, y);
        } else {
            const OverlayThin t = thin[~i];
            if (y < t.y_lo || y > t.y_hi) continue;
            ov_thin_row(t, row, W, y);
        }
    }
}

}  // namespace whenet
