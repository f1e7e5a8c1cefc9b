// frames_api.cu - the frame crops (whenet_crop_resize_u8, whenet_crop_boxes_*), head overlay (whenet_draw_heads*), text
// (whenet_put_text*) and YUV -> BGR frame conversion (whenet_yuv_to_bgr_*) of the C ABI, with their debug entries (DESIGN.md
// sections 8.2, 8.4, 8.5, 8.7, 8.8 and 8.14): the host geometry and the launches of kernels_crop.cuh, kernels_overlay.cuh and
// yuv.cuh on the context's stream.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/whenet_b200.h"
#include "api_error.h"
#include "frames_api.h"
#include "kernels_crop.cuh"
#include "kernels_overlay.cuh"

using whenet::Scope;
using whenet::api::check_yuv422_layout;
using whenet::api::check_yuv_layout;
using whenet::api::fail;
namespace F = whenet::frames;

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail(WHENET_ECUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,         \
                        cudaGetErrorString(e__));                                                  \
    } while (0)

namespace whenet {
namespace frames {

// Every buffer grows to exactly what a call needs and is kept for the next call; all are freed by destroy().
struct State {
    uint8_t* d_frame = nullptr; size_t frame_cap = 0;           // host frames, uploaded (bytes)
    int4* d_rects = nullptr; size_t rects_cap = 0;              // crop table
    int* d_frame_of = nullptr; size_t frame_of_cap = 0;
    OverlaySeg* d_segs = nullptr; size_t segs_cap = 0;          // head overlay segment table
    // text and display="full" overlay: thickness-1 segments, band table and banded item list
    OverlayThin* d_thin = nullptr; size_t thin_cap = 0;
    int* d_bands = nullptr; size_t bands_cap = 0;
    int* d_items = nullptr; size_t items_cap = 0;
};

void destroy(State* st) {
    if (!st) return;
    for (void* p : {(void*)st->d_frame, (void*)st->d_rects, (void*)st->d_frame_of, (void*)st->d_segs, (void*)st->d_thin,
                    (void*)st->d_bands, (void*)st->d_items})
        if (p) cudaFree(p);
    delete st;
}

}  // namespace frames
}  // namespace whenet

namespace {

// The context's frame state, created on first use, with its device selected
int frame_state(const F::Target& t, F::State*& st) {
    CK(cudaSetDevice(t.device));
    if (!*t.state) *t.state = new F::State();
    st = *t.state;
    return 0;
}

// *buf grown to hold n elements: reallocated to exactly n when it holds fewer (its contents are not kept), never shrunk
template <typename T>
int grow(T** buf, size_t* cap, size_t n) {
    if (*cap >= n) return 0;
    if (*buf) cudaFree(*buf);
    *buf = nullptr; *cap = 0;
    CK(cudaMalloc(buf, n * sizeof(T)));
    *cap = n;
    return 0;
}

// n host elements copied into *buf on the context's stream, *buf grown first
template <typename T>
int upload(const F::Target& t, T** buf, size_t* cap, const T* src, size_t n) {
    if (n == 0) return 0;
    if (int rc = grow(buf, cap, n)) return rc;
    CK(cudaMemcpyAsync(*buf, src, n * sizeof(T), cudaMemcpyHostToDevice, t.stream));
    return 0;
}

// ----------------------------------------------------------------------------- crop front-end
// Python's builtin max(0, t) / min(lim, u) on the numpy float32 scalars of demo_video.py:15-18: the second argument wins
// only when it compares greater / smaller, so a NaN gives the bound (np.maximum / np.minimum would propagate it).
inline float py_max0(float t) { return t > 0.f ? t : 0.f; }
inline float py_min(float lim, float u) { return u < lim ? u : lim; }

// int(v) (truncation toward zero) when it lies in [lo, hi]; false for NaN, +-inf and anything outside - decided in double
// before the conversion, so no out-of-range float is ever cast to int.
inline bool trunc_within(float v, int lo, int hi, int* out) {
    const double t = std::trunc((double)v);
    if (!(t >= lo && t <= hi)) return false;
    *out = (int)t;
    return true;
}

// The margin arithmetic of reference demo_video.py:13-21 (whenet_b200/crops.py enlarge_box) bit for bit: float32 throughout
// (numpy 2 scalar rules), correctly rounded divisions by 10 and 5, and the far side grown from the ALREADY updated near side
// as the reference does.  Returns whether the slice is non-empty and inside the frame (0 <= y0 < y1 <= H, 0 <= x0 < x1 <= W,
// the predicate whenet_crop_resize_u8 enforces); r = (y0, y1, x0, x1) then, zeros otherwise.
bool enlarge_box(const float* b, int H, int W, int32_t r[4]) {
    float y_min = b[0], x_min = b[1], y_max = b[2], x_max = b[3];
    y_min = py_max0(y_min - std::fabs(y_min - y_max) / 10.f);
    y_max = py_min((float)H, y_max + std::fabs(y_min - y_max) / 10.f);
    x_min = py_max0(x_min - std::fabs(x_min - x_max) / 5.f);
    x_max = py_min((float)W, x_max + std::fabs(x_min - x_max) / 5.f);
    int y0, y1, x0, x1;
    const bool ok = trunc_within(y_min, 0, H, &y0) && trunc_within(y_max, 0, H, &y1) && trunc_within(x_min, 0, W, &x0) &&
                    trunc_within(x_max, 0, W, &x1) && y0 < y1 && x0 < x1;
    r[0] = ok ? y0 : 0; r[1] = ok ? y1 : 0; r[2] = ok ? x0 : 0; r[3] = ok ? x1 : 0;
    return ok;
}

static_assert(whenet::kYuvNV12 == WHENET_YUV_NV12 && whenet::kYuvI420 == WHENET_YUV_I420, "layout codes of yuv.cuh and the ABI");
static_assert(whenet::kYuvYUYV == WHENET_YUV_YUYV && whenet::kYuvUYVY == WHENET_YUV_UYVY, "layout codes of yuv.cuh and the ABI");

// bytes of an H x W frame: packed 8-bit BGR / RGB (yuv_layout 0), YUV 4:2:0 (H and W even) or packed YUV 4:2:2 (W even)
size_t frame_bytes(int H, int W, int yuv_layout) {
    if (whenet::yuv422(yuv_layout)) return (size_t)H * W * 2;
    return yuv_layout ? (size_t)H * W / 2 * 3 : (size_t)H * W * 3;
}

// The crop table -> crop_resize_kernel<Frames> (yuv_layout 0) or crop_resize_yuv_kernel<Frames, yuv_layout>, one launch per 65535
// crops (the grid's y limit).  rects: m x (y0, y1, x0, x1) host int32, an empty one marks a zero crop; frame_of: m host frame
// indices or NULL (all frame 0, OneSizeFrames only).
template <class Frames>
int launch_crop_kernel(whenet_ctx* c, const F::Target& t, F::State* st, const Frames& src, const int32_t* rects, const int32_t* frame_of,
                       int m, int swap_rb, int yuv_layout, uint8_t* crops_out) {
    if (int rc = upload(t, &st->d_rects, &st->rects_cap, reinterpret_cast<const int4*>(rects), m)) return rc;
    if (frame_of)
        if (int rc = upload(t, &st->d_frame_of, &st->frame_of_cap, frame_of, m)) return rc;
    Scope sc(c, t.stream, "crop_resize", (double)m * 224 * 224 * 3 * 2, 0.0);
    for (int m0 = 0; m0 < m; m0 += 65535) {
        const int mb = std::min(65535, m - m0);
        const dim3 grid((224 * 224 + 255) / 256, mb);
        const int* fo = frame_of ? st->d_frame_of + m0 : nullptr;
        uint8_t* out = crops_out + (size_t)m0 * 224 * 224 * 3;
        if (yuv_layout == whenet::kYuvNV12)
            whenet::crop_resize_yuv_kernel<Frames, whenet::kYuvNV12><<<grid, 256, 0, t.stream>>>(src, st->d_rects + m0, fo, out);
        else if (yuv_layout == whenet::kYuvI420)
            whenet::crop_resize_yuv_kernel<Frames, whenet::kYuvI420><<<grid, 256, 0, t.stream>>>(src, st->d_rects + m0, fo, out);
        else if (yuv_layout == whenet::kYuvYUYV)
            whenet::crop_resize_yuv_kernel<Frames, whenet::kYuvYUYV><<<grid, 256, 0, t.stream>>>(src, st->d_rects + m0, fo, out);
        else if (yuv_layout == whenet::kYuvUYVY)
            whenet::crop_resize_yuv_kernel<Frames, whenet::kYuvUYVY><<<grid, 256, 0, t.stream>>>(src, st->d_rects + m0, fo, out);
        else
            whenet::crop_resize_kernel<Frames><<<grid, 256, 0, t.stream>>>(src, st->d_rects + m0, fo, out, swap_rb);
        CK(cudaGetLastError());
    }
    return 0;
}

// n frames of one size (uploaded into the context's staging buffer when on the host) -> launch_crop_kernel
int launch_crops(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, const int32_t* rects,
                 const int32_t* frame_of, int m, int swap_rb, int yuv_layout, uint8_t* crops_out) {
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    const uint8_t* d_frames = frames;
    if (!frames_are_device) {
        if (int rc = upload(t, &st->d_frame, &st->frame_cap, frames, n * frame_bytes(H, W, yuv_layout))) return rc;
        d_frames = st->d_frame;
    }
    return launch_crop_kernel(c, t, st, whenet::OneSizeFrames{d_frames, H, W}, rects, frame_of, m, swap_rb, yuv_layout, crops_out);
}

// n frames of their own sizes: host frames are uploaded into the staging buffer at 256-byte aligned offsets, device frames are
// read where they are
int launch_crops_ragged(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const int32_t* rects,
                        const int32_t* frame_of, int m, int swap_rb, int yuv_layout, uint8_t* crops_out) {
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    whenet::PerFrameSources src{};
    std::vector<size_t> off(n);
    size_t total = 0;
    for (int i = 0; i < n; ++i) {
        off[i] = total;
        total += (frame_bytes(hw[2 * i], hw[2 * i + 1], yuv_layout) + 255) & ~(size_t)255;
    }
    if (!frames_are_device) {
        if (int rc = grow(&st->d_frame, &st->frame_cap, total)) return rc;
        for (int i = 0; i < n; ++i)
            CK(cudaMemcpyAsync(st->d_frame + off[i], frames[i], frame_bytes(hw[2 * i], hw[2 * i + 1], yuv_layout), cudaMemcpyHostToDevice, t.stream));
    }
    for (int i = 0; i < n; ++i) src.f[i] = {frames_are_device ? frames[i] : st->d_frame + off[i], hw[2 * i + 1], hw[2 * i]};
    return launch_crop_kernel(c, t, st, src, rects, frame_of, m, swap_rb, yuv_layout, crops_out);
}

// whenet_crop_boxes_u8 (yuv_layout 0), whenet_crop_boxes_yuv_u8 and whenet_crop_boxes_yuv422_u8
int crop_boxes(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, const float* boxes, const int32_t* frame_of,
               int m, int swap_rb, int yuv_layout, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    // the context is checked last so that every other argument can be validated without a GPU
    if (!frames || !boxes || !frame_of || !crops_out) return fail(WHENET_EINVAL, "null frames, boxes, frame_of or crops_out");
    if (n < 1 || n > 64) return fail(WHENET_EINVAL, "n=%d frames outside [1, 64]", n);
    if (H < 1 || W < 1) return fail(WHENET_EINVAL, "bad frame size %dx%d", H, W);
    if (whenet::yuv422(yuv_layout) && (H > 16384 || W < 2 || W > 16384 || W % 2))
        return fail(WHENET_EINVAL, "frame size %dx%d: a 4:2:2 frame has an even width in [2, 16384] and a height of at most 16384", H, W);
    if (yuv_layout && !whenet::yuv422(yuv_layout) && (H > 16384 || W > 16384 || H % 2 || W % 2))
        return fail(WHENET_EINVAL, "frame size %dx%d: a 4:2:0 frame has even sides of at most 16384", H, W);
    if (m < 1) return fail(WHENET_EINVAL, "m=%d boxes", m);
    for (int i = 0; i < m; ++i)
        if (frame_of[i] < 0 || frame_of[i] >= n) return fail(WHENET_EINVAL, "box %d: frame_of=%d outside [0, %d)", i, frame_of[i], n);
    if (!c) return fail(WHENET_EINVAL, "null context");
    std::vector<int32_t> rects((size_t)m * 4);
    for (int i = 0; i < m; ++i) {
        const bool ok = enlarge_box(boxes + 4 * i, H, W, &rects[(size_t)4 * i]);
        if (valid_out) valid_out[i] = ok;
    }
    if (rects_out) memcpy(rects_out, rects.data(), rects.size() * sizeof(int32_t));
    return launch_crops(c, frames, n, H, W, frames_are_device, rects.data(), frame_of, m, swap_rb, yuv_layout, crops_out);
}

// whenet_crop_boxes_ragged_u8 (yuv_layout 0), whenet_crop_boxes_ragged_yuv_u8 and whenet_crop_boxes_ragged_yuv422_u8
int crop_boxes_ragged(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const float* boxes,
                      const int32_t* frame_of, int m, int swap_rb, int yuv_layout, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    // the context is checked last so that every other argument can be validated without a GPU
    if (!frames || !hw || !boxes || !frame_of || !crops_out) return fail(WHENET_EINVAL, "null frames, hw, boxes, frame_of or crops_out");
    if (n < 1 || n > whenet::kMaxCropFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxCropFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i]) return fail(WHENET_EINVAL, "frame %d is NULL", i);
        if (hw[2 * i] < 1 || hw[2 * i + 1] < 1 || hw[2 * i] > 16384 || hw[2 * i + 1] > 16384)
            return fail(WHENET_EINVAL, "frame %d: bad frame size %dx%d", i, hw[2 * i + 1], hw[2 * i]);
        if (whenet::yuv422(yuv_layout) && hw[2 * i + 1] % 2)
            return fail(WHENET_EINVAL, "frame %d: frame size %dx%d: a 4:2:2 frame has an even width", i, hw[2 * i + 1], hw[2 * i]);
        if (yuv_layout && !whenet::yuv422(yuv_layout) && (hw[2 * i] % 2 || hw[2 * i + 1] % 2))
            return fail(WHENET_EINVAL, "frame %d: frame size %dx%d: a 4:2:0 frame has even sides", i, hw[2 * i + 1], hw[2 * i]);
    }
    if (m < 1) return fail(WHENET_EINVAL, "m=%d boxes", m);
    for (int i = 0; i < m; ++i)
        if (frame_of[i] < 0 || frame_of[i] >= n) return fail(WHENET_EINVAL, "box %d: frame_of=%d outside [0, %d)", i, frame_of[i], n);
    if (!c) return fail(WHENET_EINVAL, "null context");
    std::vector<int32_t> rects((size_t)m * 4);
    for (int i = 0; i < m; ++i) {
        const bool ok = enlarge_box(boxes + 4 * i, hw[2 * frame_of[i]], hw[2 * frame_of[i] + 1], &rects[(size_t)4 * i]);
        if (valid_out) valid_out[i] = ok;
    }
    if (rects_out) memcpy(rects_out, rects.data(), rects.size() * sizeof(int32_t));
    return launch_crops_ragged(c, frames, hw, n, frames_are_device, rects.data(), frame_of, m, swap_rb, yuv_layout, crops_out);
}

// ----------------------------------------------------------------------------- YUV -> BGR frames (DESIGN.md section 8.14)
// the layout argument of whenet_yuv_to_bgr_*
int check_convert_layout(int layout) {
    if (layout < WHENET_YUV_NV12 || layout > WHENET_YUV_UYVY)
        return fail(WHENET_EINVAL, "layout=%d: WHENET_YUV_NV12 (%d), WHENET_YUV_I420 (%d), WHENET_YUV_YUYV (%d) or WHENET_YUV_UYVY (%d)", layout,
                    WHENET_YUV_NV12, WHENET_YUV_I420, WHENET_YUV_YUYV, WHENET_YUV_UYVY);
    return 0;
}

// an H x W frame of the layout: sides in [1, 16384], W even, H even for 4:2:0.  i: the frame's index in the message, or -1
int check_convert_size(int i, int H, int W, int layout) {
    char pre[32] = "";
    if (i >= 0) snprintf(pre, sizeof(pre), "frame %d: ", i);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "%sframe size %dx%d: sides must be in [1, 16384]", pre, W, H);
    if (whenet::yuv422(layout) && W % 2) return fail(WHENET_EINVAL, "%sframe size %dx%d: a 4:2:2 frame has an even width", pre, W, H);
    if (!whenet::yuv422(layout) && (H % 2 || W % 2)) return fail(WHENET_EINVAL, "%sframe size %dx%d: a 4:2:0 frame has even sides", pre, W, H);
    return 0;
}

// pixel pairs (4:2:2) or 2 x 2 blocks (4:2:0) of an H x W frame: the threads of yuv_to_bgr_kernel
long long convert_units(int H, int W, int layout) { return (long long)(whenet::yuv422(layout) ? H : H / 2) * (W / 2); }

// The frame table (src: device frames) -> one yuv_to_bgr_kernel launch on the context's stream
int launch_convert(whenet_ctx* c, const F::Target& t, const whenet::YuvConvertFrames& tab, int n, int layout) {
    long long units = 0;
    double bytes = 0.0;
    for (int i = 0; i < n; ++i) {
        units = std::max(units, convert_units(tab.f[i].H, tab.f[i].W, layout));
        bytes += (double)frame_bytes(tab.f[i].H, tab.f[i].W, layout) + 3.0 * tab.f[i].H * tab.f[i].W;
    }
    Scope sc(c, t.stream, "yuv_to_bgr", bytes, 0.0);
    const dim3 grid((unsigned)((units + 255) / 256), n);
    switch (layout) {
        case whenet::kYuvNV12: whenet::yuv_to_bgr_kernel<whenet::kYuvNV12><<<grid, 256, 0, t.stream>>>(tab); break;
        case whenet::kYuvI420: whenet::yuv_to_bgr_kernel<whenet::kYuvI420><<<grid, 256, 0, t.stream>>>(tab); break;
        case whenet::kYuvYUYV: whenet::yuv_to_bgr_kernel<whenet::kYuvYUYV><<<grid, 256, 0, t.stream>>>(tab); break;
        case whenet::kYuvUYVY: whenet::yuv_to_bgr_kernel<whenet::kYuvUYVY><<<grid, 256, 0, t.stream>>>(tab); break;
        default: return fail(WHENET_EINVAL, "layout=%d", layout);
    }
    CK(cudaGetLastError());
    return 0;
}

// n frames of one size; host frames are uploaded into the staging buffer in one copy
int yuv_to_bgr(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, int layout, uint8_t* out) {
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    const size_t fb = frame_bytes(H, W, layout);
    if (!frames_are_device) {
        if (int rc = upload(t, &st->d_frame, &st->frame_cap, frames, n * fb)) return rc;
        frames = st->d_frame;
    }
    whenet::YuvConvertFrames tab{};
    for (int i = 0; i < n; ++i) tab.f[i] = {frames + i * fb, out + (size_t)i * H * W * 3, H, W};
    return launch_convert(c, t, tab, n, layout);
}

// n frames of their own sizes; host frames are uploaded into the staging buffer at 256-byte aligned offsets
int yuv_to_bgr_ragged(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int layout,
                      uint8_t* const* out) {
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    std::vector<size_t> off(n);
    size_t total = 0;
    for (int i = 0; i < n; ++i) {
        off[i] = total;
        total += (frame_bytes(hw[2 * i], hw[2 * i + 1], layout) + 255) & ~(size_t)255;
    }
    if (!frames_are_device) {
        if (int rc = grow(&st->d_frame, &st->frame_cap, total)) return rc;
        for (int i = 0; i < n; ++i)
            CK(cudaMemcpyAsync(st->d_frame + off[i], frames[i], frame_bytes(hw[2 * i], hw[2 * i + 1], layout), cudaMemcpyHostToDevice, t.stream));
    }
    whenet::YuvConvertFrames tab{};
    for (int i = 0; i < n; ++i) tab.f[i] = {frames_are_device ? frames[i] : st->d_frame + off[i], out[i], hw[2 * i], hw[2 * i + 1]};
    return launch_convert(c, t, tab, n, layout);
}

// ----------------------------------------------------------------------------- head overlay (DESIGN.md section 8.7)
// One head -> the 7 segments reference demo_video.py:26,29 draws (utils.py:40-42): the rectangle as its 4 edges (cv2.rectangle
// with thickness 2 gives the pixels of these 4 cv2.line calls), then the red, green and blue axes.  Every scalar keeps the type
// numpy 2 gives it in the reference: a bound clamped by max(0, v) / min(W, v) is a Python int, so tdx and size are a Python
// float and int (double arithmetic) when BOTH x bounds clamped, float32 otherwise; likewise tdy for y.  An np.float32 meeting
// a Python float rounds that float to float32 first.  Returns false where the reference raises (empty or out-of-frame slice,
// a non-finite float32 radian): such a head is not drawn.  Compiled without FMA contraction (build.py), as CPython evaluates.
constexpr int kSegsPerHead = 7;

struct PyNum {            // a float32 or a double, as the reference's value has it
    double v; bool dbl;
};
inline PyNum py_add(PyNum a, PyNum b) {
    return (a.dbl && b.dbl) ? PyNum{a.v + b.v, true} : PyNum{(double)((float)a.v + (float)b.v), false};
}
inline PyNum py_mul(PyNum size, double e) {      // size * (double expression)
    return size.dbl ? PyNum{size.v * e, true} : PyNum{(double)((float)size.v * (float)e), false};
}

bool head_segments(const float* box, const float* ang, int H, int W, int32_t seg[kSegsPerHead][4]) {
    int32_t r[4];
    if (!enlarge_box(box, H, W, r)) return false;
    float y_min = box[0], x_min = box[1], y_max = box[2], x_max = box[3];
    const float vy0 = y_min - std::fabs(y_min - y_max) / 10.f;
    const bool cy0 = !(vy0 > 0.f);
    y_min = cy0 ? 0.f : vy0;
    const float vy1 = y_max + std::fabs(y_min - y_max) / 10.f;
    const bool cy1 = !(vy1 < (float)H);
    y_max = cy1 ? (float)H : vy1;
    const float vx0 = x_min - std::fabs(x_min - x_max) / 5.f;
    const bool cx0 = !(vx0 > 0.f);
    x_min = cx0 ? 0.f : vx0;
    const float vx1 = x_max + std::fabs(x_min - x_max) / 5.f;
    const bool cx1 = !(vx1 < (float)W);
    x_max = cx1 ? (float)W : vx1;
    const float pi = (float)M_PI;
    const float pitch = ang[1] * pi / 180.f, yaw = -(ang[0] * pi / 180.f), roll = ang[2] * pi / 180.f;
    if (!std::isfinite(pitch) || !std::isfinite(yaw) || !std::isfinite(roll)) return false;
    const bool xd = cx0 && cx1, yd = cy0 && cy1;
    const PyNum tdx = xd ? PyNum{W / 2.0, true} : PyNum{(double)((x_min + x_max) / 2.f), false};
    const PyNum tdy = yd ? PyNum{H / 2.0, true} : PyNum{(double)((y_min + y_max) / 2.f), false};
    const PyNum size = xd ? PyNum{(double)(W / 2), true} : PyNum{(double)std::floor(std::fabs(x_max - x_min) / 2.f), false};
    const double cp = std::cos((double)pitch), sp = std::sin((double)pitch), cyw = std::cos((double)yaw), syw = std::sin((double)yaw);
    const double cr = std::cos((double)roll), sr = std::sin((double)roll);
    const PyNum x1 = py_add(py_mul(size, cyw * cr), tdx);
    const PyNum y1 = py_add(py_mul(size, cp * sr + cr * sp * syw), tdy);
    const PyNum x2 = py_add(py_mul(size, -cyw * sr), tdx);
    const PyNum y2 = py_add(py_mul(size, cp * cr - sp * syw * sr), tdy);
    const PyNum x3 = py_add(py_mul(size, syw), tdx);
    const PyNum y3 = py_add(py_mul(size, -cyw * sp), tdy);
    const int X0 = r[2], Y0 = r[0], X1 = r[3], Y1 = r[1];
    const int cx = (int)tdx.v, cyc = (int)tdy.v;
    const int32_t s[kSegsPerHead][4] = {{X0, Y0, X1, Y0}, {X1, Y0, X1, Y1}, {X1, Y1, X0, Y1}, {X0, Y1, X0, Y0},
                                        {cx, cyc, (int)x1.v, (int)y1.v}, {cx, cyc, (int)x2.v, (int)y2.v}, {cx, cyc, (int)x3.v, (int)y3.v}};
    memcpy(seg, s, sizeof(s));
    return true;
}

constexpr uint32_t kSegColor[kSegsPerHead] = {0, 0, 0, 0, 0xff0000u, 0x00ff00u, 0x0000ffu};   // b | g << 8 | r << 16

// A thickness-2 segment on an H x W frame -> its device record; false when it draws nothing (oracle/draw_oracle.py)
bool overlay_seg(const int32_t p[4], uint32_t bgr, int H, int W, whenet::OverlaySeg* s) {
    long long x0 = p[0] + 2LL, y0 = p[1] + 2LL, x1 = p[2] + 2LL, y1 = p[3] + 2LL;
    if (!whenet::ov_clip(W + 4LL, H + 4LL, x0, y0, x1, y1)) return false;
    x0 -= 2; y0 -= 2; x1 -= 2; y1 -= 2;
    *s = whenet::OverlaySeg{};
    s->q0x = (int)x0; s->q0y = (int)y0; s->q1x = (int)x1; s->q1y = (int)y1;
    s->bgr = bgr;
    long long lo = std::min(y0, y1) - 1, hi = std::max(y0, y1) + 1;
    const double dx = (double)(x0 - x1), dy = (double)(y1 - y0);
    double rr = dx * dx + dy * dy;
    if (std::fabs(rr) > 2.220446049250313e-16) {
        rr = 65536.0 / std::sqrt(rr);
        const long long dpx = std::llrint(dy * rr), dpy = std::llrint(dx * rr);     // round half to even, as cvRound
        const long long X0 = x0 * 65536, Y0 = y0 * 65536, X1 = x1 * 65536, Y1 = y1 * 65536;
        const long long vx[4] = {X0 + dpx, X0 - dpx, X1 - dpx, X1 + dpx}, vy[4] = {Y0 + dpy, Y0 - dpy, Y1 - dpy, Y1 + dpy};
        s->quad = 1;
        for (int k = 0; k < 4; ++k) {
            s->vx[k] = vx[k]; s->vy[k] = vy[k];
            lo = std::min(lo, (vy[k] + 32768) >> 16);
            hi = std::max(hi, (vy[k] + 32768) >> 16);
        }
    }
    lo = std::max(lo, 0LL);
    hi = std::min(hi, (long long)H - 1);
    if (lo > hi) return false;
    s->y_lo = (int)lo; s->y_hi = (int)hi;
    return true;
}

// heads -> the segment table grouped by frame, in result order within a frame, and the launch
int draw_heads(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes, const float* angles,
               const int32_t* frame_of, int m, int32_t* drawn_out) {
    whenet::OverlayFrames fr{};
    std::vector<std::vector<whenet::OverlaySeg>> per(n);
    int32_t seg[kSegsPerHead][4];
    for (int i = 0; i < m; ++i) {
        const int f = frame_of[i], H = hw[2 * f], W = hw[2 * f + 1];
        const bool ok = head_segments(boxes + 4 * i, angles + 3 * i, H, W, seg);
        if (drawn_out) drawn_out[i] = ok;
        if (!ok) continue;
        for (int k = 0; k < kSegsPerHead; ++k) {
            whenet::OverlaySeg s;
            if (overlay_seg(seg[k], kSegColor[k], H, W, &s)) per[f].push_back(s);
        }
    }
    std::vector<whenet::OverlaySeg> segs;
    int maxH = 0;
    for (int f = 0; f < n; ++f) {
        fr.seg_begin[f] = (int)segs.size();
        segs.insert(segs.end(), per[f].begin(), per[f].end());
        fr.ptr[f] = frames[f]; fr.H[f] = hw[2 * f]; fr.W[f] = hw[2 * f + 1];
        maxH = std::max(maxH, fr.H[f]);
    }
    fr.seg_begin[n] = (int)segs.size();
    if (segs.empty()) return 0;
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    if (int rc = upload(t, &st->d_segs, &st->segs_cap, segs.data(), segs.size())) return rc;
    Scope sc(c, t.stream, "draw_heads", 0.0, 0.0);
    whenet::overlay_draw_kernel<<<dim3((maxH + 127) / 128, n), 128, 0, t.stream>>>(fr, st->d_segs);
    CK(cudaGetLastError());
    return 0;
}

int draw_heads_checked(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes, const float* angles,
                       const int32_t* frame_of, int m, int32_t* drawn_out) {
    // the context is checked last so that every other argument can be validated without a GPU
    if (n < 1 || n > whenet::kMaxCropFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxCropFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i]) return fail(WHENET_EINVAL, "frame %d is NULL", i);
        if (hw[2 * i] < 1 || hw[2 * i + 1] < 1 || hw[2 * i] > 16384 || hw[2 * i + 1] > 16384)
            return fail(WHENET_EINVAL, "frame %d: bad frame size %dx%d", i, hw[2 * i + 1], hw[2 * i]);
    }
    if (m < 0) return fail(WHENET_EINVAL, "m=%d heads", m);
    if (m == 0) return 0;
    if (!boxes || !angles || !frame_of) return fail(WHENET_EINVAL, "null boxes, angles or frame_of");
    for (int i = 0; i < m; ++i)
        if (frame_of[i] < 0 || frame_of[i] >= n) return fail(WHENET_EINVAL, "head %d: frame_of=%d outside [0, %d)", i, frame_of[i], n);
    if (!c) return fail(WHENET_EINVAL, "null context");
    return draw_heads(c, frames, hw, n, boxes, angles, frame_of, m, drawn_out);
}

// ----------------------------------------------------------------------------- text (DESIGN.md section 8.8)
// cv2.putText(img, text, org, FONT_HERSHEY_SIMPLEX, scale, color, 1) as thickness-1 segments (oracle/text_oracle.py), and the
// labels of reference demo_video.py:31-34 (display="full").
#include "hershey_simplex.inc"

constexpr int kTextMaxLen = 4096;
constexpr int kTextMaxItems = 1 << 20;
constexpr long long kTextMaxChars = 1 << 22;             // characters per put_text call (at most 40 segments each)
constexpr int kLabelMaxHeads = 1 << 16;                  // heads per display="full" call
constexpr size_t kOverlayMaxItems = 0x7fffffff;          // primitives and banded entries are indexed with int
constexpr int kTextMaxOrg = 1 << 24;
constexpr double kTextMaxScale = 256.0;
constexpr float kLabelScale = 0.4f;
constexpr uint32_t kLabelColor = 100u | 255u << 8;          // (100, 255, 0) BGR

// "{}".format(np.round(np.float32(a))) under numpy 2: round half to even in float32; an empty format spec then formats the
// value as a Python float, i.e. the shortest round-trip digits of the double, positional with a trailing ".0" below 1e16
// and scientific ("1e+16", "3.4028234663852886e+38") from there.
std::string label_number(float a) {
    const float v = std::nearbyint(a);
    if (std::isnan(v)) return "nan";
    if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
    char buf[64];
    const auto r = std::to_chars(buf, buf + sizeof(buf), (double)v, std::chars_format::scientific);
    const std::string s(buf, r.ptr);                        // [-]d[.ddd]e(+|-)xx, shortest digits
    const size_t e = s.find('e');
    const bool neg = s[0] == '-';
    std::string digits;
    for (size_t i = neg; i < e; ++i)
        if (s[i] != '.') digits += s[i];
    const int exp10 = std::atoi(s.c_str() + e + 1);
    std::string out = neg ? "-" : "";
    if (v == 0.f || std::fabs((double)v) < 1e16) {          // v is an integer, so exp10 >= digits.size() - 1
        out += digits + std::string(exp10 + 1 - (int)digits.size(), '0') + ".0";
    } else {
        out += digits.substr(0, 1);
        if (digits.size() > 1) out += "." + digits.substr(1);
        char ex[16];
        snprintf(ex, sizeof(ex), "e+%02d", exp10);
        out += ex;
    }
    return out;
}

// The 16.16 segments putText draws for `text` at `org`, in draw order (x1, y1, x2, y2)
void text_segments16(const char* text, int ox, int oy, double scale, std::vector<long long>& out) {
    const long long hscale = std::llrint(scale * 65536.0), vscale = hscale;     // cvRound
    long long pen_x = (long long)ox * 65536, pen_y = (long long)oy * 65536 + kHersheyBaseLine * vscale;
    for (const char* p = text; *p; ++p) {
        const char* g = kHersheySimplex[*p - 32];
        const long long advance = (g[1] - 'R') * hscale;
        pen_x -= (g[0] - 'R') * hscale;
        long long px = 0, py = 0;
        int npts = 0;
        for (const char* q = g + 2;; ) {
            if (*q == ' ' || !*q) {
                if (!*q) break;
                ++q;
                npts = 0;
            } else {
                const long long x = (q[0] - 'R') * hscale + pen_x, y = (q[1] - 'R') * vscale + pen_y;
                if (npts++ > 0) out.insert(out.end(), {px, py, x, y});
                px = x; py = y;
                q += 2;
            }
        }
        pen_x += advance;
    }
}

// One 16.16 segment -> its thickness-1 record on an H x W frame; false when it misses the frame
bool thin_seg(const long long* s, uint32_t bgr, int H, int W, whenet::OverlayThin* t) {
    long long x1 = (s[0] + 32768) >> 16, y1 = (s[1] + 32768) >> 16, x2 = (s[2] + 32768) >> 16, y2 = (s[3] + 32768) >> 16;
    if (!whenet::ov_clip(W, H, x1, y1, x2, y2)) return false;
    if (x2 < x1) { std::swap(x1, x2); std::swap(y1, y2); }
    *t = whenet::OverlayThin{(int)x1, (int)y1, (int)x2, (int)y2, (int)std::min(y1, y2), (int)std::max(y1, y2), bgr, 0};
    return true;
}

// The primitives of every frame in draw order, banded by kOverlayBandRows rows, and the launch
struct OverlayList {
    std::vector<whenet::OverlaySeg> segs;
    std::vector<whenet::OverlayThin> thin;
    std::vector<std::vector<std::array<int, 3>>> per;      // frame -> (item, y_lo, y_hi)
    std::vector<long long> s16;                             // one text's 16.16 segments, reused
    bool overflow = false;                                  // more primitives than an int indexes
    explicit OverlayList(int n) : per(n) {}
    void add_text(int f, const char* text, int ox, int oy, double scale, uint32_t bgr, int H, int W) {
        s16.clear();
        text_segments16(text, ox, oy, scale, s16);
        for (size_t k = 0; k < s16.size(); k += 4) {
            whenet::OverlayThin t;
            if (!thin_seg(&s16[k], bgr, H, W, &t)) continue;
            if (thin.size() >= kOverlayMaxItems) { overflow = true; return; }
            per[f].push_back({~(int)thin.size(), t.y_lo, t.y_hi});
            thin.push_back(t);
        }
    }
};

int draw_overlay_list(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const OverlayList& L) {
    whenet::OverlayFrames fr{};
    std::vector<int> band_begin(1, 0), items;
    int maxH = 0;
    size_t total = 0;                                       // banded entries, counted before anything is indexed with int
    for (int f = 0; f < n; ++f)
        for (const auto& p : L.per[f]) total += (size_t)(p[2] / whenet::kOverlayBandRows - p[1] / whenet::kOverlayBandRows + 1);
    if (L.overflow || L.segs.size() >= kOverlayMaxItems || total >= kOverlayMaxItems)
        return fail(WHENET_EINVAL, "too many segments in one call (%zu banded entries, limit %zu)", total, kOverlayMaxItems);
    for (int f = 0; f < n; ++f) {
        const int H = hw[2 * f], nb = (H + whenet::kOverlayBandRows - 1) / whenet::kOverlayBandRows;
        fr.ptr[f] = frames[f]; fr.H[f] = H; fr.W[f] = hw[2 * f + 1];
        fr.seg_begin[f] = (int)band_begin.size() - 1;
        maxH = std::max(maxH, H);
        std::vector<int> cnt(nb + 1, 0);                      // counting sort by band, stable in draw order
        for (const auto& p : L.per[f])
            for (int b = p[1] / whenet::kOverlayBandRows; b <= p[2] / whenet::kOverlayBandRows; ++b) ++cnt[b + 1];
        for (int b = 0; b < nb; ++b) cnt[b + 1] += cnt[b];
        const int base = (int)items.size();
        items.resize(base + cnt[nb]);
        std::vector<int> pos(cnt.begin(), cnt.end() - 1);
        for (const auto& p : L.per[f])
            for (int b = p[1] / whenet::kOverlayBandRows; b <= p[2] / whenet::kOverlayBandRows; ++b) items[base + pos[b]++] = p[0];
        for (int b = 0; b < nb; ++b) band_begin.push_back(base + cnt[b + 1]);
    }
    fr.seg_begin[n] = (int)band_begin.size() - 1;
    if (items.empty()) return 0;
    const F::Target t = F::target(c);
    F::State* st;
    if (int rc = frame_state(t, st)) return rc;
    if (int rc = upload(t, &st->d_segs, &st->segs_cap, L.segs.data(), L.segs.size())) return rc;
    if (int rc = upload(t, &st->d_thin, &st->thin_cap, L.thin.data(), L.thin.size())) return rc;
    if (int rc = upload(t, &st->d_bands, &st->bands_cap, band_begin.data(), band_begin.size())) return rc;
    if (int rc = upload(t, &st->d_items, &st->items_cap, items.data(), items.size())) return rc;
    Scope sc(c, t.stream, "draw_overlay", 0.0, 0.0);
    whenet::overlay_draw_banded_kernel<<<dim3((maxH + 127) / 128, n), 128, 0, t.stream>>>(fr, st->d_segs, st->d_thin, st->d_bands, st->d_items);
    CK(cudaGetLastError());
    return 0;
}

// display="full": each drawn head's 7 segments, then its yaw, pitch and roll labels at (int(x_min), int(y_min) - 0 / 15 / 30)
int draw_heads_full(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes, const float* angles,
                    const int32_t* frame_of, int m, int32_t* drawn_out) {
    OverlayList L(n);
    int32_t seg[kSegsPerHead][4];
    static const char* const kLabel[3] = {"yaw: ", "pitch: ", "roll: "};
    for (int i = 0; i < m; ++i) {
        const int f = frame_of[i], H = hw[2 * f], W = hw[2 * f + 1];
        const bool ok = head_segments(boxes + 4 * i, angles + 3 * i, H, W, seg);
        if (drawn_out) drawn_out[i] = ok;
        if (!ok) continue;
        for (int k = 0; k < kSegsPerHead; ++k) {
            whenet::OverlaySeg s;
            if (!overlay_seg(seg[k], kSegColor[k], H, W, &s)) continue;
            L.per[f].push_back({(int)L.segs.size(), s.y_lo, s.y_hi});
            L.segs.push_back(s);
        }
        const int ox = seg[0][0], oy = seg[0][1];             // the rectangle's (int(x_min), int(y_min))
        for (int k = 0; k < 3; ++k)
            L.add_text(f, (kLabel[k] + label_number(angles[3 * i + k])).c_str(), ox, oy - 15 * k, kLabelScale, kLabelColor, H, W);
    }
    return draw_overlay_list(c, frames, hw, n, L);
}

int check_frames(uint8_t* const* frames, const int32_t* hw, int n) {
    if (n < 1 || n > whenet::kMaxCropFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxCropFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i]) return fail(WHENET_EINVAL, "frame %d is NULL", i);
        if (hw[2 * i] < 1 || hw[2 * i + 1] < 1 || hw[2 * i] > 16384 || hw[2 * i + 1] > 16384)
            return fail(WHENET_EINVAL, "frame %d: bad frame size %dx%d", i, hw[2 * i + 1], hw[2 * i]);
    }
    return 0;
}

int check_text(const char* text, int ox, int oy, double scale, int thickness) {
    if (!text) return fail(WHENET_EINVAL, "null text");
    if (thickness != 1) return fail(WHENET_EINVAL, "thickness %d: only 1 is supported", thickness);
    if (!(scale > 0.0 && scale <= kTextMaxScale)) return fail(WHENET_EINVAL, "scale %g outside (0, %g]", scale, kTextMaxScale);
    if (ox < -kTextMaxOrg || ox > kTextMaxOrg || oy < -kTextMaxOrg || oy > kTextMaxOrg)
        return fail(WHENET_EINVAL, "origin (%d, %d) outside +-%d", ox, oy, kTextMaxOrg);
    int len = 0;
    for (const char* p = text; *p; ++p, ++len) {
        if (*p < 32 || *p > 126) return fail(WHENET_EINVAL, "character %d at %d is not printable ASCII", (int)(unsigned char)*p, len);
        if (len >= kTextMaxLen) return fail(WHENET_EINVAL, "text longer than %d characters", kTextMaxLen);
    }
    return 0;
}

int put_text_checked(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const int32_t* frame_of, const char* const* texts,
                     const int32_t* org, const double* scale, const uint8_t* bgr, const int32_t* thickness, int m) {
    if (int rc = check_frames(frames, hw, n)) return rc;
    if (m < 0 || m > kTextMaxItems) return fail(WHENET_EINVAL, "m=%d text items outside [0, %d]", m, kTextMaxItems);
    if (m == 0) return 0;
    if (!frame_of || !texts || !org || !scale || !bgr || !thickness) return fail(WHENET_EINVAL, "null item array");
    long long chars = 0;
    for (int i = 0; i < m; ++i) {
        if (frame_of[i] < 0 || frame_of[i] >= n) return fail(WHENET_EINVAL, "item %d: frame_of=%d outside [0, %d)", i, frame_of[i], n);
        if (int rc = check_text(texts[i], org[2 * i], org[2 * i + 1], scale[i], thickness[i])) return rc;
        chars += (long long)strlen(texts[i]);
    }
    if (chars > kTextMaxChars) return fail(WHENET_EINVAL, "%lld characters in one call, limit %lld", chars, kTextMaxChars);
    if (!c) return fail(WHENET_EINVAL, "null context");
    OverlayList L(n);
    for (int i = 0; i < m; ++i) {
        const int f = frame_of[i];
        const uint32_t col = bgr[3 * i] | (uint32_t)bgr[3 * i + 1] << 8 | (uint32_t)bgr[3 * i + 2] << 16;
        L.add_text(f, texts[i], org[2 * i], org[2 * i + 1], scale[i], col, hw[2 * f], hw[2 * f + 1]);
    }
    return draw_overlay_list(c, frames, hw, n, L);
}

int draw_heads_ex_checked(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes, const float* angles,
                          const int32_t* frame_of, int m, int display, int32_t* drawn_out) {
    if (display != 0 && display != 1) return fail(WHENET_EINVAL, "display=%d: 0 (simple) or 1 (full)", display);
    if (display == 0) return draw_heads_checked(c, frames, hw, n, boxes, angles, frame_of, m, drawn_out);
    if (int rc = check_frames(frames, hw, n)) return rc;
    if (m < 0 || m > kLabelMaxHeads) return fail(WHENET_EINVAL, "m=%d heads outside [0, %d] with display=1", m, kLabelMaxHeads);
    if (m == 0) return 0;
    if (!boxes || !angles || !frame_of) return fail(WHENET_EINVAL, "null boxes, angles or frame_of");
    for (int i = 0; i < m; ++i)
        if (frame_of[i] < 0 || frame_of[i] >= n) return fail(WHENET_EINVAL, "head %d: frame_of=%d outside [0, %d)", i, frame_of[i], n);
    if (!c) return fail(WHENET_EINVAL, "null context");
    return draw_heads_full(c, frames, hw, n, boxes, angles, frame_of, m, drawn_out);
}

int dense_frames(uint8_t* frames, int n, int H, int W, uint8_t** ptrs, int32_t* hw) {
    if (!frames) return fail(WHENET_EINVAL, "null frames");
    if (n < 1 || n > whenet::kMaxCropFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxCropFrames);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    for (int i = 0; i < n; ++i) {
        ptrs[i] = frames + (size_t)i * H * W * 3;
        hw[2 * i] = H; hw[2 * i + 1] = W;
    }
    return 0;
}

static_assert(whenet::kOverlayMaxFrames == whenet::kMaxCropFrames, "overlay frame table holds every crop frame");

}  // namespace

extern "C" {

int whenet_crop_resize_u8(whenet_ctx* c, const uint8_t* frame, int H, int W, int frame_is_device,
                          const int32_t* rects, int m, int swap_rb, uint8_t* crops_out) {
    if (!c || !frame || !rects || !crops_out) return fail(WHENET_EINVAL, "null argument");
    if (H < 1 || W < 1 || m < 1) return fail(WHENET_EINVAL, "bad frame size or box count");
    for (int i = 0; i < m; ++i) {
        const int32_t* r = rects + 4 * i;
        if (!(0 <= r[0] && r[0] < r[1] && r[1] <= H && 0 <= r[2] && r[2] < r[3] && r[3] <= W))
            return fail(WHENET_EINVAL, "box %d: slice [%d:%d, %d:%d] is empty or outside the %dx%d frame (cv2.resize would raise)",
                        i, r[0], r[1], r[2], r[3], H, W);
    }
    return launch_crops(c, frame, 1, H, W, frame_is_device, rects, nullptr, m, swap_rb, 0, crops_out);
}

int whenet_crop_boxes_u8(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, const float* boxes,
                         const int32_t* frame_of, int m, int swap_rb, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    return crop_boxes(c, frames, n, H, W, frames_are_device, boxes, frame_of, m, swap_rb, 0, crops_out, rects_out, valid_out);
}

int whenet_crop_boxes_yuv_u8(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, const float* boxes,
                             const int32_t* frame_of, int m, int yuv_layout, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    if (int rc = check_yuv_layout(yuv_layout)) return rc;
    return crop_boxes(c, frames, n, H, W, frames_are_device, boxes, frame_of, m, 1, yuv_layout, crops_out, rects_out, valid_out);
}

int whenet_crop_boxes_ragged_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const float* boxes,
                                const int32_t* frame_of, int m, int swap_rb, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    return crop_boxes_ragged(c, frames, hw, n, frames_are_device, boxes, frame_of, m, swap_rb, 0, crops_out, rects_out, valid_out);
}

int whenet_crop_boxes_ragged_yuv_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                    const float* boxes, const int32_t* frame_of, int m, int yuv_layout, uint8_t* crops_out, int32_t* rects_out,
                                    int32_t* valid_out) {
    if (int rc = check_yuv_layout(yuv_layout)) return rc;
    return crop_boxes_ragged(c, frames, hw, n, frames_are_device, boxes, frame_of, m, 1, yuv_layout, crops_out, rects_out, valid_out);
}

int whenet_crop_boxes_yuv422_u8(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, const float* boxes,
                                const int32_t* frame_of, int m, int yuv422_layout, uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out) {
    if (int rc = check_yuv422_layout(yuv422_layout)) return rc;
    return crop_boxes(c, frames, n, H, W, frames_are_device, boxes, frame_of, m, 1, yuv422_layout, crops_out, rects_out, valid_out);
}

int whenet_crop_boxes_ragged_yuv422_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                       const float* boxes, const int32_t* frame_of, int m, int yuv422_layout, uint8_t* crops_out,
                                       int32_t* rects_out, int32_t* valid_out) {
    if (int rc = check_yuv422_layout(yuv422_layout)) return rc;
    return crop_boxes_ragged(c, frames, hw, n, frames_are_device, boxes, frame_of, m, 1, yuv422_layout, crops_out, rects_out, valid_out);
}

int whenet_yuv_to_bgr_u8(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, int layout, uint8_t* out_frames) {
    // the context is checked last so that every other argument can be validated without a GPU
    if (int rc = check_convert_layout(layout)) return rc;
    if (!frames || !out_frames) return fail(WHENET_EINVAL, "null frames or out_frames");
    if (n < 1 || n > whenet::kMaxConvertFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxConvertFrames);
    if (int rc = check_convert_size(-1, H, W, layout)) return rc;
    if (!c) return fail(WHENET_EINVAL, "null context");
    return yuv_to_bgr(c, frames, n, H, W, frames_are_device, layout, out_frames);
}

int whenet_yuv_to_bgr_ragged_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int layout,
                                uint8_t* const* out_frames) {
    if (int rc = check_convert_layout(layout)) return rc;
    if (!frames || !hw || !out_frames) return fail(WHENET_EINVAL, "null frames, hw or out_frames");
    if (n < 1 || n > whenet::kMaxConvertFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxConvertFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i] || !out_frames[i]) return fail(WHENET_EINVAL, "frame %d: null frame or output", i);
        if (int rc = check_convert_size(i, hw[2 * i], hw[2 * i + 1], layout)) return rc;
    }
    if (!c) return fail(WHENET_EINVAL, "null context");
    return yuv_to_bgr_ragged(c, frames, hw, n, frames_are_device, layout, out_frames);
}

int whenet_draw_heads_u8(whenet_ctx* c, uint8_t* frames, int n, int H, int W, const float* boxes, const float* angles,
                         const int32_t* frame_of, int m, int32_t* drawn_out) {
    if (!frames) return fail(WHENET_EINVAL, "null frames");
    if (n < 1 || n > whenet::kMaxCropFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, whenet::kMaxCropFrames);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    uint8_t* ptrs[whenet::kMaxCropFrames];
    int32_t hw[2 * whenet::kMaxCropFrames];
    for (int i = 0; i < n; ++i) {
        ptrs[i] = frames + (size_t)i * H * W * 3;
        hw[2 * i] = H; hw[2 * i + 1] = W;
    }
    return draw_heads_checked(c, ptrs, hw, n, boxes, angles, frame_of, m, drawn_out);
}

int whenet_draw_heads_ragged_u8(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes,
                                const float* angles, const int32_t* frame_of, int m, int32_t* drawn_out) {
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    return draw_heads_checked(c, frames, hw, n, boxes, angles, frame_of, m, drawn_out);
}

int whenet_debug_overlay_segments(const float* boxes, const float* angles, int m, int H, int W, int32_t* seg_out, int32_t* drawn_out) {
    if (!boxes || !angles || m < 1) return fail(WHENET_EINVAL, "null boxes or angles, or m=%d heads", m);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    for (int i = 0; i < m; ++i) {
        int32_t seg[kSegsPerHead][4] = {};
        const bool ok = head_segments(boxes + 4 * i, angles + 3 * i, H, W, seg);
        if (!ok) memset(seg, 0, sizeof(seg));
        if (seg_out) memcpy(seg_out + (size_t)i * kSegsPerHead * 4, seg, sizeof(seg));
        if (drawn_out) drawn_out[i] = ok;
    }
    return 0;
}

int whenet_draw_heads_ex_u8(whenet_ctx* c, uint8_t* frames, int n, int H, int W, const float* boxes, const float* angles,
                            const int32_t* frame_of, int m, int display, int32_t* drawn_out) {
    uint8_t* ptrs[whenet::kMaxCropFrames];
    int32_t hw[2 * whenet::kMaxCropFrames];
    if (int rc = dense_frames(frames, n, H, W, ptrs, hw)) return rc;
    return draw_heads_ex_checked(c, ptrs, hw, n, boxes, angles, frame_of, m, display, drawn_out);
}

int whenet_draw_heads_ex_ragged_u8(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes,
                                   const float* angles, const int32_t* frame_of, int m, int display, int32_t* drawn_out) {
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    return draw_heads_ex_checked(c, frames, hw, n, boxes, angles, frame_of, m, display, drawn_out);
}

int whenet_put_text_u8(whenet_ctx* c, uint8_t* frames, int n, int H, int W, const int32_t* frame_of, const char* const* texts,
                       const int32_t* org, const double* scale, const uint8_t* bgr, const int32_t* thickness, int m) {
    uint8_t* ptrs[whenet::kMaxCropFrames];
    int32_t hw[2 * whenet::kMaxCropFrames];
    if (int rc = dense_frames(frames, n, H, W, ptrs, hw)) return rc;
    return put_text_checked(c, ptrs, hw, n, frame_of, texts, org, scale, bgr, thickness, m);
}

int whenet_put_text_ragged_u8(whenet_ctx* c, uint8_t* const* frames, const int32_t* hw, int n, const int32_t* frame_of,
                              const char* const* texts, const int32_t* org, const double* scale, const uint8_t* bgr,
                              const int32_t* thickness, int m) {
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    return put_text_checked(c, frames, hw, n, frame_of, texts, org, scale, bgr, thickness, m);
}

int whenet_debug_text_segments(const char* text, int org_x, int org_y, double scale, int thickness, int64_t* seg_out, int cap,
                               int32_t* count_out) {
    if (int rc = check_text(text, org_x, org_y, scale, thickness)) return rc;
    std::vector<long long> s;
    text_segments16(text, org_x, org_y, scale, s);
    const int count = (int)(s.size() / 4);
    if (count_out) *count_out = count;
    if (seg_out) memcpy(seg_out, s.data(), (size_t)std::min(count, std::max(cap, 0)) * 4 * sizeof(int64_t));
    return 0;
}

int whenet_debug_label_text(const float* angles, int m, char* out, int stride) {
    if (!angles || !out || m < 1 || stride < 32) return fail(WHENET_EINVAL, "null angles or out, m=%d, stride=%d < 32", m, stride);
    for (int i = 0; i < m; ++i) {
        const std::string t = label_number(angles[i]);
        snprintf(out + (size_t)i * stride, stride, "%s", t.c_str());
    }
    return 0;
}

int whenet_debug_enlarge_boxes(const float* boxes, int m, int H, int W, int32_t* rects_out, int32_t* valid_out) {
    if (!boxes || m < 1 || H < 1 || W < 1) return fail(WHENET_EINVAL, "bad arguments");
    for (int i = 0; i < m; ++i) {
        int32_t r[4];
        const bool ok = enlarge_box(boxes + 4 * i, H, W, r);
        if (rects_out) memcpy(rects_out + 4 * i, r, sizeof(r));
        if (valid_out) valid_out[i] = ok;
    }
    return 0;
}

}  // extern "C"
