// yolo_api.cu - C ABI of the YOLOv3 head detector (whenet_det_*): weights, workspaces, the captured forward, decode + NMS.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <initializer_list>
#include <map>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/whenet_b200.h"
#include "api_error.h"
#define WHENET_YOLO_HOST_ONLY
#define WHENET_YOLO32_HOST_ONLY
#include "kernels_yolo.cuh"
#include "kernels_yolo32.cuh"

using whenet::api::check_yuv422_layout;
using whenet::api::check_yuv_layout;
using whenet::api::fail;
namespace Y = whenet::yolo;

#define CKD(call)                                                                                  \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail(WHENET_ECUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,         \
                        cudaGetErrorString(e__));                                                  \
    } while (0)

namespace {

constexpr double kBnEps = 1e-3;     // keras BatchNormalization default (reference yolo_v3/model.py:34)
constexpr int kPoolTap = 100;       // whenet_det_debug_tap: kPoolTap + i = the max-pooled input of tiny conv i

using Y::ConvCfg;
using Y::make_table;

uint16_t bf16_bits(float f) {      // round to nearest even (finite inputs)
    uint32_t u;
    std::memcpy(&u, &f, 4);
    u += 0x7FFFu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}

// the fp32 mode's weight split: hi = bf16(v), lo = bf16(v - hi) (v - hi is exact in float)
void split_bits(float v, uint16_t& hi, uint16_t& lo) {
    hi = bf16_bits(v);
    const uint32_t u = (uint32_t)hi << 16;
    float h;
    std::memcpy(&h, &u, 4);
    lo = bf16_bits(v - h);
}

// Hi, Wi: the conv's input size (after the pool of a tiny conv); pooled: that pool's output, a buffer of its own
// plan / plan32: the tile plan of the bf16 / fp32 kernels (the one of the detector's precision is set)
struct LayerDev { int Hi, Wi, Ho, Wo, N; Y::IgemmPlan plan; Y::Igemm32Plan plan32; void* out = nullptr; void* pooled = nullptr; };

struct GraphEntry {
    cudaGraphExec_t exec = nullptr;
    void* coef = nullptr;           // letterbox tables (xb, kx, yb, ky; several frames: every frame's, then their LetterboxFrames) in one allocation
    uint8_t* tmp = nullptr;         // horizontal-pass output
};

// a graph of n frames of one size: (n, H, swap_rb ? W : -W, yuv_layout)
using OneSizeKey = std::tuple<int, int, int, int>;
// a graph of frames of several sizes: (H0, W0, H1, W1, ...), swap_rb and yuv_layout
using RaggedKey = std::tuple<std::vector<int>, int, int>;
constexpr size_t kMaxGraphs = 16;   // captured graphs kept per cache

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static_assert(whenet::kYuvNV12 == WHENET_YUV_NV12 && whenet::kYuvI420 == WHENET_YUV_I420, "layout codes of yuv.cuh and the ABI");
static_assert(whenet::kYuvYUYV == WHENET_YUV_YUYV && whenet::kYuvUYVY == WHENET_YUV_UYVY, "layout codes of yuv.cuh and the ABI");

// bytes of an H x W frame: packed 8-bit BGR / RGB (yuv_layout 0), YUV 4:2:0 (H and W even) or packed YUV 4:2:2 (W even)
size_t frame_bytes(int H, int W, int yuv_layout) {
    if (whenet::yuv422(yuv_layout)) return (size_t)H * W * 2;
    return yuv_layout ? (size_t)H * W / 2 * 3 : (size_t)H * W * 3;
}

// Pillow ImagingResample (libImaging/Resample.c) coefficient tables for BICUBIC: support 2 scaled by the downscale factor,
// weights normalised in double and quantised to 22 bits (normalize_coeffs_8bpc).
double bicubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}
int precompute_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& kk) {
    const double scale = (double)(float)in_size / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 2.0 * filterscale;
    const int ksize = (int)std::ceil(support) * 2 + 1;
    bounds.assign(2 * out_size, 0);
    kk.assign((size_t)out_size * ksize, 0);
    std::vector<double> k(ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        double ww = 0.0;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; ++x) {
            const double w = bicubic((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        for (int x = 0; x < ksize; ++x) {
            const double v = x < xmax ? k[x] : 0.0;
            kk[(size_t)xx * ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << 22)) : (int)(0.5 + v * (1 << 22));
        }
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
    return ksize;
}

}  // namespace

struct whenet_det {
    int device = 0, in_h = 0, in_w = 0, max_frames = 0, sm_count = 132;
    int num_classes = 0;
    int precision = WHENET_PRECISION_BF16;      // or WHENET_PRECISION_FP32: fp32 activations, split-bf16 MMAs (kernels_yolo32.cuh)
    bool tiny = false;                  // tiny YOLOv3 (6 anchors, 13 convs, two heads) instead of YOLOv3 (9 anchors, 75 convs)
    bool loaded = false;
    cudaStream_t own_stream = nullptr, stream = nullptr, cap_stream = nullptr;
    std::vector<ConvCfg> table;
    std::vector<LayerDev> L;
    void* warena = nullptr;             // bf16 kernels, [N][K] each, 256-byte aligned (fp32 mode: their hi parts)
    void* warena_lo = nullptr;          // fp32 mode: the lo parts, at the same offsets
    float* barena = nullptr;            // fp32 biases
    std::vector<size_t> w_off, b_off;
    float anchors[18] = {};             // in (head, anchor-in-layer) slots, see DecodeParams
    uint8_t* d_frames = nullptr; size_t frames_cap = 0;
    uint8_t* d_canvas = nullptr;
    float4* d_cand = nullptr; float* d_cand_score = nullptr;
    float* d_boxes = nullptr; float* d_scores = nullptr; int* d_classes = nullptr; int* d_count = nullptr;
    // the second decode route's kept keys and counts ([max_frames][C][kMaxBoxes], [max_frames][C]), allocated on its first use
    unsigned long long* d_keep = nullptr; int* d_keep_count = nullptr;
    bool force_large_decode = false;    // whenet_det_debug_force_large_decode
    std::map<OneSizeKey, GraphEntry> graphs;
    std::map<RaggedKey, GraphEntry> ragged_graphs;      // whenet_det_detect_ragged_u8's
    int last_n = 0;
};

namespace {

// candidates per frame: 1 + 4 + 16 cells per 32x32 block (tiny: 1 + 4)
int ncand(const whenet_det* d) { return 3 * (d->in_h / 32) * (d->in_w / 32) * (d->tiny ? 5 : 21); }
int num_heads(const whenet_det* d) { return d->tiny ? 2 : 3; }
bool is_fp32(const whenet_det* d) { return d->precision == WHENET_PRECISION_FP32; }

void free_layers(whenet_det* d) {
    for (auto& l : d->L) { cudaFree(l.out); cudaFree(l.pooled); l.out = l.pooled = nullptr; }
}

// the activations and every decode workspace (they are sized by the network, the class count and max_frames)
void free_activations(whenet_det* d) {
    free_layers(d);
    cudaFree(d->d_cand); cudaFree(d->d_cand_score); cudaFree(d->d_boxes); cudaFree(d->d_scores); cudaFree(d->d_classes); cudaFree(d->d_count);
    cudaFree(d->d_keep); cudaFree(d->d_keep_count);
    d->d_cand = nullptr; d->d_cand_score = nullptr; d->d_boxes = nullptr; d->d_scores = nullptr; d->d_classes = nullptr; d->d_count = nullptr;
    d->d_keep = nullptr; d->d_keep_count = nullptr;
}

// cudaMalloc that names the request when it fails.  The failed call's error is cleared, so that a later launch check does not
// report it and the process goes on using the device.
int dev_alloc(void** p, size_t bytes, const char* what) {
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) return 0;
    *p = nullptr;
    cudaGetLastError();
    return fail(WHENET_ECUDA, "cudaMalloc of %zu bytes (%.1f GB) for %s failed: %s", bytes, bytes / 1e9, what, cudaGetErrorString(e));
}
template <class T>
int dev_alloc(T** p, size_t bytes, const char* what) { return dev_alloc(reinterpret_cast<void**>(p), bytes, what); }

// Bytes whenet_det_load_weights allocates per frame for network T (tiny: 13 convs) with C classes at an h x w model input:
// every conv output, every pooled conv input, the decoded boxes and the class scores
size_t activation_bytes_per_frame(const std::vector<ConvCfg>& T, bool tiny, int h, int w, int C, bool f32) {
    std::vector<int> Ho(T.size()), Wo(T.size());
    size_t b = 0;
    for (size_t i = 0; i < T.size(); ++i) {
        const ConvCfg& c = T[i];
        const int Hi = Y::pooled(c.src < 0 ? h : Ho[c.src], c.pool), Wi = Y::pooled(c.src < 0 ? w : Wo[c.src], c.pool);
        Ho[i] = Hi / c.stride; Wo[i] = Wi / c.stride;
        const int N = c.head >= 0 ? 3 * (5 + C) : c.cout;
        b += (size_t)Ho[i] * Wo[i] * N * (c.head >= 0 || f32 ? 4 : 2);
        if (c.pool) b += (size_t)Hi * Wi * c.cin * (f32 ? 4 : 2);
    }
    const size_t nc = (size_t)3 * (h / 32) * (w / 32) * (tiny ? 5 : 21);
    return b + nc * 16 + (size_t)C * nc * 4;
}

// A request larger than the whole device is refused before anything is allocated for it
int check_fits(int device, size_t bytes, const char* what) {
    size_t free_b = 0, total_b = 0;
    CKD(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > total_b)
        return fail(WHENET_ECUDA, "%s needs %zu bytes (%.1f GB) of device memory; device %d has %zu bytes (%.1f GB) in all", what, bytes, bytes / 1e9,
                    device, total_b, total_b / 1e9);
    return 0;
}

void free_entry(GraphEntry& e) {
    if (e.exec) cudaGraphExecDestroy(e.exec);
    cudaFree(e.coef);
    cudaFree(e.tmp);
}

template <class Map>
void free_graph_map(Map& m) {
    for (auto& kv : m) free_entry(kv.second);
    m.clear();
}

// both caches (weights reloaded, frame buffer reallocated, detector destroyed)
void free_graphs(whenet_det* d) {
    free_graph_map(d->graphs);
    free_graph_map(d->ragged_graphs);
}

const __nv_bfloat16* bf(const whenet_det* d, size_t off) { return reinterpret_cast<const __nv_bfloat16*>((const char*)d->warena + off); }
const __nv_bfloat16* bf_lo(const whenet_det* d, size_t off) { return reinterpret_cast<const __nv_bfloat16*>((const char*)d->warena_lo + off); }

// enqueue_conv of an fp32 detector
int enqueue_conv32(whenet_det* d, cudaStream_t s, int i, int n) {
    const ConvCfg& c = d->table[i];
    const LayerDev& l = d->L[i];
    if (c.pool) {
        const LayerDev& src = d->L[c.src];
        const int rc = Y::launch_maxpool32(s, (const float*)src.out, (float*)l.pooled, n, src.Ho, src.Wo, src.N, c.pool);
        if (rc) return fail(WHENET_ECUDA, "max-pool before conv %d launch failed: %s", i, cudaGetErrorString((cudaError_t)rc));
    }
    Y::Igemm32Params p{};
    const int N = l.N;
    p.in = (const float*)(c.pool ? l.pooled : d->L[c.src].out);
    p.up = c.up >= 0 ? (const float*)d->L[c.up].out : nullptr;
    p.w_hi = bf(d, d->w_off[i]);
    p.w_lo = bf_lo(d, d->w_off[i]);
    p.bias = d->barena + d->b_off[i];
    p.resid = c.res >= 0 ? (const float*)d->L[c.res].out : nullptr;
    p.out = (float*)l.out;
    p.M = n * l.Ho * l.Wo; p.Hi = l.Hi; p.Wi = l.Wi; p.Ho = l.Ho; p.Wo = l.Wo;
    p.Cin = c.cin; p.c_up = c.up >= 0 ? d->table[c.up].cout : 0; p.N = N; p.k = c.k; p.stride = c.stride;
    p.n_tile = l.plan32.n_tile; p.n_stages = l.plan32.n_stages;
    const int rc = Y::launch_igemm32(s, p, Y::igemm_mode(c), l.plan32.un, l.plan32.smem, (N + l.plan32.n_tile - 1) / l.plan32.n_tile,
                                     (p.M + Y::BM - 1) / Y::BM);
    if (rc) return fail(WHENET_ECUDA, "conv %d launch failed: %s", i, cudaGetErrorString((cudaError_t)rc));
    return 0;
}

// enqueue one conv (every table conv but the first), with the max-pool of its input for a tiny conv, on stream s, n frames
int enqueue_conv(whenet_det* d, cudaStream_t s, int i, int n) {
    if (is_fp32(d)) return enqueue_conv32(d, s, i, n);
    const ConvCfg& c = d->table[i];
    const LayerDev& l = d->L[i];
    if (c.pool) {
        const LayerDev& src = d->L[c.src];
        const int rc = Y::launch_maxpool(s, (const __nv_bfloat16*)src.out, (__nv_bfloat16*)l.pooled, n, src.Ho, src.Wo, src.N, c.pool);
        if (rc) return fail(WHENET_ECUDA, "max-pool before conv %d launch failed: %s", i, cudaGetErrorString((cudaError_t)rc));
    }
    Y::IgemmParams p{};
    const int N = l.N;
    p.in = reinterpret_cast<const __nv_bfloat16*>(c.pool ? l.pooled : d->L[c.src].out);
    p.up = c.up >= 0 ? reinterpret_cast<const __nv_bfloat16*>(d->L[c.up].out) : nullptr;
    p.wt = bf(d, d->w_off[i]);
    p.bias = d->barena + d->b_off[i];
    p.resid = c.res >= 0 ? reinterpret_cast<const __nv_bfloat16*>(d->L[c.res].out) : nullptr;
    p.out = l.out;
    p.M = n * l.Ho * l.Wo; p.Hi = l.Hi; p.Wi = l.Wi; p.Ho = l.Ho; p.Wo = l.Wo;
    p.Cin = c.cin; p.c_up = c.up >= 0 ? d->table[c.up].cout : 0; p.N = N; p.k = c.k; p.stride = c.stride;
    p.n_tile = l.plan.n_tile; p.n_stages = l.plan.n_stages;
    const int rc = Y::launch_igemm(s, p, Y::igemm_mode(c), l.plan.un, l.plan.smem, (N + l.plan.n_tile - 1) / l.plan.n_tile, (p.M + Y::BM - 1) / Y::BM);
    if (rc) return fail(WHENET_ECUDA, "conv %d launch failed: %s", i, cudaGetErrorString((cudaError_t)rc));
    return 0;
}

// The letterbox of one H x W frame: geometry, and Pillow's tables appended to `blob`, each 256-byte aligned (int2 loads), at the
// offsets f records (src and tmp are left to the caller)
int frame_plan(const whenet_det* d, int H, int W, std::vector<char>& blob, Y::LetterboxFrame* f) {
    // letterbox geometry (reference utils.py:25-33): scale in float64, int() truncation, paste at the floor-halved offsets
    const double scale = std::min((double)d->in_w / W, (double)d->in_h / H);
    const int nw = (int)(W * scale), nh = (int)(H * scale);
    if (nw < 1 || nh < 1) return fail(WHENET_EINVAL, "a %dx%d frame letterboxes to an empty %dx%d image", W, H, nw, nh);
    std::vector<int> xb, kx, yb, ky;
    const int ksx = precompute_coeffs(W, nw, xb, kx), ksy = precompute_coeffs(H, nh, yb, ky);
    const int y0 = yb[0], rows = yb[2 * (nh - 1)] + yb[2 * nh - 1] - y0;      // Pillow's ybox_first / ybox_last
    for (int y = 0; y < nh; ++y) yb[2 * y] -= y0;
    int off[4];
    const std::vector<int>* tabs[4] = {&xb, &kx, &yb, &ky};
    for (int t = 0; t < 4; ++t) {
        off[t] = (int)blob.size();
        blob.resize(align256(blob.size() + tabs[t]->size() * 4), 0);
        std::memcpy(blob.data() + off[t], tabs[t]->data(), tabs[t]->size() * 4);
    }
    *f = Y::LetterboxFrame{0, 0, H, W, nw, nh, (d->in_w - nw) / 2, (d->in_h - nh) / 2, y0, rows, ksx, ksy, off[0], off[1], off[2], off[3]};
    return 0;
}

// The letterbox (enqueued by `letterbox` on the stream it is given), the first conv and the body for n frames, as one graph
// captured on the context's private stream
template <class Letterbox>
int capture_forward(whenet_det* d, int n, Letterbox&& letterbox, GraphEntry* e) {
    cudaStream_t s = d->cap_stream;
    CKD(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
    int rc = letterbox(s);
    if (!rc && is_fp32(d))
        rc = Y::launch_conv0_32(s, d->d_canvas, bf(d, d->w_off[0]), bf_lo(d, d->w_off[0]), d->barena + d->b_off[0], (float*)d->L[0].out, n,
                                d->in_h, d->in_w, d->table[0].cout);
    else if (!rc)
        rc = Y::launch_conv0(s, d->d_canvas, bf(d, d->w_off[0]), d->barena + d->b_off[0], (__nv_bfloat16*)d->L[0].out, n, d->in_h, d->in_w,
                             d->table[0].cout);
    int rc2 = rc ? fail(WHENET_ECUDA, "letterbox / first conv launch failed: %s", cudaGetErrorString((cudaError_t)rc)) : 0;
    for (size_t i = 1; i < d->table.size() && !rc2; ++i) rc2 = enqueue_conv(d, s, (int)i, n);
    cudaGraph_t g = nullptr;
    const cudaError_t ee = cudaStreamEndCapture(s, &g);
    if (rc2) { if (g) cudaGraphDestroy(g); return rc2; }
    CKD(ee);
    const cudaError_t ie = cudaGraphInstantiate(&e->exec, g, 0);
    cudaGraphDestroy(g);
    CKD(ie);
    return 0;
}

int make_entry(whenet_det* d, int n, int H, int W, int swap_rb, int yuv_layout, GraphEntry* e) {
    std::vector<char> blob;
    Y::LetterboxFrame f;
    if (int rc = frame_plan(d, H, W, blob, &f)) return rc;
    CKD(cudaMalloc(&e->coef, blob.size()));
    char* base = (char*)e->coef;
    CKD(cudaMemcpy(base, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    if (int rc = dev_alloc(&e->tmp, (size_t)n * f.rows * f.nw * 3, "the letterbox's horizontal pass")) return rc;
    Y::LetterboxPlan lp{H, W, f.nw, f.nh, f.ox, f.oy, f.y0, f.rows, f.ksx, f.ksy,
                        (const int2*)(base + f.xb), (const int*)(base + f.kx), (const int2*)(base + f.yb), (const int*)(base + f.ky)};
    return capture_forward(d, n, [&](cudaStream_t s) { return Y::launch_letterbox(s, lp, d->d_frames, e->tmp, d->d_canvas, n, d->in_h, d->in_w, swap_rb,
                                                                             yuv_layout); },
                           e);
}

// frame i at byte offset off[i] of d_frames, hw[2i] x hw[2i+1]
int make_ragged_entry(whenet_det* d, int n, const int32_t* hw, const std::vector<size_t>& off, int swap_rb, int yuv_layout, GraphEntry* e) {
    std::vector<char> blob;
    std::vector<Y::LetterboxFrame> plans(n);
    size_t tmp_bytes = 0;
    long long max_hx = 0;
    for (int i = 0; i < n; ++i) {
        Y::LetterboxFrame& f = plans[i];
        if (int rc = frame_plan(d, hw[2 * i], hw[2 * i + 1], blob, &f)) return rc;
        f.src = (long long)off[i];
        f.tmp = (long long)tmp_bytes;
        tmp_bytes = align256(tmp_bytes + (size_t)f.rows * f.nw * 3);
        max_hx = std::max(max_hx, (long long)f.rows * f.nw);
    }
    const size_t plans_at = blob.size();
    blob.resize(plans_at + plans.size() * sizeof(Y::LetterboxFrame));
    std::memcpy(blob.data() + plans_at, plans.data(), plans.size() * sizeof(Y::LetterboxFrame));
    CKD(cudaMalloc(&e->coef, blob.size()));
    CKD(cudaMemcpy(e->coef, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    if (int rc = dev_alloc(&e->tmp, tmp_bytes, "the letterbox's horizontal pass")) return rc;
    const char* coef = (const char*)e->coef;
    const auto* d_plans = (const Y::LetterboxFrame*)(coef + plans_at);
    return capture_forward(d, n, [&](cudaStream_t s) {
        return Y::launch_letterbox_ragged(s, d_plans, coef, d->d_frames, e->tmp, d->d_canvas, n, max_hx, d->in_h, d->in_w, swap_rb, yuv_layout);
    }, e);
}

int check_frames(const whenet_det* d, int n, int H, int W) {
    if (n < 1 || n > d->max_frames) return fail(WHENET_EINVAL, "n=%d outside [1, max_frames=%d]", n, d->max_frames);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    return 0;
}

// DecodeParams of one call of n frames, frame i img_hw[2i] x img_hw[2i+1] (img_hw NULL: every frame img_h x img_w):
// yolo_correct_boxes' float32 arithmetic (model.py:157-161) on the host, one geo row per frame
Y::DecodeParams decode_params(const whenet_det* d, int n, const int32_t* img_hw, int img_h, int img_w, float score, float iou, int max_boxes) {
    Y::DecodeParams p{};
    p.cand = d->d_cand; p.cand_score = d->d_cand_score;
    p.out_boxes = d->d_boxes; p.out_scores = d->d_scores; p.out_classes = d->d_classes; p.out_count = d->d_count;
    std::memcpy(p.anchors, d->anchors, sizeof(p.anchors));
    p.gh0 = d->in_h / 32; p.gw0 = d->in_w / 32; p.C = d->num_classes; p.NC = ncand(d); p.max_boxes = max_boxes;
    p.in_h = (float)d->in_h; p.in_w = (float)d->in_w;
    for (int i = 0; i < n; ++i) {
        Y::FrameGeo& g = p.geo[i];
        g.img_h = (float)(img_hw ? img_hw[2 * i] : img_h); g.img_w = (float)(img_hw ? img_hw[2 * i + 1] : img_w);
        const float m = std::min(p.in_h / g.img_h, p.in_w / g.img_w);
        const float nh = std::nearbyint(g.img_h * m), nw = std::nearbyint(g.img_w * m);       // K.round: half to even
        g.off_y = (p.in_h - nh) / 2.0f / p.in_h; g.off_x = (p.in_w - nw) / 2.0f / p.in_w;
        g.scale_y = p.in_h / nh; g.scale_x = p.in_w / nw;
    }
    p.score = score; p.iou = iou;
    const int heads = num_heads(d);
    for (int l = 0; l < heads; ++l) p.head[l] = (const float*)d->L[d->table.size() - heads + l].out;
    return p;
}

int run_decode(whenet_det* d, const Y::DecodeParams& p, int n, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    if ((d->force_large_decode || Y::large_decode_route(p.NC)) && !d->d_keep) {
        const size_t slots = (size_t)d->max_frames * d->num_classes;
        int rc = dev_alloc(&d->d_keep, slots * Y::kMaxBoxes * 8, "the kept NMS keys");
        if (!rc) rc = dev_alloc(&d->d_keep_count, slots * 4, "the kept NMS counts");
        if (rc) {                       // both or neither: the next call allocates them again
            cudaFree(d->d_keep);
            d->d_keep = nullptr;
            return rc;
        }
    }
    const int rc = Y::launch_decode_nms(d->stream, p, n, d->force_large_decode, d->d_keep, d->d_keep_count);
    if (rc) return fail(WHENET_ECUDA, "decode/NMS launch failed: %s", cudaGetErrorString((cudaError_t)rc));
    const size_t slots = (size_t)n * p.C * p.max_boxes;
    CKD(cudaMemcpyAsync(boxes, d->d_boxes, slots * 16, cudaMemcpyDeviceToHost, d->stream));
    CKD(cudaMemcpyAsync(scores, d->d_scores, slots * 4, cudaMemcpyDeviceToHost, d->stream));
    CKD(cudaMemcpyAsync(classes, d->d_classes, slots * 4, cudaMemcpyDeviceToHost, d->stream));
    CKD(cudaMemcpyAsync(counts, d->d_count, (size_t)n * 4, cudaMemcpyDeviceToHost, d->stream));
    CKD(cudaStreamSynchronize(d->stream));
    return 0;
}

int check_decode_args(const whenet_det* d, float score, float iou, int max_boxes, const void* boxes, const void* scores, const void* classes,
                      const void* counts) {
    if (!d->loaded) return fail(WHENET_ENOWEIGHTS, "whenet_det_load_weights has not been called");
    if (!boxes || !scores || !classes || !counts) return fail(WHENET_EINVAL, "null output pointer");
    if (max_boxes < 1 || max_boxes > Y::kMaxBoxes) return fail(WHENET_EINVAL, "max_boxes=%d outside [1, %d]", max_boxes, Y::kMaxBoxes);
    if (!(score >= 0.f && score <= 1.f) || !(iou >= 0.f && iou <= 1.f)) return fail(WHENET_EINVAL, "score / iou thresholds must be in [0, 1]");
    return 0;
}

int to_f32_tap(const void* src, bool is_f32, size_t n, float* out) {
    if (is_f32) { CKD(cudaMemcpy(out, src, n * 4, cudaMemcpyDeviceToHost)); return 0; }
    std::vector<uint16_t> h(n);
    CKD(cudaMemcpy(h.data(), src, n * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) { const uint32_t u = (uint32_t)h[i] << 16; std::memcpy(out + i, &u, 4); }
    return 0;
}

// whenet_det_debug_conv on an fp32 detector (arguments checked): the host float32 values as given, the weights split into hi
// and lo as whenet_det_load_weights splits them, conv_igemm32_kernel, fp32 output
int debug_conv32(whenet_det* d, const float* x, const float* up, int n, int H, int W, int cin, int c_up, const float* w, const float* bias,
                 int k, int stride, int cout, int leaky, const float* resid, float* out) {
    const int Ho = H / stride, Wo = W / stride;
    const size_t nx = (size_t)n * H * W * (cin - c_up), nu = (size_t)n * (H / 2) * (W / 2) * c_up, no = (size_t)n * Ho * Wo * cout;
    const int K = k * k * cin, rows = (cout + 127) / 128 * 128;
    std::vector<uint16_t> hw((size_t)rows * K, 0), hl((size_t)rows * K, 0);
    for (int o = 0; o < cout; ++o)
        for (int i = 0; i < K; ++i) split_bits(w[(size_t)i * cout + o], hw[(size_t)o * K + i], hl[(size_t)o * K + i]);
    std::vector<float> hb((size_t)rows, 0.f);
    std::copy(bias, bias + cout, hb.begin());
    void *dx = nullptr, *du = nullptr, *dw = nullptr, *dl = nullptr, *db = nullptr, *dr = nullptr, *dout = nullptr;
    auto cleanup = [&]() { cudaFree(dx); cudaFree(du); cudaFree(dw); cudaFree(dl); cudaFree(db); cudaFree(dr); cudaFree(dout); };
    if (cudaMalloc(&dx, nx * 4) || (nu && cudaMalloc(&du, nu * 4)) || cudaMalloc(&dw, hw.size() * 2) || cudaMalloc(&dl, hl.size() * 2) ||
        cudaMalloc(&db, hb.size() * 4) || (resid && cudaMalloc(&dr, no * 4)) || cudaMalloc(&dout, no * 4)) {
        cleanup();
        return fail(WHENET_ECUDA, "out of device memory");
    }
    // on the detector's stream, as whenet_det_debug_conv does (pageable copies may return before their DMA has landed)
    cudaMemcpyAsync(dx, x, nx * 4, cudaMemcpyHostToDevice, d->stream);
    if (nu) cudaMemcpyAsync(du, up, nu * 4, cudaMemcpyHostToDevice, d->stream);
    cudaMemcpyAsync(dw, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice, d->stream);
    cudaMemcpyAsync(dl, hl.data(), hl.size() * 2, cudaMemcpyHostToDevice, d->stream);
    cudaMemcpyAsync(db, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice, d->stream);
    if (resid) cudaMemcpyAsync(dr, resid, no * 4, cudaMemcpyHostToDevice, d->stream);
    Y::Igemm32Params p{};
    p.in = (const float*)dx; p.up = (const float*)du; p.w_hi = (const __nv_bfloat16*)dw; p.w_lo = (const __nv_bfloat16*)dl;
    p.bias = (const float*)db; p.resid = (const float*)dr; p.out = (float*)dout;
    p.M = n * Ho * Wo; p.Hi = H; p.Wi = W; p.Ho = Ho; p.Wo = Wo; p.Cin = cin; p.c_up = c_up; p.N = cout; p.k = k; p.stride = stride;
    const Y::Igemm32Plan pl = Y::plan_igemm32(Ho, Wo, cout, cin, k, d->sm_count);
    p.n_tile = pl.n_tile; p.n_stages = pl.n_stages;
    const int mode = !leaky ? Y::kLinearF32 : up ? Y::kLeakyCat : resid ? Y::kLeakyRes : Y::kLeaky;
    int rc = Y::launch_igemm32(d->stream, p, mode, pl.un, pl.smem, (cout + pl.n_tile - 1) / pl.n_tile, (p.M + Y::BM - 1) / Y::BM);
    if (!rc) rc = (int)cudaStreamSynchronize(d->stream);
    if (!rc) rc = to_f32_tap(dout, true, no, out) ? -1 : 0;
    cleanup();
    if (rc > 0) return fail(WHENET_ECUDA, "debug conv failed: %s", cudaGetErrorString((cudaError_t)rc));
    return rc ? WHENET_ECUDA : 0;
}

}  // namespace

extern "C" {

int whenet_det_create(whenet_det** out, int device, int input_h, int input_w, int max_frames) {
    return whenet_det_create_ex(out, device, input_h, input_w, max_frames, WHENET_PRECISION_BF16);
}

}  // extern "C"

namespace {

// whenet_det_create_ex (sides up to 608) and whenet_det_create_large (up to 4096)
int create_detector(whenet_det** out, int device, int input_h, int input_w, int max_frames, int precision, int max_side) {
    if (!out) return fail(WHENET_EINVAL, "out is NULL");
    *out = nullptr;
    for (int v : {input_h, input_w})
        if (v < 32 || v > max_side || v % 32)
            return fail(WHENET_EINVAL, "input size %dx%d: both must be multiples of 32 in [32, %d]", input_w, input_h, max_side);
    if (max_frames < 1 || max_frames > 64) return fail(WHENET_EINVAL, "max_frames=%d outside [1, 64]", max_frames);
    if (precision != WHENET_PRECISION_BF16 && precision != WHENET_PRECISION_FP32)
        return fail(WHENET_EINVAL, "precision %d: the detector runs in WHENET_PRECISION_BF16 (%d) or WHENET_PRECISION_FP32 (%d)", precision,
                    WHENET_PRECISION_BF16, WHENET_PRECISION_FP32);
    int ndev = 0;
    CKD(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(WHENET_EINVAL, "device %d not in [0,%d)", device, ndev);
    CKD(cudaSetDevice(device));
    cudaDeviceProp prop;
    CKD(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(WHENET_ECUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    // the canvases and the smallest network's activations (tiny YOLOv3, one class): a detector that cannot hold even these is
    // refused before its first buffer
    const bool f32 = precision == WHENET_PRECISION_FP32;
    const size_t least = (size_t)max_frames * ((size_t)input_h * input_w * 3 +
                                               activation_bytes_per_frame(Y::make_tiny_table(), true, input_h, input_w, 1, f32));
    if (int rc = check_fits(device, least, "a detector of this size, precision and max_frames")) return rc;
    whenet_det* d = new whenet_det();
    d->device = device; d->in_h = input_h; d->in_w = input_w; d->max_frames = max_frames; d->sm_count = prop.multiProcessorCount;
    d->precision = precision;
    d->table = make_table();
    d->L.resize(d->table.size());
    auto bail = [&](int rc) { whenet_det_destroy(d); return rc; };
    if (cudaStreamCreateWithFlags(&d->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&d->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
        return bail(fail(WHENET_ECUDA, "stream creation failed"));
    d->stream = d->own_stream;
    if (int rc = dev_alloc(&d->d_canvas, (size_t)max_frames * input_h * input_w * 3, "the letterboxed canvases")) return bail(rc);
    *out = d;
    return 0;
}

}  // namespace

extern "C" {

int whenet_det_create_ex(whenet_det** out, int device, int input_h, int input_w, int max_frames, int precision) {
    return create_detector(out, device, input_h, input_w, max_frames, precision, 608);
}

int whenet_det_create_large(whenet_det** out, int device, int input_h, int input_w, int max_frames, int precision) {
    return create_detector(out, device, input_h, input_w, max_frames, precision, Y::kMaxSide);
}

int whenet_det_load_weights(whenet_det* d, const whenet_tensor* t, int n_tensors, const float* anchors, int n_anchors) {
    // the anchor count picks the network, as the reference does (yolo_postprocess.py:73)
    if (n_anchors != 6 && n_anchors != 9) return fail(WHENET_EINVAL, "YOLOv3 needs 9 anchors and tiny YOLOv3 6, got %d", n_anchors);
    if (!d || !t || !anchors) return fail(WHENET_EINVAL, "bad arguments");
    const bool tiny = n_anchors == 6;
    const std::vector<ConvCfg> T = tiny ? Y::make_tiny_table() : make_table();
    // tensors in table order: kernel [k,k,cin,cout], then gamma, beta, moving_mean, moving_variance (BN convs) or bias (output convs)
    size_t need = 0;
    for (const ConvCfg& c : T) need += c.bn ? 5 : 2;
    if ((size_t)n_tensors != need)
        return fail(WHENET_ESHAPE, "expected %zu tensors (%s: %zu convs + BatchNorms), got %d", need, tiny ? "tiny YOLOv3" : "YOLOv3", T.size(), n_tensors);
    const whenet_tensor& h0 = t[need - 2];      // output conv of head 2 (its kernel), all heads have the same width
    if (h0.ndim != 4 || h0.dims[3] < 18 || h0.dims[3] % 3) return fail(WHENET_ESHAPE, "%s: output conv width is not 3 * (5 + classes)", h0.name ? h0.name : "?");
    const int C = (int)h0.dims[3] / 3 - 5;
    const bool f32 = is_fp32(d);
    std::vector<uint16_t> hw, hw_lo;       // hw_lo: fp32 mode, the lo parts
    std::vector<float> hb;
    std::vector<size_t> w_off, b_off;
    size_t ti = 0;
    for (size_t i = 0; i < T.size(); ++i) {
        const ConvCfg& c = T[i];
        const int co = c.head >= 0 ? 3 * (5 + C) : c.cout;
        const whenet_tensor& k = t[ti++];
        const char* kn = k.name ? k.name : "?";
        if (k.ndim != 4 || k.dims[0] != c.k || k.dims[1] != c.k || k.dims[2] != c.cin || k.dims[3] != co)
            return fail(WHENET_ESHAPE, "%s (conv %zu): kernel must be [%d,%d,%d,%d]", kn, i, c.k, c.k, c.cin, co);
        std::vector<double> scale(co, 1.0), shift(co, 0.0);
        if (c.bn) {
            const whenet_tensor* bn[4] = {&t[ti], &t[ti + 1], &t[ti + 2], &t[ti + 3]};
            ti += 4;
            for (auto* b : bn)
                if (b->ndim != 1 || b->dims[0] != co) return fail(WHENET_ESHAPE, "%s (BatchNorm of conv %zu): must be [%d]", b->name ? b->name : "?", i, co);
            for (int o = 0; o < co; ++o) {
                scale[o] = (double)bn[0]->data[o] / std::sqrt((double)bn[3]->data[o] + kBnEps);
                shift[o] = (double)bn[1]->data[o] - (double)bn[2]->data[o] * scale[o];
            }
        } else {
            const whenet_tensor& b = t[ti++];
            if (b.ndim != 1 || b.dims[0] != co) return fail(WHENET_ESHAPE, "%s (output conv %zu): bias must be [%d]", b.name ? b.name : "?", i, co);
            for (int o = 0; o < co; ++o) shift[o] = b.data[o];
        }
        // kernel -> [N][K] bf16 (K = (ky*k + kx)*cin + ci); conv 0 -> [N][64] = [w(27) 0(5) w(27) 0(5)] for the hi/lo input split.
        // fp32 mode: hw holds the hi parts in that layout, hw_lo the lo parts ([N][K]; conv 0: [N][64] = [w_lo(27) 0(37)])
        const int taps = c.k * c.k;
        const int N = co, K = i == 0 ? 64 : taps * c.cin;
        const int rows = (N + 127) / 128 * 128;     // every weight tile the kernels may touch exists (zero rows past N)
        w_off.push_back(hw.size() * 2);
        hw.resize(hw.size() + (size_t)rows * K + 128, 0);
        if (f32) hw_lo.resize(hw.size(), 0);
        uint16_t* dst = hw.data() + w_off.back() / 2;
        uint16_t* dst_lo = f32 ? hw_lo.data() + w_off.back() / 2 : nullptr;
        for (int o = 0; o < N; ++o)
            for (int tp = 0; tp < taps; ++tp)
                for (int ci = 0; ci < c.cin; ++ci) {
                    const float wf = (float)((double)k.data[((size_t)tp * c.cin + ci) * co + o] * scale[o]);
                    uint16_t v, lo = 0;
                    if (f32) split_bits(wf, v, lo);
                    else v = bf16_bits(wf);
                    const size_t j = (size_t)o * K + (i == 0 ? (size_t)tp * 3 + ci : (size_t)tp * c.cin + ci);
                    dst[j] = v;
                    if (i == 0) dst[j + 32] = v;
                    if (f32) dst_lo[j] = lo;
                }
        b_off.push_back(hb.size());
        hb.resize(hb.size() + (size_t)(N + 127) / 128 * 128, 0.f);
        for (int o = 0; o < N; ++o) hb[b_off.back() + o] = (float)shift[o];
    }
    CKD(cudaSetDevice(d->device));
    // everything the detector will hold; more than the device has is refused here, the detector left as it was
    const size_t total = (hw.size() + hw_lo.size()) * 2 + hb.size() * 4 +
                         (size_t)d->max_frames * ((size_t)d->in_h * d->in_w * 3 + activation_bytes_per_frame(T, tiny, d->in_h, d->in_w, C, f32));
    if (int rc = check_fits(d->device, total, "this network at this size, precision and max_frames")) return rc;
    CKD(cudaStreamSynchronize(d->stream));
    free_graphs(d);
    cudaFree(d->warena); cudaFree(d->warena_lo); cudaFree(d->barena);
    d->warena = nullptr; d->warena_lo = nullptr; d->barena = nullptr; d->loaded = false;
    if (int rc = dev_alloc(&d->warena, hw.size() * 2, "the conv weights")) return rc;
    if (int rc = dev_alloc(&d->barena, hb.size() * 4, "the conv biases")) return rc;
    CKD(cudaMemcpy(d->warena, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice));
    if (f32) {
        if (int rc = dev_alloc(&d->warena_lo, hw_lo.size() * 2, "the conv weights' lo parts")) return rc;
        CKD(cudaMemcpy(d->warena_lo, hw_lo.data(), hw_lo.size() * 2, cudaMemcpyHostToDevice));
    }
    CKD(cudaMemcpy(d->barena, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice));
    d->w_off = w_off; d->b_off = b_off;
    // anchors in (head, anchor-in-layer) slots: the decode reads slot 3 * l + a for either network
    for (int l = 0; l < (tiny ? 2 : 3); ++l)
        for (int a = 0; a < 3; ++a) {
            const int an = tiny ? Y::kTinyAnchorMask[l][a] : Y::kAnchorMask[l][a];
            d->anchors[2 * (3 * l + a)] = anchors[2 * an];
            d->anchors[2 * (3 * l + a) + 1] = anchors[2 * an + 1];
        }
    // activations: one buffer per conv output and per pooled conv input (the concat and residual sources and the taps stay
    // addressable), workspaces; rebuilt when the network or the class count changes.  A failed allocation frees them all and
    // leaves the detector without weights.
    if (C != d->num_classes || tiny != d->tiny || !d->L[0].out) {
        free_activations(d);
        d->num_classes = C;
        d->tiny = tiny;
        d->table = T;
        d->L.assign(T.size(), LayerDev{});
        for (size_t i = 0; i < T.size(); ++i) {
            const ConvCfg& c = T[i];
            LayerDev& l = d->L[i];
            l.Hi = Y::pooled(c.src < 0 ? d->in_h : d->L[c.src].Ho, c.pool);
            l.Wi = Y::pooled(c.src < 0 ? d->in_w : d->L[c.src].Wo, c.pool);
            l.Ho = l.Hi / c.stride; l.Wo = l.Wi / c.stride;
            l.N = c.head >= 0 ? 3 * (5 + C) : c.cout;
            if (f32) l.plan32 = Y::plan_igemm32(l.Ho, l.Wo, l.N, c.cin, c.k, d->sm_count);
            else l.plan = Y::plan_igemm(l.Ho, l.Wo, l.N, c.cin, c.k, d->sm_count);
        }
        int rc = 0;
        for (size_t i = 0; i < T.size() && !rc; ++i) {
            const ConvCfg& c = T[i];
            LayerDev& l = d->L[i];
            rc = dev_alloc(&l.out, (size_t)d->max_frames * l.Ho * l.Wo * l.N * (c.head >= 0 || f32 ? 4 : 2), "a conv output");
            if (!rc && c.pool) rc = dev_alloc(&l.pooled, (size_t)d->max_frames * l.Hi * l.Wi * c.cin * (f32 ? 4 : 2), "a max-pool output");
        }
        const size_t nc = (size_t)ncand(d), slots = (size_t)d->max_frames * C * Y::kMaxBoxes;
        if (!rc) rc = dev_alloc(&d->d_cand, (size_t)d->max_frames * nc * 16, "the decoded boxes");
        if (!rc) rc = dev_alloc(&d->d_cand_score, (size_t)d->max_frames * C * nc * 4, "the class scores");
        if (!rc) rc = dev_alloc(&d->d_boxes, slots * 16, "the output boxes");
        if (!rc) rc = dev_alloc(&d->d_scores, slots * 4, "the output scores");
        if (!rc) rc = dev_alloc(&d->d_classes, slots * 4, "the output classes");
        if (!rc) rc = dev_alloc(&d->d_count, (size_t)d->max_frames * 4, "the output counts");
        if (rc) {
            free_activations(d);
            d->num_classes = 0;
            return rc;
        }
    }
    d->loaded = true;
    return 0;
}

int whenet_det_num_classes(whenet_det* d) { return d ? d->num_classes : 0; }

int whenet_det_precision(whenet_det* d) {
    if (!d) return fail(WHENET_EINVAL, "null detector");
    return d->precision;
}

// Unlike whenet_set_stream, no event orders the new stream after the old one: every detector entry point synchronises its
// stream before it returns, so nothing of the detector is in flight at a switch.
int whenet_det_set_stream(whenet_det* d, void* s) {
    if (!d) return fail(WHENET_EINVAL, "null detector");
    d->stream = s ? (cudaStream_t)s : d->own_stream;
    return 0;
}

}  // extern "C"

namespace {

// whenet_det_detect_u8 (yuv_layout 0), whenet_det_detect_yuv_u8 and whenet_det_detect_yuv422_u8 after their argument checks
int detect_one_size(whenet_det* d, const uint8_t* frames, int n, int H, int W, int frames_are_device, int swap_rb, int yuv_layout, float score,
                    float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    CKD(cudaSetDevice(d->device));
    // frames -> the context's input buffer (the captured graph reads a fixed address); RGB order there
    const size_t bytes = n * frame_bytes(H, W, yuv_layout);
    if (d->frames_cap < bytes) {
        CKD(cudaStreamSynchronize(d->stream));
        cudaFree(d->d_frames);
        d->d_frames = nullptr; d->frames_cap = 0;
        free_graphs(d);                         // they captured the old buffer
        if (int rc = dev_alloc(&d->d_frames, bytes, "the input frames")) return rc;
        d->frames_cap = bytes;
    }
    CKD(cudaMemcpyAsync(d->d_frames, frames, bytes, frames_are_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, d->stream));
    const OneSizeKey key(n, H, swap_rb ? W : -W, yuv_layout);      // graphs keyed on (n, H, W), the channel order and the layout
    auto it = d->graphs.find(key);
    if (it == d->graphs.end()) {
        if (d->graphs.size() >= kMaxGraphs) { CKD(cudaStreamSynchronize(d->stream)); free_graph_map(d->graphs); }
        GraphEntry e{};
        int rc = make_entry(d, n, H, W, swap_rb ? 1 : 0, yuv_layout, &e);
        if (rc) { free_entry(e); return rc; }
        it = d->graphs.emplace(key, e).first;
    }
    CKD(cudaGraphLaunch(it->second.exec, d->stream));
    d->last_n = n;
    return run_decode(d, decode_params(d, n, nullptr, H, W, score, iou, max_boxes), n, boxes, scores, classes, counts);
}

// whenet_det_detect_ragged_u8 (yuv_layout 0), whenet_det_detect_ragged_yuv_u8 and whenet_det_detect_ragged_yuv422_u8
int detect_ragged(whenet_det* d, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int swap_rb, int yuv_layout,
                  float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    // the detector is checked after every argument that can be validated without a GPU
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    if (n < 1 || n > Y::kMaxFrames) return fail(WHENET_EINVAL, "n=%d outside [1, %d]", n, Y::kMaxFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i]) return fail(WHENET_EINVAL, "frame %d is NULL", i);
        if (hw[2 * i] < 1 || hw[2 * i + 1] < 1 || hw[2 * i] > 16384 || hw[2 * i + 1] > 16384)
            return fail(WHENET_EINVAL, "frame %d: bad frame size %dx%d", i, hw[2 * i + 1], hw[2 * i]);
        if (whenet::yuv422(yuv_layout) && hw[2 * i + 1] % 2)
            return fail(WHENET_EINVAL, "frame %d: frame size %dx%d: a 4:2:2 frame has an even width", i, hw[2 * i + 1], hw[2 * i]);
        if (yuv_layout && !whenet::yuv422(yuv_layout) && (hw[2 * i] % 2 || hw[2 * i + 1] % 2))
            return fail(WHENET_EINVAL, "frame %d: frame size %dx%d: a 4:2:0 frame has even sides", i, hw[2 * i + 1], hw[2 * i]);
    }
    if (!boxes || !scores || !classes || !counts) return fail(WHENET_EINVAL, "null output pointer");
    if (!d) return fail(WHENET_EINVAL, "null detector");
    if (n > d->max_frames) return fail(WHENET_EINVAL, "n=%d outside [1, max_frames=%d]", n, d->max_frames);
    if (int rc = check_decode_args(d, score, iou, max_boxes, boxes, scores, classes, counts)) return rc;
    CKD(cudaSetDevice(d->device));
    // frames -> the context's input buffer at 256-byte aligned offsets that depend on the sizes only (the captured graph reads
    // fixed addresses)
    std::vector<size_t> off(n);
    size_t bytes = 0;
    for (int i = 0; i < n; ++i) {
        off[i] = bytes;
        bytes += align256(frame_bytes(hw[2 * i], hw[2 * i + 1], yuv_layout));
    }
    if (d->frames_cap < bytes) {
        CKD(cudaStreamSynchronize(d->stream));
        cudaFree(d->d_frames);
        d->d_frames = nullptr; d->frames_cap = 0;
        free_graphs(d);                         // they captured the old buffer
        if (int rc = dev_alloc(&d->d_frames, bytes, "the input frames")) return rc;
        d->frames_cap = bytes;
    }
    const cudaMemcpyKind kind = frames_are_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    for (int i = 0; i < n; ++i) CKD(cudaMemcpyAsync(d->d_frames + off[i], frames[i], frame_bytes(hw[2 * i], hw[2 * i + 1], yuv_layout), kind, d->stream));
    RaggedKey key(std::vector<int>(hw, hw + 2 * n), swap_rb ? 1 : 0, yuv_layout);
    auto it = d->ragged_graphs.find(key);
    if (it == d->ragged_graphs.end()) {
        if (d->ragged_graphs.size() >= kMaxGraphs) { CKD(cudaStreamSynchronize(d->stream)); free_graph_map(d->ragged_graphs); }
        GraphEntry e{};
        int rc = make_ragged_entry(d, n, hw, off, swap_rb ? 1 : 0, yuv_layout, &e);
        if (rc) { free_entry(e); return rc; }
        it = d->ragged_graphs.emplace(std::move(key), e).first;
    }
    CKD(cudaGraphLaunch(it->second.exec, d->stream));
    d->last_n = n;
    return run_decode(d, decode_params(d, n, hw, 0, 0, score, iou, max_boxes), n, boxes, scores, classes, counts);
}

}  // namespace

extern "C" {

int whenet_det_detect_u8(whenet_det* d, const uint8_t* frames, int n, int H, int W, int frames_are_device, int swap_rb, float score, float iou,
                         int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    if (!d || !frames) return fail(WHENET_EINVAL, "null detector or frames");
    if (int rc = check_frames(d, n, H, W)) return rc;
    if (int rc = check_decode_args(d, score, iou, max_boxes, boxes, scores, classes, counts)) return rc;
    return detect_one_size(d, frames, n, H, W, frames_are_device, swap_rb, 0, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_detect_yuv_u8(whenet_det* d, const uint8_t* frames, int n, int H, int W, int frames_are_device, int yuv_layout, float score,
                             float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    // the detector is checked after every argument that can be validated without a GPU
    if (int rc = check_yuv_layout(yuv_layout)) return rc;
    if (!frames) return fail(WHENET_EINVAL, "null frames");
    if (n < 1 || n > Y::kMaxFrames) return fail(WHENET_EINVAL, "n=%d outside [1, %d]", n, Y::kMaxFrames);
    if (H < 2 || W < 2 || H > 16384 || W > 16384 || H % 2 || W % 2)
        return fail(WHENET_EINVAL, "frame size %dx%d: a 4:2:0 frame has even sides in [2, 16384]", W, H);
    if (!boxes || !scores || !classes || !counts) return fail(WHENET_EINVAL, "null output pointer");
    if (!d) return fail(WHENET_EINVAL, "null detector");
    if (n > d->max_frames) return fail(WHENET_EINVAL, "n=%d outside [1, max_frames=%d]", n, d->max_frames);
    if (int rc = check_decode_args(d, score, iou, max_boxes, boxes, scores, classes, counts)) return rc;
    return detect_one_size(d, frames, n, H, W, frames_are_device, 1, yuv_layout, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_detect_ragged_u8(whenet_det* d, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int swap_rb,
                                float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    return detect_ragged(d, frames, hw, n, frames_are_device, swap_rb, 0, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_detect_ragged_yuv_u8(whenet_det* d, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int yuv_layout,
                                    float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    if (int rc = check_yuv_layout(yuv_layout)) return rc;
    return detect_ragged(d, frames, hw, n, frames_are_device, 1, yuv_layout, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_detect_yuv422_u8(whenet_det* d, const uint8_t* frames, int n, int H, int W, int frames_are_device, int yuv422_layout, float score,
                                float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    // the detector is checked after every argument that can be validated without a GPU
    if (int rc = check_yuv422_layout(yuv422_layout)) return rc;
    if (!frames) return fail(WHENET_EINVAL, "null frames");
    if (n < 1 || n > Y::kMaxFrames) return fail(WHENET_EINVAL, "n=%d outside [1, %d]", n, Y::kMaxFrames);
    if (H < 1 || W < 2 || H > 16384 || W > 16384 || W % 2)
        return fail(WHENET_EINVAL, "frame size %dx%d: a 4:2:2 frame has an even width in [2, 16384] and a height in [1, 16384]", W, H);
    if (!boxes || !scores || !classes || !counts) return fail(WHENET_EINVAL, "null output pointer");
    if (!d) return fail(WHENET_EINVAL, "null detector");
    if (n > d->max_frames) return fail(WHENET_EINVAL, "n=%d outside [1, max_frames=%d]", n, d->max_frames);
    if (int rc = check_decode_args(d, score, iou, max_boxes, boxes, scores, classes, counts)) return rc;
    return detect_one_size(d, frames, n, H, W, frames_are_device, 1, yuv422_layout, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_detect_ragged_yuv422_u8(whenet_det* d, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                       int yuv422_layout, float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes,
                                       int32_t* counts) {
    if (int rc = check_yuv422_layout(yuv422_layout)) return rc;
    return detect_ragged(d, frames, hw, n, frames_are_device, 1, yuv422_layout, score, iou, max_boxes, boxes, scores, classes, counts);
}

int whenet_det_synchronize(whenet_det* d) {
    if (!d) return fail(WHENET_EINVAL, "null detector");
    CKD(cudaSetDevice(d->device));
    CKD(cudaStreamSynchronize(d->stream));
    return 0;
}

void whenet_det_destroy(whenet_det* d) {
    if (!d) return;
    cudaSetDevice(d->device);
    if (d->stream) cudaStreamSynchronize(d->stream);
    free_graphs(d);
    free_activations(d);
    cudaFree(d->warena); cudaFree(d->warena_lo); cudaFree(d->barena); cudaFree(d->d_frames); cudaFree(d->d_canvas);
    if (d->own_stream) cudaStreamDestroy(d->own_stream);
    if (d->cap_stream) cudaStreamDestroy(d->cap_stream);
    delete d;
}

int whenet_det_debug_tap(whenet_det* d, int layer, float* out, size_t cap, size_t* n_elems) {
    if (!d) return fail(WHENET_EINVAL, "null detector");
    if (!d->loaded || d->last_n < 1) return fail(WHENET_ENOTFOUND, "no detection has run yet");
    const int nl = (int)d->table.size();
    const bool pool_tap = layer >= kPoolTap && layer < kPoolTap + nl && d->table[layer - kPoolTap].pool;
    if (!pool_tap && (layer < -1 || layer >= nl))
        return fail(WHENET_ENOTFOUND, "no tap %d (conv outputs 0..%d, -1 = letterboxed canvas, %d + i = the max-pooled input of tiny conv i)", layer,
                    nl - 1, kPoolTap);
    const LayerDev* l = pool_tap ? &d->L[layer - kPoolTap] : layer >= 0 ? &d->L[layer] : nullptr;
    const size_t n = !l ? (size_t)d->last_n * d->in_h * d->in_w * 3
                        : pool_tap ? (size_t)d->last_n * l->Hi * l->Wi * d->table[layer - kPoolTap].cin : (size_t)d->last_n * l->Ho * l->Wo * l->N;
    if (n_elems) *n_elems = n;
    if (!out) return 0;
    if (cap < n) return fail(WHENET_EINVAL, "tap %d needs %zu elements, buffer holds %zu", layer, n, cap);
    CKD(cudaSetDevice(d->device));
    CKD(cudaStreamSynchronize(d->stream));
    if (!l) {
        std::vector<uint8_t> h(n);
        CKD(cudaMemcpy(h.data(), d->d_canvas, n, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n; ++i) out[i] = h[i];
        return 0;
    }
    if (pool_tap) return to_f32_tap(l->pooled, is_fp32(d), n, out);
    return to_f32_tap(l->out, d->table[layer].head >= 0 || is_fp32(d), n, out);
}

int whenet_det_debug_conv(whenet_det* d, const float* x, const float* up, int n, int H, int W, int cin, int c_up, const float* w, const float* bias,
                          int k, int stride, int cout, int leaky, const float* resid, float* out) {
    if (!d || !x || !w || !bias || !out) return fail(WHENET_EINVAL, "null argument");
    if (n < 1 || H < 1 || W < 1 || cin < 8 || cout < 1 || cin % 8) return fail(WHENET_EINVAL, "bad shape (n=%d H=%d W=%d cin=%d cout=%d)", n, H, W, cin, cout);
    if (!((k == 1 && stride == 1) || (k == 3 && (stride == 1 || (stride == 2 && H >= 2 && W >= 2)))))
        return fail(WHENET_EINVAL, "unsupported conv k=%d stride=%d", k, stride);
    if (leaky && cout % 8) return fail(WHENET_EINVAL, "bf16 outputs need cout %% 8 == 0");
    if (!leaky && (resid || up)) return fail(WHENET_EINVAL, "the linear fp32 conv has no residual or concat source");
    if (resid && up) return fail(WHENET_EINVAL, "residual and concat source together are not a YOLOv3 layer");
    if (up && (stride != 1 || c_up < 64 || c_up % 64 || c_up >= cin || H % 2 || W % 2)) return fail(WHENET_EINVAL, "bad concat shape");
    if (!up) c_up = 0;
    CKD(cudaSetDevice(d->device));
    if (is_fp32(d)) return debug_conv32(d, x, up, n, H, W, cin, c_up, w, bias, k, stride, cout, leaky, resid, out);
    const int Ho = H / stride, Wo = W / stride;
    const size_t nx = (size_t)n * H * W * (cin - c_up), nu = (size_t)n * (H / 2) * (W / 2) * c_up, no = (size_t)n * Ho * Wo * cout;
    const int K = k * k * cin, rows = (cout + 127) / 128 * 128;
    std::vector<uint16_t> hx(nx), hu(nu), hw((size_t)rows * K, 0), hr(resid ? no : 0);
    for (size_t i = 0; i < nx; ++i) hx[i] = bf16_bits(x[i]);
    for (size_t i = 0; i < nu; ++i) hu[i] = bf16_bits(up[i]);
    for (int o = 0; o < cout; ++o)
        for (int i = 0; i < K; ++i) hw[(size_t)o * K + i] = bf16_bits(w[(size_t)i * cout + o]);
    for (size_t i = 0; i < hr.size(); ++i) hr[i] = bf16_bits(resid[i]);
    std::vector<float> hb((size_t)rows, 0.f);
    std::copy(bias, bias + cout, hb.begin());
    void *dx = nullptr, *du = nullptr, *dw = nullptr, *db = nullptr, *dr = nullptr, *dout = nullptr;
    auto cleanup = [&]() { cudaFree(dx); cudaFree(du); cudaFree(dw); cudaFree(db); cudaFree(dr); cudaFree(dout); };
    const size_t osz = no * (leaky ? 2 : 4);
    if (cudaMalloc(&dx, nx * 2) || (nu && cudaMalloc(&du, nu * 2)) || cudaMalloc(&dw, hw.size() * 2) || cudaMalloc(&db, hb.size() * 4) ||
        (resid && cudaMalloc(&dr, no * 2)) || cudaMalloc(&dout, osz)) {
        cleanup();
        return fail(WHENET_ECUDA, "out of device memory");
    }
    // on the detector's stream: a cudaMemcpy from pageable memory can return before its DMA has landed, and the
    // non-blocking stream would not wait for it
    cudaMemcpyAsync(dx, hx.data(), nx * 2, cudaMemcpyHostToDevice, d->stream);
    if (nu) cudaMemcpyAsync(du, hu.data(), nu * 2, cudaMemcpyHostToDevice, d->stream);
    cudaMemcpyAsync(dw, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice, d->stream);
    cudaMemcpyAsync(db, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice, d->stream);
    if (resid) cudaMemcpyAsync(dr, hr.data(), no * 2, cudaMemcpyHostToDevice, d->stream);
    Y::IgemmParams p{};
    p.in = (const __nv_bfloat16*)dx; p.up = (const __nv_bfloat16*)du; p.wt = (const __nv_bfloat16*)dw; p.bias = (const float*)db;
    p.resid = (const __nv_bfloat16*)dr; p.out = dout;
    p.M = n * Ho * Wo; p.Hi = H; p.Wi = W; p.Ho = Ho; p.Wo = Wo; p.Cin = cin; p.c_up = c_up; p.N = cout; p.k = k; p.stride = stride;
    const Y::IgemmPlan pl = Y::plan_igemm(Ho, Wo, cout, cin, k, d->sm_count);
    p.n_tile = pl.n_tile; p.n_stages = pl.n_stages;
    const int mode = !leaky ? Y::kLinearF32 : up ? Y::kLeakyCat : resid ? Y::kLeakyRes : Y::kLeaky;
    int rc = Y::launch_igemm(d->stream, p, mode, pl.un, pl.smem, (cout + pl.n_tile - 1) / pl.n_tile, (p.M + Y::BM - 1) / Y::BM);
    if (!rc) rc = (int)cudaStreamSynchronize(d->stream);
    if (!rc) rc = to_f32_tap(dout, !leaky, no, out) ? -1 : 0;
    cleanup();
    if (rc > 0) return fail(WHENET_ECUDA, "debug conv failed: %s", cudaGetErrorString((cudaError_t)rc));
    return rc ? WHENET_ECUDA : 0;
}

int whenet_det_debug_maxpool(whenet_det* d, const float* x, int n, int H, int W, int C, int stride, float* out) {
    if (!d || !x || !out) return fail(WHENET_EINVAL, "null argument");
    if (n < 1 || H < 1 || W < 1 || C < 8 || C % 8 || (stride != 1 && stride != 2))
        return fail(WHENET_EINVAL, "bad max-pool shape (n=%d H=%d W=%d C=%d stride=%d)", n, H, W, C, stride);
    CKD(cudaSetDevice(d->device));
    const size_t ni = (size_t)n * H * W * C, no = (size_t)n * Y::pooled(H, stride) * Y::pooled(W, stride) * C;
    if (is_fp32(d)) {                   // the host values as given, the fp32 kernel
        void *dx = nullptr, *dout = nullptr;
        if (cudaMalloc(&dx, ni * 4) || cudaMalloc(&dout, no * 4)) {
            cudaFree(dx); cudaFree(dout);
            return fail(WHENET_ECUDA, "out of device memory");
        }
        int rc = (int)cudaMemcpyAsync(dx, x, ni * 4, cudaMemcpyHostToDevice, d->stream);
        if (!rc) rc = Y::launch_maxpool32(d->stream, (const float*)dx, (float*)dout, n, H, W, C, stride);
        if (!rc) rc = (int)cudaStreamSynchronize(d->stream);
        if (!rc) rc = (int)cudaMemcpy(out, dout, no * 4, cudaMemcpyDeviceToHost);
        cudaFree(dx); cudaFree(dout);
        if (rc) return fail(WHENET_ECUDA, "debug max-pool failed: %s", cudaGetErrorString((cudaError_t)rc));
        return 0;
    }
    std::vector<uint16_t> hx(ni);
    for (size_t i = 0; i < ni; ++i) hx[i] = bf16_bits(x[i]);
    void *dx = nullptr, *dout = nullptr;
    if (cudaMalloc(&dx, ni * 2) || cudaMalloc(&dout, no * 2)) {
        cudaFree(dx); cudaFree(dout);
        return fail(WHENET_ECUDA, "out of device memory");
    }
    int rc = (int)cudaMemcpyAsync(dx, hx.data(), ni * 2, cudaMemcpyHostToDevice, d->stream);     // ordered before the kernel (see above)
    if (!rc) rc = Y::launch_maxpool(d->stream, (const __nv_bfloat16*)dx, (__nv_bfloat16*)dout, n, H, W, C, stride);
    if (!rc) rc = (int)cudaStreamSynchronize(d->stream);
    if (!rc) rc = to_f32_tap(dout, false, no, out) ? -1 : 0;
    cudaFree(dx); cudaFree(dout);
    if (rc > 0) return fail(WHENET_ECUDA, "debug max-pool failed: %s", cudaGetErrorString((cudaError_t)rc));
    return rc ? WHENET_ECUDA : 0;
}

int whenet_det_debug_decode(whenet_det* d, const float* head0, const float* head1, const float* head2, int n, int img_h, int img_w, float score,
                            float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts) {
    if (!d || !head0 || !head1 || (!head2 && !d->tiny)) return fail(WHENET_EINVAL, "null argument");
    if (int rc = check_frames(d, n, img_h, img_w)) return rc;
    if (int rc = check_decode_args(d, score, iou, max_boxes, boxes, scores, classes, counts)) return rc;
    CKD(cudaSetDevice(d->device));
    const float* hs[3] = {head0, head1, head2};
    Y::DecodeParams p = decode_params(d, n, nullptr, img_h, img_w, score, iou, max_boxes);
    const int nh = num_heads(d);
    for (int l = 0; l < nh; ++l) {
        const LayerDev& L = d->L[d->table.size() - nh + l];
        const size_t bytes = (size_t)n * L.Ho * L.Wo * L.N * 4;
        CKD(cudaMemcpyAsync(L.out, hs[l], bytes, cudaMemcpyHostToDevice, d->stream));
    }
    return run_decode(d, p, n, boxes, scores, classes, counts);
}

int whenet_det_debug_force_large_decode(whenet_det* d, int on) {
    if (!d) return fail(WHENET_EINVAL, "null detector");
    d->force_large_decode = on != 0;
    return 0;
}

}  // extern "C"
