// whenet_api.cu - context, weight packing, forward orchestration and the C ABI declared in include/whenet_b200.h, except the
// frame crops and overlays (frames_api.cu) and the JPEG codec (jpeg_api.cu).  See DESIGN.md for the data layout.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <vector>

#include "../../include/whenet_b200.h"
#include "api_error.h"
#include "kernels_simt.cuh"
#include "kernels_tc.cuh"
#include "kernels_fused.cuh"
#include "kernels_k2.cuh"
#include "kernels_tc32.cuh"
#include "kernels_dwse.cuh"
#include "kernels_k1x.cuh"
#include "frames_api.h"
#include "jpeg_api.h"
#include <cudaTypedefs.h>

// The fused-kernel launchers are instantiated in their own translation units (inst_k1_bf16.cu, inst_k1_f16.cu, inst_dwse.cu)
namespace whenet {
namespace fused {
#define WHENET_EXTERN_FUSED(T)                                                                            \
    extern template int launch_k1<T>(cudaStream_t, K1Params, int, int, int, int, size_t, int);            \
    extern template int launch_dw_only<T>(cudaStream_t, K1Params, size_t, int);
WHENET_EXTERN_FUSED(__nv_bfloat16)
WHENET_EXTERN_FUSED(__half)
#undef WHENET_EXTERN_FUSED
extern template int launch_dwse<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int);
extern template int launch_dwse_x<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int);
extern template int launch_dwse_spatial<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int);
extern template int launch_k1x<__nv_bfloat16>(cudaStream_t, DwSeParams, int, int, int, int, int, int, int, int);
}  // namespace fused
namespace tc {
#define WHENET_EXTERN_PW(T)                                                                                                         \
    extern template int launch_pw_tc2<T>(cudaStream_t, const T*, const void*, const float*, const float*, const T*, T*, long long, \
                                         int, int, int, bool, int, int, int, bool);                                                 \
    extern template int launch_k2<T>(cudaStream_t, const K2Params&, size_t, bool, bool, bool, int);          \
    extern template int launch_pw_tc3<T>(cudaStream_t, const T*, const void*, const float*, const float*, const T*, T*, long long, int, int, int);
WHENET_EXTERN_PW(__nv_bfloat16)
WHENET_EXTERN_PW(__half)
#undef WHENET_EXTERN_PW
}  // namespace tc
}  // namespace whenet

namespace {

using whenet::api::fail;
using whenet::api::g_err;
using whenet::Scope;

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail(WHENET_ECUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,         \
                        cudaGetErrorString(e__));                                                  \
    } while (0)

constexpr double kBnEps = 1e-3;   // efficientnet==0.0.4 BatchNormalization epsilon (SURVEY.md 8c)
constexpr int kImgElems = 224 * 224 * 3;

struct BlockCfg {
    int idx, hin, hout, cin, cexp, cout, k, s, cse, pad;
    bool skip, has_expand;
};

// EfficientNet-B0 table (kernel, stride, expand, cin, cout, repeats); the python twin is arch.py.
std::vector<BlockCfg> make_blocks() {
    static const int st[7][6] = {{3, 1, 1, 32, 16, 1}, {3, 2, 6, 16, 24, 2}, {5, 2, 6, 24, 40, 2}, {3, 2, 6, 40, 80, 3},
                                 {5, 1, 6, 80, 112, 3}, {5, 2, 6, 112, 192, 4}, {3, 1, 6, 192, 320, 1}};
    std::vector<BlockCfg> v;
    int h = 112, idx = 0;
    for (auto& r : st)
        for (int i = 0; i < r[5]; ++i) {
            BlockCfg b{};
            b.idx = ++idx;
            b.k = r[0];
            b.s = i == 0 ? r[1] : 1;
            b.cin = i == 0 ? r[3] : r[4];
            b.cout = r[4];
            b.cexp = b.cin * r[2];
            b.has_expand = r[2] != 1;
            b.hin = h;
            b.hout = (h + b.s - 1) / b.s;
            b.cse = std::max(1, b.cin / 4);
            b.skip = b.s == 1 && b.cin == b.cout;
            int total = std::max((b.hout - 1) * b.s + b.k - b.hin, 0);
            b.pad = total / 2;   // TF SAME: floor(total/2) before, the rest after
            h = b.hout;
            v.push_back(b);
        }
    return v;
}

struct BlockW {   // device pointers into the fp32 arena
    float *w_exp = nullptr, *b_exp = nullptr;     // [cin][cexp], [cexp]
    float *w_dw = nullptr, *b_dw = nullptr;       // [k*k][cexp], [cexp]
    float *w_se1t = nullptr, *b_se1 = nullptr;    // [cse][cexp], [cse]
    float *w_se2 = nullptr, *b_se2 = nullptr;     // [cse][cexp], [cexp]
    float *w_proj = nullptr, *b_proj = nullptr;   // [cexp][cout], [cout]
    void *wt_exp = nullptr, *wt_proj = nullptr;   // 16-bit [N][K] copies for the tensor-core path
    void* wt_exp_aug = nullptr;                   // 16-bit [cexp][cin+8]: 0.5*(weights | shift_hi | shift_lo) | 0... (K1)
    float *w_dw_h = nullptr, *b_dw_h = nullptr;   // 0.5 * depthwise weights / shift (K1)
    void* w_dw16 = nullptr;                       // fp16 [k*k][cexp]: 0.5 * depthwise weights / kDwScale (HFMA2 depthwise of K1 / KD)
};

struct K1Plan { bool valid = false; whenet::fused::K1Params p{}; int R = 0; int NT = 256; size_t smem = 0; };
// Which operand a cached tensor map describes.  K2: activations keyed by (K, M), weights by (N, K).  KD and K1X: keyed by
// (block, crops), or (block, 0) for weights, whose map does not depend on the batch.
enum class TmapKind {
    K2A, K2W,                  // K2's A and W
    KdE, KdDw, KdIn, KdExp,    // KD's E tiles, depthwise weights, block input and expand weights (on-chip expand)
    K1xIn, K1xExp, K1xDw,      // K1X's block input, augmented expand weights and depthwise weights
};
struct TmapKey {
    TmapKind kind; int i, j; const void* ptr;
    bool operator<(const TmapKey& o) const { return std::tie(kind, i, j, ptr) < std::tie(o.kind, o.i, o.j, o.ptr); }
};
// One pass through the net: its stream and its views of the context's workspace buffers (see pass_view)
struct Pass {
    cudaStream_t stream;
    void *A, *B, *E, *D;       // block input / output (ping-pong), expanded tensor, depthwise output
    float *partial, *gate, *pooled;
    int* se_counter;
};
struct GraphKey {
    int n, in_u8, sig;
    const void* in;
    float *ang, *log;
    bool operator==(const GraphKey& o) const { return n == o.n && in_u8 == o.in_u8 && sig == o.sig && in == o.in && ang == o.ang && log == o.log; }
};
struct GraphEntry { GraphKey key; cudaGraphExec_t exec; int launches; };
struct EvPair { cudaEvent_t a, b; int stat; };
struct Stat { std::string name; double bytes = 0, flops = 0; int launches = 0; float ms = 0; };

}  // namespace

struct whenet_ctx {
    int device = 0, max_batch = 0, precision = 0;
    int chunk = 0;          // crops per pass through the net
    int use_tc = 0;         // tensor-core kernels for the 1x1 convs
    int* h_tflag = nullptr; // mbarrier-timeout flag: mapped pinned host memory, raised by any pipelined tensor-core kernel of this context
    int* d_tflag = nullptr; // ... its device address (kernel parameter)
    int dw_variant = 1;     // 0 = one output per thread, 1 = register-blocked strips
    int pw_variant = 4;     // tensor-core 1x1 kernel: 2 = pw_tc2 (one tile per CTA, cp.async ring), 3 = K2 (persistent, TMA, warp-specialised),
                            // 4 = per layer (launch_pw)
    std::map<TmapKey, CUtensorMap> tmaps2;  // K2 tensor maps
    int pw_stage_cap = 0, pw_smem_kb = 54, pw_min_ctas = 132;    // pw_tc2 ring: max stages (0 = up to 4) and per-CTA smem budget that trades depth for co-residency
    int stem_variant = 1;   // 0 = 4 threads / pixel straight from global, 1 = smem-tiled, weights in the constant bank
    whenet::StemParams stem_params{};
    bool async_host = false;    // set by whenet_forward_u8_async for the duration of the call
    unsigned host_pass_ctr = 0; // staging slot selector, persistent across calls so consecutive calls double-buffer
    float* d_angles_slot[2] = {nullptr, nullptr};
    float* d_logits_slot[2] = {nullptr, nullptr};
    int host_chunk = 1 << 30;   // host inputs can run in passes of at most this many crops so the H2D of pass i+1 hides behind
                                // pass i; default: whole-batch passes
    int cfg_epoch = 0;      // bumped by every set_option / plan change: part of the graph cache key
    int use_graph = 0;      // replay device-resident forwards from a captured CUDA graph (small-batch latency)
    std::vector<GraphEntry> graphs;
    int use_fused = 0;      // K1: expand + depthwise in one kernel (16-bit storage only; default on for bf16/fp16)
    int fused_max_block = 16;  // blocks 2..fused_max_block use K1
    int kd_tail = 0;           // KD computes the SE gate and gates its output itself (1) or leaves both to se_gate + the project conv (0)
    int se_batch = 1;          // batches >= 64: se_gate_batch_kernel (four crops per CTA)
    int pw3 = 1;               // gated projects with H*W >= 784: pw_tc3 (a CTA walks several tiles of one crop) instead of pw_tc2
    int dw1_kd = 1;            // bf16: the stem writes fp16 and block 1's depthwise runs on KD (spatial tiles, TMA, HFMA2) instead of K1's depthwise half
    int head_batch = 1;        // batches >= 64: GAP kernel + Dense/decode for four crops per CTA
    int k1x = 0;               // bf16: the blocks with a K1X instance (K1 fed by TMA, same bits) run it where a CTA holds all chunks of its tile; 0 = K1
    int kd_from = 7;           // bf16: blocks >= kd_from whose map fits one CTA run expand GEMM (fp16 E through L2) + KD; 0 = off
    std::vector<K1Plan> k1;
    std::map<TmapKey, CUtensorMap> tmaps;   // KD and K1X tensor maps
    int sm_count = 132;
    K1Plan dw1;                // block 1 (no expand): depthwise-only instance of K1
    int dw1_fused = 1;
    cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
    cudaEvent_t ev_switch = nullptr;    // whenet_set_stream: the new stream waits for the old one's work
    bool weights_loaded = false;
    std::vector<BlockCfg> blocks;
    std::vector<BlockW> bw;
    float* d_arena = nullptr;
    void* d_arena16 = nullptr;
    size_t split_lo_bytes = 0;     // fp32 mode: byte distance from a weight's bf16 hi part to its lo part in the 16-bit arena
    std::vector<int64_t> layout;   // offsets of every packed tensor inside the two arenas (the persisted artefact's index)
    float *w_stem = nullptr, *b_stem = nullptr, *lut = nullptr;
    float *w_head = nullptr, *b_head = nullptr, *w_fct = nullptr, *b_fc = nullptr;
    void* wt_head = nullptr;
    // workspaces
    int ws_chunk = 0;
    size_t ws_io = 0, ws_ex = 0, ws_dw = 0, ws_part = 0;   // per-crop element counts of the workspace buffers
    cudaStream_t aux_stream[4] = {nullptr, nullptr, nullptr, nullptr};   // multi-stream mode: batch parts run concurrently
    cudaEvent_t ev_fork = nullptr, ev_join[4] = {nullptr, nullptr, nullptr, nullptr}, ev_half[4] = {nullptr, nullptr, nullptr, nullptr};
    int n_streams = 2;   // two half-batch streams: the late one-CTA-per-SM kernels share SMs with the other half
    void *bufA = nullptr, *bufB = nullptr, *bufE = nullptr, *bufD = nullptr;
    float *d_partial = nullptr, *d_gate = nullptr, *d_angles = nullptr, *d_logits = nullptr, *d_pooled = nullptr;
    int* d_se_counter = nullptr;   // per-crop tickets of the fused SE excite (zero between kernels)
    int se_wide = 0;               // 1024-thread SE gate CTAs also for large batches
    int se_scale_out = 1;          // ... and gate their depthwise output in place, so the project conv runs without a gate pass
    int k1_split_ctas = 120;       // small batches: split a crop's chunks over CTAs until the K1 grid has this many (measured: at 256
                                   // crops per stream the late blocks run faster unsplit, with the SE tail, than split to 296)
    int se_tail = 1;               // K1 CTAs that hold whole crops (blocks 7-16 at large batch) compute the SE gate themselves
    int se_fused = 0;              // K1's/K0's last CTA per crop computes the SE gate (no se_gate launch); off by default: the
                                   // fence + ticket tail serialises the last CTA of every crop
    void* d_in[2] = {nullptr, nullptr};
    void* h_stage = nullptr;            // pinned staging for PAGEABLE host inputs (upload_input)
    size_t h_stage_bytes = 0;
    cudaEvent_t ev_stage = nullptr;     // the last H2D copy out of h_stage
    int stage_threads = 8;              // host threads that fill the staging buffer (0 = plain cudaMemcpyAsync from the pageable buffer)
    cudaEvent_t ev_ready[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
    // frame crop and overlay buffers (frames_api.cu), created by the first call that needs one
    whenet::frames::State* frames = nullptr;
    // JPEG encoder scratch (jpeg_api.cu), created by the first encode
    whenet::jpeg::State* jpeg = nullptr;
    // taps (whenet_debug_enable_taps): 0 off, 1 first chunk of <= 8 crops on the one-stream route, 2 every chunk on the
    // untapped route.  Keyed by the canonical name ("dw%d" also holds a gated "dwg%d"); `valid`: written by the last forward.
    struct Tap { float* p = nullptr; size_t cap = 0, n = 0; bool valid = false; int forms = 0; };   // forms: 1 ungated, 2 gated rows
    int taps_mode = 0;
    std::map<std::string, Tap> taps;
    std::vector<int> tap_sel;                 // mode 2: the crops to tap, in tap-row order (empty: all)
    std::vector<int2> tap_map;                // this forward: (crop, tap row), sorted by crop
    int2* d_tap_map = nullptr; int tap_map_cap = 0;
    // profile
    bool prof_on = false;
    std::vector<EvPair> ev_used;
    std::vector<cudaEvent_t> ev_pool;
    std::vector<Stat> stats;
    std::map<std::string, int> stat_idx;
    int64_t launches = 0;
};

// ----------------------------------------------------------------------------- profiling scope
whenet::Scope::Scope(whenet_ctx* ctx, cudaStream_t stream, const char* name, double bytes, double flops) : c(ctx), s(stream) {
    c->launches++;
    if (!c->prof_on) return;
    auto it = c->stat_idx.find(name);
    int si;
    if (it == c->stat_idx.end()) {
        si = (int)c->stats.size();
        Stat s; s.name = name;
        c->stats.push_back(s);
        c->stat_idx[name] = si;
    } else si = it->second;
    c->stats[si].bytes += bytes;
    c->stats[si].flops += flops;
    c->stats[si].launches++;
    EvPair p{};
    for (cudaEvent_t* e : {&p.a, &p.b}) {
        if (!c->ev_pool.empty()) { *e = c->ev_pool.back(); c->ev_pool.pop_back(); }
        else cudaEventCreate(e);
    }
    p.stat = si;
    cudaEventRecord(p.a, s);
    c->ev_used.push_back(p);
    ev = (int)c->ev_used.size() - 1;
}

whenet::Scope::~Scope() {
    if (ev >= 0) cudaEventRecord(c->ev_used[ev].b, s);
}

namespace {

size_t esize(int precision) { return precision == WHENET_PRECISION_FP32 ? 4 : 2; }

// The stream has been synchronised: did any pipelined tensor-core kernel of this context give up on an mbarrier?  (plain host read of
// the mapped pinned flag; the flag is cleared so the context stays usable)
int check_timeout(whenet_ctx* c) {
    if (c->h_tflag && *reinterpret_cast<volatile int*>(c->h_tflag)) {
        *reinterpret_cast<volatile int*>(c->h_tflag) = 0;
        return fail(WHENET_ECUDA, "a tensor-core kernel timed out waiting on an mbarrier (results invalid)");
    }
    return 0;
}

// Before the first kernel of a tapped forward: invalidate every tap, map the tapped crops (`crops`: crop indices of the call in
// tap-row order) to their rows, and size every tap buffer for them, so that no allocation runs between launches.
int prepare_taps(whenet_ctx* c, const std::vector<int>& crops) {
    for (auto& kv : c->taps) { kv.second.valid = false; kv.second.forms = 0; }
    c->tap_map.clear();
    const int k = (int)crops.size();
    if (k == 0) return 0;
    if (k > 65535) return fail(WHENET_EINVAL, "%d tapped crops: select at most 65535 (whenet_debug_tap_crops)", k);
    for (int r = 0; r < k; ++r) c->tap_map.push_back(make_int2(crops[r], r));
    std::stable_sort(c->tap_map.begin(), c->tap_map.end(), [](const int2& a, const int2& b) { return a.x < b.x; });
    std::vector<std::pair<std::string, size_t>> per{{"stem", (size_t)112 * 112 * 32}, {"head", (size_t)49 * 1280}, {"pooled", 1280}};
    for (const BlockCfg& b : c->blocks) {
        per.push_back({"dw" + std::to_string(b.idx), (size_t)b.hout * b.hout * b.cexp});
        per.push_back({"gate" + std::to_string(b.idx), (size_t)b.cexp});
        per.push_back({"block" + std::to_string(b.idx), (size_t)b.hout * b.hout * b.cout});
    }
    CK(cudaStreamSynchronize(c->stream));                 // the previous forward's tap copies are done with the map and buffers
    for (auto& pr : per) {
        whenet_ctx::Tap& t = c->taps[pr.first];
        t.n = (size_t)k * pr.second;
        if (t.cap < t.n) {
            if (t.p) cudaFree(t.p);
            t.p = nullptr; t.cap = 0;
            CK(cudaMalloc(&t.p, t.n * sizeof(float)));
            t.cap = t.n;
        }
    }
    if (c->tap_map_cap < k) {
        if (c->d_tap_map) cudaFree(c->d_tap_map);
        c->d_tap_map = nullptr; c->tap_map_cap = 0;
        CK(cudaMalloc(&c->d_tap_map, (size_t)k * sizeof(int2)));
        c->tap_map_cap = k;
    }
    CK(cudaMemcpy(c->d_tap_map, c->tap_map.data(), (size_t)k * sizeof(int2), cudaMemcpyHostToDevice));
    return 0;
}

// Copy the tapped crops among [off, off + nb) of the call out of `src` (this chunk's tensor, per_crop elements per crop) into
// their rows of tap `name`, on the chunk's stream `s`.  `gated`: a depthwise output gated in place (read back as "dwg%d").
template <typename T>
int add_tap(whenet_ctx* c, cudaStream_t s, const std::string& name, const T* src, size_t per_crop, int off, int nb, bool gated = false) {
    auto it = c->taps.find(name);
    if (it == c->taps.end() || it->second.n != c->tap_map.size() * per_crop)
        return fail(WHENET_EINVAL, "tap %s was not prepared for this forward", name.c_str());
    const auto lo = std::lower_bound(c->tap_map.begin(), c->tap_map.end(), off, [](const int2& a, int v) { return a.x < v; });
    const auto hi = std::lower_bound(c->tap_map.begin(), c->tap_map.end(), off + nb, [](const int2& a, int v) { return a.x < v; });
    if (hi > lo) {
        whenet::tap_gather_kernel<T><<<dim3((unsigned)((per_crop + 255) / 256), (unsigned)(hi - lo)), 256, 0, s>>>(
            src, it->second.p, c->d_tap_map + (lo - c->tap_map.begin()), off, (long long)per_crop);
        CK(cudaGetLastError());
        it->second.forms |= gated ? 2 : 1;
    }
    it->second.valid = true;
    return 0;
}

// ----------------------------------------------------------------------------- workspace
void drop_graphs(whenet_ctx* c);
void free_ws(whenet_ctx* c) {
    drop_graphs(c);
    for (void** p : {&c->bufA, &c->bufB, &c->bufE, &c->bufD, &c->d_in[0], &c->d_in[1]}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    for (float** p : {&c->d_partial, &c->d_gate, &c->d_pooled}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    if (c->d_se_counter) cudaFree(c->d_se_counter);
    c->d_se_counter = nullptr;
    c->ws_chunk = 0;
}

int ensure_ws(whenet_ctx* c) {
    if (c->ws_chunk == c->chunk && c->bufA) return 0;
    free_ws(c);
    const size_t es = esize(c->precision), ch = (size_t)c->chunk;
    // per-crop element counts from the block table (SURVEY.md 8a): block io (stem out 112*112*32 is the largest),
    // expanded tensor (block 2: 112*112*96; also holds the 7*7*1280 head features), depthwise output (block 3: 56*56*144)
    size_t io = 112ull * 112 * 32, ex = 49ull * 1280, dw = 0, part = 0;
    for (const BlockCfg& b : c->blocks) {
        io = std::max(io, (size_t)b.hout * b.hout * b.cout);
        if (b.has_expand) ex = std::max(ex, (size_t)b.hin * b.hin * b.cexp);
        dw = std::max(dw, (size_t)b.hout * b.hout * b.cexp);
        part = std::max(part, (size_t)((b.hout + 7) / 8) * b.cexp);
    }
    for (const K1Plan& pl : c->k1)
        if (pl.valid) part = std::max(part, (size_t)pl.p.tiles_x * pl.p.tiles_y * pl.p.Cexp);
    // block 1 on KD (bf16): squeeze partials per 14x14 output tile
    const BlockCfg& b1 = c->blocks[0];
    if (c->precision == WHENET_PRECISION_BF16) part = std::max(part, (size_t)(b1.hin / 14) * (b1.hin / 14) * b1.cexp);
    if (c->dw1.valid) part = std::max(part, (size_t)c->dw1.p.tiles_x * c->dw1.p.tiles_y * c->dw1.p.Cexp);
    c->ws_io = io; c->ws_ex = ex; c->ws_dw = dw; c->ws_part = part;
    CK(cudaMalloc(&c->bufA, ch * io * es));
    CK(cudaMalloc(&c->bufB, ch * io * es));
    CK(cudaMalloc(&c->bufE, ch * ex * es));
    CK(cudaMalloc(&c->bufD, ch * dw * es));
    CK(cudaMalloc(&c->d_partial, ch * part * sizeof(float)));         // [crop][<= ceil(hout/8) tiles][cexp]
    CK(cudaMalloc(&c->d_gate, ch * 1152 * sizeof(float)));
    CK(cudaMalloc(&c->d_pooled, ch * 1280 * sizeof(float)));
    CK(cudaMalloc(&c->d_se_counter, ch * sizeof(int)));
    CK(cudaMemset(c->d_se_counter, 0, ch * sizeof(int)));
    for (int i = 0; i < 2; ++i) CK(cudaMalloc(&c->d_in[i], ch * kImgElems * sizeof(float)));
    c->ws_chunk = c->chunk;
    return 0;
}

// The workspace of crops off, off + 1, ... for a pass on stream s.  A two-stream forward runs each part of the batch on its own
// stream with its own crop range of every buffer.
Pass pass_view(const whenet_ctx* c, int off, cudaStream_t s) {
    const size_t es = esize(c->precision), o = (size_t)off;
    return {s,
            (char*)c->bufA + o * c->ws_io * es, (char*)c->bufB + o * c->ws_io * es,
            (char*)c->bufE + o * c->ws_ex * es, (char*)c->bufD + o * c->ws_dw * es,
            c->d_partial + o * c->ws_part, c->d_gate + o * 1152, c->d_pooled + o * 1280, c->d_se_counter + o};
}

// ----------------------------------------------------------------------------- TMA tensor maps (K2, KD, K1X)
// cuTensorMapEncodeTiled for a dense 16-bit tensor: dims[0] is contiguous and each stride is the product of the dims before it
int encode_tmap16(CUtensorMap* tm, const char* what, const void* base, bool is_bf16, std::initializer_list<long long> dims,
                  std::initializer_list<int> box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2) {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
    }
    if (!fn) return fail(WHENET_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const int rank = (int)dims.size();
    cuuint64_t dim[4], stride[4];
    cuuint32_t bx[4], estr[4] = {1, 1, 1, 1};
    for (int d = 0; d < rank; ++d) {
        dim[d] = (cuuint64_t)dims.begin()[d];
        bx[d] = (cuuint32_t)box.begin()[d];
        stride[d] = (d ? stride[d - 1] : 2) * dim[d];     // bytes between steps of dim d + 1
    }
    const CUresult r = fn(tm, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), dim,
                          stride, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        std::string dims_s, box_s;
        for (int d = 0; d < rank; ++d) { dims_s += " " + std::to_string(dim[d]); box_s += " " + std::to_string(bx[d]); }
        return fail(WHENET_ECUDA, "cuTensorMapEncodeTiled(%s, dims%s, box%s) failed: %d", what, dims_s.c_str(), box_s.c_str(), (int)r);
    }
    return 0;
}

// K-major weight matrix [rows][K] (16-bit): box = {64, box_rows} in SWIZZLE_128B rows, or {32, box_rows} in SWIZZLE_64B rows
// when row_bytes is 64
int make_tmap_w(CUtensorMap* tm, const void* base, int rows, int K, int box_rows, bool is_bf16, int row_bytes = 128) {
    return encode_tmap16(tm, "K-major matrix", base, is_bf16, {K, rows}, {row_bytes / 2, box_rows},
                         row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}
// KD operands (fp16, no swizzle): E [n][H][H][C] with box {cc, pw, pw, 1} (started at (-pad, -pad) the out-of-image part of the
// box is zero-filled = TF-SAME padding), depthwise weights [kk][C] with box {cc, kk}
int make_tmap_kd_e(CUtensorMap* tm, const void* base, int n, int H, int C, int cc, int pw) {
    return encode_tmap16(tm, "KD tile", base, false, {C, H, H, n}, {cc, pw, pw, 1}, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
int make_tmap_kd_w(CUtensorMap* tm, const void* base, int kk, int C, int cc) {
    return encode_tmap16(tm, "KD weights", base, false, {C, kk}, {cc, kk}, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// K1X's block input (bf16) [n][H][H][C]: box {row_bytes / 2, iw, iw, 1}, SWIZZLE_128B (128-byte rows) or SWIZZLE_64B (64-byte
// rows) - a halo tile lands as the K-major A operand, one row per pixel; channels >= C and pixels outside the image are
// zero-filled
int make_tmap_k1x_in(CUtensorMap* tm, const void* base, int n, int H, int C, int iw, int row_bytes) {
    return encode_tmap16(tm, "K1X input", base, true, {C, H, H, n}, {row_bytes / 2, iw, iw, 1},
                         row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Copy the map cached under `key` to *out, encoding it with make(&map) on a miss.  A cache holding more than `limit` maps is
// emptied first, so that buffers of past batch sizes do not pile up.
template <class Make>
int cached_tmap(std::map<TmapKey, CUtensorMap>& cache, size_t limit, const TmapKey& key, CUtensorMap* out, Make make) {
    if (cache.size() > limit) cache.clear();
    auto it = cache.find(key);
    if (it == cache.end()) {
        CUtensorMap tm;
        if (int rc = make(&tm)) return rc;
        it = cache.emplace(key, tm).first;
    }
    *out = it->second;
    return 0;
}

// ----------------------------------------------------------------------------- launches
// A 1x1 conv on stream s.  use_tc, variant: the kernel family (a forward passes the context's use_tc and pw_variant)
template <typename T>
int launch_pw(whenet_ctx* c, cudaStream_t s, int use_tc, int variant, const char* name, const T* A, const float* W, const void* Wt16,
              const float* bias, const float* gate, const T* resid, T* out, long long M, int K, int N, int hw, bool swish, bool out_half = false) {
    const double bytes = (double)M * (K + N + (resid ? N : 0)) * sizeof(T);
    const double flops = 2.0 * (double)M * K * N;
    Scope sc(c, s, name, bytes, flops);
    if constexpr (sizeof(T) == 2) {
        // pw_variant 4 (default): K2 for the ungated convs (expands, head, projects whose input is already gated) and for the gated
        // projects of the small maps; pw_tc2 (per-crop gate on W) for the gated projects of blocks 1-6 and for the fp16-output
        // expands that feed KD at small batches
        const bool want_k2 = variant == 3 || (variant == 4 && (gate == nullptr || hw <= 196));
        if (use_tc && Wt16 && want_k2 && !out_half) {
            whenet::tc::K2Params kp{};
            size_t smem = 0;
            // (the persistent kernel needs enough tiles to keep every SM busy for a while; below that pw_tc2's N split wins)
            if (whenet::tc::plan_k2(M, K, N, hw, gate != nullptr, c->precision == WHENET_PRECISION_BF16, &kp, &smem) &&
                (variant == 3 || kp.tiles >= 2 * c->sm_count)) {
                const bool bf16 = c->precision == WHENET_PRECISION_BF16;
                int rc = cached_tmap(c->tmaps2, 1024, {TmapKind::K2A, K, (int)M, A}, &kp.tmA,
                                     [&](CUtensorMap* tm) { return make_tmap_w(tm, A, (int)M, K, whenet::tc::BM, bf16); });
                if (!rc)
                    rc = cached_tmap(c->tmaps2, 1024, {TmapKind::K2W, N, K, Wt16}, &kp.tmW,
                                     [&](CUtensorMap* tm) { return make_tmap_w(tm, Wt16, N, K, kp.n_tile, bf16); });
                if (rc) return rc;
                kp.bias = bias; kp.gate = gate; kp.resid = resid; kp.out = out; kp.tflag = c->d_tflag;
                rc = whenet::tc::launch_k2<T>(s, kp, smem, swish, gate != nullptr, resid != nullptr, c->sm_count);
                if (rc == 0) { CK(cudaGetLastError()); return 0; }
                if (rc < 0) return fail(WHENET_ECUDA, "K2 launch failed for %s (rc=%d)", name, rc);
            }
            // shape or epilogue not covered by K2 -> pw_tc2 below
        }
        if (use_tc && Wt16 && gate && hw >= 784 && c->pw3 && !out_half && !swish) {
            // gated projects of the large maps: several tiles of one crop per CTA (pw_tc3; same bits as pw_tc2's per-crop route)
            int rc = whenet::tc::launch_pw_tc3<T>(s, A, Wt16, bias, gate, resid, out, M, K, N, hw);
            if (rc == 0) { CK(cudaGetLastError()); return 0; }
            if (rc < 0) return fail(WHENET_ECUDA, "pw_tc3 launch failed for %s (rc=%d)", name, rc);
        }
        if (use_tc && Wt16) {
            int rc = whenet::tc::launch_pw_tc2<T>(s, A, Wt16, bias, gate, resid, out, M, K, N, hw, swish, c->pw_stage_cap, c->pw_smem_kb, c->pw_min_ctas, out_half);
            if (rc == 0) { CK(cudaGetLastError()); return 0; }
            if (rc < 0) return fail(WHENET_ECUDA, "tensor-core 1x1 launch failed for %s (rc=%d)", name, rc);
            // rc > 0: shape not supported by the tensor-core kernel -> CUDA-core kernel below
        }
    }
    if constexpr (sizeof(T) == 4) {
        if (use_tc && Wt16 && c->split_lo_bytes) {
            int rc = whenet::tc::launch_pw_tc32(s, A, Wt16, (const char*)Wt16 + c->split_lo_bytes, bias, gate, resid, out, M, K, N, hw, swish);
            if (rc == 0) { CK(cudaGetLastError()); return 0; }
            if (rc < 0) return fail(WHENET_ECUDA, "split-bf16 tensor-core 1x1 launch failed for %s (rc=%d)", name, rc);
        }
    }
    if (out_half) return fail(WHENET_EINVAL, "fp16-output 1x1 conv needs the tensor-core kernel (%s)", name);
    dim3 grid((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
#define PW(SW, GA, RE) whenet::pw_conv_kernel<T, SW, GA, RE><<<grid, 256, 0, s>>>(A, W, bias, gate, resid, out, M, K, N, hw)
    if (swish && !gate && !resid) PW(true, false, false);
    else if (!swish && gate && !resid) PW(false, true, false);
    else if (!swish && gate && resid) PW(false, true, true);
    else if (!swish && !gate && !resid) PW(false, false, false);
    else if (!swish && !gate && resid) PW(false, false, true);
    else return fail(WHENET_EINVAL, "unsupported 1x1 epilogue combination");
#undef PW
    CK(cudaGetLastError());
    return 0;
}

template <typename T>
int launch_dw(whenet_ctx* c, const Pass& ps, const char* name, const BlockCfg& b, const BlockW& w, const T* in, T* out, int nb, int* tiles_out) {
    const int rows = b.hout >= 28 ? 8 : b.hout;     // output rows per CTA
    const int tiles = (b.hout + rows - 1) / rows;
    *tiles_out = tiles;
    const int cv = b.cexp / 8;
    const int py = std::max(1, 256 / cv);
    dim3 grid(tiles, nb), block(cv, py);
    const size_t smem = (size_t)py * b.cexp * sizeof(float);
    const double bytes = (double)nb * ((double)b.hin * b.hin + (double)b.hout * b.hout) * b.cexp * sizeof(T);
    const double flops = 2.0 * nb * (double)b.hout * b.hout * b.k * b.k * b.cexp;
    Scope sc(c, ps.stream, name, bytes, flops);
#define DW(KS, S) whenet::dw_conv_kernel<T, KS, S><<<grid, block, smem, ps.stream>>>(in, w.w_dw, w.b_dw, out, ps.partial, b.hin, b.hout, b.cexp, b.pad, rows)
#define DWS(KS, S, R) whenet::dw_strip_kernel<T, KS, S, R, (sizeof(T) == 2)><<<grid, block, smem, ps.stream>>>(in, w.w_dw, w.b_dw, out, ps.partial, b.hin, b.hout, b.cexp, b.pad, rows)
    if (c->dw_variant == 0) {
        if (b.k == 3 && b.s == 1) DW(3, 1);
        else if (b.k == 3 && b.s == 2) DW(3, 2);
        else if (b.k == 5 && b.s == 1) DW(5, 1);
        else if (b.k == 5 && b.s == 2) DW(5, 2);
        else return fail(WHENET_EINVAL, "unsupported depthwise config");
    } else {
        // strip length: 4 outputs where the row is long enough, 7 = a whole row at the 7x7 / 14x14 stages
        if (b.k == 3 && b.s == 1) { if (b.hout % 4 == 0) DWS(3, 1, 4); else DWS(3, 1, 7); }
        else if (b.k == 3 && b.s == 2) { if (b.hout % 4 == 0) DWS(3, 2, 4); else DWS(3, 2, 7); }
        else if (b.k == 5 && b.s == 1) { if (b.hout % 4 == 0) DWS(5, 1, 4); else DWS(5, 1, 7); }
        else if (b.k == 5 && b.s == 2) { if (b.hout % 4 == 0) DWS(5, 2, 4); else DWS(5, 2, 7); }
        else return fail(WHENET_EINVAL, "unsupported depthwise config");
    }
#undef DWS
#undef DW
    CK(cudaGetLastError());
    return 0;
}

// ----------------------------------------------------------------------------- forward: stem, block routes, SE gate, head
template <typename T, bool IN_U8>
int run_stem(whenet_ctx* c, const Pass& ps, const void* d_in, int nb, bool stem_half) {
    T* out = (T*)ps.A;
    Scope sc(c, ps.stream, "stem", (double)nb * (kImgElems * (IN_U8 ? 1.0 : 4.0) + 112.0 * 112 * 32 * sizeof(T)),
             2.0 * nb * 112.0 * 112 * 27 * 32);
    if (stem_half) {
        // block 1's depthwise is KD (HFMA2 over an fp16 tile): the stem output, read by nothing else, is written as fp16
        CK((whenet::launch_stem_tile<__half, IN_U8, true>(ps.stream, d_in, reinterpret_cast<__half*>(out), c->stem_params, c->lut, nb)));
    } else if (c->stem_variant == 0) {
        const long long total = (long long)nb * 112 * 112 * 4;
        whenet::stem_kernel<T, IN_U8><<<(unsigned)((total + 255) / 256), 256, 0, ps.stream>>>(d_in, out, c->w_stem, c->b_stem, c->lut, nb);
        CK(cudaGetLastError());
    } else {
        CK((whenet::launch_stem_tile<T, IN_U8, (sizeof(T) == 2)>(ps.stream, d_in, out, c->stem_params, c->lut, nb)));
    }
    return 0;
}

// What a block's depthwise route leaves for the SE gate and the project conv
struct DwResult {
    int tiles = 0;            // squeeze partials per crop in Pass::partial
    bool gate_done = false;   // the route computed the SE gate itself (options se_fused / se_tail)
    bool d_gated = false;     // ... and D already carries it
};

// Block 1, bf16, stem output in fp16: KD over 14x14 spatial tiles of the stem output (TMA, HFMA2)
int kd_stem_tiles(whenet_ctx* c, const Pass& ps, const __nv_bfloat16* cur, int nb, DwResult* r) {
    using T = __nv_bfloat16;
    const BlockCfg& b = c->blocks[0];
    const BlockW& w = c->bw[0];
    whenet::fused::DwSeParams p{};
    int rc = cached_tmap(c->tmaps, 512, {TmapKind::KdE, b.idx, nb, cur}, &p.tmE,
                         [&](CUtensorMap* tm) { return make_tmap_kd_e(tm, cur, nb, b.hin, b.cexp, 32, 16); });
    if (!rc)
        rc = cached_tmap(c->tmaps, 512, {TmapKind::KdDw, b.idx, 0, w.w_dw16}, &p.tmW,
                         [&](CUtensorMap* tm) { return make_tmap_kd_w(tm, w.w_dw16, 9, b.cexp, 32); });
    if (rc) return rc;
    p.b_dw = w.b_dw_h; p.tflag = c->d_tflag; p.out = ps.D; p.partial = ps.partial;
    p.C = b.cexp; p.pad = b.pad; p.Cse = b.cse; p.inv_hw = 1.0f / (float)(b.hout * b.hout);
    int split = 1;
    {
        const int n_tiles = (b.hin / 14) * (b.hin / 14);
        while (split < n_tiles && (long long)nb * split < c->k1_split_ctas) ++split;
    }
    char nm[48];
    snprintf(nm, sizeof nm, "b%02d.dw", b.idx);
    Scope sc(c, ps.stream, nm, (double)nb * 2.0 * b.hin * b.hin * b.cexp * sizeof(T), 2.0 * nb * (double)b.hout * b.hout * b.k * b.k * b.cexp);
    rc = whenet::fused::launch_dwse_spatial<T>(ps.stream, p, b.hin, nb, split);
    if (rc != 0) return fail(WHENET_ECUDA, "KD (block 1) launch failed (rc=%d)", rc);
    CK(cudaGetLastError());
    r->tiles = (b.hin / 14) * (b.hin / 14);
    return 0;
}

// Late blocks, bf16 (whole map in one CTA): KD (depthwise + SE + gating, one CTA per crop).  Small batches spread one crop's
// channel chunks over several CTAs (the gate then comes from se_gate_kernel) and read E from an expand GEMM; otherwise each CTA
// computes its crop's expand conv on chip and E never leaves the SM.
int kd_block(whenet_ctx* c, const Pass& ps, size_t i, const __nv_bfloat16* cur, int nb, bool plain_dw, DwResult* r) {
    using T = __nv_bfloat16;
    const BlockCfg& b = c->blocks[i];
    const BlockW& w = c->bw[i];
    T* E = (T*)ps.E;
    char nm[48];
    const int cc = whenet::fused::dwse_chunk(b.k, b.s, b.hin, b.cexp);
    int split = 1;
    while (split < b.cexp / cc && (long long)nb * split < c->k1_split_ctas) ++split;
    int rc = 0;
    if (split > 1) {
        snprintf(nm, sizeof nm, "b%02d.expand", b.idx);
        rc = launch_pw<T>(c, ps.stream, c->use_tc, c->pw_variant, nm, cur, w.w_exp, w.wt_exp, w.b_exp, nullptr, nullptr, E,
                          (long long)nb * b.hin * b.hin, b.cin, b.cexp, b.hin * b.hin, true, true);
        if (rc) return rc;
    }
    whenet::fused::DwSeParams p{};
    const int pw = (b.hout - 1) * b.s + b.k;
    rc = cached_tmap(c->tmaps, 512, {TmapKind::KdDw, b.idx, 0, w.w_dw16}, &p.tmW,
                     [&](CUtensorMap* tm) { return make_tmap_kd_w(tm, w.w_dw16, b.k * b.k, b.cexp, cc); });
    if (rc) return rc;
    if (split > 1) {
        rc = cached_tmap(c->tmaps, 512, {TmapKind::KdE, b.idx, nb, E}, &p.tmE,
                         [&](CUtensorMap* tm) { return make_tmap_kd_e(tm, E, nb, b.hin, b.cexp, cc, pw); });
    } else {
        // block input [nb*H*W][Cin]: box rows = one crop's pixels rounded up to a swizzle atom; expand weights [Cexp][Cin]
        rc = cached_tmap(c->tmaps, 512, {TmapKind::KdIn, b.idx, nb, cur}, &p.tmX,
                         [&](CUtensorMap* tm) { return make_tmap_w(tm, cur, nb * b.hin * b.hin, b.cin, (b.hin * b.hin + 7) / 8 * 8, true); });
        if (!rc)
            rc = cached_tmap(c->tmaps, 512, {TmapKind::KdExp, b.idx, 0, w.wt_exp}, &p.tmWx,
                             [&](CUtensorMap* tm) { return make_tmap_w(tm, w.wt_exp, b.cexp, b.cin, cc, true); });
        p.b_exp = w.b_exp;
    }
    if (rc) return rc;
    p.b_dw = w.b_dw_h; p.tflag = c->d_tflag;
    p.out = ps.D; p.partial = ps.partial;
    p.w_se1t = w.w_se1t; p.b_se1 = w.b_se1; p.w_se2 = w.w_se2; p.b_se2 = w.b_se2; p.gate = ps.gate; p.Cse = b.cse;
    p.inv_hw = 1.0f / (float)(b.hout * b.hout);
    p.C = b.cexp; p.pad = b.pad;
    if (split == 1 && c->se_tail && c->kd_tail) {
        p.se_tail = 1;
        r->gate_done = true;
        if (c->se_scale_out && !plain_dw) { p.scale_out = 1; r->d_gated = true; }
    }
    snprintf(nm, sizeof nm, "b%02d.kd", b.idx);
    if (split == 1) {
        Scope sc(c, ps.stream, nm, (double)nb * ((double)b.hin * b.hin * b.cin + (double)b.hout * b.hout * b.cexp) * sizeof(T),
                 2.0 * nb * ((double)b.hin * b.hin * b.cin * b.cexp + (double)b.hout * b.hout * b.k * b.k * b.cexp));
        rc = whenet::fused::launch_dwse_x<T>(ps.stream, p, b.k, b.s, b.hin, b.cin, nb);
        if (rc != 0) return fail(WHENET_ECUDA, "KD (on-chip expand) launch failed for block %d (rc=%d)", b.idx, rc);
        CK(cudaGetLastError());
    } else {
        Scope sc(c, ps.stream, nm, (double)nb * ((double)b.hin * b.hin + (double)b.hout * b.hout) * b.cexp * sizeof(T),
                 2.0 * nb * (double)b.hout * b.hout * b.k * b.k * b.cexp);
        rc = whenet::fused::launch_dwse<T>(ps.stream, p, b.k, b.s, b.hin, nb, split);
        if (rc != 0) return fail(WHENET_ECUDA, "KD launch failed for block %d (rc=%d)", b.idx, rc);
        CK(cudaGetLastError());
    }
    r->tiles = 1;
    return 0;
}

// Block 1, 16-bit: K1's depthwise-only instance
template <typename T>
int k1_dw_only(whenet_ctx* c, const Pass& ps, const T* cur, int nb, DwResult* r) {
    const BlockCfg& b = c->blocks[0];
    const BlockW& w = c->bw[0];
    whenet::fused::K1Params p = c->dw1.p;
    p.in = cur; p.wt_aug = nullptr; p.w_dw = w.w_dw_h; p.b_dw = w.b_dw_h; p.out = ps.D; p.partial = ps.partial; p.tflag = c->d_tflag;
    p.w_se1t = w.w_se1t; p.b_se1 = w.b_se1; p.w_se2 = w.w_se2; p.b_se2 = w.b_se2; p.gate = ps.gate; p.Cse = b.cse;
    r->gate_done = c->se_fused != 0;
    p.se_counter = r->gate_done ? ps.se_counter : nullptr;
    char nm[48];
    snprintf(nm, sizeof nm, "b%02d.dw", b.idx);
    Scope sc(c, ps.stream, nm, (double)nb * 2.0 * b.hin * b.hin * b.cexp * sizeof(T), 2.0 * nb * (double)b.hout * b.hout * b.k * b.k * b.cexp);
    int rc = whenet::fused::launch_dw_only<T>(ps.stream, p, c->dw1.smem, nb);
    if (rc != 0) return fail(WHENET_ECUDA, "depthwise-only K1 launch failed (rc=%d)", rc);
    CK(cudaGetLastError());
    r->tiles = p.tiles_x * p.tiles_y;
    return 0;
}

// K1X, bf16: the tiles and bits of K1's plan `p`, with the block input and the weights fed by TMA
int launch_k1x_block(whenet_ctx* c, const Pass& ps, size_t i, const __nv_bfloat16* cur, int nb, const whenet::fused::K1Params& p) {
    const BlockCfg& b = c->blocks[i];
    const BlockW& w = c->bw[i];
    const int rowb = whenet::fused::k1x_row_bytes(b.cin);          // A and W rows: 64 or 128 bytes
    whenet::fused::DwSeParams q{};
    int rc = cached_tmap(c->tmaps, 512, {TmapKind::K1xIn, b.idx, nb, cur}, &q.tmX,
                         [&](CUtensorMap* tm) { return make_tmap_k1x_in(tm, cur, nb, b.hin, b.cin, p.IW, rowb); });
    if (!rc)
        rc = cached_tmap(c->tmaps, 512, {TmapKind::K1xExp, b.idx, 0, w.wt_exp_aug}, &q.tmWx,
                         [&](CUtensorMap* tm) { return make_tmap_w(tm, w.wt_exp_aug, b.cexp, b.cin + 8, p.CC, true, rowb); });
    if (!rc)
        rc = cached_tmap(c->tmaps, 512, {TmapKind::K1xDw, b.idx, 0, w.w_dw16}, &q.tmW,
                         [&](CUtensorMap* tm) { return make_tmap_kd_w(tm, w.w_dw16, b.k * b.k, b.cexp, p.CC); });
    if (rc) return rc;
    q.b_dw = w.b_dw_h; q.tflag = c->d_tflag; q.out = ps.D; q.partial = ps.partial; q.C = b.cexp; q.pad = b.pad;
    rc = whenet::fused::launch_k1x<__nv_bfloat16>(ps.stream, q, b.k, b.s, b.hin, b.cin, p.TH, c->k1[i].R, p.CC, nb);
    if (rc != 0) return fail(WHENET_ECUDA, "K1X launch failed for block %d (rc=%d)", b.idx, rc);
    CK(cudaGetLastError());
    return 0;
}

// 16-bit blocks with a K1 plan: expand + depthwise in one kernel (K1, or K1X where its conditions hold)
template <typename T>
int k1_block(whenet_ctx* c, const Pass& ps, size_t i, const T* cur, int nb, bool plain_dw, DwResult* r) {
    const BlockCfg& b = c->blocks[i];
    const BlockW& w = c->bw[i];
    whenet::fused::K1Params p = c->k1[i].p;
    p.in = cur; p.wt_aug = w.wt_exp_aug; p.w_dw = w.w_dw_h; p.w_dw16 = w.w_dw16; p.b_dw = w.b_dw_h; p.out = ps.D; p.partial = ps.partial; p.tflag = c->d_tflag;
    p.w_se1t = w.w_se1t; p.b_se1 = w.b_se1; p.w_se2 = w.w_se2; p.b_se2 = w.b_se2; p.gate = ps.gate; p.Cse = b.cse;
    r->gate_done = c->se_fused && p.NB == 1;
    p.se_counter = r->gate_done ? ps.se_counter : nullptr;
    // small batches: spread one crop's chunks over several CTAs until the grid covers the SMs about twice
    {
        const long long ctas = (long long)p.tiles_x * p.tiles_y * ((nb + p.NB - 1) / p.NB);
        int split = 1;
        while (split < p.n_chunks && ctas * split < c->k1_split_ctas) ++split;
        p.chunks_per_cta = (p.n_chunks + split - 1) / split;
        // one tile per image and no chunk split: the CTA sees every pixel and channel of its crops and
        // computes their SE gate in its tail (same bits as se_gate_kernel, which is then not launched)
        if (c->se_tail && !r->gate_done && p.tiles_x * p.tiles_y == 1 && split == 1) {
            p.se_tail = 1;
            p.inv_hw = 1.0f / (float)(b.hout * b.hout);
            r->gate_done = true;
            // ... and applies it to its depthwise output (not under mode-1 taps, whose dw tap is the ungated tensor)
            if (c->se_scale_out && !plain_dw) { p.scale_out = 1; r->d_gated = true; }
        }
    }
    r->tiles = p.tiles_x * p.tiles_y;
    char nm[48];
    snprintf(nm, sizeof nm, "b%02d.k1", b.idx);
    Scope sc(c, ps.stream, nm, (double)nb * ((double)b.hin * b.hin * b.cin + (double)b.hout * b.hout * b.cexp) * sizeof(T),
             2.0 * nb * ((double)b.hin * b.hin * b.cin * b.cexp + (double)b.hout * b.hout * b.k * b.k * b.cexp));
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        // throughput batches (a CTA holds every chunk of its tile): K1X, the same tiles and bits fed by TMA
        if (c->k1x && c->use_tc && p.chunks_per_cta == p.n_chunks && !r->gate_done &&
            whenet::fused::k1x_has_instance(b.k, b.s, b.hin, b.cin, b.pad, p, c->k1[i].R))
            return launch_k1x_block(c, ps, i, cur, nb, p);
    }
    int rc = whenet::fused::launch_k1<T>(ps.stream, p, b.k, b.s, c->k1[i].R, c->k1[i].NT, c->k1[i].smem, nb);
    if (rc != 0) return fail(WHENET_ECUDA, "K1 launch failed for block %d (rc=%d)", b.idx, rc);
    CK(cudaGetLastError());
    return 0;
}

// Any block: expand GEMM (if the block has an expand conv) + stand-alone depthwise
template <typename T>
int expand_dw(whenet_ctx* c, const Pass& ps, size_t i, const T* cur, int nb, DwResult* r) {
    const BlockCfg& b = c->blocks[i];
    const BlockW& w = c->bw[i];
    char nm[48];
    const T* dw_in = cur;
    if (b.has_expand) {
        snprintf(nm, sizeof nm, "b%02d.expand", b.idx);
        int rc = launch_pw<T>(c, ps.stream, c->use_tc, c->pw_variant, nm, cur, w.w_exp, w.wt_exp, w.b_exp, nullptr, nullptr, (T*)ps.E,
                              (long long)nb * b.hin * b.hin, b.cin, b.cexp, b.hin * b.hin, true);
        if (rc) return rc;
        dw_in = (const T*)ps.E;
    }
    snprintf(nm, sizeof nm, "b%02d.dw", b.idx);
    return launch_dw<T>(c, ps, nm, b, w, dw_in, (T*)ps.D, nb, &r->tiles);
}

// Block i's expand and depthwise (D and the squeeze partials), on the first route whose conditions hold
template <typename T>
int run_dw_route(whenet_ctx* c, const Pass& ps, size_t i, const T* cur, int nb, bool stem_half, bool plain_dw, DwResult* r) {
    const BlockCfg& b = c->blocks[i];
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        if (i == 0 && stem_half) return kd_stem_tiles(c, ps, cur, nb, r);
        // late blocks (whole map in one CTA): expand GEMM + KD, or KD with the expand on chip, instead of K1
        const bool use_kd = c->use_fused && c->use_tc && c->kd_from > 0 && b.idx >= c->kd_from &&
                            b.has_expand && whenet::fused::dwse_chunk(b.k, b.s, b.hin, b.cexp) > 0;
        if (use_kd) return kd_block(c, ps, i, cur, nb, plain_dw, r);
    }
    if constexpr (sizeof(T) == 2) {
        // (block 1 has no expand conv, so this route and KD's never compete)
        if (i == 0 && c->use_fused && c->dw1_fused && c->dw1.valid) return k1_dw_only<T>(c, ps, cur, nb, r);
        if (c->use_fused && c->k1[i].valid && b.idx <= c->fused_max_block) return k1_block<T>(c, ps, i, cur, nb, plain_dw, r);
    }
    return expand_dw<T>(c, ps, i, cur, nb, r);
}

// Block b's SE gate from the squeeze partials its depthwise left (`tiles` per crop)
int se_gate(whenet_ctx* c, const Pass& ps, const BlockCfg& b, const BlockW& w, int nb, int tiles) {
    char nm[48];
    snprintf(nm, sizeof nm, "b%02d.se", b.idx);
    Scope sc(c, ps.stream, nm, (double)nb * (tiles + 1) * b.cexp * 4.0, 4.0 * nb * b.cexp * b.cse);
    const float inv_hw = 1.0f / (float)(b.hout * b.hout);
    const size_t se_smem = (b.cexp + b.cse) * sizeof(float);
    if (nb >= 64 && c->se_batch) {
        // throughput batches: four crops per CTA share every FC weight load (bit-identical gates)
        constexpr int SEB = 4;
        whenet::se_gate_batch_kernel<SEB, 512><<<(nb + SEB - 1) / SEB, 512, SEB * se_smem, ps.stream>>>(
            ps.partial, tiles, inv_hw, w.w_se1t, w.b_se1, w.w_se2, w.b_se2, ps.gate, b.cexp, b.cse, nb);
    } else if (nb < 64 || c->se_wide)     // 32 warps per crop cut the FC latency chain
        whenet::se_gate_kernel<1024><<<nb, 1024, se_smem, ps.stream>>>(
            ps.partial, tiles, inv_hw, w.w_se1t, w.b_se1, w.w_se2, w.b_se2, ps.gate, b.cexp, b.cse);
    else
        whenet::se_gate_kernel<256><<<nb, 256, se_smem, ps.stream>>>(
            ps.partial, tiles, inv_hw, w.w_se1t, w.b_se1, w.w_se2, w.b_se2, ps.gate, b.cexp, b.cse);
    CK(cudaGetLastError());
    return 0;
}

// Global average pool of the head features in E, Dense and the angle decode
template <typename T>
int head_fc_decode(whenet_ctx* c, const Pass& ps, int nb, float* d_angles, float* d_logits, bool taps) {
    const T* E = (const T*)ps.E;
    Scope sc(c, ps.stream, "head.fc_decode", (double)nb * (49.0 * 1280 * sizeof(T) + 12), 2.0 * nb * (1280.0 * 252 + 49 * 1280));
    if (nb >= 64 && c->head_batch) {
        // throughput batches: GAP kernel + Dense/decode for four crops per CTA (same bits as the one-CTA-per-crop kernel)
        constexpr int HB = 4;
        whenet::head_pool_kernel<T><<<nb, 160, 0, ps.stream>>>(E, ps.pooled);
        c->launches++;                     // two kernels under one profile scope
        auto kfn = whenet::head_fc_decode_batch_kernel<HB>;
        const size_t hsm = (size_t)HB * (1280 + 256) * sizeof(float);
        CK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsm));
        kfn<<<(nb + HB - 1) / HB, 512, hsm, ps.stream>>>(ps.pooled, c->w_fct, c->b_fc, d_angles, d_logits, nb);
    } else
        whenet::head_pool_fc_decode_kernel<T><<<nb, 256, 0, ps.stream>>>(E, nullptr, c->w_fct, c->b_fc, d_angles, d_logits,
                                                                          taps ? ps.pooled : nullptr);
    CK(cudaGetLastError());
    return 0;
}

// One pass of nb crops through the net on ps.stream, in ps's workspace
template <typename T, bool IN_U8>
int forward_chunk(whenet_ctx* c, const Pass& ps, const void* d_in, int nb, float* d_angles, float* d_logits, bool taps, int off) {
    char nm[48];
    // taps: record this chunk (crops off .. off + nb - 1 of the call).  Mode 1 also leaves the depthwise outputs ungated;
    // mode 2 changes no launch and no kernel parameter.
    const bool plain_dw = taps && c->taps_mode == 1;
    T* cur = (T*)ps.A;
    T* oth = (T*)ps.B;
    const T* D = (const T*)ps.D;
    const bool stem_half = std::is_same<T, __nv_bfloat16>::value && c->use_fused && c->use_tc && c->dw1_kd && c->stem_variant != 0 && !c->blocks.empty() &&
                           !c->blocks[0].has_expand && c->blocks[0].cexp == 32 && c->blocks[0].k == 3 && c->blocks[0].s == 1 && c->blocks[0].hin % 14 == 0;
    int rc = run_stem<T, IN_U8>(c, ps, d_in, nb, stem_half);
    if (rc) return rc;
    if (taps) {
        rc = stem_half ? add_tap<__half>(c, ps.stream, "stem", reinterpret_cast<const __half*>(cur), (size_t)112 * 112 * 32, off, nb)
                       : add_tap<T>(c, ps.stream, "stem", cur, (size_t)112 * 112 * 32, off, nb);
        if (rc) return rc;
    }
    for (size_t i = 0; i < c->blocks.size(); ++i) {
        const BlockCfg& b = c->blocks[i];
        const BlockW& w = c->bw[i];
        DwResult r;
        if ((rc = run_dw_route<T>(c, ps, i, cur, nb, stem_half, plain_dw, &r))) return rc;
        if (!r.gate_done && (rc = se_gate(c, ps, b, w, nb, r.tiles))) return rc;
        snprintf(nm, sizeof nm, "b%02d.project", b.idx);
        rc = launch_pw<T>(c, ps.stream, c->use_tc, c->pw_variant, nm, D, w.w_proj, w.wt_proj, w.b_proj, r.d_gated ? nullptr : ps.gate,
                          b.skip ? cur : nullptr, oth, (long long)nb * b.hout * b.hout, b.cexp, b.cout, b.hout * b.hout, false);
        if (rc) return rc;
        if (taps) {
            snprintf(nm, sizeof nm, "dw%d", b.idx);
            if ((rc = add_tap<T>(c, ps.stream, nm, D, (size_t)b.hout * b.hout * b.cexp, off, nb, r.d_gated))) return rc;
            snprintf(nm, sizeof nm, "gate%d", b.idx);
            if ((rc = add_tap<float>(c, ps.stream, nm, ps.gate, (size_t)b.cexp, off, nb))) return rc;
            snprintf(nm, sizeof nm, "block%d", b.idx);
            if ((rc = add_tap<T>(c, ps.stream, nm, oth, (size_t)b.hout * b.hout * b.cout, off, nb))) return rc;
        }
        std::swap(cur, oth);
    }
    rc = launch_pw<T>(c, ps.stream, c->use_tc, c->pw_variant, "head.conv", cur, c->w_head, c->wt_head, c->b_head, nullptr, nullptr,
                      (T*)ps.E, (long long)nb * 49, 320, 1280, 49, true);
    if (rc) return rc;
    if (taps && (rc = add_tap<T>(c, ps.stream, "head", (const T*)ps.E, (size_t)49 * 1280, off, nb))) return rc;
    if ((rc = head_fc_decode<T>(c, ps, nb, d_angles, d_logits, taps))) return rc;
    if (taps && (rc = add_tap<float>(c, ps.stream, "pooled", ps.pooled, (size_t)1280, off, nb))) return rc;
    return 0;
}

void drop_graphs(whenet_ctx* c) {
    for (auto& g : c->graphs) cudaGraphExecDestroy(g.exec);
    c->graphs.clear();
}


// Host -> device upload of an input batch.  Pinned (or registered) buffers go straight to cudaMemcpyAsync.  A PAGEABLE buffer - what
// the reference's callers pass to get_angle (a plain numpy array, demo.py:12-14) - would be staged by the driver through its own
// bounce buffer by one thread (~10 GB/s: 7 ms for 512 crops, longer than the whole forward); here `stage_threads` host threads copy
// 4 MB pieces into the context's pinned staging buffer and each piece starts its DMA as soon as it is staged.
// `stage_off` / `stage_total`: where this piece of the batch sits in the staging buffer and how large the buffer has to be (the halves
// of a two-stream forward use disjoint regions, so the second half is staged while the first one is still in flight); `first`:
// first upload of a forward call - the only one that has to wait for the previous call's DMA out of the staging buffer.
int upload_input(whenet_ctx* c, void* dst, const void* src, size_t bytes, cudaStream_t stream, size_t stage_off = 0, size_t stage_total = 0,
                 bool first = true) {
    constexpr size_t kPiece = 4u << 20;
    bool pageable = false;
    if (c->stage_threads > 0 && bytes >= 2 * kPiece) {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, src) == cudaSuccess) pageable = at.type == cudaMemoryTypeUnregistered;
        else cudaGetLastError();
    }
    if (!pageable) {
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
        return 0;
    }
    if (stage_total < stage_off + bytes) stage_total = stage_off + bytes;
    if (c->h_stage_bytes < stage_total) {
        if (c->h_stage) { cudaEventSynchronize(c->ev_stage); cudaFreeHost(c->h_stage); c->h_stage = nullptr; c->h_stage_bytes = 0; }
        if (cudaHostAlloc(&c->h_stage, stage_total, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));       // no pinned memory left: the plain route
            return 0;
        }
        c->h_stage_bytes = stage_total;
        if (!c->ev_stage) CK(cudaEventCreateWithFlags(&c->ev_stage, cudaEventDisableTiming));
    } else if (first) {
        CK(cudaEventSynchronize(c->ev_stage));              // the previous call's uploads have left the staging buffer
    }
    char* const stage = (char*)c->h_stage + stage_off;
    const size_t n_pieces = (bytes + kPiece - 1) / kPiece;
    std::vector<std::atomic<int>> done(n_pieces);
    for (auto& d : done) d.store(0, std::memory_order_relaxed);
    std::atomic<size_t> next{0};
    const int nt = (int)std::min<size_t>((size_t)c->stage_threads, n_pieces);
    auto work = [&]() {
        for (;;) {
            const size_t i = next.fetch_add(1, std::memory_order_relaxed);
            if (i >= n_pieces) break;
            const size_t off = i * kPiece, len = std::min(kPiece, bytes - off);
            memcpy(stage + off, (const char*)src + off, len);
            done[i].store(1, std::memory_order_release);
        }
    };
    std::vector<std::thread> pool;
    pool.reserve(nt);
    for (int t = 0; t < nt; ++t) pool.emplace_back(work);
    cudaError_t err = cudaSuccess;
    for (size_t i = 0; i < n_pieces; ++i) {
        while (!done[i].load(std::memory_order_acquire)) std::this_thread::yield();
        const size_t off = i * kPiece, len = std::min(kPiece, bytes - off);
        if (err == cudaSuccess) err = cudaMemcpyAsync((char*)dst + off, stage + off, len, cudaMemcpyHostToDevice, stream);
    }
    for (auto& th : pool) th.join();
    if (err != cudaSuccess) return fail(WHENET_ECUDA, "staged upload failed: %s", cudaGetErrorString(err));
    CK(cudaEventRecord(c->ev_stage, stream));
    return 0;
}

template <typename T, bool IN_U8>
int forward_all(whenet_ctx* c, const void* in, int n, int in_is_device, float* angles_out, float* logits_out, int out_is_device) {
    for (auto& kv : c->taps) kv.second.valid = false;     // a tap is only ever read from the forward that wrote it
    int rc = ensure_ws(c);
    if (rc) return rc;
    const size_t in_es = IN_U8 ? 1 : 4;
    const int oslot = (int)(c->host_pass_ctr & 1u);       // result buffers alternate too: two host calls may be in flight
    float* d_ang = out_is_device ? angles_out : c->d_angles_slot[oslot];
    float* d_log = logits_out ? (out_is_device ? logits_out : c->d_logits_slot[oslot]) : nullptr;
    // ---- device-resident forwards can be replayed from a captured graph (66 -> 1 launch; small-batch latency)
    const bool graphable = c->use_graph && in_is_device && out_is_device && !c->prof_on && !c->taps_mode;
    GraphKey key{n, IN_U8 ? 1 : 0, c->cfg_epoch, in, d_ang, d_log};
    if (graphable) {
        for (auto& g : c->graphs)
            if (g.key == key) {
                CK(cudaGraphLaunch(g.exec, c->stream));
                c->launches += g.launches;
                return 0;
            }
        CK(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    }
    const int64_t launches0 = c->launches;
    // ---- two-stream mode (device-resident input, one pass): the two half batches run on two streams so that the
    //      low-occupancy kernels of one half (late K1 blocks: one CTA per SM) share the SMs with kernels of the other
    const bool two_streams = c->n_streams >= 2 && !graphable && c->taps_mode != 1 && n <= c->chunk && n >= 64;
    const int step = in_is_device ? c->chunk : std::max(1, std::min(c->chunk, c->host_chunk));
    if (c->taps_mode) {
        // mode 1: the first chunk if it has at most 8 crops (one stream); mode 2: the selected crops, or all of them
        std::vector<int> crops;
        if (c->taps_mode == 2 && !c->tap_sel.empty()) {
            for (int i : c->tap_sel)
                if (i >= n) return fail(WHENET_EINVAL, "tapped crop %d outside the call's %d crops", i, n);
            crops = c->tap_sel;
        }
        else if (c->taps_mode == 2 || std::min(step, n) <= 8)
            for (int i = 0; i < (c->taps_mode == 2 ? n : std::min(step, n)); ++i) crops.push_back(i);
        if ((rc = prepare_taps(c, crops))) return rc;
    }
    if (two_streams) {
        const int parts = c->n_streams;
        const int per = (n + parts - 1) / parts;
        CK(cudaEventRecord(c->ev_fork, c->stream));
        const int slot = in_is_device ? 0 : (int)(c->host_pass_ctr++ & 1u);
        if (!in_is_device) CK(cudaStreamWaitEvent(c->copy_stream, c->ev_free[slot], 0));   // staging slot reusable
        for (int h = 0; h < parts; ++h) {
            const int off = h * per, nb = std::min(per, n - off);
            if (nb <= 0) { CK(cudaEventRecord(c->ev_join[h], c->aux_stream[h])); continue; }
            const Pass ps = pass_view(c, off, c->aux_stream[h]);
            CK(cudaStreamWaitEvent(ps.stream, c->ev_fork, 0));
            const void* d_src = (const char*)in + (size_t)off * kImgElems * in_es;
            if (!in_is_device) {
                // half h uploads on the copy stream while half h-1 (and the previous call) compute
                char* dst = (char*)c->d_in[slot] + (size_t)off * kImgElems * in_es;
                if (int urc = upload_input(c, dst, d_src, (size_t)nb * kImgElems * in_es, c->copy_stream, (size_t)off * kImgElems * in_es,
                                           (size_t)n * kImgElems * in_es, h == 0)) return urc;
                CK(cudaEventRecord(c->ev_half[h], c->copy_stream));
                CK(cudaStreamWaitEvent(ps.stream, c->ev_half[h], 0));
                d_src = dst;
            }
            rc = forward_chunk<T, IN_U8>(c, ps, d_src, nb, d_ang + (size_t)off * 3,
                                         d_log ? d_log + (size_t)off * WHENET_N_LOGITS : nullptr, c->taps_mode == 2, off);
            if (rc) return rc;
            CK(cudaEventRecord(c->ev_join[h], ps.stream));
        }
        for (int h = 0; h < parts; ++h) CK(cudaStreamWaitEvent(c->stream, c->ev_join[h], 0));
        if (!in_is_device) CK(cudaEventRecord(c->ev_free[slot], c->stream));
        if (!out_is_device) {
            CK(cudaMemcpyAsync(angles_out, d_ang, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
            if (logits_out)
                CK(cudaMemcpyAsync(logits_out, d_log, (size_t)n * WHENET_N_LOGITS * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
            if (in_is_device) c->host_pass_ctr++;
            if (!c->async_host) {
                CK(cudaStreamSynchronize(c->stream));
                return check_timeout(c);
            }
        }
        return 0;
    }
    const Pass ps = pass_view(c, 0, c->stream);
    int ci = 0;
    for (int off = 0; off < n; off += step, ++ci) {
        const int nb = std::min(step, n - off);
        const void* d_in;
        const int slot = in_is_device ? 0 : (int)(c->host_pass_ctr++ & 1u);
        if (in_is_device) {
            d_in = (const char*)in + (size_t)off * kImgElems * in_es;
        } else {
            // stage through the copy stream so chunk i+1 uploads while chunk i computes
            CK(cudaStreamWaitEvent(c->copy_stream, c->ev_free[slot], 0));
            if (int urc = upload_input(c, c->d_in[slot], (const char*)in + (size_t)off * kImgElems * in_es, (size_t)nb * kImgElems * in_es, c->copy_stream)) return urc;
            CK(cudaEventRecord(c->ev_ready[slot], c->copy_stream));
            CK(cudaStreamWaitEvent(c->stream, c->ev_ready[slot], 0));
            d_in = c->d_in[slot];
        }
        rc = forward_chunk<T, IN_U8>(c, ps, d_in, nb, d_ang + (size_t)off * 3, d_log ? d_log + (size_t)off * WHENET_N_LOGITS : nullptr,
                                     c->taps_mode == 2 || (c->taps_mode == 1 && off == 0 && nb <= 8), off);
        if (rc) {
            if (graphable) { cudaGraph_t g = nullptr; cudaStreamEndCapture(c->stream, &g); if (g) cudaGraphDestroy(g); }
            return rc;
        }
        if (!in_is_device) CK(cudaEventRecord(c->ev_free[slot], c->stream));
    }
    if (graphable) {
        cudaGraph_t graph = nullptr;
        CK(cudaStreamEndCapture(c->stream, &graph));
        cudaGraphExec_t exec = nullptr;
        cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) return fail(WHENET_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
        if (c->graphs.size() >= 8) { cudaGraphExecDestroy(c->graphs.front().exec); c->graphs.erase(c->graphs.begin()); }
        c->graphs.push_back({key, exec, (int)(c->launches - launches0)});
        CK(cudaGraphLaunch(exec, c->stream));
        return 0;
    }
    if (!out_is_device) {
        CK(cudaMemcpyAsync(angles_out, d_ang, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (logits_out)
            CK(cudaMemcpyAsync(logits_out, d_log, (size_t)n * WHENET_N_LOGITS * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (in_is_device) c->host_pass_ctr++;            // keep alternating result buffers for device-in / host-out calls too
        if (c->async_host) return 0;                     // the caller synchronises (whenet_synchronize) before reading
        CK(cudaStreamSynchronize(c->stream));
        return check_timeout(c);
    }
    return 0;
}

template <bool IN_U8>
int forward_dispatch(whenet_ctx* c, const void* in, int n, int in_is_device, float* angles_out, float* logits_out, int out_is_device) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    if (!in || !angles_out) return fail(WHENET_EINVAL, "null input or output pointer");
    if (n < 1 || n > c->max_batch) return fail(WHENET_EINVAL, "n=%d outside [1, max_batch=%d]", n, c->max_batch);
    if (!c->weights_loaded) return fail(WHENET_ENOWEIGHTS, "whenet_load_weights has not been called");
    CK(cudaSetDevice(c->device));
    switch (c->precision) {
        case WHENET_PRECISION_FP32: return forward_all<float, IN_U8>(c, in, n, in_is_device, angles_out, logits_out, out_is_device);
        case WHENET_PRECISION_BF16: return forward_all<__nv_bfloat16, IN_U8>(c, in, n, in_is_device, angles_out, logits_out, out_is_device);
        case WHENET_PRECISION_FP16: return forward_all<__half, IN_U8>(c, in, n, in_is_device, angles_out, logits_out, out_is_device);
    }
    return fail(WHENET_EINVAL, "bad precision %d", c->precision);
}

// ----------------------------------------------------------------------------- weight packing
struct TensorMap {
    std::map<std::string, const whenet_tensor*> m;
    const whenet_tensor* get(const std::string& name, std::initializer_list<int64_t> dims, std::string* err) const {
        auto it = m.find(name);
        if (it == m.end()) { *err = "missing tensor " + name; return nullptr; }
        const whenet_tensor* t = it->second;
        bool ok = t->ndim == (int)dims.size();
        int i = 0;
        for (int64_t d : dims) { if (ok && t->dims[i] != d) ok = false; ++i; }
        if (!ok || !t->data) { *err = "tensor " + name + " has the wrong shape"; return nullptr; }
        return t;
    }
};

struct BnFold { std::vector<double> scale, shift; };

bool fold_bn(const TensorMap& tm, int bn_id, int c, BnFold* out, std::string* err) {
    const std::string p = "batch_normalization_" + std::to_string(bn_id) + "/";
    const whenet_tensor *g = tm.get(p + "gamma:0", {c}, err), *b = tm.get(p + "beta:0", {c}, err),
                        *m = tm.get(p + "moving_mean:0", {c}, err), *v = tm.get(p + "moving_variance:0", {c}, err);
    if (!g || !b || !m || !v) return false;
    out->scale.resize(c);
    out->shift.resize(c);
    for (int i = 0; i < c; ++i) {
        const double s = (double)g->data[i] / std::sqrt((double)v->data[i] + kBnEps);
        out->scale[i] = s;
        out->shift[i] = (double)b->data[i] - (double)m->data[i] * s;
    }
    return true;
}

inline void whenet_host_cvt(float v, float* o) { *o = v; }
inline void whenet_host_cvt(float v, __nv_bfloat16* o) { *o = __float2bfloat16_rn(v); }
inline void whenet_host_cvt(float v, __half* o) { *o = __float2half_rn(v); }
inline float whenet_host_cvt_back(float v) { return v; }
inline float whenet_host_cvt_back(__nv_bfloat16 v) { return __bfloat162float(v); }
inline float whenet_host_cvt_back(__half v) { return __half2float(v); }

template <typename T16> T16 to16(float v);
template <> __nv_bfloat16 to16<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __half to16<__half>(float v) { return __float2half_rn(v); }

constexpr int64_t kPackMagic = 0x57484e3242323030LL;   // "WHN2B200"
constexpr int64_t kPackVersion = 4;
constexpr int kPackHeader = 14, kPackPerBlock = 16;

// Upload a packed weight image (fp32 arena + 16-bit arena + index) and point the context at it.  Shared by
// whenet_load_weights (which has just built the image from the raw Keras tensors) and whenet_import_packed (which read it
// from the persisted artefact): folding, transposition and rounding are NOT repeated on import.
int bind_packed(whenet_ctx* c, const float* arena, size_t n_f32, const uint16_t* h16, size_t n_16, const std::vector<int64_t>& L) {
    const size_t nb = c->blocks.size();
    if (L.size() != (size_t)kPackHeader + nb * kPackPerBlock || L[0] != kPackMagic || L[1] != kPackVersion)
        return fail(WHENET_ESHAPE, "packed weights: bad index (size %zu, magic/version mismatch)", L.size());
    if (L[2] != c->precision) return fail(WHENET_ESHAPE, "packed weights were exported for precision %lld, this context is %d", (long long)L[2], c->precision);
    if ((size_t)L[3] != n_f32 || (size_t)L[4] != n_16 || (size_t)L[13] != nb) return fail(WHENET_ESHAPE, "packed weights: arena sizes do not match the index");
    if (n_16 == 0) return fail(WHENET_ESHAPE, "packed weights: the 16-bit arena is missing");
    c->split_lo_bytes = c->precision == WHENET_PRECISION_FP32 ? n_16 : 0;       // fp32: [hi | lo], n_16 / 2 elements each = n_16 bytes apart
    for (size_t i = 5; i < L.size(); ++i)
        if (i != 13 && (L[i] < 0 || (size_t)L[i] >= std::max(n_f32, n_16))) return fail(WHENET_ESHAPE, "packed weights: offset %zu out of range", i);
    if (c->d_arena) { cudaFree(c->d_arena); c->d_arena = nullptr; }
    if (c->d_arena16) { cudaFree(c->d_arena16); c->d_arena16 = nullptr; }
    CK(cudaMalloc(&c->d_arena, n_f32 * sizeof(float)));
    CK(cudaMemcpy(c->d_arena, arena, n_f32 * sizeof(float), cudaMemcpyHostToDevice));
    char* base16 = nullptr;
    if (n_16) {
        CK(cudaMalloc(&c->d_arena16, n_16 * 2 + 256));
        CK(cudaMemcpy(c->d_arena16, h16, n_16 * 2, cudaMemcpyHostToDevice));
        base16 = (char*)c->d_arena16;
    }
    float* A = c->d_arena;
    c->w_stem = A + L[5]; c->b_stem = A + L[6]; c->lut = A + L[7];
    if ((size_t)L[5] + 27 * 32 > n_f32 || (size_t)L[6] + 32 > n_f32) return fail(WHENET_ESHAPE, "packed weights: stem out of range");
    memcpy(c->stem_params.w, arena + L[5], sizeof(c->stem_params.w));
    memcpy(c->stem_params.b, arena + L[6], sizeof(c->stem_params.b));
    c->w_head = A + L[8]; c->b_head = A + L[9]; c->wt_head = base16 ? base16 + L[10] * 2 : nullptr;
    c->w_fct = A + L[11]; c->b_fc = A + L[12];
    for (size_t i = 0; i < nb; ++i) {
        const int64_t* o = &L[kPackHeader + i * kPackPerBlock];
        BlockW& w = c->bw[i];
        w = BlockW{};
        if (c->blocks[i].has_expand) {
            w.w_exp = A + o[0]; w.b_exp = A + o[1];
            w.wt_exp = base16 ? base16 + o[10] * 2 : nullptr;
            w.wt_exp_aug = base16 ? base16 + o[12] * 2 : nullptr;
        }
        w.w_dw = A + o[2]; w.b_dw = A + o[3];
        w.w_se1t = A + o[4]; w.b_se1 = A + o[5]; w.w_se2 = A + o[6]; w.b_se2 = A + o[7];
        w.w_proj = A + o[8]; w.b_proj = A + o[9];
        w.wt_proj = base16 ? base16 + o[11] * 2 : nullptr;
        w.w_dw_h = A + o[13]; w.b_dw_h = A + o[14];
        w.w_dw16 = base16 ? base16 + o[15] * 2 : nullptr;
    }
    c->layout = L;
    c->weights_loaded = true;
    c->tmaps.clear();
    c->tmaps2.clear();
    drop_graphs(c);
    return 0;
}

}  // namespace

// ============================================================================= C ABI
extern "C" {

const char* whenet_last_error(void) { return g_err; }
const char* whenet_version(void) { return "whenet_b200 0.1 (sm_90a)"; }

int whenet_create(whenet_ctx** out, int device, int max_batch, int precision) {
    if (!out) return fail(WHENET_EINVAL, "out is NULL");
    *out = nullptr;
    if (max_batch < 1) return fail(WHENET_EINVAL, "max_batch must be >= 1");
    if (precision < 0 || precision > 2) return fail(WHENET_EINVAL, "precision must be 0 (fp32), 1 (bf16) or 2 (fp16)");
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(WHENET_EINVAL, "device %d not in [0,%d)", device, ndev);
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(WHENET_ECUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    whenet_ctx* c = new whenet_ctx();
    c->device = device;
    c->max_batch = max_batch;
    c->precision = precision;
    c->sm_count = prop.multiProcessorCount;
    const char* ev = getenv("WHENET_CHUNK");
    int chunk = ev ? atoi(ev) : max_batch;   // one pass over the whole batch is fastest (8.2 ms vs 13 ms per 512 crops at chunk 128)
    if (chunk < 1) chunk = max_batch;
    c->chunk = std::min(chunk, max_batch);
    c->use_tc = precision != WHENET_PRECISION_FP32;
    if (const char* e2 = getenv("WHENET_TC")) c->use_tc = atoi(e2) && precision != WHENET_PRECISION_FP32;
    c->blocks = make_blocks();
    c->bw.resize(c->blocks.size());
    c->k1.resize(c->blocks.size());
    if (precision != WHENET_PRECISION_FP32) {
        const BlockCfg& b1 = c->blocks[0];
        c->dw1.valid = !b1.has_expand && whenet::fused::plan_dw_only(b1.hin, b1.cexp, b1.k, b1.s, b1.pad, &c->dw1.p, &c->dw1.smem);
        c->dw1.R = 7;
    }
    if (precision != WHENET_PRECISION_FP32)
        for (size_t i = 0; i < c->blocks.size(); ++i) {
            const BlockCfg& b = c->blocks[i];
            if (!b.has_expand) continue;
            K1Plan& pl = c->k1[i];
            whenet::fused::K1Choice ch{};
            pl.valid = whenet::fused::plan_k1(b.hin, b.hout, b.cin, b.cexp, b.k, b.s, b.pad, precision == WHENET_PRECISION_BF16, true,
                                              &pl.p, &ch, &pl.smem);
            pl.R = ch.r;
            pl.NT = ch.nt;
        }
    c->use_fused = precision != WHENET_PRECISION_FP32;
    c->k1x = precision == WHENET_PRECISION_BF16;
    if (const char* e3 = getenv("WHENET_FUSED")) c->use_fused = atoi(e3) && precision != WHENET_PRECISION_FP32;
    CK(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    c->stream = c->own_stream;
    CK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&c->ev_switch, cudaEventDisableTiming));
    for (int i = 0; i < 4; ++i) {
        CK(cudaStreamCreateWithFlags(&c->aux_stream[i], cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->ev_half[i], cudaEventDisableTiming));
    }
    for (int i = 0; i < 2; ++i) {
        CK(cudaEventCreateWithFlags(&c->ev_ready[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->ev_free[i], cudaEventDisableTiming));
    }
    CK(cudaHostAlloc((void**)&c->h_tflag, sizeof(int), cudaHostAllocMapped));
    *c->h_tflag = 0;
    CK(cudaHostGetDevicePointer((void**)&c->d_tflag, c->h_tflag, 0));
    CK(cudaMalloc(&c->d_angles, (size_t)max_batch * 3 * sizeof(float) * 2));
    CK(cudaMalloc(&c->d_logits, (size_t)max_batch * WHENET_N_LOGITS * sizeof(float) * 2));
    for (int i = 0; i < 2; ++i) {
        c->d_angles_slot[i] = c->d_angles + (size_t)i * max_batch * 3;
        c->d_logits_slot[i] = c->d_logits + (size_t)i * max_batch * WHENET_N_LOGITS;
    }
    *out = c;
    return 0;
}

int whenet_load_weights(whenet_ctx* c, const whenet_tensor* tensors, int n_tensors) {
    if (!c || !tensors || n_tensors < 1) return fail(WHENET_EINVAL, "bad arguments");
    CK(cudaSetDevice(c->device));
    TensorMap tm;
    for (int i = 0; i < n_tensors; ++i)
        if (tensors[i].name) tm.m[tensors[i].name] = &tensors[i];
    std::string err;
    std::vector<float> arena;          // fp32 host staging; offsets recorded then rebased
    std::vector<float> arena16src;     // values for the 16-bit [N][K] tensor-core copies
    auto put = [&](const std::vector<float>& v) { size_t off = arena.size(); arena.insert(arena.end(), v.begin(), v.end());
                                                  while (arena.size() % 4) arena.push_back(0.f); return off; };
    auto put16 = [&](const std::vector<float>& v) { size_t off = arena16src.size(); arena16src.insert(arena16src.end(), v.begin(), v.end());
                                                    while (arena16src.size() % 8) arena16src.push_back(0.f); return off; };
    struct Off { size_t w_exp, b_exp, w_dw, b_dw, w_se1t, b_se1, w_se2, b_se2, w_proj, b_proj, t_exp, t_proj, t_aug, w_dw_h, b_dw_h, w_dw16; };
    std::vector<std::pair<size_t, size_t>> force_f16;     // ranges of the 16-bit arena that are fp16 whatever the storage type
    // values of the augmented expand weights; shift columns are filled after 16-bit rounding of the high part
    std::vector<std::pair<size_t, float>> shift_lo_fix;   // (index in arena16src of the hi column, full-precision shift)
    std::vector<Off> offs(c->blocks.size());
    int conv = 0, dwc = 0, bn = 0;
    auto conv_name = [&]() { return "conv2d_" + std::to_string(++conv); };

    // 1x1 conv [1,1,K,N] + BN(N) -> W'[K][N], bias[N], and the transposed [N][K] copy
    auto pack_pw = [&](int K, int N, size_t* w_off, size_t* b_off, size_t* t_off) -> bool {
        const std::string nm = conv_name();
        const whenet_tensor* t = tm.get(nm + "/kernel:0", {1, 1, K, N}, &err);
        if (!t) return false;
        if (tm.m.count(nm + "/bias:0")) { err = nm + " unexpectedly has a bias"; return false; }
        BnFold f;
        if (!fold_bn(tm, ++bn, N, &f, &err)) return false;
        std::vector<float> w((size_t)K * N), b(N), wt((size_t)K * N);
        for (int k = 0; k < K; ++k)
            for (int n = 0; n < N; ++n) {
                const float v = (float)((double)t->data[(size_t)k * N + n] * f.scale[n]);
                w[(size_t)k * N + n] = v;
                wt[(size_t)n * K + k] = v;
            }
        for (int n = 0; n < N; ++n) b[n] = (float)f.shift[n];
        *w_off = put(w);
        *b_off = put(b);
        *t_off = put16(wt);
        return true;
    };

    // ---- stem: conv2d_1 [3,3,3,32] + BN1
    size_t o_wstem, o_bstem, o_lut;
    {
        const whenet_tensor* t = tm.get(conv_name() + "/kernel:0", {3, 3, 3, 32}, &err);
        BnFold f;
        if (!t || !fold_bn(tm, ++bn, 32, &f, &err)) return fail(WHENET_ESHAPE, "%s", err.c_str());
        std::vector<float> w(27 * 32), b(32), lut(768);
        for (int i = 0; i < 27; ++i)
            for (int co = 0; co < 32; ++co) w[i * 32 + co] = (float)((double)t->data[i * 32 + co] * f.scale[co]);
        for (int co = 0; co < 32; ++co) b[co] = (float)f.shift[co];
        // reference whenet.py:23-26, evaluated in float64 like numpy, then the float32 feed cast
        const double mean[3] = {0.485, 0.456, 0.406}, sd[3] = {0.229, 0.224, 0.225};
        for (int ch = 0; ch < 3; ++ch)
            for (int v = 0; v < 256; ++v) lut[ch * 256 + v] = (float)((((double)v / 255.0) - mean[ch]) / sd[ch]);
        o_wstem = put(w); o_bstem = put(b); o_lut = put(lut);
    }
    // ---- 16 MBConv blocks
    for (size_t i = 0; i < c->blocks.size(); ++i) {
        const BlockCfg& b = c->blocks[i];
        Off& o = offs[i];
        if (b.has_expand) {
            if (!pack_pw(b.cin, b.cexp, &o.w_exp, &o.b_exp, &o.t_exp)) return fail(WHENET_ESHAPE, "%s", err.c_str());
            // [cexp][cin+8] copy for K1: the BN shift rides in two extra K columns (hi + lo 16-bit parts)
            const int ka = b.cin + 8;
            std::vector<float> aug((size_t)b.cexp * ka, 0.f);
            for (int n = 0; n < b.cexp; ++n) {
                for (int k = 0; k < b.cin; ++k) aug[(size_t)n * ka + k] = 0.5f * arena16src[o.t_exp + (size_t)n * b.cin + k];
                aug[(size_t)n * ka + b.cin] = 0.5f * arena[o.b_exp + n];
            }
            o.t_aug = put16(aug);
            for (int n = 0; n < b.cexp; ++n) shift_lo_fix.push_back({o.t_aug + (size_t)n * ka + b.cin, 0.5f * arena[o.b_exp + n]});
        }
        {
            const std::string nm = "depthwise_conv2d_" + std::to_string(++dwc);
            const whenet_tensor* t = tm.get(nm + "/depthwise_kernel:0", {b.k, b.k, b.cexp, 1}, &err);
            BnFold f;
            if (!t || !fold_bn(tm, ++bn, b.cexp, &f, &err)) return fail(WHENET_ESHAPE, "%s", err.c_str());
            std::vector<float> w((size_t)b.k * b.k * b.cexp), bb(b.cexp);
            for (int tap = 0; tap < b.k * b.k; ++tap)
                for (int ch = 0; ch < b.cexp; ++ch) w[(size_t)tap * b.cexp + ch] = (float)((double)t->data[(size_t)tap * b.cexp + ch] * f.scale[ch]);
            for (int ch = 0; ch < b.cexp; ++ch) bb[ch] = (float)f.shift[ch];
            o.w_dw = put(w); o.b_dw = put(bb);
            for (float& v : w) v *= 0.5f;
            for (float& v : bb) v *= 0.5f;
            o.w_dw_h = put(w); o.b_dw_h = put(bb);
            for (float& v : w) v *= 1.0f / whenet::fused::kDwScale;
            o.w_dw16 = put16(w);
            force_f16.push_back({o.w_dw16, w.size()});
        }
        {
            const std::string n1 = conv_name();
            const whenet_tensor *w1 = tm.get(n1 + "/kernel:0", {1, 1, b.cexp, b.cse}, &err), *b1 = tm.get(n1 + "/bias:0", {b.cse}, &err);
            const std::string n2 = conv_name();
            const whenet_tensor *w2 = tm.get(n2 + "/kernel:0", {1, 1, b.cse, b.cexp}, &err), *b2 = tm.get(n2 + "/bias:0", {b.cexp}, &err);
            if (!w1 || !b1 || !w2 || !b2) return fail(WHENET_ESHAPE, "%s", err.c_str());
            std::vector<float> w1t((size_t)b.cse * b.cexp);
            for (int ch = 0; ch < b.cexp; ++ch)
                for (int j = 0; j < b.cse; ++j) w1t[(size_t)j * b.cexp + ch] = w1->data[(size_t)ch * b.cse + j];
            o.w_se1t = put(w1t);
            o.b_se1 = put(std::vector<float>(b1->data, b1->data + b.cse));
            o.w_se2 = put(std::vector<float>(w2->data, w2->data + (size_t)b.cse * b.cexp));
            o.b_se2 = put(std::vector<float>(b2->data, b2->data + b.cexp));
        }
        if (!pack_pw(b.cexp, b.cout, &o.w_proj, &o.b_proj, &o.t_proj)) return fail(WHENET_ESHAPE, "%s", err.c_str());
    }
    // ---- head conv + BN49, three Dense heads
    size_t o_whead, o_bhead, o_thead, o_wfct, o_bfc;
    if (!pack_pw(320, 1280, &o_whead, &o_bhead, &o_thead)) return fail(WHENET_ESHAPE, "%s", err.c_str());
    {
        std::vector<float> wt((size_t)WHENET_N_LOGITS * 1280), bb(WHENET_N_LOGITS);
        const char* names[3] = {"yaw_new", "pitch_new", "roll_new"};   // reference whenet.py:11-13
        const int units[3] = {WHENET_N_YAW, WHENET_N_PITCH, WHENET_N_ROLL};
        int row = 0;
        for (int h = 0; h < 3; ++h) {
            const whenet_tensor *k = tm.get(std::string(names[h]) + "/kernel:0", {1280, units[h]}, &err),
                                *bi = tm.get(std::string(names[h]) + "/bias:0", {units[h]}, &err);
            if (!k || !bi) return fail(WHENET_ESHAPE, "%s", err.c_str());
            for (int u = 0; u < units[h]; ++u, ++row) {
                for (int ch = 0; ch < 1280; ++ch) wt[(size_t)row * 1280 + ch] = k->data[(size_t)ch * units[h] + u];
                bb[row] = bi->data[u];
            }
        }
        o_wfct = put(wt); o_bfc = put(bb);
    }
    if (conv != 65 || dwc != 16 || bn != 49)
        return fail(WHENET_ESHAPE, "consumed %d/%d/%d conv/dw/bn layers, expected 65/16/49", conv, dwc, bn);

    // ---- 16-bit arena in the storage type of this context
    std::vector<uint16_t> h16;
    if (c->precision == WHENET_PRECISION_FP32) {
        // parity mode on the tensor core (option tensor_cores=1): every K-major weight as bf16 hi | lo (x = hi + lo to 2^-18)
        const size_t n = arena16src.size();
        h16.resize(2 * n);
        for (size_t i = 0; i < n; ++i) {
            const __nv_bfloat16 hi = __float2bfloat16_rn(arena16src[i]);
            const __nv_bfloat16 lo = __float2bfloat16_rn(arena16src[i] - __bfloat162float(hi));
            memcpy(&h16[i], &hi, 2);
            memcpy(&h16[n + i], &lo, 2);
        }
    } else {
        h16.resize(arena16src.size());
        for (size_t i = 0; i < h16.size(); ++i) {
            if (c->precision == WHENET_PRECISION_BF16) { __nv_bfloat16 v = to16<__nv_bfloat16>(arena16src[i]); memcpy(&h16[i], &v, 2); }
            else { __half v = to16<__half>(arena16src[i]); memcpy(&h16[i], &v, 2); }
        }
        for (auto& rg : force_f16)
            for (size_t i = rg.first; i < rg.first + rg.second; ++i) { __half v = to16<__half>(arena16src[i]); memcpy(&h16[i], &v, 2); }
        // lo part of every K1 shift: what the 16-bit rounding of the hi part lost
        for (auto& fx : shift_lo_fix) {
            float hi;
            if (c->precision == WHENET_PRECISION_BF16) { __nv_bfloat16 v; memcpy(&v, &h16[fx.first], 2); hi = __bfloat162float(v);
                                                         __nv_bfloat16 lo = __float2bfloat16_rn(fx.second - hi); memcpy(&h16[fx.first + 1], &lo, 2); }
            else { __half v; memcpy(&v, &h16[fx.first], 2); hi = __half2float(v);
                   __half lo = __float2half_rn(fx.second - hi); memcpy(&h16[fx.first + 1], &lo, 2); }
        }
    }
    // ---- the index of the packed image: everything bind_packed needs to find a tensor again
    std::vector<int64_t> layout = {kPackMagic, kPackVersion, c->precision, (int64_t)arena.size(), (int64_t)h16.size(),
                                   (int64_t)o_wstem, (int64_t)o_bstem, (int64_t)o_lut, (int64_t)o_whead, (int64_t)o_bhead, (int64_t)o_thead,
                                   (int64_t)o_wfct, (int64_t)o_bfc, (int64_t)c->blocks.size()};
    for (size_t i = 0; i < c->blocks.size(); ++i) {
        const Off& o = offs[i];
        const bool e = c->blocks[i].has_expand;
        for (size_t v : {e ? o.w_exp : 0, e ? o.b_exp : 0, o.w_dw, o.b_dw, o.w_se1t, o.b_se1, o.w_se2, o.b_se2, o.w_proj, o.b_proj, e ? o.t_exp : 0, o.t_proj,
                         e ? o.t_aug : 0, o.w_dw_h, o.b_dw_h, o.w_dw16})
            layout.push_back((int64_t)v);
    }
    return bind_packed(c, arena.data(), arena.size(), h16.data(), h16.size(), layout);
}


int whenet_export_packed(whenet_ctx* c, float* arena_f32, uint16_t* arena_16, int64_t* index, int64_t sizes[3]) {
    if (!c || !sizes) return fail(WHENET_EINVAL, "bad arguments");
    if (!c->weights_loaded) return fail(WHENET_ENOWEIGHTS, "no weights loaded");
    sizes[0] = c->layout[3]; sizes[1] = c->layout[4]; sizes[2] = (int64_t)c->layout.size();
    CK(cudaSetDevice(c->device));
    if (arena_f32) CK(cudaMemcpy(arena_f32, c->d_arena, (size_t)sizes[0] * sizeof(float), cudaMemcpyDeviceToHost));
    if (arena_16 && sizes[1]) CK(cudaMemcpy(arena_16, c->d_arena16, (size_t)sizes[1] * 2, cudaMemcpyDeviceToHost));
    if (index) memcpy(index, c->layout.data(), c->layout.size() * sizeof(int64_t));
    return 0;
}

int whenet_import_packed(whenet_ctx* c, const float* arena_f32, int64_t n_f32, const uint16_t* arena_16, int64_t n_16, const int64_t* index, int64_t n_index) {
    if (!c || !arena_f32 || !index || n_f32 < 1 || n_16 < 0 || n_index < 1 || (n_16 > 0 && !arena_16)) return fail(WHENET_EINVAL, "bad arguments");
    CK(cudaSetDevice(c->device));
    return bind_packed(c, arena_f32, (size_t)n_f32, arena_16, (size_t)n_16, std::vector<int64_t>(index, index + n_index));
}

int whenet_set_stream(whenet_ctx* c, void* s) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    const cudaStream_t next = s ? (cudaStream_t)s : c->own_stream;
    if (next != c->stream) {
        // every call shares the workspace, the staging and result slots and the crop tables: work queued on the new stream
        // waits for everything queued on the old one, so it cannot overwrite buffers still in use and whenet_synchronize on
        // the new stream covers both
        CK(cudaSetDevice(c->device));
        CK(cudaEventRecord(c->ev_switch, c->stream));
        CK(cudaStreamWaitEvent(next, c->ev_switch, 0));
        c->stream = next;
    }
    return 0;   // captured graphs are stream independent: they are launched on whatever stream is current
}

int whenet_forward_u8(whenet_ctx* c, const uint8_t* in, int n, int in_is_device, float* angles, float* logits, int out_is_device) {
    return forward_dispatch<true>(c, in, n, in_is_device, angles, logits, out_is_device);
}

int whenet_forward_u8_async(whenet_ctx* c, const uint8_t* in_host, int n, float* angles_host, float* logits_host) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    c->async_host = true;
    const int rc = forward_dispatch<true>(c, in_host, n, 0, angles_host, logits_host, 0);
    c->async_host = false;
    return rc;
}

int whenet_forward_f32(whenet_ctx* c, const float* in, int n, int in_is_device, float* angles, float* logits, int out_is_device) {
    return forward_dispatch<false>(c, in, n, in_is_device, angles, logits, out_is_device);
}

}  // extern "C"

whenet::jpeg::Target whenet::jpeg::target(whenet_ctx* c) { return {&c->jpeg, c->device, c->stream}; }
whenet::frames::Target whenet::frames::target(whenet_ctx* c) { return {&c->frames, c->device, c->stream}; }

extern "C" {

int whenet_synchronize(whenet_ctx* c) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    return check_timeout(c);
}

void* whenet_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
        fail(WHENET_ECUDA, "cudaHostAlloc(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
void whenet_host_free(void* p) { if (p) cudaFreeHost(p); }

int whenet_debug_enable_taps(whenet_ctx* c, int enable) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    if (enable < 0 || enable > 2) return fail(WHENET_EINVAL, "tap mode %d is not 0, 1 or 2", enable);
    c->taps_mode = enable;
    return 0;
}

int whenet_debug_tap_crops(whenet_ctx* c, const int* idx, int k) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    if (k < 0 || k > 64 || (k > 0 && !idx)) return fail(WHENET_EINVAL, "select 0..64 crops (got %d)", k);
    for (int i = 0; i < k; ++i)
        if (idx[i] < 0) return fail(WHENET_EINVAL, "negative crop index %d", idx[i]);
    c->tap_sel.assign(idx, idx + k);
    return 0;
}

int whenet_debug_tap(whenet_ctx* c, const char* name, float* out, size_t cap, size_t* n_elems) {
    if (!c || !name) return fail(WHENET_EINVAL, "bad arguments");
    // "dwg%d" reads the "dw%d" buffer when the last forward gated that block's depthwise output in place
    const bool want_gated = !strncmp(name, "dwg", 3);
    const std::string key = want_gated ? "dw" + std::string(name + 3) : std::string(name);
    auto it = c->taps.find(key);
    if (it == c->taps.end() || !it->second.valid)
        return fail(WHENET_ENOTFOUND, "the last forward wrote no tap named %s (taps off, or mode 1 with more than 8 crops)", name);
    const whenet_ctx::Tap& t = it->second;
    if (!strncmp(name, "dw", 2) && t.forms == 3) return fail(WHENET_EINVAL, "tap %s holds gated and ungated crops", name);
    if (!strncmp(name, "dw", 2) && t.forms != 0 && (t.forms == 2) != want_gated)
        return fail(WHENET_ENOTFOUND, "no tap named %s: the last forward wrote %s%s", name, want_gated ? "dw" : "dwg", key.c_str() + 2);
    if (n_elems) *n_elems = t.n;
    if (!out) return 0;
    if (cap < t.n) return fail(WHENET_EINVAL, "tap %s needs %zu elements, buffer holds %zu", name, t.n, cap);
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));                 // the halves' streams (and their tap copies) joined it
    CK(cudaMemcpy(out, t.p, t.n * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"

namespace {
template <typename T>
int debug_conv_impl(whenet_ctx* c, int use_tc, const float* A, const float* W, const float* bias, const float* gate,
                    const float* resid, float* out, long long M, int K, int N, int hw, int swish) {
    std::vector<T> hA((size_t)M * K), hWt((size_t)N * K), hR(resid ? (size_t)M * N : 0), hO((size_t)M * N);
    auto cv = [](float v) { T t; whenet_host_cvt(v, &t); return t; };
    for (size_t i = 0; i < hA.size(); ++i) hA[i] = cv(A[i]);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) hWt[(size_t)n * K + k] = cv(W[(size_t)k * N + n]);
    for (size_t i = 0; i < hR.size(); ++i) hR[i] = cv(resid[i]);
    T *dA = nullptr, *dWt = nullptr, *dR = nullptr, *dO = nullptr;
    float *dW = nullptr, *dB = nullptr, *dG = nullptr;
    const long long ncrops = (M + hw - 1) / hw;
    CK(cudaMalloc(&dA, hA.size() * sizeof(T)));
    CK(cudaMalloc(&dWt, hWt.size() * sizeof(T) + 256));
    CK(cudaMalloc(&dO, hO.size() * sizeof(T)));
    CK(cudaMalloc(&dW, (size_t)K * N * 4));
    CK(cudaMalloc(&dB, (size_t)N * 4));
    CK(cudaMemcpy(dA, hA.data(), hA.size() * sizeof(T), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dWt, hWt.data(), hWt.size() * sizeof(T), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dW, W, (size_t)K * N * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dB, bias, (size_t)N * 4, cudaMemcpyHostToDevice));
    if (gate) { CK(cudaMalloc(&dG, (size_t)ncrops * K * 4)); CK(cudaMemcpy(dG, gate, (size_t)ncrops * K * 4, cudaMemcpyHostToDevice)); }
    if (resid) { CK(cudaMalloc(&dR, hR.size() * sizeof(T))); CK(cudaMemcpy(dR, hR.data(), hR.size() * sizeof(T), cudaMemcpyHostToDevice)); }
    // on the context's stream: a legacy-stream memset is not ordered against kernels of a non-blocking stream and could land on
    // rows the first tiles had already written (seen once in ~20 runs as NaN rows at the start of the output)
    CK(cudaMemsetAsync(dO, 0xFF, hO.size() * sizeof(T), c->stream));
    int rc;
    if (use_tc) {
        rc = 1;
        if constexpr (sizeof(T) == 2)
            if (use_tc == 3) {
                rc = launch_pw<T>(c, c->stream, use_tc, 3, "debug.conv1x1", dA, dW, dWt, dB, dG, dR, dO, M, K, N, hw, swish != 0);
            } else if (use_tc == 5) {
                rc = whenet::tc::launch_pw_tc3<T>(c->stream, dA, dWt, dB, dG, dR, dO, M, K, N, hw);
            } else
            rc = whenet::tc::launch_pw_tc2<T>(c->stream, dA, dWt, dB, dG, dR, dO, M, K, N, hw, swish != 0);
        uint16_t* dS = nullptr;
        if constexpr (sizeof(T) == 4) {
            // fp32 parity mode on the tensor core: bf16 hi | lo split of the K-major weights, as whenet_load_weights builds it
            std::vector<uint16_t> hs((size_t)2 * N * K);
            for (size_t i = 0; i < (size_t)N * K; ++i) {
                const float wv = whenet_host_cvt_back(hWt[i]);
                const __nv_bfloat16 hi = __float2bfloat16_rn(wv), lo = __float2bfloat16_rn(wv - __bfloat162float(hi));
                memcpy(&hs[i], &hi, 2);
                memcpy(&hs[(size_t)N * K + i], &lo, 2);
            }
            if (cudaMalloc(&dS, hs.size() * 2 + 256) == cudaSuccess) {
                cudaMemcpyAsync(dS, hs.data(), hs.size() * 2, cudaMemcpyHostToDevice, c->stream);
                cudaStreamSynchronize(c->stream);
                rc = whenet::tc::launch_pw_tc32(c->stream, (const float*)dA, dS, dS + (size_t)N * K, dB, dG, (const float*)dR, (float*)dO, M, K, N, hw, swish != 0);
                cudaStreamSynchronize(c->stream);
                cudaFree(dS);
            } else rc = -1;
        }
        if (rc == 0 && cudaGetLastError() != cudaSuccess) rc = -1;
        if (rc != 0) rc = fail(WHENET_EINVAL, "tensor-core family cannot run M=%lld K=%d N=%d (rc=%d)", M, K, N, rc);
    } else {
        rc = launch_pw<T>(c, c->stream, 0, c->pw_variant, "debug.conv1x1", dA, dW, nullptr, dB, dG, dR, dO, M, K, N, hw, swish != 0);
    }
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (rc == 0 && e != cudaSuccess) rc = fail(WHENET_ECUDA, "debug conv failed: %s", cudaGetErrorString(e));
    if (rc == 0 && use_tc) rc = check_timeout(c);
    if (rc == 0) {
        e = cudaMemcpy(hO.data(), dO, hO.size() * sizeof(T), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(WHENET_ECUDA, "copy back failed: %s", cudaGetErrorString(e));
        else for (size_t i = 0; i < hO.size(); ++i) out[i] = whenet_host_cvt_back(hO[i]);
    }
    for (void* p : {(void*)dA, (void*)dWt, (void*)dR, (void*)dO, (void*)dW, (void*)dB, (void*)dG}) if (p) cudaFree(p);
    return rc;
}
}  // namespace

extern "C" {

int whenet_debug_conv1x1(whenet_ctx* c, int use_tc, const float* A, const float* W, const float* bias, const float* gate,
                         const float* resid, float* out, int64_t M, int K, int N, int hw, int swish) {
    if (!c || !A || !W || !bias || !out || M < 1 || K < 8 || N < 8 || hw < 1) return fail(WHENET_EINVAL, "bad arguments");
    CK(cudaSetDevice(c->device));
    switch (c->precision) {
        case WHENET_PRECISION_FP32: return debug_conv_impl<float>(c, use_tc, A, W, bias, gate, resid, out, M, K, N, hw, swish);
        case WHENET_PRECISION_BF16: return debug_conv_impl<__nv_bfloat16>(c, use_tc, A, W, bias, gate, resid, out, M, K, N, hw, swish);
        case WHENET_PRECISION_FP16: return debug_conv_impl<__half>(c, use_tc, A, W, bias, gate, resid, out, M, K, N, hw, swish);
    }
    return fail(WHENET_EINVAL, "bad precision");
}

int whenet_debug_decode(whenet_ctx* c, const float* logits_host, int n, float* angles_host) {
    if (!c || !logits_host || !angles_host || n < 1) return fail(WHENET_EINVAL, "bad arguments");
    CK(cudaSetDevice(c->device));
    float *dl = nullptr, *da = nullptr;
    CK(cudaMalloc(&dl, (size_t)n * WHENET_N_LOGITS * sizeof(float)));
    if (cudaMalloc(&da, (size_t)n * 3 * sizeof(float)) != cudaSuccess) { cudaFree(dl); return fail(WHENET_ECUDA, "cudaMalloc failed"); }
    cudaMemcpyAsync(dl, logits_host, (size_t)n * WHENET_N_LOGITS * sizeof(float), cudaMemcpyHostToDevice, c->stream);
    whenet::decode_only_kernel<<<n, 96, 0, c->stream>>>(dl, da);
    cudaMemcpyAsync(angles_host, da, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, c->stream);
    const cudaError_t e = cudaStreamSynchronize(c->stream);
    cudaFree(dl); cudaFree(da);
    if (e != cudaSuccess) return fail(WHENET_ECUDA, "decode failed: %s", cudaGetErrorString(e));
    return 0;
}

int whenet_debug_raise_timeout(whenet_ctx* c) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    CK(cudaSetDevice(c->device));
    whenet::raise_flag_kernel<<<1, 1, 0, c->stream>>>(c->d_tflag);
    CK(cudaGetLastError());
    return 0;
}

int whenet_debug_set_k1_plan(whenet_ctx* c, int block, int th, int tw, int r, int cc, int nt, int nb) {
    if (!c || block < 2 || block > (int)c->blocks.size()) return fail(WHENET_EINVAL, "bad block index");
    if (c->precision == WHENET_PRECISION_FP32) return fail(WHENET_EINVAL, "K1 needs a 16-bit storage mode");
    const BlockCfg& b = c->blocks[block - 1];
    if (cc < 16 || cc > 128 || (cc & 15) || r < 1 || th < 1 || tw < 1 || (nt != 256 && nt != 512) || nb < 1 || nb > 2)
        return fail(WHENET_EINVAL, "bad plan parameters");
    if (!whenet::fused::k1_has_instance(b.k, b.s, r)) return fail(WHENET_EINVAL, "no K1 instantiation for k=%d s=%d r=%d", b.k, b.s, r);
    K1Plan pl;
    if (!whenet::fused::plan_k1_candidate(b.hin, b.hout, b.cin, b.cexp, b.k, b.s, b.pad, c->precision == WHENET_PRECISION_BF16,
                                          th, tw, r, cc, nt, nb, &pl.p, &pl.smem))
        return fail(WHENET_EINVAL, "plan %dx%d r%d cc%d nt%d nb%d does not fit block %d", th, tw, r, cc, nt, nb, block);
    pl.valid = true;
    pl.R = r;
    pl.NT = nt;
    c->k1[block - 1] = pl;
    c->cfg_epoch++;
    free_ws(c);      // the squeeze-partials buffer depends on the tile count
    return 0;
}

int whenet_profile_enable(whenet_ctx* c, int enable) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    c->prof_on = enable != 0;
    return 0;
}

int whenet_profile_read(whenet_ctx* c, whenet_kernel_stat* out, int cap) {
    if (!c) return fail(WHENET_EINVAL, "null context");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    for (auto& p : c->ev_used) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) c->stats[p.stat].ms += ms;
        c->ev_pool.push_back(p.a);
        c->ev_pool.push_back(p.b);
    }
    c->ev_used.clear();
    int n = 0;
    for (auto& s : c->stats) {
        if (out && n < cap) {
            memset(&out[n], 0, sizeof(out[n]));
            snprintf(out[n].name, sizeof(out[n].name), "%s", s.name.c_str());
            out[n].ms = s.ms; out[n].launches = s.launches; out[n].bytes = s.bytes; out[n].flops = s.flops;
        }
        ++n;
    }
    if (out) { c->stats.clear(); c->stat_idx.clear(); }
    return n;
}

int64_t whenet_launch_count(whenet_ctx* c) { return c ? c->launches : 0; }

int whenet_set_option(whenet_ctx* c, const char* key, int value) {
    if (!c || !key) return fail(WHENET_EINVAL, "bad arguments");
    drop_graphs(c);        // every option may change the launch sequence a captured graph froze
    c->cfg_epoch++;
    if (!strcmp(key, "tensor_cores")) { c->use_tc = value; return 0; }      // fp32: 1 = split-bf16 (3 MMAs per product) parity mode
    if (!strcmp(key, "streams")) { c->n_streams = value < 1 ? 1 : (value > 4 ? 4 : value); return 0; }
    if (!strcmp(key, "se_fused")) { c->se_fused = value; return 0; }
    if (!strcmp(key, "se_tail")) { c->se_tail = value; return 0; }
    if (!strcmp(key, "se_scale_out")) { c->se_scale_out = value; return 0; }
    if (!strcmp(key, "k1_split_ctas")) { c->k1_split_ctas = value; return 0; }
    if (!strcmp(key, "se_wide")) { c->se_wide = value; return 0; }
    if (!strcmp(key, "host_chunk")) { if (value < 1) return fail(WHENET_EINVAL, "host_chunk must be >= 1"); c->host_chunk = value; return 0; }
    if (!strcmp(key, "graph")) { c->use_graph = value; if (!value) drop_graphs(c); return 0; }
    if (!strcmp(key, "dw_variant")) { c->dw_variant = value; return 0; }
    if (!strcmp(key, "stem_variant")) { c->stem_variant = value; return 0; }
    if (!strcmp(key, "dw1_fused")) { c->dw1_fused = value; return 0; }
    if (!strcmp(key, "pw_variant")) { c->pw_variant = value; return 0; }
    if (!strcmp(key, "pw_stage_cap")) { c->pw_stage_cap = value; return 0; }
    if (!strcmp(key, "pw_smem_kb")) { c->pw_smem_kb = value; return 0; }
    if (!strcmp(key, "pw_min_ctas")) { c->pw_min_ctas = value; return 0; }
    if (!strcmp(key, "fused")) { c->use_fused = value && c->precision != WHENET_PRECISION_FP32; return 0; }
    if (!strcmp(key, "fused_max_block")) { c->fused_max_block = value; return 0; }
    if (!strcmp(key, "kd_from")) { c->kd_from = value; return 0; }
    if (!strcmp(key, "k1x")) { c->k1x = value && c->precision == WHENET_PRECISION_BF16; return 0; }
    if (!strcmp(key, "kd_tail")) { c->kd_tail = value; return 0; }
    if (!strcmp(key, "se_batch")) { c->se_batch = value; return 0; }
    if (!strcmp(key, "head_batch")) { c->head_batch = value; return 0; }
    if (!strcmp(key, "dw1_kd")) { c->dw1_kd = value; return 0; }
    if (!strcmp(key, "pw3")) { c->pw3 = value; return 0; }
    if (!strcmp(key, "stage_threads")) { c->stage_threads = value < 0 ? 0 : (value > 32 ? 32 : value); return 0; }
    if (!strcmp(key, "chunk")) {
        if (value < 1) return fail(WHENET_EINVAL, "chunk must be >= 1");
        c->chunk = std::min(value, c->max_batch);
        return 0;
    }
    return fail(WHENET_ENOTFOUND, "unknown option %s", key);
}

void whenet_destroy(whenet_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    drop_graphs(c);
    free_ws(c);
    whenet::frames::destroy(c->frames);
    whenet::jpeg::destroy(c->jpeg);
    for (auto& kv : c->taps) cudaFree(kv.second.p);
    if (c->d_tap_map) cudaFree(c->d_tap_map);
    for (auto& p : c->ev_used) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
    for (auto e : c->ev_pool) cudaEventDestroy(e);
    if (c->d_arena) cudaFree(c->d_arena);
    if (c->d_arena16) cudaFree(c->d_arena16);
    if (c->d_angles) cudaFree(c->d_angles);
    if (c->d_logits) cudaFree(c->d_logits);
    if (c->h_tflag) cudaFreeHost(c->h_tflag);
    for (int i = 0; i < 2; ++i) {
        if (c->ev_ready[i]) cudaEventDestroy(c->ev_ready[i]);
        if (c->ev_free[i]) cudaEventDestroy(c->ev_free[i]);
    }
    for (int i = 0; i < 4; ++i) {
        if (c->aux_stream[i]) cudaStreamDestroy(c->aux_stream[i]);
        if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]);
        if (c->ev_half[i]) cudaEventDestroy(c->ev_half[i]);
    }
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_switch) cudaEventDestroy(c->ev_switch);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (c->ev_stage) cudaEventDestroy(c->ev_stage);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    delete c;
}

}  // extern "C"
