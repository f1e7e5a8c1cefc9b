// The YOLOv3 detector's kernels (kernels_yolo.cuh) and their launchers, in a unit of their own.
#include "kernels_yolo.cuh"

namespace whenet {
namespace yolo {

int launch_letterbox(cudaStream_t s, const LetterboxPlan& lp, const uint8_t* in, uint8_t* tmp, uint8_t* out, int n, int S_h, int S_w, int swap_rb,
                     int yuv_layout) {
    const long long hx = (long long)lp.rows * lp.nw;
    const dim3 grid_h((unsigned)((hx + 255) / 256), n);
    switch (yuv_layout) {
        case 0: letterbox_h_kernel<<<grid_h, 256, 0, s>>>(in, tmp, lp.H, lp.W, lp.nw, lp.y0, lp.rows, lp.xb, lp.kx, lp.ksx, swap_rb); break;
        case kYuvNV12:
            letterbox_h_yuv_kernel<kYuvNV12><<<grid_h, 256, 0, s>>>(in, tmp, lp.H, lp.W, lp.nw, lp.y0, lp.rows, lp.xb, lp.kx, lp.ksx);
            break;
        case kYuvI420:
            letterbox_h_yuv_kernel<kYuvI420><<<grid_h, 256, 0, s>>>(in, tmp, lp.H, lp.W, lp.nw, lp.y0, lp.rows, lp.xb, lp.kx, lp.ksx);
            break;
        case kYuvYUYV:
            letterbox_h_yuv_kernel<kYuvYUYV><<<grid_h, 256, 0, s>>>(in, tmp, lp.H, lp.W, lp.nw, lp.y0, lp.rows, lp.xb, lp.kx, lp.ksx);
            break;
        case kYuvUYVY:
            letterbox_h_yuv_kernel<kYuvUYVY><<<grid_h, 256, 0, s>>>(in, tmp, lp.H, lp.W, lp.nw, lp.y0, lp.rows, lp.xb, lp.kx, lp.ksx);
            break;
        default: return (int)cudaErrorInvalidValue;
    }
    letterbox_v_kernel<<<dim3((unsigned)((S_h * S_w + 255) / 256), n), 256, 0, s>>>(tmp, out, lp.nw, lp.nh, lp.rows, S_h, S_w, lp.ox, lp.oy,
                                                                                   lp.yb, lp.ky, lp.ksy);
    return (int)cudaGetLastError();
}

int launch_letterbox_ragged(cudaStream_t s, const LetterboxFrame* plans, const char* coef, const uint8_t* in, uint8_t* tmp, uint8_t* out, int n,
                            long long max_hx, int S_h, int S_w, int swap_rb, int yuv_layout) {
    const dim3 grid_h((unsigned)((max_hx + 255) / 256), n);
    switch (yuv_layout) {
        case 0: letterbox_h_ragged_kernel<<<grid_h, 256, 0, s>>>(plans, coef, in, tmp, swap_rb); break;
        case kYuvNV12: letterbox_h_ragged_yuv_kernel<kYuvNV12><<<grid_h, 256, 0, s>>>(plans, coef, in, tmp); break;
        case kYuvI420: letterbox_h_ragged_yuv_kernel<kYuvI420><<<grid_h, 256, 0, s>>>(plans, coef, in, tmp); break;
        case kYuvYUYV: letterbox_h_ragged_yuv_kernel<kYuvYUYV><<<grid_h, 256, 0, s>>>(plans, coef, in, tmp); break;
        case kYuvUYVY: letterbox_h_ragged_yuv_kernel<kYuvUYVY><<<grid_h, 256, 0, s>>>(plans, coef, in, tmp); break;
        default: return (int)cudaErrorInvalidValue;
    }
    letterbox_v_ragged_kernel<<<dim3((unsigned)((S_h * S_w + 255) / 256), n), 256, 0, s>>>(plans, coef, tmp, out, S_h, S_w);
    return (int)cudaGetLastError();
}

template <int N>
int launch_conv0_t(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w0, const float* bias, __nv_bfloat16* out, int n, int S_h, int S_w) {
    constexpr size_t smem = 128 * 128 + N * 128 + 256 * 4 + tc::acc_tile_bytes(N) + 1024;
    cudaError_t e = cudaFuncSetAttribute(yolo_conv0_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    const long long tiles = (long long)n * S_h * S_w / 128;           // S_h * S_w is a multiple of 1024
    yolo_conv0_kernel<N><<<(unsigned)tiles, 128, smem, s>>>(img, w0, bias, out, S_h, S_w);
    return (int)cudaGetLastError();
}

int launch_conv0(cudaStream_t s, const uint8_t* img, const __nv_bfloat16* w0, const float* bias, __nv_bfloat16* out, int n, int S_h, int S_w,
                 int cout) {
    switch (cout) {
        case 16: return launch_conv0_t<16>(s, img, w0, bias, out, n, S_h, S_w);
        case 32: return launch_conv0_t<32>(s, img, w0, bias, out, n, S_h, S_w);
    }
    return (int)cudaErrorInvalidValue;
}

int launch_maxpool(cudaStream_t s, const __nv_bfloat16* in, __nv_bfloat16* out, int n, int H, int W, int C, int stride) {
    const long long threads = (long long)n * ((H + stride - 1) / stride) * ((W + stride - 1) / stride) * (C / 8);
    yolo_maxpool_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(in, out, n, H, W, C, stride);
    return (int)cudaGetLastError();
}

template <int MODE, int UN>
int launch_igemm_t(cudaStream_t s, const IgemmParams& p, size_t smem, int grid_n, int grid_m) {
    auto kfn = conv_igemm_kernel<MODE, UN>;
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    kfn<<<dim3(grid_n, grid_m), 128, smem, s>>>(p);
    return (int)cudaGetLastError();
}

template <int MODE>
int launch_igemm_m(cudaStream_t s, const IgemmParams& p, int un, size_t smem, int grid_n, int grid_m) {
    switch (un) {
        case 32: return launch_igemm_t<MODE, 32>(s, p, smem, grid_n, grid_m);
        case 64: return launch_igemm_t<MODE, 64>(s, p, smem, grid_n, grid_m);
        case 128: return launch_igemm_t<MODE, 128>(s, p, smem, grid_n, grid_m);
    }
    return (int)cudaErrorInvalidValue;
}

int launch_igemm_mode(cudaStream_t s, const IgemmParams& p, int mode, int un, size_t smem, int grid_n, int grid_m) {
    switch (mode) {
        case kLeaky: return launch_igemm_m<kLeaky>(s, p, un, smem, grid_n, grid_m);
        case kLeakyRes: return launch_igemm_m<kLeakyRes>(s, p, un, smem, grid_n, grid_m);
        case kLeakyCat: return launch_igemm_m<kLeakyCat>(s, p, un, smem, grid_n, grid_m);
        case kLinearF32: return launch_igemm_m<kLinearF32>(s, p, un, smem, grid_n, grid_m);
    }
    return (int)cudaErrorInvalidValue;
}

// More M tiles than gridDim.y holds: one launch per group of whole frames (igemm_group_frames), each with its frames' in, up,
// resid and out.  A frame's tiles and their results do not depend on the frames around it.
// grid_m: the tiles of all p.M rows.  One group (every call that fits) launches p itself.
int launch_igemm(cudaStream_t s, const IgemmParams& p, int mode, int un, size_t smem, int grid_n, int grid_m) {
    const long long hw = (long long)p.Ho * p.Wo;
    const size_t out_elem = mode == kLinearF32 ? 4 : 2;
    return for_each_frame_group((int)(p.M / hw), hw, [&](int f0, int nf) {
        if (nf * hw == p.M) return launch_igemm_mode(s, p, mode, un, smem, grid_n, grid_m);
        IgemmParams q = p;
        q.in = p.in + (size_t)f0 * p.Hi * p.Wi * (p.Cin - p.c_up);
        if (p.up) q.up = p.up + (size_t)f0 * (p.Hi / 2) * (p.Wi / 2) * p.c_up;
        if (p.resid) q.resid = p.resid + (size_t)f0 * hw * p.N;
        q.out = (char*)p.out + (size_t)f0 * hw * p.N * out_elem;
        q.M = (int)(nf * hw);
        return launch_igemm_mode(s, q, mode, un, smem, grid_n, (q.M + BM - 1) / BM);
    });
}

int launch_decode_nms(cudaStream_t s, const DecodeParams& p, int n, bool force_large, unsigned long long* keep, int* keep_count) {
    if (!force_large && !large_decode_route(p.NC)) {
        yolo_decode_nms_kernel<<<n, kNmsThreads, 0, s>>>(p);
        return (int)cudaGetLastError();
    }
    if (!keep || !keep_count || p.NC > kMaxCandidates) return (int)cudaErrorInvalidValue;
    const int alive_bytes = (p.NC + 31) / 32 * 4;
    cudaError_t e = cudaFuncSetAttribute(yolo_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLargeAliveBytes);
    if (e != cudaSuccess) return (int)e;
    yolo_decode_kernel<<<dim3((p.NC + 255) / 256, n), 256, 0, s>>>(p);
    yolo_nms_kernel<<<dim3(p.C, n), kNmsThreads, alive_bytes, s>>>(p, keep, keep_count);
    yolo_pack_kernel<<<n, 256, 0, s>>>(p, keep, keep_count);
    return (int)cudaGetLastError();
}

}  // namespace yolo
}  // namespace whenet
