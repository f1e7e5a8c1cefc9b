// kernels_jpeg.cuh - baseline JPEG encoding of packed BGR or gray frames, byte-identical to cv2.imencode (libjpeg-turbo: islow
// FDCT; 4:2:0, 4:2:2, 4:4:4 or gray; Annex K or optimised Huffman tables; restart intervals).  DESIGN.md sections 8.9 and 8.11;
// oracle/jpeg_oracle.py restates every step.
//
// One call encodes up to 64 frames of their own sizes with one option set.  Every kernel reads the call's frame table and works
// on global indices (transform CTAs, blocks, segments, 16-byte chunks) that it maps back to a frame, so a frame's bytes never
// depend on the other frames.  A segment is one restart interval, or the whole frame without restarts.
//   jpeg_transform_kernel<S>   colour conversion, downsampling of MCU shape S, FDCT, quantisation, zigzag: int16 per block
//   jpeg_code_kernel<2, S>     optimised tables only: per-frame symbol histograms, then jpeg_huff_build_kernel builds the tables
//   jpeg_code_kernel<0, S>     each block's Huffman bit length
//   jpeg_scan_*                exclusive int64 scan (bit offsets of blocks; chunks of segments; output bytes of chunks)
//   jpeg_seg_chunks_kernel     16-byte chunks of each segment's unstuffed stream (every segment starts on a chunk)
//   jpeg_code_kernel<1, S>     each block writes its codes at its bit offset (atomicOr into a zeroed buffer where words are shared)
//   jpeg_out_count_kernel / jpeg_stuff_kernel   0x00 after every 0xFF and RSTm between segments, each frame at its place
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace whenet {
namespace jpeg {

constexpr int kMaxFrames = 64;
constexpr int kStripBlocks = 48;       // a transform CTA codes 48 blocks of one MCU row (8 MCUs at 4:2:0)
constexpr int kTransformThreads = 256;
constexpr int kCodeThreads = 128;
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;
constexpr int kChunk = 16;             // bytes per stuffing thread; every segment's unstuffed stream starts on a chunk
constexpr int kDhtBytes = 16 + 256;    // one optimised table as DHT carries it: counts per length 1..16, then the symbols

// MCU shapes: luma sampling h x v, luma blocks row by row, then Cb and Cr; gray has one block of samples per MCU
enum Shape { k420 = 0, k422 = 1, k444 = 2, kGray = 3 };
template <int S>
struct Mcu {
    static constexpr int kShape = S;
    static constexpr int h = S <= k422 ? 2 : 1, v = S == k420 ? 2 : 1;
    static constexpr int luma = h * v, blocks = luma + (S == kGray ? 0 : 2);
    static constexpr int strip = kStripBlocks / blocks;     // MCUs per transform CTA
    static constexpr int tables = S == kGray ? 2 : 4;       // DC0 AC0 (DC1 AC1)
};

struct Frame {
    const uint8_t* src;     // H x W x 3 BGR, or H x W gray
    int H, W, mcux, mcuy, strips;   // strips: transform CTAs per MCU row
    int rst;                // MCUs per segment: the restart interval, or mcux * mcuy
    int nseg;               // segments of the frame
    int hdr;                // header bytes (SOI .. SOS) before the frame's entropy-coded data
    long long cta0;         // first transform CTA of the frame
    long long blk0;         // first block (scan order) of the frame in the call
    long long seg0;         // first segment of the frame in the call
};

struct Quant {
    uint16_t q8[2][64];     // 8 x the luma / chroma table, natural order (the islow FDCT's output is scaled by 8)
};

// The frame whose range [start, next frame's start) holds v; `field` selects the start (n <= 64: six steps).
template <long long Frame::*field>
__device__ __forceinline__ int find_frame(const Frame* __restrict__ fr, int n, long long v) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (fr[mid].*field <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__host__ __device__ constexpr int fix16(double c) { return (int)(c * 65536.0 + 0.5); }
__host__ __device__ constexpr int fix13(double c) { return (int)(c * 8192.0 + 0.5); }

__device__ __forceinline__ void load_bgr(const uint8_t* __restrict__ p, int& b, int& g, int& r) {
    b = __ldg(p); g = __ldg(p + 1); r = __ldg(p + 2);
}
__device__ __forceinline__ int rgb_y(int r, int g, int b) {
    return (fix16(0.29900) * r + fix16(0.58700) * g + fix16(0.11400) * b + (1 << 15)) >> 16;
}
__device__ __forceinline__ int rgb_cb(int r, int g, int b) {
    return (-fix16(0.16874) * r - fix16(0.33126) * g + fix16(0.5) * b + (128 << 16) + (1 << 15) - 1) >> 16;
}
__device__ __forceinline__ int rgb_cr(int r, int g, int b) {
    return (fix16(0.5) * r - fix16(0.41869) * g - fix16(0.08131) * b + (128 << 16) + (1 << 15) - 1) >> 16;
}

// One 8-point pass of libjpeg's islow FDCT (CONST_BITS 13, PASS1_BITS 2) over d[0], d[s], ..., d[7s], in place.
template <bool kRows>
__device__ __forceinline__ void fdct_pass(int* d, int s) {
    constexpr int kShift = kRows ? 13 - 2 : 13 + 2;
    auto descale = [](int x, int n) { return (x + (1 << (n - 1))) >> n; };
    const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
    const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    if (kRows) { d[0] = (t10 + t11) * 4; d[4 * s] = (t10 - t11) * 4; }
    else { d[0] = descale(t10 + t11, 2); d[4 * s] = descale(t10 - t11, 2); }
    const int z1e = (t12 + t13) * fix13(0.541196100);
    d[2 * s] = descale(z1e + t13 * fix13(0.765366865), kShift);
    d[6 * s] = descale(z1e - t12 * fix13(1.847759065), kShift);
    const int z5 = (t4 + t6 + t5 + t7) * fix13(1.175875602);
    const int z1 = -(t4 + t7) * fix13(0.899976223), z2 = -(t5 + t6) * fix13(2.562915447);
    const int z3 = -(t4 + t6) * fix13(1.961570560) + z5, z4 = -(t5 + t7) * fix13(0.390180644) + z5;
    d[7 * s] = descale(t4 * fix13(0.298631336) + z1 + z3, kShift);
    d[5 * s] = descale(t5 * fix13(2.053119869) + z2 + z4, kShift);
    d[3 * s] = descale(t6 * fix13(3.072711026) + z2 + z3, kShift);
    d[s] = descale(t7 * fix13(1.501321110) + z1 + z4, kShift);
}

__device__ __forceinline__ int quantise(int v, int q8) {
    const int a = ((v < 0 ? -v : v) + (q8 >> 1)) / q8;
    return v < 0 ? -a : a;
}

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

constexpr int kBlkStride = 72;   // 8 rows of 9 ints: row and column passes are both free of bank conflicts

// One CTA per strip of Mcu<S>::strip MCUs of one MCU row.  Writes the strip's blocks as zigzag int16 at
// coef[(blk0 + blocks * mcu + b) * 64].  Luma (and gray) replicates the last row and column to the block boundary.  Chroma
// replicates the last column to h x its block boundary and the last row to a multiple of v, sums the h x v pixels with a bias
// that alternates along a row (4:2:0: 1, 2; 4:2:2: 0, 1), shifts, and then replicates the last downsampled row.  A luma block
// past the image (a dummy block, only where an MCU has two luma blocks along an axis) gets AC 0 and the DC of the block before
// it in the MCU.  Quantisation takes qt.q8[0] for luma and qt.q8[1] for chroma.
template <int S>
__global__ void __launch_bounds__(kTransformThreads) jpeg_transform_kernel(const Frame* __restrict__ frames, int n, Quant qt,
                                                                           int16_t* __restrict__ coef) {
    using M = Mcu<S>;
    __shared__ int ws[kStripBlocks * kBlkStride];
    const int f = find_frame<&Frame::cta0>(frames, n, blockIdx.x);
    const Frame fr = frames[f];
    const long long cta = blockIdx.x - fr.cta0;
    const int my = (int)(cta / fr.strips), mx0 = (int)(cta % fr.strips) * M::strip;
    const int nm = min(M::strip, fr.mcux - mx0);
    const int H = fr.H, W = fr.W, ch = (H + M::v - 1) / M::v;
    const uint8_t* __restrict__ src = fr.src;

    // samples minus 128: 64 chroma cells per MCU, each with its h x v luma pixels
    for (int i = threadIdx.x; i < nm * 64; i += kTransformThreads) {
        const int m = i >> 6, ly = (i >> 3) & 7, lx = i & 7;
        const int cy = my * 8 + ly, cx = (mx0 + m) * 8 + lx;
        int* blk = ws + m * M::blocks * kBlkStride;
        if (S == kGray) {
            blk[ly * 9 + lx] = __ldg(src + (size_t)min(cy, H - 1) * W + min(cx, W - 1)) - 128;
            continue;
        }
        int sb = 0, sr = 0;
        const int yc = min(cy, ch - 1);
        for (int dy = 0; dy < M::v; ++dy)
            for (int dx = 0; dx < M::h; ++dx) {
                const int x = min(M::h * cx + dx, W - 1);
                int b, g, r;
                load_bgr(src + ((size_t)min(M::v * cy + dy, H - 1) * W + x) * 3, b, g, r);
                const int yy = M::v * ly + dy, xx = M::h * lx + dx;
                blk[((yy >> 3) * M::h + (xx >> 3)) * kBlkStride + (yy & 7) * 9 + (xx & 7)] = rgb_y(r, g, b) - 128;
                if (M::v == 2) load_bgr(src + ((size_t)min(2 * yc + dy, H - 1) * W + x) * 3, b, g, r);
                sb += rgb_cb(r, g, b);
                sr += rgb_cr(r, g, b);
            }
        const int bias = S == k420 ? 1 + (lx & 1) : S == k422 ? lx & 1 : 0, shift = S == k420 ? 2 : S == k422 ? 1 : 0;
        blk[M::luma * kBlkStride + ly * 9 + lx] = ((sb + bias) >> shift) - 128;
        blk[(M::luma + 1) * kBlkStride + ly * 9 + lx] = ((sr + bias) >> shift) - 128;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nm * M::blocks * 8; i += kTransformThreads) fdct_pass<true>(ws + (i >> 3) * kBlkStride + (i & 7) * 9, 1);
    __syncthreads();
    for (int i = threadIdx.x; i < nm * M::blocks * 8; i += kTransformThreads) fdct_pass<false>(ws + (i >> 3) * kBlkStride + (i & 7), 9);
    __syncthreads();

    const int bx = (W + 7) >> 3, by = (H + 7) >> 3;
    int16_t* __restrict__ out = coef + (fr.blk0 + (long long)M::blocks * ((long long)my * fr.mcux + mx0)) * 64;
    for (int i = threadIdx.x; i < nm * M::blocks * 64; i += kTransformThreads) {
        const int k = i & 63, blkn = i >> 6, m = blkn / M::blocks, b = blkn - M::blocks * m;
        const int comp = b < M::luma ? 0 : 1;
        int src_b = b;      // a dummy luma block takes the DC of the last real block before it in the MCU
        if (M::luma > 1 && b < M::luma) {
            auto dummy = [&](int bb) { return M::h * (mx0 + m) + bb % M::h >= bx || M::v * my + bb / M::h >= by; };
            while (src_b > 0 && dummy(src_b)) --src_b;
        }
        int v;
        if (src_b != b) v = k == 0 ? quantise(ws[(m * M::blocks + src_b) * kBlkStride], qt.q8[0][0]) : 0;
        else {
            const int nat = kZigzag[k];
            v = quantise(ws[blkn * kBlkStride + (nat >> 3) * 9 + (nat & 7)], qt.q8[comp][nat]);
        }
        out[i] = (int16_t)v;
    }
}

// Huffman table: huff[t * 256 + symbol] = length << 16 | code, t = 0 DC luma, 1 AC luma, 2 DC chroma, 3 AC chroma
struct BitSink {
    uint32_t* words;     // the segment's stream as little-endian words of big-endian bit order (bswap on store)
    long long w;         // word being filled
    unsigned long long acc;
    int nacc;            // bits in acc; the first word starts with (bit offset & 31) bits owned by the blocks before
    bool first;
    __device__ __forceinline__ void put(uint32_t code, int len) {
        acc = (acc << len) | code;
        nacc += len;
        if (nacc >= 32) {
            nacc -= 32;
            const uint32_t word = __byte_perm((uint32_t)(acc >> nacc), 0, 0x0123);
            if (first) atomicOr(words + w, word); else words[w] = word;
            first = false;
            ++w;
        }
    }
    __device__ __forceinline__ void flush() {
        if (nacc > 0) atomicOr(words + w, __byte_perm((uint32_t)(acc << (32 - nacc)), 0, 0x0123));
    }
};

__device__ __forceinline__ int bit_length(int a) { return a ? 32 - __clz(a) : 0; }

// The bit total of segment k of a frame: its blocks' lengths from the exclusive scan excl.
__device__ __forceinline__ long long seg_bits(const Frame& fr, int k, int bpm, const long long* __restrict__ excl) {
    const long long b0 = fr.blk0 + (long long)k * fr.rst * bpm;
    const long long b1 = fr.blk0 + (long long)min((k + 1) * fr.rst, fr.mcux * fr.mcuy) * bpm;
    return excl[b1] - excl[b0];
}

// One thread per block of the call.  The DC prediction is the previous block of the same component in the block's segment.
//   kMode 0: bits[g] = the block's coded length.
//   kMode 1: the block's codes at bit offset excl[g] - excl[first block of its segment] of the segment's stream, which starts
//            at chunk seg_cx[segment]; the segment's last block pads the final byte with 1s.
//   kMode 2: the block's symbols counted into hist[frame * 1024 + table * 256 + symbol], through a CTA histogram for the
//            frame of the CTA's first block (EOB alone would contend on one global counter per frame).
// huff_stride: 0 = one table set for the call (Annex K), 1024 = one per frame (optimised).
template <int kMode, int S>
__global__ void __launch_bounds__(kCodeThreads) jpeg_code_kernel(const Frame* __restrict__ frames, int n, long long nblocks,
                                                                 const int16_t* __restrict__ coef, const uint32_t* __restrict__ huff,
                                                                 int huff_stride, int* __restrict__ bits, const long long* __restrict__ excl,
                                                                 const long long* __restrict__ seg_cx, uint32_t* __restrict__ raw,
                                                                 int* __restrict__ hist) {
    using M = Mcu<S>;
    __shared__ int sh[kMode == 2 ? 4 * 256 : 1];
    const long long g0 = (long long)blockIdx.x * kCodeThreads;
    long long g = g0 + threadIdx.x;
    const bool live = g < nblocks;
    int f0 = 0;
    if (kMode == 2) {
        for (int i = threadIdx.x; i < 4 * 256; i += kCodeThreads) sh[i] = 0;
        f0 = find_frame<&Frame::blk0>(frames, n, g0);
        __syncthreads();
        if (!live) g = nblocks - 1;         // walks a real block but counts nothing
    } else if (!live) {
        return;
    }
    const int f = find_frame<&Frame::blk0>(frames, n, g);
    const Frame& fr = frames[f];
    const int l = (int)(g - fr.blk0), mcu = l / M::blocks;
    const int b = l - M::blocks * mcu, comp = b < M::luma ? 0 : 1;
    const int seg = mcu / fr.rst;
    long long prev = -1;                       // previous block of the same component in the segment
    if (b >= 1 && b < M::luma) prev = g - 1;
    else if (mcu != seg * fr.rst) prev = b == 0 ? g - M::blocks + M::luma - 1 : g - M::blocks;
    // a mask of the nonzero coefficients; the values themselves are read again (from L1) only where the mask has a bit
    const int16_t* __restrict__ c = coef + g * 64;
    unsigned long long nz = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int4 q = __ldg(reinterpret_cast<const int4*>(c) + i);
        const uint32_t w[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            nz |= (unsigned long long)((w[j] & 0xffffu) != 0) << (8 * i + 2 * j) | (unsigned long long)((w[j] >> 16) != 0) << (8 * i + 2 * j + 1);
    }
    const int pred = prev >= 0 ? coef[prev * 64] : 0;
    const int t_dc = comp * 2;
    const uint32_t* __restrict__ dc_t = huff + (long long)f * huff_stride + t_dc * 256;
    const uint32_t* __restrict__ ac_t = dc_t + 256;
    int* __restrict__ h_dc = (f == f0 ? sh : hist + (long long)f * 1024) + t_dc * 256;
    int* __restrict__ h_ac = h_dc + 256;

    BitSink s{};
    long long total = 0;
    const long long gs = fr.blk0 + (long long)seg * fr.rst * M::blocks;    // the segment's first block
    if (kMode == 1) {
        const long long off = excl[g] - excl[gs];
        s.words = raw + seg_cx[fr.seg0 + seg] * (kChunk / 4);
        s.w = off >> 5;
        s.nacc = (int)(off & 31);
        s.first = true;
    }
    auto put = [&](const uint32_t* __restrict__ t, int* __restrict__ h, int sym, int extra, int nb) {    // a code then nb extra bits
        if (kMode == 2) {
            if (live) atomicAdd(h + sym, 1);
            return;
        }
        const uint32_t hc = __ldg(t + sym);
        const int len = (int)(hc >> 16);
        if (kMode == 1) s.put(((hc & 0xffff) << nb) | (uint32_t)(extra & ((1 << nb) - 1)), len + nb);
        else total += len + nb;
    };
    {
        const int diff = __ldg(c) - pred;
        const int nb = bit_length(diff < 0 ? -diff : diff);
        put(dc_t, h_dc, nb, diff < 0 ? diff - 1 : diff, nb);
    }
    nz &= ~1ull;
    int last = 0;
    while (nz) {
        const int k = __ffsll((long long)nz) - 1;
        nz &= nz - 1;
        int run = k - last - 1;
        for (; run > 15; run -= 16) put(ac_t, h_ac, 0xF0, 0, 0);
        const int v = __ldg(c + k);
        const int nb = bit_length(v < 0 ? -v : v);
        put(ac_t, h_ac, run << 4 | nb, v < 0 ? v - 1 : v, nb);
        last = k;
    }
    if (last < 63) put(ac_t, h_ac, 0, 0, 0);
    if (kMode == 0) { bits[g] = (int)total; return; }
    if (kMode == 2) {
        __syncthreads();
        int* __restrict__ hf = hist + (long long)f0 * 1024;
        for (int i = threadIdx.x; i < M::tables * 256; i += kCodeThreads)
            if (sh[i]) atomicAdd(hf + i, sh[i]);
        return;
    }
    if (g == fr.blk0 + (long long)min((seg + 1) * fr.rst, fr.mcux * fr.mcuy) * M::blocks - 1) {
        const int pad = (int)((8 - ((excl[g + 1] - excl[gs]) & 7)) & 7);
        if (pad) s.put((1u << pad) - 1, pad);
    }
    s.flush();
}

// ---- optimised Huffman tables: libjpeg's jpeg_gen_optimal_table, one warp per (frame, table)
constexpr int kSymsPerLane = 9;        // 32 x 9 >= 257 symbols: 0..255 and the reserved 256

// The warp's smallest (count << 9 | 511 - symbol) over live symbols other than `skip`: the smallest count, ties to the
// largest symbol, as libjpeg's "<=" scan picks.  ~0 when there is none.
__device__ __forceinline__ unsigned long long warp_min_sym(const long long (&freq)[kSymsPerLane], int lane, int skip) {
    unsigned long long key = ~0ull;
#pragma unroll
    for (int k = 0; k < kSymsPerLane; ++k) {
        const int j = lane * kSymsPerLane + k;
        if (freq[k] && j != skip) key = min(key, (unsigned long long)freq[k] << 9 | (unsigned)(511 - j));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
    return key;
}

// hist: nfreq[f * 1024 + t * 256 + symbol] counts; one 32-thread CTA per (frame f, table t < tables).  Writes the code table
// huff[f * 1024 + t * 256 + symbol] (0 for unused symbols) and dht[(f * 4 + t) * kDhtBytes]: counts per length 1..16, then the
// symbols by length, then value.
__global__ void __launch_bounds__(32) jpeg_huff_build_kernel(const int* __restrict__ hist, int tables, uint32_t* __restrict__ huff,
                                                             uint8_t* __restrict__ dht) {
    __shared__ int nbits[33];
    __shared__ uint8_t vals[256];
    const int f = blockIdx.x / tables, t = blockIdx.x - f * tables, lane = threadIdx.x;
    const int* __restrict__ h = hist + f * 1024 + t * 256;
    long long freq[kSymsPerLane];
    int size[kSymsPerLane], group[kSymsPerLane];
#pragma unroll
    for (int k = 0; k < kSymsPerLane; ++k) {
        const int j = lane * kSymsPerLane + k;
        freq[k] = j < 256 ? h[j] : j == 256;
        size[k] = 0;
        group[k] = j;         // the live symbol whose count holds this one's
    }
    for (;;) {
        const unsigned long long k1 = warp_min_sym(freq, lane, -1);
        const int c1 = 511 - (int)(k1 & 511);
        const unsigned long long k2 = warp_min_sym(freq, lane, c1);
        if (k2 == ~0ull) break;
        const int c2 = 511 - (int)(k2 & 511);
#pragma unroll
        for (int k = 0; k < kSymsPerLane; ++k) {
            const int j = lane * kSymsPerLane + k;
            if (j == c1) freq[k] += (long long)(k2 >> 9);
            if (j == c2) freq[k] = 0;
            if (group[k] == c1 || group[k] == c2) { ++size[k]; group[k] = c1; }
        }
    }
    // codes per length, then libjpeg's adjustment of lengths past 16 and the removal of the reserved code.  libjpeg refuses
    // a length past 32 (counts that grow like Fibonacci numbers past ~2^22 per table); dht's first byte 0xFF reports it.
    int over = 0;
#pragma unroll
    for (int k = 0; k < kSymsPerLane; ++k) over += size[k] > 32;
    if (__reduce_add_sync(0xffffffffu, over)) {
        if (lane == 0) dht[(f * 4 + t) * kDhtBytes] = 0xFF;
        return;
    }
    if (lane == 0) nbits[0] = 0;
    for (int len = 1; len <= 32; ++len) {
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < kSymsPerLane; ++k) cnt += size[k] == len;
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) nbits[len] = cnt;
    }
    // symbols 0..255 by length, then value: the symbols of a lane are consecutive, so lanes take places in order
    int base = 0;
    for (int len = 1; len <= 32; ++len) {
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < kSymsPerLane; ++k) cnt += size[k] == len && lane * kSymsPerLane + k < 256;
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        int p = base + incl - cnt;
#pragma unroll
        for (int k = 0; k < kSymsPerLane; ++k) {
            const int j = lane * kSymsPerLane + k;
            if (size[k] == len && j < 256) vals[p++] = (uint8_t)j;
        }
        base += __shfl_sync(0xffffffffu, incl, 31);
    }
    uint32_t* __restrict__ table = huff + f * 1024 + t * 256;
    for (int j = lane; j < 256; j += 32) table[j] = 0;
    __syncwarp();
    if (lane == 0) {
        for (int i = 32; i > 16; --i)
            while (nbits[i] > 0) {
                int j = i - 2;
                while (nbits[j] == 0) --j;
                nbits[i] -= 2;
                nbits[i - 1] += 1;
                nbits[j + 1] += 2;
                nbits[j] -= 1;
            }
        int i = 16;
        while (nbits[i] == 0) --i;
        nbits[i] -= 1;
        uint8_t* __restrict__ d = dht + (f * 4 + t) * kDhtBytes;
        uint32_t code = 0;
        int p = 0;
        for (int len = 1; len <= 16; ++len) {
            d[len - 1] = (uint8_t)nbits[len];
            for (int q = 0; q < nbits[len]; ++q, ++p) {
                table[vals[p]] = (uint32_t)len << 16 | code++;
                d[16 + p] = vals[p];
            }
            code <<= 1;
        }
    }
}

// ---- exclusive scan of int32 or int64 values into int64 (out[count] = total): tile sums, one CTA over the sums, tile re-scan
__device__ __forceinline__ long long cta_exclusive_scan(long long v, long long* warp_sums, long long& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        long long w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < kScanThreads / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    total = warp_sums[kScanThreads / 32 - 1];
    const long long r = x - v + (wid ? warp_sums[wid - 1] : 0);
    __syncthreads();
    return r;
}

template <typename T>
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_tiles_kernel(const T* __restrict__ in, long long count, long long* __restrict__ tile_sum) {
    __shared__ long long ws[kScanThreads / 32];
    const long long base = (long long)blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    long long s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) s += base + i < count ? (long long)in[base + i] : 0;
    long long total;
    cta_exclusive_scan(s, ws, total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// one CTA: tile_sum becomes its exclusive scan; *grand = the total
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_sums_kernel(long long* __restrict__ tile_sum, long long ntiles, long long* __restrict__ grand) {
    __shared__ long long ws[kScanThreads / 32];
    long long carry = 0;
    for (long long base = 0; base < ntiles; base += kScanThreads) {
        const long long i = base + threadIdx.x;
        const long long v = i < ntiles ? tile_sum[i] : 0;
        long long total;
        const long long e = cta_exclusive_scan(v, ws, total);
        if (i < ntiles) tile_sum[i] = carry + e;
        carry += total;
    }
    if (threadIdx.x == 0) *grand = carry;
}

template <typename T>
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_apply_kernel(const T* __restrict__ in, long long count,
                                                                       const long long* __restrict__ tile_excl, long long* __restrict__ out) {
    __shared__ long long ws[kScanThreads / 32];
    const long long base = (long long)blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    long long v[kScanItems], s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) { v[i] = base + i < count ? (long long)in[base + i] : 0; s += v[i]; }
    long long total;
    long long e = cta_exclusive_scan(s, ws, total) + tile_excl[blockIdx.x];
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        if (base + i < count) out[base + i] = e;
        e += v[i];
    }
}

// ---- segments, output placement and stuffing
// chunks[s] = 16-byte chunks of segment s's unstuffed stream (at least one: a segment has a block, a block a DC code)
__global__ void __launch_bounds__(256) jpeg_seg_chunks_kernel(const Frame* __restrict__ frames, int n, long long nseg, int bpm,
                                                              const long long* __restrict__ excl, int* __restrict__ chunks) {
    const long long s = (long long)blockIdx.x * 256 + threadIdx.x;
    if (s >= nseg) return;
    const int f = find_frame<&Frame::seg0>(frames, n, s);
    const long long bytes = (seg_bits(frames[f], (int)(s - frames[f].seg0), bpm, excl) + 7) >> 3;
    chunks[s] = (int)((bytes + kChunk - 1) / kChunk);
}

// The segment whose chunks [seg_cx[s], seg_cx[s + 1]) hold chunk i.
__device__ __forceinline__ long long find_seg(const long long* __restrict__ seg_cx, long long nseg, long long i) {
    long long lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (seg_cx[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Where chunk i is in its segment: frame f, segment k of the frame, byte pos in the segment, m stream bytes in the chunk, and
// whether an RSTm follows it (the last chunk of a segment other than the frame's last).
struct ChunkPlace {
    int f, k, m;
    bool rst;
};
__device__ __forceinline__ ChunkPlace place_chunk(const Frame* __restrict__ frames, int n, const long long* __restrict__ seg_cx, long long nseg,
                                                  int bpm, const long long* __restrict__ excl, long long i) {
    const long long s = find_seg(seg_cx, nseg, i);
    ChunkPlace p;
    p.f = find_frame<&Frame::seg0>(frames, n, s);
    const Frame& fr = frames[p.f];
    p.k = (int)(s - fr.seg0);
    const long long pos = (i - seg_cx[s]) * kChunk, nbytes = (seg_bits(fr, p.k, bpm, excl) + 7) >> 3;
    p.m = (int)min((long long)kChunk, nbytes - pos);
    p.rst = pos + kChunk >= nbytes && p.k + 1 < fr.nseg;
    return p;
}

// count[i] = output bytes of chunk i: its stream bytes, a 0x00 after each 0xFF, and 2 for an RSTm after it
__global__ void __launch_bounds__(256) jpeg_out_count_kernel(const Frame* __restrict__ frames, int n, const long long* __restrict__ seg_cx,
                                                             long long nseg, int bpm, const long long* __restrict__ excl,
                                                             const uint4* __restrict__ raw, long long nchunks, int* __restrict__ count) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const ChunkPlace p = place_chunk(frames, n, seg_cx, nseg, bpm, excl, i);
    const uint4 v = __ldg(raw + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int c = p.m + (p.rst ? 2 : 0);      // bytes past the stream inside the chunk are zero, so they never count as 0xFF
#pragma unroll
    for (int j = 0; j < 16; ++j) c += ((w[j >> 2] >> (8 * (j & 3))) & 0xff) == 0xff;
    count[i] = c;
}

// offsets[f] = where frame f's file starts in the output: header, stuffed stream with its RSTm, EOI; offsets[n] = the total
__global__ void jpeg_place_kernel(const Frame* __restrict__ frames, int n, const long long* __restrict__ seg_cx,
                                  const long long* __restrict__ outx, long long* __restrict__ offsets) {
    if (threadIdx.x != 0) return;
    long long o = 0;
    for (int f = 0; f < n; ++f) {
        const Frame& fr = frames[f];
        offsets[f] = o;
        o += fr.hdr + (outx[seg_cx[fr.seg0 + fr.nseg]] - outx[seg_cx[fr.seg0]]) + 2;
    }
    offsets[n] = o;
}

__global__ void __launch_bounds__(256) jpeg_stuff_kernel(const Frame* __restrict__ frames, int n, const long long* __restrict__ seg_cx,
                                                        long long nseg, int bpm, const long long* __restrict__ excl,
                                                        const uint4* __restrict__ raw, long long nchunks, const long long* __restrict__ outx,
                                                        const long long* __restrict__ offsets, uint8_t* __restrict__ out) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const ChunkPlace p = place_chunk(frames, n, seg_cx, nseg, bpm, excl, i);
    const Frame& fr = frames[p.f];
    uint8_t* dst = out + offsets[p.f] + fr.hdr + (outx[i] - outx[seg_cx[fr.seg0]]);
    const uint4 v = __ldg(raw + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < kChunk; ++j) {
        if (j >= p.m) break;
        const uint8_t byte = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        *dst++ = byte;
        if (byte == 0xff) *dst++ = 0;
    }
    if (p.rst) { dst[0] = 0xFF; dst[1] = (uint8_t)(0xD0 + (p.k & 7)); }
}

// ---- progressive files (DESIGN.md section 8.12): the same coefficients, coded as libjpeg's scan script
// A unit is one MCU of an interleaved (DC) scan, or one block of a one-component scan in the component's own raster order.
// Every scan of every frame of the call is one entry of the scan table, and its units follow the previous scan's units, so
// each kernel below runs all scans of the call in one grid.  For placement, output counting and stuffing each scan is a
// Frame of the existing kernels: units are its blocks (bpm 1), a restart interval of units its segment.
//   jpeg_prog_code_kernel<kProgShape, S>   flags: emits a symbol, ends in an EOB run (joins), correction bits it adds to a run
//   jpeg_prog_partition_kernel             splits each EOB run at 0x7FFF blocks and 937 buffered correction bits
//   jpeg_prog_code_kernel<kProgHist, S>    per-scan symbol histograms (jpeg_huff_build_kernel then builds each table)
//   jpeg_prog_code_kernel<kProgBits, S>    each unit's bit length;  <kProgEmit, S> its bits at its offset
constexpr int kEobRunMax = 0x7FFF;
constexpr int kMaxCorrBits = 1000 - 64 + 1;    // a run is flushed once its buffered correction bits pass this (libjpeg)
enum ProgMode { kProgShape = 0, kProgHist = 1, kProgBits = 2, kProgEmit = 3 };

struct ProgScan {
    long long u0;           // first unit of the scan in the call
    long long blk0;         // the frame's first block in coef
    long long seg0;         // first segment of the scan in the call
    int units, rst;         // units of the scan; units per segment
    int mcux, bw;           // MCUs per row of the frame; blocks per row of the component (one-component scans)
    int slot;               // table slot of component 0 (DC) or of the scan's AC table; DC chroma is slot + 1; -1: no table
    int comp;               // the component of a one-component scan; -1 for all (interleaved)
    int Ss, Se, Ah, Al;
};

__device__ __forceinline__ int find_scan(const ProgScan* __restrict__ sc, int n, long long u) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sc[mid].u0 <= u) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// One thread per unit of the call.  kMode:
//   kProgShape: emit[u] = the unit codes a symbol, join[u] = it ends in zeros (so it joins an EOB run), corr[u] = the
//               correction bits it adds to that run; eob[u] = 0.  DC units emit and never join.
//   kProgHist:  the unit's symbols, and the EOBn symbol of a run piece starting at it (eob[u] > 0), counted into
//               hist[slot * 256 + symbol] through a CTA histogram for the two slots of the CTA's first unit.
//   kProgBits:  bits[u] = its coded length;  kProgEmit: its bits at excl[u] - excl[first unit of its segment] in the
//               segment's stream at chunk seg_cx[segment], the segment's last unit padding the final byte with 1s.
// A unit's bits are its symbols (with the correction bits refinement buffers between them), then the EOBn symbol and its run
// length of a piece starting at it, then its own correction bits that the run carries: the stream order, as the blocks of a
// piece after its first send nothing but their correction bits.
template <int kMode, int S>
__global__ void __launch_bounds__(kCodeThreads) jpeg_prog_code_kernel(const ProgScan* __restrict__ scans, int nscans, long long nunits,
                                                                      const int16_t* __restrict__ coef, const uint32_t* __restrict__ huff,
                                                                      int* __restrict__ bits, uint8_t* __restrict__ emit,
                                                                      uint8_t* __restrict__ join, int* __restrict__ eob,
                                                                      const long long* __restrict__ excl, const long long* __restrict__ seg_cx,
                                                                      uint32_t* __restrict__ raw, int* __restrict__ hist) {
    using M = Mcu<S>;
    __shared__ int sh[kMode == kProgHist ? 2 * 256 : 1];
    const long long g0 = (long long)blockIdx.x * kCodeThreads;
    long long u = g0 + threadIdx.x;
    const bool live = u < nunits;
    int slot0 = -1;
    if (kMode == kProgHist) {
        for (int i = threadIdx.x; i < 2 * 256; i += kCodeThreads) sh[i] = 0;
        slot0 = scans[find_scan(scans, nscans, g0)].slot;
        __syncthreads();
        if (!live) u = nunits - 1;          // walks a real unit but counts nothing
    } else if (!live) {
        return;
    }
    const ProgScan p = scans[find_scan(scans, nscans, u)];
    const int l = (int)(u - p.u0), seg = l / p.rst;
    const bool seg_first = l == seg * p.rst;
    const long long us = p.u0 + (long long)seg * p.rst;        // the segment's first unit
    const bool seg_last = l + 1 == min((seg + 1) * p.rst, p.units);
    const int run = kMode == kProgShape ? 0 : eob[u];

    BitSink s{};
    long long total = 0;
    if (kMode == kProgEmit) {
        if (excl[u + 1] == excl[u] && !seg_last) return;
        const long long off = excl[u] - excl[us];
        s.words = raw + seg_cx[p.seg0 + seg] * (kChunk / 4);
        s.w = off >> 5;
        s.nacc = (int)(off & 31);
        s.first = true;
    }
    auto sym = [&](int t, int symbol, uint32_t extra, int nb) {     // table slot p.slot + t, then nb extra bits
        if (kMode == kProgHist) {
            if (!live) return;
            const int sl = p.slot + t;
            if (slot0 >= 0 && (unsigned)(sl - slot0) < 2u) atomicAdd(sh + (sl - slot0) * 256 + symbol, 1);
            else atomicAdd(hist + sl * 256 + symbol, 1);
            return;
        }
        if (kMode == kProgShape) return;
        const uint32_t hc = __ldg(huff + (p.slot + t) * 256 + symbol);
        const int len = (int)(hc >> 16);
        if (kMode == kProgEmit) s.put(((hc & 0xffff) << nb) | (extra & ((1u << nb) - 1)), len + nb);
        else total += len + nb;
    };
    auto put_bits = [&](unsigned long long v, int nb) {             // nb <= 63 raw bits
        if (kMode == kProgEmit) {
            for (; nb > 32; nb -= 32) s.put((uint32_t)(v >> (nb - 32)), 32);
            s.put((uint32_t)(v & ((1ull << nb) - 1)), nb);
        } else if (kMode == kProgBits) {
            total += nb;
        }
    };

    bool emits = true, joins = false;
    int ncorr = 0;
    unsigned long long corr = 0;        // the correction bits this unit hands to its run
    if (p.Ss == 0) {
        // DC: every block of the MCU (one block for gray), the prediction being the previous block of the same component in
        // the segment, shifted by Al
        const long long g = p.blk0 + (long long)l * M::blocks;
#pragma unroll
        for (int b = 0; b < M::blocks; ++b) {
            const int v = coef[(g + b) * 64] >> p.Al;
            if (p.Ah) { put_bits(v & 1, 1); continue; }
            long long prev = -1;
            if (b >= 1 && b < M::luma) prev = g + b - 1;
            else if (!seg_first) prev = b == 0 ? g - M::blocks + M::luma - 1 : g + b - M::blocks;
            const int diff = v - (prev >= 0 ? coef[prev * 64] >> p.Al : 0);
            const int nb = bit_length(diff < 0 ? -diff : diff);
            sym(b < M::luma ? 0 : 1, nb, (uint32_t)(diff < 0 ? diff - 1 : diff), nb);
        }
    } else {
        long long g;
        if (p.comp == 0) {
            const int by = l / p.bw, bx = l - by * p.bw;
            g = p.blk0 + (long long)((by / M::v) * p.mcux + bx / M::h) * M::blocks + (by % M::v) * M::h + bx % M::h;
        } else {
            g = p.blk0 + (long long)l * M::blocks + M::luma + p.comp - 1;
        }
        // masks of the band's coefficients with |c| >> Al == 1 and > 1
        const int16_t* __restrict__ c = coef + g * 64;
        unsigned long long one = 0, big = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int4 q = __ldg(reinterpret_cast<const int4*>(c) + i);
            const uint32_t w[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int v = (int16_t)(w[j >> 1] >> (16 * (j & 1)));
                const int a = (v < 0 ? -v : v) >> p.Al;
                one |= (unsigned long long)(a == 1) << (8 * i + j);
                big |= (unsigned long long)(a > 1) << (8 * i + j);
            }
        }
        const unsigned long long band = (~0ull >> (63 - p.Se)) & (~0ull << p.Ss);
        one &= band;
        big &= band;
        int last = p.Ss - 1;
        if (p.Ah == 0) {
            unsigned long long nz = one | big;
            emits = nz != 0;
            while (nz) {
                const int k = __ffsll((long long)nz) - 1;
                nz &= nz - 1;
                int r = k - last - 1;
                for (; r > 15; r -= 16) sym(0, 0xF0, 0, 0);
                const int v = __ldg(c + k), a = (v < 0 ? -v : v) >> p.Al;
                const int nb = bit_length(a);
                sym(0, r << 4 | nb, (uint32_t)(v < 0 ? ~a : a), nb);
                last = k;
            }
            joins = last < p.Se;
        } else {
            // refinement: a coefficient that was nonzero before sends one correction bit, buffered until the next symbol;
            // zero runs past 15 send ZRL only up to the last newly nonzero coefficient
            const int eob_k = one ? 63 - __clzll((long long)one) : -1;
            unsigned long long nz = one | big;
            emits = one != 0;
            int r = 0;
            while (nz) {
                const int k = __ffsll((long long)nz) - 1;
                nz &= nz - 1;
                r += k - last - 1;
                last = k;
                for (; r > 15 && k <= eob_k; r -= 16) {
                    sym(0, 0xF0, 0, 0);
                    put_bits(corr, ncorr);
                    corr = 0; ncorr = 0;
                }
                const int v = __ldg(c + k);
                if ((big >> k) & 1) {
                    corr = corr << 1 | (((v < 0 ? -v : v) >> p.Al) & 1);
                    ++ncorr;
                    continue;
                }
                sym(0, r << 4 | 1, v < 0 ? 0 : 1, 1);
                put_bits(corr, ncorr);
                corr = 0; ncorr = 0; r = 0;
            }
            r += p.Se - last;
            joins = r > 0 || ncorr > 0;
        }
    }
    if (kMode == kProgShape) {
        emit[u] = emits;
        join[u] = joins;
        bits[u] = joins ? ncorr : 0;
        eob[u] = 0;
        return;
    }
    if (run > 0) {
        const int nb = 31 - __clz(run);
        sym(0, nb << 4, (uint32_t)run, nb);
    }
    if (joins) put_bits(corr, ncorr);
    if (kMode == kProgBits) { bits[u] = (int)total; return; }
    if (kMode == kProgHist) {
        __syncthreads();
        if (slot0 >= 0)
            for (int i = threadIdx.x; i < 2 * 256; i += kCodeThreads)
                if (sh[i]) atomicAdd(hist + slot0 * 256 + i, sh[i]);
        return;
    }
    if (seg_last) {
        const int pad = (int)((8 - ((excl[u + 1] - excl[us]) & 7)) & 7);
        if (pad) s.put((1u << pad) - 1, pad);
    }
    s.flush();
}

// One thread per unit.  A run starts at a joining unit that is its segment's first, emits a symbol, or follows a unit that
// did not join; it ends before the next emitting unit or at the segment's end.  Its starting thread splits it greedily where
// libjpeg flushes: after 0x7FFF units, or after the unit that takes the buffered correction bits past kMaxCorrBits.  corr_x
// and emit_x are exclusive scans of the units' correction bits and emit flags; eob[first unit of each piece] = its length.
__global__ void __launch_bounds__(256) jpeg_prog_partition_kernel(const ProgScan* __restrict__ scans, int nscans, long long nunits,
                                                                  const uint8_t* __restrict__ emit, const uint8_t* __restrict__ join,
                                                                  const long long* __restrict__ corr_x, const long long* __restrict__ emit_x,
                                                                  int* __restrict__ eob) {
    const long long u = (long long)blockIdx.x * 256 + threadIdx.x;
    if (u >= nunits || !join[u]) return;
    const ProgScan& p = scans[find_scan(scans, nscans, u)];
    const int l = (int)(u - p.u0), seg = l / p.rst;
    if (l != seg * p.rst && !emit[u] && join[u - 1]) return;
    long long lo = u, hi = p.u0 + min((seg + 1) * p.rst, p.units) - 1;    // the run's end: no emitting unit in (u, end]
    const long long e0 = emit_x[u + 1];
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (emit_x[mid + 1] == e0) lo = mid; else hi = mid - 1;
    }
    const long long end = lo;
    for (long long q = u; q <= end;) {
        long long e = min(q + kEobRunMax - 1, end);
        if (p.Ah && corr_x[e + 1] - corr_x[q] > kMaxCorrBits) {     // the first unit that passes the cap
            long long a = q, b = e;
            while (a < b) {
                const long long mid = (a + b) >> 1;
                if (corr_x[mid + 1] - corr_x[q] > kMaxCorrBits) b = mid; else a = mid + 1;
            }
            e = a;
        }
        eob[q] = (int)(e - q + 1);
        q = e + 1;
    }
}

}  // namespace jpeg
}  // namespace whenet
