// kernels_jpeg.cuh - baseline JPEG encoding of packed BGR frames, byte-identical to cv2.imencode (libjpeg-turbo defaults: 4:2:0,
// Annex K Huffman tables, islow FDCT, no restart markers).  DESIGN.md section 8.9; oracle/jpeg_oracle.py restates every step.
//
// One call encodes up to 64 frames of their own sizes.  Every kernel reads the call's frame table and works on global indices
// (transform CTAs, blocks, 16-byte chunks) that it maps back to a frame, so a frame's bytes never depend on the other frames.
//   jpeg_transform_kernel   colour conversion, 4:2:0 downsampling, FDCT, quantisation, zigzag: int16 coefficients per block
//   jpeg_code_kernel<0>     each block's Huffman bit length
//   jpeg_scan_*             exclusive int64 scan (bit offsets of blocks; 0xFF counts of chunks)
//   jpeg_code_kernel<1>     each block writes its codes at its bit offset (atomicOr into a zeroed buffer where words are shared)
//   jpeg_ff_count_kernel / jpeg_stuff_kernel   0x00 after every 0xFF, each frame's stream at its place in the output
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace whenet {
namespace jpeg {

constexpr int kMaxFrames = 64;
constexpr int kStripMcus = 8;          // a transform CTA codes 8 MCUs (128 x 16 pixels) of one MCU row
constexpr int kStripBlocks = 6 * kStripMcus;
constexpr int kTransformThreads = 256;
constexpr int kCodeThreads = 128;
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;
constexpr int kChunk = 16;             // bytes per stuffing thread; every frame's unstuffed stream starts on a chunk
constexpr int kHeaderBytes = 623;      // SOI .. SOS of this encoder's files (the same for every size and quality)

struct Frame {
    const uint8_t* src;     // H x W x 3 BGR
    int H, W, mcux, mcuy, strips;   // strips: transform CTAs per MCU row
    long long cta0;         // first transform CTA of the frame
    long long blk0;         // first block (scan order) of the frame in the call
    long long raw0;         // first byte of its unstuffed stream (a multiple of kChunk)
    long long nbytes;       // unstuffed bytes, last byte padded with 1s
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

// One CTA per strip of kStripMcus MCUs of one MCU row.  Writes the strip's blocks (6 per MCU: Y00 Y01 Y10 Y11 Cb Cr) as zigzag
// int16 at coef[(blk0 + 6 * mcu + b) * 64].  Luma replicates the last row and column to the block boundary; chroma replicates
// the last column to the chroma block boundary and (odd H) the last row once, downsamples with bias 1, 2, 1, 2, ..., and then
// replicates the last downsampled row.  Luma blocks past the image (dummy blocks) get AC 0 and the DC of the block before them.
__global__ void __launch_bounds__(kTransformThreads) jpeg_transform_kernel(const Frame* __restrict__ frames, int n, Quant qt,
                                                                           int16_t* __restrict__ coef) {
    __shared__ int ws[kStripBlocks * kBlkStride];
    const int f = find_frame<&Frame::cta0>(frames, n, blockIdx.x);
    const Frame fr = frames[f];
    const long long cta = blockIdx.x - fr.cta0;
    const int my = (int)(cta / fr.strips), mx0 = (int)(cta % fr.strips) * kStripMcus;
    const int nm = min(kStripMcus, fr.mcux - mx0);
    const int H = fr.H, W = fr.W, ch = (H + 1) >> 1;
    const uint8_t* __restrict__ src = fr.src;

    // samples minus 128: 64 chroma cells per MCU, each with its 2 x 2 luma pixels
    for (int i = threadIdx.x; i < nm * 64; i += kTransformThreads) {
        const int m = i >> 6, ly = (i >> 3) & 7, lx = i & 7;
        const int cy = my * 8 + ly, cx = (mx0 + m) * 8 + lx;
        int* blk = ws + m * 6 * kBlkStride;
        int sb = 0, sr = 0;
        const int yc = min(cy, ch - 1);
        for (int dy = 0; dy < 2; ++dy)
            for (int dx = 0; dx < 2; ++dx) {
                const int x = min(2 * cx + dx, W - 1);
                int b, g, r;
                load_bgr(src + ((size_t)min(2 * cy + dy, H - 1) * W + x) * 3, b, g, r);
                const int yy = 2 * ly + dy, xx = 2 * lx + dx;
                blk[((yy >> 3) * 2 + (xx >> 3)) * kBlkStride + (yy & 7) * 9 + (xx & 7)] = rgb_y(r, g, b) - 128;
                load_bgr(src + ((size_t)min(2 * yc + dy, H - 1) * W + x) * 3, b, g, r);
                sb += rgb_cb(r, g, b);
                sr += rgb_cr(r, g, b);
            }
        const int bias = 1 + (lx & 1);
        blk[4 * kBlkStride + ly * 9 + lx] = ((sb + bias) >> 2) - 128;
        blk[5 * kBlkStride + ly * 9 + lx] = ((sr + bias) >> 2) - 128;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nm * 48; i += kTransformThreads) fdct_pass<true>(ws + (i >> 3) * kBlkStride + (i & 7) * 9, 1);
    __syncthreads();
    for (int i = threadIdx.x; i < nm * 48; i += kTransformThreads) fdct_pass<false>(ws + (i >> 3) * kBlkStride + (i & 7), 9);
    __syncthreads();

    const int bx = (W + 7) >> 3, by = (H + 7) >> 3;
    int16_t* __restrict__ out = coef + (fr.blk0 + 6LL * ((long long)my * fr.mcux + mx0)) * 64;
    for (int i = threadIdx.x; i < nm * 6 * 64; i += kTransformThreads) {
        const int k = i & 63, blkn = i >> 6, m = blkn / 6, b = blkn - 6 * m;
        const int comp = b < 4 ? 0 : 1;
        int src_b = b;      // a dummy luma block takes the DC of the last real block before it in the MCU
        if (b < 4) {
            auto dummy = [&](int bb) { return 2 * (mx0 + m) + (bb & 1) >= bx || 2 * my + (bb >> 1) >= by; };
            while (src_b > 0 && dummy(src_b)) --src_b;
        }
        int v;
        if (src_b != b) v = k == 0 ? quantise(ws[(m * 6 + src_b) * kBlkStride], qt.q8[0][0]) : 0;
        else {
            const int nat = kZigzag[k];
            v = quantise(ws[blkn * kBlkStride + (nat >> 3) * 9 + (nat & 7)], qt.q8[comp][nat]);
        }
        out[i] = (int16_t)v;
    }
}

// Huffman table: huff[t * 256 + symbol] = length << 16 | code, t = 0 DC luma, 1 AC luma, 2 DC chroma, 3 AC chroma
struct BitSink {
    uint32_t* words;     // the frame's stream as little-endian words of big-endian bit order (bswap on store)
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

// One thread per block of the call.  kEmit = 0: bits[g] = the block's coded length.  kEmit = 1: the block's codes at bit
// offset excl[g] - excl[blk0] of its frame's stream, and the frame's last block pads the final byte with 1s.
template <int kEmit>
__global__ void __launch_bounds__(kCodeThreads) jpeg_code_kernel(const Frame* __restrict__ frames, int n, long long nblocks,
                                                                 const int16_t* __restrict__ coef, const uint32_t* __restrict__ huff,
                                                                 int* __restrict__ bits, const long long* __restrict__ excl,
                                                                 uint32_t* __restrict__ raw) {
    const long long g = (long long)blockIdx.x * kCodeThreads + threadIdx.x;
    if (g >= nblocks) return;
    const int f = find_frame<&Frame::blk0>(frames, n, g);
    const Frame& fr = frames[f];
    const long long l = g - fr.blk0, mcu = l / 6;
    const int b = (int)(l - 6 * mcu), comp = b < 4 ? 0 : 1;
    long long prev = -1;                       // previous block of the same component in scan order
    if (b >= 1 && b <= 3) prev = g - 1;
    else if (mcu > 0) prev = b == 0 ? g - 3 : g - 6;
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
    const uint32_t* __restrict__ dc_t = huff + comp * 512;
    const uint32_t* __restrict__ ac_t = dc_t + 256;

    BitSink s{};
    long long total = 0;
    if (kEmit) {
        const long long off = excl[g] - excl[fr.blk0];
        s.words = raw + (fr.raw0 >> 2);
        s.w = off >> 5;
        s.nacc = (int)(off & 31);
        s.first = true;
    }
    auto put = [&](uint32_t hc, int extra, int nb) {      // a Huffman code then nb extra bits
        const int len = (int)(hc >> 16);
        if (kEmit) s.put(((hc & 0xffff) << nb) | (uint32_t)(extra & ((1 << nb) - 1)), len + nb);
        else total += len + nb;
    };
    {
        const int diff = __ldg(c) - pred;
        const int nb = bit_length(diff < 0 ? -diff : diff);
        put(__ldg(dc_t + nb), diff < 0 ? diff - 1 : diff, nb);
    }
    nz &= ~1ull;
    int last = 0;
    while (nz) {
        const int k = __ffsll((long long)nz) - 1;
        nz &= nz - 1;
        int run = k - last - 1;
        for (; run > 15; run -= 16) put(__ldg(ac_t + 0xF0), 0, 0);
        const int v = __ldg(c + k);
        const int nb = bit_length(v < 0 ? -v : v);
        put(__ldg(ac_t + (run << 4 | nb)), v < 0 ? v - 1 : v, nb);
        last = k;
    }
    if (last < 63) put(__ldg(ac_t), 0, 0);
    if (!kEmit) { bits[g] = (int)total; return; }
    if (l == 6LL * fr.mcux * fr.mcuy - 1) {
        const int pad = (int)((8 - ((excl[g + 1] - excl[fr.blk0]) & 7)) & 7);
        if (pad) s.put((1u << pad) - 1, pad);
    }
    s.flush();
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

// ---- per-frame totals and output placement (one thread per frame)
__global__ void jpeg_frame_bits_kernel(const Frame* __restrict__ frames, int n, const long long* __restrict__ excl, long long* __restrict__ fbits) {
    const int f = threadIdx.x;
    if (f >= n) return;
    const Frame& fr = frames[f];
    fbits[f] = excl[fr.blk0 + 6LL * fr.mcux * fr.mcuy] - excl[fr.blk0];
}

// offsets[f] = where frame f's file starts in the output: header, stuffed stream, EOI; offsets[n] = the total
__global__ void jpeg_place_kernel(const Frame* __restrict__ frames, int n, const long long* __restrict__ ffx, long long* __restrict__ offsets) {
    if (threadIdx.x != 0) return;
    long long o = 0;
    for (int f = 0; f < n; ++f) {
        const Frame& fr = frames[f];
        offsets[f] = o;
        const long long c0 = fr.raw0 / kChunk, c1 = (fr.raw0 + fr.nbytes + kChunk - 1) / kChunk;
        o += kHeaderBytes + fr.nbytes + (ffx[c1] - ffx[c0]) + 2;
    }
    offsets[n] = o;
}

__global__ void __launch_bounds__(256) jpeg_ff_count_kernel(const uint4* __restrict__ raw, long long nchunks, int* __restrict__ count) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const uint4 v = __ldg(raw + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int c = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) c += ((w[j >> 2] >> (8 * (j & 3))) & 0xff) == 0xff;
    count[i] = c;
}

// bytes past a frame's stream inside its last chunk are zero, so they never count as 0xFF
__global__ void __launch_bounds__(256) jpeg_stuff_kernel(const Frame* __restrict__ frames, int n, const uint4* __restrict__ raw, long long nchunks,
                                                        const long long* __restrict__ ffx, const long long* __restrict__ offsets,
                                                        uint8_t* __restrict__ out) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const int f = find_frame<&Frame::raw0>(frames, n, i * kChunk);
    const Frame& fr = frames[f];
    const long long pos = i * kChunk - fr.raw0;
    if (pos >= fr.nbytes) return;
    uint8_t* dst = out + offsets[f] + kHeaderBytes + pos + (ffx[i] - ffx[fr.raw0 / kChunk]);
    const uint4 v = __ldg(raw + i);
    const int m = (int)min((long long)kChunk, fr.nbytes - pos);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < kChunk; ++j) {
        if (j >= m) return;
        const uint8_t byte = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        *dst++ = byte;
        if (byte == 0xff) *dst++ = 0;
    }
}

}  // namespace jpeg
}  // namespace whenet
