// jpeg_api.cu - whenet_encode_jpeg_u8 / _ragged_u8 / _ex_u8 and their debug entries (DESIGN.md sections 8.9, 8.11 and 8.12):
// baseline or progressive JPEG files of device or host BGR or gray frames, byte-identical to cv2.imencode(".jpg", frame, params)
// with the quality, sampling, restart-interval, optimised-Huffman, luma/chroma-quality and progressive parameters.  The
// decoder (section 8.10) is jpeg_decode.inc, included at the end.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/whenet_b200.h"
#include "api_error.h"
#include "jpeg_api.h"
#include "kernels_jpeg.cuh"

using whenet::api::fail;
namespace J = whenet::jpeg;

#define JCK(call)                                                                                  \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail(WHENET_ECUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,         \
                        cudaGetErrorString(e__));                                                  \
    } while (0)

namespace whenet {
namespace jpeg {

// Every buffer grows to what a call needs and is kept for the next call; all are freed by destroy().
struct State {
    uint32_t* d_huff = nullptr;                 // 4 x 256 entries: length << 16 | code (Annex K)
    uint32_t* d_ohuff = nullptr;                // optimised: 4 x 256 entries per frame
    int* d_hist = nullptr;                      // optimised: 4 x 256 symbol counts per frame
    uint8_t* d_dht = nullptr;                   // optimised: 4 x kDhtBytes per frame, read back with the segment chunk total
    uint8_t* h_dht = nullptr;                   // pinned
    Frame* d_frames = nullptr;
    long long* d_small = nullptr;               // the n + 1 output offsets
    long long* h_small = nullptr;               // pinned
    uint8_t* d_in = nullptr; size_t in_cap = 0;                 // host frames, uploaded
    int16_t* d_coef = nullptr; size_t coef_cap = 0;             // elements
    int* d_bits = nullptr; size_t bits_cap = 0;                 // per block
    long long* d_excl = nullptr; size_t excl_cap = 0;           // per block + 1
    int* d_segc = nullptr; size_t segc_cap = 0;                 // chunks per segment
    long long* d_segx = nullptr; size_t segx_cap = 0;           // per segment + 1: first chunk
    long long* d_tiles = nullptr; size_t tiles_cap = 0;
    uint32_t* d_raw = nullptr; size_t raw_cap = 0;              // bytes
    int* d_ffc = nullptr; size_t ffc_cap = 0;                   // output bytes per chunk
    long long* d_ffx = nullptr; size_t ffx_cap = 0;
    uint8_t* d_out = nullptr; size_t out_cap = 0;
    uint8_t* h_out = nullptr; size_t h_cap = 0;                 // pinned: the files handed to the caller
    // progressive (section 8.12): the scan table, each scan as a Frame, its n * scans + 1 offsets, optimal tables per slot
    ProgScan* d_pscans = nullptr;
    Frame* d_pframes = nullptr;
    long long* d_psmall = nullptr;
    long long* h_psmall = nullptr;              // pinned
    int* d_phist = nullptr;
    uint32_t* d_phuff = nullptr;
    uint8_t* d_pdht = nullptr;
    uint8_t* h_pdht = nullptr;                  // pinned
    uint8_t* d_pemit = nullptr; size_t pemit_cap = 0;           // per unit: codes a symbol
    uint8_t* d_pjoin = nullptr; size_t pjoin_cap = 0;           // per unit: ends in an EOB run
    int* d_peob = nullptr; size_t peob_cap = 0;                 // per unit: the length of the EOB run piece starting there
    long long* d_pemitx = nullptr; size_t pemitx_cap = 0;       // per unit + 1: exclusive scan of d_pemit
    DecState* dec = nullptr;                                    // the decoder's scratch (jpeg_decode.inc)
};

}  // namespace jpeg
}  // namespace whenet

namespace {

// T.81 Annex K.1 (natural order) and K.3
const uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,
                            69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55,  64,
                            81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                              99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                              99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZigzagHost[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t kDcCounts[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
const uint8_t kDcSyms[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcCounts[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
const uint8_t kAcSyms[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// IJG quality scaling, clamped to baseline's [1, 255]; natural order
void quant_table(int quality, int chroma, int out[64]) {
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; ++i) out[i] = std::min(255, std::max(1, ((chroma ? kChromaQ : kLumaQ)[i] * s + 50) / 100));
}

// canonical codes (T.81 Annex C): table[symbol] = length << 16 | code
void huff_table(const uint8_t counts[16], const uint8_t* syms, uint32_t table[256]) {
    uint32_t code = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int i = 0; i < counts[len - 1]; ++i) table[syms[k++]] = (uint32_t)len << 16 | code++;
        code <<= 1;
    }
}

// What a call encodes: luma and chroma qualities, MCU shape (J::Shape, kGray for one channel), restart interval in MCUs
// (0 = none), optimised tables.
struct Opts {
    int quality, chroma_quality, shape, restart, optimize, progressive;
};
constexpr int kMaxHeaderBytes = 2 + 18 + 2 * 69 + 19 + 4 * (5 + J::kDhtBytes) + 6 + 14;

// SOI, APP0 (JFIF 1.01, density 1:1, no thumbnail), DQT luma and chroma (zigzag), and SOF0 (baseline) or SOF2 (progressive);
// gray has one DQT and one component.  Returns the bytes written.
int frame_header(int H, int W, const Opts& o, uint8_t sof, uint8_t* out) {
    const bool gray = o.shape == J::kGray;
    const int nc = gray ? 1 : 3;
    uint8_t* p = out;
    auto seg = [&](uint8_t marker, int len) { *p++ = 0xFF; *p++ = marker; *p++ = (uint8_t)((len + 2) >> 8); *p++ = (uint8_t)(len + 2); };
    *p++ = 0xFF; *p++ = 0xD8;
    seg(0xE0, 14);
    const uint8_t app0[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    memcpy(p, app0, 14); p += 14;
    for (int t = 0; t < (gray ? 1 : 2); ++t) {
        int q[64];
        quant_table(t ? o.chroma_quality : o.quality, t, q);
        seg(0xDB, 65);
        *p++ = (uint8_t)t;
        for (int k = 0; k < 64; ++k) *p++ = (uint8_t)q[kZigzagHost[k]];
    }
    seg(sof, 6 + 3 * nc);
    const uint8_t ysf = o.shape == J::k420 ? 0x22 : o.shape == J::k422 ? 0x21 : 0x11;
    const uint8_t sofb[15] = {8, (uint8_t)(H >> 8), (uint8_t)H, (uint8_t)(W >> 8), (uint8_t)W, (uint8_t)nc, 1, ysf, 0, 2, 0x11, 1, 3, 0x11, 1};
    memcpy(p, sofb, 6 + 3 * nc); p += 6 + 3 * nc;
    return (int)(p - out);
}

// frame_header with SOF0, then DHT DC0 AC0 DC1 AC1, DRI when restarts, SOS; gray has DHT DC0 AC0.  dht: the optimised tables
// (4 x kDhtBytes), or nullptr for Annex K.
int header_bytes(int H, int W, const Opts& o, const uint8_t* dht, uint8_t* out) {
    const bool gray = o.shape == J::kGray;
    const int nc = gray ? 1 : 3;
    uint8_t* p = out + frame_header(H, W, o, 0xC0, out);
    auto seg = [&](uint8_t marker, int len) { *p++ = 0xFF; *p++ = marker; *p++ = (uint8_t)((len + 2) >> 8); *p++ = (uint8_t)(len + 2); };
    for (int t = 0; t < (gray ? 2 : 4); ++t) {
        const int chroma = t >> 1, ac = t & 1;
        const uint8_t* counts = dht ? dht + t * J::kDhtBytes : ac ? kAcCounts[chroma] : kDcCounts[chroma];
        const uint8_t* syms = dht ? counts + 16 : ac ? kAcSyms[chroma] : kDcSyms;
        int nsym = 0;
        for (int i = 0; i < 16; ++i) nsym += counts[i];
        seg(0xC4, 17 + nsym);
        *p++ = (uint8_t)(ac << 4 | chroma);
        memcpy(p, counts, 16); p += 16;
        memcpy(p, syms, nsym); p += nsym;
    }
    if (o.restart) {
        seg(0xDD, 2);
        *p++ = (uint8_t)(o.restart >> 8); *p++ = (uint8_t)o.restart;
    }
    seg(0xDA, 4 + 2 * nc);
    const uint8_t sos[10] = {(uint8_t)nc, 1, 0x00, 2, 0x11, 3, 0x11};
    memcpy(p, sos, 1 + 2 * nc); p += 1 + 2 * nc;
    *p++ = 0; *p++ = 63; *p++ = 0;
    return (int)(p - out);
}

// libjpeg's jpeg_gen_optimal_table on the host, as jpeg_huff_build_kernel runs it on the device: bits = codes per length
// 1..16, vals = the symbols by length then value.  Returns the number of symbols, or -1 for a code longer than 32 bits
// (libjpeg refuses those).
int gen_optimal_table(const int32_t* counts, uint8_t bits[16], uint8_t vals[256]) {
    long long freq[257];
    int codesize[257], others[257], nb[33] = {0};
    for (int i = 0; i < 257; ++i) { freq[i] = i < 256 ? counts[i] : 1; codesize[i] = 0; others[i] = -1; }
    for (;;) {
        int c1 = -1, c2 = -1;
        long long v = 1000000000LL;
        for (int i = 0; i <= 256; ++i)
            if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = 1000000000LL;
        for (int i = 0; i <= 256; ++i)
            if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
        if (c2 < 0) break;
        freq[c1] += freq[c2];
        freq[c2] = 0;
        ++codesize[c1];
        while (others[c1] >= 0) { c1 = others[c1]; ++codesize[c1]; }
        others[c1] = c2;
        ++codesize[c2];
        while (others[c2] >= 0) { c2 = others[c2]; ++codesize[c2]; }
    }
    for (int i = 0; i <= 256; ++i)
        if (codesize[i]) {
            if (codesize[i] > 32) return -1;
            ++nb[codesize[i]];
        }
    for (int i = 32; i > 16; --i)
        while (nb[i] > 0) {
            int j = i - 2;
            while (nb[j] == 0) --j;
            nb[i] -= 2; nb[i - 1] += 1; nb[j + 1] += 2; nb[j] -= 1;
        }
    int i = 16;
    while (nb[i] == 0) --i;
    nb[i] -= 1;
    for (int l = 1; l <= 16; ++l) bits[l - 1] = (uint8_t)nb[l];
    int p = 0;
    for (int l = 1; l <= 32; ++l)
        for (int j = 0; j < 256; ++j)
            if (codesize[j] == l) vals[p++] = (uint8_t)j;
    return p;
}

template <class T>
int grow(T*& p, size_t& cap, size_t need) {
    if (need <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    JCK(cudaMalloc(&p, need * sizeof(T)));
    cap = need;
    return 0;
}

int grow_host(uint8_t*& p, size_t& cap, size_t need) {
    if (need <= cap) return 0;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    JCK(cudaHostAlloc((void**)&p, need, cudaHostAllocDefault));
    cap = need;
    return 0;
}

int create(J::State*& st) {
    st = new J::State();
    JCK(cudaMalloc(&st->d_huff, 4 * 256 * sizeof(uint32_t)));
    JCK(cudaMalloc(&st->d_frames, J::kMaxFrames * sizeof(J::Frame)));
    JCK(cudaMalloc(&st->d_small, (J::kMaxFrames + 1) * sizeof(long long)));
    JCK(cudaHostAlloc((void**)&st->h_small, (J::kMaxFrames + 1) * sizeof(long long), cudaHostAllocDefault));
    std::vector<uint32_t> huff(4 * 256, 0);
    for (int t = 0; t < 4; ++t) {
        const int chroma = t >> 1, ac = t & 1;
        huff_table(ac ? kAcCounts[chroma] : kDcCounts[chroma], ac ? kAcSyms[chroma] : kDcSyms, huff.data() + 256 * t);
    }
    JCK(cudaMemcpy(st->d_huff, huff.data(), huff.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    return 0;
}

// exclusive scan of count values into out[0 .. count]; out[count] = the total
template <typename T>
int scan(J::State* st, cudaStream_t s, const T* in, long long count, long long* out) {
    const long long tiles = (count + J::kScanTile - 1) / J::kScanTile;
    if (int rc = grow(st->d_tiles, st->tiles_cap, (size_t)tiles)) return rc;
    J::jpeg_scan_tiles_kernel<T><<<(unsigned)tiles, J::kScanThreads, 0, s>>>(in, count, st->d_tiles);
    J::jpeg_scan_sums_kernel<<<1, J::kScanThreads, 0, s>>>(st->d_tiles, tiles, out + count);
    J::jpeg_scan_apply_kernel<T><<<(unsigned)tiles, J::kScanThreads, 0, s>>>(in, count, st->d_tiles, out);
    JCK(cudaGetLastError());
    return 0;
}

// Runs f(J::Mcu<shape>{}) for the call's MCU shape.
template <class F>
void by_shape(int shape, F&& f) {
    switch (shape) {
    case J::k420: f(J::Mcu<J::k420>{}); break;
    case J::k422: f(J::Mcu<J::k422>{}); break;
    case J::k444: f(J::Mcu<J::k444>{}); break;
    default: f(J::Mcu<J::kGray>{}); break;
    }
}

// The call's frame table (fr, uploaded to st->d_frames) and the quantised coefficients of every block in st->d_coef, on
// stream s; *blocks_out = the blocks of the call.  Host frames are uploaded first.
int transform(J::State* st, cudaStream_t s, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const Opts& o,
              std::vector<J::Frame>& fr, long long* blocks_out) {
    int bpm = 0, mw = 0, mh = 0, strip = 0;
    by_shape(o.shape, [&](auto m) {
        using M = decltype(m);
        bpm = M::blocks; mw = 8 * M::h; mh = 8 * M::v; strip = M::strip;
    });
    const int channels = o.shape == J::kGray ? 1 : 3;
    fr.assign(n, J::Frame{});
    long long ctas = 0, blocks = 0, segs = 0;
    size_t in_bytes = 0;
    for (int i = 0; i < n; ++i) {
        J::Frame& f = fr[i];
        f.H = hw[2 * i]; f.W = hw[2 * i + 1];
        f.mcux = (f.W + mw - 1) / mw; f.mcuy = (f.H + mh - 1) / mh;
        f.strips = (f.mcux + strip - 1) / strip;
        const int mcus = f.mcux * f.mcuy;
        f.rst = o.restart ? std::min(o.restart, mcus) : mcus;
        f.nseg = (mcus + f.rst - 1) / f.rst;
        f.hdr = 0;
        f.cta0 = ctas; f.blk0 = blocks; f.seg0 = segs;
        ctas += (long long)f.strips * f.mcuy;
        blocks += (long long)bpm * mcus;
        segs += f.nseg;
        in_bytes += (size_t)f.H * f.W * channels;
        f.src = frames[i];
    }
    if (!frames_are_device) {
        if (int rc = grow(st->d_in, st->in_cap, in_bytes)) return rc;
        size_t off = 0;
        for (int i = 0; i < n; ++i) {
            const size_t b = (size_t)fr[i].H * fr[i].W * channels;
            JCK(cudaMemcpyAsync(st->d_in + off, frames[i], b, cudaMemcpyHostToDevice, s));
            fr[i].src = st->d_in + off;
            off += b;
        }
    }
    J::Quant qt;
    for (int c = 0; c < 2; ++c) {
        int q[64];
        quant_table(c ? o.chroma_quality : o.quality, c, q);
        for (int k = 0; k < 64; ++k) qt.q8[c][k] = (uint16_t)(8 * q[k]);
    }
    if (int rc = grow(st->d_coef, st->coef_cap, (size_t)blocks * 64)) return rc;
    JCK(cudaMemcpyAsync(st->d_frames, fr.data(), n * sizeof(J::Frame), cudaMemcpyHostToDevice, s));
    by_shape(o.shape, [&](auto m) {
        J::jpeg_transform_kernel<decltype(m)::kShape><<<(unsigned)ctas, J::kTransformThreads, 0, s>>>(st->d_frames, n, qt, st->d_coef);
    });
    JCK(cudaGetLastError());
    *blocks_out = blocks;
    return 0;
}

int encode(J::Target t, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const Opts& o,
           const uint8_t** data_out, int64_t* offsets_out) {
    JCK(cudaSetDevice(t.device));
    if (!*t.state)
        if (int rc = create(*t.state)) return rc;
    J::State* st = *t.state;
    const cudaStream_t s = t.stream;
    int bpm = 0, tables = 0;
    by_shape(o.shape, [&](auto m) {
        using M = decltype(m);
        bpm = M::blocks; tables = M::tables;
    });
    std::vector<J::Frame> fr;
    long long blocks = 0;
    if (int rc = transform(st, s, frames, hw, n, frames_are_device, o, fr, &blocks)) return rc;
    const long long segs = fr[n - 1].seg0 + fr[n - 1].nseg;
    if (int rc = grow(st->d_bits, st->bits_cap, (size_t)blocks)) return rc;
    if (int rc = grow(st->d_excl, st->excl_cap, (size_t)blocks + 1)) return rc;
    if (int rc = grow(st->d_segc, st->segc_cap, (size_t)segs)) return rc;
    if (int rc = grow(st->d_segx, st->segx_cap, (size_t)segs + 1)) return rc;

    // optimised tables from the frames' own symbols; bit lengths, bit offsets, chunks per segment
    const unsigned code_grid = (unsigned)((blocks + J::kCodeThreads - 1) / J::kCodeThreads);
    const uint32_t* huff = st->d_huff;
    int huff_stride = 0;
    if (o.optimize) {
        if (!st->d_hist) {
            JCK(cudaMalloc(&st->d_hist, J::kMaxFrames * 1024 * sizeof(int)));
            JCK(cudaMalloc(&st->d_ohuff, J::kMaxFrames * 1024 * sizeof(uint32_t)));
            JCK(cudaMalloc(&st->d_dht, J::kMaxFrames * 4 * J::kDhtBytes));
            JCK(cudaHostAlloc((void**)&st->h_dht, J::kMaxFrames * 4 * J::kDhtBytes, cudaHostAllocDefault));
        }
        JCK(cudaMemsetAsync(st->d_hist, 0, (size_t)n * 1024 * sizeof(int), s));
        JCK(cudaMemsetAsync(st->d_dht, 0, (size_t)n * 4 * J::kDhtBytes, s));
        by_shape(o.shape, [&](auto m) {
            J::jpeg_code_kernel<2, decltype(m)::kShape><<<code_grid, J::kCodeThreads, 0, s>>>(st->d_frames, n, blocks, st->d_coef, nullptr, 0, nullptr,
                                                                                             nullptr, nullptr, nullptr, st->d_hist);
        });
        J::jpeg_huff_build_kernel<<<n * tables, 32, 0, s>>>(st->d_hist, tables, st->d_ohuff, st->d_dht);
        huff = st->d_ohuff;
        huff_stride = 1024;
    }
    by_shape(o.shape, [&](auto m) {
        J::jpeg_code_kernel<0, decltype(m)::kShape><<<code_grid, J::kCodeThreads, 0, s>>>(st->d_frames, n, blocks, st->d_coef, huff, huff_stride,
                                                                                         st->d_bits, nullptr, nullptr, nullptr, nullptr);
    });
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_bits, blocks, st->d_excl)) return rc;
    J::jpeg_seg_chunks_kernel<<<(unsigned)((segs + 255) / 256), 256, 0, s>>>(st->d_frames, n, segs, bpm, st->d_excl, st->d_segc);
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_segc, segs, st->d_segx)) return rc;
    JCK(cudaMemcpyAsync(st->h_small, st->d_segx + segs, sizeof(long long), cudaMemcpyDeviceToHost, s));
    if (o.optimize) JCK(cudaMemcpyAsync(st->h_dht, st->d_dht, (size_t)n * 4 * J::kDhtBytes, cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));
    const long long chunks = st->h_small[0];
    uint8_t hdr[kMaxHeaderBytes];
    for (int i = 0; i < n; ++i) {
        const uint8_t* dht = o.optimize ? st->h_dht + (size_t)i * 4 * J::kDhtBytes : nullptr;
        if (dht && dht[0] == 0xFF) return fail(WHENET_EINVAL, "frame %d: an optimised Huffman code is longer than 32 bits", i);
        fr[i].hdr = header_bytes(fr[i].H, fr[i].W, o, dht, hdr);
    }

    // the codes, then 0x00 after every 0xFF and RSTm between segments
    if (int rc = grow(st->d_raw, st->raw_cap, (size_t)chunks * J::kChunk / 4)) return rc;
    JCK(cudaMemsetAsync(st->d_raw, 0, (size_t)chunks * J::kChunk, s));
    JCK(cudaMemcpyAsync(st->d_frames, fr.data(), n * sizeof(J::Frame), cudaMemcpyHostToDevice, s));
    by_shape(o.shape, [&](auto m) {
        J::jpeg_code_kernel<1, decltype(m)::kShape><<<code_grid, J::kCodeThreads, 0, s>>>(st->d_frames, n, blocks, st->d_coef, huff, huff_stride,
                                                                                         nullptr, st->d_excl, st->d_segx, st->d_raw, nullptr);
    });
    if (int rc = grow(st->d_ffc, st->ffc_cap, (size_t)chunks)) return rc;
    if (int rc = grow(st->d_ffx, st->ffx_cap, (size_t)chunks + 1)) return rc;
    const unsigned chunk_grid = (unsigned)((chunks + 255) / 256);
    const uint4* raw4 = reinterpret_cast<const uint4*>(st->d_raw);
    J::jpeg_out_count_kernel<<<chunk_grid, 256, 0, s>>>(st->d_frames, n, st->d_segx, segs, bpm, st->d_excl, raw4, chunks, st->d_ffc);
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_ffc, chunks, st->d_ffx)) return rc;
    J::jpeg_place_kernel<<<1, 32, 0, s>>>(st->d_frames, n, st->d_segx, st->d_ffx, st->d_small);
    JCK(cudaGetLastError());
    JCK(cudaMemcpyAsync(st->h_small, st->d_small, (n + 1) * sizeof(long long), cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));
    const long long total = st->h_small[n];
    if (int rc = grow(st->d_out, st->out_cap, (size_t)total)) return rc;
    J::jpeg_stuff_kernel<<<chunk_grid, 256, 0, s>>>(st->d_frames, n, st->d_segx, segs, bpm, st->d_excl, raw4, chunks, st->d_ffx, st->d_small,
                                                    st->d_out);
    JCK(cudaGetLastError());
    if (int rc = grow_host(st->h_out, st->h_cap, (size_t)total)) return rc;
    JCK(cudaMemcpyAsync(st->h_out, st->d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));

    // the host frames each stream: header before, EOI after
    for (int i = 0; i <= n; ++i) offsets_out[i] = st->h_small[i];
    for (int i = 0; i < n; ++i) {
        header_bytes(fr[i].H, fr[i].W, o, o.optimize ? st->h_dht + (size_t)i * 4 * J::kDhtBytes : nullptr, st->h_out + offsets_out[i]);
        st->h_out[offsets_out[i + 1] - 2] = 0xFF;
        st->h_out[offsets_out[i + 1] - 1] = 0xD9;
    }
    *data_out = st->h_out;
    return 0;
}

// ---- progressive files (DESIGN.md section 8.12)
// libjpeg's jpeg_simple_progression: (component, -1 for all; Ss, Se, Ah, Al)
struct ScanDef {
    int comp, Ss, Se, Ah, Al;
};
const ScanDef kScriptColor[10] = {{-1, 0, 0, 0, 1}, {0, 1, 5, 0, 2},  {2, 1, 63, 0, 1}, {1, 1, 63, 0, 1}, {0, 6, 63, 0, 2},
                                  {0, 1, 63, 2, 1}, {-1, 0, 0, 1, 0}, {2, 1, 63, 1, 0}, {1, 1, 63, 1, 0}, {0, 1, 63, 1, 0}};
const ScanDef kScriptGray[6] = {{-1, 0, 0, 0, 1}, {0, 1, 5, 0, 2}, {0, 6, 63, 0, 2}, {0, 1, 63, 2, 1}, {-1, 0, 0, 1, 0}, {0, 1, 63, 1, 0}};
constexpr int kMaxScans = 10, kMaxSlots = 10;      // per frame: scans, optimal tables
constexpr int kMaxScanHeaderBytes = 2 * (4 + J::kDhtBytes + 1) + 6 + 14;

// One scan's DHTs (its optimal tables, dht = slot p.slot's kDhtBytes; none for DC refinement), DRI before the first scan when
// restarts, and SOS.  Returns the bytes written.
int scan_header(const ScanDef& d, int nc, int restart, bool first, const uint8_t* dht, uint8_t* out) {
    uint8_t* p = out;
    auto seg = [&](uint8_t marker, int len) { *p++ = 0xFF; *p++ = marker; *p++ = (uint8_t)((len + 2) >> 8); *p++ = (uint8_t)(len + 2); };
    if (!(d.Ss == 0 && d.Ah)) {
        const int ntab = d.Ss == 0 ? (nc == 3 ? 2 : 1) : 1;
        for (int t = 0; t < ntab; ++t) {
            const uint8_t* counts = dht + t * J::kDhtBytes;
            int nsym = 0;
            for (int i = 0; i < 16; ++i) nsym += counts[i];
            seg(0xC4, 17 + nsym);
            *p++ = (uint8_t)(d.Ss == 0 ? t : 0x10 | (d.comp == 0 ? 0 : 1));
            memcpy(p, counts, 16 + nsym); p += 16 + nsym;
        }
    }
    if (first && restart) {
        seg(0xDD, 2);
        *p++ = (uint8_t)(restart >> 8); *p++ = (uint8_t)restart;
    }
    const int ns = d.comp < 0 ? nc : 1;
    seg(0xDA, 4 + 2 * ns);
    *p++ = (uint8_t)ns;
    for (int i = 0; i < ns; ++i) {
        const int c = d.comp < 0 ? i : d.comp, t = c == 0 ? 0 : 1;
        *p++ = (uint8_t)(c + 1);
        *p++ = (uint8_t)(d.Ss ? t : d.Ah ? 0 : t << 4);
    }
    *p++ = (uint8_t)d.Ss; *p++ = (uint8_t)d.Se; *p++ = (uint8_t)(d.Ah << 4 | d.Al);
    return (int)(p - out);
}

// The progressive files: the baseline transform, then every scan of every frame coded by the jpeg_prog_* kernels with its own
// optimal tables.  For placement and stuffing each scan is a Frame (pf) of the baseline kernels whose header is its DHT, DRI
// and SOS bytes and whose two closing bytes are the next scan's first two, or EOI: a frame's first scan also carries SOI ..
// SOF2, and a later scan's header is two bytes shorter.  The same three synchronisations as the baseline call.
int encode_progressive(J::Target t, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, const Opts& o,
                       const uint8_t** data_out, int64_t* offsets_out) {
    JCK(cudaSetDevice(t.device));
    if (!*t.state)
        if (int rc = create(*t.state)) return rc;
    J::State* st = *t.state;
    const cudaStream_t s = t.stream;
    const bool gray = o.shape == J::kGray;
    const int nc = gray ? 1 : 3, ns = gray ? 6 : 10;
    const ScanDef* script = gray ? kScriptGray : kScriptColor;
    int slots = 0;          // tables per frame
    for (int k = 0; k < ns; ++k) slots += script[k].Ss == 0 ? (script[k].Ah ? 0 : nc == 3 ? 2 : 1) : 1;

    std::vector<J::Frame> fr;
    long long blocks = 0;
    if (int rc = transform(st, s, frames, hw, n, frames_are_device, o, fr, &blocks)) return rc;
    const int nv = n * ns;
    std::vector<J::ProgScan> ps(nv);
    std::vector<J::Frame> pf(nv);
    long long units = 0, segs = 0;
    for (int i = 0; i < n; ++i) {
        const int mcus = fr[i].mcux * fr[i].mcuy, bw = (fr[i].W + 7) / 8, bh = (fr[i].H + 7) / 8;
        int slot = i * slots;
        for (int k = 0; k < ns; ++k) {
            const ScanDef& d = script[k];
            J::ProgScan& p = ps[i * ns + k];
            p.units = d.comp == 0 ? bw * bh : mcus;       // a one-component luma scan skips the dummy blocks
            p.rst = o.restart ? std::min(o.restart, p.units) : p.units;
            p.u0 = units; p.blk0 = fr[i].blk0; p.seg0 = segs;
            p.mcux = fr[i].mcux; p.bw = bw;
            p.slot = d.Ss == 0 && d.Ah ? -1 : slot;
            slot += d.Ss == 0 ? (d.Ah ? 0 : nc == 3 ? 2 : 1) : 1;
            p.comp = d.comp; p.Ss = d.Ss; p.Se = d.Se; p.Ah = d.Ah; p.Al = d.Al;
            J::Frame& f = pf[i * ns + k];
            f = J::Frame{};
            f.mcux = p.units; f.mcuy = 1; f.rst = p.rst;
            f.nseg = (p.units + p.rst - 1) / p.rst;
            f.blk0 = p.u0; f.seg0 = p.seg0;
            units += p.units;
            segs += f.nseg;
        }
    }
    if (!st->d_pscans) {
        JCK(cudaMalloc(&st->d_pscans, J::kMaxFrames * kMaxScans * sizeof(J::ProgScan)));
        JCK(cudaMalloc(&st->d_pframes, J::kMaxFrames * kMaxScans * sizeof(J::Frame)));
        JCK(cudaMalloc(&st->d_psmall, (J::kMaxFrames * kMaxScans + 1) * sizeof(long long)));
        JCK(cudaHostAlloc((void**)&st->h_psmall, (J::kMaxFrames * kMaxScans + 1) * sizeof(long long), cudaHostAllocDefault));
        JCK(cudaMalloc(&st->d_phist, J::kMaxFrames * kMaxSlots * 256 * sizeof(int)));
        JCK(cudaMalloc(&st->d_phuff, J::kMaxFrames * kMaxSlots * 256 * sizeof(uint32_t)));
        JCK(cudaMalloc(&st->d_pdht, J::kMaxFrames * kMaxSlots * J::kDhtBytes));
        JCK(cudaHostAlloc((void**)&st->h_pdht, J::kMaxFrames * kMaxSlots * J::kDhtBytes, cudaHostAllocDefault));
    }
    if (int rc = grow(st->d_bits, st->bits_cap, (size_t)units)) return rc;
    if (int rc = grow(st->d_excl, st->excl_cap, (size_t)units + 1)) return rc;
    if (int rc = grow(st->d_pemit, st->pemit_cap, (size_t)units)) return rc;
    if (int rc = grow(st->d_pjoin, st->pjoin_cap, (size_t)units)) return rc;
    if (int rc = grow(st->d_peob, st->peob_cap, (size_t)units)) return rc;
    if (int rc = grow(st->d_pemitx, st->pemitx_cap, (size_t)units + 1)) return rc;
    if (int rc = grow(st->d_segc, st->segc_cap, (size_t)segs)) return rc;
    if (int rc = grow(st->d_segx, st->segx_cap, (size_t)segs + 1)) return rc;
    JCK(cudaMemcpyAsync(st->d_pscans, ps.data(), nv * sizeof(J::ProgScan), cudaMemcpyHostToDevice, s));
    JCK(cudaMemcpyAsync(st->d_pframes, pf.data(), nv * sizeof(J::Frame), cudaMemcpyHostToDevice, s));

    // flags; EOB run pieces; per-scan tables; bit lengths, bit offsets, chunks per segment
    const unsigned grid = (unsigned)((units + J::kCodeThreads - 1) / J::kCodeThreads);
    auto code = [&](auto mode) {
        by_shape(o.shape, [&](auto m) {
            J::jpeg_prog_code_kernel<decltype(mode)::value, decltype(m)::kShape><<<grid, J::kCodeThreads, 0, s>>>(
                st->d_pscans, nv, units, st->d_coef, st->d_phuff, st->d_bits, st->d_pemit, st->d_pjoin, st->d_peob, st->d_excl, st->d_segx,
                st->d_raw, st->d_phist);
        });
    };
    code(std::integral_constant<int, J::kProgShape>{});
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_bits, units, st->d_excl)) return rc;
    if (int rc = scan(st, s, st->d_pemit, units, st->d_pemitx)) return rc;
    J::jpeg_prog_partition_kernel<<<(unsigned)((units + 255) / 256), 256, 0, s>>>(st->d_pscans, nv, units, st->d_pemit, st->d_pjoin, st->d_excl,
                                                                                  st->d_pemitx, st->d_peob);
    JCK(cudaMemsetAsync(st->d_phist, 0, (size_t)n * slots * 256 * sizeof(int), s));
    JCK(cudaMemsetAsync(st->d_pdht, 0, (size_t)n * slots * J::kDhtBytes, s));
    code(std::integral_constant<int, J::kProgHist>{});
    // slot q's histogram, table and DHT bytes are at q * 256 and q * kDhtBytes: the layout of (frame q / 4, table q % 4)
    J::jpeg_huff_build_kernel<<<n * slots, 32, 0, s>>>(st->d_phist, 4, st->d_phuff, st->d_pdht);
    code(std::integral_constant<int, J::kProgBits>{});
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_bits, units, st->d_excl)) return rc;
    J::jpeg_seg_chunks_kernel<<<(unsigned)((segs + 255) / 256), 256, 0, s>>>(st->d_pframes, nv, segs, 1, st->d_excl, st->d_segc);
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_segc, segs, st->d_segx)) return rc;
    JCK(cudaMemcpyAsync(st->h_psmall, st->d_segx + segs, sizeof(long long), cudaMemcpyDeviceToHost, s));
    JCK(cudaMemcpyAsync(st->h_pdht, st->d_pdht, (size_t)n * slots * J::kDhtBytes, cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));
    const long long chunks = st->h_psmall[0];
    uint8_t hdr[kMaxHeaderBytes + kMaxScanHeaderBytes];
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < ns; ++k) {
            const J::ProgScan& p = ps[i * ns + k];
            const uint8_t* dht = p.slot >= 0 ? st->h_pdht + (size_t)p.slot * J::kDhtBytes : nullptr;
            if (dht && (dht[0] == 0xFF || (script[k].Ss == 0 && nc == 3 && dht[J::kDhtBytes] == 0xFF)))
                return fail(WHENET_EINVAL, "frame %d scan %d: an optimal Huffman code is longer than 32 bits", i, k);
            pf[i * ns + k].hdr = scan_header(script[k], nc, o.restart, k == 0, dht, hdr) +
                                 (k == 0 ? frame_header(fr[i].H, fr[i].W, o, 0xC2, hdr) : -2);
        }

    // the codes, then 0x00 after every 0xFF and RSTm between segments
    if (int rc = grow(st->d_raw, st->raw_cap, (size_t)chunks * J::kChunk / 4)) return rc;
    JCK(cudaMemsetAsync(st->d_raw, 0, (size_t)chunks * J::kChunk, s));
    JCK(cudaMemcpyAsync(st->d_pframes, pf.data(), nv * sizeof(J::Frame), cudaMemcpyHostToDevice, s));
    code(std::integral_constant<int, J::kProgEmit>{});
    if (int rc = grow(st->d_ffc, st->ffc_cap, (size_t)chunks)) return rc;
    if (int rc = grow(st->d_ffx, st->ffx_cap, (size_t)chunks + 1)) return rc;
    const unsigned chunk_grid = (unsigned)((chunks + 255) / 256);
    const uint4* raw4 = reinterpret_cast<const uint4*>(st->d_raw);
    J::jpeg_out_count_kernel<<<chunk_grid, 256, 0, s>>>(st->d_pframes, nv, st->d_segx, segs, 1, st->d_excl, raw4, chunks, st->d_ffc);
    JCK(cudaGetLastError());
    if (int rc = scan(st, s, st->d_ffc, chunks, st->d_ffx)) return rc;
    J::jpeg_place_kernel<<<1, 32, 0, s>>>(st->d_pframes, nv, st->d_segx, st->d_ffx, st->d_psmall);
    JCK(cudaGetLastError());
    JCK(cudaMemcpyAsync(st->h_psmall, st->d_psmall, (nv + 1) * sizeof(long long), cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));
    const long long total = st->h_psmall[nv];
    if (int rc = grow(st->d_out, st->out_cap, (size_t)total)) return rc;
    J::jpeg_stuff_kernel<<<chunk_grid, 256, 0, s>>>(st->d_pframes, nv, st->d_segx, segs, 1, st->d_excl, raw4, chunks, st->d_ffx, st->d_psmall,
                                                    st->d_out);
    JCK(cudaGetLastError());
    if (int rc = grow_host(st->h_out, st->h_cap, (size_t)total)) return rc;
    JCK(cudaMemcpyAsync(st->h_out, st->d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
    JCK(cudaStreamSynchronize(s));

    // the host writes the headers between the scans' streams, and EOI
    for (int i = 0; i < n; ++i) {
        offsets_out[i] = st->h_psmall[i * ns];
        for (int k = 0; k < ns; ++k) {
            const J::ProgScan& p = ps[i * ns + k];
            uint8_t* d = st->h_out + st->h_psmall[i * ns + k] - (k ? 2 : 0);
            if (k == 0) d += frame_header(fr[i].H, fr[i].W, o, 0xC2, d);
            scan_header(script[k], nc, o.restart, k == 0, p.slot >= 0 ? st->h_pdht + (size_t)p.slot * J::kDhtBytes : nullptr, d);
        }
        const long long end = st->h_psmall[(i + 1) * ns];
        st->h_out[end - 2] = 0xFF;
        st->h_out[end - 1] = 0xD9;
    }
    offsets_out[n] = st->h_psmall[nv];
    *data_out = st->h_out;
    return 0;
}

// Checks the options of one call (channels 1 or 3) and fills o; WHENET_EINVAL otherwise.
int check_options(int channels, const whenet_jpeg_options* opts, Opts& o) {
    if (channels != 1 && channels != 3) return fail(WHENET_EINVAL, "channels %d is neither 1 nor 3", channels);
    if (!opts) return fail(WHENET_EINVAL, "null options");
    const whenet_jpeg_options& p = *opts;
    if (p.quality < 1 || p.quality > 100) return fail(WHENET_EINVAL, "quality %d outside [1, 100]", p.quality);
    if (p.chroma_quality < 1 || p.chroma_quality > 100) return fail(WHENET_EINVAL, "chroma_quality %d outside [1, 100]", p.chroma_quality);
    if (p.sampling != 420 && p.sampling != 422 && p.sampling != 444) return fail(WHENET_EINVAL, "sampling %d is not 420, 422 or 444", p.sampling);
    if (p.restart_interval < 0 || p.restart_interval > 65535) return fail(WHENET_EINVAL, "restart_interval %d outside [0, 65535]", p.restart_interval);
    if (p.optimize != 0 && p.optimize != 1) return fail(WHENET_EINVAL, "optimize %d is neither 0 nor 1", p.optimize);
    if (p.progressive != 0 && p.progressive != 1) return fail(WHENET_EINVAL, "progressive %d is neither 0 nor 1", p.progressive);
    if (channels == 1 && (p.sampling != 420 || p.chroma_quality != p.quality))
        return fail(WHENET_EINVAL, "one-channel frames take sampling 420 and chroma_quality = quality (a gray file has no chroma)");
    if (p.chroma_quality != p.quality && p.sampling != 444)
        return fail(WHENET_EINVAL, "chroma_quality %d != quality %d needs sampling 444 (libjpeg codes it as 4:4:4)", p.chroma_quality, p.quality);
    o.quality = p.quality;
    o.chroma_quality = p.chroma_quality;
    o.shape = channels == 1 ? J::kGray : p.sampling == 420 ? J::k420 : p.sampling == 422 ? J::k422 : J::k444;
    o.restart = p.restart_interval;
    o.optimize = p.optimize;
    o.progressive = p.progressive;
    return 0;
}

int encode_checked(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int channels, int frames_are_device,
                   const whenet_jpeg_options* opts, const uint8_t** data_out, int64_t* offsets_out) {
    // the context is checked last so that every other argument can be validated without a GPU
    if (n < 1 || n > J::kMaxFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, J::kMaxFrames);
    for (int i = 0; i < n; ++i) {
        if (!frames[i]) return fail(WHENET_EINVAL, "frame %d is NULL", i);
        if (hw[2 * i] < 1 || hw[2 * i + 1] < 1 || hw[2 * i] > 16384 || hw[2 * i + 1] > 16384)
            return fail(WHENET_EINVAL, "frame %d: bad frame size %dx%d", i, hw[2 * i + 1], hw[2 * i]);
    }
    Opts o;
    if (int rc = check_options(channels, opts, o)) return rc;
    if (!data_out || !offsets_out) return fail(WHENET_EINVAL, "null data_out or offsets_out");
    if (!c) return fail(WHENET_EINVAL, "null context");
    if (o.progressive) return encode_progressive(J::target(c), frames, hw, n, frames_are_device, o, data_out, offsets_out);
    return encode(J::target(c), frames, hw, n, frames_are_device, o, data_out, offsets_out);
}

whenet_jpeg_options default_options(int quality) { return whenet_jpeg_options{quality, quality, 420, 0, 0, 0}; }

}  // namespace

namespace whenet {
namespace jpeg {

int dec_state(Target t, DecState**& slot) {
    JCK(cudaSetDevice(t.device));
    if (!*t.state)
        if (int rc = create(*t.state)) return rc;
    slot = &(*t.state)->dec;
    return 0;
}

void destroy(State* st) {
    if (!st) return;
    destroy_dec(st->dec);
    for (void* p : {(void*)st->d_huff, (void*)st->d_ohuff, (void*)st->d_hist, (void*)st->d_dht, (void*)st->d_frames, (void*)st->d_small,
                    (void*)st->d_in, (void*)st->d_coef, (void*)st->d_bits, (void*)st->d_excl, (void*)st->d_segc, (void*)st->d_segx,
                    (void*)st->d_tiles, (void*)st->d_raw, (void*)st->d_ffc, (void*)st->d_ffx, (void*)st->d_out, (void*)st->d_pscans,
                    (void*)st->d_pframes, (void*)st->d_psmall, (void*)st->d_phist, (void*)st->d_phuff, (void*)st->d_pdht, (void*)st->d_pemit,
                    (void*)st->d_pjoin, (void*)st->d_peob, (void*)st->d_pemitx})
        if (p) cudaFree(p);
    if (st->h_small) cudaFreeHost(st->h_small);
    if (st->h_psmall) cudaFreeHost(st->h_psmall);
    if (st->h_pdht) cudaFreeHost(st->h_pdht);
    if (st->h_dht) cudaFreeHost(st->h_dht);
    if (st->h_out) cudaFreeHost(st->h_out);
    delete st;
}

}  // namespace jpeg
}  // namespace whenet

extern "C" {

int whenet_encode_jpeg_u8(whenet_ctx* c, const uint8_t* frames, int n, int H, int W, int frames_are_device, int quality,
                          const uint8_t** data_out, int64_t* offsets_out) {
    if (!frames) return fail(WHENET_EINVAL, "null frames");
    if (n < 1 || n > J::kMaxFrames) return fail(WHENET_EINVAL, "n=%d frames outside [1, %d]", n, J::kMaxFrames);
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    const uint8_t* ptrs[J::kMaxFrames];
    int32_t hw[2 * J::kMaxFrames];
    for (int i = 0; i < n; ++i) {
        ptrs[i] = frames + (size_t)i * H * W * 3;
        hw[2 * i] = H; hw[2 * i + 1] = W;
    }
    const whenet_jpeg_options o = default_options(quality);
    return encode_checked(c, ptrs, hw, n, 3, frames_are_device, &o, data_out, offsets_out);
}

int whenet_encode_jpeg_ragged_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device, int quality,
                                 const uint8_t** data_out, int64_t* offsets_out) {
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    const whenet_jpeg_options o = default_options(quality);
    return encode_checked(c, frames, hw, n, 3, frames_are_device, &o, data_out, offsets_out);
}

int whenet_encode_jpeg_ex_u8(whenet_ctx* c, const uint8_t* const* frames, const int32_t* hw, int n, int channels, int frames_are_device,
                             const whenet_jpeg_options* opts, const uint8_t** data_out, int64_t* offsets_out) {
    if (!frames || !hw) return fail(WHENET_EINVAL, "null frames or hw");
    return encode_checked(c, frames, hw, n, channels, frames_are_device, opts, data_out, offsets_out);
}

int whenet_debug_jpeg_header(int H, int W, int quality, uint8_t* out, int cap, int* len) {
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    if (quality < 1 || quality > 100) return fail(WHENET_EINVAL, "quality %d outside [1, 100]", quality);
    constexpr int kDefaultHeaderBytes = 623;
    if (!out || !len || cap < kDefaultHeaderBytes) return fail(WHENET_EINVAL, "null out or len, or cap %d < %d", cap, kDefaultHeaderBytes);
    *len = header_bytes(H, W, Opts{quality, quality, J::k420, 0, 0, 0}, nullptr, out);
    return 0;
}

int whenet_debug_jpeg_header_ex(int H, int W, int channels, const whenet_jpeg_options* opts, uint8_t* out, int cap, int* len) {
    if (H < 1 || W < 1 || H > 16384 || W > 16384) return fail(WHENET_EINVAL, "bad frame size %dx%d", W, H);
    Opts o;
    if (int rc = check_options(channels, opts, o)) return rc;
    if (o.optimize) return fail(WHENET_EINVAL, "an optimised header depends on the frame's symbols");
    if (o.progressive) return fail(WHENET_EINVAL, "a progressive file's scan headers depend on the frame's symbols");
    uint8_t buf[kMaxHeaderBytes];
    const int n = header_bytes(H, W, o, nullptr, buf);
    if (!out || !len || cap < n) return fail(WHENET_EINVAL, "null out or len, or cap %d < %d", cap, n);
    memcpy(out, buf, n);
    *len = n;
    return 0;
}

int whenet_debug_jpeg_optimal_table(const int32_t* counts, uint8_t* bits_out, uint8_t* vals_out, int* nvals_out) {
    if (!counts || !bits_out || !vals_out || !nvals_out) return fail(WHENET_EINVAL, "null counts, bits_out, vals_out or nvals_out");
    for (int i = 0; i < 256; ++i)
        if (counts[i] < 0) return fail(WHENET_EINVAL, "counts[%d] = %d is negative", i, counts[i]);
    const int nv = gen_optimal_table(counts, bits_out, vals_out);
    if (nv < 0) return fail(WHENET_EINVAL, "a code would be longer than 32 bits");
    *nvals_out = nv;
    return 0;
}

int whenet_debug_jpeg_optimal_table_gpu(whenet_ctx* c, const int32_t* counts, uint8_t* bits_out, uint8_t* vals_out, int* nvals_out) {
    if (!counts || !bits_out || !vals_out || !nvals_out) return fail(WHENET_EINVAL, "null counts, bits_out, vals_out or nvals_out");
    for (int i = 0; i < 256; ++i)
        if (counts[i] < 0) return fail(WHENET_EINVAL, "counts[%d] = %d is negative", i, counts[i]);
    if (!c) return fail(WHENET_EINVAL, "null context");
    const J::Target t = J::target(c);
    JCK(cudaSetDevice(t.device));
    int* d_hist = nullptr;
    uint32_t* d_huff = nullptr;
    uint8_t* d_dht = nullptr;
    uint8_t dht[J::kDhtBytes];
    cudaError_t e = cudaMalloc(&d_hist, 1024 * sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc(&d_huff, 1024 * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc(&d_dht, 4 * J::kDhtBytes);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_hist, counts, 256 * sizeof(int), cudaMemcpyHostToDevice, t.stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_dht, 0, J::kDhtBytes, t.stream);
    if (e == cudaSuccess) {
        J::jpeg_huff_build_kernel<<<1, 32, 0, t.stream>>>(d_hist, 1, d_huff, d_dht);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(dht, d_dht, J::kDhtBytes, cudaMemcpyDeviceToHost, t.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(t.stream);
    cudaFree(d_hist); cudaFree(d_huff); cudaFree(d_dht);
    if (e != cudaSuccess) return fail(WHENET_ECUDA, "optimal table on the device: %s", cudaGetErrorString(e));
    if (dht[0] == 0xFF) return fail(WHENET_EINVAL, "a code would be longer than 32 bits");
    int nv = 0;
    for (int i = 0; i < 16; ++i) nv += dht[i];
    memcpy(bits_out, dht, 16);
    memcpy(vals_out, dht + 16, nv);
    *nvals_out = nv;
    return 0;
}

}  // extern "C"

#include "jpeg_decode.inc"
