// kernels_jpeg_dec.cuh - baseline / extended-sequential Huffman JPEG decoding into packed BGR frames, pixel-identical to
// cv2.imdecode(buf, cv2.IMREAD_COLOR) (libjpeg-turbo defaults: islow IDCT, fancy upsampling, EXIF orientation applied).
// DESIGN.md section 8.10.
//
// The parse, the Huffman state machine, the IDCT, the upsampling and the colour conversion are __host__ __device__ (or host)
// functions, so tools/jpeg_decode_dump.cu runs the same arithmetic on the CPU.  One call decodes up to 64 files of their own
// sizes; every kernel maps call-wide indices (16-byte chunks, intervals, subsequences, blocks, pixels) back to a file through
// the per-file table, so a file's pixels never depend on the other files.
//   jd_end_kernel / jd_unstuff_kernel<0, 1>               the first marker that ends the data; 0x00 stuffing and RSTn removed,
//                                                          RST numbers checked, each restart interval's start byte recorded
//   jd_frame_kernel / jd_interval_kernel                  per file: stream length, RST count, EOI; per interval: subsequences
//   jd_piece_kernel / jd_sync_kernel                       self-synchronising Huffman decode (Weissenberger & Schmidt): every
//                                                          subsequence decodes from a guessed state, then again from its
//                                                          predecessor's end state until no state changes
//   jd_check_kernel / jd_write_kernel                      per-interval block counts; coefficients written in natural order
//   jd_idct_kernel / jd_color_kernel                       dequantise + islow IDCT; fancy upsampling, YCbCr->BGR, orientation
// The reduced and gray modes (cv2's IMREAD_REDUCED_* and IMREAD_GRAYSCALE, DESIGN.md section 8.13) share every stage up to the
// coefficients; jd_idct_kernel<true> stores each component at its own IDCT size (8, 4, 2 or 1 samples square) and
// jd_color_kernel<kColorScaled / kColorGray> converts those planes.
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "kernels_jpeg.cuh"

#define JD_HD __host__ __device__ __forceinline__

namespace whenet {
namespace jpegdec {

constexpr int kMaxFrames = jpeg::kMaxFrames;
constexpr int kMaxSide = 16384;
constexpr int kChunk = 16;                 // bytes per unstuffing thread; every file's data starts on a chunk
constexpr int kDefaultPieceBits = 2048;    // subsequence length of the Huffman decode
constexpr int kMinPieceBits = 32, kMaxPieceBits = 65536;

// per-file status bits (whenet_decode_jpeg_u8's status_out)
constexpr int kStTruncated = 1;     // the data ends before EOI, or a code runs past the end of its interval
constexpr int kStRst = 2;           // a restart marker out of sequence, or too many or too few of them
constexpr int kStMarker = 4;        // a marker other than RSTn, APPn, COM or EOI in or after the entropy-coded data
constexpr int kStBadCode = 8;       // a bit pattern that is no Huffman code of its table
constexpr int kStRun = 16;          // an AC run past coefficient 63
constexpr int kStBlocks = 32;       // an interval codes more or fewer blocks than its MCUs hold

// Decoder state: (bit position, block slot in the MCU, zigzag index); two decodes that reach the same state agree from then
// on.  A decode that meets an error records its status bit and carries on (an invalid code skips one bit, a run past 63 ends
// the block, a code past the interval's end ends the decode there), so that a decode from a wrong guess can still meet the
// true state; the errors count only for the decode from a subsequence's final start state.
JD_HD uint64_t pack_state(long long pos, int slot, int zz) { return (uint64_t)pos << 16 | (uint64_t)slot << 8 | (uint64_t)zz; }

// Canonical Huffman table (T.81 Annex C / F.2.2.3): a 9-bit lookup, then maxcode / valoff for codes of 10..16 bits.
struct HuffTable {
    int32_t maxcode[17];    // largest code of each length, -1 if none
    int32_t valoff[17];     // symbol index = code + valoff[length]
    uint8_t val[256];
    uint16_t look[512];     // length << 8 | symbol for codes of <= 9 bits; 0: a longer code or none
};

struct Tables {
    HuffTable h[6];         // component c: h[2c] DC, h[2c + 1] AC
    uint16_t q[3][64];      // dequantisation per component, natural order
};

struct Header {             // what the host parse gives
    int H, W;               // coded size
    int oH, oW, orient;     // output size after the EXIF orientation (1..8)
    int ncomp, hs, vs;      // 1 or 3 components; luma sampling (chroma is 1 x 1)
    int mcux, mcuy, bpm;    // MCU grid; blocks per MCU
    int ri;                 // restart interval in MCUs, 0: none
    long long ecs;          // offset of the first entropy-coded byte in the file
    Tables t;
};

struct DecFrame {
    int H, W, oH, oW, orient, ncomp, hs, vs, mcux, mcuy, bpm, ri;
    long long nint;         // restart intervals
    int slot_comp[6], slot_dx[6], slot_dy[6];   // each MCU slot's component and block offset inside the MCU
    int pw[3], ph[3];       // component planes (whole MCUs)
    long long in0, in_len;  // the file's entropy-coded bytes in the call's input (in0 a multiple of kChunk)
    long long iv0;          // first interval in the call
    long long blk0, nblk;   // first block in the call; blocks
    long long plane0[3];    // component planes in the call's plane buffer
    long long pix0;         // first coded pixel in the call
    uint8_t* out;           // oH x oW x 3 BGR (x 1 in gray mode)
};

struct DecScaled {          // what the reduced and gray modes add to a DecFrame (frame_scaled)
    int sc[3];              // IDCT size of each component: 8, 4, 2 or 1
    int dH, dW;             // decoded size before the orientation: ceil(H / d) x ceil(W / d)
    int gray;               // the luma plane alone, oH x oW x 1
    int uh, uv;             // chroma upsampling factors (1 or 2) from its plane to dH x dW
    int cw, ch;             // chroma plane extent; cw = 1 where libjpeg replicates instead of fancy upsampling
};

struct Piece {              // one subsequence: frame-local bit range [start, end) of interval iv (call-wide), which ends at iend
    long long start, end, iend, iv;
    int f, first;
};

// ---------------------------------------------------------------------------------------------------- Huffman decoding
// 32 bits of the stream from bit pos, big-endian; bytes past nbytes read as 0xFF
JD_HD uint32_t peek32(const uint8_t* b, long long nbytes, long long pos) {
    const long long i = pos >> 3;
    uint64_t v = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) v = v << 8 | (i + k < nbytes ? b[i + k] : 0xFFu);
    return (uint32_t)(v >> (8 - (pos & 7)));
}

JD_HD int huff_decode(const HuffTable& t, uint32_t bits, int& sym) {
    const int e = t.look[bits >> 23];
    if (e) { sym = e & 0xff; return e >> 8; }
    for (int l = 10; l <= 16; ++l) {
        const int code = (int)(bits >> (32 - l));
        if (code <= t.maxcode[l]) { sym = t.val[(code + t.valoff[l]) & 0xff]; return l; }
    }
    return 0;
}

// the bits [pos, end) are all ones (the padding before a restart marker or EOI)
JD_HD bool all_ones(const uint8_t* b, long long nbytes, long long pos, long long end) {
    const int n = (int)(end - pos);
    return n <= 0 || (peek32(b, nbytes, pos) >> (32 - n)) == (1u << n) - 1;
}

struct PieceResult {
    uint64_t state;
    int nblocks;
    int dc[3];              // sums of the DC differences per component
    int err;                // status bits met on the way
};

// Decode the symbols that start in [state's position, end) of a stream whose interval ends at iend.  kWrite: coefficient k of
// the current block goes to coef[blk * 64 + natural[k]] while blk < blk_end, with DC predictions starting at pred0.
template <bool kWrite>
JD_HD PieceResult decode_piece(const DecFrame& fr, const Tables& t, const uint8_t* natural, const uint8_t* bytes, long long nbytes,
                               uint64_t in, long long end, long long iend, int16_t* coef, long long blk, long long blk_end,
                               const int* pred0) {
    PieceResult r{in, 0, {0, 0, 0}, 0};
    long long pos = (long long)(in >> 16);
    int slot = (int)(in >> 8) & 0xff, zz = (int)in & 0xff;
    // the DC sums and predictions stay in registers: the component selects them by branch, never by index
    int d0 = 0, d1 = 0, d2 = 0, p0 = 0, p1 = 0, p2 = 0;
    if (kWrite) { p0 = pred0[0]; p1 = pred0[1]; p2 = pred0[2]; }
    while (pos < end) {
        if (iend - pos < 8 && all_ones(bytes, nbytes, pos, iend)) { pos = iend; break; }
        const int c = fr.slot_comp[slot];
        const uint32_t bits = peek32(bytes, nbytes, pos);
        int sym;
        const int len = huff_decode(t.h[2 * c + (zz ? 1 : 0)], bits, sym);
        if (!len) { r.err |= kStBadCode; ++pos; continue; }
        const int run = zz ? sym >> 4 : 0, s = zz ? sym & 15 : sym;
        if (pos + len + s > iend) { r.err |= kStTruncated; pos = iend; break; }
        int v = 0;
        if (s) {
            v = (int)((bits << len) >> (32 - s));
            if (v < (1 << (s - 1))) v += (int)(~0u << s) + 1;     // HUFF_EXTEND
        }
        pos += len + s;
        if (zz == 0) {
            int pv;
            if (c == 0) { d0 += v; pv = p0 += v; }
            else if (c == 1) { d1 += v; pv = p1 += v; }
            else { d2 += v; pv = p2 += v; }
            if (kWrite && blk < blk_end) coef[blk * 64] = (int16_t)pv;
            zz = 1;
        } else if (s) {
            zz += run;
            if (zz > 63) {
                r.err |= kStRun;
                zz = 64;
            } else {
                if (kWrite && blk < blk_end) coef[blk * 64 + natural[zz]] = (int16_t)v;
                ++zz;
            }
        } else if (run == 15) {
            zz += 16;
            if (zz > 64) { r.err |= kStRun; zz = 64; }
        } else {
            zz = 64;        // EOB
        }
        if (zz == 64) {
            zz = 0;
            ++r.nblocks;
            ++blk;
            if (++slot == fr.bpm) slot = 0;
        }
    }
    r.dc[0] = d0; r.dc[1] = d1; r.dc[2] = d2;
    r.state = pack_state(pos, slot, zz);
    return r;
}

// ---------------------------------------------------------------------------------------------------- pixels
// libjpeg's islow IDCT (jidctint.c, CONST_BITS 13, PASS1_BITS 2), columns first, with the 16-bit steps of libjpeg-turbo's SIMD
// version, which cv2.imdecode runs (the numpy model in oracle/jpeg_decode_oracle.py pins each one against cv2):
//   - the coefficient x quantiser product is taken modulo 2^16;
//   - a block whose coefficient rows 1..7 are all zero skips the column pass: every workspace row is the dequantised row 0
//     shifted left by PASS1_BITS modulo 2^16;
//   - the pairwise sums d0 + d4, d0 - d4, d7 + d3 and d5 + d1 of both passes are taken modulo 2^16 (the other sums of the C
//     code are folded into 32-bit multiply-adds there, so they stay exact here);
//   - each pass saturates its descaled output to int16; the row pass then clamps to [-128, 127] and adds 128.
// No 32-bit sum can overflow: the largest, |tmp12 +- o1|, stays below 2^31 - 2^17 for any int16 inputs.  For coefficients an
// encoder makes from 8-bit samples nothing wraps or saturates, and the result is the C code's.
__host__ __device__ constexpr int c13(double x) { return (int)(x * 8192.0 + 0.5); }
JD_HD int s16(int x) { return (int)(int16_t)x; }

template <int kShift, typename In, typename F>
JD_HD void idct_pass(const In* d, int s, int16_t* o, int os, F load) {
    const int z2e = load(d[2 * s], 2), z3e = load(d[6 * s], 6);
    const int z1 = (z2e + z3e) * c13(0.541196100);
    const int tmp2 = z1 - z3e * c13(1.847759065), tmp3 = z1 + z2e * c13(0.765366865);
    const int a = load(d[0], 0), b = load(d[4 * s], 4);
    const int tmp0 = s16(a + b) * 8192, tmp1 = s16(a - b) * 8192;
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    int o0 = load(d[7 * s], 7), o1 = load(d[5 * s], 5), o2 = load(d[3 * s], 3), o3 = load(d[s], 1);
    int z1o = o0 + o3, z2o = o1 + o2, z3o = s16(o0 + o2), z4o = s16(o1 + o3);
    const int z5 = (z3o + z4o) * c13(1.175875602);
    o0 *= c13(0.298631336); o1 *= c13(2.053119869); o2 *= c13(3.072711026); o3 *= c13(1.501321110);
    z1o *= -c13(0.899976223); z2o *= -c13(2.562915447); z3o *= -c13(1.961570560); z4o *= -c13(0.390180644);
    z3o += z5; z4o += z5;
    o0 += z1o + z3o; o1 += z2o + z4o; o2 += z2o + z3o; o3 += z1o + z4o;
    auto put = [&](int i, int x) {
        const int v = (x + (1 << (kShift - 1))) >> kShift;
        o[i * os] = (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v);
    };
    put(0, tmp10 + o3); put(7, tmp10 - o3); put(1, tmp11 + o2); put(6, tmp11 - o2);
    put(2, tmp12 + o1); put(5, tmp12 - o1); put(3, tmp13 + o0); put(4, tmp13 - o0);
}

// column `col` of a block has a non-zero coefficient in rows 1..7 (no block with one takes the DC-only column pass)
JD_HD bool idct_column_ac(const int16_t* coef, int col) {
    int nz = 0;
#pragma unroll
    for (int r = 1; r < 8; ++r) nz |= coef[r * 8 + col];
    return nz != 0;
}
// column `col` of a block (natural-order coefficients) -> ws[col], ws[8 + col], ...; dc_only: no column of the block has a
// non-zero coefficient in rows 1..7
JD_HD void idct_column(const int16_t* coef, const uint16_t* q, int col, bool dc_only, int16_t* ws) {
    auto deq = [&](int16_t c, int row) { return s16(c * q[row * 8 + col]); };
    if (dc_only) {
        const int16_t v = (int16_t)(deq(coef[col], 0) * 4);
#pragma unroll
        for (int r = 0; r < 8; ++r) ws[r * 8 + col] = v;
    } else {
        idct_pass<13 - 2>(coef + col, 8, ws + col, 8, deq);
    }
}
// row `row` of the workspace -> 8 samples
JD_HD void idct_row(const int16_t* ws, int row, uint8_t* out) {
    int16_t v[8];
    idct_pass<13 + 2 + 3>(ws + row * 8, 1, v, 1, [](int16_t x, int) { return (int)x; });
    for (int i = 0; i < 8; ++i) out[i] = (uint8_t)(v[i] < -128 ? 0 : v[i] > 127 ? 255 : v[i] + 128);
}

// libjpeg's reduced IDCTs (jidctred.c: jpeg_idct_4x4, jpeg_idct_2x2, jpeg_idct_1x1), columns first, with the 16- and 32-bit
// steps of libjpeg-turbo's SSE2 versions, which cv2.imdecode runs (oracle/jpeg_scaled_decode_oracle.py pins each one):
//   - the coefficient x quantiser product is taken modulo 2^16;
//   - every multiply-add sum and its rounding constant are taken modulo 2^32 (each product of an int16 and a constant fits
//     an int32, so unsigned sums give the SIMD lanes' result), then shifted arithmetically;
//   - 4x4: a block whose coefficient rows 1, 2, 3, 5, 6, 7 are all zero skips the column pass (every workspace row is the
//     dequantised row 0 shifted left by PASS1_BITS modulo 2^16); otherwise the column pass saturates to int16;
//   - 2x2: columns 1, 3, 5, 7 of the column pass saturate to int16, column 0 stays 32-bit, and its row-pass even term
//     (<< 15) is taken modulo 2^32;
//   - the row pass saturates to int16, then clamps to [-128, 127] and adds 128.
// 4x4 reads no coefficient of row or column 4; 2x2 reads only rows and columns 0, 1, 3, 5 and 7.
JD_HD int desc32(uint32_t sum, int shift) { return (int)(sum + (1u << (shift - 1))) >> shift; }
JD_HD int16_t sat16(int v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }
JD_HD uint8_t clamp_sample(int v) { return (uint8_t)(v < -128 ? 0 : v > 127 ? 255 : v + 128); }

// 1-D 4-point transform of d[0], d[s], ... d[7 s] (index 4 unused) -> 4 descaled int32 outputs
template <typename In, typename F>
JD_HD void idct4_pass(const In* d, int s, int shift, F load, int* o) {
    const uint32_t t0 = (uint32_t)(load(d[0], 0) * 16384);
    const uint32_t t2 = (uint32_t)(load(d[2 * s], 2) * 15137) - (uint32_t)(load(d[6 * s], 6) * 6270);
    const int z1 = load(d[7 * s], 7), z2 = load(d[5 * s], 5), z3 = load(d[3 * s], 3), z4 = load(d[s], 1);
    const uint32_t o0 = (uint32_t)(z2 * 11893) + (uint32_t)(z4 * 8697) - (uint32_t)(z1 * 1730) - (uint32_t)(z3 * 17799);
    const uint32_t o2 = (uint32_t)(z3 * 7373) + (uint32_t)(z4 * 20995) - (uint32_t)(z1 * 4176) - (uint32_t)(z2 * 4926);
    o[0] = desc32(t0 + t2 + o2, shift);
    o[1] = desc32(t0 - t2 + o0, shift);
    o[2] = desc32(t0 - t2 - o0, shift);
    o[3] = desc32(t0 + t2 - o2, shift);
}
// the 2-point odd part of d[s], d[3 s], d[5 s], d[7 s]
template <typename In, typename F>
JD_HD uint32_t idct2_odd(const In* d, int s, F load) {
    return (uint32_t)(load(d[5 * s], 5) * 6967) + (uint32_t)(load(d[s], 1) * 29692) - (uint32_t)(load(d[7 * s], 7) * 5906) -
           (uint32_t)(load(d[3 * s], 3) * 10426);
}

// rows 1, 2, 3, 5, 6, 7 of column `col` hold a non-zero coefficient (no block with one takes the 4x4 shortcut)
JD_HD bool idct4_column_ac(const int16_t* coef, int col) {
    return (coef[8 + col] | coef[16 + col] | coef[24 + col] | coef[40 + col] | coef[48 + col] | coef[56 + col]) != 0;
}
// column `col` (not 4) of a block -> ws[col], ws[8 + col], ws[16 + col], ws[24 + col]
JD_HD void idct4_column(const int16_t* coef, const uint16_t* q, int col, bool dc_only, int16_t* ws) {
    auto deq = [&](int16_t c, int row) { return s16(c * q[row * 8 + col]); };
    if (dc_only) {
        const int16_t v = (int16_t)(deq(coef[col], 0) * 4);
        for (int r = 0; r < 4; ++r) ws[r * 8 + col] = v;
        return;
    }
    int o[4];
    idct4_pass(coef + col, 8, 13 - 2 + 1, deq, o);
    for (int r = 0; r < 4; ++r) ws[r * 8 + col] = sat16(o[r]);
}
// row `row` (0..3) of the workspace -> 4 samples
JD_HD void idct4_row(const int16_t* ws, int row, uint8_t* out) {
    int o[4];
    idct4_pass(ws + row * 8, 1, 13 + 2 + 3 + 1, [](int16_t x, int) { return (int)x; }, o);
    for (int i = 0; i < 4; ++i) out[i] = clamp_sample(sat16(o[i]));
}
// column `col` (0, 1, 3, 5 or 7) -> rows 0 and 1 of the workspace.  Column 0 keeps its 32-bit value, stored as two halves in
// columns 2 (low) and 4 (high), which the 2x2 IDCT never reads.
JD_HD void idct2_column(const int16_t* coef, const uint16_t* q, int col, int16_t* ws) {
    auto deq = [&](int16_t c, int row) { return s16(c * q[row * 8 + col]); };
    const uint32_t t10 = (uint32_t)(deq(coef[col], 0) * 32768), od = idct2_odd(coef + col, 8, deq);
    const int v[2] = {desc32(t10 + od, 13 - 2 + 2), desc32(t10 - od, 13 - 2 + 2)};
    for (int r = 0; r < 2; ++r) {
        if (col) {
            ws[r * 8 + col] = sat16(v[r]);
        } else {
            ws[r * 8 + 2] = (int16_t)(uint16_t)(uint32_t)v[r];
            ws[r * 8 + 4] = (int16_t)(uint16_t)((uint32_t)v[r] >> 16);
        }
    }
}
JD_HD void idct2_row(const int16_t* ws, int row, uint8_t* out) {
    const int16_t* w = ws + row * 8;
    const uint32_t c0 = (uint32_t)(uint16_t)w[2] | (uint32_t)(uint16_t)w[4] << 16;
    const uint32_t e = c0 << 15, od = idct2_odd(w, 1, [](int16_t x, int) { return (int)x; });
    out[0] = clamp_sample(sat16(desc32(e + od, 13 + 2 + 3 + 2)));
    out[1] = clamp_sample(sat16(desc32(e - od, 13 + 2 + 3 + 2)));
}
// DC only: (DC x q + 4) >> 3 through libjpeg's 1024-entry range-limit table (jdmaster.c, index masked by RANGE_MASK); the
// quantiser is a signed 16-bit multiplier there
JD_HD uint8_t idct1(const int16_t* coef, const uint16_t* q) {
    const int v = ((int)coef[0] * (int)(int16_t)q[0] + 4) >> 3;
    const int i = v & 1023;
    return (uint8_t)(i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896);
}

// one chroma sample at coded pixel (y, x) with libjpeg's fancy upsampling; the plane's real extent is cw x ch, replicated.
// libjpeg upsamples a chroma plane of width <= 2 by plain replication instead (jdsample.c).
JD_HD int chroma_at(const uint8_t* p, int pw, int cw, int ch, int hs, int vs, int y, int x) {
    if (hs == 1) return p[(size_t)y * pw + x];
    if (cw <= 2) return p[(size_t)(y / vs) * pw + (x >> 1)];
    const int cx = x >> 1, nx = (x & 1) ? (cx + 1 < cw ? cx + 1 : cw - 1) : (cx > 0 ? cx - 1 : 0);
    if (vs == 1) {
        const uint8_t* r = p + (size_t)y * pw;
        return (x & 1) ? (3 * r[cx] + r[nx] + 2) >> 2 : (3 * r[cx] + r[nx] + 1) >> 2;
    }
    const int cy = y >> 1, fy = (y & 1) ? (cy + 1 < ch ? cy + 1 : ch - 1) : (cy > 0 ? cy - 1 : 0);
    const uint8_t* near = p + (size_t)cy * pw;
    const uint8_t* far = p + (size_t)fy * pw;
    const int t = 3 * near[cx] + far[cx], n = 3 * near[nx] + far[nx];
    return (x & 1) ? (3 * t + n + 7) >> 4 : (3 * t + n + 8) >> 4;
}

// libjpeg's YCbCr -> RGB tables (jdcolor.c, 16 fraction bits), written as BGR
JD_HD void ycc_bgr(int y, int cb, int cr, uint8_t* o) {
    constexpr int kR = (int)(1.40200 * 65536 + 0.5), kB = (int)(1.77200 * 65536 + 0.5);
    constexpr int kGr = (int)(0.71414 * 65536 + 0.5), kGb = (int)(0.34414 * 65536 + 0.5);
    cb -= 128; cr -= 128;
    auto clamp = [](int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); };
    o[0] = clamp(y + ((kB * cb + 32768) >> 16));
    o[1] = clamp(y + ((-kGb * cb - kGr * cr + 32768) >> 16));
    o[2] = clamp(y + ((kR * cr + 32768) >> 16));
}

// where coded pixel (y, x) of an H x W image lands under EXIF orientation o (what cv2's flip / transpose sequence does)
JD_HD void orient_dst(int o, int H, int W, int y, int x, int& oy, int& ox) {
    switch (o) {
        case 2: oy = y; ox = W - 1 - x; break;
        case 3: oy = H - 1 - y; ox = W - 1 - x; break;
        case 4: oy = H - 1 - y; ox = x; break;
        case 5: oy = x; ox = y; break;
        case 6: oy = x; ox = H - 1 - y; break;
        case 7: oy = W - 1 - x; ox = H - 1 - y; break;
        case 8: oy = W - 1 - x; ox = y; break;
        default: oy = y; ox = x; break;
    }
}

// the BGR pixel of coded position (y, x), from the component planes
JD_HD void pixel_bgr(const DecFrame& fr, const uint8_t* planes, int y, int x, uint8_t* o) {
    const int yv = planes[fr.plane0[0] + (size_t)y * fr.pw[0] + x];
    if (fr.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)yv; return; }
    const int cw = (fr.W + fr.hs - 1) / fr.hs, ch = (fr.H + fr.vs - 1) / fr.vs;
    const int cb = chroma_at(planes + fr.plane0[1], fr.pw[1], cw, ch, fr.hs, fr.vs, y, x);
    const int cr = chroma_at(planes + fr.plane0[2], fr.pw[2], cw, ch, fr.hs, fr.vs, y, x);
    ycc_bgr(yv, cb, cr, o);
}

// the BGR pixel of decoded position (y, x) of a reduced frame: chroma without upsampling, or h2v1 / h2v2 (fancy, or replicated
// where cw says so)
JD_HD void pixel_bgr_scaled(const DecFrame& fr, const DecScaled& z, const uint8_t* planes, int y, int x, uint8_t* o) {
    const int yv = planes[fr.plane0[0] + (size_t)y * fr.pw[0] + x];
    if (fr.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)yv; return; }
    const int cb = chroma_at(planes + fr.plane0[1], fr.pw[1], z.cw, z.ch, z.uh, z.uv, y, x);
    const int cr = chroma_at(planes + fr.plane0[2], fr.pw[2], z.cw, z.ch, z.uh, z.uv, y, x);
    ycc_bgr(yv, cb, cr, o);
}

// block b (frame-local, scan order) -> component and its block position in the component plane
JD_HD int block_place(const DecFrame& fr, long long b, int& bx, int& by) {
    const long long mcu = b / fr.bpm;
    const int slot = (int)(b - mcu * fr.bpm), c = fr.slot_comp[slot];
    const int mx = (int)(mcu % fr.mcux), my = (int)(mcu / fr.mcux);
    const int h = c ? 1 : fr.hs, v = c ? 1 : fr.vs;
    bx = mx * h + fr.slot_dx[slot];
    by = my * v + fr.slot_dy[slot];
    return c;
}

// ---------------------------------------------------------------------------------------------------- host parse
// T.81 Annex K.3 tables: what libjpeg uses for a table slot 0 / 1 that no DHT defines (Motion-JPEG frames have none)
inline const uint8_t* std_counts(int ac, int chroma) {
    static const uint8_t k[2][2][16] = {{{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}},
                                        {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}}};
    return k[ac][chroma];
}
inline const uint8_t* std_syms(int ac, int chroma) {
    static const uint8_t dc[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
    static const uint8_t acs[2][162] = {
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
    return ac ? acs[chroma] : dc;
}

inline const uint8_t* natural_order_host() {
    static const uint8_t k[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                  41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                  30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return k;
}

// Refused: more than 256 symbols, a code of all ones (as libjpeg refuses them), and a DC symbol above 15, a category no 8-bit
// DC difference has (stricter than cv2, which decodes a file whose table holds such a symbol if the data never uses it)
inline const char* build_huff(const uint8_t counts[16], const uint8_t* syms, int dc, HuffTable& t) {
    memset(&t, 0, sizeof(t));
    int k = 0, code = 0;
    for (int l = 1; l <= 16; ++l) {
        const int n = counts[l - 1];
        if (k + n > 256) return "Huffman table with more than 256 codes";
        t.valoff[l] = k - code;
        t.maxcode[l] = n ? code + n - 1 : -1;
        for (int i = 0; i < n; ++i, ++k, ++code) {
            if (dc && syms[k] > 15) return "DC Huffman symbol above 15";
            t.val[k] = syms[k];
            if (l <= 9)
                for (int j = code << (9 - l); j < (code + 1) << (9 - l); ++j) t.look[j] = (uint16_t)(l << 8 | syms[k]);
        }
        if (code >= (1 << l)) return "Huffman table with an all-ones or overflowing code";
        code <<= 1;
    }
    return nullptr;
}

// OpenCV's ExifReader as cv2.imdecode applies it: the first APP1 after its 6-byte header is a TIFF block ("II" / "MM", 0x2A,
// IFD0); IFD0 entries are read until one would pass the end, and the first orientation entry (tag 0x0112) counts if in 1..8.
inline int exif_orientation(const uint8_t* d, size_t n) {
    if (n < 1) return 1;
    const bool intel = d[0] == 'I' && (n < 2 || d[1] == 'I');
    auto u16 = [&](size_t o, bool& ok) -> int {
        if (o + 1 >= n) { ok = false; return 0; }
        return intel ? d[o] | d[o + 1] << 8 : d[o] << 8 | d[o + 1];
    };
    auto u32 = [&](size_t o, bool& ok) -> uint32_t {
        if (o + 3 >= n) { ok = false; return 0; }
        return intel ? (uint32_t)d[o] | (uint32_t)d[o + 1] << 8 | (uint32_t)d[o + 2] << 16 | (uint32_t)d[o + 3] << 24
                     : (uint32_t)d[o] << 24 | (uint32_t)d[o + 1] << 16 | (uint32_t)d[o + 2] << 8 | (uint32_t)d[o + 3];
    };
    bool ok = true;
    if (u16(2, ok) != 0x2A || !ok) return 1;
    size_t off = u32(4, ok);
    if (!ok) return 1;
    const int entries = u16(off, ok);
    if (!ok) return 1;
    off += 2;
    for (int e = 0; e < entries; ++e, off += 12) {
        const int tag = u16(off, ok);
        if (!ok) return 1;
        if (tag == 0x0112) {
            const int v = u16(off + 8, ok);
            if (!ok) return 1;
            return v >= 1 && v <= 8 ? v : 1;
        }
    }
    return 1;
}

// Parse a file's markers up to its SOS.  Returns nullptr and fills h, or the reason the file is not decoded.
inline const char* parse_header(const uint8_t* d, size_t n, Header& h) {
    memset(&h, 0, sizeof(h));
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return "not a JPEG file (no SOI)";
    uint16_t qt[4][64];
    bool have_q[4] = {}, have_h[2][4] = {};
    uint8_t hcounts[2][4][16], hsyms[2][4][256];
    bool sof = false, jfif = false, adobe = false, app1 = false;
    int adobe_transform = 0, cid[3] = {}, ctq[3] = {}, hsamp[3] = {}, vsamp[3] = {};
    h.orient = 1;
    size_t p = 2;
    for (;;) {
        if (p >= n || d[p] != 0xFF) return "truncated or malformed marker segment";
        while (p < n && d[p] == 0xFF) ++p;
        if (p >= n) return "truncated marker segment";
        const int m = d[p++];
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
        if (m == 0xD8) return "a second SOI";
        if (m == 0xD9) return "EOI before any scan";
        if (p + 2 > n) return "truncated marker segment";
        const size_t len = (size_t)d[p] << 8 | d[p + 1];
        if (len < 2 || p + len > n) return "truncated marker segment";
        const uint8_t* s = d + p + 2;
        const size_t sl = len - 2;
        p += len;
        switch (m) {
            case 0xC0: case 0xC1: {
                if (sof) return "a second SOF";
                if (sl < 6) return "short SOF segment";
                if (s[0] != 8) return "not 8-bit (12-bit or other sample precision)";
                h.H = s[1] << 8 | s[2];
                h.W = s[3] << 8 | s[4];
                h.ncomp = s[5];
                if (h.H == 0) return "height defined by DNL";
                if (h.ncomp != 1 && h.ncomp != 3) return "not 1 or 3 components";
                if (sl < 6 + 3u * h.ncomp) return "short SOF segment";
                if (h.W < 1 || h.W > kMaxSide || h.H > kMaxSide) return "a side outside [1, 16384]";
                for (int c = 0; c < h.ncomp; ++c) {
                    cid[c] = s[6 + 3 * c];
                    hsamp[c] = s[7 + 3 * c] >> 4;
                    vsamp[c] = s[7 + 3 * c] & 15;
                    ctq[c] = s[8 + 3 * c];
                    if (ctq[c] > 3) return "quantisation table id above 3";
                    if (hsamp[c] < 1 || hsamp[c] > 4 || vsamp[c] < 1 || vsamp[c] > 4) return "bad sampling factor";
                }
                sof = true;
                break;
            }
            case 0xC2: case 0xC6: case 0xCA: case 0xCE: return "progressive JPEG";
            case 0xC3: case 0xC7: case 0xCB: case 0xCF: return "lossless JPEG";
            case 0xC5: return "hierarchical JPEG";
            case 0xC9: case 0xCD: case 0xCC: return "arithmetic coding";
            case 0xDC: return "DNL marker";
            case 0xDB: {
                size_t o = 0;
                while (o < sl) {
                    const int pq = s[o] >> 4, tq = s[o] & 15;
                    if (tq > 3 || pq > 1) return "bad DQT segment";
                    if (o + 1 + 64u * (pq + 1) > sl) return "short DQT segment";
                    for (int k = 0; k < 64; ++k)
                        qt[tq][natural_order_host()[k]] = pq ? (uint16_t)(s[o + 1 + 2 * k] << 8 | s[o + 2 + 2 * k]) : s[o + 1 + k];
                    have_q[tq] = true;
                    o += 1 + 64 * (pq + 1);
                }
                break;
            }
            case 0xC4: {
                size_t o = 0;
                while (o < sl) {
                    if (o + 17 > sl) return "short DHT segment";
                    const int tc = s[o] >> 4, th = s[o] & 15;
                    if (tc > 1 || th > 3) return "bad DHT segment";
                    int cnt = 0;
                    for (int i = 0; i < 16; ++i) cnt += s[o + 1 + i];
                    if (cnt > 256 || o + 17 + cnt > sl) return "bad DHT segment";
                    memcpy(hcounts[tc][th], s + o + 1, 16);
                    memcpy(hsyms[tc][th], s + o + 17, cnt);
                    have_h[tc][th] = true;
                    o += 17 + cnt;
                }
                break;
            }
            case 0xDD:
                if (sl < 2) return "short DRI segment";
                h.ri = s[0] << 8 | s[1];
                break;
            case 0xE0:
                if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) jfif = true;
                break;
            case 0xE1:
                if (!app1) {
                    app1 = true;
                    if (sl > 6) h.orient = exif_orientation(s + 6, sl - 6);
                }
                break;
            case 0xEE:
                if (sl >= 12 && !memcmp(s, "Adobe", 5)) { adobe = true; adobe_transform = s[11]; }
                break;
            case 0xDA: {
                if (!sof) return "SOS before SOF";
                if (sl < 1) return "short SOS segment";
                const int ns = s[0];
                if (sl < 4 + 2u * ns) return "short SOS segment";
                if (ns != h.ncomp) return "non-interleaved scan (a scan without every component)";
                int tdc[3], tac[3];
                for (int i = 0; i < ns; ++i) {
                    if (s[1 + 2 * i] != cid[i]) return "scan components out of frame order";
                    tdc[i] = s[2 + 2 * i] >> 4;
                    tac[i] = s[2 + 2 * i] & 15;
                    if (tdc[i] > 3 || tac[i] > 3) return "bad Huffman table id";
                }
                const uint8_t* t = s + 1 + 2 * ns;
                if (t[0] != 0 || t[1] != 63 || t[2] != 0) return "spectral selection or successive approximation in a sequential scan";
                if (h.ncomp == 3) {
                    const bool rgb = !jfif && (adobe ? adobe_transform == 0 : (cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B'));
                    if (rgb) return "RGB colour transform (Adobe transform 0 or RGB component ids)";
                    for (int c = 1; c < 3; ++c)
                        if (hsamp[c] != 1 || vsamp[c] != 1) return "unsupported sampling (chroma not 1x1)";
                    const int hv = hsamp[0] * 10 + vsamp[0];
                    if (hv != 11 && hv != 21 && hv != 22) return "unsupported sampling (not 4:4:4, 4:2:2 or 4:2:0)";
                    h.hs = hsamp[0]; h.vs = vsamp[0];
                    h.mcux = (h.W + 8 * h.hs - 1) / (8 * h.hs);
                    h.mcuy = (h.H + 8 * h.vs - 1) / (8 * h.vs);
                    h.bpm = h.hs * h.vs + 2;
                } else {
                    h.hs = h.vs = 1;        // a single-component scan is non-interleaved: one block per MCU
                    h.mcux = (h.W + 7) / 8;
                    h.mcuy = (h.H + 7) / 8;
                    h.bpm = 1;
                }
                for (int c = 0; c < h.ncomp; ++c) {
                    if (!have_q[ctq[c]]) return "quantisation table not defined";
                    memcpy(h.t.q[c], qt[ctq[c]], sizeof(qt[0]));
                    for (int ac = 0; ac < 2; ++ac) {
                        const int id = ac ? tac[c] : tdc[c];
                        const uint8_t *cnt, *sym;
                        if (have_h[ac][id]) { cnt = hcounts[ac][id]; sym = hsyms[ac][id]; }
                        else if (id < 2) { cnt = std_counts(ac, id); sym = std_syms(ac, id); }
                        else return "Huffman table not defined";
                        if (const char* e = build_huff(cnt, sym, !ac, h.t.h[2 * c + ac])) return e;
                    }
                }
                if (h.orient >= 5) { h.oH = h.W; h.oW = h.H; } else { h.oH = h.H; h.oW = h.W; }
                h.ecs = (long long)p;
                return nullptr;
            }
            default:        // other APPn and COM are skipped; libjpeg refuses DHP, EXP, JPGn and RESn
                if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) return "unknown marker";
                break;
        }
    }
}

// the device frame of a parsed header (buffer offsets are filled by the caller)
inline void frame_of(const Header& h, DecFrame& f) {
    memset(&f, 0, sizeof(f));
    f.H = h.H; f.W = h.W; f.oH = h.oH; f.oW = h.oW; f.orient = h.orient;
    f.ncomp = h.ncomp; f.hs = h.hs; f.vs = h.vs; f.mcux = h.mcux; f.mcuy = h.mcuy; f.bpm = h.bpm; f.ri = h.ri;
    const long long mcus = (long long)h.mcux * h.mcuy;
    f.nint = h.ri ? (mcus + h.ri - 1) / h.ri : 1;
    f.nblk = mcus * h.bpm;
    int s = 0;
    for (int y = 0; y < h.vs; ++y)
        for (int x = 0; x < h.hs; ++x, ++s) { f.slot_comp[s] = 0; f.slot_dx[s] = x; f.slot_dy[s] = y; }
    for (int c = 1; c < h.ncomp; ++c, ++s) f.slot_comp[s] = c;
    for (int c = 0; c < h.ncomp; ++c) {
        f.pw[c] = h.mcux * (c ? 1 : h.hs) * 8;
        f.ph[c] = h.mcuy * (c ? 1 : h.vs) * 8;
    }
}

// the reduced / gray frame of a parsed header: 1 / d scale (d = 1, 2, 4, 8), colour or gray.  libjpeg's
// jpeg_core_output_dimensions rule (jdmaster.c): the luma IDCT is m = 8 / d square; a chroma component's doubles from m while
// it stays <= 8 and both the luma's sampling factors times m divide by twice it.  libjpeg turns fancy upsampling off at m = 1.
inline void frame_scaled(const Header& h, int d, bool gray, DecFrame& f, DecScaled& z) {
    frame_of(h, f);
    memset(&z, 0, sizeof(z));
    const int m = 8 / d;
    z.dH = (h.H + d - 1) / d;
    z.dW = (h.W + d - 1) / d;
    if (h.orient >= 5) { f.oH = z.dW; f.oW = z.dH; } else { f.oH = z.dH; f.oW = z.dW; }
    z.gray = gray;
    z.sc[0] = m;
    for (int c = 1; c < h.ncomp; ++c) {
        int s = m;
        while (s < 8 && (h.hs * m) % (2 * s) == 0 && (h.vs * m) % (2 * s) == 0) s *= 2;
        z.sc[c] = s;
    }
    for (int c = 0; c < h.ncomp; ++c) {
        f.pw[c] = h.mcux * (c ? 1 : h.hs) * z.sc[c];
        f.ph[c] = h.mcuy * (c ? 1 : h.vs) * z.sc[c];
    }
    if (h.ncomp == 3) {
        z.uh = h.hs * m / z.sc[1];
        z.uv = h.vs * m / z.sc[1];
        z.cw = (z.dW + z.uh - 1) / z.uh;
        z.ch = (z.dH + z.uv - 1) / z.uv;
        if (m == 1) z.cw = 1;
    }
}

// ---------------------------------------------------------------------------------------------------- unstuffing (GPU)
JD_HD bool is_rst(int b) { return b >= 0xD0 && b <= 0xD7; }

template <typename F>
__device__ __forceinline__ int find_by(int n, F start_of, long long v) {     // the last frame whose start <= v
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start_of(mid) <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// What byte p of a file's entropy-coded bytes is (T.81 B.1.1.2, read as libjpeg reads it): a run of 0xFF is fill up to its
// last byte, which is one data 0xFF when 0x00 follows, a restart marker when RSTn follows, and otherwise the marker that ends
// the data; the 0x00 or RSTn byte after it is dropped.
enum { kByteData, kByteDrop, kByteRst, kByteEnd };
JD_HD int byte_kind(const uint8_t* b, long long len, long long p) {
    const int c = b[p], nx = p + 1 < len ? b[p + 1] : -1;
    if (c == 0xFF) {
        if (nx == 0xFF) return kByteDrop;
        if (nx == 0) return kByteData;
        return is_rst(nx) ? kByteRst : kByteEnd;
    }
    return p > 0 && b[p - 1] == 0xFF && (c == 0 || is_rst(c)) ? kByteDrop : kByteData;
}

// What follows the data that ends at e: APPn and COM segments, which libjpeg reads after the scan, then EOI.  0, or the status.
JD_HD int after_data_status(const uint8_t* b, long long len, long long e) {
    long long p = e;
    for (;;) {
        while (p < len && b[p] == 0xFF) ++p;
        if (p >= len) return kStTruncated;
        const int m = b[p];
        if (m == 0xD9) return 0;
        if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) return kStMarker;
        if (p + 2 >= len) return kStTruncated;
        p += 1 + ((long long)b[p + 1] << 8 | b[p + 2]);       // advances by at least one byte
        if (p >= len) return kStTruncated;
        if (b[p] != 0xFF) return kStMarker;
    }
}

// per file: end[f] = the first byte of the marker that ends the data (initialised to in_len)
__global__ void __launch_bounds__(256) jd_end_kernel(const DecFrame* __restrict__ fr, int n, const uint8_t* __restrict__ in, long long nchunks,
                                                     unsigned long long* __restrict__ end) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const int f = find_by(n, [&](int k) { return fr[k].in0; }, i * kChunk);
    const long long p0 = i * kChunk - fr[f].in0, len = fr[f].in_len;
    const uint8_t* b = in + fr[f].in0;
    for (long long p = p0; p < p0 + kChunk && p < len; ++p)
        if (byte_kind(b, len, p) == kByteEnd) { atomicMin(end + f, (unsigned long long)p); return; }
}

// per chunk: kept bytes + (RST markers << 32) before the file's end
template <bool kScatter>
__global__ void __launch_bounds__(256) jd_unstuff_kernel(const DecFrame* __restrict__ fr, int n, const uint8_t* __restrict__ in, long long nchunks,
                                                         const unsigned long long* __restrict__ end, long long* __restrict__ counts,
                                                         const long long* __restrict__ excl, uint8_t* __restrict__ out,
                                                         long long* __restrict__ ival_start, int* __restrict__ status) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nchunks) return;
    const int f = find_by(n, [&](int k) { return fr[k].in0; }, i * kChunk);
    const DecFrame& F = fr[f];
    const long long p0 = i * kChunk - F.in0, e = (long long)end[f];
    const uint8_t* b = in + F.in0;
    long long kept = 0, rst = 0;
    if (kScatter) {
        const long long d = excl[i] - excl[F.in0 / kChunk];
        kept = d & 0xffffffffll;
        rst = d >> 32;
    }
    for (long long p = p0; p < p0 + kChunk && p < e; ++p) {
        const int k = byte_kind(b, F.in_len, p);
        if (k == kByteRst) {
            if (kScatter) {
                if (b[p + 1] != 0xD0 + (rst & 7)) atomicOr(status + f, kStRst);
                if (rst + 1 < F.nint) ival_start[F.iv0 + rst + 1] = kept;
                else atomicOr(status + f, kStRst);
            }
            ++rst;
        } else if (k == kByteData) {
            if (kScatter) out[F.in0 + kept] = b[p];
            ++kept;
        }
    }
    if (!kScatter) counts[i] = kept + (rst << 32);
}

// one thread per file: stream length, RST count, what follows the data
__global__ void jd_frame_kernel(const DecFrame* __restrict__ fr, int n, const uint8_t* __restrict__ in, const unsigned long long* __restrict__ end,
                                const long long* __restrict__ excl, long long* __restrict__ nbytes, long long* __restrict__ ival_start,
                                int* __restrict__ status) {
    const int f = threadIdx.x;
    if (f >= n) return;
    const DecFrame& F = fr[f];
    const long long c0 = F.in0 / kChunk, c1 = (F.in0 + F.in_len + kChunk - 1) / kChunk;
    const long long d = excl[c1] - excl[c0];
    nbytes[f] = d & 0xffffffffll;
    if ((d >> 32) < F.nint - 1) atomicOr(status + f, kStRst);
    if (const int st = after_data_status(in + F.in0, F.in_len, (long long)end[f])) atomicOr(status + f, st);
    ival_start[F.iv0] = 0;
}

// one thread per interval of the call: its bit range and number of subsequences
__global__ void __launch_bounds__(256) jd_interval_kernel(const DecFrame* __restrict__ fr, int n, long long nint, const long long* __restrict__ nbytes,
                                                          const long long* __restrict__ ival_start, long long* __restrict__ ibits,
                                                          int* __restrict__ npieces, int piece_bits) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= nint) return;
    const int f = find_by(n, [&](int k) { return fr[k].iv0; }, i);
    const long long nb = nbytes[f];
    auto at = [&](long long k) { const long long v = ival_start[k]; return v < 0 || v > nb ? nb : v; };
    const long long s = at(i), e = i + 1 < fr[f].iv0 + fr[f].nint ? max(s, at(i + 1)) : nb;
    ibits[2 * i] = s * 8;
    ibits[2 * i + 1] = max(s, e) * 8;
    npieces[i] = (int)max(1ll, (e * 8 - s * 8 + piece_bits - 1) / piece_bits);
}

// ---------------------------------------------------------------------------------------------------- Huffman decode (GPU)
struct Bufs {
    const DecFrame* fr;
    const Tables* tabs;
    const uint8_t* bytes;         // compacted streams, file f at fr[f].in0
    const long long* nbytes;
    Piece* pieces;
    uint64_t* in_state;
    int* nblk;                    // per piece
    int* dc[3];                   // per piece and component
    int* err;                     // per piece: status bits of its latest decode
};

__device__ __forceinline__ void decode_into(const Bufs& B, long long j, uint64_t in, uint64_t* out_state) {
    const Piece P = B.pieces[j];
    const DecFrame& F = B.fr[P.f];
    const PieceResult r = decode_piece<false>(F, B.tabs[P.f], jpeg::kZigzag, B.bytes + F.in0, B.nbytes[P.f], in, P.end, P.iend, nullptr, 0, 0,
                                              nullptr);
    out_state[j] = r.state;
    B.nblk[j] = r.nblocks;
    B.err[j] = r.err;
    for (int c = 0; c < 3; ++c) B.dc[c][j] = r.dc[c];
}

// one thread per subsequence: its place, and a decode from its guessed start state (known at an interval's start)
__global__ void __launch_bounds__(128) jd_piece_kernel(Bufs B, int n, long long npieces, long long nint, const long long* __restrict__ pc0,
                                                       const long long* __restrict__ ibits, int piece_bits, uint64_t* __restrict__ out_state) {
    const long long j = (long long)blockIdx.x * 128 + threadIdx.x;
    if (j >= npieces) return;
    long long lo = 0, hi = nint - 1;
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (pc0[mid] <= j) lo = mid; else hi = mid - 1;
    }
    Piece P;
    P.iv = lo;
    P.f = find_by(n, [&](int k) { return B.fr[k].iv0; }, lo);
    P.first = j == pc0[lo];
    P.iend = ibits[2 * lo + 1];
    P.start = ibits[2 * lo] + (j - pc0[lo]) * piece_bits;
    P.end = min(P.start + piece_bits, P.iend);
    B.pieces[j] = P;
    const uint64_t in = pack_state(P.start, 0, 0);
    B.in_state[j] = in;
    decode_into(B, j, in, out_state);
}

// one round: a subsequence whose predecessor ended in a state other than its start state decodes again from that state
__global__ void __launch_bounds__(128) jd_sync_kernel(Bufs B, long long npieces, const uint64_t* __restrict__ cur, uint64_t* __restrict__ next,
                                                      int* __restrict__ changed) {
    const long long j = (long long)blockIdx.x * 128 + threadIdx.x;
    if (j >= npieces) return;
    const uint64_t s = j > 0 ? cur[j - 1] : 0;
    if (B.pieces[j].first || s == B.in_state[j]) { next[j] = cur[j]; return; }
    B.in_state[j] = s;
    decode_into(B, j, s, next);
    *changed = 1;
}

// errors of the synchronised decode, and intervals with the wrong number of blocks
__global__ void __launch_bounds__(128) jd_check_kernel(Bufs B, long long npieces, const long long* __restrict__ pc0,
                                                       const uint64_t* __restrict__ out_state, const long long* __restrict__ bx,
                                                       int* __restrict__ status) {
    const long long j = (long long)blockIdx.x * 128 + threadIdx.x;
    if (j >= npieces) return;
    const Piece& P = B.pieces[j];
    const DecFrame& F = B.fr[P.f];
    if (B.err[j]) atomicOr(status + P.f, B.err[j]);
    if (P.first) {
        const long long k = P.iv - F.iv0, per = F.ri ? (long long)F.ri * F.bpm : F.nblk;
        const long long want = min(per, F.nblk - k * per), got = bx[pc0[P.iv + 1]] - bx[pc0[P.iv]];
        if (got != want) atomicOr(status + P.f, kStBlocks);
    }
}

// one thread per subsequence: decode again from its final start state and write the coefficients (natural order, DC values)
__global__ void __launch_bounds__(128) jd_write_kernel(Bufs B, long long npieces, const long long* __restrict__ pc0, const long long* __restrict__ bx,
                                                       const long long* __restrict__ dcx0, const long long* __restrict__ dcx1,
                                                       const long long* __restrict__ dcx2, int16_t* __restrict__ coef) {
    const long long j = (long long)blockIdx.x * 128 + threadIdx.x;
    if (j >= npieces) return;
    const Piece P = B.pieces[j];
    const DecFrame& F = B.fr[P.f];
    const long long first = pc0[P.iv], k = P.iv - F.iv0, per = F.ri ? (long long)F.ri * F.bpm : F.nblk;
    const long long blk = k * per + bx[j] - bx[first], blk_end = min(F.nblk, (k + 1) * per);
    const int pred[3] = {(int)(dcx0[j] - dcx0[first]), (int)(dcx1[j] - dcx1[first]), (int)(dcx2[j] - dcx2[first])};
    decode_piece<true>(F, B.tabs[P.f], jpeg::kZigzag, B.bytes + F.in0, B.nbytes[P.f], B.in_state[j], P.end, P.iend, coef + F.blk0 * 64,
                       blk, blk_end, pred);
}

// ---------------------------------------------------------------------------------------------------- pixels (GPU)
constexpr int kIdctBlocks = 32;      // blocks per CTA, 8 threads each

// kScaled: each component at its IDCT size zs[f].sc[c] (8 threads per block still: columns, then rows), chroma skipped in gray
// mode; otherwise every block 8x8 and zs is unused
template <bool kScaled>
__global__ void __launch_bounds__(256) jd_idct_kernel(const DecFrame* __restrict__ fr, int n, const Tables* __restrict__ tabs, long long nblocks,
                                                      const int16_t* __restrict__ coef, uint8_t* __restrict__ planes,
                                                      const DecScaled* __restrict__ zs) {
    __shared__ int16_t ws[kIdctBlocks][64];
    const int lb = threadIdx.x >> 3, t = threadIdx.x & 7;
    const long long g = (long long)blockIdx.x * kIdctBlocks + lb;
    bool live = g < nblocks;            // the same for the 8 threads of a block
    int f = 0, c = 0, bx = 0, by = 0, sz = 8;
    if (live) {
        f = find_by(n, [&](int k) { return fr[k].blk0; }, g);
        c = block_place(fr[f], g - fr[f].blk0, bx, by);
        if (kScaled) {
            sz = zs[f].sc[c];
            if (c && zs[f].gray) live = false;
        }
        if (!kScaled || (live && sz == 8)) {
            const bool ac = __any_sync(0xffu << (threadIdx.x & 24), idct_column_ac(coef + g * 64, t));
            idct_column(coef + g * 64, tabs[f].q[c], t, !ac, ws[lb]);
        } else if (live && sz == 4) {
            const bool ac = __any_sync(0xffu << (threadIdx.x & 24), idct4_column_ac(coef + g * 64, t));
            if (t != 4) idct4_column(coef + g * 64, tabs[f].q[c], t, !ac, ws[lb]);
        } else if (live && sz == 2) {
            if (t < 2 || (t & 1)) idct2_column(coef + g * 64, tabs[f].q[c], t, ws[lb]);
        }
    }
    __syncthreads();
    if (!live) return;
    if (kScaled && sz < 8) {
        const DecFrame& F = fr[f];
        uint8_t* dst = planes + F.plane0[c] + ((size_t)by * sz + t) * F.pw[c] + (size_t)bx * sz;
        if (sz == 4 && t < 4) {
            uint8_t v[4];
            idct4_row(ws[lb], t, v);
            *reinterpret_cast<uint32_t*>(dst) = v[0] | v[1] << 8 | v[2] << 16 | (uint32_t)v[3] << 24;
        } else if (sz == 2 && t < 2) {
            uint8_t v[2];
            idct2_row(ws[lb], t, v);
            *reinterpret_cast<uint16_t*>(dst) = (uint16_t)(v[0] | v[1] << 8);
        } else if (sz == 1 && t == 0) {
            *dst = idct1(coef + g * 64, tabs[f].q[c]);
        }
        return;
    }
    uint8_t v[8];
    idct_row(ws[lb], t, v);
    const DecFrame& F = fr[f];
    uint8_t* dst = planes + F.plane0[c] + ((size_t)by * 8 + t) * F.pw[c] + (size_t)bx * 8;
    uint2 w;
    w.x = v[0] | v[1] << 8 | v[2] << 16 | (uint32_t)v[3] << 24;
    w.y = v[4] | v[5] << 8 | v[6] << 16 | (uint32_t)v[7] << 24;
    *reinterpret_cast<uint2*>(dst) = w;
}

enum { kColorFull, kColorScaled, kColorGray };

// one thread per decoded pixel: kColorFull the full-size BGR frame (zs unused), kColorScaled a reduced one (H x W is then
// zs[f].dH x dW), kColorGray the luma plane alone into oH x oW x 1
template <int kMode>
__global__ void __launch_bounds__(256) jd_color_kernel(const DecFrame* __restrict__ fr, int n, long long npix, const uint8_t* __restrict__ planes,
                                                       const DecScaled* __restrict__ zs) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= npix) return;
    const int f = find_by(n, [&](int k) { return fr[k].pix0; }, i);
    const DecFrame& F = fr[f];
    const long long l = i - F.pix0;
    const int W = kMode == kColorFull ? F.W : zs[f].dW;
    const int y = (int)(l / W), x = (int)(l - (long long)y * W);
    uint8_t o[3];
    if (kMode == kColorFull) pixel_bgr(F, planes, y, x, o);
    else if (kMode == kColorScaled) pixel_bgr_scaled(F, zs[f], planes, y, x, o);
    else o[0] = planes[F.plane0[0] + (size_t)y * F.pw[0] + x];
    int oy, ox;
    if (kMode == kColorFull) orient_dst(F.orient, F.H, F.W, y, x, oy, ox);
    else orient_dst(F.orient, zs[f].dH, zs[f].dW, y, x, oy, ox);
    if (kMode == kColorGray) {
        F.out[(size_t)oy * F.oW + ox] = o[0];
        return;
    }
    uint8_t* d = F.out + ((size_t)oy * F.oW + ox) * 3;
    d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
}

}  // namespace jpegdec
}  // namespace whenet
