// Host-only run of the GPU JPEG decoder's algorithm (csrc/kernels_jpeg_dec.cuh): the same parse, Huffman state machine, IDCT,
// upsampling and colour conversion, with the subsequences and their synchronisation rounds emulated one after another.
//   nvcc -std=c++17 -arch=sm_90a -O1 -g -Xcompiler -fsanitize=address -lasan -o jpeg_decode_dump tools/jpeg_decode_dump.cu
//   jpeg_decode_dump PIECE_BITS [--scale D C] in.jpg out.bgr [in.jpg out.bgr ...]
// Prints one line per file: "ok H W rounds", "einval <reason>" (the header is refused) or "status <bits> rounds"; for "ok"
// the H x W x 3 BGR bytes go to out.bgr.  --scale decodes at 1 / D (1, 2, 4 or 8) into C channels (3: BGR, 1: the luma
// plane), as whenet_decode_jpeg_ex_u8 (DESIGN.md section 8.13); out.bgr then holds H x W x C bytes.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../headposeestimation-whenet_b200/csrc/kernels_jpeg_dec.cuh"

using namespace whenet::jpegdec;

static std::vector<uint8_t> read_file(const char* path) {
    std::vector<uint8_t> d;
    FILE* f = fopen(path, "rb");
    if (!f) return d;
    fseek(f, 0, SEEK_END);
    d.resize((size_t)ftell(f));
    fseek(f, 0, SEEK_SET);
    if (!d.empty() && fread(d.data(), 1, d.size(), f) != d.size()) d.clear();
    fclose(f);
    return d;
}

// jd_idct_kernel<true> and jd_color_kernel<kColorScaled / kColorGray> on the CPU
static int pixels_scaled(DecFrame& fr, const DecScaled& z, const Header& h, const std::vector<int16_t>& coef, std::vector<uint8_t>& out) {
    const int np = z.gray ? 1 : fr.ncomp;
    long long planes = 0;
    for (int c = 0; c < np; ++c) { fr.plane0[c] = planes; planes += (long long)fr.pw[c] * fr.ph[c]; }
    std::vector<uint8_t> pl((size_t)planes);
    for (long long g = 0; g < fr.nblk; ++g) {
        int bx, by;
        const int c = block_place(fr, g, bx, by), sz = z.sc[c];
        if (c >= np) continue;
        const int16_t* cf = coef.data() + g * 64;
        uint8_t* dst = pl.data() + fr.plane0[c] + (size_t)by * sz * fr.pw[c] + (size_t)bx * sz;
        int16_t ws[64];
        if (sz == 8) {
            bool ac = false;
            for (int col = 0; col < 8; ++col) ac |= idct_column_ac(cf, col);
            for (int col = 0; col < 8; ++col) idct_column(cf, h.t.q[c], col, !ac, ws);
            for (int row = 0; row < 8; ++row) idct_row(ws, row, dst + (size_t)row * fr.pw[c]);
        } else if (sz == 4) {
            bool ac = false;
            for (int col = 0; col < 8; ++col) ac |= idct4_column_ac(cf, col);
            for (int col = 0; col < 8; ++col)
                if (col != 4) idct4_column(cf, h.t.q[c], col, !ac, ws);
            for (int row = 0; row < 4; ++row) idct4_row(ws, row, dst + (size_t)row * fr.pw[c]);
        } else if (sz == 2) {
            for (int col : {0, 1, 3, 5, 7}) idct2_column(cf, h.t.q[c], col, ws);
            for (int row = 0; row < 2; ++row) idct2_row(ws, row, dst + (size_t)row * fr.pw[c]);
        } else {
            *dst = idct1(cf, h.t.q[c]);
        }
    }
    const int C = z.gray ? 1 : 3;
    out.assign((size_t)fr.oH * fr.oW * C, 0);
    for (int y = 0; y < z.dH; ++y)
        for (int x = 0; x < z.dW; ++x) {
            int oy, ox;
            orient_dst(fr.orient, z.dH, z.dW, y, x, oy, ox);
            uint8_t* o = out.data() + ((size_t)oy * fr.oW + ox) * C;
            if (z.gray) *o = pl[fr.plane0[0] + (size_t)y * fr.pw[0] + x];
            else pixel_bgr_scaled(fr, z, pl.data(), y, x, o);
        }
    return 0;
}

// returns the status bits; out gets the BGR frame
static int decode(const std::vector<uint8_t>& file, const Header& h, int S, std::vector<uint8_t>& out, int& rounds, int scale,
                  bool gray) {
    const bool scaled = scale != 1 || gray;
    DecFrame fr;
    DecScaled z;
    if (scaled) frame_scaled(h, scale, gray, fr, z);
    else frame_of(h, fr);
    const uint8_t* b = file.data() + h.ecs;
    const long long len = (long long)file.size() - h.ecs;
    int status = 0;

    // unstuffing, as jd_end_kernel / jd_unstuff_kernel / jd_frame_kernel
    long long end = len;
    for (long long p = 0; p < len; ++p)
        if (byte_kind(b, len, p) == kByteEnd) { end = p; break; }
    std::vector<uint8_t> comp;
    std::vector<long long> ival(fr.nint, -1);
    ival[0] = 0;
    long long rst = 0;
    for (long long p = 0; p < end; ++p) {
        const int k = byte_kind(b, len, p);
        if (k == kByteRst) {
            if (b[p + 1] != 0xD0 + (rst & 7)) status |= kStRst;
            if (rst + 1 < fr.nint) ival[rst + 1] = (long long)comp.size();
            else status |= kStRst;
            ++rst;
        } else if (k == kByteData) {
            comp.push_back(b[p]);
        }
    }
    if (rst < fr.nint - 1) status |= kStRst;
    status |= after_data_status(b, len, end);
    const long long nb = (long long)comp.size();
    comp.resize(comp.size() + 8, 0);      // nothing reads past nb (peek32 fills with 0xFF), but keep the vector non-empty

    // intervals and subsequences, as jd_interval_kernel / jd_piece_kernel
    std::vector<Piece> pieces;
    for (long long i = 0; i < fr.nint; ++i) {
        auto at = [&](long long k) { const long long v = ival[k]; return v < 0 || v > nb ? nb : v; };
        const long long s = at(i), e = i + 1 < fr.nint ? std::max(s, at(i + 1)) : nb;
        const long long np = std::max(1ll, (e * 8 - s * 8 + S - 1) / S);
        for (long long k = 0; k < np; ++k) {
            Piece P;
            P.iv = i; P.f = 0; P.first = k == 0;
            P.iend = e * 8;
            P.start = s * 8 + k * S;
            P.end = std::min(P.start + S, P.iend);
            pieces.push_back(P);
        }
    }
    const long long np = (long long)pieces.size();
    std::vector<uint64_t> in(np), cur(np), nxt(np);
    std::vector<PieceResult> res(np);
    auto run = [&](long long j, uint64_t st) {
        res[j] = decode_piece<false>(fr, h.t, natural_order_host(), comp.data(), nb, st, pieces[j].end, pieces[j].iend, nullptr, 0, 0,
                                     nullptr);
        return res[j].state;
    };
    for (long long j = 0; j < np; ++j) { in[j] = pack_state(pieces[j].start, 0, 0); cur[j] = run(j, in[j]); }
    rounds = 0;
    for (bool changed = true; changed;) {       // jd_sync_kernel: every subsequence reads the previous round's end states
        changed = false;
        ++rounds;
        for (long long j = 0; j < np; ++j) {
            const uint64_t s = j > 0 ? cur[j - 1] : 0;
            if (pieces[j].first || s == in[j]) { nxt[j] = cur[j]; continue; }
            in[j] = s;
            nxt[j] = run(j, s);
            changed = true;
        }
        cur.swap(nxt);
    }

    // block counts and DC predictions (the exclusive scans), the checks, the coefficients
    const long long per = fr.ri ? (long long)fr.ri * fr.bpm : fr.nblk;
    std::vector<int16_t> coef((size_t)fr.nblk * 64, 0);
    long long blk_in_iv = 0;
    int dcsum[3] = {0, 0, 0};
    for (long long j = 0; j < np; ++j) {
        if (pieces[j].first) { blk_in_iv = 0; dcsum[0] = dcsum[1] = dcsum[2] = 0; }
        status |= res[j].err;
        const long long k = pieces[j].iv;
        decode_piece<true>(fr, h.t, natural_order_host(), comp.data(), nb, in[j], pieces[j].end, pieces[j].iend, coef.data(),
                           k * per + blk_in_iv, std::min(fr.nblk, (k + 1) * per), dcsum);
        blk_in_iv += res[j].nblocks;
        for (int c = 0; c < 3; ++c) dcsum[c] += res[j].dc[c];
        if (j + 1 == np || pieces[j + 1].first)
            if (blk_in_iv != std::min(per, fr.nblk - k * per)) status |= kStBlocks;
    }
    if (status) return status;

    if (scaled) return pixels_scaled(fr, z, h, coef, out);

    // IDCT into component planes, then upsampling, colour and orientation
    long long planes = 0;
    for (int c = 0; c < fr.ncomp; ++c) { fr.plane0[c] = planes; planes += (long long)fr.pw[c] * fr.ph[c]; }
    std::vector<uint8_t> pl((size_t)planes);
    for (long long g = 0; g < fr.nblk; ++g) {
        int bx, by;
        const int c = block_place(fr, g, bx, by);
        int16_t ws[64];
        bool ac = false;
        for (int col = 0; col < 8; ++col) ac |= idct_column_ac(coef.data() + g * 64, col);
        for (int col = 0; col < 8; ++col) idct_column(coef.data() + g * 64, h.t.q[c], col, !ac, ws);
        for (int row = 0; row < 8; ++row) idct_row(ws, row, pl.data() + fr.plane0[c] + ((size_t)by * 8 + row) * fr.pw[c] + (size_t)bx * 8);
    }
    out.assign((size_t)fr.oH * fr.oW * 3, 0);
    for (int y = 0; y < fr.H; ++y)
        for (int x = 0; x < fr.W; ++x) {
            int oy, ox;
            orient_dst(fr.orient, fr.H, fr.W, y, x, oy, ox);
            pixel_bgr(fr, pl.data(), y, x, out.data() + ((size_t)oy * fr.oW + ox) * 3);
        }
    return 0;
}

int main(int argc, char** argv) {
    int first = 2, scale = 1, channels = 3;
    if (argc > 4 && !strcmp(argv[2], "--scale")) {
        scale = atoi(argv[3]);
        channels = atoi(argv[4]);
        first = 5;
        if ((scale != 1 && scale != 2 && scale != 4 && scale != 8) || (channels != 1 && channels != 3)) {
            fprintf(stderr, "--scale D C: D in {1, 2, 4, 8}, C in {1, 3}\n");
            return 2;
        }
    }
    if (argc < first + 2 || (argc - first) % 2) {
        fprintf(stderr, "usage: %s PIECE_BITS [--scale D C] in out [in out ...]\n", argv[0]);
        return 2;
    }
    const int S = atoi(argv[1]);
    if (S < kMinPieceBits || S > kMaxPieceBits) { fprintf(stderr, "PIECE_BITS outside [%d, %d]\n", kMinPieceBits, kMaxPieceBits); return 2; }
    Header* h = new Header;
    for (int a = first; a + 1 < argc; a += 2) {
        const std::vector<uint8_t> file = read_file(argv[a]);
        if (const char* e = parse_header(file.data(), file.size(), *h)) { printf("einval %s\n", e); continue; }
        std::vector<uint8_t> out;
        int rounds = 0;
        const int st = decode(file, *h, S, out, rounds, scale, channels == 1);
        if (st) { printf("status %d %d\n", st, rounds); continue; }
        FILE* f = fopen(argv[a + 1], "wb");
        if (!f || fwrite(out.data(), 1, out.size(), f) != out.size()) { fprintf(stderr, "cannot write %s\n", argv[a + 1]); return 1; }
        fclose(f);
        printf("ok %d %d %d\n", (h->oH + scale - 1) / scale, (h->oW + scale - 1) / scale, rounds);
    }
    delete h;
    return 0;
}
