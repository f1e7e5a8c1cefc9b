// Host-only dump of the round-2 route planners (no GPU): K2 (persistent 1x1 conv) plans of the late expands / projects / head conv,
// KD chunk widths, thread counts and shared memory (both KD kernels), the K1X instances, pw_tc3's tile walk of the
// early gated projects.
//   nvcc -std=c++17 -arch=sm_90a -o build_tmp/route_plan_dump tools/route_plan_dump.cu && build_tmp/route_plan_dump [crops]
#include <cstdio>
#include <cstdlib>
#include "../headposeestimation-whenet_b200/csrc/kernels_simt.cuh"
#include "../headposeestimation-whenet_b200/csrc/kernels_tc.cuh"
#include "../headposeestimation-whenet_b200/csrc/kernels_k2.cuh"
#include "../headposeestimation-whenet_b200/csrc/kernels_dwse.cuh"
#include "../headposeestimation-whenet_b200/csrc/kernels_k1x.cuh"
using namespace whenet;
struct Blk { int idx, hin, ho, cin, cexp, cout, k, s, cse; };
static const Blk blocks[] = {
    {1, 112, 112, 32, 32, 16, 3, 1, 8},     {2, 112, 56, 16, 96, 24, 3, 2, 4},      {3, 56, 56, 24, 144, 24, 3, 1, 6},      {4, 56, 28, 24, 144, 40, 5, 2, 6},
    {5, 28, 28, 40, 240, 40, 5, 1, 10},     {6, 28, 14, 40, 240, 80, 3, 2, 10},     {7, 14, 14, 80, 480, 80, 3, 1, 20},     {9, 14, 14, 80, 480, 112, 5, 1, 20},
    {10, 14, 14, 112, 672, 112, 5, 1, 28},  {12, 14, 7, 112, 672, 192, 5, 2, 28},   {13, 7, 7, 192, 1152, 192, 5, 1, 48},   {16, 7, 7, 192, 1152, 320, 3, 1, 48}};
template <int KS, int S, int HIN, int CC> static void kd_line(const Blk& b) {
    printf("  kd b%02d cc %d threads %d strips %d pw %d smem %zu chunks %d\n", b.idx, CC, fused::DwSeThreads<KS, S, HIN, CC>::value,
           fused::DwSeGeom<KS, S, HIN>::NSTRIPS, fused::DwSeGeom<KS, S, HIN>::PW, fused::dwse_smem<KS, S, HIN, CC>(b.cexp, b.cse), b.cexp / CC);
}
// KD with the on-chip expand (one CTA per crop): CIN input channels
template <int KS, int S, int HIN, int CC, int CIN> static void kdx_line(const Blk& b) {
    using X = fused::DwSeX<KS, S, HIN, CC, CIN>;
    printf("  kdx b%02d cc %d cin %d threads %d halves %d nwg %d smem %zu chunks %d ctas_per_sm %d\n", b.idx, CC, CIN, X::NT, X::HALVES,
           X::NWG, X::smem(b.cexp, b.cse), b.cexp / CC, X::CTAS_PER_SM);
}
// K1X (K1 fed by TMA): geometry and shared memory of the instance
template <int KS, int S, int HIN, int TH, int R, int CC, int CIN> static void k1x_line(const Blk& b) {
    using X = fused::K1X<KS, S, HIN, TH, R, CC, CIN>;
    if (b.k == KS && b.s == S && b.hin == HIN && b.cin == CIN)
        printf("  k1x b%02d th %d r %d cc %d cin %d tiles %d pix %d halves %d ksteps %d lanes %d smem %zu chunks %d ctas_per_sm %d row_bytes %d\n", b.idx,
               TH, R, CC, CIN, X::TILES, X::NPIX, X::HALVES, X::KSTEPS, X::PY, X::SMEM, b.cexp / CC, X::CTAS_PER_SM, X::ROWB);
}
static void k2_line(const char* what, int idx, long long M, int K, int N, int hw, bool gate) {
    tc::K2Params p{};
    size_t smem = 0;
    if (!tc::plan_k2(M, K, N, hw, gate, true, &p, &smem)) { printf("  k2 %s b%02d: no plan\n", what, idx); return; }
    printf("  k2 %s b%02d M %lld K %d N %d gate %d : n_tile %d n_tiles %d tiles %d nkb %d stages %d resident %d smem %zu\n", what, idx, M, K, N,
           (int)gate, p.n_tile, p.n_tiles, p.tiles, p.nkb, p.stages, p.w_resident, smem);
}
int main(int argc, char** argv) {
    const int crops = argc > 1 ? atoi(argv[1]) : 256;
    for (const Blk& b : blocks) {
        const int cc = b.idx == 1 ? 32 : fused::dwse_chunk(b.k, b.s, b.hin, b.cexp);
        printf("b%02d kd_chunk %d\n", b.idx, b.idx == 1 ? 32 : cc);
        if (b.idx >= 7) {
            if (b.hin == 14 && b.s == 1 && b.k == 3) kd_line<3, 1, 14, 32>(b);
            if (b.hin == 14 && b.s == 1 && b.k == 5) kd_line<5, 1, 14, 32>(b);
            if (b.hin == 14 && b.s == 2 && b.k == 5) kd_line<5, 2, 14, 96>(b);
            if (b.hin == 7 && b.k == 5) kd_line<5, 1, 7, 128>(b);
            if (b.hin == 7 && b.k == 3) kd_line<3, 1, 7, 128>(b);
            if (b.hin == 14 && b.s == 1 && b.k == 3) kdx_line<3, 1, 14, 32, 80>(b);
            if (b.hin == 14 && b.s == 1 && b.k == 5 && b.cin == 80) kdx_line<5, 1, 14, 32, 80>(b);
            if (b.hin == 14 && b.s == 1 && b.k == 5 && b.cin == 112) kdx_line<5, 1, 14, 32, 112>(b);
            if (b.hin == 14 && b.s == 2 && b.k == 5) kdx_line<5, 2, 14, 96, 112>(b);
            if (b.hin == 7 && b.k == 5) kdx_line<5, 1, 7, 128, 192>(b);
            if (b.hin == 7 && b.k == 3) kdx_line<3, 1, 7, 128, 192>(b);
            k2_line("expand ", b.idx, (long long)crops * b.hin * b.hin, b.cin, b.cexp, b.hin * b.hin, false);
            k2_line("project", b.idx, (long long)crops * b.ho * b.ho, b.cexp, b.cout, b.ho * b.ho, true);
        } else {
            if (b.idx == 1) kd_line<3, 1, 14, 32>(b);
#define K1X_LINE(KS, S, HIN, TH, R, CC, CIN) k1x_line<KS, S, HIN, TH, R, CC, CIN>(b);
            WHENET_K1X_INSTANCES(K1X_LINE)
#undef K1X_LINE
            tc::Pw3Plan pl{};
            const bool ok = tc::plan_pw_tc3((long long)crops * b.ho * b.ho, b.cexp, b.cout, b.ho * b.ho, true, &pl);
            if (ok) printf("  pw3 b%02d tiles_per_crop %d tpc %d groups %d umma_n %d smem %zu\n", b.idx, pl.tiles_per_crop, pl.tpc, pl.groups, pl.umma_n, pl.smem);
            else printf("  pw3 b%02d: not taken\n", b.idx);
        }
    }
    k2_line("head   ", 17, (long long)crops * 49, 320, 1280, 49, false);
    return 0;
}
