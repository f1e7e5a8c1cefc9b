// Host-only dump of the K1 tile plans (default choice per block + any plan given on the command line):
//   nvcc -std=c++17 -arch=sm_90a -o build_tmp/k1_plan_dump tools/k1_plan_dump.cu && build_tmp/k1_plan_dump [th tw r cc nt nb]
#include <cstdio>
#include <cstdlib>
#include "../headposeestimation-whenet_b200/csrc/kernels_fused.cuh"
using namespace whenet::fused;
struct Blk { int idx, hin, ho, cin, cexp, k, s, pad; };
static const Blk blocks[] = {
    {2, 112, 56, 16, 96, 3, 2, 0},   {3, 56, 56, 24, 144, 3, 1, 1},   {4, 56, 28, 24, 144, 5, 2, 1},   {5, 28, 28, 40, 240, 5, 1, 2},
    {6, 28, 14, 40, 240, 3, 2, 0},   {7, 14, 14, 80, 480, 3, 1, 1},   {9, 14, 14, 80, 480, 5, 1, 2},   {10, 14, 14, 112, 672, 5, 1, 2},
    {12, 14, 7, 112, 672, 5, 2, 1},  {13, 7, 7, 192, 1152, 5, 1, 2},  {16, 7, 7, 192, 1152, 3, 1, 1}};
static void show(const Blk& b, const K1Params& p, int R, int NT, size_t smem) {
    printf("  b%02d %3d->%2d k%d s%d cin%3d cexp%4d : %2dx%-2d r%d cc%-3d nt%d nb%d  mtiles %d rows_alloc %3d chunks %2d PY %2d PYc %2d "
           "smem %6zu (A %6d W %5d C %5d E %6d) %s\n",
           b.idx, b.hin, b.ho, b.k, b.s, b.cin, b.cexp, p.TH, p.TW, R, p.CC, NT, p.NB, p.mtiles, p.rows_alloc, p.n_chunks, p.PY,
           p.PYc, smem, p.smem_A, p.smem_W, p.smem_C, p.smem_E, k1_two_per_sm(p, smem, NT) ? "2/SM" : "1/SM");
}
int main(int argc, char** argv) {
    for (const Blk& b : blocks) {
        K1Params p{}; K1Choice c{}; size_t smem = 0;
        if (plan_k1(b.hin, b.ho, b.cin, b.cexp, b.k, b.s, b.pad, true, true, &p, &c, &smem)) show(b, p, c.r, c.nt, smem);
        else printf("  b%02d: no plan\n", b.idx);
        for (int a = 1; a + 5 < argc; a += 6) {
            K1Params q{};
            const int th = atoi(argv[a]), tw = atoi(argv[a + 1]), r = atoi(argv[a + 2]), cc = atoi(argv[a + 3]), nt = atoi(argv[a + 4]), nb = atoi(argv[a + 5]);
            if (plan_k1_candidate(b.hin, b.ho, b.cin, b.cexp, b.k, b.s, b.pad, true, th, tw, r, cc, nt, nb, &q, &smem)) { printf("    alt"); show(b, q, r, nt, smem); }
        }
    }
    return 0;
}
