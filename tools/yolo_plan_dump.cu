// Host-only dump of the YOLOv3 detector's implicit-GEMM tile plans (no GPU): plan_igemm of convs 1-74 of the library's own table
// (tiny YOLOv3: convs 1-12) for a model input size, class count and SM count, or of single debug-conv shapes, plus the
// decode/NMS capacity constants.
//   nvcc -std=c++17 -arch=sm_90a -o build_tmp/yolo_plan_dump tools/yolo_plan_dump.cu
//   build_tmp/yolo_plan_dump net C SM [H W]         every legal input size (32..608 step 32 per side), or one
//   build_tmp/yolo_plan_dump tiny C SM [H W]        the same for tiny YOLOv3 (lines start with "tiny" instead of "net")
//   build_tmp/yolo_plan_dump conv SM Ho Wo N Cin k [Ho Wo N Cin k ...]
// and the fp32 parity mode's plans (plan_igemm32, with the CTAs per SM each plan assumes):
//   build_tmp/yolo_plan_dump net32 C SM [H W] | tiny32 C SM [H W] | conv32 SM Ho Wo N Cin k [...]
// and the frame groups launch_igemm / launch_igemm32 split a conv of n frames of Ho x Wo output pixels into:
//   build_tmp/yolo_plan_dump split Ho Wo n [Ho Wo n ...]
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#define WHENET_YOLO_HOST_ONLY
#define WHENET_YOLO32_HOST_ONLY
#include "../headposeestimation-whenet_b200/csrc/kernels_yolo.cuh"
#include "../headposeestimation-whenet_b200/csrc/kernels_yolo32.cuh"
using namespace whenet::yolo;

static const char* mode_name(int m) { return m == kLeaky ? "leaky" : m == kLeakyRes ? "res" : m == kLeakyCat ? "cat" : "f32"; }

static void plan_line(int Ho, int Wo, int N, int Cin, int k, int sm) {
    const IgemmPlan pl = plan_igemm(Ho, Wo, N, Cin, k, sm);
    const int n_tiles = (N + pl.n_tile - 1) / pl.n_tile;
    printf("Ho %d Wo %d N %d Cin %d k %d n_tile %d un %d n_stages %d smem %zu n_tail %d m_tail %d\n", Ho, Wo, N, Cin, k, pl.n_tile, pl.un,
           pl.n_stages, pl.smem, N - (n_tiles - 1) * pl.n_tile, (Ho * Wo) % BM);
}

static void plan32_line(int Ho, int Wo, int N, int Cin, int k, int sm) {
    const Igemm32Plan pl = plan_igemm32(Ho, Wo, N, Cin, k, sm);
    const int n_tiles = (N + pl.n_tile - 1) / pl.n_tile;
    printf("Ho %d Wo %d N %d Cin %d k %d n_tile %d un %d n_stages %d ctas %d smem %zu n_tail %d m_tail %d\n", Ho, Wo, N, Cin, k, pl.n_tile,
           pl.un, pl.n_stages, pl.ctas_per_sm, pl.smem, N - (n_tiles - 1) * pl.n_tile, (Ho * Wo) % BM);
}

// the per-layer shapes whenet_det_load_weights derives from the table; fp32: the fp32 mode's plans (lines "net32" / "tiny32")
static void net(int h, int w, int C, int sm, bool tiny, bool fp32 = false) {
    const std::vector<ConvCfg> T = tiny ? make_tiny_table() : make_table();
    std::vector<int> Ho(T.size()), Wo(T.size());
    for (size_t i = 0; i < T.size(); ++i) {
        const ConvCfg& c = T[i];
        Ho[i] = pooled(c.src < 0 ? h : Ho[c.src], c.pool) / c.stride;
        Wo[i] = pooled(c.src < 0 ? w : Wo[c.src], c.pool) / c.stride;
        if (i == 0) continue;                       // conv 0 is yolo_conv0_kernel
        printf("%s%s %d %d conv %zu mode %s stride %d ", tiny ? "tiny" : "net", fp32 ? "32" : "", h, w, i, mode_name(igemm_mode(c)), c.stride);
        (fp32 ? plan32_line : plan_line)(Ho[i], Wo[i], c.head >= 0 ? 3 * (5 + C) : c.cout, c.cin, c.k, sm);
    }
}

int main(int argc, char** argv) {
    printf("nms per %d threads %d max_boxes %d\n", kNmsPer, kNmsThreads, kMaxBoxes);
    printf("large nms above %d candidates max_candidates %d alive_bytes %d max_side %d grid_y %d\n", kNmsPer * kNmsThreads, kMaxCandidates,
           kLargeAliveBytes, kMaxSide, kMaxGridY);
    const std::string cmd = argc >= 2 ? argv[1] : "";
    if (argc >= 4 && (cmd == "net" || cmd == "tiny" || cmd == "net32" || cmd == "tiny32")) {
        const bool tiny = cmd.rfind("tiny", 0) == 0, fp32 = cmd.size() > 2 && cmd.substr(cmd.size() - 2) == "32";
        const int C = atoi(argv[2]), sm = atoi(argv[3]);
        if (argc >= 6) net(atoi(argv[4]), atoi(argv[5]), C, sm, tiny, fp32);
        else
            for (int h = 32; h <= 608; h += 32)
                for (int w = 32; w <= 608; w += 32) net(h, w, C, sm, tiny, fp32);
        return 0;
    }
    if (argc >= 3 && (cmd == "conv" || cmd == "conv32") && (argc - 3) % 5 == 0) {
        const int sm = atoi(argv[2]);
        for (int a = 3; a < argc; a += 5) {
            printf("%s ", cmd.c_str());
            (cmd == "conv32" ? plan32_line : plan_line)(atoi(argv[a]), atoi(argv[a + 1]), atoi(argv[a + 2]), atoi(argv[a + 3]), atoi(argv[a + 4]), sm);
        }
        return 0;
    }
    if (argc >= 5 && cmd == "split" && (argc - 2) % 3 == 0) {
        for (int a = 2; a < argc; a += 3) {
            const int Ho = atoi(argv[a]), Wo = atoi(argv[a + 1]), n = atoi(argv[a + 2]);
            const long long hw = (long long)Ho * Wo;
            printf("split Ho %d Wo %d n %d", Ho, Wo, n);
            for_each_frame_group(n, hw, [&](int f0, int nf) {          // the launchers' own grouping
                printf(" | f0 %d nf %d tiles %lld", f0, nf, (nf * hw + BM - 1) / BM);
                return 0;
            });
            printf("\n");
        }
        return 0;
    }
    fprintf(stderr, "usage: %s net|net32 C SM [H W] | tiny|tiny32 C SM [H W] | conv|conv32 SM Ho Wo N Cin k [...] | split Ho Wo n [...]\n", argv[0]);
    return 2;
}
