// frames_api.h - what the frame crops and overlays' translation unit (frames_api.cu) and the WHENet context's (whenet_api.cu)
// know of each other: the frame code keeps its device buffers in a State that the context owns, runs on the context's device
// and stream, and counts and profiles its launches through the context's Scope.
#pragma once
#include <cuda_runtime.h>

struct whenet_ctx;

namespace whenet {

// A launch of the context (defined in whenet_api.cu): counted by whenet_launch_count and, while profiling is on, timed on
// `stream` from construction to destruction under `name` for whenet_profile_read.
struct Scope {
    Scope(whenet_ctx* ctx, cudaStream_t stream, const char* name, double bytes, double flops);
    ~Scope();
    whenet_ctx* c;
    cudaStream_t s;
    int ev = -1;
};

namespace frames {

struct State;
struct Target {
    State** state;          // created on first use, freed by destroy() when the context is destroyed
    int device;
    cudaStream_t stream;
};
Target target(whenet_ctx* c);   // whenet_api.cu
void destroy(State* s);         // frames_api.cu

}  // namespace frames
}  // namespace whenet
