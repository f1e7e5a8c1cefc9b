// jpeg_api.h - what the JPEG encoder's translation unit (jpeg_api.cu) and the WHENet context's (whenet_api.cu) know of each
// other: the encoder keeps its scratch in a State that the context owns, and runs on the context's device and stream.
#pragma once
#include <cuda_runtime.h>

struct whenet_ctx;

namespace whenet {
namespace jpeg {

struct State;
struct Target {
    State** state;          // created on the first encode, freed by destroy() when the context is destroyed
    int device;
    cudaStream_t stream;
};
Target target(whenet_ctx* c);   // whenet_api.cu
void destroy(State* s);         // jpeg_api.cu

}  // namespace jpeg
}  // namespace whenet
