// jpeg_api.h - what the JPEG encoder's and decoder's translation units (jpeg_api.cu, with jpeg_decode.inc) and the WHENet
// context's (whenet_api.cu) know of each other: the codecs keep their scratch in a State that the context owns, and run on the
// context's device and stream.
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

// The decoder (jpeg_decode.inc) keeps its scratch inside the encoder's State: dec_state selects the context's device,
// creates the State on first use and points slot at the decoder's pointer; destroy() frees it through destroy_dec.
struct DecState;
int dec_state(Target t, DecState**& slot);   // jpeg_api.cu
void destroy_dec(DecState* d);               // jpeg_decode.inc

}  // namespace jpeg
}  // namespace whenet
