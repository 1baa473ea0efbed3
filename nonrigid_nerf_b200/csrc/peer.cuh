// Peer-memory (NVLink, CUDA IPC) gradient reduction fused into the optimizer step, and a small row all-gather (peer.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "adam.cuh"

namespace nrn {

constexpr int kPeerMaxRanks = 8;       // one NVSwitch domain of an 8-GPU H100 node
constexpr int kPeerArrive = 0;         // flag rows inside a window: [3][kPeerMaxRanks] u32, then padding to kPeerFlagBytes
constexpr int kPeerDone = 1;
constexpr int kPeerGather = 2;
constexpr size_t kPeerFlagBytes = 1024;

struct PeerCtx {
  uint8_t* window[kPeerMaxRanks];      // every rank's window as mapped into THIS process (own rank: the local allocation)
  int world, rank;
  size_t slot_off, slot_bytes;         // two row slots (double buffered) behind the flags
  size_t arena_off;                    // gradient arena behind the slots
};

// epoch_word: device u32[3] (one epoch per flag row, zero-initialised); done_counter: device u32, zero-initialised
cudaError_t launch_peer_reduce_adam(const PeerCtx& c, const AdamParams& a, int n_tensors, int n_blocks, long long total,
                                    uint32_t* epoch_word, float* gsum, unsigned int* done_counter, int* err, cudaStream_t st);
cudaError_t launch_peer_gather(const PeerCtx& c, uint32_t* epoch_word, const float* local, int n_per_rank, float* out, int* err,
                               cudaStream_t st);

}  // namespace nrn
