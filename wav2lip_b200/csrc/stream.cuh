// stream.cuh — the one kernel of a streaming lip-sync step that the offline path does not have: the 16-frame mel
// chunks of a step's rows gathered out of the session's mel ring (mel.cuh, mel_ring_kernel) into the (N,1,80,16) layout
// the generator reads.  Chunk starts are absolute mel frame indices, read from the step's device table, so the launch
// itself has no per-step arguments and can be replayed from a CUDA graph.
#pragma once

#include <stdint.h>

namespace w2l {

// out[n][m][t] = ring[m][(starts[n] + t) & (pitch - 1)]
__global__ void mel_ring_gather_kernel(const float* ring, long long pitch, const int* starts, int N, float* out) {
    const int total = N * 80 * 16;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int t = i & 15, m = (i >> 4) % 80, n = i / 1280;
        out[i] = ring[(long long)m * pitch + (((long long)__ldg(starts + n) + t) & (pitch - 1))];
    }
}

}  // namespace w2l
