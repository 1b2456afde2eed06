// stream.cuh — the kernels of a streaming lip-sync step that the offline path does not have, for the lone session
// (w2l_stream_*) and stream groups (w2l_stream_group_*) alike: the 16-frame mel chunks of a step's rows gathered out of
// their sessions' mel rings (mel.cuh, mel_ring_kernel) into the (N,1,80,16) layout the generator reads, and per-row
// forms of the offline crop and paste; for stream groups, the audio scatter into many rings.
#pragma once

#include <stdint.h>

#include "resize.cuh"

namespace w2l {

// Every pointer a step reads or writes is in its device table, one GroupRow per row, so the whole step (gather, crop,
// generator, paste) is captured once per bucket size and replayed whatever sessions the rows belong to.  Chunk starts
// are absolute mel frame indices.
struct GroupRow {
    const float* mel;        // the session's mel ring, (80, pitch) row-major by absolute frame
    long long pitch;
    long long start;         // chunk start (absolute mel frame)
    const uint8_t* frames;   // the session's (F, H, W, 3) video
    uint8_t* dst;            // the output frame (H, W, 3); null for a padding row, which is not pasted
    int H, W, frame, y1, y2, x1, x2, pad;
};

// A piece of one session's new samples into its audio ring (or its input ring, when it resamples) at absolute
// positions [at, at + n): copied by the lone session, one block row (blockIdx.y) of group_scatter_kernel in a group.
struct GroupScatter {
    const float* src;        // the caller's pcm; in a group, host pcm is read from the packed upload
    float* ring;
    long long mask, at, n;
};

__global__ void group_scatter_kernel(const GroupScatter* d) {
    const GroupScatter s = d[blockIdx.y];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < s.n; i += (long long)gridDim.x * blockDim.x)
        s.ring[(s.at + i) & s.mask] = __ldg(s.src + i);
}

// out[n][m][t] = ring_n[m][(start_n + t) & (pitch_n - 1)]
__global__ void group_gather_kernel(const GroupRow* rows, int N, float* out) {
    const int total = N * 80 * 16;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int t = i & 15, m = (i >> 4) % 80, n = i / 1280;
        const GroupRow& r = rows[n];
        out[i] = r.mel[(long long)m * r.pitch + ((r.start + t) & (r.pitch - 1))];
    }
}

// crop_resize_kernel with a video, frame size and box per row
__global__ void group_crop_kernel(const GroupRow* rows, int N, int S, uint8_t* crops) {
    const long long total = (long long)N * S * S;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % S), oy = (int)((i / S) % S), n = (int)(i / ((long long)S * S));
        const GroupRow& r = rows[n];
        const ResizeAxis ax = resize_axis(ox, S, r.x2 - r.x1, true);
        const ResizeAxis ay = resize_axis(oy, S, r.y2 - r.y1, false);
        const uint8_t* src = r.frames + (((long long)r.frame * r.H + r.y1) * r.W + r.x1) * 3;
        uint8_t o[3];
        resize_pixel(src, (long long)r.W * 3, ax, ay, o);
        uint8_t* d = crops + i * 3;
        d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
    }
}

__device__ __forceinline__ void set_byte(uint32_t* w, int k, uint32_t v) {
    w[k >> 2] = (w[k >> 2] & ~(0xffu << (8 * (k & 3)))) | (v << (8 * (k & 3)));
}

// Bytes [o0, o0 + nb) (nb <= 16, o0 = 16 c) of one output frame: the source frame's bytes, with the pixels inside the box
// replaced by the prediction resized to the box (paste_kernel's arithmetic).  The first pixel touched starts R = o0 % 3
// = c % 3 bytes before o0; with R a template constant every byte index is a constant and the 16 bytes stay in registers.
template <int R>
__device__ __forceinline__ void paste_chunk(const GroupRow& r, const uint8_t* pred, int S, const uint8_t* src, int o0, int nb,
                                            bool vec) {
    uint32_t w[4];
    if (vec) {
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(src + o0));
        w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
    } else {
        w[0] = w[1] = w[2] = w[3] = 0;
#pragma unroll
        for (int k = 0; k < 16; ++k)
            if (k < nb) set_byte(w, k, __ldg(src + o0 + k));
    }
    const int p0 = o0 / 3;
    int y = p0 / r.W, x = p0 - y * r.W;
#pragma unroll
    for (int j = 0; j < 6; ++j) {   // pixels p0 .. p0 + 5 hold bytes o0 - R .. o0 - R + 17; past the frame, y >= H >= y2
        if (y >= r.y1 && y < r.y2 && x >= r.x1 && x < r.x2) {
            const ResizeAxis ax = resize_axis(x - r.x1, r.x2 - r.x1, S, true);
            const ResizeAxis ay = resize_axis(y - r.y1, r.y2 - r.y1, S, false);
            uint8_t o[3];
            resize_pixel(pred, (long long)S * 3, ax, ay, o);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int k = 3 * j + c - R;
                if (k >= 0 && k < 16) set_byte(w, k, o[c]);
            }
        }
        if (++x == r.W) { x = 0; ++y; }
    }
    if (vec) {
        *reinterpret_cast<uint4*>(r.dst + o0) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
        for (int k = 0; k < 16; ++k)
            if (k < nb) r.dst[o0 + k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    }
}

// paste_kernel with a video, frame size, box and destination per row: row blockIdx.y, its frame in 16-byte pieces
// striding over gridDim.x blocks (16-byte loads and stores when the source and destination frames are 16-byte aligned).
// Offsets within a frame are 32-bit (the host admits frames below 2^31 bytes): 64-bit division would bound the kernel.
__global__ void __launch_bounds__(256) group_paste_kernel(const uint8_t* pred, int S, const GroupRow* rows) {
    const GroupRow& r = rows[blockIdx.y];
    if (!r.dst) return;
    const int bytes = r.H * r.W * 3;
    const uint8_t* src = r.frames + (long long)r.frame * bytes;
    const uint8_t* pr = pred + (long long)blockIdx.y * S * S * 3;
    const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(r.dst)) & 15) == 0;
    const int chunks = (bytes + 15) / 16;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < chunks; c += gridDim.x * blockDim.x) {
        const int o0 = c * 16;
        const int nb = min(16, bytes - o0);
        const bool vec = aligned && nb == 16;
        switch (c % 3) {
            case 0: paste_chunk<0>(r, pr, S, src, o0, nb, vec); break;
            case 1: paste_chunk<1>(r, pr, S, src, o0, nb, vec); break;
            default: paste_chunk<2>(r, pr, S, src, o0, nb, vec); break;
        }
    }
}

}  // namespace w2l
