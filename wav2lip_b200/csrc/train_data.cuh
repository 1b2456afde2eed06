// train_data.cuh — the training scripts' batch assembly on the GPU: one gather launch turns B sampled (frame slots, mel rows)
// rows into exactly the tensors `default_collate` of B `Dataset.__getitem__` calls holds.
//   train_batch_wav2lip_kernel   wav2lip_train.py:111-164 (= hq_wav2lip_train.py): x, indiv_mels, mel, gt
//   train_batch_syncnet_kernel   color_syncnet_train.py:69-131: x, mel, y
// Frames are the cache's uint8 (96,96,3) BGR crops (device or pinned host memory, read through the same pointer); mels
// are the cache's (rows, 80) fp32 `orig_mel` rows.  A pixel is `float32(u / 255.)` with the division in float64, as NumPy
// does (u * (1/255.f) differs on 126 of the 256 byte values): a 256-entry shared-memory table built per block.
// HBM-bound: each thread reads 4 pixels (12 bytes, three 32-bit loads) and writes one float4 per channel.
#pragma once

#include <stdint.h>

namespace w2l {

constexpr int TD_W2L_FIELDS = 17;   // [0,5) window slots, [5,10) wrong-window slots, 10 mel row, [11,16) indiv rows, 16 video end
constexpr int TD_SYNC_FIELDS = 8;   // [0,5) window slots, 5 mel row, 6 label, 7 video end
constexpr int TD_T = 5, TD_S = 96, TD_MEL = 80, TD_STEP = 16;
constexpr long long TD_FRAME = TD_S * TD_S * 3;   // 27 648 bytes

__device__ __forceinline__ void td_build_lut(float* lut) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = (float)((double)i / 255.0);
    __syncthreads();
}

// 4 consecutive pixels of one frame row -> one float4 per channel (channel c = BGR byte c)
__device__ __forceinline__ void td_load_quad(const uint8_t* src, const float* lut, float4 ch[3]) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(src);
    const uint32_t w[3] = {p[0], p[1], p[2]};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int byte = 3 * k + c;
            v[k] = lut[(w[byte >> 2] >> (8 * (byte & 3))) & 0xffu];
        }
        ch[c] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// out (80,16) = mels[row : row + 16, :].T, as float4 stores of 4 consecutive columns: item = (m, j4)
__device__ __forceinline__ void td_mel_quad(const float* mels, long long row, int item, float* out) {
    const int j4 = item & 3, m = item >> 2;
    const float* s = mels + (row + 4 * j4) * TD_MEL + m;
    *reinterpret_cast<float4*>(out + m * TD_STEP + 4 * j4) = make_float4(s[0], s[TD_MEL], s[2 * TD_MEL], s[3 * TD_MEL]);
}

// x (B,6,5,96,96): channels 0-2 the window with rows 48-95 zeroed, 3-5 the wrong window; gt (B,3,5,96,96) the window;
// indiv_mels (B,5,1,80,16) windows at rows samples[11..15]; mel (B,1,80,16) the window at samples[10]
__global__ void __launch_bounds__(256) train_batch_wav2lip_kernel(const uint8_t* __restrict__ frames, const float* __restrict__ mels,
                                                                  const int* __restrict__ samples, int B, float* __restrict__ x,
                                                                  float* __restrict__ indiv, float* __restrict__ mel, float* __restrict__ gt) {
    __shared__ float lut[256];
    td_build_lut(lut);
    constexpr int Q = TD_S / 4, PLANE = TD_S * TD_S;
    const long long n_pix = (long long)B * 2 * TD_T * TD_S * Q;      // (b, window|wrong, t, y, quad)
    const long long n_mel = (long long)B * 6 * TD_MEL * 4;            // (b, mel|indiv 0..4, m, j4)
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_pix + n_mel; i += (long long)gridDim.x * blockDim.x) {
        if (i < n_pix) {
            const int q = (int)(i % Q), y = (int)((i / Q) % TD_S), t = (int)((i / (Q * TD_S)) % TD_T);
            const int w = (int)((i / (Q * TD_S * TD_T)) & 1), b = (int)(i / (2 * Q * TD_S * TD_T));
            const long long slot = samples[b * TD_W2L_FIELDS + w * TD_T + t];
            float4 ch[3];
            td_load_quad(frames + slot * TD_FRAME + y * TD_S * 3 + q * 12, lut, ch);
            const int pix = y * TD_S + 4 * q;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (w == 0) {
                    *reinterpret_cast<float4*>(gt + (((long long)b * 3 + c) * TD_T + t) * PLANE + pix) = ch[c];
                    // prepare_window + window[:, :, H//2:] = 0. (wav2lip_train.py:153-155)
                    *reinterpret_cast<float4*>(x + (((long long)b * 6 + c) * TD_T + t) * PLANE + pix) =
                        y >= TD_S / 2 ? make_float4(0.f, 0.f, 0.f, 0.f) : ch[c];
                } else {
                    *reinterpret_cast<float4*>(x + (((long long)b * 6 + 3 + c) * TD_T + t) * PLANE + pix) = ch[c];
                }
            }
        } else {
            const long long r = i - n_pix;
            const int item = (int)(r % (TD_MEL * 4)), k = (int)((r / (TD_MEL * 4)) % 6), b = (int)(r / (TD_MEL * 4 * 6));
            const int* s = samples + b * TD_W2L_FIELDS;
            float* out = k == 0 ? mel + (long long)b * TD_MEL * TD_STEP : indiv + ((long long)b * TD_T + k - 1) * TD_MEL * TD_STEP;
            td_mel_quad(mels, s[10 + k], item, out);
        }
    }
}

// x (B,15,48,96): channel 3t+c = rows 48-95 of frame t, channel c; mel (B,1,80,16) at samples[5]; y (B,1) = samples[6]
__global__ void __launch_bounds__(256) train_batch_syncnet_kernel(const uint8_t* __restrict__ frames, const float* __restrict__ mels,
                                                                  const int* __restrict__ samples, int B, float* __restrict__ x,
                                                                  float* __restrict__ mel, float* __restrict__ y) {
    __shared__ float lut[256];
    td_build_lut(lut);
    constexpr int Q = TD_S / 4, H2 = TD_S / 2;
    const long long n_pix = (long long)B * TD_T * H2 * Q;            // (b, t, row - 48, quad)
    const long long n_mel = (long long)B * TD_MEL * 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_pix + n_mel; i += (long long)gridDim.x * blockDim.x) {
        if (i < n_pix) {
            const int q = (int)(i % Q), yy = (int)((i / Q) % H2), t = (int)((i / (Q * H2)) % TD_T), b = (int)(i / (Q * H2 * TD_T));
            const long long slot = samples[b * TD_SYNC_FIELDS + t];
            float4 ch[3];
            td_load_quad(frames + slot * TD_FRAME + (H2 + yy) * TD_S * 3 + q * 12, lut, ch);
#pragma unroll
            for (int c = 0; c < 3; ++c)
                *reinterpret_cast<float4*>(x + (((long long)b * 15 + 3 * t + c) * H2 + yy) * TD_S + 4 * q) = ch[c];
        } else {
            const long long r = i - n_pix;
            const int item = (int)(r % (TD_MEL * 4)), b = (int)(r / (TD_MEL * 4));
            const int* s = samples + b * TD_SYNC_FIELDS;
            td_mel_quad(mels, s[5], item, mel + (long long)b * TD_MEL * TD_STEP);
            if (item == 0) y[b] = (float)s[6];
        }
    }
}

}  // namespace w2l
