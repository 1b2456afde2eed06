// train_kernels.cuh — the memory-bound kernels of the training step (SURVEY.md section 8 f1) around the tensor-core
// convs: train-mode BatchNorm (batch statistics over the T*B flatten, conv.py:8-11 / wav2lip.py:93-94), its backward
// fused with the ReLU mask and the residual split (conv.py:16-19), the LeakyReLU backward of nonorm_Conv2d (conv.py:21-31),
// the generator head (wav2lip.py:84-85) forward / backward, the loss gradients of wav2lip_train.py:178-198,:227-229 and
// a multi-tensor Adam (torch.optim.Adam defaults, wav2lip_train.py:357-360).
//
// Activations are NHWC 16-bit (bf16 in training).  A "view" is (pointer to channel 0 of pixel 0, pixel pitch in
// elements): a dense tensor or a channel slice of a skip-concat buffer.  Every kernel handles 8 channels per thread
// (16-byte accesses); all channel counts of the three networks are multiples of 16.
// Reductions are two-pass and deterministic: per-block partial sums in fp32 (a few hundred terms per thread), final
// sums over the blocks in fp64.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "aux_kernels.cuh"

namespace w2l {

constexpr int kBnThreads = 256;
constexpr float kBnEps = 1e-5f;       // nn.BatchNorm2d default, conv.py:10
constexpr float kBnMomentum = 0.1f;

template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        f[2 * j] = from16<kBF16>((uint16_t)(w[j] & 0xFFFFu));
        f[2 * j + 1] = from16<kBF16>((uint16_t)(w[j] >> 16));
    }
}
template <bool kBF16>
__device__ __forceinline__ uint4 pack8(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = (uint32_t)to16<kBF16>(f[2 * j]) | ((uint32_t)to16<kBF16>(f[2 * j + 1]) << 16);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// Per-channel partial reductions over pixels.  Thread layout: C/8 threads cover the channels of one pixel, blockDim /
// (C/8) pixels per block iteration.  MODE 0: sum z, sum z^2.  MODE 1 (BatchNorm backward): du = dy * (y > 0),
// sum du, sum du * zhat.  MODE 2 (nonorm backward): dz = dy * (y > 0 ? 1 : 0.01) is also WRITTEN to dz, sum dz.
struct ChanReduceParams {
    const uint16_t* z; long long z_pitch;    // pre-BN conv output (modes 0, 1)
    const uint16_t* dy; long long dy_pitch;  // modes 1, 2
    const uint16_t* y; long long y_pitch;    // modes 1, 2
    uint16_t* dz; long long dz_pitch;        // mode 2 output
    const float* stats;                      // mode 1: [4][C] mean, invstd, G = gamma * invstd, H = beta - mean * G
                                             // with y == nullptr (non-residual block) the ReLU mask is recomputed as
                                             // G z + H > 0 instead of re-reading y (one tensor pass less)
    float* partial;                          // [gridDim.x][2][C]
    long long M;                             // pixels
    int C;
};

template <bool kBF16, int MODE>
__global__ void __launch_bounds__(kBnThreads) chan_reduce_kernel(const ChanReduceParams p) {
    extern __shared__ float red_smem[];      // [rows][2][C]
    const int tpr = p.C >> 3;
    const int rows = kBnThreads / tpr;
    const int g = threadIdx.x % tpr, r = threadIdx.x / tpr;
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.0f;
    float G[8], H[8];
    if (MODE == 1 && r < rows && p.y == nullptr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { G[j] = p.stats[2 * p.C + g * 8 + j]; H[j] = p.stats[3 * p.C + g * 8 + j]; }
    }
    if (r < rows) {
        for (long long pix = (long long)blockIdx.x * rows + r; pix < p.M; pix += (long long)gridDim.x * rows) {
            float a[8];
            if (MODE == 0) {
                unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.z + pix * p.z_pitch) + g), a);
#pragma unroll
                for (int j = 0; j < 8; ++j) { s0[j] += a[j]; s1[j] = fmaf(a[j], a[j], s1[j]); }
            } else {
                float d[8], yv[8];
                unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.dy + pix * p.dy_pitch) + g), d);
                if (MODE != 1 || p.y != nullptr) unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.y + pix * p.y_pitch) + g), yv);
                if (MODE == 1) {
                    unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.z + pix * p.z_pitch) + g), a);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {   // sum du and sum du * z; the finalize kernel turns the latter into sum du * zhat
                        const bool on = p.y != nullptr ? yv[j] > 0.0f : fmaf(G[j], a[j], H[j]) > 0.0f;
                        const float du = on ? d[j] : 0.0f;
                        s0[j] += du;
                        s1[j] = fmaf(du, a[j], s1[j]);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        d[j] = yv[j] > 0.0f ? d[j] : 0.01f * d[j];
                        s0[j] += d[j];
                    }
                    *(reinterpret_cast<uint4*>(p.dz + pix * p.dz_pitch) + g) = pack8<kBF16>(d);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            red_smem[(r * 2 + 0) * p.C + g * 8 + j] = s0[j];
            red_smem[(r * 2 + 1) * p.C + g * 8 + j] = s1[j];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * p.C; i += kBnThreads) {
        float s = 0.0f;
        for (int rr = 0; rr < rows; ++rr) s += red_smem[rr * 2 * p.C + i];
        p.partial[(long long)blockIdx.x * 2 * p.C + i] = s;
    }
}

// Sum of the per-block partials of 32 consecutive channels in fp64: block = 32 channels x 32 slices of the block range
// (a one-thread-per-channel loop over ~600 partials is a 70 us latency chain; this is ~3 us).
constexpr int kFinThreads = 1024;
__device__ __forceinline__ void sum_partials_2(const float* partial, int nblk, int C, int c, bool cvalid, double* s_out, double* q_out) {
    __shared__ double sh[2][32][33];
    const int cl = threadIdx.x & 31, j = threadIdx.x >> 5;
    double s = 0.0, q = 0.0;
    if (cvalid)
        for (int b = j; b < nblk; b += 32) { s += (double)partial[(long long)b * 2 * C + c]; q += (double)partial[(long long)b * 2 * C + C + c]; }
    sh[0][j][cl] = s; sh[1][j][cl] = q;
    __syncthreads();
    if (j == 0) {
        s = 0.0; q = 0.0;
#pragma unroll 8
        for (int k = 0; k < 32; ++k) { s += sh[0][k][cl]; q += sh[1][k][cl]; }
    }
    *s_out = s; *q_out = q;
}

// Batch statistics from the partial sums; running averages updated as nn.BatchNorm2d does in train mode (momentum 0.1,
// unbiased variance).  The conv bias never enters the conv kernel in train mode (BatchNorm removes any per-channel
// constant): it only shifts the batch mean, so it is added here, for running_mean.   grid = ceil(C / 32), block = 1024.
__global__ void __launch_bounds__(kFinThreads) bn_finalize_kernel(const float* partial, int nblk, int C, double m, const float* bias, float* rmean,
                                                                  float* rvar, const float* gamma, const float* beta, float* stats) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    double s, q;
    sum_partials_2(partial, nblk, C, c, c < C, &s, &q);
    if ((threadIdx.x >> 5) != 0 || c >= C) return;
    const double mean = s / m;
    double var = q / m - mean * mean;
    if (var < 0.0) var = 0.0;
    const float istd = (float)(1.0 / sqrt(var + (double)kBnEps));
    stats[c] = (float)mean;
    stats[C + c] = istd;
    if (gamma) {   // y = relu(G z + H [+ x])
        const float G = gamma[c] * istd;
        stats[2 * C + c] = G;
        stats[3 * C + c] = beta[c] - (float)mean * G;
    }
    if (rmean) rmean[c] = (1.0f - kBnMomentum) * rmean[c] + kBnMomentum * (float)(mean + (bias ? (double)bias[c] : 0.0));
    if (rvar) rvar[c] = (1.0f - kBnMomentum) * rvar[c] + kBnMomentum * (float)(m > 1.0 ? var * m / (m - 1.0) : var);
}

// y = relu(gamma * zhat + beta [+ res])   (conv.py:15-19 with batch statistics); optional fp32 copy (last block of SyncNet)
struct BnApplyParams {
    const uint16_t* z; long long z_pitch;
    const uint16_t* res; long long res_pitch;   // nullptr = no residual
    uint16_t* y; long long y_pitch;
    float* y_f32;                               // nullptr or dense [M][C]
    const float* stats;                         // [4][C]: mean, invstd, G, H
    long long M; int C;
};

// Thread layout as in chan_reduce_kernel: thread = (pixel row r, channel group g); the per-channel constants of the
// thread's 8 channels live in registers for the whole pixel loop (no per-element table loads).
template <bool kBF16>
__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(const BnApplyParams p) {
    const int tpr = p.C >> 3;
    const int rows = kBnThreads / tpr;
    const int g = threadIdx.x % tpr, r = threadIdx.x / tpr;
    if (r >= rows) return;
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = p.stats[2 * p.C + g * 8 + j]; sh[j] = p.stats[3 * p.C + g * 8 + j]; }   // G, H
    for (long long pix = (long long)blockIdx.x * rows + r; pix < p.M; pix += (long long)gridDim.x * rows) {
        float a[8], o[8];
        unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.z + pix * p.z_pitch) + g), a);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(a[j], sc[j], sh[j]);
        if (p.res) {
            float rr[8];
            unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.res + pix * p.res_pitch) + g), rr);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += rr[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j], 0.0f);
        *(reinterpret_cast<uint4*>(p.y + pix * p.y_pitch) + g) = pack8<kBF16>(o);
        if (p.y_f32) {
            float4* f = reinterpret_cast<float4*>(p.y_f32 + pix * p.C + g * 8);
            f[0] = make_float4(o[0], o[1], o[2], o[3]);
            f[1] = make_float4(o[4], o[5], o[6], o[7]);
        }
    }
}

// BatchNorm backward, second half: per-channel sums -> dgamma, dbeta and the three coefficients of
//   dz = c1 * (du - c2 - zhat * c3) = P du + Q z + R,   c1 = gamma * invstd, c2 = mean(du), c3 = mean(du * zhat).
__global__ void __launch_bounds__(kFinThreads) bn_bwd_finalize_kernel(const float* partial, int nblk, int C, double m, const float* gamma,
                                                                      const float* stats, float* dgamma, float* dbeta, int accumulate, float* coef) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    double s, q;
    sum_partials_2(partial, nblk, C, c, c < C, &s, &q);      // s = sum du, q = sum du * z
    if ((threadIdx.x >> 5) != 0 || c >= C) return;
    const double mean = stats[c], istd = stats[C + c];
    const double dg = istd * (q - mean * s);                 // sum du * zhat
    if (dbeta) dbeta[c] = accumulate ? dbeta[c] + (float)s : (float)s;
    if (dgamma) dgamma[c] = accumulate ? dgamma[c] + (float)dg : (float)dg;
    // dz = c1 (du - c2 - zhat c3), c1 = gamma istd, c2 = s/m, c3 = dg/m, zhat = istd z - mean istd
    //    = P du + Q z + R
    const double c1 = (double)gamma[c] * istd, c2 = s / m, c3 = dg / m;
    coef[c] = (float)c1;
    coef[C + c] = (float)(-c1 * c3 * istd);
    coef[2 * C + c] = (float)(c1 * c3 * mean * istd - c1 * c2);
}

struct BnBwdApplyParams {
    const uint16_t* z; long long z_pitch;
    const uint16_t* dy; long long dy_pitch;
    const uint16_t* y; long long y_pitch;
    uint16_t* dz;          // dense [M][C]
    uint16_t* du;          // dense [M][C] or nullptr: gradient of the residual branch (conv.py:16-18: joins before the ReLU)
    const float* stats; const float* coef;   // stats [4][C] (mean, invstd, G, H), coef [3][C] (P, Q, R)
    long long M; int C;                      // y == nullptr (non-residual block): mask from G z + H > 0
};

template <bool kBF16>
__global__ void __launch_bounds__(kBnThreads, 4) bn_bwd_apply_kernel(const BnBwdApplyParams p) {
    const int tpr = p.C >> 3;
    const int rows = kBnThreads / tpr;
    const int g = threadIdx.x % tpr, r = threadIdx.x / tpr;
    if (r >= rows) return;
    const bool from_z = p.y == nullptr;
    float P[8], Q[8], R[8], G[8], H[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = g * 8 + j;
        P[j] = p.coef[c]; Q[j] = p.coef[p.C + c]; R[j] = p.coef[2 * p.C + c];
        G[j] = from_z ? p.stats[2 * p.C + c] : 0.0f; H[j] = from_z ? p.stats[3 * p.C + c] : 0.0f;
    }
    for (long long pix = (long long)blockIdx.x * rows + r; pix < p.M; pix += (long long)gridDim.x * rows) {
        float a[8], d[8], yv[8], o[8];
        unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.z + pix * p.z_pitch) + g), a);
        unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.dy + pix * p.dy_pitch) + g), d);
        if (!from_z) unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.y + pix * p.y_pitch) + g), yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const bool on = from_z ? fmaf(G[j], a[j], H[j]) > 0.0f : yv[j] > 0.0f;
            d[j] = on ? d[j] : 0.0f;
            o[j] = fmaf(P[j], d[j], fmaf(Q[j], a[j], R[j]));
        }
        *(reinterpret_cast<uint4*>(p.dz + pix * p.C) + g) = pack8<kBF16>(o);
        if (p.du) *(reinterpret_cast<uint4*>(p.du + pix * p.C) + g) = pack8<kBF16>(d);
    }
}

// per-channel sums of MODE 2 -> conv bias gradient of a nonorm block
__global__ void __launch_bounds__(kFinThreads) bias_grad_finalize_kernel(const float* partial, int nblk, int C, float* db, int accumulate) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    double s, q;
    sum_partials_2(partial, nblk, C, c, c < C, &s, &q);
    if ((threadIdx.x >> 5) != 0 || c >= C) return;
    db[c] = accumulate ? db[c] + (float)s : (float)s;
}

__global__ void fill_kernel(float* p, long long n, float v) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

// ---- generator head: output_block.1 (Conv2d(32,3,1)) + Sigmoid, wav2lip.py:84-85, with the 5-D unflatten of :119-120 ----
// n = t*B + b  ->  g[b][oc][t][y][x]   (T = 1, B = N for the 4-D call)
struct HeadParams {
    const uint16_t* y32; long long y_pitch;   // output_block.0 result, 32 channels
    const float* w; const float* b;           // (3,32), (3)
    float* g;                                 // generator output, fp32
    const float* dg;                          // backward: dL/dg, same layout
    uint16_t* dy32;                           // backward: dense [M][32]
    float* partial;                           // backward: [gridDim.x][99]  (96 dW + 3 db)
    int N, B, T, HW;                          // HW = 96*96
};

template <bool kBF16>
__global__ void __launch_bounds__(256) head_fwd_kernel(const HeadParams p) {
    __shared__ float sw[99];
    if (threadIdx.x < 96) sw[threadIdx.x] = p.w[threadIdx.x];
    if (threadIdx.x < 3) sw[96 + threadIdx.x] = p.b[threadIdx.x];
    __syncthreads();
    const long long M = (long long)p.N * p.HW;
    for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < M; pix += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(pix / p.HW), hw = (int)(pix % p.HW);
        const int b = n % p.B, t = n / p.B;
        float f[32];
#pragma unroll
        for (int q = 0; q < 4; ++q) unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.y32 + pix * p.y_pitch) + q), f + 8 * q);
#pragma unroll
        for (int oc = 0; oc < 3; ++oc) {
            float s = sw[96 + oc];
#pragma unroll
            for (int j = 0; j < 32; ++j) s = fmaf(f[j], sw[oc * 32 + j], s);
            p.g[(((long long)b * 3 + oc) * p.T + t) * p.HW + hw] = 1.0f / (1.0f + __expf(-s));
        }
    }
}

template <bool kBF16>
__global__ void __launch_bounds__(256) head_bwd_kernel(const HeadParams p) {
    __shared__ float sw[96];
    __shared__ float red[8][99];
    if (threadIdx.x < 96) sw[threadIdx.x] = p.w[threadIdx.x];
    __syncthreads();
    float acc[99];
#pragma unroll
    for (int i = 0; i < 99; ++i) acc[i] = 0.0f;
    const long long M = (long long)p.N * p.HW;
    for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < M; pix += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(pix / p.HW), hw = (int)(pix % p.HW);
        const int b = n % p.B, t = n / p.B;
        float f[32], dl[3], o[32];
#pragma unroll
        for (int q = 0; q < 4; ++q) unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.y32 + pix * p.y_pitch) + q), f + 8 * q);
#pragma unroll
        for (int oc = 0; oc < 3; ++oc) {
            const long long gi = (((long long)b * 3 + oc) * p.T + t) * p.HW + hw;
            const float gv = __ldg(p.g + gi);
            dl[oc] = __ldg(p.dg + gi) * gv * (1.0f - gv);   // through the sigmoid
            acc[96 + oc] += dl[oc];
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            o[j] = dl[0] * sw[j] + dl[1] * sw[32 + j] + dl[2] * sw[64 + j];
            acc[j] = fmaf(dl[0], f[j], acc[j]);
            acc[32 + j] = fmaf(dl[1], f[j], acc[32 + j]);
            acc[64 + j] = fmaf(dl[2], f[j], acc[64 + j]);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) *(reinterpret_cast<uint4*>(p.dy32 + pix * 32) + q) = pack8<kBF16>(o + 8 * q);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 99; ++i) {
        float v = acc[i];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < 99) {
        float v = 0.0f;
        for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
        p.partial[(long long)blockIdx.x * 99 + threadIdx.x] = v;
    }
}

__global__ void head_bwd_finalize_kernel(const float* partial, int nblk, float* dw, float* db, int accumulate) {
    const int i = threadIdx.x;
    if (i >= 99) return;
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += (double)partial[(long long)b * 99 + i];
    float* o = i < 96 ? dw + i : db + (i - 96);
    *o = accumulate ? *o + (float)s : (float)s;
}

// ---- disc head: binary_pred = Conv2d(512,1,1) + Sigmoid on the (N,512) feature (wav2lip.py:152), backward ----
// given dL/dprob: dfeat[n][c] = dlogit[n] * w[c]; dw[c] = sum_n dlogit[n] * feat[n][c]; db = sum_n dlogit[n]
template <bool kBF16>
__global__ void disc_head_bwd_kernel(const uint16_t* feat, int pitch, const float* w, const float* prob, const float* dprob, int N,
                                     int D, uint16_t* dfeat, float* dw, float* db, int accumulate) {
    // one block; N is a few thousand rows at most, D = 512: column sums in a fixed order
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        float s = 0.0f;
        const float wc = w[c];
        for (int n = 0; n < N; ++n) {
            const float pv = prob[n];
            const float dl = dprob[n] * pv * (1.0f - pv);
            s = fmaf(dl, from16<kBF16>(feat[(long long)n * pitch + c]), s);
            dfeat[(long long)n * D + c] = to16<kBF16>(dl * wc);
        }
        dw[c] = accumulate ? dw[c] + s : s;
    }
    if (threadIdx.x == 0) {
        float s = 0.0f;
        for (int n = 0; n < N; ++n) { const float pv = prob[n]; s += dprob[n] * pv * (1.0f - pv); }
        db[0] = accumulate ? db[0] + s : s;
    }
}

// ---- losses of wav2lip_train.py:178-198 / :227-229, gradients ----
// F.normalize backward (syncnet.py:62-63): e = r / max(||r||, 1e-12); dr = (de - e (e . de)) / max(||r||, 1e-12), 16-bit out
template <bool kBF16>
__global__ void l2norm_bwd_kernel(const float* raw, const float* de, uint16_t* draw, int B, int D) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* r = raw + (long long)row * D;
    const float* d = de + (long long)row * D;
    float srr = 0.0f, srd = 0.0f;
    for (int i = lane; i < D; i += 32) { srr = fmaf(r[i], r[i], srr); srd = fmaf(r[i], d[i], srd); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { srr += __shfl_xor_sync(0xffffffffu, srr, o); srd += __shfl_xor_sync(0xffffffffu, srd, o); }
    const float nrm = sqrtf(srr);
    const float inv = 1.0f / fmaxf(nrm, 1e-12f);
    // e . de = (r . de) * inv  (when the clamp is inactive); clamp active means e = r * 1e12 and the projection term vanishes
    const float proj = nrm > 1e-12f ? srd * inv * inv : 0.0f;
    for (int i = lane; i < D; i += 32) draw[(long long)row * D + i] = to16<kBF16>((d[i] - r[i] * proj) * inv);
}

// cosine_loss backward (wav2lip_train.py:178-183): d = cos_sim(a, v) (eps 1e-8), L = mean BCE(d, y) * scale.
//   dL/dd = scale / B * (d - y) / max(d (1 - d), 1e-12)  (torch's binary_cross_entropy backward)
//   dd/da = v / (|a||v|) - d a / |a|^2,  dd/dv symmetric.
__global__ void cosine_bce_bwd_kernel(const float* a, const float* v, const float* y, float scale, float* da, float* dv, int B, int D) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* ar = a + (long long)row * D;
    const float* vr = v + (long long)row * D;
    float saa = 0.0f, svv = 0.0f, sav = 0.0f;
    for (int i = lane; i < D; i += 32) { saa = fmaf(ar[i], ar[i], saa); svv = fmaf(vr[i], vr[i], svv); sav = fmaf(ar[i], vr[i], sav); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        saa += __shfl_xor_sync(0xffffffffu, saa, o);
        svv += __shfl_xor_sync(0xffffffffu, svv, o);
        sav += __shfl_xor_sync(0xffffffffu, sav, o);
    }
    const float na = fmaxf(sqrtf(saa), 1e-8f), nv = fmaxf(sqrtf(svv), 1e-8f);
    const float d = sav / (na * nv);
    const float t = y ? y[row] : 1.0f;
    const float dLdd = scale / (float)B * (d - t) / fmaxf(d * (1.0f - d), 1e-12f);
    for (int i = lane; i < D; i += 32) {
        da[(long long)row * D + i] = dLdd * (vr[i] / (na * nv) - d * ar[i] / (na * na));
        dv[(long long)row * D + i] = dLdd * (ar[i] / (na * nv) - d * vr[i] / (nv * nv));
    }
}

// dL/dg of the generator step (wav2lip_train.py:227-229 / hq_wav2lip_train.py:229-240):
//   l1_scale * sign(g - gt)  [+ dsync scattered from the expert's input gradient: lower half, channel 3t + c (:193-194)]
//   [+ ddisc scattered from the quality discriminator's input gradient: lower half, n = t*B + b (wav2lip.py:155-161)]
struct GenLossGradParams {
    const float* g; const float* gt; float* dg;
    const uint16_t* dsync;   // [B][48][96][16] or nullptr
    const uint16_t* ddisc;   // [T*B][48][96][16] or nullptr
    float l1_scale;
    int B, T;
};

template <bool kBF16>
__global__ void gen_loss_grad_kernel(const GenLossGradParams p) {
    const long long total = (long long)p.B * 3 * p.T * 9216;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % 96), yy = (int)((i / 96) % 96);
        const int t = (int)((i / 9216) % p.T), c = (int)((i / (9216LL * p.T)) % 3), b = (int)(i / (9216LL * p.T * 3));
        float d = 0.0f;
        if (p.g) {   // (null in the stand-alone bridge: only an input gradient is scattered, w2l_train_backward)
            const float diff = p.g[i] - p.gt[i];
            d = diff > 0.0f ? p.l1_scale : (diff < 0.0f ? -p.l1_scale : 0.0f);
        }
        if (yy >= 48) {
            if (p.dsync) d += from16<kBF16>(p.dsync[(((long long)b * 48 + (yy - 48)) * 96 + x) * 16 + 3 * t + c]);
            if (p.ddisc) d += from16<kBF16>(p.ddisc[((((long long)t * p.B + b) * 48 + (yy - 48)) * 96 + x) * 16 + c]);
        }
        p.dg[i] = d;
    }
}

// The three BCE terms of hq_wav2lip_train.py:233-252 from the discriminator's probabilities on g (p_fake) and on gt
// (p_real), n each, in one block (a fixed reduction order: deterministic):
//   loss[2] = BCE(p_fake, 1) (perceptual, 0 when disc_wt == 0), loss[4] = BCE(p_real, 1), loss[5] = BCE(p_fake, 0)
//   d_perc = disc_wt * dBCE(p_fake, 1)/dp;   d_fake = dBCE(p_fake, 0)/dp;   d_real = dBCE(p_real, 1)/dp
// torch's arithmetic: logs clamped at -100, dBCE/dp = (p - t) / max(p (1 - p), 1e-12) / n.
__global__ void __launch_bounds__(1024) disc_bce_kernel(const float* p_fake, const float* p_real, int n, float disc_wt, float* loss,
                                                        float* d_perc, float* d_fake, float* d_real) {
    __shared__ float sh[3][32];
    float s_perc = 0.0f, s_fake = 0.0f, s_real = 0.0f;
    const float inv_n = 1.0f / (float)n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float pf = p_fake[i], pr = p_real[i];
        s_perc -= fmaxf(logf(pf), -100.0f);
        s_fake -= fmaxf(log1pf(-pf), -100.0f);
        s_real -= fmaxf(logf(pr), -100.0f);
        const float qf = fmaxf(pf * (1.0f - pf), 1e-12f), qr = fmaxf(pr * (1.0f - pr), 1e-12f);
        // (torch's order: grad * (p - t) / max(...), then the mean's reciprocal — the autograd bridge's values bit for bit)
        d_perc[i] = disc_wt * (pf - 1.0f) / qf * inv_n;
        d_fake[i] = pf / qf * inv_n;
        d_real[i] = (pr - 1.0f) / qr * inv_n;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s_perc += __shfl_xor_sync(0xffffffffu, s_perc, o);
        s_fake += __shfl_xor_sync(0xffffffffu, s_fake, o);
        s_real += __shfl_xor_sync(0xffffffffu, s_real, o);
    }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s_perc; sh[1][threadIdx.x >> 5] = s_fake; sh[2][threadIdx.x >> 5] = s_real; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const bool on = threadIdx.x < (blockDim.x >> 5);
        s_perc = on ? sh[0][threadIdx.x] : 0.0f; s_fake = on ? sh[1][threadIdx.x] : 0.0f; s_real = on ? sh[2][threadIdx.x] : 0.0f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s_perc += __shfl_xor_sync(0xffffffffu, s_perc, o);
            s_fake += __shfl_xor_sync(0xffffffffu, s_fake, o);
            s_real += __shfl_xor_sync(0xffffffffu, s_real, o);
        }
        if (threadIdx.x == 0) {
            loss[2] = disc_wt > 0.0f ? s_perc * inv_n : 0.0f;
            loss[4] = s_real * inv_n;
            loss[5] = s_fake * inv_n;
        }
    }
}

// ---- multi-tensor Adam (torch.optim.Adam defaults: no weight decay, no amsgrad) ----
struct AdamTensor { float* p; const float* g; float* m; float* v; long long n; };
struct AdamParams {
    const AdamTensor* t;   // device table
    float lr, beta1, beta2, eps, bc1, bc2_sqrt;   // bias corrections 1 - beta1^t, sqrt(1 - beta2^t)
    float grad_scale;                             // 1 / world when the all-reduce summed
};

__global__ void adam_kernel(const AdamParams a) {
    const AdamTensor t = a.t[blockIdx.y];
    const float step = a.lr / a.bc1;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < t.n; i += (long long)gridDim.x * blockDim.x) {
        const float g = t.g[i] * a.grad_scale;
        const float m = a.beta1 * t.m[i] + (1.0f - a.beta1) * g;
        const float v = a.beta2 * t.v[i] + (1.0f - a.beta2) * g * g;
        t.m[i] = m;
        t.v[i] = v;
        t.p[i] -= step * m / (sqrtf(v) / a.bc2_sqrt + a.eps);
    }
}

// fp32 NCHW gradient <- NHWC 16-bit (tests / the autograd bridge: dL/dx of a block or a network input)
template <bool kBF16>
__global__ void export_grad_kernel(const uint16_t* src, long long pitch, float* dst, int N, int H, int W, int C) {
    const long long total = (long long)N * C * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        const int c = (int)((i / ((long long)W * H)) % C), n = (int)(i / ((long long)W * H * C));
        dst[i] = from16<kBF16>(src[(((long long)n * H + y) * W + x) * pitch + c]);
    }
}

}  // namespace w2l
