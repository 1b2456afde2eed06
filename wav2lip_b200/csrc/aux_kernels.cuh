// aux_kernels.cuh — the small data-movement / packing kernels around the conv kernel.
//   ingest:   fp32 NCHW / 5-D caller tensors -> NHWC 16-bit with channel padding, t-major flatten
//             (wav2lip.py:93-94, :158-161) and the lower-half crop (wav2lip.py:155-156) as index math.
//   pack_w:   fp32 conv / convT weights -> [tap][Cout_pad][Cin_pad] 16-bit K-major slabs.
//   fold_bn:  conv bias + BatchNorm running stats (conv.py:8-11, eps 1e-5) -> per-channel scale/shift.
//   l2norm:   F.normalize(p=2, dim=1) of syncnet.py:62-63.
//   disc_head: Conv2d(512,1,1) + Sigmoid of wav2lip.py:152.
//   export:   NHWC 16-bit slice -> NCHW fp32 (tests / debug only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace w2l {

template <bool kBF16>
__device__ __forceinline__ uint16_t to16(float f) {
    if constexpr (kBF16) {
        __nv_bfloat16 h = __float2bfloat16_rn(f);
        return *reinterpret_cast<uint16_t*>(&h);
    } else {
        __half h = __float2half_rn(f);
        return *reinterpret_cast<uint16_t*>(&h);
    }
}
template <bool kBF16>
__device__ __forceinline__ float from16(uint16_t u) {
    if constexpr (kBF16) {
        return __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&u));
    } else {
        return __half2float(*reinterpret_cast<__half*>(&u));
    }
}

struct IngestParams {
    const float* src;
    uint16_t* dst;      // [N][H][Wp][Cpad], image column x stored at column x + x_off (zero borders pre-set)
    int N, B;           // n = t*B + b
    int C, H, W, Cpad;
    int Wp, x_off;      // destination row pitch (pixels) and left border
    long long sB, sC, sT;  // source strides in elements for b, c, t
    int y_off, Wsrc;       // source row offset / row pitch
    int lo_off;            // > 0: split-operand mode, also write lo = x - fp16(x) at channel + lo_off
    int Cpix;              // channels per pixel of the destination (= Cpad, or 2*Cpad with a lo plane)
    int cgrp;              // > 0: destination channel c comes from source (group c / cgrp, channel c % cgrp):
    long long sG;          //      offset (c / cgrp) * sG + (c % cgrp) * sC — frames stacked on channels, wav2lip_train.py:194
};

__device__ __forceinline__ long long src_off(const IngestParams& p, int c) {
    return p.cgrp > 0 ? (long long)(c / p.cgrp) * p.sG + (long long)(c % p.cgrp) * p.sC : (long long)c * p.sC;
}

template <bool kBF16>
__global__ void ingest_kernel(const IngestParams p) {
    const long long total = (long long)p.N * p.H * p.W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % p.W);
        const int y = (int)((i / p.W) % p.H);
        const int n = (int)(i / ((long long)p.W * p.H));
        const int b = n % p.B, t = n / p.B;
        const float* s = p.src + b * p.sB + t * p.sT + (long long)(y + p.y_off) * p.Wsrc + x;
        uint16_t* d = p.dst + ((((long long)n * p.H + y) * p.Wp) + x + p.x_off) * p.Cpix;
        for (int c0 = 0; c0 < p.Cpad; c0 += 8) {
            uint16_t h[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = c0 + j;
                h[j] = (c < p.C) ? to16<kBF16>(__ldg(s + src_off(p, c))) : (uint16_t)0;
            }
            uint4 o;
            o.x = h[0] | ((uint32_t)h[1] << 16);
            o.y = h[2] | ((uint32_t)h[3] << 16);
            o.z = h[4] | ((uint32_t)h[5] << 16);
            o.w = h[6] | ((uint32_t)h[7] << 16);
            *reinterpret_cast<uint4*>(d + c0) = o;
            if (p.lo_off > 0) {
                uint16_t l[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = c0 + j;
                    l[j] = (c < p.C) ? to16<kBF16>(__ldg(s + src_off(p, c)) - from16<kBF16>(h[j])) : (uint16_t)0;
                }
                uint4 q;
                q.x = l[0] | ((uint32_t)l[1] << 16);
                q.y = l[2] | ((uint32_t)l[3] << 16);
                q.z = l[4] | ((uint32_t)l[5] << 16);
                q.w = l[6] | ((uint32_t)l[7] << 16);
                *reinterpret_cast<uint4*>(d + p.lo_off + c0) = q;
            }
        }
    }
}

// Same conversion, four horizontally adjacent pixels per thread: one 16-byte load per source channel (the NCHW planes
// are read with 4x the bytes in flight) and four 16-byte stores per 8 destination channels.  Needs W, the source row
// pitch and all source strides to be multiples of 4 elements and a 16-byte aligned source (checked by the caller);
// 16-bit modes only (no lo plane).
template <bool kBF16>
__global__ void ingest4_kernel(const IngestParams p) {
    const int W4 = p.W >> 2;
    const long long total = (long long)p.N * p.H * W4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W4) << 2;
        const int y = (int)((i / W4) % p.H);
        const int n = (int)(i / ((long long)W4 * p.H));
        const int b = n % p.B, t = n / p.B;
        const float* s = p.src + b * p.sB + t * p.sT + (long long)(y + p.y_off) * p.Wsrc + x;
        uint16_t* d = p.dst + ((((long long)n * p.H + y) * p.Wp) + x + p.x_off) * p.Cpix;
        for (int c0 = 0; c0 < p.Cpad; c0 += 8) {
            float4 v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = c0 + j;
                v[j] = (c < p.C) ? __ldg(reinterpret_cast<const float4*>(s + src_off(p, c))) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int px = 0; px < 4; ++px) {
                uint16_t h[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float f = px == 0 ? v[j].x : px == 1 ? v[j].y : px == 2 ? v[j].z : v[j].w;
                    h[j] = to16<kBF16>(f);
                }
                uint4 o;
                o.x = h[0] | ((uint32_t)h[1] << 16);
                o.y = h[2] | ((uint32_t)h[3] << 16);
                o.z = h[4] | ((uint32_t)h[5] << 16);
                o.w = h[6] | ((uint32_t)h[7] << 16);
                *reinterpret_cast<uint4*>(d + (long long)px * p.Cpix + c0) = o;
            }
        }
    }
}

// Batch assembly of inference.py:134-140 on the GPU: uint8 BGR crops (N,96,96,3) -> 6 channels
// [crop with rows >= H/2 zeroed | crop] / 255 (float64 division rounded to float32, as np.concatenate(...)/255.
// followed by torch.FloatTensor does), written in the first conv's input layout.
struct IngestU8Params {
    const unsigned char* src;  // (N, H, W, 3)
    uint16_t* dst;
    int N, H, W, Cpad, Wp, x_off;
    int lo_off;  // > 0: split-operand mode, also write the lo plane
    int Cpix;    // channels per pixel of the destination
};

template <bool kBF16>
__global__ void ingest_u8_kernel(const IngestU8Params p) {
    const long long total = (long long)p.N * p.H * p.W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % p.W);
        const int y = (int)((i / p.W) % p.H);
        const int n = (int)(i / ((long long)p.W * p.H));
        const unsigned char* s = p.src + i * 3;
        uint16_t h[8], l[8];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = (float)((double)s[c] / 255.0);
            h[3 + c] = to16<kBF16>(v);
            l[3 + c] = to16<kBF16>(v - from16<kBF16>(h[3 + c]));
            h[c] = (y >= p.H / 2) ? (uint16_t)0 : h[3 + c];
            l[c] = (y >= p.H / 2) ? (uint16_t)0 : l[3 + c];
        }
        h[6] = h[7] = 0;
        l[6] = l[7] = 0;
        uint16_t* d = p.dst + ((((long long)n * p.H + y) * p.Wp) + x + p.x_off) * p.Cpix;
        uint4 o;
        o.x = h[0] | ((uint32_t)h[1] << 16);
        o.y = h[2] | ((uint32_t)h[3] << 16);
        o.z = h[4] | ((uint32_t)h[5] << 16);
        o.w = 0u;
        *reinterpret_cast<uint4*>(d) = o;
        for (int c0 = 8; c0 < p.Cpad; c0 += 8) *reinterpret_cast<uint4*>(d + c0) = make_uint4(0u, 0u, 0u, 0u);
        if (p.lo_off > 0) {
            uint4 q;
            q.x = l[0] | ((uint32_t)l[1] << 16);
            q.y = l[2] | ((uint32_t)l[3] << 16);
            q.z = l[4] | ((uint32_t)l[5] << 16);
            q.w = 0u;
            *reinterpret_cast<uint4*>(d + p.lo_off) = q;
            for (int c0 = 8; c0 < p.Cpad; c0 += 8) *reinterpret_cast<uint4*>(d + p.lo_off + c0) = make_uint4(0u, 0u, 0u, 0u);
        }
    }
}

// Mel chunking of inference.py:231-240: chunk i = mel[:, start_i : start_i + 16], start_i = int(i * 80./fps);
// the last chunk is right-aligned (mel[:, F-16:]).  out is (n_chunks, 1, 80, 16) fp32.
__global__ void mel_chunk_kernel(const float* mel, long long F, double mult, int n_chunks, float* out) {
    const long long total = (long long)n_chunks * 80 * 16;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % 16);
        const int m = (int)((i / 16) % 80);
        const int c = (int)(i / 1280);
        long long start = (long long)((double)c * mult);
        if (start + 16 > F) start = F - 16;
        out[i] = mel[(long long)m * F + start + t];
    }
}

// NHWC 16-bit (channel slice of a buffer with channel pitch Cs) -> NCHW fp32
template <bool kBF16>
__global__ void export_kernel(const uint16_t* src, float* dst, int N, int H, int W, int C, int Cs, int f32src, int lo_off) {
    const long long total = (long long)N * C * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const int y = (int)((i / W) % H);
        const int c = (int)((i / ((long long)W * H)) % C);
        const int n = (int)(i / ((long long)W * H * C));
        const long long so = (((long long)n * H + y) * W + x) * Cs + c;
        dst[i] = f32src ? reinterpret_cast<const float*>(src)[so]
                        : from16<kBF16>(src[so]) + (lo_off > 0 ? from16<kBF16>(src[so + lo_off]) : 0.0f);
    }
}

struct PackParams {
    const float* src;
    uint16_t* dst;  // [ntaps][cout_pad][cin_pad]
    int ntaps, cout, cin, cout_pad, cin_pad;
    long long s_co, s_ci, s_r, s_s;  // source strides (elements)
    signed char r[49], s[49];        // filter coordinates of each packed tap
    int lo;                          // 1: pack w - fp16(w) (the lo plane of the split-operand mode)
};

template <bool kBF16>
__global__ void pack_w_kernel(const PackParams p) {
    const long long total = (long long)p.ntaps * p.cout_pad * p.cin_pad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % p.cin_pad);
        const int co = (int)((i / p.cin_pad) % p.cout_pad);
        const int t = (int)(i / ((long long)p.cin_pad * p.cout_pad));
        float v = 0.0f;
        if (ci < p.cin && co < p.cout) v = p.src[co * p.s_co + ci * p.s_ci + p.r[t] * p.s_r + p.s[t] * p.s_s];
        if (p.lo) v -= from16<kBF16>(to16<kBF16>(v));
        p.dst[i] = to16<kBF16>(v);
    }
}

// All weight slabs of a training plan in ONE launch (the slabs are re-packed from the fp32 masters every step: ~240 jobs).
// blk_job[b] = job of block b, blk_first[j] = first block of job j.
template <bool kBF16>
__global__ void pack_multi_kernel(const PackParams* jobs, const int* blk_job, const int* blk_first) {
    const int j = blk_job[blockIdx.x];
    const PackParams& p = jobs[j];
    const long long total = (long long)p.ntaps * p.cout_pad * p.cin_pad;
    const long long nblk = (total + 4095) / 4096;      // blocks of this job: 4096 elements each
    const long long b = blockIdx.x - blk_first[j];
    const long long end = (b + 1) * 4096 < total ? (b + 1) * 4096 : total;
    (void)nblk;
    for (long long i = b * 4096 + threadIdx.x; i < end; i += blockDim.x) {
        const int ci = (int)(i % p.cin_pad);
        const int co = (int)((i / p.cin_pad) % p.cout_pad);
        const int t = (int)(i / ((long long)p.cin_pad * p.cout_pad));
        float v = 0.0f;
        if (ci < p.cin && co < p.cout) v = p.src[co * p.s_co + ci * p.s_ci + p.r[t] * p.s_r + p.s[t] * p.s_s];
        p.dst[i] = to16<kBF16>(v);
    }
}

// "kw folded into K" packing for the first layers (tiny Cin): dst[r][co][s*Cp + c] = w[co][c][r][s]
struct PackFoldParams {
    const float* src;  // (cout, cin, kh, kw)
    uint16_t* dst;     // [kh][cout_pad][kfold]
    int kh, kw, cout, cin, cout_pad, kfold, Cp;
};

template <bool kBF16>
__global__ void pack_fold_kernel(const PackFoldParams p) {
    const long long total = (long long)p.kh * p.cout_pad * p.kfold;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % p.kfold);
        const int co = (int)((i / p.kfold) % p.cout_pad);
        const int r = (int)(i / ((long long)p.kfold * p.cout_pad));
        const int s = k / p.Cp, c = k % p.Cp;
        float v = 0.0f;
        if (s < p.kw && c < p.cin && co < p.cout) v = p.src[(((long long)co * p.cin + c) * p.kh + r) * p.kw + s];
        p.dst[i] = to16<kBF16>(v);
    }
}

// scale/shift of length reps*cout (replicated), padded with (0,0) up to n_pad
__global__ void fold_bn_kernel(const float* bias, const float* gamma, const float* beta, const float* mean,
                               const float* var, float eps, int cout, int reps, int n_pad, float* scale,
                               float* shift) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    if (i >= cout * reps) {
        scale[i] = 0.0f;
        shift[i] = 0.0f;
        return;
    }
    const int c = i % cout;
    const float b = bias ? bias[c] : 0.0f;
    if (gamma) {
        const float s = gamma[c] / sqrtf(var[c] + eps);
        scale[i] = s;
        shift[i] = (b - mean[c]) * s + beta[c];
    } else {
        scale[i] = 1.0f;
        shift[i] = b;
    }
}

// one warp per row of a (B, D) fp32 matrix: y = x / max(||x||_2, 1e-12)
__global__ void l2norm_kernel(const float* x, float* y, int B, int D) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* xr = x + (long long)row * D;
    float s = 0.0f;
    for (int i = lane; i < D; i += 32) s = fmaf(xr[i], xr[i], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv = 1.0f / fmaxf(sqrtf(s), 1e-12f);
    for (int i = lane; i < D; i += 32) y[(long long)row * D + i] = xr[i] * inv;
}

// one warp per row: prob = sigmoid(dot(x[row,:D], w) + b), x is 16-bit
template <bool kBF16>
__global__ void disc_head_kernel(const uint16_t* x, const float* w, const float* b, float* prob, int rows, int D, int pitch,
                                 int lo_off) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float s = 0.0f;
    for (int i = lane; i < D; i += 32) {
        float xv = from16<kBF16>(x[(long long)row * pitch + i]);
        if (lo_off > 0) xv += from16<kBF16>(x[(long long)row * pitch + lo_off + i]);
        s = fmaf(xv, w[i], s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) prob[row] = 1.0f / (1.0f + __expf(-(s + b[0])));
}

// ---- S3FD (face_detection/detection/sfd/net_s3fd.py) glue kernels ---------------------------------------------------------
// Both read and write NHWC 16-bit activations with pixel pitch Cs.  lo_off > 0 (split-operand mode, Cs = 2C): every value
// is hi + lo, the lo plane lo_off channels after the hi plane; both planes are read and both are written.

__device__ __forceinline__ uint16_t half_of(const uint4& q, int j) {
    const uint32_t w = (&q.x)[j >> 1];
    return (uint16_t)((j & 1) ? (w >> 16) : (w & 0xFFFFu));
}
__device__ __forceinline__ uint4 pack8(const uint16_t* o) {
    return make_uint4(o[0] | ((uint32_t)o[1] << 16), o[2] | ((uint32_t)o[3] << 16), o[4] | ((uint32_t)o[5] << 16),
                      o[6] | ((uint32_t)o[7] << 16));
}

// F.max_pool2d(h, 2, 2) (net_s3fd.py:74,78,84,90,96): floor semantics, 8 channels per thread.  Split operands: the
// window's largest hi + lo wins and both of its planes are copied, so the pool is exact in every mode.
template <bool kBF16>
__global__ void maxpool2_kernel(const uint16_t* in, uint16_t* out, int N, int H, int W, int C, int Cs, int lo_off) {
    const int Ho = H >> 1, Wo = W >> 1, cg = C >> 3;
    const long long total = (long long)N * Ho * Wo * cg;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int g = (int)(i % cg);
        const int x = (int)((i / cg) % Wo), y = (int)((i / ((long long)cg * Wo)) % Ho), n = (int)(i / ((long long)cg * Wo * Ho));
        const long long row = (long long)W * Cs;
        const uint16_t* p = in + ((((long long)n * H + 2 * y) * W + 2 * x) * Cs) + g * 8;
        const uint16_t* po[4] = {p, p + Cs, p + row, p + row + Cs};
        uint4 q[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) q[k] = __ldg(reinterpret_cast<const uint4*>(po[k]));
        uint16_t* d = out + ((((long long)n * Ho + y) * Wo + x) * Cs) + g * 8;
        uint16_t o[8];
        if (lo_off > 0) {
            uint4 l[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) l[k] = __ldg(reinterpret_cast<const uint4*>(po[k] + lo_off));
            uint16_t ol[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                int best = 0;
                float m = from16<kBF16>(half_of(q[0], j)) + from16<kBF16>(half_of(l[0], j));
#pragma unroll
                for (int k = 1; k < 4; ++k) {
                    const float v = from16<kBF16>(half_of(q[k], j)) + from16<kBF16>(half_of(l[k], j));
                    if (v > m) { m = v; best = k; }
                }
                o[j] = half_of(q[best], j);
                ol[j] = half_of(l[best], j);
            }
            *reinterpret_cast<uint4*>(d + lo_off) = pack8(ol);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float m = -3.4e38f;
#pragma unroll
                for (int k = 0; k < 4; ++k) m = fmaxf(m, from16<kBF16>(half_of(q[k], j)));
                o[j] = to16<kBF16>(m);
            }
        }
        *reinterpret_cast<uint4*>(d) = pack8(o);
    }
}

// L2Norm (net_s3fd.py:6-19): x / (sqrt(sum_c x^2) + 1e-10) * weight[c]; one warp per pixel.  Split operands: x = hi + lo
// (exact in fp32), y is stored as to16(y) and to16(y - hi).
template <bool kBF16>
__global__ void chan_l2norm_kernel(const uint16_t* in, uint16_t* out, const float* weight, long long pixels, int C, int Cs,
                                   int lo_off) {
    const long long pix = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pix >= pixels) return;
    const uint16_t* p = in + pix * Cs;
    uint16_t* q = out + pix * Cs;
    auto val = [&](int c) { return lo_off > 0 ? from16<kBF16>(p[c]) + from16<kBF16>(p[c + lo_off]) : from16<kBF16>(p[c]); };
    float s = 0.0f;
    for (int c = lane; c < C; c += 32) { const float v = val(c); s = fmaf(v, v, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv = 1.0f / (sqrtf(s) + 1e-10f);
    for (int c = lane; c < C; c += 32) {
        const float y = val(c) * inv * __ldg(weight + c);
        const uint16_t h = to16<kBF16>(y);
        q[c] = h;
        if (lo_off > 0) q[c + lo_off] = to16<kBF16>(y - from16<kBF16>(h));
    }
}

// mbox head (fp32 NHWC, 16-channel pitch) -> the module's NCHW fp32 output; maxout: cls1 = [max(c0,c1,c2), c3] (net_s3fd.py:123-126)
__global__ void s3fd_export_kernel(const float* in, float* out, int N, int H, int W, int Cout, int maxout) {
    const long long total = (long long)N * Cout * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        const int c = (int)((i / ((long long)W * H)) % Cout), n = (int)(i / ((long long)W * H * Cout));
        const float* p = in + (((long long)n * H + y) * W + x) * 16;
        out[i] = maxout ? (c == 0 ? fmaxf(fmaxf(p[0], p[1]), p[2]) : p[3]) : p[c];
    }
}

// ---- evaluation-loop losses (wav2lip_train.py:178-198, 262-292; color_syncnet_train.py:133-138) -------------------------
// cosine_loss: d = F.cosine_similarity(a, v) (eps 1e-8), loss = nn.BCELoss()(d.unsqueeze(1), y) — mean over the batch,
// log terms clamped at -100 as torch does.  One warp per row, per-row terms to `terms`, then a single block sums them in
// a fixed order (deterministic).  y == nullptr means a vector of ones (get_sync_loss, wav2lip_train.py:197).
__global__ void cosine_bce_terms_kernel(const float* a, const float* v, const float* y, float* terms, int B, int D) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* ar = a + (long long)row * D;
    const float* vr = v + (long long)row * D;
    float saa = 0.0f, svv = 0.0f, sav = 0.0f;
    for (int i = lane; i < D; i += 32) {
        const float x = ar[i], z = vr[i];
        saa = fmaf(x, x, saa); svv = fmaf(z, z, svv); sav = fmaf(x, z, sav);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        saa += __shfl_xor_sync(0xffffffffu, saa, o);
        svv += __shfl_xor_sync(0xffffffffu, svv, o);
        sav += __shfl_xor_sync(0xffffffffu, sav, o);
    }
    if (lane == 0) {
        const float d = sav / (fmaxf(sqrtf(saa), 1e-8f) * fmaxf(sqrtf(svv), 1e-8f));
        const float t = y ? y[row] : 1.0f;
        const float l1 = fmaxf(logf(d), -100.0f), l0 = fmaxf(logf(1.0f - d), -100.0f);
        terms[row] = -(t * l1 + (1.0f - t) * l0);
    }
}

// out[0] = scale * sum(x[0..n)) in a fixed order (one block)
__global__ void sum_scale_kernel(const float* x, float* out, int n, float scale) {
    __shared__ float sh[32];
    float s = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += x[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (threadIdx.x == 0) out[0] = s * scale;
    }
}

// nn.L1Loss() partial sums: partial[block] = sum |x - y| over the block's grid-stride share (16-byte loads; HBM-bound:
// 8 bytes read per element pair).  The tail (n % 4) is handled by block 0.
__global__ void l1_partial_kernel(const float* x, const float* y, float* partial, long long n) {
    __shared__ float sh[32];
    const long long n4 = n >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* y4 = reinterpret_cast<const float4*>(y);
    float s = 0.0f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n4; i += 4 * stride) {  // four independent 16-byte load pairs in flight per thread
        float4 a[4], b[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { a[u] = __ldg(x4 + i + u * stride); b[u] = __ldg(y4 + i + u * stride); }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            s += fabsf(a[u].x - b[u].x) + fabsf(a[u].y - b[u].y) + fabsf(a[u].z - b[u].z) + fabsf(a[u].w - b[u].w);
    }
    for (; i < n4; i += stride) {
        const float4 a = __ldg(x4 + i), b = __ldg(y4 + i);
        s += fabsf(a.x - b.x) + fabsf(a.y - b.y) + fabsf(a.z - b.z) + fabsf(a.w - b.w);
    }
    if (blockIdx.x == 0)
        for (long long i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) s += fabsf(x[i] - y[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (threadIdx.x == 0) partial[blockIdx.x] = s;
    }
}

}  // namespace w2l
