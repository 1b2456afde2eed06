// wgrad.cuh — weight gradients of the conv blocks (training row, SURVEY.md section 8 f1) on the Hopper tensor cores
// (wgmma): the contraction runs over PIXELS.
//
//   Conv2d           (conv.py:5-19)   dW[co][ci][r][s]   = sum_{n,y,x} dz[n,y,x,co] * x[n, y*sy - ph + r, x*sx - pw + s, ci]
//   Conv2dTranspose  (conv.py:33-44)  dW_t[ci][co][r][s] = sum_{n,y,x} x[n,y,x,ci]  * dz[n, y*sy - ph + r, x*sx - pw + s, co]
//
// i.e. in both cases  D_t[m][n] = sum_pix S[pix][m] * T_t[pix'(pix, t)][n]  per filter tap t, where S ("shared") is the
// tensor living on the dense pixel grid of the sum (dz for a conv, x for a transposed conv) and T ("per tap") is the other
// one, read at a strided, tap-shifted position (zero outside the image: exactly the forward's zero padding).  Both tensors
// are NHWC 16-bit, channels contiguous — so as GEMM operands with K = pixels they are **MN-major**: a TMA box of
// (64 channels x P pixels) lands as P rows of 128 bytes with the hardware 128-byte swizzle, which is the canonical
// MN-major SWIZZLE_128B layout of the wgmma shared-memory descriptor (rows = K, 8-row groups SBO = 1024 B apart,
// 64-channel atoms LBO = P*128 B apart); both operands are issued transposed (imm-trans-a = imm-trans-b = 1).  No
// transposed copy of any activation is ever made.
//
//   warp 0  : TMA producer.  Per K chunk (a bw x bh x bn box of P pixels of the shared grid): 2 loads of the shared
//             operand's 128-channel tile and, for each tap of the CTA's tap group, the per-tap operand's BN-channel tile
//             at the shifted / strided position (TMA element strides = the conv stride, out-of-bounds zero fill).
//   warps 4-7: one consumer warpgroup.  Every tap owns BN accumulator columns (registers; taps x BN <= 128), so the shared
//             operand is loaded ONCE per chunk for the whole tap group: per chunk P/16 x taps x 2 wgmma m64nBNk16.  Then
//             the fp32 partial tile goes to the workspace ws[split][tap][m][n].
// Split-K over CTAs (a unit = m tile x n tile x tap group x K split) with a deterministic second pass
// (wgrad_reduce_kernel) that sums the splits in a fixed order and writes the PyTorch parameter layout [m][n][tap].
#pragma once

#include "conv_igemm.cuh"

namespace w2l {

constexpr int kWgThreads = 256;  // the producer warpgroup + one consumer warpgroup
constexpr int kWgMaxTaps = 49;
constexpr int kWgMaxCols = 128;  // accumulator columns (taps x BN) of one unit: registers of one warpgroup

struct alignas(64) WgradParams {
    CUtensorMap tmS;  // shared operand: dims (C, W, H, N), box (64, bw, bh, bn), SWIZZLE_128B
    CUtensorMap tmT;  // per-tap operand: dims (C, W, H, N), box (min(BN,64), bw*sx, bh*sy, bn), element strides (1,sx,sy,1)
    int tiles_x, tiles_y, tiles_n;  // K chunks = boxes over the shared operand's pixel grid
    int bw, bh, bn, P;              // P = bw*bh*bn pixels per chunk (multiple of 16)
    int sx, sy;                     // pixels of the per-tap operand per pixel of the shared one
    int m_tiles, n_tiles;           // 128-channel tiles of S, BN-channel tiles of T
    int ntaps, ngroups, tg;         // taps, tap groups, taps per group (the last group may be shorter)
    int splits;                     // K splits
    long long chunks;               // total K chunks
    int stages;
    unsigned stage_bytes;           // shared memory per pipeline stage
    unsigned a_bytes;               // bytes of the S part of a stage = 2 atoms * P * 128
    unsigned tap_bytes;             // bytes of one tap's T part = P * BN * 2
    float* ws;                      // [splits][ntaps][m_tiles*128][n_tiles*BN] fp32 partial sums
    signed char dx[kWgMaxTaps], dy[kWgMaxTaps];  // offset of the per-tap operand for each tap (r - ph, s - pw)
};

template <int BN, bool kBF16>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const __grid_constant__ WgradParams p) {
    pdl_launch_dependents();
    constexpr int kRowB = (BN >= 64 ? 64 : BN) * 2;                           // bytes of one K row of a T atom
    constexpr int kAtomsT = BN >= 64 ? BN / 64 : 1;
    constexpr int kTg = kWgMaxCols / BN;                                       // most taps of one unit
    constexpr int kMaxStages = 8;

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_raw_u32 = smem_u32(smem_raw);
    const uint32_t smem_base = (smem_raw_u32 + 1023u) & ~1023u;
    const uint32_t xb_base = smem_base + p.stages * p.stage_bytes;
    const uint32_t bar_base = xb_base + xbuf_bytes<16>();
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kMaxStages + s); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmS);
        tma_prefetch_desc(&p.tmT);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);  // one arrive per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    const int units_per_split = p.m_tiles * p.n_tiles * p.ngroups;
    const int total_units = units_per_split * p.splits;
    auto decode = [&](int u, int* g, int* nt, int* mt, long long* c0, long long* c1) {
        const int s = u / units_per_split;   // the K split is the slowest index: CTAs running together share pixels (L2)
        const int r = u % units_per_split;
        *g = r % p.ngroups;
        *nt = (r / p.ngroups) % p.n_tiles;
        *mt = r / (p.ngroups * p.n_tiles);
        *c0 = p.chunks * s / p.splits;
        *c1 = p.chunks * (s + 1) / p.splits;
    };

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
                int g, nt, mt;
                long long c0, c1;
                decode(u, &g, &nt, &mt, &c0, &c1);
                const int t0 = g * p.tg;
                const int nt_g = min(p.tg, p.ntaps - t0);
                for (long long c = c0; c < c1; ++c) {
                    const int tx = (int)(c % p.tiles_x);
                    const int ty = (int)((c / p.tiles_x) % p.tiles_y);
                    const int tn = (int)(c / ((long long)p.tiles_x * p.tiles_y));
                    const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = tn * p.bn;
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    const uint32_t base = smem_base + stage * p.stage_bytes;
                    mbar_arrive_expect_tx(full_bar(stage), p.a_bytes + nt_g * p.tap_bytes);
                    tma_load_4d(base, &p.tmS, full_bar(stage), mt * 128, x0, y0, n0);
                    tma_load_4d(base + (p.a_bytes >> 1), &p.tmS, full_bar(stage), mt * 128 + 64, x0, y0, n0);
                    for (int t = 0; t < nt_g; ++t) {
                        const uint32_t tb = base + p.a_bytes + t * p.tap_bytes;
#pragma unroll
                        for (int a = 0; a < kAtomsT; ++a)
                            tma_load_4d(tb + a * (p.tap_bytes / kAtomsT), &p.tmT, full_bar(stage), nt * BN + a * 64,
                                        x0 * p.sx + p.dx[t0 + t], y0 * p.sy + p.dy[t0 + t], n0);
                    }
                    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else if (warp >= 4) {
        // =============================== consumer warpgroup: MMA + epilogue ===============================
        // A = the 128 channels of S (two 64-channel MN-major atoms, one per m64 half), B = the BN channels of one tap's T
        // tile; every tap owns BN accumulator columns, so the shared operand is loaded ONCE per chunk for the whole group.
        const int q = warp - 4;
        const int row = q * 32 + lane;  // after the transpose: the channel of the shared operand inside the m tile
        float* const xb = reinterpret_cast<float*>(smem_raw + (xb_base - smem_raw_u32));
        const long long Mp = (long long)p.m_tiles * 128, Np = (long long)p.n_tiles * BN;
        const int ksteps = p.P >> 4;
        const uint32_t a_lbo = p.a_bytes >> 1;              // second 64-channel atom of S
        const uint32_t t_lbo = p.tap_bytes / kAtomsT;       // next 64-channel atom of a T tile
        float acc[2][kWgMaxCols / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
            int g, nt, mt;
            long long c0, c1;
            decode(u, &g, &nt, &mt, &c0, &c1);
            const int s = u / units_per_split;
            const int t0 = g * p.tg;
            const int nt_g = min(p.tg, p.ntaps - t0);
            int prev = -1;
            for (long long c = c0; c < c1; ++c) {
                mbar_wait(full_bar(stage), phase);
                const uint32_t base = smem_base + stage * p.stage_bytes;
                wg_fence();
                for (int k = 0; k < ksteps; ++k) {   // 16 pixels further along K: 16 rows of the operand tiles
                    const uint32_t on = (c > c0 || k > 0) ? 1u : 0u;
                    const uint64_t a0 = wg_desc(base + k * 16 * 128, a_lbo, 1024, 128);
                    const uint64_t a1 = wg_desc(base + a_lbo + k * 16 * 128, a_lbo, 1024, 128);
#pragma unroll
                    for (int t = 0; t < kTg; ++t) {
                        if (t < nt_g) {
                            const uint64_t bd = wg_desc(base + p.a_bytes + t * p.tap_bytes + k * 16 * kRowB, t_lbo, 8 * kRowB, kRowB);
                            wgmma_m64k16<BN, kBF16>(acc[0] + t * (BN / 2), a0, bd, on, 1);
                            wgmma_m64k16<BN, kBF16>(acc[1] + t * (BN / 2), a1, bd, on, 1);
                        }
                    }
                }
                wg_commit();
                wg_wait<1>();
                if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
                prev = stage;
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
            wg_wait<0>();
            wg_fence_regs<kWgMaxCols / 2>(acc[0]);
            wg_fence_regs<kWgMaxCols / 2>(acc[1]);
            if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
            // fp32 partial tile -> workspace ws[split][tap][m][n]
#pragma unroll
            for (int t = 0; t < kTg; ++t) {
                if (t < nt_g) {
                    float* dst = p.ws + (((long long)s * p.ntaps + t0 + t) * Mp + (long long)mt * 128 + row) * Np + (long long)nt * BN;
#pragma unroll
                    for (int cc = 0; cc < BN; cc += 16) {
                        uint32_t v[16];
                        acc_to_rows<16>(acc[0], acc[1], t * BN + cc, xb, 1, v);
                        float4* o = reinterpret_cast<float4*>(dst + cc);
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            o[j] = make_float4(__uint_as_float(v[4 * j]), __uint_as_float(v[4 * j + 1]), __uint_as_float(v[4 * j + 2]),
                                               __uint_as_float(v[4 * j + 3]));
                    }
                }
            }
        }
    }
}

// Second pass of the split-K: out[m][n][tap] (the PyTorch parameter layout: (Cout,Cin,kh,kw) for a conv with m = co,
// n = ci; (Cin,Cout,kh,kw) for a transposed conv with m = ci, n = co) = [out +] sum over splits, in a fixed order.
struct WgradReduceParams {
    const float* ws;
    float* out;
    int splits, ntaps, Cm, Cn;
    long long Mp, Np;
    int accumulate;
    int transpose;   // 1: the parameter layout is [n][m][tap] (a conv whose operand roles were swapped: m = ci, n = co)
    // K-folded first layers: a "tap" is a filter ROW r and column n = s*fold_cp + c is horizontal tap s, input channel c
    // (fold_kw = 0: off); the parameter element is out[m][c][r][s]
    int fold_kw, fold_cp, fold_cin;
};

// grid = (ceil(Cn / 64), Cm), block = 256: a block sums the splits of one row m, 64 columns n, all taps — reading the
// workspace in 256-byte runs along n — and transposes through shared memory so that the (n, tap) values leave as one
// contiguous run of 64 * ntaps floats of the parameter tensor.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const WgradReduceParams p) {
    extern __shared__ float red_t[];           // [64][ntaps + 1]
    const int m = blockIdx.y, n0 = blockIdx.x * 64;
    const int pitch = p.ntaps + 1;
    const int items = p.ntaps * 64;
    for (int i = threadIdx.x; i < items; i += 256) {
        const int t = i >> 6, n = i & 63;
        float s = 0.0f;
        if (n0 + n < p.Cn) {
            const float* src = p.ws + ((long long)t * p.Mp + m) * p.Np + n0 + n;
            const long long split_stride = (long long)p.ntaps * p.Mp * p.Np;
            // four loads in flight per thread (the split loop is otherwise one dependent-latency chain per item)
            float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
            int k = 0;
            for (; k + 3 < p.splits; k += 4) {
                s0 += __ldg(src + (k + 0) * split_stride); s1 += __ldg(src + (k + 1) * split_stride);
                s2 += __ldg(src + (k + 2) * split_stride); s3 += __ldg(src + (k + 3) * split_stride);
            }
            for (; k < p.splits; ++k) s0 += __ldg(src + k * split_stride);
            s = (s0 + s1) + (s2 + s3);
        }
        red_t[n * pitch + t] = s;
    }
    __syncthreads();
    const int ncols = min(64, p.Cn - n0);
    if (p.fold_kw > 0) {
        for (int i = threadIdx.x; i < ncols * p.ntaps; i += 256) {
            const int n = i / p.ntaps, r = i - n * p.ntaps;
            const int sx = (n0 + n) / p.fold_cp, c = (n0 + n) - sx * p.fold_cp;
            if (sx >= p.fold_kw || c >= p.fold_cin) continue;
            const float v = red_t[n * pitch + r];
            float* o = p.out + (((long long)m * p.fold_cin + c) * p.ntaps + r) * p.fold_kw + sx;
            *o = p.accumulate ? *o + v : v;
        }
        return;
    }
    for (int i = threadIdx.x; i < ncols * p.ntaps; i += 256) {
        const int n = i / p.ntaps, t = i - n * p.ntaps;
        const float v = red_t[n * pitch + t];
        float* o = p.transpose ? p.out + ((long long)(n0 + n) * p.Cm + m) * p.ntaps + t
                               : p.out + ((long long)m * p.Cn + n0) * p.ntaps + i;
        *o = p.accumulate ? *o + v : v;
    }
}

}  // namespace w2l
