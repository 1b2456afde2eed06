// conv_igemm.cuh — the generic fused conv-block kernel of the Wav2Lip hot path for sm_90a, plus the PTX
// wrappers and the epilogue helpers shared by the specialised kernels (conv_patch.cuh, convt_fused.cuh).
//
// One persistent, warp-specialised kernel computes, for every block kind of
// /root/reference/models/conv.py (Conv2d :5-19, nonorm_Conv2d :21-31 and, phase by phase,
// Conv2dTranspose :33-44):
//
//     y = act( scale[c] * conv(x, w)[., c] + shift[c]  (+ residual) )
//
// as an implicit GEMM on the Hopper tensor cores (wgmma):
//     M = output pixels (a 128-row tile = a bw x bh x bn box of the NHWC output grid),
//     N = output channels (BN per tile), K = filter taps x input channels (BK per step).
//
//   warp 0  : TMA producer. For each K step one 4-D tiled TMA load per M tile brings the input box of the
//             current filter tap (start coordinate = tile origin * stride + tap offset; out-of-bounds
//             coordinates are zero-filled by the TMA unit, which IS the conv zero padding) and one
//             3-D TMA load brings the [BN x BK] weight slice of that tap. Both land K-major with the
//             hardware 128/64/32-byte swizzle that the wgmma shared-memory descriptors expect.
//   warps 4-11: two consumer warpgroups.  MT = 2: one per M tile of a unit (two tiles that share every weight
//             slab, half the weight traffic per FLOP).  MT = 1 (ping-pong): they take alternate tiles of the CTA and
//             their K loops alternate (a pair of named barriers hands the ring over), so one warpgroup's epilogue
//             runs while the other issues MMAs.  The producer warpgroup gives registers to the consumers
//             (setmaxnreg).  A warpgroup issues wgmma.mma_async m64nBNk16 for both 64-row halves of its tile,
//             accumulating in registers (fp32), keeps one K step in flight and releases each shared-memory
//             stage as soon as the step that read it has retired.  Then the epilogue: the folded BatchNorm
//             scale/shift (conv bias folded in), the residual add (conv.py:16-18: after BN, before ReLU), ReLU /
//             LeakyReLU(0.01), and NHWC 16-bit straight into the channel slice of the consumer's buffer (so
//             torch.cat of wav2lip.py:108 never exists).
//             Staged mode (tma_epi): works on the wgmma accumulator fragment itself.  The residual arrives by TMA
//             in the warpgroup's swizzled staging boxes (the full tile width, one box per 64 channels), every
//             column pair is combined in place at its swizzled address, and the boxes leave by TMA tensor stores
//             (which also clip ragged tiles); the next tile's residual is requested as soon as the stores have
//             read the boxes.  Direct mode (fp32 outputs, split-operand mode, fused generator head
//             wav2lip.py:84-85): a shared-memory transpose (wgmma.cuh: acc_to_rows) makes thread = GEMM row =
//             output pixel, then per-thread global accesses.
//   Channel-major form (kCM, BN = 128, BK = 64): the operand roles swap.  The 128 output channels are M (warpgroup g takes
//             weight rows 64g.. as the K-major A operand), a box of kCmPixels = 256 output pixels is N (the activation box,
//             the K-major B operand of m64n256k16, shared by both warpgroups), so a tile reads 80 instead of 96 bytes of
//             shared memory per tensor clock.  Both warpgroups consume every stage and run their epilogues together
//             (chmajor_epilogue: residual by ldmatrix.trans from the staging box, stmatrix.trans, one TMA store each).
//
// Everything a launch needs is in ConvParams (a __grid_constant__), built once per plan on the host.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace w2l {

constexpr int kTileM = 128;
constexpr int kMaxTaps = 49;              // filter taps of one launch
constexpr int kMaxSteps = 3 * kMaxTaps;   // K-loop entries: x3 in the split-operand (fp32-faithful) precision mode
constexpr int kSmemExtra = 2048;         // 1024 alignment slack + barriers
constexpr int kSmemMax = 227 * 1024;     // dynamic shared memory limit per CTA on sm_90

enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_LRELU = 2 };

// What the epilogue needs, shared by every conv kernel variant.
struct EpiParams {
    int Wout, Hout, N;      // logical output grid of this launch (rows outside are masked)
    int act;
    int out_f32;
    void* out;              // element (n,y,x,c) at out + n*out_sn + y*out_sy + x*out_sx + c  (elements)
    long long out_sn, out_sy, out_sx;
    const void* res;        // nullptr = no residual; same addressing
    long long res_sn, res_sy, res_sx;
    const float* scale;     // [n_tiles*BN]
    const float* shift;
    // fused generator head (kHead kernels only): out = sigmoid(W[3x32] relu(y) + b), fp32 NCHW/5-D
    const float* head_w;
    const float* head_b;
    // split-operand (fp32-faithful) mode: every value is stored as hi + lo (two fp16 planes, lo_off channels apart)
    int x2;
    int out_lo_off, res_lo_off;
    float* head_out;
    unsigned char* head_out_u8;  // if set: (N,H,W,3) uint8 = trunc(sigmoid * 255.f), inference.py:265,269
    int head_B, head_T;     // n = t*head_B + b ; T=1,B=N for the 4-D call
};

struct alignas(64) ConvParams {
    CUtensorMap tmA;  // activations, dims (C, W, H, N), box (BK, bw*sx, bh*sy, bn), elem strides (1,sx,sy,1)
    CUtensorMap tmB;  // weights, dims (Cin_pad, Cout_pad, taps), box (BK, BN, 1)
    CUtensorMap tmO;  // output slice (Cout, Wl, Hl, N) with the launch's pixel strides, box (EW, bw, bh, bn)   [tma_epi]
    CUtensorMap tmR;  // residual, same geometry                                                              [tma_epi]
    int tma_epi;             // 1: epilogue stages through swizzled smem and uses TMA for the residual and the output
    unsigned epi_box_bytes;  // bytes of one epilogue box (bw*bh*bn rows x EW channels)
    // M tiling of the logical output grid
    int tiles_x, tiles_y, tiles_n, n_tiles;
    int bw, bh, bn;
    int sx, sy;
    // K loop
    int ntaps, kc_per_tap;
    unsigned stage_tx_bytes;  // bytes both TMA loads of one stage deliver
    EpiParams ep;
    // K-loop entries ("steps"): one per filter tap, or three per tap in the split-operand mode
    // (x_hi*w_hi, x_lo*w_hi, x_hi*w_lo).  a_lo selects the lo plane of the activations, b_slab the weight slab.
    int a_lo_off;                    // channel offset of the lo plane inside a pixel (0 in the 16-bit modes)
    signed char dx[kMaxSteps];
    signed char dy[kMaxSteps];
    unsigned char a_lo[kMaxSteps];
    unsigned char b_slab[kMaxSteps];
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "W2L_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra W2L_DONE_%=;\n\t"
        "bra W2L_WAIT_%=;\n\t"
        "W2L_DONE_%=:\n\t"
        "}" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* desc, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* desc, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// Programmatic dependent launch: the next kernel in the stream may start its prologue (barrier init, descriptor
// prefetch) while this one drains; it touches global memory only after pdl_wait().
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// K-major operand tile in shared memory: rows of BK*2 bytes, 8-row groups, hardware swizzle = row bytes.
template <int BK>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr) {
    return wg_desc(saddr, 16, 8 * BK * 2, BK * 2);
}

// One K step of BK channels for a warpgroup's 128-row tile: a = first row of the A tile, b = the [BN x BK] B slab,
// sbo_a = bytes between the A tile's 8-row groups; acc = 0 starts a new accumulation.
template <int BN, int BK, bool kBF16>
__device__ __forceinline__ void wg_mma_tile(float (&acc)[2][BN / 2], uint32_t a, uint32_t sbo_a, uint32_t b, bool accumulate) {
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {  // 16 elements further along K = 32 bytes inside the swizzle atom
        const uint64_t bd = make_kmajor_desc<BK>(b + 32u * k);
        const uint32_t on = (accumulate || k > 0) ? 1u : 0u;
        wgmma_m64k16<BN, kBF16>(acc[0], wg_desc(a + 32u * k, 16, sbo_a, BK * 2), bd, on, 0);
        wgmma_m64k16<BN, kBF16>(acc[1], wg_desc(a + 8u * sbo_a + 32u * k, 16, sbo_a, BK * 2), bd, on, 0);
    }
}

// MT = number of 128-row M tiles a CTA works on at once (sharing each weight slab).  Either way the CTA has two
// consumer warpgroups: MT = 2 gives each one of the unit's two tiles, MT = 1 gives them alternate tiles (ping-pong).
// Shared memory: the K-step ring, then one region per consumer warpgroup that holds either the staging boxes of the
// staged epilogue (the full tile width, BN / kEW boxes) or the transpose buffer of the direct one (a launch uses one
// epilogue form), then the barriers.
// Channel-major form (CM): the tile is BN = 128 channels x kCmPixels pixels, each consumer warpgroup owns one 64-channel half
// and its staging box (64 channels x kCmPixels pixels); the ring stage holds the pixel box and the weight slab.
constexpr int kCmPixels = 256;
template <int BN, int BK, int MT = 1, bool kCM = false>
struct ConvCfg {
    static constexpr int kRowsA = kCM ? kCmPixels : kTileM;       // pixel rows of one A (activation) tile
    static constexpr int kATile = kRowsA * BK * 2;
    static constexpr int kABytes = MT * kATile;
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kEW = BN < 64 ? BN : 64;                 // channels per epilogue box (one TMA box)
    static constexpr int kCW = BN < 32 ? BN : 32;                 // accumulator columns per transpose chunk (direct epilogue)
    static constexpr int kPasses = kCM ? 1 : BN / kEW;            // epilogue boxes per warpgroup and tile
    static constexpr int kBoxBytes = kRowsA * kEW * 2;            // one staging box: kRowsA rows x kEW 16-bit channels
    // CM always stages its epilogue (no transpose buffer)
    static constexpr int kGrpRaw = (kCM || kPasses * kBoxBytes > xbuf_bytes<kCW>()) ? kPasses * kBoxBytes : xbuf_bytes<kCW>();
    static constexpr int kGrpBytes = (kGrpRaw + 1023) / 1024 * 1024;  // epilogue region of one consumer warpgroup
    static constexpr int kStagesRaw = (kSmemMax - kSmemExtra - 2 * kGrpBytes) / kStageBytes;
    static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
    static constexpr int kRingBytes = (kStages * kStageBytes + 1023) / 1024 * 1024;
    static constexpr int kSmemBytes = kRingBytes + 2 * kGrpBytes + kSmemExtra;
    static constexpr int kThreads = 384;  // the producer warpgroup + two consumer warpgroups
    static_assert(BN <= 128, "a warpgroup holds at most 128 fp32 accumulator columns per row");
    static_assert(!kCM || (BN == 128 && BK == 64 && MT == 1), "channel-major form: 128 channels, 128-byte K rows, one tile");
    static_assert(kBoxBytes % 1024 == 0, "staging boxes must keep the 1024-byte swizzle alignment");
    static_assert(kStages >= 2, "need a pipeline");
    static_assert(kSmemBytes <= kSmemMax, "shared-memory carve-up exceeds the per-CTA limit");
};

// Sticky range flag of the fp16 modes: set by any epilogue that rounds a value beyond the fp16 range (|v| > 65504 ->
// inf, or a NaN) when it stores an activation.  One instance per device (module-scope __device__ variable); read and
// cleared through w2l_f16_overflow().  bf16 has fp32's exponent range and never sets it.
__device__ int g_f16_overflow = 0;

// `live` = the value belongs to a real output pixel.  (GEMM rows beyond a partial tile box are computed from stale shared
// memory — any bit pattern, NaN included — and never stored; they must not raise the flag.)  pack2_live takes it per
// half: bit 15 = a is live, bit 31 = b is live.
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2_live(float a, float b, uint32_t live_bits) {
    if constexpr (kBF16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    } else {
        __half2 h = __floats2half2_rn(a, b);
        const uint32_t u = *reinterpret_cast<uint32_t*>(&h);
        // exponent field all ones (inf / NaN) in either half: adding 0x0400 to the magnitude bits carries into bit 15
        if (((u & 0x7FFF7FFFu) + 0x04000400u) & live_bits) g_f16_overflow = 1;
        return u;
    }
}
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2(float a, float b, bool live = true) {
    return pack2_live<kBF16>(a, b, live ? 0x80008000u : 0u);
}
template <bool kBF16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
    if constexpr (kBF16) {
        return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
    } else {
        return __half22float2(*reinterpret_cast<__half2*>(&u));
    }
}

// One accumulator tile (this thread's row = one output pixel, BN columns) -> epilogue math -> global memory.
template <int BN, bool kBF16, bool kHead>
__device__ __forceinline__ void epilogue_tile(const EpiParams& e, const float (&acc)[2][BN / 2], float* xb, uint32_t bar_id,
                                              bool valid, int n, int y, int x, int nt) {
    constexpr int CH = (BN >= 32) ? 32 : 16;  // columns per transpose chunk
    const long long o_off = (long long)n * e.out_sn + (long long)y * e.out_sy + (long long)x * e.out_sx;
    const long long r_off = (long long)n * e.res_sn + (long long)y * e.res_sy + (long long)x * e.res_sx;
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += CH) {
        uint32_t v[CH];
        acc_to_rows<CH>(acc[0], acc[1], c0, xb, bar_id, v);
        if (valid) {
            const int cg = nt * BN + c0;  // first output channel of this batch
            float f[CH];
#pragma unroll
            for (int j = 0; j < CH; j += 4) {
                const float4 sc = __ldg(reinterpret_cast<const float4*>(e.scale + cg + j));
                const float4 sh = __ldg(reinterpret_cast<const float4*>(e.shift + cg + j));
                f[j + 0] = fmaf(__uint_as_float(v[j + 0]), sc.x, sh.x);
                f[j + 1] = fmaf(__uint_as_float(v[j + 1]), sc.y, sh.y);
                f[j + 2] = fmaf(__uint_as_float(v[j + 2]), sc.z, sh.z);
                f[j + 3] = fmaf(__uint_as_float(v[j + 3]), sc.w, sh.w);
            }
            if (e.res != nullptr) {
                const uint4* rp = reinterpret_cast<const uint4*>(
                    reinterpret_cast<const uint16_t*>(e.res) + r_off + cg);
#pragma unroll
                for (int j = 0; j < CH / 8; ++j) {
                    const uint4 r = __ldg(rp + j);
                    const float2 a = unpack2<kBF16>(r.x), b = unpack2<kBF16>(r.y);
                    const float2 c = unpack2<kBF16>(r.z), d = unpack2<kBF16>(r.w);
                    f[8 * j + 0] += a.x; f[8 * j + 1] += a.y; f[8 * j + 2] += b.x; f[8 * j + 3] += b.y;
                    f[8 * j + 4] += c.x; f[8 * j + 5] += c.y; f[8 * j + 6] += d.x; f[8 * j + 7] += d.y;
                }
                if (e.x2) {  // lo plane of the residual
#pragma unroll
                    for (int j = 0; j < CH / 8; ++j) {
                        const uint4 r = __ldg(rp + (e.res_lo_off >> 3) + j);
                        const float2 a = unpack2<kBF16>(r.x), b = unpack2<kBF16>(r.y);
                        const float2 c = unpack2<kBF16>(r.z), d = unpack2<kBF16>(r.w);
                        f[8 * j + 0] += a.x; f[8 * j + 1] += a.y; f[8 * j + 2] += b.x; f[8 * j + 3] += b.y;
                        f[8 * j + 4] += c.x; f[8 * j + 5] += c.y; f[8 * j + 6] += d.x; f[8 * j + 7] += d.y;
                    }
                }
            }
            if (e.act == ACT_RELU) {
#pragma unroll
                for (int j = 0; j < CH; ++j) f[j] = fmaxf(f[j], 0.0f);
            } else if (e.act == ACT_LRELU) {
#pragma unroll
                for (int j = 0; j < CH; ++j) f[j] = f[j] > 0.0f ? f[j] : 0.01f * f[j];
            }
            if constexpr (kHead) {
                // wav2lip.py:84-85: Conv2d(32,3,1) + Sigmoid on the fp32 block output still in registers
                const int hb = n % e.head_B, ht = n / e.head_B;
                const long long plane = (long long)e.Hout * e.Wout;
#pragma unroll
                for (int oc = 0; oc < 3; ++oc) {
                    float s = __ldg(e.head_b + oc);
#pragma unroll
                    for (int j = 0; j < 32; ++j) s = fmaf(f[j], __ldg(e.head_w + oc * 32 + j), s);
                    s = 1.0f / (1.0f + __expf(-s));
                    if (e.head_out_u8 != nullptr)
                        e.head_out_u8[(((long long)n * e.Hout + y) * e.Wout + x) * 3 + oc] = (unsigned char)__fmul_rn(s, 255.0f);
                    else
                        e.head_out[(((long long)hb * 3 + oc) * e.head_T + ht) * plane + (long long)y * e.Wout + x] = s;
                }
            } else if (e.out_f32) {
                float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + o_off + cg);
#pragma unroll
                for (int j = 0; j < CH / 4; ++j) op[j] = make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
            } else {
                uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.out) + o_off + cg);
#pragma unroll
                for (int j = 0; j < CH / 8; ++j) {
                    uint4 o;
                    o.x = pack2<kBF16>(f[8 * j + 0], f[8 * j + 1]);
                    o.y = pack2<kBF16>(f[8 * j + 2], f[8 * j + 3]);
                    o.z = pack2<kBF16>(f[8 * j + 4], f[8 * j + 5]);
                    o.w = pack2<kBF16>(f[8 * j + 6], f[8 * j + 7]);
                    op[j] = o;
                    if (e.x2) {  // lo = fp16(v - fp16(v)): together the two planes carry ~22 significant bits
                        const float2 h0 = unpack2<kBF16>(o.x), h1 = unpack2<kBF16>(o.y);
                        const float2 h2 = unpack2<kBF16>(o.z), h3 = unpack2<kBF16>(o.w);
                        uint4 l;
                        l.x = pack2<kBF16>(f[8 * j + 0] - h0.x, f[8 * j + 1] - h0.y);
                        l.y = pack2<kBF16>(f[8 * j + 2] - h1.x, f[8 * j + 3] - h1.y);
                        l.z = pack2<kBF16>(f[8 * j + 4] - h2.x, f[8 * j + 5] - h2.y);
                        l.w = pack2<kBF16>(f[8 * j + 6] - h3.x, f[8 * j + 7] - h3.y);
                        op[(e.out_lo_off >> 3) + j] = l;
                    }
                }
            }
        }
    }
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Epilogue of a channel-major tile (conv_patch_kernel<64, 64> and conv_igemm_kernel<128, 64, ., ., 1, true>): one
// warpgroup's m64n256 accumulator, rows = 64 output channels, columns = 256 output pixels.  Fragment: warp q holds channels
// 16q + lane/4 (acc[4j + 0..1], scale / shift sc0 / sh0) and that + 8 (acc[4j + 2..3], sc1 / sh1) at pixels
// 8j + 2(lane%4) + {0,1}.  The staging tile `stg` is pixel-major: pixel p is row p of 128 bytes (64 16-bit channels,
// 128-byte swizzle), exactly the box the TMA store `tmO` writes at (c0, c1, c2, c3).
//   res       : 0 = no residual, else the address of residual pixel 0 in a pixel-major 128-byte-row tile whose pixel rows of
//               8 are res_pitch rows apart (the staging tile itself when the residual was TMA-loaded into it, pitch 8);
//               read by ldmatrix.trans straight into the fragment layout
//   after_res : called by every thread once its residual reads are done (the patch kernel releases its ring slot there)
//   live(j)   : pack2_live bits of the pixel pair of column chunk j (only pixels inside the image may raise the fp16 flag)
// Every warp reads and writes only its own 32-byte channel stripe of the tiles; the named barrier bar_id orders the
// warpgroup's stmatrix writes after the previous TMA store has read the staging tile, and the store after the writes.
template <bool kBF16, typename AfterRes, typename Live>
__device__ __forceinline__ void chmajor_epilogue(float (&acc)[128], float sc0, float sh0, float sc1, float sh1, int act,
                                                 uint32_t res, int res_pitch, AfterRes&& after_res, Live&& live, uint32_t stg,
                                                 uint32_t bar_id, bool leader, const CUtensorMap* tmO, int c0, int c1, int c2,
                                                 int c3) {
    constexpr uint32_t kRowB = 128;
    const int lane = threadIdx.x & 31, q = (threadIdx.x >> 5) & 3;
    // ldmatrix / stmatrix .x4: lanes 8m .. 8m+7 address the 8 pixels of matrix m = (pixels 8(2i + m/2) .., 16-byte channel
    // chunk 2q + m%2), which land in / come from the fragment registers of (column chunk 2i + m/2, channel half m%2)
    const int lm_row = lane >> 4, lm_px = lane & 7;
    const uint32_t lm_chunk = 16u * (2 * q + ((lane >> 3) & 1));
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float* a = acc + 8 * i + 4 * h;
            a[0] = fmaf(a[0], sc0, sh0); a[1] = fmaf(a[1], sc0, sh0);
            a[2] = fmaf(a[2], sc1, sh1); a[3] = fmaf(a[3], sc1, sh1);
        }
        if (res != 0) {
            uint32_t ad = res + static_cast<uint32_t>((2 * i + lm_row) * res_pitch + lm_px) * kRowB + lm_chunk;
            ad ^= ((ad >> 7) & 7u) << 4;
            uint32_t rv[4];
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                         : "=r"(rv[0]), "=r"(rv[1]), "=r"(rv[2]), "=r"(rv[3]) : "r"(ad));
#pragma unroll
            for (int m = 0; m < 4; ++m) {
                const float2 v = unpack2<kBF16>(rv[m]);
                acc[8 * i + 2 * m] += v.x;
                acc[8 * i + 2 * m + 1] += v.y;
            }
        }
    }
    after_res();
    if (act == ACT_RELU) {
#pragma unroll
        for (int j = 0; j < 128; ++j) acc[j] = fmaxf(acc[j], 0.0f);
    } else if (act == ACT_LRELU) {
#pragma unroll
        for (int j = 0; j < 128; ++j) acc[j] = acc[j] > 0.0f ? acc[j] : 0.01f * acc[j];
    }
    if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // previous store has read the staging tile
    named_bar_sync(bar_id, 128);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        uint32_t ad = stg + static_cast<uint32_t>((2 * i + lm_row) * 8 + lm_px) * kRowB + lm_chunk;
        ad ^= ((ad >> 7) & 7u) << 4;
        const uint32_t l0 = live(2 * i), l1 = live(2 * i + 1);
        const uint32_t o0 = pack2_live<kBF16>(acc[8 * i + 0], acc[8 * i + 1], l0);
        const uint32_t o1 = pack2_live<kBF16>(acc[8 * i + 2], acc[8 * i + 3], l0);
        const uint32_t o2 = pack2_live<kBF16>(acc[8 * i + 4], acc[8 * i + 5], l1);
        const uint32_t o3 = pack2_live<kBF16>(acc[8 * i + 6], acc[8 * i + 7], l1);
        asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1,%2,%3,%4};"
                     ::"r"(ad), "r"(o0), "r"(o1), "r"(o2), "r"(o3) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
    named_bar_sync(bar_id, 128);
    if (leader) {
        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                     ::"l"(reinterpret_cast<uint64_t>(tmO)), "r"(stg), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------------
// Register split between the warpgroups (all four warps of a warpgroup execute it): the producer needs few registers, the
// consumers hold a 128 x BN fp32 accumulator tile each.  __launch_bounds__(384, 1) gives every thread 168; 128 x 40 +
// 256 x 232 = 64 512 of the SM's 65 536.
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

template <int BN, int BK, bool kBF16, bool kHead, int MT = 1, bool kCM = false>
__global__ void __launch_bounds__(ConvCfg<BN, BK, MT, kCM>::kThreads, 1) conv_igemm_kernel(const __grid_constant__ ConvParams p) {
    pdl_launch_dependents();
    using Cfg = ConvCfg<BN, BK, MT, kCM>;
    constexpr int kStages = Cfg::kStages;
    static_assert(!kHead || BN == 32, "fused head expects the 32-channel output block");
    static_assert(MT == 1 || MT == 2, "one or two M tiles per unit");
    static_assert(!kCM || !kHead, "the channel-major form stages its epilogue");

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_raw_u32 = smem_u32(smem_raw);
    const uint32_t smem_base = (smem_raw_u32 + 1023u) & ~1023u;  // swizzle atoms need 1024-B alignment
    const uint32_t grp_base = smem_base + Cfg::kRingBytes;       // the two consumer warpgroups' epilogue regions
    const uint32_t bar_base = grp_base + 2 * Cfg::kGrpBytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
    auto res_bar = [&](int g) { return bar_base + 8u * (2 * kStages + g); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        if (p.tma_epi) {
            tma_prefetch_desc(&p.tmO);
            tma_prefetch_desc(&p.tmR);
        }
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), kCM ? 8 : 4 * MT);  // one arrive per warp of the warpgroup(s) that consume the step
        }
        for (int g = 0; g < 2; ++g) mbar_init(res_bar(g), 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlaps the previous kernel's tail; global memory is touched only below

    const int m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
    const int m_units = (m_tiles + MT - 1) / MT;  // a unit = MT consecutive M tiles x one N tile (a tile index past the
    const int total_tiles = m_units * p.n_tiles;  // end decodes to n >= N: its loads are zero-filled, its rows masked)
    const int k_steps = p.ntaps * p.kc_per_tap;

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();
        // =============================== TMA producer: K steps in tile order into the one ring ===============================
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int nt = tile % p.n_tiles;
                const int mu = tile / p.n_tiles;
                int x_in0[MT], y_in0[MT], n0[MT];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    const int m = mu * MT + mt;
                    const int tx = m % p.tiles_x;
                    const int ty = (m / p.tiles_x) % p.tiles_y;
                    const int tn = m / (p.tiles_x * p.tiles_y);
                    x_in0[mt] = tx * p.bw * p.sx;
                    y_in0[mt] = ty * p.bh * p.sy;
                    n0[mt] = tn * p.bn;
                }
                for (int t = 0; t < p.ntaps; ++t) {
                    for (int kc = 0; kc < p.kc_per_tap; ++kc) {
                        mbar_wait(empty_bar(stage), phase ^ 1u);
                        const uint32_t a_dst = smem_base + stage * Cfg::kStageBytes;
                        const uint32_t b_dst = a_dst + Cfg::kABytes;
                        mbar_arrive_expect_tx(full_bar(stage), p.stage_tx_bytes);
#pragma unroll
                        for (int mt = 0; mt < MT; ++mt)
                            tma_load_4d(a_dst + mt * Cfg::kATile, &p.tmA, full_bar(stage), kc * BK + (p.a_lo[t] ? p.a_lo_off : 0),
                                        x_in0[mt] + p.dx[t], y_in0[mt] + p.dy[t], n0[mt]);
                        tma_load_3d(b_dst, &p.tmB, full_bar(stage), kc * BK, nt * BN, p.b_slab[t]);
                        if (++stage == kStages) { stage = 0; phase ^= 1u; }
                    }
                }
            }
        }
    } else if constexpr (kCM) {
        setmaxnreg_inc<kConsumerRegs>();
        // ===== channel-major consumers: both warpgroups work on every tile of the CTA.  Warpgroup g computes
        // D[64 channels x 256 pixels] = W[64 x K] * box[K x 256]: its 64-row half of the weight slab is the K-major A
        // operand, the pixel box (rows = pixels, 8-row groups 1024 B apart) the K-major B operand of m64n256k16.  Each warp
        // releases a ring stage once the step that read it has retired (8 arrivals per stage). =====
        const int g = (warp - 4) >> 2;
        const int q = (warp - 4) & 3;
        const uint32_t bar_id = 1 + g;
        const bool leader = (q == 0 && lane == 0);
        const uint32_t stg = grp_base + g * Cfg::kGrpBytes;  // this warpgroup's staging box (64 channels x 256 pixels)
        const bool has_res = p.ep.res != nullptr;
        const int rows_valid = p.bw * p.bh * p.bn;
        const int ch = 64 * g + 16 * q + (lane >> 2);         // fragment channels ch and ch + 8 of the tile
        auto tile_origin = [&](int tile_, int* nt_, int* x0_, int* y0_, int* n0_) {
            *nt_ = tile_ % p.n_tiles;
            const int m_ = tile_ / p.n_tiles;
            *x0_ = (m_ % p.tiles_x) * p.bw;
            *y0_ = ((m_ / p.tiles_x) % p.tiles_y) * p.bh;
            *n0_ = (m_ / (p.tiles_x * p.tiles_y)) * p.bn;
        };
        // leader: request the tile's residual half into the staging box (the previous store must have read it)
        auto fetch_res = [&](int tile_) {
            int nt_, x0_, y0_, n0_;
            tile_origin(tile_, &nt_, &x0_, &y0_, &n0_);
            mbar_arrive_expect_tx(res_bar(g), p.epi_box_bytes);
            tma_load_4d(stg, &p.tmR, res_bar(g), nt_ * BN + 64 * g, x0_, y0_, n0_);
        };
        if (has_res && leader && static_cast<int>(blockIdx.x) < total_tiles) fetch_res(blockIdx.x);
        float acc[128];
        int stage = 0;
        uint32_t phase = 0, rphase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            int prev = -1;
            for (int ks = 0; ks < k_steps; ++ks) {
                mbar_wait(full_bar(stage), phase);
                const uint32_t box = smem_base + stage * Cfg::kStageBytes;
                const uint32_t wts = box + Cfg::kABytes + g * (64 * BK * 2);
                wg_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)  // 16 elements further along K = 32 bytes inside the swizzle atom
                    wgmma_m64k16<256, kBF16>(acc, make_kmajor_desc<BK>(wts + 32u * k), make_kmajor_desc<BK>(box + 32u * k),
                                             (ks | k) != 0 ? 1u : 0u, 0);
                wg_commit();
                wg_wait<1>();
                if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1u; }
            }
            wg_wait<0>();
            wg_fence_regs<128>(acc);
            if (lane == 0) mbar_arrive(empty_bar(prev));

            int nt, x0, y0, n0;
            tile_origin(tile, &nt, &x0, &y0, &n0);
            // fp16: which of this thread's pixels 8j + 2(lane%4) + {0,1} are real output pixels (bit 2j + e); GEMM columns
            // past the box or outside the image are computed from stale or zero-filled rows and never stored
            uint64_t live = ~0ull;
            if constexpr (!kBF16) {
                const int xr = p.ep.Wout - x0, yr = p.ep.Hout - y0, nr = p.ep.N - n0;
                if (rows_valid < kCmPixels || xr < p.bw || yr < p.bh || nr < p.bn) {
                    live = 0;
#pragma unroll 1
                    for (int b = 0; b < 64; ++b) {
                        const int px = 8 * (b >> 1) + 2 * (lane & 3) + (b & 1);
                        const int xx = px % p.bw, yy = (px / p.bw) % p.bh, nn = px / (p.bw * p.bh);
                        if (px < rows_valid && xx < xr && yy < yr && nn < nr) live |= 1ull << b;
                    }
                }
            }
            if (has_res) {
                mbar_wait(res_bar(g), rphase);
                rphase ^= 1u;
            }
            const float* const sc = p.ep.scale + nt * BN + ch;
            const float* const sh = p.ep.shift + nt * BN + ch;
            chmajor_epilogue<kBF16>(
                acc, __ldg(sc), __ldg(sh), __ldg(sc + 8), __ldg(sh + 8), p.ep.act, has_res ? stg : 0u, 8, [] {},
                [&](int j) {
                    return (static_cast<uint32_t>(live >> (2 * j)) & 1u) << 15 | (static_cast<uint32_t>(live >> (2 * j + 1)) & 1u) << 31;
                },
                stg, bar_id, leader, &p.tmO, nt * BN + 64 * g, x0, y0, n0);
            if (has_res && leader && tile + static_cast<int>(gridDim.x) < total_tiles) {
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the store has read the staging box
                fetch_res(tile + gridDim.x);  // lands while both warpgroups run the next tile's MMAs
            }
        }
        if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete before exit
    } else {
        setmaxnreg_inc<kConsumerRegs>();
        // =============================== consumer warpgroups: MMA + epilogue ===============================
        // MT = 2: group g computes M tile g of every unit of the CTA.  MT = 1 (ping-pong): group g takes the CTA's tiles
        // i = g, g + 2, ..., so one group's epilogue runs while the other issues MMAs.  Tile i of the CTA is
        // blockIdx.x + i * gridDim.x; its K steps are the CTA-global ring steps i * k_steps + ks.
        const int g = (warp - 4) >> 2;     // consumer warpgroup
        const int q = (warp - 4) & 3;      // warp of the warpgroup
        const int mt = MT == 2 ? g : 0;    // which of the unit's M tiles this warpgroup computes
        constexpr int kItStride = MT == 2 ? 1 : 2;
        const int it0 = MT == 2 ? 0 : g;
        const int rows_valid = p.bw * p.bh * p.bn;
        const uint32_t bar_id = 1 + g;     // named barrier of this warpgroup (0 is __syncthreads)
        // MT = 1: the two groups' K loops alternate.  Group g waits on named barrier 3 + g before its K loop; the other
        // group arrives there once it has waited for the last full barrier of its own tile.  So every ring step before
        // a group's first one has been loaded when the group starts, and a parity wait can never see a stage two
        // phases behind.
        const uint32_t my_turn = 3 + g, their_turn = 3 + (g ^ 1);
        const uint32_t grp = grp_base + g * Cfg::kGrpBytes;
        float acc[2][BN / 2];
        // the K loop of one tile (ring steps s0 ..); one wgmma group stays in flight, the stage of the step before it is
        // released; hand_off = the other group has a next tile and waits for this K loop
        auto mainloop = [&](int s0, bool hand_off) {
            int stage = s0 % kStages;
            uint32_t phase = static_cast<uint32_t>(s0 / kStages) & 1u;
            int prev = -1;
            for (int ks = 0; ks < k_steps; ++ks) {
                mbar_wait(full_bar(stage), phase);
                const uint32_t a_addr = smem_base + stage * Cfg::kStageBytes + mt * Cfg::kATile;
                wg_fence();
                wg_mma_tile<BN, BK, kBF16>(acc, a_addr, 8 * BK * 2, smem_base + stage * Cfg::kStageBytes + Cfg::kABytes, ks > 0);
                wg_commit();
                wg_wait<1>();
                if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1u; }
            }
            if (hand_off) named_bar_arrive(their_turn, 256);
            wg_wait<0>();
            wg_fence_regs<BN / 2>(acc[0]);
            wg_fence_regs<BN / 2>(acc[1]);
            if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        };
        // every tile of this warpgroup: K loop, then epilogue(tile, next tile of this group exists)
        auto for_each_tile = [&](auto&& epilogue) {
            for (int it = it0;; it += kItStride) {
                const int tile = blockIdx.x + it * static_cast<int>(gridDim.x);
                if (tile >= total_tiles) break;
                if (MT == 1 && it > 0) named_bar_sync(my_turn, 256);
                mainloop(it * k_steps, MT == 1 && tile + static_cast<int>(gridDim.x) < total_tiles);
                epilogue(tile, tile + kItStride * static_cast<int>(gridDim.x) < total_tiles);
            }
        };
        auto tile_origin = [&](int tile_, int* nt_, int* x0_, int* y0_, int* n0_) {
            *nt_ = tile_ % p.n_tiles;
            const int m_ = (tile_ / p.n_tiles) * MT + mt;
            *x0_ = (m_ % p.tiles_x) * p.bw;
            *y0_ = ((m_ / p.tiles_x) % p.tiles_y) * p.bh;
            *n0_ = (m_ / (p.tiles_x * p.tiles_y)) * p.bn;
        };
        if (!kHead && p.tma_epi) {
            // ---- staged epilogue on the accumulator fragment: the residual arrives by TMA in the warpgroup's swizzled
            // staging boxes (one per kEW channels), every value is combined in place and the boxes leave by TMA stores ----
            constexpr int EW = Cfg::kEW;
            constexpr int kPasses = Cfg::kPasses;
            constexpr uint32_t kRowB = EW * 2;
            constexpr uint32_t kSwz = (kRowB == 128) ? 7u : (kRowB == 64) ? 3u : 1u;
            const bool leader = (q == 0 && lane == 0);
            const bool has_res = p.ep.res != nullptr;
            const EpiParams& e = p.ep;
            // leader: request all residual boxes of a tile (the staging boxes must be free)
            auto fetch_res = [&](int tile_) {
                int nt_, x0_, y0_, n0_;
                tile_origin(tile_, &nt_, &x0_, &y0_, &n0_);
                mbar_arrive_expect_tx(res_bar(g), kPasses * p.epi_box_bytes);
#pragma unroll
                for (int ps = 0; ps < kPasses; ++ps)
                    tma_load_4d(grp + ps * Cfg::kBoxBytes, &p.tmR, res_bar(g), nt_ * BN + ps * EW, x0_, y0_, n0_);
            };
            if (has_res && leader) {
                const int first = blockIdx.x + it0 * static_cast<int>(gridDim.x);
                if (first < total_tiles) fetch_res(first);
            }
            uint32_t rphase = 0;
            for_each_tile([&](int tile, bool more) {
                int nt, x0, y0, n0;
                tile_origin(tile, &nt, &x0, &y0, &n0);
                if (has_res) {
                    mbar_wait(res_bar(g), rphase);
                    rphase ^= 1u;
                }
                // fragment of m64nBNk16: this thread holds rows 16q + lane/4 (+8) of each 64-row half and, in every
                // 8-column chunk j, the column pair 8j + 2(lane%4)
                const float* const scale = e.scale + nt * BN;
                const float* const shift = e.shift + nt * BN;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    const float2 sc = __ldg(reinterpret_cast<const float2*>(scale + c));
                    const float2 sh = __ldg(reinterpret_cast<const float2*>(shift + c));
                    const uint32_t box = grp + (8 * j / EW) * Cfg::kBoxBytes;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
#pragma unroll
                        for (int r8 = 0; r8 < 2; ++r8) {
                            const int row = 64 * h + 16 * q + (lane >> 2) + 8 * r8;
                            float f0 = fmaf(acc[h][4 * j + 2 * r8], sc.x, sh.x);
                            float f1 = fmaf(acc[h][4 * j + 2 * r8 + 1], sc.y, sh.y);
                            uint32_t a = box + row * kRowB + (c % EW) * 2;
                            a ^= ((a >> 7) & kSwz) << 4;
                            if (has_res) {
                                uint32_t r;
                                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(a));
                                const float2 rv = unpack2<kBF16>(r);
                                f0 += rv.x;
                                f1 += rv.y;
                            }
                            if (e.act == ACT_RELU) {
                                f0 = fmaxf(f0, 0.0f);
                                f1 = fmaxf(f1, 0.0f);
                            } else if (e.act == ACT_LRELU) {
                                f0 = f0 > 0.0f ? f0 : 0.01f * f0;
                                f1 = f1 > 0.0f ? f1 : 0.01f * f1;
                            }
                            const uint32_t o = pack2<kBF16>(f0, f1, row < rows_valid);
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(o) : "memory");
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
                named_bar_sync(bar_id, 128);
                if (leader) {
#pragma unroll
                    for (int ps = 0; ps < kPasses; ++ps)
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(reinterpret_cast<uint64_t>(&p.tmO)), "r"(grp + ps * Cfg::kBoxBytes), "r"(nt * BN + ps * EW),
                                       "r"(x0), "r"(y0), "r"(n0)
                                     : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the stores have read the boxes
                    // the next tile's residual lands while the other warpgroup runs its MMAs
                    if (has_res && more) fetch_res(tile + kItStride * static_cast<int>(gridDim.x));
                }
                // nobody writes the boxes again before the stores have read them: with a residual the next epilogue
                // waits for its TMA load (issued after the read), without one the whole group waits here
                if (has_res)
                    __syncwarp();
                else
                    named_bar_sync(bar_id, 128);
            });
            if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        } else {
            // ---- direct epilogue (fused head, fp32 outputs, split-operand mode): transpose through the warpgroup's
            // region so that thread = GEMM row = output pixel, then per-thread global accesses ----
            const int row = q * 32 + lane;
            const int px = row % p.bw;
            const int py = (row / p.bw) % p.bh;
            const int pn = row / (p.bw * p.bh);
            float* const xb = reinterpret_cast<float*>(smem_raw + (grp - smem_raw_u32));
            for_each_tile([&](int tile, bool) {
                int nt, x0, y0, n0;
                tile_origin(tile, &nt, &x0, &y0, &n0);
                const int x = x0 + px, y = y0 + py, n = n0 + pn;
                const bool valid = (row < rows_valid) && (x < p.ep.Wout) && (y < p.ep.Hout) && (n < p.ep.N);
                epilogue_tile<BN, kBF16, kHead>(p.ep, acc, xb, bar_id, valid, n, y, x, nt);
            });
        }
    }
}

}  // namespace w2l
