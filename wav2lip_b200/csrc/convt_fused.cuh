// convt_fused.cuh — Conv2dTranspose(k=3, stride=2, pad=1, output_padding=1) + BatchNorm + ReLU
// (/root/reference/models/conv.py:33-44, used for the 48x48 -> 96x96 stage at wav2lip.py:79) with all FOUR
// output phases computed by one kernel from one read of the input.
//
// out[2y+py, 2x+px] = sum over the taps (r,s) with r = (py+1) mod 2 (+2), s likewise, of
// in[y + dy, x + dx] * w[:, :, r, s], dy = (py + 1 - r)/2 in {0,1}: 1/2/2/4 taps for the four phases, 9 in total —
// only true MACs, no zero-insertion.  The generic path runs one launch per phase and therefore reads the input
// four times from HBM (4 x 472 MB at N=640).
// Here a work unit is one 8 x 16 tile of INPUT pixels of one image:
//   * a K step = one chunk of BK input channels: ONE TMA load of the (9 x 17 pixel) input patch chunk (the +1
//     halo on the right/bottom is zero-filled at the border) and ONE 3-D TMA load of the 9 weight slabs
//     [tap][64][BK] of that chunk;
//   * the four output phases live side by side in one 256-column accumulator, in the order [00 | 11 | 01 | 10], and
//     the 9 taps are issued as wide instructions, one per input shift (dy,dx) and consumer warpgroup — an input pixel
//     feeds every phase it touches:   (0,0) -> all four phases;   (0,1) -> phases 01,11;   (1,0) -> phases 11,10;
//     (1,1) -> 11.  With the weight slabs packed in the order of host_weights.cuh every B operand is a contiguous window;
//   * two consumer warpgroups each own half of the accumulator (registers): group 0 the columns of phases 00,11
//     (N = 128 from shift (0,0), then N = 64 from (0,1), (1,0), (1,1) into phase 11: 5 tap products per k16), group 1
//     those of 01,10 (N = 128 from (0,0), N = 64 from (0,1) into 01 and from (1,0) into 10: 4 tap products);  every
//     phase accumulates over (chunk, k16, shift) in that order;
//   * each group then drains its two phases on the accumulator fragment itself: scale/shift + activation, packed
//     16-bit pairs into the swizzled staging tile at the fragment's (row, column pair), one TMA tensor store per phase
//     through a strided (every-other-pixel) view of the output channel slice.  No transpose buffer: the shared memory
//     goes to ring stages, so the producer loads the next unit's K steps while both groups run their epilogues.
#pragma once

#include "conv_igemm.cuh"

namespace w2l {

constexpr int kCtThreads = 384;
constexpr int kCtBN = 64;
constexpr int kCtPW = 9, kCtPH = 17;
constexpr int kCtMaxStages = 6;

struct alignas(64) ConvTParams {
    CUtensorMap tmA;     // input (C, W, H, N), box (BK, 9, 17, 1)
    CUtensorMap tmB;     // weights (Cin_pad, 64, 9), box (BK, 64, 9)
    CUtensorMap tmO[4];  // output phase views (64, W, H, N) with doubled pixel strides, box (64, 8, 16, 1)
    int tiles_x, tiles_y, N;
    int kc;              // K steps per unit
    int stages;
    int patch_bytes, patch_stride;
    int act;
    float cscale[64], cshift[64];
};

// Consumer warpgroup G (MMA + epilogue) of every unit of the CTA.  G is a template parameter so that each group's wgmma
// chain is straight-line code (no branch on the group between the instructions of one K step).
template <int G, int BK, bool kBF16>
__device__ __forceinline__ void convt_consumer(const ConvTParams& p, uint32_t smem_base, uint32_t stg, uint32_t bar_base) {
    constexpr int BN = kCtBN;
    constexpr int kRowBytes = BK * 2;
    constexpr int kSlab = BN * BK * 2;
    constexpr uint32_t kSboA = kCtPW * kRowBytes;   // next output row = next patch row
    constexpr uint32_t kSboB = 8 * kRowBytes;
    constexpr uint32_t kRowB = BN * 2;              // staging tile: 128 pixel rows of 64 16-bit channels, 128-byte swizzle
    const int kc = p.kc;
    const int stages = p.stages;
    const uint32_t stage_bytes = p.patch_stride + 9u * kSlab;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kCtMaxStages + s); };
    const int lane = threadIdx.x & 31;
    const int q = (threadIdx.x >> 5) & 3;
    const bool leader = (q == 0 && lane == 0);
    const uint32_t bar_id = 1 + G;
    const int tiles_per_img = p.tiles_x * p.tiles_y;
    const int total_units = tiles_per_img * p.N;
    float acc[2][64];
    int stage = 0;
    uint32_t phase = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const int n = unit / tiles_per_img;
        const int r = unit - n * tiles_per_img;
        const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
        int prev = -1;
        for (int c = 0; c < kc; ++c) {
            mbar_wait(full_bar(stage), phase);
            const uint32_t patch = smem_base + stage * stage_bytes;
            const uint32_t wslab = patch + p.patch_stride;
            wg_fence();
            // input shifts (dy,dx) = patch rows dy*9 + dx; weight slabs in the packed order of host_weights.cuh:
            // (0,0) -> 00 11 01 10 (slabs 0-3), into 11: (0,1) (1,0) (1,1) (slabs 4-6), (0,1) -> 01 (slab 7), (1,0) -> 10 (slab 8)
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                const uint32_t on = (c | k) != 0 ? 1u : 0u;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t a0 = patch + h * 8 * kSboA + 32u * k;
                    auto ad = [&](uint32_t rows) { return wg_desc(a0 + rows * kRowBytes, 16, kSboA, kRowBytes); };
                    auto bd = [&](int slab) { return wg_desc(wslab + slab * kSlab + 32u * k, 16, kSboB, kRowBytes); };
                    if constexpr (G == 0) {  // [00 | 11]
                        wgmma_m64k16<128, kBF16>(acc[h], ad(0), bd(0), on, 0);
                        wgmma_m64k16<64, kBF16>(acc[h] + 32, ad(1), bd(4), 1u, 0);
                        wgmma_m64k16<64, kBF16>(acc[h] + 32, ad(kCtPW), bd(5), 1u, 0);
                        wgmma_m64k16<64, kBF16>(acc[h] + 32, ad(kCtPW + 1), bd(6), 1u, 0);
                    } else {                 // [01 | 10]
                        wgmma_m64k16<128, kBF16>(acc[h], ad(0), bd(2), on, 0);
                        wgmma_m64k16<64, kBF16>(acc[h], ad(1), bd(7), 1u, 0);
                        wgmma_m64k16<64, kBF16>(acc[h] + 32, ad(kCtPW), bd(8), 1u, 0);
                    }
                }
            }
            wg_commit();
            wg_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
        wg_wait<0>();
        wg_fence_regs<64>(acc[0]);
        wg_fence_regs<64>(acc[1]);
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        // epilogue on the fragment of m64n128k16: this thread holds rows 16q + lane/4 (+8) of each 64-row half and, in
        // every 8-column chunk, the column pair 2(lane%4); chunks 0-7 are the group's first phase, 8-15 its second
#pragma unroll
        for (int lp = 0; lp < 2; ++lp) {
            const int ph = G == 0 ? 3 * lp : 1 + lp;  // tmO index py*2 + px: group 0 holds 00, 11, group 1 holds 01, 10
            if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // previous store has read the tile
            named_bar_sync(bar_id, 128);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int cc = 8 * j + 2 * (lane & 3);
                const float sc0 = p.cscale[cc], sc1 = p.cscale[cc + 1], sh0 = p.cshift[cc], sh1 = p.cshift[cc + 1];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int r8 = 0; r8 < 2; ++r8) {
                        const int row = 64 * h + 16 * q + (lane >> 2) + 8 * r8;
                        float f0 = fmaf(acc[h][4 * (8 * lp + j) + 2 * r8], sc0, sh0);
                        float f1 = fmaf(acc[h][4 * (8 * lp + j) + 2 * r8 + 1], sc1, sh1);
                        if (p.act == ACT_RELU) {
                            f0 = fmaxf(f0, 0.0f);
                            f1 = fmaxf(f1, 0.0f);
                        } else if (p.act == ACT_LRELU) {
                            f0 = f0 > 0.0f ? f0 : 0.01f * f0;
                            f1 = f1 > 0.0f ? f1 : 0.01f * f1;
                        }
                        uint32_t a = stg + row * kRowB + cc * 2;
                        a ^= ((a >> 7) & 7u) << 4;
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack2<kBF16>(f0, f1)) : "memory");
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
            named_bar_sync(bar_id, 128);
            if (leader) {
                asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                             ::"l"(reinterpret_cast<uint64_t>(&p.tmO[ph])), "r"(stg), "r"(0), "r"(tx * 8), "r"(ty * 16), "r"(n)
                             : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <int BK, bool kBF16>
__global__ void __launch_bounds__(kCtThreads, 1) convt_fused_kernel(const __grid_constant__ ConvTParams p) {
    pdl_launch_dependents();
    constexpr uint32_t kStgBytes = kTileM * kCtBN * 2;  // 16 KB staging tile per consumer warpgroup
    constexpr int kSlab = kCtBN * BK * 2;

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int kc = p.kc;
    const int stages = p.stages;
    const uint32_t stage_bytes = p.patch_stride + 9u * kSlab;
    const uint32_t stg_base = smem_base + stages * stage_bytes;
    const uint32_t bar_base = stg_base + 2u * kStgBytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kCtMaxStages + s); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
#pragma unroll
        for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.tmO[i]);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 8);  // both consumer warpgroups read every stage
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlaps the previous kernel's tail; global memory is touched only below

    const int tiles_per_img = p.tiles_x * p.tiles_y;
    const int total_units = tiles_per_img * p.N;

    if (warp < 4) {
        setmaxnreg_dec<kProducerRegs>();  // registers go to the consumers' 128 accumulators
        // =============================== TMA producer ===============================
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
                const int n = unit / tiles_per_img;
                const int r = unit - n * tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                for (int c = 0; c < kc; ++c) {
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    const uint32_t a_dst = smem_base + stage * stage_bytes;
                    mbar_arrive_expect_tx(full_bar(stage), static_cast<uint32_t>(p.patch_bytes) + 9u * kSlab);
                    tma_load_4d(a_dst, &p.tmA, full_bar(stage), c * BK, tx * 8, ty * 16, n);
                    tma_load_3d(a_dst + p.patch_stride, &p.tmB, full_bar(stage), c * BK, 0, 0);
                    if (++stage == stages) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        setmaxnreg_inc<kConsumerRegs>();
        if (warp >= 8)
            convt_consumer<1, BK, kBF16>(p, smem_base, stg_base + kStgBytes, bar_base);
        else
            convt_consumer<0, BK, kBF16>(p, smem_base, stg_base, bar_base);
    }
}

}  // namespace w2l
