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
//   * the four output phases live side by side in one 256-column accumulator, in the order [00 | 01 | 11 | 10], and
//     the 9 taps are issued as wide instructions, one per input shift (dy,dx) — an input pixel feeds every phase it
//     touches at once:   (0,0) -> all four phases;   (0,1) -> phases 01,11;   (1,0) -> phases 11,10;   (1,1) -> 11.
//     With the weight slabs packed in that order every B operand is a contiguous window;
//   * two consumer warpgroups each own half of the accumulator (registers): group 0 the columns of phases 00,01
//     (N = 128 from shift (0,0), N = 64 from (0,1)), group 1 those of 11,10 (N = 128, 64, 128, 64); each then drains
//     its two phases: scale/shift + ReLU, swizzled staging tile, one TMA tensor store per phase through a strided
//     (every-other-pixel) view of the output channel slice.
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

template <int BK, bool kBF16>
__global__ void __launch_bounds__(kCtThreads, 1) convt_fused_kernel(const __grid_constant__ ConvTParams p) {
    pdl_launch_dependents();
    constexpr int BN = kCtBN;
    constexpr int kRowBytes = BK * 2;
    constexpr int kSlab = BN * BK * 2;
    constexpr uint32_t kStgBytes = kTileM * BN * 2;  // 16 KB staging tile per consumer warpgroup

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_raw_u32 = smem_u32(smem_raw);
    const uint32_t smem_base = (smem_raw_u32 + 1023u) & ~1023u;
    const int kc = p.kc;
    const int stages = p.stages;
    const uint32_t stage_bytes = p.patch_stride + 9u * kSlab;
    const uint32_t stg_base = smem_base + stages * stage_bytes;
    const uint32_t xb_base = stg_base + 2u * kStgBytes;
    const uint32_t bar_base = xb_base + 2u * xbuf_bytes<16>();
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

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
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
    } else if (warp >= 4) {
        // ===== consumer warpgroup g: accumulator columns [128 g, 128 g + 128) = phases 2g and 2g+1, MMA + epilogue =====
        const int grp = (warp - 4) >> 2;
        const int q = (warp - 4) & 3;
        const int row = q * 32 + lane;
        const uint32_t stg = stg_base + grp * kStgBytes;
        float* const xb = reinterpret_cast<float*>(smem_raw + (xb_base - smem_raw_u32) + grp * xbuf_bytes<16>());
        const bool leader = (q == 0 && lane == 0);
        const uint32_t bar_id = 1 + grp;
        constexpr uint32_t kSboA = kCtPW * kRowBytes;   // next output row = next patch row
        constexpr uint32_t kSboB = 8 * kRowBytes;
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
                // input shifts (dy,dx) = patch rows dy*9 + dx; weight slabs in the packed order of host_weights.cuh.  Column
                // order of the full accumulator is [00 | 01 | 11 | 10] (64 each): (0,0) feeds all four phases (slabs 0-3),
                // (0,1) phases 01,11 (slabs 4,5), (1,0) phases 11,10 (slabs 6,7), (1,1) phase 11 (slab 8).
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint32_t on = (c | k) != 0 ? 1u : 0u;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t a0 = patch + h * 8 * kSboA + 32u * k;
                        auto ad = [&](uint32_t rows) { return wg_desc(a0 + rows * kRowBytes, 16, kSboA, kRowBytes); };
                        auto bd = [&](int slab) { return wg_desc(wslab + slab * kSlab + 32u * k, 16, kSboB, kRowBytes); };
                        if (grp == 0) {
                            wgmma_m64k16<128, kBF16>(acc[h], ad(0), bd(0), on, 0);
                            wgmma_m64k16<64, kBF16>(acc[h] + 32, ad(1), bd(4), 1u, 0);
                        } else {
                            wgmma_m64k16<128, kBF16>(acc[h], ad(0), bd(2), on, 0);
                            wgmma_m64k16<64, kBF16>(acc[h], ad(1), bd(5), 1u, 0);
                            wgmma_m64k16<128, kBF16>(acc[h], ad(kCtPW), bd(6), 1u, 0);
                            wgmma_m64k16<64, kBF16>(acc[h], ad(kCtPW + 1), bd(8), 1u, 0);
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
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                // local columns [64 h, 64 h + 64) of this warpgroup's half; the full accumulator's column order is
                // [00 | 01 | 11 | 10], so group 1 holds phase 11 (index 3) first, then 10 (index 2)
                const int ph = grp == 0 ? h : 3 - h;
                const int col0 = h * BN;
                if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
                for (int c0 = 0; c0 < BN; c0 += 16) {
                    uint32_t v[16];
                    acc_to_rows<16>(acc[0], acc[1], col0 + c0, xb, bar_id, v);
#pragma unroll
                    for (int jj = 0; jj < 2; ++jj) {
                        const int j = c0 / 8 + jj;
                        float f[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            f[i] = fmaf(__uint_as_float(v[8 * jj + i]), p.cscale[8 * j + i], p.cshift[8 * j + i]);
                            if (p.act == ACT_RELU) f[i] = fmaxf(f[i], 0.0f);
                            else if (p.act == ACT_LRELU) f[i] = f[i] > 0.0f ? f[i] : 0.01f * f[i];
                        }
                        uint32_t a = stg + row * (BN * 2) + j * 16;
                        a ^= ((a >> 7) & 7u) << 4;
                        const uint32_t o0 = pack2<kBF16>(f[0], f[1]), o1 = pack2<kBF16>(f[2], f[3]);
                        const uint32_t o2 = pack2<kBF16>(f[4], f[5]), o3 = pack2<kBF16>(f[6], f[7]);
                        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(o0), "r"(o1), "r"(o2), "r"(o3) : "memory");
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
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
}

}  // namespace w2l
