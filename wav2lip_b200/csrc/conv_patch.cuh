// conv_patch.cuh — "patch" variant of the implicit-GEMM conv for layers with few channels, where the generic
// kernel (conv_igemm.cuh) is bound by L2->SM operand traffic because it re-loads the input box for every
// filter tap.  Used for
//   * 3x3 / stride 1 / pad 1 blocks with Cout <= 64 (conv.py:5-19 at wav2lip.py:16-22,40-45,79-83; the
//     80->32 output block with the fused 1x1+sigmoid head, wav2lip.py:83-85),
//   * the output phases of the last transposed conv (conv.py:33-44 at wav2lip.py:79), and
//   * the first layers with tiny Cin whose kw horizontal taps are folded into K (7x7 / 3x3 on 1..15 channels).
//
// A persistent CTA
//   * keeps ALL weights of the launch resident in shared memory (taps x Cin x Cout x 2 B <= ~100 KB), loaded
//     once by TMA, and
//   * per output tile (8 wide x 16 tall pixels of one image = 128 GEMM rows) loads ONE input patch per channel
//     chunk (PW x PH pixels x BK channels, e.g. 10 x 18 for a 3x3 conv; out-of-bounds zero-filled by TMA =
//     the conv padding).
// Every tap is a shifted VIEW of that patch: in the K-major swizzled layout a pixel is one shared-memory row,
// the 8 pixels of an output row are 8 consecutive rows (one 8-row group of the wgmma descriptor) and the next output
// row starts exactly one patch row (PW pixels) further, so the descriptor of tap t is
//     start = patch + tap_row[t] * row_bytes,     stride-byte-offset = PW * row_bytes.
// The hardware swizzle is a function of the shared-memory ADDRESS bits (TMA writes and wgmma reads apply the
// same XOR), so group starts need not be aligned to the 8-row swizzle atom.  Operand traffic per tile drops from
// taps x (A + B) to one patch.
//
// Two consumer warpgroups take alternate tiles; each issues the wgmma chain of its tile into registers and runs
// the epilogue, so one group's epilogue overlaps the other's MMAs.  The ring has an even number of stages, so a
// stage is always consumed by the same warpgroup and its parity waits are in order.  The epilogue works on the
// accumulator fragment itself (no shared-memory transpose):
//   * the residual of a residual block is the block's own input, i.e. the centre of the patch that is already
//     in shared memory: each thread reads its channel pairs from there (the warpgroup releases the patch after that read);
//   * results are staged as packed 16-bit pairs at the fragment's (pixel, channel pair) in swizzled shared memory and
//     written with ONE TMA tensor store per tile (which also clips ragged edges);
//   * the fused 32 -> 3 head gathers each pixel's 32 channels into one lane of its quad (two shuffle steps) and runs
//     the dot products there in channel order;
//   * scale/shift/head weights come from the constant bank (kernel params).
//
// Channel-major form (BN = 64, BK = 64, no head: the 64 -> 64 residual blocks).  With pixels on M and 64 channels on N,
// every m64n64k16 reads 2 KB of A and 2 KB of B from shared memory per 64 tensor clocks, which is the SM's whole
// shared-memory bandwidth before the epilogue touches it.  This form swaps the operand roles: the 64 output channels
// are M (the resident weight slab [tap][cout][cin] is already the K-major A operand) and a tile of 8 x 32 = 256 pixels
// is N (the haloed 10 x 34 patch is the K-major B operand, tap t at patch + tap_row[t] rows, one 8-row group per output
// row).  One m64n256k16 reads 2 + 8 KB per 128 clocks.  The epilogue works on the accumulator fragment (rows =
// channels, so a thread needs the scale / shift of 2 channels): the residual comes from the patch centre by
// ldmatrix.trans, the output goes to a pixel-major swizzled staging tile by stmatrix.trans and leaves by one TMA store.
// A warpgroup holds 64 x 256 fp32 accumulators (128 registers per thread): setmaxnreg moves registers from the
// producer warpgroup to the consumers.
#pragma once

#include "conv_igemm.cuh"

namespace w2l {

constexpr int kPatchTileW = 8, kPatchTileH = 16;  // output tile (pixels)
constexpr int kChTileH = 32;                       // output tile height of the channel-major form (8 x 32 pixels)
__host__ __device__ constexpr bool patch_chmajor(int BN, int BK, bool head) { return BN == 64 && BK == 64 && !head; }
constexpr int kPatchThreads = 384;       // warps: 0 TMA, 1 barrier init, 2-3 idle, 4-7 consumer A, 8-11 consumer B
constexpr int kPatchMaxTaps = 9;
constexpr int kPatchMaxStages = 8;

struct alignas(64) PatchParams {
    CUtensorMap tmA;  // activations (C, W, H, N), box (BK, PW, PH, 1)
    CUtensorMap tmB;  // weights (Cin_pad, Cout_pad, taps), box (BK, BN, 1)
    CUtensorMap tmO;  // output channel slice (BN, Wl, Hl, N) with the launch's pixel strides, box (BN, 8, tile height, 1)
    CUtensorMap tmO2; // optional second destination of the same tile (a dense zero-bordered copy for a folded consumer)
    int has_out2;
    int tiles_x, tiles_y;   // tiles per image
    int kc;                 // channel chunks of BK
    int stages;             // depth of the patch ring (even)
    int PW, PH;             // patch size in pixels
    int ox, oy;             // patch origin relative to the tile origin (-1,-1 for a padded 3x3)
    int ntaps;
    int patch_bytes;        // PW*PH*BK*2 (TMA transaction size)
    int patch_stride;       // ring slot size (patch_bytes rounded up to 1024)
    int tap_row[kPatchMaxTaps];  // first patch row (pixel index) of each tap's view
    int res_row;            // >= 0: the residual IS the block input: patch row of the tile's first pixel (centre tap)
    EpiParams ep;
    float cscale[64], cshift[64];  // folded BatchNorm, constant bank
    float chead_w[96], chead_b[4]; // fused generator head
};

template <int BN, int BK, bool kBF16, bool kHead>
__global__ void __launch_bounds__(kPatchThreads, 1) conv_patch_kernel(const __grid_constant__ PatchParams p) {
    pdl_launch_dependents();
    constexpr int kSlab = BN * BK * 2;  // one (tap, chunk) weight slab
    constexpr int kRowBytes = BK * 2;
    static_assert(BN <= 64, "resident-weight variant is for narrow layers");
    static_assert(!kHead || BN == 32, "fused head expects the 32-channel output block");
    constexpr bool kCM = patch_chmajor(BN, BK, kHead);
    constexpr int kTileH = kCM ? kChTileH : kPatchTileH;

    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_raw_u32 = smem_u32(smem_raw);
    const uint32_t smem_base = (smem_raw_u32 + 1023u) & ~1023u;
    const int kc = p.kc;
    const int stages = p.stages;
    const int ntaps = p.ntaps;
    const uint32_t w_base = smem_base;
    const uint32_t a_base = w_base + static_cast<uint32_t>(ntaps * kc) * kSlab;
    const uint32_t stg_base = a_base + static_cast<uint32_t>(stages * kc) * p.patch_stride;  // a stage = all chunks of one tile
    constexpr uint32_t kStgBytes = ((kPatchTileW * kTileH * BN * 2 + 1023) / 1024) * 1024;    // one staging tile per group
    const uint32_t bar_base = stg_base + 2u * kStgBytes;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (kPatchMaxStages + s); };
    const uint32_t w_bar = bar_base + 8u * (2 * kPatchMaxStages);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&p.tmA);
        tma_prefetch_desc(&p.tmB);
        tma_prefetch_desc(&p.tmO);
        if (p.has_out2) tma_prefetch_desc(&p.tmO2);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 4);  // the 4 warps of the warpgroup that consumed the patch (MMAs retired, residual read)
        }
        mbar_init(w_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlaps the previous kernel's tail; global memory is touched only below

    const int tiles_per_img = p.tiles_x * p.tiles_y;
    const int total_tiles = tiles_per_img * p.ep.N;

    if (warp < 4) {
        if constexpr (kCM) setmaxnreg_dec<kProducerRegs>();
        // =============================== TMA producer ===============================
        if (warp == 0 && lane == 0) {
            mbar_arrive_expect_tx(w_bar, static_cast<uint32_t>(ntaps * kc) * kSlab);
            for (int tap = 0; tap < ntaps; ++tap)
                for (int c = 0; c < kc; ++c)
                    tma_load_3d(w_base + (tap * kc + c) * kSlab, &p.tmB, w_bar, c * BK, 0, tap);
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int n = tile / tiles_per_img;
                const int r = tile - n * tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                mbar_wait(empty_bar(stage), phase ^ 1u);
                mbar_arrive_expect_tx(full_bar(stage), static_cast<uint32_t>(kc) * p.patch_bytes);
                for (int c = 0; c < kc; ++c)
                    tma_load_4d(a_base + (stage * kc + c) * p.patch_stride, &p.tmA, full_bar(stage), c * BK,
                                tx * kPatchTileW + p.ox, ty * kTileH + p.oy, n);
                if (++stage == stages) { stage = 0; phase ^= 1u; }
            }
        }
    } else if constexpr (kCM) {
        setmaxnreg_inc<kConsumerRegs>();
        // ===== channel-major consumer warpgroups, alternating tiles: D[64 channels x 256 pixels] = W[64 x K] * patch[K x 256] =====
        // Fragment of m64n256k16: warp q of the group holds channels c = 16q + lane/4 (acc[4j + 0..1]) and c + 8
        // (acc[4j + 2..3]) at pixels 8j + 2(lane%4) + {0,1}, i.e. row j of the 8 x 32 tile, columns 2(lane%4) + {0,1}.
        const int grp = (warp - 4) >> 2;
        const int q = (warp - 4) & 3;
        const int ch = 16 * q + (lane >> 2);
        const float sc0 = p.cscale[ch], sh0 = p.cshift[ch], sc1 = p.cscale[ch + 8], sh1 = p.cshift[ch + 8];
        const int px = 2 * (lane & 3);
        const EpiParams& e = p.ep;
        const uint32_t stg = stg_base + grp * kStgBytes;
        const bool leader = (q == 0 && lane == 0);
        const uint32_t bar_id = 1 + grp;
        const uint32_t sbo_b = static_cast<uint32_t>(p.PW) * kRowBytes;
        uint32_t tap_off[kPatchMaxTaps];
#pragma unroll
        for (int t = 0; t < kPatchMaxTaps; ++t) tap_off[t] = (t < ntaps ? p.tap_row[t] : 0) * kRowBytes;
        mbar_wait(w_bar, 0);
        float acc[128];
        for (int it = grp;; it += 2) {
            const int tile = blockIdx.x + it * gridDim.x;
            if (tile >= total_tiles) break;
            const int stage = it % stages;
            const int n = tile / tiles_per_img;
            const int r = tile - n * tiles_per_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;

            mbar_wait(full_bar(stage), static_cast<uint32_t>(it / stages) & 1u);
            wg_fence();
            for (int c = 0; c < kc; ++c) {
                const uint32_t patch = a_base + (stage * kc + c) * p.patch_stride;
#pragma unroll
                for (int tap = 0; tap < kPatchMaxTaps; ++tap)
                    if (tap < ntaps) {
#pragma unroll
                        for (int k = 0; k < BK / 16; ++k)  // 16 channels further along K = 32 bytes inside the swizzle atom
                            wgmma_m64k16<256, kBF16>(acc, make_kmajor_desc<BK>(w_base + (tap * kc + c) * kSlab + 32u * k),
                                                     wg_desc(patch + tap_off[tap] + 32u * k, 16, sbo_b, kRowBytes),
                                                     (c | tap | k) != 0 ? 1u : 0u, 0);
                    }
            }
            wg_commit();
            wg_wait<0>();
            wg_fence_regs<128>(acc);
            if (p.res_row < 0 && lane == 0) mbar_arrive(empty_bar(stage));  // the MMAs were the patch's last readers

            // folded BatchNorm, the residual = this block's input = centre of the patch (pixel-major, swizzled by address
            // bits as TMA wrote it, output rows PW pixels apart), the activation, then the 8 x 32 tile leaves by one TMA
            // store.  Column chunk j of the fragment is tile row j: only pixels inside the image may raise the fp16 flag.
            const int x = tx * kPatchTileW + px;
            const uint32_t live_x = (x < e.Wout ? 0x8000u : 0u) | (x + 1 < e.Wout ? 0x80000000u : 0u);
            const int rows_live = e.Hout - ty * kTileH;
            const uint32_t res = p.res_row >= 0 ? a_base + (stage * kc * p.patch_stride + p.res_row * kRowBytes) : 0u;
            chmajor_epilogue<kBF16>(
                acc, sc0, sh0, sc1, sh1, e.act, res, p.PW,
                [&] {
                    if (p.res_row >= 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(empty_bar(stage));  // this warp is done with the patch
                    }
                },
                [&](int j) { return j < rows_live ? live_x : 0u; }, stg, bar_id, leader, &p.tmO, 0, tx * kPatchTileW,
                ty * kTileH, n);
        }
        if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete before exit
    } else {
        // ============ consumer warpgroups (MMA + epilogue), alternating tiles: group g takes tiles g, g+2, .. ============
        // Fragment of m64nBNk16: warp q holds the GEMM rows 64h + 16q + lane/4 + 8r8 (h, r8 in {0,1}), i.e. tile pixel
        // x = lane/4 of the rows 8h + 2q + r8 of the 8 x 16 tile, and in every 8-column chunk j the channel pair
        // 8j + 2(lane%4) (acc[h][4j + 2r8 + {0,1}]).
        const int grp = (warp - 4) >> 2;
        const int q = (warp - 4) & 3;
        const int px = lane >> 2;
        const int cq = 2 * (lane & 3);
        const EpiParams& e = p.ep;
        constexpr uint32_t kOutRow = BN * 2;                                   // bytes per pixel in the staging tile
        constexpr uint32_t kOutSwz = (kOutRow == 128) ? 7u : (kOutRow == 64) ? 3u : 1u;   // matches tmO's swizzle mode
        constexpr uint32_t kInSwz = (BK == 64) ? 7u : (BK == 32) ? 3u : 1u;
        const uint32_t stg = stg_base + grp * kStgBytes;
        const bool leader = (q == 0 && lane == 0);
        const uint32_t bar_id = 1 + grp;  // named barrier of this group (0 is __syncthreads)
        // Every tap is a shifted view of the patch: the 8 pixels of an output row are 8 consecutive patch rows (one 8-row
        // group of the descriptor) and the next output row starts one patch row (PW pixels) further.
        const uint32_t sbo_a = static_cast<uint32_t>(p.PW) * kRowBytes;
        uint32_t tap_off[kPatchMaxTaps];
#pragma unroll
        for (int t = 0; t < kPatchMaxTaps; ++t) tap_off[t] = (t < ntaps ? p.tap_row[t] : 0) * kRowBytes;
        mbar_wait(w_bar, 0);
        float acc[2][BN / 2];
        for (int it = grp;; it += 2) {
            const int tile = blockIdx.x + it * gridDim.x;
            if (tile >= total_tiles) break;
            const int stage = it % stages;
            const int n = tile / tiles_per_img;
            const int r = tile - n * tiles_per_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;

            mbar_wait(full_bar(stage), static_cast<uint32_t>(it / stages) & 1u);
            wg_fence();
            for (int c = 0; c < kc; ++c) {
                const uint32_t patch = a_base + (stage * kc + c) * p.patch_stride;
#pragma unroll
                for (int tap = 0; tap < kPatchMaxTaps; ++tap)
                    if (tap < ntaps)
                        wg_mma_tile<BN, BK, kBF16>(acc, patch + tap_off[tap], sbo_a, w_base + (tap * kc + c) * kSlab, (c | tap) != 0);
            }
            wg_commit();
            wg_wait<0>();
            wg_fence_regs<BN / 2>(acc[0]);
            wg_fence_regs<BN / 2>(acc[1]);
            if (p.res_row < 0 && lane == 0) mbar_arrive(empty_bar(stage));  // the MMAs were the patch's last readers

            // folded BatchNorm, the residual = this block's input = centre of the patch still resident in shared memory
            // (K-major, swizzled by address bits exactly as TMA wrote it), the activation: all on the fragment
            const uint32_t res = a_base + stage * kc * p.patch_stride + (p.res_row + px) * kRowBytes;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int cc = 8 * j + cq;
                const float sc0 = p.cscale[cc], sc1 = p.cscale[cc + 1], sh0 = p.cshift[cc], sh1 = p.cshift[cc + 1];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int r8 = 0; r8 < 2; ++r8) {
                        float* const a = &acc[h][4 * j + 2 * r8];
                        a[0] = fmaf(a[0], sc0, sh0);
                        a[1] = fmaf(a[1], sc1, sh1);
                        if (p.res_row >= 0) {
                            uint32_t ad = res + static_cast<uint32_t>((8 * h + 2 * q + r8) * p.PW) * kRowBytes + cc * 2;
                            ad ^= ((ad >> 7) & kInSwz) << 4;
                            uint32_t rv;
                            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rv) : "r"(ad));
                            const float2 v = unpack2<kBF16>(rv);
                            a[0] += v.x;
                            a[1] += v.y;
                        }
                    }
            }
            if (p.res_row >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(stage));  // this warp is done with the patch
            }
            if (e.act == ACT_RELU) {
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) { acc[0][j] = fmaxf(acc[0][j], 0.0f); acc[1][j] = fmaxf(acc[1][j], 0.0f); }
            } else if (e.act == ACT_LRELU) {
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) {
                    acc[0][j] = acc[0][j] > 0.0f ? acc[0][j] : 0.01f * acc[0][j];
                    acc[1][j] = acc[1][j] > 0.0f ? acc[1][j] : 0.01f * acc[1][j];
                }
            }
            if constexpr (kHead) {
                // wav2lip.py:84-85: Conv2d(32,3,1) + Sigmoid on the fp32 block output still in registers.  The four lanes of
                // a quad hold the same four pixels (rows (h, r8)) and each 8 of their 32 channels; a two-step butterfly
                // inside the quad gives lane t = 2h + r8 all 32 channels of row (h, r8), so each thread finishes one pixel
                // with the dot products in channel order.
                const int lh = (lane >> 1) & 1, lr = lane & 1;  // quad lane = 2 lh + lr holds pixel row (lh, lr)
                float z[2][2][8];  // after the xor-2 step: z[s][r8][2j + e] = channel 8j + 2(2s + lr) + e of row (lh, r8)
#pragma unroll
                for (int r8 = 0; r8 < 2; ++r8)
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int k = 4 * (i >> 1) + 2 * r8 + (i & 1);
                        const float recv = __shfl_xor_sync(0xffffffffu, lh ? acc[0][k] : acc[1][k], 2);
                        z[0][r8][i] = lh ? recv : acc[0][k];
                        z[1][r8][i] = lh ? acc[1][k] : recv;
                    }
                float f[32];
#pragma unroll
                for (int sh = 0; sh < 2; ++sh)
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const float recv = __shfl_xor_sync(0xffffffffu, lr ? z[sh][0][i] : z[sh][1][i], 1);
                        // source lane (sh, sb) holds channels 8j + 2(2 sh + sb) + e of chunk j = i / 2, e = i % 2
                        const int c0 = 8 * (i >> 1) + 2 * (2 * sh) + (i & 1);
                        f[c0] = lr ? recv : z[sh][0][i];
                        f[c0 + 2] = lr ? z[sh][1][i] : recv;
                    }
                const int x = tx * kPatchTileW + px, y = ty * kPatchTileH + 8 * lh + 2 * q + lr;
                if (x < e.Wout && y < e.Hout) {
                    const int hb = n % e.head_B, ht = n / e.head_B;
                    const long long plane = (long long)e.Hout * e.Wout;
#pragma unroll
                    for (int oc = 0; oc < 3; ++oc) {
                        float s = p.chead_b[oc];
#pragma unroll
                        for (int j = 0; j < 32; ++j) s = fmaf(f[j], p.chead_w[oc * 32 + j], s);
                        s = 1.0f / (1.0f + __expf(-s));
                        if (e.head_out_u8 != nullptr)
                            e.head_out_u8[(((long long)n * e.Hout + y) * e.Wout + x) * 3 + oc] = (unsigned char)__fmul_rn(s, 255.0f);
                        else
                            e.head_out[(((long long)hb * 3 + oc) * e.head_T + ht) * plane + (long long)y * e.Wout + x] = s;
                    }
                }
            } else {
                // stage the tile (pixel-major rows of BN 16-bit channels, hardware swizzle pattern) and TMA-store it
                if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // previous store has read the buffer
                named_bar_sync(bar_id, 128);
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int r8 = 0; r8 < 2; ++r8) {
                            uint32_t a = stg + (64 * h + 16 * q + 8 * r8 + px) * kOutRow + (8 * j + cq) * 2;
                            a ^= ((a >> 7) & kOutSwz) << 4;
                            const uint32_t o = pack2<kBF16>(acc[h][4 * j + 2 * r8], acc[h][4 * j + 2 * r8 + 1]);
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(o) : "memory");
                        }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
                named_bar_sync(bar_id, 128);
                if (leader) {
                    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                 ::"l"(reinterpret_cast<uint64_t>(&p.tmO)), "r"(stg), "r"(0), "r"(tx * kPatchTileW), "r"(ty * kPatchTileH), "r"(n)
                                 : "memory");
                    if (p.has_out2)
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(reinterpret_cast<uint64_t>(&p.tmO2)), "r"(stg), "r"(0), "r"(tx * kPatchTileW), "r"(ty * kPatchTileH), "r"(n)
                                     : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (!kHead && leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete before exit
    }
}

}  // namespace w2l
