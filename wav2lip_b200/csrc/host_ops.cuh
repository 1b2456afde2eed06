// host_ops.cuh — turning one conv block of a spec table into launches: tile/box selection, TMA tensor maps for the
// activations / weights / outputs, the parameter blocks of the three kernel families, transposed-conv phases.
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// building one conv launch
// ------------------------------------------------------------------------------------------------
static int pick_bk(int cin_pad) { return (cin_pad % 64 == 0) ? 64 : (cin_pad % 32 == 0) ? 32 : 16; }
static int round_up(int a, int b) { return (a + b - 1) / b * b; }
// channel-major selection (make_conv_op), set from the per-launch times of the generator at N = 640 on an H100 SXM (DESIGN
// section 6): least K steps per tile, least K steps per CTA (rounds x K steps: the pipeline fill and the exposed epilogues are
// amortised over it), and how much worse than the row-major tiles' the fill of the grid's rounds may be
constexpr int kCmMinSteps = 18;
constexpr int kCmMinCtaSteps = 48;
constexpr double kCmFillMargin = 0.06;

// A tile of `pixels` GEMM rows (columns in the channel-major form) is a (bw x bh x bn) box of output pixels; choose the
// box with the least padding waste.
static void pick_box(int W, int H, int N, int sx, int sy, int* bw, int* bh, int* bn, int pixels = kTileM) {
    double best = 1e30;
    int b_w = 1, b_h = 1, b_n = 1;
    for (int w = 1; w <= std::min(W, pixels); ++w) {
        if (w * sx > 256) break;
        for (int h = 1; h <= std::min(H, pixels / w); ++h) {
            if (h * sy > 256) break;
            int n = std::min(pixels / (w * h), std::max(N, 1));
            if (n < 1) continue;
            if (n > 256) n = 256;
            const double tiles = (double)((W + w - 1) / w) * ((H + h - 1) / h) * ((N + n - 1) / n);
            // prefer wide boxes (longer contiguous runs) on ties
            const double cost = tiles - 1e-6 * w - 1e-9 * h;
            if (cost < best) { best = cost; b_w = w; b_h = h; b_n = n; }
        }
    }
    *bw = b_w; *bh = b_h; *bn = b_n;
}

struct ConvArgs {
    std::string name;
    Act in, out;
    const PackedW* w = nullptr;
    int sx = 1, sy = 1;        // input stride per logical output pixel
    int Hl = 0, Wl = 0;        // logical output grid handled by this launch
    int osy = 1, osx = 1;      // output pixel = logical * os + phase
    int phy = 0, phx = 0;
    const Act* res = nullptr;
    const float* scale = nullptr;
    const float* shift = nullptr;
    int ch_off = 0;            // offset into scale/shift
    int act = ACT_RELU;
    int cout = 0;              // channels produced
    double macs_per_pixel = 0; // true MACs per logical output pixel (for flop accounting)
    // fused head
    bool head = false;
    const float* head_w = nullptr;
    const float* head_b = nullptr;
    int head_B = 1, head_T = 1;
};

static void fill_epi(EpiParams* e, const ConvArgs& a) {
    memset(e, 0, sizeof(*e));
    e->Wout = a.Wl; e->Hout = a.Hl; e->N = a.in.N;
    e->act = a.act;
    e->out_f32 = a.out.f32 ? 1 : 0;
    const long long oCs = a.out.Cs;
    const long long Wfull = a.out.W;
    if (!a.head) {
        const long long base_off = ((long long)a.phy * Wfull + a.phx) * oCs + a.out.c_off;
        e->out = a.out.f32 ? (void*)((float*)a.out.base + base_off) : (void*)(a.out.base + base_off);
        e->out_sn = (long long)a.out.H * Wfull * oCs;
        e->out_sy = (long long)a.osy * Wfull * oCs;
        e->out_sx = (long long)a.osx * oCs;
    }
    if (a.res) {
        // same pixel mapping as the output: logical pixel (y, x) of a phase launch is pixel (y*osy + phy, x*osx + phx)
        // (the forward never adds a residual to a transposed conv; the dgrad of a strided conv does: the skip gradient)
        const long long rCs = a.res->Cs, rW = a.res->W;
        e->res = a.res->ptr() + ((long long)a.phy * rW + a.phx) * rCs;
        e->res_sn = (long long)a.res->H * rW * rCs;
        e->res_sy = (long long)a.osy * rW * rCs;
        e->res_sx = (long long)a.osx * rCs;
    }
    e->scale = a.scale + a.ch_off;
    e->shift = a.shift + a.ch_off;
    e->head_w = a.head_w; e->head_b = a.head_b; e->head_out = nullptr; e->head_B = a.head_B; e->head_T = a.head_T;
    e->x2 = (a.out.lo_off > 0 || (a.res && a.res->lo_off > 0)) ? 1 : 0;
    e->out_lo_off = a.out.lo_off;
    e->res_lo_off = a.res ? a.res->lo_off : 0;
}

static int encode_act_map(w2l_ctx* ctx, CUtensorMap* tm, const Act& in, int BK, int bx, int by, int bn, int sx, int sy,
                          const char* name) {
    EncodeTiledFn enc = get_encode_fn();
    const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUtensorMapSwizzle sw = BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : BK == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    cuuint64_t dims[4] = {(cuuint64_t)(in.lo_off + in.C), (cuuint64_t)(in.nwin ? in.nwin : in.W), (cuuint64_t)in.H, (cuuint64_t)in.N};
    cuuint64_t strides[3] = {(cuuint64_t)in.Cs * in.wstride * 2, (cuuint64_t)in.pitch() * in.Cs * 2, (cuuint64_t)in.H * in.pitch() * in.Cs * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)bx, (cuuint32_t)by, (cuuint32_t)bn};
    cuuint32_t es[4] = {1, (cuuint32_t)sx, (cuuint32_t)sy, 1};
    CUresult r = enc(tm, dt, 4, in.ptr(), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(A) failed with %d (dims %d,%d,%d,%d box %d,%d,%d,%d)", name, (int)r,
                    in.C, in.W, in.H, in.N, BK, bx, by, bn);
    return W2L_OK;
}

static int encode_w_map(w2l_ctx* ctx, CUtensorMap* tm, const PackedW& w, int BK, int BN, const char* name) {
    EncodeTiledFn enc = get_encode_fn();
    const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUtensorMapSwizzle sw = BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : BK == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad, (cuuint64_t)w.cout_pad, (cuuint64_t)(w.nslabs ? w.nslabs : w.ntaps)};
    cuuint64_t strides[2] = {(cuuint64_t)w.cin_pad * 2, (cuuint64_t)w.cin_pad * w.cout_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BN, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = enc(tm, dt, 3, w.w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(B) failed with %d", name, (int)r);
    return W2L_OK;
}

// Few-channel stride-1 layers: one input patch per tile + resident weights (conv_patch.cuh)
struct PatchGeom { int ox, oy, PW, PH, BK, TH, patch_bytes, patch_stride, wbytes, stg_bytes, res_tap; };

// weights + patch ring + staging; the barriers come on top
constexpr int kPatchSmemBudget = kSmemMax - kSmemExtra;

static bool patch_eligible(const w2l_ctx* ctx, const ConvArgs& a, PatchGeom* g) {
    if (!ctx->use_patch) return false;
    const PackedW& w = *a.w;
    if (a.sx != 1 || a.sy != 1 || w.ntaps > kPatchMaxTaps) return false;
    if (a.cout != 16 && a.cout != 32 && a.cout != 64) return false;
    if (w.cout_pad != a.cout) return false;
    if (a.head && a.cout != 32) return false;
    if (a.Wl < kPatchTileW || a.Hl < kPatchTileW) return false;
    if (a.out.f32) return false;
    g->BK = pick_bk(w.cin_pad);
    // the 64 -> 64 form runs channel-major on 8 x 32 tiles (conv_patch.cuh)
    g->TH = patch_chmajor(a.cout, g->BK, a.head) ? kChTileH : kPatchTileH;
    const double tiles = (double)((a.Wl + kPatchTileW - 1) / kPatchTileW) * ((a.Hl + g->TH - 1) / g->TH);
    if ((double)a.Wl * a.Hl / (tiles * kPatchTileW * g->TH) < 0.6) return false;
    int mnx = 127, mxx = -127, mny = 127, mxy = -127;
    for (int t = 0; t < w.ntaps; ++t) {
        mnx = std::min(mnx, (int)w.dx[t]); mxx = std::max(mxx, (int)w.dx[t]);
        mny = std::min(mny, (int)w.dy[t]); mxy = std::max(mxy, (int)w.dy[t]);
    }
    g->ox = mnx; g->oy = mny;
    g->PW = kPatchTileW + (mxx - mnx); g->PH = g->TH + (mxy - mny);
    g->patch_bytes = g->PW * g->PH * g->BK * 2;
    g->patch_stride = (g->patch_bytes + 1023) / 1024 * 1024;
    g->wbytes = w.ntaps * w.cin_pad * a.cout * 2;
    g->stg_bytes = 2 * ((kPatchTileW * g->TH * a.cout * 2 + 1023) / 1024 * 1024);  // the kernel always carves two staging tiles
    if (g->PW > 256 || g->PH > 256) return false;
    if (g->wbytes + g->stg_bytes + 2 * (w.cin_pad / g->BK) * g->patch_stride > kPatchSmemBudget) return false;
    g->res_tap = -1;
    if (a.res) {
        // the patch kernel takes the residual from the input patch in shared memory: it must BE the block input
        if (a.res->base != a.in.base || a.res->c_off != a.in.c_off || a.res->Cs != a.in.Cs) return false;
        if (w.cin_pad != a.cout || w.cin_pad != g->BK) return false;
        for (int t = 0; t < w.ntaps; ++t)
            if (w.dx[t] == 0 && w.dy[t] == 0) g->res_tap = t;
        if (g->res_tap < 0) return false;
    }
    return true;
}

static int make_patch_op(w2l_ctx* ctx, Plan* pl, const ConvArgs& a, const PatchGeom& g) {
    Op op;
    op.type = OP_CONV;
    op.name = a.name + (a.w->fold ? " [fold+patch]" : " [patch]");
    op.patch = true;
    op.head = a.head;
    const PackedW& w = *a.w;
    const int BK = g.BK, BN = a.cout;
    op.BN = BN; op.BK = BK;
    PatchParams& h = op.pp;
    memset(&h, 0, sizeof(h));
    CKR(encode_act_map(ctx, &h.tmA, a.in, BK, g.PW, g.PH, 1, 1, 1, a.name.c_str()));
    CKR(encode_w_map(ctx, &h.tmB, w, BK, BN, a.name.c_str()));
    h.tiles_x = (a.Wl + kPatchTileW - 1) / kPatchTileW;
    h.tiles_y = (a.Hl + g.TH - 1) / g.TH;
    h.kc = w.cin_pad / BK;
    h.PW = g.PW; h.PH = g.PH; h.ox = g.ox; h.oy = g.oy;
    h.ntaps = w.ntaps;
    h.patch_bytes = g.patch_bytes; h.patch_stride = g.patch_stride;
    for (int t = 0; t < w.ntaps; ++t) h.tap_row[t] = (w.dy[t] - g.oy) * g.PW + (w.dx[t] - g.ox);
    // even: the two consumer warpgroups take alternate tiles, so each stage always goes to the same one
    h.stages = std::min(kPatchMaxStages, (kPatchSmemBudget - g.wbytes - g.stg_bytes) / (h.kc * g.patch_stride)) & ~1;
    op.dyn_smem = g.wbytes + h.stages * h.kc * g.patch_stride + g.stg_bytes + kSmemExtra;
    if (op.dyn_smem > kSmemMax || h.stages < 2) return fail(W2L_EINVAL, "%s: patch kernel smem plan %d B / %d stages", a.name.c_str(), op.dyn_smem, h.stages);
    fill_epi(&h.ep, a);
    h.res_row = g.res_tap >= 0 ? h.tap_row[g.res_tap] : -1;
    if (!a.head) {
        // TMA-store view of the output: the BN-channel slice, with this launch's pixel strides (transposed-conv phases
        // interleave), box = one tile; out-of-range pixels of ragged tiles are clipped by the TMA unit
        EncodeTiledFn enc = get_encode_fn();
        const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
        const CUtensorMapSwizzle sw = BN == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : BN == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
        cuuint64_t dims[4] = {(cuuint64_t)BN, (cuuint64_t)a.Wl, (cuuint64_t)a.Hl, (cuuint64_t)a.in.N};
        cuuint64_t strides[3] = {(cuuint64_t)h.ep.out_sx * 2, (cuuint64_t)h.ep.out_sy * 2, (cuuint64_t)h.ep.out_sn * 2};
        cuuint32_t box[4] = {(cuuint32_t)BN, (cuuint32_t)kPatchTileW, (cuuint32_t)g.TH, 1};
        cuuint32_t es[4] = {1, 1, 1, 1};
        if (a.out.f32) return fail(W2L_EINVAL, "%s: patch kernel stores 16-bit outputs only", a.name.c_str());
        CUresult r = enc(&h.tmO, dt, 4, h.ep.out, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(out) failed with %d", a.name.c_str(), (int)r);
    } else {
        h.tmO = h.tmA;  // never used by the head variant; keep the descriptor valid for the prefetch
    }
    // constant-bank copies of the folded BatchNorm and the head (plan-build time only)
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(h.cscale, a.scale + a.ch_off, (size_t)BN * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(h.cshift, a.shift + a.ch_off, (size_t)BN * 4, cudaMemcpyDeviceToHost));
    if (a.head) {
        CK(cudaMemcpy(h.chead_w, a.head_w, 96 * 4, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(h.chead_b, a.head_b, 3 * 4, cudaMemcpyDeviceToHost));
    }
    const long long total = (long long)h.tiles_x * h.tiles_y * a.in.N;
    op.grid = (int)std::min<long long>(total, ctx->num_sms);
    op.fold = w.fold; op.m_tiles = (int)total; op.n_tiles = 1; op.patch_th = g.TH;
    op.flops = 2.0 * a.macs_per_pixel * (double)a.Wl * a.Hl * a.in.N;
    pl->ops.push_back(op);
    return W2L_OK;
}

static int make_conv_op(w2l_ctx* ctx, Plan* pl, const ConvArgs& a) {
    if (!get_encode_fn()) return fail(W2L_ENODEV, "cuTensorMapEncodeTiled is not available (no CUDA driver?)");
    const PackedW& w = *a.w;
    if (a.in.C != w.cin_pad) return fail(W2L_EINVAL, "%s: input view has %d channels, weights packed for %d", a.name.c_str(), a.in.C, w.cin_pad);
    if (a.cout % 16 != 0) return fail(W2L_EINVAL, "%s: cout %d not a multiple of 16", a.name.c_str(), a.cout);
    PatchGeom geom;
    if (patch_eligible(ctx, a, &geom)) return make_patch_op(ctx, pl, a, geom);
    Op op;
    op.type = OP_CONV;
    op.name = a.name + (w.fold ? " [fold]" : "");
    const int BK = pick_bk(w.cin_pad);
    int bw, bh, bn;
    pick_box(a.Wl, a.Hl, a.in.N, a.sx, a.sy, &bw, &bh, &bn);
    int tiles_x = (a.Wl + bw - 1) / bw, tiles_y = (a.Hl + bh - 1) / bh, tiles_n = (a.in.N + bn - 1) / bn;
    int m_tiles = tiles_x * tiles_y * tiles_n;
    int BN = 16;
    for (int cand : {128, 64, 32, 16})
        if (a.cout % cand == 0) { BN = cand; break; }
    if (a.head) BN = 32;
    else
        while (BN > 32 && m_tiles * (a.cout / BN) < ctx->num_sms && a.cout % (BN / 2) == 0) BN /= 2;
    // Channel-major form (conv_igemm.cuh, kCM): 128 output channels x a box of kCmPixels pixels per tile, both consumer
    // warpgroups on every tile, so no epilogue hides behind the other warpgroup's MMAs.  Taken for 16-bit staged outputs
    // with unit pixel strides (the interleaved phase stores of transposed convs did not gain) when a tile has at least
    // kCmMinSteps K steps and a CTA at least kCmMinCtaSteps, and the tiles fill the persistent grid's rounds nearly as
    // well as 128 x 128 row-major tiles: fill = useful pixels x channels over rounds x SMs x tile size.
    const int k_steps = w.ntaps * (w.cin_pad / BK);
    if (ctx->use_tma_epi && !ctx->x2 && !a.head && !a.out.f32 && a.cout % 128 == 0 && w.cout_pad % 128 == 0 && BK == 64 &&
        a.osx == 1 && a.osy == 1 && k_steps >= kCmMinSteps) {
        int cw, ch, cn;
        pick_box(a.Wl, a.Hl, a.in.N, a.sx, a.sy, &cw, &ch, &cn, kCmPixels);
        const long long cm_tiles = (long long)((a.Wl + cw - 1) / cw) * ((a.Hl + ch - 1) / ch) * ((a.in.N + cn - 1) / cn);
        const int S = ctx->num_sms, nt = a.cout / 128;
        auto fill = [&](long long tiles, int pixels) {
            const long long rounds = (tiles * nt + S - 1) / S;
            return (double)a.Wl * a.Hl * a.in.N / ((double)rounds * S * pixels / nt);
        };
        if ((cm_tiles * nt + S - 1) / S * k_steps >= kCmMinCtaSteps &&
            fill(cm_tiles, kCmPixels) >= (1.0 - kCmFillMargin) * fill(m_tiles, kTileM)) {
            op.cm = true;
            op.name += " [cm]";
            BN = 128;
            bw = cw; bh = ch; bn = cn;
            tiles_x = (a.Wl + bw - 1) / bw; tiles_y = (a.Hl + bh - 1) / bh; tiles_n = (a.in.N + bn - 1) / bn;
            m_tiles = tiles_x * tiles_y * tiles_n;
        }
    }
    if (w.cout_pad % BN != 0) return fail(W2L_EINVAL, "%s: cout_pad %d vs BN %d", a.name.c_str(), w.cout_pad, BN);
    op.BN = BN; op.BK = BK; op.head = a.head;
    // two M tiles per CTA (shared weight slab, one consumer warpgroup each) once there is plenty of work
    const int n_tiles_ = a.cout / BN;
    if (ctx->use_mt2 && !a.head && !op.cm && find_conv_kernel(BN, BK, ctx->bf16, false, 2) &&
        (long long)((m_tiles + 1) / 2) * n_tiles_ >= 2LL * ctx->num_sms)
        op.MT = 2;
    if (op.MT == 2) op.name += " [2M]";

    ConvParams& p = op.cp;
    memset(&p, 0, sizeof(p));
    CKR(encode_act_map(ctx, &p.tmA, a.in, BK, bw * a.sx, bh * a.sy, bn, a.sx, a.sy, a.name.c_str()));
    CKR(encode_w_map(ctx, &p.tmB, w, BK, BN, a.name.c_str()));
    p.tiles_x = tiles_x; p.tiles_y = tiles_y; p.tiles_n = tiles_n; p.n_tiles = a.cout / BN;
    p.bw = bw; p.bh = bh; p.bn = bn;
    p.sx = a.sx; p.sy = a.sy;
    p.ntaps = w.ntaps; p.kc_per_tap = w.cin_pad / BK;
    p.stage_tx_bytes = (unsigned)(op.MT * bw * bh * bn * BK * 2 + BN * BK * 2);
    fill_epi(&p.ep, a);
    // staged epilogue (TMA residual load + TMA store) for 16-bit outputs; the head / fp32 outputs keep direct stores
    p.tma_epi = 0;
    if (ctx->use_tma_epi && !ctx->x2 && !a.head && !a.out.f32) {
        EncodeTiledFn enc = get_encode_fn();
        const int EW = BN < 64 ? BN : 64;
        const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
        const CUtensorMapSwizzle esw = EW == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : EW == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
        // the channel extent is the destination view's: a launch may compute more (zero) channels than it stores (dgrad of
        // the 80-channel output block runs as one 128-wide tile), the TMA store clips them
        cuuint64_t dims[4] = {(cuuint64_t)std::min(a.cout, a.out.C), (cuuint64_t)a.Wl, (cuuint64_t)a.Hl, (cuuint64_t)a.in.N};
        cuuint32_t box[4] = {(cuuint32_t)EW, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
        cuuint32_t es[4] = {1, 1, 1, 1};
        cuuint64_t os[3] = {(cuuint64_t)p.ep.out_sx * 2, (cuuint64_t)p.ep.out_sy * 2, (cuuint64_t)p.ep.out_sn * 2};
        CUresult r = enc(&p.tmO, dt, 4, p.ep.out, dims, os, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, esw,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(out) failed with %d", a.name.c_str(), (int)r);
        if (a.res) {
            cuuint64_t rs[3] = {(cuuint64_t)p.ep.res_sx * 2, (cuuint64_t)p.ep.res_sy * 2, (cuuint64_t)p.ep.res_sn * 2};
            r = enc(&p.tmR, dt, 4, const_cast<void*>(p.ep.res), dims, rs, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, esw,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(res) failed with %d", a.name.c_str(), (int)r);
        } else {
            p.tmR = p.tmO;
        }
        p.tma_epi = 1;
        p.epi_box_bytes = (unsigned)(bw * bh * bn * EW * 2);
    }
    if (w.ntaps > kMaxTaps) return fail(W2L_EINVAL, "%s: too many taps", a.name.c_str());
    if (a.cout > a.out.C && !p.tma_epi && !a.head) return fail(W2L_ESTATE, "%s: %d computed channels for a %d-channel destination need the TMA-store epilogue", a.name.c_str(), a.cout, a.out.C);
    if (ctx->x2) {
        // split operands: x*w ~= x_hi*w_hi + x_lo*w_hi + x_hi*w_lo (the dropped x_lo*w_lo term is ~2^-22 relative)
        if (a.in.lo_off <= 0 || w.nslabs != 2 * w.ntaps) return fail(W2L_ESTATE, "%s: split-operand mode needs hi/lo planes", a.name.c_str());
        int k = 0;
        for (int t = 0; t < w.ntaps; ++t)
            for (int v = 0; v < 3; ++v, ++k) {
                p.dx[k] = w.dx[t]; p.dy[k] = w.dy[t];
                p.a_lo[k] = (v == 1) ? 1 : 0;
                p.b_slab[k] = (unsigned char)((v == 2) ? w.ntaps + t : t);
            }
        p.ntaps = 3 * w.ntaps;
        p.a_lo_off = a.in.lo_off;
    } else {
        for (int t = 0; t < w.ntaps; ++t) { p.dx[t] = w.dx[t]; p.dy[t] = w.dy[t]; p.a_lo[t] = 0; p.b_slab[t] = (unsigned char)t; }
    }
    const int total = ((m_tiles + op.MT - 1) / op.MT) * p.n_tiles;
    op.grid = std::min(total, ctx->num_sms);
    op.fold = w.fold; op.m_tiles = m_tiles; op.n_tiles = p.n_tiles;
    op.flops = 2.0 * a.macs_per_pixel * (double)a.Wl * a.Hl * a.in.N;
    pl->ops.push_back(op);
    return W2L_OK;
}

// Conv2dTranspose k3 s2 p1 op1 with 64 output channels: all four phases in one launch (convt_fused.cuh)
static int make_convt_fused_op(w2l_ctx* ctx, Plan* pl, const Layer& L, const LayerW& lw, const Act& in, const Act& out, int act = ACT_RELU) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return fail(W2L_ENODEV, "cuTensorMapEncodeTiled is not available");
    const PackedW& w = lw.ph.back();  // all 9 taps, grouped by input shift (load_layer)
    Op op;
    op.type = OP_CONV;
    op.name = L.name + " [fused 4-phase]";
    op.ctf = true;
    // K steps of 32 channels whatever cin is: one 64-channel stage (patch + nine 64x64 weight slabs, 94 KB) would not
    // double-buffer in shared memory
    const int BK = 32;
    if (w.cin_pad % BK != 0) return fail(W2L_EINVAL, "%s: fused convT needs cin %% 32 == 0", L.name.c_str());
    op.BK = BK; op.BN = kCtBN;
    ConvTParams& t = op.tp;
    memset(&t, 0, sizeof(t));
    CKR(encode_act_map(ctx, &t.tmA, in, BK, kCtPW, kCtPH, 1, 1, 1, L.name.c_str()));
    {
        const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
        const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_64B;  // 64-byte (BK = 32) rows
        cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad, (cuuint64_t)w.cout_pad, 9};
        cuuint64_t strides[2] = {(cuuint64_t)w.cin_pad * 2, (cuuint64_t)w.cin_pad * w.cout_pad * 2};
        cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)kCtBN, 9};
        cuuint32_t es[3] = {1, 1, 1};
        CUresult r = enc(&t.tmB, dt, 3, w.w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(B9) failed with %d", L.name.c_str(), (int)r);
        for (int py = 0; py < 2; ++py)
            for (int px = 0; px < 2; ++px) {
                uint16_t* base = out.base + ((long long)py * out.W + px) * out.Cs + out.c_off;
                cuuint64_t od[4] = {(cuuint64_t)kCtBN, (cuuint64_t)in.W, (cuuint64_t)in.H, (cuuint64_t)in.N};
                cuuint64_t os[3] = {(cuuint64_t)2 * out.Cs * 2, (cuuint64_t)2 * out.W * out.Cs * 2, (cuuint64_t)out.H * out.W * out.Cs * 2};
                cuuint32_t ob[4] = {(cuuint32_t)kCtBN, 8, 16, 1};
                cuuint32_t oe[4] = {1, 1, 1, 1};
                CUresult r2 = enc(&t.tmO[py * 2 + px], dt, 4, base, od, os, ob, oe, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
                if (r2 != CUDA_SUCCESS) return fail(W2L_ECUDA, "%s: cuTensorMapEncodeTiled(out phase) failed with %d", L.name.c_str(), (int)r2);
            }
    }
    t.tiles_x = (in.W + 7) / 8; t.tiles_y = (in.H + 15) / 16; t.N = in.N;
    t.kc = w.cin_pad / BK;
    t.patch_bytes = kCtPW * kCtPH * BK * 2;
    t.patch_stride = (t.patch_bytes + 1023) / 1024 * 1024;
    const int stage_bytes = t.patch_stride + 9 * kCtBN * BK * 2;
    const int fixed = 2 * kTileM * kCtBN * 2 + kSmemExtra;  // two staging tiles, alignment slack + barriers
    t.stages = std::min(kCtMaxStages, (kCtSmemMax - fixed) / stage_bytes);
    if (t.stages < 2) return fail(W2L_EINVAL, "%s: fused convT does not fit shared memory", L.name.c_str());
    op.dyn_smem = t.stages * stage_bytes + fixed;
    t.act = act;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(t.cscale, lw.scale, kCtBN * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(t.cshift, lw.shift, kCtBN * 4, cudaMemcpyDeviceToHost));
    const long long units = (long long)t.tiles_x * t.tiles_y * in.N;
    op.grid = (int)std::min<long long>(units, ctx->num_sms);
    op.m_tiles = (int)units; op.n_tiles = 1;
    op.flops = 2.0 * (double)L.cin * L.cout * 9 * (double)in.W * in.H * in.N;
    pl->ops.push_back(op);
    return W2L_OK;
}

// Emit the launches of one block (conv / convT) of a spec table.
// act_override >= 0 replaces the block kind's activation (training: the conv stores the pre-BatchNorm output; dgrad: none).
static int emit_block(w2l_ctx* ctx, Plan* pl, const NetW& nw, int li, const Layer& L, const Act& in, const Act& out,
                      const Act* res, bool head = false, int head_B = 1, int head_T = 1, int act_override = -1) {
    const LayerW& lw = nw.layers[li];
    ConvArgs a;
    a.in = in; a.out = out; a.res = res;
    a.scale = lw.scale; a.shift = lw.shift;
    a.act = (L.kind == W2L_BLOCK_CONV_LRELU) ? ACT_LRELU : (L.kind == W2L_BLOCK_CONV_PLAIN ? ACT_NONE : ACT_RELU);
    if (act_override >= 0) a.act = act_override;
    a.cout = L.cout;
    a.head = head; a.head_w = nw.head_w; a.head_b = nw.head_b; a.head_B = head_B; a.head_T = head_T;
    if (L.kind != W2L_BLOCK_CONVT_BN_RELU) {
        a.name = L.name;
        a.w = &lw.ph[0];
        a.sx = lw.ph[0].fold ? 1 : L.sw; a.sy = L.sh;  // folded first layers: the tensor map already strides the windows
        a.Hl = out.H; a.Wl = out.W;
        a.macs_per_pixel = (double)L.cin * L.cout * L.kh * L.kw;
        return make_conv_op(ctx, pl, a);
    }
    if (lw.gemm_convT) {
        // 1x1 -> kh x kw transposed conv == GEMM with kh*kw*cout output columns landing NHWC-contiguous
        Act o = out;
        o.H = 1; o.W = 1; o.Cs = out.Cs * out.H * out.W; o.C = L.cout * L.kh * L.kw;
        if (out.c_off != 0 || out.C != out.Cs) return fail(W2L_EINVAL, "%s: gemm convT needs a dense output", L.name.c_str());
        a.name = L.name;
        a.out = o;
        a.w = &lw.ph[0];
        a.Hl = 1; a.Wl = 1;
        a.cout = L.cout * L.kh * L.kw;
        a.macs_per_pixel = (double)L.cin * L.cout * L.kh * L.kw;
        return make_conv_op(ctx, pl, a);
    }
    // the fused kernel steps K by 32 channels (g_ct_kernels): a cin that is not a multiple of 32 (16, 48, 80, ...) takes
    // the four phase launches
    if (lw.has_all_taps && ctx->use_ctfused && lw.ph.back().cin_pad % 32 == 0 && in.W >= 8 && in.H >= 8 && !res &&
        out.H == 2 * in.H && out.W == 2 * in.W &&
        (double)in.W * in.H / ((double)((in.W + 7) / 8) * ((in.H + 15) / 16) * kTileM) >= 0.6 && !out.f32)
        return make_convt_fused_op(ctx, pl, L, lw, in, out, a.act);
    const size_t nph = lw.ph.size() - (lw.has_all_taps ? 1 : 0);
    for (size_t i = 0; i < nph; ++i) {
        const PackedW& w = lw.ph[i];
        ConvArgs b = a;
        b.name = L.name + ".ph" + std::to_string(w.py) + std::to_string(w.px);
        b.w = &w;
        b.osy = L.sh; b.osx = L.sw; b.phy = w.py; b.phx = w.px;
        b.Hl = (out.H - w.py + L.sh - 1) / L.sh;
        b.Wl = (out.W - w.px + L.sw - 1) / L.sw;
        b.macs_per_pixel = (double)L.cin * L.cout * w.ntaps;
        CKR(make_conv_op(ctx, pl, b));
    }
    return W2L_OK;
}

static void conv_out_dims(const Layer& L, int H, int W, int* Ho, int* Wo) {
    if (L.kind == W2L_BLOCK_CONVT_BN_RELU) {
        *Ho = (H - 1) * L.sh - 2 * L.ph + L.kh + L.out_pad;
        *Wo = (W - 1) * L.sw - 2 * L.pw + L.kw + L.out_pad;
    } else {
        *Ho = (H + 2 * L.ph - L.kh) / L.sh + 1;
        *Wo = (W + 2 * L.pw - L.kw) / L.sw + 1;
    }
}
