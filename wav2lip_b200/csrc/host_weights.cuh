// host_weights.cuh — w2l_load_weights' back end: re-packing the reference's fp32 tensors into 16-bit K-major tap slabs
// (plain, K-folded, per transposed-conv phase, grouped for the fused kernel) and folding BatchNorm into scale/shift.
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// weights
// ------------------------------------------------------------------------------------------------
struct TensorRef { const float* p; int64_t n; };
typedef std::map<std::string, TensorRef> TensorMap;

static int need(const TensorMap& tm, const std::string& name, int64_t numel, const float** out) {
    auto it = tm.find(name);
    if (it == tm.end()) return fail(W2L_EINVAL, "missing tensor '%s'", name.c_str());
    if (it->second.n != numel) return fail(W2L_EINVAL, "tensor '%s' has %lld elements, expected %lld", name.c_str(), (long long)it->second.n, (long long)numel);
    *out = it->second.p;
    return W2L_OK;
}

// The slabs go to lw's memory.  log != nullptr (training): the job is also recorded there, to be replayed after every
// optimizer step
static int pack_taps(w2l_ctx* ctx, LayerW* lw, PackedW* pw, const float* src, int cout, int cin, int kh, int kw, bool transposed,
                     const std::vector<std::pair<int, int>>& rs, int cout_pad_to, RepackLog* log, cudaStream_t st,
                     uint16_t* dst_override = nullptr) {
    PackParams pp;
    memset(&pp, 0, sizeof(pp));
    pp.src = src;
    pp.ntaps = (int)rs.size();
    pp.cout = cout; pp.cin = cin;
    pp.cin_pad = round_up(cin, 16);
    pp.cout_pad = round_up(cout, cout_pad_to);
    if (transposed) { pp.s_ci = (long long)cout * kh * kw; pp.s_co = (long long)kh * kw; }
    else { pp.s_co = (long long)cin * kh * kw; pp.s_ci = (long long)kh * kw; }
    pp.s_r = kw; pp.s_s = 1;
    for (size_t t = 0; t < rs.size(); ++t) { pp.r[t] = (signed char)rs[t].first; pp.s[t] = (signed char)rs[t].second; }
    const size_t n = (size_t)pp.ntaps * pp.cout_pad * pp.cin_pad;
    const int planes = (ctx->x2 && !dst_override) ? 2 : 1;
    if (dst_override) pp.dst = dst_override;
    else {
        CKR(alloc_in(ctx, &lw->mem, &pp.dst, n * 2 * planes));
        pw->w = pp.dst;
        pw->ntaps = pp.ntaps; pw->cout_pad = pp.cout_pad; pw->cin_pad = pp.cin_pad;
        pw->nslabs = pp.ntaps * planes;
    }
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
    if (log) log->pack.push_back(pp);
    for (int pl_ = 0; pl_ < planes; ++pl_) {  // hi slabs, then (split-operand mode) the lo slabs w - fp16(w)
        pp.lo = pl_;
        if (ctx->bf16) pack_w_kernel<true><<<blocks, 256, 0, st>>>(pp);
        else pack_w_kernel<false><<<blocks, 256, 0, st>>>(pp);
        ctx->launches++;
        pp.dst += n;
    }
    CK(cudaGetLastError());
    return W2L_OK;
}

// Pack one block's parameters. in_hw1: the block is applied to a 1x1 input (enables the GEMM form of convT).
//   fold: the block may read a K-folded input (first layers fed by the ingest kernel);  log: see pack_taps
static int load_layer(w2l_ctx* ctx, LayerW* lw, const Layer& L, const float* W, const float* bias, const float* gamma,
                      const float* beta, const float* mean, const float* var, bool in_hw1, bool fold, RepackLog* log,
                      cudaStream_t st) {
    *lw = LayerW();
    const int pad_to = 16;
    int reps = 1;
    if (fold && L.kind != W2L_BLOCK_CONVT_BN_RELU && L.cin <= 16 && L.kw >= 3 && (L.sw == 1 || L.sw == 2)) {
        // tiny-Cin first layer: fold the kw horizontal taps into K (one K row per filter row r)
        PackedW pw;
        pw.fold = true;
        pw.Cp = L.cin <= 8 ? 8 : 16;
        const int raw = L.kw * pw.Cp;
        pw.kfold = raw <= 32 ? 32 : round_up(raw, 64);
        pw.win = pw.kfold / pw.Cp;
        pw.ntaps = L.kh; pw.cin_pad = pw.kfold; pw.cout_pad = round_up(L.cout, pad_to);
        for (int r = 0; r < L.kh; ++r) { pw.dy.push_back((signed char)(r - L.ph)); pw.dx.push_back(0); }
        const size_t n = (size_t)pw.ntaps * pw.cout_pad * pw.kfold;
        CKR(alloc_in(ctx, &lw->mem, &pw.w, n * 2));
        PackFoldParams fp;
        fp.src = W; fp.dst = pw.w; fp.kh = L.kh; fp.kw = L.kw; fp.cout = L.cout; fp.cin = L.cin;
        fp.cout_pad = pw.cout_pad; fp.kfold = pw.kfold; fp.Cp = pw.Cp;
        const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
        if (log) log->pack_fold.push_back(fp);
        if (ctx->bf16) pack_fold_kernel<true><<<blocks, 256, 0, st>>>(fp);
        else pack_fold_kernel<false><<<blocks, 256, 0, st>>>(fp);
        ctx->launches++;
        CK(cudaGetLastError());
        lw->ph.push_back(pw);
    } else if (L.kind != W2L_BLOCK_CONVT_BN_RELU) {
        std::vector<std::pair<int, int>> rs;
        PackedW pw;
        for (int r = 0; r < L.kh; ++r)
            for (int s = 0; s < L.kw; ++s) { rs.push_back({r, s}); pw.dy.push_back((signed char)(r - L.ph)); pw.dx.push_back((signed char)(s - L.pw)); }
        CKR(pack_taps(ctx, lw, &pw, W, L.cout_real > 0 ? L.cout_real : L.cout, L.cin, L.kh, L.kw, false, rs, pad_to, log, st));
        lw->ph.push_back(pw);
    } else if (in_hw1 && !ctx->x2 && L.sh == 1 && L.sw == 1 && L.ph == 0 && L.pw == 0) {
        // out[n, y, x, co] = sum_ci in[n, ci] * W[ci, co, y, x]  -> GEMM with columns (y, x, co)
        lw->gemm_convT = true;
        reps = L.kh * L.kw;
        PackedW pw;
        pw.ntaps = 1; pw.cin_pad = round_up(L.cin, 16); pw.cout_pad = round_up(L.cout, pad_to) * reps;
        pw.dx.push_back(0); pw.dy.push_back(0);
        CKR(alloc_in(ctx, &lw->mem, &pw.w, (size_t)pw.cout_pad * pw.cin_pad * 2));
        if (L.cout % pad_to != 0) return fail(W2L_EINVAL, "%s: gemm convT needs cout %% 16 == 0", L.name.c_str());
        for (int r = 0; r < L.kh; ++r)
            for (int s = 0; s < L.kw; ++s) {
                std::vector<std::pair<int, int>> rs = {{r, s}};
                CKR(pack_taps(ctx, lw, nullptr, W, L.cout, L.cin, L.kh, L.kw, true, rs, pad_to, log, st,
                              pw.w + (size_t)(r * L.kw + s) * L.cout * pw.cin_pad));
            }
        lw->ph.push_back(pw);
    } else {
        // transposed conv: oy = iy*s - p + r.  Output phase py uses the taps r == (py + p) mod s at input row y + (py + p - r)/s
        for (int py = 0; py < L.sh; ++py)
            for (int px = 0; px < L.sw; ++px) {
                std::vector<std::pair<int, int>> rs;
                PackedW pw;
                pw.py = py; pw.px = px;
                for (int r = 0; r < L.kh; ++r) {
                    if ((py + L.ph - r) % L.sh != 0) continue;
                    for (int s = 0; s < L.kw; ++s) {
                        if ((px + L.pw - s) % L.sw != 0) continue;
                        rs.push_back({r, s});
                        pw.dy.push_back((signed char)((py + L.ph - r) / L.sh));
                        pw.dx.push_back((signed char)((px + L.pw - s) / L.sw));
                    }
                }
                if (rs.empty()) return fail(W2L_EINVAL, "%s: empty transposed-conv phase", L.name.c_str());
                CKR(pack_taps(ctx, lw, &pw, W, L.cout, L.cin, L.kh, L.kw, true, rs, pad_to, log, st));
                lw->ph.push_back(pw);
            }
        if (!ctx->x2 && L.cout == kCtBN && L.kh == 3 && L.kw == 3 && L.sh == 2 && L.sw == 2 && L.ph == 1 && L.pw == 1 && L.out_pad == 1) {
            // all nine taps for the fused four-phase kernel in the slab order of its two consumer warpgroups
            // (convt_fused.cuh): shift (0,0) for the accumulator's phase order [00 | 11 | 01 | 10] (each group's half one
            // contiguous 128-column window), then the other taps of group 0's phase 11, then those of group 1's phases
            // 01 and 10.  Tap (r,s) belongs to phase ((r+1)&1, (s+1)&1) and reads in[y + (r==0), x + (s==0)]
            std::vector<std::pair<int, int>> rs = {{1, 1}, {2, 2}, {1, 2}, {2, 1},   // shift (0,0): phases 00 11 01 10
                                                   {2, 0}, {0, 2}, {0, 0},           // phase 11: shifts (0,1) (1,0) (1,1)
                                                   {1, 0},                           // phase 01: shift (0,1)
                                                   {0, 1}};                          // phase 10: shift (1,0)
            PackedW pw;
            for (int t = 0; t < 9; ++t) { pw.dy.push_back(0); pw.dx.push_back(0); }
            CKR(pack_taps(ctx, lw, &pw, W, L.cout, L.cin, L.kh, L.kw, true, rs, pad_to, log, st));
            lw->ph.push_back(pw);
            lw->has_all_taps = true;
        }
    }
    const int n_pad = round_up(L.cout, pad_to) * reps;
    CKR(alloc_in(ctx, &lw->mem, &lw->scale, (size_t)n_pad * 4));
    CKR(alloc_in(ctx, &lw->mem, &lw->shift, (size_t)n_pad * 4));
    lw->n_scale = n_pad;
    fold_bn_kernel<<<(n_pad + 127) / 128, 128, 0, st>>>(bias, gamma, beta, mean, var, 1e-5f, L.cout_real > 0 ? L.cout_real : L.cout, reps, n_pad, lw->scale, lw->shift);
    if (log && bias) log->fold.push_back(FoldJob{bias, L.cout, reps, n_pad, lw->scale, lw->shift});
    ctx->launches++;
    CK(cudaGetLastError());
    lw->loaded = true;
    return W2L_OK;
}

static int fetch_block_tensors(const TensorMap& tm, const Layer& L, const float** W, const float** b, const float** g,
                               const float** be, const float** m, const float** v) {
    const int cout = L.cout_real > 0 ? L.cout_real : L.cout;
    const int64_t wn = (int64_t)L.cin * cout * L.kh * L.kw;
    CKR(need(tm, L.name + (L.bare_keys ? ".weight" : ".conv_block.0.weight"), wn, W));
    CKR(need(tm, L.name + (L.bare_keys ? ".bias" : ".conv_block.0.bias"), cout, b));
    *g = *be = *m = *v = nullptr;
    if (L.kind == W2L_BLOCK_CONV_BN_RELU || L.kind == W2L_BLOCK_CONVT_BN_RELU) {
        CKR(need(tm, L.name + ".conv_block.1.weight", L.cout, g));
        CKR(need(tm, L.name + ".conv_block.1.bias", L.cout, be));
        CKR(need(tm, L.name + ".conv_block.1.running_mean", L.cout, m));
        CKR(need(tm, L.name + ".conv_block.1.running_var", L.cout, v));
    }
    return W2L_OK;
}

static void drop_plans(w2l_ctx* ctx, int net) {
    for (auto it = ctx->plans.begin(); it != ctx->plans.end();) {
        if (it->second->net == net) it = ctx->plans.erase(it);
        else ++it;
    }
    ctx->last_plan[net] = nullptr;
    ctx->plan_epoch[net]++;
}
