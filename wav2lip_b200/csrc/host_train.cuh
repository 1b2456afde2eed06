// host_train.cuh — the training step behind wav2lip_train.py:210-231, color_syncnet_train.py:146-163 and
// hq_wav2lip_train.py:213-255 (SURVEY.md section 8 f1): train-mode plans of the three networks.
//
// A training plan keeps every block's input, pre-BatchNorm output z and output y (bf16 NHWC) and replays, per block,
//   forward : conv (the inference kernels, epilogue = identity)  ->  per-channel sum z / sum z^2  ->  batch statistics
//             (+ running-average update)  ->  y = relu(gamma * zhat + beta [+ x])
//   backward: du = dy * (y > 0), sums of du and du * zhat  ->  dgamma, dbeta, dz  ->  dgrad = the inference kernels on
//             re-packed weights (flipped taps / the transposed-conv phases / a strided conv: oracle/backward_recipe.py)
//             with the residual or skip gradient added in its epilogue  ->  wgrad = wgrad_kernel (pixels as K) + the
//             deterministic split-K reduction into the bound fp32 gradient tensor.
// Master parameters, BatchNorm buffers and gradients are caller-owned fp32 device tensors bound by name
// (w2l_train_bind); the 16-bit weight slabs are re-packed from them at the start of every training forward.
// Part of the single translation unit w2l_api.cu (included there, after host_plans.cuh).
#pragma once

struct ParamRef { float* value = nullptr; float* grad = nullptr; long long n = 0; };

enum WgForm { WG_PLAIN = 0, WG_STRIDED = 1, WG_TRANSPOSED = 2, WG_SWAP = 3, WG_FOLDED = 4 };   // = W2L_WG_*

struct WgradOp {
    bool on = false;
    int BN = 0;
    int form = WG_PLAIN;
    WgradParams wp;
    WgradReduceParams rp;
    int grid = 0, smem = 0;
    double flops = 0;
};

static bool starts_with(const std::string& s, const char* prefix) { return s.rfind(prefix, 0) == 0; }

struct TBlock {
    int li = 0;
    Layer L, Ld;                 // the block, and its input-gradient computation written as a block of the same table
    Act x, y, z;                 // input view, output view, pre-BatchNorm output (dense; BN blocks only)
    Act dy, dz, du;              // gradient of y (view), of z (dense), of the residual branch (dense, residual blocks)
    Act dx, dx_add;              // where the input gradient goes (base == nullptr: not needed) and what is added to it
    float* y_f32 = nullptr;      // optional fp32 copy of y (embeddings)
    bool bn = true;
    bool wgrad_only = false;     // backward of this block only serves parameter gradients (the expert's audio branch)
    int lane = 0;                // 1: audio-encoder block — independent of the face encoder, runs on the auxiliary stream beside it
    Act x_fold;                  // first blocks: the K-folded copy of the input the forward reads (base == nullptr: none)
    int fold_cp = 0;             // ... and its channel pitch: window element s*fold_cp + c = horizontal tap s, channel c
    float *stats = nullptr, *coef = nullptr, *partial = nullptr;
    int nblk = 0;
    long long M = 0;             // output pixels N*Ho*Wo
    size_t fwd0 = 0, fwd1 = 0, dg0 = 0, dg1 = 0;   // op ranges in the plan's op list
    WgradOp wg;
    // bound tensors
    float *W = nullptr, *b = nullptr, *gamma = nullptr, *beta = nullptr, *rmean = nullptr, *rvar = nullptr;
    float *gW = nullptr, *gb = nullptr, *ggamma = nullptr, *gbeta = nullptr;
};

struct TrainPlan {
    explicit TrainPlan(w2l_ctx* ctx) : pl(ctx) {}
    int net = 0, B = 0, T = 0, N = 0;
    Plan pl;                       // op storage + allocations
    NetW wf, wd;                   // forward / dgrad weight slabs (16-bit), repacked every step
    RepackLog repack;              // ... by these launches
    DevMem<PackParams> pack_dev; DevMem<int> pack_blk_job, pack_blk_first; int pack_blocks = 0;   // one-launch repack
    std::vector<TBlock> blocks;    // forward order
    std::vector<size_t> ingest;    // indices of the ingest ops
    // generator
    Act y32, dy32; float* head_partial = nullptr; int head_blocks = 0;
    const float* g_out = nullptr;  // caller's generator output of the last forward (the head backward re-reads it)
    // syncnet
    float *fe_raw = nullptr, *ae_raw = nullptr; Act dfe, dae; Act dface_in;
    const float *a_out = nullptr, *v_out = nullptr;
    // disc
    Act feat, dfeat, dframes_in; const float* prob_out = nullptr;
    // split-K workspace of the wgrads, one per lane: with the wgrad side stream off, each block's wgrad runs on its own
    // lane's stream, and the audio encoder's (auxiliary stream) run concurrently with the face encoder's (main stream)
    float* wg_ws[2] = {nullptr, nullptr}; size_t wg_ws_bytes[2] = {0, 0};
    bool input_grad = false;       // the first block's dgrad is part of the plan (expert / discriminator inside a generator step)
    double fwd_flops = 0;
};

// Adam moments of one net's bound tensors that have a gradient, in the order of the name map (alphabetical): names[i] owns
// host[i]; step is the count the bias correction uses (torch.optim.Adam's state['step'])
struct AdamSlot { std::vector<std::string> names; std::vector<DevMem<>> moments; std::vector<AdamTensor> host; DevMem<AdamTensor> dev; long long step = 0; };

// NCCL entry points resolved at run time from the libnccl.so.2 that torch already loaded (no link-time dependency)
typedef int (*NcclGetUniqueIdFn)(void*);
struct NcclId { char bytes[128]; };
typedef int (*NcclCommInitRankFn)(void**, int, NcclId, int);
typedef int (*NcclAllReduceFn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*NcclCommDestroyFn)(void*);
typedef const char* (*NcclGetErrorStringFn)(int);

struct TrainState {
    std::map<std::string, ParamRef> bound[3];
    bool is_bound[3] = {false, false, false};
    std::map<std::string, std::unique_ptr<TrainPlan>> plans;
    TrainPlan* last[3] = {nullptr, nullptr, nullptr};
    AdamSlot adam[3];
    // losses of the fused steps
    DevMem<float> loss_dev;        // [8]
    DevMem<float> a_emb, v_emb, da, dv;
    DevMem<float> g_buf, dg_buf;
    DevMem<float> prob, dprob;     // disc probabilities on g | gt (2N), their gradients (3N)
    // data-parallel gradient all-reduce
    void* nccl_lib = nullptr; void* comm = nullptr; int rank = 0, world = 1;
    NcclAllReduceFn all_reduce = nullptr; NcclCommDestroyFn comm_destroy = nullptr; NcclGetErrorStringFn err_string = nullptr;
    Stream s_comm; Event ev_bucket, ev_comm;
    double last_allreduce_bytes = 0;
    // the weight-gradient GEMMs are leaves of the backward graph: they run on a side stream beside the dgrad chain, so that
    // they fill the SMs the chain's partial rounds (and, at small batches, its latency-bound launches) leave idle
    Stream s_wg; Event ev_dz, ev_wg, ev_wgb;
    // the audio encoder (small, latency-bound launches) runs beside the face encoder, forward and backward
    Stream s_aux; Event ev_aux_fork, ev_aux_join;
    // the discriminator's step of the hq iteration (its two backward passes, all-reduce, Adam) beside the generator's backward
    Stream s_disc; Event ev_disc_fork, ev_disc_join;
    std::vector<w2l_train_block_info> last_block_info;   // the block of the last w2l_conv_block_train (its plan is freed)
    ~TrainState() { if (comm && comm_destroy) comm_destroy(comm); }   // before s_comm goes
};

static TrainState* train_state(w2l_ctx* ctx) {
    if (!ctx->train) ctx->train.reset(new TrainState());
    return ctx->train.get();
}

// ------------------------------------------------------------------------------------------------
// building blocks
// ------------------------------------------------------------------------------------------------
static int bound_ptr(TrainState* ts, int net, const std::string& name, long long numel, float** value, float** grad, bool required = true) {
    auto it = ts->bound[net].find(name);
    if (it == ts->bound[net].end()) {
        if (!required) { *value = nullptr; if (grad) *grad = nullptr; return W2L_OK; }
        return fail(W2L_ESTATE, "training: tensor '%s' is not bound (w2l_train_bind)", name.c_str());
    }
    if (it->second.n != numel) return fail(W2L_EINVAL, "training: tensor '%s' has %lld elements, expected %lld", name.c_str(), it->second.n, numel);
    *value = it->second.value;
    if (grad) *grad = it->second.grad;
    return W2L_OK;
}

// The input gradient of a block, written as a block of the same table (oracle/backward_recipe.py: conv_dgrad).
//   widen: the staged (TMA-store) epilogue is on, which can store fewer channels than a launch computes
static Layer dgrad_layer(const Layer& L, int Hin, int Win, int Ho, int Wo, bool widen) {
    Layer d = L;
    d.residual = false;
    d.cin = L.cout;
    d.cout = round_up(L.cin, 16);
    if (L.kind == W2L_BLOCK_CONVT_BN_RELU) {   // transposed conv  ->  strided conv with the same tensor read as (out=Cin_t, in=Cout_t)
        d.kind = W2L_BLOCK_CONV_PLAIN;
        d.out_pad = 0;
    } else if (L.sh == 1 && L.sw == 1) {       // stride-1 conv     ->  conv with flipped taps, pad k-1-p
        d.kind = W2L_BLOCK_CONV_PLAIN;
        d.ph = L.kh - 1 - L.ph; d.pw = L.kw - 1 - L.pw;
        // 80 input channels (the output block) would tile as 5 x 16 output channels, each pass re-reading dz: compute 128
        // (48 zero rows) in one pass instead; the TMA store clips at the real channel count (the direct epilogue cannot:
        // with W2L_DISABLE_TMAEPI the plan keeps the real width)
        if (widen && d.cout > 64 && d.cout % 64 != 0 && d.cout < 128) d.cout = 128;
    } else {                                   // strided conv      ->  transposed conv with the SAME tensor
        d.kind = W2L_BLOCK_CONVT_BN_RELU;
        d.out_pad = Hin - ((Ho - 1) * L.sh - 2 * L.ph + L.kh);   // rows the forward's floor division dropped (per axis: emit uses out dims)
        (void)Win; (void)Wo;
    }
    return d;
}

// Pack the dgrad weights of block L from the master tensor W (fp32, the reference's layout).
static int load_dgrad_layer(w2l_ctx* ctx, LayerW* lw, const Layer& L, const Layer& Ld, const float* W, RepackLog* log, cudaStream_t st) {
    if (L.kind == W2L_BLOCK_CONVT_BN_RELU)     // (Cin_t, Cout_t, kh, kw) == conv layout (out, in, kh, kw): plain pack
        return load_layer(ctx, lw, Ld, W, nullptr, nullptr, nullptr, nullptr, nullptr, false, false, log, st);
    if (Ld.kind == W2L_BLOCK_CONVT_BN_RELU) {  // (Cout, Cin, kh, kw) == transposed-conv layout (in, out, kh, kw): phase packs
        Layer t = Ld;
        t.cout = L.cin;                        // real channel count of the source tensor (cout_pad rounds up)
        return load_layer(ctx, lw, t, W, nullptr, nullptr, nullptr, nullptr, nullptr, false, false, log, st);
    }
    // stride 1: dst[tap][ci][co] = W[co][ci][r][s], tap (r,s) reads dz at (y + ph - r, x + pw - s)
    // (Ld.cout may have been widened to a multiple of 128 — see dgrad_layer — the extra rows are zero and never stored)
    *lw = LayerW();
    std::vector<std::pair<int, int>> rs;
    PackedW pw;
    for (int r = 0; r < L.kh; ++r)
        for (int s = 0; s < L.kw; ++s) { rs.push_back({r, s}); pw.dy.push_back((signed char)(L.ph - r)); pw.dx.push_back((signed char)(L.pw - s)); }
    CKR(pack_taps(ctx, lw, &pw, W, L.cin, L.cout, L.kh, L.kw, true, rs, Ld.cout, log, st));
    lw->ph.push_back(pw);
    const int n_pad = Ld.cout;
    CKR(alloc_in(ctx, &lw->mem, &lw->scale, (size_t)n_pad * 4));
    CKR(alloc_in(ctx, &lw->mem, &lw->shift, (size_t)n_pad * 4));
    lw->n_scale = n_pad;
    fold_bn_kernel<<<(n_pad + 127) / 128, 128, 0, st>>>(nullptr, nullptr, nullptr, nullptr, nullptr, 1e-5f, n_pad, 1, n_pad, lw->scale, lw->shift);
    ctx->launches++;
    CK(cudaGetLastError());
    lw->loaded = true;
    return W2L_OK;
}

// K chunk of the wgrad: a (bw x bh x bn) box of the shared operand's pixel grid with P = bw*bh*bn a multiple of 16
static void pick_kbox(int W, int H, int N, int sx, int sy, int maxP, int* bw, int* bh, int* bn) {
    double best = 1e30;
    int b_w = 1, b_h = 1, b_n = 16;
    for (int w = 1; w <= std::min(W, maxP); ++w) {
        if (w * sx > 256) break;
        for (int h = 1; h <= std::min(H, maxP / w); ++h) {
            if (h * sy > 256) break;
            for (int n = 1; n <= 256 && w * h * n <= maxP; ++n) {
                const int P = w * h * n;
                if (P % 16 != 0) continue;
                const double rows = (double)((W + w - 1) / w) * ((H + h - 1) / h) * ((N + n - 1) / n) * P;
                const double cost = rows * (1.0 + 2.0 / P);   // fewer, larger chunks on ties (per-chunk overhead)
                if (cost < best) { best = cost; b_w = w; b_h = h; b_n = n; }
            }
        }
    }
    *bw = b_w; *bh = b_h; *bn = b_n;
}

typedef void (*WgKernelFn)(const WgradParams);
struct WgKernelEntry { int BN; WgKernelFn fn; uint64_t attr_set; };
static WgKernelEntry g_wg_kernels[] = {   // bf16 operands only: training refuses fp16 contexts (get_train_plan)
    {16, wgrad_kernel<16, true>, 0}, {32, wgrad_kernel<32, true>, 0}, {64, wgrad_kernel<64, true>, 0}, {128, wgrad_kernel<128, true>, 0},
};
constexpr int kWgSmemMax = 225 * 1024;

// ws_need[lane]: the largest split-K workspace of the lane's blocks
static int make_wgrad_op(w2l_ctx* ctx, TrainPlan* tp, TBlock* b, size_t* ws_need) {
    const Layer& L = b->L;
    const bool convT = L.kind == W2L_BLOCK_CONVT_BN_RELU;
    // A stride-1 conv is symmetric in its two tensors (sum over y,x of dz[y,x] x[y+d] == sum over y',x' of x[y',x'] dz[y'-d]):
    // when the input is wide and the output narrow (the 80 -> 32 output block) put x on the M side and dz, with all its taps
    // in one group, on the N side — one pass over the pixels instead of three
    const bool swap = !convT && L.sh == 1 && L.sw == 1 && L.cin > 64 && L.cout <= 64;
    // K-folded first layers (7x7 on 6 / 3 channels): the shifted operand is the forward's folded copy of the input, whose
    // 64-element window at pixel x holds the kw horizontal taps side by side — kh loads of 128-byte rows per pixel chunk
    // instead of kh*kw loads of 32-byte rows (the plain form was TMA-request-bound: 1.5 ms for 28 GFLOP)
    const bool folded = !convT && !swap && b->x_fold.base != nullptr && b->x_fold.C == 64 && L.sh == 1 && L.sw == 1 &&
                        L.kw * b->fold_cp <= 64;
    const Act& S = (convT || swap) ? b->x : b->dz;     // on the dense pixel grid of the sum
    const Act& Tt = folded ? b->x_fold : ((convT || swap) ? b->dz : b->x);    // read shifted / strided
    const int Cm = (convT || swap) ? L.cin : L.cout, Cn = folded ? 64 : ((convT || swap) ? L.cout : L.cin);
    WgradOp& w = b->wg;
    w.on = true;
    const int cn_pad = Tt.C;                 // channels of the view (first layers: padded to 16)
    int BN = cn_pad <= 16 ? 16 : cn_pad <= 32 ? 32 : cn_pad <= 64 ? 64 : 128;
    w.BN = BN;
    w.form = folded ? WG_FOLDED : swap ? WG_SWAP : convT ? WG_TRANSPOSED : (L.sh > 1 || L.sw > 1) ? WG_STRIDED : WG_PLAIN;
    WgradParams& p = w.wp;
    memset(&p, 0, sizeof(p));
    p.ntaps = folded ? L.kh : L.kh * L.kw;
    if (p.ntaps > kWgMaxTaps) return fail(W2L_EINVAL, "%s: too many taps for wgrad", L.name.c_str());
    const int max_tg = kWgMaxCols / BN;
    p.ngroups = (p.ntaps + max_tg - 1) / max_tg;
    p.tg = (p.ntaps + p.ngroups - 1) / p.ngroups;
    p.ngroups = (p.ntaps + p.tg - 1) / p.tg;
    if (folded) {
        for (int r = 0; r < L.kh; ++r) { p.dy[r] = (signed char)(r - L.ph); p.dx[r] = 0; }   // the window already starts at the leftmost tap
    } else {
        for (int r = 0; r < L.kh; ++r)
            for (int s = 0; s < L.kw; ++s) {
                p.dy[r * L.kw + s] = (signed char)(swap ? L.ph - r : r - L.ph);
                p.dx[r * L.kw + s] = (signed char)(swap ? L.pw - s : s - L.pw);
            }
    }
    p.sx = L.sw; p.sy = L.sh;
    // pixels per chunk: at least three pipeline stages must fit
    int maxP = (kWgSmemMax - xbuf_bytes<16>()) / 3 / (256 + p.tg * BN * 2) / 16 * 16;
    maxP = std::max(16, std::min(128, maxP));
    pick_kbox(S.W, S.H, S.N, p.sx, p.sy, maxP, &p.bw, &p.bh, &p.bn);
    p.P = p.bw * p.bh * p.bn;
    p.tiles_x = (S.W + p.bw - 1) / p.bw; p.tiles_y = (S.H + p.bh - 1) / p.bh; p.tiles_n = (S.N + p.bn - 1) / p.bn;
    p.chunks = (long long)p.tiles_x * p.tiles_y * p.tiles_n;
    p.m_tiles = (S.C + 127) / 128;
    p.n_tiles = (cn_pad + BN - 1) / BN;
    p.a_bytes = (unsigned)(2 * p.P * 128);
    p.tap_bytes = (unsigned)(p.P * BN * 2);
    p.stage_bytes = (p.a_bytes + p.tg * p.tap_bytes + 1023u) / 1024u * 1024u;
    p.stages = std::min(8, (int)((kWgSmemMax - xbuf_bytes<16>()) / p.stage_bytes));
    if (p.stages < 2) return fail(W2L_EINVAL, "%s: wgrad stage of %u bytes does not pipeline", L.name.c_str(), p.stage_bytes);
    w.smem = p.stages * p.stage_bytes + xbuf_bytes<16>() + 2048;
    // split K so that about two waves of units exist, each with enough chunks to amortise the pipeline fill
    const long long base_units = (long long)p.m_tiles * p.n_tiles * p.ngroups;
    // (rounded DOWN: units are dealt round-robin to one persistent CTA per SM, so 2 * SMs + 1 units would cost three rounds)
    long long splits = (2LL * ctx->num_sms) / base_units;
    splits = std::max(1LL, std::min(splits, std::max(1LL, p.chunks / 8)));
    splits = std::min(splits, 256LL);
    p.splits = (int)splits;
    CKR(encode_act_map(ctx, &p.tmS, S, 64, p.bw, p.bh, p.bn, 1, 1, L.name.c_str()));
    CKR(encode_act_map(ctx, &p.tmT, Tt, std::min(BN, 64), p.bw * p.sx, p.bh * p.sy, p.bn, p.sx, p.sy, L.name.c_str()));
    const long long Mp = (long long)p.m_tiles * 128, Np = (long long)p.n_tiles * BN;
    ws_need[b->lane] = std::max<size_t>(ws_need[b->lane], (size_t)((long long)p.splits * p.ntaps * Mp * Np * 4));
    w.grid = (int)std::min<long long>(base_units * p.splits, ctx->num_sms);
    WgradReduceParams& r = w.rp;
    r.ws = nullptr; r.out = b->gW; r.splits = p.splits; r.ntaps = p.ntaps; r.Cm = Cm; r.Cn = Cn; r.Mp = Mp; r.Np = Np; r.accumulate = 0;
    r.transpose = swap ? 1 : 0;
    r.fold_kw = folded ? L.kw : 0; r.fold_cp = folded ? b->fold_cp : 0; r.fold_cin = folded ? L.cin : 0;
    w.flops = 2.0 * (double)L.cin * L.cout * L.kh * L.kw * (double)S.N * S.H * S.W;
    return W2L_OK;
}

static int launch_wgrad(w2l_ctx* ctx, TrainPlan* tp, TBlock& b, bool accumulate, cudaStream_t st, bool pdl = true) {
    WgKernelEntry* e = nullptr;
    for (auto& k : g_wg_kernels) if (k.BN == b.wg.BN) e = &k;
    if (!e) return fail(W2L_EINVAL, "no wgrad kernel for BN=%d", b.wg.BN);
    CKR(ensure_smem_attr(&e->attr_set, ctx->device, (const void*)e->fn, kWgSmemMax + 2048));
    b.wg.wp.ws = tp->wg_ws[b.lane];
    CK(launch_k(e->fn, b.wg.grid, kWgThreads, (size_t)b.wg.smem, st, b.wg.wp, pdl && ctx->use_pdl));
    WgradReduceParams rp = b.wg.rp;
    rp.ws = tp->wg_ws[b.lane]; rp.out = b.gW; rp.accumulate = accumulate ? 1 : 0;
    const int n_tiles64 = (rp.Cn + 63) / 64;
    wgrad_reduce_kernel<<<dim3((unsigned)n_tiles64, (unsigned)rp.Cm), 256, (size_t)64 * (rp.ntaps + 1) * 4, st>>>(rp);
    ctx->launches += 2;
    return W2L_OK;
}

// dense 16-bit activation owned by the plan
static int tp_act(TrainPlan* tp, Act* a, int N, int H, int W, int C) { return plan_act(&tp->pl, a, N, H, W, C); }

static void add_train_ingest(TrainPlan* tp, const char* name, const IngestSpec& s, const Act& dst) {
    add_ingest(&tp->pl, name, s, dst);
    tp->ingest.push_back(tp->pl.ops.size() - 1);
}

// Add one block to a training plan: forward launches, statistics buffers, dgrad launches, wgrad.
//   x / y: input and output views;   dy: gradient view of y;   dx: where the input gradient goes (base nullptr: none);
//   dx_add: extra gradient added to dx (skip half of a concat gradient), base nullptr: none.
//   fold_in: the caller tensor x is ingested from (first blocks). Without an input gradient, the forward conv may then read
//   a second, K-folded copy of it (the inference plan's first-layer layout, 10-20x faster on the 7x7 / 6-channel layer)
//   written by one more ingest launch; the backward (wgrad) reads the plain NHWC copy.
static int add_train_block(w2l_ctx* ctx, TrainPlan* tp, int net, int li, const Layer& L, const Act& x, const Act& y, const Act& dy,
                           const Act& dx, const Act& dx_add, bool want_wgrad, bool in_hw1, size_t* ws_need, float* y_f32 = nullptr,
                           const IngestSpec* fold_in = nullptr) {
    TrainState* ts = train_state(ctx);
    TBlock b;
    b.li = li; b.L = L; b.x = x; b.y = y; b.dy = dy; b.dx = dx; b.dx_add = dx_add; b.y_f32 = y_f32;
    b.bn = (L.kind == W2L_BLOCK_CONV_BN_RELU || L.kind == W2L_BLOCK_CONVT_BN_RELU);
    b.M = (long long)y.N * y.H * y.W;
    const long long wn = (long long)L.cin * L.cout * L.kh * L.kw;
    CKR(bound_ptr(ts, net, L.name + ".conv_block.0.weight", wn, &b.W, &b.gW));
    CKR(bound_ptr(ts, net, L.name + ".conv_block.0.bias", L.cout, &b.b, &b.gb));
    if (b.bn) {
        CKR(bound_ptr(ts, net, L.name + ".conv_block.1.weight", L.cout, &b.gamma, &b.ggamma));
        CKR(bound_ptr(ts, net, L.name + ".conv_block.1.bias", L.cout, &b.beta, &b.gbeta));
        CKR(bound_ptr(ts, net, L.name + ".conv_block.1.running_mean", L.cout, &b.rmean, nullptr, false));
        CKR(bound_ptr(ts, net, L.name + ".conv_block.1.running_var", L.cout, &b.rvar, nullptr, false));
    }
    if (want_wgrad && !b.gW) want_wgrad = false;   // frozen / no gradient tensor bound
    cudaStream_t st = nullptr;
    // ---- forward weights + launches ----
    if ((int)tp->wf.layers.size() <= li) { tp->wf.layers.resize(li + 1); tp->wd.layers.resize(li + 1); }
    const bool fold = fold_in && ctx->use_fold && ctx->use_patch && !dx.base;
    CKR(load_layer(ctx, &tp->wf.layers[li], L, b.W, b.bn ? nullptr : b.b, nullptr, nullptr, nullptr, nullptr, in_hw1, fold,
                   &tp->repack, st));
    if (dx.base) {
        b.Ld = dgrad_layer(L, x.H, x.W, y.H, y.W, ctx->use_tma_epi);
        CKR(load_dgrad_layer(ctx, &tp->wd.layers[li], L, b.Ld, b.W, &tp->repack, st));
    }
    Act conv_out = y;
    if (b.bn) { CKR(tp_act(tp, &b.z, y.N, y.H, y.W, L.cout)); conv_out = b.z; }
    Act x_fwd = x;
    if (tp->wf.layers[li].ph[0].fold) {
        CKR(plan_input_act(&tp->pl, &x_fwd, x.N, x.H, x.W, L.cin, tp->wf.layers[li], L));
        add_train_ingest(tp, "ingest.fold", *fold_in, x_fwd);
        b.x_fold = x_fwd; b.fold_cp = tp->wf.layers[li].ph[0].Cp;
    }
    b.fwd0 = tp->pl.ops.size();
    CKR(emit_block(ctx, &tp->pl, tp->wf, li, L, x_fwd, conv_out, nullptr, false, 1, 1, b.bn ? ACT_NONE : -1));
    b.fwd1 = tp->pl.ops.size();
    for (size_t i = b.fwd0; i < b.fwd1; ++i) tp->fwd_flops += tp->pl.ops[i].flops;
    // ---- statistics / reduction buffers ----
    const int rows = kBnThreads / (L.cout / 8);
    b.nblk = (int)std::max<long long>(1, std::min<long long>((b.M + rows - 1) / rows, (long long)ctx->num_sms * 4));
    CKR(plan_alloc(&tp->pl, &b.partial, (size_t)b.nblk * 2 * L.cout * 4));
    CKR(plan_alloc(&tp->pl, &b.stats, (size_t)4 * L.cout * 4));   // mean, invstd, G, H
    CKR(plan_alloc(&tp->pl, &b.coef, (size_t)3 * L.cout * 4));
    // ---- backward ----
    CKR(tp_act(tp, &b.dz, y.N, y.H, y.W, L.cout));
    if (b.bn && L.residual) CKR(tp_act(tp, &b.du, y.N, y.H, y.W, L.cout));
    b.dg0 = b.dg1 = tp->pl.ops.size();
    if (dx.base) {
        const Act* add = nullptr;
        if (b.bn && L.residual) add = &b.du;
        if (dx_add.base) {
            if (add) return fail(W2L_ESTATE, "%s: residual block with a second gradient source", L.name.c_str());
            add = &b.dx_add;
        }
        // (b is copied into the plan below; emit_block bakes the pointers, not &b)
        Act add_copy;
        if (add) add_copy = *add;
        CKR(emit_block(ctx, &tp->pl, tp->wd, li, b.Ld, b.dz, dx, add ? &add_copy : nullptr, false, 1, 1, ACT_NONE));
        b.dg1 = tp->pl.ops.size();
    }
    b.lane = starts_with(L.name, "audio_encoder.") ? 1 : 0;
    if (want_wgrad) CKR(make_wgrad_op(ctx, tp, &b, ws_need));
    tp->blocks.push_back(b);
    return W2L_OK;
}

// the w2l_train_block_info row of one block (test aid)
static void train_block_info(const w2l_ctx* ctx, const TrainPlan* tp, const TBlock& b, w2l_train_block_info* o) {
    memset(o, 0, sizeof(*o));
    const Layer& L = b.L;
    snprintf(o->name, sizeof(o->name), "%s", L.name.c_str());
    o->layer = b.li;
    o->kind = L.kind; o->cin = L.cin; o->cout = L.cout; o->kh = L.kh; o->kw = L.kw; o->sh = L.sh; o->sw = L.sw;
    o->ph = L.ph; o->pw = L.pw; o->out_pad = L.out_pad; o->residual = L.residual ? 1 : 0;
    o->n = b.x.N; o->h_in = b.x.H; o->w_in = b.x.W; o->h_out = b.y.H; o->w_out = b.y.W;
    o->lane = b.lane;
    o->has_dx = b.dx.base ? 1 : 0; o->has_dx_add = b.dx_add.base ? 1 : 0; o->has_du = b.du.base ? 1 : 0;
    o->has_wgrad = b.wg.on ? 1 : 0;
    if (b.wg.on) {
        const WgradParams& p = b.wg.wp;
        o->wg_bn = b.wg.BN; o->wg_form = b.wg.form; o->wg_ntaps = p.ntaps; o->wg_tg = p.tg; o->wg_ngroups = p.ngroups;
        o->wg_p = p.P; o->wg_bw = p.bw; o->wg_bh = p.bh; o->wg_bnb = p.bn;
        o->wg_chunks = (int32_t)p.chunks; o->wg_m_tiles = p.m_tiles; o->wg_n_tiles = p.n_tiles; o->wg_splits = p.splits;
        o->wg_grid = b.wg.grid;
    }
    for (size_t i = b.fwd0; i < b.fwd1 && o->n_fwd < 4; ++i)
        if (tp->pl.ops[i].type == OP_CONV) op_kernel_info(ctx, tp->pl.ops[i], &o->fwd[o->n_fwd++]);
    for (size_t i = b.dg0; i < b.dg1 && o->n_dgrad < 4; ++i)
        if (tp->pl.ops[i].type == OP_CONV) op_kernel_info(ctx, tp->pl.ops[i], &o->dgrad[o->n_dgrad++]);
}

// a straight chain of blocks; value and gradient buffers of the intermediate tensors are dense and owned by the plan
//   x0 / dx0: input view and where its gradient goes (base nullptr: none); last / dlast: output view of the final block and
//   its gradient view (base nullptr: allocate dense ones, returned through out / dout)
static int add_train_chain(w2l_ctx* ctx, TrainPlan* tp, int net, const std::vector<Layer>& layers, const std::vector<int>& idx,
                           Act x0, Act dx0, Act dx0_add, const Act* last, const Act* dlast, bool want_wgrad, size_t* ws_need,
                           Act* out, Act* dout, float* last_f32 = nullptr, const IngestSpec* fold_in = nullptr) {
    // values and gradients of every block output first (the gradient view of y[k] is the dx of block k+1)
    std::vector<Act> ys(idx.size()), dys(idx.size());
    int H = x0.H, W = x0.W;
    for (size_t k = 0; k < idx.size(); ++k) {
        const Layer& L = layers[idx[k]];
        int Ho, Wo;
        conv_out_dims(L, H, W, &Ho, &Wo);
        if (k + 1 == idx.size() && last) {
            ys[k] = *last; dys[k] = *dlast;
            if (ys[k].H != Ho || ys[k].W != Wo || ys[k].C != L.cout) return fail(W2L_EINVAL, "%s: destination shape mismatch", L.name.c_str());
        } else {
            CKR(tp_act(tp, &ys[k], x0.N, Ho, Wo, L.cout));
            CKR(tp_act(tp, &dys[k], x0.N, Ho, Wo, L.cout));
        }
        H = Ho; W = Wo;
    }
    Act none;
    for (size_t k = 0; k < idx.size(); ++k) {
        const Layer& L = layers[idx[k]];
        const Act& x = k == 0 ? x0 : ys[k - 1];
        const Act& dx = k == 0 ? dx0 : dys[k - 1];
        const bool hw1 = L.kind == W2L_BLOCK_CONVT_BN_RELU && x.H == 1 && x.W == 1;
        CKR(add_train_block(ctx, tp, net, idx[k], L, x, ys[k], dys[k], dx, k == 0 ? dx0_add : none, want_wgrad, hw1, ws_need,
                            k + 1 == idx.size() ? last_f32 : nullptr, k == 0 ? fold_in : nullptr));
    }
    if (out) *out = ys.back();
    if (dout) *dout = dys.back();
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// the three networks
// ------------------------------------------------------------------------------------------------
static int build_generator_train_plan(w2l_ctx* ctx, TrainPlan* tp, size_t* ws_need) {
    const GeneratorSpec& g = gen_spec();
    const int N = tp->N, B = tp->B, T = tp->T;
    const int net = W2L_NET_GENERATOR;
    Act faceIn, melIn, none;
    CKR(tp_act(tp, &faceIn, N, 96, 96, 16));
    CKR(tp_act(tp, &melIn, N, 80, 16, 16));
    IngestSpec mel, face;
    generator_inputs(B, T, &mel, &face);
    add_train_ingest(tp, "ingest.mel", mel, melIn);
    add_train_ingest(tp, "ingest.face", face, faceIn);
    Act D[7], dD[7];   // [decoder output | encoder skip] and its gradient (wav2lip.py:108)
    for (int k = 0; k < 7; ++k) {
        CKR(tp_act(tp, &D[k], N, g.hw[k], g.hw[k], g.dec_c[k] + g.skip_c[k]));
        CKR(tp_act(tp, &dD[k], N, g.hw[k], g.hw[k], g.dec_c[k] + g.skip_c[k]));
    }
    // audio encoder
    Act AE, dAE;
    CKR(add_train_chain(ctx, tp, net, g.layers, g.audio_enc, melIn, none, none, nullptr, nullptr, true, ws_need, &AE, &dAE, nullptr, &mel));
    // face encoder: stage i ends in the skip half of D[6-i]; the gradient of a stage output is
    //   (input gradient of the next stage's first block) + (skip half of dD[6-i])  — the latter joins in that dgrad's epilogue
    Act x = faceIn, dx = none;
    Act G[7];          // total gradient of stage i's output
    for (int i = 0; i < 6; ++i) CKR(tp_act(tp, &G[i], N, g.hw[6 - i], g.hw[6 - i], g.skip_c[6 - i]));
    G[6] = dD[0].slice(g.dec_c[0], g.skip_c[0]);
    for (int i = 0; i < 7; ++i) {
        Act dst = D[6 - i].slice(g.dec_c[6 - i], g.skip_c[6 - i]);
        Act add = i > 0 ? dD[6 - (i - 1)].slice(g.dec_c[6 - (i - 1)], g.skip_c[6 - (i - 1)]) : none;
        CKR(add_train_chain(ctx, tp, net, g.layers, g.face_enc[i], x, dx, add, &dst, &G[i], true, ws_need, nullptr, nullptr, nullptr,
                            i == 0 ? &face : nullptr));
        x = dst; dx = G[i];
    }
    // decoder
    x = AE; dx = dAE;
    for (int k = 0; k < 7; ++k) {
        Act dst = D[k].slice(0, g.dec_c[k]), ddst = dD[k].slice(0, g.dec_c[k]);
        CKR(add_train_chain(ctx, tp, net, g.layers, g.face_dec[k], x, dx, none, &dst, &ddst, true, ws_need, nullptr, nullptr));
        x = D[k]; dx = dD[k];
    }
    // output block, then the head (its own kernels)
    CKR(tp_act(tp, &tp->y32, N, 96, 96, 32));
    CKR(tp_act(tp, &tp->dy32, N, 96, 96, 32));
    CKR(add_train_block(ctx, tp, net, g.output_block0, g.layers[g.output_block0], x, tp->y32, tp->dy32, dx, none, true, false, ws_need));
    tp->head_blocks = ctx->num_sms * 2;
    CKR(plan_alloc(&tp->pl, &tp->head_partial, (size_t)tp->head_blocks * 99 * 4));
    return W2L_OK;
}

static int build_syncnet_train_plan(w2l_ctx* ctx, TrainPlan* tp, size_t* ws_need, bool want_wgrad, bool input_grad) {
    const SyncnetSpec& s = sync_spec();
    const int N = tp->N, net = W2L_NET_SYNCNET;
    Act faceIn, melIn, none;
    CKR(tp_act(tp, &faceIn, N, 48, 96, 16));
    CKR(tp_act(tp, &melIn, N, 80, 16, 16));
    IngestSpec mel, face;
    syncnet_inputs(N, tp->T, &mel, &face);
    add_train_ingest(tp, "ingest.mel", mel, melIn);
    add_train_ingest(tp, tp->T > 0 ? "ingest.frames" : "ingest.face", face, faceIn);
    CKR(plan_alloc(&tp->pl, &tp->fe_raw, (size_t)N * 512 * 4));
    CKR(plan_alloc(&tp->pl, &tp->ae_raw, (size_t)N * 512 * 4));
    if (input_grad) CKR(tp_act(tp, &tp->dface_in, N, 48, 96, 16));
    Act ae, fe;
    CKR(add_train_chain(ctx, tp, net, s.layers, s.audio_enc, melIn, none, none, nullptr, nullptr, want_wgrad, ws_need, &ae, &tp->dae, tp->ae_raw));
    for (TBlock& b : tp->blocks) b.wgrad_only = true;   // the mel is an input: nothing upstream of the audio branch wants a gradient
    CKR(add_train_chain(ctx, tp, net, s.layers, s.face_enc, faceIn, input_grad ? tp->dface_in : none, none, nullptr, nullptr, want_wgrad,
                        ws_need, &fe, &tp->dfe, tp->fe_raw));
    return W2L_OK;
}

static int build_disc_train_plan(w2l_ctx* ctx, TrainPlan* tp, size_t* ws_need, bool want_wgrad, bool input_grad) {
    const DiscSpec& d = disc_spec();
    const int N = tp->N, B = tp->B, T = tp->T, net = W2L_NET_DISC;
    Act in, none;
    CKR(tp_act(tp, &in, N, 48, 96, 16));
    add_train_ingest(tp, "ingest.frames", disc_input(B, T), in);
    if (input_grad) CKR(tp_act(tp, &tp->dframes_in, N, 48, 96, 16));
    std::vector<int> idx;
    for (size_t i = 0; i < d.layers.size(); ++i) idx.push_back((int)i);
    CKR(add_train_chain(ctx, tp, net, d.layers, idx, in, input_grad ? tp->dframes_in : none, none, nullptr, nullptr, want_wgrad, ws_need,
                        &tp->feat, &tp->dfeat));
    return W2L_OK;
}

enum : int { TRAIN_WGRAD = 1, TRAIN_ACCUMULATE = 2, TRAIN_INPUT_GRAD = 4, TRAIN_NO_STAT_UPDATE = 8,   // = W2L_TRAIN_*
             // passes of the fused steps only:
             TRAIN_SKIP_INPUT_GRAD = 16,   // a plan built with its input gradient: leave that last dgrad out of this pass
             TRAIN_ONE_STREAM = 32 };      // every launch on the caller's stream (a lane of its own beside another backward)

static int get_train_plan(w2l_ctx* ctx, int net, int B, int T, bool want_wgrad, bool input_grad, TrainPlan** out) {
    TrainState* ts = train_state(ctx);
    if (!ctx->bf16) return fail(W2L_ESTATE, "training runs with bf16 operands (gradients leave the fp16 range): create the context with W2L_PREC_BF16");
    if (!ts->is_bound[net]) return fail(W2L_ESTATE, "training: parameters of net %d are not bound (w2l_train_bind)", net);
    char key[64];
    snprintf(key, sizeof(key), "%d:%d:%d:%d:%d", net, B, T, (int)want_wgrad, (int)input_grad);
    auto it = ts->plans.find(key);
    if (it != ts->plans.end()) { *out = it->second.get(); return W2L_OK; }
    std::unique_ptr<TrainPlan> tp(new TrainPlan(ctx));
    tp->net = net; tp->B = B; tp->T = T; tp->input_grad = input_grad;
    tp->N = (net == W2L_NET_SYNCNET) ? B : (T > 0 ? B * T : B);
    size_t ws_need[2] = {0, 0};
    int r;
    if (net == W2L_NET_GENERATOR) r = build_generator_train_plan(ctx, tp.get(), ws_need);
    else if (net == W2L_NET_SYNCNET) r = build_syncnet_train_plan(ctx, tp.get(), ws_need, want_wgrad, input_grad);
    else r = build_disc_train_plan(ctx, tp.get(), ws_need, want_wgrad, input_grad);
    CKR(r);
    for (int lane = 0; lane < 2; ++lane) {
        if (!ws_need[lane]) continue;
        CKR(plan_alloc(&tp->pl, &tp->wg_ws[lane], ws_need[lane]));
        tp->wg_ws_bytes[lane] = ws_need[lane];
    }
    CK(cudaDeviceSynchronize());
    *out = tp.get();
    ts->plans[key] = std::move(tp);
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// replay (training plans exist only on bf16 contexts, get_train_plan: every launch below is the bf16 instantiation)
// ------------------------------------------------------------------------------------------------
static int repack_weights(w2l_ctx* ctx, TrainPlan* tp, cudaStream_t st) {
    const std::vector<PackParams>& jobs = tp->repack.pack;
    if (!jobs.empty()) {
        if (!tp->pack_blocks) {   // job table + block map, built once per plan
            std::vector<int> blk_job, blk_first;
            for (size_t j = 0; j < jobs.size(); ++j) {
                const PackParams& pp = jobs[j];
                const long long total = (long long)pp.ntaps * pp.cout_pad * pp.cin_pad;
                blk_first.push_back((int)blk_job.size());
                for (long long b = 0; b < (total + 4095) / 4096; ++b) blk_job.push_back((int)j);
            }
            CKR(tp->pack_dev.grow(ctx, jobs.size() * sizeof(PackParams)));
            CKR(tp->pack_blk_job.grow(ctx, blk_job.size() * 4));
            CKR(tp->pack_blk_first.grow(ctx, blk_first.size() * 4));
            CK(cudaMemcpy(tp->pack_dev, jobs.data(), jobs.size() * sizeof(PackParams), cudaMemcpyHostToDevice));
            CK(cudaMemcpy(tp->pack_blk_job, blk_job.data(), blk_job.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(tp->pack_blk_first, blk_first.data(), blk_first.size() * 4, cudaMemcpyHostToDevice));
            tp->pack_blocks = (int)blk_job.size();
        }
        pack_multi_kernel<true><<<tp->pack_blocks, 256, 0, st>>>(tp->pack_dev, tp->pack_blk_job, tp->pack_blk_first);
        ctx->launches++;
    }
    for (const PackFoldParams& fp : tp->repack.pack_fold) {
        const size_t n = (size_t)fp.kh * fp.cout_pad * fp.kfold;
        const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
        pack_fold_kernel<true><<<blocks, 256, 0, st>>>(fp);
        ctx->launches++;
    }
    for (const FoldJob& f : tp->repack.fold) {
        fold_bn_kernel<<<(f.n_pad + 127) / 128, 128, 0, st>>>(f.bias, nullptr, nullptr, nullptr, nullptr, 1e-5f, f.cout, f.reps, f.n_pad, f.scale, f.shift);
        ctx->launches++;
    }
    CK(cudaGetLastError());
    return W2L_OK;
}

static int elem_grid(w2l_ctx* ctx, long long work_items) {
    return (int)std::max<long long>(1, std::min<long long>((work_items + kBnThreads - 1) / kBnThreads, (long long)ctx->num_sms * 8));
}
constexpr int kRedSmem = 2 * 2048 * 4;   // chan_reduce_kernel: [rows][2][C] floats, rows * C <= 2048

template <int MODE>
static void launch_chan_reduce(w2l_ctx* ctx, const ChanReduceParams& rp, int nblk, cudaStream_t st) {
    chan_reduce_kernel<true, MODE><<<nblk, kBnThreads, kRedSmem, st>>>(rp);
    ctx->launches++;
}

static int block_forward(w2l_ctx* ctx, TrainPlan* tp, TBlock& b, bool update_running, cudaStream_t st) {
    for (size_t i = b.fwd0; i < b.fwd1; ++i) CKR(launch_conv(ctx, tp->pl.ops[i], st));
    if (!b.bn) return W2L_OK;   // nonorm: bias + LeakyReLU in the conv epilogue
    const int C = b.L.cout;
    ChanReduceParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.z = b.z.ptr(); rp.z_pitch = b.z.Cs; rp.partial = b.partial; rp.M = b.M; rp.C = C;
    launch_chan_reduce<0>(ctx, rp, b.nblk, st);
    bn_finalize_kernel<<<(C + 31) / 32, kFinThreads, 0, st>>>(b.partial, b.nblk, C, (double)b.M, b.b, update_running ? b.rmean : nullptr,
                                                       update_running ? b.rvar : nullptr, b.gamma, b.beta, b.stats);
    ctx->launches++;
    BnApplyParams ap;
    memset(&ap, 0, sizeof(ap));
    ap.z = b.z.ptr(); ap.z_pitch = b.z.Cs;
    if (b.L.residual) { ap.res = b.x.ptr(); ap.res_pitch = b.x.Cs; }
    ap.y = b.y.ptr(); ap.y_pitch = b.y.Cs; ap.y_f32 = b.y_f32;
    ap.stats = b.stats; ap.M = b.M; ap.C = C;
    const int grid = b.nblk * 2;   // rows-of-pixels layout (kBnThreads / (C/8) pixels per block iteration), as the reductions
    bn_apply_kernel<true><<<grid, kBnThreads, 0, st>>>(ap);
    ctx->launches++;
    return W2L_OK;
}

static int ensure_wg_stream(TrainState* ts) {
    if (ts->s_wg) return W2L_OK;
    CKR(ts->s_wg.create());
    CKR(ts->ev_dz.create());
    CKR(ts->ev_wg.create());
    CKR(ts->ev_wgb.create());
    return W2L_OK;
}

static int ensure_aux_stream(TrainState* ts) {
    if (ts->s_aux) return W2L_OK;
    CKR(ts->s_aux.create());
    CKR(ts->ev_aux_fork.create());
    CKR(ts->ev_aux_join.create());
    return W2L_OK;
}
static int ensure_disc_stream(TrainState* ts) {
    if (ts->s_disc) return W2L_OK;
    CKR(ts->s_disc.create());
    CKR(ts->ev_disc_fork.create());
    CKR(ts->ev_disc_join.create());
    return W2L_OK;
}
static bool has_aux_lane(const TrainPlan* tp) {
    for (const TBlock& b : tp->blocks) if (b.lane == 1) return true;
    return false;
}

// s_wg != nullptr: the block's wgrad (+ its split-K reduction) goes to that stream, ordered after this block's dz (ev);
// the caller joins the stream before anything consumes the parameter gradients.
//   dgrad == false: the input gradient of this block is not wanted in this pass (TRAIN_SKIP_INPUT_GRAD)
static int block_backward(w2l_ctx* ctx, TrainPlan* tp, TBlock& b, bool wgrad, bool accumulate, bool dgrad, cudaStream_t st,
                          cudaStream_t s_wg = nullptr, cudaEvent_t ev = nullptr) {
    const int C = b.L.cout;
    ChanReduceParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.dy = b.dy.ptr(); rp.dy_pitch = b.dy.Cs; rp.y = b.y.ptr(); rp.y_pitch = b.y.Cs;
    rp.partial = b.partial; rp.M = b.M; rp.C = C;
    // non-residual BatchNorm blocks: y > 0  <=>  gamma * zhat + beta > 0 (the value the forward rounded to bf16 has the same
    // sign unless it underflows): recompute the mask from z instead of reading y a second and third time
    const bool mask_from_z = b.bn && !b.L.residual;
    if (b.bn) {
        if (mask_from_z) rp.y = nullptr;
        rp.z = b.z.ptr(); rp.z_pitch = b.z.Cs; rp.stats = b.stats;
        launch_chan_reduce<1>(ctx, rp, b.nblk, st);
        const bool pg = wgrad && b.ggamma;
        bn_bwd_finalize_kernel<<<(C + 31) / 32, kFinThreads, 0, st>>>(b.partial, b.nblk, C, (double)b.M, b.gamma, b.stats, pg ? b.ggamma : nullptr,
                                                           pg ? b.gbeta : nullptr, accumulate ? 1 : 0, b.coef);
        ctx->launches++;
        BnBwdApplyParams ap;
        memset(&ap, 0, sizeof(ap));
        ap.z = b.z.ptr(); ap.z_pitch = b.z.Cs; ap.dy = b.dy.ptr(); ap.dy_pitch = b.dy.Cs; ap.y = b.y.ptr(); ap.y_pitch = b.y.Cs;
        ap.dz = b.dz.ptr(); ap.du = b.L.residual ? b.du.ptr() : nullptr; ap.stats = b.stats; ap.coef = b.coef; ap.M = b.M; ap.C = C;
        if (mask_from_z) ap.y = nullptr;
        const int grid = b.nblk * 2;
        bn_bwd_apply_kernel<true><<<grid, kBnThreads, 0, st>>>(ap);
        ctx->launches++;
        // the conv bias under a BatchNorm has an exactly zero gradient (sum of dz over the batch is 0 by construction)
        if (wgrad && b.gb && !accumulate) { fill_kernel<<<1, 128, 0, st>>>(b.gb, C, 0.0f); ctx->launches++; }
    } else {
        rp.dz = b.dz.ptr(); rp.dz_pitch = b.dz.Cs;
        launch_chan_reduce<2>(ctx, rp, b.nblk, st);
        if (wgrad && b.gb) {
            bias_grad_finalize_kernel<<<(C + 31) / 32, kFinThreads, 0, st>>>(b.partial, b.nblk, C, b.gb, accumulate ? 1 : 0);
            ctx->launches++;
        }
    }
    const bool side = s_wg != nullptr && wgrad && b.wg.on;
    if (side) {
        CK(cudaEventRecord(ev, st));
        CK(cudaStreamWaitEvent(s_wg, ev, 0));
        CKR(launch_wgrad(ctx, tp, b, accumulate, s_wg));
    }
    if (dgrad) for (size_t i = b.dg0; i < b.dg1; ++i) CKR(launch_conv(ctx, tp->pl.ops[i], st));
    if (!side && wgrad && b.wg.on) CKR(launch_wgrad(ctx, tp, b, accumulate, st));
    return W2L_OK;
}

static int train_forward(w2l_ctx* ctx, TrainPlan* tp, const void* in0, const void* in1, void* out0, void* out1, int flags, cudaStream_t st) {
    TrainState* ts = train_state(ctx);
    CKR(repack_weights(ctx, tp, st));
    for (size_t i : tp->ingest) {
        const Op& op = tp->pl.ops[i];
        CKR(launch_ingest(ctx, op, op.ingest_src == 0 ? in0 : in1, st));
    }
    const bool upd = !(flags & TRAIN_NO_STAT_UPDATE);
    // the audio-encoder blocks (lane 1) run on the auxiliary stream beside the face encoder; the first consumer of the audio
    // embedding (face_decoder_blocks.0.0; the embedding normalisation for SyncNet) waits for them
    const bool aux = ctx->use_aux_stream && tp->blocks.size() > 1 && has_aux_lane(tp);
    bool joined = !aux;
    if (aux) {
        CKR(ensure_aux_stream(ts));
        CK(cudaEventRecord(ts->ev_aux_fork, st));
        CK(cudaStreamWaitEvent(ts->s_aux, ts->ev_aux_fork, 0));
    }
    auto join_aux = [&]() -> int {
        CK(cudaEventRecord(ts->ev_aux_join, ts->s_aux));
        CK(cudaStreamWaitEvent(st, ts->ev_aux_join, 0));
        joined = true;
        return W2L_OK;
    };
    for (TBlock& b : tp->blocks) {
        if (aux && b.lane == 1) { CKR(block_forward(ctx, tp, b, upd, ts->s_aux)); continue; }
        if (!joined && starts_with(b.L.name, "face_decoder_blocks.")) CKR(join_aux());
        CKR(block_forward(ctx, tp, b, upd, st));
    }
    if (!joined) CKR(join_aux());
    if (tp->net == W2L_NET_GENERATOR) {
        HeadParams hp;
        memset(&hp, 0, sizeof(hp));
        float *hw, *hb;
        CKR(bound_ptr(ts, tp->net, "output_block.1.weight", 96, &hw, nullptr));
        CKR(bound_ptr(ts, tp->net, "output_block.1.bias", 3, &hb, nullptr));
        hp.y32 = tp->y32.ptr(); hp.y_pitch = tp->y32.Cs; hp.w = hw; hp.b = hb; hp.g = (float*)out0;
        hp.N = tp->N; hp.B = tp->T > 0 ? tp->B : tp->N; hp.T = tp->T > 0 ? tp->T : 1; hp.HW = 9216;
        const int grid = elem_grid(ctx, (long long)tp->N * 9216);
        head_fwd_kernel<true><<<grid, 256, 0, st>>>(hp);
        ctx->launches++;
        tp->g_out = (const float*)out0;
    } else if (tp->net == W2L_NET_SYNCNET) {
        l2norm_kernel<<<(tp->N + 3) / 4, 128, 0, st>>>(tp->ae_raw, (float*)out0, tp->N, 512);
        l2norm_kernel<<<(tp->N + 3) / 4, 128, 0, st>>>(tp->fe_raw, (float*)out1, tp->N, 512);
        ctx->launches += 2;
        tp->a_out = (const float*)out0; tp->v_out = (const float*)out1;
    } else {
        float *hw, *hb;
        CKR(bound_ptr(ts, tp->net, "binary_pred.0.weight", 512, &hw, nullptr));
        CKR(bound_ptr(ts, tp->net, "binary_pred.0.bias", 1, &hb, nullptr));
        disc_head_kernel<true><<<(tp->N + 3) / 4, 128, 0, st>>>(tp->feat.ptr(), hw, hb, (float*)out0, tp->N, 512, tp->feat.Cs, 0);
        ctx->launches++;
        tp->prob_out = (const float*)out0;
    }
    CK(cudaGetLastError());
    ts->last[tp->net] = tp;
    return W2L_OK;
}

// gradient buckets of the generator, in the order the backward completes them (blocks are visited in reverse)
static int train_backward(w2l_ctx* ctx, TrainPlan* tp, const float* d0, const float* d1, int flags, cudaStream_t st,
                          const std::function<int(size_t)>* after_block = nullptr) {
    TrainState* ts = train_state(ctx);
    const bool wgrad = (flags & TRAIN_WGRAD) != 0, acc = (flags & TRAIN_ACCUMULATE) != 0;
    if (tp->net == W2L_NET_GENERATOR) {
        if (!tp->g_out) return fail(W2L_ESTATE, "generator backward before a training forward");
        HeadParams hp;
        memset(&hp, 0, sizeof(hp));
        float *hw, *hb, *ghw, *ghb;
        CKR(bound_ptr(ts, tp->net, "output_block.1.weight", 96, &hw, &ghw));
        CKR(bound_ptr(ts, tp->net, "output_block.1.bias", 3, &hb, &ghb));
        hp.y32 = tp->y32.ptr(); hp.y_pitch = tp->y32.Cs; hp.w = hw; hp.b = hb; hp.g = const_cast<float*>(tp->g_out); hp.dg = d0;
        hp.dy32 = tp->dy32.ptr(); hp.partial = tp->head_partial;
        hp.N = tp->N; hp.B = tp->T > 0 ? tp->B : tp->N; hp.T = tp->T > 0 ? tp->T : 1; hp.HW = 9216;
        head_bwd_kernel<true><<<tp->head_blocks, 256, 0, st>>>(hp);
        ctx->launches++;
        if (wgrad && ghw && ghb) { head_bwd_finalize_kernel<<<1, 128, 0, st>>>(tp->head_partial, tp->head_blocks, ghw, ghb, acc ? 1 : 0); ctx->launches++; }
    } else if (tp->net == W2L_NET_SYNCNET) {
        if (!tp->a_out) return fail(W2L_ESTATE, "syncnet backward before a training forward");
        // through F.normalize (syncnet.py:62-63): d0 = dL/d audio_embedding, d1 = dL/d face_embedding
        l2norm_bwd_kernel<true><<<(tp->N + 3) / 4, 128, 0, st>>>(tp->ae_raw, d0, tp->dae.ptr(), tp->N, 512);
        l2norm_bwd_kernel<true><<<(tp->N + 3) / 4, 128, 0, st>>>(tp->fe_raw, d1, tp->dfe.ptr(), tp->N, 512);
        ctx->launches += 2;
    } else {
        if (!tp->prob_out) return fail(W2L_ESTATE, "disc backward before a training forward");
        float *hw, *hb, *ghw, *ghb;
        CKR(bound_ptr(ts, tp->net, "binary_pred.0.weight", 512, &hw, &ghw));
        CKR(bound_ptr(ts, tp->net, "binary_pred.0.bias", 1, &hb, &ghb));
        float* dw = (wgrad && ghw) ? ghw : ts->loss_dev + 8;   // scratch when the head's gradient is not wanted
        float* db = (wgrad && ghb) ? ghb : ts->loss_dev + 8 + 512;
        const int accf = (wgrad && ghw && acc) ? 1 : 0;
        disc_head_bwd_kernel<true><<<1, 512, 0, st>>>(tp->feat.ptr(), tp->feat.Cs, hw, tp->prob_out, d0, tp->N, 512, tp->dfeat.ptr(), dw, db, accf);
        ctx->launches++;
    }
    const bool one_stream = (flags & TRAIN_ONE_STREAM) != 0;
    cudaStream_t s_wg = nullptr;
    if (wgrad && ctx->use_wg_stream && !one_stream) { CKR(ensure_wg_stream(ts)); s_wg = ts->s_wg; }
    // the plan's own input gradient (first block's dx), left out of a pass that only wants parameter gradients
    const void* skip_dx = nullptr;
    if ((flags & TRAIN_SKIP_INPUT_GRAD) && tp->input_grad) skip_dx = tp->net == W2L_NET_DISC ? tp->dframes_in.base : tp->dface_in.base;
    // audio-encoder blocks (lane 1): their backward chain starts at the gradient of the audio embedding — produced by
    // face_decoder_blocks.0.0's dgrad (generator) or by the normalisation backward above (SyncNet) — and shares nothing with
    // the face encoder's: it runs on the auxiliary stream, forked at that point, joined before the last block's hook
    const bool aux = ctx->use_aux_stream && !one_stream && tp->blocks.size() > 1 && has_aux_lane(tp);
    bool forked = false, waited = false, joined = false;
    if (aux) {
        CKR(ensure_aux_stream(ts));
        if (tp->net != W2L_NET_GENERATOR) { CK(cudaEventRecord(ts->ev_aux_fork, st)); forked = true; }
    }
    auto join_aux = [&]() -> int {
        if (waited && !joined) {
            CK(cudaEventRecord(ts->ev_aux_join, ts->s_aux));
            CK(cudaStreamWaitEvent(st, ts->ev_aux_join, 0));
        }
        joined = true;
        return W2L_OK;
    };
    for (size_t k = tp->blocks.size(); k-- > 0;) {
        TBlock& b = tp->blocks[k];
        // a frozen expert inside the generator step only needs the face branch: skip blocks whose gradient goes nowhere
        if (!wgrad && b.wgrad_only) continue;
        cudaStream_t bs = st;
        if (aux && forked && b.lane == 1) {
            if (!waited) { CK(cudaStreamWaitEvent(ts->s_aux, ts->ev_aux_fork, 0)); waited = true; }
            bs = ts->s_aux;
        }
        const bool dgrad = !(skip_dx && b.dx.base == skip_dx);
        CKR(block_backward(ctx, tp, b, wgrad, acc, dgrad, bs, s_wg, ts->ev_dz));
        if (aux && !forked && b.L.name == "face_decoder_blocks.0.0") { CK(cudaEventRecord(ts->ev_aux_fork, st)); forked = true; }
        if (k == 0) CKR(join_aux());
        if (after_block) CKR((*after_block)(k));
    }
    CKR(join_aux());
    if (s_wg) {   // join: whatever follows on `st` (Adam, the caller's optimizer, the next forward) sees every gradient
        CK(cudaEventRecord(ts->ev_wg, s_wg));
        CK(cudaStreamWaitEvent(st, ts->ev_wg, 0));
    }
    CK(cudaGetLastError());
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// optimizer, collective, fused steps
// ------------------------------------------------------------------------------------------------
static int ensure_train_scratch(w2l_ctx* ctx, int B, int T) {
    TrainState* ts = train_state(ctx);
    if (!ts->loss_dev) { CKR(ts->loss_dev.grow(ctx, 2048 * 4)); CK(cudaMemset(ts->loss_dev, 0, 2048 * 4)); }
    const int N = B * std::max(T, 1);
    for (DevMem<float>* q : {&ts->a_emb, &ts->v_emb, &ts->da, &ts->dv}) CKR(q->grow(ctx, (size_t)B * 512 * 4));
    CKR(ts->prob.grow(ctx, (size_t)2 * N * 4));
    CKR(ts->dprob.grow(ctx, (size_t)3 * N * 4));
    for (DevMem<float>* q : {&ts->g_buf, &ts->dg_buf}) CKR(q->grow(ctx, (size_t)N * 3 * 9216 * 4));
    return W2L_OK;
}

// the moments (zero) of every bound tensor of `net` that has a gradient, allocated at the first use
static int ensure_adam_slot(w2l_ctx* ctx, int net, cudaStream_t st) {
    TrainState* ts = train_state(ctx);
    AdamSlot& a = ts->adam[net];
    if (a.dev) return W2L_OK;
    AdamSlot t;   // stored in the slot only once every allocation has succeeded
    for (auto& kv : ts->bound[net]) {
        if (!kv.second.grad) continue;
        const size_t bytes = (size_t)kv.second.n * 4;
        float *m, *v;
        CKR(alloc_in(ctx, &t.moments, &m, bytes));
        CKR(alloc_in(ctx, &t.moments, &v, bytes));
        CK(cudaMemsetAsync(m, 0, bytes, st));
        CK(cudaMemsetAsync(v, 0, bytes, st));
        t.names.push_back(kv.first);
        t.host.push_back(AdamTensor{kv.second.value, kv.second.grad, m, v, kv.second.n});
    }
    if (t.host.empty()) return fail(W2L_ESTATE, "adam: no gradient tensors bound for net %d", net);
    CKR(t.dev.grow(ctx, t.host.size() * sizeof(AdamTensor)));
    CK(cudaMemcpyAsync(t.dev, t.host.data(), t.host.size() * sizeof(AdamTensor), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    a = std::move(t);
    return W2L_OK;
}

static int adam_step(w2l_ctx* ctx, int net, float lr, float beta1, float beta2, float eps, float grad_scale, cudaStream_t st) {
    TrainState* ts = train_state(ctx);
    AdamSlot& a = ts->adam[net];
    CKR(ensure_adam_slot(ctx, net, st));
    a.step++;
    AdamParams p;
    p.t = a.dev; p.lr = lr; p.beta1 = beta1; p.beta2 = beta2; p.eps = eps;
    p.bc1 = (float)(1.0 - std::pow((double)beta1, (double)a.step));
    p.bc2_sqrt = (float)std::sqrt(1.0 - std::pow((double)beta2, (double)a.step));
    p.grad_scale = grad_scale;
    adam_kernel<<<dim3(32, (unsigned)a.host.size()), 256, 0, st>>>(p);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

// ---- gradient all-reduce: NCCL resolved from the process (torch has loaded libnccl.so.2) ----
static void* nccl_sym(TrainState* ts, const char* name) {
    if (!ts->nccl_lib) {
        ts->nccl_lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!ts->nccl_lib) ts->nccl_lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!ts->nccl_lib) ts->nccl_lib = dlopen(nullptr, RTLD_NOW);
    }
    return ts->nccl_lib ? dlsym(ts->nccl_lib, name) : nullptr;
}

struct GradRange { float* p; long long n; };

// one contiguous [ptr, ptr + n) range per bucket when the caller laid the gradients out contiguously (the Python side
// allocates one arena in state_dict order); otherwise one range per tensor
static std::vector<GradRange> bucket_ranges(TrainState* ts, int net, const std::vector<std::string>& prefixes) {
    std::vector<GradRange> t;
    for (auto& kv : ts->bound[net]) {
        if (!kv.second.grad) continue;
        for (const std::string& pre : prefixes)
            if (kv.first.compare(0, pre.size(), pre) == 0) { t.push_back(GradRange{kv.second.grad, kv.second.n}); break; }
    }
    std::sort(t.begin(), t.end(), [](const GradRange& a, const GradRange& b) { return a.p < b.p; });
    std::vector<GradRange> out;
    for (const GradRange& r : t) {
        if (!out.empty() && out.back().p + out.back().n == r.p) out.back().n += r.n;
        else out.push_back(r);
    }
    return out;
}

static int all_reduce_ranges(w2l_ctx* ctx, const std::vector<GradRange>& ranges, cudaStream_t compute) {
    TrainState* ts = train_state(ctx);
    if (ts->world <= 1 || !ts->comm) return W2L_OK;
    CK(cudaEventRecord(ts->ev_bucket, compute));
    CK(cudaStreamWaitEvent(ts->s_comm, ts->ev_bucket, 0));
    if (ts->s_wg) {   // the bucket's weight gradients were queued on the wgrad stream
        CK(cudaEventRecord(ts->ev_wgb, ts->s_wg));
        CK(cudaStreamWaitEvent(ts->s_comm, ts->ev_wgb, 0));
    }
    for (const GradRange& r : ranges) {
        const int rc = ts->all_reduce(r.p, r.p, (size_t)r.n, /*ncclFloat32*/ 7, /*ncclAvg*/ 4, ts->comm, ts->s_comm);
        if (rc != 0) return fail(W2L_ECUDA, "ncclAllReduce failed: %s", ts->err_string ? ts->err_string(rc) : "?");
        ts->last_allreduce_bytes += (double)r.n * 4;
    }
    return W2L_OK;
}

static int join_comm(w2l_ctx* ctx, cudaStream_t compute) {
    TrainState* ts = train_state(ctx);
    if (ts->world <= 1 || !ts->comm) return W2L_OK;
    CK(cudaEventRecord(ts->ev_comm, ts->s_comm));
    CK(cudaStreamWaitEvent(compute, ts->ev_comm, 0));
    return W2L_OK;
}

// generator backward with the bucketed all-reduce launched as soon as a bucket's last wgrad is queued
static int generator_backward_dp(w2l_ctx* ctx, TrainPlan* tp, const float* dg, cudaStream_t st) {
    TrainState* ts = train_state(ctx);
    if (ts->world <= 1 || !ts->comm) return train_backward(ctx, tp, dg, nullptr, TRAIN_WGRAD, st);
    size_t k_a = 0, k_b = 0;
    for (size_t k = 0; k < tp->blocks.size(); ++k) {
        if (tp->blocks[k].L.name == "face_decoder_blocks.4.0") k_a = k;
        if (tp->blocks[k].L.name == "face_decoder_blocks.0.0") k_b = k;
    }
    const std::vector<GradRange> ra = bucket_ranges(ts, tp->net, {"output_block.", "face_decoder_blocks.4.", "face_decoder_blocks.5.", "face_decoder_blocks.6."});
    const std::vector<GradRange> rb = bucket_ranges(ts, tp->net, {"face_decoder_blocks.0.", "face_decoder_blocks.1.", "face_decoder_blocks.2.", "face_decoder_blocks.3."});
    const std::vector<GradRange> rc = bucket_ranges(ts, tp->net, {"face_encoder_blocks.", "audio_encoder."});
    ts->last_allreduce_bytes = 0;
    std::function<int(size_t)> hook = [&](size_t k) -> int {
        if (k == k_a) return all_reduce_ranges(ctx, ra, st);
        if (k == k_b) return all_reduce_ranges(ctx, rb, st);
        if (k == 0) return all_reduce_ranges(ctx, rc, st);
        return W2L_OK;
    };
    CKR(train_backward(ctx, tp, dg, nullptr, TRAIN_WGRAD, st, &hook));
    return join_comm(ctx, st);
}

__global__ void combine_losses_kernel(float* l, float wt_sync, float wt_disc) {
    // l[0] = sync, l[1] = l1, l[2] = perceptual  ->  l[3] = total (wav2lip_train.py:229 / hq_wav2lip_train.py:239-240)
    if (threadIdx.x == 0) l[3] = wt_sync * l[0] + wt_disc * l[2] + (1.0f - wt_sync - wt_disc) * l[1];
}
