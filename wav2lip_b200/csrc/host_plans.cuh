// host_plans.cuh — execution plans of the three networks (buffers, op lists, side-stream lanes), the plan cache and
// the replay loop.
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// plans
// ------------------------------------------------------------------------------------------------
struct TmpPool {  // two ping-pong temporaries per chain, grown on demand
    Act slot[2];
    size_t cap[2] = {0, 0};
    int next = 0;
};

static int tmp_act(w2l_ctx* ctx, Plan* pl, TmpPool* tp, Act* a, int N, int H, int W, int C, const uint16_t* avoid) {
    int s = tp->next;
    if (tp->slot[s].base != nullptr && tp->slot[s].base == avoid) s ^= 1;
    const size_t need_b = (size_t)N * H * W * C * 2 * (pl->x2 ? 2 : 1);
    if (ctx->keep_all || tp->cap[s] < need_b) {
        CKR(plan_act(pl, &tp->slot[s], N, H, W, C));
        tp->cap[s] = need_b;
    }
    Act v = tp->slot[s];
    v.N = N; v.H = H; v.W = W; v.Cs = pl->x2 ? 2 * C : C; v.c_off = 0; v.C = C; v.lo_off = pl->x2 ? C : 0;
    *a = v;
    tp->next = s ^ 1;
    return W2L_OK;
}

// How the ingest kernel reads one fp32 caller tensor (IngestParams): destination image n = t*B + b, channel c, row y
// comes from src + b*sB + t*sT + c*sC + (y + y_off)*Wsrc;  cgrp > 0: c*sC becomes (c / cgrp)*sG + (c % cgrp)*sC
struct IngestSpec {
    int src_id;          // which caller tensor: 0 = mel / frames, 1 = face
    int B, C;
    long long sB, sC, sT;
    int y_off, Wsrc;
    int cgrp = 0;
    long long sG = 0;
};

// The caller tensors of each network, for its inference and its training plans.
// Generator: mel (B,T,1,80,16) and face (B,6,T,96,96); T == 0: (B,1,80,16) and (B,6,96,96)
static void generator_inputs(int B, int T, IngestSpec* mel, IngestSpec* face) {
    if (T > 0) {
        *mel = IngestSpec{0, B, 1, (long long)T * 1280, 1280, 1280, 0, 16};
        *face = IngestSpec{1, B, 6, (long long)6 * T * 9216, (long long)T * 9216, 9216, 0, 96};
    } else {
        *mel = IngestSpec{0, B, 1, 1280, 1280, 0, 0, 16};
        *face = IngestSpec{1, B, 6, 6 * 9216, 9216, 0, 0, 96};
    }
}

// SyncNet: mel (B,1,80,16) and the face window (B,15,48,96); T > 0: generated / ground-truth frames (B,3,T,96,96) instead,
// lower half, the T frames stacked on channels (c' = 3 t + c) — wav2lip_train.py:193-194 as addressing
static void syncnet_inputs(int B, int T, IngestSpec* mel, IngestSpec* face) {
    *mel = IngestSpec{0, B, 1, 1280, 1280, 0, 0, 16};
    if (T > 0) *face = IngestSpec{1, B, 3 * T, (long long)3 * T * 9216, (long long)T * 9216, 0, 48, 96, 3, 9216};
    else *face = IngestSpec{1, B, 15, 15 * 4608, 4608, 0, 0, 96};
}

// Discriminator: frames (B,3,T,96,96), t-major flatten + rows 48..95   (wav2lip.py:155-161)
static IngestSpec disc_input(int B, int T) { return IngestSpec{0, B, 3, (long long)3 * T * 9216, (long long)T * 9216, 9216, 48, 96}; }

static void add_ingest(Plan* pl, const char* name, const IngestSpec& s, const Act& dst) {
    Op op;
    op.type = OP_INGEST;
    op.name = name;
    op.ingest_src = s.src_id;
    IngestParams& ip = op.ip;
    ip.src = nullptr; ip.dst = dst.base;
    ip.N = dst.N; ip.B = s.B; ip.C = s.C; ip.H = dst.H; ip.W = dst.W;
    ip.Cpad = dst.lo_off > 0 ? dst.lo_off : dst.Cs;  // logical (padded) channels; Cs is the pixel pitch
    ip.Cpix = dst.Cs;
    ip.Wp = dst.pitch(); ip.x_off = dst.x_off;
    ip.lo_off = dst.lo_off;
    ip.sB = s.sB; ip.sC = s.sC; ip.sT = s.sT; ip.y_off = s.y_off; ip.Wsrc = s.Wsrc;
    ip.cgrp = s.cgrp; ip.sG = s.sG;
    pl->ops.push_back(op);
}

static int launch_ingest(w2l_ctx* ctx, const Op& op, const void* src, cudaStream_t st) {
    IngestParams ip = op.ip;
    ip.src = (const float*)src;
    const long long total = (long long)ip.N * ip.H * ip.W;
    const bool vec4 = ip.lo_off == 0 && ((ip.W | ip.Wsrc) & 3) == 0 && ((ip.sB | ip.sC | ip.sT | ip.sG) & 3) == 0 &&
                      (((uintptr_t)ip.src) & 15) == 0;
    if (vec4) {
        const int blocks = (int)std::min<long long>((total / 4 + 255) / 256, ctx->num_sms * 16);
        if (ctx->bf16) ingest4_kernel<true><<<blocks, 256, 0, st>>>(ip);
        else ingest4_kernel<false><<<blocks, 256, 0, st>>>(ip);
    } else {
        const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
        if (ctx->bf16) ingest_kernel<true><<<blocks, 256, 0, st>>>(ip);
        else ingest_kernel<false><<<blocks, 256, 0, st>>>(ip);
    }
    ctx->launches++;
    return W2L_OK;
}

// a straight chain of blocks (encoders): ping-pong temporaries, optional final destination
static int emit_chain(w2l_ctx* ctx, Plan* pl, int net, const std::vector<Layer>& layers, const std::vector<int>& idx,
                      Act x, TmpPool* tp, const Act* final_dst, Act* result) {
    for (size_t k = 0; k < idx.size(); ++k) {
        const Layer& L = layers[idx[k]];
        int Ho, Wo;
        conv_out_dims(L, x.H, x.W, &Ho, &Wo);
        Act out;
        if (k + 1 == idx.size() && final_dst) {
            out = *final_dst;
            if (out.H != Ho || out.W != Wo || out.C != L.cout) return fail(W2L_EINVAL, "%s: destination shape mismatch (%dx%dx%d vs %dx%dx%d)", L.name.c_str(), out.H, out.W, out.C, Ho, Wo, L.cout);
        } else {
            CKR(tmp_act(ctx, pl, tp, &out, x.N, Ho, Wo, L.cout, x.base));
        }
        CKR(emit_block(ctx, pl, ctx->nets[net], idx[k], L, x, out, L.residual ? &x : nullptr));
        pl->layer_out[idx[k]] = out;
        x = out;
    }
    if (result) *result = x;
    return W2L_OK;
}

static int build_generator_plan(w2l_ctx* ctx, Plan* pl) {
    const GeneratorSpec& g = gen_spec();
    const int N = pl->N, B = pl->B, T = pl->T;
    Act faceIn, melIn;
    const NetW& nw = ctx->nets[W2L_NET_GENERATOR];
    CKR(plan_input_act(pl, &faceIn, N, 96, 96, 6, nw.layers[g.face_enc[0][0]], g.layers[g.face_enc[0][0]]));
    CKR(plan_input_act(pl, &melIn, N, 80, 16, 1, nw.layers[g.audio_enc[0]], g.layers[g.audio_enc[0]]));
    IngestSpec mel, face;
    generator_inputs(B, T, &mel, &face);
    add_ingest(pl, "ingest.mel", mel, melIn);
    add_ingest(pl, "ingest.face", face, faceIn);
    // skip-concat buffers D[k]: [decoder output | encoder feature] at resolution hw[k]   (wav2lip.py:108)
    Act D[7];
    for (int k = 0; k < 7; ++k) CKR(plan_act(pl, &D[k], N, g.hw[k], g.hw[k], g.dec_c[k] + g.skip_c[k]));

    // audio encoder -> (N,1,1,512)
    Act AE;
    CKR(plan_act(pl, &AE, N, 1, 1, 512));
    TmpPool tpa;
    const size_t audio_first = 0;  // ingest.mel is op 0; ingest.face (op 1) stays on the main lane
    CKR(emit_chain(ctx, pl, W2L_NET_GENERATOR, g.layers, g.audio_enc, melIn, &tpa, &AE, nullptr));
    // the audio encoder (small, latency-bound launches) runs on a side stream while the face encoder runs on the main one
    pl->ops[audio_first].lane = 1;
    for (size_t i = 2; i < pl->ops.size(); ++i) pl->ops[i].lane = 1;
    pl->has_side = true;

    // face encoder: stage i ends in the skip half of D[6-i] and the next stage reads it from there
    TmpPool tpe;
    Act x = faceIn;
    for (int i = 0; i < 7; ++i) {
        Act dst = D[6 - i].slice(g.dec_c[6 - i], g.skip_c[6 - i]);
        CKR(emit_chain(ctx, pl, W2L_NET_GENERATOR, g.layers, g.face_enc[i], x, &tpe, &dst, &x));
        if (i == 0 && nw.layers[g.face_enc[1][0]].ph[0].fold) {
            // The 16->32 stride-2 block gathers every other pixel of a 16-channel slice of D[6]: 32-byte TMA rows, the
            // slowest layer per FLOP. Give it a dense zero-bordered copy of the first block's output instead (second
            // TMA store of the same staged tile), read through the overlapping-window map with the 3 horizontal taps
            // folded into K.
            Op& prev = pl->ops.back();
            if (!prev.patch || prev.head) return fail(W2L_ESTATE, "folded stride-2 block needs the patch kernel on the first block");
            const Layer& L1 = g.layers[g.face_enc[1][0]];
            Act e0;
            CKR(plan_input_act(pl, &e0, N, 96, 96, L1.cin, nw.layers[g.face_enc[1][0]], L1));
            EncodeTiledFn enc = get_encode_fn();
            const CUtensorMapDataType dt = ctx->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
            cuuint64_t od[4] = {16, 96, 96, (cuuint64_t)N};
            cuuint64_t os[3] = {(cuuint64_t)e0.Cs * 2, (cuuint64_t)e0.Wp * e0.Cs * 2, (cuuint64_t)96 * e0.Wp * e0.Cs * 2};
            cuuint32_t ob[4] = {16, (cuuint32_t)kPatchTileW, (cuuint32_t)kPatchTileH, 1};
            cuuint32_t oe[4] = {1, 1, 1, 1};
            CUresult r = enc(&prev.pp.tmO2, dt, 4, e0.base + (size_t)e0.x_off * e0.Cs, od, os, ob, oe, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return fail(W2L_ECUDA, "cuTensorMapEncodeTiled(dense copy) failed with %d", (int)r);
            prev.pp.has_out2 = 1;
            x = e0;
        }
    }
    // decoder
    TmpPool tpd;
    x = AE;
    const size_t dec_first = pl->ops.size();
    for (int k = 0; k < 7; ++k) {
        Act dst = D[k].slice(0, g.dec_c[k]);
        CKR(emit_chain(ctx, pl, W2L_NET_GENERATOR, g.layers, g.face_dec[k], x, &tpd, &dst, nullptr));
        x = D[k];
    }
    // output block with the fused 1x1 + sigmoid head; writes the caller's fp32 tensor
    const Layer& L = g.layers[g.output_block0];
    Act none;
    none.N = N; none.H = 96; none.W = 96; none.Cs = 32; none.C = 32;
    CKR(emit_block(ctx, pl, ctx->nets[W2L_NET_GENERATOR], g.output_block0, L, x, none, nullptr, true, T > 0 ? B : N, T > 0 ? T : 1));
    pl->ops[dec_first].join_side = true;  // the decoder's first block consumes the audio embedding
    return W2L_OK;
}

static int build_syncnet_plan(w2l_ctx* ctx, Plan* pl) {
    const SyncnetSpec& s = sync_spec();
    const int N = pl->N;
    Act faceIn, melIn, fe, ae;
    const NetW& nw = ctx->nets[W2L_NET_SYNCNET];
    CKR(plan_input_act(pl, &faceIn, N, 48, 96, 15, nw.layers[s.face_enc[0]], s.layers[s.face_enc[0]]));
    CKR(plan_input_act(pl, &melIn, N, 80, 16, 1, nw.layers[s.audio_enc[0]], s.layers[s.audio_enc[0]]));
    CKR(plan_act(pl, &fe, N, 1, 1, 512, true));
    CKR(plan_act(pl, &ae, N, 1, 1, 512, true));
    IngestSpec mel, face;
    syncnet_inputs(N, pl->T, &mel, &face);
    add_ingest(pl, "ingest.mel", mel, melIn);
    add_ingest(pl, pl->T > 0 ? "ingest.frames" : "ingest.face", face, faceIn);
    TmpPool tpf, tpa;
    // the two encoders are independent until the embeddings: the audio one (short launches, issued first) runs on the
    // side stream while the face encoder runs on the main one
    CKR(emit_chain(ctx, pl, W2L_NET_SYNCNET, s.layers, s.audio_enc, melIn, &tpa, &ae, nullptr));
    pl->ops[0].lane = 1;  // ingest.mel
    for (size_t i = 2; i < pl->ops.size(); ++i) pl->ops[i].lane = 1;
    pl->has_side = true;
    CKR(emit_chain(ctx, pl, W2L_NET_SYNCNET, s.layers, s.face_enc, faceIn, &tpf, &fe, nullptr));
    const size_t join_at = pl->ops.size();
    for (int which = 0; which < 2; ++which) {
        Op op;
        op.type = OP_L2NORM;
        op.name = which == 0 ? "l2norm.audio" : "l2norm.face";
        op.aux_in = which == 0 ? ae.base : fe.base;
        op.aux_rows = N; op.aux_dim = 512; op.aux_out = which;
        pl->ops.push_back(op);
    }
    pl->ops[join_at].join_side = true;
    return W2L_OK;
}

static int build_disc_plan(w2l_ctx* ctx, Plan* pl) {
    const DiscSpec& d = disc_spec();
    const int N = pl->N, B = pl->B, T = pl->T;
    Act in, feat;
    CKR(plan_input_act(pl, &in, N, 48, 96, 3, ctx->nets[W2L_NET_DISC].layers[0], d.layers[0]));
    CKR(plan_act(pl, &feat, N, 1, 1, 512));
    add_ingest(pl, "ingest.frames", disc_input(B, T), in);
    std::vector<int> idx;
    for (size_t i = 0; i < d.layers.size(); ++i) idx.push_back((int)i);
    TmpPool tp;
    CKR(emit_chain(ctx, pl, W2L_NET_DISC, d.layers, idx, in, &tp, &feat, nullptr));
    Op op;
    op.type = OP_DISC_HEAD;
    op.name = "binary_pred";
    op.aux_in = feat.base; op.aux_rows = N; op.aux_dim = 512; op.aux_out = 0;
    op.aux_pitch = feat.Cs; op.aux_lo = feat.lo_off;
    pl->ops.push_back(op);
    return W2L_OK;
}


// face_detection/detection/sfd/net_s3fd.py:71-128: backbone with taps, L2Norm on the first three, two 3x3 heads per tap.
static void s3fd_dims(int H, int W, int hs[6], int ws[6]) {
    int h = H, w = W;
    h /= 2; w /= 2; h /= 2; w /= 2;          // pool1, pool2 -> conv3_x
    hs[0] = h; ws[0] = w;
    h /= 2; w /= 2; hs[1] = h; ws[1] = w;    // conv4_x
    h /= 2; w /= 2; hs[2] = h; ws[2] = w;    // conv5_x
    h /= 2; w /= 2;                          // pool5
    h += 4; w += 4; hs[3] = h; ws[3] = w;    // fc6: kernel 3, padding 3
    h = (h + 2 - 3) / 2 + 1; w = (w + 2 - 3) / 2 + 1; hs[4] = h; ws[4] = w;   // conv6_2, stride 2
    h = (h + 2 - 3) / 2 + 1; w = (w + 2 - 3) / 2 + 1; hs[5] = h; ws[5] = w;   // conv7_2
}

static int build_s3fd_plan(w2l_ctx* ctx, Plan* pl) {
    const S3fdSpec& sp = s3fd_spec();
    const NetW& nw = ctx->nets[W2L_NET_S3FD];
    const int N = pl->N, H = pl->H, W = pl->W;
    if (H < 32 || W < 32) return fail(W2L_EINVAL, "S3FD needs an image of at least 32 x 32 (five 2x2 pools)");
    Act x;
    CKR(plan_input_act(pl, &x, N, H, W, 3, nw.layers[0], sp.layers[0]));
    add_ingest(pl, "ingest.img", IngestSpec{0, N, 3, (long long)3 * H * W, (long long)H * W, 0, 0, W}, x);
    auto conv = [&](int li, const Act& in, Act* out, bool f32 = false) -> int {
        const Layer& L = sp.layers[li];
        int Ho, Wo;
        conv_out_dims(L, in.H, in.W, &Ho, &Wo);
        CKR(plan_act(pl, out, N, Ho, Wo, L.cout, f32));
        CKR(emit_block(ctx, pl, nw, li, L, in, *out, nullptr));
        pl->layer_out[li] = *out;
        return W2L_OK;
    };
    // pools and L2Norms are exported by w2l_debug_layer_output after the 31 conv layers: pool k at 31 + k, norm i at 36 + i
    int npool = 0;
    auto pool = [&](const Act& in, Act* out) -> int {
        CKR(plan_act(pl, out, N, in.H / 2, in.W / 2, in.C));
        Op op;
        op.type = OP_MAXPOOL; op.name = "max_pool2d";
        op.sp_in = in.base; op.sp_out = out->base; op.sp_N = N; op.sp_H = in.H; op.sp_W = in.W; op.sp_C = in.C;
        op.aux_pitch = in.Cs; op.aux_lo = in.lo_off;   // the output has the input's layout
        pl->ops.push_back(op);
        pl->layer_out[(int)sp.layers.size() + npool++] = *out;
        return W2L_OK;
    };
    Act a, b, taps[6];
    CKR(conv(0, x, &a)); CKR(conv(1, a, &b)); CKR(pool(b, &a));
    CKR(conv(2, a, &b)); CKR(conv(3, b, &a)); CKR(pool(a, &b));
    CKR(conv(4, b, &a)); CKR(conv(5, a, &b)); CKR(conv(6, b, &taps[0])); CKR(pool(taps[0], &a));
    CKR(conv(7, a, &b)); CKR(conv(8, b, &a)); CKR(conv(9, a, &taps[1])); CKR(pool(taps[1], &a));
    CKR(conv(10, a, &b)); CKR(conv(11, b, &a)); CKR(conv(12, a, &taps[2])); CKR(pool(taps[2], &a));
    CKR(conv(13, a, &b)); CKR(conv(14, b, &taps[3]));
    CKR(conv(15, taps[3], &a)); CKR(conv(16, a, &taps[4]));
    CKR(conv(17, taps[4], &a)); CKR(conv(18, a, &taps[5]));
    for (int i = 0; i < 6; ++i) {
        Act f = taps[i];
        if (i < 3) {   // L2Norm(scale 10 / 8 / 5), net_s3fd.py:108-110
            CKR(plan_act(pl, &f, N, taps[i].H, taps[i].W, taps[i].C));
            Op op;
            op.type = OP_CHAN_L2NORM; op.name = "L2Norm";
            op.sp_in = taps[i].base; op.sp_out = f.base; op.sp_w = ctx->s3fd_l2w[i];
            op.sp_N = N; op.sp_H = f.H; op.sp_W = f.W; op.sp_C = f.C;
            op.aux_pitch = f.Cs; op.aux_lo = f.lo_off;
            pl->ops.push_back(op);
            pl->layer_out[(int)sp.layers.size() + 5 + i] = f;
        }
        for (int h = 0; h < 2; ++h) {
            const int li = 19 + 2 * i + h;
            Act o;
            CKR(conv(li, f, &o, true));
            Op op;
            op.type = OP_S3FD_EXPORT; op.name = sp.layers[li].name + ".export";
            op.sp_f32 = (const float*)o.base; op.sp_N = N; op.sp_H = o.H; op.sp_W = o.W;
            op.sp_Cout = h == 0 ? 2 : 4; op.sp_maxout = (i == 0 && h == 0) ? 1 : 0;
            op.aux_out = 2 * i + h;
            pl->ops.push_back(op);
        }
    }
    return W2L_OK;
}

// Detection on an S3FD plan: the select / NMS kernels read the fp32 head outputs the plan already writes (found through its
// export ops); their workspace is allocated once per plan, sized for every anchor of every image.
static int ensure_s3fd_detect(w2l_ctx* ctx, Plan* pl) {
    if (pl->det) return W2L_OK;
    std::unique_ptr<S3fdDetWork> dw(new S3fdDetWork());
    S3fdDetParams& p = dw->p;
    memset(&p, 0, sizeof(p));
    int found = 0;
    for (const Op& op : pl->ops) {
        if (op.type != OP_S3FD_EXPORT) continue;
        S3fdScale& sc = p.sc[op.aux_out / 2];
        if (op.aux_out % 2 == 0) sc.cls = op.sp_f32; else sc.reg = op.sp_f32;
        sc.h = op.sp_H; sc.w = op.sp_W;
        ++found;
    }
    if (found != 12) return fail(W2L_ESTATE, "S3FD plan has %d head outputs, expected 12", found);
    int L = 0;
    for (int i = 0; i < 6; ++i) { p.sc[i].first = L; L += p.sc[i].h * p.sc[i].w; }
    const int B = pl->N;
    p.B = B; p.L = L;
    p.Lpad = 1;
    while (p.Lpad < L) p.Lpad <<= 1;
    p.nchunk = (L + kSelChunk - 1) / kSelChunk;
    CKR(plan_alloc(pl, &p.chunk_count, (size_t)B * p.nchunk * 4));
    CKR(plan_alloc(pl, &p.ncand, (size_t)B * 4));
    CKR(plan_alloc(pl, &p.cbox, (size_t)B * L * 16));
    CKR(plan_alloc(pl, &p.cloc, (size_t)B * L * 4));
    CKR(plan_alloc(pl, &p.keys, (size_t)B * p.Lpad * 8));
    CKR(plan_alloc(pl, &p.sup, (size_t)B * L));
    CKR(plan_alloc(pl, &p.path, (size_t)B * 4));
    CK(cudaFuncSetAttribute(s3fd_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kNmsSmemBytes));
    pl->det = std::move(dw);
    return W2L_OK;
}

// arguments of a detection replay of an S3FD plan (w2l_s3fd_detect_u8)
struct S3fdRun {
    const uint8_t* frames;  // (B, H, W, 3) uint8 on the device
    int reverse;            // 1: frames are RGB
    int max_det;
    float* dets;            // (B, max_det, 5)
    int32_t* counts;        // (B)
    const uint8_t* const* frame_ptrs = nullptr;   // device table of B (H, W, 3) frames, read instead of `frames`
};

static int get_plan(w2l_ctx* ctx, int net, int B, int T, Plan** out, int H = 0, int W = 0) {
    char key[96];
    snprintf(key, sizeof(key), "%d:%d:%d:%d:%d:%d", net, B, T, (int)ctx->keep_all, H, W);
    auto it = ctx->plans.find(key);
    if (it != ctx->plans.end()) { it->second->last_used = ++ctx->plan_clock; *out = it->second.get(); return W2L_OK; }
    if (!ctx->nets[net].loaded) return fail(W2L_ESTATE, "weights of net %d not loaded", net);
    // keep at most a few plans per net alive (activation arenas are large): evict the least recently used one that no
    // streaming session has pinned (a pinned plan is baked into that session's CUDA graph)
    for (;;) {
        int count = 0;
        auto lru = ctx->plans.end();
        for (auto p = ctx->plans.begin(); p != ctx->plans.end(); ++p)
            if (p->second->net == net) {
                ++count;
                if (p->second->pins == 0 && (lru == ctx->plans.end() || p->second->last_used < lru->second->last_used)) lru = p;
            }
        if (count < 6 || lru == ctx->plans.end()) break;
        CK(cudaDeviceSynchronize());  // the plan's buffers may still be in use by queued launches
        if (ctx->last_plan[net] == lru->second.get()) ctx->last_plan[net] = nullptr;
        ctx->plans.erase(lru);
    }
    std::unique_ptr<Plan> pl(new Plan(ctx));
    pl->net = net; pl->B = B; pl->T = T; pl->H = H; pl->W = W;
    pl->x2 = ctx->x2;
    pl->N = (net == W2L_NET_SYNCNET) ? B : (T > 0 ? B * T : B);
    int r = W2L_OK;
    if (net == W2L_NET_GENERATOR) r = build_generator_plan(ctx, pl.get());
    else if (net == W2L_NET_SYNCNET) r = build_syncnet_plan(ctx, pl.get());
    else if (net == W2L_NET_S3FD) r = build_s3fd_plan(ctx, pl.get());
    else r = build_disc_plan(ctx, pl.get());
    CKR(r);
    pl->last_used = ++ctx->plan_clock;
    *out = pl.get();
    ctx->plans[key] = std::move(pl);
    return W2L_OK;
}

static int run_plan(w2l_ctx* ctx, Plan* pl, const void* in0, const void* in1, void* out0, void* out1, cudaStream_t st,
                    bool u8 = false, float* const* outs = nullptr, const S3fdRun* det = nullptr) {
    const bool side = pl->has_side && ctx->use_side;
    cudaStream_t main_st = st;
    if (side) {
        CK(cudaEventRecord(ctx->ev_fork, main_st));
        CK(cudaStreamWaitEvent(ctx->s_side, ctx->ev_fork, 0));
    }
    for (Op& op : pl->ops) {
        if (side && op.join_side) {
            CK(cudaEventRecord(ctx->ev_join, ctx->s_side));
            CK(cudaStreamWaitEvent(main_st, ctx->ev_join, 0));
        }
        st = (side && op.lane == 1) ? ctx->s_side : main_st;
        switch (op.type) {
            case OP_INGEST: {
                if (det) {  // S3FD detection: uint8 frames, mean subtraction (and RGB -> BGR) fused into the ingest
                    S3fdIngestParams sp;
                    sp.src = det->frames; sp.dst = op.ip.dst;
                    sp.N = op.ip.N; sp.H = op.ip.H; sp.W = op.ip.W; sp.Cpad = op.ip.Cpad; sp.Wp = op.ip.Wp; sp.x_off = op.ip.x_off;
                    sp.Cpix = op.ip.Cpix; sp.lo_off = op.ip.lo_off; sp.reverse = det->reverse;
                    sp.srcs = det->frame_ptrs;
                    const long long tot = (long long)sp.N * sp.H * sp.W;
                    const int blk = (int)std::min<long long>((tot + 255) / 256, ctx->num_sms * 16);
                    if (det->frame_ptrs) {
                        if (ctx->bf16) s3fd_ingest_u8_kernel<true, true><<<blk, 256, 0, st>>>(sp);
                        else s3fd_ingest_u8_kernel<false, true><<<blk, 256, 0, st>>>(sp);
                    } else if (ctx->bf16) s3fd_ingest_u8_kernel<true><<<blk, 256, 0, st>>>(sp);
                    else s3fd_ingest_u8_kernel<false><<<blk, 256, 0, st>>>(sp);
                    ctx->launches++;
                    break;
                }
                if (u8 && op.ingest_src == 1) {  // uint8 crops: mask + concat + /255 fused into the ingest
                    IngestU8Params up;
                    up.src = (const unsigned char*)in1; up.dst = op.ip.dst;
                    up.N = op.ip.N; up.H = op.ip.H; up.W = op.ip.W; up.Cpad = op.ip.Cpad; up.Wp = op.ip.Wp; up.x_off = op.ip.x_off; up.lo_off = op.ip.lo_off; up.Cpix = op.ip.Cpix;
                    const long long tot = (long long)up.N * up.H * up.W;
                    const int blk = (int)std::min<long long>((tot + 255) / 256, ctx->num_sms * 16);
                    if (ctx->bf16) ingest_u8_kernel<true><<<blk, 256, 0, st>>>(up);
                    else ingest_u8_kernel<false><<<blk, 256, 0, st>>>(up);
                    ctx->launches++;
                    break;
                }
                CKR(launch_ingest(ctx, op, op.ingest_src == 0 ? in0 : in1, st));
                break;
            }
            case OP_CONV: {
                if (op.head) {
                    op.cp.ep.head_out = u8 ? nullptr : (float*)out0; op.pp.ep.head_out = op.cp.ep.head_out;
                    op.cp.ep.head_out_u8 = u8 ? (unsigned char*)out0 : nullptr; op.pp.ep.head_out_u8 = op.cp.ep.head_out_u8;
                }
                CKR(launch_conv(ctx, op, st));
                break;
            }
            case OP_L2NORM: {
                float* o = (float*)(op.aux_out == 0 ? out0 : out1);
                l2norm_kernel<<<(op.aux_rows + 3) / 4, 128, 0, st>>>((const float*)op.aux_in, o, op.aux_rows, op.aux_dim);
                ctx->launches++;
                break;
            }
            case OP_MAXPOOL: {
                const long long total = (long long)op.sp_N * (op.sp_H / 2) * (op.sp_W / 2) * (op.sp_C / 8);
                const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
                if (ctx->bf16) maxpool2_kernel<true><<<blocks, 256, 0, st>>>(op.sp_in, op.sp_out, op.sp_N, op.sp_H, op.sp_W, op.sp_C, op.aux_pitch, op.aux_lo);
                else maxpool2_kernel<false><<<blocks, 256, 0, st>>>(op.sp_in, op.sp_out, op.sp_N, op.sp_H, op.sp_W, op.sp_C, op.aux_pitch, op.aux_lo);
                ctx->launches++;
                break;
            }
            case OP_CHAN_L2NORM: {
                const long long pixels = (long long)op.sp_N * op.sp_H * op.sp_W;
                if (ctx->bf16) chan_l2norm_kernel<true><<<(unsigned)((pixels + 7) / 8), 256, 0, st>>>(op.sp_in, op.sp_out, op.sp_w, pixels, op.sp_C, op.aux_pitch, op.aux_lo);
                else chan_l2norm_kernel<false><<<(unsigned)((pixels + 7) / 8), 256, 0, st>>>(op.sp_in, op.sp_out, op.sp_w, pixels, op.sp_C, op.aux_pitch, op.aux_lo);
                ctx->launches++;
                break;
            }
            case OP_S3FD_EXPORT: {
                if (!outs && det) break;   // detection without the maps
                if (!outs) return fail(W2L_EINVAL, "S3FD plan needs its 12 output pointers");
                const long long total = (long long)op.sp_N * op.sp_Cout * op.sp_H * op.sp_W;
                const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
                s3fd_export_kernel<<<blocks, 256, 0, st>>>(op.sp_f32, outs[op.aux_out], op.sp_N, op.sp_H, op.sp_W, op.sp_Cout, op.sp_maxout);
                ctx->launches++;
                break;
            }
            case OP_DISC_HEAD: {
                const NetW& nw = ctx->nets[W2L_NET_DISC];
                if (ctx->bf16) disc_head_kernel<true><<<(op.aux_rows + 3) / 4, 128, 0, st>>>((const uint16_t*)op.aux_in, nw.head_w, nw.head_b, (float*)out0, op.aux_rows, op.aux_dim, op.aux_pitch, op.aux_lo);
                else disc_head_kernel<false><<<(op.aux_rows + 3) / 4, 128, 0, st>>>((const uint16_t*)op.aux_in, nw.head_w, nw.head_b, (float*)out0, op.aux_rows, op.aux_dim, op.aux_pitch, op.aux_lo);
                ctx->launches++;
                break;
            }
        }
    }
    if (det) {
        S3fdDetParams p = pl->det->p;
        p.max_det = det->max_det; p.dets = det->dets; p.counts = det->counts;
        const dim3 grid(p.nchunk, p.B);
        s3fd_count_kernel<<<grid, kSelChunk, 0, main_st>>>(p);
        s3fd_select_kernel<<<grid, kSelChunk, 0, main_st>>>(p);
        s3fd_nms_kernel<<<p.B, kNmsThreads, kNmsSmemBytes, main_st>>>(p);
        ctx->launches += 3;
    }
    if (pl->det) pl->det->last = det != nullptr;
    CK(cudaGetLastError());
    ctx->last_plan[pl->net] = pl;
    return W2L_OK;
}
