// w2l_api.cu — the C-ABI of include/w2l.h (libw2l.so).  The host side behind it lives in the host_*.h / host_*.cuh
// headers included below (one translation unit): data model, kernel launch tables, op builders, weight packing, plans,
// mel tables.  No torch, no CPU compute path.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <functional>
#include <initializer_list>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/w2l.h"
#include "aux_kernels.cuh"
#include "conv_igemm.cuh"
#include "conv_patch.cuh"
#include "convt_fused.cuh"
#include "mel.cuh"
#include "netspec.h"
#include "resize.cuh"
#include "s3fd_detect.cuh"
#include "stream.cuh"
#include "train_data.cuh"
#include "train_kernels.cuh"
#include "wgrad.cuh"

using namespace w2l;

#include "host_types.h"
#include "host_launch.cuh"
#include "host_ops.cuh"
#include "host_weights.cuh"
#include "host_plans.cuh"
#include "host_mel_tables.h"
#include "host_train.cuh"
#include "host_stream.cuh"
#include "host_stream_group.cuh"

// ------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int w2l_abi_version(void) { return W2L_ABI_VERSION; }
const char* w2l_last_error(void) { return g_err.c_str(); }

int w2l_net_num_layers(int net) {
    const std::vector<Layer>* L = net_layers(net);
    return L ? (int)L->size() : fail(W2L_EINVAL, "unknown net %d", net);
}

int w2l_net_layer_info(int net, int index, w2l_layer_info* out) {
    const std::vector<Layer>* Ls = net_layers(net);
    if (!Ls || !out || index < 0 || index >= (int)Ls->size()) return fail(W2L_EINVAL, "bad net/index %d/%d", net, index);
    const Layer& L = (*Ls)[index];
    memset(out, 0, sizeof(*out));
    snprintf(out->name, sizeof(out->name), "%s", L.name.c_str());
    out->kind = L.kind; out->cin = L.cin; out->cout = L.cout; out->kh = L.kh; out->kw = L.kw;
    out->sh = L.sh; out->sw = L.sw; out->ph = L.ph; out->pw = L.pw; out->out_pad = L.out_pad; out->residual = L.residual ? 1 : 0;
    out->cout_real = L.cout_real;
    return W2L_OK;
}

/* product's own mel filterbank, dense (80 x 401) fp32, host memory — for the parity tests */
int w2l_mel_basis_host(float* out) {
    if (!out) return fail(W2L_EINVAL, "null output");
    std::vector<float> d;
    build_mel_basis(&d);
    memcpy(out, d.data(), d.size() * 4);
    return W2L_OK;
}

int w2l_create(int device, int precision, w2l_ctx** out) {
    if (!out) return fail(W2L_EINVAL, "null out");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(W2L_ENODEV, "no CUDA device (this library has no CPU path)"); }
    if (device < 0 || device >= ndev) return fail(W2L_EINVAL, "device %d out of range (%d devices)", device, ndev);
    if (precision != W2L_PREC_F16 && precision != W2L_PREC_BF16 && precision != W2L_PREC_F32X) return fail(W2L_EINVAL, "unknown precision %d", precision);
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(W2L_ENODEV, "device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
    if (!get_encode_fn()) return fail(W2L_ENODEV, "cuTensorMapEncodeTiled not found in the driver");
    DeviceGuard g(device);
    std::unique_ptr<w2l_ctx> ctx(new w2l_ctx());   // released here, device current, if anything below fails
    ctx->device = device;
    ctx->bf16 = precision == W2L_PREC_BF16;
    ctx->x2 = precision == W2L_PREC_F32X;
    ctx->num_sms = prop.multiProcessorCount;
    for (Stream* s : {&ctx->stream, &ctx->s_h2d, &ctx->s_d2h, &ctx->s_side}) CKR(s->create());
    for (Event* e : {&ctx->ev_fork, &ctx->ev_join, &ctx->ev_in[0], &ctx->ev_done[0], &ctx->ev_out[0], &ctx->ev_in[1],
                     &ctx->ev_done[1], &ctx->ev_out[1]})
        CKR(e->create());
    CKR(init_mel_tables(ctx.get()));
    {
        // A/B switches, read once per context: W2L_DISABLE_<NAME>=1 turns one specialised path off (tests/test_gpu_variants.py)
        auto enabled = [](const char* name) { const char* v = getenv(name); return !(v && v[0] == '1'); };
        ctx->use_patch = enabled("W2L_DISABLE_HALO");
        ctx->use_fold = enabled("W2L_DISABLE_FOLD");
        ctx->use_fold_s2 = enabled("W2L_DISABLE_FOLDS2");
        ctx->use_mt2 = enabled("W2L_DISABLE_MT2");
        ctx->use_wg_stream = enabled("W2L_DISABLE_WGSTREAM");
        ctx->use_aux_stream = enabled("W2L_DISABLE_AUXSTREAM");
        ctx->use_tma_epi = enabled("W2L_DISABLE_TMAEPI");
        ctx->use_ctfused = enabled("W2L_DISABLE_CTFUSED");
        ctx->use_side = enabled("W2L_DISABLE_SIDESTREAM");
        ctx->use_pdl = enabled("W2L_DISABLE_PDL");
        ctx->use_stream_graph = enabled("W2L_DISABLE_STREAMGRAPH");
        if (ctx->x2) {  // the split-operand mode runs on the generic kernel with the direct epilogue only
            ctx->use_patch = ctx->use_fold = ctx->use_fold_s2 = ctx->use_ctfused = ctx->use_tma_epi = false;
        }
        if (ctx->use_fold) {
            // the folded first layers need a tensor map whose pixel stride (16 B) is smaller than its inner extent
            // (128 B): probe once that the driver encodes such overlapping windows
            Act probe;
            probe.base = (uint16_t*)ctx->mel_tw.p; probe.N = 2; probe.H = 16; probe.W = 16; probe.Cs = 8; probe.C = 64; probe.Wp = 24;
            CUtensorMap tm;
            if (encode_act_map(ctx.get(), &tm, probe, 64, 8, 8, 2, 1, 1, "probe") != W2L_OK) { ctx->use_fold = false; g_err.clear(); }
        }
    }
    *out = ctx.release();
    return W2L_OK;
}

int w2l_destroy(w2l_ctx* ctx) {
    if (!ctx) return W2L_OK;
    DeviceGuard g(ctx->device);
    cudaDeviceSynchronize();
    delete ctx;
    return W2L_OK;
}

int w2l_set_debug(w2l_ctx* ctx, int keep_all_layer_outputs) {
    if (!ctx) return fail(W2L_EINVAL, "null ctx");
    ctx->keep_all = keep_all_layer_outputs != 0;
    return W2L_OK;
}

int w2l_load_weights(w2l_ctx* ctx, int net, int n_tensors, const char* const* names, const void* const* dev_ptrs,
                     const int64_t* numels, void* stream) {
    if (!ctx || !names || !dev_ptrs || !numels) return fail(W2L_EINVAL, "null argument");
    const std::vector<Layer>* Ls = net_layers(net);
    if (!Ls) return fail(W2L_EINVAL, "unknown net %d", net);
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    TensorMap tm;
    for (int i = 0; i < n_tensors; ++i) {
        std::string nm = names[i];
        if (nm.rfind("module.", 0) == 0) nm = nm.substr(7);  // DataParallel-era checkpoints, inference.py:174-175
        tm[nm] = TensorRef{(const float*)dev_ptrs[i], numels[i]};
    }
    CK(cudaDeviceSynchronize());  // queued forwards (asynchronous host submissions included) still read the old weights
    drop_plans(ctx, net);
    NetW& nw = ctx->nets[net];
    nw.loaded = false;
    nw.layers.resize(Ls->size());
    // which blocks see a 1x1 input (GEMM form of the transposed conv): generator decoder stage 1
    for (size_t i = 0; i < Ls->size(); ++i) {
        const Layer& L = (*Ls)[i];
        const float *W, *b, *gm, *be, *m, *v;
        CKR(fetch_block_tensors(tm, L, &W, &b, &gm, &be, &m, &v));
        const bool hw1 = (net == W2L_NET_GENERATOR && L.name == "face_decoder_blocks.1.0");
        // blocks fed directly by the ingest kernel (caller tensors): the only ones with a tiny Cin
        bool first = L.name == "face_encoder_blocks.0.0" || L.name == "audio_encoder.0" || L.name == "face_encoder.0" ||
                     (net == W2L_NET_S3FD && L.name == "conv1_1");
        // the generator's 16->32 stride-2 block reads a dense zero-bordered copy of the first block's output (written by
        // the patch kernel's second TMA store) through the same overlapping-window trick
        if (net == W2L_NET_GENERATOR && L.name == "face_encoder_blocks.1.0" && ctx->use_patch && ctx->use_fold && ctx->use_fold_s2) first = true;
        CKR(load_layer(ctx, &nw.layers[i], L, W, b, gm, be, m, v, hw1, first && ctx->use_fold, nullptr, st));
    }
    if (net == W2L_NET_GENERATOR || net == W2L_NET_DISC) {
        const char* wn = net == W2L_NET_GENERATOR ? "output_block.1.weight" : "binary_pred.0.weight";
        const char* bn = net == W2L_NET_GENERATOR ? "output_block.1.bias" : "binary_pred.0.bias";
        const int64_t wcount = net == W2L_NET_GENERATOR ? 96 : 512, bcount = net == W2L_NET_GENERATOR ? 3 : 1;
        const float *hw, *hb;
        CKR(need(tm, wn, wcount, &hw));
        CKR(need(tm, bn, bcount, &hb));
        CKR(nw.head_w.grow(ctx, wcount * 4));
        CKR(nw.head_b.grow(ctx, bcount * 4));
        CK(cudaMemcpyAsync(nw.head_w, hw, wcount * 4, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(nw.head_b, hb, bcount * 4, cudaMemcpyDeviceToDevice, st));
    }
    if (net == W2L_NET_S3FD) {   // L2Norm weights (net_s3fd.py:12-14, :64-66)
        const char* names3[3] = {"conv3_3_norm.weight", "conv4_3_norm.weight", "conv5_3_norm.weight"};
        const int64_t n3[3] = {256, 512, 512};
        for (int i = 0; i < 3; ++i) {
            const float* w;
            CKR(need(tm, names3[i], n3[i], &w));
            CKR(ctx->s3fd_l2w[i].grow(ctx, 512 * 4));
            CK(cudaMemcpyAsync(ctx->s3fd_l2w[i], w, n3[i] * 4, cudaMemcpyDeviceToDevice, st));
        }
    }
    CK(cudaStreamSynchronize(st));  // the caller may free / mutate the fp32 sources after we return
    nw.loaded = true;
    return W2L_OK;
}

int w2l_generator_forward(w2l_ctx* ctx, const float* mel, const float* face, float* out, int B, int T, void* stream) {
    if (!ctx || !mel || !face || !out) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T < 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_GENERATOR, B, T, &pl));
    return run_plan(ctx, pl, mel, face, out, nullptr, (cudaStream_t)stream);
}

// ---- host-buffer entry points: a two-slot software pipeline over three streams --------------------------------
// Every submission (a whole call, or one chunk of a synchronous call) goes H2D (s_h2d) -> kernels (ctx->stream) ->
// D2H (s_d2h) through device staging slot seq & 1, so the copies of one submission overlap the kernels of its
// neighbours.  At most two submissions are in flight.
static int host_drain(w2l_ctx* ctx, int keep) {
    while (ctx->host_inflight > keep) {
        const long long oldest = ctx->host_seq - ctx->host_inflight;
        CK(cudaEventSynchronize(ctx->ev_out[oldest & 1]));
        ctx->host_inflight--;
    }
    return W2L_OK;
}

static int host_submit(w2l_ctx* ctx, int B, int T, const void* mel_h, size_t mel_bytes, const void* face_h, size_t face_bytes,
                       void* out_h, size_t out_bytes, bool u8) {
    if (ctx->host_inflight >= 2) CKR(host_drain(ctx, 1));
    const int sl = (int)(ctx->host_seq & 1);
    if (ctx->stage[0 + sl].cap < mel_bytes || ctx->stage[2 + sl].cap < face_bytes || ctx->stage[4 + sl].cap < out_bytes) {
        CKR(host_drain(ctx, 0));  // growing a staging buffer frees the old one
        CKR(ctx->stage[0 + sl].grow(ctx, mel_bytes));
        CKR(ctx->stage[2 + sl].grow(ctx, face_bytes));
        CKR(ctx->stage[4 + sl].grow(ctx, out_bytes));
    }
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_GENERATOR, B, T, &pl));
    // (waiting on an event that was never recorded is a no-op)
    CK(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_done[sl], 0));   // the kernels that read staging_in[sl] two submissions ago
    CK(cudaMemcpyAsync(ctx->stage[0 + sl], mel_h, mel_bytes, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(ctx->stage[2 + sl], face_h, face_bytes, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaEventRecord(ctx->ev_in[sl], ctx->s_h2d));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[sl], 0));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_out[sl], 0));   // staging_out[sl] drained
    CKR(run_plan(ctx, pl, ctx->stage[0 + sl], ctx->stage[2 + sl], ctx->stage[4 + sl], nullptr, ctx->stream, u8));
    CK(cudaEventRecord(ctx->ev_done[sl], ctx->stream));
    CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_done[sl], 0));
    CK(cudaMemcpyAsync(out_h, ctx->stage[4 + sl], out_bytes, cudaMemcpyDeviceToHost, ctx->s_d2h));
    CK(cudaEventRecord(ctx->ev_out[sl], ctx->s_d2h));
    ctx->host_seq++;
    ctx->host_inflight++;
    return W2L_OK;
}

// fewer, larger chunks: small batches run the low-resolution layers inefficiently
static int host_chunks(int B) { return B >= 64 ? 2 : 1; }

int w2l_generator_forward_host(w2l_ctx* ctx, const float* mel_h, const float* face_h, float* out_h, int B, int T) {
    if (!ctx || !mel_h || !face_h || !out_h) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T < 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    DeviceGuard g(ctx->device);
    // A synchronous call cuts the batch along B (whole T-windows, so every chunk is itself a legal call) so that the
    // copies of one chunk overlap the kernels of the other.
    const int tt = T > 0 ? T : 1;
    const int cb = (B + host_chunks(B) - 1) / host_chunks(B);
    const size_t per_b_mel = (size_t)tt * 1280 * 4, per_b_face = (size_t)tt * 6 * 9216 * 4, per_b_out = (size_t)tt * 3 * 9216 * 4;
    for (int b0 = 0; b0 < B; b0 += cb) {
        const int bc = std::min(cb, B - b0);
        CKR(host_submit(ctx, bc, T, (const char*)mel_h + b0 * per_b_mel, bc * per_b_mel, (const char*)face_h + b0 * per_b_face,
                        bc * per_b_face, (char*)out_h + b0 * per_b_out, bc * per_b_out, false));
    }
    return host_drain(ctx, 0);
}

int w2l_generator_submit_host(w2l_ctx* ctx, const float* mel_h, const float* face_h, float* out_h, int B, int T) {
    if (!ctx || !mel_h || !face_h || !out_h) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T < 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    DeviceGuard g(ctx->device);
    const size_t n = (size_t)B * (T > 0 ? T : 1);
    return host_submit(ctx, B, T, mel_h, n * 1280 * 4, face_h, n * 6 * 9216 * 4, out_h, n * 3 * 9216 * 4, false);
}

int w2l_generator_submit_u8_host(w2l_ctx* ctx, const float* mel_h, const uint8_t* faces_h, uint8_t* out_h, int N) {
    if (!ctx || !mel_h || !faces_h || !out_h) return fail(W2L_EINVAL, "null argument");
    if (N <= 0) return fail(W2L_EINVAL, "bad batch %d", N);
    DeviceGuard g(ctx->device);
    return host_submit(ctx, N, 0, mel_h, (size_t)N * 1280 * 4, faces_h, (size_t)N * 96 * 96 * 3, out_h, (size_t)N * 96 * 96 * 3, true);
}

int w2l_host_wait(w2l_ctx* ctx, int keep_in_flight) {
    if (!ctx) return fail(W2L_EINVAL, "null argument");
    if (keep_in_flight < 0) keep_in_flight = 0;
    DeviceGuard g(ctx->device);
    return host_drain(ctx, keep_in_flight);
}

int w2l_generator_forward_u8(w2l_ctx* ctx, const float* mel, const uint8_t* faces, uint8_t* out, int N, void* stream) {
    if (!ctx || !mel || !faces || !out) return fail(W2L_EINVAL, "null argument");
    if (N <= 0) return fail(W2L_EINVAL, "bad batch %d", N);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_GENERATOR, N, 0, &pl));
    return run_plan(ctx, pl, mel, faces, out, nullptr, (cudaStream_t)stream, true);
}

int w2l_generator_forward_u8_host(w2l_ctx* ctx, const float* mel_h, const uint8_t* faces_h, uint8_t* out_h, int N) {
    if (!ctx || !mel_h || !faces_h || !out_h) return fail(W2L_EINVAL, "null argument");
    if (N <= 0) return fail(W2L_EINVAL, "bad batch %d", N);
    DeviceGuard g(ctx->device);
    const int cb = (N + host_chunks(N) - 1) / host_chunks(N);
    const size_t per_mel = 1280 * 4, per_face = 96 * 96 * 3, per_out = 96 * 96 * 3;
    for (int b0 = 0; b0 < N; b0 += cb) {
        const int bc = std::min(cb, N - b0);
        CKR(host_submit(ctx, bc, 0, (const char*)mel_h + b0 * per_mel, bc * per_mel, faces_h + b0 * per_face, bc * per_face,
                        out_h + b0 * per_out, bc * per_out, true));
    }
    return host_drain(ctx, 0);
}


// ---- scope row f2: the two cv2.resize calls and the paste around the generator call (inference.py:126, :269-271) ----
static int upload_boxes(w2l_ctx* ctx, const int32_t* boxes, int N, int F, int H, int W, cudaStream_t st) {
    for (int n = 0; n < N; ++n) {
        const int32_t* b = boxes + 5 * n;
        if (b[0] < 0 || b[0] >= F || b[1] < 0 || b[2] > H || b[1] >= b[2] || b[3] < 0 || b[4] > W || b[3] >= b[4])
            return fail(W2L_EINVAL, "box %d = (frame %d, y %d:%d, x %d:%d) is empty or outside the %d frames of %dx%d", n, b[0], b[1], b[2], b[3], b[4], F, H, W);
    }
    CKR(ctx->boxes_dev.grow(ctx, (size_t)N * 5 * 4));
    CK(cudaMemcpyAsync(ctx->boxes_dev, boxes, (size_t)N * 5 * 4, cudaMemcpyHostToDevice, st));
    return W2L_OK;
}

int w2l_crop_resize_u8(w2l_ctx* ctx, const uint8_t* frames, int F, int H, int W, const int32_t* boxes_host, int N, uint8_t* crops,
                       void* stream) {
    if (!ctx || !frames || !boxes_host || !crops) return fail(W2L_EINVAL, "null argument");
    if (F <= 0 || H <= 0 || W <= 0 || N <= 0) return fail(W2L_EINVAL, "bad shape");
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(upload_boxes(ctx, boxes_host, N, F, H, W, st));
    const long long total = (long long)N * 96 * 96;
    crop_resize_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16), 256, 0, st>>>(frames, H, W, ctx->boxes_dev, N, 96, crops);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_paste_u8(w2l_ctx* ctx, const uint8_t* pred, const uint8_t* frames, int F, int H, int W, const int32_t* boxes_host, int N,
                 uint8_t* out_frames, void* stream) {
    if (!ctx || !pred || !frames || !boxes_host || !out_frames) return fail(W2L_EINVAL, "null argument");
    if (F <= 0 || H <= 0 || W <= 0 || N <= 0) return fail(W2L_EINVAL, "bad shape");
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(upload_boxes(ctx, boxes_host, N, F, H, W, st));
    const long long total = (long long)N * H * W;
    paste_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 32), 256, 0, st>>>(pred, 96, frames, H, W, ctx->boxes_dev, N, out_frames);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_lipsync_frames_u8(w2l_ctx* ctx, const float* mel, const uint8_t* frames, int F, int H, int W, const int32_t* boxes_host, int N,
                          uint8_t* out_frames, void* stream) {
    if (!ctx || !mel || !frames || !boxes_host || !out_frames) return fail(W2L_EINVAL, "null argument");
    if (F <= 0 || H <= 0 || W <= 0 || N <= 0) return fail(W2L_EINVAL, "bad shape");
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t cb = (size_t)N * 96 * 96 * 3;
    CKR(ctx->crops_dev.grow(ctx, cb));
    CKR(ctx->preds_dev.grow(ctx, cb));
    CKR(w2l_crop_resize_u8(ctx, frames, F, H, W, boxes_host, N, ctx->crops_dev, stream));
    CKR(w2l_generator_forward_u8(ctx, mel, ctx->crops_dev, ctx->preds_dev, N, stream));
    const long long total = (long long)N * H * W;
    paste_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 32), 256, 0, st>>>(ctx->preds_dev, 96, frames, H, W, ctx->boxes_dev, N, out_frames);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}


// ---- scope row f3: the training scripts' Dataset.__getitem__ + default_collate, one gather per batch ----
// The gather reads the cache through `p` itself: device (or managed) memory of this context's device, or page-locked host
// memory, which unified addressing maps at the same address.  Pageable memory cannot be read by a kernel.
static int train_source(w2l_ctx* ctx, const void* p, const char* what, const void** dev) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(W2L_EINVAL, "%s: cudaPointerGetAttributes: %s", what, cudaGetErrorString(e)); }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
        if (a.type == cudaMemoryTypeDevice && a.device != ctx->device)
            return fail(W2L_EINVAL, "%s is on device %d, the context on device %d", what, a.device, ctx->device);
        *dev = p;
        return W2L_OK;
    }
    if (a.type == cudaMemoryTypeHost && a.devicePointer) { *dev = a.devicePointer; return W2L_OK; }
    return fail(W2L_EINVAL, "%s is pageable host memory: the batch gather reads device or pinned (page-locked) memory only", what);
}

// every row of the host sample table, before anything touches the device
static int check_samples(const int32_t* s, int B, int fields, int n_slots, int mel_at, int n_mel, int label_at,
                         int64_t n_frames, int64_t n_mel_rows) {
    for (int b = 0; b < B; ++b) {
        const int32_t* r = s + (size_t)b * fields;
        for (int k = 0; k < n_slots; ++k)
            if (r[k] < 0 || r[k] >= n_frames) return fail(W2L_EINVAL, "sample %d: frame slot %d is outside the %lld cached frames", b, r[k], (long long)n_frames);
        const int32_t end = r[fields - 1];
        if (end > n_mel_rows) return fail(W2L_EINVAL, "sample %d: video end row %d is past the %lld cached mel rows", b, end, (long long)n_mel_rows);
        for (int k = 0; k < n_mel; ++k)
            if (r[mel_at + k] < 0 || (int64_t)r[mel_at + k] + 16 > end)
                return fail(W2L_EINVAL, "sample %d: mel window at row %d does not end by its video's end row %d", b, r[mel_at + k], end);
        if (label_at >= 0 && r[label_at] != 0 && r[label_at] != 1) return fail(W2L_EINVAL, "sample %d: label %d is not 0 or 1", b, r[label_at]);
    }
    return W2L_OK;
}

// argument checks shared by both entries: host-side ones first (no context needed), then the two cache pointers
static int train_batch_args(w2l_ctx* ctx, const uint8_t* frames, int64_t n_frames, const float* mels, int64_t n_mel_rows,
                            const int32_t* samples, int B, std::initializer_list<const void*> outs, int fields, int n_slots,
                            int mel_at, int n_mel, int label_at, const void** fdev, const void** mdev) {
    if (!frames || !mels || !samples) return fail(W2L_EINVAL, "null argument");
    for (const void* o : outs)
        if (!o || ((uintptr_t)o & 15)) return fail(W2L_EINVAL, "outputs must be non-null and 16-byte aligned");
    if (B <= 0 || n_frames <= 0 || n_mel_rows < 16 || n_mel_rows > INT32_MAX)
        return fail(W2L_EINVAL, "bad batch %d / %lld frames / %lld mel rows", B, (long long)n_frames, (long long)n_mel_rows);
    CKR(check_samples(samples, B, fields, n_slots, mel_at, n_mel, label_at, n_frames, n_mel_rows));
    if (!ctx) return fail(W2L_EINVAL, "null context");
    CKR(train_source(ctx, frames, "frames", fdev));
    return train_source(ctx, mels, "mels", mdev);
}

static int upload_samples(w2l_ctx* ctx, const int32_t* s, size_t n, cudaStream_t st) {
    CKR(ctx->samples_dev.grow(ctx, n * 4));
    CK(cudaMemcpyAsync(ctx->samples_dev, s, n * 4, cudaMemcpyHostToDevice, st));
    return W2L_OK;
}

int w2l_train_batch_wav2lip(w2l_ctx* ctx, const uint8_t* frames, int64_t n_frames, const float* mels, int64_t n_mel_rows,
                            const int32_t* samples_host, int B, float* x, float* indiv_mels, float* mel, float* gt, void* stream) {
    const void *fd = nullptr, *md = nullptr;
    CKR(train_batch_args(ctx, frames, n_frames, mels, n_mel_rows, samples_host, B, {x, indiv_mels, mel, gt},
                         TD_W2L_FIELDS, 10, 10, 6, -1, &fd, &md));
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(upload_samples(ctx, samples_host, (size_t)B * TD_W2L_FIELDS, st));
    const long long total = (long long)B * (2 * 5 * 96 * 24 + 6 * 80 * 4);
    train_batch_wav2lip_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16), 256, 0, st>>>(
        (const uint8_t*)fd, (const float*)md, ctx->samples_dev, B, x, indiv_mels, mel, gt);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_train_batch_syncnet(w2l_ctx* ctx, const uint8_t* frames, int64_t n_frames, const float* mels, int64_t n_mel_rows,
                            const int32_t* samples_host, int B, float* x, float* mel, float* y, void* stream) {
    const void *fd = nullptr, *md = nullptr;
    CKR(train_batch_args(ctx, frames, n_frames, mels, n_mel_rows, samples_host, B, {x, mel, y},
                         TD_SYNC_FIELDS, 5, 5, 1, 6, &fd, &md));
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(upload_samples(ctx, samples_host, (size_t)B * TD_SYNC_FIELDS, st));
    const long long total = (long long)B * (5 * 48 * 24 + 80 * 4);
    train_batch_syncnet_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16), 256, 0, st>>>(
        (const uint8_t*)fd, (const float*)md, ctx->samples_dev, B, x, mel, y);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}


// ---- scope row f4: S3FD network (face_detection/detection/sfd/net_s3fd.py:22-129) ----
int w2l_s3fd_out_dims(int H, int W, int32_t* dims12) {
    if (!dims12 || H < 32 || W < 32) return fail(W2L_EINVAL, "S3FD needs an image of at least 32 x 32");
    int hs[6], ws[6];
    s3fd_dims(H, W, hs, ws);
    for (int i = 0; i < 6; ++i) { dims12[2 * i] = hs[i]; dims12[2 * i + 1] = ws[i]; }
    return W2L_OK;
}

int w2l_s3fd_forward(w2l_ctx* ctx, const float* img, float* const* outs, int B, int H, int W, void* stream) {
    if (!ctx || !img || !outs) return fail(W2L_EINVAL, "null argument");
    for (int i = 0; i < 12; ++i) if (!outs[i]) return fail(W2L_EINVAL, "null output %d", i);
    if (B <= 0 || H < 32 || W < 32) return fail(W2L_EINVAL, "bad shape B=%d H=%d W=%d", B, H, W);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_S3FD, B, 0, &pl, H, W));
    return run_plan(ctx, pl, img, nullptr, nullptr, nullptr, (cudaStream_t)stream, false, outs);
}

int w2l_s3fd_detect_u8(w2l_ctx* ctx, const uint8_t* frames, int B, int H, int W, int reverse_channels, int max_det, float* dets,
                       int32_t* counts, float* const* outs, void* stream) {
    if (!ctx || !frames || !dets || !counts) return fail(W2L_EINVAL, "null argument");
    if (outs)
        for (int i = 0; i < 12; ++i) if (!outs[i]) return fail(W2L_EINVAL, "null output %d", i);
    if (B <= 0 || H < 32 || W < 32) return fail(W2L_EINVAL, "bad shape B=%d H=%d W=%d", B, H, W);
    if (reverse_channels != 0 && reverse_channels != 1) return fail(W2L_EINVAL, "reverse_channels must be 0 or 1");
    if (max_det < 1) return fail(W2L_EINVAL, "max_det must be at least 1, got %d", max_det);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_S3FD, B, 0, &pl, H, W));
    CKR(ensure_s3fd_detect(ctx, pl));
    const S3fdRun run{frames, reverse_channels, max_det, dets, counts};
    return run_plan(ctx, pl, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream, false, outs, &run);
}

int w2l_debug_s3fd_candidates(w2l_ctx* ctx, int image, int cap, float* out, int* n, int* nms_path) {
    if (!ctx) return fail(W2L_EINVAL, "null ctx");
    Plan* pl = ctx->last_plan[W2L_NET_S3FD];
    if (!pl || !pl->det || !pl->det->last) return fail(W2L_ESTATE, "the last S3FD call was not a detection");
    const S3fdDetParams& p = pl->det->p;
    if (image < 0 || image >= p.B) return fail(W2L_EINVAL, "image %d out of range (%d images)", image, p.B);
    if (cap < 0 || (cap > 0 && !out)) return fail(W2L_EINVAL, "bad output buffer");
    DeviceGuard g(ctx->device);
    CK(cudaDeviceSynchronize());
    int cnt = 0, path = 0;
    CK(cudaMemcpy(&cnt, p.ncand + image, 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&path, p.path + image, 4, cudaMemcpyDeviceToHost));
    if (n) *n = cnt;
    if (nms_path) *nms_path = path;
    const int k = std::min(cnt, cap);
    if (k > 0) {
        std::vector<uint64_t> keys(k);
        std::vector<float4> box(cnt);
        std::vector<int> loc(cnt);
        CK(cudaMemcpy(keys.data(), p.keys + (size_t)image * p.Lpad, (size_t)k * 8, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(box.data(), p.cbox + (size_t)image * p.L, (size_t)cnt * 16, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(loc.data(), p.cloc + (size_t)image * p.L, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
        for (int r = 0; r < k; ++r) {
            const uint32_t slot = (uint32_t)keys[r];
            if (slot >= (uint32_t)cnt) return fail(W2L_ESTATE, "sorted candidate %d refers to slot %u of %d", r, slot, cnt);
            const uint32_t sb = (uint32_t)(keys[r] >> 32);
            float sc;
            memcpy(&sc, &sb, 4);
            float* o = out + (size_t)r * 6;
            o[0] = box[slot].x; o[1] = box[slot].y; o[2] = box[slot].z; o[3] = box[slot].w; o[4] = sc; o[5] = (float)loc[slot];
        }
    }
    return W2L_OK;
}

int w2l_syncnet_forward(w2l_ctx* ctx, const float* mel, const float* face, float* a_emb, float* v_emb, int B, void* stream) {
    if (!ctx || !mel || !face || !a_emb || !v_emb) return fail(W2L_EINVAL, "null argument");
    if (B <= 0) return fail(W2L_EINVAL, "bad batch %d", B);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_SYNCNET, B, 0, &pl));
    return run_plan(ctx, pl, mel, face, a_emb, v_emb, (cudaStream_t)stream);
}

int w2l_syncnet_forward_frames(w2l_ctx* ctx, const float* mel, const float* frames, float* a_emb, float* v_emb, int B, int T,
                               void* stream) {
    if (!ctx || !mel || !frames || !a_emb || !v_emb) return fail(W2L_EINVAL, "null argument");
    if (B <= 0) return fail(W2L_EINVAL, "bad batch %d", B);
    if (T != 5) return fail(W2L_EINVAL, "SyncNet_color takes syncnet_T = 5 frames (15 channels), got T=%d", T);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_SYNCNET, B, T, &pl));
    return run_plan(ctx, pl, mel, frames, a_emb, v_emb, (cudaStream_t)stream);
}

int w2l_cosine_bce_loss(w2l_ctx* ctx, const float* a_emb, const float* v_emb, const float* y, int B, int D, float* loss, void* stream) {
    if (!ctx || !a_emb || !v_emb || !loss) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || D <= 0) return fail(W2L_EINVAL, "bad shape B=%d D=%d", B, D);
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(ctx->scratch.grow(ctx, (size_t)std::max(B, 4096) * 4));
    cosine_bce_terms_kernel<<<(B + 3) / 4, 128, 0, st>>>(a_emb, v_emb, y, ctx->scratch, B, D);
    sum_scale_kernel<<<1, 1024, 0, st>>>(ctx->scratch, loss, B, 1.0f / (float)B);
    ctx->launches += 2;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_l1_loss(w2l_ctx* ctx, const float* x, const float* y, int64_t n, float* loss, void* stream) {
    if (!ctx || !x || !y || !loss) return fail(W2L_EINVAL, "null argument");
    if (n <= 0) return fail(W2L_EINVAL, "bad element count");
    if ((((uintptr_t)x) | ((uintptr_t)y)) & 15) return fail(W2L_EINVAL, "inputs must be 16-byte aligned");
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int blocks = (int)std::min<long long>(std::max<long long>((n / 4 + 255) / 256, 1), (long long)ctx->num_sms * 8);
    CKR(ctx->scratch.grow(ctx, (size_t)std::max(blocks, 4096) * 4));
    l1_partial_kernel<<<blocks, 256, 0, st>>>(x, y, ctx->scratch, (long long)n);
    sum_scale_kernel<<<1, 1024, 0, st>>>(ctx->scratch, loss, blocks, (float)(1.0 / (double)n));
    ctx->launches += 2;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_disc_forward(w2l_ctx* ctx, const float* frames, float* prob, int B, int T, void* stream) {
    if (!ctx || !frames || !prob) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T <= 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    DeviceGuard g(ctx->device);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_DISC, B, T, &pl));
    return run_plan(ctx, pl, frames, nullptr, prob, nullptr, (cudaStream_t)stream);
}

// The block of a single-block entry, from the caller's description: every field is checked here, before anything is
// allocated or launched.  Ho / Wo: the output size on an N x H x W input.
static int block_from_info(const w2l_layer_info* spec, const char* name, int N, int H, int W, Layer* L, int* Ho, int* Wo) {
    if (N <= 0 || H <= 0 || W <= 0) return fail(W2L_EINVAL, "bad shape N=%d H=%d W=%d", N, H, W);
    const w2l_layer_info& s = *spec;
    if (s.kind < W2L_BLOCK_CONV_BN_RELU || s.kind > W2L_BLOCK_CONV_RELU) return fail(W2L_EINVAL, "unknown block kind %d", s.kind);
    if (s.cin < 1) return fail(W2L_EINVAL, "cin %d < 1", s.cin);
    if (s.cout <= 0 || s.cout % 16 != 0) return fail(W2L_EINVAL, "cout %d: must be a positive multiple of 16", s.cout);
    if (s.kh < 1 || s.kw < 1 || (long long)s.kh * s.kw > kMaxTaps)
        return fail(W2L_EINVAL, "kernel %dx%d: needs 1 to %d taps", s.kh, s.kw, kMaxTaps);
    if (s.sh < 1 || s.sw < 1) return fail(W2L_EINVAL, "stride %dx%d < 1", s.sh, s.sw);
    if (s.ph < 0 || s.pw < 0 || s.out_pad < 0) return fail(W2L_EINVAL, "negative padding");
    L->name = name;
    L->kind = s.kind; L->cin = s.cin; L->cout = s.cout; L->kh = s.kh; L->kw = s.kw;
    L->sh = s.sh; L->sw = s.sw; L->ph = s.ph; L->pw = s.pw; L->out_pad = s.out_pad; L->residual = s.residual != 0;
    conv_out_dims(*L, H, W, Ho, Wo);
    if (*Ho <= 0 || *Wo <= 0) return fail(W2L_EINVAL, "empty output");
    if (L->residual && (L->cin != L->cout || *Ho != H || *Wo != W)) return fail(W2L_EINVAL, "residual needs same shape");
    return W2L_OK;
}

int w2l_conv_block_forward(w2l_ctx* ctx, const w2l_layer_info* spec, const float* x, int N, int H, int W,
                           const float* weight, const float* bias, const float* bn_w, const float* bn_b,
                           const float* bn_m, const float* bn_v, float* y, void* stream) {
    if (!ctx || !spec || !x || !weight || !y) return fail(W2L_EINVAL, "null argument");
    Layer L;
    int Ho, Wo;
    const std::string name(spec->name, strnlen(spec->name, sizeof(spec->name)));
    CKR(block_from_info(spec, name.empty() ? "block" : name.c_str(), N, H, W, &L, &Ho, &Wo));
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    ctx->last_block_kernels.clear();
    // a private one-block "network" and plan, released on return; a residual is read from the block input, which then
    // stays in the plain NHWC layout
    NetW scratch;
    scratch.layers.resize(1);
    CKR(load_layer(ctx, &scratch.layers[0], L, weight, bias, bn_w, bn_b, bn_m, bn_v, H == 1 && W == 1,
                   ctx->use_fold && !L.residual, nullptr, st));
    Plan pl(ctx);
    pl.net = W2L_NET_DISC; pl.N = N; pl.B = N; pl.T = 0;
    pl.x2 = ctx->x2;
    Act in, out;
    CKR(plan_input_act(&pl, &in, N, H, W, L.cin, scratch.layers[0], L));
    CKR(plan_act(&pl, &out, N, Ho, Wo, L.cout));
    add_ingest(&pl, "ingest.x", IngestSpec{0, N, L.cin, (long long)L.cin * H * W, (long long)H * W, 0, 0, W}, in);
    CKR(emit_block(ctx, &pl, scratch, 0, L, in, out, L.residual ? &in : nullptr));
    for (const Op& op : pl.ops)
        if (op.type == OP_CONV) { ctx->last_block_kernels.emplace_back(); op_kernel_info(ctx, op, &ctx->last_block_kernels.back()); }
    Plan* lp = ctx->last_plan[W2L_NET_DISC];
    const int r = run_plan(ctx, &pl, x, nullptr, nullptr, nullptr, st);  // (pl.net only labels the plan)
    ctx->last_plan[W2L_NET_DISC] = lp;
    CKR(r);
    const long long total = (long long)N * L.cout * Ho * Wo;
    const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
    if (ctx->bf16) export_kernel<true><<<blocks, 256, 0, st>>>(out.base, y, N, Ho, Wo, L.cout, out.Cs, 0, out.lo_off);
    else export_kernel<false><<<blocks, 256, 0, st>>>(out.base, y, N, Ho, Wo, L.cout, out.Cs, 0, out.lo_off);
    ctx->launches++;
    CK(cudaStreamSynchronize(st));
    return W2L_OK;
}

int w2l_debug_kernel_table(int cap, w2l_kernel_info* out) {
    std::vector<w2l_kernel_info> t;
    auto add = [&](int fam, int bn, int bk, int mt, bool head, bool bf16) {
        w2l_kernel_info k;
        memset(&k, 0, sizeof(k));
        k.family = fam; k.bn = bn; k.bk = bk; k.mt = mt; k.head = head ? 1 : 0; k.bf16 = bf16 ? 1 : 0;
        t.push_back(k);
    };
    // one row per (family, BN, BK, MT, head, precision); an instantiation that also has the channel-major form is
    // named "[cm]"
    for (const auto& e : g_conv_kernels)
        if (!e.cm) add(W2L_KFAM_IGEMM, e.BN, e.BK, e.mt, e.head, e.bf16);
    for (const auto& e : g_conv_kernels)
        if (e.cm)
            for (auto& k : t)
                if (k.family == W2L_KFAM_IGEMM && k.bn == e.BN && k.bk == e.BK && k.mt == e.mt && k.head == (e.head ? 1 : 0) &&
                    k.bf16 == (e.bf16 ? 1 : 0))
                    snprintf(k.name, sizeof(k.name), "[cm]");
    for (const auto& e : g_patch_kernels) add(W2L_KFAM_PATCH, e.BN, e.BK, 1, e.head, e.bf16);
    for (const auto& e : g_ct_kernels) add(W2L_KFAM_CONVT_FUSED, kCtBN, e.BK, 1, false, e.bf16);
    if (!out) return (int)t.size();
    const int k = std::min<int>(std::max(cap, 0), (int)t.size());
    for (int i = 0; i < k; ++i) out[i] = t[i];
    return k;
}

int w2l_debug_plan_kernels(w2l_ctx* ctx, int net, int cap, w2l_kernel_info* out) {
    if (!ctx || net < -1 || net > 3) return fail(W2L_EINVAL, "bad argument");
    std::vector<w2l_kernel_info> t;
    if (net < 0) {
        t = ctx->last_block_kernels;
    } else {
        const Plan* pl = ctx->last_plan[net];
        if (!pl) return fail(W2L_ESTATE, "no forward has run for net %d", net);
        for (const Op& op : pl->ops)
            if (op.type == OP_CONV) { t.emplace_back(); op_kernel_info(ctx, op, &t.back()); }
    }
    if (!out) return (int)t.size();
    const int k = std::min<int>(std::max(cap, 0), (int)t.size());
    for (int i = 0; i < k; ++i) out[i] = t[i];
    return k;
}

int w2l_debug_layer_output(w2l_ctx* ctx, int net, int layer, float* y, int* n, int* c, int* h, int* w, void* stream) {
    if (!ctx || net < 0 || net > 3) return fail(W2L_EINVAL, "bad argument");
    Plan* pl = ctx->last_plan[net];
    if (!pl) return fail(W2L_ESTATE, "no forward has run for net %d", net);
    auto it = pl->layer_out.find(layer);
    if (it == pl->layer_out.end()) return fail(W2L_EINVAL, "layer %d has no materialised output (fused head?)", layer);
    const Act& a = it->second;
    if (n) *n = a.N;
    if (c) *c = a.C;
    if (h) *h = a.H;
    if (w) *w = a.W;
    if (!y) return W2L_OK;
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)a.N * a.C * a.H * a.W;
    const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
    const uint16_t* src = a.f32 ? (const uint16_t*)((const float*)a.base + a.c_off) : a.ptr();
    if (ctx->bf16) export_kernel<true><<<blocks, 256, 0, st>>>(src, y, a.N, a.H, a.W, a.C, a.Cs, a.f32 ? 1 : 0, a.f32 ? 0 : a.lo_off);
    else export_kernel<false><<<blocks, 256, 0, st>>>(src, y, a.N, a.H, a.W, a.C, a.Cs, a.f32 ? 1 : 0, a.f32 ? 0 : a.lo_off);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int64_t w2l_mel_num_frames(int64_t n_samples) { return n_samples < 0 ? 0 : 1 + n_samples / MEL_HOP; }

int w2l_melspectrogram(w2l_ctx* ctx, const float* wav, int64_t n_samples, float* mel, void* stream) {
    if (!ctx || !wav || !mel) return fail(W2L_EINVAL, "null argument");
    if (n_samples < 2) return fail(W2L_EINVAL, "need at least 2 samples (got %lld)", (long long)n_samples);
    DeviceGuard g(ctx->device);
    MelParams p;
    p.wav = wav; p.L = n_samples; p.mel = mel; p.F = w2l_mel_num_frames(n_samples);
    p.tw = ctx->mel_tw; p.bvals = ctx->mel_bvals; p.boff = ctx->mel_boff; p.bstart = ctx->mel_bstart; p.blen = ctx->mel_blen;
    const long long blocks = (p.F + MEL_FPB - 1) / MEL_FPB;
    mel_kernel<<<(unsigned)blocks, MEL_THREADS, kMelSmemBytes, (cudaStream_t)stream>>>(p);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_melspectrogram_host(w2l_ctx* ctx, const float* wav_h, int64_t n_samples, float* mel_h) {
    if (!ctx || !wav_h || !mel_h) return fail(W2L_EINVAL, "null argument");
    if (n_samples < 2) return fail(W2L_EINVAL, "need at least 2 samples (got %lld)", (long long)n_samples);
    DeviceGuard g(ctx->device);
    CKR(host_drain(ctx, 0));  // the staging buffers below are slot 0 of the asynchronous host pipeline
    const int64_t F = w2l_mel_num_frames(n_samples);
    CKR(ctx->stage[0].grow(ctx, (size_t)n_samples * 4));
    CKR(ctx->stage[4].grow(ctx, (size_t)F * MEL_BANDS * 4));
    CK(cudaMemcpyAsync(ctx->stage[0], wav_h, (size_t)n_samples * 4, cudaMemcpyHostToDevice, ctx->stream));
    CKR(w2l_melspectrogram(ctx, (const float*)ctx->stage[0].p, n_samples, (float*)ctx->stage[4].p, ctx->stream));
    CK(cudaMemcpyAsync(mel_h, ctx->stage[4], (size_t)F * MEL_BANDS * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return W2L_OK;
}

int64_t w2l_mel_num_chunks(int64_t n_frames, double fps) {
    if (n_frames < 16 || !(fps > 0)) return 0;
    const double mult = 80.0 / fps;  // inference.py:232
    int64_t i = 0;
    while ((int64_t)((double)i * mult) + 16 <= n_frames) ++i;  // :235-239: the first i that overruns becomes the last chunk
    return i + 1;
}

int w2l_mel_chunks(w2l_ctx* ctx, const float* mel, int64_t n_frames, double fps, float* chunks, int64_t n_chunks, void* stream) {
    if (!ctx || !mel || !chunks) return fail(W2L_EINVAL, "null argument");
    if (n_frames < 16) return fail(W2L_EINVAL, "mel shorter than one 16-frame chunk");
    if (n_chunks != w2l_mel_num_chunks(n_frames, fps)) return fail(W2L_EINVAL, "n_chunks %lld does not match w2l_mel_num_chunks = %lld", (long long)n_chunks, (long long)w2l_mel_num_chunks(n_frames, fps));
    DeviceGuard g(ctx->device);
    const long long total = (long long)n_chunks * 1280;
    const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
    mel_chunk_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(mel, n_frames, 80.0 / fps, (int)n_chunks, chunks);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int w2l_f16_overflow(w2l_ctx* ctx, int clear, int* flag, void* stream) {
    if (!ctx || !flag) return fail(W2L_EINVAL, "null argument");
    DeviceGuard g(ctx->device);
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    CK(cudaStreamSynchronize(ctx->s_side));
    CK(cudaStreamSynchronize(ctx->stream));
    int v = 0;
    CK(cudaMemcpyFromSymbol(&v, g_f16_overflow, sizeof(int)));
    *flag = v;
    if (clear && v) { const int z = 0; CK(cudaMemcpyToSymbol(g_f16_overflow, &z, sizeof(int))); }
    return W2L_OK;
}


// ================================================================================================
// training (SURVEY.md section 8 f1)
// ================================================================================================
int w2l_train_bind(w2l_ctx* ctx, int net, int n_tensors, const char* const* names, void* const* value_ptrs, void* const* grad_ptrs,
                   const int64_t* numels) {
    if (!ctx || !names || !value_ptrs || !numels) return fail(W2L_EINVAL, "null argument");
    if (net < 0 || net > 2) return fail(W2L_EINVAL, "unknown net %d", net);
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    CK(cudaDeviceSynchronize());
    // plans bake the bound pointers: drop the ones of this net
    for (auto it = ts->plans.begin(); it != ts->plans.end();) {
        if (it->second->net == net) it = ts->plans.erase(it);
        else ++it;
    }
    ts->last[net] = nullptr;
    ts->adam[net] = AdamSlot();
    ts->bound[net].clear();
    for (int i = 0; i < n_tensors; ++i) {
        std::string nm = names[i];
        if (nm.rfind("module.", 0) == 0) nm = nm.substr(7);
        ts->bound[net][nm] = ParamRef{(float*)value_ptrs[i], grad_ptrs ? (float*)grad_ptrs[i] : nullptr, (long long)numels[i]};
    }
    ts->is_bound[net] = true;
    return ensure_train_scratch(ctx, 1, 1);
}

int w2l_train_forward(w2l_ctx* ctx, int net, const float* in0, const float* in1, float* out0, float* out1, int B, int T, int flags,
                      void* stream) {
    if (!ctx || !in0 || !out0) return fail(W2L_EINVAL, "null argument");
    if (net < 0 || net > 2 || B <= 0 || T < 0) return fail(W2L_EINVAL, "bad argument net=%d B=%d T=%d", net, B, T);
    if (net != W2L_NET_DISC && !in1) return fail(W2L_EINVAL, "null argument");
    if (net == W2L_NET_SYNCNET && (!out1 || (T != 0 && T != 5))) return fail(W2L_EINVAL, "SyncNet_color: T must be 0 (stacked faces) or 5 (frames)");
    if (net == W2L_NET_DISC && T <= 0) return fail(W2L_EINVAL, "Wav2Lip_disc_qual takes (B,3,T,96,96)");
    DeviceGuard g(ctx->device);
    TrainPlan* tp;
    const bool wg = net == W2L_NET_GENERATOR ? true : (flags & TRAIN_WGRAD) != 0;
    const bool ig = net == W2L_NET_GENERATOR ? false : (flags & TRAIN_INPUT_GRAD) != 0;
    CKR(get_train_plan(ctx, net, B, T, wg, ig, &tp));
    return train_forward(ctx, tp, in0, in1, out0, out1, flags, (cudaStream_t)stream);
}

int w2l_train_backward(w2l_ctx* ctx, int net, const float* d0, const float* d1, float* dinput, int flags, void* stream) {
    if (!ctx || !d0) return fail(W2L_EINVAL, "null argument");
    if (net < 0 || net > 2) return fail(W2L_EINVAL, "unknown net %d", net);
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    TrainPlan* tp = ts->last[net];
    if (!tp) return fail(W2L_ESTATE, "backward of net %d before a training forward", net);
    cudaStream_t st = (cudaStream_t)stream;
    if (net == W2L_NET_SYNCNET && !d1) return fail(W2L_EINVAL, "null argument");
    if (dinput && !tp->input_grad) return fail(W2L_ESTATE, "the forward was not run with W2L_TRAIN_INPUT_GRAD");
    flags &= TRAIN_WGRAD | TRAIN_ACCUMULATE | TRAIN_INPUT_GRAD | TRAIN_NO_STAT_UPDATE;   // (the fused steps' own passes are internal)
    if (net == W2L_NET_GENERATOR) flags |= TRAIN_WGRAD;
    CKR(train_backward(ctx, tp, d0, d1, flags, st));
    if (dinput) {
        if (net == W2L_NET_SYNCNET && tp->T == 0) {
            const long long total = (long long)tp->N * 15 * 48 * 96;
            const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
            export_grad_kernel<true><<<blocks, 256, 0, st>>>(tp->dface_in.ptr(), tp->dface_in.Cs, dinput, tp->N, 48, 96, 15);
        } else {
            GenLossGradParams lp;
            memset(&lp, 0, sizeof(lp));
            lp.dg = dinput; lp.B = tp->B; lp.T = tp->T;
            if (net == W2L_NET_SYNCNET) lp.dsync = tp->dface_in.ptr(); else lp.ddisc = tp->dframes_in.ptr();
            const long long total = (long long)tp->B * 3 * tp->T * 9216;
            const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
            gen_loss_grad_kernel<true><<<blocks, 256, 0, st>>>(lp);
        }
        ctx->launches++;
        CK(cudaGetLastError());
    }
    return W2L_OK;
}

int w2l_adam_step(w2l_ctx* ctx, int net, float lr, float beta1, float beta2, float eps, void* stream) {
    if (!ctx || net < 0 || net > 2) return fail(W2L_EINVAL, "bad argument");
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    if (!ts->is_bound[net]) return fail(W2L_ESTATE, "adam: net %d is not bound", net);
    return adam_step(ctx, net, lr, beta1, beta2, eps, 1.0f, (cudaStream_t)stream);
}

int w2l_comm_unique_id(w2l_ctx* ctx, char* id128) {
    if (!ctx || !id128) return fail(W2L_EINVAL, "null argument");
    TrainState* ts = train_state(ctx);
    NcclGetUniqueIdFn f = (NcclGetUniqueIdFn)nccl_sym(ts, "ncclGetUniqueId");
    if (!f) return fail(W2L_ENODEV, "NCCL not found in the process (libnccl.so.2)");
    const int rc = f(id128);
    if (rc != 0) return fail(W2L_ECUDA, "ncclGetUniqueId failed (%d)", rc);
    return W2L_OK;
}

int w2l_comm_init(w2l_ctx* ctx, const char* id128, int rank, int world) {
    if (!ctx || !id128 || world < 1 || rank < 0 || rank >= world) return fail(W2L_EINVAL, "bad argument");
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    if (ts->comm) return fail(W2L_ESTATE, "communicator already initialised");
    ts->rank = rank; ts->world = world;
    if (world == 1) return W2L_OK;
    NcclCommInitRankFn init = (NcclCommInitRankFn)nccl_sym(ts, "ncclCommInitRank");
    ts->all_reduce = (NcclAllReduceFn)nccl_sym(ts, "ncclAllReduce");
    ts->comm_destroy = (NcclCommDestroyFn)nccl_sym(ts, "ncclCommDestroy");
    ts->err_string = (NcclGetErrorStringFn)nccl_sym(ts, "ncclGetErrorString");
    if (!init || !ts->all_reduce) return fail(W2L_ENODEV, "NCCL not found in the process (libnccl.so.2)");
    NcclId id;
    memcpy(id.bytes, id128, 128);
    const int rc = init(&ts->comm, world, id, rank);
    if (rc != 0) { ts->comm = nullptr; return fail(W2L_ECUDA, "ncclCommInitRank failed: %s", ts->err_string ? ts->err_string(rc) : "?"); }
    CKR(ts->s_comm.create());
    CKR(ts->ev_bucket.create());
    CKR(ts->ev_comm.create());
    return W2L_OK;
}

// get_sync_loss (wav2lip_train.py:192-198) on the generator output of the step, and its input gradient scaled by
// syncnet_wt (sp->dface_in); the scripts leave the frozen expert in train mode (:187-189): batch statistics, running
// averages move
static int sync_loss_grad(w2l_ctx* ctx, TrainPlan* sp, const float* mel, int B, float syncnet_wt, float* loss, cudaStream_t st) {
    TrainState* ts = train_state(ctx);
    CKR(train_forward(ctx, sp, mel, ts->g_buf, ts->a_emb, ts->v_emb, 0, st));
    CKR(w2l_cosine_bce_loss(ctx, ts->a_emb, ts->v_emb, nullptr, B, 512, loss, st));
    cosine_bce_bwd_kernel<<<(B + 3) / 4, 128, 0, st>>>(ts->a_emb, ts->v_emb, nullptr, syncnet_wt, ts->da, ts->dv, B, 512);
    ctx->launches++;
    return train_backward(ctx, sp, ts->da, ts->dv, 0, st);
}

/* one iteration of wav2lip_train.py:210-231 on the bound generator (+ frozen expert), everything on `stream` */
int w2l_wav2lip_train_step(w2l_ctx* ctx, const float* indiv_mels, const float* x, const float* mel, const float* gt, int B, int T,
                           float syncnet_wt, float lr, float* losses_dev, void* stream) {
    if (!ctx || !indiv_mels || !x || !gt) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T <= 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    if (syncnet_wt > 0.0f && (!mel || T != 5)) return fail(W2L_EINVAL, "the sync loss needs mel and T == 5 (syncnet_T)");
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(ensure_train_scratch(ctx, B, T));
    TrainPlan *gp, *sp = nullptr;
    CKR(get_train_plan(ctx, W2L_NET_GENERATOR, B, T, true, false, &gp));
    if (syncnet_wt > 0.0f) CKR(get_train_plan(ctx, W2L_NET_SYNCNET, B, T, false, true, &sp));
    float* L = ts->loss_dev;   // [0] sync, [1] l1, [2] perceptual, [3] total
    CK(cudaMemsetAsync(L, 0, 4 * 4, st));
    CKR(train_forward(ctx, gp, indiv_mels, x, ts->g_buf, nullptr, 0, st));
    const long long numel = (long long)B * 3 * T * 9216;
    GenLossGradParams lp;
    memset(&lp, 0, sizeof(lp));
    if (sp) {
        CKR(sync_loss_grad(ctx, sp, mel, B, syncnet_wt, L + 0, st));
        lp.dsync = sp->dface_in.ptr();
    }
    CKR(w2l_l1_loss(ctx, ts->g_buf, gt, numel, L + 1, st));
    lp.g = ts->g_buf; lp.gt = gt; lp.dg = ts->dg_buf; lp.l1_scale = (1.0f - syncnet_wt) / (float)numel; lp.B = B; lp.T = T;
    {
        const int blocks = (int)std::min<long long>((numel + 255) / 256, ctx->num_sms * 16);
        gen_loss_grad_kernel<true><<<blocks, 256, 0, st>>>(lp);
        ctx->launches++;
    }
    CKR(generator_backward_dp(ctx, gp, ts->dg_buf, st));
    CKR(adam_step(ctx, W2L_NET_GENERATOR, lr, 0.9f, 0.999f, 1e-8f, 1.0f, st));
    combine_losses_kernel<<<1, 32, 0, st>>>(L, syncnet_wt, 0.0f);
    ctx->launches++;
    if (losses_dev) CK(cudaMemcpyAsync(losses_dev, L, 4 * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return W2L_OK;
}

/* one iteration of hq_wav2lip_train.py:212-256 on the bound generator, (frozen) expert and discriminator.
 *
 * The discriminator runs forward twice, on g (plan with input gradient) and on gt: disc(g.detach()) at :252 is the
 * value disc(g) had at :233 (same weights — disc_optimizer.step() comes at :256 — same input, no BatchNorm or dropout),
 * so the g tape serves two backward passes: the perceptual one (input gradient only; :246 zeroes the disc gradients it
 * would make) and the fake term's (parameter gradients added to the real term's, no input gradient).  The two passes share
 * the plan's gradient buffers, so they are ordered on the main stream: the perceptual pass first, then the discriminator's
 * step (real pass, fake pass, all-reduce, Adam) forks onto its own stream and runs beside the generator's backward and
 * Adam; the caller's stream joins it before the losses are final (and so before the next step repacks the disc slabs). */
int w2l_hq_wav2lip_train_step(w2l_ctx* ctx, const float* indiv_mels, const float* x, const float* mel, const float* gt, int B, int T,
                              float syncnet_wt, float disc_wt, float lr, float disc_lr, float* losses_dev, void* stream) {
    if (!ctx || !indiv_mels || !x || !gt) return fail(W2L_EINVAL, "null argument");
    if (B <= 0 || T <= 0) return fail(W2L_EINVAL, "bad batch B=%d T=%d", B, T);
    if (!(syncnet_wt >= 0.0f) || !(disc_wt >= 0.0f)) return fail(W2L_EINVAL, "loss weights must be >= 0 (syncnet_wt %g, disc_wt %g)", syncnet_wt, disc_wt);
    if (syncnet_wt > 0.0f && (!mel || T != 5)) return fail(W2L_EINVAL, "the sync loss needs mel and T == 5 (syncnet_T)");
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    if (!ts->is_bound[W2L_NET_DISC]) return fail(W2L_ESTATE, "hq step: the discriminator is not bound (w2l_train_bind, W2L_NET_DISC)");
    cudaStream_t st = (cudaStream_t)stream;
    CKR(ensure_train_scratch(ctx, B, T));
    TrainPlan *gp, *sp = nullptr, *dg, *dr;
    CKR(get_train_plan(ctx, W2L_NET_GENERATOR, B, T, true, false, &gp));
    if (syncnet_wt > 0.0f) CKR(get_train_plan(ctx, W2L_NET_SYNCNET, B, T, false, true, &sp));
    CKR(get_train_plan(ctx, W2L_NET_DISC, B, T, true, true, &dg));    // on g: input gradient (perceptual) + wgrad (fake term)
    CKR(get_train_plan(ctx, W2L_NET_DISC, B, T, true, false, &dr));   // on gt: wgrad (real term)
    const int N = B * T;
    float* L = ts->loss_dev;   // [0] sync, [1] l1, [2] perceptual, [3] total, [4] disc real, [5] disc fake
    float *p_fake = ts->prob, *p_real = ts->prob + N;
    float *d_perc = ts->dprob, *d_fake = ts->dprob + N, *d_real = ts->dprob + 2 * N;
    CK(cudaMemsetAsync(L, 0, 6 * 4, st));
    CKR(train_forward(ctx, gp, indiv_mels, x, ts->g_buf, nullptr, 0, st));
    const long long numel = (long long)B * 3 * T * 9216;
    GenLossGradParams lp;
    memset(&lp, 0, sizeof(lp));
    if (sp) {
        CKR(sync_loss_grad(ctx, sp, mel, B, syncnet_wt, L + 0, st));
        lp.dsync = sp->dface_in.ptr();
    }
    CKR(train_forward(ctx, dg, ts->g_buf, nullptr, p_fake, nullptr, 0, st));
    CKR(train_forward(ctx, dr, gt, nullptr, p_real, nullptr, 0, st));
    disc_bce_kernel<<<1, 1024, 0, st>>>(p_fake, p_real, N, disc_wt, L, d_perc, d_fake, d_real);
    ctx->launches++;
    if (disc_wt > 0.0f) {   // perceptual_forward (wav2lip.py:163-174) backward: dL/dg through the disc, no disc gradients
        CKR(train_backward(ctx, dg, d_perc, nullptr, 0, st));
        lp.ddisc = dg->dframes_in.ptr();
    }
    // ---- the discriminator's step (:245-256) on its own lane ----
    cudaStream_t sd = st;
    if (ctx->use_aux_stream) {
        CKR(ensure_disc_stream(ts));
        sd = ts->s_disc;
        CK(cudaEventRecord(ts->ev_disc_fork, st));
        CK(cudaStreamWaitEvent(sd, ts->ev_disc_fork, 0));
    }
    CKR(train_backward(ctx, dr, d_real, nullptr, TRAIN_WGRAD | TRAIN_ONE_STREAM, sd));
    CKR(train_backward(ctx, dg, d_fake, nullptr, TRAIN_WGRAD | TRAIN_ACCUMULATE | TRAIN_SKIP_INPUT_GRAD | TRAIN_ONE_STREAM, sd));
    // ---- the generator's backward and Adam (:242-243) on the caller's stream ----
    CKR(w2l_l1_loss(ctx, ts->g_buf, gt, numel, L + 1, st));
    // dL/dg of the L1 term in autograd's operation order — the weight (1 - syncnet_wt - disc_wt, formed in double as the
    // script's Python floats are, rounded once) times the mean's reciprocal 1/numel, times sign(g - gt) — so that with
    // syncnet_wt = 0 the generator's gradient equals the script's loss.backward() bit for bit
    const float wt_l1 = (float)(1.0 - (double)syncnet_wt - (double)disc_wt);
    lp.g = ts->g_buf; lp.gt = gt; lp.dg = ts->dg_buf; lp.l1_scale = wt_l1 * (1.0f / (float)numel); lp.B = B; lp.T = T;
    {
        const int blocks = (int)std::min<long long>((numel + 255) / 256, ctx->num_sms * 16);
        gen_loss_grad_kernel<true><<<blocks, 256, 0, st>>>(lp);
        ctx->launches++;
    }
    CKR(generator_backward_dp(ctx, gp, ts->dg_buf, st));
    CKR(adam_step(ctx, W2L_NET_GENERATOR, lr, 0.5f, 0.999f, 1e-8f, 1.0f, st));   // :421-422
    // the discriminator's bucket goes to the communication stream AFTER the generator's three, so that none of those waits
    // for the discriminator's backward; its Adam waits for it (last_allreduce_bytes, reset by the generator's backward,
    // ends as this step's total)
    if (ts->world > 1 && ts->comm) {
        CKR(all_reduce_ranges(ctx, bucket_ranges(ts, W2L_NET_DISC, {""}), sd));
        CKR(join_comm(ctx, sd));
    }
    CKR(adam_step(ctx, W2L_NET_DISC, disc_lr, 0.5f, 0.999f, 1e-8f, 1.0f, sd));   // hq_wav2lip_train.py:423-424
    if (sd != st) {
        CK(cudaEventRecord(ts->ev_disc_join, sd));
        CK(cudaStreamWaitEvent(st, ts->ev_disc_join, 0));
    }
    combine_losses_kernel<<<1, 32, 0, st>>>(L, syncnet_wt, disc_wt);
    ctx->launches++;
    if (losses_dev) CK(cudaMemcpyAsync(losses_dev, L, 6 * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return W2L_OK;
}

/* one iteration of color_syncnet_train.py:149-163 on the bound expert, everything on `stream` (the audio encoder on the
 * auxiliary lane) */
int w2l_syncnet_train_step(w2l_ctx* ctx, const float* mel, const float* x, const float* y, int B, float lr, float* loss_dev, void* stream) {
    if (!ctx || !mel || !x || !y) return fail(W2L_EINVAL, "null argument");
    if (B <= 0) return fail(W2L_EINVAL, "bad batch B=%d", B);
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(ensure_train_scratch(ctx, B, 0));
    TrainPlan* sp;
    CKR(get_train_plan(ctx, W2L_NET_SYNCNET, B, 0, true, false, &sp));
    float* L = ts->loss_dev;
    CKR(train_forward(ctx, sp, mel, x, ts->a_emb, ts->v_emb, 0, st));
    CKR(w2l_cosine_bce_loss(ctx, ts->a_emb, ts->v_emb, y, B, 512, L, st));
    cosine_bce_bwd_kernel<<<(B + 3) / 4, 128, 0, st>>>(ts->a_emb, ts->v_emb, y, 1.0f, ts->da, ts->dv, B, 512);
    ctx->launches++;
    if (ts->world > 1 && ts->comm) {
        // two buckets in the order the backward completes them: the face encoder (main stream), then the audio encoder
        // (auxiliary lane, joined at the last block)
        size_t k_face = 0;
        for (size_t k = 0; k < sp->blocks.size(); ++k)
            if (sp->blocks[k].lane == 0) { k_face = k; break; }
        const std::vector<GradRange> rf = bucket_ranges(ts, W2L_NET_SYNCNET, {"face_encoder."});
        const std::vector<GradRange> ra = bucket_ranges(ts, W2L_NET_SYNCNET, {"audio_encoder."});
        ts->last_allreduce_bytes = 0;
        std::function<int(size_t)> hook = [&](size_t k) -> int {
            if (k == k_face) return all_reduce_ranges(ctx, rf, st);
            if (k == 0) return all_reduce_ranges(ctx, ra, st);
            return W2L_OK;
        };
        CKR(train_backward(ctx, sp, ts->da, ts->dv, TRAIN_WGRAD, st, &hook));
        CKR(join_comm(ctx, st));
    } else {
        CKR(train_backward(ctx, sp, ts->da, ts->dv, TRAIN_WGRAD, st));
    }
    CKR(adam_step(ctx, W2L_NET_SYNCNET, lr, 0.9f, 0.999f, 1e-8f, 1.0f, st));   // color_syncnet_train.py:270-271
    if (loss_dev) CK(cudaMemcpyAsync(loss_dev, L, 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return W2L_OK;
}

/* Adam moments and step count of named bound tensors of `net`, out of the context (direction 0) or into it (1). */
int w2l_adam_state(w2l_ctx* ctx, int net, int direction, int n, const char* const* names, float* const* m_ptrs, float* const* v_ptrs,
                   int64_t* step, void* stream) {
    if (!ctx || !step || (n > 0 && (!names || !m_ptrs || !v_ptrs))) return fail(W2L_EINVAL, "null argument");
    if (net < 0 || net > 2 || n < 0 || (direction != 0 && direction != 1)) return fail(W2L_EINVAL, "bad argument net=%d n=%d direction=%d", net, n, direction);
    if (direction == 1 && *step < 0) return fail(W2L_EINVAL, "negative step count %lld", (long long)*step);
    DeviceGuard g(ctx->device);
    TrainState* ts = train_state(ctx);
    if (!ts->is_bound[net]) return fail(W2L_ESTATE, "adam state: net %d is not bound", net);
    cudaStream_t st = (cudaStream_t)stream;
    CKR(ensure_adam_slot(ctx, net, st));
    AdamSlot& a = ts->adam[net];
    std::vector<size_t> idx((size_t)n);
    for (int i = 0; i < n; ++i) {   // resolve every name before anything is copied
        if (!names[i] || !m_ptrs[i] || !v_ptrs[i]) return fail(W2L_EINVAL, "null argument");
        std::string nm = names[i];
        if (nm.rfind("module.", 0) == 0) nm = nm.substr(7);
        auto it = std::lower_bound(a.names.begin(), a.names.end(), nm);
        if (it == a.names.end() || *it != nm) return fail(W2L_EINVAL, "adam state: '%s' is not a bound tensor with a gradient", nm.c_str());
        idx[i] = (size_t)(it - a.names.begin());
    }
    for (int i = 0; i < n; ++i) {
        const AdamTensor& t = a.host[idx[i]];
        const size_t bytes = (size_t)t.n * 4;
        if (direction == 0) {
            CK(cudaMemcpyAsync(m_ptrs[i], t.m, bytes, cudaMemcpyDeviceToDevice, st));
            CK(cudaMemcpyAsync(v_ptrs[i], t.v, bytes, cudaMemcpyDeviceToDevice, st));
        } else {
            CK(cudaMemcpyAsync(t.m, m_ptrs[i], bytes, cudaMemcpyDeviceToDevice, st));
            CK(cudaMemcpyAsync(t.v, v_ptrs[i], bytes, cudaMemcpyDeviceToDevice, st));
        }
    }
    if (direction == 0) *step = (int64_t)a.step;
    else a.step = (long long)*step;
    return W2L_OK;
}

/* generator output of the last fused step (B,3,T,96,96) fp32, device pointer owned by the context (tests / logging) */
int w2l_train_last_output(w2l_ctx* ctx, float* out, int64_t n, void* stream) {
    if (!ctx || !out || !ctx->train || !ctx->train->g_buf) return fail(W2L_ESTATE, "no fused training step has run");
    if (n <= 0 || (size_t)n > ctx->train->g_buf.cap / 4) return fail(W2L_EINVAL, "bad element count");
    DeviceGuard g(ctx->device);
    CK(cudaMemcpyAsync(out, ctx->train->g_buf, (size_t)n * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return W2L_OK;
}

double w2l_train_flops(w2l_ctx* ctx, int net) {
    if (!ctx || !ctx->train || net < 0 || net > 2 || !ctx->train->last[net]) return 0.0;
    return ctx->train->last[net]->fwd_flops;
}


/* Per-stage CUDA-event times of the last training plan of `net` (after a forward + backward have run, so every buffer holds
 * real data): for each block "<name> fwd / stats+apply / bwd_bn / dgrad / wgrad", `iters` back-to-back repetitions each.
 * Returns the number of rows written (<= cap). */
int w2l_train_profile(w2l_ctx* ctx, int net, int iters, int cap, float* ms_out, double* flop_out, char (*names_out)[64], void* stream) {
    if (!ctx || net < 0 || net > 2 || iters <= 0 || !ctx->train) return fail(W2L_EINVAL, "bad argument");
    TrainPlan* tp = ctx->train->last[net];
    if (!tp) return fail(W2L_ESTATE, "no training forward has run for net %d", net);
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    Event e0, e1;
    CKR(e0.create(cudaEventDefault));
    CKR(e1.create(cudaEventDefault));
    int k = 0;
    auto timed = [&](const std::string& name, double flops, const std::function<int()>& fn) -> int {
        if (k >= cap) return W2L_OK;
        CKR(fn());
        CK(cudaEventRecord(e0, st));
        for (int i = 0; i < iters; ++i) CKR(fn());
        CK(cudaEventRecord(e1, st));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms_out) ms_out[k] = ms / iters;
        if (flop_out) flop_out[k] = flops;
        if (names_out) snprintf(names_out[k], 64, "%s", name.c_str());
        ++k;
        return W2L_OK;
    };
    for (TBlock& b : tp->blocks) {
        double f = 0;
        for (size_t i = b.fwd0; i < b.fwd1; ++i) f += tp->pl.ops[i].flops;
        // forward conv only, then the statistics + normalise passes (running averages untouched)
        CKR(timed(b.L.name + " fwd", f, [&]() -> int { for (size_t i = b.fwd0; i < b.fwd1; ++i) CKR(launch_conv(ctx, tp->pl.ops[i], st, false)); return W2L_OK; }));
        if (b.bn) {
            TBlock c = b; c.fwd0 = c.fwd1 = 0;
            CKR(timed(b.L.name + " bn", 0, [&]() -> int { return block_forward(ctx, tp, c, false, st); }));
        }
        {
            TBlock c = b; c.dg0 = c.dg1 = 0; c.wg.on = false;
            CKR(timed(b.L.name + " bwd_bn", 0, [&]() -> int { return block_backward(ctx, tp, c, false, false, true, st); }));
        }
        if (b.dg1 > b.dg0) {
            double fd = 0;
            for (size_t i = b.dg0; i < b.dg1; ++i) fd += tp->pl.ops[i].flops;
            CKR(timed(b.L.name + " dgrad", fd, [&]() -> int { for (size_t i = b.dg0; i < b.dg1; ++i) CKR(launch_conv(ctx, tp->pl.ops[i], st, false)); return W2L_OK; }));
        }
        if (b.wg.on) CKR(timed(b.L.name + " wgrad", b.wg.flops, [&]() -> int { return launch_wgrad(ctx, tp, b, false, st, false); }));
    }
    return k;
}

/* One block, train mode, forward + backward (the operator-level entry of the per-geometry gradient tests):
 *   y = block(x) with batch statistics; given dy: dx, dw, db, dgamma, dbeta; running stats updated in place. */
int w2l_conv_block_train(w2l_ctx* ctx, const w2l_layer_info* spec, const float* x, int N, int H, int W, float* weight, float* bias,
                         float* bn_weight, float* bn_bias, float* bn_mean, float* bn_var, const float* dy, float* y, float* dx,
                         float* dw, float* db, float* dgamma, float* dbeta, void* stream) {
    if (!ctx || !spec || !x || !weight || !y) return fail(W2L_EINVAL, "null argument");
    if (!ctx->bf16) return fail(W2L_ESTATE, "training runs with bf16 operands: create the context with W2L_PREC_BF16");
    Layer L;
    int Ho, Wo;
    CKR(block_from_info(spec, "block", N, H, W, &L, &Ho, &Wo));   // the name its tensors are bound under below
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    TrainState* ts = train_state(ctx);
    ts->last_block_info.clear();
    CKR(ensure_train_scratch(ctx, 1, 1));
    const int slot = W2L_NET_DISC;
    // the block's tensors are bound in the discriminator's slot for this call; the caller's binding comes back on return
    struct Rebind {
        std::map<std::string, ParamRef>& live;
        std::map<std::string, ParamRef> saved;
        explicit Rebind(std::map<std::string, ParamRef>& m) : live(m) { saved.swap(live); }
        ~Rebind() { live.swap(saved); }
    } rebind(ts->bound[slot]);
    const long long wn = (long long)L.cin * L.cout * L.kh * L.kw;
    ts->bound[slot]["block.conv_block.0.weight"] = ParamRef{weight, dw, wn};
    ts->bound[slot]["block.conv_block.0.bias"] = ParamRef{bias, db, L.cout};
    const bool bn = L.kind == W2L_BLOCK_CONV_BN_RELU || L.kind == W2L_BLOCK_CONVT_BN_RELU;
    if (bn) {
        ts->bound[slot]["block.conv_block.1.weight"] = ParamRef{bn_weight, dgamma, L.cout};
        ts->bound[slot]["block.conv_block.1.bias"] = ParamRef{bn_bias, dbeta, L.cout};
        if (bn_mean) ts->bound[slot]["block.conv_block.1.running_mean"] = ParamRef{bn_mean, nullptr, L.cout};
        if (bn_var) ts->bound[slot]["block.conv_block.1.running_var"] = ParamRef{bn_var, nullptr, L.cout};
    }
    TrainPlan tp(ctx);   // released on return, before the binding
    tp.net = slot; tp.N = N; tp.B = N; tp.T = 0;
    Act xin, dxin, yv, dyv, none;
    size_t ws_need[2] = {0, 0};
    CKR(tp_act(&tp, &xin, N, H, W, round_up(L.cin, 16)));
    CKR(tp_act(&tp, &dxin, N, H, W, round_up(L.cin, 16)));
    CKR(tp_act(&tp, &yv, N, Ho, Wo, L.cout));
    CKR(tp_act(&tp, &dyv, N, Ho, Wo, L.cout));
    add_train_ingest(&tp, "ingest.x", IngestSpec{0, N, L.cin, (long long)L.cin * H * W, (long long)H * W, 0, 0, W}, xin);
    add_train_ingest(&tp, "ingest.dy", IngestSpec{1, N, L.cout, (long long)L.cout * Ho * Wo, (long long)Ho * Wo, 0, 0, Wo}, dyv);
    CKR(add_train_block(ctx, &tp, slot, 0, L, xin, yv, dyv, dx ? dxin : none, none, dw != nullptr,
                        L.kind == W2L_BLOCK_CONVT_BN_RELU && H == 1 && W == 1, ws_need));
    if (ws_need[0]) CKR(plan_alloc(&tp.pl, &tp.wg_ws[0], ws_need[0]));
    CK(cudaDeviceSynchronize());
    CKR(repack_weights(ctx, &tp, st));
    CKR(launch_ingest(ctx, tp.pl.ops[tp.ingest[0]], x, st));
    CKR(block_forward(ctx, &tp, tp.blocks[0], true, st));
    {
        const long long total = (long long)N * L.cout * Ho * Wo;
        const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
        export_kernel<true><<<blocks, 256, 0, st>>>(yv.base, y, N, Ho, Wo, L.cout, yv.Cs, 0, 0);
        ctx->launches++;
    }
    if (dy) {
        CKR(launch_ingest(ctx, tp.pl.ops[tp.ingest[1]], dy, st));
        CKR(block_backward(ctx, &tp, tp.blocks[0], dw != nullptr, false, true, st));
        if (dx) {
            const long long total = (long long)N * L.cin * H * W;
            const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
            export_grad_kernel<true><<<blocks, 256, 0, st>>>(dxin.ptr(), dxin.Cs, dx, N, H, W, L.cin);
            ctx->launches++;
        }
    }
    CK(cudaStreamSynchronize(st));
    ts->last_block_info.emplace_back();
    train_block_info(ctx, &tp, tp.blocks[0], &ts->last_block_info.back());
    return W2L_OK;
}

int w2l_debug_train_blocks(w2l_ctx* ctx, int net, int cap, w2l_train_block_info* out) {
    if (!ctx || net < -1 || net > 2) return fail(W2L_EINVAL, "bad argument");
    TrainState* ts = train_state(ctx);
    std::vector<w2l_train_block_info> t;
    if (net < 0) {
        t = ts->last_block_info;
    } else {
        const TrainPlan* tp = ts->last[net];
        if (!tp) return fail(W2L_ESTATE, "no training forward has run for net %d", net);
        t.resize(tp->blocks.size());
        for (size_t i = 0; i < tp->blocks.size(); ++i) train_block_info(ctx, tp, tp->blocks[i], &t[i]);
    }
    if (!out) return (int)t.size();
    const int k = std::min<int>(std::max(cap, 0), (int)t.size());
    for (int i = 0; i < k; ++i) out[i] = t[i];
    return k;
}

int w2l_debug_train_tensor(w2l_ctx* ctx, int net, int block, int which, float* out, int* n, int* c, int* h, int* w, void* stream) {
    if (!ctx || net < 0 || net > 2) return fail(W2L_EINVAL, "bad argument");
    const TrainPlan* tp = train_state(ctx)->last[net];
    if (!tp) return fail(W2L_ESTATE, "no training forward has run for net %d", net);
    if (block < 0 || block >= (int)tp->blocks.size()) return fail(W2L_EINVAL, "block %d out of range", block);
    const TBlock& b = tp->blocks[block];
    const Act* a = nullptr;
    int C = b.L.cout;
    switch (which) {
        case W2L_TAPE_X: a = &b.x; C = b.L.cin; break;
        case W2L_TAPE_Z: a = &b.z; break;
        case W2L_TAPE_Y: a = &b.y; break;
        case W2L_TAPE_DY: a = &b.dy; break;
        case W2L_TAPE_DZ: a = &b.dz; break;
        case W2L_TAPE_DU: a = &b.du; break;
        case W2L_TAPE_DX: a = &b.dx; C = b.L.cin; break;
        case W2L_TAPE_DX_ADD: a = &b.dx_add; C = b.L.cin; break;
        case W2L_TAPE_STATS: break;
        default: return fail(W2L_EINVAL, "unknown tape tensor %d", which);
    }
    if (which == W2L_TAPE_STATS) {
        if (!b.bn) return fail(W2L_EINVAL, "%s has no BatchNorm statistics", b.L.name.c_str());
        if (n) *n = 2;
        if (c) *c = C;
        if (h) *h = 1;
        if (w) *w = 1;
        if (out) CK(cudaMemcpyAsync(out, b.stats, (size_t)2 * C * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
        return W2L_OK;
    }
    if (!a->base) return fail(W2L_EINVAL, "%s has no tape tensor %d", b.L.name.c_str(), which);
    if (n) *n = a->N;
    if (c) *c = C;
    if (h) *h = a->H;
    if (w) *w = a->W;
    if (!out) return W2L_OK;
    DeviceGuard g(ctx->device);
    const long long total = (long long)a->N * C * a->H * a->W;
    const int blocks = (int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16);
    export_grad_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(a->ptr(), a->Cs, out, a->N, a->H, a->W, C);
    ctx->launches++;
    CK(cudaGetLastError());
    return W2L_OK;
}

int64_t w2l_launch_count(const w2l_ctx* ctx) { return ctx ? ctx->launches : 0; }

int64_t w2l_device_bytes(const w2l_ctx* ctx) { return ctx ? (int64_t)ctx->device_bytes : 0; }

int w2l_profile_plan(w2l_ctx* ctx, int net, int iters, int cap, float* ms_out, double* flop_out, char (*names_out)[64], void* stream) {
    if (!ctx || net < 0 || net > 3 || iters <= 0) return fail(W2L_EINVAL, "bad argument");
    Plan* pl = ctx->last_plan[net];
    if (!pl) return fail(W2L_ESTATE, "no forward has run for net %d", net);
    DeviceGuard g(ctx->device);
    cudaStream_t st = (cudaStream_t)stream;
    Event e0, e1;
    CKR(e0.create(cudaEventDefault));
    CKR(e1.create(cudaEventDefault));
    // Cold-cache timing: the 126 MB L2 is flushed (a 256 MB buffer is overwritten) before EVERY timed launch, so that layers
    // whose tensors fit the L2 are not timed warm (the timing rule: flush L2 between timed iterations).
    const size_t flush_bytes = (size_t)256 << 20;
    DevMem<> flush;
    if (flush.grow(ctx, flush_bytes) != W2L_OK) g_err.clear();   // without it the timings are warm-cache
    int k = 0;
    for (Op& op : pl->ops) {
        if (op.type != OP_CONV || k >= cap) continue;
        if (op.head && op.cp.ep.head_out == nullptr && op.pp.ep.head_out == nullptr && op.cp.ep.head_out_u8 == nullptr) continue;
        CKR(launch_conv(ctx, op, st, false));  // warm the instruction cache / attributes
        float total = 0.0f;
        for (int i = 0; i < iters; ++i) {
            if (flush) cudaMemsetAsync(flush, i, flush_bytes, st);
            cudaEventRecord(e0, st);
            const int r = launch_conv(ctx, op, st, false);
            cudaEventRecord(e1, st);
            if (cudaEventSynchronize(e1) != cudaSuccess) return fail(W2L_ECUDA, "profile: %s", cudaGetErrorString(cudaGetLastError()));
            CKR(r);
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            total += ms;
        }
        if (ms_out) ms_out[k] = total / iters;
        if (flop_out) flop_out[k] = op.flops;
        if (names_out) snprintf(names_out[k], 64, "%s", op.name.c_str());
        ++k;
    }
    return k;
}

}  // extern "C"
