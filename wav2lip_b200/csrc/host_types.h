// host_types.h — host-side data model of libw2l.so: error reporting, the architecture specs, the tensor-map encoder entry
// point, activation views (Act), packed weights, launch descriptors (Op), plans and the context.
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess)                                                                           \
            return fail(W2L_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)
#define CKR(expr)               \
    do {                        \
        int r_ = (expr);        \
        if (r_ != W2L_OK) return r_; \
    } while (0)

// ------------------------------------------------------------------------------------------------
// specs (built once, host only)
// ------------------------------------------------------------------------------------------------
static const GeneratorSpec& gen_spec() { static GeneratorSpec s = build_generator_spec(); return s; }
static const SyncnetSpec& sync_spec() { static SyncnetSpec s = build_syncnet_spec(); return s; }
static const DiscSpec& disc_spec() { static DiscSpec s = build_disc_spec(); return s; }
static const S3fdSpec& s3fd_spec() { static S3fdSpec s = build_s3fd_spec(); return s; }
static const std::vector<Layer>* net_layers(int net) {
    switch (net) {
        case W2L_NET_GENERATOR: return &gen_spec().layers;
        case W2L_NET_SYNCNET: return &sync_spec().layers;
        case W2L_NET_DISC: return &disc_spec().layers;
        case W2L_NET_S3FD: return &s3fd_spec().layers;
    }
    return nullptr;
}

// ------------------------------------------------------------------------------------------------
// driver entry point for tensor-map encoding (no link-time dependency on libcuda)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// ------------------------------------------------------------------------------------------------
// tensors in HBM
// ------------------------------------------------------------------------------------------------
// Activations are NHWC, 16-bit (fp16 or bf16), channel pitch Cs; a view may select a channel slice
// [c_off, c_off + C) of a wider buffer (the skip-concat buffers of the decoder).
struct Act {
    uint16_t* base = nullptr;  // start of the buffer (not of the slice)
    int N = 0, H = 0, W = 0;
    int Cs = 0;     // channel pitch of the buffer
    int c_off = 0;  // first channel of this view
    int C = 0;      // channels of this view
    bool f32 = false;
    int Wp = 0;     // row pitch in pixels (0 = W); > W only for the zero-bordered first-layer inputs
    int x_off = 0;  // left border of those inputs
    int lo_off = 0;   // split-operand mode: channel distance from the hi plane to the lo plane of the same pixel
    int wstride = 1;  // folded views: pixels between consecutive windows (= the conv's horizontal stride)
    int nwin = 0;     // folded views: number of windows per row (= output width); 0 = W
    int pitch() const { return Wp ? Wp : W; }
    uint16_t* ptr() const { return base + c_off; }
    Act slice(int off, int c) const { Act a = *this; a.c_off = c_off + off; a.C = c; return a; }
};

struct PackedW {
    uint16_t* w = nullptr;  // [ntaps][cout_pad][cin_pad]
    int ntaps = 0, cout_pad = 0, cin_pad = 0;
    int nslabs = 0;                   // weight slabs stored: ntaps, or 2*ntaps (hi then lo) in the split-operand mode
    std::vector<signed char> dx, dy;  // input offset of each tap relative to (out * stride)
    int py = 0, px = 0;               // output phase (transposed conv)
    // "kw folded into K" form for tiny-Cin first layers: one K row = kw taps x Cp channels (zero padded to kfold)
    bool fold = false;
    int Cp = 0, kfold = 0, win = 0;   // channel pitch of the input, folded K per filter row, pixels spanned by a window
};

struct LayerW {
    std::vector<PackedW> ph;  // 1 for conv, 4 for stride-2 convT, 1 (as GEMM) for the 1x1->3x3 convT
    float* scale = nullptr;
    float* shift = nullptr;
    int n_scale = 0;
    bool gemm_convT = false;
    bool has_all_taps = false;  // ph.back() holds all 9 taps of a stride-2 transposed conv (fused 4-phase kernel)
    bool loaded = false;
};

struct NetW {
    std::vector<LayerW> layers;
    float* head_w = nullptr;  // generator output_block.1 (3x32) / disc binary_pred (512)
    float* head_b = nullptr;
    bool loaded = false;
};

enum OpType { OP_CONV = 0, OP_INGEST = 1, OP_L2NORM = 2, OP_DISC_HEAD = 3, OP_MAXPOOL = 4, OP_CHAN_L2NORM = 5, OP_S3FD_EXPORT = 6 };

struct Op {
    int type = OP_CONV;
    std::string name;
    // conv
    ConvParams cp;
    int BN = 0, BK = 0, MT = 1;
    bool head = false;
    int grid = 0;
    double flops = 0;  // algorithmic (true MACs*2), not padded
    bool patch = false;  // conv_patch_kernel instead of conv_igemm_kernel
    PatchParams pp;
    int dyn_smem = 0;
    bool ctf = false;   // convt_fused_kernel
    ConvTParams tp;
    bool fold = false;  // K-folded first layer
    int m_tiles = 0, n_tiles = 0;  // output tiles along pixels / channels (w2l_debug_plan_kernels)
    // ingest
    IngestParams ip;
    int ingest_src = 0;  // which caller tensor: 0 = mel / frames, 1 = face
    // l2norm / disc head
    const void* aux_in = nullptr;
    int aux_rows = 0, aux_dim = 0;
    int aux_out = 0;  // which caller output
    int aux_pitch = 0, aux_lo = 0;  // pixel pitch and lo-plane offset of aux_in (also of the S3FD max-pool / L2Norm buffers)
    // S3FD: max-pool / channel L2Norm / head export
    const uint16_t* sp_in = nullptr; uint16_t* sp_out = nullptr; const float* sp_f32 = nullptr; const float* sp_w = nullptr;
    int sp_N = 0, sp_H = 0, sp_W = 0, sp_C = 0, sp_Cout = 0, sp_maxout = 0;
    int lane = 0;          // 1: runs on the context's side stream (the audio encoder, concurrently with the face encoder)
    bool join_side = false;  // wait for the side stream before this op
};

// detection work of an S3FD plan (s3fd_detect.cuh), added the first time the plan is used for detection
struct S3fdDetWork {
    S3fdDetParams p;       // head pointers, sizes and workspace; max_det / dets / counts are set per call
    bool last = false;     // the plan's last replay was a detection (its candidates are readable)
};

struct Plan {
    int net = 0, B = 0, T = 0, N = 0;
    int H = 0, W = 0;              // S3FD: image size
    std::vector<Op> ops;
    std::vector<void*> allocs;
    size_t bytes = 0;
    std::map<int, Act> layer_out;  // layer index -> activation view (debug export)
    long long last_used = 0;       // LRU stamp
    bool x2 = false;               // split-operand precision: activations carry hi and lo planes
    bool has_side = false;         // some ops run on the side stream
    std::unique_ptr<S3fdDetWork> det;  // S3FD: detection workspace (nullptr until the first w2l_s3fd_detect_u8)
};

struct FoldJob { const float* bias; int cout, reps, n_pad; float* scale; float* shift; };  // nonorm blocks: shift = conv bias
// the launches that pack a training plan's 16-bit weight slabs from the fp32 master tensors, replayed after every
// optimizer step (repack_weights)
struct RepackLog { std::vector<PackParams> pack; std::vector<PackFoldParams> pack_fold; std::vector<FoldJob> fold; };
struct TrainState;  // host_train.cuh

struct w2l_ctx {
    TrainState* train = nullptr;
    int device = 0;
    bool bf16 = false;
    bool x2 = false;        // W2L_PREC_F32X: split fp16 operands (hi + lo), generic kernel only
    int num_sms = 132;
    bool keep_all = false;  // debug: no buffer reuse, every layer output stays readable
    bool use_patch = true;   // W2L_DISABLE_HALO=1 turns the patch kernel off (A/B testing)
    bool use_mt2 = true;    // W2L_DISABLE_MT2=1
    bool use_aux_stream = true; // W2L_DISABLE_AUXSTREAM=1: training audio-encoder blocks on the main stream
    bool use_wg_stream = true; // W2L_DISABLE_WGSTREAM=1: training wgrads on the main stream instead of a side stream
    bool use_tma_epi = true;  // W2L_DISABLE_TMAEPI=1
    bool use_fold_s2 = true;  // W2L_DISABLE_FOLDS2=1
    bool use_ctfused = true;  // W2L_DISABLE_CTFUSED=1
    bool use_fold = true;   // W2L_DISABLE_FOLD=1 / driver rejects overlapping-stride tensor maps
    bool use_pdl = true;      // W2L_DISABLE_PDL=1
    NetW nets[4];
    float* s3fd_l2w[3] = {nullptr, nullptr, nullptr};   // conv3_3_norm / conv4_3_norm / conv5_3_norm weights (fp32 copies)
    std::map<std::string, std::unique_ptr<Plan>> plans;
    Plan* last_plan[4] = {nullptr, nullptr, nullptr, nullptr};
    std::vector<w2l_kernel_info> last_block_kernels;  // conv launches of the last w2l_conv_block_forward (its plan is freed)
    int64_t launches = 0;
    long long plan_clock = 0;
    size_t weight_bytes = 0;
    // host-buffer entry points: compute stream + copy streams, double-buffered device staging
    cudaStream_t stream = nullptr;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaStream_t s_side = nullptr;   // audio-encoder lane of the generator plan
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool use_side = true;            // W2L_DISABLE_SIDESTREAM=1
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
    void* stage[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    int* boxes_dev = nullptr; int box_cap = 0;                 // crop / paste boxes (row f2)
    int* samples_dev = nullptr; size_t sample_cap = 0;         // training-batch sample table (ints)
    uint8_t *crops_dev = nullptr, *preds_dev = nullptr; size_t crop_cap = 0;
    float* scratch = nullptr;  // partial sums of the loss kernels
    size_t scratch_bytes = 0;
    long long host_seq = 0;   // host-buffer submissions so far (staging slot = seq & 1)
    int host_inflight = 0;    // submitted and not yet retired by host_drain
    size_t stage_bytes[6] = {0, 0, 0, 0, 0, 0};
    // mel tables
    double2* mel_tw = nullptr;
    float* mel_bvals = nullptr;
    int* mel_boff = nullptr;
    int* mel_bstart = nullptr;
    int* mel_blen = nullptr;
};

static int dev_alloc(void** p, size_t bytes) {
    cudaError_t e = cudaMalloc(p, bytes ? bytes : 16);
    if (e != cudaSuccess) return fail(W2L_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return W2L_OK;
}

static int plan_alloc(Plan* pl, void** p, size_t bytes) {
    CKR(dev_alloc(p, bytes));
    pl->allocs.push_back(*p);
    pl->bytes += bytes;
    return W2L_OK;
}

static int plan_act(Plan* pl, Act* a, int N, int H, int W, int C, bool f32 = false) {
    void* p = nullptr;
    const bool planes = pl->x2 && !f32;
    const size_t bytes = (size_t)N * H * W * C * (f32 ? 4 : 2) * (planes ? 2 : 1);
    CKR(plan_alloc(pl, &p, bytes));
    a->base = (uint16_t*)p;
    a->N = N; a->H = H; a->W = W; a->Cs = planes ? 2 * C : C; a->c_off = 0; a->C = C; a->f32 = f32;
    a->lo_off = planes ? C : 0;
    return W2L_OK;
}

// Buffer the ingest kernel fills for the first block of a chain. Folded first layers read it through an
// overlapping-window tensor map: channel pitch Cp, rows padded with pw zero pixels on the left and enough
// on the right for the last window; the view handed to the conv is (C = kfold, W windows).
static int plan_input_act(Plan* pl, Act* a, int N, int H, int W, int cin, const LayerW& lw, const Layer& L) {
    const PackedW& w = lw.ph[0];
    if (!w.fold) return plan_act(pl, a, N, H, W, ((cin + 15) / 16) * 16);
    const int Wout = (W + 2 * L.pw - L.kw) / L.sw + 1;
    const int Wp = (std::max(W + L.pw, (Wout - 1) * L.sw + w.win) + 1) / 2 * 2;
    void* p = nullptr;
    const size_t bytes = ((size_t)N * H * Wp * w.Cp + w.kfold) * 2;  // + one window of slack at the very end
    CKR(plan_alloc(pl, &p, bytes));
    CK(cudaMemset(p, 0, bytes));
    a->base = (uint16_t*)p;
    a->N = N; a->H = H; a->W = W; a->Cs = w.Cp; a->c_off = 0; a->C = w.kfold; a->f32 = false;
    a->Wp = Wp; a->x_off = L.pw;
    a->wstride = L.sw; a->nwin = Wout;
    return W2L_OK;
}

static void free_plan(Plan* pl) {
    for (void* p : pl->allocs) cudaFree(p);
    pl->allocs.clear();
}
