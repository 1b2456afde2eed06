// host_types.h — host-side data model of libw2l.so: error reporting, the architecture specs, the tensor-map encoder entry
// point, owning handles (device memory, streams, events), activation views (Act), packed weights, launch descriptors (Op),
// plans and the context.
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
// owning handles
// ------------------------------------------------------------------------------------------------
// Every device buffer, stream and event belongs to one of these, held by the context, a plan, a weight layer or the
// training state, and is released when its holder is destroyed.  Releases run with the context's device current: every
// entry point holds a DeviceGuard.
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int dev_alloc(void** p, size_t bytes) {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) return W2L_OK;
    cudaGetLastError();  // a failed allocation is not sticky: clear it, or the next launch check reports it again
    *p = nullptr;
    return fail(W2L_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
}

struct w2l_ctx;

// One cudaMalloc block, counted on its context's device_bytes while it is held.
template <class T = void>
struct DevMem {
    T* p = nullptr;
    size_t cap = 0;              // bytes
    size_t* counter = nullptr;   // &w2l_ctx::device_bytes
    DevMem() = default;
    DevMem(DevMem&& o) noexcept : p(o.p), cap(o.cap), counter(o.counter) { o.p = nullptr; o.cap = 0; }
    DevMem& operator=(DevMem&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); std::swap(counter, o.counter); return *this; }
    ~DevMem() { if (p) { cudaFree(p); *counter -= cap; } }
    operator T*() const { return p; }
    // at least `bytes`: a smaller block is released once the device is idle (queued work may still read it) and
    // replaced; when that allocation fails the block is left empty
    int grow(w2l_ctx* ctx, size_t bytes);
};

struct Stream {
    cudaStream_t h = nullptr;
    Stream() = default;
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() { if (h) cudaStreamDestroy(h); }
    int create() { CK(cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking)); return W2L_OK; }
    operator cudaStream_t() const { return h; }
};

struct Event {
    cudaEvent_t h = nullptr;
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (h) cudaEventDestroy(h); }
    int create(unsigned flags = cudaEventDisableTiming) { CK(cudaEventCreateWithFlags(&h, flags)); return W2L_OK; }
    operator cudaEvent_t() const { return h; }
};

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
    std::vector<DevMem<>> mem;  // the slabs of ph, scale and shift
    int n_scale = 0;
    bool gemm_convT = false;
    bool has_all_taps = false;  // ph.back() holds all 9 taps of a stride-2 transposed conv (fused 4-phase kernel)
    bool loaded = false;
};

struct NetW {
    std::vector<LayerW> layers;
    DevMem<float> head_w;  // generator output_block.1 (3x32) / disc binary_pred (512)
    DevMem<float> head_b;
    bool loaded = false;
};

enum OpType { OP_CONV = 0, OP_INGEST = 1, OP_L2NORM = 2, OP_DISC_HEAD = 3, OP_MAXPOOL = 4, OP_CHAN_L2NORM = 5, OP_S3FD_EXPORT = 6 };

struct Op {
    int type = OP_CONV;
    std::string name;
    // conv
    ConvParams cp;
    int BN = 0, BK = 0, MT = 1;
    bool cm = false;     // channel-major form of the generic kernel (BN channels on wgmma's M, kCmPixels pixels on N)
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
    int patch_th = 0;    // patch kernel: output rows per tile (kPatchTileH, or kChTileH in the channel-major form)
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
    explicit Plan(w2l_ctx* c) : ctx(c) {}
    w2l_ctx* ctx;                  // its allocations count on this context's device_bytes
    int net = 0, B = 0, T = 0, N = 0;
    int H = 0, W = 0;              // S3FD: image size
    std::vector<Op> ops;
    std::vector<DevMem<>> allocs;
    std::map<int, Act> layer_out;  // layer index -> activation view (debug export)
    long long last_used = 0;       // LRU stamp
    int pins = 0;                  // streaming sessions replaying it from a CUDA graph: exempt from LRU eviction
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
    size_t device_bytes = 0;   // every block the members below hold (w2l_device_bytes); declared first, destroyed last
    int device = 0;
    bool bf16 = false;
    bool x2 = false;        // W2L_PREC_F32X: split fp16 operands (hi + lo), generic kernel only
    int num_sms = 132;      // SMs plans are built for: the device's own count unless w2l_debug_set_sm_count lowered it
    int device_sms = 132;   // the device's own count
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
    bool use_stream_graph = true;  // W2L_DISABLE_STREAMGRAPH=1: streaming-session steps launched one by one, not replayed
    NetW nets[4];
    DevMem<float> s3fd_l2w[3];   // conv3_3_norm / conv4_3_norm / conv5_3_norm weights (fp32 copies)
    std::map<std::string, std::unique_ptr<Plan>> plans;
    Plan* last_plan[4] = {nullptr, nullptr, nullptr, nullptr};
    // bumped whenever drop_plans erases the plans of a net (new weights): a streaming session whose graph was captured
    // under an older epoch drops its plan pointer and graph and captures again
    uint64_t plan_epoch[4] = {0, 0, 0, 0};
    std::vector<w2l_kernel_info> last_block_kernels;  // conv launches of the last w2l_conv_block_forward (its plan is freed)
    int64_t launches = 0;
    long long plan_clock = 0;
    // host-buffer entry points: compute stream + copy streams, double-buffered device staging
    Stream stream;
    Stream s_h2d, s_d2h;
    Stream s_side;                   // audio-encoder lane of the generator plan
    Event ev_fork, ev_join;
    bool use_side = true;            // W2L_DISABLE_SIDESTREAM=1
    Event ev_in[2], ev_done[2], ev_out[2];
    DevMem<> stage[6];
    DevMem<int> boxes_dev;           // crop / paste boxes (row f2)
    DevMem<int> samples_dev;         // training-batch sample table (ints)
    DevMem<uint8_t> crops_dev, preds_dev;
    DevMem<float> scratch;           // partial sums of the loss kernels
    long long host_seq = 0;   // host-buffer submissions so far (staging slot = seq & 1)
    int host_inflight = 0;    // submitted and not yet retired by host_drain
    // mel tables
    DevMem<double2> mel_tw;
    DevMem<float> mel_bvals;
    DevMem<int> mel_boff;
    DevMem<int> mel_bstart;
    DevMem<int> mel_blen;
    // resampling: (win, delta) tables by ratio (1.0 for every upsampling ratio), made when a ratio is first used, and the
    // block start registers of w2l_resample
    std::map<double, DevMem<double2>> rs_tables;
    DevMem<double> rs_reg0;
    Event ev_rs;                     // after the last w2l_resample kernel: the next call's upload of rs_reg0 waits for it
    std::unique_ptr<TrainState> train;   // declared last: released first
};

template <class T>
int DevMem<T>::grow(w2l_ctx* ctx, size_t bytes) {
    if (p && cap >= bytes) return W2L_OK;
    if (p) {
        CK(cudaDeviceSynchronize());
        *this = DevMem();
    }
    const size_t n = bytes ? bytes : 16;
    void* q;
    CKR(dev_alloc(&q, n));
    p = (T*)q; cap = n; counter = &ctx->device_bytes;
    *counter += n;
    return W2L_OK;
}

// a new block of `bytes`, held by `owner`
template <class T>
static int alloc_in(w2l_ctx* ctx, std::vector<DevMem<>>* owner, T** p, size_t bytes) {
    owner->emplace_back();
    CKR(owner->back().grow(ctx, bytes));
    *p = (T*)owner->back().p;
    return W2L_OK;
}

template <class T>
static int plan_alloc(Plan* pl, T** p, size_t bytes) { return alloc_in(pl->ctx, &pl->allocs, p, bytes); }

static int plan_act(Plan* pl, Act* a, int N, int H, int W, int C, bool f32 = false) {
    const bool planes = pl->x2 && !f32;
    const size_t bytes = (size_t)N * H * W * C * (f32 ? 4 : 2) * (planes ? 2 : 1);
    CKR(plan_alloc(pl, &a->base, bytes));
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
    const size_t bytes = ((size_t)N * H * Wp * w.Cp + w.kfold) * 2;  // + one window of slack at the very end
    CKR(plan_alloc(pl, &a->base, bytes));
    CK(cudaMemset(a->base, 0, bytes));
    a->N = N; a->H = H; a->W = W; a->Cs = w.Cp; a->c_off = 0; a->C = w.kfold; a->f32 = false;
    a->Wp = Wp; a->x_off = L.pw;
    a->wstride = L.sw; a->nwin = Wout;
    return W2L_OK;
}
