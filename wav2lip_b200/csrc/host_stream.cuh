// host_stream.cuh — streaming: the mel rings behind w2l_melstream_* and the lip-sync session behind w2l_stream_*
// (DESIGN.md section 3.8).  The scheduling rules (which rows the audio received so far fixes) are host code with no
// device state, exported as w2l_stream_schedule so that they can be tested without a GPU.
// Part of the single translation unit w2l_api.cu (included there, after the plans).
#pragma once

static const char kMelNanMsg[] =
    "Mel contains nan! Using a TTS voice? Add a small epsilon noise to the wav file and try again";  // inference.py:228-229

struct PinnedMem {
    void* p = nullptr;
    PinnedMem() = default;
    PinnedMem(const PinnedMem&) = delete;
    PinnedMem& operator=(const PinnedMem&) = delete;
    ~PinnedMem() { if (p) cudaFreeHost(p); }
    int alloc(size_t bytes) { CK(cudaHostAlloc(&p, bytes, cudaHostAllocDefault)); return W2L_OK; }
};

struct GraphExec {
    cudaGraphExec_t h = nullptr;
    GraphExec() = default;
    GraphExec(const GraphExec&) = delete;
    GraphExec& operator=(const GraphExec&) = delete;
    ~GraphExec() { reset(); }
    void reset() { if (h) cudaGraphExecDestroy(h); h = nullptr; }
};

static long long pow2_at_least(long long v) { long long p = 1; while (p < v) p <<= 1; return p; }

// mel frames that L received samples make final: 200 f + 400 <= L
static long long mel_final_frames(long long L) { return L >= 400 ? (L - 400) / MEL_HOP + 1 : 0; }

// Where a piece of audio lives.  An asynchronous copy from pageable memory has read it when cudaMemcpyAsync returns;
// from pinned or device memory it reads it when the copy runs.
enum PcmKind { PCM_PAGEABLE = 0, PCM_PINNED = 1, PCM_DEVICE = 2 };
static int pcm_kind(const w2l_ctx* ctx, const float* p, int* kind) {
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(W2L_EINVAL, "pcm: cudaPointerGetAttributes: %s", cudaGetErrorString(e)); }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
        if (a.type == cudaMemoryTypeDevice && a.device != ctx->device)
            return fail(W2L_EINVAL, "pcm is on device %d, the context on device %d", a.device, ctx->device);
        *kind = PCM_DEVICE;
    } else {
        *kind = a.type == cudaMemoryTypeHost ? PCM_PINNED : PCM_PAGEABLE;
    }
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// mel rings: audio by absolute sample index, mel by absolute frame index, both power-of-two long
// ------------------------------------------------------------------------------------------------
struct MelRing {
    w2l_ctx* ctx = nullptr;
    long long ra = 0, rm = 0;   // audio ring (samples), mel ring (frames)
    DevMem<float> audio, mel;
    DevMem<int> nan;
    PinnedMem nan_host;
    Event ev_nan;
    long long L = 0;            // samples received
    long long f_next = 0;       // frames computed: [0, f_next)
    bool finished = false;

    int init(w2l_ctx* c, int audio_log2, long long min_mel_frames) {
        ctx = c;
        if (audio_log2 == 0) audio_log2 = 16;
        if (audio_log2 < 11 || audio_log2 > 24) return fail(W2L_EINVAL, "audio ring of 2^%d samples: need 2^11 .. 2^24", audio_log2);
        ra = 1LL << audio_log2;
        rm = pow2_at_least(std::max(ra / MEL_HOP + 16, min_mel_frames));
        CKR(audio.grow(ctx, (size_t)ra * 4));
        CKR(mel.grow(ctx, (size_t)rm * MEL_BANDS * 4));
        CKR(nan.grow(ctx, 4));
        CK(cudaMemset(nan, 0, 4));
        CKR(nan_host.alloc(4));
        CKR(ev_nan.create());
        return W2L_OK;
    }

    // Longest next piece of audio that overwrites neither an audio sample a frame not yet computed reads (frame f reads
    // from 200 f - 401) nor a mel column at or after keep_frame, the oldest frame the consumer still needs.
    long long max_piece(long long keep_frame) const {
        const long long oldest = std::max(0LL, f_next * MEL_HOP - MEL_NFFT / 2 - 1);
        const long long by_audio = ra - (L - oldest);
        const long long by_mel = (long long)MEL_HOP * (rm - (f_next - keep_frame) - 1);
        return std::min(by_audio, by_mel);
    }

    // pcm: host (any kind) or device memory; copied into the ring at absolute positions [L, L + n)
    int append(const float* pcm, long long n, cudaStream_t st) {
        long long done = 0;
        while (done < n) {
            const long long at = (L + done) & (ra - 1);
            const long long k = std::min(n - done, ra - at);
            CK(cudaMemcpyAsync(audio.p + at, pcm + done, (size_t)k * 4, cudaMemcpyDefault, st));
            done += k;
        }
        L += n;
        return W2L_OK;
    }

    // frames [f_next, f_end); L_end >= 0 only at finish (reflection at the end of the utterance)
    int compute(const MelParams& tables, long long f_end, long long L_end, cudaStream_t st) {
        if (f_end <= f_next) return W2L_OK;
        MelRingParams r;
        r.audio = audio; r.audio_mask = ra - 1; r.mel = mel; r.mel_pitch = rm;
        r.L = L_end >= 0 ? L_end : (1LL << 62);
        r.f0 = f_next; r.f1 = f_end; r.nan = nan;
        const long long blocks = (f_end - f_next + MEL_FPB - 1) / MEL_FPB;
        mel_ring_kernel<<<(unsigned)blocks, MEL_THREADS, kMelSmemBytes, st>>>(tables, r);
        ctx->launches++;
        CK(cudaGetLastError());
        f_next = f_end;
        return W2L_OK;
    }

    // the sticky NaN flag (waits for the work queued on st)
    int nan_seen(cudaStream_t st, bool* seen) {
        CK(cudaMemcpyAsync(nan_host.p, nan, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(ev_nan, st));
        CK(cudaEventSynchronize(ev_nan));
        *seen = *(const int*)nan_host.p != 0;
        return W2L_OK;
    }

    // frames [a, b) -> columns [col, col + b - a) of an (80, pitch) row-major block
    int copy_out(long long a, long long b, float* dst, long long pitch, long long col, cudaStream_t st) {
        while (a < b) {
            const long long at = a & (rm - 1);
            const long long k = std::min(b - a, rm - at);
            CK(cudaMemcpy2DAsync(dst + col, (size_t)pitch * 4, mel.p + at, (size_t)rm * 4, (size_t)k * 4, MEL_BANDS,
                                 cudaMemcpyDeviceToDevice, st));
            a += k; col += k;
        }
        return W2L_OK;
    }
};

static MelParams mel_tables(const w2l_ctx* ctx) {
    MelParams p;
    memset(&p, 0, sizeof(p));
    p.tw = ctx->mel_tw; p.bvals = ctx->mel_bvals; p.boff = ctx->mel_boff; p.bstart = ctx->mel_bstart; p.blen = ctx->mel_blen;
    return p;
}

struct w2l_melstream {
    w2l_ctx* ctx = nullptr;
    MelRing ring;
};

// ------------------------------------------------------------------------------------------------
// scheduling (rules 1-4 of DESIGN.md section 3.8), host only
// ------------------------------------------------------------------------------------------------
struct StreamSched {
    w2l_stream_desc d;
    double mult = 0;                          // 80. / fps, inference.py:232
    std::vector<long long> padded;            // F x (x1, y1, x2, y2): rects padded and clipped (inference.py:89-96)
    std::map<long long, std::vector<long long>> smoothed;  // n -> the first n padded rows smoothed as inference.py:59-66

    struct At {
        long long M = 0;         // final mel frames
        long long n_total = -1;  // frames the video is cut to (inference.py:244), -1 while unknown
        long long n_fixed = 0;   // rows fixed
        bool final = false;
    };

    // detect: the rects arrive frame by frame through set_rect (rects unused, d.has_box must be 0)
    int init(const w2l_stream_desc* desc, const int32_t* rects, bool detect = false) {
        if (!desc) return fail(W2L_EINVAL, "null stream description");
        d = *desc;
        if (d.F < 1 || d.H < 1 || d.W < 1) return fail(W2L_EINVAL, "bad video shape F=%d H=%d W=%d", d.F, d.H, d.W);
        if (!(d.fps > 0) || !std::isfinite(d.fps)) return fail(W2L_EINVAL, "fps must be positive and finite (got %g)", d.fps);
        mult = 80. / d.fps;
        if (detect && d.has_box) return fail(W2L_EINVAL, "a fixed box and face detection exclude each other");
        if (d.has_box) {
            const int32_t* b = d.box;
            if (b[0] < 0 || b[1] > d.H || b[0] >= b[1] || b[2] < 0 || b[3] > d.W || b[2] >= b[3])
                return fail(W2L_EINVAL, "box (y %d:%d, x %d:%d) is empty or outside the %dx%d frame", b[0], b[1], b[2], b[3], d.H, d.W);
            return W2L_OK;
        }
        if (!rects && !detect) return fail(W2L_EINVAL, "neither detector rects nor a fixed box");
        padded.assign((size_t)d.F * 4, 0);
        if (!detect)
            for (int j = 0; j < d.F; ++j) set_rect(j, rects + 4 * j);
        return W2L_OK;
    }

    void set_rect(long long j, const int32_t* r) {
        padded[4 * j + 0] = std::max(0, r[0] - d.pads[2]);
        padded[4 * j + 1] = std::max(0, r[1] - d.pads[0]);
        padded[4 * j + 2] = std::min(d.W, r[2] + d.pads[3]);
        padded[4 * j + 3] = std::min(d.H, r[3] + d.pads[1]);
    }

    long long start(long long i) const { return (long long)((double)i * mult); }

    // chunks i with s_i + 16 <= M (the regular ones of a mel of M frames)
    long long n_regular(long long M) const {
        if (M < 16) return 0;
        long long i = (long long)((double)(M - 16) / mult) + 2;
        while (i > 0 && start(i - 1) + 16 > M) --i;
        while (start(i) + 16 <= M) ++i;
        return i;
    }

    int at(long long L, bool final, At* a) const {
        a->final = final;
        if (final) {
            a->M = L >= 2 ? 1 + L / MEL_HOP : 0;
            if (a->M < 16)
                return fail(W2L_EINVAL, "audio of %lld samples gives %lld mel frames: shorter than one 16-frame chunk", L, a->M);
            a->n_fixed = n_regular(a->M) + 1;  // the first chunk that overruns is the last one, right-aligned
            a->n_total = std::min<long long>(a->n_fixed, d.F);
            return W2L_OK;
        }
        a->M = mel_final_frames(L);
        const long long n_reg = n_regular(a->M);
        const long long n_lb = n_reg > 0 ? n_reg + 1 : 0;   // the chunk count the audio so far guarantees
        a->n_total = n_lb >= d.F ? d.F : -1;
        const bool box_now = d.has_box || d.nosmooth || d.F == 1 || a->n_total >= 0;
        // otherwise output i shows frame i, whose smoothed box is final once i + 5 <= n_lb
        a->n_fixed = box_now ? n_reg : std::max(0LL, std::min(n_reg, n_lb - 4));
        return W2L_OK;
    }

    // The frames whose rects rows [0, a.n_fixed) read: always a prefix [0, need).  F == 1: frame 0.  nosmooth: the
    // frames shown.  Smoothing: the padded rows i .. i+4 of each row i while n_total is unknown (n_fixed + 4 <= n_lb < F),
    // all of [0, n_total) once it is known (the tail window's in-place smoothing reads every earlier row).  At final this
    // is n_total: the frames inference.py detects on (:244, :113), and none past them.
    long long need(const At& a) const {
        if (d.has_box) return 0;
        if (d.F == 1) return 1;
        if (a.n_fixed == 0) return 0;
        if (d.nosmooth) return a.n_total >= 0 ? std::min(a.n_fixed, a.n_total) : a.n_fixed;
        return a.n_total >= 0 ? a.n_total : a.n_fixed + 4;
    }

    const std::vector<long long>& smooth_first(long long n) {
        auto it = smoothed.find(n);
        if (it != smoothed.end()) return it->second;
        std::vector<long long> b(padded.begin(), padded.begin() + 4 * n);
        for (long long i = 0; i < n; ++i) {        // in place, as get_smoothened_boxes does
            long long lo = i, hi = i + 5;
            if (i + 5 > n) {                       // boxes[len - T:], a negative start counting from the end
                lo = n - 5;
                if (lo < 0) lo = (-lo <= n) ? n + lo : 0;
                hi = n;
            }
            for (int c = 0; c < 4; ++c) {
                double s = 0;
                for (long long k = lo; k < hi; ++k) s += (double)b[4 * k + c];
                b[4 * i + c] = (long long)(s / (double)(hi - lo));   // np.mean, truncated into the int array
            }
        }
        return smoothed[n] = std::move(b);
    }

    // row i (< a.n_fixed): (i, chunk start, frame, y1, y2, x1, x2)
    int row(long long i, const At& a, int32_t* r) {
        const long long frame = a.n_total >= 0 ? i % a.n_total : i;
        long long s = start(i);
        if (a.final && s + 16 > a.M) s = a.M - 16;
        long long y1, y2, x1, x2;
        if (d.has_box) {
            y1 = d.box[0]; y2 = d.box[1]; x1 = d.box[2]; x2 = d.box[3];
        } else if (d.nosmooth) {
            const long long* p = &padded[4 * frame];
            x1 = p[0]; y1 = p[1]; x2 = p[2]; y2 = p[3];
        } else {
            long long v[4];
            if (a.n_total >= 0 && frame + 5 > a.n_total) {
                const std::vector<long long>& b = smooth_first(a.n_total);
                for (int c = 0; c < 4; ++c) v[c] = b[4 * frame + c];
            } else {                               // rows before the tail window: the mean of the next five padded rows
                for (int c = 0; c < 4; ++c) {
                    double sum = 0;
                    for (long long k = frame; k < frame + 5; ++k) sum += (double)padded[4 * k + c];
                    v[c] = (long long)(sum / 5.0);
                }
            }
            x1 = v[0]; y1 = v[1]; x2 = v[2]; y2 = v[3];
        }
        if (y1 < 0 || y2 > d.H || y1 >= y2 || x1 < 0 || x2 > d.W || x1 >= x2)
            return fail(W2L_EINVAL, "output %lld: box of frame %lld (y %lld:%lld, x %lld:%lld) is empty or outside the %dx%d frame",
                        i, frame, y1, y2, x1, x2, d.H, d.W);
        r[0] = (int32_t)i; r[1] = (int32_t)s; r[2] = (int32_t)frame;
        r[3] = (int32_t)y1; r[4] = (int32_t)y2; r[5] = (int32_t)x1; r[6] = (int32_t)x2;
        return W2L_OK;
    }
};

// ------------------------------------------------------------------------------------------------
// the session
// ------------------------------------------------------------------------------------------------
constexpr int kStreamSlots = 4;   // pinned staging rows of the per-step table in flight

struct w2l_stream {
    w2l_ctx* ctx = nullptr;
    StreamSched sched;
    MelRing mel;
    const uint8_t* frames = nullptr;
    int batch = 0;
    long long emitted = 0;          // rows whose step has been queued
    bool nan = false, finished = false;
    // per-step device table: [batch][5] (frame, y1, y2, x1, x2) for crop and paste, then [batch] chunk starts
    DevMem<int> table;
    PinnedMem stage;                // kStreamSlots x the table
    Event slot_done[kStreamSlots];  // the H2D copy out of each staging slot
    // The mel work (audio copy, ring kernel, NaN flag read-back) runs on a private stream, so that the host, which waits
    // for each piece's NaN flag before it schedules rows, waits for this session's mel frames only, not for the steps
    // queued on the caller's stream.  The ring kernel overwrites mel columns that queued steps may still read: before
    // it runs, the mel stream waits for the last step that reads a column it overwrites (step_done / step_lo).
    Stream s_mel;
    Event ev_caller;                // the caller's stream, before a piece of device audio is copied
    Event step_done[kStreamSlots];  // recorded after the gather of step k (slot k % kStreamSlots) on the caller's stream
    long long step_lo[kStreamSlots] = {0, 0, 0, 0};   // the lowest mel frame step k reads
    long long first_lo = -1;        // that of the session's first step
    long long steps = 0;
    DevMem<float> chunks;
    DevMem<uint8_t> crops, preds;
    // the generator plan the step replays, pinned against LRU eviction while held; valid while epoch matches
    Plan* plan = nullptr;
    uint64_t epoch = 0;
    Stream cap;                     // capture stream (the graph is launched on the caller's stream)
    GraphExec exec;
    bool warm = false;              // one uncaptured step ran on the current plan (kernel attributes are set)
};

static void stream_release_plan(w2l_stream* s) {
    if (s->plan && s->epoch == s->ctx->plan_epoch[W2L_NET_GENERATOR]) s->plan->pins--;
    s->plan = nullptr;
    s->exec.reset();
    s->warm = false;
}

// The plan is erased, with every generator plan, only by drop_plans (new weights), which bumps the epoch; LRU eviction
// skips pinned plans.  So a matching epoch means the plan, and every buffer the graph bakes, is alive and current.
static int stream_acquire_plan(w2l_stream* s) {
    w2l_ctx* ctx = s->ctx;
    if (s->plan && s->epoch == ctx->plan_epoch[W2L_NET_GENERATOR]) return W2L_OK;
    stream_release_plan(s);
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_GENERATOR, s->batch, 0, &pl));
    pl->pins++;
    s->plan = pl;
    s->epoch = ctx->plan_epoch[W2L_NET_GENERATOR];
    return W2L_OK;
}

// gather + crop/resize + generator: every argument is a session buffer, so the launches can be captured once
static int stream_body(w2l_stream* s, cudaStream_t st) {
    w2l_ctx* ctx = s->ctx;
    const int B = s->batch;
    const StreamSched& sc = s->sched;
    mel_ring_gather_kernel<<<(B * 1280 + 255) / 256, 256, 0, st>>>(s->mel.mel, s->mel.rm, s->table.p + 5 * B, B, s->chunks);
    const long long total = (long long)B * 96 * 96;
    crop_resize_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16), 256, 0, st>>>(
        s->frames, sc.d.H, sc.d.W, s->table, B, 96, s->crops);
    ctx->launches += 2;
    CK(cudaGetLastError());
    return run_plan(ctx, s->plan, s->chunks, s->crops, s->preds, nullptr, st, true);
}

static int stream_capture(w2l_stream* s) {
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(s->cap, cudaStreamCaptureModeThreadLocal));
    const int r = stream_body(s, s->cap);
    const cudaError_t e = cudaStreamEndCapture(s->cap, &g);
    if (r != W2L_OK) { if (g) cudaGraphDestroy(g); cudaGetLastError(); return r; }
    CK(e);
    const cudaError_t ei = cudaGraphInstantiate(&s->exec.h, g, 0);
    cudaGraphDestroy(g);
    CK(ei);
    return W2L_OK;
}

// one generator step over rows[0, n) (n <= batch), output frames to out (n, H, W, 3)
static int stream_step(w2l_stream* s, const int32_t* rows, int n, uint8_t* out, cudaStream_t st) {
    w2l_ctx* ctx = s->ctx;
    const int B = s->batch;
    CKR(stream_acquire_plan(s));
    const int slot = (int)(s->steps++ % kStreamSlots);
    CK(cudaEventSynchronize(s->slot_done[slot]));       // its previous copy has read the staging row
    int32_t* h = (int32_t*)s->stage.p + (size_t)slot * B * 6;
    for (int b = 0; b < B; ++b) {
        const int32_t* r = rows + W2L_STREAM_ROW * std::min(b, n - 1);   // rows past n repeat the last one
        h[5 * b + 0] = r[2]; h[5 * b + 1] = r[3]; h[5 * b + 2] = r[4]; h[5 * b + 3] = r[5]; h[5 * b + 4] = r[6];
        h[5 * B + b] = r[1];
    }
    CK(cudaMemcpyAsync(s->table, h, (size_t)B * 6 * 4, cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(s->slot_done[slot], st));
    if (!ctx->use_stream_graph || !s->warm) {
        CKR(stream_body(s, st));
        s->warm = true;
    } else {
        if (!s->exec.h) CKR(stream_capture(s));
        CK(cudaGraphLaunch(s->exec.h, st));
    }
    CK(cudaEventRecord(s->step_done[slot], st));      // its gather has read the mel ring
    s->step_lo[slot] = rows[1];                        // rows are in output order: the first has the lowest start
    if (s->first_lo < 0) s->first_lo = rows[1];
    // the paste writes into the caller's buffer and only the n real rows: launched outside the graph
    const StreamSched& sc = s->sched;
    const long long total = (long long)n * sc.d.H * sc.d.W;
    paste_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 32), 256, 0, st>>>(
        s->preds, 96, s->frames, sc.d.H, sc.d.W, s->table, n, out);
    ctx->launches++;
    CK(cudaGetLastError());
    s->emitted += n;
    return W2L_OK;
}

// Before the ring kernel writes frames [f_next, f_end) into columns that held frames below f_end - rm: make the mel
// stream wait for the last queued step that reads such a frame.  Steps read from their lowest chunk start upwards and
// those starts never decrease from step to step, so that step is the newest one with step_lo < cutoff; if it is older
// than the tracked slots, the oldest tracked step (after it on the caller's stream) stands in for it.
static int stream_wait_readers(w2l_stream* s, long long f_end) {
    const long long cutoff = f_end - s->mel.rm;
    if (s->steps == 0 || cutoff <= s->first_lo) return W2L_OK;
    const long long tracked = std::min<long long>(s->steps, kStreamSlots);
    long long k = s->steps - 1;
    while (k > s->steps - tracked && s->step_lo[k % kStreamSlots] >= cutoff) --k;
    CK(cudaStreamWaitEvent(s->s_mel, s->step_done[k % kStreamSlots], 0));
    return W2L_OK;
}

// mel frames up to f_end on the mel stream, then the NaN flag; the caller's stream is ordered after them
static int stream_mel(w2l_stream* s, const MelParams& tables, long long f_end, long long L_end, cudaStream_t st) {
    CKR(stream_wait_readers(s, f_end));
    CKR(s->mel.compute(tables, f_end, L_end, s->s_mel));
    bool nan;
    CKR(s->mel.nan_seen(s->s_mel, &nan));     // before any row reads the new frames (and the audio copy is done)
    if (nan) { s->nan = true; return fail(W2L_EINVAL, "%s", kMelNanMsg); }
    CK(cudaStreamWaitEvent(st, s->mel.ev_nan, 0));
    return W2L_OK;
}

static int stream_pending(const w2l_stream* s, long long n_samples, bool finish, long long* n_out) {
    StreamSched::At a;
    CKR(s->sched.at(s->mel.L + n_samples, finish, &a));
    *n_out = std::max(0LL, a.n_fixed - s->emitted);
    return W2L_OK;
}

// rows [s->emitted + pend, a.n_fixed) join pend; full batches of pend run
static int stream_advance(w2l_stream* s, const StreamSched::At& a, std::vector<int32_t>* pend, uint8_t* out,
                          long long first, cudaStream_t st) {
    const size_t frame_bytes = (size_t)s->sched.d.H * s->sched.d.W * 3;
    long long next = s->emitted + (long long)(pend->size() / W2L_STREAM_ROW);
    for (; next < a.n_fixed; ++next) {
        int32_t r[W2L_STREAM_ROW];
        CKR(s->sched.row(next, a, r));
        pend->insert(pend->end(), r, r + W2L_STREAM_ROW);
    }
    while ((long long)(pend->size() / W2L_STREAM_ROW) >= s->batch) {
        CKR(stream_step(s, pend->data(), s->batch, out + (size_t)(s->emitted - first) * frame_bytes, st));
        pend->erase(pend->begin(), pend->begin() + (size_t)s->batch * W2L_STREAM_ROW);
    }
    return W2L_OK;
}

static int stream_run(w2l_stream* s, const float* pcm, long long n, bool finish, uint8_t* out, long long cap,
                      long long* first_index, long long* n_out, cudaStream_t st) {
    if (s->nan) return fail(W2L_EINVAL, "%s", kMelNanMsg);
    if (s->finished) return fail(W2L_ESTATE, "the stream is finished");
    if (n < 0 || (n > 0 && !pcm)) return fail(W2L_EINVAL, "bad audio piece (%lld samples)", n);
    long long need;
    CKR(stream_pending(s, n, finish, &need));
    if (need > cap || (need > 0 && !out)) return fail(W2L_EINVAL, "output holds %lld frames, this call emits %lld", cap, need);
    DeviceGuard g(s->ctx->device);
    const long long first = s->emitted;
    *first_index = first;
    *n_out = 0;
    const MelParams tables = mel_tables(s->ctx);
    if (n > 0) {
        int kind;
        CKR(pcm_kind(s->ctx, pcm, &kind));
        if (kind == PCM_DEVICE) {   // device audio may be produced by work queued on the caller's stream
            CK(cudaEventRecord(s->ev_caller, st));
            CK(cudaStreamWaitEvent(s->s_mel, s->ev_caller, 0));
        }
    }
    std::vector<int32_t> pend;
    StreamSched::At a;
    long long done = 0;
    while (done < n) {
        const long long keep = std::min(s->mel.f_next, s->sched.start(s->emitted));
        const long long piece = std::min(n - done, s->mel.max_piece(keep));
        if (piece <= 0) return fail(W2L_ESTATE, "mel ring too small for the pending rows");
        CKR(s->mel.append(pcm + done, piece, s->s_mel));
        done += piece;
        CKR(stream_mel(s, tables, mel_final_frames(s->mel.L), -1, st));
        CKR(s->sched.at(s->mel.L, false, &a));
        CKR(stream_advance(s, a, &pend, out, first, st));
    }
    if (finish) {
        CKR(s->sched.at(s->mel.L, true, &a));
        const long long keep = std::min(std::min(s->mel.f_next, s->sched.start(s->emitted)), a.M - 16);
        if (a.M - keep > s->mel.rm) return fail(W2L_ESTATE, "mel ring too small for the pending rows");
        CKR(stream_mel(s, tables, a.M, s->mel.L, st));
        CKR(stream_advance(s, a, &pend, out, first, st));
        s->finished = true;
    }
    if (!pend.empty()) {
        const size_t frame_bytes = (size_t)s->sched.d.H * s->sched.d.W * 3;
        CKR(stream_step(s, pend.data(), (int)(pend.size() / W2L_STREAM_ROW), out + (size_t)(s->emitted - first) * frame_bytes, st));
    }
    *n_out = s->emitted - first;
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// C-ABI (declared in include/w2l.h)
// ------------------------------------------------------------------------------------------------
int w2l_melstream_create(w2l_ctx* ctx, int audio_ring_log2, w2l_melstream** out) {
    if (!ctx || !out) return fail(W2L_EINVAL, "null argument");
    *out = nullptr;
    DeviceGuard g(ctx->device);
    std::unique_ptr<w2l_melstream> ms(new w2l_melstream());
    ms->ctx = ctx;
    CKR(ms->ring.init(ctx, audio_ring_log2, 0));
    *out = ms.release();
    return W2L_OK;
}

int64_t w2l_melstream_pending(const w2l_melstream* ms, int64_t n_samples, int finish) {
    if (!ms || n_samples < 0) return 0;
    const MelRing& r = ms->ring;
    if (r.finished) return 0;
    const long long L = r.L + n_samples;
    const long long total = finish ? (L >= 2 ? 1 + L / MEL_HOP : 0) : mel_final_frames(L);
    return std::max(0LL, total - r.f_next);
}

static int melstream_run(w2l_melstream* ms, const float* pcm, long long n, bool finish, float* mel_out, long long cap,
                         int64_t* n_new, int* nan_seen, cudaStream_t st) {
    if (!ms || !n_new) return fail(W2L_EINVAL, "null argument");
    MelRing& r = ms->ring;
    if (r.finished) return fail(W2L_ESTATE, "the stream is finished");
    if (n < 0 || (n > 0 && !pcm)) return fail(W2L_EINVAL, "bad audio piece (%lld samples)", n);
    if (finish && r.L + n < 2) return fail(W2L_EINVAL, "need at least 2 samples (got %lld)", r.L + n);
    const long long need = w2l_melstream_pending(ms, n, finish);
    if (need > cap || (need > 0 && !mel_out)) return fail(W2L_EINVAL, "output holds %lld frames, this call gives %lld", cap, need);
    DeviceGuard g(ms->ctx->device);
    const MelParams tables = mel_tables(ms->ctx);
    int kind = PCM_PAGEABLE;
    if (n > 0) CKR(pcm_kind(ms->ctx, pcm, &kind));
    const long long first = r.f_next;
    long long done = 0;
    while (done < n) {
        const long long piece = std::min(n - done, r.max_piece(r.f_next));
        CKR(r.append(pcm + done, piece, st));
        done += piece;
        const long long a = r.f_next;
        CKR(r.compute(tables, mel_final_frames(r.L), -1, st));
        CKR(r.copy_out(a, r.f_next, mel_out, need, a - first, st));
    }
    if (finish) {
        const long long a = r.f_next;
        CKR(r.compute(tables, 1 + r.L / MEL_HOP, r.L, st));
        CKR(r.copy_out(a, r.f_next, mel_out, need, a - first, st));
        r.finished = true;
    }
    *n_new = r.f_next - first;
    if (kind == PCM_PINNED) {   // the copies read pinned memory when they run: let the caller reuse it on return
        CK(cudaEventRecord(r.ev_nan, st));
        CK(cudaEventSynchronize(r.ev_nan));
    }
    if (nan_seen) {
        bool nan;
        CKR(r.nan_seen(st, &nan));
        *nan_seen = nan ? 1 : 0;
    }
    return W2L_OK;
}

int w2l_melstream_push(w2l_melstream* ms, const float* pcm, int64_t n_samples, float* mel_dev, int64_t cap_frames,
                       int64_t* n_new, int* nan_seen, void* stream) {
    return melstream_run(ms, pcm, n_samples, false, mel_dev, cap_frames, n_new, nan_seen, (cudaStream_t)stream);
}

int w2l_melstream_finish(w2l_melstream* ms, float* mel_dev, int64_t cap_frames, int64_t* n_new, int* nan_seen, void* stream) {
    return melstream_run(ms, nullptr, 0, true, mel_dev, cap_frames, n_new, nan_seen, (cudaStream_t)stream);
}

int w2l_melstream_destroy(w2l_melstream* ms) {
    if (!ms) return W2L_OK;
    DeviceGuard g(ms->ctx->device);
    cudaDeviceSynchronize();   // queued kernels may still read the rings
    delete ms;
    return W2L_OK;
}

int w2l_stream_schedule(const w2l_stream_desc* d, const int32_t* rects_host, int64_t n_samples, int final_,
                        int64_t first_row, int64_t cap, int32_t* rows_host, int64_t* n_fixed) {
    if (!n_fixed || n_samples < 0 || first_row < 0 || cap < 0 || (cap > 0 && !rows_host)) return fail(W2L_EINVAL, "bad argument");
    StreamSched sc;
    CKR(sc.init(d, rects_host));
    StreamSched::At a;
    CKR(sc.at(n_samples, final_ != 0, &a));
    *n_fixed = a.n_fixed;
    for (long long i = first_row; i < a.n_fixed && i < first_row + cap; ++i)
        CKR(sc.row(i, a, rows_host + (size_t)(i - first_row) * W2L_STREAM_ROW));
    return W2L_OK;
}

int w2l_stream_detect_need(const w2l_stream_desc* d, int64_t n_samples, int final_, int64_t* n_frames) {
    if (!n_frames || n_samples < 0) return fail(W2L_EINVAL, "bad argument");
    StreamSched sc;
    CKR(sc.init(d, nullptr, true));
    StreamSched::At a;
    CKR(sc.at(n_samples, final_ != 0, &a));
    *n_frames = sc.need(a);
    return W2L_OK;
}

int w2l_stream_create(w2l_ctx* ctx, const uint8_t* frames_dev, const w2l_stream_desc* d, const int32_t* rects_host,
                      int batch, w2l_stream** out) {
    if (!ctx || !frames_dev || !d || !out) return fail(W2L_EINVAL, "null argument");
    *out = nullptr;
    if (batch < 1 || batch > 4096) return fail(W2L_EINVAL, "batch %d: need 1 .. 4096", batch);
    std::unique_ptr<w2l_stream> s(new w2l_stream());
    s->ctx = ctx;
    CKR(s->sched.init(d, rects_host));
    DeviceGuard g(ctx->device);
    cudaPointerAttributes pa;
    const cudaError_t e = cudaPointerGetAttributes(&pa, frames_dev);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(W2L_EINVAL, "frames: cudaPointerGetAttributes: %s", cudaGetErrorString(e)); }
    if (pa.type != cudaMemoryTypeDevice || pa.device != ctx->device)
        return fail(W2L_EINVAL, "frames must be device memory of the context's device %d", ctx->device);
    if (!ctx->nets[W2L_NET_GENERATOR].loaded) return fail(W2L_ESTATE, "generator weights not loaded");
    s->frames = frames_dev;
    s->batch = batch;
    // the mel ring holds the frames of every row not yet run (< batch + 4 chunks) beside a whole audio ring of new ones
    CKR(s->mel.init(ctx, 0, (long long)std::ceil((batch + 4) * s->sched.mult) + 64 + (1LL << 16) / MEL_HOP + 16));
    CKR(s->table.grow(ctx, (size_t)batch * 6 * 4));
    CKR(s->stage.alloc((size_t)kStreamSlots * batch * 6 * 4));
    for (Event& ev : s->slot_done) CKR(ev.create());
    for (Event& ev : s->step_done) CKR(ev.create());
    CKR(s->ev_caller.create());
    CKR(s->s_mel.create());
    CKR(s->chunks.grow(ctx, (size_t)batch * 1280 * 4));
    CKR(s->crops.grow(ctx, (size_t)batch * 96 * 96 * 3));
    CKR(s->preds.grow(ctx, (size_t)batch * 96 * 96 * 3));
    CKR(s->cap.create());
    *out = s.release();
    return W2L_OK;
}

int w2l_stream_pending(const w2l_stream* s, int64_t n_samples, int finish, int64_t* n_out) {
    if (!s || !n_out || n_samples < 0) return fail(W2L_EINVAL, "bad argument");
    if (s->nan) return fail(W2L_EINVAL, "%s", kMelNanMsg);
    if (s->finished) { *n_out = 0; return W2L_OK; }
    long long n;
    CKR(stream_pending(s, n_samples, finish != 0, &n));
    *n_out = n;
    return W2L_OK;
}

int w2l_stream_push(w2l_stream* s, const float* pcm, int64_t n_samples, uint8_t* out_dev, int64_t cap,
                    int64_t* first_index, int64_t* n_out, void* stream) {
    if (!s || !first_index || !n_out) return fail(W2L_EINVAL, "null argument");
    long long f, n;
    const int r = stream_run(s, pcm, n_samples, false, out_dev, cap, &f, &n, (cudaStream_t)stream);
    *first_index = f; *n_out = n;
    return r;
}

int w2l_stream_finish(w2l_stream* s, uint8_t* out_dev, int64_t cap, int64_t* first_index, int64_t* n_out, void* stream) {
    if (!s || !first_index || !n_out) return fail(W2L_EINVAL, "null argument");
    long long f, n;
    const int r = stream_run(s, nullptr, 0, true, out_dev, cap, &f, &n, (cudaStream_t)stream);
    *first_index = f; *n_out = n;
    return r;
}

int w2l_stream_destroy(w2l_stream* s) {
    if (!s) return W2L_OK;
    DeviceGuard g(s->ctx->device);
    cudaDeviceSynchronize();   // queued steps may still read the session's buffers
    stream_release_plan(s);
    delete s;
    return W2L_OK;
}
