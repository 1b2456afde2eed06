// host_stream.cuh — streaming: the mel rings behind w2l_melstream_* and the lip-sync session behind w2l_stream_*
// (DESIGN.md section 3.8).  The scheduling rules (which rows the audio received so far fixes) are host code with no
// device state, exported as w2l_stream_schedule so that they can be tested without a GPU.  The piece planner
// (MelRing::plan), the generator steps (StepRunner) and the ring-reader tracking (RingReaders) serve stream groups
// (host_stream_group.cuh) as well.
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
// The next piece of a stream's input and what it makes final (MelRing::plan).
struct MelPiece {
    long long n = 0;            // input samples
    ResampleClock clk;          // the resampling clock after them
    long long L = 0;            // the 16 kHz length after them
    bool input_end = false;     // the end of the input is resampled with them (its right wings stop there)
    long long f_end = 0;        // mel frames final after them
    long long L_end = -1;       // at finish: the final length, where the last frames reflect; else -1
    bool fin = false;           // the piece ends the stream: frames [f_next, f_end) are all there are
};

struct MelRing {
    w2l_ctx* ctx = nullptr;
    long long ra = 0, rm = 0;   // audio ring (samples), mel ring (frames)
    DevMem<float> audio, mel;
    DevMem<int> nan;
    PinnedMem nan_host;
    Event ev_nan;
    long long L = 0;            // 16 kHz samples in the audio ring: received, or resampled from the input
    long long f_next = 0;       // frames computed: [0, f_next)
    bool finished = false;
    // Resampling (set_rate, DESIGN.md section 3.11): the input arrives at sr into a ring of its own and the outputs its
    // samples make final are resampled into the audio ring, so L stays the 16 kHz count everything downstream uses.
    int sr = 16000;
    ResampleClock clk;          // clk.t == L
    long long n_in = 0;         // input samples received
    long long rsrc = 0;         // input ring length (samples)
    DevMem<float> src;
    DevMem<double> reg0;        // block start registers of one launch
    const double2* wd = nullptr;

    bool resampling() const { return sr != 16000; }

    int set_rate(int rate) {
        if (!rs_rate_ok(rate)) return fail(W2L_EINVAL, "input rate %d Hz: need an integer rate of 4000 .. 192000 Hz", rate);
        if (L > 0 || n_in > 0 || finished) return fail(W2L_ESTATE, "the input rate must be set before the first audio");
        if (rate == 16000 || rate == sr) { sr = rate; return W2L_OK; }
        ResampleClock c;
        CKR(c.init(rate, 16000));
        const double2* t;
        CKR(resample_table(ctx, c.ratio, &t));
        // the input of a full audio ring, plus the left wing of the oldest pending output, rounded up to a power of two
        const long long n = pow2_at_least((long long)std::ceil((double)ra * c.inc) + 2 * (RS_NWIN / c.step + 2));
        CKR(src.grow(ctx, (size_t)n * 4));
        CKR(reg0.grow(ctx, (size_t)(ra / RS_THREADS + 2) * 8));
        rsrc = n; clk = c; wd = t; sr = rate;
        return W2L_OK;
    }

    // L after n more input samples (final: and the end of the input)
    long long samples_after(long long n, bool final) const {
        if (!resampling()) return L + n;
        ResampleClock c = clk;
        return c.advance(n_in + n, final, nullptr);
    }

    // Longest next piece of input whose outputs fit max_out more 16 kHz samples and which overwrites no input sample
    // that a pending output's left wing reads.
    long long max_input(long long max_out) const {
        if (!resampling()) return max_out;
        const long long by_src = rsrc - (n_in - clk.oldest_read());
        // outputs of n_in + k samples are at most n_res(n_in + k) <= (n_in + k) * ratio
        const long long by_out = (long long)((double)(L + max_out) * clk.inc) - n_in - 2;
        return std::min(by_src, by_out);
    }

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

    // The next piece: at most `left` input samples (ends: the input ends after them), as many as overwrite nothing that
    // is still read (max_piece, max_input; keep: the oldest mel frame the consumer still needs).  starts gets the
    // register of every RS_THREADS-th output the piece resamples.  The end of the input is taken only once its last
    // outputs fit the audio ring and its last frames, from the right-aligned last chunk (M - 16) on, fit the mel ring;
    // until then the piece stops short of it and a later one, after the consumer has moved on, ends the stream.  A piece
    // that would make no progress is W2L_ESTATE.
    int plan(long long left, bool ends, long long keep, MelPiece* out, std::vector<double>* starts) const {
        const long long room = max_piece(keep);
        MelPiece p;
        p.n = std::max(0LL, std::min(left, max_input(room)));
        p.input_end = ends && p.n == left;
        p.L = L + p.n;
        starts->clear();
        if (resampling()) {
            p.clk = clk;
            p.L = p.clk.advance(n_in + p.n, p.input_end, starts);
            if (p.input_end && p.L - L > room) {
                starts->clear();
                p.clk = clk;
                p.L = p.clk.advance(n_in + p.n, false, starts);
                p.input_end = false;
            }
        }
        p.f_end = mel_final_frames(p.L);
        if (p.input_end) {
            const long long M = 1 + p.L / MEL_HOP;   // the mel frames of the whole input (StreamSched::at at final)
            if (M - std::min(keep, M - 16) <= rm) { p.fin = true; p.f_end = M; p.L_end = p.L; }
        }
        if (p.n == 0 && p.L == L && !p.fin) return fail(W2L_ESTATE, "audio or mel ring too small for the next piece");
        *out = p;
        return W2L_OK;
    }

    // where a piece's input goes: the input ring of a resampling stream, else the audio ring
    GroupScatter input_of(const MelPiece& p, const float* pcm) const {
        if (resampling()) return GroupScatter{pcm, src.p, rsrc - 1, n_in, p.n};
        return GroupScatter{pcm, audio.p, ra - 1, L, p.n};
    }

    void resample_args(const MelPiece& p, const double* reg, int* flag, ResampleParams* rp, ResampleRingParams* r) const {
        const long long n1 = n_in + p.n;
        *rp = resample_params(clk, wd, reg, L, p.L, p.input_end ? clk.n_res(n1) : (1LL << 62));
        r->src = src; r->src_mask = rsrc - 1; r->n_in = p.input_end ? n1 : (1LL << 62);
        r->audio = audio; r->audio_mask = ra - 1; r->nan = flag;
    }

    // the piece's frames [f_next, p.f_end); L_end >= 0 only at finish (reflection at the end of the utterance)
    MelRingParams mel_args(const MelPiece& p, int* flag) const {
        MelRingParams r;
        r.audio = audio; r.audio_mask = ra - 1; r.mel = mel; r.mel_pitch = rm;
        r.L = p.L_end >= 0 ? p.L_end : (1LL << 62);
        r.f0 = f_next; r.f1 = p.f_end; r.nan = flag;
        return r;
    }

    // Queues a planned piece on st: its input (pcm: host memory of any kind, or device memory) copied into its ring at
    // absolute positions, the outputs it makes final resampled into the audio ring, and, once `readers` (if any) has
    // completed, its mel frames.  The ring is unchanged until commit.
    int launch(const MelPiece& p, const float* pcm, const std::vector<double>& starts, const MelParams& tables,
               cudaEvent_t readers, cudaStream_t st) {
        const GroupScatter in = input_of(p, pcm);
        for (long long done = 0; done < in.n;) {
            const long long at = (in.at + done) & in.mask;
            const long long k = std::min(in.n - done, in.mask + 1 - at);
            CK(cudaMemcpyAsync(in.ring + at, pcm + done, (size_t)k * 4, cudaMemcpyDefault, st));
            done += k;
        }
        if (!starts.empty()) {
            CK(cudaMemcpyAsync(reg0.p, starts.data(), starts.size() * 8, cudaMemcpyHostToDevice, st));
            ResampleParams rp;
            ResampleRingParams r;
            resample_args(p, reg0, nan, &rp, &r);
            resample_ring_kernel<<<(unsigned)starts.size(), RS_THREADS, 0, st>>>(rp, r);
            ctx->launches++;
            CK(cudaGetLastError());
        }
        if (p.f_end > f_next) {
            if (readers) CK(cudaStreamWaitEvent(st, readers, 0));
            const long long blocks = (p.f_end - f_next + MEL_FPB - 1) / MEL_FPB;
            mel_ring_kernel<<<(unsigned)blocks, MEL_THREADS, kMelSmemBytes, st>>>(tables, mel_args(p, nan));
            ctx->launches++;
            CK(cudaGetLastError());
        }
        return W2L_OK;
    }

    void commit(const MelPiece& p) {
        if (resampling()) { clk = p.clk; n_in += p.n; }
        L = p.L;
        f_next = std::max(f_next, p.f_end);
        finished = p.fin;
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
// generator steps over stream rows: the lone session's and the stream group's (host_stream_group.cuh)
// ------------------------------------------------------------------------------------------------
constexpr int kStepSlots = 4;     // pinned staging slots of the per-step table in flight
constexpr int kStepEvents = 16;   // step-completion events the ring-safety wait chooses from
constexpr int kReaderTrack = 4;   // the last steps each session remembers (step id, lowest chunk start)

// One step size: its generator plan and the CUDA graph of its step.  The plan is pinned against LRU eviction while held
// and valid while epoch matches: it is erased, with every generator plan, only by drop_plans (new weights), which
// bumps the epoch.  So a matching epoch means the plan, and every buffer the graph bakes, is alive and current.
struct StepBucket {
    int B = 0;
    Plan* plan = nullptr;
    uint64_t epoch = 0;
    GraphExec exec;
    bool warm = false;               // one uncaptured step ran on the current plan (kernel attributes are set)
};

// The step buffers.  Every pointer a step reads or writes is in its device table, one GroupRow per row, so the whole
// step (gather, crop, generator, paste) is captured once per bucket and replayed whatever rows it runs.  The table
// (max_batch rows) is shared by the buckets because steps run in order on the caller's stream; each step fills it with
// one copy from a pinned slot.
struct StepRunner {
    w2l_ctx* ctx = nullptr;
    int max_batch = 0;
    DevMem<GroupRow> table;
    PinnedMem table_host;            // kStepSlots x max_batch rows
    Event table_done[kStepSlots];
    Event step_done[kStepEvents];    // after step k (k % kStepEvents) on the caller's stream
    long long count = 0;             // steps queued
    DevMem<float> chunks;
    DevMem<uint8_t> crops, preds;
    Stream cap;                      // capture stream (the graph is launched on the caller's stream)
    int64_t calls = 0, waits = 0;    // CUDA API submissions (launches, graph launches, copies, event records and waits)
                                     // and host synchronisations (a stream group counts its ticks' here)

    int init(w2l_ctx* c, int max_b) {
        ctx = c;
        max_batch = max_b;
        for (Event& e : table_done) CKR(e.create());
        for (Event& e : step_done) CKR(e.create());
        CKR(table.grow(ctx, (size_t)max_batch * sizeof(GroupRow)));
        CKR(table_host.alloc((size_t)kStepSlots * max_batch * sizeof(GroupRow)));
        CKR(chunks.grow(ctx, (size_t)max_batch * 1280 * 4));
        CKR(crops.grow(ctx, (size_t)max_batch * 96 * 96 * 3));
        CKR(preds.grow(ctx, (size_t)max_batch * 96 * 96 * 3));
        return cap.create();
    }

    void release(StepBucket* b) {
        if (b->plan && b->epoch == ctx->plan_epoch[W2L_NET_GENERATOR]) b->plan->pins--;
        b->plan = nullptr;
        b->exec.reset();
        b->warm = false;
    }

    int acquire(StepBucket* b) {
        if (b->plan && b->epoch == ctx->plan_epoch[W2L_NET_GENERATOR]) return W2L_OK;
        release(b);
        Plan* pl;
        CKR(get_plan(ctx, W2L_NET_GENERATOR, b->B, 0, &pl));
        pl->pins++;
        b->plan = pl;
        b->epoch = ctx->plan_epoch[W2L_NET_GENERATOR];
        return W2L_OK;
    }

    // gather + crop + generator + paste of B table rows
    int body(const StepBucket& b, cudaStream_t st) {
        const int B = b.B;
        group_gather_kernel<<<(B * 1280 + 255) / 256, 256, 0, st>>>(table, B, chunks);
        const long long total = (long long)B * 96 * 96;
        group_crop_kernel<<<(int)std::min<long long>((total + 255) / 256, ctx->num_sms * 16), 256, 0, st>>>(table, B, 96, crops);
        ctx->launches += 2;
        CK(cudaGetLastError());
        CKR(run_plan(ctx, b.plan, chunks, crops, preds, nullptr, st, true));
        // about 8 blocks per SM over the step, each row's frame split across gridDim.x of them
        const dim3 grid((unsigned)std::max(1, (ctx->num_sms * 8 + B - 1) / B), (unsigned)B);
        group_paste_kernel<<<grid, 256, 0, st>>>(preds, 96, table);
        ctx->launches++;
        CK(cudaGetLastError());
        return W2L_OK;
    }

    int capture(StepBucket* b) {
        cudaGraph_t gr = nullptr;
        CK(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
        const int r = body(*b, cap);
        const cudaError_t e = cudaStreamEndCapture(cap, &gr);
        if (r != W2L_OK) { if (gr) cudaGraphDestroy(gr); cudaGetLastError(); return r; }
        CK(e);
        const cudaError_t ei = cudaGraphInstantiate(&b->exec.h, gr, 0);
        cudaGraphDestroy(gr);
        CK(ei);
        return W2L_OK;
    }

    // One step of bucket b over rows [0, n) (n <= b->B): row(k) gives the GroupRow of row k.  Rows past n repeat the
    // last one and are not pasted.  *id gets the step's id; step_done[*id % kStepEvents] is recorded after it.
    template <class Row>
    int step(StepBucket* b, int n, Row row, cudaStream_t st, long long* id) {
        CKR(acquire(b));
        *id = count++;
        const int slot = (int)(*id % kStepSlots);
        CK(cudaEventSynchronize(table_done[slot]));       // its previous copy has read the staging slot
        waits++;
        GroupRow* h = (GroupRow*)table_host.p + (size_t)slot * max_batch;
        for (int k = 0; k < b->B; ++k) {
            if (k < n) h[k] = row(k);
            else { h[k] = h[n - 1]; h[k].dst = nullptr; }
        }
        CK(cudaMemcpyAsync(table, h, (size_t)b->B * sizeof(GroupRow), cudaMemcpyHostToDevice, st));
        CK(cudaEventRecord(table_done[slot], st));
        calls += 2;
        if (!ctx->use_stream_graph || !b->warm) {
            CKR(body(*b, st));
            b->warm = true;
        } else {
            if (!b->exec.h) CKR(capture(b));
            CK(cudaGraphLaunch(b->exec.h, st));
            calls++;
        }
        CK(cudaEventRecord(step_done[*id % kStepEvents], st));   // its gather has read the mel rings
        calls++;
        return W2L_OK;
    }
};

// a row (W2L_STREAM_ROW ints) of a session with mel ring m, video frames and description d, pasted into dst
static GroupRow step_row(const MelRing& m, const uint8_t* frames, const w2l_stream_desc& d, const int32_t* r, uint8_t* dst) {
    GroupRow g;
    g.mel = m.mel; g.pitch = m.rm; g.start = r[1];
    g.frames = frames; g.dst = dst;
    g.H = d.H; g.W = d.W; g.frame = r[2];
    g.y1 = r[3]; g.y2 = r[4]; g.x1 = r[5]; g.x2 = r[6]; g.pad = 0;
    return g;
}

// The steps that read a session's mel ring.  Before the ring kernel writes frames [f_next, f_end) into columns that
// held frames below f_end - rm, the mel stream waits for the last queued step that reads such a frame.  Steps read
// from their lowest chunk start upwards and a session's starts never decrease from step to step, so that step is the
// newest one whose lowest start is below the cutoff.
struct RingReaders {
    long long first_lo = -1;                          // the lowest mel frame of the session's first step
    long long step[kReaderTrack], lo[kReaderTrack];   // its last steps and their lowest mel frames, oldest first
    int n = 0;

    void track(long long id, long long start) {
        if (first_lo < 0) first_lo = start;
        if (n > 0 && step[n - 1] == id) return;   // rows of one step: the first has the lowest start
        if (n == kReaderTrack) {
            for (int k = 1; k < kReaderTrack; ++k) { step[k - 1] = step[k]; lo[k - 1] = lo[k]; }
            --n;
        }
        step[n] = id; lo[n] = start; ++n;
    }

    // The step to wait for before frames below f_end are written into a ring of rm columns (-1: none).  When it is
    // older than the steps remembered, the oldest remembered one (after it on the caller's stream) stands in for it.
    long long reader(long long f_end, long long rm) const {
        const long long cutoff = f_end - rm;
        if (n == 0 || cutoff <= first_lo) return -1;
        int k = n - 1;
        while (k > 0 && lo[k] >= cutoff) --k;
        return step[k];
    }
};

// The video of a session: device memory on the context's device, frames under 2^31 bytes (the paste's offsets within
// a frame are 32-bit), and the generator to run on it loaded.
static int check_stream_frames(const w2l_ctx* ctx, const uint8_t* frames, const w2l_stream_desc& d) {
    if ((long long)d.H * d.W * 3 > INT32_MAX) return fail(W2L_EINVAL, "a %dx%d frame: need fewer than 2^31 bytes", d.H, d.W);
    cudaPointerAttributes pa;
    const cudaError_t e = cudaPointerGetAttributes(&pa, frames);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(W2L_EINVAL, "frames: cudaPointerGetAttributes: %s", cudaGetErrorString(e)); }
    if (pa.type != cudaMemoryTypeDevice || pa.device != ctx->device)
        return fail(W2L_EINVAL, "frames must be device memory of the context's device %d", ctx->device);
    if (!ctx->nets[W2L_NET_GENERATOR].loaded) return fail(W2L_ESTATE, "generator weights not loaded");
    return W2L_OK;
}

// ------------------------------------------------------------------------------------------------
// the session
// ------------------------------------------------------------------------------------------------
struct w2l_stream {
    w2l_ctx* ctx = nullptr;
    StreamSched sched;
    MelRing mel;
    const uint8_t* frames = nullptr;
    long long emitted = 0;          // rows whose step has been queued
    bool nan = false;
    // The mel work (audio copy, ring kernel, NaN flag read-back) runs on a private stream, so that the host, which waits
    // for each piece's NaN flag before it schedules rows, waits for this session's mel frames only, not for the steps
    // queued on the caller's stream.
    Stream s_mel;
    Event ev_caller;                // the caller's stream, before a piece of device audio is copied
    StepRunner steps;
    StepBucket bucket;              // every step runs at B = batch
    RingReaders readers;
};

// Full batches of pend run (all: and the rest, in one step padded to the batch); output frames go to out from row first.
static int stream_flush(w2l_stream* s, std::vector<int32_t>* pend, uint8_t* out, long long first, bool all, cudaStream_t st) {
    const size_t frame_bytes = (size_t)s->sched.d.H * s->sched.d.W * 3;
    const size_t B = (size_t)s->bucket.B;
    while (pend->size() >= B * W2L_STREAM_ROW || (all && !pend->empty())) {
        const int n = (int)std::min(B, pend->size() / W2L_STREAM_ROW);
        const int32_t* rows = pend->data();
        uint8_t* o = out + (size_t)(s->emitted - first) * frame_bytes;
        long long id;
        CKR(s->steps.step(&s->bucket, n, [&](int k) {
            return step_row(s->mel, s->frames, s->sched.d, rows + (size_t)k * W2L_STREAM_ROW, o + (size_t)k * frame_bytes);
        }, st, &id));
        s->readers.track(id, rows[1]);   // rows are in output order: the first has the lowest start
        s->emitted += n;
        pend->erase(pend->begin(), pend->begin() + (size_t)n * W2L_STREAM_ROW);
    }
    return W2L_OK;
}

static int stream_pending(const w2l_stream* s, long long n_samples, bool finish, long long* n_out) {
    StreamSched::At a;
    CKR(s->sched.at(s->mel.samples_after(n_samples, finish), finish, &a));
    *n_out = std::max(0LL, a.n_fixed - s->emitted);
    return W2L_OK;
}

static int stream_run(w2l_stream* s, const float* pcm, long long n, bool finish, uint8_t* out, long long cap,
                      long long* first_index, long long* n_out, cudaStream_t st) {
    if (s->nan) return fail(W2L_EINVAL, "%s", kMelNanMsg);
    if (s->mel.finished) return fail(W2L_ESTATE, "the stream is finished");
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
    MelRing& m = s->mel;
    std::vector<int32_t> pend;
    std::vector<double> starts;
    for (long long done = 0; done < n || (finish && !m.finished); ) {
        MelPiece p;
        CKR(m.plan(n - done, finish, std::min(m.f_next, s->sched.start(s->emitted)), &p, &starts));
        const long long rd = s->readers.reader(p.f_end, m.rm);
        CKR(m.launch(p, pcm + done, starts, tables, rd >= 0 ? (cudaEvent_t)s->steps.step_done[rd % kStepEvents] : nullptr,
                     s->s_mel));
        m.commit(p);
        done += p.n;
        bool nan;
        CKR(m.nan_seen(s->s_mel, &nan));     // before any row reads the new frames (and the audio copy is done)
        if (nan) { s->nan = true; return fail(W2L_EINVAL, "%s", kMelNanMsg); }
        CK(cudaStreamWaitEvent(st, m.ev_nan, 0));
        StreamSched::At a;
        CKR(s->sched.at(m.L, p.fin, &a));
        for (long long i = s->emitted + (long long)(pend.size() / W2L_STREAM_ROW); i < a.n_fixed; ++i) {
            int32_t r[W2L_STREAM_ROW];
            CKR(s->sched.row(i, a, r));
            pend.insert(pend.end(), r, r + W2L_STREAM_ROW);
        }
        CKR(stream_flush(s, &pend, out, first, false, st));
    }
    CKR(stream_flush(s, &pend, out, first, true, st));
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
    const long long L = r.samples_after(n_samples, finish != 0);
    const long long total = finish ? (L >= 2 ? 1 + L / MEL_HOP : 0) : mel_final_frames(L);
    return std::max(0LL, total - r.f_next);
}

static int melstream_run(w2l_melstream* ms, const float* pcm, long long n, bool finish, float* mel_out, long long cap,
                         int64_t* n_new, int* nan_seen, cudaStream_t st) {
    if (!ms || !n_new) return fail(W2L_EINVAL, "null argument");
    MelRing& r = ms->ring;
    if (r.finished) return fail(W2L_ESTATE, "the stream is finished");
    if (n < 0 || (n > 0 && !pcm)) return fail(W2L_EINVAL, "bad audio piece (%lld samples)", n);
    if (finish && r.samples_after(n, true) < 2)
        return fail(W2L_EINVAL, "need at least 2 samples at 16 kHz (got %lld)", r.samples_after(n, true));
    const long long need = w2l_melstream_pending(ms, n, finish);
    if (need > cap || (need > 0 && !mel_out)) return fail(W2L_EINVAL, "output holds %lld frames, this call gives %lld", cap, need);
    DeviceGuard g(ms->ctx->device);
    const MelParams tables = mel_tables(ms->ctx);
    int kind = PCM_PAGEABLE;
    if (n > 0) CKR(pcm_kind(ms->ctx, pcm, &kind));
    const long long first = r.f_next;
    std::vector<double> starts;
    for (long long done = 0; done < n || (finish && !r.finished); ) {
        MelPiece p;
        CKR(r.plan(n - done, finish, r.f_next, &p, &starts));
        CKR(r.launch(p, pcm + done, starts, tables, nullptr, st));
        CKR(r.copy_out(r.f_next, p.f_end, mel_out, need, r.f_next - first, st));
        r.commit(p);
        done += p.n;
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

int w2l_melstream_set_input_rate(w2l_melstream* ms, int sr) {
    if (!ms) return fail(W2L_EINVAL, "null argument");
    DeviceGuard g(ms->ctx->device);
    return ms->ring.set_rate(sr);
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
    CKR(check_stream_frames(ctx, frames_dev, *d));
    s->frames = frames_dev;
    s->bucket.B = batch;
    // the mel ring holds the frames of every row not yet run (< batch + 4 chunks) beside a whole audio ring of new ones
    CKR(s->mel.init(ctx, 0, (long long)std::ceil((batch + 4) * s->sched.mult) + 64 + (1LL << 16) / MEL_HOP + 16));
    CKR(s->steps.init(ctx, batch));
    CKR(s->ev_caller.create());
    CKR(s->s_mel.create());
    *out = s.release();
    return W2L_OK;
}

int w2l_stream_pending(const w2l_stream* s, int64_t n_samples, int finish, int64_t* n_out) {
    if (!s || !n_out || n_samples < 0) return fail(W2L_EINVAL, "bad argument");
    if (s->nan) return fail(W2L_EINVAL, "%s", kMelNanMsg);
    if (s->mel.finished) { *n_out = 0; return W2L_OK; }
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

int w2l_stream_set_input_rate(w2l_stream* s, int sr) {
    if (!s) return fail(W2L_EINVAL, "null argument");
    DeviceGuard g(s->ctx->device);
    return s->mel.set_rate(sr);
}

int w2l_stream_destroy(w2l_stream* s) {
    if (!s) return W2L_OK;
    DeviceGuard g(s->ctx->device);
    cudaDeviceSynchronize();   // queued steps may still read the session's buffers
    s->steps.release(&s->bucket);
    delete s;
    return W2L_OK;
}
