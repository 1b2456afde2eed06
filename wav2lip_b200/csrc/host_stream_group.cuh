// host_stream_group.cuh — stream groups behind w2l_stream_group_* (DESIGN.md section 3.9): many lip-sync sessions that
// share one context, one caller stream and one set of generator steps.  Each session keeps the rules of section 3.8
// (StreamSched) and a MelRing; a tick scatters every session's new audio and computes every session's new mel frames in
// one launch each, reads every NaN flag back in one copy, pools the rows that the audio fixes and runs them in as few
// steps as possible, each step one graph launch of a bucket size.
// Part of the single translation unit w2l_api.cu (included there, after host_stream.cuh).
#pragma once

// Bucket sizes: powers of two below max_batch, then max_batch.  n rows run as full max_batch steps, then the remainder
// in the smallest bucket that holds it.  Host only (w2l_stream_group_buckets).
static int group_bucket(int max_batch, long long n) {
    int b = 1;
    while (b < n && b < max_batch) b <<= 1;
    return std::min(b, max_batch);
}

// Face detection inside the group (DESIGN.md section 3.10).  Constants, not options: the detector batch of
// inference.py's --face_det_batch_size default, and the look-ahead that lets a tick at real-time audio find the rects it
// needs already read back.
constexpr int kDetMaxBatch = 16;
constexpr long long kDetOpenSamples = 6400;    // open: the frames the first 400 ms of audio need
constexpr long long kDetAheadSamples = 3200;   // after a tick: the frames need(L + 200 ms) adds

// S3FD batch of the next launch for r frames of one size: full 16s, a remainder above 8 as one 16, above 1 as 4s, else
// 1.  Three plans per frame size; padding (the last frame repeated) is at most 7 frames.
static int det_bucket(long long r) { return r > 8 ? 16 : r > 1 ? 4 : 1; }

struct GroupSession {
    int32_t id = -1;
    int slot = 0;                    // its NaN flag: w2l_stream_group::nan[slot]
    StreamSched sched;
    MelRing mel;
    const uint8_t* frames = nullptr;
    long long emitted = 0;           // rows whose step has been queued
    bool failed = false;
    std::string msg;                 // why it failed: the NaN message, or a detection's
    bool detect = false;             // rects found by the group's detector
    long long det_launched = 0;      // frames [0, det_launched) have a detection queued or read back
    long long det_ok = 0;            // frames [0, det_ok) were read back with a face
    std::vector<int8_t> det_status;  // per frame: -1 not read back yet, else kRectFace / kRectNone / kRectNonFinite
    RingReaders readers;             // the steps that read its mel ring, among the group's
};

// an S3FD plan of one (H, W, B), pinned while a detecting session of that frame size is open; valid while epoch matches
struct DetPlan {
    int H = 0, W = 0, B = 0;
    Plan* plan = nullptr;
    uint64_t epoch = 0;
};

// One detection launch: up to kDetMaxBatch frames of one size.  Device block: [frame pointers][dets (B, 1, 5) fp32]
// [counts][rects (B, 5) int32]; pinned block: [frame pointers][rects].
constexpr size_t kDetDevPtrs = 0, kDetDevDets = 128, kDetDevCounts = 448, kDetDevRects = 512, kDetDevBytes = 832;
constexpr size_t kDetHostRects = 128, kDetHostBytes = 448;
struct DetJob {
    int n = 0;                       // real frames (the rest repeat the last one)
    int32_t sid[kDetMaxBatch];
    int32_t frame[kDetMaxBatch];
    DevMem<uint8_t> dev;
    PinnedMem host;
};

struct w2l_stream_group {
    w2l_ctx* ctx = nullptr;
    int ring_log2 = 0;
    std::map<int32_t, std::unique_ptr<GroupSession>> sessions;
    int32_t next_id = 0;
    std::vector<int> free_slots;
    int n_slots = 0;
    // one sticky NaN flag per session slot, read back in one copy per round
    DevMem<int> nan;
    PinnedMem nan_host;
    int nan_cap = 0;
    // the round's upload: [GroupScatter x sessions][MelGroupBlock x blocks][host pcm], one H2D.  The mel stream is idle
    // after every round (its NaN read-back is waited for), so one device buffer and one pinned buffer serve every round.
    DevMem<uint8_t> up;
    PinnedMem up_host;
    size_t up_host_cap = 0;
    // The mel work runs on a stream of the group's own, so the round's host wait is for the new mel frames only, not for
    // the steps queued on the caller's stream.
    Stream s_mel;
    Event ev_mel, ev_caller;
    StepRunner steps;                // at max_batch; its counters count every call and host wait of the ticks
    std::vector<std::unique_ptr<StepBucket>> buckets;
    // Face detection runs on a stream of its own; ev_det follows the last launch.  Every launch is read back by the
    // next round's host wait (the mel stream waits for ev_det before its NaN read-back), so jobs are busy until then.
    Stream s_det;
    Event ev_det, ev_open;
    std::vector<std::unique_ptr<DetJob>> det_busy, det_free;
    std::vector<DetPlan> det_plans;
    std::map<std::pair<int, int>, int> det_sizes;   // open detecting sessions per (H, W)
};

static void group_det_release(w2l_stream_group* g, int H, int W) {
    auto& v = g->det_plans;
    for (DetPlan& p : v)
        if (p.H == H && p.W == W && p.plan && p.epoch == g->ctx->plan_epoch[W2L_NET_S3FD]) p.plan->pins--;
    v.erase(std::remove_if(v.begin(), v.end(), [&](const DetPlan& p) { return p.H == H && p.W == W; }), v.end());
}

// the S3FD plan of (H, W, B), pinned; after new weights (drop_plans) the old one is gone and a new one is taken
static int group_det_plan(w2l_stream_group* g, int H, int W, int B, Plan** out) {
    w2l_ctx* ctx = g->ctx;
    size_t k = 0;
    while (k < g->det_plans.size() && !(g->det_plans[k].H == H && g->det_plans[k].W == W && g->det_plans[k].B == B)) ++k;
    if (k < g->det_plans.size() && g->det_plans[k].plan && g->det_plans[k].epoch == ctx->plan_epoch[W2L_NET_S3FD]) {
        *out = g->det_plans[k].plan;
        return W2L_OK;
    }
    if (k == g->det_plans.size()) {
        DetPlan p;
        p.H = H; p.W = W; p.B = B;
        g->det_plans.push_back(p);
    }
    g->det_plans[k].plan = nullptr;
    Plan* pl;
    CKR(get_plan(ctx, W2L_NET_S3FD, B, 0, &pl, H, W));
    CKR(ensure_s3fd_detect(ctx, pl));
    pl->pins++;
    g->det_plans[k].plan = pl;
    g->det_plans[k].epoch = ctx->plan_epoch[W2L_NET_S3FD];
    *out = pl;
    return W2L_OK;
}

// one S3FD launch over fr[0, n) (n <= B frames of one size) on the detection stream, its rects read back to pinned memory
static int group_det_launch(w2l_stream_group* g, const std::pair<GroupSession*, long long>* fr, int n, int B) {
    w2l_ctx* ctx = g->ctx;
    const int H = fr[0].first->sched.d.H, W = fr[0].first->sched.d.W;
    Plan* pl;
    CKR(group_det_plan(g, H, W, B, &pl));
    std::unique_ptr<DetJob> j;
    if (!g->det_free.empty()) { j = std::move(g->det_free.back()); g->det_free.pop_back(); }
    else {
        j.reset(new DetJob());
        CKR(j->dev.grow(ctx, kDetDevBytes));
        CKR(j->host.alloc(kDetHostBytes));
    }
    const uint8_t** ptrs = (const uint8_t**)j->host.p;
    const size_t frame_bytes = (size_t)H * W * 3;
    for (int k = 0; k < B; ++k) {
        const auto& f = fr[std::min(k, n - 1)];
        ptrs[k] = f.first->frames + (size_t)f.second * frame_bytes;
    }
    for (int k = 0; k < n; ++k) { j->sid[k] = fr[k].first->id; j->frame[k] = (int32_t)fr[k].second; }
    j->n = n;
    uint8_t* dv = j->dev.p;
    CK(cudaMemcpyAsync(dv + kDetDevPtrs, ptrs, (size_t)B * sizeof(void*), cudaMemcpyHostToDevice, g->s_det));
    const long long l0 = ctx->launches;
    S3fdRun run{nullptr, 1, 1, (float*)(dv + kDetDevDets), (int32_t*)(dv + kDetDevCounts)};
    run.frame_ptrs = (const uint8_t* const*)(dv + kDetDevPtrs);
    CKR(run_plan(ctx, pl, nullptr, nullptr, nullptr, nullptr, g->s_det, false, nullptr, &run));
    s3fd_rect_export_kernel<<<1, 32, 0, g->s_det>>>((const float*)(dv + kDetDevDets), (const int*)(dv + kDetDevCounts), n, 1,
                                                    (int32_t*)(dv + kDetDevRects));
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync((uint8_t*)j->host.p + kDetHostRects, dv + kDetDevRects, (size_t)n * 5 * 4, cudaMemcpyDeviceToHost, g->s_det));
    g->steps.calls += 2 + (ctx->launches - l0);
    g->det_busy.push_back(std::move(j));
    return W2L_OK;
}

// Queue the detection of frames [det_launched, upto) of each (session, upto), pooled per frame size in launches of
// det_bucket frames, then record ev_det.
static int group_detect(w2l_stream_group* g, const std::vector<std::pair<GroupSession*, long long>>& upto) {
    std::map<std::pair<int, int>, std::vector<std::pair<GroupSession*, long long>>> by_size;
    for (const auto& u : upto) {
        GroupSession* s = u.first;
        for (long long f = s->det_launched; f < u.second; ++f) by_size[{s->sched.d.H, s->sched.d.W}].push_back({s, f});
    }
    if (by_size.empty()) return W2L_OK;
    for (const auto& kv : by_size) {
        const auto& fr = kv.second;
        for (size_t i = 0; i < fr.size();) {
            const int B = det_bucket((long long)(fr.size() - i));
            const int n = (int)std::min<size_t>((size_t)B, fr.size() - i);
            CKR(group_det_launch(g, fr.data() + i, n, B));
            i += n;
        }
    }
    for (const auto& u : upto) u.first->det_launched = std::max(u.first->det_launched, u.second);
    CK(cudaEventRecord(g->ev_det, g->s_det));
    g->steps.calls++;
    return W2L_OK;
}

// every busy job has completed (the caller waited): its rects go to their sessions, the job to the free list
static void group_det_resolve(w2l_stream_group* g) {
    for (auto& j : g->det_busy) {
        const int32_t* o = (const int32_t*)((const uint8_t*)j->host.p + kDetHostRects);
        for (int k = 0; k < j->n; ++k) {
            auto f = g->sessions.find(j->sid[k]);
            if (f == g->sessions.end()) continue;      // closed since
            GroupSession* s = f->second.get();
            s->det_status[j->frame[k]] = (int8_t)o[5 * k + 4];
            if (o[5 * k + 4] == kRectFace) s->sched.set_rect(j->frame[k], o + 5 * k);
        }
        g->det_free.push_back(std::move(j));
    }
    g->det_busy.clear();
}

// The first frame below n whose detection failed: face_boxes' message (inference.py:91-93), or the non-finite box's.
// Frames below n are read back by the time this is asked.
static bool group_det_failed(GroupSession* s, long long n, std::string* msg) {
    while (s->det_ok < n && s->det_status[s->det_ok] == kRectFace) ++s->det_ok;
    if (s->det_ok >= n) return false;
    const long long f = s->det_ok;
    char buf[160];
    if (s->det_status[f] == kRectNone)
        snprintf(buf, sizeof(buf), "Face not detected in frame %lld! Ensure the video contains a face in all the frames.", f);
    else if (s->det_status[f] == kRectNonFinite)
        snprintf(buf, sizeof(buf), "Face detector returned a non-finite box in frame %lld", f);
    else
        snprintf(buf, sizeof(buf), "frame %lld: its detection was not read back", f);
    *msg = buf;
    return true;
}

static StepBucket* group_bucket_of(w2l_stream_group* g, int B) {
    for (auto& b : g->buckets) if (b->B == B) return b.get();
    g->buckets.emplace_back(new StepBucket());
    g->buckets.back()->B = B;
    return g->buckets.back().get();
}

// one pooled row of a tick: the session, its row (W2L_STREAM_ROW ints) and its output frame
struct GroupPend {
    GroupSession* s;
    const int32_t* row;
    uint8_t* dst;
};

// one step over pend[0, n) (n <= max_batch) in the smallest bucket that holds it
static int group_step(w2l_stream_group* g, const GroupPend* pend, int n, cudaStream_t st) {
    long long id;
    CKR(g->steps.step(group_bucket_of(g, group_bucket(g->steps.max_batch, n)), n, [&](int k) {
        const GroupPend& p = pend[k];
        return step_row(p.s->mel, p.s->frames, p.s->sched.d, p.row, p.dst);
    }, st, &id));
    for (int k = 0; k < n; ++k) {
        pend[k].s->readers.track(id, pend[k].row[1]);
        pend[k].s->emitted++;
    }
    return W2L_OK;
}

// what a tick does with one of its sessions
struct GroupItem {
    GroupSession* s = nullptr;       // null: skipped (the session failed in an earlier tick)
    const float* pcm = nullptr;
    long long n = 0, done = 0;       // samples, and those already in the ring
    bool finish = false, device = false, failed = false;
    uint8_t* out = nullptr;
    long long first = 0;             // s->emitted when the tick began
    StreamSched::At last;            // the schedule once all of the tick's audio is in
    std::vector<int32_t> rows;       // rows [first, last.n_fixed), computed and checked before any launch
    long long queued = 0;            // rows of `rows` pooled so far
};

static int group_nan_capacity(w2l_stream_group* g, int slots) {
    if (slots <= g->nan_cap) return W2L_OK;
    const int cap = std::max(64, 2 * slots);
    DevMem<int> d;
    CKR(d.grow(g->ctx, (size_t)cap * 4));
    CK(cudaStreamSynchronize(g->s_mel));     // the ring kernels write the old flags on the mel stream
    CK(cudaMemset(d, 0, (size_t)cap * 4));
    if (g->nan_cap) CK(cudaMemcpy(d, g->nan, (size_t)g->nan_cap * 4, cudaMemcpyDeviceToDevice));
    g->nan = std::move(d);
    PinnedMem hm;
    CKR(hm.alloc((size_t)cap * 4));
    std::swap(g->nan_host.p, hm.p);
    g->nan_cap = cap;
    return W2L_OK;
}

static int group_upload_capacity(w2l_stream_group* g, size_t bytes) {
    CKR(g->up.grow(g->ctx, bytes));
    if (bytes > g->up_host_cap) {
        PinnedMem hm;
        CKR(hm.alloc(bytes + bytes / 2));
        std::swap(g->up_host.p, hm.p);
        g->up_host_cap = bytes + bytes / 2;
    }
    return W2L_OK;
}

// One round: every item's next piece of audio (at most what its rings take), its new mel frames, the NaN flags, and
// the rows that fixes pooled into pend; full max_batch steps of pend run.  *more: some item has audio left.
static int group_round(w2l_stream_group* g, std::vector<GroupItem>& items, std::vector<GroupPend>* pend, int32_t* status,
                       cudaStream_t st, bool* more) {
    w2l_ctx* ctx = g->ctx;
    const MelParams tables = mel_tables(ctx);
    std::vector<MelPiece> pl(items.size());
    std::vector<char> live(items.size(), 0);   // the item has a piece this round
    std::vector<GroupScatter> sc;
    std::vector<MelGroupBlock> mb;
    std::vector<ResampleGroupBlock> rb;
    std::vector<double> starts;
    size_t host_samples = 0;
    bool any_device = false, any = false;
    long long wait_step = -1;
    for (size_t i = 0; i < items.size(); ++i) {
        GroupItem& it = items[i];
        if (!it.s || it.failed || it.s->mel.finished) continue;
        GroupSession* s = it.s;
        if (it.done == it.n && !it.finish) continue;
        MelRing& m = s->mel;
        MelPiece& p = pl[i];
        if (m.plan(it.n - it.done, it.finish, std::min(m.f_next, s->sched.start(s->emitted)), &p, &starts) != W2L_OK)
            return fail(W2L_ESTATE, "session %d: %s", s->id, g_err.c_str());
        live[i] = any = true;
        int* flag = g->nan.p + s->slot;
        for (size_t b = 0; b < starts.size(); ++b) {   // only when the session resamples
            ResampleGroupBlock blk;
            m.resample_args(p, nullptr, flag, &blk.p, &blk.r);
            blk.tb = m.L + (long long)b * RS_THREADS;
            blk.reg = starts[b];
            rb.push_back(blk);
        }
        if (p.n > 0) {   // host pcm: an offset into the packed upload until it is packed
            sc.push_back(m.input_of(p, it.device ? it.pcm + it.done : (const float*)(uintptr_t)host_samples));
            if (it.device) any_device = true; else host_samples += (size_t)p.n;
        }
        const MelRingParams r = m.mel_args(p, flag);
        for (long long f = r.f0; f < r.f1; f += MEL_FPB)
            mb.push_back(MelGroupBlock{r.audio, r.audio_mask, r.mel, r.mel_pitch, r.L, f, r.f1, r.nan});
        if (p.f_end > m.f_next) wait_step = std::max(wait_step, s->readers.reader(p.f_end, m.rm));
    }
    *more = false;
    if (!any) return W2L_OK;

    // ---- the upload: descriptors and host pcm, packed into one pinned buffer, one copy ----
    const size_t o_mb = sc.size() * sizeof(GroupScatter);
    const size_t o_rb = (o_mb + mb.size() * sizeof(MelGroupBlock) + 15) / 16 * 16;
    const size_t o_pcm = (o_rb + rb.size() * sizeof(ResampleGroupBlock) + 15) / 16 * 16;
    const size_t bytes = o_pcm + host_samples * 4;
    CKR(group_upload_capacity(g, bytes));
    uint8_t* hp = (uint8_t*)g->up_host.p;
    {
        size_t k = 0;
        for (size_t i = 0; i < items.size(); ++i) {
            GroupItem& it = items[i];
            if (pl[i].n == 0) continue;
            GroupScatter& d = sc[k++];
            if (!it.device) {
                const size_t at = (size_t)(uintptr_t)d.src;
                memcpy(hp + o_pcm + at * 4, it.pcm + it.done, (size_t)pl[i].n * 4);
                d.src = (const float*)(g->up.p + o_pcm) + at;
            }
        }
    }
    memcpy(hp, sc.data(), o_mb);
    memcpy(hp + o_mb, mb.data(), mb.size() * sizeof(MelGroupBlock));
    memcpy(hp + o_rb, rb.data(), rb.size() * sizeof(ResampleGroupBlock));
    CK(cudaMemcpyAsync(g->up, hp, bytes, cudaMemcpyHostToDevice, g->s_mel));
    g->steps.calls++;
    if (any_device) {   // device audio may be produced by work queued on the caller's stream
        CK(cudaEventRecord(g->ev_caller, st));
        CK(cudaStreamWaitEvent(g->s_mel, g->ev_caller, 0));
        g->steps.calls += 2;
    }
    // the newest queued step that reads a mel column this round overwrites (the steps before it are done by then)
    if (wait_step >= 0) {
        CK(cudaStreamWaitEvent(g->s_mel, g->steps.step_done[wait_step % kStepEvents], 0));
        g->steps.calls++;
    }
    if (!sc.empty()) {
        long long longest = 0;
        for (const GroupScatter& d : sc) longest = std::max(longest, d.n);
        const dim3 grid((unsigned)std::min<long long>((longest + 255) / 256, 64), (unsigned)sc.size());
        group_scatter_kernel<<<grid, 256, 0, g->s_mel>>>((const GroupScatter*)g->up.p);
        ctx->launches++; g->steps.calls++;
        CK(cudaGetLastError());
    }
    if (!rb.empty()) {   // only when some session resamples: its new outputs into its audio ring
        resample_group_kernel<<<(unsigned)rb.size(), RS_THREADS, 0, g->s_mel>>>((const ResampleGroupBlock*)(g->up.p + o_rb));
        ctx->launches++; g->steps.calls++;
        CK(cudaGetLastError());
    }
    if (!mb.empty()) {
        mel_group_kernel<<<(unsigned)mb.size(), MEL_THREADS, kMelSmemBytes, g->s_mel>>>(tables, (const MelGroupBlock*)(g->up.p + o_mb));
        ctx->launches++; g->steps.calls++;
        CK(cudaGetLastError());
    }
    // the detection launched so far is read back within the same wait
    if (!g->det_busy.empty()) {
        CK(cudaStreamWaitEvent(g->s_mel, g->ev_det, 0));
        g->steps.calls++;
    }
    // every flag in one copy: the round's host wait (the upload's pinned buffer and host pcm are read by then)
    CK(cudaMemcpyAsync(g->nan_host.p, g->nan, (size_t)g->n_slots * 4, cudaMemcpyDeviceToHost, g->s_mel));
    CK(cudaEventRecord(g->ev_mel, g->s_mel));
    CK(cudaEventSynchronize(g->ev_mel));
    CK(cudaStreamWaitEvent(st, g->ev_mel, 0));
    g->steps.calls += 3; g->steps.waits++;
    group_det_resolve(g);

    const int* flags = (const int*)g->nan_host.p;
    for (size_t i = 0; i < items.size(); ++i) {
        GroupItem& it = items[i];
        const MelPiece& p = pl[i];
        if (!live[i]) continue;
        GroupSession* s = it.s;
        s->mel.commit(p);
        it.done += p.n;
        if (it.done < it.n || (it.finish && !p.fin)) *more = true;
        auto fail_session = [&](const std::string& msg) {   // its rows of this tick do not run
            s->failed = true;
            s->msg = msg;
            it.failed = true;
            status[i] = W2L_EINVAL;
            pend->erase(std::remove_if(pend->begin(), pend->end(), [s](const GroupPend& q) { return q.s == s; }), pend->end());
        };
        std::string msg;
        if (flags[s->slot]) { fail_session(kMelNanMsg); continue; }
        // a detected session fails at the tick whose rows first read a frame without a usable box
        if (s->detect && group_det_failed(s, s->sched.need(it.last), &msg)) { fail_session(msg); continue; }
        StreamSched::At a;
        if (p.fin) a = it.last;
        else CKR(s->sched.at(s->mel.L, false, &a));
        if (s->detect) {   // its rows need the rects read back above
            bool bad = false;
            for (long long r = it.first + it.queued; r < a.n_fixed && !bad; ++r)
                if (s->sched.row(r, a, &it.rows[(size_t)(r - it.first) * W2L_STREAM_ROW]) != W2L_OK) bad = true;
            if (bad) { fail_session(g_err); continue; }
        }
        const size_t frame_bytes = (size_t)s->sched.d.H * s->sched.d.W * 3;
        for (long long r = it.first + it.queued; r < a.n_fixed; ++r, ++it.queued)
            pend->push_back(GroupPend{s, &it.rows[(size_t)(r - it.first) * W2L_STREAM_ROW],
                                      it.out + (size_t)(r - it.first) * frame_bytes});
    }
    size_t k = 0;
    const int B = g->steps.max_batch;
    for (; pend->size() - k >= (size_t)B; k += B) CKR(group_step(g, pend->data() + k, B, st));
    pend->erase(pend->begin(), pend->begin() + k);
    return W2L_OK;
}

static int group_tick(w2l_stream_group* g, int n, const int32_t* ids, const float* const* pcm, const int64_t* n_samples,
                      const int32_t* finish, uint8_t* const* out, const int64_t* cap, int64_t* first_index,
                      int64_t* n_out, int32_t* status, cudaStream_t st) {
    if (!g || n < 0) return fail(W2L_EINVAL, "bad argument");
    if (n > 0 && (!ids || !n_samples || !out || !cap || !first_index || !n_out || !status)) return fail(W2L_EINVAL, "null argument");
    // ---- every argument, index, pointer and row is checked before anything is launched ----
    std::vector<GroupItem> items((size_t)n);
    DeviceGuard dg(g->ctx->device);
    for (int i = 0; i < n; ++i) {
        auto f = g->sessions.find(ids[i]);
        if (f == g->sessions.end()) return fail(W2L_EINVAL, "session %d is not open in this group", ids[i]);
        for (int j = 0; j < i; ++j)
            if (ids[j] == ids[i]) return fail(W2L_EINVAL, "session %d is named twice in one tick", ids[i]);
        GroupSession* s = f->second.get();
        GroupItem& it = items[i];
        status[i] = W2L_OK;
        first_index[i] = s->emitted;
        n_out[i] = 0;
        if (s->failed) { status[i] = W2L_EINVAL; continue; }
        if (s->mel.finished) return fail(W2L_ESTATE, "session %d is finished", ids[i]);
        const long long ns = n_samples[i];
        const float* p = pcm ? pcm[i] : nullptr;
        if (ns < 0 || (ns > 0 && !p)) return fail(W2L_EINVAL, "session %d: bad audio piece (%lld samples)", ids[i], ns);
        if (ns > 0) {
            int kind;
            CKR(pcm_kind(g->ctx, p, &kind));
            it.device = kind == PCM_DEVICE;
        }
        it.pcm = p; it.n = ns;
        it.finish = finish && finish[i] != 0;
        CKR(s->sched.at(s->mel.samples_after(ns, it.finish), it.finish, &it.last));
        const long long need = std::max(0LL, it.last.n_fixed - s->emitted);
        if (need > cap[i] || (need > 0 && !out[i]))
            return fail(W2L_EINVAL, "session %d: output holds %lld frames, this tick emits %lld", ids[i], (long long)cap[i], need);
        it.out = out[i];
        it.first = s->emitted;
        it.rows.resize((size_t)need * W2L_STREAM_ROW);
        if (!s->detect)   // a detected session's rows are made once its rects are read back (group_round)
            for (long long r = 0; r < need; ++r) CKR(s->sched.row(it.first + r, it.last, &it.rows[(size_t)r * W2L_STREAM_ROW]));
        it.s = s;
    }
    // ---- detection of the frames this tick's rows read that no launch covers yet ----
    std::vector<std::pair<GroupSession*, long long>> upto;
    for (const GroupItem& it : items)
        if (it.s && it.s->detect) upto.push_back({it.s, it.s->sched.need(it.last)});
    CKR(group_detect(g, upto));
    // ---- rounds (one unless a piece exceeds what a session's rings take), then the partial last step ----
    std::vector<GroupPend> pend;
    bool more = true;
    while (more) CKR(group_round(g, items, &pend, status, st, &more));
    if (!pend.empty()) CKR(group_step(g, pend.data(), (int)pend.size(), st));
    for (int i = 0; i < n; ++i)
        if (items[i].s && !items[i].failed) n_out[i] = items[i].s->emitted - items[i].first;
    // ---- prefetch: the frames 200 ms more audio would need, read back by a later tick's wait ----
    upto.clear();
    for (const GroupItem& it : items) {
        GroupSession* s = it.s;
        if (!s || !s->detect || s->failed || s->mel.finished) continue;
        StreamSched::At a;
        CKR(s->sched.at(s->mel.L + kDetAheadSamples, false, &a));
        upto.push_back({s, s->sched.need(a)});
    }
    return group_detect(g, upto);
}

// ------------------------------------------------------------------------------------------------
// C-ABI (declared in include/w2l.h)
// ------------------------------------------------------------------------------------------------
int w2l_stream_group_buckets(int max_batch, int64_t n_rows, int32_t* sizes, int64_t cap) {
    if (max_batch < 1 || n_rows < 0 || cap < 0 || (cap > 0 && !sizes)) return fail(W2L_EINVAL, "bad argument");
    int64_t k = 0;
    for (long long left = n_rows; left > 0; ++k) {
        const int b = left >= max_batch ? max_batch : group_bucket(max_batch, left);
        if (k < cap) sizes[k] = b;
        left -= std::min<long long>(left, b);
    }
    return (int)k;
}

int w2l_stream_group_create(w2l_ctx* ctx, int max_batch, int audio_ring_log2, w2l_stream_group** out) {
    if (!ctx || !out) return fail(W2L_EINVAL, "null argument");
    *out = nullptr;
    if (max_batch < 1 || max_batch > 4096) return fail(W2L_EINVAL, "max_batch %d: need 1 .. 4096", max_batch);
    if (audio_ring_log2 != 0 && (audio_ring_log2 < 11 || audio_ring_log2 > 24))
        return fail(W2L_EINVAL, "audio ring of 2^%d samples: need 2^11 .. 2^24", audio_ring_log2);
    DeviceGuard dg(ctx->device);
    std::unique_ptr<w2l_stream_group> g(new w2l_stream_group());
    g->ctx = ctx;
    g->ring_log2 = audio_ring_log2 ? audio_ring_log2 : 16;
    CKR(g->s_mel.create());
    CKR(g->ev_mel.create());
    CKR(g->ev_caller.create());
    CKR(g->s_det.create());
    CKR(g->ev_det.create());
    CKR(g->ev_open.create());
    CKR(g->steps.init(ctx, max_batch));
    CKR(group_nan_capacity(g.get(), 1));
    *out = g.release();
    return W2L_OK;
}

static int group_open(w2l_stream_group* g, const uint8_t* frames_dev, const w2l_stream_desc* d, const int32_t* rects_host,
                      bool detect, int32_t* session_id) {
    if (!g || !frames_dev || !d || !session_id) return fail(W2L_EINVAL, "null argument");
    w2l_ctx* ctx = g->ctx;
    DeviceGuard dg(ctx->device);
    std::unique_ptr<GroupSession> s(new GroupSession());
    CKR(s->sched.init(d, rects_host, detect));
    CKR(check_stream_frames(ctx, frames_dev, *d));
    if (detect) {
        if (!ctx->nets[W2L_NET_S3FD].loaded) return fail(W2L_ESTATE, "S3FD weights not loaded");
        if (d->H < 32 || d->W < 32) return fail(W2L_EINVAL, "S3FD needs frames of at least 32 x 32, got %dx%d", d->H, d->W);
        s->detect = true;
        s->det_status.assign((size_t)d->F, (int8_t)-1);
    }
    s->frames = frames_dev;
    // as the session's: the frames of every row not yet run (< max_batch + 4 chunks) beside a whole audio ring of new ones
    const long long ra = 1LL << g->ring_log2;
    CKR(s->mel.init(ctx, g->ring_log2, (long long)std::ceil((g->steps.max_batch + 4) * s->sched.mult) + 64 + ra / MEL_HOP + 16));
    int slot;
    if (!g->free_slots.empty()) { slot = g->free_slots.back(); g->free_slots.pop_back(); }
    else { CKR(group_nan_capacity(g, g->n_slots + 1)); slot = g->n_slots++; }
    CK(cudaMemsetAsync(g->nan.p + slot, 0, 4, g->s_mel));   // a reused slot may hold the flag of a closed session
    s->slot = slot;
    s->id = g->next_id++;
    *session_id = s->id;
    if (detect) {
        // The frames the first 400 ms of audio need, launched without waiting.  They were written by work the caller
        // queued before this call on the legacy default stream (or completed).
        StreamSched::At a;
        int r = s->sched.at(kDetOpenSamples, false, &a);
        if (r == W2L_OK && cudaEventRecord(g->ev_open, cudaStreamLegacy) == cudaSuccess &&
            cudaStreamWaitEvent(g->s_det, g->ev_open, 0) == cudaSuccess)
            r = group_detect(g, {{s.get(), s->sched.need(a)}});
        else if (r == W2L_OK)
            r = fail(W2L_ECUDA, "%s", cudaGetErrorString(cudaGetLastError()));
        if (r != W2L_OK) { g->free_slots.push_back(slot); return r; }   // launches already queued find no session
        g->det_sizes[{d->H, d->W}]++;
    }
    g->sessions[s->id] = std::move(s);
    return W2L_OK;
}

int w2l_stream_group_open(w2l_stream_group* g, const uint8_t* frames_dev, const w2l_stream_desc* d,
                          const int32_t* rects_host, int32_t* session_id) {
    return group_open(g, frames_dev, d, rects_host, false, session_id);
}

int w2l_stream_group_open_detect(w2l_stream_group* g, const uint8_t* frames_dev, const w2l_stream_desc* d,
                                 int32_t* session_id) {
    return group_open(g, frames_dev, d, nullptr, true, session_id);
}

int w2l_stream_group_set_input_rate(w2l_stream_group* g, int32_t session_id, int sr) {
    if (!g) return fail(W2L_EINVAL, "null argument");
    auto f = g->sessions.find(session_id);
    if (f == g->sessions.end()) return fail(W2L_EINVAL, "session %d is not open in this group", session_id);
    DeviceGuard dg(g->ctx->device);
    return f->second->mel.set_rate(sr);
}

int w2l_stream_group_close(w2l_stream_group* g, int32_t session_id) {
    if (!g) return fail(W2L_EINVAL, "null argument");
    auto f = g->sessions.find(session_id);
    if (f == g->sessions.end()) return fail(W2L_EINVAL, "session %d is not open in this group", session_id);
    DeviceGuard dg(g->ctx->device);
    CK(cudaDeviceSynchronize());   // queued steps may still read the session's rings
    g->free_slots.push_back(f->second->slot);
    if (f->second->detect) {
        const std::pair<int, int> hw(f->second->sched.d.H, f->second->sched.d.W);
        if (--g->det_sizes[hw] == 0) {   // the last detecting session of its size: unpin that size's plans
            g->det_sizes.erase(hw);
            group_det_release(g, hw.first, hw.second);
        }
    }
    g->sessions.erase(f);
    group_det_resolve(g);          // every launch is complete: its buffers are free again
    return W2L_OK;
}

int w2l_stream_group_pending(const w2l_stream_group* g, int n, const int32_t* ids, const int64_t* n_samples,
                             const int32_t* finish, int64_t* n_out) {
    if (!g || n < 0 || (n > 0 && (!ids || !n_samples || !n_out))) return fail(W2L_EINVAL, "bad argument");
    for (int i = 0; i < n; ++i) {
        auto f = g->sessions.find(ids[i]);
        if (f == g->sessions.end()) return fail(W2L_EINVAL, "session %d is not open in this group", ids[i]);
        const GroupSession* s = f->second.get();
        n_out[i] = 0;
        if (s->failed || s->mel.finished) continue;
        if (n_samples[i] < 0) return fail(W2L_EINVAL, "session %d: bad audio piece (%lld samples)", ids[i], (long long)n_samples[i]);
        StreamSched::At a;
        CKR(s->sched.at(s->mel.samples_after(n_samples[i], finish && finish[i] != 0), finish && finish[i] != 0, &a));
        n_out[i] = std::max(0LL, a.n_fixed - s->emitted);
    }
    return W2L_OK;
}

int w2l_stream_group_tick(w2l_stream_group* g, int n, const int32_t* ids, const float* const* pcm, const int64_t* n_samples,
                          const int32_t* finish, uint8_t* const* out_dev, const int64_t* cap, int64_t* first_index,
                          int64_t* n_out, int32_t* status, void* stream) {
    return group_tick(g, n, ids, pcm, n_samples, finish, out_dev, cap, first_index, n_out, status, (cudaStream_t)stream);
}

const char* w2l_stream_group_error(const w2l_stream_group* g, int32_t session_id) {
    if (!g) return "";
    auto f = g->sessions.find(session_id);
    return f != g->sessions.end() && f->second->failed ? f->second->msg.c_str() : "";
}

int w2l_stream_group_counters(const w2l_stream_group* g, int64_t* calls, int64_t* host_waits, int64_t* steps) {
    if (!g) return fail(W2L_EINVAL, "null argument");
    if (calls) *calls = g->steps.calls;
    if (host_waits) *host_waits = g->steps.waits;
    if (steps) *steps = g->steps.count;
    return W2L_OK;
}

int w2l_stream_group_destroy(w2l_stream_group* g) {
    if (!g) return W2L_OK;
    DeviceGuard dg(g->ctx->device);
    cudaDeviceSynchronize();   // queued steps may still read the group's buffers
    for (auto& b : g->buckets) g->steps.release(b.get());
    for (const DetPlan& p : g->det_plans)
        if (p.plan && p.epoch == g->ctx->plan_epoch[W2L_NET_S3FD]) p.plan->pins--;
    delete g;
    return W2L_OK;
}
