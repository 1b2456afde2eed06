// s3fd_detect.cuh — the S3FD detector around the network, on the device (face_detection/detection/sfd: detect.py:58-94,
// bbox.py:44-64, sfd_detector.py:40-46).
//   s3fd_ingest_u8_kernel:  uint8 NHWC frames (optionally channel-reversed) minus (104, 117, 123) -> conv1_1's input layout.
//   s3fd_count_kernel / s3fd_select_kernel:  softmax of the class maps, p > 0.5, prior decode, a per-image compaction in
//                           location order (scale, row, column) through per-chunk counts: no atomics, deterministic.
//   s3fd_nms_kernel:        one CTA per image: bitonic sort by (score, location) descending, greedy NMS at IoU 0.3 until
//                           max_det boxes are kept.  Shared memory up to kNmsSmemCap candidates, global memory above.
// Why only p > 0.5 and what the tie / NaN rules are: DESIGN.md §3.6.  Every float op that the reference rounds on its own
// is written with an explicit-rounding intrinsic so that nvcc cannot contract it into an FMA.
#pragma once

#include <stdint.h>

namespace w2l {

// ---- (a) ingest --------------------------------------------------------------------------------------------------------
// detect.py:60-65 on uint8: x - (104, 117, 123) is an integer in [-123, 151], exact in fp16 and bf16, so the activation is
// bit-identical to the fp32 path's.  reverse: channel c reads source channel 2 - c (api.py:64 reverses the channels).
struct S3fdIngestParams {
    const unsigned char* src;  // (N, H, W, 3)
    uint16_t* dst;             // [N][H][Wp][Cpix], image column x at column x + x_off (zero borders pre-set)
    int N, H, W, Cpad, Wp, x_off, Cpix, lo_off;
    int reverse;
    const unsigned char* const* srcs;   // kGather: image n is the (H, W, 3) frame srcs[n]; src unused
};

// kGather: each image through the frame-pointer table, so one launch takes frames of several videos of one size
template <bool kBF16, bool kGather = false>
__global__ void s3fd_ingest_u8_kernel(const S3fdIngestParams p) {
    const long long total = (long long)p.N * p.H * p.W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % p.W);
        const int y = (int)((i / p.W) % p.H);
        const int n = (int)(i / ((long long)p.W * p.H));
        const unsigned char* s;
        if constexpr (kGather) s = p.srcs[n] + (i - (long long)n * p.W * p.H) * 3;
        else s = p.src + i * 3;
        const int m[3] = {104, 117, 123};
        uint16_t h[4];
#pragma unroll
        for (int c = 0; c < 3; ++c) h[c] = to16<kBF16>((float)((int)s[p.reverse ? 2 - c : c] - m[c]));
        uint16_t* d = p.dst + ((((long long)n * p.H + y) * p.Wp) + x + p.x_off) * p.Cpix;
        *reinterpret_cast<uint4*>(d) = make_uint4(h[0] | ((uint32_t)h[1] << 16), h[2], 0u, 0u);
        for (int c0 = 8; c0 < p.Cpad; c0 += 8) *reinterpret_cast<uint4*>(d + c0) = make_uint4(0u, 0u, 0u, 0u);
        if (p.lo_off > 0)  // split-operand mode: the values are exact, the lo plane is zero
            for (int c0 = 0; c0 < p.Cpad; c0 += 8) *reinterpret_cast<uint4*>(d + p.lo_off + c0) = make_uint4(0u, 0u, 0u, 0u);
    }
}

// ---- (b) select + decode -----------------------------------------------------------------------------------------------
constexpr int kSelChunk = 512;      // locations per CTA of the select kernels (= threads)
constexpr int kNmsThreads = 512;
constexpr int kNmsSmemCap = 4096;   // candidates per image sorted and suppressed in shared memory
constexpr size_t kNmsSmemBytes = (size_t)kNmsSmemCap * (8 + 16 + 1);

struct S3fdScale {
    const float* cls;  // head output, fp32 NHWC with a 16-channel pitch (4 used at scale 0, 2 elsewhere)
    const float* reg;  // fp32 NHWC, 16-channel pitch, 4 used
    int h, w, first;   // map size, location index of its (0, 0)
};

struct S3fdDetParams {
    S3fdScale sc[6];
    int B, L, Lpad, nchunk;
    int* chunk_count;  // [B][nchunk]
    int* ncand;        // [B] candidates (p > 0.5) per image
    float4* cbox;      // [B][L] compacted boxes (x1, y1, x2, y2), location order
    int* cloc;         // [B][L] their location indices
    uint64_t* keys;    // [B][Lpad] (score bits << 32 | slot); sorted descending by s3fd_nms_kernel
    uint8_t* sup;      // [B][L] suppression flags of the global-memory path
    int* path;         // [B] 0: shared-memory NMS, 1: global-memory NMS
    int max_det;
    float* dets;       // [B][max_det][5]
    int* counts;       // [B]
};

// softmax(cls)[1] and the decoded box at location l of image b (detect.py:70-91, bbox.py:124-128 in float32, op by op)
__device__ __forceinline__ bool s3fd_location(const S3fdDetParams& p, int b, int l, float* score, float4* box) {
    int s = 0;
#pragma unroll
    for (int k = 1; k < 6; ++k) s += l >= p.sc[k].first ? 1 : 0;
    const S3fdScale& sc = p.sc[s];
    const int r = l - sc.first, y = r / sc.w, x = r - y * sc.w;
    const long long pix = ((long long)b * sc.h + y) * sc.w + x;
    const float* c = sc.cls + pix * 16;
    const float x0 = s == 0 ? fmaxf(fmaxf(c[0], c[1]), c[2]) : c[0];   // max-out background, net_s3fd.py:123-126
    const float x1 = s == 0 ? c[3] : c[1];
    const float mx = fmaxf(x0, x1);
    const float e0 = expf(__fsub_rn(x0, mx)), e1 = expf(__fsub_rn(x1, mx));
    const float pr = __fdiv_rn(e1, __fadd_rn(e0, e1));
    *score = pr;
    if (!(pr > 0.5f)) return false;
    const float* g = sc.reg + pix * 16;
    const int stride = 4 << s;
    const float A = (float)(4 * stride);
    const float axc = 0.5f * stride + (float)(x * stride), ayc = 0.5f * stride + (float)(y * stride);   // exact
    const float cx = __fadd_rn(axc, __fmul_rn(__fmul_rn(g[0], 0.1f), A));
    const float cy = __fadd_rn(ayc, __fmul_rn(__fmul_rn(g[1], 0.1f), A));
    const float w = __fmul_rn(A, expf(__fmul_rn(g[2], 0.2f)));
    const float h = __fmul_rn(A, expf(__fmul_rn(g[3], 0.2f)));
    const float bx1 = __fsub_rn(cx, __fmul_rn(w, 0.5f)), by1 = __fsub_rn(cy, __fmul_rn(h, 0.5f));
    *box = make_float4(bx1, by1, __fadd_rn(w, bx1), __fadd_rn(h, by1));
    return true;
}

// pass 1: number of candidates in each chunk of kSelChunk locations
__global__ void __launch_bounds__(kSelChunk) s3fd_count_kernel(const S3fdDetParams p) {
    const int b = blockIdx.y, l = blockIdx.x * kSelChunk + threadIdx.x;
    float sc = 0.0f;
    float4 box;
    const bool hit = l < p.L && s3fd_location(p, b, l, &sc, &box);
    const int n = __syncthreads_count(hit);
    if (threadIdx.x == 0) p.chunk_count[b * p.nchunk + blockIdx.x] = n;
}

// pass 2: chunk offset = sum of the preceding chunks' counts, rank inside the chunk by ballot: candidates land in
// location order
__global__ void __launch_bounds__(kSelChunk) s3fd_select_kernel(const S3fdDetParams p) {
    __shared__ int warp_n[kSelChunk / 32];
    __shared__ int s_base;
    const int b = blockIdx.y, l = blockIdx.x * kSelChunk + threadIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (wid == 0) {
        int s = 0;
        for (int c = lane; c < (int)blockIdx.x; c += 32) s += p.chunk_count[b * p.nchunk + c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) s_base = s;
    }
    float sc = 0.0f;
    float4 box;
    const bool hit = l < p.L && s3fd_location(p, b, l, &sc, &box);
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_n[wid] = __popc(m);
    __syncthreads();
    int rank = s_base + __popc(m & ((1u << lane) - 1u));
    for (int k = 0; k < wid; ++k) rank += warp_n[k];
    if (hit) {
        const size_t o = (size_t)b * p.L + rank;
        p.cbox[o] = box;
        p.cloc[o] = l;
        p.keys[(size_t)b * p.Lpad + rank] = ((uint64_t)__float_as_uint(sc) << 32) | (uint32_t)rank;
    }
    if (blockIdx.x == p.nchunk - 1 && threadIdx.x == kSelChunk - 1) {
        int tot = s_base;
        for (int k = 0; k < kSelChunk / 32; ++k) tot += warp_n[k];
        p.ncand[b] = tot;
    }
}

// ---- (c) sort + greedy NMS ---------------------------------------------------------------------------------------------
// bbox.py:44-64 in float32, every op rounded: area = ((x2 - x1) + 1) * ((y2 - y1) + 1), w = max(0, (xx2 - xx1) + 1),
// ovr = inter / ((area_i + area_j) - inter).  Returns whether j survives: ovr <= 0.3, so a NaN overlap suppresses, as
// np.where(ovr <= thresh) does.
__device__ __forceinline__ float s3fd_area(const float4 a) {
    return __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.0f), __fadd_rn(__fsub_rn(a.w, a.y), 1.0f));
}
__device__ __forceinline__ bool s3fd_survives(const float4 a, float area_a, const float4 c) {
    const float xx1 = fmaxf(a.x, c.x), yy1 = fmaxf(a.y, c.y), xx2 = fminf(a.z, c.z), yy2 = fminf(a.w, c.w);
    const float w = fmaxf(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
    const float h = fmaxf(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
    const float inter = __fmul_rn(w, h);
    const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, s3fd_area(c)), inter));
    return ovr <= 0.3f;
}

__global__ void __launch_bounds__(kNmsThreads) s3fd_nms_kernel(const S3fdDetParams p) {
    extern __shared__ __align__(16) unsigned char nms_smem[];
    __shared__ int red[kNmsThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = p.ncand[b];
    const bool fast = n <= kNmsSmemCap;
    uint64_t* gkeys = p.keys + (size_t)b * p.Lpad;
    uint64_t* keys = fast ? reinterpret_cast<uint64_t*>(nms_smem) : gkeys;
    float4* sbox = reinterpret_cast<float4*>(nms_smem + (size_t)kNmsSmemCap * 8);
    uint8_t* sup = fast ? nms_smem + (size_t)kNmsSmemCap * 24 : p.sup + (size_t)b * p.L;
    const float4* cbox = p.cbox + (size_t)b * p.L;
    int P = 1;
    while (P < n) P <<= 1;
    for (int i = tid; i < P; i += kNmsThreads) {
        if (i >= n) keys[i] = 0ull;
        else if (fast) keys[i] = gkeys[i];
    }
    __syncthreads();
    // bitonic sort, descending: score first, then the slot, which is in location order (ties: larger index first)
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += kNmsThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t a = keys[i], c = keys[ixj];
                    if ((i & k) == 0 ? a < c : a > c) { keys[i] = c; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += kNmsThreads) {
        sup[i] = 0;
        if (fast) {
            gkeys[i] = keys[i];   // the sorted list stays readable (w2l_debug_s3fd_candidates)
            sbox[i] = cbox[(uint32_t)keys[i]];
        }
    }
    __syncthreads();
    float* dets = p.dets + (size_t)b * p.max_det * 5;
    int kept = 0, i = 0;
    while (i < n) {
        const float4 bi = fast ? sbox[i] : cbox[(uint32_t)keys[i]];
        if (tid == 0) {
            float* d = dets + (size_t)kept * 5;
            d[0] = bi.x; d[1] = bi.y; d[2] = bi.z; d[3] = bi.w; d[4] = __uint_as_float((uint32_t)(keys[i] >> 32));
        }
        if (++kept == p.max_det) break;
        // suppress against box i; the next kept box is the first survivor after it
        const float ai = s3fd_area(bi);
        int next = n;
        for (int j = i + 1 + tid; j < n; j += kNmsThreads) {
            if (sup[j]) continue;
            const float4 bj = fast ? sbox[j] : cbox[(uint32_t)keys[j]];
            if (s3fd_survives(bi, ai, bj)) next = min(next, j);
            else sup[j] = 1;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) next = min(next, __shfl_xor_sync(0xffffffffu, next, o));
        if ((tid & 31) == 0) red[tid >> 5] = next;
        __syncthreads();
        next = n;
#pragma unroll
        for (int w = 0; w < kNmsThreads / 32; ++w) next = min(next, red[w]);
        __syncthreads();   // red is rewritten by the next round
        i = next;
    }
    for (long long r = (long long)kept * 5 + tid; r < (long long)p.max_det * 5; r += kNmsThreads) dets[r] = 0.0f;
    if (tid == 0) {
        p.counts[b] = kept;
        p.path[b] = fast ? 0 : 1;
    }
}

// ---- (d) rect export -----------------------------------------------------------------------------------------------------
// get_detections_for_batch_u8's result for image b < n (api.py: the first box, np.clip(d[:4], 0, None), int() of each):
// out[b] = (x1, y1, x2, y2, status).  Finiteness is tested before the clip, because fmaxf(NaN, 0) is 0 while np.clip
// keeps the NaN and int() then raises.  Coordinates are clamped to 2^30 before the truncating conversion, so that the
// padding arithmetic after it cannot overflow int32.
constexpr int kRectFace = 0, kRectNone = 1, kRectNonFinite = 2;

__global__ void s3fd_rect_export_kernel(const float* dets, const int* counts, int n, int max_det, int32_t* out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    int32_t* o = out + (size_t)b * 5;
    const float* d = dets + (size_t)b * max_det * 5;
    int status = counts[b] > 0 ? kRectFace : kRectNone;
    for (int k = 0; k < 4; ++k) {
        const float v = status == kRectNone ? 0.0f : d[k];
        if (!isfinite(v)) status = kRectNonFinite;
        o[k] = isfinite(v) ? (int32_t)fminf(fmaxf(v, 0.0f), 1073741824.0f) : 0;
    }
    o[4] = status;
}

}  // namespace w2l
