// face_crops.cuh — preprocess.py's per-frame step on the device (preprocess.py:38-67, :82-89 around
// face_detection/api.py:64-79): the detector's top box -> get_detections_for_batch's clip and int() -> the crop
// fb[j][y1:y2, x1:x2] -> cv2.resize(crop, (96, 96)) into a cache slot, with the script's abort rules, no host round trip.
//   face_crops_rows_kernel:    one CTA per call: each frame's status and slice bounds, the call's abort point, the frame
//                              that caused it, slots by a block scan over kept frames (frame order), the carried state.
//   face_crops_resize_kernel:  (96·96 / 256, frames) CTAs, one thread per destination pixel of a kept frame, through
//                              resize.cuh's cv2.resize-exact resize_axis / resize_pixel.
// The rules (DESIGN.md §3.12, restated in NumPy by oracle/preprocess_oracle.py):
//   - no detection: no file (status 1);
//   - np.clip(d, 0, None) then int(): -inf -> 0, finite values truncate toward zero, NaN / +inf raise (status 2), before
//     any file of the detector batch is written, so the video ends at the start of that batch;
//   - NumPy slicing clamps the ends to H / W; an empty slice makes cv2.imwrite raise (status 3): the video ends at that
//     frame;  the earliest abort point wins, every later frame is lost (status 4), the files before it stay.
#pragma once

#include <stdint.h>

namespace w2l {

constexpr int kFcThreads = 1024;
constexpr int kFcKept = 0, kFcNoFace = 1, kFcNonFinite = 2, kFcEmpty = 3, kFcAborted = 4;
constexpr int kFcRow = 6;   // status, slot, y1, y2, x1, x2
constexpr int kFcNoAbort = 0x7fffffff;

struct FaceCropParams {
    const uint8_t* frames;   // (B, H, W, 3)
    const float* dets;       // (B, max_det, 5): x1 y1 x2 y2 score, only row 0 is read
    const int32_t* counts;   // (B)
    int32_t* state;          // [0] next free slot, [1] abort frame (kFcNoAbort: none yet; not read when frame0 = 0)
    int32_t* rows;           // (B, 6)
    uint8_t* crops;          // (cap, 96, 96, 3)
    long long cap;
    int B, H, W, max_det, frame0, batch;
};

// The frame's own status (0..3, before the video's abort is applied), its slice bounds and the abort point it causes.
// Coordinates are clamped to 2^30 before the truncating conversion, so 1e30 cannot overflow int32; the slice ends then
// clamp to H / W as NumPy's do.  A non-finite coordinate leaves 0 in its bound.
__device__ __forceinline__ int face_crop_own(const FaceCropParams& p, int b, int* y1, int* y2, int* x1, int* x2, int* abort_at) {
    const int i = p.frame0 + b;
    int s = p.counts[b] > 0 ? kFcKept : kFcNoFace;
    int c[4] = {0, 0, 0, 0};   // x1, y1, x2, y2
    if (s == kFcKept) {
        const float* d = p.dets + (size_t)b * p.max_det * 5;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float v = d[k];
            if (isnan(v) || v == INFINITY) s = kFcNonFinite;
            else c[k] = (int)fminf(fmaxf(v, 0.0f), 1073741824.0f);
        }
    }
    *x1 = min(c[0], p.W); *y1 = min(c[1], p.H); *x2 = min(c[2], p.W); *y2 = min(c[3], p.H);
    if (s == kFcKept && (*y1 >= *y2 || *x1 >= *x2)) s = kFcEmpty;
    *abort_at = s == kFcNonFinite ? i - i % p.batch : s == kFcEmpty ? i : kFcNoAbort;
    return s;
}

__global__ void __launch_bounds__(kFcThreads) face_crops_rows_kernel(const FaceCropParams p) {
    __shared__ int s_abort, s_cause;
    __shared__ int warp_n[kFcThreads / 32];
    __shared__ int s_carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // a call at frame 0 starts its video: no frame precedes it, so the incoming abort frame is not read (a zeroed state works)
    const int slot0 = p.state[0], abort_prev = p.frame0 == 0 ? kFcNoAbort : p.state[1];
    if (tid == 0) { s_abort = abort_prev; s_cause = kFcNoAbort; s_carry = 0; }
    __syncthreads();
    int y1, y2, x1, x2, a;
    // pass 1: the earliest abort point of the video so far
    for (int b = tid; b < p.B; b += kFcThreads) {
        face_crop_own(p, b, &y1, &y2, &x1, &x2, &a);
        if (a < kFcNoAbort) atomicMin(&s_abort, a);
    }
    __syncthreads();
    const int A = s_abort;
    // pass 2: the frame that raised.  If A is a batch start with a non-finite box in that batch, the first such box raised
    // (get_detections_for_batch converts the boxes in order); otherwise A is the empty crop's own frame.
    const bool here = A != abort_prev && A >= p.frame0;
    if (here) {
        for (int b = tid; b < p.B; b += kFcThreads) {
            const int i = p.frame0 + b;
            if (face_crop_own(p, b, &y1, &y2, &x1, &x2, &a) == kFcNonFinite && i / p.batch == A / p.batch) atomicMin(&s_cause, i);
        }
        __syncthreads();
    }
    const int cause = !here ? -1 : s_cause < kFcNoAbort ? s_cause : A;
    // pass 3: final statuses, slots by a block scan over kept frames, in frame order
    for (int b0 = 0; b0 < p.B; b0 += kFcThreads) {
        const int b = b0 + tid;
        int s = kFcAborted;
        if (b < p.B) {
            const int i = p.frame0 + b;
            const int own = face_crop_own(p, b, &y1, &y2, &x1, &x2, &a);
            if (i < A || i == cause) s = own;
        }
        const bool kept = b < p.B && s == kFcKept;
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (lane == 0) warp_n[wid] = __popc(m);
        __syncthreads();
        int rank = s_carry + __popc(m & ((1u << lane) - 1u));
        for (int k = 0; k < wid; ++k) rank += warp_n[k];
        if (b < p.B) {
            int32_t* r = p.rows + (size_t)b * kFcRow;
            r[0] = s; r[1] = kept ? slot0 + rank : -1; r[2] = y1; r[3] = y2; r[4] = x1; r[5] = x2;
        }
        __syncthreads();   // every thread has read s_carry and warp_n
        if (tid == 0) {
            int n = 0;
            for (int k = 0; k < kFcThreads / 32; ++k) n += warp_n[k];
            s_carry += n;
        }
        __syncthreads();
    }
    if (tid == 0) {
        p.state[0] = slot0 + s_carry;   // > cap: the crops past cap were not written, the caller reports the overflow
        p.state[1] = A;
    }
}

constexpr int kFcPix = 96 * 96;
constexpr int kFcResizeThreads = 256;

__global__ void __launch_bounds__(kFcResizeThreads) face_crops_resize_kernel(const FaceCropParams p) {
    const int px = blockIdx.x * kFcResizeThreads + threadIdx.x;
    if (px >= kFcPix) return;
    const int ox = px % 96, oy = px / 96;
    for (int b = blockIdx.y; b < p.B; b += gridDim.y) {
        const int32_t* r = p.rows + (size_t)b * kFcRow;
        if (r[0] != kFcKept || (long long)r[1] >= p.cap) continue;
        const int y1 = r[2], y2 = r[3], x1 = r[4], x2 = r[5];
        const ResizeAxis ax = resize_axis(ox, 96, x2 - x1, true);
        const ResizeAxis ay = resize_axis(oy, 96, y2 - y1, false);
        const uint8_t* src = p.frames + (((long long)b * p.H + y1) * p.W + x1) * 3;
        uint8_t o[3];
        resize_pixel(src, (long long)p.W * 3, ax, ay, o);
        uint8_t* d = p.crops + ((long long)r[1] * kFcPix + px) * 3;
        d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
    }
}

}  // namespace w2l
