// mel.cuh — fused audio.melspectrogram for sm_90a.
//
// One kernel does what /root/reference/audio.py:45-51 does in six NumPy/librosa passes:
//   pre-emphasis (audio.py:20-23) -> reflect-padded framing + periodic Hann window + 800-point real FFT
//   (audio.py:57-61 -> librosa.stft) -> |.| -> 80-band Slaney mel filterbank (audio.py:92-101)
//   -> 20*log10(max(1e-5, .)) - 20 (audio.py:103-105, :47) -> symmetric normalise + clip (audio.py:110-114).
//
// Numerics follow the reference's dtypes: pre-emphasis, window and FFT in float64 (scipy.lfilter and
// the FFT of a float64 frame), spectrum rounded to complex64, magnitude / mel / log / clip in float32.
// float64 matters: with a loud tone in the frame, a float32 FFT's noise floor (-144 dB re peak) reaches
// the mel bands near the 1e-5 clipping floor and breaks the 1e-4 tolerance; the H100 has the FP64 rate.
//
// Work split: a block owns MEL_FPB consecutive frames (so the (80, F) row-major output is written in runs of
// MEL_FPB floats). The real 800-point FFT is the 400-point complex FFT of the even/odd-packed frame followed by
// the real-FFT split X[k] = E[k] + W800^k O[k] (800 = 2^5 5^2 is not a power of two, and zero-padding would
// change the result). 400 = 25 x 16 is split Cooley-Tukey style across threads:
//   step 1  (25 threads per frame, thread = n1): the 16 packed samples z[n1 + 25 n2] are gathered straight from
//           HBM/L1 (coalesced across n1), pre-emphasised, windowed (periodic Hann from the cos table) and transformed
//           by a 16-point FFT (4 x 4) in registers; the result is multiplied by W400^(n1 k2) and written to shared
//           memory, the one exchange between the two steps;
//   step 3  (16 threads per frame, thread = k2): 25-point FFT (5 x 5) in registers over n1, then the real-FFT
//           split, whose partner Z[400 - k] lives in thread 16 - k2 of the same 16-lane group: warp shuffles,
//           no second exchange; |X| goes to shared memory as fp32.
// The twiddles inside the small FFTs are compile-time constants (mel_consts.h). The FFT lives in registers because
// a shared-memory round trip of the float64 data per radix pass would make the kernel shared-memory bound; with one
// exchange (~18 KB of shared-memory traffic per frame) it is bound by the FP64 pipe instead. The mel product uses
// the filterbank's sparsity (739 non-zeros, <= 27 per band) straight from the magnitudes in shared memory.
#pragma once

#include <stdint.h>

#include "mel_consts.h"

namespace w2l {

constexpr int MEL_FPB = 5;        // frames per block: 125 of 128 threads busy in step 1, 80 in step 3
constexpr int MEL_THREADS = 128;
constexpr int MEL_NFFT = 800;
constexpr int MEL_HOP = 200;
constexpr int MEL_BINS = 401;
constexpr int MEL_BANDS = 80;
constexpr int kMelSmemBytes = 404 * 16 + MEL_FPB * 400 * 16 + MEL_FPB * 404 * 4 + MEL_BANDS * MEL_FPB * 4;

struct MelParams {
    const float* wav;
    long long L;
    float* mel;          // (80, F) row-major
    long long F;
    const double2* tw;   // [0,401): exp(-2 pi i m / 800) (Hann window, W400 twiddles of step 1, real-FFT split)
    const float* bvals;  // packed non-zero filterbank weights
    const int* boff;     // [80] offset into bvals
    const int* bstart;   // [80] first FFT bin of the band
    const int* blen;     // [80] number of bins
};

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }

template <int R>
__device__ __forceinline__ void butterfly(double2* v);

template <>
__device__ __forceinline__ void butterfly<4>(double2* v) {
    const double2 a = cadd(v[0], v[2]), b = csub(v[0], v[2]);
    const double2 c = cadd(v[1], v[3]), d = csub(v[1], v[3]);
    v[0] = cadd(a, c);
    v[2] = csub(a, c);
    v[1] = make_double2(b.x + d.y, b.y - d.x);  // b - i d
    v[3] = make_double2(b.x - d.y, b.y + d.x);  // b + i d
}

template <>
__device__ __forceinline__ void butterfly<5>(double2* v) {
    const double c1 = 0.30901699437494742410229341718282;   // cos(2 pi / 5)
    const double c2 = -0.80901699437494742410229341718282;  // cos(4 pi / 5)
    const double s1 = 0.95105651629515357211643933337938;   // sin(2 pi / 5)
    const double s2 = 0.58778525229247312916870595463907;   // sin(4 pi / 5)
    const double2 a1 = cadd(v[1], v[4]), a2 = cadd(v[2], v[3]);
    const double2 b1 = csub(v[1], v[4]), b2 = csub(v[2], v[3]);
    const double2 t1 = make_double2(v[0].x + c1 * a1.x + c2 * a2.x, v[0].y + c1 * a1.y + c2 * a2.y);
    const double2 t2 = make_double2(v[0].x + c2 * a1.x + c1 * a2.x, v[0].y + c2 * a1.y + c1 * a2.y);
    const double2 u1 = make_double2(s1 * b1.x + s2 * b2.x, s1 * b1.y + s2 * b2.y);
    const double2 u2 = make_double2(s2 * b1.x - s1 * b2.x, s2 * b1.y - s1 * b2.y);
    v[0] = make_double2(v[0].x + a1.x + a2.x, v[0].y + a1.y + a2.y);
    v[1] = make_double2(t1.x + u1.y, t1.y - u1.x);  // t1 - i u1
    v[4] = make_double2(t1.x - u1.y, t1.y + u1.x);  // t1 + i u1
    v[2] = make_double2(t2.x + u2.y, t2.y - u2.x);
    v[3] = make_double2(t2.x - u2.y, t2.y + u2.x);
}

__device__ __forceinline__ double2 shfl_d2(double2 v, int src_lane) {
    return make_double2(__shfl_sync(0xffffffffu, v.x, src_lane, 16), __shfl_sync(0xffffffffu, v.y, src_lane, 16));
}

// The load stage and the store stage are template parameters; everything between them (window, FFT, magnitude, mel
// product, dB, normalise, clip) is shared, so a frame computed by either kernel below has the same bits.
//   Src::len()     the length the reflection at the end uses
//   Src::x(j, d)   sample j + d (absolute index, 0 <= j + d < len())
//   Dst::put(m, t, v)   writes band m of frame t (called with consecutive t across a block's frames)
//   Dst::note(s)   sees every pre-clip mel sum
// The block computes frames [f0 + blockIdx.x * MEL_FPB, ...) below f1.
struct MelWavSrc {      // the whole utterance in device memory (w2l_melspectrogram)
    const MelParams& p;
    __device__ __forceinline__ long long len() const { return p.L; }
    __device__ __forceinline__ double x(long long j, int d) const { return (double)__ldg(p.wav + j + d); }
};
struct MelDenseDst {    // (80, F) row-major
    const MelParams& p;
    __device__ __forceinline__ void note(float) const {}
    __device__ __forceinline__ void put(int m, long long t, float v) const { p.mel[(long long)m * p.F + t] = v; }
};

template <class Src, class Dst>
__device__ __forceinline__ void mel_frames(const MelParams& p, const Src& src, const Dst& dst, long long f0, long long f1) {
    extern __shared__ uint8_t mel_smem[];
    double2* tw = reinterpret_cast<double2*>(mel_smem);                 // [401] exp(-2 pi i m / 800)  (+3 pad)
    double2* ybuf = tw + 404;                                            // [FPB][16][25]
    float* mags = reinterpret_cast<float*>(ybuf + MEL_FPB * 400);        // [FPB][404]
    float* outs = mags + MEL_FPB * 404;                                  // [80][FPB]
    const int tid = threadIdx.x;
    for (int i = tid; i < 401; i += MEL_THREADS) tw[i] = p.tw[i];
    __syncthreads();

    // ---------------- step 1: thread = (frame f, n1) ----------------
    if (tid < MEL_FPB * 25) {
        const int f = tid / 25, n1 = tid % 25;
        const long long t = f0 + (long long)blockIdx.x * MEL_FPB + f;
        if (t < f1) {
            double2 v[16];
            const long long base = t * MEL_HOP - MEL_NFFT / 2 + 2 * n1;
#pragma unroll
            for (int n2 = 0; n2 < 16; ++n2) {
                const long long j0 = base + 50 * n2;
                double y0, y1;
                if (j0 >= 1 && j0 + 1 < src.len()) {   // interior: three consecutive samples
                    const double xm = src.x(j0, -1), x0 = src.x(j0, 0), x1 = src.x(j0, 1);
                    y0 = x0 + (-0.97) * xm;
                    y1 = x1 + (-0.97) * x0;
                } else {                         // np.pad(mode="reflect") of the PRE-EMPHASISED signal
                    double yy[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        long long j = j0 + e;
                        while (j < 0 || j >= src.len()) j = j < 0 ? -j : 2 * (src.len() - 1) - j;
                        const double x0 = src.x(j, 0);
                        yy[e] = (j > 0) ? x0 + (-0.97) * src.x(j, -1) : x0;
                    }
                    y0 = yy[0]; y1 = yy[1];
                }
                // periodic Hann 0.5 - 0.5 cos(2 pi n / 800), n = 2 n1 + 50 n2 (+1), from the table (cos is even around 400)
                const int n = 2 * n1 + 50 * n2;
                const double c0 = tw[n <= 400 ? n : MEL_NFFT - n].x;
                const double c1 = tw[n + 1 <= 400 ? n + 1 : MEL_NFFT - n - 1].x;
                v[n2] = make_double2((0.5 - 0.5 * c0) * y0, (0.5 - 0.5 * c1) * y1);
            }
            // 16-point FFT over n2 = 4 a + b  ->  k2 = c + 4 d
            double2 u[4][4];
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                double2 q[4] = {v[b], v[4 + b], v[8 + b], v[12 + b]};
                butterfly<4>(q);
#pragma unroll
                for (int c = 0; c < 4; ++c) u[b][c] = (b * c == 0) ? q[c] : cmul(q[c], kMelW16[b * c]);
            }
            double2 Y[16];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                double2 q[4] = {u[0][c], u[1][c], u[2][c], u[3][c]};
                butterfly<4>(q);
#pragma unroll
                for (int d = 0; d < 4; ++d) Y[c + 4 * d] = q[d];
            }
            double2* dst = ybuf + f * 400 + n1;
            dst[0] = Y[0];
#pragma unroll
            for (int k2 = 1; k2 < 16; ++k2) {      // W400^(n1 k2) = W800^(2 n1 k2 mod 800), upper half by conjugate symmetry
                const int m = (2 * n1 * k2) % MEL_NFFT;
                double2 w = tw[m <= 400 ? m : MEL_NFFT - m];
                if (m > 400) w.y = -w.y;
                dst[k2 * 25] = cmul(Y[k2], w);
            }
        }
    }
    __syncthreads();

    // ---------------- step 3: thread = (frame f, k2), whole warps so that the shuffles below are convergent ----------------
    if (tid < 96) {
        const int f = tid >> 4, k2 = tid & 15;
        const long long t = f0 + (long long)blockIdx.x * MEL_FPB + f;
        const bool live = f < MEL_FPB && t < f1;
        double2 y[25];
#pragma unroll
        for (int n1 = 0; n1 < 25; ++n1) y[n1] = live ? ybuf[f * 400 + k2 * 25 + n1] : make_double2(0.0, 0.0);
        // 25-point FFT over n1 = 5 a + b  ->  k1 = c + 5 d
        double2 u[5][5];
#pragma unroll
        for (int b = 0; b < 5; ++b) {
            double2 q[5] = {y[b], y[5 + b], y[10 + b], y[15 + b], y[20 + b]};
            butterfly<5>(q);
#pragma unroll
            for (int c = 0; c < 5; ++c) u[b][c] = (b * c == 0) ? q[c] : cmul(q[c], kMelW25[b * c]);
        }
        double2 Z[25];
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            double2 q[5] = {u[0][c], u[1][c], u[2][c], u[3][c], u[4][c]};
            butterfly<5>(q);
#pragma unroll
            for (int d = 0; d < 5; ++d) Z[c + 5 * d] = q[d];
        }
        // real-FFT split: bin k = k2 + 16 k1 pairs with 400 - k = (16 - k2) + 16 (24 - k1): lane (16 - k2) & 15, register 24 - k1
        const int partner = (16 - k2) & 15;
        const double2 wk2 = live ? tw[k2] : make_double2(1.0, 0.0);
        float* mag = mags + f * 404;
#pragma unroll
        for (int k1 = 0; k1 < 25; ++k1) {
            double2 zp = shfl_d2(Z[24 - k1], partner);
            if (k2 == 0) zp = (k1 == 0) ? Z[0] : Z[25 - k1];    // 400 - 16 k1 = 16 (25 - k1): same lane
            const double2 zk = Z[k1];
            const double2 e = make_double2(0.5 * (zk.x + zp.x), 0.5 * (zk.y - zp.y));
            const double2 dd = make_double2(0.5 * (zk.x - zp.x), 0.5 * (zk.y + zp.y));
            const double2 o = make_double2(dd.y, -dd.x);         // -i d
            const double2 x = cadd(e, cmul(cmul(wk2, kMelW50[k1]), o));
            const float re = (float)x.x, im = (float)x.y;        // complex64 store of librosa.stft
            if (live) mag[k2 + 16 * k1] = (float)sqrt((double)re * (double)re + (double)im * (double)im);
        }
        if (live && k2 == 0) {                                   // Nyquist bin: X[400] = E[0] - O[0] = Re Z[0] - Im Z[0]
            const float re = (float)(Z[0].x - Z[0].y);
            mag[400] = fabsf(re);
        }
    }
    __syncthreads();
    // ---------------- sparse mel product + dB + normalise / clip, fp32 as NumPy does on float32 arrays ----------------
    for (int i = tid; i < MEL_BANDS * MEL_FPB; i += MEL_THREADS) {
        const int f = i / MEL_BANDS, m = i % MEL_BANDS;
        const long long t = f0 + (long long)blockIdx.x * MEL_FPB + f;
        if (t >= f1) continue;
        const float* mag = mags + f * 404;
        const int off = p.boff[m], st = p.bstart[m], len = p.blen[m];
        float s = 0.0f;
        for (int j = 0; j < len; ++j) s = fmaf(__ldg(p.bvals + off + j), mag[st + j], s);
        dst.note(s);
        const float db = 20.0f * log10f(fmaxf(1e-5f, s)) - 20.0f;
        float v = 8.0f * ((db + 100.0f) / 100.0f) - 4.0f;
        v = fminf(fmaxf(v, -4.0f), 4.0f);
        outs[m * MEL_FPB + f] = v;
    }
    __syncthreads();
    for (int i = tid; i < MEL_BANDS * MEL_FPB; i += MEL_THREADS) {
        const int m = i / MEL_FPB, ff = i % MEL_FPB;
        const long long tt = f0 + (long long)blockIdx.x * MEL_FPB + ff;
        if (tt < f1) dst.put(m, tt, outs[i]);
    }
}

__global__ void __launch_bounds__(MEL_THREADS, 4) mel_kernel(const MelParams p) {
    mel_frames(p, MelWavSrc{p}, MelDenseDst{p}, 0, p.F);
}

// ---- streaming form (w2l_melstream_*): audio and mel live in power-of-two rings indexed by absolute position ----
// Frame f reads pre-emphasised samples [200 f - 400, 200 f + 400) and x[200 f - 401]: the reflection at the start uses
// absolute indices, so frames 0 and 1 are exact whatever has arrived.  A frame is final once 200 f + 400 <= L; only the
// frames that reach the end of the utterance reflect there, and they are computed with L = L_end (finish).  A ring slot
// is read only while it still holds the sample of that absolute index (the host never lets the writer lap the oldest
// sample a pending frame reads).
struct MelRingSrc {
    const float* ring;
    long long mask;      // ring length - 1
    long long L;         // L_end at finish; otherwise larger than any index read, so only the start reflects
    __device__ __forceinline__ long long len() const { return L; }
    __device__ __forceinline__ double x(long long j, int d) const { return (double)__ldg(ring + ((j + d) & mask)); }
};
struct MelRingDst {     // (80, R) row-major ring of frame columns; NaN anywhere in a frame sets *nan (sticky)
    float* mel;
    long long pitch;     // R
    int* nan;
    __device__ __forceinline__ void note(float s) const { if (s != s) atomicOr(nan, 1); }
    __device__ __forceinline__ void put(int m, long long t, float v) const { mel[(long long)m * pitch + (t & (pitch - 1))] = v; }
};

struct MelRingParams {
    const float* audio;
    long long audio_mask;
    float* mel;
    long long mel_pitch;
    long long L;          // see MelRingSrc::L
    long long f0, f1;     // frames to compute
    int* nan;
};

__global__ void __launch_bounds__(MEL_THREADS, 4) mel_ring_kernel(const MelParams p, const MelRingParams r) {
    mel_frames(p, MelRingSrc{r.audio, r.audio_mask, r.L}, MelRingDst{r.mel, r.mel_pitch, r.nan}, r.f0, r.f1);
}

// ---- many rings in one launch (w2l_stream_group_*): block b computes up to MEL_FPB frames of one session ----
// Each block reads its own descriptor, so one launch covers every session of a tick however few frames each has.  The
// body indexes frames from f0 + blockIdx.x * MEL_FPB; passing f0 = fb - blockIdx.x * MEL_FPB leaves that indexing, and
// with it the instruction sequence of mel_kernel and mel_ring_kernel, as it was.
struct MelGroupBlock {
    const float* audio;
    long long audio_mask;
    float* mel;
    long long mel_pitch;
    long long L;          // see MelRingSrc::L
    long long fb, f1;     // frames [fb, min(fb + MEL_FPB, f1))
    int* nan;             // the session's sticky flag
};

__global__ void __launch_bounds__(MEL_THREADS, 4) mel_group_kernel(const MelParams p, const MelGroupBlock* blocks) {
    const MelGroupBlock b = blocks[blockIdx.x];
    mel_frames(p, MelRingSrc{b.audio, b.audio_mask, b.L}, MelRingDst{b.mel, b.mel_pitch, b.nan},
               b.fb - (long long)blockIdx.x * MEL_FPB, b.f1);
}

}  // namespace w2l
