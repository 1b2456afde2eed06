/*
 * w2l.h — C-ABI of the H100-native Wav2Lip compute core (libw2l.so).
 *
 * The reference (Rudrabha/Wav2Lip) has no FFI: its boundary is the Python module surface
 * `models` / `audio` that the scripts import by bare name.  Each entry point below replaces
 * one of those Python call targets; the reference-side binding (a ctypes-backed `models`
 * package with the same class names, ctor/forward signatures and state_dict keys) lives in
 * wav2lip_b200/models/ and is described in INTEGRATION.md.
 *
 * Conventions
 *  - plain C types only: pointers, sizes, ints.  No torch / C++ types cross this boundary.
 *  - every function returns 0 on success, a negative W2L_E* code on failure; the message is
 *    available through w2l_last_error() (thread local).  Nothing throws across the ABI.
 *  - "dev" pointers are CUDA device pointers on the context's device; tensors are fp32,
 *    contiguous, in the layout the reference's callers build (NCHW / 5-D B,C,T,H,W).
 *  - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); calls are
 *    asynchronous on that stream unless stated otherwise.
 *  - a context is bound to one device and is not thread safe (one context per GPU / stream).
 *  - there is NO CPU fallback: every compute entry point fails with W2L_ENODEV when no
 *    sm_90 (H100) device is usable.
 */
#ifndef W2L_H_
#define W2L_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define W2L_ABI_VERSION 1

/* error codes */
#define W2L_OK        0
#define W2L_EINVAL   -1   /* bad argument / shape */
#define W2L_ENODEV   -2   /* no usable sm_90 CUDA device */
#define W2L_ECUDA    -3   /* CUDA runtime / driver error (see w2l_last_error) */
#define W2L_ENOMEM   -4
#define W2L_ESTATE   -5   /* e.g. forward before weights were loaded */

/* networks */
#define W2L_NET_GENERATOR 0   /* models.Wav2Lip            /root/reference/models/wav2lip.py:8-125   */
#define W2L_NET_SYNCNET   1   /* models.SyncNet_color      /root/reference/models/syncnet.py:7-66    */
#define W2L_NET_DISC      2   /* models.Wav2Lip_disc_qual  /root/reference/models/wav2lip.py:127-184 */
#define W2L_NET_S3FD      3   /* face_detection s3fd       /root/reference/face_detection/detection/sfd/net_s3fd.py:22-129 */

/* block kinds — /root/reference/models/conv.py */
#define W2L_BLOCK_CONV_BN_RELU   0   /* Conv2d           conv.py:5-19  */
#define W2L_BLOCK_CONVT_BN_RELU  1   /* Conv2dTranspose  conv.py:33-44 */
#define W2L_BLOCK_CONV_LRELU     2   /* nonorm_Conv2d    conv.py:21-31 */
#define W2L_BLOCK_CONV_PLAIN     3   /* bare nn.Conv2d heads: wav2lip.py:84, :152 (followed by Sigmoid); S3FD's mbox convs */
#define W2L_BLOCK_CONV_RELU      4   /* F.relu(nn.Conv2d(x)): the S3FD backbone, net_s3fd.py:72-106 */

/* operand precision of the tensor-core path (accumulation is always fp32) */
#define W2L_PREC_F16  0   /* fp16 operands: 10-bit mantissa, same as TF32 (default) */
#define W2L_PREC_BF16 1   /* bf16 operands: for checkpoints whose activations exceed the fp16 range */
#define W2L_PREC_F32X 2   /* fp32-faithful: every activation and weight is carried as hi + lo (two fp16 values, ~22
                             significant bits) and each product as x_hi*w_hi + x_lo*w_hi + x_hi*w_lo on the tensor
                             cores (3 MMAs, generic kernel only): ~1e-6 relative per block, ~1/4 of the throughput */

typedef struct w2l_ctx w2l_ctx;

/* One row of an architecture table: a conv block with the reference's own module path. */
typedef struct w2l_layer_info {
    char name[64];      /* e.g. "face_decoder_blocks.3.1" — state_dict prefix of the block */
    int32_t kind;       /* W2L_BLOCK_* */
    int32_t cin, cout;
    int32_t kh, kw, sh, sw, ph, pw;
    int32_t out_pad;    /* ConvTranspose2d output_padding */
    int32_t residual;   /* conv.py:16-18 */
    int32_t cout_real;  /* 0, or the parameter tensor's real output-channel count when `cout` is its 16-padded width (S3FD heads) */
} w2l_layer_info;

/* ---- introspection (host only; usable without a GPU) ---- */
int         w2l_abi_version(void);
const char* w2l_last_error(void);
int         w2l_net_num_layers(int net);
int         w2l_net_layer_info(int net, int index, w2l_layer_info* out);

/* ---- context ---- */
/* Replaces `Model().to(device)` (inference.py:169,178; wav2lip_train.py:356). */
int w2l_create(int device, int precision, w2l_ctx** out);
int w2l_destroy(w2l_ctx* ctx);

/* Replaces `model.load_state_dict(sd)` (inference.py:176): hands the context the fp32 device
 * tensors of one network by their reference state_dict names ("<block>.conv_block.0.weight",
 * "<block>.conv_block.1.running_var", "output_block.1.weight", ...).  Weights are re-packed
 * (fp16/bf16, tap-major K-major tiles; BatchNorm running stats folded into per-channel
 * scale/shift) on `stream`; the source tensors may be freed afterwards.  Re-callable.
 * Unknown names are ignored ("...num_batches_tracked"); a missing tensor is W2L_EINVAL. */
int w2l_load_weights(w2l_ctx* ctx, int net, int n_tensors, const char* const* names,
                     const void* const* dev_ptrs, const int64_t* numels, void* stream);

/* Replaces `Wav2Lip.forward(audio_sequences, face_sequences)` (wav2lip.py:87-125), eval mode.
 *   T == 0 : mel (B,1,80,16), face (B,6,96,96)      -> out (B,3,96,96)
 *   T  > 0 : mel (B,T,1,80,16), face (B,6,T,96,96)  -> out (B,3,T,96,96)   (t-major flatten inside) */
int w2l_generator_forward(w2l_ctx* ctx, const float* mel_dev, const float* face_dev, float* out_dev,
                          int B, int T, void* stream);

/* Same, with HOST buffers: H2D of the inputs, forward, D2H of the result, then a stream sync.
 * Buffers should be pinned for full PCIe bandwidth (pageable memory works, slower). */
int w2l_generator_forward_host(w2l_ctx* ctx, const float* mel_host, const float* face_host,
                               float* out_host, int B, int T);

/* Asynchronous form of the two host-buffer calls, for a serving loop that keeps the PCIe link and the GPU busy at
 * the same time (the reference's loop, inference.py:259-265, is copy -> forward -> copy, strictly serial):
 *   w2l_generator_submit_host / _submit_u8_host enqueue H2D -> forward -> D2H for one batch and return at once;
 *   at most two submissions are in flight (a third call first waits for the oldest);
 *   w2l_host_wait(ctx, keep) blocks until at most `keep` submissions are still in flight — their out_host buffers are
 *   complete when it returns, in submission order.  Host buffers must stay valid (and should be pinned) until retired.
 *       submit(batch 0); for k = 1..: submit(batch k); w2l_host_wait(ctx, 1); consume(batch k-1); ... w2l_host_wait(ctx, 0) */
int w2l_generator_submit_host(w2l_ctx* ctx, const float* mel_host, const float* face_host, float* out_host, int B, int T);
int w2l_generator_submit_u8_host(w2l_ctx* ctx, const float* mel_host, const uint8_t* faces_host, uint8_t* out_host, int N);
int w2l_host_wait(w2l_ctx* ctx, int keep_in_flight);

/* Scope row (f): the batch assembly around the generator call of inference.py, fused on the GPU.
 * Replaces inference.py:134-140 (mask the lower half, concat [masked | full] on channels, /255, NHWC->NCHW),
 * :259-263 (to device, forward) and :265,:269 (transpose, *255., astype(uint8)) — everything between the
 * cv2.resize of the crop (:126) and the cv2.resize of the prediction (:269):
 *   mel (N,1,80,16) fp32, faces (N,96,96,3) uint8 BGR crops -> out (N,96,96,3) uint8 BGR.
 * 8x fewer H2D and 4x fewer D2H bytes than the fp32 call. */
int w2l_generator_forward_u8(w2l_ctx* ctx, const float* mel_dev, const uint8_t* faces_dev, uint8_t* out_dev,
                             int N, void* stream);
int w2l_generator_forward_u8_host(w2l_ctx* ctx, const float* mel_host, const uint8_t* faces_host,
                                  uint8_t* out_host, int N);

/* Scope row (f2), the rest of the batch assembly: the two cv2.resize calls and the paste-back of inference.py, bit-identical
 * to OpenCV's fixed-point 8-bit INTER_LINEAR (11-bit coefficients; restated and pinned against cv2 in oracle/pipeline_oracle.py).
 *   frames (F,H,W,3) uint8 BGR on the device; boxes_host: N rows (frame index, y1, y2, x1, x2) in HOST memory (validated).
 *   w2l_crop_resize_u8    replaces `cv2.resize(face, (96, 96))` of every frames[f][y1:y2, x1:x2] (inference.py:102,:126)
 *                         -> crops (N,96,96,3) uint8, the input of w2l_generator_forward_u8.
 *   w2l_paste_u8          replaces `p = cv2.resize(p.astype(np.uint8), (x2-x1, y2-y1)); f[y1:y2, x1:x2] = p` on a copy of the
 *                         frame (inference.py:123, :267-271): pred (N,96,96,3) uint8 -> out_frames (N,H,W,3) uint8.
 *   w2l_lipsync_frames_u8 the whole inner loop of inference.py:120-140 + :259-271 in one call: crop + resize -> mask / concat
 *                         / 255 -> generator -> x255 -> uint8 -> resize -> paste.  mel (N,1,80,16) fp32. */
int w2l_crop_resize_u8(w2l_ctx* ctx, const uint8_t* frames_dev, int F, int H, int W, const int32_t* boxes_host, int N,
                       uint8_t* crops_dev, void* stream);
int w2l_paste_u8(w2l_ctx* ctx, const uint8_t* pred_dev, const uint8_t* frames_dev, int F, int H, int W,
                 const int32_t* boxes_host, int N, uint8_t* out_frames_dev, void* stream);
int w2l_lipsync_frames_u8(w2l_ctx* ctx, const float* mel_dev, const uint8_t* frames_dev, int F, int H, int W,
                          const int32_t* boxes_host, int N, uint8_t* out_frames_dev, void* stream);

/* Scope row (f3): the training scripts' batch assembly, `default_collate` of B `Dataset.__getitem__` calls
 * (wav2lip_train.py:111-164, identical in hq_wav2lip_train.py; color_syncnet_train.py:69-131) from a cache, in one launch.
 *   frames (n_frames,96,96,3) uint8 BGR = cv2.resize(cv2.imread(f), (96, 96)) (wav2lip_train.py:63-70); mels (n_mel_rows,80) fp32
 *   = every video's `audio.melspectrogram(wav).T` (:138-141) stacked.  Both in device or pinned host memory; pageable is refused.
 *   samples_host: B rows of int32 in HOST memory, validated before any launch (slot < n_frames, row + 16 <= end <= n_mel_rows,
 *   label 0 / 1).  Mel rows are absolute cache rows, `end` is the row after the sample's video.
 *   Pixels are float32(u / 255.) with the division in float64 (prepare_window, :101-106).  Outputs: 16-byte aligned device memory.
 * w2l_train_batch_wav2lip   rows of 17: window slots[5], wrong-window slots[5], mel row, indiv rows[5], end
 *                           -> x (B,6,5,96,96) (channels 0-2 the window with rows 48-95 zeroed, :152-157), indiv_mels (B,5,1,80,16)
 *                           (get_segmented_mels, :88-99), mel (B,1,80,16) (crop_audio_window, :75-86), gt (B,3,5,96,96) (:154)
 * w2l_train_batch_syncnet   rows of 8: window slots[5], mel row, label, end
 *                           -> x (B,15,48,96) (channel 3t+c, rows 48-95: color_syncnet_train.py:123-126), mel (B,1,80,16), y (B,1) */
int w2l_train_batch_wav2lip(w2l_ctx* ctx, const uint8_t* frames, int64_t n_frames, const float* mels, int64_t n_mel_rows,
                            const int32_t* samples_host, int B, float* x, float* indiv_mels, float* mel, float* gt, void* stream);
int w2l_train_batch_syncnet(w2l_ctx* ctx, const uint8_t* frames, int64_t n_frames, const float* mels, int64_t n_mel_rows,
                            const int32_t* samples_host, int B, float* x, float* mel, float* y, void* stream);

/* Scope row (f4): the S3FD face detector's network (face_detection/detection/sfd/net_s3fd.py:22-129), the per-frame GPU
 * work of inference.py's face_detect (:73-100): 19 conv+ReLU layers (VGG16 backbone + fc6/fc7 + conv6/7), 5 max-pools,
 * 3 L2Norm layers and the 12 mbox heads, max-out of the first scale's background logits included.
 *   img (B,3,H,W) fp32, BGR minus (104,117,123) as detect.py:21-23 / :60-61 prepare it  ->  12 maps
 *   outs[2i] = cls_i (B,2,h_i,w_i), outs[2i+1] = reg_i (B,4,h_i,w_i), i = 0..5 (strides 4..128), raw logits as the module
 *   returns them (softmax / threshold / decode / NMS of detect.py:31-56 and bbox.py:44-64: w2l_s3fd_detect_u8 below).
 * w2l_s3fd_out_dims writes the six (h_i, w_i) pairs for an H x W input.  Weights: w2l_load_weights(ctx, W2L_NET_S3FD, ...)
 * with the module's own state_dict names ("conv1_1.weight", ..., "conv3_3_norm.weight", "conv7_2_mbox_loc.bias"). */
int w2l_s3fd_out_dims(int H, int W, int32_t* dims12);
int w2l_s3fd_forward(w2l_ctx* ctx, const float* img_dev, float* const* outs12_dev, int B, int H, int W, void* stream);

/* The whole detector on the device: face_detection/detection/sfd detect.py:58-94 + bbox.py:44-64 + sfd_detector.py:40-46.
 *   frames (B,H,W,3) uint8 in the order detect_from_batch takes them (reverse_channels = 1: reversed first, as api.py:64
 *   does to the frames inference.py passes) -> per image the boxes that
 *   survive greedy NMS at IoU 0.3 with score > 0.5, best first, at most max_det (>= 1) of them:
 *   dets (B, max_det, 5) fp32 = x1 y1 x2 y2 score (rows past counts[b] are zero), counts (B) int32.
 *   outs12: NULL, or the 12 maps of w2l_s3fd_forward, bit-identical to that call on the same frames.
 * Only locations whose own score exceeds 0.5 can reach the output, so the reference's 0.05 threshold, its cross-image
 * candidate union and their duplicates are not materialised; ties in score are ordered by descending location index
 * (DESIGN.md §3.6).  Shares the S3FD plan of (B,H,W) with w2l_s3fd_forward. */
int w2l_s3fd_detect_u8(w2l_ctx* ctx, const uint8_t* frames_dev, int B, int H, int W, int reverse_channels, int max_det,
                       float* dets_dev, int32_t* counts_dev, float* const* outs12_dev, void* stream);

/* Replaces `SyncNet_color.forward(audio, face)` (syncnet.py:55-66):
 *   mel (B,1,80,16), face (B,15,48,96) -> audio_emb (B,512), face_emb (B,512), both L2-normalised. */
int w2l_syncnet_forward(w2l_ctx* ctx, const float* mel_dev, const float* face_dev,
                        float* audio_emb_dev, float* face_emb_dev, int B, void* stream);

/* Scope row (a8) + evaluation loops (wav2lip_train.py:262-292, hq_wav2lip_train.py eval): the expert-discriminator
 * call on generated frames, `get_sync_loss` (wav2lip_train.py:192-198) up to the embeddings:
 *   g[:, :, :, H/2:]  ->  cat([g[:, :, i] for i in range(syncnet_T)], dim=1)  ->  syncnet(mel, .)
 * with the slice and the channel stack done as addressing by the ingest kernel:
 *   mel (B,1,80,16), frames (B,3,T,96,96) with T == 5 -> audio_emb (B,512), face_emb (B,512). */
int w2l_syncnet_forward_frames(w2l_ctx* ctx, const float* mel_dev, const float* frames_dev, float* audio_emb_dev,
                               float* face_emb_dev, int B, int T, void* stream);

/* Replaces `cosine_loss(a, v, y)` (wav2lip_train.py:178-183, color_syncnet_train.py:133-138):
 *   d = F.cosine_similarity(a, v) (eps 1e-8);  loss = nn.BCELoss()(d.unsqueeze(1), y)  (mean; log clamped at -100).
 *   a, v (B,D) fp32; y (B) fp32 targets or NULL for all ones (get_sync_loss, :197); loss: 1 float on the device.
 *   Forward value only (the evaluation loops); deterministic summation order. */
int w2l_cosine_bce_loss(w2l_ctx* ctx, const float* a_dev, const float* v_dev, const float* y_dev, int B, int D,
                        float* loss_dev, void* stream);

/* Replaces `recon_loss = nn.L1Loss()` (wav2lip_train.py:191, :228, :281): loss = mean |x - y| over n fp32 elements
 * (16-byte aligned pointers); loss: 1 float on the device.  HBM-bound: 8 bytes read per element pair. */
int w2l_l1_loss(w2l_ctx* ctx, const float* x_dev, const float* y_dev, int64_t n, float* loss_dev, void* stream);

/* Replaces `Wav2Lip_disc_qual.forward(face_sequences)` (wav2lip.py:176-184):
 *   frames (B,3,T,96,96) -> prob (B*T,1), rows t-major (row = t*B + b). */
int w2l_disc_forward(w2l_ctx* ctx, const float* frames_dev, float* prob_dev, int B, int T, void* stream);

/* Replaces one `models.conv.{Conv2d,Conv2dTranspose,nonorm_Conv2d}.forward` (conv.py:15-19,29-31,
 * 42-44), eval mode — the operator-level entry used by the per-geometry parity tests.
 *   x (N,cin,H,W) fp32 -> y (N,cout,Hout,Wout) fp32.  weight is (cout,cin,kh,kw), or
 *   (cin,cout,kh,kw) for the transposed block; bn_* are NULL for nonorm/plain blocks. */
int w2l_conv_block_forward(w2l_ctx* ctx, const w2l_layer_info* spec,
                           const float* x_dev, int N, int H, int W,
                           const float* weight_dev, const float* bias_dev,
                           const float* bn_weight_dev, const float* bn_bias_dev,
                           const float* bn_mean_dev, const float* bn_var_dev,
                           float* y_dev, void* stream);

/* Debug/test aid: copy the output of block `layer` (index into the net's table) of the LAST
 * forward of `net` to y (N,cout,H,W) fp32.  *h,*w,*c receive the dims (any may be NULL).
 * W2L_NET_S3FD also exports its glue ops after the 31 conv layers: 31..35 = the five max-pools (pool1..pool5),
 * 36..38 = the three L2Norm outputs (conv3_3_norm, conv4_3_norm, conv5_3_norm).  The mbox heads (19..30) export all
 * 16 stored channels; channels cout_real..15 are padding. */
int w2l_debug_layer_output(w2l_ctx* ctx, int net, int layer, float* y_dev, int* n, int* c, int* h, int* w,
                           void* stream);

/* Replaces `audio.melspectrogram(wav)` (audio.py:45-51 with hparams.py:33-73):
 *   wav (L) fp32 -> mel (80, 1 + L/200) fp32 in [-4,4], row-major as numpy returns it.
 *   L >= 2; clips shorter than n_fft/2 = 400 samples reflect more than once, as np.pad(mode="reflect") does.
 *   w2l_melspectrogram_host first retires every asynchronous host submission of the context (w2l_host_wait(ctx, 0)):
 *   it shares their staging buffers. */
int w2l_melspectrogram(w2l_ctx* ctx, const float* wav_dev, int64_t n_samples, float* mel_dev, void* stream);
int w2l_melspectrogram_host(w2l_ctx* ctx, const float* wav_host, int64_t n_samples, float* mel_host);
/* number of frames for n_samples: 1 + n_samples/200 (librosa center=True) */
int64_t w2l_mel_num_frames(int64_t n_samples);

/* Scope row (f): replaces the mel chunking loop of inference.py:231-240 — chunk i = mel[:, s_i : s_i+16] with
 * s_i = int(i * 80./fps), the last chunk right-aligned; chunks out is (n_chunks,1,80,16) fp32, i.e. already the
 * `mel_batch` layout of inference.py:260.  w2l_mel_num_chunks gives n_chunks for a mel of n_frames columns. */
int64_t w2l_mel_num_chunks(int64_t n_frames, double fps);
int w2l_mel_chunks(w2l_ctx* ctx, const float* mel_dev, int64_t n_frames, double fps, float* chunks_dev,
                   int64_t n_chunks, void* stream);

/* ---- streaming ---- */
/* Streaming form of w2l_melspectrogram: audio arrives in pieces, frames come out as soon as they are final, and every
 * frame is bit-identical to the same column of w2l_melspectrogram on the whole utterance.  Frame f is final once
 * 200 f + 400 <= L (L = samples received); the frames that reach the end of the utterance need its length and come out
 * of _finish.  Audio and mel live in device rings of fixed size (audio_ring_log2: log2 of the audio ring in samples,
 * 11..24, 0 = 16; the mel ring follows from it); a push of any length is split internally, so device memory does not
 * grow with the stream.
 *   pcm: fp32 16 kHz samples in host memory (pageable or pinned) or in device memory of the context's device.
 *   _push writes the newly final frames to mel_dev as an (80, n_new) row-major block; *n_new may be 0.  The caller
 *   sizes mel_dev with w2l_melstream_pending (frames a push of n_samples more, or the finish, will write).
 *   _finish writes the remaining frames; the stream then has 1 + L/200 frames in all (L >= 2).
 *   *nan_seen (optional, synchronises the stream) reports whether any frame so far held a NaN (the reference raises
 *   on that, inference.py:228-229).
 * Calls are asynchronous on `stream` except where stated.  pcm may be reused when _push returns if it is host memory
 * (for pinned memory _push waits for its copies, and so for the work queued on `stream` before them); device pcm is
 * read by work queued on `stream`, ordered like any other asynchronous copy there. */
typedef struct w2l_melstream w2l_melstream;
int w2l_melstream_create(w2l_ctx* ctx, int audio_ring_log2, w2l_melstream** out);
int64_t w2l_melstream_pending(const w2l_melstream* ms, int64_t n_samples, int finish);
int w2l_melstream_push(w2l_melstream* ms, const float* pcm, int64_t n_samples, float* mel_dev, int64_t cap_frames,
                       int64_t* n_new, int* nan_seen, void* stream);
int w2l_melstream_finish(w2l_melstream* ms, float* mel_dev, int64_t cap_frames, int64_t* n_new, int* nan_seen,
                         void* stream);
int w2l_melstream_destroy(w2l_melstream* ms);

/* Streaming lip-sync session: the whole inference loop of inference.py (:224-244 mel and chunks, :87-103 boxes,
 * :120-140 and :259-271 generator and paste) on audio that arrives in pieces, for a fixed face video.  Each output
 * frame is emitted as soon as the audio received so far fixes it, and the concatenated output equals the offline loop
 * bit for bit.  Output i shows frame i % n_total (n_total = min(chunk count, F), inference.py:244) with mel chunk i.
 *
 * The video and its boxes: frames_dev (F,H,W,3) uint8 on the device (it must stay valid while the session lives), and
 * either F detector rects (x1,y1,x2,y2 per frame, as get_detections_for_batch returns them) that the session pads,
 * clips and smooths as inference.py:87-103 does (the smoothing of inference.py:59-66 over the first n_total frames;
 * d->nosmooth turns it off), or one fixed box (d->has_box, d->box = y1,y2,x1,x2: inference.py:116-119). */
typedef struct w2l_stream_desc {
    int32_t F, H, W;     /* video frames and size */
    double fps;          /* chunk start s_i = int(i * 80./fps), inference.py:232 */
    int32_t nosmooth;
    int32_t has_box;     /* 1: box below for every frame; rects unused */
    int32_t box[4];      /* y1, y2, x1, x2 */
    int32_t pads[4];     /* top, bottom, left, right (inference.py --pads, default 0 10 0 0) */
} w2l_stream_desc;

/* One emitted row: output index, mel chunk start (absolute mel frame), video frame index, box y1, y2, x1, x2. */
#define W2L_STREAM_ROW 7

/* Pure host function (no device, no context): the rows that n_samples received audio samples fix, or, with
 * final != 0, all rows of an utterance of n_samples.  *n_fixed gets their count; rows [first_row, first_row + cap)
 * of them (those that exist) are written to rows_host as W2L_STREAM_ROW int32 each.  rects_host: F x 4, unused with a
 * fixed box.  A final length with fewer than 16 mel frames is W2L_EINVAL (there is no chunk). */
int w2l_stream_schedule(const w2l_stream_desc* d, const int32_t* rects_host, int64_t n_samples, int final_,
                        int64_t first_row, int64_t cap, int32_t* rows_host, int64_t* n_fixed);

/* Pure host function: *n_frames gets need, the count of the prefix [0, need) of frames whose rects the rows that
 * n_samples fix read (all rows of an utterance of n_samples with final != 0).  Rects of frames at or past need do not
 * change those rows.  F == 1: 1.  nosmooth: the frames shown.  Smoothing: rows i read rects i .. i+4 while n_total is
 * unknown, all of [0, n_total) once it is known.  At final it is n_total (inference.py:244, :113).  d must not have
 * has_box; its rects are not needed. */
int w2l_stream_detect_need(const w2l_stream_desc* d, int64_t n_samples, int final_, int64_t* n_frames);

/* Every step runs the generator at exactly `batch` rows (one plan; rows past the ready ones repeat the last ready row
 * and are dropped), from a CUDA graph captured once per session and replayed (W2L_DISABLE_STREAMGRAPH=1 launches the
 * same kernels directly).  The generator weights must be loaded; loading new ones between pushes is allowed.
 * _push / _finish write n_out output frames (n_out, H, W, 3) uint8 to out_dev; they are output indices
 * first_index .. first_index + n_out - 1.  Size out_dev with w2l_stream_pending.  A push whose audio gives a mel frame
 * holding a NaN fails with W2L_EINVAL and the reference's message (inference.py:228-229) and writes no frame of a
 * chunk that contains it; so does every later call.  The session must be destroyed before its context.
 * The mel work runs on a stream of the session's own: a push waits on the host for its own new mel frames and their
 * NaN flag (host pcm is then copied), not for the steps already queued on `stream`; device pcm makes the mel work wait
 * for the work queued on `stream` first.  Steps, pastes and outputs are ordered on `stream`. */
typedef struct w2l_stream w2l_stream;
int w2l_stream_create(w2l_ctx* ctx, const uint8_t* frames_dev, const w2l_stream_desc* d, const int32_t* rects_host,
                      int batch, w2l_stream** out);
int w2l_stream_pending(const w2l_stream* s, int64_t n_samples, int finish, int64_t* n_out);
int w2l_stream_push(w2l_stream* s, const float* pcm, int64_t n_samples, uint8_t* out_dev, int64_t cap,
                    int64_t* first_index, int64_t* n_out, void* stream);
int w2l_stream_finish(w2l_stream* s, uint8_t* out_dev, int64_t cap, int64_t* first_index, int64_t* n_out,
                      void* stream);
int w2l_stream_destroy(w2l_stream* s);

/* Stream group: many streaming sessions (each as w2l_stream_*: the loop of inference.py:224-244, :87-103, :120-140 and
 * :259-271 on audio that arrives in pieces) sharing one context, one caller stream and one set of generator steps.  A
 * tick takes the new audio of any subset of the sessions (and may finish some); it computes every row that audio fixes
 * within the tick, pooled across sessions into as few steps as possible: full max_batch steps, then the rest in the
 * smallest bucket (a power of two below max_batch, or max_batch) that holds it.  Each session's output equals a lone
 * w2l_stream (and the offline loop) fed the same pieces, bit for bit.  Per tick the host makes one upload copy, one
 * audio scatter and one mel launch, one NaN read-back (its only wait, apart from reusing a table staging slot), and per
 * step one table copy and one graph launch, however many sessions take part.
 *   _create: max_batch 1..4096; audio_ring_log2 as w2l_melstream_create (0 = 16).  The generator weights must be
 *     loaded; new ones may be loaded between ticks.  The group must be destroyed before its context.
 *   _open: frames_dev, d and rects_host as w2l_stream_create; *session_id gets the session's id.
 *   _open_detect: as _open without rects or box (d->has_box = 0): the group finds each frame's box with the S3FD weights
 *     of its context (w2l_load_weights(ctx, W2L_NET_S3FD, ...); W2L_ESTATE without them), as
 *     get_detections_for_batch_u8 does on inference.py's BGR frames (inference.py:68-103: reversed channels, the first
 *     box, clipped at 0 and truncated), on a stream of the group's own.  Frames of at least 32 x 32, written by work
 *     queued on the legacy default stream before the call (or complete).  Only the frames a tick's rows read are
 *     detected (w2l_stream_detect_need), just before that tick needs them: _open queues the frames of the first 400 ms of
 *     audio without waiting, each tick the frames its own audio needs that no launch covers yet, then those of 200 ms
 *     more, and each tick's one host wait covers every launch queued before it.  Launches take up to 16 frames of one
 *     size from any sessions; S3FD plans of batch 1, 4 and 16 per frame size stay pinned while a detecting session of
 *     that size is open.  A frame a tick's rows need without a face (or with a non-finite box) fails its session as a
 *     NaN does, with face_boxes' message (inference.py:91-93) or the non-finite box's, both naming the frame.  A frame
 *     past the ones the utterance needs fails nothing.
 *   _close: the session's rings are released (waits for the device).
 *   _pending (host only): for each named session, the frames a tick with n_samples more (and finish) would emit.
 *   _tick: n sessions ids[i] with pcm[i] (n_samples[i] fp32 16 kHz samples, host or device memory; pcm may be null
 *     when every n_samples is 0) and finish[i] (finish may be null); frames go to out_dev[i] (cap[i] frames of
 *     (H, W, 3) uint8), output indices first_index[i] .. + n_out[i] - 1.  Every argument, pointer and row is checked
 *     before anything is launched; a bad one fails the whole tick (W2L_EINVAL / W2L_ESTATE) with nothing done.  A mel
 *     frame holding a NaN fails its session only: status[i] = W2L_EINVAL, its rows of the tick are not run, and so on
 *     for every later tick that names it; w2l_stream_group_error gives the reference's message (inference.py:228-229),
 *     "" for a session that has not failed.  The return code is for group-wide errors.
 *   _buckets (host only, no context): the bucket of each step that n_rows pooled rows take; returns the step count and
 *     writes the first cap sizes.
 *   _counters: CUDA API submissions (launches, graph launches, copies, event records and waits), host waits and steps
 *     made by all ticks so far (any may be null). */
typedef struct w2l_stream_group w2l_stream_group;
int w2l_stream_group_create(w2l_ctx* ctx, int max_batch, int audio_ring_log2, w2l_stream_group** out);
int w2l_stream_group_open(w2l_stream_group* g, const uint8_t* frames_dev, const w2l_stream_desc* d,
                          const int32_t* rects_host, int32_t* session_id);
int w2l_stream_group_open_detect(w2l_stream_group* g, const uint8_t* frames_dev, const w2l_stream_desc* d,
                                 int32_t* session_id);
int w2l_stream_group_close(w2l_stream_group* g, int32_t session_id);
int w2l_stream_group_pending(const w2l_stream_group* g, int n, const int32_t* ids, const int64_t* n_samples,
                             const int32_t* finish, int64_t* n_out);
int w2l_stream_group_tick(w2l_stream_group* g, int n, const int32_t* ids, const float* const* pcm,
                          const int64_t* n_samples, const int32_t* finish, uint8_t* const* out_dev, const int64_t* cap,
                          int64_t* first_index, int64_t* n_out, int32_t* status, void* stream);
const char* w2l_stream_group_error(const w2l_stream_group* g, int32_t session_id);
int w2l_stream_group_buckets(int max_batch, int64_t n_rows, int32_t* sizes, int64_t cap);
int w2l_stream_group_counters(const w2l_stream_group* g, int64_t* calls, int64_t* host_waits, int64_t* steps);
int w2l_stream_group_destroy(w2l_stream_group* g);

/* ---- test aids ---- */
/* keep every block output of subsequent plans addressable (no buffer reuse) for w2l_debug_layer_output */
int w2l_set_debug(w2l_ctx* ctx, int keep_all_layer_outputs);
/* the kernel's own (80 x 401) Slaney mel filterbank, dense fp32, written to HOST memory */
int w2l_mel_basis_host(float* out_host);

/* Which conv kernel a launch uses, so that a parity test can assert the path it exercises. */
#define W2L_KFAM_IGEMM        0   /* generic implicit-GEMM kernel (conv_igemm.cuh) */
#define W2L_KFAM_PATCH        1   /* patch kernel with resident weights (conv_patch.cuh) */
#define W2L_KFAM_CONVT_FUSED  2   /* fused 4-phase transposed conv (convt_fused.cuh) */
typedef struct w2l_kernel_info {
    char    name[64];   /* the op's plan label ("b [patch]", "b.ph01 [2M]", "b [cm]", ...); in the table listing "[cm]" for
                         * an instantiation that also has the channel-major form, else empty */
    int32_t family;     /* W2L_KFAM_* */
    int32_t bn, bk, mt, head, bf16, x2, tma_epi, fold;
    int32_t m_tiles, n_tiles, grid;
} w2l_kernel_info;
/* every compiled conv kernel instantiation (generic, patch, fused transposed conv); host only */
int w2l_debug_kernel_table(int cap, w2l_kernel_info* out);
/* the conv launches of the last plan of `net`; net = -1: of the last w2l_conv_block_forward call */
int w2l_debug_plan_kernels(w2l_ctx* ctx, int net, int cap, w2l_kernel_info* out);
/* Both return the number of entries written (at most cap), or a negative W2L_E* code; out == NULL returns the count. */
/* The sorted pre-NMS candidates (score > 0.5) of `image` of the last S3FD call, which must have been w2l_s3fd_detect_u8:
 * min(n, cap) rows of x1 y1 x2 y2 score location-index to HOST memory, *n = all candidates of the image, *nms_path = 0 if
 * its NMS ran in shared memory, 1 if in global memory.  Synchronises the device. */
int w2l_debug_s3fd_candidates(w2l_ctx* ctx, int image, int cap, float* out_host, int* n, int* nms_path);

/* ---- training step (scope row f1): wav2lip_train.py:210-231, color_syncnet_train.py:146-163, hq_wav2lip_train.py:213-255 ----
 * Train-mode forward (BatchNorm on batch statistics over the T*B flatten, conv.py:8-11 / wav2lip.py:93-94; running
 * averages updated with momentum 0.1) and backward through every block, as kernels: conv / dgrad on the wgmma conv
 * kernels, wgrad on a wgmma kernel whose K dimension is the pixel index, BatchNorm / ReLU / residual passes,
 * loss gradients, multi-tensor Adam, bucketed NCCL all-reduce of the gradients.  bf16 operands, fp32 accumulation,
 * fp32 master parameters and gradients (the context must be created with W2L_PREC_BF16).
 *
 * w2l_train_bind replaces `optimizer = optim.Adam([p for p in model.parameters() ...])` + the module's own tensors
 * (wav2lip_train.py:356-360): it hands the context, by reference state_dict name, the caller's fp32 device tensors —
 * parameters (value + gradient pointer; NULL gradient = frozen, wav2lip_train.py:188-189) and BatchNorm buffers
 * (running_mean / running_var, gradient NULL).  The pointers must stay valid; values are re-read (and the 16-bit weight
 * slabs re-packed) at every training forward, gradients are written by the backward, running averages are updated in
 * place.  Gradients laid out contiguously (one arena in state_dict order) are all-reduced as three large buckets. */
#define W2L_TRAIN_WGRAD           1   /* compute parameter gradients into the bound gradient tensors */
#define W2L_TRAIN_ACCUMULATE      2   /* add to the bound gradient tensors instead of overwriting (two backward() calls, hq_wav2lip_train.py:248-253) */
#define W2L_TRAIN_INPUT_GRAD      4   /* the plan also produces dL/d(input frames) (expert / discriminator inside a generator step) */
#define W2L_TRAIN_NO_STAT_UPDATE  8   /* leave running_mean / running_var untouched */
int w2l_train_bind(w2l_ctx* ctx, int net, int n_tensors, const char* const* names, void* const* value_ptrs,
                   void* const* grad_ptrs, const int64_t* numels);

/* Train-mode forward; keeps the tape (block inputs, pre-BatchNorm outputs, outputs) for w2l_train_backward.
 *   W2L_NET_GENERATOR: in0 = mel, in1 = face (4-D with T == 0 or 5-D with T > 0, as w2l_generator_forward), out0 = g.
 *                      out0 must stay valid until the backward (the head's backward re-reads it).
 *   W2L_NET_SYNCNET  : in0 = mel (B,1,80,16); in1 = face (B,15,48,96) [T == 0] or frames (B,3,5,96,96) [T == 5];
 *                      out0 = audio_embedding, out1 = face_embedding (B,512), L2-normalised.
 *   W2L_NET_DISC     : in0 = frames (B,3,T,96,96), out0 = prob (B*T,1) t-major. */
int w2l_train_forward(w2l_ctx* ctx, int net, const float* in0_dev, const float* in1_dev, float* out0_dev, float* out1_dev,
                      int B, int T, int flags, void* stream);

/* Backward of the last w2l_train_forward of `net`.  d0 (/ d1) = dL/d out0 (/ out1) fp32, same shapes; with
 * W2L_TRAIN_WGRAD the bound gradient tensors receive dL/dparameter (`loss.backward()`, wav2lip_train.py:230);
 * dinput (needs W2L_TRAIN_INPUT_GRAD at the forward) receives dL/d in1 (SyncNet: frames (B,3,5,96,96) — zero in the
 * upper half — or face (B,15,48,96)) or dL/d in0 (disc frames), fp32. */
int w2l_train_backward(w2l_ctx* ctx, int net, const float* d0_dev, const float* d1_dev, float* dinput_dev, int flags,
                       void* stream);

/* Replaces `optimizer.step()` (torch.optim.Adam, no weight decay / amsgrad; wav2lip_train.py:231, :357-360) on every
 * bound tensor of `net` that has a gradient: one multi-tensor kernel; moments live in the context. */
int w2l_adam_step(w2l_ctx* ctx, int net, float lr, float beta1, float beta2, float eps, void* stream);

/* One whole iteration of wav2lip_train.py:210-231 on the bound generator and (frozen, train-mode as in the scripts,
 * :187-189) expert: g = model(indiv_mels, x); sync_loss = get_sync_loss(mel, g) if syncnet_wt > 0; l1 = L1(g, gt);
 * loss = syncnet_wt*sync + (1-syncnet_wt)*l1; backward; [gradient all-reduce, overlapped]; Adam(lr, (0.9,0.999), 1e-8).
 *   indiv_mels (B,T,1,80,16), x (B,6,T,96,96), mel (B,1,80,16), gt (B,3,T,96,96); losses_dev: 4 floats on the device
 *   [sync_loss, l1, 0, loss] or NULL. */
int w2l_wav2lip_train_step(w2l_ctx* ctx, const float* indiv_mels_dev, const float* x_dev, const float* mel_dev,
                           const float* gt_dev, int B, int T, float syncnet_wt, float lr, float* losses_dev, void* stream);
/* One whole iteration of hq_wav2lip_train.py:212-256 on the bound generator, (frozen, train-mode) expert and
 * discriminator, all bound to this context (the discriminator's gradients in one contiguous arena):
 *   g = model(indiv_mels, x); sync_loss if syncnet_wt > 0; perceptual = BCE(disc(g), 1) if disc_wt > 0; l1;
 *   loss = syncnet_wt*sync + disc_wt*perceptual + (1-syncnet_wt-disc_wt)*l1; backward; Adam(lr, (0.5,0.999), 1e-8);
 *   then the discriminator: BCE(disc(gt), 1) + BCE(disc(g.detach()), 0), backward, Adam(disc_lr, (0.5,0.999), 1e-8).
 * The discriminator's forward on g runs once (the value :252 recomputes); its step runs beside the generator's backward.
 * With a communicator (w2l_comm_init) both networks' gradients are averaged over the ranks.
 *   inputs as w2l_wav2lip_train_step; losses_dev: 6 floats on the device
 *   [sync_loss, l1, perceptual, loss, disc_real_loss, disc_fake_loss] or NULL. */
int w2l_hq_wav2lip_train_step(w2l_ctx* ctx, const float* indiv_mels_dev, const float* x_dev, const float* mel_dev,
                              const float* gt_dev, int B, int T, float syncnet_wt, float disc_wt, float lr, float disc_lr,
                              float* losses_dev, void* stream);
/* One whole iteration of color_syncnet_train.py:149-163 on the bound expert: a, v = model(mel, x) in train mode;
 * loss = cosine_loss(a, v, y); backward; [gradient all-reduce, overlapped]; Adam(lr, (0.9,0.999), 1e-8).
 *   mel (B,1,80,16), x (B,15,48,96), y (B,1) in {0, 1}; loss_dev: 1 float on the device or NULL. */
int w2l_syncnet_train_step(w2l_ctx* ctx, const float* mel_dev, const float* x_dev, const float* y_dev, int B, float lr,
                           float* loss_dev, void* stream);
/* `optimizer.state_dict()` / `optimizer.load_state_dict()` of the fused steps' Adam: the first and second moments of the
 * n named bound tensors of `net` (each with a gradient; m_ptrs[i] / v_ptrs[i] are fp32 device buffers of the tensor's
 * size) are copied out of the context (direction 0) or into it (direction 1), and *step, the step count of the bias
 * correction, is read (0) or set (1).  Before the first step the moments are zero and the count is 0. */
int w2l_adam_state(w2l_ctx* ctx, int net, int direction, int n, const char* const* names, float* const* m_ptrs,
                   float* const* v_ptrs, int64_t* step, void* stream);
/* copies the generator output g (B,3,T,96,96) of the last fused step into out_dev (n floats) */
int w2l_train_last_output(w2l_ctx* ctx, float* out_dev, int64_t n, void* stream);
/* algorithmic forward FLOPs of the last training plan of `net` (2 x true MACs of its convs) */
double w2l_train_flops(w2l_ctx* ctx, int net);

/* Per-stage CUDA-event times of the last training plan of `net` (run one forward + backward first): rows
 * "<block> fwd | bn | bwd_bn | dgrad | wgrad" with the stage's algorithmic FLOPs; returns the number of rows (<= cap). */
int w2l_train_profile(w2l_ctx* ctx, int net, int iters, int cap, float* ms_out, double* flop_out, char (*names_out)[64],
                      void* stream);

/* Data-parallel training: the gradient all-reduce is the one collective of the system (SURVEY.md 8e).  NCCL is
 * resolved at run time from the process (torch loads libnccl.so.2); rank 0 creates the 128-byte unique id, the host
 * side broadcasts it (torch.distributed), every rank calls w2l_comm_init.  w2l_wav2lip_train_step then averages the
 * gradients over the ranks (ncclAvg) in three buckets launched on a side stream as the backward completes them. */
int w2l_comm_unique_id(w2l_ctx* ctx, char* id128);
int w2l_comm_init(w2l_ctx* ctx, const char* id128, int rank, int world);

/* One conv.py block in train mode, forward + backward (operator-level entry of the per-geometry gradient tests):
 *   x (N,cin,H,W), dy (N,cout,Ho,Wo) fp32 -> y, dx (same layouts; dy/dx/dw may be NULL), dw in the parameter's own
 *   layout, db, dgamma, dbeta; bn_mean / bn_var (running averages) are updated in place when given. */
int w2l_conv_block_train(w2l_ctx* ctx, const w2l_layer_info* spec, const float* x_dev, int N, int H, int W,
                         float* weight_dev, float* bias_dev, float* bn_weight_dev, float* bn_bias_dev, float* bn_mean_dev,
                         float* bn_var_dev, const float* dy_dev, float* y_dev, float* dx_dev, float* dw_dev, float* db_dev,
                         float* dgamma_dev, float* dbeta_dev, void* stream);

/* Range guard of the fp16 modes (W2L_PREC_F16 / _F32X): every epilogue that stores an activation sets a sticky
 * per-device flag when the rounded value leaves the fp16 range (|v| > 65504 -> inf, or NaN).  Synchronises `stream`,
 * writes the flag to *flag (0 = every activation stored so far was finite) and, if `clear`, resets it.  A checkpoint
 * that trips it must run in W2L_PREC_BF16 (fp32's exponent range).  bf16 contexts never set it. */
int w2l_f16_overflow(w2l_ctx* ctx, int clear, int* flag, void* stream);

/* ---- training test aids: the blocks of a training plan and their tape, for per-block parity tests ---- */
#define W2L_WG_PLAIN       0   /* stride-1 conv: dz on the dense pixel grid, x read at the tap offset */
#define W2L_WG_STRIDED     1   /* strided conv: x read at stride x output pixel + tap offset */
#define W2L_WG_TRANSPOSED  2   /* transposed conv: x on the dense grid, dz read strided */
#define W2L_WG_SWAP        3   /* stride-1 conv with wide input, narrow output: x on the dense grid, dz per tap */
#define W2L_WG_FOLDED      4   /* K-folded first layer: a "tap" is a filter row of the folded input copy */
typedef struct w2l_train_block_info {
    char    name[64];            /* the block's state_dict prefix ("block" for w2l_conv_block_train) */
    int32_t layer;               /* index into the net's table */
    int32_t kind, cin, cout, kh, kw, sh, sw, ph, pw, out_pad, residual;
    int32_t n, h_in, w_in, h_out, w_out;
    int32_t lane;                /* 1: audio-encoder block (runs on the auxiliary stream beside the face encoder) */
    int32_t has_dx, has_dx_add, has_du, has_wgrad;
    /* the weight-gradient op (zero when has_wgrad == 0): wgrad_kernel<wg_bn> + the split-K reduction */
    int32_t wg_bn, wg_form, wg_ntaps, wg_tg, wg_ngroups;
    int32_t wg_p, wg_bw, wg_bh, wg_bnb;   /* pixels per K chunk = the box wg_bw x wg_bh x wg_bnb images */
    int32_t wg_chunks, wg_m_tiles, wg_n_tiles, wg_splits, wg_grid;
    /* the conv launches of the block's forward and of its input gradient (dgrad) */
    int32_t n_fwd, n_dgrad;
    w2l_kernel_info fwd[4], dgrad[4];
} w2l_train_block_info;
/* The blocks of the last training plan of `net` in forward order; net = -1: the block of the last w2l_conv_block_train.
 * Returns the number of entries written (at most cap), or a negative W2L_E* code; out == NULL returns the count. */
int w2l_debug_train_blocks(w2l_ctx* ctx, int net, int cap, w2l_train_block_info* out);

/* One tape tensor of block `block` (forward order) of the last training plan of `net`, as fp32 NCHW with exactly the
 * stored 16-bit values: X input, Z pre-BatchNorm conv output, Y output, DY its gradient, DZ gradient of Z (of the conv
 * output), DU gradient of the residual branch, DX input gradient, DX_ADD the skip gradient added to it; STATS is the
 * batch statistics (n = 2: mean, invstd; c = cout; h = w = 1) in fp32.  *n,*c,*h,*w receive the dims (any may be NULL);
 * out_dev == NULL only queries them.  A tensor the block does not have is W2L_EINVAL. */
#define W2L_TAPE_X      0
#define W2L_TAPE_Z      1
#define W2L_TAPE_Y      2
#define W2L_TAPE_DY     3
#define W2L_TAPE_DZ     4
#define W2L_TAPE_DU     5
#define W2L_TAPE_DX     6
#define W2L_TAPE_DX_ADD 7
#define W2L_TAPE_STATS  8
int w2l_debug_train_tensor(w2l_ctx* ctx, int net, int block, int which, float* out_dev, int* n, int* c, int* h, int* w,
                           void* stream);

/* ---- instrumentation ---- */
/* kernels launched by this library since the context was created (all streams) */
int64_t w2l_launch_count(const w2l_ctx* ctx);
/* bytes of device memory the context holds: weights, inference and training plans, Adam moments, staging and scratch
 * buffers, mel tables — every block it has allocated and not yet released */
int64_t w2l_device_bytes(const w2l_ctx* ctx);
/* Time the conv kernels of the last-built plan of `net` individually: runs every launch `iters`
 * times with CUDA events on `stream`, the L2 flushed before each timed launch (cold cache, as in the step), and writes
 * per-launch mean milliseconds and flop counts.
 * Returns the number of launches written (<= cap). */
int w2l_profile_plan(w2l_ctx* ctx, int net, int iters, int cap, float* ms_out, double* flop_out,
                     char (*names_out)[64], void* stream);

#ifdef __cplusplus
}
#endif
#endif /* W2L_H_ */
