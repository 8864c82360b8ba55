/* iss_b200.h -- C ABI of libiss_b200.so: the H100 (sm_90a) implementation of
 * inaSpeechSegmenter's per-frame hot path.
 *
 * The reference (ina-foss/inaSpeechSegmenter) is pure Python and has no FFI;
 * its seams are Python call signatures.  Every entry point below names the
 * reference call it replaces (path:line relative to the reference tree).
 * Conventions:
 *   - plain C types only; all `d_*` pointers are DEVICE pointers owned by the
 *     caller (e.g. torch.Tensor.data_ptr()), `h_*` pointers are HOST pointers;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     calls are asynchronous on that stream unless stated otherwise;
 *   - return value: 0 = ISS_OK, negative = error; iss_last_error() returns a
 *     thread-local message for the last failing call on this thread;
 *   - handles are opaque; distinct contexts may be used concurrently from
 *     different host threads (the reference extracts features on a worker
 *     thread while the main thread runs the CNNs, segmenter.py:377-387);
 *   - there is NO CPU fallback anywhere behind this ABI.
 */
#ifndef ISS_B200_H
#define ISS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ISS_OK              0
#define ISS_ERR_INVALID    -1   /* bad argument */
#define ISS_ERR_CUDA       -2   /* a CUDA runtime call failed */
#define ISS_ERR_NOMEM      -3
#define ISS_ERR_UNSUPPORTED -4  /* e.g. layer type / shape the kernels do not cover */
#define ISS_ERR_STATE      -5   /* tables not uploaded, model not loaded, ... */

typedef struct iss_ctx iss_ctx;
typedef struct iss_cnn iss_cnn;
typedef struct iss_resnet iss_resnet;
typedef struct iss_mlp iss_mlp;

/* ---- library / context ------------------------------------------------- */

#define ISS_ABI_VERSION 9
int         iss_version(void);               /* == ISS_ABI_VERSION of the header the library was built from */
const char *iss_last_error(void);
/* Creates a context bound to CUDA device `device` (one per host thread that
 * issues work).  Fails with ISS_ERR_CUDA if the device is not compute
 * capability 10.x. */
int iss_ctx_create(int device, iss_ctx **out);
int iss_ctx_destroy(iss_ctx *ctx);
/* Number of kernels this library has launched in this process so far (all
 * contexts); bench.py reports the delta over its timed region. */
int64_t iss_launch_count(void);
/* GEMM engine used by the conv / dense layers of K2 and K5 (process-wide):
 * 0 = fp32 CUDA cores; 2 = 3xTF32 split on wgmma (tf32) for every layer with C, K and N
 * multiples of 32; 3 (default) = fp16 hi/lo split on wgmma (f16) for layers with C and N
 * multiples of 64, engine 2 for every other layer.  All are sm_90a code
 * paths of this library with fp32-class accuracy (<= 1e-5 on the softmax against the fp32
 * oracle); the default can be overridden with ISS_B200_GEMM=fp32|tc_ts|tc_f16. */
int iss_set_gemm_mode(int mode);
int iss_get_gemm_mode(void);

/* ---- K1: SIDEKIT log-mel + log-energy front-end -------------------------
 * Replaces mfcc(sig, get_mspec=True) as used by _media2feats
 * (inaSpeechSegmenter/sidekit_mfcc.py:278-352 via segmenter.py:53-58):
 * framing 400/160 (:240-263), per-frame pre-emphasis 0.97 (:266-275),
 * loge = log(sum y^2) before windowing (:226), Hann(400) (:223), 512-point
 * real FFT power (:232-233), 24-band mel filterbank (:118-197) and log (:334).
 * The dead DCT (:337) is not computed. */

#define ISS_PCM_F32 0   /* float32 samples in [-1, 1) (what soundfile returns, io.py:51) */
#define ISS_PCM_S16 1   /* int16 PCM; converted as s / 32768.0f, exactly what soundfile does */
/* WAV encodings only the resampler reads (ISS_ERR_INVALID everywhere else), with their float64 value: */
#define ISS_PCM_U8  2   /* unsigned 8-bit, (s - 128) / 128 */
#define ISS_PCM_S24 3   /* signed 24-bit, 3 bytes little-endian, packed; s / 2^23 */
#define ISS_PCM_S32 4   /* signed 32-bit, s / 2^31 */
#define ISS_PCM_F64 5   /* IEEE float64, as is */

#define ISS_FFT_FP32 0  /* single-precision FFT (fast) */
#define ISS_FFT_FP64 1  /* double-precision window + FFT, power rounded to f32: the
                           reference's own precision recipe (sidekit_mfcc.py:231-233) */

/* L = int((n - 400) / 160) + 1 frames, 0 if n < 400 (sidekit_mfcc.py:254). */
int64_t iss_sidekit_num_frames(int64_t n_samples);

/* Host-precomputed tables: fbank = trfbank(16000,512,100,8000,0,24)[0]
 * (float32 [24][257], sidekit_mfcc.py:332) and window = numpy.hanning(400)
 * (float64 [400], :223).  Must be called once per context before
 * iss_sidekit_features.  Synchronous. */
int iss_sidekit_upload_tables(iss_ctx *ctx, const float *h_fbank, const double *h_window);

/* d_pcm: n_samples samples (format pcm_format) in device memory.
 * d_mspec: float32 [L][24]; d_loge: float32 [L];
 * d_loge_stats: double[2] = { sum of finite loge, count of finite loge } --
 * the global reduction _energy_activity needs (segmenter.py:70); written by a
 * deterministic two-stage reduction (no atomics).  A time-shard passes a
 * pointer to its own first sample (frame f starts at sample 160*f); int16
 * input needs 2-byte and float input 4-byte alignment only. */
int iss_sidekit_features(iss_ctx *ctx, const void *d_pcm, int pcm_format, int64_t n_samples,
                         int fft_precision, float *d_mspec, float *d_loge,
                         double *d_loge_stats, void *stream);

/* The same for n_rec recordings in one launch (iss_sidekit_features is its n_rec = 1 case).
 * Recording r is h_pcm[r] (a DEVICE pointer held in a host array) with h_n_samples[r] samples,
 * all in one pcm_format; its L_r frames go to the mspec rows h_row_off[r] .. + L_r of d_mspec
 * ([rows][24]) and to d_loge[h_loge_off[r] .. + L_r], and its {sum, count} to
 * d_loge_stats[2r], [2r + 1].  Every recording is tiled from its own first frame, so its
 * mspec, loge and statistics are bit-identical to those of an iss_sidekit_features call on it. */
int iss_sidekit_features_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_samples,
                               int pcm_format, int fft_precision, float *d_mspec, const int64_t *h_row_off,
                               float *d_loge, const int64_t *h_loge_off, double *d_loge_stats, void *stream);

/* Stand-alone version of the {sum, count} reduction over a float32 loge array
 * (e.g. the all-gathered loge of a time-sharded recording): same summation
 * order as the fused reduction inside iss_sidekit_features, hence bit-identical
 * d_loge_stats for the same loge values. */
int iss_loge_stats(iss_ctx *ctx, const float *d_loge, int64_t L, double *d_loge_stats, void *stream);
/* iss_loge_stats on each of n_seq sequences of one buffer in one pass: sequence i is d_loge[h_loge_off[i] ..
 * + h_len[i]) (h_len[i] >= 1), its {sum, count} goes to d_loge_stats[2i ..].  Bit-identical to iss_loge_stats on
 * the sequence alone.  Live streams use it for the calibration prefixes of their energy thresholds. */
int iss_loge_stats_multi(iss_ctx *ctx, const float *d_loge, const int64_t *h_loge_off, const int64_t *h_len,
                         int n_seq, double *d_loge_stats, void *stream);

/* ---- K3: Viterbi smoothing ------------------------------------------------
 * Replaces viterbi_decoding(emission, transition) for the two ways the hot
 * path calls it (inaSpeechSegmenter/pyannote_viterbi.py:118-224; callers
 * segmenter.py:72 and :176).  Exact IEEE-double max-sum recursion in the
 * reference's evaluation order, first-max tie break, uniform prior log(1/K). */

/* Energy activity (segmenter.py:69-73 + viterbi_utils.py:29-42):
 *   thr   = (double)(float)(stats[0]/stats[1]) + log_ratio   (NaN if count == 0)
 *   raw_t = (double)loge[t] > thr
 *   E_t   = { raw_t ? h_emis[1] : h_emis[0],  raw_t ? h_emis[0] : h_emis[1] }
 *           with h_emis = { log(1-1e-10), log(1e-10) } computed by the host the
 *           way the reference does (numpy), A = h_trans (row-major [2][2],
 *           from->to), prior = log_prior = log(1/2).
 * d_states: uint8 [ceil(L / out_stride)] -- state of every out_stride-th frame
 * (the reference keeps [::2], segmenter.py:262).  d_work: scratch of at least
 * iss_viterbi_work_bytes(L, 1) bytes.
 * Tracks of >= 65536 frames are decoded chunk-parallel (16384-frame chunks: max-plus transfer
 * matrices -> entry scores -> concurrent true passes); iss_set_energy_viterbi_serial(1), or
 * ISS_B200_VITERBI=serial, forces the single serial chain (the checker of the GPU tests). */
int iss_set_energy_viterbi_serial(int serial);
int iss_energy_viterbi(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                       double log_ratio, const double *h_emis, const double *h_trans,
                       double log_prior, int out_stride, uint8_t *d_states, void *d_work,
                       void *stream);
/* One independent energy chain per recording, all in one launch: recording r is
 * d_loge[h_loge_off[r] .. h_loge_off[r+1]) thresholded with d_loge_stats[2r], [2r + 1]
 * (as iss_sidekit_features_multi writes them); its every out_stride-th state goes to
 * d_states[h_out_off[r] ..].  d_work: iss_viterbi_work_bytes(h_loge_off[n_rec], n_rec) bytes.
 * Each chain is decoded serially, so a recording of 4 * 16384 = 65536 frames or more
 * (which iss_energy_viterbi decodes chunk-parallel) is refused with ISS_ERR_INVALID. */
int iss_energy_viterbi_multi(iss_ctx *ctx, const float *d_loge, const int64_t *h_loge_off, int n_rec,
                             const double *d_loge_stats, double log_ratio, const double *h_emis,
                             const double *h_trans, double log_prior, int out_stride,
                             const int64_t *h_out_off, uint8_t *d_states, void *d_work, void *stream);

/* Batched decode of CNN posteriors (segmenter.py:167-178): for segment s the
 * rows d_probs[seg_off[s] .. seg_off[s+1]) (float32 [n][K], already carrying
 * the 0.5 override of :175) are turned into emissions log(p) (float32 log,
 * widened to double like numpy's promotion) and decoded independently with a
 * fresh uniform prior log_prior = log(1/K).  h_seg_off: n_seg+1 int64 host
 * offsets.  2 <= K <= 4.  d_states: uint8 [n]. */
int iss_viterbi_segments(iss_ctx *ctx, const float *d_probs, int K, const int64_t *h_seg_off,
                         int n_seg, const double *h_trans, double log_prior, uint8_t *d_states,
                         void *d_work, void *stream);
int64_t iss_viterbi_work_bytes(int64_t total_steps, int n_seg);

/* Online decoding of many Viterbi chains in one launch (live streams: inaspeechsegmenter_b200/stream.py).  Chain i
 * is h_chains[6i .. 6i+6) = {src, n, slot, pend, out, flags} (int64, host):
 *   - its n new steps are d_src entries src .. src+n: energy mode (h_emis != NULL, K == 2) thresholds loge against
 *     the threshold of iss_energy_viterbi from d_stats[2*slot ..]; CNN mode (h_emis == NULL) takes log(p) of the
 *     posterior rows d_src[(src+t)*K ..];
 *   - flags & ISS_ONLINE_START: the chain starts here (V = E + log_prior on its first step, pend must be 0);
 *     otherwise it continues from the scores d_scores[slot*4 .. +K) left by its previous call;
 *   - the back-pointers of its pend undecided steps are d_hist[slot*hist_cap ..]; the new steps' are appended
 *     (pend + n <= hist_cap);
 *   - every state up to the latest step at which the backtracks from all K end states meet is final; with
 *     flags & ISS_ONLINE_END the chain ends and all its states are final (backtrack from the first argmax).
 * The decided states (one byte each, oldest first) go to d_out[out ..], their count to d_ndec[i]; the history row
 * keeps only the still undecided steps.  Same arithmetic as iss_energy_viterbi / iss_viterbi_segments, so the
 * decided states of a chain are those of the offline decode of all its steps.  d_scores, d_hist and d_stats are
 * caller-owned and live across calls; d_work holds iss_viterbi_online_work_bytes(n_chain) bytes.  Sizes, checked
 * against every chain before the launch: d_src holds src_len steps (entries or rows), d_scores / d_hist / d_stats
 * n_slots slots, d_out out_len bytes (chain i needs out + pend + n of them). */
#define ISS_ONLINE_START 1
#define ISS_ONLINE_END   2
int iss_viterbi_online(iss_ctx *ctx, int K, int n_chain, const int64_t *h_chains, const float *d_src,
                       int64_t src_len, const double *d_stats, double log_ratio, const double *h_emis,
                       const double *h_trans, double log_prior, double *d_scores, uint8_t *d_hist, int64_t n_slots,
                       int64_t hist_cap, uint8_t *d_out, int64_t out_len, int64_t *d_ndec, void *d_work, void *stream);
int64_t iss_viterbi_online_work_bytes(int n_chain);

/* Partial chains of the energy Viterbi for a recording that is time-sharded across GPUs
 * (the whole-file chain of pyannote_viterbi.py:202-220 cut at rank boundaries):
 *  iss_energy_transfer: max-plus transfer matrix of this rank's L frames, h_matrix[j*2+i] = best
 *      score of ending in state j given the chain entered (before the first frame) in state i --
 *      two basis-vector forward chains, no back-pointers.  Synchronous.
 *  iss_energy_forward: the true forward pass over the L frames, from the sequence start
 *      (h_vin == NULL: V[0] = E[0] + log_prior) or continuing from the predecessor's outgoing
 *      scores h_vin[2]; stores back-pointers in d_work, returns the outgoing scores h_vout[2] and
 *      the composite back map h_backmap[x] = state just before the first frame given state x at
 *      the last frame.  Synchronous.
 *  iss_energy_emit: backtrack from end_state (-1: argmax of the outgoing scores of the preceding
 *      iss_energy_forward on the same d_work) and write every out_stride-th state.
 * d_work: iss_viterbi_work_bytes(L, 1) bytes, the same buffer for forward and emit. */
int iss_energy_transfer(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                        double log_ratio, const double *h_emis, const double *h_trans,
                        double *h_matrix, void *d_work, void *stream);
int iss_energy_forward(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                       double log_ratio, const double *h_emis, const double *h_trans, double log_prior,
                       const double *h_vin, double *h_vout, uint8_t *h_backmap, void *d_work, void *stream);
int iss_energy_emit(iss_ctx *ctx, int64_t L, int end_state, int out_stride, uint8_t *d_states,
                    void *d_work, void *stream);

/* ---- K2: patch z-normalisation + CNN forward ------------------------------
 * Replaces _get_patches (segmenter.py:76-88) + keras Model.predict
 * (segmenter.py:131-133,163) + the non-finite override (:175). */

#define ISS_LAYER_CONV2D  1
#define ISS_LAYER_DENSE   2
#define ISS_LAYER_MAXPOOL 3

#define ISS_F_BIAS        1   /* + bias[cout] */
#define ISS_F_AFFINE_PRE  2   /* then  x*pre_scale[c] + pre_shift[c]   (BatchNorm before the activation) */
#define ISS_F_RELU        4   /* then  max(x, 0) */
#define ISS_F_AFFINE_POST 8   /* then  x*post_scale[c] + post_shift[c] (BatchNorm after the activation) */
#define ISS_F_SOFTMAX     16  /* softmax over cout (last layer only) */
#define ISS_F_SIGMOID     32

typedef struct iss_layer_desc {
    int32_t kind;                 /* ISS_LAYER_* */
    int32_t kh, kw;               /* kernel / pool window (rows = time, cols = mel band) */
    int32_t sh, sw;               /* strides */
    int32_t pad_top, pad_left, pad_bottom, pad_right;  /* zero (conv) / -inf (pool) padding */
    int32_t cin, cout;            /* DENSE: cin = flattened (H*W*C, Keras channels_last order) */
    int32_t flags;                /* ISS_F_* */
    int64_t w_off;                /* float offsets into the weight blob; -1 when unused.     */
    int64_t bias_off;             /* CONV2D kernel is [kh][kw][cin][cout] (Keras layout),     */
    int64_t pre_scale_off, pre_shift_off;    /* DENSE kernel is [cin][cout].                */
    int64_t post_scale_off, post_shift_off;
} iss_layer_desc;

/* Builds a model for input patches of in_h x in_w x 1 (68 x nmel).  The blob is
 * copied to the device.  Synchronous. */
int iss_cnn_create(iss_ctx *ctx, const iss_layer_desc *layers, int n_layers,
                   const float *h_blob, int64_t blob_len, int in_h, int in_w, iss_cnn **out);
int iss_cnn_destroy(iss_cnn *cnn);
int iss_cnn_num_classes(const iss_cnn *cnn);
double iss_cnn_flops_per_patch(const iss_cnn *cnn);     /* 2 * MACs of all conv/dense layers */
/* scratch needed by iss_cnn_forward for `n` patches in `n_seg` index ranges
 * (activations ping-pong, patch statistics, index map). */
int64_t iss_cnn_workspace_bytes(const iss_cnn *cnn, int64_t n, int n_seg);

/* d_mspec: float32 [L][ld] log-mel rows (ld = 24; the first in_w bands are
 * used, segmenter.py:146-147).  Patch p (0 <= p < ceil(L/2)) is frames
 * 2*clamp(p-17, 0, U-1) .. +67 with U = (L-68)/2+1 un-replicated windows
 * (edge replication of segmenter.py:83-85); edge_left/edge_right = 0 disable
 * the replication on that side for a time-shard that is not at a file end
 * (then patch p is frames 2p .. 2p+67 and p < U).
 * The patches evaluated are those of the index ranges
 * [h_seg_start[s], h_seg_stop[s]) concatenated (segmenter.py:156-162).
 * d_probs: float32 [n][K] softmax, rows of non-finite patches forced to 0.5
 * (segmenter.py:175).  n = sum of range lengths. */
int iss_cnn_forward(iss_ctx *ctx, iss_cnn *cnn, const float *d_mspec, int64_t L, int ld,
                    int edge_left, int edge_right,
                    const int32_t *h_seg_start, const int32_t *h_seg_stop, int n_seg,
                    float *d_probs, void *d_work, int64_t work_bytes, void *stream);

/* The same over n_rec recordings packed in one d_mspec of `rows` rows (iss_cnn_forward is its
 * one-recording case): recording r is rows h_row_off[r] .. + h_len[r] (h_len[r] >= 68, short
 * recordings padded first), with edge replication at both of its ends; range s is the padded
 * patches [h_seg_start[s], h_seg_stop[s]) of recording h_seg_rec[s], so patch p of recording r
 * is rows h_row_off[r] + 2*clamp(p-17, 0, U_r-1) .. +67.  A patch's posteriors do not depend on
 * the other patches of the call. */
int iss_cnn_forward_multi(iss_ctx *ctx, iss_cnn *cnn, const float *d_mspec, int64_t rows, int ld,
                          const int64_t *h_row_off, const int64_t *h_len, int n_rec,
                          const int32_t *h_seg_rec, const int32_t *h_seg_start, const int32_t *h_seg_stop, int n_seg,
                          float *d_probs, void *d_work, int64_t work_bytes, void *stream);

/* ---- K4: VBx / HTK 64-band log-mel front-end + floating CMVN ----------------
 * Replaces get_features(signal) (inaSpeechSegmenter/vbx_segmenter.py:72-89 on top
 * of features_vbx.py:62-148): trunc(signal*2^15) + dither, mirror pad 120/200,
 * frames 400/160, per-frame mean removal + pre-emphasis, Povey window, 512-point
 * power spectrum, log(max(1, . fbank)), cmvn_floating_kaldi(150, 149), float32. */

/* M = (n + 320 - 400) / 160 + 1 feature frames (0 if n < 200). */
int64_t iss_vbx_num_frames(int64_t n_samples);
/* h_fbank = mel_fbank_mx(400, 16000, NUMCHANS=64, LOFREQ=20, HIFREQ=7600,
 * htk_bug=False) (float64 [257][64]); h_window = povey_window(400) (float64). */
int iss_vbx_upload_tables(iss_ctx *ctx, const double *h_fbank, const double *h_window);
int64_t iss_vbx_work_bytes(int64_t n_samples);
/* d_dither: float64 [n] = 8*(2u-1), u the np.random.seed(3); np.random.rand(n)
 * stream (a prefix of one fixed MT19937 sequence -- keep it resident), or NULL for
 * no dither.  d_fea: float32 [M][64].  d_work: iss_vbx_work_bytes(n) of scratch. */
int iss_vbx_features(iss_ctx *ctx, const void *d_pcm, int pcm_format, int64_t n_samples,
                     const double *d_dither, float *d_fea, void *d_work, void *stream);
/* The same for n_rec recordings in one pair of launches (iss_vbx_features is its n_rec = 1 case).
 * Recording r is h_pcm[r] (a DEVICE pointer held in a host array) with h_n_samples[r] samples, all
 * in one pcm_format; its M_r = iss_vbx_num_frames(h_n_samples[r]) rows go to d_fea rows
 * h_fea_off[r] .. + M_r.  Every recording is padded, dithered (d_dither[0 ..] again for each one,
 * as the reference reseeds per get_features call), tiled and CMVN-windowed on its own, so its rows
 * are bit-identical to those of an iss_vbx_features call on it.  Recordings under 200 samples get
 * no rows.  d_work: 8 * 64 * sum(M_r) + 256 bytes of scratch. */
int iss_vbx_features_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_samples,
                           int pcm_format, const double *d_dither, float *d_fea, const int64_t *h_fea_off,
                           void *d_work, void *stream);
/* The same front end over windows of streams fed piece by piece (live streams), in two steps that run the kernels of
 * iss_vbx_features_multi (which is the window s_base = r_first = r_base = t_first = 0 with ISS_VBX_END of each
 * recording), so every row equals, bit for bit, the same row of iss_vbx_features on the whole stream.
 * Raw rows (float64 log-fbank before CMVN), n_rec records of one pcm_format in one launch: record r is the int64 row
 * h_win[6 r ..] = {s_base, s_known, r_first, rows, raw_off, flags}.  h_pcm[r] and h_dither[r] (DEVICE pointers, the
 * dither as d_dither above, or NULL for none) hold samples [s_base, s_known) of the stream; raw rows r_first ..
 * r_first + rows - 1 go to d_raw rows raw_off ...  Row t reads samples max(0, 160 t - 120) .. 160 t + 279 and is final
 * once 160 t + 280 <= s_known; the mirrored rows past that read around s_known, the stream's last sample, and are
 * allowed only once it has ended (ISS_VBX_END).  Checked on the host before the launch, ISS_ERR_INVALID with the
 * record's index: no row reads a sample before s_base; without ISS_VBX_END no row reads a sample at or past s_known;
 * with it, rows < iss_vbx_num_frames(s_known). */
#define ISS_VBX_END 1
int iss_vbx_fbank_window_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const double *const *h_dither,
                               const int64_t *h_win, int pcm_format, double *d_raw, void *stream);
/* CMVN rows, n_rec records in one launch: record r is h_win[7 r ..] = {r_base, r_known, t_first, rows, raw_off,
 * fea_off, flags}: d_raw rows raw_off .. hold raw rows [r_base, r_known) of the stream; feature rows t_first ..
 * t_first + rows - 1 go to d_fea rows fea_off ...  r_known is the M of the sliding window.  Each row is computed by
 * replaying its 128-row chunk of the whole-recording grid from the chunk's start, so it is the same sum in the same
 * order.  Checked on the host: rows < r_known; without ISS_VBX_END, r_known >= 300 and t_first + rows - 1 + 150 <=
 * r_known (rows whose window can no longer change); the window start of the chunk of t_first is >= r_base. */
int iss_vbx_cmvn_window_multi(iss_ctx *ctx, int n_rec, const int64_t *h_win, const double *d_raw, float *d_fea,
                              void *stream);
/* The dither of d_dither above, drawn on the device for many streams, each from its own MT19937 state, in one launch.
 * d_state: uint32 [n_slots][625], row s = the 624 key words and the position of numpy's RandomState(3).get_state()
 * when stream slot s opens; record r = h_rec[3 r ..] = {slot, n, out_off} writes the slot's next n dither values to
 * d_out[out_off ..] and advances its state, so a stream's values concatenate to 8 * (2 RandomState(3).rand(N) - 1).
 * A state position that is odd or past 624 is read as 624 (the next draw twists first).  ISS_ERR_INVALID (host check,
 * no launch) for a slot out of range or drawn twice in one call, or n_slots >= 2^31. */
int iss_dither_mt19937_multi(iss_ctx *ctx, int n_rec, const int64_t *h_rec, uint32_t *d_state, int64_t n_slots,
                             double *d_out, void *stream);

/* ---- Resampling to 16 kHz mono -----------------------------------------------
 * No reference counterpart: the reference has ffmpeg decode with `-ar 16000 -ac 1`
 * (io.py:37-55).  This is NOT ffmpeg's resampler.  A recording of n frames of C
 * interleaved channels at integer rate R (8000 <= R <= 192000, 1 <= C <= 8, samples of
 * any ISS_PCM_* format laid out [frames][channels]) becomes int16 16 kHz mono PCM:
 *   x[m]   = mean of the C samples of frame m in float64 (each as its format's value:
 *            int16 s as s / 32768.0, float32 as is, the WAV encodings as listed above),
 *   y      = scipy.signal.resample_poly(x, up, down) with up = 16000 / g, down = R / g,
 *            g = gcd(16000, R) (scipy's default Kaiser(5.0) design, zero padding),
 *   out[k] = clip(rint(y[k] * 32768), -32768, 32767)  (round half to even),
 * k < ceil(n * up / down).  Each output is one float64 dot product in a fixed tap
 * order, so every recording's output is the same in any call. */

/* ceil(n_frames * up / down); -1 for a rate outside [8000, 192000] or n_frames < 0. */
int64_t iss_resample_num_frames(int64_t n_frames, int rate);
/* h_taps: the float64 prototype filter of rate `rate`, scipy.signal.firwin(2H + 1,
 * 1 / max(up, down), window=('kaiser', 5.0)) * up with H = 10 max(up, down) (n_taps =
 * 2H + 1; the single tap {1.0} when up == down == 1).  Arranged by phase and kept on
 * the device by the context until iss_resample_release_taps or iss_ctx_destroy; an
 * upload for a rate that has taps replaces them.  Synchronous. */
int iss_resample_upload_taps(iss_ctx *ctx, int rate, const double *h_taps, int64_t n_taps);
int iss_resample_release_taps(iss_ctx *ctx, int rate);
/* Resamples n_rec recordings of one (rate, channels, pcm_format) in one launch.  Recording
 * r is h_pcm[r] (a DEVICE pointer held in a host array) with h_n_frames[r] frames; its
 * iss_resample_num_frames(h_n_frames[r], rate) int16 outputs go to d_out[h_out_off[r] ..].
 * Any pointer alignment of the sample type works (16-byte aligned recordings are read
 * with vector loads; packed 24-bit recordings at any byte address).  No load reads a byte
 * outside a recording's frames.  ISS_ERR_STATE if no taps were uploaded for `rate`. */
int iss_resample_to16k_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_frames,
                             int channels, int rate, int pcm_format, int16_t *d_out, const int64_t *h_out_off,
                             void *stream);
/* The same resampling over windows of streams fed piece by piece (live streams), n_rec
 * records of one (rate, channels, pcm_format) in one launch.  Record r is the int64 row
 * h_win[6 r ..] = {f_base, n_known, k_first, n_out, out_off, flags}: h_pcm[r] (a DEVICE
 * pointer) holds frames [f_base, n_known) of its stream, and outputs k_first ..
 * k_first + n_out - 1 of the stream go to d_out[out_off ..].  Frames at or past n_known
 * read as zero, which is the definition's padding only once the stream has ended
 * (flags ISS_RESAMPLE_END).  Every output equals, bit for bit, the same output of
 * iss_resample_to16k_multi on the whole stream.  Output k reads frames a + s_q ..
 * a + s_q + n_q - 1 (k down = a up + q, the phase table of iss_resample_upload_taps).
 * Checked on the host before the launch, ISS_ERR_INVALID with the record's index: no
 * output reads a frame in [0, f_base); without ISS_RESAMPLE_END no output reads a frame at
 * or past n_known; k_first + n_out <= iss_resample_num_frames(n_known, rate). */
#define ISS_RESAMPLE_END 1
int iss_resample_window_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_win,
                              int channels, int rate, int pcm_format, int16_t *d_out, void *stream);

/* ---- K5: ResNet101 x-vector extractor ----------------------------------------
 * Replaces VBxExtractor.get_embedding / OnnxBackendExtractor (vbx_segmenter.py:
 * 249-266) == ResNet.forward (resnet.py:115-130), batched over the windows of
 * VBxExtractor.__call__ (vbx_segmenter.py:217-246).
 * Blob layout (float32), in module order conv1, layer1.0 ... layer4.2, each
 * Bottleneck as conv1, conv2, conv3[, shortcut]; every convolution contributes
 * kernel [kh][kw][cin][cout], then BatchNorm folded to scale[cout], shift[cout];
 * finally embedding weight transposed [2*C*H][embed] and bias [embed]. */
int64_t iss_resnet_blob_len(int m_channels, int feat_dim, int embed_dim, const int *num_blocks);
int iss_resnet_create(iss_ctx *ctx, const float *h_blob, int64_t blob_len, int m_channels, int feat_dim,
                      int embed_dim, const int *num_blocks, iss_resnet **out);
int iss_resnet_destroy(iss_resnet *net);
double iss_resnet_flops_per_window(const iss_resnet *net, int win_len);
int64_t iss_resnet_workspace_bytes(const iss_resnet *net, int n_windows, int win_len);
/* d_fea: float32 [M][feat_dim] (CMVN'd features); window i = rows
 * [h_win_start[i], h_win_start[i] + win_len); d_emb: float32 [n_windows][embed]. */
int iss_resnet_embed(iss_ctx *ctx, iss_resnet *net, const float *d_fea, int64_t M,
                     const int32_t *h_win_start, int n_windows, int win_len, float *d_emb,
                     void *d_work, int64_t work_bytes, void *stream);

/* ---- Dense stack applied to x-vectors ------------------------------------------------
 * Replaces gender_detection_mlp_model.predict(x) of VoiceFemininityScoring
 * (inaSpeechSegmenter/vbx_segmenter.py:116-124,188-191).  layers: ISS_LAYER_DENSE records
 * only (flags as for the CNN head, ISS_F_SIGMOID supported, no softmax). */
int iss_mlp_create(iss_ctx *ctx, const iss_layer_desc *layers, int n_layers, const float *h_blob,
                   int64_t blob_len, int in_dim, iss_mlp **out);
int iss_mlp_destroy(iss_mlp *mlp);
int iss_mlp_out_dim(const iss_mlp *mlp);
int64_t iss_mlp_workspace_bytes(const iss_mlp *mlp, int64_t n_rows);
/* d_x: float32 [n_rows][in_dim]; d_y: float32 [n_rows][out_dim].  d_x, d_y and d_work must be
 * 16-byte aligned (ISS_ERR_INVALID otherwise). */
int iss_mlp_forward(iss_ctx *ctx, iss_mlp *mlp, const float *d_x, int64_t n_rows, float *d_y,
                    void *d_work, int64_t work_bytes, void *stream);

/* Live roofline support: record CUDA events around every launch of layer
 * `layer` (index into the iss_layer_desc list; -1 switches profiling off) on
 * the stream the launch uses.  iss_cnn_profile_read synchronises those events,
 * returns the summed device time (ms), the number of launches and the FLOPs
 * those launches performed, and resets the accumulators. */
int iss_cnn_profile(iss_cnn *cnn, int layer);
int iss_cnn_profile_read(iss_cnn *cnn, double *total_ms, int64_t *launches, double *flops);
/* FLOPs of one layer for one patch (2 * MACs); 0 for pooling. */
double iss_cnn_layer_flops(const iss_cnn *cnn, int layer);
int iss_cnn_num_layers(const iss_cnn *cnn);
/* Input rows that one 128-row tile of the gather convolution kernel reads at most
 * (rows of the batch as one tall image), over every tile start: the size of
 * its shared-memory halo for a layer of input height H, output OH x OW, KH
 * filter rows, row stride SH and top padding PT. */
int iss_gather_halo_rows_bound(int H, int OH, int OW, int KH, int SH, int PT);
/* Shared memory (bytes) of the gather convolution kernel with that halo for an
 * fp16-split layer with a 2x2 max-pooling folded in, C -> N channels, pooled
 * input width W and a KH x KW filter; 0 when the layer keeps the global-memory
 * operand fill (C != 64, one tap, or the halo does not fit in shared memory). */
int iss_gather_halo_smem(int H, int W, int OH, int OW, int KH, int KW, int SH, int PT, int C, int N);
/* Shared memory (bytes) of the pipelined form of that layer: two such halos,
 * restaged as hi / lo planes, next to a three-stage weight ring, so that the
 * halo of the next tile is staged while the tensor cores work on this one; 0
 * when the layer keeps the single halo or the global-memory fill. */
int iss_gather_pipe_smem(int H, int W, int OH, int OW, int KH, int KW, int SH, int PT, int C, int N);

#ifdef __cplusplus
}
#endif
#endif /* ISS_B200_H */
