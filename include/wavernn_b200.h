/* wavernn_b200.h -- C ABI of the Hopper-native (sm_90a) WaveRNN generate() engine.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference (fatchord/WaveRNN) has no
 * native interface of its own: its hot path is the Python loop
 *     models/fatchord_version.py:201-241   (per-sample: I, rnn1, rnn2, fc1, fc2, fc3)
 *     utils/distribution.py:87-123         (MoL sampling)      /  :231-237 (RAW softmax head)
 * run between `self.upsample(...)` (:186) and the numpy epilogue (:243).  These entry
 * points are what a Python/ctypes (or any FFI) binding of that span binds; the
 * reference-side stub is shown in INTEGRATION.md and implemented in
 * wavernn_b200/cabi.py.
 *
 * Conventions: plain C types only; every function returns 0 on success or a negative
 * WRNN_E_* code and never throws; `wrnn_last_error()` gives a thread-local message.
 * The caller owns every buffer it passes; a handle owns only its packed weights and
 * scratch.  One handle per device; one generate in flight per handle.  All device
 * work is enqueued on the given stream; no host synchronisation inside
 * `wrnn_generate` (errors detected on the device -- e.g. a watchdog abort -- are
 * reported by `wrnn_check`, to be called after the stream has been synchronised).
 */
#ifndef WAVERNN_B200_H_
#define WAVERNN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WRNN_ABI_VERSION 5

enum {
  WRNN_OK = 0,
  WRNN_E_INVALID = -1,      /* bad argument / unsupported configuration            */
  WRNN_E_CUDA = -2,         /* a CUDA runtime call failed (see wrnn_last_error)     */
  WRNN_E_NO_DEVICE = -3,    /* no sm_90 device: there is NO CPU fallback            */
  WRNN_E_WATCHDOG = -4,     /* the persistent kernel aborted on its spin watchdog   */
  WRNN_E_BUSY = -5
};

enum { WRNN_MODE_MOL = 0, WRNN_MODE_RAW = 1 };   /* fatchord_version.py:98-104 */

/* Arithmetic of the dense contractions.
 *   F16 : weights and activations rounded (RNE, saturating) to IEEE fp16 as tensor-core
 *         operands, fp32 accumulate; state, gates and sampler fp32.  The product path:
 *         same tensor throughput as bf16 with 8x finer operand rounding (all operands of
 *         this network are O(1)..O(100), far inside fp16 range).
 *   BF16: as F16 with bfloat16 operands.
 *   FP32: strict mode -- fp32 weights/activations on CUDA cores; a debugging and
 *         parity tool (matches the reference to reassociation error).               */
enum { WRNN_PREC_F16 = 0, WRNN_PREC_FP32 = 1, WRNN_PREC_BF16 = 2 };

/* Which kernel family executes the job.  AUTO picks the fastest that supports it:
 *   TCGEN05: weights stationary in the shared memory of 128 SMs, activations exchanged through L2 -- lowest latency
 *            per step, tiles of <= 64 folds one after the other (BASELINE configs[1], [2]);
 *   STREAM : activations stationary (one CTA per 16/32 folds, any number of CTAs), weights streamed from L2 every
 *            step -- highest throughput for jobs with hundreds of folds (configs[3], [4]); MoL head;
 *   SIMT   : CUDA-core engine, the only one with strict fp32 arithmetic.                                       */
enum { WRNN_ENGINE_AUTO = 0, WRNN_ENGINE_SIMT = 1, WRNN_ENGINE_TCGEN05 = 2, WRNN_ENGINE_STREAM = 3 };

/* Where frame-rate conditioning (wrnn_job::mel_frames) is turned into per-sample rows. */
enum { WRNN_COND_AUTO = 0, WRNN_COND_EXPAND = 1, WRNN_COND_IN_KERNEL = 2 };

typedef struct wrnn_handle wrnn_t;

/* Mirrors the WaveRNN ctor arguments that size the hot path
 * (fatchord_version.py:93-123; hparams.py:44-50).                                  */
typedef struct {
  int32_t rnn_dims;     /* 512 */
  int32_t fc_dims;      /* 512 */
  int32_t feat_dims;    /* 80  */
  int32_t aux_dims;     /* res_out_dims / 4 = 32 */
  int32_t n_classes;    /* 30 (MOL) or 2**bits (RAW) */
  int32_t mode;         /* WRNN_MODE_* */
  int32_t precision;    /* WRNN_PREC_* */
  int32_t engine;       /* WRNN_ENGINE_* */
} wrnn_cfg;

/* The 16 hot-path tensors exactly as they sit in the reference state_dict
 * (fp32, row-major [out, in]); host or device pointers (resolved with UVA).
 *   I.weight (rnn, 1+feat+aux)            col 0 = previous sample, 1..feat = mel, rest = aux[0:d]
 *   rnn1.weight_ih_l0 (3*rnn, rnn)        gate rows [r, z, n]   (fatchord_version.py:273-279)
 *   rnn2.weight_ih_l0 (3*rnn, rnn+aux)    cols rnn.. = aux[d:2d]
 *   fc1.weight (fc, rnn+aux)              cols rnn.. = aux[2d:3d]
 *   fc2.weight (fc, fc+aux)               cols fc..  = aux[3d:4d]
 *   fc3.weight (n_classes, fc)                                                     */
typedef struct {
  const float *I_weight, *I_bias;
  const float *rnn1_weight_ih, *rnn1_weight_hh, *rnn1_bias_ih, *rnn1_bias_hh;
  const float *rnn2_weight_ih, *rnn2_weight_hh, *rnn2_bias_ih, *rnn2_bias_hh;
  const float *fc1_weight, *fc1_bias, *fc2_weight, *fc2_bias, *fc3_weight, *fc3_bias;
} wrnn_weights;

/* One generate call == the loop fatchord_version.py:194-241 over `n_seg` folds.
 * Folds are strided windows of the UN-folded conditioning stream: fold b, step t
 * reads row  b*seg_stride + t  of mels_up / aux; rows >= L read as zeros, which is
 * what fold_with_overlap's right padding produces (fatchord_version.py:319-338).
 * Unbatched generation is n_seg = 1, seg_len = L.                                  */
typedef struct {
  const float *mels_up;   /* device, [L, feat_dims]                                  */
  const float *aux;       /* device, [L, 4*aux_dims]                                 */
  int64_t L;
  int64_t seg_stride;     /* target + overlap                                        */
  int32_t n_seg;          /* folds handled by this call (this rank)                  */
  int32_t seg_len;        /* target + 2*overlap == steps per fold                    */
  int32_t seg_first;      /* global index of fold 0 (keys the in-kernel Philox)      */
  int32_t steps;          /* 0 = seg_len; otherwise generate only the first `steps`  */
  /* Randomness.  Parity mode: the caller supplies the draws the reference would have
   * made from torch's generator (utils/distribution.py:106,118):
   *   uniforms [seg_len, 11*n_seg], row t = [n_seg*10 mixture draws, fold-major |
   *   n_seg logistic draws], values in [1e-5, 1-1e-5].
   *   expo     [seg_len, n_seg, n_classes] Exp(1) draws (RAW head: Categorical.sample()
   *   == argmax(p / e), fatchord_version.py:233-235).
   * NULL selects the in-kernel counter-based Philox4x32-10 keyed by
   * (philox_seed, philox_offset, global fold, step).                               */
  const float *uniforms;
  const float *expo;
  uint64_t philox_seed;
  uint64_t philox_offset;
  float *out;             /* device, [n_seg, seg_len] generated samples (pre-xfade)  */
  /* Instrumentation (NULL when unused) */
  const float *x_force;   /* [seg_len, n_seg] teacher forcing: step t consumes
                             x_force[t-1] instead of its own previous sample        */
  float *logits_out;      /* [seg_len, n_seg, n_classes] fc3 outputs per step        */
  /* Optional fold tables (device, [n_seg] int64 each; NULL = the strided windows above).
   * fold b, step t reads conditioning row  fold_row0[b] + t ; rows >= fold_row_end[b] read as zeros.
   * Lets one job carry the folds of SEVERAL utterances laid end to end in mels_up / aux
   * (WaveRNN.generate_many; the reference vocodes sentences one at a time, gen_tacotron.py:139-163). */
  const int64_t *fold_row0;
  const int64_t *fold_row_end;
  /* Optional frame-rate conditioning (device; tensor-core engines).  When mel_frames != NULL the library builds the
   * conditioning rows itself and mels_up / aux are ignored (may be NULL; L stays the stream length in samples):
   *   aux row n  = aux_frames[n / hop]                      (Stretch2d is a nearest-neighbour repeat, :57-61)
   *   mel row n  = sum_{d<5} up_taps[n % hop][d] * mel_frames[n / hop + d]
   * mel_frames [T + 2*pad, feat] is the zero-padded mel, aux_frames [T, 4*aux] the MelResNet output, and
   * up_taps [hop, 5] the composed impulse response of the three stretch+conv stages of UpsampleNetwork
   * (fatchord_version.py:73-88), exact for every output sample that survives the `indent` crop.
   * The frame tensors always describe the WHOLE stream: without fold tables, fold b reads rows
   * (seg_first + b)*seg_stride + t  (so a rank's shard passes the same tensors and its seg_first).
   * cond_mode picks where the rows are formed (same arithmetic, bit-identical samples):
   *   WRNN_COND_AUTO     : EXPAND when the job has no fold tables, else IN_KERNEL
   *   WRNN_COND_EXPAND   : an HBM-rate pre-pass writes each 64-fold tile's rows to engine scratch
   *                        (<= 64*seg_stride*832 B) just before that tile's persistent launch
   *   WRNN_COND_IN_KERNEL: the persistent kernel's staging warps form the rows step by step (no scratch) */
  const float *mel_frames;
  const float *aux_frames;
  const float *up_taps;
  int32_t hop;
  int32_t cond_mode;
  /* Optional (MoL parity mode, tensor-core engines): `uniforms` may still be in flight when the job is enqueued.
   * *uniforms_ready (device, uint32) = number of leading rows of `uniforms` that are valid; the kernel consumes row t at
   * step t and waits (bounded by the watchdog) until rows t .. min(t+3, steps-1) are valid (a margin that keeps its
   * cached loads from ever touching a line that is still in flight).  The caller uploads the draws in step
   * chunks on another stream and bumps the counter after each chunk (a 4-byte copy on that same stream), so the
   * host-side replay of torch's generator overlaps the kernel instead of preceding it.  NULL: all rows are valid.  */
  const uint32_t *uniforms_ready;
} wrnn_job;

int wrnn_abi_version(void);
const char *wrnn_last_error(void);

/* Packs the weights for the chosen engine on `device` (bf16 tiles + folded
 * conditioning matrices) and allocates per-handle scratch.                         */
int wrnn_create(wrnn_t **out, const wrnn_cfg *cfg, const wrnn_weights *w, int device);
void wrnn_destroy(wrnn_t *h);

/* Enqueues the persistent kernel on `stream` (a cudaStream_t; NULL = default).     */
int wrnn_generate(wrnn_t *h, const wrnn_job *job, void *stream);

/* After the stream has been synchronised: 0, or WRNN_E_WATCHDOG / WRNN_E_CUDA if the
 * last job aborted on the device.                                                  */
int wrnn_check(wrnn_t *h);

/* Convenience for non-torch callers: same job but mels_up / aux / uniforms / expo /
 * out / x_force / logits_out are HOST pointers; copies in, runs, copies out and
 * synchronises.                                                                    */
int wrnn_generate_host(wrnn_t *h, const wrnn_job *job);

/* Introspection: name of the engine serving the handle ("simt", "tcgen05"), number
 * of CTAs of the persistent grid, and kernel launches issued so far.               */
const char *wrnn_engine_name(const wrnn_t *h);
int wrnn_grid_ctas(const wrnn_t *h);
int64_t wrnn_launch_count(const wrnn_t *h);

/* The conditioning pre-pass on its own (what WRNN_COND_EXPAND runs per tile): rows [row_lo, row_lo + n_rows) of the
 * per-sample stream -- mels_up [n_rows, feat], aux [n_rows, 4*aux] -- from the frame-rate tensors of wrnn_job
 * (same arithmetic, so the rows are bit-identical to the ones a frame-rate job forms internally).  All DEVICE
 * pointers; asynchronous on `stream`.  mel_frames must hold frames up to (row_lo + n_rows - 1) / hop + 4.
 * Used by WaveRNN.generate_many to lay several utterances end to end for one job with fold tables.           */
int wrnn_expand_conditioning(const float *mel_frames, const float *aux_frames, const float *up_taps, int32_t hop,
                             int64_t row_lo, int64_t n_rows, float *mels_up, float *aux, void *stream);

/* The tail of generate() on the device (fatchord_version.py:243-258, :342-405; utils/dsp.py:98-103): float64
 * mu-law expansion, cross-fade + overlap-add of the folds, final fade-out -- one HBM-bound pass, asynchronous on
 * `stream`.  All pointers are DEVICE pointers.
 *   samples [n_seg, seg_len] fp32 as written by wrnn_generate (after the all-gather on multi-GPU jobs)
 *   fade_in / fade_out [overlap] float64: the windows of xfade_and_unfold (:385-391); NULL with overlap = 0 (unbatched)
 *   mu_table [n_classes] float64 or NULL: expansion of label k (RAW head with mu_law)
 *   tail [tail_len] float64 or NULL: linspace(1, 0, 20*hop) applied to the last tail_len samples (:255-258)
 *   wav [wave_len] float64
 * The tables are built by the caller with the reference's own numpy expressions, so the result is bit-identical
 * to the host epilogue (multiplications and additions in the reference's order, folds ascending).            */
int wrnn_epilogue(const float *samples, int32_t n_seg, int32_t seg_len, int64_t seg_stride, int32_t overlap,
                  const double *fade_in, const double *fade_out, const double *mu_table, int32_t n_classes,
                  const double *tail, int64_t tail_len, int64_t wave_len, double *wav, void *stream);

/* Host helper for parity mode: replays torch's default CPU generator (MT19937) natively, so the
 * draws the reference makes before / inside its loop cost a few ms instead of ~30.
 *   state : the generator's 624 words and its position `pos` in [0, 624] (624 = block exhausted)
 *   skip  : outputs to discard first -- the reference builds two nn.GRUCell per generate() call
 *           (fatchord_version.py:178-179 via :266-271), whose reset_parameters() draws one value
 *           per parameter element
 *   out   : n floats  lo + u24 * 2^-24 * (hi - lo), u24 = low 24 bits of each tempered output --
 *           torch's CPU uniform_() for float32 (utils/distribution.py:106,118 via torch.rand_like
 *           on a CPU tensor).  out may be NULL with n = 0 (skip only).
 * Returns the new position; `state` is updated in place.                               */
int32_t wrnn_mt19937_uniform(uint32_t *state, int32_t pos, uint64_t skip, float *out, uint64_t n,
                             float lo, float hi);
/* Same stream, but the n_rows x row_len draws that follow `skip` are a matrix of which only the columns
 * [a_lo, a_hi) and [b_lo, b_hi) (a_hi <= b_lo) are wanted: `out` is [n_rows, (a_hi-a_lo) + (b_hi-b_lo)], the other
 * draws are discarded without being converted.  A rank of a sharded job needs only its own folds' columns of the
 * reference's [steps, 11*B] draw matrix (10*B mixture draws fold-major, then B logistic draws per row).        */
int32_t wrnn_mt19937_uniform_cols(uint32_t *state, int32_t pos, uint64_t skip, float *out, uint64_t n_rows,
                                  uint64_t row_len, uint64_t a_lo, uint64_t a_hi, uint64_t b_lo, uint64_t b_hi,
                                  float lo, float hi);

#ifdef __cplusplus
}
#endif
#endif /* WAVERNN_B200_H_ */
