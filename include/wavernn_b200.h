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
 *            step -- highest throughput for jobs with hundreds of folds (configs[3], [4]); MoL head (30 classes) and
 *            9-bit RAW head (512 classes); AUTO routes only MoL jobs here;
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
 * synchronises.  It takes per-sample conditioning rows; a caller holding a mel
 * spectrogram and no conditioning network uses wrnn_vocode_host below.             */
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

/* ---------------------------------------------------------------------------------------------------------------
 * From a mel spectrogram, without PyTorch: the conditioning network (MelResNet, fatchord_version.py:26-48) and the
 * rest of generate() (:169-264) restated in the library.  A caller holding a state_dict exported as plain float32
 * arrays attaches the `upsample.*` tensors once, then vocodes mels.  Draws are the in-kernel Philox ones
 * (generate(gen_rng='philox')); there is no torch generator to replay.
 * --------------------------------------------------------------------------------------------------------------- */

/* One state_dict entry: its key and its fp32 values, row-major as torch stores them (host or device pointer). */
typedef struct {
  const char *name;
  const float *data;
  int64_t numel;
} wrnn_tensor;

/* The UpsampleNetwork arguments of the WaveRNN ctor (hparams voc_*).  feat_dims is the handle's (80). */
typedef struct {
  int32_t compute_dims;   /* 128 */
  int32_t res_out_dims;   /* 128 (= 4 * aux_dims) */
  int32_t res_blocks;     /* 10 */
  int32_t pad;            /* 2 */
  int32_t n_factors;      /* 3 */
  int32_t factors[4];     /* (5, 5, 11) */
  int32_t hop_length;     /* 275 == product of the factors */
} wrnn_upsample_cfg;

/* Reads the upsample.* tensors among t[0..n) by their state_dict keys (entries outside upsample.* and the BatchNorms'
 * num_batches_tracked are ignored), folds each eval-mode BatchNorm (eps 1e-5) into the convolution before it -- in
 * double, on the host -- builds the 5-tap interpolation table of the three stretch + conv stages and uploads both.
 * Refused (WRNN_E_INVALID): a missing, repeated or unknown upsample.* key or one with the wrong number of elements
 * (the message names it); compute_dims or res_out_dims other than 128; a geometry the 5-tap table does not encode
 * (pad != 2, product of the factors != hop_length, or an impulse response wider than +-2 frames).  Replaces any
 * upsampler attached before.                                                                                     */
int wrnn_attach_upsampler(wrnn_t *h, const wrnn_upsample_cfg *cfg, const wrnn_tensor *t, int32_t n);

/* The frame-rate conditioning of wrnn_job from a mel spectrogram, on the device (fp32 FFMA, no tensor cores):
 *   mel        [feat, T]          the layout of the reference's mel .npy (gen_wavernn.py)
 *   mel_frames [T + 2*pad, feat]  the zero-padded mel, transposed (F.pad(mel, (pad, pad))[0].T)
 *   aux_frames [T, res_out]       MelResNet output, transposed
 *   up_taps    [hop, 5]           the interpolation table; NULL when not wanted
 * All DEVICE pointers; asynchronous on `stream`.                                                                 */
int wrnn_conditioning_frames(wrnn_t *h, const float *mel, int64_t T, float *mel_frames, float *aux_frames,
                             float *up_taps, void *stream);

/* generate(mel, None, batched, target, overlap, mu_law) with gen_rng='philox', as one call: fold geometry
 * (fold_with_overlap, :319-338; one fold of T*hop samples when unbatched), wrnn_conditioning_frames into handle
 * scratch, the sample loop on the engine wrnn_generate would pick (Philox keyed by philox_seed, offset 0, folds
 * numbered from 0), and wrnn_epilogue with float64 fade, fade-out and mu-law tables built on the host with the
 * reference's expressions.  A handle whose engine is the SIMT one (fp32 strict arithmetic) takes the per-sample
 * rows: they are expanded into scratch first, 832 B per sample of T*hop.                                        */
typedef struct {
  const float *mel;        /* [feat, T]                                                          */
  int64_t T;               /* mel frames, >= 21 (the fade-out spans the last 20 hops)            */
  int32_t batched;         /* fold with overlap (1) or one fold for the whole stream (0)         */
  int32_t target;          /* samples per fold (batched)                                         */
  int32_t overlap;         /* cross-faded samples between folds (batched; > 0)                   */
  int32_t mu_law;          /* RAW head: labels are mu-law codes (ignored by the MoL head)        */
  uint64_t philox_seed;    /* key of the in-kernel draws (WaveRNN.gen_philox_seed)               */
  double *wav;             /* [(T - 1) * hop] float64                                            */
} wrnn_vocode_job;

/* DEVICE pointers; asynchronous on `stream`, no host synchronisation (device errors: wrnn_check after a sync).
 * Refused: T < 21, a batched job with target <= 0 or overlap <= 0, a handle with no upsampler attached.        */
int wrnn_vocode(wrnn_t *h, const wrnn_vocode_job *job, void *stream);
/* The same with HOST mel and wav: copies in, runs, copies out, synchronises and returns wrnn_check's verdict. */
int wrnn_vocode_host(wrnn_t *h, const wrnn_vocode_job *job);

/* A batch of mels as ONE job: one launch of the conditioning network, one engine job over the folds of every utterance
 * (folds ordered by utterance, then ascending; one tile-launch per 64 folds on TCGEN05, one launch on STREAM) and one
 * epilogue launch.  A step of the sample loop costs about the same for 1 fold as for 64, so k short utterances cost
 * about as much as one.
 *
 * Contract: utterance i's waveform is bit-identical to wrnn_vocode on the same handle with {mel_i, T_i, batched,
 * target, overlap, mu_law, philox_seed_i} whenever the batch and that single call are served by the same engine: each
 * fold's draws are keyed by (its utterance's philox_seed, its index within the utterance), not by its place in the
 * batch.  A handle created with a fixed engine (TCGEN05, STREAM, SIMT) always serves both with that engine.  An AUTO
 * handle routes the batch by its TOTAL fold count with wrnn_generate's rule (MoL jobs of 257 folds or more go to the
 * stream engine), so a batch can land on another engine than its single calls; its waveforms then agree with them
 * to DESIGN.md section 5's tolerances, not bit for bit.
 *
 * Unbatched (batched = 0): each utterance is one fold and every fold runs max_i(T_i) * hop steps; a shorter
 * utterance's fold runs past its end on zero conditioning and those samples are discarded (the recurrence is causal,
 * so its first T_i * hop samples are unchanged).  That costs sum_i (max T - T_i) * hop wasted fold-steps.
 *
 * Refused (WRNN_E_INVALID, the handle stays usable): n_utts < 1 or > 65535, a null utts / mel / wav, any T_i < 21
 * (the message names i), a batched job with target <= 0 or overlap <= 0, a laid-out stream of 2^31 samples or more
 * (sum_i (T_i + 4) * hop), a total of 2^31 folds or more, a handle with no upsampler attached.                  */
typedef struct {
  const float *mel;        /* [feat, T], the layout of wrnn_vocode_job::mel */
  int64_t T;               /* >= 21                                          */
  uint64_t philox_seed;    /* this utterance's key                           */
  double *wav;             /* [(T - 1) * hop] float64                        */
} wrnn_utterance;

typedef struct {
  const wrnn_utterance *utts;   /* HOST array of n_utts descriptors (mel / wav: device or host per entry point) */
  int32_t n_utts;
  int32_t batched, target, overlap, mu_law;   /* shared, meaning as in wrnn_vocode_job */
} wrnn_vocode_batch;

/* DEVICE mel / wav pointers; asynchronous on `stream` (device errors: wrnn_check after a sync). */
int wrnn_vocode_many(wrnn_t *h, const wrnn_vocode_batch *b, void *stream);
/* The same with HOST mel / wav: copies in, runs, copies out, synchronises and returns wrnn_check's verdict. */
int wrnn_vocode_many_host(wrnn_t *h, const wrnn_vocode_batch *b);

/* Live unbatched vocoding ("Slow Unbatched Generation", gen_tacotron.py:31): the waveform reaches the caller while the
 * persistent kernel is still generating it.  Unbatched generation is one fold with no cross-fade, so sample n of the
 * waveform depends on generated sample n alone (and on the fade-out table over the last 20 hops).  The kernel stores
 * its samples straight into a pinned host buffer the library owns and publishes how many it has stored every 64
 * steps; each poll turns the newly published ones into float64 samples of wav with wrnn_epilogue's arithmetic.
 *
 * Contract: the concatenated waveform is bit-identical to wrnn_vocode_host on the same handle with the same {mel, T,
 * batched = 0, mu_law, philox_seed}: the draws are Philox, keyed as in wrnn_vocode.
 *
 * Refused (WRNN_E_INVALID, the message names the cause, the handle stays usable): batched != 0 (a batched job's folds
 * all finish at its last step); a handle whose engine for the job is not the persistent one (TCGEN05: the stream
 * engine's cluster form is slower than real time for one fold, the SIMT engine is not timed); a null job, mel or wav;
 * T < 21; a handle with no upsampler attached.
 *
 * While a live job is in flight every other entry point on the handle returns WRNN_E_BUSY (a second
 * wrnn_vocode_live_start included); wrnn_destroy waits for the job and then frees.  A live job cannot be cancelled. */

/* Starts wrnn_vocode of an UNBATCHED job (job->batched must be 0; target / overlap ignored) whose waveform is
 * delivered while it is generated.  job->mel: host or device (UVA); job->wav: HOST, [(T - 1) * hop] float64.
 * Enqueued on `stream`; returns without waiting for the kernel. */
int wrnn_vocode_live_start(wrnn_t *h, const wrnn_vocode_job *job, void *stream);

/* Waits up to wait_us for more samples, writes every newly final sample into job->wav and sets *n_ready to the
 * number of leading samples of wav that are final (never decreases; never rewritten).
 * Returns 1 while the job runs, 0 once all (T - 1) * hop samples are in wav, or a negative WRNN_E_* code
 * (device errors as wrnn_check: samples delivered before the error stay valid).  After 0 or an error the handle is free.
 * The wait sleeps in intervals of 100 us; wait_us <= 0 returns at once.  A null n_ready, or a handle with no live job,
 * is refused (WRNN_E_INVALID) without touching the job. */
int wrnn_vocode_live_poll(wrnn_t *h, int32_t wait_us, int64_t *n_ready);

/* Live batch vocoding: up to 64 unbatched utterances in ONE persistent job, each delivered while it is generated, so
 * that one GPU serves several listeners at once.  The layout is wrnn_vocode_many's unbatched one: utterance i is fold
 * i, every fold runs max_i(T_i) * hop steps, and fold i's draws are keyed by (philox_seed_i, 0).  Each fold publishes
 * its own sample count every 64 steps and at the last step, so a short utterance completes before the job ends.
 *
 * Contract: utterance i's concatenated waveform is bit-identical to wrnn_vocode_many_host on the same handle and batch,
 * and so (wrnn_vocode_many's contract, fixed-engine handle) to wrnn_vocode_host with {mel_i, T_i, batched = 0, mu_law,
 * philox_seed_i}.
 *
 * Refused (WRNN_E_INVALID, the message names the cause, the handle stays usable): batched != 0; n_utts < 1 or > 64
 * (one persistent tile holds 64 folds, and a second tile would start only after the first had finished, so it would
 * not be live); a null b, utts, mel or wav; any T_i < 21 (the message names i); a handle whose engine for the job is
 * not the persistent one; a handle with no upsampler attached.
 *
 * Busy rules are those of wrnn_vocode_live_start, shared with it: while either kind of live job is in flight every other
 * entry point returns WRNN_E_BUSY (both live starts included), and wrnn_destroy waits for the job.  Each poll serves
 * only the jobs of its own start: the other poll refuses (WRNN_E_INVALID, naming the right poll) without touching the
 * job. */

/* Starts wrnn_vocode_many of an UNBATCHED batch (b->batched must be 0; target / overlap ignored) whose waveforms are
 * delivered while they are generated.  utts[i].mel: host or device (UVA); utts[i].wav: HOST, [(T_i - 1) * hop] float64.
 * Enqueued on `stream`; returns without waiting for the kernel. */
int wrnn_vocode_many_live_start(wrnn_t *h, const wrnn_vocode_batch *b, void *stream);

/* Waits up to wait_us for more samples of any utterance, writes every newly final sample into its utts[i].wav and sets
 * n_ready[i] (an array of n_utts) to the number of leading samples of utterance i that are final (never decreases; never
 * rewritten; utterance i is complete once n_ready[i] == (T_i - 1) * hop, possibly while the job still runs).
 * Returns 1 while the kernel runs, 0 once every utterance is complete, or a negative WRNN_E_* code (device errors as
 * wrnn_check: samples delivered before the error stay valid).  After 0 or an error the handle is free.  The wait is
 * wrnn_vocode_live_poll's.  A null n_ready, or a handle with no batch live job in flight, is refused (WRNN_E_INVALID)
 * without touching the job. */
int wrnn_vocode_many_live_poll(wrnn_t *h, int32_t wait_us, int64_t *n_ready);

/* Live session: listeners that arrive at any time.  The session holds a persistent tile of `capacity` slots (1 to 64);
 * each submitted utterance takes a free slot and is admitted into the RUNNING kernel at its next admission boundary
 * (every 64 steps), then delivered as a wrnn_vocode_many_live utterance.  An idle session's kernel exits; the next
 * submit relaunches it.
 *
 * Contract: a ticket's delivered waveform is bit-identical to wrnn_vocode_host with {mel, T, batched = 0, mu_law,
 * philox_seed} on the same handle, whatever its slot, its admission step, the launch that served it and whatever else
 * was in flight.  n_ready never decreases and a delivered sample is never rewritten.
 *
 * While a session is open every other entry point returns WRNN_E_BUSY (both live starts included; their polls refuse
 * it); wrnn_destroy closes it.  Refused (WRNN_E_INVALID, with a message) before the handle is looked at: capacity
 * outside 1..64, max_T < 21, null pointers, T < 21; then a null handle, a handle whose engine is not the persistent one
 * or without an upsampler, max_T beyond 2^27 samples per utterance, T > max_T, any call but wrnn_live_open without an
 * open session. */
enum { WRNN_LIVE_RUNNING = 0, WRNN_LIVE_DONE = 1, WRNN_LIVE_CANCELLED = 2 };
typedef struct {
  int64_t ticket;
  int64_t n_ready;    /* leading samples of the ticket's wav that are final */
  int32_t state;      /* WRNN_LIVE_*: DONE / CANCELLED once, by the poll that releases the ticket's slot */
  int32_t pad;
} wrnn_live_ticket;

/* Opens a session of `capacity` slots for utterances of up to max_T frames (mu_law: RAW head, as wrnn_vocode_job).
 * Allocates a pinned, mapped buffer [progress words | mailboxes | capacity x (max_T - 1) * hop samples] and a device
 * frame arena of `capacity` regions of max_T + 4 frames.  The kernel runs on `stream`. */
int wrnn_live_open(wrnn_t *h, int32_t capacity, int64_t max_T, int32_t mu_law, void *stream);

/* Submits one utterance (u->mel: host or device; u->wav: HOST, [(T - 1) * hop] float64, written by wrnn_live_poll) and
 * returns its ticket (1, 2, ... in submission order).  The conditioning network runs into the slot's region on a side
 * stream, on the SMs the kernel leaves free; the request is posted to the kernel once it is complete.  WRNN_E_BUSY when
 * every slot holds an utterance (there is no host queue): poll until one is released. */
int wrnn_live_submit(wrnn_t *h, const wrnn_utterance *u, int64_t *ticket);

/* Submits one utterance for BATCHED generation (wrnn_vocode_job with batched = 1, target, overlap): its n_seg folds
 * (fold_with_overlap's geometry) each take a free slot of the session and are admitted into the running kernel, each at
 * the next boundary it is seen (not necessarily the same one).  Fold b's draws are keyed by (philox_seed, b), as
 * wrnn_vocode's are, and every fold runs target + 2 * overlap steps.
 *
 * Contract: the ticket's delivered wav is bit-identical to wrnn_vocode_host on the same handle with {mel, T, batched = 1,
 * target, overlap, mu_law = the session's, philox_seed}, whatever its slots, the boundaries its folds were admitted at,
 * the launches that served them and whatever else was in flight.  Sample n is final once every fold whose window
 * [b * (target + overlap), + target + 2 * overlap) covers n has stored its sample for n; n_ready is the longest final
 * prefix (fold 0's samples lead it, one per step, so the waveform starts to play as early as an unbatched ticket's).
 * It never decreases and a delivered sample is never rewritten.  A batched ticket is ONE wrnn_live_ticket:
 * wrnn_live_cancel cancels all its folds, and wrnn_live_poll releases all its slots together, once every fold has
 * retired, and only then reports it DONE or CANCELLED.
 *
 * Refused (WRNN_E_INVALID, with a message; the handle and the session are unchanged): those of wrnn_live_submit;
 * target <= 0 or overlap <= 0; more folds than the session's capacity (it could never be admitted); target + 2 * overlap
 * > (max_T - 1) * hop (a fold's samples would not fit a slot's row).  WRNN_E_BUSY, taking no slot, while fewer slots
 * are free than the utterance has folds: poll until enough are released. */
int wrnn_live_submit_batched(wrnn_t *h, const wrnn_utterance *u, int32_t target, int32_t overlap, int64_t *ticket);

/* Cancels a ticket: its slots stop at the next boundary and are released by a later poll (state CANCELLED). */
int wrnn_live_cancel(wrnn_t *h, int64_t ticket);

/* Waits up to wait_us for progress, writes every newly final sample into its ticket's wav and reports in out[0 ..
 * *n_out) the tickets whose slot was released since the last poll (state DONE or CANCELLED), then every ticket still
 * held (state RUNNING).  max_out must be at least 2 * capacity.  Returns 1 while any ticket is held, 0 when none is,
 * or a negative WRNN_E_* code (device errors as wrnn_check).  The wait is wrnn_vocode_live_poll's. */
int wrnn_live_poll(wrnn_t *h, int32_t wait_us, wrnn_live_ticket *out, int32_t max_out, int32_t *n_out);

/* Closes the session: cancels every ticket still held, waits for the kernel to exit and frees the session's buffers. */
int wrnn_live_close(wrnn_t *h);

/* ---------------------------------------------------------------------------------------------------------------
 * Scoring: how likely a given waveform is under the model, on the engine that generates it.  The loss the reference
 * trains with (train_wavernn.py:83), per sample, teacher-forced and reduced inside the kernel where the logits are:
 *   MoL: discretized_mix_logistic_loss(reduce=False) (utils/distribution.py:16-84; num_classes 65536, log_scale_min
 *        log(1e-14)), all of its branches, in fp32 in the reference's order;
 *   RAW: F.cross_entropy, logsumexp(logits) - logits[label] with label = rint((y + 1)(n_classes - 1) / 2) clamped to
 *        [0, n_classes - 1] -- pass label_2_float(label) as the target (utils/dataset.py:88).
 * In nats, with accurate expf / logf / log1pf.  No draws are made.  The stream engine scores the MoL head only.
 * --------------------------------------------------------------------------------------------------------------- */

/* nll[t][b] (device, [seg_len, n_seg], the layout of x_force) = the loss of target x_force[t][b] given x_force[0..t-1][b]
 * and the conditioning rows up to t.  job->x_force (device) is required and holds the targets; step t consumes
 * x_force[t-1] exactly as wrnn_generate does.  Rows >= steps of nll are untouched.  job->out may be NULL and is never
 * written; logits_out works as in wrnn_generate (the same chains, so the same bits); the draw fields are ignored.
 * The engine is the one wrnn_generate would pick.  Asynchronous on `stream` (device errors: wrnn_check after a sync). */
int wrnn_score(wrnn_t *h, const wrnn_job *job, float *nll, void *stream);

/* One recording to score from its mel spectrogram.  Scored UNBATCHED, as one fold: step t conditions on row t of the
 * T*hop-row stream wrnn_vocode would build from `mel` and on x[t-1] (0 at t = 0) -- the model's likelihood of the
 * whole recording (folding with overlap would change it).                                                          */
typedef struct {
  const float *mel;        /* [feat, T], the layout of wrnn_vocode_job::mel           */
  int64_t T;               /* mel frames                                               */
  const float *x;          /* [n] the waveform, samples in [-1, 1] (RAW: label_2_float) */
  int64_t n;               /* samples to score, 1 <= n <= T * hop                       */
  float *nll;              /* [n] per-sample loss in nats                               */
} wrnn_score_utt;

/* All utterances as ONE job: one launch of the conditioning network, one engine job over n_utts folds of max_i n_i steps
 * (rows past an utterance read as zeros; nothing is written past n_i), engine chosen as for wrnn_vocode_many (a SIMT
 * handle expands the rows into scratch first).  Each utterance's losses are bit-identical to its own single-utterance
 * call whenever both are served by the same engine (always on a handle created with a fixed engine).
 * Refused (WRNN_E_INVALID, the handle stays usable): n_utts < 1 or > 65535; a null utts, mel, x or nll; n_i < 1 or
 * n_i > T_i * hop (the message names i); a laid-out stream of 2^31 samples or more (sum_i (T_i + 4) * hop); a handle
 * with no upsampler attached; a RAW head on the stream engine.  DEVICE mel / x / nll pointers; asynchronous.        */
int wrnn_score_many(wrnn_t *h, const wrnn_score_utt *utts, int32_t n_utts, void *stream);
/* The same with HOST mel / x / nll: copies in, runs, copies out, synchronises and returns wrnn_check's verdict. */
int wrnn_score_many_host(wrnn_t *h, const wrnn_score_utt *utts, int32_t n_utts);

/* ---------------------------------------------------------------------------------------------------------------
 * Mel analysis: the reference's melspectrogram(y) (utils/dsp.py:72-81: librosa 0.6.3 STFT -> Slaney mel filterbank ->
 * amp_to_db -> normalize) on the device, so that a recording can be analysed, vocoded again or scored without librosa.
 * An analysis object needs no weights.  Per frame: the reflect-padded samples (np.pad(y, n_fft / 2, 'reflect')) times
 * the periodic Hann window of win_length centred in n_fft, a float64 real FFT, each bin rounded to complex64 as
 * librosa's stft(dtype=np.complex64) stores it, its magnitude, the band sums with the float64 filterbank, then
 * clip((20 log10(max(1e-5, M)) - min_level_db) / -min_level_db, 0, 1) stored as float32 (DESIGN.md §3.8).
 * --------------------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t sample_rate;   /* 22050; > 0                                             */
  int32_t n_fft;         /* 2048; a power of two, 256..4096                        */
  int32_t hop_length;    /* 275; >= 1                                              */
  int32_t win_length;    /* 1100; 1..n_fft                                         */
  int32_t n_mels;        /* 80; 1..128                                             */
  float fmin;            /* 40; 0 <= fmin < sample_rate / 2                        */
  float min_level_db;    /* -100; < 0                                              */
} wrnn_mel_cfg;          /* the hparams fields utils/dsp.py reads; fmax is sample_rate / 2 as in linear_to_mel */

typedef struct wrnn_mel_plan wrnn_mel_t;

/* Builds the tables once, in float64 on the host (window, twiddles, Slaney filterbank with Slaney norm and each band's
 * nonzero bin range: librosa 0.6.3 filters.mel(sr, n_fft, n_mels, fmin), htk=False, norm=1) and uploads them to
 * `device`.  A configuration outside the ranges above is refused (WRNN_E_INVALID, with a message) before the device is
 * looked at.  An analysis object has no busy state: any number of calls may use it at once, on any streams. */
int wrnn_mel_create(wrnn_mel_t **out, const wrnn_mel_cfg *cfg, int device);
void wrnn_mel_destroy(wrnn_mel_t *m);

typedef struct {
  const float *y;        /* [n] waveform, float32 as librosa.load returns it                             */
  int64_t n;             /* > n_fft / 2 (one reflection of the centre padding)                           */
  float *mel;            /* [n_mels, 1 + n / hop_length], the layout of the reference's mel .npy          */
} wrnn_mel_utt;

/* Every frame of every utterance in one kernel launch.  Each utterance's mel is bit-identical to its own call.
 * Refused (WRNN_E_INVALID): a null m or u, n_utts < 1, a null y or mel, n_i <= n_fft / 2 (the message names i), a
 * batch of 2^31 frames or more.  DEVICE pointers; asynchronous on `stream`. */
int wrnn_melspectrogram_many(const wrnn_mel_t *m, const wrnn_mel_utt *u, int32_t n_utts, void *stream);
/* The same with HOST y / mel: copies in, runs, copies out and synchronises. */
int wrnn_melspectrogram_many_host(const wrnn_mel_t *m, const wrnn_mel_utt *u, int32_t n_utts);

/* Griffin-Lim: the reference's reconstruct_waveform(mel, n_iter) (utils/dsp.py:105-116, librosa 0.7 mel_to_stft and
 * griffinlim), the inverse of the analysis above with the same configuration and tables.  Per utterance:
 *   1. S = the non-negative least-squares inversion of db_to_amp(denormalize(mel)) (float32) through the float32
 *      filterbank, per frame in float64: the clipped minimum-norm least-squares start, then a fixed number of
 *      accelerated projected-gradient steps (DESIGN.md §3.9);
 *   2. angles = exp(2 pi i u), u a Philox4x32-10 draw keyed by (phase_seed, frame, bin);
 *   3. n_iter times: inverse = istft(S angles) (float64 inverse FFT times the window, overlap-added into float32 in
 *      frame order, divided by the float32 window sum-square, centre-trimmed), rebuilt = stft(inverse) (complex64),
 *      angles = rebuilt - (0.99 / 1.99) tprev, angles /= |angles| + 1e-16;
 *   4. wav = istft(S angles).
 * Contract: each utterance's wav is bit-identical to its own call; the same phase_seed gives the same bits. */
typedef struct {
  const float *mel;      /* [n_mels, T] normalized mel, the layout of the reference's mel .npy          */
  int64_t T;             /* frames; hop_length * (T - 1) > n_fft / 2                                   */
  uint64_t phase_seed;   /* key of the initial phases                                                  */
  float *wav;            /* [hop_length * (T - 1)] float32, as reconstruct_waveform returns it          */
} wrnn_gl_utt;
/* Every frame of every utterance in each launch: one launch for the solve, then two per iteration and two more.
 * n_iter >= 0 (0 is the istft of the initial phases).  Refused (WRNN_E_INVALID): a null m or u, n_utts < 1, a null
 * mel or wav, hop_length * (T_i - 1) <= n_fft / 2 (the message names i), a batch of 2^31 frames or more, n_iter < 0.
 * Scratch (about 29 KB per frame at n_fft = 2048) is allocated stream-ordered inside the call, in batches of at most
 * 1 GiB; a failed allocation is WRNN_E_CUDA.  DEVICE mel / wav; asynchronous on `stream`. */
int wrnn_griffinlim_many(const wrnn_mel_t *m, const wrnn_gl_utt *u, int32_t n_utts, int32_t n_iter, void *stream);
/* The same with HOST mel / wav: copies in, runs, copies out and synchronises. */
int wrnn_griffinlim_many_host(const wrnn_mel_t *m, const wrnn_gl_utt *u, int32_t n_utts, int32_t n_iter);

/* Resampling: the reference's load_wav (utils/dsp.py: librosa.load(path, sr=hp.sample_rate), librosa 0.6.3) after
 * decoding and mixing to mono, on the device: resampy's `kaiser_best` band-limited interpolation to the analysis
 * object's sample_rate, then librosa's fix_length.  Per utterance, with ratio = (double)sample_rate_out / sample_rate:
 *   1. int(n * ratio) samples of resampy's resample_f with the kaiser_best half-window (64 zero crossings, Kaiser
 *      beta 14.769656459379492, rolloff 0.9475937167399596, 2^16 table entries per zero crossing), scaled by ratio
 *      when it is below 1; output t reads the time register t * (1 / ratio), and each tap's weighted sample is added
 *      in float64 and the sum rounded to float32 (DESIGN.md §3.10);
 *   2. zero padding to wrnn_resample_length(n, sample_rate, sample_rate_out) = ceil(n * ratio) samples.
 * Equal rates copy x, as librosa does not resample them.  The result feeds wrnn_melspectrogram_many,
 * wrnn_score_wav_many and wrnn_vocode built for the same sample_rate.
 * Contracts: a batch gives the same bits as each utterance resampled alone; the _host entry point gives the same bits
 * as the device one; nothing is written past wrnn_resample_length samples of y.
 * The filter table (33.6 MB of float64) is uploaded once per analysis object, by its first resampling call. */
typedef struct {
  const float *x;        /* [n] the decoded mono recording, float32                                  */
  int64_t n;             /* samples, >= 1                                                             */
  int32_t sample_rate;   /* its rate, > 0; each utterance of a batch may have its own                 */
  int32_t pad;
  float *y;              /* [wrnn_resample_length(n, sample_rate, m's sample_rate)]                   */
} wrnn_resample_utt;
/* ceil(n * ((double)sr_out / sr_in)): the samples librosa.load returns; -1 if n < 0 or a rate is <= 0. */
int64_t wrnn_resample_length(int64_t n, int32_t sr_in, int32_t sr_out);
/* Every output sample of every utterance in one kernel launch.  Refused (WRNN_E_INVALID; the message names i): a null
 * m or u, n_utts < 1, a null x or y, sample_rate <= 0, n < 1, int(n * ratio) < 1 (resampy refuses it too), a ratio
 * below 2^-16 (the filter would have no taps), a batch of 2^31 output samples or more.  DEVICE x / y; asynchronous on
 * `stream` (the first call on an object also uploads the table, synchronously). */
int wrnn_resample_many(const wrnn_mel_t *m, const wrnn_resample_utt *u, int32_t n_utts, void *stream);
/* The same with HOST x / y: copies in, runs, copies out and synchronises. */
int wrnn_resample_many_host(const wrnn_mel_t *m, const wrnn_resample_utt *u, int32_t n_utts);

/* Scoring a recording from its audio alone: what preprocess.py:36-47 and utils/dataset.py:86-91 do, on the device.
 *   1. y /= max|y| (float32) when peak_norm is set or the peak exceeds 1;
 *   2. mel = the analysis of that y by `m` (T = 1 + n / hop frames, so T * hop >= n);
 *   3. the stored labels, evaluated in float32: MoL trunc(clip((y + 1) * 65535 / 2, 0, 65535)); RAW with mu_law
 *      encode_mu_law(y, n_classes); RAW without it trunc(float_2_label(y, bits)); mapped back with label_2_float;
 *   4. wrnn_score_many's job on {mel, those targets}.
 * Contract: nll is bit-identical to wrnn_score_many on the same handle given the mel wrnn_melspectrogram_many makes of
 * the normalised y and those targets.  mu_law is wrnn_vocode_job::mu_law, a property of the training data that the
 * handle does not know; the MoL head ignores it.
 * Refused (WRNN_E_INVALID, the handle stays usable): those of wrnn_score_many; a null m; m->n_mels != feat_dims, or
 * m->hop_length other than the attached upsampler's hop_length, or m on another device (the message names both);
 * any n_i <= n_fft / 2 (the message names i).  Busy rules are the handle's.  DEVICE y / nll; asynchronous. */
typedef struct {
  const float *y;        /* [n] the recording, float32                                        */
  int64_t n;             /* samples, > n_fft / 2                                               */
  float *nll;            /* [n] per-sample loss in nats                                        */
} wrnn_score_wav_utt;
int wrnn_score_wav_many(wrnn_t *h, const wrnn_mel_t *m, const wrnn_score_wav_utt *u, int32_t n_utts, int32_t peak_norm,
                        int32_t mu_law, void *stream);
/* The same with HOST y / nll: copies in, runs, copies out, synchronises and returns wrnn_check's verdict. */
int wrnn_score_wav_many_host(wrnn_t *h, const wrnn_mel_t *m, const wrnn_score_wav_utt *u, int32_t n_utts,
                             int32_t peak_norm, int32_t mu_law);

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
