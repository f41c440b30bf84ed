// wrnn_engine.h -- internal C++ interface between the C ABI (wrnn_capi.cu) and the engines.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/wavernn_b200.h"
#include "wrnn_fold.h"

namespace wrnn {

void set_error(const std::string& msg);          // thread-local last error (wrnn_capi.cu)

#define WRNN_CUDA_OK(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::wrnn::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e));           \
      return WRNN_E_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

// Grid of a grid-stride kernel: `blocks`, capped at 8 blocks per SM of the current device.
inline int grid_stride_blocks(long long blocks) {
  int dev = 0, n_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const long long cap = 8ll * (n_sm > 0 ? n_sm : 1);
  return (int)(blocks < cap ? blocks : cap);
}

// Staging of the host-memory entry points.  place puts each item at a 256-B-aligned offset of the device buffer d
// (staged_bytes(items) long) and copies it there on st (cudaMemcpyDefault: src may be host or device memory; src NULL:
// a region the job writes); dev[k] is item k's device address, NULL for an empty item.  copy_back copies results back
// (host or device destinations) on stream 0 and synchronises.  Static, so that none is exported by the library.
struct Staged { const void* src; size_t bytes; };
struct Unstaged { void* dst; const void* src; size_t bytes; };
static inline size_t align256(size_t bytes) { return (bytes + 255) & ~size_t(255); }

static inline size_t staged_bytes(const std::vector<Staged>& items) {
  size_t total = 0;
  for (const Staged& it : items) total += align256(it.bytes);
  return total;
}

static inline int place(void* d, const std::vector<Staged>& items, cudaStream_t st, std::vector<void*>& dev) {
  char* p = static_cast<char*>(d);
  dev.assign(items.size(), nullptr);
  for (size_t k = 0; k < items.size(); ++k) {
    if (!items[k].bytes) continue;
    dev[k] = p;
    if (items[k].src) WRNN_CUDA_OK(cudaMemcpyAsync(p, items[k].src, items[k].bytes, cudaMemcpyDefault, st));
    p += align256(items[k].bytes);
  }
  return WRNN_OK;
}

static inline int copy_back(const std::vector<Unstaged>& items) {
  for (const Unstaged& it : items)
    if (it.bytes) WRNN_CUDA_OK(cudaMemcpyAsync(it.dst, it.src, it.bytes, cudaMemcpyDefault, 0));
  WRNN_CUDA_OK(cudaStreamSynchronize(0));
  return WRNN_OK;
}

// A host-memory entry point of the analysis object (wrnn_mel_t): the items staged in one device allocation of this
// call alone, so that calls on any streams share the object, and freed on every path.  run(dev, out) launches on
// stream 0 with the items' device addresses and sets out[k] for each item k whose region copy_back returns.
template <class F>
int with_staging(int device, const std::vector<Staged>& items, F run) {
  WRNN_CUDA_OK(cudaSetDevice(device));
  void* d = nullptr;
  WRNN_CUDA_OK(cudaMalloc(&d, staged_bytes(items)));
  std::vector<void*> dev;
  std::vector<Unstaged> out(items.size(), Unstaged{nullptr, nullptr, 0});
  int rc = place(d, items, 0, dev);
  if (rc == WRNN_OK) rc = run(dev, out);
  if (rc == WRNN_OK) rc = copy_back(out);
  cudaFree(d);
  return rc;
}

// A launch whose table of n utterances lives on the device for that launch only, allocated and freed in stream order
// on st, so that calls on any streams share one analysis object.  launch(d_tab) enqueues on st.
template <class T, class F>
int with_device_table(const T* tab, size_t n, cudaStream_t st, F launch) {
  const size_t bytes = n * sizeof(T);
  void* d = nullptr;
  WRNN_CUDA_OK(cudaMallocAsync(&d, bytes, st));
  WRNN_CUDA_OK(cudaMemcpyAsync(d, tab, bytes, cudaMemcpyHostToDevice, st));
  const int rc = launch(static_cast<const T*>(d));
  if (rc != WRNN_OK) return rc;
  WRNN_CUDA_OK(cudaFreeAsync(d, st));
  return WRNN_OK;
}

// ---- live session (wrnn_live_open / _submit / _cancel / _poll / _close; DESIGN §3.7) ------------------------------------
// A session launch runs an open-ended tile of C slots.  Slot f's utterance runs from its admission step a to its end step
// e (global steps of the launch), at local step t - a.  Admissions, cancellations and the launch's stop are decided by
// CTA 0 at boundaries b = k * SES_PERIOD and take effect at the next boundary.
constexpr int SES_PERIOD = 64;
constexpr int SES_DRAIN = 4;                        // a slot is retired at the first boundary >= e + SES_DRAIN (staging runs <= 3 steps ahead)
constexpr int SES_ADMIT_LIMIT = 1 << 27;            // no admission at a boundary from here on: every step index stays below 2^28
constexpr long long SES_MAX_STEPS = 1ll << 27;      // samples of one utterance: (T - 1) * hop <= 2^27
constexpr unsigned SES_RETIRED = 1u << 31;          // progress word: (tag << 32) | [retired bit] | samples stored
// Slot table entry (device, [2 versions][64]): version k is written at boundary k * SES_PERIOD.  The occupant is fold
// `fold` of its utterance (the Philox counter fold of its draws); local step ts reads arena row row0 + ts, or zeros from
// ts = rows on (an unbatched occupant: fold 0, its region's first row, rows its steps never reach).
struct SesEntry {
  int a, e;
  unsigned long long seed;
  unsigned fold;
  int row0, rows, pad;
};
// One slot's mailbox (mapped host memory, written by the host only): the tag of the latest request and of the latest
// cancellation, and the request's Philox seed, step count, fold and rows (written before `req`).
struct SesMail {
  unsigned long long req, cancel, seed;
  long long steps;
  unsigned fold;
  int row0, rows, pad;
};
// A ticket's 32-bit tag in the progress word and the mailbox: never 0 (the tag of a slot that never held a request).
inline unsigned ses_tag(long long ticket) { return (unsigned)((unsigned long long)(ticket - 1) % 0xffffffffull) + 1u; }
// CTA 0's state of one slot and its decisions at boundary b, shared by the kernel and the CPU test hook.
struct SesSlot {
  unsigned tag;                  // the occupant's (or last occupant's) ticket tag
  int a, e;
  unsigned long long seed;
  bool retired;
  unsigned fold;
  int row0, rows;
};
// Retirement (returns the progress word to publish, or 0) and cancellation at boundary b.
__host__ __device__ inline unsigned long long ses_retire_cancel(SesSlot& s, int b, unsigned cancel_tag) {
  unsigned long long word = 0;
  if (!s.retired && s.e + SES_DRAIN <= b) {
    s.retired = true;
    word = ((unsigned long long)s.tag << 32) | SES_RETIRED | (unsigned)(s.e - s.a);
  }
  if (!s.retired && cancel_tag == s.tag && s.e > b + SES_PERIOD) s.e = b + SES_PERIOD;
  return word;
}
__host__ __device__ inline bool ses_admits(const SesSlot& s, int b, unsigned req_tag) {
  return s.retired && req_tag != s.tag && b < SES_ADMIT_LIMIT;
}
// Admission at boundary b: the utterance runs steps [b + SES_PERIOD, + steps).  Returns the progress word to publish.
__host__ __device__ inline unsigned long long ses_admit(SesSlot& s, int b, unsigned req_tag, unsigned long long seed, long long steps,
                                                     unsigned fold, int row0, int rows) {
  s.tag = req_tag; s.a = b + SES_PERIOD; s.e = s.a + (int)steps; s.seed = seed; s.retired = false;
  s.fold = fold; s.row0 = row0; s.rows = rows;
  return (unsigned long long)req_tag << 32;
}
struct SesCtl {
  SesEntry* tab;                 // [2][64] (device)
  int* stop;                     // [2]: the step at which each version stops the launch, or INT_MAX (device)
  const SesMail* mail;           // [64] (device alias of mapped host memory)
  unsigned long long* progress;  // [64] (device alias of mapped host memory)
};

class Engine {
 public:
  virtual ~Engine() {}
  // async; keys: optional per-fold Philox keys ([job.n_seg], device; NULL = keyed by seg_first + fold, philox_seed)
  virtual int generate(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys) = 0;
  // The same job with the loss of target x_force[t] in the sampler's place: nll [steps][n_seg] (device), out unused.
  virtual int score(const wrnn_job& job, float* nll, cudaStream_t stream, const FoldKey* keys) = 0;
  virtual int check() = 0;                                              // after stream sync
  virtual bool supports(const wrnn_job& job) const { (void)job; return true; }   // job inside this engine's envelope?
  virtual bool scores() const { return true; }                          // serves wrnn_score for this handle's head?
  // Live vocoding (wrnn_vocode_live_start, wrnn_vocode_many_live_start): NULL when this engine serves it, else why not.
  // generate_live runs a job of one tile (up to 64 folds, keyed by `keys` as generate) whose `out` is mapped host memory
  // and publishes the samples of fold f stored so far to progress[f] (mapped host memory).
  virtual const char* live_refusal() const { return "live vocoding runs on the persistent engine only"; }
  virtual int generate_live(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys, unsigned long long* progress) {
    (void)job; (void)stream; (void)keys; (void)progress;
    set_error(live_refusal());
    return WRNN_E_INVALID;
  }
  // One launch of a live session (same refusal): job.n_seg slots, slot f's conditioning rows from its table entry's row0 of
  // the frame tensors, its samples at job.out + f * job.seg_len (mapped host memory).
  virtual int generate_session(const wrnn_job& job, cudaStream_t stream, const SesCtl& c) {
    (void)job; (void)stream; (void)c;
    set_error(live_refusal());
    return WRNN_E_INVALID;
  }
  virtual const char* name() const = 0;
  virtual int grid_ctas() const = 0;
  int64_t launches = 0;
  int device = 0;
  wrnn_cfg cfg{};
};

// SIMT engine: CUDA-core FMA contractions, fp32-strict or bf16-operand arithmetic.
int make_simt_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// persistent tensor-core engine (wrnn_tc.cu): weights stationary in 128 SMs, wgmma contractions (fp16 / bf16 operands).
int make_tc_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// stream engine (wrnn_stream.cu): activation-stationary, weights streamed from L2; the throughput form for many folds
int make_stream_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// conditioning pre-pass (wrnn_tc.cu): rows [row_lo, row_lo + n_rows) of the per-sample stream from frame-rate tensors
int expand_conditioning(const float* mel_frames, const float* aux_frames, const float* up_taps, int hop, long long row_lo,
                        long long n_rows, float* mels_up, float* aux, cudaStream_t stream);

// One utterance of an epilogue batch: folds [fold0, fold0 + n_seg) of the sample block unfold into wav [wave_len].
struct EpUtt {
  long long fold0;
  int n_seg;
  long long wave_len;
  double* wav;
};
// The epilogue (wrnn_epilogue.cu) over n_utts utterances in one launch: the table `utts` (device) or, with utts == NULL
// and n_utts == 1, `one`.  max_wave_len: the longest wave_len.  Every utterance's samples are bit-identical to its own
// wrnn_epilogue call.  Arguments are checked by the callers.
int epilogue_launch(const float* samples, int seg_len, long long seg_stride, int overlap, const double* fade_in,
                    const double* fade_out, const double* mu_table, int n_classes, const double* tail, long long tail_len,
                    const EpUtt* utts, const EpUtt& one, int n_utts, long long max_wave_len, cudaStream_t stream);

struct Upsampler;                                // conditioning network on the device (wrnn_cond.h)
void destroy_upsampler(Upsampler* u);
struct LiveJob;                                  // a live job and its pinned buffer (wrnn_capi.cu)
struct LiveSession;                              // a live session, its buffers and its slots (wrnn_capi.cu)

}  // namespace wrnn

struct wrnn_handle {
  wrnn::Engine* engine = nullptr;          // engine chosen at create time
  wrnn::Engine* fallback = nullptr;        // ENGINE_AUTO only: SIMT engine, created on first job outside `engine`'s envelope
  wrnn::Engine* stream = nullptr;          // ENGINE_AUTO only: stream engine, created on the first job with many folds
  wrnn::Engine* last = nullptr;            // engine that served the most recent job
  wrnn::HostWeights* host_weights = nullptr;
  bool auto_engine = false;
  bool stream_failed = false;
  // staging of the host-memory entry points (wrnn_generate_host, wrnn_vocode_host, ..., and a live start's mels)
  void* d_stage = nullptr;
  size_t stage_bytes = 0;
  // wrnn_score_wav_many: the normalised recordings, their mels and their targets
  void* d_audio = nullptr;
  size_t audio_bytes = 0;
  // wrnn_attach_upsampler: folded MelResNet, tap table and the scratch of wrnn_vocode
  wrnn::Upsampler* upsampler = nullptr;
  // wrnn_vocode_live_start / wrnn_vocode_many_live_start: the live job (in flight while live_busy) and its pinned, mapped
  // host buffer
  wrnn::LiveJob* live = nullptr;
  bool live_busy = false;
  // wrnn_live_open .. wrnn_live_close: the open live session (every other entry point is busy while it is open)
  wrnn::LiveSession* session = nullptr;
};

namespace wrnn {
// WRNN_E_BUSY with its message while a live job is in flight on h, else WRNN_OK (every entry point but the live poll)
int idle_or_busy(const wrnn_handle* h);
// The rule of every vocoded utterance: T >= 21 mel frames, the fade-out spanning the last 20 hops.  `name` is what the
// message calls T.  check_utterance also requires mel and wav; `at` prefixes its messages ("utterance i: " or "").
int check_frames(const std::string& name, long long T);
int check_utterance(const std::string& at, const void* mel, const void* wav, long long T);
}  // namespace wrnn
