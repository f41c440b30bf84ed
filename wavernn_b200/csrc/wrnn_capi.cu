// wrnn_capi.cu -- the extern "C" surface declared in include/wavernn_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <optional>
#include <string>
#include <thread>
#include <vector>

#include "wrnn_cond.h"
#include "wrnn_engine.h"
#include "wrnn_mel.h"
#include "wrnn_stream_plan.h"

namespace wrnn {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }

int check_frames(const std::string& name, long long T) {
  if (T >= 21) return WRNN_OK;
  set_error(name + " must be >= 21 mel frames: the fade-out spans the last 20 hops of the (T-1)*hop samples");
  return WRNN_E_INVALID;
}

int check_utterance(const std::string& at, const void* mel, const void* wav, long long T) {
  if (!mel || !wav) { set_error(at + "mel and wav are required"); return WRNN_E_INVALID; }
  return check_frames(at + "T", T);
}

// The 16 tensors of `w` into hw, in the style of cond::build_host_upsampler: host_only reads host memory with no CUDA
// call, otherwise cudaMemcpyDefault resolves host or device pointers through UVA.
static int read_weights(const wrnn_cfg& cfg, const wrnn_weights& w, bool host_only, HostWeights& hw) {
  const size_t W2W = H + AUXD, NC = (size_t)cfg.n_classes;
#define WT(dst, src, n) {&hw.dst, w.src, (n), #src}
  const struct { std::vector<float>* dst; const float* src; size_t n; const char* name; } list[] = {
      WT(I_w, I_weight, (size_t)H * (1 + F1IN)), WT(I_b, I_bias, H),
      WT(w1i, rnn1_weight_ih, (size_t)G3 * H), WT(w1h, rnn1_weight_hh, (size_t)G3 * H),
      WT(b1i, rnn1_bias_ih, G3), WT(b1h, rnn1_bias_hh, G3),
      WT(w2i, rnn2_weight_ih, (size_t)G3 * W2W), WT(w2h, rnn2_weight_hh, (size_t)G3 * H),
      WT(b2i, rnn2_bias_ih, G3), WT(b2h, rnn2_bias_hh, G3),
      WT(f1w, fc1_weight, (size_t)H * W2W), WT(f1b, fc1_bias, H),
      WT(f2w, fc2_weight, (size_t)H * W2W), WT(f2b, fc2_bias, H),
      WT(f3w, fc3_weight, NC * H), WT(f3b, fc3_bias, NC)};
#undef WT
  hw.n_classes = cfg.n_classes;
  for (const auto& t : list) {
    if (!t.src) { set_error(std::string("null weight pointer: ") + t.name); return WRNN_E_INVALID; }
    t.dst->resize(t.n);
    if (host_only) { std::memcpy(t.dst->data(), t.src, t.n * sizeof(float)); continue; }
    const cudaError_t e = cudaMemcpy(t.dst->data(), t.src, t.n * sizeof(float), cudaMemcpyDefault);
    if (e != cudaSuccess) { set_error(std::string("copying ") + t.name + ": " + cudaGetErrorString(e)); return WRNN_E_CUDA; }
  }
  return WRNN_OK;
}

static int grow(void** buf, size_t* bytes, size_t want) {
  if (want <= *bytes) return WRNN_OK;
  if (*buf) cudaFree(*buf);
  *buf = nullptr; *bytes = 0;
  WRNN_CUDA_OK(cudaMalloc(buf, want));
  *bytes = want;
  return WRNN_OK;
}

// grow for a pinned host buffer mapped into the device's address space; *dev is its device alias.
static int grow_mapped(void** host, void** dev, size_t* bytes, size_t want) {
  if (want <= *bytes) return WRNN_OK;
  if (*host) cudaFreeHost(*host);
  *host = *dev = nullptr; *bytes = 0;
  WRNN_CUDA_OK(cudaHostAlloc(host, want, cudaHostAllocMapped));
  WRNN_CUDA_OK(cudaHostGetDevicePointer(dev, *host, 0));
  *bytes = want;
  return WRNN_OK;
}

// Staging of the handle's host-memory entry points (place / copy_back, wrnn_engine.h) in its one device staging buffer,
// grown as needed.  unstage, their common end, copies the results back, synchronises and returns the engine's check().
static int stage(wrnn_t* h, const std::vector<Staged>& items, cudaStream_t st, std::vector<void*>& dev) {
  WRNN_CUDA_OK(cudaSetDevice(h->engine->device));
  const int rc = grow(&h->d_stage, &h->stage_bytes, staged_bytes(items));
  if (rc != WRNN_OK) return rc;
  return place(h->d_stage, items, st, dev);
}

static int unstage(wrnn_t* h, const std::vector<Unstaged>& items) {
  const int rc = copy_back(items);
  return rc != WRNN_OK ? rc : h->last->check();
}

// The host epilogue's tables (wrnn_vocode's geometry: unbatched with overlap 0, else batched): mu is empty unless mu-law
// applies, which it does on a RAW head only.
struct LiveTables {
  std::vector<double> mu, tail, fade_in, fade_out;
  long long tail_len = 0;
  int n_classes = 0, overlap = 0;
};
static LiveTables live_tables(int mode, bool mu_law, int n_classes, int hop, int overlap = 0) {
  LiveTables t;
  cond::epilogue_tables(overlap, mu_law && mode == WRNN_MODE_RAW, n_classes, hop, t.fade_in, t.fade_out, t.mu, t.tail);
  t.tail_len = 20ll * hop;
  t.n_classes = n_classes;
  t.overlap = overlap;
  return t;
}

// A live job: wrnn_vocode_live_start's one utterance or wrnn_vocode_many_live_start's n, utterance i being fold i.  The
// pinned buffer is mapped into the device's address space: one progress word per fold (the samples of that fold stored
// so far, published by the kernel), padded to 512 B, then the fp32 samples [n][steps] the kernel's sample store writes.
// The host reads both in place.
struct LiveJob {
  static constexpr int MAX_UTTS = 64;   // one persistent tile
  static constexpr size_t SAMPLES_OFF = MAX_UTTS * sizeof(unsigned long long);
  void* host = nullptr;                 // pinned and mapped (grow_mapped)
  void* dev = nullptr;                  // its device alias
  size_t bytes = 0;
  cudaEvent_t done = nullptr;           // recorded after the kernel
  Engine* e = nullptr;
  bool many = false;                    // started by wrnn_vocode_many_live_start (served by its poll only)
  long long steps = 0;                  // samples per fold (the row pitch of the sample block)
  LiveTables tabs;
  std::vector<double*> wav;             // per utterance: the caller's [wave_len[i]]
  std::vector<long long> wave_len, delivered;
  int n() const { return (int)wav.size(); }
  unsigned long long progress(int i) const {
    return __atomic_load_n(static_cast<const unsigned long long*>(host) + i, __ATOMIC_ACQUIRE);
  }
  const float* samples(int i) const {
    return reinterpret_cast<const float*>(static_cast<const char*>(host) + SAMPLES_OFF) + (size_t)i * steps;
  }
};

int idle_or_busy(const wrnn_handle* h) {
  if (h && h->session) {
    set_error("a live session is open on this handle: wrnn_live_close it first");
    return WRNN_E_BUSY;
  }
  if (h && h->live_busy) {
    set_error(std::string("a live job is in flight on this handle: ") +
              (h->live->many ? "wrnn_vocode_many_live_poll" : "wrnn_vocode_live_poll") + " until it returns 0 or an error");
    return WRNN_E_BUSY;
  }
  return WRNN_OK;
}
}  // namespace wrnn

using namespace wrnn;

extern "C" {

int wrnn_abi_version(void) { return WRNN_ABI_VERSION; }
const char* wrnn_last_error(void) { return g_last_error.c_str(); }

int wrnn_create(wrnn_t** out, const wrnn_cfg* cfg, const wrnn_weights* w, int device) {
  if (!out || !cfg || !w) { set_error("null argument"); return WRNN_E_INVALID; }
  *out = nullptr;
  if (cfg->rnn_dims != H || cfg->fc_dims != H || cfg->feat_dims != FEAT || cfg->aux_dims != AUXD) {
    set_error("unsupported dims: the kernels are specialised for rnn_dims=fc_dims=512, feat_dims=80, "
              "aux_dims=32 (hparams.py:46-50)");
    return WRNN_E_INVALID;
  }
  if (cfg->mode != WRNN_MODE_MOL && cfg->mode != WRNN_MODE_RAW) { set_error("Unknown model mode value"); return WRNN_E_INVALID; }
  if (cfg->n_classes <= 0) { set_error("n_classes must be positive"); return WRNN_E_INVALID; }
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || device < 0 || device >= n_dev) {
    cudaGetLastError();
    set_error("no CUDA device: wavernn_b200 has no CPU fallback");
    return WRNN_E_NO_DEVICE;
  }
  WRNN_CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  WRNN_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {         // only an sm_90a cubin is built (wgmma and TMA of Hopper)
    set_error(std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major * 10 + prop.minor) +
              "; this library is built for sm_90a only");
    return WRNN_E_NO_DEVICE;
  }
  HostWeights hw;
  int rc = read_weights(*cfg, *w, false, hw);
  if (rc != WRNN_OK) return rc;
  Engine* eng = nullptr;
  int engine = cfg->engine;
  if (cfg->precision == WRNN_PREC_FP32) {
    if (engine == WRNN_ENGINE_TCGEN05) { set_error("fp32 strict arithmetic is served by the SIMT engine only"); return WRNN_E_INVALID; }
    engine = WRNN_ENGINE_SIMT;
  }
  if (engine == WRNN_ENGINE_AUTO) engine = WRNN_ENGINE_TCGEN05;
  if (engine == WRNN_ENGINE_STREAM) {
    rc = make_stream_engine(*cfg, hw, device, &eng);
  } else if (engine == WRNN_ENGINE_TCGEN05) {
    rc = make_tc_engine(*cfg, hw, device, &eng);
    if (rc != WRNN_OK && cfg->engine == WRNN_ENGINE_AUTO && rc == WRNN_E_INVALID) {
      // configuration outside the tensor-core engine's envelope: AUTO may pick the SIMT engine
      rc = make_simt_engine(*cfg, hw, device, &eng);
    }
  } else {
    rc = make_simt_engine(*cfg, hw, device, &eng);
  }
  if (rc != WRNN_OK) return rc;
  wrnn_handle* h = new (std::nothrow) wrnn_handle();
  if (!h) { delete eng; set_error("out of host memory"); return WRNN_E_INVALID; }
  h->engine = eng;
  h->last = eng;
  h->auto_engine = (cfg->engine == WRNN_ENGINE_AUTO);
  if (h->auto_engine && engine == WRNN_ENGINE_TCGEN05) h->host_weights = new HostWeights(hw);   // for a lazy SIMT fallback
  *out = h;
  return WRNN_OK;
}

// Folds from which ENGINE_AUTO hands a job to the stream engine: the persistent engine serves tiles of 64 folds one
// after the other, the stream engine all tiles at once.  Measured on an H100 SXM (400 W limit), end to end: a persistent
// tile costs ~15.5 us per step, the stream engine's cluster form ~64 us per step for up to a few hundred folds, so the
// stream engine wins from the fifth tile on.  WRNN_STREAM_MIN_FOLDS overrides (experiments).
static int stream_min_folds() {
  static const int v = [] { const char* e = getenv("WRNN_STREAM_MIN_FOLDS"); return e ? atoi(e) : 4 * 64 + 1; }();
  return v;
}

// ENGINE_AUTO: many-fold MoL jobs go to the stream engine; jobs outside the tensor-core engine's envelope go to the
// SIMT engine (same arithmetic contract).
static int pick_engine(wrnn_t* h, const wrnn_job* job, Engine** out) {
  if (h->auto_engine && h->host_weights && job->n_seg >= stream_min_folds() && h->engine->cfg.mode == WRNN_MODE_MOL &&
      h->engine->cfg.n_classes == 30 && h->engine->cfg.precision != WRNN_PREC_FP32 && !h->stream_failed) {
    if (!h->stream) {
      const int rc = make_stream_engine(h->engine->cfg, *h->host_weights, h->engine->device, &h->stream);
      if (rc != WRNN_OK) h->stream_failed = true;
    }
    if (h->stream && h->stream->supports(*job)) { *out = h->stream; return WRNN_OK; }
  }
  if (h->engine->supports(*job)) { *out = h->engine; return WRNN_OK; }
  if (!h->auto_engine || !h->host_weights) {
    set_error(std::string("job is outside the envelope of engine '") + h->engine->name() + "'");
    return WRNN_E_INVALID;
  }
  if (!h->fallback) {
    int rc = make_simt_engine(h->engine->cfg, *h->host_weights, h->engine->device, &h->fallback);
    if (rc != WRNN_OK) return rc;
  }
  *out = h->fallback;
  return WRNN_OK;
}

void wrnn_destroy(wrnn_t* h) {
  if (!h) return;
  if (h->session) wrnn_live_close(h);                  // cancels every ticket and waits for the kernel
  if (h->live) {                                       // a live job still in flight finishes first
    if (h->live->done) {
      cudaSetDevice(h->engine->device);
      cudaEventSynchronize(h->live->done);
      cudaEventDestroy(h->live->done);
    }
    if (h->live->host) cudaFreeHost(h->live->host);
    delete h->live;
  }
  if (h->d_stage) cudaFree(h->d_stage);
  if (h->d_audio) cudaFree(h->d_audio);
  delete h->engine;
  delete h->fallback;
  delete h->stream;
  delete h->host_weights;
  destroy_upsampler(h->upsampler);
  delete h;
}

static int validate(const wrnn_t* h, const wrnn_job* job, bool host, bool score = false) {
  if (!h || !h->engine || !job) { set_error("null handle or job"); return WRNN_E_INVALID; }
  if (!job->out && !score) { set_error("out is required"); return WRNN_E_INVALID; }
  if (job->mel_frames) {
    if (!job->aux_frames || !job->up_taps || job->hop <= 0) { set_error("mel_frames needs aux_frames, up_taps and hop"); return WRNN_E_INVALID; }
    if (host) { set_error("frame-rate conditioning is a device-pointer feature (use wrnn_generate)"); return WRNN_E_INVALID; }
    if (job->cond_mode < WRNN_COND_AUTO || job->cond_mode > WRNN_COND_IN_KERNEL) { set_error("cond_mode must be a WRNN_COND_* value"); return WRNN_E_INVALID; }
    if (job->cond_mode == WRNN_COND_EXPAND && job->fold_row0) { set_error("WRNN_COND_EXPAND needs strided folds (no fold tables)"); return WRNN_E_INVALID; }
    if (job->L >= (1ll << 31)) { set_error("frame-rate conditioning: stream longer than 2^31 samples"); return WRNN_E_INVALID; }
  } else if (!job->mels_up || !job->aux) { set_error("mels_up and aux (or mel_frames / aux_frames / up_taps) are required"); return WRNN_E_INVALID; }
  if (job->n_seg <= 0 || job->seg_len <= 0 || job->L <= 0 || job->seg_stride <= 0) {
    set_error("n_seg, seg_len, L and seg_stride must be positive"); return WRNN_E_INVALID;
  }
  if (job->steps < 0 || job->steps > job->seg_len) { set_error("steps must be in [0, seg_len]"); return WRNN_E_INVALID; }
  if ((job->fold_row0 == nullptr) != (job->fold_row_end == nullptr)) { set_error("fold_row0 and fold_row_end go together"); return WRNN_E_INVALID; }
  if (job->uniforms_ready && (!job->uniforms || host)) { set_error("uniforms_ready needs device `uniforms` (wrnn_generate)"); return WRNN_E_INVALID; }
  (void)host;
  return WRNN_OK;
}

int wrnn_generate(wrnn_t* h, const wrnn_job* job, void* stream) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate(h, job, false);
  if (rc != WRNN_OK) return rc;
  Engine* e = nullptr;
  if ((rc = pick_engine(h, job, &e)) != WRNN_OK) return rc;
  h->last = e;
  return e->generate(*job, static_cast<cudaStream_t>(stream), nullptr);
}

static const char* kNoRawStreamScore = "the stream engine scores the MoL head only (RAW scoring runs on the persistent or SIMT engine)";

int wrnn_score(wrnn_t* h, const wrnn_job* job, float* nll, void* stream) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate(h, job, false, true);
  if (rc != WRNN_OK) return rc;
  if (!job->x_force || !nll) { set_error("wrnn_score needs x_force (the targets) and nll"); return WRNN_E_INVALID; }
  Engine* e = nullptr;
  if ((rc = pick_engine(h, job, &e)) != WRNN_OK) return rc;
  if (!e->scores()) { set_error(kNoRawStreamScore); return WRNN_E_INVALID; }
  h->last = e;
  return e->score(*job, nll, static_cast<cudaStream_t>(stream), nullptr);
}

int wrnn_check(wrnn_t* h) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (h->live_busy || h->session) return idle_or_busy(h);
  return h->last->check();
}

int wrnn_generate_host(wrnn_t* h, const wrnn_job* job) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate(h, job, true);
  if (rc != WRNN_OK) return rc;
  Engine* e = nullptr;
  if ((rc = pick_engine(h, job, &e)) != WRNN_OK) return rc;
  h->last = e;
  const size_t S = job->steps > 0 ? job->steps : job->seg_len;
  const size_t B = job->n_seg, NC = e->cfg.n_classes, F = sizeof(float);
  const size_t b_tab = job->fold_row0 ? B * sizeof(int64_t) : 0, b_out = B * S * F, b_log = job->logits_out ? S * B * NC * F : 0;
  std::vector<void*> d;
  rc = stage(h, {{job->mels_up, (size_t)job->L * FEAT * F}, {job->aux, (size_t)job->L * 4 * AUXD * F},
                 {job->uniforms, job->uniforms ? S * 11 * B * F : 0}, {job->expo, job->expo ? S * B * NC * F : 0},
                 {job->x_force, job->x_force ? S * B * F : 0}, {job->fold_row0, b_tab}, {job->fold_row_end, b_tab},
                 {nullptr, b_out}, {nullptr, b_log}},
             0, d);
  if (rc != WRNN_OK) return rc;
  wrnn_job dj = *job;
  dj.mels_up = static_cast<float*>(d[0]); dj.aux = static_cast<float*>(d[1]);
  dj.uniforms = static_cast<float*>(d[2]); dj.expo = static_cast<float*>(d[3]); dj.x_force = static_cast<float*>(d[4]);
  dj.fold_row0 = static_cast<int64_t*>(d[5]); dj.fold_row_end = static_cast<int64_t*>(d[6]);
  dj.out = static_cast<float*>(d[7]); dj.logits_out = static_cast<float*>(d[8]);
  if ((rc = e->generate(dj, 0, nullptr)) != WRNN_OK) return rc;
  return unstage(h, {{job->out, dj.out, b_out}, {job->logits_out, dj.logits_out, b_log}});
}

const char* wrnn_engine_name(const wrnn_t* h) { return (h && h->last) ? h->last->name() : ""; }
int wrnn_grid_ctas(const wrnn_t* h) { return (h && h->last) ? h->last->grid_ctas() : 0; }
int64_t wrnn_launch_count(const wrnn_t* h) {
  return (h && h->engine) ? h->engine->launches + (h->fallback ? h->fallback->launches : 0) + (h->stream ? h->stream->launches : 0) : 0;
}

int wrnn_expand_conditioning(const float* mel_frames, const float* aux_frames, const float* up_taps, int32_t hop, int64_t row_lo,
                             int64_t n_rows, float* mels_up, float* aux, void* stream) {
  if (!mel_frames || !aux_frames || !up_taps || !mels_up || !aux || hop <= 0 || row_lo < 0 || n_rows <= 0 ||
      row_lo + n_rows >= (1ll << 31)) {
    set_error("wrnn_expand_conditioning: bad argument");
    return WRNN_E_INVALID;
  }
  return expand_conditioning(mel_frames, aux_frames, up_taps, hop, row_lo, n_rows, mels_up, aux, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// wrnn_vocode: generate(gen_rng='philox') restated -- the frame-rate branch of WaveRNN._run_segments and the device branch
// of WaveRNN._finish, with the conditioning network of wrnn_cond.cu in place of torch's.
// ---------------------------------------------------------------------------------------------------------------------
static int validate_vocode(const wrnn_t* h, const wrnn_vocode_job* job) {
  if (!h || !h->engine || !job) { set_error("null handle or job"); return WRNN_E_INVALID; }
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  const int rc = check_utterance("", job->mel, job->wav, job->T);
  if (rc != WRNN_OK) return rc;
  if (job->T * h->upsampler->hop >= (1ll << 31)) { set_error("stream longer than 2^31 samples"); return WRNN_E_INVALID; }
  if (job->batched && (job->target <= 0 || job->overlap <= 0)) {
    set_error("a batched job needs target > 0 and overlap > 0"); return WRNN_E_INVALID;
  }
  return WRNN_OK;
}

static size_t align_floats(size_t n) { return (n + 63) & ~size_t(63); }   // 256-byte aligned regions

// The engine of a vocode job (frame-rate conditioning).  The SIMT engine takes per-sample rows: pick_engine refuses the
// frame-rate job on a handle that has no other engine, and *expanded tells the caller to expand the rows into scratch.
static int pick_vocode_engine(wrnn_t* h, wrnn_job& j, Engine** e, bool* expanded) {
  const void* tag = h->upsampler;                      // placeholders: only tested against NULL
  j.mel_frames = j.aux_frames = j.up_taps = static_cast<const float*>(tag);
  *expanded = pick_engine(h, &j, e) != WRNN_OK;
  if (!*expanded) return WRNN_OK;
  j.mel_frames = j.aux_frames = j.up_taps = nullptr;
  j.mels_up = j.aux = static_cast<const float*>(tag);
  return pick_engine(h, &j, e);
}

// Scratch floats of the expanded rows of a stream of L rows.
static size_t rows_floats(long long L) { return align_floats((size_t)L * FEAT) + align_floats((size_t)L * 4 * AUXD); }

// The conditioning of job j: the frames, or on an engine that takes per-sample rows (expanded), rows [0, n_rows) of the
// stream of L rows expanded into `rows` (rows_floats(L) of scratch), enqueued on st.
static int frames_or_rows(const Upsampler& u, float* mel_frames, float* aux_frames, bool expanded, long long L,
                          long long n_rows, float* rows, cudaStream_t st, wrnn_job& j) {
  if (!expanded) {
    j.mel_frames = mel_frames; j.aux_frames = aux_frames; j.up_taps = u.d_taps;
    return WRNN_OK;
  }
  j.mels_up = rows; j.aux = rows + align_floats((size_t)L * FEAT);
  return expand_conditioning(mel_frames, aux_frames, u.d_taps, u.hop, 0, n_rows, rows, rows + align_floats((size_t)L * FEAT), st);
}

// fade_in / fade_out / mu / tail of the epilogue on the device, rebuilt and uploaded only when (overlap, mu_law,
// n_classes) changes.  mu-law applies to a RAW head only.
struct EpTables { const double *fade_in, *fade_out, *mu, *tail; };
static int epilogue_tables(wrnn_t* h, int ov, int mu_law_flag, cudaStream_t st, EpTables* t) {
  Upsampler& u = *h->upsampler;
  const int nc = h->engine->cfg.n_classes;
  const bool mu_law = mu_law_flag && h->engine->cfg.mode == WRNN_MODE_RAW;
  if (u.tabs_key[0] != ov || u.tabs_key[1] != (mu_law ? 1 : 0) || u.tabs_key[2] != nc) {
    u.tabs_key[0] = u.tabs_key[1] = u.tabs_key[2] = -1;
    std::vector<double> fi, fo, mu, tail;
    cond::epilogue_tables(ov, mu_law, nc, u.hop, fi, fo, mu, tail);
    u.host_tabs.clear();
    for (const auto* v : {&fi, &fo, &mu, &tail}) u.host_tabs.insert(u.host_tabs.end(), v->begin(), v->end());
    if (u.host_tabs.size() > u.tabs_len) {
      if (u.d_tabs) cudaFree(u.d_tabs);
      u.d_tabs = nullptr; u.tabs_len = 0;
      WRNN_CUDA_OK(cudaMalloc(&u.d_tabs, u.host_tabs.size() * sizeof(double)));
      u.tabs_len = u.host_tabs.size();
    }
    WRNN_CUDA_OK(cudaMemcpyAsync(u.d_tabs, u.host_tabs.data(), u.host_tabs.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    u.tabs_key[0] = ov; u.tabs_key[1] = mu_law ? 1 : 0; u.tabs_key[2] = nc;
  }
  t->fade_in = ov ? u.d_tabs : nullptr;
  t->fade_out = ov ? u.d_tabs + ov : nullptr;
  t->mu = mu_law ? u.d_tabs + 2 * ov : nullptr;
  t->tail = u.d_tabs + 2 * ov + (mu_law ? nc : 0);
  return WRNN_OK;
}

// The job of wrnn_vocode or wrnn_vocode_many up to the engine launch: fold geometry, the engine, scratch, the epilogue
// tables (not for a live job, whose epilogue runs on the host) and the conditioning frames (or the expanded rows of a
// SIMT engine), enqueued on st.  j.out is the sample block in scratch.  wrnn_vocode_many's job also has per-fold Philox
// keys and the utterance table of its epilogue, both in scratch.
struct VocodeJob {
  cond::Geometry g;
  wrnn_job j;
  Engine* e = nullptr;
  EpTables tabs{};
  const FoldKey* keys = nullptr;
  const EpUtt* eu = nullptr;
};

static int vocode_job(wrnn_t* h, const wrnn_vocode_job* job, cudaStream_t st, VocodeJob* v) {
  Upsampler& u = *h->upsampler;
  const int hop = u.hop;
  const long long T = job->T, L = T * hop;
  const cond::Geometry g = cond::fold_geometry(L, job->batched != 0, job->target, job->overlap);
  if (g.n_seg < 1 || g.n_seg >= (1ll << 31) || g.seg_len >= (1ll << 31)) {
    set_error("target / overlap give no fold, or folds beyond 2^31"); return WRNN_E_INVALID;
  }
  WRNN_CUDA_OK(cudaSetDevice(h->engine->device));

  wrnn_job& j = v->j;
  std::memset(&j, 0, sizeof(j));
  j.L = L; j.seg_stride = g.seg_stride; j.n_seg = (int32_t)g.n_seg; j.seg_len = (int32_t)g.seg_len;
  j.philox_seed = job->philox_seed;
  j.hop = hop; j.cond_mode = WRNN_COND_AUTO;
  Engine* e = nullptr;
  bool expanded = false;
  int rc = pick_vocode_engine(h, j, &e, &expanded);
  if (rc != WRNN_OK) return rc;

  const size_t n_mf = align_floats((size_t)(T + 4) * FEAT), n_af = align_floats((size_t)T * cond::CD);
  const size_t n_smp = align_floats((size_t)g.n_seg * g.seg_len);
  rc = grow(&u.d_scratch, &u.scratch_bytes, (n_mf + n_af + n_smp + (expanded ? rows_floats(L) : 0)) * sizeof(float));
  if (rc != WRNN_OK) return rc;
  float* mel_frames = static_cast<float*>(u.d_scratch);
  float* aux_frames = mel_frames + n_mf;
  float* samples = aux_frames + n_af;

  if ((rc = epilogue_tables(h, (int)g.overlap, job->mu_law, st, &v->tabs)) != WRNN_OK) return rc;
  if ((rc = conditioning_frames(u, job->mel, T, mel_frames, aux_frames, nullptr, st)) != WRNN_OK) return rc;
  if ((rc = frames_or_rows(u, mel_frames, aux_frames, expanded, L, L, samples + n_smp, st, j)) != WRNN_OK) return rc;
  j.out = samples;
  v->g = g;
  v->e = e;
  h->last = e;
  return WRNN_OK;
}

static int vocode(wrnn_t* h, const wrnn_vocode_job* job, cudaStream_t st) {
  VocodeJob v;
  int rc = vocode_job(h, job, st, &v);
  if (rc != WRNN_OK) return rc;
  const wrnn_job& j = v.j;
  const int hop = h->upsampler->hop;
  if ((rc = v.e->generate(j, st, nullptr)) != WRNN_OK) return rc;
  return wrnn_epilogue(j.out, j.n_seg, j.seg_len, j.seg_stride, (int)v.g.overlap, v.tabs.fade_in, v.tabs.fade_out, v.tabs.mu,
                       h->engine->cfg.n_classes, v.tabs.tail, 20ll * hop, (job->T - 1) * hop, job->wav, st);
}

// The job of a batch laid out by cond::batch_plan or cond::score_plan (mels[i]: utterance i's DEVICE mel), up to what
// its caller adds: the fold tables, the engine, scratch and the conditioning frames (or the expanded rows of a SIMT
// engine), enqueued on st.  Scratch: [row0 | row_end | CondUtt table | the caller's table (tab_bytes) | mel_frames |
// aux_frames | the caller's regions (n_floats) | expanded rows].  The frame regions span every utterance's T + 4 frames
// (aux_frames included, so that no row of the laid-out stream maps outside them).  Once the engine e is picked,
// fill(e, tab) refuses it (returning its code, message set) or writes the caller's table into the host image at tab;
// the tables then go up in one copy.
struct BatchJob {
  wrnn_job j;                          // fold tables and conditioning set; out and x_force are the caller's
  Engine* e = nullptr;
  const unsigned char* tab = nullptr;  // the caller's table (device)
  float* regions = nullptr;            // the caller's regions (device)
};

template <class Fill>
static int batch_job(wrnn_t* h, const cond::BatchPlan& pl, const float* const* mels, size_t tab_bytes, size_t n_floats,
                     cudaStream_t st, BatchJob* bj, Fill fill) {
  Upsampler& u = *h->upsampler;
  const int n = (int)pl.frame0.size() - 1;
  const size_t nf = (size_t)pl.g.n_seg;
  WRNN_CUDA_OK(cudaSetDevice(h->engine->device));

  wrnn_job& j = bj->j;
  std::memset(&j, 0, sizeof(j));
  j.L = pl.L; j.seg_stride = pl.g.seg_stride; j.n_seg = (int32_t)nf; j.seg_len = (int32_t)pl.g.seg_len;
  j.hop = u.hop; j.cond_mode = WRNN_COND_AUTO;
  const void* tag = h->upsampler;                      // placeholders: only tested against NULL
  j.fold_row0 = j.fold_row_end = static_cast<const int64_t*>(tag);
  bool expanded = false;
  int rc = pick_vocode_engine(h, j, &bj->e, &expanded);
  if (rc != WRNN_OK) return rc;

  const size_t b_row = align256(nf * sizeof(int64_t)), b_cu = align256(n * sizeof(CondUtt));
  const size_t o_tab = 2 * b_row + b_cu, b_tab = o_tab + align256(tab_bytes);
  u.host_plan.assign(b_tab, 0);
  unsigned char* hp = u.host_plan.data();
  if ((rc = fill(*bj->e, hp + o_tab)) != WRNN_OK) return rc;
  std::memcpy(hp, pl.row0.data(), nf * sizeof(int64_t));
  std::memcpy(hp + b_row, pl.row_end.data(), nf * sizeof(int64_t));
  CondUtt* cu = reinterpret_cast<CondUtt*>(hp + 2 * b_row);
  for (int i = 0; i < n; ++i) cu[i] = CondUtt{mels[i], pl.frame0[i + 1] - pl.frame0[i] - 4, pl.frame0[i]};

  const size_t n_frames = (size_t)pl.frame0.back();
  const size_t n_mf = align_floats(n_frames * FEAT), n_af = align_floats(n_frames * cond::CD);
  rc = grow(&u.d_scratch, &u.scratch_bytes, b_tab + (n_mf + n_af + n_floats + (expanded ? rows_floats(pl.L) : 0)) * sizeof(float));
  if (rc != WRNN_OK) return rc;
  unsigned char* d = static_cast<unsigned char*>(u.d_scratch);
  float* mel_frames = reinterpret_cast<float*>(d + b_tab);
  float* aux_frames = mel_frames + n_mf;
  bj->regions = aux_frames + n_af;
  WRNN_CUDA_OK(cudaMemcpyAsync(d, hp, b_tab, cudaMemcpyHostToDevice, st));
  j.fold_row0 = reinterpret_cast<const int64_t*>(d);
  j.fold_row_end = reinterpret_cast<const int64_t*>(d + b_row);
  bj->tab = d + o_tab;

  const CondUtt* d_cu = reinterpret_cast<const CondUtt*>(d + 2 * b_row);
  if ((rc = conditioning_frames_batch(u, d_cu, n, pl.max_T, mel_frames, aux_frames, st)) != WRNN_OK) return rc;
  // rows [0, L - 4*hop): the last utterance's 4*hop gap rows would read frames past the end and no fold reads them
  rc = frames_or_rows(u, mel_frames, aux_frames, expanded, pl.L, pl.L - 4ll * u.hop, bj->regions + n_floats, st, j);
  if (rc != WRNN_OK) return rc;
  h->last = bj->e;
  return WRNN_OK;
}

// wrnn_vocode_many's job (layout: cond::batch_plan): batch_job with the per-fold Philox keys and the epilogue's
// utterance table as its table and the sample block as its region.  A live job refuses an engine without live
// vocoding and has no device epilogue.  `b` holds DEVICE mel pointers (and DEVICE wav pointers unless live).
static int vocode_many_job(wrnn_t* h, const wrnn_vocode_batch* b, const cond::BatchPlan& pl, cudaStream_t st, bool live,
                           VocodeJob* v) {
  const int hop = h->upsampler->hop, n = b->n_utts;
  const size_t nf = (size_t)pl.g.n_seg, b_key = align256(nf * sizeof(FoldKey));
  std::vector<const float*> mels(n);
  for (int i = 0; i < n; ++i) mels[i] = b->utts[i].mel;
  BatchJob bj;
  int rc = batch_job(h, pl, mels.data(), b_key + n * sizeof(EpUtt), align_floats(nf * pl.g.seg_len), st, &bj,
                     [&](const Engine& e, unsigned char* tab) -> int {
                       if (live && e.live_refusal()) { set_error(e.live_refusal()); return WRNN_E_INVALID; }
                       std::memcpy(tab, pl.keys.data(), nf * sizeof(FoldKey));
                       EpUtt* eu = reinterpret_cast<EpUtt*>(tab + b_key);
                       for (int i = 0; i < n; ++i)
                         eu[i] = EpUtt{pl.fold0[i], (int)(pl.fold0[i + 1] - pl.fold0[i]), (b->utts[i].T - 1) * hop, b->utts[i].wav};
                       return WRNN_OK;
                     });
  if (rc != WRNN_OK) return rc;
  v->j = bj.j;
  v->j.out = bj.regions;
  v->g = pl.g;
  v->e = bj.e;
  v->keys = reinterpret_cast<const FoldKey*>(bj.tab);
  v->eu = reinterpret_cast<const EpUtt*>(bj.tab + b_key);
  return live ? WRNN_OK : epilogue_tables(h, (int)pl.g.overlap, b->mu_law, st, &v->tabs);
}

static int vocode_many(wrnn_t* h, const wrnn_vocode_batch* b, const cond::BatchPlan& pl, cudaStream_t st) {
  VocodeJob v;
  int rc = vocode_many_job(h, b, pl, st, false, &v);
  if (rc != WRNN_OK) return rc;
  const wrnn_job& j = v.j;
  if ((rc = v.e->generate(j, st, v.keys)) != WRNN_OK) return rc;
  return epilogue_launch(j.out, j.seg_len, j.seg_stride, (int)v.g.overlap, v.tabs.fade_in, v.tabs.fade_out, v.tabs.mu,
                         h->engine->cfg.n_classes, v.tabs.tail, 20ll * h->upsampler->hop, v.eu, EpUtt{0, 0, 0, nullptr},
                         b->n_utts, pl.max_wave, st);
}

// wrnn_score_many: each utterance one fold (layout: cond::score_plan).  Its samples are gathered into the x_force block
// of the job ([steps][n_utts], zeros past n_i) and its losses scattered back from the nll block, one launch each.
struct ScoreUtt {
  const float* x;
  float* nll;
  long long n;
};
__global__ void score_gather_kernel(const ScoreUtt* __restrict__ u, int n_utts, long long steps, float* __restrict__ xf) {
  const long long total = steps * n_utts;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / n_utts;
    const int b = (int)(i - t * n_utts);
    xf[i] = t < u[b].n ? __ldg(u[b].x + t) : 0.f;
  }
}
__global__ void score_scatter_kernel(const ScoreUtt* __restrict__ u, int n_utts, long long steps, const float* __restrict__ nl) {
  const long long total = steps * n_utts;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / n_utts;
    const int b = (int)(i - t * n_utts);
    if (t < u[b].n) u[b].nll[t] = __ldcg(nl + i);
  }
}

static int score_many(wrnn_t* h, const wrnn_score_utt* utts, int n, const cond::BatchPlan& pl, cudaStream_t st) {
  const long long steps = pl.g.seg_len;
  const size_t n_xf = align_floats((size_t)steps * n);
  std::vector<const float*> mels(n);
  for (int i = 0; i < n; ++i) mels[i] = utts[i].mel;
  BatchJob bj;
  int rc = batch_job(h, pl, mels.data(), n * sizeof(ScoreUtt), 2 * n_xf, st, &bj, [&](const Engine& e, unsigned char* tab) -> int {
    if (!e.scores()) { set_error(kNoRawStreamScore); return WRNN_E_INVALID; }
    ScoreUtt* su = reinterpret_cast<ScoreUtt*>(tab);
    for (int i = 0; i < n; ++i) su[i] = ScoreUtt{utts[i].x, utts[i].nll, utts[i].n};
    return WRNN_OK;
  });
  if (rc != WRNN_OK) return rc;
  // regions: [x_force | nll]
  const ScoreUtt* d_su = reinterpret_cast<const ScoreUtt*>(bj.tab);
  float* xf = bj.regions;
  float* nl = xf + n_xf;
  const int grid = grid_stride_blocks((steps * n + 255) / 256);
  score_gather_kernel<<<grid, 256, 0, st>>>(d_su, n, steps, xf);
  WRNN_CUDA_OK(cudaGetLastError());
  bj.j.x_force = xf;
  if ((rc = bj.e->score(bj.j, nl, st, nullptr)) != WRNN_OK) return rc;
  score_scatter_kernel<<<grid, 256, 0, st>>>(d_su, n, steps, nl);
  WRNN_CUDA_OK(cudaGetLastError());
  return WRNN_OK;
}

static int validate_score_many(const wrnn_t* h, const wrnn_score_utt* utts, int n, cond::BatchPlan& pl) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  if (!h->engine->scores()) { set_error(kNoRawStreamScore); return WRNN_E_INVALID; }
  return cond::score_plan(h->upsampler->hop, utts, n, pl);
}

static int validate_many(const wrnn_t* h, const wrnn_vocode_batch* b, cond::BatchPlan& pl) {
  if (!h || !h->engine || !b) { set_error("null handle or batch"); return WRNN_E_INVALID; }
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  return cond::batch_plan(h->upsampler->hop, *b, pl);
}

extern "C" {

int wrnn_vocode(wrnn_t* h, const wrnn_vocode_job* job, void* stream) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_vocode(h, job);
  if (rc != WRNN_OK) return rc;
  return vocode(h, job, static_cast<cudaStream_t>(stream));
}

int wrnn_vocode_host(wrnn_t* h, const wrnn_vocode_job* job) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_vocode(h, job);
  if (rc != WRNN_OK) return rc;
  const size_t b_wav = (size_t)(job->T - 1) * h->upsampler->hop * sizeof(double);
  std::vector<void*> d;
  if ((rc = stage(h, {{job->mel, (size_t)job->T * FEAT * sizeof(float)}, {nullptr, b_wav}}, 0, d)) != WRNN_OK) return rc;
  wrnn_vocode_job dj = *job;
  dj.mel = static_cast<float*>(d[0]); dj.wav = static_cast<double*>(d[1]);
  if ((rc = vocode(h, &dj, 0)) != WRNN_OK) return rc;
  return unstage(h, {{job->wav, dj.wav, b_wav}});
}

int wrnn_vocode_many(wrnn_t* h, const wrnn_vocode_batch* b, void* stream) {
  cond::BatchPlan pl;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_many(h, b, pl);
  if (rc != WRNN_OK) return rc;
  return vocode_many(h, b, pl, static_cast<cudaStream_t>(stream));
}

int wrnn_vocode_many_host(wrnn_t* h, const wrnn_vocode_batch* b) {
  cond::BatchPlan pl;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_many(h, b, pl);
  if (rc != WRNN_OK) return rc;
  const int n = b->n_utts;
  std::vector<Staged> in(2 * n);                       // [mels | waveforms]
  for (int i = 0; i < n; ++i) {
    in[i] = {b->utts[i].mel, (size_t)b->utts[i].T * FEAT * sizeof(float)};
    in[n + i] = {nullptr, (size_t)(pl.wav0[i + 1] - pl.wav0[i]) * sizeof(double)};
  }
  std::vector<void*> d;
  if ((rc = stage(h, in, 0, d)) != WRNN_OK) return rc;
  std::vector<wrnn_utterance> du(b->utts, b->utts + n);
  std::vector<Unstaged> out(n);
  for (int i = 0; i < n; ++i) {
    du[i].mel = static_cast<float*>(d[i]);
    du[i].wav = static_cast<double*>(d[n + i]);
    out[i] = {b->utts[i].wav, d[n + i], in[n + i].bytes};
  }
  wrnn_vocode_batch db = *b;
  db.utts = du.data();
  if ((rc = vocode_many(h, &db, pl, 0)) != WRNN_OK) return rc;
  return unstage(h, out);
}

int wrnn_score_many(wrnn_t* h, const wrnn_score_utt* utts, int32_t n_utts, void* stream) {
  cond::BatchPlan pl;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_score_many(h, utts, n_utts, pl);
  if (rc != WRNN_OK) return rc;
  return score_many(h, utts, n_utts, pl, static_cast<cudaStream_t>(stream));
}

int wrnn_score_many_host(wrnn_t* h, const wrnn_score_utt* utts, int32_t n_utts) {
  cond::BatchPlan pl;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  rc = validate_score_many(h, utts, n_utts, pl);
  if (rc != WRNN_OK) return rc;
  const int n = n_utts;
  std::vector<Staged> in(3 * n);                       // [mels | waveforms | losses]
  for (int i = 0; i < n; ++i) {
    in[i] = {utts[i].mel, (size_t)utts[i].T * FEAT * sizeof(float)};
    in[n + i] = {utts[i].x, (size_t)utts[i].n * sizeof(float)};
    in[2 * n + i] = {nullptr, (size_t)utts[i].n * sizeof(float)};
  }
  std::vector<void*> d;
  if ((rc = stage(h, in, 0, d)) != WRNN_OK) return rc;
  std::vector<wrnn_score_utt> du(utts, utts + n);
  std::vector<Unstaged> out(n);
  for (int i = 0; i < n; ++i) {
    du[i].mel = static_cast<float*>(d[i]); du[i].x = static_cast<float*>(d[n + i]); du[i].nll = static_cast<float*>(d[2 * n + i]);
    out[i] = {utts[i].nll, du[i].nll, in[2 * n + i].bytes};
  }
  if ((rc = score_many(h, du.data(), n, pl, 0)) != WRNN_OK) return rc;
  return unstage(h, out);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// wrnn_score_wav_many: preprocess.py:36-47 and utils/dataset.py:86-91 on the device, then wrnn_score_many's job.
// ---------------------------------------------------------------------------------------------------------------------
// A float32 product that is never contracted into an FMA with the addition after it (numpy rounds both).
__host__ __device__ inline float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
// The stored label of sample y (float32, as numpy 1.22 evaluates preprocess.py) mapped back to the float target with
// label_2_float (float32, as torch evaluates dataset.py).  Logarithms are the correctly rounded float of the double
// logarithm, so the host and the device agree.
__host__ __device__ inline float wav_target(float y, int mode, int n_classes, bool mu_law) {
  const int bits = mode == WRNN_MODE_MOL ? 16 : (int)log2((double)n_classes);
  const float top = (float)((1 << bits) - 1);
  float label;
  if (mode == WRNN_MODE_RAW && mu_law) {                 // encode_mu_law(y, 2^bits)
    const float mu = top;
    const float s = y > 0.f ? 1.f : (y < 0.f ? -1.f : 0.f);
    const float fx = s * (float)log((double)(1.f + mul_rn(mu, fabsf(y)))) / (float)log((double)(1 << bits));
    label = floorf(mul_rn((fx + 1.f) / 2.f, mu) + 0.5f);
  } else {                                               // trunc(float_2_label(y, bits))
    const float v = (y + 1.f) * top / 2.f;
    label = truncf(v < 0.f ? 0.f : (v > top ? top : v));
  }
  return 2.f * label / top - 1.f;
}

struct WavUtt {
  const float* y;
  long long n;
  float* yn;      // the normalised recording
  float* x;       // its targets
};

// One block per recording: max |y|.
__global__ void wav_peak_kernel(const WavUtt* __restrict__ u, float* __restrict__ peak) {
  __shared__ float red[256];
  const WavUtt w = u[blockIdx.x];
  float p = 0.f;
  for (long long i = threadIdx.x; i < w.n; i += blockDim.x) p = fmaxf(p, fabsf(__ldg(w.y + i)));
  red[threadIdx.x] = p;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) peak[blockIdx.x] = red[0];
}

// Recording blockIdx.y: y / peak when peak_norm is set or the peak exceeds 1, and the targets of that y.
__global__ void wav_targets_kernel(const WavUtt* __restrict__ u, const float* __restrict__ peak, int peak_norm, int mode,
                                   int n_classes, int mu_law) {
  const WavUtt w = u[blockIdx.y];
  const float p = peak[blockIdx.y];
  const bool norm = peak_norm || p > 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < w.n; i += (long long)gridDim.x * blockDim.x) {
    float y = __ldg(w.y + i);
    if (norm) y = y / p;
    w.yn[i] = y;
    w.x[i] = wav_target(y, mode, n_classes, mu_law != 0);
  }
}

// Enqueues the peak, normalisation and target kernels over the DEVICE table `d_u` of n recordings.
static int wav_targets(const WavUtt* d_u, int n, long long max_n, float* peak, int peak_norm, int mode, int n_classes,
                       int mu_law, cudaStream_t st) {
  wav_peak_kernel<<<n, 256, 0, st>>>(d_u, peak);
  WRNN_CUDA_OK(cudaGetLastError());
  const dim3 grid((unsigned)std::min<long long>((max_n + 255) / 256, 64), (unsigned)n);
  wav_targets_kernel<<<grid, 256, 0, st>>>(d_u, peak, peak_norm, mode, n_classes, mu_law);
  WRNN_CUDA_OK(cudaGetLastError());
  return WRNN_OK;
}

// The batch's checks, on the host: the analysis against the model, each recording, then wrnn_score_many's plan of the
// job it becomes (T_i = 1 + n_i / hop frames) and the analysis's frame table.
static int score_wav_plan(int feat, int hop, const wrnn_mel_t* m, const wrnn_score_wav_utt* u, int n, cond::BatchPlan& pl,
                          std::vector<int64_t>& frame0) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  if (m->cfg.n_mels != feat) {
    set_error("the analysis makes n_mels = " + std::to_string(m->cfg.n_mels) + " bands, the model takes feat_dims = " + std::to_string(feat));
    return WRNN_E_INVALID;
  }
  if (m->cfg.hop_length != hop) {
    set_error("the analysis has hop_length " + std::to_string(m->cfg.hop_length) + ", the attached upsampler hop_length " + std::to_string(hop));
    return WRNN_E_INVALID;
  }
  if (!u || n < 1 || n > 65535) return cond::score_plan(hop, nullptr, 0, pl);
  const void* tag = m;                                 // placeholders: the plans only test these against NULL
  std::vector<wrnn_mel_utt> mu(n);
  std::vector<wrnn_score_utt> su(n);
  for (int i = 0; i < n; ++i) {
    if (!u[i].y || !u[i].nll) { set_error("utterance " + std::to_string(i) + ": y and nll are required"); return WRNN_E_INVALID; }
    mu[i] = wrnn_mel_utt{u[i].y, u[i].n, static_cast<float*>(const_cast<void*>(tag))};
  }
  int rc = mel::plan(m->cfg, mu.data(), n, frame0);
  if (rc != WRNN_OK) return rc;
  for (int i = 0; i < n; ++i)
    su[i] = wrnn_score_utt{static_cast<const float*>(tag), frame0[i + 1] - frame0[i], u[i].y, u[i].n, u[i].nll};
  return cond::score_plan(hop, su.data(), n, pl);
}

static int validate_score_wav(const wrnn_t* h, const wrnn_mel_t* m, const wrnn_score_wav_utt* u, int n, cond::BatchPlan& pl,
                              std::vector<int64_t>& frame0) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  if (!h->engine->scores()) { set_error(kNoRawStreamScore); return WRNN_E_INVALID; }
  int rc = score_wav_plan(h->engine->cfg.feat_dims, h->upsampler->hop, m, u, n, pl, frame0);
  if (rc != WRNN_OK) return rc;
  if (m->device != h->engine->device) {
    set_error("the analysis object is on device " + std::to_string(m->device) + ", the handle on device " + std::to_string(h->engine->device));
    return WRNN_E_INVALID;
  }
  return WRNN_OK;
}

// Handle scratch d_audio: [WavUtt table | peaks | normalised recordings | mels | targets], each region 256-B aligned.
static int score_wav_many(wrnn_t* h, const wrnn_mel_t* m, const wrnn_score_wav_utt* u, int n, int peak_norm, int mu_law,
                          const cond::BatchPlan& pl, const std::vector<int64_t>& frame0, cudaStream_t st) {
  const int nm = m->cfg.n_mels;
  std::vector<Staged> items(3 * n + 2);
  items[0].bytes = n * sizeof(WavUtt);
  items[1].bytes = n * sizeof(float);
  long long max_n = 0;
  for (int i = 0; i < n; ++i) {
    items[2 + i].bytes = items[2 + 2 * n + i].bytes = (size_t)u[i].n * sizeof(float);
    items[2 + n + i].bytes = (size_t)nm * (frame0[i + 1] - frame0[i]) * sizeof(float);
    max_n = std::max<long long>(max_n, u[i].n);
  }
  WRNN_CUDA_OK(cudaSetDevice(h->engine->device));
  int rc = grow(&h->d_audio, &h->audio_bytes, staged_bytes(items));
  if (rc != WRNN_OK) return rc;
  std::vector<void*> d;
  if ((rc = place(h->d_audio, items, st, d)) != WRNN_OK) return rc;
  auto region = [&](int kind, int i) { return static_cast<float*>(d[2 + kind * n + i]); };
  std::vector<WavUtt> wu(n);
  std::vector<wrnn_mel_utt> mu(n);
  std::vector<wrnn_score_utt> su(n);
  for (int i = 0; i < n; ++i) {
    wu[i] = WavUtt{u[i].y, u[i].n, region(0, i), region(2, i)};
    mu[i] = wrnn_mel_utt{region(0, i), u[i].n, region(1, i)};
    su[i] = wrnn_score_utt{region(1, i), frame0[i + 1] - frame0[i], region(2, i), u[i].n, u[i].nll};
  }
  WRNN_CUDA_OK(cudaMemcpyAsync(d[0], wu.data(), n * sizeof(WavUtt), cudaMemcpyHostToDevice, st));
  const wrnn_cfg& c = h->engine->cfg;
  if ((rc = wav_targets(static_cast<const WavUtt*>(d[0]), n, max_n, static_cast<float*>(d[1]), peak_norm, c.mode,
                        c.n_classes, mu_law, st)) != WRNN_OK)
    return rc;
  if ((rc = wrnn_melspectrogram_many(m, mu.data(), n, st)) != WRNN_OK) return rc;
  return score_many(h, su.data(), n, pl, st);
}

extern "C" {

int wrnn_score_wav_many(wrnn_t* h, const wrnn_mel_t* m, const wrnn_score_wav_utt* u, int32_t n_utts, int32_t peak_norm,
                        int32_t mu_law, void* stream) {
  cond::BatchPlan pl;
  std::vector<int64_t> frame0;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  if ((rc = validate_score_wav(h, m, u, n_utts, pl, frame0)) != WRNN_OK) return rc;
  return score_wav_many(h, m, u, n_utts, peak_norm, mu_law, pl, frame0, static_cast<cudaStream_t>(stream));
}

int wrnn_score_wav_many_host(wrnn_t* h, const wrnn_mel_t* m, const wrnn_score_wav_utt* u, int32_t n_utts, int32_t peak_norm,
                             int32_t mu_law) {
  cond::BatchPlan pl;
  std::vector<int64_t> frame0;
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  if ((rc = validate_score_wav(h, m, u, n_utts, pl, frame0)) != WRNN_OK) return rc;
  const int n = n_utts;
  std::vector<Staged> in(2 * n);                       // [recordings | losses]
  for (int i = 0; i < n; ++i) {
    in[i] = {u[i].y, (size_t)u[i].n * sizeof(float)};
    in[n + i] = {nullptr, (size_t)u[i].n * sizeof(float)};
  }
  std::vector<void*> d;
  if ((rc = stage(h, in, 0, d)) != WRNN_OK) return rc;
  std::vector<wrnn_score_wav_utt> du(u, u + n);
  std::vector<Unstaged> out(n);
  for (int i = 0; i < n; ++i) {
    du[i].y = static_cast<float*>(d[i]); du[i].nll = static_cast<float*>(d[n + i]);
    out[i] = {u[i].nll, du[i].nll, in[n + i].bytes};
  }
  if ((rc = score_wav_many(h, m, du.data(), n, peak_norm, mu_law, pl, frame0, 0)) != WRNN_OK) return rc;
  return unstage(h, out);
}

// ---- test hooks (not declared in the header) ------------------------------------------------------------------------
// wrnn_score_wav_many's plan without a handle: its refusals, and T_i (T [n_utts]) of the job it becomes.
int wrnn_debug_score_wav_plan(int32_t feat_dims, int32_t hop, const wrnn_mel_cfg* cfg, const wrnn_score_wav_utt* u,
                              int32_t n_utts, int64_t* T) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  wrnn_mel_plan m;
  m.cfg = *cfg;
  cond::BatchPlan pl;
  std::vector<int64_t> frame0;
  if ((rc = score_wav_plan(feat_dims, hop, &m, u, n_utts, pl, frame0)) != WRNN_OK) return rc;
  for (int i = 0; T && i < n_utts; ++i) T[i] = frame0[i + 1] - frame0[i];
  return WRNN_OK;
}

// The targets of each sample of y [n] (HOST), without normalisation: wav_target on the host.
int wrnn_debug_wav_targets(const float* y, int64_t n, int32_t mode, int32_t n_classes, int32_t mu_law, float* x) {
  for (int64_t i = 0; i < n; ++i) x[i] = wav_target(y[i], mode, n_classes, mu_law != 0);
  return WRNN_OK;
}

// What wrnn_score_wav_many runs before the analysis, for one recording (DEVICE pointers, asynchronous on `stream`):
// the normalised recording yn [n] and its targets x [n].  peak: one float of device scratch.
int wrnn_debug_score_wav_targets(const float* y, int64_t n, int32_t mode, int32_t n_classes, int32_t peak_norm,
                                 int32_t mu_law, float* yn, float* x, float* peak, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const WavUtt w{y, n, yn, x};
  return with_device_table(&w, 1, st, [&](const WavUtt* d) {
    return wav_targets(d, 1, n, peak, peak_norm, mode, n_classes, mu_law, st);
  });
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// wrnn_vocode_live_start / _poll: an unbatched wrnn_vocode whose samples the host turns into the waveform while the
// persistent kernel is still generating.  One fold, overlap 0: sample n < wave_len is final as soon as it is stored.
// wrnn_vocode_many_live_start / _poll: the same for an unbatched wrnn_vocode_many of up to 64 utterances, one fold each,
// in one tile; each fold publishes its own progress.
// ---------------------------------------------------------------------------------------------------------------------
// wrnn_epilogue_kernel on the host: samples [n0, n1) of a waveform of wave_len samples unfolded from x[0 .. n_seg), fold
// b's seg_len samples starting at waveform sample b * stride (unbatched: one fold, stride = seg_len >= wave_len).  The
// same operations in the same order: per fold sample, the mu-law label recovered in fp32 and rounded half to even
// (saturating, NaN -> 0, then clamped), times fade_in on the fold's first overlap samples and fade_out on its last; per
// waveform sample 0.0 + the earlier fold's sample + the later one's (a -0.0 sample becomes +0.0), then the fade-out over
// the last tail_len samples.
static void live_epilogue(const LiveTables& t, const float* const* x, int n_seg, long long seg_len, long long stride, long long n0,
                          long long n1, long long wave_len, double* wav) {
  const int nc = t.n_classes, ov = t.overlap;
  auto value = [&](long long i, long long k) {
    const float xf = x[i][k];
    double y = (double)xf;
    if (!t.mu.empty()) {
      const float r = std::nearbyint((xf + 1.0f) * (0.5f * (float)(nc - 1)));
      y = t.mu[!(r > 0.f) ? 0 : (r >= (float)(nc - 1) ? nc - 1 : (int)r)];
    }
    if (k < ov) y *= t.fade_in[k];
    if (k >= seg_len - ov) y *= t.fade_out[k - (seg_len - ov)];
    return y;
  };
  for (long long n = n0; n < n1; ++n) {
    const long long i = std::min(n / stride, (long long)n_seg - 1), k = n - i * stride;
    double v = 0.0;
    if (i >= 1 && k + stride < seg_len) v += value(i - 1, k + stride);
    if (k < seg_len) v += value(i, k);
    if (n >= wave_len - t.tail_len) v *= t.tail[n - (wave_len - t.tail_len)];
    wav[n] = v;
  }
}

// One utterance's delivery, for both kinds of live job: its samples [delivered, min(count, wave_len)) of x, count being
// what its fold has published, through live_epilogue into wav.  Returns whether any were delivered.
static bool live_deliver_one(const LiveTables& t, const float* x, long long count, long long wave_len, long long& delivered,
                             double* wav) {
  const long long ready = count < wave_len ? count : wave_len;
  if (ready <= delivered) return false;
  live_epilogue(t, &x, 1, wave_len, wave_len, delivered, ready, wave_len, wav);
  delivered = ready;
  return true;
}

// Calls f until it returns a value, sleeping in short intervals in between (a few hundred steps of the kernel each), for
// at most wait_us in all (no limit when wait_us < 0).  Returns f's value, or nothing at the deadline.
template <class F>
static std::optional<int> wait_for(long long wait_us, F f) {
  const auto end = std::chrono::steady_clock::now() + std::chrono::microseconds(wait_us);
  const std::chrono::steady_clock::duration interval = std::chrono::microseconds(100);
  for (;;) {
    if (const std::optional<int> r = f()) return r;
    const auto left = wait_us < 0 ? interval : end - std::chrono::steady_clock::now();
    if (left <= left.zero()) return std::nullopt;
    std::this_thread::sleep_for(std::min(left, interval));
  }
}

// Delivers, per utterance, the samples its fold has published so far (at most its wave_len) into the caller's wav.
// Returns whether any utterance received samples.
static bool live_deliver(LiveJob& lj) {
  bool more = false;
  for (int i = 0; i < lj.n(); ++i)
    more = live_deliver_one(lj.tabs, lj.samples(i), (long long)lj.progress(i), lj.wave_len[i], lj.delivered[i], lj.wav[i]) || more;
  return more;
}

// The launch of a live job set up by vocode_many_job: fold i (utterance i, of T[i] frames) stores its
// samples into row i of the pinned buffer and publishes its progress word; the poll delivers them into wav[i].
static int live_launch(wrnn_t* h, VocodeJob& v, bool many, bool mu_law, const std::vector<double*>& wav,
                       const std::vector<long long>& T, cudaStream_t st) {
  if (!h->live && !(h->live = new (std::nothrow) LiveJob())) { set_error("out of host memory"); return WRNN_E_INVALID; }
  LiveJob& lj = *h->live;
  const int n = (int)wav.size(), hop = h->upsampler->hop;
  const long long steps = v.j.seg_len;
  int rc = grow_mapped(&lj.host, &lj.dev, &lj.bytes, LiveJob::SAMPLES_OFF + (size_t)n * steps * sizeof(float));
  if (rc != WRNN_OK) return rc;
  for (int i = 0; i < n; ++i)                                   // no kernel of this handle runs
    __atomic_store_n(static_cast<unsigned long long*>(lj.host) + i, 0ull, __ATOMIC_RELEASE);
  if (!lj.done) WRNN_CUDA_OK(cudaEventCreateWithFlags(&lj.done, cudaEventDisableTiming));
  v.j.out = reinterpret_cast<float*>(static_cast<char*>(lj.dev) + LiveJob::SAMPLES_OFF);
  if ((rc = v.e->generate_live(v.j, st, v.keys, static_cast<unsigned long long*>(lj.dev))) != WRNN_OK) return rc;
  WRNN_CUDA_OK(cudaEventRecord(lj.done, st));

  lj.tabs = live_tables(h->engine->cfg.mode, mu_law, h->engine->cfg.n_classes, hop);
  lj.e = v.e;
  lj.many = many;
  lj.steps = steps;
  lj.wav = wav;
  lj.wave_len.resize(n);
  for (int i = 0; i < n; ++i) lj.wave_len[i] = (T[i] - 1) * hop;
  lj.delivered.assign(n, 0);
  h->live_busy = true;
  return WRNN_OK;
}

// Both polls: waits up to wait_us for more samples of the job the matching start began and delivers them; n_ready[i] =
// the final samples of utterance i.
static int live_poll(wrnn_t* h, int32_t wait_us, bool many, int64_t* n_ready) {
  if (!h || !h->engine || !n_ready) { set_error("null handle or n_ready"); return WRNN_E_INVALID; }
  if (h->session) { set_error("a live session is open on this handle: poll it with wrnn_live_poll"); return WRNN_E_INVALID; }
  if (!h->live_busy) {
    set_error(many ? "no batch live job on this handle (wrnn_vocode_many_live_start)" : "no live job on this handle (wrnn_vocode_live_start)");
    return WRNN_E_INVALID;
  }
  LiveJob& lj = *h->live;
  if (lj.many != many) {
    set_error(many ? "the live job in flight was started by wrnn_vocode_live_start: poll it with wrnn_vocode_live_poll"
                   : "the live job in flight was started by wrnn_vocode_many_live_start: poll it with wrnn_vocode_many_live_poll");
    return WRNN_E_INVALID;
  }
  const std::optional<int> rc = wait_for(wait_us > 0 ? wait_us : 0, [&]() -> std::optional<int> {
    const cudaError_t q = cudaEventQuery(lj.done);
    if (q == cudaSuccess) {                            // the kernel has finished: every sample is published
      h->live_busy = false;
      int rc = lj.e->check();
      if (rc == WRNN_OK) {
        live_deliver(lj);
        for (int i = 0; i < lj.n() && rc == WRNN_OK; ++i)
          if (lj.delivered[i] < lj.wave_len[i]) {
            set_error("live job: the kernel finished with " + std::to_string(lj.delivered[i]) + " of " +
                      std::to_string(lj.wave_len[i]) + " samples of utterance " + std::to_string(i) + " published");
            rc = WRNN_E_CUDA;
          }
      }
      return rc;
    }
    if (q != cudaErrorNotReady) {
      h->live_busy = false;
      set_error(std::string("live job: ") + cudaGetErrorString(q));
      return WRNN_E_CUDA;
    }
    return live_deliver(lj) ? std::optional<int>(1) : std::nullopt;
  });
  for (int i = 0; i < lj.n(); ++i) n_ready[i] = lj.delivered[i];
  return rc ? *rc : 1;
}

// Both live starts, after their own refusals (b is unbatched, of 1 to 64 utterances with mel, wav and T >= 21): the
// batch laid out as wrnn_vocode_many's job, launched live.
static int live_start(wrnn_t* h, const wrnn_vocode_batch* b, bool many, cudaStream_t st) {
  int rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  cond::BatchPlan pl;
  if ((rc = validate_many(h, b, pl)) != WRNN_OK) return rc;

  // the mels (host or device) into staging, so that the conditioning network reads device memory
  const int n = b->n_utts;
  std::vector<Staged> in(n);
  for (int i = 0; i < n; ++i) in[i] = {b->utts[i].mel, (size_t)b->utts[i].T * FEAT * sizeof(float)};
  std::vector<void*> d;
  if ((rc = stage(h, in, st, d)) != WRNN_OK) return rc;
  std::vector<wrnn_utterance> du(b->utts, b->utts + n);
  std::vector<double*> wav(n);
  std::vector<long long> T(n);
  for (int i = 0; i < n; ++i) {
    du[i].mel = static_cast<float*>(d[i]);
    wav[i] = b->utts[i].wav;
    T[i] = b->utts[i].T;
  }
  wrnn_vocode_batch db = *b;
  db.utts = du.data();
  VocodeJob v;
  if ((rc = vocode_many_job(h, &db, pl, st, true, &v)) != WRNN_OK) return rc;
  return live_launch(h, v, many, b->mu_law, wav, T, st);
}

extern "C" {

int wrnn_vocode_live_start(wrnn_t* h, const wrnn_vocode_job* job, void* stream) {
  if (!job) { set_error("null job"); return WRNN_E_INVALID; }
  if (job->batched) {
    set_error("a live job must be unbatched (batched = 0): a batched job's folds all finish at its last step, so no "
              "sample is final before the whole job is");
    return WRNN_E_INVALID;
  }
  const int rc = check_utterance("", job->mel, job->wav, job->T);
  if (rc != WRNN_OK) return rc;
  // the batch of one utterance: the same fold, keyed (philox_seed, 0), as wrnn_vocode's unbatched job
  const wrnn_utterance u{job->mel, job->T, job->philox_seed, job->wav};
  const wrnn_vocode_batch b{&u, 1, 0, 0, 0, job->mu_law};
  return live_start(h, &b, false, static_cast<cudaStream_t>(stream));
}

int wrnn_vocode_live_poll(wrnn_t* h, int32_t wait_us, int64_t* n_ready) { return live_poll(h, wait_us, false, n_ready); }

int wrnn_vocode_many_live_start(wrnn_t* h, const wrnn_vocode_batch* b, void* stream) {
  if (!b) { set_error("null batch"); return WRNN_E_INVALID; }
  if (b->batched) {
    set_error("a live batch must be unbatched (batched = 0): a batched job's folds all finish at its last step, so no "
              "sample is final before the whole job is");
    return WRNN_E_INVALID;
  }
  if (b->n_utts < 1 || b->n_utts > LiveJob::MAX_UTTS) {
    set_error("a live batch holds 1 to 64 utterances: one persistent tile holds 64 folds, and a second tile would start "
              "only after the first has finished");
    return WRNN_E_INVALID;
  }
  if (!b->utts) { set_error("utts is required"); return WRNN_E_INVALID; }
  for (int i = 0; i < b->n_utts; ++i) {
    const wrnn_utterance& u = b->utts[i];
    const int rc = check_utterance("utterance " + std::to_string(i) + ": ", u.mel, u.wav, u.T);
    if (rc != WRNN_OK) return rc;
  }
  return live_start(h, b, true, static_cast<cudaStream_t>(stream));
}

int wrnn_vocode_many_live_poll(wrnn_t* h, int32_t wait_us, int64_t* n_ready) { return live_poll(h, wait_us, true, n_ready); }

// Test hook (CPU-only, no device needed): wrnn_vocode_live_poll's epilogue over samples x [n] (n <= wave_len) of an
// unbatched job of wave_len samples at this hop, with the tables wrnn_vocode builds (mu_law: a RAW head's).  Checked in
// tests/test_live_abi.py.
int wrnn_debug_live_epilogue(const float* x, int64_t n, int64_t wave_len, int32_t hop, int32_t mu_law, int32_t n_classes,
                             double* wav) {
  if (!x || !wav || hop <= 0 || n < 0 || n > wave_len || wave_len < 20ll * hop || (mu_law && n_classes < 2)) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  live_epilogue(live_tables(WRNN_MODE_RAW, mu_law != 0, n_classes, hop), &x, 1, wave_len, wave_len, 0, n, wave_len, wav);
  return WRNN_OK;
}

// Test hook (CPU-only, no device needed): one delivery of a poll of wrnn_vocode_many_live_poll, on a host buffer laid
// out as the live job's pinned one.  Utterance i (T[i] frames) is fold i with samples x [n_utts][steps] and published
// progress[i]; delivered [n_utts] holds what earlier polls delivered and receives what this one did; wav is the
// concatenation of the n_utts waveforms.  Checked in tests/test_live_many_abi.py.
int wrnn_debug_live_many_deliver(const float* x, int64_t steps, const uint64_t* progress, int32_t n_utts, const int64_t* T,
                                 int32_t hop, int32_t mu_law, int32_t n_classes, int64_t* delivered, double* wav) {
  if (!x || !progress || !T || !delivered || !wav || steps <= 0 || hop <= 0 || n_utts < 1 || n_utts > LiveJob::MAX_UTTS ||
      (mu_law && n_classes < 2)) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  for (int i = 0; i < n_utts; ++i)
    if (T[i] < 21 || T[i] * hop > steps || delivered[i] < 0 || delivered[i] > (T[i] - 1) * hop) { set_error("bad argument"); return WRNN_E_INVALID; }
  std::vector<unsigned char> buf(LiveJob::SAMPLES_OFF + (size_t)n_utts * steps * sizeof(float));
  std::memcpy(buf.data(), progress, (size_t)n_utts * sizeof(uint64_t));
  std::memcpy(buf.data() + LiveJob::SAMPLES_OFF, x, (size_t)n_utts * steps * sizeof(float));
  LiveJob lj;
  lj.host = buf.data();
  lj.steps = steps;
  lj.tabs = live_tables(WRNN_MODE_RAW, mu_law != 0, n_classes, hop);
  double* w = wav;
  for (int i = 0; i < n_utts; ++i) {
    lj.wav.push_back(w);
    lj.wave_len.push_back((T[i] - 1) * hop);
    lj.delivered.push_back(delivered[i]);
    w += (T[i] - 1) * hop;
  }
  live_deliver(lj);
  for (int i = 0; i < n_utts; ++i) delivered[i] = lj.delivered[i];
  return WRNN_OK;
}

}  // extern "C"

extern "C" {

// Test hook (CPU-only, no device needed): the stream engine's packed weight stream and step program for host-resident
// weights, so the packing and the schedule can be interpreted and checked without a GPU (tests/test_stream_plan.py,
// tests/test_stream_plan_raw.py).  cfg->mode selects the head: the MoL plan (n_classes <= 128) or the RAW plan
// (n_classes == 512).  Call with blob == NULL to obtain the sizes.  Not part of the reference-facing surface.
int wrnn_debug_stream_plan(const wrnn_cfg* cfg, const wrnn_weights* w, uint8_t* blob, uint64_t* blob_bytes, uint8_t* prog,
                           uint64_t* n_chunks,
                           float* vectors /* qk[4096] vq[4096] b1h[1536] b2h[1536] b3[n_classes padded to a multiple of 128:
                                             128 for MoL, 512 for RAW] */,
                           uint16_t* mine /* [4][n_chunks]: per issuing warp, its chunk indices; unused tail = 0xffff */,
                           int32_t only_block /* -1: the whole program; 0..3: the share of that rank of a 4-CTA cluster */) {
  if (!cfg || !w || !blob_bytes || !n_chunks) { set_error("null argument"); return WRNN_E_INVALID; }
  if (cfg->mode == WRNN_MODE_RAW ? cfg->n_classes != 512 : (cfg->n_classes <= 0 || cfg->n_classes > stream::MROWS)) {
    set_error("stream plan: the MoL head needs n_classes <= 128, the RAW head n_classes == 512");
    return WRNN_E_INVALID;
  }
  HostWeights hw;
  const int rc = read_weights(*cfg, *w, true, hw);
  if (rc != WRNN_OK) return rc;
  stream::Plan plan;
  stream::build_plan(hw, cfg->precision == WRNN_PREC_BF16, plan, only_block);
  if (blob) {
    if (*blob_bytes < plan.blob.size() || *n_chunks < plan.prog.size()) { set_error("buffers too small"); return WRNN_E_INVALID; }
    std::memcpy(blob, plan.blob.data(), plan.blob.size());
    std::memcpy(prog, plan.prog.data(), plan.prog.size() * sizeof(stream::Chunk));
    float* v = vectors;
    std::memcpy(v, plan.qk.data(), 8 * H * 4); v += 8 * H;
    std::memcpy(v, plan.vq.data(), 8 * H * 4); v += 8 * H;
    std::memcpy(v, plan.b1h.data(), G3 * 4); v += G3;
    std::memcpy(v, plan.b2h.data(), G3 * 4); v += G3;
    std::memcpy(v, plan.b3.data(), plan.b3.size() * 4);
    if (mine) {
      std::memset(mine, 0xff, sizeof(uint16_t) * stream::N_ISSUERS * plan.prog.size());
      for (int o = 0; o < stream::N_ISSUERS; ++o) std::memcpy(mine + (size_t)o * plan.prog.size(), plan.mine[o].data(), plan.mine[o].size() * sizeof(uint16_t));
    }
  }
  *blob_bytes = plan.blob.size(); *n_chunks = plan.prog.size();
  return WRNN_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// wrnn_live_open .. wrnn_live_close: a live session.  Slot s of the persistent tile owns region s of the frame arena, row
// s of the pinned sample block, progress word s and mailbox s.  A ticket holds one slot per fold: an unbatched one a single
// fold, a batched one the n_seg folds of fold_with_overlap.  The host picks free slots, writes the utterance's conditioning
// frames into the region of the ticket's first slot on a side stream and, once they are complete, posts each fold's
// request to its slot's mailbox; CTA 0 admits each at the next boundary it sees it (DESIGN §3.7).  A launch that has
// exited is relaunched with the posted requests admitted at its step 0.
// ---------------------------------------------------------------------------------------------------------------------
namespace wrnn {
struct LiveSession {
  static constexpr int MAX_SLOTS = 64;
  static constexpr size_t MAIL_OFF = MAX_SLOTS * sizeof(unsigned long long);
  static constexpr size_t SAMPLES_OFF = 4096;     // [progress words | mailboxes | pad | samples [C][max_steps]]
  static_assert(MAIL_OFF + MAX_SLOTS * sizeof(SesMail) <= SAMPLES_OFF, "pinned layout");
  enum { FREE, PREP, POSTED };
  // A ticket, kept at the index of its first slot.  Fold b runs seg_len steps from arena row row0 + b * stride (rows
  // past `rows` read as zeros), covers waveform samples [b * stride, + seg_len) and is held by slot slot[b].
  struct Ticket {
    int state = FREE;
    long long ticket = 0;
    unsigned tag = 0;
    unsigned long long seed = 0;
    long long wave_len = 0, delivered = 0;
    long long seg_len = 0, stride = 0, row0 = 0, rows = 0;
    std::vector<int> slot;
    int posted = 0;                  // folds 0 .. posted - 1 have their request in their slot's mailbox
    LiveTables tabs;                 // the session's, or a batched ticket's own (its overlap's fade tables)
    double* wav = nullptr;
    bool cancelled = false;
  };
  int C = 0, hop = 0;
  long long max_T = 0, max_steps = 0;
  LiveTables tabs;
  Engine* e = nullptr;
  cudaStream_t st = nullptr, side = nullptr;
  void* host = nullptr; void* dev = nullptr;         // pinned, mapped
  void* d_ctl = nullptr;                             // [tab 2 x 64 | stop 2]
  void* d_arena = nullptr;                           // [mel_frames C x (max_T + 4) | aux_frames C x (max_T + 4) | mel stage C x max_T]
  float *mel_frames = nullptr, *aux_frames = nullptr, *mel_stage = nullptr;
  const float* taps = nullptr;                       // the upsampler's [hop][5] tap table
  size_t stage_pitch = 0;
  cudaEvent_t done = nullptr;                        // recorded after the running launch
  bool running = false;
  std::vector<Ticket> tickets;                       // [C]: the ticket whose first slot is s, if any
  std::vector<int> owner;                            // [C]: the first slot of the ticket holding slot s, or -1
  std::vector<cudaEvent_t> ready;                    // [C]: the frames of the ticket whose first slot is s are complete
  std::vector<SesEntry> tab;                         // host image of the table for a launch: [2][64], version -1 in buffer 1
  long long next_ticket = 1;
  int post_limit = MAX_SLOTS;                        // folds posted by one pump at most (wrnn_debug_live_post_limit)
  std::vector<wrnn_live_ticket> released;            // tickets whose slots were released since the last poll
  unsigned long long* progress() const { return static_cast<unsigned long long*>(host); }
  SesMail* mail() const { return reinterpret_cast<SesMail*>(static_cast<char*>(host) + MAIL_OFF); }
  const float* samples(int s) const {
    return reinterpret_cast<const float*>(static_cast<const char*>(host) + SAMPLES_OFF) + (size_t)s * max_steps;
  }
  // Releases all of a ticket's slots at once: a retired fold's samples stay in its slot's row until the prefix has
  // passed them.
  void release(Ticket& tk) {
    released.push_back(wrnn_live_ticket{tk.ticket, tk.delivered,
                                        (!tk.cancelled && tk.delivered == tk.wave_len) ? WRNN_LIVE_DONE : WRNN_LIVE_CANCELLED, 0});
    for (const int s : tk.slot) owner[s] = -1;
    tk = Ticket();
  }
};

// Delivers, per posted ticket, the longest prefix of its waveform whose every sample each covering fold has published
// (words of an earlier occupant of a slot carry another tag and count as nothing published), and releases the tickets
// whose every fold CTA 0 retired (a cancelled ticket: every fold it posted).  Returns whether anything changed.
static bool session_deliver(LiveSession& ss) {
  bool more = false;
  for (LiveSession::Ticket& tk : ss.tickets) {
    if (tk.state != LiveSession::POSTED) continue;
    const int n_seg = (int)tk.slot.size();
    long long ready = tk.wave_len;
    bool retired = tk.posted == n_seg || tk.cancelled;
    const float* x[LiveSession::MAX_SLOTS];
    for (int b = 0; b < n_seg; ++b) {
      const unsigned long long w = __atomic_load_n(ss.progress() + tk.slot[b], __ATOMIC_ACQUIRE);
      const bool mine = (unsigned)(w >> 32) == tk.tag;
      const long long count = mine ? (long long)(w & (SES_RETIRED - 1u)) : 0;
      if (b < tk.posted) retired = retired && mine && (w & SES_RETIRED);
      if (count < tk.seg_len) ready = std::min(ready, b * tk.stride + count);
      x[b] = ss.samples(tk.slot[b]);
    }
    if (!tk.cancelled && ready > tk.delivered) {
      live_epilogue(tk.tabs, x, n_seg, tk.seg_len, tk.stride, tk.delivered, ready, tk.wave_len, tk.wav);
      tk.delivered = ready;
      more = true;
    }
    if (retired) { ss.release(tk); more = true; }
  }
  return more;
}

// A relaunch's decision for one posted ticket (no launch runs, so every fold a launch admitted has retired).  Each posted
// fold whose slot carries the ticket's tag has finished, whatever launch served it; the others were never admitted.
// Those go into version -1 of the table, admitted at step 0 with the ticket's tag written to their progress words, or
// are withdrawn if the ticket is cancelled, which then releases it.  Its folds may so be served by several launches: a
// launch exits at a boundary where no slot is held, which can fall between two folds' posts.  Sets `launch` when a
// fold was admitted; WRNN_E_CUDA if a fold with the ticket's tag is not retired.
static int relaunch_ticket(LiveSession& ss, LiveSession::Ticket& tk, bool& launch) {
  for (int b = 0; b < tk.posted; ++b) {
    const int s = tk.slot[b];
    const unsigned long long w = __atomic_load_n(ss.progress() + s, __ATOMIC_ACQUIRE);
    if ((unsigned)(w >> 32) == tk.tag) {
      if (w & SES_RETIRED) continue;
      set_error("live session: a launch exited with slot " + std::to_string(s) + " still held");
      return WRNN_E_CUDA;
    }
    if (tk.cancelled) {
      __atomic_store_n(&ss.mail()[s].req, w >> 32, __ATOMIC_RELEASE);
      continue;
    }
    ss.tab[LiveSession::MAX_SLOTS + s] = SesEntry{0, (int)tk.seg_len, tk.seed, (unsigned)b, (int)(tk.row0 + b * tk.stride),
                                                  (int)(tk.rows - b * tk.stride), 0};
    __atomic_store_n(ss.progress() + s, (unsigned long long)tk.tag << 32, __ATOMIC_RELEASE);
    launch = true;
  }
  if (tk.cancelled) ss.release(tk);
  return WRNN_OK;
}

// Posts the folds of the tickets whose frames are complete (at most post_limit per call), and relaunches the kernel when
// the last launch has exited and a posted request was not admitted by it.
static int session_pump(LiveSession& ss) {
  if (ss.running) {
    const cudaError_t q = cudaEventQuery(ss.done);
    if (q == cudaSuccess) {
      ss.running = false;
      session_deliver(ss);                             // the launch's last words
      const int rc = ss.e->check();
      if (rc != WRNN_OK) return rc;
    } else if (q != cudaErrorNotReady) {
      set_error(std::string("live session: ") + cudaGetErrorString(q));
      return WRNN_E_CUDA;
    }
  }
  for (int s = 0; s < ss.C; ++s) {
    LiveSession::Ticket& tk = ss.tickets[s];
    if (tk.state != LiveSession::PREP) continue;
    const cudaError_t q = cudaEventQuery(ss.ready[s]);
    if (q == cudaErrorNotReady) continue;
    if (q != cudaSuccess) { set_error(std::string("live session: conditioning: ") + cudaGetErrorString(q)); return WRNN_E_CUDA; }
    if (tk.cancelled) { ss.release(tk); continue; }
    tk.state = LiveSession::POSTED;
  }
  int budget = ss.post_limit;
  for (LiveSession::Ticket& tk : ss.tickets) {
    for (; tk.state == LiveSession::POSTED && !tk.cancelled && tk.posted < (int)tk.slot.size() && budget > 0; ++tk.posted, --budget) {
      const int b = tk.posted;
      SesMail& m = ss.mail()[tk.slot[b]];
      m.seed = tk.seed;
      m.steps = tk.seg_len;
      m.fold = (unsigned)b;
      m.row0 = (int)(tk.row0 + b * tk.stride);
      m.rows = (int)(tk.rows - b * tk.stride);
      __atomic_store_n(&m.req, (unsigned long long)tk.tag, __ATOMIC_RELEASE);   // the body before the tag
    }
  }
  if (ss.running) return WRNN_OK;
  bool launch = false;
  for (int s = 0; s < LiveSession::MAX_SLOTS; ++s) ss.tab[LiveSession::MAX_SLOTS + s] = SesEntry{};
  for (LiveSession::Ticket& tk : ss.tickets) {
    if (tk.state != LiveSession::POSTED) continue;
    const int rc = relaunch_ticket(ss, tk, launch);
    if (rc != WRNN_OK) return rc;
  }
  if (!launch) return WRNN_OK;
  WRNN_CUDA_OK(cudaSetDevice(ss.e->device));
  WRNN_CUDA_OK(cudaMemcpyAsync(ss.d_ctl, ss.tab.data(), ss.tab.size() * sizeof(SesEntry), cudaMemcpyHostToDevice, ss.st));
  wrnn_job j;
  std::memset(&j, 0, sizeof(j));
  j.n_seg = ss.C; j.seg_len = (int32_t)ss.max_steps; j.seg_stride = (ss.max_T + 4) * ss.hop; j.L = j.seg_stride * ss.C;
  j.mel_frames = ss.mel_frames; j.aux_frames = ss.aux_frames; j.up_taps = ss.taps; j.hop = ss.hop;
  j.out = reinterpret_cast<float*>(static_cast<char*>(ss.dev) + LiveSession::SAMPLES_OFF);
  SesCtl c;
  c.tab = static_cast<SesEntry*>(ss.d_ctl);
  c.stop = reinterpret_cast<int*>(c.tab + 2 * LiveSession::MAX_SLOTS);
  c.mail = reinterpret_cast<const SesMail*>(static_cast<char*>(ss.dev) + LiveSession::MAIL_OFF);
  c.progress = static_cast<unsigned long long*>(ss.dev);
  int rc = ss.e->generate_session(j, ss.st, c);
  if (rc != WRNN_OK) return rc;
  WRNN_CUDA_OK(cudaEventRecord(ss.done, ss.st));
  ss.running = true;
  return WRNN_OK;
}

static void session_free(LiveSession* ss) {
  if (ss->done) { cudaEventSynchronize(ss->done); cudaEventDestroy(ss->done); }
  if (ss->side) { cudaStreamSynchronize(ss->side); cudaStreamDestroy(ss->side); }
  for (const cudaEvent_t ev : ss->ready) if (ev) cudaEventDestroy(ev);
  if (ss->host) cudaFreeHost(ss->host);
  cudaFree(ss->d_ctl);
  cudaFree(ss->d_arena);
  delete ss;
}

// The refusals shared by both submits, then the open session of h (nullptr after a refusal).
static LiveSession* submit_session(wrnn_t* h, const wrnn_utterance* u) {
  if (!h || !h->engine) { set_error("null handle"); return nullptr; }
  if (!h->session) { set_error("no live session is open on this handle (wrnn_live_open)"); return nullptr; }
  if (u->T > h->session->max_T) { set_error("T exceeds the session's max_T (" + std::to_string(h->session->max_T) + ")"); return nullptr; }
  return h->session;
}

// Both submits, after their refusals: g is the ticket's fold geometry (unbatched: one fold of wave_len steps).  Takes
// g.n_seg free slots (none when fewer are free), runs the conditioning network into the first one's region on the side
// stream and records that slot's ready event; session_pump posts the folds once it has completed.
static int session_submit(wrnn_t* h, const wrnn_utterance* u, const cond::Geometry& g, LiveTables tabs, int64_t* ticket) {
  LiveSession& ss = *h->session;
  int rc = session_pump(ss);                           // releases what has finished, so that its slots can be reused
  if (rc != WRNN_OK) return rc;
  session_deliver(ss);
  std::vector<int> slot;
  for (int s = 0; s < ss.C && (long long)slot.size() < g.n_seg; ++s)
    if (ss.owner[s] < 0) slot.push_back(s);
  if ((long long)slot.size() < g.n_seg) {
    set_error(g.n_seg == 1 ? "all " + std::to_string(ss.C) + " slots of the live session hold an utterance: poll until one is released"
                           : std::to_string(slot.size()) + " of the live session's " + std::to_string(ss.C) + " slots are free and the utterance has " +
                                 std::to_string(g.n_seg) + " folds: poll until enough are released");
    return WRNN_E_BUSY;
  }
  WRNN_CUDA_OK(cudaSetDevice(ss.e->device));
  const int s0 = slot[0];
  float* stage = ss.mel_stage + (size_t)s0 * ss.stage_pitch;
  const size_t frame0 = (size_t)s0 * (ss.max_T + 4);
  WRNN_CUDA_OK(cudaMemcpyAsync(stage, u->mel, (size_t)u->T * FEAT * sizeof(float), cudaMemcpyDefault, ss.side));
  if ((rc = conditioning_frames(*h->upsampler, stage, u->T, ss.mel_frames + frame0 * FEAT, ss.aux_frames + frame0 * cond::CD,
                                nullptr, ss.side)) != WRNN_OK)
    return rc;
  WRNN_CUDA_OK(cudaEventRecord(ss.ready[s0], ss.side));
  LiveSession::Ticket& tk = ss.tickets[s0];
  tk.state = LiveSession::PREP;
  tk.ticket = ss.next_ticket++;
  tk.tag = ses_tag(tk.ticket);
  tk.seed = u->philox_seed;
  tk.wave_len = (u->T - 1) * ss.hop;
  tk.delivered = 0;
  tk.seg_len = g.seg_len;
  tk.stride = g.seg_stride;
  tk.row0 = (long long)frame0 * ss.hop;
  tk.rows = u->T * ss.hop;
  tk.slot = slot;
  tk.posted = 0;
  tk.tabs = std::move(tabs);
  tk.wav = u->wav;
  tk.cancelled = false;
  for (const int s : slot) ss.owner[s] = s0;
  *ticket = tk.ticket;
  return session_pump(ss);
}
}  // namespace wrnn

extern "C" {

int wrnn_live_open(wrnn_t* h, int32_t capacity, int64_t max_T, int32_t mu_law, void* stream) {
  if (capacity < 1 || capacity > LiveSession::MAX_SLOTS) {
    set_error("a live session holds 1 to 64 slots: one persistent tile holds 64 folds"); return WRNN_E_INVALID;
  }
  int rc = check_frames("max_T", max_T);
  if (rc != WRNN_OK) return rc;
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  rc = idle_or_busy(h);
  if (rc != WRNN_OK) return rc;
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  if (h->engine->live_refusal()) { set_error(h->engine->live_refusal()); return WRNN_E_INVALID; }
  const int hop = h->upsampler->hop;
  if ((max_T - 1) * hop > SES_MAX_STEPS || (max_T + 4) * hop * capacity >= (1ll << 31)) {
    set_error("max_T too large: an utterance is at most 2^27 samples and the session's frame arena below 2^31 rows"); return WRNN_E_INVALID;
  }
  LiveSession* ss = new (std::nothrow) LiveSession();
  if (!ss) { set_error("out of host memory"); return WRNN_E_INVALID; }
  ss->C = capacity; ss->hop = hop; ss->max_T = max_T; ss->max_steps = (max_T - 1) * hop;
  ss->tabs = live_tables(h->engine->cfg.mode, mu_law != 0, h->engine->cfg.n_classes, hop);
  ss->e = h->engine; ss->st = static_cast<cudaStream_t>(stream); ss->taps = h->upsampler->d_taps;
  ss->tickets.resize(capacity);
  ss->owner.assign(capacity, -1);
  ss->ready.assign(capacity, nullptr);
  ss->tab.assign(2 * LiveSession::MAX_SLOTS, SesEntry{});
  auto fail = [&](int code) { session_free(ss); return code; };
#define SES_OK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e)); return fail(WRNN_E_CUDA); } } while (0)
  SES_OK(cudaSetDevice(h->engine->device));
  size_t host_bytes = 0;
  rc = grow_mapped(&ss->host, &ss->dev, &host_bytes, LiveSession::SAMPLES_OFF + (size_t)capacity * ss->max_steps * sizeof(float));
  if (rc != WRNN_OK) return fail(rc);
  std::memset(ss->host, 0, LiveSession::SAMPLES_OFF);
  SES_OK(cudaMalloc(&ss->d_ctl, 2 * LiveSession::MAX_SLOTS * sizeof(SesEntry) + 64));
  const size_t rf = (size_t)(max_T + 4) * capacity;
  ss->stage_pitch = align_floats((size_t)max_T * FEAT);
  const size_t n_mf = align_floats(rf * FEAT), n_af = align_floats(rf * cond::CD);
  SES_OK(cudaMalloc(&ss->d_arena, (n_mf + n_af + ss->stage_pitch * capacity) * sizeof(float)));
  ss->mel_frames = static_cast<float*>(ss->d_arena);
  ss->aux_frames = ss->mel_frames + n_mf;
  ss->mel_stage = ss->aux_frames + n_af;
  SES_OK(cudaStreamCreateWithFlags(&ss->side, cudaStreamNonBlocking));
  SES_OK(cudaEventCreateWithFlags(&ss->done, cudaEventDisableTiming));
  for (auto& ev : ss->ready) SES_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
#undef SES_OK
  h->session = ss;
  return WRNN_OK;
}

int wrnn_live_submit(wrnn_t* h, const wrnn_utterance* u, int64_t* ticket) {
  if (!u || !ticket) { set_error("null utterance or ticket"); return WRNN_E_INVALID; }
  const int rc = check_utterance("", u->mel, u->wav, u->T);
  if (rc != WRNN_OK) return rc;
  LiveSession* ss = submit_session(h, u);
  if (!ss) return WRNN_E_INVALID;
  const long long wave_len = (u->T - 1) * ss->hop;
  return session_submit(h, u, cond::Geometry{1, wave_len, wave_len, 0, wave_len}, ss->tabs, ticket);
}

int wrnn_live_submit_batched(wrnn_t* h, const wrnn_utterance* u, int32_t target, int32_t overlap, int64_t* ticket) {
  if (!u || !ticket) { set_error("null utterance or ticket"); return WRNN_E_INVALID; }
  const int rc = check_utterance("", u->mel, u->wav, u->T);
  if (rc != WRNN_OK) return rc;
  if (target <= 0 || overlap <= 0) { set_error("a batched ticket needs target > 0 and overlap > 0"); return WRNN_E_INVALID; }
  LiveSession* ss = submit_session(h, u);
  if (!ss) return WRNN_E_INVALID;
  const cond::Geometry g = cond::fold_geometry(u->T * ss->hop, true, target, overlap);
  if (g.n_seg < 1) { set_error("target / overlap give no fold"); return WRNN_E_INVALID; }
  if (g.n_seg > ss->C) {
    set_error("the utterance has " + std::to_string(g.n_seg) + " folds, more than the session's " + std::to_string(ss->C) +
              " slots: it could never be admitted");
    return WRNN_E_INVALID;
  }
  if (g.seg_len > ss->max_steps) {
    set_error("a fold's target + 2 * overlap = " + std::to_string(g.seg_len) + " samples exceed a slot's row of (max_T - 1) * hop = " +
              std::to_string(ss->max_steps));
    return WRNN_E_INVALID;
  }
  return session_submit(h, u, g, live_tables(ss->e->cfg.mode, !ss->tabs.mu.empty(), ss->e->cfg.n_classes, ss->hop, overlap),
                        ticket);
}

int wrnn_live_cancel(wrnn_t* h, int64_t ticket) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (!h->session) { set_error("no live session is open on this handle (wrnn_live_open)"); return WRNN_E_INVALID; }
  LiveSession& ss = *h->session;
  for (LiveSession::Ticket& tk : ss.tickets) {
    if (tk.state == LiveSession::FREE || tk.ticket != ticket) continue;
    if (!tk.cancelled) {
      tk.cancelled = true;
      for (int b = 0; b < tk.posted; ++b) __atomic_store_n(&ss.mail()[tk.slot[b]].cancel, (unsigned long long)tk.tag, __ATOMIC_RELEASE);
    }
    return WRNN_OK;
  }
  set_error("ticket " + std::to_string(ticket) + " is not in flight in this session");
  return WRNN_E_INVALID;
}

int wrnn_live_poll(wrnn_t* h, int32_t wait_us, wrnn_live_ticket* out, int32_t max_out, int32_t* n_out) {
  if (!out || !n_out) { set_error("null out or n_out"); return WRNN_E_INVALID; }
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (!h->session) { set_error("no live session is open on this handle (wrnn_live_open)"); return WRNN_E_INVALID; }
  LiveSession& ss = *h->session;
  if (max_out < 2 * ss.C) { set_error("max_out must be at least twice the session's capacity"); return WRNN_E_INVALID; }
  *n_out = 0;
  const std::optional<int> rc = wait_for(wait_us > 0 ? wait_us : 0, [&]() -> std::optional<int> {
    const int rc = session_pump(ss);
    if (rc != WRNN_OK || session_deliver(ss) || !ss.released.empty()) return rc;
    return std::nullopt;
  });
  if (rc && *rc != WRNN_OK) return *rc;
  // released tickets first, then every ticket still held (at most C)
  int n = 0, held = 0;
  size_t k = 0;
  for (; k < ss.released.size() && n < max_out - ss.C; ++k) out[n++] = ss.released[k];
  ss.released.erase(ss.released.begin(), ss.released.begin() + k);   // the rest: next poll
  for (const auto& tk : ss.tickets) {
    if (tk.state == LiveSession::FREE) continue;
    ++held;
    out[n++] = wrnn_live_ticket{tk.ticket, tk.delivered, WRNN_LIVE_RUNNING, 0};
  }
  *n_out = n;
  return held > 0 ? 1 : 0;
}

int wrnn_live_close(wrnn_t* h) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (!h->session) { set_error("no live session is open on this handle (wrnn_live_open)"); return WRNN_E_INVALID; }
  LiveSession* ss = h->session;
  for (const auto& tk : ss->tickets)
    if (tk.state != LiveSession::FREE && !tk.cancelled) wrnn_live_cancel(h, tk.ticket);
  const std::optional<int> rc = wait_for(-1, [&]() -> std::optional<int> {   // the launch stops once every cancelled slot is retired
    const int rc = session_pump(*ss);
    if (rc != WRNN_OK) return rc;
    session_deliver(*ss);
    bool held = false;
    for (const auto& tk : ss->tickets) held = held || tk.state != LiveSession::FREE;
    return (!held && !ss->running) ? std::optional<int>(WRNN_OK) : std::nullopt;
  });
  h->session = nullptr;
  session_free(ss);
  return *rc;
}

// Test hook (CPU-only, no device needed): one delivery of wrnn_live_poll on a host buffer laid out as the session's
// pinned one.  Slot s holds ticket[s] (0: free) of T[s] frames, whose samples are x [C][max_steps], published word
// progress[s]; delivered[s] holds what earlier polls delivered and receives what this one did, released[s] whether the
// slot was released; wav is the concatenation of the held tickets' waveforms.  Checked in tests/test_live_session_abi.py.
int wrnn_debug_live_session_deliver(const float* x, int64_t max_steps, const uint64_t* progress, int32_t C,
                                    const int64_t* ticket, const int64_t* T, int32_t hop, int32_t mu_law, int32_t n_classes,
                                    int64_t* delivered, int32_t* released, double* wav) {
  if (!x || !progress || !ticket || !T || !delivered || !released || !wav || max_steps <= 0 || hop <= 0 || C < 1 ||
      C > LiveSession::MAX_SLOTS || (mu_law && n_classes < 2)) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  for (int s = 0; s < C; ++s)
    if (ticket[s] && (T[s] < 21 || (T[s] - 1) * hop > max_steps || delivered[s] < 0 || delivered[s] > (T[s] - 1) * hop)) {
      set_error("bad argument"); return WRNN_E_INVALID;
    }
  std::vector<unsigned char> buf(LiveSession::SAMPLES_OFF + (size_t)C * max_steps * sizeof(float));
  std::memcpy(buf.data(), progress, (size_t)C * sizeof(uint64_t));
  std::memcpy(buf.data() + LiveSession::SAMPLES_OFF, x, (size_t)C * max_steps * sizeof(float));
  LiveSession ss;
  ss.host = buf.data();
  ss.C = C; ss.hop = hop; ss.max_steps = max_steps;
  ss.tickets.resize(C);
  ss.owner.assign(C, -1);
  const LiveTables tabs = live_tables(WRNN_MODE_RAW, mu_law != 0, n_classes, hop);
  double* w = wav;
  for (int s = 0; s < C; ++s) {
    if (!ticket[s]) continue;
    LiveSession::Ticket& tk = ss.tickets[s];
    tk.state = LiveSession::POSTED; tk.ticket = ticket[s]; tk.tag = ses_tag(ticket[s]);
    tk.wave_len = (T[s] - 1) * hop; tk.seg_len = tk.stride = tk.wave_len; tk.delivered = delivered[s]; tk.wav = w;
    tk.slot = {s}; tk.posted = 1; tk.tabs = tabs;
    ss.owner[s] = s;
    w += tk.wave_len;
  }
  session_deliver(ss);
  for (int s = 0; s < C; ++s) {
    released[s] = 0;
    if (!ticket[s]) continue;
    for (const auto& r : ss.released) if (r.ticket == ticket[s]) { released[s] = 1; delivered[s] = r.n_ready; }
    if (!released[s]) delivered[s] = ss.tickets[s].delivered;
  }
  ss.host = nullptr;
  return WRNN_OK;
}

// Test hook (CPU-only, no device needed): one delivery of wrnn_live_poll for ONE batched ticket (T frames, target,
// overlap), on a host buffer laid out as the session's pinned one of C slots: fold b is held by slot slot[b] (n_seg
// entries, fold_with_overlap's count), its samples are row slot[b] of x [C][max_steps] and its published word
// progress[slot[b]].  *delivered holds what earlier polls delivered and receives what this one did; *released whether the
// ticket was released, and free_slots [C] whether each slot is free afterwards.  Checked in tests/test_live_batched_abi.py.
int wrnn_debug_live_batched_deliver(const float* x, int64_t max_steps, const uint64_t* progress, int32_t C, int64_t ticket,
                                    int64_t T, int32_t target, int32_t overlap, const int32_t* slot, int32_t n_seg, int32_t hop,
                                    int32_t mu_law, int32_t n_classes, int64_t* delivered, int32_t* released,
                                    int32_t* free_slots, double* wav) {
  if (!x || !progress || !slot || !delivered || !released || !free_slots || !wav || max_steps <= 0 || hop <= 0 || C < 1 ||
      C > LiveSession::MAX_SLOTS || T < 21 || target <= 0 || overlap <= 0 || (mu_law && n_classes < 2)) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  const cond::Geometry g = cond::fold_geometry(T * hop, true, target, overlap);
  if (g.n_seg != n_seg || g.seg_len > max_steps || *delivered < 0 || *delivered > (T - 1) * hop) { set_error("bad argument"); return WRNN_E_INVALID; }
  std::vector<int> owner(C, -1);
  for (int b = 0; b < n_seg; ++b) {
    if (slot[b] < 0 || slot[b] >= C || owner[slot[b]] >= 0) { set_error("bad argument"); return WRNN_E_INVALID; }
    owner[slot[b]] = slot[0];
  }
  std::vector<unsigned char> buf(LiveSession::SAMPLES_OFF + (size_t)C * max_steps * sizeof(float));
  std::memcpy(buf.data(), progress, (size_t)C * sizeof(uint64_t));
  std::memcpy(buf.data() + LiveSession::SAMPLES_OFF, x, (size_t)C * max_steps * sizeof(float));
  LiveSession ss;
  ss.host = buf.data();
  ss.C = C; ss.hop = hop; ss.max_steps = max_steps;
  ss.tickets.resize(C);
  ss.owner = owner;
  LiveSession::Ticket& tk = ss.tickets[slot[0]];
  tk.state = LiveSession::POSTED; tk.ticket = ticket; tk.tag = ses_tag(ticket);
  tk.wave_len = (T - 1) * hop; tk.seg_len = g.seg_len; tk.stride = g.seg_stride; tk.delivered = *delivered; tk.wav = wav;
  tk.slot.assign(slot, slot + n_seg);
  tk.posted = n_seg;
  tk.tabs = live_tables(WRNN_MODE_RAW, mu_law != 0, n_classes, hop, overlap);
  session_deliver(ss);
  *released = ss.released.empty() ? 0 : 1;
  *delivered = ss.released.empty() ? tk.delivered : ss.released[0].n_ready;
  for (int s = 0; s < C; ++s) free_slots[s] = ss.owner[s] < 0 ? 1 : 0;
  ss.host = nullptr;
  return WRNN_OK;
}

// Test hook (CPU-only, no device needed): a relaunch's decision for ONE posted batched ticket (T frames, target, overlap;
// cancelled or not) on a session of C slots whose launch has exited: fold b is held by slot slot[b] (n_seg entries) and
// folds 0 .. posted - 1 were posted.  progress [C] holds each slot's word and receives what the host wrote; req [C]
// receives each slot's mailbox tag (0 where nothing was posted or withdrawn); entry [C][4] the version -1 table entry of
// each slot (steps, fold, row0 - the ticket's first row, rows; steps 0: not admitted); *launch whether a launch is
// needed, *released whether the ticket was released.  Returns the decision's code (WRNN_E_CUDA: a fold still held).
// Checked in tests/test_live_batched_abi.py.
int wrnn_debug_live_batched_relaunch(uint64_t* progress, int32_t C, int64_t ticket, int64_t T, int32_t target, int32_t overlap,
                                     const int32_t* slot, int32_t n_seg, int32_t posted, int32_t cancelled, int32_t hop,
                                     uint64_t* req, int64_t* entry, int32_t* launch, int32_t* released) {
  if (!progress || !slot || !req || !entry || !launch || !released || C < 1 || C > LiveSession::MAX_SLOTS || T < 21 ||
      target <= 0 || overlap <= 0 || hop <= 0 || posted < 0 || posted > n_seg) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  const cond::Geometry g = cond::fold_geometry(T * hop, true, target, overlap);
  if (g.n_seg != n_seg) { set_error("bad argument"); return WRNN_E_INVALID; }
  std::vector<int> owner(C, -1);
  for (int b = 0; b < n_seg; ++b) {
    if (slot[b] < 0 || slot[b] >= C || owner[slot[b]] >= 0) { set_error("bad argument"); return WRNN_E_INVALID; }
    owner[slot[b]] = slot[0];
  }
  std::vector<unsigned char> buf(LiveSession::SAMPLES_OFF, 0);
  std::memcpy(buf.data(), progress, (size_t)C * sizeof(uint64_t));
  LiveSession ss;
  ss.host = buf.data();
  ss.C = C; ss.hop = hop;
  ss.tickets.resize(C);
  ss.owner = owner;
  ss.tab.assign(2 * LiveSession::MAX_SLOTS, SesEntry{});
  for (int b = 0; b < posted; ++b) ss.mail()[slot[b]].req = ses_tag(ticket);
  LiveSession::Ticket& tk = ss.tickets[slot[0]];
  tk.state = LiveSession::POSTED; tk.ticket = ticket; tk.tag = ses_tag(ticket);
  tk.wave_len = (T - 1) * hop; tk.seg_len = g.seg_len; tk.stride = g.seg_stride; tk.rows = T * hop;
  tk.slot.assign(slot, slot + n_seg);
  tk.posted = posted;
  tk.cancelled = cancelled != 0;
  bool go = false;
  const int rc = relaunch_ticket(ss, tk, go);
  std::memcpy(progress, buf.data(), (size_t)C * sizeof(uint64_t));
  for (int s = 0; s < C; ++s) {
    const SesEntry& e = ss.tab[LiveSession::MAX_SLOTS + s];
    req[s] = ss.mail()[s].req;
    entry[4 * s] = e.e - e.a; entry[4 * s + 1] = e.fold; entry[4 * s + 2] = e.row0; entry[4 * s + 3] = e.rows;
  }
  *launch = go ? 1 : 0;
  *released = ss.released.empty() ? 0 : 1;
  ss.host = nullptr;
  return rc;
}

// Test hook (device tests): at most n folds are posted per pass of the open session's host loop on h (a submit makes one,
// a poll one per 100 us of its wait, one with wait_us <= 0), so that a ticket's folds reach the kernel at different
// boundaries or launches.  The default is 64.
int wrnn_debug_live_post_limit(wrnn_t* h, int32_t n) {
  if (!h || !h->session || n < 1) { set_error("bad argument: an open live session and n >= 1"); return WRNN_E_INVALID; }
  h->session->post_limit = n;
  return WRNN_OK;
}

// Test hook (CPU-only): a ticket's 32-bit tag, and CTA 0's decision for one slot at boundary b (the functions the kernel
// runs).  state = {tag, a, e, retired}; words[0] / words[1]: the retirement and admission words published (0: none).
uint32_t wrnn_debug_live_tag(int64_t ticket) { return ses_tag(ticket); }
int wrnn_debug_live_session_slot(int64_t* state, uint64_t* seed, int32_t b, uint32_t req_tag, uint32_t cancel_tag,
                                 uint64_t req_seed, int64_t req_steps, uint64_t* words) {
  if (!state || !seed || !words || b < 0 || b % SES_PERIOD || req_steps < 1 || req_steps > SES_MAX_STEPS) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  SesSlot s{(unsigned)state[0], (int)state[1], (int)state[2], *seed, state[3] != 0};
  words[0] = ses_retire_cancel(s, b, cancel_tag);
  words[1] = 0;
  if (ses_admits(s, b, req_tag)) words[1] = ses_admit(s, b, req_tag, req_seed, req_steps, 0u, 0, (int)req_steps);
  state[0] = s.tag; state[1] = s.a; state[2] = s.e; state[3] = s.retired ? 1 : 0;
  *seed = s.seed;
  return WRNN_OK;
}

// Test hook (CPU-only): the same decision for a slot whose occupant (and request) is a fold of a batched utterance.
// state = {tag, a, e, retired, fold, row0, rows}; the request's fold, first row and row count are req_fold, req_row0 and
// req_rows.
int wrnn_debug_live_session_fold_slot(int64_t* state, uint64_t* seed, int32_t b, uint32_t req_tag, uint32_t cancel_tag,
                                      uint64_t req_seed, int64_t req_steps, uint32_t req_fold, int32_t req_row0, int32_t req_rows,
                                      uint64_t* words) {
  if (!state || !seed || !words || b < 0 || b % SES_PERIOD || req_steps < 1 || req_steps > SES_MAX_STEPS || req_row0 < 0 ||
      req_rows < 1) {
    set_error("bad argument"); return WRNN_E_INVALID;
  }
  SesSlot s{(unsigned)state[0], (int)state[1], (int)state[2], *seed, state[3] != 0, (unsigned)state[4], (int)state[5], (int)state[6]};
  words[0] = ses_retire_cancel(s, b, cancel_tag);
  words[1] = 0;
  if (ses_admits(s, b, req_tag)) words[1] = ses_admit(s, b, req_tag, req_seed, req_steps, req_fold, req_row0, req_rows);
  state[0] = s.tag; state[1] = s.a; state[2] = s.e; state[3] = s.retired ? 1 : 0;
  state[4] = s.fold; state[5] = s.row0; state[6] = s.rows;
  *seed = s.seed;
  return WRNN_OK;
}

}  // extern "C"
