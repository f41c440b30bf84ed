// wrnn_capi.cu -- the extern "C" surface declared in include/wavernn_b200.h.
#include <cuda_runtime.h>

#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "wrnn_engine.h"
#include "wrnn_stream_plan.h"

namespace wrnn {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }

static int fetch(std::vector<float>& dst, const float* src, size_t n, const char* what) {
  if (!src) { set_error(std::string("null weight pointer: ") + what); return WRNN_E_INVALID; }
  dst.resize(n);
  // cudaMemcpyDefault resolves host or device pointers through UVA
  cudaError_t e = cudaMemcpy(dst.data(), src, n * sizeof(float), cudaMemcpyDefault);
  if (e != cudaSuccess) { set_error(std::string("copying ") + what + ": " + cudaGetErrorString(e)); return WRNN_E_CUDA; }
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
  hw.n_classes = cfg->n_classes;
  const size_t W2W = H + AUXD;
  int rc;
#define FETCH(field, src, n) if ((rc = fetch(hw.field, w->src, (n), #src)) != WRNN_OK) return rc
  FETCH(I_w, I_weight, (size_t)H * (1 + F1IN)); FETCH(I_b, I_bias, H);
  FETCH(w1i, rnn1_weight_ih, (size_t)G3 * H); FETCH(w1h, rnn1_weight_hh, (size_t)G3 * H);
  FETCH(b1i, rnn1_bias_ih, G3); FETCH(b1h, rnn1_bias_hh, G3);
  FETCH(w2i, rnn2_weight_ih, (size_t)G3 * W2W); FETCH(w2h, rnn2_weight_hh, (size_t)G3 * H);
  FETCH(b2i, rnn2_bias_ih, G3); FETCH(b2h, rnn2_bias_hh, G3);
  FETCH(f1w, fc1_weight, (size_t)H * W2W); FETCH(f1b, fc1_bias, H);
  FETCH(f2w, fc2_weight, (size_t)H * W2W); FETCH(f2b, fc2_bias, H);
  FETCH(f3w, fc3_weight, (size_t)cfg->n_classes * H); FETCH(f3b, fc3_bias, cfg->n_classes);
#undef FETCH
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
  if (h->d_stage) cudaFree(h->d_stage);
  delete h->engine;
  delete h->fallback;
  delete h->stream;
  delete h->host_weights;
  delete h;
}

static int validate(const wrnn_t* h, const wrnn_job* job, bool host) {
  if (!h || !h->engine || !job) { set_error("null handle or job"); return WRNN_E_INVALID; }
  if (!job->out) { set_error("out is required"); return WRNN_E_INVALID; }
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
  int rc = validate(h, job, false);
  if (rc != WRNN_OK) return rc;
  Engine* e = nullptr;
  if ((rc = pick_engine(h, job, &e)) != WRNN_OK) return rc;
  h->last = e;
  return e->generate(*job, static_cast<cudaStream_t>(stream));
}

int wrnn_check(wrnn_t* h) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  return h->last->check();
}

int wrnn_generate_host(wrnn_t* h, const wrnn_job* job) {
  int rc = validate(h, job, true);
  if (rc != WRNN_OK) return rc;
  Engine* e = nullptr;
  if ((rc = pick_engine(h, job, &e)) != WRNN_OK) return rc;
  h->last = e;
  WRNN_CUDA_OK(cudaSetDevice(e->device));
  const size_t S = job->steps > 0 ? job->steps : job->seg_len;
  const size_t B = job->n_seg, NC = e->cfg.n_classes;
  const size_t n_mel = (size_t)job->L * FEAT, n_aux = (size_t)job->L * 4 * AUXD;
  const size_t n_uni = job->uniforms ? S * 11 * B : 0, n_exp = job->expo ? S * B * NC : 0;
  const size_t n_xf = job->x_force ? S * B : 0, n_out = B * S, n_log = job->logits_out ? S * B * NC : 0;
  const size_t n_tab = job->fold_row0 ? 4 * B : 0;   // two int64 tables, counted in floats
  const size_t total = (n_mel + n_aux + n_uni + n_exp + n_xf + n_out + n_log + n_tab + 2) * sizeof(float);
  if (total > h->stage_bytes) {
    if (h->d_stage) cudaFree(h->d_stage);
    h->d_stage = nullptr; h->stage_bytes = 0;
    WRNN_CUDA_OK(cudaMalloc(&h->d_stage, total));
    h->stage_bytes = total;
  }
  float* d = static_cast<float*>(h->d_stage);
  wrnn_job dj = *job;
  auto up = [&](const float* src, size_t n) -> float* {
    if (!n) return nullptr;
    float* p = d; d += n;
    cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyHostToDevice, 0);
    return p;
  };
  dj.mels_up = up(job->mels_up, n_mel); dj.aux = up(job->aux, n_aux);
  dj.uniforms = up(job->uniforms, n_uni); dj.expo = up(job->expo, n_exp); dj.x_force = up(job->x_force, n_xf);
  dj.out = d; d += n_out;
  dj.logits_out = n_log ? d : nullptr; d += n_log;
  if (n_tab) {
    d = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(d) + 7) & ~uintptr_t(7));
    int64_t* t0 = reinterpret_cast<int64_t*>(d);
    cudaMemcpyAsync(t0, job->fold_row0, B * 8, cudaMemcpyHostToDevice, 0);
    cudaMemcpyAsync(t0 + B, job->fold_row_end, B * 8, cudaMemcpyHostToDevice, 0);
    dj.fold_row0 = t0; dj.fold_row_end = t0 + B;
  }
  rc = e->generate(dj, 0);
  if (rc != WRNN_OK) return rc;
  WRNN_CUDA_OK(cudaMemcpyAsync(job->out, dj.out, n_out * sizeof(float), cudaMemcpyDeviceToHost, 0));
  if (n_log) WRNN_CUDA_OK(cudaMemcpyAsync(job->logits_out, dj.logits_out, n_log * sizeof(float), cudaMemcpyDeviceToHost, 0));
  WRNN_CUDA_OK(cudaStreamSynchronize(0));
  return e->check();
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

// Test hook (CPU-only, no device needed): the stream engine's packed weight stream and step program for host-resident
// weights, so the packing and the schedule can be interpreted and checked without a GPU (tests/test_stream_plan.py).
// Call with blob == NULL to obtain the sizes.  Not part of the reference-facing surface.
int wrnn_debug_stream_plan(const wrnn_cfg* cfg, const wrnn_weights* w, uint8_t* blob, uint64_t* blob_bytes, uint8_t* prog,
                           uint64_t* n_chunks, float* vectors /* qk[4096] vq[4096] b1h[1536] b2h[1536] b3[128] */,
                           uint16_t* mine /* [4][n_chunks]: per issuing warp, its chunk indices; unused tail = 0xffff */,
                           int32_t only_block /* -1: the whole program; 0..3: the share of that rank of a 4-CTA cluster */) {
  if (!cfg || !w || !blob_bytes || !n_chunks) { set_error("null argument"); return WRNN_E_INVALID; }
  HostWeights hw;
  hw.n_classes = cfg->n_classes;
  const size_t W2W = H + AUXD;
  auto take = [&](std::vector<float>& dst, const float* src, size_t n) { dst.assign(src, src + n); };
  take(hw.I_w, w->I_weight, (size_t)H * (1 + F1IN)); take(hw.I_b, w->I_bias, H);
  take(hw.w1i, w->rnn1_weight_ih, (size_t)G3 * H); take(hw.w1h, w->rnn1_weight_hh, (size_t)G3 * H);
  take(hw.b1i, w->rnn1_bias_ih, G3); take(hw.b1h, w->rnn1_bias_hh, G3);
  take(hw.w2i, w->rnn2_weight_ih, (size_t)G3 * W2W); take(hw.w2h, w->rnn2_weight_hh, (size_t)G3 * H);
  take(hw.b2i, w->rnn2_bias_ih, G3); take(hw.b2h, w->rnn2_bias_hh, G3);
  take(hw.f1w, w->fc1_weight, (size_t)H * W2W); take(hw.f1b, w->fc1_bias, H);
  take(hw.f2w, w->fc2_weight, (size_t)H * W2W); take(hw.f2b, w->fc2_bias, H);
  take(hw.f3w, w->fc3_weight, (size_t)cfg->n_classes * H); take(hw.f3b, w->fc3_bias, cfg->n_classes);
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
    std::memcpy(v, plan.b3.data(), stream::MROWS * 4);
    if (mine) {
      std::memset(mine, 0xff, sizeof(uint16_t) * stream::N_ISSUERS * plan.prog.size());
      for (int o = 0; o < stream::N_ISSUERS; ++o) std::memcpy(mine + (size_t)o * plan.prog.size(), plan.mine[o].data(), plan.mine[o].size() * sizeof(uint16_t));
    }
  }
  *blob_bytes = plan.blob.size(); *n_chunks = plan.prog.size();
  return WRNN_OK;
}

}  // extern "C"
