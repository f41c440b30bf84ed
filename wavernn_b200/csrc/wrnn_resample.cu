// wrnn_resample.cu -- the resampling step of the reference's load_wav (librosa.load(path, sr) with librosa 0.6.3's
// default res_type, resampy's kaiser_best) on the device: wrnn_resample_many and its host hook.
//
// One thread per output sample of every utterance of a batch, in one launch; each block stages the input span its
// outputs read in shared memory and reads the filter table through L2.  Every output is a __host__ __device__ function
// of its index alone (the time register is t * (1 / ratio), not a running sum), so wrnn_debug_resample runs the same
// source on the host.  The arithmetic is resampy's resample_f, rounded step by step (DESIGN.md §3.10).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "wrnn_device.cuh"
#include "wrnn_engine.h"
#include "wrnn_mel.h"

namespace wrnn {
namespace rs {

constexpr int THREADS = 256;
constexpr int ZEROS = 64;                                     // zero crossings of the half-window
constexpr int PRECISION = 16;                                 // table entries per zero crossing: 2^PRECISION
constexpr long long NUM_TABLE = 1ll << PRECISION;
constexpr long long NWIN = ZEROS * NUM_TABLE + 1;             // entries of the half-window
constexpr double BETA = 14.769656459379492;
constexpr double ROLLOFF = 0.9475937167399596;
constexpr int STAGE_MAX = 12288;                              // staged input floats per block (48 KB)

// The half-window as resampy's sinc_window builds it in float64, plus one copy of its last entry, so that the
// difference formed at the last entry is interp_delta's 0:
//   rolloff * sinc(rolloff * linspace(0, 64, 64 * 2^p + 1)) * kaiser(2 * 64 * 2^p + 1, beta)[64 * 2^p:]
// np.sinc(x) = sin(pi x') / (pi x') with x' = x, or 1e-20 at 0; scipy's kaiser is i0(beta sqrt(1 - (k / N)^2)) /
// i0(beta), i0 here by its power series in long double (positive terms), rounded once.
static double bessel_i0(double x) {
  const long double q = 0.25L * x * x;
  long double term = 1.0L, sum = 1.0L;
  for (int k = 1; term > 1e-21L * sum; ++k) {
    term *= q / ((long double)k * k);
    sum += term;
  }
  return (double)sum;
}

static void build_table(std::vector<double>& win) {
  win.resize(NWIN + 1);
  const double i0b = bessel_i0(BETA), N = (double)(NWIN - 1);
  for (long long k = 0; k < NWIN; ++k) {
    const double x = ROLLOFF * std::ldexp((double)k, -PRECISION);
    const double y = M_PI * (x == 0.0 ? 1.0e-20 : x);
    const double sinc = ROLLOFF * (std::sin(y) / y);
    const double r = (double)k / N;
    const double taper = bessel_i0(BETA * std::sqrt(1.0 - r * r)) / i0b;
    win[k] = taper * sinc;
  }
  win[NWIN] = win[NWIN - 1];
}

static const std::vector<double>& host_table() {
  static std::vector<double> win;
  static std::once_flag once;
  std::call_once(once, [] { build_table(win); });
  return win;
}

// One utterance of a launch, its blocks block0 .. block0 + ceil(n_len / THREADS) - 1 of the grid.
struct RsUtt {
  const float* x;
  long long n;          // input samples
  float* y;
  long long n_out;      // int(n * ratio): resampy's samples
  long long n_len;      // ceil(n * ratio): written samples (the ones past n_out are 0)
  long long block0;
  double ratio;         // sr_out / sr_in
  double scale;         // min(1, ratio)
  double inc;           // 1 / ratio
  int step;             // index_step = int(scale * 2^p)
  int copy;             // equal rates: y = x
};

__host__ __device__ inline long long lmin(long long a, long long b) { return a < b ? a : b; }
__host__ __device__ inline long long lmax(long long a, long long b) { return a > b ? a : b; }

// The time register of output t and its input index n = int(t * inc).
__host__ __device__ inline double time_of(const RsUtt& u, long long t) { return dmul_rn((double)t, u.inc); }

// Taps of one wing: weight = w[j] + eta * (w[j + 1] - w[j]) on the table scaled by ratio when it is below 1, and
// y = float32(y + weight * x) after each tap.  xs[j - lo] is input sample j; `dir` -1 reads n, n - 1, ..., +1 reads
// n + 1, n + 2, ...
__host__ __device__ inline float wing(const double* __restrict__ win, const RsUtt& u, const float* xs, long long lo,
                                      long long n, double frac, long long limit, int dir, float y) {
  const double index_frac = dmul_rn(frac, (double)NUM_TABLE);
  const long long offset = (long long)index_frac;
  const double eta = dadd_rn(index_frac, -(double)offset);
  const long long taps = lmin(limit, (NWIN - offset) / u.step);
  const bool down = u.ratio < 1.0;
  const float* src = xs + (n - lo) + (dir > 0 ? 1 : 0);
  for (long long i = 0; i < taps; ++i) {
    const long long j = offset + i * u.step;
#ifdef __CUDA_ARCH__
    double w0 = __ldg(win + j), w1 = __ldg(win + j + 1);
#else
    double w0 = win[j], w1 = win[j + 1];
#endif
    if (down) {
      w0 = dmul_rn(w0, u.ratio);
      w1 = dmul_rn(w1, u.ratio);
    }
    const double weight = dadd_rn(w0, dmul_rn(eta, dadd_rn(w1, -w0)));
    const float xv = src[dir > 0 ? i : -i];
    y = (float)dadd_rn((double)y, dmul_rn(weight, (double)xv));
  }
  return y;
}

// Output t < n_out of utterance u: resampy's left wing, then its right wing.
__host__ __device__ inline float output(const double* __restrict__ win, const RsUtt& u, const float* xs, long long lo,
                                        long long t) {
  const double tr = time_of(u, t);
  const long long n = (long long)tr;
  const double frac = dmul_rn(u.scale, dadd_rn(tr, -(double)n));
  float y = wing(win, u, xs, lo, n, frac, n + 1, -1, 0.f);
  return wing(win, u, xs, lo, n, dadd_rn(u.scale, -frac), u.n - n - 1, +1, y);
}

// Widest wing: (NWIN - offset) / step taps at most.
__host__ __device__ inline long long max_taps(const RsUtt& u) { return (NWIN + u.step - 1) / u.step; }

__global__ void __launch_bounds__(THREADS) resample_kernel(const double* __restrict__ win, const RsUtt* __restrict__ utts,
                                                           int n_utts, int stage_cap) {
  extern __shared__ float xs[];
  const long long b = blockIdx.x;
  int lo_u = 0, hi_u = n_utts - 1;
  while (lo_u < hi_u) {
    const int mid = (lo_u + hi_u + 1) >> 1;
    if (utts[mid].block0 <= b) lo_u = mid; else hi_u = mid - 1;
  }
  const RsUtt u = utts[lo_u];
  const long long t0 = (b - u.block0) * THREADS, t = t0 + threadIdx.x;
  if (u.copy) {
    if (t < u.n_len) u.y[t] = u.x[t];
    return;
  }
  // the span of input this block's outputs read, staged when it fits
  const long long t_last = lmin(t0 + THREADS, u.n_out) - 1;
  const float* src = u.x;
  long long lo = 0;
  if (t_last >= t0) {
    const long long w = max_taps(u);
    const long long a = lmax(0, (long long)time_of(u, t0) - w);
    const long long e = lmin(u.n - 1, (long long)time_of(u, t_last) + w + 1);
    if (e - a + 1 <= stage_cap) {
      for (long long j = threadIdx.x; j <= e - a; j += THREADS) xs[j] = u.x[a + j];
      __syncthreads();
      src = xs;
      lo = a;
    }
  }
  if (t < u.n_out) u.y[t] = output(win, u, src, lo, t);
  else if (t < u.n_len) u.y[t] = 0.f;
}

// Checks a batch and lays out its launch table (pointers as given).  WRNN_E_INVALID with a message; no CUDA call.
static int plan(int sr_out, const wrnn_resample_utt* u, int n_utts, std::vector<RsUtt>& tab) {
  if (!u || n_utts < 1) { set_error("wrnn_resample_many needs a non-null utterance array and n_utts >= 1"); return WRNN_E_INVALID; }
  tab.assign(n_utts, RsUtt{});
  long long total = 0, block = 0;
  for (int i = 0; i < n_utts; ++i) {
    const std::string at = "utterance " + std::to_string(i) + ": ";
    if (!u[i].x || !u[i].y) { set_error(at + "x and y are required"); return WRNN_E_INVALID; }
    if (u[i].sample_rate <= 0) { set_error(at + "sample_rate must be > 0"); return WRNN_E_INVALID; }
    if (u[i].n < 1) { set_error(at + "n must be >= 1"); return WRNN_E_INVALID; }
    RsUtt& r = tab[i];
    r.x = u[i].x;
    r.n = u[i].n;
    r.y = u[i].y;
    r.copy = u[i].sample_rate == sr_out;
    r.ratio = (double)sr_out / u[i].sample_rate;
    r.scale = std::min(1.0, r.ratio);
    r.inc = 1.0 / r.ratio;
    const double len = (double)u[i].n * r.ratio;
    r.n_out = r.copy ? r.n : (long long)len;
    r.n_len = r.copy ? r.n : (long long)std::ceil(len);
    if (r.n_out < 1) {
      set_error(at + "n = " + std::to_string(u[i].n) + " at " + std::to_string(u[i].sample_rate) + " Hz gives no output sample at " +
                std::to_string(sr_out) + " Hz");
      return WRNN_E_INVALID;
    }
    const double step = r.scale * (double)NUM_TABLE;
    if (!r.copy && step < 1.0) {
      set_error(at + "the ratio " + std::to_string(sr_out) + " / " + std::to_string(u[i].sample_rate) + " is below 2^-16");
      return WRNN_E_INVALID;
    }
    r.step = (int)step;
    if (r.n_len >= (1ll << 31) - total) { set_error("a batch must have fewer than 2^31 output samples"); return WRNN_E_INVALID; }
    total += r.n_len;
    r.block0 = block;
    block += (r.n_len + THREADS - 1) / THREADS;
  }
  return WRNN_OK;
}

// Staged floats per block: the widest span any block of the batch reads, at most STAGE_MAX.
static int stage_cap(const std::vector<RsUtt>& tab) {
  long long cap = 0;
  for (const RsUtt& r : tab)
    if (!r.copy) cap = std::max<long long>(cap, (long long)std::ceil((THREADS - 1) * r.inc) + 2 * max_taps(r) + 4);
  return (int)std::min<long long>(cap, STAGE_MAX);
}

static int ensure_table(const wrnn_mel_plan& m) {
  std::lock_guard<std::mutex> lock(m.rs_mu);
  if (m.d_rs_win) return WRNN_OK;
  const std::vector<double>& win = host_table();
  double* d = nullptr;
  cudaError_t e = cudaMalloc(&d, win.size() * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(d, win.data(), win.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    cudaGetLastError();
    set_error(std::string("wrnn_resample_many: filter table upload failed: ") + cudaGetErrorString(e));
    return WRNN_E_CUDA;
  }
  m.d_rs_win = d;
  return WRNN_OK;
}

static int launch(const wrnn_mel_plan& m, std::vector<RsUtt> tab, cudaStream_t st) {
  const int n = (int)tab.size();
  WRNN_CUDA_OK(cudaSetDevice(m.device));
  const int rc = ensure_table(m);
  if (rc != WRNN_OK) return rc;
  const RsUtt& last = tab.back();
  const long long blocks = last.block0 + (last.n_len + THREADS - 1) / THREADS;
  const int cap = stage_cap(tab);
  // the table lives for this launch only, so that calls on any streams share the analysis object
  void* d = nullptr;
  WRNN_CUDA_OK(cudaMallocAsync(&d, n * sizeof(RsUtt), st));
  WRNN_CUDA_OK(cudaMemcpyAsync(d, tab.data(), n * sizeof(RsUtt), cudaMemcpyHostToDevice, st));
  resample_kernel<<<(unsigned)blocks, THREADS, (size_t)cap * sizeof(float), st>>>(m.d_rs_win, static_cast<RsUtt*>(d), n, cap);
  WRNN_CUDA_OK(cudaGetLastError());
  WRNN_CUDA_OK(cudaFreeAsync(d, st));
  return WRNN_OK;
}

}  // namespace rs
}  // namespace wrnn

using namespace wrnn;

extern "C" {

int64_t wrnn_resample_length(int64_t n, int32_t sr_in, int32_t sr_out) {
  if (n < 0 || sr_in <= 0 || sr_out <= 0) return -1;
  if (sr_in == sr_out) return n;
  return (int64_t)std::ceil((double)n * ((double)sr_out / sr_in));
}

int wrnn_resample_many(const wrnn_mel_t* m, const wrnn_resample_utt* u, int32_t n_utts, void* stream) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<rs::RsUtt> tab;
  const int rc = rs::plan(m->cfg.sample_rate, u, n_utts, tab);
  if (rc != WRNN_OK) return rc;
  return rs::launch(*m, std::move(tab), static_cast<cudaStream_t>(stream));
}

int wrnn_resample_many_host(const wrnn_mel_t* m, const wrnn_resample_utt* u, int32_t n_utts) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<rs::RsUtt> tab;
  int rc = rs::plan(m->cfg.sample_rate, u, n_utts, tab);
  if (rc != WRNN_OK) return rc;
  const int n = n_utts;
  // one device block [x_0 | .. | x_{n-1} | y_0 | ..], each region 256-B aligned
  std::vector<size_t> off(2 * n + 1, 0);
  for (int i = 0; i < 2 * n; ++i) {
    const size_t bytes = (size_t)(i < n ? tab[i].n : tab[i - n].n_len) * sizeof(float);
    off[i + 1] = off[i] + ((bytes + 255) & ~size_t(255));
  }
  WRNN_CUDA_OK(cudaSetDevice(m->device));
  char* d = nullptr;
  WRNN_CUDA_OK(cudaMalloc(&d, off[2 * n]));
  std::vector<rs::RsUtt> dtab = tab;
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < n && e == cudaSuccess; ++i) {
    dtab[i].x = reinterpret_cast<float*>(d + off[i]);
    dtab[i].y = reinterpret_cast<float*>(d + off[n + i]);
    e = cudaMemcpyAsync(d + off[i], u[i].x, (size_t)u[i].n * sizeof(float), cudaMemcpyDefault, 0);
  }
  if (e == cudaSuccess) {
    rc = rs::launch(*m, dtab, 0);
    for (int i = 0; i < n && rc == WRNN_OK && e == cudaSuccess; ++i)
      e = cudaMemcpyAsync(u[i].y, dtab[i].y, (size_t)tab[i].n_len * sizeof(float), cudaMemcpyDefault, 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);
  }
  cudaFree(d);
  if (e != cudaSuccess) { set_error(std::string("wrnn_resample_many_host: ") + cudaGetErrorString(e)); return WRNN_E_CUDA; }
  return rc;
}

// ---- test hooks (not declared in the header) ------------------------------------------------------------------------
// The host half-window: its entry count, and the entries themselves into win unless it is NULL.
int64_t wrnn_debug_resample_table(double* win) {
  const std::vector<double>& t = rs::host_table();
  if (win) std::copy(t.begin(), t.begin() + rs::NWIN, win);
  return rs::NWIN;
}

// The kernel's per-output function run on the host, output after output, for a batch resampled to sr_out (HOST x / y;
// the same checks and messages as wrnn_resample_many).
int wrnn_debug_resample(const wrnn_resample_utt* u, int32_t n_utts, int32_t sr_out) {
  if (sr_out <= 0) { set_error("wrnn_debug_resample: sr_out must be > 0"); return WRNN_E_INVALID; }
  std::vector<rs::RsUtt> tab;
  const int rc = rs::plan(sr_out, u, n_utts, tab);
  if (rc != WRNN_OK) return rc;
  const double* win = rs::host_table().data();
  for (const rs::RsUtt& r : tab) {
    if (r.copy) { std::memcpy(r.y, r.x, (size_t)r.n * sizeof(float)); continue; }
    for (long long t = 0; t < r.n_len; ++t) r.y[t] = t < r.n_out ? rs::output(win, r, r.x, 0, t) : 0.f;
  }
  return WRNN_OK;
}

}  // extern "C"
