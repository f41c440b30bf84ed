// wrnn_mel.cu -- the reference's melspectrogram(y) (utils/dsp.py:72-81) on the device: wrnn_mel_create,
// wrnn_melspectrogram_many and their host hooks.
//
// One CTA per frame of every utterance of a batch, in one launch.  The frame's n_fft windowed samples are packed as
// n_fft / 2 complex points (even samples real, odd imaginary), transformed by a radix-2 Stockham FFT in float64 in
// shared memory and unpacked into the n_fft / 2 + 1 bins of the real transform.  Each bin is rounded to complex64, as
// librosa 0.6.3's stft(dtype=np.complex64) stores it, before its magnitude is taken; everything after that sums
// non-negative terms in float64 (DESIGN.md §3.8).  Each step of a frame is a __host__ __device__ function of
// (thread index, stage), so wrnn_debug_mel_frames runs the same source on the host.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "wrnn_engine.h"
#include "wrnn_mel.h"

namespace wrnn {
namespace mel {

constexpr int THREADS = 256;

// The tables, host or device: window [n_fft], twiddles tw[m] = e^{-2 pi i m / n_fft} for m < n_fft / 2, the packed
// filterbank and, per band, its first nonzero bin, bin count and offset into basis.
struct Tabs {
  int n_fft, hop, n_mels;
  double min_level_db;
  const double* window;
  const double2* tw;
  const double* basis;
  const int* bands;   // [n_mels][3]: lo, count, offset
};

struct HostTabs {
  std::vector<double> window, tw, basis;   // tw interleaved (re, im)
  std::vector<int> bands;
  std::vector<double> dense;               // [n_mels][n_fft / 2 + 1], the filterbank before packing
};

// librosa 0.6.3's Slaney mel scale (filters.py hz_to_mel / mel_to_hz, htk=False).
static double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
static double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}
// numpy.linspace(start, stop, num): i * step + start, the last element stop.
static std::vector<double> linspace(double start, double stop, int num) {
  std::vector<double> y(num);
  const double step = (stop - start) / (num - 1);
  for (int i = 0; i < num; ++i) y[i] = i * step + start;
  y[num - 1] = stop;
  return y;
}

static void build_tables(const wrnn_mel_cfg& c, HostTabs& t) {
  const int N = c.n_fft, nb = N / 2 + 1, W = c.win_length, M = c.n_mels;
  // scipy.signal.get_window('hann', W, fftbins=True): 0.5 + 0.5 cos(linspace(-pi, pi, W + 1)[n]), centred as pad_center;
  // a one-sample window is [1] (scipy's length guard, as torch.hann_window(1)), not the formula's 0
  t.window.assign(N, 0.0);
  const double step = 2 * M_PI / W;
  for (int n = 0; n < W; ++n) t.window[(N - W) / 2 + n] = W == 1 ? 1.0 : 0.5 + 0.5 * std::cos(n * step + -M_PI);
  t.tw.resize(N);
  for (int m = 0; m < N / 2; ++m) {
    t.tw[2 * m] = std::cos(2 * M_PI * m / N);
    t.tw[2 * m + 1] = -std::sin(2 * M_PI * m / N);
  }
  // filters.mel(sr, n_fft, n_mels, fmin, fmax = sr / 2, htk=False, norm=1)
  const std::vector<double> fft = linspace(0, c.sample_rate / 2.0, nb);
  const std::vector<double> mls = linspace(hz_to_mel(c.fmin), hz_to_mel(c.sample_rate / 2.0), M + 2);
  std::vector<double> mel_f(M + 2);
  for (int i = 0; i < M + 2; ++i) mel_f[i] = mel_to_hz(mls[i]);
  t.dense.assign((size_t)M * nb, 0.0);
  t.basis.clear();
  t.bands.assign(3 * M, 0);
  for (int i = 0; i < M; ++i) {
    const double fd0 = mel_f[i + 1] - mel_f[i], fd1 = mel_f[i + 2] - mel_f[i + 1];
    const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
    int lo = -1, hi = -1;
    for (int k = 0; k < nb; ++k) {
      const double lower = -(mel_f[i] - fft[k]) / fd0, upper = (mel_f[i + 2] - fft[k]) / fd1;
      const double w = std::fmax(0.0, std::fmin(lower, upper)) * enorm;
      t.dense[(size_t)i * nb + k] = w;
      if (w > 0) { if (lo < 0) lo = k; hi = k; }
    }
    t.bands[3 * i] = lo < 0 ? 0 : lo;
    t.bands[3 * i + 1] = lo < 0 ? 0 : hi - lo + 1;
    t.bands[3 * i + 2] = (int)t.basis.size();
    for (int k = lo; lo >= 0 && k <= hi; ++k) t.basis.push_back(t.dense[(size_t)i * nb + k]);
  }
}

static Tabs host_view(const wrnn_mel_cfg& c, const HostTabs& t) {
  return Tabs{c.n_fft, c.hop_length, c.n_mels, (double)c.min_level_db, t.window.data(),
              reinterpret_cast<const double2*>(t.tw.data()), t.basis.data(), t.bands.data()};
}

// ---- one frame, step by step ---------------------------------------------------------------------------------------
// np.pad(y, n_fft / 2, mode='reflect')[i], computed by index (n > n_fft / 2: one reflection suffices).
__host__ __device__ inline double padded(const float* y, long long n, int half, long long i) {
  long long j = i - half;
  if (j < 0) j = -j;
  if (j >= n) j = 2 * (n - 1) - j;
  return (double)y[j];
}
// Packed point k < n_fft / 2 of the frame starting at padded sample `start`: samples 2k and 2k + 1, windowed.
__host__ __device__ inline void load_point(const Tabs& tb, const float* y, long long n, long long start, int k, double2* z) {
  const int half = tb.n_fft / 2;
  z[k] = make_double2(tb.window[2 * k] * padded(y, n, half, start + 2 * k),
                      tb.window[2 * k + 1] * padded(y, n, half, start + 2 * k + 1));
}
// Butterfly j < n_fft / 4 of the Stockham stage whose sub-transforms have Ns points (Ns = 1, 2, 4, ... < n_fft / 2).
__host__ __device__ inline void fft_stage(const Tabs& tb, int j, int Ns, const double2* in, double2* out) {
  const int H = tb.n_fft / 2;
  const int k = j & (Ns - 1);
  const double2 w = tb.tw[k * (tb.n_fft / (2 * Ns))];   // e^{-2 pi i k / (2 Ns)}
  const double2 a = in[j], c = in[j + H / 2];
  const double2 b = make_double2(c.x * w.x - c.y * w.y, c.x * w.y + c.y * w.x);
  const int d = (j - k) * 2 + k;
  out[d] = make_double2(a.x + b.x, a.y + b.y);
  out[d + Ns] = make_double2(a.x - b.x, a.y - b.y);
}
// |X[k]| for bin k <= n_fft / 2 of the real transform, from the packed transform Z: X[k] = E[k] + e^{-2 pi i k / n_fft}
// O[k] with E = (Z[k] + conj Z[H - k]) / 2, O = (Z[k] - conj Z[H - k]) / 2i.  X[k] is rounded to complex64 first, and
// its magnitude is the correctly rounded hypotf of the two floats (as glibc's hypotf, which numpy's abs uses).
__host__ __device__ inline float bin_magnitude(const Tabs& tb, int k, const double2* Z) {
  const int H = tb.n_fft / 2;
  const double2 zk = Z[k == H ? 0 : k], zm = Z[k == 0 ? 0 : H - k];
  const double ex = 0.5 * (zk.x + zm.x), ey = 0.5 * (zk.y - zm.y);
  const double ox = 0.5 * (zk.y + zm.y), oy = -0.5 * (zk.x - zm.x);
  const double2 w = k < H ? tb.tw[k] : make_double2(-1.0, 0.0);
  const float xr = (float)(ex + (w.x * ox - w.y * oy)), xi = (float)(ey + (w.x * oy + w.y * ox));
  return (float)sqrt((double)xr * xr + (double)xi * xi);
}
// Band m: its float64 sum, amp_to_db and normalize, stored as float32.  20 log10(1e-5) is -100 exactly (as numpy
// evaluates it), so a frame of digital silence is exactly 0 at min_level_db = -100.  A NaN sum (a frame that read a
// NaN sample) stays NaN through the floor and the clamp, as np.maximum and np.clip keep it; a band with no filter
// weight sums nothing and keeps its silent value, where numpy's 0 x NaN would make it NaN.
__host__ __device__ inline float band_value(const Tabs& tb, int m, const float* mag) {
  const int lo = tb.bands[3 * m], cnt = tb.bands[3 * m + 1], off = tb.bands[3 * m + 2];
  double acc = 0.0;
  for (int i = 0; i < cnt; ++i) acc += tb.basis[off + i] * (double)mag[lo + i];
  const double S = !(acc <= 1e-5) ? 20.0 * log10(acc) : -100.0;
  const double v = (S - tb.min_level_db) / -tb.min_level_db;
  return (float)(v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v));
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
struct FrameUtt {          // one entry of the frame table: utterance i owns frames frame0 .. frame0 + T - 1 of the grid
  const float* y;
  long long n;
  float* mel;
  long long T;
  long long frame0;
};

__global__ void __launch_bounds__(THREADS) mel_frames_kernel(Tabs tb, const FrameUtt* __restrict__ utts, int n_utts) {
  extern __shared__ double2 sm[];   // [2][n_fft / 2]; the magnitudes reuse the free half
  const long long f = blockIdx.x;
  int lo = 0, hi = n_utts - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (utts[mid].frame0 <= f) lo = mid; else hi = mid - 1;
  }
  const FrameUtt u = utts[lo];
  const long long t = f - u.frame0;
  const int H = tb.n_fft / 2;
  double2 *in = sm, *out = sm + H;
  for (int k = threadIdx.x; k < H; k += THREADS) load_point(tb, u.y, u.n, t * tb.hop, k, in);
  __syncthreads();
  for (int Ns = 1; Ns < H; Ns *= 2) {
    for (int j = threadIdx.x; j < H / 2; j += THREADS) fft_stage(tb, j, Ns, in, out);
    __syncthreads();
    double2* s = in; in = out; out = s;
  }
  float* mag = reinterpret_cast<float*>(out);
  for (int k = threadIdx.x; k <= H; k += THREADS) mag[k] = bin_magnitude(tb, k, in);
  __syncthreads();
  for (int m = threadIdx.x; m < tb.n_mels; m += THREADS) u.mel[(long long)m * u.T + t] = band_value(tb, m, mag);
}

static size_t smem_bytes(int n_fft) { return (size_t)n_fft * sizeof(double2); }

static Tabs device_view(const wrnn_mel_plan& m) {
  const wrnn_mel_cfg& c = m.cfg;
  const double* d = static_cast<const double*>(m.d_tabs);
  const double* basis = d + 2 * c.n_fft;
  return Tabs{c.n_fft, c.hop_length, c.n_mels, (double)c.min_level_db, d, reinterpret_cast<const double2*>(d + c.n_fft),
              basis, reinterpret_cast<const int*>(basis + m.n_basis)};
}

int check_cfg(const wrnn_mel_cfg* c) {
  auto bad = [](const std::string& s) { set_error("wrnn_mel_cfg: " + s); return WRNN_E_INVALID; };
  if (!c) return bad("null cfg");
  if (c->sample_rate <= 0) return bad("sample_rate must be > 0");
  if (c->n_fft < 256 || c->n_fft > 4096 || (c->n_fft & (c->n_fft - 1))) return bad("n_fft must be a power of two in 256..4096");
  if (c->hop_length < 1) return bad("hop_length must be >= 1");
  if (c->win_length < 1 || c->win_length > c->n_fft) return bad("win_length must be in 1..n_fft");
  if (c->n_mels < 1 || c->n_mels > 128) return bad("n_mels must be in 1..128");
  if (!(c->fmin >= 0.f) || !(c->fmin < c->sample_rate / 2.0)) return bad("fmin must be in [0, sample_rate / 2)");
  if (!(c->min_level_db < 0.f) || !std::isfinite(c->min_level_db)) return bad("min_level_db must be finite and < 0");
  return WRNN_OK;
}

int plan(const wrnn_mel_cfg& c, const wrnn_mel_utt* u, int n_utts, std::vector<int64_t>& frame0) {
  if (!u || n_utts < 1) { set_error("wrnn_melspectrogram_many needs a non-null utterance array and n_utts >= 1"); return WRNN_E_INVALID; }
  frame0.assign(n_utts + 1, 0);
  for (int i = 0; i < n_utts; ++i) {
    const std::string at = "utterance " + std::to_string(i) + ": ";
    if (!u[i].y || !u[i].mel) { set_error(at + "y and mel are required"); return WRNN_E_INVALID; }
    if (u[i].n <= c.n_fft / 2) {
      set_error(at + "n must be > n_fft / 2 = " + std::to_string(c.n_fft / 2) + " (one reflection of the centre padding)");
      return WRNN_E_INVALID;
    }
    frame0[i + 1] = frame0[i] + 1 + u[i].n / c.hop_length;
    if (frame0[i + 1] >= (1ll << 31)) { set_error("a batch must have fewer than 2^31 frames"); return WRNN_E_INVALID; }
  }
  return WRNN_OK;
}

static int launch(const wrnn_mel_plan& m, const wrnn_mel_utt* u, int n, const std::vector<int64_t>& frame0, cudaStream_t st) {
  std::vector<FrameUtt> tab(n);
  for (int i = 0; i < n; ++i) tab[i] = FrameUtt{u[i].y, u[i].n, u[i].mel, frame0[i + 1] - frame0[i], frame0[i]};
  WRNN_CUDA_OK(cudaSetDevice(m.device));
  // the table lives for this launch only, so that calls on any streams share the analysis object
  void* d = nullptr;
  WRNN_CUDA_OK(cudaMallocAsync(&d, tab.size() * sizeof(FrameUtt), st));
  WRNN_CUDA_OK(cudaMemcpyAsync(d, tab.data(), tab.size() * sizeof(FrameUtt), cudaMemcpyHostToDevice, st));
  mel_frames_kernel<<<(unsigned)frame0[n], THREADS, smem_bytes(m.cfg.n_fft), st>>>(device_view(m), static_cast<FrameUtt*>(d), n);
  WRNN_CUDA_OK(cudaGetLastError());
  WRNN_CUDA_OK(cudaFreeAsync(d, st));
  return WRNN_OK;
}

}  // namespace mel
}  // namespace wrnn

using namespace wrnn;

extern "C" {

int wrnn_mel_create(wrnn_mel_t** out, const wrnn_mel_cfg* cfg, int device) {
  if (!out) { set_error("wrnn_mel_create: null out"); return WRNN_E_INVALID; }
  *out = nullptr;
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  mel::HostTabs t;
  mel::build_tables(*cfg, t);
  // [window | twiddles | basis | bands]
  const long long n_basis = (long long)t.basis.size();
  std::vector<double> blob(2 * cfg->n_fft + n_basis + (t.bands.size() + 1) / 2, 0.0);
  std::copy(t.window.begin(), t.window.end(), blob.begin());
  std::copy(t.tw.begin(), t.tw.end(), blob.begin() + cfg->n_fft);
  std::copy(t.basis.begin(), t.basis.end(), blob.begin() + 2 * cfg->n_fft);
  std::memcpy(&blob[2 * cfg->n_fft + n_basis], t.bands.data(), t.bands.size() * sizeof(int));
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
    cudaGetLastError();
    set_error("wrnn_mel_create: no such CUDA device");
    return WRNN_E_NO_DEVICE;
  }
  WRNN_CUDA_OK(cudaSetDevice(device));
  WRNN_CUDA_OK(cudaFuncSetAttribute(mel::mel_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)mel::smem_bytes(4096)));
  wrnn_mel_plan* m = new (std::nothrow) wrnn_mel_plan;
  if (!m) { set_error("out of host memory"); return WRNN_E_INVALID; }
  m->cfg = *cfg;
  m->device = device;
  m->n_basis = n_basis;
  cudaError_t e = cudaMalloc(&m->d_tabs, blob.size() * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(m->d_tabs, blob.data(), blob.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error(std::string("wrnn_mel_create: ") + cudaGetErrorString(e));
    wrnn_mel_destroy(m);
    return WRNN_E_CUDA;
  }
  *out = m;
  return WRNN_OK;
}

void wrnn_mel_destroy(wrnn_mel_t* m) {
  if (!m) return;
  if (m->d_tabs) {
    cudaSetDevice(m->device);
    cudaFree(m->d_tabs);
  }
  delete m;
}

int wrnn_melspectrogram_many(const wrnn_mel_t* m, const wrnn_mel_utt* u, int32_t n_utts, void* stream) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<int64_t> frame0;
  const int rc = mel::plan(m->cfg, u, n_utts, frame0);
  if (rc != WRNN_OK) return rc;
  return mel::launch(*m, u, n_utts, frame0, static_cast<cudaStream_t>(stream));
}

int wrnn_melspectrogram_many_host(const wrnn_mel_t* m, const wrnn_mel_utt* u, int32_t n_utts) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<int64_t> frame0;
  int rc = mel::plan(m->cfg, u, n_utts, frame0);
  if (rc != WRNN_OK) return rc;
  const int n = n_utts;
  // one device block [y_0 | .. | y_{n-1} | mel_0 | ..], each region 256-B aligned
  std::vector<size_t> off(2 * n + 1, 0);
  for (int i = 0; i < 2 * n; ++i) {
    const size_t bytes = i < n ? (size_t)u[i].n * sizeof(float) : (size_t)m->cfg.n_mels * (frame0[i - n + 1] - frame0[i - n]) * sizeof(float);
    off[i + 1] = off[i] + ((bytes + 255) & ~size_t(255));
  }
  WRNN_CUDA_OK(cudaSetDevice(m->device));
  char* d = nullptr;
  WRNN_CUDA_OK(cudaMalloc(&d, off[2 * n]));
  std::vector<wrnn_mel_utt> du(n);
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < n && e == cudaSuccess; ++i) {
    du[i] = wrnn_mel_utt{reinterpret_cast<float*>(d + off[i]), u[i].n, reinterpret_cast<float*>(d + off[n + i])};
    e = cudaMemcpyAsync(d + off[i], u[i].y, (size_t)u[i].n * sizeof(float), cudaMemcpyDefault, 0);
  }
  if (e == cudaSuccess) {
    rc = mel::launch(*m, du.data(), n, frame0, 0);
    for (int i = 0; i < n && rc == WRNN_OK && e == cudaSuccess; ++i)
      e = cudaMemcpyAsync(u[i].mel, du[i].mel, (size_t)m->cfg.n_mels * (frame0[i + 1] - frame0[i]) * sizeof(float),
                          cudaMemcpyDefault, 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(0);
  }
  cudaFree(d);
  if (e != cudaSuccess) { set_error(std::string("wrnn_melspectrogram_many_host: ") + cudaGetErrorString(e)); return WRNN_E_CUDA; }
  return rc;
}

// ---- test hooks (not declared in the header) ------------------------------------------------------------------------
// The host tables: window [n_fft], the dense filterbank [n_mels][n_fft / 2 + 1] and the bands [n_mels][2] (first
// nonzero bin, count); NULL outputs are skipped.
int wrnn_debug_mel_tables(const wrnn_mel_cfg* cfg, double* window, double* basis, int32_t* bands) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  mel::HostTabs t;
  mel::build_tables(*cfg, t);
  if (window) std::copy(t.window.begin(), t.window.end(), window);
  if (basis) std::copy(t.dense.begin(), t.dense.end(), basis);
  for (int i = 0; bands && i < cfg->n_mels; ++i) { bands[2 * i] = t.bands[3 * i]; bands[2 * i + 1] = t.bands[3 * i + 1]; }
  return WRNN_OK;
}

// The frame table wrnn_melspectrogram_many lays out (frame0 [n_utts + 1]), or its refusal.
int wrnn_debug_mel_plan(const wrnn_mel_cfg* cfg, const wrnn_mel_utt* u, int32_t n_utts, int64_t* frame0) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  std::vector<int64_t> f0;
  if ((rc = mel::plan(*cfg, u, n_utts, f0)) != WRNN_OK) return rc;
  if (frame0) std::copy(f0.begin(), f0.end(), frame0);
  return WRNN_OK;
}

// The kernel's per-frame functions run on the host, frame after frame: y [n] -> mel [n_mels, 1 + n / hop_length].
int wrnn_debug_mel_frames(const wrnn_mel_cfg* cfg, const float* y, int64_t n, float* mel) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  const wrnn_mel_utt u{y, n, mel};
  std::vector<int64_t> f0;
  if ((rc = mel::plan(*cfg, &u, 1, f0)) != WRNN_OK) return rc;
  mel::HostTabs t;
  mel::build_tables(*cfg, t);
  const mel::Tabs tb = mel::host_view(*cfg, t);
  const int H = cfg->n_fft / 2;
  std::vector<double2> a(H), b(H);
  std::vector<float> mag(H + 1);
  const long long T = f0[1];
  for (long long f = 0; f < T; ++f) {
    double2 *in = a.data(), *out = b.data();
    for (int k = 0; k < H; ++k) mel::load_point(tb, y, n, f * cfg->hop_length, k, in);
    for (int Ns = 1; Ns < H; Ns *= 2) {
      for (int j = 0; j < H / 2; ++j) mel::fft_stage(tb, j, Ns, in, out);
      std::swap(in, out);
    }
    for (int k = 0; k <= H; ++k) mag[k] = mel::bin_magnitude(tb, k, in);
    for (int m = 0; m < cfg->n_mels; ++m) mel[(long long)m * T + f] = mel::band_value(tb, m, mag.data());
  }
  return WRNN_OK;
}

}  // extern "C"
