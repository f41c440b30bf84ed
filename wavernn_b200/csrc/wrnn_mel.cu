// wrnn_mel.cu -- the reference's melspectrogram(y) (utils/dsp.py:72-81) and its inverse, reconstruct_waveform(mel)
// (utils/dsp.py:105-116, Griffin-Lim), on the device: wrnn_mel_create, wrnn_melspectrogram_many,
// wrnn_griffinlim_many and their host hooks.
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

#include "wrnn_device.cuh"
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
  std::vector<double> basis32;             // basis as librosa 0.7 builds it in float32 (Griffin-Lim's NNLS), same ranges
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
  t.basis32.clear();
  t.bands.assign(3 * M, 0);
  std::vector<double> tri(nb);
  for (int i = 0; i < M; ++i) {
    const double fd0 = mel_f[i + 1] - mel_f[i], fd1 = mel_f[i + 2] - mel_f[i + 1];
    const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
    int lo = -1, hi = -1;
    for (int k = 0; k < nb; ++k) {
      const double lower = -(mel_f[i] - fft[k]) / fd0, upper = (mel_f[i + 2] - fft[k]) / fd1;
      tri[k] = std::fmax(0.0, std::fmin(lower, upper));
      const double w = tri[k] * enorm;
      t.dense[(size_t)i * nb + k] = w;
      if (w > 0) { if (lo < 0) lo = k; hi = k; }
    }
    t.bands[3 * i] = lo < 0 ? 0 : lo;
    t.bands[3 * i + 1] = lo < 0 ? 0 : hi - lo + 1;
    t.bands[3 * i + 2] = (int)t.basis.size();
    for (int k = lo; lo >= 0 && k <= hi; ++k) {
      t.basis.push_back(t.dense[(size_t)i * nb + k]);
      // filters.mel(dtype=float32): the triangle stored as float32, scaled by the float64 norm, stored again
      t.basis32.push_back((double)(float)((double)(float)tri[k] * enorm));
    }
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
// Bin k <= n_fft / 2 of the real transform, from the packed transform Z: X[k] = E[k] + e^{-2 pi i k / n_fft} O[k] with
// E = (Z[k] + conj Z[H - k]) / 2, O = (Z[k] - conj Z[H - k]) / 2i, rounded to complex64 as librosa's stft stores it.
__host__ __device__ inline float2 bin_value(const Tabs& tb, int k, const double2* Z) {
  const int H = tb.n_fft / 2;
  const double2 zk = Z[k == H ? 0 : k], zm = Z[k == 0 ? 0 : H - k];
  const double ex = 0.5 * (zk.x + zm.x), ey = 0.5 * (zk.y - zm.y);
  const double ox = 0.5 * (zk.y + zm.y), oy = -0.5 * (zk.x - zm.x);
  const double2 w = k < H ? tb.tw[k] : make_double2(-1.0, 0.0);
  return make_float2((float)(ex + (w.x * ox - w.y * oy)), (float)(ey + (w.x * oy + w.y * ox)));
}
// |x| of a complex64 value: the correctly rounded hypotf of the two floats (as glibc's hypotf, which numpy's abs uses).
__host__ __device__ inline float cabs64(float2 x) { return (float)sqrt((double)x.x * x.x + (double)x.y * x.y); }
__host__ __device__ inline float bin_magnitude(const Tabs& tb, int k, const double2* Z) { return cabs64(bin_value(tb, k, Z)); }
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
  const FrameUtt u = utts[find_utt(utts, n_utts, f, &FrameUtt::frame0)];
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
  return with_device_table(tab.data(), tab.size(), st, [&](const FrameUtt* d) {
    mel_frames_kernel<<<(unsigned)frame0[n], THREADS, smem_bytes(m.cfg.n_fft), st>>>(device_view(m), d, n);
    WRNN_CUDA_OK(cudaGetLastError());
    return WRNN_OK;
  });
}

// ---- Griffin-Lim: the inverse of the analysis (DESIGN.md §3.9) -------------------------------------------------------
// Per utterance: S = NNLS(A, db_to_amp(denormalize(mel))) frame by frame, then librosa 0.7's griffinlim on S.  One CTA
// per frame for the solve and for each iteration's rfft -> phase update -> irfft; one thread per sample for each
// overlap-add, which writes the signal straight into wav (the last one is the result).
constexpr int NNLS_ITERS = 100;        // accelerated projected-gradient steps per frame (tests/gl_oracle.py FISTA_ITERS)
constexpr double PIVOT_DROP = 1e-10;   // a band whose LDL^T pivot falls below this share of its diagonal leaves the start
constexpr float GL_MOMENTUM_C = (float)(0.99 / 1.99);   // momentum / (1 + momentum), as numpy casts it to complex64
constexpr size_t GL_CHUNK_BYTES = size_t(1) << 30;       // scratch per launch batch

struct GLTabs {             // the solve's constants, host or device
  const double* basis32;    // the float32 filterbank, packed as Tabs::basis
  const double* inv_d;      // [n_mels] inverse LDL^T pivots of A A^T (0: band left out of the start)
  const double* sub;        // [n_mels] LDL^T subdiagonal multipliers (sub[m] couples bands m - 1 and m)
  const int* bin_band;      // [n_fft / 2 + 1] the first band holding bin k, or -1; the second can only be the next one
  double step;              // 1 / lambda_max(A A^T)
};
struct HostGL {
  std::vector<double> inv_d, sub;
  std::vector<int> bin_band;
  double step = 0.0;
};

// The LDL^T factor of the tridiagonal A A^T (a Slaney bin lies in at most two adjacent bands) and its largest
// eigenvalue by Sturm-sequence bisection, from the float32 filterbank.
static void build_gl(const wrnn_mel_cfg& c, const HostTabs& t, HostGL& g) {
  const int M = c.n_mels, nb = c.n_fft / 2 + 1;
  std::vector<double> dense((size_t)M * nb, 0.0), a(M, 0.0), e(M, 0.0);
  g.bin_band.assign(nb, -1);
  for (int m = M - 1; m >= 0; --m)
    for (int i = 0; i < t.bands[3 * m + 1]; ++i) {
      const int k = t.bands[3 * m] + i;
      dense[(size_t)m * nb + k] = t.basis32[t.bands[3 * m + 2] + i];
      g.bin_band[k] = m;
    }
  for (int m = 0; m < M; ++m)
    for (int k = 0; k < nb; ++k) {
      const double v = dense[(size_t)m * nb + k];
      a[m] += v * v;
      if (m > 0) e[m] += v * dense[(size_t)(m - 1) * nb + k];
    }
  g.inv_d.assign(M, 0.0);
  g.sub.assign(M, 0.0);
  double prev = 0.0;
  for (int m = 0; m < M; ++m) {
    double l = m > 0 && prev > 0 ? e[m] / prev : 0.0;
    double d = m > 0 ? a[m] - l * e[m] : a[m];
    if (!(d > PIVOT_DROP * a[m])) { l = 0.0; d = 0.0; }
    g.sub[m] = l;
    g.inv_d[m] = d > 0 ? 1.0 / d : 0.0;
    prev = d;
  }
  double lo = 0.0, hi = 0.0;   // Gershgorin bound, then bisection on the count of eigenvalues below x
  for (int m = 0; m < M; ++m) hi = std::max(hi, a[m] + std::fabs(e[m]) + (m + 1 < M ? std::fabs(e[m + 1]) : 0.0));
  auto below = [&](double x) {
    int n = 0;
    double q = 1.0;
    for (int m = 0; m < M; ++m) {
      q = a[m] - x - (m > 0 ? e[m] * e[m] / q : 0.0);
      if (q == 0.0) q = -1e-300;
      n += q < 0;
    }
    return n;
  };
  for (int it = 0; it < 200 && hi - lo > 1e-15 * hi; ++it) {
    const double mid = 0.5 * (lo + hi);
    (below(mid) == M ? hi : lo) = mid;
  }
  g.step = hi > 0 ? 1.0 / hi : 0.0;
}

// ---- the solve, step by step ----
// b_m = db_to_amp(denormalize(mel)) in float32: (clip(v, 0, 1) * -L + L) * 0.05, then 10^x rounded once.  NaN stays NaN.
__host__ __device__ inline double nnls_rhs(const Tabs& tb, float v) {
  const float L = (float)tb.min_level_db;
  const float c = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
  const float x = fmul_rn(fmul_rn(c, -L) + L, 0.05f);
  return (double)(float)pow(10.0, (double)x);
}
// The minimum-norm least-squares start's multipliers: z = (A A^T)^-1 b over the bands kept (one thread).
__host__ __device__ inline void nnls_start(const GLTabs& g, int M, const double* b, double* z) {
  double u = 0.0;
  for (int m = 0; m < M; ++m) {
    u = b[m] - g.sub[m] * u;
    z[m] = u;
  }
  for (int m = 0; m < M; ++m) z[m] = g.inv_d[m] == 0.0 ? 0.0 : z[m] * g.inv_d[m];
  for (int m = M - 2; m >= 0; --m) z[m] -= g.sub[m + 1] * z[m + 1];
}
// (A^T v)[k]: at most two terms
__host__ __device__ inline double nnls_at(const Tabs& tb, const GLTabs& g, int k, const double* v) {
  const int m = g.bin_band[k];
  if (m < 0) return 0.0;
  double s = g.basis32[tb.bands[3 * m + 2] + k - tb.bands[3 * m]] * v[m];
  if (m + 1 < tb.n_mels) {
    const int lo = tb.bands[3 * (m + 1)], cnt = tb.bands[3 * (m + 1) + 1];
    if (k >= lo && k < lo + cnt) s += g.basis32[tb.bands[3 * (m + 1) + 2] + k - lo] * v[m + 1];
  }
  return s;
}
__host__ __device__ inline double clip0(double v) { return v < 0.0 ? 0.0 : v; }   // np.maximum(v, 0): NaN stays
// r_m = (A y)_m - b_m
__host__ __device__ inline double nnls_residual(const Tabs& tb, const GLTabs& g, int m, const double* y, const double* b) {
  const int lo = tb.bands[3 * m], cnt = tb.bands[3 * m + 1], off = tb.bands[3 * m + 2];
  double acc = 0.0;
  for (int i = 0; i < cnt; ++i) acc += g.basis32[off + i] * y[lo + i];
  return acc - b[m];
}
// one projected-gradient step of bin k with momentum beta
__host__ __device__ inline void nnls_step(const Tabs& tb, const GLTabs& g, int k, const double* r, double beta, double* x,
                                          double* y) {
  const double xn = clip0(y[k] - nnls_at(tb, g, k, r) * g.step);
  y[k] = xn + beta * (xn - x[k]);
  x[k] = xn;
}
// FISTA's momentum after step i: t_{i+1} = (1 + sqrt(1 + 4 t_i^2)) / 2, beta = (t_i - 1) / t_{i+1}
__host__ __device__ inline double fista_next(double& t) {
  const double tn = (1.0 + sqrt(1.0 + 4.0 * t * t)) / 2.0, beta = (t - 1.0) / tn;
  t = tn;
  return beta;
}

// ---- one Griffin-Lim frame, step by step ----
// The initial phase of bin k of frame t: exp(2 pi i u) rounded to complex64, u = u01 of word k % 4 of the Philox block
// at counter (t, k / 4, 0, 0) under key seed.
__host__ __device__ inline float2 gl_phase0(unsigned long long seed, long long t, int k) {
  const Philox4 r = philox4x32_10((unsigned)t, (unsigned)(k >> 2), 0u, 0u, (unsigned)seed, (unsigned)(seed >> 32));
  const unsigned w = (k & 3) == 0 ? r.x : (k & 3) == 1 ? r.y : (k & 3) == 2 ? r.z : r.w;
  const double th = 6.283185307179586 * (double)u01(w);
  return make_float2((float)cos(th), (float)sin(th));
}
// S * angles in complex64: each part scaled by the float32 magnitude
__host__ __device__ inline float2 gl_scale(float s, float2 a) { return make_float2(fmul_rn(s, a.x), fmul_rn(s, a.y)); }
// rebuilt = bin k of the frame's transform Z; angles = rebuilt - c tprev (tprev = 0 on the first iteration), then
// angles / (|angles| + 1e-16) as numpy divides complex64 by a real (times the float32 reciprocal); tprev = rebuilt.
// Returns S_k * angles.
__host__ __device__ inline float2 gl_update(const Tabs& tb, int k, const double2* Z, float s, float2* tprev, bool first) {
  const float2 x = bin_value(tb, k, Z);
  float2 a = x;
  if (!first) {
    const float2 p = tprev[k];
    a = make_float2(x.x - fmul_rn(GL_MOMENTUM_C, p.x), x.y - fmul_rn(GL_MOMENTUM_C, p.y));
  }
  tprev[k] = x;
  const float r = 1.0f / (cabs64(a) + 1e-16f);
  return gl_scale(s, make_float2(fmul_rn(a.x, r), fmul_rn(a.y, r)));
}
// Packs the bins P[0 .. H] of a real signal into point k < H of conj(Z), Z the H-point transform of its (even, odd)
// sample pairs, so that the forward stages compute the inverse: Z[k] = E[k] + i O[k], E = (X[k] + conj X[H - k]) / 2,
// O = (X[k] - conj X[H - k]) e^{2 pi i k / n_fft} / 2.  The imaginary parts of the DC and Nyquist bins are dropped,
// as irfft drops them.
__host__ __device__ inline void gl_pack(const Tabs& tb, int k, const float2* P, double2* out) {
  const int H = tb.n_fft / 2;
  const float2 pk = P[k], pm = P[H - k];
  const double xr = pk.x, xi = k == 0 ? 0.0 : pk.y, mr = pm.x, mi = k == 0 ? 0.0 : pm.y;
  const double er = 0.5 * (xr + mr), ei = 0.5 * (xi - mi), dr = 0.5 * (xr - mr), di = 0.5 * (xi + mi);
  const double2 w = tb.tw[k];   // e^{-2 pi i k / n_fft}; O = D conj(w)
  const double orr = dr * w.x + di * w.y, oi = di * w.x - dr * w.y;
  out[k] = make_double2(er - oi, -(ei + orr));
}
// Samples 2n, 2n + 1 of irfft, from the forward transform R of conj(Z): conj(R[n]) / H, times the window.
__host__ __device__ inline void gl_unpack(const Tabs& tb, int n, const double2* R, double* y) {
  const double s = 1.0 / (tb.n_fft / 2);
  y[2 * n] = tb.window[2 * n] * (R[n].x * s);
  y[2 * n + 1] = tb.window[2 * n + 1] * (-R[n].y * s);
}
// Sample p of the padded signal: the float64 frames added into float32 in frame order, divided by the float32
// window sum-square built the same way where it exceeds float32 tiny.  frames: [T][n_fft] float64.
__host__ __device__ inline float gl_ola(const Tabs& tb, const double* frames, long long T, long long p) {
  const int N = tb.n_fft, hop = tb.hop;
  const long long i0 = p - N + 1 <= 0 ? 0 : (p - N + hop) / hop, i1 = p / hop < T - 1 ? p / hop : T - 1;
  float y = 0.f, w = 0.f;
  for (long long i = i0; i <= i1; ++i) {
    const int q = (int)(p - i * hop);
    y = (float)((double)y + frames[i * N + q]);
    w = (float)((double)w + dmul_rn(tb.window[q], tb.window[q]));
  }
  return w > 1.17549435e-38f ? y / w : y;
}

struct GLUtt {              // one utterance of a launch batch
  const float* mel;
  float* wav;
  long long T, frame0, sample0;   // frames, first frame and first sample in the whole call
  unsigned long long seed;
};
struct GLScratch {          // per frame of a launch batch, indexed by frame - the batch's first frame
  float* S;                 // [n_fft / 2 + 1]
  float2* tprev;            // [n_fft / 2 + 1]
  double* frames;           // [n_fft], the windowed inverse transform
};

__global__ void __launch_bounds__(THREADS) gl_nnls_kernel(Tabs tb, GLTabs g, const GLUtt* __restrict__ utts, int n,
                                                          float* __restrict__ S) {
  extern __shared__ double sd[];   // b [M] | z [M] | r [M] | x [nb] | y [nb]
  const int M = tb.n_mels, nb = tb.n_fft / 2 + 1;
  double *b = sd, *z = b + M, *r = z + M, *x = r + M, *y = x + nb;
  const long long f = utts[0].frame0 + blockIdx.x;
  const GLUtt u = utts[find_utt(utts, n, f, &GLUtt::frame0)];
  const long long t = f - u.frame0;
  for (int m = threadIdx.x; m < M; m += THREADS) b[m] = nnls_rhs(tb, u.mel[(long long)m * u.T + t]);
  __syncthreads();
  if (threadIdx.x == 0) nnls_start(g, M, b, z);
  __syncthreads();
  for (int k = threadIdx.x; k < nb; k += THREADS) x[k] = y[k] = clip0(nnls_at(tb, g, k, z));
  __syncthreads();
  double tk = 1.0;
  for (int it = 0; it < NNLS_ITERS; ++it) {
    for (int m = threadIdx.x; m < M; m += THREADS) r[m] = nnls_residual(tb, g, m, y, b);
    __syncthreads();
    const double beta = fista_next(tk);
    for (int k = threadIdx.x; k < nb; k += THREADS) nnls_step(tb, g, k, r, beta, x, y);
    __syncthreads();
  }
  float* out = S + (size_t)blockIdx.x * nb;
  for (int k = threadIdx.x; k < nb; k += THREADS) out[k] = (float)x[k];
}

// Iteration `it` of frame f: it = 0 takes the initial phases; it >= 1 analyses the signal the last overlap-add wrote
// and updates the phases.  Either way it ends with the windowed inverse transform of S * angles.
__global__ void __launch_bounds__(THREADS) gl_frames_kernel(Tabs tb, const GLUtt* __restrict__ utts, int n, GLScratch s,
                                                            int it) {
  extern __shared__ double2 sm[];   // [2][n_fft / 2]; the products S * angles (complex64) reuse the free half
  const int H = tb.n_fft / 2, nb = H + 1;
  const long long f = utts[0].frame0 + blockIdx.x;
  const GLUtt u = utts[find_utt(utts, n, f, &GLUtt::frame0)];
  const long long t = f - u.frame0;
  const float* S = s.S + (size_t)blockIdx.x * nb;
  double2 *in = sm, *out = sm + H;
  float2* P = reinterpret_cast<float2*>(out);
  if (it == 0) {
    for (int k = threadIdx.x; k < nb; k += THREADS) P[k] = gl_scale(S[k], gl_phase0(u.seed, t, k));
  } else {
    const long long len = (long long)tb.hop * (u.T - 1);
    for (int k = threadIdx.x; k < H; k += THREADS) load_point(tb, u.wav, len, t * tb.hop, k, in);
    __syncthreads();
    for (int Ns = 1; Ns < H; Ns *= 2) {
      for (int j = threadIdx.x; j < H / 2; j += THREADS) fft_stage(tb, j, Ns, in, out);
      __syncthreads();
      double2* q = in; in = out; out = q;
    }
    P = reinterpret_cast<float2*>(out);
    float2* tprev = s.tprev + (size_t)blockIdx.x * nb;
    for (int k = threadIdx.x; k < nb; k += THREADS) P[k] = gl_update(tb, k, in, S[k], tprev, it == 1);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < H; k += THREADS) gl_pack(tb, k, P, in);
  __syncthreads();
  for (int Ns = 1; Ns < H; Ns *= 2) {
    for (int j = threadIdx.x; j < H / 2; j += THREADS) fft_stage(tb, j, Ns, in, out);
    __syncthreads();
    double2* q = in; in = out; out = q;
  }
  double* y = s.frames + (size_t)blockIdx.x * tb.n_fft;
  for (int k = threadIdx.x; k < H; k += THREADS) gl_unpack(tb, k, in, y);
}

// One thread per sample of the batch: wav[j] = sample j + n_fft / 2 of the padded signal (the centre trim).
__global__ void __launch_bounds__(THREADS) gl_ola_kernel(Tabs tb, const GLUtt* __restrict__ utts, int n, const double* frames,
                                                         long long n_samples) {
  const long long j = utts[0].sample0 + (long long)blockIdx.x * THREADS + threadIdx.x;
  if (j >= utts[0].sample0 + n_samples) return;
  const GLUtt u = utts[find_utt(utts, n, j, &GLUtt::sample0)];
  const double* fr = frames + (size_t)(u.frame0 - utts[0].frame0) * tb.n_fft;
  u.wav[j - u.sample0] = gl_ola(tb, fr, u.T, j - u.sample0 + tb.n_fft / 2);
}

static size_t nnls_smem(const wrnn_mel_cfg& c) { return (size_t)(3 * c.n_mels + 2 * (c.n_fft / 2 + 1)) * sizeof(double); }
static size_t gl_frame_bytes(int n_fft) {
  const size_t nb = n_fft / 2 + 1;
  return align256(nb * sizeof(float)) + align256(nb * sizeof(float2)) + n_fft * sizeof(double);
}

static GLTabs gl_device_view(const wrnn_mel_plan& m) {
  const double* d = static_cast<const double*>(m.d_tabs) + m.gl_off;
  const int M = m.cfg.n_mels;
  return GLTabs{d, d + m.n_basis, d + m.n_basis + M, reinterpret_cast<const int*>(d + m.n_basis + 2 * M), m.gl_step};
}

int gl_plan(const wrnn_mel_cfg& c, const wrnn_gl_utt* u, int n_utts, int n_iter, std::vector<int64_t>& frame0) {
  if (!u || n_utts < 1) { set_error("wrnn_griffinlim_many needs a non-null utterance array and n_utts >= 1"); return WRNN_E_INVALID; }
  if (n_iter < 0) { set_error("wrnn_griffinlim_many: n_iter must be >= 0"); return WRNN_E_INVALID; }
  frame0.assign(n_utts + 1, 0);
  for (int i = 0; i < n_utts; ++i) {
    const std::string at = "utterance " + std::to_string(i) + ": ";
    if (!u[i].mel || !u[i].wav) { set_error(at + "mel and wav are required"); return WRNN_E_INVALID; }
    if (u[i].T < 2 || u[i].T - 1 <= (c.n_fft / 2) / c.hop_length) {
      set_error(at + "hop_length * (T - 1) must be > n_fft / 2 = " + std::to_string(c.n_fft / 2) +
                " (one reflection of the centre padding)");
      return WRNN_E_INVALID;
    }
    if (u[i].T >= (1ll << 31) - frame0[i]) { set_error("a batch must have fewer than 2^31 frames"); return WRNN_E_INVALID; }
    frame0[i + 1] = frame0[i] + u[i].T;
  }
  return WRNN_OK;
}

static int gl_launch(const wrnn_mel_plan& m, const wrnn_gl_utt* u, int n, int n_iter, const std::vector<int64_t>& frame0,
                     cudaStream_t st) {
  const wrnn_mel_cfg& c = m.cfg;
  const int nb = c.n_fft / 2 + 1;
  std::vector<GLUtt> tab(n);
  long long s0 = 0;
  for (int i = 0; i < n; ++i) {
    tab[i] = GLUtt{u[i].mel, u[i].wav, u[i].T, frame0[i], s0, u[i].phase_seed};
    s0 += (long long)c.hop_length * (u[i].T - 1);
  }
  // launch batches: runs of whole utterances within GL_CHUNK_BYTES of scratch (an utterance larger than that alone)
  const size_t per_frame = gl_frame_bytes(c.n_fft);
  const long long cap = std::max<long long>(1, (long long)(GL_CHUNK_BYTES / per_frame));
  std::vector<int> first{0};
  long long biggest = 0;
  for (int i = 0; i < n; ++i) {
    if (i > first.back() && frame0[i + 1] - frame0[first.back()] > cap) first.push_back(i);
    biggest = std::max<long long>(biggest, frame0[i + 1] - frame0[first.back()]);
  }
  first.push_back(n);
  const size_t tab_bytes = align256(n * sizeof(GLUtt));
  const size_t S_bytes = align256(nb * sizeof(float)), P_bytes = align256(nb * sizeof(float2));
  WRNN_CUDA_OK(cudaSetDevice(m.device));
  char* d = nullptr;
  if (cudaMallocAsync(reinterpret_cast<void**>(&d), tab_bytes + (size_t)biggest * per_frame, st) != cudaSuccess) {
    cudaGetLastError();
    set_error("wrnn_griffinlim_many: scratch allocation of " + std::to_string(tab_bytes + (size_t)biggest * per_frame) +
              " bytes failed");
    return WRNN_E_CUDA;
  }
  WRNN_CUDA_OK(cudaMemcpyAsync(d, tab.data(), n * sizeof(GLUtt), cudaMemcpyHostToDevice, st));
  const GLUtt* dtab = reinterpret_cast<const GLUtt*>(d);
  char* base = d + tab_bytes;
  const GLScratch s{reinterpret_cast<float*>(base), reinterpret_cast<float2*>(base + biggest * S_bytes),
                    reinterpret_cast<double*>(base + biggest * (S_bytes + P_bytes))};
  const Tabs tb = device_view(m);
  const GLTabs g = gl_device_view(m);
  for (size_t b = 0; b + 1 < first.size(); ++b) {
    const int i0 = first[b], cnt = first[b + 1] - first[b];
    const unsigned frames = (unsigned)(frame0[first[b + 1]] - frame0[i0]);
    const long long samples = (b + 2 < first.size() ? tab[first[b + 1]].sample0 : s0) - tab[i0].sample0;
    const unsigned ola_blocks = (unsigned)((samples + THREADS - 1) / THREADS);
    gl_nnls_kernel<<<frames, THREADS, nnls_smem(c), st>>>(tb, g, dtab + i0, cnt, s.S);
    for (int it = 0; it <= n_iter; ++it) {
      gl_frames_kernel<<<frames, THREADS, smem_bytes(c.n_fft), st>>>(tb, dtab + i0, cnt, s, it);
      gl_ola_kernel<<<ola_blocks, THREADS, 0, st>>>(tb, dtab + i0, cnt, s.frames, samples);
    }
  }
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
  mel::HostGL g;
  mel::build_gl(*cfg, t, g);
  // [window | twiddles | basis | bands], then Griffin-Lim's [basis32 | inv_d | sub | bin_band]
  const long long n_basis = (long long)t.basis.size(), M = cfg->n_mels;
  const long long gl_off = 2 * cfg->n_fft + n_basis + (long long)(t.bands.size() + 1) / 2;
  std::vector<double> blob(gl_off + n_basis + 2 * M + (g.bin_band.size() + 1) / 2, 0.0);
  std::copy(t.window.begin(), t.window.end(), blob.begin());
  std::copy(t.tw.begin(), t.tw.end(), blob.begin() + cfg->n_fft);
  std::copy(t.basis.begin(), t.basis.end(), blob.begin() + 2 * cfg->n_fft);
  std::memcpy(&blob[2 * cfg->n_fft + n_basis], t.bands.data(), t.bands.size() * sizeof(int));
  std::copy(t.basis32.begin(), t.basis32.end(), blob.begin() + gl_off);
  std::copy(g.inv_d.begin(), g.inv_d.end(), blob.begin() + gl_off + n_basis);
  std::copy(g.sub.begin(), g.sub.end(), blob.begin() + gl_off + n_basis + M);
  std::memcpy(&blob[gl_off + n_basis + 2 * M], g.bin_band.data(), g.bin_band.size() * sizeof(int));
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
    cudaGetLastError();
    set_error("wrnn_mel_create: no such CUDA device");
    return WRNN_E_NO_DEVICE;
  }
  WRNN_CUDA_OK(cudaSetDevice(device));
  WRNN_CUDA_OK(cudaFuncSetAttribute(mel::mel_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)mel::smem_bytes(4096)));
  WRNN_CUDA_OK(cudaFuncSetAttribute(mel::gl_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)mel::smem_bytes(4096)));
  wrnn_mel_plan* m = new (std::nothrow) wrnn_mel_plan;
  if (!m) { set_error("out of host memory"); return WRNN_E_INVALID; }
  m->cfg = *cfg;
  m->device = device;
  m->n_basis = n_basis;
  m->gl_off = gl_off;
  m->gl_step = g.step;
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
  if (m->d_tabs || m->d_rs_win) {
    cudaSetDevice(m->device);
    cudaFree(m->d_tabs);
    cudaFree(m->d_rs_win);
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
  std::vector<Staged> in(2 * n);                       // [recordings | mels]
  for (int i = 0; i < n; ++i) {
    in[i] = {u[i].y, (size_t)u[i].n * sizeof(float)};
    in[n + i] = {nullptr, (size_t)m->cfg.n_mels * (frame0[i + 1] - frame0[i]) * sizeof(float)};
  }
  return with_staging(m->device, in, [&](const std::vector<void*>& d, std::vector<Unstaged>& out) {
    std::vector<wrnn_mel_utt> du(u, u + n);
    for (int i = 0; i < n; ++i) {
      du[i].y = static_cast<float*>(d[i]);
      du[i].mel = static_cast<float*>(d[n + i]);
      out[n + i] = {u[i].mel, d[n + i], in[n + i].bytes};
    }
    return mel::launch(*m, du.data(), n, frame0, 0);
  });
}

int wrnn_griffinlim_many(const wrnn_mel_t* m, const wrnn_gl_utt* u, int32_t n_utts, int32_t n_iter, void* stream) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<int64_t> frame0;
  const int rc = mel::gl_plan(m->cfg, u, n_utts, n_iter, frame0);
  if (rc != WRNN_OK) return rc;
  return mel::gl_launch(*m, u, n_utts, n_iter, frame0, static_cast<cudaStream_t>(stream));
}

int wrnn_griffinlim_many_host(const wrnn_mel_t* m, const wrnn_gl_utt* u, int32_t n_utts, int32_t n_iter) {
  if (!m) { set_error("null analysis object"); return WRNN_E_INVALID; }
  std::vector<int64_t> frame0;
  int rc = mel::gl_plan(m->cfg, u, n_utts, n_iter, frame0);
  if (rc != WRNN_OK) return rc;
  const int n = n_utts;
  const long long M = m->cfg.n_mels, hop = m->cfg.hop_length;
  std::vector<Staged> in(2 * n);                       // [mels | waveforms]
  for (int i = 0; i < n; ++i) {
    in[i] = {u[i].mel, (size_t)(M * u[i].T) * sizeof(float)};
    in[n + i] = {nullptr, (size_t)(hop * (u[i].T - 1)) * sizeof(float)};
  }
  return with_staging(m->device, in, [&](const std::vector<void*>& d, std::vector<Unstaged>& out) {
    std::vector<wrnn_gl_utt> du(u, u + n);
    for (int i = 0; i < n; ++i) {
      du[i].mel = static_cast<float*>(d[i]);
      du[i].wav = static_cast<float*>(d[n + i]);
      out[n + i] = {u[i].wav, d[n + i], in[n + i].bytes};
    }
    return mel::gl_launch(*m, du.data(), n, n_iter, frame0, 0);
  });
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

// The frame table wrnn_griffinlim_many lays out (frame0 [n_utts + 1]), or its refusal.
int wrnn_debug_griffinlim_plan(const wrnn_mel_cfg* cfg, const wrnn_gl_utt* u, int32_t n_utts, int32_t n_iter,
                               int64_t* frame0) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  std::vector<int64_t> f0;
  if ((rc = mel::gl_plan(*cfg, u, n_utts, n_iter, f0)) != WRNN_OK) return rc;
  if (frame0) std::copy(f0.begin(), f0.end(), frame0);
  return WRNN_OK;
}

// The Griffin-Lim kernels' per-frame and per-sample functions run on the host, in launch order: mel [n_mels, T] ->
// wav [hop_length * (T - 1)].  S (optional, [T][n_fft / 2 + 1]) receives the solve's magnitudes.
int wrnn_debug_griffinlim(const wrnn_mel_cfg* cfg, const float* mel, int64_t T, uint64_t seed, int32_t n_iter, float* wav,
                          float* S_out) {
  int rc = mel::check_cfg(cfg);
  if (rc != WRNN_OK) return rc;
  const wrnn_gl_utt u{mel, T, seed, wav};
  std::vector<int64_t> f0;
  if ((rc = mel::gl_plan(*cfg, &u, 1, n_iter, f0)) != WRNN_OK) return rc;
  mel::HostTabs t;
  mel::build_tables(*cfg, t);
  mel::HostGL hg;
  mel::build_gl(*cfg, t, hg);
  const mel::Tabs tb = mel::host_view(*cfg, t);
  const mel::GLTabs g{t.basis32.data(), hg.inv_d.data(), hg.sub.data(), hg.bin_band.data(), hg.step};
  const int M = cfg->n_mels, N = cfg->n_fft, H = N / 2, nb = H + 1, hop = cfg->hop_length;
  std::vector<float> S((size_t)T * nb);
  std::vector<float2> tprev((size_t)T * nb), P(nb);
  std::vector<double> frames((size_t)T * N), b(M), z(M), r(M), x(nb), y(nb);
  for (long long f = 0; f < T; ++f) {
    for (int m = 0; m < M; ++m) b[m] = mel::nnls_rhs(tb, mel[(long long)m * T + f]);
    mel::nnls_start(g, M, b.data(), z.data());
    for (int k = 0; k < nb; ++k) x[k] = y[k] = mel::clip0(mel::nnls_at(tb, g, k, z.data()));
    double tk = 1.0;
    for (int it = 0; it < mel::NNLS_ITERS; ++it) {
      for (int m = 0; m < M; ++m) r[m] = mel::nnls_residual(tb, g, m, y.data(), b.data());
      const double beta = mel::fista_next(tk);
      for (int k = 0; k < nb; ++k) mel::nnls_step(tb, g, k, r.data(), beta, x.data(), y.data());
    }
    for (int k = 0; k < nb; ++k) S[f * nb + k] = (float)x[k];
  }
  if (S_out) std::copy(S.begin(), S.end(), S_out);
  const long long len = (long long)hop * (T - 1);
  std::vector<double2> a(H), bb(H);
  for (int it = 0; it <= n_iter; ++it) {
    for (long long f = 0; f < T; ++f) {
      double2 *in = a.data(), *out = bb.data();
      const float* Sf = S.data() + f * nb;
      if (it == 0) {
        for (int k = 0; k < nb; ++k) P[k] = mel::gl_scale(Sf[k], mel::gl_phase0(seed, f, k));
      } else {
        for (int k = 0; k < H; ++k) mel::load_point(tb, wav, len, f * hop, k, in);
        for (int Ns = 1; Ns < H; Ns *= 2) {
          for (int j = 0; j < H / 2; ++j) mel::fft_stage(tb, j, Ns, in, out);
          std::swap(in, out);
        }
        for (int k = 0; k < nb; ++k) P[k] = mel::gl_update(tb, k, in, Sf[k], tprev.data() + f * nb, it == 1);
      }
      for (int k = 0; k < H; ++k) mel::gl_pack(tb, k, P.data(), in);
      for (int Ns = 1; Ns < H; Ns *= 2) {
        for (int j = 0; j < H / 2; ++j) mel::fft_stage(tb, j, Ns, in, out);
        std::swap(in, out);
      }
      for (int k = 0; k < H; ++k) mel::gl_unpack(tb, k, in, frames.data() + f * N);
    }
    for (long long j = 0; j < len; ++j) wav[j] = mel::gl_ola(tb, frames.data(), T, j + H);
  }
  return WRNN_OK;
}

}  // extern "C"
