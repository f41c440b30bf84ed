// wrnn_cond.cu -- the conditioning network of generate() on the device, and the host-side restatements wrnn_vocode
// needs: the UpsampleNetwork's MelResNet (reference models/fatchord_version.py:26-48) with its eval-mode BatchNorms
// folded into the convolutions, the 5-tap interpolation table of the three stretch + conv stages (:64-80), fold_with_overlap's
// geometry (:319-330) and the float64 tables of the epilogue (:255, :379-391; utils/dsp.py:98-103).
//
// MelResNet is a chain of 128-wide 1x1 convolutions over frames (conv_in is k = 5 over 80 channels: K = 400 with the
// im2col done on the fly).  A CTA owns a tile of 64 frames and keeps its activations in shared memory through every
// layer; the folded weights (about 1.6 MB fp32 for 10 blocks) come from L2.  Arithmetic is fp32 FFMA on CUDA cores:
// the output also feeds the strict fp32 SIMT engine, and the whole network is ~0.4 MMAC per frame, small next to the
// sample loop (68 GMAC for a 172,034-frame job).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

#include "wrnn_cond.h"

namespace wrnn {
namespace cond {
namespace {

constexpr int TF = 64;                  // frames per CTA
constexpr int XS = TF + 4;              // row stride of the shared activations (17 float4: conflict-free float4 stores)
constexpr int THREADS = 256;            // 32 channel groups of 4 x 8 frame groups of 8
constexpr size_t SMEM = 2ull * CD * XS * sizeof(float);   // X and Y; the mel tile [FEAT][XS] aliases Y
static_assert(FEAT * XS <= CD * XS, "mel tile fits in Y");
static_assert(THREADS == (CD / 4) * (TF / 8), "one 4x8 output block per thread");

// acc[i][f] += sum_k W[k][o0 + i] * X[k][f0 + f]   (W from global, [k][CD]; X from shared, row stride XS)
template <int K>
__device__ __forceinline__ void gemm_tile(float (&acc)[4][8], const float* __restrict__ W, const float* X, int o0, int f0) {
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * CD + o0));
    const float4 xa = *reinterpret_cast<const float4*>(X + k * XS + f0);
    const float4 xb = *reinterpret_cast<const float4*>(X + k * XS + f0 + 4);
    const float x[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
    const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int f = 0; f < 8; ++f) acc[i][f] = fmaf(wv[i], x[f], acc[i][f]);
  }
}

__device__ __forceinline__ void init_bias(float (&acc)[4][8], const float* __restrict__ b, int o0) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(b + o0));
  const float bv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int f = 0; f < 8; ++f) acc[i][f] = bv[i];
}

__device__ __forceinline__ void store_tile(float* X, const float (&acc)[4][8], int o0, int f0, bool relu) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v[8];
#pragma unroll
    for (int f = 0; f < 8; ++f) v[f] = relu ? fmaxf(acc[i][f], 0.f) : acc[i][f];
    *reinterpret_cast<float4*>(X + (o0 + i) * XS + f0) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(X + (o0 + i) * XS + f0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// Utterance blockIdx.y of the batch: utts[blockIdx.y], or `one` when the batch is a single utterance (utts == NULL).
__device__ __forceinline__ CondUtt utt_of(const CondUtt* __restrict__ utts, const CondUtt& one, unsigned i) {
  return utts ? utts[i] : one;
}

// mel [FEAT, T] -> aux_frames [T, CD] of each utterance (rows frame0 .. frame0 + T - 1); blob as cond::blob_len describes
// (fp32, transposed matrices).  Grid: (tiles of TF frames of the longest utterance, utterances); a CTA serves one tile
// of one utterance, and the CTAs past the end of a shorter utterance return at once.
__global__ void __launch_bounds__(THREADS) melresnet_kernel(const CondUtt* __restrict__ utts, const CondUtt one,
                                                            const float* __restrict__ blob, int res_blocks,
                                                            float* __restrict__ aux_frames_all) {
  extern __shared__ __align__(16) float smem[];
  float* X = smem;                      // [CD][XS] activations of the tile
  float* Y = smem + CD * XS;            // [CD][XS] inner activations of a residual block
  float* M = Y;                         // [FEAT][XS] mel frames t0-2 .. t0+TF+1 (conv_in's receptive field)
  const CondUtt ut = utt_of(utts, one, blockIdx.y);
  const float* __restrict__ mel = ut.mel;
  const long long T = ut.T;
  const long long t0 = (long long)blockIdx.x * TF;
  if (t0 >= T) return;
  float* __restrict__ aux_frames = aux_frames_all + (size_t)ut.frame0 * CD;
  const int o0 = (threadIdx.x & 31) * 4, f0 = (threadIdx.x >> 5) * 8;

  for (int e = threadIdx.x; e < FEAT * XS; e += THREADS) {
    const int c = e / XS, fr = e - c * XS;
    const long long t = t0 + fr - 2;
    M[e] = (t >= 0 && t < T) ? __ldg(mel + (size_t)c * T + t) : 0.f;   // F.pad(mel, (2, 2)) zeros
  }
  __syncthreads();

  float acc[4][8];
  // conv_in + batch_norm + relu: out[o][t] = sum_{c, j} W[o][c][j] * melpad[c][t + j], k = c*5 + j
  const float* W = blob;
  init_bias(acc, W + (size_t)KIN * CD, o0);
#pragma unroll 1
  for (int c = 0; c < FEAT; ++c) {
    const float4 m0 = *reinterpret_cast<const float4*>(M + c * XS + f0);
    const float4 m1 = *reinterpret_cast<const float4*>(M + c * XS + f0 + 4);
    const float4 m2 = *reinterpret_cast<const float4*>(M + c * XS + f0 + 8);
    const float m[12] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w, m2.x, m2.y, m2.z, m2.w};
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(W + (size_t)(c * 5 + j) * CD + o0));
      const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int f = 0; f < 8; ++f) acc[i][f] = fmaf(wv[i], m[f + j], acc[i][f]);
    }
  }
  store_tile(X, acc, o0, f0, true);
  __syncthreads();
  W += (size_t)KIN * CD + CD;

  // residual blocks: x = bn2(conv2(relu(bn1(conv1(x))))) + x
#pragma unroll 1
  for (int r = 0; r < res_blocks; ++r) {
    init_bias(acc, W + CD * CD, o0);
    gemm_tile<CD>(acc, W, X, o0, f0);
    store_tile(Y, acc, o0, f0, true);
    __syncthreads();
    W += CD * CD + CD;
    init_bias(acc, W + CD * CD, o0);
    gemm_tile<CD>(acc, W, Y, o0, f0);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int f = 0; f < 8; ++f) acc[i][f] += X[(o0 + i) * XS + f0 + f];   // each thread owns these elements of X
    store_tile(X, acc, o0, f0, false);
    __syncthreads();
    W += CD * CD + CD;
  }

  // conv_out (with bias), written transposed: aux_frames[t][o]
  init_bias(acc, W + CD * CD, o0);
  gemm_tile<CD>(acc, W, X, o0, f0);
#pragma unroll
  for (int f = 0; f < 8; ++f) {
    const long long t = t0 + f0 + f;
    if (t < T) *reinterpret_cast<float4*>(aux_frames + (size_t)t * CD + o0) = make_float4(acc[0][f], acc[1][f], acc[2][f], acc[3][f]);
  }
}

// mel [FEAT, T] -> mel_frames [T + 4, FEAT] of each utterance (rows frame0 .. frame0 + T + 3): the zero-padded mel,
// transposed through a 32 x 32 shared tile.  Grid: (32-frame tiles of the longest padded utterance, channel tiles,
// utterances).
__global__ void __launch_bounds__(256) pad_transpose_kernel(const CondUtt* __restrict__ utts, const CondUtt one,
                                                            float* __restrict__ mel_frames_all) {
  __shared__ float tile[32][33];
  const CondUtt ut = utt_of(utts, one, blockIdx.z);
  const float* __restrict__ mel = ut.mel;
  const long long T = ut.T;
  const long long r0 = (long long)blockIdx.x * 32;            // padded frame
  if (r0 >= T + 4) return;
  float* __restrict__ mel_frames = mel_frames_all + (size_t)ut.frame0 * FEAT;
  const int c0 = blockIdx.y * 32;                             // channel
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i;
    const long long t = r0 + threadIdx.x - 2;
    tile[i][threadIdx.x] = (c < FEAT && t >= 0 && t < T) ? __ldg(mel + (size_t)c * T + t) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const long long r = r0 + i;
    const int c = c0 + threadIdx.x;
    if (r < T + 4 && c < FEAT) mel_frames[(size_t)r * FEAT + c] = tile[threadIdx.x][i];
  }
}

// numpy.linspace(start, stop, num) for num >= 1: i*step + start with the last element set to stop.  The product is
// kept apart from the sum so that no compiler contracts them into one fma.
void linspace(double start, double stop, int num, double* y) {
  if (num == 1) { y[0] = start; return; }
  const double step = (stop - start) / (double)(num - 1);
  for (int i = 0; i < num; ++i) {
    volatile double p = (double)i * step;
    y[i] = p + start;
  }
  y[num - 1] = stop;
}

int fetch(std::vector<double>& dst, const wrnn_tensor& t, bool host_only) {
  std::vector<float> f((size_t)t.numel);
  if (t.numel > 0) {
    if (!t.data) { set_error(std::string("null data pointer: ") + t.name); return WRNN_E_INVALID; }
    if (host_only) {
      std::memcpy(f.data(), t.data, f.size() * sizeof(float));
    } else {
      const cudaError_t e = cudaMemcpy(f.data(), t.data, f.size() * sizeof(float), cudaMemcpyDefault);
      if (e != cudaSuccess) { set_error(std::string("copying ") + t.name + ": " + cudaGetErrorString(e)); return WRNN_E_CUDA; }
    }
  }
  dst.assign(f.begin(), f.end());
  return WRNN_OK;
}

}  // namespace

int build_host_upsampler(const wrnn_upsample_cfg& cfg, const wrnn_tensor* t, int n, bool host_only, HostUpsampler& out) {
  if (cfg.compute_dims != CD || cfg.res_out_dims != CD) {
    set_error("unsupported dims: the conditioning network is specialised for compute_dims = res_out_dims = 128 "
              "(aux_dims = 32, hparams.py:47-49)");
    return WRNN_E_INVALID;
  }
  if (cfg.res_blocks < 0 || cfg.res_blocks > 1024) { set_error("res_blocks must be in [0, 1024]"); return WRNN_E_INVALID; }
  if (cfg.n_factors < 1 || cfg.n_factors > 4) { set_error("n_factors must be in [1, 4]"); return WRNN_E_INVALID; }
  long long prod = 1;
  for (int i = 0; i < cfg.n_factors; ++i) {
    if (cfg.factors[i] < 1 || cfg.factors[i] > 4096) { set_error("upsample factors must be in [1, 4096]"); return WRNN_E_INVALID; }
    prod *= cfg.factors[i];
  }
  if (cfg.pad != 2 || prod != cfg.hop_length) {
    set_error("the 5-tap conditioning table needs pad == 2 and a product of the upsample factors equal to hop_length");
    return WRNN_E_INVALID;
  }
  if (n < 0 || (n > 0 && !t)) { set_error("null tensor list"); return WRNN_E_INVALID; }

  // expected keys (state_dict names of UpsampleNetwork) -> element count
  const int R = cfg.res_blocks;
  std::map<std::string, long long> want;
  const std::string rn = "upsample.resnet.";
  auto bn = [&](const std::string& p) {
    for (const char* s : {"weight", "bias", "running_mean", "running_var"}) want[p + "." + s] = CD;
  };
  want[rn + "conv_in.weight"] = (long long)CD * KIN;
  bn(rn + "batch_norm");
  for (int r = 0; r < R; ++r) {
    const std::string l = rn + "layers." + std::to_string(r) + ".";
    want[l + "conv1.weight"] = CD * CD;
    want[l + "conv2.weight"] = CD * CD;
    bn(l + "batch_norm1");
    bn(l + "batch_norm2");
  }
  want[rn + "conv_out.weight"] = CD * CD;
  want[rn + "conv_out.bias"] = CD;
  for (int i = 0; i < cfg.n_factors; ++i) want["upsample.up_layers." + std::to_string(2 * i + 1) + ".weight"] = 2 * cfg.factors[i] + 1;

  std::map<std::string, std::vector<double>> got;
  const std::string pre = "upsample.", nbt = ".num_batches_tracked";
  for (int i = 0; i < n; ++i) {
    if (!t[i].name) { set_error("wrnn_tensor without a name"); return WRNN_E_INVALID; }
    const std::string k = t[i].name;
    if (k.compare(0, pre.size(), pre) != 0) continue;
    if (k.size() >= nbt.size() && k.compare(k.size() - nbt.size(), nbt.size(), nbt) == 0) continue;
    auto it = want.find(k);
    if (it == want.end()) { set_error("unexpected key in the upsampler's tensors: " + k); return WRNN_E_INVALID; }
    if (got.count(k)) { set_error("repeated key: " + k); return WRNN_E_INVALID; }
    if (t[i].numel != it->second) {
      set_error(k + " has " + std::to_string((long long)t[i].numel) + " elements, expected " + std::to_string(it->second));
      return WRNN_E_INVALID;
    }
    const int rc = fetch(got[k], t[i], host_only);
    if (rc != WRNN_OK) return rc;
  }
  for (const auto& kv : want)
    if (!got.count(kv.first)) { set_error("missing key: " + kv.first); return WRNN_E_INVALID; }

  // interpolation table: a unit impulse at frame c of n_fr pushed through the stretch + conv stages (the same
  // construction as WaveRNN.upsample_taps), then mel_up[n] = sum_d taps[n % hop][d] * mel_padded[n / hop + d]
  const int hop = cfg.hop_length, n_fr = 9, c = 4;
  std::vector<double> x(n_fr, 0.0);
  x[c] = 1.0;
  for (int i = 0; i < cfg.n_factors; ++i) {
    const int s = cfg.factors[i];
    const std::vector<double>& w = got["upsample.up_layers." + std::to_string(2 * i + 1) + ".weight"];
    std::vector<double> rep(x.size() * s), y(x.size() * s);
    for (size_t q = 0; q < rep.size(); ++q) rep[q] = x[q / s];
    for (long long q = 0; q < (long long)y.size(); ++q) {
      double a = 0.0;
      for (int m = 0; m <= 2 * s; ++m) {
        const long long src = q + m - s;
        if (src >= 0 && src < (long long)rep.size()) a += w[m] * rep[src];
      }
      y[q] = a;
    }
    x.swap(y);
  }
  out.taps.assign((size_t)hop * TAPS, 0.0);
  for (long long q = 0; q < (long long)x.size(); ++q) {
    const long long d = c - q / hop + 2;
    if (d >= 0 && d < TAPS) out.taps[(size_t)(q % hop) * TAPS + d] = x[q];
    else if (x[q] != 0.0) {
      set_error("the interpolation cascade's impulse response is wider than the 5-tap table (+-2 frames)");
      return WRNN_E_INVALID;
    }
  }

  // BatchNorm folding: bn(conv(x)) = (W*s) x + (beta - mean*s), s = gamma / sqrt(var + eps)
  out.res_blocks = R;
  out.hop = hop;
  out.blob.assign(blob_len(R), 0.0);
  double* b = out.blob.data();
  auto put = [&](const std::string& wkey, const std::string& bnkey, int K) {
    const std::vector<double>& W = got[wkey];
    std::vector<double> s(CD, 1.0), bias(CD, 0.0);
    if (!bnkey.empty()) {
      const std::vector<double>&g = got[bnkey + ".weight"], &be = got[bnkey + ".bias"], &mu = got[bnkey + ".running_mean"],
                           &var = got[bnkey + ".running_var"];
      for (int o = 0; o < CD; ++o) { s[o] = g[o] / std::sqrt(var[o] + BN_EPS); bias[o] = be[o] - mu[o] * s[o]; }
    } else {
      bias = got[rn + "conv_out.bias"];
    }
    for (int k = 0; k < K; ++k)
      for (int o = 0; o < CD; ++o) b[(size_t)k * CD + o] = W[(size_t)o * K + k] * s[o];
    b += (size_t)K * CD;
    for (int o = 0; o < CD; ++o) b[o] = bias[o];
    b += CD;
  };
  put(rn + "conv_in.weight", rn + "batch_norm", KIN);
  for (int r = 0; r < R; ++r) {
    const std::string l = rn + "layers." + std::to_string(r) + ".";
    put(l + "conv1.weight", l + "batch_norm1", CD);
    put(l + "conv2.weight", l + "batch_norm2", CD);
  }
  put(rn + "conv_out.weight", "", CD);
  return WRNN_OK;
}

Geometry fold_geometry(int64_t total_len, bool batched, int64_t target, int64_t overlap) {
  if (!batched) return Geometry{1, total_len, total_len, 0, total_len};
  const int64_t num = total_len - overlap, den = target + overlap;
  int64_t n = num / den;
  if ((num % den != 0) && ((num < 0) != (den < 0))) --n;     // Python's floor division
  const int64_t remaining = total_len - (n * (overlap + target) + overlap);
  int64_t padded = total_len;
  if (remaining != 0) {
    n += 1;
    padded = total_len + (target + 2 * overlap - remaining);
  }
  return Geometry{n, target + 2 * overlap, target + overlap, overlap, padded};
}

int batch_plan(int hop, const wrnn_vocode_batch& b, BatchPlan& out) {
  if (b.n_utts < 1 || b.n_utts > 65535 || !b.utts) { set_error("a batch needs 1 to 65535 utterances and a non-null utts array"); return WRNN_E_INVALID; }
  if (b.batched && (b.target <= 0 || b.overlap <= 0)) { set_error("a batched job needs target > 0 and overlap > 0"); return WRNN_E_INVALID; }
  out = BatchPlan();
  int64_t frames = 0, waves = 0;
  for (int i = 0; i < b.n_utts; ++i) {
    const wrnn_utterance& u = b.utts[i];
    const std::string at = "utterance " + std::to_string(i) + ": ";
    const int rc = check_utterance(at, u.mel, u.wav, u.T);
    if (rc != WRNN_OK) return rc;
    if (u.T >= (1ll << 31) / hop) { set_error(at + "stream longer than 2^31 samples"); return WRNN_E_INVALID; }
    out.frame0.push_back(frames); out.wav0.push_back(waves);
    frames += u.T + 4; waves += (u.T - 1) * hop;
    if (frames * hop >= (1ll << 31)) { set_error("the laid-out stream of the batch is 2^31 samples or longer"); return WRNN_E_INVALID; }
    if (u.T > out.max_T) out.max_T = u.T;
  }
  out.frame0.push_back(frames); out.wav0.push_back(waves);
  out.L = frames * hop;
  out.max_wave = (out.max_T - 1) * hop;
  if (b.batched) {
    out.g = Geometry{0, (int64_t)b.target + 2ll * b.overlap, (int64_t)b.target + b.overlap, b.overlap, 0};   // fold_with_overlap's
    if (out.g.seg_len >= (1ll << 31)) { set_error("target + 2 * overlap must be below 2^31"); return WRNN_E_INVALID; }
  } else {
    out.g = Geometry{0, out.max_T * hop, out.max_T * hop, 0, 0};
  }
  int64_t folds = 0;
  for (int i = 0; i < b.n_utts; ++i) {
    const int64_t Ti = b.utts[i].T, n = b.batched ? fold_geometry(Ti * hop, true, b.target, b.overlap).n_seg : 1;
    if (n < 1) { set_error("utterance " + std::to_string(i) + ": target / overlap give no fold"); return WRNN_E_INVALID; }
    out.fold0.push_back(folds);
    folds += n;
    if (folds >= (1ll << 31)) { set_error("the batch has 2^31 folds or more"); return WRNN_E_INVALID; }
  }
  out.fold0.push_back(folds);
  out.g.n_seg = folds;
  out.row0.reserve(folds); out.row_end.reserve(folds); out.keys.reserve(folds);
  for (int i = 0; i < b.n_utts; ++i) {
    const int64_t R = out.frame0[i] * hop, end = R + b.utts[i].T * hop;
    for (int64_t j = 0; j < out.fold0[i + 1] - out.fold0[i]; ++j) {
      out.row0.push_back(R + (b.batched ? j * out.g.seg_stride : 0));
      out.row_end.push_back(end);
      out.keys.push_back(FoldKey{b.utts[i].philox_seed, (uint32_t)j, 0u});
    }
  }
  return WRNN_OK;
}

int score_plan(int hop, const wrnn_score_utt* utts, int n_utts, BatchPlan& out) {
  if (n_utts < 1 || n_utts > 65535 || !utts) { set_error("a batch needs 1 to 65535 utterances and a non-null utts array"); return WRNN_E_INVALID; }
  out = BatchPlan();
  int64_t frames = 0, losses = 0, max_n = 0;
  for (int i = 0; i < n_utts; ++i) {
    const wrnn_score_utt& u = utts[i];
    const std::string at = "utterance " + std::to_string(i) + ": ";
    if (!u.mel || !u.x || !u.nll) { set_error(at + "mel, x and nll are required"); return WRNN_E_INVALID; }
    if (u.T < 1 || u.T >= (1ll << 31) / hop) { set_error(at + "T must be >= 1 and the stream shorter than 2^31 samples"); return WRNN_E_INVALID; }
    if (u.n < 1 || u.n > u.T * hop) { set_error(at + "n must be in [1, T * hop]: one target per conditioning row"); return WRNN_E_INVALID; }
    out.frame0.push_back(frames); out.wav0.push_back(losses); out.fold0.push_back(i);
    out.row0.push_back(frames * hop); out.row_end.push_back((frames + u.T) * hop);
    frames += u.T + 4; losses += u.n;
    if (frames * hop >= (1ll << 31)) { set_error("the laid-out stream of the batch is 2^31 samples or longer"); return WRNN_E_INVALID; }
    if (u.T > out.max_T) out.max_T = u.T;
    if (u.n > max_n) max_n = u.n;
  }
  out.frame0.push_back(frames); out.wav0.push_back(losses); out.fold0.push_back(n_utts);
  out.L = frames * hop;
  out.g = Geometry{n_utts, max_n, max_n, 0, 0};
  return WRNN_OK;
}

void epilogue_tables(int overlap, bool mu_law, int n_classes, int hop, std::vector<double>& fade_in,
                     std::vector<double>& fade_out, std::vector<double>& mu, std::vector<double>& tail) {
  fade_in.clear(); fade_out.clear(); mu.clear();
  if (overlap > 0) {                    // xfade_and_unfold: silence, then an equal-power fade over linspace(-1, 1)
    const int silence = overlap / 2, m = overlap - silence;
    std::vector<double> t(m);
    linspace(-1.0, 1.0, m, t.data());
    fade_in.assign(silence, 0.0);
    fade_out.assign(silence, 1.0);
    for (int i = 0; i < m; ++i) {
      fade_in.push_back(std::sqrt(0.5 * (1.0 + t[i])));
      fade_out.push_back(std::sqrt(0.5 * (1.0 - t[i])));
    }
  }
  if (mu_law) {                         // the kernel's samples are x_k = 2k/(n-1) - 1 in fp32: expand exactly those
    const double m = (double)(n_classes - 1);
    for (int k = 0; k < n_classes; ++k) {
      const float x2 = 2.0f * (float)k;
      const float xq = x2 / (float)(n_classes - 1);
      const double y = (double)(xq - 1.0f);
      const double sgn = y > 0.0 ? 1.0 : (y < 0.0 ? -1.0 : 0.0);
      mu.push_back(sgn / m * (std::pow((double)n_classes, std::fabs(y)) - 1.0));
    }
  }
  tail.resize((size_t)20 * hop);
  linspace(1.0, 0.0, 20 * hop, tail.data());
}

}  // namespace cond

Upsampler::~Upsampler() {
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(device);
  if (d_blob) cudaFree(d_blob);
  if (d_taps) cudaFree(d_taps);
  if (d_scratch) cudaFree(d_scratch);
  if (d_tabs) cudaFree(d_tabs);
  cudaSetDevice(prev);
}

void destroy_upsampler(Upsampler* u) { delete u; }

int make_upsampler(const cond::HostUpsampler& hu, int device, Upsampler** out) {
  *out = nullptr;
  Upsampler* u = new (std::nothrow) Upsampler();
  if (!u) { set_error("out of host memory"); return WRNN_E_INVALID; }
  u->device = device; u->res_blocks = hu.res_blocks; u->hop = hu.hop;
  std::vector<float> blob(hu.blob.begin(), hu.blob.end()), taps(hu.taps.begin(), hu.taps.end());
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaMalloc(&u->d_blob, blob.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&u->d_taps, taps.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMemcpy(u->d_blob, blob.data(), blob.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(u->d_taps, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(cond::melresnet_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cond::SMEM);
  if (e != cudaSuccess) {
    set_error(std::string("uploading the conditioning network: ") + cudaGetErrorString(e));
    delete u;
    return WRNN_E_CUDA;
  }
  *out = u;
  return WRNN_OK;
}

// Both kernels over a batch: the utterance table `utts` (device) or, for one utterance, `one` passed by value.
static int launch_conditioning(const Upsampler& u, const CondUtt* utts, const CondUtt& one, int n_utts, long long max_T,
                               float* mel_frames, float* aux_frames, cudaStream_t stream) {
  using namespace cond;
  pad_transpose_kernel<<<dim3((unsigned)((max_T + 4 + 31) / 32), (FEAT + 31) / 32, (unsigned)n_utts), dim3(32, 8), 0, stream>>>(
      utts, one, mel_frames);
  WRNN_CUDA_OK(cudaGetLastError());
  melresnet_kernel<<<dim3((unsigned)((max_T + TF - 1) / TF), (unsigned)n_utts), THREADS, SMEM, stream>>>(utts, one, u.d_blob,
                                                                                                      u.res_blocks, aux_frames);
  WRNN_CUDA_OK(cudaGetLastError());
  return WRNN_OK;
}

int conditioning_frames(const Upsampler& u, const float* mel, long long T, float* mel_frames, float* aux_frames, float* up_taps,
                        cudaStream_t stream) {
  const CondUtt one{mel, T, 0};
  const int rc = launch_conditioning(u, nullptr, one, 1, T, mel_frames, aux_frames, stream);
  if (rc != WRNN_OK) return rc;
  if (up_taps) WRNN_CUDA_OK(cudaMemcpyAsync(up_taps, u.d_taps, (size_t)u.hop * cond::TAPS * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  return WRNN_OK;
}

int conditioning_frames_batch(const Upsampler& u, const CondUtt* utts, int n_utts, long long max_T, float* mel_frames,
                              float* aux_frames, cudaStream_t stream) {
  return launch_conditioning(u, utts, CondUtt{nullptr, 0, 0}, n_utts, max_T, mel_frames, aux_frames, stream);
}

}  // namespace wrnn

using namespace wrnn;

extern "C" {

int wrnn_attach_upsampler(wrnn_t* h, const wrnn_upsample_cfg* cfg, const wrnn_tensor* t, int32_t n) {
  if (!h || !h->engine || !cfg) { set_error("null handle or cfg"); return WRNN_E_INVALID; }
  if (h->live_busy || h->session) return idle_or_busy(h);
  WRNN_CUDA_OK(cudaSetDevice(h->engine->device));
  cond::HostUpsampler hu;
  int rc = cond::build_host_upsampler(*cfg, t, n, false, hu);
  if (rc != WRNN_OK) return rc;
  Upsampler* u = nullptr;
  if ((rc = make_upsampler(hu, h->engine->device, &u)) != WRNN_OK) return rc;
  destroy_upsampler(h->upsampler);
  h->upsampler = u;
  return WRNN_OK;
}

int wrnn_conditioning_frames(wrnn_t* h, const float* mel, int64_t T, float* mel_frames, float* aux_frames, float* up_taps,
                             void* stream) {
  if (!h || !h->engine) { set_error("null handle"); return WRNN_E_INVALID; }
  if (h->live_busy || h->session) return idle_or_busy(h);
  if (!h->upsampler) { set_error("no upsampler attached (wrnn_attach_upsampler)"); return WRNN_E_INVALID; }
  if (!mel || !mel_frames || !aux_frames || T <= 0 || T >= (1ll << 31)) {
    set_error("wrnn_conditioning_frames: bad argument"); return WRNN_E_INVALID;
  }
  WRNN_CUDA_OK(cudaSetDevice(h->upsampler->device));
  return conditioning_frames(*h->upsampler, mel, T, mel_frames, aux_frames, up_taps, static_cast<cudaStream_t>(stream));
}

// Test hooks (CPU-only, no device needed; not part of the reference-facing surface), checked in tests/test_vocode_abi.py.
// out[5] = n_seg, seg_len, seg_stride, overlap, padded_len of the job wrnn_vocode would run.
int wrnn_debug_fold_geometry(int64_t total_len, int32_t batched, int64_t target, int64_t overlap, int64_t* out) {
  if (!out) { set_error("null argument"); return WRNN_E_INVALID; }
  const cond::Geometry g = cond::fold_geometry(total_len, batched != 0, target, overlap);
  out[0] = g.n_seg; out[1] = g.seg_len; out[2] = g.seg_stride; out[3] = g.overlap; out[4] = g.padded_len;
  return WRNN_OK;
}

// The layout wrnn_vocode_many runs for batch b at this hop (cond::batch_plan), or its refusal.  geo[7] = n_seg, seg_len,
// seg_stride, overlap, L (rows of the laid-out stream), max_T, total waveform samples; utt [n_utts][3] = frame0, fold0,
// wav0 per utterance; folds [n_seg][4] = fold_row0, fold_row_end, key seed (bits of the uint64), key fold.  utt and
// folds may be NULL (sizes first).  mel / wav are only tested against NULL.
int wrnn_debug_vocode_many_plan(int32_t hop, const wrnn_vocode_batch* b, int64_t* geo, int64_t* utt, int64_t* folds) {
  if (!b || !geo || hop <= 0) { set_error("null argument"); return WRNN_E_INVALID; }
  cond::BatchPlan pl;
  const int rc = cond::batch_plan(hop, *b, pl);
  if (rc != WRNN_OK) return rc;
  const int64_t g[7] = {pl.g.n_seg, pl.g.seg_len, pl.g.seg_stride, pl.g.overlap, pl.L, pl.max_T, pl.wav0.back()};
  std::memcpy(geo, g, sizeof(g));
  if (utt)
    for (int i = 0; i < b->n_utts; ++i) { utt[3 * i] = pl.frame0[i]; utt[3 * i + 1] = pl.fold0[i]; utt[3 * i + 2] = pl.wav0[i]; }
  if (folds)
    for (int64_t f = 0; f < pl.g.n_seg; ++f) {
      folds[4 * f] = pl.row0[f]; folds[4 * f + 1] = pl.row_end[f];
      folds[4 * f + 2] = (int64_t)pl.keys[f].seed; folds[4 * f + 3] = pl.keys[f].fold;
    }
  return WRNN_OK;
}

// The layout wrnn_score_many runs for these utterances at this hop (cond::score_plan), or its refusal.  geo[5] = n_seg,
// steps (max n_i), L (rows of the laid-out stream), max_T, total losses; folds [n_utts][4] = fold_row0, fold_row_end,
// frame0, offset of the utterance's losses.  folds may be NULL.  mel / x / nll are only tested against NULL.
int wrnn_debug_score_many_plan(int32_t hop, const wrnn_score_utt* utts, int32_t n_utts, int64_t* geo, int64_t* folds) {
  if (!geo || hop <= 0) { set_error("null argument"); return WRNN_E_INVALID; }
  cond::BatchPlan pl;
  const int rc = cond::score_plan(hop, utts, n_utts, pl);
  if (rc != WRNN_OK) return rc;
  const int64_t g[5] = {pl.g.n_seg, pl.g.seg_len, pl.L, pl.max_T, pl.wav0.back()};
  std::memcpy(geo, g, sizeof(g));
  if (folds)
    for (int i = 0; i < n_utts; ++i) {
      folds[4 * i] = pl.row0[i]; folds[4 * i + 1] = pl.row_end[i]; folds[4 * i + 2] = pl.frame0[i]; folds[4 * i + 3] = pl.wav0[i];
    }
  return WRNN_OK;
}

// The epilogue tables wrnn_vocode uploads: fade_in / fade_out [overlap], mu [n_classes] (mu_law), tail [20*hop];
// NULL for a table not wanted.
int wrnn_debug_epilogue_tables(int32_t overlap, int32_t mu_law, int32_t n_classes, int32_t hop, double* fade_in,
                               double* fade_out, double* mu, double* tail) {
  if (overlap < 0 || hop <= 0 || (mu_law && n_classes < 2)) { set_error("bad argument"); return WRNN_E_INVALID; }
  std::vector<double> fi, fo, m, tl;
  cond::epilogue_tables(overlap, mu_law != 0, n_classes, hop, fi, fo, m, tl);
  if (fade_in) std::memcpy(fade_in, fi.data(), fi.size() * sizeof(double));
  if (fade_out) std::memcpy(fade_out, fo.data(), fo.size() * sizeof(double));
  if (mu) std::memcpy(mu, m.data(), m.size() * sizeof(double));
  if (tail) std::memcpy(tail, tl.data(), tl.size() * sizeof(double));
  return WRNN_OK;
}

// wrnn_attach_upsampler's host half on HOST tensors: the checks, the folded parameters in double before the fp32 upload
// (layout of cond::blob_len; *blob_len receives the element count, blob may be NULL) and the tap table [hop][5] in double.
int wrnn_debug_upsampler(const wrnn_upsample_cfg* cfg, const wrnn_tensor* t, int32_t n, double* blob, uint64_t* blob_len,
                         double* taps) {
  if (!cfg) { set_error("null argument"); return WRNN_E_INVALID; }
  cond::HostUpsampler hu;
  const int rc = cond::build_host_upsampler(*cfg, t, n, true, hu);
  if (rc != WRNN_OK) return rc;
  if (blob_len) *blob_len = hu.blob.size();
  if (blob) std::memcpy(blob, hu.blob.data(), hu.blob.size() * sizeof(double));
  if (taps) std::memcpy(taps, hu.taps.data(), hu.taps.size() * sizeof(double));
  return WRNN_OK;
}

}  // extern "C"
