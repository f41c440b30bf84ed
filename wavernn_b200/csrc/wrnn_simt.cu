// wrnn_simt.cu -- SIMT engine: the whole generate() loop (reference
// models/fatchord_version.py:201-241 + utils/distribution.py:87-123) as ONE persistent
// cooperative kernel, contractions on CUDA cores.
//
// Role: the strict-arithmetic engine.  In FP32 mode it reproduces the reference to
// re-association error (weights, activations and accumulation all fp32), which proves the
// folded algebra (wrnn_fold.h), the exchange protocol, the fold indexing and the samplers
// independently of tensor-core rounding; in BF16 mode it applies exactly the rounding
// contract of the tensor-core engines (operands rounded to bf16, fp32 accumulate).
//
// Decomposition: P = 128 CTAs; CTA c owns hidden units [4c, 4c+4) of every layer and keeps
// its slice of all matrices resident in shared memory for the whole launch.  Per step the
// CTAs exchange the four 512-wide activation vectors (h1', h2', y1, y2) through L2-resident
// buffers laid out [unit][fold] (coalesced for producers and consumers) with a grid
// barrier after each; fold tiles of 32 are sampled by CTA (tile % P).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <vector>

#include "wrnn_device.cuh"
#include "wrnn_engine.h"

namespace wrnn {
namespace {

constexpr int P = 128;            // CTAs == weight shards
constexpr int U = H / P;          // hidden units per CTA (4)
constexpr int NT = 256;           // threads per CTA
constexpr int FT = 32;            // folds per tile (== warp width)
constexpr int AP = FT + 1;        // activation tile pitch (bank-conflict padding)

constexpr int QROWS = 8 * U;      // 32
constexpr int S1ROWS = 8 * U;     // 28 real + 4 zero rows
constexpr int S2ROWS = 4 * U;     // 16
constexpr int S3ROWS = U;         // 4
constexpr int S4ROWS = U;         // RAW: rows of fc3 owned by this CTA (n_classes == 4*P)
constexpr int MAT_ELEMS = CDIM * QROWS + H * (S1ROWS + S2ROWS + S3ROWS + S4ROWS);
constexpr int NVEC = 96;          // qk[32] vq[32] b1h[12] b2h[12] b3s[4] (+4 pad)
constexpr int F3ROWS = 32;        // MOL: fc3 rows padded 30 -> 32, read from global by sampler CTAs

// per-fold state kept by the owning CTA (fp32), field-major [field][Bp]
enum { ST_H1 = 0, ST_H2 = 4, ST_GH1 = 8, ST_GH2 = 20, ST_FC1P = 32, ST_PGI2 = 36, ST_PFC1 = 48, ST_PFC2 = 52,
       NSTATE = 56 };

struct SimtParams {
  const unsigned char* blob; size_t blob_stride;
  const void* f3t; const float* b3;
  const float* mels_up; const float* aux; long long L; long long seg_stride;
  int n_seg, seg_len, seg_first, steps, Bp, out_pitch, n_classes, mode;
  const float* uniforms; const float* expo; unsigned long long seed, offset;
  float* out; const float* x_force; float* logits_out;
  const long long* fold_row0; const long long* fold_row_end;
  const FoldKey* keys;   // optional per-fold Philox keys [n_seg]
  float* xch;      // 4 x [H][Bp]: h1', h2', y1, y2
  float* xs;       // [Bp] previous sample per fold
  float* state;    // [P][NSTATE][Bp]
  float* xlog;     // RAW: [n_classes][Bp]
  unsigned* counter; int* abort_flag;
  float* nll;      // scoring: [steps][n_seg] loss of target x_force[t] (out is not written)
};

__device__ __forceinline__ float4 load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load4(const __nv_bfloat16* p) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u),
                     __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xffff0000u));
}

// outs[task][4][AP], task = ks*RG + rg.  Warp `task` accumulates rows 4rg..4rg+3 over its k-slice
// for the 32 folds of the tile (lane == fold).  W is k-major [K][ROWS].
__device__ __forceinline__ float4 load4(const __half* p) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
// operand rounding of the arithmetic contract (identity for the fp32 strict mode)
template <typename T> __device__ __forceinline__ float round_op(float v);
template <> __device__ __forceinline__ float round_op<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_op<__nv_bfloat16>(float v) { return bf16_round(v); }
template <> __device__ __forceinline__ float round_op<__half>(float v) { return f16_round(v); }

template <typename T, int ROWS>
__device__ __forceinline__ void gemv_tile(const T* __restrict__ W, int K, const float* __restrict__ act,
                                          float* __restrict__ outs) {
  constexpr int RG = ROWS / 4;
  constexpr int KS = 8 / RG;
  static_assert(RG * KS == 8, "ROWS must be 4, 8, 16 or 32");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rg = warp % RG, ks = warp / RG;
  const int kn = K / KS, k0 = ks * kn;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 8
  for (int k = k0; k < k0 + kn; ++k) {
    const float a = act[k * AP + lane];
    const float4 w = load4(W + (size_t)k * ROWS + 4 * rg);
    a0 = fmaf(w.x, a, a0); a1 = fmaf(w.y, a, a1); a2 = fmaf(w.z, a, a2); a3 = fmaf(w.w, a, a3);
  }
  float* o = outs + (warp * 4) * AP + lane;
  o[0] = a0; o[AP] = a1; o[2 * AP] = a2; o[3 * AP] = a3;
}
template <int ROWS>
__device__ __forceinline__ float out_row(const float* outs, int row, int f) {
  constexpr int RG = ROWS / 4;
  constexpr int KS = 8 / RG;
  float s = 0.f;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) s += outs[((ks * RG + row / 4) * 4 + (row & 3)) * AP + f];
  return s;
}

// SCORE: the sampler's place takes the loss of target x_force[t] (wrnn_score); no draws are made.
template <typename T, bool SCORE>
__global__ void __launch_bounds__(NT, 1) wrnn_simt_kernel(const SimtParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  T* wQ = reinterpret_cast<T*>(smem);
  T* wS1 = wQ + CDIM * QROWS;
  T* wS2 = wS1 + H * S1ROWS;
  T* wS3 = wS2 + H * S2ROWS;
  T* wS4 = wS3 + H * S3ROWS;
  float* fv = reinterpret_cast<float*>(wS4 + H * S4ROWS);
  const float* qk = fv; const float* vq = fv + 32; const float* b1h = fv + 64; const float* b2h = fv + 76;
  const float* b3s = fv + 88;
  float* act = fv + NVEC;
  float* outs = act + H * AP;

  const int cta = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int B = p.n_seg, Bp = p.Bp, ntiles = Bp / FT, u0 = cta * U;
  const int S = p.steps;

  {  // stage this CTA's weight shard once
    const int4* src = reinterpret_cast<const int4*>(p.blob + (size_t)cta * p.blob_stride);
    const int n16 = (int)((MAT_ELEMS * sizeof(T) + NVEC * sizeof(float)) / 16);
    for (int i = tid; i < n16; i += NT) reinterpret_cast<int4*>(smem)[i] = src[i];
  }
  __syncthreads();
  float* st = p.state + (size_t)cta * NSTATE * Bp;
  for (int idx = tid; idx < NSTATE * Bp; idx += NT) {   // h = 0  =>  W_hh h + b_hh = b_hh  (:194-196)
    const int f = idx / Bp;
    float v = 0.f;
    if (f >= ST_GH1 && f < ST_GH1 + 12) v = b1h[f - ST_GH1];
    if (f >= ST_GH2 && f < ST_GH2 + 12) v = b2h[f - ST_GH2];
    st[idx] = v;
  }
  __syncthreads();

  float* xh1 = p.xch; float* xh2 = p.xch + (size_t)H * Bp; float* xy1 = p.xch + (size_t)2 * H * Bp;
  float* xy2 = p.xch + (size_t)3 * H * Bp;
  unsigned nbar = 0;
#define WRNN_BARRIER()                                                              \
  do {                                                                              \
    ++nbar;                                                                         \
    if (!grid_barrier(p.counter, nbar * (unsigned)gridDim.x, p.abort_flag)) return; \
  } while (0)

  auto load_xch_tile = [&](const float* x, int b0) {    // [H][Bp] global -> act[k][fold]
    for (int idx = tid; idx < H * FT; idx += NT) {
      const int k = idx >> 5, f = idx & 31;
      act[k * AP + f] = __ldcg(x + (size_t)k * Bp + b0 + f);
    }
  };
  auto rnd = [&](float v) { return round_op<T>(v); };

  for (int t = 0; t < S; ++t) {
    // ---- phase A: pre = Q cond_t + qk + x vq ; GRU1 (gi1 is conditioning + rank-1 in x) -----------
    for (int tile = 0; tile < ntiles; ++tile) {
      const int b0 = tile * FT;
      for (int idx = tid; idx < CDIM * FT; idx += NT) {
        const int c = idx % CDIM, f = idx / CDIM, b = b0 + f;
        long long row = (long long)b * p.seg_stride + t, row_end = p.L;
        if (p.fold_row0 && b < B) { row = __ldg(p.fold_row0 + b) + t; row_end = __ldg(p.fold_row_end + b); }
        float v = 0.f;
        if (b < B && row < row_end) v = (c < FEAT) ? __ldg(p.mels_up + row * FEAT + c) : __ldg(p.aux + row * (4 * AUXD) + (c - FEAT));
        act[c * AP + f] = rnd(v);
      }
      __syncthreads();
      gemv_tile<T, QROWS>(wQ, CDIM, act, outs);
      __syncthreads();
      if (tid < U * FT) {
        const int f = tid & 31, j = tid >> 5, b = b0 + f;
        if (b < B) {
          float x = 0.f;
          if (t > 0) x = p.x_force ? __ldg(p.x_force + (size_t)(t - 1) * B + b) : __ldcg(p.xs + b);
          auto pre = [&](int q) { return out_row<QROWS>(outs, q, f) + qk[q] + x * vq[q]; };
          const float h = st[(ST_H1 + j) * Bp + b];
          const float hn = gru_unit(pre(j), pre(U + j), pre(2 * U + j), st[(ST_GH1 + j) * Bp + b],
                                    st[(ST_GH1 + U + j) * Bp + b], st[(ST_GH1 + 2 * U + j) * Bp + b], h);
          st[(ST_H1 + j) * Bp + b] = hn;
          st[(ST_PGI2 + j) * Bp + b] = pre(3 * U + j);
          st[(ST_PGI2 + U + j) * Bp + b] = pre(4 * U + j);
          st[(ST_PGI2 + 2 * U + j) * Bp + b] = pre(5 * U + j);
          st[(ST_PFC1 + j) * Bp + b] = pre(6 * U + j);
          st[(ST_PFC2 + j) * Bp + b] = pre(7 * U + j);
          xh1[(size_t)(u0 + j) * Bp + b] = rnd(hn);
        }
      }
      __syncthreads();
    }
    WRNN_BARRIER();
    // ---- phase B: [W2x ; W1h ; F1x] h1'  -> GRU2, next step's gh1, fc1 partial --------------------
    for (int tile = 0; tile < ntiles; ++tile) {
      const int b0 = tile * FT;
      load_xch_tile(xh1, b0);
      __syncthreads();
      gemv_tile<T, S1ROWS>(wS1, H, act, outs);
      __syncthreads();
      if (tid < U * FT) {
        const int f = tid & 31, j = tid >> 5, b = b0 + f;
        if (b < B) {
          auto o = [&](int r) { return out_row<S1ROWS>(outs, r, f); };
          const float h = st[(ST_H2 + j) * Bp + b];
          const float hn = gru_unit(o(j) + st[(ST_PGI2 + j) * Bp + b], o(U + j) + st[(ST_PGI2 + U + j) * Bp + b],
                                    o(2 * U + j) + st[(ST_PGI2 + 2 * U + j) * Bp + b], st[(ST_GH2 + j) * Bp + b],
                                    st[(ST_GH2 + U + j) * Bp + b], st[(ST_GH2 + 2 * U + j) * Bp + b], h);
          st[(ST_H2 + j) * Bp + b] = hn;
          st[(ST_GH1 + j) * Bp + b] = o(3 * U + j) + b1h[j];
          st[(ST_GH1 + U + j) * Bp + b] = o(4 * U + j) + b1h[U + j];
          st[(ST_GH1 + 2 * U + j) * Bp + b] = o(5 * U + j) + b1h[2 * U + j];
          st[(ST_FC1P + j) * Bp + b] = o(6 * U + j);
          xh2[(size_t)(u0 + j) * Bp + b] = rnd(hn);
        }
      }
      __syncthreads();
    }
    WRNN_BARRIER();
    // ---- phase C: [F1x ; W2h] h2' -> y1 = relu(fc1), next step's gh2 -------------------------------
    for (int tile = 0; tile < ntiles; ++tile) {
      const int b0 = tile * FT;
      load_xch_tile(xh2, b0);
      __syncthreads();
      gemv_tile<T, S2ROWS>(wS2, H, act, outs);
      __syncthreads();
      if (tid < U * FT) {
        const int f = tid & 31, j = tid >> 5, b = b0 + f;
        if (b < B) {
          auto o = [&](int r) { return out_row<S2ROWS>(outs, r, f); };
          const float y = fmaxf(st[(ST_FC1P + j) * Bp + b] + o(j) + st[(ST_PFC1 + j) * Bp + b], 0.f);
          st[(ST_GH2 + j) * Bp + b] = o(U + j) + b2h[j];
          st[(ST_GH2 + U + j) * Bp + b] = o(2 * U + j) + b2h[U + j];
          st[(ST_GH2 + 2 * U + j) * Bp + b] = o(3 * U + j) + b2h[2 * U + j];
          xy1[(size_t)(u0 + j) * Bp + b] = rnd(y);
        }
      }
      __syncthreads();
    }
    WRNN_BARRIER();
    // ---- phase D: F2x y1 -> y2 = relu(fc2) ---------------------------------------------------------
    for (int tile = 0; tile < ntiles; ++tile) {
      const int b0 = tile * FT;
      load_xch_tile(xy1, b0);
      __syncthreads();
      gemv_tile<T, S3ROWS>(wS3, H, act, outs);
      __syncthreads();
      if (tid < U * FT) {
        const int f = tid & 31, j = tid >> 5, b = b0 + f;
        if (b < B) {
          const float y = fmaxf(out_row<S3ROWS>(outs, j, f) + st[(ST_PFC2 + j) * Bp + b], 0.f);
          xy2[(size_t)(u0 + j) * Bp + b] = rnd(y);
        }
      }
      __syncthreads();
    }
    WRNN_BARRIER();
    // ---- phase E: fc3 + sampling ---------------------------------------------------------------------
    if (p.mode == WRNN_MODE_MOL) {
      for (int tile = cta; tile < ntiles; tile += P) {      // fold tiles are owned round-robin
        const int b0 = tile * FT;
        load_xch_tile(xy2, b0);
        __syncthreads();
        gemv_tile<T, F3ROWS>(reinterpret_cast<const T*>(p.f3t), H, act, outs);
        __syncthreads();
        if (tid < FT) {
          const int f = tid, b = b0 + f;
          if (b < B) {
            auto lget = [&](int i) { return out_row<F3ROWS>(outs, i, f) + __ldg(p.b3 + i); };
            float s;
            if constexpr (SCORE) {
              s = __ldg(p.x_force + (size_t)t * B + b);
              p.nll[(size_t)t * B + b] = mol_nll(lget, s);
            } else if (p.uniforms) {
              const float* ur = p.uniforms + (size_t)t * 11 * B;
              s = mol_sample(lget, [&](int i) { return i < 10 ? __ldg(ur + b * 10 + i) : __ldg(ur + 10 * B + b); });
            } else {
              const FoldPhilox k = fold_philox(p.keys, b, p.seg_first, p.seed);
              const unsigned g = k.fold, k0 = k.k0, k1 = k.k1;
              const unsigned o0 = (unsigned)p.offset;
              const Philox4 r0 = philox4x32_10((unsigned)t, g, 0u, o0, k0, k1);
              const Philox4 r1 = philox4x32_10((unsigned)t, g, 1u, o0, k0, k1);
              const Philox4 r2 = philox4x32_10((unsigned)t, g, 2u, o0, k0, k1);
              const unsigned rv[12] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
              s = mol_sample(lget, [&](int i) { return u_ref_range(rv[i]); });
            }
            p.xs[b] = s;
            if (!SCORE) p.out[(size_t)b * p.out_pitch + t] = s;
            if (p.logits_out)
              for (int i = 0; i < 30; ++i) p.logits_out[((size_t)t * B + b) * 30 + i] = lget(i);
          }
        }
        __syncthreads();
      }
      WRNN_BARRIER();
    } else {
      // RAW: fc3 has n_classes == 4*P rows; every CTA computes its 4 logits for all folds
      for (int tile = 0; tile < ntiles; ++tile) {
        const int b0 = tile * FT;
        load_xch_tile(xy2, b0);
        __syncthreads();
        gemv_tile<T, S4ROWS>(wS4, H, act, outs);
        __syncthreads();
        if (tid < U * FT) {
          const int f = tid & 31, j = tid >> 5, b = b0 + f;
          if (b < B) p.xlog[(size_t)(u0 + j) * Bp + b] = out_row<S4ROWS>(outs, j, f) + b3s[j];
        }
        __syncthreads();
      }
      WRNN_BARRIER();
      // softmax + Categorical.sample() == argmax(p / e), e ~ Exp(1)  (:232-235)
      const int NC = p.n_classes;
      for (int tile = cta; tile < ntiles; tile += P) {
        const int b0 = tile * FT;
        for (int f = warp; f < FT; f += NT / 32) {
          const int b = b0 + f;
          if (b >= B) continue;
          float mx = -INFINITY;
          for (int i = lane; i < NC; i += 32) mx = fmaxf(mx, __ldcg(p.xlog + (size_t)i * Bp + b));
          for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
          float sum = 0.f;
          for (int i = lane; i < NC; i += 32) sum += expf(__ldcg(p.xlog + (size_t)i * Bp + b) - mx);
          for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
          if constexpr (SCORE) {
            const float y = __ldg(p.x_force + (size_t)t * B + b);
            if (p.logits_out)
              for (int i = lane; i < NC; i += 32) p.logits_out[((size_t)t * B + b) * NC + i] = __ldcg(p.xlog + (size_t)i * Bp + b);
            if (lane == 0) {
              p.nll[(size_t)t * B + b] = raw_nll(mx, sum, __ldcg(p.xlog + (size_t)raw_label(y, NC) * Bp + b));
              p.xs[b] = y;
            }
            continue;
          }
          float bestq = -1.f; int besti = 0x7fffffff;
          const FoldPhilox key = p.expo ? FoldPhilox{0u, 0u, 0u} : fold_philox(p.keys, b, p.seg_first, p.seed);
          for (int i = lane; i < NC; i += 32) {
            const float l = __ldcg(p.xlog + (size_t)i * Bp + b);
            const float pr = expf(l - mx) / sum;
            float e;
            if (p.expo) e = __ldg(p.expo + ((size_t)t * B + b) * NC + i);
            else {
              const Philox4 r = philox4x32_10((unsigned)t, key.fold, 16u + (unsigned)(i >> 2), (unsigned)p.offset, key.k0, key.k1);
              const unsigned rv[4] = {r.x, r.y, r.z, r.w};
              e = -logf(u01_open(rv[i & 3]));
            }
            const float q = pr / e;
            if (q > bestq) { bestq = q; besti = i; }
            if (p.logits_out) p.logits_out[((size_t)t * B + b) * NC + i] = l;
          }
          for (int o = 16; o; o >>= 1) {
            const float oq = __shfl_xor_sync(0xffffffffu, bestq, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (oq > bestq || (oq == bestq && oi < besti)) { bestq = oq; besti = oi; }
          }
          if (lane == 0) {
            const float s = 2.0f * (float)besti / ((float)NC - 1.0f) - 1.0f;     // :235
            p.xs[b] = s;
            p.out[(size_t)b * p.out_pitch + t] = s;
          }
        }
      }
      WRNN_BARRIER();
    }
  }
#undef WRNN_BARRIER
}

// --------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------
struct HostBf16 { uint16_t bits; };
struct HostF16 { uint16_t bits; };
template <typename T> T cvt(double v);
template <> float cvt<float>(double v) { return (float)v; }
template <> HostBf16 cvt<HostBf16>(double v) { return HostBf16{f2bf((float)v)}; }
template <> HostF16 cvt<HostF16>(double v) { return HostF16{f2h((float)v)}; }

template <typename T>   // T = float, HostBf16 or HostF16
void pack_blob(const HostWeights& w, const Folded& f, std::vector<unsigned char>& blob, size_t& stride,
               std::vector<unsigned char>& f3t, int n_classes, int mode) {
  stride = (MAT_ELEMS * sizeof(T) + NVEC * sizeof(float) + 15) / 16 * 16;
  blob.assign(stride * P, 0);
  CtaSlice s;
  for (int c = 0; c < P; ++c) {
    slice_for_cta(w, f, c, U, s);
    T* m = reinterpret_cast<T*>(blob.data() + stride * c);
    T* q = m; T* s1 = q + CDIM * QROWS; T* s2 = s1 + H * S1ROWS; T* s3 = s2 + H * S2ROWS; T* s4 = s3 + H * S3ROWS;
    float* fv = reinterpret_cast<float*>(s4 + H * S4ROWS);
    for (int k = 0; k < CDIM; ++k) for (int r = 0; r < 8 * U; ++r) q[k * QROWS + r] = cvt<T>(s.Q[(size_t)r * CDIM + k]);
    for (int k = 0; k < H; ++k) {
      for (int r = 0; r < 7 * U; ++r) s1[k * S1ROWS + r] = cvt<T>(s.S1[(size_t)r * H + k]);
      for (int r = 0; r < 4 * U; ++r) s2[k * S2ROWS + r] = cvt<T>(s.S2[(size_t)r * H + k]);
      for (int r = 0; r < U; ++r) s3[k * S3ROWS + r] = cvt<T>(s.S3[(size_t)r * H + k]);
      if (mode == WRNN_MODE_RAW)
        for (int r = 0; r < U; ++r) s4[k * S4ROWS + r] = cvt<T>(w.f3w[(size_t)(c * U + r) * H + k]);
    }
    for (int r = 0; r < 8 * U; ++r) { fv[r] = s.qk[r]; fv[32 + r] = s.vq[r]; }
    for (int r = 0; r < 3 * U; ++r) { fv[64 + r] = s.b1h[r]; fv[76 + r] = s.b2h[r]; }
    if (mode == WRNN_MODE_RAW) for (int r = 0; r < U; ++r) fv[88 + r] = w.f3b[c * U + r];
  }
  f3t.assign((size_t)H * F3ROWS * sizeof(T), 0);
  if (mode == WRNN_MODE_MOL) {
    T* t3 = reinterpret_cast<T*>(f3t.data());
    for (int k = 0; k < H; ++k) for (int r = 0; r < n_classes; ++r) t3[k * F3ROWS + r] = cvt<T>(w.f3w[(size_t)r * H + k]);
  }
}

class SimtEngine : public Engine {
 public:
  ~SimtEngine() override {
    cudaSetDevice(device);
    cudaFree(d_blob_); cudaFree(d_f3t_); cudaFree(d_b3_); cudaFree(d_scratch_); cudaFree(d_sync_);
  }
  const char* name() const override {
    return cfg.precision == WRNN_PREC_FP32 ? "simt-fp32" : cfg.precision == WRNN_PREC_BF16 ? "simt-bf16" : "simt-fp16";
  }
  const char* live_refusal() const override {
    return "live vocoding runs on the persistent engine only: the SIMT engine's step has not been timed against real time";
  }
  template <bool SCORE> const void* kernel_of() const {
    return cfg.precision == WRNN_PREC_FP32   ? (const void*)wrnn_simt_kernel<float, SCORE>
           : cfg.precision == WRNN_PREC_BF16 ? (const void*)wrnn_simt_kernel<__nv_bfloat16, SCORE>
                                             : (const void*)wrnn_simt_kernel<__half, SCORE>;
  }
  const void* kernel(bool score) const { return score ? kernel_of<true>() : kernel_of<false>(); }
  int grid_ctas() const override { return P; }

  int init(const HostWeights& w) {
    Folded f; fold(w, f);
    std::vector<unsigned char> blob, f3t;
    if (cfg.precision == WRNN_PREC_FP32) pack_blob<float>(w, f, blob, stride_, f3t, cfg.n_classes, cfg.mode);
    else if (cfg.precision == WRNN_PREC_BF16) pack_blob<HostBf16>(w, f, blob, stride_, f3t, cfg.n_classes, cfg.mode);
    else pack_blob<HostF16>(w, f, blob, stride_, f3t, cfg.n_classes, cfg.mode);
    WRNN_CUDA_OK(cudaMalloc(&d_blob_, blob.size()));
    WRNN_CUDA_OK(cudaMemcpy(d_blob_, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    WRNN_CUDA_OK(cudaMalloc(&d_f3t_, f3t.size()));
    WRNN_CUDA_OK(cudaMemcpy(d_f3t_, f3t.data(), f3t.size(), cudaMemcpyHostToDevice));
    std::vector<float> b3(64, 0.f);
    for (int i = 0; i < cfg.n_classes && i < 64; ++i) b3[i] = w.f3b[i];
    WRNN_CUDA_OK(cudaMalloc(&d_b3_, b3.size() * 4));
    WRNN_CUDA_OK(cudaMemcpy(d_b3_, b3.data(), b3.size() * 4, cudaMemcpyHostToDevice));
    WRNN_CUDA_OK(cudaMalloc(&d_sync_, 64));
    WRNN_CUDA_OK(cudaMemset(d_sync_, 0, 64));
    const size_t elem = cfg.precision == WRNN_PREC_FP32 ? 4 : 2;
    smem_bytes_ = MAT_ELEMS * elem + NVEC * 4 + (size_t)H * AP * 4 + 8 * 4 * AP * 4;
    WRNN_CUDA_OK(cudaFuncSetAttribute(kernel(false), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes_));
    WRNN_CUDA_OK(cudaFuncSetAttribute(kernel(true), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes_));
    int n_sm = 0;
    WRNN_CUDA_OK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
    if (n_sm < P) { set_error("SIMT engine needs >= 128 SMs for its co-resident weight shards"); return WRNN_E_NO_DEVICE; }
    return WRNN_OK;
  }

  bool supports(const wrnn_job& job) const override { return job.mel_frames == nullptr; }   // upsampled streams only

  int generate(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys) override { return run(job, stream, keys, nullptr); }
  int score(const wrnn_job& job, float* nll, cudaStream_t stream, const FoldKey* keys) override { return run(job, stream, keys, nll); }

  // nll != NULL: scoring (the loss of x_force[t] in the sampler's place)
  int run(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys, float* nll) {
    if (job.mel_frames) { set_error("the SIMT engine takes the upsampled conditioning streams (mels_up / aux)"); return WRNN_E_INVALID; }
    if (job.uniforms_ready) { set_error("the SIMT engine needs all draws resident (no uniforms_ready)"); return WRNN_E_INVALID; }
    WRNN_CUDA_OK(cudaSetDevice(device));
    const int Bp = (job.n_seg + FT - 1) / FT * FT;
    const size_t need = ((size_t)4 * H * Bp + Bp + (size_t)P * NSTATE * Bp + (size_t)cfg.n_classes * Bp) * sizeof(float);
    if (need > scratch_bytes_) {
      WRNN_CUDA_OK(cudaStreamSynchronize(stream));
      cudaFree(d_scratch_); d_scratch_ = nullptr; scratch_bytes_ = 0;
      WRNN_CUDA_OK(cudaMalloc(&d_scratch_, need));
      scratch_bytes_ = need;
    }
    WRNN_CUDA_OK(cudaMemsetAsync(d_sync_, 0, 64, stream));
    WRNN_CUDA_OK(cudaMemsetAsync(d_scratch_, 0, need, stream));
    SimtParams p{};
    p.blob = static_cast<const unsigned char*>(d_blob_); p.blob_stride = stride_;
    p.f3t = d_f3t_; p.b3 = static_cast<const float*>(d_b3_);
    p.mels_up = job.mels_up; p.aux = job.aux; p.L = job.L; p.seg_stride = job.seg_stride;
    p.n_seg = job.n_seg; p.seg_len = job.seg_len; p.seg_first = job.seg_first;
    p.steps = job.steps > 0 ? job.steps : job.seg_len; p.Bp = Bp; p.out_pitch = p.steps;
    p.n_classes = cfg.n_classes; p.mode = cfg.mode;
    p.uniforms = job.uniforms; p.expo = job.expo; p.seed = job.philox_seed; p.offset = job.philox_offset;
    p.out = job.out; p.x_force = job.x_force; p.logits_out = job.logits_out;
    p.fold_row0 = reinterpret_cast<const long long*>(job.fold_row0); p.fold_row_end = reinterpret_cast<const long long*>(job.fold_row_end);
    p.keys = keys;
    float* s = static_cast<float*>(d_scratch_);
    p.xch = s; s += (size_t)4 * H * Bp;
    p.xs = s; s += Bp;
    p.state = s; s += (size_t)P * NSTATE * Bp;
    p.xlog = s;
    p.counter = static_cast<unsigned*>(d_sync_); p.abort_flag = reinterpret_cast<int*>(static_cast<unsigned*>(d_sync_) + 8);
    p.nll = nll;
    void* args[] = {&p};
    const void* fn = kernel(nll != nullptr);
    // cooperative launch: all P CTAs must be co-resident for the spin barriers to be safe
    WRNN_CUDA_OK(cudaLaunchCooperativeKernel(fn, dim3(P), dim3(NT), args, smem_bytes_, stream));
    ++launches;
    return WRNN_OK;
  }

  int check() override {
    int flags[16];
    WRNN_CUDA_OK(cudaSetDevice(device));
    WRNN_CUDA_OK(cudaMemcpy(flags, d_sync_, 64, cudaMemcpyDeviceToHost));
    if (flags[8] != 0) { set_error("persistent kernel aborted on its grid-barrier watchdog"); return WRNN_E_WATCHDOG; }
    return WRNN_OK;
  }

 private:
  void *d_blob_ = nullptr, *d_f3t_ = nullptr, *d_b3_ = nullptr, *d_scratch_ = nullptr, *d_sync_ = nullptr;
  size_t stride_ = 0, scratch_bytes_ = 0, smem_bytes_ = 0;
};

}  // namespace

int make_simt_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out) {
  if (cfg.mode == WRNN_MODE_RAW && cfg.n_classes != 4 * P) {
    set_error("SIMT engine: RAW head supports n_classes == 512 (bits = 9) only");
    return WRNN_E_INVALID;
  }
  if (cfg.mode == WRNN_MODE_MOL && cfg.n_classes != 30) { set_error("MOL head needs n_classes == 30"); return WRNN_E_INVALID; }
  SimtEngine* e = new SimtEngine();
  e->cfg = cfg; e->device = device;
  const int rc = e->init(w);
  if (rc != WRNN_OK) { delete e; return rc; }
  *out = e;
  return WRNN_OK;
}

}  // namespace wrnn
