// wrnn_device.cuh -- device helpers shared by the engines: memory-ordering primitives,
// the grid barrier with a watchdog, Philox4x32-10, and the two samplers
// (reference utils/distribution.py:87-123 and models/fatchord_version.py:231-237).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wrnn_fold.h"

namespace wrnn {

// -------------------------------------------------------------------------------------
// memory ordering
// -------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add_u32(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_relaxed_s32(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Spin budget before a waiter declares the grid dead and raises the abort flag.  SM clock
// is <= ~2 GHz, so 2^32 cycles is > 2 s: far beyond any legitimate wait (a step is ~10 us)
// and far below gpurun's own limits, so a protocol bug ends in an error, not a hung box.
constexpr long long kWatchdogCycles = 1ll << 32;

// Grid-wide barrier over a monotonically increasing counter: the k-th barrier of a launch
// waits for counter >= k * gridDim.x.  Returns false when the launch must be abandoned.
// The comparison is wrap-safe (signed distance): the 32-bit counter may roll over on very long unbatched jobs
// (6 barriers x 128 CTAs per step wrap after ~5.6 M steps); CTAs are never more than one barrier apart, so the
// distance between counter and target is always far below 2^31.
__device__ __forceinline__ bool counter_behind(unsigned value, unsigned target) { return (int)(value - target) < 0; }
__device__ __forceinline__ bool grid_barrier(unsigned* counter, unsigned target, int* abort_flag) {
  __shared__ int s_ok;
  __syncthreads();
  if (threadIdx.x == 0) {
    red_release_add_u32(counter, 1u);   // release: orders this CTA's prior writes (made visible to
                                        // thread 0 by the bar.sync above) before the increment
    int ok = 1;
    const long long t0 = clock64();
    while (counter_behind(ld_acquire_u32(counter), target)) {
      if (clock64() - t0 > kWatchdogCycles || ld_relaxed_s32(abort_flag) != 0) {
        atomicExch(abort_flag, 1);
        ok = 0;
        break;
      }
    }
    s_ok = ok;
  }
  __syncthreads();
  return s_ok != 0;
}

// -------------------------------------------------------------------------------------
// numerics
// -------------------------------------------------------------------------------------
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
// RNE to IEEE half, saturating to +-65504 (cvt.rn.satfinite.f16.f32), back to float
__device__ __forceinline__ float f16_round(float x) {
  unsigned short h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
  return __half2float(__ushort_as_half(h));
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// PyTorch GRUCell update for one hidden unit (gate order r, z, n).
__device__ __forceinline__ float gru_unit(float gi_r, float gi_z, float gi_n, float gh_r, float gh_z,
                                          float gh_n, float h) {
  const float r = sigmoidf_(gi_r + gh_r);
  const float z = sigmoidf_(gi_z + gh_z);
  const float n = tanhf(gi_n + r * gh_n);
  return (1.0f - z) * n + z * h;
}

// float32 / float64 arithmetic rounded step by step, as numpy evaluates it (no fused multiply-add on the device); the
// host hooks of wrnn_mel.cu and wrnn_resample.cu run the same source on the CPU
__host__ __device__ inline float fmul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double dmul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double dadd_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// -------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011), counter-based: (seed) x (step, fold, lane, offset)
// -------------------------------------------------------------------------------------
struct Philox4 { unsigned x, y, z, w; };
__host__ __device__ __forceinline__ unsigned umulhi32(unsigned a, unsigned b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (unsigned)(((unsigned long long)a * b) >> 32);
#endif
}
// host and device (wrnn_debug_griffinlim runs the Griffin-Lim phase draws on the host)
__host__ __device__ __forceinline__ Philox4 philox4x32_10(unsigned c0, unsigned c1, unsigned c2, unsigned c3,
                                                           unsigned k0, unsigned k1) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int i = 0; i < 10; ++i) {
    const unsigned hi0 = umulhi32(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned hi1 = umulhi32(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const unsigned n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
// 24 random bits -> [2^-25, 1].  Closed at 1: above 2^23 the float sum (m + 0.5f) rounds to nearest even, so
// x >> 8 == 0xffffff gives exactly 1.0f (once per 2^24 words).
__host__ __device__ __forceinline__ float u01(unsigned x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// u01 clamped into the open interval (0, 1): the RAW head's Exp(1) draws -logf(u) must be > 0 (at u = 1 they were -0.0,
// which forced the class in the persistent engine and excluded it in the SIMT engine).  Every other word maps as u01.
__device__ __forceinline__ float u01_open(unsigned x) { return fminf(u01(x), 0x1.fffffep-1f); }
// the reference's uniform_(1e-5, 1 - 1e-5): rand*(to-from)+from, contracted to one FFMA.  u01 = 1 maps to
// 1 - 1e-5 (rounded), inside the reference's range, so the MoL draws keep the closed u01.
__device__ __forceinline__ float u_ref_range(unsigned x) { return u01(x) * (1.0f - 2e-5f) + 1e-5f; }

// Philox counter fold and key words of job fold f: the per-fold table when present (one 16-byte read-only load),
// else (seg_first + f, philox_seed).
struct FoldPhilox { unsigned fold, k0, k1; };
__device__ __forceinline__ FoldPhilox fold_philox(const FoldKey* keys, int f, int seg_first, unsigned long long seed) {
  if (keys) {
    const ulonglong2 k = __ldg(reinterpret_cast<const ulonglong2*>(keys + f));
    return FoldPhilox{(unsigned)k.y, (unsigned)k.x, (unsigned)(k.x >> 32)};
  }
  return FoldPhilox{(unsigned)(seg_first + f), (unsigned)seed, (unsigned)(seed >> 32)};
}
// the key of a live-session slot: its occupant's seed, counter fold 0
__device__ __forceinline__ FoldPhilox slot_philox(unsigned long long seed) {
  return FoldPhilox{0u, (unsigned)seed, (unsigned)(seed >> 32)};
}
// The in-kernel draws of one step of a fold, the same on every tensor-core engine.  MoL: words 0-9 (mixture) and 10
// (logistic) of Philox blocks 0-2 at counter (step, fold, block, offset), each mapped by u_ref_range.
__device__ __forceinline__ void mol_uniforms(const FoldPhilox& k, unsigned step, unsigned offset, float (&ur)[11]) {
  const unsigned g = k.fold, k0 = k.k0, k1 = k.k1, o0 = offset;
  const Philox4 r0 = philox4x32_10(step, g, 0u, o0, k0, k1), r1 = philox4x32_10(step, g, 1u, o0, k0, k1),
                r2 = philox4x32_10(step, g, 2u, o0, k0, k1);
  ur[0] = u_ref_range(r0.x); ur[1] = u_ref_range(r0.y); ur[2] = u_ref_range(r0.z); ur[3] = u_ref_range(r0.w);
  ur[4] = u_ref_range(r1.x); ur[5] = u_ref_range(r1.y); ur[6] = u_ref_range(r1.z); ur[7] = u_ref_range(r1.w);
  ur[8] = u_ref_range(r2.x); ur[9] = u_ref_range(r2.y); ur[10] = u_ref_range(r2.z);
}
// RAW: class c draws Exp(1) from word c % 4 of block 16 + c / 4.
__device__ __forceinline__ Philox4 raw_block(const FoldPhilox& k, unsigned step, unsigned cls_block, unsigned offset) {
  return philox4x32_10(step, k.fold, 16u + cls_block, offset, k.k0, k.k1);
}
__device__ __forceinline__ float raw_exp(const Philox4& r, unsigned word) {
  return -logf(u01_open(word == 0 ? r.x : word == 1 ? r.y : word == 2 ? r.z : r.w));
}

// -------------------------------------------------------------------------------------
// samplers
// -------------------------------------------------------------------------------------
// utils/distribution.py:99-121.  l: 30 logits = [10 mixture | 10 means | 10 log-scales].
// `lget(i)` fetches logit i, `uget(i)` uniform i (0..9 mixture draws, 10 = logistic draw).
template <typename LGet, typename UGet>
__device__ __forceinline__ float mol_sample(LGet lget, UGet uget) {
  int best = 0;
  float bestv = -INFINITY;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const float g = lget(k) - logf(-logf(uget(k)));            // :107
    if (g > bestv) { bestv = g; best = k; }                     // :108 first maximum wins
  }
  const float mean = lget(10 + best);                           // :113
  const float log_scale = fmaxf(lget(20 + best), -32.23619130191664f);   // :114 log(1e-14)
  const float u = uget(10);
  float x = mean + expf(log_scale) * (logf(u) - logf(1.0f - u));         // :119
  return fminf(fmaxf(x, -1.0f), 1.0f);                          // :121
}

// -------------------------------------------------------------------------------------
// scoring: the reference's training loss per sample, in nats (train_wavernn.py:83).  Accurate expf / logf / log1pf
// (never the SFU intrinsics) in fp32, in the reference's order, so that the value is a measurement of the logits.
// -------------------------------------------------------------------------------------
// torch.sigmoid and F.softplus (beta 1, threshold 20) as torch evaluates them in fp32
__device__ __forceinline__ float ref_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float ref_softplus(float x) { return x > 20.0f ? x : log1pf(expf(x)); }

// discretized_mix_logistic_loss(reduce=False) of utils/distribution.py:16-84 for target y, num_classes = 65536 and
// log_scale_min = log(1e-14).  `lget(i)` fetches logit i of [10 mixture | 10 means | 10 log-scales].  The reference
// blends its branches with 0/1 masks; every branch value is finite, so the blend is the selection made here.
template <typename LGet>
__device__ __forceinline__ float mol_nll(LGet lget, float y) {
  const float half_bin = (float)(1.0 / 65535.0);                 // 1. / (num_classes - 1), a float32 scalar
  const float log_half_classes = 10.397192449493701f;            // np.log((num_classes - 1) / 2)
  float mx = lget(0);
#pragma unroll
  for (int k = 1; k < 10; ++k) mx = fmaxf(mx, lget(k));
  float se = 0.f;
#pragma unroll
  for (int k = 0; k < 10; ++k) se += expf(lget(k) - mx);
  const float lse_pi = logf(se);                                 // F.log_softmax(logit_probs): (x - max) - log(sum)
  float lp[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const float log_scale = fmaxf(lget(20 + k), -32.23619130191664f);
    const float centered = y - lget(10 + k);
    const float inv_stdv = expf(-log_scale);
    const float plus_in = inv_stdv * (centered + half_bin);
    const float min_in = inv_stdv * (centered - half_bin);
    const float cdf_delta = ref_sigmoid(plus_in) - ref_sigmoid(min_in);
    float v;
    if (y < -0.999f) v = plus_in - ref_softplus(plus_in);                       // log_cdf_plus
    else if (y > 0.999f) v = -ref_softplus(min_in);                             // log_one_minus_cdf_min
    else if (cdf_delta > 1e-5f) v = logf(fmaxf(cdf_delta, 1e-12f));
    else {
      const float mid_in = inv_stdv * centered;
      v = __fsub_rn(__fsub_rn(mid_in, log_scale), __fmul_rn(2.0f, ref_softplus(mid_in))) - log_half_classes;   // log_pdf_mid
    }
    lp[k] = v + ((lget(k) - mx) - lse_pi);
  }
  float m = lp[0];
#pragma unroll
  for (int k = 1; k < 10; ++k) m = fmaxf(m, lp[k]);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 10; ++k) s += expf(lp[k] - m);
  return -(m + logf(s));                                         // -log_sum_exp(log_probs)
}

// F.cross_entropy of one sample from the logits' maximum, the sum of exp(l - max) and the target's logit: the negated
// log_softmax entry, -((l_y - max) - log(sum)).
__device__ __forceinline__ float raw_nll(float mx, float sum, float l_y) { return -((l_y - mx) - logf(sum)); }

// RAW head: the class of a target sample y as the reference labels it (the inverse of label_2_float,
// utils/dataset.py:88): rint((y + 1) (n_classes - 1) / 2), clamped to [0, n_classes - 1].
__device__ __forceinline__ int raw_label(float y, int n_classes) {
  const float v = rintf(__fmul_rn(__fmul_rn(y + 1.0f, (float)(n_classes - 1)), 0.5f));
  return (int)fminf(fmaxf(v, 0.0f), (float)(n_classes - 1));
}

}  // namespace wrnn
