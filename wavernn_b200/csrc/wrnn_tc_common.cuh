// wrnn_tc_common.cuh -- PTX wrappers (wgmma, TMA, mbarrier) and epilogue math shared by the tensor-core engines
// (wrnn_tc.cu, wrnn_stream.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "wrnn_device.cuh"

namespace wrnn {
namespace tc {

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  // SM90 shared-memory matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout [62,64) = 0
  // (no swizzle: 8-row x 16-byte core matrices, contiguous 128 B each), K-major.  LBO = byte distance of the two core
  // matrices of one K = 16 step, SBO = byte distance of consecutive 8-row groups.
  return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) | ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// D[64, N] (+)= A[64, 16] * B[N, 16]^T, both operands K-major in shared memory, fp32 accumulators in registers
// (m64nNk16 fragment: thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8j + 2*(t%4) (+1)).
// Executed by all 128 threads of a warpgroup; scale_d == 0 overwrites D.  FMT 0 = fp16, 1 = bf16 operands.
template <int N, int FMT> __device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_ss<8, 0>(float* d, uint64_t da, uint64_t db, uint32_t s) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "l"(da), "l"(db), "r"(s) : "memory");
}
template <> __device__ __forceinline__ void wgmma_ss<8, 1>(float* d, uint64_t da, uint64_t db, uint32_t s) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "l"(da), "l"(db), "r"(s) : "memory");
}
#define WRNN_WGMMA_N16(FMT, TY)                                                                                              \
  template <> __device__ __forceinline__ void wgmma_ss<16, FMT>(float* d, uint64_t da, uint64_t db, uint32_t s) {          \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"                                                      \
                 "wgmma.mma_async.sync.aligned.m64n16k16" TY " {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n" \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])           \
                 : "l"(da), "l"(db), "r"(s) : "memory");                                                                     \
  }
#define WRNN_WGMMA_N32(FMT, TY)                                                                                              \
  template <> __device__ __forceinline__ void wgmma_ss<32, FMT>(float* d, uint64_t da, uint64_t db, uint32_t s) {          \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                                      \
                 "wgmma.mma_async.sync.aligned.m64n32k16" TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "  \
                 "%14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"                                                                 \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),          \
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])    \
                 : "l"(da), "l"(db), "r"(s) : "memory");                                                                     \
  }
WRNN_WGMMA_N16(0, ".f32.f16.f16")
WRNN_WGMMA_N16(1, ".f32.bf16.bf16")
WRNN_WGMMA_N32(0, ".f32.f16.f16")
WRNN_WGMMA_N32(1, ".f32.bf16.bf16")
#undef WRNN_WGMMA_N16
#undef WRNN_WGMMA_N32

// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (whole warp, one lane elected)
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t"
               "@e mbarrier.arrive.expect_tx.shared::cta.b64 _, [%3], %2;\n\t"
               "@e cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}\n"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void proxy_fence_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void proxy_fence_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory"); }

// bounded waits: a protocol bug must end in an error code, never in a hung GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* abort_flag) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  unsigned spins = 0;
  while (!mbar_try(bar, parity)) {
    if ((++spins & 1023u) == 0) {                       // rarely: has another wait already given up?
      if (ld_relaxed_s32(abort_flag) != 0) return;
      if (clock64() - t0 > kWatchdogCycles) { atomicExch(abort_flag, 2); return; }
    }
  }
}
__device__ __forceinline__ void counter_wait(const unsigned* ctr, unsigned target, int* abort_flag) {
  if (!counter_behind(ld_acquire_u32(ctr), target)) return;          // wrap-safe, see grid_barrier
  const long long t0 = clock64();
  unsigned spins = 0;
  while (counter_behind(ld_acquire_u32(ctr), target)) {
    // watchdog / abort check (a second L2 load) only every 64th poll.  Measured: no change of the step (12.10 us either
    // way) -- the exchange is bound by when the last of the 128 producers arrives, not by the polling period.
    if ((++spins & 63u) == 0 && (clock64() - t0 > kWatchdogCycles || ld_relaxed_s32(abort_flag) != 0)) { atomicExch(abort_flag, 1); return; }
  }
}

// Streamed draws (wrnn_job::uniforms_ready): returns the number of valid rows once it exceeds `need - 1`
// (0xffffffff if the job is being abandoned, so the caller stops asking).
__device__ __forceinline__ unsigned rows_wait(const unsigned* ready, unsigned need, int* abort_flag) {
  unsigned v = ld_acquire_u32(ready);
  if (v >= need) return v;
  const long long t0 = clock64();
  while ((v = ld_acquire_u32(ready)) < need) {
    if (ld_relaxed_s32(abort_flag) != 0) return 0xffffffffu;
    if (clock64() - t0 > kWatchdogCycles) { atomicExch(abort_flag, 1); return 0xffffffffu; }
    __nanosleep(200);
  }
  return v;
}

template <int FMT> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<0>(float a, float b) {      // fp16, RNE, saturating
  uint32_t r;
  asm("{\n\t.reg .b16 lo, hi;\n\tcvt.rn.satfinite.f16.f32 lo, %1;\n\tcvt.rn.satfinite.f16.f32 hi, %2;\n\tmov.b32 %0, {lo, hi};\n\t}\n"
      : "=r"(r) : "f"(a), "f"(b));
  return r;
}
template <> __device__ __forceinline__ uint32_t pack2<1>(float a, float b) {      // bf16, RNE
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}

// Epilogue transcendentals on the SFU (ex2/rcp/lg2 approx, rel. error ~1e-6 -- two orders below the
// fp16 operand rounding of the contractions).  The strict SIMT engine keeps the libm versions.
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.0f - __fdividef(2.0f, __expf(2.0f * x) + 1.0f); }
__device__ __forceinline__ float gru_unit_fast(float gi_r, float gi_z, float gi_n, float gh_r, float gh_z, float gh_n, float h) {
  const float r = fast_sigmoid(gi_r + gh_r);
  const float z = fast_sigmoid(gi_z + gh_z);
  const float n = fast_tanh(gi_n + r * gh_n);
  return (1.0f - z) * n + z * h;
}
// utils/distribution.py:99-121 on SFU logs/exp
__device__ __forceinline__ float mol_sample_fast(const float* lg, const float* u) {
  int best = 0;
  float bestv = -INFINITY;
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    const float g = lg[k] - __logf(-__logf(u[k]));
    if (g > bestv) { bestv = g; best = k; }
  }
  float mean = lg[10], ls = lg[20];
#pragma unroll
  for (int k = 1; k < 10; ++k) { if (best == k) { mean = lg[10 + k]; ls = lg[20 + k]; } }
  ls = fmaxf(ls, -32.23619130191664f);
  const float x = mean + __expf(ls) * (__logf(u[10]) - __logf(1.0f - u[10]));
  return fminf(fmaxf(x, -1.0f), 1.0f);
}


// K-major no-swizzle operand image (host side): element (r, k) at (r/8)*(K/8)*64 + (k/8)*64 + (r%8)*8 + k%8
inline size_t img_index(int r, int k, int K) { return (size_t)(r / 8) * (K / 8) * 64 + (size_t)(k / 8) * 64 + (r % 8) * 8 + (k % 8); }

}  // namespace tc
}  // namespace wrnn
