// wrnn_stream.cu -- STREAM engine: the throughput form of the generate() loop (reference models/fatchord_version.py:
// 201-241 + utils/distribution.py:87-123) for jobs with many folds (BASELINE configs[3], configs[4]).
//
// wrnn_tc.cu keeps the weights stationary (row-sharded over 128 SMs) and pays four all-to-all exchanges of the
// activations per step: right for 19 folds, wrong for 4096 (every exchange broadcasts the whole tile's activations to
// 128 SMs through L2).  Here the ACTIVATIONS are stationary: one CTA owns NF folds (16 or 32) for the whole sequence,
// runs every layer for them, and streams the 7.4 MB of fp16 weights from L2 each step through a shared-memory ring of
// TMA bulk copies -- no inter-SM synchronisation at all, one independent CTA per fold tile, any number of tiles.
// The step is the static program of wrnn_stream_plan.h (chunk list with accumulator / operand / barrier fields).
//
// Swap-AB wgmma: D[128 weight rows, NF folds] (+)= W[128, 16] * act[NF, 16]^T, fp32 accumulators in registers.  Two
// consumer warpgroups split every 128-row chunk (rows 0-63 / 64-127) and walk the program grouped by (phase, unit
// block): each holds the four accumulators of the current group (r / z / in / hn of a GRU block, or the four K
// partials of an fc block) and runs the group's epilogue itself when its last chunk is done.  The r / z / n
// pre-activations of a unit sit in the same fragment position of different accumulators, so the gate math is
// thread-local.  The fp32 hidden state lives in L2-resident global scratch ([2][512][NF] per tile); the fp16 operand
// images of h1', h2', y1, y2 live in shared memory.
//
// Warp roles (320 threads):
//   warps 0-7  consumers : two warpgroups; per chunk: operand readiness, ring slot, wgmma, slot release; epilogues
//   warp 8     producer  : walks the chunk list, one cp.async.bulk per chunk into the ring (full/empty mbarriers)
//   warp 9     staging   : conditioning row of step t+1 for the NF folds (stream or frame-rate form) -> fp16 image
//
// Cluster form (template CL = 4; jobs whose clusters are co-resident): a tile belongs to a thread-block cluster of four
// CTAs.  CTA r runs the program of unit block r of every layer (a quarter of the weight stream and of the MMAs; MoL:
// fc3 + sampling in rank 0, which hands the sample to its peers; RAW: fc3 block r in rank r, whose best (score, class)
// goes into every rank's candidate table, and every rank reduces the four), keeps all four K = 512 operand images, and pushes the block
// it has just computed into the peers' images with cp.async.bulk.shared::cluster.shared::cta (complete_tx on the PEER's
// readiness barrier, arrive.expect_tx by the sender), so that a peer's block arrives exactly like a TMA load.  Same MMAs
// in the same order: results are bit-identical to the one-CTA form.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "wrnn_device.cuh"
#include "wrnn_engine.h"
#include "wrnn_stream_plan.h"
#include "wrnn_tc_common.cuh"

namespace wrnn {
namespace {
using namespace tc;
using namespace stream;

constexpr int NT = 320;
constexpr int N_CONSUMERS = 256;             // warps 0-7
constexpr int PRODUCER_WARP = 8, STAGING_WARP = 9;
constexpr int KQ = CDIM / 8;                 // 26 16-byte chunks per conditioning row
constexpr int SBO_Q = KQ * 128;              // 3328: stride between 8-fold groups of the conditioning image
constexpr int SBO_H = (H / 8) * 128;         // 8192: same for the K = 512 images
constexpr int NBAR = 48;
constexpr int MAX_STAGES = 9;               // ring slots (one chunk each)

// RAW: the 9-bit head's classes (fc3 in four unit blocks of 128)
constexpr int NCLS_RAW = 512;

template <int NF, bool RAW = false> struct Smem {
  static constexpr int GROUPS = NF / 8;
  static constexpr int ACT = GROUPS * SBO_H;                 // one K = 512 activation image
  static constexpr int COND = GROUPS * SBO_Q;                // one conditioning image
  // Four K = 512 operand images: X0 / X1 = h1 ping-pong (this step's h1 is X[cur], h1' goes to X[cur^1]), H0 / H1 = h2
  // ping-pong likewise; y1 goes to X[cur] and y2 to H[cur] once their old contents have been read.
  static constexpr int OFF_X0 = 0, OFF_X1 = ACT, OFF_H2 = 2 * ACT, OFF_H2B = 3 * ACT;
  static constexpr int OFF_COND = 4 * ACT;                   // two conditioning images (double buffer)
  static constexpr int OFF_RING = (OFF_COND + 2 * COND + 1023) / 1024 * 1024;
  static constexpr int SLOT_BYTES = CHUNK_BYTES;
  static constexpr int LOGP = 33;                                            // padded row of the logits transpose (conflict-free both ways)
  // RAW, cluster form: [4 ranks][NF] (score, class) candidates of the step, written by every rank into every rank
  static constexpr int CAND = RAW ? 4 * NF * 8 : 0;
  static constexpr int MISC = LOGP * NF * 4 + NF * 4 + NBAR * 8 + 64 + 256 + CAND;  // logits transpose, x, barriers, flags, zero block
  static constexpr int STAGES = (227 * 1024 - OFF_RING - MISC) / SLOT_BYTES > MAX_STAGES ? MAX_STAGES : (227 * 1024 - OFF_RING - MISC) / SLOT_BYTES;
  static constexpr int OFF_LOG = OFF_RING + STAGES * SLOT_BYTES;             // [NF][LOGP] fp32 (RAW: [2][8 warps][NF] candidates)
  static constexpr int OFF_XS = OFF_LOG + LOGP * NF * 4;                       // [NF] fp32: previous sample per fold
  static constexpr int OFF_BAR = OFF_XS + NF * 4;
  static constexpr int OFF_ZERO = OFF_BAR + NBAR * 8 + 64;                  // 256 B of zeros: B operand of padding MMAs
  static constexpr int OFF_CAND = OFF_ZERO + 256;
  static constexpr int BYTES = OFF_CAND + CAND;
  static_assert(STAGES >= 3, "ring too shallow");
  static_assert(BYTES <= 227 * 1024, "shared memory budget");
  static_assert(2 * 8 * NF * 8 <= LOGP * NF * 4, "RAW: the per-warp candidates of two blocks fit the logits transpose");
};
// the RAW head's candidate tables take shared memory the ring could not use anyway: as many ring slots as MoL
static_assert(Smem<16, true>::STAGES == Smem<16>::STAGES && Smem<32, true>::STAGES == Smem<32>::STAGES, "RAW ring depth");
// barrier indices
constexpr int BAR_FULL = 0, BAR_EMPTY = MAX_STAGES,
              BAR_READY = 2 * MAX_STAGES /* + {0, 1: cond[parity]; 2..5: h1' block b; 6..9: h2' block b; 10..13: y1 block b; 14..17: y2 block b} */,
              BAR_COND_FREE = BAR_READY + 18;
constexpr int BAR_X = BAR_COND_FREE + 2;    // cluster form: "the sample of this step has been written into this CTA's x_s"
constexpr int BAR_CAND = BAR_X + 1;         // RAW cluster form: "every rank's candidates of this step are in this CTA's table"
static_assert(BAR_CAND + 1 <= NBAR, "barrier table");

struct StreamParams {
  // per cluster rank (one-CTA form: rank 0 only): the weight stream and the chunk list of one step
  const unsigned char* blob[4]; const uint4* prog[4]; int n_prog[4];
  const float* qk; const float* vq; const float* b1h; const float* b2h; const float* b3;
  const float* mels_up; const float* aux; long long L; long long seg_stride; long long row_base;
  int n_total, steps, out_pitch, seg_first;
  const float* uniforms; const unsigned* uniforms_ready; unsigned long long seed, offset;
  float* out; const float* x_force; float* logits_out;
  const long long* fold_row0; const long long* fold_row_end;
  const FoldKey* keys;          // optional per-fold Philox keys [n_total]
  const float* mel_frames; const float* aux_frames; const float* up_taps; int hop;
  float* state;                 // [tiles][2][H][NF] fp32 hidden state
  int* abort_flag;
  long long* prof;              // optional cycle counters of CTA 0
  const float* expo;            // RAW: optional explicit Exp(1) draws [steps][n_total][512] (else Philox)
  float* nll;                   // scoring (MoL): [steps][n_total] loss of target x_force[t] (out is not written)
};

__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_rank(uint32_t addr, uint32_t rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}

// SCORE (wrnn_score, MoL only): rank 0's sampler threads write the loss of target x_force[t] instead of a sample and
// make no draws; the cluster form broadcasts x_force[t] as it broadcasts a sample.
template <int NF, int FMT, bool FRAMES, bool PROF, int CL, bool RAW, bool SCORE>
__global__ void __launch_bounds__(NT, 1) wrnn_stream_kernel(const StreamParams p) {
  static_assert(!(RAW && SCORE), "the stream engine scores the MoL head only");
  using SM = Smem<NF, RAW>;
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::OFF_BAR);
  volatile int* s_abort = reinterpret_cast<volatile int*>(smem + SM::OFF_BAR + NBAR * 8 + 16);   // CTA-local copy of the abort flag
  float* x_s = reinterpret_cast<float*>(smem + SM::OFF_XS);
  float* log_s = reinterpret_cast<float*>(smem + SM::OFF_LOG);
  auto bar = [&](int i) -> uint32_t { return smem_u32(&bars[i]); };

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (CL == 1) ? 0 : (int)cluster_rank();                  // which 128-unit block of every layer this CTA computes
  const int tile = blockIdx.x / CL, f0 = tile * NF;
  const int B = (p.n_total - f0 < NF) ? (p.n_total - f0) : NF;          // real folds of this tile
  const int S = p.steps;
  const uint4* prog = p.prog[rank];
  const int n_prog = p.n_prog[rank];

  // ---- setup ----------------------------------------------------------------------------------------------------
  {
    int4* z = reinterpret_cast<int4*>(smem);
    // operand images start as zeros; the ring too, so that the padding MMAs of a K = 16 chunk (ring bytes x 0) add exact zeros
    for (int i = tid; i < SM::OFF_LOG / 16; i += NT) z[i] = make_int4(0, 0, 0, 0);
    for (int i = tid; i < 256 / 16; i += NT) z[SM::OFF_ZERO / 16 + i] = make_int4(0, 0, 0, 0);
    if (tid < NF) x_s[tid] = 0.f;
    if (tid == 0) *s_abort = 0;
  }
  if (tid == 0) {
    for (int i = 0; i < SM::STAGES; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar(BAR_FULL + i)));
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 8;" :: "r"(bar(BAR_EMPTY + i)));            // one arrival per consumer warp
    }
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 32;" :: "r"(bar(BAR_READY + 0)));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 32;" :: "r"(bar(BAR_READY + 1)));
    // operand blocks: written here by the 256 consumer threads (one arrival each), or -- cluster form, a peer's block --
    // delivered by the peer's bulk copies (one arrive.expect_tx by the sender + the bytes)
    for (int i = 2; i < 18; ++i)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar(BAR_READY + i)), "r"((CL == 1 || ((i - 2) & 3) == rank) ? N_CONSUMERS : 1));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 8;" :: "r"(bar(BAR_COND_FREE + 0)));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 8;" :: "r"(bar(BAR_COND_FREE + 1)));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar(BAR_X)));
    if constexpr (RAW) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar(BAR_CAND)), "r"((uint32_t)CL));   // one arrival per rank
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  proxy_fence_smem();
  __syncthreads();
  if constexpr (CL > 1) cluster_sync_all();                  // every peer's barriers and zeroed images exist before anyone writes into them
  // Bounded wait (a protocol bug must end in WRNN_E_WATCHDOG, never in a hung GPU): once any wait of this CTA has given
  // up, or another CTA has raised the global flag, every later wait returns at once and the role loops end.
  auto wait = [&](uint32_t b, uint32_t parity) {
    if (mbar_try(b, parity)) return;
    if (*s_abort) return;
    const long long t0 = clock64();
    unsigned spins = 0;
    while (!mbar_try(b, parity)) {
      if ((++spins & 1023u) == 0) {
        if (*s_abort) return;
        if (ld_relaxed_s32(p.abort_flag) != 0) { *s_abort = 1; return; }
        if (clock64() - t0 > kWatchdogCycles) { atomicExch(p.abort_flag, 2); *s_abort = 1; return; }
      }
    }
  };

  // same, for barriers peers arrive on after writing into this CTA's shared memory (acquire at cluster scope)
  auto wait_peer = [&](uint32_t b, uint32_t parity) {
    if constexpr (CL == 1) { wait(b, parity); return; }
    auto try_cl = [&]() -> bool {
      uint32_t ok;
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                   : "=r"(ok) : "r"(b), "r"(parity) : "memory");
      return ok != 0;
    };
    if (try_cl()) return;
    if (*s_abort) return;
    const long long t0 = clock64();
    unsigned spins = 0;
    while (!try_cl()) {
      if ((++spins & 1023u) == 0) {
        if (*s_abort) return;
        if (ld_relaxed_s32(p.abort_flag) != 0) { *s_abort = 1; return; }
        if (clock64() - t0 > kWatchdogCycles) { atomicExch(p.abort_flag, 2); *s_abort = 1; return; }
      }
    }
  };

  if (warp == PRODUCER_WARP) {
    // ===================================================================================================== producer
    // one TMA (and one full / empty barrier) per chunk, in the order the consumers take them
    unsigned g = 0;                                           // chunk loads issued so far (ring position)
    for (int t = 0; t < S && !*s_abort; ++t) {
      for (int c = 0; c < n_prog; ++c) {
        const uint4 r = __ldg(prog + c);
        const uint32_t flags = (r.z >> 8) & 0xffu;
        if (flags & DF_SAME_SLOT) continue;                   // operand of the previous record's chunk
        const uint32_t bytes = (flags & DF_NK1) ? (uint32_t)(CHUNK_BYTES / 4) : (uint32_t)CHUNK_BYTES;
        const int slot = g % SM::STAGES;
        wait(bar(BAR_EMPTY + slot), ((g / SM::STAGES) & 1) ^ 1);      // slot drained by the MMAs of its chunk
        tma_bulk_g2s(smem_u32(smem + SM::OFF_RING + slot * SM::SLOT_BYTES), p.blob[rank] + (size_t)r.x * 16, bytes, bar(BAR_FULL + slot));
        ++g;
      }
    }
  } else if (warp == STAGING_WARP) {
    // ====================================================================================================== staging
    // cond_s (fp32 rows of the per-sample conditioning stream, or built from frame-rate tensors) -> fp16 image of step s,
    // one step ahead of the MMAs.  (fold, 8-column chunk) tasks, 32 threads.
    const int st = lane;
    auto row0_of = [&](int f) -> long long {
      return p.fold_row0 ? __ldg(p.fold_row0 + f0 + f) : (long long)(f0 + f + (FRAMES ? p.seg_first : 0)) * p.seg_stride - p.row_base;
    };
    auto end_of = [&](int f) -> long long { return p.fold_row_end ? __ldg(p.fold_row_end + f0 + f) : p.L; };
    for (int s = 0; s < S && !*s_abort; ++s) {
      const int par = s & 1;
      if (s >= 2) wait(bar(BAR_COND_FREE + par), (uint32_t)((s >> 1) - 1) & 1);   // step s-2 has consumed this buffer
      unsigned char* img = smem + SM::OFF_COND + par * SM::COND;
#pragma unroll 2
      for (int task = st; task < NF * KQ; task += 32) {
        const int f = task / KQ, c8 = task - f * KQ;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
        const long long row = (f < B) ? row0_of(f) + s : 0;
        if (f < B && row < end_of(f)) {
          if constexpr (!FRAMES) {
            const float* src = (c8 < FEAT / 8) ? p.mels_up + row * FEAT + c8 * 8 : p.aux + row * (4 * AUXD) + (c8 - FEAT / 8) * 8;
            a = __ldg(reinterpret_cast<const float4*>(src)); b = __ldg(reinterpret_cast<const float4*>(src) + 1);
          } else {
            const unsigned r = (unsigned)row, frame = r / (unsigned)p.hop, phase = r - frame * (unsigned)p.hop;
            if (c8 >= FEAT / 8) {
              const float4* src = reinterpret_cast<const float4*>(p.aux_frames + (size_t)frame * (4 * AUXD) + (c8 - FEAT / 8) * 8);
              a = __ldg(src); b = __ldg(src + 1);
            } else {                                           // same fmaf order as wrnn_expand_rows_kernel -> identical rows
              const float* k = p.up_taps + phase * 5;
#pragma unroll
              for (int d = 0; d < 5; ++d) {
                const float wgt = __ldg(k + d);
                const float4* src = reinterpret_cast<const float4*>(p.mel_frames + (size_t)(frame + d) * FEAT + c8 * 8);
                const float4 x0 = __ldg(src), x1 = __ldg(src + 1);
                a.x = fmaf(wgt, x0.x, a.x); a.y = fmaf(wgt, x0.y, a.y); a.z = fmaf(wgt, x0.z, a.z); a.w = fmaf(wgt, x0.w, a.w);
                b.x = fmaf(wgt, x1.x, b.x); b.y = fmaf(wgt, x1.y, b.y); b.z = fmaf(wgt, x1.z, b.z); b.w = fmaf(wgt, x1.w, b.w);
              }
            }
          }
        }
        uint4 v;
        v.x = pack2<FMT>(a.x, a.y); v.y = pack2<FMT>(a.z, a.w); v.z = pack2<FMT>(b.x, b.y); v.w = pack2<FMT>(b.z, b.w);
        *reinterpret_cast<uint4*>(img + (f >> 3) * SBO_Q + c8 * 128 + (f & 7) * 16) = v;
      }
      proxy_fence_smem();                                      // generic-proxy stores -> async-proxy (MMA) reads
      mbar_arrive(bar(BAR_READY + par));
    }
  } else if (warp < PRODUCER_WARP) {
    // ===================================================================================================== consumers
    const int wg = warp >> 2;                                  // rows [64 wg, 64 wg + 64) of every 128-row chunk
    // this thread's fragment: rows rw and rw + 8 of the chunk, folds 8j + fc (+1), j < NF / 8
    const int rw = 64 * wg + 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
    float* st_h1 = p.state + ((size_t)tile * 2 + 0) * H * NF;
    float* st_h2 = p.state + ((size_t)tile * 2 + 1) * H * NF;
    unsigned rows_known = p.uniforms_ready ? 0u : 0xffffffffu;   // rows of p.uniforms known to have landed (streamed draws)
    const bool profiling = PROF && blockIdx.x == 0 && tid == 0;
    long long t_ring = 0, t_b = 0, t_issue = 0, t_epi = 0;
    const uint32_t s0_lo = smem_u32(smem) >> 4, ring_lo = smem_u32(smem + SM::OFF_RING) >> 4;
    constexpr uint64_t LBO = (uint64_t)(128u >> 4) << 16;
    const uint64_t dz = (uint64_t)((smem_u32(smem + SM::OFF_ZERO) >> 4) & 0x3fffu) | LBO;     // zero block, SBO 0
    unsigned g_next = 0;                                       // chunk loads consumed so far (ring position)
    int slot = 0;
    float d[NF / 2];                                           // the chain being accumulated
    float acc[4][NF / 2];                                      // the finished chains of the current (phase, block)

    // This CTA's part of operand `kind`, unit block `blk` (GLOBAL block id) of the image at `off` is written.  Cluster
    // form: the block is written LOCALLY like in the one-CTA form, then three elected threads (one per peer) push it into
    // the same place of the peers' images with bulk copies (shared::cta -> shared::cluster, NF/8 pieces of 2 KB: the 16
    // K-chunks of the block are contiguous within a fold group) that complete_tx on the peer's readiness barrier.
    auto publish_ready = [&](int kind, int blk, int off) {
      const uint32_t b = bar(BAR_READY + 2 + (kind - W_H1NEW) * 4 + blk);
      proxy_fence_smem();
      mbar_arrive(b);
      if constexpr (CL > 1) {
        named_bar_sync(2, N_CONSUMERS);                        // every consumer thread's stores (and proxy fences) are done
        if (lane == 0 && warp >= 1 && warp <= 3) {
          const uint32_t peer = (uint32_t)((rank + warp) & 3);
          if (RAW || kind != W_Y2 || peer == 0u) {              // y2: MoL's fc3 runs in rank 0 only, RAW's in every rank
            const uint32_t rb = map_to_rank(b, peer);
            asm volatile("mbarrier.arrive.expect_tx.relaxed.cluster.shared::cluster.b64 _, [%0], %1;" :: "r"(rb), "r"((uint32_t)(NF * 256)) : "memory");
#pragma unroll
            for (int g = 0; g < NF / 8; ++g) {
              const uint32_t src = smem_u32(smem + off + g * SBO_H + blk * (MROWS / 8) * 128);
              asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                           :: "r"(map_to_rank(src, peer)), "r"(src), "r"((uint32_t)((MROWS / 8) * 128)), "r"(rb) : "memory");
            }
          }
        }
      }
    };
    // element (fold f, unit k) of a K = 512 operand image
    auto img_store = [&](int off, int f, int k, float v) {
      *reinterpret_cast<uint16_t*>(smem + off + (f >> 3) * SBO_H + (k >> 3) * 128 + (f & 7) * 16 + (k & 7) * 2) = (uint16_t)(pack2<FMT>(v, 0.f) & 0xffffu);
    };

    volatile int* ep_stop = s_abort + 1;                      // the consumers leave the loop together (named barriers inside)
    if (tid == 0) *ep_stop = 0;
    named_bar_sync(1, N_CONSUMERS);
    for (int t = 0; t < S; ++t) {
      const int cur = t & 1;
      const int off_h1new = cur ? SM::OFF_X0 : SM::OFF_X1, off_y1 = cur ? SM::OFF_X1 : SM::OFF_X0;
      const int off_h2new = cur ? SM::OFF_H2 : SM::OFF_H2B, off_y2 = cur ? SM::OFF_H2B : SM::OFF_H2;
      // draws of this step for the fold this thread samples (rank 0, threads 0 .. B-1)
      float ur[11];
#pragma unroll
      for (int i = 0; i < 11; ++i) ur[i] = 0.5f;
      const bool sampler = rank == 0 && tid < B;
      if (!RAW && !SCORE && p.uniforms && rank == 0 && warp == 0) {      // streamed draws: read row t once rows t .. t+3 have landed (see wrnn_tc.cu)
        const unsigned need = min((unsigned)S, (unsigned)t + 4u);
        if (rows_known < need) rows_known = rows_wait(p.uniforms_ready, need, p.abort_flag);
      }
      if (!RAW && !SCORE && sampler) {                         // (RAW: the fc3 epilogue draws per class)
        const int gf = f0 + tid;
        if (p.uniforms) {
          const float* u = p.uniforms + (size_t)t * 11 * p.n_total;
#pragma unroll
          for (int i = 0; i < 10; ++i) ur[i] = __ldca(u + gf * 10 + i);
          ur[10] = __ldca(u + 10 * p.n_total + gf);
        } else {
          mol_uniforms(fold_philox(p.keys, gf, p.seg_first, p.seed), (unsigned)t, (unsigned)p.offset, ur);
        }
      }

      // RAW, one-CTA form: the best (score, class) of fold `lane` over the fc3 blocks done so far (warp 0, lanes < NF)
      float run_best = -INFINITY;
      int run_k = 0x7fffffff;
      auto better = [](float s, int k, float bs, int bk) { return s > bs || (s == bs && k < bk); };   // ties: lowest class

      // ---- epilogue of one (phase, block) group: accumulators -> gates / relu / logits -----------------------------------
      auto epilogue = [&](int phase, int blk) {
        if (phase <= 1) {                                      // P1 / P2: the two GRU cells
          const int cell = phase;
          float* stt = cell ? st_h2 : st_h1;
          const float* bh = cell ? p.b2h : p.b1h;
          const int qbase = cell * 3 * H;                      // rows of qk / vq: gi1 = 0.., gi2 = 3H..
          const int off_out = cell ? off_h2new : off_h1new;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int u = blk * MROWS + rw + 8 * hr;
            const float qk_r = __ldg(p.qk + qbase + u), qk_z = __ldg(p.qk + qbase + H + u), qk_n = __ldg(p.qk + qbase + 2 * H + u);
            const float vq_r = __ldg(p.vq + qbase + u), vq_z = __ldg(p.vq + qbase + H + u), vq_n = __ldg(p.vq + qbase + 2 * H + u);
            const float bh_r = __ldg(bh + u), bh_z = __ldg(bh + H + u), bh_n = __ldg(bh + 2 * H + u);
            float* hrow = stt + (size_t)u * NF;
#pragma unroll
            for (int j = 0; j < NF / 8; ++j) {
              const int f = 8 * j + fc;
              float2 hp = make_float2(0.f, 0.f);
              if (t > 0) hp = __ldcg(reinterpret_cast<const float2*>(hrow + f));
              float hv[2] = {hp.x, hp.y};
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int i = 4 * j + 2 * hr + e;
                const float x = x_s[f + e];
                // (the recurrent r / z contributions are already inside acc[0] / acc[1]: one accumulator per gate)
                hv[e] = gru_unit_fast(acc[0][i] + qk_r + x * vq_r, acc[1][i] + qk_z + x * vq_z, acc[2][i] + qk_n + x * vq_n,
                                      bh_r, bh_z, acc[3][i] + bh_n, hv[e]);
                img_store(off_out, f + e, u, hv[e]);
              }
              __stcg(reinterpret_cast<float2*>(hrow + f), make_float2(hv[0], hv[1]));
            }
          }
          publish_ready(cell ? W_H2NEW : W_H1NEW, blk, off_out);
        } else if (phase <= 3) {                               // P3 fc1 -> y1 into X[cur], P4 fc2 -> y2 into H[cur]
          const int qbase = (phase == 2 ? 6 : 7) * H;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int u = blk * MROWS + rw + 8 * hr;
            const float qk_u = __ldg(p.qk + qbase + u), vq_u = phase == 2 ? __ldg(p.vq + qbase + u) : 0.f;
#pragma unroll
            for (int j = 0; j < NF / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int i = 4 * j + 2 * hr + e, f = 8 * j + fc + e;
                const float a = (acc[0][i] + acc[1][i]) + (acc[2][i] + acc[3][i]);
                const float y = phase == 2 ? fmaxf(a + qk_u + x_s[f] * vq_u, 0.f) : fmaxf(a + qk_u, 0.f);
                img_store(phase == 2 ? off_y1 : off_y2, f, u, y);
              }
            }
          }
          publish_ready(phase == 2 ? W_Y1 : W_Y2, blk, phase == 2 ? off_y1 : off_y2);
        } else if constexpr (RAW) {
          // P5, RAW head, classes [128 blk, 128 blk + 128): logit = F3 y2 + b3, score = logit - log e with e the class's
          // Exp(1) draw (raw_block / raw_exp: block 16 + class / 4, word class % 4; or `expo`);
          // the pick is the best score, ties to the lowest class.  This thread holds rows rw, rw + 8 of folds 8j + fc (+1):
          // two words of two different Philox blocks per fold, each block computed for the one word it gives.
          uint2* cw = reinterpret_cast<uint2*>(smem + SM::OFF_LOG) + (blk & 1) * 8 * NF;      // [warp][fold] best of the warp's 16 rows
          const unsigned o0 = (unsigned)p.offset;
#pragma unroll
          for (int j = 0; j < NF / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int f = 8 * j + fc + e;
              const size_t row_out = ((size_t)t * p.n_total + f0 + f) * NCLS_RAW;
              FoldPhilox key{0u, 0u, 0u};
              if (f < B && !p.expo) key = fold_philox(p.keys, f0 + f, p.seg_first, p.seed);
              float best = 0.f;
              int bk = 0;
#pragma unroll
              for (int hr = 0; hr < 2; ++hr) {
                const int i = 4 * j + 2 * hr + e, k = blk * MROWS + rw + 8 * hr;
                const float lg = ((acc[0][i] + acc[1][i]) + (acc[2][i] + acc[3][i])) + __ldg(p.b3 + k);
                float ex = 1.f;
                if (f < B) {
                  if (p.expo) {
                    ex = __ldg(p.expo + row_out + k);
                  } else {
                    ex = raw_exp(raw_block(key, (unsigned)t, (unsigned)(k >> 2), o0), (unsigned)(k & 3));
                  }
                  if (p.logits_out) p.logits_out[row_out + k] = lg;
                }
                const float sc = lg - __logf(ex);
                if (hr == 0 || better(sc, k, best, bk)) { best = sc; bk = k; }
              }
              // the warp's 8 row groups (lanes 4, 8, 16 apart)
#pragma unroll
              for (int m = 4; m < 32; m <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, m);
                const int ok = __shfl_xor_sync(0xffffffffu, bk, m);
                if (better(ob, ok, best, bk)) { best = ob; bk = ok; }
              }
              if (lane < 4) cw[warp * NF + f] = make_uint2(__float_as_uint(best), (unsigned)bk);
            }
          }
          named_bar_sync(3, N_CONSUMERS);                      // every warp's candidates of this block are in cw
          if (warp == 0) {
            float bs = -INFINITY;
            int bk = 0x7fffffff;
            if (lane < NF) {
#pragma unroll
              for (int w = 0; w < 8; ++w) {                    // warps in ascending class order
                const uint2 v = cw[w * NF + lane];
                if (better(__uint_as_float(v.x), (int)v.y, bs, bk)) { bs = __uint_as_float(v.x); bk = (int)v.y; }
              }
            }
            bool done = false;
            if constexpr (CL == 1) {
              if (better(bs, bk, run_best, run_k)) { run_best = bs; run_k = bk; }
              bs = run_best; bk = run_k;
              done = blk == NCLS_RAW / MROWS - 1;
            } else {
              // this rank's candidate into slot `rank` of every rank's table, then a release at cluster scope on every
              // rank's candidate barrier; every rank then reduces the same four candidates the same way
              uint2* ct = reinterpret_cast<uint2*>(smem + SM::OFF_CAND);                        // [rank][fold]
              if (lane < NF) {
                const uint32_t a = smem_u32(ct + rank * NF + lane);
#pragma unroll
                for (int r = 0; r < CL; ++r)
                  asm volatile("st.shared::cluster.v2.u32 [%0], {%1, %2};" :: "r"(map_to_rank(a, (uint32_t)r)), "r"(__float_as_uint(bs)), "r"((uint32_t)bk) : "memory");
              }
              __syncwarp();
              if (lane == 0) {
#pragma unroll
                for (int r = 0; r < CL; ++r)
                  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" :: "r"(map_to_rank(bar(BAR_CAND), (uint32_t)r)) : "memory");
                wait_peer(bar(BAR_CAND), (uint32_t)t & 1);
              }
              __syncwarp();
              bs = -INFINITY; bk = 0x7fffffff;
              if (lane < NF) {
#pragma unroll
                for (int r = 0; r < CL; ++r) {
                  const uint2 v = ct[r * NF + lane];
                  if (better(__uint_as_float(v.x), (int)v.y, bs, bk)) { bs = __uint_as_float(v.x); bk = (int)v.y; }
                }
              }
              done = true;
            }
            if (done && lane < NF) {
              float xnew = 0.f;
              if (lane < B) {
                const int gf = f0 + lane;
                xnew = 2.0f * (float)bk / ((float)NCLS_RAW - 1.0f) - 1.0f;          // reference :235
                if (rank == 0) p.out[(size_t)gf * p.out_pitch + t] = xnew;
                if (p.x_force) xnew = __ldg(p.x_force + (size_t)t * p.n_total + gf);
              }
              x_s[lane] = xnew;                                // read after the end-of-step barrier
            }
          }
        } else {                                               // P5 (rank 0): logits -> transpose -> one thread per fold samples
          if (wg == 0 && rw < 32) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const int row = rw + 8 * hr;
              const float b3 = __ldg(p.b3 + row);
#pragma unroll
              for (int j = 0; j < NF / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int i = 4 * j + 2 * hr + e;
                  log_s[(8 * j + fc + e) * SM::LOGP + row] = ((acc[0][i] + acc[1][i]) + (acc[2][i] + acc[3][i])) + b3;   // [fold][class]
                }
              }
            }
          }
          named_bar_sync(3, N_CONSUMERS);                      // the logits of every fold are in log_s
          if (warp == 0) {
            float xnew = 0.f;
            if (sampler) {
              float lgo[32];
#pragma unroll
              for (int i = 0; i < 32; ++i) lgo[i] = log_s[lane * SM::LOGP + i];
              const int gf = f0 + lane;
              if constexpr (SCORE) {
                xnew = __ldg(p.x_force + (size_t)t * p.n_total + gf);
                p.nll[(size_t)t * p.n_total + gf] = mol_nll([&](int i) { return lgo[i]; }, xnew);
              } else {
                xnew = mol_sample_fast(lgo, ur);
                p.out[(size_t)gf * p.out_pitch + t] = xnew;
              }
              if (p.logits_out) {
#pragma unroll
                for (int i = 0; i < 30; ++i) p.logits_out[((size_t)t * p.n_total + gf) * 30 + i] = lgo[i];
              }
              if (!SCORE && p.x_force) xnew = __ldg(p.x_force + (size_t)t * p.n_total + gf);   // teacher forcing: step t+1 consumes x_force[t]
            }
            __syncwarp();
            if constexpr (CL == 1) {
              if (lane < NF) x_s[lane] = xnew;
            } else {
              if (lane < NF) {
                const uint32_t a = smem_u32(x_s + lane);
#pragma unroll
                for (int r = 0; r < CL; ++r)
                  asm volatile("st.shared::cluster.f32 [%0], %1;" :: "r"(map_to_rank(a, (uint32_t)r)), "f"(xnew) : "memory");
              }
              __syncwarp();
              if (lane == 0) {
#pragma unroll
                for (int r = 0; r < CL; ++r)
                  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" :: "r"(map_to_rank(bar(BAR_X), (uint32_t)r)) : "memory");
              }
            }
          }
        }
      };

      // ---- the step program ---------------------------------------------------------------------------------------------
      uint4 nx = __ldg(prog);
#pragma unroll 1
      for (int c = 0; c < n_prog; ++c) {
        const uint4 r = nx;
        if (c + 1 < n_prog) nx = __ldg(prog + c + 1);
        const uint32_t accsel = r.z & 0xffu, flags = (r.z >> 8) & 0xffu, wait_b = (r.z >> 16) & 0xffu;
        const uint32_t phase = (r.z >> 24) & 0xfu, blk = r.z >> 28;
        long long c0 = 0, c1 = 0, c2 = 0;
        if (profiling) c0 = clock64();
        const uint32_t wkind = wait_b & 15u;
        if (wkind == W_COND) wait(bar(BAR_READY + cur), (uint32_t)(t >> 1) & 1);
        else if (wkind != W_NONE) {
          // the block this K range reads: written here through the generic proxy (fenced by its writers), or a peer's
          // block that arrived by bulk copy (async proxy, complete_tx on this barrier) -- like a TMA load, no fence
          wait(bar(BAR_READY + 2 + (wkind - W_H1NEW) * 4 + (wait_b >> 4)), (uint32_t)t & 1);
        }
        if (profiling) c1 = clock64();
        if (!(flags & DF_SAME_SLOT)) {
          slot = g_next % SM::STAGES;
          wait(bar(BAR_FULL + slot), (g_next / SM::STAGES) & 1);
          ++g_next;
        }
        if (profiling) c2 = clock64();
        {
          const bool one = (flags & DF_NK1) != 0;
          // (address field: 14 bits of byte address >> 4 -- masked, because in a cluster launch the shared::cta window of
          //  ranks > 0 need not start at 0)
          const uint32_t a_lo = (ring_lo + (uint32_t)slot * (SM::SLOT_BYTES >> 4) + (uint32_t)wg * (one ? (2048u >> 4) : (8192u >> 4))) & 0x3fffu;
          const uint64_t da = (uint64_t)a_lo | LBO | ((uint64_t)((one ? 256u : 1024u) >> 4) << 32);
          const uint64_t sbo_b = (uint64_t)(((flags & DF_B_COND) ? (uint32_t)SBO_Q : (uint32_t)SBO_H) >> 4) << 32;
          const uint32_t blo = cur ? (r.y >> 16) : (r.y & 0xffffu);
          const uint64_t db = (uint64_t)((s0_lo + blo) & 0x3fffu) | LBO | sbo_b;
          const uint32_t scale0 = (flags & DF_FIRST) ? 0u : 1u;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)           // K = 16 chunk: steps 1-3 multiply the zero block (SBO 0: every row group)
            wgmma_ss<NF, FMT>(d, da + (uint64_t)(16 * k), (one && k > 0) ? dz : db + (uint64_t)(16 * k), k == 0 ? scale0 : 1u);
          wgmma_commit();
          wgmma_wait<0>();
        }
        __syncwarp();
        if (lane == 0) {
          if (!(flags & DF_KEEP_SLOT)) mbar_arrive(bar(BAR_EMPTY + slot));   // this warp's reads of the slot are complete
          if (flags & DF_COND_RELEASE) mbar_arrive(bar(BAR_COND_FREE + cur));
        }
        if (flags & DF_ACC_END) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int i = 0; i < NF / 2; ++i) acc[j][i] = (accsel == (uint32_t)j) ? d[i] : acc[j][i];
          }
        }
        if (profiling) { const long long c3 = clock64(); t_b += c1 - c0; t_ring += c2 - c1; t_issue += c3 - c2; }
        if (flags & DF_END) {
          long long e0 = 0;
          if (profiling) e0 = clock64();
          epilogue((int)phase, (int)blk);
          if (profiling) t_epi += clock64() - e0;
        }
      }
      // x of this step has landed here (cluster form: rank 0's remote stores, released at cluster scope).  One thread
      // acquires -- every poll of an acquire.cluster wait invalidates L1 --, the named barrier below hands it on.
      if (tid == 0) {
        if constexpr (CL > 1 && !RAW) wait_peer(bar(BAR_X), (uint32_t)t & 1);   // (RAW: every rank computed x itself)
        *ep_stop = *s_abort;
      }
      named_bar_sync(1, N_CONSUMERS);                          // x of this step (and the stop decision) visible to all consumers
      if (*ep_stop) break;
    }
    if (profiling) { p.prof[0] = t_b; p.prof[1] = t_ring; p.prof[2] = t_issue; p.prof[3] = t_epi; }
  }

  __syncthreads();
  if constexpr (CL > 1) cluster_sync_all();                  // nobody leaves while a peer may still write into its shared memory
}

// --------------------------------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------------------------------
class StreamEngine : public Engine {
 public:
  ~StreamEngine() override {
    cudaSetDevice(device);
    for (auto& v : var_) { cudaFree(v.d_blob); cudaFree(v.d_prog); }
    cudaFree(d_vec_); cudaFree(d_state_); cudaFree(d_sync_);
  }
  // (engine names are part of the C ABI's introspection surface and predate the Hopper port)
  const char* name() const override {
    if (last_cluster_) return cfg.precision == WRNN_PREC_BF16 ? "tcgen05-stream-x4-bf16" : "tcgen05-stream-x4-fp16";
    return cfg.precision == WRNN_PREC_BF16 ? "tcgen05-stream-bf16" : "tcgen05-stream-fp16";
  }
  int grid_ctas() const override { return last_grid_; }

  template <int NF, int CL, bool PROF, bool RAW, bool SC = false> const void* kernel_r(bool frames) const {
    if (cfg.precision == WRNN_PREC_BF16) return frames ? (const void*)wrnn_stream_kernel<NF, 1, true, PROF, CL, RAW, SC> : (const void*)wrnn_stream_kernel<NF, 1, false, PROF, CL, RAW, SC>;
    return frames ? (const void*)wrnn_stream_kernel<NF, 0, true, PROF, CL, RAW, SC> : (const void*)wrnn_stream_kernel<NF, 0, false, PROF, CL, RAW, SC>;
  }
  // MoL scoring (no profiling variant)
  template <int NF, int CL> const void* kernel_score(bool frames) const { return kernel_r<NF, CL, false, false, true>(frames); }
  template <int NF, int CL, bool PROF> const void* kernel_p(bool frames) const {
    return raw() ? kernel_r<NF, CL, PROF, true>(frames) : kernel_r<NF, CL, PROF, false>(frames);
  }
  template <int NF, int CL> const void* kernel_nf(bool frames, bool prof) const { return prof ? kernel_p<NF, CL, true>(frames) : kernel_p<NF, CL, false>(frames); }
  template <int NF> static SmemLayout layout() {
    using S = Smem<NF>;
    return SmemLayout{S::OFF_X0, S::OFF_X1, {S::OFF_H2, S::OFF_H2B}, S::OFF_COND, S::COND};
  }
  bool raw() const { return cfg.mode == WRNN_MODE_RAW; }
  template <int NF> int smem_bytes() const { return raw() ? Smem<NF, true>::BYTES : Smem<NF>::BYTES; }

  // one (cluster size, folds per CTA) combination: its weight streams (one per cluster rank) and device programs
  struct Variant {
    int nf = 0, cl = 1, smem = 0;
    void *d_blob = nullptr, *d_prog = nullptr;
    size_t blob_off[4] = {0, 0, 0, 0}, prog_off[4] = {0, 0, 0, 0};
    int n_prog[4] = {0, 0, 0, 0};
  };

  int upload(Variant& v, const std::vector<Plan>& plans, const SmemLayout& L) {
    std::vector<uint8_t> blob; std::vector<DevChunk> prog;
    for (size_t r = 0; r < plans.size(); ++r) {
      const Plan& pl = plans[r];
      std::vector<DevChunk> dp;
      compile_device(pl, L, plans.size() > 1 ? (int)r : -1, dp);
      v.blob_off[r] = blob.size(); blob.insert(blob.end(), pl.blob.begin(), pl.blob.end());
      while (blob.size() % 16) blob.push_back(0);
      v.prog_off[r] = prog.size(); v.n_prog[r] = (int)dp.size(); prog.insert(prog.end(), dp.begin(), dp.end());
    }
    WRNN_CUDA_OK(cudaMalloc(&v.d_blob, blob.size()));
    WRNN_CUDA_OK(cudaMemcpy(v.d_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    WRNN_CUDA_OK(cudaMalloc(&v.d_prog, prog.size() * sizeof(DevChunk)));
    WRNN_CUDA_OK(cudaMemcpy(v.d_prog, prog.data(), prog.size() * sizeof(DevChunk), cudaMemcpyHostToDevice));
    return WRNN_OK;
  }

  int init(const HostWeights& w) {
    const bool bf = cfg.precision == WRNN_PREC_BF16;
    std::vector<Plan> whole(1), split(4);
    build_plan(w, bf, whole[0]);
    for (int r = 0; r < 4; ++r) build_plan(w, bf, split[r], r);
    n_chunks_ = (int)whole[0].prog.size(); n_mma_ = whole[0].n_mma;
    int rc;
    var_[0].nf = 16; var_[0].cl = 1; var_[0].smem = smem_bytes<16>(); if ((rc = upload(var_[0], whole, layout<16>())) != WRNN_OK) return rc;
    var_[1].nf = 32; var_[1].cl = 1; var_[1].smem = smem_bytes<32>(); if ((rc = upload(var_[1], whole, layout<32>())) != WRNN_OK) return rc;
    var_[2].nf = 16; var_[2].cl = 4; var_[2].smem = smem_bytes<16>(); if ((rc = upload(var_[2], split, layout<16>())) != WRNN_OK) return rc;
    var_[3].nf = 32; var_[3].cl = 4; var_[3].smem = smem_bytes<32>(); if ((rc = upload(var_[3], split, layout<32>())) != WRNN_OK) return rc;
    const Plan& plan = whole[0];
    std::vector<float> vec;
    off_qk_ = 0; vec.insert(vec.end(), plan.qk.begin(), plan.qk.end());
    off_vq_ = vec.size(); vec.insert(vec.end(), plan.vq.begin(), plan.vq.end());
    off_b1h_ = vec.size(); vec.insert(vec.end(), plan.b1h.begin(), plan.b1h.end());
    off_b2h_ = vec.size(); vec.insert(vec.end(), plan.b2h.begin(), plan.b2h.end());
    off_b3_ = vec.size(); vec.insert(vec.end(), plan.b3.begin(), plan.b3.end());
    WRNN_CUDA_OK(cudaMalloc(&d_vec_, vec.size() * sizeof(float)));
    WRNN_CUDA_OK(cudaMemcpy(d_vec_, vec.data(), vec.size() * sizeof(float), cudaMemcpyHostToDevice));
    WRNN_CUDA_OK(cudaMalloc(&d_sync_, 256));
    WRNN_CUDA_OK(cudaMemset(d_sync_, 0, 256));
    for (int k = 0; k < 4; ++k) {
      const bool fr = (k & 1) != 0, pr = (k & 2) != 0;
      WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_nf<16, 1>(fr, pr), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<16>()));
      WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_nf<32, 1>(fr, pr), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<32>()));
      WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_nf<16, 4>(fr, pr), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<16>()));
      WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_nf<32, 4>(fr, pr), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<32>()));
    }
    if (!raw()) {
      for (int fr = 0; fr < 2; ++fr) {
        WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_score<16, 1>(fr != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<16>()));
        WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_score<32, 1>(fr != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<32>()));
        WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_score<16, 4>(fr != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<16>()));
        WRNN_CUDA_OK(cudaFuncSetAttribute(kernel_score<32, 4>(fr != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<32>()));
      }
    }
    WRNN_CUDA_OK(cudaDeviceGetAttribute(&n_sm_, cudaDevAttrMultiProcessorCount, device));
    // clusters of four that fit the device at once (GPC granularity); both tile sizes use the same shared memory class
    {
      cudaLaunchConfig_t lc{};
      lc.gridDim = dim3(4 * n_sm_); lc.blockDim = dim3(NT); lc.dynamicSmemBytes = smem_bytes<32>();
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 4; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      lc.attrs = at; lc.numAttrs = 1;
      int n_cl = 0;
      WRNN_CUDA_OK(cudaOccupancyMaxActiveClusters(&n_cl, kernel_nf<32, 4>(false, false), &lc));
      max_clusters_ = n_cl;
    }
    return WRNN_OK;
  }

  static bool supports_cfg(const wrnn_cfg& c) {
    return c.precision != WRNN_PREC_FP32 && ((c.mode == WRNN_MODE_MOL && c.n_classes == 30) || (c.mode == WRNN_MODE_RAW && c.n_classes == NCLS_RAW));
  }
  // explicit Exp(1) draws (`expo`) belong to the RAW head; streamed uniforms (`uniforms_ready`) are MoL draws and unused by it
  bool supports(const wrnn_job& job) const override {
    return (raw() || job.expo == nullptr) && !(job.mel_frames && job.cond_mode == WRNN_COND_EXPAND && job.fold_row0);
  }

  // Which form serves n folds:
  //   one CTA per tile : 16 folds per CTA while the tiles fit one wave (one tile per SM), 32 folds per CTA beyond
  //   cluster of 4     : the rows of every layer split over four CTAs -> a quarter of the stream per SM; used while the
  //                      clusters of the job are co-resident (cudaOccupancyMaxActiveClusters at init)
  void choose(int n_seg, int& nf, int& cl) const {
    const int max_cl = max_clusters_;
    if ((n_seg + 15) / 16 <= max_cl) { nf = 16; cl = 4; }
    else if ((n_seg + 31) / 32 <= max_cl) { nf = 32; cl = 4; }
    else if ((n_seg + 15) / 16 <= n_sm_) { nf = 16; cl = 1; }
    else { nf = 32; cl = 1; }
    if (const char* e = getenv("WRNN_STREAM_NF")) { const int v = atoi(e); if (v == 16 || v == 32) nf = v; }   // experiments
    if (const char* e = getenv("WRNN_STREAM_CL")) { const int v = atoi(e); if (v == 1 || v == 4) cl = v; }
  }

  int generate(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys) override { return run(job, stream, keys, nullptr); }
  bool scores() const override { return !raw(); }
  const char* live_refusal() const override {
    return "live vocoding runs on the persistent engine only: the stream engine's cluster form takes about 66 us per step, "
           "slower than real time for one fold (DESIGN.md section 3.2)";
  }
  int score(const wrnn_job& job, float* nll, cudaStream_t stream, const FoldKey* keys) override {
    if (raw()) { set_error("the stream engine scores the MoL head only: score RAW jobs on the persistent or SIMT engine"); return WRNN_E_INVALID; }
    return run(job, stream, keys, nll);
  }

  // nll != NULL: MoL scoring (the loss of x_force[t] in the sampler's place; the draws are not read)
  int run(const wrnn_job& job, cudaStream_t stream, const FoldKey* keys, float* nll) {
    WRNN_CUDA_OK(cudaSetDevice(device));
    int nf = 16, cl = 1;
    choose(job.n_seg, nf, cl);
    const Variant& V = var_[(cl == 4 ? 2 : 0) + (nf == 32 ? 1 : 0)];
    const int tiles = (job.n_seg + nf - 1) / nf;
    const size_t need = (size_t)tiles * 2 * H * nf * sizeof(float);
    if (need > state_bytes_) {
      cudaFree(d_state_); d_state_ = nullptr; state_bytes_ = 0;
      WRNN_CUDA_OK(cudaMalloc(&d_state_, need));
      state_bytes_ = need;
    }
    StreamParams p{};
    const float* v = static_cast<const float*>(d_vec_);
    for (int r = 0; r < cl; ++r) {
      p.blob[r] = static_cast<const unsigned char*>(V.d_blob) + V.blob_off[r];
      p.prog[r] = static_cast<const uint4*>(V.d_prog) + V.prog_off[r];
      p.n_prog[r] = V.n_prog[r];
    }
    p.qk = v + off_qk_; p.vq = v + off_vq_; p.b1h = v + off_b1h_; p.b2h = v + off_b2h_; p.b3 = v + off_b3_;
    p.mels_up = job.mels_up; p.aux = job.aux; p.L = job.L; p.seg_stride = job.seg_stride; p.row_base = 0;
    p.n_total = job.n_seg; p.steps = job.steps > 0 ? job.steps : job.seg_len; p.out_pitch = p.steps; p.seg_first = job.seg_first;
    p.uniforms = job.uniforms; p.uniforms_ready = job.uniforms_ready; p.seed = job.philox_seed; p.offset = job.philox_offset;
    p.out = job.out; p.x_force = job.x_force; p.logits_out = job.logits_out; p.expo = raw() ? job.expo : nullptr;
    p.fold_row0 = reinterpret_cast<const long long*>(job.fold_row0); p.fold_row_end = reinterpret_cast<const long long*>(job.fold_row_end);
    p.keys = keys;
    p.mel_frames = job.mel_frames; p.aux_frames = job.aux_frames; p.up_taps = job.up_taps; p.hop = job.hop;
    p.state = static_cast<float*>(d_state_);
    p.abort_flag = reinterpret_cast<int*>(static_cast<unsigned*>(d_sync_) + 8);
    p.nll = nll;
    if (nll) { p.uniforms = nullptr; p.uniforms_ready = nullptr; p.expo = nullptr; }
    const bool prof = !nll && getenv("WRNN_STREAM_PROF") != nullptr;
    p.prof = reinterpret_cast<long long*>(static_cast<unsigned char*>(d_sync_) + 64);
    const bool frames = job.mel_frames != nullptr;             // rows are formed by the staging warps (no scratch of size L)
    const void* fn = nll ? (cl == 4 ? (nf == 16 ? kernel_score<16, 4>(frames) : kernel_score<32, 4>(frames))
                                    : (nf == 16 ? kernel_score<16, 1>(frames) : kernel_score<32, 1>(frames)))
                         : cl == 4 ? (nf == 16 ? kernel_nf<16, 4>(frames, prof) : kernel_nf<32, 4>(frames, prof))
                                   : (nf == 16 ? kernel_nf<16, 1>(frames, prof) : kernel_nf<32, 1>(frames, prof));
    void* args[] = {&p};
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(tiles * cl); lc.blockDim = dim3(NT); lc.dynamicSmemBytes = V.smem; lc.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    lc.attrs = at; lc.numAttrs = cl > 1 ? 1 : 0;
    WRNN_CUDA_OK(cudaLaunchKernelExC(&lc, fn, args));
    ++launches;
    last_grid_ = tiles * cl; last_steps_ = p.steps; last_nf_ = nf; last_cluster_ = cl > 1;
    return WRNN_OK;
  }

  int check() override {
    unsigned char buf[256];
    WRNN_CUDA_OK(cudaSetDevice(device));
    WRNN_CUDA_OK(cudaMemcpy(buf, d_sync_, 256, cudaMemcpyDeviceToHost));
    const int flag = reinterpret_cast<int*>(buf)[8];
    if (getenv("WRNN_STREAM_PROF") && last_steps_ > 0) {
      long long prof[16]; std::memcpy(prof, buf + 64, sizeof(prof));
      const long long n = last_steps_;
      fprintf(stderr, "[wrnn_stream prof] NF=%d cluster=%d CTAs=%d steps=%d mma/step=%d chunks/step=%d | consumer thread 0: operand-wait=%lld "
              "ring-wait=%lld mma=%lld epilogue=%lld (cycles per step)\n",
              last_nf_, last_cluster_ ? 4 : 1, last_grid_, last_steps_, n_mma_, n_chunks_, prof[0] / n, prof[1] / n, prof[2] / n, prof[3] / n);
    }
    if (flag != 0) { set_error("stream kernel aborted: an mbarrier wait (TMA / MMA / operand hand-off) timed out"); return WRNN_E_WATCHDOG; }
    return WRNN_OK;
  }

 private:
  Variant var_[4];
  void *d_vec_ = nullptr, *d_state_ = nullptr, *d_sync_ = nullptr;
  size_t state_bytes_ = 0, off_qk_ = 0, off_vq_ = 0, off_b1h_ = 0, off_b2h_ = 0, off_b3_ = 0;
  int n_chunks_ = 0, n_mma_ = 0, n_sm_ = 0, max_clusters_ = 0, last_grid_ = 0, last_steps_ = 0, last_nf_ = 0;
  bool last_cluster_ = false;
};

}  // namespace

int make_stream_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out) {
  if (!StreamEngine::supports_cfg(cfg)) {
    set_error("stream engine serves the MoL head (30 classes) and the 9-bit RAW head (512 classes) with fp16/bf16 operands");
    return WRNN_E_INVALID;
  }
  StreamEngine* e = new StreamEngine();
  e->cfg = cfg; e->device = device;
  const int rc = e->init(w);
  if (rc != WRNN_OK) { delete e; return rc; }
  *out = e;
  return WRNN_OK;
}

}  // namespace wrnn
