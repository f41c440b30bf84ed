// wrnn_stream_plan.h -- host side of the STREAM engine (wrnn_stream.cu): the packed weight stream and the static
// per-step MMA program one CTA interprets.  Pure C++ (no CUDA), so the packing and the schedule can be checked on a
// CPU-only box (wrnn_debug_stream_plan + tests/test_stream_plan.py interpret the program with numpy and compare it
// with the engine-arithmetic emulation oracle/contract.py).
//
// Decomposition ("activation-stationary"; the opposite of wrnn_tc.cu).  A CTA owns NF folds for the whole sequence
// and runs EVERY layer for them; nothing is exchanged between SMs.  The weights (7.4 MB as fp16) do not fit one SM,
// so they are streamed from L2 every step, in the order the step consumes them, through a shared-memory ring (TMA
// bulk copies; every CTA of the grid reads the same stream, which the 50 MB L2 serves to every SM).  Contractions are
// "swap-AB": the weight rows are the MMA M dimension (tiles of 128 rows, two wgmma M tiles of 64), the CTA's folds are
// N (NF = 16 or 32), D[rows, folds] += W[rows, k0:k0+16] * act[folds, k0:k0+16]^T.
// A GRU unit's r / z / n pre-activations sit in the SAME fragment position of different accumulators, so the gate math is
// thread-local (one thread per unit row, NF folds each).
//
// Per step (folded algebra of wrnn_fold.h; reference models/fatchord_version.py:208-223), unit blocks b = 0..3 of 128:
//   P1 GRU1 :  acc r,z = Q1[g,b] cond + W1h[g,b] h1   | acc in = Q1[n,b] cond          | acc hn = W1h[n,b] h1
//   P2 GRU2 :  acc r,z = Q2[g,b] cond + W2h[g,b] h2 + W2x[g,b] h1' | acc in = Q2[n,b] cond + W2x[n,b] h1' | acc hn = W2h[n,b] h2
//   P3 fc1  :  acc = Q3[b] cond + F1x[b] h1' + F1x[b] h2'      (one streamed F1x chunk feeds two MMAs)
//   P4 fc2  :  acc = Q4[b] cond + F2x[b] y1
//   P5 fc3  :  acc = F3 y2        (MoL: 30 rows in one 128-row tile; RAW: 512 rows, four unit blocks like fc1 / fc2)
// The program lists the weight chunks in exactly this order; within P2 every chunk that does not depend on h1' is
// issued first, so those MMAs (and the epilogue-free h2 reads) overlap the P1 gate math.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "wrnn_fold.h"

namespace wrnn {
namespace stream {

constexpr int MROWS = 128;          // weight rows per streamed chunk (two wgmma M tiles)
constexpr int KCH = 64;             // K elements per streamed chunk (4 MMAs of K = 16)
constexpr int CHUNK_BYTES = MROWS * KCH * 2;   // 16 KB: one chunk
constexpr int PAIR_BYTES = 2 * CHUNK_BYTES;    // 32 KB ring slot: chunks are loaded two at a time (halves the producer's work per byte)

// B operand (activation image) selectors
enum : uint8_t { B_COND = 0, B_H1PREV = 1, B_H1NEW = 2, B_H2 = 3, B_Y1 = 4, B_Y2 = 5, B_NONE = 0xff };
// readiness barriers an issuer may have to wait for before a chunk
enum : uint8_t { W_NONE = 0, W_COND = 1, W_H1NEW = 2, W_H2NEW = 3, W_Y1 = 4, W_Y2 = 5 };
enum : uint8_t { F_FIRST = 1, F_COND_RELEASE = 2 };
constexpr int N_ISSUERS = 4;        // owners: every accumulator chain of a (phase, block) belongs to exactly one of them
constexpr int N_PHASES = 5;

struct Chunk {            // 16 bytes, read as one uint4
  uint16_t size16;        // size of this chunk in the weight stream in 16-byte units (chunks are consecutive): 128 rows x (16*nk) x 2 B
  uint16_t a_off16;       // where the chunk lands inside its ring slot (16-byte units): chunks travel in PAIRS (one TMA, one
                          // barrier per pair), the second chunk of a pair sits right behind the first
  uint8_t acc;            // accumulator index: 4 * block + owner
  uint8_t nk;             // K = 16 steps in this chunk
  uint8_t b_buf;          // B operand image (B_*)
  uint8_t b_buf2;         // second B operand for the same weight chunk (fc1: h2'), B_NONE otherwise
  uint16_t k0;            // K offset of the chunk inside the B image (elements)
  uint8_t flags;          // F_FIRST: first MMA of the accumulator in this phase overwrites; F_COND_RELEASE: this issuer's last cond read
  uint8_t wait_b;         // W_* | block << 4: readiness barrier to wait for before issuing.  h1', h2' and y1 become ready BLOCK by
                          // block (128 units = 128 K columns each), y2 too (in the cluster form each CTA delivers its own block): a chunk waits only for
                          // the block its K range reads
  uint8_t wait_acc;       // 0, or block + 1: first chunk of this issuer in (phase, block): the previous phase's epilogue must have drained the block
  uint8_t commit;         // 0, or block + 1: last chunk of this issuer in (phase, block): signal "my accumulators of the block are full"
  uint8_t owner;          // owner 0..3 (the accumulator within its (phase, block) group)
  uint8_t phase;          // 0..4 (P1..P5)
};
static_assert(sizeof(Chunk) == 16, "Chunk must stay one uint4");

struct Plan {
  std::vector<uint8_t> blob;      // the weight stream: chunk images back to back (fp16 / bf16 bits), in program order
  std::vector<Chunk> prog;        // one step of the program, in stream order (what the producer walks)
  std::vector<uint16_t> mine[N_ISSUERS];   // per issuing warp: indices into prog, ascending
  std::vector<float> qk, vq;      // [4096] conditioning-row constants, row order gi1 | gi2 | fc1 | fc2 (gate-major inside the GRUs)
  std::vector<float> b1h, b2h;    // [1536] gate-major
  std::vector<float> b3;          // [n_classes padded to a multiple of 128]
  int n_classes = 0;
  int n_mma = 0;                  // MMA instructions per step (for the roofline bookkeeping)
};

// K-major no-swizzle operand image of a [128 x kc] tile: element (r, k) at (r/8)*(kc/8)*64 + (k/8)*64 + (r%8)*8 + k%8
inline size_t tile_index(int r, int k, int kc) { return (size_t)(r / 8) * (kc / 8) * 64 + (size_t)(k / 8) * 64 + (r % 8) * 8 + (k % 8); }

// Builds the plan.  `bf` selects bf16 instead of fp16 operand bits.  n_classes <= 128 (MoL: 30: one fc3 block) or
// 512 (RAW: four fc3 blocks of 128 classes, in class order, each like an fc1 / fc2 block).
//
// Ownership (one owner per accumulator chain, four chains per unit block in every phase; the stream order below
// interleaves the four owners' chunks -- the kernel regroups them per owner, see compile_device):
//   GRU phases : warp 0 = r, 1 = z, 2 = in (input-side n), 3 = hn (hidden-side n)            accumulators 4b + q
//   fc phases  : the K dimension is split in four: warp q owns conditioning K-chunk q and K = [128q, 128q + 128) of the
//                recurrent operand, into its own partial accumulator 4b + q (the epilogue adds the four partials)
// Stream order: the chains of one (phase, block) are interleaved round-robin, so consecutive ring slots go to different
// warps; within P2 everything that does not depend on h1' is issued (for all blocks) before the W2x h1' chunks.
// `only_block` >= 0 builds the program of ONE 128-unit block of every layer (accumulator set = phase, see ab() below;
// MoL's fc3 only for block 0, RAW's fc3 block r for block r): the share of CTA `only_block` of a 4-CTA cluster that splits the rows of every layer
// (wrnn_stream.cu, cluster form).  Operand readiness codes (wait_b) keep the GLOBAL block of the K range they read.
inline void build_plan(const HostWeights& w, bool bf, Plan& p, int only_block = -1) {
  Folded f; fold(w, f);
  CtaSlice s; slice_for_cta(w, f, 0, H, s);          // P = 1: the dense matrices in the row order documented in wrnn_fold.h
  auto cvt = [&](double v) -> uint16_t { return bf ? f2bf((float)v) : f2h((float)v); };
  p.blob.clear(); p.prog.clear(); p.n_mma = 0;
  for (auto& m : p.mine) m.clear();
  p.n_classes = w.n_classes;
  p.qk = s.qk; p.vq = s.vq; p.b1h = s.b1h; p.b2h = s.b2h;
  const bool raw = w.n_classes > MROWS;                    // RAW: fc3 in four unit blocks
  const int NC3 = raw ? (w.n_classes + MROWS - 1) / MROWS * MROWS : MROWS;   // fc3 rows, zero-padded
  p.b3.assign(NC3, 0.f);
  for (int r = 0; r < w.n_classes && r < NC3; ++r) p.b3[r] = w.f3b[r];

  struct Pending { Chunk c; std::vector<uint16_t> img; };
  std::vector<Pending> q[N_ISSUERS];
  bool fresh[N_ISSUERS] = {true, true, true, true};       // no chunk of this issuer yet in the current (phase, block)

  // queues the chunks of rows [row0, row0 + 128) x columns [kbeg, kend) of a dense row-major [rows][K] matrix for `owner`
  auto emit = [&](int owner, int phase, int blk, const double* M, int K, int n_rows_valid, int row0, int kbeg, int kend, uint8_t acc,
                  uint8_t b_buf, uint8_t b_buf2, bool& first, uint8_t wait_b) {
    for (int k0 = kbeg; k0 < kend; k0 += KCH) {
      const int kc = (kend - k0 < KCH) ? (kend - k0) : KCH;        // 64, or the 16-wide tail of K = 208
      Pending pd;
      pd.img.assign((size_t)MROWS * kc, 0);
      for (int r = 0; r < MROWS; ++r) {
        if (row0 + r >= n_rows_valid) continue;                    // rows beyond the matrix stay zero (fc3: 30 of 128)
        for (int k = 0; k < kc; ++k) pd.img[tile_index(r, k, kc)] = cvt(M[(size_t)(row0 + r) * K + k0 + k]);
      }
      Chunk c{};
      c.size16 = (uint16_t)(MROWS * kc * 2 / 16); c.a_off16 = 0; c.acc = acc; c.nk = (uint8_t)(kc / 16); c.b_buf = b_buf; c.b_buf2 = b_buf2;
      c.k0 = (uint16_t)k0; c.flags = first ? F_FIRST : 0; c.wait_acc = fresh[owner] ? (uint8_t)(blk + 1) : 0;
      c.wait_b = wait_b;
      if (wait_b >= W_H1NEW) c.wait_b = (uint8_t)(wait_b | ((k0 / MROWS) << 4));   // per-block readiness (h1', h2', y1, y2)
      c.commit = 0; c.owner = (uint8_t)owner; c.phase = (uint8_t)phase;
      first = false; fresh[owner] = false;
      pd.c = c;
      q[owner].push_back(std::move(pd));
      p.n_mma += c.nk * (b_buf2 == B_NONE ? 1 : 2);
    }
  };
  auto mark_commit = [&](int owner, int blk) { q[owner].back().c.commit = (uint8_t)(blk + 1); };
  // appends the queued chunks to the stream, round-robin over the issuers TWO chunks at a time: chunks travel through the
  // ring in pairs (one TMA, one full / empty barrier per pair) and both chunks of a pair belong to the same issuer, which
  // therefore pays the ring hand-shake once per eight MMAs.  Every flush group has an even chunk count per issuer.
  auto flush = [&]() {
    size_t pos[N_ISSUERS] = {0, 0, 0, 0};
    for (bool any = true; any;) {
      any = false;
      for (int o = 0; o < N_ISSUERS; ++o) {
        if (pos[o] >= q[o].size()) continue;
        any = true;
        for (int j = 0; j < 2 && pos[o] < q[o].size(); ++j) {
          Pending& pd = q[o][pos[o]++];
          p.mine[o].push_back((uint16_t)p.prog.size());
          if (p.prog.size() & 1) pd.c.a_off16 = p.prog.back().size16;     // second chunk of a pair
          p.prog.push_back(pd.c);
          const size_t base = p.blob.size();
          p.blob.resize(base + pd.img.size() * 2);
          std::memcpy(p.blob.data() + base, pd.img.data(), pd.img.size() * 2);
        }
      }
    }
    for (auto& v : q) v.clear();
  };
  auto new_block = [&]() { for (bool& b : fresh) b = true; };

  const double* Q = s.Q.data();         // [8H][CDIM]: gi1 (g*H+u) | gi2 (3H + g*H+u) | fc1 (6H+u) | fc2 (7H+u)
  const double* S1 = s.S1.data();       // [7H][H]: W2x (g*H+u) | W1h (3H + g*H+u) | F1x (6H+u)
  const double* S2 = s.S2.data();       // [4H][H]: F1x (u) | W2h (H + g*H+u)
  const double* S3 = s.S3.data();       // [H][H] : F2x
  const double* W2x = S1; const double* W1h = S1 + (size_t)3 * H * H; const double* F1x = S1 + (size_t)6 * H * H;
  const double* W2h = S2 + (size_t)H * H; const double* F2x = S3;
  const int NB = H / MROWS;             // 4 unit blocks
  const int B0 = only_block >= 0 ? only_block : 0, B1 = only_block >= 0 ? only_block + 1 : NB;     // blocks of this program
  // block id used for accumulators and their barriers: the unit block, or -- one-block programs -- the PHASE (P1..P4 ->
  // sets 0..3, fc3 -> set 0 again): nothing else is computed in the other three, and with a set per phase the
  // MMAs of a phase never wait for the previous phase's epilogue to drain.
  auto ab = [&](int b, int phase) -> int { return only_block >= 0 ? (phase & 3) : b; };
  std::vector<double> F3((size_t)NC3 * H, 0.0);
  for (int r = 0; r < w.n_classes && r < NC3; ++r) for (int k = 0; k < H; ++k) F3[(size_t)r * H + k] = w.f3w[(size_t)r * H + k];
  const int QK[5] = {0, 64, 128, 192, CDIM};              // the four K-chunks of a conditioning row (64, 64, 64, 16)

  // ---- P1: GRU1 (phase 0).  Accumulators of block b: 4b + {0: r, 1: z, 2: in, 3: hn}
  for (int b = B0; b < B1; ++b) {
    new_block();
    for (int g = 0; g < 2; ++g) {                                  // r, z: conditioning + recurrent part in one accumulator
      bool first = true;
      emit(g, 0, ab(b, 0), Q, CDIM, 8 * H, g * H + b * MROWS, 0, CDIM, (uint8_t)(4 * ab(b, 0) + g), B_COND, B_NONE, first, W_COND);
      emit(g, 0, ab(b, 0), W1h, H, 3 * H, g * H + b * MROWS, 0, H, (uint8_t)(4 * ab(b, 0) + g), B_H1PREV, B_NONE, first, W_NONE);
      mark_commit(g, ab(b, 0));
    }
    { bool first = true; emit(2, 0, ab(b, 0), Q, CDIM, 8 * H, 2 * H + b * MROWS, 0, CDIM, (uint8_t)(4 * ab(b, 0) + 2), B_COND, B_NONE, first, W_COND); mark_commit(2, ab(b, 0)); }
    { bool first = true; emit(3, 0, ab(b, 0), W1h, H, 3 * H, 2 * H + b * MROWS, 0, H, (uint8_t)(4 * ab(b, 0) + 3), B_H1PREV, B_NONE, first, W_NONE); mark_commit(3, ab(b, 0)); }
    flush();
  }
  // ---- P2: GRU2 (phase 1).  First everything that does not need h1' (overlaps the P1 gate math), then W2x h1'.
  for (int b = B0; b < B1; ++b) {
    new_block();
    for (int g = 0; g < 3; ++g) {
      bool first = true;
      emit(g, 1, ab(b, 1), Q, CDIM, 8 * H, 3 * H + g * H + b * MROWS, 0, CDIM, (uint8_t)(4 * ab(b, 1) + g), B_COND, B_NONE, first, W_COND);
      if (g < 2) emit(g, 1, ab(b, 1), W2h, H, 3 * H, g * H + b * MROWS, 0, H, (uint8_t)(4 * ab(b, 1) + g), B_H2, B_NONE, first, W_NONE);
    }
    { bool first = true; emit(3, 1, ab(b, 1), W2h, H, 3 * H, 2 * H + b * MROWS, 0, H, (uint8_t)(4 * ab(b, 1) + 3), B_H2, B_NONE, first, W_NONE); mark_commit(3, ab(b, 1)); }
    flush();
  }
  for (int b = B0; b < B1; ++b) {
    for (bool& fr : fresh) fr = false;                             // the accumulators were opened by the independent part
    for (int g = 0; g < 3; ++g) {
      bool first = false;
      emit(g, 1, ab(b, 1), W2x, H, 3 * H, g * H + b * MROWS, 0, H, (uint8_t)(4 * ab(b, 1) + g), B_H1NEW, B_NONE, first, W_H1NEW);
      mark_commit(g, ab(b, 1));
    }
    flush();
  }
  // ---- P3 / P4: fc1 (phase 2), fc2 (phase 3): K split over the four issuers, partial accumulators 4b + q
  for (int layer = 0; layer < 2; ++layer) {
    const double* F = layer ? F2x : F1x;
    for (int b = B0; b < B1; ++b) {
      new_block();
      for (int o = 0; o < N_ISSUERS; ++o) {
        bool first = true;
        emit(o, 2 + layer, ab(b, 2 + layer), Q, CDIM, 8 * H, (6 + layer) * H + b * MROWS, QK[o], QK[o + 1], (uint8_t)(4 * ab(b, 2 + layer) + o), B_COND, B_NONE, first, W_COND);
        if (layer == 1 && b == B1 - 1) q[o].back().c.flags |= F_COND_RELEASE;      // this issuer's last read of the step's conditioning
        if (layer == 0) emit(o, 2, ab(b, 2 + layer), F, H, H, b * MROWS, 128 * o, 128 * o + 128, (uint8_t)(4 * ab(b, 2 + layer) + o), B_H1NEW, B_H2, first, W_H2NEW);
        else emit(o, 3, ab(b, 2 + layer), F, H, H, b * MROWS, 128 * o, 128 * o + 128, (uint8_t)(4 * ab(b, 2 + layer) + o), B_Y1, B_NONE, first, W_Y1);
        mark_commit(o, ab(b, 2 + layer));
      }
    }
    flush();            // per layer: 3 chunks per issuer and block -> 12 per issuer, even (one-block programs: 3, their ring slots hold one chunk)
  }
  // ---- P5: fc3 (phase 4).  RAW: classes [128b, 128b + 128) are unit block b, K split over the four issuers like fc1 /
  // fc2 (partial accumulators 4b + q, two chunks each); every chunk waits for the y2 block its K range reads.
  if (raw) {
    for (int b = B0; b < B1; ++b) {
      new_block();
      for (int o = 0; o < N_ISSUERS; ++o) {
        bool first = true;
        emit(o, 4, ab(b, 4), F3.data(), H, NC3, b * MROWS, 128 * o, 128 * o + 128, (uint8_t)(4 * ab(b, 4) + o), B_Y2, B_NONE, first, W_Y2);
        mark_commit(o, ab(b, 4));
      }
      flush();
    }
  } else if (only_block <= 0) {
    // MoL: partial accumulators 0..3 of block 0
    new_block();
    for (int o = 0; o < N_ISSUERS; ++o) {
      bool first = true;
      emit(o, 4, 0, F3.data(), H, MROWS, 0, 128 * o, 128 * o + 128, (uint8_t)o, B_Y2, B_NONE, first, W_Y2);
      mark_commit(o, 0);
    }
    flush();
  }
}

// ---- what the kernel reads -----------------------------------------------------------------------------------------
// The kernel's consumer warpgroups accumulate ONE chain at a time in registers and keep the finished chains of the current
// (phase, block) until that block's epilogue, which they run as soon as its last chunk is done.  So they consume the
// program grouped by (phase, block) and, inside a group, by accumulator: a stable reordering of the stream that keeps the
// order of every accumulator's chunks (hence its floating-point sums) and only moves chunks of other accumulators (of P2:
// the h1'-independent chunks of block b next to the W2x h1' chunks of block b).  The producer loads the chunks in that
// order from their places in the weight stream.  Since block b's GRU2 epilogue now runs before block b+1's W2h h2
// chunks, h2 ping-pongs (H0 / H1) in both forms, and y2 goes to the stale h2 image.
// Every record is exactly four K = 16 MMAs (no branch around the MMAs: a branch makes the compiler serialize them):
// the K = 16 tail of the conditioning row multiplies a zero operand in its last three, and an fc1 chunk, which feeds
// h1' and h2', becomes two records on the same ring slot.
enum : uint8_t { DF_FIRST = 1, DF_COND_RELEASE = 2, DF_B_COND = 4, DF_NK1 = 8, DF_SAME_SLOT = 16, DF_END = 32, DF_ACC_END = 64,
                 DF_KEEP_SLOT = 128 };
struct DevChunk {
  uint32_t src16;         // offset of the chunk in the weight stream, >> 4 (its size: 4 KB if DF_NK1, else 16 KB)
  uint16_t b_lo[2];       // B operand start (byte offset from the start of dynamic shared memory, >> 4), step parity 0 / 1
  uint8_t acc;            // accumulator of the (phase, block) group: 0..3 (the plan's owner)
  uint8_t flags;          // DF_*: SAME_SLOT = operand of the previous record's slot (no load), KEEP_SLOT = the next record
                          // reuses this slot, ACC_END / END = last record of its accumulator / of its (phase, block) group,
                          // COND_RELEASE = last conditioning read of the step
  uint8_t wait_b;         // W_* | block << 4: readiness barrier to wait for before issuing
  uint8_t phase_blk;      // phase | (global unit block) << 4
  uint32_t reserved;      // keeps the record one uint4
};
static_assert(sizeof(DevChunk) == 16, "DevChunk must stay one uint4");

// byte offsets of the operand images: h1 and h2 ping-pong (X[cur] / H[cur] hold the previous step's values), y1 goes
// to the stale h1 image X[cur], y2 to the stale h2 image H[cur]
struct SmemLayout { int off_x0, off_x1, off_h2[2], off_cond, cond_bytes; };

// `block`: the unit block of a one-block program (cluster rank), or -1 for the whole program
inline void compile_device(const Plan& p, const SmemLayout& L, int block, std::vector<DevChunk>& d) {
  d.clear();
  auto base_of = [&](uint8_t buf, int cur, int phase) -> int {
    switch (buf) {
      case B_COND: return L.off_cond + cur * L.cond_bytes;
      case B_H1NEW: return cur ? L.off_x0 : L.off_x1;
      case B_H2: return L.off_h2[phase <= 1 ? cur : cur ^ 1];       // GRU2 reads the previous h2 (H[cur]), fc1 the new one (H[cur^1])
      case B_Y2: return L.off_h2[cur];
      default: return cur ? L.off_x1 : L.off_x0;          // B_H1PREV, B_Y1
    }
  };
  std::vector<size_t> src(p.prog.size() + 1, 0);
  for (size_t i = 0; i < p.prog.size(); ++i) src[i + 1] = src[i] + (size_t)p.prog[i].size16;
  auto group = [&](const Chunk& c) { return c.phase * 4 + c.acc / 4; };
  std::vector<size_t> order(p.prog.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) {
    const Chunk &x = p.prog[a], &y = p.prog[b];
    return group(x) != group(y) ? group(x) < group(y) : x.acc % 4 < y.acc % 4;
  });
  int last_cond = -1;
  for (size_t j = 0; j < order.size(); ++j) {
    const Chunk& c = p.prog[order[j]];
    const bool last_of_group = j + 1 == order.size() || group(p.prog[order[j + 1]]) != group(c);
    const bool last_of_acc = last_of_group || p.prog[order[j + 1]].acc != c.acc;
    for (int part = 0; part < (c.b_buf2 == B_NONE ? 1 : 2); ++part) {
      const uint8_t buf = part ? c.b_buf2 : c.b_buf;
      const bool last = c.b_buf2 == B_NONE || part == 1;
      DevChunk r{};
      r.src16 = (uint32_t)src[order[j]];
      for (int cur = 0; cur < 2; ++cur) r.b_lo[cur] = (uint16_t)((base_of(buf, cur, c.phase) + c.k0 * 16) >> 4);
      r.acc = (uint8_t)(c.acc % 4);
      r.flags = (uint8_t)(((c.flags & F_FIRST) && part == 0 ? DF_FIRST : 0) | (buf == B_COND ? DF_B_COND : 0) | (c.nk == 1 ? DF_NK1 : 0) |
                          (part == 1 ? DF_SAME_SLOT : 0) | (!last ? DF_KEEP_SLOT : 0) | (last && last_of_acc ? DF_ACC_END : 0) |
                          (last && last_of_group ? DF_END : 0));
      r.wait_b = c.wait_b;
      r.phase_blk = (uint8_t)(c.phase | ((block >= 0 ? block : c.acc / 4) << 4));
      if (buf == B_COND) last_cond = (int)d.size();
      d.push_back(r);
    }
  }
  if (last_cond >= 0) d[last_cond].flags |= DF_COND_RELEASE;
}

}  // namespace stream
}  // namespace wrnn
