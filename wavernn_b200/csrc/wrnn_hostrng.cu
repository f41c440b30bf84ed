// Host-side replay of torch's default CPU generator (MT19937) for parity mode.
//
// The reference draws all of its randomness from torch's global CPU generator: two nn.GRUCell constructions per
// generate() call (fatchord_version.py:178-179 -> :266-271; reset_parameters() draws one uniform per parameter
// element, 3.2 M values that are thrown away) and then 11 uniforms per fold and step inside the loop
// (utils/distribution.py:106,118).  Reproducing that stream with torch operators costs ~30 ms of single-thread CPU
// time per call -- a large share of the whole GPU job.  Here the discarded part is skipped with bare state twists (no
// tempering, no stores) and the used part is written straight into the caller's (pinned) staging buffer.
//
// The caller (wavernn_b200/vocoder.py) reads / writes the generator state through torch.get_rng_state() /
// set_rng_state() and self-checks this routine against torch before trusting it.
#include <cmath>
#include <cstdint>

#include "../../include/wavernn_b200.h"

namespace {

constexpr int N = 624, M = 397;
constexpr uint32_t UPPER = 0x80000000u, LOWER = 0x7fffffffu, MAG = 0x9908b0dfu;

inline uint32_t mix(uint32_t a, uint32_t b, uint32_t far) {
  const uint32_t y = (a & UPPER) | (b & LOWER);
  return far ^ (y >> 1) ^ ((0u - (y & 1u)) & MAG);
}

// next block of 624 words, in place.  The first loop only reads words that are still old, the second reads words
// written at least 227 iterations earlier: both vectorise (8 words per instruction with AVX2 -- the skipped / foreign
// part of the draw matrix of a sharded job costs one twist per 624 words, so this loop IS the replay's cost).
inline __attribute__((always_inline)) void twist_body(uint32_t* __restrict__ mt) {
  int i = 0;
  for (; i < N - M; ++i) mt[i] = mix(mt[i], mt[i + 1], mt[i + M]);
  for (; i < N - 1; ++i) mt[i] = mix(mt[i], mt[i + 1], mt[i + M - N]);
  mt[N - 1] = mix(mt[N - 1], mt[0], mt[M - 1]);
}
#if defined(__x86_64__)
__attribute__((target("avx2"))) void twist_avx2(uint32_t* __restrict__ mt) { twist_body(mt); }
#endif
void twist_base(uint32_t* __restrict__ mt) { twist_body(mt); }
using twist_fn = void (*)(uint32_t*);
twist_fn pick_twist() {
#if defined(__x86_64__)
  if (__builtin_cpu_supports("avx2")) return twist_avx2;
#endif
  return twist_base;
}
const twist_fn twist = pick_twist();

inline uint32_t temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// One body, two instantiations: with the FMA unit (every x86-64 host an H100 sits in) the conversion is one
// instruction per draw; otherwise libm's correctly rounded fmaf gives the same bits.
template <bool HW>
inline __attribute__((always_inline)) void convert_body(const uint32_t* s, float* o, uint64_t take, float range, float lo) {
  constexpr float kInv = 1.0f / 16777216.0f;
  for (uint64_t i = 0; i < take; ++i) {
    const float x = (float)(int32_t)(temper(s[i]) & 0xffffffu) * kInv;
    o[i] = HW ? __builtin_fmaf(x, range, lo) : std::fmaf(x, range, lo);
  }
}
template <bool HW> void convert(const uint32_t* s, float* o, uint64_t take, float range, float lo);
#if defined(__x86_64__)
template <> __attribute__((target("fma,avx2"))) void convert<true>(const uint32_t* s, float* o, uint64_t take, float range, float lo) {
  convert_body<true>(s, o, take, range, lo);
}
#else
template <> void convert<true>(const uint32_t* s, float* o, uint64_t take, float range, float lo) { convert_body<false>(s, o, take, range, lo); }
#endif
template <> void convert<false>(const uint32_t* s, float* o, uint64_t take, float range, float lo) { convert_body<false>(s, o, take, range, lo); }

// position in the generator's output stream + the two operations the replay needs
struct Stream {
  uint32_t* state; int32_t pos; float range, lo; bool hw;
  Stream(uint32_t* st, int32_t p, float lo_, float hi_) : state(st), pos(p), range(hi_ - lo_), lo(lo_) {
#if defined(__x86_64__)
    hw = __builtin_cpu_supports("fma") && __builtin_cpu_supports("avx2");
#else
    hw = false;
#endif
  }
  void skip(uint64_t n) {                                // discard: whole blocks cost one twist each
    while (n) {
      if (pos == N) { twist(state); pos = 0; }
      const uint64_t take = n < (uint64_t)(N - pos) ? n : (uint64_t)(N - pos);
      pos += (int32_t)take;
      n -= take;
    }
  }
  // torch's uniform_real<float>: x = (y & (2^24 - 1)) * 2^-24 ; x * (hi - lo) + lo with one rounding (its CPU kernels
  // are built with FMA contraction)
  void draw(float* out, uint64_t n) {
    uint64_t done = 0;
    while (done < n) {
      if (pos == N) { twist(state); pos = 0; }
      const uint64_t take = (n - done) < (uint64_t)(N - pos) ? (n - done) : (uint64_t)(N - pos);
      if (hw) convert<true>(state + pos, out + done, take, range, lo);
      else convert<false>(state + pos, out + done, take, range, lo);
      pos += (int32_t)take;
      done += take;
    }
  }
};

}  // namespace

extern "C" int32_t wrnn_mt19937_uniform(uint32_t* state, int32_t pos, uint64_t skip, float* out, uint64_t n, float lo, float hi) {
  if (!state || pos < 0 || pos > N || (n && !out)) return -1;
  Stream s(state, pos, lo, hi);
  s.skip(skip);
  s.draw(out, n);
  return s.pos;
}

extern "C" int32_t wrnn_mt19937_uniform_cols(uint32_t* state, int32_t pos, uint64_t skip, float* out, uint64_t n_rows, uint64_t row_len,
                                             uint64_t a_lo, uint64_t a_hi, uint64_t b_lo, uint64_t b_hi, float lo, float hi) {
  if (!state || pos < 0 || pos > N || a_lo > a_hi || a_hi > b_lo || b_lo > b_hi || b_hi > row_len) return -1;
  if (!out && n_rows && (a_hi - a_lo) + (b_hi - b_lo) > 0) return -1;
  Stream s(state, pos, lo, hi);
  s.skip(skip);
  const uint64_t wa = a_hi - a_lo, wb = b_hi - b_lo;
  for (uint64_t r = 0; r < n_rows; ++r) {
    float* o = out + r * (wa + wb);
    s.skip(a_lo);
    s.draw(o, wa);
    s.skip(b_lo - a_hi);
    s.draw(o + wa, wb);
    s.skip(row_len - b_hi);
  }
  return s.pos;
}
