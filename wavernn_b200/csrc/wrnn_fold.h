// wrnn_fold.h -- host-side algebra shared by every engine: "linear folding" of the
// conditioning path out of the recurrence, and the per-CTA row ownership.
//
// Reference step (models/fatchord_version.py:208-223), H = rnn_dims, x = previous sample,
// cond = [m_t (feat) | a1 | a2 | a3 | a4] (the row of mels_up concatenated with the row of aux):
//     x0 = I [x ; m ; a1] + bI                  = x*i0 + Ic cond[0:F1] + bI        (F1 = feat+aux)
//     gi1 = W1i x0 + b1i ,  gh1 = W1h h1 + b1h   -> h1' ;  x1 = x0 + h1'
//     gi2 = W2i [x1 ; a2] + b2i , gh2 = W2h h2 + b2h -> h2' ;  x2 = x1 + h2'
//     y1 = relu(F1 [x2 ; a3] + bf1) ; y2 = relu(F2 [y1 ; a4] + bf2) ; logits = F3 y2 + b3
// Everything that does not depend on the recurrent state is linear in (x, cond), so with
//     v1 = W1i i0, A1 = W1i Ic, k1 = W1i bI + b1i
//     v2 = W2x i0, A2 = W2x Ic, k2 = W2x bI + b2i         (W2x = W2i[:, :H], W2a = W2i[:, H:])
//     v3 = F1x i0, A3 = F1x Ic, k3 = F1x bI + bf1         (F1x = F1[:, :H],  F1a = F1[:, H:])
// the step becomes
//     gi1 = x v1 + A1 cond[0:F1] + k1
//     gi2 = W2x h1' + x v2 + A2 cond[0:F1] + W2a a2 + k2
//     y1  = relu(F1x h1' + F1x h2' + x v3 + A3 cond[0:F1] + F1a a3 + k3)
//     y2  = relu(F2x y1 + F2a a4 + bf2)
// i.e. per step only FOUR dependent K=H contractions remain on the critical path
// (h1'->gi2, h2'->y1, y1->y2, y2->logits); W1h h1' and W2h h2' ride along with them
// for the next step, and every conditioning term is one small K=(feat+4*aux)
// contraction  pre = Q cond + qk + x vq  that can run ahead of the recurrence.
// The products of matrices are formed here in double precision, so the folded path is
// not less accurate than the reference order (it removes one bf16 rounding of x0).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

namespace wrnn {

constexpr int H = 512;        // rnn_dims == fc_dims
constexpr int FEAT = 80;
constexpr int AUXD = 32;
constexpr int F1IN = FEAT + AUXD;          // 112: conditioning columns of I
constexpr int CDIM = FEAT + 4 * AUXD;      // 208: full conditioning row
constexpr int G3 = 3 * H;

struct HostWeights {   // fp32 copies of the state_dict tensors, row-major [out, in]
  std::vector<float> I_w, I_b, w1i, w1h, b1i, b1h, w2i, w2h, b2i, b2h, f1w, f1b, f2w, f2b, f3w, f3b;
  int n_classes = 0;
};

// Optional per-fold key of the in-kernel Philox draws (device table of n_seg entries, indexed by the job's fold).
// Without the table, fold f of a job draws with (counter fold = seg_first + f, key = philox_seed); with it, with
// (key[f].fold, key[f].seed) -- so a fold's draws follow its utterance, not its place in a batch (wrnn_vocode_many).
struct alignas(16) FoldKey {
  uint64_t seed;
  uint32_t fold;
  uint32_t pad;
};

// Dense folded model in double precision; row order is the reference's ([r,z,n] gate blocks).
struct Folded {
  std::vector<double> v1, k1, v2, k2, v3, k3;        // G3, G3, G3, G3, H, H
  std::vector<double> A1, A2, A3;                    // [G3][F1IN], [G3][F1IN], [H][F1IN]
};

inline void fold(const HostWeights& w, Folded& f) {
  f.v1.assign(G3, 0); f.k1.assign(G3, 0); f.v2.assign(G3, 0); f.k2.assign(G3, 0);
  f.v3.assign(H, 0); f.k3.assign(H, 0);
  f.A1.assign((size_t)G3 * F1IN, 0); f.A2.assign((size_t)G3 * F1IN, 0); f.A3.assign((size_t)H * F1IN, 0);
  const int IW = 1 + F1IN;            // I.weight row length (113)
  const int W2W = H + AUXD;           // rnn2.weight_ih / fc1 / fc2 row length (544)
  auto fold_rows = [&](const float* W, int ldw, int rows, const float* bias, double* v, double* k, double* A) {
    for (int r = 0; r < rows; ++r) {
      double sv = 0, sk = bias[r];
      double* Ar = A + (size_t)r * F1IN;
      for (int j = 0; j < H; ++j) {
        const double wj = W[(size_t)r * ldw + j];
        const float* Irow = w.I_w.data() + (size_t)j * IW;
        sv += wj * Irow[0];
        sk += wj * w.I_b[j];
        for (int c = 0; c < F1IN; ++c) Ar[c] += wj * Irow[1 + c];
      }
      v[r] = sv; k[r] = sk;
    }
  };
  fold_rows(w.w1i.data(), H, G3, w.b1i.data(), f.v1.data(), f.k1.data(), f.A1.data());
  fold_rows(w.w2i.data(), W2W, G3, w.b2i.data(), f.v2.data(), f.k2.data(), f.A2.data());
  fold_rows(w.f1w.data(), W2W, H, w.f1b.data(), f.v3.data(), f.k3.data(), f.A3.data());
}

// ---- row ownership: CTA c of P owns hidden units [c*U, (c+1)*U), U = H / P ------------
// Local row orders (j = unit within the CTA, g = gate 0/1/2 = r/z/n):
//   Q  (cond rows) : gi1(g,j) = g*U+j | gi2(g,j) = 3U+g*U+j | fc1(j) = 6U+j | fc2(j) = 7U+j   -> 8U rows
//   S1 (x h1')     : W2x(g,j) = g*U+j | W1h(g,j) = 3U+g*U+j | F1x(j) = 6U+j                    -> 7U rows
//   S2 (x h2')     : F1x(j) = j       | W2h(g,j) = U+g*U+j                                     -> 4U rows
//   S3 (x y1)      : F2x(j) = j                                                                -> U rows
struct RowMaps {
  static int q_rows(int U) { return 8 * U; }
  static int s1_rows(int U) { return 7 * U; }
  static int s2_rows(int U) { return 4 * U; }
  static int s3_rows(int U) { return U; }
};

// Fills dense per-CTA matrices in double, row-major [rows][K]; also the fp32 vectors.
struct CtaSlice {
  std::vector<double> Q, S1, S2, S3;     // [8U][CDIM], [7U][H], [4U][H], [U][H]
  std::vector<float> qk, vq;             // [8U]
  std::vector<float> b1h, b2h;           // [3U] gate-major (g*U+j)
};

inline void slice_for_cta(const HostWeights& w, const Folded& f, int cta, int U, CtaSlice& s) {
  const int u0 = cta * U;
  const int W2W = H + AUXD;
  s.Q.assign((size_t)8 * U * CDIM, 0); s.S1.assign((size_t)7 * U * H, 0);
  s.S2.assign((size_t)4 * U * H, 0); s.S3.assign((size_t)U * H, 0);
  s.qk.assign(8 * U, 0); s.vq.assign(8 * U, 0); s.b1h.assign(3 * U, 0); s.b2h.assign(3 * U, 0);
  for (int j = 0; j < U; ++j) {
    const int u = u0 + j;
    for (int g = 0; g < 3; ++g) {
      const int R = g * H + u;                 // reference row in the [r,z,n] stacks
      // Q: gi1
      { int q = g * U + j; for (int c = 0; c < F1IN; ++c) s.Q[(size_t)q * CDIM + c] = f.A1[(size_t)R * F1IN + c];
        s.qk[q] = (float)f.k1[R]; s.vq[q] = (float)f.v1[R]; }
      // Q: gi2 (cond[0:112] through A2, a2 = cond[112:144] through W2a)
      { int q = 3 * U + g * U + j; for (int c = 0; c < F1IN; ++c) s.Q[(size_t)q * CDIM + c] = f.A2[(size_t)R * F1IN + c];
        for (int c = 0; c < AUXD; ++c) s.Q[(size_t)q * CDIM + F1IN + c] = w.w2i[(size_t)R * W2W + H + c];
        s.qk[q] = (float)f.k2[R]; s.vq[q] = (float)f.v2[R]; }
      for (int k = 0; k < H; ++k) {
        s.S1[(size_t)(g * U + j) * H + k] = w.w2i[(size_t)R * W2W + k];
        s.S1[(size_t)(3 * U + g * U + j) * H + k] = w.w1h[(size_t)R * H + k];
        s.S2[(size_t)(U + g * U + j) * H + k] = w.w2h[(size_t)R * H + k];
      }
      s.b1h[g * U + j] = w.b1h[R];
      s.b2h[g * U + j] = w.b2h[R];
    }
    // Q: fc1 (A3 on cond[0:112], F1a on a3 = cond[144:176]) and fc2 (F2a on a4 = cond[176:208])
    { int q = 6 * U + j; for (int c = 0; c < F1IN; ++c) s.Q[(size_t)q * CDIM + c] = f.A3[(size_t)u * F1IN + c];
      for (int c = 0; c < AUXD; ++c) s.Q[(size_t)q * CDIM + F1IN + AUXD + c] = w.f1w[(size_t)u * W2W + H + c];
      s.qk[q] = (float)f.k3[u]; s.vq[q] = (float)f.v3[u]; }
    { int q = 7 * U + j; for (int c = 0; c < AUXD; ++c) s.Q[(size_t)q * CDIM + F1IN + 2 * AUXD + c] = w.f2w[(size_t)u * W2W + H + c];
      s.qk[q] = w.f2b[u]; s.vq[q] = 0.f; }
    for (int k = 0; k < H; ++k) {
      s.S1[(size_t)(6 * U + j) * H + k] = w.f1w[(size_t)u * W2W + k];
      s.S2[(size_t)j * H + k] = w.f1w[(size_t)u * W2W + k];
      s.S3[(size_t)j * H + k] = w.f2w[(size_t)u * W2W + k];
    }
  }
}

// round-to-nearest-even float -> bf16 bits (host)
inline uint16_t f2bf(float x) {
  uint32_t u; std::memcpy(&u, &x, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);   // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

// round-to-nearest-even float -> IEEE half bits, saturating to +-65504 (host)
inline uint16_t f2h(float x) {
  uint32_t u; std::memcpy(&u, &x, 4);
  const uint32_t sign = (u >> 16) & 0x8000u;
  u &= 0x7fffffffu;
  if (u > 0x7f800000u) return (uint16_t)(sign | 0x7e00u);          // NaN
  if (u >= 0x477ff000u) return (uint16_t)(sign | 0x7bffu);         // >= 65520 (rounds past max) -> 65504
  if (u < 0x33000001u) return (uint16_t)sign;                      // < 2^-25 (or == ties-to-even) -> 0
  int exp = (int)(u >> 23) - 127;
  uint32_t man = (u & 0x7fffffu) | 0x800000u;
  int shift; uint32_t base;
  if (exp >= -14) { shift = 13; base = (uint32_t)(exp + 15) << 10; man &= 0x7fffffu; }
  else { shift = 13 + (-14 - exp); base = 0; }                     // subnormal half
  uint32_t q = man >> shift, rem = man & ((1u << shift) - 1), half = 1u << (shift - 1);
  uint32_t h = base + q;
  if (rem > half || (rem == half && (h & 1u))) ++h;                // RNE (carry into exponent is correct)
  return (uint16_t)(sign | h);
}

}  // namespace wrnn
