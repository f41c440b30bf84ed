// wrnn_epilogue.cu -- the tail of generate() on the device (SURVEY 8f-3): float64 mu-law expansion, equal-power
// cross-fade + overlap-add of the folds and the final fade-out (reference models/fatchord_version.py:243-258,
// :342-405; utils/dsp.py:98-103) in one pass over the (n_seg, seg_len) sample block the persistent kernel (or the
// all-gather) left in HBM.
//
// Bit-exactness with the host (numpy float64) epilogue is by construction: every weight the reference computes
// with a transcendental (sqrt of the fade windows, the 512-entry mu-law expansion, the linspace of the fade-out)
// is passed in as a float64 TABLE built by the caller with the reference's own numpy expressions; the kernel only
// converts fp32 -> fp64 (exact), multiplies and adds in the reference's order (folds ascending).
//
// HBM-bound and tiny: reads 4 B per fold-sample, writes 8 B per output sample.
#include <cuda_runtime.h>

#include <cstdint>

#include "wrnn_engine.h"

namespace wrnn {
namespace {

struct EpParams {
  const float* samples; int seg_len; long long seg_stride; int overlap;   // samples: [folds of every utterance, seg_len]
  const double* fade_in; const double* fade_out;      // [overlap] each (NULL when overlap == 0: unbatched)
  const double* mu_table; int n_classes;               // RAW + mu_law: expansion of label k (NULL = none)
  const double* tail; long long tail_len;              // final fade-out over the last tail_len samples of each utterance
  const EpUtt* utts; EpUtt one;                        // utterance table (device), or the one utterance when utts == NULL
};

__device__ __forceinline__ double fold_value(const EpParams& p, const float* s, int i, long long k) {
  const float xf = __ldg(s + (size_t)i * p.seg_len + k);
  double y = (double)xf;
  if (p.mu_table) {                                     // x = 2k/(n-1) - 1  ->  label k (exact: labels are 2/(n-1) apart)
    int lbl = __float2int_rn((xf + 1.0f) * (0.5f * (float)(p.n_classes - 1)));
    lbl = lbl < 0 ? 0 : (lbl >= p.n_classes ? p.n_classes - 1 : lbl);
    y = __ldg(p.mu_table + lbl);
  }
  if (k < p.overlap) y = __dmul_rn(y, __ldg(p.fade_in + k));                          // y[:, :overlap] *= fade_in   (:394)
  if (k >= p.seg_len - p.overlap) y = __dmul_rn(y, __ldg(p.fade_out + (k - (p.seg_len - p.overlap))));   // (:395)
  return y;
}

// Grid: (grid-stride blocks over the longest waveform, utterances); blockIdx.y unfolds utterance blockIdx.y alone.
__global__ void __launch_bounds__(256) wrnn_epilogue_kernel(const EpParams p) {
  const EpUtt u = p.utts ? p.utts[blockIdx.y] : p.one;
  const float* s = p.samples + (size_t)u.fold0 * p.seg_len;
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < u.wave_len; n += (long long)gridDim.x * blockDim.x) {
    long long i_hi = n / p.seg_stride;
    if (i_hi > u.n_seg - 1) i_hi = u.n_seg - 1;
    const long long k_hi = n - i_hi * p.seg_stride;
    double v = 0.0;                                      // unfolded = zeros; unfolded[...] += y[i], i ascending (:397-403)
    if (i_hi >= 1 && k_hi + p.seg_stride < p.seg_len) v = __dadd_rn(v, fold_value(p, s, (int)i_hi - 1, k_hi + p.seg_stride));
    if (k_hi < p.seg_len) v = __dadd_rn(v, fold_value(p, s, (int)i_hi, k_hi));
    if (p.tail && n >= u.wave_len - p.tail_len) v = __dmul_rn(v, __ldg(p.tail + (n - (u.wave_len - p.tail_len))));   // (:255-258)
    u.wav[n] = v;
  }
}

}  // namespace

// Shared by wrnn_epilogue (one utterance, passed by value) and wrnn_vocode_many (a device table of n_utts utterances).
int epilogue_launch(const float* samples, int seg_len, long long seg_stride, int overlap, const double* fade_in,
                    const double* fade_out, const double* mu_table, int n_classes, const double* tail, long long tail_len,
                    const EpUtt* utts, const EpUtt& one, int n_utts, long long max_wave_len, cudaStream_t stream) {
  EpParams p{samples, seg_len, seg_stride, overlap, fade_in, fade_out, mu_table, n_classes, tail, tail_len, utts, one};
  const long long blocks = (max_wave_len + 255) / 256;
  const int grid = grid_stride_blocks(blocks);
  wrnn_epilogue_kernel<<<dim3(grid, n_utts), 256, 0, stream>>>(p);
  WRNN_CUDA_OK(cudaGetLastError());
  return WRNN_OK;
}

}  // namespace wrnn

extern "C" int wrnn_epilogue(const float* samples, int32_t n_seg, int32_t seg_len, int64_t seg_stride, int32_t overlap,
                             const double* fade_in, const double* fade_out, const double* mu_table, int32_t n_classes,
                             const double* tail, int64_t tail_len, int64_t wave_len, double* wav, void* stream) {
  using namespace wrnn;
  if (!samples || !wav || n_seg <= 0 || seg_len <= 0 || seg_stride <= 0 || overlap < 0 || wave_len <= 0) {
    set_error("wrnn_epilogue: bad argument"); return WRNN_E_INVALID;
  }
  if (overlap > 0 && (!fade_in || !fade_out)) { set_error("wrnn_epilogue: fade tables are required when overlap > 0"); return WRNN_E_INVALID; }
  if (2 * (int64_t)overlap > seg_len) { set_error("wrnn_epilogue: overlap windows must not intersect"); return WRNN_E_INVALID; }
  if (wave_len > (int64_t)(n_seg - 1) * seg_stride + seg_len) { set_error("wrnn_epilogue: wave_len exceeds the unfolded length"); return WRNN_E_INVALID; }
  if (tail && (tail_len <= 0 || tail_len > wave_len)) { set_error("wrnn_epilogue: tail_len must be in (0, wave_len]"); return WRNN_E_INVALID; }
  if (mu_table && n_classes < 2) { set_error("wrnn_epilogue: n_classes"); return WRNN_E_INVALID; }
  return epilogue_launch(samples, seg_len, seg_stride, overlap, fade_in, fade_out, mu_table, n_classes, tail, tail_len, nullptr,
                         EpUtt{0, n_seg, wave_len, wav}, 1, wave_len, static_cast<cudaStream_t>(stream));
}
