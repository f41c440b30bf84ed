// wrnn_cond.h -- the conditioning network (MelResNet with its BatchNorms folded) and the host-side pieces of
// wrnn_vocode: fold geometry and the float64 epilogue tables (wrnn_cond.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "wrnn_engine.h"

namespace wrnn {
namespace cond {

constexpr int CD = 128;                 // compute_dims == res_out_dims
constexpr int KIN = FEAT * 5;           // conv_in: k = 5 over 80 channels, k index = c*5 + j (torch's weight layout)
constexpr int TAPS = 5;                 // mel frames n/hop .. n/hop + 4 of the padded mel per output sample
constexpr double BN_EPS = 1e-5;

// Parameter blob (fp32 on the device, float64 as folded on the host); every matrix transposed to [k][out]:
//   conv_in  W [KIN][CD], b [CD]               (BatchNorm folded)
//   block r  W1 [CD][CD], b1 [CD], W2 [CD][CD], b2 [CD]   (batch_norm1 / batch_norm2 folded), r < res_blocks
//   conv_out W [CD][CD], b [CD]
inline size_t blob_len(int res_blocks) {
  return (size_t)KIN * CD + CD + (size_t)res_blocks * (2 * CD * CD + 2 * CD) + CD * CD + CD;
}

struct HostUpsampler {
  int res_blocks = 0, hop = 0;
  std::vector<double> blob;             // blob_len(res_blocks)
  std::vector<double> taps;             // [hop][TAPS]
};

// Reads and checks the upsample.* tensors, folds the BatchNorms and builds the tap table, all in double.
// host_only: the data pointers are host memory (no CUDA call is made).
int build_host_upsampler(const wrnn_upsample_cfg& cfg, const wrnn_tensor* t, int n, bool host_only, HostUpsampler& out);

struct Geometry {
  int64_t n_seg, seg_len, seg_stride, overlap, padded_len;
};
// fold_with_overlap's index math (fatchord_version.py:319-330); unbatched: one fold of total_len samples
Geometry fold_geometry(int64_t total_len, bool batched, int64_t target, int64_t overlap);

// The job wrnn_vocode_many runs, laid out on the host after the batch has been checked.  Utterance i's frames start
// at frame0[i] = sum_{j<i} (T_j + 4) of mel_frames / aux_frames, its conditioning rows at hop * frame0[i]; its folds
// are fold0[i] .. fold0[i+1] - 1 (batched: its own fold_with_overlap geometry; unbatched: one fold of max_T * hop steps),
// with the fold tables of wrnn_job and the Philox key (philox_seed_i, index within the utterance).  wav0[i] is its
// offset in the concatenation of the waveforms.
struct BatchPlan {
  Geometry g;                                 // seg_len, seg_stride, overlap shared; n_seg = folds of the whole batch
  int64_t L = 0;                              // rows of the laid-out stream: hop * sum (T_i + 4)
  int64_t max_T = 0, max_wave = 0;
  std::vector<int64_t> frame0, fold0, wav0;   // [n_utts + 1] each (last entry: the totals)
  std::vector<int64_t> row0, row_end;         // [n_seg]
  std::vector<FoldKey> keys;                  // [n_seg]
};
// Checks the batch (WRNN_E_INVALID with a message naming the bad utterance) and lays it out.
int batch_plan(int hop, const wrnn_vocode_batch& b, BatchPlan& out);
// The job wrnn_score_many runs: batch_plan's unbatched layout for utterances of n_i scored samples.  Utterance i is
// fold i, reading rows frame0[i] * hop + t (rows >= frame0[i] * hop + T_i * hop read as zeros) for max_i n_i steps
// (g.seg_len); wav0[i] is the offset of its n_i losses in the concatenation of the nll arrays.  keys are not used.
int score_plan(int hop, const wrnn_score_utt* utts, int n_utts, BatchPlan& out);

// generate()'s float64 epilogue tables, with numpy's arithmetic (linspace = i*step + start, last element = stop):
//   fade_in / fade_out [overlap] (xfade_and_unfold, :379-391; empty when overlap == 0), tail [20*hop] (:255),
//   mu [n_classes] (decode_mu_law of the fp32 class values, utils/dsp.py:98-103; empty without mu_law)
void epilogue_tables(int overlap, bool mu_law, int n_classes, int hop, std::vector<double>& fade_in,
                     std::vector<double>& fade_out, std::vector<double>& mu, std::vector<double>& tail);

}  // namespace cond

struct Upsampler {
  int device = 0, res_blocks = 0, hop = 0;
  float* d_blob = nullptr;              // cond::blob_len(res_blocks) fp32
  float* d_taps = nullptr;              // [hop][5] fp32
  // wrnn_vocode scratch: frames, samples and expanded rows (grown on demand), epilogue tables (cached by key)
  void* d_scratch = nullptr;
  size_t scratch_bytes = 0;
  std::vector<double> host_tabs;        // [fade_in | fade_out | mu | tail], kept alive for the asynchronous upload
  std::vector<unsigned char> host_plan; // a batch job's fold tables and utterance tables, uploaded in one copy
  double* d_tabs = nullptr;
  size_t tabs_len = 0;
  long long tabs_key[3] = {-1, -1, -1}; // overlap, mu_law, n_classes of the tables in d_tabs
  ~Upsampler();
};

// One utterance of a conditioning batch: mel [FEAT, T] (device); its padded mel and its MelResNet output are rows
// frame0 .. frame0 + T + 3 of mel_frames and frame0 .. frame0 + T - 1 of aux_frames.
struct CondUtt {
  const float* mel;
  long long T;
  long long frame0;
};

int make_upsampler(const cond::HostUpsampler& hu, int device, Upsampler** out);
// mel [FEAT, T] -> mel_frames [T + 4, FEAT], aux_frames [T, 128] (and up_taps [hop, 5] when not NULL); device, async
int conditioning_frames(const Upsampler& u, const float* mel, long long T, float* mel_frames, float* aux_frames,
                        float* up_taps, cudaStream_t stream);
// The same for n_utts utterances in one launch of each kernel: utts [n_utts] is a DEVICE table, max_T the longest T.
// Each utterance's frames are bit-identical to its own conditioning_frames.
int conditioning_frames_batch(const Upsampler& u, const CondUtt* utts, int n_utts, long long max_T, float* mel_frames,
                              float* aux_frames, cudaStream_t stream);

}  // namespace wrnn
