// wrnn_mel.h -- the mel analysis object of wrnn_mel_create and its host-side checks (wrnn_mel.cu).
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/wavernn_b200.h"

struct wrnn_mel_plan {
  wrnn_mel_cfg cfg{};
  int device = 0;
  void* d_tabs = nullptr;   // [window n_fft | twiddles n_fft/2 x (re, im) | basis n_basis | bands] (wrnn::mel::Tabs),
                            // then the Griffin-Lim solve's [basis32 n_basis | inv_d n_mels | sub n_mels | bin_band]
  long long n_basis = 0;    // nonzero filterbank weights
  long long gl_off = 0;     // offset of basis32 in d_tabs, in doubles
  double gl_step = 0.0;     // 1 / lambda_max(A A^T) of the float32 filterbank A
};

namespace wrnn {
namespace mel {

// The configuration's ranges (WRNN_E_INVALID with a message); no CUDA call.
int check_cfg(const wrnn_mel_cfg* cfg);
// Checks a batch (WRNN_E_INVALID with a message naming the bad utterance; no CUDA call) and lays out its frame table:
// utterance i's frames are frame0[i] .. frame0[i + 1] - 1 of the launch, T_i = 1 + n_i / hop_length.
int plan(const wrnn_mel_cfg& cfg, const wrnn_mel_utt* u, int n_utts, std::vector<int64_t>& frame0);
// The same for wrnn_griffinlim_many: utterance i's frames are frame0[i] .. frame0[i + 1] - 1, T_i of them.
int gl_plan(const wrnn_mel_cfg& cfg, const wrnn_gl_utt* u, int n_utts, int n_iter, std::vector<int64_t>& frame0);

}  // namespace mel
}  // namespace wrnn
