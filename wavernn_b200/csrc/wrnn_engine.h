// wrnn_engine.h -- internal C++ interface between the C ABI (wrnn_capi.cu) and the engines.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <string>

#include "../../include/wavernn_b200.h"
#include "wrnn_fold.h"

namespace wrnn {

void set_error(const std::string& msg);          // thread-local last error (wrnn_capi.cu)

#define WRNN_CUDA_OK(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::wrnn::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e));           \
      return WRNN_E_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

// Grid of a grid-stride kernel: `blocks`, capped at 8 blocks per SM of the current device.
inline int grid_stride_blocks(long long blocks) {
  int dev = 0, n_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const long long cap = 8ll * (n_sm > 0 ? n_sm : 1);
  return (int)(blocks < cap ? blocks : cap);
}

class Engine {
 public:
  virtual ~Engine() {}
  virtual int generate(const wrnn_job& job, cudaStream_t stream) = 0;   // async
  virtual int check() = 0;                                              // after stream sync
  virtual bool supports(const wrnn_job& job) const { (void)job; return true; }   // job inside this engine's envelope?
  virtual const char* name() const = 0;
  virtual int grid_ctas() const = 0;
  int64_t launches = 0;
  int device = 0;
  wrnn_cfg cfg{};
};

// SIMT engine: CUDA-core FMA contractions, fp32-strict or bf16-operand arithmetic.
int make_simt_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// persistent tensor-core engine (wrnn_tc.cu): weights stationary in 128 SMs, wgmma contractions (fp16 / bf16 operands).
int make_tc_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// stream engine (wrnn_stream.cu): activation-stationary, weights streamed from L2; the throughput form for many folds
int make_stream_engine(const wrnn_cfg& cfg, const HostWeights& w, int device, Engine** out);
// conditioning pre-pass (wrnn_tc.cu): rows [row_lo, row_lo + n_rows) of the per-sample stream from frame-rate tensors
int expand_conditioning(const float* mel_frames, const float* aux_frames, const float* up_taps, int hop, long long row_lo,
                        long long n_rows, float* mels_up, float* aux, cudaStream_t stream);

}  // namespace wrnn

struct wrnn_handle {
  wrnn::Engine* engine = nullptr;          // engine chosen at create time
  wrnn::Engine* fallback = nullptr;        // ENGINE_AUTO only: SIMT engine, created on first job outside `engine`'s envelope
  wrnn::Engine* stream = nullptr;          // ENGINE_AUTO only: stream engine, created on the first job with many folds
  wrnn::Engine* last = nullptr;            // engine that served the most recent job
  wrnn::HostWeights* host_weights = nullptr;
  bool auto_engine = false;
  bool stream_failed = false;
  // staging for wrnn_generate_host
  void* d_stage = nullptr;
  size_t stage_bytes = 0;
};
