// Native gradient-ready -> bucket-launch sequencing (SURVEY.md N2: the reference's torch binding of Horovod —
// `hvd.DistributedOptimizer` registers one hook per parameter, horovod/torch/optimizer.py, and the C++ core decides what
// is communicated when, PyTorch_benchmark/src/pytorch_synthetic_benchmark.py:72-74).
//
// One StepLauncher per optimizer.  The per-parameter autograd hook IS StepLauncher::on_ready (bound as a C++ callable):
// it counts the parameter into its bucket and, strictly in plan order (so that every rank issues the same kernel
// sequence), launches each bucket whose parameters are all ready — event-joins the compute stream and the weight-gradient
// side stream into the communication stream and launches the fused allreduce+SGD kernel — without touching Python.
// Python is called back ONCE per step (first bucket): for the framework's current stream and for the hyper-parameter
// upload, which follows the optimizer's param_groups (LR schedules).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <vector>

#include "../comm/comm.h"

namespace ddl {

// ---- weight-gradient side stream (module-wide): ops note work enqueued on it, consumers join what is pending ------------
void wgrad_note(cudaStream_t side);
// makes `consumer` wait for everything noted since the last join; false when nothing was pending
bool wgrad_join(cudaStream_t consumer);

struct StepLauncherConfig {
  std::vector<int32_t> param_bucket;         // bucket of each parameter, ready order
  std::vector<int32_t> bucket_param_count;
  std::vector<int64_t> bucket_start, bucket_numel;
  CommCtx ctx{};
  int world = 1;
  float* W = nullptr;                        // fp32 master weights, gradient accumulators, momentum: arena bases
  float* G = nullptr;
  float* M = nullptr;
  void* Wb = nullptr;                        // bf16 compute copy of the weights
  const SgdHyper* hyper_dev = nullptr;
  int comm_blocks = 32, sms = 132;         // callers pass the device's SM count; 132 = H100 SXM
  bool use_mc = false, wire_bf16 = false;
  int64_t oneshot_bytes = 0;
  uint64_t scalars_off = 0;
  float* scalars_out = nullptr;
  cudaStream_t comm_stream = nullptr;        // nullptr: buckets are launched on the compute stream
};

class StepLauncher {
 public:
  using StreamFn = std::function<cudaStream_t()>;        // the framework's current compute stream
  using HyperFn = std::function<void(cudaStream_t)>;     // upload this step's hyper-parameters on that stream

  StepLauncher(StepLauncherConfig cfg, StreamFn stream_fn, HyperFn hyper_fn);
  ~StepLauncher();
  StepLauncher(const StepLauncher&) = delete;
  StepLauncher& operator=(const StepLauncher&) = delete;

  int on_ready(int idx);     // gradient of parameter idx is final; returns the number of kernels launched
  int finish();              // launch what is left (parameters without a gradient), join the communication stream
  void reset();              // next step
  void set_hold(bool hold) { hold_ = hold; }
  void set_scalars_pending(bool on) { scalars_pending_ = on; }
  int next_bucket() const { return next_; }
  int launches() const { return launches_; }             // kernels launched since construction

 private:
  void launch(int b);
  cudaEvent_t next_event();

  StepLauncherConfig c_;
  StreamFn stream_fn_;
  HyperFn hyper_fn_;
  std::vector<int32_t> pending_;
  std::vector<uint8_t> seen_;
  std::vector<cudaEvent_t> events_;
  size_t ev_next_ = 0;
  int next_ = 0;
  int launches_ = 0;
  bool hold_ = false, scalars_pending_ = false, hyper_uploaded_ = false, have_stream_ = false;
  cudaStream_t cur_ = nullptr;
};

}  // namespace ddl
