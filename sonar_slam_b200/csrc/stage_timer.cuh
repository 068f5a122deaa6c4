// Optional per-stage device timing (sfe_frontend_*, sfe_jpeg_*, sfe_png_* set_timing / get_timing): a pair of CUDA
// events brackets every timed interval on the stream its work runs on, and collect() adds the elapsed times of the
// closed intervals to running totals per stage.
#pragma once
#include <vector>

#include "common.cuh"

namespace sfe {

struct StageTimer {
  static constexpr int MAX_STAGES = 8;
  static_assert(SFE_FE_STAGES <= MAX_STAGES && SFE_JPEG_STAGES <= MAX_STAGES && SFE_PNG_STAGES <= MAX_STAGES, "");

  bool on = false;

  StageTimer() = default;
  StageTimer(const StageTimer &) = delete;
  StageTimer &operator=(const StageTimer &) = delete;
  ~StageTimer() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }

  // drop the totals and any interval not collected yet; time from now on when `enable`
  void reset(bool enable) {
    on = enable;
    stage.clear();
    for (int i = 0; i < MAX_STAGES; ++i) ms[i] = 0.0, calls[i] = 0;
  }

  void tic(cudaStream_t st, int s) {
    if (!on) return;
    const size_t k = stage.size();
    while (ev.size() < 2 * k + 2) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      ev.push_back(e);
    }
    cudaEventRecord(ev[2 * k], st);
    open = s;
  }

  void toc(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(ev[2 * stage.size() + 1], st);
    stage.push_back(open);
  }

  // waits for `st` (the stream every interval was recorded on), adds the closed intervals to the totals and writes
  // the totals of the first n_stages stages (stage_calls may be null)
  int collect(cudaStream_t st, int n_stages, double *stage_ms, int64_t *stage_calls) {
    SFE_CUDA(cudaStreamSynchronize(st));
    for (size_t k = 0; k < stage.size(); ++k) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, ev[2 * k], ev[2 * k + 1]) == cudaSuccess) ms[stage[k]] += t, calls[stage[k]]++;
    }
    stage.clear();
    for (int i = 0; i < n_stages; ++i) {
      stage_ms[i] = ms[i];
      if (stage_calls) stage_calls[i] = calls[i];
    }
    return SFE_OK;
  }

 private:
  std::vector<cudaEvent_t> ev;  // pool; events [2k, 2k + 1] bracket closed interval k
  std::vector<int> stage;       // stage of closed interval k: pushed when it closes, so it never runs ahead of ev
  int open = 0;                 // stage of the interval tic() opened
  double ms[MAX_STAGES] = {};
  int64_t calls[MAX_STAGES] = {};
};

}  // namespace sfe
