// workspace.h -- host-side scaffolding of the point-cloud entry points (normals, outliers, subsample, plane, objects)
// and mesh_score: workspace carving, the stage-timing hook, launch sizes and the error tail.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "internal.h"

namespace ma {

// every workspace buffer starts on a 256-byte boundary
constexpr size_t ws_align(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// Hands out aligned typed buffers from a workspace, in the order they are taken; with a null base it only counts
// the bytes, so a stage's size query and its entry point share one function.
struct Carver {
  char* base;
  size_t total = 0;
  explicit Carver(void* ws) : base(static_cast<char*>(ws)) {}
  template <class T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + total) : nullptr;
    total += ws_align(count * sizeof(T));
    return p;
  }
};

// The stage-timing hook behind ma_*_set_events: while set, mark(i) records the caller's event i on the stream.
template <int N>
struct StageEvents {
  cudaEvent_t ev[N];
  bool on = false;
  void set(void* const* events) {
    on = events != nullptr;
    if (events)
      for (int i = 0; i < N; i++) ev[i] = (cudaEvent_t)events[i];
  }
  void mark(int at, cudaStream_t st) const {
    if (on) cudaEventRecord(ev[at], st);
  }
};

inline int blocks(size_t count, int threads) { return (int)((count + threads - 1) / threads); }

// SMs of the current device; 132 (an H100 SXM) when the query fails
inline int sm_count() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    sms = 132;
  return sms;
}

// The status of an entry point after it enqueued work, given the first error of its runtime calls: 1 with
// "<what>: <error>" set and the non-sticky error cleared, so that the next call does not report it; otherwise the
// launch check.
inline int stage_status(const char* what, cudaError_t e) {
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    cudaGetLastError();
    return 1;
  }
  return check_launch(what) ? 0 : 1;
}

}  // namespace ma
