// owned.cuh -- owners of the engine's CUDA resources, the only code of the engine that allocates or releases CUDA memory or
// destroys a stream, event or graph.  Each owner is move-only and releases what it holds in its destructor, so a resource is
// freed exactly once, whichever way the handle or scope that holds it ends.  The live-byte counters are a test hook
// (vtts_debug_live_bytes): what this process holds through these types right now.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <utility>

namespace vtts {

inline std::atomic<uint64_t> g_live_device_bytes{0}, g_live_pinned_bytes{0};

enum class Mem { Device, Pinned, Mapped };   // cudaMalloc, cudaMallocHost, cudaHostAlloc(Mapped)

// `cap` elements of device or pinned host memory at p; mapped host memory also has its device alias at d.
template <typename T, Mem M = Mem::Device>
struct Buf {
  T* p = nullptr;
  T* d = nullptr;
  size_t cap = 0;

  Buf() = default;
  Buf(Buf&& o) noexcept { *this = std::move(o); }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) { reset(); p = std::exchange(o.p, nullptr); d = std::exchange(o.d, nullptr); cap = std::exchange(o.cap, 0); }
    return *this;
  }
  ~Buf() { reset(); }

  // Releases the old memory, then allocates exactly n elements (contents undefined).  Returns the runtime's status.
  cudaError_t alloc(size_t n) {
    reset();
    void* q = nullptr;
    const size_t bytes = n * sizeof(T);
    cudaError_t e = M == Mem::Device ? cudaMalloc(&q, bytes)
                    : M == Mem::Pinned ? cudaMallocHost(&q, bytes) : cudaHostAlloc(&q, bytes, cudaHostAllocMapped);
    if (e != cudaSuccess) return e;
    p = static_cast<T*>(q);
    cap = n;
    live() += bytes;
    return M == Mem::Mapped ? cudaHostGetDevicePointer(reinterpret_cast<void**>(&d), q, 0) : cudaSuccess;
  }
  // Workspace growth: room for n elements plus a quarter and some slack, so that slowly growing calls reallocate rarely.
  cudaError_t grow(size_t n) { return alloc(n + n / 4 + (M == Mem::Device ? 256 : 4096)); }
  void reset() {
    if (!p) return;
    if (M == Mem::Device) cudaFree(p);
    else cudaFreeHost(p);
    live() -= cap * sizeof(T);
    p = d = nullptr;
    cap = 0;
  }

 private:
  static std::atomic<uint64_t>& live() { return M == Mem::Device ? g_live_device_bytes : g_live_pinned_bytes; }
};
template <typename T>
using PinnedBuf = Buf<T, Mem::Pinned>;
template <typename T>
using MappedBuf = Buf<T, Mem::Mapped>;

// A stream, event, graph or graph exec, destroyed with `release`.  Converts to the raw handle, so it is passed to the runtime
// as it is; out() releases what it held and hands a create function the slot to fill.
template <typename H, cudaError_t (*release)(H)>
class Handle {
 public:
  Handle() = default;
  Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Handle& operator=(Handle&& o) noexcept {
    if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); }
    return *this;
  }
  ~Handle() { reset(); }
  operator H() const { return h_; }
  H* out() { reset(); return &h_; }
  void reset() {
    if (h_) release(h_);
    h_ = nullptr;
  }

 private:
  H h_ = nullptr;
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Graph = Handle<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Handle<cudaGraphExec_t, cudaGraphExecDestroy>;

}  // namespace vtts
