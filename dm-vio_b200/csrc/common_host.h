// Host-side helpers shared by the C-ABI translation units: thread-local error string, CK, the owners of the handles' CUDA memory, streams
// and events, a lazily dlopen()ed NCCL (so the library loads on hosts without libnccl and uses the copy already mapped by the process, e.g.
// PyTorch's), and the launchers of the image-plane kernels that the BA, coarse-tracker and initialiser uploads share.
#pragma once
#include "../../include/dmvio_b200.h"
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <utility>

namespace dmv {
// Owner of one device (cudaMalloc) or pinned host (cudaMallocHost) buffer of T: move-only, freed by its destructor, and converted to T*
// wherever the buffer is used.  The caller keeps the stream ordering: a buffer is released or replaced only once no queued work reads it.
template <typename T, bool Pinned>
class CudaBuf {
 public:
  CudaBuf() = default;
  CudaBuf(CudaBuf&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  CudaBuf& operator=(CudaBuf&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
  ~CudaBuf() { if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_); }
  operator T*() const { return p_; }
  T* operator->() const { return p_; }
  T* get() const { return p_; }
  size_t size() const { return n_; }   // elements
  // n elements, after releasing what the buffer held; on failure the buffer is left empty
  cudaError_t alloc(size_t n) {
    *this = CudaBuf();
    void* p = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e == cudaSuccess) { p_ = static_cast<T*>(p); n_ = n; }
    return e;
  }
  // grow-only: a buffer of at least n elements stays as it is, a smaller one is replaced by alloc(n)
  cudaError_t reserve(size_t n) { return n <= n_ ? cudaSuccess : alloc(n); }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};
template <typename T> using DevBuf = CudaBuf<T, false>;
template <typename T> using PinnedBuf = CudaBuf<T, true>;

// Owner of a stream or an event: destroyed with its handle; put() receives it from the create call
template <typename H, cudaError_t (*Destroy)(H)>
class CudaObj {
 public:
  CudaObj() = default;
  CudaObj(const CudaObj&) = delete;
  CudaObj& operator=(const CudaObj&) = delete;
  ~CudaObj() { if (h_) Destroy(h_); }
  operator H() const { return h_; }
  H* put() { return &h_; }

 private:
  H h_ = nullptr;
};
using Stream = CudaObj<cudaStream_t, cudaStreamDestroy>;
using Event = CudaObj<cudaEvent_t, cudaEventDestroy>;

int set_error(int code, const char* fmt, ...);
int nccl_unique_id(void* id128);
int nccl_init(void** comm, int nranks, int rank, const void* id128);
int nccl_allreduce_double(void* comm, double* buf, size_t count, cudaStream_t s);
void nccl_destroy(void* comm);

// image_planes.cu: AoS3 [I, dx, dy] -> float4 texels; level-0 [I, dx, dy, 0] from intensities; level l+1 intensities from level l's texels
void launch_repack(const float* src, float4* dst, int n, cudaStream_t s);
void launch_make_dI(const float* img, float4* dst, int w, int h, cudaStream_t s);
void launch_pyr_down(const float4* src, float* dst, int wl, int hl, int wlm1, cudaStream_t s);
}  // namespace dmv

// returns DMV_ERR_CUDA with the failing call's text from the enclosing C-ABI function
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) return dmv::set_error(DMV_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(_e)); \
  } while (0)
