// Host-side helpers shared by the C-ABI translation units: thread-local error string, CK, a lazily dlopen()ed NCCL (so the library
// loads on hosts without libnccl and uses the copy already mapped by the process, e.g. PyTorch's), and the launchers of the image-plane
// kernels that the BA, coarse-tracker and initialiser uploads share.
#pragma once
#include "../../include/dmvio_b200.h"
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>

namespace dmv {
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
