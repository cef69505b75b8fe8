#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include <dlfcn.h>
#include <cstring>

namespace dmv {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// ---- NCCL through dlopen -------------------------------------------------------------------------------------
typedef struct { char internal[128]; } ncclUniqueId_t;
typedef int (*fn_getuid)(ncclUniqueId_t*);
typedef int (*fn_initrank)(void**, int, ncclUniqueId_t, int);
typedef int (*fn_allreduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*fn_destroy)(void*);
typedef const char* (*fn_errstr)(int);
static void* g_nccl = nullptr;
static fn_getuid p_getuid; static fn_initrank p_initrank; static fn_allreduce p_allreduce; static fn_destroy p_destroy; static fn_errstr p_errstr;

static int load_nccl() {
  if (g_nccl) return DMV_OK;
  g_nccl = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!g_nccl) g_nccl = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!g_nccl) return set_error(DMV_ERR_NCCL, "cannot dlopen libnccl: %s", dlerror());
  p_getuid = (fn_getuid)dlsym(g_nccl, "ncclGetUniqueId");
  p_initrank = (fn_initrank)dlsym(g_nccl, "ncclCommInitRank");
  p_allreduce = (fn_allreduce)dlsym(g_nccl, "ncclAllReduce");
  p_destroy = (fn_destroy)dlsym(g_nccl, "ncclCommDestroy");
  p_errstr = (fn_errstr)dlsym(g_nccl, "ncclGetErrorString");
  if (!p_getuid || !p_initrank || !p_allreduce || !p_destroy) return set_error(DMV_ERR_NCCL, "libnccl lacks required symbols");
  return DMV_OK;
}
int nccl_unique_id(void* id128) {
  int rc = load_nccl();
  if (rc != DMV_OK) return rc;
  ncclUniqueId_t id;
  int e = p_getuid(&id);
  if (e != 0) return set_error(DMV_ERR_NCCL, "ncclGetUniqueId: %s", p_errstr ? p_errstr(e) : "?");
  std::memcpy(id128, &id, 128);
  return DMV_OK;
}
int nccl_init(void** comm, int nranks, int rank, const void* id128) {
  int rc = load_nccl();
  if (rc != DMV_OK) return rc;
  ncclUniqueId_t id;
  std::memcpy(&id, id128, 128);
  int e = p_initrank(comm, nranks, id, rank);
  if (e != 0) return set_error(DMV_ERR_NCCL, "ncclCommInitRank: %s", p_errstr ? p_errstr(e) : "?");
  return DMV_OK;
}
int nccl_allreduce_double(void* comm, double* buf, size_t count, cudaStream_t s) {
  const int ncclFloat64 = 8, ncclSum = 0;
  int e = p_allreduce(buf, buf, count, ncclFloat64, ncclSum, comm, s);
  if (e != 0) return set_error(DMV_ERR_NCCL, "ncclAllReduce: %s", p_errstr ? p_errstr(e) : "?");
  return DMV_OK;
}
void nccl_destroy(void* comm) { if (comm && p_destroy) p_destroy(comm); }

}  // namespace dmv

extern "C" {
const char* dmv_last_error(void) { return dmv::g_err; }
const char* dmv_version(void) { return "dmvio_b200 0.1 (sm_90a)"; }
int dmv_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}
}
