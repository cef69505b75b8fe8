// dmv_ip_store — a window's immature points resident on one device between frames (include/dmvio_b200.h).  The store keeps the points of
// every slot in ip_trace_kernel's ipw layout (ip_trace.h), concatenated in slot order, with set = slot, and its own table area: a trace
// over the store is then one ip_trace_kernel member {the handle's frame, the store's buffer, its capacity, its point count}, and a frame
// uploads 14 floats per slot and downloads nothing.
// put and remove rebuild the point list by one gather (ip_store_gather_kernel) into the second of two buffers: new row j = old row
// perm[j], or a row of the slot just uploaded.  The kernel only copies words, so an edit changes no bit of a point that stays.
#include "ba_handle.h"
#include "ct_handle.h"
#include "ip_store.h"
#include "ip_trace.h"
#include "remove_outliers.h"
#include <cstring>
#include <vector>

namespace dmv {

// address of word w (0 .. 30) of point i in an ipw array of capacity cap
__device__ __forceinline__ size_t ipw_word(int w, size_t i, size_t cap) {
  int b = w, width = 1;
  if (w >= ipw::color && w < ipw::weights) { b = ipw::color; width = 8; }
  else if (w >= ipw::weights && w < ipw::gradH) { b = ipw::weights; width = 8; }
  else if (w >= ipw::gradH && w < ipw::energyTH) { b = ipw::gradH; width = 4; }
  else if (w >= ipw::uv && w < ipw::interval) { b = ipw::uv; width = 2; }
  return (size_t)b * cap + width * i + (w - b);
}

// row j of dst (all 31 words) = row perm[j] of src, or row -1 - perm[j] of add; one thread per (row, word), the word in blockIdx.y
__global__ void __launch_bounds__(128) ip_store_gather_kernel(unsigned* __restrict__ dst, int dcap, const unsigned* __restrict__ src, int scap,
                                                              const unsigned* __restrict__ add, int acap, const int* __restrict__ perm, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int w = blockIdx.y, p = perm[j];
  dst[ipw_word(w, j, dcap)] = p >= 0 ? src[ipw_word(w, p, scap)] : add[ipw_word(w, -1 - p, acap)];
}

constexpr int kWords = ipw::tables;                       // 31 words per point
constexpr size_t kTableWords = 14 * DMV_IP_STORE_SLOTS;

static int ip_store_total(const dmv_ip_store* s) {
  int n = 0;
  for (int k = 0; k < DMV_IP_STORE_SLOTS; k++) n += s->count[k];
  return n;
}

int ip_store_first(const dmv_ip_store* s, int slot) {
  int at = 0;
  for (int k = 0; k < slot; k++) at += s->count[k];
  return at;
}

// buffer k holds at least n points
static cudaError_t ip_store_reserve(dmv_ip_store* s, int k, int n) {
  if (n <= s->cap[k]) return cudaSuccess;
  s->cap[k] = 0;
  const int cap = std::max(2048, n + n / 2);
  const cudaError_t e = s->d_pts[k].alloc((size_t)kWords * cap + kTableWords);
  if (e == cudaSuccess) s->cap[k] = cap;
  return e;
}

// The edit shared by put and remove: the new list is perm (perm.size() rows) over the current buffer and the m rows that the caller wrote
// into h_edit (ipw layout of capacity m), or, rows_on_device, into d_edit on the store's stream; uploaded (the row map only when the rows
// are already there), gathered into the other buffer on the store's stream.  Returns the buffer the list lands in; ip_store_commit makes it
// current.  h_edit / d_edit already hold room for the rows and perm (ip_store_stage).
static int ip_store_gather(dmv_ip_store* s, const std::vector<int>& perm, int m, bool rows_on_device, int* dst_out) {
  const int n = (int)perm.size();
  const int dst = 1 - s->cur;
  CK(ip_store_reserve(s, dst, n));
  const size_t rows = (size_t)kWords * m, words = rows + n;
  std::memcpy(s->h_edit.get() + rows, perm.data(), sizeof(int) * (size_t)n);
  if (n > 0) {
    const size_t first = rows_on_device ? rows : 0;
    CK(cudaMemcpyAsync(s->d_edit + first, s->h_edit + first, sizeof(float) * (words - first), cudaMemcpyHostToDevice, s->stream));
    const dim3 grid((n + 127) / 128, kWords);
    ip_store_gather_kernel<<<grid, 128, 0, s->stream>>>(reinterpret_cast<unsigned*>(s->d_pts[dst].get()), s->cap[dst],
                                                        reinterpret_cast<const unsigned*>(s->d_pts[s->cur].get()), s->cap[s->cur],
                                                        reinterpret_cast<const unsigned*>(s->d_edit.get()), m,
                                                        reinterpret_cast<const int*>(s->d_edit.get() + rows), n);
    CK(cudaGetLastError());
  }
  *dst_out = dst;
  return DMV_OK;
}

// synchronises the store's stream, then buffer dst holds the list and count_after its slot counts
static int ip_store_commit(dmv_ip_store* s, int dst, const int* count_after) {
  CK(cudaStreamSynchronize(s->stream));
  s->cur = dst;
  std::memcpy(s->count, count_after, sizeof(s->count));
  return DMV_OK;
}

static int ip_store_apply(dmv_ip_store* s, const std::vector<int>& perm, int m, const int* count_after) {
  int dst = 0;
  const int rc = ip_store_gather(s, perm, m, false, &dst);
  if (rc != DMV_OK) return rc;
  return ip_store_commit(s, dst, count_after);
}

// h_edit / d_edit hold an edit of m uploaded rows and an n-row map
static int ip_store_stage(dmv_ip_store* s, int m, int n) {
  const size_t words = (size_t)kWords * m + n;
  CK(s->h_edit.reserve(words));
  CK(s->d_edit.reserve(words));
  return DMV_OK;
}

int ip_store_remove_dead(dmv_ip_store* s, const std::vector<char> (&alive)[DMV_IP_STORE_SLOTS], std::vector<int> (&order)[DMV_IP_STORE_SLOTS]) {
  int count[DMV_IP_STORE_SLOTS], total = 0, removed = 0;
  for (int k = 0; k < DMV_IP_STORE_SLOTS; k++) {
    const int m = s->count[k];
    if (alive[k].empty()) {
      order[k].resize(m);
      for (int q = 0; q < m; q++) order[k][q] = q;
    } else {
      order[k] = remove_outliers_order(0, m, alive[k]);   // activatePointsMT's loop (FullSystem.cpp:L761-769), on indices
    }
    count[k] = (int)order[k].size();
    total += count[k];
    removed += m - count[k];
  }
  if (removed == 0) return DMV_OK;
  CK(cudaSetDevice(s->device));
  const int rc = ip_store_stage(s, 0, total);
  if (rc != DMV_OK) return rc;
  std::vector<int> perm;
  perm.reserve(total);
  for (int k = 0, first = 0; k < DMV_IP_STORE_SLOTS; first += s->count[k], k++)
    for (int o : order[k]) perm.push_back(first + o);
  return ip_store_apply(s, perm, 0, count);
}

// the checks of one store job (dmv_ct_trace_store's arguments after the NULL checks); *n = the points it traces.  No CUDA call.
static int ip_store_job_check(const dmv_ct* c, const dmv_ip_store* s, int nslots, const float* tables14, int* n) {
  if (!s) return set_error(DMV_ERR_INVALID, "null argument");
  if (nslots < 0 || nslots > DMV_IP_STORE_SLOTS) return set_error(DMV_ERR_INVALID, "nslots = %d: expected 0 to %d", nslots, DMV_IP_STORE_SLOTS);
  if (s->device != c->device) return set_error(DMV_ERR_INVALID, "the store is on device %d, the handle on device %d", s->device, c->device);
  *n = 0;
  for (int k = 0; k < DMV_IP_STORE_SLOTS; k++) {
    if (k >= nslots && s->count[k] > 0) return set_error(DMV_ERR_INVALID, "slot %d holds %d points but nslots = %d", k, s->count[k], nslots);
    *n += s->count[k];
  }
  if (*n > 0 && !tables14) return set_error(DMV_ERR_INVALID, "null tables14 with %d points in the store", *n);
  return DMV_OK;
}

// The stores of n handles traced in one launch (n = 1, !many: dmv_ct_trace_store).  Every job is checked first; each store's tables go to
// its table area on handles[0]'s stream, the launch follows there behind every member's queued work, and one synchronisation ends the call.
static int ip_store_trace_run(dmv_ct* const* hs, int n, const dmv_ct_trace_store_job* jobs, const dmv_ip_settings* settings, bool many) {
  int np[DMV_CT_TRACE_MANY_MAX];
  int total = 0;
  for (int i = 0; i < n; i++) {
    const int rc = ip_store_job_check(hs[i], jobs[i].store, jobs[i].nslots, jobs[i].tables14, &np[i]);
    if (rc != DMV_OK) return many ? ct_member_error(rc, i) : rc;
    for (int j = 0; j < i; j++)
      if (jobs[j].store == jobs[i].store) return set_error(DMV_ERR_INVALID, "jobs[%d] and jobs[%d] name the same store", j, i);
    total += np[i];
  }
  if (total == 0) return DMV_OK;
  CK(cudaSetDevice(hs[0]->device));
  IPTraceArgs A;
  ip_trace_args(A, n, settings);
  const cudaStream_t st = hs[0]->stream;
  for (int i = 0; i < n; i++) {
    dmv_ip_store* s = jobs[i].store;
    ip_trace_member(A, i, hs[i], s->d_pts[s->cur], s->cap[s->cur], np[i]);
    if (np[i] == 0) continue;
    const size_t nt = 14 * (size_t)jobs[i].nslots;
    std::memcpy(s->h_tab, jobs[i].tables14, sizeof(float) * nt);
    CK(cudaMemcpyAsync(s->d_pts[s->cur] + (size_t)kWords * s->cap[s->cur], s->h_tab, sizeof(float) * nt, cudaMemcpyHostToDevice, st));
  }
  const int rc = ip_trace_launch(hs, A);
  if (rc != DMV_OK) return rc;
  CK(cudaStreamSynchronize(st));
  for (int i = 0; i < n; i++) hs[i]->staging_busy = false;   // every member's queued work completed before the kernel started
  return DMV_OK;
}

}  // namespace dmv

using namespace dmv;

int dmv_ip_store_create(int device, dmv_ip_store** out) {
  if (!out) return set_error(DMV_ERR_INVALID, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return set_error(DMV_ERR_NO_DEVICE, "no CUDA device: dmvio_b200 has no CPU path");
  }
  if (device < 0 || device >= ndev) return set_error(DMV_ERR_INVALID, "device out of range");
  CK(cudaSetDevice(device));
  std::unique_ptr<dmv_ip_store> s(new dmv_ip_store());
  s->device = device;
  CK(cudaStreamCreateWithFlags(s->stream.put(), cudaStreamNonBlocking));
  CK(s->h_tab.alloc(kTableWords));
  *out = s.release();
  return DMV_OK;
}

int dmv_ip_store_destroy(dmv_ip_store* s) {
  if (!s) return DMV_OK;
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  delete s;
  return DMV_OK;
}

static int ip_store_slot_check(const dmv_ip_store* s, int slot) {
  if (!s) return set_error(DMV_ERR_INVALID, "null argument");
  if (slot < 0 || slot >= DMV_IP_STORE_SLOTS) return set_error(DMV_ERR_INVALID, "slot %d: expected 0 to %d", slot, DMV_IP_STORE_SLOTS - 1);
  return DMV_OK;
}

// put's row map: every slot's rows in place, slot `slot` replaced by the m uploaded rows; count = the slot counts after the edit
static void ip_store_put_map(const dmv_ip_store* s, int slot, int m, std::vector<int>& perm, int* count) {
  perm.clear();
  perm.reserve(ip_store_total(s) - s->count[slot] + m);
  int at = 0;
  for (int k = 0; k < DMV_IP_STORE_SLOTS; k++) {
    if (k == slot)
      for (int q = 0; q < m; q++) perm.push_back(-1 - q);
    else
      for (int q = 0; q < s->count[k]; q++) perm.push_back(at + q);
    at += s->count[k];
  }
  std::memcpy(count, s->count, sizeof(s->count));
  count[slot] = m;
}

int dmv_ip_store_put(dmv_ip_store* s, int slot, const dmv_ip_points* p) {
  int rc = ip_store_slot_check(s, slot);
  if (rc != DMV_OK) return rc;
  if (!p) return set_error(DMV_ERR_INVALID, "null argument");
  if (p->n < 0 || (p->n > 0 && (!p->u || !p->v || !p->color8 || !p->weights8 || !p->gradH4 || !p->energyTH || !p->idepth_min || !p->idepth_max ||
                                !p->quality || !p->lastTraceStatus || !p->lastTraceUV2 || !p->lastTracePixelInterval)))
    return set_error(DMV_ERR_INVALID, "incomplete dmv_ip_points");
  const int m = p->n, old = s->count[slot];
  if (m == 0 && old == 0) return DMV_OK;
  const int total = ip_store_total(s) - old + m;
  CK(cudaSetDevice(s->device));
  rc = ip_store_stage(s, m, total);
  if (rc != DMV_OK) return rc;
  float* hb = s->h_edit;
  const size_t cap = (size_t)m, n = (size_t)m;
  if (m > 0) {   // the slot's rows, ipw layout of capacity m
    std::memcpy(hb + ipw::u * cap, p->u, 4 * n); std::memcpy(hb + ipw::v * cap, p->v, 4 * n);
    std::memcpy(hb + ipw::color * cap, p->color8, 32 * n); std::memcpy(hb + ipw::weights * cap, p->weights8, 32 * n);
    std::memcpy(hb + ipw::gradH * cap, p->gradH4, 16 * n); std::memcpy(hb + ipw::energyTH * cap, p->energyTH, 4 * n);
    std::memcpy(hb + ipw::idepth_min * cap, p->idepth_min, 4 * n); std::memcpy(hb + ipw::idepth_max * cap, p->idepth_max, 4 * n);
    std::memcpy(hb + ipw::quality * cap, p->quality, 4 * n); std::memcpy(hb + ipw::status * cap, p->lastTraceStatus, 4 * n);
    std::memcpy(hb + ipw::uv * cap, p->lastTraceUV2, 8 * n); std::memcpy(hb + ipw::interval * cap, p->lastTracePixelInterval, 4 * n);
    int* setp = reinterpret_cast<int*>(hb + ipw::set * cap);
    for (size_t q = 0; q < n; q++) setp[q] = slot;
  }
  std::vector<int> perm;
  int count[DMV_IP_STORE_SLOTS];
  ip_store_put_map(s, slot, m, perm, count);
  return ip_store_apply(s, perm, m, count);
}

namespace dmv {
// put with rows the caller writes on the device (ip_store.h).  d_edit: the m rows (ipw layout of capacity m), the row map, then m words for
// the caller; h_edit: the row map at the same offset, and the downloaded outputs in front of it (24 words per point <= kWords)
int ip_store_rows_stage(dmv_ip_store* s, int slot, int m, float** d_rows, float** d_extra) {
  const int total = ip_store_total(s) - s->count[slot] + m;
  CK(cudaSetDevice(s->device));
  const int rc = ip_store_stage(s, m, total + m);
  if (rc != DMV_OK) return rc;
  *d_rows = s->d_edit;
  *d_extra = s->d_edit + (size_t)kWords * m + total;
  return DMV_OK;
}

int ip_store_rows_put(dmv_ip_store* s, int slot, int m, const dmv_new_traces_args* out) {
  const int old = s->count[slot];
  if (m == 0 && old == 0) {   // put leaves the store as it is; the caller's copy kernel has nothing to write
    CK(cudaStreamSynchronize(s->stream));
    return DMV_OK;
  }
  std::vector<int> perm;
  int count[DMV_IP_STORE_SLOTS];
  ip_store_put_map(s, slot, m, perm, count);
  const float* d_extra = s->d_edit + (size_t)kWords * m + perm.size();
  int dst = 0;
  const int rc = ip_store_gather(s, perm, m, true, &dst);
  if (rc != DMV_OK) return rc;
  // the requested outputs from the slot's rows in the new buffer; type, which the store does not hold, from the words beside the rows
  const size_t cap = s->cap[dst], at = ip_store_first(s, slot), n = m;
  const float* d = s->d_pts[dst];
  float* hb = s->h_edit;
  struct Field { const void* want; const float* src; size_t words; };
  const Field f[7] = {{out->u, d + ipw::u * cap + at, n},
                      {out->v, d + ipw::v * cap + at, n},
                      {out->color8, d + ipw::color * cap + 8 * at, 8 * n},
                      {out->weights8, d + ipw::weights * cap + 8 * at, 8 * n},
                      {out->gradH4, d + ipw::gradH * cap + 4 * at, 4 * n},
                      {out->energyTH, d + ipw::energyTH * cap + at, n},
                      {out->type, d_extra, n}};
  size_t o = 0;
  for (const Field& x : f) {
    if (x.want && n > 0) CK(cudaMemcpyAsync(hb + o, x.src, sizeof(float) * x.words, cudaMemcpyDeviceToHost, s->stream));
    o += x.words;
  }
  const int rc2 = ip_store_commit(s, dst, count);
  if (rc2 != DMV_OK) return rc2;
  for (size_t i = 0; out->u && i < n; i++) out->u[i] = (int32_t)hb[i];
  for (size_t i = 0; out->v && i < n; i++) out->v[i] = (int32_t)hb[n + i];
  if (out->color8) std::memcpy(out->color8, hb + 2 * n, 32 * n);
  if (out->weights8) std::memcpy(out->weights8, hb + 10 * n, 32 * n);
  if (out->gradH4) std::memcpy(out->gradH4, hb + 18 * n, 16 * n);
  if (out->energyTH) std::memcpy(out->energyTH, hb + 22 * n, 4 * n);
  if (out->type) std::memcpy(out->type, hb + 23 * n, 4 * n);
  return DMV_OK;
}
}  // namespace dmv

int dmv_ip_store_get(dmv_ip_store* s, int slot, dmv_ip_points* p) {
  const int rc = ip_store_slot_check(s, slot);
  if (rc != DMV_OK) return rc;
  if (!p) return set_error(DMV_ERR_INVALID, "null argument");
  const int m = s->count[slot];
  if (p->n != m) return set_error(DMV_ERR_INVALID, "pts->n = %d: slot %d holds %d points", p->n, slot, m);
  if (m > 0 && (!p->idepth_min || !p->idepth_max || !p->quality || !p->lastTraceStatus || !p->lastTraceUV2 || !p->lastTracePixelInterval))
    return set_error(DMV_ERR_INVALID, "incomplete dmv_ip_points");
  if (m == 0) return DMV_OK;
  CK(cudaSetDevice(s->device));
  CK(s->h_edit.reserve((size_t)ipw::inout * m));
  const size_t cap = s->cap[s->cur], at = ip_store_first(s, slot), n = m;
  const float* d = s->d_pts[s->cur];
  float* hb = s->h_edit;
  // idepth_min, idepth_max, quality, status: four arrays of one word per point; then uv (two) and interval (one)
  CK(cudaMemcpy2DAsync(hb, 4 * n, d + ipw::idepth_min * cap + at, 4 * cap, 4 * n, 4, cudaMemcpyDeviceToHost, s->stream));
  CK(cudaMemcpyAsync(hb + 4 * n, d + ipw::uv * cap + 2 * at, 8 * n, cudaMemcpyDeviceToHost, s->stream));
  CK(cudaMemcpyAsync(hb + 6 * n, d + ipw::interval * cap + at, 4 * n, cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  std::memcpy(p->idepth_min, hb, 4 * n); std::memcpy(p->idepth_max, hb + n, 4 * n); std::memcpy(p->quality, hb + 2 * n, 4 * n);
  std::memcpy(p->lastTraceStatus, hb + 3 * n, 4 * n); std::memcpy(p->lastTraceUV2, hb + 4 * n, 8 * n); std::memcpy(p->lastTracePixelInterval, hb + 6 * n, 4 * n);
  return DMV_OK;
}

int dmv_ip_store_remove(dmv_ip_store* s, int slot, int n, const int32_t* idx, int32_t* order_out) {
  int rc = ip_store_slot_check(s, slot);
  if (rc != DMV_OK) return rc;
  if (n < 0 || (n > 0 && !idx)) return set_error(DMV_ERR_INVALID, "null argument");
  const int m = s->count[slot];
  if (n > m) return set_error(DMV_ERR_INVALID, "n = %d: slot %d holds %d points", n, slot, m);
  std::vector<char> alive[DMV_IP_STORE_SLOTS];
  alive[slot].assign(m, 1);
  for (int q = 0; q < n; q++) {
    if (idx[q] < 0 || idx[q] >= m) return set_error(DMV_ERR_INVALID, "idx[%d] = %d: slot %d holds %d points", q, idx[q], slot, m);
    if (!alive[slot][idx[q]]) return set_error(DMV_ERR_INVALID, "idx[%d] = %d appears twice", q, idx[q]);
    alive[slot][idx[q]] = 0;
  }
  std::vector<int> order[DMV_IP_STORE_SLOTS];
  rc = ip_store_remove_dead(s, alive, order);
  if (rc != DMV_OK) return rc;
  if (order_out) std::memcpy(order_out, order[slot].data(), sizeof(int32_t) * order[slot].size());
  return DMV_OK;
}

int dmv_ct_trace_store(dmv_ct* c, dmv_ip_store* s, int nslots, const float* tables14, const dmv_ip_settings* settings) {
  if (!c || !s) return set_error(DMV_ERR_INVALID, "null argument");
  dmv_ct_trace_store_job j;
  j.store = s; j.nslots = nslots; j.tables14 = tables14;
  return ip_store_trace_run(&c, 1, &j, settings, false);
}

int dmv_ct_trace_store_many(dmv_ct* const* handles, int n, const dmv_ct_trace_store_job* jobs, const dmv_ip_settings* settings) {
  if (!handles || !jobs) return set_error(DMV_ERR_INVALID, "null argument");
  const int rc = ct_check_members(handles, n, DMV_CT_TRACE_MANY_MAX);
  if (rc != DMV_OK) return rc;
  return ip_store_trace_run(handles, n, jobs, settings, true);
}

// dmv_ba_activate_store: the selection and the activation on rows gathered from the store on the device, then the removal as one edit
int dmv_ba_activate_store(dmv_ba* b, dmv_ip_store* s, const dmv_ba_activate_store_args* a) {
  if (!b || !s || !a) return set_error(DMV_ERR_INVALID, "null argument");
  if (b->nf < 2 || !b->have_state) return set_error(DMV_ERR_STATE, "dmv_ba_set_window + dmv_ba_set_state first");
  const int nf = a->nf;
  if (nf != b->nf) return set_error(DMV_ERR_INVALID, "nf = %d: the window has %d frames", nf, b->nf);
  if (s->device != b->device) return set_error(DMV_ERR_INVALID, "the store is on device %d, the handle on device %d", s->device, b->device);
  if (!a->slot || !a->my_type) return set_error(DMV_ERR_INVALID, "incomplete dmv_ba_activate_store_args");
  int off[MAXF + 1] = {0};
  for (int f = 0; f < nf; f++) {
    const int k = a->slot[f];
    if (k < -1 || k >= DMV_IP_STORE_SLOTS) return set_error(DMV_ERR_INVALID, "slot[%d] = %d: expected -1 to %d", f, k, DMV_IP_STORE_SLOTS - 1);
    for (int g = 0; g < f; g++)
      if (k >= 0 && a->slot[g] == k) return set_error(DMV_ERR_INVALID, "slot[%d] and slot[%d] are both %d", g, f, k);
    const int m = k >= 0 ? s->count[k] : 0;
    if (m > 0 && !a->my_type[f]) return set_error(DMV_ERR_INVALID, "my_type[%d] is NULL for %d points", f, m);
    off[f + 1] = off[f] + m;
  }
  const int n = off[nf];
  std::vector<int32_t> action(a->action ? 0 : n), opt(std::max(a->cap, 0));
  dmv_ba_select_args sa;
  std::memset(&sa, 0, sizeof(sa));
  sa.nf = nf; sa.newest = a->newest; sa.tables12 = a->tables12; sa.flagged = a->flagged; sa.n_active = a->n_active;
  sa.act_u = a->act_u; sa.act_v = a->act_v; sa.act_idepth_scaled = a->act_idepth_scaled; sa.act_host = a->act_host; sa.imm_offset = off;
  sa.currentMinActDist = a->currentMinActDist; sa.minTraceQuality = a->minTraceQuality; sa.cap = a->cap; sa.n_opt = a->n_opt;
  sa.action = a->action ? a->action : action.data(); sa.opt_idx = opt.data(); sa.map = a->map; sa.stats = a->stats;
  int rc = sel_check(b, &sa, true);
  if (rc != DMV_OK) return rc;
  if (a->cap > 0 && (!a->RT || !a->opt_frame || !a->opt_index || !a->status || !a->idepth || !a->res_state))
    return set_error(DMV_ERR_INVALID, "incomplete dmv_ba_activate_store_args");
  const int* d_opt = nullptr;
  rc = ip_select_from_store(b, &sa, s, a->slot, a->my_type, &d_opt);
  if (rc != DMV_OK) return rc;
  const int nopt = *a->n_opt;
  std::vector<int32_t> trace_status(nopt);
  rc = ip_act_from_store(b, s, off, a->slot, d_opt, nopt, a->RT, a->minObs, a->status, a->idepth, a->res_state, trace_status.data());
  if (rc != DMV_OK) return rc;
  // activatePointsMT's removals (FullSystem.cpp:L732-770): deleted by the selection, activated (1), outliers (-1), and not activated but OOB
  std::vector<char> alive[DMV_IP_STORE_SLOTS];
  for (int f = 0; f < nf; f++)
    if (a->slot[f] >= 0 && f != a->newest) alive[a->slot[f]].assign(off[f + 1] - off[f], 1);
  for (int f = 0; f < nf; f++)
    for (int i = off[f]; f != a->newest && i < off[f + 1]; i++)
      if (sa.action[i] == DMV_ACT_DELETE) alive[a->slot[f]][i - off[f]] = 0;
  int32_t* act_host = nopt > 0 ? reinterpret_cast<int32_t*>(b->h_act.get() + act_layout(b->act_cap).host) : nullptr;   // as the gather wrote d_act
  for (int j = 0; j < nopt; j++) {
    const int i = opt[j];
    int f = 0;
    while (off[f + 1] <= i) f++;
    act_host[j] = f;
    a->opt_frame[j] = f;
    a->opt_index[j] = i - off[f];
    if (a->status[j] != 0 || trace_status[j] == 1) alive[a->slot[f]][i - off[f]] = 0;   // IPS_OOB
  }
  std::vector<int> order[DMV_IP_STORE_SLOTS];
  b->act_n = nopt;
  rc = ip_store_remove_dead(s, alive, order);
  if (rc != DMV_OK) return rc;
  for (int f = 0, at = 0; f < nf; f++) {
    const int kept = a->slot[f] >= 0 ? (int)order[a->slot[f]].size() : 0;
    if (a->order_out && kept > 0) std::memcpy(a->order_out + at, order[a->slot[f]].data(), sizeof(int32_t) * kept);
    if (a->n_kept) a->n_kept[f] = kept;
    at += kept;
  }
  return DMV_OK;
}
