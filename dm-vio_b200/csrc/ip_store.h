// The immature-point store's internals (ip_store.cu), shared with the activation fed from a store (dmv_ba_activate_store): the BA side
// reads the current buffer and the slot counts, and its removals go through the store's one edit path; pixel selection straight into a
// store (dmv_ct_make_new_traces_store) writes its rows into the same edit.
#pragma once
#include "../../include/dmvio_b200.h"
#include "common_host.h"
#include <vector>

struct dmv_ip_store {
  int device = 0;
  dmv::Stream stream;                 // put, get and remove; a trace runs on its handle's stream
  dmv::DevBuf<float> d_pts[2];        // ipw layout of cap[k] points, then 14 x DMV_IP_STORE_SLOTS table floats; d_pts[cur] holds the points
  int cap[2] = {0, 0};
  int cur = 0;
  int count[DMV_IP_STORE_SLOTS] = {0};   // points per slot, in slot order in d_pts[cur]
  dmv::DevBuf<float> d_edit;          // an edit's uploaded words: put's rows (ipw layout, capacity = their count), then the row map perm
  dmv::PinnedBuf<float> h_edit;       // its host side; get's downloaded words
  dmv::PinnedBuf<float> h_tab;        // a trace's tables
};

namespace dmv {
// row of the current buffer where slot k's points begin
int ip_store_first(const dmv_ip_store* s, int slot);
// Removes from every slot k with a non-empty alive[k] (one entry per point of the slot) the points q with !alive[k][q], each slot by
// activatePointsMT's swap-with-back loop (FullSystem.cpp:L761-769, remove_outliers_order), in one gather.  order[k] = slot k's survivors'
// old indices in their new order (the identity for a slot without alive entries).  No edit, copy or synchronisation when nothing is removed.
int ip_store_remove_dead(dmv_ip_store* s, const std::vector<char> (&alive)[DMV_IP_STORE_SLOTS], std::vector<int> (&order)[DMV_IP_STORE_SLOTS]);

// dmv_ip_store_put of a slot's m rows that the caller writes on the device instead of uploading them (dmv_ct_make_new_traces_store).
// ip_store_rows_stage makes room in the edit staging: *d_rows = the rows (ipw layout of capacity m, every word put uploads, set included),
// *d_extra = m words beside them that the store does not keep.  The caller writes both on the store's stream; ip_store_rows_put then
// uploads the row map only, gathers as put does, downloads out's non-NULL per-point outputs (u, v, color8, weights8, gradH4, energyTH from
// the slot's rows after the edit, type from *d_extra) and synchronises once.  Neither checks slot or m.
int ip_store_rows_stage(dmv_ip_store* s, int slot, int m, float** d_rows, float** d_extra);
int ip_store_rows_put(dmv_ip_store* s, int slot, int m, const dmv_new_traces_args* out);

// dmv_ba_select_activation's argument checks (ip_select.cu); from_store: the immature points' arrays and action are not the caller's
int sel_check(const dmv_ba* b, const dmv_ba_select_args* a, bool from_store);

// The two halves of dmv_ba_activate_store fed from a store.  Frame f's immature points are slot slot[f]'s (none for -1), the selection's
// group f.  a->imm_offset holds the groups' offsets; a->u .. a->quality are not read.
// ip_select.cu: dmv_ba_select_activation's staging, launches and read-back on those groups, type from my_type[f]; *d_opt = toOptimize on
// the device (the indexes into the groups' concatenation) for ip_act_from_store.  Results land where a's out pointers say.
int ip_select_from_store(dmv_ba* b, const dmv_ba_select_args* a, const dmv_ip_store* s, const int* slot, const float* const* my_type, const int** d_opt);
// ip_trace.cu: dmv_ba_activate_points on the n rows d_opt names, gathered from the store on the device; trace_status[j] = their
// lastTraceStatus.  Leaves the BA handle's launch count as dmv_ba_activate_points does.
int ip_act_from_store(dmv_ba* b, const dmv_ip_store* s, const int* imm_offset, const int* slot, const int* d_opt, int n, const float* RT, int minObs,
                      int32_t* status, float* idepth, int32_t* res_state, int32_t* trace_status);
}  // namespace dmv
