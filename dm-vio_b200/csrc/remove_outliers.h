// FullSystem::removeOutliers (FullSystemOptimize.cpp:L680-697): in each host frame's fh->pointHessians, a point without residuals leaves by
// swap-with-back (the host's last point moves into the hole, i-- re-checks it).  makeKeyFrame runs it right before setCoarseTrackingRef
// (FullSystem.cpp:L1438, L1458), so this is the point order makeCoarseDepthL0 folds colliding splats in.  Shared by the BA handle
// (dmv_ba_ref_source) and the host adapter (WindowBA::coarseTrackingRefInputs).
#pragma once
#include <vector>

namespace dmv {
// one host frame's points [b, e) (indices of a list ordered by host frame); alive[i] = point i still has a residual.
// Returns the surviving points in their order after the removal: the reference's loop, replayed on indices.
inline std::vector<int> remove_outliers_order(int b, int e, const std::vector<char>& alive) {
  std::vector<int> list;
  list.reserve(e > b ? e - b : 0);
  for (int i = b; i < e; i++) list.push_back(i);
  for (int i = 0; i < (int)list.size(); i++)
    if (!alive[list[i]]) {
      list[i] = list.back();
      list.pop_back();
      i--;
    }
  return list;
}
}  // namespace dmv
