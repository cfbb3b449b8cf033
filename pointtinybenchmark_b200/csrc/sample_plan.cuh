// The RandomSampler plan shared by the RPN targets (rpn_train.cu) and the RoI targets (roi_head.cu): a header [B][2] of (offset, count)
// for the positives and the negatives of each image (count -1: every candidate is sampled, no draw), then each (image, kind)'s drawn
// candidate ranks in ascending order (ptb_rpn_anchor_targets in include/ptb_b200.h).
#pragma once
#include "ptb_common.cuh"

namespace ptb {

// output slot of candidate rank r of (image b, kind 0 pos / 1 neg) in the sampled list, -1 when it is not sampled
__device__ __forceinline__ int sampled_slot(const int32_t* __restrict__ plan, int b, int kind, int r) {
  const int off = plan[(b * 2 + kind) * 2], cnt = plan[(b * 2 + kind) * 2 + 1];
  if (cnt < 0) return r;
  int lo = 0, hi = cnt;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (plan[off + mid] < r) lo = mid + 1; else hi = mid;
  }
  return (lo < cnt && plan[off + lo] == r) ? lo : -1;
}

}  // namespace ptb
