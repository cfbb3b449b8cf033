// DeltaXYWHBBoxCoder arithmetic shared by the RPN targets (rpn_train.cu) and the RoI head (roi_head.cu), in the reference's fp32
// operation order (delta_xywh_bbox_coder.py:98-270).  __f*_rn intrinsics are never contracted, so every step rounds as torch's CPU ops do.
#pragma once
#include "ptb_common.cuh"

namespace ptb {

// bbox2delta(p, g) then (delta - mean) / std
__device__ __forceinline__ float4 bbox2delta(const float4 p, const float4 q, const float (&mean)[4], const float (&stdv)[4]) {
  const float px = __fmul_rn(__fadd_rn(p.x, p.z), 0.5f), py = __fmul_rn(__fadd_rn(p.y, p.w), 0.5f);
  const float pw = __fsub_rn(p.z, p.x), ph = __fsub_rn(p.w, p.y);
  const float gx = __fmul_rn(__fadd_rn(q.x, q.z), 0.5f), gy = __fmul_rn(__fadd_rn(q.y, q.w), 0.5f);
  const float gw = __fsub_rn(q.z, q.x), gh = __fsub_rn(q.w, q.y);
  const float dx = __fdiv_rn(__fsub_rn(gx, px), pw), dy = __fdiv_rn(__fsub_rn(gy, py), ph);
  const float dw = logf(__fdiv_rn(gw, pw)), dh = logf(__fdiv_rn(gh, ph));
  return make_float4(__fdiv_rn(__fsub_rn(dx, mean[0]), stdv[0]), __fdiv_rn(__fsub_rn(dy, mean[1]), stdv[1]),
                     __fdiv_rn(__fsub_rn(dw, mean[2]), stdv[2]), __fdiv_rn(__fsub_rn(dh, mean[3]), stdv[3]));
}

}  // namespace ptb
