// Loss term of the CPR positive bags, as a functor pair (value, d/dp) shared by the MIL forward / backward kernels (mil.cu) and the
// map-level backward (loss_bwd.cu):
//   GfocalTerm  MILLoss.gfocal_loss (multi_instance_learning_loss.py:148-151), multiplied by the label weight of the bag / sample;
//   BceTerm     F.binary_cross_entropy(p, t, weight=None) as MILLoss / AllPosLoss call it (:187-202, :229-240): NOT weighted, so a bag
//               whose weights are all zero (prob = 0 exactly) still adds 100 at its label column (ATen clamps log at -100).
// BceTerm follows ATen's CPU formula: (t - 1) * max(log1p(-p), -100) - t * max(log p, -100), d/dp = (p - t) / max((1 - p) p, 1e-12).
// The clamps are written as ATen's std::max(x, -100) so that a NaN (p > 1 after rounding, where ATen raises) stays NaN.
#pragma once

namespace ptb {

enum CprLossKind { LOSS_GFOCAL = 0, LOSS_BCE = 1 };

__device__ __forceinline__ float gfocal_elem(float p, float q, float eps) {
  // -( (p-q)^2 * ( q*log(p+eps) + (1-q)*log(1-p+eps) ) )
  const float l1 = (p - q) * (p - q);
  const float l2 = q * logf(p + eps) + (1.f - q) * logf(1.f - p + eps);
  return -(l1 * l2);
}
__device__ __forceinline__ float gfocal_dp(float p, float q, float eps) {
  const float d = p - q;
  const float L = q * logf(p + eps) + (1.f - q) * logf(1.f - p + eps);
  const float dL = q / (p + eps) - (1.f - q) / (1.f - p + eps);
  return -(2.f * d * L + d * d * dL);
}
__device__ __forceinline__ float gfocal_dp_f(float p, float q, float eps) {      // fast-intrinsic form used by the map backward
  const float d = p - q;
  const float L = q * __logf(p + eps) + (1.f - q) * __logf(1.f - p + eps);
  const float dL = __fdividef(q, p + eps) - __fdividef(1.f - q, 1.f - p + eps);
  return -(2.f * d * L + d * d * dL);
}

__device__ __forceinline__ float aten_log_clamp(float x) { return x < -100.f ? -100.f : x; }   // std::max(x, -100.f)

struct GfocalTerm {
  static constexpr bool label_weighted = true;
  float eps;
  __device__ __forceinline__ float value(float p, float q) const { return gfocal_elem(p, q, eps); }
  __device__ __forceinline__ float dp(float p, float q) const { return gfocal_dp(p, q, eps); }
  __device__ __forceinline__ float dp_fast(float p, float q) const { return gfocal_dp_f(p, q, eps); }
};

struct BceTerm {
  static constexpr bool label_weighted = false;
  float eps;                                    // unused: F.binary_cross_entropy has no eps
  __device__ __forceinline__ float value(float p, float q) const {
    return (q - 1.f) * aten_log_clamp(log1pf(-p)) - q * aten_log_clamp(logf(p));
  }
  __device__ __forceinline__ float dp(float p, float q) const {
    const float v = (1.f - p) * p;
    return (p - q) / (v < 1e-12f ? 1e-12f : v);                               // std::max(v, 1e-12f)
  }
  __device__ __forceinline__ float dp_fast(float p, float q) const { return dp(p, q); }
};

}  // namespace ptb
