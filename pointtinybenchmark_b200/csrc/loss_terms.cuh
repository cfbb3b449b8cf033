// The elementwise loss terms and the fixed-order loss-sum kernel shared by the P2P head (p2p.cu) and the RPN head (rpn_train.cu).
#pragma once
#include "ptb_common.cuh"

namespace ptb {

// An elementwise loss is a functor over element e:  op(e, want_loss, grad, sc) returns e's term of the loss sum (read only when
// want_loss) and, when grad is set, stores grad[e] = sc * d term / dx[e].  The kernel owns the loop and the sum.
template <class Loss>
__global__ void __launch_bounds__(256)
loss_sum_kernel(Loss op, long long n, float* loss_sum, const float* __restrict__ scale, float* __restrict__ grad,
                SumScratch* __restrict__ scr) {
  const float sc = (grad && scale) ? scale[0] : 1.f;
  float acc = 0.f;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < n; e += (long long)gridDim.x * 256)
    acc += op(e, loss_sum != nullptr, grad, sc);
  if (loss_sum) block_partial_finish(acc, *scr, loss_sum);
}

// SmoothL1Loss (smooth_l1_loss.py:25-31) on the normalised points
struct SmoothL1Loss {
  const float* pred; const float* target; const float* weight; float inv_norm, beta;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const float w = weight ? weight[e] : 1.f;
    const float diff = (pred[e] - target[e]) * inv_norm;
    const float d = fabsf(diff);
    // a NaN diff keeps its NaN gradient (0 * |diff|), as torch's does through the unselected branch of torch.where
    if (grad) grad[e] = sc * w * inv_norm * (d < beta ? diff / beta : (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f * d)));
    return (d < beta ? 0.5f * d * d / beta : d - 0.5f * beta) * w;
  }
};

// CrossEntropyLoss(use_sigmoid=True) = binary_cross_entropy (cross_entropy_loss.py:42-89): labels expanded to one-hot rows
// (_expand_onehot_labels; a label outside [0, C), e.g. the background label C, is an all-zero row), the per-proposal weight
// broadcast over the classes, F.binary_cross_entropy_with_logits(reduction='none') in ATen's CPU form
//   (1 - t) * x - log_sigmoid(x),   log_sigmoid(x) = min(x, 0) - log1p(exp(-|x|)),
// then the weighted sum of weight_reduce_loss (the caller divides by avg_factor).  d/dx = sigmoid(x) - t.
// POS_WEIGHT: CrossEntropyLoss.class_weight, which binary_cross_entropy passes as pos_weight (cross_entropy_loss.py:85-86), in
// ATen's CPU order: log_weight = (pw_c - 1) * t + 1, loss = (1 - t) * x - log_sigmoid(x) * log_weight; d/dx = (pw_c t + 1 - t)
// sigmoid(x) - pw_c t (binary_cross_entropy_with_logits_backward).  Without it this is the class_weight=None form above.
// The log is computed only when the sum is wanted: the backward launch skips it.
template <bool POS_WEIGHT>
struct SigmoidBCELoss {
  const float* x; const int64_t* labels; const float* weight; const float* pos_weight; int C;
  __device__ __forceinline__ float operator()(long long e, bool want_loss, float* grad, float sc) const {
    const long long m = e / C;
    const int c = (int)(e - m * C);
    const float w = weight ? weight[m] : 1.f;
    const float t = (labels[m] == c) ? 1.f : 0.f;
    const float v = x[e];
    float term = 0.f;
    if constexpr (POS_WEIGHT) {
      const float pw = pos_weight[c];
      if (want_loss) {
        const float log_sig = __fsub_rn(fminf(v, 0.f), log1pf(expf(-fabsf(v))));
        const float log_w = __fadd_rn(__fmul_rn(__fsub_rn(pw, 1.f), t), 1.f);
        term = __fmul_rn(__fsub_rn(__fmul_rn(1.f - t, v), __fmul_rn(log_sig, log_w)), w);
      }
      if (grad) {
        const float pt = __fmul_rn(pw, t);
        grad[e] = sc * w * __fsub_rn(__fmul_rn(__fsub_rn(__fadd_rn(pt, 1.f), t), sigmoidf_acc(v)), pt);
      }
    } else {
      if (want_loss) {
        const float log_sig = __fsub_rn(fminf(v, 0.f), log1pf(expf(-fabsf(v))));
        term = __fmul_rn(__fsub_rn(__fmul_rn(1.f - t, v), log_sig), w);
      }
      if (grad) grad[e] = sc * w * (sigmoidf_acc(v) - t);
    }
    return term;
  }
};

// L1Loss on the normalised points (row_inv_norm NULL: on the raw values): |d| * weight; d/dpred = sgn(d) * inv * weight.  ATen's abs backward multiplies by sgn(d), which is
// 0 at d == 0 and at a NaN d, so a NaN difference has gradient 0 (its loss term is NaN)
struct L1RowsLoss {
  const float* pred; const float* target; const float* weight; const float* row_inv_norm;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const float inv = row_inv_norm ? row_inv_norm[e >> 1] : 1.f;
    const float w = weight ? weight[e] : 1.f;
    const float d = (pred[e] - target[e]) * inv;
    if (grad) grad[e] = sc * w * inv * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
    return fabsf(d) * w;
  }
};

// The RoI head's box loss (bbox_head.py:282-306): element e = 4 m + k of the (R, 4) targets.  Only positive rows (label in
// [0, num_classes)) count; their prediction is column 4 * label + k of bbox_pred (R, ld), or column k when class-agnostic.  L1Loss
// |d| * w or SmoothL1Loss (beta) on d = pred - target; the gradient is written at that column only (the caller zeroes the rest).
template <bool SMOOTH>
struct RoIBoxLoss {
  const float* pred; const int64_t* labels; const float* target; const float* weight; int ld, num_classes, agnostic; float beta;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const long long m = e >> 2;
    const int k = (int)(e & 3);
    const long long lab = labels[m];
    if (lab < 0 || lab >= num_classes) return 0.f;
    const long long col = m * ld + (agnostic ? k : 4 * lab + k);
    const float w = weight[e];
    const float diff = pred[col] - target[e];
    const float d = fabsf(diff);
    const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
    if constexpr (SMOOTH) {
      if (grad) grad[col] = sc * w * (d < beta ? diff / beta : sgn);
      return (d < beta ? 0.5f * d * d / beta : d - 0.5f * beta) * w;
    } else {
      if (grad) grad[col] = sc * w * sgn;
      return d * w;
    }
  }
};

}  // namespace ptb
