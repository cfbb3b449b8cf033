// RPN training targets and losses for dense anchors (SURVEY.md §8f rank 4, BASELINE.json configs[3]) — replaces the per-image Python
// of AnchorHead.get_targets / loss (mmdet/models/dense_heads/anchor_head.py:171-267, 269-365, 422-482) and the index work of
// RandomSampler (mmdet/core/bbox/samplers/random_sampler.py:31-80, base_sampler.py:34-99).  Per batch of B images:
//
//   rpn_inside_kernel     CTA per image: walks the image's anchors in the reference's flat (level, y, x, anchor) order, tests each
//                         against the host-made inside box of its (level, anchor) — valid flags of pad_shape and, when allowed_border
//                         >= 0, the border test against img_shape (core/anchor/utils.py:20-45) — and compacts the inside anchors
//                         (base[a] + (x*sx, y*sy, x*sx, y*sy) in fp32, AnchorGenerator.single_level_grid_anchors) with a block scan.
//   ptb_max_iou_assign    per image on its inside anchors (assign.cu, unchanged).
//   rpn_candidate_kernel  CTA per image: segmented scan of the assignment: each inside anchor's rank among the image's positives
//                         (gt_inds > 0) or negatives (gt_inds == 0), and the two counts — the only data the host reads back.
//   (host)                the reference's randperm draws from the counts; the chosen ranks come back in one upload.
//   rpn_targets_kernel    thread per anchor, in the layout of the head's output maps (labels / label_weights like cls_score
//                         (B, A, H, W), bbox_targets / bbox_weights like bbox_pred (B, 4A, H, W), levels one after the other), so
//                         the loss reads the maps in place: unmap, sampling, bbox2delta (delta_xywh_bbox_coder.py:98-140) in fp32.
//   rpn_sampled_kernel    RandomSampler alone: the sampled positive / negative index lists (SamplingResult.pos_inds / neg_inds).
//   ptb_rpn_level_loss    per level the fixed-order sums of CrossEntropyLoss(use_sigmoid=True) and L1Loss / SmoothL1Loss over the
//                         maps (loss_terms.cuh), or their gradients in the maps' layout.
// Integer results (ranks, counts, labels, weights, sampled sets) are exact; every sum has a fixed order.
#include "ptb_common.cuh"
#include "loss_terms.cuh"
#include "box_coder.cuh"
#include "sample_plan.cuh"

namespace ptb {
namespace {

constexpr int RT_THREADS = 1024;

// exclusive block prefix of a 0/1 flag over RT_THREADS threads; *total gets the block's count.  s must hold 33 ints.
__device__ __forceinline__ int block_excl_scan(bool flag, int* s, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  const int pre = __popc(m & ((1u << lane) - 1u));
  if (lane == 0) s[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    const int v = s[lane];
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    s[lane] = inc - v;
    if (lane == 31) s[32] = inc;
  }
  __syncthreads();
  const int r = s[warp] + pre;
  *total = s[32];
  __syncthreads();
  return r;
}

struct RtLevels {                     // by-value kernel argument
  int L, A;
  int H[PTB_RPN_MAX_LEVELS], W[PTB_RPN_MAX_LEVELS], sx[PTB_RPN_MAX_LEVELS], sy[PTB_RPN_MAX_LEVELS];
  int anchor_off[PTB_RPN_MAX_LEVELS + 1];      // flat anchor offset of each level inside one image
};

__device__ __forceinline__ int level_of(const RtLevels& lv, int i) {
  int l = 0;
  while (l + 1 < lv.L && i >= lv.anchor_off[l + 1]) ++l;
  return l;
}

__global__ void __launch_bounds__(RT_THREADS)
rpn_inside_kernel(const float4* __restrict__ base /*[L][A]*/, RtLevels lv, const int4* __restrict__ inside_box /*[B][L][A]*/,
                  float4* __restrict__ inside_anchors /*[B][N]*/, int32_t* __restrict__ inside_idx /*[B][N]*/,
                  int32_t* __restrict__ n_inside /*[B]*/) {
  __shared__ int s[33];
  const int b = blockIdx.x, N = lv.anchor_off[lv.L];
  int done = 0;
  for (int i0 = 0; i0 < N; i0 += RT_THREADS) {
    const int i = i0 + threadIdx.x;
    bool in = false;
    float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < N) {
      const int l = level_of(lv, i);
      const int q = i - lv.anchor_off[l];
      const int cell = q / lv.A, a = q - cell * lv.A;
      const int y = cell / lv.W[l], x = cell - y * lv.W[l];
      const int4 r = inside_box[(b * lv.L + l) * lv.A + a];                  // [x0, x1) x [y0, y1)
      in = x >= r.x && x < r.y && y >= r.z && y < r.w;
      const float4 ba = base[l * lv.A + a];
      const float fx = (float)(x * lv.sx[l]), fy = (float)(y * lv.sy[l]);
      box = make_float4(__fadd_rn(ba.x, fx), __fadd_rn(ba.y, fy), __fadd_rn(ba.z, fx), __fadd_rn(ba.w, fy));
    }
    int tot;
    const int r = block_excl_scan(in, s, &tot);
    if (i < N) {
      inside_idx[(long long)b * N + i] = in ? done + r : -1;
      if (in) inside_anchors[(long long)b * N + done + r] = box;
    }
    done += tot;
  }
  if (threadIdx.x == 0) n_inside[b] = done;
}

__global__ void __launch_bounds__(RT_THREADS)
rpn_candidate_kernel(const int64_t* __restrict__ gt_inds /*[B][N]*/, const int32_t* __restrict__ n_inside, int N,
                     int32_t* __restrict__ rank /*[B][N]*/, int32_t* __restrict__ counts /*[B][2]*/) {
  __shared__ int s[33];
  const int b = blockIdx.x, n = n_inside[b];
  int npos = 0, nneg = 0;
  for (int j0 = 0; j0 < n; j0 += RT_THREADS) {
    const int j = j0 + threadIdx.x;
    const long long g = j < n ? gt_inds[(long long)b * N + j] : -1;
    int tp, tn;
    const int rp = block_excl_scan(g > 0, s, &tp);
    const int rn = block_excl_scan(g == 0, s, &tn);
    if (j < n) rank[(long long)b * N + j] = g > 0 ? npos + rp : (g == 0 ? nneg + rn : -1);
    npos += tp;
    nneg += tn;
  }
  if (threadIdx.x == 0) { counts[2 * b] = npos; counts[2 * b + 1] = nneg; }
}

struct EncodeCfg {
  float mean[4], stdv[4];
  float pos_weight;
};

__global__ void __launch_bounds__(256)
rpn_targets_kernel(RtLevels lv, int B, const int32_t* __restrict__ inside_idx, const float4* __restrict__ inside_anchors,
                   const int64_t* __restrict__ gt_inds, const int32_t* __restrict__ rank, const int32_t* __restrict__ plan,
                   const float4* __restrict__ gt /*concatenated*/, const int32_t* __restrict__ gt_off /*[B+1]*/, EncodeCfg ec,
                   int64_t* __restrict__ labels, float* __restrict__ label_w, float* __restrict__ bbox_t, float* __restrict__ bbox_w) {
  const int N = lv.anchor_off[lv.L];
  const long long total = (long long)B * N;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    // e runs over the maps' layout: level l's block of B*A*H*W elements starts at B * anchor_off[l]
    const int l = level_of(lv, (int)(e / B));
    const long long lo = (long long)B * lv.anchor_off[l];
    const int H = lv.H[l], W = lv.W[l], A = lv.A, HW = H * W;
    long long t = e - lo;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H); t /= H;
    const int a = (int)(t % A);
    const int b = (int)(t / A);
    const int i = lv.anchor_off[l] + (y * W + x) * A + a;
    const long long row = (long long)b * N;
    int64_t lab = 1;                                      // background = num_classes (1)
    float lw = 0.f;
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    float bw = 0.f;
    const int j = inside_idx[row + i];
    if (j >= 0) {
      const long long g = gt_inds[row + j];
      const int r = rank[row + j];
      if (g > 0 && sampled_slot(plan, b, 0, r) >= 0) {
        lab = 0;
        lw = ec.pos_weight > 0.f ? ec.pos_weight : 1.f;
        bw = 1.f;
        d = bbox2delta(inside_anchors[row + j], gt[gt_off[b] + (int)(g - 1)], ec.mean, ec.stdv);
      } else if (g == 0 && sampled_slot(plan, b, 1, r) >= 0) {
        lw = 1.f;
      }
    }
    labels[e] = lab;
    label_w[e] = lw;
    const long long rb = 4 * lo + ((long long)(b * 4 * A + a * 4) * H + y) * W + x;    // channel a*4 + k of bbox_pred
    const float dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      bbox_t[rb + (long long)k * HW] = dv[k];
      bbox_w[rb + (long long)k * HW] = bw;
    }
  }
}

__global__ void __launch_bounds__(256)
rpn_sampled_kernel(const int64_t* __restrict__ gt_inds, const int32_t* __restrict__ rank, int n, const int32_t* __restrict__ plan,
                   int64_t* __restrict__ pos_inds, int64_t* __restrict__ neg_inds) {
  for (int j = blockIdx.x * 256 + threadIdx.x; j < n; j += gridDim.x * 256) {
    const long long g = gt_inds[j];
    if (g < 0) continue;
    const int slot = sampled_slot(plan, 0, g > 0 ? 0 : 1, rank[j]);
    if (slot >= 0) (g > 0 ? pos_inds : neg_inds)[slot] = j;
  }
}

int set_levels(RtLevels& lv, int L, int A, const int32_t* hw, const int32_t* strides) {
  if (L < 1 || L > PTB_RPN_MAX_LEVELS || A < 1) return 0;
  lv.L = L; lv.A = A;
  long long off = 0;
  for (int l = 0; l < L; ++l) {
    lv.H[l] = hw[2 * l]; lv.W[l] = hw[2 * l + 1]; lv.sx[l] = strides[2 * l]; lv.sy[l] = strides[2 * l + 1];
    if (lv.H[l] < 1 || lv.W[l] < 1) return 0;
    lv.anchor_off[l] = (int)off;
    off += (long long)lv.H[l] * lv.W[l] * A;
    if (off >= (1LL << 30)) return 0;
  }
  lv.anchor_off[L] = (int)off;
  return 1;
}

}  // namespace
}  // namespace ptb

using namespace ptb;

extern "C" int ptb_rpn_inside_anchors(const float* base_anchors, const int32_t* featmap_hw, const int32_t* strides, int L, int A, int B,
                                      const int32_t* inside_box, float* inside_anchors, int32_t* inside_idx, int32_t* n_inside,
                                      void* stream) {
  PTB_REQUIRE(featmap_hw && strides && B > 0, "shape");
  RtLevels lv;
  PTB_REQUIRE(set_levels(lv, L, A, featmap_hw, strides), "levels: 1..PTB_RPN_MAX_LEVELS non-empty maps, fewer than 2^30 anchors per image");
  PTB_REQUIRE(base_anchors && inside_box && inside_anchors && inside_idx && n_inside, "NULL input");
  PTB_REQUIRE((uintptr_t)base_anchors % 16 == 0 && (uintptr_t)inside_anchors % 16 == 0 && (uintptr_t)inside_box % 16 == 0,
              "16-byte aligned arrays");
  rpn_inside_kernel<<<B, RT_THREADS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(base_anchors), lv,
                                                                  reinterpret_cast<const int4*>(inside_box),
                                                                  reinterpret_cast<float4*>(inside_anchors), inside_idx, n_inside);
  return check_launch("ptb_rpn_inside_anchors");
}

extern "C" int ptb_rpn_candidate_ranks(const int64_t* gt_inds, const int32_t* n_inside, int B, int N, int32_t* rank, int32_t* counts,
                                       void* stream) {
  PTB_REQUIRE(B > 0 && N >= 0, "shape");
  PTB_REQUIRE(gt_inds && n_inside && rank && counts, "NULL input");
  rpn_candidate_kernel<<<B, RT_THREADS, 0, (cudaStream_t)stream>>>(gt_inds, n_inside, N, rank, counts);
  return check_launch("ptb_rpn_candidate_ranks");
}

extern "C" int ptb_rpn_anchor_targets(const int32_t* featmap_hw, const int32_t* strides, int L, int A, int B, const int32_t* inside_idx,
                                      const float* inside_anchors, const int64_t* gt_inds, const int32_t* rank, const int32_t* plan,
                                      const float* gt_bboxes, const int32_t* gt_off, const float* means, const float* stds,
                                      float pos_weight, int64_t* labels, float* label_weights, float* bbox_targets, float* bbox_weights,
                                      void* stream) {
  PTB_REQUIRE(featmap_hw && strides && means && stds && B > 0, "shape");
  RtLevels lv;
  PTB_REQUIRE(set_levels(lv, L, A, featmap_hw, strides), "levels: 1..PTB_RPN_MAX_LEVELS non-empty maps, fewer than 2^30 anchors per image");
  PTB_REQUIRE(inside_idx && inside_anchors && gt_inds && rank && plan && gt_off && labels && label_weights && bbox_targets && bbox_weights,
              "NULL input");
  PTB_REQUIRE((uintptr_t)inside_anchors % 16 == 0 && (uintptr_t)gt_bboxes % 16 == 0, "16-byte aligned boxes");
  EncodeCfg ec;
  for (int k = 0; k < 4; ++k) { ec.mean[k] = means[k]; ec.stdv[k] = stds[k]; }
  ec.pos_weight = pos_weight;
  const long long total = (long long)B * lv.anchor_off[L];
  const int blocks = (int)std::min<long long>((total + 255) / 256, 16LL * sm_count());
  rpn_targets_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(lv, B, inside_idx, reinterpret_cast<const float4*>(inside_anchors), gt_inds,
                                                               rank, plan, reinterpret_cast<const float4*>(gt_bboxes), gt_off, ec, labels,
                                                               label_weights, bbox_targets, bbox_weights);
  return check_launch("ptb_rpn_anchor_targets");
}

extern "C" int ptb_rpn_sampled_indices(const int64_t* gt_inds, const int32_t* rank, int n, const int32_t* plan, int64_t* pos_inds,
                                       int64_t* neg_inds, void* stream) {
  PTB_REQUIRE(n >= 0, "shape");
  if (n == 0) return 0;
  PTB_REQUIRE(gt_inds && rank && plan, "NULL input");
  const int blocks = std::min((n + 255) / 256, 8 * sm_count());
  rpn_sampled_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(gt_inds, rank, n, plan, pos_inds, neg_inds);
  return check_launch("ptb_rpn_sampled_indices");
}

extern "C" int ptb_rpn_level_loss(const float* cls_score, const float* bbox_pred, const int64_t* labels, const float* label_weights,
                                  const float* bbox_targets, const float* bbox_weights, int64_t M, int bbox_loss, float beta,
                                  float* loss_sum, const float* scale, float* grad_cls, float* grad_bbox, void* stream) {
  PTB_REQUIRE(M >= 0 && (bbox_loss == PTB_RPN_LOSS_L1 || (bbox_loss == PTB_RPN_LOSS_SMOOTH_L1 && beta > 0.f)),
              "shape / loss kind (SmoothL1 needs beta > 0)");
  if (M == 0) return 0;
  PTB_REQUIRE(cls_score && bbox_pred && labels && label_weights && bbox_targets && bbox_weights, "NULL input");
  PTB_REQUIRE(loss_sum ? !(grad_cls || grad_bbox) : (grad_cls && grad_bbox), "either loss_sum or both gradients");
  const char* name = "ptb_rpn_level_loss";
  int rc = launch_sum(loss_sum_kernel<SigmoidBCELoss<false>>, stream, name,
                      SigmoidBCELoss<false>{cls_score, labels, label_weights, nullptr, 1}, M, loss_sum, scale, grad_cls);
  if (rc) return rc;
  float* bsum = loss_sum ? loss_sum + 1 : nullptr;
  const float* bscale = scale ? scale + 1 : nullptr;
  if (bbox_loss == PTB_RPN_LOSS_L1)
    return launch_sum(loss_sum_kernel<L1RowsLoss>, stream, name, L1RowsLoss{bbox_pred, bbox_targets, bbox_weights, nullptr}, 4 * M,
                      bsum, bscale, grad_bbox);
  return launch_sum(loss_sum_kernel<SmoothL1Loss>, stream, name, SmoothL1Loss{bbox_pred, bbox_targets, bbox_weights, 1.f, beta}, 4 * M,
                    bsum, bscale, grad_bbox);
}
