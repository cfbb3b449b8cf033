// FCOS head (mmdet/models/dense_heads/fcos_head.py): point targets, the centerness-weighted IoU / GIoU box loss, the soft-target
// centerness loss and the per-level top-k decode.  Rows are ordered as the reference flattens them in `loss`: level after level, image
// after image inside a level, then y, x.  Every row's point is x * stride + stride // 2 (fcos_head.py:472-482), formed from the row index.
#include "ptb_common.cuh"
#include "loss_terms.cuh"
#include "topk_select.cuh"
#include <math_constants.h>

namespace ptb {

constexpr int FCOS_MAX_LEVELS = 8;
constexpr float FCOS_INF = 1e8f;         // fcos_head.py:12, exact in fp32

struct FcosLevels {
  int L, B;
  long long row0[FCOS_MAX_LEVELS + 1];   // first row of level l; row0[L] = every row of the batch
  int H[FCOS_MAX_LEVELS], W[FCOS_MAX_LEVELS];
  float stride[FCOS_MAX_LEVELS], half[FCOS_MAX_LEVELS];
};

struct FcosPoint {
  int l, b;
  long long cell;
  float x, y;
};

__device__ __forceinline__ FcosPoint fcos_point(const FcosLevels& lv, long long m) {
  int l = 0;
  while (l + 1 < lv.L && m >= lv.row0[l + 1]) ++l;
  const long long r = m - lv.row0[l], hw = (long long)lv.H[l] * lv.W[l];
  FcosPoint p;
  p.l = l;
  p.b = (int)(r / hw);
  p.cell = r - (long long)p.b * hw;
  const int yi = (int)(p.cell / lv.W[l]), xi = (int)(p.cell - (long long)yi * lv.W[l]);
  p.x = __fadd_rn(__fmul_rn((float)xi, lv.stride[l]), lv.half[l]);
  p.y = __fadd_rn(__fmul_rn((float)yi, lv.stride[l]), lv.half[l]);
  return p;
}

// centerness_target (fcos_head.py:629-648): sqrt(min(l, r) / max(l, r) * (min(t, b) / max(t, b)))
__device__ __forceinline__ float fcos_centerness(const float* t) {
  return __fsqrt_rn(__fmul_rn(__fdiv_rn(fminf(t[0], t[2]), fmaxf(t[0], t[2])), __fdiv_rn(fminf(t[1], t[3]), fmaxf(t[1], t[3]))));
}

__device__ __forceinline__ bool fcos_pos(const int64_t* labels, long long m, int C) { return labels[m] >= 0 && labels[m] < C; }

// ------------------------------------------------------------------------------------------------
// targets: _get_target_single (fcos_head.py:552-627) for every (image, point), one thread per row, the image's GTs scanned in order
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fcos_targets_kernel(FcosLevels lv, const float* __restrict__ gt, const int64_t* __restrict__ gt_labels, const int32_t* __restrict__ gt_off,
                    const float* __restrict__ ranges, const float* __restrict__ radius_px, int norm_on_bbox, int num_classes,
                    int64_t* __restrict__ labels, float* __restrict__ targets) {
  const long long N = lv.row0[lv.L];
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < N; m += (long long)gridDim.x * blockDim.x) {
    const FcosPoint p = fcos_point(lv, m);
    const int g0 = gt_off[p.b], g1 = gt_off[p.b + 1];
    float* out = targets + m * 4;
    if (g1 == g0) {                                     // no GT: background and zero targets (fcos_head.py:557-559)
      labels[m] = num_classes;
      out[0] = out[1] = out[2] = out[3] = 0.f;
      continue;
    }
    const float lo = ranges[2 * p.l], hi = ranges[2 * p.l + 1];
    float best = 0.f;
    int bi = g0;
    for (int j = g0; j < g1; ++j) {
      const float* g = gt + (size_t)j * 4;
      const float d0 = __fsub_rn(p.x, g[0]), d1 = __fsub_rn(p.y, g[1]), d2 = __fsub_rn(g[2], p.x), d3 = __fsub_rn(g[3], p.y);
      bool inside;
      if (radius_px) {
        // centre box of stride * radius around the GT centre, clipped to the GT with torch.where (fcos_head.py:584-607)
        const float cx = __fdiv_rn(__fadd_rn(g[0], g[2]), 2.f), cy = __fdiv_rn(__fadd_rn(g[1], g[3]), 2.f), s = radius_px[p.l];
        const float xmin = __fsub_rn(cx, s), ymin = __fsub_rn(cy, s), xmax = __fadd_rn(cx, s), ymax = __fadd_rn(cy, s);
        const float c0 = xmin > g[0] ? xmin : g[0], c1 = ymin > g[1] ? ymin : g[1];
        const float c2 = xmax > g[2] ? g[2] : xmax, c3 = ymax > g[3] ? g[3] : ymax;
        inside = fminf(fminf(__fsub_rn(p.x, c0), __fsub_rn(p.y, c1)), fminf(__fsub_rn(c2, p.x), __fsub_rn(c3, p.y))) > 0.f;
      } else {
        inside = fminf(fminf(d0, d1), fminf(d2, d3)) > 0.f;
      }
      const float mx = fmaxf(fmaxf(d0, d1), fmaxf(d2, d3));
      const bool in_range = mx >= lo && mx <= hi;
      const float area = (inside && in_range) ? __fmul_rn(__fsub_rn(g[2], g[0]), __fsub_rn(g[3], g[1])) : FCOS_INF;
      if (j == g0 || area < best) {                     // ties: the first minimum, as Tensor.min(dim) on the CPU
        best = area;
        bi = j;
      }
    }
    const float* g = gt + (size_t)bi * 4;
    float t[4] = {__fsub_rn(p.x, g[0]), __fsub_rn(p.y, g[1]), __fsub_rn(g[2], p.x), __fsub_rn(g[3], p.y)};
    labels[m] = best == FCOS_INF ? (int64_t)num_classes : gt_labels[bi];
#pragma unroll
    for (int k = 0; k < 4; ++k) out[k] = norm_on_bbox ? __fdiv_rn(t[k], lv.stride[p.l]) : t[k];
  }
}

// ------------------------------------------------------------------------------------------------
// loss normalisers and losses over the fixed-order sum shell (loss_terms.cuh); negative rows add 0 and get a zero gradient
// ------------------------------------------------------------------------------------------------
struct FcosPosCount {
  const int64_t* labels; int C;
  __device__ __forceinline__ float operator()(long long m, bool, float*, float) const { return fcos_pos(labels, m, C) ? 1.f : 0.f; }
};

struct FcosCenternessSum {
  const int64_t* labels; const float* target; int C;
  __device__ __forceinline__ float operator()(long long m, bool, float*, float) const {
    return fcos_pos(labels, m, C) ? fcos_centerness(target + m * 4) : 0.f;
  }
};

// gradient share of torch.maximum / torch.minimum: the winner takes it all, a tie splits it
__device__ __forceinline__ float win(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }

// IoULoss (linear or -log) / GIoULoss (iou_loss.py:14-34, 87-101, 223-260, 330-365) on distance2bbox of the prediction and the target
// (transforms.py:144-160), aligned bbox_overlaps in mmdet's fp32 order (iou2d_calculator.py:213-260), weighted by the centerness target
enum { FCOS_IOU_LOG = 0, FCOS_IOU_LINEAR = 1, FCOS_GIOU = 2 };

struct FcosBoxLoss {
  FcosLevels lv; const int64_t* labels; const float* pred; const float* target; int C, mode; float overlap_eps, eps;
  __device__ __forceinline__ float operator()(long long m, bool, float* grad, float sc) const {
    if (!fcos_pos(labels, m, C)) {
      if (grad) reinterpret_cast<float4*>(grad)[m] = make_float4(0.f, 0.f, 0.f, 0.f);
      return 0.f;
    }
    const FcosPoint p = fcos_point(lv, m);
    const float* d = pred + m * 4;
    const float* t = target + m * 4;
    const float w = fcos_centerness(t);
    const float x1 = __fsub_rn(p.x, d[0]), y1 = __fsub_rn(p.y, d[1]), x2 = __fadd_rn(p.x, d[2]), y2 = __fadd_rn(p.y, d[3]);
    const float u1 = __fsub_rn(p.x, t[0]), v1 = __fsub_rn(p.y, t[1]), u2 = __fadd_rn(p.x, t[2]), v2 = __fadd_rn(p.y, t[3]);
    const float w1 = __fsub_rn(x2, x1), h1 = __fsub_rn(y2, y1);
    const float area1 = __fmul_rn(w1, h1), area2 = __fmul_rn(__fsub_rn(u2, u1), __fsub_rn(v2, v1));
    const float ltx = fmaxf(x1, u1), lty = fmaxf(y1, v1), rbx = fminf(x2, u2), rby = fminf(y2, v2);
    const float wx = __fsub_rn(rbx, ltx), wy = __fsub_rn(rby, lty);
    const float iw = fmaxf(wx, 0.f), ih = fmaxf(wy, 0.f);
    const float overlap = __fmul_rn(iw, ih);
    const float uni = __fsub_rn(__fadd_rn(area1, area2), overlap);
    const float eps_o = mode == FCOS_GIOU ? eps : overlap_eps;
    const float uc = fmaxf(uni, eps_o);
    const float iou = __fdiv_rn(overlap, uc);
    float loss, g_iou = 0.f, g_union = 0.f, g_earea = 0.f;
    float ex1 = 0.f, ey1 = 0.f, ex2 = 0.f, ey2 = 0.f, ew = 0.f, eh = 0.f, ea_raw = 0.f, ea = 1.f;
    if (mode == FCOS_GIOU) {
      ex1 = fminf(x1, u1); ey1 = fminf(y1, v1); ex2 = fmaxf(x2, u2); ey2 = fmaxf(y2, v2);
      ew = fmaxf(__fsub_rn(ex2, ex1), 0.f); eh = fmaxf(__fsub_rn(ey2, ey1), 0.f);
      ea_raw = __fmul_rn(ew, eh);
      ea = fmaxf(ea_raw, eps);
      const float giou = __fsub_rn(iou, __fdiv_rn(__fsub_rn(ea, uc), ea));
      loss = __fsub_rn(1.f, giou);
      g_iou = -1.f;
      g_union = -1.f / ea;                      // d loss / d union through the enclose term
      g_earea = uc / (ea * ea);
    } else {
      const float ic = fmaxf(iou, eps);
      loss = mode == FCOS_IOU_LINEAR ? __fsub_rn(1.f, ic) : -logf(ic);
      g_iou = iou >= eps ? (mode == FCOS_IOU_LINEAR ? -1.f : -1.f / ic) : 0.f;
    }
    if (grad) {
      const float s = sc * w;
      // union = maximum(uni, eps), iou = overlap / union
      const float g_uc = g_union + g_iou * (-iou / uc);
      const float g_uni = g_uc * win(uni, eps_o);
      const float g_ov = g_iou / uc - g_uni;
      const float g_iw = wx >= 0.f ? g_ov * ih : 0.f, g_ih = wy >= 0.f ? g_ov * iw : 0.f;
      // area1 = (x2 - x1) * (y2 - y1), lt = maximum, rb = minimum
      float gx1 = -g_uni * h1 - g_iw * win(x1, u1), gx2 = g_uni * h1 + g_iw * win(u2, x2);
      float gy1 = -g_uni * w1 - g_ih * win(y1, v1), gy2 = g_uni * w1 + g_ih * win(v2, y2);
      if (mode == FCOS_GIOU) {
        const float g_ea = g_earea * win(ea_raw, eps);
        const float g_ew = __fsub_rn(ex2, ex1) >= 0.f ? g_ea * eh : 0.f, g_eh = __fsub_rn(ey2, ey1) >= 0.f ? g_ea * ew : 0.f;
        gx1 -= g_ew * win(u1, x1); gx2 += g_ew * win(x2, u2);
        gy1 -= g_eh * win(v1, y1); gy2 += g_eh * win(y2, v2);
      }
      // x1 = px - l, y1 = py - t, x2 = px + r, y2 = py + b
      reinterpret_cast<float4*>(grad)[m] = make_float4(-s * gx1, -s * gy1, s * gx2, s * gy2);
    }
    return __fmul_rn(loss, w);
  }
};

// CrossEntropyLoss(use_sigmoid=True) of the centerness logit against the soft centerness target: binary_cross_entropy_with_logits in
// ATen's CPU form (1 - t) x - log_sigmoid(x); d/dx = sigmoid(x) - t
struct FcosCenternessLoss {
  const int64_t* labels; const float* target; const float* x; int C;
  __device__ __forceinline__ float operator()(long long m, bool want_loss, float* grad, float sc) const {
    if (!fcos_pos(labels, m, C)) {
      if (grad) grad[m] = 0.f;
      return 0.f;
    }
    const float t = fcos_centerness(target + m * 4), v = x[m];
    if (grad) grad[m] = sc * __fsub_rn(sigmoidf_acc(v), t);
    if (!want_loss) return 0.f;
    const float log_sig = __fsub_rn(fminf(v, 0.f), log1pf(expf(-fabsf(v))));
    return __fsub_rn(__fmul_rn(__fsub_rn(1.f, t), v), log_sig);
  }
};

// ------------------------------------------------------------------------------------------------
// decode (fcos_head.py:384-431): per level and image the key max_c sigmoid(cls_c) * sigmoid(ctr), top nms_pre of it, then the gather
// ------------------------------------------------------------------------------------------------
struct FcosMaps {
  const float* cls[FCOS_MAX_LEVELS]; const float* reg[FCOS_MAX_LEVELS]; const float* ctr[FCOS_MAX_LEVELS];
  int rofs[FCOS_MAX_LEVELS + 1];          // first output row of level l; rofs[L] = R rows per image
  int select[FCOS_MAX_LEVELS];            // 1: the level's rows are a top-k of its keys, 0: all of them in index order
};

// one warp per (image, cell) of one level; sigmoid is monotone and fl(s * k) is monotone in s, so max_c fl(s_c * k) = fl(max_c s_c * k)
__global__ void __launch_bounds__(256)
fcos_key_kernel(const float* __restrict__ cls, const float* __restrict__ ctr, long long BQ, int C, float* __restrict__ key) {
  const long long wq = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wq >= BQ) return;
  const float* row = cls + wq * C;
  float mx = -CUDART_INF_F;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, sigmoidf_acc(row[c]));
  mx = warp_max(mx);
  if (lane == 0) key[wq] = __fmul_rn(mx, sigmoidf_acc(ctr[wq]));
}

// one warp per output row (image b, row r): the C scores, the centerness and the box, clipped to img_shape with torch.where
// (transforms.py:172-185) and divided by scale_factor when given (fcos_head.py:433-435)
__global__ void __launch_bounds__(256)
fcos_gather_kernel(FcosLevels lv, FcosMaps mp, int C, const float* __restrict__ img_hw, const float* __restrict__ scale_factor,
                   int32_t* __restrict__ idx, float* __restrict__ boxes, float* __restrict__ scores, float* __restrict__ ctr_out) {
  const int R = mp.rofs[lv.L];
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)lv.B * R) return;
  const int b = (int)(w / R), r = (int)(w - (long long)b * R);
  int l = 0;
  while (l + 1 < lv.L && r >= mp.rofs[l + 1]) ++l;
  int q;
  if (mp.select[l]) {
    q = idx[w];
  } else {
    q = r - mp.rofs[l];
    if (lane == 0) idx[w] = q;
  }
  const long long cell = (long long)b * lv.H[l] * lv.W[l] + q;
  const float* crow = mp.cls[l] + cell * C;
  float* srow = scores + w * C;
  for (int c = lane; c < C; c += 32) srow[c] = sigmoidf_acc(crow[c]);
  if (lane != 0) return;
  ctr_out[w] = sigmoidf_acc(mp.ctr[l][cell]);
  const int yi = q / lv.W[l], xi = q - yi * lv.W[l];
  const float px = __fadd_rn(__fmul_rn((float)xi, lv.stride[l]), lv.half[l]);
  const float py = __fadd_rn(__fmul_rn((float)yi, lv.stride[l]), lv.half[l]);
  const float* d = mp.reg[l] + cell * 4;
  float o[4] = {__fsub_rn(px, d[0]), __fsub_rn(py, d[1]), __fadd_rn(px, d[2]), __fadd_rn(py, d[3])};
  const float mh = img_hw[2 * b], mw = img_hw[2 * b + 1];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float mx = (k & 1) ? mh : mw;
    o[k] = o[k] < 0.f ? 0.f : o[k];
    o[k] = o[k] > mx ? mx : o[k];
    if (scale_factor) o[k] = __fdiv_rn(o[k], scale_factor[4 * b + k]);
  }
  reinterpret_cast<float4*>(boxes)[w] = make_float4(o[0], o[1], o[2], o[3]);
}

static int fcos_levels(FcosLevels& lv, int B, int L, const int32_t* hw, const float* strides) {
  PTB_REQUIRE(B > 0 && L >= 1 && L <= FCOS_MAX_LEVELS && hw && strides, "1 to 8 levels, B > 0");
  lv.L = L;
  lv.B = B;
  long long n = 0;
  for (int l = 0; l < L; ++l) {
    PTB_REQUIRE(hw[2 * l] > 0 && hw[2 * l + 1] > 0 && strides[l] > 0.f, "level shape");
    lv.H[l] = hw[2 * l]; lv.W[l] = hw[2 * l + 1];
    lv.stride[l] = strides[l];
    lv.half[l] = (float)((int)strides[l] / 2);
    lv.row0[l] = n;
    n += (long long)B * hw[2 * l] * hw[2 * l + 1];
  }
  lv.row0[L] = n;
  PTB_REQUIRE(n <= 0x7fffffffLL, "more than 2^31 - 1 points in the batch");
  return 0;
}

static unsigned grid_for(long long n, int per_block = 256) {
  const long long blocks = (n + per_block - 1) / per_block, cap = (long long)sm_count() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_fcos_targets(const float* gt_bboxes, const int64_t* gt_labels, const int32_t* gt_off, int B, int L, const int32_t* hw,
                                const float* strides, const float* ranges, const float* radius_px, int norm_on_bbox, int num_classes,
                                int64_t* out_labels, float* out_targets, void* stream) {
  FcosLevels lv = {};
  int rc;
  if ((rc = fcos_levels(lv, B, L, hw, strides))) return rc;
  PTB_REQUIRE(gt_off && ranges && out_labels && out_targets && num_classes > 0, "ptb_fcos_targets: arguments");
  fcos_targets_kernel<<<grid_for(lv.row0[L]), 256, 0, (cudaStream_t)stream>>>(lv, gt_bboxes, gt_labels, gt_off, ranges, radius_px,
                                                                               norm_on_bbox, num_classes, out_labels, out_targets);
  return check_launch("ptb_fcos_targets");
}

extern "C" int ptb_fcos_norm_sums(const int64_t* labels, const float* targets, int64_t N, int num_classes, float* out, void* stream) {
  PTB_REQUIRE(labels && targets && out && N >= 0 && num_classes > 0, "ptb_fcos_norm_sums: arguments");
  int rc;
  if ((rc = launch_sum(loss_sum_kernel<FcosPosCount>, stream, "ptb_fcos_norm_sums/count", FcosPosCount{labels, num_classes}, (long long)N,
                       out, (const float*)nullptr, (float*)nullptr)))
    return rc;
  return launch_sum(loss_sum_kernel<FcosCenternessSum>, stream, "ptb_fcos_norm_sums/centerness",
                    FcosCenternessSum{labels, targets, num_classes}, (long long)N, out + 1, (const float*)nullptr, (float*)nullptr);
}

extern "C" int ptb_fcos_bbox_loss(const float* pred, const float* targets, const int64_t* labels, int B, int L, const int32_t* hw,
                                  const float* strides, int num_classes, int mode, float overlap_eps, float eps, float* loss_sum,
                                  const float* scale, float* grad, void* stream) {
  FcosLevels lv = {};
  int rc;
  if ((rc = fcos_levels(lv, B, L, hw, strides))) return rc;
  PTB_REQUIRE(pred && targets && labels && num_classes > 0, "ptb_fcos_bbox_loss: arguments");
  PTB_REQUIRE(mode == FCOS_IOU_LOG || mode == FCOS_IOU_LINEAR || mode == FCOS_GIOU, "mode: 0 IoU (log), 1 IoU (linear), 2 GIoU");
  return launch_sum(loss_sum_kernel<FcosBoxLoss>, stream, "ptb_fcos_bbox_loss",
                    FcosBoxLoss{lv, labels, pred, targets, num_classes, mode, overlap_eps, eps}, lv.row0[L], loss_sum, scale, grad);
}

extern "C" int ptb_fcos_centerness_loss(const float* logits, const float* targets, const int64_t* labels, int64_t N, int num_classes,
                                        float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(logits && targets && labels && N >= 0 && num_classes > 0, "ptb_fcos_centerness_loss: arguments");
  return launch_sum(loss_sum_kernel<FcosCenternessLoss>, stream, "ptb_fcos_centerness_loss",
                    FcosCenternessLoss{labels, targets, logits, num_classes}, (long long)N, loss_sum, scale, grad);
}

extern "C" uint64_t ptb_fcos_decode_workspace(int B, int L, const int32_t* hw) {
  uint64_t m = 0;
  for (int l = 0; l < L && hw; ++l) m = max(m, (uint64_t)hw[2 * l] * hw[2 * l + 1]);
  return (uint64_t)B * m * sizeof(float);
}

extern "C" int ptb_fcos_decode(const float* const* cls_maps, const float* const* reg_maps, const float* const* ctr_maps, int L,
                               const int32_t* hw, const float* strides, int B, int num_classes, const float* img_hw,
                               const float* scale_factor, int nms_pre, int32_t* out_idx, float* out_boxes, float* out_scores,
                               float* out_ctr, void* workspace, uint64_t workspace_bytes, void* stream) {
  FcosLevels lv = {};
  int rc;
  if ((rc = fcos_levels(lv, B, L, hw, strides))) return rc;
  PTB_REQUIRE(cls_maps && reg_maps && ctr_maps && img_hw && out_idx && out_boxes && out_scores && out_ctr && num_classes > 0,
              "ptb_fcos_decode: arguments");
  FcosMaps mp = {};
  int R = 0;
  for (int l = 0; l < L; ++l) {
    PTB_REQUIRE(cls_maps[l] && reg_maps[l] && ctr_maps[l], "ptb_fcos_decode: NULL map");
    mp.cls[l] = cls_maps[l]; mp.reg[l] = reg_maps[l]; mp.ctr[l] = ctr_maps[l];
    const int hwl = hw[2 * l] * hw[2 * l + 1];
    mp.select[l] = nms_pre > 0 && nms_pre < hwl;       // get_k_for_topk (onnx_helper.py:45-78)
    mp.rofs[l] = R;
    R += mp.select[l] ? nms_pre : hwl;
  }
  mp.rofs[L] = R;
  cudaStream_t st = (cudaStream_t)stream;
  char what[64];
  for (int l = 0; l < L; ++l) {
    if (!mp.select[l]) continue;
    PTB_REQUIRE(nms_pre <= TOPK_MAX, "nms_pre > 4096 is not supported");
    PTB_REQUIRE(workspace && workspace_bytes >= ptb_fcos_decode_workspace(B, L, hw), "ptb_fcos_decode: workspace too small");
    float* key = reinterpret_cast<float*>(workspace);
    const long long BQ = (long long)B * lv.H[l] * lv.W[l];
    fcos_key_kernel<<<(unsigned)((BQ * 32 + 255) / 256), 256, 0, st>>>(cls_maps[l], ctr_maps[l], BQ, num_classes, key);
    snprintf(what, sizeof(what), "ptb_fcos_decode/key%d", l);
    if ((rc = check_launch(what))) return rc;
    p2p_select_kernel<<<B, SEL_THREADS, 0, st>>>(key, lv.H[l] * lv.W[l], nms_pre, out_idx + mp.rofs[l], R);
    snprintf(what, sizeof(what), "ptb_fcos_decode/select%d", l);
    if ((rc = check_launch(what))) return rc;
  }
  const long long rows = (long long)B * R;
  fcos_gather_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(lv, mp, num_classes, img_hw, scale_factor, out_idx, out_boxes,
                                                                          out_scores, out_ctr);
  return check_launch("ptb_fcos_decode/gather");
}
