// The bbox branch of StandardRoIHead (mmdet/models/roi_heads/standard_roi_head.py, bbox_heads/bbox_head.py, roi_extractors/
// single_level_roi_extractor.py) with mmcv's RoIAlign(aligned=True, pool_mode='avg').  Per batch:
//
//   roi_align_fwd_kernel   CTA per RoI: the RoI's FPN level (floor(log2(sqrt(w h) / finest_scale + 1e-6)) clamped to [0, L-1]) and
//                          mmcv's aligned bilinear sampling from that level's channels-last map; the (C, out, out) block is staged in
//                          shared memory and written coalesced in the (R, C, out, out) layout the first Linear flattens.
//   roi_align_bwd_kernel   CTA per RoI: the block's gradient scattered into its level's gradient map with float4 atomics.
//   roi_targets_kernel     thread per candidate ([GTs; proposals] of each image, assigned by ptb_max_iou_assign and ranked by
//                          ptb_rpn_candidate_ranks): the sampled rows in the reference's order (image-major, positives then negatives):
//                          rois, labels, label weights, bbox2delta targets, bbox weights (bbox_head.py:117-181).
//   RoIBoxLoss             loss_terms.cuh: L1 / SmoothL1 over the positive rows' class columns, fixed-order sum.
//   roi_accuracy_kernel    top-1 accuracy (losses/accuracy.py), torch.argmax of each row (its first NaN, else its first maximum).
//   roi_decode_kernel      warp per RoI row: the padding rows zeroed (test_mixins.py:79-119), softmax, class-specific delta2bbox,
//                          img_shape clip and rescale, written [B][N][C][4] / [B][N][C] for the batched multiclass NMS.
#include "ptb_common.cuh"
#include "loss_terms.cuh"
#include "box_coder.cuh"
#include "sample_plan.cuh"

namespace ptb {
namespace {

struct RoiLevels {                   // by-value kernel argument
  int L, B, C;
  const float* map[PTB_ROI_MAX_LEVELS];       // channels-last [B][H][W][C]
  float* grad[PTB_ROI_MAX_LEVELS];
  int H[PTB_ROI_MAX_LEVELS], W[PTB_ROI_MAX_LEVELS];
  float scale[PTB_ROI_MAX_LEVELS];            // spatial_scale = 1 / stride
};

// lv.X[l] without indexing the by-value argument dynamically (which would copy it to the local stack)
template <class T>
__device__ __forceinline__ T pick(const T (&a)[PTB_ROI_MAX_LEVELS], int l) {
  T v = a[0];
#pragma unroll
  for (int i = 1; i < PTB_ROI_MAX_LEVELS; ++i)
    if (l == i) v = a[i];
  return v;
}

// SingleRoIExtractor.map_roi_levels (single_level_roi_extractor.py:50-54) in fp32 as torch's CPU ops round it; log2 is taken in
// double and rounded once, which is the correctly rounded fp32 log2 that torch returns next to the level boundaries.  -1: NaN scale
// (the reference's mask matches no level and the RoI keeps its zero features).
__device__ __forceinline__ int roi_level(const float* r, int L, float finest_scale) {
  if (L == 1) return 0;
  const float s = __fsqrt_rn(__fmul_rn(__fsub_rn(r[3], r[1]), __fsub_rn(r[4], r[2])));
  const float v = __fadd_rn(__fdiv_rn(s, finest_scale), 1e-6f);
  const float lg = floorf(__double2float_rn(log2((double)v)));
  if (lg != lg) return -1;
  return lg < 0.f ? 0 : (lg > (float)(L - 1) ? L - 1 : (int)lg);
}

struct RoiGeom {
  int lvl, b, gh, gw;
  float sh, sw, bh, bw, count;
};

// mmcv roi_align (aligned=True): coordinates * spatial_scale - 0.5, bins of roi / out, a grid of ceil(roi / out) samples per bin when
// sampling_ratio <= 0, the bin value averaged over max(gh * gw, 1) samples.
__device__ __forceinline__ RoiGeom roi_geom(const float* r, const RoiLevels& lv, int lvl, int out, int sampling_ratio) {
  RoiGeom g;
  g.lvl = lvl;
  g.b = (int)r[0];
  const float sc = pick(lv.scale, lvl);
  g.sw = __fsub_rn(__fmul_rn(r[1], sc), 0.5f);
  g.sh = __fsub_rn(__fmul_rn(r[2], sc), 0.5f);
  const float rw = __fsub_rn(__fsub_rn(__fmul_rn(r[3], sc), 0.5f), g.sw);
  const float rh = __fsub_rn(__fsub_rn(__fmul_rn(r[4], sc), 0.5f), g.sh);
  g.bh = __fdiv_rn(rh, (float)out);
  g.bw = __fdiv_rn(rw, (float)out);
  g.gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(g.bh);
  g.gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(g.bw);
  g.count = (float)max(g.gh * g.gw, 1);
  return g;
}

// one sample's bilinear taps (mmcv bilinear_interpolate): false when the sample lies beyond [-1, H] x [-1, W]
__device__ __forceinline__ bool roi_taps(float y, float x, int H, int W, int& o1, int& o2, int& o3, int& o4, float& w1, float& w2,
                                         float& w3, float& w4) {
  if (y < -1.f || y > (float)H || x < -1.f || x > (float)W) return false;
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else { yh = yl + 1; }
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else { xh = xl + 1; }
  const float ly = __fsub_rn(y, (float)yl), lx = __fsub_rn(x, (float)xl);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  w1 = __fmul_rn(hy, hx); w2 = __fmul_rn(hy, lx); w3 = __fmul_rn(ly, hx); w4 = __fmul_rn(ly, lx);
  o1 = yl * W + xl; o2 = yl * W + xh; o3 = yh * W + xl; o4 = yh * W + xh;
  return true;
}

// sample coordinate: roi_start + p * bin + ((i + .5) * bin) / grid
__device__ __forceinline__ float roi_sample(float start, int p, float bin, int i, int grid) {
  return __fadd_rn(__fadd_rn(start, __fmul_rn((float)p, bin)), __fdiv_rn(__fmul_rn((float)i + 0.5f, bin), (float)grid));
}

__device__ __forceinline__ float lerp4(float a, float b, float c, float d, float w1, float w2, float w3, float w4) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w1, a), __fmul_rn(w2, b)), __fmul_rn(w3, c)), __fmul_rn(w4, d));
}

// work item idx -> (channel vector cv, bin): G consecutive channel vectors (G = the largest power of two <= 8 dividing C4) run fastest,
// then the bins.  A warp covers G channel vectors x 32 / G bins, so its float4 tap loads stay 16 G bytes contiguous, and the staging
// addresses (4 cv + k) * bins + bin of its lanes fall in different banks for an odd bin count (4 * 49 = 4 mod 32), where a
// channel-fastest order would put four lanes on each bank.
__device__ __forceinline__ void work_item(int idx, int C4, int bins, int& cv, int& bin) {
  const int G = min(C4 & -C4, 8);
  const int t = idx / G;
  bin = t % bins;
  cv = (t / bins) * G + (idx & (G - 1));
}

__global__ void __launch_bounds__(256)
roi_align_fwd_kernel(RoiLevels lv, const float* __restrict__ rois, int out, int sampling_ratio, float finest_scale,
                     float* __restrict__ y, int32_t* __restrict__ levels) {
  extern __shared__ float blk[];                 // [C][out * out]
  const int r = blockIdx.x, C = lv.C, C4 = C >> 2, bins = out * out;
  const float* roi = rois + 5LL * r;
  const int lvl = roi_level(roi, lv.L, finest_scale);
  const RoiGeom g = roi_geom(roi, lv, lvl, out, sampling_ratio);
  if (threadIdx.x == 0) levels[r] = lvl;
  const bool live = lvl >= 0 && g.b >= 0 && g.b < lv.B;
  const int H = live ? pick(lv.H, lvl) : 1, W = live ? pick(lv.W, lvl) : 1;
  const float4* fm = live ? reinterpret_cast<const float4*>(pick(lv.map, lvl) + (size_t)g.b * H * W * C) : nullptr;
  for (int idx = threadIdx.x; idx < C4 * bins; idx += blockDim.x) {
    int cv, bin;
    work_item(idx, C4, bins, cv, bin);
    const int ph = bin / out, pw = bin - ph * out;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
      for (int iy = 0; iy < g.gh; ++iy) {
        const float sy = roi_sample(g.sh, ph, g.bh, iy, g.gh);
        for (int ix = 0; ix < g.gw; ++ix) {
          const float sx = roi_sample(g.sw, pw, g.bw, ix, g.gw);
          int o1, o2, o3, o4;
          float w1, w2, w3, w4;
          if (!roi_taps(sy, sx, H, W, o1, o2, o3, o4, w1, w2, w3, w4)) continue;
          const float4 a = fm[(size_t)o1 * C4 + cv], b = fm[(size_t)o2 * C4 + cv], c = fm[(size_t)o3 * C4 + cv],
                       d = fm[(size_t)o4 * C4 + cv];
          acc.x = __fadd_rn(acc.x, lerp4(a.x, b.x, c.x, d.x, w1, w2, w3, w4));
          acc.y = __fadd_rn(acc.y, lerp4(a.y, b.y, c.y, d.y, w1, w2, w3, w4));
          acc.z = __fadd_rn(acc.z, lerp4(a.z, b.z, c.z, d.z, w1, w2, w3, w4));
          acc.w = __fadd_rn(acc.w, lerp4(a.w, b.w, c.w, d.w, w1, w2, w3, w4));
        }
      }
      acc = make_float4(__fdiv_rn(acc.x, g.count), __fdiv_rn(acc.y, g.count), __fdiv_rn(acc.z, g.count), __fdiv_rn(acc.w, g.count));
    }
    blk[(4 * cv + 0) * bins + bin] = acc.x;
    blk[(4 * cv + 1) * bins + bin] = acc.y;
    blk[(4 * cv + 2) * bins + bin] = acc.z;
    blk[(4 * cv + 3) * bins + bin] = acc.w;
  }
  __syncthreads();
  float* dst = y + (size_t)r * C * bins;
  for (int i = threadIdx.x; i < C * bins; i += blockDim.x) __stcs(dst + i, blk[i]);
}

__global__ void __launch_bounds__(256)
roi_align_bwd_kernel(RoiLevels lv, const float* __restrict__ rois, const int32_t* __restrict__ levels, int out, int sampling_ratio,
                     const float* __restrict__ grad_y) {
  extern __shared__ float blk[];
  const int r = blockIdx.x, C = lv.C, C4 = C >> 2, bins = out * out;
  const float* roi = rois + 5LL * r;
  const int lvl = levels[r];
  const RoiGeom g = roi_geom(roi, lv, lvl, out, sampling_ratio);
  if (lvl < 0 || g.b < 0 || g.b >= lv.B) return;
  const float* src = grad_y + (size_t)r * C * bins;
  for (int i = threadIdx.x; i < C * bins; i += blockDim.x) blk[i] = __ldcs(src + i);
  __syncthreads();
  const int H = pick(lv.H, lvl), W = pick(lv.W, lvl);
  float4* gm = reinterpret_cast<float4*>(pick(lv.grad, lvl) + (size_t)g.b * H * W * C);
  for (int idx = threadIdx.x; idx < C4 * bins; idx += blockDim.x) {
    int cv, bin;
    work_item(idx, C4, bins, cv, bin);
    const int ph = bin / out, pw = bin - ph * out;
    const float4 go = make_float4(blk[(4 * cv + 0) * bins + bin], blk[(4 * cv + 1) * bins + bin], blk[(4 * cv + 2) * bins + bin],
                                  blk[(4 * cv + 3) * bins + bin]);
    for (int iy = 0; iy < g.gh; ++iy) {
      const float sy = roi_sample(g.sh, ph, g.bh, iy, g.gh);
      for (int ix = 0; ix < g.gw; ++ix) {
        const float sx = roi_sample(g.sw, pw, g.bw, ix, g.gw);
        int o[4];
        float w[4];
        if (!roi_taps(sy, sx, H, W, o[0], o[1], o[2], o[3], w[0], w[1], w[2], w[3])) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (w[q] == 0.f) continue;
          // mmcv: grad * w / count
          atomicAdd(gm + (size_t)o[q] * C4 + cv,
                    make_float4(__fdiv_rn(__fmul_rn(go.x, w[q]), g.count), __fdiv_rn(__fmul_rn(go.y, w[q]), g.count),
                                __fdiv_rn(__fmul_rn(go.z, w[q]), g.count), __fdiv_rn(__fmul_rn(go.w, w[q]), g.count)));
        }
      }
    }
  }
}

struct TargetCfg {
  float mean[4], stdv[4];
  float pos_weight;
  int num_classes;
};

__global__ void __launch_bounds__(256)
roi_targets_kernel(int B, int N, const float4* __restrict__ cand, const int64_t* __restrict__ gt_inds, const int32_t* __restrict__ rank,
                   const int32_t* __restrict__ plan, const int32_t* __restrict__ row_off, const float4* __restrict__ gt,
                   const int32_t* __restrict__ gt_off, const int64_t* __restrict__ gt_labels, TargetCfg tc, float* __restrict__ rois,
                   int64_t* __restrict__ labels, float* __restrict__ label_w, float4* __restrict__ bbox_t, float4* __restrict__ bbox_w) {
  const long long total = (long long)B * N;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    const int b = (int)(e / N);
    const long long g = gt_inds[e];
    if (g < 0) continue;
    const int kind = g > 0 ? 0 : 1;
    const int slot = sampled_slot(plan, b, kind, rank[e]);
    if (slot < 0) continue;
    const long long row = (long long)row_off[2 * b + kind] + slot;
    const float4 box = cand[e];
    float* rr = rois + 5 * row;
    rr[0] = (float)b; rr[1] = box.x; rr[2] = box.y; rr[3] = box.z; rr[4] = box.w;
    if (kind == 0) {
      const int gi = gt_off[b] + (int)(g - 1);
      labels[row] = gt_labels[gi];
      label_w[row] = tc.pos_weight > 0.f ? tc.pos_weight : 1.f;
      bbox_t[row] = bbox2delta(box, gt[gi], tc.mean, tc.stdv);
      bbox_w[row] = make_float4(1.f, 1.f, 1.f, 1.f);
    } else {
      labels[row] = tc.num_classes;
      label_w[row] = 1.f;
      bbox_t[row] = make_float4(0.f, 0.f, 0.f, 0.f);
      bbox_w[row] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// top-1 accuracy over R rows of num_cols logits: one CTA, a warp per row; out = correct * scale.  The prediction follows torch.argmax,
// which agrees with the reference's pred.topk(1) wherever the winner is unique: NaN ranks above every number, so a row containing NaN
// predicts its first NaN column, and any other row its first maximum.
__global__ void __launch_bounds__(1024)
roi_accuracy_kernel(const float* __restrict__ x, const int64_t* __restrict__ labels, long long R, int num_cols, float scale,
                    float* __restrict__ out) {
  __shared__ int correct;
  if (threadIdx.x == 0) correct = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int mine = 0;
  for (long long m = warp; m < R; m += 32) {
    float best = -INFINITY;
    int arg = num_cols;                        // num_cols: the lane holds no column
    for (int c = lane; c < num_cols; c += 32) {           // ascending columns: a tie keeps the earlier one
      const float v = x[m * num_cols + c];
      if (arg == num_cols || (best == best && (v != v || v > best))) { best = v; arg = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      const bool take = ob != ob ? (best == best || oa < arg) : (best == best && (ob > best || (ob == best && oa < arg)));
      if (take) { best = ob; arg = oa; }
    }
    if (lane == 0 && arg == labels[m]) ++mine;
  }
  if (lane == 0 && mine) atomicAdd(&correct, mine);
  __syncthreads();
  if (threadIdx.x == 0) out[0] = __fmul_rn((float)correct, scale);
}

struct DecodeCfg {
  float mean[4], stdv[4];
  float max_ratio;
  int num_classes, agnostic, rescale;
};

// warp per RoI row of the padded batch (B * N rows)
__global__ void __launch_bounds__(256)
roi_decode_kernel(long long rows, int N, const float* __restrict__ rois, const float* __restrict__ cls_score,
                  const float* __restrict__ bbox_pred, const float* __restrict__ img_hw /*[B][2]*/,
                  const float* __restrict__ scale_factor /*[B][4]*/, DecodeCfg dc, float* __restrict__ boxes, float* __restrict__ scores) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int C = dc.num_classes, C1 = C + 1, ld = dc.agnostic ? 4 : 4 * C;
  for (long long m = warp; m < rows; m += n_warps) {
    const float* roi = rois + 5 * m;
    const int b = (int)(m / N);
    // the padding rows (every coordinate 0) get cls_score = 0 and bbox_pred = 0
    const bool pad = __fadd_rn(__fadd_rn(__fadd_rn(fabsf(roi[1]), fabsf(roi[2])), fabsf(roi[3])), fabsf(roi[4])) == 0.f;
    const float* xs = cls_score + m * C1;
    float mx = -INFINITY;
    for (int c = lane; c < C1; c += 32) mx = fmaxf(mx, pad ? 0.f : xs[c]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane; c < C1; c += 32) sum = __fadd_rn(sum, sleef_expf_u10(__fsub_rn(pad ? 0.f : xs[c], mx)));
    sum = warp_sum(sum);
    const float inv = __fdiv_rn(1.f, sum);
    const float x1 = roi[1], y1 = roi[2], x2 = roi[3], y2 = roi[4];
    const float px = __fmul_rn(__fadd_rn(x1, x2), 0.5f), py = __fmul_rn(__fadd_rn(y1, y2), 0.5f);
    const float pw = __fsub_rn(x2, x1), ph = __fsub_rn(y2, y1);
    const float H = img_hw[2 * b], W = img_hw[2 * b + 1];
    for (int c = lane; c < C; c += 32) {
      scores[m * C + c] = __fmul_rn(sleef_expf_u10(__fsub_rn(pad ? 0.f : xs[c], mx)), inv);
      const float* d = bbox_pred + m * ld + (dc.agnostic ? 0 : 4 * c);
      float dd[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) dd[k] = __fadd_rn(__fmul_rn(pad ? 0.f : d[k], dc.stdv[k]), dc.mean[k]);
      const float mr = dc.max_ratio;
      const float dw = dd[2] < -mr ? -mr : (dd[2] > mr ? mr : dd[2]);
      const float dh = dd[3] < -mr ? -mr : (dd[3] > mr ? mr : dd[3]);
      const float gw = __fmul_rn(pw, sleef_expf_u10(dw)), gh = __fmul_rn(ph, sleef_expf_u10(dh));
      const float gx = __fadd_rn(px, __fmul_rn(pw, dd[0])), gy = __fadd_rn(py, __fmul_rn(ph, dd[1]));
      float o[4] = {__fsub_rn(gx, __fmul_rn(gw, 0.5f)), __fsub_rn(gy, __fmul_rn(gh, 0.5f)), __fadd_rn(gx, __fmul_rn(gw, 0.5f)),
                    __fadd_rn(gy, __fmul_rn(gh, 0.5f))};
      const float lim[4] = {W, H, W, H};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        o[k] = o[k] < 0.f ? 0.f : o[k];
        o[k] = o[k] > lim[k] ? lim[k] : o[k];
        if (dc.rescale) o[k] = __fdiv_rn(o[k], scale_factor[4 * b + k]);
      }
      reinterpret_cast<float4*>(boxes)[m * C + c] = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

int set_levels(RoiLevels& lv, int L, int B, int C, const float* const* maps, float* const* grads, const int32_t* hw,
               const float* strides) {
  if (L < 1 || L > PTB_ROI_MAX_LEVELS || B < 1 || C < 4 || C % 4) return 0;
  lv.L = L; lv.B = B; lv.C = C;
  for (int l = 0; l < L; ++l) {
    lv.map[l] = maps ? maps[l] : nullptr;
    lv.grad[l] = grads ? grads[l] : nullptr;
    lv.H[l] = hw[2 * l]; lv.W[l] = hw[2 * l + 1];
    if (lv.H[l] < 1 || lv.W[l] < 1 || !(strides[l] > 0.f)) return 0;
    if ((maps && ((uintptr_t)maps[l] % 16)) || (grads && ((uintptr_t)grads[l] % 16))) return 0;
    lv.scale[l] = (float)(1.0 / (double)strides[l]);
  }
  return 1;
}

int roi_smem(int C, int out) { return C * out * out * (int)sizeof(float); }

}  // namespace
}  // namespace ptb

using namespace ptb;

extern "C" int ptb_roi_align_fwd(const float* const* maps, const int32_t* featmap_hw, const float* strides, int L, int B, int C,
                                 const float* rois, int R, int out, int sampling_ratio, float finest_scale, float* y, int32_t* levels,
                                 void* stream) {
  PTB_REQUIRE(maps && featmap_hw && strides && R >= 0 && out >= 1 && finest_scale > 0.f, "shape");
  RoiLevels lv;
  PTB_REQUIRE(set_levels(lv, L, B, C, maps, nullptr, featmap_hw, strides),
              "levels: 1..PTB_ROI_MAX_LEVELS non-empty 16-byte aligned maps, C a positive multiple of 4, stride > 0");
  const int smem = roi_smem(C, out);
  PTB_REQUIRE(smem <= 227 * 1024, "C * out * out floats must fit in shared memory");
  if (R == 0) return 0;
  PTB_REQUIRE(rois && y && levels, "NULL input");
  if (cudaFuncSetAttribute(roi_align_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return fail("%s", "ptb_roi_align_fwd: cudaFuncSetAttribute failed");
  roi_align_fwd_kernel<<<R, 256, smem, (cudaStream_t)stream>>>(lv, rois, out, sampling_ratio, finest_scale, y, levels);
  return check_launch("ptb_roi_align_fwd");
}

extern "C" int ptb_roi_align_bwd(float* const* grad_maps, const int32_t* featmap_hw, const float* strides, int L, int B, int C,
                                 const float* rois, const int32_t* levels, int R, int out, int sampling_ratio, const float* grad_y,
                                 void* stream) {
  PTB_REQUIRE(grad_maps && featmap_hw && strides && R >= 0 && out >= 1, "shape");
  RoiLevels lv;
  PTB_REQUIRE(set_levels(lv, L, B, C, nullptr, grad_maps, featmap_hw, strides),
              "levels: 1..PTB_ROI_MAX_LEVELS non-empty 16-byte aligned maps, C a positive multiple of 4, stride > 0");
  const int smem = roi_smem(C, out);
  PTB_REQUIRE(smem <= 227 * 1024, "C * out * out floats must fit in shared memory");
  if (R == 0) return 0;
  PTB_REQUIRE(rois && levels && grad_y, "NULL input");
  if (cudaFuncSetAttribute(roi_align_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return fail("%s", "ptb_roi_align_bwd: cudaFuncSetAttribute failed");
  roi_align_bwd_kernel<<<R, 256, smem, (cudaStream_t)stream>>>(lv, rois, levels, out, sampling_ratio, grad_y);
  return check_launch("ptb_roi_align_bwd");
}

extern "C" int ptb_roi_targets(int B, int N, const float* cand, const int64_t* gt_inds, const int32_t* rank, const int32_t* plan,
                               const int32_t* row_off, const float* gt_bboxes, const int32_t* gt_off, const int64_t* gt_labels,
                               int num_classes, const float* means, const float* stds, float pos_weight, float* rois, int64_t* labels,
                               float* label_weights, float* bbox_targets, float* bbox_weights, void* stream) {
  PTB_REQUIRE(B > 0 && N >= 0 && num_classes >= 1 && means && stds, "shape");
  if (N == 0) return 0;
  PTB_REQUIRE(cand && gt_inds && rank && plan && row_off && gt_off && rois && labels && label_weights && bbox_targets && bbox_weights,
              "NULL input");
  PTB_REQUIRE((uintptr_t)cand % 16 == 0 && (uintptr_t)gt_bboxes % 16 == 0 && (uintptr_t)bbox_targets % 16 == 0 &&
              (uintptr_t)bbox_weights % 16 == 0, "16-byte aligned boxes");
  TargetCfg tc;
  for (int k = 0; k < 4; ++k) { tc.mean[k] = means[k]; tc.stdv[k] = stds[k]; }
  tc.pos_weight = pos_weight;
  tc.num_classes = num_classes;
  const long long total = (long long)B * N;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 8LL * sm_count());
  roi_targets_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(B, N, reinterpret_cast<const float4*>(cand), gt_inds, rank, plan, row_off,
                                                               reinterpret_cast<const float4*>(gt_bboxes), gt_off, gt_labels, tc, rois,
                                                               labels, label_weights, reinterpret_cast<float4*>(bbox_targets),
                                                               reinterpret_cast<float4*>(bbox_weights));
  return check_launch("ptb_roi_targets");
}

extern "C" int ptb_roi_bbox_loss(const float* bbox_pred, int ld, const int64_t* labels, const float* bbox_targets, const float* bbox_weights,
                                 int64_t R, int num_classes, int class_agnostic, int bbox_loss, float beta, float* loss_sum,
                                 const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(R >= 0 && num_classes >= 1 && ld == (class_agnostic ? 4 : 4 * num_classes) &&
              (bbox_loss == PTB_RPN_LOSS_L1 || (bbox_loss == PTB_RPN_LOSS_SMOOTH_L1 && beta > 0.f)),
              "shape / loss kind (SmoothL1 needs beta > 0)");
  if (R == 0) return 0;
  PTB_REQUIRE(bbox_pred && labels && bbox_targets && bbox_weights, "NULL input");
  PTB_REQUIRE(loss_sum ? !grad : grad != nullptr, "either loss_sum or grad");
  const char* name = "ptb_roi_bbox_loss";
  if (bbox_loss == PTB_RPN_LOSS_L1)
    return launch_sum(loss_sum_kernel<RoIBoxLoss<false>>, stream, name,
                      RoIBoxLoss<false>{bbox_pred, labels, bbox_targets, bbox_weights, ld, num_classes, class_agnostic, 0.f}, 4 * R,
                      loss_sum, scale, grad);
  return launch_sum(loss_sum_kernel<RoIBoxLoss<true>>, stream, name,
                    RoIBoxLoss<true>{bbox_pred, labels, bbox_targets, bbox_weights, ld, num_classes, class_agnostic, beta}, 4 * R,
                    loss_sum, scale, grad);
}

extern "C" int ptb_roi_accuracy(const float* cls_score, const int64_t* labels, int64_t R, int num_cols, float scale, float* out,
                                void* stream) {
  PTB_REQUIRE(R >= 1 && num_cols >= 1 && cls_score && labels && out, "shape / NULL input");
  roi_accuracy_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(cls_score, labels, R, num_cols, scale, out);
  return check_launch("ptb_roi_accuracy");
}

extern "C" int ptb_roi_decode(const float* rois, const float* cls_score, const float* bbox_pred, int B, int N, int num_classes,
                              int class_agnostic, const float* means, const float* stds, float max_ratio, const float* img_hw,
                              const float* scale_factor, float* boxes, float* scores, void* stream) {
  PTB_REQUIRE(B >= 1 && N >= 0 && num_classes >= 1 && means && stds && max_ratio >= 0.f, "shape");
  if (N == 0) return 0;
  PTB_REQUIRE(rois && cls_score && bbox_pred && img_hw && boxes && scores, "NULL input");
  PTB_REQUIRE((uintptr_t)boxes % 16 == 0, "16-byte aligned boxes");
  DecodeCfg dc;
  for (int k = 0; k < 4; ++k) { dc.mean[k] = means[k]; dc.stdv[k] = stds[k]; }
  dc.max_ratio = max_ratio;
  dc.num_classes = num_classes;
  dc.agnostic = class_agnostic ? 1 : 0;
  dc.rescale = scale_factor ? 1 : 0;
  const long long rows = (long long)B * N;
  const int blocks = (int)std::min<long long>((rows + 7) / 8, 16LL * sm_count());
  roi_decode_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, N, rois, cls_score, bbox_pred, img_hw, scale_factor, dc, boxes, scores);
  return check_launch("ptb_roi_decode");
}
