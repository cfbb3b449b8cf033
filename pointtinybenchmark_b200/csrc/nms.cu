// multiclass NMS for point pseudo-boxes (multiclass_nms, mmdet/core/post_processing/bbox_nms.py:7-94, and the
// third-party mmcv.ops.nms.batched_nms it calls — semantics restated in oracle/p2p.py).
//
// The class-offset trick of batched_nms makes boxes of different classes disjoint, so greedy NMS decomposes
// exactly into independent per-class problems; the global result (descending score, first max_per_img) is a
// C-way merge of the per-class keep lists.  Three launches per batch:
//   K0  one CTA / image : per-point candidate counts, exclusive scan (candidate ranks = `keep` indices of the
//                         reference), max box coordinate (the batched_nms offset unit), candidate count
//   K1  one CTA / (image, class): compact the class's candidates, bitonic sort by (score desc, flat id asc) in
//                         shared memory, then warp-batched greedy suppression against the <= max_per_img kept boxes
//   K2  one warp / image: C-way merge of the sorted per-class lists -> first max_per_img detections
// IoU is evaluated on the offset fp32 coordinates with the reference's operation order, so `keep` is bit-exact.
#include "ptb_common.cuh"
#include <math_constants.h>

namespace ptb {

constexpr int NMS_MAXP = 4096;      // points per image supported (nms_pre)
// the *_wide entry points: up to 8192 points per image (nms_pre over several FPN levels, e.g. 5 x 1000).  Their class kernel keeps
// its sort keys in dynamic shared memory and their soft-NMS class kernel recomputes each box area instead of storing it.
constexpr int NMS_MAXP_WIDE = 8192;
constexpr int NMS_T0 = 1024;
// mmcv batched_nms's default split_thr: from this many candidates on it runs NMS class by class and sorts the kept entries by
// score, so the classes never interact whatever the offset does - the per-class kernels and the merge are that branch exactly
constexpr int NMS_SPLIT_THR = 10000;
// The 1024-thread kernels are templates over the box layout (cs = 1: class-specific boxes).  Their cs = 1 forms state one CTA per
// SM, which lets ptxas use the full 64 registers per thread instead of spilling; the shared-box forms keep their plain bounds.
#define NMS_T0_BOUNDS(cs) __launch_bounds__(NMS_T0, (cs) ? 1 : 0)

struct NmsImg {       // per-image header in the workspace
  float max_coord;
  int cand_count;
  int slow;           // 1: boxes of adjacent classes may overlap despite the class offset (and cand_count < NMS_SPLIT_THR)
                      //    -> exact global path
  int degenerate;     // gaussian soft-NMS: candidates whose offset box has zero area (1 each) or a negative / NaN area (2 each)
};

// Gaussian soft-NMS weighs by exp(-IoU^2 / sigma) even where IoU = 0/0 = NaN: two zero-area boxes (of any classes, disjoint or
// not) turn a score into NaN in mmcv's loop, and what happens next depends on mmcv's swap arrangement (the NaN never compares
// above anything, never drops below min_score), which neither the per-class decomposition nor the global kernel reproduce.  A
// box of negative area can meet any box with a union of 0.  The gaussian method therefore refuses an image whose candidates
// weigh >= 2 here: its out_count is -1.  Hard NMS, naive and linear only compare the IoU, and NaN compares false everywhere.
__device__ __forceinline__ int degenerate_weight(float area) { return area > 0.f ? 0 : (area == 0.f ? 1 : 2); }


// un-offset box of point / proposal p: either given explicitly (row p of the image's boxes, see box_row) or the pseudo box
// pts[p] -/+ (hw, hh)
struct RawBox {
  float x1, y1, x2, y2;
};
__device__ __forceinline__ RawBox raw_box(const float* __restrict__ pp, const float* __restrict__ bx, int p, float hw, float hh) {
  RawBox r;
  if (bx) {
    r.x1 = bx[4 * p]; r.y1 = bx[4 * p + 1]; r.x2 = bx[4 * p + 2]; r.y2 = bx[4 * p + 3];
  } else {
    const float px = pp[2 * p], py = pp[2 * p + 1];
    r.x1 = __fsub_rn(px, hw); r.y1 = __fsub_rn(py, hh); r.x2 = __fadd_rn(px, hw); r.y2 = __fadd_rn(py, hh);
  }
  return r;
}
// image b's boxes: [P][4] shared by the classes, or [P][C][4] with one box per (point, class) (cs = 1, class-specific boxes);
// candidate (p, c) uses row box_row(p, c) of them
__device__ __forceinline__ const float* img_boxes(const float* boxes, int b, int P, int C, int cs) {
  return boxes ? boxes + (size_t)b * P * (cs ? C : 1) * 4 : nullptr;
}
__device__ __forceinline__ int box_row(int p, int c, int C, int cs) { return cs ? p * C + c : p; }
__device__ __forceinline__ Box offset_box(const RawBox& r, float off) {
  Box b;   // + label*(max_coord+1) on every coordinate (mmcv batched_nms)
  b.x1 = __fadd_rn(r.x1, off); b.y1 = __fadd_rn(r.y1, off); b.x2 = __fadd_rn(r.x2, off); b.y2 = __fadd_rn(r.y2, off);
  b.area = __fmul_rn(__fsub_rn(b.x2, b.x1), __fsub_rn(b.y2, b.y1));
  return b;
}

template <int cs, bool WIDE>
__global__ void NMS_T0_BOUNDS(cs)
nms_prepare_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C, float hw, float hh,
                   float score_thr, NmsImg* __restrict__ hdr, int32_t* __restrict__ base /*[B][P]*/,
                   int32_t* __restrict__ out_cand_count) {
  __shared__ int s_cnt[WIDE ? NMS_MAXP_WIDE : NMS_MAXP];
  __shared__ float s_max[NMS_T0 / 32];
  __shared__ int s_wsum[NMS_T0 / 32];
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* sc = scores + (size_t)b * P * C;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  float mx = -CUDART_INF_F;
  float ax = CUDART_INF_F, ay = CUDART_INF_F;   // min x1 / y1 over candidate boxes in the negative corner zone
  // warp per point: count classes over threshold
  for (int p = wid; p < P; p += NMS_T0 / 32) {
    int cnt = 0;
    for (int c = lane; c < C; c += 32) {
      const bool is = sc[(size_t)p * C + c] > score_thr;
      cnt += is;
      if (cs && is) {  // class-specific boxes: every candidate brings its own box
        const RawBox rb = raw_box(pp, bx, box_row(p, c, C, cs), hw, hh);
        mx = fmaxf(mx, fmaxf(fmaxf(rb.x1, rb.y1), fmaxf(rb.x2, rb.y2)));
        if (rb.x1 < -0.95f && rb.y1 < -0.95f) { ax = fminf(ax, rb.x1); ay = fminf(ay, rb.y1); }
      }
    }
    cnt = (int)warp_sum((float)cnt);
    if (lane == 0) {
      s_cnt[p] = cnt;
      if (!cs && cnt > 0) {   // boxes.max() over the candidate boxes = max over (x2, y2)
        const RawBox rb = raw_box(pp, bx, p, hw, hh);
        mx = fmaxf(mx, fmaxf(fmaxf(rb.x1, rb.y1), fmaxf(rb.x2, rb.y2)));
        if (rb.x1 < -0.95f && rb.y1 < -0.95f) { ax = fminf(ax, rb.x1); ay = fminf(ay, rb.y1); }
      }
    }
  }
  mx = warp_max(mx);
  ax = -warp_max(-ax);
  ay = -warp_max(-ay);
  __shared__ float s_ax[NMS_T0 / 32], s_ay[NMS_T0 / 32];
  __shared__ int s_slow;
  if (lane == 0) { s_max[wid] = mx; s_ax[wid] = ax; s_ay[wid] = ay; }
  if (threadIdx.x == 0) s_slow = 0;
  __syncthreads();
  {
    // The class offset label*(max_coord+1) only separates classes when every coordinate is >= -1.  A box of class c
    // in the negative corner (x1<-1 and y1<-1) can still intersect a class c-1 box whose x2 and y2 are both within
    // that margin of max_coord (near-square images only).  Detect conservatively; such images take the exact path.
    float m = s_max[0], mnx = s_ax[0], mny = s_ay[0];
    for (int w = 1; w < NMS_T0 / 32; ++w) { m = fmaxf(m, s_max[w]); mnx = fminf(mnx, s_ax[w]); mny = fminf(mny, s_ay[w]); }
    if (mnx < CUDART_INF_F) {
      const float m1 = m + 1.f;
      if (!cs) {
        for (int p = threadIdx.x; p < P; p += NMS_T0) {
          if (s_cnt[p] <= 0) continue;
          const RawBox rb = raw_box(pp, bx, p, hw, hh);
          if (rb.x2 > mnx + m1 - 0.05f && rb.y2 > mny + m1 - 0.05f) s_slow = 1;
        }
      } else {         // the same test over every candidate's own box, warp per point
        for (int p = wid; p < P; p += NMS_T0 / 32) {
          if (s_cnt[p] <= 0) continue;
          for (int c = lane; c < C; c += 32) {
            if (!(sc[(size_t)p * C + c] > score_thr)) continue;
            const RawBox rb = raw_box(pp, bx, box_row(p, c, C, cs), hw, hh);
            if (rb.x2 > mnx + m1 - 0.05f && rb.y2 > mny + m1 - 0.05f) s_slow = 1;
          }
        }
      }
    }
  }
  __syncthreads();
  // exclusive scan of s_cnt[0..P) with the whole CTA, chunks of NMS_T0
  int running = 0;
  for (int base0 = 0; base0 < P; base0 += NMS_T0) {
    const int i = base0 + threadIdx.x;
    const int v = i < P ? s_cnt[i] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += n;
    }
    if (lane == 31) s_wsum[wid] = incl;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < wid; ++w) woff += s_wsum[w];
    if (i < P) base[(size_t)b * P + i] = running + woff + incl - v;
    int tot = 0;
    for (int w = 0; w < NMS_T0 / 32; ++w) tot += s_wsum[w];
    running += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float m = s_max[0];
    for (int w = 1; w < NMS_T0 / 32; ++w) m = fmaxf(m, s_max[w]);
    hdr[b].max_coord = m;
    hdr[b].cand_count = running;
    hdr[b].slow = s_slow && running < NMS_SPLIT_THR;   // the exact global path replays the offset branch only
    hdr[b].degenerate = 0;
    out_cand_count[b] = running;
  }
}

__device__ __forceinline__ void bitonic_sort_u64_blk(unsigned long long* a, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long x = a[lo], y = a[hi];
        if ((x > y) == up) { a[lo] = y; a[hi] = x; }
      }
    }
  }
  __syncthreads();
}

constexpr int NMS_T1 = 256;

// per (image, class): list[b][c][0..n) = kept point indices in descending score order (n <= max_keep)
template <int cs, bool WIDE>
__global__ void __launch_bounds__(NMS_T1)
nms_class_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C, float hw, float hh,
                 float score_thr, float iou_thr, int max_keep, const NmsImg* __restrict__ hdr,
                 int32_t* __restrict__ cls_cnt /*[B][C]*/, int32_t* __restrict__ cls_list /*[B][C][max_keep]*/) {
  __shared__ unsigned long long keys_static[WIDE ? 1 : NMS_MAXP];
  __shared__ int s_n;
  __shared__ int s_wbase[NMS_T1 / 32];
  extern __shared__ unsigned long long dyn_sm[];     // WIDE: keys [NMS_MAXP_WIDE], then the kept list; else the kept list
  unsigned long long* keys = WIDE ? dyn_sm : keys_static;
  float* kept = reinterpret_cast<float*>(WIDE ? dyn_sm + NMS_MAXP_WIDE : dyn_sm);   // [max_keep][5]
  const int b = blockIdx.y, c = blockIdx.x;
  if (hdr[b].slow) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* sc = scores + (size_t)b * P * C + c;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  // ---- compact candidates of this class (order irrelevant: sorted next)
  for (int base0 = 0; base0 < P; base0 += NMS_T1) {
    const int p = base0 + threadIdx.x;
    const float s = p < P ? sc[(size_t)p * C] : 0.f;
    const bool is = p < P && s > score_thr;
    const unsigned int bal = __ballot_sync(0xffffffffu, is);
    if (lane == 0) s_wbase[wid] = atomicAdd(&s_n, __popc(bal));
    __syncwarp();
    if (is) {
      const int slot = s_wbase[wid] + __popc(bal & ((1u << lane) - 1u));
      keys[slot] = ((unsigned long long)(~__float_as_uint(s)) << 32) | (unsigned int)p;   // score desc, point asc
    }
    __syncwarp();
  }
  __syncthreads();
  const int n = s_n;
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int i = n + threadIdx.x; i < n2; i += NMS_T1) keys[i] = 0xFFFFFFFFFFFFFFFFull;
  bitonic_sort_u64_blk(keys, n2);
  // ---- greedy suppression, 32 candidates per step, by warp 0
  int nk = 0;
  if (wid == 0 && n > 0) {
    const float off = __fmul_rn((float)c, __fadd_rn(hdr[b].max_coord, 1.f));
    for (int base0 = 0; base0 < n && nk < max_keep; base0 += 32) {
      const int i = base0 + lane;
      const bool have = i < n;
      const int p = have ? (int)(keys[i] & 0xFFFFFFFFull) : 0;
      const Box me = offset_box(raw_box(pp, bx, box_row(p, c, C, cs), hw, hh), off);
      bool alive = have;
      for (int t = 0; t < nk && alive; ++t) {
        Box kb;
        kb.x1 = kept[5 * t]; kb.y1 = kept[5 * t + 1]; kb.x2 = kept[5 * t + 2]; kb.y2 = kept[5 * t + 3]; kb.area = kept[5 * t + 4];
        if (iou_gt(kb, me, iou_thr)) alive = false;
      }
      // intra-batch: suppression by earlier lanes that survive
      unsigned int alive_mask = __ballot_sync(0xffffffffu, alive);
      for (int jl = 0; jl < 32; ++jl) {
        if (!((alive_mask >> jl) & 1u)) continue;       // uniform: alive_mask is warp-uniform
        Box ob;
        ob.x1 = __shfl_sync(0xffffffffu, me.x1, jl); ob.y1 = __shfl_sync(0xffffffffu, me.y1, jl);
        ob.x2 = __shfl_sync(0xffffffffu, me.x2, jl); ob.y2 = __shfl_sync(0xffffffffu, me.y2, jl);
        ob.area = __shfl_sync(0xffffffffu, me.area, jl);
        const int pj = __shfl_sync(0xffffffffu, p, jl);
        // lane jl is kept
        if (nk < max_keep) {
          if (lane == 0) {
            kept[5 * nk] = ob.x1; kept[5 * nk + 1] = ob.y1; kept[5 * nk + 2] = ob.x2; kept[5 * nk + 3] = ob.y2; kept[5 * nk + 4] = ob.area;
            cls_list[((size_t)b * C + c) * max_keep + nk] = pj;
          }
          ++nk;
        }
        if (lane > jl && alive && iou_gt(ob, me, iou_thr)) alive = false;
        alive_mask = __ballot_sync(0xffffffffu, alive);
        if (nk >= max_keep) break;
      }
      __syncwarp();
    }
  }
  if (threadIdx.x == 0) cls_cnt[(size_t)b * C + c] = nk;
}

// one warp per image: merge
template <int cs>
__global__ void __launch_bounds__(32)
nms_merge_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C, float hw, float hh,
                 float score_thr, int max_keep, const NmsImg* __restrict__ hdr, const int32_t* __restrict__ base,
                 const int32_t* __restrict__ cls_cnt, const int32_t* __restrict__ cls_list, int32_t* __restrict__ out_count,
                 float* __restrict__ out_det, int32_t* __restrict__ out_label, int32_t* __restrict__ out_keep,
                 const float* __restrict__ cls_score /*soft-NMS: decayed score per list entry, else NULL*/) {
  extern __shared__ int head[];   // [C]
  const int b = blockIdx.x, lane = threadIdx.x;
  if (hdr[b].slow) return;
  if (hdr[b].degenerate >= 2) {   // gaussian soft-NMS only (the class kernel counts nothing otherwise)
    if (lane == 0) out_count[b] = -1;
    return;
  }
  for (int c = lane; c < C; c += 32) head[c] = 0;
  __syncwarp();
  const float* sc = scores + (size_t)b * P * C;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  int r = 0;
  for (; r < max_keep; ++r) {
    unsigned long long best = 0xFFFFFFFFFFFFFFFFull;   // (~score bits, flat id) : smaller is better
    for (int c = lane; c < C; c += 32) {
      const int h = head[c];
      if (h < cls_cnt[(size_t)b * C + c]) {
        const int p = cls_list[((size_t)b * C + c) * max_keep + h];
        const float sv = cls_score ? cls_score[((size_t)b * C + c) * max_keep + h] : sc[(size_t)p * C + c];
        const unsigned long long k = ((unsigned long long)(~__float_as_uint(sv)) << 32) | (unsigned int)(p * C + c);
        if (k < best) best = k;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      if (other < best) best = other;
    }
    if (best == 0xFFFFFFFFFFFFFFFFull) break;
    const int flat = (int)(best & 0xFFFFFFFFull);
    const int p = flat / C, c = flat - p * C;
    if (lane == 0) {
      const float sv = cls_score ? cls_score[((size_t)b * C + c) * max_keep + head[c]] : sc[(size_t)p * C + c];
      head[c] += 1;
      float* d = out_det + ((size_t)b * max_keep + r) * 5;
      const RawBox rb = raw_box(pp, bx, box_row(p, c, C, cs), hw, hh);
      d[0] = rb.x1; d[1] = rb.y1; d[2] = rb.x2; d[3] = rb.y2;
      d[4] = sv;
      out_label[(size_t)b * max_keep + r] = c;
      // rank of (p,c) in the flat candidate list = base[p] + #candidate classes below c at point p
      int rank = base[(size_t)b * P + p];
      for (int cc = 0; cc < c; ++cc) rank += sc[(size_t)p * C + cc] > score_thr;
      out_keep[(size_t)b * max_keep + r] = rank;
    }
    __syncwarp();
  }
  if (lane == 0) out_count[b] = r;
}

// ---------------------------------------------------------------------------------------------------------------
// soft-NMS (mmcv.ops.nms.soft_nms through batched_nms; third-party, restated in oracle/p2p.py::soft_nms).  Boxes of different
// classes are disjoint after the class offset and every soft-NMS weight is exactly 1 at IoU 0, so the sequential algorithm
// decomposes per class exactly like hard NMS; scores only decay, so a class's selections come out in non-increasing score
// order and the image's first max_per_img detections are a C-way merge of the first <= max_per_img selections of every class.
// (The gaussian weight is exactly 1 at IoU 0 but NaN at 0/0: images with degenerate boxes are refused, see degenerate_weight.)
// One CTA per (image, class): candidates (ascending point index = the reference's array order) live in shared memory; per
// selection one block-wide arg-max (highest score, lowest position) and one parallel decay pass.
// method: 0 naive (weight 0 when IoU >= thr), 1 linear (1 - IoU when IoU >= thr), 2 gaussian (exp(-IoU^2 / sigma)).
// Difference from mmcv's CPU loop: exact score ties are broken by candidate position (mmcv: by the position after its
// swap-with-last deletions).  Images flagged `slow` (the class offset does not separate the classes) take
// soft_nms_global_kernel: the same loop over ALL candidates of the image with the state in global memory.
// ---------------------------------------------------------------------------------------------------------------
constexpr int SNMS_T = 256;

__device__ __forceinline__ float soft_weight(float ovr, float iou_thr, float sigma, int method) {
  if (method == 0) return ovr >= iou_thr ? 0.f : 1.f;
  if (method == 1) return ovr >= iou_thr ? __fsub_rn(1.f, ovr) : 1.f;
  return expf(__fdiv_rn(-__fmul_rn(ovr, ovr), sigma));
}


template <int cs, bool WIDE>
__global__ void __launch_bounds__(SNMS_T)
soft_nms_class_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C,
                      float hw, float hh, float score_thr, float iou_thr, float sigma, float min_score, int method, int max_keep,
                      NmsImg* __restrict__ hdr, int32_t* __restrict__ cls_cnt, int32_t* __restrict__ cls_list,
                      float* __restrict__ cls_score) {
  // x1 | y1 | x2 | y2 | area | score : [P] each, then idx [P] (int), alive [P] (u8).  WIDE: no area array (recomputed from the
  // offset box by offset_box's formula, the same bits), so 8192 candidates fit
  extern __shared__ float sm[];
  constexpr int NA = WIDE ? 0 : 1;
  float* bx1 = sm; float* by1 = sm + P; float* bx2 = sm + 2 * P; float* by2 = sm + 3 * P; float* bar = sm + 4 * P;
  float* bsc = sm + (4 + NA) * P;
  int* bidx = reinterpret_cast<int*>(sm + (5 + NA) * P);
  unsigned char* alive = reinterpret_cast<unsigned char*>(sm + (6 + NA) * P);
  auto area_of = [&](int j) { return WIDE ? __fmul_rn(__fsub_rn(bx2[j], bx1[j]), __fsub_rn(by2[j], by1[j])) : bar[j]; };
  __shared__ int s_wcnt[SNMS_T / 32];
  __shared__ unsigned long long s_red[SNMS_T / 32];
  __shared__ unsigned long long s_best;
  const int b = blockIdx.y, c = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (hdr[b].slow) return;
  const float* sc = scores + (size_t)b * P * C + c;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  const float off = __fmul_rn((float)c, __fadd_rn(hdr[b].max_coord, 1.f));
  // ---- ordered compaction of this class's candidates
  int n = 0;
  for (int base0 = 0; base0 < P; base0 += SNMS_T) {
    const int p = base0 + threadIdx.x;
    const float s = p < P ? sc[(size_t)p * C] : 0.f;
    const bool is = p < P && s > score_thr;
    const unsigned int bal = __ballot_sync(0xffffffffu, is);
    if (lane == 0) s_wcnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < SNMS_T / 32; ++w) { if (w < wid) before += s_wcnt[w]; total += s_wcnt[w]; }
    if (is) {
      const int slot = n + before + __popc(bal & ((1u << lane) - 1u));
      const Box me = offset_box(raw_box(pp, bx, box_row(p, c, C, cs), hw, hh), off);
      bx1[slot] = me.x1; by1[slot] = me.y1; bx2[slot] = me.x2; by2[slot] = me.y2;
      if (!WIDE) bar[slot] = me.area;
      bsc[slot] = s; bidx[slot] = p; alive[slot] = 1;
    }
    n += total;
    __syncthreads();
  }
  if (method == 2) {          // degenerate boxes of the whole image, summed over its classes; the merge refuses the image
    int d = 0;
    for (int j = threadIdx.x; j < n; j += SNMS_T) d += degenerate_weight(area_of(j));
    if (d) atomicAdd(&hdr[b].degenerate, d);
  }
  int nk = 0;
  while (nk < max_keep) {
    // ---- arg-max over the alive candidates: (score desc, position asc)
    unsigned long long mine = 0xFFFFFFFFFFFFFFFFull;
    for (int j = threadIdx.x; j < n; j += SNMS_T)
      if (alive[j]) {
        const unsigned long long k = ((unsigned long long)(~__float_as_uint(bsc[j])) << 32) | (unsigned int)j;
        if (k < mine) mine = k;
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, o);
      if (other < mine) mine = other;
    }
    if (lane == 0) s_red[wid] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long m = s_red[0];
      for (int w = 1; w < SNMS_T / 32; ++w) if (s_red[w] < m) m = s_red[w];
      s_best = m;
      if (m != 0xFFFFFFFFFFFFFFFFull) {
        const int w0 = (int)(m & 0xFFFFFFFFull);
        alive[w0] = 0;
        cls_list[((size_t)b * C + c) * max_keep + nk] = bidx[w0];
        cls_score[((size_t)b * C + c) * max_keep + nk] = bsc[w0];
      }
    }
    __syncthreads();
    const unsigned long long best = s_best;
    if (best == 0xFFFFFFFFFFFFFFFFull) break;
    ++nk;
    const int w0 = (int)(best & 0xFFFFFFFFull);
    const float ix1 = bx1[w0], iy1 = by1[w0], ix2 = bx2[w0], iy2 = by2[w0], iarea = area_of(w0);
    // ---- decay every remaining candidate (mmcv's operation order: offset 0)
    for (int j = threadIdx.x; j < n; j += SNMS_T)
      if (alive[j]) {
        const float w = fmaxf(0.f, __fsub_rn(fminf(ix2, bx2[j]), fmaxf(ix1, bx1[j])));
        const float h = fmaxf(0.f, __fsub_rn(fminf(iy2, by2[j]), fmaxf(iy1, by1[j])));
        const float inter = __fmul_rn(w, h);
        const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(iarea, area_of(j)), inter));
        const float ns = __fmul_rn(bsc[j], soft_weight(ovr, iou_thr, sigma, method));
        bsc[j] = ns;
        if (ns < min_score) alive[j] = 0;
      }
    __syncthreads();
  }
  if (threadIdx.x == 0) cls_cnt[(size_t)b * C + c] = nk;
}

// soft-NMS over ALL candidates of a flagged image (class offsets applied, classes may interact): state[e] = current score of
// candidate (p, c) = e / C, e % C, or -1 when dead / selected / not a candidate.  One CTA per flagged image.
template <int cs>
__global__ void NMS_T0_BOUNDS(cs)
soft_nms_global_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C,
                       float hw, float hh, float score_thr, float iou_thr, float sigma, float min_score, int method, int max_keep,
                       const NmsImg* __restrict__ hdr, const int32_t* __restrict__ base, float* __restrict__ state /*[B][P*C]*/,
                       int32_t* __restrict__ out_count, float* __restrict__ out_det, int32_t* __restrict__ out_label,
                       int32_t* __restrict__ out_keep) {
  __shared__ unsigned long long s_red[NMS_T0 / 32];
  __shared__ unsigned long long s_best;
  const int b = blockIdx.x;
  if (!hdr[b].slow) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* sc = scores + (size_t)b * P * C;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  float* st = state + (size_t)b * P * C;
  const float m1 = __fadd_rn(hdr[b].max_coord, 1.f);
  const int N = P * C;
  __shared__ int s_deg;
  if (threadIdx.x == 0) s_deg = 0;
  __syncthreads();
  int deg = 0;
  for (int e = threadIdx.x; e < N; e += NMS_T0) {
    st[e] = sc[e] > score_thr ? sc[e] : -1.f;
    if (method == 2 && sc[e] > score_thr) {
      const int p = e / C, c = e - p * C;
      deg += degenerate_weight(offset_box(raw_box(pp, bx, box_row(p, c, C, cs), hw, hh), __fmul_rn((float)c, m1)).area);
    }
  }
  if (deg) atomicAdd(&s_deg, deg);
  __syncthreads();
  if (s_deg >= 2) {           // see degenerate_weight
    if (threadIdx.x == 0) out_count[b] = -1;
    return;
  }
  int nk = 0;
  while (nk < max_keep) {
    unsigned long long mine = 0xFFFFFFFFFFFFFFFFull;
    for (int e = threadIdx.x; e < N; e += NMS_T0) {
      const float v = st[e];
      if (v >= 0.f) {
        const unsigned long long k = ((unsigned long long)(~__float_as_uint(v)) << 32) | (unsigned int)e;
        if (k < mine) mine = k;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, o);
      if (other < mine) mine = other;
    }
    if (lane == 0) s_red[wid] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long m = s_red[0];
      for (int w = 1; w < NMS_T0 / 32; ++w) if (s_red[w] < m) m = s_red[w];
      s_best = m;
    }
    __syncthreads();
    const unsigned long long best = s_best;
    if (best == 0xFFFFFFFFFFFFFFFFull) break;
    const int e0 = (int)(best & 0xFFFFFFFFull);
    const int p0 = e0 / C, c0 = e0 - p0 * C;
    const RawBox rb0 = raw_box(pp, bx, box_row(p0, c0, C, cs), hw, hh);
    const Box b0 = offset_box(rb0, __fmul_rn((float)c0, m1));
    if (threadIdx.x == 0) {
      float* d = out_det + ((size_t)b * max_keep + nk) * 5;
      d[0] = rb0.x1; d[1] = rb0.y1; d[2] = rb0.x2; d[3] = rb0.y2;
      d[4] = st[e0];
      out_label[(size_t)b * max_keep + nk] = c0;
      int rank = base[(size_t)b * P + p0];
      for (int cc = 0; cc < c0; ++cc) rank += sc[(size_t)p0 * C + cc] > score_thr;
      out_keep[(size_t)b * max_keep + nk] = rank;
    }
    ++nk;
    __syncthreads();                       // everyone has read st[e0] / s_best before they change
    for (int e = threadIdx.x; e < N; e += NMS_T0) {
      const float v = st[e];
      if (e == e0) { st[e] = -1.f; continue; }
      if (v < 0.f) continue;
      const int p = e / C, c = e - p * C;
      const Box me = offset_box(raw_box(pp, bx, box_row(p, c, C, cs), hw, hh), __fmul_rn((float)c, m1));
      const float w = fmaxf(0.f, __fsub_rn(fminf(b0.x2, me.x2), fmaxf(b0.x1, me.x1)));
      const float h = fmaxf(0.f, __fsub_rn(fminf(b0.y2, me.y2), fmaxf(b0.y1, me.y1)));
      const float inter = __fmul_rn(w, h);
      const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(b0.area, me.area), inter));
      const float ns = __fmul_rn(v, soft_weight(ovr, iou_thr, sigma, method));
      st[e] = ns < min_score ? -1.f : ns;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out_count[b] = nk;
}

// Exact global path (rare: near-square images with candidates in both extreme corners and fewer than NMS_SPLIT_THR
// candidates; from NMS_SPLIT_THR on, batched_nms itself goes class by class).  One CTA per flagged image
// walks the candidates in descending (score, flat id) order - one block-wide arg-min per examined candidate - and
// tests each against the <= max_keep kept boxes of ALL classes on the offset coordinates, i.e. the reference's
// batched_nms literally, stopping at max_keep.
template <int cs>
__global__ void NMS_T0_BOUNDS(cs)
nms_global_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, const float* __restrict__ scores, int P, int C, float hw, float hh,
                  float score_thr, float iou_thr, int max_keep, const NmsImg* __restrict__ hdr,
                  const int32_t* __restrict__ base, int32_t* __restrict__ out_count, float* __restrict__ out_det,
                  int32_t* __restrict__ out_label, int32_t* __restrict__ out_keep) {
  extern __shared__ float kept[];     // [max_keep][5]
  __shared__ unsigned long long s_red[NMS_T0 / 32];
  __shared__ unsigned long long s_best;
  const int b = blockIdx.x;
  if (!hdr[b].slow) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* sc = scores + (size_t)b * P * C;
  const float* pp = pts ? pts + (size_t)b * P * 2 : nullptr;
  const float* bx = img_boxes(boxes, b, P, C, cs);
  const float m1 = __fadd_rn(hdr[b].max_coord, 1.f);
  const int N = P * C;
  unsigned long long prev = 0ull;
  bool first = true;
  int nk = 0;
  while (nk < max_keep) {
    unsigned long long mine = 0xFFFFFFFFFFFFFFFFull;
    for (int e = threadIdx.x; e < N; e += NMS_T0) {
      const float s = sc[e];
      if (s > score_thr) {
        const unsigned long long k = ((unsigned long long)(~__float_as_uint(s)) << 32) | (unsigned int)e;
        if ((first || k > prev) && k < mine) mine = k;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, o);
      if (other < mine) mine = other;
    }
    if (lane == 0) s_red[wid] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long m = s_red[0];
      for (int w = 1; w < NMS_T0 / 32; ++w) if (s_red[w] < m) m = s_red[w];
      s_best = m;
    }
    __syncthreads();
    const unsigned long long best = s_best;
    if (best == 0xFFFFFFFFFFFFFFFFull) break;
    prev = best;
    first = false;
    const int flat = (int)(best & 0xFFFFFFFFull);
    const int p = flat / C, c = flat - p * C;
    const RawBox rb = raw_box(pp, bx, box_row(p, c, C, cs), hw, hh);
    const Box me = offset_box(rb, __fmul_rn((float)c, m1));
    int sup = 0;
    for (int t = threadIdx.x; t < nk; t += NMS_T0) {
      Box kb;
      kb.x1 = kept[5 * t]; kb.y1 = kept[5 * t + 1]; kb.x2 = kept[5 * t + 2]; kb.y2 = kept[5 * t + 3]; kb.area = kept[5 * t + 4];
      sup |= iou_gt(kb, me, iou_thr);
    }
    sup = __syncthreads_or(sup);
    if (!sup) {
      if (threadIdx.x == 0) {
        kept[5 * nk] = me.x1; kept[5 * nk + 1] = me.y1; kept[5 * nk + 2] = me.x2; kept[5 * nk + 3] = me.y2; kept[5 * nk + 4] = me.area;
        float* d = out_det + ((size_t)b * max_keep + nk) * 5;
        d[0] = rb.x1; d[1] = rb.y1; d[2] = rb.x2; d[3] = rb.y2;
        d[4] = sc[flat];
        out_label[(size_t)b * max_keep + nk] = c;
        int rank = base[(size_t)b * P + p];
        for (int cc = 0; cc < c; ++cc) rank += sc[(size_t)p * C + cc] > score_thr;
        out_keep[(size_t)b * max_keep + nk] = rank;
      }
      ++nk;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out_count[b] = nk;
}

}  // namespace ptb

using namespace ptb;

static inline size_t nms_hdr_bytes(int B) { return (((size_t)B * sizeof(NmsImg) + 255) / 256) * 256; }

extern "C" uint64_t ptb_multiclass_nms_workspace(int B, int P, int num_classes) {
  // header | base[B][P] | cls_cnt[B][C] | cls_list[B][C][1024]
  return nms_hdr_bytes(B) + ((uint64_t)B * P + (uint64_t)B * num_classes + (uint64_t)B * num_classes * 1024) * 4;
}

// class-specific boxes index row p * C + c of a [P][C][4] image: keep 4 * P * C within int
#define NMS_REQUIRE_CS_ROWS(cs, P, C) \
  PTB_REQUIRE(!(cs) || (uint64_t)(P) * (uint64_t)(C) * 4 <= 0x7fffffffull, "class-specific boxes: 4 * P * num_classes must fit in int")

template <int cs, bool WIDE = false>
static int nms_run(const float* pts, const float* boxes, const float* scores, int B, int P, int num_classes, float pseudo_w,
                   float pseudo_h, float score_thr, float iou_thr, int max_per_img, int32_t* out_count, float* out_det,
                   int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                   void* stream) {
  PTB_REQUIRE(B > 0 && P > 0 && num_classes > 0, "shape");
  if (WIDE) PTB_REQUIRE(P <= NMS_MAXP_WIDE, "more than 8192 points per image not supported");
  else PTB_REQUIRE(P <= NMS_MAXP, "more than 4096 points per image not supported");
  PTB_REQUIRE(max_per_img > 0 && max_per_img <= 1024, "max_per_img must be in [1,1024]");
  PTB_REQUIRE(iou_thr >= 0.f, "iou_thr must be >= 0 (per-class decomposition)");
  PTB_REQUIRE((pts || boxes) && scores && out_count && out_det && out_label && out_keep && out_cand_count, "NULL input");
  PTB_REQUIRE(workspace && workspace_bytes >= ptb_multiclass_nms_workspace(B, P, num_classes), "workspace too small");
  NMS_REQUIRE_CS_ROWS(cs, P, num_classes);
  NmsImg* hdr = reinterpret_cast<NmsImg*>(workspace);
  int32_t* base = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(workspace) + nms_hdr_bytes(B));
  int32_t* cls_cnt = base + (size_t)B * P;
  int32_t* cls_list = cls_cnt + (size_t)B * num_classes;
  const float hw = pseudo_w * 0.5f, hh = pseudo_h * 0.5f;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  nms_prepare_kernel<cs, WIDE><<<B, NMS_T0, 0, st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, hdr, base, out_cand_count);
  if ((rc = check_launch("ptb_multiclass_nms/prepare"))) return rc;
  // keys (32 KB static, or 64 KB dynamic when WIDE) + kept list (dynamic) can exceed the 48 KB default; the attribute is per device
  // -> set on every call
  const int keys_dyn = WIDE ? NMS_MAXP_WIDE * (int)sizeof(unsigned long long) : 0;
  if (cudaFuncSetAttribute(nms_class_kernel<cs, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           keys_dyn + 1024 * 5 * (int)sizeof(float)) != cudaSuccess ||
      cudaFuncSetAttribute(nms_global_kernel<cs>, cudaFuncAttributeMaxDynamicSharedMemorySize, 1024 * 5 * (int)sizeof(float)) != cudaSuccess)
    return fail("%s", "ptb_multiclass_nms: shared memory opt-in failed");
  dim3 g1(num_classes, B);
  nms_class_kernel<cs, WIDE><<<g1, NMS_T1, keys_dyn + (size_t)max_per_img * 5 * sizeof(float), st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr,
                                                                              iou_thr, max_per_img, hdr, cls_cnt, cls_list);
  if ((rc = check_launch("ptb_multiclass_nms/class"))) return rc;
  nms_merge_kernel<cs><<<B, 32, (size_t)num_classes * sizeof(int), st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, max_per_img,
                                                                   hdr, base, cls_cnt, cls_list, out_count, out_det, out_label,
                                                                   out_keep, nullptr);
  if ((rc = check_launch("ptb_multiclass_nms/merge"))) return rc;
  nms_global_kernel<cs><<<B, NMS_T0, (size_t)max_per_img * 5 * sizeof(float), st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr,
                                                                                iou_thr, max_per_img, hdr, base, out_count,
                                                                                out_det, out_label, out_keep);
  return check_launch("ptb_multiclass_nms/global");
}

extern "C" int ptb_multiclass_nms(const float* pts, const float* scores, int B, int P, int num_classes, float pseudo_w,
                                  float pseudo_h, float score_thr, float iou_thr, int max_per_img, int32_t* out_count,
                                  float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                                  void* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(pts, "NULL pts");
  return nms_run<0>(pts, nullptr, scores, B, P, num_classes, pseudo_w, pseudo_h, score_thr, iou_thr, max_per_img, out_count, out_det,
                 out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

extern "C" int ptb_multiclass_nms_boxes(const float* boxes, const float* scores, int B, int P, int num_classes, float score_thr,
                                        float iou_thr, int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label,
                                        int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                                        void* stream) {
  PTB_REQUIRE(boxes, "NULL boxes");
  return nms_run<0>(nullptr, boxes, scores, B, P, num_classes, 0.f, 0.f, score_thr, iou_thr, max_per_img, out_count, out_det,
                 out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

extern "C" int ptb_multiclass_nms_cls_boxes(const float* boxes, const float* scores, int B, int P, int num_classes, float score_thr,
                                            float iou_thr, int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label,
                                            int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                                            void* stream) {
  PTB_REQUIRE(boxes, "NULL boxes");
  return nms_run<1>(nullptr, boxes, scores, B, P, num_classes, 0.f, 0.f, score_thr, iou_thr, max_per_img, out_count, out_det,
                 out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

extern "C" uint64_t ptb_multiclass_soft_nms_workspace(int B, int P, int num_classes) {
  // header | base[B][P] | cls_cnt[B][C] | cls_list[B][C][1024] | cls_score[B][C][1024] | state[B][P*C] (global fallback)
  return nms_hdr_bytes(B) +
         ((uint64_t)B * P + (uint64_t)B * num_classes + 2 * (uint64_t)B * num_classes * 1024 + (uint64_t)B * P * num_classes) * 4;
}

template <int cs, bool WIDE = false>
static int soft_nms_run(const float* pts, const float* boxes, const float* scores, int B, int P, int num_classes,
                        float pseudo_w, float pseudo_h, float score_thr, float iou_thr, float sigma, float min_score, int method,
                        int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep,
                        int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(B > 0 && P > 0 && num_classes > 0, "shape");
  if (WIDE) PTB_REQUIRE(P <= NMS_MAXP_WIDE, "more than 8192 points per image not supported");
  else PTB_REQUIRE(P <= NMS_MAXP, "more than 4096 points per image not supported");
  PTB_REQUIRE(max_per_img > 0 && max_per_img <= 1024, "max_per_img must be in [1,1024]");
  PTB_REQUIRE(method >= 0 && method <= 2, "method: 0 naive, 1 linear, 2 gaussian");
  PTB_REQUIRE(method != 2 || sigma > 0.f, "sigma must be > 0 for the gaussian method");
  // naive weight at IoU 0 is 0 when iou_thr <= 0: a selection would zero every other class too (no per-class decomposition)
  PTB_REQUIRE(method != 0 || iou_thr > 0.f, "the naive method needs iou_thr > 0 (per-class decomposition)");
  PTB_REQUIRE((pts != nullptr) != (boxes != nullptr), "give either pts (pseudo boxes) or boxes");
  PTB_REQUIRE(scores && out_count && out_det && out_label && out_keep && out_cand_count, "NULL input");
  PTB_REQUIRE(workspace && workspace_bytes >= ptb_multiclass_soft_nms_workspace(B, P, num_classes), "workspace too small");
  NMS_REQUIRE_CS_ROWS(cs, P, num_classes);
  NmsImg* hdr = reinterpret_cast<NmsImg*>(workspace);
  int32_t* base = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(workspace) + nms_hdr_bytes(B));
  int32_t* cls_cnt = base + (size_t)B * P;
  int32_t* cls_list = cls_cnt + (size_t)B * num_classes;
  float* cls_score = reinterpret_cast<float*>(cls_list + (size_t)B * num_classes * 1024);
  float* state = cls_score + (size_t)B * num_classes * 1024;
  const float hw = pseudo_w * 0.5f, hh = pseudo_h * 0.5f;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  nms_prepare_kernel<cs, WIDE><<<B, NMS_T0, 0, st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, hdr, base, out_cand_count);
  if ((rc = check_launch("ptb_multiclass_soft_nms/prepare"))) return rc;
  const size_t smem = (size_t)P * ((WIDE ? 6 : 7) * sizeof(float) + 1) + 16;
  // the kernel's own 104 B of static shared memory count against the 48 KB default too (P = 1691..1694 have smem <= 48 KB but fail
  // to launch without the opt-in): set the per-device attribute on every call (a process may drive several devices)
  if (cudaFuncSetAttribute(soft_nms_class_kernel<cs, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("%s", "ptb_multiclass_soft_nms: shared memory opt-in failed");
  dim3 g1(num_classes, B);
  soft_nms_class_kernel<cs, WIDE><<<g1, SNMS_T, smem, st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, iou_thr, sigma, min_score, method,
                                                max_per_img, hdr, cls_cnt, cls_list, cls_score);
  if ((rc = check_launch("ptb_multiclass_soft_nms/class"))) return rc;
  nms_merge_kernel<cs><<<B, 32, (size_t)num_classes * sizeof(int), st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, max_per_img,
                                                                   hdr, base, cls_cnt, cls_list, out_count, out_det, out_label,
                                                                   out_keep, cls_score);
  if ((rc = check_launch("ptb_multiclass_soft_nms/merge"))) return rc;
  soft_nms_global_kernel<cs><<<B, NMS_T0, 0, st>>>(pts, boxes, scores, P, num_classes, hw, hh, score_thr, iou_thr, sigma, min_score, method,
                                             max_per_img, hdr, base, state, out_count, out_det, out_label, out_keep);
  return check_launch("ptb_multiclass_soft_nms/global");
}

extern "C" int ptb_multiclass_soft_nms(const float* pts, const float* boxes, const float* scores, int B, int P, int num_classes,
                                       float pseudo_w, float pseudo_h, float score_thr, float iou_thr, float sigma, float min_score,
                                       int method, int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label,
                                       int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                                       void* stream) {
  return soft_nms_run<0>(pts, boxes, scores, B, P, num_classes, pseudo_w, pseudo_h, score_thr, iou_thr, sigma, min_score, method,
                      max_per_img, out_count, out_det, out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

extern "C" int ptb_multiclass_soft_nms_cls_boxes(const float* boxes, const float* scores, int B, int P, int num_classes,
                                                 float score_thr, float iou_thr, float sigma, float min_score, int method,
                                                 int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label,
                                                 int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                                                 void* stream) {
  PTB_REQUIRE(boxes, "NULL boxes");
  return soft_nms_run<1>(nullptr, boxes, scores, B, P, num_classes, 0.f, 0.f, score_thr, iou_thr, sigma, min_score, method,
                      max_per_img, out_count, out_det, out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

// up to 8192 points per image: the multi-level P2P head's candidates (L levels x nms_pre).  Same arguments, workspaces and results as
// ptb_multiclass_nms / ptb_multiclass_soft_nms.
extern "C" int ptb_multiclass_nms_wide(const float* pts, const float* scores, int B, int P, int num_classes, float pseudo_w,
                                       float pseudo_h, float score_thr, float iou_thr, int max_per_img, int32_t* out_count,
                                       float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                                       void* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(pts, "NULL pts");
  return nms_run<0, true>(pts, nullptr, scores, B, P, num_classes, pseudo_w, pseudo_h, score_thr, iou_thr, max_per_img, out_count,
                          out_det, out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}

extern "C" int ptb_multiclass_soft_nms_wide(const float* pts, const float* boxes, const float* scores, int B, int P, int num_classes,
                                            float pseudo_w, float pseudo_h, float score_thr, float iou_thr, float sigma, float min_score,
                                            int method, int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label,
                                            int32_t* out_keep, int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes,
                                            void* stream) {
  return soft_nms_run<0, true>(pts, boxes, scores, B, P, num_classes, pseudo_w, pseudo_h, score_thr, iou_thr, sigma, min_score, method,
                               max_per_img, out_count, out_det, out_label, out_keep, out_cand_count, workspace, workspace_bytes, stream);
}
