// P2P head point path: decode + per-image top-k with sigmoid or softmax scores (p2p_head.py:125-170, 362-376), Hungarian cost
// matrix (match_cost.py:94-99, 197-214), PointAssigner (point_assigner.py:23-133) and the elementwise losses
// (focal_loss.py:11-56, smooth_l1_loss.py:25-31, cross_entropy_loss.py:9-89 sigmoid with or without class_weight and softmax,
// mse_loss.py:9-48).  All HBM-bound scan / select work: coalesced channels-last
// reads, warp-shuffle reductions, radix select + bitonic sort in shared memory (no library sort).
#include "ptb_common.cuh"
#include "loss_terms.cuh"
#include "topk_select.cuh"
#include <math_constants.h>

namespace ptb {

// ------------------------------------------------------------------------------------------------
// decode + top-k
// ------------------------------------------------------------------------------------------------
// key[b][q] = max_c sigmoid(cls[b][cell][a*C + c]),  q = cell*k + a.   One warp per proposal.
__global__ void __launch_bounds__(256)
p2p_score_kernel(const float* __restrict__ cls_map, long long BQ, int C, float* __restrict__ key) {
  const long long wq = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wq >= BQ) return;
  const float* row = cls_map + wq * C;     // [B][H][W][k*C] flattened: (b,cell,a) -> contiguous C floats
  float mx = -CUDART_INF_F;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, sigmoidf_acc(row[c]));
  mx = warp_max(mx);
  if (lane == 0) key[wq] = mx;
}

// Softmax over one row of C1 logits (background last), by one warp: m = max_c x_c, s = sum_c exp(x_c - m) (lane-strided partial
// sums, then the xor butterfly: a fixed order, the same bits in every lane and in every kernel that calls this), e_fg =
// max_{c < C1-1} exp(x_c - m).  softmax(row)[c] = exp(x_c - m) / s; division by s > 0 is monotone, so the largest foreground
// probability is exactly e_fg / s.
__device__ __forceinline__ void softmax_row_stats(const float* __restrict__ row, int C1, int lane, float& m, float& s, float& e_fg) {
  float mx = -CUDART_INF_F;
  for (int c = lane; c < C1; c += 32) mx = fmaxf(mx, row[c]);
  m = warp_max(mx);
  float acc = 0.f, ef = 0.f;
  for (int c = lane; c < C1; c += 32) {
    const float e = sleef_expf_u10(__fsub_rn(row[c], m));
    acc = __fadd_rn(acc, e);
    if (c < C1 - 1) ef = fmaxf(ef, e);
  }
  s = warp_sum(acc);
  e_fg = warp_max(ef);
}

// softmax classification (use_sigmoid=False, p2p_head.py:363,370): key[b][q] = max_{c<C} softmax(cls[b][q])[c] over a row of C+1
// logits.  One warp per proposal.
__global__ void __launch_bounds__(256)
p2p_softmax_score_kernel(const float* __restrict__ cls_map, long long BQ, int C, float* __restrict__ key) {
  const long long wq = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wq >= BQ) return;
  float m, s, e_fg;
  softmax_row_stats(cls_map + wq * (C + 1), C + 1, lane, m, s, e_fg);
  if (lane == 0) key[wq] = __fdiv_rn(e_fg, s);
}

// (radix select + bitonic sort: topk_select.cuh, shared with the RPN proposal path of rpn.cu)

// gather: decode the selected proposals.  SOFTMAX: rows of C+1 logits, out_scores = the C foreground probabilities (the background
// column is what multiclass_nms drops, bbox_nms.py:34,42), computed by softmax_row_stats like the key of p2p_softmax_score_kernel, so
// max_c out_scores[r][c] equals the key bit for bit.
template <bool SOFTMAX>
__global__ void __launch_bounds__(256)
p2p_gather_kernel(const float* __restrict__ cls_map, const float* __restrict__ reg_map, int H, int W, int C, int k,
                  const float* __restrict__ point_anchor, float stride, float gamma, const int32_t* __restrict__ img_hw,
                  const float* __restrict__ scale_xy, int P, int identity, const int32_t* __restrict__ idx,
                  int32_t* __restrict__ out_idx, float* __restrict__ out_pts, float* __restrict__ out_scores, long long BP) {
  const long long wr = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wr >= BP) return;
  const int b = (int)(wr / P);
  const int r = (int)(wr - (long long)b * P);
  const int q = identity ? r : idx[wr];
  const int Q = H * W * k;
  const int cell = q / k, a = q - cell * k;
  const int i = cell / W, j = cell - i * W;
  if (lane == 0) {
    if (identity) out_idx[wr] = q;
    // p2p_head.py:155-165 with PointGenerator.grid_points (no half-stride): anchor = (j*s, i*s) + point_anchor*s
    const float ax = __fadd_rn(__fmul_rn((float)j, stride), __fmul_rn(point_anchor[2 * a], stride));
    const float ay = __fadd_rn(__fmul_rn((float)i, stride), __fmul_rn(point_anchor[2 * a + 1], stride));
    const float* rg = reg_map + ((size_t)b * H * W + cell) * (2 * k) + 2 * a;
    float x = __fadd_rn(ax, __fmul_rn(__fmul_rn(rg[0], gamma), stride));
    float y = __fadd_rn(ay, __fmul_rn(__fmul_rn(rg[1], gamma), stride));
    x = fminf(fmaxf(x, 0.f), (float)img_hw[2 * b + 1]);      // p2p_head.py:374-375
    y = fminf(fmaxf(y, 0.f), (float)img_hw[2 * b]);
    if (scale_xy) { x = __fdiv_rn(x, scale_xy[2 * b]); y = __fdiv_rn(y, scale_xy[2 * b + 1]); }
    out_pts[wr * 2] = x; out_pts[wr * 2 + 1] = y;
  }
  float* orow = out_scores + wr * C;
  if constexpr (SOFTMAX) {
    const float* row = cls_map + ((size_t)b * Q + q) * (C + 1);
    float m, s, e_fg;
    softmax_row_stats(row, C + 1, lane, m, s, e_fg);
    for (int c = lane; c < C; c += 32) orow[c] = __fdiv_rn(sleef_expf_u10(__fsub_rn(row[c], m)), s);
  } else {
    const float* row = cls_map + ((size_t)b * Q + q) * C;
    for (int c = lane; c < C; c += 32) orow[c] = sigmoidf_acc(row[c]);
  }
}

// ------------------------------------------------------------------------------------------------
// decode + top-k over several FPN levels (p2p_head.py:125-170, 355-381).  An image's rows t in [0, T), T = sum_l H_l W_l k, are the
// levels' proposals concatenated level-major (cell-major, anchor-minor inside a level).  The reference's _get_bboxes_single then
// reshapes them into L equal chunks of T / L rows - not into levels - and takes the top nms_pre of each chunk, so a chunk may
// straddle two or more levels.  The key / select / gather steps below reproduce exactly that.
// ------------------------------------------------------------------------------------------------
constexpr int P2P_MAX_LEVELS = 8;
struct P2PLevels {
  const float* cls[P2P_MAX_LEVELS];      // [B][H_l][W_l][k*C1]
  const float* reg[P2P_MAX_LEVELS];      // [B][H_l][W_l][2k]
  int W[P2P_MAX_LEVELS];
  float stride[P2P_MAX_LEVELS];
  int row0[P2P_MAX_LEVELS + 1];          // first row of level l in an image; row0[L] = T
  int L;
  __device__ __forceinline__ int level_of(int t) const {
    int l = 0;
    while (l + 1 < L && t >= row0[l + 1]) ++l;
    return l;
  }
};

// key[b][t] as p2p_score_kernel / p2p_softmax_score_kernel compute it for row t's level.  One warp per row.
template <bool SOFTMAX>
__global__ void __launch_bounds__(256)
p2p_levels_score_kernel(P2PLevels lv, int B, int C, float* __restrict__ key) {
  const long long wq = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int T = lv.row0[lv.L];
  if (wq >= (long long)B * T) return;
  const int b = (int)(wq / T), t = (int)(wq - (long long)b * T);
  const int l = lv.level_of(t);
  const long long q = (long long)b * (lv.row0[l + 1] - lv.row0[l]) + (t - lv.row0[l]);
  if constexpr (SOFTMAX) {
    float m, s, e_fg;
    softmax_row_stats(lv.cls[l] + q * (C + 1), C + 1, lane, m, s, e_fg);
    if (lane == 0) key[wq] = __fdiv_rn(e_fg, s);
  } else {
    const float* row = lv.cls[l] + q * C;
    float mx = -CUDART_INF_F;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, sigmoidf_acc(row[c]));
    mx = warp_max(mx);
    if (lane == 0) key[wq] = mx;
  }
}

// gather: output row r of image b is entry r % P of chunk r / P; its image row is t = chunk * (T / L) + the chunk-local index
// (the select's output, or r itself when every chunk keeps all its rows).  Decode and scores as p2p_gather_kernel, at t's level.
template <bool SOFTMAX>
__global__ void __launch_bounds__(256)
p2p_levels_gather_kernel(P2PLevels lv, int C, int k, const float* __restrict__ point_anchor, float gamma,
                         const int32_t* __restrict__ img_hw, const float* __restrict__ scale_xy, int P, int identity,
                         int32_t* __restrict__ topk_idx, float* __restrict__ out_pts, float* __restrict__ out_scores, long long BR) {
  const long long wr = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wr >= BR) return;
  const int LP = lv.L * P, T = lv.row0[lv.L];
  const int b = (int)(wr / LP);
  const int r = (int)(wr - (long long)b * LP);
  const int chunk = r / P;
  const int local = identity ? r - chunk * P : topk_idx[wr];
  const int t = chunk * (T / lv.L) + local;
  const int l = lv.level_of(t);
  const int Ql = lv.row0[l + 1] - lv.row0[l];
  const int q = t - lv.row0[l];
  const int cell = q / k, a = q - cell * k;
  const int i = cell / lv.W[l], j = cell - i * lv.W[l];
  const float stride = lv.stride[l];
  if (lane == 0) {
    if (identity) topk_idx[wr] = local;
    const float ax = __fadd_rn(__fmul_rn((float)j, stride), __fmul_rn(point_anchor[2 * a], stride));
    const float ay = __fadd_rn(__fmul_rn((float)i, stride), __fmul_rn(point_anchor[2 * a + 1], stride));
    const float* rg = lv.reg[l] + ((size_t)b * (Ql / k) + cell) * (2 * k) + 2 * a;
    float x = __fadd_rn(ax, __fmul_rn(__fmul_rn(rg[0], gamma), stride));
    float y = __fadd_rn(ay, __fmul_rn(__fmul_rn(rg[1], gamma), stride));
    x = fminf(fmaxf(x, 0.f), (float)img_hw[2 * b + 1]);
    y = fminf(fmaxf(y, 0.f), (float)img_hw[2 * b]);
    if (scale_xy) { x = __fdiv_rn(x, scale_xy[2 * b]); y = __fdiv_rn(y, scale_xy[2 * b + 1]); }
    out_pts[wr * 2] = x; out_pts[wr * 2 + 1] = y;
  }
  float* orow = out_scores + wr * C;
  if constexpr (SOFTMAX) {
    const float* row = lv.cls[l] + ((size_t)b * Ql + q) * (C + 1);
    float m, s, e_fg;
    softmax_row_stats(row, C + 1, lane, m, s, e_fg);
    for (int c = lane; c < C; c += 32) orow[c] = __fdiv_rn(sleef_expf_u10(__fsub_rn(row[c], m)), s);
  } else {
    const float* row = lv.cls[l] + ((size_t)b * Ql + q) * C;
    for (int c = lane; c < C; c += 32) orow[c] = sigmoidf_acc(row[c]);
  }
}

// ------------------------------------------------------------------------------------------------
// cost matrix
// ------------------------------------------------------------------------------------------------
// FocalLossCost (match_cost.py:94-100) of one logit
__device__ __forceinline__ float focal_cost(float x, float alpha, float gamma, float eps, float w) {
  const float p = sigmoidf_acc(x);
  const float pg = (gamma == 2.f) ? __fmul_rn(p, p) : powf(p, gamma);
  const float omp = __fsub_rn(1.f, p);
  const float og = (gamma == 2.f) ? __fmul_rn(omp, omp) : powf(omp, gamma);
  const float neg = __fmul_rn(__fmul_rn(-logf(__fadd_rn(omp, eps)), __fsub_rn(1.f, alpha)), pg);
  const float pos = __fmul_rn(__fmul_rn(-logf(__fadd_rn(p, eps)), alpha), og);
  return __fmul_rn(__fsub_rn(pos, neg), w);
}

// torch.cdist(p=1) of two points already divided by the image size: |dx| + |dy|
__device__ __forceinline__ float l1_dist(float px, float py, float gx, float gy) {
  return __fadd_rn(fabsf(__fsub_rn(px, gx)), fabsf(__fsub_rn(py, gy)));
}

// torch.cdist(p=2) with both sides <= 25 rows (ATen's direct path, Distance.cpp cdist_impl), as the CPU build computes it:
// sqrt(fma(dy, dy, dx * dx)).  The plain formula without the FMA (ptb_common.cuh's cdist_direct) mismatched 5 646 of 69 271
// random pairs against torch 2.11's CPU cdist on an AVX-512 host; this order mismatched none.
__device__ __forceinline__ float l2_dist_direct(float px, float py, float gx, float gy) {
  const float dx = __fsub_rn(px, gx), dy = __fsub_rn(py, gy);
  return __fsqrt_rn(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

// The cost of one (row, GT) element.  row r of the matrix is proposal q = row_idx[r] of cls / pts.
// FocalL1Cost: the shipped pair FocalLossCost + DisCostV2(p=1), cost = focal + w_dis * |d|_1 (one add, as before the term lists).
struct FocalL1Cost {
  const float* cls; const float* pts; int ldp, C; const float* gts; const int32_t* gt_labels;
  float w_cls, alpha, gamma, eps, w_dis, fx, fy;
  __device__ __forceinline__ float operator()(long long, long long q, int g) const {
    const float cc = focal_cost(cls[q * C + gt_labels[g]], alpha, gamma, eps, w_cls);
    const float d = l1_dist(__fdiv_rn(pts[q * ldp], fx), __fdiv_rn(pts[q * ldp + 1], fy), __fdiv_rn(gts[2 * g], fx),
                            __fdiv_rn(gts[2 * g + 1], fy));
    return __fadd_rn(cc, __fmul_rn(d, w_dis));
  }
};

// TermListCost: HungarianAssignerV2's `sum(cls_costs) + sum(reg_costs)` (hungarian_assigner.py:223-227) over an ordered term list.
// Python's sum starts from 0, so each partial sum is 0 + t_1 + t_2 + ... in fp32 (0 + -0 is +0, as torch's tensor + 0), then one add
// of the two partials.  Classification kinds go to the first partial, DisCostV2 to the second, each in list order.
constexpr int MAX_COST_TERMS = 2 * PTB_MAX_MATCH_COST_TERMS;
struct CostTerms {
  ptb_match_cost t[MAX_COST_TERMS];
  int n;
};
struct TermListCost {
  const float* cls; const float* pts; int ldp, C; const float* gts; const int32_t* gt_labels;
  const float2* sm_stats;            // [n_rows] (max, sum of exp) of each row's softmax, when a ClassificationCostV2 softmax term is listed
  float img_w, img_h;
  bool use_mm;                       // torch.cdist(p=2)'s matmul formulation: either side has more than 25 rows
  CostTerms terms;
  __device__ __forceinline__ float operator()(long long r, long long q, int g) const {
    float cs = 0.f, rs = 0.f;
    const float x = cls[q * C + gt_labels[g]];
    for (int i = 0; i < terms.n; ++i) {
      const ptb_match_cost& t = terms.t[i];
      switch (t.kind) {
        case PTB_MATCH_COST_FOCAL: cs = __fadd_rn(cs, focal_cost(x, t.alpha, t.gamma, t.eps, t.weight)); break;
        case PTB_MATCH_COST_CLS_SIGMOID: cs = __fadd_rn(cs, __fmul_rn(-sigmoidf_acc(x), t.weight)); break;
        case PTB_MATCH_COST_CLS_SOFTMAX: {    // -(exp(x - m) / s) * w, the numerics of the softmax decode (softmax_row_stats)
          const float2 st = sm_stats[r];
          cs = __fadd_rn(cs, __fmul_rn(-__fdiv_rn(sleef_expf_u10(__fsub_rn(x, st.x)), st.y), t.weight));
          break;
        }
        case PTB_MATCH_COST_ZERO: cs = __fadd_rn(cs, 0.f); break;
        default: {                            // PTB_MATCH_COST_DIS: match_cost.py:208-214, the division by (w, h) first
          const float fx = t.norm_with_img_wh ? img_w : 1.f, fy = t.norm_with_img_wh ? img_h : 1.f;
          const float px = __fdiv_rn(pts[q * ldp], fx), py = __fdiv_rn(pts[q * ldp + 1], fy);
          const float gx = __fdiv_rn(gts[2 * g], fx), gy = __fdiv_rn(gts[2 * g + 1], fy);
          float d;
          if (t.p == 1) d = l1_dist(px, py, gx, gy);
          else if (use_mm) d = cdist_mm(px, py, sq_norm2(px, py), gx, gy, sq_norm2(gx, gy));
          else d = l2_dist_direct(px, py, gx, gy);
          rs = __fadd_rn(rs, __fmul_rn(d, t.weight));
        }
      }
    }
    return __fadd_rn(cs, rs);
  }
};

template <class Cost>
__global__ void __launch_bounds__(256)
cost_matrix_kernel(Cost cost_of, const int32_t* __restrict__ row_idx, long long n_rows, int n_gt, float* __restrict__ cost) {
  const long long total = n_rows * n_gt;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    const long long r = e / n_gt;
    const int g = (int)(e - r * n_gt);
    cost[e] = cost_of(r, row_idx ? row_idx[r] : r, g);
  }
}

// per-row softmax statistics (m, s) of the rows the matching uses, for ClassificationCostV2(use_sigmoid=False).  One warp per row.
__global__ void __launch_bounds__(256)
cost_softmax_stats_kernel(const float* __restrict__ cls, int C, const int32_t* __restrict__ row_idx, long long n_rows,
                          float2* __restrict__ stats) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const long long q = row_idx ? row_idx[r] : r;
  float m, s, e_fg;
  softmax_row_stats(cls + q * C, C, lane, m, s, e_fg);
  if (lane == 0) stats[r] = make_float2(m, s);
}

// ------------------------------------------------------------------------------------------------
// PointAssigner
// ------------------------------------------------------------------------------------------------
struct PaScratch {
  int lmin, lmax;
};

__global__ void pa_init_kernel(const float* __restrict__ points, int N, unsigned long long* __restrict__ best, PaScratch* sc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && blockIdx.x == 0) { /* lmin/lmax set by host memset pattern below */ }
  if (i < N) {
    best[i] = 0xFFFFFFFFFFFFFFFFull;
    const int lv = (int)log2f(points[3 * i + 2]);
    atomicMin(&sc->lmin, lv);
    atomicMax(&sc->lmax, lv);
  }
}
__global__ void pa_reset_kernel(PaScratch* sc) { sc->lmin = 0x7fffffff; sc->lmax = -0x7fffffff; }

// one CTA per GT: pos_num nearest points of its level claim the GT through a packed 64-bit atomicMin
__global__ void __launch_bounds__(256)
pa_assign_kernel(const float* __restrict__ points, int N, const float* __restrict__ gts, float scale, int pos_num,
                 const PaScratch* __restrict__ sc, unsigned long long* __restrict__ best) {
  __shared__ unsigned long long red[8];
  __shared__ unsigned long long chosen_prev;
  const int j = blockIdx.x;
  const float x1 = gts[4 * j], y1 = gts[4 * j + 1], x2 = gts[4 * j + 2], y2 = gts[4 * j + 3];
  const float cx = __fdiv_rn(__fadd_rn(x1, x2), 2.f), cy = __fdiv_rn(__fadd_rn(y1, y2), 2.f);
  const float w = fmaxf(__fsub_rn(x2, x1), 1e-6f), h = fmaxf(__fsub_rn(y2, y1), 1e-6f);
  int lvl = (int)(__fdiv_rn(__fadd_rn(log2f(__fdiv_rn(w, scale)), log2f(__fdiv_rn(h, scale))), 2.f));
  lvl = min(max(lvl, sc->lmin), sc->lmax);
  unsigned long long prev = 0ull;   // selections are strictly increasing in (dist, idx): pick the next one above `prev`
  for (int round = 0; round < pos_num; ++round) {
    unsigned long long mine = 0xFFFFFFFFFFFFFFFFull;
    for (int i = threadIdx.x; i < N; i += 256) {
      if ((int)log2f(points[3 * i + 2]) != lvl) continue;
      const float dx = __fdiv_rn(__fsub_rn(points[3 * i], cx), w), dy = __fdiv_rn(__fsub_rn(points[3 * i + 1], cy), h);
      const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)i;
      if ((round == 0 || key > prev) && key < mine) mine = key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, o);
      if (other < mine) mine = other;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long m = red[0];
      for (int wv = 1; wv < 8; ++wv) if (red[wv] < m) m = red[wv];
      chosen_prev = m;
      if (m != 0xFFFFFFFFFFFFFFFFull) {
        const unsigned int pi = (unsigned int)(m & 0xFFFFFFFFull);
        const unsigned long long claim = (m & 0xFFFFFFFF00000000ull) | (unsigned int)j;   // (dist, gt index)
        atomicMin(&best[pi], claim);
      }
    }
    __syncthreads();
    prev = chosen_prev;
    if (prev == 0xFFFFFFFFFFFFFFFFull) break;
  }
}

__global__ void pa_finish_kernel(const unsigned long long* __restrict__ best, int N, int64_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) out[i] = best[i] == 0xFFFFFFFFFFFFFFFFull ? 0 : (int64_t)(best[i] & 0xFFFFFFFFull) + 1;
}

// ------------------------------------------------------------------------------------------------
// losses with fused forward / backward and a fixed-order sum
// ------------------------------------------------------------------------------------------------
// FocalLoss (focal_loss.py:11-56) over M x C logits, the per-proposal weight broadcast over the classes
struct FocalLoss {
  const float* x; const int64_t* labels; const float* weight; int C; float gamma, alpha;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const long long m = e / C;
    const int c = (int)(e - m * C);
    const float w = weight ? weight[m] : 1.f;
    const float t = (labels[m] == c) ? 1.f : 0.f;
    const float v = x[e];
    const float p = sigmoidf_acc(v);
    const float pt = (1.f - p) * t + p * (1.f - t);
    const float a = alpha * t + (1.f - alpha) * (1.f - t);
    const float ptg = (gamma == 2.f) ? pt * pt : powf(pt, gamma);
    const float bce = fmaxf(v, 0.f) - v * t + log1pf(expf(-fabsf(v)));
    if (grad) {
      const float dpt = (t > 0.5f ? -1.f : 1.f) * p * (1.f - p);
      // d pt^gamma / d pt.  At gamma 0 it is 0, as torch's pow_backward makes it: gamma * powf(pt, -1) would be 0 * inf = NaN
      // for a saturated, correctly classified element (pt == 0)
      const float ptg1 = (gamma == 2.f) ? 2.f * pt : (gamma == 0.f ? 0.f : gamma * powf(pt, gamma - 1.f));
      grad[e] = sc * w * a * (ptg1 * dpt * bce + ptg * (p - t));
    }
    return bce * (a * ptg) * w;
  }
};

// The regression losses over several FPN levels: each proposal row m brings its own 1 / (stride_m * reg_norm) (p2p_head.py:234-240
// divides by the row's own stride), the rest is the single-level functor.
template <class Loss>
struct PerRowNorm {
  Loss base; const float* row_inv_norm;
  __device__ __forceinline__ float operator()(long long e, bool want_loss, float* grad, float sc) const {
    Loss l = base;
    l.inv_norm = row_inv_norm[e >> 1];
    return l(e, want_loss, grad, sc);
  }
};

// MSELoss (mse_loss.py:9-48): sum ((pred - target) * inv_norm)^2 * weight on the normalised points; d/dpred = 2 diff inv_norm w
struct MSELoss {
  const float* pred; const float* target; const float* weight; float inv_norm;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const float w = weight ? weight[e] : 1.f;
    const float diff = (pred[e] - target[e]) * inv_norm;
    if (grad) grad[e] = sc * w * inv_norm * 2.f * diff;
    return __fmul_rn(__fmul_rn(diff, diff), w);
  }
};

// CrossEntropyLoss(use_sigmoid=False) = cross_entropy (cross_entropy_loss.py:9-39): F.cross_entropy(x, y, weight=class_weight,
// reduction='none') over rows of C1 logits (background label C1-1 is an ordinary column), times the per-proposal weight, summed
// (the caller divides by avg_factor):  loss_m = w_m cw[y_m] (logsumexp(x_m) - x_m[y_m]),  d/dx = w_m cw[y_m] (softmax(x_m) - onehot(y_m)).
// One warp per row (softmax_row_stats); lane 0 carries the row's loss into the ordered block-partial sum.  A label outside [0, C1)
// makes its row's loss and gradient NaN: the library cannot report device data as an error code.
__global__ void __launch_bounds__(256)
softmax_ce_kernel(const float* __restrict__ x, const int64_t* __restrict__ labels, const float* __restrict__ weight,
                  const float* __restrict__ class_weight, long long M, int C1, float* loss_sum, const float* __restrict__ scale,
                  float* __restrict__ grad, SumScratch* __restrict__ scr) {
  const int lane = threadIdx.x & 31;
  const float sc = (grad && scale) ? scale[0] : 1.f;
  float acc = 0.f;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < M; r += (long long)gridDim.x * 8) {
    const float* row = x + r * C1;
    const int64_t y = labels[r];
    const bool ok = y >= 0 && y < C1;
    float m, s, e_fg;
    softmax_row_stats(row, C1, lane, m, s, e_fg);
    const float w = !ok ? CUDART_NAN_F : __fmul_rn(weight ? weight[r] : 1.f, class_weight ? class_weight[y] : 1.f);
    if (loss_sum && lane == 0) {
      const float lse = __fadd_rn(m, logf(s));
      acc += __fmul_rn(__fsub_rn(lse, ok ? row[y] : 0.f), w);
    }
    if (grad) {
      const float g = sc * w;
      float* grow = grad + r * C1;
      for (int c = lane; c < C1; c += 32) {
        const float p = __fdiv_rn(sleef_expf_u10(__fsub_rn(row[c], m)), s);
        grow[c] = __fmul_rn(g, __fsub_rn(p, c == y ? 1.f : 0.f));
      }
    }
  }
  if (loss_sum) block_partial_finish(acc, *scr, loss_sum);
}

}  // namespace ptb

using namespace ptb;

extern "C" uint64_t ptb_p2p_decode_topk_workspace(int B, int H, int W, int k) {
  return (uint64_t)B * H * W * k * sizeof(float) + (uint64_t)B * TOPK_MAX * sizeof(int32_t);
}

// decode + top-k of both score forms: sigmoid over rows of C logits, or softmax over rows of C+1 (background last)
template <bool SOFTMAX>
static int p2p_decode_topk(const float* cls_map, const float* reg_map, int B, int H, int W, int num_classes, int k,
                           const float* point_anchor, float stride, float pts_gamma, const int32_t* img_hw, const float* scale_xy,
                           int nms_pre, int32_t* out_topk_idx, float* out_pts, float* out_scores, void* workspace,
                           uint64_t workspace_bytes, void* stream) {
  const char* name = SOFTMAX ? "ptb_p2p_decode_topk_softmax" : "ptb_p2p_decode_topk";
  char what[64];
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && num_classes > 0 && k > 0, "shape");
  PTB_REQUIRE(cls_map && reg_map && point_anchor && img_hw && out_topk_idx && out_pts && out_scores, "NULL input");
  const int Q = H * W * k;
  const bool identity = !(nms_pre > 0 && nms_pre < Q);
  const int P = identity ? Q : nms_pre;
  PTB_REQUIRE(identity || nms_pre <= TOPK_MAX, "nms_pre > 4096 not supported");
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (!identity) {
    PTB_REQUIRE(workspace && workspace_bytes >= ptb_p2p_decode_topk_workspace(B, H, W, k), "workspace too small");
    float* key = reinterpret_cast<float*>(workspace);
    const long long BQ = (long long)B * Q;
    if (SOFTMAX)
      p2p_softmax_score_kernel<<<(unsigned)((BQ * 32 + 255) / 256), 256, 0, st>>>(cls_map, BQ, num_classes, key);
    else
      p2p_score_kernel<<<(unsigned)((BQ * 32 + 255) / 256), 256, 0, st>>>(cls_map, BQ, num_classes, key);
    snprintf(what, sizeof(what), "%s/score", name);
    if ((rc = check_launch(what))) return rc;
    p2p_select_kernel<<<B, SEL_THREADS, 0, st>>>(key, Q, P, out_topk_idx, P);
    snprintf(what, sizeof(what), "%s/select", name);
    if ((rc = check_launch(what))) return rc;
  }
  const long long BP = (long long)B * P;
  p2p_gather_kernel<SOFTMAX><<<(unsigned)((BP * 32 + 255) / 256), 256, 0, st>>>(cls_map, reg_map, H, W, num_classes, k,
                                                                              point_anchor, stride, pts_gamma, img_hw, scale_xy, P,
                                                                              identity ? 1 : 0, out_topk_idx, out_topk_idx, out_pts,
                                                                              out_scores, BP);
  snprintf(what, sizeof(what), "%s/gather", name);
  return check_launch(what);
}

extern "C" int ptb_p2p_decode_topk(const float* cls_map, const float* reg_map, int B, int H, int W, int num_classes, int k,
                                   const float* point_anchor, float stride, float pts_gamma, const int32_t* img_hw,
                                   const float* scale_xy, int nms_pre, int32_t* out_topk_idx, float* out_pts, float* out_scores,
                                   void* workspace, uint64_t workspace_bytes, void* stream) {
  return p2p_decode_topk<false>(cls_map, reg_map, B, H, W, num_classes, k, point_anchor, stride, pts_gamma, img_hw, scale_xy,
                                nms_pre, out_topk_idx, out_pts, out_scores, workspace, workspace_bytes, stream);
}

extern "C" int ptb_p2p_decode_topk_softmax(const float* cls_map, const float* reg_map, int B, int H, int W, int num_classes, int k,
                                           const float* point_anchor, float stride, float pts_gamma, const int32_t* img_hw,
                                           const float* scale_xy, int nms_pre, int32_t* out_topk_idx, float* out_pts,
                                           float* out_scores, void* workspace, uint64_t workspace_bytes, void* stream) {
  return p2p_decode_topk<true>(cls_map, reg_map, B, H, W, num_classes, k, point_anchor, stride, pts_gamma, img_hw, scale_xy,
                               nms_pre, out_topk_idx, out_pts, out_scores, workspace, workspace_bytes, stream);
}

extern "C" uint64_t ptb_p2p_decode_topk_levels_workspace(int B, int L, const int32_t* hw, int k) {
  uint64_t T = 0;
  for (int l = 0; l < L && hw; ++l) T += (uint64_t)hw[2 * l] * hw[2 * l + 1] * k;
  return (uint64_t)B * T * sizeof(float);
}

template <bool SOFTMAX>
static int p2p_decode_topk_levels(const float* const* cls_maps, const float* const* reg_maps, int L, const int32_t* hw,
                                  const float* strides, int B, int num_classes, int k, const float* point_anchor, float pts_gamma,
                                  const int32_t* img_hw, const float* scale_xy, int nms_pre, int32_t* out_topk_idx, float* out_pts,
                                  float* out_scores, void* workspace, uint64_t workspace_bytes, void* stream) {
  const char* name = SOFTMAX ? "ptb_p2p_decode_topk_levels_softmax" : "ptb_p2p_decode_topk_levels";
  char what[64];
  PTB_REQUIRE(L >= 1 && L <= P2P_MAX_LEVELS, "1 to 8 levels");
  PTB_REQUIRE(B > 0 && num_classes > 0 && k > 0, "shape");
  PTB_REQUIRE(cls_maps && reg_maps && hw && strides && point_anchor && img_hw && out_topk_idx && out_pts && out_scores, "NULL input");
  P2PLevels lv = {};
  lv.L = L;
  long long T = 0;
  for (int l = 0; l < L; ++l) {
    PTB_REQUIRE(cls_maps[l] && reg_maps[l] && hw[2 * l] > 0 && hw[2 * l + 1] > 0 && strides[l] > 0.f, "level shape");
    lv.cls[l] = cls_maps[l]; lv.reg[l] = reg_maps[l]; lv.W[l] = hw[2 * l + 1]; lv.stride[l] = strides[l];
    lv.row0[l] = (int)T;
    T += (long long)hw[2 * l] * hw[2 * l + 1] * k;
    PTB_REQUIRE(T <= 0x7fffffffLL, "more than 2^31 - 1 proposals per image");
  }
  lv.row0[L] = (int)T;
  // p2p_head.py:357-358 reshapes the rows into L equal chunks, which raises when L does not divide them
  PTB_REQUIRE(T % L == 0, "the number of proposals per image is not a multiple of the number of levels");
  const int chunk = (int)(T / L);
  const bool identity = !(nms_pre > 0 && nms_pre < chunk);
  const int P = identity ? chunk : nms_pre;
  PTB_REQUIRE(identity || nms_pre <= TOPK_MAX, "nms_pre > 4096 not supported");
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (!identity) {
    PTB_REQUIRE(workspace && workspace_bytes >= ptb_p2p_decode_topk_levels_workspace(B, L, hw, k), "workspace too small");
    float* key = reinterpret_cast<float*>(workspace);
    const long long BT = (long long)B * T;
    p2p_levels_score_kernel<SOFTMAX><<<(unsigned)((BT * 32 + 255) / 256), 256, 0, st>>>(lv, B, num_classes, key);
    snprintf(what, sizeof(what), "%s/score", name);
    if ((rc = check_launch(what))) return rc;
    // the B * L chunks are consecutive runs of T / L keys: one select CTA each, output row (b, chunk) at (b * L + chunk) * P
    p2p_select_kernel<<<B * L, SEL_THREADS, 0, st>>>(key, chunk, P, out_topk_idx, P);
    snprintf(what, sizeof(what), "%s/select", name);
    if ((rc = check_launch(what))) return rc;
  }
  const long long BR = (long long)B * L * P;
  p2p_levels_gather_kernel<SOFTMAX><<<(unsigned)((BR * 32 + 255) / 256), 256, 0, st>>>(lv, num_classes, k, point_anchor, pts_gamma,
                                                                                      img_hw, scale_xy, P, identity ? 1 : 0,
                                                                                      out_topk_idx, out_pts, out_scores, BR);
  snprintf(what, sizeof(what), "%s/gather", name);
  return check_launch(what);
}

extern "C" int ptb_p2p_decode_topk_levels(const float* const* cls_maps, const float* const* reg_maps, int L, const int32_t* hw,
                                          const float* strides, int B, int num_classes, int k, const float* point_anchor,
                                          float pts_gamma, const int32_t* img_hw, const float* scale_xy, int nms_pre,
                                          int32_t* out_topk_idx, float* out_pts, float* out_scores, void* workspace,
                                          uint64_t workspace_bytes, void* stream) {
  return p2p_decode_topk_levels<false>(cls_maps, reg_maps, L, hw, strides, B, num_classes, k, point_anchor, pts_gamma, img_hw,
                                       scale_xy, nms_pre, out_topk_idx, out_pts, out_scores, workspace, workspace_bytes, stream);
}

extern "C" int ptb_p2p_decode_topk_levels_softmax(const float* const* cls_maps, const float* const* reg_maps, int L,
                                                  const int32_t* hw, const float* strides, int B, int num_classes, int k,
                                                  const float* point_anchor, float pts_gamma, const int32_t* img_hw,
                                                  const float* scale_xy, int nms_pre, int32_t* out_topk_idx, float* out_pts,
                                                  float* out_scores, void* workspace, uint64_t workspace_bytes, void* stream) {
  return p2p_decode_topk_levels<true>(cls_maps, reg_maps, L, hw, strides, B, num_classes, k, point_anchor, pts_gamma, img_hw,
                                      scale_xy, nms_pre, out_topk_idx, out_pts, out_scores, workspace, workspace_bytes, stream);
}

static unsigned cost_matrix_blocks(int n_rows, int n_gt) {
  const long long blocks = ((long long)n_rows * n_gt + 255) / 256, cap = (long long)sm_count() * 8;
  return (unsigned)(blocks > cap ? cap : blocks);
}

extern "C" int ptb_p2p_cost_matrix(const float* cls_logits, const float* pts, int ldp, const int32_t* row_idx, int n_rows,
                                   int num_classes, const float* gts, const int32_t* gt_labels, int n_gt, float w_cls,
                                   float alpha, float gamma, float eps, float w_dis, float fx, float fy, float* cost,
                                   void* stream) {
  PTB_REQUIRE(n_rows >= 0 && n_gt >= 0 && num_classes > 0 && ldp >= 2, "shape");
  if (n_rows == 0 || n_gt == 0) return 0;
  PTB_REQUIRE(cls_logits && pts && gts && gt_labels && cost, "NULL input");
  cost_matrix_kernel<<<cost_matrix_blocks(n_rows, n_gt), 256, 0, (cudaStream_t)stream>>>(
      FocalL1Cost{cls_logits, pts, ldp, num_classes, gts, gt_labels, w_cls, alpha, gamma, eps, w_dis, fx, fy}, row_idx, n_rows, n_gt,
      cost);
  return check_launch("ptb_p2p_cost_matrix");
}

extern "C" uint64_t ptb_p2p_cost_matrix_terms_workspace(int n_rows) { return (uint64_t)(n_rows > 0 ? n_rows : 0) * sizeof(float2); }

extern "C" int ptb_p2p_cost_matrix_terms(const float* cls_logits, const float* pts, int ldp, const int32_t* row_idx, int n_rows,
                                         int num_cols, const float* gts, const int32_t* gt_labels, int n_gt, const ptb_match_cost* terms,
                                         int n_terms, float img_w, float img_h, float* cost, void* workspace, uint64_t workspace_bytes,
                                         void* stream) {
  PTB_REQUIRE(n_rows >= 0 && n_gt >= 0 && num_cols > 0 && ldp >= 2, "shape");
  PTB_REQUIRE(terms && n_terms > 0, "no cost terms");
  int n_cls = 0, n_reg = 0;
  bool softmax = false;
  for (int i = 0; i < n_terms && i <= MAX_COST_TERMS; ++i) {
    const ptb_match_cost& t = terms[i];
    PTB_REQUIRE(t.kind >= PTB_MATCH_COST_FOCAL && t.kind <= PTB_MATCH_COST_DIS, "unknown cost kind");
    PTB_REQUIRE(t.kind != PTB_MATCH_COST_DIS || t.p == 1 || t.p == 2, "DisCostV2 p must be 1 or 2");
    (t.kind == PTB_MATCH_COST_DIS ? n_reg : n_cls) += 1;
    softmax = softmax || t.kind == PTB_MATCH_COST_CLS_SOFTMAX;
  }
  PTB_REQUIRE(n_cls <= PTB_MAX_MATCH_COST_TERMS && n_reg <= PTB_MAX_MATCH_COST_TERMS,
              "at most 8 classification and 8 DisCostV2 terms");
  if (n_rows == 0 || n_gt == 0) return 0;
  PTB_REQUIRE(cls_logits && pts && gts && gt_labels && cost, "NULL input");
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  float2* stats = nullptr;
  if (softmax) {
    PTB_REQUIRE(workspace && workspace_bytes >= ptb_p2p_cost_matrix_terms_workspace(n_rows), "workspace too small");
    stats = reinterpret_cast<float2*>(workspace);
    cost_softmax_stats_kernel<<<(unsigned)(((long long)n_rows * 32 + 255) / 256), 256, 0, st>>>(cls_logits, num_cols, row_idx, n_rows,
                                                                                              stats);
    if ((rc = check_launch("ptb_p2p_cost_matrix_terms/softmax_stats"))) return rc;
  }
  TermListCost c{cls_logits, pts, ldp, num_cols, gts, gt_labels, stats, img_w, img_h, n_rows > 25 || n_gt > 25, {}};
  for (int i = 0; i < n_terms; ++i) c.terms.t[i] = terms[i];
  c.terms.n = n_terms;
  cost_matrix_kernel<<<cost_matrix_blocks(n_rows, n_gt), 256, 0, st>>>(c, row_idx, n_rows, n_gt, cost);
  return check_launch("ptb_p2p_cost_matrix_terms");
}

extern "C" uint64_t ptb_point_assigner_workspace(int N, int n) {
  (void)n;
  return (uint64_t)N * sizeof(unsigned long long) + 64;
}

extern "C" int ptb_point_assigner(const float* points, int N, const float* gt_bboxes, int n, float scale, int pos_num,
                                  int64_t* out_gt_inds, void* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(N >= 0 && n >= 0 && pos_num > 0 && scale > 0.f, "shape");
  if (N == 0) return 0;
  PTB_REQUIRE(points && out_gt_inds, "NULL input");
  PTB_REQUIRE(workspace && workspace_bytes >= ptb_point_assigner_workspace(N, n), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  PaScratch* sc = reinterpret_cast<PaScratch*>(workspace);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(workspace) + 64);
  int rc;
  pa_reset_kernel<<<1, 1, 0, st>>>(sc);
  if ((rc = check_launch("ptb_point_assigner/reset"))) return rc;
  pa_init_kernel<<<(N + 255) / 256, 256, 0, st>>>(points, N, best, sc);
  if ((rc = check_launch("ptb_point_assigner/init"))) return rc;
  if (n > 0) {
    PTB_REQUIRE(gt_bboxes, "NULL gt_bboxes");
    pa_assign_kernel<<<n, 256, 0, st>>>(points, N, gt_bboxes, scale, pos_num, sc, best);
    if ((rc = check_launch("ptb_point_assigner/assign"))) return rc;
  }
  pa_finish_kernel<<<(N + 255) / 256, 256, 0, st>>>(best, N, out_gt_inds);
  return check_launch("ptb_point_assigner/finish");
}

extern "C" int ptb_sigmoid_focal_fwd_bwd(const float* logits, const int64_t* labels, const float* weight, int64_t M,
                                         int num_classes, float gamma, float alpha, float* loss_sum, const float* scale,
                                         float* grad, void* stream) {
  PTB_REQUIRE(M >= 0 && num_classes > 0, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(logits && labels && (loss_sum || grad), "NULL input");
  return launch_sum(loss_sum_kernel<FocalLoss>, stream, "ptb_sigmoid_focal_fwd_bwd",
                    FocalLoss{logits, labels, weight, num_classes, gamma, alpha}, M * num_classes, loss_sum, scale, grad);
}

extern "C" int ptb_smooth_l1_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M, float inv_norm,
                                     float beta, float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0 && beta > 0.f, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && (loss_sum || grad), "NULL input");
  return launch_sum(loss_sum_kernel<SmoothL1Loss>, stream, "ptb_smooth_l1_fwd_bwd", SmoothL1Loss{pred, target, weight, inv_norm, beta},
                    M * 2, loss_sum, scale, grad);
}

extern "C" int ptb_sigmoid_bce_cw_fwd_bwd(const float* logits, const int64_t* labels, const float* weight, const float* pos_weight,
                                          int64_t M, int num_classes, float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0 && num_classes > 0, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(logits && labels && (loss_sum || grad), "NULL input");
  const char* name = "ptb_sigmoid_bce_cw_fwd_bwd";
  if (pos_weight)
    return launch_sum(loss_sum_kernel<SigmoidBCELoss<true>>, stream, name,
                      SigmoidBCELoss<true>{logits, labels, weight, pos_weight, num_classes}, M * num_classes, loss_sum, scale, grad);
  return launch_sum(loss_sum_kernel<SigmoidBCELoss<false>>, stream, name,
                    SigmoidBCELoss<false>{logits, labels, weight, nullptr, num_classes}, M * num_classes, loss_sum, scale, grad);
}

extern "C" int ptb_sigmoid_bce_fwd_bwd(const float* logits, const int64_t* labels, const float* weight, int64_t M, int num_classes,
                                       float* loss_sum, const float* scale, float* grad, void* stream) {
  return ptb_sigmoid_bce_cw_fwd_bwd(logits, labels, weight, nullptr, M, num_classes, loss_sum, scale, grad, stream);
}

extern "C" int ptb_softmax_ce_fwd_bwd(const float* logits, const int64_t* labels, const float* weight, const float* class_weight,
                                      int64_t M, int num_cols, float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0 && num_cols >= 2, "shape (softmax needs at least two columns)");
  if (M == 0) return 0;
  PTB_REQUIRE(logits && labels && (loss_sum || grad), "NULL input");
  return launch_sum(softmax_ce_kernel, stream, "ptb_softmax_ce_fwd_bwd", logits, labels, weight, class_weight, M, num_cols, loss_sum,
                    scale, grad);
}

extern "C" int ptb_mse_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M, float inv_norm,
                               float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && (loss_sum || grad), "NULL input");
  return launch_sum(loss_sum_kernel<MSELoss>, stream, "ptb_mse_fwd_bwd", MSELoss{pred, target, weight, inv_norm}, M * 2, loss_sum,
                    scale, grad);
}

extern "C" int ptb_smooth_l1_rows_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M,
                                          const float* row_inv_norm, float beta, float* loss_sum, const float* scale, float* grad,
                                          void* stream) {
  PTB_REQUIRE(M >= 0 && beta > 0.f, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && row_inv_norm && (loss_sum || grad), "NULL input");
  using L = PerRowNorm<SmoothL1Loss>;
  return launch_sum(loss_sum_kernel<L>, stream, "ptb_smooth_l1_rows_fwd_bwd", L{SmoothL1Loss{pred, target, weight, 0.f, beta}, row_inv_norm},
                    M * 2, loss_sum, scale, grad);
}

extern "C" int ptb_mse_rows_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M, const float* row_inv_norm,
                                    float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && row_inv_norm && (loss_sum || grad), "NULL input");
  using L = PerRowNorm<MSELoss>;
  return launch_sum(loss_sum_kernel<L>, stream, "ptb_mse_rows_fwd_bwd", L{MSELoss{pred, target, weight, 0.f}, row_inv_norm}, M * 2,
                    loss_sum, scale, grad);
}

// ------------------------------------------------------------------------------------------------
// GHM-C / GHM-R (ghm_loss.py:21-172), L1Loss (smooth_l1_loss.py:33-45) and BalancedL1Loss (balanced_l1_loss.py:12-49)
// ------------------------------------------------------------------------------------------------
// GHM runs in three launches over a batch of B images and nothing returns to the host:
//   1. ghm_hist_kernel: per (image, chunk) CTA, integer shared-memory counts of the valid elements per gradient-length bin, added to
//      the image's global counts with integer atomics (the same counts in any order);
//   2. ghm_weights_kernel: one thread walks the images in order and forms, with the reference's fp32 operation order, the image's
//      tot, its number of non-empty bins n, its per-bin weights and the in-place momentum update of acc_sum;
//   3. the loss pass per image (loss_sum_kernel with GHMCLoss / GHMRLoss): the element's bin again, its weight, the loss term into the
//      fixed-order sum, and with grad the gradient in the same launch.  Its backward reuses the bin weights of step 2.
// Bins are [edges[i], edges[i+1]) on fp32 g, as `(g >= edges[i]) & (g < edges[i+1])`; edges must be nondecreasing (the head checks a
// loaded buffer), so an element lies in at most one bin: the last i with edges[i] <= g, if g < edges[i+1].
namespace ptb {

__device__ __forceinline__ int ghm_bin(float g, const float* edges, int bins) {
  int lo = 0, hi = bins + 1;                // first index with edges[idx] > g, in [0, bins + 1]; a NaN g finds 0: no bin
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (edges[mid] <= g) lo = mid + 1; else hi = mid;
  }
  const int i = lo - 1;
  return (i >= 0 && i < bins && g < edges[i + 1]) ? i : -1;
}

// g of GHM-C: |sigmoid(x) - t| with ATen's CPU sigmoid bits (sigmoidf_acc)
struct GHMCGrad {
  const float* x; const int64_t* labels; const float* label_weight; long long Q; int C;
  __device__ __forceinline__ float operator()(int b, long long e, bool& valid) const {
    const long long m = e / C;
    const int c = (int)(e - m * C);
    valid = label_weight[b * Q + m] > 0.f;
    const float t = labels[b * Q + m] == c ? 1.f : 0.f;
    return fabsf(__fsub_rn(sigmoidf_acc(x[b * Q * C + e]), t));
  }
};

// GHM-R's normalised difference and g = |d / sqrt(mu^2 + d^2)| (mu2 = fp32(mu * mu), the reference's python-float square)
__device__ __forceinline__ float ghmr_diff(float p, float t, float inv) { return (p - t) * inv; }
__device__ __forceinline__ float ghmr_root(float d, float mu2) { return __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), mu2)); }

struct GHMRGrad {
  const float* pred; const float* target; const float* weight; const float* row_inv_norm; long long Q; float mu2;
  __device__ __forceinline__ float operator()(int b, long long e, bool& valid) const {
    const long long o = b * Q * 2 + e;
    valid = weight[o] > 0.f;
    const float d = ghmr_diff(pred[o], target[o], row_inv_norm[e >> 1]);
    return fabsf(__fdiv_rn(d, ghmr_root(d, mu2)));
  }
};

constexpr int GHM_HIST_ITEMS = 8;        // elements per thread and CTA sweep before the grid strides

// counts[b][i] (i < bins) = valid elements of image b in bin i; counts[b][bins] = valid elements of image b.  The warp aggregates
// equal bins (__match_any_sync) before the shared atomics: most of GHM-C's elements share the lowest bin.
template <class G>
__global__ void __launch_bounds__(256)
ghm_hist_kernel(G gf, long long n, const float* __restrict__ edges, int bins, int* __restrict__ counts) {
  __shared__ float se[PTB_GHM_MAX_BINS + 1];
  __shared__ int sc[PTB_GHM_MAX_BINS + 1];
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i <= bins; i += 256) { se[i] = edges[i]; sc[i] = 0; }
  __syncthreads();
  int nvalid = 0;
  for (long long base = (long long)blockIdx.x * 256; base < n; base += (long long)gridDim.x * 256) {
    const long long e = base + threadIdx.x;
    int key = -2;                                   // -2: out of range or invalid, -1: valid but in no bin
    if (e < n) {
      bool valid;
      const float g = gf(b, e, valid);
      if (valid) { key = ghm_bin(g, se, bins); ++nvalid; }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && lane == __ffs(peers) - 1) atomicAdd(&sc[key], __popc(peers));
  }
  nvalid = warp_sum_int(nvalid);
  if (lane == 0 && nvalid) atomicAdd(&sc[bins], nvalid);
  __syncthreads();
  for (int i = threadIdx.x; i <= bins; i += 256)
    if (sc[i]) atomicAdd(&counts[(long long)b * (bins + 1) + i], sc[i]);
}

// ghm_loss.py:76-90 / 154-168 per image, images in order.  tot = max(valid, 1) (GHM-R: the number of points with weight > 0, which is
// the reference's sum of its weights for the head's 0/1 point weights) is the exact count rounded once to fp32.  The reference sums
// the valid mask in fp32: the same value while the count stays below 2^24, within one ulp above it.  Without momentum w_i = fp32(tot / cnt_i) in double
// (python floats); with it acc_i = fp32(mmt) * acc_i + fp32((1 - mmt) * cnt_i), w_i = (1 / acc_i) * tot (python's float / tensor is
// reciprocal() * other).  Then w_i / n in fp32.  Empty bins weigh 0.
__global__ void ghm_weights_kernel(const int* __restrict__ counts, int B, int bins, double mmt, float* __restrict__ acc_sum,
                                   float* __restrict__ bin_weight, float* __restrict__ tot) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int b = 0; b < B; ++b) {
    const int* cb = counts + (long long)b * (bins + 1);
    const float t = fmaxf((float)cb[bins], 1.f);
    int nb = 0;
    for (int i = 0; i < bins; ++i) nb += cb[i] > 0;
    for (int i = 0; i < bins; ++i) {
      float w = 0.f;
      if (cb[i] > 0) {
        if (mmt > 0.0) {
          acc_sum[i] = __fadd_rn(__fmul_rn((float)mmt, acc_sum[i]), (float)((1.0 - mmt) * (double)cb[i]));
          w = __fmul_rn(__frcp_rn(acc_sum[i]), t);
        } else {
          w = (float)((double)t / (double)cb[i]);
        }
        w = __fdiv_rn(w, (float)nb);
      }
      bin_weight[(long long)b * bins + i] = w;
    }
    tot[b] = t;
  }
}

template <class G>
static int ghm_bin_weights(const char* name, G gf, int B, long long n, const float* edges, int bins, double momentum, float* acc_sum,
                           int* counts, float* bin_weight, float* tot, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)B * (bins + 1), st) != cudaSuccess) return fail("%s: cudaMemsetAsync failed", name);
  if (n > 0) {
    const long long per_cta = 256LL * GHM_HIST_ITEMS;
    const long long want = (n + per_cta - 1) / per_cta, cap = (4LL * sm_count() + B - 1) / B;
    const dim3 grid((unsigned)(want < cap ? want : cap), (unsigned)B);
    ghm_hist_kernel<G><<<grid, 256, 0, st>>>(gf, n, edges, bins, counts);
    int rc = check_launch(name);
    if (rc) return rc;
  }
  ghm_weights_kernel<<<1, 32, 0, st>>>(counts, B, bins, momentum, acc_sum, bin_weight, tot);
  return check_launch(name);
}

// GHMC's loss pass over one image's Q x C logits: binary_cross_entropy_with_logits(x, t, weights, reduction='sum') in ATen's CPU form
// ((1 - t) x - log_sigmoid(x), times the element weight); d/dx = (sigmoid(x) - t) * weight.
struct GHMCLoss {
  const float* x; const int64_t* labels; const float* label_weight; int C; const float* edges; int bins; const float* bin_weight;
  __device__ __forceinline__ float operator()(long long e, bool want_loss, float* grad, float sc) const {
    const long long m = e / C;
    const int c = (int)(e - m * C);
    const float t = labels[m] == c ? 1.f : 0.f;
    const float v = x[e];
    const float p = sigmoidf_acc(v);
    float w = 0.f;
    if (label_weight[m] > 0.f) {
      const int i = ghm_bin(fabsf(__fsub_rn(p, t)), edges, bins);
      if (i >= 0) w = bin_weight[i];
    }
    if (grad) grad[e] = sc * w * (p - t);
    if (!want_loss) return 0.f;
    const float log_sig = __fsub_rn(fminf(v, 0.f), log1pf(expf(-fabsf(v))));
    return __fmul_rn(__fsub_rn(__fmul_rn(1.f - t, v), log_sig), w);
  }
};

// GHMR's loss pass over one image's (Q, 2) points: (sqrt(d^2 + mu^2) - mu) * weight; d/dpred = d / sqrt(d^2 + mu^2) * inv * weight
struct GHMRLoss {
  const float* pred; const float* target; const float* weight; const float* row_inv_norm; float mu, mu2; const float* edges; int bins;
  const float* bin_weight;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const float inv = row_inv_norm[e >> 1];
    const float d = ghmr_diff(pred[e], target[e], inv);
    const float r = ghmr_root(d, mu2);
    float w = 0.f;
    if (weight[e] > 0.f) {
      const int i = ghm_bin(fabsf(__fdiv_rn(d, r)), edges, bins);
      if (i >= 0) w = bin_weight[i];
    }
    if (grad) grad[e] = sc * w * inv * (d / r);
    return (r - mu) * w;
  }
};

// BalancedL1Loss on the normalised points, a = |d|, b = e^(gamma / alpha) - 1 (kb = fp32(b), kab = fp32(alpha / b)):
//   a < beta:  kab (kb a + 1) log(kb a / beta + 1) - alpha a;   else gamma a + gamma / b - alpha beta.
// d/da = kab kb log(u) + kab (kb a + 1) kb / (beta u) - alpha with u = kb a / beta + 1, or gamma; times sign(d) (0 at 0) * inv * weight.
struct BalancedL1RowsLoss {
  const float* pred; const float* target; const float* weight; const float* row_inv_norm; float alpha, gamma, beta, kb, kab, kgb;
  __device__ __forceinline__ float operator()(long long e, bool, float* grad, float sc) const {
    const float inv = row_inv_norm[e >> 1];
    const float w = weight ? weight[e] : 1.f;
    const float d = (pred[e] - target[e]) * inv;
    const float a = fabsf(d);
    const bool in = a < beta;
    const float u = kb * a / beta + 1.f;
    if (grad) {
      const float da = in ? kab * kb * logf(u) + kab * (kb * a + 1.f) * kb / (beta * u) - alpha : gamma;
      grad[e] = sc * w * inv * da * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f * d));
    }
    return (in ? kab * (kb * a + 1.f) * logf(u) - alpha * a : gamma * a + kgb - alpha * beta) * w;
  }
};

}  // namespace ptb

extern "C" int ptb_ghmc_bin_weights(const float* logits, const int64_t* labels, const float* label_weight, int B, int64_t Q,
                                    int num_classes, const float* edges, int bins, double momentum, float* acc_sum, int32_t* counts,
                                    float* bin_weight, float* tot, void* stream) {
  PTB_REQUIRE(B > 0 && Q >= 0 && num_classes > 0 && Q * num_classes < (1LL << 31), "shape (Q x num_classes must stay below 2^31)");
  PTB_REQUIRE(bins >= 1 && bins <= PTB_GHM_MAX_BINS, "GHMC bins must lie in [1, PTB_GHM_MAX_BINS]");
  PTB_REQUIRE(logits && labels && label_weight && edges && counts && bin_weight && tot && (momentum <= 0.0 || acc_sum), "NULL input");
  return ghm_bin_weights("ptb_ghmc_bin_weights", GHMCGrad{logits, labels, label_weight, Q, num_classes}, B, Q * num_classes, edges,
                         bins, momentum, acc_sum, counts, bin_weight, tot, stream);
}

extern "C" int ptb_ghmc_fwd_bwd(const float* logits, const int64_t* labels, const float* label_weight, int64_t Q, int num_classes,
                                const float* edges, int bins, const float* bin_weight, float* loss_sum, const float* scale, float* grad,
                                void* stream) {
  PTB_REQUIRE(Q >= 0 && num_classes > 0 && bins >= 1 && bins <= PTB_GHM_MAX_BINS, "shape");
  if (Q == 0) return 0;
  PTB_REQUIRE(logits && labels && label_weight && edges && bin_weight && (loss_sum || grad), "NULL input");
  return launch_sum(loss_sum_kernel<GHMCLoss>, stream, "ptb_ghmc_fwd_bwd",
                    GHMCLoss{logits, labels, label_weight, num_classes, edges, bins, bin_weight}, Q * num_classes, loss_sum, scale, grad);
}

extern "C" int ptb_ghmr_bin_weights(const float* pred, const float* target, const float* weight, const float* row_inv_norm, float mu,
                                    int B, int64_t Q, const float* edges, int bins, double momentum, float* acc_sum, int32_t* counts,
                                    float* bin_weight, float* tot, void* stream) {
  PTB_REQUIRE(B > 0 && Q >= 0 && Q < (1LL << 30), "shape");
  PTB_REQUIRE(bins >= 1 && bins <= PTB_GHM_MAX_BINS, "GHMR bins must lie in [1, PTB_GHM_MAX_BINS]");
  PTB_REQUIRE(pred && target && weight && row_inv_norm && edges && counts && bin_weight && tot && (momentum <= 0.0 || acc_sum),
              "NULL input");
  const float mu2 = (float)((double)mu * (double)mu);
  return ghm_bin_weights("ptb_ghmr_bin_weights", GHMRGrad{pred, target, weight, row_inv_norm, Q, mu2}, B, Q * 2, edges, bins, momentum,
                         acc_sum, counts, bin_weight, tot, stream);
}

extern "C" int ptb_ghmr_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t Q, const float* row_inv_norm,
                                float mu, const float* edges, int bins, const float* bin_weight, float* loss_sum, const float* scale,
                                float* grad, void* stream) {
  PTB_REQUIRE(Q >= 0 && bins >= 1 && bins <= PTB_GHM_MAX_BINS, "shape");
  if (Q == 0) return 0;
  PTB_REQUIRE(pred && target && weight && row_inv_norm && edges && bin_weight && (loss_sum || grad), "NULL input");
  const float mu2 = (float)((double)mu * (double)mu);
  return launch_sum(loss_sum_kernel<GHMRLoss>, stream, "ptb_ghmr_fwd_bwd",
                    GHMRLoss{pred, target, weight, row_inv_norm, mu, mu2, edges, bins, bin_weight}, Q * 2, loss_sum, scale, grad);
}

extern "C" int ptb_l1_rows_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M, const float* row_inv_norm,
                                   float* loss_sum, const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0, "shape");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && row_inv_norm && (loss_sum || grad), "NULL input");
  return launch_sum(loss_sum_kernel<L1RowsLoss>, stream, "ptb_l1_rows_fwd_bwd", L1RowsLoss{pred, target, weight, row_inv_norm}, M * 2,
                    loss_sum, scale, grad);
}

extern "C" int ptb_balanced_l1_rows_fwd_bwd(const float* pred, const float* target, const float* weight, int64_t M,
                                            const float* row_inv_norm, float alpha, float gamma, float beta, float* loss_sum,
                                            const float* scale, float* grad, void* stream) {
  PTB_REQUIRE(M >= 0 && alpha > 0.f && beta > 0.f, "shape (alpha and beta must be positive)");
  // b = e^(gamma / alpha) - 1 divides the loss: mmdet raises at gamma == 0, and a NaN gamma makes every term NaN
  PTB_REQUIRE(gamma != 0.f && gamma == gamma, "gamma must be non-zero and not NaN (b = e^(gamma / alpha) - 1 must not be 0)");
  if (M == 0) return 0;
  PTB_REQUIRE(pred && target && row_inv_norm && (loss_sum || grad), "NULL input");
  const double b = exp((double)gamma / (double)alpha) - 1.0;
  return launch_sum(loss_sum_kernel<BalancedL1RowsLoss>, stream, "ptb_balanced_l1_rows_fwd_bwd",
                    BalancedL1RowsLoss{pred, target, weight, row_inv_norm, alpha, gamma, beta, (float)b, (float)((double)alpha / b),
                                       (float)((double)gamma / b)},
                    M * 2, loss_sum, scale, grad);
}
