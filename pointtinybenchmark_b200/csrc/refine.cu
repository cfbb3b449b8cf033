// Point refinement (PointRefiner.refine_single, cpr_head.py:780-850) — stage form and fused form.
//
// One CTA (4 warps) per GT.  A warp owns one bag sample at a time:
//   * lanes span the classes (128-bit loads of channels-last logits / probabilities) -> argmax for the classify
//     filter (cpr_head.py:745-756) by shuffle reduction, prob of the GT's label by broadcast;
//   * lanes span the same-(image,label) GT group for the nearest filter (cpr_head.py:711-743), distances in
//     torch.cdist's fp32 matmul formulation, first-index argmin by shuffle reduction;
//   * thresholds (cpr_head.py:823) and inside-image (773-778) are scalar;
// then the CTA reduces the surviving samples: weights, weighted mean, score, not_refine fallback (829-838).
// The fused form never materialises the (G,K,classes) probability tensor: it bilinearly samples the class-logit map
// (linearity: Linear(bilinear(feat)) == bilinear(Linear(feat)), border padding keeps the 4 weights summing to 1).
#include "tc_ptx.cuh"
#include <math_constants.h>
#include <stdlib.h>
#include <string.h>

namespace ptb {

constexpr int RF_THREADS = 128;          // stage kernel
constexpr int RF_WARPS = RF_THREADS / 32;
constexpr int RF_MAXWARPS = 32;

struct ArgMin {
  float d;
  int i;
};
__device__ __forceinline__ ArgMin warp_argmin_first(ArgMin a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float od = __shfl_xor_sync(0xffffffffu, a.d, o);
    const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
    if (od < a.d || (od == a.d && oi < a.i)) { a.d = od; a.i = oi; }
  }
  return a;
}
// argmax with lowest index on ties (torch.max(dim) on CPU keeps the first maximum)
__device__ __forceinline__ ArgMin warp_argmax_first(ArgMin a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float od = __shfl_xor_sync(0xffffffffu, a.d, o);
    const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
    if (od > a.d || (od == a.d && oi < a.i)) { a.d = od; a.i = oi; }
  }
  return a;
}

__device__ __forceinline__ float block_sum(float v, float* red /*[RF_MAXWARPS]*/) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  const int nw = (int)(blockDim.x >> 5);
  for (int w = 0; w < nw; ++w) s += red[w];
  return s;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = red[0];
  const int nw = (int)(blockDim.x >> 5);
  for (int w = 1; w < nw; ++w) s = fmaxf(s, red[w]);
  return s;
}

// nearest filter for one sample, evaluated by a full warp.  Candidates = (member j, refine r) centres in group order.
//   cand(j, r, &cx, &cy) supplies centre coordinates.  Returns true iff argmin == own.
template <class CandFn>
__device__ __forceinline__ bool nearest_is_own(float px, float py, int t, int R, int own, bool use_mm, CandFn cand, int lane) {
  const float pn = sq_norm2(px, py);
  ArgMin best;
  best.d = CUDART_INF_F;
  best.i = 0x7fffffff;
  const int total = t * R;
  for (int q = lane; q < total; q += 32) {
    float cx, cy;
    cand(q / R, q % R, cx, cy);
    const float d = use_mm ? cdist_mm(px, py, pn, cx, cy, sq_norm2(cx, cy)) : cdist_direct(px, py, cx, cy);
    if (d < best.d) { best.d = d; best.i = q; }   // ascending q per lane: keeps the first minimum
  }
  best = warp_argmin_first(best);
  return best.i == own;
}

// three block sums with ONE pair of barriers (fixed order: deterministic); red holds 3 * RF_MAXWARPS floats
__device__ __forceinline__ void block_sum3(float& a, float& b, float& c, float* red) {
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  __syncthreads();
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[w] = a; red[RF_MAXWARPS + w] = b; red[2 * RF_MAXWARPS + w] = c; }
  __syncthreads();
  a = b = c = 0.f;
  const int nw = (int)(blockDim.x >> 5);
  for (int i = 0; i < nw; ++i) { a += red[i]; b += red[RF_MAXWARPS + i]; c += red[2 * RF_MAXWARPS + i]; }
}

// tail shared by both forms: pm/x/y in shared memory (red: 3 * RF_MAXWARPS floats)
__device__ __forceinline__ void refine_tail(const float* pm, const float* sx, const float* sy, int Kt, float gt_x, float gt_y,
                                            const uint8_t* not_refine_in, int g, const ptb_refine_cfg& cfg, float* red,
                                            float* out_pts, float* out_score, uint8_t* out_not_refine, uint8_t* out_chosen) {
  const int tid = threadIdx.x;
  float s = 0.f, c = 0.f, mx = 0.f;
  for (int k = tid; k < Kt; k += blockDim.x) {
    const float v = pm[k];
    s += v;
    c += (v > 0.f) ? 1.f : 0.f;
    mx = fmaxf(mx, v);
  }
  float sum = s, cnt = c, dummy = 0.f;
  block_sum3(sum, cnt, dummy, red);
  const float denom = __fadd_rn(sum, 1e-8f);        // cpr_head.py:832
  float ax = 0.f, ay = 0.f;
  for (int k = tid; k < Kt; k += blockDim.x) {
    const float w = __fdiv_rn(pm[k], denom);
    ax += __fmul_rn(sx[k], w);
    ay += __fmul_rn(sy[k], w);
    if (out_chosen) out_chosen[(size_t)g * Kt + k] = w > 0.f;     // cpr_head.py:849
  }
  float rx = ax, ry = ay;
  dummy = 0.f;
  block_sum3(rx, ry, dummy, red);
  float score = __fdiv_rn(sum, __fadd_rn(cnt, 1e-8f));   // cpr_head.py:835
  bool nr = score < cfg.refine_th;                        // cpr_head.py:836
  if (not_refine_in) nr = nr || (not_refine_in[g] != 0);
  if (cfg.flags & 4) {                                    // return_score_type == 'max' (cpr_head.py:840-842)
    const float m = block_max(mx, red);
    score = (m == 0.f) ? __fmul_rn(cfg.refine_th, 0.5f) : m;
  }
  if (tid == 0) {
    out_pts[2 * g] = nr ? gt_x : rx;
    out_pts[2 * g + 1] = nr ? gt_y : ry;
    out_score[g] = score;
    out_not_refine[g] = nr;
  }
}

// ------------------------------------------------------------------------------------------------
// stage form: probabilities given
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RF_THREADS)
refine_stage_kernel(const float* __restrict__ prob, const float* __restrict__ pts, const uint8_t* __restrict__ valid,
                    int Kt, int K, int ncls, const int32_t* __restrict__ labels, const int32_t* __restrict__ bag_img,
                    const int32_t* __restrict__ img_hw, const int32_t* __restrict__ grp_of,
                    const int32_t* __restrict__ grp_ptr, const int32_t* __restrict__ grp_idx,
                    const uint8_t* __restrict__ not_refine_in, ptb_refine_cfg cfg, float* __restrict__ out_pts,
                    float* __restrict__ out_score, uint8_t* __restrict__ out_not_refine, uint8_t* __restrict__ out_chosen,
                    uint8_t* __restrict__ out_merge_valid) {
  extern __shared__ float sm[];
  float* pm = sm;            // [Kt]
  float* sx = sm + Kt;       // [Kt]
  float* sy = sm + 2 * Kt;   // [Kt]
  __shared__ float red[3 * RF_MAXWARPS];
  const int g = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l = labels[g], b = bag_img[g];
  const int R = Kt / K;
  const float ih = (float)img_hw[2 * b], iw = (float)img_hw[2 * b + 1];
  const int gi = grp_of[g];
  const int m0 = grp_ptr[gi], t = grp_ptr[gi + 1] - m0;
  int pos = 0;
  for (int j = 0; j < t; ++j) if (grp_idx[m0 + j] == g) pos = j;
  const bool use_mm = ((long long)t * R * K > 25) || (t * R > 25);
  const float* gprob = prob + (size_t)g * Kt * ncls;
  const float pg = gprob[(size_t)(K - 1) * ncls + l];           // centre of refine 0 (cpr_head.py:807,821)
  const float pg_a = __fmul_rn(pg, cfg.gt_alpha);

  for (int s = warp; s < Kt; s += RF_WARPS) {
    const float* pr = gprob + (size_t)s * ncls;
    const float px = pts[((size_t)g * Kt + s) * 3], py = pts[((size_t)g * Kt + s) * 3 + 1];
    bool m = valid[(size_t)g * Kt + s] != 0;
    if (cfg.flags & 2) {
      ArgMin a;
      a.d = -CUDART_INF_F;
      a.i = 0x7fffffff;
      for (int c = lane; c < ncls; c += 32) {
        const float v = pr[c];
        if (v > a.d) { a.d = v; a.i = c; }
      }
      a = warp_argmax_first(a);
      m = m && (a.i == l);
    }
    if ((cfg.flags & 1) && t > 1) {
      auto cand = [&](int j, int r, float& cx, float& cy) {
        const size_t o = ((size_t)grp_idx[m0 + j] * Kt + (size_t)r * K + (K - 1)) * 3;
        cx = pts[o]; cy = pts[o + 1];
      };
      m = m && nearest_is_own(px, py, t, R, pos * R + s / K, use_mm, cand, lane);
    }
    const float p = pr[l];
    m = m && (p > cfg.merge_th) && (p > pg_a);
    m = m && (px < iw) && (px >= 0.f) && (py < ih) && (py >= 0.f);
    if (lane == 0) {
      pm[s] = m ? p : 0.f;      // bag_cls_prob * merge_valid.float()   (p * 1.0 or p * 0.0)
      sx[s] = px; sy[s] = py;
      if (out_merge_valid) out_merge_valid[(size_t)g * Kt + s] = m;
    }
  }
  __syncthreads();
  const float gx = pts[((size_t)g * Kt + (K - 1)) * 3], gy = pts[((size_t)g * Kt + (K - 1)) * 3 + 1];
  refine_tail(pm, sx, sy, Kt, gx, gy, not_refine_in, g, cfg, red, out_pts, out_score, out_not_refine, out_chosen);
}

// ------------------------------------------------------------------------------------------------
// fused form: logits sampled from the map on the fly (num_refine == 1).  One CTA per GT.
//
// TMA staging (round 2).  The 289 samples x 4 taps of a bag fall in a window of (2r+2)^2 map cells around the GT (18 x 18 at r = 8):
// ONE cp.async.bulk.tensor box {ld channels, WS, WS, 1 image} brings the bag's logit tile (104 KB at 80 classes) into shared memory
// and every tap is served from there (1156 tap reads of 320 B = 370 KB per GT against 104 KB moved: round 1 pulled all of them
// through L1, 1.48 GB of L2->L1 traffic per batch for a 43 MB map).  The box origin is the tap of the bag's extreme sample (the
// coordinate pipeline is monotone, so no sample can fall left / above it); cells beyond the map edge are the TMA unit's zero fill and
// are never addressed because taps are clamped like the reference's border padding.  A bag whose window does not fit (a rounding
// straddle gives 2r+3 cells once in ~1e5 bags) takes the same code on global memory.  While the box is in flight the CTA does the
// map-independent work (coordinates, validity, nearest-GT filter); two CTAs per SM overlap one's load with the other's math.
//
// Lane mappings per warp and 32 samples: "owner" phases (lane = sample: coordinates, nearest filter, sigmoids, thresholds) and a
// "class" phase (8 lanes per sample, 4 samples per round: the 8 lanes read 128 contiguous bytes of each tap).
// Classify filter without per-class bookkeeping: the reference takes the FIRST maximum of the PROBABILITIES (cpr_head.py:745-756);
// sigmoid is monotone, so  argmax_first(prob) == l  <=>  p_l >= sigmoid(max_c logit)  and  p_l > sigmoid(max_{c<l} logit):
// the class loop keeps two running maxima (3 + 2 instructions per 4 classes instead of 20 for arg-max + runner-up tracking) and the
// owner evaluates three sigmoids per sample.  Saturated ties (both 1.0f) resolve to the lower class exactly like torch.max.
// ------------------------------------------------------------------------------------------------
constexpr int RF_GCAP = 256;              // group members staged in shared memory (larger groups read the rest from global memory)
constexpr int RF_SUB = 8;                 // lanes per sample in the class phase
constexpr int RF_SPW = 32 / RF_SUB;       // samples per round

__device__ __forceinline__ float4 ld_tap(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 lds_tap(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}

struct RfTile {           // where the taps of this CTA live
  const float* gbase;     // image base in global memory (fallback)
  uint32_t sbase;         // window base in shared memory (staged)
  int pitch, ox, oy;      // cells per row and origin of the addressed array (staged: WS, window origin; global: W, 0, 0)
};

// class phase for the 32 samples a warp owns: returns (to the owner lane) max logit, max logit over classes < l, logit of class l.
// NT = float4 class groups per lane (ceil(ceil(ncls/4) / 8)); requires ncls % 4 == 0 and (NT-1)*8 < cg4 (only the LAST trip is partial).
// Shape of the code (per-trip branches and predicated -inf initialisation / select chains cost many SASS instructions per trip): trips 0..NT-2 are unconditional (all tap loads first, then the FMA chains), the
// last trip sits under one branch, and the label's own group is loaded a second time as a broadcast (4 LDS + 16 FFMA) instead of being
// picked out of the trips with selects.
template <bool STAGED, int NT>
__device__ __forceinline__ void rf_class_phase(const RfTile& tl, float ix, float iy, int H, int W, int ld, int cg4, int l4, int lq,
                                               int lane, int n_rounds, float& o_max, float& o_maxlt, float& o_llab) {
  const int sub = lane & (RF_SUB - 1), slot = lane / RF_SUB;
  const bool last_on = sub + 8 * (NT - 1) < cg4;
  const int n_below = min(max((l4 - sub + 7) >> 3, 0), NT);            // trips of this lane whose group lies entirely below the label's
  auto tap = [&](int off) -> float4 {
    if (STAGED) return lds_tap(tl.sbase + 4u * (uint32_t)off);
    return ld_tap(tl.gbase + (size_t)off);
  };
#pragma unroll 1
  for (int r = 0; r < n_rounds; ++r) {            // rounds without an active sample are skipped (the last warp of a 289-sample bag owns ONE)
    const int src = RF_SPW * r + slot;
    const float sxi = __shfl_sync(0xffffffffu, ix, src), syi = __shfl_sync(0xffffffffu, iy, src);
    const float x0f = floorf(sxi), y0f = floorf(syi);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);        // east / south tap has weight 0 when clamped
    const float ex = __fsub_rn(__fadd_rn(x0f, 1.f), sxi), wx = __fsub_rn(sxi, x0f);
    const float ey = __fsub_rn(__fadd_rn(y0f, 1.f), syi), wy = __fsub_rn(syi, y0f);
    const float w00 = __fmul_rn(ex, ey), w01 = __fmul_rn(wx, ey), w10 = __fmul_rn(ex, wy), w11 = __fmul_rn(wx, wy);
    const int r0 = (y0 - tl.oy) * tl.pitch - tl.ox, r1 = (y1 - tl.oy) * tl.pitch - tl.ox;
    const int b00 = (r0 + x0) * ld, b01 = (r0 + x1) * ld, b10 = (r1 + x0) * ld, b11 = (r1 + x1) * ld;
    const int c00 = b00 + 4 * sub, c01 = b01 + 4 * sub, c10 = b10 + 4 * sub, c11 = b11 + 4 * sub;
    float m4[NT];
    {
      float4 q0[NT], q1[NT], q2[NT], q3[NT];
#pragma unroll
      for (int i = 0; i < NT - 1; ++i) {
        q0[i] = tap(c00 + 32 * i); q1[i] = tap(c01 + 32 * i); q2[i] = tap(c10 + 32 * i); q3[i] = tap(c11 + 32 * i);
      }
#pragma unroll
      for (int i = 0; i < NT - 1; ++i) {
        const float4 lg = bilerp4(q0[i], q1[i], q2[i], q3[i], w00, w01, w10, w11);
        m4[i] = fmaxf(fmaxf(lg.x, lg.y), fmaxf(lg.z, lg.w));
      }
      m4[NT - 1] = -CUDART_INF_F;
      if (last_on) {
        const float4 lg = bilerp4(tap(c00 + 32 * (NT - 1)), tap(c01 + 32 * (NT - 1)), tap(c10 + 32 * (NT - 1)), tap(c11 + 32 * (NT - 1)),
                                  w00, w01, w10, w11);
        m4[NT - 1] = fmaxf(fmaxf(lg.x, lg.y), fmaxf(lg.z, lg.w));
      }
    }
    float mx = m4[0], mlt = -CUDART_INF_F;
#pragma unroll
    for (int i = 1; i < NT; ++i) mx = fmaxf(mx, m4[i]);
#pragma unroll
    for (int i = 0; i < NT; ++i) mlt = fmaxf(mlt, i < n_below ? m4[i] : -CUDART_INF_F);
    // the label's own group (same addresses for the 8 lanes of a sample: broadcast): its logit and the classes below it inside the group
    const float4 lgl = bilerp4(tap(b00 + 4 * l4), tap(b01 + 4 * l4), tap(b10 + 4 * l4), tap(b11 + 4 * l4), w00, w01, w10, w11);
    const float llab = lq == 0 ? lgl.x : lq == 1 ? lgl.y : lq == 2 ? lgl.z : lgl.w;
    float part = -CUDART_INF_F;
    if (lq > 0) part = lgl.x;
    if (lq > 1) part = fmaxf(part, lgl.y);
    if (lq > 2) part = fmaxf(part, lgl.z);
    mlt = fmaxf(mlt, part);
#pragma unroll
    for (int d = 1; d < RF_SUB; d <<= 1) {
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
      mlt = fmaxf(mlt, __shfl_xor_sync(0xffffffffu, mlt, d));
    }
    // hand the result to the owner lane (lanes 4r .. 4r+3 own the samples of this round); every lane of a sample holds the same triple
    const int from = (lane & (RF_SPW - 1)) * RF_SUB;
    const float tm = __shfl_sync(0xffffffffu, mx, from);
    const float tlt = __shfl_sync(0xffffffffu, mlt, from);
    const float tlab = __shfl_sync(0xffffffffu, llab, from);
    if ((lane / RF_SPW) == r) { o_max = tm; o_maxlt = tlt; o_llab = tlab; }
  }
}

// generic form for more than 128 classes (NT > 4): one float4 group per trip, no unrolling
template <bool STAGED>
__device__ __noinline__ void rf_class_phase_loop(const RfTile& tl, float ix, float iy, int H, int W, int ld, int ncls, int cg4, int l4, int lq,
                                                 int lane, int n_rounds, float& o_max, float& o_maxlt, float& o_llab) {
  const int sub = lane & (RF_SUB - 1), slot = lane / RF_SUB;
  const int l_sub = l4 & (RF_SUB - 1);
#pragma unroll 1
  for (int r = 0; r < n_rounds; ++r) {
    const int src = RF_SPW * r + slot;
    const float sxi = __shfl_sync(0xffffffffu, ix, src), syi = __shfl_sync(0xffffffffu, iy, src);
    const float x0f = floorf(sxi), y0f = floorf(syi);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float ex = __fsub_rn(__fadd_rn(x0f, 1.f), sxi), wx = __fsub_rn(sxi, x0f);
    const float ey = __fsub_rn(__fadd_rn(y0f, 1.f), syi), wy = __fsub_rn(syi, y0f);
    const float w00 = __fmul_rn(ex, ey), w01 = __fmul_rn(wx, ey), w10 = __fmul_rn(ex, wy), w11 = __fmul_rn(wx, wy);
    const int r0 = (y0 - tl.oy) * tl.pitch - tl.ox, r1 = (y1 - tl.oy) * tl.pitch - tl.ox;
    const int c00 = (r0 + x0) * ld, c01 = (r0 + x1) * ld, c10 = (r1 + x0) * ld, c11 = (r1 + x1) * ld;
    float mx = -CUDART_INF_F, mlt = -CUDART_INF_F, llab = 0.f;
#pragma unroll 1
    for (int c4 = sub; c4 < cg4; c4 += RF_SUB) {
      float4 q0, q1, q2, q3;
      if (STAGED) {
        q0 = lds_tap(tl.sbase + 4u * (uint32_t)(c00 + 4 * c4)); q1 = lds_tap(tl.sbase + 4u * (uint32_t)(c01 + 4 * c4));
        q2 = lds_tap(tl.sbase + 4u * (uint32_t)(c10 + 4 * c4)); q3 = lds_tap(tl.sbase + 4u * (uint32_t)(c11 + 4 * c4));
      } else {
        q0 = ld_tap(tl.gbase + (size_t)c00 + 4 * c4); q1 = ld_tap(tl.gbase + (size_t)c01 + 4 * c4);
        q2 = ld_tap(tl.gbase + (size_t)c10 + 4 * c4); q3 = ld_tap(tl.gbase + (size_t)c11 + 4 * c4);
      }
      const float4 lg4 = bilerp4(q0, q1, q2, q3, w00, w01, w10, w11);
      float lg[4] = {lg4.x, lg4.y, lg4.z, lg4.w};
#pragma unroll
      for (int q = 1; q < 4; ++q)
        if (4 * c4 + q >= ncls) lg[q] = -CUDART_INF_F;
      const float m4 = fmaxf(fmaxf(lg[0], lg[1]), fmaxf(lg[2], lg[3]));
      mx = fmaxf(mx, m4);
      if (c4 < l4) mlt = fmaxf(mlt, m4);
      else if (c4 == l4) {
        llab = lq == 0 ? lg[0] : lq == 1 ? lg[1] : lq == 2 ? lg[2] : lg[3];
        float part = -CUDART_INF_F;
        if (lq > 0) part = lg[0];
        if (lq > 1) part = fmaxf(part, lg[1]);
        if (lq > 2) part = fmaxf(part, lg[2]);
        mlt = fmaxf(mlt, part);
      }
    }
#pragma unroll
    for (int d = 1; d < RF_SUB; d <<= 1) {
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
      mlt = fmaxf(mlt, __shfl_xor_sync(0xffffffffu, mlt, d));
    }
    const int from = (lane & (RF_SPW - 1)) * RF_SUB;
    const float tm = __shfl_sync(0xffffffffu, mx, from);
    const float tlt = __shfl_sync(0xffffffffu, mlt, from);
    const float tlab = __shfl_sync(0xffffffffu, llab, from + l_sub);
    if ((lane / RF_SPW) == r) { o_max = tm; o_maxlt = tlt; o_llab = tlab; }
  }
}

template <bool STAGED>
__device__ __forceinline__ void rf_class_phase_nt(int nt, const RfTile& tl, float ix, float iy, int H, int W, int ld, int ncls, int cg4, int l4,
                                                  int lq, int lane, int n_rounds, float& o_max, float& o_maxlt, float& o_llab) {
  const bool fast = (ncls & 3) == 0 && nt <= 4;         // CTA-uniform
  if (fast && nt == 3) rf_class_phase<STAGED, 3>(tl, ix, iy, H, W, ld, cg4, l4, lq, lane, n_rounds, o_max, o_maxlt, o_llab);      // 68..96 classes
  else if (fast && nt == 1) rf_class_phase<STAGED, 1>(tl, ix, iy, H, W, ld, cg4, l4, lq, lane, n_rounds, o_max, o_maxlt, o_llab);
  else if (fast && nt == 2) rf_class_phase<STAGED, 2>(tl, ix, iy, H, W, ld, cg4, l4, lq, lane, n_rounds, o_max, o_maxlt, o_llab);
  else if (fast && nt == 4) rf_class_phase<STAGED, 4>(tl, ix, iy, H, W, ld, cg4, l4, lq, lane, n_rounds, o_max, o_maxlt, o_llab);
  else rf_class_phase_loop<STAGED>(tl, ix, iy, H, W, ld, ncls, cg4, l4, lq, lane, n_rounds, o_max, o_maxlt, o_llab);
}

__global__ void __launch_bounds__(320, 2)
refine_fused_kernel(const __grid_constant__ CUtensorMap tm_map, int use_tma, int WS, float reach_px,
                    const float* __restrict__ lmap, int H, int W, int ncls, int ld, const float* __restrict__ centers,
                    const int32_t* __restrict__ labels, const int32_t* __restrict__ bag_img,
                    const float* __restrict__ offsets, int K, float stride, const int32_t* __restrict__ pad_hw,
                    const int32_t* __restrict__ img_hw, const int32_t* __restrict__ grp_of,
                    const int32_t* __restrict__ grp_ptr, const int32_t* __restrict__ grp_idx,
                    const uint8_t* __restrict__ not_refine_in, ptb_refine_cfg cfg, float* __restrict__ out_pts,
                    float* __restrict__ out_score, uint8_t* __restrict__ out_not_refine, uint8_t* __restrict__ out_chosen) {
  extern __shared__ uint8_t sm_raw[];
  // layout: [window (128 B aligned, only when use_tma)] [pm, sx, sy, pl : K floats each] [mk : K bytes] ; barrier in static smem
  const uint32_t raw = smem_u32(sm_raw);
  const uint32_t win = use_tma ? ((raw + 127u) & ~127u) : raw;      // (no window, no slack bytes: do not shift the arrays)
  const size_t win_bytes = use_tma ? (size_t)WS * WS * ld * sizeof(float) : 0;
  float* pm = reinterpret_cast<float*>(sm_raw + (win - raw) + win_bytes);
  float* sx = pm + K;
  float* sy = pm + 2 * K;
  float* pl = pm + 3 * K;     // prob of the GT label per sample (thresholds need the centre's first)
  uint8_t* mk = reinterpret_cast<uint8_t*>(pm + 4 * K);   // partial mask per sample
  __shared__ float red[3 * RF_MAXWARPS];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_staged, s_ox, s_oy;
  __shared__ float s_gcx[RF_GCAP], s_gcy[RF_GCAP];     // centres (+ centre offset) of the same-(image,label) GTs: nearest filter
  __shared__ int s_gid[RF_GCAP];
  const int g = blockIdx.x;
  const int l = labels[g], b = bag_img[g];
  const float ih = (float)img_hw[2 * b], iw = (float)img_hw[2 * b + 1];
  const float ph = (float)pad_hw[2 * b], pw = (float)pad_hw[2 * b + 1];
  const int gi = grp_of[g];
  const int m0 = grp_ptr[gi], t = grp_ptr[gi + 1] - m0;
  const bool use_mm = ((long long)t * K > 25) || (t > 25);
  const float cxg = centers[2 * g], cyg = centers[2 * g + 1];
  const float ox_last = offsets[2 * (K - 1)], oy_last = offsets[2 * (K - 1) + 1];
  const int cg4 = (ncls + 3) >> 2;
  const int nt = (cg4 + RF_SUB - 1) / RF_SUB;          // float4 class groups per lane of the class phase
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int l4 = l >> 2, lq = l & 3;                  // float4 / component that holds the label's logit
  const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
  const uint32_t bar = smem_u32(&s_bar);

  if (threadIdx.x == 0) {
    int staged = 0, ox = 0, oy = 0;
    if (use_tma) {
      // extreme taps of the bag: every sample's coordinate lies in [c - reach, c + reach] and the pipeline is monotone
      const float xl = sample_coord(__fadd_rn(-reach_px, cxg), stride, (float)W, hw), xr = sample_coord(__fadd_rn(reach_px, cxg), stride, (float)W, hw);
      const float yl = sample_coord(__fadd_rn(-reach_px, cyg), stride, (float)H, hh), yr = sample_coord(__fadd_rn(reach_px, cyg), stride, (float)H, hh);
      ox = (int)floorf(xl); oy = (int)floorf(yl);
      const int x_hi = min((int)floorf(xr) + 1, W - 1), y_hi = min((int)floorf(yr) + 1, H - 1);
      staged = (x_hi - ox + 1 <= WS) && (y_hi - oy + 1 <= WS);
      if (staged) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(bar, (uint32_t)win_bytes);
        tma_load_4d(&tm_map, bar, win, 0, ox, oy, b);
      }
    }
    s_staged = staged; s_ox = ox; s_oy = oy;
  }
  if ((cfg.flags & 1) && t > 1) {        // one independent global load per member instead of a dependent chain per sample
    for (int j = threadIdx.x; j < min(t, RF_GCAP); j += blockDim.x) {
      const int gj = grp_idx[m0 + j];
      s_gid[j] = gj;
      s_gcx[j] = __fadd_rn(ox_last, centers[2 * gj]);
      s_gcy[j] = __fadd_rn(oy_last, centers[2 * gj + 1]);
    }
  }
  __syncthreads();
  const bool staged = s_staged != 0;
  RfTile tl;
  tl.gbase = lmap + (size_t)b * H * W * ld;
  tl.sbase = win;
  tl.pitch = staged ? WS : W;
  tl.ox = staged ? s_ox : 0;
  tl.oy = staged ? s_oy : 0;
  bool waited = false;

  for (int s0 = warp * 32; s0 < K; s0 += nwarps * 32) {              // warp-uniform trip count
    // ---- owner phase 1 (map independent, runs under the TMA load): lane = sample
    const bool act = s0 + lane < K;
    const int s = act ? s0 + lane : K - 1;                            // idle lanes shadow the centre sample
    const float px = __fadd_rn(offsets[2 * s], cxg), py = __fadd_rn(offsets[2 * s + 1], cyg);
    const float ix = sample_coord(px, stride, (float)W, hw), iy = sample_coord(py, stride, (float)H, hh);
    bool m = (0.f <= px) && (px < pw) && (0.f <= py) && (py < ph);   // bag_valid (cpr_head.py:179)
    if ((cfg.flags & 1) && t > 1) {
      // nearest filter (cpr_head.py:711-743): candidates = same-(image,label) GT centres in ascending GT order
      const float pn = sq_norm2(px, py);
      float bd = CUDART_INF_F;
      int bj = -1;
      for (int j = 0; j < t; ++j) {                                    // t is CTA-uniform
        int gj;
        float cx, cy;
        if (j < RF_GCAP) { gj = s_gid[j]; cx = s_gcx[j]; cy = s_gcy[j]; }
        else { gj = grp_idx[m0 + j]; cx = __fadd_rn(ox_last, centers[2 * gj]); cy = __fadd_rn(oy_last, centers[2 * gj + 1]); }
        const float d = use_mm ? cdist_mm(px, py, pn, cx, cy, sq_norm2(cx, cy)) : cdist_direct(px, py, cx, cy);
        if (d < bd) { bd = d; bj = gj; }
      }
      m = m && (bj == g);
    }
    m = m && (px < iw) && (px >= 0.f) && (py < ih) && (py >= 0.f);
    // ---- class phase
    if (staged && !waited) { mbar_wait(bar, 0u); waited = true; }
    float v_max = 0.f, v_maxlt = 0.f, v_llab = 0.f;
    const int n_rounds = (min(32, K - s0) + RF_SPW - 1) / RF_SPW;
    if (staged) rf_class_phase_nt<true>(nt, tl, ix, iy, H, W, ld, ncls, cg4, l4, lq, lane, n_rounds, v_max, v_maxlt, v_llab);
    else rf_class_phase_nt<false>(nt, tl, ix, iy, H, W, ld, ncls, cg4, l4, lq, lane, n_rounds, v_max, v_maxlt, v_llab);
    // ---- owner phase 2: three sigmoids per sample
    const float p_label = sigmoidf_acc(v_llab);
    if (cfg.flags & 2) {
      bool first = p_label >= sigmoidf_acc(v_max);
      if (first && v_maxlt > -CUDART_INF_F) first = p_label > sigmoidf_acc(v_maxlt);
      m = m && first;
    }
    if (act) { pl[s] = p_label; mk[s] = m; sx[s] = px; sy[s] = py; }
  }
  __syncthreads();
  const float pg_a = __fmul_rn(pl[K - 1], cfg.gt_alpha);
  for (int s = threadIdx.x; s < K; s += blockDim.x) {
    const float p = pl[s];
    const bool m = mk[s] && (p > cfg.merge_th) && (p > pg_a);
    pm[s] = m ? p : 0.f;
  }
  __syncthreads();
  refine_tail(pm, sx, sy, K, sx[K - 1], sy[K - 1], not_refine_in, g, cfg, red, out_pts, out_score, out_not_refine, out_chosen);
}

// ------------------------------------------------------------------------------------------------
// same-(image,label) GT groups as CSR — the device-side group_by_label (cpr_head.py:64-70 does labels.cpu()).
// One CTA per image: a stable counting sort by label (members of a group stay in ascending GT order); groups are numbered
// image-major, label-minor, so CTA b first counts the distinct labels of images 0..b-1 (a few thousand labels: cheaper than
// a second launch or a grid-wide scan).  Deterministic: no cross-CTA communication at all.
// ------------------------------------------------------------------------------------------------
constexpr int LG_THREADS = 512;
constexpr int LG_MAX_N = 8192;       // GTs per image held in shared memory
constexpr int LG_MAX_C = 1024;

__global__ void __launch_bounds__(LG_THREADS)
label_groups_kernel(const int32_t* __restrict__ labels, const int32_t* __restrict__ img_ptr, int B, int G, int C,
                    int32_t* __restrict__ grp_of, int32_t* __restrict__ grp_ptr, int32_t* __restrict__ grp_idx) {
  __shared__ int s_lab[LG_MAX_N];
  __shared__ int s_cnt[LG_MAX_C], s_start[LG_MAX_C], s_rank[LG_MAX_C];
  __shared__ int s_groups, s_base;
  const int tid = threadIdx.x;
  const int b = blockIdx.x;
  if (tid == 0) s_base = 0;
  __syncthreads();          // (racecheck, round 2: image 0 runs no iteration of the loop below, so nothing ordered this write before the read)
  // distinct labels of the images before this one
  for (int pb = 0; pb < b; ++pb) {
    const int q0 = img_ptr[pb], qn = img_ptr[pb + 1] - q0;
    for (int c = tid; c < C; c += LG_THREADS) s_cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < qn; i += LG_THREADS) s_cnt[labels[q0 + i]] = 1;       // benign same-value race
    __syncthreads();
    int mine = 0;
    for (int c = tid; c < C; c += LG_THREADS) mine += s_cnt[c];
    mine = warp_sum_int(mine);
    if ((tid & 31) == 0 && mine) atomicAdd(&s_base, mine);                      // integer sum: order-independent
    __syncthreads();
  }
  const int group_base = s_base;
  const int g0 = img_ptr[b], n = img_ptr[b + 1] - g0;
  for (int c = tid; c < C; c += LG_THREADS) s_cnt[c] = 0;
  __syncthreads();
  for (int i = tid; i < n; i += LG_THREADS) {
    const int l = labels[g0 + i];
    s_lab[i] = l;
    atomicAdd(&s_cnt[l], 1);
  }
  __syncthreads();
  if (tid == 0) {           // C <= 1024: serial exclusive scans are negligible
    int run = 0, ng = 0;
    for (int c = 0; c < C; ++c) {
      s_start[c] = run;
      s_rank[c] = ng;
      if (s_cnt[c] > 0) {
        grp_ptr[group_base + ng] = g0 + run;
        ++ng;
      }
      run += s_cnt[c];
    }
    s_groups = ng;
  }
  __syncthreads();
  for (int i = tid; i < n; i += LG_THREADS) {
    const int l = s_lab[i];
    int before = 0;
    for (int j = 0; j < i; ++j) before += (s_lab[j] == l);      // stable rank inside the label
    grp_idx[g0 + s_start[l] + before] = g0 + i;
    grp_of[g0 + i] = group_base + s_rank[l];
  }
  if (b == B - 1)
    for (int k = group_base + s_groups + tid; k <= G; k += LG_THREADS) grp_ptr[k] = G;   // closing entry (+ unused tail)
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_cpr_refine(const float* bag_prob, const float* bag_pts, const uint8_t* bag_valid, int G, int Kt, int K,
                              int num_classes, const int32_t* labels, const int32_t* bag_img, const int32_t* img_hw,
                              const int32_t* grp_of, const int32_t* grp_ptr, const int32_t* grp_idx,
                              const uint8_t* not_refine_in, ptb_refine_cfg cfg, float* out_pts, float* out_score,
                              uint8_t* out_not_refine, uint8_t* out_chosen, uint8_t* out_merge_valid, void* stream) {
  PTB_REQUIRE(G >= 0 && Kt > 0 && K > 0 && Kt % K == 0 && num_classes > 0, "shape");
  if (G == 0) return 0;
  PTB_REQUIRE(bag_prob && bag_pts && bag_valid && labels && bag_img && img_hw && grp_of && grp_ptr && grp_idx, "NULL input");
  PTB_REQUIRE(out_pts && out_score && out_not_refine, "NULL output");
  const size_t smem = (size_t)3 * Kt * sizeof(float);
  PTB_REQUIRE(smem <= 48 * 1024, "bag too large for shared memory");
  if (smem > 40 * 1024 &&     // static (384 B) + dynamic beyond the 48 KB default needs the opt-in; per-device attribute -> per call
      cudaFuncSetAttribute(refine_stage_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("%s", "ptb_cpr_refine: shared memory opt-in failed");
  refine_stage_kernel<<<G, RF_THREADS, smem, (cudaStream_t)stream>>>(bag_prob, bag_pts, bag_valid, Kt, K, num_classes, labels,
                                                                   bag_img, img_hw, grp_of, grp_ptr, grp_idx, not_refine_in,
                                                                   cfg, out_pts, out_score, out_not_refine, out_chosen,
                                                                   out_merge_valid);
  return check_launch("ptb_cpr_refine");
}

extern "C" int ptb_cpr_refine_fused(const float* logit_map, int B, int H, int W, int num_classes, int ld, const float* centers,
                                    const int32_t* labels, const int32_t* bag_img, int G, const float* offsets, int K,
                                    float stride, float reach_px, const int32_t* pad_hw, const int32_t* img_hw, const int32_t* grp_of,
                                    const int32_t* grp_ptr, const int32_t* grp_idx, const uint8_t* not_refine_in,
                                    ptb_refine_cfg cfg, float* out_pts, float* out_score, uint8_t* out_not_refine,
                                    uint8_t* out_chosen, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && G >= 0 && K > 0 && num_classes > 0 && stride > 0.f, "shape");
  PTB_REQUIRE(ld % 4 == 0 && ld >= ((num_classes + 3) / 4) * 4, "ld must be a multiple of 4 covering num_classes");
  PTB_REQUIRE((uintptr_t)logit_map % 16 == 0, "logit_map must be 16-byte aligned");
  if (G == 0) return 0;
  PTB_REQUIRE(logit_map && centers && labels && bag_img && offsets && pad_hw && img_hw && grp_of && grp_ptr && grp_idx,
              "NULL input");
  PTB_REQUIRE(out_pts && out_score && out_not_refine, "NULL output");
  const size_t tail = (size_t)4 * K * sizeof(float) + (size_t)((K + 15) / 16) * 16;
  PTB_REQUIRE(tail <= 48 * 1024, "bag too large for shared memory");
  int warps = (K + 31) / 32;              // a warp takes 32 samples per pass
  if (warps < 2) warps = 2;
  if (warps > 10) warps = 10;             // 320 threads x 2 CTAs per SM; larger bags take several passes per warp
  const int threads = warps * 32;
  // ---- TMA staging of the bag's logit tile: window of 2*ceil(reach/stride) + 2 cells; PTB_REFINE_TMA=0 forces the global path
  int use_tma = 0, WS = 0;
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  const char* e_tma = getenv("PTB_REFINE_TMA");        // read per call: tools/profile_refine.py times both paths in one process
  const int tma_mode = (e_tma && e_tma[0] == '0') ? 0 : 1;
  if (tma_mode && reach_px > 0.f && ld <= 256) {
    WS = 2 * (int)ceilf(reach_px / stride) + 2;
    const size_t win_bytes = (size_t)WS * WS * ld * sizeof(float);
    // two CTAs per SM must fit (227 KB usable, 1 KB reserved per CTA): otherwise the load of one bag cannot hide behind another's math
    if (WS <= 256 && win_bytes + tail + 128 <= 112 * 1024) {
      EncodeTiledFn enc = tc_get_encode();
      if (enc) {
        cuuint64_t dims[4] = {(cuuint64_t)ld, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
        cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4};
        cuuint32_t box[4] = {(cuuint32_t)ld, (cuuint32_t)WS, (cuuint32_t)WS, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(logit_map), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS)
          use_tma = 1;
      }
    }
  }
  const size_t smem = tail + (use_tma ? (size_t)WS * WS * ld * sizeof(float) + 128 : 0);
  if (smem > 40 * 1024 &&     // static (3.2 KB) + dynamic beyond the 48 KB default needs the opt-in; per-device attribute -> per call
      cudaFuncSetAttribute(refine_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return fail("%s", "ptb_cpr_refine_fused: shared memory opt-in failed");
  refine_fused_kernel<<<G, threads, smem, (cudaStream_t)stream>>>(tm, use_tma, WS, reach_px, logit_map, H, W, num_classes, ld, centers,
                                                                   labels, bag_img, offsets, K, stride, pad_hw, img_hw, grp_of,
                                                                   grp_ptr, grp_idx, not_refine_in, cfg, out_pts, out_score,
                                                                   out_not_refine, out_chosen);
  return check_launch("ptb_cpr_refine_fused");
}

extern "C" int ptb_label_groups(const int32_t* labels, const int32_t* img_ptr, int B, int G, int num_classes, int max_per_image,
                                int32_t* grp_of, int32_t* grp_ptr, int32_t* grp_idx, void* stream) {
  PTB_REQUIRE(B > 0 && G >= 0 && num_classes > 0, "shape");
  PTB_REQUIRE(num_classes <= LG_MAX_C, "num_classes > 1024 not supported");
  PTB_REQUIRE(max_per_image <= LG_MAX_N, "more than 8192 GT points per image not supported");
  PTB_REQUIRE(img_ptr && grp_ptr && (G == 0 || (labels && grp_of && grp_idx)), "NULL input");
  label_groups_kernel<<<B, LG_THREADS, 0, (cudaStream_t)stream>>>(labels, img_ptr, B, G, num_classes, grp_of, grp_ptr, grp_idx);
  return check_launch("ptb_label_groups");
}
