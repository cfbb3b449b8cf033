// Test-time augmentation and tile testing of the two-stage detector (TwoStageDetector.tile_aug_test, StandardRoIHead.aug_test):
//   box_map_kernel        bbox_mapping (core/bbox/transforms.py): * scale_factor, flip, tile shift + clamp + keep mask, per RoI row.
//   aug_merge_kernel      bbox_mapping_back of every aug, then merge_aug_bboxes' torch.stack(...).mean(0) over the augs of a tile, in
//                         ATen's CPU summation order (see aten_mean).
//   batched_nms_kernel    mmcv batched_nms / nms for up to 65536 rows per segment, one CTA per segment, no kept-count cap.
//   tile_concat_kernel    each tile's detections: * scale_factor, + tile offset, rows in bbox2result's class-major order.
#include "ptb_common.cuh"

namespace ptb {
namespace {

constexpr int TT_META = 12;         // per-aug meta row: seg, roi batch, sf[4], flip, img_h, img_w, has_off, dx, dy
constexpr int BNMS_T = 1024;        // threads of the NMS CTA = candidates per greedy block
constexpr int BNMS_SORT_CHUNK = 8192;   // keys sorted in shared memory at once
constexpr int BNMS_MAX_ROWS = 65536;

struct NBox {
  Box b;
  int label;
};

// from split_thr rows on (mmcv's class-by-class branch) only boxes of one label suppress each other
__device__ __forceinline__ bool nbox_suppresses(const NBox& a, const NBox& b, float thr, bool split) {
  return (!split || a.label == b.label) && iou_gt(a.b, b.b, thr);
}

// bbox_flip of one (x1, y1, x2, y2) group: h / w are the img_shape the flip uses
__device__ __forceinline__ void flip4(float* o, int dir, float h, float w) {
  const float x1 = o[0], y1 = o[1], x2 = o[2], y2 = o[3];
  if (dir == 1 || dir == 3) { o[0] = __fsub_rn(w, x2); o[2] = __fsub_rn(w, x1); }
  if (dir == 2 || dir == 3) { o[1] = __fsub_rn(h, y2); o[3] = __fsub_rn(h, y1); }
}

// row r of aug g: proposals[seg][r] * sf, flipped, shifted by -offset and clamped to [0, w-1] x [0, h-1]; keep = W >= 2 & H >= 2
__global__ void box_map_kernel(const float* __restrict__ boxes, int ld, const int32_t* __restrict__ counts, int N, int G,
                               const float* __restrict__ meta, float* __restrict__ rois, uint8_t* __restrict__ keep) {
  const long long total = (long long)G * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i / N), r = (int)(i % N);
    const float* m = meta + (size_t)g * TT_META;
    const int seg = (int)m[0];
    float* out = rois + 5 * i;
    const bool valid = r < (counts ? counts[seg] : N);
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    bool k = false;
    if (valid) {
      const float* b = boxes + ((size_t)seg * N + r) * ld;
#pragma unroll
      for (int c = 0; c < 4; ++c) o[c] = __fmul_rn(b[c], m[2 + c]);
      flip4(o, (int)m[6], m[7], m[8]);
      k = true;
      if (m[9] != 0.f) {
        const float dx = m[10], dy = m[11], wm = __fsub_rn(m[8], 1.f), hm = __fsub_rn(m[7], 1.f);
        o[0] = fminf(fmaxf(__fsub_rn(o[0], dx), 0.f), wm); o[2] = fminf(fmaxf(__fsub_rn(o[2], dx), 0.f), wm);
        o[1] = fminf(fmaxf(__fsub_rn(o[1], dy), 0.f), hm); o[3] = fminf(fmaxf(__fsub_rn(o[3], dy), 0.f), hm);
        k = __fsub_rn(o[2], o[0]) >= 2.f && __fsub_rn(o[3], o[1]) >= 2.f;
      }
    }
    out[0] = m[1];
#pragma unroll
    for (int c = 0; c < 4; ++c) out[1 + c] = o[c];
    if (keep) keep[i] = k;
  }
}

// merge_aug_proposals' recovery: bbox_mapping_back of the first counts[g] proposals (box, score) of every aug g = t * A + a, the augs of
// tile t concatenated in order into out [T][A*N][5]; out_count[t] = their number
__global__ void proposal_map_back_kernel(const float* __restrict__ det, const int32_t* __restrict__ counts, int N, int T, int A,
                                         const float* __restrict__ meta, float* __restrict__ out, int32_t* __restrict__ out_count) {
  const long long total = (long long)T * A * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i / N), r = (int)(i % N), t = g / A, a = g % A;
    int base = 0;
    for (int u = t * A; u < g; ++u) base += min(max(counts[u], 0), N);
    const int n = min(max(counts[g], 0), N);
    if (a == A - 1 && r == 0) out_count[t] = base + n;
    if (r >= n) continue;
    const float* m = meta + (size_t)g * TT_META;
    const float* d = det + ((size_t)g * N + r) * 5;
    float o[4] = {d[0], d[1], d[2], d[3]};
    flip4(o, (int)m[6], m[7], m[8]);
    float* y = out + ((size_t)t * A * N + base + r) * 5;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      y[k] = __fdiv_rn(o[k], m[2 + k]);
      if (m[9] != 0.f) y[k] = __fadd_rn(y[k], (k & 1) ? m[11] : m[10]);
    }
    y[4] = d[4];
  }
}

// torch.stack(x_0..x_{A-1}).mean(0) on the CPU: the stack is reduced over dim 0 with its other dims flattened to M columns.  ATen's
// cascade_sum sums the first floor(M / 32) * 32 columns row by row from 0 (four levels folding every 16 rows), and every later column
// with row_sum: partial sums p_k over rows 4i + k (i < A / 4), the remaining rows added to p_0, then p_0 + p_1 + p_2 + p_3.  The sum is
// then divided by A.  A < 64 (row_sum's partials do not cascade below 16 blocks of 4).
template <class Load>
__device__ __forceinline__ float aten_mean(Load x, int A, bool vec_part) {
  float s;
  if (vec_part) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    int i = 0;
    for (; i + 16 <= A;) {
      for (int j = 0; j < 16; ++j, ++i) acc[0] = __fadd_rn(acc[0], x(i));
      for (int j = 1; j < 4; ++j) {
        acc[j] = __fadd_rn(acc[j], acc[j - 1]);
        acc[j - 1] = 0.f;
        if ((i & (15 << (4 * j))) != 0) break;
      }
    }
    for (; i < A; ++i) acc[0] = __fadd_rn(acc[0], x(i));
    s = __fadd_rn(__fadd_rn(__fadd_rn(acc[0], acc[1]), acc[2]), acc[3]);
  } else {
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    const int q = A / 4;
    for (int i = 0; i < q; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k) p[k] = __fadd_rn(p[k], x(4 * i + k));
    for (int i = 4 * q; i < A; ++i) p[0] = __fadd_rn(p[0], x(i));
    s = __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[1]), p[2]), p[3]);
  }
  return __fdiv_rn(s, (float)A);
}

// thread per (tile, row, class, coordinate) of the merged boxes and per (tile, row, class) of the merged scores.
// boxes [G][N][C][4] / scores [G][N][C] of roi_decode, G = T * A (tile-major); box_cols = the reference's 4 (class-agnostic) or 4C.
__global__ void aug_merge_kernel(const float* __restrict__ boxes, const float* __restrict__ scores, int N, int C, int box_cols,
                                 const int32_t* __restrict__ counts, int T, int A, const float* __restrict__ meta,
                                 float* __restrict__ out_boxes, float* __restrict__ out_scores) {
  const long long per_tile = (long long)N * C * 5, total = per_tile * T;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / per_tile);
    const long long e = i % per_tile;
    const int n = counts ? counts[t] : N;
    if (e < (long long)N * C) {               // score (row, class)
      const int r = (int)(e / C), c = (int)(e % C);
      float v = -INFINITY;                     // padding rows never pass a score threshold
      if (r < n) {
        const long long col = (long long)r * (C + 1) + c;          // the reference stacks (n, C + 1) scores
        const bool vp = col < ((long long)n * (C + 1) / 32) * 32;
        v = aten_mean([&](int a) { return scores[(((size_t)(t * A + a)) * N + r) * C + c]; }, A, vp);
      }
      out_scores[((size_t)t * N + r) * C + c] = v;
      continue;
    }
    const long long f = e - (long long)N * C;   // box (row, class, coordinate)
    const int r = (int)(f / (4 * C)), c = (int)((f / 4) % C), k = (int)(f % 4);
    float v = 0.f;
    if (r < n) {
      const int cc = box_cols == 4 ? 0 : c;
      const long long col = (long long)r * box_cols + 4 * cc + k;
      const bool vp = col < ((long long)n * box_cols / 32) * 32;
      v = aten_mean([&](int a) {
        const float* m = meta + (size_t)(t * A + a) * TT_META;
        float o[4];
        const float* b = boxes + ((((size_t)(t * A + a)) * N + r) * C + cc) * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = b[j];
        flip4(o, (int)m[6], m[7], m[8]);                            // bbox_mapping_back: flip, / scale_factor, + offset
        float y = __fdiv_rn(o[k], m[2 + k]);
        if (m[9] != 0.f) y = __fadd_rn(y, (k & 1) ? m[11] : m[10]);
        return y;
      }, A, vp);
    }
    out_boxes[(((size_t)t * N + r) * C + c) * 4 + k] = v;
  }
}

__device__ __forceinline__ unsigned long long nms_key(float s, int pos) {
  unsigned int u = __float_as_uint(s);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);      // ascending order of the scores
  return ((unsigned long long)(~u) << 32) | (unsigned int)pos;   // score descending, position ascending
}

__device__ __forceinline__ void bitonic_pass(unsigned long long* a, int lo_base, int n_pairs, int size, int stride) {
  for (int i = threadIdx.x; i < n_pairs; i += blockDim.x) {
    const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
    const bool up = (((lo + lo_base) & size) == 0);
    const unsigned long long x = a[lo], y = a[hi];
    if ((x > y) == up) { a[lo] = y; a[hi] = x; }
  }
}

// ascending bitonic sort of keys[0..n2) (n2 a power of two) by one CTA: every stride below a shared-memory chunk runs there
__device__ void sort_keys(unsigned long long* keys, int n2, unsigned long long* sm) {
  const int ch = n2 < BNMS_SORT_CHUNK ? n2 : BNMS_SORT_CHUNK;
  for (int size = ch; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride >= ch; stride >>= 1) {
      __syncthreads();
      bitonic_pass(keys, 0, n2 / 2, size, stride);
    }
    for (int base = 0; base < n2; base += ch) {
      __syncthreads();
      for (int i = threadIdx.x; i < ch; i += blockDim.x) sm[i] = keys[base + i];
      for (int sz = size == ch ? 2 : size; sz <= size; sz <<= 1)       // the first round sorts each chunk from size 2
        for (int st = min(sz, ch) >> 1; st > 0; st >>= 1) {
          __syncthreads();
          bitonic_pass(sm, base, ch / 2, sz, st);
        }
      __syncthreads();
      for (int i = threadIdx.x; i < ch; i += blockDim.x) keys[base + i] = sm[i];
    }
  }
  __syncthreads();
}

struct BnmsSmem {
  unsigned int mask[BNMS_T][BNMS_T / 32];   // survivor i suppresses survivor j > i
  NBox tile[BNMS_T];                        // kept boxes streamed from the workspace / the block's survivors
  NBox surv[BNMS_T];
  int surv_pos[BNMS_T];
  unsigned char kflag[BNMS_T];
  int wsum[BNMS_T / 32];
  float wmax[BNMS_T / 32];
  int n_keep;
};

// One CTA per segment.  Candidates are the first counts[s] rows; they are sorted by (score desc, position asc) and processed in blocks
// of BNMS_T: each candidate is tested against every box kept so far (streamed through shared memory), the block's survivors get a
// pairwise suppression mask, and one warp resolves the block greedily.  Labels given: coordinates offset by label * (max + 1) as mmcv
// batched_nms; from split_thr rows on only boxes of the same label suppress (its class-by-class branch; the kept rows sorted by score
// are exactly the greedy order here).  Output rows: the kept ones in that order, at most max_num (> 0).
__global__ void __launch_bounds__(BNMS_T, 1)
batched_nms_kernel(const float* __restrict__ boxes, int ld, const float* __restrict__ scores, int lds, const int32_t* __restrict__ labels,
                   const int32_t* __restrict__ counts, int N, int N2, float iou_thr, int split_thr, int max_num,
                   unsigned long long* __restrict__ keys_ws, NBox* __restrict__ kept_ws, int32_t* __restrict__ out_count,
                   float* __restrict__ out_det, int32_t* __restrict__ out_label, int32_t* __restrict__ out_keep) {
  extern __shared__ __align__(16) unsigned char smraw[];
  BnmsSmem& S = *reinterpret_cast<BnmsSmem*>(smraw);
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float* bx = boxes + (size_t)s * N * ld;
  const float* sc = scores + (size_t)s * N * lds;
  const int32_t* lb = labels ? labels + (size_t)s * N : nullptr;
  unsigned long long* keys = keys_ws + (size_t)s * N2;
  NBox* kept = kept_ws + (size_t)s * N;
  const int n = counts ? min(max(counts[s], 0), N) : N;
  // boxes.max() of batched_nms (the class offset unit)
  float mx = -INFINITY;
  if (lb)
    for (int i = tid; i < n; i += BNMS_T) mx = fmaxf(mx, fmaxf(fmaxf(bx[(size_t)i * ld], bx[(size_t)i * ld + 1]), fmaxf(bx[(size_t)i * ld + 2], bx[(size_t)i * ld + 3])));
  mx = warp_max(mx);
  if (lane == 0) S.wmax[wid] = mx;
  __syncthreads();
  mx = S.wmax[0];
  for (int w = 1; w < BNMS_T / 32; ++w) mx = fmaxf(mx, S.wmax[w]);
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int i = tid; i < n2; i += BNMS_T) keys[i] = i < n ? nms_key(sc[(size_t)i * lds], i) : ~0ull;
  __syncthreads();
  if (n > 1) sort_keys(keys, n2, reinterpret_cast<unsigned long long*>(&S.mask[0][0]));
  const float m1 = __fadd_rn(mx, 1.f);        // batched_nms: offsets = label * (boxes.max() + 1)
  const bool split = lb && n >= split_thr;
  const int cap = max_num > 0 ? min(max_num, n) : n;
  int n_kept = 0;
  for (int base = 0; base < n && n_kept < cap; base += BNMS_T) {
    const int i = base + tid;
    const bool have = i < n;
    const int pos = have ? (int)(keys[i] & 0xffffffffull) : 0;
    NBox me;
    {
      const float* b = bx + (size_t)pos * ld;
      me.label = lb && have ? lb[pos] : 0;
      const float off = lb ? __fmul_rn((float)me.label, m1) : 0.f;
      Box& q = me.b;
      q.x1 = __fadd_rn(b[0], off); q.y1 = __fadd_rn(b[1], off); q.x2 = __fadd_rn(b[2], off); q.y2 = __fadd_rn(b[3], off);
      q.area = __fmul_rn(__fsub_rn(q.x2, q.x1), __fsub_rn(q.y2, q.y1));
    }
    bool alive = have;
    for (int k0 = 0; k0 < n_kept; k0 += BNMS_T) {
      const int kn = min(BNMS_T, n_kept - k0);
      __syncthreads();
      if (tid < kn) S.tile[tid] = kept[k0 + tid];
      __syncthreads();
      if (alive)
        for (int t = 0; t < kn; ++t)
          if (nbox_suppresses(S.tile[t], me, iou_thr, split)) { alive = false; break; }
    }
    // survivors of the kept set, compacted in order
    const unsigned int bal = __ballot_sync(0xffffffffu, alive);
    if (lane == 0) S.wsum[wid] = __popc(bal);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < BNMS_T / 32; ++w) { const int v = S.wsum[w]; woff += w < wid ? v : 0; tot += v; }
    if (alive) {
      const int slot = woff + __popc(bal & ((1u << lane) - 1u));
      S.surv[slot] = me;
      S.surv_pos[slot] = pos;
    }
    __syncthreads();
    const int m = tot;
    if (tid < m) {
      const NBox a = S.surv[tid];
      for (int w = 0; w < BNMS_T / 32; ++w) {
        unsigned int bits = 0;
        const int j0 = 32 * w;
        if (j0 + 31 > tid && j0 < m)
          for (int j = max(j0, tid + 1); j < min(j0 + 32, m); ++j)
            if (nbox_suppresses(a, S.surv[j], iou_thr, split)) bits |= 1u << (j - j0);
        S.mask[tid][w] = bits;
      }
    }
    __syncthreads();
    if (wid == 0) {                       // greedy over the block's survivors: lane w holds removal word w
      unsigned int removed = 0;
      int nk = 0;
      for (int t = 0; t < m; ++t) {
        const unsigned int word = __shfl_sync(0xffffffffu, removed, t >> 5);
        const bool keep = !((word >> (t & 31)) & 1u) && n_kept + nk < cap;
        if (keep) { removed |= S.mask[t][lane]; ++nk; }
        if (lane == 0) S.kflag[t] = keep;
      }
      if (lane == 0) S.n_keep = nk;
    }
    __syncthreads();
    // append the block's kept rows in order
    const bool kf = tid < m && S.kflag[tid];
    const unsigned int kb = __ballot_sync(0xffffffffu, kf);
    __syncthreads();
    if (lane == 0) S.wsum[wid] = __popc(kb);
    __syncthreads();
    int koff = 0;
    for (int w = 0; w < wid; ++w) koff += S.wsum[w];
    if (kf) {
      const int o = n_kept + koff + __popc(kb & ((1u << lane) - 1u));
      const NBox a = S.surv[tid];
      const int p = S.surv_pos[tid];
      kept[o] = a;
      const float* b = bx + (size_t)p * ld;
      float* d = out_det + ((size_t)s * N + o) * 5;
      d[0] = b[0]; d[1] = b[1]; d[2] = b[2]; d[3] = b[3]; d[4] = sc[(size_t)p * lds];
      out_keep[(size_t)s * N + o] = p;
      if (out_label) out_label[(size_t)s * N + o] = a.label;
    }
    n_kept += S.n_keep;
    __syncthreads();
  }
  if (tid == 0) out_count[s] = n_kept;
}

// one CTA per tile: row k of tile t's NMS output goes to concat row tile_base + class_base(label) + rank within its class, with its box
// * scale_factor[t] (when given) and + (dx, dy) in fp32; out_count[0] = the number of rows
__global__ void tile_concat_kernel(const float* __restrict__ det, const int32_t* __restrict__ lab, const int32_t* __restrict__ cnt, int T,
                                   int K, const float* __restrict__ sf, const float* __restrict__ off, float* __restrict__ out,
                                   int32_t* __restrict__ out_label, int32_t* __restrict__ out_count) {
  const int t = blockIdx.x;
  int tile_base = 0;
  for (int u = 0; u < t; ++u) tile_base += min(max(cnt[u], 0), K);
  const int n = min(max(cnt[t], 0), K);
  if (t == T - 1 && threadIdx.x == 0) out_count[0] = tile_base + n;
  const int32_t* L = lab + (size_t)t * K;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int l = L[k];
    int r = 0;
    for (int j = 0; j < n; ++j) r += (L[j] < l) || (L[j] == l && j < k);
    const float* d = det + ((size_t)t * K + k) * 5;
    float* o = out + (size_t)(tile_base + r) * 5;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float v = sf ? __fmul_rn(d[c], sf[4 * t + c]) : d[c];
      o[c] = __fadd_rn(v, off[2 * t + (c & 1)]);
    }
    o[4] = d[4];
    out_label[tile_base + r] = l;
  }
}

}  // namespace
}  // namespace ptb

using namespace ptb;

extern "C" int ptb_box_map(const float* boxes, int ld, const int32_t* counts, int N, int G, const float* meta, float* rois, uint8_t* keep,
                           void* stream) {
  PTB_REQUIRE(ld >= 4 && N >= 0 && G >= 0, "ptb_box_map: arguments");
  if ((long long)G * N == 0) return 0;                  // no proposal: nothing to map (an empty tensor's pointer may be NULL)
  PTB_REQUIRE(boxes && meta && rois, "ptb_box_map: NULL argument");
  const long long total = (long long)G * N;
  box_map_kernel<<<(int)min((total + 255) / 256, 4096ll), 256, 0, (cudaStream_t)stream>>>(boxes, ld, counts, N, G, meta, rois, keep);
  return check_launch("ptb_box_map");
}

extern "C" int ptb_proposal_map_back(const float* det, const int32_t* counts, int N, int T, int A, const float* meta, float* out,
                                     int32_t* out_count, void* stream) {
  PTB_REQUIRE(det && counts && meta && out && out_count && N > 0 && T > 0 && A > 0, "ptb_proposal_map_back: arguments");
  const long long total = (long long)T * A * N;
  proposal_map_back_kernel<<<(int)min((total + 255) / 256, 4096ll), 256, 0, (cudaStream_t)stream>>>(det, counts, N, T, A, meta, out, out_count);
  return check_launch("ptb_proposal_map_back");
}

extern "C" int ptb_aug_merge(const float* boxes, const float* scores, int N, int num_classes, int box_cols, const int32_t* counts, int T,
                             int A, const float* meta, float* out_boxes, float* out_scores, void* stream) {
  PTB_REQUIRE(boxes && scores && meta && out_boxes && out_scores && num_classes > 0, "ptb_aug_merge: arguments");
  PTB_REQUIRE(box_cols == 4 || box_cols == 4 * num_classes, "ptb_aug_merge: box_cols must be 4 or 4 * num_classes");
  PTB_REQUIRE(A >= 1 && A <= 63, "ptb_aug_merge: 1 to 63 augs per tile");
  if ((long long)T * N == 0) return 0;
  const long long total = (long long)T * N * num_classes * 5;
  aug_merge_kernel<<<(int)min((total + 255) / 256, 8192ll), 256, 0, (cudaStream_t)stream>>>(boxes, scores, N, num_classes, box_cols, counts,
                                                                                          T, A, meta, out_boxes, out_scores);
  return check_launch("ptb_aug_merge");
}

extern "C" uint64_t ptb_batched_nms_workspace(int S, int N) {
  int n2 = 1;
  while (n2 < N) n2 <<= 1;
  return (uint64_t)S * n2 * sizeof(unsigned long long) + (uint64_t)S * N * sizeof(NBox);
}

extern "C" int ptb_batched_nms(const float* boxes, int ld, const float* scores, int lds, const int32_t* labels, const int32_t* counts, int S,
                               int N, float iou_thr, int split_thr, int max_num, int32_t* out_count, float* out_det, int32_t* out_label,
                               int32_t* out_keep, void* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(boxes && scores && out_count && out_det && out_keep && ld >= 4 && lds >= 1 && S >= 0 && N >= 0, "ptb_batched_nms: arguments");
  PTB_REQUIRE(N <= BNMS_MAX_ROWS, "ptb_batched_nms: more than 65536 rows per segment");
  if (S == 0) return 0;
  PTB_REQUIRE(workspace && workspace_bytes >= ptb_batched_nms_workspace(S, N), "ptb_batched_nms: workspace too small");
  int n2 = 1;
  while (n2 < N) n2 <<= 1;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(workspace);
  NBox* kept = reinterpret_cast<NBox*>(keys + (size_t)S * n2);
  const int smem = (int)sizeof(BnmsSmem);
  if (cudaFuncSetAttribute(batched_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return fail("%s", "ptb_batched_nms: shared memory opt-in failed");
  batched_nms_kernel<<<S, BNMS_T, smem, (cudaStream_t)stream>>>(boxes, ld, scores, lds, labels, counts, N, n2, iou_thr, split_thr, max_num,
                                                                keys, kept, out_count, out_det, out_label, out_keep);
  return check_launch("ptb_batched_nms");
}

extern "C" int ptb_tile_concat(const float* det, const int32_t* labels, const int32_t* counts, int T, int K, const float* scale_factor,
                               const float* offsets, float* out, int32_t* out_label, int32_t* out_count, void* stream) {
  PTB_REQUIRE(det && labels && counts && offsets && out && out_label && out_count && T > 0 && K > 0, "ptb_tile_concat: arguments");
  tile_concat_kernel<<<T, 256, 0, (cudaStream_t)stream>>>(det, labels, counts, T, K, scale_factor, offsets, out, out_label, out_count);
  return check_launch("ptb_tile_concat");
}
