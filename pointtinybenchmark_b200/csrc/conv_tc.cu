// Dense convolutions of the head on the Hopper tensor cores (wgmma + TMA + mbarrier), fp32-accurate by operand splitting:
// conv3x3 (stride 1, pad 1) and conv1x1 / per-cell Linear, Cin % 32 == 0 (fp16 mode) or Cin % 16 == 0 (TF32 mode), up to 512
// output channels (fp16 mode; 256 in TF32 mode and whenever GroupNorm statistics are requested), optional bias, optional
// GroupNorm statistics in the epilogue; GroupNorm-apply + ReLU + operand split runs either inside the conv kernel, in warps that
// are idle otherwise, as each image's statistics complete (GnFuse, ptb_conv3x3_c256_f16_gn: what the towers run), or as a second,
// HBM-bound kernel.  Replaces the cuDNN / cuBLAS calls behind CPRHead.forward_single / P2PHead.forward_single
// (cpr_head.py:1033-1043, p2p_head.py:113-123: 4 x ConvModule(conv3x3 + GN(32) + ReLU), 79.3 GFLOP per image), the
// per-sample cls_out / ins_out Linear of CPRHead.get_pts_outs (cpr_head.py:1045-1078, applied once per map cell here) and
// P2PHead's cls_out / reg_out conv3x3 (k * num_classes channels: 320 at the reference's default 4 anchors x 80 classes).
//
// Implicit GEMM:  M = output pixels (tile = 128 pixels of one image), N = output channels in slices of NT <= 128,
//                 K = taps x Cin.  One K-block = (tap, 64 B of input channels) = one SWIZZLE_64B row.
//   Outputs wider than 128 channels run as ceil(n_mma / 128) slices of 128 in ONE launch (2 at 256, 3 at 320, 4 at 512); the
//   persistent CTAs walk the (tile, slice) items, the weight TMA box of slice s starts at row 128 s (rows >= n_mma zero-filled).
//   * A operand: 4-D TMA box {64 B ch, tile w, tile h + 2, 1 img} of the channels-last activation at (h0 - 1, w0 + kw - 1): one
//     box serves the three vertical taps kh = 0, 1, 2 of column offset kw, as the same shared memory at + kh x tile w x 64 B (whole
//     512 B swizzle atoms for every tile shape, so the wgmma descriptors only move their start address).  A 1-tap conv loads the
//     tile itself.  Out-of-bounds (the zero padding of the conv and partial edge tiles) is zero-filled by the TMA unit.
//   * B operand: 2-D TMA box {64 B k, NT co} of the packed weights W2[co][tap*Cin + ci]; rows beyond n_mma are zero-filled.
//   * K order (9 taps): (kw, channel block, kh); one activation box (hi + lo) serves 3 K-blocks, each with its own weight box
//     (hi + lo) of tap (kh, kw).  That is 22.7 KB of TMA traffic per K-block instead of 32 KB with one box per tap.
//   * fp32 accuracy (the head's logits must match the fp32 reference to 1e-4).  Every operand is split x = hi + lo and three
//     MMAs per k-step accumulate hi*hi + lo*hi + hi*lo (the lo*lo term is below 2^-22 |a||b|):
//       F16 = true  (default): hi = fp16(x*s), lo = fp16(x*s - hi) with one power-of-two scale s per tensor (undone exactly in
//                    the epilogue), m64nNk16, 32 channels per K-block;
//       F16 = false: hi = x with the 13 low mantissa bits cleared (exact TF32), lo = x - hi (exact), m64n128k8 tf32, 16 channels
//                    per K-block (half the MMA rate).
//   * The tensor core adds into its fp32 accumulator without round-to-nearest, i.e. every accumulate step costs up to ~0.5 ulp of
//     the accumulator.  The two small correction products therefore go to their OWN accumulator (their error is 2^-11 smaller in
//     absolute terms); the epilogue adds the two in fp32 (round-to-nearest).
//   * warp roles (384 threads, 1 CTA / SM, persistent over (tile, channel slice) items): warpgroup 0 = TMA producer (one thread;
//     with GnFuse its warps 1-3 apply GroupNorm + ReLU to the CTA's finished items),
//     warpgroups 1 and 2 = MMA + epilogue for pixel rows 0-63 / 64-127 of the tile, each holding two 64 x NT fp32 accumulators in
//     registers (128 per thread at NT = 128).  Two mbarrier full / empty rings in shared memory: 4 x 24 KB activation boxes,
//     released after their last K-block, and 8 x 16 KB weight boxes, released after every K-block, so the weight loads of the
//     next K-blocks never wait for a whole activation box to retire.  The producer runs ahead into the next item while the MMA
//     warpgroups store the previous one.
//   * epilogue: straight from the accumulator registers (add, scale, bias) to global memory (8-byte stores, 32 contiguous bytes per
//     row and quad); GroupNorm sum / sum of squares per (image, group of 8 channels) by a halving butterfly over the 32 lanes of a
//     warp + one fp64 atomic per lane.
//   * half-precision activations (an autocast backbone's fp16 / bf16 feature map) are operand pairs already.  An fp16 tensor is its
//     own hi with lo == 0 and scale 1: A_LO_ZERO drops the lo * W_hi MMA (8 MMAs per K-block instead of 12) and the lo activation
//     box (half the activation TMA bytes); the ring keeps its layout, the lo half of a slot stays unused.  A bf16 tensor goes
//     through split_f16_from_bf16_kernel (2 B / element read) and the ordinary three-MMA kernel.  OutT = __half / __nv_bfloat16
//     stores the epilogue's fp32 value rounded to nearest even: the input gradient of such a tensor, in its dtype.
#include "tc_ptx.cuh"
#include <cuda_bf16.h>
#include <stdlib.h>
#include <type_traits>

namespace ptb {

constexpr int CV_N = 256;                       // output channels of the tower convolutions
constexpr int CV_N_MAX = 512;                   // widest output of ptb_conv_tc_f16x2 (4 slices of CV_NT)
constexpr int CV_BM = 128;                      // output pixels per tile
constexpr int CV_NT = 128;                      // widest output-channel slice of one item
constexpr int CV_KB = 16;                       // fp32/TF32 input channels per K-block (64 B = one SWIZZLE_64B row)
constexpr int CV_KB_F16 = 32;                   // fp16 input channels per K-block (also 64 B)
constexpr int CV_KH = 3;                        // K-blocks per activation box: the vertical taps kh = 0, 1, 2 share one box
constexpr int CV_A_STAGES = 4;                  // activation ring: 4 x 24 KB (hi + lo box)
constexpr int CV_B_STAGES = 8;                  // weight ring: 8 x 16 KB (hi + lo box of one K-block)
constexpr uint32_t CV_A_BYTES = (CV_BM + 2 * 32) * 64;      // 12 KB: the tallest box, (4 + 2) x 32 pixels (tile shape 1)
constexpr uint32_t CV_B_BYTES = CV_NT * 64;                 // 8 KB (a narrower slice uses the front of it)
constexpr uint32_t CV_A_STAGE_BYTES = 2 * CV_A_BYTES;       // 24 KB
constexpr uint32_t CV_B_STAGE_BYTES = 2 * CV_B_BYTES;       // 16 KB
constexpr uint32_t CV_RING_BYTES = CV_A_STAGES * CV_A_STAGE_BYTES + CV_B_STAGES * CV_B_STAGE_BYTES;   // 224 KB
constexpr uint32_t CV_SMEM_BYTES = CV_RING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(CV_SMEM_BYTES <= 227 * 1024, "the conv rings must fit the 227 KB of opt-in shared memory");
static_assert(2 * 8 * (CV_A_STAGES + CV_B_STAGES) + 8 <= 256, "the conv barriers and the item counter must fit their 256 B");
constexpr int CV_THREADS = 384;

// Output tiling.  A tile is always 128 pixels; the main region uses 8 x 16 tiles and the two edge strips that 8 x 16 tiles would
// cover half-empty get their own shapes: a bottom strip of <= 4 rows is covered by 4 x 32 tiles, a right strip of <= 8 columns by
// 16 x 8 tiles.  At the 100 x 168 map that is 132 tiles per image instead of 143 (13 x 11 with the last tile row and column half
// outside the image): 7.7 % fewer MMAs and loads for the same output.
//   shape 0: 8 h x 16 w (main)     shape 1: 4 h x 32 w (bottom strip, all columns)     shape 2: 16 h x 8 w (right strip, rows above the bottom strip)
struct ConvShape {
  int B, H, W, Cin;
  int tiles_h, tiles_w;   // main region, in 8 x 16 tiles
  int n_main, n_right, n_bottom, per_img, n_tiles;
  int right_w0, right_h;  // right strip: first column, number of rows it covers (rows below belong to the bottom strip)
  int bottom_h0;          // bottom strip: first row
  int n_slices;           // output-channel slices of NT channels per tile: item = tile * n_slices + slice
  int taps;       // 9: conv3x3 (pad 1), 1: conv1x1 / per-cell Linear
  int n_out;      // output channels actually stored
  int ldy;        // floats per output pixel row
};

struct ConvMaps {          // by-value __grid_constant__ kernel argument
  CUtensorMap x[3][2];     // activations (hi, lo) with the box of tile shape 0 / 1 / 2
  CUtensorMap w[2];        // packed weights (hi, lo); box rows = NT
};
struct TileAt {
  int b, h0, w0, shape, twl;     // image, origin, shape id, log2(tile width)
};
__device__ __forceinline__ TileAt tile_at(const ConvShape& cs, int tile) {
  TileAt t;
  t.b = tile / cs.per_img;
  const int r = tile - t.b * cs.per_img;
  if (r < cs.n_main) {
    t.shape = 0; t.twl = 4; t.h0 = (r / cs.tiles_w) * 8; t.w0 = (r % cs.tiles_w) * 16;
  } else if (r < cs.n_main + cs.n_right) {
    t.shape = 2; t.twl = 3; t.h0 = (r - cs.n_main) * 16; t.w0 = cs.right_w0;
  } else {
    t.shape = 1; t.twl = 5; t.h0 = cs.bottom_h0; t.w0 = (r - cs.n_main - cs.n_right) * 32;
  }
  return t;
}

// ---- GroupNorm + ReLU applied inside the conv kernel (GN != CV_GN_NONE) ----
// The statistics of image b are complete once every item of b has been stored by all 8 MMA warps of the CTA that computed it.  After
// its epilogue stores and statistics atomics an MMA warp only counts the item in shared memory (a CTA-scope release: no wait for its
// stores to reach L2).  Warp 1 publishes them: once the MMA warps have counted all of the CTA's items of image b it adds them to
// done[b] with a gpu-scope release, which makes those stores visible to the whole GPU (the release is cumulative) off the MMA warps'
// critical path.  Warps 1-3 of warpgroup 0 (idle besides the TMA producer thread) walk the CTA's own items behind the MMA
// warpgroups, wait for done[b] (gpu-scope acquire) and write
// relu(GroupNorm(y)) of the item's 128 pixels x 128 channels, read back through L2: while the tensor cores run image b + 1.  The MMA
// warps join the apply of the last image, which has nothing left to hide behind.  Only the wait crosses CTAs, so the launch is
// cooperative (every CTA resident).  The arithmetic is gn_relu_apply_f16_v8_kernel's (CV_GN_F16) or gn_relu_apply_kernel's
// (CV_GN_F32), element by element: the same bits.
constexpr int CV_GN_NONE = 0, CV_GN_F16 = 1, CV_GN_F32 = 2;
constexpr int CV_APPLY_WARPS = 3;                // warps 1-3 of warpgroup 0
constexpr int CV_MMA_WARPS = 8;
struct GnFuse {             // by-value kernel argument (unused when GN == CV_GN_NONE)
  const float* gamma;
  const float* beta;
  float eps;
  void* out;                // CV_GN_F16: __half h [B][H][W][256]; CV_GN_F32: float [B][H][W][256]
  __half* out_l;            // CV_GN_F16: __half l
  int* overflow_flag;       // optional, CV_GN_F16: raised when |GN output| > 60000 was clamped
  int* done;                // [B] (item, MMA warp) completions, zero on entry
};
constexpr uint32_t CV_CNT_OFFSET = 2 * 8 * (CV_A_STAGES + CV_B_STAGES);   // shared item counters of MMA warpgroups 1, 2 (4 B each)

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_cta_shared(uint32_t a) {
  int v;
  asm volatile("ld.acquire.cta.shared::cta.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_cta_shared_add(uint32_t a, int v) {
  asm volatile("red.release.cta.shared::cta.add.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
// lane 0 polls with backoff, then the warp proceeds (bounded: a protocol bug must not hang the GPU — trap after > 10 s)
__device__ __forceinline__ void wait_count(const int* p, int target, int lane) {
  if (lane == 0) {
    uint32_t ns = 32, polls = 0;
    while (ld_acquire_gpu(p) < target) {
      __nanosleep(ns);
      if (ns < 1024) ns <<= 1;
      if (++polls > (1u << 24)) __trap();
    }
  }
  __syncwarp();
}
// warp 1: publish this CTA's items of image b (item = its first one, last = the image's last item overall) to done[b], once the MMA
// warps have counted them in shared memory (cnt, cnt + 4: (item, warp) completions of MMA warpgroup 1 / 2, in the CTA's walk order;
// one counter per warpgroup, as the two may be an item apart)
__device__ __forceinline__ void publish_image(uint32_t cnt, int* done_b, int item, int last, int lane) {
  if (lane == 0) {
    const int n = (last - item) / (int)gridDim.x + 1;                          // the CTA's items of the image
    const int through = (item - (int)blockIdx.x) / (int)gridDim.x + n;         // CTA items up to and including the image's last
    uint32_t ns = 32, polls = 0;
    while (ld_acquire_cta_shared(cnt) < through * (CV_MMA_WARPS / 2) || ld_acquire_cta_shared(cnt + 4) < through * (CV_MMA_WARPS / 2)) {
      __nanosleep(ns);
      if (ns < 1024) ns <<= 1;
      if (++polls > (1u << 24)) __trap();
    }
    red_release_gpu_add(done_b, n * CV_MMA_WARPS);
  }
  __syncwarp();
}

// relu(GroupNorm(y)) of one item (128 pixels x 128 channels at n0) by member `member` of a team of `team` warps: lane L owns channels
// n0 + 4 L .. + 3 (one group of 8 per lane pair), a warp one pixel row (512 B of y) per step, four rows in flight.
template <int GN>
__device__ __forceinline__ void gn_apply_item(const ConvShape& cs, const GnFuse& gf, const float* __restrict__ y,
                                              const double* __restrict__ stats, int item, int member, int team, int lane,
                                              bool& clamped) {
  const int tile = item / cs.n_slices, n0 = (item - tile * cs.n_slices) * CV_NT;
  const TileAt ta = tile_at(cs, tile);
  const int c = n0 + 4 * lane, g = c >> 3;
  const int HW = cs.H * cs.W, cpg = CV_N / 32;
  const double inv_n = 1.0 / ((double)HW * cpg);
  const double s = __ldcg(stats + ((size_t)ta.b * 32 + g) * 2), ss = __ldcg(stats + ((size_t)ta.b * 32 + g) * 2 + 1);
  const double mean = s * inv_n;
  double var = ss * inv_n - mean * mean;
  var = var < 0.0 ? 0.0 : var;
  const float rstd = (float)(1.0 / sqrt(var + (double)gf.eps));
  const float mu = (float)mean;
  const float4 ga = __ldg(reinterpret_cast<const float4*>(gf.gamma + c)), be = __ldg(reinterpret_cast<const float4*>(gf.beta + c));
  const int h_end = ta.shape == 2 ? cs.right_h : cs.H;     // the epilogue's edge rules
  const int tw_mask = (1 << ta.twl) - 1;
  const size_t img = (size_t)ta.b * HW * CV_N + c;           // element offsets below are relative to (image b, channel c)
  const float* __restrict__ yb = y + img;
  constexpr int U = 4;
  for (int p0 = member; p0 < CV_BM; p0 += U * team) {
    float4 v[U];
    int at[U];                                                 // < H * W * 256 elements: one image
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = p0 + u * team;
      const int h = ta.h0 + (p >> ta.twl), w = ta.w0 + (p & tw_mask);
      at[u] = p < CV_BM && h < h_end && w < cs.W ? (h * cs.W + w) * CV_N : -1;
      if (at[u] >= 0) v[u] = __ldcg(reinterpret_cast<const float4*>(yb + at[u]));
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (at[u] < 0) continue;
      float o[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      o[0] = fmaf((o[0] - mu) * rstd, ga.x, be.x); o[1] = fmaf((o[1] - mu) * rstd, ga.y, be.y);
      o[2] = fmaf((o[2] - mu) * rstd, ga.z, be.z); o[3] = fmaf((o[3] - mu) * rstd, ga.w, be.w);
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
      if constexpr (GN == CV_GN_F16) {
        __align__(8) __half h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (fabsf(o[j]) > 60000.f) { o[j] = copysignf(60000.f, o[j]); clamped = true; }
          split_h2(o[j], h[j], l[j]);
        }
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(gf.out) + img + at[u]) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(gf.out_l + img + at[u]) = *reinterpret_cast<uint2*>(l);
      } else {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(gf.out) + img + at[u]) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// F16 = false: 3xTF32 (operands fp32 hi/lo).  F16 = true: 2-term fp16 split (x = h + l, 22 significant bits): h*h + l*h + h*l,
// the same three MMAs per k-step but K = 16 per MMA, i.e. half the tensor-pipe time and half the operand bytes.  out_scale undoes
// the power-of-two scaling of the fp16 operands (exact).  NT: output channels per item (16, 32, 64 or 128; 128 in TF32 mode).
// A_LO_ZERO: the activation's lo term is identically zero (an fp16 input): its box is not loaded and its MMA not issued; the result
// has the bits of the full kernel fed an explicit all-zero lo.  OutT: element type of y (float, or __half / __nv_bfloat16 rounded
// to nearest even from the same fp32 value; cs.ldy counts elements of OutT).
// GN: CV_GN_NONE, or GroupNorm + ReLU applied in the kernel (see GnFuse; fp16 mode, NT = 128, fp32 y, statistics on, no bias).
template <bool F16, int NT, bool A_LO_ZERO = false, typename OutT = float, int GN = CV_GN_NONE>
__global__ void __launch_bounds__(CV_THREADS, 1)
conv_tc_kernel(const __grid_constant__ ConvMaps mp, ConvShape cs, OutT* __restrict__ y, double* __restrict__ stats /*[B][32][2] or NULL*/,
               float out_scale, const float* __restrict__ dev_out_scale, const float* __restrict__ bias, GnFuse gf) {
  static_assert(F16 || NT == 128, "the TF32 mode runs 128-channel slices");
  static_assert(F16 || (!A_LO_ZERO && std::is_same<OutT, float>::value), "half-precision inputs and outputs belong to the fp16 mode");
  static_assert(GN == CV_GN_NONE || (F16 && NT == 128 && std::is_same<OutT, float>::value), "the fused GroupNorm apply runs on fp32 y, NT 128");
  constexpr int KBC = F16 ? CV_KB_F16 : CV_KB;      // channels per K-block
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;      // swizzle atoms need (at least) 512 B alignment
  const uint32_t sA_base = smem_base, sB_base = smem_base + CV_A_STAGES * CV_A_STAGE_BYTES;
  const uint32_t bar_base = smem_base + CV_RING_BYTES;
  auto full_a = [&](int s) { return bar_base + 8u * s; };
  auto empty_a = [&](int s) { return bar_base + 8u * (CV_A_STAGES + s); };
  auto full_b = [&](int s) { return bar_base + 8u * (2 * CV_A_STAGES + s); };
  auto empty_b = [&](int s) { return bar_base + 8u * (2 * CV_A_STAGES + CV_B_STAGES + s); };

  const int wg = threadIdx.x >> 7;
  const int kblocks_per_tap = cs.Cin / KBC;
  const int n_kh = cs.taps == 9 ? CV_KH : 1;             // K-blocks per activation box
  const int n_boxes_item = (cs.taps / n_kh) * kblocks_per_tap;   // activation boxes per item: (kw, channel block), kh innermost
  const int n_items = cs.n_tiles * cs.n_slices;

  if (threadIdx.x == 0) {
    for (int s = 0; s < CV_A_STAGES; ++s) {
      mbar_init(full_a(s), 1);
      mbar_init(empty_a(s), 8);                      // one arrive per MMA warp
    }
    for (int s = 0; s < CV_B_STAGES; ++s) {
      mbar_init(full_b(s), 1);
      mbar_init(empty_b(s), 8);
    }
    if constexpr (GN != CV_GN_NONE) asm volatile("st.shared.v2.u32 [%0], {0, 0};" ::"r"(bar_base + CV_CNT_OFFSET) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // =============================== TMA producer (+ GroupNorm apply: warps 1-3) ===============================
    if constexpr (GN != CV_GN_NONE) {
      regs_dealloc<72>();
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      if (warp >= 1) {
        const int items_per_img = cs.per_img * cs.n_slices;      // items are image-major
        bool clamped = false;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
          const int b = item / items_per_img;
          if (b == cs.B - 1) break;                          // the last image: the tail below, with the MMA warps
          // the image's first item in this CTA's walk: warp 1 publishes the CTA's items of it
          if (warp == 1 && item - (int)gridDim.x < b * items_per_img)
            publish_image(bar_base + CV_CNT_OFFSET, gf.done + b, item, (b + 1) * items_per_img - 1, lane);
          wait_count(gf.done + b, items_per_img * CV_MMA_WARPS, lane);
          gn_apply_item<GN>(cs, gf, y, stats, item, warp - 1, CV_APPLY_WARPS, lane, clamped);
        }
        if (clamped && gf.overflow_flag) *gf.overflow_flag = 1;
      }
    } else {
      regs_dealloc<40>();
    }
    if (threadIdx.x == 0) {
      int a_st = 0, b_st = 0;
      uint32_t a_ph = 0, b_ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tile = item / cs.n_slices, n0 = (item - tile * cs.n_slices) * NT;
        const TileAt ta = tile_at(cs, tile);
        // 9 taps: the box is the tile shifted by kw - 1 columns and grown by one row above and below (the maps' box height is
        // tile h + 2); 1 tap: the tile itself
        const uint32_t a_bytes = (uint32_t)(CV_BM + ((n_kh - 1) << ta.twl)) * 64u;
        for (int ks = 0; ks < n_boxes_item; ++ks) {
          const int kw = cs.taps == 9 ? ks / kblocks_per_tap : 1, cblk = ks - (ks / kblocks_per_tap) * kblocks_per_tap;
          mbar_wait(empty_a(a_st), a_ph ^ 1u);
          const uint32_t sA_hi = sA_base + a_st * CV_A_STAGE_BYTES;
          mbar_expect_tx(full_a(a_st), (A_LO_ZERO ? 1 : 2) * a_bytes);
          const int aw = ta.w0 + kw - 1, ah = ta.h0 - (n_kh > 1 ? 1 : 0);
          tma_load_4d(&mp.x[ta.shape][0], full_a(a_st), sA_hi, cblk * KBC, aw, ah, ta.b);
          if constexpr (!A_LO_ZERO) tma_load_4d(&mp.x[ta.shape][1], full_a(a_st), sA_hi + CV_A_BYTES, cblk * KBC, aw, ah, ta.b);
          if (++a_st == CV_A_STAGES) { a_st = 0; a_ph ^= 1u; }
          for (int kh = 0; kh < n_kh; ++kh) {                // the weight rows of taps (kh, kw), kh = 0 .. n_kh - 1
            const int tap = cs.taps == 9 ? 3 * kh + kw : 0;
            const int kcol = tap * cs.Cin + cblk * KBC;
            mbar_wait(empty_b(b_st), b_ph ^ 1u);
            const uint32_t sB_hi = sB_base + b_st * CV_B_STAGE_BYTES;
            mbar_expect_tx(full_b(b_st), 2 * NT * 64);
            tma_load_2d(&mp.w[0], full_b(b_st), sB_hi, kcol, n0);
            tma_load_2d(&mp.w[1], full_b(b_st), sB_hi + CV_B_BYTES, kcol, n0);
            if (++b_st == CV_B_STAGES) { b_st = 0; b_ph ^= 1u; }
          }
        }
      }
    }
  } else {
    // =============================== MMA + epilogue (warpgroups 1, 2) ===============================
    if constexpr (GN != CV_GN_NONE) regs_alloc<216>();       // 128 x 72 + 256 x 216 <= 64 K registers
    else regs_alloc<232>();
    const int cw = wg - 1;                                  // pixel rows 64 cw .. 64 cw + 63 of the tile
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const float sc = F16 ? (dev_out_scale ? __fmul_rn(out_scale, *dev_out_scale) : out_scale) : 1.f;   // powers of two: exact
    float acc[NT / 2], cor[NT / 2];
    int a_st = 0, b_st = 0;
    uint32_t a_ph = 0, b_ph = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int tile = item / cs.n_slices, n0 = (item - tile * cs.n_slices) * NT;
      const TileAt ta = tile_at(cs, tile);
      // pixel p of the tile sits at box row p + kh * tile w for vertical tap kh: kh * (512 / 1024 / 2048 B), whole swizzle atoms
      const uint32_t kh_step = 64u << ta.twl;
      // the K loop of one item with a compile-time count of K-blocks per box (a run-time count inside the MMA sequence makes
      // ptxas fence the accumulators between the K-blocks).  Each K-block is one commit group; once the next one is issued and
      // the previous one has completed, its weight slot goes back, and its activation slot too after the box's last K-block.
      auto k_loop = [&](auto kh_n_) {
        constexpr int KH_N = decltype(kh_n_)::value;
        int prev_a = 0, prev_b = 0;
        for (int ks = 0; ks < n_boxes_item; ++ks) {
          mbar_wait(full_a(a_st), a_ph);
          const uint32_t sA_hi = sA_base + a_st * CV_A_STAGE_BYTES + (uint32_t)cw * (CV_BM * 64 / 2);
          const uint32_t sA_lo = sA_hi + CV_A_BYTES;
#pragma unroll
          for (int kh = 0; kh < KH_N; ++kh) {
            mbar_wait(full_b(b_st), b_ph);
            const uint32_t a_off = kh_step * kh, sB_hi = sB_base + b_st * CV_B_STAGE_BYTES, sB_lo = sB_hi + CV_B_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 2; ++k) {                    // 32 B (16 fp16 / 8 tf32) of K per MMA inside the 64 B swizzle row
              const uint64_t a_hi = gmma_desc(sA_hi + a_off + 32u * k, 16u, 512u, GMMA_SW64);
              const uint64_t a_lo = gmma_desc(sA_lo + a_off + 32u * k, 16u, 512u, GMMA_SW64);
              const uint64_t b_hi = gmma_desc(sB_hi + 32u * k, 16u, 512u, GMMA_SW64), b_lo = gmma_desc(sB_lo + 32u * k, 16u, 512u, GMMA_SW64);
              const uint32_t first = (ks | kh | k) != 0;
              if constexpr (F16) {
                wgmma_f16<0, 0>(acc, a_hi, b_hi, first);
                if constexpr (A_LO_ZERO) {
                  wgmma_f16<0, 0>(cor, a_hi, b_lo, first);
                } else {
                  wgmma_f16<0, 0>(cor, a_lo, b_hi, first);
                  wgmma_f16<0, 0>(cor, a_hi, b_lo, 1u);
                }
              } else {
                wgmma_tf32(acc, a_hi, b_hi, first);
                wgmma_tf32(cor, a_lo, b_hi, first);
                wgmma_tf32(cor, a_hi, b_lo, 1u);
              }
            }
            wgmma_commit();
            if ((ks | kh) != 0) {                            // the previous K-block's MMAs have read their slots: hand them back
              wgmma_wait<1>();
              if (lane == 0) {
                mbar_arrive(empty_b(prev_b));
                if (kh == 0) mbar_arrive(empty_a(prev_a));   // the previous K-block was the last one of its box
              }
            }
            prev_b = b_st;
            if (++b_st == CV_B_STAGES) { b_st = 0; b_ph ^= 1u; }
          }
          prev_a = a_st;
          if (++a_st == CV_A_STAGES) { a_st = 0; a_ph ^= 1u; }
        }
        wgmma_wait<0>();
        if (lane == 0) { mbar_arrive(empty_b(prev_b)); mbar_arrive(empty_a(prev_a)); }
      };
      if (n_kh == CV_KH) k_loop(std::integral_constant<int, CV_KH>{});
      else k_loop(std::integral_constant<int, 1>{});

      // ---- epilogue: rows r0 and r0 + 8, columns n0 + 8 i + 2 (lane % 4) (+1) ----
      const int h_end = ta.shape == 2 ? cs.right_h : cs.H;   // the right strip stops where the bottom strip begins
      OutT* row_ptr[2];
      bool valid[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = 64 * cw + 16 * warp + (lane >> 2) + 8 * j;
        const int h = ta.h0 + (r >> ta.twl), w = ta.w0 + (r & ((1 << ta.twl) - 1));
        valid[j] = h < h_end && w < cs.W;
        row_ptr[j] = y + (((size_t)ta.b * cs.H + h) * cs.W + w) * cs.ldy;
      }
      float part[NT == 128 ? 32 : 1];                        // per group of 8 channels: (sum, sum of squares) of this thread's values
#pragma unroll
      for (int i = 0; i < NT / 8; ++i) {
        const int col = n0 + 8 * i + 2 * (lane & 3);
        float s = 0.f, ss = 0.f;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float v0 = __fadd_rn(acc[4 * i + 2 * j], cor[4 * i + 2 * j]);
          float v1 = __fadd_rn(acc[4 * i + 2 * j + 1], cor[4 * i + 2 * j + 1]);
          if (F16) { v0 = __fmul_rn(v0, sc); v1 = __fmul_rn(v1, sc); }
          if (bias) {
            if (col < cs.n_out) v0 = v0 + __ldg(bias + col);
            if (col + 1 < cs.n_out) v1 = v1 + __ldg(bias + col + 1);
          }
          if (valid[j]) {
            if constexpr (std::is_same<OutT, float>::value) {
              if (col + 1 < cs.n_out) *reinterpret_cast<float2*>(row_ptr[j] + col) = make_float2(v0, v1);
              else if (col < cs.n_out) row_ptr[j][col] = v0;
            } else if constexpr (std::is_same<OutT, __half>::value) {
              if (col + 1 < cs.n_out) *reinterpret_cast<__half2*>(row_ptr[j] + col) = __halves2half2(__float2half_rn(v0), __float2half_rn(v1));
              else if (col < cs.n_out) row_ptr[j][col] = __float2half_rn(v0);
            } else {
              if (col + 1 < cs.n_out) *reinterpret_cast<__nv_bfloat162*>(row_ptr[j] + col) = __halves2bfloat162(__float2bfloat16_rn(v0), __float2bfloat16_rn(v1));
              else if (col < cs.n_out) row_ptr[j][col] = __float2bfloat16_rn(v0);
            }
            s += v0 + v1;
            ss = fmaf(v0, v0, ss);
            ss = fmaf(v1, v1, ss);
          }
        }
        if constexpr (NT == 128) { part[2 * i] = s; part[2 * i + 1] = ss; }
      }
      if constexpr (NT == 128) {
        if (stats) {
          // halving butterfly: 32 values (16 groups x {sum, sumsq}) over 32 lanes in 31 shuffles; lane L ends with value L
          auto level = [&](auto o_) {
            constexpr int o = decltype(o_)::value;
            const bool up = (lane & o) != 0;
#pragma unroll
            for (int i = 0; i < o; ++i) {
              const float send = up ? part[i] : part[i + o];
              const float recv = __shfl_xor_sync(0xffffffffu, send, o);
              part[i] = (up ? part[i + o] : part[i]) + recv;
            }
          };
          level(std::integral_constant<int, 16>{}); level(std::integral_constant<int, 8>{}); level(std::integral_constant<int, 4>{});
          level(std::integral_constant<int, 2>{}); level(std::integral_constant<int, 1>{});
          atomicAdd(stats + ((size_t)ta.b * 32 + (n0 >> 3) + (lane >> 1)) * 2 + (lane & 1), (double)part[0]);
        }
      }
      if constexpr (GN != CV_GN_NONE) {      // this warp's stores and statistics of the item are done: count them (warp 1 publishes)
        __syncwarp();
        if (lane == 0) red_release_cta_shared_add(bar_base + CV_CNT_OFFSET + 4u * cw, 1);
      }
    }
  }
  if constexpr (GN != CV_GN_NONE) {
    // tail: the apply warps and the 8 MMA warps (11 warps, once each has run out of items) share this CTA's items of the last image,
    // which has no MMA work left to hide behind.  One copy of this code serves both roles, so it fits the apply warps' registers.
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 1) {
      const int items_per_img = cs.per_img * cs.n_slices, last0 = (cs.B - 1) * items_per_img;
      bool clamped = false;
      int item = (int)blockIdx.x;
      if (item < last0) item += (last0 - item + (int)gridDim.x - 1) / (int)gridDim.x * (int)gridDim.x;   // first item of the last image
      if (warp == 1 && item < n_items) publish_image(bar_base + CV_CNT_OFFSET, gf.done + cs.B - 1, item, n_items - 1, lane);
      for (; item < n_items; item += gridDim.x) {
        wait_count(gf.done + cs.B - 1, items_per_img * CV_MMA_WARPS, lane);
        gn_apply_item<GN>(cs, gf, y, stats, item, warp - 1, CV_APPLY_WARPS + CV_MMA_WARPS, lane, clamped);
      }
      if (clamped && gf.overflow_flag) *gf.overflow_flag = 1;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// elementwise helpers (HBM-bound, 128-bit vectors)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

__global__ void __launch_bounds__(256)
split_tf32_kernel(const float4* __restrict__ x, long long n4, float4* __restrict__ hi, float4* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const float4 v = __ldcs(x + i);
    float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    hi[i] = h;
    lo[i] = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
  }
}

// y: raw conv output [B][HW][C]; stats: [B][G][2] (sum, sumsq) fp64.  out = relu((y-mean)*rstd*gamma + beta)
// written either as fp32 (out_lo == NULL) or as the TF32 hi/lo pair the next conv consumes.
__global__ void __launch_bounds__(256)
gn_relu_apply_kernel(const float4* __restrict__ y, const double* __restrict__ stats, const float* __restrict__ gamma,
                     const float* __restrict__ beta, int HW, int C, int groups, float eps, int relu, long long n4,
                     float4* __restrict__ out_hi, float4* __restrict__ out_lo) {
  const int c4n = C >> 2;
  const int cpg = C / groups;
  const double inv_n = 1.0 / ((double)HW * cpg);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % c4n) * 4;
    const long long pix = i / c4n;
    const int b = (int)(pix / HW);
    const int g = c / cpg;            // cpg is a multiple of 4 or the 4 channels share... (host guarantees cpg % 4 == 0)
    const double s = stats[((size_t)b * groups + g) * 2], ss = stats[((size_t)b * groups + g) * 2 + 1];
    const double mean = s * inv_n;
    double var = ss * inv_n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float mu = (float)mean;
    const float4 v = __ldcs(y + i);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    float4 o;
    o.x = fmaf((v.x - mu) * rstd, ga.x, be.x);
    o.y = fmaf((v.y - mu) * rstd, ga.y, be.y);
    o.z = fmaf((v.z - mu) * rstd, ga.z, be.z);
    o.w = fmaf((v.w - mu) * rstd, ga.w, be.w);
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    if (out_lo) {
      const float4 h = make_float4(tf32_hi(o.x), tf32_hi(o.y), tf32_hi(o.z), tf32_hi(o.w));
      out_hi[i] = h;
      out_lo[i] = make_float4(o.x - h.x, o.y - h.y, o.z - h.z, o.w - h.w);
    } else {
      out_hi[i] = o;
    }
  }
}

// ---- fp16 two-term split (split_h2, tc_ptx.cuh) ----
// power-of-two scale that brings amax into [2^11, 2^12) (fp16 max is 65504; small values keep 3e-8*|scale| absolute precision)
__device__ __forceinline__ float pow2_scale_for(float amax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
  int e;
  frexpf(amax, &e);                 // amax = m * 2^e, m in [0.5, 1)
  return ldexpf(1.f, 12 - e);       // amax*scale in [2^11, 2^12)
}

__device__ __forceinline__ float amax4(float m, const float4 v) {
  return fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
}

// pure HBM read: four independent 16-byte loads in flight per thread (tens of KB in flight per SM are needed to saturate HBM)
__global__ void __launch_bounds__(256) amax_abs_kernel(const float4* __restrict__ x, long long n4, unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  const long long step = (long long)gridDim.x * 256;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  for (; i + 3 * step < n4; i += 4 * step) {
    const float4 v0 = x[i], v1 = x[i + step], v2 = x[i + 2 * step], v3 = x[i + 3 * step];
    m = amax4(amax4(amax4(amax4(m, v0), v1), v2), v3);
  }
  for (; i < n4; i += step) m = amax4(m, x[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));     // non-negative floats order like their bits
}

__device__ __forceinline__ void split8(const float4 a, const float4 b, float scale, uint4& ph, uint4& pl) {
  __align__(16) __half h[8], l[8];
  split_h2(a.x * scale, h[0], l[0]); split_h2(a.y * scale, h[1], l[1]);
  split_h2(a.z * scale, h[2], l[2]); split_h2(a.w * scale, h[3], l[3]);
  split_h2(b.x * scale, h[4], l[4]); split_h2(b.y * scale, h[5], l[5]);
  split_h2(b.z * scale, h[6], l[6]); split_h2(b.w * scale, h[7], l[7]);
  ph = *reinterpret_cast<uint4*>(h);
  pl = *reinterpret_cast<uint4*>(l);
}

// hi/lo are [n] fp16; dev_amax (optional) selects a power-of-two scale on the device, its inverse is written to inv_scale_out.
// 8 elements per thread and step: 2 x 16-byte loads, 2 x 16-byte stores; two steps in flight.
__global__ void __launch_bounds__(256)
split_f16_kernel(const float4* __restrict__ x, long long n4, const unsigned int* __restrict__ dev_amax_bits,
                 uint2* __restrict__ hi, uint2* __restrict__ lo, float* __restrict__ inv_scale_out) {
  const float scale = dev_amax_bits ? pow2_scale_for(__uint_as_float(*dev_amax_bits)) : 1.f;
  if (inv_scale_out && blockIdx.x == 0 && threadIdx.x == 0) *inv_scale_out = 1.f / scale;
  const long long n8 = n4 >> 1;
  const long long step = (long long)gridDim.x * 256;
  uint4* hi8 = reinterpret_cast<uint4*>(hi);
  uint4* lo8 = reinterpret_cast<uint4*>(lo);
  const bool al16 = ((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (al16) {
    for (; i + step < n8; i += 2 * step) {
      const float4 a0 = __ldcs(x + 2 * i), a1 = __ldcs(x + 2 * i + 1);
      const float4 b0 = __ldcs(x + 2 * (i + step)), b1 = __ldcs(x + 2 * (i + step) + 1);
      uint4 ph, pl;
      split8(a0, a1, scale, ph, pl);
      hi8[i] = ph; lo8[i] = pl;
      split8(b0, b1, scale, ph, pl);
      hi8[i + step] = ph; lo8[i + step] = pl;
    }
    for (; i < n8; i += step) {
      uint4 ph, pl;
      split8(__ldcs(x + 2 * i), __ldcs(x + 2 * i + 1), scale, ph, pl);
      hi8[i] = ph; lo8[i] = pl;
    }
    i = 2 * n8 + (long long)blockIdx.x * 256 + threadIdx.x;       // odd float4 tail
  }
  for (; i < n4; i += step) {
    const float4 v = __ldcs(x + i);
    __half h[4], l[4];
    split_h2(v.x * scale, h[0], l[0]); split_h2(v.y * scale, h[1], l[1]);
    split_h2(v.z * scale, h[2], l[2]); split_h2(v.w * scale, h[3], l[3]);
    hi[i] = *reinterpret_cast<uint2*>(h);
    lo[i] = *reinterpret_cast<uint2*>(l);
  }
}

// ---- bf16 activations: the same (hi, lo, scale) as split_f16_kernel on the upcast tensor (bf16 -> fp32 is exact, so bit for bit),
// read at 2 B / element.  8 values (one 16-byte load) per thread and step.
__device__ __forceinline__ void bf16x8_to_f32(const uint4 v, float4& a, float4& b) {
  a = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xFFFF0000u), __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xFFFF0000u));
  b = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xFFFF0000u), __uint_as_float(v.w << 16), __uint_as_float(v.w & 0xFFFF0000u));
}

__global__ void __launch_bounds__(256) amax_abs_bf16_kernel(const uint4* __restrict__ x, long long n8, unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  const long long step = (long long)gridDim.x * 256;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  float4 a, b;
  for (; i + 3 * step < n8; i += 4 * step) {
    const uint4 v0 = x[i], v1 = x[i + step], v2 = x[i + 2 * step], v3 = x[i + 3 * step];
    bf16x8_to_f32(v0, a, b); m = amax4(amax4(m, a), b);
    bf16x8_to_f32(v1, a, b); m = amax4(amax4(m, a), b);
    bf16x8_to_f32(v2, a, b); m = amax4(amax4(m, a), b);
    bf16x8_to_f32(v3, a, b); m = amax4(amax4(m, a), b);
  }
  for (; i < n8; i += step) { bf16x8_to_f32(x[i], a, b); m = amax4(amax4(m, a), b); }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(256)
split_f16_from_bf16_kernel(const uint4* __restrict__ x, long long n8, const unsigned int* __restrict__ dev_amax_bits,
                           uint4* __restrict__ hi, uint4* __restrict__ lo, float* __restrict__ inv_scale_out) {
  const float scale = pow2_scale_for(__uint_as_float(*dev_amax_bits));
  if (blockIdx.x == 0 && threadIdx.x == 0) *inv_scale_out = 1.f / scale;
  const long long step = (long long)gridDim.x * 256;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  float4 a, b;
  uint4 ph, pl;
  for (; i + step < n8; i += 2 * step) {
    const uint4 v0 = __ldcs(x + i), v1 = __ldcs(x + i + step);
    bf16x8_to_f32(v0, a, b); split8(a, b, scale, ph, pl);
    hi[i] = ph; lo[i] = pl;
    bf16x8_to_f32(v1, a, b); split8(a, b, scale, ph, pl);
    hi[i + step] = ph; lo[i + step] = pl;
  }
  for (; i < n8; i += step) {
    bf16x8_to_f32(__ldcs(x + i), a, b); split8(a, b, scale, ph, pl);
    hi[i] = ph; lo[i] = pl;
  }
}

// GroupNorm + ReLU written directly as the fp16 (h, l) pair of the next conv; |out| is clamped to 60000 (never reached by
// a GroupNorm output with sane affine parameters) and *overflow_flag is raised if the clamp ever fires.
__global__ void __launch_bounds__(256)
gn_relu_apply_f16_kernel(const float4* __restrict__ y, const double* __restrict__ stats, const float* __restrict__ gamma,
                         const float* __restrict__ beta, int HW, int C, int groups, float eps, int relu, long long n4,
                         uint2* __restrict__ out_h, uint2* __restrict__ out_l, int* __restrict__ overflow_flag) {
  const int c4n = C >> 2;
  const int cpg = C / groups;
  const double inv_n = 1.0 / ((double)HW * cpg);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % c4n) * 4;
    const long long pix = i / c4n;
    const int b = (int)(pix / HW);
    const int g = c / cpg;
    const double s = stats[((size_t)b * groups + g) * 2], ss = stats[((size_t)b * groups + g) * 2 + 1];
    const double mean = s * inv_n;
    double var = ss * inv_n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float mu = (float)mean;
    const float4 v = __ldcs(y + i);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    float o[4];
    o[0] = fmaf((v.x - mu) * rstd, ga.x, be.x); o[1] = fmaf((v.y - mu) * rstd, ga.y, be.y);
    o[2] = fmaf((v.z - mu) * rstd, ga.z, be.z); o[3] = fmaf((v.w - mu) * rstd, ga.w, be.w);
    __half h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (relu) o[j] = fmaxf(o[j], 0.f);
      if (fabsf(o[j]) > 60000.f) { o[j] = copysignf(60000.f, o[j]); if (overflow_flag) *overflow_flag = 1; }
      split_h2(o[j], h[j], l[j]);
    }
    out_h[i] = *reinterpret_cast<uint2*>(h);
    out_l[i] = *reinterpret_cast<uint2*>(l);
  }
}

// Fast path of the above for C/8 | 256 and 8 | C/groups: a thread owns 8 channels of one group (mean, rstd, gamma, beta live in
// registers for the whole kernel: no per-element double math or integer division), C/8 threads cover a pixel, blockIdx.y is the
// image and blockIdx.x a contiguous range of pixels; 32-byte loads, 2 x 16-byte stores, two pixels in flight per thread.
__global__ void __launch_bounds__(256)
gn_relu_apply_f16_v8_kernel(const float4* __restrict__ y, const double* __restrict__ stats, const float* __restrict__ gamma,
                            const float* __restrict__ beta, int HW, int C, int groups, float eps, int relu, int pix_per_cta,
                            uint4* __restrict__ out_h, uint4* __restrict__ out_l, int* __restrict__ overflow_flag) {
  const int tpp = C >> 3;                 // threads per pixel
  const int ppp = 256 / tpp;              // pixels per pass
  const int c = (threadIdx.x % tpp) * 8;
  const int b = blockIdx.y;
  const int cpg = C / groups;
  const int g = c / cpg;
  const double inv_n = 1.0 / ((double)HW * cpg);
  const double s = stats[((size_t)b * groups + g) * 2], ss = stats[((size_t)b * groups + g) * 2 + 1];
  const double mean = s * inv_n;
  double var = ss * inv_n - mean * mean;
  var = var < 0.0 ? 0.0 : var;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float mu = (float)mean;
  float ga[8], be[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { ga[j] = gamma[c + j]; be[j] = beta[c + j]; }
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  const size_t img = (size_t)b * HW;
  bool clamped = false;
  auto apply = [&](const float4 a, const float4 q, size_t idx8) {
    float o[8] = {a.x, a.y, a.z, a.w, q.x, q.y, q.z, q.w};
    __align__(16) __half h[8], l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] = fmaf((o[j] - mu) * rstd, ga[j], be[j]);
      if (relu) o[j] = fmaxf(o[j], 0.f);
      if (fabsf(o[j]) > 60000.f) { o[j] = copysignf(60000.f, o[j]); clamped = true; }
      split_h2(o[j], h[j], l[j]);
    }
    out_h[idx8] = *reinterpret_cast<uint4*>(h);
    out_l[idx8] = *reinterpret_cast<uint4*>(l);
  };
  int p = p0 + threadIdx.x / tpp;
  for (; p + ppp < p1; p += 2 * ppp) {
    const size_t i0 = ((img + p) * C + c) >> 3, i1 = ((img + p + ppp) * C + c) >> 3;
    const float4 a0 = __ldcs(y + 2 * i0), a1 = __ldcs(y + 2 * i0 + 1);
    const float4 b0 = __ldcs(y + 2 * i1), b1 = __ldcs(y + 2 * i1 + 1);
    apply(a0, a1, i0);
    apply(b0, b1, i1);
  }
  for (; p < p1; p += ppp) {
    const size_t i0 = ((img + p) * C + c) >> 3;
    apply(__ldcs(y + 2 * i0), __ldcs(y + 2 * i0 + 1), i0);
  }
  if (clamped && overflow_flag) *overflow_flag = 1;
}

// w [n_out][Cin][taps] (nn.Conv2d / nn.Linear) -> packed [n_mma][tap*Cin + ci] (rows >= n_out are zero) as fp16 h / l
__global__ void pack_conv_weight_f16_kernel(const float* __restrict__ w, int n_out, int n_mma, int Cin, int taps, float scale,
                                            __half* __restrict__ hi, __half* __restrict__ lo) {
  const long long n = (long long)n_mma * Cin * taps;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % Cin);
    const int tap = (int)((i / Cin) % taps);
    const int co = (int)(i / ((long long)Cin * taps));
    const float v = co < n_out ? w[((size_t)co * Cin + ci) * taps + tap] * scale : 0.f;
    split_h2(v, hi[i], lo[i]);
  }
}

// w [Cout][Cin][3][3] (nn.Conv2d) -> packed [Cout][tap][Cin] split into TF32 hi / lo
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, int Cout, int Cin, float* __restrict__ hi,
                                        float* __restrict__ lo) {
  const long long n = (long long)Cout * Cin * 9;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % Cin);
    const int tap = (int)((i / Cin) % 9);
    const int co = (int)(i / ((long long)Cin * 9));
    const float v = w[((size_t)co * Cin + ci) * 9 + tap];
    const float h = tf32_hi(v);
    hi[i] = h;
    lo[i] = v - h;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
EncodeTiledFn tc_get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

constexpr int CV_SHAPE_TW[3] = {16, 32, 8}, CV_SHAPE_TH[3] = {8, 4, 16};
static_assert((CV_SHAPE_TH[0] + 2) * CV_SHAPE_TW[0] * 64 <= CV_A_BYTES && (CV_SHAPE_TH[1] + 2) * CV_SHAPE_TW[1] * 64 <= CV_A_BYTES &&
              (CV_SHAPE_TH[2] + 2) * CV_SHAPE_TW[2] * 64 <= CV_A_BYTES, "a conv3x3 activation box overflows its stage slot");

// halo: extra image rows of the box (2 for a conv3x3: the three vertical taps of one column offset read one box)
static int make_act_map(CUtensorMap* tm, const void* ptr, int B, int H, int W, int C, bool f16, int shape, int halo) {
  EncodeTiledFn enc = tc_get_encode();
  if (!enc) return fail("%s", "cuTensorMapEncodeTiled is unavailable (driver too old?)");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t es = f16 ? 2 : 4;
  cuuint64_t strides[3] = {(cuuint64_t)C * es, (cuuint64_t)W * C * es, (cuuint64_t)H * W * C * es};
  cuuint32_t box[4] = {(cuuint32_t)(f16 ? CV_KB_F16 : CV_KB), (cuuint32_t)CV_SHAPE_TW[shape], (cuuint32_t)(CV_SHAPE_TH[shape] + halo), 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(activation) failed: %s%lld", "", (long long)r);
  return 0;
}
static int make_w_map(CUtensorMap* tm, const void* ptr, int n_mma, int Ktot, bool f16, int box_rows) {
  EncodeTiledFn enc = tc_get_encode();
  if (!enc) return fail("%s", "cuTensorMapEncodeTiled is unavailable (driver too old?)");
  cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)n_mma};
  cuuint64_t strides[1] = {(cuuint64_t)Ktot * (f16 ? 2 : 4)};
  cuuint32_t box[2] = {(cuuint32_t)(f16 ? CV_KB_F16 : CV_KB), (cuuint32_t)box_rows};   // one channel slice per TMA request
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(weights) failed: %s%lld", "", (long long)r);
  return 0;
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream) {
  PTB_REQUIRE(n >= 0 && n % 4 == 0, "n must be a multiple of 4");
  PTB_REQUIRE(((uintptr_t)x % 16 == 0) && ((uintptr_t)hi % 16 == 0) && ((uintptr_t)lo % 16 == 0), "16-byte alignment");
  if (n == 0) return 0;
  long long blocks = (n / 4 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  split_tf32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), n / 4,
                                                                       reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo));
  return check_launch("ptb_split_tf32");
}

extern "C" int ptb_conv3x3_pack_weight(const float* w_oihw, int Cout, int Cin, float* w_hi, float* w_lo, void* stream) {
  PTB_REQUIRE(Cout > 0 && Cin > 0 && w_oihw && w_hi && w_lo, "shape / NULL");
  const long long n = (long long)Cout * Cin * 9;
  pack_conv_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w_oihw, Cout, Cin, w_hi, w_lo);
  return check_launch("ptb_conv3x3_pack_weight");
}

template <bool F16, int NT, bool A_LO_ZERO = false, typename OutT = float>
static int conv_launch_nt(const ConvMaps& mp, const ConvShape& cs, OutT* y, double* gn_stats, float out_scale, const float* dev_out_scale,
                          const float* bias, void* stream) {
  // a function attribute is per DEVICE and a process may drive several: set it on every call (a few hundred ns)
  if (cudaFuncSetAttribute(conv_tc_kernel<F16, NT, A_LO_ZERO, OutT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CV_SMEM_BYTES) != cudaSuccess)
    return fail("%s", "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed for the conv kernel");
  int grid = sm_count();                                     // persistent: one CTA per SM
  if (grid > cs.n_tiles * cs.n_slices) grid = cs.n_tiles * cs.n_slices;
  conv_tc_kernel<F16, NT, A_LO_ZERO, OutT><<<grid, CV_THREADS, CV_SMEM_BYTES, (cudaStream_t)stream>>>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias,
                                                                                                    GnFuse{});
  return 0;
}

// the fused GroupNorm-apply conv: a cooperative launch, as its CTAs wait on each other's items.  *launched = false (nothing enqueued,
// no error) when the grid cannot be co-resident or the device refuses the cooperative launch: the caller runs the two kernels.
template <bool A_LO_ZERO, int GN>
static int conv_gn_launch(const ConvMaps& mp, const ConvShape& cs, float* y, double* stats, float out_scale, const float* dev_out_scale,
                          const GnFuse& gf, cudaStream_t st, bool* launched) {
  *launched = false;
  auto kern = conv_tc_kernel<true, CV_NT, A_LO_ZERO, float, GN>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CV_SMEM_BYTES) != cudaSuccess)
    return fail("%s", "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed for the fused conv kernel");
  const int n_items = cs.n_tiles * cs.n_slices;
  const int grid = sm_count() < n_items ? sm_count() : n_items;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CV_THREADS, CV_SMEM_BYTES) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  if (per_sm * sm_count() < grid) return 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(CV_THREADS);
  cfg.dynamicSmemBytes = CV_SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const float* no_bias = nullptr;
  if (cudaLaunchKernelEx(&cfg, kern, mp, cs, y, stats, out_scale, dev_out_scale, no_bias, gf) != cudaSuccess) {
    (void)cudaGetLastError();          // a refused launch is not sticky: clear it and let the caller run the two kernels
    return 0;
  }
  *launched = true;
  return 0;
}

// tile plan, output-channel slice width (*nt) and tensor maps of one conv launch.  A_LO_ZERO: x_lo is not read (NULL).
template <bool F16, bool A_LO_ZERO>
static int conv_prepare(ConvShape& cs, ConvMaps& mp, int* nt_out, const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo,
                        int B, int H, int W, int Cin, int taps, int n_out, int n_mma, int ldy, const double* gn_stats) {
  cs.B = B; cs.H = H; cs.W = W; cs.Cin = Cin;
  {   // tile plan (see ConvShape)
    const int rh = H % 8, rw = W % 16;
    const bool bottom = rh >= 1 && rh <= 4;
    cs.tiles_h = bottom ? H / 8 : (H + 7) / 8;
    cs.bottom_h0 = cs.tiles_h * 8;
    cs.n_bottom = bottom ? (W + 31) / 32 : 0;
    const bool right = rw >= 1 && rw <= 8 && cs.tiles_h > 0;
    cs.tiles_w = right ? W / 16 : (W + 15) / 16;
    cs.right_w0 = cs.tiles_w * 16;
    cs.right_h = cs.tiles_h * 8 < H ? cs.tiles_h * 8 : H;
    cs.n_right = right ? (cs.right_h + 15) / 16 : 0;
    cs.n_main = cs.tiles_h * cs.tiles_w;
    cs.per_img = cs.n_main + cs.n_right + cs.n_bottom;
    cs.n_tiles = B * cs.per_img;
  }
  // narrowest slice width that covers the output channels (the MMA N); wider outputs run as ceil(n_mma / 128) slices of 128
  // (two at 256 channels, up to four at CV_N_MAX)
  const int nt = (!F16 || n_mma > 64) ? CV_NT : n_mma > 32 ? 64 : n_mma > 16 ? 32 : 16;
  // the epilogue's statistics index [B][32][2] as (slice start / 8 + group in slice): 256 channels = 32 groups of 8, 128-channel slices
  PTB_REQUIRE(!gn_stats || (n_out == CV_N && n_mma == CV_N && nt == CV_NT), "GroupNorm statistics need 256 output channels (32 groups of 8)");
  cs.n_slices = (n_mma + nt - 1) / nt;
  cs.taps = taps; cs.n_out = n_out; cs.ldy = ldy;
  int rc;
  for (int sh = 0; sh < 3; ++sh) {
    if ((rc = make_act_map(&mp.x[sh][0], x_hi, B, H, W, Cin, F16, sh, taps == 9 ? 2 : 0))) return rc;
    if (A_LO_ZERO) mp.x[sh][1] = mp.x[sh][0];            // never used by the kernel
    else if ((rc = make_act_map(&mp.x[sh][1], x_lo, B, H, W, Cin, F16, sh, taps == 9 ? 2 : 0))) return rc;
  }
  if ((rc = make_w_map(&mp.w[0], w_hi, n_mma, taps * Cin, F16, nt))) return rc;
  if ((rc = make_w_map(&mp.w[1], w_lo, n_mma, taps * Cin, F16, nt))) return rc;
  *nt_out = nt;
  return 0;
}

// A_LO_ZERO: x_lo is not read (NULL).  OutT != float runs 128-channel slices only (n_mma > 64: the callers' input gradients).
template <bool F16, bool A_LO_ZERO = false, typename OutT = float>
static int conv_launch(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, int B, int H, int W, int Cin, int taps,
                       int n_out, int n_mma, OutT* y, int ldy, const float* bias, double* gn_stats, float out_scale,
                       const float* dev_out_scale, void* stream, const char* what) {
  ConvShape cs;
  ConvMaps mp;
  int nt = 0;
  int rc = conv_prepare<F16, A_LO_ZERO>(cs, mp, &nt, x_hi, x_lo, w_hi, w_lo, B, H, W, Cin, taps, n_out, n_mma, ldy, gn_stats);
  if (rc) return rc;
  if constexpr (!F16) rc = conv_launch_nt<false, 128>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias, stream);
  else if (nt == 128) rc = conv_launch_nt<true, 128, A_LO_ZERO, OutT>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias, stream);
  else if constexpr (!std::is_same<OutT, float>::value) return fail("%s: a half-precision output needs more than 64 output channels", what);
  else if (nt == 64) rc = conv_launch_nt<true, 64, A_LO_ZERO>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias, stream);
  else if (nt == 32) rc = conv_launch_nt<true, 32, A_LO_ZERO>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias, stream);
  else rc = conv_launch_nt<true, 16, A_LO_ZERO>(mp, cs, y, gn_stats, out_scale, dev_out_scale, bias, stream);
  if (rc) return rc;
  return check_launch(what);
}

extern "C" int ptb_conv3x3_c256_tf32x3(const float* x_hi, const float* x_lo, const float* w_hi, const float* w_lo, int B, int H,
                                       int W, int Cin, float* y, double* gn_stats, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0, "shape");
  PTB_REQUIRE(Cin % CV_KB == 0, "Cin must be a multiple of 16");
  PTB_REQUIRE(x_hi && x_lo && w_hi && w_lo && y, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_hi % 16 == 0) && ((uintptr_t)x_lo % 16 == 0) && ((uintptr_t)w_hi % 16 == 0) &&
                  ((uintptr_t)w_lo % 16 == 0) && ((uintptr_t)y % 16 == 0), "16-byte alignment");
  return conv_launch<false>(x_hi, x_lo, w_hi, w_lo, B, H, W, Cin, 9, CV_N, CV_N, y, CV_N, nullptr, gn_stats, 1.f, nullptr, stream,
                            "ptb_conv3x3_c256_tf32x3");
}

extern "C" int ptb_conv3x3_c256_f16x2(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                                      float out_scale, const float* dev_out_scale, float* y, double* gn_stats, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0, "shape");
  PTB_REQUIRE(Cin % CV_KB_F16 == 0, "Cin must be a multiple of 32");
  PTB_REQUIRE(x_h && x_l && w_h && w_l && y, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_h % 16 == 0) && ((uintptr_t)x_l % 16 == 0) && ((uintptr_t)w_h % 16 == 0) && ((uintptr_t)w_l % 16 == 0) &&
                  ((uintptr_t)y % 16 == 0), "16-byte alignment");
  return conv_launch<true>(x_h, x_l, w_h, w_l, B, H, W, Cin, 9, CV_N, CV_N, y, CV_N, nullptr, gn_stats, out_scale, dev_out_scale, stream,
                           "ptb_conv3x3_c256_f16x2");
}

extern "C" int ptb_split_f16(const float* x, int64_t n, int auto_scale, void* hi, void* lo, float* dev_inv_scale, void* workspace,
                             void* stream) {
  PTB_REQUIRE(n >= 0 && n % 4 == 0, "n must be a multiple of 4");
  PTB_REQUIRE(((uintptr_t)x % 16 == 0) && ((uintptr_t)hi % 8 == 0) && ((uintptr_t)lo % 8 == 0), "alignment");
  PTB_REQUIRE(!auto_scale || (workspace && dev_inv_scale), "auto_scale needs a 4-byte workspace and dev_inv_scale");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  long long blocks = (n / 4 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  unsigned int* amax = nullptr;
  if (auto_scale) {
    amax = reinterpret_cast<unsigned int*>(workspace);
    if (cudaMemsetAsync(amax, 0, 4, st) != cudaSuccess) return fail("%s", "ptb_split_f16: cudaMemsetAsync failed");
    amax_abs_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(x), n / 4, amax);
    int rc = check_launch("ptb_split_f16/amax");
    if (rc) return rc;
  }
  split_f16_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(x), n / 4, amax, reinterpret_cast<uint2*>(hi),
                                                    reinterpret_cast<uint2*>(lo), dev_inv_scale);
  return check_launch("ptb_split_f16");
}

extern "C" int ptb_split_f16_amax(const float* x, int64_t n, const unsigned int* dev_amax_bits, void* hi, void* lo,
                                  float* dev_inv_scale, void* stream) {
  PTB_REQUIRE(n >= 0 && n % 4 == 0, "n must be a multiple of 4");
  PTB_REQUIRE(((uintptr_t)x % 16 == 0) && ((uintptr_t)hi % 8 == 0) && ((uintptr_t)lo % 8 == 0), "alignment");
  PTB_REQUIRE(dev_amax_bits && dev_inv_scale, "dev_amax_bits and dev_inv_scale are required");
  if (n == 0) return 0;
  long long blocks = (n / 4 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  split_f16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), n / 4, dev_amax_bits,
                                                                      reinterpret_cast<uint2*>(hi), reinterpret_cast<uint2*>(lo),
                                                                      dev_inv_scale);
  return check_launch("ptb_split_f16_amax");
}

extern "C" int ptb_conv3x3_pack_weight_f16(const float* w_oihw, int Cout, int Cin, float scale, void* w_h, void* w_l, void* stream) {
  PTB_REQUIRE(Cout > 0 && Cin > 0 && w_oihw && w_h && w_l && scale > 0.f, "shape / NULL");
  const long long n = (long long)Cout * Cin * 9;
  pack_conv_weight_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w_oihw, Cout, Cout, Cin, 9, scale,
                                                                                           reinterpret_cast<__half*>(w_h),
                                                                                           reinterpret_cast<__half*>(w_l));
  return check_launch("ptb_conv3x3_pack_weight_f16");
}

extern "C" int ptb_conv_tc_pack_weight_f16(const float* w, int n_out, int n_mma, int Cin, int taps, float scale, void* w_h, void* w_l,
                                           void* stream) {
  PTB_REQUIRE(n_out > 0 && Cin > 0 && (taps == 1 || taps == 9) && w && w_h && w_l && scale > 0.f, "shape / NULL");
  PTB_REQUIRE(n_mma >= n_out && n_mma % 16 == 0 && n_mma <= CV_N_MAX, "n_mma must be a multiple of 16 in [n_out, 512]");
  const long long n = (long long)n_mma * Cin * taps;
  pack_conv_weight_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, n_out, n_mma, Cin, taps, scale,
                                                                                           reinterpret_cast<__half*>(w_h),
                                                                                           reinterpret_cast<__half*>(w_l));
  return check_launch("ptb_conv_tc_pack_weight_f16");
}

extern "C" int ptb_conv_tc_f16x2(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                                 int taps, int n_out, int n_mma, float out_scale, const float* dev_out_scale, const float* bias,
                                 float* y, int ldy, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && (taps == 1 || taps == 9), "shape");
  PTB_REQUIRE(Cin % CV_KB_F16 == 0, "Cin must be a multiple of 32");
  PTB_REQUIRE(n_out > 0 && n_mma >= n_out && n_mma % 16 == 0 && n_mma <= CV_N_MAX, "n_mma must be a multiple of 16 in [n_out, 512]");
  PTB_REQUIRE(ldy >= n_out && ldy % 4 == 0, "ldy must be a multiple of 4 and >= n_out");
  PTB_REQUIRE(x_h && x_l && w_h && w_l && y, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_h % 16 == 0) && ((uintptr_t)x_l % 16 == 0) && ((uintptr_t)w_h % 16 == 0) && ((uintptr_t)w_l % 16 == 0) &&
                  ((uintptr_t)y % 16 == 0), "16-byte alignment");
  return conv_launch<true>(x_h, x_l, w_h, w_l, B, H, W, Cin, taps, n_out, n_mma, y, ldy, bias, nullptr, out_scale, dev_out_scale, stream,
                           "ptb_conv_tc_f16x2");
}

// the checks ptb_conv_tc_f16x2 makes on its shape arguments, shared by the half-precision entry points
static int conv_tc_check_shape(int B, int H, int W, int Cin, int taps, int n_out, int n_mma, int ldy) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && (taps == 1 || taps == 9), "shape");
  PTB_REQUIRE(Cin % CV_KB_F16 == 0, "Cin must be a multiple of 32");
  PTB_REQUIRE(n_out > 0 && n_mma >= n_out && n_mma % 16 == 0 && n_mma <= CV_N_MAX, "n_mma must be a multiple of 16 in [n_out, 512]");
  PTB_REQUIRE(ldy >= n_out && ldy % 4 == 0, "ldy must be a multiple of 4 and >= n_out");
  return 0;
}

extern "C" int ptb_conv_tc_f16x1a(const void* x_h, const void* w_h, const void* w_l, int B, int H, int W, int Cin, int taps, int n_out,
                                  int n_mma, float out_scale, const float* dev_out_scale, const float* bias, float* y, int ldy,
                                  double* gn_stats, void* stream) {
  if (int rc = conv_tc_check_shape(B, H, W, Cin, taps, n_out, n_mma, ldy)) return rc;
  PTB_REQUIRE(x_h && w_h && w_l && y, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_h % 16 == 0) && ((uintptr_t)w_h % 16 == 0) && ((uintptr_t)w_l % 16 == 0) && ((uintptr_t)y % 16 == 0),
              "16-byte alignment");
  return conv_launch<true, true>(x_h, nullptr, w_h, w_l, B, H, W, Cin, taps, n_out, n_mma, y, ldy, bias, gn_stats, out_scale, dev_out_scale,
                                 stream, "ptb_conv_tc_f16x1a");
}

extern "C" int ptb_conv3x3_c256_f16_gn(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                                       float out_scale, const float* dev_out_scale, float* y, void* workspace, const float* gamma,
                                       const float* beta, float eps, void* out, void* out_l, int* overflow_flag, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0, "shape");
  PTB_REQUIRE(Cin % CV_KB_F16 == 0, "Cin must be a multiple of 32");
  PTB_REQUIRE(x_h && w_h && w_l && y && workspace && gamma && beta && out, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_h % 16 == 0) && ((uintptr_t)x_l % 16 == 0) && ((uintptr_t)w_h % 16 == 0) && ((uintptr_t)w_l % 16 == 0) &&
                  ((uintptr_t)y % 16 == 0) && ((uintptr_t)workspace % 8 == 0) && ((uintptr_t)gamma % 16 == 0) && ((uintptr_t)beta % 16 == 0) &&
                  ((uintptr_t)out % 16 == 0) && ((uintptr_t)out_l % 16 == 0), "alignment");
  cudaStream_t st = (cudaStream_t)stream;
  double* stats = reinterpret_cast<double*>(workspace);
  GnFuse gf;
  gf.gamma = gamma; gf.beta = beta; gf.eps = eps; gf.out = out; gf.out_l = reinterpret_cast<__half*>(out_l);
  gf.overflow_flag = overflow_flag;
  gf.done = reinterpret_cast<int*>(stats + (size_t)B * 32 * 2);
  ConvShape cs;
  ConvMaps mp;
  int nt = 0, rc;
  bool launched = false;
  if (x_l) {
    if ((rc = conv_prepare<true, false>(cs, mp, &nt, x_h, x_l, w_h, w_l, B, H, W, Cin, 9, CV_N, CV_N, CV_N, stats))) return rc;
    rc = out_l ? conv_gn_launch<false, CV_GN_F16>(mp, cs, y, stats, out_scale, dev_out_scale, gf, st, &launched)
               : conv_gn_launch<false, CV_GN_F32>(mp, cs, y, stats, out_scale, dev_out_scale, gf, st, &launched);
  } else {
    if ((rc = conv_prepare<true, true>(cs, mp, &nt, x_h, nullptr, w_h, w_l, B, H, W, Cin, 9, CV_N, CV_N, CV_N, stats))) return rc;
    rc = out_l ? conv_gn_launch<true, CV_GN_F16>(mp, cs, y, stats, out_scale, dev_out_scale, gf, st, &launched)
               : conv_gn_launch<true, CV_GN_F32>(mp, cs, y, stats, out_scale, dev_out_scale, gf, st, &launched);
  }
  if (rc) return rc;
  if (launched) return check_launch("ptb_conv3x3_c256_f16_gn");
  // the grid cannot be co-resident: the conv and the apply as two kernels (the same bits)
  if (x_l) rc = conv_launch<true>(x_h, x_l, w_h, w_l, B, H, W, Cin, 9, CV_N, CV_N, y, CV_N, nullptr, stats, out_scale, dev_out_scale, stream,
                                  "ptb_conv3x3_c256_f16_gn/conv");
  else rc = conv_launch<true, true>(x_h, nullptr, w_h, w_l, B, H, W, Cin, 9, CV_N, CV_N, y, CV_N, nullptr, stats, out_scale, dev_out_scale,
                                    stream, "ptb_conv3x3_c256_f16_gn/conv");
  if (rc) return rc;
  if (out_l) return ptb_gn_relu_apply_f16(y, stats, gamma, beta, B, H * W, CV_N, 32, eps, 1, out, out_l, overflow_flag, stream);
  return ptb_gn_relu_apply(y, stats, gamma, beta, B, H * W, CV_N, 32, eps, 1, reinterpret_cast<float*>(out), nullptr, stream);
}

extern "C" int ptb_conv_tc_f16x2_half_out(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                                          int taps, int n_out, int n_mma, float out_scale, const float* dev_out_scale, const float* bias,
                                          void* y, int y_dtype, int ldy, void* stream) {
  if (int rc = conv_tc_check_shape(B, H, W, Cin, taps, n_out, n_mma, ldy)) return rc;
  PTB_REQUIRE(y_dtype == PTB_DTYPE_F16 || y_dtype == PTB_DTYPE_BF16, "y_dtype must be PTB_DTYPE_F16 or PTB_DTYPE_BF16");
  PTB_REQUIRE(x_h && x_l && w_h && w_l && y, "NULL input");
  PTB_REQUIRE(((uintptr_t)x_h % 16 == 0) && ((uintptr_t)x_l % 16 == 0) && ((uintptr_t)w_h % 16 == 0) && ((uintptr_t)w_l % 16 == 0) &&
                  ((uintptr_t)y % 16 == 0), "16-byte alignment");
  if (y_dtype == PTB_DTYPE_F16)
    return conv_launch<true, false, __half>(x_h, x_l, w_h, w_l, B, H, W, Cin, taps, n_out, n_mma, reinterpret_cast<__half*>(y), ldy, bias,
                                            nullptr, out_scale, dev_out_scale, stream, "ptb_conv_tc_f16x2_half_out");
  return conv_launch<true, false, __nv_bfloat16>(x_h, x_l, w_h, w_l, B, H, W, Cin, taps, n_out, n_mma, reinterpret_cast<__nv_bfloat16*>(y),
                                                 ldy, bias, nullptr, out_scale, dev_out_scale, stream, "ptb_conv_tc_f16x2_half_out");
}

extern "C" int ptb_split_f16_from_bf16(const void* x, int64_t n, void* hi, void* lo, float* dev_inv_scale, void* workspace, void* stream) {
  PTB_REQUIRE(n >= 0 && n % 8 == 0, "n must be a multiple of 8");
  PTB_REQUIRE(((uintptr_t)x % 16 == 0) && ((uintptr_t)hi % 16 == 0) && ((uintptr_t)lo % 16 == 0), "16-byte alignment");
  PTB_REQUIRE(workspace && dev_inv_scale, "a 4-byte workspace and dev_inv_scale are required");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  long long blocks = (n / 8 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  unsigned int* amax = reinterpret_cast<unsigned int*>(workspace);
  if (cudaMemsetAsync(amax, 0, 4, st) != cudaSuccess) return fail("%s", "ptb_split_f16_from_bf16: cudaMemsetAsync failed");
  amax_abs_bf16_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 8, amax);
  if (int rc = check_launch("ptb_split_f16_from_bf16/amax")) return rc;
  split_f16_from_bf16_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 8, amax, reinterpret_cast<uint4*>(hi),
                                                              reinterpret_cast<uint4*>(lo), dev_inv_scale);
  return check_launch("ptb_split_f16_from_bf16");
}

extern "C" int ptb_gn_relu_apply_f16(const float* y, const double* gn_stats, const float* gamma, const float* beta, int B, int HW,
                                     int C, int groups, float eps, int relu, void* out_h, void* out_l, int* overflow_flag,
                                     void* stream) {
  PTB_REQUIRE(B > 0 && HW > 0 && C > 0 && groups > 0 && C % groups == 0, "shape");
  PTB_REQUIRE((C / groups) % 4 == 0 && C % 4 == 0, "channels per group must be a multiple of 4");
  PTB_REQUIRE(y && gn_stats && gamma && beta && out_h && out_l, "NULL input");
  const int cpg = C / groups;
  if (C % 8 == 0 && cpg % 8 == 0 && C <= 2048 && 256 % (C / 8) == 0 && ((uintptr_t)y % 32 == 0) && ((uintptr_t)out_h % 16 == 0) &&
      ((uintptr_t)out_l % 16 == 0)) {
    const int ppp2 = 2 * (256 / (C / 8));                         // pixels per CTA and double-pass
    int chunks = (sm_count() * 4 + B - 1) / B;                   // one wave of 4 CTAs (64 regs x 256 thr) per SM over all images
    int pix_per_cta = (HW + chunks - 1) / chunks;
    pix_per_cta = ((pix_per_cta + ppp2 - 1) / ppp2) * ppp2;
    chunks = (HW + pix_per_cta - 1) / pix_per_cta;
    gn_relu_apply_f16_v8_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(y), gn_stats, gamma, beta, HW, C, groups, eps, relu, pix_per_cta,
        reinterpret_cast<uint4*>(out_h), reinterpret_cast<uint4*>(out_l), overflow_flag);
    return check_launch("ptb_gn_relu_apply_f16");
  }
  const long long n4 = (long long)B * HW * C / 4;
  long long blocks = (n4 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  gn_relu_apply_f16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(y), gn_stats, gamma, beta,
                                                                              HW, C, groups, eps, relu, n4,
                                                                              reinterpret_cast<uint2*>(out_h),
                                                                              reinterpret_cast<uint2*>(out_l), overflow_flag);
  return check_launch("ptb_gn_relu_apply_f16");
}

extern "C" int ptb_gn_relu_apply(const float* y, const double* gn_stats, const float* gamma, const float* beta, int B, int HW,
                                 int C, int groups, float eps, int relu, float* out_hi, float* out_lo, void* stream) {
  PTB_REQUIRE(B > 0 && HW > 0 && C > 0 && groups > 0 && C % groups == 0, "shape");
  PTB_REQUIRE((C / groups) % 4 == 0 && C % 4 == 0, "channels per group must be a multiple of 4");
  PTB_REQUIRE(y && gn_stats && gamma && beta && out_hi, "NULL input");
  const long long n4 = (long long)B * HW * C / 4;
  long long blocks = (n4 + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  gn_relu_apply_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(y), gn_stats, gamma, beta,
                                                                          HW, C, groups, eps, relu, n4,
                                                                          reinterpret_cast<float4*>(out_hi),
                                                                          reinterpret_cast<float4*>(out_lo));
  return check_launch("ptb_gn_relu_apply");
}
