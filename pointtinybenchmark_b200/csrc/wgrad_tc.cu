// Weight gradient of the tower's conv3x3 (256 -> 256, stride 1, pad 1) on the Hopper tensor cores (wgmma), fp32-accurate:
//     dW[co][ci][kh][kw] = sum_{b,h,w} dy[b][h][w][co] * x[b][h+kh-1][w+kw-1][ci]          (autograd of cpr_head.py:1033-1043's convs)
// A GEMM with M = co, N = ci and K = PIXELS: both operands are channels-last activations, i.e. their contiguous dimension is
// M / N, not K.  wgmma reads such "MN-major" fp16 operands directly (the transpose immediates of wgmma.mma_async; canonical layout
// of 64-element x 8-deep SWIZZLE_128B atoms), so no transpose pass:
//   * a 4-D TMA box {64 channels, 16 w, 2 h, 1 image} of fp16 lands in shared memory as 32 pixel rows of 128 B with the
//     SWIZZLE_128B XOR — exactly one MN-major atom column (64 channels) x 4 K-atoms (8 pixels each, SBO = 1024 B);
//     128 channels = 2 such boxes (LBO = 4096 B).  The x box is fetched at the tap-shifted origin; its out-of-bounds part (the
//     conv's zero padding, partial edge tiles) is zero-filled by the TMA unit, and dy's out-of-image rows are zero too, so edge
//     tiles need no masks.
//   * fp32 accuracy as in conv_tc.cu: dy*s1 = h + l and x*s2 = h + l as fp16 pairs, h*h -> main accumulator, l*h + h*l ->
//     correction accumulator, summed in fp32 at the end.
//   * the tensor core adds into the fp32 accumulator without round-to-nearest (see conv_tc.cu); over the thousands of accumulation
//     steps of a pixel split that would be a visible error on dW.  The main accumulator is therefore FLUSHED every WG_FLUSH pixel
//     blocks: the MMA warpgroups store it as one more fp32 partial and restart it from zero; the correction accumulator is 2^-11
//     smaller and runs through.  The reduction kernel adds runs and splits with round-to-nearest fp32 adds in a fixed order.
//   * work: 2 co halves x 2 ci halves x 9 taps x S pixel splits = 36*S CTAs (S chosen so the CTAs fill whole waves of the SMs);
//     a CTA streams its pixel blocks through a 6 x 32 KB mbarrier ring (warpgroup 0: TMA producer, warpgroups 1 and 2: 64 output
//     channels each, two 64 x 128 fp32 accumulators in registers) and writes 128 x 128 fp32 partials; `wgrad_reduce_kernel` adds
//     the partials in a fixed order, applies the (power-of-two) inverse operand scales and writes OIHW.  Deterministic.
#include "tc_ptx.cuh"
#include <stdlib.h>

namespace ptb {

constexpr int WG_PX = 32;                         // pixels per K-block: box {64 ch, 16 w, 2 h}
constexpr int WG_TW = 16, WG_TH = 2;
constexpr int WG_STAGES = 6;
constexpr uint32_t WG_BOX_BYTES = WG_PX * 128;    // 4 KB: 32 pixel rows x 64 fp16 channels
constexpr uint32_t WG_OP_BYTES = 2 * WG_BOX_BYTES;  // 128 channels of one operand half (hi or lo)
constexpr uint32_t WG_STAGE_BYTES = 4 * WG_OP_BYTES;  // dy hi, dy lo, x hi, x lo: 32 KB
constexpr uint32_t WG_SMEM_BYTES = WG_STAGES * WG_STAGE_BYTES + 1024 + 256;
constexpr int WG_THREADS = 384;
constexpr int WG_C = 256;                         // Cout = Cin = 256
constexpr int WG_FLUSH = 128;                     // pixel blocks (256 accumulation steps) between two flushes of the main accumulator

// Accumulation runs of a pixel split: the FIRST run of split s is shortened to WG_FLUSH * (s + 1) / splits blocks, later runs have WG_FLUSH
// blocks.  All CTAs stream at the same pace, so equal runs would make them all flush their accumulators in the same few microseconds;
// staggered, the splits flush 1/splits of a run apart and the stores of one hide behind the MMAs of the others.
__host__ __device__ inline int wg_first_run(int split, int splits) {
  const int f = (int)(((long long)WG_FLUSH * (split + 1)) / splits);
  return f < 1 ? 1 : f;
}
__host__ __device__ inline int wg_runs(int n_my, int first) {
  if (n_my <= 0) return 0;
  return n_my <= first ? 1 : 1 + (n_my - first + WG_FLUSH - 1) / WG_FLUSH;
}

struct WgradShape {
  int B, H, W;
  int tiles_h, tiles_w, n_blocks;    // pixel blocks of 16 x 2
  int splits;
  int max_runs;                      // partial slots per split (upper bound of wg_runs())
  int taps;                          // 9: conv3x3 (pad 1), 1: conv1x1 / per-cell Linear (CPRHead's cls_out / ins_out logit map)
  int Cout;                          // rows of dW actually wanted (<= 256); rows beyond it are the TMA unit's zero fill of dy
};

__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_dyh, const __grid_constant__ CUtensorMap tm_dyl,
                const __grid_constant__ CUtensorMap tm_xh, const __grid_constant__ CUtensorMap tm_xl, WgradShape ws,
                float* __restrict__ partial /*[splits][max_runs][taps][256 co][256 ci]*/) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;     // SWIZZLE_128B atoms need 1024 B alignment
  const uint32_t bar_base = smem_base + WG_STAGES * WG_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };

  const int wg = threadIdx.x >> 7;
  // unit = (split, tap, ci half, co half)
  const int unit = blockIdx.x;
  const int m_half = unit & 1, n_half = (unit >> 1) & 1;
  const int tap = (unit >> 2) % ws.taps;
  const int split = unit / (4 * ws.taps);
  const int kh = ws.taps == 9 ? tap / 3 : 1, kw = ws.taps == 9 ? tap - (tap / 3) * 3 : 1;
  const int blk0 = (int)(((long long)ws.n_blocks * split) / ws.splits);
  const int blk1 = (int)(((long long)ws.n_blocks * (split + 1)) / ws.splits);
  const int n_my = blk1 - blk0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);                    // one arrive per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // =============================== TMA producer ===============================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int per_img = ws.tiles_h * ws.tiles_w;
      int b = blk0 / per_img;
      int th = (blk0 - b * per_img) / ws.tiles_w;
      int tw = (blk0 - b * per_img) - th * ws.tiles_w;
      for (int blk = blk0; blk < blk1; ++blk) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const int h0 = th * WG_TH, w0 = tw * WG_TW;
        const uint32_t sA_h = smem_base + stage * WG_STAGE_BYTES;
        const uint32_t sA_l = sA_h + WG_OP_BYTES;
        const uint32_t sB_h = sA_l + WG_OP_BYTES;
        const uint32_t sB_l = sB_h + WG_OP_BYTES;
        mbar_expect_tx(full_bar(stage), WG_STAGE_BYTES);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          tma_load_4d(&tm_dyh, full_bar(stage), sA_h + i * WG_BOX_BYTES, m_half * 128 + 64 * i, w0, h0, b);
          tma_load_4d(&tm_dyl, full_bar(stage), sA_l + i * WG_BOX_BYTES, m_half * 128 + 64 * i, w0, h0, b);
          tma_load_4d(&tm_xh, full_bar(stage), sB_h + i * WG_BOX_BYTES, n_half * 128 + 64 * i, w0 + kw - 1, h0 + kh - 1, b);
          tma_load_4d(&tm_xl, full_bar(stage), sB_l + i * WG_BOX_BYTES, n_half * 128 + 64 * i, w0 + kw - 1, h0 + kh - 1, b);
        }
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1u; }
        if (++tw == ws.tiles_w) { tw = 0; if (++th == ws.tiles_h) { th = 0; ++b; } }
      }
    }
  } else {
    // =============================== MMA + flushes (warpgroups 1, 2) ===============================
    regs_alloc<232>();
    const int cw = wg - 1;                                   // output channels m_half * 128 + 64 cw .. + 63
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    float acc[64], cor[64];
    int stage = 0;
    uint32_t phase = 0;
    const int co = m_half * 128 + cw * 64 + warp * 16 + (lane >> 2);
    const int ci = n_half * 128 + 2 * (lane & 3);
    int it = 0;
    for (int run = 0; it < n_my; ++run) {
      const int run_len = min(run == 0 ? wg_first_run(split, ws.splits) : WG_FLUSH, n_my - it);
      int prev = 0;
      for (int r = 0; r < run_len; ++r, ++it) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sA_h = smem_base + stage * WG_STAGE_BYTES + (uint32_t)cw * WG_BOX_BYTES;
        const uint32_t sA_l = sA_h + WG_OP_BYTES;
        const uint32_t sB_h = smem_base + stage * WG_STAGE_BYTES + 2 * WG_OP_BYTES;
        const uint32_t sB_l = sB_h + WG_OP_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_PX / 16; ++k) {               // 16 pixels per MMA = two 8-deep atoms = 2048 B
          const uint64_t a_h = gmma_desc(sA_h + 2048u * k, WG_BOX_BYTES, 1024u, GMMA_SW128);
          const uint64_t a_l = gmma_desc(sA_l + 2048u * k, WG_BOX_BYTES, 1024u, GMMA_SW128);
          const uint64_t b_h = gmma_desc(sB_h + 2048u * k, WG_BOX_BYTES, 1024u, GMMA_SW128);
          const uint64_t b_l = gmma_desc(sB_l + 2048u * k, WG_BOX_BYTES, 1024u, GMMA_SW128);
          wgmma_f16<1, 1>(acc, a_h, b_h, (r | k) != 0);
          wgmma_f16<1, 1>(cor, a_l, b_h, (it | k) != 0);
          wgmma_f16<1, 1>(cor, a_h, b_l, 1u);
        }
        wgmma_commit();
        if (r > 0) {                                         // the previous block's MMAs have read their stage: hand it back
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stage;
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      // run complete: store it as one partial (the last run adds the correction accumulator)
      const bool last = it == n_my;
      float* out = partial + ((((size_t)split * ws.max_runs + run) * ws.taps + tap) * WG_C + co) * WG_C + ci;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float2 o = make_float2(acc[4 * i + 2 * j], acc[4 * i + 2 * j + 1]);
          if (last) { o.x = __fadd_rn(o.x, cor[4 * i + 2 * j]); o.y = __fadd_rn(o.y, cor[4 * i + 2 * j + 1]); }
          __stcg(reinterpret_cast<float2*>(out + (size_t)8 * j * WG_C + 8 * i), o);     // L2-resident: the reduction re-reads it
        }
      }
    }
  }
}

// dw[co][ci][tap] = scale * sum_{split, run} partial[split][run][tap][co][ci]   (fixed order; scale = product of the inverse
// operand scales).  A split owns blocks [n*s/S, n*(s+1)/S) and has wg_runs() runs (0 for an empty split).
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ partial, WgradShape ws, float scale, const float* __restrict__ dev_scale_a,
                    const float* __restrict__ dev_scale_b, float* __restrict__ dw, int accumulate) {
  const int i = blockIdx.x * 256 + threadIdx.x;      // over [tap][co][ci]
  if (i >= ws.taps * WG_C * WG_C) return;
  const int ci = i % WG_C, co = (i / WG_C) % WG_C, tap = i / (WG_C * WG_C);
  if (co >= ws.Cout) return;
  const size_t slot = (size_t)ws.taps * WG_C * WG_C;
  float s = 0.f;
  for (int k = 0; k < ws.splits; ++k) {
    const int n_my = (int)(((long long)ws.n_blocks * (k + 1)) / ws.splits) - (int)(((long long)ws.n_blocks * k) / ws.splits);
    const int runs = wg_runs(n_my, wg_first_run(k, ws.splits));
    for (int r = 0; r < runs; ++r) s += __ldcg(partial + ((size_t)k * ws.max_runs + r) * slot + i);
  }
  float sc = scale;
  if (dev_scale_a) sc *= *dev_scale_a;
  if (dev_scale_b) sc *= *dev_scale_b;
  float* o = dw + ((size_t)co * WG_C + ci) * ws.taps + tap;
  *o = accumulate ? *o + s * sc : s * sc;
}

// column sums of a row-major [M][ld] matrix (bias gradient of the logit-map Linear): per-slice partials, then reduce_cols in slice order
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ y, long long M, int N, int ld, int rows_per_slice, float* __restrict__ part /*[slices][N]*/) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  const long long m0 = (long long)blockIdx.y * rows_per_slice;
  long long m1 = m0 + rows_per_slice;
  if (m1 > M) m1 = M;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;      // four independent chains (fixed association: deterministic)
  long long m = m0;
  for (; m + 3 < m1; m += 4) {
    a0 += y[m * ld + n]; a1 += y[(m + 1) * ld + n]; a2 += y[(m + 2) * ld + n]; a3 += y[(m + 3) * ld + n];
  }
  for (; m < m1; ++m) a0 += y[m * ld + n];
  part[(size_t)blockIdx.y * N + n] = (a0 + a1) + (a2 + a3);
}
__global__ void __launch_bounds__(256) colsum_reduce_kernel(const float* __restrict__ part, int slices, int N, float* __restrict__ out) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float s = 0.f;
  for (int i = 0; i < slices; ++i) s += part[(size_t)i * N + n];
  out[n] = s;
}

// C channels of pixel rows `ld` fp16 apart (ld = C: dense); channels past C read as zeros (TMA out-of-bounds fill)
static int make_px_map(CUtensorMap* tm, const void* ptr, int B, int H, int W, int C, int ld) {
  EncodeTiledFn enc = tc_get_encode();
  if (!enc) return fail("%s", "cuTensorMapEncodeTiled is unavailable (driver too old?)");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
  cuuint32_t box[4] = {64, WG_TW, WG_TH, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled(wgrad operand) failed: %s%lld", "", (long long)r);
  return 0;
}

}  // namespace ptb

using namespace ptb;

// pixel splits: 4 * taps * S CTAs of one block each per SM; S is picked for the least wave-quantised time ceil(CTAs / SMs) / S
static int wgrad_splits(int taps) {
  const int sms = sm_count(), units = 4 * taps;
  int s_max = 4 * (sms / units > 1 ? sms / units : 1);
  if (s_max > 96) s_max = 96;
  int best = 1;
  for (int s = 2; s <= s_max; ++s)
    if ((long long)((units * s + sms - 1) / sms) * best < (long long)((units * best + sms - 1) / sms) * s) best = s;
  return best;
}

static int wgrad_max_runs(int n_blocks, int splits) {
  const int per_split = (n_blocks + splits - 1) / splits;
  return 1 + (per_split + WG_FLUSH - 1) / WG_FLUSH;      // upper bound of wg_runs(): a shortened first run + full runs
}

static uint64_t wgrad_ws_bytes(int B, int H, int W, int taps) {
  if (B <= 0 || H <= 0 || W <= 0 || (taps != 1 && taps != 9)) return 0;
  const int n_blocks = B * ((H + WG_TH - 1) / WG_TH) * ((W + WG_TW - 1) / WG_TW);
  const int splits = wgrad_splits(taps);
  return (uint64_t)splits * wgrad_max_runs(n_blocks, splits) * taps * WG_C * WG_C * sizeof(float);
}

extern "C" uint64_t ptb_conv_tc_wgrad_workspace(int B, int H, int W, int taps) { return wgrad_ws_bytes(B, H, W, taps); }

static int wgrad_run(const void* dy_h, const void* dy_l, int ld_dy, const void* x_h, const void* x_l, int B, int H, int W, int Cout, int Cin,
                     int taps, float scale, const float* dev_scale_dy, const float* dev_scale_x, void* workspace, float* dw, int accumulate,
                     void* stream) {
  const char* what = "ptb_conv_tc_wgrad_f16x2_ld";
  CUtensorMap tm_dyh, tm_dyl, tm_xh, tm_xl;
  int rc;
  if ((rc = make_px_map(&tm_dyh, dy_h, B, H, W, Cout, ld_dy))) return rc;
  if ((rc = make_px_map(&tm_dyl, dy_l, B, H, W, Cout, ld_dy))) return rc;
  if ((rc = make_px_map(&tm_xh, x_h, B, H, W, Cin, Cin))) return rc;
  if ((rc = make_px_map(&tm_xl, x_l, B, H, W, Cin, Cin))) return rc;
  WgradShape ws;
  ws.B = B; ws.H = H; ws.W = W;
  ws.tiles_h = (H + WG_TH - 1) / WG_TH;
  ws.tiles_w = (W + WG_TW - 1) / WG_TW;
  ws.n_blocks = B * ws.tiles_h * ws.tiles_w;
  ws.splits = wgrad_splits(taps);
  ws.max_runs = wgrad_max_runs(ws.n_blocks, ws.splits);
  ws.taps = taps; ws.Cout = Cout;
  // per-device function attribute: set on every call (a process may drive several devices)
  if (cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM_BYTES) != cudaSuccess)
    return fail("%s", "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed for the wgrad kernel");
  cudaStream_t st = (cudaStream_t)stream;
  // CTAs of the upper co half have nothing to do when Cout <= 128: they still run (zero operands) to keep the unit decomposition uniform
  wgrad_tc_kernel<<<4 * taps * ws.splits, WG_THREADS, WG_SMEM_BYTES, st>>>(tm_dyh, tm_dyl, tm_xh, tm_xl, ws, reinterpret_cast<float*>(workspace));
  if ((rc = check_launch(what))) return rc;
  const int n = taps * WG_C * WG_C;
  wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float*>(workspace), ws, scale, dev_scale_dy,
                                                      dev_scale_x, dw, accumulate);
  return check_launch(what);
}

extern "C" int ptb_conv_tc_wgrad_f16x2_ld(const void* dy_h, const void* dy_l, int ld_dy, const void* x_h, const void* x_l, int B, int H,
                                          int W, int Cout, int Cin, int taps, float scale, const float* dev_scale_dy,
                                          const float* dev_scale_x, void* workspace, float* dw, int accumulate, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && (taps == 1 || taps == 9), "shape");
  PTB_REQUIRE(Cin == WG_C && Cout > 0 && Cout <= WG_C && Cout % 8 == 0, "Cin must be 256, Cout a multiple of 8 up to 256");
  PTB_REQUIRE(ld_dy >= Cout && ld_dy % 8 == 0, "ld_dy must be a multiple of 8 and >= Cout");
  PTB_REQUIRE(dy_h && dy_l && x_h && x_l && workspace && dw, "NULL input");
  PTB_REQUIRE(((uintptr_t)dy_h % 16 == 0) && ((uintptr_t)dy_l % 16 == 0) && ((uintptr_t)x_h % 16 == 0) && ((uintptr_t)x_l % 16 == 0) &&
                  ((uintptr_t)workspace % 16 == 0), "16-byte alignment");
  return wgrad_run(dy_h, dy_l, ld_dy, x_h, x_l, B, H, W, Cout, Cin, taps, scale, dev_scale_dy, dev_scale_x, workspace, dw, accumulate,
                   stream);
}

extern "C" uint64_t ptb_col_sum_workspace(int64_t M, int N) {
  if (M <= 0 || N <= 0) return 0;
  return (uint64_t)SCRATCH_BLOCKS * N * sizeof(float);
}

extern "C" int ptb_col_sum(const float* y, int64_t M, int N, int ld, float* workspace, float* out, void* stream) {
  PTB_REQUIRE(M > 0 && N > 0 && ld >= N, "shape");
  PTB_REQUIRE(y && workspace && out, "NULL input");
  int slices = SCRATCH_BLOCKS;
  if ((int64_t)slices > M) slices = (int)M;
  const int rps = (int)((M + slices - 1) / slices);
  slices = (int)((M + rps - 1) / rps);
  cudaStream_t st = (cudaStream_t)stream;
  colsum_partial_kernel<<<dim3((N + 255) / 256, slices), 256, 0, st>>>(y, M, N, ld, rps, workspace);
  int rc = check_launch("ptb_col_sum/partial");
  if (rc) return rc;
  colsum_reduce_kernel<<<(N + 255) / 256, 256, 0, st>>>(workspace, slices, N, out);
  return check_launch("ptb_col_sum");
}
