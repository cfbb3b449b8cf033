// Neighbor (bag) gather over channels-last maps — forward and backward.
// Replaces cpr_head.py:182-199 + 73-93 (extract_point_feat / grid_sample), 453-497 (CirclePtFeatGenerator) and
// 172-180 (get_point_valid) of the reference, for ALL images and bags of a batch in one launch.
//
// Layout / mapping (HBM-bound kernel; algorithmic bytes = map + coords in, G*K*C*4 out):
//   * a warp owns a group of 32 consecutive samples (flattened g*K+k); lane j derives the 4 taps + weights of
//     sample j ONCE (fp32 coordinate pipeline identical to ATen's), writes pts/valid for it;
//   * the warp then walks the flattened (sample, float4-channel-group) space 32 lanes at a time, fetching the
//     sample's taps from a per-warp shared-memory table (3 broadcast reads; the first version pulled them from the
//     owning lane with 10 shuffles per step, and the L1 data pipe — which also executes shuffles — spent a large share of
//     its wavefronts on them): every 128-bit load reads a contiguous channels-last run
//     (1 KB per tap at C=256) and every 128-bit store lands in a contiguous output row -> fully coalesced both ways;
//   * map reads go through the read-only path (L1-cached: neighbouring samples of a bag share taps, the map of one
//     image (17 MB) stays L2 resident); output uses streaming stores.
#include "tc_ptx.cuh"
#include <stdlib.h>
#include <string.h>

namespace ptb {

// dynamic chunk scheduler state lives in the per-stream scratch block (ptb_common.cuh): self-resetting — the last CTA to drain
// restores both counters, so consecutive launches on one stream need no memset, and launches on different streams do not share it.

constexpr int GATHER_CHUNK = 256;   // samples per CTA work item (8 warps x 32 samples)

template <int CG_T>  // CG_T = C/4 when known at compile time (64, 40, 20), 0 = runtime
__global__ void __launch_bounds__(256)
bag_gather_kernel(const float* __restrict__ map, int H, int W, int C, int ld,
                  const float* __restrict__ centers, const int32_t* __restrict__ bag_img, long long S /*=G*K*/, int K,
                  const float* __restrict__ offsets, float stride, const int32_t* __restrict__ pad_hw,
                  float* __restrict__ out_feats, float* __restrict__ out_pts, uint8_t* __restrict__ out_valid,
                  StreamScratch* __restrict__ sched) {
  const int CG = CG_T ? CG_T : (C >> 2);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned int n_chunks = (unsigned int)((S + GATHER_CHUNK - 1) / GATHER_CHUNK);
  const size_t img_cells = (size_t)H * W;
  __shared__ unsigned int s_chunk;
  __shared__ int4 s_off[8][32];        // per warp: tap cell offsets of its 32 samples
  __shared__ float4 s_wgt[8][32];      //           tap weights (nw, ne, sw, se)
  __shared__ long long s_cb[8][32];    //           first cell of the sample's image

  for (;;) {
    if (threadIdx.x == 0) s_chunk = atomicAdd(&sched->gather_ticket, 1u);
    __syncthreads();
    const unsigned int chunk = s_chunk;
    __syncthreads();
    if (chunk >= n_chunks) break;
    // The 8 warps of the CTA interleave over the chunk's 256 consecutive samples: lane j of warp w owns sample
    // base + 8*j + w, so at any moment the warps work on ring-adjacent samples that share bilinear taps -> the
    // CTA's live window stays L1 resident (hit rate ~2x the one-warp-per-32-samples mapping).
    const long long base = (long long)chunk * GATHER_CHUNK;
    const long long s_mine = base + 8 * lane + wid;
    Taps t;
    t.o00 = t.o01 = t.o10 = t.o11 = 0;
    t.w00 = t.w01 = t.w10 = t.w11 = 0.f;
    long long cell_base = 0;  // (b*H*W) in cells
    if (s_mine < S) {
      const int g = (int)(s_mine / K);
      const int k = (int)(s_mine - (long long)g * K);
      const int b = bag_img[g];
      const float px = __fadd_rn(offsets[2 * k], centers[2 * g]);       // cpr_head.py:492  off + centre
      const float py = __fadd_rn(offsets[2 * k + 1], centers[2 * g + 1]);
      t = make_taps(px, py, stride, H, W);
      cell_base = (long long)b * img_cells;
      if (out_pts) {
        float* p = out_pts + s_mine * 3;
        p[0] = px; p[1] = py; p[2] = stride;
      }
      if (out_valid) {
        const float ph = (float)pad_hw[2 * b], pw = (float)pad_hw[2 * b + 1];
        out_valid[s_mine] = (0.f <= px) && (px < pw) && (0.f <= py) && (py < ph);   // cpr_head.py:179
      }
    }
    if (!out_feats) continue;
    s_off[wid][lane] = make_int4(t.o00, t.o01, t.o10, t.o11);
    s_wgt[wid][lane] = make_float4(t.w00, t.w01, t.w10, t.w11);
    s_cb[wid][lane] = cell_base;
    __syncwarp();
    // number of this warp's samples inside S
    const long long rem = S - base - wid;
    const int n_mine = rem <= 0 ? 0 : (int)min((long long)32, (rem + 7) / 8);
    const int total = n_mine * CG;
    if constexpr (CG_T > 0 && CG_T % 32 == 0) {
      // whole samples per step (C = 256: two 512-byte halves): the tap record is read once per sample and the 4 x CG_T/32
      // loads of a sample are issued back to back
#pragma unroll 2
      for (int sidx = 0; sidx < n_mine; ++sidx) {
        const long long cb = s_cb[wid][sidx];
        const int4 o4 = s_off[wid][sidx];
        const float4 w4 = s_wgt[wid][sidx];
        const float* mb = map + (size_t)cb * ld + 4 * lane;
        const float* p00 = mb + (size_t)o4.x * ld;
        const float* p01 = mb + (size_t)o4.y * ld;
        const float* p10 = mb + (size_t)o4.z * ld;
        const float* p11 = mb + (size_t)o4.w * ld;
        float* dst = out_feats + (size_t)(base + 8 * sidx + wid) * C + 4 * lane;
#pragma unroll
        for (int it = 0; it < (CG_T > 0 ? CG_T / 32 : 1); ++it) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(p00 + 128 * it));
          const float4 bq = __ldg(reinterpret_cast<const float4*>(p01 + 128 * it));
          const float4 c = __ldg(reinterpret_cast<const float4*>(p10 + 128 * it));
          const float4 d = __ldg(reinterpret_cast<const float4*>(p11 + 128 * it));
          const float4 r = bilerp4(a, bq, c, d, w4.x, w4.y, w4.z, w4.w);   // ATen's FMA chain, bit-exact vs the CPU kernel
          st_cs(reinterpret_cast<float4*>(dst + 128 * it), r);
        }
      }
    } else {
#pragma unroll 2
    for (int idx = lane; idx < ((total + 31) & ~31); idx += 32) {
      const bool act = idx < total;
      const int sidx = act ? idx / CG : 0;
      const int cg = idx - sidx * CG;
      const long long cb = s_cb[wid][sidx];
      const int4 o4 = s_off[wid][sidx];
      const float4 w4 = s_wgt[wid][sidx];
      const int o00 = o4.x, o01 = o4.y, o10 = o4.z, o11 = o4.w;
      const float w00 = w4.x, w01 = w4.y, w10 = w4.z, w11 = w4.w;
      if (act) {
        const float* mb = map + (size_t)cb * ld + 4 * cg;
        const float4 a = __ldg(reinterpret_cast<const float4*>(mb + (size_t)o00 * ld));
        const float4 bq = __ldg(reinterpret_cast<const float4*>(mb + (size_t)o01 * ld));
        const float4 c = __ldg(reinterpret_cast<const float4*>(mb + (size_t)o10 * ld));
        const float4 d = __ldg(reinterpret_cast<const float4*>(mb + (size_t)o11 * ld));
        const float4 r = bilerp4(a, bq, c, d, w00, w01, w10, w11);   // ATen's FMA chain, bit-exact vs the CPU kernel
        float* dst = out_feats + (size_t)(base + 8 * sidx + wid) * C + 4 * cg;
        st_cs(reinterpret_cast<float4*>(dst), r);
      }
    }
    }
  }
  // self-reset of the scheduler
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&sched->gather_done, 1u) == gridDim.x - 1) {
      sched->gather_ticket = 0;
      sched->gather_done = 0;
      __threadfence();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// TMA-staged variant (round 2).  Work item = (bag, channel chunk of CC = 64 or 32 channels): ONE cp.async.bulk.tensor box
// {CC channels, WS, WS, 1 image} brings the bag's (2r+2)^2-cell window of the chunk into shared memory (83 KB at CC = 64, r = 8); the
// 289 x 4 tap reads are then shared-memory reads.  Why: the LDG version is limited by the L1 data pipe (a warp-wide LDG.128 that touches 4 lines costs ~2 cycles per line, ~62 B/clk, while this kernel needs 4 tap bytes per output byte);
// LDS serves 128 B/clk and the window moves 1.33 GB through L2 instead of the ~2.4 GB of L1 misses.  Two CTAs per SM overlap one's
// box load with the other's interpolation.  Bags whose window does not fit (rounding straddle) read global memory in the same code.
// Outputs are bit-identical to bag_gather_kernel (same tap arithmetic, same FMA chain).
// ---------------------------------------------------------------------------------------------------------------------------------
struct GtTap { int o[4]; float w[4]; };      // tap offsets in floats relative to the addressed array (window or image), weights

template <int CC>
__global__ void __launch_bounds__(256, 2)
bag_gather_tma_kernel(const __grid_constant__ CUtensorMap tm_map, int WS, float reach_px, const float* __restrict__ map, int H, int W,
                      int C, int ld, const float* __restrict__ centers, const int32_t* __restrict__ bag_img, int K,
                      const float* __restrict__ offsets, float stride, const int32_t* __restrict__ pad_hw,
                      float* __restrict__ out_feats, float* __restrict__ out_pts, uint8_t* __restrict__ out_valid) {
  extern __shared__ uint8_t sm_raw[];
  const uint32_t raw = smem_u32(sm_raw);
  const uint32_t win = (raw + 127u) & ~127u;
  const size_t win_bytes = (size_t)WS * WS * CC * sizeof(float);
  GtTap* s_tap = reinterpret_cast<GtTap*>(sm_raw + (win - raw) + win_bytes);
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_staged, s_ox, s_oy;
  const int n_cc = C / CC;
  const int g = blockIdx.x / n_cc, cc = blockIdx.x - g * n_cc;
  const int b = bag_img[g];
  const float cxg = centers[2 * g], cyg = centers[2 * g + 1];
  const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
  const uint32_t bar = smem_u32(&s_bar);
  if (threadIdx.x == 0) {
    const float xl = sample_coord(__fadd_rn(-reach_px, cxg), stride, (float)W, hw), xr = sample_coord(__fadd_rn(reach_px, cxg), stride, (float)W, hw);
    const float yl = sample_coord(__fadd_rn(-reach_px, cyg), stride, (float)H, hh), yr = sample_coord(__fadd_rn(reach_px, cyg), stride, (float)H, hh);
    const int ox = (int)floorf(xl), oy = (int)floorf(yl);
    const int x_hi = min((int)floorf(xr) + 1, W - 1), y_hi = min((int)floorf(yr) + 1, H - 1);
    const int staged = (x_hi - ox + 1 <= WS) && (y_hi - oy + 1 <= WS);
    if (staged) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      mbar_expect_tx(bar, (uint32_t)win_bytes);
      tma_load_4d(&tm_map, bar, win, cc * CC, ox, oy, b);
    }
    s_staged = staged; s_ox = ox; s_oy = oy;
  }
  __syncthreads();
  const bool staged = s_staged != 0;
  const int ox = s_ox, oy = s_oy;
  // tap table (runs under the box load); chunk 0 also writes the points / validity of the bag
  for (int k = threadIdx.x; k < K; k += 256) {
    const float px = __fadd_rn(offsets[2 * k], cxg), py = __fadd_rn(offsets[2 * k + 1], cyg);
    const Taps t = make_taps(px, py, stride, H, W);
    GtTap r;
    const int o[4] = {t.o00, t.o01, t.o10, t.o11};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int y = o[i] / W, x = o[i] - y * W;
      r.o[i] = staged ? ((y - oy) * WS + (x - ox)) * CC : o[i] * ld + cc * CC;
    }
    r.w[0] = t.w00; r.w[1] = t.w01; r.w[2] = t.w10; r.w[3] = t.w11;
    s_tap[k] = r;
    if (cc == 0) {
      const size_t sidx = (size_t)g * K + k;
      if (out_pts) { float* p = out_pts + sidx * 3; p[0] = px; p[1] = py; p[2] = stride; }
      if (out_valid) {
        const float ph = (float)pad_hw[2 * b], pw = (float)pad_hw[2 * b + 1];
        out_valid[sidx] = (0.f <= px) && (px < pw) && (0.f <= py) && (py < ph);   // cpr_head.py:179
      }
    }
  }
  __syncthreads();
  if (!out_feats) { if (staged) mbar_wait(bar, 0u); return; }     // (never exit with a bulk copy in flight)
  if (staged) mbar_wait(bar, 0u);
  constexpr int GP = CC / 4;                 // float4 groups per sample chunk (16 or 8)
  constexpr int SPW = 32 / GP;               // samples per warp instruction
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = lane % GP, sl = lane / GP;
  const float* gimg = map + (size_t)b * H * W * ld;
  float* obase = out_feats + (size_t)g * K * C + cc * CC + 4 * grp;
  for (int k0 = warp * SPW; k0 < K; k0 += 8 * SPW) {
    const int k = k0 + sl;
    if (k < K) {
      const GtTap t = s_tap[k];
      float4 q0, q1, q2, q3;
      if (staged) {
        const uint32_t a = win + 16u * (uint32_t)grp;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q0.x), "=f"(q0.y), "=f"(q0.z), "=f"(q0.w) : "r"(a + 4u * (uint32_t)t.o[0]));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q1.x), "=f"(q1.y), "=f"(q1.z), "=f"(q1.w) : "r"(a + 4u * (uint32_t)t.o[1]));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q2.x), "=f"(q2.y), "=f"(q2.z), "=f"(q2.w) : "r"(a + 4u * (uint32_t)t.o[2]));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q3.x), "=f"(q3.y), "=f"(q3.z), "=f"(q3.w) : "r"(a + 4u * (uint32_t)t.o[3]));
      } else {
        const float* a = gimg + 4 * grp;
        q0 = __ldg(reinterpret_cast<const float4*>(a + t.o[0])); q1 = __ldg(reinterpret_cast<const float4*>(a + t.o[1]));
        q2 = __ldg(reinterpret_cast<const float4*>(a + t.o[2])); q3 = __ldg(reinterpret_cast<const float4*>(a + t.o[3]));
      }
      st_cs(reinterpret_cast<float4*>(obase + (size_t)k * C), bilerp4(q0, q1, q2, q3, t.w[0], t.w[1], t.w[2], t.w[3]));
    }
  }
}

// backward: grad_map[b][tap][c] += w_tap * grad_out[g][k][c]   (vector atomics: red.global.add.v4.f32 on sm_90+)
__global__ void __launch_bounds__(256)
bag_gather_bwd_kernel(const float* __restrict__ grad_out, int H, int W, int C, int ld,
                      const float* __restrict__ centers, const int32_t* __restrict__ bag_img, long long S, int K,
                      const float* __restrict__ offsets, float stride, float* __restrict__ grad_map) {
  const int CG = C >> 2;
  const int lane = threadIdx.x & 31;
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long n_groups = (S + 31) >> 5;
  const size_t img_cells = (size_t)H * W;
  for (long long grp = warp_global; grp < n_groups; grp += n_warps) {
    const long long s_mine = grp * 32 + lane;
    Taps t;
    t.o00 = t.o01 = t.o10 = t.o11 = 0;
    t.w00 = t.w01 = t.w10 = t.w11 = 0.f;
    long long cell_base = 0;
    if (s_mine < S) {
      const int g = (int)(s_mine / K);
      const int k = (int)(s_mine - (long long)g * K);
      const float px = __fadd_rn(offsets[2 * k], centers[2 * g]);
      const float py = __fadd_rn(offsets[2 * k + 1], centers[2 * g + 1]);
      t = make_taps(px, py, stride, H, W);
      cell_base = (long long)bag_img[g] * img_cells;
    }
    const int n_in_grp = (int)min((long long)32, S - grp * 32);
    const int total = n_in_grp * CG;
    const float* go_base = grad_out + (size_t)grp * 32 * C;
    for (int idx = lane; idx < ((total + 31) & ~31); idx += 32) {
      const bool act = idx < total;
      const int sidx = act ? idx / CG : 0;
      const int cg = idx - sidx * CG;
      const long long cb = __shfl_sync(0xffffffffu, cell_base, sidx);
      const int o00 = __shfl_sync(0xffffffffu, t.o00, sidx), o01 = __shfl_sync(0xffffffffu, t.o01, sidx);
      const int o10 = __shfl_sync(0xffffffffu, t.o10, sidx), o11 = __shfl_sync(0xffffffffu, t.o11, sidx);
      const float w00 = __shfl_sync(0xffffffffu, t.w00, sidx), w01 = __shfl_sync(0xffffffffu, t.w01, sidx);
      const float w10 = __shfl_sync(0xffffffffu, t.w10, sidx), w11 = __shfl_sync(0xffffffffu, t.w11, sidx);
      if (act) {
        const float4 gq = __ldcs(reinterpret_cast<const float4*>(go_base + (size_t)idx * 4));
        float* base = grad_map + (size_t)cb * ld + 4 * cg;
        const int offs[4] = {o00, o01, o10, o11};
        const float ws[4] = {w00, w01, w10, w11};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (ws[q] != 0.f) {
            float4 v = make_float4(gq.x * ws[q], gq.y * ws[q], gq.z * ws[q], gq.w * ws[q]);
            atomicAdd(reinterpret_cast<float4*>(base + (size_t)offs[q] * ld), v);
          }
        }
      }
    }
  }
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_cpr_bag_gather(const float* map, int B, int H, int W, int C, int ld, const float* centers,
                                  const int32_t* bag_img, int G, const float* offsets, int K, float stride,
                                  float reach_px, const int32_t* pad_hw, float* out_feats, float* out_pts, uint8_t* out_valid,
                                  void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && K > 0 && G >= 0, "shape");
  PTB_REQUIRE(stride > 0.f, "stride");
  PTB_REQUIRE(!out_feats || (C % 4 == 0 && ld % 4 == 0 && ld >= C), "C and ld must be multiples of 4, ld >= C");
  PTB_REQUIRE(!out_feats || map, "map is NULL");
  PTB_REQUIRE(((uintptr_t)map % 16 == 0) && ((uintptr_t)out_feats % 16 == 0), "map/out_feats must be 16-byte aligned");
  PTB_REQUIRE(!out_valid || pad_hw, "pad_hw required for out_valid");
  if (G == 0) return 0;
  PTB_REQUIRE(centers && bag_img && offsets, "NULL input");
  const long long S = (long long)G * K;
  const long long n_chunks = (S + GATHER_CHUNK - 1) / GATHER_CHUNK;
  const int threads = 256;
  cudaStream_t st = (cudaStream_t)stream;
  const int CG = C / 4;
  // ---- TMA-staged variant: (bag, channel chunk) work items, the bag's window of the chunk in shared memory (PTB_GATHER_TMA=0: LDG kernel)
  const char* e_tma = getenv("PTB_GATHER_TMA");
  const char* e_cc = getenv("PTB_GATHER_CC");
  int CCk = (C % 64 == 0) ? 64 : ((C % 32 == 0) ? 32 : 0);
  if (e_cc && e_cc[0] == '3' && C % 32 == 0) CCk = 32;
  if (!e_cc && C % 32 == 0 && C < 256) CCk = 32;            // small windows: 4 CTAs per SM
  // The kernel is bound by the L1 / shared-memory data pipe either way (4 tap bytes read per byte written), and at C = 256 the two
  // 92 KB staging windows leave few warps resident per SM, so the staged form only pays where its windows are small.  Default: TMA for
  // C <= 192; tools/profile_gather2.py times both forms.
  const bool want_tma = e_tma ? (e_tma[0] != '0') : (C <= 192);
  if (want_tma && out_feats && reach_px > 0.f && CCk && (long long)G * (C / CCk) < (1ll << 31)) {
    const int WS = 2 * (int)ceilf(reach_px / stride) + 2;
    const size_t smem = (size_t)WS * WS * CCk * sizeof(float) + 128 + (size_t)K * sizeof(GtTap);
    EncodeTiledFn enc = tc_get_encode();
    if (WS <= 256 && smem <= 112 * 1024 && enc) {
      CUtensorMap tm;
      cuuint64_t dims[4] = {(cuuint64_t)ld, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4};
      cuuint32_t box[4] = {(cuuint32_t)CCk, (cuuint32_t)WS, (cuuint32_t)WS, 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(map), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS) {
        const unsigned grid = (unsigned)((long long)G * (C / CCk));
        if (CCk == 64) {
          if (cudaFuncSetAttribute(bag_gather_tma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return fail("%s", "ptb_cpr_bag_gather: shared memory opt-in failed");
          bag_gather_tma_kernel<64><<<grid, 256, smem, st>>>(tm, WS, reach_px, map, H, W, C, ld, centers, bag_img, K, offsets, stride, pad_hw,
                                                             out_feats, out_pts, out_valid);
        } else {
          if (cudaFuncSetAttribute(bag_gather_tma_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return fail("%s", "ptb_cpr_bag_gather: shared memory opt-in failed");
          bag_gather_tma_kernel<32><<<grid, 256, smem, st>>>(tm, WS, reach_px, map, H, W, C, ld, centers, bag_img, K, offsets, stride, pad_hw,
                                                             out_feats, out_pts, out_valid);
        }
        return check_launch("ptb_cpr_bag_gather");
      }
    }
  }
  StreamScratch* sched = stream_scratch(stream);
  if (!sched) return 1;
  // one wave of resident CTAs, work handed out dynamically (no tail wave, no static imbalance)
#define LAUNCH(CGT)                                                                                             \
  do {                                                                                                          \
    static int occ = 0;                                                                                         \
    if (occ == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bag_gather_kernel<CGT>, threads, 0) != cudaSuccess || occ <= 0)) \
      occ = 4;                                                                                                  \
    long long blocks = (long long)sm_count() * occ;                                                             \
    if (blocks > n_chunks) blocks = n_chunks;                                                                   \
    bag_gather_kernel<CGT><<<(unsigned)blocks, threads, 0, st>>>(map, H, W, C, ld, centers, bag_img, S, K, offsets, \
                                                                 stride, pad_hw, out_feats, out_pts, out_valid, sched);  \
  } while (0)
  if (CG == 64) LAUNCH(64);
  else if (CG == 40) LAUNCH(40);
  else if (CG == 20) LAUNCH(20);
  else LAUNCH(0);
#undef LAUNCH
  return check_launch("ptb_cpr_bag_gather");
}

extern "C" int ptb_cpr_bag_gather_bwd(const float* grad_out, int B, int H, int W, int C, int ld, const float* centers,
                                      const int32_t* bag_img, int G, const float* offsets, int K, float stride,
                                      float* grad_map, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && K > 0 && G >= 0, "shape");
  PTB_REQUIRE(C % 4 == 0 && ld % 4 == 0 && ld >= C, "C and ld must be multiples of 4, ld >= C");
  PTB_REQUIRE(((uintptr_t)grad_map % 16 == 0) && ((uintptr_t)grad_out % 16 == 0), "16-byte alignment");
  if (G == 0) return 0;
  PTB_REQUIRE(grad_out && centers && bag_img && offsets && grad_map, "NULL input");
  const long long S = (long long)G * K;
  const long long n_groups = (S + 31) / 32;
  long long blocks = (n_groups + 7) / 8;
  const long long max_blocks = (long long)sm_count() * 8;
  if (blocks > max_blocks) blocks = max_blocks;
  bag_gather_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(grad_out, H, W, C, ld, centers, bag_img, S, K,
                                                                           offsets, stride, grad_map);
  return check_launch("ptb_cpr_bag_gather_bwd");
}
