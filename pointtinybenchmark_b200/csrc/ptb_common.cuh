// Shared helpers for the sm_90a kernels of libptb_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/ptb_b200.h"

namespace ptb {

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

inline int fail(const char* fmt, const char* a = "", long long b = 0, long long c = 0) {
  snprintf(g_err, sizeof(g_err), fmt, a, b, c);
  return 1;
}

#define PTB_REQUIRE(cond, msg)                                                          \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      snprintf(ptb::g_err, sizeof(ptb::g_err), "%s: requirement failed: %s (%s)", __func__, #cond, msg); \
      return 2;                                                                         \
    }                                                                                   \
  } while (0)

inline int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return 3;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// per-(device, stream) scratch: self-resetting scheduler tickets / "last block" counters and block partials of the fixed-order
// reductions.  Launches on ONE stream are serialised, and the last block of every fixed-order sum resets `done` before its
// kernel ends, so one SumScratch serves every sum kernel of the stream; a block per stream keeps concurrent launches on
// different streams apart.  Allocated lazily (cudaMalloc + cudaMemsetAsync on its stream, once per stream) by capi.cu; ptb_reset_stream_state()
// zeroes it after an aborted launch.
// ---------------------------------------------------------------------------------------------
constexpr int SCRATCH_BLOCKS = 528;      // 4 x 132 (H100 SMs): grid of the fixed-order sum kernels
struct SumScratch {
  float partials[SCRATCH_BLOCKS];
  unsigned int done;
};
struct StreamScratch {
  unsigned int gather_ticket, gather_done;       // bag_gather chunk scheduler
  SumScratch sum;
  unsigned int spare[60];
};
StreamScratch* stream_scratch(void* stream);     // NULL on failure (g_err set)

inline int sm_count() {       // of the CURRENT device (cached per device: a process may drive several)
  static int n[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;  // H100 SXM
  if (n[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev] = v;
  }
  return n[dev];
}

// ---------------------------------------------------------------------------------------------
// numerics that define parity with the reference's CPU (ATen) path
// ---------------------------------------------------------------------------------------------

// Sample coordinate pipeline of cpr_head.py:192 + 88 followed by ATen grid_sampler_2d (align_corners=False,
// padding_mode='border') on CPU:  u = p/stride;  g = (2u+1)/size - 1;  ix = fma(g+1, size/2, -0.5);  clip to [0,size-1].
// (the fma in the un-normalise step was identified empirically: it reproduces ATen's CPU output to 5e-7.)
__device__ __forceinline__ float sample_coord(float img_coord, float stride, float size, float half_size) {
  float u = __fdiv_rn(img_coord, stride);
  float t = __fadd_rn(__fmul_rn(2.f, u), 1.f);
  float g = __fadd_rn(__fdiv_rn(t, size), -1.f);
  float ix = __fmaf_rn(__fadd_rn(g, 1.f), half_size, -0.5f);
  return fminf(fmaxf(ix, 0.f), size - 1.f);
}

struct Taps {
  int o00, o01, o10, o11;   // cell offsets (y*W + x), to be multiplied by the cell stride
  float w00, w01, w10, w11; // nw, ne, sw, se weights
};

// taps from the (clamped) source-pixel coordinates ix, iy of sample_coord
__device__ __forceinline__ Taps make_taps_at(float ix, float iy, int H, int W) {
  float x0f = floorf(ix), y0f = floorf(iy);
  int x0 = (int)x0f, y0 = (int)y0f;
  int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);  // east/south tap has weight 0 when clamped
  float ex = __fsub_rn(__fadd_rn(x0f, 1.f), ix), wx = __fsub_rn(ix, x0f);
  float ey = __fsub_rn(__fadd_rn(y0f, 1.f), iy), wy = __fsub_rn(iy, y0f);
  Taps t;
  t.o00 = y0 * W + x0; t.o01 = y0 * W + x1; t.o10 = y1 * W + x0; t.o11 = y1 * W + x1;
  t.w00 = __fmul_rn(ex, ey); t.w01 = __fmul_rn(wx, ey); t.w10 = __fmul_rn(ex, wy); t.w11 = __fmul_rn(wx, wy);
  return t;
}

__device__ __forceinline__ Taps make_taps(float px, float py, float stride, int H, int W) {
  return make_taps_at(sample_coord(px, stride, (float)W, 0.5f * (float)W), sample_coord(py, stride, (float)H, 0.5f * (float)H), H, W);
}

// bilinear combination of four 128-bit taps in ATen's operation order (nw*w + ne*w + sw*w + se*w as an FMA chain, bit-exact vs the
// CPU grid_sample kernel).  __f*_rn intrinsics are never contracted or reassociated, so every element rounds exactly as ATen's does.
__device__ __forceinline__ float bilerp1(float q0, float q1, float q2, float q3, float w00, float w01, float w10, float w11) {
  return __fmaf_rn(q3, w11, __fmaf_rn(q2, w10, __fmaf_rn(q1, w01, __fmul_rn(q0, w00))));
}
__device__ __forceinline__ float4 bilerp4(const float4 q0, const float4 q1, const float4 q2, const float4 q3, float w00, float w01,
                                          float w10, float w11) {
  return make_float4(bilerp1(q0.x, q1.x, q2.x, q3.x, w00, w01, w10, w11), bilerp1(q0.y, q1.y, q2.y, q3.y, w00, w01, w10, w11),
                     bilerp1(q0.z, q1.z, q2.z, q3.z, w00, w01, w10, w11), bilerp1(q0.w, q1.w, q2.w, q3.w, w00, w01, w10, w11));
}

// torch.cdist(p=2) as ATen computes it.
//  - matmul formulation (rows1 > 25 || rows2 > 25; aten/src/ATen/native/Distance.cpp _euclidean_dist):
//      [-2x0, -2x1, |x|^2, 1] . [y0, y1, 1, |y|^2]  accumulated k=0..3 with FMAs (MKL sgemm order, verified bit-exact
//      on 8.7e5 pairs in the build container), clamp_min(0), sqrt.
//  - direct formulation otherwise: sqrt((x0-y0)^2 + (x1-y1)^2), no FMA.
// __f*_rn intrinsics are never contracted by nvcc, so the rounding sequence is fixed.
__device__ __forceinline__ float sq_norm2(float x, float y) { return __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)); }

__device__ __forceinline__ float cdist_mm(float px, float py, float pn, float cx, float cy, float cn) {
  float acc = __fmul_rn(__fmul_rn(-2.f, px), cx);
  acc = __fmaf_rn(__fmul_rn(-2.f, py), cy, acc);
  acc = __fadd_rn(acc, pn);
  acc = __fadd_rn(acc, cn);
  return __fsqrt_rn(fmaxf(acc, 0.f));
}

__device__ __forceinline__ float cdist_direct(float px, float py, float cx, float cy) {
  float dx = fabsf(__fsub_rn(px, cx)), dy = fabsf(__fsub_rn(py, cy));
  return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
}

// torch.sigmoid on the CPU (ATen UnaryOpsKernel.cpp sigmoid_kernel, vectorised path):  a = 0 - x;  a = Sleef_expf_u10(a);  a = 1 + a;
// a = 1 / a (true division).  Sleef's expf (sleefsimdsp.c xexpf: Cody-Waite reduction with L2Uf / L2Lf, degree-6 polynomial as an FMA
// chain, ldexp2) is restated operation by operation, so the probabilities are BIT-IDENTICAL to the reference's: verified in the build
// container against torch.sigmoid on 4e6 random inputs (0 mismatches; cf. ~24 % mismatching bits with libm / CUDA expf).  This makes
// every thresholded / sorted probability (top-k order, score_thr, merge_th, classify arg-max) reproduce the reference exactly whenever
// the logits agree, instead of "up to 1-ulp ties".
__device__ __forceinline__ float sleef_expf_u10(float d) {
  const int q = __float2int_rn(__fmul_rn(d, 1.442695040888963407359924681001892137426645954152985934135449406931f));
  const float qf = (float)q;
  float s = __fmaf_rn(qf, -0.693145751953125f, d);
  s = __fmaf_rn(qf, -1.428606765330187045e-06f, s);
  float u = 0.000198527617612853646278381f;
  u = __fmaf_rn(u, s, 0.00139304355252534151077271f);
  u = __fmaf_rn(u, s, 0.00833336077630519866943359f);
  u = __fmaf_rn(u, s, 0.0416664853692054748535156f);
  u = __fmaf_rn(u, s, 0.166666671633720397949219f);
  u = __fmaf_rn(u, s, 0.5f);
  u = __fadd_rn(1.0f, __fmaf_rn(__fmul_rn(s, s), u, s));
  const int h = q >> 1;                                                     // vldexp2: u * 2^(q>>1) * 2^(q - (q>>1))
  u = __fmul_rn(__fmul_rn(u, __int_as_float((h + 127) << 23)), __int_as_float((q - h + 127) << 23));
  if (d < -104.f) u = 0.f;
  if (d > 100.f) u = __int_as_float(0x7f800000);
  return u;
}
__device__ __forceinline__ float sigmoidf_acc(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, sleef_expf_u10(__fsub_rn(0.f, x)))); }

// ---------------------------------------------------------------------------------------------
// warp / block reductions (fixed order => deterministic)
// ---------------------------------------------------------------------------------------------
// an NMS box on the coordinates the IoU sees, area = (x2 - x1) * (y2 - y1); iou_gt: mmcv / torchvision nms (offset 0), IoU > thr in
// their fp32 operation order.  Shared by every NMS kernel so that they cannot disagree.
struct Box {
  float x1, y1, x2, y2, area;
};
__device__ __forceinline__ bool iou_gt(const Box& a, const Box& b, float thr) {
  const float w = fmaxf(0.f, __fsub_rn(fminf(a.x2, b.x2), fmaxf(a.x1, b.x1)));
  const float h = fmaxf(0.f, __fsub_rn(fminf(a.y2, b.y2), fmaxf(a.y1, b.y1)));
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(a.area, b.area), inter));
  return ovr > thr;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// deterministic sum over launch_sum's fixed grid of SCRATCH_BLOCKS x 256 threads: each block writes its partial, the last block
// to finish adds them in block order into out[0] and resets the counter, so the next sum kernel on the stream finds `done` at 0.
// The trip counts are the grid's constants: the final loop is latency-bound, and a known count lets the compiler batch its loads.
__device__ __forceinline__ void block_partial_finish(float acc, SumScratch& sc, float* out) {
  __shared__ float red[8];
  __shared__ bool last;
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    sc.partials[blockIdx.x] = t;
    __threadfence();
    last = (atomicAdd(&sc.done, 1u) == SCRATCH_BLOCKS - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float t = 0.f;
    for (int b = 0; b < SCRATCH_BLOCKS; ++b) t += reinterpret_cast<volatile float*>(sc.partials)[b];
    out[0] += t;
    sc.done = 0;
  }
}

// launches a kernel that ends in block_partial_finish on SCRATCH_BLOCKS x 256 threads, with the stream's SumScratch appended to args
template <class... Params, class... Args>
inline int launch_sum(void (*kernel)(Params...), void* stream, const char* name, Args... args) {
  StreamScratch* scr = stream_scratch(stream);
  if (!scr) return 1;
  kernel<<<SCRATCH_BLOCKS, 256, 0, (cudaStream_t)stream>>>(args..., &scr->sum);
  return check_launch(name);
}

// streaming 128-bit store (output that is not re-read by this kernel: keep it out of the way of the map in L2)
__device__ __forceinline__ void st_cs(float4* p, float4 v) { __stcs(p, v); }

}  // namespace ptb
