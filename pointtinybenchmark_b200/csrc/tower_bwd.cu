// Backward of the tower's GroupNorm + ReLU (mmcv ConvModule order conv -> GN -> ReLU; cpr_head.py:983-995, p2p_head.py:82-102) on the
// channels-last layout of the tensor-core convolution:  a = relu(z), z = gamma * yhat + beta, yhat = (y - mean) * rstd per (image, group).
//   dz        = da * [z > 0]
//   dgamma_c  = sum_{b,p} dz * yhat,   dbeta_c = sum_{b,p} dz
//   dy        = rstd * (gamma * dz - (s1 + yhat * s2) / n),   s1 = sum_{c in g, p} gamma * dz,  s2 = sum gamma * dz * yhat,  n = HW * C/groups
// Three launches, all HBM-bound streaming passes over (da, y):
//   1. gn_bwd_partial_kernel : per-(image, pixel-chunk, channel) partial sums of dz and dz*yhat   (reads 2 x B*HW*C*4 bytes)
//   2. gn_bwd_finalize_kernel: one CTA per image; fixed-order fp64 sums over chunks -> per-(image, group) coefficients + per-image
//      channel sums (dgamma / dbeta are their fixed-order sum over images, done by the first CTA of pass 3)
//   3. gn_bwd_apply_kernel   : dy (fp32) + max|dy| (for the power-of-two scale of the fp16 operand pair fed to dgrad / wgrad)
// Deterministic: no floating-point atomics (the max is an integer atomic on the bit pattern).
#include "ptb_common.cuh"

namespace ptb {

constexpr int GNB_THREADS = 256;

struct GnCoef {           // per (image, group)
  float mean, rstd, k1, k2;   // dy = (rstd*gamma_c) * dz - k1 - k2 * yhat
};

__device__ __forceinline__ void gn_mean_rstd(const double* __restrict__ stats, int b, int g, int groups, double inv_n, float eps,
                                             float& mu, float& rstd) {
  const double s = stats[((size_t)b * groups + g) * 2], ss = stats[((size_t)b * groups + g) * 2 + 1];
  const double mean = s * inv_n;
  double var = ss * inv_n - mean * mean;
  var = var < 0.0 ? 0.0 : var;
  rstd = (float)(1.0 / sqrt(var + (double)eps));
  mu = (float)mean;
}

// a thread owns 8 channels of one group; C/8 threads cover a pixel; blockIdx.y = image, blockIdx.x = pixel chunk
__global__ void __launch_bounds__(GNB_THREADS)
gn_bwd_partial_kernel(const float4* __restrict__ da, const float4* __restrict__ y, const double* __restrict__ stats,
                      const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C, int groups, float eps,
                      int relu, int pix_per_cta, float* __restrict__ partial /*[B][chunks][C][2]*/) {
  __shared__ float red[GNB_THREADS][17];
  const int tpp = C >> 3, ppp = GNB_THREADS / tpp;
  const int c = (threadIdx.x % tpp) * 8;
  const int b = blockIdx.y;
  const int cpg = C / groups;
  float mu, rstd;
  gn_mean_rstd(stats, b, c / cpg, groups, 1.0 / ((double)HW * cpg), eps, mu, rstd);
  float ga[8], be[8], a1[8], a2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { ga[j] = gamma[c + j]; be[j] = beta[c + j]; a1[j] = 0.f; a2[j] = 0.f; }
  const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
  const size_t img = (size_t)b * HW;
  for (int p = p0 + threadIdx.x / tpp; p < p1; p += ppp) {
    const size_t i8 = ((img + p) * C + c) >> 3;
    const float4 d0 = __ldcs(da + 2 * i8), d1 = __ldcs(da + 2 * i8 + 1);
    const float4 y0 = __ldcs(y + 2 * i8), y1 = __ldcs(y + 2 * i8 + 1);
    const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
    const float yv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float yh = (yv[j] - mu) * rstd;
      const float z = fmaf(yh, ga[j], be[j]);
      const float dz = (!relu || z > 0.f) ? dv[j] : 0.f;
      a1[j] += dz;
      a2[j] = fmaf(dz, yh, a2[j]);
    }
  }
  // fixed-order reduction over the ppp pixel rows of the CTA
#pragma unroll
  for (int j = 0; j < 8; ++j) { red[threadIdx.x][j] = a1[j]; red[threadIdx.x][8 + j] = a2[j]; }
  __syncthreads();
  if (threadIdx.x < tpp) {
    float s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
    for (int r = 0; r < ppp; ++r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { s1[j] += red[r * tpp + threadIdx.x][j]; s2[j] += red[r * tpp + threadIdx.x][8 + j]; }
    }
    float* out = partial + (((size_t)b * gridDim.x + blockIdx.x) * C + c) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) { out[2 * j] = s1[j]; out[2 * j + 1] = s2[j]; }
  }
}

// one CTA per image, 1024 threads (C <= 1024): 1024 / C threads per channel add interleaved subsets of its chunk partials in a fixed
// order (fp64, 4 independent chains each), thread c adds those in a fixed order, the first `groups` threads turn the channel sums into
// the per-(image, group) coefficients
__global__ void __launch_bounds__(1024)
gn_bwd_finalize_kernel(const float* __restrict__ partial, const double* __restrict__ stats, const float* __restrict__ gamma,
                       int chunks, int HW, int C, int groups, float eps, GnCoef* __restrict__ coef /*[B][groups]*/,
                       double* __restrict__ img_sums /*[B][C][2]: sum dz, sum dz*yhat per image*/) {
  __shared__ double sh1[1024], sh2[1024];
  const int b = blockIdx.x;
  const int cpg = C / groups;
  const double inv_n = 1.0 / ((double)HW * cpg);
  // 1024 / C threads share a channel (chunk k goes to part k % nparts): the loop over chunks is a chain of dependent-latency loads,
  // with one thread per channel that chain, not the few KB of data, set the launch time
  const int nparts = 1024 / C;                       // >= 1 (C <= 1024)
  const int c = threadIdx.x % C, part = threadIdx.x / C;
  double r1 = 0.0, r2 = 0.0;
  if (part < nparts) {
    double a1[4] = {0.0, 0.0, 0.0, 0.0}, a2[4] = {0.0, 0.0, 0.0, 0.0};
    const float2* p = reinterpret_cast<const float2*>(partial) + (size_t)b * chunks * C + c;
    int k = part;
    for (; k + 3 * nparts < chunks; k += 4 * nparts) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float2 v = __ldg(p + (size_t)(k + u * nparts) * C);
        a1[u] += (double)v.x;
        a2[u] += (double)v.y;
      }
    }
    for (; k < chunks; k += nparts) {
      const float2 v = __ldg(p + (size_t)k * C);
      a1[0] += (double)v.x;
      a2[0] += (double)v.y;
    }
    sh1[threadIdx.x] = (a1[0] + a1[1]) + (a1[2] + a1[3]);
    sh2[threadIdx.x] = (a2[0] + a2[1]) + (a2[2] + a2[3]);
  }
  __syncthreads();
  if (threadIdx.x < C) {                             // parts in a fixed order
    for (int q = 0; q < nparts; ++q) { r1 += sh1[q * C + c]; r2 += sh2[q * C + c]; }
    img_sums[((size_t)b * C + c) * 2] = r1;
    img_sums[((size_t)b * C + c) * 2 + 1] = r2;
  }
  __syncthreads();
  if (threadIdx.x < C) {
    const double g_c = (double)gamma[c];
    sh1[c] = g_c * r1;
    sh2[c] = g_c * r2;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    double s1 = 0.0, s2 = 0.0;
    for (int j = 0; j < cpg; ++j) { s1 += sh1[g * cpg + j]; s2 += sh2[g * cpg + j]; }
    float mu, rstd;
    gn_mean_rstd(stats, b, g, groups, inv_n, eps, mu, rstd);
    GnCoef k;
    k.mean = mu; k.rstd = rstd;
    k.k1 = (float)((double)rstd * s1 * inv_n);
    k.k2 = (float)((double)rstd * s2 * inv_n);
    coef[(size_t)b * groups + g] = k;
  }
}

__global__ void __launch_bounds__(GNB_THREADS)
gn_bwd_apply_kernel(const float4* __restrict__ da, const float4* __restrict__ y, const GnCoef* __restrict__ coef,
                    const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int C, int groups, int relu,
                    int pix_per_cta, float4* __restrict__ dy, unsigned int* __restrict__ amax_bits,
                    const double* __restrict__ img_sums, int B, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  if (blockIdx.x == 0 && blockIdx.y == 0) {          // dbeta_c = sum_b sum dz, dgamma_c = sum_b sum dz*yhat  (fixed order over images)
    for (int ch = threadIdx.x; ch < C; ch += GNB_THREADS) {
      double d1 = 0.0, d2 = 0.0;
      for (int bb = 0; bb < B; ++bb) { d1 += img_sums[((size_t)bb * C + ch) * 2]; d2 += img_sums[((size_t)bb * C + ch) * 2 + 1]; }
      if (dbeta) dbeta[ch] = (float)d1;
      if (dgamma) dgamma[ch] = (float)d2;
    }
  }
  const int tpp = C >> 3, ppp = GNB_THREADS / tpp;
  const int c = (threadIdx.x % tpp) * 8;
  const int b = blockIdx.y;
  const GnCoef k = coef[(size_t)b * groups + c / (C / groups)];
  float ga[8], be[8], rg[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { ga[j] = gamma[c + j]; be[j] = beta[c + j]; rg[j] = k.rstd * ga[j]; }
  const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
  const size_t img = (size_t)b * HW;
  float m = 0.f;
  for (int p = p0 + threadIdx.x / tpp; p < p1; p += ppp) {
    const size_t i8 = ((img + p) * C + c) >> 3;
    const float4 d0 = __ldcs(da + 2 * i8), d1 = __ldcs(da + 2 * i8 + 1);
    const float4 y0 = __ldcs(y + 2 * i8), y1 = __ldcs(y + 2 * i8 + 1);
    const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
    const float yv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float yh = (yv[j] - k.mean) * k.rstd;
      const float z = fmaf(yh, ga[j], be[j]);
      const float dz = (!relu || z > 0.f) ? dv[j] : 0.f;
      o[j] = fmaf(rg[j], dz, -fmaf(k.k2, yh, k.k1));
      m = fmaxf(m, fabsf(o[j]));
    }
    dy[2 * i8] = make_float4(o[0], o[1], o[2], o[3]);
    dy[2 * i8 + 1] = make_float4(o[4], o[5], o[6], o[7]);
  }
  if (amax_bits) {
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));   // non-negative floats order like their bits
  }
}

}  // namespace ptb

using namespace ptb;

static int gnb_grid(int B, int HW, int C, int* pix_per_cta) {
  const int ppp = GNB_THREADS / (C / 8);
  int chunks = (sm_count() * 4 + B - 1) / B;
  int ppc = (HW + chunks - 1) / chunks;
  ppc = ((ppc + ppp - 1) / ppp) * ppp;
  *pix_per_cta = ppc;
  return (HW + ppc - 1) / ppc;
}

extern "C" uint64_t ptb_gn_relu_bwd_workspace(int B, int HW, int C, int groups) {
  if (B <= 0 || HW <= 0 || C <= 0 || groups <= 0 || C % 8 != 0 || GNB_THREADS % (C / 8) != 0) return 0;
  int ppc;
  const int chunks = gnb_grid(B, HW, C, &ppc);
  return (size_t)B * chunks * C * 2 * sizeof(float) + (size_t)B * groups * sizeof(GnCoef) + (size_t)B * C * 2 * sizeof(double) + 256;
}

extern "C" int ptb_gn_relu_bwd(const float* da, const float* y, const double* gn_stats, const float* gamma, const float* beta, int B,
                               int HW, int C, int groups, float eps, int relu, void* workspace, float* dy, float* dgamma,
                               float* dbeta, unsigned int* amax_bits, void* stream) {
  PTB_REQUIRE(B > 0 && HW > 0 && C > 0 && groups > 0 && C % groups == 0, "shape");
  PTB_REQUIRE(C % 8 == 0 && (C / groups) % 8 == 0 && C <= 1024 && GNB_THREADS % (C / 8) == 0,
              "C/groups must be a multiple of 8 and C/8 must divide 256");
  PTB_REQUIRE(da && y && gn_stats && gamma && beta && workspace && dy, "NULL input");
  PTB_REQUIRE(((uintptr_t)da % 32 == 0) && ((uintptr_t)y % 32 == 0) && ((uintptr_t)dy % 32 == 0) && ((uintptr_t)workspace % 16 == 0),
              "alignment");
  cudaStream_t st = (cudaStream_t)stream;
  int ppc;
  const int chunks = gnb_grid(B, HW, C, &ppc);
  float* partial = reinterpret_cast<float*>(workspace);
  size_t off = (size_t)B * chunks * C * 2 * sizeof(float);
  off = (off + 15) / 16 * 16;
  GnCoef* coef = reinterpret_cast<GnCoef*>(reinterpret_cast<char*>(workspace) + off);
  off += (size_t)B * groups * sizeof(GnCoef);
  off = (off + 15) / 16 * 16;
  double* img_sums = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + off);
  const dim3 grid((unsigned)chunks, (unsigned)B);
  gn_bwd_partial_kernel<<<grid, GNB_THREADS, 0, st>>>(reinterpret_cast<const float4*>(da), reinterpret_cast<const float4*>(y), gn_stats,
                                                       gamma, beta, HW, C, groups, eps, relu, ppc, partial);
  int rc = check_launch("ptb_gn_relu_bwd/partial");
  if (rc) return rc;
  gn_bwd_finalize_kernel<<<B, 1024, 0, st>>>(partial, gn_stats, gamma, chunks, HW, C, groups, eps, coef, img_sums);
  if ((rc = check_launch("ptb_gn_relu_bwd/finalize"))) return rc;
  if (amax_bits && cudaMemsetAsync(amax_bits, 0, 4, st) != cudaSuccess) return fail("%s", "ptb_gn_relu_bwd: cudaMemsetAsync failed");
  gn_bwd_apply_kernel<<<grid, GNB_THREADS, 0, st>>>(reinterpret_cast<const float4*>(da), reinterpret_cast<const float4*>(y), coef, gamma,
                                                     beta, HW, C, groups, relu, ppc, reinterpret_cast<float4*>(dy), amax_bits, img_sums, B, dgamma, dbeta);
  return check_launch("ptb_gn_relu_bwd/apply");
}
