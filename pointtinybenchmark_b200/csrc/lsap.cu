// HungarianAssignerV2 on the GPU — kernels and C entry points around lsap_core.cuh (read its header first).
//   lsap_prep_kernel        grid (tiles, images): validates the cost entries the way scipy does (NaN / -inf -> status 2) and writes
//                           the transposed copy T[n][N] the solver scans row-wise (coalesced) when there are more proposals
//                           than GTs (scipy transposes in that case too, rectangular_lsap.cpp).
//   hungarian_v2_kernel     one CTA (1024 threads) per image: <= topk_k rounds of shortest-augmenting-path matching on the
//                           still-free proposals (hungarian_assigner.py:248-268), results scattered straight into
//                           assigned_gt_inds.  Latency-bound by construction (a sequential algorithm: one block-wide arg-min
//                           per Dijkstra step; the step's read-write column state sits in shared memory, the read-only cost row
//                           streams from L2 with 4 loads in flight per thread); images run concurrently on different SMs, nothing returns to the host:
//                           the reference's cost.cpu() + scipy loop (140 ms per solve at 16 800 x 500) disappears.
#include "ptb_common.cuh"
#include "lsap_core.cuh"
#include "lsap_cluster.cuh"
#include <stdlib.h>

namespace ptb {

constexpr int LSAP_THREADS = 1024;
constexpr int LSAP_DESC = 6;      // int64 per image: cost_off, ws_off, out_off, rowidx_off (-1: none), N, n

__global__ void __launch_bounds__(1024)
lsap_prep_kernel(const float* __restrict__ cost, const int64_t* __restrict__ desc, char* __restrict__ workspace,
                 int32_t* __restrict__ status) {
  __shared__ float tile[32][33];
  const int64_t* d = desc + (int64_t)blockIdx.y * LSAP_DESC;
  const int N = (int)d[4], n = (int)d[5];
  if (N <= 0 || n <= 0) return;
  const float* c = cost + d[0];
  const bool tr = n < N;
  float* T = tr ? ptb_lsap::ws_carve(workspace + d[1], N, n).T : nullptr;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int tiles_g = (n + 31) >> 5, tiles_p = (N + 31) >> 5;
  bool bad = false;
  for (long long t = blockIdx.x; t < (long long)tiles_g * tiles_p; t += gridDim.x) {
    const int p0 = (int)(t / tiles_g) << 5, g0 = (int)(t % tiles_g) << 5;
    const int p = p0 + ty, g = g0 + tx;
    float v = 0.f;
    if (p < N && g < n) {
      v = c[(size_t)p * n + g];
      bad |= (v != v) || (v == __int_as_float(0xff800000));
    }
    if (tr) {
      tile[ty][tx] = v;
      __syncthreads();
      const int pp = p0 + tx, gg = g0 + ty;
      if (pp < N && gg < n) T[(size_t)gg * N + pp] = tile[tx][ty];
      __syncthreads();
    }
  }
  if (bad) status[blockIdx.y] = 2;      // same value from every writer
}

__global__ void __launch_bounds__(LSAP_THREADS, 1)
hungarian_v2_kernel(const float* __restrict__ cost, const int64_t* __restrict__ desc, int topk_k,
                    const int32_t* __restrict__ row_idx, int64_t* __restrict__ gt_inds, char* __restrict__ workspace,
                    int32_t* __restrict__ status, int smem_cols) {
  extern __shared__ double s_dyn[];     // [smem_cols] spc (fp64) + [smem_cols] colstate (int32) + [smem_cols] flags (uint8): the per-step column state
  __shared__ ptb_lsap::Bcast s_bc;
  __shared__ ptb_lsap::Cand s_part[32];
  __shared__ int s_scan[33];
  const int64_t* d = desc + (int64_t)blockIdx.x * LSAP_DESC;
  const int N = (int)d[4], n = (int)d[5];
  if (N <= 0 || n <= 0) return;
  if (status[blockIdx.x] != 0) return;  // invalid entries found by the prep kernel (uniform per CTA)
  if (threadIdx.x == 0) s_bc.err = 0;
  __syncthreads();
  ptb_lsap::Ctx cx(s_bc, s_part, s_scan);
  ptb_lsap::Ws w = ptb_lsap::ws_carve(workspace + d[1], N, n);
  if ((N > n ? N : n) <= smem_cols) {   // the arrays every Dijkstra step reads AND writes live in shared memory when they fit
    w.spc = s_dyn;                      // (16 800 columns = 213 KB of the 227 KB); larger problems keep them in the L2-resident workspace
    w.colstate = reinterpret_cast<int32_t*>(s_dyn + smem_cols);
    w.flags = reinterpret_cast<uint8_t*>(w.colstate + smem_cols);
  }
  const int rc = ptb_lsap::hungarian_v2_image(cx, cost + d[0], N, n, topk_k, w, d[3] >= 0 ? row_idx + d[3] : nullptr, gt_inds + d[2]);
  if (rc && threadIdx.x == 0) status[blockIdx.x] = rc;
}

// cluster of `ncta` (8, 6 or 5) CTAs per image (lsap_cluster.cuh); blockIdx.x / ncta = image
__global__ void __launch_bounds__(ptb_lsap::CL_T, 1)
hungarian_v2_cluster_kernel(const float* __restrict__ cost, const int64_t* __restrict__ desc, int topk_k, const int32_t* __restrict__ row_idx,
                            int64_t* __restrict__ gt_inds, char* __restrict__ workspace, int32_t* __restrict__ status, int ncta) {
  extern __shared__ __align__(16) unsigned char cl_smem[];
  ptb_lsap::ClShared& S = *reinterpret_cast<ptb_lsap::ClShared*>(cl_smem);
  const int image = blockIdx.x / ncta;
  const uint32_t rank = ptb_lsap::cl_rank();
  const int64_t* d = desc + (int64_t)image * LSAP_DESC;
  const int N = (int)d[4], n = (int)d[5];
  if (N <= 0 || n <= 0) return;                 // uniform over the cluster
  if (status[image] != 0) return;               // invalid entries found by the prep kernel (uniform: written by an earlier launch)
  ptb_lsap::Ws w = ptb_lsap::ws_carve(workspace + d[1], N, n);
  const int rc = ptb_lsap::hungarian_v2_image_cl(S, rank, ncta, cost + d[0], N, n, topk_k, w, d[3] >= 0 ? row_idx + d[3] : nullptr, gt_inds + d[2]);
  if (rc && rank == 0 && threadIdx.x == 0) status[image] = rc;
}

}  // namespace ptb

extern "C" uint64_t ptb_hungarian_v2_workspace(int N, int n) {
  if (N <= 0 || n <= 0) return 64;
  return (uint64_t)ptb_lsap::ws_bytes(N, n);
}

extern "C" int ptb_hungarian_v2_batch(const float* cost, const int64_t* desc, int num_images, int max_N, int max_n, int topk_k,
                                      const int32_t* row_idx, int64_t* gt_inds, void* workspace, int32_t* status, void* stream) {
  using namespace ptb;
  PTB_REQUIRE(num_images >= 0 && topk_k >= 1 && max_N >= 0 && max_n >= 0, "shape");
  if (num_images == 0 || max_N == 0 || max_n == 0) return 0;
  PTB_REQUIRE(cost && desc && gt_inds && workspace && status, "NULL input");
  cudaStream_t st = (cudaStream_t)stream;
  const long long tiles = (long long)((max_N + 31) / 32) * ((max_n + 31) / 32);
  long long gx = tiles < 1 ? 1 : tiles;
  const long long cap = (long long)sm_count() * 2;
  if (gx > cap) gx = cap;
  int rc;
  lsap_prep_kernel<<<dim3((unsigned)gx, (unsigned)num_images), 1024, 0, st>>>(cost, desc, reinterpret_cast<char*>(workspace), status);
  if ((rc = check_launch("ptb_hungarian_v2_batch/prep"))) return rc;
  // default: one CTA cluster per image (lsap_cluster.cuh); PTB_LSAP_CLUSTER=0, problems beyond 17 600 columns / 1024 rows and devices
  // that cannot host such a cluster use the one-CTA kernel below
  const char* e_cl = getenv("PTB_LSAP_CLUSTER");
  const int max_cols = max_N > max_n ? max_N : max_n;
  const int min_dim = max_N < max_n ? max_N : max_n;            // rows of any solve <= min(N, n) <= this
  if (!(e_cl && e_cl[0] == '0') && max_cols <= ptb_lsap::CL_MAXC && min_dim <= ptb_lsap::CL_ROWS) {
    if (cudaFuncSetAttribute(hungarian_v2_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)ptb_lsap::cl_smem_bytes(ptb_lsap::CL_NMIN)) != cudaSuccess)
      return fail("%s", "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed for hungarian_v2_cluster_kernel");
    // cluster size: the largest of 8 / 6 / 5 CTAs per image with which every image of the batch is resident at once (a cluster lives
    // inside one GPC, so fewer clusters of 8 than SMs / 8 may fit, and a batch that does not fit runs as two waves); else the one with the most clusters
    int ncta = 8, best_active = -1;
    const int cand[3] = {8, 6, 5};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    for (int k = 0; k < 3; ++k) {
      cudaLaunchConfig_t q = {};
      q.gridDim = dim3((unsigned)num_images * cand[k]);
      q.blockDim = dim3(ptb_lsap::CL_T);
      q.dynamicSmemBytes = ptb_lsap::cl_smem_bytes(cand[k]);
      attr[0].val.clusterDim.x = cand[k]; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      q.attrs = attr; q.numAttrs = 1;
      int active = 0;
      if (cudaOccupancyMaxActiveClusters(&active, hungarian_v2_cluster_kernel, &q) != cudaSuccess) { (void)cudaGetLastError(); active = 0; }
      if (active >= num_images) { ncta = cand[k]; best_active = active; break; }
      if (active > best_active) { best_active = active; ncta = cand[k]; }
    }
    const char* e_n = getenv("PTB_LSAP_NCTA");
    if (e_n && (e_n[0] == '8' || e_n[0] == '6' || e_n[0] == '5')) ncta = e_n[0] - '0';
    if (best_active > 0) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)num_images * ncta);
    cfg.blockDim = dim3(ptb_lsap::CL_T);
    cfg.dynamicSmemBytes = ptb_lsap::cl_smem_bytes(ncta);
    cfg.stream = st;
    attr[0].val.clusterDim.x = ncta; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, hungarian_v2_cluster_kernel, cost, desc, topk_k, row_idx, gt_inds, reinterpret_cast<char*>(workspace),
                                       status, ncta);
    if (e != cudaSuccess) return fail("ptb_hungarian_v2_batch: cluster launch failed: %s", cudaGetErrorString(e));
    return check_launch("ptb_hungarian_v2_batch/cluster");
    }
  }
  constexpr int SMEM_COLS_MAX = 17600;      // 17600 * 13 B = 223.4 KB of dynamic shared memory
  // per device and cheap: set on every call (a process may drive several devices)
  if (cudaFuncSetAttribute(hungarian_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_COLS_MAX * 13) != cudaSuccess)
    return fail("%s", "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed for hungarian_v2_kernel");
  int smem_cols = max_N > max_n ? max_N : max_n;
  if (smem_cols > SMEM_COLS_MAX) smem_cols = SMEM_COLS_MAX;
  smem_cols = (smem_cols + 7) & ~7;
  hungarian_v2_kernel<<<num_images, LSAP_THREADS, (size_t)smem_cols * 13, st>>>(cost, desc, topk_k, row_idx, gt_inds,
                                                                               reinterpret_cast<char*>(workspace), status, smem_cols);
  return check_launch("ptb_hungarian_v2_batch");
}
