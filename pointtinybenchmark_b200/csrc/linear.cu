// Row-wise linear classifier over channels-last maps (the 1x1-conv form of CPRHead.cls_out / ins_out,
// cpr_head.py:1008-1014, 1045-1078) and its two backward products.  fp32 FFMA ("parity mode", no TF32):
// logits must match the reference CPU head to 1e-4, see DESIGN.md for the tensor-core plan.
//
// forward  Y[M][N]   = X[M][Cin] * Wt[N][Cin]^T + b       128x80 output tile / CTA, 8x5 micro-tile / thread
// bwd_x    dX[M][Cin] = dY[M][N] * W[N][Cin]              same kernel with operand roles swapped (B given as [K][N])
// bwd_w    dW[N][Cin] = dY^T[N][M] * X[M][Cin]            split-M partial tiles + fixed-order reduction
#include "ptb_common.cuh"

namespace ptb {

constexpr int BM = 128, BN = 80, BK = 16, TM = 8, TN = 5;   // 16x16 threads

// C[m][n] (+)= sum_k A[m][k] * Bop[k][n] (+ bias[n])
//   A: [M][lda] row-major (k contiguous).
//   B_IS_NK = true : B given as [N][ldb] (k contiguous)   -> forward (W is [N][Cin])
//   B_IS_NK = false: B given as [K][ldb] (n contiguous)   -> bwd_x   (W is [N][Cin] = [K][n])
template <bool B_IS_NK>
__global__ void __launch_bounds__(256)
sgemm_rows_kernel(const float* __restrict__ A, int M, int Kd, int lda, const float* __restrict__ Bm, int N, int ldb,
                  const float* __restrict__ bias, float* __restrict__ Cc, int ldc, int accumulate) {
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // global->smem staging assignment
  const int a_row = tid >> 2, a_k4 = (tid & 3) * 4;     // A: 2 x (64 rows x 16 k) per thread-pass
  float4 a_reg[2];
  float b_reg[5];                                        // B tile: 16 x 80 = 1280 floats = 5 per thread

  auto load_tile = [&](int k0) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int r = m0 + a_row + 64 * p;
      if (r < M) a_reg[p] = __ldg(reinterpret_cast<const float4*>(A + (size_t)r * lda + k0 + a_k4));
      else a_reg[p] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int p = 0; p < 5; ++p) {
      const int e = tid + 256 * p;           // 0..1279
      int kk, nn;
      if (B_IS_NK) { nn = e >> 4; kk = e & 15; }        // consecutive threads walk k (contiguous in memory)
      else { kk = e / BN; nn = e - kk * BN; }            // consecutive threads walk n (contiguous in memory)
      const int n = n0 + nn;
      float v = 0.f;
      if (n < N) v = B_IS_NK ? __ldg(Bm + (size_t)n * ldb + k0 + kk) : __ldg(Bm + (size_t)(k0 + kk) * ldb + n);
      b_reg[p] = v;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int r = a_row + 64 * p;
      As[buf][a_k4 + 0][r] = a_reg[p].x; As[buf][a_k4 + 1][r] = a_reg[p].y;
      As[buf][a_k4 + 2][r] = a_reg[p].z; As[buf][a_k4 + 3][r] = a_reg[p].w;
    }
#pragma unroll
    for (int p = 0; p < 5; ++p) {
      const int e = tid + 256 * p;
      int kk, nn;
      if (B_IS_NK) { nn = e >> 4; kk = e & 15; }
      else { kk = e / BN; nn = e - kk * BN; }
      Bs[buf][kk][nn] = b_reg[p];
    }
  };

  const int n_k = Kd / BK;   // host guarantees Kd % 16 == 0
  load_tile(0);
  store_tile(0);
  __syncthreads();
  for (int kt = 0; kt < n_k; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_k) load_tile((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[buf][k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < n_k) {
      store_tile(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int j = 0; j < TN; ++j) {
    const int n = n0 + tx + 16 * j;
    if (n >= N) continue;
    const float bv = bias ? __ldg(bias + n) : 0.f;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = m0 + ty * TM + i;
      if (m < M) {
        float* p = Cc + (size_t)m * ldc + n;
        const float v = acc[i][j] + bv;
        *p = accumulate ? (*p + v) : v;
      }
    }
  }
}

// dW partials: part[s][n][c] = sum_{m in slice s} dY[m][n] * X[m][c];   dbp[s][n] = sum_{m in slice s} dY[m][n]
// CTA: 80 (n) x 128 (c) tile, slice of M rows;  thread micro-tile 5 (n) x 8 (c).
__global__ void __launch_bounds__(256)
dw_partial_kernel(const float* __restrict__ dY, int M, int N, int ldy, const float* __restrict__ X, int Cin, int ldx,
                  int rows_per_slice, float* __restrict__ part, float* __restrict__ dbp) {
  __shared__ __align__(16) float Ys[BK][BN];        // [m][n]
  __shared__ __align__(16) float Xs[BK][BM];        // [m][c]
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;        // ty -> c block of 8, tx -> n (tx + 16 j)
  const int c0 = blockIdx.x * BM, n0 = blockIdx.y * BN, s = blockIdx.z;
  const int m_begin = s * rows_per_slice, m_end = min(M, m_begin + rows_per_slice);
  float acc[TN][TM];
#pragma unroll
  for (int j = 0; j < TN; ++j)
#pragma unroll
    for (int i = 0; i < TM; ++i) acc[j][i] = 0.f;
  float dbj[TN] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int mt = m_begin; mt < m_end; mt += BK) {
    // stage 16 rows
    for (int e = tid; e < BK * BN; e += 256) {
      const int mm = e / BN, nn = e - mm * BN;
      const int m = mt + mm, n = n0 + nn;
      Ys[mm][nn] = (m < m_end && n < N) ? __ldg(dY + (size_t)m * ldy + n) : 0.f;
    }
    for (int e = tid; e < BK * BM / 4; e += 256) {
      const int mm = e / (BM / 4), c4 = (e - mm * (BM / 4)) * 4;
      const int m = mt + mm, c = c0 + c4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < m_end && c < Cin) v = __ldg(reinterpret_cast<const float4*>(X + (size_t)m * ldx + c));
      *reinterpret_cast<float4*>(&Xs[mm][c4]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float y[TN], x[TM];
#pragma unroll
      for (int j = 0; j < TN; ++j) y[j] = Ys[k][tx + 16 * j];
      const float4 x0 = *reinterpret_cast<const float4*>(&Xs[k][ty * TM]);
      const float4 x1 = *reinterpret_cast<const float4*>(&Xs[k][ty * TM + 4]);
      x[0] = x0.x; x[1] = x0.y; x[2] = x0.z; x[3] = x0.w; x[4] = x1.x; x[5] = x1.y; x[6] = x1.z; x[7] = x1.w;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        dbj[j] += y[j];
#pragma unroll
        for (int i = 0; i < TM; ++i) acc[j][i] = fmaf(y[j], x[i], acc[j][i]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < TN; ++j) {
    const int n = n0 + tx + 16 * j;
    if (n >= N) continue;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int c = c0 + ty * TM + i;
      if (c < Cin) part[((size_t)s * N + n) * Cin + c] = acc[j][i];
    }
    if (ty == 0 && blockIdx.x == 0) dbp[(size_t)s * N + n] = dbj[j];
  }
}

// out[e] = sum_s part[s][e]  in slice order (deterministic)
__global__ void reduce_slices_kernel(const float* __restrict__ part, int n_slices, size_t n_elem, float* __restrict__ out) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elem) return;
  float s = 0.f;
  for (int i = 0; i < n_slices; ++i) s += part[(size_t)i * n_elem + e];
  out[e] = s;
}

static inline int dw_slices(int M) {
  int s = (M + 2047) / 2048;   // >= 2048 rows per slice
  if (s > 74) s = 74;
  if (s < 1) s = 1;
  return s;
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_linear_rows(const float* x, int M, int Cin, int ldx, const float* w, const float* bias, int N,
                               float* y, int ldy, void* stream) {
  PTB_REQUIRE(M >= 0 && Cin > 0 && N > 0, "shape");
  PTB_REQUIRE(Cin % 16 == 0 && ldx % 4 == 0 && ldx >= Cin && ldy >= N, "Cin % 16 == 0, ldx % 4 == 0");
  PTB_REQUIRE((uintptr_t)x % 16 == 0, "x must be 16-byte aligned");
  if (M == 0) return 0;
  PTB_REQUIRE(x && w && y, "NULL input");
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN);
  sgemm_rows_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, M, Cin, ldx, w, N, Cin, bias, y, ldy, 0);
  return check_launch("ptb_linear_rows");
}

extern "C" int ptb_linear_rows_bwd_x(const float* dy, int M, int N, int ldy, const float* w, int Cin, float* dx, int ldx,
                                     int accumulate, void* stream) {
  PTB_REQUIRE(M >= 0 && Cin > 0 && N > 0, "shape");
  PTB_REQUIRE(N % 16 == 0 && ldy % 4 == 0 && ldy >= N && ldx >= Cin, "N % 16 == 0, ldy % 4 == 0");
  PTB_REQUIRE((uintptr_t)dy % 16 == 0, "dy must be 16-byte aligned");
  if (M == 0) return 0;
  PTB_REQUIRE(dy && w && dx, "NULL input");
  // dX[M][Cin] = dY[M][N] * W[N][Cin] : A = dY (K = N), B = W as [K][n] with n = c
  dim3 grid((M + BM - 1) / BM, (Cin + BN - 1) / BN);
  sgemm_rows_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(dy, M, N, ldy, w, Cin, Cin, nullptr, dx, ldx, accumulate);
  return check_launch("ptb_linear_rows_bwd_x");
}

extern "C" uint64_t ptb_linear_rows_bwd_w_workspace(int M, int N, int Cin) {
  return (uint64_t)dw_slices(M) * ((uint64_t)N * Cin + N) * sizeof(float);
}

extern "C" int ptb_linear_rows_bwd_w(const float* dy, int M, int N, int ldy, const float* x, int Cin, int ldx, float* dw,
                                     float* db, float* workspace, uint64_t workspace_bytes, void* stream) {
  PTB_REQUIRE(M > 0 && Cin > 0 && N > 0, "shape");
  PTB_REQUIRE(Cin % 4 == 0 && ldx % 4 == 0 && (uintptr_t)x % 16 == 0, "Cin/ldx % 4, x 16-byte aligned");
  PTB_REQUIRE(workspace_bytes >= ptb_linear_rows_bwd_w_workspace(M, N, Cin), "workspace too small");
  PTB_REQUIRE(dy && x && dw && workspace, "NULL input");
  const int S = dw_slices(M);
  int rps = (M + S - 1) / S;
  rps = (rps + BK - 1) / BK * BK;
  float* part = workspace;
  float* dbp = workspace + (size_t)S * N * Cin;
  dim3 grid((Cin + BM - 1) / BM, (N + BN - 1) / BN, S);
  cudaStream_t st = (cudaStream_t)stream;
  dw_partial_kernel<<<grid, 256, 0, st>>>(dy, M, N, ldy, x, Cin, ldx, rps, part, dbp);
  int rc = check_launch("ptb_linear_rows_bwd_w/partial");
  if (rc) return rc;
  const size_t ne = (size_t)N * Cin;
  reduce_slices_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, st>>>(part, S, ne, dw);
  rc = check_launch("ptb_linear_rows_bwd_w/reduce");
  if (rc) return rc;
  if (db) {
    reduce_slices_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(dbp, S, (size_t)N, db);
    rc = check_launch("ptb_linear_rows_bwd_w/reduce_b");
  }
  return rc;
}
