// HungarianAssignerV2's matching with the column scan of every Dijkstra step split over an 8-CTA thread-block cluster (round 2).
//
// Why: the one-CTA-per-image kernel (lsap_core.cuh) runs hundreds of instructions per thread and Dijkstra step for the columns a thread
// owns, on the ONE SM an image runs on, and spends the rest of the time at the block barrier: the step is bound by one SM's instruction
// issue, not by memory.  Here an image is solved by a cluster of CL_N CTAs:
//   * CTA r owns the contiguous column range [r*Cc, (r+1)*Cc) and keeps ITS part of the per-step read-write column state (spc fp64,
//     colstate int32, flags) in its own shared memory; a thread scans <= 5 columns, all global loads of a step in flight at once;
//   * per step: block arg-best -> every CTA stores its candidate into the leader's shared memory (st.shared::cluster) -> cluster
//     barrier A -> the leader's thread 0 picks the winner of the 8 (the same total order: identical to the sequential scan) and runs the
//     bookkeeping of lsap_core.cuh's solve() (swap-with-last removal, next row), reaching into the owners' shared memory for the two
//     column states it touches, then stores the broadcast record (minVal, column, next row) into every CTA -> cluster barrier B;
//   * dual update, augmentation, free-list compaction and the output scatter are the leader's (a handful of entries each); the
//     per-round gather of the cost matrix is shared by all CTAs.
//   * v2 of this file: the first cluster version kept v, path, row4col, remaining, u, col4row in the L2-resident workspace like the
//     one-CTA kernel and was NOT faster (10.3 vs 9.6 ms per 16 images): an augmentation is a chain of ~10 dependent L2 round trips in
//     the serial sections (remstamp -> remaining, row4col, the dual update's read-modify-writes, the path walk), not instruction
//     issue.  Now every per-column array lives in its owner's shared memory (33 B per column; the leader reaches it with
//     ld/st.shared::cluster, ~215 cycles instead of an L2 trip), `remaining` + stamps (uint16) and the row arrays u / col4row are in
//     the leader's shared memory; the only global traffic of a Dijkstra step is the cost row.
//   * v3: the bookkeeping is REPLICATED instead of led.  A CTA's candidate message carries everything the bookkeeping needs about its
//     best column (value, list state, row4col, path predecessor); every CTA stores its message into ALL CTAs (double-buffered slots),
//     ONE cluster barrier per Dijkstra step, and every CTA then runs the identical sequential bookkeeping on its own copies of the row
//     arrays (u, col4row, predecessor rows) and of the `remaining` list, touching only the column state it owns.  spc[j] of a scanned
//     column is frozen at the value it was selected with (= that step's minVal), so the dual update needs no column state either: the
//     step records (column, minVal, row) are replicated too.  No leader sections, no second / third barrier per step, and the cost row
//     of the next augmentation (row cur+1: known in advance) is prefetched into registers one augmentation ahead.
// Arrays that cross CTAs through GLOBAL memory (free list, gathered matrix) are read with ld.global.cg: an SM's L1 is not coherent
// with another SM's stores; the cluster barriers (arrive.release / wait.acquire) order them.
// The algorithm, its fp64 operation order and its tie rule are those of lsap_core.cuh (read its header first): assignments are
// bit-identical to scipy and to the single-CTA kernel (tests/test_lsap.py runs both).
#pragma once
#include "lsap_core.cuh"

namespace ptb_lsap {

constexpr int CL_N = 8;            // largest cluster (CTAs per image; the portable limit).  The host picks 8, 6 or 5 CTAs per image so that all
                                   // images of a batch are resident at once (a cluster lives inside one GPC, so fewer clusters of 8 than SMs / 8
                                   // may fit; a batch that does not fit runs as two waves)
constexpr int CL_T = 512;          // threads per CTA
constexpr int CL_MAXC = 17600;     // columns of a problem (= the single-CTA kernel's shared-memory limit)
constexpr int CL_NMIN = 5;         // smallest cluster the shared-memory budget allows (3520 columns per CTA)
constexpr int CL_U = (CL_MAXC / CL_NMIN + CL_T - 1) / CL_T;     // <= 7 columns per thread, one group

constexpr int CL_ROWS = 1024;      // rows (min(N, n)) whose arrays every CTA replicates in shared memory; larger problems use the one-CTA kernel
constexpr int CL_SC = 256;         // scanned-column list entries cached in shared memory (the rest goes through the workspace)

struct ClMsg {                     // a CTA's candidate of one Dijkstra step (32 bytes, stored into every CTA)
  double val;                      // spc of the column
  int st, j;                       // list state (0: none) and column
  int r4c, pth;                    // row4col[j];  path[j] if it was set in this augmentation, else cur
  int pad0, pad1;
};

struct ClShared {                  // head of the dynamic shared memory of every CTA; the per-column state follows it (cl_cols)
  // replicated in every CTA (identical contents: every CTA runs the same bookkeeping on the same messages)
  double u[CL_ROWS];
  int32_t col4row[CL_ROWS];
  int32_t pred_row[CL_ROWS];       // row r was reached through a column whose path predecessor is pred_row[r] (current augmentation)
  uint16_t remaining[CL_MAXC];
  uint16_t remstamp[CL_MAXC];     // 0xFFFF = no entry of the current augmentation
  double rec_min[CL_ROWS];         // step records of the current augmentation (<= assigned columns + 1 <= rows steps)
  int32_t rec_j[CL_ROWS];
  int32_t rec_row[CL_ROWS];
  ClMsg slot[2][CL_N];             // messages of the current / next step
  // per CTA
  Cand part[CL_T / 32];
  int scan[33];
  int step_j, step_next, step_err, nfree;     // result of thread 0's bookkeeping for the other threads; nfree: broadcast by rank 0 between rounds
  double step_min, step_ui;
};
// per-column state of the columns this CTA owns: `cap` columns (= ceil(CL_MAXC / cluster size), a multiple of 8), carved behind ClShared
struct ClColState {
  double *spc, *v;
  int32_t *colstate, *row4col, *path, *pathstamp;
  uint8_t* flags;
};
__host__ __device__ inline int cl_cap(int ncta) { return ((CL_MAXC + ncta - 1) / ncta + 7) & ~7; }
__host__ __device__ inline size_t cl_smem_bytes(int ncta) { return sizeof(ClShared) + (size_t)cl_cap(ncta) * 33 + 16; }
__device__ __forceinline__ ClColState cl_cols(ClShared& S, int ncta) {
  const int cap = cl_cap(ncta);
  unsigned char* p = reinterpret_cast<unsigned char*>(&S) + ((sizeof(ClShared) + 15) & ~(size_t)15);
  ClColState c;
  c.spc = reinterpret_cast<double*>(p); p += (size_t)cap * 8;
  c.v = reinterpret_cast<double*>(p); p += (size_t)cap * 8;
  c.colstate = reinterpret_cast<int32_t*>(p); p += (size_t)cap * 4;
  c.row4col = reinterpret_cast<int32_t*>(p); p += (size_t)cap * 4;
  c.path = reinterpret_cast<int32_t*>(p); p += (size_t)cap * 4;
  c.pathstamp = reinterpret_cast<int32_t*>(p); p += (size_t)cap * 4;
  c.flags = p;
  return c;
}

__device__ __forceinline__ uint32_t cl_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cl_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `p` (a pointer into this CTA's shared memory) in CTA `rank`
__device__ __forceinline__ uint32_t cl_map(const void* p, uint32_t rank) {
  uint32_t r;
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
  return r;
}
__device__ __forceinline__ void cl_st_u64(uint32_t a, unsigned long long v) { asm volatile("st.shared::cluster.b64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ void cl_st_u32(uint32_t a, uint32_t v) { asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void cl_st_u8(uint32_t a, uint32_t v) { asm volatile("st.shared::cluster.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t cl_ld_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared::cluster.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t cl_ld_u8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long cl_ld_u64(uint32_t a) {
  unsigned long long v;
  asm volatile("ld.shared::cluster.b64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
  return v;
}

__device__ __forceinline__ Cand cl_warp_reduce(Cand c) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Cand d;
    d.val = __shfl_xor_sync(0xffffffffu, c.val, o);
    d.st = __shfl_xor_sync(0xffffffffu, c.st, o);
    d.j = __shfl_xor_sync(0xffffffffu, c.j, o);
    c = better(c, d);
  }
  return c;
}

// One linear_sum_assignment of R rows x C columns (R <= C, R <= CL_ROWS, C <= CL_MAXC), entered by every thread of every CTA of the
// cluster.  Returns 0 / 1 (infeasible) / 3 (internal), the same value in every CTA.  S.col4row[R] out (in every CTA).
__device__ __forceinline__ int solve_cl(ClShared& S, const ClColState& L, const uint32_t rank, const int ncta, const float* cost, const float* Tm,
                                        const Ws& w, int N, int n, int R, int C, bool transposed) {
  const int tid = threadIdx.x;
  constexpr int T = CL_T;
  const int Cc = (C + ncta - 1) / ncta;                  // columns per CTA this round (<= cl_cap(ncta): C <= CL_MAXC checked by the host)
  const int c0 = min(C, (int)rank * Cc), c1 = min(C, c0 + Cc);
  for (int i = tid; i < R; i += T) { S.u[i] = 0.0; S.col4row[i] = -1; }
  for (int j = tid; j < C; j += T) S.remstamp[j] = 0xFFFFu;
  for (int j = c0 + tid; j < c1; j += T) {
    const int jl = j - c0;
    L.v[jl] = 0.0; L.row4col[jl] = -1; L.pathstamp[jl] = -1; L.flags[jl] = 0;
  }
  __syncthreads();
  auto row_ptr = [&](int i) -> const float* {
    return transposed ? Tm + (size_t)i * (size_t)N : cost + (size_t)__ldcg(&w.freelist[i]) * (size_t)n;
  };
  float cfn[CL_U];                                       // the cost row of the NEXT augmentation's first step (row cur+1), prefetched
  {
    const float* r0 = row_ptr(0);
#pragma unroll
    for (int q = 0; q < CL_U; ++q) { const int j = c0 + tid + q * T; cfn[q] = (c0 < c1) ? __ldcg(r0 + (j < c1 ? j : c0)) : 0.f; }
  }
  int gstep = 0;                                         // Dijkstra steps since the start of the solve: message buffer parity
  for (int cur = 0; cur < R; ++cur) {
    int i = cur, nrem = C, nsc = 0, sink = -1, sink_pth = cur;
    double minVal = 0.0, ui = 0.0;                       // u[cur] is still 0: a row's dual only changes once the row is assigned
    bool first = true;
    float cf[CL_U];
#pragma unroll
    for (int q = 0; q < CL_U; ++q) cf[q] = cfn[q];
    if (cur + 1 < R && c0 < c1) {                        // in flight during this whole augmentation
      const float* rn = row_ptr(cur + 1);
#pragma unroll
      for (int q = 0; q < CL_U; ++q) { const int j = c0 + tid + q * T; cfn[q] = __ldcg(rn + (j < c1 ? j : c0)); }
    }
    while (sink < 0) {
      Cand best;
      best.val = 0.0; best.st = 0; best.j = -1;
      if (c0 < c1) {
        if (!first) {
          const float* crow = row_ptr(i);
#pragma unroll
          for (int q = 0; q < CL_U; ++q) { const int j = c0 + tid + q * T; cf[q] = __ldcg(crow + (j < c1 ? j : c0)); }
        }
#pragma unroll
        for (int q = 0; q < CL_U; ++q) {
          const int j = c0 + tid + q * T;
          if (j >= c1) continue;
          const int jl = j - c0;
          const double r = ((minVal + (double)cf[q]) - ui) - L.v[jl];        // v[j] is exactly 0 for a column never scanned
          if (first) {
            const int st = (L.flags[jl] & 1) ? -(C - j) : (C - j);         // it = C-1-j  ->  it+1 = C-j
            L.colstate[jl] = st;
            const double s = (r < LSAP_INF) ? r : LSAP_INF;
            L.spc[jl] = s;
            if (s < LSAP_INF) {
              Cand c2;
              c2.val = s; c2.st = st; c2.j = j;
              best = better(best, c2);
            }
          } else {
            const int st = L.colstate[jl];
            if (st == 0) continue;
            double s = L.spc[jl];
            if (r < s) { L.path[jl] = i; L.pathstamp[jl] = cur; L.spc[jl] = r; s = r; }
            if (s < LSAP_INF) {
              Cand c2;
              c2.val = s; c2.st = st; c2.j = j;
              best = better(best, c2);
            }
          }
        }
      }
      first = false;
      // block arg-best -> this CTA's message, stored into every CTA of the cluster
      best = cl_warp_reduce(best);
      if ((tid & 31) == 0) S.part[tid >> 5] = best;
      __syncthreads();                                         // (also: this step's path / spc writes are visible to thread 0)
      const int par = gstep & 1;
      if (tid < 32) {
        Cand r2;
        r2.val = 0.0; r2.st = 0; r2.j = -1;
        if (tid < T / 32) r2 = S.part[tid];
        r2 = cl_warp_reduce(r2);
        if (tid < ncta) {                                      // lane r stores the message into CTA r
          int r4c = -1, pth = cur;
          if (r2.st != 0) {
            const int jl = r2.j - c0;
            r4c = L.row4col[jl];
            pth = (L.pathstamp[jl] == cur) ? L.path[jl] : cur;
          }
          const uint32_t a = cl_map(&S.slot[par][rank], (uint32_t)tid);
          cl_st_u64(a, (unsigned long long)__double_as_longlong(r2.val));
          cl_st_u64(a + 8u, ((unsigned long long)(uint32_t)r2.j << 32) | (uint32_t)r2.st);
          cl_st_u64(a + 16u, ((unsigned long long)(uint32_t)pth << 32) | (uint32_t)r4c);
        }
      }
      cl_sync();                                               // the ONE cluster barrier of the step: all 8 messages are here
      if (tid < 32) {                                          // identical bookkeeping in every CTA: warp 0 picks the winner, lane 0 does the rest
        Cand g;
        g.val = 0.0; g.st = 0; g.j = -1;
        int gi = tid & (CL_N - 1);
        if (tid < ncta) { g.val = S.slot[par][tid].val; g.st = S.slot[par][tid].st; g.j = S.slot[par][tid].j; }
#pragma unroll
        for (int o = CL_N / 2; o > 0; o >>= 1) {
          Cand c2;
          c2.val = __shfl_xor_sync(0xffffffffu, g.val, o);
          c2.st = __shfl_xor_sync(0xffffffffu, g.st, o);
          c2.j = __shfl_xor_sync(0xffffffffu, g.j, o);
          const int ci = __shfl_xor_sync(0xffffffffu, gi, o);
          const Cand b2 = better(g, c2);
          if (b2.j != g.j || b2.st != g.st) { g = b2; gi = ci; }
        }
        if (tid == 0) {
        if (g.st == 0) {
          S.step_err = 1; S.step_j = -1; S.step_next = -1; S.step_min = LSAP_INF; S.step_ui = 0.0;
        } else {
          const int j = g.j;
          const int idx = (g.st > 0 ? g.st : -g.st) - 1;                    // position of j in `remaining`
          const int r4c = S.slot[par][gi].r4c, pth = S.slot[par][gi].pth;
          if (j >= c0 && j < c1) L.colstate[j - c0] = 0;
          if (nsc >= CL_ROWS) { S.step_err = 3; }               // cannot happen: a non-sink step consumes an assigned column (<= rows)
          else { S.rec_j[nsc] = j; S.rec_min[nsc] = g.val; S.rec_row[nsc] = g.st > 0 ? -1 : r4c; }
          const int last = nrem - 1;                                         // swap-with-last removal
          const int jm = (S.remstamp[last] == (uint16_t)cur) ? (int)S.remaining[last] : (C - 1 - last);
          if (jm != j) {
            S.remaining[idx] = (uint16_t)jm;
            S.remstamp[idx] = (uint16_t)cur;
            if (jm >= c0 && jm < c1) {
              const int sm = L.colstate[jm - c0];
              L.colstate[jm - c0] = sm > 0 ? (idx + 1) : -(idx + 1);
            }
          }
          S.step_err = nsc >= CL_ROWS ? 3 : 0; S.step_min = g.val; S.step_j = j;
          if (g.st > 0) {                                                    // an unassigned column: the sink
            S.step_next = -1; S.step_ui = 0.0;
            S.pred_row[cur] = pth;                                           // (slot `cur` is free: row cur is the root) the sink's predecessor
          } else {
            S.step_next = r4c; S.step_ui = S.u[r4c];
            S.pred_row[r4c] = pth;                                           // row r4c is entered through column j, reached from row pth
          }
        }
        }
      }
      __syncthreads();
      if (S.step_err) return S.step_err;
      minVal = S.step_min;
      ++nsc; --nrem; ++gstep;
      if (S.step_next < 0) { sink = S.step_j; sink_pth = S.pred_row[cur]; } else { i = S.step_next; ui = S.step_ui; }
    }
    // dual variables: spc[j] of a scanned column is frozen at the minVal of the step that selected it (rec_min), so every CTA updates its
    // own copy of u and the v / flags of the scanned columns it owns; augmentation: every CTA walks the path on its own row arrays
    __syncthreads();                                           // (thread 0 read pred_row[cur] above before it may be rewritten below)
    if (tid == 0) S.u[cur] += minVal;
    for (int k = tid; k < nsc; k += T) {
      const int j = S.rec_j[k];
      const double d = minVal - S.rec_min[k];
      if (j >= c0 && j < c1) { L.v[j - c0] -= d; L.flags[j - c0] |= (k == nsc - 1) ? 3 : 2; }     // the last record is the sink: now assigned
      if (k < nsc - 1) S.u[S.rec_row[k]] += d;             // distinct rows per k
    }
    if (tid == 32 || (T <= 32 && tid == 0)) {                // another warp than the u[cur] writer's: no ordering needed, distinct data
      int j = sink, r = sink_pth, hops = 0, err = 0;           // (the sink's assigned bit is set by the dual loop: same byte)
      for (;;) {
        if (j >= c0 && j < c1) L.row4col[j - c0] = r;
        const int t = S.col4row[r];
        S.col4row[r] = j;
        if (r == cur) break;
        j = t;
        r = S.pred_row[r];
        if (++hops > R || j < 0) { err = 3; break; }
      }
      S.step_err = err;
    }
    __syncthreads();
    if (S.step_err) return S.step_err;
  }
  cl_sync();                                                   // nobody leaves the solve while a peer may still store a message into it
  return 0;
}

// hungarian_assigner.py:229-270 for one image on a cluster (see hungarian_v2_image in lsap_core.cuh)
__device__ __forceinline__ int hungarian_v2_image_cl(ClShared& S, const uint32_t rank, const int ncta, const float* cost, int N, int n, int topk_k,
                                                     const Ws& w, const int32_t* row_idx, int64_t* out) {
  const ClColState L = cl_cols(S, ncta);
  const int tid = threadIdx.x;
  constexpr int T = CL_T;
  const bool leader = rank == 0;
  if (leader) for (int p = tid; p < N; p += T) w.freelist[p] = p;
  __syncthreads();
  cl_sync();
  int nfree = N;
  const float* Tm = w.T;
  for (int round = 0; round < topk_k; ++round) {
    if (topk_k > 1 && nfree < n) break;                 // `cost_new.shape[0] // num_gts != 0`
    const bool transposed = n < nfree;                  // scipy: transpose iff more rows than columns
    const int R = transposed ? n : nfree, C = transposed ? nfree : n;
    { const int rc = solve_cl(S, L, rank, ncta, cost, Tm, w, N, n, R, C, transposed); if (rc) return rc; }
    if (leader) {
      for (int i = tid; i < R; i += T) {
        const int p = transposed ? w.freelist[S.col4row[i]] : w.freelist[i];
        const int g = transposed ? i : S.col4row[i];
        out[row_idx ? row_idx[p] : p] = (int64_t)g + 1;
      }
      __syncthreads();
    }
    if (!transposed) { nfree = 0; continue; }           // every free proposal got a GT (uniform over the cluster)
    if (leader) {
      for (int i = tid; i < R; i += T) w.freelist[S.col4row[i]] = -1;
      __syncthreads();
      {                                                 // ordered compaction of the free list (see lsap_core.cuh): the leader's 512 threads
        const int seg = (nfree + T - 1) / T;
        const int e0 = min(nfree, tid * seg), e1 = min(nfree, e0 + seg);
        int cnt = 0;
        for (int e = e0; e < e1; ++e) cnt += (w.freelist[e] >= 0) ? 1 : 0;
        const int lane = tid & 31, wi = tid >> 5;
        int inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += t;
        }
        if (lane == 31) S.scan[wi] = inc;
        __syncthreads();
        if (wi == 0) {
          const int t = lane < T / 32 ? S.scan[lane] : 0;
          int ti = t;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int x = __shfl_up_sync(0xffffffffu, ti, o);
            if (lane >= o) ti += x;
          }
          S.scan[lane] = ti - t;
          if (lane == 31) S.scan[32] = ti;
        }
        __syncthreads();
        const int total = S.scan[32];
        int o = S.scan[wi] + inc - cnt;
        for (int e = e0; e < e1; ++e) {
          const int val = w.freelist[e];
          if (val >= 0) w.sc_list[o++] = val;
        }
        __syncthreads();
        for (int e = tid; e < total; e += T) w.freelist[e] = w.sc_list[e];
        if (tid == 0) {
#pragma unroll
          for (int r = 0; r < ncta; ++r) cl_st_u32(cl_map(&S.nfree, (uint32_t)r), (uint32_t)total);
        }
      }
    }
    __syncthreads();
    cl_sync();
    nfree = S.nfree;
    // the next round's matrix, columns = the proposals still free: T2[g][e] = T[g][freelist[e]] — rows dealt to the CTAs; every Dijkstra
    // step of the round then reads its cost row directly (coalesced, no indirection)
    if (round + 1 < topk_k && n < nfree) {
      for (int e0 = tid; e0 < nfree; e0 += 8 * T) {
        int fe[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) { const int e = e0 + q * T; fe[q] = __ldcg(&w.freelist[e < nfree ? e : e0]); }
        for (int g = (int)rank; g < n; g += ncta) {
          const float* s0 = w.T + (size_t)g * (size_t)N;
          float* d0 = w.T2 + (size_t)g * (size_t)N;
          float a0[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) a0[q] = s0[fe[q]];
#pragma unroll
          for (int q = 0; q < 8; ++q) { const int e = e0 + q * T; if (e < nfree) d0[e] = a0[q]; }
        }
      }
      Tm = w.T2;
    }
    __syncthreads();
    cl_sync();
  }
  return 0;
}

}  // namespace ptb_lsap
