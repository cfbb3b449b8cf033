// Negative (out-of-circle) mask over the anchor grid of one FPN level.
// Replaces OutCirclePtFeatGenerator.generate (cpr_head.py:254-290): the per-label Python loop + torch.cdist + min
// becomes one launch; a cell is negative for class c unless some GT of class c lies closer than `thresh`.
// The distance is torch.cdist's fp32 matmul formulation (ptb_common.cuh) so the bool mask is bit-identical to the
// reference CPU head's.  HBM traffic: G*12 B in, B*H*W*num_classes B out.
// The flag tile of a CTA holds NEG_TILE cells x `cc` classes of shared memory; above NEG_MAX_CC classes the classes are split into
// chunks of at most NEG_MAX_CC (grid z), each CTA writing its chunk's columns of the cells' rows.  One chunk is the whole row.
#include "ptb_common.cuh"

namespace ptb {

constexpr int NEG_TILE = 64;   // grid cells per CTA
constexpr int NEG_MAX_CC = (48 * 1024 - 2048) / NEG_TILE;   // classes per chunk: the flag tile stays under the 48 KB default (736)

__global__ void __launch_bounds__(256)
neg_mask_kernel(int H, int W, float stride, const int32_t* __restrict__ pad_hw, const float* __restrict__ centers,
                const int32_t* __restrict__ labels, const int32_t* __restrict__ img_ptr, float thresh, int ncls,
                int class_wise, int cc, uint8_t* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  const int b = blockIdx.y;
  const int cell0 = blockIdx.x * NEG_TILE;
  const int c0 = blockIdx.z * cc;                              // first class of the chunk
  const int nc = min(cc, ncls - c0);                           // classes in the chunk
  const int HW = H * W;
  const int g0 = img_ptr[b], g1 = img_ptr[b + 1];
  const int n = g1 - g0;
  uint8_t* flags = smem_raw;                                   // [NEG_TILE][nc]
  __shared__ float s_px[NEG_TILE], s_py[NEG_TILE], s_pn[NEG_TILE];
  __shared__ uint8_t s_valid[NEG_TILE];
  const int tid = threadIdx.x;
  const float ph = (float)pad_hw[2 * b], pw = (float)pad_hw[2 * b + 1];
  if (tid < NEG_TILE) {
    const int cell = cell0 + tid;
    float px = 0.f, py = 0.f;
    uint8_t v = 0;
    if (cell < HW) {
      const int i = cell / W, j = cell - i * W;
      // cpr_head.py:243  pts = (int grid) * stride + stride / 2
      px = __fadd_rn(__fmul_rn((float)j, stride), __fmul_rn(stride, 0.5f));
      py = __fadd_rn(__fmul_rn((float)i, stride), __fmul_rn(stride, 0.5f));
      v = (0.f <= px) && (px < pw) && (0.f <= py) && (py < ph);
    }
    s_px[tid] = px; s_py[tid] = py; s_pn[tid] = sq_norm2(px, py); s_valid[tid] = v;
  }
  __syncthreads();
  for (int e = tid; e < NEG_TILE * nc; e += blockDim.x) flags[e] = s_valid[e / nc];
  __syncthreads();
  // ATen takes the matmul path when either operand has > 25 rows: rows1 = H*W grid points, rows2 = #centres of the
  // label group (class_wise) or of the image.  Group sizes are only needed when H*W <= 25.
  const bool big_grid = HW > 25;
  // thread layout: 4 threads per cell stride over the GTs
  const int c_local = tid >> 2, sub = tid & 3;
  {
    const float px = s_px[c_local], py = s_py[c_local], pn = s_pn[c_local];
    // conservative pre-filter: a centre further than thresh + 4 px along one axis cannot come out below thresh even with the matmul
    // formulation's rounding (its error near d = thresh is |x|^2 * 2^-23 / (2 thresh) << 1 px at image-scale coordinates; the 0.5 px
    // worst case of SURVEY.md §7.1 is at d ~ 0).  Only ~2 % of an image's GTs pass it: 108 -> ~15 us at the headline batch.
    const float pre = thresh + 4.f;
    for (int g = g0 + sub; g < g1; g += 4) {
      const float cx = centers[2 * g], cy = centers[2 * g + 1];
      if (fabsf(cx - px) > pre || fabsf(cy - py) > pre) continue;
      bool use_mm = big_grid;
      if (!use_mm) {
        int cnt = 0;
        if (class_wise) { for (int q = g0; q < g1; ++q) cnt += (labels[q] == labels[g]); }
        else cnt = n;
        use_mm = cnt > 25;
      }
      const float d = use_mm ? cdist_mm(px, py, pn, cx, cy, sq_norm2(cx, cy)) : cdist_direct(px, py, cx, cy);
      if (!(d >= thresh)) {            // inside the circle: not a negative for that class  (cpr_head.py:278-279)
        if (class_wise) {
          const int c = labels[g] - c0;
          if (0 <= c && c < nc) flags[c_local * nc + c] = 0;
        } else {
          for (int c = 0; c < nc; ++c) flags[c_local * nc + c] = 0;
        }
      }
    }
  }
  __syncthreads();
  const size_t out_base = ((size_t)b * HW + cell0) * ncls + c0;
  const int n_bytes = min(NEG_TILE, HW - cell0) * nc;
  if (nc == ncls) {
    for (int e = tid; e < n_bytes; e += blockDim.x) out[out_base + e] = flags[e];
  } else {
    for (int e = tid; e < n_bytes; e += blockDim.x) {
      const int cell = e / nc;
      out[out_base + (size_t)cell * ncls + (e - cell * nc)] = flags[e];
    }
  }
}

}  // namespace ptb

using namespace ptb;

extern "C" int ptb_cpr_neg_mask(int B, int H, int W, float stride, const int32_t* pad_hw, const float* centers,
                                const int32_t* labels, const int32_t* img_ptr, int G, float thresh, int num_classes,
                                int class_wise, uint8_t* out, void* stream) {
  PTB_REQUIRE(B > 0 && H > 0 && W > 0 && num_classes > 0 && G >= 0, "shape");
  PTB_REQUIRE(pad_hw && img_ptr && out, "NULL input");
  PTB_REQUIRE(G == 0 || (centers && labels), "NULL centers/labels");
  const int chunks = (num_classes + NEG_MAX_CC - 1) / NEG_MAX_CC;
  const int cc = (num_classes + chunks - 1) / chunks;          // balanced chunks of at most NEG_MAX_CC classes
  dim3 grid((H * W + NEG_TILE - 1) / NEG_TILE, B, chunks);
  neg_mask_kernel<<<grid, 256, NEG_TILE * cc, (cudaStream_t)stream>>>(H, W, stride, pad_hw, centers, labels, img_ptr, thresh,
                                                                     num_classes, class_wise, cc, out);
  return check_launch("ptb_cpr_neg_mask");
}
