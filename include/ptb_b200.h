/* ptb_b200.h — C ABI of libptb_b200.so: the H100 (sm_90a) CPR / P2P point-localization hot path.
 *
 * The reference (ucas-vg/PointTinyBenchmark, TOV_mmdetection) is pure Python: it has NO FFI for this path.  Its
 * "plugin boundary" is the mmdet dense-head protocol (HEADS registry).  This header is the C ABI that sits directly
 * under the Python head classes in pointtinybenchmark_b200/ (ctypes binding, see INTEGRATION.md); every entry point
 * names the reference code (file:line under TOV_mmdetection/) it replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers (cudaMalloc'ed / torch CUDA storage) unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); every call is asynchronous on it;
 *   - every function returns 0 on success, non-zero on error; ptb_last_error() gives the message of the last failure
 *     on the calling thread (argument validation errors and CUDA launch errors alike);
 *   - feature / logit maps are channels-last:  map[b][y][x][c], c fastest;  `ld` = floats per (b,y,x) cell;
 *   - point sets of a batch are concatenated over images ("CSR"): img_ptr[b]..img_ptr[b+1] are the GTs of image b;
 *   - bool outputs are uint8_t 0/1;  indices are int32_t unless stated.
 */
#ifndef PTB_B200_H_
#define PTB_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PTB_ABI_VERSION 2

int ptb_abi_version(void);
const char* ptb_last_error(void);
/* number of kernels launched by this library since load (all threads) — bench.py's `gpu_launches` claim */
uint64_t ptb_launch_count(void);
/* The dynamic chunk schedulers and the fixed-order block reductions keep their tickets / partials in a small scratch block owned by
 * the library PER (device, stream) — created on first use — so launches on different streams never share counters.  The counters reset
 * themselves at the end of every kernel; after an ABORTED launch (device fault, killed context) call this to zero the block of `stream`. */
int ptb_reset_stream_state(void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Neighbor gather  — replaces PtFeatGenerator.extract_point_feat + grid_sample
 *   (mmdet/models/point/dense_heads/cpr_head.py:182-199, 73-93) together with
 *   CirclePtFeatGenerator.generate / get_point_neighbours / get_point_valid (cpr_head.py:453-497, 172-180).
 * For every bag g (centre centers[g], image bag_img[g]) and every offset k:  p = centers[g] + offsets[k];
 *   out_pts[g][k]   = (p.x, p.y, stride)
 *   out_valid[g][k] = 0<=p.x<pad_w && 0<=p.y<pad_h                        (pad_hw[b] = {pad_h, pad_w})
 *   out_feats[g][k][0..C) = bilinear sample of map[b] at p/stride, align_corners=False, border padding,
 *                           using ATen's fp32 coordinate pipeline  ix = fma((2u+1)/W-1+1, W/2, -0.5).
 * C must be a multiple of 4 and ld >= C (ld multiple of 4).  Any of out_feats/out_pts/out_valid may be NULL.
 * The same entry point samples the 80-channel logit maps of the fused path (C = num classes).
 */
int ptb_cpr_bag_gather(const float* map, int B, int H, int W, int C, int ld,
                       const float* centers /*[G][2]*/, const int32_t* bag_img /*[G]*/, int G,
                       const float* offsets /*[K][2]*/, int K, float stride,
                       float reach_px /* max_k |offsets[k]| (radius * stride), 0 = unknown: with it and C % 32 == 0 the bag's window of
                                         2*ceil(reach/stride)+2 cells per side is staged per channel chunk by one TMA box */,
                       const int32_t* pad_hw /*[B][2]*/,
                       float* out_feats /*[G][K][C]*/, float* out_pts /*[G][K][3]*/, uint8_t* out_valid /*[G][K]*/,
                       void* stream);

/* backward of the gather w.r.t. the map (scatter-add of bilinear taps; grid_sampler_2d_backward semantics).
 * grad_map must be zero-initialised by the caller; accumulation uses fp32 atomics (red.global.add.v4.f32). */
int ptb_cpr_bag_gather_bwd(const float* grad_out /*[G][K][C]*/, int B, int H, int W, int C, int ld,
                           const float* centers, const int32_t* bag_img, int G,
                           const float* offsets, int K, float stride,
                           float* grad_map /*[B][H][W][ld]*/, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Per-cell linear classifier  y[m][n] = sum_c x[m][c] * w[n][c] + bias[n]   — replaces CPRHead.get_pts_outs
 *   (cpr_head.py:1045-1078: nn.Linear cls_out / ins_out) applied to every map cell (1x1 conv form).
 * x: [M][ldx] (first Cin used), w: [N][Cin] row-major (nn.Linear layout), y: [M][ldy].  Cin % 4 == 0.
 * fp32 FFMA accumulation (parity mode: no TF32).
 */
int ptb_linear_rows(const float* x, int M, int Cin, int ldx, const float* w, const float* bias, int N,
                    float* y, int ldy, void* stream);
/* dX[m][c] = sum_n dY[m][n] w[n][c]   (accumulate=0: overwrite, 1: add) */
int ptb_linear_rows_bwd_x(const float* dy, int M, int N, int ldy, const float* w, int Cin,
                          float* dx, int ldx, int accumulate, void* stream);
/* dW[n][c] = sum_m dY[m][n] x[m][c];  db[n] = sum_m dY[m][n]   (overwrite; fixed-order tree reduction) */
int ptb_linear_rows_bwd_w(const float* dy, int M, int N, int ldy, const float* x, int Cin, int ldx,
                          float* dw /*[N][Cin]*/, float* db /*[N]*/, float* workspace, uint64_t workspace_bytes,
                          void* stream);
uint64_t ptb_linear_rows_bwd_w_workspace(int M, int N, int Cin);

/* ------------------------------------------------------------------------------------------------------------------
 * Negative (out-of-circle) mask — replaces OutCirclePtFeatGenerator.generate (cpr_head.py:254-290) and
 * AnchorPtFeatGenerator.anchor_points (cpr_head.py:240-244) for one FPN level.
 *   grid point (x,y) of cell (i,j) = (j*stride + stride/2, i*stride + stride/2);  cell_valid = inside pad_hw[b];
 *   class_wise:  out[b][i][j][c] = cell_valid && min_{g in image b, labels[g]==c} dist(p, centers[g]) >= thresh
 *   otherwise :  out[b][i][j][c] = cell_valid && min_{g in image b} dist(p, centers[g]) >= thresh       (all c)
 * dist reproduces torch.cdist's matmul formulation in fp32 (the reference's integer mask is defined by it; DESIGN.md).
 */
int ptb_cpr_neg_mask(int B, int H, int W, float stride, const int32_t* pad_hw,
                     const float* centers /*[G][2]*/, const int32_t* labels /*[G]*/, const int32_t* img_ptr /*[B+1]*/,
                     int G, float thresh, int num_classes, int class_wise,
                     uint8_t* out /*[B][H][W][num_classes]*/, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Point refinement — replaces PointRefiner.refine_single with nearest_filter / classify_filter / inside_img
 *   (cpr_head.py:780-850, 711-756, 773-778).
 * Kt = num_refine * K samples per GT; the centre of refine 0 is sample `center_idx` (= K-1).
 * grp_ptr/grp_idx: CSR of same-(image,label) GT groups: members of GT g's group are
 *   grp_idx[grp_ptr[grp_of[g]] .. grp_ptr[grp_of[g]+1]) in ascending GT order (host builds it; it is the
 *   group_by_label of cpr_head.py:64-70 without the device->host sync).
 * flags: bit0 nearest_filter, bit1 classify_filter, bit2 return_score_type=='max'.
 */
typedef struct {
  float merge_th, gt_alpha, refine_th;
  int32_t flags;
} ptb_refine_cfg;

/* ---------------------------------------------------------------------------------------------------------
 * a8  grid-cell ("neighbour index") bags: GridPtFeatGenerator.generate + GridCirclesPtFeatGenerator.get_chosen_neighbours
 *     (cpr_head.py:296-350, 418-444), num_refine == 1.
 * Bag of GT g = [cells whose centre (j*stride + stride/2, i*stride + stride/2) lies within radius_px of the GT, row-major |
 *                zero padding up to max_pos_num + 1 slots | the GT centre], Kt = max_pos_num + 2 slots.
 *   out_feats [G][Kt][C]  exact copies of the map's cell vectors, zeros in the padding, bilinear sample for the centre
 *   out_pts   [G][Kt][3]  (x, y, stride); zeros in the padding
 *   out_valid [G][Kt]     1 for filled cell slots and the centre (not tested against pad_shape: cpr_head.py:329)
 *   out_cell  [G][Kt]     int32 linear cell index i*W + j of the slot (the neighbour index; bit-exact target),
 *                         -1 = padding, -2 = the centre sample
 *   overflow  device int32 set to 1 if some GT has more than max_pos_num + 1 chosen cells (the reference raises there)
 * Any output pointer may be NULL.  map is channels-last [B][H][W][ld], C % 4 == 0. */
int ptb_cpr_grid_bag(const float* map, int B, int H, int W, int C, int ld, const float* centers /*[G][2]*/,
                     const int32_t* bag_img /*[G]*/, int G, float stride, float radius_px, int max_pos_num,
                     float* out_feats, float* out_pts, uint8_t* out_valid, int32_t* out_cell, int32_t* overflow,
                     void* stream);
/* backward of the above w.r.t. the map: grad_map [B][H][W][ld] += scatter(grad_out [G][Kt][C]) (caller zero-fills) */
int ptb_cpr_grid_bag_bwd(const float* grad_out, int B, int H, int W, int C, int ld, const float* centers,
                         const int32_t* bag_img, const int32_t* cell_idx /*[G][Kt] from the forward*/, int G, int Kt,
                         float stride, float* grad_map, void* stream);

/* builds that CSR on the device (no host sync): groups numbered image-major / label-minor, members in ascending GT order.
 * grp_of [G], grp_ptr [G+1] (entries past the last group are filled with G), grp_idx [G].  max_per_image <= 8192. */
int ptb_label_groups(const int32_t* labels /*[G]*/, const int32_t* img_ptr /*[B+1]*/, int B, int G, int num_classes,
                     int max_per_image, int32_t* grp_of, int32_t* grp_ptr, int32_t* grp_idx, void* stream);

/* stage form: consumes materialised probabilities (bit-exact masks vs the oracle given the same probs) */
int ptb_cpr_refine(const float* bag_prob /*[G][Kt][num_classes]*/, const float* bag_pts /*[G][Kt][3]*/,
                   const uint8_t* bag_valid /*[G][Kt]*/, int G, int Kt, int K, int num_classes,
                   const int32_t* labels /*[G]*/, const int32_t* bag_img /*[G]*/, const int32_t* img_hw /*[B][2]*/,
                   const int32_t* grp_of /*[G]*/, const int32_t* grp_ptr, const int32_t* grp_idx,
                   const uint8_t* not_refine_in /*[G] or NULL*/, ptb_refine_cfg cfg,
                   float* out_pts /*[G][2]*/, float* out_score /*[G]*/, uint8_t* out_not_refine /*[G]*/,
                   uint8_t* out_chosen /*[G][Kt] or NULL*/, uint8_t* out_merge_valid /*[G][Kt] or NULL*/,
                   void* stream);

/* fused form (production): samples the class-logit map on the fly (bilinear), sigmoid, filters, merge — the
 * (G,K,num_classes) probability tensor is never written.  num_refine == 1.  Replaces CPRHead.get_bboxes'
 * extract -> get_pts_outs -> get_cls_prob -> PointRefiner chain (cpr_head.py:1248-1257). */
int ptb_cpr_refine_fused(const float* logit_map /*[B][H][W][ld]*/, int B, int H, int W, int num_classes, int ld,
                         const float* centers /*[G][2]*/, const int32_t* labels, const int32_t* bag_img, int G,
                         const float* offsets /*[K][2]*/, int K, float stride,
                         float reach_px /* max_k |offsets[k]| (e.g. radius*stride), 0 = unknown: selects the shared-memory window
                                           of 2*ceil(reach/stride)+2 cells per side that one TMA box stages per GT */,
                         const int32_t* pad_hw, const int32_t* img_hw,
                         const int32_t* grp_of, const int32_t* grp_ptr, const int32_t* grp_idx,
                         const uint8_t* not_refine_in, ptb_refine_cfg cfg,
                         float* out_pts, float* out_score, uint8_t* out_not_refine,
                         uint8_t* out_chosen /*[G][K] or NULL*/, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * MIL bag loss — replaces MILLoss.forward (mmdet/models/losses/multi_instance_learning_loss.py:153-203,
 * binary_ins=False, gfocal) on bags whose cls/ins logits are given as [G][Kt][ld] rows (cls at column 0,
 * ins at column ins_off).  weight[g][k] = valid * gt_weight (cpr_head.py:1211).
 *   out_bag_prob[g][c] = sum_k sigmoid(cls) * normalize_L1(softmax_k(ins) * weight)
 *       (the buffer must hold G*num_classes + 3*G floats: the trailing 3*G are per-bag loss / weight / hit scratch)
 *   out_loss_sum[0]   += sum_g term(bag_prob[g], onehot(labels[g])) * (any_k weight>0)      (un-normalised; term below)
 *   out_stats[0] += #bags with any weight>0 ; out_stats[1] += #bags whose argmax (first maximum) == label
 * num_classes <= 1280; above 256 the classes are processed in chunks of 256 lanes, each per-(bag, class) sum in the same order.
 * bwd: d(loss_sum)/d(cls logits), d/d(ins logits) scaled by `scale` (= loss_weight / num_sample).
 * loss_kind selects the loss term of the positive bags (MILLoss / AllPosLoss `loss_type`, multi_instance_learning_loss.py:187-202, 229-240):
 *   PTB_LOSS_GFOCAL  gfocal_loss(p, onehot) x label weight (the bag's any-weight flag for MIL, w_k for AllPos)
 *   PTB_LOSS_BCE     F.binary_cross_entropy(p, onehot) UNWEIGHTED: (t-1) max(log1p(-p), -100) - t max(log p, -100), as ATen on the CPU;
 *                    a MIL bag whose weights are all zero (prob = 0) still adds 100 at its label column, with zero gradient.
 *                    A probability above 1 (rounding of saturated sigmoids; ATen raises) gives NaN.
 */
#define PTB_LOSS_GFOCAL 0
#define PTB_LOSS_BCE 1
int ptb_mil_loss_fwd(const float* logits /*[G][Kt][ld]*/, int G, int Kt, int num_classes, int ld, int ins_off,
                     const float* weight /*[G][Kt]*/, const int32_t* labels, float eps, int loss_kind,
                     float* out_bag_prob /*[G][num_classes]*/, float* out_loss_sum /*[1]*/, float* out_stats /*[2]*/,
                     float* out_mt /*[G][num_classes][2] = (max_k ins, 1/T or 0 if the L1-normalisation clamp is active) or NULL:
                                     what ptb_cpr_loss_bwd_map needs of the forward*/,
                     void* stream);
int ptb_mil_loss_bwd(const float* logits, int G, int Kt, int num_classes, int ld, int ins_off,
                     const float* weight, const int32_t* labels, float eps, int loss_kind, const float* bag_prob,
                     const float* scale /*[1] device scalar*/, float* grad_logits /*[G][Kt][ld], cls+ins columns written*/,
                     void* stream);
/* AllPosLoss forward (multi_instance_learning_loss.py:206-243): every bag sample is a row p = sigmoid(logits[g][k][0..num_classes)) with
 * the label of its bag.  aux [3*G] scratch; fixed-order sums (deterministic):
 *   out_loss_sum[0] += sum_{g,k,c} term(p, onehot) (x weight[g][k] for PTB_LOSS_GFOCAL; unweighted over ALL samples for PTB_LOSS_BCE)
 *   out_stats[0] += #samples with weight > 0 ;  out_stats[1] += #samples whose top-1 class (first maximum) == label */
int ptb_cpr_allpos_fwd(const float* logits /*[G][K][ld]*/, int G, int K, int num_classes, int ld, const float* weight /*[G][K]*/,
                       const int32_t* labels, float eps, int loss_kind, float* aux, float* out_loss_sum /*[1]*/, float* out_stats /*[2]*/,
                       void* stream);

/* Fused bag gather + MIL forward (ring bags, num_classes <= 128): samples the [cls | ins] logit map (columns 0.. and ins_off..) at every
 * bag point like ptb_cpr_bag_gather, writes the sampled rows (out_bag_logits [G][K][ld], needed by the backward), the sample validity
 * as weights (out_weight [G][K] = 0/1), and evaluates ptb_mil_loss_fwd on the fly with online softmax accumulators: the (G,K,ld) tensor
 * is written once and never re-read by the forward.  out_bag_prob needs G*num_classes + 3*G floats like ptb_mil_loss_fwd. */
int ptb_cpr_bag_mil_fwd(const float* logit_map /*[B][H][W][ld]*/, int B, int H, int W, int ld, int num_classes, int ins_off,
                        const float* centers, const int32_t* bag_img, int G, const float* offsets, int K, float stride,
                        const int32_t* pad_hw, const int32_t* labels, float eps, int loss_kind, float* out_bag_logits, float* out_weight,
                        float* out_bag_prob, float* out_loss_sum /*[1]*/, float* out_stats /*[2]*/, float* out_mt /*[G][N][2] or NULL*/,
                        void* stream);

/* Backward of the whole CPR training loss w.r.t. the LOGIT MAP in one deterministic kernel (gather formulation, no atomics on global
 * memory): replaces autograd of MILLoss (multi_instance_learning_loss.py:153-203), of the gt / neg gfocal terms (cpr_head.py:1159-1184,
 * 1219-1228) and of grid_sample (cpr_head.py:73-93) for ring bags.
 *   grad_map[b][y][x][ch] = sum_{bag g of image b, sample k, tap t on (y,x)} w_t * dLoss/d bag_logits[g][k][ch]
 *                         + [ch < num_classes] scale_neg * neg_mask * d gfocal(sigmoid(logit_map), 0)           (if logit_map != NULL)
 * with dLoss/d bag_logits from scale_mil (MIL term; needs bag_prob, mil_mt, label_weight = the trailing [G..2G) aux floats of
 * ptb_mil_loss_fwd's out_bag_prob buffer) and scale_gt * valid_center (gt term on the centre sample k = K-1).  Every element of
 * grad_map is written (no zero-init needed).  One CTA per 8x8-cell tile; every sum is formed by one thread in a fixed order, so the
 * result is bit-identical run to run.  ld must be a multiple of 32 and at most 160 (every such ld, 32 to 160, is exact: narrow rows run
 * smaller blocks and rounds of blockDim / 4 samples); K <= 320; reach_px must be at least the largest |offset| component, or samples
 * outside the window are lost.
 * loss_kind is that of the bag term and of the per-sample positive term (AllPosLoss):
 *   mil_mt == NULL      no MIL term (bag_prob, label_weight, scale_mil unused; the ins columns get no gradient);
 *   scale_pos != NULL   every sample k of every bag adds scale_pos * w * term'(sigmoid(cls)) * sigmoid'(cls) to its cls columns, with
 *                       w = weight[g][k] for PTB_LOSS_GFOCAL and w = 1 for PTB_LOSS_BCE (samples outside pad_shape included). */
int ptb_cpr_loss_bwd_map(const float* bag_logits /*[G][K][ld]*/, const float* weight /*[G][K]*/, const float* mil_mt /*[G][N][2] or NULL*/,
                         const float* bag_prob /*[G][N]*/, const float* label_weight /*[G]*/, const int32_t* labels,
                         const float* centers /*[G][2]*/, const int32_t* img_ptr /*[B+1]*/, const float* offsets /*[K][2]*/,
                         int B, int H, int W, int G, int K, int num_classes, int ins_off, int ld, float stride, float reach_px, float eps,
                         const float* scale_mil /*[1] or NULL*/, const float* scale_gt /*[1] or NULL*/,
                         const float* valid_center /*[G] or NULL*/, const float* logit_map /*[B][H][W][ld] or NULL*/,
                         const uint8_t* neg_mask /*[B][H][W][N]*/, const float* scale_neg /*[1]*/,
                         int loss_kind, const float* scale_pos /*[1] or NULL*/,
                         void* workspace /*ptb_cpr_loss_bwd_map_workspace(G, N) bytes, 16-byte aligned*/,
                         float* grad_map /*[B][H][W][ld]*/, void* stream);
uint64_t ptb_cpr_loss_bwd_map_workspace(int G, int num_classes);
/* Scatter form of the MIL + gt part of the same gradient (fastest; fp32 vector atomics, so NOT bit-reproducible): one CTA per bag adds
 * w_tap * dLoss/d bag_logits straight into grad_map, which the caller has initialised (zeros, or the neg-loss term written by
 * ptb_sigmoid_loss_bwd).  Same inputs as ptb_cpr_loss_bwd_map except bag_img [G] instead of img_ptr; workspace as above. */
int ptb_cpr_loss_bwd_scatter(const float* bag_logits, const float* weight, const float* mil_mt, const float* bag_prob,
                             const float* label_weight, const int32_t* labels, const float* centers, const int32_t* bag_img,
                             const float* offsets, int B, int H, int W, int G, int K, int num_classes, int ins_off, int ld,
                             float stride, float eps, const float* scale_mil, const float* scale_gt, const float* valid_center,
                             int loss_kind, const float* scale_pos /*[1] or NULL*/,
                             void* workspace, float* grad_map /*[B][H][W][ld], accumulated into*/, void* stream);

/* gfocal on sigmoid(logits) vs a one-hot / all-zero target with per-element weights — replaces
 * MILLoss.gfocal_loss (multi_instance_learning_loss.py:148-151) as used for gt_loss and neg_loss
 * (cpr_head.py:1159-1184, 1219-1228).  rows: logits[m*row_stride + c], c<num_classes;
 * target_label[m] in [0,num_classes) or -1 (all-zero target); weight is uint8 [M][num_classes] (wmode 0),
 * float [M] (wmode 1) or NULL (all ones).  loss_sum[0] += sum.   bwd: grad = scale[0] * dloss/dlogit (overwrite or add), where the loss
 * is this gfocal for PTB_LOSS_GFOCAL and weight * BCE(sigmoid(logit), target) for PTB_LOSS_BCE. */
int ptb_gfocal_sigmoid_fwd(const float* logits, int64_t M, int num_classes, int64_t row_stride,
                           const int32_t* target_label, const void* weight, int wmode, float eps,
                           float* loss_sum, void* stream);
int ptb_sigmoid_loss_bwd(const float* logits, int64_t M, int num_classes, int64_t row_stride, const int32_t* target_label,
                         const void* weight, int wmode, float eps, int loss_kind, const float* scale, float* grad,
                         int64_t grad_row_stride, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * P2P decode + top-k — replaces P2PHead.get_pred_points (p2p_head.py:125-170) and the per-level
 * max-over-classes + topk(nms_pre) of _get_bboxes_single (p2p_head.py:362-376).
 * cls_map [B][H][W][k*C] logits, reg_map [B][H][W][2k]; proposal index q = (i*W+j)*k + a.
 *   out_topk_idx[b][r]  = index of the r-th largest max_c sigmoid(cls[q][c]) (ties: lower index first)
 *   out_pts[b][r]       = clamp(anchor + reg*gamma*stride, [0,img_w]x[0,img_h])   (optionally / scale_factor)
 *   out_scores[b][r][c] = sigmoid(cls[topk][c])
 * nms_pre >= number of proposals keeps every proposal in index order (reference skips top-k then).
 */
int ptb_p2p_decode_topk(const float* cls_map, const float* reg_map, int B, int H, int W, int num_classes, int k,
                        const float* point_anchor /*[k][2]*/, float stride, float pts_gamma,
                        const int32_t* img_hw, const float* scale_xy /*[B][2] or NULL*/, int nms_pre,
                        int32_t* out_topk_idx /*[B][P]*/, float* out_pts /*[B][P][2]*/, float* out_scores /*[B][P][C]*/,
                        void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_p2p_decode_topk_workspace(int B, int H, int W, int k);
/* Softmax classification (CrossEntropyLoss(use_sigmoid=False), p2p_head.py:63-67,363,370): the same arguments, workspace and outputs,
 * but a cls row holds num_classes + 1 logits, background last (cls_map [B][H][W][k*(C+1)]):
 *   key[q]              = max_{c<C} softmax(cls[q])[c] = exp(max_{c<C} x_c - m) / s,  m = max over the C+1 logits, s = sum exp(x - m)
 *   out_topk_idx[b][r]  = index of the r-th largest key (ties: lower index first)
 *   out_scores[b][r][c] = softmax(cls[topk])[c] for the C foreground classes (multiclass_nms drops the background column);
 *                         max_c out_scores[b][r][c] equals that proposal's key bit for bit.
 * Probabilities are within a few ulps of ATen's CPU softmax, not bit-identical to it. */
int ptb_p2p_decode_topk_softmax(const float* cls_map, const float* reg_map, int B, int H, int W, int num_classes, int k,
                                const float* point_anchor /*[k][2]*/, float stride, float pts_gamma,
                                const int32_t* img_hw, const float* scale_xy /*[B][2] or NULL*/, int nms_pre,
                                int32_t* out_topk_idx /*[B][P]*/, float* out_pts /*[B][P][2]*/, float* out_scores /*[B][P][C]*/,
                                void* workspace, uint64_t workspace_bytes, void* stream);
/* Several FPN levels (P2PHead with strides [s_0, ..., s_{L-1}], p2p_head.py:125-170, 345-381), sigmoid or softmax scores as above.
 * Level l: cls_maps[l] [B][H_l][W_l][k*C1], reg_maps[l] [B][H_l][W_l][2k], hw[l] = (H_l, W_l), strides[l] (host arrays of L <= 8
 * entries; the maps are device pointers).  An image's T = sum_l H_l W_l k rows are the levels' proposals, level-major.  As the
 * reference's _get_bboxes_single, the rows are split into L equal chunks of T / L rows (not into levels: a chunk may straddle
 * levels), and each chunk keeps its top nms_pre rows by the max foreground score (ties: lower index first), or all of its rows when
 * nms_pre <= 0 or nms_pre >= T / L.  P = rows kept per chunk; output row r of image b is entry r % P of chunk r / P:
 *   out_topk_idx[b][r] = the chunk-local row index (reference topk_inds),  out_pts / out_scores as above with the row's own stride.
 * T % L != 0 is refused (the reference's reshape raises there).  nms_pre <= 4096.  workspace: ptb_p2p_decode_topk_levels_workspace. */
int ptb_p2p_decode_topk_levels(const float* const* cls_maps, const float* const* reg_maps, int L, const int32_t* hw /*[L][2]*/,
                               const float* strides /*[L]*/, int B, int num_classes, int k, const float* point_anchor /*[k][2]*/,
                               float pts_gamma, const int32_t* img_hw, const float* scale_xy /*[B][2] or NULL*/, int nms_pre,
                               int32_t* out_topk_idx /*[B][L*P]*/, float* out_pts /*[B][L*P][2]*/, float* out_scores /*[B][L*P][C]*/,
                               void* workspace, uint64_t workspace_bytes, void* stream);
int ptb_p2p_decode_topk_levels_softmax(const float* const* cls_maps, const float* const* reg_maps, int L, const int32_t* hw,
                                       const float* strides, int B, int num_classes, int k, const float* point_anchor, float pts_gamma,
                                       const int32_t* img_hw, const float* scale_xy, int nms_pre, int32_t* out_topk_idx,
                                       float* out_pts, float* out_scores, void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_p2p_decode_topk_levels_workspace(int B, int L, const int32_t* hw /*[L][2]*/, int k);

/* ------------------------------------------------------------------------------------------------------------------
 * multiclass NMS — replaces multiclass_nms (mmdet/core/post_processing/bbox_nms.py:7-94) and the third-party
 * mmcv.ops.nms.batched_nms it calls (mmcv-full 1.3.x, not vendored; semantics restated in oracle/p2p.py).
 * Per image b: candidates = (point p, class c) with scores[b][p][c] > score_thr, flat id = p*C+c, in flat order;
 * box = pts[p] -/+ pseudo_wh/2 offset by c*(max_coord+1);  greedy NMS by descending score (ties: lower flat id first),
 * suppress IoU > iou_thr;  keep the first max_per_img.
 *   out_count[b], out_det[b][r] = (x1,y1,x2,y2,score), out_label[b][r], out_keep[b][r] = index into the candidate list,
 *   out_cand_count[b] = number of candidates.
 */
int ptb_multiclass_nms(const float* pts /*[B][P][2]*/, const float* scores /*[B][P][C]*/, int B, int P, int num_classes,
                       float pseudo_w, float pseudo_h, float score_thr, float iou_thr, int max_per_img,
                       int32_t* out_count /*[B]*/, float* out_det /*[B][max][5]*/, int32_t* out_label /*[B][max]*/,
                       int32_t* out_keep /*[B][max]*/, int32_t* out_cand_count /*[B]*/,
                       void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_multiclass_nms_workspace(int B, int P, int num_classes);
/* same with explicit boxes [B][P][4] (x1,y1,x2,y2) instead of point pseudo-boxes: the second NMS of the test-time-aug /
 * tile merge path (P2PHead.aug_test_bboxes, p2p_head.py:487-572; dense_test_mixins.py:173-204). */
int ptb_multiclass_nms_boxes(const float* boxes /*[B][P][4]*/, const float* scores /*[B][P][C]*/, int B, int P, int num_classes,
                             float score_thr, float iou_thr, int max_per_img,
                             int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                             void* workspace, uint64_t workspace_bytes, void* stream);

/* soft-NMS variant (nms=dict(type='soft_nms', iou_threshold, sigma=0.5, min_score=1e-3, method='linear'|'gaussian'|'naive') through
 * batched_nms; mmcv.ops.nms.soft_nms is third-party (mmcv-full 1.3.x) — its published CPU kernel is restated in
 * oracle/p2p.py::soft_nms; no reference test pins it: parity unpinned).  Same candidate list, class offset and outputs as
 * ptb_multiclass_nms, but out_det[..][4] is the DECAYED score and the order is the soft-NMS selection order (non-increasing decayed
 * score).  Give either pts (pseudo boxes) or boxes.  method: 0 naive, 1 linear, 2 gaussian.
 * Images whose classes are not separated by the class offset (negative coordinates on near-square images) take an exact global
 * path, like ptb_multiclass_nms.  Naive needs iou_thr > 0.  Gaussian refuses an image with two candidate boxes of zero area (after
 * the class offset) or one of negative / NaN area, where mmcv's weight exp(-(0/0)^2 / sigma) is NaN: out_count[b] = -1 there. */
int ptb_multiclass_soft_nms(const float* pts /*[B][P][2] or NULL*/, const float* boxes /*[B][P][4] or NULL*/,
                            const float* scores /*[B][P][C]*/, int B, int P, int num_classes, float pseudo_w, float pseudo_h,
                            float score_thr, float iou_thr, float sigma, float min_score, int method, int max_per_img,
                            int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                            void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_multiclass_soft_nms_workspace(int B, int P, int num_classes);

/* class-specific boxes [B][P][C][4] (x1,y1,x2,y2): candidate (p, c) uses boxes[b][p][c] - the RoI head's multiclass_nms with
 * bboxes (n, 4*C).  Everything else as ptb_multiclass_nms_boxes / ptb_multiclass_soft_nms with boxes: the candidate list, the
 * `keep` ranks (box-major, class-minor), max_coord over the candidates' own boxes, the `slow` test over every candidate box and
 * the exact global path below 10000 candidates, the per-class kernels and the merge from 10000 on.  Limits as there: P <= 4096
 * boxes per image, max_per_img in [1, 1024]; the workspaces are ptb_multiclass_nms_workspace(B, P, C) and
 * ptb_multiclass_soft_nms_workspace(B, P, C).  Gaussian soft-NMS refuses an image on its candidates' own boxes. */
int ptb_multiclass_nms_cls_boxes(const float* boxes /*[B][P][C][4]*/, const float* scores /*[B][P][C]*/, int B, int P, int num_classes,
                                 float score_thr, float iou_thr, int max_per_img,
                                 int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                                 void* workspace, uint64_t workspace_bytes, void* stream);
int ptb_multiclass_soft_nms_cls_boxes(const float* boxes /*[B][P][C][4]*/, const float* scores /*[B][P][C]*/, int B, int P,
                                      int num_classes, float score_thr, float iou_thr, float sigma, float min_score, int method,
                                      int max_per_img, int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep,
                                      int32_t* out_cand_count, void* workspace, uint64_t workspace_bytes, void* stream);
/* ptb_multiclass_nms / ptb_multiclass_soft_nms (point pseudo-boxes or shared boxes) for up to 8192 points per image, e.g. the
 * multi-level P2P head's L x nms_pre candidates.  Same arguments, workspaces (ptb_multiclass_nms_workspace,
 * ptb_multiclass_soft_nms_workspace) and results. */
int ptb_multiclass_nms_wide(const float* pts /*[B][P][2]*/, const float* scores /*[B][P][C]*/, int B, int P, int num_classes,
                            float pseudo_w, float pseudo_h, float score_thr, float iou_thr, int max_per_img,
                            int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                            void* workspace, uint64_t workspace_bytes, void* stream);
int ptb_multiclass_soft_nms_wide(const float* pts /*[B][P][2] or NULL*/, const float* boxes /*[B][P][4] or NULL*/,
                                 const float* scores /*[B][P][C]*/, int B, int P, int num_classes, float pseudo_w, float pseudo_h,
                                 float score_thr, float iou_thr, float sigma, float min_score, int method, int max_per_img,
                                 int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep, int32_t* out_cand_count,
                                 void* workspace, uint64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Hungarian cost matrix — replaces FocalLossCost + DisCostV2 (mmdet/core/bbox/match_costs/match_cost.py:94-99,
 * 197-214) as summed by HungarianAssignerV2.assign (hungarian_assigner.py:222-227).
 *   cost[q][g] = w_cls*(pos(p)-neg(p)) at column labels[g] + w_dis * sum_d |pts[q][d]/f_d - gts[g][d]/f_d|
 * rows = the n_rows proposals listed in row_idx (the valid ones), written densely [n_rows][n_gt].
 */
int ptb_p2p_cost_matrix(const float* cls_logits /*[Q][C]*/, const float* pts /*[Q][ldp]*/, int ldp,
                        const int32_t* row_idx /*[n_rows] or NULL*/, int n_rows, int num_classes,
                        const float* gts /*[n_gt][2]*/, const int32_t* gt_labels, int n_gt,
                        float w_cls, float alpha, float gamma, float eps, float w_dis, float fx, float fy,
                        float* cost, void* stream);

/* Hungarian cost matrix over a list of match costs — HungarianAssignerV2.assign's `sum(cls_costs) + sum(reg_costs)`
 * (hungarian_assigner.py:223-227) for the point costs of match_cost.py:
 *   PTB_MATCH_COST_FOCAL        FocalLossCost(weight, alpha, gamma, eps)                    (classification)
 *   PTB_MATCH_COST_CLS_SIGMOID  ClassificationCostV2(use_sigmoid=True):  -sigmoid(x)[:, l] * w
 *   PTB_MATCH_COST_CLS_SOFTMAX  ClassificationCostV2(use_sigmoid=False): -softmax(x, -1)[:, l] * w over all num_cols columns
 *   PTB_MATCH_COST_ZERO         ZeroCost (contributes 0)
 *   PTB_MATCH_COST_DIS          DisCostV2(weight, norm_with_img_wh, p = 1 or 2) on (x, y)     (regression)
 * The classification terms are summed in list order from 0, the DisCostV2 terms likewise, then the two sums are added.  At most
 * PTB_MAX_MATCH_COST_TERMS of each.  DisCostV2 divides by (img_w, img_h) when norm_with_img_wh is set.  p = 2 follows torch.cdist's
 * CPU dispatch: the matmul formulation when n_rows > 25 or n_gt > 25, the direct one otherwise.
 * workspace: ptb_p2p_cost_matrix_terms_workspace(n_rows) bytes when a CLS_SOFTMAX term is listed (per-row softmax statistics),
 * else may be NULL. */
#define PTB_MATCH_COST_FOCAL 0
#define PTB_MATCH_COST_CLS_SIGMOID 1
#define PTB_MATCH_COST_CLS_SOFTMAX 2
#define PTB_MATCH_COST_ZERO 3
#define PTB_MATCH_COST_DIS 4
#define PTB_MAX_MATCH_COST_TERMS 8
typedef struct {
  int32_t kind;                             /* PTB_MATCH_COST_* */
  float weight, alpha, gamma, eps;          /* alpha, gamma, eps: FocalLossCost only */
  int32_t p;                                /* DisCostV2 only: 1 or 2 */
  int32_t norm_with_img_wh;                 /* DisCostV2 only */
} ptb_match_cost;
int ptb_p2p_cost_matrix_terms(const float* cls_logits /*[Q][num_cols]*/, const float* pts /*[Q][ldp]*/, int ldp,
                              const int32_t* row_idx /*[n_rows] or NULL*/, int n_rows, int num_cols,
                              const float* gts /*[n_gt][2]*/, const int32_t* gt_labels, int n_gt,
                              const ptb_match_cost* terms, int n_terms, float img_w, float img_h,
                              float* cost, void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_p2p_cost_matrix_terms_workspace(int n_rows);

/* ------------------------------------------------------------------------------------------------------------------
 * RPN proposals for dense anchors — replaces RPNHead._get_bboxes (mmdet/models/dense_heads/rpn_head.py:78-186) with the grid
 * anchors of AnchorGenerator (mmdet/core/anchor/anchor_generator.py:207-270), DeltaXYWHBBoxCoder.decode
 * (mmdet/core/bbox/coder/delta_xywh_bbox_coder.py:144-270, clip_border=True) and mmcv batched_nms over level ids, for a batch.
 *   cls_scores[l] : device (B, A, H_l, W_l) NCHW logits (use_sigmoid_cls);  bbox_preds[l] : device (B, 4A, H_l, W_l)
 *   level_hw      : HOST [L][2] (H_l, W_l);  strides_wh : HOST [L][2] (stride_w, stride_h);  base_anchors : DEVICE [L][A][4]
 *   img_hw        : DEVICE [B][2] = img_shape (h, w) -> clip range;  means, stds : HOST [4]
 *   per level: sigmoid, top-nms_pre by (score desc, anchor index asc) when the level has more than nms_pre anchors (else all, in
 *   index order), decode, clip;  then drop boxes with w <= min_bbox_size or h <= min_bbox_size (min_bbox_size < 0: keep all),
 *   greedy NMS (IoU > iou_thr) per level on coordinates offset by level*(boxes.max()+1), merge by descending score, first max_per_img.
 *   out_det [B][max_per_img][5] (x1,y1,x2,y2,score), out_count[B], out_level[B][max_per_img];
 *   optional (may be NULL): out_pos [B][max_per_img] position in the candidate list, out_cand_box [B][Ptot][4] (16-byte aligned),
 *   out_cand_score [B][Ptot], out_cand_idx [B][Ptot] (anchor index q = (y*W+x)*A + a inside its level), Ptot = sum_l min(nms_pre, H_l*W_l*A).
 * Limits: L <= 8, nms_pre <= 4096 (every level keeps <= 4096 candidates), max_per_img <= 2048.
 */
uint64_t ptb_rpn_proposals_workspace(const int32_t* level_hw, int L, int B, int A, int nms_pre, int max_per_img);
int ptb_rpn_proposals(const float* const* cls_scores, const float* const* bbox_preds, const int32_t* level_hw,
                      const int32_t* strides_wh, const float* base_anchors, int L, int B, int A, const int32_t* img_hw,
                      const float* means, const float* stds, float wh_ratio_clip, int nms_pre, float min_bbox_size,
                      float iou_thr, int max_per_img, int32_t* out_count, float* out_det, int32_t* out_level,
                      int32_t* out_pos, float* out_cand_box, float* out_cand_score, int32_t* out_cand_idx,
                      void* workspace, uint64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * HungarianAssignerV2 matching — replaces `cost.detach().cpu()` + the <= topk_k scipy.optimize.linear_sum_assignment solves of
 * HungarianAssignerV2.assign (mmdet/core/bbox/assigners/hungarian_assigner.py:229-270) for a whole batch, without a host
 * round trip.  scipy's algorithm (rectangular_lsap: shortest augmenting paths, fp64 duals, transpose rule, tie rule) is
 * restated bit-for-bit (oracle/lsap.c is pinned to scipy; pointtinybenchmark_b200/csrc/lsap_core.cuh is the parallel form, one CTA per
 * image; csrc/lsap_cluster.cuh solves an image on a cluster of 8 / 6 / 5 CTAs — the default up to 17 600 columns x 1024 rows).
 *   cost      : concatenated per-image cost matrices, image b = [N_b][n_b] fp32 row-major (proposals x GTs, as the reference
 *               builds it) at element offset desc[b][0]
 *   desc      : DEVICE int64 [num_images][6] = {cost_off, workspace byte offset (multiple of 8), gt_inds element offset,
 *               row_idx element offset or -1, N_b, n_b}
 *   row_idx   : optional map from the cost row to the slot inside the image's gt_inds slice (the valid proposals)
 *   gt_inds   : int64, PRE-ZEROED by the caller; matched proposals receive gt index + 1 (`assigned_gt_inds`)
 *   workspace : >= sum of ptb_hungarian_v2_workspace(N_b, n_b) bytes
 *   status    : DEVICE int32 [num_images], PRE-ZEROED; 0 ok, 1 = scipy's "cost matrix is infeasible",
 *               2 = scipy's "matrix contains invalid numeric entries" (NaN / -inf), 3 = internal error
 *   topk_k    : 1 = one solve (any orientation); > 1 = rounds on the still-unassigned proposals while they are >= n_b
 */
uint64_t ptb_hungarian_v2_workspace(int N, int n);
int ptb_hungarian_v2_batch(const float* cost, const int64_t* desc, int num_images, int max_N, int max_n, int topk_k,
                           const int32_t* row_idx, int64_t* gt_inds, void* workspace, int32_t* status, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * PointAssigner — replaces PointAssigner.assign (mmdet/core/bbox/assigners/point_assigner.py:23-133).
 * points [N][3] (x,y,stride), gts [n][4];  out_gt_inds[N] (0 = background, j+1 = gt j), int64 like the reference.
 */
int ptb_point_assigner(const float* points, int N, const float* gt_bboxes, int n, float scale, int pos_num,
                       int64_t* out_gt_inds, void* workspace, uint64_t workspace_bytes, void* stream);
uint64_t ptb_point_assigner_workspace(int N, int n);

/* elementwise P2P losses — replace FocalLoss (mmdet/models/losses/focal_loss.py:11-56 formula) and SmoothL1Loss
 * (smooth_l1_loss.py:25-31) as used by P2PHead.loss_single (p2p_head.py:220-248). sums are atomically added. */
int ptb_sigmoid_focal_fwd_bwd(const float* logits /*[M][C]*/, const int64_t* labels /*[M], ==C: background*/,
                              const float* weight /*[M]*/, int64_t M, int num_classes, float gamma, float alpha,
                              float* loss_sum /*[1]*/, const float* scale /*[1] or NULL*/, float* grad /*[M][C] or NULL*/,
                              void* stream);
int ptb_smooth_l1_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2]*/, int64_t M,
                          float inv_norm /* 1/(stride*reg_norm) */, float beta,
                          float* loss_sum, const float* scale, float* grad /*[M][2] or NULL*/, void* stream);
/* the reference P2PHead's default losses (p2p_head.py:37-45), same conventions as the pair above (loss_sum += the weighted,
 * un-normalised sum, deterministic; with grad != NULL the gradient scale * d sum / d input is written instead):
 *   ptb_sigmoid_bce_fwd_bwd  CrossEntropyLoss(use_sigmoid=True, class_weight=None) (cross_entropy_loss.py:42-89):
 *                            sum_m,c [(1 - t) x - log_sigmoid(x)] * weight[m], t = one-hot(labels[m]) (label outside [0, C): 0)
 *   ptb_mse_fwd_bwd          MSELoss (mse_loss.py:9-48): sum ((pred - target) * inv_norm)^2 * weight */
int ptb_sigmoid_bce_fwd_bwd(const float* logits /*[M][C]*/, const int64_t* labels /*[M], ==C: background*/,
                            const float* weight /*[M] or NULL*/, int64_t M, int num_classes, float* loss_sum /*[1]*/,
                            const float* scale /*[1] or NULL*/, float* grad /*[M][C] or NULL*/, void* stream);
int ptb_mse_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2] or NULL*/, int64_t M,
                    float inv_norm /* 1/(stride*reg_norm) */, float* loss_sum, const float* scale, float* grad /*[M][2] or NULL*/,
                    void* stream);
/* CrossEntropyLoss with its class_weight option and in softmax mode, same conventions:
 *   ptb_sigmoid_bce_cw_fwd_bwd  use_sigmoid=True with class_weight, which mmdet passes as pos_weight of
 *                               binary_cross_entropy_with_logits (cross_entropy_loss.py:85-86), in ATen's CPU order:
 *                               sum_m,c [(1 - t) x - log_sigmoid(x) ((pw_c - 1) t + 1)] * weight[m];
 *                               grad (pw_c t + 1 - t) sigmoid(x) - pw_c t.  pos_weight NULL: the bits of ptb_sigmoid_bce_fwd_bwd
 *   ptb_softmax_ce_fwd_bwd      use_sigmoid=False (cross_entropy_loss.py:9-39): over rows of num_cols = C + 1 logits,
 *                               sum_m weight[m] cw[y_m] (logsumexp(x_m) - x_m[y_m]); grad weight[m] cw[y_m] (softmax(x_m) - onehot(y_m)).
 *                               Labels lie in [0, num_cols) (background = num_cols - 1); a row with a label outside it gets a NaN
 *                               loss and gradient.  num_cols >= 2. */
int ptb_sigmoid_bce_cw_fwd_bwd(const float* logits /*[M][C]*/, const int64_t* labels /*[M], ==C: background*/,
                               const float* weight /*[M] or NULL*/, const float* pos_weight /*[C] or NULL*/, int64_t M,
                               int num_classes, float* loss_sum /*[1]*/, const float* scale /*[1] or NULL*/,
                               float* grad /*[M][C] or NULL*/, void* stream);
int ptb_softmax_ce_fwd_bwd(const float* logits /*[M][num_cols]*/, const int64_t* labels /*[M]*/, const float* weight /*[M] or NULL*/,
                           const float* class_weight /*[num_cols] or NULL*/, int64_t M, int num_cols, float* loss_sum /*[1]*/,
                           const float* scale /*[1] or NULL*/, float* grad /*[M][num_cols] or NULL*/, void* stream);
/* ptb_smooth_l1_fwd_bwd / ptb_mse_fwd_bwd with one normalisation per proposal row, row_inv_norm[m] = 1 / (stride_m * reg_norm):
 * the multi-level P2P head, where each row is divided by its own level's stride (p2p_head.py:234-240). */
int ptb_smooth_l1_rows_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2]*/, int64_t M,
                               const float* row_inv_norm /*[M]*/, float beta, float* loss_sum, const float* scale, float* grad,
                               void* stream);
int ptb_mse_rows_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2] or NULL*/, int64_t M,
                         const float* row_inv_norm /*[M]*/, float* loss_sum, const float* scale, float* grad, void* stream);
/* P2PHead's other point losses on the normalised points d = (pred - target) * row_inv_norm[m], same conventions:
 *   ptb_l1_rows_fwd_bwd           L1Loss (smooth_l1_loss.py:33-45): sum |d| * weight; the gradient of |d| is sgn(d), 0 at d == 0
 *                                 and at a NaN d, as torch's
 *   ptb_balanced_l1_rows_fwd_bwd  BalancedL1Loss (balanced_l1_loss.py:12-49) with its alpha, gamma, beta; alpha > 0, beta > 0 and
 *                                 gamma != 0 (b = e^(gamma / alpha) - 1 divides the loss), else it returns an error */
int ptb_l1_rows_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2] or NULL*/, int64_t M,
                        const float* row_inv_norm /*[M]*/, float* loss_sum, const float* scale, float* grad, void* stream);
int ptb_balanced_l1_rows_fwd_bwd(const float* pred /*[M][2]*/, const float* target, const float* weight /*[M][2] or NULL*/, int64_t M,
                                 const float* row_inv_norm /*[M]*/, float alpha, float gamma, float beta, float* loss_sum,
                                 const float* scale, float* grad, void* stream);
/* GHM-C and GHM-R (ghm_loss.py:21-172) as P2PHead calls them, one image at a time, in two steps, all on the device:
 *   ptb_ghm{c,r}_bin_weights  over a batch of B images: counts[b][i] (i < bins) = valid elements of image b whose gradient length g
 *                             lies in [edges[i], edges[i+1]) (edges nondecreasing), counts[b][bins] = valid elements; then, image by
 *                             image in order, tot[b] = max(counts[b][bins], 1) and the per-bin element weights bin_weight[b][i] =
 *                             (tot / cnt_i) / n, or with momentum > 0 (tot / acc_sum[i]) / n after the in-place update
 *                             acc_sum[i] = momentum * acc_sum[i] + (1 - momentum) * cnt_i of every non-empty bin; n = non-empty bins.
 *                             GHMC: g = |sigmoid(x) - t| over B x Q x C logits, t = one-hot(labels) (label outside [0, C): zero row),
 *                             valid = label_weight[b][q] > 0.  GHMR: g = |d / sqrt(d^2 + mu^2)|, valid = weight > 0.
 *                             tot counts the valid elements.  For GHMR the reference sums the weights instead: the two agree for
 *                             P2PHead's 0/1 point weights, not for fractional ones.  Above 2^24 valid elements tot is the count
 *                             rounded to fp32, which can differ by one ulp from the reference's fp32 sum.
 *   ptb_ghm{c,r}_fwd_bwd      one image: loss_sum += sum of the element losses times their bin's weight (GHMC: binary cross-entropy
 *                             with logits, GHMR: sqrt(d^2 + mu^2) - mu); with grad != NULL the gradient scale * d sum / d input instead.
 * At most PTB_GHM_MAX_BINS bins. */
#define PTB_GHM_MAX_BINS 256
int ptb_ghmc_bin_weights(const float* logits /*[B][Q][C]*/, const int64_t* labels /*[B][Q], ==C: background*/,
                         const float* label_weight /*[B][Q]*/, int B, int64_t Q, int num_classes, const float* edges /*[bins+1]*/,
                         int bins, double momentum, float* acc_sum /*[bins], NULL without momentum*/, int32_t* counts /*[B][bins+1]*/,
                         float* bin_weight /*[B][bins]*/, float* tot /*[B]*/, void* stream);
int ptb_ghmc_fwd_bwd(const float* logits /*[Q][C]*/, const int64_t* labels /*[Q]*/, const float* label_weight /*[Q]*/, int64_t Q,
                     int num_classes, const float* edges /*[bins+1]*/, int bins, const float* bin_weight /*[bins]*/, float* loss_sum,
                     const float* scale, float* grad /*[Q][C] or NULL*/, void* stream);
int ptb_ghmr_bin_weights(const float* pred /*[B][Q][2]*/, const float* target, const float* weight /*[B][Q][2]*/,
                         const float* row_inv_norm /*[Q]*/, float mu, int B, int64_t Q, const float* edges /*[bins+1]*/, int bins,
                         double momentum, float* acc_sum /*[bins] or NULL*/, int32_t* counts /*[B][bins+1]*/,
                         float* bin_weight /*[B][bins]*/, float* tot /*[B]*/, void* stream);
int ptb_ghmr_fwd_bwd(const float* pred /*[Q][2]*/, const float* target, const float* weight /*[Q][2]*/, int64_t Q,
                     const float* row_inv_norm /*[Q]*/, float mu, const float* edges /*[bins+1]*/, int bins,
                     const float* bin_weight /*[bins]*/, float* loss_sum, const float* scale, float* grad /*[Q][2] or NULL*/,
                     void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Conv towers on the tensor cores — replace the cuDNN calls behind CPRHead.forward_single / P2PHead.forward_single
 * (cpr_head.py:983-995,1033-1043; p2p_head.py:82-97,113-123): ConvModule = conv3x3(256 out, no bias) + GroupNorm + ReLU.
 * fp32-accurate 3xTF32 implicit GEMM (wgmma.mma_async tf32, TMA-staged operands, fp32 accumulators in registers).
 *   ptb_split_tf32           x -> hi (13 low mantissa bits cleared) + lo (= x - hi, exact)
 *   ptb_conv3x3_pack_weight  nn.Conv2d weight [Cout][Cin][3][3] -> [Cout][tap][Cin] as hi / lo
 *   ptb_conv3x3_c256_tf32x3  y[b][h][w][0..256) = sum_{tap,ci} x[b][h+kh-1][w+kw-1][ci] * w[co][tap][ci]  (zero padding);
 *                            gn_stats (optional, zero-initialised by the caller) [B][32][2] fp64 += per-(image, group of 8
 *                            channels) sum / sum of squares of y
 *   ptb_gn_relu_apply        out = relu((y-mean)*rstd*gamma+beta) from those statistics, written as fp32 (out_lo == NULL)
 *                            or directly as the hi/lo pair the next conv consumes
 */
int ptb_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream);
int ptb_conv3x3_pack_weight(const float* w_oihw, int Cout, int Cin, float* w_hi, float* w_lo, void* stream);
int ptb_conv3x3_c256_tf32x3(const float* x_hi, const float* x_lo /*[B][H][W][Cin]*/, const float* w_hi, const float* w_lo,
                            int B, int H, int W, int Cin, float* y /*[B][H][W][256]*/, double* gn_stats, void* stream);
int ptb_gn_relu_apply(const float* y, const double* gn_stats, const float* gamma, const float* beta, int B, int HW, int C,
                      int groups, float eps, int relu, float* out_hi, float* out_lo, void* stream);
/* Same tower at HALF the tensor-pipe time: two-term fp16 split  x*scale = h + l  (22 significant bits), three
 * wgmma.mma_async f16 products per k-step (h*h + l*h + h*l), fp32 accumulate.  Operands are IEEE fp16 arrays (void* = __half*).
 *   ptb_split_f16: auto_scale != 0 picks a power-of-two scale from max|x| ON THE DEVICE (workspace: 4 bytes) and writes
 *                  its inverse to dev_inv_scale (a device float), else scale = 1.
 *   ptb_conv3x3_pack_weight_f16: weights * scale (a power of two chosen by the caller) as h / l.
 *   ptb_conv3x3_c256_f16x2: y = conv * out_scale * (*dev_out_scale if given): undoes the operand scales exactly.
 *   ptb_gn_relu_apply_f16: GroupNorm(+ReLU) written as the (h, l) pair of the next conv (scale 1); |out| > 60000 is clamped
 *                  and *overflow_flag set (cannot happen for a GroupNorm output with sane affine parameters).
 */
int ptb_split_f16(const float* x, int64_t n, int auto_scale, void* hi, void* lo, float* dev_inv_scale, void* workspace, void* stream);
int ptb_conv3x3_pack_weight_f16(const float* w_oihw, int Cout, int Cin, float scale, void* w_h, void* w_l, void* stream);
int ptb_conv3x3_c256_f16x2(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                           float out_scale, const float* dev_out_scale, float* y, double* gn_stats, void* stream);
/* General form of the same kernel for the head's other GEMMs: taps = 1 (the per-cell Linear cls_out / ins_out of CPRHead,
 * cpr_head.py:1008-1014) or 9 (P2PHead's cls_out / reg_out conv3x3 WITH bias, p2p_head.py:98-102), n_out <= 512 output
 * channels (P2PHead at its default 4 anchors x 80 classes has 320), MMA N = n_mma (multiple of 16 in [n_out, 512]; the
 * packed weight has zero rows beyond n_out), bias added in the epilogue, output row stride ldy (a multiple of 4, >= n_out).
 * One launch at every width: outputs wider than 128 channels run as ceil(n_mma / 128) channel slices of 128 over the same
 * persistent grid, so n_out <= 256 keeps its slicing (and its bits).  GroupNorm statistics stay with the 256-channel
 * ptb_conv3x3_c256_* entry points. */
int ptb_conv_tc_pack_weight_f16(const float* w /*[n_out][Cin][taps]*/, int n_out, int n_mma, int Cin, int taps, float scale,
                                void* w_h, void* w_l, void* stream);
int ptb_conv_tc_f16x2(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin, int taps,
                      int n_out, int n_mma, float out_scale, const float* dev_out_scale, const float* bias, float* y, int ldy,
                      void* stream);
int ptb_gn_relu_apply_f16(const float* y, const double* gn_stats, const float* gamma, const float* beta, int B, int HW, int C,
                          int groups, float eps, int relu, void* out_h, void* out_l, int* overflow_flag, void* stream);
/* Half-precision feature maps (the fp16 / bf16 FPN output of a backbone under autocast) are operand pairs without an fp32 copy:
 *   fp16  the tensor is its own h with l == 0 and scale 1.  ptb_conv_tc_f16x1a is ptb_conv_tc_f16x2 without x_l: the l * w_h product
 *         and the l activation loads are dropped (8 MMAs per K-block instead of 12, half the activation bytes); the result has the
 *         bits of ptb_conv_tc_f16x2 given the same x_h and an all-zero x_l.  gn_stats (optional, zero-initialised, [B][32][2] fp64)
 *         as in ptb_conv3x3_c256_f16x2: needs n_out == n_mma == 256.
 *   bf16  ptb_split_f16_from_bf16: x (void* = __nv_bfloat16*, n % 8 == 0, 16-byte aligned) -> (h, l, *dev_inv_scale), bit for bit
 *         what ptb_split_f16(auto_scale = 1) gives on the tensor converted to fp32, reading 2 bytes per element (workspace: 4 bytes).
 *   ptb_conv_tc_f16x2_half_out: ptb_conv_tc_f16x2 storing y as fp16 / bf16 (y_dtype = PTB_DTYPE_*, ldy in elements), each value the
 *         fp32 result rounded to nearest even (overflow to +-inf), i.e. the cast of the fp32 output without a second pass: the input
 *         gradient (dgrad) of a half-precision feature map.  n_mma > 64 (128-channel slices). */
#define PTB_DTYPE_F16 1
#define PTB_DTYPE_BF16 2
int ptb_split_f16_from_bf16(const void* x, int64_t n, void* hi, void* lo, float* dev_inv_scale, void* workspace, void* stream);
int ptb_conv_tc_f16x1a(const void* x_h, const void* w_h, const void* w_l, int B, int H, int W, int Cin, int taps, int n_out, int n_mma,
                       float out_scale, const float* dev_out_scale, const float* bias, float* y, int ldy, double* gn_stats /*or NULL*/,
                       void* stream);
int ptb_conv_tc_f16x2_half_out(const void* x_h, const void* x_l, const void* w_h, const void* w_l, int B, int H, int W, int Cin, int taps,
                               int n_out, int n_mma, float out_scale, const float* dev_out_scale, const float* bias, void* y, int y_dtype,
                               int ldy, void* stream);
/* One tower layer in one launch: ptb_conv3x3_c256_f16x2 (x_l == NULL: the lo == 0 variant of ptb_conv_tc_f16x1a) followed by
 * GroupNorm(32 groups) + ReLU, the apply running inside the conv kernel as each image's statistics complete.
 *   workspace  zero-filled by the caller, 8-byte aligned: B * 32 * 2 doubles (the statistics [B][32][2], as gn_stats of
 *              ptb_conv3x3_c256_f16x2) followed by B int32 completion counters.
 *   out_l != NULL: out / out_l = the fp16 (h, l) pair ptb_gn_relu_apply_f16 writes (|value| > 60000 clamped, *overflow_flag raised
 *              when given);  out_l == NULL: out = fp32 relu(GroupNorm(y)) as ptb_gn_relu_apply writes it (out_lo == NULL).
 * y (fp32 [B][H][W][256]) and the statistics are written as by ptb_conv3x3_c256_f16x2.  Outputs have the bits of the two kernels
 * run one after the other on this y and these statistics.  The launch is cooperative (the CTAs wait on each other's images); when
 * the grid cannot be co-resident it runs as those two kernels. */
int ptb_conv3x3_c256_f16_gn(const void* x_h, const void* x_l /*or NULL*/, const void* w_h, const void* w_l, int B, int H, int W, int Cin,
                            float out_scale, const float* dev_out_scale, float* y, void* workspace, const float* gamma, const float* beta,
                            float eps, void* out, void* out_l /*or NULL*/, int* overflow_flag /*or NULL*/, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Dense-anchor assignment (SURVEY.md §8f rank 4, BASELINE.json configs[3]): MaxIoUAssigner.assign
 * (mmdet/core/bbox/assigners/max_iou_assigner.py:60-212) over BboxOverlaps2D (iou_calculators/iou2d_calculator.py:211-256)
 * without materialising the (k, n) IoU matrix.  Boxes are [.][4] fp32 (x1,y1,x2,y2), 16-byte aligned.
 *   out_gt_inds[i]      int64: -1 ignored / between thresholds, 0 negative, g+1 assigned to GT g          (bit-exact target)
 *   out_max_overlaps[i] max IoU of anchor i over the GTs (-1 for anchors hit by gt_bboxes_ignore)
 *   out_labels[i]       int64 gt_labels[g] for positives, -1 otherwise (NULL to skip)
 * neg_iou_lo/hi: a float neg_iou_thr t is (0, t); a tuple (a, b) is (a, b).  ignore_iof_thr <= 0 or no ignore boxes: no ignoring;
 * ignore_wrt_candidates selects which box's area normalises the IoF (max_iou_assigner.py:109-116).
 * ptb_bbox_overlaps writes the matrix itself (mode_iof: 0 IoU, 1 IoF w.r.t. boxes1). */
uint64_t ptb_max_iou_assign_workspace(int N, int n_gt);
int ptb_max_iou_assign(const float* bboxes, int N, const float* gt_bboxes, int n_gt, const int32_t* gt_labels /*or NULL*/,
                       const float* gt_bboxes_ignore /*or NULL*/, int n_ignore, float pos_iou_thr, float neg_iou_lo, float neg_iou_hi,
                       float min_pos_iou, int gt_max_assign_all, int match_low_quality, float ignore_iof_thr, int ignore_wrt_candidates,
                       int64_t* out_gt_inds, float* out_max_overlaps, int64_t* out_labels, void* workspace, uint64_t workspace_bytes,
                       void* stream);
int ptb_bbox_overlaps(const float* boxes1, int m, const float* boxes2, int n, int mode_iof, float* out /*[m][n]*/, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Tower backward (autograd of CPRHead.forward_single / P2PHead.forward_single, cpr_head.py:1033-1043, p2p_head.py:113-123;
 * the reference gets it from ATen/cuDNN autograd).  Per ConvModule, in reverse order:
 *   ptb_gn_relu_bwd          da (grad of the ReLU output) + saved conv output y + epilogue statistics -> dy (fp32), dgamma, dbeta,
 *                            max|dy| as float bits (device) for the operand scale.  Deterministic (no fp atomics).
 *   ptb_split_f16_amax       dy -> fp16 (h, l) pair with the power-of-two scale derived from that device max; 1/scale -> dev_inv_scale
 *   ptb_conv_tc_f16x2        dgrad: the forward kernel on (dy pair, weights transposed + flipped and packed by the host layer)
 *   ptb_conv_tc_wgrad_f16x2_ld  taps 9, ld_dy = Cout: dW[co][ci][3][3] (+)= scale * s_dy * s_x * sum_pixels dy (x) x_shifted
 *                            on wgmma with MN-major operands
 * All tensors channels-last; C = 256 for the tensor-core kernels.
 */
uint64_t ptb_gn_relu_bwd_workspace(int B, int HW, int C, int groups);
int ptb_gn_relu_bwd(const float* da, const float* y, const double* gn_stats, const float* gamma, const float* beta, int B, int HW, int C,
                    int groups, float eps, int relu, void* workspace, float* dy, float* dgamma /*[C] or NULL*/,
                    float* dbeta /*[C] or NULL*/, unsigned int* amax_bits /*device, or NULL*/, void* stream);
int ptb_split_f16_amax(const float* x, int64_t n, const unsigned int* dev_amax_bits, void* hi, void* lo, float* dev_inv_scale,
                       void* stream);

/* The weight gradient of any channels-last GEMM with K = pixels:
 *   dW[co][ci][tap] (+)= scale * s_dy * s_x * sum_pixels dy[p][co] * x[p + tap][ci]
 * with taps = 9 (conv3x3, pad 1: the towers) or taps = 1 (conv1x1 / per-cell Linear: the weight gradient of CPRHead's cls_out / ins_out
 * logit map, cpr_head.py:1045-1078 under autograd), Cin = 256, Cout a multiple of 8 up to 256 (rows beyond Cout are never written).
 * dy (fp16 pair [B][H][W][.], 16-byte aligned) has rows ld_dy fp16 apart (ld_dy >= Cout, a multiple of 8): ld_dy = Cout for a dense
 * map, or one column slice [c0, c0 + Cout) of a wider pair (dy + c0), e.g. the logit map's gradient of more than 256 columns, without
 * a copy.  x is [B][H][W][256] fp16.  dw is [Cout][256][taps] fp32; dev_scale_dy / dev_scale_x may be NULL.  Deterministic
 * (fixed-order reduction of the pixel splits). */
uint64_t ptb_conv_tc_wgrad_workspace(int B, int H, int W, int taps);
int ptb_conv_tc_wgrad_f16x2_ld(const void* dy_h, const void* dy_l, int ld_dy, const void* x_h, const void* x_l, int B, int H, int W,
                               int Cout, int Cin, int taps, float scale, const float* dev_scale_dy, const float* dev_scale_x,
                               void* workspace, float* dw, int accumulate, void* stream);

/* column sums of a row-major fp32 matrix: out[n] = sum_m y[m][n] (bias gradient of the logit-map Linear); fixed-order, deterministic */
uint64_t ptb_col_sum_workspace(int64_t M, int N);
int ptb_col_sum(const float* y /*[M][ld]*/, int64_t M, int N, int ld, float* workspace, float* out /*[N]*/, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * RPN training (SURVEY.md §8f rank 4, BASELINE.json configs[3]): AnchorHead.get_targets / loss (anchor_head.py:171-267, 269-365,
 * 422-482) with RandomSampler (random_sampler.py:31-80) for B images of L levels, A anchors per cell, N = sum_l H_l W_l A anchors
 * per image in the reference's flat (level, y, x, anchor) order.  featmap_hw [L][2] = (H, W), strides [L][2] = (sx, sy), host arrays.
 *   ptb_rpn_inside_anchors   inside_box [B][L][A] int32 (x0, x1, y0, y1): anchor (l, y, x, a) of image b is inside iff
 *                            x0 <= x < x1 and y0 <= y < y1 (the host restates valid_flags and anchor_inside_flags as these boxes).
 *                            Writes the inside anchors compacted in flat order (inside_anchors [B][N][4], the first n_inside[b] rows
 *                            of each image), inside_idx [B][N] (the anchor's row there, -1 outside) and n_inside [B].
 *   ptb_rpn_candidate_ranks  gt_inds [B][N] (MaxIoUAssigner's result on image b's first n_inside[b] rows): rank [B][N] = the row's
 *                            rank among the image's positives (gt_inds > 0) or negatives (== 0), -1 for ignored rows, and
 *                            counts [B][2] = (positives, negatives).
 *   plan                     int32: [B][2] x (offset, count) for the positives and the negatives of each image, then the sampled ranks
 *                            of each (image, kind) ascending at plan[offset ...]; count -1: every candidate is sampled.
 *   ptb_rpn_anchor_targets   the reference's unmapped targets in the layout of the output maps: labels (int64; 0 foreground, 1
 *                            background) and label_weights like cls_score [B][A][H][W], bbox_targets and bbox_weights like
 *                            bbox_pred [B][4A][H][W], one level after the other.  gt_bboxes: the images' GTs concatenated, image b's
 *                            at rows [gt_off[b], gt_off[b+1]).  A sampled positive gets pos_weight (> 0) or 1 as label weight.
 *   ptb_rpn_sampled_indices  one image (plan of B = 1): pos_inds / neg_inds = the sampled rows, ascending (SamplingResult).
 *   ptb_rpn_level_loss       one level's sums of CrossEntropyLoss(use_sigmoid=True) over M = B*A*H*W logits (loss_sum[0]) and of
 *                            L1Loss / SmoothL1Loss(beta) over the 4M box deltas (loss_sum[1]), weighted, un-normalised, fixed-order;
 *                            or (loss_sum NULL) the gradients scale[0] * d/dcls_score and scale[1] * d/dbbox_pred in the maps' layout. */
#define PTB_RPN_MAX_LEVELS 8
#define PTB_RPN_LOSS_L1 0
#define PTB_RPN_LOSS_SMOOTH_L1 1
int ptb_rpn_inside_anchors(const float* base_anchors /*[L][A][4]*/, const int32_t* featmap_hw, const int32_t* strides, int L, int A, int B,
                           const int32_t* inside_box, float* inside_anchors, int32_t* inside_idx, int32_t* n_inside, void* stream);
int ptb_rpn_candidate_ranks(const int64_t* gt_inds, const int32_t* n_inside, int B, int N, int32_t* rank, int32_t* counts, void* stream);
int ptb_rpn_anchor_targets(const int32_t* featmap_hw, const int32_t* strides, int L, int A, int B, const int32_t* inside_idx,
                           const float* inside_anchors, const int64_t* gt_inds, const int32_t* rank, const int32_t* plan,
                           const float* gt_bboxes, const int32_t* gt_off, const float* means /*[4]*/, const float* stds /*[4]*/,
                           float pos_weight, int64_t* labels, float* label_weights, float* bbox_targets, float* bbox_weights,
                           void* stream);
int ptb_rpn_sampled_indices(const int64_t* gt_inds, const int32_t* rank, int n, const int32_t* plan, int64_t* pos_inds,
                            int64_t* neg_inds, void* stream);
int ptb_rpn_level_loss(const float* cls_score, const float* bbox_pred, const int64_t* labels, const float* label_weights,
                       const float* bbox_targets, const float* bbox_weights, int64_t M, int bbox_loss, float beta, float* loss_sum /*[2]*/,
                       const float* scale /*[2] or NULL*/, float* grad_cls, float* grad_bbox, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * The bbox branch of StandardRoIHead (roi_heads/standard_roi_head.py, bbox_heads/bbox_head.py) with SingleRoIExtractor and mmcv's
 * RoIAlign(aligned=True, pool_mode='avg').  featmap_hw [L][2] and strides [L] (spatial_scale = 1 / stride) are host arrays.
 *   ptb_roi_align_fwd   maps[l]: channels-last [B][H_l][W_l][C] (C a multiple of 4, 16-byte aligned); rois [R][5] (batch index, x1, y1,
 *                       x2, y2).  levels[R] = floor(log2(sqrt(w h) / finest_scale + 1e-6)) clamped to [0, L-1] (-1 for a NaN scale,
 *                       whose features stay 0; L == 1: level 0); y [R][C][out][out] = the RoI's bins on its level, ceil(roi / out)
 *                       samples per bin side when sampling_ratio <= 0.
 *   ptb_roi_align_bwd   grad_maps[l] (channels-last like the maps, zeroed by the caller) += the scatter of grad_y through the forward's
 *                       taps (float atomics); levels from ptb_roi_align_fwd.
 *   ptb_roi_targets     candidates cand [B][N][4] = each image's [GTs; proposals] padded to N, gt_inds [B][N] (MaxIoUAssigner with the
 *                       GTs assigned to themselves, -1 on padding), rank from ptb_rpn_candidate_ranks, the sample plan of
 *                       ptb_rpn_anchor_targets, row_off [B][2] = first output row of image b's positives / negatives.  Writes the
 *                       sampled rows: rois [R][5], labels [R] (gt label or num_classes), label_weights [R] (pos_weight > 0 or 1 for
 *                       positives, 1 for negatives), bbox_targets [R][4] (bbox2delta, then (delta - mean) / std) and bbox_weights [R][4].
 *   ptb_roi_bbox_loss   sum over the positive rows of L1Loss / SmoothL1Loss(beta) * bbox_weights between bbox_pred's class columns
 *                       (4 label .. 4 label + 3 of [R][ld], ld = 4 num_classes; columns 0..3 when class_agnostic, ld = 4) and the
 *                       targets; or (loss_sum NULL) the gradient scale[0] * d/dbbox_pred at those columns (the caller zeroes grad).
 *   ptb_roi_accuracy    out[0] = (number of rows whose first maximum is the label) * scale.
 *   ptb_roi_decode      over B x N padded RoI rows: rows whose four coordinates are 0 take cls_score = 0 and bbox_pred = 0; softmax of
 *                       cls_score [B*N][C+1]; delta2bbox of bbox_pred [B*N][4C] (or [B*N][4]) with dw, dh clamped to +-max_ratio,
 *                       clipped to img_hw [B][2] (h, w, fp32), divided by scale_factor [B][4] when it is given.  boxes [B][N][C][4],
 *                       scores [B][N][C] (the background column dropped). */
#define PTB_ROI_MAX_LEVELS 4
int ptb_roi_align_fwd(const float* const* maps, const int32_t* featmap_hw, const float* strides, int L, int B, int C, const float* rois,
                      int R, int out, int sampling_ratio, float finest_scale, float* y, int32_t* levels, void* stream);
int ptb_roi_align_bwd(float* const* grad_maps, const int32_t* featmap_hw, const float* strides, int L, int B, int C, const float* rois,
                      const int32_t* levels, int R, int out, int sampling_ratio, const float* grad_y, void* stream);
int ptb_roi_targets(int B, int N, const float* cand, const int64_t* gt_inds, const int32_t* rank, const int32_t* plan,
                    const int32_t* row_off, const float* gt_bboxes, const int32_t* gt_off, const int64_t* gt_labels, int num_classes,
                    const float* means /*[4]*/, const float* stds /*[4]*/, float pos_weight, float* rois, int64_t* labels,
                    float* label_weights, float* bbox_targets, float* bbox_weights, void* stream);
int ptb_roi_bbox_loss(const float* bbox_pred, int ld, const int64_t* labels, const float* bbox_targets, const float* bbox_weights, int64_t R,
                      int num_classes, int class_agnostic, int bbox_loss, float beta, float* loss_sum, const float* scale, float* grad,
                      void* stream);
int ptb_roi_accuracy(const float* cls_score, const int64_t* labels, int64_t R, int num_cols, float scale, float* out, void* stream);
int ptb_roi_decode(const float* rois, const float* cls_score, const float* bbox_pred, int B, int N, int num_classes, int class_agnostic,
                   const float* means /*[4]*/, const float* stds /*[4]*/, float max_ratio, const float* img_hw, const float* scale_factor,
                   float* boxes, float* scores, void* stream);

/* ---- test-time augmentation and tile testing of the two-stage detector (csrc/tile_test.cu): StandardRoIHead.aug_test and
 * TwoStageDetector.tile_aug_test.  An aug meta row is 12 floats: segment, RoI batch index, scale_factor[4], flip (0 none, 1 horizontal,
 * 2 vertical, 3 diagonal), img_h, img_w, has_offset, dx, dy.
 *   ptb_box_map        bbox_mapping of rows [0, counts[seg]) of boxes [S][N][ld] for every aug g of meta [G][12]: * scale_factor, flip,
 *                      and with an offset - (dx, dy), clamp to [0, w-1] x [0, h-1] and keep = (W >= 2 & H >= 2).  rois [G][N][5]
 *                      (batch index, box; zero boxes past the count), keep [G][N] (or NULL).  counts NULL: N rows.
 *   ptb_proposal_map_back  merge_aug_proposals' recovery: bbox_mapping_back (flip, / scale_factor, + offset) of the first counts[g]
 *                      rows of det [T*A][N][5] (box, score; aug g = t * A + a), the augs of tile t concatenated in order into
 *                      out [T][A*N][5]; out_count [T].
 *   ptb_aug_merge      merge_aug_bboxes of T tiles of A augs (meta row t * A + a): bbox_mapping_back (flip, / scale_factor, + offset)
 *                      of boxes [T*A][N][C][4] and torch.stack(...).mean(0) of them and of scores [T*A][N][C], in ATen's CPU order for
 *                      a stack of (counts[t], box_cols) boxes and (counts[t], C + 1) scores.  box_cols: 4 (class-agnostic) or 4C.
 *                      out_boxes [T][N][C][4], out_scores [T][N][C] (-inf past the count).  A <= 63.
 *   ptb_batched_nms    mmcv batched_nms (labels given) or nms (labels NULL) of each of S segments of N <= 65536 rows: the first
 *                      counts[s] rows (NULL: N) of boxes [S][N][ld], scores [S][N][lds], labels [S][N].  Greedy IoU > iou_thr in the
 *                      order score descending, position ascending on boxes offset by label * (max + 1); from split_thr rows on only
 *                      equal labels suppress.  out_count [S], out_det [S][N][5] (box, score), out_label [S][N] (or NULL), out_keep
 *                      [S][N] row positions, at most max_num rows when max_num > 0.  workspace: ptb_batched_nms_workspace(S, N).
 *   ptb_tile_concat    the first counts[t] rows of det [T][K][5] / labels [T][K] of each tile, boxes * scale_factor [T][4] (or NULL)
 *                      + offsets [T][2] (dx, dy), concatenated in tile order, class-major within a tile (the rows of one class in
 *                      their order): out [T*K][5], out_label [T*K], out_count[0] = the number of rows. */
#define PTB_BATCHED_NMS_MAX_ROWS 65536
int ptb_box_map(const float* boxes, int ld, const int32_t* counts, int N, int G, const float* meta, float* rois, uint8_t* keep,
                void* stream);
int ptb_proposal_map_back(const float* det, const int32_t* counts, int N, int T, int A, const float* meta, float* out, int32_t* out_count,
                          void* stream);
int ptb_aug_merge(const float* boxes, const float* scores, int N, int num_classes, int box_cols, const int32_t* counts, int T, int A,
                  const float* meta, float* out_boxes, float* out_scores, void* stream);
uint64_t ptb_batched_nms_workspace(int S, int N);
int ptb_batched_nms(const float* boxes, int ld, const float* scores, int lds, const int32_t* labels, const int32_t* counts, int S, int N,
                    float iou_thr, int split_thr, int max_num, int32_t* out_count, float* out_det, int32_t* out_label, int32_t* out_keep,
                    void* workspace, uint64_t workspace_bytes, void* stream);
int ptb_tile_concat(const float* det, const int32_t* labels, const int32_t* counts, int T, int K, const float* scale_factor,
                    const float* offsets, float* out, int32_t* out_label, int32_t* out_count, void* stream);

/* FCOS head (fcos_head.py).  Rows of a batch: level after level, image after image inside a level, then y, x (the order of the
 * reference's flattened maps); the point of a row is x * stride + stride // 2 of its level (L <= 8 levels of hw [L][2], strides [L]).
 *   ptb_fcos_targets   _get_target_single of every (image, point): GTs gt_bboxes [G][4] / gt_labels [G] of image b at rows
 *                      gt_off[b] .. gt_off[b+1]; regress ranges [L][2]; radius_px [L] = fp32(stride * center_sample_radius) or NULL
 *                      (no centre sampling); the minimum-area GT wins, ties to the first; label num_classes where every area is
 *                      excluded.  out_labels [N] int64, out_targets [N][4] (l, t, r, b; / stride when norm_on_bbox).
 *   ptb_fcos_norm_sums out[0] += the number of positive rows, out[1] += the sum of their centerness targets (fixed order).
 *   ptb_fcos_bbox_loss the centerness-weighted IoU (mode 0: -log, 1: linear; bbox_overlaps eps overlap_eps, clamp eps) or GIoU (mode 2,
 *                      eps) loss of distance2bbox(point, pred [N][4]) against distance2bbox(point, targets): loss_sum [1] += the sum,
 *                      or grad [N][4] = scale[0] * d/dpred (zero rows for negatives).
 *   ptb_fcos_centerness_loss  binary_cross_entropy_with_logits(logits [N], centerness target) of the positive rows, same convention.
 *   ptb_fcos_decode    per level and image: rows of the top nms_pre keys max_c sigmoid(cls) * sigmoid(ctr) when 0 < nms_pre < H*W
 *                      (else every row in order), maps channels-last cls [B][H][W][C], reg [B][H][W][4], ctr [B][H][W]; out_idx
 *                      [B][R] cell of each row, out_boxes [B][R][4] clipped to img_hw [B][2] (float) and / scale_factor [B][4] (or
 *                      NULL), out_scores [B][R][C] sigmoid, out_ctr [B][R] sigmoid.  workspace: ptb_fcos_decode_workspace(B, L, hw). */
int ptb_fcos_targets(const float* gt_bboxes, const int64_t* gt_labels, const int32_t* gt_off, int B, int L, const int32_t* hw,
                     const float* strides, const float* ranges, const float* radius_px, int norm_on_bbox, int num_classes,
                     int64_t* out_labels, float* out_targets, void* stream);
int ptb_fcos_norm_sums(const int64_t* labels, const float* targets, int64_t N, int num_classes, float* out, void* stream);
int ptb_fcos_bbox_loss(const float* pred, const float* targets, const int64_t* labels, int B, int L, const int32_t* hw, const float* strides,
                       int num_classes, int mode, float overlap_eps, float eps, float* loss_sum, const float* scale, float* grad,
                       void* stream);
int ptb_fcos_centerness_loss(const float* logits, const float* targets, const int64_t* labels, int64_t N, int num_classes, float* loss_sum,
                             const float* scale, float* grad, void* stream);
uint64_t ptb_fcos_decode_workspace(int B, int L, const int32_t* hw);
int ptb_fcos_decode(const float* const* cls_maps, const float* const* reg_maps, const float* const* ctr_maps, int L, const int32_t* hw,
                    const float* strides, int B, int num_classes, const float* img_hw, const float* scale_factor, int nms_pre,
                    int32_t* out_idx, float* out_boxes, float* out_scores, float* out_ctr, void* workspace, uint64_t workspace_bytes,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PTB_B200_H_ */
