"""CPRHead — host-side mirror of the reference's Coarse-Point-Refine head over the sm_90a kernels.

Interface (same names / argument meaning / output structure as the reference, SURVEY.md §8b):
  reference: TOV_mmdetection/mmdet/models/point/dense_heads/cpr_head.py:898-1309 (CPRHead), registered in HEADS.
  forward(feats) -> (list[cls_feat], list[ins_feat]);  loss(...) -> dict(gt_loss, pos_loss, bag_acc, neg_loss);
  get_bboxes(...) -> [(det (n,6) [x1,y1,x2,y2,score,ann_id], labels (n,))];  forward_train / simple_test as mmdet.
  state_dict keys: cls_convs.{i}.conv.weight, cls_convs.{i}.gn.{weight,bias}, cls_out.*, ins_out.*.

Data flow (GPU-first, see DESIGN.md): the per-point Linear(256->C) of the reference commutes with bilinear sampling,
so the head computes ONE class/instance logit map (a 1-tap wgmma convolution, `ptb_conv_tc_f16x2`; `ptb_linear_rows` is the
fp32 FFMA alternative) and samples that (C channels instead of 256); the (G,K,256) gathered-feature tensor of the reference is
never built, and at inference not even the (G,K,C) probability tensor is (ptb_cpr_refine_fused).  All images of the batch go
through each kernel in one launch.  Positive bags: ring bags (CirclePtFeatGenerator) or grid-cell bags (GridCirclesPtFeatGenerator);
`other_info.out_geo` appends the chosen bag points to the output rows.
"""
import os
import warnings

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .layers import ConvModule, PackedWeightsMixin, bias_init_with_prob, normal_init_, tower, tc_enabled, _packed_tc
from .registry import register_head

_SUPPORTED_POS = ('CirclePtFeatGenerator', 'GridCirclesPtFeatGenerator')
_SUPPORTED_NEG = ('OutCirclePtFeatGenerator', 'OutGridCirclesPtFeatGenerator')


def _merge(default, given):
    out = dict(default)
    out.update(given or {})
    return out


_GT_INDEX_CACHE = {}       # (lens, pad shapes, img shapes, device) -> packed int32 device tensor; bounded, see _BatchGT


class _BatchGT:
    """CSR view of the per-image GT lists (device tensors + host lengths).  The index arrays (bag -> image, image offsets, pad / image
    shapes) depend only on the per-image GT counts and the image metas: they are built and uploaded ONCE per distinct key and cached,
    so a steady-state step does no numpy work and no pageable host->device copy (an implicit sync on the hot path in round 1)."""

    def __init__(self, gt_bboxes, gt_labels, img_metas, device):
        self.lens = [int(l.shape[0]) for l in gt_labels]
        n_ref = [int(b.shape[0]) // max(n, 1) for b, n in zip(gt_bboxes, self.lens)]
        if any(r != 1 for r, n in zip(n_ref, self.lens) if n > 0):
            raise NotImplementedError('num_refine > 1 (CPR++ cascade, unreleased in the reference) is not supported')
        boxes = torch.cat([b.reshape(-1, 4) for b in gt_bboxes]).to(device=device, dtype=torch.float32)
        self.centers = ((boxes[:, :2] + boxes[:, 2:]) / 2).contiguous()          # cpr_head.py:1293-1301
        self.labels64 = torch.cat(list(gt_labels)).to(device)
        self.labels = self.labels64.int().contiguous()
        B = len(self.lens)
        self.G = int(sum(self.lens))
        pad_t = tuple(tuple(int(v) for v in m['pad_shape'][:2]) for m in img_metas)
        img_t = tuple(tuple(int(v) for v in m['img_shape'][:2]) for m in img_metas)
        key = (tuple(self.lens), pad_t, img_t, str(device))
        packed = _GT_INDEX_CACHE.get(key)
        if packed is None:
            bag_img = np.repeat(np.arange(B, dtype=np.int32), self.lens)
            img_ptr = np.concatenate([[0], np.cumsum(self.lens)]).astype(np.int32)
            host = torch.from_numpy(np.concatenate([bag_img, img_ptr, np.array(pad_t, dtype=np.int32).reshape(-1),
                                                    np.array(img_t, dtype=np.int32).reshape(-1)]))
            packed = host.to(device)
            if len(_GT_INDEX_CACHE) >= 256:          # ragged training batches: bounded, oldest entry out
                _GT_INDEX_CACHE.pop(next(iter(_GT_INDEX_CACHE)))
            _GT_INDEX_CACHE[key] = packed
        o = 0
        self.bag_img = packed[o:o + self.G]; o += self.G
        self.img_ptr = packed[o:o + B + 1]; o += B + 1
        self.pad_hw = packed[o:o + 2 * B].view(B, 2); o += 2 * B
        self.img_hw = packed[o:o + 2 * B].view(B, 2)


class _CircleBags:
    """CirclePtFeatGenerator (cpr_head.py:447-497): ring offsets + centre, bilinear samples (ptb_cpr_bag_gather).
    `reach` = max |offset| in pixels, taken from the host copy of the table when it is built; it sizes the sample windows of the
    gather, the fused refine and the deterministic loss backward (a reach that is too small loses samples)."""

    def __init__(self, offsets, stride, reach=None):
        self.offsets, self.stride = offsets, stride
        self.reach = ops.offsets_reach(offsets) if reach is None else float(reach)

    def gather(self, lmap, gt, pts=False):
        f, p, valid = ops.bag_gather(lmap, gt.centers, gt.bag_img, self.offsets, self.stride, gt.pad_hw, pts=pts, reach_px=self.reach)
        return f, p, valid, None

    def gather_bwd(self, grad, map_shape, gt, aux):
        return ops.bag_gather_bwd(grad, map_shape, gt.centers, gt.bag_img, self.offsets, self.stride)


class _GridCircleBags:
    """GridCirclesPtFeatGenerator (cpr_head.py:296-350, 413-444): grid cells within radius*stride + centre (ptb_cpr_grid_bag)."""

    def __init__(self, radius, max_pos_num, stride):
        self.radius, self.max_pos_num, self.stride = radius, max_pos_num, stride

    def gather(self, lmap, gt, pts=False):
        return ops.grid_bag(lmap, gt.centers, gt.bag_img, self.stride, self.radius, self.max_pos_num, pts=pts)

    def gather_bwd(self, grad, map_shape, gt, cell):
        return ops.grid_bag_bwd(grad, map_shape, gt.centers, gt.bag_img, cell, self.stride)


def _loss_gemm_on_tc(C, LD):
    """the two GEMMs of the loss that are plain 1x1 convolutions (logit map forward, its input gradient) run on the wgmma kernel
    when the channel counts fit it (Cin % 32 == 0, N <= 256); PTB_LOSS_GEMM=ffma keeps the fp32 FFMA kernels."""
    import os
    return os.environ.get('PTB_LOSS_GEMM', 'tc') == 'tc' and C % 32 == 0 and LD % 32 == 0 and C <= 256 and LD <= 256


class _BagGatherFn(torch.autograd.Function):
    """differentiable bag gather over a channels-last map (ptb_cpr_bag_gather / ptb_cpr_grid_bag and their backward kernels): the
    reference's extract_point_feat + grid_sample (cpr_head.py:73-93, 182-199) for all bags of the batch; used by the generic loss path."""

    @staticmethod
    def forward(ctx, fmap, gt, bags):
        f, _, valid, aux = bags.gather(fmap, gt)
        ctx.gt, ctx.bags, ctx.aux, ctx.shape = gt, bags, aux, tuple(fmap.shape)
        ctx.mark_non_differentiable(valid)
        return f, valid

    @staticmethod
    def backward(ctx, g, _gv):
        return ctx.bags.gather_bwd(g.contiguous(), ctx.shape, ctx.gt, ctx.aux), None, None


LB_MAX_LD = 160        # ptb_cpr_loss_bwd_map: logit rows of at most 160 columns (5 channel groups x 64 cells = 320 threads per tile)
LB_MAX_K = 320         # ... and at most 320 samples per bag


def loss_bwd_plan(N, K, circle_bags, with_mil_loss, env_mode=None, deterministic=False):
    """Column padding and backward path of the fused CPR loss (_CPRLossFn).  A pure function of the configuration.

    env_mode is PTB_LOSS_BWD (None when unset); deterministic is torch.are_deterministic_algorithms_enabled().  Returns
    (NP, path, reason):
      NP      ins column offset of the logit map, LD = 2 * NP.  ceil8(N) by default; ceil16(N) when bit-reproducible gradients are
              asked for, so that LD is a multiple of 32 (the tile kernel's channel groups) for every N.
      path    'tiles'   ptb_cpr_loss_bwd_map: deterministic, ring bags with the MIL loss, LD <= 160 (N <= 80), K <= 320
              'scatter' ptb_cpr_loss_bwd_scatter: fp32 atomics, ring bags with the MIL loss (the default)
              'staged'  mil_loss_bwd + gfocal_bwd + bag_gather_bwd / grid_bag_bwd: fp32 atomics, every configuration
      reason  None, or why bit-reproducible gradients were asked for (PTB_LOSS_BWD=tiles or deterministic mode) but cannot be
              given; `path` is then the atomic path that would run instead.  The caller raises, or warns in warn-only mode."""
    want_tiles = env_mode == 'tiles' or (env_mode is None and deterministic)
    NP = (N + 15) // 16 * 16 if want_tiles else (N + 7) // 8 * 8
    LD = 2 * NP
    circle = circle_bags and with_mil_loss
    fallback = 'scatter' if circle and env_mode in (None, 'scatter', 'tiles') else 'staged'
    if want_tiles:
        if not circle_bags:
            reason = 'grid-cell bags (GridCirclesPtFeatGenerator) have no deterministic loss backward'
        elif not with_mil_loss:
            reason = 'the deterministic loss backward needs with_mil_loss=True'
        elif LD % 32 or LD > LB_MAX_LD:
            reason = f'num_classes={N} gives logit rows of {LD} columns; the deterministic loss backward handles at most {LB_MAX_LD} (num_classes <= 80)'
        elif K > LB_MAX_K:
            reason = f'{K} samples per bag; the deterministic loss backward handles at most {LB_MAX_K}'
        else:
            return NP, 'tiles', None
        return NP, fallback, reason
    if deterministic:
        return NP, fallback, f'PTB_LOSS_BWD={env_mode} selects a backward with fp32 atomics'
    return NP, fallback, None


def _gfocal(p, q, w, eps):
    """MILLoss.gfocal_loss (multi_instance_learning_loss.py:148-151)."""
    return -(((p - q) ** 2) * (q * (p + eps).log() + (1 - q) * (1 - p + eps).log()) * w).sum(dim=-1)


class _CPRLossFn(torch.autograd.Function):
    """fused CPR training loss (CPRHead.loss + loss0, cpr_head.py:1101-1229) on the logit-map data flow."""

    @staticmethod
    def forward(ctx, fmap, w_cls, b_cls, w_ins, b_ins, gt, bags, hp):
        B, H, W, C = fmap.shape
        N = hp['num_classes']
        K = bags.offsets.shape[0] if isinstance(bags, _CircleBags) else 0
        env_mode = os.environ.get('PTB_LOSS_BWD')
        NP, bwd_path, bwd_reason = loss_bwd_plan(N, K, isinstance(bags, _CircleBags), hp['with_mil_loss'], env_mode,
                                                 torch.are_deterministic_algorithms_enabled())
        ctx.bwd = (NP, bwd_path, bwd_reason, env_mode)
        LD = 2 * NP                            # logit row: [cls(0..N) pad | ins(NP..NP+N) pad]
        M = B * H * W
        dev = fmap.device
        wcat = torch.zeros((LD, C), device=dev)
        bcat = torch.zeros((LD,), device=dev)
        wcat[:N], wcat[NP:NP + N], bcat[:N], bcat[NP:NP + N] = w_cls, w_ins, b_cls, b_ins
        x2d = fmap.reshape(M, C)
        use_tc = _loss_gemm_on_tc(C, LD)
        if use_tc:       # logit map on the tensor cores: 1-tap conv of the fp16 operand pair (fp32-accurate two-term split)
            fh, fl, finv = ops.split_f16(fmap, auto_scale=True)
            lmap = ops.conv_tc_f16(fh, fl, ops.conv_tc_pack_weight_f16(wcat, 1), 1, LD, bias=bcat, dev_out_scale=finv, ldy=LD).view(M, LD)
        else:
            lmap = ops.linear_rows(x2d, wcat, bcat)                              # (M, LD) fp32 FFMA GEMM
        fused_fwd = isinstance(bags, _CircleBags) and hp['with_mil_loss'] and N <= 128 and os.environ.get('PTB_LOSS_FWD', 'fused') == 'fused'
        if fused_fwd:   # ring-bag gather + MIL forward in ONE kernel (online softmax): the (G,K,LD) tensor is written once, never re-read
            bl, weight, bag_prob, mil_sum, mil_stats, mil_mt, mil_lw = ops.bag_mil_fwd(
                lmap.view(B, H, W, LD), N, NP, gt.centers, gt.bag_img, bags.offsets, bags.stride, gt.pad_hw, gt.labels, hp['eps'])
            aux = None
        else:
            bl, _, valid, aux = bags.gather(lmap.view(B, H, W, LD), gt)          # (G,K,LD), (G,K)
            weight = valid.float().contiguous()                                  # gt_weights == 1 (cpr_head.py:1114)
        G, K, _ = bl.shape
        one = torch.ones((), device=dev)
        zero = torch.zeros((), device=dev)
        gt_loss = pos_loss = neg_loss = bag_acc = zero
        num_pos = one
        saved = dict(valid_center=None, bag_prob=None, num_pos_gt=one, num_sample=one, neg_mask=None)
        if hp['with_gt_loss']:
            wc = weight[:, K - 1].contiguous()                                   # validity of the centre sample
            s = ops.gfocal_fwd(bl[:, K - 1], G, N, K * LD, gt.labels, wc, hp['eps'])
            num_pos = torch.clamp((wc > 0).sum().float(), min=1.0)               # cpr_head.py:1180
            gt_loss = hp['gt_loss_weight'] * (s[0] / num_pos)
            saved['valid_center'], saved['num_pos_gt'] = wc, num_pos
        if hp['with_mil_loss']:
            if fused_fwd:
                s, stats = mil_sum, mil_stats
            else:
                bag_prob, s, stats, mil_mt, mil_lw = ops.mil_loss_fwd(bl, N, NP, weight, gt.labels, hp['eps'], want_aux=True)
            saved['mil_mt'], saved['mil_lw'] = mil_mt, mil_lw
            num_sample = torch.clamp(stats[0], min=1.0)                          # multi_instance_learning_loss.py:176
            pos_loss = hp['mil_loss_weight'] * (s[0] / num_sample)
            bag_acc = stats[1] * (100.0 / max(G, 1))
            num_pos = num_sample                                                 # cpr_head.py:1216 rebinds num_pos
            saved['bag_prob'], saved['num_sample'] = bag_prob, num_sample
        if hp['with_neg']:
            nm = ops.neg_mask(B, H, W, hp['stride'], gt.pad_hw, gt.centers, gt.labels, gt.img_ptr,
                              hp['stride'] * hp['neg_radius'], N, hp['neg_class_wise'], as_bool=False)
            s = ops.gfocal_fwd(lmap, M, N, LD, None, nm, hp['eps'])
            neg_loss = hp['neg_loss_weight'] * (s[0] / num_pos)
            saved['neg_mask'] = nm
        ctx.hp, ctx.gt, ctx.bags, ctx.aux, ctx.saved = hp, gt, bags, aux, saved
        ctx.num_pos = num_pos
        ctx.fpair = (fh, fl, finv) if use_tc else None        # fp16 operand pair of the feature map: the wgrad's second operand
        ctx.save_for_backward(fmap, wcat, lmap, bl, weight)
        return gt_loss, pos_loss, neg_loss, bag_acc

    @staticmethod
    def _bwd_map_staged(ctx, g_gt, g_pos, g_neg, bl, weight, lmap, B, H, W, N, NP, LD, M, G, K):
        """round-1 chain (kept for grid-cell bags and as PTB_LOSS_BWD=staged): (G,K,LD) gradient tensor -> scatter-add with fp32 atomics."""
        hp, gt, sv = ctx.hp, ctx.gt, ctx.saved
        full = hp['with_mil_loss'] and NP == N       # MIL backward then writes every column of every row
        dbl = torch.empty_like(bl) if full else torch.zeros_like(bl)
        if hp['with_mil_loss']:
            scale = (g_pos * hp['mil_loss_weight'] / sv['num_sample']).reshape(1).float().contiguous()
            ops.mil_loss_bwd(bl, N, NP, weight, gt.labels, hp['eps'], sv['bag_prob'], scale, grad_out=dbl)
        if hp['with_gt_loss']:
            scale = (g_gt * hp['gt_loss_weight'] / sv['num_pos_gt']).reshape(1).float().contiguous()
            ops.gfocal_bwd(bl[:, K - 1], G, N, K * LD, gt.labels, sv['valid_center'], hp['eps'], scale, dbl[:, K - 1],
                           K * LD, accumulate=True)
        dlmap = ctx.bags.gather_bwd(dbl, (B, H, W, LD), gt, ctx.aux)
        if hp['with_neg']:
            scale = (g_neg * hp['neg_loss_weight'] / ctx.num_pos).reshape(1).float().contiguous()
            ops.gfocal_bwd(lmap, M, N, LD, None, sv['neg_mask'], hp['eps'], scale, dlmap, LD, accumulate=True)
        return dlmap

    @staticmethod
    def backward(ctx, g_gt, g_pos, g_neg, _g_acc):
        fmap, wcat, lmap, bl, weight = ctx.saved_tensors
        hp, gt, sv = ctx.hp, ctx.gt, ctx.saved
        B, H, W, C = fmap.shape
        N = hp['num_classes']
        NP, path, reason, env_mode = ctx.bwd
        LD = 2 * NP
        M = B * H * W
        G, K, _ = bl.shape
        if reason is not None:
            # bit-reproducible gradients were asked for and the tile kernel cannot give them: torch's convention for an op without a
            # deterministic implementation (raise; warn instead in warn-only mode, unless PTB_LOSS_BWD=tiles asks for it explicitly)
            msg = f'CPRHead loss backward: no deterministic implementation here ({reason}); the {path} path uses fp32 atomics'
            if env_mode == 'tiles' or not torch.is_deterministic_algorithms_warn_only_enabled():
                raise RuntimeError(msg)
            warnings.warn(msg)
        f1 = lambda t: t.reshape(1).float().contiguous()
        if path == 'tiles':
            # DETERMINISTIC mode (torch.use_deterministic_algorithms(True) or PTB_LOSS_BWD=tiles): MIL + gt + neg gfocal backward and the
            # grid_sample backward in one gather-formulated kernel, one CTA per 8x8 map tile, every sum formed by one thread in a fixed
            # order: bit-identical gradients run to run (2.2 ms at the headline batch)
            dlmap = ops.cpr_loss_bwd_map(
                bl, weight, sv['mil_mt'], sv['bag_prob'], sv['mil_lw'], gt.labels, gt.centers, gt.img_ptr, ctx.bags.offsets, (B, H, W, LD), N, NP,
                ctx.bags.stride, ctx.bags.reach, hp['eps'],
                scale_mil=f1(g_pos * hp['mil_loss_weight'] / sv['num_sample']),
                scale_gt=f1(g_gt * hp['gt_loss_weight'] / sv['num_pos_gt']) if hp['with_gt_loss'] else None,
                valid_center=sv['valid_center'] if hp['with_gt_loss'] else None,
                logit_map=lmap if hp['with_neg'] else None, neg_mask=sv['neg_mask'] if hp['with_neg'] else None,
                scale_neg=f1(g_neg * hp['neg_loss_weight'] / ctx.num_pos) if hp['with_neg'] else None)
        elif path == 'scatter':
            # default: the neg term initialises the map (no memset + read-modify-write), then one kernel per batch computes the MIL + gt
            # gradient of every bag sample from the forward's per-(bag, class) statistics and scatters it with fp32 vector atomics; the
            # (G,K,LD) gradient tensor of round 1 (740 MB written and re-read) and mil_bwd's three passes are gone
            dlmap = torch.empty((B, H, W, LD), dtype=torch.float32, device=bl.device)
            if hp['with_neg'] and NP == N:
                dlmap.view(M, LD)[:, N:].zero_()
                ops.gfocal_bwd(lmap, M, N, LD, None, sv['neg_mask'], hp['eps'], f1(g_neg * hp['neg_loss_weight'] / ctx.num_pos), dlmap, LD,
                               accumulate=False)
            else:
                dlmap.zero_()
                if hp['with_neg']:
                    ops.gfocal_bwd(lmap, M, N, LD, None, sv['neg_mask'], hp['eps'], f1(g_neg * hp['neg_loss_weight'] / ctx.num_pos), dlmap, LD,
                                   accumulate=True)
            ops.cpr_loss_bwd_scatter(bl, weight, sv['mil_mt'], sv['bag_prob'], sv['mil_lw'], gt.labels, gt.centers, gt.bag_img, ctx.bags.offsets,
                                     dlmap, N, NP, ctx.bags.stride, hp['eps'],
                                     scale_mil=f1(g_pos * hp['mil_loss_weight'] / sv['num_sample']),
                                     scale_gt=f1(g_gt * hp['gt_loss_weight'] / sv['num_pos_gt']) if hp['with_gt_loss'] else None,
                                     valid_center=sv['valid_center'] if hp['with_gt_loss'] else None)
        else:
            dlmap = _CPRLossFn._bwd_map_staged(ctx, g_gt, g_pos, g_neg, bl, weight, lmap, B, H, W, N, NP, LD, M, G, K)
        d2 = dlmap.view(M, LD)
        x2d = fmap.reshape(M, C)
        if _loss_gemm_on_tc(C, LD) and ctx.fpair is not None and C == 256 and LD % 8 == 0:
            # both GEMMs of the Linear's backward on the tensor cores (fp16 two-term split, fp32-accurate, deterministic):
            #   dW = dL^T @ X  : K = pixels, MN-major operands (the tower's wgrad kernel with one tap)
            #   dX = dL @ W    : 1-tap conv with W^T (Cin = LD)
            dh, dl_, dinv = ops.split_f16(dlmap.view(B, H, W, LD), auto_scale=True)
            fh, fl, finv = ctx.fpair
            dw = ops.conv_tc_wgrad_f16(dh, dl_, fh, fl, 1, 1.0, dinv, finv)
            db = ops.col_sum(d2)
            dx = ops.conv_tc_f16(dh, dl_, ops.conv_tc_pack_weight_f16(wcat.t().contiguous(), 1), 1, C, dev_out_scale=dinv, ldy=C)
        else:
            dw, db = ops.linear_rows_bwd_w(d2, x2d)
            dx = ops.linear_rows_bwd_x(d2, wcat).view(B, H, W, C)
        return dx, dw[:N], db[:N], dw[NP:NP + N], db[NP:NP + N], None, None, None


@register_head
class CPRHead(PackedWeightsMixin, nn.Module):
    """Coarse Point Refine head (drop-in for the reference class of the same name)."""

    def __init__(self, num_classes, in_channels, feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64),
                 num_cls_fcs=0, fc_out_channels=1024,
                 train_pts_extractor=None, refine_pts_extractor=None, point_refiner=None,
                 ins_share_head_feat=True, ins_share_head_classifier=False,
                 loss_mil=None, loss_type=0, loss_cfg=None, normal_cfg=None, init_cfg=None,
                 debug=False, debug_info=None, other_info=None,
                 conv_cfg=None, norm_cfg=None, conv_bias='auto', dcn_on_last_conv=False,
                 loss_bbox=None, train_cfg=None, test_cfg=None, **kwargs):
        super().__init__()
        if kwargs:
            raise TypeError(f'CPRHead: unexpected kwargs {sorted(kwargs)}')
        self.num_classes, self.in_channels, self.feat_channels = num_classes, in_channels, feat_channels
        self.stacked_convs, self.strides = stacked_convs, list(strides)
        self.num_cls_fcs, self.fc_out_channels = num_cls_fcs, fc_out_channels
        self.ins_share_head_feat, self.ins_share_head_classifier = ins_share_head_feat, ins_share_head_classifier
        self.train_cfg, self.test_cfg, self.norm_cfg, self.conv_cfg = train_cfg, test_cfg, norm_cfg, conv_cfg
        self.loss_type = loss_type
        self.loss_mil_cfg = _merge(dict(type='MILLoss', binary_ins=False, loss_weight=1.0, eps=1e-6, loss_type='gfocal_loss'),
                                   loss_mil)
        self.loss_cfg = _merge(dict(with_neg=True, neg_loss_weight=1.0, refine_bag_policy='independent_with_gt_bag',
                                    random_remove_rate=0.4, with_gt_loss=False, gt_loss_weight=1.0, with_mil_loss=True),
                               loss_cfg)
        self.normal_cfg = _merge(dict(prob_cls_type='sigmoid', out_bg_cls=False), normal_cfg)
        self.train_pts_extractor = _merge(dict(pos_generator=dict(type='CirclePtFeatGenerator', radius=5),
                                               neg_generator=dict(type='OutCirclePtFeatGenerator', radius=3)),
                                          train_pts_extractor)
        self.refine_pts_extractor = _merge(dict(pos_generator=dict(type='CirclePtFeatGenerator', radius=5),
                                                neg_generator=dict(type='AnchorPtFeatGenerator', scale_factor=1.0)),
                                           refine_pts_extractor)
        self.point_refiner = _merge(dict(gt_alpha=0.5, merge_th=0.05, refine_th=0.05, classify_filter=False,
                                         nearest_filter=True, return_score_type='mean'), point_refiner)
        self.other_info = other_info or {}
        self.debug = debug
        self._check_supported()
        # ---- layers (cpr_head.py:983-1014)
        self.cls_convs = nn.ModuleList()
        chn = in_channels
        for _ in range(stacked_convs):
            self.cls_convs.append(ConvModule(chn, feat_channels, 3, 1, 1, norm_cfg=norm_cfg, bias=conv_bias))
            chn = feat_channels
        self.ins_convs = nn.ModuleList()
        self.cls_fcs, self.ins_fcs = nn.ModuleList(), nn.ModuleList()
        for _ in range(num_cls_fcs):                                             # cpr_head.py:1000-1006
            self.cls_fcs.append(nn.Linear(chn, fc_out_channels))
            chn = fc_out_channels
        self.num_cls_out = num_classes
        self.binary_ins = bool(self.loss_mil_cfg.get('binary_ins', False))
        self.cls_out = nn.Linear(chn, self.num_cls_out)
        if ins_share_head_classifier:
            assert not self.binary_ins                                           # cpr_head.py:1012
            self.ins_out = self.cls_out
        else:
            self.ins_out = nn.Linear(chn, self.num_cls_out * (2 if self.binary_ins else 1))
        self.init_weights()
        self._offset_cache = {}
        self._init_packed_hooks()

    # ------------------------------------------------------------------------------------------------
    def _check_supported(self):
        def need(cond, what):
            if not cond:
                raise NotImplementedError(f'CPRHead: {what} is not supported by the CUDA path')
        need(len(self.strides) == 1, 'more than one FPN level (the reference asserts a single level too, cpr_head.py:799,1152)')
        need(self.ins_share_head_feat, 'ins_share_head_feat=False')
        need(self.loss_mil_cfg.get('type', 'MILLoss') == 'MILLoss', 'loss_mil.type != MILLoss')
        need(self.loss_mil_cfg.get('loss_type', 'gfocal_loss') == 'gfocal_loss', 'MILLoss.loss_type != gfocal_loss')
        need(self.normal_cfg['prob_cls_type'] in ('sigmoid', 'softmax', 'normed_sigmoid'), f"prob_cls_type {self.normal_cfg['prob_cls_type']}")
        need(not self.normal_cfg['out_bg_cls'], 'out_bg_cls=True')
        need(self.loss_type == 0, 'loss_type != 0')
        for ex in (self.train_pts_extractor, self.refine_pts_extractor):
            need(ex['pos_generator']['type'] in _SUPPORTED_POS, f"pos_generator {ex['pos_generator']['type']}")
        need(self.train_pts_extractor['neg_generator']['type'] in _SUPPORTED_NEG,
             f"train neg_generator {self.train_pts_extractor['neg_generator']['type']}")
        need(self.loss_cfg.get('gt_loss_type', 'gt_refine') in ('gt_refine', 'gt'), 'gt_loss_type')
        need(self.point_refiner['return_score_type'] in ('mean', 'max'), 'return_score_type')

    def init_weights(self):
        """Normal(0, 0.01) for conv/linear, cls_out bias = bias_init_with_prob(0.01) (cpr_head.py:939-948)."""
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                normal_init_(m, 0.01, 0.0)
        nn.init.constant_(self.cls_out.bias, bias_init_with_prob(0.01))

    def _bags(self, gen_cfg, device):
        if gen_cfg['type'] == 'GridCirclesPtFeatGenerator':
            return _GridCircleBags(gen_cfg['radius'], gen_cfg.get('max_pos_num', -1), float(self.strides[0]))
        off, reach = self._offset_table(gen_cfg, device)
        return _CircleBags(off, float(self.strides[0]), reach)

    def _offsets(self, gen_cfg, device):
        return self._offset_table(gen_cfg, device)[0]

    def _offset_table(self, gen_cfg, device):
        """(device offset table, its reach in pixels); the reach comes from the host table when the table is built."""
        key = (gen_cfg.get('radius'), gen_cfg.get('start_angle', 0), gen_cfg.get('base_num_point', 8),
               gen_cfg.get('same_num_all_radius', False), gen_cfg.get('append_center', True), str(device))
        if key not in self._offset_cache:
            off = ops.circle_offsets(gen_cfg['radius'], self.strides[0], gen_cfg.get('start_angle', 0),
                                     gen_cfg.get('base_num_point', 8), gen_cfg.get('same_num_all_radius', False),
                                     gen_cfg.get('append_center', True))
            reach = ops.offsets_reach(off)
            self._offset_cache[key] = (ops.with_reach(off.to(device), reach), reach)
        return self._offset_cache[key]

    # ------------------------------------------------------------------------------------------------
    # ------------------------------------------------------------------------------------------------
    # generic path for the non-default variants the reference class accepts (num_cls_fcs > 0, binary_ins, prob_cls_type softmax /
    # normed_sigmoid, gt_weights): the reference's own data flow — gather the feat_channels-d bag features with the CUDA gather
    # (differentiable through ptb_cpr_bag_gather_bwd), then FC stack / classifiers / probabilities / losses as torch elementwise + GEMM
    # calls on the GPU (fp32, TF32 off).  The shipped configs (sigmoid, no FCs) never take it: they run the fused kernels.
    def _default_variant(self):
        return self.num_cls_fcs == 0 and not self.binary_ins and self.normal_cfg['prob_cls_type'] == 'sigmoid'

    def get_cls_prob(self, cls_out):
        """cpr_head.py:1080-1099."""
        t = self.normal_cfg['prob_cls_type']
        if t == 'sigmoid':
            return cls_out.sigmoid()
        if t == 'softmax':
            return cls_out.softmax(dim=-1)
        return torch.nn.functional.normalize(cls_out.sigmoid(), p=self.normal_cfg.get('normed_sigmoid_p', 1), dim=-1)

    def get_pts_outs(self, pts_cls_feats, want_ins=True):
        """cpr_head.py:1045-1078 for one level: FC stack (+ReLU) then cls_out / ins_out on (..., C) features."""
        shape = pts_cls_feats.shape
        x = pts_cls_feats.reshape(-1, shape[-1])
        for fc in self.cls_fcs:
            x = torch.relu(fc(x))
        cls_o = self.cls_out(x).reshape(*shape[:-1], -1)
        if not want_ins:
            return cls_o
        return cls_o, (cls_o if self.ins_out is self.cls_out else self.ins_out(x).reshape(*shape[:-1], -1))

    def _loss_generic(self, fmap, gt, hp, gt_weights):
        """CPRHead.loss0 (cpr_head.py:1131-1229) + MILLoss.forward (multi_instance_learning_loss.py:153-203), R = 1."""
        B, H, W, C = fmap.shape
        N, eps, dev = self.num_classes, hp['eps'], fmap.device
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            bags = self._bags(self.train_pts_extractor['pos_generator'], dev)
            feats, valid = _BagGatherFn.apply(fmap, gt, bags)                     # (G,K,C), (G,K)
            G, K, _ = feats.shape
            pos_cls, pos_ins = self.get_pts_outs(feats)
            neg_cls = self.get_pts_outs(fmap.reshape(B * H * W, C), want_ins=False)
            gw = torch.ones(G, device=dev) if gt_weights is None else torch.cat(list(gt_weights)).to(dev).float()
            labels = gt.labels64
            onehot = torch.zeros(G, N, device=dev)
            onehot[torch.arange(G, device=dev), labels] = 1
            losses, num_pos = {}, None
            vf = valid.float()
            if hp['with_gt_loss']:
                gt_prob = self.get_cls_prob(pos_cls[:, K - 1])
                wrep = (vf[:, K - 1] * gw).reshape(-1, 1)
                num_pos = torch.clamp((wrep > 0).sum(), min=1)
                losses['gt_loss'] = hp['gt_loss_weight'] * (_gfocal(gt_prob, onehot, wrep, eps).sum() / num_pos)
            if hp['with_mil_loss']:
                pw = vf * gw.reshape(-1, 1)                                       # (G,K) = valid * gt_weight (cpr_head.py:1211)
                prob_cls = self.get_cls_prob(pos_cls)
                nb = 2 if self.binary_ins else 1
                prob_ins = pos_ins.reshape(G, K, N, nb).softmax(dim=1) * pw[:, :, None, None]
                prob_ins = torch.nn.functional.normalize(prob_ins, dim=1, p=1)
                prob = (prob_cls.unsqueeze(-1) * prob_ins).sum(dim=1)             # (G,N,nb)
                acc = (prob[..., 0].argmax(dim=1) == labels).float().sum().reshape(1) * (100.0 / max(G, 1))
                lw = (pw.sum(dim=1, keepdim=True) > 0).float()                    # (G,1)
                num_sample = torch.clamp((lw.sum(dim=-1) > 0).float().sum(), min=1.0)
                if self.binary_ins:                                               # negative bag probability trained towards 0 (:179-186)
                    p_all = torch.cat([prob[..., 0], prob[..., 1]])
                    l_all = _gfocal(p_all, torch.cat([onehot, torch.zeros_like(onehot)]), torch.cat([lw, lw]), eps)
                else:
                    l_all = _gfocal(prob[..., 0], onehot, lw, eps)
                losses['pos_loss'] = hp['mil_loss_weight'] * (l_all.sum() / num_sample)
                losses['bag_acc'] = acc.detach()
                num_pos = num_sample
            if hp['with_neg']:
                nm = ops.neg_mask(B, H, W, hp['stride'], gt.pad_hw, gt.centers, gt.labels, gt.img_ptr, hp['stride'] * hp['neg_radius'], N,
                                  hp['neg_class_wise'], as_bool=False).reshape(-1, N).float()
                neg_prob = self.get_cls_prob(neg_cls)
                losses['neg_loss'] = hp['neg_loss_weight'] * (_gfocal(neg_prob, torch.zeros_like(neg_prob), nm, eps).sum() / num_pos)
            return losses
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32

    @torch.no_grad()
    def _refine_generic(self, fmap, gt, not_refine=None, want_chosen=False, want_bag_pts=False):
        """refine for the variants: bag features (CUDA gather) -> FC stack / cls_out / get_cls_prob (torch) -> ptb_cpr_refine (staged)."""
        pr = self.point_refiner
        dev = fmap.device
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            f, pts, valid, _ = self._bags(self.refine_pts_extractor['pos_generator'], dev).gather(fmap, gt, pts=True)
            prob = self.get_cls_prob(self.get_pts_outs(f, want_ins=False)).contiguous()
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
        groups = ops.label_groups(gt.bag_img, gt.labels, self.num_classes)
        cfg = ops._refine_cfg(pr['merge_th'], pr['gt_alpha'], pr['refine_th'], pr['nearest_filter'], pr['classify_filter'],
                              pr['return_score_type'] == 'max')
        o_pts, o_sc, o_nr, o_ch, _ = ops.refine(prob, pts, valid, pts.shape[1], gt.labels, gt.bag_img, gt.img_hw, groups, cfg,
                                                not_refine=not_refine, want_masks=want_chosen)
        return (o_pts, o_sc, o_nr, o_ch, pts[..., :2]) if want_bag_pts else (o_pts, o_sc, o_nr, o_ch)

    def forward(self, feats):
        """cpr_head.py:1030-1043: returns feature maps (not logits)."""
        cls_feats, ins_feats = [], []
        info = {}
        for x in feats:
            c = tower(self.cls_convs, x, info)
            self.last_tower_backend = info.get('backend')
            cls_feats.append(c)
            ins_feats.append(c)
        return cls_feats, ins_feats

    def forward_train(self, x, img_metas, gt_bboxes, gt_labels=None, gt_bboxes_ignore=None, gt_true_bboxes=None,
                      proposal_cfg=None, **kwargs):
        outs = self(x)
        losses = self.loss(*outs, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=gt_bboxes_ignore,
                           gt_true_bboxes=gt_true_bboxes)
        if proposal_cfg is None:
            return losses
        raise NotImplementedError('proposal_cfg')

    def simple_test(self, feats, img_metas, rescale=False, **kwargs):
        """dense_test_mixins.py:15-36 (forward -> get_bboxes).  Inference fast path: the towers hand their output over
        as the fp16 operand pair and the class-logit map comes from the same wgmma kernel (1 tap, N = num_classes),
        so neither the fp32 feature map nor an FFMA GEMM appears in the step; results are identical within 1e-4."""
        x = feats[0]
        if len(feats) == 1 and self._default_variant() and tc_enabled(x, self.cls_convs, self.cls_out) and not torch.is_grad_enabled() \
                and self.in_channels % 32 == 0 and self.feat_channels == 256:
            info = {}
            pair = tower(self.cls_convs, x, info, want='f16pair')
            if pair is not None:
                self.last_tower_backend = info.get('backend')
                self.last_overflow_flag = info.get('overflow_flag')
                if self.debug and self.last_overflow_flag is not None and int(self.last_overflow_flag) != 0:    # host sync: debug only
                    raise FloatingPointError('CPRHead: a GroupNorm output exceeded the fp16 operand range (|x| > 6e4) and was clamped')
                h, l = pair
                lmap = ops.conv_tc_f16(h, l, _packed_tc(self.cls_out, 1, 'lin'), 1, self.num_classes, bias=self.cls_out.bias.detach())
                return self._get_bboxes_from_logit_map(lmap, img_metas, rescale=rescale, **kwargs)
        outs = self.forward(feats)
        return self.get_bboxes(*outs, img_metas, rescale=rescale, **kwargs)

    # ------------------------------------------------------------------------------------------------
    def loss(self, cls_feat, ins_feat, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=None, gt_true_bboxes=None,
             gt_weights=None):
        assert len(gt_labels) > 0
        feat = cls_feat[0]
        if not feat.is_cuda:
            raise RuntimeError('CPRHead runs on CUDA tensors only; there is no CPU fallback')
        gt = _BatchGT(gt_bboxes, gt_labels, img_metas, feat.device)
        pos, neg = self.train_pts_extractor['pos_generator'], self.train_pts_extractor['neg_generator']
        hp = dict(num_classes=self.num_classes, stride=float(self.strides[0]), eps=float(self.loss_mil_cfg.get('eps', 1e-6)),
                  mil_loss_weight=float(self.loss_mil_cfg.get('loss_weight', 1.0)),
                  with_gt_loss=bool(self.loss_cfg.get('with_gt_loss', False)),
                  gt_loss_weight=float(self.loss_cfg.get('gt_loss_weight', 1.0)),
                  with_mil_loss=bool(self.loss_cfg.get('with_mil_loss', True)),
                  with_neg=bool(self.loss_cfg.get('with_neg', True)),
                  neg_loss_weight=float(self.loss_cfg.get('neg_loss_weight', 1.0)),
                  neg_radius=float(neg['radius']), neg_class_wise=bool(neg.get('class_wise', False)))
        fmap = ops.to_nhwc(feat)
        if gt_weights is not None or not self._default_variant():
            return self._loss_generic(fmap.contiguous(), gt, hp, gt_weights)
        gt_loss, pos_loss, neg_loss, bag_acc = _CPRLossFn.apply(
            fmap, self.cls_out.weight, self.cls_out.bias, self.ins_out.weight, self.ins_out.bias, gt,
            self._bags(pos, feat.device), hp)
        losses = {}
        if hp['with_gt_loss']:
            losses['gt_loss'] = gt_loss
        if hp['with_mil_loss']:
            losses['pos_loss'] = pos_loss
            losses['bag_acc'] = bag_acc.detach().reshape(1)
        if hp['with_neg']:
            losses['neg_loss'] = neg_loss
        return losses

    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def refine_points(self, feat, gt, not_refine=None, want_chosen=False, want_bag_pts=False):
        """logit map -> fused sample/sigmoid/filter/merge kernel.  returns pts (G,2), scores (G,), not_refine (G,) bool,
        chosen (G,K) bool | None [, bag points (G,K,2) when want_bag_pts]."""
        fmap = ops.to_nhwc(feat)
        if not self._default_variant():
            return self._refine_generic(fmap.contiguous(), gt, not_refine, want_chosen, want_bag_pts)
        B, H, W, C = fmap.shape
        lmap = ops.linear_rows(fmap.reshape(-1, C), self.cls_out.weight, self.cls_out.bias).view(B, H, W, self.num_classes) \
            if self.num_classes % 4 == 0 else self._padded_logit_map(fmap)
        return self._refine_from_logit_map(lmap, gt, not_refine, want_chosen, want_bag_pts)

    @torch.no_grad()
    def _refine_from_logit_map(self, lmap, gt, not_refine=None, want_chosen=False, want_bag_pts=False):
        pr = self.point_refiner
        dev = lmap.device
        if max(gt.lens) <= 8192 and self.num_classes <= 1024:
            groups = ops.label_groups_csr(gt.labels, gt.img_ptr, self.num_classes, max(gt.lens))
        else:
            groups = ops.label_groups(gt.bag_img, gt.labels, self.num_classes)
        cfg = ops._refine_cfg(pr['merge_th'], pr['gt_alpha'], pr['refine_th'], pr['nearest_filter'], pr['classify_filter'],
                              pr['return_score_type'] == 'max')
        gen = self.refine_pts_extractor['pos_generator']
        if gen['type'] == 'GridCirclesPtFeatGenerator':
            # staged: grid-cell bags of class logits -> sigmoid -> ptb_cpr_refine (bags are ragged, no offset table)
            f, pts, valid, _ = self._bags(gen, dev).gather(lmap, gt, pts=True)
            prob = torch.sigmoid(f[..., :self.num_classes]).contiguous()
            o_pts, o_sc, o_nr, o_ch, _ = ops.refine(prob, pts, valid, pts.shape[1], gt.labels, gt.bag_img, gt.img_hw, groups, cfg,
                                                    not_refine=not_refine, want_masks=want_chosen)
            return (o_pts, o_sc, o_nr, o_ch, pts[..., :2]) if want_bag_pts else (o_pts, o_sc, o_nr, o_ch)
        off, reach = self._offset_table(gen, dev)
        out = ops.refine_fused(lmap, self.num_classes, gt.centers, gt.labels, gt.bag_img, off, self.strides[0], gt.pad_hw,
                               gt.img_hw, groups, cfg, not_refine=not_refine, want_chosen=want_chosen, reach_px=reach)
        if want_bag_pts:
            return out + (off[None, :, :] + gt.centers[:, None, :],)        # cpr_head.py:492-497 (same fp32 add as the kernel)
        return out

    def _padded_logit_map(self, fmap):
        B, H, W, C = fmap.shape
        n4 = (self.num_classes + 3) // 4 * 4
        w = torch.zeros((n4, C), device=fmap.device)
        b = torch.zeros((n4,), device=fmap.device)
        w[:self.num_classes], b[:self.num_classes] = self.cls_out.weight, self.cls_out.bias
        return ops.linear_rows(fmap.reshape(-1, C), w, b).view(B, H, W, n4)

    @torch.no_grad()
    def get_bboxes(self, cls_feat, ins_feat, img_metas, cfg=None, rescale=False, with_nms=True, gt_bboxes=None,
                   gt_labels=None, gt_bboxes_ignore=None, gt_true_bboxes=None, gt_anns_id=None, not_refine=None,
                   cascade_out_fmt=False):
        """cpr_head.py:1231-1283; one row per GT point: [x1,y1,x2,y2,score,ann_id]."""
        assert gt_labels is not None and len(gt_labels) > 0
        feat = cls_feat[0]
        if not feat.is_cuda:
            raise RuntimeError('CPRHead runs on CUDA tensors only; there is no CPU fallback')
        gt = _BatchGT(gt_bboxes, gt_labels, img_metas, feat.device)
        nr_in = torch.cat(list(not_refine)).to(feat.device) if not_refine is not None else None
        geo = bool(self.other_info.get('out_geo', False))
        out = self.refine_points(feat, gt, nr_in, want_chosen=geo, want_bag_pts=geo)
        return self._format_results(out, gt, img_metas, rescale, gt_labels, gt_anns_id, cascade_out_fmt, with_nms)

    @torch.no_grad()
    def _get_bboxes_from_logit_map(self, lmap, img_metas, rescale=False, gt_bboxes=None, gt_labels=None, gt_anns_id=None,
                                   not_refine=None, cascade_out_fmt=False, with_nms=True, **unused):
        assert gt_labels is not None and len(gt_labels) > 0
        gt = _BatchGT(gt_bboxes, gt_labels, img_metas, lmap.device)
        nr_in = torch.cat(list(not_refine)).to(lmap.device) if not_refine is not None else None
        geo = bool(self.other_info.get('out_geo', False))
        out = self._refine_from_logit_map(lmap, gt, nr_in, want_chosen=geo, want_bag_pts=geo)
        return self._format_results(out, gt, img_metas, rescale, gt_labels, gt_anns_id, cascade_out_fmt, with_nms)

    def _format_results(self, refined, gt, img_metas, rescale, gt_labels, gt_anns_id, cascade_out_fmt, with_nms):
        pts, scores, nr = refined[:3]
        feat = pts
        boxes = torch.cat([pts - 8.0, pts + 8.0], dim=-1)                        # center_to_pseudo_bbox (16x16)
        sf = None
        if rescale:
            sf = torch.tensor(np.array([m['scale_factor'] for m in img_metas], dtype=np.float32), device=feat.device)
            sf = sf[gt.bag_img.long()]
            boxes = boxes / sf
        ann = torch.cat(list(gt_anns_id)).to(feat.device).type_as(boxes) if gt_anns_id is not None \
            else torch.arange(gt.G, device=feat.device).type_as(boxes)
        det = torch.cat([boxes, scores[:, None], ann[:, None]], dim=-1)
        dets = list(torch.split(det, gt.lens))
        if self.other_info.get('out_geo', False):
            # geometry columns (cpr_head.py:855-866, 1262-1273): [refined point, chosen bag points ...] per GT, flattened, padded
            # with -1 to the longest list OF THE IMAGE.  Chosen points keep their bag order (stable partition of the mask).
            chosen, bag_pts = refined[3], refined[4]
            K = chosen.shape[1]
            cnt = chosen.sum(dim=1)
            order = torch.argsort((~chosen).to(torch.uint8), dim=1, stable=True)
            cp = torch.gather(bag_pts, 1, order[..., None].expand(-1, -1, 2))
            geo = torch.cat([pts[:, None, :], cp], dim=1)                        # (G, 1+K, 2)
            if sf is not None:
                geo = geo / sf[:, None, :2]
            keep = torch.arange(K + 1, device=feat.device)[None, :] <= cnt[:, None]
            geo = torch.where(keep[..., None], geo, torch.full_like(geo, -1.0))
            lmax = [int(c.max()) + 1 if len(c) else 1 for c in torch.split(cnt.cpu(), gt.lens)]
            dets = [torch.cat([d, g[:, :m].reshape(len(g), -1)], dim=-1) for d, g, m in zip(dets, torch.split(geo, gt.lens), lmax)]
        res = list(zip(dets, [l.to(feat.device) for l in gt_labels]))
        if cascade_out_fmt:
            return res, list(torch.split(nr, gt.lens))
        if not with_nms:
            raise NotImplementedError
        return res
