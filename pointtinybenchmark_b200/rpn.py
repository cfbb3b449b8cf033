"""Dense-anchor proposal path (SURVEY.md §8f rank 4, BASELINE.json configs[3]) — host-side mirror of the reference pieces around
ptb_rpn_proposals:

  AnchorGenerator   mmdet/core/anchor/anchor_generator.py:9-330 (base anchors, grid anchors, valid flags; same ctor kwargs).  The base
                    anchors are input-independent (a few floats per level): computed once with torch CPU ops in the reference's
                    order, so they are bit-identical; the H*W*A grid anchors are NOT materialised on the proposal path — the decode
                    kernel forms `base[a] + shift(x, y)` on the fly — `grid_anchors` exists for callers that want the tensor
                    (e.g. to feed MaxIoUAssigner).
  RPNProposals      the `get_bboxes` of RPNHead (AnchorHead.get_bboxes, anchor_head.py:551-590 -> RPNHead._get_bboxes,
                    rpn_head.py:78-186): same arguments (cls_scores, bbox_preds, img_metas, cfg, rescale, with_nms), same result
                    (list of (n, 5) tensors), one library call for the whole batch instead of the per-level / per-image Python loop.
There is no CPU path: CUDA tensors only.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .assigners import MaxIoUAssigner, random_sample_plan, sampled_counts, upload_sample_plan
from .post_processing import parse_nms_cfg
from .registry import CfgNode


def _as_wh(stride):
    """a stride given as one number means the same step along x and y"""
    if isinstance(stride, (tuple, list)):
        if len(stride) != 2:
            raise ValueError(f'a stride is one number or an (x, y) pair, got {stride!r}')
        return int(stride[0]), int(stride[1])
    return int(stride), int(stride)


class AnchorGenerator:
    """Same constructor keywords, attributes and method names as the reference generator (anchor_generator.py:9-330), organised around
    one table per pyramid level: `strides[l]` = (step_x, step_y), `base_sizes[l]`, `base_anchors[l]` = (A, 4) fp32 boxes around the
    level's anchor centre.  Only the base-anchor arithmetic has to follow the reference operation by operation (it is the one place where
    fp32 rounding enters: sqrt of the ratios, two products per side); grid anchors are `base + (x * step_x, y * step_y)` — one exact
    integer-valued shift and one fp32 add per coordinate however the shift grid is laid out — and the valid flags are index comparisons."""

    def __init__(self, strides, ratios, scales=None, base_sizes=None, scale_major=True, octave_base_scale=None, scales_per_octave=None,
                 centers=None, center_offset=0.):
        self.strides = [_as_wh(st) for st in strides]
        n_lvl = len(self.strides)
        if not 0 <= center_offset <= 1:
            raise ValueError(f'center_offset must lie in [0, 1] (fraction of the base size), got {center_offset}')
        if centers is not None and center_offset != 0:
            raise AssertionError(f'explicit centers ({centers}) and a non-zero center_offset exclude each other')
        if centers is not None and len(centers) != n_lvl:
            raise AssertionError(f'{len(centers)} centers for {n_lvl} levels')
        self.base_sizes = [min(st) for st in self.strides] if base_sizes is None else list(base_sizes)
        if len(self.base_sizes) != n_lvl:
            raise AssertionError(f'{len(self.base_sizes)} base sizes for {n_lvl} strides')
        octave = octave_base_scale is not None and scales_per_octave is not None
        if octave == (scales is not None):
            raise AssertionError('give either `scales` or (`octave_base_scale`, `scales_per_octave`), not both and not neither')
        if octave:
            steps = np.array([2 ** (k / scales_per_octave) for k in range(scales_per_octave)])
            self.scales = torch.Tensor(steps * octave_base_scale)
        else:
            self.scales = torch.Tensor(scales)
        self.ratios = torch.Tensor(ratios)
        self.octave_base_scale, self.scales_per_octave = octave_base_scale, scales_per_octave
        self.scale_major, self.centers, self.center_offset = scale_major, centers, center_offset
        self.base_anchors = self.gen_base_anchors()

    num_levels = property(lambda self: len(self.strides))
    num_base_anchors = property(lambda self: [int(t.shape[0]) for t in self.base_anchors])

    def gen_base_anchors(self):
        return [self.gen_single_level_base_anchors(size, self.scales, self.ratios, self.centers[lvl] if self.centers is not None else None)
                for lvl, size in enumerate(self.base_sizes)]

    def gen_single_level_base_anchors(self, base_size, scales, ratios, center=None):
        """(A, 4) boxes of side base_size * scale, aspect h / w = ratio, around the level's centre — the reference's fp32 operation order
        (anchor_generator.py:112-151): sqrt(ratio) and its reciprocal, then (size * ratio_term) * scale, or scale first when not scale_major."""
        cx, cy = center if center is not None else (self.center_offset * base_size, self.center_offset * base_size)
        tall = torch.sqrt(ratios)
        wide = 1 / tall
        if self.scale_major:
            half_w = 0.5 * (base_size * wide[:, None] * scales[None, :]).view(-1)
            half_h = 0.5 * (base_size * tall[:, None] * scales[None, :]).view(-1)
        else:
            half_w = 0.5 * (base_size * scales[:, None] * wide[None, :]).view(-1)
            half_h = 0.5 * (base_size * scales[:, None] * tall[None, :]).view(-1)
        return torch.stack([cx - half_w, cy - half_h, cx + half_w, cy + half_h], dim=-1)

    def single_level_grid_anchors(self, base_anchors, featmap_size, stride=(16, 16), device='cuda'):
        """(H*W*A, 4): cell (y, x) major, base anchor minor — the order of the head's permute(0, 2, 3, 1) logits."""
        rows, cols = featmap_size
        step_x, step_y = stride
        xs = (torch.arange(cols, device=device) * step_x).to(base_anchors.dtype)
        ys = (torch.arange(rows, device=device) * step_y).to(base_anchors.dtype)
        shift = torch.stack([xs[None, :].expand(rows, cols), ys[:, None].expand(rows, cols)], dim=-1).repeat(1, 1, 2)      # (H, W, 4) = x, y, x, y
        return (shift[:, :, None, :] + base_anchors[None, None, :, :]).reshape(-1, 4)

    def grid_anchors(self, featmap_sizes, device='cuda'):
        if len(featmap_sizes) != self.num_levels:
            raise AssertionError(f'{len(featmap_sizes)} feature maps for {self.num_levels} levels')
        return [self.single_level_grid_anchors(self.base_anchors[lvl].to(device), size, self.strides[lvl], device=device)
                for lvl, size in enumerate(featmap_sizes)]

    def valid_extent(self, featmap_sizes, pad_shape):
        """per level (rows, cols) of valid cells: min(ceil(padded image extent / stride), map size) (anchor_generator.py:292-296)"""
        img_h, img_w = pad_shape[:2]
        out = []
        for lvl, (rows, cols) in enumerate(featmap_sizes):
            step_x, step_y = self.strides[lvl]
            ok_cols = min(-(-int(img_w) // step_x) if float(img_w).is_integer() else int(np.ceil(img_w / step_x)), cols)
            ok_rows = min(-(-int(img_h) // step_y) if float(img_h).is_integer() else int(np.ceil(img_h / step_y)), rows)
            out.append((ok_rows, ok_cols))
        return out

    def valid_flags(self, featmap_sizes, pad_shape, device='cuda'):
        """per level a bool (H*W*A,): the anchors of the cells whose index is below ceil(padded image extent / stride)
        (anchor_generator.py:272-330)"""
        if len(featmap_sizes) != self.num_levels:
            raise AssertionError(f'{len(featmap_sizes)} feature maps for {self.num_levels} levels')
        flags = []
        for lvl, ((rows, cols), (ok_rows, ok_cols)) in enumerate(zip(featmap_sizes, self.valid_extent(featmap_sizes, pad_shape))):
            cell_ok = (torch.arange(rows, device=device) < ok_rows)[:, None] & (torch.arange(cols, device=device) < ok_cols)[None, :]
            flags.append(cell_ok.reshape(-1, 1).expand(rows * cols, self.num_base_anchors[lvl]).reshape(-1))
        return flags


class RPNProposals:
    """get_bboxes of the reference RPNHead (sigmoid classification, DeltaXYWHBBoxCoder) over ptb_rpn_proposals."""

    def __init__(self, anchor_generator, bbox_coder=None, test_cfg=None, use_sigmoid_cls=True):
        ag = dict(anchor_generator)
        if ag.pop('type', 'AnchorGenerator') != 'AnchorGenerator':
            raise NotImplementedError('only AnchorGenerator is implemented')
        self.anchor_generator = AnchorGenerator(**ag)
        bc = dict(bbox_coder or dict(type='DeltaXYWHBBoxCoder'))
        if bc.pop('type', 'DeltaXYWHBBoxCoder') != 'DeltaXYWHBBoxCoder':
            raise NotImplementedError('only DeltaXYWHBBoxCoder is implemented')
        if bc.get('add_ctr_clamp', False) or not bc.get('clip_border', True):
            raise NotImplementedError('DeltaXYWHBBoxCoder(add_ctr_clamp=True / clip_border=False)')
        self.means, self.stds = tuple(bc.get('target_means', (0., 0., 0., 0.))), tuple(bc.get('target_stds', (1., 1., 1., 1.)))
        self.wh_ratio_clip = 16 / 1000                       # DeltaXYWHBBoxCoder.decode default (delta_xywh_bbox_coder.py:88)
        if not use_sigmoid_cls:
            raise NotImplementedError('RPN softmax classification (loss_cls.use_sigmoid=False)')
        if len(set(self.anchor_generator.num_base_anchors)) != 1:
            raise NotImplementedError('levels with different numbers of base anchors')
        self.test_cfg = CfgNode(test_cfg) if test_cfg is not None else None
        self._base_dev = {}

    def _base(self, device):
        if device not in self._base_dev:
            self._base_dev[device] = torch.stack(self.anchor_generator.base_anchors).to(device).contiguous()
        return self._base_dev[device]

    @torch.no_grad()
    def get_bboxes_padded(self, cls_scores, bbox_preds, img_metas, cfg=None):
        """one ptb_rpn_proposals launch for the batch, no synchronisation: count (B,) int32, det (B, max_per_img, 5), level (B, max)"""
        assert len(cls_scores) == len(bbox_preds) == self.anchor_generator.num_levels
        if not cls_scores[0].is_cuda:
            raise RuntimeError('RPNProposals runs on CUDA tensors only; there is no CPU fallback')
        cfg = CfgNode(cfg) if cfg is not None else self.test_cfg
        nms = parse_nms_cfg(cfg.get('nms', dict(iou_threshold=cfg.get('nms_thr', 0.7))), default_iou=0.7)
        if nms.kind != 'nms':
            raise NotImplementedError(f'rpn nms type {nms.kind}')
        max_per_img = cfg.get('max_per_img', cfg.get('max_num', cfg.get('nms_post', 1000)))   # older configs spell it max_num / nms_post
        dev = cls_scores[0].device
        img_hw = torch.tensor([[int(m['img_shape'][0]), int(m['img_shape'][1])] for m in img_metas], dtype=torch.int32).to(dev)
        return ops.rpn_proposals([c.detach().float().contiguous() for c in cls_scores], [r.detach().float().contiguous() for r in bbox_preds],
                                 self._base(dev), self.anchor_generator.strides, img_hw, self.means, self.stds, self.wh_ratio_clip,
                                 cfg.get('nms_pre', -1), cfg.get('min_bbox_size', 0), nms.iou, max_per_img)

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, img_metas, cfg=None, rescale=False, with_nms=True, return_levels=False):
        if not with_nms:
            raise NotImplementedError('with_nms=False')
        cnt, det, lvl = self.get_bboxes_padded(cls_scores, bbox_preds, img_metas, cfg)
        cnt = cnt.cpu().tolist()                      # ragged result lists, like the reference's per-image dets
        out = [det[b, :cnt[b]] for b in range(len(cnt))]
        if return_levels:
            return out, [lvl[b, :cnt[b]] for b in range(len(cnt))]
        return out


def inside_boxes(anchor_generator, featmap_sizes, img_metas, allowed_border):
    """(B, L, A, 4) int32 (x0, x1, y0, y1): anchor (l, y, x, a) of image b is inside — valid_flags of pad_shape and, when
    allowed_border >= 0, anchor_inside_flags against img_shape (core/anchor/utils.py:20-45) — iff x0 <= x < x1 and y0 <= y < y1.  The
    border test compares the fp32 anchor coordinates base[a] + x * stride, which grow with x (y), so each test keeps an interval."""
    ag = anchor_generator
    L, A = ag.num_levels, ag.num_base_anchors[0]
    out = np.zeros((len(img_metas), L, A, 4), np.int32)
    for b, meta in enumerate(img_metas):
        ext = ag.valid_extent(featmap_sizes, meta['pad_shape'])
        img_h, img_w = meta['img_shape'][:2]
        for l, (ok_rows, ok_cols) in enumerate(ext):
            sx, sy = ag.strides[l]
            base = ag.base_anchors[l].numpy()
            xs = (np.arange(ok_cols) * sx).astype(np.float32)
            ys = (np.arange(ok_rows) * sy).astype(np.float32)
            for a in range(A):
                if allowed_border >= 0:
                    mx = (base[a, 0] + xs >= np.float32(-allowed_border)) & (base[a, 2] + xs < np.float32(img_w + allowed_border))
                    my = (base[a, 1] + ys >= np.float32(-allowed_border)) & (base[a, 3] + ys < np.float32(img_h + allowed_border))
                else:
                    mx, my = np.ones(ok_cols, bool), np.ones(ok_rows, bool)
                ix, iy = np.flatnonzero(mx), np.flatnonzero(my)
                if len(ix) and len(iy):
                    out[b, l, a] = (ix[0], ix[-1] + 1, iy[0], iy[-1] + 1)
    return out


_SAMPLING_OFF = ('FocalLoss', 'GHMC', 'QualityFocalLoss')      # anchor_head.py:66-68: these turn sampling off (PseudoSampler)


class _RPNLevelSums(torch.autograd.Function):
    """the (L, 2) un-normalised loss sums (cls, bbox) per level over the maps, read in place; backward writes the maps' gradients."""

    @staticmethod
    def forward(ctx, tg, *maps):
        L = len(maps) // 2
        ctx.tg = tg
        ctx.save_for_backward(*maps)
        return torch.stack([ops.rpn_level_loss(maps[l], maps[L + l], *tg.level(l), tg.bbox_loss, tg.beta) for l in range(L)])

    @staticmethod
    def backward(ctx, g):
        maps = ctx.saved_tensors
        L = len(maps) // 2
        g = g.float().contiguous()
        gc, gb = zip(*[ops.rpn_level_loss(maps[l], maps[L + l], *ctx.tg.level(l), ctx.tg.bbox_loss, ctx.tg.beta, scale=g[l],
                                          want_grad=True) for l in range(L)])
        return (None, *gc, *gb)


class RPNTargets:
    """AnchorHead.get_targets of one batch on the device.  labels / label_weights in the layout of the concatenated cls_score maps,
    bbox_targets / bbox_weights in that of the bbox_pred maps (level after level); `pos_inds` / `neg_inds` per image (flat anchor
    index) on request; `num_total_samples` the loss's avg_factor (anchor_head.py:352-353, 467-468)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def level(self, l):
        a, b = self.cls_off[l], self.cls_off[l + 1]
        return self.labels[a:b], self.label_weights[a:b], self.bbox_targets[4 * a:4 * b], self.bbox_weights[4 * a:4 * b]

    def level_targets(self, l):
        """level l's targets in the reference's layout (images_to_levels): (B, H*W*A) and (B, H*W*A, 4)"""
        B, A, (H, W) = self.B, self.A, self.featmap_sizes[l]
        lab, lw, bt, bw = self.level(l)
        p = lambda t, k: t.view(B, A, k, H, W).permute(0, 3, 4, 1, 2).reshape(B, H * W * A, k)
        return p(lab, 1)[..., 0], p(lw, 1)[..., 0], p(bt, 4), p(bw, 4)

    def sampled_sets(self):
        """per image the sampled positive and negative anchors (AnchorHead's pos_inds / neg_inds: indices of the inside anchors)"""
        out = []
        for b in range(self.B):
            n = self.n_inside[b]
            g, r = self.gt_inds[b, :n], self.rank[b, :n]
            pos, neg = self.plan[b]
            sel = []
            for kind, s in ((g > 0, pos), (g == 0, neg)):
                idx = torch.nonzero(kind).squeeze(1)
                sel.append(idx if s is None else idx[s.to(idx.device)])
            out.append(tuple(sel))
        return out


class RPNHead(nn.Module):
    """mmdet/models/dense_heads/rpn_head.py:12-75 (AnchorHead with one sigmoid class): same constructor keywords, parameter names
    (rpn_conv, rpn_cls, rpn_reg), `forward`, `forward_single`, `loss`, `forward_train`, `get_bboxes` and the detector's test entry
    `simple_test_rpn` (`aug_test_rpn` raises NotImplementedError).  The convs stay nn.Conv2d;
    `loss` runs AnchorHead.get_targets (inside flags, MaxIoUAssigner, RandomSampler, bbox2delta, unmap) and the per-level
    CrossEntropyLoss(use_sigmoid=True) + L1Loss / SmoothL1Loss in the ptb_rpn_* kernels, one autograd function over the output maps."""

    def __init__(self, in_channels, feat_channels=256,
                 anchor_generator=dict(type='AnchorGenerator', scales=[8, 16, 32], ratios=[0.5, 1.0, 2.0], strides=[4, 8, 16, 32, 64]),
                 bbox_coder=dict(type='DeltaXYWHBBoxCoder', clip_border=True, target_means=(.0, .0, .0, .0), target_stds=(1.0, 1.0, 1.0, 1.0)),
                 reg_decoded_bbox=False, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.0), train_cfg=None, test_cfg=None,
                 init_cfg=dict(type='Normal', layer='Conv2d', std=0.01)):
        super().__init__()
        lc, lb = dict(loss_cls), dict(loss_bbox)
        t = lc.get('type')
        if t in _SAMPLING_OFF:
            raise NotImplementedError(f'RPNHead with loss_cls {t}: it turns sampling off (PseudoSampler), which is not implemented')
        if t != 'CrossEntropyLoss':
            raise NotImplementedError(f'RPNHead loss_cls {t}: CrossEntropyLoss(use_sigmoid=True) is implemented')
        if not lc.get('use_sigmoid', False):
            raise NotImplementedError('RPN softmax classification (loss_cls.use_sigmoid=False)')
        if lc.get('use_mask', False) or lc.get('class_weight') is not None or lc.get('reduction', 'mean') != 'mean':
            raise NotImplementedError("RPNHead CrossEntropyLoss with use_mask, class_weight or a reduction other than 'mean'")
        tb = lb.get('type')
        if tb not in ('L1Loss', 'SmoothL1Loss'):
            raise NotImplementedError(f'RPNHead loss_bbox {tb}: L1Loss and SmoothL1Loss are implemented')
        if lb.get('reduction', 'mean') != 'mean':
            raise NotImplementedError(f"RPNHead {tb} with reduction {lb.get('reduction')!r}: 'mean' is implemented")
        if reg_decoded_bbox:
            raise NotImplementedError('RPNHead(reg_decoded_bbox=True)')
        self.in_channels, self.feat_channels, self.num_classes, self.cls_out_channels = in_channels, feat_channels, 1, 1
        self.use_sigmoid_cls, self.sampling, self.reg_decoded_bbox = True, True, False
        self.cls_loss_weight = float(lc.get('loss_weight', 1.0))
        self.bbox_loss_kind = ops.RPN_LOSS_L1 if tb == 'L1Loss' else ops.RPN_LOSS_SMOOTH_L1
        self.bbox_beta = float(lb.get('beta', 1.0)) if tb == 'SmoothL1Loss' else 0.0
        if tb == 'SmoothL1Loss' and not self.bbox_beta > 0:
            raise ValueError(f'SmoothL1Loss beta must be > 0, got {self.bbox_beta}')
        self.bbox_loss_weight = float(lb.get('loss_weight', 1.0))
        self.proposals = RPNProposals(anchor_generator, bbox_coder, test_cfg)
        self.anchor_generator = self.proposals.anchor_generator
        self.num_anchors = self.anchor_generator.num_base_anchors[0]
        self.means, self.stds = self.proposals.means, self.proposals.stds
        self.train_cfg = CfgNode(train_cfg) if train_cfg is not None else None
        self.test_cfg = self.proposals.test_cfg
        self.init_cfg = init_cfg
        if self.train_cfg is not None:
            asg = dict(self.train_cfg.get('assigner') or {})
            t = asg.pop('type', None)
            if t != 'MaxIoUAssigner':
                raise NotImplementedError(f'RPNHead assigner {t}: MaxIoUAssigner is implemented')
            self.assigner = MaxIoUAssigner(**asg)
            smp = dict(self.train_cfg.get('sampler') or {})
            t = smp.pop('type', 'PseudoSampler')
            if t != 'RandomSampler':
                raise NotImplementedError(f'RPNHead sampler {t}: RandomSampler is implemented')
            self.sampler_cfg = dict(num=smp['num'], pos_fraction=smp['pos_fraction'], neg_pos_ub=smp.get('neg_pos_ub', -1))
            # AnchorHead samples without gt_labels (anchor_head.py:220-221), so the reference's BaseSampler raises for an image with GTs
            # when add_gt_as_proposals is set (its default); get_targets raises the same error
            self.sampler_add_gt = bool(smp.get('add_gt_as_proposals', True))
        self.rpn_conv = nn.Conv2d(in_channels, feat_channels, 3, padding=1)
        self.rpn_cls = nn.Conv2d(feat_channels, self.num_anchors * self.cls_out_channels, 1)
        self.rpn_reg = nn.Conv2d(feat_channels, self.num_anchors * 4, 1)
        self.init_weights()

    def init_weights(self):
        """init_cfg Normal(std=0.01) on every Conv2d, bias 0 (mmcv normal_init)"""
        std = float(dict(self.init_cfg or {}).get('std', 0.01))
        for m in (self.rpn_conv, self.rpn_cls, self.rpn_reg):
            nn.init.normal_(m.weight, 0.0, std)
            nn.init.constant_(m.bias, 0.0)

    def forward_single(self, x):
        x = F.relu(self.rpn_conv(x), inplace=True)
        return self.rpn_cls(x), self.rpn_reg(x)

    def forward(self, feats):
        return tuple(map(list, zip(*[self.forward_single(x) for x in feats])))

    def get_targets(self, featmap_sizes, gt_bboxes, img_metas, gt_bboxes_ignore=None, device='cuda'):
        """AnchorHead.get_targets for the whole batch; None when an image has no inside anchor (anchor_head.py:212-213, 349-350),
        after the draws of the images before and after it, as the reference makes them."""
        if self.train_cfg is None:
            raise RuntimeError('RPNHead.loss needs train_cfg')
        if self.sampler_add_gt and any(len(g) > 0 for g in gt_bboxes):
            raise ValueError('gt_labels must be given when add_gt_as_proposals is True (base_sampler.py:73-76: AnchorHead samples '
                             'without gt_labels; RPN configs set train_cfg.rpn.sampler.add_gt_as_proposals=False)')
        ag, B, A = self.anchor_generator, len(img_metas), self.num_anchors
        if len(featmap_sizes) != ag.num_levels:
            raise AssertionError(f'{len(featmap_sizes)} feature maps for {ag.num_levels} levels')
        boxes = inside_boxes(ag, featmap_sizes, img_metas, self.train_cfg.get('allowed_border', 0))
        n_inside = ((boxes[..., 1] - boxes[..., 0]) * (boxes[..., 3] - boxes[..., 2])).sum(axis=(1, 2)).tolist()
        base = self.proposals._base(device)
        anchors, inside_idx, n_dev = ops.rpn_inside_anchors(base, featmap_sizes, ag.strides, torch.from_numpy(boxes).to(device))
        N = anchors.shape[1]
        gt_inds = torch.full((B, N), -1, dtype=torch.int64, device=device)
        max_ov = torch.empty((B, N), dtype=torch.float32, device=device)
        asg = self.assigner
        for b in range(B):
            n = n_inside[b]
            if n == 0:
                continue
            ign = gt_bboxes_ignore[b] if gt_bboxes_ignore is not None else None
            ign = ign[:, :4].float().contiguous() if ign is not None and ign.numel() > 0 else None
            ops.max_iou_assign(anchors[b, :n], gt_bboxes[b][:, :4].float().contiguous(), None, ign, asg.pos_iou_thr, asg.neg_iou_thr,
                               asg.min_pos_iou, asg.gt_max_assign_all, asg.ignore_iof_thr, asg.ignore_wrt_candidates,
                               asg.match_low_quality, out=(gt_inds[b, :n], max_ov[b, :n]))
        rank, counts = ops.rpn_candidate_ranks(gt_inds, n_dev)
        counts = [tuple(c) for c in counts.cpu().tolist()]            # the batch's one device-to-host copy
        plan = random_sample_plan(counts, **self.sampler_cfg)
        if min(n_inside) == 0:
            return None
        gt_cat = torch.cat([g[:, :4].float() for g in gt_bboxes]).contiguous() if B else None
        gt_off = torch.tensor(np.concatenate([[0], np.cumsum([len(g) for g in gt_bboxes])]), dtype=torch.int32).to(device)
        labels, lw, bt, bw = ops.rpn_anchor_targets(featmap_sizes, ag.strides, A, inside_idx, anchors, gt_inds, rank,
                                                    upload_sample_plan(plan, device), gt_cat, gt_off, self.means, self.stds,
                                                    self.train_cfg.get('pos_weight', -1))
        ns = sampled_counts(plan, counts)
        cls_off = np.concatenate([[0], np.cumsum([B * h * w * A for h, w in featmap_sizes])]).tolist()
        return RPNTargets(B=B, A=A, featmap_sizes=[tuple(s) for s in featmap_sizes], labels=labels, label_weights=lw, bbox_targets=bt,
                          bbox_weights=bw, cls_off=cls_off, n_inside=n_inside, gt_inds=gt_inds, rank=rank, plan=plan, counts=counts,
                          num_total_samples=sum(max(p, 1) for p, _ in ns) + sum(max(q, 1) for _, q in ns),
                          bbox_loss=self.bbox_loss_kind, beta=self.bbox_beta)

    def loss(self, cls_scores, bbox_preds, gt_bboxes, img_metas, gt_bboxes_ignore=None):
        """dict(loss_rpn_cls=[L], loss_rpn_bbox=[L]) as rpn_head.py:44-75, or None when an image has no inside anchor"""
        featmap_sizes = [tuple(int(v) for v in c.shape[-2:]) for c in cls_scores]
        if not cls_scores[0].is_cuda:
            raise RuntimeError('RPNHead.loss runs on CUDA tensors only; there is no CPU fallback')
        tg = self.get_targets(featmap_sizes, gt_bboxes, img_metas, gt_bboxes_ignore, device=cls_scores[0].device)
        if tg is None:
            return None
        maps = [c.float().contiguous() for c in cls_scores] + [r.float().contiguous() for r in bbox_preds]
        sums = _RPNLevelSums.apply(tg, *maps)
        avg = float(tg.num_total_samples)
        cls = sums[:, 0] / avg * self.cls_loss_weight
        box = sums[:, 1] / avg * self.bbox_loss_weight
        return dict(loss_rpn_cls=list(cls.unbind(0)), loss_rpn_bbox=list(box.unbind(0)))

    def forward_train(self, x, img_metas, gt_bboxes, gt_labels=None, gt_bboxes_ignore=None, proposal_cfg=None, **kwargs):
        """base_dense_head.py:22-59"""
        outs = self(x)
        if gt_labels is None:
            losses = self.loss(*outs, gt_bboxes, img_metas, gt_bboxes_ignore=gt_bboxes_ignore)
        else:
            losses = self.loss(*outs, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=gt_bboxes_ignore)
        if proposal_cfg is None:
            return losses
        return losses, self.get_bboxes(*outs, img_metas, cfg=proposal_cfg)

    def get_bboxes(self, cls_scores, bbox_preds, img_metas, cfg=None, rescale=False, with_nms=True):
        return self.proposals.get_bboxes(cls_scores, bbox_preds, img_metas, cfg=cfg, rescale=rescale, with_nms=with_nms)

    def simple_test_rpn(self, x, img_metas):
        """RPNTestMixin.simple_test_rpn (dense_test_mixins.py:109-124), what TwoStageDetector.simple_test calls: proposals per image"""
        return self.get_bboxes(*self(x), img_metas)

    def aug_test_rpn(self, feats, img_metas):
        """RPNTestMixin.aug_test_rpn (dense_test_mixins.py:126-160) merges the augmentations with merge_aug_proposals, which is not built"""
        raise NotImplementedError('RPNHead.aug_test_rpn (test-time augmentation of the RPN: merge_aug_proposals) is not implemented')
