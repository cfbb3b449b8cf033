"""The second stage of the two-stage detector (BASELINE.json configs[3], the TinyPerson Faster R-CNN): the bbox branch of
StandardRoIHead (mmdet/models/roi_heads/standard_roi_head.py) with SingleRoIExtractor (roi_extractors/single_level_roi_extractor.py,
mmcv RoIAlign(aligned=True, pool_mode='avg')) and Shared2FCBBoxHead (bbox_heads/convfc_bbox_head.py:193-205, bbox_head.py), with the
reference's constructor keywords, parameter names and method signatures.

  * SingleRoIExtractor   one ptb_roi_align_fwd launch over every RoI of the batch and every level (each RoI mapped to its level on the
                         device), reading the FPN maps channels-last; backward ptb_roi_align_bwd.
  * Shared2FCBBoxHead    shared_fcs.0 / shared_fcs.1 / fc_cls / fc_reg stay nn.Linear under autograd (the reference's arithmetic);
                         `loss` runs CrossEntropyLoss(use_sigmoid=False) on ptb_softmax_ce_fwd_bwd, L1Loss / SmoothL1Loss on
                         ptb_roi_bbox_loss and the accuracy on ptb_roi_accuracy.
  * StandardRoIHead      forward_train: MaxIoUAssigner (ptb_max_iou_assign per image), RandomSampler over the whole batch (one
                         device-to-host copy of the candidate counts, the reference's randperm draws on the host, one upload of the
                         plan) and the targets of every sampled RoI in one ptb_roi_targets launch.  simple_test: the reference's padded
                         batch, ptb_roi_decode and one batched multiclass NMS call.
There is no CPU path: CUDA tensors only."""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .assigners import MaxIoUAssigner, random_sample_plan, sampled_counts, upload_sample_plan
from .post_processing import check_kept, check_split_thr, keep_limit, parse_nms_cfg, run_multiclass_nms
from .registry import CfgNode
from .results import bbox2result


def _pair(v):
    return (int(v), int(v)) if isinstance(v, int) else tuple(int(t) for t in v)


class _RoIAlignLevels(torch.autograd.Function):
    """features (R, C, out, out) of the RoIs on their levels; backward: the gradient of every level's map (0 where no RoI reads)."""

    @staticmethod
    def forward(ctx, ext, rois, *feats):
        maps = [ops.to_nhwc(f.detach().float()) for f in feats]
        y, levels = ops.roi_align_fwd(maps, ext.featmap_strides, rois, ext.out_size, ext.sampling_ratio, ext.finest_scale)
        ext.last_levels = levels
        ctx.ext, ctx.shapes, ctx.dtypes = ext, [tuple(m.shape) for m in maps], [f.dtype for f in feats]
        ctx.save_for_backward(rois, levels)
        return y

    @staticmethod
    def backward(ctx, gy):
        rois, levels = ctx.saved_tensors
        ext = ctx.ext
        grads = ops.roi_align_bwd(gy.float().contiguous(), ctx.shapes, ext.featmap_strides, rois, levels, ext.sampling_ratio)
        return (None, None, *[g.permute(0, 3, 1, 2).to(dt) for g, dt in zip(grads, ctx.dtypes)])


class SingleRoIExtractor(nn.Module):
    """single_level_roi_extractor.py with base_roi_extractor.py: same constructor keywords, `num_inputs`, `forward(feats, rois)`.
    RoIAlign only, with mmcv's defaults aligned=True and pool_mode='avg'.  `last_levels` holds the level of each RoI of the last call
    (-1 for a RoI whose scale is NaN, which keeps zero features as in the reference)."""

    def __init__(self, roi_layer, out_channels, featmap_strides, finest_scale=56, init_cfg=None):
        super().__init__()
        rl = dict(roi_layer)
        t = rl.pop('type', None)
        if t != 'RoIAlign':
            raise NotImplementedError(f'SingleRoIExtractor roi_layer {t}: RoIAlign is implemented')
        if rl.pop('pool_mode', 'avg') != 'avg':
            raise NotImplementedError("RoIAlign(pool_mode='max'): pool_mode='avg' is implemented")
        if not rl.pop('aligned', True):
            raise NotImplementedError('RoIAlign(aligned=False): aligned=True is implemented')
        if rl.pop('use_torchvision', False):
            raise NotImplementedError('RoIAlign(use_torchvision=True)')
        oh, ow = _pair(rl.pop('output_size'))
        if oh != ow:
            raise NotImplementedError(f'RoIAlign output_size {(oh, ow)}: square outputs are implemented')
        self.out_size, self.sampling_ratio = oh, int(rl.pop('sampling_ratio', 0))
        if rl:
            raise TypeError(f'RoIAlign: unexpected arguments {sorted(rl)}')
        if not 1 <= len(featmap_strides) <= ops.ROI_MAX_LEVELS:
            raise NotImplementedError(f'SingleRoIExtractor over {len(featmap_strides)} levels: 1 to {ops.ROI_MAX_LEVELS} are implemented')
        if out_channels % 4:
            raise NotImplementedError(f'SingleRoIExtractor out_channels={out_channels}: a multiple of 4 is implemented')
        self.out_channels, self.featmap_strides, self.finest_scale = out_channels, list(featmap_strides), finest_scale
        self.init_cfg = init_cfg
        self.last_levels = None

    @property
    def num_inputs(self):
        return len(self.featmap_strides)

    def forward(self, feats, rois, roi_scale_factor=None):
        if roi_scale_factor is not None:
            raise NotImplementedError('SingleRoIExtractor roi_scale_factor (RoI rescaling)')
        if len(feats) != self.num_inputs:
            raise ValueError(f'{len(feats)} feature maps for {self.num_inputs} strides')
        if not feats[0].is_cuda:
            raise RuntimeError('SingleRoIExtractor runs on CUDA tensors only; there is no CPU fallback')
        if feats[0].shape[1] != self.out_channels:
            raise ValueError(f'feature maps have {feats[0].shape[1]} channels, out_channels is {self.out_channels}')
        return _RoIAlignLevels.apply(self, rois.detach().float().contiguous(), *feats)


def _delta_coder(bbox_coder):
    bc = dict(bbox_coder)
    if bc.pop('type', 'DeltaXYWHBBoxCoder') != 'DeltaXYWHBBoxCoder':
        raise NotImplementedError('only DeltaXYWHBBoxCoder is implemented')
    if bc.get('add_ctr_clamp', False) or not bc.get('clip_border', True):
        raise NotImplementedError('DeltaXYWHBBoxCoder(add_ctr_clamp=True / clip_border=False)')
    return tuple(float(v) for v in bc.get('target_means', (0., 0., 0., 0.))), \
        tuple(float(v) for v in bc.get('target_stds', (1., 1., 1., 1.)))


class _RoILossSums(torch.autograd.Function):
    """(2,) un-normalised sums: the weighted softmax cross-entropy over every row, the box loss over the positive rows."""

    @staticmethod
    def forward(ctx, head, tg, cls_score, bbox_pred):
        labels, lw, bt, bw = tg
        ctx.head, ctx.tg = head, tg
        ctx.save_for_backward(cls_score, bbox_pred)
        c = ops.softmax_ce(cls_score, labels, lw, head._class_weight(cls_score.device))
        b = ops.roi_bbox_loss(bbox_pred, labels, bt, bw, head.num_classes, head.reg_class_agnostic, head.bbox_loss_kind, head.bbox_beta)
        return torch.cat([c, b])

    @staticmethod
    def backward(ctx, g):
        cls_score, bbox_pred = ctx.saved_tensors
        labels, lw, bt, bw = ctx.tg
        head = ctx.head
        g = g.float().contiguous()
        gc = ops.softmax_ce(cls_score, labels, lw, head._class_weight(cls_score.device), scale=g[0:1], want_grad=True)
        gb = ops.roi_bbox_loss(bbox_pred, labels, bt, bw, head.num_classes, head.reg_class_agnostic, head.bbox_loss_kind, head.bbox_beta,
                               scale=g[1:2], want_grad=True)
        return None, None, gc, gb


class Shared2FCBBoxHead(nn.Module):
    """Shared2FCBBoxHead = ConvFCBBoxHead(num_shared_fcs=2) over BBoxHead: same constructor keywords and parameter names
    (shared_fcs.0, shared_fcs.1, fc_cls, fc_reg), the reference init (Xavier-uniform shared FCs, fc_cls Normal(0.01), fc_reg
    Normal(0.001), biases 0), `forward`, `get_targets`-free `loss` and DeltaXYWHBBoxCoder decoding (in StandardRoIHead.simple_test)."""

    def __init__(self, fc_out_channels=1024, conv_out_channels=256, conv_cfg=None, norm_cfg=None, init_cfg=None, with_avg_pool=False,
                 with_cls=True, with_reg=True, roi_feat_size=7, in_channels=256, num_classes=80,
                 bbox_coder=dict(type='DeltaXYWHBBoxCoder', clip_border=True, target_means=[0., 0., 0., 0.],
                                 target_stds=[0.1, 0.1, 0.2, 0.2]),
                 reg_class_agnostic=False, reg_decoded_bbox=False, reg_predictor_cfg=dict(type='Linear'),
                 cls_predictor_cfg=dict(type='Linear'), loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0)):
        super().__init__()
        if with_avg_pool:
            raise NotImplementedError('Shared2FCBBoxHead(with_avg_pool=True)')
        if not (with_cls and with_reg):
            raise NotImplementedError('Shared2FCBBoxHead without the cls or the reg branch')
        if reg_decoded_bbox:
            raise NotImplementedError('Shared2FCBBoxHead(reg_decoded_bbox=True)')
        for name, c in (('reg_predictor_cfg', reg_predictor_cfg), ('cls_predictor_cfg', cls_predictor_cfg)):
            if dict(c).get('type', 'Linear') != 'Linear':
                raise NotImplementedError(f"{name} type {dict(c).get('type')}: Linear is implemented")
        lc, lb = dict(loss_cls), dict(loss_bbox)
        if lc.get('type') != 'CrossEntropyLoss':
            raise NotImplementedError(f"Shared2FCBBoxHead loss_cls {lc.get('type')}: CrossEntropyLoss(use_sigmoid=False) is implemented")
        if lc.get('use_sigmoid', False):
            raise NotImplementedError('sigmoid classification in the box head (CrossEntropyLoss(use_sigmoid=True))')
        if lc.get('use_mask', False) or lc.get('reduction', 'mean') != 'mean':
            raise NotImplementedError("CrossEntropyLoss with use_mask or a reduction other than 'mean'")
        tb = lb.get('type')
        if tb not in ('L1Loss', 'SmoothL1Loss'):
            raise NotImplementedError(f'Shared2FCBBoxHead loss_bbox {tb}: L1Loss and SmoothL1Loss are implemented')
        if lb.get('reduction', 'mean') != 'mean':
            raise NotImplementedError(f"{tb} with reduction {lb.get('reduction')!r}: 'mean' is implemented")
        self.fc_out_channels, self.conv_out_channels = fc_out_channels, conv_out_channels
        self.roi_feat_size = _pair(roi_feat_size)
        self.roi_feat_area = self.roi_feat_size[0] * self.roi_feat_size[1]
        self.in_channels, self.num_classes = in_channels, num_classes
        self.reg_class_agnostic, self.reg_decoded_bbox = bool(reg_class_agnostic), False
        self.means, self.stds = _delta_coder(bbox_coder)
        self.cls_loss_weight = float(lc.get('loss_weight', 1.0))
        cw = lc.get('class_weight')
        if cw is not None and len(cw) != num_classes + 1:
            raise ValueError(f'CrossEntropyLoss class_weight has {len(cw)} entries for {num_classes + 1} classes')
        self.class_weight = None if cw is None else [float(v) for v in cw]
        self._cw_dev = {}
        self.bbox_loss_kind = ops.RPN_LOSS_L1 if tb == 'L1Loss' else ops.RPN_LOSS_SMOOTH_L1
        self.bbox_beta = float(lb.get('beta', 1.0)) if tb == 'SmoothL1Loss' else 0.0
        if tb == 'SmoothL1Loss' and not self.bbox_beta > 0:
            raise ValueError(f'SmoothL1Loss beta must be > 0, got {self.bbox_beta}')
        self.bbox_loss_weight = float(lb.get('loss_weight', 1.0))
        self.init_cfg = init_cfg
        # the reference's registration order (BBoxHead makes fc_cls / fc_reg before ConvFCBBoxHead makes shared_fcs): optimizer state
        # saved with a reference checkpoint is indexed by parameter position
        self.fc_cls = nn.Linear(fc_out_channels, num_classes + 1)
        self.fc_reg = nn.Linear(fc_out_channels, 4 if reg_class_agnostic else 4 * num_classes)
        self.shared_fcs = nn.ModuleList([nn.Linear(in_channels * self.roi_feat_area, fc_out_channels),
                                         nn.Linear(fc_out_channels, fc_out_channels)])
        self.relu = nn.ReLU(inplace=True)
        self.init_weights()

    def init_weights(self):
        for fc in self.shared_fcs:
            nn.init.xavier_uniform_(fc.weight)
            nn.init.constant_(fc.bias, 0.0)
        nn.init.normal_(self.fc_cls.weight, 0.0, 0.01)
        nn.init.constant_(self.fc_cls.bias, 0.0)
        nn.init.normal_(self.fc_reg.weight, 0.0, 0.001)
        nn.init.constant_(self.fc_reg.bias, 0.0)

    def _class_weight(self, device):
        if self.class_weight is None:
            return None
        if device not in self._cw_dev:
            self._cw_dev[device] = torch.tensor(self.class_weight, dtype=torch.float32).to(device)
        return self._cw_dev[device]

    def forward(self, x):
        x = x.flatten(1)
        for fc in self.shared_fcs:
            x = self.relu(fc(x))
        return self.fc_cls(x), self.fc_reg(x)

    def loss(self, cls_score, bbox_pred, rois, labels, label_weights, bbox_targets, bbox_weights, reduction_override=None,
             avg_factor=None):
        """bbox_head.py:261-306: dict(loss_cls, acc, loss_bbox).  avg_factor: #(label_weights > 0) when the caller knows it (one device
        read otherwise, as the reference's .item())."""
        if reduction_override is not None:
            raise NotImplementedError('Shared2FCBBoxHead.loss reduction_override')
        if not cls_score.is_cuda:
            raise RuntimeError('Shared2FCBBoxHead.loss runs on CUDA tensors only; there is no CPU fallback')
        R = cls_score.shape[0]
        if avg_factor is None:
            avg_factor = int((label_weights > 0).sum())
        tg = (labels.contiguous(), label_weights.float().contiguous(), bbox_targets.float().contiguous(), bbox_weights.float().contiguous())
        cs, bp = cls_score.float().contiguous(), bbox_pred.float().contiguous()
        sums = _RoILossSums.apply(self, tg, cs, bp)
        return dict(loss_cls=sums[0] / float(max(avg_factor, 1)) * self.cls_loss_weight,
                    acc=ops.roi_accuracy(cs.detach(), tg[0]),
                    loss_bbox=sums[1] / float(R) * self.bbox_loss_weight)


class StandardRoIHead(nn.Module):
    """standard_roi_head.py over base_roi_head.py, bbox branch only: same constructor keywords, `forward_train` (returns
    dict(loss_cls, loss_bbox, acc)), `simple_test` (per image the bbox2result lists), `_bbox_forward`.  Refused with
    NotImplementedError: a mask branch, a shared head, other extractors and bbox heads, samplers other than RandomSampler,
    and `aug_test` under test_cfg do_tile_as_aug=True.  `aug_test` / `aug_test_bboxes` run the reference's test-time augmentation for
    one image; pointtinybenchmark_b200.tile_test.tile_aug_test runs the detector's tile testing."""

    def __init__(self, bbox_roi_extractor=None, bbox_head=None, mask_roi_extractor=None, mask_head=None, shared_head=None,
                 train_cfg=None, test_cfg=None, pretrained=None, init_cfg=None):
        super().__init__()
        if mask_head is not None or mask_roi_extractor is not None:
            raise NotImplementedError('StandardRoIHead mask branch (mask_head / mask_roi_extractor)')
        if shared_head is not None:
            raise NotImplementedError('StandardRoIHead shared_head')
        if bbox_head is None or bbox_roi_extractor is None:
            raise NotImplementedError('StandardRoIHead without a bbox branch')
        ex, bh = dict(bbox_roi_extractor), dict(bbox_head)
        t = ex.pop('type', None)
        if t != 'SingleRoIExtractor':
            raise NotImplementedError(f'RoI extractor {t}: SingleRoIExtractor is implemented')
        t = bh.pop('type', None)
        if t != 'Shared2FCBBoxHead':
            raise NotImplementedError(f'bbox head {t}: Shared2FCBBoxHead is implemented')
        self.bbox_roi_extractor = SingleRoIExtractor(**ex)
        self.bbox_head = Shared2FCBBoxHead(**bh)
        self.train_cfg = CfgNode(train_cfg) if train_cfg is not None else None
        self.test_cfg = CfgNode(test_cfg) if test_cfg is not None else None
        self.init_cfg = init_cfg
        self.bbox_assigner = self.bbox_sampler = None
        if self.train_cfg is not None:
            asg = dict(self.train_cfg.get('assigner') or {})
            t = asg.pop('type', None)
            if t != 'MaxIoUAssigner':
                raise NotImplementedError(f'StandardRoIHead assigner {t}: MaxIoUAssigner is implemented')
            self.bbox_assigner = MaxIoUAssigner(**asg)
            smp = dict(self.train_cfg.get('sampler') or {})
            t = smp.pop('type', None)
            if t != 'RandomSampler':
                raise NotImplementedError(f'StandardRoIHead sampler {t}: RandomSampler is implemented')
            self.sampler_cfg = dict(num=smp['num'], pos_fraction=smp['pos_fraction'], neg_pos_ub=smp.get('neg_pos_ub', -1))
            self.sampler_add_gt = bool(smp.get('add_gt_as_proposals', True))
        self.last_sampling = None

    with_bbox = property(lambda self: True)
    with_mask = property(lambda self: False)
    with_shared_head = property(lambda self: False)

    def _bbox_forward(self, x, rois):
        bbox_feats = self.bbox_roi_extractor(x[:self.bbox_roi_extractor.num_inputs], rois)
        cls_score, bbox_pred = self.bbox_head(bbox_feats)
        return dict(cls_score=cls_score, bbox_pred=bbox_pred, bbox_feats=bbox_feats)

    def get_targets(self, proposal_list, gt_bboxes, gt_labels, gt_bboxes_ignore=None):
        """assign + sample + BBoxHead.get_targets for the batch: rois (R, 5), labels, label_weights, bbox_targets, bbox_weights in the
        reference's row order, and the sampled counts per image.  One device-to-host copy (the candidate counts)."""
        if self.train_cfg is None:
            raise RuntimeError('StandardRoIHead.forward_train needs train_cfg')
        B = len(proposal_list)
        dev = proposal_list[0].device
        n_gt = [int(g.shape[0]) for g in gt_bboxes]
        g0 = [n if self.sampler_add_gt else 0 for n in n_gt]
        n_prop = [int(p.shape[0]) for p in proposal_list]
        n_cand = [a + b for a, b in zip(g0, n_prop)]
        N = max(max(n_cand), 1)
        cand = torch.zeros((B, N, 4), dtype=torch.float32, device=dev)
        gt_inds = torch.full((B, N), -1, dtype=torch.int64, device=dev)
        max_ov = torch.empty((B, N), dtype=torch.float32, device=dev)
        ones = torch.arange(1, max(n_gt + [1]) + 1, dtype=torch.int64, device=dev)
        gts = [g[:, :4].float().contiguous() for g in gt_bboxes]
        asg = self.bbox_assigner
        for b in range(B):
            if g0[b]:                                          # RandomSampler add_gt_as_proposals: GTs first, assigned to themselves
                cand[b, :g0[b]] = gts[b]
                gt_inds[b, :g0[b]] = ones[:g0[b]]
            if n_prop[b]:
                cand[b, g0[b]:n_cand[b]] = proposal_list[b][:, :4]
                ign = gt_bboxes_ignore[b] if gt_bboxes_ignore is not None else None
                ign = ign[:, :4].float().contiguous() if ign is not None and ign.numel() > 0 else None
                ops.max_iou_assign(cand[b, g0[b]:n_cand[b]], gts[b], None, ign, asg.pos_iou_thr, asg.neg_iou_thr, asg.min_pos_iou,
                                   asg.gt_max_assign_all, asg.ignore_iof_thr, asg.ignore_wrt_candidates, asg.match_low_quality,
                                   out=(gt_inds[b, g0[b]:n_cand[b]], max_ov[b, g0[b]:n_cand[b]]))
        # host-to-device copies go from pinned memory without a stream synchronisation: the counts below are the batch's one sync
        n_cand_dev = torch.tensor(n_cand, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
        rank, counts = ops.rpn_candidate_ranks(gt_inds, n_cand_dev)
        counts = [tuple(c) for c in counts.cpu().tolist()]              # the batch's one device-to-host copy
        plan = random_sample_plan(counts, **self.sampler_cfg)
        ns = sampled_counts(plan, counts)
        row_off, R = [], 0
        for p, q in ns:
            row_off += [R, R + p]
            R += p + q
        gt_off = np.concatenate([[0], np.cumsum(n_gt)]).astype(np.int64).tolist()
        buf = upload_sample_plan(plan, dev, tail=row_off + gt_off)             # the plan, the row offsets and the GT offsets in one copy
        n = buf.numel()
        row_off_dev, gt_off = buf[n - 3 * B - 1:n - B - 1], buf[n - B - 1:]
        gt_cat = torch.cat(gts).contiguous() if sum(n_gt) else torch.zeros((0, 4), dtype=torch.float32, device=dev)
        lab_cat = torch.cat([l.long() for l in gt_labels]).contiguous() if sum(n_gt) else torch.zeros((0,), dtype=torch.int64, device=dev)
        bh = self.bbox_head
        rois, labels, lw, bt, bw = ops.roi_targets(cand, gt_inds, rank, buf, row_off_dev, gt_cat, gt_off, lab_cat,
                                                   bh.num_classes, bh.means, bh.stds, self.train_cfg.get('pos_weight', -1), R)
        self.last_sampling = dict(gt_inds=gt_inds, rank=rank, plan=plan, counts=counts, sampled=ns, n_cand=n_cand)
        return rois, labels, lw, bt, bw, ns

    def forward_train(self, x, img_metas, proposal_list, gt_bboxes, gt_labels, gt_bboxes_ignore=None, gt_masks=None, **kwargs):
        if gt_masks is not None:
            raise NotImplementedError('StandardRoIHead mask branch (gt_masks)')
        if not proposal_list[0].is_cuda:
            raise RuntimeError('StandardRoIHead runs on CUDA tensors only; there is no CPU fallback')
        rois, labels, lw, bt, bw, ns = self.get_targets(proposal_list, gt_bboxes, gt_labels, gt_bboxes_ignore)
        res = self._bbox_forward(x, rois)
        # every sampled row has a positive label weight (pos_weight > 0 or 1, negatives 1): avg_factor is the sample count
        return self.bbox_head.loss(res['cls_score'], res['bbox_pred'], rois, labels, lw, bt, bw, avg_factor=rois.shape[0])

    def _multiclass_nms(self, boxes, scores, cfg):
        """the batched multiclass NMS of (B, P, C, 4) boxes and (B, P, C) scores with the test cfg's nms / max_per_img:
        count (B,), det (B, kmax, 5), label (B, kmax) and keep_limit's (kmax, unlimited)"""
        nms_cfg = cfg.get('nms') or {}
        check_split_thr(nms_cfg)
        nms = parse_nms_cfg(nms_cfg, default_iou=0.5)
        if nms.class_agnostic:
            raise NotImplementedError('RoI head class_agnostic NMS')
        kmax, unlimited = keep_limit(cfg.get('max_per_img', -1))
        cnt, det, lab, _, _ = run_multiclass_nms(boxes, scores, float(cfg.score_thr), nms, kmax)
        return cnt, det, lab, kmax, unlimited

    def simple_test_bboxes(self, x, img_metas, proposals, rcnn_test_cfg, rescale=False):
        """test_mixins.py:57-155: per image (dets (k, 5), labels (k,)) from one decode launch and one batched NMS call"""
        cfg = CfgNode(rcnn_test_cfg)
        B = len(proposals)
        dev = proposals[0].device
        N = max(int(p.shape[0]) for p in proposals)
        # the reference's padding: shorter proposal lists get zero boxes at the FRONT
        rois = torch.zeros((B, N, 5), dtype=torch.float32, device=dev)
        rois[:, :, 0] = torch.arange(B, dtype=torch.float32, device=dev)[:, None]
        for b, p in enumerate(proposals):
            if p.shape[0]:
                rois[b, N - p.shape[0]:, 1:] = p[:, :4]
        rois = rois.view(B * N, 5)
        res = self._bbox_forward(x, rois)
        bh = self.bbox_head
        img_hw = torch.tensor([[float(m['img_shape'][0]), float(m['img_shape'][1])] for m in img_metas], dtype=torch.float32).to(dev)
        sf = None
        if rescale and N > 0:
            sf = torch.tensor(np.stack([np.asarray(m['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32)
                                        for m in img_metas]), dtype=torch.float32).to(dev)
        boxes, scores = ops.roi_decode(rois, res['cls_score'].detach().float().contiguous(), res['bbox_pred'].detach().float().contiguous(), B,
                                       bh.num_classes, bh.reg_class_agnostic, bh.means, bh.stds, abs(np.log(16 / 1000)), img_hw, sf)
        cnt, det, lab, kmax, unlimited = self._multiclass_nms(boxes, scores, cfg)
        cnt = cnt.cpu().tolist()
        check_kept(max(cnt), kmax, unlimited)
        return [det[b, :cnt[b]] for b in range(B)], [lab[b, :cnt[b]].long() for b in range(B)]

    def simple_test(self, x, proposal_list, img_metas, proposals=None, rescale=False):
        """standard_roi_head.py:221-245: per image the bbox2result list (one (k, 5) array per class)"""
        if self.test_cfg is None:
            raise RuntimeError('StandardRoIHead.simple_test needs test_cfg')
        if not proposal_list[0].is_cuda:
            raise RuntimeError('StandardRoIHead runs on CUDA tensors only; there is no CPU fallback')
        det, lab = self.simple_test_bboxes(x, img_metas, list(proposal_list), self.test_cfg, rescale=rescale)
        n = [int(d.shape[0]) for d in det]
        det_h, lab_h = torch.cat(det).cpu().split(n), torch.cat(lab).cpu().split(n)          # one copy for the batch
        return [bbox2result(d, l, self.bbox_head.num_classes) for d, l in zip(det_h, lab_h)]

    def _refuse_tile_as_aug(self, cfg):
        if CfgNode(cfg or {}).get('do_tile_as_aug', False):
            raise NotImplementedError(
                'StandardRoIHead.aug_test with test_cfg do_tile_as_aug=True: the detector then feeds every tile of an image as an aug of '
                "one aug_test call, and the reference's bbox_mapping keeps different proposals per tile, so merge_aug_bboxes' torch.stack "
                'fails for any image of more than one tile; use do_tile_as_aug=False (tile_aug_test, pointtinybenchmark_b200.tile_test)')

    def shape_batches(self, feats):
        """the position of every aug among the augs of its FPN shape (its RoI batch index in that shape's one RoIAlign)"""
        L, seen, out = self.bbox_roi_extractor.num_inputs, {}, []
        for f in feats:
            key = tuple(tuple(m.shape[-2:]) for m in f[:L])
            out.append(seen.get(key, 0))
            seen[key] = out[-1] + 1
        return out

    def aug_forward_merge(self, feats, metas, meta, rois, counts, A):
        """the RoI forward of every aug of T tiles at once and merge_aug_bboxes per tile.  feats: per aug (tile-major, A per tile) its
        level maps (1, C, H, W); metas: per aug its meta dict; rois (T*A, N, 5) of ptb_box_map (batch index = position of the aug in its
        FPN-shape group), counts (T,) int32 rows per tile or None.  returns boxes (T, N, C, 4) and scores (T, N, C), -inf past the count."""
        G, N = rois.shape[:2]
        dev = rois.device
        L = self.bbox_roi_extractor.num_inputs
        groups = {}
        for g, f in enumerate(feats):
            groups.setdefault(tuple(tuple(m.shape[-2:]) for m in f[:L]), []).append(g)
        order = [g for gs in groups.values() for g in gs]
        parts = []
        for gs in groups.values():                    # augs at other scales have other map sizes: one RoIAlign per shape group
            x = [torch.cat([feats[g][l] for g in gs]) for l in range(L)]
            r = rois if len(groups) == 1 else rois[torch.tensor(gs, device=dev)]
            parts.append(self.bbox_roi_extractor(x, r.reshape(-1, 5)))
        bbox_feats = parts[0] if len(parts) == 1 else torch.cat(parts)
        cls_score, bbox_pred = self.bbox_head(bbox_feats)
        if len(groups) > 1:                           # back to aug order
            inv = torch.empty(G, dtype=torch.int64)
            inv[torch.tensor(order)] = torch.arange(G)
            rows = (inv.to(dev)[:, None] * N + torch.arange(N, device=dev)[None]).reshape(-1)
            cls_score, bbox_pred = cls_score[rows], bbox_pred[rows]
        bh = self.bbox_head
        img_hw = torch.tensor([[float(m['img_shape'][0]), float(m['img_shape'][1])] for m in metas], dtype=torch.float32)
        boxes, scores = ops.roi_decode(rois.reshape(-1, 5).contiguous(), cls_score.detach().float().contiguous(),
                                       bbox_pred.detach().float().contiguous(), G, bh.num_classes, bh.reg_class_agnostic, bh.means, bh.stds,
                                       abs(np.log(16 / 1000)), img_hw.to(dev, non_blocking=True), None)
        return ops.aug_merge(boxes, scores, counts, meta, A, 4 if bh.reg_class_agnostic else 4 * bh.num_classes)

    def aug_test_bboxes(self, feats, img_metas, proposal_list, rcnn_test_cfg):
        """test_mixins.py:157-189 for one image: bbox_mapping of the proposals into every aug, one RoI forward over the augs,
        merge_aug_bboxes (mean over the augs) and multiclass_nms.  returns (det_bboxes (k, 5), det_labels (k,))."""
        self._refuse_tile_as_aug(rcnn_test_cfg if rcnn_test_cfg is not None else self.test_cfg)
        cfg = CfgNode(rcnn_test_cfg)
        metas = [m[0] for m in img_metas]
        A = len(feats)
        prop = proposal_list[0][:, :4].float().contiguous()
        dev = prop.device
        if not prop.is_cuda:
            raise RuntimeError('StandardRoIHead runs on CUDA tensors only; there is no CPU fallback')
        meta = ops.aug_meta(metas, [0] * A, self.shape_batches(feats), dev)
        n = prop.shape[0]
        if any(m.get('tile_offset') is not None for m in metas):
            rois, keep = ops.box_map(prop[None], None, meta, want_keep=True)
            kept = keep.sum(1).cpu().tolist()
            if len(set(kept)) > 1:               # merge_aug_bboxes' torch.stack of the augs' box sets
                raise RuntimeError(f'stack expects each tensor to be equal size: the tile offsets keep {kept} proposals per aug')
            n = kept[0]
            rois = rois[keep].view(A, n, 5)
        else:
            rois = ops.box_map(prop[None], None, meta)
        if n == 0:                                # the reference forwards no RoI and multiclass_nms returns nothing
            return torch.zeros((0, 5), dtype=torch.float32, device=dev), torch.zeros((0,), dtype=torch.long, device=dev)
        boxes, scores = self.aug_forward_merge(feats, metas, meta, rois, None, A)
        cnt, det, lab, kmax, unlimited = self._multiclass_nms(boxes, scores, cfg)
        c = int(cnt[0])
        check_kept(c, kmax, unlimited)
        return det[0, :c], lab[0, :c].long()

    def aug_test(self, x, proposal_list, img_metas, rescale=False):
        """standard_roi_head.py:246-270: [bbox_results] of one image; without rescale the boxes are multiplied by the first aug's
        scale_factor"""
        self._refuse_tile_as_aug(self.test_cfg)
        det, lab = self.aug_test_bboxes(x, img_metas, proposal_list, self.test_cfg)
        if not rescale:
            sf = np.asarray(img_metas[0][0]['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32)
            det = torch.cat([det[:, :4] * torch.from_numpy(sf).to(det.device), det[:, 4:]], 1)
        return [bbox2result(det.cpu(), lab.cpu(), self.bbox_head.num_classes)]
