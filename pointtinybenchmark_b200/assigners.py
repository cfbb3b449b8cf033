"""MaxIoUAssigner — host-side mirror of mmdet/core/bbox/assigners/max_iou_assigner.py:9-212 over ptb_max_iou_assign
(SURVEY.md §8f rank 4: the dense-anchor assignment of BASELINE.json configs[3]).  Same ctor kwargs, `assign` signature and result
fields (`num_gts`, `gt_inds`, `max_overlaps`, `labels`) as the reference's AssignResult (assign_result.py:42-46).

Also here: PointAssigner, HungarianAssignerV2 (the P2P point assigner named by BASELINE.json north_star) and PseudoSampler /
SamplingResult mirrors.  `registry.register_core()` registers them into mmdet's BBOX_ASSIGNERS / BBOX_SAMPLERS when mmdet is importable."""
import torch

from . import ops


class AssignResult:
    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels

    @property
    def num_preds(self):
        return len(self.gt_inds)


class MaxIoUAssigner:
    def __init__(self, pos_iou_thr, neg_iou_thr, min_pos_iou=.0, gt_max_assign_all=True, ignore_iof_thr=-1, ignore_wrt_candidates=True,
                 match_low_quality=True, gpu_assign_thr=-1, iou_calculator=None):
        if iou_calculator is not None and dict(iou_calculator).get('type', 'BboxOverlaps2D') != 'BboxOverlaps2D':
            raise NotImplementedError(f'iou_calculator {iou_calculator}')
        if iou_calculator is not None and dict(iou_calculator).get('dtype') == 'fp16':
            raise NotImplementedError('BboxOverlaps2D(dtype=fp16)')
        self.pos_iou_thr, self.neg_iou_thr, self.min_pos_iou = pos_iou_thr, neg_iou_thr, min_pos_iou
        self.gt_max_assign_all, self.ignore_iof_thr, self.ignore_wrt_candidates = gt_max_assign_all, ignore_iof_thr, ignore_wrt_candidates
        self.match_low_quality = match_low_quality
        self.gpu_assign_thr = gpu_assign_thr          # accepted for config compatibility: there is no CPU assignment path here

    def assign(self, bboxes, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None):
        if not bboxes.is_cuda:
            raise RuntimeError('MaxIoUAssigner runs on CUDA tensors only; there is no CPU fallback')
        b = bboxes[:, :4].float().contiguous()
        g = gt_bboxes[:, :4].float().contiguous()
        ign = gt_bboxes_ignore[:, :4].float().contiguous() if gt_bboxes_ignore is not None else None
        gt_inds, max_ov, labels = ops.max_iou_assign(b, g, gt_labels, ign, self.pos_iou_thr, self.neg_iou_thr, self.min_pos_iou,
                                                     self.gt_max_assign_all, self.ignore_iof_thr, self.ignore_wrt_candidates,
                                                     self.match_low_quality)
        if g.shape[0] == 0 and gt_labels is None:
            labels = None
        return AssignResult(g.shape[0], gt_inds, max_ov, labels)


class PointAssigner:
    """mmdet/core/bbox/assigners/point_assigner.py:9-133 over ptb_point_assigner: same ctor kwargs, `assign` signature and result
    (gt_inds: 0 background, i+1 positive; labels: -1 background)."""

    def __init__(self, scale=4, pos_num=3):
        self.scale, self.pos_num = scale, pos_num

    def assign(self, points, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None):
        if not points.is_cuda:
            raise RuntimeError('PointAssigner runs on CUDA tensors only; there is no CPU fallback')
        p = (points.reshape(-1, 3) if points.numel() == 0 else points[:, :3]).float().contiguous()      # the reference's tests pass 1-D empties
        g = (gt_bboxes.reshape(-1, 4) if gt_bboxes.numel() == 0 else gt_bboxes[:, :4]).float().contiguous()
        gt_inds = ops.point_assigner(p, g, self.scale, self.pos_num)
        labels = None
        if gt_labels is not None:
            labels = gt_inds.new_full((p.shape[0],), -1)
            if g.shape[0] > 0:
                pos = gt_inds > 0
                labels = labels.masked_scatter(pos, gt_labels.to(gt_inds.device)[gt_inds[pos] - 1].to(labels.dtype))
        return AssignResult(g.shape[0], gt_inds, None, labels)


class HungarianAssignerV2:
    """mmdet/core/bbox/assigners/hungarian_assigner.py:149-270 for the point setting the reference uses it in (P2PHead: FocalLossCost +
    DisCostV2 on (x, y) points): cost matrix and the <= topk_k matching rounds both on the device (ptb_p2p_cost_matrix,
    ptb_hungarian_v2_batch); `assign` keeps the reference's argument order.  P2PHead.loss uses the batched form directly."""

    def __init__(self, cls_costs=None, reg_costs=None, topk_k=1):
        # the reference's defaults are the DETR costs (ClassificationCost; BBoxL1Cost + IoUCost, hungarian_assigner.py:153-158), which no
        # CPR / P2P config uses: they are rejected below like every other unsupported cost, never silently replaced
        cc = cls_costs if cls_costs is not None else [dict(type='ClassificationCost', weight=1.)]
        rc = reg_costs if reg_costs is not None else [dict(type='BBoxL1Cost', weight=1.0, norm_with_img_size=True),
                                                      dict(type='IoUCost', iou_mode='giou', weight=1.0)]
        cc = cc[0] if isinstance(cc, (list, tuple)) and len(cc) == 1 else cc
        rc = rc[0] if isinstance(rc, (list, tuple)) and len(rc) == 1 else rc
        if not isinstance(cc, dict) or not isinstance(rc, dict) or cc.get('type') != 'FocalLossCost' or rc.get('type') != 'DisCostV2':
            raise NotImplementedError('HungarianAssignerV2: one FocalLossCost + one DisCostV2 (the P2P configs) are implemented')
        if rc.get('p', 1) != 1:
            raise NotImplementedError('DisCostV2 p != 1')
        self.w_cls, self.alpha, self.gamma, self.eps = cc.get('weight', 1.0), cc.get('alpha', 0.25), cc.get('gamma', 2), cc.get('eps', 1e-12)
        self.w_dis, self.norm_wh = rc.get('weight', 1.0), rc.get('norm_with_img_wh', True)
        self.topk_k = topk_k

    def assign(self, bbox_pred, cls_pred, gt_bboxes, gt_labels, img_meta, gt_bboxes_ignore=None, eps=1e-7):
        assert gt_bboxes_ignore is None, 'Only case when gt_bboxes_ignore is None is supported.'
        if not bbox_pred.is_cuda:
            raise RuntimeError('HungarianAssignerV2 runs on CUDA tensors only; there is no CPU fallback')
        if bbox_pred.shape[-1] != 2 or (gt_bboxes.numel() > 0 and gt_bboxes.shape[-1] != 2):
            raise NotImplementedError('HungarianAssignerV2: (x, y) points only (DisCostV2 with k*2 = 2 coordinates, as P2PHead uses it)')
        N, n = bbox_pred.shape[0], gt_bboxes.shape[0]
        dev = bbox_pred.device
        gt_inds = torch.zeros((N,), dtype=torch.long, device=dev)
        labels = torch.full((N,), -1, dtype=torch.long, device=dev)
        if N == 0 or n == 0:                        # hungarian_assigner.py:211-219: no GT -> everything background
            return AssignResult(n, gt_inds, None, labels)
        fx, fy = (img_meta['img_shape'][1], img_meta['img_shape'][0]) if self.norm_wh else (1.0, 1.0)
        cost = ops.p2p_cost_matrix(cls_pred.detach().float().contiguous(), bbox_pred.detach()[:, :2].float().contiguous(), None,
                                   gt_bboxes[:, :2].float().contiguous(), gt_labels.int().contiguous(), self.w_cls, self.alpha, self.gamma,
                                   self.eps, self.w_dis, fx, fy)
        status = ops.hungarian_v2_batch(cost.view(-1), [(N, n)], self.topk_k, gt_inds, [0])
        st = int(status[0])
        if st:
            raise ValueError({1: 'cost matrix is infeasible', 2: 'matrix contains invalid numeric entries'}.get(st, f'hungarian kernel status {st}'))
        pos = gt_inds > 0
        labels = labels.masked_scatter(pos, gt_labels.to(dev)[gt_inds[pos] - 1].to(labels.dtype))
        return AssignResult(n, gt_inds, None, labels)


class SamplingResult:
    """mmdet/core/bbox/samplers/sampling_result.py:25-53 (the fields P2PHead._get_target_single reads)."""

    def __init__(self, pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags):
        self.pos_inds, self.neg_inds = pos_inds, neg_inds
        self.pos_bboxes, self.neg_bboxes = bboxes[pos_inds], bboxes[neg_inds]
        self.pos_is_gt = gt_flags[pos_inds]
        self.num_gts = gt_bboxes.shape[0]
        self.pos_assigned_gt_inds = assign_result.gt_inds[pos_inds] - 1
        if gt_bboxes.numel() == 0:
            assert self.pos_assigned_gt_inds.numel() == 0
            self.pos_gt_bboxes = torch.empty_like(gt_bboxes).view(-1, gt_bboxes.shape[-1] if gt_bboxes.dim() > 1 else 4)
        else:
            self.pos_gt_bboxes = gt_bboxes[self.pos_assigned_gt_inds, :]
        self.pos_gt_labels = assign_result.labels[pos_inds] if assign_result.labels is not None else None

    @property
    def bboxes(self):
        return torch.cat([self.pos_bboxes, self.neg_bboxes])


class PseudoSampler:
    """mmdet/core/bbox/samplers/pseudo_sampler.py:9-41: every assigned proposal is a sample."""

    def __init__(self, **kwargs):
        pass

    def sample(self, assign_result, bboxes, gt_bboxes, **kwargs):
        pos_inds = torch.nonzero(assign_result.gt_inds > 0, as_tuple=False).squeeze(-1).unique()
        neg_inds = torch.nonzero(assign_result.gt_inds == 0, as_tuple=False).squeeze(-1).unique()
        gt_flags = bboxes.new_zeros(bboxes.shape[0], dtype=torch.uint8)
        return SamplingResult(pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags)
