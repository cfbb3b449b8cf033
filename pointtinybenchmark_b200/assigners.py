"""MaxIoUAssigner — host-side mirror of mmdet/core/bbox/assigners/max_iou_assigner.py:9-212 over ptb_max_iou_assign
(SURVEY.md §8f rank 4: the dense-anchor assignment of BASELINE.json configs[3]).  Same ctor kwargs, `assign` signature and result
fields (`num_gts`, `gt_inds`, `max_overlaps`, `labels`) as the reference's AssignResult (assign_result.py:42-46).

Also here: PointAssigner, HungarianAssignerV2 (the P2P point assigner named by BASELINE.json north_star), PseudoSampler /
SamplingResult mirrors and RandomSampler with its host draw plan.  `registry.register_core()` registers them into mmdet's BBOX_ASSIGNERS / BBOX_SAMPLERS when mmdet is importable."""
import torch

from . import _lib, ops


class AssignResult:
    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels

    @property
    def num_preds(self):
        return len(self.gt_inds)

    def add_gt_(self, gt_labels):
        """assign_result.py:190-204: the GT boxes prepended as proposals assigned to themselves."""
        self_inds = torch.arange(1, len(gt_labels) + 1, dtype=torch.long, device=gt_labels.device)
        self.gt_inds = torch.cat([self_inds, self.gt_inds])
        if self.max_overlaps is not None:
            self.max_overlaps = torch.cat([self.max_overlaps.new_ones(len(gt_labels)), self.max_overlaps])
        if self.labels is not None:
            self.labels = torch.cat([gt_labels, self.labels])


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


MAX_MATCH_COST_TERMS = _lib.DEFINES['PTB_MAX_MATCH_COST_TERMS']        # per list
_BOX_COSTS = ('BBoxL1Cost', 'IoUCost', 'IoUCostV2')


def match_cost_terms(cls_costs, reg_costs):
    """HungarianAssignerV2's cls_costs / reg_costs (a dict or a list of dicts each, hungarian_assigner.py:160-163) -> the ordered term
    list of ops.p2p_cost_matrix_terms: the classification terms, then the DisCostV2 terms, each in config order.  Raises
    NotImplementedError, naming the type, for every cost this matching does not compute."""
    def as_list(c):
        return list(c) if isinstance(c, (list, tuple)) else [c]

    def common(c, t):
        if t == 'ClassificationCost':
            raise NotImplementedError('ClassificationCost is not implemented: it computes -softmax(x)[:, label] * weight, which '
                                      "ClassificationCostV2(use_sigmoid=False) computes; use that")
        if t in _BOX_COSTS:
            raise NotImplementedError(f'{t} is a box cost; the point matching takes FocalLossCost, ClassificationCostV2, ZeroCost '
                                      'and DisCostV2')
        raise NotImplementedError(f'match cost {t}')

    terms = []
    cls_l, reg_l = as_list(cls_costs), as_list(reg_costs)
    for name, lst in (('cls_costs', cls_l), ('reg_costs', reg_l)):
        if len(lst) > MAX_MATCH_COST_TERMS:
            raise NotImplementedError(f'{name}: {len(lst)} costs; at most {MAX_MATCH_COST_TERMS} per list are implemented')
    for c in cls_l:
        c = dict(c)
        t = c.get('type')
        w = c.get('weight', 1.0)
        if t == 'FocalLossCost':
            terms.append(dict(kind=t, weight=w, alpha=c.get('alpha', 0.25), gamma=c.get('gamma', 2), eps=c.get('eps', 1e-12)))
        elif t == 'ClassificationCostV2':
            terms.append(dict(kind='ClassificationCostV2_sigmoid' if c.get('use_sigmoid', False) else 'ClassificationCostV2_softmax',
                              weight=w))
        elif t == 'ZeroCost':
            terms.append(dict(kind=t, weight=0.0))
        elif t == 'DisCostV2':
            raise NotImplementedError('DisCostV2 as a classification cost: the reference calls cls_costs with (cls_pred, gt_labels)')
        else:
            common(c, t)
    for c in reg_l:
        c = dict(c)
        t = c.get('type')
        if t == 'DisCostV2':
            p = c.get('p', 1)
            if p not in (1, 2):
                raise NotImplementedError(f'DisCostV2 p={p}: p = 1 and p = 2 are implemented')
            terms.append(dict(kind=t, weight=c.get('weight', 1.0), p=int(p), norm_with_img_wh=bool(c.get('norm_with_img_wh', True))))
        elif t == 'ZeroCost':
            raise NotImplementedError('ZeroCost as a regression cost: the reference calls reg_costs with three arguments and '
                                      'ZeroCost takes two (TypeError)')
        elif t in ('FocalLossCost', 'ClassificationCostV2'):
            raise NotImplementedError(f'{t} as a regression cost: the reference calls reg_costs with (bbox_pred, gt_bboxes, img_meta)')
        else:
            common(c, t)
    if not terms:
        raise NotImplementedError('HungarianAssignerV2: no match costs')
    return terms


def is_focal_l1_pair(terms):
    """the shipped pair, one FocalLossCost + one DisCostV2(p=1), which ops.p2p_cost_matrix computes"""
    return len(terms) == 2 and terms[0]['kind'] == 'FocalLossCost' and terms[1]['kind'] == 'DisCostV2' and terms[1]['p'] == 1


def cost_matrix(cls, pts, row_idx, gts, gt_labels, terms, img_shape, out=None):
    """the matching's cost matrix for one image on the device: the shipped pair through ops.p2p_cost_matrix, every other term list
    through ops.p2p_cost_matrix_terms.  img_shape: (h, w, ...) of img_meta, read only when a DisCostV2 has norm_with_img_wh."""
    norm = any(t.get('norm_with_img_wh', False) for t in terms)
    fx, fy = (float(img_shape[1]), float(img_shape[0])) if norm else (1.0, 1.0)
    if is_focal_l1_pair(terms):
        fc, dc = terms
        return ops.p2p_cost_matrix(cls, pts, row_idx, gts, gt_labels, fc['weight'], fc['alpha'], fc['gamma'], fc['eps'], dc['weight'],
                                   fx, fy, out=out)
    return ops.p2p_cost_matrix_terms(cls, pts, row_idx, gts, gt_labels, terms, fx, fy, out=out)


class HungarianAssignerV2:
    """mmdet/core/bbox/assigners/hungarian_assigner.py:149-270 for the point setting the reference uses it in (P2PHead: cost lists of
    FocalLossCost, ClassificationCostV2, ZeroCost and DisCostV2(p=1 or 2) on (x, y) points): cost matrix and the <= topk_k matching
    rounds both on the device (ptb_p2p_cost_matrix or ptb_p2p_cost_matrix_terms, ptb_hungarian_v2_batch); `assign` keeps the
    reference's argument order.  P2PHead.loss uses the batched form directly."""

    def __init__(self, cls_costs=None, reg_costs=None, topk_k=1):
        # the reference's defaults are the DETR costs (ClassificationCost; BBoxL1Cost + IoUCost, hungarian_assigner.py:153-158), which no
        # CPR / P2P config uses: they are rejected like every other unsupported cost, never silently replaced
        cc = cls_costs if cls_costs is not None else [dict(type='ClassificationCost', weight=1.)]
        rc = reg_costs if reg_costs is not None else [dict(type='BBoxL1Cost', weight=1.0, norm_with_img_size=True),
                                                      dict(type='IoUCost', iou_mode='giou', weight=1.0)]
        self.terms = match_cost_terms(cc, rc)
        self.topk_k = topk_k

    def assign(self, bbox_pred, cls_pred, gt_bboxes, gt_labels, img_meta, gt_bboxes_ignore=None, eps=1e-7):
        assert gt_bboxes_ignore is None, 'Only case when gt_bboxes_ignore is None is supported.'
        if not bbox_pred.is_cuda:
            raise RuntimeError('HungarianAssignerV2 runs on CUDA tensors only; there is no CPU fallback')
        if bbox_pred.shape[-1] != 2 or (gt_bboxes.numel() > 0 and gt_bboxes.shape[-1] != 2):
            raise NotImplementedError('HungarianAssignerV2: DisCostV2 on (x, y) points only (k*2 = 2 coordinates, as P2PHead uses it)')
        N, n = bbox_pred.shape[0], gt_bboxes.shape[0]
        dev = bbox_pred.device
        gt_inds = torch.zeros((N,), dtype=torch.long, device=dev)
        labels = torch.full((N,), -1, dtype=torch.long, device=dev)
        if N == 0 or n == 0:                        # hungarian_assigner.py:211-219: no GT -> everything background
            return AssignResult(n, gt_inds, None, labels)
        cost = cost_matrix(cls_pred.detach().float().contiguous(), bbox_pred.detach()[:, :2].float().contiguous(), None,
                           gt_bboxes[:, :2].float().contiguous(), gt_labels.int().contiguous(), self.terms, img_meta.get('img_shape'))
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


def random_sample_plan(counts, num, pos_fraction, neg_pos_ub=-1):
    """The draws of BaseSampler.sample + RandomSampler (base_sampler.py:82-97, random_sampler.py:31-81) for images whose assignment has
    counts = [(positives, negatives), ...], image by image.  Makes exactly the reference's torch.randperm calls on the CPU default
    generator, in its order, so the sampled sets and the generator state after the call are the reference's.  Per image returns
    (pos, neg): None when every candidate of that kind is sampled (no draw), else the sorted ranks (int64) of the sampled candidates
    among the image's positives / negatives — the reference's `gallery[randperm(n)[:k]].unique()` with an ascending gallery."""
    plan = []
    num_expected_pos = int(num * pos_fraction)
    for n_pos, n_neg in counts:
        pos = torch.randperm(n_pos)[:num_expected_pos].unique() if n_pos > num_expected_pos else None
        n_sampled_pos = n_pos if pos is None else pos.numel()
        num_expected_neg = num - n_sampled_pos
        if neg_pos_ub >= 0:
            neg_upper_bound = int(neg_pos_ub * max(1, n_sampled_pos))
            if num_expected_neg > neg_upper_bound:
                num_expected_neg = neg_upper_bound
        neg = torch.randperm(n_neg)[:num_expected_neg].unique() if n_neg > num_expected_neg else None
        plan.append((pos, neg))
    return plan


def sampled_counts(plan, counts):
    """per image (sampled positives, sampled negatives) of a random_sample_plan"""
    return [tuple(c if sel is None else sel.numel() for sel, c in zip(p, cnt)) for p, cnt in zip(plan, counts)]


def upload_sample_plan(plan, device, tail=()):
    """the plan in the layout of ptb_rpn_anchor_targets / ptb_rpn_sampled_indices (include/ptb_b200.h), one copy from pinned memory;
    `tail` (ints) is appended after the drawn ranks, in the same copy"""
    head, body, off = [], [], 4 * len(plan)
    for p in plan:
        for sel in p:
            if sel is None:
                head += [0, -1]
            else:
                head += [off, sel.numel()]
                body.append(sel)
                off += sel.numel()
    buf = torch.empty((off + len(tail),), dtype=torch.int32, pin_memory=True)
    buf[:len(head)] = torch.tensor(head, dtype=torch.int32)
    if body:
        buf[len(head):off] = torch.cat(body)
    if len(tail):
        buf[off:] = torch.tensor(list(tail), dtype=torch.int32)
    return buf.to(device, non_blocking=True)


class RandomSampler:
    """mmdet/core/bbox/samplers/random_sampler.py:7-81 with base_sampler.py:8-101: same ctor kwargs and `sample` signature and result.
    The candidate ranks and counts come from ptb_rpn_candidate_ranks, the draws from random_sample_plan (the reference's randperm
    calls on the CPU generator), the sampled index lists from ptb_rpn_sampled_indices: one device-to-host copy (the two counts)."""

    def __init__(self, num, pos_fraction, neg_pos_ub=-1, add_gt_as_proposals=True, **kwargs):
        # kwargs may carry the reference's `rng`, which its random_choice never reads (it draws with torch.randperm)
        self.num, self.pos_fraction, self.neg_pos_ub, self.add_gt_as_proposals = num, pos_fraction, neg_pos_ub, add_gt_as_proposals

    def sample(self, assign_result, bboxes, gt_bboxes, gt_labels=None, **kwargs):
        if not assign_result.gt_inds.is_cuda:
            raise RuntimeError('RandomSampler runs on CUDA tensors only; there is no CPU fallback')
        if len(bboxes.shape) < 2:
            bboxes = bboxes[None, :]
        bboxes = bboxes[:, :4]
        gt_flags = bboxes.new_zeros((bboxes.shape[0],), dtype=torch.uint8)
        if self.add_gt_as_proposals and len(gt_bboxes) > 0:
            if gt_labels is None:
                raise ValueError('gt_labels must be given when add_gt_as_proposals is True')
            bboxes = torch.cat([gt_bboxes, bboxes], dim=0)
            assign_result.add_gt_(gt_labels)
            gt_flags = torch.cat([bboxes.new_ones(gt_bboxes.shape[0], dtype=torch.uint8), gt_flags])
        gt_inds = assign_result.gt_inds.contiguous()
        n = gt_inds.numel()
        rank, counts = ops.rpn_candidate_ranks(gt_inds.view(1, n), torch.full((1,), n, dtype=torch.int32, device=gt_inds.device))
        counts = [tuple(c) for c in counts.cpu().tolist()]
        plan = random_sample_plan(counts, self.num, self.pos_fraction, self.neg_pos_ub)
        (n_pos, n_neg), = sampled_counts(plan, counts)
        pos_inds, neg_inds = ops.rpn_sampled_indices(gt_inds, rank.view(-1), upload_sample_plan(plan, gt_inds.device), n_pos, n_neg)
        return SamplingResult(pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags)
