"""multiclass_nms — host-side mirror of mmdet/core/post_processing/bbox_nms.py:7-94 (which calls the third-party
mmcv.ops.nms.batched_nms) over ptb_multiclass_nms_boxes / ptb_multiclass_soft_nms: same arguments and return values
(`dets (k,5)`, `labels (k,)`, optionally `keep` = indices into the score-filtered candidate list, as the reference returns them).
CUDA tensors only; limits of the kernels: n <= 4096 boxes (n * #class <= 4096 for class_agnostic), max_num <= 1024.
Class-specific boxes (n, #class*4) go through ptb_multiclass_nms_cls_boxes / ptb_multiclass_soft_nms_cls_boxes."""
from collections import namedtuple

import torch

from . import ops

NmsCfg = namedtuple('NmsCfg', 'kind iou sigma min_score method class_agnostic split_thr')
HARD_NMS_KEYS = frozenset(('type', 'iou_threshold', 'iou_thr', 'class_agnostic', 'split_thr'))     # what hard NMS reads of a config


def parse_nms_cfg(nms_cfg, default_iou=None):
    """an NmsCfg as mmcv reads an nms config (mmcv/ops/nms.py batched_nms, nms, soft_nms): kind = `type`, 'nms' (default) or
    'soft_nms'; iou = `iou_threshold` (mmcv >= 1.3), else its older spelling `iou_thr`, else `default_iou`, else soft_nms' own 0.3;
    soft_nms' defaults for sigma, min_score and method.  Other keys are ignored: each caller refuses what its kernels cannot run."""
    kind = nms_cfg.get('type', 'nms')
    if kind not in ('nms', 'soft_nms'):
        raise NotImplementedError(f'nms type {kind}')
    if 'iou_threshold' not in nms_cfg and 'iou_thr' not in nms_cfg and default_iou is None:
        if kind == 'nms':
            raise KeyError("test_cfg.nms needs 'iou_threshold' (or 'iou_thr')")
        default_iou = 0.3
    return NmsCfg(kind, float(nms_cfg.get('iou_threshold', nms_cfg.get('iou_thr', default_iou))), nms_cfg.get('sigma', 0.5),
                  nms_cfg.get('min_score', 1e-3), nms_cfg.get('method', 'linear'), bool(nms_cfg.get('class_agnostic', False)),
                  nms_cfg.get('split_thr', 10000))


def check_split_thr(nms_cfg):
    """mmcv's batched_nms switches to class-by-class NMS at `split_thr` candidates (default 10000); the NMS kernels hard-code that
    default, so any other value would silently give the other branch's answer."""
    if nms_cfg.get('split_thr', 10000) != 10000:
        raise NotImplementedError(f"nms split_thr={nms_cfg.get('split_thr')}: only mmcv's default 10000 is implemented")


def keep_limit(max_per_img):
    """(kmax, unlimited) of mmdet's max_per_img / max_num: the kernels keep at most 1024 per image; -1 (or 0) runs them at 1024"""
    max_per_img = int(max_per_img)
    if max_per_img > 1024:
        raise NotImplementedError('max_per_img must be <= 1024')
    return (1024, True) if max_per_img <= 0 else (max_per_img, False)


def check_kept(count, kmax, unlimited):
    """refuses an unlimited result whose largest count (a host int) fills all kmax slots: detections may have been cut"""
    if unlimited and count >= kmax:
        raise NotImplementedError('max_per_img=-1: more than 1023 detections survive the NMS (kernel limit 1024)')


def run_multiclass_nms(geom, scores, score_thr, nms, kmax, pseudo_wh=None, wide=False):
    """the NMS kernel for `nms` (a parse_nms_cfg record), hard or soft, of points (B, P, 2) with boxes of pseudo_wh, boxes shared by
    the classes (B, P, 4) or class-specific boxes (B, P, C, 4), and scores (B, P, C): ops' count, det, label, keep, cand_count"""
    if nms.kind == 'soft_nms':
        return ops.multiclass_soft_nms(geom, scores, pseudo_wh, score_thr, nms.iou, kmax, nms.sigma, nms.min_score, nms.method, wide=wide)
    if pseudo_wh is not None:
        return ops.multiclass_nms(geom, scores, pseudo_wh, score_thr, nms.iou, kmax, wide=wide)
    return ops.multiclass_nms_boxes(geom, scores, score_thr, nms.iou, kmax)


def multiclass_nms(multi_bboxes, multi_scores, score_thr, nms_cfg, max_num=-1, score_factors=None, return_inds=False):
    """bbox_nms.py:7-94 with nms_cfg type 'nms' or 'soft_nms' (sigma, min_score, method 'linear' | 'gaussian' | 'naive').
    Options beyond what the point heads use (pinned by tests/golden/multiclass_nms_options.npz and multiclass_nms_roi.npz):
      * `score_factors` (>= 0), hard and soft NMS: the threshold sees the raw scores, the NMS ranks by the products
        (bbox_nms.py:52-62); soft-NMS decays the products.
      * class-specific boxes (n, #class*4), the RoI head's call, hard and soft NMS: candidate (box p, class c) uses its own box
        through ptb_multiclass_nms_cls_boxes / ptb_multiclass_soft_nms_cls_boxes; n <= 4096 boxes at any number of classes.
      * `class_agnostic` NMS, hard and soft: one kernel candidate per (box, class) in a single class, so n * #class <= 4096.
      * `max_num=-1`: exact while at most 1023 detections survive, else NotImplementedError.
    Limits of the kernels: n <= 4096 boxes, max_num <= 1024, mmcv's default split_thr."""
    if not multi_bboxes.is_cuda:
        raise RuntimeError('multiclass_nms runs on CUDA tensors only; there is no CPU fallback')
    n, C = multi_scores.shape[0], multi_scores.shape[1] - 1
    class_specific = multi_bboxes.shape[1] > 4
    if class_specific and multi_bboxes.shape[1] != 4 * C:
        raise ValueError(f'multi_bboxes must be (n, 4) or (n, {4 * C})')
    kmax, unlimited = keep_limit(max_num)
    check_split_thr(nms_cfg)
    nms = parse_nms_cfg(nms_cfg, default_iou=0.5)
    scores = multi_scores[:, :-1].float()                                  # the last column is the background class
    thr = float(score_thr)
    if score_factors is not None:
        # the kernel filters and ranks by ONE number: candidates that fail the raw-score threshold become -inf, the rest the product
        valid = scores > score_thr
        scores = torch.where(valid, scores * score_factors.float().view(-1, 1), scores.new_full((), float('-inf')))
        thr = -3.4028234663852886e38
    if nms.class_agnostic:
        if n * C > 4096:
            raise NotImplementedError('class_agnostic NMS: n * #class must be <= 4096')
        boxes = (multi_bboxes.float().view(n, C, 4) if class_specific else multi_bboxes.float()[:, None].expand(n, C, 4)).reshape(1, n * C, 4).contiguous()
        flat = scores.reshape(-1)
        k_scores = flat.view(1, n * C, 1).contiguous()                     # one class for the kernel: no per-class separation
    else:
        # class-specific boxes as (1, n, C, 4): the ops take them to the *_cls_boxes entry points
        boxes = (multi_bboxes.float().reshape(1, n, C, 4) if class_specific else multi_bboxes.float()[None]).contiguous()
        k_scores = scores.contiguous()[None]
    cnt, det, lab, keep, _ = run_multiclass_nms(boxes, k_scores, thr, nms, kmax)
    k = int(cnt[0])
    check_kept(k, kmax, unlimited)
    keep_k = keep[0, :k].long()
    # class_agnostic: the labels from the flat (box, class) index of the kept candidates
    labels = (flat > thr).nonzero(as_tuple=False).squeeze(1)[keep_k] % C if nms.class_agnostic else lab[0, :k].long()
    dets = det[0, :k]
    return (dets, labels, keep_k) if return_inds else (dets, labels)
