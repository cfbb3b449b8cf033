"""multiclass_nms — host-side mirror of mmdet/core/post_processing/bbox_nms.py:7-94 (which calls the third-party
mmcv.ops.nms.batched_nms) over ptb_multiclass_nms_boxes / ptb_multiclass_soft_nms: same arguments and return values
(`dets (k,5)`, `labels (k,)`, optionally `keep` = indices into the score-filtered candidate list, as the reference returns them).
CUDA tensors only; limits of the kernels: n <= 4096 boxes (n * #class <= 4096 for class_agnostic), max_num <= 1024.
Class-specific boxes (n, #class*4) go through ptb_multiclass_nms_cls_boxes / ptb_multiclass_soft_nms_cls_boxes."""
import torch

from . import ops


def check_split_thr(nms_cfg):
    """mmcv's batched_nms switches to class-by-class NMS at `split_thr` candidates (default 10000); the NMS kernels hard-code that
    default, so any other value would silently give the other branch's answer."""
    if nms_cfg.get('split_thr', 10000) != 10000:
        raise NotImplementedError(f"nms split_thr={nms_cfg.get('split_thr')}: only mmcv's default 10000 is implemented")


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
    unlimited = max_num <= 0
    if max_num > 1024:
        raise NotImplementedError('max_num must be <= 1024')
    kmax = 1024 if unlimited else int(max_num)
    check_split_thr(nms_cfg)
    cfg = dict(nms_cfg)
    kind = cfg.pop('type', 'nms')
    if kind not in ('nms', 'soft_nms'):
        raise NotImplementedError(f'nms type {kind}')
    agnostic = bool(cfg.pop('class_agnostic', False))
    iou = cfg.pop('iou_threshold', cfg.pop('iou_thr', 0.5))
    soft = dict(sigma=cfg.get('sigma', 0.5), min_score=cfg.get('min_score', 1e-3), method=cfg.get('method', 'linear'))
    scores = multi_scores[:, :-1].float()                                  # the last column is the background class
    thr = float(score_thr)
    if score_factors is not None:
        # the kernel filters and ranks by ONE number: candidates that fail the raw-score threshold become -inf, the rest the product
        valid = scores > score_thr
        scores = torch.where(valid, scores * score_factors.float().view(-1, 1), scores.new_full((), float('-inf')))
        thr = -3.4028234663852886e38
    if agnostic:
        if n * C > 4096:
            raise NotImplementedError('class_agnostic NMS: n * #class must be <= 4096')
        boxes = (multi_bboxes.float().view(n, C, 4) if class_specific else multi_bboxes.float()[:, None].expand(n, C, 4)).reshape(1, n * C, 4).contiguous()
        flat = scores.reshape(-1)
        k_scores = flat.view(1, n * C, 1).contiguous()                     # one class for the kernel: no per-class separation
        if kind == 'nms':
            cnt, det, lab, keep, _ = ops.multiclass_nms_boxes(boxes, k_scores, thr, iou, kmax)
        else:
            cnt, det, lab, keep, _ = ops.multiclass_soft_nms(boxes, k_scores, None, thr, iou, kmax, **soft)
        k = int(cnt[0])
        keep_k = keep[0, :k].long()
        inds = (flat > thr).nonzero(as_tuple=False).squeeze(1)             # labels from the flat (box, class) index of the kept candidates
        labels = inds[keep_k] % C
    else:
        # class-specific boxes as (1, n, C, 4): the ops take them to the *_cls_boxes entry points
        boxes = (multi_bboxes.float().reshape(1, n, C, 4) if class_specific else multi_bboxes.float()[None]).contiguous()
        k_scores = scores.contiguous()[None]
        if kind == 'nms':
            cnt, det, lab, keep, _ = ops.multiclass_nms_boxes(boxes, k_scores, thr, iou, kmax)
        else:
            cnt, det, lab, keep, _ = ops.multiclass_soft_nms(boxes, k_scores, None, thr, iou, kmax, **soft)
        k = int(cnt[0])
        keep_k = keep[0, :k].long()
        labels = lab[0, :k].long()
    if unlimited and k >= kmax:
        raise NotImplementedError('max_num=-1: more than 1023 detections survive the NMS (kernel limit 1024)')
    dets = det[0, :k]
    return (dets, labels, keep_k) if return_inds else (dets, labels)
