"""multiclass_nms — host-side mirror of mmdet/core/post_processing/bbox_nms.py:7-94 (which calls the third-party
mmcv.ops.nms.batched_nms) over ptb_multiclass_nms_boxes / ptb_multiclass_soft_nms: same arguments and return values
(`dets (k,5)`, `labels (k,)`, optionally `keep` = indices into the score-filtered candidate list, as the reference returns them).
CUDA tensors only; limits of the kernel: n <= 4096 candidates boxes, max_num <= 1024."""
import torch

from . import ops


def check_split_thr(nms_cfg):
    """mmcv's batched_nms switches to class-by-class NMS at `split_thr` candidates (default 10000); the NMS kernels hard-code that
    default, so any other value would silently give the other branch's answer."""
    if nms_cfg.get('split_thr', 10000) != 10000:
        raise NotImplementedError(f"nms split_thr={nms_cfg.get('split_thr')}: only mmcv's default 10000 is implemented")


def multiclass_nms(multi_bboxes, multi_scores, score_thr, nms_cfg, max_num=-1, score_factors=None, return_inds=False):
    """bbox_nms.py:7-94.  Options beyond what the point heads use (round 2, pinned by tests/golden/multiclass_nms_options.npz):
    `score_factors` (>= 0; the threshold sees the raw scores, the NMS ranks by the products, bbox_nms.py:52-62), class-specific boxes
    (n, #class*4) and `class_agnostic` NMS (both through one kernel candidate per (box, class): n * #class <= 4096), `max_num=-1`
    (exact while at most 1024 detections survive, else NotImplementedError)."""
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
    agnostic = bool(cfg.pop('class_agnostic', False))
    iou = cfg.pop('iou_threshold', cfg.pop('iou_thr', 0.5))
    scores = multi_scores[:, :-1].float()                                  # the last column is the background class
    thr = float(score_thr)
    valid = None
    if score_factors is not None:
        # the kernel filters and ranks by ONE number: candidates that fail the raw-score threshold become -inf, the rest the product
        valid = scores > score_thr
        scores = torch.where(valid, scores * score_factors.float().view(-1, 1), scores.new_full((), float('-inf')))
        thr = -3.4028234663852886e38
    if class_specific or agnostic:
        if n * C > 4096:
            raise NotImplementedError('class-specific boxes / class_agnostic NMS: n * #class must be <= 4096')
        if kind != 'nms':
            raise NotImplementedError('soft_nms with class-specific boxes or class_agnostic')
        boxes = (multi_bboxes.float().view(n, C, 4) if class_specific else multi_bboxes.float()[:, None].expand(n, C, 4)).reshape(1, n * C, 4).contiguous()
        flat = scores.reshape(-1)
        if agnostic:                                                       # one class for the kernel: no per-class separation
            k_scores = flat.view(1, n * C, 1).contiguous()
        else:                                                              # candidate (box p, class c) scores only in its own class
            k_scores = flat.new_full((n * C, C), float('-inf'))
            k_scores[torch.arange(n * C, device=flat.device), torch.arange(n * C, device=flat.device) % C] = flat
            k_scores = k_scores[None]
        cnt, det, lab, keep, _ = ops.multiclass_nms_boxes(boxes, k_scores, thr, iou, kmax)
        k = int(cnt[0])
        keep_k = keep[0, :k].long()
        if agnostic:                                                       # labels from the flat (box, class) index of the kept candidates
            inds = (flat > thr).nonzero(as_tuple=False).squeeze(1)
            labels = inds[keep_k] % C
        else:
            labels = lab[0, :k].long()
    else:
        boxes = multi_bboxes.float().contiguous()[None]
        k_scores = scores.contiguous()[None]
        if kind == 'nms':
            cnt, det, lab, keep, _ = ops.multiclass_nms_boxes(boxes, k_scores, thr, iou, kmax)
        elif kind == 'soft_nms':
            if score_factors is not None:
                raise NotImplementedError('soft_nms with score_factors')
            cnt, det, lab, keep, _ = ops.multiclass_soft_nms(boxes, k_scores, None, score_thr, iou, kmax, sigma=cfg.get('sigma', 0.5),
                                                             min_score=cfg.get('min_score', 1e-3), method=cfg.get('method', 'linear'))
        else:
            raise NotImplementedError(f'nms type {kind}')
        k = int(cnt[0])
        keep_k = keep[0, :k].long()
        labels = lab[0, :k].long()
    if unlimited and k >= kmax:
        raise NotImplementedError('max_num=-1: more than 1023 detections survive the NMS (kernel limit 1024)')
    dets = det[0, :k]
    return (dets, labels, keep_k) if return_inds else (dets, labels)
