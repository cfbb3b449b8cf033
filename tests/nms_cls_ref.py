"""Host restatement of the class-specific box layout of csrc/nms.cu (ptb_multiclass_nms_cls_boxes, ptb_multiclass_soft_nms_cls_boxes):
boxes [P][C][4], candidate (p, c) uses boxes[p, c].  Built on tests/nms_ref.py (same fp32 operation order, the same branch rules of
mmcv's batched_nms); only where the candidates' boxes come from differs:
  * max_coord is the maximum over the candidates' own boxes;
  * the `slow` test runs over every candidate box;
  * a candidate's offset box and its det row are its own box.
"""
import numpy as np

from tests import nms_ref as ref

F32 = ref.F32


def cand_boxes(boxes, flat):
    """(n,4) fp32 boxes of the candidates with flat ids `flat` (point * C + class) of a (P,C,4) array."""
    return np.asarray(boxes, dtype=F32).reshape(-1, 4)[flat]


def slow_flag(boxes, scores, score_thr):
    """nms_prepare_kernel's test for images whose class offset may not separate the classes, over every candidate's own box."""
    flat = ref.candidates(scores, score_thr)
    if not len(flat):
        return False
    b = cand_boxes(boxes, flat)
    corner = (b[:, 0] < F32(-0.95)) & (b[:, 1] < F32(-0.95))
    if not corner.any():
        return False
    mnx, mny = b[corner, 0].min(), b[corner, 1].min()
    m1 = F32(b.max()) + F32(1)
    return bool(((b[:, 2] > (mnx + m1) - F32(0.05)) & (b[:, 3] > (mny + m1) - F32(0.05))).any())


def image(boxes, scores, score_thr, iou_thr, max_keep, soft_cfg=None, branch='auto', split_thr=ref.SPLIT_THR):
    """multiclass NMS of one image with class-specific boxes (P,C,4), scores (P,C); arguments and result as nms_ref.image."""
    s = np.asarray(scores, dtype=F32)
    P, C = s.shape
    flat = ref.candidates(s, score_thr)
    n = len(flat)
    if branch == 'auto':
        branch = 'offset' if n < split_thr else 'split'
    gauss = soft_cfg is not None and soft_cfg['method'] == 'gaussian'
    sure, refused, all_lists_sure = None, False, True
    cb = cand_boxes(boxes, flat)
    if n == 0:
        kf, ks = np.zeros(0, np.int64), np.zeros(0, F32)
    else:
        m = F32(cb.max())
        c = flat % C
        ob = ref.offset_boxes(cb, c, m)
        cs = s.reshape(-1)[flat]
        refused = gauss and ref.degenerate(ob) >= 2
        method = None if soft_cfg is None else ref.SOFT_METHODS[soft_cfg['method']]
        if refused:
            branch = 'refused'
            kf, ks = np.zeros(0, np.int64), np.zeros(0, F32)
        elif branch == 'offset':
            if soft_cfg is None:
                k = ref.greedy(ob, cs, flat, iou_thr, max_keep)
                kf, ks = flat[k], cs[k]
            else:
                k, ks, sure = ref.soft(ob, cs, flat, iou_thr, soft_cfg['sigma'], soft_cfg['min_score'], method, max_keep)
                kf = flat[k]
                adj = np.array([ref._near(a, b) for a, b in zip(ks[:-1], ks[1:])], bool)
                sure[:-1] &= ~adj
                sure[1:] &= ~adj
        else:
            lists = []
            for cl in np.unique(c):
                idx = np.nonzero(c == cl)[0]
                if soft_cfg is None:
                    k = ref.greedy(ob[idx], cs[idx], flat[idx], iou_thr, max_keep)
                    lists.append((flat[idx][k], cs[idx][k]))
                else:
                    k, v, su = ref.soft(ob[idx], cs[idx], flat[idx], iou_thr, soft_cfg['sigma'], soft_cfg['min_score'], method, max_keep)
                    lists.append((flat[idx][k], v, su))
            kf, ks, sure = ref.merge(lists, max_keep)
            if soft_cfg is not None:
                all_lists_sure = all(bool(l[2].all()) for l in lists)
    det = np.concatenate([cand_boxes(boxes, kf), ks[:, None]], 1).astype(F32) if len(kf) else np.zeros((0, 5), F32)
    if gauss and sure is not None:
        bad = np.nonzero(~sure)[0]
        exact_upto = int(bad[0]) if len(bad) else len(kf)
        all_exact = not len(bad) and (branch == 'offset' or all_lists_sure)
    else:
        exact_upto, all_exact = len(kf), True
    return dict(count=len(kf), cand_count=n, keep=np.searchsorted(flat, kf).astype(np.int64), labels=(kf % C).astype(np.int64), flat=kf,
                det=det, branch=branch, refused=refused, exact_upto=exact_upto, all_exact=all_exact)


def expected_path(boxes, scores, score_thr):
    """which kernels produce the image's result: 'global' (`slow` and fewer than 10000 candidates) or 'class'."""
    n = len(ref.candidates(scores, score_thr))
    slow = slow_flag(boxes, scores, score_thr)
    return dict(path='global' if slow and n < ref.SPLIT_THR else 'class', slow=slow, split=n >= ref.SPLIT_THR, empty=n == 0)


def glue_scores(scores_bg, score_thr, factors=None):
    """post_processing.multiclass_nms's kernel scores and threshold: the (n, C) foreground scores, or with score_factors the products
    where the raw score passes score_thr and -inf elsewhere, under a threshold of -FLT_MAX."""
    s = np.asarray(scores_bg, dtype=F32)[:, :-1]
    if factors is None:
        return s, score_thr
    prod = (s * np.asarray(factors, dtype=F32)[:, None]).astype(F32)
    return np.where(s > F32(score_thr), prod, F32(-np.inf)).astype(F32), float(-np.finfo(np.float32).max)
