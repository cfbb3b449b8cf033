"""Host restatement of the multiclass NMS and soft-NMS kernels of csrc/nms.cu (ptb_multiclass_nms, ptb_multiclass_nms_boxes,
ptb_multiclass_soft_nms), in numpy fp32 with the kernels' operation order.  It imports no kernel code.

Every `__f*_rn` of nms.cu is one plain fp32 operation here (numpy never fuses a multiply-add), and fminf / fmaxf are np.minimum /
np.maximum (no NaN reaches them: a zero-area pair gives its NaN only in the final division, where `NaN > thr` is false).

What mmcv's `batched_nms` (mmcv-full 1.3.x, third-party and not in this tree) does is restated from SURVEY.md's description and is
**unpinned** by any vector, like `oracle.p2p.soft_nms`:
  * fewer than `split_thr` (10000) candidates: offset every box by label * (max_coord + 1) and run ONE NMS over all of them
    (the offset branch);
  * `split_thr` candidates or more: the same offset boxes, NMS run class by class, and the kept entries sorted by (decayed) score,
    descending (the split branch).  That sort has no tie contract; the kernels break ties by flat id (point * C + class), and so
    does `merge` here.
"""
import numpy as np

F32 = np.float32
SPLIT_THR = 10000
SOFT_METHODS = {'naive': 0, 'linear': 1, 'gaussian': 2}
MAX_P, MAX_KEEP = 4096, 1024
SOFT_SMEM_DEFAULT = 48 * 1024


def raw_boxes(pts_or_boxes, pseudo_wh=None):
    """(P,4) fp32 un-offset boxes: explicit boxes as given, or the pseudo box pts -/+ (w * 0.5, h * 0.5) (nms.cu raw_box)."""
    a = np.asarray(pts_or_boxes, dtype=F32)
    if a.shape[-1] == 4:
        return a.copy()
    hw, hh = F32(pseudo_wh[0]) * F32(0.5), F32(pseudo_wh[1]) * F32(0.5)
    return np.stack([a[:, 0] - hw, a[:, 1] - hh, a[:, 0] + hw, a[:, 1] + hh], 1).astype(F32)


def candidates(scores, score_thr):
    """flat ids (point * C + class) of the candidates `score > score_thr`, ascending: position in this list = the `keep` rank."""
    s = np.asarray(scores, dtype=F32)
    return np.nonzero(s.reshape(-1) > F32(score_thr))[0]


def max_coord(rb, scores, score_thr):
    """boxes.max() over the candidate boxes (nms_prepare_kernel: every coordinate of every point with a candidate class)."""
    pts = np.nonzero((np.asarray(scores, dtype=F32) > F32(score_thr)).any(1))[0]
    return F32(rb[pts].max()) if len(pts) else F32(-np.inf)


def offset_boxes(rb, labels, m):
    """nms.cu offset_box: coordinates + fl(label * fl(max_coord + 1)), area = fl(fl(x2 - x1) * fl(y2 - y1)) -> (n,5) fp32."""
    off = np.asarray(labels).astype(F32) * (F32(m) + F32(1))
    b = (rb + off[:, None]).astype(F32)
    area = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(F32)
    return np.concatenate([b, area[:, None]], 1)


def iou(a, b):
    """IoU of one offset box a (5,) against boxes b (n,5) in nms.cu's order: max(0, min - max) per axis, fl(w*h),
    fl(inter / fl(fl(area_a + area_b) - inter))."""
    with np.errstate(invalid='ignore', divide='ignore'):
        w = np.maximum(F32(0), np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0]))
        h = np.maximum(F32(0), np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1]))
        inter = w * h
        return (inter / ((a[4] + b[:, 4]) - inter)).astype(F32)


def iou_gt(a, b, thr):
    """nms.cu iou_gt: suppression test of hard NMS, strictly greater."""
    return iou(a, b) > F32(thr)


def soft_weight(ovr, iou_thr, sigma, method):
    """nms.cu soft_weight.  The gaussian branch uses np.exp in fp32; the kernel's expf is within 2 ulp of it."""
    ovr = np.asarray(ovr, dtype=F32)
    thr = F32(iou_thr)
    with np.errstate(invalid='ignore'):
        if method == 0:
            return np.where(ovr >= thr, F32(0), F32(1)).astype(F32)
        if method == 1:
            return np.where(ovr >= thr, F32(1) - ovr, F32(1)).astype(F32)
        return np.exp(-(ovr * ovr) / F32(sigma)).astype(F32)


def _order(s, ids):
    """(score desc, id asc): the kernels' 64-bit keys (~score bits << 32 | id) for non-negative scores."""
    return np.lexsort((ids, -s.astype(np.float64)))


def greedy(ob, s, ids, iou_thr, max_keep):
    """greedy NMS of offset boxes ob (n,5) visited in (score desc, id asc) order, stopping at max_keep kept -> indices into ob."""
    order = _order(s, ids)
    sup = np.zeros(len(s), bool)
    keep = []
    for pos, i in enumerate(order):
        if sup[i]:
            continue
        keep.append(i)
        if len(keep) == max_keep:
            break
        rest = order[pos + 1:]
        sup[rest[iou_gt(ob[i], ob[rest], iou_thr)]] = True
    return np.array(keep, np.int64)


NEAR = 1e-5    # relative margin under which a gaussian decision (expf against np.exp, a few ulp apart) counts as a near-tie


def _near(a, b):
    a, b = np.float64(a), np.float64(b)
    return abs(a - b) <= NEAR * max(abs(a), abs(b), 1e-30)


def soft(ob, s, ids, iou_thr, sigma, min_score, method, max_keep):
    """soft-NMS as the kernels run it: select the alive entry of highest score, lowest position (`ids` ascending = position), decay
    every other alive entry by soft_weight(IoU with the selected one), drop those below min_score, stop at max_keep selections.
    returns (indices into ob in selection order, decayed score at selection, sure): sure[k] is False from the first selection whose
    runner-up, or an earlier min_score decision, lies within NEAR of it - there the gaussian method's outcome is not decided by
    the restatement."""
    sc = s.astype(F32).copy()
    alive = np.ones(len(sc), bool)
    sel, val, sure, ok = [], [], [], True
    while len(sel) < max_keep and alive.any():
        cand = np.nonzero(alive)[0]
        o = cand[_order(sc[cand], ids[cand])]
        i = o[0]
        if len(o) > 1 and _near(sc[i], sc[o[1]]):
            ok = False
        sel.append(i)
        val.append(sc[i])
        sure.append(ok)
        alive[i] = False
        rest = np.nonzero(alive)[0]
        if len(rest):
            ns = (sc[rest] * soft_weight(iou(ob[i], ob[rest]), iou_thr, sigma, method)).astype(F32)
            sc[rest] = ns
            with np.errstate(invalid='ignore'):
                alive[rest[ns < F32(min_score)]] = False
                if (np.abs(ns.astype(np.float64) - np.float64(F32(min_score))) <= NEAR * np.float64(F32(min_score))).any():
                    ok = False
    return np.array(sel, np.int64), np.array(val, F32), np.array(sure, bool)


def degenerate(ob):
    """nms.cu degenerate_weight summed over offset boxes (n,5): 1 per zero area, 2 per negative or NaN area.  Gaussian soft-NMS
    refuses an image at >= 2 (IoU 0/0 = NaN gives NaN weights in mmcv's loop)."""
    a = ob[:, 4]
    return int((a == 0).sum() + 2 * (~(a >= 0)).sum())


def merge(lists, max_keep):
    """C-way merge of per-class (flat id, score[, sure]) lists by (score desc, flat id asc), first max_keep.  returns ids, scores
    and, per row, whether the row is decided (its list entry sure, no neighbour of the full merge within NEAR)."""
    if not lists:
        return np.zeros(0, np.int64), np.zeros(0, F32), np.zeros(0, bool)
    ids = np.concatenate([l[0] for l in lists]).astype(np.int64)
    sc = np.concatenate([l[1] for l in lists]).astype(F32)
    sure = np.concatenate([l[2] if len(l) > 2 else np.ones(len(l[0]), bool) for l in lists])
    o = _order(sc, ids)
    ids, sc, sure = ids[o], sc[o], sure[o].copy()
    adj = np.array([_near(a, b) for a, b in zip(sc[:-1], sc[1:])], bool)
    sure[:-1] &= ~adj
    sure[1:] &= ~adj
    return ids[:max_keep], sc[:max_keep], sure[:max_keep]


def slow_flag(pts_or_boxes, scores, score_thr, pseudo_wh=None):
    """fp32 mirror of nms_prepare_kernel's test for images whose class offset may not separate the classes: min x1 / min y1 over
    the candidate boxes with x1 < -0.95 and y1 < -0.95 (mnx, mny), then any candidate box with x2 > fl(fl(mnx + m1) - 0.05) and
    y2 > fl(fl(mny + m1) - 0.05), m1 = fl(max_coord + 1)."""
    rb = raw_boxes(pts_or_boxes, pseudo_wh)
    s = np.asarray(scores, dtype=F32)
    cp = (s > F32(score_thr)).any(1)
    if not cp.any():
        return False
    b = rb[cp]
    corner = (b[:, 0] < F32(-0.95)) & (b[:, 1] < F32(-0.95))
    if not corner.any():
        return False
    mnx, mny = b[corner, 0].min(), b[corner, 1].min()
    m1 = F32(b.max()) + F32(1)
    return bool(((b[:, 2] > (mnx + m1) - F32(0.05)) & (b[:, 3] > (mny + m1) - F32(0.05))).any())


def image(pts_or_boxes, scores, score_thr, iou_thr, max_keep, pseudo_wh=None, soft_cfg=None, branch='auto', split_thr=SPLIT_THR):
    """multiclass NMS of one image.  scores (P,C); soft_cfg None (hard NMS) or dict(sigma, min_score, method).
    branch: 'offset' (one NMS over all offset boxes), 'split' (class by class, then the merge), or 'auto' (mmcv's choice:
    'offset' below split_thr candidates, else 'split').
    returns dict(count, cand_count, keep (ranks), labels, flat, det (count,5) raw boxes + (decayed) score, refused, exact_upto,
    all_exact).  refused: gaussian soft-NMS on an image with degenerate boxes (the kernels' out_count is -1).  exact_upto / all_exact:
    the gaussian method's rows before exact_upto are decided (keep, labels, boxes exact), and so is the count when all_exact;
    every other kind is exact throughout."""
    s = np.asarray(scores, dtype=F32)
    P, C = s.shape
    rb = raw_boxes(pts_or_boxes, pseudo_wh)
    flat = candidates(s, score_thr)
    n = len(flat)
    if branch == 'auto':
        branch = 'offset' if n < split_thr else 'split'
    gauss = soft_cfg is not None and soft_cfg['method'] == 'gaussian'
    sure, refused = None, False
    if n == 0:
        kf, ks = np.zeros(0, np.int64), np.zeros(0, F32)
    else:
        m = max_coord(rb, s, score_thr)
        p, c = flat // C, flat % C
        ob = offset_boxes(rb[p], c, m)
        cs = s.reshape(-1)[flat]
        refused = gauss and degenerate(ob) >= 2
        if refused:
            branch = 'refused'
            kf, ks = np.zeros(0, np.int64), np.zeros(0, F32)
        elif branch == 'offset':
            if soft_cfg is None:
                k = greedy(ob, cs, flat, iou_thr, max_keep)
                kf, ks = flat[k], cs[k]
            else:
                k, ks, sure = soft(ob, cs, flat, iou_thr, soft_cfg['sigma'], soft_cfg['min_score'], SOFT_METHODS[soft_cfg['method']],
                                   max_keep)
                kf = flat[k]
                adj = np.array([_near(a, b) for a, b in zip(ks[:-1], ks[1:])], bool)
                sure[:-1] &= ~adj
                sure[1:] &= ~adj
        else:
            lists = []
            for cl in np.unique(c):
                idx = np.nonzero(c == cl)[0]
                if soft_cfg is None:
                    k = greedy(ob[idx], cs[idx], flat[idx], iou_thr, max_keep)
                    lists.append((flat[idx][k], cs[idx][k]))
                else:
                    k, v, su = soft(ob[idx], cs[idx], flat[idx], iou_thr, soft_cfg['sigma'], soft_cfg['min_score'],
                                    SOFT_METHODS[soft_cfg['method']], max_keep)
                    lists.append((flat[idx][k], v, su))
            kf, ks, sure = merge(lists, max_keep)
            if soft_cfg is not None:
                all_lists_sure = all(bool(l[2].all()) for l in lists)
    kp, kc = kf // C, kf % C
    det = np.concatenate([rb[kp], ks[:, None]], 1).astype(F32) if len(kf) else np.zeros((0, 5), F32)
    if gauss and sure is not None:
        bad = np.nonzero(~sure)[0]
        exact_upto = int(bad[0]) if len(bad) else len(kf)
        all_exact = not len(bad) and (branch == 'offset' or all_lists_sure)
    else:
        exact_upto, all_exact = len(kf), True
    return dict(count=len(kf), cand_count=n, keep=np.searchsorted(flat, kf).astype(np.int64), labels=kc.astype(np.int64), flat=kf,
                det=det, branch=branch, refused=refused, exact_upto=exact_upto, all_exact=all_exact)


def batched(pts_or_boxes, scores, score_thr, iou_thr, max_keep, pseudo_wh=None, soft_cfg=None, split_thr=SPLIT_THR):
    """mmcv's batched_nms as restated above (branch on the candidate count), per image of a (B,P,C) batch."""
    return [image(pts_or_boxes[b], scores[b], score_thr, iou_thr, max_keep, pseudo_wh, soft_cfg, 'auto', split_thr)
            for b in range(len(scores))]


SOFT_SMEM_STATIC = 8 * 4 + 8 * 8 + 8      # soft_nms_class_kernel's static shared memory: s_wcnt, s_red, s_best


def soft_smem_bytes(P):
    """shared memory of soft_nms_class_kernel: six fp32 arrays, one int and one byte per point, + 16 (dynamic), + the static part."""
    return P * (7 * 4 + 1) + 16 + SOFT_SMEM_STATIC


def expected_path(pts_or_boxes, scores, score_thr, kind, pseudo_wh=None):
    """which kernels produce one image's result: 'global' (nms_global_kernel / soft_nms_global_kernel: `slow` set and fewer than
    10000 candidates) or 'class' (the per-class kernel and the merge), with the flags that select it and, for soft-NMS, whether
    the class kernel's shared memory (dynamic + static) is above the 48 KB default.  kind: 'hard' or 'soft'."""
    s = np.asarray(scores, dtype=F32)
    n = len(candidates(s, score_thr))
    slow = slow_flag(pts_or_boxes, s, score_thr, pseudo_wh)
    path = 'global' if slow and n < SPLIT_THR else 'class'
    optin = kind == 'soft' and soft_smem_bytes(s.shape[0]) > SOFT_SMEM_DEFAULT
    return dict(kind=kind, path=path, slow=slow, split=n >= SPLIT_THR, empty=n == 0, optin=optin)


def planted_slow(P, C, many, seed, side=256.0):
    """a square side x side image (pseudo boxes 32 x 32) with points in both extreme corners, so `slow` is set.  The class C-1 box of
    corner point 0 (score 0.99) intersects the class C-2 box of far point 3 (score 0.98) after the class offset, with IoU 0.12:
    the offset branch suppresses the far box, the split branch keeps it.  many: ~90 % of the (point, class) pairs are candidates
    (>= 10000 at P * C >= 12000), else ~10 %.  P >= 7."""
    rng = np.random.default_rng(seed)
    pts = (rng.random((P, 2)) * (side - 16) + 8).astype(F32)
    pts[:3] = [[0, 0], [1, 2], [2, 1]]
    pts[3:6] = [[side, side], [side - 1, side], [side, side - 1]]
    sc = (rng.random((P, C)) * 0.85 * (rng.random((P, C)) < (0.9 if many else 0.1))).astype(F32)
    sc += (np.arange(P * C).reshape(P, C) * 1e-7 * (sc > 0)).astype(F32)
    sc[0, C - 1], sc[3, C - 2] = F32(0.99), F32(0.98)
    pts[6], sc[6] = 4 * side, 0                     # far outside, no candidate: neither max_coord nor the `slow` test sees it
    return pts, sc, (32.0, 32.0)


def largest_reaching_x1(m, C):
    """for max coordinates m (fp32 array) at C classes: the largest fp32 corner x1 of a class C-1 box whose offset x1,
    fl(x1 + fl((C-1) * m1)), still lies below the offset x2 = m of a class C-2 box, fl(m + fl((C-2) * m1)), m1 = fl(m + 1).
    Bisection over float64 values, each rounded to fp32 before the test.  returns (x1, m1)."""
    m = np.asarray(m, dtype=F32)
    m1 = m + F32(1)
    A, X2 = F32(C - 1) * m1, m + F32(C - 2) * m1
    u = np.spacing(A).astype(np.float64)
    lo = X2.astype(np.float64) - A - 2 * u                   # reaches: fl(x1 + A) < X2
    hi = X2.astype(np.float64) - A + 2 * u                   # does not
    for _ in range(48):
        mid = (lo + hi) / 2
        r = (mid.astype(F32) + A) < X2
        lo, hi = np.where(r, mid, lo), np.where(r, hi, mid)
    x1 = lo.astype(F32)
    assert ((x1 + A) < X2).all()
    return x1, m1
