"""ORACLE (test infrastructure, NOT product code) — CPU restatement of the reference P2P head path.

Follows /root/reference/TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py (P2PHead),
mmdet/core/bbox/assigners/hungarian_assigner.py:149-270 (HungarianAssignerV2),
mmdet/core/bbox/match_costs/match_cost.py:54-100,190-214 (FocalLossCost, DisCostV2),
mmdet/core/bbox/assigners/point_assigner.py:8-133 (PointAssigner),
mmdet/core/post_processing/bbox_nms.py:7-94 (multiclass_nms) and the third-party
mmcv.ops.nms.batched_nms (mmcv-full 1.3.2..1.4.0, NOT in /root/reference; published algorithm restated in
`nms`/`batched_nms` below and cross-checked against torchvision.ops.nms in tests/test_oracle_*.py).
"ref:" = p2p_head.py unless a file is named.  Only tests/, smoke() and bench.py's baseline legs import this.
"""
import numpy as np
import torch
import torch.nn.functional as F


def default_cfg(**over):
    """P2PHead ctor/test_cfg/train_cfg values of configs2/COCO/p2p/p2p_r50_fpns4_1x_fl_sl1_coco.py:85-127."""
    cfg = dict(
        num_classes=80, in_channels=256, feat_channels=256, stacked_convs=4, stride=4, gn_groups=32,
        point_anchor=[(0., 0.)], pts_gamma=1.0, reg_norm=1.0, assign_before_pred=False,
        focal_gamma=2.0, focal_alpha=0.25, loss_cls_weight=1.0, sl1_beta=1.0 / 9.0, loss_reg_weight=0.5,
        cls_cost_weight=2.0, dis_cost_weight=0.1, dis_norm_with_img_wh=False, dis_p=1, topk_k=5,
        neg_weight=1.0, pos_weight=1.0,
        nms_pre=1000, score_thr=0.05, pseudo_wh=(32, 32), nms_iou=0.01, max_per_img=100,
    )
    cfg.update(over)
    return cfg


# ----------------------------------------------------------------------------------------------
def head_forward(x, weights, cfg):
    """ref:113-123: cls tower + reg tower (conv3x3+GN+ReLU) then conv3x3 out layers."""
    def tower(x, prefix):
        for i in range(cfg['stacked_convs']):
            x = F.conv2d(x, weights[f'{prefix}.{i}.conv.weight'], None, 1, 1)
            x = F.group_norm(x, cfg['gn_groups'], weights[f'{prefix}.{i}.gn.weight'], weights[f'{prefix}.{i}.gn.bias'])
            x = F.relu(x)
        return x
    cls_out = F.conv2d(tower(x, 'cls_convs'), weights['cls_out.weight'], weights['cls_out.bias'], 1, 1)
    pts_out = F.conv2d(tower(x, 'reg_convs'), weights['reg_out.weight'], weights['reg_out.bias'], 1, 1)
    return cls_out, pts_out


def grid_points(h, w, stride):
    """core/anchor/point_generator.py:17-25: (j*s, i*s, s) row-major, NO half-stride offset."""
    sx = torch.arange(0., w) * stride
    sy = torch.arange(0., h) * stride
    xx = sx.repeat(len(sy))
    yy = sy.view(-1, 1).repeat(1, len(sx)).view(-1)
    return torch.stack([xx, yy, xx.new_full((xx.shape[0],), stride)], dim=-1)


def valid_flags(h, w, pad_h, pad_w, stride):
    """ref:452-463 + point_generator.py:27-37."""
    vh = min(int(np.ceil(pad_h / stride)), h)
    vw = min(int(np.ceil(pad_w / stride)), w)
    vx = torch.zeros(w, dtype=torch.bool)
    vy = torch.zeros(h, dtype=torch.bool)
    vx[:vw] = 1
    vy[:vh] = 1
    return vx.repeat(len(vy)) & vy.view(-1, 1).repeat(1, len(vx)).view(-1)


def pred_points(cls_out, pts_out, img_metas, cfg):
    """ref:125-170 get_pred_points for ONE level.
    cls_out (B,k*C,H,W), pts_out (B,2k,H,W) -> anchor (B,HWk,3), pred (B,HWk,3), valid (B,HWk), cls (B,HWk,C)."""
    B, _, H, W = cls_out.shape
    k = len(cfg['point_anchor'])
    C = cfg['num_classes']
    s = cfg['stride']
    cls = cls_out.reshape(B, cls_out.size(1), -1).permute(0, 2, 1).reshape(B, H * W, k, C)
    reg = pts_out.reshape(B, pts_out.size(1), -1).permute(0, 2, 1).reshape(B, H * W, k, 2)
    centers = grid_points(H, W, s).unsqueeze(0).repeat(B, 1, 1)
    flags = torch.stack([valid_flags(H, W, *m['pad_shape'][:2], s) for m in img_metas])
    anchor = centers.unsqueeze(2).repeat(1, 1, k, 1)
    anchor[..., :2] += torch.FloatTensor(cfg['point_anchor']) * anchor[..., -1:]
    flags = flags.unsqueeze(2).repeat(1, 1, k)
    pred = anchor[..., :2] + reg * cfg['pts_gamma'] * anchor[..., -1:]
    pred = torch.cat([pred, anchor[..., -1:]], dim=-1)
    return (anchor.reshape(B, -1, 3), pred.reshape(B, -1, 3), flags.reshape(B, -1), cls.reshape(B, -1, C))


# ----------------------------------------------------------------------------------------------
# assignment
# ----------------------------------------------------------------------------------------------
def focal_loss_cost(cls_pred, gt_labels, weight=1., alpha=0.25, gamma=2, eps=1e-12):
    """match_cost.py:94-99"""
    p = cls_pred.sigmoid()
    neg = -(1 - p + eps).log() * (1 - alpha) * p.pow(gamma)
    pos = -(p + eps).log() * alpha * (1 - p).pow(gamma)
    return (pos[:, gt_labels] - neg[:, gt_labels]) * weight


def dis_cost_v2(pts, gts, img_shape, weight=1., norm_with_img_wh=True, p=1):
    """match_cost.py:197-214"""
    factor = 1.0
    if norm_with_img_wh:
        k = pts.shape[-1] // 2
        factor = gts.new_tensor([img_shape[1], img_shape[0]] * k).unsqueeze(0)
    return torch.cdist(pts / factor, gts / factor, p=p) * weight


def cost_matrix(pts, cls_pred, gts, gt_labels, img_shape, cfg):
    """hungarian_assigner.py:222-227"""
    return (focal_loss_cost(cls_pred, gt_labels, cfg['cls_cost_weight'], cfg['focal_alpha'], cfg['focal_gamma'])
            + dis_cost_v2(pts, gts, img_shape, cfg['dis_cost_weight'], cfg['dis_norm_with_img_wh'], cfg['dis_p']))


def hungarian_v2_from_cost(cost, gt_labels, topk_k):
    """hungarian_assigner.py:229-270: <=topk_k rounds of scipy linear_sum_assignment on unassigned rows.
    cost (N,n) CPU float -> assigned_gt_inds (N,) int64 (0 bg, j+1 fg), assigned_labels (N,) (-1 bg)."""
    from scipy.optimize import linear_sum_assignment
    N, n = cost.shape
    gt_inds = torch.zeros(N, dtype=torch.long)
    labels = torch.full((N,), -1, dtype=torch.long)
    if n == 0 or N == 0:
        return gt_inds, labels
    cost = cost.detach().cpu()
    if topk_k == 1:
        r, c = linear_sum_assignment(cost)
        r, c = torch.from_numpy(r), torch.from_numpy(c)
        gt_inds[r] = c + 1
        labels[r] = gt_labels[c]
        return gt_inds, labels
    assign = torch.zeros(N, dtype=torch.long)
    index = torch.nonzero(assign == 0).squeeze(1)
    cost_new = cost[assign == 0]
    num = 0
    while cost_new.shape[0] // n != 0 and num + 1 <= topk_k:
        num += 1
        r, c = linear_sum_assignment(cost_new)
        r, c = torch.from_numpy(r), torch.from_numpy(c)
        r = index[r]
        gt_inds[r] = c + 1
        assign[r] = c + 1
        labels[r] = gt_labels[c]
        index = torch.nonzero(assign == 0).squeeze(1)
        cost_new = cost[assign == 0]
    return gt_inds, labels


def target_single(pred_pts, valid, cls_outs, gt_points, gt_labels, img_shape, cfg):
    """ref:275-328 _get_target_single + sample_result_to_target + unmap (fill=0).
    returns labels (N,) long, label_weights (N,), gt_pts (N,2), pts_weights (N,2), gt_inds (N,) (unmapped)."""
    N = pred_pts.shape[0]
    props, cls = pred_pts[valid], cls_outs[valid]
    cost = cost_matrix(props, cls, gt_points, gt_labels, img_shape, cfg)
    gt_inds, _ = hungarian_v2_from_cost(cost, gt_labels, cfg['topk_k'])
    nv = props.shape[0]
    bbox_gt = props.new_zeros(nv, 2)
    pw = props.new_zeros(nv, 2)
    labels = props.new_full((nv,), cfg['num_classes'], dtype=torch.long)
    lw = props.new_zeros(nv)
    pos = torch.nonzero(gt_inds > 0).squeeze(-1)
    neg = torch.nonzero(gt_inds == 0).squeeze(-1)
    if len(pos) > 0:
        bbox_gt[pos] = gt_points[gt_inds[pos] - 1]
        pw[pos] = 1.0
        labels[pos] = gt_labels[gt_inds[pos] - 1]
        lw[pos] = cfg['pos_weight']
    if len(neg) > 0:
        lw[neg] = 1.0 if cfg['neg_weight'] <= 0 else cfg['neg_weight']

    def unmap(d):
        out = d.new_zeros((N,) + d.shape[1:])
        out[valid] = d
        return out
    return unmap(labels), unmap(lw), unmap(bbox_gt), unmap(pw), unmap(gt_inds)


def sigmoid_focal_loss_elem(pred, target_labels, gamma, alpha):
    """losses/focal_loss.py:11-56 py_sigmoid_focal_loss elementwise part; labels==num_classes -> bg row."""
    C = pred.size(1)
    t = F.one_hot(target_labels, num_classes=C + 1)[:, :C].type_as(pred)
    p = pred.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    fw = (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    return F.binary_cross_entropy_with_logits(pred, t, reduction='none') * fw


def smooth_l1_elem(pred, target, beta):
    """losses/smooth_l1_loss.py:25-31"""
    d = torch.abs(pred - target)
    return torch.where(d < beta, 0.5 * d * d / beta, d - 0.5 * beta)


def p2p_loss(cls_out, pts_out, gt_bboxes, gt_labels, img_metas, cfg, return_all=False):
    """ref:172-248: returns dict(loss_cls=[B], loss_pts=[B])."""
    anchor, pred, valid, cls = pred_points(cls_out, pts_out, img_metas, cfg)
    gt_points = [(b[:, :2] + b[:, 2:]) / 2 for b in gt_bboxes]
    prop = anchor if cfg['assign_before_pred'] else pred
    tg = [target_single(prop[b][..., :2].detach(), valid[b], cls[b].detach(), gt_points[b], gt_labels[b],
                        img_metas[b]['img_shape'], cfg) for b in range(len(img_metas))]
    num_total_pos = sum([(t[3][..., 0] > 0).sum() for t in tg])
    loss_cls, loss_pts = [], []
    for b, (labels, lw, gpts, pw, _) in enumerate(tg):
        l = sigmoid_focal_loss_elem(cls[b].contiguous(), labels, cfg['focal_gamma'], cfg['focal_alpha'])
        l = (l * lw.view(-1, 1)).sum() / num_total_pos
        loss_cls.append(cfg['loss_cls_weight'] * l)
        s = pred[b][..., -1:]
        r = smooth_l1_elem(pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm'], cfg['sl1_beta'])
        loss_pts.append(cfg['loss_reg_weight'] * ((r * pw).sum() / num_total_pos))
    out = dict(loss_cls=loss_cls, loss_pts=loss_pts)
    if return_all:
        return out, dict(targets=tg, pred=pred, valid=valid, cls=cls)
    return out


# ----------------------------------------------------------------------------------------------
# NMS (third-party mmcv-full semantics restated)
# ----------------------------------------------------------------------------------------------
def nms(boxes, scores, iou_threshold):
    """mmcv.ops.nms(offset=0) CPU semantics: visit boxes by descending score; a box is suppressed when its
    IoU with an already-kept box is > iou_threshold; area=(x2-x1)*(y2-y1); returns keep indices in
    descending-score order.  Ties in score are visited lower-index first (stable order) here."""
    b = boxes.detach().cpu().numpy().astype(np.float32)
    s = scores.detach().cpu().numpy()
    order = np.argsort(-s, kind='stable')
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    areas = (x2 - x1) * (y2 - y1)
    suppressed = np.zeros(len(b), dtype=bool)
    keep = []
    thr = np.float32(iou_threshold)
    for _i in range(len(order)):
        i = order[_i]
        if suppressed[i]:
            continue
        keep.append(i)
        rest = order[_i + 1:]
        xx1 = np.maximum(x1[i], x1[rest]); yy1 = np.maximum(y1[i], y1[rest])
        xx2 = np.minimum(x2[i], x2[rest]); yy2 = np.minimum(y2[i], y2[rest])
        w = np.maximum(np.float32(0), xx2 - xx1); h = np.maximum(np.float32(0), yy2 - yy1)
        inter = w * h
        ovr = inter / (areas[i] + areas[rest] - inter)
        suppressed[rest[ovr > thr]] = True
    return torch.as_tensor(np.array(keep, dtype=np.int64))


SOFT_NMS_METHODS = {'naive': 0, 'linear': 1, 'gaussian': 2}


def soft_nms(boxes, scores, iou_threshold=0.3, sigma=0.5, min_score=1e-3, method='linear', offset=0):
    """mmcv.ops.nms.soft_nms (mmcv-full 1.3.x, third-party, NOT under /root/reference: parity unpinned).  Restated from the
    published CPU kernel `softnms_cpu_kernel` (mmcv/ops/csrc/pytorch/cpu/nms.cpp), array swaps included:
      for i in 0..n-1:  move the first maximum of sc[i:] to position i (swap);  for every later box: sc *= weight(iou with box i)
        naive: weight 0 if iou >= thr;  linear: 1 - iou if iou >= thr;  gaussian: exp(-iou^2 / sigma)   (fp32 arithmetic)
        a box whose score drops below min_score is overwritten by the last box and n shrinks (the moved box is examined next).
    returns dets (k,5) [box, decayed score] in selection order (non-increasing score) and inds (k,) into the input."""
    b = boxes.detach().cpu().numpy().astype(np.float32).copy()
    sc = scores.detach().cpu().numpy().astype(np.float32).copy()
    n = len(b)
    off = np.float32(offset)
    x1, y1, x2, y2 = b[:, 0].copy(), b[:, 1].copy(), b[:, 2].copy(), b[:, 3].copy()
    areas = (x2 - x1 + off) * (y2 - y1 + off)
    inds = np.arange(n, dtype=np.int64)
    dets = np.zeros((n, 5), dtype=np.float32)
    thr, sg, ms, m = np.float32(iou_threshold), np.float32(sigma), np.float32(min_score), SOFT_NMS_METHODS[method]
    arrays = (x1, y1, x2, y2, sc, areas, inds)
    i = 0
    while i < n:
        mp = i + int(np.argmax(sc[i:n]))                   # first maximum (strict '<' update in the C++ loop)
        for arr in arrays:
            arr[i], arr[mp] = arr[mp], arr[i]
        dets[i] = (x1[i], y1[i], x2[i], y2[i], sc[i])
        # the C++ inner loop visits every later box exactly once (a box moved in by a deletion is examined at its new place), so
        # the score update is order independent and can be vectorised; only the ARRANGEMENT left by the swap-deletions is sequential
        r = slice(i + 1, n)
        w = np.maximum(np.float32(0), np.minimum(x2[i], x2[r]) - np.maximum(x1[i], x1[r]) + off)
        h = np.maximum(np.float32(0), np.minimum(y2[i], y2[r]) - np.maximum(y1[i], y1[r]) + off)
        inter = w * h
        ovr = inter / ((areas[i] + areas[r]) - inter)
        if m == 0:
            weight = np.where(ovr >= thr, np.float32(0), np.float32(1))
        elif m == 1:
            weight = np.where(ovr >= thr, np.float32(1) - ovr, np.float32(1))
        else:
            weight = np.exp(-(ovr * ovr) / sg).astype(np.float32)
        sc[r] = sc[r] * weight.astype(np.float32)
        pos = i + 1
        while pos < n:
            dead = sc[pos:n] < ms
            if not dead.any():
                break
            pos += int(np.argmax(dead))                    # next box below min_score: overwritten by the last box, n shrinks,
            for arr in arrays:                             # and the moved box is looked at next (pos does not advance)
                arr[pos] = arr[n - 1]
            n -= 1
        i += 1
    return torch.from_numpy(dets[:n].copy()), torch.from_numpy(inds[:n].copy())


SPLIT_THR = 10000


def _split_branch(boxes_for_nms, scores, idxs, nms_op):
    """batched_nms at split_thr candidates or more: nms_op(boxes, scores) -> (dets, keep) class by class (by `idxs`, also when
    class_agnostic dropped the offset) on the boxes given, then the kept entries sorted by their score after NMS, descending - for
    soft-NMS the DECAYED score (dets[:, -1]); versions early in mmcv's 1.3.2..1.4.0 window may sort by the original scores.  mmcv's
    sort has no tie contract; here ties keep the candidate order (ascending flat id), as the kernels' merge does.  Restated from
    SURVEY.md's description of mmcv 1.3.x: unpinned."""
    total = torch.zeros(scores.shape, dtype=torch.bool)
    after = scores.new_zeros(scores.shape)
    for c in torch.unique(idxs):
        m = (idxs == c).nonzero(as_tuple=False).view(-1)
        dets, keep = nms_op(boxes_for_nms[m], scores[m])
        total[m[keep]] = True
        after[m[keep]] = dets[:, -1]
    keep = total.nonzero(as_tuple=False).view(-1)
    sc, inds = after[keep].sort(descending=True, stable=True)
    return sc, keep[inds]


def batched_soft_nms(boxes, scores, idxs, nms_cfg):
    """batched_nms with nms_cfg['type'] == 'soft_nms' (mmcv/ops/nms.py): class offset, then soft_nms on everything (fewer than
    nms_cfg.get('split_thr', 10000) candidates) or class by class (the split branch); boxes[keep] with the DECAYED scores."""
    cfg = {k: v for k, v in nms_cfg.items() if k not in ('type', 'split_thr', 'class_agnostic')}
    agnostic = nms_cfg.get('class_agnostic', False)
    b = boxes if agnostic else boxes + (idxs.to(boxes) * (boxes.max() + 1))[:, None]
    if len(boxes) < nms_cfg.get('split_thr', SPLIT_THR):
        dets, keep = soft_nms(b, scores, **cfg)
        return torch.cat([boxes[keep], dets[:, -1:]], -1), keep
    sc, keep = _split_branch(b, scores, idxs, lambda bb, ss: soft_nms(bb, ss, **cfg))
    return torch.cat([boxes[keep], sc[:, None]], -1), keep


def batched_nms(boxes, scores, idxs, iou_threshold, class_agnostic=False, split_thr=SPLIT_THR):
    """mmcv.ops.nms.batched_nms: offset every box by label*(boxes.max()+1), then plain NMS over everything (fewer than split_thr
    boxes) or class by class with the kept entries sorted by score (the split branch, which loops over `idxs` even when class_agnostic).
    returns dets (k,5) [original boxes, score] and keep."""
    if class_agnostic:
        b = boxes
    else:
        b = boxes + (idxs.to(boxes) * (boxes.max() + 1))[:, None]
    if len(boxes) < split_thr:
        keep = nms(b, scores, iou_threshold)
        return torch.cat([boxes[keep], scores[keep, None]], -1), keep

    def op(bb, ss):
        k = nms(bb, ss, iou_threshold)
        return ss[k, None], k
    sc, keep = _split_branch(b, scores, idxs, op)
    return torch.cat([boxes[keep], sc[:, None]], -1), keep


def multiclass_nms(multi_bboxes, multi_scores, score_thr, iou_threshold, max_num=-1, nms_cfg=None, score_factors=None):
    """core/post_processing/bbox_nms.py:7-94 (boxes (n,4) shared by the classes or (n,C*4) class-specific, scores (n,C+1) with a bg column).
    returns dets (k,5), labels (k,), keep (k,) indices into the score-filtered candidate list,
    and inds = flat (point*C+class) index of every candidate.  nms_cfg with type='soft_nms' selects mmcv's soft-NMS,
    nms_cfg['class_agnostic'] drops the per-class coordinate offset; `score_factors` (n,) multiply the scores AFTER the
    `score > score_thr` filter (bbox_nms.py:52-62: the threshold sees the raw scores, the NMS ranks by the product)."""
    C = multi_scores.size(1) - 1
    if multi_bboxes.shape[1] > 4:
        bboxes = multi_bboxes.view(multi_scores.size(0), -1, 4).reshape(-1, 4)
    else:
        bboxes = multi_bboxes[:, None].expand(multi_scores.size(0), C, 4).reshape(-1, 4)
    scores = multi_scores[:, :-1].reshape(-1)
    labels = torch.arange(C, dtype=torch.long).view(1, -1).expand(multi_scores.size(0), C).reshape(-1)
    valid = scores > score_thr
    if score_factors is not None:
        scores = scores * score_factors.view(-1, 1).expand(multi_scores.size(0), C).reshape(-1)
    inds = valid.nonzero(as_tuple=False).squeeze(1)
    bboxes, scores, labels = bboxes[inds], scores[inds], labels[inds]
    if bboxes.numel() == 0:
        return torch.cat([bboxes, scores[:, None]], -1), labels, inds.new_zeros(0), inds
    if nms_cfg is not None and nms_cfg.get('type', 'nms') == 'soft_nms':
        dets, keep = batched_soft_nms(bboxes, scores, labels, nms_cfg)
    else:
        dets, keep = batched_nms(bboxes, scores, labels, iou_threshold, class_agnostic=bool(nms_cfg and nms_cfg.get('class_agnostic', False)),
                                 split_thr=(nms_cfg or {}).get('split_thr', SPLIT_THR))
    if max_num > 0:
        dets, keep = dets[:max_num], keep[:max_num]
    return dets, labels[keep], keep, inds


def get_bboxes_single(pred_pts, cls_outs, img_shape, scale_factor, cfg, rescale=False, return_all=False):
    """ref:345-405 _get_bboxes_single (one level, sigmoid cls): top-k -> clamp -> pseudo boxes -> NMS."""
    scores = cls_outs.sigmoid()
    nms_pre = cfg['nms_pre']
    topk_inds = None
    pts = pred_pts
    if 0 < nms_pre < scores.shape[0]:
        max_scores, _ = scores.max(dim=1)
        _, topk_inds = max_scores.topk(nms_pre)
        scores = scores[topk_inds, :]
        pts = pts[topk_inds, :]
    x = pts[:, 0].clamp(min=0, max=img_shape[1])
    y = pts[:, 1].clamp(min=0, max=img_shape[0])
    pts = torch.stack([x, y], dim=-1)
    if rescale:
        pts = pts / pts.new_tensor(scale_factor[:2])
    scores_bg = torch.cat([scores, scores.new_zeros(scores.shape[0], 1)], dim=1)
    wh = pts.new_tensor(cfg['pseudo_wh'])
    boxes = torch.cat([pts - wh / 2, pts + wh / 2], dim=-1)
    dets, labels, keep, inds = multiclass_nms(boxes, scores_bg, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    cxcy = torch.stack([(dets[:, 0] + dets[:, 2]) / 2, (dets[:, 1] + dets[:, 3]) / 2], dim=-1)
    out = torch.cat([cxcy, dets[:, 4:5]], dim=1)
    if return_all:
        return out, labels, dict(topk_inds=topk_inds, cand_inds=inds, keep=keep, boxes=boxes, scores=scores)
    return out, labels


def p2p_get_bboxes(cls_out, pts_out, img_metas, cfg, rescale=False):
    """ref:330-343: per image result (pseudo box (m,5), labels (m,))."""
    _, pred, _, cls = pred_points(cls_out, pts_out, img_metas, cfg)
    res = []
    wh = pred.new_tensor(cfg['pseudo_wh'])
    for b, m in enumerate(img_metas):
        ps, labels = get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, rescale)
        res.append((torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], dim=-1), labels))
    return res


# ----------------------------------------------------------------------------------------------
# test-time augmentation / cropped-tile merge (ref:487-572)
# ----------------------------------------------------------------------------------------------
def bbox_flip(bboxes, img_shape, direction='horizontal'):
    """core/bbox/transforms.py:5-31."""
    assert bboxes.shape[-1] % 4 == 0 and direction in ('horizontal', 'vertical', 'diagonal')
    f = bboxes.clone()
    if direction in ('horizontal', 'diagonal'):
        f[..., 0::4] = img_shape[1] - bboxes[..., 2::4]
        f[..., 2::4] = img_shape[1] - bboxes[..., 0::4]
    if direction in ('vertical', 'diagonal'):
        f[..., 1::4] = img_shape[0] - bboxes[..., 3::4]
        f[..., 3::4] = img_shape[0] - bboxes[..., 1::4]
    return f


def bbox_mapping_back(bboxes, img_shape, scale_factor, flip, flip_direction, tile_offset=None):
    """core/bbox/transforms.py:62-85 (with the reference's tile_offset extension)."""
    nb = bbox_flip(bboxes, img_shape, flip_direction) if flip else bboxes
    nb = nb.view(-1, 4) / nb.new_tensor(scale_factor)
    if tile_offset is not None:
        dx, dy = tile_offset
        nb[:, [0, 2]] += dx
        nb[:, [1, 3]] += dy
    return nb.view(bboxes.shape)


def aug_test_bboxes(aug_outs, aug_img_metas, cfg, rescale=False):
    """ref:487-572 P2PHead.aug_test_bboxes + dense_test_mixins.py:173-204 merge_aug_bboxes, AFTER `self.forward(x)`:
    aug_outs = [(cls_out (1,C,H,W), pts_out (1,2k,H,W))] per augmentation / tile, aug_img_metas = [[meta]] per augmentation.
    Per aug: get_bboxes with NMS (not rescaled) -> scatter the kept scores into an (m, Ncls) matrix (ref:534-535) -> map the boxes
    back (flip / scale / tile_offset) -> concat -> bg column -> SECOND multiclass_nms (ref:556-562) -> un-rescale unless `rescale`."""
    C = cfg['num_classes']
    aug_b, aug_s = [], []
    for (cls_out, pts_out), metas in zip(aug_outs, aug_img_metas):
        assert len(metas) == 1
        boxes5, labels = p2p_get_bboxes(cls_out, pts_out, metas, cfg, rescale=False)[0]
        sc = boxes5.new_full((boxes5.shape[0], C), 0)
        sc[torch.arange(boxes5.shape[0]), labels] = boxes5[:, 4]
        m = metas[0]
        aug_b.append(bbox_mapping_back(boxes5[:, :4], m['img_shape'], m['scale_factor'], m['flip'], m['flip_direction'],
                                       m.get('tile_offset', None)))
        aug_s.append(sc)
    mb, ms = torch.cat(aug_b, dim=0), torch.cat(aug_s, dim=0)
    ms = torch.cat([ms, ms.new_zeros(ms.shape[0], 1)], dim=1)
    dets, labels, keep, inds = multiclass_nms(mb, ms, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    if not rescale:
        dets = dets.clone()
        dets[:, :4] *= dets.new_tensor(aug_img_metas[0][0]['scale_factor'])
    return [(dets, labels)], dict(merged_boxes=mb, merged_scores=ms, keep=keep, cand_inds=inds)


# ----------------------------------------------------------------------------------------------
# PointAssigner (RepPoints style; the reference's own golden vectors: tests/test_utils/test_assigner.py:155-194)
# ----------------------------------------------------------------------------------------------
def point_assigner(points, gt_bboxes, scale=4, pos_num=3):
    """core/bbox/assigners/point_assigner.py:23-133 -> assigned_gt_inds (N,) int64 (0 = bg, j+1 = gt j)."""
    N, n = points.shape[0], gt_bboxes.shape[0]
    if n == 0 or N == 0:
        return points.new_full((N,), 0, dtype=torch.long)
    xy, st = points[:, :2], points[:, 2]
    lvl = torch.log2(st).int()
    lmin, lmax = lvl.min(), lvl.max()
    gxy = (gt_bboxes[:, :2] + gt_bboxes[:, 2:]) / 2
    gwh = (gt_bboxes[:, 2:] - gt_bboxes[:, :2]).clamp(min=1e-6)
    glvl = ((torch.log2(gwh[:, 0] / scale) + torch.log2(gwh[:, 1] / scale)) / 2).int()
    glvl = torch.clamp(glvl, min=lmin, max=lmax)
    out = points.new_zeros((N,), dtype=torch.long)
    best = points.new_full((N,), float('inf'))
    rng = torch.arange(N)
    for j in range(n):
        m = glvl[j] == lvl
        pidx = rng[m]
        d = ((xy[m, :] - gxy[[j], :]) / gwh[[j], :]).norm(dim=1)
        md, mi = torch.topk(d, pos_num, largest=False)
        sel = pidx[mi]
        less = md < best[sel]
        sel = sel[less]
        out[sel] = j + 1
        best[sel] = md[less]
    return out
