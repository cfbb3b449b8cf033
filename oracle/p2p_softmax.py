"""ORACLE (test infrastructure, NOT product code) — P2PHead with CrossEntropyLoss in softmax mode and with class_weight.

Follows /root/reference/TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py:63-67 (num_cls_out = num_classes + 1 when
use_sigmoid is False), :220-232 (loss_single), :355-405 (_get_bboxes_single: softmax scores, top-k on the foreground columns, no
background padding) and :487-572 (aug_test_bboxes: an (n, num_classes) score matrix and, in softmax mode, no background column
before multiclass_nms, so the last real class is taken for the background), and mmdet/models/losses/cross_entropy_loss.py:9-39
(cross_entropy with class_weight) and :58-91 (binary_cross_entropy: class_weight passed as pos_weight).
Everything else (pred_points, Hungarian targets, NMS, the regression losses) is oracle/p2p.py and oracle/p2p_defaults.py, used as is.
Only tests/ and oracle/make_golden_p2p_softmax.py import this.
"""
import math

import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_defaults as odef
from oracle.synth import sample_points


def softmax_cfg(use_sigmoid=False, class_weight=None, **over):
    """oracle/p2p_defaults.py's cfg (the reference defaults) with CrossEntropyLoss(use_sigmoid, class_weight)."""
    cfg = odef.reference_defaults_cfg(use_sigmoid=use_sigmoid, class_weight=class_weight)
    cfg.update(over)
    return cfg


def num_cls_out(cfg):
    """ref:63-67"""
    return cfg['num_classes'] if cfg.get('use_sigmoid', True) else cfg['num_classes'] + 1


def pred_points(cls_out, pts_out, img_metas, cfg):
    """oracle/p2p.py's pred_points with rows of num_cls_out logits."""
    return op2p.pred_points(cls_out, pts_out, img_metas, dict(cfg, num_classes=num_cls_out(cfg)))


def cross_entropy_elem(pred, labels, class_weight=None):
    """cross_entropy_loss.py:31: F.cross_entropy(pred, label, weight=class_weight, reduction='none'); label C = background."""
    return F.cross_entropy(pred, labels, weight=class_weight, reduction='none')


def binary_cross_entropy_elem(pred, labels, class_weight=None):
    """cross_entropy_loss.py:79-86: one-hot expansion, then binary_cross_entropy_with_logits with class_weight as pos_weight."""
    C = pred.size(1)
    t = pred.new_zeros(pred.shape)
    inds = torch.nonzero((labels >= 0) & (labels < C), as_tuple=False).squeeze(1)
    if inds.numel() > 0:
        t[inds, labels[inds]] = 1
    return F.binary_cross_entropy_with_logits(pred, t, pos_weight=class_weight, reduction='none')


def p2p_loss(cls_out, pts_out, gt_bboxes, gt_labels, img_metas, cfg, return_all=False):
    """ref:172-248 with CrossEntropyLoss (softmax or sigmoid, class_weight or None) -> dict(loss_cls=[B], loss_pts=[B]).  The
    classification loss is averaged over num_total (every proposal of the batch), the regression loss over num_total_pos."""
    assert cfg['loss_cls'] == 'CrossEntropyLoss', cfg['loss_cls']
    anchor, pred, valid, cls = pred_points(cls_out, pts_out, img_metas, cfg)
    gt_points = [(b[:, :2] + b[:, 2:]) / 2 for b in gt_bboxes]
    prop = anchor if cfg['assign_before_pred'] else pred
    tg = [op2p.target_single(prop[b][..., :2].detach(), valid[b], cls[b].detach(), gt_points[b], gt_labels[b],
                             img_metas[b]['img_shape'], cfg) for b in range(len(img_metas))]
    num_total = sum([len(t[0]) for t in tg])
    num_total_pos = sum([(t[3][..., 0] > 0).sum() for t in tg])
    cw = None if cfg.get('class_weight') is None else cls.new_tensor(cfg['class_weight'])
    loss_cls, loss_pts = [], []
    for b, (labels, lw, gpts, pw, _) in enumerate(tg):
        if cfg.get('use_sigmoid', True):
            l = binary_cross_entropy_elem(cls[b].contiguous(), labels, cw)
            l = (l * lw.view(-1, 1).expand(lw.size(0), l.size(1)).float()).sum() / num_total
        else:
            l = (cross_entropy_elem(cls[b].contiguous(), labels, cw) * lw.float()).sum() / num_total
        loss_cls.append(cfg['loss_cls_weight'] * l)
        s = pred[b][..., -1:]
        if cfg['loss_reg'] == 'MSELoss':
            r = odef.mse_elem(pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm'])
        else:
            r = op2p.smooth_l1_elem(pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm'], cfg['sl1_beta'])
        loss_pts.append(cfg['loss_reg_weight'] * ((r * pw).sum() / num_total_pos))
    out = dict(loss_cls=loss_cls, loss_pts=loss_pts)
    if return_all:
        return out, dict(targets=tg, pred=pred, valid=valid, cls=cls)
    return out


def get_bboxes_single(pred_pts, cls_outs, img_shape, scale_factor, cfg, rescale=False, return_all=False):
    """ref:355-405 _get_bboxes_single (one level, softmax cls): softmax over the C+1 columns, top-k on the foreground max, clamp,
    pseudo boxes, multiclass_nms on the C+1 columns (it drops the background column itself)."""
    scores = cls_outs.softmax(-1)
    nms_pre = cfg['nms_pre']
    topk_inds, keys = None, None
    pts = pred_pts
    if 0 < nms_pre < scores.shape[0]:
        keys, _ = scores[:, :-1].max(dim=1)
        _, topk_inds = keys.topk(nms_pre)
        scores = scores[topk_inds, :]
        pts = pts[topk_inds, :]
    x = pts[:, 0].clamp(min=0, max=img_shape[1])
    y = pts[:, 1].clamp(min=0, max=img_shape[0])
    pts = torch.stack([x, y], dim=-1)
    if rescale:
        pts = pts / pts.new_tensor(scale_factor[:2])
    wh = pts.new_tensor(cfg['pseudo_wh'])
    boxes = torch.cat([pts - wh / 2, pts + wh / 2], dim=-1)
    dets, labels, keep, inds = op2p.multiclass_nms(boxes, scores, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    cxcy = torch.stack([(dets[:, 0] + dets[:, 2]) / 2, (dets[:, 1] + dets[:, 3]) / 2], dim=-1)
    out = torch.cat([cxcy, dets[:, 4:5]], dim=1)
    if return_all:
        return out, labels, dict(topk_inds=topk_inds, keys=keys, cand_inds=inds, keep=keep, boxes=boxes, scores=scores[:, :-1])
    return out, labels


def p2p_get_bboxes(cls_out, pts_out, img_metas, cfg, rescale=False):
    """ref:330-343 in softmax mode: per image (pseudo box (m,5), labels (m,))."""
    _, pred, _, cls = pred_points(cls_out, pts_out, img_metas, cfg)
    res = []
    wh = pred.new_tensor(cfg['pseudo_wh'])
    for b, m in enumerate(img_metas):
        ps, labels = get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, rescale)
        res.append((torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], dim=-1), labels))
    return res


def aug_test_bboxes(aug_outs, aug_img_metas, cfg, rescale=False):
    """ref:487-572 in softmax mode, after `self.forward(x)` (see oracle/p2p.py's aug_test_bboxes): the per-aug detections are scattered
    into an (m, num_classes) matrix and, unlike sigmoid mode, NO background column is appended before the second multiclass_nms
    (ref:549-554), which therefore treats class C-1 as the background: it never appears in the merged detections."""
    C = cfg['num_classes']
    aug_b, aug_s = [], []
    for (cls_out, pts_out), metas in zip(aug_outs, aug_img_metas):
        assert len(metas) == 1
        boxes5, labels = p2p_get_bboxes(cls_out, pts_out, metas, cfg, rescale=False)[0]
        sc = boxes5.new_full((boxes5.shape[0], C), 0)
        sc[torch.arange(boxes5.shape[0]), labels] = boxes5[:, 4]
        m = metas[0]
        aug_b.append(op2p.bbox_mapping_back(boxes5[:, :4], m['img_shape'], m['scale_factor'], m['flip'], m['flip_direction'],
                                            m.get('tile_offset', None)))
        aug_s.append(sc)
    mb, ms = torch.cat(aug_b, dim=0), torch.cat(aug_s, dim=0)
    dets, labels, keep, inds = op2p.multiclass_nms(mb, ms, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    if not rescale:
        dets = dets.clone()
        dets[:, :4] *= dets.new_tensor(aug_img_metas[0][0]['scale_factor'])
    return [(dets, labels)], dict(merged_boxes=mb, merged_scores=ms, keep=keep, cand_inds=inds)


def inputs(seed=4267, B=2, C=256, num_classes=80, k=4, stride=8, n=12, bg_bias=3.0):
    """seeded inputs whose cls_out has k * (num_classes + 1) channels (background channel last in every anchor group): towers as
    oracle/p2p_defaults.py's inputs, foreground biases ~ N(-1, 1), background bias `bg_bias`, so that softmax scores
    spread over (0, 1) with a few dozen foreground probabilities above score_thr per image.  Image 1 has a smaller pad shape.
    CPU generator: bit-reproducible."""
    gen = torch.Generator().manual_seed(seed)
    anchors = list(odef.ANCHORS) if k == 4 else [(0., 0.)] * k
    pads = [(128, 128), (112, 120)][:B] + [(128, 128)] * max(0, B - 2)
    imgs = [(125, 126), (110, 117)][:B] + [(125, 126)] * max(0, B - 2)
    H, W = 128 // stride, 128 // stride
    C1 = num_classes + 1
    w = {}
    for prefix in ('cls_convs', 'reg_convs'):
        for i in range(4):
            w[f'{prefix}.{i}.conv.weight'] = torch.randn(C, C, 3, 3, generator=gen) * (1.4 / math.sqrt(C * 9))
            w[f'{prefix}.{i}.gn.weight'] = 1 + 0.1 * torch.randn(C, generator=gen)
            w[f'{prefix}.{i}.gn.bias'] = 0.1 * torch.randn(C, generator=gen)
    w['cls_out.weight'] = torch.randn(k * C1, C, 3, 3, generator=gen) * 0.02
    bias = -1.0 + torch.randn(k, C1, generator=gen)
    bias[:, -1] = bg_bias
    bias[:, -2] += 1.5          # the last foreground class gets detections: the softmax aug-test merge drops exactly that class
    w['cls_out.bias'] = bias.reshape(-1)
    w['reg_out.weight'] = torch.randn(2 * k, C, 3, 3, generator=gen) * 0.001
    w['reg_out.bias'] = torch.zeros(2 * k)
    x = torch.relu(torch.randn(B, C, H, W, generator=gen))
    gt_bboxes, gt_labels, img_metas = [], [], []
    for b in range(B):
        ih, iw = imgs[b]
        pts = sample_points(n, iw, ih, gen)
        gt_bboxes.append(torch.cat([pts - 8, pts + 8], dim=1))
        gt_labels.append(torch.randint(0, num_classes, (n,), generator=gen))
        img_metas.append(dict(pad_shape=pads[b] + (3,), img_shape=(ih, iw, 3), scale_factor=[1.0, 1.0, 1.0, 1.0]))
    cfgd = dict(B=B, C=C, num_classes=num_classes, stride=stride, n=n, point_anchor=anchors)
    return dict(cfgd=cfgd, x=x, weights=w, gt_bboxes=gt_bboxes, gt_labels=gt_labels, img_metas=img_metas)


def aug_inputs(cls_out, pts_out, img_metas):
    """test-time-augmentation case from one batch of head outputs: 4 "augmentations" of one image, each a (cls_out, pts_out) pair of
    ONE image and its meta: image 0 as is, image 0 with a lower background logit and a tile offset (overlapping boxes: the second NMS
    has work to do), image 1 horizontally flipped at scale 1.5, image 1 with a higher background logit, vertically flipped with a tile
    offset.  The shifts go to the background channel only: softmax is invariant under a shift of every logit, which would make the
    copies' scores equal up to rounding."""
    k = pts_out.shape[1] // 2

    def shift_bg(c, d):
        c = c.clone().reshape(c.shape[0], k, -1, *c.shape[2:])
        c[:, :, -1] += d
        return c.reshape(c.shape[0], -1, *c.shape[3:])
    def meta(b, scale, flip, direction, tile):
        m = dict(img_metas[b], scale_factor=[scale] * 4, flip=flip, flip_direction=direction)
        if tile is not None:
            m['tile_offset'] = tile
        return [m]
    outs = [(cls_out[:1], pts_out[:1]), (shift_bg(cls_out[:1], -0.8), pts_out[:1]), (cls_out[1:2], pts_out[1:2]),
            (shift_bg(cls_out[1:2], 0.9), pts_out[1:2])]
    metas = [meta(0, 1.0, False, 'horizontal', None), meta(0, 1.0, False, 'horizontal', (3, 2)),
             meta(1, 1.5, True, 'horizontal', None), meta(1, 1.0, True, 'vertical', (40, 24))]
    return outs, metas
