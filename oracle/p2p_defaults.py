"""ORACLE (test infrastructure, NOT product code) — P2PHead at the reference class's OWN defaults.

Follows /root/reference/TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py:25-45 (defaults: four point anchors per cell,
pts_gamma 100/8, reg_norm 1/8, CrossEntropyLoss(use_sigmoid=True), MSELoss(loss_weight=2e-4)), :172-248 (loss, loss_single),
mmdet/models/losses/cross_entropy_loss.py:42-89 (_expand_onehot_labels, binary_cross_entropy) and mse_loss.py:9-48.
Everything else (pred_points, Hungarian targets, focal / smooth-L1, get_bboxes) is oracle/p2p.py, used as is.
Only tests/ and oracle/make_golden_p2p_defaults.py import this.
"""
import math

import torch
import torch.nn.functional as F

from oracle import p2p as op2p
from oracle.synth import sample_points

ANCHORS = [(-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)]


def reference_defaults_cfg(**over):
    """oracle/p2p.py's cfg at the reference defaults (ref:25-45); assigner / test settings as op2p.default_cfg.
    'loss_cls' selects FocalLoss or CrossEntropyLoss, 'loss_reg' SmoothL1Loss or MSELoss."""
    cfg = op2p.default_cfg(point_anchor=list(ANCHORS), pts_gamma=100. / 8, reg_norm=1. / 8,
                           loss_cls='CrossEntropyLoss', loss_cls_weight=1.0, loss_reg='MSELoss', loss_reg_weight=2e-4)
    cfg.update(over)
    return cfg


def sigmoid_bce_elem(pred, target_labels):
    """cross_entropy_loss.py:42-89 binary_cross_entropy (class_weight=None) elementwise part: _expand_onehot_labels (a label outside
    [0, C), e.g. the background label C, is an all-zero row), then F.binary_cross_entropy_with_logits(reduction='none')."""
    C = pred.size(1)
    t = pred.new_zeros(pred.shape)
    inds = torch.nonzero((target_labels >= 0) & (target_labels < C), as_tuple=False).squeeze(1)
    if inds.numel() > 0:
        t[inds, target_labels[inds]] = 1
    return F.binary_cross_entropy_with_logits(pred, t, reduction='none')


def mse_elem(pred, target):
    """mse_loss.py:9-12"""
    return F.mse_loss(pred, target, reduction='none')


def p2p_loss(cls_out, pts_out, gt_bboxes, gt_labels, img_metas, cfg, return_all=False):
    """ref:172-248 with any of the two classification / regression losses -> dict(loss_cls=[B], loss_pts=[B]).
    loss_single (ref:218-240): CrossEntropyLoss is averaged over num_total = every proposal of the batch, FocalLoss over
    num_total_pos; both regression losses over num_total_pos."""
    anchor, pred, valid, cls = op2p.pred_points(cls_out, pts_out, img_metas, cfg)
    gt_points = [(b[:, :2] + b[:, 2:]) / 2 for b in gt_bboxes]
    prop = anchor if cfg['assign_before_pred'] else pred
    tg = [op2p.target_single(prop[b][..., :2].detach(), valid[b], cls[b].detach(), gt_points[b], gt_labels[b],
                             img_metas[b]['img_shape'], cfg) for b in range(len(img_metas))]
    num_total = sum([len(t[0]) for t in tg])
    num_total_pos = sum([(t[3][..., 0] > 0).sum() for t in tg])
    cls_type, reg_type = cfg.get('loss_cls', 'FocalLoss'), cfg.get('loss_reg', 'SmoothL1Loss')
    assert cls_type in ('FocalLoss', 'CrossEntropyLoss') and reg_type in ('SmoothL1Loss', 'MSELoss'), (cls_type, reg_type)
    loss_cls, loss_pts = [], []
    for b, (labels, lw, gpts, pw, _) in enumerate(tg):
        if cls_type == 'CrossEntropyLoss':
            l = sigmoid_bce_elem(cls[b].contiguous(), labels)
            l = (l * lw.view(-1, 1).expand(lw.size(0), l.size(1)).float()).sum() / num_total
        else:
            l = op2p.sigmoid_focal_loss_elem(cls[b].contiguous(), labels, cfg['focal_gamma'], cfg['focal_alpha'])
            l = (l * lw.view(-1, 1)).sum() / num_total_pos
        loss_cls.append(cfg['loss_cls_weight'] * l)
        s = pred[b][..., -1:]
        if reg_type == 'MSELoss':
            r = mse_elem(pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm'])
        else:
            r = op2p.smooth_l1_elem(pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm'], cfg['sl1_beta'])
        loss_pts.append(cfg['loss_reg_weight'] * ((r * pw).sum() / num_total_pos))
    out = dict(loss_cls=loss_cls, loss_pts=loss_pts)
    if return_all:
        return out, dict(targets=tg, pred=pred, valid=valid, cls=cls)
    return out


def inputs(seed=8086, B=2, C=256, num_classes=80, stride=8, n=12):
    """seeded inputs at the default geometry (cls_out has 4 x num_classes channels): state_dict-shaped weights (GroupNorm towers,
    cls_out logits ~ N(-4.6, 1.5), reg_out offsets of a few pixels at pts_gamma 100/8), a ReLU feature map and GT points.  Image 1
    has a smaller pad shape than image 0, so its valid flags cut the map.  CPU generator: bit-reproducible."""
    gen = torch.Generator().manual_seed(seed)
    k = len(ANCHORS)
    pads = [(128, 128), (112, 120)][:B] + [(128, 128)] * max(0, B - 2)
    imgs = [(125, 126), (110, 117)][:B] + [(125, 126)] * max(0, B - 2)
    H, W = 128 // stride, 128 // stride
    w = {}
    for prefix in ('cls_convs', 'reg_convs'):
        for i in range(4):
            w[f'{prefix}.{i}.conv.weight'] = torch.randn(C, C, 3, 3, generator=gen) * (1.4 / math.sqrt(C * 9))
            w[f'{prefix}.{i}.gn.weight'] = 1 + 0.1 * torch.randn(C, generator=gen)
            w[f'{prefix}.{i}.gn.bias'] = 0.1 * torch.randn(C, generator=gen)
    w['cls_out.weight'] = torch.randn(k * num_classes, C, 3, 3, generator=gen) * 0.045
    w['cls_out.bias'] = torch.full((k * num_classes,), -math.log(99.0)) + 0.3 * torch.randn(k * num_classes, generator=gen)
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
    cfgd = dict(B=B, C=C, num_classes=num_classes, stride=stride, n=n, point_anchor=list(ANCHORS))
    return dict(cfgd=cfgd, x=x, weights=w, gt_bboxes=gt_bboxes, gt_labels=gt_labels, img_metas=img_metas)
