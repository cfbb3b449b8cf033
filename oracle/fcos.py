"""Functional torch-CPU restatement of the reference FCOSHead (test infrastructure).  Line numbers refer to TOV_mmdetection/mmdet:
  forward        models/dense_heads/fcos_head.py:131-160 (towers: anchor_free_head.py:88-140, mmcv ConvModule conv -> GN -> ReLU)
  points         fcos_head.py:472-482 over anchor_free_head.py:288-300
  targets        fcos_head.py:484-627 (get_targets, _get_target_single), centerness_target 629-648
  loss           fcos_head.py:163-260 with FocalLoss (losses/focal_loss.py:11-56), IoULoss / GIoULoss (losses/iou_loss.py:14-34, 87-101,
                 223-260, 330-365), aligned bbox_overlaps (core/bbox/iou_calculators/iou2d_calculator.py:213-260), CrossEntropyLoss
                 (losses/cross_entropy_loss.py:42-89), reduce_mean on one process (core/utils/dist_utils.py:63-69)
  get_bboxes     fcos_head.py:263-470, get_k_for_topk (core/export/onnx_helper.py:45-78), distance2bbox (core/bbox/transforms.py:144-187),
                 multiclass_nms (oracle.p2p, core/post_processing/bbox_nms.py:7-94)
  aug_test       models/dense_heads/dense_test_mixins.py:38-108, merge_aug_bboxes 173-204 (bbox_mapping_back with tile_offset)
Seeded inputs of the golden cases (tests/golden/fcos_*.npz) are made here from the CPU generator, so the fixtures store no inputs."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.p2p import multiclass_nms
from oracle.tile_test import bbox_mapping_back

INF = 1e8


# ---------------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------------
def tower(x, w, prefix, n):
    for i in range(n):
        x = F.conv2d(x, w[f'{prefix}.{i}.conv.weight'], None, padding=1)
        x = F.relu(F.group_norm(x, 32, w[f'{prefix}.{i}.gn.weight'], w[f'{prefix}.{i}.gn.bias']))
    return x


def forward(feats, w, cfg, training):
    """fcos_head.py:131-160 per level -> (cls_scores, bbox_preds, centernesses)"""
    cls, reg, ctr = [], [], []
    for l, (x, s) in enumerate(zip(feats, cfg['strides'])):
        fc, fr = tower(x, w, 'cls_convs', cfg['stacked_convs']), tower(x, w, 'reg_convs', cfg['stacked_convs'])
        cls.append(F.conv2d(fc, w['conv_cls.weight'], w['conv_cls.bias'], padding=1))
        b = F.conv2d(fr, w['conv_reg.weight'], w['conv_reg.bias'], padding=1)
        ctr.append(F.conv2d(fr if cfg.get('centerness_on_reg') else fc, w['conv_centerness.weight'], w['conv_centerness.bias'], padding=1))
        b = (b * w[f'scales.{l}.scale']).float()
        if cfg.get('norm_on_bbox'):
            b = F.relu(b)
            if not training:
                b = b * s
        else:
            b = b.exp()
        reg.append(b)
    return cls, reg, ctr


def points(featmap_sizes, strides, device='cpu'):
    out = []
    for (h, w), s in zip(featmap_sizes, strides):
        y, x = torch.meshgrid(torch.arange(h, device=device).float(), torch.arange(w, device=device).float(), indexing='ij')
        out.append(torch.stack((x.reshape(-1) * s, y.reshape(-1) * s), dim=-1) + s // 2)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# targets
# ---------------------------------------------------------------------------------------------------------------------------
def target_single(gt, gl, pts, ranges, npl, cfg):
    """fcos_head.py:552-627"""
    C = cfg['num_classes']
    P, G = pts.size(0), gl.size(0)
    if G == 0:
        return gl.new_full((P,), C), gt.new_zeros((P, 4))
    areas = ((gt[:, 2] - gt[:, 0]) * (gt[:, 3] - gt[:, 1]))[None].repeat(P, 1)
    rr = ranges[:, None, :].expand(P, G, 2)
    g = gt[None].expand(P, G, 4)
    xs, ys = pts[:, 0][:, None].expand(P, G), pts[:, 1][:, None].expand(P, G)
    bt = torch.stack((xs - g[..., 0], ys - g[..., 1], g[..., 2] - xs, g[..., 3] - ys), -1)
    if cfg.get('center_sampling'):
        cx, cy = (g[..., 0] + g[..., 2]) / 2, (g[..., 1] + g[..., 3]) / 2
        st = cx.new_zeros(cx.shape)
        b0 = 0
        for l, n in enumerate(npl):
            st[b0:b0 + n] = cfg['strides'][l] * cfg.get('center_sample_radius', 1.5)
            b0 += n
        xmin, ymin, xmax, ymax = cx - st, cy - st, cx + st, cy + st
        cg = torch.stack((torch.where(xmin > g[..., 0], xmin, g[..., 0]), torch.where(ymin > g[..., 1], ymin, g[..., 1]),
                          torch.where(xmax > g[..., 2], g[..., 2], xmax), torch.where(ymax > g[..., 3], g[..., 3], ymax)), -1)
        inside = torch.stack((xs - cg[..., 0], ys - cg[..., 1], cg[..., 2] - xs, cg[..., 3] - ys), -1).min(-1)[0] > 0
    else:
        inside = bt.min(-1)[0] > 0
    mx = bt.max(-1)[0]
    in_range = (mx >= rr[..., 0]) & (mx <= rr[..., 1])
    areas[inside == 0] = INF
    areas[in_range == 0] = INF
    min_area, idx = areas.min(dim=1)
    labels = gl[idx]
    labels[min_area == INF] = C
    return labels, bt[range(P), idx]


def get_targets(pts, gts, gls, cfg):
    """fcos_head.py:484-550 -> per level labels (B*HW,), bbox_targets (B*HW, 4)"""
    L = len(pts)
    ranges = torch.cat([pts[i].new_tensor(cfg['regress_ranges'][i])[None].expand_as(pts[i]) for i in range(L)])
    cp = torch.cat(pts)
    npl = [p.size(0) for p in pts]
    res = [target_single(g, lab, cp, ranges, npl, cfg) for g, lab in zip(gts, gls)]
    labs = [r[0].split(npl, 0) for r in res]
    bts = [r[1].split(npl, 0) for r in res]
    out_l, out_t = [], []
    for i in range(L):
        out_l.append(torch.cat([lb[i] for lb in labs]))
        t = torch.cat([b[i] for b in bts])
        if cfg.get('norm_on_bbox'):
            t = t / cfg['strides'][i]
        out_t.append(t)
    return out_l, out_t


def centerness_target(t):
    lr, tb = t[:, [0, 2]], t[:, [1, 3]]
    if len(lr) == 0:
        return torch.sqrt(lr[..., 0])
    return torch.sqrt((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) * (tb.min(dim=-1)[0] / tb.max(dim=-1)[0]))


# ---------------------------------------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------------------------------------
def distance2bbox(p, d, max_shape=None):
    b = torch.stack([p[..., 0] - d[..., 0], p[..., 1] - d[..., 1], p[..., 0] + d[..., 2], p[..., 1] + d[..., 3]], -1)
    if max_shape is not None:
        ms = b.new_tensor(max_shape)[..., :2]
        mxy = torch.cat([ms, ms], dim=-1).flip(-1).unsqueeze(-2)
        b = torch.where(b < b.new_tensor(0), b.new_tensor(0), b)
        b = torch.where(b > mxy, mxy, b)
    return b


def overlaps_aligned(b1, b2, mode='iou', eps=1e-6):
    a1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    a2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt, rb = torch.max(b1[..., :2], b2[..., :2]), torch.min(b1[..., 2:], b2[..., 2:])
    wh = (rb - lt).clamp(min=0)
    ov = wh[..., 0] * wh[..., 1]
    union = torch.max(a1 + a2 - ov, union_eps := a1.new_tensor([eps]))
    ious = ov / union
    if mode == 'iou':
        return ious
    ewh = (torch.max(b1[..., 2:], b2[..., 2:]) - torch.min(b1[..., :2], b2[..., :2])).clamp(min=0)
    ea = torch.max(ewh[..., 0] * ewh[..., 1], union_eps)
    return ious - (ea - union) / ea


def focal_sum(x, labels, gamma, alpha):
    C = x.size(1)
    t = F.one_hot(labels, num_classes=C + 1)[:, :C].type_as(x)
    p = x.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    fw = (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    return (F.binary_cross_entropy_with_logits(x, t, reduction='none') * fw).sum()


def loss(cls_scores, bbox_preds, centernesses, gts, gls, cfg):
    """fcos_head.py:163-260 on one process -> dict(loss_cls, loss_bbox, loss_centerness), targets"""
    C = cfg['num_classes']
    sizes = [c.shape[-2:] for c in cls_scores]
    pts = points(sizes, cfg['strides'], cls_scores[0].device)
    labels, bts = get_targets(pts, gts, gls, cfg)
    B = cls_scores[0].size(0)
    fc = torch.cat([c.permute(0, 2, 3, 1).reshape(-1, C) for c in cls_scores])
    fb = torch.cat([b.permute(0, 2, 3, 1).reshape(-1, 4) for b in bbox_preds])
    fk = torch.cat([k.permute(0, 2, 3, 1).reshape(-1) for k in centernesses])
    fl, ft = torch.cat(labels), torch.cat(bts)
    fp = torch.cat([p.repeat(B, 1) for p in pts])
    pos = ((fl >= 0) & (fl < C)).nonzero().reshape(-1)
    num_pos = max(torch.tensor(len(pos), dtype=torch.float), 1.0)
    lc = cfg['loss_cls']
    loss_cls = lc.get('loss_weight', 1.0) * (focal_sum(fc, fl, lc.get('gamma', 2.0), lc.get('alpha', 0.25)) / num_pos)
    pb, pk, pt = fb[pos], fk[pos], ft[pos]
    ctr_t = centerness_target(pt)
    denorm = max(ctr_t.sum().detach(), 1e-6)
    lb, lk = cfg['loss_bbox'], cfg['loss_centerness']
    if len(pos) > 0:
        pp = fp[pos]
        db, dt = distance2bbox(pp, pb), distance2bbox(pp, pt)
        if not torch.any(ctr_t > 0):
            loss_bbox = (db * ctr_t[:, None]).sum()
        else:
            if lb['type'] == 'IoULoss':
                ious = overlaps_aligned(db, dt).clamp(min=lb.get('eps', 1e-6))
                l = 1 - ious if lb.get('linear', False) else -ious.log()
            else:
                l = 1 - overlaps_aligned(db, dt, 'giou', lb.get('eps', 1e-6))
            loss_bbox = lb.get('loss_weight', 1.0) * ((l * ctr_t).sum() / denorm)
        lkx = F.binary_cross_entropy_with_logits(pk, ctr_t, reduction='none')
        loss_ctr = lk.get('loss_weight', 1.0) * (lkx.sum() / num_pos)
    else:
        loss_bbox, loss_ctr = pb.sum(), pk.sum()
    return dict(loss_cls=loss_cls, loss_bbox=loss_bbox, loss_centerness=loss_ctr), dict(labels=labels, bbox_targets=bts)


# ---------------------------------------------------------------------------------------------------------------------------
# get_bboxes / aug_test
# ---------------------------------------------------------------------------------------------------------------------------
def decode(cls_scores, bbox_preds, centernesses, metas, cfg, test_cfg, rescale=False):
    """fcos_head.py:328-431 up to the NMS -> boxes (B,R,4), scores (B,R,C), centerness (B,R), topk (per level (B,k) or None)"""
    C = cfg['num_classes']
    B = cls_scores[0].shape[0]
    pts = points([c.shape[-2:] for c in cls_scores], cfg['strides'], cls_scores[0].device)
    nms_pre = test_cfg.get('nms_pre', -1)
    mb, ms, mk, tk = [], [], [], []
    for c, b, k, p in zip(cls_scores, bbox_preds, centernesses, pts):
        s = c.permute(0, 2, 3, 1).reshape(B, -1, C).sigmoid()
        k = k.permute(0, 2, 3, 1).reshape(B, -1).sigmoid()
        b = b.permute(0, 2, 3, 1).reshape(B, -1, 4)
        p = p.expand(B, -1, 2)
        n = nms_pre if 0 < nms_pre < b.shape[1] else -1
        inds = None
        if n > 0:
            mx, _ = (s * k[..., None]).max(-1)
            _, inds = mx.topk(n)
            bi = torch.arange(B, device=inds.device).view(-1, 1).expand_as(inds).long()
            p, b, s, k = p[bi, inds, :], b[bi, inds, :], s[bi, inds, :], k[bi, inds]
        tk.append(inds)
        mb.append(distance2bbox(p, b, max_shape=[m['img_shape'] for m in metas]))
        ms.append(s)
        mk.append(k)
    bb = torch.cat(mb, dim=1)
    if rescale:
        bb = bb / bb.new_tensor(np.array([m['scale_factor'] for m in metas])).unsqueeze(1)
    return bb, torch.cat(ms, dim=1), torch.cat(mk, dim=1), tk


def nms_dets(boxes, scores, factors, test_cfg):
    """multiclass_nms with score_factors of one image -> dets (k, 5), labels (k,), keep"""
    padded = torch.cat([scores, scores.new_zeros(scores.shape[0], 1)], -1)
    d, l, keep, _ = multiclass_nms(boxes, padded, test_cfg['score_thr'], test_cfg['nms']['iou_threshold'], test_cfg['max_per_img'],
                                   score_factors=factors)
    return d, l, keep


def get_bboxes(cls_scores, bbox_preds, centernesses, metas, cfg, test_cfg, rescale=False):
    bb, sc, kk, tk = decode(cls_scores, bbox_preds, centernesses, metas, cfg, test_cfg, rescale)
    return [nms_dets(bb[b], sc[b], kk[b], test_cfg)[:2] for b in range(bb.shape[0])], tk


def aug_test_bboxes(aug_maps, metas, cfg, test_cfg, rescale=False):
    """dense_test_mixins.py:38-108: aug_maps[a] = the (cls, reg, ctr) level lists of aug a, metas[a] = [meta]"""
    boxes, scores, facs = [], [], []
    for (c, r, k), m in zip(aug_maps, metas):
        bb, sc, kk, _ = decode(c, r, k, m, cfg, test_cfg, False)
        boxes.append(bbox_mapping_back(bb[0], m[0]))
        scores.append(sc[0])
        facs.append(kk[0])
    d, l, _ = nms_dets(torch.cat(boxes), torch.cat(scores), torch.cat(facs), test_cfg)
    if not rescale:
        d = d.clone()
        d[:, :4] *= d.new_tensor(metas[0][0]['scale_factor'])
    return d, l, sum(len(b) for b in boxes)


# ---------------------------------------------------------------------------------------------------------------------------
# golden cases
# ---------------------------------------------------------------------------------------------------------------------------
TINY = dict(num_classes=1, regress_ranges=((-1, 16), (16, 32), (32, 64), (64, 128), (128, INF)), strides=[8, 16, 32, 64, 128],
            loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0), loss_bbox=dict(type='IoULoss', loss_weight=1.0),
            loss_centerness=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0))
TINY_TEST = dict(nms_pre=2000, min_bbox_size=0, score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=1000)
COCO = dict(TINY, num_classes=80, regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)))
COCO_TEST = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=100)
OPTIONS = dict(COCO, num_classes=3, strides=[4, 8, 16, 32, 64], center_sampling=True, center_sample_radius=1.5, norm_on_bbox=True,
               centerness_on_reg=True, loss_bbox=dict(type='GIoULoss', loss_weight=1.0))

# name -> head cfg, test cfg, batch, image (h, w), padded (h, w) per image, towers run by the reference, GTs per image, seed
CASES = {
    'tinyperson': dict(head=TINY, test=TINY_TEST, img=[(512, 640), (512, 640)], pad=(512, 640), towers=True, n_gt=[24, 24], seed=11),
    'coco80': dict(head=COCO, test=COCO_TEST, img=[(320, 416), (288, 400)], pad=(320, 416), towers=False, n_gt=[9, 6], seed=12,
                   rescale=True, scale_factor=[[0.65, 0.65, 0.65, 0.65], [0.5, 0.52, 0.5, 0.52]]),
    'options': dict(head=OPTIONS, test=dict(COCO_TEST, nms_pre=300), img=[(128, 160), (128, 160)], pad=(128, 160), towers=True,
                    n_gt=[10, 0], seed=13),
    'no_pos': dict(head=TINY, test=TINY_TEST, img=[(128, 160), (128, 160)], pad=(128, 160), towers=False, n_gt=[0, 1], seed=14,
                   far_gt=True),
}
TILE_OFFSETS = [(x, y) for y in (0, 412, 568) for x in (0, 540, 1080, 1280)]      # 1920 x 1080 in 640 x 512 tiles, 100 px overlap


def head_kwargs(name):
    h = dict(CASES[name]['head'])
    return dict(h, in_channels=256, feat_channels=256, stacked_convs=4, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                test_cfg=dict(CASES[name]['test']))


def featmap_sizes(pad, strides):
    return [(math.ceil(pad[0] / s), math.ceil(pad[1] / s)) for s in strides]


def weights(gen, num_classes, C=256, n=4, n_lvl=5):
    """state_dict-shaped weights; towers scaled to keep activations O(1), output convs at the reference's Normal(0.01)"""
    w = {}
    for p in ('cls_convs', 'reg_convs'):
        for i in range(n):
            w[f'{p}.{i}.conv.weight'] = torch.randn(C, C, 3, 3, generator=gen) * (1.4 / math.sqrt(C * 9))
            w[f'{p}.{i}.gn.weight'] = 1 + 0.1 * torch.randn(C, generator=gen)
            w[f'{p}.{i}.gn.bias'] = 0.1 * torch.randn(C, generator=gen)
    w['conv_cls.weight'] = torch.randn(num_classes, C, 3, 3, generator=gen) * 0.05
    w['conv_cls.bias'] = torch.full((num_classes,), -math.log(99.0))
    w['conv_reg.weight'] = torch.randn(4, C, 3, 3, generator=gen) * 0.02
    w['conv_reg.bias'] = torch.full((4,), 1.0)
    w['conv_centerness.weight'] = torch.randn(1, C, 3, 3, generator=gen) * 0.05
    w['conv_centerness.bias'] = torch.zeros(1)
    for l in range(n_lvl):
        w[f'scales.{l}.scale'] = torch.tensor(1.0 + 0.1 * l)
    return w


def gt_boxes(gen, n, img, tiny_specials=False, far=False):
    h, w = img
    if far:
        return torch.tensor([[2000., 2000., 2012., 2010.]] * n), torch.zeros(n, dtype=torch.long)
    wh = torch.exp(torch.rand(n, 2, generator=gen) * math.log(12.0)) * 4.0          # 4 .. 48 px
    c = torch.rand(n, 2, generator=gen) * torch.tensor([w, h])
    b = torch.cat([c - wh / 2, c + wh / 2], 1)
    if tiny_specials and n >= 4:
        b[1] = b[0]                                   # two identical GTs: the area tie goes to the first
        b[2] = torch.tensor([100., 60., 116., 70.])   # at the stride-8 point (108, 68): left = 8, right = 8, top 8, bottom 2
        b[3] = torch.tensor([-12., 200., 10., 230.])  # partly outside the image
        b[4] = torch.tensor([228., 300., 260., 316.]) # at the point (244, 308): max distance 16, the (-1, 16) / (16, 32) boundary
    return b.float(), torch.zeros(n, dtype=torch.long)


def case_inputs(name):
    c = CASES[name]
    gen = torch.Generator().manual_seed(c['seed'])
    hc = c['head']
    B = len(c['img'])
    sizes = featmap_sizes(c['pad'], hc['strides'])
    out = dict(sizes=sizes)
    out['weights'] = weights(gen, hc['num_classes'])
    out['feats'] = [torch.randn(B, 256, h, w, generator=gen) for h, w in sizes]
    gts, gls = [], []
    for b in range(B):
        g, l = gt_boxes(gen, c['n_gt'][b], c['img'][b], tiny_specials=name == 'tinyperson', far=c.get('far_gt', False))
        if hc['num_classes'] > 1 and len(l):
            l = torch.randint(0, hc['num_classes'], (len(l),), generator=gen)
        gts.append(g)
        gls.append(l)
    out['gt_bboxes'], out['gt_labels'] = gts, gls
    sf = c.get('scale_factor', [[1.0] * 4] * B)
    out['img_metas'] = [dict(img_shape=(h, w, 3), pad_shape=c['pad'] + (3,), ori_shape=(h, w, 3), scale_factor=np.array(sf[b], np.float32),
                             flip=False, flip_direction=None) for b, (h, w) in enumerate(c['img'])]
    if not c['towers']:       # the output maps themselves: logits and exp-scaled distances of a plausible spread
        C = hc['num_classes']
        out['maps'] = ([torch.randn(B, C, h, w, generator=gen) * 1.5 - 3.0 for h, w in sizes],
                       [torch.exp(torch.randn(B, 4, h, w, generator=gen) * 0.6) * s * 2 for (h, w), s in zip(sizes, hc['strides'])],
                       [torch.randn(B, 1, h, w, generator=gen) for h, w in sizes])
    return out


def tile_case(name):
    """'tiles': 12 tiles of one 1920 x 1080 image; 'flip_scale': one 320 x 400 image as itself, flipped, and scaled by 1.5.
    Per aug the seed of its maps, its meta and its feature map sizes."""
    hc = TINY
    augs = []
    if name == 'tiles':
        for i, off in enumerate(TILE_OFFSETS):
            augs.append(dict(seed=100 + i, meta=dict(img_shape=(512, 640, 3), pad_shape=(512, 640, 3), ori_shape=(1080, 1920, 3),
                                                     scale_factor=np.ones(4, np.float32), flip=False, flip_direction=None,
                                                     tile_offset=off), sizes=featmap_sizes((512, 640), hc['strides'])))
    else:
        for i, (flip, s) in enumerate(((False, 1.0), (True, 1.0), (False, 1.5))):
            h, w = int(320 * s), int(400 * s)
            augs.append(dict(seed=200 + i, meta=dict(img_shape=(h, w, 3), pad_shape=(h, w, 3), ori_shape=(320, 400, 3),
                                                     scale_factor=np.array([s] * 4, np.float32), flip=flip,
                                                     flip_direction='horizontal' if flip else None),
                             sizes=featmap_sizes((h, w), hc['strides'])))
    return augs


def aug_maps(aug):
    gen = torch.Generator().manual_seed(aug['seed'])
    sizes = aug['sizes']
    return ([torch.randn(1, 1, h, w, generator=gen) * 1.5 - 2.5 for h, w in sizes],
            [torch.exp(torch.randn(1, 4, h, w, generator=gen) * 0.5) * s for (h, w), s in zip(sizes, TINY['strides'])],
            [torch.randn(1, 1, h, w, generator=gen) for h, w in sizes])


def fcos_rows(hw, nms_pre):
    """rows a level of hw points keeps per image (get_k_for_topk)"""
    return nms_pre if 0 < nms_pre < hw else hw
