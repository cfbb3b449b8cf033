"""Restatement of the bbox branch of StandardRoIHead (mmdet/models/roi_heads/standard_roi_head.py, bbox_heads/bbox_head.py,
convfc_bbox_head.py, roi_extractors/single_level_roi_extractor.py, test_mixins.py:57-155) with torch-CPU ops in the reference's order.
Test infrastructure — only tests/ and tools/ may import this.

mmcv's RoIAlign is third-party arithmetic outside the reference tree: `roi_align` restates mmcv's published CPU kernel
(roi_align_cpu.cpp: aligned=True, pool_mode='avg', pre_calc_for_bilinear_interpolate) operation by operation in fp32; it is pinned
against torchvision.ops.roi_align(aligned=True) on CPU by tests/test_roi_head_golden.py, and `RoIAlign` is the module the reference's
SingleRoIExtractor builds when oracle/make_golden_roi_head.py runs the real reference head.

Pinned: oracle/make_golden_roi_head.py runs the real reference StandardRoIHead.forward_train (+ backward) and simple_test on the seeded
CASES below, asserts that this restatement equals it and writes tests/golden/roi_head_*.npz."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import anchors as oa
from oracle import rpn_loss as orl

STRIDES = [4, 8, 16, 32]
C_FEAT, FC = 8, 32


def roi_align(feat, rois, out, spatial_scale, sampling_ratio):
    """mmcv RoIAlign(aligned=True, pool_mode='avg') on CPU: feat (B, C, H, W) fp32, rois (R, 5) -> (R, C, out, out).  Differentiable
    (the gather and the weights are torch ops); RoIs are grouped by their sample grid so each group is one vectorised pass."""
    B, C, H, W = feat.shape
    R = rois.shape[0]
    res = feat.new_zeros((R, C, out, out))
    if R == 0:
        return res
    sc = torch.tensor(spatial_scale, dtype=torch.float32)
    sw, sh = rois[:, 1] * sc - 0.5, rois[:, 2] * sc - 0.5
    rw, rh = (rois[:, 3] * sc - 0.5) - sw, (rois[:, 4] * sc - 0.5) - sh
    bw, bh = rw / out, rh / out
    gh = torch.full((R,), sampling_ratio, dtype=torch.int64) if sampling_ratio > 0 else torch.ceil(bh).long()
    gw = torch.full((R,), sampling_ratio, dtype=torch.int64) if sampling_ratio > 0 else torch.ceil(bw).long()
    p = torch.arange(out, dtype=torch.float32)
    parts = []
    for g_h, g_w in sorted(set(zip(gh.tolist(), gw.tolist()))):
        idx = ((gh == g_h) & (gw == g_w)).nonzero().squeeze(1)
        count = torch.tensor(float(max(g_h * g_w, 1)))
        acc = feat.new_zeros((idx.numel(), C, out, out))
        if g_h > 0 and g_w > 0:
            bi = rois[idx, 0].long()
            ys = (sh[idx, None] + p[None, :] * bh[idx, None])[:, :, None] + \
                ((torch.arange(g_h, dtype=torch.float32) + 0.5)[None, :] * bh[idx, None] / float(g_h))[:, None, :]     # (n, out, gh)
            xs = (sw[idx, None] + p[None, :] * bw[idx, None])[:, :, None] + \
                ((torch.arange(g_w, dtype=torch.float32) + 0.5)[None, :] * bw[idx, None] / float(g_w))[:, None, :]     # (n, out, gw)

            def axis(v, size):
                ok = ~((v < -1.0) | (v > size))
                v = torch.where(v <= 0, torch.zeros_like(v), v)
                lo = v.long()
                top = lo >= size - 1
                lo = torch.where(top, torch.full_like(lo, size - 1), lo)
                hi = torch.where(top, lo, lo + 1)
                v = torch.where(top, lo.float(), v)
                l = v - lo.float()
                return ok, lo, hi, l, 1. - l
            oky, yl, yh, ly, hy = axis(ys, H)
            okx, xl, xh, lx, hx = axis(xs, W)
            fb = feat[bi]                                                    # (n, C, H, W)
            n = idx.numel()

            def tap(yi, xi):                                                 # yi (n, out, gh), xi (n, out, gw) -> (n, C, out, gh, out, gw)
                flat = (yi[:, :, :, None, None] * W + xi[:, None, None, :, :]).reshape(n, 1, -1).expand(n, C, -1)
                return fb.reshape(n, C, H * W).gather(2, flat).reshape(n, C, out, g_h, out, g_w)
            wy = lambda t: t[:, None, :, :, None, None]
            wx = lambda t: t[:, None, None, None, :, :]
            ok = (wy(oky) & wx(okx))
            w1, w2, w3, w4 = wy(hy) * wx(hx), wy(hy) * wx(lx), wy(ly) * wx(hx), wy(ly) * wx(lx)
            val = ((w1 * tap(yl, xl) + w2 * tap(yl, xh)) + w3 * tap(yh, xl)) + w4 * tap(yh, xh)
            val = torch.where(ok, val, torch.zeros_like(val))
            for iy in range(g_h):
                for ix in range(g_w):
                    acc = acc + val[:, :, :, iy, :, ix]
        parts.append((idx, acc / count))
    for idx, v in parts:
        res = res.index_copy(0, idx, v)
    return res


class RoIAlign(nn.Module):
    """mmcv.ops.RoIAlign's constructor and forward over `roi_align` (the module the reference extractor builds in the golden run)"""

    def __init__(self, output_size, spatial_scale=1.0, sampling_ratio=0, pool_mode='avg', aligned=True, use_torchvision=False):
        super().__init__()
        assert pool_mode == 'avg' and aligned and not use_torchvision
        self.output_size = (output_size, output_size) if isinstance(output_size, int) else tuple(output_size)
        self.spatial_scale, self.sampling_ratio = float(spatial_scale), int(sampling_ratio)

    def forward(self, input, rois):
        return roi_align(input, rois, self.output_size[0], self.spatial_scale, self.sampling_ratio)


def map_roi_levels(rois, num_levels, finest_scale=56):
    """single_level_roi_extractor.py:50-54"""
    scale = torch.sqrt((rois[:, 3] - rois[:, 1]) * (rois[:, 4] - rois[:, 2]))
    lv = torch.floor(torch.log2(scale / finest_scale + 1e-6))
    return lv.clamp(min=0, max=num_levels - 1).long()


def extract(feats, rois, out=7, sampling_ratio=0, finest_scale=56, strides=STRIDES):
    """SingleRoIExtractor.forward (single_level_roi_extractor.py:56-103)"""
    L = len(feats)
    res = feats[0].new_zeros(rois.shape[0], feats[0].shape[1], out, out)
    if L == 1:
        return roi_align(feats[0], rois, out, 1.0 / strides[0], sampling_ratio)
    lv = map_roi_levels(rois, L, finest_scale)
    for i in range(L):
        inds = (lv == i).nonzero(as_tuple=False).squeeze(1)
        if inds.numel() > 0:
            res = res.index_put((inds,), roi_align(feats[i], rois[inds], out, 1.0 / strides[i], sampling_ratio))
        else:
            res = res + feats[i].sum() * 0.
    return res


def bbox_forward(feats, rois, w, out=7, sampling_ratio=0, finest_scale=56, strides=STRIDES):
    """_bbox_forward: extractor, then Shared2FCBBoxHead.forward (convfc_bbox_head.py:148-187)"""
    x = extract(feats[:len(strides)], rois, out, sampling_ratio, finest_scale, strides).flatten(1)
    x = F.relu(F.linear(x, w['shared_fcs.0.weight'], w['shared_fcs.0.bias']))
    x = F.relu(F.linear(x, w['shared_fcs.1.weight'], w['shared_fcs.1.bias']))
    return F.linear(x, w['fc_cls.weight'], w['fc_cls.bias']), F.linear(x, w['fc_reg.weight'], w['fc_reg.bias'])


def sample(proposals, gts, labels, ign, train):
    """per image MaxIoUAssigner + RandomSampler(add_gt_as_proposals) in the reference's order (the draws on the CPU generator):
    (bboxes [GTs; proposals], gt_inds, pos_inds, neg_inds)"""
    a = {k: v for k, v in train['assigner'].items() if k != 'type'}
    s = train['sampler']
    out = []
    for b in range(len(proposals)):
        gt_inds, _, _ = oa.max_iou_assign(proposals[b][:, :4], gts[b], labels[b], ign[b] if ign is not None else None, **a)
        bboxes = proposals[b][:, :4]
        if s.get('add_gt_as_proposals', True) and len(gts[b]) > 0:
            bboxes = torch.cat([gts[b], bboxes])
            gt_inds = torch.cat([torch.arange(1, len(gts[b]) + 1), gt_inds])
        pos, neg = orl.random_sample(gt_inds, s['num'], s['pos_fraction'], s.get('neg_pos_ub', -1))
        out.append((bboxes, gt_inds, pos, neg))
    return out


def targets(samples, gts, labels, num_classes, means, stds, pos_weight):
    """bbox2roi + BBoxHead.get_targets (bbox_head.py:117-259): rois, labels, label_weights, bbox_targets, bbox_weights"""
    rois, lab, lw, bt, bw = [], [], [], [], []
    for b, (bboxes, gt_inds, pos, neg) in enumerate(samples):
        pb, nb = bboxes[pos], bboxes[neg]
        np_, nn_ = pb.shape[0], nb.shape[0]
        l = torch.full((np_ + nn_,), num_classes, dtype=torch.long)
        w = torch.zeros(np_ + nn_)
        t, tw = torch.zeros(np_ + nn_, 4), torch.zeros(np_ + nn_, 4)
        if np_:
            l[:np_] = labels[b][gt_inds[pos] - 1]
            w[:np_] = 1.0 if pos_weight <= 0 else pos_weight
            t[:np_] = orl.bbox2delta(pb, gts[b][gt_inds[pos] - 1], means, stds)
            tw[:np_] = 1
        if nn_:
            w[-nn_:] = 1.0
        rois.append(torch.cat([torch.full((np_ + nn_, 1), float(b)), torch.cat([pb, nb])], 1))
        lab.append(l); lw.append(w); bt.append(t); bw.append(tw)
    return torch.cat(rois), torch.cat(lab), torch.cat(lw), torch.cat(bt), torch.cat(bw)


def loss(cls_score, bbox_pred, labels, lw, bt, bw, num_classes, agnostic, loss_cls, loss_bbox):
    """BBoxHead.loss (bbox_head.py:261-306) with CrossEntropyLoss(use_sigmoid=False) and L1Loss / SmoothL1Loss"""
    avg = max(float((lw > 0).sum()), 1.)
    cw = loss_cls.get('class_weight')
    ce = F.cross_entropy(cls_score, labels, weight=None if cw is None else torch.tensor(cw, dtype=torch.float32), reduction='none')
    out = dict(loss_cls=loss_cls.get('loss_weight', 1.0) * ((ce * lw).sum() / avg))
    pred_label = cls_score.argmax(1)
    out['acc'] = (pred_label == labels).float().sum(0, keepdim=True) * (100.0 / cls_score.shape[0])
    pos = (labels >= 0) & (labels < num_classes)
    if pos.any():
        p = bbox_pred.view(bbox_pred.shape[0], 4)[pos] if agnostic else bbox_pred.view(bbox_pred.shape[0], -1, 4)[pos, labels[pos]]
        d = torch.abs(p - bt[pos])
        if loss_bbox['type'] == 'SmoothL1Loss':
            beta = loss_bbox.get('beta', 1.0)
            d = torch.where(d < beta, 0.5 * d * d / beta, d - 0.5 * beta)
        out['loss_bbox'] = loss_bbox.get('loss_weight', 1.0) * ((d * bw[pos]).sum() / bt.shape[0])
    else:
        out['loss_bbox'] = bbox_pred[pos].sum()
    return out


def pad_rois(proposals):
    """test_mixins.py:79-93: shorter lists padded at the FRONT with zero boxes -> rois (B * N, 5), N"""
    N = max(p.shape[0] for p in proposals)
    padded = [torch.cat([p.new_zeros(N - p.shape[0], p.shape[1]), p]) for p in proposals]
    r = torch.stack(padded)
    bi = torch.arange(r.shape[0]).float().view(-1, 1, 1).expand(r.shape[0], r.shape[1], 1)
    return torch.cat([bi, r[..., :4]], -1).view(-1, 5), N


def decode(rois, cls_score, bbox_pred, B, img_shapes, means, stds, scale_factors=None):
    """test_mixins.py:94-119 + BBoxHead.get_bboxes (bbox_head.py:310-436) up to the NMS: (boxes (B, N, 4C or 4), scores (B, N, C+1))"""
    N = rois.shape[0] // B
    rois = rois.reshape(B, N, 5)
    cls_score = cls_score.reshape(B, N, -1).clone()
    bbox_pred = bbox_pred.reshape(B, N, -1).clone()
    pad = rois.abs()[..., 1:].sum(dim=-1) == 0
    cls_score[pad, :] = 0
    bbox_pred[pad, :] = 0
    scores = F.softmax(cls_score, dim=-1)
    bboxes = oa.delta2bbox(rois[..., 1:], bbox_pred, means, stds, max_shape=img_shapes)
    if scale_factors is not None:
        bboxes = bboxes / bboxes.new_tensor(np.stack(scale_factors)).unsqueeze(1).repeat(1, 1, bboxes.size(-1) // 4)
    return bboxes, scores


TRAIN = dict(assigner=dict(type='MaxIoUAssigner', pos_iou_thr=0.5, neg_iou_thr=0.5, min_pos_iou=0.5, match_low_quality=False,
                           ignore_iof_thr=-1),
             sampler=dict(type='RandomSampler', num=64, pos_fraction=0.25, neg_pos_ub=-1, add_gt_as_proposals=True),
             pos_weight=-1, debug=False)
TEST = dict(score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=-1)
TINYPERSON = dict(num_classes=1, reg_class_agnostic=False,
                  bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0., 0., 0., 0.], target_stds=[0.1, 0.1, 0.2, 0.2]),
                  loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0), loss_bbox=dict(type='L1Loss', loss_weight=1.0))


def _case(seed, n_gt, n_prop, head=None, train=None, test=None, img=(128, 160), near=0.7, boundary=False):
    t = {k: (dict(v) if isinstance(v, dict) else v) for k, v in TRAIN.items()}
    for k, v in (train or {}).items():
        if k in ('assigner', 'sampler'):
            t[k].update(v)
        else:
            t[k] = v
    h = {k: (dict(v) if isinstance(v, dict) else v) for k, v in TINYPERSON.items()}
    h.update(head or {})
    te = dict(TEST)
    te.update(test or {})
    return dict(seed=seed, n_gt=n_gt, n_prop=n_prop, head=h, train=t, test=te, img=img, near=near, boundary=boundary)


# name -> seed, GTs and proposals per image, head / train / test overrides
CASES = {
    'tinyperson': _case(31, [6, 9], [120, 120]),
    'classes80_smoothl1': _case(32, [7, 5], [100, 100], head=dict(num_classes=80, loss_bbox=dict(type='SmoothL1Loss', beta=1.0, loss_weight=1.0)),
                                test=dict(max_per_img=100)),
    'agnostic': _case(33, [5, 8], [90, 110], head=dict(num_classes=3, reg_class_agnostic=True)),
    'cw_posweight': _case(34, [6, 6], [100, 100], head=dict(num_classes=3, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False,
                                                                                        class_weight=[1.5, 0.5, 2.0, 0.8], loss_weight=1.2)),
                          train=dict(pos_weight=2.0)),
    'no_gt_image': _case(35, [0, 7], [80, 100]),
    'no_pos': _case(36, [3, 4], [60, 60], train=dict(sampler=dict(add_gt_as_proposals=False)), near=0.0),
    'uneven': _case(37, [4, 6], [40, 130]),
    'levels': _case(38, [5, 5], [100, 100], boundary=True, img=(512, 640)),
}
N_LEVELS_IN = 5                                  # the FPN gives 5 maps; the extractor reads x[:4]


def head_kwargs(name):
    c = CASES[name]['head']
    ex = dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0), out_channels=C_FEAT,
              featmap_strides=STRIDES)
    bh = dict(type='Shared2FCBBoxHead', in_channels=C_FEAT, fc_out_channels=FC, roi_feat_size=7, **c)
    return dict(bbox_roi_extractor=ex, bbox_head=bh)


def level_boundary_rois():
    """square RoIs whose v = sqrt(w h) / 56 + 1e-6 lies within 6 ulps of the side on each of the boundaries v = 1, 2, 4, 8"""
    rows = []
    for k in (1.0, 2.0, 4.0, 8.0):
        s = np.float32((k - 1e-6) * 56)
        for d in range(-6, 7):
            side = s
            for _ in range(abs(d)):
                side = np.nextafter(side, np.float32(np.inf if d > 0 else -np.inf))
            rows.append([0.0, 10.0, 20.0, np.float32(10.0 + side), np.float32(20.0 + side)])
    return torch.tensor(np.array(rows, np.float32))


def boundary_boxes(n, size):
    """boxes whose scale sqrt(w h) sits on the level boundaries 112, 224, 448 (and 1 ulp either side), some beyond the image"""
    out = []
    ulp = lambda v, k: float(np.nextafter(np.float32(v), np.float32(np.inf if k > 0 else -np.inf)))
    for i in range(n):
        s = [112.0, 224.0, 448.0][i % 3] - 1e-6 * 56 * (1 - (i // 3) % 2)
        s = ulp(s, (i % 5) - 2) if i % 5 != 2 else s
        x0, y0 = (i * 37) % size[1] - 40.0, (i * 53) % size[0] - 40.0
        out.append([x0, y0, x0 + s, y0 + s])
    return torch.tensor(out, dtype=torch.float32)


def case_inputs(name):
    """seeded FPN features (5 levels, C_FEAT channels), FC weights, GTs, labels, proposals (n, 5) and img_metas of a case"""
    c = CASES[name]
    g = torch.Generator().manual_seed(c['seed'])
    H, W = c['img']
    B = len(c['n_gt'])
    feats = [torch.randn(B, C_FEAT, -(-H // s), -(-W // s), generator=g) for s in STRIDES + [64]]
    C = c['head']['num_classes']
    reg = 4 if c['head'].get('reg_class_agnostic') else 4 * C
    k = C_FEAT * 49
    weights = {'shared_fcs.0.weight': torch.randn(FC, k, generator=g) / k ** 0.5, 'shared_fcs.0.bias': torch.randn(FC, generator=g) * 0.1,
               'shared_fcs.1.weight': torch.randn(FC, FC, generator=g) / FC ** 0.5, 'shared_fcs.1.bias': torch.randn(FC, generator=g) * 0.1,
               'fc_cls.weight': torch.randn(C + 1, FC, generator=g) * 0.3, 'fc_cls.bias': torch.randn(C + 1, generator=g) * 0.3,
               'fc_reg.weight': torch.randn(reg, FC, generator=g) * 0.1, 'fc_reg.bias': torch.randn(reg, generator=g) * 0.1}
    gts, labels, props, metas = [], [], [], []
    for b in range(B):
        gt = orl._boxes(g, c['n_gt'][b], H, W, 8.0, 120.0 if c['boundary'] else 48.0)
        gts.append(gt)
        labels.append(torch.randint(0, C, (c['n_gt'][b],), generator=g))
        n = c['n_prop'][b]
        if c['boundary']:
            p = boundary_boxes(n, (H, W))
        else:
            p = orl._boxes(g, n, H, W, 4.0, 64.0)
            if c['near'] > 0 and len(gt):                  # a share of the proposals jittered around the GTs, so some are positive
                m = int(n * c['near'])
                src = gt[torch.randint(0, len(gt), (m,), generator=g)]
                p[:m] = src + torch.randn(m, 4, generator=g) * 3.0
            elif len(gt):                                  # no positive: proposals kept clear of every GT
                p = p + torch.tensor([W, H, W, H], dtype=torch.float32) * 2
        props.append(torch.cat([p, torch.rand(n, 1, generator=g)], 1))
        metas.append(dict(img_shape=(H - 8 * b, W - 8 * b, 3), pad_shape=(H, W, 3), ori_shape=(H, W, 3),
                          scale_factor=np.array([1.25, 1.5, 1.25, 1.5], np.float32)))
    return dict(feats=feats, weights=weights, gt_bboxes=gts, gt_labels=labels, proposals=props, img_metas=metas)


def forward_train(inp, name, feats=None, w=None):
    """StandardRoIHead.forward_train: (losses, dict(samples, rois, labels, label_weights, bbox_targets, bbox_weights, cls_score, bbox_pred))"""
    c = CASES[name]
    h = c['head']
    feats = inp['feats'] if feats is None else feats
    w = inp['weights'] if w is None else w
    smp = sample(inp['proposals'], inp['gt_bboxes'], inp['gt_labels'], None, c['train'])
    bc = h['bbox_coder']
    rois, lab, lw, bt, bw = targets(smp, inp['gt_bboxes'], inp['gt_labels'], h['num_classes'], bc['target_means'], bc['target_stds'],
                                    c['train']['pos_weight'])
    cls, reg = bbox_forward(feats, rois, w)
    out = loss(cls, reg, lab, lw, bt, bw, h['num_classes'], h.get('reg_class_agnostic', False), h['loss_cls'], h['loss_bbox'])
    return out, dict(samples=smp, rois=rois, labels=lab, label_weights=lw, bbox_targets=bt, bbox_weights=bw, cls_score=cls, bbox_pred=reg)


def multiclass_nms_per_image(boxes, scores, num_classes, test_cfg):
    """bbox_nms.py:7-94 (multiclass_nms) of each image of a decoded batch, boxes (B, N, 4C or 4) and scores (B, N, C+1), over
    oracle/p2p.py's restatement of mmcv's batched_nms: per image (dets (k, 5), labels (k,))"""
    from oracle.p2p import batched_nms
    B, N = scores.shape[:2]
    C = num_classes
    dets, labs = [], []
    for b in range(B):
        bb = boxes[b].view(N, -1, 4) if boxes.shape[-1] > 4 else boxes[b][:, None].expand(N, C, 4)
        sc = scores[b][:, :-1]
        labels = torch.arange(C, dtype=torch.long).view(1, -1).expand_as(sc)
        bb, sc, labels = bb.reshape(-1, 4), sc.reshape(-1), labels.reshape(-1)
        inds = torch.nonzero(sc > test_cfg['score_thr'], as_tuple=False).squeeze(1)
        bb, sc, labels = bb[inds], sc[inds], labels[inds]
        if bb.numel() == 0:
            dets.append(bb.new_zeros((0, 5))); labs.append(labels)
            continue
        nms = dict(test_cfg['nms'])
        assert nms.pop('type', 'nms') == 'nms'
        d, keep = batched_nms(bb, sc, labels, nms['iou_threshold'])
        if test_cfg['max_per_img'] > 0:
            d, keep = d[:test_cfg['max_per_img']], keep[:test_cfg['max_per_img']]
        dets.append(d); labs.append(labels[keep])
    return dets, labs


def simple_test(inp, name, rescale=False):
    """StandardRoIHead.simple_test up to bbox2result: per image (dets (k, 5), labels (k,))"""
    c = CASES[name]
    h = c['head']
    B = len(inp['proposals'])
    rois, N = pad_rois([p.clone() for p in inp['proposals']])
    cls, reg = bbox_forward(inp['feats'], rois, inp['weights'])
    bc = h['bbox_coder']
    reps = reg.shape[-1] // 4
    boxes, scores = decode(rois, cls, reg, B, [m['img_shape'] for m in inp['img_metas']], list(bc['target_means']) * reps,
                           list(bc['target_stds']) * reps, [m['scale_factor'] for m in inp['img_metas']] if rescale else None)
    return multiclass_nms_per_image(boxes, scores, h['num_classes'], c['test'])
