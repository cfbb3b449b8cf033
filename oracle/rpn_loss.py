"""Restatement of RPNHead.loss (mmdet/models/dense_heads/rpn_head.py:44-75 over anchor_head.py:171-489): inside flags, MaxIoUAssigner,
RandomSampler, bbox2delta, unmap, images_to_levels and the per-level CrossEntropyLoss(use_sigmoid=True) + L1Loss / SmoothL1Loss, with
torch ops in the reference's order, on the device of the GT boxes (torch CPU in the tests; the draws always on the CPU generator, as the
reference's).  Test infrastructure — only tests/ and tools/ may import this.  Pinned: oracle/make_golden_rpn_loss.py
runs the real reference RPNHead.loss (through oracle/_mmcv_stub.py) on the seeded CASES below, asserts that this restatement equals it and
stores tests/golden/rpn_loss_*.npz."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import anchors as oa

C_FEAT = 8
STRIDES = [4, 8, 16, 32, 64]
TINYPERSON = dict(anchor_generator=dict(type='AnchorGenerator', scales=[2], ratios=[0.5, 1.0, 2.0], strides=STRIDES),
                  bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0.0, 0.0, 0.0, 0.0], target_stds=[1.0, 1.0, 1.0, 1.0]),
                  loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0), loss_bbox=dict(type='L1Loss', loss_weight=1.0))
TRAIN = dict(assigner=dict(type='MaxIoUAssigner', pos_iou_thr=0.7, neg_iou_thr=0.3, min_pos_iou=0.3, match_low_quality=True,
                           ignore_iof_thr=-1),
             sampler=dict(type='RandomSampler', num=256, pos_fraction=0.5, neg_pos_ub=-1, add_gt_as_proposals=False),
             allowed_border=-1, pos_weight=-1, debug=False)


def _train(**kw):
    t = {k: (dict(v) if isinstance(v, dict) else v) for k, v in TRAIN.items()}
    for k, v in kw.items():
        if k in ('assigner', 'sampler'):
            t[k].update(v)
        else:
            t[k] = v
    return t


# name -> seed, image size (h, w), per image (img_shape h, w, pad h, w), GTs per image, head / train overrides
CASES = {
    'tinyperson': dict(seed=11, size=(128, 160), imgs=[(128, 160, 128, 160), (120, 150, 128, 160)], n_gt=[9, 14], train=_train()),
    'border0': dict(seed=12, size=(128, 160), imgs=[(128, 160, 128, 160), (100, 130, 128, 160)], n_gt=[7, 10],
                    train=_train(allowed_border=0)),
    'negposub_posweight': dict(seed=13, size=(128, 160), imgs=[(128, 160, 128, 160), (128, 160, 128, 160)], n_gt=[3, 12],
                               train=_train(sampler=dict(neg_pos_ub=1), pos_weight=2.0)),
    'smooth_l1': dict(seed=14, size=(128, 160), imgs=[(128, 160, 128, 160), (128, 160, 128, 160)], n_gt=[8, 8], train=_train(),
                      head=dict(loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=1.5),
                                loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=0.5))),
    'no_gt': dict(seed=15, size=(128, 160), imgs=[(128, 160, 128, 160), (128, 160, 128, 160)], n_gt=[0, 6], train=_train()),
    'ignore': dict(seed=16, size=(128, 160), imgs=[(128, 160, 128, 160), (128, 160, 128, 160)], n_gt=[10, 10], n_ign=[3, 2],
                   train=_train(assigner=dict(ignore_iof_thr=0.5))),
    'many_pos': dict(seed=17, size=(128, 160), imgs=[(128, 160, 128, 160), (128, 160, 128, 160)], n_gt=[160, 40], train=_train()),
    'few_neg': dict(seed=18, size=(32, 32), imgs=[(32, 32, 32, 32), (28, 30, 32, 32)], n_gt=[3, 2], train=_train()),
    'pad_shapes': dict(seed=19, size=(128, 160), imgs=[(100, 150, 104, 152), (128, 120, 128, 128)], n_gt=[6, 9],
                       train=_train(allowed_border=0)),
}
ROI_SAMPLER = dict(num=512, pos_fraction=0.25, neg_pos_ub=-1, add_gt_as_proposals=True)


def head_kwargs(name):
    c = CASES[name]
    kw = {k: (dict(v) if isinstance(v, dict) else v) for k, v in TINYPERSON.items()}
    kw.update(c.get('head', {}))
    return dict(in_channels=C_FEAT, feat_channels=C_FEAT, **kw)


def _boxes(g, n, h, w, lo=4.0, hi=40.0):
    c = torch.rand(n, 2, generator=g) * torch.tensor([w, h], dtype=torch.float32)
    s = torch.rand(n, 2, generator=g) * (hi - lo) + lo
    return torch.cat([c - s / 2, c + s / 2], 1).clamp(min=0)


def case_inputs(name):
    """seeded features (B, C_FEAT, H/4, W/4 ... ) per level, conv weights, GTs, ignore boxes and img_metas of a case"""
    c = CASES[name]
    g = torch.Generator().manual_seed(c['seed'])
    H, W = c['size']
    B = len(c['imgs'])
    feats = [torch.randn(B, C_FEAT, -(-H // s), -(-W // s), generator=g) for s in STRIDES]
    A = 3
    weights = {'rpn_conv.weight': torch.randn(C_FEAT, C_FEAT, 3, 3, generator=g) * 0.1, 'rpn_conv.bias': torch.randn(C_FEAT, generator=g) * 0.1,
               'rpn_cls.weight': torch.randn(A, C_FEAT, 1, 1, generator=g) * 0.3, 'rpn_cls.bias': torch.randn(A, generator=g) * 0.3 - 1.0,
               'rpn_reg.weight': torch.randn(4 * A, C_FEAT, 1, 1, generator=g) * 0.1, 'rpn_reg.bias': torch.randn(4 * A, generator=g) * 0.1}
    gts, igns, metas = [], [], []
    for b, (ih, iw, ph, pw) in enumerate(c['imgs']):
        gts.append(_boxes(g, c['n_gt'][b], ih, iw))
        n_ign = c.get('n_ign', [0] * B)[b]
        igns.append(_boxes(g, n_ign, ih, iw, 20.0, 60.0))
        metas.append(dict(img_shape=(ih, iw, 3), pad_shape=(ph, pw, 3), ori_shape=(ih, iw, 3), scale_factor=np.ones(4, np.float32)))
    return dict(feats=feats, weights=weights, gt_bboxes=gts, gt_bboxes_ignore=igns if 'n_ign' in c else None, img_metas=metas)


def forward(feats, w):
    """RPNHead.forward_single on every level (rpn_head.py:36-42)"""
    cls, reg = [], []
    for x in feats:
        y = F.relu(F.conv2d(x, w['rpn_conv.weight'], w['rpn_conv.bias'], padding=1))
        cls.append(F.conv2d(y, w['rpn_cls.weight'], w['rpn_cls.bias']))
        reg.append(F.conv2d(y, w['rpn_reg.weight'], w['rpn_reg.bias']))
    return cls, reg


def grid_anchors(base, feat_hw, stride, device='cpu'):
    """AnchorGenerator.single_level_grid_anchors (anchor_generator.py:233-270) on `device`, as the reference builds them on the head's"""
    fh, fw = feat_hw
    sx, sy = torch.arange(0, fw, device=device) * stride, torch.arange(0, fh, device=device) * stride
    xx, yy = sx.repeat(fh), sy.view(-1, 1).repeat(1, fw).view(-1)
    shifts = torch.stack([xx, yy, xx, yy], dim=-1).type_as(base)
    return (base[None, :, :] + shifts[:, None, :]).view(-1, 4)


def valid_flags(featmap_sizes, pad_shape, A, device='cpu'):
    """AnchorGenerator.valid_flags (anchor_generator.py:272-330)"""
    out = []
    for (fh, fw), s in zip(featmap_sizes, STRIDES):
        vh, vw = min(int(np.ceil(pad_shape[0] / s)), fh), min(int(np.ceil(pad_shape[1] / s)), fw)
        vx, vy = torch.zeros(fw, dtype=torch.bool, device=device), torch.zeros(fh, dtype=torch.bool, device=device)
        vx[:vw] = True
        vy[:vh] = True
        xx, yy = vx.repeat(fh), vy.view(-1, 1).repeat(1, fw).view(-1)
        out.append((xx & yy)[:, None].expand(fh * fw, A).contiguous().view(-1))
    return out


def inside_flags(anchors, valid, img_shape, allowed_border):
    """anchor_inside_flags (core/anchor/utils.py:20-45)"""
    if allowed_border < 0:
        return valid
    h, w = img_shape[:2]
    return valid & (anchors[:, 0] >= -allowed_border) & (anchors[:, 1] >= -allowed_border) & \
        (anchors[:, 2] < w + allowed_border) & (anchors[:, 3] < h + allowed_border)


def random_sample(gt_inds, num, pos_fraction, neg_pos_ub=-1):
    """BaseSampler.sample + RandomSampler._sample_pos / _sample_neg / random_choice (base_sampler.py:82-97, random_sampler.py:31-81) on
    an assignment without GT proposals: the same torch.randperm calls on the CPU generator."""
    def choose(inds, k):
        if inds.numel() != 0:
            inds = inds.squeeze(1)
        if inds.numel() <= k:
            return inds
        return inds[torch.randperm(inds.numel())[:k].to(inds.device)]
    nep = int(num * pos_fraction)
    pos = choose(torch.nonzero(gt_inds > 0, as_tuple=False), nep).unique()
    nen = num - pos.numel()
    if neg_pos_ub >= 0:
        ub = int(neg_pos_ub * max(1, pos.numel()))
        if nen > ub:
            nen = ub
    neg = choose(torch.nonzero(gt_inds == 0, as_tuple=False), nen).unique()
    return pos, neg


def bbox2delta(p, g, means, stds):
    """delta_xywh_bbox_coder.py:98-140"""
    px, py = (p[..., 0] + p[..., 2]) * 0.5, (p[..., 1] + p[..., 3]) * 0.5
    pw, ph = p[..., 2] - p[..., 0], p[..., 3] - p[..., 1]
    gx, gy = (g[..., 0] + g[..., 2]) * 0.5, (g[..., 1] + g[..., 3]) * 0.5
    gw, gh = g[..., 2] - g[..., 0], g[..., 3] - g[..., 1]
    d = torch.stack([(gx - px) / pw, (gy - py) / ph, torch.log(gw / pw), torch.log(gh / ph)], dim=-1)
    return d.sub_(d.new_tensor(means).unsqueeze(0)).div_(d.new_tensor(stds).unsqueeze(0))


def get_targets(featmap_sizes, gt_bboxes, img_metas, gt_bboxes_ignore, head_kw, train):
    """AnchorHead.get_targets (anchor_head.py:171-369) -> dict(levels=[(labels, label_weights, bbox_targets, bbox_weights) per level],
    pos_inds / neg_inds per image, num_total_samples) or None"""
    ag = head_kw['anchor_generator']
    A = len(ag['scales']) * len(ag['ratios'])
    dev = gt_bboxes[0].device
    base = [oa.base_anchors(s, ag['scales'], ag['ratios']).to(dev) for s in ag['strides']]
    mlvl = [grid_anchors(b, fs, s, dev) for b, fs, s in zip(base, featmap_sizes, ag['strides'])]
    flat = torch.cat(mlvl)
    bc = head_kw['bbox_coder']
    a_cfg = {k: v for k, v in train['assigner'].items() if k != 'type'}
    s_cfg = train['sampler']
    res = []
    for b, meta in enumerate(img_metas):
        valid = torch.cat(valid_flags(featmap_sizes, meta['pad_shape'], A, dev))
        inside = inside_flags(flat, valid, meta['img_shape'], train['allowed_border'])
        if not inside.any():
            res.append(None)
            continue
        anchors = flat[inside, :]
        ign = gt_bboxes_ignore[b] if gt_bboxes_ignore is not None else None
        gt_inds, _, _ = oa.max_iou_assign(anchors, gt_bboxes[b], None, ign, **a_cfg)
        pos, neg = random_sample(gt_inds, s_cfg['num'], s_cfg['pos_fraction'], s_cfg.get('neg_pos_ub', -1))
        n = anchors.shape[0]
        bt, bw = torch.zeros_like(anchors), torch.zeros_like(anchors)
        labels = anchors.new_full((n,), 1, dtype=torch.long)
        lw = anchors.new_zeros(n, dtype=torch.float)
        if len(pos) > 0:
            bt[pos, :] = bbox2delta(anchors[pos], gt_bboxes[b][gt_inds[pos] - 1, :], bc['target_means'], bc['target_stds'])
            bw[pos, :] = 1.0
            labels[pos] = 0
            lw[pos] = 1.0 if train['pos_weight'] <= 0 else train['pos_weight']
        if len(neg) > 0:
            lw[neg] = 1.0
        N = flat.shape[0]

        def unmap(t, fill=0):
            o = t.new_full((N,) + t.shape[1:], fill)
            o[inside] = t
            return o
        res.append((unmap(labels, 1), unmap(lw), unmap(bt), unmap(bw), pos, neg))
    if any(r is None for r in res):
        return None
    nl = [m.shape[0] for m in mlvl]
    off = np.concatenate([[0], np.cumsum(nl)])
    levels = [tuple(torch.stack([r[k] for r in res])[:, off[l]:off[l + 1]] for k in range(4)) for l in range(len(nl))]
    return dict(levels=levels, pos_inds=[r[4] for r in res], neg_inds=[r[5] for r in res],
                num_total_samples=sum(max(r[4].numel(), 1) for r in res) + sum(max(r[5].numel(), 1) for r in res))


def loss(cls_scores, bbox_preds, gt_bboxes, img_metas, gt_bboxes_ignore, head_kw, train):
    """RPNHead.loss: (dict(loss_rpn_cls=[L], loss_rpn_bbox=[L]) or None, targets)"""
    tg = get_targets([tuple(c.shape[-2:]) for c in cls_scores], gt_bboxes, img_metas, gt_bboxes_ignore, head_kw, train)
    if tg is None:
        return None, None
    lc, lb = head_kw['loss_cls'], head_kw['loss_bbox']
    avg = tg['num_total_samples']
    out_c, out_b = [], []
    for c, r, (lab, lw, bt, bw) in zip(cls_scores, bbox_preds, tg['levels']):
        x = c.permute(0, 2, 3, 1).reshape(-1, 1)
        lab, lw = lab.reshape(-1), lw.reshape(-1)
        t = torch.zeros_like(x)
        t[lab == 0, 0] = 1.0
        l = F.binary_cross_entropy_with_logits(x, t, reduction='none') * lw.view(-1, 1)
        out_c.append(lc.get('loss_weight', 1.0) * (l.sum() / avg))
        p = r.permute(0, 2, 3, 1).reshape(-1, 4)
        d = torch.abs(p - bt.reshape(-1, 4))
        if lb['type'] == 'SmoothL1Loss':
            beta = lb.get('beta', 1.0)
            d = torch.where(d < beta, 0.5 * d * d / beta, d - 0.5 * beta)
        out_b.append(lb.get('loss_weight', 1.0) * ((d * bw.reshape(-1, 4)).sum() / avg))
    return dict(loss_rpn_cls=out_c, loss_rpn_bbox=out_b), tg


def roi_sampler_inputs(seed=21, n=600, n_gt=12):
    """an R-CNN-stage assignment for RandomSampler(num=512, pos_fraction=0.25, add_gt_as_proposals=True) alone"""
    anchors, gts, labels, ign = oa.synth_anchor_case(seed, n_anchor=n, n_gt=n_gt, n_ign=0, size=(256, 320))
    gt_inds, max_ov, lab = oa.max_iou_assign(anchors, gts, labels, None, pos_iou_thr=0.5, neg_iou_thr=0.5, min_pos_iou=0.5,
                                             match_low_quality=False)
    return anchors, gts, labels, gt_inds, max_ov, lab
