"""Restatement of the detector's tile testing with torch-CPU ops in the reference's order: TwoStageDetector.tile_aug_test
(detectors/two_stage.py:195-258) from the RPN's per-aug proposals on, merge_aug_proposals / merge_aug_bboxes
(core/post_processing/merge_augs.py:12-109), bbox_flip / bbox_mapping / bbox_mapping_back (core/bbox/transforms.py:5-85),
StandardRoIHead.aug_test / aug_test_bboxes (standard_roi_head.py:246-270, test_mixins.py:157-189) and mmcv's batched_nms as
oracle/p2p.py restates it.  Test infrastructure — only tests/ and tools/ may import this."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import anchors as oa
from oracle import roi_head as orh
from oracle.p2p import batched_nms, nms


def bbox_flip(b, img_shape, direction):
    f = b.clone()
    if direction in ('horizontal', 'diagonal'):
        f[..., 0::4] = img_shape[1] - b[..., 2::4]
        f[..., 2::4] = img_shape[1] - b[..., 0::4]
    if direction in ('vertical', 'diagonal'):
        f[..., 1::4] = img_shape[0] - b[..., 3::4]
        f[..., 3::4] = img_shape[0] - b[..., 1::4]
    return f


def _sf(m):
    return torch.from_numpy(np.asarray(m['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32))


def bbox_mapping(b, m):
    n = b * _sf(m)
    if m.get('flip', False):
        n = bbox_flip(n, m['img_shape'], m['flip_direction'])
    off = m.get('tile_offset', None)
    if off is not None:
        dx, dy = off
        n[:, [0, 2]] -= dx
        n[:, [1, 3]] -= dy
        h, w = m['img_shape'][:2]
        n[:, [0, 2]] = n[:, [0, 2]].clamp(0, w - 1)
        n[:, [1, 3]] = n[:, [1, 3]].clamp(0, h - 1)
        n = n[((n[:, 2] - n[:, 0]) >= 2) & ((n[:, 3] - n[:, 1]) >= 2)]
    return n


def bbox_mapping_back(b, m):
    n = bbox_flip(b, m['img_shape'], m['flip_direction']) if m.get('flip', False) else b
    n = n.reshape(-1, 4) / _sf(m)
    off = m.get('tile_offset', None)
    if off is not None:
        n[:, [0, 2]] += off[0]
        n[:, [1, 3]] += off[1]
    return n.view(b.shape)


def merge_aug_proposals(props, metas, iou_threshold, max_per_img):
    rec = []
    for p, m in zip(props, metas):
        p = p.clone()
        p[:, :4] = bbox_mapping_back(p[:, :4], m)
        rec.append(p)
    p = torch.cat(rec)
    keep = nms(p[:, :4].contiguous(), p[:, 4].contiguous(), iou_threshold)
    p = p[keep]
    _, order = p[:, 4].sort(dim=0, descending=True, stable=True)
    return p[order[:min(max_per_img, p.shape[0])]]


def aug_test_bboxes(feats, metas, proposals, w, head, test_cfg):
    """feats per aug the level maps (1, C, H, W), metas per aug dict, proposals (n, >=4): (det_bboxes, det_labels)"""
    C = head['num_classes']
    bc = head['bbox_coder']
    reps = 1 if head.get('reg_class_agnostic') else C
    aug_b, aug_s = [], []
    for x, m in zip(feats, metas):
        p = bbox_mapping(proposals[:, :4], m)
        rois = torch.cat([p.new_zeros(p.shape[0], 1), p], 1)
        cls, reg = orh.bbox_forward(x, rois, w)
        scores = F.softmax(cls, dim=-1)
        b = oa.delta2bbox(rois[None, :, 1:], reg[None], list(bc['target_means']) * reps, list(bc['target_stds']) * reps,
                          max_shape=[m['img_shape']])[0]
        aug_b.append(b)
        aug_s.append(scores)
    b = torch.stack([bbox_mapping_back(bb, m) for bb, m in zip(aug_b, metas)]).mean(dim=0)
    s = torch.stack(aug_s).mean(dim=0)
    dets, labs = orh.multiclass_nms_per_image(b[None], s[None], C, test_cfg)
    return dets[0], labs[0]


def aug_test(feats, metas, proposals, w, head, test_cfg, rescale=False):
    d, l = aug_test_bboxes(feats, metas, proposals, w, head, test_cfg)
    if not rescale:
        d = d.clone()
        d[:, :4] *= _sf(metas[0])
    return d, l


def tile_aug_test(feats, metas, rpn_props, w, head, rpn_test_cfg, test_cfg, rescale=False, stats=None):
    """from the per-aug RPN proposals on: (det_bboxes (k, 5), det_labels (k,)) of the image; metas keep their tile_offset.
    stats (a dict) receives merge_rows, the number of rows the cross-tile batched_nms sees."""
    C = head['num_classes']
    tiles = {}
    for i, m in enumerate(metas):
        m = dict(m)
        off = m.pop('tile_offset')
        tiles.setdefault(off, []).append((i, m))
    boxes, labels = [], []
    for off, augs in tiles.items():
        ix = [i for i, _ in augs]
        ms = [m for _, m in augs]
        props = merge_aug_proposals([rpn_props[i] for i in ix], ms, rpn_test_cfg['nms']['iou_threshold'], rpn_test_cfg['max_per_img'])
        d, l = aug_test([feats[i] for i in ix], ms, props, w, head, test_cfg, rescale)
        dn = d.numpy().copy()
        for c in range(C):                               # bbox2result's class split, then the tile offset added in numpy fp32
            r = dn[l.numpy() == c]
            r[:, [0, 2]] += off[0]
            r[:, [1, 3]] += off[1]
            boxes.append(r)
            labels.append(torch.full((len(r),), c, dtype=torch.long))
    allb = torch.from_numpy(np.concatenate(boxes, 0))
    alll = torch.cat(labels)
    if stats is not None:
        stats['merge_rows'] = len(allb)
    if len(allb) == 0:
        return torch.zeros((0, 5)), torch.zeros((0,), dtype=torch.long)
    nmsc = dict(test_cfg['nms'])
    d, keep = batched_nms(allb[:, :4].contiguous(), allb[:, 4].contiguous(), alll, nmsc['iou_threshold'],
                          split_thr=nmsc.get('split_thr', 10000))
    if test_cfg['max_per_img'] > 0:
        d, keep = d[:test_cfg['max_per_img']], keep[:test_cfg['max_per_img']]
    return d, alll[keep]


def aten_mean0(x):
    """torch.stack(...).mean(0) of x (A, M) in ATen's CPU order, as ptb_aug_merge restates it"""
    A, M = x.shape
    x = np.asarray(x, np.float32)
    out = np.empty(M, np.float32)
    g = (M // 32) * 32
    acc = np.zeros((4, g), np.float32)
    i = 0
    while i + 16 <= A:
        for _ in range(16):
            acc[0] = acc[0] + x[i, :g]
            i += 1
        for j in range(1, 4):
            acc[j] = acc[j] + acc[j - 1]
            acc[j - 1] = 0
            if (i & (15 << (4 * j))) != 0:
                break
    while i < A:
        acc[0] = acc[0] + x[i, :g]
        i += 1
    out[:g] = ((acc[0] + acc[1]) + acc[2]) + acc[3]
    t = x[:, g:]
    p = np.zeros((4, M - g), np.float32)
    for i in range(A // 4):
        for k in range(4):
            p[k] = p[k] + t[4 * i + k]
    for i in range(4 * (A // 4), A):
        p[0] = p[0] + t[i]
    out[g:] = ((p[0] + p[1]) + p[2]) + p[3]
    return out / np.float32(A)


# ---- seeded cases pinned against the real reference by oracle/make_golden_tile_test.py (tests/golden/tile_test_*.npz)
# The RoI head's Linear layers are selection matrices (one weight of 1 or a power of two per output row, the rest 0) and the feature
# maps hold multiples of 1/64: every FC output is then exact in fp32 whatever the GEMM's summation order, so the GPU's RoI forward
# gives the CPU reference's logits bit for bit and the post-processing is compared on equal inputs.
C_FEAT, FC = 8, 64
RPN_CFG = dict(nms_pre=1000, max_per_img=1000, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
TILE_1080P = [(x, y) for y in (0, 284, 568) for x in (0, 540, 1080, 1280)]


def _case(seed, offsets, tile=(512, 640), C=1, rcnn_max=-1, rpn_max=1000, flips=(None,), scales=(1.0,), cls_gain=4.0, bg_bias=0.0,
          direct=False):
    return dict(seed=seed, offsets=offsets, tile=tile, C=C, flips=flips, scales=scales, cls_gain=cls_gain, bg_bias=bg_bias,
                direct=direct, rpn=dict(RPN_CFG, max_per_img=rpn_max),
                rcnn=dict(score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=rcnn_max))


CASES = {
    'tinyperson12': _case(61, TILE_1080P),                                       # >= 10 000 rows at the cross-tile merge (split branch)
    'classes3': _case(62, [(0, 0), (100, 0), (0, 80), (100, 80)], tile=(128, 160), C=3, rcnn_max=60, rpn_max=300, cls_gain=1.0),
    'flip_scale': _case(63, [(0, 0), (120, 0)], tile=(128, 160), rpn_max=200,
                        flips=(None, 'horizontal', None, 'vertical'), scales=(0.5, 1.0)),
    'one_tile': _case(64, [(0, 0)], tile=(128, 160), C=2, rpn_max=300),
    'empty': _case(65, [(0, 0), (130, 0)], tile=(128, 160), rpn_max=200, bg_bias=40.0),
    'direct': _case(66, [(40, 8)], tile=(128, 160), C=2, rcnn_max=50, flips=(None, 'diagonal'), scales=(1.5,), direct=True),
}


def head_kwargs(name):
    c = CASES[name]
    rpn = dict(in_channels=C_FEAT, feat_channels=C_FEAT, anchor_generator=dict(type='AnchorGenerator', scales=[2], ratios=[0.5, 1.0, 2.0],
                                                                                strides=[4, 8, 16, 32, 64]),
               bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0.] * 4, target_stds=[1.0] * 4))
    roi = dict(bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0),
                                       out_channels=C_FEAT, featmap_strides=orh.STRIDES),
               bbox_head=dict(type='Shared2FCBBoxHead', in_channels=C_FEAT, fc_out_channels=FC, roi_feat_size=7, num_classes=c['C'],
                              bbox_coder=dict(type='DeltaXYWHBBoxCoder', target_means=[0.] * 4, target_stds=[0.1, 0.1, 0.2, 0.2]),
                              reg_class_agnostic=False, loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0),
                              loss_bbox=dict(type='L1Loss', loss_weight=1.0)))
    return rpn, roi


def _select(g, rows, cols, gain):
    w = torch.zeros(rows, cols)
    w[torch.arange(rows), torch.randperm(cols, generator=g)[:rows] if rows <= cols else torch.randint(0, cols, (rows,), generator=g)] = gain
    return w


def case_inputs(name):
    """feats per aug (levels (1, C_FEAT, H, W), multiples of 1/64), img_metas per aug [meta] with tile_offset, the RPN's conv weights,
    the RoI head's selection weights, and for the direct case seeded proposals (n, 5)"""
    c = CASES[name]
    g = torch.Generator().manual_seed(c['seed'])
    C = c['C']
    rpn_w = {'rpn_conv.weight': torch.randn(C_FEAT, C_FEAT, 3, 3, generator=g) * 0.2, 'rpn_conv.bias': torch.zeros(C_FEAT),
             'rpn_cls.weight': torch.randn(3, C_FEAT, 1, 1, generator=g) * 0.5, 'rpn_cls.bias': torch.zeros(3),
             'rpn_reg.weight': torch.randn(12, C_FEAT, 1, 1, generator=g) * 0.05, 'rpn_reg.bias': torch.zeros(12)}
    k = C_FEAT * 49
    cls_w = _select(g, C + 1, FC, c['cls_gain'])
    roi_w = {'shared_fcs.0.weight': _select(g, FC, k, 1.0), 'shared_fcs.0.bias': torch.zeros(FC),
             'shared_fcs.1.weight': _select(g, FC, FC, 1.0), 'shared_fcs.1.bias': torch.zeros(FC),
             'fc_cls.weight': cls_w, 'fc_cls.bias': torch.tensor([0.5] * C + [c['bg_bias']]),
             'fc_reg.weight': _select(g, 4 * C, FC, 0.125), 'fc_reg.bias': torch.zeros(4 * C)}
    feats, metas = [], []
    th, tw = c['tile']
    for off in c['offsets']:
        for s in c['scales']:
            for d in c['flips']:
                h, w = int(th * s), int(tw * s)
                feats.append([torch.round(torch.randn(1, C_FEAT, -(-h // st), -(-w // st), generator=g) * 64) / 64
                              for st in (4, 8, 16, 32, 64)])
                metas.append([dict(img_shape=(h, w, 3), pad_shape=(h, w, 3), ori_shape=(th, tw, 3),
                                   scale_factor=np.array([s] * 4, np.float32), flip=d is not None, flip_direction=d, tile_offset=off)])
    out = dict(feats=feats, img_metas=metas, rpn_weights=rpn_w, roi_weights=roi_w)
    if c['direct']:
        xy = 40 + torch.rand(60, 2, generator=g) * 50          # inside the window at the offset in every aug: none clamped or dropped
        wh = 6 + torch.rand(60, 2, generator=g) * 30
        out['proposals'] = torch.cat([xy, xy + wh, torch.rand(60, 1, generator=g)], 1)
    return out


def roi_head_spec(name):
    c = CASES[name]
    return dict(num_classes=c['C'], reg_class_agnostic=False,
                bbox_coder=dict(target_means=[0.] * 4, target_stds=[0.1, 0.1, 0.2, 0.2]))
