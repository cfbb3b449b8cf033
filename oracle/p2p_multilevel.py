"""ORACLE (test infrastructure, NOT product code) — P2PHead over several FPN levels (strides=[s_0, ..., s_{L-1}]).

Follows /root/reference/TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py:104-123 (forward: the same towers on every level),
:125-170 (get_pred_points: the levels' rows concatenated level-major, each row carrying its stride), :172-248 (loss: one Hungarian
matching over every level's valid rows of an image; loss_single divides the points by each row's own stride), :345-405
(_get_bboxes_single: the rows reshaped into len(strides) EQUAL chunks - not levels - and the top nms_pre of each chunk) and
:425-465 (get_points: per-level grid points without a half-stride offset and per-level valid flags from pad_shape).
Everything per level is oracle/p2p.py; the losses are oracle/p2p.py, oracle/p2p_defaults.py and oracle/p2p_softmax.py.
Only tests/ and oracle/make_golden_p2p_multilevel.py import this.
"""
import math

import torch

from oracle import p2p as op2p, p2p_defaults as odef, p2p_softmax as osm
from oracle.synth import sample_points

# (a) strides [8, 16, 32], one anchor, Focal + SmoothL1, T = 336 rows in 3 chunks of 112 (the last chunk straddles all three levels);
# (b) strides [8, 16], the reference defaults (four anchors, CrossEntropy + MSE), T = 1280 in 2 chunks of 640 inside level 0 and
#     across the level boundary; (c) softmax CrossEntropy with class_weight over (b)'s maps; (d) maps whose T = 320 is not a multiple
#     of 3: training only, inference raises in the reference; (e) aug_test_bboxes of (a)'s head at two scales.
CASES = {
    'a_focal_sl1': dict(seed=5101, strides=[8, 16, 32], k=1, loss_cls='FocalLoss', loss_reg='SmoothL1Loss', maps=[(16, 16), (8, 8), (4, 4)],
                        nms_pre=50),
    'b_defaults': dict(seed=5102, strides=[8, 16], k=4, loss_cls='CrossEntropyLoss', loss_reg='MSELoss', maps=[(16, 16), (8, 8)],
                       nms_pre=300),
    'c_softmax_cw': dict(seed=5103, strides=[8, 16], k=4, loss_cls='CrossEntropyLoss', loss_reg='MSELoss', maps=[(16, 16), (8, 8)],
                         nms_pre=300, use_sigmoid=False),
    'd_uneven': dict(seed=5104, strides=[8, 16, 32], k=1, loss_cls='FocalLoss', loss_reg='SmoothL1Loss', maps=[(16, 15), (8, 8), (4, 4)],
                     nms_pre=50),
}
AUG_CASE = dict(base='a_focal_sl1', seed=5105, scales=[1.0, 0.75], maps=[[(16, 16), (8, 8), (4, 4)], [(12, 12), (6, 6), (3, 3)]])
NUM_CLASSES = 80
C_FEAT = 256


def case_cfg(name):
    c = CASES[name]
    anchors = list(odef.ANCHORS) if c['k'] == 4 else [(0., 0.)]
    cfg = odef.reference_defaults_cfg(num_classes=NUM_CLASSES, point_anchor=anchors, strides=list(c['strides']), stride=c['strides'][0],
                                      loss_cls=c['loss_cls'], loss_reg=c['loss_reg'], nms_pre=c['nms_pre'], nms_iou=0.5)
    if c['k'] == 1:          # the shipped single-anchor configs: pts_gamma 1, reg_norm 1, FocalLoss + SmoothL1Loss(beta 1/9, 0.5)
        cfg.update(pts_gamma=1.0, reg_norm=1.0, loss_cls_weight=1.0, loss_reg_weight=0.5)
    if c.get('use_sigmoid', True) is False:
        cfg.update(use_sigmoid=False, class_weight=[1.0 + 0.01 * (i % 7) for i in range(NUM_CLASSES)] + [0.5])
    return cfg


def num_cls_out(cfg):
    return osm.num_cls_out(cfg)


def weights(gen, k, n_out, softmax):
    w = {}
    for prefix in ('cls_convs', 'reg_convs'):
        for i in range(4):
            w[f'{prefix}.{i}.conv.weight'] = torch.randn(C_FEAT, C_FEAT, 3, 3, generator=gen) * (1.4 / math.sqrt(C_FEAT * 9))
            w[f'{prefix}.{i}.gn.weight'] = 1 + 0.1 * torch.randn(C_FEAT, generator=gen)
            w[f'{prefix}.{i}.gn.bias'] = 0.1 * torch.randn(C_FEAT, generator=gen)
    w['cls_out.weight'] = torch.randn(k * n_out, C_FEAT, 3, 3, generator=gen) * 0.045
    if softmax:
        bias = -1.0 + torch.randn(k, n_out, generator=gen)
        bias[:, -1] = 3.0
        w['cls_out.bias'] = bias.reshape(-1)
    else:
        w['cls_out.bias'] = torch.full((k * n_out,), -math.log(99.0)) + 0.3 * torch.randn(k * n_out, generator=gen)
    w['reg_out.weight'] = torch.randn(2 * k, C_FEAT, 3, 3, generator=gen) * 0.001
    w['reg_out.bias'] = torch.zeros(2 * k)
    return w


def case_inputs(name, B=2, n=12):
    """seeded weights, one ReLU feature map per level (sizes CASES[name]['maps']), GT points and metas.  Image 1 has a smaller pad shape,
    so every level's valid flags cut its map.  CPU generator: bit-reproducible."""
    c = CASES[name]
    cfg = case_cfg(name)
    gen = torch.Generator().manual_seed(c['seed'])
    w = weights(gen, c['k'], num_cls_out(cfg), not cfg.get('use_sigmoid', True))
    xs = [torch.relu(torch.randn(B, C_FEAT, h, wd, generator=gen)) for h, wd in c['maps']]
    H0, W0 = c['maps'][0]
    s0 = c['strides'][0]
    pads = [(H0 * s0, W0 * s0), (H0 * s0 - 16, W0 * s0 - 8)]
    imgs = [(pads[0][0] - 3, pads[0][1] - 2), (pads[1][0] - 2, pads[1][1] - 3)]
    gt_bboxes, gt_labels, metas = [], [], []
    for b in range(B):
        ih, iw = imgs[b]
        pts = sample_points(n, iw, ih, gen)
        gt_bboxes.append(torch.cat([pts - 8, pts + 8], dim=1))
        gt_labels.append(torch.randint(0, NUM_CLASSES, (n,), generator=gen))
        metas.append(dict(pad_shape=pads[b] + (3,), img_shape=(ih, iw, 3), scale_factor=[1.0, 1.0, 1.0, 1.0]))
    return dict(xs=xs, weights=w, gt_bboxes=gt_bboxes, gt_labels=gt_labels, img_metas=metas), cfg


def aug_inputs():
    """AUG_CASE: one image seen at two scales, (a)'s head.  The second view's maps are smaller and its meta carries scale 0.75."""
    base = AUG_CASE['base']
    gen = torch.Generator().manual_seed(AUG_CASE['seed'])
    cfg = case_cfg(base)
    w = weights(gen, CASES[base]['k'], num_cls_out(cfg), False)
    feats, metas = [], []
    for scale, maps in zip(AUG_CASE['scales'], AUG_CASE['maps']):
        feats.append([torch.relu(torch.randn(1, C_FEAT, h, wd, generator=gen)) for h, wd in maps])
        ph, pw = maps[0][0] * 8, maps[0][1] * 8
        metas.append([dict(pad_shape=(ph, pw, 3), img_shape=(ph - 2, pw - 3, 3), scale_factor=[scale] * 4, flip=False,
                           flip_direction='horizontal')])
    return feats, metas, w, cfg


def head_forward(xs, weights_, cfg):
    """ref:104-123: the same towers and output convs over every level."""
    outs = [op2p.head_forward(x, weights_, cfg) for x in xs]
    return [o[0] for o in outs], [o[1] for o in outs]


def pred_points(cls_outs, pts_outs, img_metas, cfg):
    """ref:125-170: oracle/p2p.py's pred_points per level with that level's stride, concatenated level-major -> anchor (B,T,3),
    pred (B,T,3) (column 2 = the row's stride), valid (B,T), cls (B,T,num_cls_out)."""
    per = [op2p.pred_points(c, p, img_metas, dict(cfg, stride=s, num_classes=num_cls_out(cfg)))
           for c, p, s in zip(cls_outs, pts_outs, cfg['strides'])]
    return tuple(torch.cat([o[i] for o in per], 1) for i in range(4))


def p2p_loss(cls_outs, pts_outs, gt_bboxes, gt_labels, img_metas, cfg, return_all=False):
    """ref:172-248 over every level's rows: one matching per image, CrossEntropyLoss averaged over num_total, FocalLoss and the point
    losses over num_total_pos, each row's points divided by its own stride."""
    anchor, pred, valid, cls = pred_points(cls_outs, pts_outs, img_metas, cfg)
    gt_points = [(b[:, :2] + b[:, 2:]) / 2 for b in gt_bboxes]
    prop = anchor if cfg['assign_before_pred'] else pred
    tg = [op2p.target_single(prop[b][..., :2].detach(), valid[b], cls[b].detach(), gt_points[b], gt_labels[b],
                             img_metas[b]['img_shape'], cfg) for b in range(len(img_metas))]
    num_total = sum([len(t[0]) for t in tg])
    num_total_pos = sum([(t[3][..., 0] > 0).sum() for t in tg])
    cw = None if cfg.get('class_weight') is None else cls.new_tensor(cfg['class_weight'])
    loss_cls, loss_pts = [], []
    for b, (labels, lw, gpts, pw, _) in enumerate(tg):
        x = cls[b].contiguous()
        if cfg['loss_cls'] == 'FocalLoss':
            l = (op2p.sigmoid_focal_loss_elem(x, labels, cfg['focal_gamma'], cfg['focal_alpha']) * lw.view(-1, 1)).sum() / num_total_pos
        elif cfg.get('use_sigmoid', True):
            l = osm.binary_cross_entropy_elem(x, labels, cw)
            l = (l * lw.view(-1, 1).expand(lw.size(0), l.size(1)).float()).sum() / num_total
        else:
            l = (osm.cross_entropy_elem(x, labels, cw) * lw.float()).sum() / num_total
        loss_cls.append(cfg['loss_cls_weight'] * l)
        s = pred[b][..., -1:]
        p_, g_ = pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm']
        r = odef.mse_elem(p_, g_) if cfg['loss_reg'] == 'MSELoss' else op2p.smooth_l1_elem(p_, g_, cfg['sl1_beta'])
        loss_pts.append(cfg['loss_reg_weight'] * ((r * pw).sum() / num_total_pos))
    out = dict(loss_cls=loss_cls, loss_pts=loss_pts)
    if return_all:
        return out, dict(targets=tg, pred=pred, valid=valid, cls=cls)
    return out


def get_bboxes_single(pred_pts, cls_outs, L, img_shape, scale_factor, cfg, rescale=False):
    """ref:345-405: reshape the T rows into L equal chunks (RuntimeError when L does not divide T, as torch's reshape), per chunk the
    scores, the top nms_pre by the max foreground score, the clamp; then the chunk-major concatenation, the optional rescale and
    multiclass_nms.  Returns (cx, cy, score) (m,3), labels, dict(topk_inds [L x (nms_pre,)] or None, keep, cand_inds, pts, scores)."""
    sig = cfg.get('use_sigmoid', True)
    pred_pts = pred_pts.reshape(L, -1, 2)
    cls_outs = cls_outs.reshape(L, -1, cls_outs.shape[-1])
    pts_l, sc_l, topk_l = [], [], []
    for cs, pp in zip(cls_outs, pred_pts):
        scores = cs.sigmoid() if sig else cs.softmax(-1)
        nms_pre = cfg['nms_pre']
        if 0 < nms_pre < scores.shape[0]:
            mx, _ = (scores if sig else scores[:, :-1]).max(dim=1)
            _, ti = mx.topk(nms_pre)
            scores, pp = scores[ti, :], pp[ti, :]
            topk_l.append(ti)
        x = pp[:, 0].clamp(min=0, max=img_shape[1])
        y = pp[:, 1].clamp(min=0, max=img_shape[0])
        pts_l.append(torch.stack([x, y], dim=-1))
        sc_l.append(scores)
    pts, scores = torch.cat(pts_l), torch.cat(sc_l)
    if rescale:
        pts = pts / pts.new_tensor(scale_factor[:2])
    if sig:
        scores = torch.cat([scores, scores.new_zeros(scores.shape[0], 1)], dim=1)
    wh = pts.new_tensor(cfg['pseudo_wh'])
    boxes = torch.cat([pts - wh / 2, pts + wh / 2], dim=-1)
    dets, labels, keep, inds = op2p.multiclass_nms(boxes, scores, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    cxcy = torch.stack([(dets[:, 0] + dets[:, 2]) / 2, (dets[:, 1] + dets[:, 3]) / 2], dim=-1)
    return torch.cat([cxcy, dets[:, 4:5]], dim=1), labels, dict(topk_inds=topk_l or None, keep=keep, cand_inds=inds, pts=pts,
                                                               scores=scores[:, :-1])


def p2p_get_bboxes(cls_outs, pts_outs, img_metas, cfg, rescale=False, return_all=False):
    """ref:330-343 over the levels: per image (pseudo box (m,5), labels (m,))."""
    _, pred, _, cls = pred_points(cls_outs, pts_outs, img_metas, cfg)
    wh = pred.new_tensor(cfg['pseudo_wh'])
    res, aux = [], []
    for b, m in enumerate(img_metas):
        ps, labels, al = get_bboxes_single(pred[b][..., :2], cls[b], len(cls_outs), m['img_shape'], m['scale_factor'], cfg, rescale)
        res.append((torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], dim=-1), labels))
        aux.append(al)
    return (res, aux) if return_all else res


def aug_test_bboxes(aug_outs, aug_img_metas, cfg, rescale=False):
    """ref:487-572 after `self.forward(x)` per augmentation (aug_outs = [(cls_outs, pts_outs)] of one image each): the multi-level
    get_bboxes per view, then oracle/p2p.py's merge (sigmoid: a background column before the second multiclass_nms)."""
    C = cfg['num_classes']
    aug_b, aug_s = [], []
    for (cls_outs, pts_outs), metas in zip(aug_outs, aug_img_metas):
        boxes5, labels = p2p_get_bboxes(cls_outs, pts_outs, metas, cfg)[0]
        sc = boxes5.new_zeros((boxes5.shape[0], C))
        sc[torch.arange(boxes5.shape[0]), labels] = boxes5[:, 4]
        m = metas[0]
        aug_b.append(op2p.bbox_mapping_back(boxes5[:, :4], m['img_shape'], m['scale_factor'], m['flip'], m['flip_direction'],
                                            m.get('tile_offset', None)))
        aug_s.append(sc)
    mb, ms = torch.cat(aug_b), torch.cat(aug_s)
    if cfg.get('use_sigmoid', True):
        ms = torch.cat([ms, ms.new_zeros(ms.shape[0], 1)], dim=1)
    dets, labels, keep, inds = op2p.multiclass_nms(mb, ms, cfg['score_thr'], cfg['nms_iou'], cfg['max_per_img'])
    if not rescale:
        dets = dets.clone()
        dets[:, :4] *= dets.new_tensor(aug_img_metas[0][0]['scale_factor'])
    return [(dets, labels)], dict(keep=keep)
