"""ORACLE (test infrastructure, NOT product code) — P2PHead trained with GHMC, GHMR, L1Loss or BalancedL1Loss.

Follows /root/reference/TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py:172-248 (loss: loss_single per image through
multi_apply) with mmdet/models/losses/ghm_loss.py:21-172 (GHMC, GHMR), smooth_l1_loss.py:33-45 (L1Loss) and balanced_l1_loss.py:12-49
(BalancedL1Loss).  The GHM losses are restated without their per-bin loop: every element's bin comes from one comparison against all
edges, the bin counts from a sum, and the weights from the fp32 operation order the reference's python / 0-d tensor arithmetic has:
  tot = max(valid count, 1);  no momentum:  w_i = fp32(tot / cnt_i) (python floats);
  momentum:  acc_i = fp32(mmt) * acc_i + fp32((1 - mmt) * cnt_i),  w_i = (1 / acc_i) * tot (python float / tensor = reciprocal * tot);
  then w_i / n (fp32), n = non-empty bins.
oracle/make_golden_p2p_loss_types.py asserts acc_sum bit-equal to the reference's and the losses and gradients equal within 1e-6.
The proposal rows and targets are oracle/p2p_multilevel.py's (one level or several).  Only tests/ and that recipe import this.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_defaults as odef, p2p_multilevel as oml
from oracle.synth import sample_points

C_FEAT = oml.C_FEAT
# Each case: seed, strides, anchors k, classes, map sizes per level, the two loss configs as a P2PHead config writes them, the
# number of consecutive training steps (the momentum cases record acc_sum after each), and `pad_small`: image 1's pad shape leaves
# it 2 x 2 valid cells (the reference cannot train an image without a valid row: its get_targets fails).
CASES = {
    # TinyPerson: one class, one anchor, stride 4, GHMC bins=10 (with the shipped SmoothL1 points)
    'tinyperson_ghmc': dict(seed=6101, strides=[4], k=1, num_classes=1, maps=[(16, 16)],
                            loss_cls=dict(type='GHMC', bins=10, momentum=0, use_sigmoid=True, loss_weight=1.0),
                            loss_reg=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5)),
    # the reference defaults (80 classes, four anchors) with GHMC bins=30, momentum=0.75 over three steps
    'defaults_ghmc_mmt': dict(seed=6102, strides=[8], k=4, num_classes=80, maps=[(6, 6)], steps=3,
                              loss_cls=dict(type='GHMC', bins=30, momentum=0.75, use_sigmoid=True, loss_weight=1.0),
                              loss_reg=dict(type='MSELoss', loss_weight=2e-4)),
    # GHMR mu=0.02 with momentum over two steps, Focal classification
    'ghmr_mmt': dict(seed=6103, strides=[8], k=1, num_classes=4, maps=[(12, 12)], steps=2,
                     loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                     loss_reg=dict(type='GHMR', mu=0.02, bins=10, momentum=0.7, loss_weight=1.0)),
    'l1': dict(seed=6104, strides=[8], k=1, num_classes=4, maps=[(12, 12)],
               loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
               loss_reg=dict(type='L1Loss', loss_weight=0.5)),
    'balanced_l1': dict(seed=6105, strides=[8], k=1, num_classes=4, maps=[(12, 12)],
                        loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                        loss_reg=dict(type='BalancedL1Loss')),
    'balanced_l1_custom': dict(seed=6106, strides=[8], k=1, num_classes=4, maps=[(12, 12)],
                               loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                               loss_reg=dict(type='BalancedL1Loss', alpha=0.3, gamma=1.0, beta=0.5, loss_weight=2.0)),
    # two levels, GHMC + GHMR without momentum
    'two_level_ghm': dict(seed=6107, strides=[8, 16], k=1, num_classes=4, maps=[(12, 12), (6, 6)],
                          loss_cls=dict(type='GHMC', bins=10, use_sigmoid=True, loss_weight=1.0),
                          loss_reg=dict(type='GHMR', mu=0.02, bins=10, loss_weight=1.0)),
    # image 1 almost all invalid rows; GHMC with momentum and GHMR, most bins empty
    'edge_invalid_image': dict(seed=6108, strides=[8], k=1, num_classes=4, maps=[(10, 10)], pad_small=True,
                               loss_cls=dict(type='GHMC', bins=30, momentum=0.75, use_sigmoid=True, loss_weight=1.0),
                               loss_reg=dict(type='GHMR', mu=0.02, bins=30, loss_weight=1.0)),
}
# GHMR's g must lie at least this far from every bin edge: its d = (pred - target) / stride rounds differently on the device.  GHMC's
# margin is recorded only: its g is bit-exact from the same logits, and the tests that recompute the logits read the recorded margin.
SAFE_MARGIN = 1e-5


def case_cfg(name):
    c = CASES[name]
    anchors = list(odef.ANCHORS) if c['k'] == 4 else [(0., 0.)]
    cfg = odef.reference_defaults_cfg(num_classes=c['num_classes'], point_anchor=anchors, strides=list(c['strides']),
                                      stride=c['strides'][0], loss_cls=c['loss_cls']['type'], loss_reg=c['loss_reg']['type'])
    if c['k'] == 1:
        cfg.update(pts_gamma=1.0, reg_norm=1.0)
    cfg.update(loss_cls_cfg=dict(c['loss_cls']), loss_reg_cfg=dict(c['loss_reg']))
    return cfg


def case_inputs(name, step=0, B=2, n=6):
    """seeded weights (the same at every step) and, per step, ReLU feature maps per level, GT points and metas.  CPU generator."""
    c = CASES[name]
    cfg = case_cfg(name)
    gen = torch.Generator().manual_seed(c['seed'])
    w = oml.weights(gen, c['k'], c['num_classes'], False)
    gen = torch.Generator().manual_seed(c['seed'] * 10 + step)
    xs = [torch.relu(torch.randn(B, C_FEAT, h, wd, generator=gen)) for h, wd in c['maps']]
    H0, W0 = c['maps'][0]
    s0 = c['strides'][0]
    pads = [(H0 * s0, W0 * s0), (2 * s0, 2 * s0) if c.get('pad_small') else (H0 * s0 - 2 * s0, W0 * s0 - s0)]
    gt_bboxes, gt_labels, metas = [], [], []
    for b in range(B):
        ih, iw = max(pads[b][0] - 3, s0), max(pads[b][1] - 2, s0)
        pts = sample_points(n, iw, ih, gen)
        gt_bboxes.append(torch.cat([pts - 4, pts + 4], dim=1))
        gt_labels.append(torch.randint(0, c['num_classes'], (n,), generator=gen))
        metas.append(dict(pad_shape=pads[b] + (3,), img_shape=(ih, iw, 3), scale_factor=[1.0, 1.0, 1.0, 1.0]))
    return dict(xs=xs, weights=w, gt_bboxes=gt_bboxes, gt_labels=gt_labels, img_metas=metas), cfg


def ghm_edges(bins, last):
    """ghm_loss.py:39-41 / 117-119: arange(bins + 1) / bins in fp32, the last edge + 1e-6 (GHMC) or 1e3 (GHMR)."""
    e = torch.arange(bins + 1).float() / bins
    e[-1] = e[-1] + 1e-6 if last is None else last
    return e


def bin_of(g, valid, edges):
    """(n,) bin index of every valid element, -1 for none: the edges are nondecreasing, so at most one bin holds g."""
    inside = (g[:, None] >= edges[None, :-1]) & (g[:, None] < edges[None, 1:]) & valid[:, None]
    return torch.where(inside.any(1), inside.float().argmax(1), torch.full_like(g, -1, dtype=torch.long))


def bin_weights(counts, n_valid, mmt, acc_sum):
    """per-bin element weights of one image and its tot; acc_sum (fp32 tensor) is updated in place when mmt > 0."""
    tot = np.float32(max(float(n_valid), 1.0))
    nb = int((counts > 0).sum())
    w = np.zeros(len(counts), np.float32)
    for i, cnt in enumerate(counts.tolist()):
        if cnt == 0:
            continue
        if mmt > 0:
            a = np.float32(np.float32(mmt) * np.float32(acc_sum[i].item())) + np.float32((1 - mmt) * cnt)
            acc_sum[i] = float(np.float32(a))
            w[i] = np.float32(np.float32(1) / np.float32(a)) * tot
        else:
            w[i] = np.float32(float(tot) / cnt)
        w[i] = np.float32(w[i] / np.float32(nb))
    return torch.from_numpy(w), float(tot)


def ghm_margin(g, valid, edges):
    """smallest |g - edge| over the valid elements: how far the bin decision is from flipping."""
    gv = g[valid].double()
    return float((gv[:, None] - edges.double()[None, :]).abs().min()) if gv.numel() else float('inf')


def ghmc(pred, labels, label_weight, edges, mmt=0.0, acc_sum=None, loss_weight=1.0):
    """GHMC of one image (Q, C): returns loss, counts (bins,), n_valid, margin."""
    C = pred.shape[1]
    t = F.one_hot(labels.clamp(0, C), C + 1)[:, :C].float()
    valid = (label_weight[:, None] > 0).expand_as(pred).reshape(-1)
    g = (pred.detach().sigmoid() - t).abs().reshape(-1)
    b = bin_of(g, valid, edges)
    bins = edges.numel() - 1
    counts = torch.bincount(b[b >= 0], minlength=bins)
    bw, tot = bin_weights(counts, int(valid.sum()), mmt, acc_sum)
    w = torch.where(b >= 0, bw[b.clamp(min=0)], torch.zeros_like(g)).reshape(pred.shape)
    loss = F.binary_cross_entropy_with_logits(pred, t, w, reduction='sum') / tot
    return loss * loss_weight, counts, int(valid.sum()), ghm_margin(g, valid, edges)


def ghmr(pred, target, label_weight, edges, mu=0.02, mmt=0.0, acc_sum=None, loss_weight=1.0):
    """GHMR of one image's normalised (Q, 2) points: returns loss, counts, n_valid, margin."""
    d = pred - target
    root = torch.sqrt(d * d + mu * mu)
    valid = (label_weight > 0).reshape(-1)
    g = (d / root).abs().detach().reshape(-1)
    b = bin_of(g, valid, edges)
    counts = torch.bincount(b[b >= 0], minlength=edges.numel() - 1)
    bw, tot = bin_weights(counts, int(label_weight.float().sum()), mmt, acc_sum)
    w = torch.where(b >= 0, bw[b.clamp(min=0)], torch.zeros_like(g)).reshape(d.shape)
    return ((root - mu) * w).sum() / tot * loss_weight, counts, int(valid.sum()), ghm_margin(g, valid, edges)


def l1_elem(pred, target):
    return (pred - target).abs()


def balanced_l1_elem(pred, target, alpha=0.5, gamma=1.5, beta=1.0):
    a = (pred - target).abs()
    b = np.e ** (gamma / alpha) - 1
    inner = alpha / b * (b * a + 1) * torch.log(b * a / beta + 1) - alpha * a
    return torch.where(a < beta, inner, gamma * a + gamma / b - alpha * beta)


def make_state(cfg):
    """the GHM buffers of a head built from cfg: {'loss_cls.edges': ..., 'loss_cls.acc_sum': ...} as the reference names them."""
    st = {}
    for key, last in (('loss_cls', None), ('loss_reg', 1e3)):
        c = cfg[key + '_cfg']
        if c['type'] in ('GHMC', 'GHMR'):
            bins = c.get('bins', 10)
            st[f'{key}.edges'] = ghm_edges(bins, last)
            if c.get('momentum', 0) > 0:
                st[f'{key}.acc_sum'] = torch.zeros(bins)
    return st


def p2p_loss(cls_outs, pts_outs, gt_bboxes, gt_labels, img_metas, cfg, state, return_all=False):
    """ref:172-248 with the configured losses; state (make_state) is updated in place.  Returns dict(loss_cls=[B], loss_pts=[B])
    and, with return_all, the targets and per image the GHM counts (bins + 1 columns: the last is the valid count) and margins."""
    anchor, pred, valid, cls = oml.pred_points(cls_outs, pts_outs, img_metas, cfg)
    gt_points = [(b[:, :2] + b[:, 2:]) / 2 for b in gt_bboxes]
    prop = anchor if cfg['assign_before_pred'] else pred
    tg = [op2p.target_single(prop[b][..., :2].detach(), valid[b], cls[b].detach(), gt_points[b], gt_labels[b],
                             img_metas[b]['img_shape'], cfg) for b in range(len(img_metas))]
    num_total_pos = sum([(t[3][..., 0] > 0).sum() for t in tg])
    cc, rc = cfg['loss_cls_cfg'], cfg['loss_reg_cfg']
    loss_cls, loss_pts, aux = [], [], dict(targets=tg, cls_counts=[], reg_counts=[], cls_margin=[], reg_margin=[])
    for b, (labels, lw, gpts, pw, _) in enumerate(tg):
        x = cls[b].contiguous()
        if cc['type'] == 'GHMC':
            l, cnt, nv, mg = ghmc(x, labels, lw, state['loss_cls.edges'], cc.get('momentum', 0), state.get('loss_cls.acc_sum'),
                                  cc.get('loss_weight', 1.0))
            aux['cls_counts'].append(torch.cat([cnt, torch.tensor([nv])]))
            aux['cls_margin'].append(mg)
        else:
            l = (op2p.sigmoid_focal_loss_elem(x, labels, cc['gamma'], cc['alpha']) * lw.view(-1, 1)).sum() / num_total_pos
            l = cc.get('loss_weight', 1.0) * l
        loss_cls.append(l)
        s = pred[b][..., -1:]
        p_, g_ = pred[b][..., :2] / s / cfg['reg_norm'], gpts / s / cfg['reg_norm']
        if rc['type'] == 'GHMR':
            r, cnt, nv, mg = ghmr(p_, g_, pw, state['loss_reg.edges'], rc.get('mu', 0.02), rc.get('momentum', 0),
                                  state.get('loss_reg.acc_sum'), rc.get('loss_weight', 1.0))
            aux['reg_counts'].append(torch.cat([cnt, torch.tensor([nv])]))
            aux['reg_margin'].append(mg)
            loss_pts.append(r)
            continue
        if rc['type'] == 'L1Loss':
            e = l1_elem(p_, g_)
        elif rc['type'] == 'BalancedL1Loss':
            e = balanced_l1_elem(p_, g_, rc.get('alpha', 0.5), rc.get('gamma', 1.5), rc.get('beta', 1.0))
        elif rc['type'] == 'MSELoss':
            e = odef.mse_elem(p_, g_)
        else:
            e = op2p.smooth_l1_elem(p_, g_, rc['beta'])
        loss_pts.append(rc.get('loss_weight', 1.0) * ((e * pw).sum() / num_total_pos))
    out = dict(loss_cls=loss_cls, loss_pts=loss_pts)
    if return_all:
        return out, dict(aux, pred=pred, valid=valid, cls=cls)
    return out
