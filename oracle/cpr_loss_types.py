"""ORACLE (test infrastructure, NOT product code) — CPU restatement of the positive-bag losses the reference registers for
CPRHead's `loss_mil` beyond the gfocal MILLoss of oracle/cpr.py:

  MILLoss(loss_type='binary_cross_entropy')   multi_instance_learning_loss.py:153-203 (:187-202 the loss-type switch)
  AllPosLoss(loss_type='gfocal_loss' | 'binary_cross_entropy')   multi_instance_learning_loss.py:206-243

and CPRHead.loss + loss0 (ref:1101-1117, 1131-1229) with either of them in place of the MIL loss.  Everything else (bag extraction, the
point classifiers, get_cls_prob, gfocal_loss, the MIL bag probability, the gt and neg terms) is oracle/cpr.py's.

Config: oracle.cpr.default_cfg(..., loss_mil='MILLoss' | 'AllPosLoss', mil_loss_type='gfocal_loss' | 'binary_cross_entropy').
PINNED: oracle/make_golden_cpr_loss_types.py runs the real reference head on the same inputs and asserts this restatement reproduces it.
"""
import torch
import torch.nn.functional as F

from oracle import cpr as ocpr


def bce_loss(p, q):
    """F.binary_cross_entropy(p, q, None, reduction='none') as MILLoss / AllPosLoss call it (multi_instance_learning_loss.py:202, 240):
    no weight, so zero-weight bags and invalid samples count too."""
    return F.binary_cross_entropy(p, q, None, reduction='none')


def bag_term(p, q, w, eps, loss_type):
    """per-row loss of the positive bags: gfocal_loss(p, q, w) (summed over classes) or the unweighted BCE summed over classes."""
    if loss_type == 'gfocal_loss':
        return ocpr.gfocal_loss(p, q, w, eps)
    if loss_type == 'binary_cross_entropy':
        return bce_loss(p, q).sum(dim=-1)
    raise ValueError(loss_type)


def mil_loss(bag_cls_prob, bag_ins_outs, labels, valid, loss_weight=1.0, eps=1e-6, binary_ins=False, loss_type='gfocal_loss'):
    """MILLoss.forward (multi_instance_learning_loss.py:153-203) with either loss_type; binary_ins doubles the instance head (a positive
    and a negative bag probability per class, the negative one trained towards 0, :179-186).  returns loss, acc (top-1 %), num_sample,
    prob (B,C) of the positive head."""
    B, N, C = bag_cls_prob.shape
    nb = 2 if binary_ins else 1
    prob_ins = bag_ins_outs.reshape(B, N, C, nb).softmax(dim=1) * valid.unsqueeze(-1)
    prob_ins = F.normalize(prob_ins, dim=1, p=1)
    prob2 = (bag_cls_prob.unsqueeze(-1) * prob_ins).sum(dim=1)                          # (B, C, nb)
    pred_label = prob2[..., 0].topk(1, dim=1)[1][:, 0]
    acc = (pred_label == labels).float().sum(0, keepdim=True) * (100.0 / max(B, 1))
    label_weights = (valid.sum(dim=1) > 0).float()
    onehot = torch.zeros(B, C)
    onehot[torch.arange(B), labels] = 1
    num_sample = max(torch.sum(label_weights.sum(dim=-1) > 0).float().item(), 1.)
    if binary_ins:
        prob = torch.cat([prob2[..., 0], prob2[..., 1]])
        loss = bag_term(prob, torch.cat([onehot, torch.zeros_like(onehot)]), torch.cat([label_weights, label_weights]), eps, loss_type)
    else:
        loss = bag_term(prob2[..., 0], onehot, label_weights, eps, loss_type)
    return loss.sum() / num_sample * loss_weight, acc, num_sample, prob2[..., 0]


def allpos_loss(bag_cls_prob, bag_ins_outs, labels, valid, loss_weight=1.0, eps=1e-6, loss_type='gfocal_loss'):
    """AllPosLoss.forward (multi_instance_learning_loss.py:206-243): every bag sample is a row with its bag's label; gfocal rows are
    weighted by valid, BCE rows are not.  The reference returns loss + bag_ins_outs * 0; mmdet's _parse_losses reduces that with
    .mean(), which is what this returns (the scalar, with a zero gradient to the instance logits).  returns loss, acc, num_sample."""
    B, N, C = bag_cls_prob.shape
    prob = bag_cls_prob.reshape(B * N, C)
    lab = labels.unsqueeze(-1).repeat(1, N).flatten()
    w = valid.reshape(B * N, -1).float()
    pred_label = prob.topk(1, dim=1)[1][:, 0]
    acc = (pred_label == lab).float().sum(0, keepdim=True) * (100.0 / max(B * N, 1))
    onehot = torch.zeros(B * N, C)
    onehot[torch.arange(B * N), lab] = 1
    num_sample = max(torch.sum(w.sum(dim=-1) > 0).float().item(), 1.)
    loss = bag_term(prob, onehot, w, eps, loss_type).sum() / num_sample * loss_weight
    return loss + (bag_ins_outs * 0).mean(), acc, num_sample


def cpr_loss(cls_feat, weights, gt_bboxes, gt_labels, img_metas, cfg, return_all=False, gt_weights=None):
    """oracle.cpr.cpr_loss with cfg['loss_mil'] / cfg['mil_loss_type'] selecting the positive-bag loss (ins_share_head_feat=True,
    refine_bag_policy 'only_refine_bag' at num_refine = 1, the policy every test here uses)."""
    gt_points = ocpr.pseudo_bbox_to_center(gt_bboxes)
    gt_r_points = [p.reshape(len(l), -1, *p.shape[1:]) for p, l in zip(gt_points, gt_labels)]
    ex = ocpr.extract(cls_feat, gt_r_points, gt_labels, img_metas, cfg)
    nf = cfg.get('num_cls_fcs', 0)
    pos_cls = ocpr.pts_outs(ex['pos_feats'], weights, 'cls_out', nf)
    pos_ins = ocpr.pts_outs(ex['pos_feats'], weights, 'ins_out', nf)
    neg_cls = ocpr.pts_outs(ex['neg_feats'], weights, 'cls_out', nf)
    labels_all = torch.cat(gt_labels)
    gt_weights = torch.ones(len(labels_all)) if gt_weights is None else torch.cat(list(gt_weights)).float()      # ref:1108-1114
    pos_valid, neg_valid = ex['pos_valid'], ex['neg_valid']
    G, R, K, _ = ex['pos_pts'].shape
    assert R == 1 and cfg['refine_bag_policy'] == 'only_refine_bag'
    losses = {}
    num_pos = None
    if cfg['with_gt_loss']:
        gt_cls_prob = ocpr.cls_prob(pos_cls[..., -1, :].reshape(G, -1), cfg)
        w_rep = pos_valid[..., -1, :].reshape(G, -1).float() * gt_weights.reshape(-1, 1)
        onehot = torch.zeros_like(gt_cls_prob)
        onehot[torch.arange(G), labels_all] = 1
        num_pos = max((w_rep > 0).sum(), 1)
        losses['gt_loss'] = cfg['gt_loss_weight'] * (ocpr.gfocal_loss(gt_cls_prob, onehot, w_rep, cfg['mil_eps']).sum() / num_pos)
    bag_prob = None
    if cfg['with_mil_loss']:
        c_, i_, v_ = (t.reshape(G, K, -1) for t in (pos_cls, pos_ins, pos_valid))
        pos_w = v_.float() * gt_weights.reshape(-1, 1, 1)
        loss_type = cfg.get('mil_loss_type', 'gfocal_loss')
        if cfg.get('loss_mil', 'MILLoss') == 'AllPosLoss':
            pos_loss, acc, num_pos = allpos_loss(ocpr.cls_prob(c_, cfg), i_, labels_all, pos_w, cfg['mil_loss_weight'], cfg['mil_eps'],
                                                 loss_type)
        else:
            pos_loss, acc, num_pos, bag_prob = mil_loss(ocpr.cls_prob(c_, cfg), i_, labels_all, pos_w, cfg['mil_loss_weight'],
                                                        cfg['mil_eps'], cfg.get('binary_ins', False), loss_type)
        losses['pos_loss'] = pos_loss
        losses['bag_acc'] = acc
    if cfg['with_neg']:
        neg_prob = ocpr.cls_prob(neg_cls, cfg)
        nl = ocpr.gfocal_loss(neg_prob, torch.zeros_like(neg_prob), neg_valid.float(), cfg['mil_eps'])
        losses['neg_loss'] = cfg['neg_loss_weight'] * (nl.sum() / num_pos)
    if return_all:
        return losses, dict(ex=ex, pos_cls=pos_cls, pos_ins=pos_ins, neg_cls=neg_cls, bag_prob=bag_prob)
    return losses
