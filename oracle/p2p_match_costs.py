"""ORACLE (test infrastructure, NOT product code) — HungarianAssignerV2's cost lists for the point costs.

Follows /root/reference/TOV_mmdetection/mmdet/core/bbox/assigners/hungarian_assigner.py:223-227 (`sum(cls_costs) + sum(reg_costs)`,
Python's sum from 0) and mmdet/core/bbox/match_costs/match_cost.py: FocalLossCost (:94-100), DisCostV2 (:197-214, torch.cdist with p
passed through), ZeroCost (:223-226), ClassificationCostV2 (:229-245).  A term is a dict as pointtinybenchmark_b200.assigners
.match_cost_terms makes it: 'kind' one of FocalLossCost, ClassificationCostV2_sigmoid, ClassificationCostV2_softmax, ZeroCost,
DisCostV2, and its parameters.  Only tests/ and oracle/make_golden_p2p_match_costs.py import this.
"""
from oracle import p2p as op2p

# the cost sets of tests/golden/p2p_match_costs.npz (oracle/make_golden_p2p_match_costs.py)
FOCAL = dict(kind='FocalLossCost', weight=2.0, alpha=0.25, gamma=2, eps=1e-12)
SIG = dict(kind='ClassificationCostV2_sigmoid', weight=1.0)
SOFT = dict(kind='ClassificationCostV2_softmax', weight=2.0)
ZERO = dict(kind='ZeroCost', weight=0.0)


def dis(p, weight, norm=True):
    return dict(kind='DisCostV2', weight=weight, p=p, norm_with_img_wh=norm)


PAPER = [SOFT, dis(2, 5e-2)]
# name -> (terms, N rows, n GTs, logit columns)
CASES = {
    'paper': (PAPER, 150, 12, 81),
    'sig_l1_norm': ([SIG, dis(1, 0.1, True)], 150, 12, 80),
    'zero_l2': ([ZERO, dis(2, 0.1, False)], 150, 12, 80),
    'multi': ([FOCAL, SIG, dis(1, 0.1), dis(2, 5e-2, False)], 150, 12, 80),
    'direct25': (PAPER, 25, 7, 81),
    'mm26': (PAPER, 26, 5, 81),
}
IMG_SHAPE = (110, 117, 3)

CLS_KINDS = ('FocalLossCost', 'ClassificationCostV2_sigmoid', 'ClassificationCostV2_softmax', 'ZeroCost')


def cls_cost(term, cls_pred, gt_labels):
    k, w = term['kind'], term['weight']
    if k == 'FocalLossCost':
        return op2p.focal_loss_cost(cls_pred, gt_labels, w, term['alpha'], term['gamma'], term['eps'])
    if k == 'ClassificationCostV2_sigmoid':
        return -cls_pred.sigmoid()[:, gt_labels] * w
    if k == 'ClassificationCostV2_softmax':
        return -cls_pred.softmax(dim=-1)[:, gt_labels] * w
    assert k == 'ZeroCost', k
    return 0


def cost_matrix(pts, cls_pred, gts, gt_labels, img_shape, terms):
    """(N, 2) points, (N, num_cols) logits, (n, 2) GT points -> (N, n) cost, summed as the reference sums it."""
    cls = [cls_cost(t, cls_pred, gt_labels) for t in terms if t['kind'] in CLS_KINDS]
    reg = [op2p.dis_cost_v2(pts, gts, img_shape, t['weight'], t['norm_with_img_wh'], t['p']) for t in terms if t['kind'] == 'DisCostV2']
    return sum(cls) + sum(reg)


def cost_config(terms):
    """the term list back as HungarianAssignerV2's (cls_costs, reg_costs) config lists"""
    cc, rc = [], []
    for t in terms:
        k = t['kind']
        if k == 'FocalLossCost':
            cc.append(dict(type=k, weight=t['weight'], alpha=t['alpha'], gamma=t['gamma'], eps=t['eps']))
        elif k.startswith('ClassificationCostV2'):
            cc.append(dict(type='ClassificationCostV2', weight=t['weight'], use_sigmoid=k.endswith('sigmoid')))
        elif k == 'ZeroCost':
            cc.append(dict(type=k))
        else:
            rc.append(dict(type=k, weight=t['weight'], p=t['p'], norm_with_img_wh=t['norm_with_img_wh']))
    return cc, rc
