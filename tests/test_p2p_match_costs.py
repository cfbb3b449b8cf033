"""CPU: HungarianAssignerV2's cost lists (assigners.match_cost_terms): the refusals, that a list of several costs is parsed whole,
which library function each list is sent to, and the oracle against the golden vectors of the real reference
(tests/golden/p2p_match_costs.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p, p2p_match_costs as omc
from pointtinybenchmark_b200 import assigners, ops

FOCAL = dict(type='FocalLossCost', weight=2.0)
DIS = dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False)


class FakeCuda(torch.Tensor):
    """a CPU tensor that reports is_cuda: lets the assigner's CUDA-only guard pass in this dry run"""
    is_cuda = property(lambda s: True)


@pytest.mark.parametrize('cls_costs, reg_costs, match', [
    (dict(type='ClassificationCost', weight=1.0), DIS, 'ClassificationCostV2'),
    (FOCAL, dict(type='BBoxL1Cost', weight=1.0), 'BBoxL1Cost'),
    (FOCAL, dict(type='IoUCost', iou_mode='giou'), 'IoUCost'),
    (FOCAL, dict(type='IoUCostV2', iou_mode='giou'), 'IoUCostV2'),
    (FOCAL, dict(type='ZeroCost'), 'ZeroCost'),
    (FOCAL, [DIS, dict(type='FocalLossCost')], 'FocalLossCost'),
    (DIS, DIS, 'DisCostV2'),
    (FOCAL, dict(type='DisCostV2', p=3), 'DisCostV2 p=3'),
    (FOCAL, dict(type='PointsDisCost', p=2), 'PointsDisCost'),
    ([FOCAL] * 9, DIS, 'at most 8'),
    (FOCAL, [DIS] * 9, 'at most 8'),
])
def test_refused_costs(cls_costs, reg_costs, match):
    with pytest.raises(NotImplementedError, match=match):
        assigners.match_cost_terms(cls_costs, reg_costs)
    with pytest.raises(NotImplementedError, match=match):
        assigners.HungarianAssignerV2(cls_costs=cls_costs, reg_costs=reg_costs)


def test_discost_on_more_than_xy_is_refused():
    A = assigners.HungarianAssignerV2(cls_costs=FOCAL, reg_costs=DIS)
    fc = lambda t: t.as_subclass(FakeCuda)  # noqa: E731
    with pytest.raises(NotImplementedError, match='DisCostV2'):
        A.assign(fc(torch.zeros(4, 4)), fc(torch.zeros(4, 3)), fc(torch.zeros(2, 4)), fc(torch.zeros(2, dtype=torch.long)),
                 dict(img_shape=(10, 10, 3)))


def test_two_entry_lists_are_parsed_whole():
    sig = dict(type='ClassificationCostV2', use_sigmoid=True, weight=0.5)
    l2 = dict(type='DisCostV2', weight=5e-2, p=2)
    terms = assigners.match_cost_terms([FOCAL, sig], [DIS, l2])
    assert [t['kind'] for t in terms] == ['FocalLossCost', 'ClassificationCostV2_sigmoid', 'DisCostV2', 'DisCostV2']
    assert terms[1]['weight'] == 0.5 and (terms[2]['p'], terms[3]['p']) == (1, 2)
    assert (terms[2]['norm_with_img_wh'], terms[3]['norm_with_img_wh']) == (False, True)
    from pointtinybenchmark_b200.p2p_head import P2PHead
    head = P2PHead(num_classes=4, in_channels=32, feat_channels=32, stacked_convs=1, strides=[8],
                   norm_cfg=dict(type='GN', num_groups=8, requires_grad=True),
                   train_cfg=dict(assigner=dict(type='HungarianAssignerV2', cls_costs=[FOCAL, sig], reg_costs=[DIS, l2], topk_k=5)))
    assert head.assign['terms'] == terms and head.assign['topk_k'] == 5


def test_softmax_and_zero_terms():
    terms = assigners.match_cost_terms(dict(type='ZeroCost'), dict(type='DisCostV2', weight=5e-2, p=2))
    assert [t['kind'] for t in terms] == ['ZeroCost', 'DisCostV2']
    terms = assigners.match_cost_terms(dict(type='ClassificationCostV2', weight=2.0), [])
    assert terms == [dict(kind='ClassificationCostV2_softmax', weight=2.0)]      # use_sigmoid defaults to False (match_cost.py:231)


def test_dispatch(monkeypatch):
    """the shipped pair goes to ops.p2p_cost_matrix with its scalars, every other list to ops.p2p_cost_matrix_terms"""
    calls = []
    monkeypatch.setattr(ops, 'p2p_cost_matrix', lambda *a, **k: calls.append(('pair', a[5:], k)))
    monkeypatch.setattr(ops, 'p2p_cost_matrix_terms', lambda *a, **k: calls.append(('terms', a[5:], k)))
    x = torch.zeros(1)
    pair = assigners.match_cost_terms(dict(FOCAL, alpha=0.3), dict(DIS, norm_with_img_wh=True))
    assigners.cost_matrix(x, x, None, x, x, pair, (110, 117, 3))
    assert calls[-1][0] == 'pair' and calls[-1][1] == (2.0, 0.3, 2, 1e-12, 0.1, 117.0, 110.0)
    assigners.cost_matrix(x, x, None, x, x, assigners.match_cost_terms(FOCAL, DIS), (110, 117, 3))
    assert calls[-1][1][-2:] == (1.0, 1.0)
    for cc, rc in ((FOCAL, dict(DIS, p=2)), ([FOCAL, FOCAL], DIS), (FOCAL, [DIS, DIS]), (dict(type='ZeroCost'), DIS),
                   (dict(type='ClassificationCostV2'), DIS)):
        terms = assigners.match_cost_terms(cc, rc)
        assigners.cost_matrix(x, x, None, x, x, terms, (110, 117, 3))
        assert calls[-1][0] == 'terms' and calls[-1][1][0] == terms


@pytest.mark.parametrize('name', list(omc.CASES))
def test_oracle_matches_golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, 'p2p_match_costs.npz'))
    terms = omc.CASES[name][0]
    t = lambda k: torch.from_numpy(g[f'{name}_{k}'])  # noqa: E731
    cost = omc.cost_matrix(t('pts'), t('cls'), t('gts'), t('labels'), omc.IMG_SHAPE, terms)
    assert np.array_equal(cost.numpy().view(np.int32), g[f'{name}_cost'].view(np.int32)), name
    for k in (1, 5):
        gi, _ = op2p.hungarian_v2_from_cost(cost, t('labels'), k)
        assert np.array_equal(gi.numpy().astype(np.int32), g[f'{name}_gt_inds_k{k}']), (name, k)
