"""CPU: MILLoss(loss_type='binary_cross_entropy') and AllPosLoss — the oracle against the golden vectors recorded from the REAL reference
(oracle/make_golden_cpr_loss_types.py), the float64 BCE term against torch's binary_cross_entropy, and the head's config checks."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cpr_loss_types as olt
from oracle.make_golden_cpr_loss_types import LOSS_TYPE_CASES, loss_type_inputs, oracle_cfg
from tests.cpr_loss_types_ref import bce


@pytest.mark.parametrize('case', list(LOSS_TYPE_CASES))
def test_oracle_matches_reference_golden(golden_dir, case):
    gold = np.load(os.path.join(golden_dir, f'cpr_lite_loss_{case}.npz'))
    inp, w, gtw = loss_type_inputs(case, int(gold['seed']))
    cfg = oracle_cfg(case, inp['cfgd'])
    f = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    ol = olt.cpr_loss(f, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, gt_weights=gtw)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
        np.testing.assert_allclose(ol[k].detach().reshape(-1).numpy(), gold['loss_' + k], rtol=1e-6, atol=1e-7, err_msg=k)
    sub = f.grad.flatten()[::211].numpy()
    assert np.abs(sub - gold['grad_feat_sub']).max() <= 1e-6 * max(1.0, np.abs(gold['grad_feat_sub']).max())
    for name, key in (('cls_out.weight', 'grad_cls_w'), ('cls_out.bias', 'grad_cls_b'), ('ins_out.weight', 'grad_ins_w'),
                      ('ins_out.bias', 'grad_ins_b')):
        np.testing.assert_allclose(wo[name].grad.numpy(), gold[key], rtol=0, atol=1e-6 * max(1.0, np.abs(gold[key]).max()), err_msg=name)
    if cfg.get('loss_mil', 'MILLoss') == 'AllPosLoss':
        assert not gold['grad_ins_w'].any() and not gold['grad_ins_b'].any()


def test_fully_invalid_bag_scores_100_under_bce():
    """the appended GT lies outside pad_shape: its bag probability is exactly 0 and BCE adds 100 at its label column."""
    inp, w, _ = loss_type_inputs('mil_bce')
    cfg = oracle_cfg('mil_bce', inp['cfgd'])
    _, oall = olt.cpr_loss(inp['cls_feat'], w, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    assert not oall['ex']['pos_valid'][-1].any()
    p = oall['bag_prob'][-1]
    assert torch.equal(p, torch.zeros_like(p))
    onehot = torch.zeros_like(p)
    onehot[int(inp['gt_labels'][0][-1])] = 1
    assert float(olt.bce_loss(p, onehot).sum()) == 100.0


@pytest.mark.parametrize('t', [0.0, 1.0])
def test_bce_term_matches_torch(t):
    """float64 restatement of ATen's BCE (value and gradient) against F.binary_cross_entropy on the CPU, at the edges and at random p."""
    g = torch.Generator().manual_seed(7)
    edges = torch.tensor([0.0, 1.0, 1e-30, 1.0 - 2.0 ** -24], dtype=torch.float64)
    p = torch.cat([edges, torch.rand(200, generator=g, dtype=torch.float64)])
    tt = torch.full_like(p, t)
    for dtype in (torch.float64, torch.float32):
        a = p.to(dtype).clone().requires_grad_(True)
        b = p.to(dtype).clone().requires_grad_(True)
        va = bce(a, tt.to(dtype))
        vb = F.binary_cross_entropy(b, tt.to(dtype), reduction='none')
        torch.testing.assert_close(va, vb, rtol=1e-6 if dtype == torch.float32 else 1e-12, atol=0)
        va.sum().backward()
        vb.sum().backward()
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-6 if dtype == torch.float32 else 1e-12, atol=0)
    # the clamps: log(0) -> -100, and the gradient's denominator 1e-12
    assert float(bce(torch.tensor([0.0], dtype=torch.float64), torch.tensor([1.0], dtype=torch.float64))) == 100.0


def _head(loss_mil, pos='CirclePtFeatGenerator'):
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    gen = dict(type=pos, radius=2)
    return build_head(dict(type='CPRHead', num_classes=4, in_channels=32, feat_channels=32, stacked_convs=1, strides=[8],
                           norm_cfg=dict(type='GN', num_groups=8), loss_mil=loss_mil,
                           train_pts_extractor=dict(pos_generator=gen, neg_generator=dict(type='OutCirclePtFeatGenerator', radius=2)),
                           refine_pts_extractor=dict(pos_generator=gen, neg_generator=dict(type='AnchorPtFeatGenerator'))))


@pytest.mark.parametrize('typ', ['MILLoss', 'AllPosLoss'])
@pytest.mark.parametrize('loss_type', ['gfocal_loss', 'binary_cross_entropy'])
def test_configs_with_either_loss_build(typ, loss_type):
    head = _head(dict(type=typ, loss_weight=0.25, loss_type=loss_type))
    assert head.loss_mil_cfg['type'] == typ and head.loss_mil_cfg['loss_type'] == loss_type


@pytest.mark.parametrize('loss_mil', [dict(type='MILLoss', loss_type='focal_loss'), dict(type='AllPosLoss', loss_type='ce'),
                                      dict(type='MIL2Loss')])
def test_unknown_loss_types_raise(loss_mil):
    with pytest.raises(NotImplementedError):
        _head(loss_mil)


def test_allpos_with_grid_bags_raises():
    with pytest.raises(NotImplementedError):
        _head(dict(type='AllPosLoss'), pos='GridCirclesPtFeatGenerator')
