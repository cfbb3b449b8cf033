"""CPU: P2PHead with GHMC, GHMR, L1Loss and BalancedL1Loss.  The oracle (oracle/p2p_loss_types.py) against the vectors the REAL
reference head produced (tests/golden/p2p_loss_types_*.npz, written by oracle/make_golden_p2p_loss_types.py): losses, per-image bin
counts, acc_sum after every step and the output-map gradients; the GHM heads' state_dict names and shapes against the reference's,
with a strict load both ways; and the refusals: GHMC(use_sigmoid=False), more than 256 bins, a loaded edges buffer that decreases,
and the reference losses that cannot run on P2PHead's targets."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_loss_types as olt, p2p_multilevel as oml
from oracle.make_golden_p2p_loss_types import head_kwargs
from pointtinybenchmark_b200.p2p_head import P2PHead


def _close(a, ref, tol, what):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    d = np.abs(a - ref).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref).max()), f'{what}: max |diff| {d:.3e}'


@pytest.mark.parametrize('name', sorted(olt.CASES))
def test_oracle_matches_reference_golden(golden_dir, name):
    gold = np.load(os.path.join(golden_dir, f'p2p_loss_types_{name}.npz'))
    assert int(gold['seed']) == olt.CASES[name]['seed']
    _, cfg = olt.case_inputs(name)
    state = olt.make_state(cfg)
    for k, v in state.items():
        assert np.array_equal(v.numpy(), gold[f'edges_init/{k}'])
    steps = olt.CASES[name].get('steps', 1)
    for step in range(steps):
        inp, _ = olt.case_inputs(name, step)
        oc, opo = oml.head_forward(inp['xs'], inp['weights'], cfg)
        oc = [c.detach().requires_grad_(True) for c in oc]
        opo = [p.detach().requires_grad_(True) for p in opo]
        loss, aux = olt.p2p_loss(oc, opo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, state, return_all=True)
        (sum(loss['loss_cls']) + sum(loss['loss_pts'])).backward()
        for k in ('loss_cls', 'loss_pts'):
            _close(torch.stack([v.reshape(()) for v in loss[k]]).detach().numpy(), gold[f'{k}/{step}'], 1e-6, f'{name} {k}')
        for k, v in state.items():
            if k.endswith('acc_sum'):
                assert np.array_equal(v.numpy(), gold[f'{k}/{step}']), f'{name} step {step} {k}'
        for kind in ('cls', 'reg'):
            if f'{kind}_counts/{step}' in gold.files:
                assert np.array_equal(torch.stack(aux[f'{kind}_counts']).numpy(), gold[f'{kind}_counts/{step}'])
    assert np.array_equal(torch.stack([t[4] for t in aux['targets']]).numpy().astype(np.int32), gold['gt_inds'])
    for l in range(len(oc)):
        _close(oc[l].grad.numpy(), gold[f'dmap_cls/{l}'], 1e-5, f'{name} d/dcls_out[{l}]')
        _close(opo[l].grad.numpy(), gold[f'dmap_pts/{l}'], 1e-5, f'{name} d/dpts_out[{l}]')


def test_edge_cases_are_covered(golden_dir):
    """the fixtures hold an empty bin, an image with almost every row invalid, and GHMR margins safe for the device's rounding."""
    gold = np.load(os.path.join(golden_dir, 'p2p_loss_types_edge_invalid_image.npz'))
    cls, reg = gold['cls_counts/0'], gold['reg_counts/0']
    assert (cls[:, :-1] == 0).any() and (reg[:, :-1] == 0).any()
    assert cls[1, -1] == 4 * olt.CASES['edge_invalid_image']['num_classes']          # 2 x 2 valid cells
    for name in olt.CASES:
        g = np.load(os.path.join(golden_dir, f'p2p_loss_types_{name}.npz'))
        for k in g.files:
            if k.startswith('reg_margin'):
                assert float(g[k]) >= olt.SAFE_MARGIN, (name, k)


@pytest.mark.parametrize('name', ['tinyperson_ghmc', 'defaults_ghmc_mmt', 'ghmr_mmt', 'two_level_ghm', 'l1'])
def test_state_dict_matches_reference(golden_dir, name):
    gold = np.load(os.path.join(golden_dir, f'p2p_loss_types_{name}.npz'))
    inp, cfg = olt.case_inputs(name)
    head = P2PHead(**head_kwargs(cfg))
    sd = head.state_dict()
    assert sorted(sd) == gold['state_keys'].tolist()
    for k, shp in zip(gold['state_keys'].tolist(), gold['state_shapes'].tolist()):
        assert list(sd[k].shape) == [v for v in shp if v >= 0], k
    for k in olt.make_state(cfg):
        assert torch.equal(sd[k], torch.from_numpy(gold[f'edges_init/{k}'])), k
    # a reference checkpoint (its weights and GHM buffers) loads with strict=True, and the head's own state loads back
    ref_sd = dict(inp['weights'], **{k: torch.rand_like(v) if k.endswith('acc_sum') else v for k, v in olt.make_state(cfg).items()})
    head.load_state_dict(ref_sd, strict=True)
    for k, v in ref_sd.items():
        assert torch.equal(head.state_dict()[k], v), k
    P2PHead(**head_kwargs(cfg)).load_state_dict(head.state_dict(), strict=True)


def test_ghmc_without_use_sigmoid_builds_the_reference_softmax_head():
    """p2p_head.py:63 reads use_sigmoid from the config as written: a GHMC config without it gives num_classes + 1 columns."""
    h = P2PHead(3, 256, point_anchor=[(0., 0.)], loss_cls=dict(type='GHMC'))
    assert h.num_cls_out == 4 and h.cls_out.out_channels == 4 and h.loss_cls_cfg['loss_weight'] == 1.0
    assert sorted(k for k in h.state_dict() if k.startswith('loss')) == ['loss_cls.edges']


def _head(loss_cls=None, loss_reg=None):
    return P2PHead(2, 256, point_anchor=[(0., 0.)], strides=[8], loss_cls=loss_cls, loss_reg=loss_reg,
                   train_cfg=dict(assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='FocalLossCost', weight=2.0),
                                                reg_costs=dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False), topk_k=1)))


def test_refusals():
    with pytest.raises(NotImplementedError, match='use_sigmoid=True only'):
        _head(loss_cls=dict(type='GHMC', use_sigmoid=False))
    with pytest.raises(NotImplementedError, match='1 to 256 bins'):
        _head(loss_cls=dict(type='GHMC', bins=257, use_sigmoid=True))
    with pytest.raises(NotImplementedError, match='1 to 256 bins'):
        _head(loss_reg=dict(type='GHMR', bins=300))
    with pytest.raises(NotImplementedError, match="reduction='mean'"):
        _head(loss_reg=dict(type='L1Loss', reduction='sum'))
    h = _head(loss_cls=dict(type='GHMC', bins=4, use_sigmoid=True))
    bad = dict(h.state_dict())
    bad['loss_cls.edges'] = torch.tensor([0., 0.5, 0.25, 0.75, 1.0])
    with pytest.raises(ValueError, match='nondecreasing'):
        h.load_state_dict(bad)
    x = [torch.zeros(1, 2, 4, 4)], [torch.zeros(1, 2, 4, 4)]
    metas = [dict(pad_shape=(32, 32, 3), img_shape=(32, 32, 3))]
    gt = [torch.tensor([[4., 4., 8., 8.]])], [torch.tensor([0])]
    for cls_t, reg_t, what in (('VarifocalLoss', 'SmoothL1Loss', 'soft IoU-aware'), ('QualityFocalLoss', 'SmoothL1Loss', 'quality'),
                               ('SeesawLoss', 'SmoothL1Loss', 'num_classes \\+ 2'), ('FocalLoss', 'GIoULoss', 'compares boxes'),
                               ('FocalLoss', 'IoULoss', 'compares boxes')):
        h = _head(loss_cls=dict(type=cls_t, use_sigmoid=cls_t != 'SeesawLoss'), loss_reg=dict(type=reg_t))
        with pytest.raises(NotImplementedError, match=f'cannot train with .*{what}'):
            h.loss(*x, *gt, metas)
