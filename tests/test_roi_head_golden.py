"""CPU checks of the RoI head's oracle and host side (no GPU): oracle/roi_head.py against the fixtures the real reference wrote
(tests/golden/roi_head_*.npz: sampled sets, rois, targets, losses, acc, generator state, gradients, detections), the RoIAlign restatement
against torchvision.ops.roi_align(aligned=True), the FPN level rule at the level boundaries, the constructor keywords and state_dict
against the reference classes, the refusals and the registration."""
import inspect
import os

import numpy as np
import pytest
import torch
import torchvision

from oracle import roi_head as orh

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _gold(name):
    return np.load(os.path.join(GOLD, f'roi_head_{name}.npz'))


def _close(a, b, tol, what):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    assert a.shape == b.shape, f'{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}'
    if a.numel():
        d = float((a - b).abs().max())
        assert d <= tol * max(1.0, float(b.abs().max())), f'{what}: {d}'


@pytest.mark.parametrize('name', list(orh.CASES))
def test_oracle_matches_reference_fixture(name):
    g = _gold(name)
    inp = orh.case_inputs(name)
    feats = [f.clone().requires_grad_(True) for f in inp['feats']]
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    torch.manual_seed(orh.CASES[name]['seed'])
    losses, tg = orh.forward_train(inp, name, feats=feats, w=w)
    assert np.array_equal(torch.get_rng_state().numpy(), g['rng_state'])
    for b, (_, _, pos, neg) in enumerate(tg['samples']):
        assert np.array_equal(pos.numpy(), g[f'pos_inds{b}']) and np.array_equal(neg.numpy(), g[f'neg_inds{b}'])
    assert np.array_equal(tg['rois'].numpy(), g['rois'])
    for k in ('labels', 'label_weights', 'bbox_weights'):
        assert np.array_equal(tg[k].numpy(), g[k]), k
    _close(tg['bbox_targets'], g['bbox_targets'], 1e-6, 'bbox_targets')
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        _close(losses[k].detach().reshape(-1), g[k].reshape(-1), 1e-6, k)
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    for l in range(len(orh.STRIDES)):
        _close(feats[l].grad.flatten()[::97], g[f'grad_feat{l}_sub'], 1e-5, f'grad feat{l}')
    for k, v in w.items():
        _close(v.grad.flatten()[::41], g[f'grad/{k}_sub'], 1e-5, f'grad {k}')
    dets, labs = orh.simple_test(inp, name)
    for b in range(len(dets)):
        _close(dets[b], g[f'dets{b}'], 1e-6, f'dets {b}')
        assert np.array_equal(labs[b].numpy(), g[f'det_labels{b}'])


def test_padding_rows_become_detections():
    """test_mixins.py:79-119: the shorter list is padded at the front; the padded rows score 1 / (C + 1) = 0.5 at one class and
    survive the NMS as (0, 0, 0, 0) boxes — the reference's own output, pinned by the `uneven` fixture"""
    g = _gold('uneven')
    d0 = g['dets0']                                        # image 0 has 40 proposals, padded to 130
    zero = (np.abs(d0[:, :4]).sum(1) == 0)
    assert zero.sum() == 130 - 40 and np.allclose(d0[zero, 4], 0.5)


def _random_rois(seed, n, B, H, W, stride):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 2, generator=g) * torch.tensor([W * stride * 1.2, H * stride * 1.2]) - 0.1 * stride * torch.tensor([W, H])
    wh = torch.rand(n, 2, generator=g) * 40 * stride / 4
    rois = torch.cat([torch.randint(0, B, (n, 1), generator=g).float(), c, c + wh], 1)
    rois[:6, 3:] = rois[:6, 1:3]                           # zero size
    rois[6:12, 1:] -= 1000.0                               # beyond the map, negative coordinates
    rois[12:18, 1:3] = -3.0                                # negative corner inside the reach of the first row / column
    return rois


@pytest.mark.parametrize('sampling_ratio', [0, 2])
@pytest.mark.parametrize('stride', [4, 16])
def test_roi_align_restatement_matches_torchvision(sampling_ratio, stride):
    g = torch.Generator().manual_seed(5)
    feat = torch.randn(3, 8, 24, 30, generator=g)
    rois = _random_rois(stride, 400, 3, 24, 30, stride)
    a = orh.roi_align(feat, rois, 7, 1.0 / stride, sampling_ratio)
    b = torchvision.ops.roi_align(feat, rois, 7, 1.0 / stride, sampling_ratio, aligned=True)
    assert torch.equal(a, b)


def test_level_boundaries_follow_the_correctly_rounded_log2():
    """the kernel takes floor(fp32(log2(double(v)))): equal to torch's CPU levels at +-1 ulp of every boundary"""
    rois = orh.level_boundary_rois()
    want = orh.map_roi_levels(rois, 4)
    scale = torch.sqrt((rois[:, 3] - rois[:, 1]) * (rois[:, 4] - rois[:, 2]))
    v = (scale / 56 + 1e-6).numpy()
    rule = np.clip(np.floor(np.log2(v.astype(np.float64)).astype(np.float32)), 0, 3).astype(np.int64)
    assert np.array_equal(want.numpy(), rule)
    assert len(set(want.tolist())) == 4                    # every level is hit


def test_constructor_keywords_and_state_dict_match_reference():
    from pointtinybenchmark_b200.roi_head import Shared2FCBBoxHead, SingleRoIExtractor, StandardRoIHead
    g = np.load(os.path.join(GOLD, 'roi_head_ctor.npz'))
    mine = lambda cls: [p for p in inspect.signature(cls.__init__).parameters if p != 'self']
    assert mine(StandardRoIHead) == list(g['roi_head'])
    assert mine(SingleRoIExtractor) == list(g['extractor'])
    assert set(mine(Shared2FCBBoxHead)) == set(g['bbox_head'])
    for name in orh.CASES:
        kw = orh.head_kwargs(name)
        bh = dict(kw['bbox_head'])
        bh.pop('type')
        sd = Shared2FCBBoxHead(**bh).state_dict()
        gold = _gold(name)
        keys = [k[len('bbox_head.'):] for k in gold['state_keys']]
        assert list(sd) == keys                             # the reference's registration order
        for k, shp in zip(keys, gold['state_shapes']):
            assert list(sd[k].shape) == [s for s in shp if s >= 0], k


def test_reference_init():
    from pointtinybenchmark_b200.roi_head import Shared2FCBBoxHead
    torch.manual_seed(0)
    h = Shared2FCBBoxHead(in_channels=16, fc_out_channels=256, num_classes=3)
    bound = float(np.sqrt(6.0 / (16 * 49 + 256)))
    assert float(h.shared_fcs[0].weight.abs().max()) <= bound and float(h.shared_fcs[0].bias.abs().max()) == 0
    assert abs(float(h.fc_cls.weight.std()) - 0.01) < 0.002 and abs(float(h.fc_reg.weight.std()) - 0.001) < 0.0002


@pytest.mark.parametrize('change, word', [
    (dict(mask_head=dict(type='FCNMaskHead')), 'mask'),
    (dict(shared_head=dict(type='ResLayer')), 'shared_head'),
    (dict(ex=dict(type='GenericRoIExtractor')), 'GenericRoIExtractor'),
    (dict(bh=dict(type='Shared4Conv1FCBBoxHead')), 'Shared4Conv1FCBBoxHead'),
    (dict(layer=dict(pool_mode='max')), 'max'),
    (dict(layer=dict(aligned=False)), 'aligned=False'),
    (dict(bhkw=dict(reg_decoded_bbox=True)), 'reg_decoded_bbox'),
    (dict(bhkw=dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True))), 'sigmoid'),
    (dict(train=dict(sampler=dict(type='OHEMSampler', num=512, pos_fraction=0.25))), 'OHEMSampler'),
])
def test_refusals(change, word):
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    kw = orh.head_kwargs('tinyperson')
    ex, bh = dict(kw['bbox_roi_extractor']), dict(kw['bbox_head'])
    ex['roi_layer'] = dict(ex['roi_layer'], **change.get('layer', {}))
    ex.update(change.get('ex', {}))
    bh.update(change.get('bh', {}))
    bh.update(change.get('bhkw', {}))
    train = dict(orh.TRAIN, **change.get('train', {}))
    test = dict(orh.TEST, **change.get('test', {}))
    extra = {k: v for k, v in change.items() if k in ('mask_head', 'shared_head')}
    with pytest.raises(NotImplementedError, match=word):
        StandardRoIHead(bbox_roi_extractor=ex, bbox_head=bh, train_cfg=train, test_cfg=test, **extra)


def test_roi_scale_factor_and_aug_test_refused():
    """a test_cfg with do_tile_as_aug builds (training is unaffected); the detector's tile paths end in aug_test, which raises"""
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    h = StandardRoIHead(**orh.head_kwargs('tinyperson'), train_cfg=orh.TRAIN, test_cfg=dict(orh.TEST, do_tile_as_aug=True))
    with pytest.raises(NotImplementedError, match='roi_scale_factor'):
        h.bbox_roi_extractor([torch.zeros(1, 8, 4, 4)] * 4, torch.zeros(1, 5), roi_scale_factor=1.5)
    with pytest.raises(NotImplementedError, match='tile_aug_test'):
        h.aug_test(None, None, None)
    with pytest.raises(NotImplementedError, match='aug_test'):
        h.aug_test_bboxes(None, None, None, None)


def test_register_roi():
    from pointtinybenchmark_b200 import registry, roi_head
    registry.register_roi()
    assert registry.HEADS.get('StandardRoIHead') is roi_head.StandardRoIHead
    assert registry.HEADS.get('Shared2FCBBoxHead') is roi_head.Shared2FCBBoxHead
    assert registry.ROI_EXTRACTORS.get('SingleRoIExtractor') is roi_head.SingleRoIExtractor
