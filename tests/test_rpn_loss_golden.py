"""RPNHead.loss (rpn_head.py:44-75 over anchor_head.py:171-489) and RandomSampler, CPU side:
- the oracle (oracle/rpn_loss.py) reproduces every tests/golden/rpn_loss_*.npz fixture recorded from the REAL reference
  (oracle/make_golden_rpn_loss.py): sampled sets, labels and weights exact, floats within 1e-6, the generator state after the call;
- the host draw plan (assigners.random_sample_plan) makes the reference sampler's randperm calls for hand-made counts;
- the inside-box plan (rpn.inside_boxes) equals the reference's valid / inside flags;
- the mirror's constructor keywords and state_dict, the refusals, and that RPNHead / RandomSampler register only through register_rpn()."""
import os

import numpy as np
import pytest
import torch

from oracle import rpn_loss as orl

CASES = list(orl.CASES)


def _gold(golden_dir, name):
    return np.load(os.path.join(golden_dir, f'rpn_loss_{name}.npz'))


def _close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.all(np.abs(a - b) <= tol * max(1.0, float(np.abs(b).max()) if b.size else 1.0))


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_golden(golden_dir, name):
    gold = _gold(golden_dir, name)
    c = orl.CASES[name]
    inp = orl.case_inputs(name)
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    cls, reg = orl.forward(inp['feats'], w)
    for t in cls + reg:
        t.retain_grad()
    torch.manual_seed(c['seed'])
    losses, tg = orl.loss(cls, reg, inp['gt_bboxes'], inp['img_metas'], inp['gt_bboxes_ignore'], orl.head_kwargs(name), c['train'])
    assert np.array_equal(torch.get_rng_state().numpy(), gold['rng_state'])
    assert tg['num_total_samples'] == int(gold['num_total_samples'])
    sum(sum(v) for v in losses.values()).backward()
    for b in range(len(c['imgs'])):
        assert np.array_equal(tg['pos_inds'][b].numpy(), gold[f'pos_inds{b}'])
        assert np.array_equal(tg['neg_inds'][b].numpy(), gold[f'neg_inds{b}'])
    for l, (lab, lw, bt, bw) in enumerate(tg['levels']):
        assert np.array_equal(lab.numpy(), gold[f'labels{l}']) and np.array_equal(lw.numpy(), gold[f'label_weights{l}'])
        assert np.array_equal(bw.numpy(), gold[f'bbox_weights{l}'])
        assert _close(bt.numpy(), gold[f'bbox_targets{l}'], 1e-6)
        assert _close(losses['loss_rpn_cls'][l].detach(), gold[f'loss_cls{l}'], 1e-6)
        assert _close(losses['loss_rpn_bbox'][l].detach(), gold[f'loss_bbox{l}'], 1e-6)
        assert _close(cls[l].grad.flatten()[::7], gold[f'grad_cls{l}_sub'], 1e-6)
        assert _close(reg[l].grad.flatten()[::7], gold[f'grad_reg{l}_sub'], 1e-6)
    for k, v in w.items():
        assert _close(v.grad, gold[f'grad/{k}'], 1e-6), k


def _reference_sampler_draws(counts, num, pos_fraction, neg_pos_ub):
    """the reference sampler on synthetic assignments with these counts (oracle.rpn_loss.random_sample, pinned by the fixtures)"""
    out = []
    for n_pos, n_neg in counts:
        gt_inds = torch.cat([torch.ones(n_pos, dtype=torch.long), torch.zeros(n_neg, dtype=torch.long),
                             torch.full((3,), -1, dtype=torch.long)])
        gt_inds = gt_inds[torch.from_numpy(np.random.default_rng(n_pos * 7 + n_neg).permutation(gt_inds.numel()))]
        out.append((gt_inds, orl.random_sample(gt_inds, num, pos_fraction, neg_pos_ub)))
    return out


@pytest.mark.parametrize('counts,num,pos_fraction,neg_pos_ub', [
    ([(300, 5000), (10, 9000), (0, 40), (128, 128)], 256, 0.5, -1),
    ([(3, 900), (0, 900), (50, 10)], 256, 0.5, 1),
    ([(7, 300), (200, 0)], 512, 0.25, 0),
    ([(0, 0), (129, 127)], 256, 0.5, 3),
])
def test_draw_plan_makes_the_reference_draws(counts, num, pos_fraction, neg_pos_ub):
    from pointtinybenchmark_b200.assigners import random_sample_plan, sampled_counts
    torch.manual_seed(5)
    ref = _reference_sampler_draws(counts, num, pos_fraction, neg_pos_ub)
    ref_state = torch.get_rng_state()
    torch.manual_seed(5)
    plan = random_sample_plan(counts, num, pos_fraction, neg_pos_ub)
    assert torch.equal(torch.get_rng_state(), ref_state)
    for (gt_inds, (rpos, rneg)), (pos, neg), (np_, nn_) in zip(ref, plan, sampled_counts(plan, counts)):
        for kind, r, sel, n in ((gt_inds > 0, rpos, pos, np_), (gt_inds == 0, rneg, neg, nn_)):
            gallery = torch.nonzero(kind).squeeze(1)
            mine = gallery if sel is None else gallery[sel]
            assert torch.equal(mine, r) and n == r.numel()


@pytest.mark.parametrize('name', ['tinyperson', 'border0', 'pad_shapes', 'few_neg'])
def test_inside_boxes_equal_the_reference_flags(name):
    from pointtinybenchmark_b200.rpn import AnchorGenerator, inside_boxes
    from oracle import anchors as oa
    c = orl.CASES[name]
    inp = orl.case_inputs(name)
    sizes = [tuple(f.shape[-2:]) for f in inp['feats']]
    ag_cfg = orl.TINYPERSON['anchor_generator']
    ag = AnchorGenerator(strides=ag_cfg['strides'], ratios=ag_cfg['ratios'], scales=ag_cfg['scales'])
    boxes = inside_boxes(ag, sizes, inp['img_metas'], c['train']['allowed_border'])
    flat = torch.cat([oa.grid_anchors(oa.base_anchors(s, ag_cfg['scales'], ag_cfg['ratios']), fs, (s, s))
                      for s, fs in zip(ag_cfg['strides'], sizes)])
    for b, meta in enumerate(inp['img_metas']):
        want = orl.inside_flags(flat, torch.cat(orl.valid_flags(sizes, meta['pad_shape'], 3)), meta['img_shape'],
                                c['train']['allowed_border'])
        got = []
        for l, (h, w) in enumerate(sizes):
            y, x, a = np.meshgrid(np.arange(h), np.arange(w), np.arange(3), indexing='ij')
            r = boxes[b, l][a]
            got.append(((x >= r[..., 0]) & (x < r[..., 1]) & (y >= r[..., 2]) & (y < r[..., 3])).reshape(-1))
        assert np.array_equal(np.concatenate(got), want.numpy()), (name, b)


def _head(name='tinyperson', **over):
    from pointtinybenchmark_b200.rpn import RPNHead
    kw = orl.head_kwargs(name)
    kw.update(over)
    return RPNHead(**kw, train_cfg=orl.CASES[name]['train'])


def test_signature_and_state_dict_match_reference(golden_dir):
    import inspect
    from pointtinybenchmark_b200.rpn import RPNHead
    gold = _gold(golden_dir, 'tinyperson')
    mine = list(inspect.signature(RPNHead.__init__).parameters)
    for p in gold['ctor_params']:
        assert str(p) in mine, p
    sd = _head().state_dict()
    assert sorted(sd) == [str(k) for k in gold['state_keys']]
    for k, shp in zip(gold['state_keys'], gold['state_shapes']):
        assert list(sd[str(k)].shape) == [int(v) for v in shp if v >= 0]
    h = _head()
    assert abs(float(h.rpn_conv.weight.detach().std()) - 0.01) < 0.002 and float(h.rpn_cls.bias.abs().max()) == 0.0


@pytest.mark.parametrize('over,match', [
    (dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False)), 'softmax'),
    (dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True)), 'FocalLoss.*sampling'),
    (dict(loss_cls=dict(type='GHMC', use_sigmoid=True)), 'GHMC.*sampling'),
    (dict(loss_cls=dict(type='QualityFocalLoss', use_sigmoid=True)), 'QualityFocalLoss.*sampling'),
    (dict(loss_cls=dict(type='VarifocalLoss', use_sigmoid=True)), 'VarifocalLoss'),
    (dict(reg_decoded_bbox=True), 'reg_decoded_bbox'),
    (dict(loss_bbox=dict(type='GIoULoss')), 'GIoULoss'),
    (dict(loss_bbox=dict(type='L1Loss', reduction='sum')), 'reduction'),
])
def test_refusals(over, match):
    with pytest.raises(NotImplementedError, match=match):
        _head(**over)


@pytest.mark.parametrize('sampler', ['OHEMSampler', 'InstanceBalancedPosSampler', 'IoUBalancedNegSampler', 'ScoreHLRSampler',
                                     'PseudoSampler'])
def test_other_samplers_are_refused(sampler):
    from pointtinybenchmark_b200.rpn import RPNHead
    train = dict(orl.TRAIN, sampler=dict(type=sampler, num=256, pos_fraction=0.5))
    with pytest.raises(NotImplementedError, match=sampler):
        RPNHead(**orl.head_kwargs('tinyperson'), train_cfg=train)


def test_rpn_head_registers_only_through_register_rpn():
    import pointtinybenchmark_b200  # noqa: F401
    from pointtinybenchmark_b200 import registry
    from pointtinybenchmark_b200.assigners import RandomSampler
    from pointtinybenchmark_b200.rpn import RPNHead
    registry.register_core()
    if not registry.USING_MMDET:
        assert registry.HEADS.get('RPNHead') is not RPNHead
        assert registry.BBOX_SAMPLERS.get('RandomSampler') is not RandomSampler
    else:
        assert registry.HEADS.get('RPNHead') is not RPNHead
    registry.register_rpn()
    assert registry.HEADS.get('RPNHead') is RPNHead and registry.BBOX_SAMPLERS.get('RandomSampler') is RandomSampler


def test_add_gt_as_proposals_raises_as_the_reference():
    """AnchorHead samples without gt_labels, so the reference's sampler raises for an image with GTs when add_gt_as_proposals is set"""
    from pointtinybenchmark_b200.rpn import RPNHead
    train = dict(orl.TRAIN, sampler=dict(orl.TRAIN['sampler'], add_gt_as_proposals=True))
    head = RPNHead(**orl.head_kwargs('tinyperson'), train_cfg=train)
    inp = orl.case_inputs('tinyperson')
    with pytest.raises(ValueError, match='add_gt_as_proposals'):
        head.get_targets([tuple(f.shape[-2:]) for f in inp['feats']], inp['gt_bboxes'], inp['img_metas'], device='cpu')


def test_aug_test_rpn_is_refused():
    with pytest.raises(NotImplementedError, match='aug_test_rpn'):
        _head().aug_test_rpn([], [])
