"""RPNHead.loss and RandomSampler on the GPU (ptb_rpn_* kernels) against the reference-pinned oracle (oracle/rpn_loss.py) on the same
seed: sampled sets, labels, label / bbox weights bit-exact, bbox targets 1e-6 scale-relative, the CPU generator state after the call equal,
per-level losses 1e-4 scale-relative, gradients of the output maps and of the three convs 2e-4; repeats and deterministic mode bit for
bit; forward_train's proposals; every fixture case and the 16 x 81 840-anchor TinyPerson tile shape."""
import os

import numpy as np
import pytest
import torch

from oracle import rpn_loss as orl

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / max(1.0, float(b.abs().max()))) if b.numel() else 0.0


def _run(name, inp, seed, train=None, head_kw=None, deterministic=False):
    from pointtinybenchmark_b200.rpn import RPNHead
    train = train or orl.CASES[name]['train']
    head = RPNHead(**(head_kw or orl.head_kwargs(name)), train_cfg=train).to(DEV)
    head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    feats = [f.to(DEV) for f in inp['feats']]
    gtb = [g.to(DEV) for g in inp['gt_bboxes']]
    ign = [g.to(DEV) for g in inp['gt_bboxes_ignore']] if inp['gt_bboxes_ignore'] is not None else None
    cls, reg = head(feats)
    for t in cls + reg:
        t.retain_grad()
    torch.manual_seed(seed)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        losses = head.loss(cls, reg, gtb, inp['img_metas'], gt_bboxes_ignore=ign)
        state = torch.get_rng_state()
        sum(sum(v) for v in losses.values()).backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    # the targets the loss used: get_targets again from the same seed makes the same draws
    torch.manual_seed(seed)
    tg = head.get_targets([tuple(c.shape[-2:]) for c in cls], gtb, inp['img_metas'], ign, device=DEV)
    torch.set_rng_state(state)
    return (head, tg), cls, reg, losses, state


def _oracle(name, inp, seed, train=None, head_kw=None):
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    cls, reg = orl.forward(inp['feats'], w)
    for t in cls + reg:
        t.retain_grad()
    torch.manual_seed(seed)
    losses, tg = orl.loss(cls, reg, inp['gt_bboxes'], inp['img_metas'], inp['gt_bboxes_ignore'], head_kw or orl.head_kwargs(name),
                          train or orl.CASES[name]['train'])
    state = torch.get_rng_state()
    sum(sum(v) for v in losses.values()).backward()
    return w, cls, reg, losses, tg, state


def _compare(head_tg, cls, reg, losses, state, ow, ocls, oreg, ol, tg, ostate, grad_tol=2e-4):
    assert torch.equal(state, ostate), 'CPU generator state after the call'
    head, t = head_tg
    assert t.num_total_samples == tg['num_total_samples']
    for b, (pos, neg) in enumerate(t.sampled_sets()):
        assert torch.equal(pos.cpu(), tg['pos_inds'][b]) and torch.equal(neg.cpu(), tg['neg_inds'][b]), f'sampled sets, image {b}'
    for l, (lab, lw, bt, bw) in enumerate(tg['levels']):
        glab, glw, gbt, gbw = (x.cpu() for x in t.level_targets(l))
        assert torch.equal(glab, lab) and torch.equal(glw, lw) and torch.equal(gbw, bw), f'labels / weights, level {l}'
        assert _rel(gbt, bt) <= 1e-6, f'bbox_targets level {l}: {_rel(gbt, bt)}'
        for k in ('loss_rpn_cls', 'loss_rpn_bbox'):
            assert _rel(losses[k][l].detach(), ol[k][l].detach()) <= 1e-4, (k, l)
        assert _rel(cls[l].grad, ocls[l].grad) <= grad_tol and _rel(reg[l].grad, oreg[l].grad) <= grad_tol, f'map gradients, level {l}'
    for k, p in head.named_parameters():
        assert _rel(p.grad, ow[k].grad) <= grad_tol, k


@pytest.mark.parametrize('name', list(orl.CASES))
def test_rpn_loss_matches_oracle_on_fixture_cases(name, golden_dir):
    c = orl.CASES[name]
    inp = orl.case_inputs(name)
    out = _run(name, inp, c['seed'])
    _compare(*out, *_oracle(name, inp, c['seed']))
    gold = np.load(os.path.join(golden_dir, f'rpn_loss_{name}.npz'))
    assert np.array_equal(out[4].numpy(), gold['rng_state'])
    for l in range(len(orl.STRIDES)):
        assert _rel(out[3]['loss_rpn_cls'][l].detach(), gold[f'loss_cls{l}']) <= 1e-4
        assert _rel(out[3]['loss_rpn_bbox'][l].detach(), gold[f'loss_bbox{l}']) <= 1e-4


def _tile_inputs(seed=3, B=16, n_gt=24):
    """configs[3]'s shape: 16 tiles of 640 x 512 (w x h), strides 4-64, 3 anchors: 81 840 anchors per tile; n_gt small boxes per tile"""
    g = torch.Generator().manual_seed(seed)
    H, W = 512, 640
    feats = [torch.randn(B, orl.C_FEAT, H // s, W // s, generator=g) for s in orl.STRIDES]
    inp = orl.case_inputs('tinyperson')
    gts = [orl._boxes(g, n_gt, H, W, 4.0, 32.0) for _ in range(B)]
    metas = [dict(img_shape=(H, W, 3), pad_shape=(H, W, 3), ori_shape=(H, W, 3), scale_factor=np.ones(4, np.float32)) for _ in range(B)]
    return dict(feats=feats, weights=inp['weights'], gt_bboxes=gts, gt_bboxes_ignore=None, img_metas=metas)


def test_rpn_loss_at_the_tile_shape_repeats_bit_for_bit():
    inp = _tile_inputs()
    assert sum(f.shape[-2] * f.shape[-1] * 3 for f in inp['feats']) == 81840
    out = _run('tinyperson', inp, 7)
    _compare(*out, *_oracle('tinyperson', inp, 7))
    # a second run and a run in deterministic mode: the losses and the output maps' gradients bit for bit (the conv weights' gradients
    # come from cuDNN, whose algorithm choice differs between the two modes)
    for det in (False, True):
        again = _run('tinyperson', inp, 7, deterministic=det)
        for k in ('loss_rpn_cls', 'loss_rpn_bbox'):
            assert all(torch.equal(a, b) for a, b in zip(out[3][k], again[3][k]))
        assert all(torch.equal(a.grad, b.grad) for a, b in zip(out[1] + out[2], again[1] + again[2]))


def test_forward_train_proposals_equal_rpn_proposals():
    from pointtinybenchmark_b200.rpn import RPNHead, RPNProposals
    name = 'tinyperson'
    inp = orl.case_inputs(name)
    head = RPNHead(**orl.head_kwargs(name), train_cfg=orl.CASES[name]['train']).to(DEV)
    head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    feats = [f.to(DEV) for f in inp['feats']]
    cfg = dict(nms_pre=300, max_per_img=100, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
    torch.manual_seed(1)
    losses, props = head.forward_train(feats, inp['img_metas'], [g.to(DEV) for g in inp['gt_bboxes']], proposal_cfg=cfg)
    assert set(losses) == {'loss_rpn_cls', 'loss_rpn_bbox'} and len(losses['loss_rpn_cls']) == 5
    cls, reg = head(feats)
    ref = RPNProposals(orl.TINYPERSON['anchor_generator'], orl.TINYPERSON['bbox_coder']).get_bboxes(cls, reg, inp['img_metas'], cfg=cfg)
    assert len(props) == len(ref) and all(torch.equal(a, b) for a, b in zip(props, ref))


def test_simple_test_rpn_equals_rpn_proposals():
    """TwoStageDetector.simple_test calls rpn_head.simple_test_rpn(x, img_metas): the proposals of get_bboxes with the head's test_cfg"""
    from pointtinybenchmark_b200.rpn import RPNHead, RPNProposals
    name = 'tinyperson'
    inp = orl.case_inputs(name)
    cfg = dict(nms_pre=1000, max_per_img=200, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
    head = RPNHead(**orl.head_kwargs(name), train_cfg=orl.CASES[name]['train'], test_cfg=cfg).to(DEV).eval()
    head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    feats = tuple(f.to(DEV) for f in inp['feats'])
    with torch.no_grad():
        props = head.simple_test_rpn(feats, inp['img_metas'])
        cls, reg = head(feats)
        ref = RPNProposals(orl.TINYPERSON['anchor_generator'], orl.TINYPERSON['bbox_coder'], test_cfg=cfg).get_bboxes(cls, reg,
                                                                                                                    inp['img_metas'])
    assert len(props) == len(ref) == 2 and all(p.shape[0] > 0 for p in props)
    assert all(torch.equal(a, b) for a, b in zip(props, ref))
    with pytest.raises(NotImplementedError, match='aug_test_rpn'):
        head.aug_test_rpn([feats], [inp['img_metas']])


def test_loss_is_none_when_an_image_has_no_inside_anchor():
    name = 'border0'
    inp = orl.case_inputs(name)
    inp['img_metas'][1] = dict(inp['img_metas'][1], img_shape=(2, 2, 3))       # allowed_border=0: no 8-px anchor fits a 2 x 2 image
    from pointtinybenchmark_b200.rpn import RPNHead
    head = RPNHead(**orl.head_kwargs(name), train_cfg=orl.CASES[name]['train']).to(DEV)
    head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    cls, reg = head([f.to(DEV) for f in inp['feats']])
    torch.manual_seed(4)
    assert head.loss(cls, reg, [g.to(DEV) for g in inp['gt_bboxes']], inp['img_metas']) is None
    mine = torch.get_rng_state()
    torch.manual_seed(4)
    ol, _ = orl.loss(*orl.forward(inp['feats'], inp['weights']), inp['gt_bboxes'], inp['img_metas'], None, orl.head_kwargs(name),
                     orl.CASES[name]['train'])
    assert ol is None and torch.equal(mine, torch.get_rng_state())


def test_random_sampler_at_roi_head_settings_equals_fixture(golden_dir):
    from pointtinybenchmark_b200.assigners import AssignResult, RandomSampler
    gold = np.load(os.path.join(golden_dir, 'rpn_loss_roi_sampler.npz'))
    anchors, gts, labels, gt_inds, max_ov, lab = orl.roi_sampler_inputs()
    s = RandomSampler(**orl.ROI_SAMPLER)
    torch.manual_seed(21)
    r = s.sample(AssignResult(gts.shape[0], gt_inds.to(DEV), max_ov.to(DEV), lab.to(DEV)), anchors.to(DEV), gts.to(DEV), labels.to(DEV))
    assert np.array_equal(torch.get_rng_state().numpy(), gold['rng_state'])
    for k in ('pos_inds', 'neg_inds', 'pos_is_gt', 'pos_assigned_gt_inds', 'pos_gt_labels'):
        assert np.array_equal(getattr(r, k).cpu().numpy(), gold[k]), k
