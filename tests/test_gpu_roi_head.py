"""StandardRoIHead's bbox branch on the GPU (ptb_roi_* kernels) against the reference-pinned oracle (oracle/roi_head.py) and the fixtures
the real reference wrote: levels, sampled sets, rois, labels and the CPU generator state bit-exact; targets 1e-6; RoI features,
cls_score, bbox_pred, losses and acc 1e-4 scale-relative; gradients of the FPN maps and of every FC parameter 2e-4; detections (counts,
labels, boxes 1e-4).  Every fixture case, the 16-tile TinyPerson training shape, the 8-image 80-class test shape, the two heads driven
as TwoStageDetector drives them, and repeated calls."""
import os
import warnings

import numpy as np
import pytest
import torch
import torchvision

from oracle import roi_head as orh

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    assert a.shape == b.shape, (tuple(a.shape), tuple(b.shape))
    return float((a - b).abs().max() / max(1.0, float(b.abs().max()))) if b.numel() else 0.0


def _head(name=None, head_kw=None, train=None, test=None):
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    c = orh.CASES[name] if name else {}
    return StandardRoIHead(**(head_kw or orh.head_kwargs(name)), train_cfg=train or c['train'], test_cfg=test or c['test']).to(DEV)


def _dev(inp):
    return ([f.to(DEV) for f in inp['feats']], [g.to(DEV) for g in inp['gt_bboxes']], [l.to(DEV) for l in inp['gt_labels']],
            [p.to(DEV) for p in inp['proposals']])


def _train(head, inp, seed):
    feats, gtb, gtl, props = _dev(inp)
    feats = [f.requires_grad_(True) for f in feats]
    torch.manual_seed(seed)
    targets = head.get_targets(props, gtb, gtl)
    state = torch.get_rng_state()
    res = head._bbox_forward(feats, targets[0])
    for k in ('cls_score', 'bbox_pred', 'bbox_feats'):
        res[k].retain_grad()
    rois, labels, lw, bt, bw, _ = targets
    losses = head.bbox_head.loss(res['cls_score'], res['bbox_pred'], rois, labels, lw, bt, bw, avg_factor=rois.shape[0])
    (losses['loss_cls'] + losses['loss_bbox']).backward()
    torch.cuda.synchronize()
    return dict(feats=feats, targets=targets, state=state, res=res, losses=losses)


@pytest.mark.parametrize('name', list(orh.CASES))
def test_forward_train_matches_reference(name):
    g = np.load(os.path.join(GOLD, f'roi_head_{name}.npz'))
    inp = orh.case_inputs(name)
    head = _head(name)
    head.bbox_head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    out = _train(head, inp, orh.CASES[name]['seed'])
    rois, labels, lw, bt, bw, _ = out['targets']
    assert np.array_equal(out['state'].numpy(), g['rng_state'])
    assert np.array_equal(rois.cpu().numpy(), g['rois'])
    assert np.array_equal(labels.cpu().numpy(), g['labels']) and np.array_equal(lw.cpu().numpy(), g['label_weights'])
    assert np.array_equal(bw.cpu().numpy(), g['bbox_weights'])
    assert _rel(bt, g['bbox_targets']) <= 1e-6
    lv = head.bbox_roi_extractor.last_levels.cpu()
    assert _same_levels(lv, torch.from_numpy(g['rois']))
    # the oracle on the same rois with autograd
    of = [f.clone().requires_grad_(True) for f in inp['feats']]
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    r = torch.from_numpy(g['rois'])
    feat = orh.extract(of[:4], r)
    cls, reg = orh.bbox_forward(of, r, w)
    h = orh.CASES[name]['head']
    ol = orh.loss(cls, reg, torch.from_numpy(g['labels']), torch.from_numpy(g['label_weights']), torch.from_numpy(g['bbox_targets']),
                  torch.from_numpy(g['bbox_weights']), h['num_classes'], h.get('reg_class_agnostic', False), h['loss_cls'], h['loss_bbox'])
    (ol['loss_cls'] + ol['loss_bbox']).backward()
    assert _rel(out['res']['bbox_feats'].detach(), feat.detach()) <= 1e-4
    assert _rel(out['res']['cls_score'].detach(), cls.detach()) <= 1e-4
    assert _rel(out['res']['bbox_pred'].detach(), reg.detach()) <= 1e-4
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        assert _rel(out['losses'][k].detach().reshape(-1), g[k].reshape(-1)) <= 1e-4, k
    for l in range(4):
        assert _rel(out['feats'][l].grad, of[l].grad) <= 2e-4, f'grad feat{l}'
    assert out['feats'][4].grad is None
    for k, p in head.bbox_head.named_parameters():
        assert _rel(p.grad, w[k].grad) <= 2e-4, f'grad {k}'


def _same_levels(got, rois):
    """the kernel's levels against map_roi_levels; a NaN scale (a RoI with one negative side) has no level in the reference (its
    .long() matches no mask) and -1 here: both leave the RoI's features at zero"""
    want = orh.map_roi_levels(rois.cpu(), 4)
    want = torch.where((want >= 0) & (want <= 3), want, torch.full_like(want, -1))
    return torch.equal(got.cpu().long(), want)


def _same_dets(got, want, what):
    assert got.shape == want.shape, f'{what}: {tuple(got.shape)} vs {tuple(want.shape)}'
    if len(want):
        k = lambda d: np.lexsort(np.round(np.asarray(d, np.float64)[:, ::-1], 3).T)
        assert _rel(np.asarray(got)[k(got)], np.asarray(want)[k(want)]) <= 1e-4, what


@pytest.mark.parametrize('name', list(orh.CASES))
def test_simple_test_matches_reference(name):
    g = np.load(os.path.join(GOLD, f'roi_head_{name}.npz'))
    inp = orh.case_inputs(name)
    head = _head(name)
    head.bbox_head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    feats, _, _, props = _dev(inp)
    with torch.no_grad():
        res = head.simple_test(tuple(feats), props, inp['img_metas'])
    C = orh.CASES[name]['head']['num_classes']
    for b in range(len(res)):
        d, lab = g[f'dets{b}'], g[f'det_labels{b}']
        for k in range(C):
            _same_dets(res[b][k], d[lab == k], f'{name} image {b} class {k}')


def test_rescale_matches_oracle():
    inp = orh.case_inputs('tinyperson')
    head = _head('tinyperson')
    head.bbox_head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    feats, _, _, props = _dev(inp)
    with torch.no_grad():
        res = head.simple_test(tuple(feats), props, inp['img_metas'], rescale=True)
    dets, labs = orh.simple_test(inp, 'tinyperson', rescale=True)
    for b in range(len(res)):
        _same_dets(res[b][0], dets[b].numpy(), f'rescaled image {b}')


def test_repeat_calls_are_identical():
    inp = orh.case_inputs('cw_posweight')
    head = _head('cw_posweight')
    head.bbox_head.load_state_dict({k: v.to(DEV) for k, v in inp['weights'].items()})
    a, b = _train(head, inp, 7), _train(head, inp, 7)
    for x, y in zip(a['targets'][:5], b['targets'][:5]):
        assert torch.equal(x, y)
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        assert torch.equal(a['losses'][k], b['losses'][k])


def _tiles(seed, B, H, W, n_gt, n_prop, C_feat=256):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(B, C_feat, H // s, W // s, generator=g).to(DEV) for s in (4, 8, 16, 32, 64)]
    gts, labels, props = [], [], []
    from oracle import rpn_loss as orl
    for b in range(B):
        gt = orl._boxes(g, n_gt, H, W, 6.0, 60.0)
        p = orl._boxes(g, n_prop, H, W, 4.0, 200.0)
        m = n_prop // 3
        p[:m] = gt[torch.randint(0, n_gt, (m,), generator=g)] + torch.randn(m, 4, generator=g) * 2.0
        gts.append(gt); labels.append(torch.zeros(n_gt, dtype=torch.long)); props.append(torch.cat([p, torch.rand(n_prop, 1, generator=g)], 1))
    return feats, gts, labels, props


def _config_head(num_classes=1, num=512):
    kw = dict(bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0),
                                      out_channels=256, featmap_strides=[4, 8, 16, 32]),
              bbox_head=dict(type='Shared2FCBBoxHead', in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=num_classes,
                             **{k: v for k, v in orh.TINYPERSON.items() if k != 'num_classes'}))
    train = dict(orh.TRAIN, sampler=dict(orh.TRAIN['sampler'], num=num))
    return _head(head_kw=kw, train=train, test=dict(orh.TEST))


def test_tinyperson_tiles_at_full_size():
    """16 tiles of 640 x 512, 1 000 proposals and 24 GTs each, 512 sampled RoIs per tile"""
    feats, gts, labels, props = _tiles(3, 16, 512, 640, 24, 1000)
    head = _config_head()
    torch.manual_seed(5)
    rois, lab, lw, bt, bw, ns = head.get_targets([p.to(DEV) for p in props], [g.to(DEV) for g in gts], [l.to(DEV) for l in labels])
    state = torch.get_rng_state()
    torch.manual_seed(5)
    smp = orh.sample(props, gts, labels, None, orh.TRAIN | dict(sampler=dict(orh.TRAIN['sampler'], num=512)))
    assert torch.equal(torch.get_rng_state(), state)
    o = orh.targets(smp, gts, labels, 1, [0.] * 4, [0.1, 0.1, 0.2, 0.2], -1)
    assert rois.shape[0] == 16 * 512
    assert torch.equal(rois.cpu(), o[0]) and torch.equal(lab.cpu(), o[1]) and torch.equal(lw.cpu(), o[2]) and torch.equal(bw.cpu(), o[4])
    assert _rel(bt, o[3]) <= 1e-6
    # RoI features and their map gradients against torchvision's CUDA RoIAlign on each level
    x = [f.clone().requires_grad_(True) for f in feats]
    y = head.bbox_roi_extractor(x[:4], rois)
    lv = head.bbox_roi_extractor.last_levels.long()
    assert _same_levels(lv, rois)
    xr = [f.clone().requires_grad_(True) for f in feats]
    yr = torch.zeros_like(y)
    for l, s in enumerate((4, 8, 16, 32)):
        m = (lv == l).nonzero().squeeze(1)
        yr = yr.index_put((m,), torchvision.ops.roi_align(xr[l], rois[m], 7, 1.0 / s, 0, aligned=True))
    assert _rel(y.detach(), yr.detach()) <= 1e-4
    gy = torch.randn_like(y)
    (y * gy).sum().backward()
    (yr * gy).sum().backward()
    for l in range(4):
        assert _rel(x[l].grad, xr[l].grad if xr[l].grad is not None else torch.zeros_like(x[l])) <= 2e-4
    # losses on the head's outputs against the oracle's loss on the same outputs
    cls, reg = head.bbox_head(y.detach())
    losses = head.bbox_head.loss(cls, reg, rois, lab, lw, bt, bw, avg_factor=rois.shape[0])
    ol = orh.loss(cls.detach().cpu(), reg.detach().cpu(), o[1], o[2], o[3], o[4], 1, False, orh.TINYPERSON['loss_cls'],
                  orh.TINYPERSON['loss_bbox'])
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        assert _rel(losses[k].detach().reshape(-1), ol[k].reshape(-1)) <= 1e-4, k


def _realistic_scores(head, seed):
    """seeded weights with fc_cls / fc_reg at the spread of a trained head: the reference init (fc_cls Normal(0.01)) puts every one of 81
    softmax scores near 1 / 81, below score_thr 0.05, and would leave the NMS without a candidate"""
    torch.manual_seed(seed)
    head.bbox_head.init_weights()
    with torch.no_grad():
        head.bbox_head.fc_cls.weight.normal_(0.0, 0.1)
        head.bbox_head.fc_reg.weight.normal_(0.0, 0.05)


def test_simple_test_80_classes_1333x800():
    """8 images of 1333 x 800, 1 000 proposals each, 80 classes, max_per_img 100: decode + one batched NMS call against the oracle's
    decode and per-image multiclass_nms on the same head outputs; thousands of candidates per image pass score_thr"""
    feats, _, _, props = _tiles(9, 8, 800, 1344, 10, 1000)
    props = [p.to(DEV) for p in props]
    head = _config_head(num_classes=80)
    _realistic_scores(head, 17)
    test_cfg = dict(orh.TEST, max_per_img=100)
    head.test_cfg = type(head.test_cfg)(test_cfg)
    metas = [dict(img_shape=(800, 1333, 3), scale_factor=np.ones(4, np.float32)) for _ in range(8)]
    with torch.no_grad():
        res = head.simple_test(tuple(feats), props, metas)
        rois, N = orh.pad_rois([p.cpu() for p in props])
        out = head._bbox_forward(feats, rois.to(DEV))
    boxes, scores = orh.decode(rois, out['cls_score'].cpu(), out['bbox_pred'].cpu(), 8, [m['img_shape'] for m in metas], [0.] * 320,
                               [0.1, 0.1, 0.2, 0.2] * 80)
    n_cand = (scores[..., :-1] > 0.05).sum(dim=(1, 2))
    assert int(n_cand.min()) >= 500, n_cand.tolist()
    dets, labs = orh.multiclass_nms_per_image(boxes, scores, 80, test_cfg)
    for b in range(8):
        assert len(dets[b]) >= 50 and sum(len(r) for r in res[b]) == len(dets[b])
        for c in range(80):
            _same_dets(res[b][c], dets[b][labs[b] == c].numpy(), f'image {b} class {c}')


def test_levels_at_the_boundaries():
    """the kernel's level of RoIs within 6 ulps of every level boundary equals torch's CPU map_roi_levels"""
    from pointtinybenchmark_b200.roi_head import SingleRoIExtractor
    ex = SingleRoIExtractor(dict(type='RoIAlign', output_size=7, sampling_ratio=0), 8, [4, 8, 16, 32])
    rois = orh.level_boundary_rois()
    feats = [torch.randn(1, 8, 128 // s, 128 // s, device=DEV) for s in (4, 8, 16, 32)]
    ex(feats, rois.to(DEV))
    want = orh.map_roi_levels(rois, 4)
    assert len(set(want.tolist())) == 4
    assert torch.equal(ex.last_levels.cpu().long(), want)


def test_two_stage_detector_flow(monkeypatch):
    """TwoStageDetector.forward_train / simple_test (two_stage.py) with the TinyPerson head settings: RPNHead.forward_train(proposal_cfg)
    then StandardRoIHead.forward_train; simple_test_rpn then StandardRoIHead.simple_test.  The RoI stage's sampled rows and targets
    against the oracle on the same proposals, one synchronising copy (the sampled counts, device to host) in its training step and one NMS call for the test batch"""
    from oracle import rpn_loss as orl
    from pointtinybenchmark_b200 import ops
    from pointtinybenchmark_b200.rpn import RPNHead
    B, H, W = 2, 256, 320
    feats, gts, labels, _ = _tiles(11, B, H, W, 12, 10)
    feats = [f[:, :64].contiguous() for f in feats]
    torch.manual_seed(12)                                  # the heads' init: the same proposals whatever ran before
    rpn = RPNHead(in_channels=64, feat_channels=64, **{k: v for k, v in orl.TINYPERSON.items()}, train_cfg=orl.TRAIN,
                  test_cfg=dict(nms_pre=1000, max_per_img=1000, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)).to(DEV)
    kw = dict(bbox_roi_extractor=dict(type='SingleRoIExtractor', roi_layer=dict(type='RoIAlign', output_size=7, sampling_ratio=0),
                                      out_channels=64, featmap_strides=[4, 8, 16, 32]),
              bbox_head=dict(type='Shared2FCBBoxHead', in_channels=64, fc_out_channels=128, roi_feat_size=7, **orh.TINYPERSON))
    train = dict(orh.TRAIN, sampler=dict(orh.TRAIN['sampler'], num=512))
    roi = _head(head_kw=kw, train=train, test=orh.TEST)
    metas = [dict(img_shape=(H, W, 3), pad_shape=(H, W, 3), scale_factor=np.ones(4, np.float32)) for _ in range(B)]
    gtb, gtl = [g.to(DEV) for g in gts], [l.to(DEV) for l in labels]
    x = [f.requires_grad_(True) for f in feats]
    proposal_cfg = dict(nms_pre=2000, max_per_img=1000, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
    rpn_losses, proposals = rpn.forward_train(x, metas, gtb, None, proposal_cfg=proposal_cfg)
    seen = {}
    real_targets = ops.roi_targets
    monkeypatch.setattr(ops, 'roi_targets', lambda *a, **k: seen.setdefault('targets', real_targets(*a, **k)))
    torch.cuda.synchronize()
    torch.manual_seed(13)
    # every synchronising CUDA operation torch issues (device-to-host copies, blocking host-to-device copies) warns in this mode
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            roi_losses = roi.forward_train(x, metas, proposals, gtb, gtl)
        finally:
            torch.cuda.set_sync_debug_mode('default')
    syncs = [str(w.message) for w in caught if 'called a synchronizing CUDA operation' in str(w.message)]
    assert len(syncs) == 1, syncs                          # the sampled counts
    total = sum(sum(v) for v in rpn_losses.values()) + roi_losses['loss_cls'] + roi_losses['loss_bbox']
    total.backward()
    assert all(bool(torch.isfinite(f.grad).all()) for f in x[:4])
    torch.manual_seed(13)
    smp = orh.sample([p.detach().cpu() for p in proposals], gts, labels, None, train)
    o = orh.targets(smp, gts, labels, 1, [0.] * 4, [0.1, 0.1, 0.2, 0.2], -1)
    rois, lab, lw, bt, bw = seen['targets']
    for name, got, want in (('rois', rois, o[0]), ('labels', lab, o[1]), ('label_weights', lw, o[2]), ('bbox_weights', bw, o[4])):
        assert torch.equal(got.cpu(), want), name
    assert _rel(bt, o[3]) <= 1e-6
    ol = orh.loss(*orh.bbox_forward([f.detach().cpu() for f in x], o[0], {k: v.detach().cpu() for k, v in roi.bbox_head.state_dict().items()}),
                  o[1], o[2], o[3], o[4], 1, False, orh.TINYPERSON['loss_cls'], orh.TINYPERSON['loss_bbox'])
    for k in ('loss_cls', 'loss_bbox', 'acc'):
        assert _rel(roi_losses[k].detach().reshape(-1), ol[k].reshape(-1)) <= 1e-4, k
    calls = []
    real_nms = ops.multiclass_nms_boxes
    monkeypatch.setattr(ops, 'multiclass_nms_boxes', lambda *a, **k: calls.append(1) or real_nms(*a, **k))
    with torch.no_grad():
        props = rpn.simple_test_rpn([f.detach() for f in x], metas)
        res = roi.simple_test([f.detach() for f in x], props, metas)
    assert len(calls) == 1, calls
    assert len(res) == B and res[0][0].shape[1] == 5
