"""CPU: the P2P oracles at 365 and 1203 classes (cls_out of 1203 to 4812 channels, wider than one 512-channel conv launch) against the
golden vectors the REAL reference head produced (tests/golden/p2p_many_classes_*.npz, written by
oracle/make_golden_p2p_many_classes.py), the wide output conv's shape rule (layers.wide_out_conv_plan) at its boundaries, and the
head's construction-time class limit."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p
from oracle.make_golden_p2p_many_classes import (CASES, GRAD_X_STEP, MAP_STEP, case_inputs, oracle_bboxes_single, oracle_loss,
                                                 oracle_pred_points, weight_rows)


def _close(a, ref, tol, what):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    d = np.abs(a - ref).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref).max()), f'{what}: max |diff| {d:.3e}'


@pytest.fixture(scope='module', params=sorted(CASES))
def case(request, golden_dir):
    name = request.param
    gold = np.load(os.path.join(golden_dir, f'p2p_many_classes_{name}.npz'))
    inp, cfg, _ = case_inputs(name)
    assert int(gold['seed']) == CASES[name]['seed']
    x = inp['x'].clone().requires_grad_(True)
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    cls_out, pts_out = op2p.head_forward(x, w, cfg)
    loss, aux = oracle_loss(name)(cls_out, pts_out, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    (sum(loss['loss_cls']) + sum(loss['loss_pts'])).backward()
    return name, gold, inp, cfg, cls_out.detach(), pts_out.detach(), loss, aux, x, w


def test_cls_out_is_wider_than_one_conv_launch(case):
    name, gold, inp, cfg, cls_out, *_ = case
    k = len(cfg['point_anchor'])
    n_cls = CASES[name]['num_classes'] + (1 if CASES[name]['kind'] == 'softmax' else 0)
    assert cls_out.shape[1] == k * n_cls > 512
    if name == 'shipped_1203':
        assert cls_out.shape[1] % 4 != 0


def test_oracle_forward_matches_reference_golden(case):
    name, gold, inp, cfg, cls_out, pts_out, *_ = case
    _close(cls_out.flatten()[::MAP_STEP].numpy(), gold['cls_out_sub'], 1e-6, f'{name} cls_out')
    _close(float(cls_out.double().sum()), gold['cls_out_sum'], 1e-6, f'{name} sum cls_out')
    _close(pts_out.flatten().numpy(), gold['pts_out_sub'], 1e-6, f'{name} pts_out')


def test_oracle_loss_assignments_and_gradients_match_reference_golden(case):
    name, gold, inp, cfg, cls_out, pts_out, loss, aux, x, w = case
    assert np.array_equal(torch.stack([t[4] for t in aux['targets']]).numpy().astype(np.int32), gold['gt_inds'])
    for k in ('loss_cls', 'loss_pts'):
        _close(torch.stack(loss[k]).detach().numpy(), gold[k], 1e-6, f'{name} {k}')
    _close(x.grad.flatten()[::GRAD_X_STEP].numpy(), gold['grad_x_sub'], 1e-6, f'{name} d/dx')
    _close(float(x.grad.double().sum()), gold['grad_x_sum'], 1e-6, f'{name} sum d/dx')
    rows = gold['grad_w_cls_rows']
    assert np.array_equal(rows, weight_rows(name, cls_out.shape[1], len(cfg['point_anchor'])))
    assert rows[0] == 0 and rows[-1] == cls_out.shape[1] - 1
    _close(w['cls_out.weight'].grad[torch.from_numpy(rows)].numpy(), gold['grad_w_cls'], 1e-6, f'{name} d/d cls_out.weight rows')
    _close(w['cls_out.bias'].grad.numpy(), gold['grad_b_cls'], 1e-6, f'{name} d/d cls_out.bias')
    _close(w['reg_out.weight'].grad.numpy(), gold['grad_w_reg'], 1e-6, f'{name} d/d reg_out.weight')
    _close(w['reg_out.bias'].grad.numpy(), gold['grad_b_reg'], 1e-6, f'{name} d/d reg_out.bias')


def test_oracle_get_bboxes_matches_reference_golden(case):
    name, gold, inp, cfg, cls_out, pts_out, *_ = case
    _, pred, _, cls = oracle_pred_points(name)(cls_out, pts_out, inp['img_metas'], cfg)
    topk, keep, det, labels = [], [], [], []
    for b, m in enumerate(inp['img_metas']):
        ps, lab, al = oracle_bboxes_single(name)(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        wh = torch.tensor(cfg['pseudo_wh'])
        det.append(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1)); labels.append(lab)
        topk.append(al['topk_inds'] if al['topk_inds'] is not None else torch.zeros(0, dtype=torch.long)); keep.append(al['keep'])
        assert len(al['cand_inds']) == int(gold['cand_len'][b])
    assert np.array_equal(torch.cat(topk).numpy().astype(np.int32), gold['topk'])
    assert np.array_equal(torch.cat(keep).numpy(), gold['keep'])
    assert np.array_equal(torch.cat(labels).numpy(), gold['det_labels'])
    _close(torch.cat(det).numpy(), gold['det'], 1e-6, f'{name} detections')


def test_wide_out_conv_plan_row_stride_and_32_bit_limits():
    from pointtinybenchmark_b200.layers import INT32_MAX, wide_out_conv_plan
    # inference: ceil4, so the (B,H,W,n_out) view is the whole map when 4 | n_out; training: ceil32 (dX is a conv with Cin = ldy)
    assert wide_out_conv_plan(16, 100, 168, 4812, 4) == 4812
    assert wide_out_conv_plan(16, 100, 168, 1460, 4) == 1460
    assert wide_out_conv_plan(16, 100, 168, 1203, 1) == 1204
    assert wide_out_conv_plan(16, 100, 168, 4812, 4, backward=True) == 4832
    assert wide_out_conv_plan(16, 100, 168, 1460, 4, backward=True) == 1472
    assert wide_out_conv_plan(16, 100, 168, 1464, 4, backward=True) == 1472
    assert wide_out_conv_plan(16, 100, 168, 513, 1, backward=True) == 544
    # the headline batch and twice it: 1.3e9 and 2.6e9 map elements (past 2^31); every element offset of the path is 64-bit
    assert 16 * 100 * 168 * 4832 < 2 ** 31 < 32 * 100 * 168 * 4832
    assert wide_out_conv_plan(32, 100, 168, 4812, 4, backward=True) == 4832
    # the decode's proposal index is int32: H * W * k at the limit passes, one more cell fails
    H = INT32_MAX // (4 * 1024)
    assert wide_out_conv_plan(1, H, 1024, 516, 4) == 516
    assert H * 1024 * 4 <= INT32_MAX < (H + 1) * 1024 * 4
    with pytest.raises(ValueError, match='32 bits'):
        wide_out_conv_plan(1, H + 1, 1024, 516, 4)
    # the conv / wgrad tensor maps of the fp16 gradient take per-image strides below 2^40 bytes
    assert wide_out_conv_plan(1, 2 ** 14, 2 ** 13, 4064, 1, backward=True) == 4064
    with pytest.raises(ValueError, match='2\\^40'):
        wide_out_conv_plan(1, 2 ** 14, 2 ** 13, 4065, 1, backward=True)             # ldy 4096: exactly 2^40 bytes
    with pytest.raises(ValueError, match='empty'):
        wide_out_conv_plan(0, 100, 168, 4812, 4)


def _build(**over):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    base = dict(type='P2PHead', num_classes=80, in_channels=256, feat_channels=256, stacked_convs=1, strides=[8],
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
    base.update(over)
    return build_head(base)


def test_p2p_head_class_limit_at_construction():
    """above 256 classes (the many-class path, CPRHead's threshold) up to 1280 (CPRHead's limit) at any anchor count and in both
    classification modes; 1281 fails in the constructor, naming the limit.  Up to 256 classes cls_out must still fit one 512-channel
    launch, and reg_out always does."""
    sm = dict(type='CrossEntropyLoss', use_sigmoid=False)
    assert _build(num_classes=128).cls_out.out_channels == 512
    assert _build(num_classes=127, loss_cls=sm).cls_out.out_channels == 512
    for kw in (dict(num_classes=129), dict(num_classes=256), dict(num_classes=128, loss_cls=sm), dict(num_classes=255, loss_cls=sm),
               dict(num_classes=80, point_anchor=[(0., 0.)] * 7)):
        with pytest.raises(NotImplementedError, match='512'):
            _build(**kw)
    assert _build(num_classes=256, point_anchor=[(0., 0.)] * 2).cls_out.out_channels == 512
    assert _build(num_classes=257).cls_out.out_channels == 1028
    with pytest.raises(NotImplementedError, match='512'):
        _build(num_classes=256, loss_cls=sm, point_anchor=[(0., 0.)] * 2)            # 2 x 257 = 514 channels
    assert _build(num_classes=257, loss_cls=sm).cls_out.out_channels == 1032
    assert _build(num_classes=1280).cls_out.out_channels == 5120
    assert _build(num_classes=1280, loss_cls=sm).cls_out.out_channels == 5124
    assert _build(num_classes=1203, point_anchor=[(0., 0.)]).cls_out.out_channels == 1203
    for kw in (dict(), dict(loss_cls=sm), dict(point_anchor=[(0., 0.)])):
        with pytest.raises(NotImplementedError, match='1280'):
            _build(num_classes=1281, **kw)
    with pytest.raises(NotImplementedError, match='512'):
        _build(num_classes=1, point_anchor=[(0., 0.)] * 257)
    with pytest.raises(NotImplementedError, match='feat_channels=256'):
        _build(num_classes=365, feat_channels=128, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
    # class_weight length checks are unchanged at these widths
    with pytest.raises(ValueError, match='366'):
        _build(num_classes=365, loss_cls=dict(sm, class_weight=[1.0] * 365))


def test_wide_output_conv_has_no_cpu_path():
    head = _build(num_classes=365)
    with pytest.raises(RuntimeError, match='CUDA'):
        head.forward((torch.zeros(1, 256, 4, 4),))
