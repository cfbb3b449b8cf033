"""CPU: the oracle of P2PHead at the reference class's own defaults (four point anchors per cell, CrossEntropyLoss(use_sigmoid) +
MSELoss) against the golden vectors the REAL reference head produced (tests/golden/p2p_defaults_lite.npz, written by
oracle/make_golden_p2p_defaults.py), and the construction-time limit on the output conv width."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p, p2p_defaults as odef


@pytest.fixture(scope='module')
def case(golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_defaults_lite.npz'))
    inp = odef.inputs(int(gold['seed']))
    cfg = odef.reference_defaults_cfg(num_classes=inp['cfgd']['num_classes'], stride=inp['cfgd']['stride'], nms_iou=0.5)
    with torch.no_grad():
        cls_out, pts_out = op2p.head_forward(inp['x'], inp['weights'], cfg)
    return gold, inp, cfg, cls_out, pts_out


def _close(a, ref, tol, what):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    d = np.abs(a - ref).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref).max()), f'{what}: max |diff| {d:.3e}'


def test_oracle_forward_matches_reference_golden(case):
    gold, inp, cfg, cls_out, pts_out = case
    assert cls_out.shape[1] == 4 * inp['cfgd']['num_classes'] == 320 and pts_out.shape[1] == 8
    _close(cls_out.flatten()[::37].numpy(), gold['cls_out_sub'], 1e-6, 'cls_out')
    _close(pts_out.flatten().numpy(), gold['pts_out_sub'], 1e-6, 'pts_out')


def test_oracle_loss_and_gradients_match_reference_golden(case):
    gold, inp, cfg, cls_out, pts_out = case
    co, po = cls_out.clone().requires_grad_(True), pts_out.clone().requires_grad_(True)
    ol, oall = odef.p2p_loss(co, po, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    (sum(ol['loss_cls']) + sum(ol['loss_pts'])).backward()
    assert np.array_equal(torch.stack([t[4] for t in oall['targets']]).numpy().astype(np.int32), gold['gt_inds'])
    for k in ('loss_cls', 'loss_pts'):
        _close(torch.stack(ol[k]).detach().numpy(), gold[k], 1e-6, k)
    _close(co.grad.flatten()[::37].numpy(), gold['grad_cls_sub'], 1e-6, 'd loss / d cls_out')
    _close(po.grad.flatten().numpy(), gold['grad_pts_sub'], 1e-6, 'd loss / d pts_out')
    _close(float(co.grad.double().sum()), gold['grad_cls_sum'], 1e-6, 'sum d/d cls_out')


def test_ce_averages_over_all_proposals_and_mse_over_positives(case):
    """p2p_head.py:200,220-240: CrossEntropyLoss divides by num_total (every proposal of the batch), MSELoss by num_total_pos."""
    gold, inp, cfg, cls_out, pts_out = case
    ol, oall = odef.p2p_loss(cls_out, pts_out, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    tg = oall['targets']
    n_total = sum(len(t[0]) for t in tg)
    n_pos = int(sum((t[3][:, 0] > 0).sum() for t in tg))
    assert n_total == inp['cfgd']['B'] * cls_out.shape[2] * cls_out.shape[3] * 4 and 0 < n_pos < n_total
    l0 = odef.sigmoid_bce_elem(oall['cls'][0], tg[0][0])
    assert abs(float((l0 * tg[0][1][:, None]).sum() / n_total) - float(ol['loss_cls'][0])) <= 1e-6 * abs(float(ol['loss_cls'][0]))


def test_oracle_get_bboxes_matches_reference_golden(case):
    gold, inp, cfg, cls_out, pts_out = case
    _, pred, _, cls = op2p.pred_points(cls_out, pts_out, inp['img_metas'], cfg)
    topk, keep, det, labels = [], [], [], []
    for b, m in enumerate(inp['img_metas']):
        ps, lab, al = op2p.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        wh = torch.tensor(cfg['pseudo_wh'])
        det.append(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1)); labels.append(lab)
        topk.append(al['topk_inds']); keep.append(al['keep'])
        assert len(al['cand_inds']) == int(gold['cand_len'][b])
    assert np.array_equal(torch.cat(topk).numpy().astype(np.int32), gold['topk'])
    assert np.array_equal(torch.cat(keep).numpy(), gold['keep'])
    assert np.array_equal(torch.cat(labels).numpy(), gold['det_labels'])
    _close(torch.cat(det).numpy(), gold['det'], 1e-6, 'detections')


def test_p2p_head_rejects_output_convs_wider_than_the_kernel_at_construction():
    """4 anchors x C classes must fit the 512-channel output conv: C = 128 builds, C = 129 fails in the constructor (not inside the
    library at the first forward)."""
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    base = dict(type='P2PHead', in_channels=256, feat_channels=256, stacked_convs=1, strides=[8],
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
    head = build_head(dict(base, num_classes=128))
    assert head.num_points == 4 and head.cls_out.out_channels == 512
    with pytest.raises(NotImplementedError, match='512'):
        build_head(dict(base, num_classes=129))
    with pytest.raises(NotImplementedError, match='512'):
        build_head(dict(base, num_classes=80, point_anchor=[(0., 0.)] * 7))
    assert build_head(dict(base, num_classes=80, point_anchor=[(0., 0.)])).cls_out.out_channels == 80
