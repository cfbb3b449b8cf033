"""CPU: the oracle of P2PHead with CrossEntropyLoss in softmax mode and with class_weight against the golden vectors the REAL
reference head produced (tests/golden/p2p_softmax_lite.npz, written by oracle/make_golden_p2p_softmax.py), the constructor's host
logic, and the argument checks of the softmax decode and the two class-weighted loss entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import p2p as op2p, p2p_softmax as osm


@pytest.fixture(scope='module')
def case(golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_softmax_lite.npz'))
    inp = osm.inputs(int(gold['seed']))
    d = inp['cfgd']
    cfg = osm.softmax_cfg(use_sigmoid=False, class_weight=gold['class_weight_softmax'].tolist(), num_classes=d['num_classes'],
                          stride=d['stride'], nms_iou=0.5, nms_pre=int(gold['nms_pre']))
    with torch.no_grad():
        cls_out, pts_out = op2p.head_forward(inp['x'], inp['weights'], cfg)
    return gold, inp, cfg, cls_out, pts_out


def _close(a, ref, tol, what):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    d = np.abs(a - ref).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref).max()), f'{what}: max |diff| {d:.3e}'


def sigmoid_maps(cls_out, num_classes):
    """the foreground columns of a softmax cls_out: the sigmoid-mode maps of case (b)."""
    B, _, H, W = cls_out.shape
    return cls_out.reshape(B, -1, num_classes + 1, H, W)[:, :, :num_classes].reshape(B, -1, H, W).contiguous()


def test_oracle_forward_matches_reference_golden(case):
    gold, inp, cfg, cls_out, pts_out = case
    assert cls_out.shape[1] == 4 * (inp['cfgd']['num_classes'] + 1) == 324 and pts_out.shape[1] == 8
    _close(cls_out.flatten()[::37].numpy(), gold['cls_out_sub'], 1e-6, 'cls_out')
    _close(pts_out.flatten().numpy(), gold['pts_out_sub'], 1e-6, 'pts_out')


@pytest.mark.parametrize('mode', ['softmax', 'sigmoid'])
def test_oracle_loss_and_gradients_match_reference_golden(case, mode):
    """(a) softmax cross_entropy with C+1 class weights, (b) binary_cross_entropy with C class weights as pos_weight."""
    gold, inp, cfg, cls_out, pts_out = case
    p = 'sm_' if mode == 'softmax' else 'sg_'
    if mode == 'sigmoid':
        cfg = dict(cfg, use_sigmoid=True, class_weight=gold['class_weight_sigmoid'].tolist())
        cls_out = sigmoid_maps(cls_out, inp['cfgd']['num_classes'])
    co, po = cls_out.clone().requires_grad_(True), pts_out.clone().requires_grad_(True)
    ol, oall = osm.p2p_loss(co, po, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    (sum(ol['loss_cls']) + sum(ol['loss_pts'])).backward()
    assert np.array_equal(torch.stack([t[4] for t in oall['targets']]).numpy().astype(np.int32), gold[p + 'gt_inds'])
    assert np.array_equal(torch.stack([t[0] for t in oall['targets']]).numpy(), gold[p + 'labels'])
    for k in ('loss_cls', 'loss_pts'):
        _close(torch.stack(ol[k]).detach().numpy(), gold[p + k], 1e-6, k)
    _close(co.grad.flatten()[::37].numpy(), gold[p + 'grad_cls_sub'], 1e-6, 'd loss / d cls_out')
    _close(po.grad.flatten().numpy(), gold[p + 'grad_pts_sub'], 1e-6, 'd loss / d pts_out')
    _close(float(co.grad.double().sum()), gold[p + 'grad_cls_sum'], 1e-6, 'sum d/d cls_out')


def test_oracle_get_bboxes_matches_reference_golden(case):
    gold, inp, cfg, cls_out, pts_out = case
    _, pred, _, cls = osm.pred_points(cls_out, pts_out, inp['img_metas'], cfg)
    topk, keep, det, labels = [], [], [], []
    for b, m in enumerate(inp['img_metas']):
        ps, lab, al = osm.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        wh = torch.tensor(cfg['pseudo_wh'])
        det.append(torch.cat([ps[:, :2] - wh / 2, ps[:, :2] + wh / 2, ps[:, 2:]], -1)); labels.append(lab)
        topk.append(al['topk_inds']); keep.append(al['keep'])
        assert len(al['topk_inds']) == cfg['nms_pre'] < cls[b].shape[0]
        assert len(al['cand_inds']) == int(gold['cand_len'][b])
    assert np.array_equal(torch.cat(topk).numpy().astype(np.int32), gold['topk'])
    assert np.array_equal(torch.cat(keep).numpy(), gold['keep'])
    assert np.array_equal(torch.cat(labels).numpy(), gold['det_labels'])
    _close(torch.cat(det).numpy(), gold['det'], 1e-6, 'detections')


def test_oracle_aug_test_matches_reference_golden_without_the_last_class(case):
    """p2p_head.py:534-556: in softmax mode no background column is padded, so multiclass_nms drops class C-1."""
    gold, inp, cfg, cls_out, pts_out = case
    C = inp['cfgd']['num_classes']
    aug_outs, aug_metas = osm.aug_inputs(cls_out, pts_out, inp['img_metas'])
    for rescale in (False, True):
        res, aux = osm.aug_test_bboxes(aug_outs, aug_metas, cfg, rescale=rescale)
        assert np.array_equal(res[0][1].numpy(), gold[f'aug_labels_rescale{int(rescale)}'])
        _close(res[0][0].numpy(), gold[f'aug_det_rescale{int(rescale)}'], 1e-6, f'aug det (rescale={rescale})')
        assert not bool((res[0][1] == C - 1).any())
    assert np.array_equal(aux['keep'].numpy(), gold['aug_keep'])
    assert len(aux['merged_boxes']) == int(gold['aug_n_merged']) > len(gold['aug_keep'])
    assert int(gold['aug_per_aug_last_class']) > 0, 'the per-aug detections include class C-1, which the merge drops'


# ---------------------------------------------------------------------------------------------------------------------------------
def _build(**over):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    base = dict(type='P2PHead', num_classes=80, in_channels=256, feat_channels=256, stacked_convs=4, strides=[8],
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
    base.update(over)
    return build_head(base)


def test_softmax_head_has_a_background_column_per_anchor(case):
    gold, inp, cfg, cls_out, pts_out = case
    head = _build(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, class_weight=gold['class_weight_softmax'].tolist()))
    assert not head.use_sigmoid_cls and head.num_cls_out == 81 and head.cls_out.out_channels == 324
    # the fixture's weights were loaded into the reference head with strict=True: same keys and shapes
    assert {k: tuple(v.shape) for k, v in head.state_dict().items()} == {k: tuple(v.shape) for k, v in inp['weights'].items()}
    # bias_prob=0.01 covers the background channel too (init_cfg override of cls_out)
    assert torch.allclose(head.cls_out.bias, torch.full((324,), -float(np.log(99.0))))
    assert torch.equal(head.class_weight, torch.tensor(gold['class_weight_softmax']))
    assert _build(point_anchor=[(0., 0.)], loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False)).cls_out.out_channels == 81
    assert _build().num_cls_out == 80


def test_softmax_head_channel_limit_counts_the_background_column():
    sm = dict(type='CrossEntropyLoss', use_sigmoid=False)
    assert _build(num_classes=127, loss_cls=sm).cls_out.out_channels == 512
    with pytest.raises(NotImplementedError, match='512'):
        _build(num_classes=128, loss_cls=sm)


def test_class_weight_of_the_wrong_length_and_softmax_focal_are_refused():
    with pytest.raises(ValueError, match='81'):
        _build(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, class_weight=[1.0] * 80))
    with pytest.raises(ValueError, match='80'):
        _build(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, class_weight=[1.0] * 81))
    assert _build(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, class_weight=[2.0] * 80)).class_weight.shape == (80,)
    with pytest.raises(NotImplementedError, match='FocalLoss'):
        _build(loss_cls=dict(type='FocalLoss', use_sigmoid=False, gamma=2.0, alpha=0.25, loss_weight=1.0))


def test_argument_validation_of_the_softmax_entry_points_without_a_gpu():
    """argument checks run before any CUDA call: a bad call returns non-zero and sets ptb_last_error()."""
    from pointtinybenchmark_b200 import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(16)      # never dereferenced: the checks fire first
    # ptb_softmax_ce_fwd_bwd: C1 < 2, NULL logits / labels, no output at all
    assert lib.ptb_softmax_ce_fwd_bwd(d, d, None, None, 10, 1, d, None, None, None) != 0 and b'num_cols' in lib.ptb_last_error()
    assert lib.ptb_softmax_ce_fwd_bwd(None, d, None, None, 10, 81, d, None, None, None) != 0 and b'NULL' in lib.ptb_last_error()
    assert lib.ptb_softmax_ce_fwd_bwd(d, None, None, None, 10, 81, d, None, None, None) != 0 and b'NULL' in lib.ptb_last_error()
    assert lib.ptb_softmax_ce_fwd_bwd(d, d, None, None, 10, 81, None, None, None, None) != 0 and b'NULL' in lib.ptb_last_error()
    assert lib.ptb_softmax_ce_fwd_bwd(d, d, None, None, -1, 81, d, None, None, None) != 0
    # ptb_sigmoid_bce_cw_fwd_bwd
    assert lib.ptb_sigmoid_bce_cw_fwd_bwd(d, d, None, d, 10, 0, d, None, None, None) != 0 and b'num_classes' in lib.ptb_last_error()
    assert lib.ptb_sigmoid_bce_cw_fwd_bwd(None, d, None, d, 10, 80, d, None, None, None) != 0 and b'NULL' in lib.ptb_last_error()
    assert lib.ptb_sigmoid_bce_cw_fwd_bwd(d, d, None, d, 10, 80, None, None, None, None) != 0 and b'NULL' in lib.ptb_last_error()
    # ptb_p2p_decode_topk_softmax: C + 1 < 2, NULL inputs, nms_pre > 4096
    args = lambda ncls, nms_pre, cls=d: (cls, d, 1, 100, 168, ncls, 4, d, 8.0, 12.5, d, None, nms_pre, d, d, d, d, 1 << 30, None)  # noqa: E731
    assert lib.ptb_p2p_decode_topk_softmax(*args(0, 1000)) != 0 and b'num_classes' in lib.ptb_last_error()
    assert lib.ptb_p2p_decode_topk_softmax(*args(80, 1000, cls=None)) != 0 and b'NULL' in lib.ptb_last_error()
    assert lib.ptb_p2p_decode_topk_softmax(*args(80, 5000)) != 0 and b'4096' in lib.ptb_last_error()
