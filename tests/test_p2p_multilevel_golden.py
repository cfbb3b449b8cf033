"""CPU: P2PHead over several FPN levels.  The multi-level oracle (oracle/p2p_multilevel.py) against the vectors the REAL reference head
produced (tests/golden/p2p_multilevel_*.npz, written by oracle/make_golden_p2p_multilevel.py), the head's construction with the
reference's state_dict names and shapes, its level-major proposal rows, and the host chunk plan of the multi-level decode: chunk
boundaries, the T % L refusal, and the unchanged single-level plan."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_multilevel as oml
from oracle.make_golden_p2p_multilevel import GRAD_STEP
from pointtinybenchmark_b200 import ops
from pointtinybenchmark_b200.p2p_head import P2PHead


def _close(a, ref, tol, what):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape, (what, a.shape, ref.shape)
    d = np.abs(a - ref).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref).max()), f'{what}: max |diff| {d:.3e}'


def head_kwargs(cfg):
    if cfg['loss_cls'] == 'FocalLoss':
        loss_cls = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=cfg['loss_cls_weight'])
    else:
        loss_cls = dict(type='CrossEntropyLoss', use_sigmoid=cfg.get('use_sigmoid', True), loss_weight=cfg['loss_cls_weight'],
                        class_weight=cfg.get('class_weight'))
    loss_reg = (dict(type='SmoothL1Loss', beta=cfg['sl1_beta'], loss_weight=cfg['loss_reg_weight']) if cfg['loss_reg'] == 'SmoothL1Loss'
                else dict(type='MSELoss', loss_weight=cfg['loss_reg_weight']))
    return dict(num_classes=cfg['num_classes'], in_channels=oml.C_FEAT, feat_channels=oml.C_FEAT, stacked_convs=4,
                strides=list(cfg['strides']), point_anchor=[tuple(a) for a in cfg['point_anchor']], pts_gamma=cfg['pts_gamma'],
                reg_norm=cfg['reg_norm'], loss_cls=loss_cls, loss_reg=loss_reg, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))


@pytest.fixture(scope='module', params=sorted(oml.CASES))
def case(request, golden_dir):
    name = request.param
    gold = np.load(os.path.join(golden_dir, f'p2p_multilevel_{name}.npz'))
    inp, cfg = oml.case_inputs(name)
    assert int(gold['seed']) == oml.CASES[name]['seed']
    w = {k: v.clone().requires_grad_(True) for k, v in inp['weights'].items()}
    cls_outs, pts_outs = oml.head_forward(inp['xs'], w, cfg)
    loss, aux = oml.p2p_loss(cls_outs, pts_outs, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    (sum(loss['loss_cls']) + sum(loss['loss_pts'])).backward()
    return name, gold, inp, cfg, [c.detach() for c in cls_outs], [p.detach() for p in pts_outs], loss, aux, w


def test_oracle_training_matches_reference_golden(case):
    name, gold, inp, cfg, cls_outs, pts_outs, loss, aux, w = case
    assert np.array_equal(torch.stack([t[4] for t in aux['targets']]).numpy().astype(np.int32), gold['gt_inds'])
    assert np.array_equal(torch.stack([t[0] for t in aux['targets']]).numpy(), gold['labels'])
    _close(torch.stack([t[2] for t in aux['targets']]).numpy(), gold['gt_pts'], 0, f'{name} gt_pts')
    for k in ('loss_cls', 'loss_pts'):
        _close(torch.stack(loss[k]).detach().numpy(), gold[k], 1e-6, f'{name} {k}')
    for k, v in w.items():
        step = GRAD_STEP if v.dim() == 4 else 1
        _close(v.grad.flatten()[::step].numpy(), gold[f'grad/{k}'], 1e-5, f'{name} d/d{k}')


def test_oracle_inference_matches_reference_golden(case):
    name, gold, inp, cfg, cls_outs, pts_outs, *_ = case
    metas = inp['img_metas']
    if 'ref_error' in gold.files:
        assert int(gold['T']) % len(cls_outs) != 0
        with pytest.raises(RuntimeError):
            oml.p2p_get_bboxes(cls_outs, pts_outs, metas, cfg)
        with pytest.raises(RuntimeError, match='equal chunks'):
            ops.p2p_chunk_plan([c.shape[-2:] for c in cls_outs], len(cfg['point_anchor']), cfg['nms_pre'])
        return
    res, aux = oml.p2p_get_bboxes(cls_outs, pts_outs, metas, cfg, return_all=True)
    assert np.array_equal(np.array([len(r[0]) for r in res]), gold['det_len'])
    _close(torch.cat([r[0] for r in res]).numpy(), gold['det'], 1e-6, f'{name} det')
    assert np.array_equal(torch.cat([r[1] for r in res]).numpy(), gold['det_labels'])
    assert np.array_equal(torch.cat([a['keep'] for a in aux]).numpy(), gold['keep'])
    assert np.array_equal(torch.stack([torch.stack(a['topk_inds']) for a in aux]).numpy(), gold['topk'])


def test_oracle_aug_test_matches_reference_golden(golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_multilevel_aug.npz'))
    feats, metas, w, cfg = oml.aug_inputs()
    outs = [oml.head_forward(x, w, cfg) for x in feats]
    res, _ = oml.aug_test_bboxes(outs, metas, cfg)
    _close(res[0][0].numpy(), gold['det'], 1e-6, 'aug det')
    assert np.array_equal(res[0][1].numpy(), gold['det_labels'])


@pytest.mark.parametrize('name', sorted(oml.CASES))
def test_head_builds_with_reference_state_dict(name):
    inp, cfg = oml.case_inputs(name)
    head = P2PHead(**head_kwargs(cfg))
    sd = head.state_dict()
    assert sorted(sd) == sorted(inp['weights'])
    assert all(tuple(sd[k].shape) == tuple(v.shape) for k, v in inp['weights'].items())
    head.load_state_dict(inp['weights'], strict=True)


def test_head_proposal_rows_are_level_major_as_the_reference():
    """get_pred_points_levels (pure torch) against the oracle's per-level rows: anchors, points, valid flags, logits, strides."""
    inp, cfg = oml.case_inputs('b_defaults')
    head = P2PHead(**head_kwargs(cfg))
    gen = torch.Generator().manual_seed(3)
    cls_outs = [torch.randn(2, 4 * 80, h, w, generator=gen) for h, w in oml.CASES['b_defaults']['maps']]
    pts_outs = [torch.randn(2, 8, h, w, generator=gen) for h, w in oml.CASES['b_defaults']['maps']]
    anchor, pred, valid, cls = head.get_pred_points_levels(cls_outs, pts_outs, inp['img_metas'])
    oa, op_, ov, oc = oml.pred_points(cls_outs, pts_outs, inp['img_metas'], cfg)
    assert torch.equal(anchor, oa[..., :2]) and torch.equal(valid, ov) and torch.equal(cls, oc)
    inv = head.row_inv_norm(oml.CASES['b_defaults']['maps'], 'cpu')
    assert torch.equal(inv, (1.0 / (op_[0, :, 2].double() * cfg['reg_norm'])).float())
    assert head.row_inv_norm(oml.CASES['b_defaults']['maps'], 'cpu') is inv
    _close(pred.numpy(), op_[..., :2].numpy(), 1e-6, 'pred points')


def test_single_level_rows_and_plan_are_unchanged():
    """strides=[s]: the multi-level builder gives the single-level rows, and the chunk plan is one chunk of every row."""
    inp, cfg = oml.case_inputs('a_focal_sl1')
    kw = dict(head_kwargs(cfg), strides=[8])
    head = P2PHead(**kw)
    gen = torch.Generator().manual_seed(4)
    c, p = torch.randn(2, 80, 16, 16, generator=gen), torch.randn(2, 2, 16, 16, generator=gen)
    one = head.get_pred_points(c, p, inp['img_metas'])
    lv = head.get_pred_points_levels([c], [p], inp['img_metas'])
    for a, b in zip(one, lv):
        assert torch.equal(a, b)
    for nms_pre, P in ((-1, 256), (0, 256), (100, 100), (255, 255), (256, 256), (1000, 256)):
        assert ops.p2p_chunk_plan([(16, 16)], 1, nms_pre) == dict(T=256, L=1, chunk=256, P=P, level_row0=[0, 256])


@pytest.mark.parametrize('maps,k,nms_pre,chunk,row0', [
    ([(16, 16), (8, 8), (4, 4)], 1, 50, 112, [0, 256, 320, 336]),      # boundaries 112, 224 inside level 0; the last chunk spans 3 levels
    ([(16, 16), (8, 8)], 4, 300, 640, [0, 1024, 1280]),                 # boundary 640 inside level 0
    ([(4, 4), (4, 4)], 1, 5, 16, [0, 16, 32]),                          # the chunk boundary is the level boundary
    ([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], 4, 1000, 17920, [0, 67200, 84000, 88200, 89292, 89600]),  # 1333 x 800
])
def test_chunk_plan(maps, k, nms_pre, chunk, row0):
    plan = ops.p2p_chunk_plan(maps, k, nms_pre)
    assert plan == dict(T=row0[-1], L=len(maps), chunk=chunk, P=min(nms_pre, chunk) if nms_pre < chunk else chunk, level_row0=row0)


@pytest.mark.parametrize('maps,k', [([(16, 15), (8, 8), (4, 4)], 1), ([(3, 3), (2, 2)], 1), ([(5, 5), (3, 3), (1, 1)], 1)])
def test_chunk_plan_refuses_uneven_chunks(maps, k):
    with pytest.raises(RuntimeError, match='equal chunks'):
        ops.p2p_chunk_plan(maps, k, 100)


def test_level_count_limit():
    _, cfg = oml.case_inputs('a_focal_sl1')
    P2PHead(**dict(head_kwargs(cfg), strides=[4, 8, 16, 32, 64, 128, 256, 512]))
    with pytest.raises(NotImplementedError, match='1 to 8'):
        P2PHead(**dict(head_kwargs(cfg), strides=[4, 8, 16, 32, 64, 128, 256, 512, 1024]))
