"""GPU: P2PHead at 365 and 1203 classes, where cls_out is wider than one 512-channel conv launch — the wide output conv
(layers._WideOutConvFn: column-sliced forward, deterministic wgrad / col-sum / dgrad backward) against float64, the 512-channel
boundary, the head against the golden vectors of the real reference head (tests/golden/p2p_many_classes_*.npz) and against the
oracle at a mid-size map, aug_test_bboxes in softmax mode and deterministic training."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_defaults as odef, p2p_softmax as osm
from oracle.make_golden_p2p_many_classes import CASES, GRAD_X_STEP, case_inputs, oracle_bboxes_single, oracle_pred_points
from oracle.synth import sample_points
from tests.helpers import assert_close
from tests.test_gpu_p2p_defaults import TEST_CFG, TRAIN_CFG
from tests.test_gpu_p2p_softmax import check_topk_tie_groups

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def build(inp, **over):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    d = inp['cfgd']
    hc = dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
              strides=[d['stride']], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), train_cfg=TRAIN_CFG, test_cfg=TEST_CFG)
    hc.update(over)
    head = build_head(hc)
    head.load_state_dict(inp['weights'], strict=True)
    return head.cuda()


def _graph_names(t, depth=4):
    """names of the autograd nodes within `depth` steps of t.grad_fn"""
    names, level = set(), [t.grad_fn]
    for _ in range(depth):
        level = [f for f in level if f is not None]
        names |= {type(f).__name__ for f in level}
        level = [n for f in level for n, _ in f.next_functions]
    return names


def _wide_conv_run(conv, x, g):
    from pointtinybenchmark_b200.layers import wide_out_conv
    for p in conv.parameters():
        p.grad = None
    xr = x.clone().requires_grad_(True)
    y = wide_out_conv(conv, xr)
    y.backward(g)
    return y.detach(), xr.grad, conv.weight.grad.clone(), conv.bias.grad.clone()


@pytest.mark.parametrize('n_out,H,W', [(513, 19, 27), (1203, 19, 27), (1460, 19, 27), (4812, 19, 27), (4812, 50, 84)])
def test_wide_conv_forward_and_backward_match_float64(ops, n_out, H, W):
    """forward 1e-4 and dW / db / dX 2e-4 (scale-relative) against a float64 conv on maps with partial edge tiles (a bottom strip at
    19 x 27, bottom and right strips at 50 x 84); two backward passes give the same bits."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(n_out)
    B, C = 2, 256
    x = torch.relu(torch.randn(B, C, H, W, generator=g)).to(dev)
    conv = nn.Conv2d(C, n_out, 3, padding=1).to(dev)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(n_out, C, 3, 3, generator=g) * 0.02)
        conv.bias.copy_(torch.randn(n_out, generator=g))
    gy = torch.randn(B, n_out, H, W, generator=g).to(dev)
    y, dx, dw, db = _wide_conv_run(conv, x, gy)
    x64, w64, b64 = x.double().requires_grad_(True), conv.weight.detach().double().requires_grad_(True), \
        conv.bias.detach().double().requires_grad_(True)
    ref = F.conv2d(x64, w64, b64, 1, 1)
    ref.backward(gy.double())
    assert y.shape == (B, n_out, H, W)
    assert_close(y, ref.detach(), 1e-4, f'forward N={n_out}')
    assert_close(dw, w64.grad, 2e-4, f'dW N={n_out}')
    assert_close(db, b64.grad, 2e-4, f'db N={n_out}')
    assert_close(dx, x64.grad, 2e-4, f'dX N={n_out}')
    y2, dx2, dw2, db2 = _wide_conv_run(conv, x, gy)
    assert torch.equal(y, y2) and torch.equal(dx, dx2) and torch.equal(dw, dw2) and torch.equal(db, db2), 'bit-identical reruns'


def test_512_channels_keep_one_slice_and_cudnn_training(ops):
    """at 512 channels (128 classes x 4 anchors) inference is the one ptb_conv_tc_f16x2 launch, bit for bit, and training runs cuDNN;
    at 257 classes (1028 channels) training runs the wide conv."""
    from pointtinybenchmark_b200.layers import _packed_tc, tower
    dev = torch.device('cuda:0')
    inp = odef.inputs(5120, num_classes=128, n=6)
    head = build(inp).eval()
    assert head.cls_out.out_channels == 512
    x = inp['x'].to(dev)
    with torch.no_grad():
        cls_outs, _ = head.forward((x,))
        h, l = tower(head.cls_convs, x, {}, want='f16pair')
        ref = ops.conv_tc_f16(h, l, _packed_tc(head.cls_out, 9), 9, 512, bias=head.cls_out.bias.detach())
    assert torch.equal(cls_outs[0], ref.permute(0, 3, 1, 2))
    head.train()
    cls_outs, _ = head.forward((x,))
    names = _graph_names(cls_outs[0])
    assert 'ConvolutionBackward0' in names and '_WideOutConvFnBackward' not in names, names
    inp = odef.inputs(5160, num_classes=257, n=6)
    head = build(inp).train()
    cls_outs, _ = head.forward((inp['x'].to(dev),))
    assert '_WideOutConvFnBackward' in _graph_names(cls_outs[0])


@pytest.fixture(scope='module', params=sorted(CASES))
def case(request, ops, golden_dir):
    name = request.param
    gold = np.load(os.path.join(golden_dir, f'p2p_many_classes_{name}.npz'))
    inp, cfg, head_kw = case_inputs(name)
    with torch.no_grad():
        oc, op_ = op2p.head_forward(inp['x'], inp['weights'], cfg)
    return name, gold, inp, cfg, head_kw, oc, op_


def check_own_topk(name, got, cls, P, what):
    """top-k of the head's own map: sigmoid keys bit-exact up to exact ties (the GPU's sigmoid is ATen's bit for bit); softmax keys by
    the tie-group rule of tests/test_gpu_p2p_softmax.py (the CUDA softmax is within a few ulps of ATen's)"""
    if CASES[name]['kind'] == 'softmax':
        check_topk_tie_groups(got.numpy(), cls.double().softmax(-1)[:, :-1].max(-1)[0].numpy(), P, what)
        return
    keys = cls.sigmoid().max(-1)[0]
    _, topk = keys.topk(P)
    assert torch.equal(torch.sort(keys[got], descending=True)[0], keys[topk]), what


def test_simple_test_against_reference_golden(ops, case):
    """the head's own maps 1e-4 and its top-k under exact ties; get_bboxes on the oracle's maps: top-k indices, NMS keep and labels bit
    for bit against the golden, detections 1e-4."""
    name, gold, inp, cfg, head_kw, oc, op_ = case
    dev = torch.device('cuda:0')
    head = build(inp, **head_kw).eval()
    metas = inp['img_metas']
    x = inp['x'].to(dev)
    with torch.no_grad():
        cls_outs, pts_outs = head.forward((x,))
        res, aux = head.get_bboxes(cls_outs, pts_outs, metas, return_all=True)
        res2 = head.simple_test((x,), metas)
    assert head.last_tower_backend == 'wgmma-f16x2'
    for a, b in zip(res, res2):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert cls_outs[0].shape[1] == head.cls_out.out_channels > 512
    if cls_outs[0].shape[1] % 4 == 0:       # ldy = n_out: the per-anchor view is the map itself, no copy
        assert cls_outs[0].is_contiguous(memory_format=torch.channels_last)
    assert_close(cls_outs[0], oc, 1e-4, f'{name} cls_out vs oracle')
    assert_close(pts_outs[0], op_, 1e-4, f'{name} pts_out vs oracle')
    _, _, _, cls = oracle_pred_points(name)(cls_outs[0].cpu(), pts_outs[0].cpu(), metas, cfg)
    for b in range(len(metas)):
        check_own_topk(name, aux['topk_idx'][b].cpu().long(), cls[b], min(cfg['nms_pre'], cls[b].shape[0]),
                       f'{name} own-map top-k, image {b}')
    with torch.no_grad():
        res_o, aux_o = head.get_bboxes([oc.to(dev)], [op_.to(dev)], metas, return_all=True)
    _, pred, _, cls = oracle_pred_points(name)(oc, op_, metas, cfg)
    topks, keeps = [], []
    for b, m in enumerate(metas):
        ps, labels, al = oracle_bboxes_single(name)(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        n = int(aux_o['count'][b])
        assert int(aux_o['cand_count'][b]) == len(al['cand_inds']) == int(gold['cand_len'][b])
        assert torch.equal(aux_o['keep'][b, :n].cpu().long(), al['keep']), f'{name} NMS keep image {b}'
        assert torch.equal(res_o[b][1].cpu(), labels)
        topks.append(aux_o['topk_idx'][b].cpu()); keeps.append(aux_o['keep'][b, :n].cpu())
    if len(gold['topk']):
        assert np.array_equal(torch.cat(topks).numpy().astype(np.int32), gold['topk']), f'{name} top-k vs golden'
    assert np.array_equal(torch.cat(keeps).numpy().astype(np.int64), gold['keep']), f'{name} keep vs golden'
    assert np.array_equal(torch.cat([r[1] for r in res_o]).cpu().numpy(), gold['det_labels'])
    assert_close(torch.cat([r[0] for r in res_o]), torch.from_numpy(gold['det']), 1e-4, f'{name} det vs golden')


def _train_step(head, inp, dev):
    head.train()
    head.zero_grad(set_to_none=True)
    x = inp['x'].to(dev).requires_grad_(True)
    cls_outs, pts_outs = head.forward((x,))
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    loss = head.loss(cls_outs, pts_outs, gtb, gtl, inp['img_metas'])
    (sum(loss['loss_cls']) + sum(loss['loss_pts'])).backward()
    return loss, x, cls_outs[0], pts_outs[0]


def test_training_step_against_reference_golden(ops, case):
    """towers + wide output conv + matching + loss + backward of the head: assignments equal the golden, losses 1e-4, the input gradient
    and the stored cls_out / reg_out gradients 2e-4."""
    name, gold, inp, cfg, head_kw, oc, op_ = case
    dev = torch.device('cuda:0')
    head = build(inp, **head_kw)
    loss, x, cls_out, _ = _train_step(head, inp, dev)
    assert '_WideOutConvFnBackward' in _graph_names(cls_out)
    assert np.array_equal(head._last_assign['gt_inds'].cpu().numpy().astype(np.int32), gold['gt_inds']), f'{name} assignments'
    for k in ('loss_cls', 'loss_pts'):
        assert_close(torch.stack(loss[k]), torch.from_numpy(gold[k]), 1e-4, f'{name} {k} vs golden')
    assert_close(x.grad.flatten()[::GRAD_X_STEP], torch.from_numpy(gold['grad_x_sub']), 2e-4, f'{name} d/dx vs golden')
    rows = torch.from_numpy(gold['grad_w_cls_rows']).to(dev)
    assert_close(head.cls_out.weight.grad[rows], torch.from_numpy(gold['grad_w_cls']), 2e-4, f'{name} d/d cls_out.weight rows')
    assert_close(head.cls_out.bias.grad, torch.from_numpy(gold['grad_b_cls']), 2e-4, f'{name} d/d cls_out.bias')
    assert_close(head.reg_out.weight.grad, torch.from_numpy(gold['grad_w_reg']), 2e-4, f'{name} d/d reg_out.weight')
    assert_close(head.reg_out.bias.grad, torch.from_numpy(gold['grad_b_reg']), 2e-4, f'{name} d/d reg_out.bias')


def test_mid_shape_1203_classes_against_oracle(ops):
    """2 images x 50 x 84 at 1203 classes and the reference defaults (cls_out 4812 channels): simple_test, the loss and the gradients
    of the input, cls_out and reg_out against the oracle: the float64 head forward on the GPU, the oracle loss on the CPU over the
    head's own fp32 maps (so both sides match the same assignments), and its map gradients through the float64 head backward."""
    dev = torch.device('cuda:0')
    N, B, H, W, s = 1203, 2, 50, 84, 8
    inp = odef.inputs(12033, num_classes=N, n=10)
    gen = torch.Generator().manual_seed(12034)
    inp['x'] = torch.relu(torch.randn(B, 256, H, W, generator=gen))
    metas, gtb, gtl = [], [], []
    for b, (ih, iw) in enumerate([(H * s - 3, W * s - 5), (H * s - 60, W * s - 90)]):
        pad = (H * s, W * s) if b == 0 else (ih + 4, iw + 4)
        metas.append(dict(pad_shape=pad + (3,), img_shape=(ih, iw, 3), scale_factor=[1.0, 1.0, 1.0, 1.0]))
        pts = sample_points(24, iw, ih, gen)
        gtb.append(torch.cat([pts - 8, pts + 8], dim=1)); gtl.append(torch.randint(0, N, (24,), generator=gen))
    inp.update(img_metas=metas, gt_bboxes=gtb, gt_labels=gtl)
    cfg = odef.reference_defaults_cfg(num_classes=N, stride=s, nms_iou=0.5)
    head = build(inp)
    loss, x, cls_out, pts_out = _train_step(head, inp, dev)
    x64 = inp['x'].to(dev).double().requires_grad_(True)
    w64 = {k: v.to(dev).double().requires_grad_(k.startswith(('cls_out', 'reg_out'))) for k, v in inp['weights'].items()}
    oc64, op64 = op2p.head_forward(x64, w64, cfg)
    co, po = cls_out.detach().cpu().requires_grad_(True), pts_out.detach().cpu().requires_grad_(True)
    ol, oall = odef.p2p_loss(co, po, gtb, gtl, metas, cfg, return_all=True)
    (sum(ol['loss_cls']) + sum(ol['loss_pts'])).backward()
    assert torch.equal(head._last_assign['gt_inds'].cpu(), torch.stack([t[4] for t in oall['targets']])), 'mid assignments vs scipy'
    params = [w64['cls_out.weight'], w64['cls_out.bias'], w64['reg_out.weight'], w64['reg_out.bias']]
    grads = torch.autograd.grad([oc64, op64], [x64] + params, [co.grad.to(dev).double(), po.grad.to(dev).double()])
    assert_close(cls_out, oc64, 1e-4, 'mid cls_out (training forward) vs float64')
    assert_close(pts_out, op64, 1e-4, 'mid pts_out (training forward) vs float64')
    for k in ('loss_cls', 'loss_pts'):
        assert_close(torch.stack(loss[k]), torch.stack(ol[k]).detach(), 1e-4, f'mid {k}')
    for (nm, p), gref in zip([('cls_out.weight', head.cls_out.weight), ('cls_out.bias', head.cls_out.bias),
                              ('reg_out.weight', head.reg_out.weight), ('reg_out.bias', head.reg_out.bias)], grads[1:]):
        assert_close(p.grad, gref, 2e-4, f'mid d/d {nm}')
    # the input gradient passes 8 GroupNorm + ReLU layers of 16 800 pixels x 256 channels: where a pre-activation lies within rounding of
    # zero, the fp32 and float64 forwards gate it differently and that element's gradient differs outright (a few per layer at this
    # size, none at the fixtures' 16 x 16).  So it is compared by its norm here; the output conv's own dX is compared elementwise at
    # 50 x 84 by test_wide_conv_forward_and_backward_match_float64
    rel = float((x.grad.double() - grads[0]).norm() / grads[0].norm())
    print(f'[mid d/dx] norm-relative error {rel:.2e}')
    assert rel <= 5e-3, f'mid d/dx: norm-relative error {rel:.3e}'
    head.eval()
    with torch.no_grad():
        cls_outs, pts_outs = head.forward((inp['x'].to(dev),))
        res, aux = head.get_bboxes(cls_outs, pts_outs, metas, return_all=True)
    assert cls_outs[0].is_contiguous(memory_format=torch.channels_last)
    assert_close(cls_outs[0], oc64, 1e-4, 'mid simple_test cls_out vs float64')
    _, pred, _, cls = op2p.pred_points(cls_outs[0].cpu(), pts_outs[0].cpu(), metas, cfg)
    for b, m in enumerate(metas):
        keys = cls[b].sigmoid().max(dim=1)[0]
        got = aux['topk_idx'][b].cpu().long()
        _, topk = keys.topk(cfg['nms_pre'])
        assert torch.equal(torch.sort(keys[got], descending=True)[0], keys[topk]), f'mid top-k keys, image {b}'
        ps, labels, al = op2p.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        if torch.equal(torch.sort(got)[0], torch.sort(al['topk_inds'])[0]):      # same selected set: NMS must agree bit for bit
            assert int(aux['count'][b]) == len(al['keep'])
            assert torch.equal(res[b][1].cpu(), labels), f'mid labels, image {b}'


def test_aug_test_bboxes_softmax_at_365_classes(ops):
    """aug_test_bboxes through the head's own forward (cls_out 4 x 366 = 1464 channels) against the oracle's merge over the same maps:
    class C-1 is absent, labels equal, detections 1e-4."""
    dev = torch.device('cuda:0')
    inp, cfg, head_kw = case_inputs('softmax_365')
    C = inp['cfgd']['num_classes']
    head = build(inp, **head_kw).eval()
    x = inp['x'].to(dev)
    feats = [(x[:1],), (x[:1].flip(3),), (x[1:2],)]
    metas = [[dict(inp['img_metas'][0], flip=False, flip_direction='horizontal')],
             [dict(inp['img_metas'][0], flip=True, flip_direction='horizontal', tile_offset=(3, 2))],
             [dict(inp['img_metas'][1], scale_factor=[1.5] * 4, flip=False, flip_direction='horizontal')]]
    with torch.no_grad():
        outs = [head.forward(f) for f in feats]
        res = head.aug_test_bboxes(feats, metas, rescale=False)
    aug_outs = [(c[0].cpu(), p[0].cpu()) for c, p in outs]
    ores, _ = osm.aug_test_bboxes(aug_outs, metas, cfg, rescale=False)
    det, lab = res[0][0].cpu(), res[0][1].cpu()
    assert len(lab) > 0 and not bool((lab == C - 1).any())
    assert torch.equal(lab, ores[0][1]), 'labels after the second NMS'
    assert_close(det, ores[0][0], 1e-4, 'merged detections')


def test_deterministic_training_at_1203_classes(ops):
    """under torch.use_deterministic_algorithms(True) the training step at 4 x 1203 channels runs and repeats bit for bit."""
    dev = torch.device('cuda:0')
    inp, _, head_kw = case_inputs('defaults_1203')
    head = build(inp, **head_kw)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            loss, x, _, _ = _train_step(head, inp, dev)
            runs.append([torch.stack(loss['loss_cls']), x.grad] + [p.grad.clone() for p in head.parameters()])
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert torch.equal(a, b)
