"""GPU: P2PHead at the reference class's own defaults — four point anchors per cell (cls_out = 4 x 80 = 320 channels, wider than one
256-channel conv) and the CrossEntropyLoss(use_sigmoid) + MSELoss pair — against fp32 torch, the CPU oracle and the golden vectors
of the real reference head (tests/golden/p2p_defaults_lite.npz)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_defaults as odef
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

TRAIN_CFG = dict(neg_weight=1.0, assigner=dict(type='HungarianAssignerV2', cls_costs=dict(type='FocalLossCost', weight=2.0),
                                               reg_costs=dict(type='DisCostV2', weight=0.1, norm_with_img_wh=False), topk_k=5),
                 sampler=dict(type='PseudoSampler'))
TEST_CFG = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, pseudo_wh=(32, 32), nms=dict(type='nms', iou_threshold=0.5),
                max_per_img=100)


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


@pytest.fixture(scope='module')
def case(ops, golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_defaults_lite.npz'))
    inp = odef.inputs(int(gold['seed']))
    d = inp['cfgd']
    cfg = odef.reference_defaults_cfg(num_classes=d['num_classes'], stride=d['stride'], nms_iou=0.5)
    with torch.no_grad():
        oc, op_ = op2p.head_forward(inp['x'], inp['weights'], cfg)
    return gold, inp, cfg, oc, op_


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


@pytest.mark.parametrize('n_out', [264, 320, 512])
@pytest.mark.parametrize('taps', [1, 9])
def test_wide_conv_one_slice_matches_fp32(ops, n_out, taps):
    """ptb_conv_tc_f16x2 beyond 256 output channels (3 / 3 / 4 channel slices of 128 in one launch), with bias, on a map with partial
    edge tiles, against torch's fp32 conv (float64 reference)."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(n_out + taps)
    B, H, W, C = 2, 19, 27, 256
    x = torch.relu(torch.randn(B, C, H, W, generator=g))
    w = torch.randn(n_out, C, 3, 3, generator=g) * 0.02 if taps == 9 else torch.randn(n_out, C, 1, 1, generator=g) * 0.05
    b = torch.randn(n_out, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), 1, 1 if taps == 9 else 0).float()
    h, l, dinv = ops.split_f16(ops.to_nhwc(x.to(dev)).contiguous(), auto_scale=True)
    packed = ops.conv_tc_pack_weight_f16(w.reshape(n_out, C, taps).to(dev), taps)
    [(c0, n, (_, _, _, n_mma))] = packed                 # one slice, one launch, up to 512 channels
    assert (c0, n, n_mma) == (0, n_out, (n_out + 15) // 16 * 16)
    y = ops.conv_tc_f16(h, l, packed, taps, n_out, bias=b.to(dev), dev_out_scale=dinv)
    assert y.shape[-1] == (n_out + 3) // 4 * 4
    assert_close(y[..., :n_out].permute(0, 3, 1, 2), ref, 1e-4, f'wide tc conv taps={taps} N={n_out}')
    # fp32 torch on the GPU (cuDNN, TF32 off) agrees as well
    ref32 = F.conv2d(x.to(dev), w.to(dev), b.to(dev), 1, 1 if taps == 9 else 0)
    assert_close(y[..., :n_out].permute(0, 3, 1, 2), ref32, 1e-4, f'wide tc conv vs cuDNN fp32 taps={taps} N={n_out}')


def test_simple_test_at_reference_defaults(ops, case):
    gold, inp, cfg, oc, op_ = case
    dev = torch.device('cuda:0')
    head = build(inp).eval()
    assert head.num_points == 4 and head.cls_out.out_channels == 320
    x = inp['x'].to(dev)
    metas = inp['img_metas']
    with torch.no_grad():
        cls_outs, pts_outs = head.forward((x,))
        res, aux = head.get_bboxes(cls_outs, pts_outs, metas, return_all=True)
        res2 = head.simple_test((x,), metas)
    assert head.last_tower_backend == 'wgmma-f16x2', 'towers and output convs on the wgmma path'
    for a, b in zip(res, res2):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert_close(cls_outs[0], oc, 1e-4, 'cls_out (320 channels) vs oracle')
    assert_close(pts_outs[0], op_, 1e-4, 'pts_out vs oracle')
    assert_close(cls_outs[0].flatten()[::37], torch.from_numpy(gold['cls_out_sub']), 1e-4, 'cls_out vs golden')
    # post-processing of the head's own maps: top-k keys / set exact (order free only inside exact ties), NMS vs the oracle
    _, pred, _, cls = op2p.pred_points(cls_outs[0].cpu(), pts_outs[0].cpu(), metas, cfg)
    for b, m in enumerate(metas):
        keys = cls[b].sigmoid().max(dim=1)[0]
        _, topk = keys.topk(cfg['nms_pre'])
        got = aux['topk_idx'][b].cpu().long()
        assert torch.equal(keys[got], keys[topk]) and torch.equal(torch.sort(got)[0], torch.sort(topk)[0]), f'top-k, image {b}'
        ps, labels, al = op2p.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        n = int(aux['count'][b])
        assert n == len(al['keep'])
        assert torch.equal(res[b][1].cpu(), labels), f'labels of the kept detections, image {b}'
        assert_close(res[b][0][:, :4], torch.cat([ps[:, :2] - 16, ps[:, :2] + 16], -1), 1e-4, f'kept boxes, image {b}')
    # get_bboxes on the oracle's maps: top-k indices and NMS keep bit-exact against the oracle and the golden
    with torch.no_grad():
        res_o, aux_o = head.get_bboxes([oc.to(dev)], [op_.to(dev)], metas, return_all=True)
    _, pred, _, cls = op2p.pred_points(oc, op_, metas, cfg)
    topks, keeps = [], []
    for b, m in enumerate(metas):
        ps, labels, al = op2p.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        assert torch.equal(aux_o['topk_idx'][b].cpu().long(), al['topk_inds']), f'top-k indices image {b}'
        n = int(aux_o['count'][b])
        assert int(aux_o['cand_count'][b]) == len(al['cand_inds']) == int(gold['cand_len'][b])
        assert torch.equal(aux_o['keep'][b, :n].cpu().long(), al['keep']), f'NMS keep image {b}'
        assert torch.equal(res_o[b][1].cpu(), labels)
        assert_close(aux_o['scores'][b], al['scores'], 1e-4, 'top-k scores')
        topks.append(aux_o['topk_idx'][b].cpu()); keeps.append(aux_o['keep'][b, :n].cpu())
    assert np.array_equal(torch.cat(topks).numpy().astype(np.int32), gold['topk']), 'top-k vs golden'
    assert np.array_equal(torch.cat(keeps).numpy().astype(np.int64), gold['keep']), 'keep vs golden'
    assert np.array_equal(torch.cat([r[1] for r in res_o]).cpu().numpy(), gold['det_labels'])
    assert_close(torch.cat([r[0] for r in res_o]), torch.from_numpy(gold['det']), 1e-4, 'det vs golden')


@pytest.mark.parametrize('losses', ['ce_mse', 'focal_sl1'])
def test_loss_and_gradients_at_four_anchors(ops, case, losses):
    """P2PHead.loss + backward with 4 anchors per cell: Hungarian assignments bit-exact against scipy (oracle) and the golden, losses
    1e-4, gradients 2e-4.  'ce_mse' = the reference defaults (golden too); 'focal_sl1' = the shipped configs' losses at k = 4."""
    gold, inp, cfg, oc, op_ = case
    dev = torch.device('cuda:0')
    if losses == 'ce_mse':
        head, ocfg = build(inp), cfg
    else:
        head = build(inp, loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                     loss_reg=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5))
        ocfg = dict(cfg, loss_cls='FocalLoss', loss_reg='SmoothL1Loss', loss_reg_weight=0.5)
    co, po = oc.to(dev).requires_grad_(True), op_.to(dev).requires_grad_(True)
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    got = head.loss([co], [po], gtb, gtl, inp['img_metas'])
    (sum(got['loss_cls']) + sum(got['loss_pts'])).backward()
    co_o, po_o = oc.clone().requires_grad_(True), op_.clone().requires_grad_(True)
    ol, oall = odef.p2p_loss(co_o, po_o, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], ocfg, return_all=True)
    (sum(ol['loss_cls']) + sum(ol['loss_pts'])).backward()
    gi = head._last_assign['gt_inds'].cpu()
    assert torch.equal(gi, torch.stack([t[4] for t in oall['targets']])), 'assignments vs scipy'
    assert np.array_equal(gi.numpy().astype(np.int32), gold['gt_inds']), 'assignments vs golden'
    for b in range(inp['cfgd']['B']):
        assert torch.equal(head._last_targets['labels'][b].cpu(), oall['targets'][b][0]), 'assigned labels'
        assert torch.equal(head._last_targets['pts_weights'][b].cpu(), oall['targets'][b][3])
    for k in ('loss_cls', 'loss_pts'):
        assert_close(torch.stack(got[k]), torch.stack(ol[k]).detach(), 1e-4, f'{losses} {k}')
        if losses == 'ce_mse':
            assert_close(torch.stack(got[k]), torch.from_numpy(gold[k]), 1e-4, f'{k} vs golden')
    assert_close(co.grad, co_o.grad, 2e-4, f'{losses} d/d cls_out')
    assert_close(po.grad, po_o.grad, 2e-4, f'{losses} d/d pts_out')
    if losses == 'ce_mse':
        assert_close(co.grad.flatten()[::37], torch.from_numpy(gold['grad_cls_sub']), 2e-4, 'd/d cls_out vs golden')
        assert_close(po.grad.flatten(), torch.from_numpy(gold['grad_pts_sub']), 2e-4, 'd/d pts_out vs golden')


def test_loss_kernels_match_torch_on_random_rows(ops):
    """ptb_sigmoid_bce_fwd_bwd / ptb_mse_fwd_bwd alone: background and out-of-range labels are all-zero rows, zero weights drop rows,
    the sums are deterministic (two runs give the same bits)."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(3)
    M, C = 5003, 80
    x = torch.randn(M, C, generator=g) * 4
    lab = torch.randint(0, C + 1, (M,), generator=g)
    lab[:7] = -1
    w = (torch.rand(M, generator=g) > 0.2).float() * torch.rand(M, generator=g)
    t = torch.zeros(M, C)
    ok = (lab >= 0) & (lab < C)
    t[ok.nonzero().squeeze(1), lab[ok]] = 1
    xr = x.clone().requires_grad_(True)
    ref = (F.binary_cross_entropy_with_logits(xr, t, reduction='none') * w[:, None]).sum()
    ref.backward()
    xd, ld, wd = x.to(dev), lab.to(dev), w.to(dev)
    l1 = ops.sigmoid_bce(xd, ld, wd)
    assert torch.equal(l1, ops.sigmoid_bce(xd, ld, wd))
    assert_close(l1, ref.detach().reshape(1), 1e-5, 'bce sum')
    gr = ops.sigmoid_bce(xd, ld, wd, scale=torch.tensor([0.5], device=dev), want_grad=True)
    assert_close(gr, 0.5 * xr.grad, 1e-5, 'bce grad')
    p = torch.randn(M, 2, generator=g) * 30
    q = torch.randn(M, 2, generator=g) * 30
    pw = (torch.rand(M, 2, generator=g) > 0.5).float()
    pr = p.clone().requires_grad_(True)
    ref = (F.mse_loss(pr / 8 / 0.5, q / 8 / 0.5, reduction='none') * pw).sum()
    ref.backward()
    l2 = ops.mse(p.to(dev), q.to(dev), pw.to(dev), 1.0 / 4)
    assert_close(l2, ref.detach().reshape(1), 1e-5, 'mse sum')
    gr = ops.mse(p.to(dev), q.to(dev), pw.to(dev), 1.0 / 4, scale=torch.tensor([2.0], device=dev), want_grad=True)
    assert_close(gr, 2.0 * pr.grad, 1e-5, 'mse grad')
