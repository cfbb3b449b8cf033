"""GPU: P2PHead with CrossEntropyLoss in softmax mode (C+1 outputs per anchor, background last) and with class_weight — the softmax
decode / top-k, the softmax cross-entropy and the pos_weight BCE kernels on their own against float64 torch, and the head against the
CPU oracle and the golden vectors of the real reference head (tests/golden/p2p_softmax_lite.npz).

The CUDA softmax is within a few ulps of ATen's CPU softmax, not bit-identical to it.  Decisions that follow softmax values are
therefore compared with a margin: float64 keys within a relative bound of each other form a tie group, inside which the order is
free, and the selected set must equal the reference's outside the group at the k-th boundary.  On the golden case, which its
generator asserts free of near-ties, top-k and NMS keep are compared bit for bit."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_softmax as osm
from tests.helpers import assert_close
from tests.test_gpu_p2p_defaults import TRAIN_CFG

pytestmark = pytest.mark.gpu

TIE_REL = 1e-6      # the fp32 keys are within ~3e-7 relative of float64; two keys further apart than this are ordered exactly


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def check_topk_tie_groups(got, keys64, P, what, rel=TIE_REL):
    """got (P,) selected indices in selection order, keys64 (Q,) float64 keys.  Asserts the tie-group rule and returns the number of
    tie groups (more than one member) among the selected."""
    got = np.asarray(got, np.int64)
    order = np.argsort(-keys64, kind='stable')
    sk = keys64[order]
    gid = np.concatenate([[0], np.cumsum(sk[:-1] - sk[1:] > rel * np.abs(sk[:-1]))])
    group = np.empty(len(order), np.int64)
    group[order] = gid
    assert len(np.unique(got)) == P == len(got), what
    kth = gid[P - 1]
    must = {int(q) for q in order[:P] if group[q] != kth}
    assert must <= set(got.tolist()), f'{what}: selected set differs outside the boundary tie group'
    assert (group[got] <= kth).all(), f'{what}: a proposal below the boundary tie group was selected'
    assert (np.diff(group[got]) >= 0).all(), f'{what}: order differs outside a tie group'
    sizes = np.bincount(gid[:P])
    n = int((sizes > 1).sum())
    print(f'[{what}] {n} tie groups of > 1 member among the top {P}')
    return n


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C1', [2, 81, 129])
@pytest.mark.parametrize('with_cw', [False, True])
def test_softmax_ce_matches_float64(ops, C1, with_cw):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(C1 * 2 + with_cw)
    M = 5003
    x = torch.randn(M, C1, generator=g) * 4
    lab = torch.randint(0, C1, (M,), generator=g)
    lab[::5] = C1 - 1                                                     # background label
    w = (torch.rand(M, generator=g) > 0.2).float() * torch.rand(M, generator=g) * 2      # zero and fractional weights
    cw = (torch.rand(C1, generator=g) * 2 + 0.1) if with_cw else None
    xr = x.double().requires_grad_(True)
    ref = (F.cross_entropy(xr, lab, weight=None if cw is None else cw.double(), reduction='none') * w.double()).sum()
    ref.backward()
    xd, ld, wd = x.to(dev), lab.to(dev), w.to(dev)
    cwd = None if cw is None else cw.to(dev)
    l1 = ops.softmax_ce(xd, ld, wd, cwd)
    assert torch.equal(l1, ops.softmax_ce(xd, ld, wd, cwd)), 'two calls give identical bits'
    assert_close(l1, ref.detach().reshape(1), 1e-5, f'softmax ce sum C1={C1}')
    sc = torch.tensor([0.25], device=dev)
    gr = ops.softmax_ce(xd, ld, wd, cwd, scale=sc, want_grad=True)
    assert torch.equal(gr, ops.softmax_ce(xd, ld, wd, cwd, scale=sc, want_grad=True))
    assert_close(gr, 0.25 * xr.grad, 1e-5, f'softmax ce grad C1={C1}')
    assert not bool(gr.cpu()[w == 0].any()), 'zero-weight rows have zero gradient'


def test_softmax_ce_out_of_range_label_gives_a_nan_row(ops):
    dev = torch.device('cuda:0')
    x = torch.randn(64, 21, device=dev)
    lab = torch.randint(0, 21, (64,), device=dev)
    lab[3] = 21
    gr = ops.softmax_ce(x, lab, None, scale=torch.ones(1, device=dev), want_grad=True)
    assert torch.isnan(ops.softmax_ce(x, lab, None)).all()
    assert torch.isnan(gr[3]).all() and torch.isfinite(torch.cat([gr[:3], gr[4:]])).all()


@pytest.mark.parametrize('C', [1, 80, 129])
def test_sigmoid_bce_pos_weight_matches_float64(ops, C):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(100 + C)
    M = 5003
    x = torch.randn(M, C, generator=g) * 4
    lab = torch.randint(0, C + 1, (M,), generator=g)                      # C = background: all-zero row
    w = (torch.rand(M, generator=g) > 0.2).float() * torch.rand(M, generator=g)
    pw = torch.rand(C, generator=g) * 3 + 0.1
    t = torch.zeros(M, C, dtype=torch.float64)
    ok = lab < C
    t[ok.nonzero().squeeze(1), lab[ok]] = 1
    xr = x.double().requires_grad_(True)
    ref = (F.binary_cross_entropy_with_logits(xr, t, pos_weight=pw.double(), reduction='none') * w.double()[:, None]).sum()
    ref.backward()
    xd, ld, wd, pwd = x.to(dev), lab.to(dev), w.to(dev), pw.to(dev)
    l1 = ops.sigmoid_bce(xd, ld, wd, pos_weight=pwd)
    assert torch.equal(l1, ops.sigmoid_bce(xd, ld, wd, pos_weight=pwd))
    assert_close(l1, ref.detach().reshape(1), 1e-5, 'bce pos_weight sum')
    sc = torch.tensor([0.5], device=dev)
    gr = ops.sigmoid_bce(xd, ld, wd, scale=sc, want_grad=True, pos_weight=pwd)
    assert torch.equal(gr, ops.sigmoid_bce(xd, ld, wd, scale=sc, want_grad=True, pos_weight=pwd))
    assert_close(gr, 0.5 * xr.grad, 1e-5, 'bce pos_weight grad')
    # pos_weight NULL through the class-weighted entry point: the bits of ptb_sigmoid_bce_fwd_bwd
    from pointtinybenchmark_b200 import _lib
    from pointtinybenchmark_b200.ops import _ptr, _stream
    lib = _lib.load()
    for want_grad in (False, True):
        outs = []
        for call in (lambda *out: lib.ptb_sigmoid_bce_cw_fwd_bwd(_ptr(xd), _ptr(ld), _ptr(wd), None, M, C, *out),
                     lambda *out: lib.ptb_sigmoid_bce_fwd_bwd(_ptr(xd), _ptr(ld), _ptr(wd), M, C, *out)):
            out = torch.zeros(1, device=dev) if not want_grad else torch.empty_like(xd)
            lsum, grad = (None, out) if want_grad else (out, None)
            rc = call(_ptr(lsum), _ptr(sc), _ptr(grad), _stream())
            assert rc == 0, lib.ptb_last_error()
            outs.append(out)
        assert torch.equal(*outs), 'NULL pos_weight = class_weight None'


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C1', [2, 21, 81])
@pytest.mark.parametrize('k', [1, 4])
@pytest.mark.parametrize('nms_pre', [-1, 100, 1000, 5000])
def test_softmax_decode_on_random_maps(ops, C1, k, nms_pre):
    from pointtinybenchmark_b200 import _lib
    from pointtinybenchmark_b200.ops import _ptr, _stream
    lib = _lib.load()
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(C1 * 10 + k + max(nms_pre, 0))
    B, H, W, C = 3, 13, 21, C1 - 1
    Q = H * W * k
    cmap = (torch.randn(B, H, W, k * C1, generator=g) * 3).to(dev)
    rmap = torch.randn(B, H, W, 2 * k, generator=g).to(dev)
    anchor = torch.tensor([(-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)][:k], device=dev)
    img_hw = torch.tensor([[100, 160], [80, 120], [100, 160]], dtype=torch.int32, device=dev)   # image 1: smaller pad / image
    P = nms_pre if 0 < nms_pre < Q else Q
    idx = torch.empty((B, P), dtype=torch.int32, device=dev)
    pts = torch.empty((B, P, 2), device=dev)
    scores = torch.empty((B, P, C), device=dev)
    nbytes = lib.ptb_p2p_decode_topk_workspace(B, H, W, k)
    ws = torch.zeros(nbytes // 4 + 1, device=dev)
    rc = lib.ptb_p2p_decode_topk_softmax(_ptr(cmap), _ptr(rmap), B, H, W, C, k, _ptr(anchor), 8.0, 12.5, _ptr(img_hw), None,
                                         nms_pre, _ptr(idx), _ptr(pts), _ptr(scores), _ptr(ws), nbytes, _stream())
    assert rc == 0, lib.ptb_last_error()
    i2, p2, s2 = ops.p2p_decode_topk_softmax(cmap.contiguous(), rmap, C, k, anchor, 8.0, 12.5, img_hw, nms_pre)
    assert torch.equal(i2, idx) and torch.equal(p2, pts) and torch.equal(s2, scores), 'the ops wrapper and the ABI agree'
    rows = cmap.reshape(B, Q, C1).double().cpu()
    prob64 = rows.softmax(-1)
    keys64 = prob64[..., :C].max(-1)[0].numpy()
    idx_h = idx.long().cpu()
    sel = torch.stack([prob64[b, idx_h[b], :C] for b in range(B)])
    assert_close(scores, sel, 1e-6, f'probabilities C1={C1} k={k}')
    if P < Q:
        key = ws[:B * Q].reshape(B, Q).cpu()
        assert torch.equal(scores.max(-1)[0].cpu(), torch.stack([key[b, idx_h[b]] for b in range(B)])), 'key = row max, bit for bit'
        for b in range(B):
            check_topk_tie_groups(idx_h[b].numpy(), keys64[b], P, f'top-k C1={C1} k={k} nms_pre={nms_pre} image {b}')
    else:
        assert torch.equal(idx_h, torch.arange(Q).expand(B, Q)), 'identity path keeps every proposal in index order'
    # the points are those of the sigmoid decode for the same indices (its identity path decodes every proposal)
    _, pall, _ = ops.p2p_decode_topk(cmap, rmap, C1, k, anchor, 8.0, 12.5, img_hw, -1)
    assert torch.equal(pts, torch.stack([pall[b, idx[b].long()] for b in range(B)]))


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def case(ops, golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_softmax_lite.npz'))
    inp = osm.inputs(int(gold['seed']))
    d = inp['cfgd']
    cfg = osm.softmax_cfg(use_sigmoid=False, class_weight=gold['class_weight_softmax'].tolist(), num_classes=d['num_classes'],
                          stride=d['stride'], nms_iou=0.5, nms_pre=int(gold['nms_pre']))
    with torch.no_grad():
        oc, op_ = op2p.head_forward(inp['x'], inp['weights'], cfg)
    return gold, inp, cfg, oc, op_


def build(inp, cfg, **over):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    d = inp['cfgd']
    test_cfg = dict(nms_pre=cfg['nms_pre'], min_bbox_size=0, score_thr=cfg['score_thr'], pseudo_wh=cfg['pseudo_wh'],
                    nms=dict(type='nms', iou_threshold=cfg['nms_iou']), max_per_img=cfg['max_per_img'])
    hc = dict(type='P2PHead', num_classes=d['num_classes'], in_channels=d['C'], feat_channels=d['C'], stacked_convs=4,
              strides=[d['stride']], point_anchor=d['point_anchor'], norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
              loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=cfg['use_sigmoid'], class_weight=cfg['class_weight'], loss_weight=1.0),
              train_cfg=TRAIN_CFG, test_cfg=test_cfg)
    hc.update(over)
    head = build_head(hc)
    if 'weights' in inp:
        head.load_state_dict(inp['weights'], strict=True)
    return head.cuda()


def check_nms_on_gpu_scores(aux, res, metas, cfg, what):
    """the GPU's NMS over its own top-k points / scores equals the oracle's multiclass_nms over the same fp32 values."""
    for b in range(len(metas)):
        pts, sc = aux['pts'][b].cpu(), aux['scores'][b].cpu()
        wh = pts.new_tensor(cfg['pseudo_wh'])
        boxes = torch.cat([pts - wh / 2, pts + wh / 2], -1)
        dets, labels, keep, inds = op2p.multiclass_nms(boxes, torch.cat([sc, sc.new_zeros(len(sc), 1)], 1), cfg['score_thr'],
                                                       cfg['nms_iou'], cfg['max_per_img'])
        n = int(aux['count'][b])
        assert int(aux['cand_count'][b]) == len(inds) and n == len(keep), what
        assert torch.equal(aux['keep'][b, :n].cpu().long(), keep), f'{what}: NMS keep, image {b}'
        assert torch.equal(res[b][1].cpu(), labels), f'{what}: labels, image {b}'
        assert_close(res[b][0][:, 4], dets[:, 4], 1e-6, f'{what}: scores, image {b}')


def test_simple_test_softmax_at_four_anchors(ops, case):
    gold, inp, cfg, oc, op_ = case
    dev = torch.device('cuda:0')
    head = build(inp, cfg).eval()
    assert head.num_cls_out == 81 and head.cls_out.out_channels == 324
    x = inp['x'].to(dev)
    metas = inp['img_metas']
    C = inp['cfgd']['num_classes']
    with torch.no_grad():
        cls_outs, pts_outs = head.forward((x,))
        res, aux = head.get_bboxes(cls_outs, pts_outs, metas, return_all=True)
        res2 = head.simple_test((x,), metas)
    assert head.last_tower_backend == 'wgmma-f16x2', 'towers and output convs on the wgmma path'
    for a, b in zip(res, res2):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert_close(cls_outs[0], oc, 1e-4, 'cls_out (324 channels) vs oracle')
    assert_close(pts_outs[0], op_, 1e-4, 'pts_out vs oracle')
    assert_close(cls_outs[0].flatten()[::37], torch.from_numpy(gold['cls_out_sub']), 1e-4, 'cls_out vs golden')
    # the head's own maps: top-k under the tie-group rule against float64 softmax of those maps, NMS against the oracle's
    _, _, _, cls = osm.pred_points(cls_outs[0].double().cpu(), pts_outs[0].cpu(), metas, cfg)
    for b in range(len(metas)):
        check_topk_tie_groups(aux['topk_idx'][b].cpu().numpy(), cls[b].softmax(-1)[:, :C].max(-1)[0].numpy(), cfg['nms_pre'],
                              f'own maps image {b}')
    check_nms_on_gpu_scores(aux, res, metas, cfg, 'own maps')
    # the oracle's maps: top-k indices and NMS keep bit-exact against the oracle and the golden
    with torch.no_grad():
        res_o, aux_o = head.get_bboxes([oc.to(dev)], [op_.to(dev)], metas, return_all=True)
    _, pred, _, cls = osm.pred_points(oc, op_, metas, cfg)
    topks, keeps = [], []
    for b, m in enumerate(metas):
        ps, labels, al = osm.get_bboxes_single(pred[b][..., :2], cls[b], m['img_shape'], m['scale_factor'], cfg, return_all=True)
        assert torch.equal(aux_o['topk_idx'][b].cpu().long(), al['topk_inds']), f'top-k indices image {b}'
        n = int(aux_o['count'][b])
        assert int(aux_o['cand_count'][b]) == len(al['cand_inds']) == int(gold['cand_len'][b])
        assert torch.equal(aux_o['keep'][b, :n].cpu().long(), al['keep']), f'NMS keep image {b}'
        assert torch.equal(res_o[b][1].cpu(), labels)
        assert_close(aux_o['scores'][b], al['scores'], 1e-6, 'top-k probabilities vs ATen softmax')
        topks.append(aux_o['topk_idx'][b].cpu()); keeps.append(aux_o['keep'][b, :n].cpu())
    assert np.array_equal(torch.cat(topks).numpy().astype(np.int32), gold['topk']), 'top-k vs golden'
    assert np.array_equal(torch.cat(keeps).numpy().astype(np.int64), gold['keep']), 'keep vs golden'
    assert np.array_equal(torch.cat([r[1] for r in res_o]).cpu().numpy(), gold['det_labels'])
    assert_close(torch.cat([r[0] for r in res_o]), torch.from_numpy(gold['det']), 1e-4, 'det vs golden')


def test_simple_test_softmax_at_one_anchor(ops, case):
    """81-channel cls_out against the oracle: conv 1e-4, top-k under the tie-group rule, NMS on the GPU's scores exact."""
    gold, _, cfg4, _, _ = case
    inp = osm.inputs(int(gold['seed']), k=1)
    cfg = dict(cfg4, point_anchor=inp['cfgd']['point_anchor'])
    dev = torch.device('cuda:0')
    head = build(inp, cfg).eval()
    assert head.cls_out.out_channels == 81
    metas = inp['img_metas']
    with torch.no_grad():
        oc, op_ = op2p.head_forward(inp['x'], inp['weights'], cfg)
        cls_outs, pts_outs = head.forward((inp['x'].to(dev),))
        res, aux = head.get_bboxes([oc.to(dev)], [op_.to(dev)], metas, return_all=True)
    assert_close(cls_outs[0], oc, 1e-4, 'cls_out (81 channels) vs oracle')
    assert_close(pts_outs[0], op_, 1e-4, 'pts_out vs oracle')
    _, _, _, cls = osm.pred_points(oc.double(), op_, metas, cfg)
    for b in range(len(metas)):
        prob = cls[b].softmax(-1)
        check_topk_tie_groups(aux['topk_idx'][b].cpu().numpy(), prob[:, :-1].max(-1)[0].numpy(), cfg['nms_pre'], f'k=1 image {b}')
        assert_close(aux['scores'][b], prob[aux['topk_idx'][b].cpu().long(), :-1], 1e-6, 'k=1 probabilities')
    check_nms_on_gpu_scores(aux, res, metas, cfg, 'k=1')


@pytest.mark.parametrize('losses', ['softmax_mse', 'softmax_sl1', 'sigmoid_cw_mse'])
def test_loss_and_gradients(ops, case, losses):
    """P2PHead.loss + backward: Hungarian assignments bit-exact against scipy (oracle) and the golden, losses 1e-4, gradients 2e-4."""
    gold, inp, cfg, oc, op_ = case
    dev = torch.device('cuda:0')
    C = inp['cfgd']['num_classes']
    p = 'sg_' if losses.startswith('sigmoid') else 'sm_'
    if losses == 'sigmoid_cw_mse':
        cfg = dict(cfg, use_sigmoid=True, class_weight=gold['class_weight_sigmoid'].tolist())
        oc = oc.reshape(oc.shape[0], 4, C + 1, *oc.shape[2:])[:, :, :C].reshape(oc.shape[0], 4 * C, *oc.shape[2:]).contiguous()
        head = build(dict(cfgd=inp['cfgd']), cfg)
    elif losses == 'softmax_sl1':
        cfg = dict(cfg, loss_reg='SmoothL1Loss', loss_reg_weight=0.5)
        head = build(inp, cfg, loss_reg=dict(type='SmoothL1Loss', beta=cfg['sl1_beta'], loss_weight=0.5))
    else:
        head = build(inp, cfg)
    co, po = oc.to(dev).requires_grad_(True), op_.to(dev).requires_grad_(True)
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    got = head.loss([co], [po], gtb, gtl, inp['img_metas'])
    (sum(got['loss_cls']) + sum(got['loss_pts'])).backward()
    co_o, po_o = oc.clone().requires_grad_(True), op_.clone().requires_grad_(True)
    ol, oall = osm.p2p_loss(co_o, po_o, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, return_all=True)
    (sum(ol['loss_cls']) + sum(ol['loss_pts'])).backward()
    gi = head._last_assign['gt_inds'].cpu()
    assert torch.equal(gi, torch.stack([t[4] for t in oall['targets']])), 'assignments vs scipy'
    assert np.array_equal(gi.numpy().astype(np.int32), gold[p + 'gt_inds']), 'assignments vs golden'
    assert np.array_equal(torch.stack(head._last_targets['labels']).cpu().numpy(), gold[p + 'labels']), 'labels vs golden'
    for k in ('loss_cls', 'loss_pts'):
        assert_close(torch.stack(got[k]), torch.stack(ol[k]).detach(), 1e-4, f'{losses} {k}')
    assert_close(torch.stack(got['loss_cls']), torch.from_numpy(gold[p + 'loss_cls']), 1e-4, 'loss_cls vs golden')
    assert_close(co.grad, co_o.grad, 2e-4, f'{losses} d/d cls_out')
    assert_close(po.grad, po_o.grad, 2e-4, f'{losses} d/d pts_out')
    assert_close(co.grad.flatten()[::37], torch.from_numpy(gold[p + 'grad_cls_sub']), 2e-4, 'd/d cls_out vs golden')
    if losses != 'softmax_sl1':
        assert_close(torch.stack(got['loss_pts']), torch.from_numpy(gold[p + 'loss_pts']), 1e-4, 'loss_pts vs golden')
        assert_close(po.grad.flatten(), torch.from_numpy(gold[p + 'grad_pts_sub']), 2e-4, 'd/d pts_out vs golden')


def test_aug_test_bboxes_softmax_drops_the_last_class(ops, case):
    """aug_test_bboxes in softmax mode (p2p_head.py:534-556): no background column before the second NMS, so class C-1 is absent."""
    gold, inp, cfg, oc, op_ = case
    dev = torch.device('cuda:0')
    C = inp['cfgd']['num_classes']
    head = build(inp, cfg).eval()
    aug_outs, aug_metas = osm.aug_inputs(oc, op_, inp['img_metas'])
    dev_outs = [(c.to(dev).contiguous(), p.to(dev).contiguous()) for c, p in aug_outs]
    table = {id(o[0]): o for o in dev_outs}
    head.forward = lambda x: ([table[id(x)][0]], [table[id(x)][1]])
    for rescale in (False, True):
        res = head.aug_test_bboxes([o[0] for o in dev_outs], aug_metas, rescale=rescale)
        ores, _ = osm.aug_test_bboxes(aug_outs, aug_metas, cfg, rescale=rescale)
        det, lab = res[0][0].cpu(), res[0][1].cpu()
        assert not bool((lab == C - 1).any()), 'class C-1 must be absent'
        assert torch.equal(lab, ores[0][1]), 'labels after the second NMS'
        assert np.array_equal(lab.numpy(), gold[f'aug_labels_rescale{int(rescale)}'])
        assert_close(det, ores[0][0], 1e-4, f'merged detections (rescale={rescale})')
        assert_close(det, torch.from_numpy(gold[f'aug_det_rescale{int(rescale)}']), 1e-4, 'vs reference golden')
