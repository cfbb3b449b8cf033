"""GPU: CPRHead above 256 classes.

  * kernels: ptb_mil_loss_fwd / _bwd (class chunks of 256 lanes) and ptb_cpr_allpos_fwd against float64 (tests/mil_chunk_ref.py) on both
    sides of every chunk boundary up to the 1280-class limit, both loss kinds, bags of 1, 33 and 289 samples and a zero-weight bag;
    bag_acc with a planted tie across a chunk boundary;
  * ptb_cpr_neg_mask in class chunks (above 736 classes) bit-exact against the oracle (torch.cdist on the host);
  * the logit-map GEMMs at LD = 256 .. 2416 on the tensor cores against fp64: the column-sliced forward (ops.conv_tc_f16), dW in
    column slices (ops.conv_tc_wgrad_f16) and dX; the head's tensor-core backward against the FFMA kernels;
  * the head at 365 and 1203 classes against the golden vectors of the reference (oracle/make_golden_cpr_many_classes.py), refine through
    the margin harness, simple_test's sliced inference map, and the refusal above 1280 classes.
Tolerances as in tests/test_gpu_cpr_loss_types.py (kernels) and tests/test_gpu_cpr_loss_types.py::test_head_against_oracle_and_golden
(head: 1e-4 on losses, 2e-4 on gradients)."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr as ocpr
from oracle.make_golden import ref_cpr_cfg
from oracle.make_golden_cpr_many_classes import CLASS_COUNTS, many_class_inputs, oracle_cfg
from tests.helpers import assert_close, check_refine_against_oracle, scale_rel_err
from tests.mil_chunk_ref import allpos_ref64, mil_ref64

pytestmark = pytest.mark.gpu

EPS = 1e-6
TOP1_BOUND = 1e-5
N_LIST = [255, 256, 257, 365, 512, 513, 1024, 1203, 1280]


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops as _ops
    return _ops


def _bags(N, K, seed, G=6):
    """bag logits (G,K,LD), LD = 2 ceil8(N), pad columns 50; bag 0 has no valid sample, the others about 70 % and their last one."""
    g = torch.Generator().manual_seed(seed)
    NP = (N + 7) // 8 * 8
    bl = torch.full((G, K, 2 * NP), 50.0)
    bl[..., :N] = torch.randn(G, K, N, generator=g) * 2.0 - 1.0
    bl[..., NP:NP + N] = torch.randn(G, K, N, generator=g) * 2.0
    weight = (torch.rand(G, K, generator=g) < 0.7).float()
    weight[0] = 0.0
    weight[1:, -1] = 1.0
    labels = torch.randint(0, N, (G,), generator=g, dtype=torch.int32)
    return bl, NP, weight, labels


def _hits_ok(got, ref, margin):
    close = int((margin <= TOP1_BOUND).sum())
    lo = ref - close
    return lo <= got <= ref + close


@pytest.mark.parametrize('kind', [0, 1])
@pytest.mark.parametrize('K', [1, 33, 289])
@pytest.mark.parametrize('N', N_LIST)
def test_mil_kernels_against_float64(ops, N, K, kind):
    bl, NP, weight, labels = _bags(N, K, 31 * N + K + kind)
    ref = mil_ref64(bl, N, NP, weight, labels, EPS, kind)
    d_bl, d_w, d_l = bl.cuda(), weight.cuda(), labels.cuda()
    bp, s, stats, mt, lw = ops.mil_loss_fwd(d_bl, N, NP, d_w, d_l, EPS, want_aux=True, loss_kind=kind)
    what = f'N={N} K={K} kind={kind}'
    assert abs(float(s[0]) - ref['sum']) <= 2e-5 * max(1.0, abs(ref['sum'])), (what, float(s[0]), ref['sum'])
    assert float(stats[0]) == ref['count'], what
    ref_hits = ref['hits']
    assert _hits_ok(float(stats[1]), ref_hits, ref['margin']), (what, float(stats[1]), ref_hits)
    assert scale_rel_err(bp, ref['prob']) <= 1e-5, what
    assert torch.equal(lw.cpu(), (weight.sum(1) > 0).float()), what
    scale = torch.ones(1, device='cuda')
    grad = ops.mil_loss_bwd(d_bl, N, NP, d_w, d_l, EPS, bp, scale, loss_kind=kind)
    g = grad.cpu().double()
    assert torch.isfinite(g).all(), what
    pad = torch.ones(2 * NP, dtype=torch.bool)
    pad[:N] = False
    pad[NP:NP + N] = False
    assert not g[..., pad].any(), f'{what}: gradient in the pad columns'
    assert not g[0].any(), f'{what}: the zero-weight bag has a gradient'
    err = float((g - ref['grad']).abs().max())
    bound = 2e-5 * max(1e-3, float(ref['grad'].abs().max()))
    assert err <= bound, f'{what}: max |grad - ref| {err:.3e} > {bound:.3e}'


@pytest.mark.parametrize('kind', [0, 1])
@pytest.mark.parametrize('K', [1, 33, 289])
@pytest.mark.parametrize('N', N_LIST)
def test_allpos_kernel_against_float64(ops, N, K, kind):
    bl, NP, weight, labels = _bags(N, K, 37 * N + K + kind)
    ref = allpos_ref64(bl, N, weight, labels, EPS, kind)
    s, stats = ops.allpos_fwd(bl.cuda(), N, weight.cuda(), labels.cuda(), EPS, kind)
    what = f'N={N} K={K} kind={kind}'
    assert abs(float(s[0]) - ref['sum']) <= 2e-5 * max(1.0, abs(ref['sum'])), (what, float(s[0]), ref['sum'])
    assert float(stats[0]) == ref['count'], what
    assert _hits_ok(float(stats[1]), ref['hits'], ref['margin']), (what, float(stats[1]), ref['hits'])


@pytest.mark.parametrize('N,c', [(300, 255), (700, 511), (1280, 1023)])
def test_bag_acc_tie_across_a_chunk_boundary(ops, N, c):
    """classes c and c + 1 sit in adjacent chunks with identical logits and the largest bag probability: the first maximum (c) is the
    top-1 class, exactly, for MIL; and for AllPos on every sample."""
    bl, NP, weight, labels = _bags(N, 9, N, G=2)
    weight[:] = 1.0                                         # both bags count (a zero-weight bag's top-1 class is 0)
    for cc in (c, c + 1):
        bl[..., cc] = 12.0                                  # above every random logit of every sample (AllPos ranks samples)
        bl[..., NP + cc] = 0.5
    for lab, hit in ((c, True), (c + 1, False)):
        labels[:] = lab
        _, _, stats = ops.mil_loss_fwd(bl.cuda(), N, NP, weight.cuda(), labels.cuda(), EPS)
        assert float(stats[1]) == (2.0 if hit else 0.0), (N, lab, float(stats[1]))
        _, st = ops.allpos_fwd(bl.cuda(), N, weight.cuda(), labels.cuda(), EPS, 0)
        assert float(st[1]) == (18.0 if hit else 0.0), (N, lab, float(st[1]))


@pytest.mark.parametrize('class_wise', [True, False])
@pytest.mark.parametrize('N', [736, 737, 1203])
def test_neg_mask_class_chunks_bit_exact(ops, N, class_wise):
    g = torch.Generator().manual_seed(N + class_wise)
    B, H, W, stride, radius = 2, 20, 24, 8.0, 3
    pad_hw = torch.tensor([[H * 8, W * 8 - 6], [H * 8 - 11, W * 8]], dtype=torch.int32)
    lens = [31, 12]
    centers = torch.rand(sum(lens), 2, generator=g) * torch.tensor([W * stride, H * stride])
    labels = torch.randint(0, N, (sum(lens),), generator=g, dtype=torch.int32)
    chunks = (N + 735) // 736
    cc = (N + chunks - 1) // chunks                         # the launcher's balanced chunk width: classes cc - 1 and cc straddle a boundary
    labels[:6] = torch.tensor([0, N - 1, cc - 1, cc, cc - 1, N - 1], dtype=torch.int32) % N
    img_ptr = torch.tensor([0, lens[0], sum(lens)], dtype=torch.int32)
    got = ops.neg_mask(B, H, W, stride, pad_hw.cuda(), centers.cuda(), labels.cuda(), img_ptr.cuda(), stride * radius, N, class_wise).cpu()
    for b in range(B):
        pts, valid = ocpr.anchor_points(H, W, int(pad_hw[b, 0]), int(pad_hw[b, 1]), stride)
        sel = slice(int(img_ptr[b]), int(img_ptr[b + 1]))
        ref = ocpr.out_circle_neg_mask(pts.reshape(-1, 2).float(), valid.reshape(-1), centers[sel][:, None, :], labels[sel].long(), stride,
                                       radius, N, class_wise)
        assert torch.equal(got[b].reshape(-1, N), ref), f'N={N} class_wise={class_wise} image {b}: {int((got[b].reshape(-1, N) != ref).sum())} flags differ'


@pytest.mark.parametrize('LD', [256, 264, 520, 2416])
def test_logit_map_gemms_in_column_slices(ops, LD):
    """the logit map's three GEMMs on the tensor cores against fp64: the forward as column slices of the wgmma conv (1e-4), dW as column
    slices of <= 256 of the gradient's fp16 pair read in place (2e-4), and dX as one conv with Cin = LD (2e-4) at the width the head
    gives it (loss_bwd_plan pads LD to a multiple of 32 above 256 classes: 264 -> 288, 520 -> 544, 2416 -> 2432)."""
    g = torch.Generator().manual_seed(LD)
    B, H, W, C = 2, 12, 20, 256
    x = torch.relu(torch.randn(B, H, W, C, generator=g))
    w = torch.randn(LD, C, generator=g) * 0.05
    bias = torch.randn(LD, generator=g) * 0.1
    dx, dw_, db_ = x.cuda(), w.cuda(), bias.cuda()
    fh, fl, finv = ops.split_f16(dx, auto_scale=True)
    y = ops.conv_tc_f16(fh, fl, ops.conv_tc_pack_weight_f16(dw_, 1), 1, LD, bias=db_, dev_out_scale=finv, ldy=LD)
    ref = x.reshape(-1, C).double() @ w.double().t() + bias.double()
    assert_close(y.reshape(-1, LD), ref, 1e-4, f'LD={LD} sliced map')
    dy = torch.randn(B, H, W, LD, generator=g)
    dh, dl, dinv = ops.split_f16(dy.cuda(), auto_scale=True)
    gw = ops.conv_tc_wgrad_f16(dh, dl, fh, fl, 1, 1.0, dinv, finv)
    assert_close(gw, dy.reshape(-1, LD).double().t() @ x.reshape(-1, C).double(), 2e-4, f'LD={LD} dW')
    LDx = (LD + 31) // 32 * 32
    dyx = torch.zeros(B, H, W, LDx)
    dyx[..., :LD] = dy
    wx = torch.zeros(LDx, C)
    wx[:LD] = w
    xh, xl, xinv = ops.split_f16(dyx.cuda(), auto_scale=True)
    gx = ops.conv_tc_f16(xh, xl, ops.conv_tc_pack_weight_f16(wx.cuda().t().contiguous(), 1), 1, C, dev_out_scale=xinv, ldy=C)
    assert_close(gx.reshape(-1, C), dyx.reshape(-1, LDx).double() @ wx.double(), 2e-4, f'LD={LDx} dX')


@pytest.mark.parametrize('N', [365, 1203])
def test_head_backward_gemms_on_tensor_cores(ops, monkeypatch, N):
    """CPRHead.loss + backward at 256 feature channels: the tensor-core logit-map GEMMs (forward slices, sliced dW, dX conv) against the
    fp32 FFMA kernels (the shape predicate forced off) on the same inputs: losses 1e-4, gradients 2e-4."""
    from oracle import synth
    from pointtinybenchmark_b200 import cpr_head
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 7000 + N, num_classes=N, n=16)
    head = _head(N, 256, dev, inp['weights'])
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    runs = {}
    for mode in ('tc', 'ffma'):
        if mode == 'ffma':
            monkeypatch.setattr(cpr_head, '_loss_map_on_tc', lambda *a: False)
        head.zero_grad(set_to_none=True)
        feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
        sum(v for k, v in losses.items() if 'loss' in k).backward()
        runs[mode] = (losses, [feat.grad.clone(), head.cls_out.weight.grad.clone(), head.cls_out.bias.grad.clone(),
                               head.ins_out.weight.grad.clone()])
    (lt, gt_), (lf, gf) = runs['tc'], runs['ffma']
    for k in ('gt_loss', 'pos_loss', 'neg_loss'):
        assert_close(lt[k].reshape(-1), lf[k].reshape(-1), 1e-4, f'N={N} {k}')
    for name, a, b in zip(('dfeat', 'dWcls', 'dbcls', 'dWins'), gt_, gf):
        assert_close(a, b, 2e-4, f'N={N} {name}')


def _head(N, C, dev, weights, **over):
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    d = dict(num_classes=N, C=C, stride=8, radius=5)
    cfg = ref_cpr_cfg(d)
    cfg['test_cfg'] = dict(cfg['test_cfg'])
    cfg.update(over)
    head = build_head(cfg).to(dev)
    sd = head.state_dict()
    sd.update({k: v.to(dev) for k, v in weights.items()})
    head.load_state_dict(sd, strict=True)
    return head


def _cat_refine(allo):
    ora = {k: torch.cat([r[k] for r in allo['refine']]) for k in allo['refine'][0]}
    ora['mask_valid'] = allo['ex']['pos_valid'][:, 0, :, 0]
    return ora


@pytest.mark.parametrize('mode', [None, 'staged'])
@pytest.mark.parametrize('N', CLASS_COUNTS)
def test_head_against_reference_golden(ops, golden_dir, N, mode):
    dev = torch.device('cuda:0')
    gold = np.load(os.path.join(golden_dir, f'cpr_many_classes_{N}.npz'))
    inp = many_class_inputs(N, int(gold['seed']))
    d = inp['cfgd']
    head = _head(N, d['C'], dev, inp['weights'])
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    os.environ.pop('PTB_LOSS_BWD', None)
    if mode:
        os.environ['PTB_LOSS_BWD'] = mode
    try:
        feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'])
        sum(v for k, v in losses.items() if 'loss' in k).backward()
    finally:
        os.environ.pop('PTB_LOSS_BWD', None)
    what = f'N={N} mode={mode}'
    for k in ('gt_loss', 'pos_loss', 'neg_loss'):
        assert_close(losses[k].reshape(-1), torch.from_numpy(gold['loss_' + k]), 1e-4, f'{what} {k}')
    assert float(losses['bag_acc'].reshape(-1)[0]) == pytest.approx(float(gold['loss_bag_acc'][0]), abs=1e-4), what
    sub = feat.grad.detach().cpu().contiguous().flatten()[::211].numpy()
    assert np.abs(sub - gold['grad_feat_sub']).max() <= 2e-4 * np.abs(gold['grad_feat_sub']).max(), what
    # ins_out.bias is not compared: the bag softmax is invariant to a per-class shift, so its gradient is zero up to rounding on both sides
    for p, key in ((head.cls_out.weight, 'grad_cls_w'), (head.cls_out.bias, 'grad_cls_b'), (head.ins_out.weight, 'grad_ins_w')):
        assert_close(p.grad, torch.from_numpy(gold[key]), 2e-4, f'{what} {key}')
    assert float(head.ins_out.bias.grad.abs().max()) <= 1e-4 * float(np.abs(gold['grad_ins_w']).max()), what
    # refine: the fused kernel against the oracle's reference data flow through the margin harness, then the golden detections
    from pointtinybenchmark_b200.cpr_head import _BatchGT
    aid = [a.to(dev) for a in inp['gt_anns_id']]
    with torch.no_grad():
        gt = _BatchGT(gtb, gtl, inp['img_metas'], dev)
        got = head.refine_points(inp['cls_feat'].to(dev), gt, want_chosen=True)
        res = head.get_bboxes([inp['cls_feat'].to(dev)], [inp['cls_feat'].to(dev)], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl,
                              gt_anns_id=aid)
        _, allo = ocpr.cpr_get_bboxes(inp['cls_feat'], inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'],
                                      inp['img_metas'], oracle_cfg(d), return_all=True)
    ora = _cat_refine(allo)
    assert torch.equal(ora['chosen'].bool(), torch.from_numpy(gold['chosen']).bool())
    check_refine_against_oracle(got, ora, allo['bag_prob'][:, 0], torch.cat(inp['gt_labels']), oracle_cfg(d), 1e-5, what)
    flips = (got[3].cpu().bool() != ora['chosen'].bool()).any(dim=1) | (got[2].cpu().bool() != torch.from_numpy(gold['not_refine']).bool())
    det = torch.cat([r[0] for r in res]).cpu()
    assert_close(det[~flips][:, :5], torch.from_numpy(gold['det'])[~flips][:, :5], 1e-4, f'{what} det rows vs golden')
    assert torch.equal(det[:, 5], torch.from_numpy(gold['det'])[:, 5])


@pytest.mark.parametrize('N', [600, 1203])
def test_simple_test_logit_map_in_column_slices(ops, monkeypatch, N):
    """simple_test above 512 classes: the class-logit map from column slices of the wgmma kernel on the towers' fp16 pair, refined; its
    probabilities against the oracle on the head's own fp32 tower output through the margin harness (bound 1e-4: fp16-split map)."""
    from oracle import synth
    from pointtinybenchmark_b200.cpr_head import _BatchGT
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 5000 + N, num_classes=N, n=16, with_towers=True, trained_like=False)
    d = inp['cfgd']
    head = _head(N, 256, dev, inp['weights']).eval()
    gtb = [b.to(dev) for b in inp['gt_bboxes']]
    gtl = [l.to(dev) for l in inp['gt_labels']]
    x = torch.randn(1, 256, 32, 32, generator=torch.Generator().manual_seed(N)).to(dev)
    calls = []
    conv = ops.conv_tc_f16
    monkeypatch.setattr(ops, 'conv_tc_f16', lambda *a, **k: calls.append((a[4], len(a[2]))) or conv(*a, **k))
    with torch.no_grad():
        res = head.simple_test((x,), inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl)
        feat = head.forward((x,))[0][0]
        ref_res = head.get_bboxes([feat], [feat], inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl)
        w = {k: v.detach().cpu() for k, v in head.state_dict().items()}
        _, allo = ocpr.cpr_get_bboxes(feat.cpu(), w, inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'], inp['img_metas'],
                                      oracle_cfg(d), return_all=True)
        gt = _BatchGT(gtb, gtl, inp['img_metas'], dev)
        got = head.refine_points(feat, gt, want_chosen=True)
    assert calls == [(N, (N + 511) // 512)], f'simple_test did not take the sliced tensor-core map: {calls}'
    check_refine_against_oracle(got, _cat_refine(allo), allo['bag_prob'][:, 0], torch.cat(inp['gt_labels']), oracle_cfg(d), 1e-4,
                                f'N={N} get_bboxes')
    det, det_ref = res[0][0].cpu(), ref_res[0][0].cpu()
    assert det.shape == det_ref.shape and torch.equal(det[:, 5], det_ref[:, 5])
    same = (det[:, :5] - det_ref[:, :5]).abs().amax(dim=1) <= 1e-3
    assert float(same.float().mean()) >= 0.9, f'N={N}: only {int(same.sum())} / {len(same)} rows of simple_test match get_bboxes'
    assert_close(det[same][:, :5], det_ref[same][:, :5], 1e-4, f'N={N} simple_test vs get_bboxes')


def test_more_than_1280_classes_is_refused(ops):
    dev = torch.device('cuda:0')
    N = 1281
    inp = many_class_inputs(365)
    from oracle import synth
    w = synth.cpr_weights(32, N, torch.Generator().manual_seed(0), with_towers=False)
    head = _head(N, 32, dev, w)
    feat = inp['cls_feat'].to(dev)
    with pytest.raises(RuntimeError, match='num_classes=1281 exceeds the 1280 classes'):
        head.loss([feat], [feat], [b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']], inp['img_metas'])
    bl, NP, weight, labels = _bags(N, 9, 1)
    with pytest.raises(RuntimeError, match='num_classes > 1280'):
        ops.mil_loss_fwd(bl.cuda(), N, NP, weight.cuda(), labels.cuda(), EPS)
