"""GPU: MILLoss(loss_type='binary_cross_entropy') and AllPosLoss on the CPR loss kernels and through CPRHead.

  * kernels: every loss kind (MIL-BCE, AllPos-gfocal, AllPos-BCE) against the float64 reference (tests/cpr_loss_types_ref.py) at the
    class counts and bag sizes the kernels dispatch on: forward sums and counts, and d loss / d logit map on the scatter, tile and
    staged backwards;
  * head: losses and gradients against the oracle and the golden vectors recorded from the reference
    (oracle/make_golden_cpr_loss_types.py) on all three backward paths, bit-identical gradients in deterministic mode, exactly zero
    instance-classifier gradients for AllPosLoss;
  * edges: zero-weight and fully invalid bags give finite gradients, an image without GTs is handled."""
import os

import numpy as np
import pytest
import torch

from oracle import cpr_loss_types as olt
from oracle.make_golden_cpr_loss_types import LOSS_TYPE_CASES, loss_type_inputs, oracle_cfg
from tests.cpr_loss_types_ref import loss_map_ref
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

KINDS = {'mil_bce': (False, 1), 'allpos_gfocal': (True, 0), 'allpos_bce': (True, 1)}
EPS = 1e-6


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')


def _problem(N, radius, seed, NP):
    """two images of 12 x 16 cells (stride 8); bags centred inside, near the borders and one wholly outside pad_shape."""
    from pointtinybenchmark_b200 import ops
    g = torch.Generator().manual_seed(seed)
    B, H, W, stride = 2, 12, 16, 8.0
    LD = 2 * NP
    lmap = torch.zeros(B, H, W, LD)
    lmap[..., :N] = torch.randn(B, H, W, N, generator=g) * 2.0 - 1.0
    lmap[..., NP:NP + N] = torch.randn(B, H, W, N, generator=g)
    G = 7
    centers = torch.rand(G, 2, generator=g) * torch.tensor([W * stride, H * stride])
    centers[0] = torch.tensor([2.0, 3.0])                                                 # partly outside
    centers[1] = torch.tensor([W * stride + radius * stride + 20.0, 40.0])                # every sample outside pad_shape
    bag_img = torch.tensor([0, 0, 0, 1, 1, 1, 1], dtype=torch.int32)
    labels = torch.randint(0, N, (G,), generator=g, dtype=torch.int32)
    offsets = ops.circle_offsets(radius, stride)
    pad_hw = torch.tensor([[H * 8, W * 8], [H * 8 - 5, W * 8 - 9]], dtype=torch.int32)
    img_ptr = torch.tensor([0, 3, 7], dtype=torch.int32)
    return dict(lmap=lmap, centers=centers, bag_img=bag_img, labels=labels, offsets=offsets, pad_hw=pad_hw, img_ptr=img_ptr, stride=stride)


@pytest.mark.parametrize('kind', list(KINDS))
@pytest.mark.parametrize('radius', [1, 5, 8])                  # K = 9, 121, 289
@pytest.mark.parametrize('N', [1, 15, 80, 81, 128])
def test_kernels_against_float64(dev, kind, radius, N):
    from pointtinybenchmark_b200 import ops
    allpos, lk = KINDS[kind]
    NP = (N + 15) // 16 * 16
    LD = 2 * NP
    P = _problem(N, radius, 1000 + 7 * N + radius, NP)
    K = P['offsets'].shape[0]
    ref = loss_map_ref(P['lmap'], N, NP, P['centers'], P['bag_img'], P['offsets'], P['stride'], P['pad_hw'], P['labels'].long(), EPS,
                       allpos, lk)
    d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in P.items()}
    lmap, offs = d['lmap'].contiguous(), d['offsets']
    offs = ops.with_reach(offs, ops.offsets_reach(offs))
    B, H, W, _ = lmap.shape
    scale = torch.ones(1, device=dev)

    def check_fwd(s, stats, what):
        assert abs(float(s[0]) - float(ref['sum'])) <= 2e-5 * max(1.0, abs(float(ref['sum']))), (what, float(s[0]), float(ref['sum']))
        assert float(stats[0]) == ref['count'] and float(stats[1]) == ref['hits'], (what, stats.tolist(), ref['count'], ref['hits'])

    bl, _, valid = ops.bag_gather(lmap, d['centers'], d['bag_img'], offs, d['stride'], d['pad_hw'], pts=False)
    weight = valid.float().contiguous()
    assert torch.equal(weight.cpu().double(), ref['weight'])
    if allpos:
        s, stats = ops.allpos_fwd(bl, N, weight, d['labels'], EPS, lk)
        check_fwd(s, stats, 'allpos_fwd')
        mt = bp = lw = None
    else:
        bp, s, stats, mt, lw = ops.mil_loss_fwd(bl, N, NP, weight, d['labels'], EPS, want_aux=True, loss_kind=lk)
        check_fwd(s, stats, 'mil_loss_fwd')
        assert_close(bp, ref['prob'], 1e-5, 'bag prob')
        if N <= 128:
            bl2, w2, bp2, s2, st2, mt2, lw2 = ops.bag_mil_fwd(lmap, N, NP, d['centers'], d['bag_img'], offs, d['stride'], d['pad_hw'],
                                                              d['labels'], EPS, loss_kind=lk)
            check_fwd(s2, st2, 'bag_mil_fwd')
            assert torch.equal(bl2[..., :N], bl[..., :N]) and torch.equal(w2, weight)
    # backward: scatter, tiles (LD <= 160), staged
    kw = dict(loss_kind=lk, scale_mil=None if allpos else scale, scale_pos=scale if allpos else None)
    grads = {}
    gmap = torch.zeros((B, H, W, LD), device=dev)
    ops.cpr_loss_bwd_scatter(bl, weight, mt, bp, lw, d['labels'], d['centers'], d['bag_img'], offs, gmap, N, NP, d['stride'], EPS, **kw)
    grads['scatter'] = gmap
    if LD <= 160:
        grads['tiles'] = ops.cpr_loss_bwd_map(bl, weight, mt, bp, lw, d['labels'], d['centers'], d['img_ptr'], offs, (B, H, W, LD), N, NP,
                                              d['stride'], ops.offsets_reach(offs), EPS, **kw)
    dbl = torch.zeros_like(bl)
    if allpos:
        ops.gfocal_bwd(bl, bl.shape[0] * K, N, LD, d['labels'].repeat_interleave(K), weight.reshape(-1) if lk == 0 else None, EPS, scale,
                       dbl, LD, accumulate=True, loss_kind=lk)
    else:
        ops.mil_loss_bwd(bl, N, NP, weight, d['labels'], EPS, bp, scale, grad_out=dbl, loss_kind=lk)
    grads['staged'] = ops.bag_gather_bwd(dbl, (B, H, W, LD), d['centers'], d['bag_img'], offs, d['stride'])
    for path, gm in grads.items():
        assert torch.isfinite(gm).all(), path
        err = float((gm.cpu().double() - ref['grad']).abs().max())
        bound = 2e-5 * max(1e-3, float(ref['grad'].abs().max()))
        assert err <= bound, f'{kind} {path}: max |grad - ref| {err:.3e} > {bound:.3e}'
        if allpos:
            assert not gm[..., NP:].any(), f'{path}: AllPosLoss must leave the instance columns at zero'


def _head(case, w, dev):
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    from oracle.make_golden import ref_cpr_cfg
    inp_d = dict(synth_lite())
    cfg = ref_cpr_cfg(inp_d)
    cfg.update(LOSS_TYPE_CASES[case][0])
    cfg['test_cfg'] = dict(cfg['test_cfg'])
    head = build_head(cfg).to(dev)
    sd = head.state_dict()
    sd.update(w)
    head.load_state_dict(sd, strict=True)
    return head


def synth_lite():
    from oracle.synth import CPR_CONFIGS
    return CPR_CONFIGS['lite']


def _run(head, inp, gtw, dev, mode=None, deterministic=False):
    os.environ.pop('PTB_LOSS_BWD', None)
    if mode is not None:
        os.environ['PTB_LOSS_BWD'] = mode
    torch.use_deterministic_algorithms(deterministic)
    try:
        head.zero_grad(set_to_none=True)
        feat = inp['cls_feat'].to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        gtb = [b.to(dev) for b in inp['gt_bboxes']]
        gtl = [l.to(dev) for l in inp['gt_labels']]
        losses = head.loss([feat], [feat], gtb, gtl, inp['img_metas'], gt_weights=gtw)
        sum(v for k, v in losses.items() if 'loss' in k).backward()
        return losses, [feat.grad] + [p.grad for p in (head.cls_out.weight, head.cls_out.bias, head.ins_out.weight, head.ins_out.bias)]
    finally:
        os.environ.pop('PTB_LOSS_BWD', None)
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize('case', list(LOSS_TYPE_CASES))
def test_head_against_oracle_and_golden(dev, golden_dir, case):
    gold = np.load(os.path.join(golden_dir, f'cpr_lite_loss_{case}.npz'))
    inp, w, gtw = loss_type_inputs(case, int(gold['seed']))
    cfg = oracle_cfg(case, inp['cfgd'])
    head = _head(case, {k: v.to(dev) for k, v in w.items()}, dev)
    fo = inp['cls_feat'].clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    ol = olt.cpr_loss(fo, wo, inp['gt_bboxes'], inp['gt_labels'], inp['img_metas'], cfg, gt_weights=gtw)
    sum(v for k, v in ol.items() if 'loss' in k).backward()
    allpos = cfg.get('loss_mil', 'MILLoss') == 'AllPosLoss'
    generic = gtw is not None
    modes = [(None, False)] if generic else [(None, False), ('staged', False), (None, True)]
    runs = {}
    for mode, det in modes:
        losses, grads = _run(head, inp, gtw, dev, mode, det)
        what = f'{case} mode={mode} deterministic={det}'
        for k in ('gt_loss', 'pos_loss', 'neg_loss', 'bag_acc'):
            assert_close(losses[k].reshape(-1), ol[k].detach().reshape(-1), 1e-4, f'{what} {k}')
            assert_close(losses[k].reshape(-1), torch.from_numpy(gold['loss_' + k]), 1e-4, f'{what} {k} vs golden')
        assert float(losses['bag_acc'].reshape(-1)[0]) == pytest.approx(float(gold['loss_bag_acc'][0]), abs=1e-4)
        assert torch.isfinite(grads[0]).all()
        assert_close(grads[0], fo.grad, 2e-4, f'{what} d feature map')
        sub = grads[0].detach().cpu().contiguous().flatten()[::211].numpy()
        assert np.abs(sub - gold['grad_feat_sub']).max() <= 2e-4 * np.abs(gold['grad_feat_sub']).max()
        assert_close(grads[1], wo['cls_out.weight'].grad, 2e-4, f'{what} d cls_out.weight')
        assert_close(grads[2], wo['cls_out.bias'].grad, 2e-4, f'{what} d cls_out.bias')
        if allpos:
            assert grads[3] is not None and grads[4] is not None, 'AllPosLoss: ins_out gradients must be zero tensors, not None'
            assert not grads[3].any() and not grads[4].any(), 'AllPosLoss: ins_out gradients must be exactly zero'
        else:
            assert_close(grads[3], wo['ins_out.weight'].grad, 2e-4, f'{what} d ins_out.weight')
        runs[(mode, det)] = [g.clone() for g in grads]
    if not generic:
        _, again = _run(head, inp, gtw, dev, None, True)
        assert all(torch.equal(a, b) for a, b in zip(runs[(None, True)], again)), f'{case}: deterministic gradients differ between runs'


@pytest.mark.parametrize('case', ['mil_bce', 'allpos_gfocal', 'allpos_bce'])
def test_image_without_gts(dev, case):
    """second image of the batch has no GT: losses and gradients stay finite (the fully invalid bag of image 0 is there too)."""
    inp, w, gtw = loss_type_inputs(case)
    inp['cls_feat'] = torch.cat([inp['cls_feat'], inp['cls_feat'].flip(-1)])
    inp['gt_bboxes'].append(torch.zeros(0, 4))
    inp['gt_labels'].append(torch.zeros(0, dtype=torch.int64))
    inp['img_metas'] = inp['img_metas'] * 2
    head = _head(case, {k: v.to(dev) for k, v in w.items()}, dev)
    for mode, det in ((None, False), ('staged', False), (None, True)):
        losses, grads = _run(head, inp, gtw, dev, mode, det)
        assert all(torch.isfinite(v).all() for v in losses.values())
        assert all(torch.isfinite(g).all() for g in grads)
