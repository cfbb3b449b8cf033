"""CPU: the host references of tests/fcos_ref.py against oracle/fcos.py, which the fcos_*.npz fixtures pin to the reference head.

  * targets        equals the fixtures' labels and bbox_targets and oracle.get_targets on the synthetic cases of the kernel tests.
  * box_terms_f32  equals the oracle's overlaps_aligned-based loss in fp32: bit for bit for linear IoU and GIoU, within 1 ulp for log IoU.
  * box_grad64     equals float64 autograd of the oracle's loss on dyadic inputs (every +, -, * exact in fp32 and float64 alike, so both
                   sides see the same ties), including every planted tie and clamp edge: torch's 0.5 split of maximum / minimum and
                   clamp's >= mask.
  * decode         equals oracle.decode on the fixtures' maps: top-k rows as sets within equal keys, boxes, scores and centerness.
"""
import os

import numpy as np
import pytest
import torch

from oracle import fcos as ofc
from tests import fcos_ref as ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FIXTURES = ['tinyperson', 'coco80', 'options', 'no_pos']
SYNTH = ['one_level', 'odd_strides', 'crowded', 'eight_levels', 'no_gt', 'planted', 'planted_cs']


def gold(name):
    return np.load(os.path.join(GOLD, f'fcos_{name}.npz'))


@pytest.mark.parametrize('name', FIXTURES)
def test_targets_equal_the_fixtures(name):
    g, inp, hc = gold(name), ofc.case_inputs(name), ofc.CASES[name]['head']
    radius = hc.get('center_sample_radius', 1.5) if hc.get('center_sampling') else None
    lab, tgt = ref.targets(inp['sizes'], hc['strides'], inp['gt_bboxes'], inp['gt_labels'], hc['regress_ranges'], radius,
                           hc.get('norm_on_bbox', False), hc['num_classes'])
    assert torch.equal(lab, torch.cat([torch.from_numpy(g[f'labels{l}'].astype(np.int64)) for l in range(5)]))
    assert torch.equal(tgt, torch.cat([torch.from_numpy(g[f'bbox_targets{l}']) for l in range(5)]))


@pytest.mark.parametrize('kind', SYNTH)
def test_targets_equal_the_oracle_on_the_synthetic_cases(kind):
    c = ref.target_case(kind)
    cfg = dict(num_classes=c['C'], strides=c['strides'], regress_ranges=c['ranges'], norm_on_bbox=c['norm'],
               center_sampling=c['radius'] is not None, center_sample_radius=c['radius'] or 1.5)
    pts = ofc.points(c['sizes'], c['strides'])
    want_l, want_t = ofc.get_targets(pts, c['gts'], c['gls'], cfg)
    lab, tgt = ref.targets(c['sizes'], c['strides'], c['gts'], c['gls'], c['ranges'], c['radius'], c['norm'], c['C'])
    assert torch.equal(lab, torch.cat(want_l))
    assert torch.equal(tgt, torch.cat(want_t))
    if kind.startswith('planted'):
        assert bool(((lab >= 0) & (lab < c['C'])).any())


def test_planted_targets_hit_their_edges():
    """the planted GTs do what their comments say on the 8-stride grid of 'planted'"""
    c = ref.target_case('planted')
    lab, tgt = ref.targets(c['sizes'], c['strides'], c['gts'], c['gls'], c['ranges'], None, False, c['C'])
    W, HW = 48, 48 * 48
    at = lambda x, y: y * W + x                                        # level 0, image 0
    assert int(lab[at(2, 3)]) == c['C']                                # on the left edge of GT 0: outside
    assert int(lab[at(3, 3)]) == 0
    assert int(lab[at(10, 3)]) == 1 and float(tgt[at(10, 3)].max()) == 16.0     # max distance 16 == hi of range 0
    assert int(lab[at(20, 6)]) == 3                                    # three GTs of area 128: the first


def _f32_oracle_terms(points, pred, tgt, mode, overlap_eps, eps):
    """the oracle's loss of fcos_head.loss per row in fp32 torch, times the centerness weight.  The weight is centerness_f32 (sqrt
    correctly rounded, as the kernel's __fsqrt_rn): ATen's vectorised CPU sqrt is not correctly rounded, so the oracle's own
    centerness_target is 1 ulp off now and then (test_centerness_is_the_correctly_rounded_oracle_formula)."""
    p, d, t = (torch.as_tensor(np.asarray(a, np.float32)) for a in (points, pred, tgt))
    db, dt = ofc.distance2bbox(p, d), ofc.distance2bbox(p, t)
    w = torch.from_numpy(ref.centerness_f32(t))
    if mode == 'giou':
        l = 1 - ofc.overlaps_aligned(db, dt, 'giou', eps)
    else:
        ious = ofc.overlaps_aligned(db, dt, eps=overlap_eps).clamp(min=eps)
        l = 1 - ious if mode == 'linear' else -ious.log()
    return (l * w).numpy()


def test_centerness_is_the_correctly_rounded_oracle_formula():
    """centerness_f32 is fl(sqrt(x)) of the oracle's fp32 product x, and within 1 ulp of the oracle's CPU centerness_target"""
    _, _, tgt = _random_rows(20000, 4)
    t = torch.from_numpy(tgt)
    lr, tb = t[:, [0, 2]], t[:, [1, 3]]
    x = ((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) * (tb.min(dim=-1)[0] / tb.max(dim=-1)[0])).numpy()
    got = ref.centerness_f32(tgt)
    assert np.array_equal(got, np.sqrt(x.astype(np.float64)).astype(np.float32))
    np.testing.assert_array_max_ulp(got, ofc.centerness_target(t).numpy(), 1)


def _random_rows(n, seed, spread=0.6):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.randint(0, 200, (n, 2), generator=g) * 8 + 4).float()
    pred = torch.exp(torch.randn(n, 4, generator=g) * spread) * 16
    tgt = torch.exp(torch.randn(n, 4, generator=g) * spread) * 16
    return pts.numpy(), pred.numpy(), tgt.numpy()


@pytest.mark.parametrize('mode', ['log', 'linear', 'giou'])
def test_box_terms_equal_the_oracle_loss_in_fp32(mode):
    pts, pred, tgt = _random_rows(20000, 3)
    pred[:500] = tgt[:500]                                            # ties
    pred[500:1000, 2] = -tgt[500:1000, 0]                              # touching
    lab = np.zeros(len(pts), np.int64)
    got = ref.box_terms_f32(pts, pred, tgt, lab, 1, mode)
    want = _f32_oracle_terms(pts, pred, tgt, mode, 1e-6, 1e-6)
    if mode == 'log':
        # the oracle's fp32 logf within 1 ulp of the correctly rounded log: one ulp of the product with w
        np.testing.assert_array_max_ulp(got.astype(np.float32), want, 1)
    else:
        assert got.dtype == np.float32 and np.array_equal(got, want)


def _dyadic_rows(seed, n=4000):
    """random multiples of 1/8 up to 32 (pred may be negative) and the planted rows, at points x * 8 + 4 below 2^11"""
    g = torch.Generator().manual_seed(seed)
    pred = (torch.randint(-16, 257, (n, 4), generator=g) / 8.0).numpy()
    tgt = (torch.randint(1, 257, (n, 4), generator=g) / 8.0).numpy()
    pred[: n // 8] = tgt[: n // 8]
    pp, pt = ref.planted_box_rows()
    pred, tgt = np.concatenate([pp, pred]).astype(np.float32), np.concatenate([pt, tgt]).astype(np.float32)
    pts = (torch.randint(0, 200, (len(pred), 2), generator=g) * 8 + 4).float().numpy()
    return pts, pred, tgt


@pytest.mark.parametrize('mode', ['log', 'linear', 'giou'])
def test_box_grad64_equals_float64_autograd_on_dyadic_inputs(mode):
    pts, pred, tgt = _dyadic_rows(5)
    eps = ref.PLANT_EPS
    n = len(pts)
    lab = np.zeros(n, np.int64)
    lab[-7:] = [1, -1, 1, -1, 1, -1, 1]                                  # negatives, C = 1
    grad, S = ref.box_grad64(pts, pred, tgt, lab, 1, mode, eps, eps, scale=0.75)
    p64 = torch.from_numpy(pred.astype(np.float64)).requires_grad_(True)
    P, T = torch.from_numpy(pts.astype(np.float64)), torch.from_numpy(tgt.astype(np.float64))
    db, dt = ofc.distance2bbox(P, p64), ofc.distance2bbox(P, T)
    w = torch.from_numpy(ref.centerness_f32(tgt).astype(np.float64))
    if mode == 'giou':
        l = 1 - ofc.overlaps_aligned(db, dt, 'giou', eps)
    else:
        ious = ofc.overlaps_aligned(db, dt, eps=eps).clamp(min=eps)
        l = 1 - ious if mode == 'linear' else -ious.log()
    pos = torch.from_numpy(ref.positive(lab, 1))
    (0.75 * (l * w)[pos]).sum().backward()
    want = p64.grad.numpy()
    err = np.abs(grad - want)
    assert np.all(err <= 1e-12 * S + 1e-300), (mode, np.argwhere(err > 1e-12 * S + 1e-300)[:8].tolist())
    assert np.all(grad[~pos.numpy()] == 0)
    # the planted rows reach the branches they were built for
    v = ref._box_f32(pts, pred, tgt, mode, eps, eps)
    assert np.any(v['x1'] == v['u1']) and np.any(v['wx'] == 0) and np.any(v['wx'] < 0) and np.any(v['uni'] == np.float32(eps))
    assert np.any(v['iou'] == np.float32(eps)) and np.any(v['uni'] < np.float32(eps))
    if mode == 'giou':
        assert np.any(v['ea_raw'] == np.float32(eps)) and np.any(v['ea_raw'] < np.float32(eps))


def test_ctr_grad_and_terms_match_float64_torch():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(5000, generator=g) * 4
    x[:15] = torch.tensor([0.0, 1e-30, -1e-30, 16.5, -16.5, 16.7, -16.7, 17.0, -17.0, 88.0, -88.0, 100.5, -100.5, 104.5, -104.5])
    tgt = torch.exp(torch.randn(5000, 4, generator=g)) * 10
    lab = torch.randint(-1, 3, (5000,), generator=g)
    terms, pieces = ref.ctr_terms64(x, tgt, lab, 2)
    t64 = torch.from_numpy(ref.centerness_f32(tgt).astype(np.float64))
    x64 = x.double().requires_grad_(True)
    bce = torch.nn.functional.binary_cross_entropy_with_logits(x64, t64, reduction='none')
    pos = torch.from_numpy(ref.positive(lab, 2))
    assert np.allclose(terms[pos.numpy()], bce.detach().numpy()[pos.numpy()], rtol=1e-12, atol=1e-300)
    assert np.all(pieces >= np.abs(terms))
    bce[pos].sum().backward()
    gr = ref.ctr_grad_f32(x, tgt, lab, 2, scale=1.0)
    assert np.allclose(gr, x64.grad.numpy(), rtol=0, atol=2 ** -22)


def _nhwc(ts):
    return [t.permute(0, 2, 3, 1).contiguous() for t in ts]


def _eval_maps(name):
    g = gold(name)
    if 'eval_cls0' in g:
        return tuple([torch.from_numpy(g[f'eval_{n}{l}']) for l in range(5)] for n in ('cls', 'reg', 'ctr'))
    return ofc.case_inputs(name)['maps']


@pytest.mark.parametrize('name', FIXTURES)
def test_decode_equals_the_oracle_on_the_fixture_maps(name):
    c, inp = ofc.CASES[name], ofc.case_inputs(name)
    cls, reg, ctr = _eval_maps(name)
    metas, rescale = inp['img_metas'], c.get('rescale', False)
    img_hw = np.array([m['img_shape'][:2] for m in metas], np.float32)
    sf = np.stack([m['scale_factor'] for m in metas]).astype(np.float32) if rescale else None
    nms_pre = c['test']['nms_pre']
    idx, boxes, scores, cts = ref.decode(_nhwc(cls), _nhwc(reg), _nhwc(ctr), c['head']['strides'], img_hw, nms_pre, sf)
    bb, sc, kk, tk = ofc.decode(cls, reg, ctr, metas, c['head'], c['test'], rescale)
    off = 0
    for l, (h, w) in enumerate(inp['sizes']):
        n = ofc.fcos_rows(h * w, nms_pre)
        key = ref.keys_f32(_nhwc([cls[l]])[0], _nhwc([ctr[l]])[0])
        for b in range(len(metas)):
            mine = idx[b, off:off + n].astype(np.int64)
            theirs = tk[l][b].numpy() if tk[l] is not None else np.arange(n)
            assert np.array_equal(np.sort(mine), np.sort(theirs)), (l, b)
            if tk[l] is not None:
                assert np.array_equal(key[b][mine], np.sort(key[b][mine])[::-1])
            o1, o2 = np.argsort(mine), np.argsort(theirs)
            assert np.array_equal(boxes[b, off:off + n][o1], bb[b, off:off + n].numpy()[o2])
            np.testing.assert_array_max_ulp(scores[b, off:off + n][o1], sc[b, off:off + n].numpy()[o2], 1)
            np.testing.assert_array_max_ulp(cts[b, off:off + n][o1], kk[b, off:off + n].numpy()[o2], 1)
        off += n
