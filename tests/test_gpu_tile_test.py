"""GPU: tile testing of the two-stage detector (pointtinybenchmark_b200/tile_test.py, csrc/tile_test.cu) against host restatements:
ptb_batched_nms against oracle/p2p.py's batched_nms / nms, ptb_aug_merge bit for bit against the reference's bbox_mapping_back +
torch.stack(...).mean(0) on the CPU, and tile_aug_test / StandardRoIHead.aug_test end to end against oracle/tile_test.py."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import roi_head as orh
from oracle import tile_test as ott
from oracle.p2p import batched_nms as ref_batched_nms, nms as ref_nms

pytestmark = pytest.mark.gpu


def _boxes(g, n, extent=2000.0, lo=8.0, hi=60.0):
    xy = torch.rand(n, 2, generator=g) * extent
    wh = lo + torch.rand(n, 2, generator=g) * (hi - lo)
    return torch.cat([xy, xy + wh], 1)


@pytest.mark.parametrize('n', [1, 9999, 10000, 10001, 65536])
@pytest.mark.parametrize('C', [1, 2, 80])
def test_batched_nms_against_host(n, C):
    from pointtinybenchmark_b200 import ops
    g = torch.Generator().manual_seed(n * 7 + C)
    b = _boxes(g, n, extent=3000.0 if n > 20000 else 1500.0)
    s = torch.rand(n, generator=g)
    lab = torch.randint(0, C, (n,), generator=g)
    d, keep = ref_batched_nms(b, s, lab, 0.5)
    rows = torch.cat([b, s[:, None]], 1).cuda()[None].contiguous()
    cnt, det, olab, okeep = ops.batched_nms(rows, rows[..., 4], lab.int().cuda()[None].contiguous(), None, 0.5)
    k = int(cnt[0])
    assert k == len(keep)
    assert torch.equal(okeep[0, :k].cpu().long(), keep)
    assert torch.equal(det[0, :k].cpu(), d)
    assert torch.equal(olab[0, :k].cpu().long(), lab[keep])


def test_batched_nms_edges():
    from pointtinybenchmark_b200 import ops
    # equal scores, identical boxes, zero-area boxes, everything suppressed, a max_num cut, an empty segment, counts per segment
    b = torch.tensor([[0., 0., 10., 10.]] * 6 + [[5., 5., 5., 5.]] * 3 + [[0., 0., 10., 10.5]] * 3)
    s = torch.tensor([0.5] * 12)
    rows = torch.cat([b, s[:, None]], 1)
    segs = torch.stack([rows, rows.flip(0), rows]).cuda().contiguous()
    counts = torch.tensor([12, 12, 0], dtype=torch.int32).cuda()
    for max_num in (-1, 1, 2):
        cnt, det, _, keep = ops.batched_nms(segs, segs[..., 4], None, counts, 0.5, max_num=max_num)
        for sidx in range(3):
            n = int(counts[sidx])
            k = ref_nms(segs[sidx, :n, :4].cpu(), segs[sidx, :n, 4].cpu(), 0.5) if n else torch.zeros(0, dtype=torch.long)
            k = k[:max_num] if max_num > 0 else k
            assert int(cnt[sidx]) == len(k)
            assert torch.equal(keep[sidx, :len(k)].cpu().long(), k)
    with pytest.raises(NotImplementedError, match='65536'):
        z = torch.zeros((1, 65537, 5), device='cuda')
        ops.batched_nms(z, z[..., 4], None, None, 0.5)


def _meta(g, direction, sf, img=(512, 640)):
    return dict(img_shape=(img[0], img[1], 3), scale_factor=np.array([sf] * 4, np.float32), flip=direction is not None,
                flip_direction=direction)


@pytest.mark.parametrize('A', [1, 2, 3, 4, 12])
@pytest.mark.parametrize('cols', ['4', '4C'])
def test_aug_merge_bit_exact(A, cols):
    from pointtinybenchmark_b200 import ops
    g = torch.Generator().manual_seed(A)
    T, N, C = 3, 37, 3
    dirs = [None, 'horizontal', 'vertical', 'diagonal']
    metas = [_meta(g, dirs[(t + a) % 4], [0.5, 1.0, 1.5][(a + t) % 3]) for t in range(T) for a in range(A)]
    counts = torch.tensor([N, 20, 1 + 7], dtype=torch.int32)
    box_cols = 4 if cols == '4' else 4 * C
    boxes = _boxes(g, T * A * N * C, 600.0).view(T * A, N, C, 4)
    if box_cols == 4:
        boxes = boxes[:, :, :1].expand(T * A, N, C, 4).contiguous()
    scores = torch.rand(T * A, N, C, generator=g)
    meta = ops.aug_meta(metas, [i // A for i in range(T * A)], [0] * (T * A), 'cuda')
    ob, os_ = ops.aug_merge(boxes.cuda(), scores.cuda(), counts.cuda(), meta, A, box_cols)
    ob, os_ = ob.cpu(), os_.cpu()
    for t in range(T):
        n = int(counts[t])
        rb = [ott.bbox_mapping_back(boxes[t * A + a, :n, :(1 if box_cols == 4 else C)].reshape(n, -1), metas[t * A + a]) for a in range(A)]
        ref_b = torch.stack(rb).mean(0).view(n, -1, 4)
        # the reference stacks (n, C + 1) softmax scores; the background column does not change the other columns' sums
        sc = [torch.cat([scores[t * A + a, :n], torch.zeros(n, 1)], 1) for a in range(A)]
        ref_s = torch.stack(sc).mean(0)[:, :C]
        assert torch.equal(ob[t, :n, :ref_b.shape[1]], ref_b)
        assert torch.equal(os_[t, :n], ref_s)
        assert bool((os_[t, n:] == -float('inf')).all())


def _heads(C=1, channels=8, fc=32, max_per_img=-1, rpn_max=300, cls_scale=4.0):
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    from pointtinybenchmark_b200.rpn import RPNHead
    rpn_cfg = dict(nms_pre=200, max_per_img=rpn_max, nms=dict(type='nms', iou_threshold=0.7), min_bbox_size=0)
    test = dict(score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=max_per_img)
    rpn = RPNHead(channels, channels, anchor_generator=dict(type='AnchorGenerator', scales=[2], ratios=[0.5, 1.0, 2.0],
                                                             strides=[4, 8, 16, 32, 64]), test_cfg=rpn_cfg).cuda()
    kw = orh.head_kwargs('tinyperson')
    kw['bbox_roi_extractor']['out_channels'] = channels
    kw['bbox_head'].update(in_channels=channels, fc_out_channels=fc, num_classes=C)
    roi = StandardRoIHead(**kw, test_cfg=test).cuda()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for p in list(rpn.parameters()) + list(roi.parameters()):
            p.copy_(torch.randn(p.shape, generator=g) * (0.3 if p.dim() > 1 else 0.1))
        roi.bbox_head.fc_cls.weight.mul_(cls_scale)      # 4: most scores saturate at 1.0, so every proposal is a detection
    return rpn, roi, rpn_cfg, test


def _tiles(T_h, T_w, th=128, tw=160, A=1, flips=(None,), scales=(1.0,), channels=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    feats, metas = [], []
    for i in range(T_h):
        for j in range(T_w):
            for d in flips:
                for s in scales:
                    h, w = int(th * s), int(tw * s)
                    feats.append([torch.randn(1, channels, -(-h // st), -(-w // st), generator=g).cuda() for st in (4, 8, 16, 32, 64)])
                    metas.append([dict(img_shape=(h, w, 3), pad_shape=(h, w, 3), ori_shape=(th, tw, 3),
                                       scale_factor=np.array([s] * 4, np.float32), flip=d is not None, flip_direction=d,
                                       tile_offset=(j * (tw - 30), i * (th - 30)))])
    return feats, metas


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
TILE_CASES = [n for n, c in ott.CASES.items() if not c['direct']]


class _CpuMapsRPN:
    """the RPNHead with its three convs run on the CPU one aug at a time, as the reference runs them, so that the RPN maps equal the
    fixtures' bit for bit (cuDNN's TF32 convs would round them differently); proposals and everything after run on the GPU"""

    def __init__(self, head):
        self.head, self.cpu = head, copy.deepcopy(head).cpu()
        self.proposals, self.test_cfg = head.proposals, head.test_cfg

    def __call__(self, x):
        n = torch.get_num_threads()
        torch.set_num_threads(1)
        try:
            outs = [self.cpu([l[b:b + 1].cpu() for l in x]) for b in range(x[0].shape[0])]
        finally:
            torch.set_num_threads(n)
        return tuple([torch.cat([o[k][l] for o in outs]).cuda() for l in range(len(x))] for k in range(2))


def _golden_heads(name):
    from pointtinybenchmark_b200.roi_head import StandardRoIHead
    from pointtinybenchmark_b200.rpn import RPNHead
    c, inp = ott.CASES[name], ott.case_inputs(name)
    rk, hk = ott.head_kwargs(name)
    rpn = RPNHead(**rk, test_cfg=c['rpn']).cuda().eval()
    rpn.load_state_dict(inp['rpn_weights'])
    roi = StandardRoIHead(**hk, test_cfg=c['rcnn']).cuda().eval()
    roi.bbox_head.load_state_dict(inp['roi_weights'])
    feats = [[l.cuda() for l in f] for f in inp['feats']]
    return c, inp, _CpuMapsRPN(rpn), roi, feats


def _split(d, lab, C):
    return [d[lab == k] for k in range(C)]


def _check_exact(res, ref, C):
    """per class the same keep set (count exact, every row within 1e-4 plus 4 ulps of its value: the tile offset moves boxes to image
    coordinates up to 1920, where one fp32 ulp of the decode's rounding is 1.2e-4), and the rows in NMS order (scores non-increasing).
    The order among rows whose scores agree to a few ulps is not compared: ptb_rpn_proposals may order near-tied proposals differently
    from the reference's CPU sigmoid, which moves such rows' positions and so their tie-break."""
    srt = lambda a: a[np.lexsort(a.T[::-1])]
    for k in range(C):
        assert res[k].shape == ref[k].shape, f'class {k}: {res[k].shape[0]} rows, reference {ref[k].shape[0]}'
        np.testing.assert_allclose(srt(res[k]), srt(ref[k]), rtol=4.8e-7, atol=1e-4)
        assert bool((np.diff(res[k][:, 4]) <= 0).all())


@pytest.mark.parametrize('name', TILE_CASES)
def test_tile_aug_test_golden(name):
    """tile_aug_test against TwoStageDetector.tile_aug_test of the real reference (tests/golden/tile_test_*.npz): the RPN's per-aug
    proposals, then every detection of the image exactly"""
    from pointtinybenchmark_b200.tile_test import tile_aug_test
    f = np.load(os.path.join(GOLD, f'tile_test_{name}.npz'))
    c, inp, rpn, roi, feats = _golden_heads(name)
    metas = copy.deepcopy(inp['img_metas'])
    props = None
    if len({tuple(x[0].shape) for x in feats}) == 1:
        with torch.no_grad():
            props = rpn.proposals.get_bboxes(*rpn([torch.cat([x[l] for x in feats]) for l in range(5)]), [m[0] for m in metas])
    if props is not None:                    # one FPN shape: the batched proposals against the reference's per-aug ones
        ref = np.split(f['rpn_props'], np.cumsum(f['rpn_counts'])[:-1])
        for p, r in zip(props, ref):
            p = p.cpu().numpy()
            assert p.shape[0] == r.shape[0]
            srt = lambda a: a[np.lexsort(a.T[::-1])]           # the same proposal set (near-tied scores may be ordered differently)
            np.testing.assert_allclose(srt(p), srt(r), rtol=0, atol=1e-4)
    res = tile_aug_test(rpn, roi, feats, metas, c['rcnn'])[0]
    assert all('tile_offset' not in m[0] for m in metas)
    _check_exact(res, _split(f['dets'], f['labels'], c['C']), c['C'])
    if name == 'tinyperson12':
        assert int(f['merge_rows']) >= 10000          # the cross-tile merge ran mmcv's class-by-class branch
    if name == 'empty':
        assert all(r.shape == (0, 5) for r in res)


def test_tile_aug_test_rescale():
    """rescale=True skips the first aug's scale_factor multiply (standard_roi_head.py:262-266); flip_scale's first augs are at 0.5"""
    from pointtinybenchmark_b200.tile_test import tile_aug_test
    name = 'flip_scale'
    f = np.load(os.path.join(GOLD, f'tile_test_{name}.npz'))
    c, inp, rpn, roi, feats = _golden_heads(name)
    res = tile_aug_test(rpn, roi, feats, copy.deepcopy(inp['img_metas']), c['rcnn'], rescale=True)[0]
    props = [torch.from_numpy(p) for p in np.split(f['rpn_props'], np.cumsum(f['rpn_counts'])[:-1])]
    d, l = ott.tile_aug_test(inp['feats'], [m[0] for m in inp['img_metas']], props, inp['roi_weights'], ott.roi_head_spec(name), c['rpn'],
                             c['rcnn'], rescale=True)
    _check_exact(res, _split(d.numpy(), l.numpy(), 1), 1)


def test_aug_test_direct_golden():
    """StandardRoIHead.aug_test with a non-zero tile_offset every aug keeps every proposal with (rescale=False, scale 1.5, diagonal
    flip) against the reference; an offset that drops proposals of one aug raises as the reference's torch.stack does"""
    name = 'direct'
    f = np.load(os.path.join(GOLD, f'tile_test_{name}.npz'))
    c, inp, _, roi, feats = _golden_heads(name)
    res = roi.aug_test(feats, [inp['proposals'].cuda()], copy.deepcopy(inp['img_metas']))[0]
    _check_exact(res, _split(f['dets'], f['labels'], c['C']), c['C'])
    assert int(f['mismatch_raises']) == 1
    bad = copy.deepcopy(inp['img_metas'])
    bad[1][0]['tile_offset'] = (110, 90)
    with pytest.raises(RuntimeError, match='stack'):
        roi.aug_test(feats, [inp['proposals'].cuda()], bad)
    empty = roi.aug_test_bboxes(feats, copy.deepcopy(inp['img_metas']), [inp['proposals'][:0].cuda()], roi.test_cfg)
    assert empty[0].shape == (0, 5) and empty[1].shape == (0,)


@pytest.mark.parametrize('C', [1, 3, 80])
def test_tile_concat_order(C):
    """ptb_tile_concat: tile order, then class-major, then the NMS order within a class; * scale_factor then + offset in fp32"""
    from pointtinybenchmark_b200 import ops
    g = torch.Generator().manual_seed(C)
    T, K = 5, 64
    det = torch.rand(T, K, 5, generator=g) * 300
    lab = torch.randint(0, C, (T, K), generator=g).int()
    cnt = torch.tensor([64, 0, 17, 1, 40], dtype=torch.int32)
    off = torch.tensor([[0., 0.], [540., 0.], [0., 284.], [1080., 568.], [1280., 568.]])
    sf = torch.rand(T, 4, generator=g) + 0.5
    rows, rlab, n = ops.tile_concat(det.cuda(), lab.cuda(), cnt.cuda(), off.cuda(), sf.cuda())
    ref, rl = [], []
    for t in range(T):
        d = det[t, :cnt[t]].numpy().copy()
        d[:, :4] *= sf[t].numpy()
        for k in range(C):
            r = d[lab[t, :cnt[t]].numpy() == k]
            r[:, [0, 2]] += off[t, 0].item()
            r[:, [1, 3]] += off[t, 1].item()
            ref.append(r)
            rl += [k] * len(r)
    ref = np.concatenate(ref)
    assert int(n[0]) == len(ref)
    assert np.array_equal(rows[:len(ref)].cpu().numpy(), ref)
    assert rlab[:len(ref)].cpu().tolist() == rl


def test_tile_aug_test_tinyperson_shape_repeatable():
    """12 tiles of a 1080 x 1920 image at 256 channels and fc_out_channels=1024: two runs give identical results"""
    from pointtinybenchmark_b200.tile_test import tile_aug_test
    rpn, roi, rpn_cfg, test = _heads(C=1, channels=256, fc=1024, rpn_max=1000)
    feats, metas = _tiles(3, 4, th=512, tw=640, channels=256)
    r1 = tile_aug_test(rpn, roi, feats, copy.deepcopy(metas), test)
    r2 = tile_aug_test(rpn, roi, feats, copy.deepcopy(metas), test)
    assert r1[0][0].shape[0] > 0
    assert np.array_equal(r1[0][0], r2[0][0])
