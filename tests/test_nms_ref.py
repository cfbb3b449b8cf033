"""CPU checks of tests/nms_ref.py, the host restatement the NMS kernel tests compare against: the offset branch against
oracle.p2p.multiclass_nms, per-class greedy NMS against torchvision.ops.nms, soft-NMS against oracle.p2p.soft_nms, the split branch
against the per-class replay of tests/helpers.py, and the claim of nms.cu's prepare kernel that its `slow` test is conservative: an
image whose offset-branch result differs from the class-by-class result is always flagged."""
import numpy as np
import pytest
import torch

from oracle import p2p as op2p
from tests import nms_ref as ref
from tests.helpers import nms_replay_per_class

F32 = np.float32


def _image(seed, P, C, extent=(300.0, 200.0), boxes=False, corner=False, frac=0.15):
    rng = np.random.default_rng(seed)
    pts = (rng.random((P, 2)) * np.array(extent)).astype(F32)
    if corner:                                                     # both extreme corners of a square image (the `slow` layout)
        pts[:3] = [[0, 0], [1, 2], [2, 1]]
        pts[3:6] = [[extent[0], extent[0]], [extent[0] - 1, extent[0]], [extent[0], extent[0] - 1]]
    sc = (rng.random((P, C)) * (rng.random((P, C)) < frac)).astype(F32)
    sc += (np.arange(P * C).reshape(P, C) * 1e-7 * (sc > 0)).astype(F32)   # distinct scores
    if corner:
        sc[:6] = (0.5 + 0.4 * rng.random((6, C))).astype(F32)
    if boxes:
        wh = (rng.random((P, 2)) * 40 + 4).astype(F32)
        return np.concatenate([pts - wh / 2, pts + wh / 2], 1).astype(F32), sc
    return pts, sc


def _as_boxes(x, wh):
    return torch.from_numpy(ref.raw_boxes(x, wh))


@pytest.mark.parametrize('seed,P,C,boxes,corner,iou,max_keep', [
    (1, 300, 5, False, False, 0.01, 100), (2, 300, 5, False, False, 0.5, 7), (3, 400, 7, True, False, 0.5, 100),
    (4, 200, 4, False, True, 0.01, 100), (5, 200, 4, False, True, 0.0, 33), (6, 500, 3, True, False, 0.0, 1024),
    (7, 250, 80, False, False, 0.3, 100)])
def test_offset_branch_matches_the_oracle(seed, P, C, boxes, corner, iou, max_keep):
    wh = (32.0, 32.0)
    x, sc = _image(seed, P, C, (256.0, 256.0) if corner else (300.0, 200.0), boxes, corner)
    got = ref.image(x, sc, 0.05, iou, max_keep, wh, branch='offset')
    d, l, k, inds = op2p.multiclass_nms(_as_boxes(x, wh), torch.from_numpy(np.concatenate([sc, np.zeros((P, 1), F32)], 1)), 0.05, iou,
                                        max_keep)
    assert got['cand_count'] == len(inds) < ref.SPLIT_THR
    assert np.array_equal(got['keep'], k.numpy()) and np.array_equal(got['labels'], l.numpy())
    assert np.array_equal(got['det'], d.numpy())
    if corner:
        assert ref.slow_flag(x, sc, 0.05, wh)


@pytest.mark.parametrize('iou', [0.0, 0.01, 0.5])
def test_per_class_greedy_matches_torchvision(iou):
    import torchvision
    x, sc = _image(11, 600, 6, boxes=True, frac=0.5)
    rb = ref.raw_boxes(x)
    flat = ref.candidates(sc, 0.05)
    p, c = flat // 6, flat % 6
    ob = ref.offset_boxes(rb[p], c, ref.max_coord(rb, sc, 0.05))
    cs = sc.reshape(-1)[flat]
    for cl in range(6):
        idx = np.nonzero(c == cl)[0]
        k = ref.greedy(ob[idx], cs[idx], flat[idx], iou, 10 ** 6)
        tv = torchvision.ops.nms(torch.from_numpy(ob[idx, :4].copy()), torch.from_numpy(cs[idx]), iou).numpy()
        assert np.array_equal(k, tv), cl
        assert np.array_equal(ref.greedy(ob[idx], cs[idx], flat[idx], iou, 5), tv[:5])


@pytest.mark.parametrize('method,iou,sigma,min_score', [('linear', 0.3, 0.5, 1e-3), ('naive', 0.3, 0.5, 1e-3),
                                                        ('gaussian', 0.5, 0.5, 0.05), ('linear', 0.0, 0.5, 0.02)])
def test_soft_nms_matches_the_oracle(method, iou, sigma, min_score):
    cfg = dict(sigma=sigma, min_score=min_score, method=method)
    nms_cfg = dict(type='soft_nms', iou_threshold=iou, **cfg)
    for seed, corner in ((21, False), (22, True)):
        wh = (32.0, 32.0)
        x, sc = _image(seed, 200, 5, (256.0, 256.0) if corner else (300.0, 200.0), corner=corner, frac=0.3)
        got = ref.image(x, sc, 0.05, iou, 100, wh, cfg, branch='offset')
        d, l, k, _ = op2p.multiclass_nms(_as_boxes(x, wh), torch.from_numpy(np.concatenate([sc, np.zeros((200, 1), F32)], 1)), 0.05,
                                         iou, 100, nms_cfg=nms_cfg)
        assert np.array_equal(got['keep'], k.numpy()) and np.array_equal(got['labels'], l.numpy())
        assert np.array_equal(got['det'][:, :4], d[:, :4].numpy())
        if method == 'gaussian':               # np.exp against the oracle's: the same fp32 function, but stated as a bound
            np.testing.assert_allclose(got['det'][:, 4], d[:, 4].numpy(), rtol=1e-6)
        else:
            assert np.array_equal(got['det'][:, 4], d[:, 4].numpy())


@pytest.mark.parametrize('soft', [False, True])
def test_split_branch_matches_the_per_class_replay_and_the_oracle(soft):
    P, C = 160, 80
    x, sc = _image(31, P, C, frac=0.9)
    wh = (16.0, 16.0)
    cfg = dict(sigma=0.5, min_score=1e-3, method='linear') if soft else None
    got = ref.image(x, sc, 0.05, 0.3, 300, wh, cfg)
    assert got['cand_count'] >= ref.SPLIT_THR and got['branch'] == 'split'
    nms_cfg = None if cfg is None else dict(type='soft_nms', iou_threshold=0.3, **cfg)
    d, l, k, _ = op2p.multiclass_nms(_as_boxes(x, wh), torch.from_numpy(np.concatenate([sc, np.zeros((P, 1), F32)], 1)), 0.05, 0.3, 300,
                                     nms_cfg=nms_cfg)
    assert np.array_equal(got['keep'], k.numpy()) and np.array_equal(got['labels'], l.numpy())
    assert np.array_equal(got['det'], d.numpy())
    if not soft:
        flat = ref.candidates(sc, 0.05)
        rk = nms_replay_per_class(ref.raw_boxes(x, wh)[flat // C], sc.reshape(-1)[flat], flat % C, 0.3, 300)
        assert np.array_equal(got['keep'], rk)


def test_split_branch_differs_from_the_offset_branch_on_a_slow_image():
    """the planted case the GPU table runs with >= 10000 candidates: a class-c box in the negative corner suppresses a class c-1 box
    near max_coord in the offset branch only."""
    x, sc, wh = ref.planted_slow(P=200, C=80, many=True, seed=3)
    assert ref.slow_flag(x, sc, 0.05, wh)
    a = ref.image(x, sc, 0.05, 0.01, 100, wh, branch='offset')
    b = ref.image(x, sc, 0.05, 0.01, 100, wh)
    assert b['branch'] == 'split' and not np.array_equal(a['flat'], b['flat'])
    assert ref.expected_path(x, sc, 0.05, 'hard', wh)['path'] == 'class'
    x2, sc2, _ = ref.planted_slow(P=200, C=4, many=False, seed=3)
    assert ref.expected_path(x2, sc2, 0.05, 'hard', wh)['path'] == 'global'


def _pair(m, g, C, c):
    """a class-c box whose top-left corner is (-1 - g, -1 - g) and a class c-1 box whose bottom-right corner is the max coordinate
    (m, m): in exact arithmetic their offset boxes intersect iff g > 0."""
    x1, w = F32(-1) - F32(g), F32(20)
    boxes = np.array([[x1, x1, x1 + w, x1 + w], [m - w, m - w, m, m]], F32)
    sc = np.zeros((2, C), F32)
    sc[0, c], sc[1, c - 1] = 0.9, 0.8
    return boxes, sc


def test_slow_flag_is_conservative_on_planted_corner_layouts():
    """nms.cu prepare: `Detect conservatively` - wherever the offset branch and the class-by-class result differ, `slow` is set.
    Sweep: max coordinates 100..4000 px, C 2..81 (the class pair at the largest offset), IoU thresholds 0, 0.01 and 0.5, corner
    gaps around the 0.05 px margin and around exact touching."""
    rng = np.random.default_rng(0)
    ms = np.concatenate([[100, 255, 256, 800, 1333, 2047, 3276, 4000], rng.uniform(100, 4000, 12)]).astype(F32)
    gaps = np.concatenate([np.linspace(-0.1, 0.1, 21), -0.05 + np.arange(-4, 5) * 2.0 ** -8, [0.0, 2.0 ** -20, 1.0, 4.0]]).astype(F32)
    differ = flagged = 0
    for m in ms:
        for C in (2, 3, 31, 80, 81):
            for g in gaps:
                x, sc = _pair(m, g, C, C - 1)
                flag = ref.slow_flag(x, sc, 0.05)
                for iou in (0.0, 0.01, 0.5):
                    a = ref.image(x, sc, 0.05, iou, 100, branch='offset')
                    b = ref.image(x, sc, 0.05, iou, 100, branch='split')
                    if not np.array_equal(a['flat'], b['flat']):
                        differ += 1
                        flagged += flag
                        assert flag, (float(m), C, float(g), iou)
    assert differ > 100 and flagged == differ


def test_slow_margin_covers_the_offset_rounding():
    """the fp32 offsets fl(c * m1) and fl(x + offset) round at magnitude C * (max_coord + 1); for the largest corner x1 whose offset
    box still reaches the class c-1 box at max_coord, the margin of 0.05 px must still flag it (x1 < -0.95 and the x2 test).
    Searched over 2e5 random max coordinates per range up to 4000 px and C up to 81."""
    rng = np.random.default_rng(1)
    for C in (2, 31, 80, 81):
        for lo, hi in ((100, 400), (400, 1500), (1500, 3300), (3300, 4000)):
            m = rng.uniform(lo, hi, 200000).astype(F32)
            x1, m1 = ref.largest_reaching_x1(m, C)
            flag = (x1 < F32(-0.95)) & (m > (x1 + m1) - F32(0.05))
            assert flag.all(), (C, lo, hi)


def test_expected_path_and_the_split_thr_refusal():
    wh = (32.0, 32.0)
    x, sc = _image(41, 300, 5)
    assert ref.expected_path(x, sc, 0.05, 'hard', wh) == dict(kind='hard', path='class', slow=False, split=False, empty=False,
                                                               optin=False)
    assert ref.expected_path(x, sc * 0, 0.05, 'soft', wh)['empty']
    assert ref.soft_smem_bytes(1690) <= ref.SOFT_SMEM_DEFAULT < ref.soft_smem_bytes(1691)
    from pointtinybenchmark_b200.post_processing import check_split_thr
    check_split_thr(dict(type='nms', iou_threshold=0.5))
    check_split_thr(dict(type='nms', iou_threshold=0.5, split_thr=10000))
    with pytest.raises(NotImplementedError):
        check_split_thr(dict(type='nms', iou_threshold=0.5, split_thr=5000))


def test_gaussian_soft_nms_refuses_degenerate_boxes():
    """IoU 0/0 = NaN between two zero-area boxes: in the offset branch mmcv's gaussian weight turns disjoint boxes of DIFFERENT
    classes into NaN scores, which the per-class decomposition cannot give.  The restatement marks such images refused (as the
    kernels do); one zero-area box, or any number under the other methods, is no refusal."""
    boxes = np.array([[10, 10, 10, 30], [100, 100, 140, 100], [50, 50, 70, 70]], F32)
    sc = np.array([[0.9, 0, 0], [0, 0.8, 0], [0, 0, 0.7]], F32)
    g = dict(sigma=0.5, min_score=1e-3, method='gaussian')
    assert ref.image(boxes, sc, 0.05, 0.3, 100, soft_cfg=g)['refused']
    off = ref.image(boxes, sc, 0.05, 0.3, 100, soft_cfg=g, branch='offset')      # what refusing avoids: a NaN score
    assert off['branch'] == 'refused'
    with np.errstate(invalid='ignore'):
        d, l, k, _ = op2p.multiclass_nms(torch.from_numpy(boxes), torch.from_numpy(np.concatenate([sc, np.zeros((3, 1), F32)], 1)),
                                         0.05, 0.3, 100, nms_cfg=dict(type='soft_nms', iou_threshold=0.3, **g))
    assert torch.isnan(d[:, 4]).any()
    for method in ('naive', 'linear'):
        r = ref.image(boxes, sc, 0.05, 0.3, 100, soft_cfg=dict(g, method=method))
        assert not r['refused'] and np.array_equal(r['labels'], [0, 1, 2])
    assert not ref.image(boxes[[0, 2]], sc[[0, 2]], 0.05, 0.3, 100, soft_cfg=g)['refused']
    assert ref.degenerate(np.array([[0, 0, 1, 1, -1.0]], F32)) == 2
