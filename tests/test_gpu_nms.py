"""GPU: the multiclass NMS and soft-NMS kernels of csrc/nms.cu against the host restatement of tests/nms_ref.py, one row per case:

  prepare   nms_prepare_kernel's 1024-wide scan chunks (P = 1023, 1024, 1025, 4096), candidate counts, max_coord, the `slow` flag
  class     nms_class_kernel: bitonic sort up to 4096 keys, greedy batches of 32, the break at max_per_img (1, 31, 32, 33, 100, 1024,
            with classes of more survivors than that); soft_nms_class_kernel on both sides of the 48 KB shared-memory default (P 1690 / 1691, dynamic +
            static)
  merge     nms_merge_kernel's warp stride over C (1, 2, 31, 32, 33, 80, 81), exact cross-class score ties (broken by flat id)
  global    nms_global_kernel / soft_nms_global_kernel on `slow` images with fewer than 10000 candidates; `slow` images with more
            take the class-by-class path (mmcv's split branch); batches mixing slow, fast and empty images
  edges     scores exactly at score_thr, IoU exactly at iou_thr (hard NMS suppresses on >, soft-NMS decays on >=), iou_thr = 0 with
            touching boxes, zero-area boxes, an image whose classes meet only through the fp32 rounding of the class offset

Every row: count, cand_count, keep and labels equal to the restatement, boxes bit-equal, scores bit-equal (hard, naive, linear) or,
for gaussian (the kernel's expf against numpy's exp), within 4 ulp per decay, i.e. 4 (k + 1) ulp at row k, with keep, labels and
boxes exact on every row before the first decision the restatement finds within 1e-5 relative (nms_ref.NEAR), nothing written
past count, and two back-to-back calls identical.  Gaussian soft-NMS on an image with two zero-area (or one negative-area)
candidate boxes is refused - IoU 0/0 = NaN - and those rows check that the op raises, naming exactly the refused images."""
import re
from typing import NamedTuple, Tuple

import numpy as np
import pytest
import torch

from tests import nms_ref as ref

F32 = np.float32


class Case(NamedTuple):
    name: str
    kind: str                    # 'hard' or a soft method
    P: int
    C: int
    layouts: Tuple[str, ...]     # one per image, see _layout
    max_keep: int = 100
    iou: float = 0.5
    thr: float = 0.05
    boxes: bool = False          # explicit boxes (ptb_multiclass_nms_boxes / soft with boxes) instead of pseudo boxes
    wh: Tuple[float, float] = (32.0, 32.0)
    sigma: float = 0.5
    min_score: float = 1e-3
    seed: int = 0


def _cases():
    out = []
    for P in (1, 31, 32, 33, 1023, 1024, 1025, 4096):
        out.append(Case(f'P{P}', 'hard', P, 3, ('rand', 'rand'), seed=P))
    for C in (1, 2, 31, 32, 33, 80, 81):
        out.append(Case(f'C{C}', 'hard', 300, C, ('rand',), iou=0.01, seed=100 + C))
    for mk in (1, 31, 32, 33, 100, 1024):
        out.append(Case(f'max{mk}', 'hard', 2000, 2, ('dense',), max_keep=mk, wh=(8.0, 8.0), seed=200 + mk))
        out.append(Case(f'max{mk}_linear', 'linear', 1500, 2, ('dense',), max_keep=mk, wh=(8.0, 8.0), iou=0.3, seed=300 + mk))
    out += [
        Case('max1024_P4096_C1', 'hard', 4096, 1, ('dense',), max_keep=1024, wh=(8.0, 8.0), seed=7),
        Case('empty_batch', 'hard', 64, 5, ('empty', 'empty')),
        Case('empty_soft', 'linear', 64, 5, ('empty', 'rand')),
        Case('mixed_hard', 'hard', 200, 4, ('rand', 'slow', 'empty', 'slow'), iou=0.01, seed=11),
        Case('mixed_linear', 'linear', 200, 4, ('slow', 'rand', 'slow', 'empty'), iou=0.3, seed=12),
        Case('mixed_gaussian', 'gaussian', 200, 4, ('slow', 'rand'), iou=0.3, seed=13),
        Case('mixed_naive', 'naive', 200, 4, ('rand', 'slow'), iou=0.3, seed=14),
        Case('slow_many_hard', 'hard', 160, 80, ('slow_many', 'slow', 'rand'), iou=0.01, seed=15),
        Case('slow_many_linear', 'linear', 160, 80, ('slow_many', 'rand'), iou=0.1, seed=16),
        Case('slow_many_naive', 'naive', 160, 80, ('slow_many',), iou=0.1, seed=17),
        Case('boxes_hard', 'hard', 500, 7, ('boxes', 'boxes_neg'), boxes=True, seed=18),
        Case('boxes_gaussian', 'gaussian', 400, 7, ('boxes', 'boxes_neg'), boxes=True, iou=0.3, seed=19),
        Case('boxes_naive', 'naive', 400, 7, ('boxes',), boxes=True, iou=0.3, seed=20),
        Case('wh_24x10', 'hard', 700, 5, ('rand', 'rand'), wh=(24.0, 10.0), iou=0.2, seed=21),
        Case('wh_24x10_linear', 'linear', 700, 5, ('rand',), wh=(24.0, 10.0), iou=0.2, seed=22),
        Case('soft_P1690', 'linear', 1690, 2, ('rand',), seed=23),
        Case('soft_P1691', 'linear', 1691, 2, ('rand',), seed=24),
        Case('soft_P1694', 'linear', 1694, 2, ('rand',), seed=39),
        Case('soft_P1695', 'gaussian', 1695, 2, ('rand',), seed=40),
        Case('soft_P4096_naive', 'naive', 4096, 1, ('dense',), max_keep=1024, wh=(8.0, 8.0), seed=25),
        Case('soft_P4096_gaussian', 'gaussian', 4096, 2, ('rand',), seed=26),
        Case('thr_equal', 'hard', 300, 6, ('thr_eq',), thr=0.25, seed=27),
        Case('thr_equal_linear', 'linear', 300, 6, ('thr_eq',), thr=0.25, seed=28),
        Case('iou_equal_hard', 'hard', 64, 3, ('iou_eq',), iou=1 / 3, seed=29),
        Case('iou_equal_naive', 'naive', 64, 3, ('iou_eq',), iou=1 / 3, seed=30),
        Case('iou_equal_linear', 'linear', 64, 3, ('iou_eq',), iou=1 / 3, seed=31),
        Case('ties', 'hard', 400, 33, ('ties',), iou=0.3, seed=32),
        Case('ties_linear', 'linear', 400, 33, ('ties',), iou=0.3, seed=33),
        Case('zero_area', 'hard', 300, 4, ('zero', 'zero'), boxes=True, iou=0.0, seed=34),
        Case('zero_area_linear', 'linear', 300, 4, ('zero',), boxes=True, iou=0.3, seed=35),
        Case('zero_area_naive', 'naive', 300, 4, ('zero', 'zero1'), boxes=True, iou=0.3, seed=41),
        Case('zero_area_gaussian', 'gaussian', 300, 4, ('boxes', 'zero', 'zero1'), boxes=True, iou=0.3, seed=42),
        Case('one_zero_area_gaussian', 'gaussian', 300, 4, ('zero1', 'zero1'), boxes=True, iou=0.3, seed=43),
        Case('slow_zero_area_gaussian', 'gaussian', 200, 4, ('slow_zero', 'slow_zero1'), boxes=True, iou=0.3, seed=44),
        Case('wh_0x8_gaussian', 'gaussian', 100, 3, ('rand', 'rand'), wh=(0.0, 8.0), iou=0.3, seed=45),
        Case('iou0_touching', 'hard', 256, 3, ('touch',), boxes=True, iou=0.0, seed=36),
        Case('iou0_touching_linear', 'linear', 256, 3, ('touch',), boxes=True, iou=0.0, seed=37),
        Case('offset_rounding', 'hard', 2, 80, ('rounding',), boxes=True, iou=0.0, seed=38),
    ]
    return out


CASES = _cases()


def rounding_pair(C=80):
    """(max coordinate m, corner x1) of the worst fp32 class offset at C classes: the corner box of class C-1 and the box of class
    C-2 ending at (m, m) intersect after the offset although x1 > -1 (so x2 = m < x1 + m + 1 in exact arithmetic).  The 0.05 px
    margin of nms_prepare_kernel still flags the image; without it the image would take the per-class path."""
    m = np.random.default_rng(1).uniform(1000, 1700, 200000).astype(F32)
    x1, m1 = ref.largest_reaching_x1(m, C)
    ok = (x1 > F32(-1)) & (m <= (x1 + m1))
    i = int(np.nonzero(ok)[0][0])
    return m[i], x1[i]


def _layout(kind, rng, P, C, wh, thr):
    """(pts (P,2) or boxes (P,4), scores (P,C)) of one image."""
    def distinct(sc):
        return (sc + np.arange(P * C).reshape(P, C) * 1e-7 * (sc > 0)).astype(F32)
    sc = distinct(rng.random((P, C)) * (rng.random((P, C)) < 0.3))
    pts = (rng.random((P, 2)) * [300.0, 200.0]).astype(F32)
    if kind == 'rand':
        return pts, sc
    if kind == 'empty':
        return pts, (rng.random((P, C)) * thr).astype(F32)
    if kind == 'dense':                                                   # almost every candidate survives: > max_keep per class
        return (rng.random((P, 2)) * 3000).astype(F32), distinct(0.1 + 0.9 * rng.random((P, C)) * (rng.random((P, C)) < 0.85))
    if kind in ('slow', 'slow_many'):
        x, s, _ = ref.planted_slow(P, C, kind == 'slow_many', int(rng.integers(1 << 30)))
        return x, s
    if kind == 'thr_eq':                                                  # exactly at score_thr: not a candidate; one ulp above: one
        t = F32(thr)
        sc[rng.random((P, C)) < 0.3] = t
        sc[rng.random((P, C)) < 0.1] = np.nextafter(t, F32(1))
        return pts, sc
    if kind == 'iou_eq':                                                  # pairs 16 px apart: IoU of the 32 x 32 boxes = 1/3 exactly
        base = np.stack([np.arange(P) % 8 * 100.0, np.arange(P) // 8 * 100.0], 1)
        base[1::2, 0] = base[0::2, 0] + 16
        s = distinct(0.3 + 0.6 * rng.random((P, C)))
        return base.astype(F32), s
    if kind == 'ties':                                                    # scores on a 1/16 grid: exact ties within and across classes
        s = (np.floor(rng.random((P, C)) * 16) / 16 * (rng.random((P, C)) < 0.3)).astype(F32)
        s[0, :] = F32(0.5)
        return pts, s
    if kind in ('slow_zero', 'slow_zero1'):                               # the `slow` layout as explicit boxes, 2 / 1 zero-area
        x, s, wh = ref.planted_slow(P, C, False, int(rng.integers(1 << 30)))
        bx = ref.raw_boxes(x, wh)
        bx[10, 2] = bx[10, 0]
        s[10] = 0                                                         # one candidate class per zero-area box: every (box, class)
        s[10, 0] = F32(0.6)                                               # candidate counts
        if kind == 'slow_zero':
            bx[11, 3] = bx[11, 1]
            s[11] = 0
            s[11, 1] = F32(0.55)
        return bx, s
    if kind in ('boxes', 'boxes_neg', 'zero', 'zero1', 'touch'):
        c = (rng.random((P, 2)) * [400.0, 260.0]).astype(F32)
        if kind == 'boxes_neg':
            c -= F32(30)
        b = (rng.random((P, 2)) * 40 + 6).astype(F32)
        bx = np.concatenate([c - b / 2, c + b / 2], 1).astype(F32)
        if kind == 'zero':                                                # points, segments and repeated zero-area boxes
            bx[::3, 2] = bx[::3, 0]
            bx[1::3, 3] = bx[1::3, 1]
            bx[2::9] = bx[2]
            bx[2::9, 2:] = bx[2, :2]
        if kind == 'zero1':                                               # exactly one zero-area candidate box
            bx[7, 2] = bx[7, 0]
            sc[7] = 0
            sc[7, 0] = F32(0.6)
        if kind == 'touch':                                               # a grid of 20 x 20 boxes sharing edges
            g = np.arange(P)
            x0, y0 = (g % 16 * 20).astype(F32), (g // 16 * 20).astype(F32)
            bx = np.stack([x0, y0, x0 + 20, y0 + 20], 1).astype(F32)
            sc = distinct(0.1 + 0.9 * rng.random((P, C)))
        return bx, sc
    if kind == 'rounding':
        m, x1 = rounding_pair(C)
        w = F32(20)
        bx = np.array([[x1, x1, x1 + w, x1 + w], [m - w, m - w, m, m]], F32)
        s = np.zeros((P, C), F32)
        s[0, C - 1], s[1, C - 2] = F32(0.9), F32(0.8)
        return bx, s
    raise KeyError(kind)


def make(case):
    rng = np.random.default_rng(case.seed)
    xs, ss = zip(*[_layout(k, rng, case.P, case.C, case.wh, case.thr) for k in case.layouts])
    return np.stack(xs), np.stack(ss)


def soft_cfg(case):
    return None if case.kind == 'hard' else dict(sigma=case.sigma, min_score=case.min_score, method=case.kind)


def expected(case, x, s):
    wh = None if case.boxes else case.wh
    return [ref.image(x[b], s[b], case.thr, case.iou, case.max_keep, wh, soft_cfg(case)) for b in range(len(s))]


def paths(case, x, s):
    wh = None if case.boxes else case.wh
    return [ref.expected_path(x[b], s[b], case.thr, 'hard' if case.kind == 'hard' else 'soft', wh) for b in range(len(s))]


def _run(ops, case, x, s):
    xt, st = torch.from_numpy(x).cuda(), torch.from_numpy(s).cuda()
    if case.kind == 'hard':
        if case.boxes:
            return ops.multiclass_nms_boxes(xt, st, case.thr, case.iou, case.max_keep)
        return ops.multiclass_nms(xt, st, case.wh, case.thr, case.iou, case.max_keep)
    return ops.multiclass_soft_nms(xt, st, None if case.boxes else case.wh, case.thr, case.iou, case.max_keep, case.sigma,
                                   case.min_score, case.kind)


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_nms_kernels_match_the_restatement(ops, case):
    x, s = make(case)
    rs = expected(case, x, s)
    refused = [b for b, r in enumerate(rs) if r['refused']]
    if refused:                                   # gaussian with degenerate boxes: the kernels set count -1, the op raises
        for _ in range(2):
            with pytest.raises(RuntimeError, match=re.escape(f'refused image(s) {refused}')):
                _run(ops, case, x, s)
        return
    out = [t.cpu() for t in _run(ops, case, x, s)]
    again = [t.cpu() for t in _run(ops, case, x, s)]
    for a, b in zip(out, again):
        assert torch.equal(a, b), f'{case.name}: two calls differ'
    cnt, det, lab, keep, cc = [t.numpy() for t in out]
    for b, r in enumerate(rs):
        what = f'{case.name} image {b} ({case.layouts[b]})'
        assert int(cc[b]) == r['cand_count'], what
        n = int(cnt[b])
        if r['all_exact']:
            assert n == r['count'], (what, n, r['count'])
        e = min(r['exact_upto'], n)                 # every row but the gaussian method's undecided tail
        assert np.array_equal(keep[b, :e], r['keep'][:e]), what
        assert np.array_equal(lab[b, :e], r['labels'][:e]), what
        assert np.array_equal(det[b, :e, :4], r['det'][:e, :4]), what
        if case.kind == 'gaussian':                 # row k has been decayed at most k times: 4 ulp per expf and product
            tol = 4 * 2.0 ** -23 * (np.arange(e) + 1) * np.abs(r['det'][:e, 4].astype(np.float64))
            assert (np.abs(det[b, :e, 4].astype(np.float64) - r['det'][:e, 4]) <= tol).all(), what
        else:
            assert np.array_equal(det[b, :n, 4], r['det'][:, 4]), what
        assert not det[b, n:].any() and not lab[b, n:].any() and not keep[b, n:].any(), f'{what}: written past count'


def test_the_table_reaches_every_path():
    """every (kind, kernel path) pair of expected_path, the slow images above 10000 candidates, the soft class kernel with and
    without the shared-memory opt-in, empty images of both kinds, and a batch mixing slow, fast and empty images."""
    seen = set()
    for case in CASES:
        x, s = make(case)
        ps = paths(case, x, s)
        for p in ps:
            seen.add((p['kind'], p['path']))
            if p['slow'] and p['split']:
                seen.add((p['kind'], 'slow_split'))
            if p['empty']:
                seen.add((p['kind'], 'empty'))
            if p['kind'] == 'soft' and p['path'] == 'class' and not p['empty']:
                seen.add(('soft', 'optin' if p['optin'] else 'default_smem'))
        if {p['path'] for p in ps} == {'class', 'global'} and any(p['empty'] for p in ps):
            seen.add((ps[0]['kind'], 'mixed'))
        if case.kind == 'gaussian':
            for p, r in zip(ps, expected(case, x, s)):
                seen.add(('gaussian', ('refused_' if r['refused'] else 'accepted_') + p['path']))
    want = {(k, p) for k in ('hard', 'soft') for p in ('class', 'global', 'slow_split', 'empty', 'mixed')}
    want |= {('soft', 'optin'), ('soft', 'default_smem')}
    want |= {('gaussian', a + p) for a in ('refused_', 'accepted_') for p in ('class', 'global')}
    assert want <= seen, sorted(want - seen)
    x, s = make(next(c for c in CASES if c.name == 'offset_rounding'))
    assert ref.slow_flag(x[0], s[0], 0.05)
    a = ref.image(x[0], s[0], 0.05, 0.0, 100, branch='offset')
    b = ref.image(x[0], s[0], 0.05, 0.0, 100, branch='split')
    assert a['count'] != b['count'], 'the rounding case must separate the two branches'


@pytest.mark.gpu
def test_refusals_are_host_errors(ops):
    from pointtinybenchmark_b200 import _lib
    dev = torch.device('cuda:0')
    pts = torch.rand(1, 4097, 2, device=dev) * 100
    sc = torch.rand(1, 4097, 3, device=dev)
    with pytest.raises(RuntimeError, match='4096'):
        ops.multiclass_nms(pts, sc, (32, 32), 0.05, 0.5, 100)
    with pytest.raises(RuntimeError, match='4096'):
        ops.multiclass_soft_nms(pts, sc, (32, 32), 0.05, 0.5, 100)
    pts, sc = pts[:, :100].contiguous(), sc[:, :100].contiguous()
    for mk in (0, 1025):
        with pytest.raises(RuntimeError, match='max_per_img'):
            ops.multiclass_nms(pts, sc, (32, 32), 0.05, 0.5, mk)
        with pytest.raises(RuntimeError, match='max_per_img'):
            ops.multiclass_soft_nms(pts, sc, (32, 32), 0.05, 0.5, mk)
    with pytest.raises(RuntimeError, match='iou_thr'):
        ops.multiclass_nms(pts, sc, (32, 32), 0.05, -0.1, 100)
    with pytest.raises(RuntimeError, match='iou_thr'):
        ops.multiclass_soft_nms(pts, sc, (32, 32), 0.05, 0.0, 100, method='naive')
    lib = _lib.load()
    B, P, C = 1, 100, 3
    out = [torch.zeros(n, dtype=dt, device=dev) for n, dt in ((B, torch.int32), (B * 100 * 5, torch.float32), (B * 100, torch.int32),
                                                              (B * 100, torch.int32), (B, torch.int32))]
    boxes = torch.cat([pts - 16, pts + 16], -1).contiguous()
    need = lib.ptb_multiclass_nms_workspace(B, P, C)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    outs = [ops._ptr(t) for t in out]
    for fn, args in ((lib.ptb_multiclass_nms, [ops._ptr(pts), ops._ptr(sc), B, P, C, 32.0, 32.0, 0.05, 0.5, 100]),
                     (lib.ptb_multiclass_nms_boxes, [ops._ptr(boxes), ops._ptr(sc), B, P, C, 0.05, 0.5, 100])):
        assert fn(*args, *outs, ops._ptr(ws), need - 1, ops._stream()) != 0
        assert 'workspace' in lib.ptb_last_error().decode()
    need = lib.ptb_multiclass_soft_nms_workspace(B, P, C)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    args = [ops._ptr(pts), None, ops._ptr(sc), B, P, C, 32.0, 32.0, 0.05, 0.5, 0.5, 1e-3, 1, 100] + [ops._ptr(t) for t in out]
    assert lib.ptb_multiclass_soft_nms(*args, ops._ptr(ws), need - 1, ops._stream()) != 0
    assert 'workspace' in lib.ptb_last_error().decode()
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_p2p_head_get_bboxes_on_a_square_image_matches_the_restatement(ops):
    """P2PHead.get_bboxes at 80 classes on a 640 x 640 meta: points clamped into both extreme corners make the image `slow`, and
    tens of thousands of candidates put it on mmcv's split branch; the head's NMS output equals the restatement's on the head's
    own top-k points and scores."""
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    from tests.test_gpu_p2p import head_cfg
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(640)
    H = W = 80
    cls_out = torch.randn(2, 80, H, W, generator=g) - 0.5
    pts_out = torch.randn(2, 2, H, W, generator=g) * 3
    cls_out[:, :, 0, 0] += 5                              # one point pushed past each extreme corner, both in the top-k
    cls_out[:, :, H - 1, W - 1] += 5
    pts_out[:, :, 0, 0], pts_out[:, :, H - 1, W - 1] = -5, 5
    cls_out, pts_out = cls_out.to(dev), pts_out.to(dev)
    metas = [dict(img_shape=(640, 640, 3), pad_shape=(640, 640, 3), ori_shape=(640, 640, 3), scale_factor=np.ones(4, F32))] * 2
    hc = head_cfg(dict(num_classes=80, C=32, stride=8), 0.01)
    head = build_head(hc).cuda().eval()
    res, aux = head.get_bboxes([cls_out], [pts_out], metas, return_all=True)
    cfg = hc['test_cfg']
    pts, sc = aux['pts'].cpu().numpy(), aux['scores'].cpu().numpy()
    for b in range(2):
        r = ref.image(pts[b], sc[b], cfg['score_thr'], 0.01, cfg['max_per_img'], cfg['pseudo_wh'])
        assert ref.slow_flag(pts[b], sc[b], cfg['score_thr'], cfg['pseudo_wh']) and r['branch'] == 'split', b
        n = int(aux['count'][b])
        assert int(aux['cand_count'][b]) == r['cand_count'] and n == r['count']
        assert np.array_equal(aux['keep'][b, :n].cpu().numpy(), r['keep'])
        assert np.array_equal(res[b][1].cpu().numpy(), r['labels'])
        assert np.array_equal(res[b][0][:, 4].cpu().numpy(), r['det'][:, 4])
