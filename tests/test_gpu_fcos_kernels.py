"""GPU: the FCOS kernels (csrc/fcos.cu) through the ops.fcos_* wrappers, against the host references of tests/fcos_ref.py.

  * fcos_targets         labels and targets bit for bit at 1, 2, 5 and 8 levels, odd strides (3, 5, 12), B = 1 to 3 with an image without
                         GTs in the middle and a batch without any, 1 to 300 GTs, up to 511 classes, centre sampling, norm_on_bbox, GTs
                         planted on grid points, on the ends of the ranges, of equal area over one point, of area 1e8 (INF) and above,
                         and at one trip of the grid-stride loop (16 x SMs x 256 rows) - 1, + 0, + 1 and past two trips.
  * fcos_norm_sums       the positive count exactly and the centerness sum bit for bit against fixed_order_sum, at the sizes where the
                         fixed 528 x 256 sum grid changes shape.
  * fcos_bbox_loss       linear IoU and GIoU sums bit for bit against fixed_order_sum(box_terms_f32); the log-IoU sum within
                         (n_add + 3) u sum|terms|; every gradient component within gamma_K S of box_grad64 (GRAD_K below); negative rows
                         exactly 0; identical bits over two calls.  Random, zero, negative and planted dyadic distances (every max / min
                         tie, touching and apart boxes, union, iou and enclose exactly at and below eps = 2^-20).
  * fcos_centerness_loss the gradient bit for bit against ctr_grad_f32; the sum within the bound of CTR_PIECE_K below.
  * fcos_decode          idx, boxes, scores and centerness bit for bit at 1, 5 and 8 levels, C = 1 to 511 (the lane loops' edges), three
                         images of distinct shapes and rescale factors, nms_pre from -1 to H*W + 1 and 4096, with large groups of equal
                         keys; idx against torch.topk as sets within equal keys.
  * refusals             0 and 9 levels, nms_pre > 4096 where it would select, maps that are not channels-last.
The largest errors seen are printed."""
import numpy as np
import pytest
import torch

from tests import fcos_ref as ref
from tests.p2p_loss_ref import SUM_GRID, fixed_order_sum
from tests.test_gpu_p2p_loss_kernels import PLANTED

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
U = ref.U
# Box-loss gradient: the longest chain of fp32 roundings from the kernel's fp32 intermediates to one chain-rule product of a gradient
# component is 10 (log IoU, the product g_iou * (iou / uc) through g_uni, g_ov and g_iw): iou = ov / uc (1), g_iou = -1 / ic (1),
# -iou / uc (1), g_iou * that (1), g_ov's subtraction (1), * ih (1), the two additions into gx1 (2), s = sc * w (1), -s * gx1 (1).
# Every other product has fewer (GIoU's enclose term 6, its g_union term 9).  With |delta| <= u per rounding the error of a sum of such
# products is at most gamma_10 = 10 u / (1 - 10 u) times S, the sum of their magnitudes; FMA contraction only removes roundings.
GRAD_K = 10
# Centerness BCE term (1 - t) x - (min(x, 0) - log1pf(expf(-|x|))): fl(1 - t) and the product (2u |a|), expf within 2 ulp and log1pf
# within 1 ulp (3u of log1p(e)), the inner and the outer subtraction (u each of the pieces): at most 5u times the pieces' magnitudes,
# and 6u covers the second-order terms.
CTR_PIECE_K = 6
SIZES = [1, SUM_GRID - 1, SUM_GRID, SUM_GRID + 1, 3 * SUM_GRID + 7]

_worst = {}


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    yield
    for k in sorted(_worst):
        print(f'[max error] {k}: {_worst[k]:.3e}')


def _note(key, e):
    _worst[key] = max(_worst.get(key, 0.0), e)


def _trip():
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * 256


def _poison(*shapes):
    """fill freed blocks of these sizes, so an output row a kernel leaves unwritten cannot hold an earlier call's right answer"""
    ts = [torch.full(s, float('nan'), device=DEV) for s in shapes]
    torch.cuda.synchronize()
    del ts


# ---------------------------------------------------------------------------------------------------------------------------------
# targets
def run_targets(ops, c):
    gts = [(g, l) for g, l in zip(c['gts'], c['gls']) if len(g)]
    gt = torch.cat([g for g, _ in gts]).to(DEV).contiguous() if gts else None
    gl = torch.cat([l for _, l in gts]).to(DEV).contiguous() if gts else None
    off = torch.tensor(np.concatenate([[0], np.cumsum([len(g) for g in c['gts']])]).astype(np.int32), device=DEV)
    ranges = torch.tensor(c['ranges'], dtype=torch.float32, device=DEV)
    radius = None
    if c['radius'] is not None:
        radius = torch.tensor([float(np.float32(s * c['radius'])) for s in c['strides']], dtype=torch.float32, device=DEV)
    N = c['B'] * sum(h * w for h, w in c['sizes'])
    _poison((N * 2,), (N * 4,))
    return ops.fcos_targets(c['sizes'], c['strides'], c['B'], gt, gl, off, ranges, radius, c['norm'], c['C'])


def check_targets(ops, c):
    lab, tgt = run_targets(ops, c)
    want_l, want_t = ref.targets(c['sizes'], c['strides'], c['gts'], c['gls'], c['ranges'], c['radius'], c['norm'], c['C'])
    bad = torch.nonzero(lab.cpu() != want_l).flatten()
    assert bad.numel() == 0, f'{bad.numel()} labels differ, first rows {bad[:6].tolist()}'
    bad = torch.nonzero((tgt.cpu() != want_t).any(1)).flatten()
    assert bad.numel() == 0, f'{bad.numel()} target rows differ, first rows {bad[:6].tolist()}'
    return want_l


@pytest.mark.parametrize('kind', ['one_level', 'odd_strides', 'crowded', 'eight_levels', 'no_gt', 'planted', 'planted_cs'])
def test_targets_bit_exact(ops, kind):
    c = ref.target_case(kind)
    lab = check_targets(ops, c)
    if kind != 'no_gt':
        assert bool(((lab >= 0) & (lab < c['C'])).any())


def test_targets_of_a_batch_without_gts(ops):
    c = ref.target_case('no_gt')
    lab, tgt = run_targets(ops, c)
    assert bool((lab == c['C']).all()) and bool((tgt == 0).all())


@pytest.mark.parametrize('where', [-1, 0, 1, 'two'])
def test_targets_around_the_grid_stride_trip(ops, where):
    trip = _trip()
    N = 2 * trip + 5 if where == 'two' else trip + where
    sizes, strides = ref.trip_sizes(N)
    g = torch.Generator().manual_seed(N)
    ext = (sizes[0][1] * strides[0], sizes[0][0] * strides[0])
    gt, gl = ref._random_gts(g, 40, ext, 3, lo=8.0, hi=400.0)
    tail = torch.tensor([[0.0, 0.0, sizes[-1][1] * strides[-1] + 40.0, 24.0]])   # over the last level's row, to its last point
    c = dict(sizes=sizes, strides=strides, B=1, gts=[torch.cat([gt, tail])], gls=[torch.cat([gl, torch.tensor([2])]).long()],
             ranges=[(-1, 64), (64, ref.ofc.INF)], radius=None, norm=False, C=3)
    lab = check_targets(ops, c)
    assert int(lab.numel()) == N and bool((lab[-4:] == 2).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# loss normalisers
@pytest.mark.parametrize('N', SIZES)
def test_norm_sums_exact(ops, N):
    g = torch.Generator().manual_seed(N)
    C = 4
    lab = torch.randint(-1, C + 1, (N,), generator=g)
    tgt = torch.exp(torch.randn(N, 4, generator=g)) * 20
    out = ops.fcos_norm_sums(lab.to(DEV), tgt.to(DEV), C).cpu().numpy()
    cnt, s = ref.norm_sums(lab, tgt, C)
    assert out[0] == np.float32(cnt), (float(out[0]), cnt)
    assert out[1].tobytes() == np.float32(s).tobytes(), (float(out[1]), float(s))


# ---------------------------------------------------------------------------------------------------------------------------------
# box and centerness losses
def loss_case(sizes, strides, B, C, seed, plant):
    """pred / target distances (N, 4) fp32 and labels (N,) of a batch: random positive distances, some rows zero (ReLU) or negative
    in a column, 15 % negatives labelled C or -1; with plant, planted_box_rows at the first cells of level 0 of every image"""
    g = torch.Generator().manual_seed(seed)
    N = B * sum(h * w for h, w in sizes)
    st = torch.cat([torch.full((B * h * w,), float(s)) for (h, w), s in zip(sizes, strides)])
    pred = (torch.exp(torch.randn(N, 4, generator=g) * 0.6) * st[:, None] * 2).numpy()
    tgt = (torch.exp(torch.randn(N, 4, generator=g) * 0.6) * st[:, None] * 2).numpy()
    r = torch.rand(N, generator=g).numpy()
    col = torch.randint(0, 4, (N,), generator=g).numpy()
    pred[r < 0.04] = 0.0
    pred[(r >= 0.04) & (r < 0.08), col[(r >= 0.04) & (r < 0.08)]] *= -0.3
    same = (r >= 0.08) & (r < 0.1)
    pred[same] = tgt[same]
    lab = torch.randint(0, C, (N,), generator=g).numpy()
    neg = torch.rand(N, generator=g).numpy() < 0.15
    lab[neg] = np.where(torch.rand(N, generator=g).numpy()[neg] < 0.5, C, -1)
    if plant:
        pp, pt = ref.planted_box_rows()
        hw0 = sizes[0][0] * sizes[0][1]
        for b in range(B):
            rows = b * hw0 + np.arange(len(pp))
            pred[rows], tgt[rows], lab[rows] = pp, pt, np.arange(len(pp)) % C
    return pred.astype(np.float32), tgt.astype(np.float32), lab.astype(np.int64)


def check_box_loss(ops, mode, sizes, strides, B, C, pred, tgt, lab, oeps, eps, key):
    pd, td, ld = (torch.from_numpy(a).to(DEV) for a in (pred, tgt, lab))
    call = lambda **kw: ops.fcos_bbox_loss(pd, td, ld, sizes, strides, B, C, ref.MODES[mode], oeps, eps, **kw)
    s1, s2 = call(), call()
    assert torch.equal(s1, s2), 'two sums differ'
    got = np.float32(s1.cpu().numpy()[0])
    pts = ref.row_points(sizes, strides, B)
    terms = ref.box_terms_f32(pts, pred, tgt, lab, C, mode, oeps, eps)
    if mode == 'log':
        # each term: logf within 1 ulp (2u) and the product with w (u); the sum: u per addition on its longest chain
        want = float(terms.sum())
        bound = (ref.sum_chain(len(terms)) + 3) * U * float(np.abs(terms).sum())
        e = abs(float(got) - want)
        _note(f'box {key} sum / bound', e / max(bound, 1e-300))
        assert e <= bound, (float(got), want, bound)
    else:
        want = fixed_order_sum(terms)
        assert got.tobytes() == want.tobytes(), (float(got), float(want))
    sc = torch.tensor([0.75], device=DEV)
    _poison(tuple(pred.shape))
    g1 = call(scale=sc, want_grad=True)
    g2 = call(scale=sc, want_grad=True)
    assert torch.equal(g1, g2), 'two gradients differ'
    g = g1.cpu().double().numpy()
    want_g, S = ref.box_grad64(pts, pred, tgt, lab, C, mode, oeps, eps, scale=0.75)
    gamma = GRAD_K * U / (1 - GRAD_K * U)
    err = np.abs(g - want_g)
    bound = gamma * S + GRAD_K * 2.0 ** -149
    _note(f'box {key} grad / (gamma_K S)', float((err / np.maximum(bound, 1e-300)).max()))
    bad = np.argwhere(err > bound)
    assert bad.size == 0, f'{len(bad)} gradient components out of bound, first {bad[:4].tolist()}: {g[tuple(bad[0])]} vs {want_g[tuple(bad[0])]}'
    neg = ~ref.positive(lab, C)
    assert np.all(g[neg] == 0)


@pytest.mark.parametrize('mode', ['log', 'linear', 'giou'])
@pytest.mark.parametrize('N', SIZES)
def test_box_loss_at_the_sum_grid_sizes(ops, mode, N):
    sizes, strides = ref.trip_sizes(N)
    pred, tgt, lab = loss_case(sizes, strides, 1, 3, N, plant=N > 100)
    check_box_loss(ops, mode, sizes, strides, 1, 3, pred, tgt, lab, 1e-6, 1e-6, mode)


@pytest.mark.parametrize('mode', ['log', 'linear', 'giou'])
def test_box_loss_planted_ties_over_levels_and_images(ops, mode):
    """B = 3 over 5 levels of odd shapes, so fcos_point's split of a row into (level, image, cell) meets the reference's points;
    eps = 2^-20 for the union clamp and the IoU / enclose clamps, where the planted rows sit exactly"""
    sizes, strides = [(32, 40), (16, 20), (9, 10), (5, 5), (3, 3)], [8, 16, 32, 64, 128]
    pred, tgt, lab = loss_case(sizes, strides, 3, 7, 11, plant=True)
    eps = ref.PLANT_EPS
    check_box_loss(ops, mode, sizes, strides, 3, 7, pred, tgt, lab, eps, eps, mode + ' planted')


@pytest.mark.parametrize('N', SIZES)
def test_centerness_loss(ops, N):
    g = torch.Generator().manual_seed(N + 1)
    C = 2
    x = (torch.randn(N, generator=g) * 4).numpy().astype(np.float32)
    if N >= len(PLANTED):
        x[:len(PLANTED)] = PLANTED
    tgt = (torch.exp(torch.randn(N, 4, generator=g)) * 10).numpy().astype(np.float32)
    lab = torch.randint(-1, C + 1, (N,), generator=g).numpy()
    xd, td, ld = (torch.from_numpy(a).to(DEV) for a in (x, tgt, lab))
    call = lambda **kw: ops.fcos_centerness_loss(xd, td, ld, C, **kw)
    s1, s2 = call(), call()
    assert torch.equal(s1, s2)
    terms, pieces = ref.ctr_terms64(x, tgt, lab, C)
    bound = CTR_PIECE_K * U * float(pieces.sum()) + ref.sum_chain(N) * U * float(np.abs(terms).sum())
    e = abs(float(s1.cpu()[0]) - float(terms.sum()))
    _note('centerness sum / bound', e / max(bound, 1e-300))
    assert e <= bound, (float(s1.cpu()[0]), float(terms.sum()), bound)
    sc = torch.tensor([0.75], device=DEV)
    _poison((N,))
    g1, g2 = call(scale=sc, want_grad=True), call(scale=sc, want_grad=True)
    assert torch.equal(g1, g2)
    want = ref.ctr_grad_f32(x, tgt, lab, C, scale=0.75)
    got = g1.cpu().numpy()
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, f'{bad.size} gradients differ, first {bad[:4].tolist()}: {got[bad[:2]]} vs {want[bad[:2]]}'


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
LEVEL_SIZES = [(40, 52), (20, 26), (10, 13), (5, 7), (3, 4), (2, 2), (1, 1), (1, 2)]
LEVEL_STRIDES = [8, 16, 32, 64, 128, 256, 512, 1024]


def decode_case(L, C, seed, sizes=None, ties=False):
    """channels-last maps of B = 3 images with distinct non-square img_shape inside the map (boxes cross every side) and four distinct
    rescale factors per image; with ties, logits quantised to 1/2 and constant regions, so keys repeat in large groups"""
    g = torch.Generator().manual_seed(seed)
    sizes = sizes or LEVEL_SIZES[:L]
    strides = LEVEL_STRIDES[:len(sizes)]
    B = 3
    cls, reg, ctr = [], [], []
    for (h, w), s in zip(sizes, strides):
        c = torch.randn(B, h, w, C, generator=g) * 1.5 - 2.0
        k = torch.randn(B, h, w, 1, generator=g)
        if ties:
            c, k = torch.round(c * 2) / 2, torch.round(k * 2) / 2
            c[:, : h // 2] = -1.0
            k[:, : h // 2] = 0.5
        cls.append(c.contiguous())
        reg.append((torch.exp(torch.randn(B, h, w, 4, generator=g) * 0.8) * s * 2).contiguous())
        ctr.append(k.contiguous())
    H0, W0 = sizes[0][0] * strides[0], sizes[0][1] * strides[0]
    img_hw = torch.tensor([[H0 * 0.8, W0 * 0.9], [H0 * 0.55, W0 * 0.7], [H0 * 0.95, W0 * 0.4]], dtype=torch.float32).floor()
    sf = torch.tensor([[0.5, 0.75, 1.25, 1.5], [2.0, 1.0, 0.8, 0.6], [1.1, 0.9, 0.7, 1.3]], dtype=torch.float32)
    return cls, reg, ctr, strides, img_hw, sf


def check_decode(ops, case, nms_pre, rescale):
    cls, reg, ctr, strides, img_hw, sf = case
    C = cls[0].shape[3]
    d = lambda ts: [t.to(DEV) for t in ts]
    got = ops.fcos_decode(d(cls), d(reg), d(ctr), strides, C, img_hw.to(DEV), nms_pre, sf.to(DEV) if rescale else None)
    want = ref.decode(cls, reg, ctr, strides, img_hw, nms_pre, sf if rescale else None)
    for name, a, b in zip(('idx', 'boxes', 'scores', 'ctr'), got, want):
        a = a.cpu().numpy()
        assert a.shape == b.shape, (name, a.shape, b.shape)
        bad = np.argwhere(a.view(np.uint32) != b.view(np.uint32)) if a.dtype == np.float32 else np.argwhere(a != b)
        assert bad.size == 0, f'{name}: {len(bad)} elements differ, first {bad[:4].tolist()}'
    # the selected levels' rows against torch.topk, as sets within equal keys
    idx, off = got[0].cpu().long(), 0
    for l, c in enumerate(cls):
        hw = c.shape[1] * c.shape[2]
        n = nms_pre if 0 < nms_pre < hw else hw
        if n < hw:
            key = torch.from_numpy(ref.keys_f32(c, ctr[l]))
            for b in range(key.shape[0]):
                mine, tk = idx[b, off:off + n], key[b].topk(n).indices
                kth = key[b][tk].min()
                above = lambda s: set(s[key[b][s] > kth].tolist())
                assert above(mine) == above(tk)
                assert int((key[b][mine] == kth).sum()) == int((key[b][tk] == kth).sum())
        off += n
    return got


DECODE_LC = [(1, 1), (5, 2), (8, 31), (5, 32), (1, 33), (5, 80), (8, 511)]


@pytest.mark.parametrize('L, C', DECODE_LC)
@pytest.mark.parametrize('nms', ['-1', '0', '1', 'hw-1', 'hw', 'hw+1'])
def test_decode_bit_exact(ops, L, C, nms):
    hw0 = LEVEL_SIZES[0][0] * LEVEL_SIZES[0][1]
    nms_pre = {'-1': -1, '0': 0, '1': 1, 'hw-1': hw0 - 1, 'hw': hw0, 'hw+1': hw0 + 1}[nms]
    check_decode(ops, decode_case(L, C, 100 * L + C), nms_pre, rescale=nms in ('1', 'hw-1'))


@pytest.mark.parametrize('L, C', [(5, 1), (8, 33), (1, 80)])
@pytest.mark.parametrize('nms_pre', [1, 5, 300, 2079])
def test_decode_large_tie_groups(ops, L, C, nms_pre):
    check_decode(ops, decode_case(L, C, 7 + L, ties=True), nms_pre, rescale=True)


def test_decode_4096_on_a_level_above_4096(ops):
    sizes = [(64, 80), (32, 40), (16, 20), (8, 10), (4, 5)]
    for ties in (False, True):
        check_decode(ops, decode_case(5, 3, 21, sizes=sizes, ties=ties), 4096, rescale=True)


def test_decode_nms_pre_above_4096_where_no_level_selects(ops):
    sizes = [(64, 78), (32, 39), (16, 20)]                         # 4 992 cells: nms_pre = 5000 keeps every level whole
    got = check_decode(ops, decode_case(3, 2, 22, sizes=sizes), 5000, rescale=False)
    assert got[0].shape[1] == sum(h * w for h, w in sizes)


# ---------------------------------------------------------------------------------------------------------------------------------
# refusals
def test_refusals(ops):
    cls, reg, ctr, strides, img_hw, sf = (decode_case(1, 3, 5, sizes=[(72, 64)]))
    d = lambda ts: [t.to(DEV) for t in ts]
    hw = img_hw.to(DEV)
    with pytest.raises(NotImplementedError, match='4096'):
        ops.fcos_decode(d(cls), d(reg), d(ctr), strides, 3, hw, 4097)
    with pytest.raises(ValueError, match='1 to 8 levels'):
        ops.fcos_decode([], [], [], [], 3, hw, 100)
    with pytest.raises(ValueError, match='1 to 8 levels'):
        ops.fcos_decode(d(cls) * 9, d(reg) * 9, d(ctr) * 9, strides * 9, 3, hw, 100)
    with pytest.raises(ValueError, match='channels-last'):
        ops.fcos_decode([c.to(DEV).permute(0, 3, 1, 2).contiguous() for c in cls], d(reg), d(ctr), strides, 3, hw, 100)
    with pytest.raises(ValueError, match='contiguous'):
        ops.fcos_decode([c.to(DEV).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1) for c in cls], d(reg), d(ctr), strides, 3,
                        hw, 100)
    c = ref.target_case('one_level')
    off = torch.tensor([0, 1], dtype=torch.int32, device=DEV)
    gt, gl = c['gts'][0].to(DEV), c['gls'][0].to(DEV)
    for L in (0, 9):
        with pytest.raises(ValueError, match='1 to 8 levels'):
            ops.fcos_targets([(4, 4)] * L, [8] * L, 1, gt, gl, off, torch.zeros(L, 2, device=DEV), None, False, 1)
    x = torch.zeros(16, 4, device=DEV)
    with pytest.raises(ValueError, match='1 to 8 levels'):
        ops.fcos_bbox_loss(x, x, torch.zeros(16, dtype=torch.int64, device=DEV), [(1, 1)] * 9, [8] * 9, 1, 1, 0, 1e-6, 1e-6)
