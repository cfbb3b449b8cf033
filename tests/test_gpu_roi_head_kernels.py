"""GPU: the RoI head kernels (csrc/roi_head.cu) through the ops.roi_* wrappers, against the host references of tests/roi_head_ref.py.

  * roi_align_fwd   bit for bit, features and levels, at every channel width G of the work-item mapping (C = 4 .. 1184, the largest
                    C whose block fits shared memory at out = 7), out in {1, 2, 3, 7, 14}, sampling_ratio in {0, 1, 2, 4} (with grids
                    of 20 x 20 and more at 0), 1 to 4 levels at finest_scale 56 and 112, 1 x 1, 1 x W, H x 1 and odd maps, RoIs that are
                    empty, inverted, outside, straddling the border, sampling exactly the last row / column, with bad batch indices or
                    a NaN scale, and R = 0, 1 and 2 000.  The host refuses C * out^2 * 4 > 227 KB and C % 4 != 0.
  * roi_align_bwd   within (n + 2) 2^-24 S_e of float64 at every element (n: the most terms any element receives, S_e: the sum of the
                    element's |terms|), exactly 0 where no RoI reads; SingleRoIExtractor + autograd with NCHW fp32 and fp16 maps.
  * roi_targets     rois, labels and weights exactly, dx / dy bit for bit, dw / dh within 2 ulp, on host-made assignments and plans
                    (every candidate, none, the first and last rank, images without GTs) and past the kernel's grid-stride trip.
  * roi_bbox_loss   sums within 1e-5 of float64, gradients at scale 0.75 within 1e-5 scale-relative and exactly 0 outside the positive
                    rows' class columns, identical bits over two calls; a single term exactly the fp32 SmoothL1 at |d| == beta.
  * roi_accuracy    bit for bit fp32(correct) * fp32(100 / R) with torch.argmax's prediction: ties, -inf rows, NaN rows.
  * roi_decode      scores within 1e-5 relative of float64 (1 / (C + 1) exactly on padding rows), boxes within 8 2^-24 M.
The largest errors seen are printed."""
import math

import numpy as np
import pytest
import torch

from tests import roi_head_ref as ref
from tests.helpers import scale_rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
TOL = 1e-5
STRIDES = [4, 8, 16, 32]
SMEM_LIMIT = 227 * 1024
C_MAX_OUT7 = SMEM_LIMIT // (4 * 49) // 4 * 4          # 1184: the widest block of 7 x 7 bins that fits shared memory

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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------------------
# RoIAlign
def _edge_rois(g, B, H, W, s, out):
    """planted RoIs (image coordinates) on a level of H x W cells of stride s"""
    rows = []
    b = lambda: float(torch.randint(0, B, (1,), generator=g))
    rows += [[b(), 3.0 * s, 2.0 * s, 3.0 * s, 2.0 * s], [b(), 0.0, 0.0, 0.0, 0.0]]                      # zero size
    rows += [[b(), 5.0 * s, 1.0 * s, 2.0 * s, 4.0 * s], [b(), 1.0 * s, 5.0 * s, 4.0 * s, 2.0 * s]]      # negative width / height
    rows += [[b(), -40.0 * s, -30.0 * s, -20.0 * s, -10.0 * s],                                        # wholly outside, both sides
             [b(), (W + 20.0) * s, (H + 10.0) * s, (W + 40.0) * s, (H + 30.0) * s],
             [b(), -9.0 * s, 0.0, -3.0 * s, H * s], [b(), 0.0, (H + 3.0) * s, W * s, (H + 9.0) * s]]
    rows += [[b(), -3.0 * s, -3.0 * s, (W + 2.0) * s, (H + 2.0) * s],                                   # straddling -1 and H / W
             [b(), -1.5 * s, (H - 1.5) * s, 1.5 * s, (H + 1.5) * s]]
    for j in range(out):                   # one bin row / column of samples exactly on y = H, x = W and y = x = -1 (one sample per bin)
        rows.append([b(), 0.0, (H - j) * s, out * s, (H - j + out) * s])
        rows.append([b(), (W - j) * s, 0.0, (W - j + out) * s, out * s])
        rows.append([b(), (-1.0 - j) * s, (-1.0 - j) * s, (-1.0 - j + out) * s, (-1.0 - j + out) * s])
    rows += [[b(), (W - 1.0) * s, (H - 1.0) * s, (W - 1.0) * s, (H - 1.0) * s],                         # on the last cell exactly
             [b(), (W + 0.5) * s, (H + 0.5) * s, (W + 0.5) * s, (H + 0.5) * s]]                         # every sample at (H, W)
    for bi in (-1.0, float(B), 0.5, B - 0.5, -0.5, B + 0.25):                                           # bad and fractional indices
        rows.append([bi, 1.0 * s, 1.0 * s, 4.0 * s, 5.0 * s])
    return torch.tensor(rows, dtype=torch.float32)


def _random_rois(g, n, B, img_h, img_w, lo, hi):
    """n RoIs with log-uniform sides in [lo, hi] and centres over [-0.2, 1.2] of the image"""
    c = torch.rand(n, 2, generator=g) * torch.tensor([img_w, img_h]) * 1.4 - 0.2 * torch.tensor([img_w, img_h])
    wh = torch.exp(torch.rand(n, 2, generator=g) * (math.log(hi) - math.log(lo)) + math.log(lo))
    wh = wh * (1.0 + 0.3 * torch.rand(n, 2, generator=g))
    return torch.cat([torch.randint(0, B, (n, 1), generator=g).float(), c - wh / 2, c + wh / 2], 1)


def _nan_scale_rois(g, n, B):
    """one negative side: sqrt of a negative area is NaN (level -1 when L > 1)"""
    r = _random_rois(g, n, B, 100.0, 100.0, 4.0, 60.0)
    r[:, 3] = r[:, 1] - 3.0
    return r


def _align_case(C, out=7, sr=0, L=1, fs=56, hw=None, B=2, n=150, lo=2.0, hi=300.0, seed=0, edges=True, img=(100, 132)):
    g = torch.Generator().manual_seed(seed)
    img_h, img_w = img
    if hw is None:
        hw = [(-(-img_h // s) + l % 2, -(-img_w // s) + (l + 1) % 2) for l, s in enumerate(STRIDES[:L])]   # unequal, some odd
    maps = [torch.randn(B, h, w, C, generator=g) for h, w in hw]
    parts = [_random_rois(g, n, B, float(img_h), float(img_w), lo, hi)] if n else []
    if edges:
        parts += [_edge_rois(g, B, h, w, s, out) for (h, w), s in zip(hw, STRIDES)]
        if L > 1:
            parts.append(_nan_scale_rois(g, 5, B))
    rois = torch.cat(parts) if parts else torch.zeros((0, 5))
    rois = rois[torch.randperm(rois.shape[0], generator=g)]
    return maps, STRIDES[:L], rois.contiguous(), out, sr, fs


ALIGN_CASES = {
    # every G = min(C4 & -C4, 8) and channel counts off the 32-lane multiple, four levels
    **{f'C{C}': dict(C=C, L=4) for C in (4, 8, 12, 16, 24, 36, 48, 64, 256)},
    f'C{C_MAX_OUT7}_largest': dict(C=C_MAX_OUT7, L=4, n=40, hi=200.0),
    # output sizes (bin counts 1, 4, 9, 196), C = 256 at out = 14 (196 KB of shared memory)
    **{f'out{o}': dict(C=16, out=o, L=4) for o in (1, 2, 3, 14)},
    'out14_C256': dict(C=256, out=14, L=4, n=60, hi=200.0),
    # sampling ratios; 0 with grids of 20 x 20 and more
    **{f'sr{r}': dict(C=12, sr=r, L=4) for r in (1, 2, 4)},
    'sr0_large_grids': dict(C=8, L=1, n=30, lo=560.0, hi=900.0, img=(400, 480)),
    # levels and finest_scale
    **{f'L{L}_fs{fs}': dict(C=8, L=L, fs=fs, lo=2.0, hi=1200.0, img=(200, 264)) for L in (1, 2, 3, 4) for fs in (56, 112)},
    # map shapes
    'map_1x1': dict(C=12, hw=[(1, 1)], n=40, hi=40.0), 'map_1xW': dict(C=12, hw=[(1, 9)], n=40, hi=40.0, sr=2),
    'map_Hx1': dict(C=20, hw=[(9, 1)], n=40, hi=40.0), 'map_odd': dict(C=16, hw=[(7, 13), (5, 3)], L=2, n=60, sr=1),
    # RoI counts
    'R1': dict(C=16, n=1, edges=False), 'R2000_C256': dict(C=256, L=4, n=2000, hi=120.0, edges=False, seed=3),
    # many overlapping RoIs on a small map: elements that receive thousands of terms
    'overlap': dict(C=8, hw=[(6, 7)], n=600, lo=8.0, hi=30.0, img=(24, 28), sr=2, edges=False),
    # only dead RoIs: nothing is written to the gradient
    'dead_only': dict(C=8, L=3, n=0),
}


def _dead_only(maps, rois, B):
    keep = (rois[:, 0].trunc() < 0) | (rois[:, 0].trunc() >= B) | torch.isnan(torch.sqrt((rois[:, 3] - rois[:, 1]) *
                                                                                          (rois[:, 4] - rois[:, 2])))
    return rois[keep].contiguous()


@pytest.mark.parametrize('name', list(ALIGN_CASES))
def test_roi_align_fwd_bit_exact_and_bwd_bound(ops, name):
    maps, strides, rois, out, sr, fs = _align_case(**ALIGN_CASES[name])
    B = maps[0].shape[0]
    if name == 'dead_only':
        rois = _dead_only(maps, rois, B)
        assert rois.shape[0] > 0
    want, want_lv = ref.roi_align_fwd(maps, strides, rois, out, sr, fs)
    dm = [m.to(DEV) for m in maps]
    y, lv = ops.roi_align_fwd(dm, strides, rois.to(DEV), out, sr, fs)
    torch.cuda.synchronize()
    assert torch.equal(lv.cpu().long(), want_lv), f'{name}: levels differ at {(lv.cpu().long() != want_lv).nonzero()[:8].tolist()}'
    diff = (y.cpu() != want) & ~(torch.isnan(y.cpu()) & torch.isnan(want))
    assert not bool(diff.any()), (f'{name}: {int(diff.sum())} features differ, first RoIs '
                                  f'{diff.flatten(1).any(1).nonzero()[:8].squeeze(1).tolist()}')
    if name == 'sr0_large_grids':
        gh, gw = ref._grid(rois, out, 1.0 / strides[0], 0)
        assert int(gh.max()) >= 20 and int(gw.max()) >= 20
    # backward
    g = torch.Generator().manual_seed(17)
    gy = torch.randn(y.shape, generator=g)
    shapes = [tuple(m.shape) for m in maps]
    grads = ops.roi_align_bwd(gy.to(DEV), shapes, strides, rois.to(DEV), lv, sr)
    res = ref.roi_align_bwd64(shapes, strides, rois, want_lv, out, sr, gy)
    n = max(int(c.max()) for _, _, c in res)
    for l, (got, (w64, s, _)) in enumerate(zip(grads, res)):
        got = got.cpu().double()
        read = s > 0
        assert bool((got[~read] == 0).all()), f'{name} level {l}: {int((got[~read] != 0).sum())} unread elements are not 0'
        err = (got - w64).abs()
        bound = (n + 2) * ref.U * s
        bad = err > bound
        assert not bool(bad.any()), (f'{name} level {l}: {int(bad.sum())} elements beyond (n + 2) u S_e (n = {n}); worst '
                                     f'{float((err / bound.clamp(min=1e-300)).max()):.3f} of the bound')
        if bool(read.any()):
            _note('roi_align_bwd |err| / (u S_e)', float((err[read] / (ref.U * s[read])).max()))
    _note('roi_align_bwd n (terms per element)', float(n))


def test_roi_align_zero_rois_launch_nothing(ops):
    maps, strides, _, out, sr, fs = _align_case(C=8, L=2, n=0, edges=False)
    dm = [m.to(DEV) for m in maps]
    rois = torch.zeros((0, 5), device=DEV)
    before = ops.launch_count()
    y, lv = ops.roi_align_fwd(dm, strides, rois, out, sr, fs)
    grads = ops.roi_align_bwd(y, [tuple(m.shape) for m in maps], strides, rois, lv, sr)
    assert ops.launch_count() == before
    assert tuple(y.shape) == (0, 8, 7, 7) and lv.numel() == 0 and all(not bool(g.any()) for g in grads)


@pytest.mark.parametrize('C, out, ok', [(C_MAX_OUT7, 7, True), (C_MAX_OUT7 + 4, 7, False), (6, 7, False), (2, 1, False),
                                        (296, 14, True), (300, 14, False)])
def test_roi_align_host_refusals(ops, C, out, ok):
    """C * out^2 floats must fit 227 KB of shared memory and C must be a multiple of 4: refused on the host, before any launch"""
    m = [torch.zeros((1, 3, 3, C), device=DEV)]
    rois = torch.tensor([[0.0, 1.0, 1.0, 2.0, 2.0]], device=DEV)
    before = ops.launch_count()
    if ok:
        ops.roi_align_fwd(m, [4], rois, out, 0, 56)
        assert ops.launch_count() == before + 1
        return
    with pytest.raises(RuntimeError, match='ptb_roi_align_fwd'):
        ops.roi_align_fwd(m, [4], rois, out, 0, 56)
    gy = torch.zeros((1, C, out, out), device=DEV)
    with pytest.raises(RuntimeError, match='ptb_roi_align_bwd'):
        ops.roi_align_bwd(gy, [(1, 3, 3, C)], [4], rois, torch.zeros(1, dtype=torch.int32, device=DEV), 0)
    assert ops.launch_count() == before


@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_extractor_autograd_nchw(ops, L, dtype):
    """SingleRoIExtractor over L NCHW maps (fp32, fp16) under autograd: features bit for bit against the reference on the maps as
    fp32, the maps' gradients within (n + 2) u S_e (fp16: plus the fp16 rounding of the gradient)"""
    from pointtinybenchmark_b200.roi_head import SingleRoIExtractor
    maps, strides, rois, out, sr, fs = _align_case(C=24, L=L, n=120, seed=5 + L, hi=500.0, img=(120, 152))
    feats = [m.permute(0, 3, 1, 2).contiguous().to(dtype) for m in maps]
    ex = SingleRoIExtractor(dict(type='RoIAlign', output_size=out, sampling_ratio=sr), 24, strides)
    x = [f.to(DEV).requires_grad_(True) for f in feats]
    y = ex(x, rois.to(DEV))
    nhwc = [f.float().permute(0, 2, 3, 1).contiguous() for f in feats]
    want, want_lv = ref.roi_align_fwd(nhwc, strides, rois, out, sr, fs)
    assert torch.equal(y.detach().cpu(), want) and torch.equal(ex.last_levels.cpu().long(), want_lv)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(2))
    y.backward(gy.to(DEV))
    res = ref.roi_align_bwd64([tuple(m.shape) for m in nhwc], strides, rois, want_lv, out, sr, gy)
    n = max(int(c.max()) for _, _, c in res)
    for l in range(L):
        got = x[l].grad
        assert got.dtype == dtype and got.shape == feats[l].shape
        got = got.cpu().double().permute(0, 2, 3, 1)
        w64, s, _ = res[l]
        bound = (n + 2) * ref.U * s
        if dtype == torch.float16:                         # the gradient rounded to fp16 (2^-25: its subnormal spacing / 2)
            bound = bound + 2.0 ** -11 * (w64.abs() + bound) + 2.0 ** -25
        assert bool(((got - w64).abs() <= bound).all()), f'level {l}'
        assert bool((got[s == 0] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# RoI targets
def _boxes(g, n, lo=2.0, hi=120.0, img=(400.0, 500.0)):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([img[1], img[0]])
    wh = torch.rand(n, 2, generator=g) * (hi - lo) + lo
    return torch.cat([xy, xy + wh], 1)


def _targets_case(seed, n_gt, N, num_classes, modes):
    """host-made assignments: per image n_gt[b] GTs (first among the candidates, assigned to themselves), the other candidates
    positive, negative or ignored at random; ranks by host cumsum; plan per (image, kind) by modes[b][kind] in
    {'all', 'none', 'draw'} ('draw' keeps the first and the last rank)"""
    g = torch.Generator().manual_seed(seed)
    B = len(n_gt)
    gts = [_boxes(g, k) for k in n_gt]
    labels = [torch.randint(0, num_classes, (k,), generator=g) for k in n_gt]
    cand = _boxes(g, B * N).view(B, N, 4)
    gt_inds = torch.zeros((B, N), dtype=torch.int64)
    for b in range(B):
        k = n_gt[b]
        cand[b, :k] = gts[b]
        gt_inds[b, :k] = torch.arange(1, k + 1)
        if k:
            r = torch.randint(0, 10, (N - k,), generator=g)
            src = torch.randint(1, k + 1, (N - k,), generator=g)
            pos = r < 4
            gt_inds[b, k:] = torch.where(pos, src, torch.where(r < 8, 0, -1))
            jitter = gts[b][src - 1] + torch.randn(N - k, 4, generator=g) * 3.0
            jitter[:, 2:] = torch.maximum(jitter[:, 2:], jitter[:, :2] + 1.0)
            cand[b, k:] = torch.where(pos[:, None], jitter, cand[b, k:])
        else:
            gt_inds[b] = torch.where(torch.rand(N, generator=g) < 0.8, 0, -1)
    rank = torch.zeros((B, N), dtype=torch.int32)
    header, body, row_off, sel, R = [], [], [], [], 0
    for b in range(B):
        for kind in (0, 1):
            m = (gt_inds[b] > 0) if kind == 0 else (gt_inds[b] == 0)
            idx = m.nonzero().squeeze(1)
            rank[b, idx] = torch.arange(idx.numel(), dtype=torch.int32)
            nk, mode = idx.numel(), modes[b][kind]
            if mode == 'all':
                ranks, cnt = torch.arange(nk), -1
            elif mode == 'none' or nk == 0:
                ranks, cnt = torch.zeros(0, dtype=torch.int64), 0
            else:                                  # a random third of the ranks, the first and the last among them
                drawn = torch.randperm(nk, generator=g)[:max(1, nk // 3)]
                ranks = torch.unique(torch.cat([drawn, torch.tensor([0, nk - 1])]))
                cnt = ranks.numel()
            header.append([0, cnt])
            body.append(ranks.int())
            row_off.append(R)
            sel.append((b, kind, idx[ranks]))
            R += ranks.numel()
    off = 4 * B
    for h, r in zip(header, body):
        h[0] = off
        off += r.numel()
    plan = torch.cat([torch.tensor(header, dtype=torch.int32).view(-1)] + body)
    gt_off = torch.tensor(np.concatenate([[0], np.cumsum(n_gt)]), dtype=torch.int32)
    gt_cat = torch.cat(gts) if sum(n_gt) else torch.zeros((0, 4))
    lab_cat = torch.cat(labels) if sum(n_gt) else torch.zeros((0,), dtype=torch.int64)
    return dict(cand=cand, gt_inds=gt_inds, rank=rank, plan=plan, row_off=torch.tensor(row_off, dtype=torch.int32), gts=gt_cat,
                gt_off=gt_off, gt_labels=lab_cat, R=R, sel=sel, B=B)


def _targets_want(c, num_classes, means, stds, pos_weight):
    R = c['R']
    rois = np.zeros((R, 5), np.float32)
    labels = np.full(R, num_classes, np.int64)
    lw, bt, bw = np.ones(R, np.float32), np.zeros((R, 4), np.float32), np.zeros((R, 4), np.float32)
    row = 0
    for b, kind, e in c['sel']:
        n = e.numel()
        rows = slice(row, row + n)
        box = c['cand'][b, e].numpy()
        rois[rows, 0], rois[rows, 1:] = b, box
        if kind == 0 and n:
            gi = (c['gt_off'][b] + c['gt_inds'][b, e] - 1).numpy()
            labels[rows] = c['gt_labels'].numpy()[gi]
            lw[rows] = pos_weight if pos_weight > 0 else 1.0
            bt[rows] = ref.bbox2delta_f32(box, c['gts'].numpy()[gi], means, stds)
            bw[rows] = 1.0
        row += n
    return rois, labels, lw, bt, bw


TARGET_MODES = {
    'mixed': ([5, 0, 9], 300, [('draw', 'draw'), ('none', 'all'), ('all', 'draw')]),
    'all_none': ([3, 4], 200, [('all', 'none'), ('none', 'all')]),
    'one_candidate': ([1], 1, [('all', 'all')]),
}


@pytest.mark.parametrize('num_classes', [1, 80, 1203])
@pytest.mark.parametrize('pos_weight', [-1.0, 0.0, 2.5])
@pytest.mark.parametrize('mode', list(TARGET_MODES))
def test_roi_targets(ops, mode, pos_weight, num_classes):
    n_gt, N, modes = TARGET_MODES[mode]
    _check_targets(ops, _targets_case(len(mode) + num_classes, n_gt, N, num_classes, modes), num_classes, pos_weight,
                   [0.05, -0.05, 0.0, 0.0], [0.1, 0.1, 0.2, 0.2])


def test_roi_targets_past_the_grid_trip(ops):
    """B * N beyond 8 SMs x 256 threads: every thread makes a second trip"""
    cap = 8 * _sms() * 256
    N = cap // 2 + 3001
    c = _targets_case(99, [40, 25], N, 80, [('draw', 'draw'), ('all', 'draw')])
    assert 2 * N > cap
    _check_targets(ops, c, 80, -1.0, [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0])


def _check_targets(ops, c, num_classes, pos_weight, means, stds):
    d = lambda t: t.contiguous().to(DEV)
    got = ops.roi_targets(d(c['cand']), d(c['gt_inds']), d(c['rank']), d(c['plan']), d(c['row_off']), d(c['gts'].view(-1, 4)),
                          d(c['gt_off']), d(c['gt_labels']), num_classes, means, stds, pos_weight, c['R'])
    rois, labels, lw, bt, bw = [t.cpu().numpy() for t in got]
    w_rois, w_labels, w_lw, w_bt, w_bw = _targets_want(c, num_classes, means, stds, pos_weight)
    assert np.array_equal(rois, w_rois) and np.array_equal(labels, w_labels)
    assert np.array_equal(lw, w_lw) and np.array_equal(bw, w_bw)
    assert np.array_equal(bt[:, :2], w_bt[:, :2]), f'dx / dy differ in {int((bt[:, :2] != w_bt[:, :2]).sum())} places'
    u = ref.ulp_diff(bt[:, 2:], w_bt[:, 2:])
    if u.size:
        _note('roi_targets dw / dh ulps', float(u.max()))
        assert int(u.max()) <= 2, f'dw / dh {int(u.max())} ulp from the correctly rounded log'


# ---------------------------------------------------------------------------------------------------------------------------------
# box loss
def check_loss(call, x, ref_sum, ref_grad, what, key, zero=None):
    """call(scale=None, want_grad=False) runs one kernel; x is its input on the GPU.  Sum, gradient (at scale 0.75), determinism,
    zero-gradient elements and NaN placement against the float64 reference."""
    l1, l2 = call(), call()
    assert torch.equal(l1, l2) or (torch.isnan(l1).all() and torch.isnan(l2).all()), f'{what}: two sums differ'
    got, want = float(l1.cpu()), float(ref_sum)
    if np.isnan(want):
        assert np.isnan(got), f'{what}: sum {got}, float64 NaN'
    else:
        e = abs(got - want) / max(abs(want), 1e-30)
        _note(key + ' sum', e)
        assert e <= TOL or got == want, f'{what}: sum {got!r} vs float64 {want!r} (relative {e:.3e})'
    sc = torch.tensor([0.75], device=x.device)
    g1 = call(scale=sc, want_grad=True)
    g2 = call(scale=sc, want_grad=True)
    assert torch.equal(torch.nan_to_num(g1, 7.0), torch.nan_to_num(g2, 7.0)), f'{what}: two gradients differ'
    g1 = g1.cpu().double()
    want_g = 0.75 * ref_grad
    nan_g, nan_w = torch.isnan(g1), torch.isnan(want_g)
    assert torch.equal(nan_g, nan_w), (f'{what}: gradient NaN at {int(nan_g.sum())} elements, float64 at {int(nan_w.sum())} '
                                       f'(first mismatch {torch.nonzero(nan_g != nan_w)[:4].tolist()})')
    ok = ~nan_w
    assert torch.isfinite(g1[ok]).all(), f'{what}: non-finite gradient where float64 is finite'
    e = scale_rel_err(g1[ok], want_g[ok])
    _note(key + ' grad', e)
    assert e <= TOL, f'{what}: gradient scale-relative error {e:.3e} > {TOL}'
    if zero is not None and bool(zero.any()):
        gz = g1[zero.cpu() & ok]
        assert bool((gz == 0).all()), f'{what}: {int((gz != 0).sum())} zero-weight / no-bin elements have a non-zero gradient'


def _loss_inputs(seed, R, C, agnostic, beta):
    g = torch.Generator().manual_seed(seed)
    ld = 4 if agnostic else 4 * C
    pred = torch.randn(R, ld, generator=g) * 2
    r = torch.randint(0, 10, (R,), generator=g)
    labels = torch.randint(0, C, (R,), generator=g)
    labels = torch.where(r == 0, torch.full_like(labels, C), torch.where(r == 1, torch.full_like(labels, -1), labels))
    bt = torch.randn(R, 4, generator=g)
    bw = torch.ones(R, 4)
    bw[torch.randint(0, 6, (R,), generator=g) == 0] = 0.0                    # zero-weight rows
    # planted |d| == fp32(beta) (target 0, so the difference is exact) and d == 0
    b32 = float(np.float32(beta))
    pos = ((labels >= 0) & (labels < C)).nonzero().squeeze(1)
    for j, m in enumerate(pos[:24].tolist()):
        k = j % 4
        col = k if agnostic else 4 * int(labels[m]) + k
        if j % 3 == 2:
            bt[m, k] = pred[m, col]
        else:
            bt[m, k] = 0.0
            pred[m, col] = b32 if j % 3 == 0 else -b32
        bw[m, k] = 1.0
    return pred, labels, bt, bw


LOSS_KINDS = {'l1': (False, 1.0), 'smooth_b1': (True, 1.0), 'smooth_b1_9': (True, 1.0 / 9.0), 'smooth_b0.11': (True, 0.11)}
LOSS_SHAPES = [(1, 1), (33791, 1), (33792, 80), (33793, 1), (70000, 80), (2000, 365), (1500, 1203)]


@pytest.mark.parametrize('R, C', LOSS_SHAPES)
@pytest.mark.parametrize('agnostic', [False, True])
@pytest.mark.parametrize('kind', list(LOSS_KINDS))
def test_roi_bbox_loss(ops, kind, agnostic, R, C):
    smooth, beta = LOSS_KINDS[kind]
    pred, labels, bt, bw = _loss_inputs(R + C, R, C, agnostic, beta)
    s, grad, read = ref.bbox_loss64(pred, labels, bt, bw, C, agnostic, smooth, beta)
    dp, dl, dt, dw = pred.to(DEV), labels.to(DEV), bt.to(DEV), bw.to(DEV)
    loss_kind = ops.RPN_LOSS_SMOOTH_L1 if smooth else ops.RPN_LOSS_L1
    call = lambda scale=None, want_grad=False: ops.roi_bbox_loss(dp, dl, dt, dw, C, agnostic, loss_kind, beta if smooth else 0.0,
                                                                 scale=scale, want_grad=want_grad)
    check_loss(call, dp, s, grad, f'{kind} agnostic={agnostic} R={R} C={C}', f'roi_bbox_loss {kind}', zero=~read)


def _split_beta():
    """the first fp32 beta >= 0.4 at which SmoothL1's two branches round apart at d == beta"""
    b = np.float32(0.4)
    while (np.float32(0.5) * b * b) / b == b - np.float32(0.5) * b:
        b = np.nextafter(b, np.float32(1.0))
    return b


@pytest.mark.parametrize('sign', [1.0, -1.0])
@pytest.mark.parametrize('agnostic', [False, True])
def test_roi_bbox_loss_single_term_at_beta(ops, sign, agnostic):
    """one non-zero term: the sum is that term, which at |d| == beta must be the linear branch d - beta / 2 (SmoothL1 takes the
    quadratic branch only for d < beta); at this beta the quadratic branch rounds to a different float"""
    beta = _split_beta()
    C = 3
    pred = torch.zeros(1, 4 if agnostic else 4 * C)
    labels = torch.tensor([1])
    col = 2 if agnostic else 4 + 2
    pred[0, col] = float(sign * beta)
    bt, bw = torch.zeros(1, 4), torch.tensor([[0.0, 0.0, 1.0, 0.0]])
    got = ops.roi_bbox_loss(pred.to(DEV), labels.to(DEV), bt.to(DEV), bw.to(DEV), C, agnostic, ops.RPN_LOSS_SMOOTH_L1, float(beta))
    d = torch.tensor([float(beta)])
    want = torch.where(d < float(beta), 0.5 * d * d / float(beta), d - 0.5 * float(beta))      # torch fp32, the reference's formula
    assert float(got.cpu()[0]) == float(want[0]) == float(beta - np.float32(0.5) * beta)


# ---------------------------------------------------------------------------------------------------------------------------------
# accuracy
def _acc_inputs(seed, R, K):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, K, generator=g)
    ints = torch.randint(0, 4, (R, K), generator=g).float()                   # integer rows: ties everywhere
    x = torch.where((torch.arange(R) % 3 == 0)[:, None], ints, x)
    for m in range(0, R, 7):                                                   # planted ties: across lanes and within a lane
        a = int(torch.randint(0, K, (1,), generator=g))
        for c in {a, (a + 1) % K, (a + 32) % K, (a + 64) % K}:
            x[m, c] = 50.0
    for m in range(1, R, 11):
        x[m] = -float('inf')                                                   # all -inf
    for m in range(2, R, 13):
        x[m, int(torch.randint(0, K, (1,), generator=g))] = float('nan')       # one NaN
    for m in range(3, R, 17):
        x[m, torch.randint(0, K, (3,), generator=g)] = float('nan')            # several NaNs
    for m in range(4, R, 19):
        x[m, -1] = float('nan')                                                # NaN at the background column
    want = ref.argmax_rule(x)
    labels = torch.randint(0, K, (R,), generator=g)
    labels = torch.where(torch.rand(R, generator=g) < 0.6, want, labels)     # most rows correct, K - 1 is the background label
    labels[::23] = K - 1
    return x, labels


@pytest.mark.parametrize('K', [2, 31, 32, 33, 81, 366, 1204])
@pytest.mark.parametrize('R', [1, 31, 32, 33, 1025, 8192])
def test_roi_accuracy_bit_exact(ops, R, K):
    x, labels = _acc_inputs(R * 7 + K, R, K)
    got = ops.roi_accuracy(x.to(DEV), labels.to(DEV))
    want = ref.accuracy_f32(x, labels)
    assert float(got.cpu()[0]) == float(want), (float(got.cpu()[0]), float(want))


def test_roi_accuracy_nan_rows_rank_first(ops):
    """the issue's rows: [1, nan, 3] and [inf, nan, 1] predict column 1, as topk(1) and argmax do"""
    x = torch.tensor([[1.0, float('nan'), 3.0], [float('inf'), float('nan'), 1.0]])
    for lab, want in (([1, 1], 100.0), ([2, 0], 0.0), ([1, 0], 50.0)):
        got = ops.roi_accuracy(x.to(DEV), torch.tensor(lab).to(DEV))
        assert float(got.cpu()[0]) == want


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
MAX_RATIO = abs(np.log(16 / 1000))


def _decode_inputs(seed, B, N, C, agnostic, means, stds):
    g = torch.Generator().manual_seed(seed)
    img_hw = torch.tensor([[200.0 + 17 * b, 260.0 - 9 * b] for b in range(B)])
    rows = []
    for b in range(B):
        H, W = img_hw[b].tolist()
        n_pad = (N // 5) if b % 2 == 0 else 0
        r = torch.cat([torch.rand(N, 2, generator=g) * torch.tensor([W, H]) * 1.2 - 20.0, torch.rand(N, 2, generator=g) * 90 + 1], 1)
        r[:, 2:] += r[:, :2]
        r[:n_pad] = 0.0                                                  # the reference's padding rows, at the front
        if N > n_pad + 3:
            r[n_pad] = torch.tensor([0.0, 0.0, 0.0, 5.0])                # one non-zero coordinate: not padding
            r[n_pad + 1] = torch.tensor([-10.0, -8.0, 12.0, 6.0])        # straddling the top-left corner
            r[n_pad + 2] = torch.tensor([W - 6.0, H - 5.0, W + 20.0, H + 9.0])
        rows.append(torch.cat([torch.full((N, 1), float(b)), r], 1))
    rois = torch.cat(rows)
    M = B * N
    spread = torch.rand(M, 1, generator=g) * 100.0
    cls = torch.rand(M, C + 1, generator=g) * spread + torch.randn(M, 1, generator=g) * 10.0
    ld = 4 if agnostic else 4 * C
    reg = torch.randn(M, ld, generator=g)
    sd = torch.tensor(stds * (ld // 4)).view(1, ld)
    mn = torch.tensor(means * (ld // 4)).view(1, ld)
    k = torch.arange(ld)
    mr = float(MAX_RATIO)
    pick = torch.randint(0, 8, (M, ld), generator=g)
    target = torch.where(pick == 0, torch.full((M, ld), 1.7 * mr), torch.where(pick == 1, torch.full((M, ld), -1.6 * mr),
                         torch.where(pick == 2, torch.full((M, ld), mr * (1 - 1e-6)), torch.full((M, ld), -mr * (1 - 1e-6)))))
    wh = (k % 4 >= 2)[None, :] & (pick < 4)
    reg = torch.where(wh, (target - mn) / sd, reg)                      # dw / dh beyond and just inside +-max_ratio
    xy = (k % 4 < 2)[None, :] & (pick >= 6)
    reg = torch.where(xy, torch.where(pick == 6, 40.0, -40.0) / sd, reg)   # centres pushed past 0 and past W / H
    return rois.contiguous(), cls.contiguous(), reg.contiguous(), img_hw


DECODE_CASES = [(C, agnostic) for C in (1, 31, 32, 33, 80, 365) for agnostic in (False, True)]


@pytest.mark.parametrize('rescale', [False, True])
@pytest.mark.parametrize('C, agnostic', DECODE_CASES)
def test_roi_decode(ops, C, agnostic, rescale):
    _check_decode(ops, C * 3 + agnostic + 7 * rescale, 3, 60, C, agnostic, rescale)


def test_roi_decode_past_the_grid_trip(ops):
    """B * N beyond 16 SMs x 8 warps rows: every warp decodes a second row"""
    rows = 16 * _sms() * 8
    _check_decode(ops, 5, 2, rows // 2 + 700, 2, False, True)


def _check_decode(ops, seed, B, N, C, agnostic, rescale):
    means, stds = [0.02, -0.03, 0.0, 0.01], [0.1, 0.1, 0.2, 0.2]
    rois, cls, reg, img_hw = _decode_inputs(seed, B, N, C, agnostic, means, stds)
    sf = torch.tensor([[1.25, 1.5, 1.25, 1.5], [0.8, 2.0, 0.8, 2.0], [3.0, 0.75, 3.0, 0.75]])[:B] if rescale else None
    boxes, scores = ops.roi_decode(rois.to(DEV), cls.to(DEV), reg.to(DEV), B, C, agnostic, means, stds, MAX_RATIO, img_hw.to(DEV),
                                   None if sf is None else sf.to(DEV))
    wb, ws, mag = ref.decode64(rois, cls, reg, B, C, agnostic, means, stds, MAX_RATIO, img_hw, sf)
    boxes, scores = boxes.cpu().double(), scores.cpu().double()
    pad = (rois[:, 1:].abs().sum(1) == 0).view(B, N)
    assert int(pad.sum()) > 0 or B * N < 10
    assert bool((scores[pad] == float(np.float32(1.0 / (C + 1)))).all()), 'padding rows must score exactly 1 / (C + 1)'
    e = (scores - ws).abs()
    bad = e > TOL * ws + 2.0 ** -126                    # below FLT_MIN fp32 has no relative precision
    assert not bool(bad.any()), f'{int(bad.sum())} scores beyond 1e-5 relative (worst {float((e / ws.clamp(min=1e-300)).max()):.3e})'
    _note('roi_decode scores relative', float((e / ws.clamp(min=2.0 ** -126)).max()))
    eb = (boxes - wb).abs() / (ref.U * mag[..., None, None])
    _note('roi_decode boxes |err| / (u M)', float(eb.max()))
    assert float(eb.max()) <= 8.0, f'boxes {float(eb.max()):.2f} u M from float64'
