"""CPU: the host restatement of the bag gather (tests/gather_ref.py) against ATen's CPU grid_sample, which the kernel reproduces bit for
bit: the fp32 forward at every channel width and map edge the GPU tests use, the float64 forward and backward against float64
grid_sample and its autograd, the correctly rounded fma the fp32 forward rests on, and the staged-window and dispatch restatements."""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cpr as ocpr
from pointtinybenchmark_b200 import ops
from tests import gather_ref as ref

U = 2.0 ** -24


def _points(g, n, H, W, s, out=0.1):
    """n fp32 points: uniform over the map and up to `out` of its size beyond every side, exact cell positions, and points a few
    ulps either side of a cell position"""
    span = torch.tensor([W * s, H * s])
    p = torch.rand(n, 2, generator=g) * span * (1 + 2 * out) - out * span
    cells = torch.stack([torch.randint(0, W, (n,), generator=g), torch.randint(0, H, (n,), generator=g)], 1).float() * s
    near = cells.clone()
    for _ in range(3):
        near = torch.nextafter(near, torch.where(torch.rand(n, 2, generator=g) < 0.5, -np.inf, np.inf).float())
    return torch.cat([p, cells, near]).float()


def _aten_f32(map_nhwc, pts, s, C):
    """oracle.cpr.sample_point_feat (F.grid_sample, fp32) of a one-image map at (N,2) points -> (N,C)"""
    return ocpr.sample_point_feat(map_nhwc[..., :C].permute(0, 3, 1, 2).contiguous(), pts[None], s)[0]


def _one_image(pts):
    """the gather_ref arguments that sample image 0 at pts: one bag per point, a centre-only offset table"""
    return pts, torch.zeros(pts.shape[0], dtype=torch.int32), torch.zeros(1, 2)


@pytest.mark.parametrize('C,H,W,s', [(4, 20, 28, 8), (16, 20, 28, 8), (48, 13, 9, 8), (80, 13, 21, 8), (128, 13, 21, 4),
                                     (160, 13, 9, 8), (192, 5, 2, 8), (256, 20, 28, 8), (272, 13, 21, 16), (16, 1, 7, 8),
                                     (16, 1, 1, 8), (4, 2, 5, 8), (16, 100, 168, 8)])
def test_gather_f32_equals_aten_grid_sample_bit_for_bit(C, H, W, s):
    g = torch.Generator().manual_seed(C * 1000 + H * 10 + W)
    ld = C + 4
    m = torch.randn(1, H, W, ld, generator=g)
    m[..., C:] = float('nan')                                  # padding columns are never read
    pts = _points(g, max(200, 60000 // C), H, W, s)
    got = ref.gather_f32(m, *_one_image(pts), s, C)[:, 0]
    want = _aten_f32(m, pts, s, C)
    assert not torch.isnan(got).any()
    nbad = int((got.view(torch.int32) != want.view(torch.int32)).sum())
    assert nbad == 0, f'{nbad} / {want.numel()} values differ from ATen grid_sample'


def test_gather_f32_bags_follow_the_image_and_offset_tables():
    """several images, unsorted bag_img, ring offsets: each bag equals grid_sample of its own image at centre + offsets"""
    g = torch.Generator().manual_seed(3)
    B, H, W, C, s, r = 3, 13, 21, 48, 8, 3
    m = torch.randn(B, H, W, C, generator=g)
    n = 30
    centers = (torch.rand(n, 2, generator=g) * torch.tensor([W * s * 1.2, H * s * 1.2]) - 10).float()
    bag_img = torch.randint(0, B, (n,), generator=g).int()
    off = ops.circle_offsets(r, s)
    got = ref.gather_f32(m, centers, bag_img, off, s)
    pts = ref.sample_points(centers, off)
    for i in range(n):
        want = _aten_f32(m[int(bag_img[i]):int(bag_img[i]) + 1], pts[i], s, C)
        assert torch.equal(got[i], want), i


def _fma_exact(a, b, c):
    """fp32 fma(a, b, c) from exact rational arithmetic: the nearest fp32 value, ties to even"""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    f = np.float32(float(x))
    cand = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    d = [abs(Fraction(float(v)) - x) for v in cand]
    best = min(d)
    ties = [v for v, e in zip(cand, d) if e == best]
    return ties[0] if len(ties) == 1 else next(v for v in ties if int(np.array(v).view(np.int32)) % 2 == 0)


def test_fma_f32_is_correctly_rounded():
    g = torch.Generator().manual_seed(11)
    n = 3000
    a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    c = -(a.double() * b.double()).float() * (1 + torch.randn(n, generator=g) * 1e-6)     # heavy cancellation
    c = torch.where(torch.rand(n, generator=g) < 0.5, c, torch.randn(n, generator=g))
    # sums that lie within a float64 ulp of an fp32 tie: one rounding in float64 and one in fp32 would round them to even
    e = torch.tensor([1 + 2 ** -23, -(1 + 2 ** -23), 3 * (1 + 2 ** -23), 1 + 2 ** -23], dtype=torch.float32)
    f = torch.tensor([1 - 2 ** -23, 1 - 2 ** -23, (1 - 2 ** -23) / 4, 1 + 2 ** -23], dtype=torch.float32)
    h = torch.tensor([2 ** 24 + 2, -(2 ** 24 + 2), 3 * 2 ** 22 + 3, 2 ** 24], dtype=torch.float32)
    a, b, c = torch.cat([a, e]), torch.cat([b, f]), torch.cat([c, h])
    got = ref.fma_f32(a, b, c)
    want = torch.tensor(np.array([_fma_exact(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], dtype=np.float32))
    assert torch.equal(got, want)
    naive = (a.double() * b.double() + c.double()).float()
    assert not torch.equal(naive[n:], want[n:]), 'the planted ties must defeat a plain float64 fma'


@pytest.mark.parametrize('C,H,W,s', [(16, 20, 28, 8), (80, 13, 9, 4), (4, 1, 7, 16)])
def test_gather_f64_agrees_with_float64_grid_sample(C, H, W, s):
    g = torch.Generator().manual_seed(C + H)
    m = torch.randn(1, H, W, C, generator=g, dtype=torch.float64)
    pts = _points(g, 3000, H, W, s)
    got = ref.gather_f64(m, *_one_image(pts), s)[:, 0]
    want = _aten_f32(m, pts.double(), s, C)
    # the kernel's taps come from fp32 coordinates and weights: each weight is within a few fp32 ulps of size of float64's
    bound = 16 * U * max(H, W) * m.abs().max()
    assert float((got - want).abs().max()) <= bound
    # and the fp32 forward is the fp32 rounding of the same blend: four roundings of partial sums bounded by sum |w q|
    m32 = m.float()
    f32 = ref.gather_f32(m32, *_one_image(pts), s)[:, 0].double()
    f64 = ref.gather_f64(m32, *_one_image(pts), s)[:, 0]
    idx, w = ref.bag_taps(*_one_image(pts), s, H, W)
    absw = sum(m32.reshape(H * W, C)[idx[:, 0, t]].double().abs() * w[:, 0, t, None].double() for t in range(4))
    assert bool(((f32 - f64).abs() <= 4.01 * U * absw).all())


@pytest.mark.parametrize('C,ld,H,W,s', [(16, 20, 20, 28, 8), (4, 4, 1, 7, 8), (80, 112, 13, 9, 16)])
def test_scatter_f64_is_the_adjoint_of_the_gather(C, ld, H, W, s):
    g = torch.Generator().manual_seed(C * 7 + H)
    B, r, n = 2, 3, 12
    m = torch.randn(B, H, W, ld, generator=g, dtype=torch.float64)
    centers = (torch.rand(n, 2, generator=g) * torch.tensor([W * s * 1.3, H * s * 1.3]) - 0.15 * torch.tensor([W * s, H * s])).float()
    centers[0] = torch.tensor([3.0 * s, 2.0 * s])
    bag_img = torch.randint(0, B, (n,), generator=g).int()
    off = ops.circle_offsets(r, s)
    K = off.shape[0]
    go = torch.randn(n, K, C, generator=g)
    grad, absum, count = ref.scatter_f64(go, (B, H, W, ld), centers, bag_img, off, s)
    # float64 autograd of grid_sample at the same fp32 points: its float64 weights differ from the kernel's fp32 ones by a few ulps
    mm = m.clone().requires_grad_(True)
    pts = ref.sample_points(centers, off).double()
    tot = 0
    for b in range(B):
        sel = (bag_img == b).nonzero().flatten()
        if len(sel):
            tot = tot + (ocpr.sample_point_feat(mm[b:b + 1, ..., :C].permute(0, 3, 1, 2), pts[sel], s) * go[sel].double()).sum()
    tot.backward()
    want = mm.grad
    assert float((grad - want).abs().max()) <= 16 * U * max(H, W) * float(absum.max()) + 1e-12
    assert bool((grad[..., C:] == 0).all()) and bool((absum[..., C:] == 0).all())
    assert bool((grad.abs() <= absum * (1 + 1e-12)).all())
    # exact adjoint of the float64 blend of the same fp32 taps
    lhs = float((ref.gather_f64(m, centers, bag_img, off, s, C) * go.double()).sum())
    rhs = float((m * grad).sum())
    assert abs(lhs - rhs) <= 1e-12 * float((m.abs() * absum).sum())
    _, w = ref.bag_taps(centers, bag_img, off, s, H, W)
    assert int(count.sum()) == int((w != 0).sum())
    assert bool(((count == 0) == (absum[..., :C] == 0).all(-1, keepdim=True)).all())


def test_window_staged_finds_staged_and_straddling_bags():
    """centres a few ulps either side of cell positions: rounding in the fp32 sample coordinate of centre -/+ reach can make the
    window one cell wider than WS; every staged bag's taps lie inside its WS x WS window"""
    H, W, s = 40, 56, 8.0
    for r in (1, 3, 8, 10):
        reach = r * s
        ks = torch.arange(r + 1, W - r - 1).float() * s
        cx = torch.cat([ks] + [torch.nextafter(ks, torch.full_like(ks, d * np.inf)) for d in (-1, 1)])
        centers = torch.stack([cx, torch.full_like(cx, 17 * s + 3.25)], 1)
        staged = ref.window_staged(centers, reach, s, H, W)
        assert bool(staged.any()) and bool((~staged).any()), r
        ws = ref.window_size(reach, s)
        off = ops.circle_offsets(r, s)
        idx, w = ref.bag_taps(centers, torch.zeros(len(cx), dtype=torch.int32), off, s, H, W)
        x, y = idx % W, idx // W
        wide_x = x.amax((1, 2)) - x.amin((1, 2)) + 1
        wide_y = y.amax((1, 2)) - y.amin((1, 2)) + 1
        assert bool(((wide_x <= ws) & (wide_y <= ws))[staged].all())
        assert int(wide_y.max()) <= ws


def test_expected_path_mirrors_the_host_dispatch():
    P = ref.expected_path
    assert P(160, 160, 289, 64.0, 8, {}) == ('tma<32>', None)
    assert P(80, 80, 289, 64.0, 8, {}) == ('ldg<20>', None)
    assert P(160, 160, 289, 64.0, 8, {'PTB_GATHER_TMA': '0'}) == ('ldg<40>', None)
    assert P(256, 256, 289, 64.0, 8, {}) == ('ldg<64>', None)
    assert P(256, 256, 289, 64.0, 8, {'PTB_GATHER_TMA': '1'}) == ('tma<64>', None)
    assert P(256, 256, 289, 64.0, 8, {'PTB_GATHER_TMA': '1', 'PTB_GATHER_CC': '32'}) == ('tma<32>', None)
    assert P(128, 128, 289, 64.0, 8, {'PTB_GATHER_CC': '64'}) == ('tma<64>', None)
    assert P(160, 160, 289, 64.0, 8, {'PTB_GATHER_CC': '64'}) == ('tma<32>', None)   # 160 channels have no 64-channel chunks
    assert P(128, 128, 441, 80.0, 8, {}) == ('tma<32>', None)                         # r = 10: 22 x 22 x 32 channels fit
    assert P(128, 128, 441, 80.0, 8, {'PTB_GATHER_CC': '64'}) == ('ldg<0>', 'window')
    assert P(128, 128, 1089, 128.0, 8, {}) == ('ldg<0>', 'window')                     # r = 16
    assert P(64, 64, 1, 0.0, 8, {}) == ('ldg<0>', 'reach0')
    assert P(64, 64, 289, 64.0, 8, {}, feats=False) == ('ldg<0>', 'reach0')
    assert P(272, 276, 289, 64.0, 8, {'PTB_GATHER_TMA': '1'}) == ('ldg<0>', None)      # 272 has no 32-channel chunks
    assert P(16, 16, 289, 64.0, 8, {}, G=0) == (None, None)
