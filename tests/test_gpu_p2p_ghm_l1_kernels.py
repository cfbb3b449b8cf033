"""GPU: the GHM-C, GHM-R, L1Loss and BalancedL1Loss kernels of P2PHead.

The bin step (ptb_ghm{c,r}_bin_weights) against the exact restatement of tests/p2p_loss_ref.py: counts equal, and tot, bin_weight and
acc_sum bit for bit, at every bin count the head allows, on planted elements whose g sits exactly on an edge or one ulp from it, with
duplicate edges, NaNs, labels outside the classes, empty and one-bin images, momentum over two steps, every grid shape of the
histogram (one CTA per image up to the grid cap and several grid-stride trips) and an image of more than 2^24 valid elements.

The loss passes against the float64 reference on the kernel's own bins, with the checks of test_gpu_p2p_loss_kernels.py: sums within
1e-5 relative, gradients at scale 0.75 within 1e-5 scale-relative, zero-weight and no-bin elements with a gradient of exactly 0, two
calls with identical bits and NaN exactly where float64 torch has it; the sum plumbing every fixed-order sum shares; and P2PHead.loss at
the bench shape against float64 built from the head's own targets.  The largest errors seen are printed."""
import numpy as np
import pytest
import torch

from oracle import p2p_loss_types as olt
from tests import p2p_loss_ref as ref
from tests.helpers import scale_rel_err
from tests.test_gpu_p2p_defaults import TRAIN_CFG

pytestmark = pytest.mark.gpu

TOL = 1e-5
GRID = ref.SUM_GRID
BENCH_Q, DEFAULT_Q = 100 * 168, 100 * 168 * 4          # proposals of one 100x168 image at 1 and at 4 anchors per cell
POINT_SIZES = [1, 128, (GRID - 1) // 2, GRID // 2, GRID // 2 + 1, DEFAULT_Q]      # n = 2Q: 2 .. one trip + 2, and the head's
BALANCED_PARAMS = [(0.5, 1.5, 1.0), (0.5, 1.5, 0.11), (0.25, 3.0, 1.0 / 9.0)]
GHMC_LAST, GHMR_LAST = None, 1e3                       # ghm_edges: GHMC's last edge 1 + 1e-6, GHMR's 1e3
# planted GHMC logits with their targets and g: 0 gives g = 0.5 (an interior edge when bins is even); +17 gives p = 1.0 and -100.5
# p = 0.0 exactly (g exactly 0 or 1 by the target); -17 with t = 1 gives g = 0.99999994, not 1
PLANTED_C = [(0.0, 0), (0.0, 1), (17.0, 0), (17.0, 1), (-100.5, 0), (-100.5, 1), (-17.0, 1), (-17.0, 0), (16.5, 0), (1e-30, 1)]

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


DEV = torch.device('cuda:0')


def _to(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


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


def _bits(t):
    return t.detach().cpu().contiguous().numpy().tobytes()


# ---------------------------------------------------------------------------------------------------------------------------------
# the bin step
def ghmc_batch(B, Q, C, seed, plant=True, empty=(), one_bin=()):
    """(B, Q, C) logits, labels (B, Q) with -1, C and C + 3 among them, 0/1 label weights with zero rows; planted logits; images in
    `empty` have no valid row, images in `one_bin` only logits whose g lies in the lowest bin."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Q, C, generator=g) * 4
    lab = torch.randint(0, C, (B, Q), generator=g)
    r = torch.randint(0, 8, (B, Q), generator=g)
    lab = torch.where(r == 0, torch.full_like(lab, C), torch.where(r == 1, torch.full_like(lab, -1), lab))
    lab = torch.where(r == 2, torch.full_like(lab, C + 3), lab)
    lw = (torch.rand(B, Q, generator=g) > 0.15).float()
    for b in range(B):
        if plant and Q * C >= 2 * len(PLANTED_C):
            rows = torch.randperm(Q, generator=g)[:len(PLANTED_C)]
            for (v, t), q in zip(PLANTED_C, rows.tolist()):
                c = int(torch.randint(0, C, (1,), generator=g))
                lw[b, q] = 1.0
                if t:
                    lab[b, q] = c
                elif lab[b, q] == c:
                    lab[b, q] = C
                x[b, q, c] = v
            nan_q = int(torch.randint(0, Q, (1,), generator=g))
            lw[b, nan_q] = 1.0
            x[b, nan_q, 0] = float('nan')                    # valid, in no bin, counted in tot
        if b in empty:
            lw[b] = 0.0
        if b in one_bin:                                     # g < 1e-3: every valid element in bin 0
            lab[b] = C
            x[b] = -20.0 - torch.rand(Q, C, generator=g)
    return x, lab, lw


def check_ghmc_bins(ops, x, lab, lw, edges, mmt=0.0, acc=None, what=''):
    """one ghmc_bin_weights call against the restatement; acc (CPU) is updated as the kernel updates its device copy."""
    B, Q, C = x.shape
    acc_d = None if acc is None else acc.to(DEV)
    xd, ld, wd, ed = _to(x, lab, lw, edges)
    counts, bw, tot = ops.ghmc_bin_weights(xd, ld, wd, ed, mmt, acc_d)
    gg = ref.ghmc_g_f32(x, lab).reshape(B, -1)
    valid = (lw > 0)[:, :, None].expand(B, Q, C).reshape(B, -1)
    c_r, idx, bw_r, tot_r = ref.ghm_bin_step(gg, valid, edges, mmt, acc)
    assert torch.equal(counts.cpu().long(), c_r), f'{what}: counts {counts.cpu().tolist()} vs {c_r.tolist()}'
    assert _bits(tot) == _bits(tot_r), f'{what}: tot {tot.cpu().tolist()} vs {tot_r.tolist()}'
    assert _bits(bw) == _bits(bw_r), f'{what}: bin weights differ'
    if acc is not None:
        assert _bits(acc_d) == _bits(acc), f'{what}: acc_sum {acc_d.cpu().tolist()} vs {acc.tolist()}'
    return counts, bw, tot, idx


@pytest.mark.parametrize('bins', [1, 2, 10, 30, 255, 256])
@pytest.mark.parametrize('last', ['+1e-6', '1.0'])
def test_ghmc_bins_at_the_default_edges(ops, bins, last):
    """g = 1 lies in the last bin with GHMC's +1e-6 and in none without it; g = 0.5 is an edge at even bins"""
    edges = olt.ghm_edges(bins, GHMC_LAST if last == '+1e-6' else 1.0)
    x, lab, lw = ghmc_batch(3, 97, 7, bins)
    counts, _, _, idx = check_ghmc_bins(ops, x, lab, lw, edges, what=f'bins={bins} last={last}')
    g = ref.ghmc_g_f32(x, lab).reshape(3, -1)
    valid = (lw > 0)[:, :, None].expand(3, 97, 7).reshape(3, -1)
    ones = (g == 1.0) & valid
    assert bool(ones.any()) and bool(((g == 0.0) & valid).any()) and bool((torch.isnan(g) & valid).any())
    assert bool((idx[ones] == (bins - 1 if last == '+1e-6' else -1)).all())
    assert bool((idx[torch.isnan(g)] == -1).all())
    if bins % 2 == 0:
        half = (g == 0.5) & valid
        assert bool(half.any()) and bool((idx[half] == bins // 2).all()), 'g = 0.5 opens the upper half'


def _planted_edges(g):
    """nondecreasing edges through the planted g values: exactly at one, one ulp either side of others, and duplicates (empty bins)"""
    v = np.unique(g[np.isfinite(g) & (g > 0.01) & (g < 0.99)].astype(np.float32))
    pick = v[np.linspace(0, len(v) - 1, 6).astype(int)]
    e = [np.float32(0), pick[0], np.nextafter(pick[1], np.float32(np.inf)), np.nextafter(pick[2], np.float32(-np.inf)),
         pick[3], pick[3], pick[3], np.float32(0.5), np.float32(0.5), pick[4], np.nextafter(pick[5], np.float32(-np.inf)),
         pick[5], np.float32(1.0) + np.float32(1e-6)]
    e = np.sort(np.array(e, np.float32))
    return torch.from_numpy(e), pick


@pytest.mark.parametrize('mmt', [0.0, 0.75])
def test_ghmc_bins_at_custom_edges_on_planted_g(ops, mmt):
    x, lab, lw = ghmc_batch(2, 300, 5, 7)
    lw[:] = 1.0
    g = ref.ghmc_g_f32(x, lab).reshape(-1).numpy()
    edges, pick = _planted_edges(g)
    acc = torch.rand(edges.numel() - 1) * 100 if mmt else None
    counts, _, _, idx = check_ghmc_bins(ops, x, lab, lw, edges, mmt, acc, what=f'custom edges mmt={mmt}')
    gi = torch.from_numpy(g).reshape(2, -1)
    e = edges.numpy()
    for p in pick[[0, 3, 5]]:                              # g exactly on an edge opens the bin that starts there
        at = gi == float(p)
        assert bool(at.any())
        first = int(np.nonzero(e == p)[0].max())
        assert bool((idx[at] == first).all())
    empty = [i for i in range(len(e) - 1) if e[i] == e[i + 1]]
    assert empty and bool((counts[:, empty] == 0).all()), 'zero-width bins stay empty'


@pytest.mark.parametrize('n', [1, 31, 255, 2047, 2048, 2049])
@pytest.mark.parametrize('B', [1, 2, 3, 16, 17])
def test_ghmc_bins_at_every_image_size_and_batch(ops, n, B):
    """n elements per image (C = 1); each image's counts equal the histogram of that image alone"""
    x, lab, lw = ghmc_batch(B, n, 1, 100 * n + B, plant=n >= 20)
    edges = olt.ghm_edges(10, GHMC_LAST)
    counts, bw, tot, _ = check_ghmc_bins(ops, x, lab, lw, edges, what=f'n={n} B={B}')
    for b in {0, B // 2, B - 1}:
        c1, bw1, t1 = ops.ghmc_bin_weights(*_to(x[b:b + 1], lab[b:b + 1], lw[b:b + 1], edges))
        assert torch.equal(c1[0], counts[b]) and torch.equal(bw1[0], bw[b]) and torch.equal(t1[0], tot[b]), f'image {b} alone'


def test_ghmc_bins_where_the_grid_cap_binds(ops):
    """one image of 3.2 M elements: 528 CTAs at most (4 per SM at 132 SMs), each several grid-stride trips; then more images than
    4 x the SM count, one CTA per image"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    x, lab, lw = ghmc_batch(1, 40_000, 80, 3)
    assert x.numel() > 4 * sms * 256 * 8 * 2
    check_ghmc_bins(ops, x, lab, lw, olt.ghm_edges(30, GHMC_LAST), what='one large image')
    B = 4 * sms + 7
    x, lab, lw = ghmc_batch(B, 700, 4, 4)
    check_ghmc_bins(ops, x, lab, lw, olt.ghm_edges(10, GHMC_LAST), 0.75, torch.rand(10) * 10, what=f'B={B}')


@pytest.mark.parametrize('mmt', [0.0, 0.75, 0.7, 1e-3])
def test_ghmc_bins_with_empty_and_one_bin_images_over_two_steps(ops, mmt):
    """image 1 has no valid element (tot 1, all weights 0, acc_sum untouched by it), image 2 one non-empty bin; two steps in a row
    with the state the first left.  0.7 is not exact in fp32: the update takes fp32(mmt)."""
    bins = 30
    edges = olt.ghm_edges(bins, GHMC_LAST)
    acc = (torch.rand(bins) * 40) if mmt else None
    for step in range(2):
        x, lab, lw = ghmc_batch(4, 400, 6, 50 + step, empty=(1,), one_bin=(2,))
        counts, bw, tot, _ = check_ghmc_bins(ops, x, lab, lw, edges, mmt, acc, what=f'mmt={mmt} step {step}')
        assert float(tot[1]) == 1.0 and bool((bw[1] == 0).all()) and int(counts[1].sum()) == 0
        assert int((counts[2, :bins] > 0).sum()) == 1 and int(counts[2, 0]) == int(counts[2, bins])
    if mmt:
        # on their own: the empty image leaves every acc_sum entry as it was, the one-bin image changes entry 0 only
        for b, changed in ((1, []), (2, [0])):
            acc_d = acc.to(DEV)
            ops.ghmc_bin_weights(*_to(x[b:b + 1], lab[b:b + 1], lw[b:b + 1], edges), mmt, acc_d)
            diff = torch.nonzero(acc_d.cpu() != acc).reshape(-1).tolist()
            assert diff == changed, f'image {b} alone changed acc_sum entries {diff}'


def test_ghmc_bins_above_2_24_valid_elements(ops):
    """1203 classes on a 67 200-row image: 27 895 valid rows give 33 557 685 valid elements, which fp32 cannot hold: tot is the count
    rounded once, within one ulp of the reference's fp32 sum of the valid mask"""
    Q, C, nv = DEFAULT_Q, 1203, 27_895
    g = torch.Generator().manual_seed(1203)
    x = torch.randn(1, Q, C, generator=g) * 4
    lab = torch.randint(0, C + 1, (1, Q), generator=g)
    lw = torch.zeros(1, Q)
    lw[0, torch.randperm(Q, generator=g)[:nv]] = 1.0
    counts, _, tot, _ = check_ghmc_bins(ops, x, lab, lw, olt.ghm_edges(10, GHMC_LAST), what='1203 classes')
    count = nv * C
    assert count > 2 ** 25 and int(counts[0, -1]) == count
    t = np.float32(tot.cpu()[0])
    assert t == np.float32(count)
    s = float((lw > 0)[:, :, None].expand(1, Q, C).float().sum())
    assert abs(float(t) - s) <= float(np.spacing(t)), (float(t), s)


def ghmr_batch(B, Q, seed, weights='points'):
    g = torch.Generator().manual_seed(seed)
    p, t = torch.randn(B, Q, 2, generator=g) * 30, torch.randn(B, Q, 2, generator=g) * 30
    inv = (1.0 / torch.tensor([8.0, 16.0, 32.0, 64.0, 128.0]))[torch.randint(0, 5, (Q,), generator=g)]
    if weights == 'points':
        w = (torch.rand(B, Q, 1, generator=g) > 0.4).float().expand(B, Q, 2).contiguous()
    else:
        w = torch.rand(B, Q, 2, generator=g) * (torch.rand(B, Q, 2, generator=g) > 0.3)
    if Q >= 4:
        p[:, 0] = t[:, 0]                                # d = 0: g = 0
        w[:, 0] = 1.0
        p[:, 1, 0] = float('nan')                        # valid, in no bin
        w[:, 1] = 1.0
        p[:, 2] = t[:, 2] + 1e-3
    return p, t, inv, w


def check_ghmr_bins(ops, p, t, inv, w, mu, edges, mmt=0.0, acc=None, what=''):
    B, Q, _ = p.shape
    acc_d = None if acc is None else acc.to(DEV)
    counts, bw, tot = ops.ghmr_bin_weights(*_to(p, t, w, inv), mu, edges.to(DEV), mmt, acc_d)
    gg = ref.ghmr_g_f32(p, t, inv, mu).reshape(B, -1)
    c_r, idx, bw_r, tot_r = ref.ghm_bin_step(gg, (w > 0).reshape(B, -1), edges, mmt, acc)
    assert torch.equal(counts.cpu().long(), c_r), f'{what}: counts {counts.cpu().tolist()} vs {c_r.tolist()}'
    assert _bits(tot) == _bits(tot_r) and _bits(bw) == _bits(bw_r), f'{what}: tot / bin weights differ'
    if acc is not None:
        assert _bits(acc_d) == _bits(acc), f'{what}: acc_sum'
    return counts, bw, tot, idx


@pytest.mark.parametrize('bins,mmt', [(1, 0.0), (10, 0.0), (10, 0.7), (30, 0.75), (256, 1e-3)])
@pytest.mark.parametrize('B,Q', [(1, 1), (2, 1000), (17, 300), (1, 700_000)])
def test_ghmr_bins(ops, bins, mmt, B, Q):
    edges = olt.ghm_edges(bins, GHMR_LAST)
    acc = torch.rand(bins) * 20 if mmt else None
    for step in range(2 if mmt else 1):
        p, t, inv, w = ghmr_batch(B, Q, 10 * bins + step)
        check_ghmr_bins(ops, p, t, inv, w, 0.02, edges, mmt, acc, what=f'bins={bins} mmt={mmt} B={B} Q={Q} step {step}')


def test_ghmr_tot_counts_positive_weights_not_their_sum(ops):
    """the documented difference from the reference: with fractional weights tot is the number of weights > 0 (the head's point
    weights are 0 or 1, where the two agree)"""
    p, t, inv, w = ghmr_batch(2, 500, 3, weights='mixed')
    counts, _, tot, _ = check_ghmr_bins(ops, p, t, inv, w, 0.02, olt.ghm_edges(10, GHMR_LAST), what='fractional weights')
    for b in range(2):
        assert float(tot[b]) == float((w[b] > 0).sum()) != float(w[b].sum())


# ---------------------------------------------------------------------------------------------------------------------------------
# the loss passes on the kernel's bins
GHMC_SHAPES = [(1, 1), (255, 1), (GRID - 1, 1), (GRID, 1), (GRID + 1, 1), (GRID // 80 + 1, 80), (DEFAULT_Q, 80)]


def _ghmc_loss_case(ops, x, lab, lw, edges, what, key):
    counts, bw, tot, idx = check_ghmc_bins(ops, x[None], lab[None], lw[None], edges, what=what)
    s, gr = ref.ghmc(x, lab, lw, idx[0], bw[0].cpu())
    xd, ld, wd, ed, bwd = _to(x, lab, lw, edges, bw[0])
    call = lambda scale=None, want_grad=False: ops.ghmc(xd, ld, wd, ed, bwd, scale=scale, want_grad=want_grad)  # noqa: E731
    Q, C = x.shape
    zero = ((lw == 0)[:, None].expand(Q, C) | (idx[0] < 0).reshape(Q, C))
    check_loss(call, xd, s, gr, what, key, zero)


@pytest.mark.parametrize('Q,C', GHMC_SHAPES)
@pytest.mark.parametrize('bins', [10, 30])
def test_ghmc_loss_matches_float64(ops, Q, C, bins):
    x, lab, lw = ghmc_batch(1, Q, C, Q + C + bins, plant=Q * C >= 100)
    x[0].view(-1)[torch.isnan(x[0].view(-1))] = 0.25       # the NaN case has its own test
    if Q == 1:
        lw[:] = 1.0
    _ghmc_loss_case(ops, x[0], lab[0], lw[0], olt.ghm_edges(bins, GHMC_LAST), f'GHMC Q={Q} C={C} bins={bins}', 'GHMC')


def test_ghmc_loss_at_1203_classes(ops):
    x, lab, lw = ghmc_batch(1, DEFAULT_Q, 1203, 12, plant=False)
    _ghmc_loss_case(ops, x[0], lab[0], lw[0], olt.ghm_edges(10, GHMC_LAST), 'GHMC Q=67200 C=1203', 'GHMC 1203')


@pytest.mark.parametrize('Q', POINT_SIZES)
@pytest.mark.parametrize('bins', [10, 30])
def test_ghmr_loss_matches_float64(ops, Q, bins):
    p, t, inv, w = ghmr_batch(1, Q, Q + bins)
    if Q > 1:
        p[0, 1, 0] = 0.5                                      # the NaN case has its own test
    _, bw, _, idx = check_ghmr_bins(ops, p, t, inv, w, 0.02, olt.ghm_edges(bins, GHMR_LAST), what=f'GHMR Q={Q}')
    s, gr = ref.ghmr(p[0], t[0], w[0], inv, 0.02, idx[0], bw[0].cpu())
    pd, td, wd, invd, ed, bwd = _to(p[0], t[0], w[0], inv, olt.ghm_edges(bins, GHMR_LAST), bw[0])
    call = lambda scale=None, want_grad=False: ops.ghmr(pd, td, wd, invd, 0.02, ed, bwd, scale=scale, want_grad=want_grad)  # noqa: E731
    check_loss(call, pd, s, gr, f'GHMR Q={Q} bins={bins}', 'GHMR', (w[0] == 0) | (idx[0] < 0).reshape(Q, 2))


def points_case(Q, seed, weights, beta=1.0):
    """(Q, 2) points with five strides; the first rows carry planted normalised differences on target 0: |d| == beta exactly, one
    ulp either side, +-0 and tiny values (the product pred * inv is exact: inv is a power of two and pred = d / inv)"""
    g = torch.Generator().manual_seed(seed)
    p, t = torch.randn(Q, 2, generator=g) * 30, torch.randn(Q, 2, generator=g) * 30
    inv = (1.0 / torch.tensor([8.0, 16.0, 32.0, 64.0, 128.0]))[torch.randint(0, 5, (Q,), generator=g)]
    b32 = np.float32(beta)
    planted = np.array([b32, -b32, np.nextafter(b32, np.float32(0)), np.nextafter(b32, np.float32(np.inf)),
                        -np.nextafter(b32, np.float32(0)), 0.0, -0.0, 1e-7, -3e-6, 1e-30], np.float32)
    k = min(len(planted), 2 * Q) if Q > 1 else 0
    if k:
        fp, ft = p.view(-1), t.view(-1)
        rows = torch.arange(k) // 2
        ft[:k] = 0.0
        fp[:k] = torch.from_numpy(planted[:k]) / inv[rows]
        got = (fp[:k].numpy() - ft[:k].numpy()) * inv[rows].numpy()
        assert np.array_equal(got, planted[:k]) and np.array_equal(np.signbit(got), np.signbit(planted[:k])), 'planted d exact'
    if weights == 'none':
        w = None
    elif weights == 'points':
        w = (torch.rand(Q, generator=g) > 0.4).float()[:, None].expand(Q, 2).contiguous()
    else:
        w = torch.rand(Q, 2, generator=g) * 2 * (torch.rand(Q, 2, generator=g) > 0.2)
    return p, t, inv, w


@pytest.mark.parametrize('weights', ['none', 'points', 'mixed'])
def test_l1_loss_matches_float64(ops, weights):
    for i, Q in enumerate(POINT_SIZES):
        p, t, inv, w = points_case(Q, 70 + i, weights)
        s, gr = ref.l1_rows(p, t, w, inv)
        pd, td, invd, wd = _to(p, t, inv, w)
        call = lambda scale=None, want_grad=False: ops.l1_rows(pd, td, wd, invd, scale=scale, want_grad=want_grad)  # noqa: E731
        zero = (p - t == 0) | (torch.zeros_like(p, dtype=torch.bool) if w is None else w == 0)
        check_loss(call, pd, s, gr, f'L1 Q={Q} w={weights}', 'L1', zero)


@pytest.mark.parametrize('alpha,gamma,beta', BALANCED_PARAMS)
@pytest.mark.parametrize('weights', ['none', 'points', 'mixed'])
def test_balanced_l1_loss_matches_float64(ops, alpha, gamma, beta, weights):
    for i, Q in enumerate(POINT_SIZES):
        p, t, inv, w = points_case(Q, 80 + i, weights, beta)
        s, gr = ref.balanced_l1_rows(p, t, w, inv, alpha, gamma, beta)
        pd, td, invd, wd = _to(p, t, inv, w)
        call = lambda scale=None, want_grad=False: ops.balanced_l1_rows(pd, td, wd, invd, alpha, gamma, beta, scale=scale,  # noqa: E731
                                                                        want_grad=want_grad)
        zero = (p - t == 0) | (torch.zeros_like(p, dtype=torch.bool) if w is None else w == 0)
        check_loss(call, pd, s, gr, f'BalancedL1 {alpha},{gamma},{beta} Q={Q} w={weights}', 'BalancedL1', zero)


@pytest.mark.parametrize('alpha,gamma,beta', BALANCED_PARAMS)
def test_balanced_l1_small_differences_stay_within_the_size_of_the_cancelling_terms(ops, alpha, gamma, beta):
    """for |d| << beta the two terms kab (kb a + 1) log(u), about alpha a / beta, and alpha a cancel (at beta = 1 to about
    alpha b a^2 / 2) in fp32, as in the reference's own fp32 arithmetic: the sum's relative error exceeds 1e-5 at beta = 1.  It is
    bounded by a few eps times the size of the cancelling terms, sum alpha a / min(beta, 1), not by the size of the result."""
    g = torch.Generator().manual_seed(int(beta * 1000))
    Q = 50_000
    inv = torch.full((Q,), 0.125)
    d = (10.0 ** (torch.rand(Q, 2, generator=g) * 3 - 6)) * beta * torch.sign(torch.rand(Q, 2, generator=g) - 0.5)
    t = torch.randn(Q, 2, generator=g)
    p = t + d / 0.125
    s, _ = ref.balanced_l1_rows(p, t, None, inv, alpha, gamma, beta)
    got = float(ops.balanced_l1_rows(*_to(p, t, None, inv), alpha, gamma, beta).cpu())
    a = ((p.double() - t.double()) * 0.125).abs()
    bound = 16 * 2.0 ** -24 * float((ref.f32(alpha) * a / min(ref.f32(beta), 1.0)).sum())
    err = abs(got - float(s))
    _note(f'BalancedL1 small |d| {alpha},{gamma},{beta} error / bound', err / bound)
    assert err <= bound, f'sum {got!r} vs float64 {float(s)!r}: error {err:.3e} > {bound:.3e}'


# ---------------------------------------------------------------------------------------------------------------------------------
NAN_LOSSES = ['ghmc', 'ghmr', 'l1', 'balanced_l1']


@pytest.mark.parametrize('loss', NAN_LOSSES)
def test_a_nan_input_makes_the_sum_nan_and_the_gradient_nan_where_torch_has_it(ops, loss):
    """one NaN in a zero-weight row, one in a weighted row past the first trip of the sum grid.  GHM: a NaN is valid but in no bin
    (weight 0), and 0 * (sigmoid(NaN) - t) is NaN in torch as in the kernel.  L1: torch's abs backward is sgn(d), 0 at NaN."""
    g = torch.Generator().manual_seed(NAN_LOSSES.index(loss))
    if loss == 'ghmc':
        Q, C = GRID // 80 + 3, 80
        x, lab, lw = ghmc_batch(1, Q, C, 5, plant=False)
        lw[0, 3], lw[0, Q - 2] = 0.0, 1.0
        x[0, 3, 5] = x[0, Q - 2, 7] = float('nan')
        edges = olt.ghm_edges(10, GHMC_LAST)
        _, bw, _, idx = check_ghmc_bins(ops, x, lab, lw, edges, what='GHMC NaN')
        s, gr = ref.ghmc(x[0], lab[0], lw[0], idx[0], bw[0].cpu())
        xd, ld, wd, ed, bwd = _to(x[0], lab[0], lw[0], edges, bw[0])
        call = lambda scale=None, want_grad=False: ops.ghmc(xd, ld, wd, ed, bwd, scale=scale, want_grad=want_grad)  # noqa: E731
        inp = x[0]
    else:
        Q = GRID // 2 + 5
        p, t, inv, w = ghmr_batch(1, Q, 6) if loss == 'ghmr' else (*points_case(Q, 6, 'points')[:3], None)
        p, t = p.reshape(Q, 2), t.reshape(Q, 2)
        w = torch.ones(Q, 2) if w is None else w.reshape(Q, 2)
        w[3] = 0
        p[1, 0] = 0.5
        p[3, 1] = p[GRID // 2 + 1, 0] = float('nan')
        w[GRID // 2 + 1] = 1.0
        pd, td, wd, invd = _to(p, t, w, inv)
        if loss == 'ghmr':
            edges = olt.ghm_edges(10, GHMR_LAST)
            _, bw, _, idx = check_ghmr_bins(ops, p[None], t[None], inv, w[None], 0.02, edges, what='GHMR NaN')
            s, gr = ref.ghmr(p, t, w, inv, 0.02, idx[0], bw[0].cpu())
            ed, bwd = _to(edges, bw[0])
            call = lambda scale=None, want_grad=False: ops.ghmr(pd, td, wd, invd, 0.02, ed, bwd, scale=scale,  # noqa: E731
                                                                want_grad=want_grad)
        elif loss == 'l1':
            s, gr = ref.l1_rows(p, t, w, inv)
            call = lambda scale=None, want_grad=False: ops.l1_rows(pd, td, wd, invd, scale=scale, want_grad=want_grad)  # noqa: E731
            # the reference model trains on the GPU: torch's CUDA float64 autograd gives the same gradient at the NaN
            pc = p.double().to(DEV).requires_grad_(True)
            ((pc - t.double().to(DEV)) * inv.double().to(DEV)[:, None]).abs().mul(w.double().to(DEV)).sum().backward()
            cuda_g = pc.grad.cpu()
            print(f'[L1 at NaN] torch CUDA float64 gradient {cuda_g[3].tolist()} / {cuda_g[GRID // 2 + 1].tolist()}, '
                  f'CPU {gr[3].tolist()} / {gr[GRID // 2 + 1].tolist()}')
            assert torch.equal(torch.isnan(cuda_g), torch.isnan(gr))
        else:
            s, gr = ref.balanced_l1_rows(p, t, w, inv, 0.5, 1.5, 1.0)
            call = lambda scale=None, want_grad=False: ops.balanced_l1_rows(pd, td, wd, invd, 0.5, 1.5, 1.0, scale=scale,  # noqa: E731
                                                                            want_grad=want_grad)
        inp = p
    assert torch.isnan(s)
    want_nan = {'ghmc': 2, 'ghmr': 2, 'l1': 0, 'balanced_l1': 2}[loss]
    assert int(torch.isnan(gr).sum()) == want_nan, f'float64 {loss}: NaN gradient at {int(torch.isnan(gr).sum())} elements'
    check_loss(call, inp.to(DEV), s, gr, f'NaN {loss}', f'NaN {loss}')


# ---------------------------------------------------------------------------------------------------------------------------------
# the fixed-order sum these four share with the other losses
def _sum_jobs(ops):
    jobs = []
    x, lab, lw = ghmc_batch(1, GRID // 80 + 1, 80, 9, plant=False)
    edges_c = olt.ghm_edges(10, GHMC_LAST).to(DEV)
    xd, ld, wd = _to(x, lab, lw)
    _, bwc, _ = ops.ghmc_bin_weights(xd, ld, wd, edges_c)
    jobs.append(('GHMC', lambda: ops.ghmc(xd[0], ld[0], wd[0], edges_c, bwc[0])))
    x1, l1, w1 = _to(torch.randn(1, 1), torch.zeros(1, dtype=torch.int64), torch.ones(1))
    _, bw1, _ = ops.ghmc_bin_weights(x1[None], l1[None], w1[None], edges_c)
    jobs.append(('GHMC n=1', lambda: ops.ghmc(x1, l1, w1, edges_c, bw1[0])))
    p, t, inv, w = ghmr_batch(1, GRID // 2 + 1, 9)
    p[:, 1, 0] = 0.5                                         # a finite sum: equal sums are compared bit for bit
    edges_r = olt.ghm_edges(10, GHMR_LAST).to(DEV)
    pr, tr, invr, wr = _to(p, t, inv, w)
    _, bwr, _ = ops.ghmr_bin_weights(pr, tr, wr, invr, 0.02, edges_r)
    jobs.append(('GHMR', lambda: ops.ghmr(pr[0], tr[0], wr[0], invr, 0.02, edges_r, bwr[0])))
    p, t, inv, w = _to(*points_case(255, 9, 'points'))
    jobs.append(('L1', lambda: ops.l1_rows(p, t, w, inv)))
    jobs.append(('BalancedL1', lambda: ops.balanced_l1_rows(p, t, w, inv, 0.5, 1.5, 1.0)))
    pb, tb, invb, _ = _to(*points_case(GRID // 2 + 3, 10, 'none'))
    jobs.append(('BalancedL1 large', lambda: ops.balanced_l1_rows(pb, tb, None, invb, 0.25, 3.0, 1.0 / 9.0)))
    xf, lf = _to(torch.randn(300, 80), torch.randint(0, 80, (300,)))
    jobs.append(('focal', lambda: ops.sigmoid_focal(xf, lf, None, 2.0, 0.25)))
    return jobs


def _solo(jobs):
    out = []
    for _, fn in jobs:
        r = fn()
        torch.cuda.synchronize()
        out.append(r.clone())
    return out


def test_back_to_back_sums_on_one_stream_leave_each_other_alone(ops):
    jobs = _sum_jobs(ops)
    solo = _solo(jobs)
    order = [0, 1, 2, 3, 4, 5, 6, 1, 0, 5, 3, 2, 4, 6, 1, 1, 5, 5, 0, 2]
    got = [jobs[i][1]() for i in order]
    torch.cuda.synchronize()
    for i, r in zip(order, got):
        assert torch.equal(r, solo[i]), f'{jobs[i][0]}: {float(r)} interleaved vs {float(solo[i])} solo'


def test_concurrent_sums_on_two_streams_use_their_own_slots(ops):
    jobs = _sum_jobs(ops)
    solo = _solo(jobs)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a, b = [0, 2, 1, 5, 0, 2], [3, 4, 6, 3, 5, 4]
    torch.cuda.synchronize()
    main = torch.cuda.current_stream()
    ra, rb = [], []
    for _ in range(3):
        torch.cuda._sleep(50_000_000)          # holds both streams back until all their launches are queued, so that they overlap
        s1.wait_stream(main)
        s2.wait_stream(main)
        for i, j in zip(a, b):
            with torch.cuda.stream(s1):
                ra.append((i, jobs[i][1]()))
            with torch.cuda.stream(s2):
                rb.append((j, jobs[j][1]()))
    torch.cuda.synchronize()
    for i, r in ra + rb:
        assert torch.equal(r, solo[i]), f'{jobs[i][0]}: {float(r)} on two streams vs {float(solo[i])} solo'


def test_sums_after_reset_stream_state(ops):
    from pointtinybenchmark_b200 import _lib
    from pointtinybenchmark_b200.ops import _stream
    jobs = _sum_jobs(ops)
    solo = _solo(jobs)
    for i, (_, fn) in enumerate(jobs):
        assert _lib.load().ptb_reset_stream_state(_stream()) == 0
        assert torch.equal(fn(), solo[i]), jobs[i][0]
    torch.cuda.synchronize()


def test_each_loss_call_is_one_launch_and_the_bin_step_two(ops):
    x, lab, lw = _to(*ghmc_batch(2, 300, 80, 1))
    p, t, inv, w = _to(*ghmr_batch(2, 300, 1))
    ec, er = _to(olt.ghm_edges(10, GHMC_LAST), olt.ghm_edges(10, GHMR_LAST))
    acc = torch.zeros(10, device=DEV)
    n0 = ops.launch_count()
    _, bwc, _ = ops.ghmc_bin_weights(x, lab, lw, ec, 0.75, acc)
    _, bwr, _ = ops.ghmr_bin_weights(p, t, w, inv, 0.02, er)
    assert ops.launch_count() - n0 == 4
    sc = torch.ones(1, device=DEV)
    calls = [lambda **k: ops.ghmc(x[0], lab[0], lw[0], ec, bwc[0], **k), lambda **k: ops.ghmr(p[0], t[0], w[0], inv, 0.02, er, bwr[0], **k),
             lambda **k: ops.l1_rows(p[0], t[0], w[0], inv, **k), lambda **k: ops.balanced_l1_rows(p[0], t[0], None, inv, 0.5, 1.5, 1.0, **k)]
    for c in calls:
        for kw in ({}, dict(scale=sc, want_grad=True)):
            n0 = ops.launch_count()
            c(**kw)
            assert ops.launch_count() - n0 == 1


def test_one_launch_with_both_outputs_gives_the_bits_of_two(ops):
    """the C entry points take loss_sum and grad together; scale NULL with a gradient means scale 1"""
    from pointtinybenchmark_b200 import _lib
    from pointtinybenchmark_b200.ops import _ptr, _stream
    lib = _lib.load()
    x, lab, lw = _to(*ghmc_batch(1, GRID // 80 + 1, 80, 2))
    x[torch.isnan(x)] = 0.5
    p, t, inv, w = _to(*ghmr_batch(1, GRID // 2 + 1, 2))
    p[torch.isnan(p)] = 0.5
    ec, er = _to(olt.ghm_edges(30, GHMC_LAST), olt.ghm_edges(10, GHMR_LAST))
    _, bwc, _ = ops.ghmc_bin_weights(x, lab, lw, ec)
    _, bwr, _ = ops.ghmr_bin_weights(p, t, w, inv, 0.02, er)
    x, lab, lw, p, t, w = x[0], lab[0], lw[0], p[0], t[0], w[0]
    Q, C = x.shape
    M = p.shape[0]
    entries = [
        ('GHMC', x, lambda *o: lib.ptb_ghmc_fwd_bwd(_ptr(x), _ptr(lab), _ptr(lw), Q, C, _ptr(ec), 30, _ptr(bwc[0]), *o)),
        ('GHMR', p, lambda *o: lib.ptb_ghmr_fwd_bwd(_ptr(p), _ptr(t), _ptr(w), M, _ptr(inv), 0.02, _ptr(er), 10, _ptr(bwr[0]), *o)),
        ('L1', p, lambda *o: lib.ptb_l1_rows_fwd_bwd(_ptr(p), _ptr(t), _ptr(w), M, _ptr(inv), *o)),
        ('BalancedL1', p, lambda *o: lib.ptb_balanced_l1_rows_fwd_bwd(_ptr(p), _ptr(t), None, M, _ptr(inv), 0.5, 1.5, 0.11, *o)),
    ]
    one = torch.ones(1, device=DEV)
    sc = torch.tensor([-2.5], device=DEV)
    for name, inp, fn in entries:
        def run(want_sum, want_grad, scale):
            s = torch.zeros(1, device=DEV) if want_sum else None
            g = torch.full_like(inp, 123.0) if want_grad else None
            assert fn(_ptr(s), _ptr(scale), _ptr(g), _stream()) == 0, lib.ptb_last_error()
            return s, g
        s_only, _ = run(True, False, None)
        _, g_only = run(False, True, sc)
        s_both, g_both = run(True, True, sc)
        assert torch.equal(s_both, s_only), f'{name}: sum of the fused launch'
        assert torch.equal(g_both, g_only), f'{name}: gradient of the fused launch'
        _, g_null = run(False, True, None)
        _, g_one = run(False, True, one)
        assert torch.equal(g_null, g_one), f'{name}: scale NULL is scale 1'


def test_the_wrappers_refuse_tensors_the_kernels_would_misread(ops):
    """every tensor of ghmc / ghmr / l1_rows / balanced_l1_rows is checked for dtype, device and shape before any launch"""
    x, lab, lw = _to(*ghmc_batch(1, 50, 4, 1, plant=False))
    x, lab, lw = x[0], lab[0], lw[0]
    ec = olt.ghm_edges(10, GHMC_LAST).to(DEV)
    bw = torch.ones(10, device=DEV)
    p, t, inv, w = _to(*ghmr_batch(1, 50, 1))
    p, t, w = p[0], t[0], w[0]
    er = olt.ghm_edges(10, GHMR_LAST).to(DEV)
    n0 = ops.launch_count()
    bad_c = [dict(labels=lab[:-1]), dict(labels=lab.int()), dict(label_weight=lw[:-1]), dict(label_weight=lw.double()),
             dict(label_weight=lw.cpu()), dict(bin_weight=bw[:-1]), dict(bin_weight=torch.ones(11, device=DEV)),
             dict(bin_weight=bw.cpu()), dict(logits=x[None])]
    for kw in bad_c:
        a = dict(logits=x, labels=lab, label_weight=lw, edges=ec, bin_weight=bw)
        a.update(kw)
        with pytest.raises((ValueError, TypeError, RuntimeError)):
            ops.ghmc(**a)
    bad_r = [dict(weight=w[:, 0].contiguous()), dict(weight=w.reshape(-1)), dict(weight=w[:-1]), dict(weight=w.double()),
             dict(weight=w.cpu()), dict(bin_weight=bw[:-1]), dict(bin_weight=bw.half()), dict(pred=p[None], target=t[None])]
    for kw in bad_r:
        a = dict(pred=p, target=t, weight=w, row_inv_norm=inv, mu=0.02, edges=er, bin_weight=bw)
        a.update(kw)
        with pytest.raises((ValueError, TypeError, RuntimeError)):
            ops.ghmr(**a)
    for fn, extra in ((ops.l1_rows, ()), (ops.balanced_l1_rows, (0.5, 1.5, 1.0))):
        for bad in (w[:, 0].contiguous(), w[:-1], w.double(), w.cpu(), w.t()):
            with pytest.raises((ValueError, TypeError, RuntimeError)):
                fn(p, t, bad, inv, *extra)
        with pytest.raises(ValueError):
            fn(p[None], t[None], None, inv, *extra)
    with pytest.raises(RuntimeError, match='gamma'):
        ops.balanced_l1_rows(p, t, w, inv, 0.5, 0.0, 1.0)
    assert ops.launch_count() == n0, 'a refused call launches nothing'


# ---------------------------------------------------------------------------------------------------------------------------------
HEAD_LOSSES = {
    'ghmc+ghmr': (dict(type='GHMC', bins=30, momentum=0.75, use_sigmoid=True, loss_weight=1.5),
                  dict(type='GHMR', mu=0.02, bins=10, loss_weight=0.5)),
    'focal+l1': (dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0), dict(type='L1Loss', loss_weight=0.5)),
    'focal+balanced_l1': (dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                          dict(type='BalancedL1Loss', alpha=0.5, gamma=1.5, beta=0.11, loss_weight=2.0)),
}


def _head(k, losses):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    lc, lr = HEAD_LOSSES[losses]
    hc = dict(type='P2PHead', num_classes=80, in_channels=256, feat_channels=256, stacked_convs=4, strides=[8],
              norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), train_cfg=TRAIN_CFG, loss_cls=dict(lc), loss_reg=dict(lr))
    if k == 1:                                                # bench.py's head: one anchor, pts_gamma 1, reg_norm 1
        hc.update(point_anchor=[(0., 0.)], pts_gamma=1, reg_norm=1)
    return build_head(hc).cuda().train()


@pytest.mark.parametrize('losses', sorted(HEAD_LOSSES))
@pytest.mark.parametrize('k,B', [(1, 3), (4, 2)])
def test_head_loss_at_the_bench_shape_matches_float64_on_its_own_targets(ops, losses, k, B):
    """P2PHead.loss + backward on random 100x168 maps with 20 GTs per image against float64 built from the head's own targets and
    the restated bins: per-image losses (the division by tot or num_total_pos, loss_weight, each image's row of bin weights) and the
    gradients of cls_out and pts_out under upstream gradients other than 1; the head's GHM counts equal the restatement's."""
    head = _head(k, losses)
    lc, lr = HEAD_LOSSES[losses]
    H, W, C, s = 100, 168, 80, 8.0
    g = torch.Generator().manual_seed(60 + k)
    cls_out = (torch.randn(B, k * C, H, W, generator=g) * 2 - 3).to(DEV).requires_grad_(True)
    pts_out = (torch.randn(B, 2 * k, H, W, generator=g) * (0.5 if k == 1 else 0.05)).to(DEV).requires_grad_(True)
    gtb, gtl = [], []
    for _ in range(B):
        cxy = torch.rand(20, 2, generator=g) * torch.tensor([1300., 780.]) + 10
        gtb.append(torch.cat([cxy - 8, cxy + 8], 1).to(DEV))
        gtl.append(torch.randint(0, C, (20,), generator=g).to(DEV))
    metas = [dict(pad_shape=(800, 1344, 3), img_shape=(800, 1333, 3), scale_factor=[1.0] * 4)] * B
    acc0 = head.loss_cls.acc_sum.detach().cpu().clone() if lc['type'] == 'GHMC' else None
    got = head.loss([cls_out], [pts_out], gtb, gtl, metas)
    got_vals = {key: [float(v.detach()) for v in vals] for key, vals in got.items()}
    up_cls = [3.7, 0.6, -1.2][:B]
    up_pts = [-0.25, 1.0, 2.0][:B]
    total = sum(a * l for a, l in zip(up_cls, got['loss_cls'])) + sum(a * l for a, l in zip(up_pts, got['loss_pts']))
    total.backward()
    tg = head._last_targets
    with torch.no_grad():
        _, pred, _, cls = head.get_pred_points(cls_out, pts_out, metas)
    Q = H * W * k
    npos = float(sum(int((p[:, 0] > 0).sum()) for p in tg['pts_weights']))
    assert npos > 0
    row_inv = torch.full((Q,), ref.f32(1.0 / (s * head.reg_norm)))
    labels = torch.stack(tg['labels']).cpu()
    lw = torch.stack(tg['label_weights']).cpu()
    gts, pws = torch.stack(tg['gt_pts']).cpu(), torch.stack(tg['pts_weights']).cpu()
    if lc['type'] == 'GHMC':
        gg = ref.ghmc_g_f32(cls, labels).reshape(B, -1)
        c_r, c_idx, c_bw, c_tot = ref.ghm_bin_step(gg, (lw > 0)[:, :, None].expand(B, Q, C).reshape(B, -1), head.loss_cls.edges.cpu(),
                                                   lc['momentum'], acc0)
        assert torch.equal(head._last_ghm['cls_counts'].cpu().long(), c_r), 'GHMC counts of the head'
        assert _bits(head.loss_cls.acc_sum) == _bits(acc0), 'GHMC acc_sum of the head'
    if lr['type'] == 'GHMR':
        gg = ref.ghmr_g_f32(pred, gts, row_inv, lr['mu']).reshape(B, -1)
        r_r, r_idx, r_bw, r_tot = ref.ghm_bin_step(gg, (pws > 0).reshape(B, -1), head.loss_reg.edges.cpu())
        assert torch.equal(head._last_ghm['reg_counts'].cpu().long(), r_r), 'GHMR counts of the head'
    g_cls, g_pts = [], []
    for b in range(B):
        if lc['type'] == 'GHMC':
            sc, gc = ref.ghmc(cls[b], labels[b], lw[b], c_idx[b], c_bw[b])
            norm_c = float(c_tot[b]) / lc['loss_weight']
        else:
            sc, gc = ref.focal(cls[b], labels[b], lw[b], lc['gamma'], lc['alpha'])
            norm_c = npos / lc['loss_weight']
        if lr['type'] == 'GHMR':
            sp, gp = ref.ghmr(pred[b], gts[b], pws[b], row_inv, lr['mu'], r_idx[b], r_bw[b])
            norm_p = float(r_tot[b]) / lr['loss_weight']
        elif lr['type'] == 'L1Loss':
            sp, gp = ref.l1_rows(pred[b], gts[b], pws[b], row_inv)
            norm_p = npos / lr['loss_weight']
        else:
            sp, gp = ref.balanced_l1_rows(pred[b], gts[b], pws[b], row_inv, lr['alpha'], lr['gamma'], lr['beta'])
            norm_p = npos / lr['loss_weight']
        for what, want in (('loss_cls', float(sc) / norm_c), ('loss_pts', float(sp) / norm_p)):
            val = got_vals[what][b]
            e = abs(val - want) / abs(want)
            _note(f'head {losses} k={k} {what}', e)
            assert e <= TOL, f'{losses} k={k} image {b} {what}: {val} vs float64 {want} (relative {e:.3e})'
        g_cls.append(gc * up_cls[b] / norm_c)
        g_pts.append(gp * up_pts[b] / norm_p * head.pts_gamma * s)       # pred = anchor + reg * pts_gamma * stride
    want_cls = torch.stack(g_cls).reshape(B, H, W, k * C).permute(0, 3, 1, 2)
    want_pts = torch.stack(g_pts).reshape(B, H, W, 2 * k).permute(0, 3, 1, 2)
    for what, got_g, want_g in (('d/d cls_out', cls_out.grad, want_cls), ('d/d pts_out', pts_out.grad, want_pts)):
        e = scale_rel_err(got_g, want_g)
        _note(f'head {losses} k={k} {what}', e)
        assert e <= TOL, f'{losses} k={k} {what}: scale-relative {e:.3e}'
