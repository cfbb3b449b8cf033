"""GPU: the fused P2P loss kernels (focal, smooth-L1, MSE, sigmoid BCE with and without pos_weight, softmax CE) against the float64
reference of tests/p2p_loss_ref.py, at the element counts where the fixed 528 x 256 sum grid changes shape (one element, one block,
one trip of the grid-stride loop and one element either side of it) and at the head's real sizes; the MSE sum bit for bit against a
numpy restatement of the fixed-order sum; the one scratch slot per stream that every fixed-order sum shares; and P2PHead.loss at the
bench shape against the float64 reference built from the head's own targets.

Checks of every case: sums within 1e-5 relative of float64, gradients within 1e-5 scale-relative, zero-weight rows with a gradient of
exactly 0, two calls with identical bits, and NaN exactly where float64 torch has it.  The largest errors seen are printed."""
import numpy as np
import pytest
import torch

from tests import p2p_loss_ref as ref
from tests.helpers import scale_rel_err
from tests.test_gpu_p2p_defaults import TRAIN_CFG

pytestmark = pytest.mark.gpu

TOL = 1e-5
GRID = ref.SUM_GRID                                   # 135 168 elements per trip
ELEM_SIZES = [1, 255, GRID - 1, GRID, GRID + 1]       # elementwise losses, in elements of the grid-stride loop
BENCH_M, DEFAULT_M = 100 * 168, 100 * 168 * 4         # proposals of one 100x168 image at 1 and at 4 anchors per cell
ROW_SIZES = [1, ref.ROWS_PER_TRIP - 1, ref.ROWS_PER_TRIP, ref.ROWS_PER_TRIP + 1, DEFAULT_M]
FOCAL_PARAMS = [(2.0, 0.25), (1.5, 0.25), (1.0, 0.5), (3.0, 0.75), (0.0, 0.25)]
# logits around the saturation points of sleef_expf_u10 (|x| > 100 / 104) and of sigmoidf_acc (p == 1 from x ~ 16.7)
PLANTED = [0.0, 1e-30, -1e-30, 16.5, -16.5, 16.7, -16.7, 17.0, -17.0, 88.0, -88.0, 100.5, -100.5, 104.5, -104.5]

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


def check_loss(call, x, ref_sum, ref_grad, what, key, zero_rows=None):
    """call(scale=None, want_grad=False) runs one kernel; x is its input on the GPU.  Sum, gradient (at scale 0.75), determinism,
    zero-weight rows and NaN placement against the float64 reference."""
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
    if zero_rows is not None and bool(zero_rows.any()):
        gz = g1[zero_rows.cpu()]
        gz = gz[~torch.isnan(gz)]
        assert bool((gz == 0).all()), f'{what}: zero-weight rows have a non-zero gradient'


def _weights(kind, n, g):
    if kind == 'none':
        return None
    w = torch.rand(n, generator=g) * 0.9 + 0.05                                      # fractional
    r = torch.rand(n, generator=g)
    w = torch.where(r < 0.2, torch.zeros_like(w), torch.where(r > 0.8, 1.0 + 3.0 * torch.rand(n, generator=g), w))  # 0 and > 1
    return w


def focal_case(M, C, seed, weights, plant=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C, generator=g) * 4
    lab = torch.randint(0, C, (M,), generator=g)
    r = torch.randint(0, 8, (M,), generator=g)
    lab = torch.where(r == 0, torch.full_like(lab, C), lab)                           # background
    lab = torch.where(r == 1, torch.full_like(lab, -1), lab)
    lab = torch.where(r == 2, torch.full_like(lab, C + 3), lab)
    lab = torch.where(r == 3, torch.zeros_like(lab), lab)                             # first and last columns
    lab = torch.where(r == 4, torch.full_like(lab, C - 1), lab)
    if M == 1:                                   # one element carries the whole sum: a background row keeps it well conditioned
        lab[:] = C
    if plant and M >= 2 * len(PLANTED):
        rows = torch.randperm(M, generator=g)[:2 * len(PLANTED)]
        for i, v in enumerate(PLANTED):
            m1, m0 = int(rows[2 * i]), int(rows[2 * i + 1])
            c1 = int(torch.randint(0, C, (1,), generator=g))
            lab[m1] = c1
            x[m1, c1] = v                                                              # t = 1
            c0 = (int(lab[m0]) + 1) % C if 0 <= int(lab[m0]) < C and C > 1 else 0
            if C == 1 and 0 <= int(lab[m0]) < C:
                lab[m0] = C
            x[m0, c0] = v                                                              # t = 0
    return x, lab, _weights(weights, M, g)


def _to(dev, *ts):
    return [None if t is None else t.to(dev) for t in ts]


def _focal_shapes(C):
    if C == 1:
        return [(n, 1) for n in ELEM_SIZES]
    return [(1, C), (255 // C + 1, C), ((GRID - 1) // C, C), (GRID // C + 1, C)]


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('gamma,alpha', FOCAL_PARAMS)
@pytest.mark.parametrize('C', [1, 7, 80, 129])
@pytest.mark.parametrize('weights', ['none', 'mixed'])
def test_focal_matches_float64(ops, gamma, alpha, C, weights):
    dev = torch.device('cuda:0')
    shapes = _focal_shapes(C) + ([(BENCH_M, 80)] if C == 80 else [])
    for i, (M, Cs) in enumerate(shapes):
        x, lab, w = focal_case(M, Cs, 1000 * C + 10 * i + int(gamma * 2), weights)
        s, gr = ref.focal(x, lab, w, gamma, alpha)
        xd, ld, wd = _to(dev, x, lab, w)
        call = lambda scale=None, want_grad=False: ops.sigmoid_focal(xd, ld, wd, gamma, alpha, scale=scale, want_grad=want_grad)  # noqa: E731
        zero = None if w is None else (w == 0)[:, None].expand(M, Cs)
        check_loss(call, xd, s, gr, f'focal gamma={gamma} alpha={alpha} M={M} C={Cs} w={weights}', f'focal g={gamma}', zero)


@pytest.mark.parametrize('gamma,alpha', [(2.0, 0.25), (0.0, 0.25)])
def test_focal_at_the_reference_default_shape(ops, gamma, alpha):
    dev = torch.device('cuda:0')
    x, lab, w = focal_case(DEFAULT_M, 80, 77 + int(gamma), 'mixed')
    s, gr = ref.focal(x, lab, w, gamma, alpha)
    xd, ld, wd = _to(dev, x, lab, w)
    call = lambda scale=None, want_grad=False: ops.sigmoid_focal(xd, ld, wd, gamma, alpha, scale=scale, want_grad=want_grad)  # noqa: E731
    check_loss(call, xd, s, gr, f'focal gamma={gamma} M={DEFAULT_M} C=80', f'focal g={gamma}', (w == 0)[:, None].expand(DEFAULT_M, 80))


def test_focal_gamma_zero_on_saturated_elements_has_the_gradient_of_torch(ops):
    """pt == 0 exactly (a positive with p == 1 in fp32, a negative with p == 0): d pt^0 / d pt is 0, as in torch, not 0 * inf."""
    dev = torch.device('cuda:0')
    x = torch.tensor([[17.0, -104.5, 0.5], [100.5, -17.0, -0.5]])
    lab = torch.tensor([0, 0])
    s, gr = ref.focal(x, lab, None, 0.0, 0.25)
    gd = ops.sigmoid_focal(x.to(dev), lab.to(dev), None, 0.0, 0.25, scale=torch.ones(1, device=dev), want_grad=True).cpu()
    assert torch.isfinite(gd).all(), f'gamma 0 gradient {gd.tolist()}'
    assert scale_rel_err(gd, gr) <= TOL


# ---------------------------------------------------------------------------------------------------------------------------------
def points_case(M, seed, weights, beta, inv_norm):
    """(M, 2) predictions and targets; the first rows carry planted diffs: exactly 0, +-beta and one fp32 ulp either side of beta.
    They are built on target 0 so that (pred - target) * inv_norm is exact whenever inv_norm is a power of two."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(M, 2, generator=g) * 30
    t = torch.randn(M, 2, generator=g) * 30
    b32 = np.float32(beta)
    edges = np.array([0.0, b32, -b32, np.nextafter(b32, np.float32(0)), np.nextafter(b32, np.float32(np.inf)),
                      -np.nextafter(b32, np.float32(0)), -np.nextafter(b32, np.float32(np.inf))], np.float32)
    k = min(len(edges), 2 * M)
    if M > 1:
        inv = np.float32(inv_norm)
        flat_p, flat_t = p.view(-1), t.view(-1)
        flat_t[:k] = 0.0
        flat_p[:k] = torch.from_numpy(edges[:k] / inv)
        if inv_norm in (0.125, 0.5, 1.0):
            got = (flat_p[:k].numpy() - flat_t[:k].numpy()) * inv
            assert np.array_equal(got, edges[:k]), 'planted diffs are exact'
    if weights == 'none':
        w = None
    else:
        w = (torch.rand(M, generator=g) > 0.4).float()[:, None].expand(M, 2).contiguous()     # the head's {0, 1} point weights
    return p, t, w


POINT_SIZES = [1, 128, (GRID - 1) // 2, GRID // 2, GRID // 2 + 1, BENCH_M, DEFAULT_M]   # n = 2M: 2 .. one trip + 2, and the head's


@pytest.mark.parametrize('beta', [1.0 / 9.0, 1.0, 1e-3])
@pytest.mark.parametrize('inv_norm', [0.125, 1.0 / 3.0])
@pytest.mark.parametrize('weights', ['none', 'points'])
def test_smooth_l1_matches_float64(ops, beta, inv_norm, weights):
    dev = torch.device('cuda:0')
    for i, M in enumerate(POINT_SIZES):
        p, t, w = points_case(M, 31 * i + int(beta * 100), weights, beta, inv_norm)
        s, gr = ref.smooth_l1(p, t, w, inv_norm, beta)
        pd, td, wd = _to(dev, p, t, w)
        call = lambda scale=None, want_grad=False: ops.smooth_l1(pd, td, wd, inv_norm, beta, scale=scale, want_grad=want_grad)  # noqa: E731
        check_loss(call, pd, s, gr, f'smooth-L1 beta={beta} inv_norm={inv_norm} M={M} w={weights}', 'smooth-L1',
                   None if w is None else w == 0)


@pytest.mark.parametrize('inv_norm', [0.125, 1.0 / 3.0])
@pytest.mark.parametrize('weights', ['none', 'points', 'mixed'])
def test_mse_matches_float64_and_the_fixed_order_sum_bit_for_bit(ops, inv_norm, weights):
    dev = torch.device('cuda:0')
    for i, M in enumerate(POINT_SIZES):
        p, t, w = points_case(M, 7 * i + 3, 'none' if weights == 'mixed' else weights, 1.0 / 9.0, inv_norm)
        if weights == 'mixed':
            w = _weights('mixed', 2 * M, torch.Generator().manual_seed(i)).view(M, 2).contiguous()
        s, gr = ref.mse(p, t, w, inv_norm)
        pd, td, wd = _to(dev, p, t, w)
        call = lambda scale=None, want_grad=False: ops.mse(pd, td, wd, inv_norm, scale=scale, want_grad=want_grad)  # noqa: E731
        check_loss(call, pd, s, gr, f'MSE inv_norm={inv_norm} M={M} w={weights}', 'MSE', None if w is None else w == 0)
        terms = ref.mse_terms_f32(p.numpy(), t.numpy(), None if w is None else w.numpy(), ref.f32(inv_norm))
        want = ref.fixed_order_sum(terms)
        got = call().cpu().numpy()[0]
        assert got.tobytes() == want.tobytes(), f'MSE M={M}: sum {got!r} != fixed-order fp32 sum {want!r}'


# ---------------------------------------------------------------------------------------------------------------------------------
def bce_case(M, C, seed, weights):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C, generator=g) * 4
    lab = torch.randint(-1, C + 2, (M,), generator=g)              # -1, C and C + 1 are all-zero rows
    if M * C >= len(PLANTED):
        x.view(-1)[:len(PLANTED)] = torch.tensor(PLANTED)
    return x, lab, _weights(weights, M, g), torch.rand(C, generator=g) * 3 + 0.1


@pytest.mark.parametrize('C', [1, 7, 80, 129, 320])
@pytest.mark.parametrize('with_pw', [False, True])
@pytest.mark.parametrize('weights', ['none', 'mixed'])
def test_sigmoid_bce_matches_float64(ops, C, with_pw, weights):
    dev = torch.device('cuda:0')
    shapes = [(GRID - 1) // C, GRID // C + 1] + ([BENCH_M, DEFAULT_M] if C == 80 else [])
    for i, M in enumerate(shapes):
        x, lab, w, pw = bce_case(M, C, 500 + 10 * C + i, weights)
        pw = pw if with_pw else None
        s, gr = ref.sigmoid_bce(x, lab, w, pw)
        xd, ld, wd, pwd = _to(dev, x, lab, w, pw)
        call = lambda scale=None, want_grad=False: ops.sigmoid_bce(xd, ld, wd, pos_weight=pwd, scale=scale, want_grad=want_grad)  # noqa: E731
        check_loss(call, xd, s, gr, f'BCE pos_weight={with_pw} M={M} C={C} w={weights}', f'BCE pos_weight={with_pw}',
                   None if w is None else (w == 0)[:, None].expand(M, C))


# ---------------------------------------------------------------------------------------------------------------------------------
def softmax_case(M, C1, seed, weights):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C1, generator=g) * 4
    lab = torch.randint(0, C1, (M,), generator=g)
    lab[::3] = C1 - 1                                                          # the background column
    if M > 8:
        x[1] = 0.5                                                             # all logits equal
        x[2, 3 % C1] += 80.0                                                   # one logit far above the rest, the label's ...
        lab[2] = 3 % C1
        x[3, 0] += 80.0                                                        # ... and another column's
        lab[3] = C1 - 1
        x[4, ::2] = -1e4                                                       # hugely negative entries
        x[5] = -1e4
        x[6, C1 - 1] = -1e4
        lab[6] = C1 - 1
    else:                                          # one row carries the whole sum: label its smallest logit (a well-conditioned loss)
        lab = x.argmin(dim=1)
    return x, lab, _weights(weights, M, g)


@pytest.mark.parametrize('C1', [2, 31, 32, 33, 64, 65, 81, 321])
@pytest.mark.parametrize('with_cw', [False, True])
def test_softmax_ce_matches_float64(ops, C1, with_cw):
    dev = torch.device('cuda:0')
    for i, M in enumerate(ROW_SIZES):
        x, lab, w = softmax_case(M, C1, 3000 + 10 * C1 + i, 'mixed' if i % 2 else 'none')
        cw = (torch.rand(C1, generator=torch.Generator().manual_seed(C1)) * 2 + 0.1) if with_cw else None
        s, gr = ref.softmax_ce(x, lab, w, cw)
        xd, ld, wd, cwd = _to(dev, x, lab, w, cw)
        call = lambda scale=None, want_grad=False: ops.softmax_ce(xd, ld, wd, cwd, scale=scale, want_grad=want_grad)  # noqa: E731
        check_loss(call, xd, s, gr, f'softmax CE class_weight={with_cw} M={M} C1={C1}', 'softmax CE',
                   None if w is None else (w == 0)[:, None].expand(M, C1))


# ---------------------------------------------------------------------------------------------------------------------------------
NAN_LOSSES = ['focal_g2', 'focal_g0', 'focal_g1.5', 'smooth_l1', 'mse', 'bce', 'bce_pw', 'softmax_ce']


@pytest.mark.parametrize('loss', NAN_LOSSES)
def test_a_nan_input_makes_the_sum_nan_and_the_gradient_nan_where_torch_has_it(ops, loss):
    """the NaN element for the elementwise losses, the NaN's whole row for softmax CE; every other gradient element stays finite.
    One NaN sits in a zero-weight row, one in a weighted row past the first trip."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(NAN_LOSSES.index(loss))
    if loss in ('smooth_l1', 'mse'):
        M = GRID // 2 + 5
        p, t = torch.randn(M, 2, generator=g) * 30, torch.randn(M, 2, generator=g) * 30
        w = torch.ones(M, 2)
        w[3] = 0
        p[3, 1] = float('nan')
        p[GRID // 2 + 1, 0] = float('nan')
        if loss == 'mse':
            s, gr = ref.mse(p, t, w, 0.125)
            call = lambda scale=None, want_grad=False: ops.mse(*_to(dev, p, t, w), 0.125, scale=scale, want_grad=want_grad)  # noqa: E731
        else:
            s, gr = ref.smooth_l1(p, t, w, 0.125, 1.0 / 9.0)
            call = lambda scale=None, want_grad=False: ops.smooth_l1(*_to(dev, p, t, w), 0.125, 1.0 / 9.0, scale=scale,  # noqa: E731
                                                                     want_grad=want_grad)
        x = p
    else:
        C = 80 if loss != 'softmax_ce' else 81
        M = GRID // C + 3
        x = torch.randn(M, C, generator=g) * 4
        lab = torch.randint(0, C, (M,), generator=g)
        w = torch.rand(M, generator=g) + 0.1
        w[3] = 0
        x[3, 5] = float('nan')
        x[M - 2, 7] = float('nan')
        if loss.startswith('focal'):
            gamma = {'focal_g2': 2.0, 'focal_g0': 0.0, 'focal_g1.5': 1.5}[loss]
            s, gr = ref.focal(x, lab, w, gamma, 0.25)
            call = lambda scale=None, want_grad=False: ops.sigmoid_focal(*_to(dev, x, lab, w), gamma, 0.25, scale=scale,  # noqa: E731
                                                                         want_grad=want_grad)
        elif loss.startswith('bce'):
            pw = torch.rand(C, generator=g) + 0.5 if loss == 'bce_pw' else None
            s, gr = ref.sigmoid_bce(x, lab, w, pw)
            call = lambda scale=None, want_grad=False: ops.sigmoid_bce(*_to(dev, x, lab, w), pos_weight=_to(dev, pw)[0],  # noqa: E731
                                                                       scale=scale, want_grad=want_grad)
        else:
            s, gr = ref.softmax_ce(x, lab, w)
            call = lambda scale=None, want_grad=False: ops.softmax_ce(*_to(dev, x, lab, w), scale=scale, want_grad=want_grad)  # noqa: E731
    assert torch.isnan(s)
    nan_rows = torch.isnan(gr).any(dim=1)
    assert int(nan_rows.sum()) == 2, 'the float64 gradient is NaN in the two rows of the NaNs'
    if loss == 'softmax_ce':
        assert torch.isnan(gr[nan_rows]).all(), 'float64 softmax CE: the whole row'
    else:
        assert int(torch.isnan(gr).sum()) == 2, 'float64 elementwise: the element only'
    check_loss(call, x.to(dev), s, gr, f'NaN {loss}', f'NaN {loss}')


# ---------------------------------------------------------------------------------------------------------------------------------
def _sum_jobs(ops, dev):
    """the fixed-order sums that share a stream's scratch slot, each with its own n, n = 1 among them"""
    g = torch.Generator().manual_seed(99)
    jobs = []
    x1 = torch.randn(1, 1, generator=g).to(dev)
    l1 = torch.ones(1, dtype=torch.int64, device=dev)
    jobs.append(('focal n=1', lambda: ops.sigmoid_focal(x1, l1, None, 2.0, 0.25)))
    xf, lf, wf = _to(dev, *focal_case(GRID // 80 + 1, 80, 5, 'mixed'))
    jobs.append(('focal', lambda: ops.sigmoid_focal(xf, lf, wf, 2.0, 0.25)))
    xg, lg = torch.rand(3001, 80, generator=g).to(dev) * 6 - 3, torch.randint(0, 80, (3001,), generator=g).int().to(dev)
    wg = torch.rand(3001, generator=g).to(dev)
    jobs.append(('gfocal', lambda: ops.gfocal_fwd(xg, 3001, 80, 80, lg, wg, 1e-6)))
    xs, ls, ws = _to(dev, *softmax_case(ref.ROWS_PER_TRIP + 1, 81, 6, 'mixed'))
    jobs.append(('softmax CE', lambda: ops.softmax_ce(xs, ls, ws)))
    xs1, ls1 = torch.randn(1, 2, generator=g).to(dev), torch.zeros(1, dtype=torch.int64, device=dev)
    jobs.append(('softmax CE M=1', lambda: ops.softmax_ce(xs1, ls1, None)))
    pm, tm, wm = _to(dev, *points_case(GRID // 2 + 1, 7, 'points', 1.0 / 9.0, 0.125))
    jobs.append(('MSE', lambda: ops.mse(pm, tm, wm, 0.125)))
    jobs.append(('smooth-L1', lambda: ops.smooth_l1(pm, tm, wm, 0.125, 1.0 / 9.0)))
    xb, lb, wb, pwb = _to(dev, *bce_case(255, 7, 8, 'mixed'))
    jobs.append(('BCE', lambda: ops.sigmoid_bce(xb, lb, wb)))
    jobs.append(('BCE pos_weight', lambda: ops.sigmoid_bce(xb, lb, wb, pos_weight=pwb)))
    return jobs


def _solo(jobs):
    out = []
    for _, fn in jobs:
        r = fn()
        torch.cuda.synchronize()
        out.append(r.clone())
    return out


def test_back_to_back_sums_on_one_stream_leave_each_other_alone(ops):
    dev = torch.device('cuda:0')
    jobs = _sum_jobs(ops, dev)
    solo = _solo(jobs)
    order = [0, 2, 1, 3, 5, 4, 6, 7, 8, 2, 0, 4, 1, 3, 8, 7, 6, 5, 0, 0, 2, 2]        # repeats and n = 1 next to the large sums
    got = [jobs[i][1]() for i in order]                                              # no synchronisation in between
    torch.cuda.synchronize()
    for i, r in zip(order, got):
        assert torch.equal(r, solo[i]), f'{jobs[i][0]}: {float(r)} interleaved vs {float(solo[i])} solo'


def test_concurrent_sums_on_two_streams_use_their_own_slots(ops):
    dev = torch.device('cuda:0')
    jobs = _sum_jobs(ops, dev)
    solo = _solo(jobs)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = [1, 6, 1, 0, 7, 1, 6, 2]                      # about 8 launches each, different losses on the two streams
    b = [3, 5, 3, 4, 8, 3, 5, 3]
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
    # and the default stream still sums correctly afterwards
    for i, (_, fn) in enumerate(jobs):
        assert torch.equal(fn(), solo[i])


def test_sums_after_reset_stream_state(ops):
    from pointtinybenchmark_b200 import _lib
    from pointtinybenchmark_b200.ops import _stream
    dev = torch.device('cuda:0')
    jobs = _sum_jobs(ops, dev)
    solo = _solo(jobs)
    assert _lib.load().ptb_reset_stream_state(_stream()) == 0
    for i, (_, fn) in enumerate(jobs):
        assert torch.equal(fn(), solo[i]), jobs[i][0]
        assert _lib.load().ptb_reset_stream_state(_stream()) == 0
    torch.cuda.synchronize()


def test_each_loss_call_is_one_launch(ops):
    dev = torch.device('cuda:0')
    x, lab, w = _to(dev, *focal_case(300, 80, 1, 'mixed'))
    pts, tgt, pw = _to(dev, *points_case(300, 1, 'points', 1.0 / 9.0, 0.125))
    sc = torch.ones(1, device=dev)
    calls = [lambda **k: ops.sigmoid_focal(x, lab, w, 2.0, 0.25, **k), lambda **k: ops.sigmoid_bce(x, lab, w, **k),
             lambda **k: ops.sigmoid_bce(x, lab, w, pos_weight=torch.ones(80, device=dev), **k),
             lambda **k: ops.softmax_ce(x, lab.clamp(0, 79), w, **k), lambda **k: ops.smooth_l1(pts, tgt, pw, 0.125, 1.0 / 9.0, **k),
             lambda **k: ops.mse(pts, tgt, pw, 0.125, **k)]
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
    dev = torch.device('cuda:0')
    x, lab, w = _to(dev, *focal_case(GRID // 80 + 1, 80, 2, 'mixed'))
    xs, ls, ws = _to(dev, *softmax_case(ref.ROWS_PER_TRIP + 1, 81, 3, 'mixed'))
    pts, tgt, pw = _to(dev, *points_case(GRID // 2 + 1, 2, 'points', 1.0 / 9.0, 0.125))
    pos_w = torch.rand(80, device=dev) + 0.5
    entries = [
        ('focal g2', x, lambda *o: lib.ptb_sigmoid_focal_fwd_bwd(_ptr(x), _ptr(lab), _ptr(w), x.shape[0], 80, 2.0, 0.25, *o)),
        ('focal g1.5', x, lambda *o: lib.ptb_sigmoid_focal_fwd_bwd(_ptr(x), _ptr(lab), _ptr(w), x.shape[0], 80, 1.5, 0.25, *o)),
        ('smooth-L1', pts, lambda *o: lib.ptb_smooth_l1_fwd_bwd(_ptr(pts), _ptr(tgt), _ptr(pw), pts.shape[0], 0.125, 1.0 / 9.0, *o)),
        ('MSE', pts, lambda *o: lib.ptb_mse_fwd_bwd(_ptr(pts), _ptr(tgt), _ptr(pw), pts.shape[0], 0.125, *o)),
        ('BCE', x, lambda *o: lib.ptb_sigmoid_bce_fwd_bwd(_ptr(x), _ptr(lab), _ptr(w), x.shape[0], 80, *o)),
        ('BCE pos_weight', x, lambda *o: lib.ptb_sigmoid_bce_cw_fwd_bwd(_ptr(x), _ptr(lab), _ptr(w), _ptr(pos_w), x.shape[0], 80, *o)),
        ('softmax CE', xs, lambda *o: lib.ptb_softmax_ce_fwd_bwd(_ptr(xs), _ptr(ls), _ptr(ws), None, xs.shape[0], 81, *o)),
    ]
    one = torch.ones(1, device=dev)
    sc = torch.tensor([-2.5], device=dev)
    for name, inp, fn in entries:
        def run(want_sum, want_grad, scale):
            s = torch.zeros(1, device=dev) if want_sum else None
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


# ---------------------------------------------------------------------------------------------------------------------------------
def _head(k):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401  (registers the head)
    from pointtinybenchmark_b200.registry import build_head
    hc = dict(type='P2PHead', num_classes=80, in_channels=256, feat_channels=256, stacked_convs=4, strides=[8],
              norm_cfg=dict(type='GN', num_groups=32, requires_grad=True), train_cfg=TRAIN_CFG,
              loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
              loss_reg=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=0.5))
    if k == 1:                                                # bench.py's head: one anchor, pts_gamma 1, reg_norm 1
        hc.update(point_anchor=[(0., 0.)], pts_gamma=1, reg_norm=1)
    return build_head(hc).cuda().train()


@pytest.mark.parametrize('k,B', [(1, 3), (4, 2)])
def test_head_loss_at_the_bench_shape_matches_float64_on_its_own_targets(ops, k, B):
    """P2PHead.loss + backward (focal + smooth-L1) on random 100x168 maps with 20 GTs per image, against the float64 losses of the
    head's own targets and normalisers; an upstream gradient other than 1 checks that the scale reaches the gradient launches."""
    dev = torch.device('cuda:0')
    head = _head(k)
    H, W, C, s = 100, 168, 80, 8.0
    g = torch.Generator().manual_seed(40 + k)
    cls_out = (torch.randn(B, k * C, H, W, generator=g) * 2 - 3).to(dev).requires_grad_(True)
    pts_out = (torch.randn(B, 2 * k, H, W, generator=g) * (0.5 if k == 1 else 0.05)).to(dev).requires_grad_(True)
    gtb, gtl = [], []
    for _ in range(B):
        cxy = torch.rand(20, 2, generator=g) * torch.tensor([1300., 780.]) + 10
        gtb.append(torch.cat([cxy - 8, cxy + 8], 1).to(dev))
        gtl.append(torch.randint(0, C, (20,), generator=g).to(dev))
    metas = [dict(pad_shape=(800, 1344, 3), img_shape=(800, 1333, 3), scale_factor=[1.0] * 4)] * B
    got = head.loss([cls_out], [pts_out], gtb, gtl, metas)
    got_vals = {key: [float(v.detach()) for v in vals] for key, vals in got.items()}
    up_cls = [3.7, 0.6, -1.2][:B]
    up_pts = [-0.25, 1.0, 2.0][:B]
    total = sum(a * l for a, l in zip(up_cls, got['loss_cls'])) + sum(a * l for a, l in zip(up_pts, got['loss_pts']))
    total.backward()
    tg = head._last_targets
    with torch.no_grad():
        _, pred, _, cls = head.get_pred_points(cls_out, pts_out, metas)
    npos = float(sum(int((p[:, 0] > 0).sum()) for p in tg['pts_weights']))
    assert npos > 0
    inv_norm = 1.0 / (s * head.reg_norm)
    g_cls, g_pts = [], []
    for b in range(B):
        lw, labels = tg['label_weights'][b], tg['labels'][b]
        sc, gc = ref.focal(cls[b], labels, lw, 2.0, 0.25)
        sp, gp = ref.smooth_l1(pred[b], tg['gt_pts'][b], tg['pts_weights'][b], inv_norm, 1.0 / 9.0)
        for what, want in (('loss_cls', float(sc) / npos), ('loss_pts', 0.5 * float(sp) / npos)):
            val = got_vals[what][b]
            e = abs(val - want) / abs(want)
            _note(f'head k={k} {what}', e)
            assert e <= TOL, f'k={k} image {b} {what}: {val} vs float64 {want} (relative {e:.3e})'
        g_cls.append(gc * up_cls[b] / npos)
        g_pts.append(gp * up_pts[b] * 0.5 / npos * head.pts_gamma * s)       # pred = anchor + reg * pts_gamma * stride
    want_cls = torch.stack(g_cls).reshape(B, H, W, k * C).permute(0, 3, 1, 2)
    want_pts = torch.stack(g_pts).reshape(B, H, W, 2 * k).permute(0, 3, 1, 2)
    for what, got_g, want_g in (('d/d cls_out', cls_out.grad, want_cls), ('d/d pts_out', pts_out.grad, want_pts)):
        e = scale_rel_err(got_g, want_g)
        _note(f'head k={k} {what}', e)
        assert e <= TOL, f'k={k} {what}: scale-relative {e:.3e}'
