"""CPU: the float64 reference of the fused P2P losses (tests/p2p_loss_ref.py) against the oracle's fp32 functions, its fixed-order
sum against an exactly rounded sum, and the argument checks of the elementwise loss entry points, which run before any CUDA call."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p as op2p, p2p_loss_types as olt
from tests import p2p_loss_ref as ref
from tests.helpers import assert_close


def _fp32_oracle(fn, x, *args):
    """sum and gradient of fn(x, *args).sum() in fp32 autograd"""
    xr = x.clone().requires_grad_(True)
    s = fn(xr, *args).sum()
    s.backward()
    return s.detach(), xr.grad


@pytest.mark.parametrize('gamma,alpha', [(2.0, 0.25), (1.5, 0.25), (0.0, 0.25), (3.0, 0.75)])
def test_focal_reference_matches_the_fp32_oracle(gamma, alpha):
    g = torch.Generator().manual_seed(int(gamma * 10))
    M, C = 700, 7
    x = torch.randn(M, C, generator=g) * 3
    lab = torch.randint(-1, C + 4, (M,), generator=g)
    w = torch.rand(M, generator=g) * 2
    s, gr = ref.focal(x, lab, w, gamma, alpha)
    lab_o = torch.where((lab < 0) | (lab >= C), torch.full_like(lab, C), lab)
    so, go = _fp32_oracle(lambda xr: op2p.sigmoid_focal_loss_elem(xr, lab_o, gamma, alpha) * w[:, None], x)
    assert s.dtype == gr.dtype == torch.float64
    assert_close(so, s, 2e-6, 'focal sum')
    assert_close(go, gr, 2e-6, 'focal grad')
    # a label outside [0, C) is an all-zero row: the row equals a background row
    bg = (lab < 0) | (lab >= C)
    assert bg.any() and (~bg).any()


@pytest.mark.parametrize('loss', ['smooth_l1', 'mse'])
def test_point_loss_references_match_the_fp32_oracle(loss):
    g = torch.Generator().manual_seed(5)
    M, inv_norm, beta = 900, 0.125, 1.0 / 9.0
    p, t = torch.randn(M, 2, generator=g) * 3, torch.randn(M, 2, generator=g) * 3
    w = (torch.rand(M, 2, generator=g) > 0.5).float()
    if loss == 'smooth_l1':
        s, gr = ref.smooth_l1(p, t, w, inv_norm, beta)
        so, go = _fp32_oracle(lambda pr: op2p.smooth_l1_elem((pr - t) * inv_norm, torch.zeros_like(t), ref.f32(beta)) * w, p)
    else:
        s, gr = ref.mse(p, t, w, inv_norm)
        so, go = _fp32_oracle(lambda pr: F.mse_loss(pr * inv_norm, t * inv_norm, reduction='none') * w, p)
    assert_close(so, s, 2e-6, f'{loss} sum')
    assert_close(go, gr, 2e-6, f'{loss} grad')
    # the fp32 MSE terms in the kernel's order sum to the float64 loss
    terms = ref.mse_terms_f32(p.numpy(), t.numpy(), w.numpy(), inv_norm)
    assert abs(float(ref.fixed_order_sum(terms)) - float(ref.mse(p, t, w, inv_norm)[0])) <= 1e-5 * float(s)


@pytest.mark.parametrize('with_w', [False, True])
def test_bce_and_softmax_references_match_the_fp32_oracle(with_w):
    g = torch.Generator().manual_seed(9 + with_w)
    M, C = 600, 13
    x = torch.randn(M, C, generator=g) * 3
    lab = torch.randint(-1, C + 1, (M,), generator=g)
    w = torch.rand(M, generator=g) * 2 if with_w else None
    pw = torch.rand(C, generator=g) * 3 + 0.1
    t = torch.zeros(M, C)
    ok = (lab >= 0) & (lab < C)
    t[ok.nonzero().squeeze(1), lab[ok]] = 1
    wr = torch.ones(M) if w is None else w
    for pos_weight in (None, pw):
        s, gr = ref.sigmoid_bce(x, lab, w, pos_weight)
        so, go = _fp32_oracle(lambda xr: F.binary_cross_entropy_with_logits(xr, t, pos_weight=pos_weight, reduction='none')
                              * wr[:, None], x)
        assert_close(so, s, 2e-6, 'bce sum')
        assert_close(go, gr, 2e-6, 'bce grad')
    labs = torch.randint(0, C, (M,), generator=g)
    for cw in (None, pw):
        s, gr = ref.softmax_ce(x, labs, w, cw)
        so, go = _fp32_oracle(lambda xr: F.cross_entropy(xr, labs, weight=cw, reduction='none') * wr, x)
        assert_close(so, s, 2e-6, 'softmax ce sum')
        assert_close(go, gr, 2e-6, 'softmax ce grad')


def test_focal_reference_at_gamma_zero_has_a_finite_gradient_on_saturated_elements():
    """torch's pow_backward is 0 for exponent 0, so a correctly classified element with pt == 0 has gradient 0, not NaN."""
    x = torch.tensor([[100.5, -100.5], [-17.0, 17.0]])
    lab = torch.tensor([0, 1])
    s, gr = ref.focal(x, lab, None, 0.0, 0.25)
    assert torch.isfinite(gr).all() and torch.isfinite(s)


@pytest.mark.parametrize('n', [1, 31, 255, 256, ref.SUM_GRID - 1, ref.SUM_GRID, ref.SUM_GRID + 1, 1_344_000])
def test_fixed_order_sum_is_an_fp32_sum(n):
    rng = np.random.default_rng(n)
    terms = (rng.random(n) * rng.choice([1e-3, 1.0, 50.0], n)).astype(np.float32)
    got = float(ref.fixed_order_sum(terms))
    exact = math.fsum(terms.astype(np.float64))
    assert abs(got - exact) <= 1e-6 * exact, (got, exact)
    # small integers add exactly in any order
    ints = rng.integers(0, 8, n).astype(np.float32)
    assert float(ref.fixed_order_sum(ints)) == float(ints.astype(np.float64).sum())


def test_fixed_order_sum_follows_the_grid_order():
    """the order, not only the value: a term of 1 is absorbed by 2^24 when it is added after it on the same thread, and kept when
    the two sit on different threads of one warp and meet in the butterfly as 2^24 + 2 (an exact fp32 value)."""
    big = np.float32(2 ** 24)
    t = np.zeros(ref.SUM_GRID + 1, np.float32)
    t[0], t[ref.SUM_GRID] = big, 1.0                 # same thread, 1 added after 2^24: lost
    assert ref.fixed_order_sum(t) == big
    t = np.zeros(ref.SUM_GRID + 2, np.float32)
    t[0], t[1], t[ref.SUM_GRID + 1] = big, 1.0, 1.0  # lanes 1 (two trips) and 0: 2 meets 2^24 in the butterfly
    assert ref.fixed_order_sum(t) == big + 2


def test_argument_validation_of_the_elementwise_loss_entry_points_without_a_gpu():
    """argument checks run before any CUDA call: a bad call returns non-zero and sets ptb_last_error(); M = 0 returns 0 at once and
    leaves the sum as it was."""
    from pointtinybenchmark_b200 import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(16)      # never dereferenced: the checks fire first
    # ptb_sigmoid_focal_fwd_bwd(logits, labels, weight, M, C, gamma, alpha, loss_sum, scale, grad, stream)
    focal = lambda x=d, lab=d, M=10, C=80, out=d, grad=None: lib.ptb_sigmoid_focal_fwd_bwd(  # noqa: E731
        x, lab, None, M, C, 2.0, 0.25, out, None, grad, None)
    assert focal(M=-1) == 2 and b'M >= 0' in lib.ptb_last_error()
    assert focal(C=0) == 2 and b'num_classes' in lib.ptb_last_error()
    assert focal(x=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert focal(lab=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert focal(out=None) == 2 and b'NULL' in lib.ptb_last_error()
    # ptb_smooth_l1_fwd_bwd(pred, target, weight, M, inv_norm, beta, loss_sum, scale, grad, stream)
    sl1 = lambda p=d, t=d, M=10, beta=1.0 / 9, out=d: lib.ptb_smooth_l1_fwd_bwd(p, t, None, M, 0.125, beta, out, None, None, None)  # noqa: E731
    assert sl1(M=-1) == 2 and b'M >= 0' in lib.ptb_last_error()
    for beta in (0.0, -1.0, float('nan')):
        assert sl1(beta=beta) == 2 and b'beta' in lib.ptb_last_error()
    assert sl1(M=0, beta=0.0) == 2, 'beta is checked even when there is nothing to sum'
    assert sl1(p=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert sl1(t=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert sl1(out=None) == 2 and b'NULL' in lib.ptb_last_error()
    # ptb_mse_fwd_bwd(pred, target, weight, M, inv_norm, loss_sum, scale, grad, stream)
    mse = lambda p=d, t=d, M=10, out=d: lib.ptb_mse_fwd_bwd(p, t, None, M, 0.125, out, None, None, None)  # noqa: E731
    assert mse(M=-1) == 2 and b'M >= 0' in lib.ptb_last_error()
    assert mse(p=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert mse(t=None) == 2 and b'NULL' in lib.ptb_last_error()
    assert mse(out=None) == 2 and b'NULL' in lib.ptb_last_error()
    # M = 0: nothing is launched (there is no device here, a launch would fail) and the host-side sum stays 0
    s = ctypes.c_float(0.0)
    ps = ctypes.c_void_p(ctypes.addressof(s))
    assert focal(M=0, x=None, lab=None, out=ps) == 0
    assert sl1(M=0, p=None, t=None, out=ps) == 0
    assert mse(M=0, p=None, t=None, out=ps) == 0
    assert s.value == 0.0


# ---------------------------------------------------------------------------------------------------------------------------------
# GHM-C, GHM-R, L1Loss and BalancedL1Loss
BALANCED_PARAMS = [(0.5, 1.5, 1.0), (0.5, 1.5, 0.11), (0.25, 3.0, 1.0 / 9.0)]


def _row_inv(M, g):
    """one normalisation per row, five strides 8 .. 128 as the multi-level head has them"""
    return (1.0 / torch.tensor([8.0, 16.0, 32.0, 64.0, 128.0]))[torch.randint(0, 5, (M,), generator=g)]


@pytest.mark.parametrize('loss', ['l1'] + [f'balanced_l1 {p}' for p in BALANCED_PARAMS])
def test_l1_and_balanced_l1_references_match_the_fp32_oracle(loss):
    g = torch.Generator().manual_seed(11)
    M = 800
    p, t = torch.randn(M, 2, generator=g) * 30, torch.randn(M, 2, generator=g) * 30
    inv = _row_inv(M, g)
    w = torch.rand(M, 2, generator=g) * (torch.rand(M, 2, generator=g) > 0.3)
    d = lambda pr: (pr - t) * inv[:, None]                                   # noqa: E731
    if loss == 'l1':
        s, gr = ref.l1_rows(p, t, w, inv)
        so, go = _fp32_oracle(lambda pr: olt.l1_elem(d(pr), torch.zeros_like(t)) * w, p)
    else:
        a, gm, b = BALANCED_PARAMS[[f'balanced_l1 {q}' for q in BALANCED_PARAMS].index(loss)]
        s, gr = ref.balanced_l1_rows(p, t, w, inv, a, gm, b)
        so, go = _fp32_oracle(lambda pr: olt.balanced_l1_elem(d(pr), torch.zeros_like(t), a, gm, b) * w, p)
    assert s.dtype == gr.dtype == torch.float64
    assert_close(so, s, 2e-6, f'{loss} sum')
    assert_close(go, gr, 2e-6, f'{loss} grad')


def test_l1_reference_gradient_at_zero_and_nan_is_zero():
    """torch's abs backward is sgn(d): 0 at d == 0 and at a NaN d, which the kernel follows"""
    p = torch.tensor([[0.0, float('nan')], [3.0, -3.0]])
    s, gr = ref.l1_rows(p, torch.zeros(2, 2), None, torch.ones(2))
    assert torch.isnan(s)
    assert gr.tolist() == [[0.0, 0.0], [1.0, -1.0]]


def _ghmc_case(Q, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(Q, C, generator=g) * 4
    lab = torch.randint(0, C + 4, (Q,), generator=g)       # the oracle clamps a negative label onto class 0: none here
    lw = (torch.rand(Q, generator=g) > 0.25).float()
    return x, lab, lw


@pytest.mark.parametrize('bins,mmt', [(10, 0.0), (30, 0.75), (1, 0.0), (256, 0.7)])
def test_ghmc_restatement_and_reference_match_the_oracle(bins, mmt):
    """the restated g, bins, counts, weights and acc_sum against oracle/p2p_loss_types.ghmc, image by image, and the float64 sum /
    gradient on those bins against the oracle's fp32 autograd"""
    edges = olt.ghm_edges(bins, None)
    acc_r, acc_o = torch.rand(bins) * 50, None
    acc_o = acc_r.clone()
    xs, labs, lws = zip(*[_ghmc_case(300, 7, 20 + b) for b in range(3)])
    x, lab, lw = torch.stack(xs), torch.stack(labs), torch.stack(lws)
    gg = ref.ghmc_g_f32(x, lab)
    for b in range(3):
        t = F.one_hot(lab[b].clamp(0, 7), 8)[:, :7].float()                 # the oracle's one-hot
        go = (x[b].sigmoid() - t).abs()
        assert torch.equal(gg[b], ref.ghmc_g_f32(x[b], lab[b])), 'g does not depend on the batch around it'
        diff = (gg[b] - go).abs()                # one ulp of p below 1 is 2^-24: ATen's scalar tail may round p the other way
        assert float(diff.max()) <= 2.0 ** -24 and int((diff > 0).sum()) <= 64, 'g is the oracle fp32 g up to ATen\'s scalar tail'
    valid = (lw[:, :, None] > 0).expand(3, 300, 7).reshape(3, -1)
    counts, idx, bw, tot = ref.ghm_bin_step(gg.reshape(3, -1), valid, edges, mmt, acc_r if mmt > 0 else None)
    for b in range(3):
        xr = x[b].clone().requires_grad_(True)
        lo, cnt, nv, _ = olt.ghmc(xr, lab[b], lw[b], edges, mmt, acc_o if mmt > 0 else None)
        assert torch.equal(counts[b, :bins], cnt) and int(counts[b, bins]) == nv
        assert float(tot[b]) == float(max(nv, 1))
        lo.backward()
        s, gr = ref.ghmc(x[b], lab[b], lw[b], idx[b], bw[b])
        assert_close(lo.detach(), s / float(tot[b]), 2e-6, 'GHMC sum')
        assert_close(xr.grad, gr / float(tot[b]), 2e-6, 'GHMC grad')
    if mmt > 0:
        assert acc_r.numpy().tobytes() == acc_o.numpy().tobytes(), 'acc_sum bit for bit'


@pytest.mark.parametrize('bins,mmt', [(10, 0.0), (10, 0.7), (30, 0.0)])
def test_ghmr_restatement_and_reference_match_the_oracle(bins, mmt):
    g = torch.Generator().manual_seed(bins + int(mmt * 10))
    B, Q, mu = 2, 500, 0.02
    edges = olt.ghm_edges(bins, 1e3)
    p, t = torch.randn(B, Q, 2, generator=g) * 30, torch.randn(B, Q, 2, generator=g) * 30
    inv = _row_inv(Q, g)
    w = (torch.rand(B, Q, 1, generator=g) > 0.4).float().expand(B, Q, 2).contiguous()
    acc_r = torch.zeros(bins)
    acc_o = acc_r.clone()
    gg = ref.ghmr_g_f32(p, t, inv, mu)
    counts, idx, bw, tot = ref.ghm_bin_step(gg.reshape(B, -1), (w > 0).reshape(B, -1), edges, mmt, acc_r if mmt > 0 else None)
    for b in range(B):
        dn = torch.from_numpy((p[b].numpy() - t[b].numpy()) * inv.numpy()[:, None])     # the normalised points, fp32 as the kernel
        dr = dn.clone().requires_grad_(True)
        lo, cnt, nv, _ = olt.ghmr(dr, torch.zeros_like(dn), w[b], edges, mu, mmt, acc_o if mmt > 0 else None)
        # every operation correctly rounded, as __fsqrt_rn / __fdiv_rn are (a float64 sqrt or quotient of fp32 values, rounded once)
        d64 = dn.numpy().astype(np.float64)
        sq = np.float32(d64 * d64) + np.float32(np.float32(mu) ** 2)
        root = np.sqrt(sq.astype(np.float64)).astype(np.float32)
        assert np.array_equal(gg[b].numpy(), np.abs((d64 / root).astype(np.float32))), 'g is correctly rounded fp32'
        # torch's CPU fp32 sqrt is not always correctly rounded: the oracle's g is within two ulps of 1
        assert float((gg[b] - (dn / torch.sqrt(dn * dn + mu * mu)).abs()).abs().max()) <= 2.0 ** -22
        assert torch.equal(counts[b, :bins], cnt) and int(counts[b, bins]) == nv
        lo.backward()
        s, gr = ref.ghmr(p[b], t[b], w[b], inv, mu, idx[b], bw[b])
        assert_close(lo.detach(), s / float(tot[b]), 2e-6, 'GHMR sum')
        assert_close(dr.grad * inv[:, None], gr / float(tot[b]), 2e-6, 'GHMR grad')
    if mmt > 0:
        assert acc_r.numpy().tobytes() == acc_o.numpy().tobytes(), 'acc_sum bit for bit'


def test_sigmoid_f32_is_atens_vector_path_on_every_element():
    """each 64-element block on its own takes only ATen's vector loop; sigmoid_f32 of the whole gives the same bits"""
    x = torch.randn(100_003, generator=torch.Generator().manual_seed(2)) * 6
    s = ref.sigmoid_f32(x)
    for i in range(0, 100_000, 64 * 37):
        assert torch.equal(s[i:i + 64], torch.sigmoid(x[i:i + 64].clone())), i


def test_ghmc_g_of_a_label_outside_the_classes_is_a_zero_row():
    """-1, C and C + 3 are all-zero rows of the one-hot, as mmdet's _expand_onehot_labels makes them"""
    x = torch.randn(4, 3)
    gg = ref.ghmc_g_f32(x, torch.tensor([-1, 3, 6, 1]))
    p = ref.sigmoid_f32(x)
    assert torch.equal(gg[:3], p[:3])
    assert torch.equal(gg[3], (p[3] - torch.tensor([0., 1., 0.])).abs())


def test_ghm_tot_above_2_24_is_within_one_ulp_of_the_fp32_sum():
    """tot is the exact count rounded once to fp32; the reference's fp32 sum of the valid mask can round differently above 2^24"""
    for n in (33_554_435, 27_895 * 1203):
        ones = torch.ones(n)
        s = float(ones.sum())
        t = np.float32(n)
        ulp = float(np.spacing(t))
        assert abs(float(t) - s) <= ulp, (n, float(t), s)


def test_argument_validation_of_the_ghm_and_l1_entry_points_without_a_gpu():
    """the six entry points of GHM-C, GHM-R, L1Loss and BalancedL1Loss check their arguments before any CUDA call; a loss pass of
    Q = 0 or M = 0 returns 0 and launches nothing (there is no device here: a launch would fail)"""
    from pointtinybenchmark_b200 import _lib
    lib = _lib.load()
    d = ctypes.c_void_p(16)      # never dereferenced: the checks fire first

    def err(rc, what):
        return rc == 2 and what in lib.ptb_last_error()

    # ptb_ghmc_bin_weights(logits, labels, label_weight, B, Q, C, edges, bins, momentum, acc_sum, counts, bin_weight, tot, stream)
    def cbw(x=d, lab=d, lw=d, B=2, Q=10, C=80, e=d, bins=10, mmt=0.0, acc=None, cnt=d, bw=d, tot=d):
        return lib.ptb_ghmc_bin_weights(x, lab, lw, B, Q, C, e, bins, mmt, acc, cnt, bw, tot, None)
    assert err(cbw(B=0), b'B > 0') and err(cbw(B=-1), b'B > 0')
    assert err(cbw(Q=-1), b'Q >= 0') and err(cbw(C=0), b'num_classes > 0')
    assert err(cbw(Q=(1 << 31) // 80 + 1), b'2^31') and err(cbw(Q=1 << 24, C=128), b'2^31')
    for bins in (0, 257):
        assert err(cbw(bins=bins), b'bins')
    assert err(cbw(mmt=0.75), b'NULL') and err(cbw(mmt=1e-3), b'NULL')
    for k in ('x', 'lab', 'lw', 'e', 'cnt', 'bw', 'tot'):
        assert err(cbw(**{k: None}), b'NULL'), k
    # ptb_ghmr_bin_weights(pred, target, weight, row_inv_norm, mu, B, Q, edges, bins, momentum, acc_sum, counts, bin_weight, tot, s)
    def rbw(p=d, t=d, w=d, inv=d, B=2, Q=10, e=d, bins=10, mmt=0.0, acc=None, cnt=d, bw=d, tot=d):
        return lib.ptb_ghmr_bin_weights(p, t, w, inv, 0.02, B, Q, e, bins, mmt, acc, cnt, bw, tot, None)
    assert err(rbw(B=0), b'B > 0') and err(rbw(Q=-1), b'Q >= 0') and err(rbw(Q=1 << 30), b'Q < (1LL << 30)')
    for bins in (0, 257):
        assert err(rbw(bins=bins), b'bins')
    assert err(rbw(mmt=0.7), b'NULL')
    for k in ('p', 't', 'w', 'inv', 'e', 'cnt', 'bw', 'tot'):
        assert err(rbw(**{k: None}), b'NULL'), k
    # ptb_ghmc_fwd_bwd(logits, labels, label_weight, Q, C, edges, bins, bin_weight, loss_sum, scale, grad, stream)
    def cfb(x=d, lab=d, lw=d, Q=10, C=80, e=d, bins=10, bw=d, out=d, grad=None):
        return lib.ptb_ghmc_fwd_bwd(x, lab, lw, Q, C, e, bins, bw, out, None, grad, None)
    assert err(cfb(Q=-1), b'Q >= 0') and err(cfb(C=0), b'num_classes > 0')
    for bins in (0, 257):
        assert err(cfb(bins=bins), b'bins')
        assert err(cfb(Q=0, bins=bins), b'bins'), 'bins are checked even when there is nothing to sum'
    for k in ('x', 'lab', 'lw', 'e', 'bw', 'out'):
        assert err(cfb(**{k: None}), b'NULL'), k
    # ptb_ghmr_fwd_bwd(pred, target, weight, Q, row_inv_norm, mu, edges, bins, bin_weight, loss_sum, scale, grad, stream)
    def rfb(p=d, t=d, w=d, Q=10, inv=d, e=d, bins=10, bw=d, out=d):
        return lib.ptb_ghmr_fwd_bwd(p, t, w, Q, inv, 0.02, e, bins, bw, out, None, None, None)
    assert err(rfb(Q=-1), b'Q >= 0')
    for bins in (0, 257):
        assert err(rfb(bins=bins), b'bins')
    for k in ('p', 't', 'w', 'inv', 'e', 'bw', 'out'):
        assert err(rfb(**{k: None}), b'NULL'), k
    # ptb_l1_rows_fwd_bwd(pred, target, weight, M, row_inv_norm, loss_sum, scale, grad, stream)
    def l1(p=d, t=d, M=10, inv=d, out=d):
        return lib.ptb_l1_rows_fwd_bwd(p, t, None, M, inv, out, None, None, None)
    assert err(l1(M=-1), b'M >= 0')
    for k in ('p', 't', 'inv', 'out'):
        assert err(l1(**{k: None}), b'NULL'), k
    # ptb_balanced_l1_rows_fwd_bwd(pred, target, weight, M, row_inv_norm, alpha, gamma, beta, loss_sum, scale, grad, stream)
    def bl1(p=d, t=d, M=10, inv=d, alpha=0.5, gamma=1.5, beta=1.0, out=d):
        return lib.ptb_balanced_l1_rows_fwd_bwd(p, t, None, M, inv, alpha, gamma, beta, out, None, None, None)
    assert err(bl1(M=-1), b'M >= 0')
    for a in (0.0, -0.5, float('nan')):
        assert err(bl1(alpha=a), b'alpha')
    for b in (0.0, -1.0, float('nan')):
        assert err(bl1(beta=b), b'beta')
    for gm in (0.0, -0.0, float('nan')):
        assert err(bl1(gamma=gm), b'gamma'), gm
        assert err(bl1(M=0, gamma=gm), b'gamma'), 'gamma is checked even when there is nothing to sum'
    for k in ('p', 't', 'inv', 'out'):
        assert err(bl1(**{k: None}), b'NULL'), k
    # Q = 0 / M = 0: 0 at once, the host-side sum untouched
    s = ctypes.c_float(0.0)
    ps = ctypes.c_void_p(ctypes.addressof(s))
    assert cfb(Q=0, x=None, lab=None, lw=None, out=ps) == 0
    assert rfb(Q=0, p=None, t=None, w=None, inv=None, out=ps) == 0
    assert l1(M=0, p=None, t=None, inv=None, out=ps) == 0
    assert bl1(M=0, p=None, t=None, inv=None, out=ps) == 0
    assert s.value == 0.0


def test_p2p_head_refuses_a_balanced_l1_loss_that_divides_by_zero():
    from pointtinybenchmark_b200.p2p_head import P2PHead
    for kw in (dict(gamma=0.0), dict(gamma=float('nan')), dict(alpha=0.0), dict(beta=0.0), dict(alpha=-0.5)):
        with pytest.raises(ValueError, match='gamma non-zero'):
            P2PHead(2, 256, point_anchor=[(0., 0.)], strides=[8], loss_reg=dict(type='BalancedL1Loss', **kw))
    h = P2PHead(2, 256, point_anchor=[(0., 0.)], strides=[8], loss_reg=dict(type='BalancedL1Loss', gamma=-1.0))
    assert h.loss_reg_cfg['gamma'] == -1.0
