"""CPU: the float64 reference of the fused P2P losses (tests/p2p_loss_ref.py) against the oracle's fp32 functions, its fixed-order
sum against an exactly rounded sum, and the argument checks of the elementwise loss entry points, which run before any CUDA call."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p as op2p
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
