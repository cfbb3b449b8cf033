"""CPU checks of tests/roi_head_ref.py (no GPU): each host reference of the RoI head kernels against what is already trusted — the
float64 RoIAlign backward against torchvision's CPU backward, its term counts against its own gradient, the forward's two extensions
against oracle/roi_head.py's extractor, decode64 against orh.decode, the accuracy rule against torch.topk(1), bbox2delta_f32 against
orh.targets and bbox_loss64 against orh.loss."""
import numpy as np
import pytest
import torch
import torchvision

from oracle import roi_head as orh
from tests import roi_head_ref as ref
from tests.test_roi_head_golden import _random_rois


@pytest.mark.parametrize('sampling_ratio', [0, 2])
@pytest.mark.parametrize('stride', [4, 16])
def test_backward64_matches_torchvision(sampling_ratio, stride):
    """the float64 gradient against torchvision's CPU roi_align backward (fp32), within fp32 accumulation error; S bounds both"""
    g = torch.Generator().manual_seed(7)
    B, C, H, W = 3, 8, 24, 30
    rois = _random_rois(stride + 1, 300, B, H, W, stride)
    lv = ref.levels(rois, 1, 56)
    gy = torch.randn(rois.shape[0], C, 7, 7, generator=g)
    (got, s, cnt), = ref.roi_align_bwd64([(B, H, W, C)], [stride], rois, lv, 7, sampling_ratio, gy)
    x = torch.zeros(B, C, H, W, requires_grad=True)
    y = torchvision.ops.roi_align(x, rois, 7, 1.0 / stride, sampling_ratio, aligned=True)
    y.backward(gy)
    want = x.grad.permute(0, 2, 3, 1).double()
    n = int(cnt.max())
    assert n > 0
    assert bool(((got - want).abs() <= (n + 2) * ref.U * s + 1e-30).all())
    assert float((got - want).abs().max()) < 1e-4 * float(want.abs().max())
    # an element receives a term exactly where it has a non-zero sum of |terms|
    assert torch.equal((s > 0).all(-1), cnt[..., None].expand_as(s).gt(0).all(-1))
    assert torch.equal((s > 0).any(-1), cnt > 0)


def test_term_counts_by_hand():
    """one RoI, one bin, one sample per axis: a sample between pixels has four taps, on a pixel row two, on the last column (clamped)
    two; a sample beyond the map none"""
    shapes = [(1, 8, 8, 4)]
    cases = [((2.25 + 0.5, 3.5 + 0.5), 4), ((2.25 + 0.5, 3.0 + 0.5), 2), ((7.0 + 0.5, 3.0 + 0.5), 1), ((9.5 + 0.5, 3.0 + 0.5), 0),
             ((8.0 + 0.5, 2.5 + 0.5), 2)]
    for (x, y), want in cases:
        rois = torch.tensor([[0.0, x, y, x, y]])
        cnt = ref.term_counts(shapes, [1], rois, torch.zeros(1, dtype=torch.int64), 1, 1)[0]
        assert int(cnt.sum()) == want and int(cnt.max()) <= 1, (x, y, cnt.nonzero().tolist())


def test_forward_extensions_and_levels():
    """live RoIs equal orh.extract over four levels; batch index -1, B and a negative side give zero features (level -1 for the NaN
    scale); a fractional index truncates toward zero"""
    g = torch.Generator().manual_seed(3)
    B, C = 2, 8
    strides = [4, 8, 16, 32]
    feats = [torch.randn(B, C, 64 // s + 1, 80 // s + 3, generator=g) for s in strides]
    rois = _random_rois(9, 120, B, 16, 20, 4) * torch.tensor([1.0, 3.0, 3.0, 3.0, 3.0])
    rois[:, 0] = torch.randint(0, B, (120,), generator=g).float()
    rois[20, 0], rois[21, 0], rois[22, 0], rois[23, 0] = -1.0, float(B), -0.5, B - 0.25
    rois[24, 3] = rois[24, 1] - 5.0                                 # negative width: NaN scale
    for i, side in enumerate((60.0, 150.0, 300.0, 600.0)):           # one RoI on each level
        rois[30 + i, 3:] = rois[30 + i, 1:3] + side
    y, lv = ref.roi_align_fwd([f.permute(0, 2, 3, 1).contiguous() for f in feats], strides, rois, 7, 0, 56)
    assert int(lv[24]) == -1 and bool((y[24] == 0).all())
    assert bool((y[20] == 0).all()) and bool((y[21] == 0).all())
    live = torch.ones(120, dtype=torch.bool)
    live[[20, 21, 24]] = False
    r = rois.clone()
    r[:, 0] = r[:, 0].trunc()
    assert torch.equal(y[live], orh.extract(feats, r[live], 7, 0, 56, strides))
    assert torch.equal(lv[live], orh.map_roi_levels(rois[live], 4, 56))
    assert set(lv[live].tolist()) == {0, 1, 2, 3}


def test_decode64_matches_oracle_decode():
    g = torch.Generator().manual_seed(11)
    B, N, C = 2, 40, 5
    H, W = 90.0, 120.0
    rois = orh.pad_rois([torch.cat([torch.rand(n, 2, generator=g) * 80, torch.rand(n, 2, generator=g) * 40 + 90], 1)
                         for n in (N, N - 7)])[0]
    rois[:, 3:] = torch.maximum(rois[:, 3:], rois[:, 1:3])
    cls = torch.randn(B * N, C + 1, generator=g) * 4
    for agnostic in (False, True):
        reg = torch.randn(B * N, 4 if agnostic else 4 * C, generator=g) * 3
        means, stds = [0.1, -0.1, 0.0, 0.05], [0.1, 0.1, 0.2, 0.2]
        sf = torch.tensor([[1.25, 1.5, 1.25, 1.5], [2.0, 0.5, 2.0, 0.5]])
        boxes, scores, _ = ref.decode64(rois, cls, reg, B, C, agnostic, means, stds, abs(np.log(16 / 1000)), torch.tensor([[H, W]] * B), sf)
        reps = reg.shape[1] // 4
        ob, osc = orh.decode(rois, cls, reg, B, [(H, W)] * B, means * reps, stds * reps, [s.numpy() for s in sf])
        ob = ob.view(B, N, reps, 4).expand(B, N, C, 4)
        assert float((boxes - ob.double()).abs().max()) <= 1e-4 * 120
        assert float((scores - osc[..., :C].double()).abs().max()) <= 1e-6


def test_accuracy_rule_matches_topk():
    """torch.argmax agrees with topk(1) on rows with a unique winner and on rows with exactly one NaN"""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(500, 41, generator=g)
    nan_rows = torch.arange(0, 500, 3)
    x[nan_rows, torch.randint(0, 41, (nan_rows.numel(),), generator=g)] = float('nan')
    x[1, :] = -float('inf')
    x[1, 17] = float('inf')
    assert torch.equal(ref.argmax_rule(x), x.topk(1, dim=1)[1].squeeze(1))
    assert torch.equal(ref.argmax_rule(torch.tensor([[1.0, float('nan'), 3.0], [float('inf'), float('nan'), 1.0], [2.0, 5.0, 5.0],
                                                     [-float('inf')] * 3])), torch.tensor([1, 1, 1, 0]))


def test_bbox2delta_f32_matches_oracle_targets():
    """dx, dy bit for bit and dw, dh within one ulp of orh.targets (torch's CPU log)"""
    g = torch.Generator().manual_seed(2)
    from oracle import rpn_loss as orl
    gts = orl._boxes(g, 30, 200, 300, 4.0, 120.0)
    p = gts[torch.randint(0, 30, (400,), generator=g)] + torch.randn(400, 4, generator=g) * 6
    p[:, 2:] = torch.maximum(p[:, 2:], p[:, :2] + 1)
    gi = torch.randint(1, 31, (400,), generator=g)
    for means, stds in (([0., 0., 0., 0.], [0.1, 0.1, 0.2, 0.2]), ([0.05, -0.05, 0., 0.], [1., 1., 1., 1.])):
        o = orh.targets([(p, gi, torch.arange(400), torch.zeros(0, dtype=torch.long))], [gts], [torch.zeros(30, dtype=torch.long)], 1,
                        means, stds, -1)
        d = ref.bbox2delta_f32(p.numpy(), gts[gi - 1].numpy(), means, stds)
        assert np.array_equal(d[:, :2], o[3][:, :2].numpy())
        assert int(ref.ulp_diff(d[:, 2:], o[3][:, 2:].numpy()).max()) <= 1


def test_bbox_loss64_matches_oracle_loss():
    g = torch.Generator().manual_seed(4)
    R, C = 300, 6
    labels = torch.randint(-1, C + 1, (R,), generator=g)
    bt, bw = torch.randn(R, 4, generator=g), (torch.rand(R, 4, generator=g) > 0.2).float()
    for agnostic in (False, True):
        pred = torch.randn(R, 4 if agnostic else 4 * C, generator=g)
        for kind in (dict(type='L1Loss'), dict(type='SmoothL1Loss', beta=0.11)):
            s, grad, read = ref.bbox_loss64(pred, labels, bt, bw, C, agnostic, kind['type'] == 'SmoothL1Loss', kind.get('beta', 1.0))
            o = orh.loss(torch.zeros(R, C + 1), pred, torch.where(labels < 0, C, labels), torch.ones(R), bt, bw, C, agnostic,
                         dict(type='CrossEntropyLoss'), dict(kind, loss_weight=1.0))
            pos = (labels >= 0) & (labels < C)
            assert abs(s / R - float(o['loss_bbox'])) <= 1e-5 * abs(s / R)
            assert int(read.sum()) == 4 * int(pos.sum()) and bool((grad[~read] == 0).all())
