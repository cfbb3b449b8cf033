"""CPU checks of the CPR loss plumbing: the backward-path choice of the fused loss (cpr_head.loss_bwd_plan), the logit map's GEMM
path, the reach of a bag offset table, and the float64 loss reference of tests/cpr_loss_ref.py against the oracle's fp32 autograd."""
import pytest
import torch

from oracle import cpr as ocpr
from pointtinybenchmark_b200 import ops
from pointtinybenchmark_b200.cpr_head import _CircleBags, _loss_map_on_tc, loss_bwd_plan
from tests.cpr_loss_ref import cpr_loss_ref, oracle_bag_logits, taps
from tests.helpers import scale_rel_err


@pytest.mark.parametrize('N', list(range(1, 130)) + [200, 256])
def test_default_mode_keeps_ceil8_and_scatter(N):
    for K in (1, 121, 289, 361):
        assert loss_bwd_plan(N, K, True, True) == ((N + 7) // 8 * 8, 'scatter', None)
        assert loss_bwd_plan(N, K, True, True, 'scatter') == ((N + 7) // 8 * 8, 'scatter', None)
        assert loss_bwd_plan(N, K, True, True, 'staged') == ((N + 7) // 8 * 8, 'staged', None)
        assert loss_bwd_plan(N, K, True, False) == ((N + 7) // 8 * 8, 'staged', None)       # no MIL term: staged chain
        assert loss_bwd_plan(N, K, False, True) == ((N + 7) // 8 * 8, 'staged', None)       # grid-cell bags


@pytest.mark.parametrize('env_mode,deterministic', [('tiles', False), (None, True), ('tiles', True)])
def test_deterministic_mode_table(env_mode, deterministic):
    """bit-reproducible gradients asked for: the tile kernel for every N <= 80 and K <= 320 on ring bags with the MIL loss (NP = ceil16,
    so LD is a multiple of 32 and at most 160), otherwise the atomic path that would run plus the reason, never a silent fallback."""
    for N in range(1, 257):
        for K in (1, 9, 121, 289, 320, 321, 361):
            NP, path, reason = loss_bwd_plan(N, K, True, True, env_mode, deterministic)
            assert NP == (N + 15) // 16 * 16 and NP >= N and (2 * NP) % 32 == 0
            if N <= 80 and K <= 320:
                assert (path, reason) == ('tiles', None), (N, K)
                assert 2 * NP <= 160
            else:
                assert path == 'scatter' and reason, (N, K)
                assert ('num_classes' in reason) == (N > 80) and (('samples per bag' in reason) == (N <= 80))
        NP, path, reason = loss_bwd_plan(N, 121, False, True, env_mode, deterministic)
        assert path == 'staged' and 'grid-cell' in reason
        NP, path, reason = loss_bwd_plan(N, 121, True, False, env_mode, deterministic)
        assert path == 'staged' and 'with_mil_loss' in reason


@pytest.mark.parametrize('env_mode', ['scatter', 'staged'])
def test_explicit_atomic_path_under_deterministic_mode_is_flagged(env_mode):
    NP, path, reason = loss_bwd_plan(80, 121, True, True, env_mode, True)
    assert (NP, path) == (80, env_mode) and f'PTB_LOSS_BWD={env_mode}' in reason


def test_n80_layout_is_the_same_in_every_mode():
    """N = 80 (COCO): NP = 80 whether or not the gradients must be bit-reproducible, so the training bits do not depend on the mode."""
    assert loss_bwd_plan(80, 289, True, True)[0] == loss_bwd_plan(80, 289, True, True, None, True)[0] == 80


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('C', [32, 48, 128, 256])
@pytest.mark.parametrize('N', [1, 20, 80, 128, 129, 200, 256, 257, 365, 1203, 1280])
def test_logit_map_path_choice(N, C, deterministic):
    """the logit map runs on the tensor cores for exactly the shapes of the two tensor-core branches it replaces (one launch: C, LD <= 256
    with C and LD multiples of 32; column slices: more than 256 classes with C % 32 == 0), FFMA for every other shape; and at C = 256
    every shape whose map ran on the tensor cores took one of those branches' tensor-core backwards, which is now the one taken."""
    NP = loss_bwd_plan(N, 121, True, True, None, deterministic)[0]
    LD = 2 * NP
    one_launch = C % 32 == 0 and LD % 32 == 0 and C <= 256 and LD <= 256
    sliced = not one_launch and N > 256 and C % 32 == 0
    assert _loss_map_on_tc(N, C, LD) == (one_launch or sliced), (N, C, LD)
    if C == 256 and (one_launch or sliced):
        assert (LD > 256 and LD % 32 == 0) or (one_launch and LD % 8 == 0), (N, LD)


def test_offsets_reach_is_cached_on_the_tensor():
    a = ops.circle_offsets(3, 4)
    assert ops.offsets_reach(a) == 12.0
    b = ops.circle_offsets(3, 8)
    assert ops.offsets_reach(b) == 24.0 and ops.offsets_reach(a) == 12.0
    a.mul_(3.0)                                   # modified in place: the cached value is stale and must not be used
    assert ops.offsets_reach(a) == 36.0
    assert _CircleBags(b, 8.0).reach == 24.0 and _CircleBags(b, 8.0, reach=30.0).reach == 30.0
    assert ops.offsets_reach(torch.zeros(0, 2)) == 0.0


def test_a_fresh_table_never_inherits_a_cached_reach():
    """the reach belongs to the tensor object: freeing a table and building one of equal size with a larger reach (the allocator may
    hand it the same address) gives the new table its own reach, and so does a new tensor over the same storage."""
    for _ in range(20):
        a = ops.circle_offsets(3, 4)
        assert ops.offsets_reach(a) == 12.0
        del a
        b = ops.circle_offsets(3, 8)
        assert ops.offsets_reach(b) == 24.0
        v = b.view(-1, 2)                        # a second tensor object on the same storage: no cached value to inherit
        assert not hasattr(v, '_ptb_reach')
        v.mul_(2.0)
        assert ops.offsets_reach(v) == 48.0 and ops.offsets_reach(b) == 48.0


def _cpu_head(radius=5, stride=8):
    from pointtinybenchmark_b200.registry import build_head
    return build_head(dict(type='CPRHead', num_classes=3, in_channels=256, feat_channels=256, stacked_convs=1, strides=[stride],
                           norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                           train_pts_extractor=dict(pos_generator=dict(type='CirclePtFeatGenerator', radius=radius),
                                                    neg_generator=dict(type='OutCirclePtFeatGenerator', radius=radius))))


def test_reach_under_inference_mode():
    """inference tensors carry no version counter: the reach must still be computed (not cached) for them, and a head whose offset
    table is first built under torch.inference_mode() keeps the reach of its host table beside it."""
    head = _cpu_head(radius=5, stride=8)
    gen = head.train_pts_extractor['pos_generator']
    with torch.inference_mode():
        t = ops.circle_offsets(3, 4)
        assert t.is_inference() and ops.offsets_reach(t) == 12.0
        t.mul_(2.0)
        assert ops.offsets_reach(t) == 24.0                                  # recomputed, never a stale cached value
        assert _CircleBags(t, 4.0).reach == 24.0
        off = head._offsets(gen, 'cpu')
        assert off.is_inference() and head._offset_table(gen, 'cpu')[1] == 40.0
        assert head._bags(gen, 'cpu').reach == 40.0 and ops.offsets_reach(off) == 40.0
    assert head._bags(gen, 'cpu').reach == 40.0                              # the same table, used outside inference mode


def _case(seed, N=5, NP=8, K_r=2, stride=8.0, B=2, H=7, W=9):
    g = torch.Generator().manual_seed(seed)
    LD = 2 * NP
    lmap = torch.full((B, H, W, LD), 50.0)
    lmap[..., :N] = torch.randn(B, H, W, N, generator=g) * 2 - 1
    lmap[..., NP:NP + N] = torch.randn(B, H, W, N, generator=g) * 2
    G = 9
    centers = (torch.rand(G, 2, generator=g) * torch.tensor([W * stride + 20, H * stride + 20]) - 10).float()
    centers[0] = 0.0
    centers[1] = torch.tensor([W * stride, H * stride])
    bag_img = torch.tensor([0] * 5 + [1] * 4, dtype=torch.int32)
    labels = torch.randint(0, N, (G,), generator=g)
    pad_hw = torch.tensor([[H * stride, W * stride], [H * stride - 5, W * stride - 3]], dtype=torch.int32)
    off = ops.circle_offsets(K_r, stride)
    nm = (torch.rand(B, H, W, N, generator=g) < 0.7).to(torch.uint8)
    return lmap, centers, bag_img, labels, pad_hw, off, nm


def test_reference_sample_points_match_grid_sample():
    """the float64 bilinear samples at the fp32 sample positions agree with F.grid_sample (fp32) to fp32 rounding: the positions, taps
    and border clamp are the same."""
    for seed in range(4):
        lmap, centers, bag_img, labels, pad_hw, off, nm = _case(seed)
        B, H, W, LD = lmap.shape
        idx, w = taps(centers, bag_img, off, 8.0, H, W)
        assert bool((w >= 0).all()) and torch.allclose(w.sum(-1), torch.ones_like(w[..., 0]), atol=1e-12)
        bl64 = (lmap.double().reshape(-1, LD)[idx] * w[..., None]).sum(2)
        bl32 = oracle_bag_logits(lmap, centers, bag_img, off, 8.0)
        assert float((bl64 - bl32.double()).abs().max()) <= 1e-5 * float(lmap.abs().max())


def test_reference_matches_the_oracle_loss_and_autograd():
    """the reference's losses and d loss / d lmap agree with the oracle's own fp32 functions (F.grid_sample + mil_loss + gfocal_loss,
    autograd in fp32) to fp32 accuracy."""
    N, NP, eps, stride = 5, 8, 1e-6, 8.0
    lmap, centers, bag_img, labels, pad_hw, off, nm = _case(7, N=N, NP=NP)
    B, H, W, LD = lmap.shape
    s = dict(mil=0.37, gt=0.29, neg=0.011)
    ref = cpr_loss_ref(lmap, N, NP, centers, bag_img, off, stride, pad_hw, labels, eps, s['mil'], s['gt'], s['neg'], neg_mask=nm)
    L = lmap.clone().requires_grad_(True)
    pts = off[None] + centers[:, None]
    bl = torch.cat([ocpr.sample_point_feat(L[b:b + 1].permute(0, 3, 1, 2), pts[bag_img.long() == b], stride) for b in range(B)])
    valid = torch.cat([ocpr.point_valid(pts[bag_img.long() == b], float(pad_hw[b, 0]), float(pad_hw[b, 1])) for b in range(B)])
    w = valid.float()
    loss, acc, num, prob = ocpr.mil_loss(bl[..., :N].sigmoid(), bl[..., NP:NP + N], labels, w[..., None], 1.0, eps)
    onehot = torch.zeros(len(labels), N)
    onehot[torch.arange(len(labels)), labels] = 1
    gt = ocpr.gfocal_loss(bl[:, -1, :N].sigmoid(), onehot, w[:, -1:], eps).sum()
    negp = L[..., :N].sigmoid()
    neg = ocpr.gfocal_loss(negp, torch.zeros_like(negp), nm.float(), eps).sum()
    total = s['mil'] * loss * num + s['gt'] * gt + s['neg'] * neg
    total.backward()
    assert scale_rel_err(prob, ref['bag_prob']) <= 1e-5
    assert scale_rel_err((loss * num).reshape(1), ref['mil_sum'].reshape(1)) <= 1e-5
    assert scale_rel_err(gt.reshape(1), ref['gt_sum'].reshape(1)) <= 1e-5
    assert scale_rel_err(total.reshape(1), ref['total'].reshape(1)) <= 1e-5
    assert ref['stats'] == (float(num), float(round(float(acc) * len(labels) / 100.0)))
    assert scale_rel_err(L.grad, ref['grad']) <= 1e-4
    assert bool((ref['grad'][..., N:NP] == 0).all()) and bool((ref['grad'][..., NP + N:] == 0).all())
