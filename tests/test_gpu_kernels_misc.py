"""GPU parity of individual kernels: MIL loss fwd/bwd, gfocal, linear backward, gather backward; size-independent
properties at the headline size (linearity of the gather, determinism, mask consistency)."""
import pytest
import torch

from oracle import cpr as ocpr
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


@pytest.mark.parametrize('G,K,C', [(7, 121, 80), (3, 9, 1), (5, 289, 20), (1, 1, 3)])
def test_mil_loss_fwd_bwd(ops, G, K, C):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(G * 1000 + K)
    NP = (C + 7) // 8 * 8
    LD = 2 * NP
    cls = torch.randn(G, K, C, generator=g) * 2
    ins = torch.randn(G, K, C, generator=g) * 2
    w = (torch.rand(G, K, generator=g) > 0.2).float()
    if G > 1:
        w[1] = 0          # a bag with no valid sample: label weight 0, excluded from num_sample
    labels = torch.randint(0, C, (G,), generator=g)
    logits = torch.zeros(G, K, LD)
    logits[..., :C], logits[..., NP:NP + C] = cls, ins
    lg = logits.to(dev)
    bag_prob, loss_sum, stats = ops.mil_loss_fwd(lg, C, NP, w.to(dev), labels.int().to(dev), 1e-6)
    c_ = cls.clone().requires_grad_(True)
    i_ = ins.clone().requires_grad_(True)
    loss, acc, num, prob = ocpr.mil_loss(c_.sigmoid(), i_, labels, w[..., None], 1.0, 1e-6)
    assert_close(bag_prob, prob.detach(), 1e-4, 'bag prob')
    assert float(stats[0]) == max(float((w.sum(1) > 0).sum()), 0.0)
    assert_close(loss_sum / max(float(stats[0]), 1.0), loss.detach().reshape(1), 1e-4, 'MIL loss')
    assert abs(float(stats[1]) * 100.0 / G - float(acc)) < 1e-3
    loss.backward()
    scale = torch.tensor([1.0 / num], device=dev)
    grad = ops.mil_loss_bwd(lg, C, NP, w.to(dev), labels.int().to(dev), 1e-6, bag_prob, scale)
    assert_close(grad[..., :C], c_.grad, 2e-4, 'd/d cls logits')
    assert_close(grad[..., NP:NP + C], i_.grad, 2e-4, 'd/d ins logits')


def test_gfocal_and_linear_backward(ops):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(5)
    M, C, Cin = 1000, 80, 256
    x = torch.randn(M, Cin, generator=g)
    wgt = torch.randn(160, Cin, generator=g) * 0.05
    b = torch.randn(160, generator=g)
    y = ops.linear_rows(x.to(dev), wgt.to(dev), b.to(dev))
    assert_close(y, torch.nn.functional.linear(x, wgt, b), 1e-5, 'linear fwd')
    dy = torch.randn(M, 160, generator=g)
    dx = ops.linear_rows_bwd_x(dy.to(dev), wgt.to(dev))
    assert_close(dx, dy @ wgt, 1e-5, 'linear bwd x')
    dw, db = ops.linear_rows_bwd_w(dy.to(dev), x.to(dev))
    assert_close(dw, dy.t() @ x, 1e-5, 'linear bwd w')
    assert_close(db, dy.sum(0), 1e-5, 'linear bwd b')
    dw2, _ = ops.linear_rows_bwd_w(dy.to(dev), x.to(dev))
    assert torch.equal(dw, dw2), 'weight-gradient reduction must be deterministic'
    # gfocal
    logits = (torch.randn(M, C, generator=g) * 2).requires_grad_(True)
    mask = (torch.rand(M, C, generator=g) > 0.3)
    ref = ocpr.gfocal_loss(logits.sigmoid(), torch.zeros(M, C), mask.float()).sum()
    ref.backward()
    got = ops.gfocal_fwd(logits.detach().to(dev), M, C, C, None, mask.to(torch.uint8).to(dev), 1e-6)
    assert_close(got, ref.detach().reshape(1), 1e-5, 'gfocal sum (neg form)')
    grad = torch.zeros(M, C, device=dev)
    ops.gfocal_bwd(logits.detach().to(dev), M, C, C, None, mask.to(torch.uint8).to(dev), 1e-6, torch.ones(1, device=dev), grad, C, False)
    assert_close(grad, logits.grad, 1e-4, 'gfocal grad')
    lab = torch.randint(0, C, (M,), generator=g)
    wrow = (torch.rand(M, generator=g) > 0.5).float()
    l2 = logits.detach().clone().requires_grad_(True)
    oh = torch.zeros(M, C); oh[torch.arange(M), lab] = 1
    r2 = ocpr.gfocal_loss(l2.sigmoid(), oh, wrow[:, None]).sum(); r2.backward()
    got2 = ops.gfocal_fwd(l2.detach().to(dev), M, C, C, lab.int().to(dev), wrow.to(dev), 1e-6)
    assert_close(got2, r2.detach().reshape(1), 1e-5, 'gfocal sum (one-hot form)')
    g2 = torch.zeros(M, C, device=dev)
    ops.gfocal_bwd(l2.detach().to(dev), M, C, C, lab.int().to(dev), wrow.to(dev), 1e-6, torch.ones(1, device=dev), g2, C, False)
    assert_close(g2, l2.grad, 1e-4, 'gfocal grad (one-hot)')


def test_gather_backward_matches_autograd(ops):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(9)
    B, H, W, C, n, r, s = 2, 20, 28, 16, 6, 3, 8
    fmap = torch.randn(B, C, H, W, generator=g)
    centers = torch.rand(B * n, 2, generator=g) * torch.tensor([W * s * 1.1, H * s * 1.1]) - 8
    bag_img = torch.arange(B, dtype=torch.int32).repeat_interleave(n)
    off = ops.circle_offsets(r, s)
    pad_hw = torch.tensor([[H * s, W * s]] * B, dtype=torch.int32)
    f = fmap.clone().requires_grad_(True)
    outs = []
    for b in range(B):
        pts = ocpr.circle_bag_points(centers[bag_img == b], s, ocpr.default_cfg(), r)
        outs.append(ocpr.sample_point_feat(f[b:b + 1], pts, s))
    ref = torch.cat(outs)
    go = torch.randn(ref.shape, generator=g)
    (ref * go).sum().backward()
    fm = ops.to_nhwc(fmap.to(dev))
    feats, _, _ = ops.bag_gather(fm, centers.to(dev), bag_img.to(dev), off.to(dev), s, pad_hw.to(dev))
    assert torch.equal(feats.cpu(), ref.detach()), 'forward gather is bit-exact vs ATen CPU grid_sample'
    gm = ops.bag_gather_bwd(go.to(dev).contiguous(), tuple(fm.shape), centers.to(dev), bag_img.to(dev), off.to(dev), s)
    assert_close(gm.permute(0, 3, 1, 2), f.grad, 1e-5, 'gather backward')


def test_headline_size_properties(ops):
    """size-independent properties at BASELINE.json configs[1] scale (8 x 100x168x256, 500 pts, r=8)."""
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    B, H, W, C, n, r, s, ncls = 8, 100, 168, 256, 500, 8, 8, 80
    f1 = torch.randn(B, H, W, C, device=dev)
    f2 = torch.randn(B, H, W, C, device=dev)
    centers = (torch.rand(B * n, 2, device=dev) * torch.tensor([1344., 800.], device=dev)).contiguous()
    bag_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(n).contiguous()
    pad_hw = torch.tensor([[800, 1344]] * B, dtype=torch.int32, device=dev)
    off = ops.circle_offsets(r, s).to(dev)
    a, pts, valid = ops.bag_gather(f1, centers, bag_img, off, s, pad_hw)
    a2, _, _ = ops.bag_gather(f1, centers, bag_img, off, s, pad_hw)
    assert torch.equal(a, a2), 'gather must be deterministic'
    b, _, _ = ops.bag_gather(f2, centers, bag_img, off, s, pad_hw, pts=False, valid=False)
    c, _, _ = ops.bag_gather(f1 + f2, centers, bag_img, off, s, pad_hw, pts=False, valid=False)
    assert_close(c, a + b, 1e-5, 'linearity of the gather')
    # the reference samples at index u = x/stride (cpr_head.py:192 + 88): x = 8*17 is exactly cell 17
    cc = torch.tensor([[8.0 * 17, 8.0 * 23]], device=dev)
    z, _, _ = ops.bag_gather(f1, cc, torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, 2, device=dev), s, pad_hw)
    assert_close(z[0, 0], f1[0, 23, 17], 1e-4, "sample on a cell index")   # (35/168-1+1)*84-0.5 is 17 up to fp32 rounding
    # valid mask == coordinate test; pts == centers + offsets
    exp_valid = (pts[..., 0] >= 0) & (pts[..., 0] < 1344) & (pts[..., 1] >= 0) & (pts[..., 1] < 800)
    assert torch.equal(valid, exp_valid)
    assert torch.equal(pts[..., :2], centers[:, None, :] + off[None])
    # Linear o gather == gather o Linear (the data-flow identity the fused path relies on)
    w = torch.randn(ncls, C, device=dev) * 0.05
    bb = torch.randn(ncls, device=dev)
    l1 = ops.linear_rows(a.reshape(-1, C), w, bb)
    lmap = ops.linear_rows(f1.reshape(-1, C), w, bb).view(B, H, W, ncls)
    l2, _, _ = ops.bag_gather(lmap, centers, bag_img, off, s, pad_hw, pts=False, valid=False)
    assert_close(l2.reshape(-1, ncls), l1, 1e-4, 'Linear(gather(x)) == gather(Linear(x))')


def test_label_groups_kernel_matches_torch_builder(ops):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(4)
    for lens, C in [([500] * 8, 80), ([3, 1, 0, 7], 5), ([1], 1), ([2000, 17], 80)]:
        labels = torch.cat([torch.randint(0, C, (n,), generator=g) for n in lens] + [torch.zeros(0, dtype=torch.long)]).int().to(dev)
        bag_img = torch.cat([torch.full((n,), i, dtype=torch.int32) for i, n in enumerate(lens)]).to(dev)
        img_ptr = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
        a = ops.label_groups(bag_img, labels, C)
        b = ops.label_groups_csr(labels, img_ptr, C, max(lens))
        G = labels.shape[0]
        assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]), (lens, C)
        ng = int(a[0].max()) + 1 if G else 0
        assert torch.equal(a[1][:ng + 1], b[1][:ng + 1])


def test_sigmoid_is_bit_identical_to_aten_cpu(ops):
    """ptb_common.cuh::sigmoidf_acc restates ATen's CPU sigmoid (0 - x, Sleef expf_u10, 1 + e, true division) operation by operation:
    the probabilities the kernels threshold / sort must equal torch.sigmoid on the CPU BIT FOR BIT (scores of ptb_p2p_decode_topk with
    nms_pre = -1 are sigmoid(logit) of every proposal in order)."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(11)
    H, W, C = 64, 96, 80
    x = torch.randn(1, H, W, C, generator=g) * 4.0 - 1.0
    x.view(-1)[:13] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 16.7, 17.0, 88.0, 100.5, -87.5, -100.5, -104.5, 50.0, -50.0])
    reg = torch.zeros(1, H, W, 2)
    img_hw = torch.tensor([[H * 8, W * 8]], dtype=torch.int32, device=dev)
    _, _, sc = ops.p2p_decode_topk(x.to(dev), reg.to(dev), C, 1, torch.zeros(1, 2, device=dev), 8, 1.0, img_hw, -1)
    ref = torch.sigmoid(x.reshape(-1, C))
    got = sc[0].cpu()
    nbad = int((got.view(torch.int32) != ref.view(torch.int32)).sum())
    assert nbad == 0, f'{nbad} / {ref.numel()} sigmoid values differ from ATen CPU in their bits'
    # every fp32 value in [-89, 89] in ascending order, in chunks: bit-identical, and non-decreasing (the fused refine's classify filter
    # compares sigmoid(label logit) with sigmoid(max logit) instead of taking an arg-max over the probabilities: that needs monotony)
    top = int(torch.tensor(89.0).view(torch.int32))
    n_neg = top + 1                                     # -89 .. -0 (descending bit patterns), then +0 .. 89
    total = 2 * n_neg
    H, W, C = 512, 512, 128
    chunk = H * W * C
    reg = torch.zeros(1, H, W, 2, device=dev)
    prev = None
    for a in range(0, total, chunk):
        i = torch.arange(a, a + chunk, dtype=torch.int64)
        bits = torch.where(i < n_neg, (1 << 31) | (top - i), i - n_neg)
        bits = torch.where(i < total, bits, torch.zeros_like(bits))                      # the last chunk's tail: +0
        x = (bits - ((bits >> 31) << 32)).to(torch.int32).view(torch.float32)
        n = min(chunk, total - a)
        _, _, sc = ops.p2p_decode_topk(x.to(dev).view(1, H, W, C), reg, C, 1, torch.zeros(1, 2, device=dev), 8, 1.0,
                                       torch.tensor([[H * 8, W * 8]], dtype=torch.int32, device=dev), -1)
        got = sc.view(-1)[:n]
        want = torch.sigmoid(x[:n]).to(dev)
        nbad = int((got.view(torch.int32) != want.view(torch.int32)).sum())
        assert nbad == 0, f'{nbad} sigmoid values in [{float(x[0])}, {float(x[n - 1])}] differ from ATen CPU in their bits'
        assert bool((got[1:] >= got[:-1]).all()), f'sigmoid decreases in [{float(x[0])}, {float(x[n - 1])}]'
        if prev is not None:
            assert float(got[0]) >= prev
        prev = float(got[-1])
    assert prev == float(torch.sigmoid(torch.tensor(89.0)))
