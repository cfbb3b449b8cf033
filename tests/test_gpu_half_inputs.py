"""GPU: fp16 / bf16 feature maps (what a backbone under torch.autocast hands the head) through the towers and both heads.

The contract is self-referential: a half input gives what the fp32 path gives on `x.float()`.  Kernel level, bit for bit:
  * ptb_split_f16_from_bf16 == ptb_split_f16(auto_scale) on the upcast tensor;
  * the lo == 0 conv (ptb_conv_tc_f16x1a) == the three-MMA kernel fed the same hi and an explicit all-zero lo;
  * the half epilogue of the dgrad launch (ptb_conv_tc_f16x2_half_out) == the fp32 output cast to that dtype.
Head level (CPRHead / P2PHead, inference and training, inside and outside an autocast region): integer outputs equal, floats within
the suite's scale-relative 1e-4, the input gradient in the input's dtype within one ulp (at the tensor's scale) of the rounded fp32 gradient."""
import contextlib

import pytest
import torch

from oracle import synth
from tests.helpers import assert_close
from tests.test_gpu_cpr_head import head_cfg as cpr_cfg
from tests.test_gpu_p2p import head_cfg as p2p_cfg

pytestmark = pytest.mark.gpu

HALF = [torch.float16, torch.bfloat16]
PATH = {torch.float32: 'fp32-split', torch.float16: 'fp16-direct', torch.bfloat16: 'bf16-split'}


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _assert_bit_equal(a, b, what, signed_zero_ok=False):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    diff = _bits(a) != _bits(b)
    if signed_zero_ok:                      # +0 vs -0: the same number
        diff &= ~((a == 0) & (b == 0))
    assert int(diff.sum()) == 0, f'{what}: {int(diff.sum())} / {a.numel()} elements differ in their bits'


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. bf16 operand load
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['plain', 'signed_zeros', 'above_fp16_max', 'subnormal_after_scale', 'one_outlier'])
@pytest.mark.parametrize('B,H,W,C', [(2, 7, 13, 32), (1, 5, 9, 64), (1, 21, 33, 256)])
def test_split_from_bf16_is_bit_equal_to_the_split_of_the_upcast_tensor(ops, case, B, H, W, C):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + C)
    x = torch.randn(B, H, W, C, generator=g)
    if case == 'signed_zeros':
        x[torch.rand(x.shape, generator=g) < 0.3] = 0.0
        x[torch.rand(x.shape, generator=g) < 0.2] = -0.0
    elif case == 'above_fp16_max':
        x = x * 3.0e5                                    # most values beyond 65 504: the scale must bring them into range
    elif case == 'subnormal_after_scale':
        x = x * torch.where(torch.rand(x.shape, generator=g) < 0.5, 1.0, 2.0 ** -30)       # 2^-19 and below after the scale
    elif case == 'one_outlier':
        x = x * 1e-3
        x[0, H // 2, W // 2, C // 3] = 3.0e38
    xb = x.to(dev).to(torch.bfloat16)
    h, l, inv = ops.split_f16_from_bf16(xb)
    h0, l0, inv0 = ops.split_f16(xb.float(), auto_scale=True)
    _assert_bit_equal(h, h0, f'{case}: hi')
    _assert_bit_equal(l, l0, f'{case}: lo')
    _assert_bit_equal(inv, inv0, f'{case}: inverse scale')
    assert bool(torch.isfinite(h.float()).all())
    if case == 'above_fp16_max':
        assert float(xb.float().abs().max()) > 65504 and 2048 <= float(h.float().abs().max()) < 4096
    if case == 'subnormal_after_scale':
        assert int(((h.float().abs() > 0) & (h.float().abs() < 2.0 ** -14)).sum()) > 0, 'the case must reach fp16 subnormals'
    assert_close((h.double() + l.double()) * inv.double(), xb.double(), 1e-6, 'the pair restores the tensor')


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. lo == 0 conv
# ---------------------------------------------------------------------------------------------------------------------------------
# full 8 x 16 tiles, the 4 x 32 bottom strip (H % 8 in 1..4), the 16 x 8 right strip (W % 16 in 1..8), maps shorter than a box
TILE_SHAPES = [(2, 16, 32), (1, 17, 40), (1, 24, 17), (1, 3, 33), (1, 100, 168)]


@pytest.mark.parametrize('Cin', [32, 256])
@pytest.mark.parametrize('B,H,W', TILE_SHAPES)
def test_lo_zero_tower_conv_is_bit_equal_to_the_full_kernel_with_zero_lo(ops, B, H, W, Cin):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + Cin)
    h = torch.randn(B, H, W, Cin, generator=g).to(dev).half()
    w = (torch.randn(256, Cin, 3, 3, generator=g) * (1.4 / (Cin * 9) ** 0.5)).to(dev)
    wh, wl, inv_w = ops.conv3x3_pack_weight_f16(w)
    y, st = ops.conv3x3_c256_f16(h, None, wh, wl, inv_w)
    y0, st0 = ops.conv3x3_c256_f16(h, torch.zeros_like(h), wh, wl, inv_w)
    _assert_bit_equal(y, y0, 'conv output', signed_zero_ok=True)
    # the statistics are sums of the same values; fp64 atomics commute only up to rounding, so they agree to fp64 precision
    assert_close(st, st0, 1e-12, 'GroupNorm statistics')
    ref = torch.nn.functional.conv2d(h.double().permute(0, 3, 1, 2), w.double(), None, 1, 1)
    assert_close(y.permute(0, 3, 1, 2), ref, 5e-5, 'lo == 0 conv vs float64')


@pytest.mark.parametrize('taps,n_out', [(9, 80), (9, 128), (9, 320), (1, 80), (1, 20)])
@pytest.mark.parametrize('B,H,W,Cin', [(1, 17, 40, 256), (2, 16, 32, 32), (1, 24, 17, 256)])
def test_lo_zero_general_conv_is_bit_equal_to_the_full_kernel_with_zero_lo(ops, B, H, W, Cin, taps, n_out):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + Cin + taps + n_out)
    h = torch.randn(B, H, W, Cin, generator=g).to(dev).half()
    w = torch.randn(n_out, Cin, taps, generator=g) * 0.03
    b = torch.randn(n_out, generator=g).to(dev)
    packed = ops.conv_tc_pack_weight_f16((w if taps == 9 else w[..., 0]).to(dev), taps)
    y = ops.conv_tc_f16(h, None, packed, taps, n_out, bias=b)
    y0 = ops.conv_tc_f16(h, torch.zeros_like(h), packed, taps, n_out, bias=b)
    _assert_bit_equal(y[..., :n_out], y0[..., :n_out], f'taps={taps} N={n_out}', signed_zero_ok=True)


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. half epilogue of the dgrad launch
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('boost', [1.0, 2.0 ** 28])
@pytest.mark.parametrize('B,H,W', [(2, 19, 37), (1, 100, 168)])
def test_half_dgrad_epilogue_is_the_cast_of_the_fp32_epilogue(ops, dtype, boost, B, H, W):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(H + W)
    C = 256
    dy = (torch.randn(B, H, W, C, generator=g) * 1e-3).to(dev)
    w = (torch.randn(C, C, 3, 3, generator=g) * 0.02).to(dev)
    dh, dl, inv_dy = ops.split_f16_amax(dy, dy.abs().max().reshape(1).view(torch.int32))
    packed = ops.conv_tc_pack_weight_f16(w.flip(2, 3).transpose(0, 1).reshape(C, C, 9).contiguous(), 9)
    scale = inv_dy * boost                     # boost 2^28: most |dx| beyond fp16's largest finite value
    dx32 = ops.conv_tc_f16(dh, dl, packed, 9, C, dev_out_scale=scale)
    dxh = ops.conv_tc_f16(dh, dl, packed, 9, C, dev_out_scale=scale, out_dtype=dtype)
    assert dxh.dtype == dtype and dxh.shape == dx32.shape
    _assert_bit_equal(dxh, dx32.to(dtype), f'dx in {dtype}')
    if boost > 1 and dtype == torch.float16:
        assert bool(torch.isinf(dxh).any()), 'the boosted gradient must overflow fp16 (round to +-inf, as the cast does)'


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. - 6. the heads
# ---------------------------------------------------------------------------------------------------------------------------------
def _autocast(on):
    return torch.autocast('cuda', dtype=torch.bfloat16) if on else contextlib.nullcontext()


def _cpr(shape, seed=2024, **cfg_over):
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    over = dict(B=2, n=60) if shape == 'full' else {}
    inp = synth.cpr_inputs('headline' if shape == 'full' else 'lite', seed, trained_like=False, with_towers=True, **over)
    hc = cpr_cfg(inp['cfgd'])
    hc.update(cfg_over)
    head = build_head(hc).cuda()
    g = torch.Generator().manual_seed(5)
    w = dict(inp['weights'])
    if hc['num_cls_fcs'] == 0:      # probabilities spread over (0, 1) with clear margins: every filter of the refiner has work to do
        w['cls_out.weight'] = torch.randn(80, 256, generator=g) * 0.16
        w['cls_out.bias'] = torch.full((80,), -2.0)
    else:
        w = {k: v for k, v in w.items() if k.startswith('cls_convs.')}
    sd = head.state_dict()
    sd.update(w)
    head.load_state_dict(sd, strict=True)
    dev = torch.device('cuda:0')
    gt = dict(gt_bboxes=[b.to(dev) for b in inp['gt_bboxes']], gt_labels=[l.to(dev) for l in inp['gt_labels']])
    aid = [a.to(dev) for a in inp['gt_anns_id']]
    return head, inp['cls_feat'].to(dev), inp['img_metas'], gt, aid


def _param_grads(head):
    out = {k: p.grad.clone() for k, p in head.named_parameters() if p.grad is not None}
    head.zero_grad(set_to_none=True)
    return out


def _check_input_grad(xh, x32, what, ulps=1):
    """the gradient of a half input arrives in its dtype and is the fp32 gradient rounded to it.  The two backward passes differ by
    fp32 rounding noise (atomics of the loss backward, cuDNN's algorithm choice for P2PHead's output convs), which can move a value
    across a rounding boundary: so at most one ulp (finfo.eps relative) at the scale of the tensor, and mostly the same bits.
    P2PHead feeds the input to two towers: autograd adds their two half-precision gradients in that dtype (as it does for two
    `.float()` casts of one half tensor), three roundings of partly cancelling terms instead of one: `ulps` = 4 there."""
    assert xh.grad is not None and xh.grad.dtype == xh.dtype and xh.grad.shape == xh.shape, what
    want = x32.grad.to(xh.dtype)
    assert bool(torch.isfinite(want.float()).all()) and float(want.float().abs().max()) > 0
    eps = torch.finfo(xh.dtype).eps
    e = assert_close(xh.grad, want, ulps * eps, f'{what}: input gradient vs the rounded fp32 gradient')
    assert_close(xh.grad, x32.grad, ulps * eps, f'{what}: input gradient vs the fp32 gradient')
    same = float((_bits(xh.grad) == _bits(want)).float().mean())
    print(f'[{what}] input gradient: {100 * same:.2f} % of the elements have the bits of the rounded fp32 gradient, worst {e / eps:.2f} ulp')
    assert same > 0.5 / ulps


def _check_param_grad(k, got, ref, what):
    if k == 'ins_out.bias' and 'ins_out.weight' in ref:
        # softmax over the bag is shift invariant: this gradient is analytically zero, rounding noise of the atomics on both sides
        assert float((got[k] - ref[k]).abs().max()) <= 1e-5 * float(ref['ins_out.weight'].abs().max()), f'd/d {k} {what}'
    else:
        assert_close(got[k], ref[k], 1e-4, f'd/d {k} {what}')


GRAD_SCALE = 4096.0      # a loss scale, as a GradScaler applies: keeps the fp16 input gradient out of fp16's subnormal range


@pytest.mark.parametrize('shape', ['lite', 'full'])
@pytest.mark.parametrize('dtype', HALF)
def test_cpr_head_inference_half_input(ops, dtype, shape):
    head, x, metas, gt, aid = _cpr(shape)
    head.eval()
    xh = x.to(dtype)
    with torch.no_grad():
        ref, nr_ref = head.simple_test((xh.float(),), metas, **gt, gt_anns_id=aid, cascade_out_fmt=True)
        assert head.last_tower_backend == 'wgmma-f16x2' and head.last_input_path == 'fp32-split'
        f_ref = head((xh.float(),))[0][0]
        for ac in (False, True):
            for xin in (xh, xh.contiguous(memory_format=torch.channels_last)):
                with _autocast(ac):
                    got, nr = head.simple_test((xin,), metas, **gt, gt_anns_id=aid, cascade_out_fmt=True)
                    f = head((xin,))[0][0]
                assert head.last_tower_backend == 'wgmma-f16x2' and head.last_input_path == PATH[dtype]
                assert f.dtype == torch.float32 and all(r[0].dtype == torch.float32 for r in got)
                assert torch.equal(torch.cat(nr), torch.cat(nr_ref)), 'not_refine'
                assert all(torch.equal(a[1], b[1]) for a, b in zip(got, ref)), 'labels'
                assert_close(torch.cat([r[0] for r in got]), torch.cat([r[0] for r in ref]), 1e-4, f'detections (autocast={ac})')
                assert_close(f, f_ref, 1e-4, f'tower output (autocast={ac})')
    assert 0.02 < float(torch.cat(nr_ref).float().mean()) < 0.98, 'both branches of the refine decision must occur'


@pytest.mark.parametrize('shape', ['lite', 'full'])
@pytest.mark.parametrize('dtype', HALF)
def test_cpr_head_training_half_input(ops, dtype, shape):
    head, x, metas, gt, _ = _cpr(shape)
    head.train()

    def step(xin, ac):
        with _autocast(ac):
            losses = head.forward_train((xin,), metas, gt['gt_bboxes'], gt['gt_labels'])
        assert all(v.dtype == torch.float32 for v in losses.values())
        (sum(v for k, v in losses.items() if 'loss' in k) * GRAD_SCALE).backward()
        return {k: v.detach().clone() for k, v in losses.items()}, _param_grads(head), head.last_tower_backend, head.last_input_path

    x32 = x.to(dtype).float().requires_grad_(True)
    l_ref, g_ref, backend, path = step(x32, False)
    assert backend == 'wgmma-f16x2-train' and path == 'fp32-split'
    for ac in (False, True):
        xh = x.to(dtype).requires_grad_(True)
        l, gr, backend, path = step(xh, ac)
        assert backend == 'wgmma-f16x2-train' and path == PATH[dtype]
        for k in l_ref:
            assert_close(l[k].reshape(-1), l_ref[k].reshape(-1), 1e-4, f'{k} (autocast={ac})')
        assert set(gr) == set(g_ref)
        for k in g_ref:
            assert gr[k].dtype == torch.float32
            _check_param_grad(k, gr, g_ref, f'(autocast={ac})')
        _check_input_grad(xh, x32, f'CPRHead {dtype} (autocast={ac})')


def _p2p(shape, seed=555):
    from pointtinybenchmark_b200 import p2p_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    inp = synth.p2p_inputs('headline', seed, B=2, n=40) if shape == 'full' else synth.p2p_inputs('lite', seed)
    d = inp['cfgd']
    torch.manual_seed(seed)
    head = build_head(p2p_cfg(d, 0.5)).cuda()
    with torch.no_grad():
        head.cls_out.weight.mul_(4.4)          # trained-like spread of the logits around the -log(99) bias
    dev = torch.device('cuda:0')
    H, W = d['pad_hw'][0] // d['stride'], d['pad_hw'][1] // d['stride']
    x = torch.randn(d['B'], 256, H, W, generator=torch.Generator().manual_seed(seed + 1)).to(dev)
    return head, x, inp['img_metas'], [b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']]


@pytest.mark.parametrize('shape', ['lite', 'full'])
@pytest.mark.parametrize('dtype', HALF)
def test_p2p_head_inference_half_input(ops, dtype, shape):
    head, x, metas, _, _ = _p2p(shape)
    head.eval()
    xh = x.to(dtype)
    with torch.no_grad():
        ref = head.simple_test((xh.float(),), metas)
        assert head.last_tower_backend == 'wgmma-f16x2' and head.last_input_path == 'fp32-split'
        c_ref, p_ref = head((xh.float(),))
        for ac in (False, True):
            with _autocast(ac):
                got = head.simple_test((xh,), metas)
                c, p = head((xh,))
            assert head.last_tower_backend == 'wgmma-f16x2' and head.last_input_path == PATH[dtype]
            assert c[0].dtype == torch.float32 and p[0].dtype == torch.float32
            assert_close(c[0], c_ref[0], 1e-4, 'cls_out')
            assert_close(p[0], p_ref[0], 1e-4, 'pts_out')
            for (b, lab), (b0, lab0) in zip(got, ref):
                assert torch.equal(lab, lab0), 'labels of the kept detections'
                assert b.dtype == torch.float32
                assert_close(b, b0, 1e-4, 'kept boxes')
    assert sum(len(r[1]) for r in ref) > 0


@pytest.mark.parametrize('shape', ['lite', 'full'])
@pytest.mark.parametrize('dtype', HALF)
def test_p2p_head_training_half_input(ops, dtype, shape):
    head, x, metas, gtb, gtl = _p2p(shape)
    head.train()

    def step(xin, ac):
        with _autocast(ac):
            losses = head.forward_train((xin,), metas, gtb, gtl)
        flat = torch.stack([v for vs in losses.values() for v in vs])
        assert flat.dtype == torch.float32
        (flat.sum() * GRAD_SCALE).backward()
        return flat.detach().clone(), _param_grads(head), [t.clone() for t in head._last_targets['labels']], head.last_input_path

    x32 = x.to(dtype).float().requires_grad_(True)
    l_ref, g_ref, t_ref, path = step(x32, False)
    assert head.last_tower_backend == 'wgmma-f16x2-train' and path == 'fp32-split'
    for ac in (False, True):
        xh = x.to(dtype).requires_grad_(True)
        l, gr, t, path = step(xh, ac)
        assert head.last_tower_backend == 'wgmma-f16x2-train' and path == PATH[dtype]
        assert all(torch.equal(a, b) for a, b in zip(t, t_ref)), 'assigned labels'
        assert_close(l, l_ref, 1e-4, f'losses (autocast={ac})')
        for k in g_ref:
            assert_close(gr[k], g_ref[k], 1e-4, f'd/d {k} (autocast={ac})')
        _check_input_grad(xh, x32, f'P2PHead {dtype} (autocast={ac})', ulps=4)


GRID = dict(type='GridCirclesPtFeatGenerator', radius=3)
VARIANTS = {
    'fcs': dict(num_cls_fcs=2, fc_out_channels=64),
    'grid': dict(train_pts_extractor=dict(pos_generator=GRID, neg_generator=dict(type='OutCirclePtFeatGenerator', radius=5, class_wise=True)),
                 refine_pts_extractor=dict(pos_generator=GRID, neg_generator=dict(type='OutCirclePtFeatGenerator', radius=5, keep_wh=True,
                                                                                  class_wise=True))),
}


@pytest.mark.parametrize('variant', sorted(VARIANTS))
def test_cpr_variants_bf16_inside_autocast(ops, variant):
    """the torch-level pieces of the head (the generic path's Linear stack and softmax, the grid-bag loss chain) stay fp32 inside an
    autocast region: a bf16 input there gives what x.float() gives outside one."""
    head, x, metas, gt, aid = _cpr('lite', **VARIANTS[variant])
    if variant == 'fcs':
        with torch.no_grad():
            for fc in head.cls_fcs:
                fc.weight.mul_(8.0)
            head.cls_out.weight.mul_(16.0)
    xb = x.to(torch.bfloat16)

    def run(xin, ac):
        head.train()
        with _autocast(ac):
            losses = head.forward_train((xin,), metas, gt['gt_bboxes'], gt['gt_labels'])
        sum(v for k, v in losses.items() if 'loss' in k).backward()
        grads = _param_grads(head)
        head.eval()
        with torch.no_grad(), _autocast(ac):
            res, nr = head.simple_test((xin.detach(),), metas, **gt, gt_anns_id=aid, cascade_out_fmt=True)
        return losses, grads, torch.cat([r[0] for r in res]), torch.cat(nr)

    l0, g0, det0, nr0 = run(xb.float().requires_grad_(True), False)
    l1, g1, det1, nr1 = run(xb.clone().requires_grad_(True), True)
    for k in l0:
        assert l1[k].dtype == torch.float32
        assert_close(l1[k].reshape(-1), l0[k].reshape(-1), 1e-4, f'{variant} {k}')
    for k in g0:
        _check_param_grad(k, g1, g0, variant)
    assert torch.equal(nr1, nr0), 'not_refine'
    assert det1.dtype == torch.float32
    assert_close(det1, det0, 1e-4, f'{variant} detections')


def test_half_inputs_outside_the_fp16_split_mode_are_refused(ops, monkeypatch):
    from pointtinybenchmark_b200.layers import tower
    head, x, _, _, _ = _cpr('lite')
    head.eval()
    monkeypatch.setenv('PTB_CONV_MODE', 'tf32x3')
    with torch.no_grad():
        info = {}
        tower(head.cls_convs, x, info)
        assert info == dict(backend='wgmma-3xtf32', input_path='fp32-split')
        with pytest.raises(NotImplementedError, match='PTB_CONV_MODE=tf32x3'):
            head((x.half(),))
    with pytest.raises(RuntimeError):          # other dtypes are not tower inputs: torch's own dtype error, as before
        head((x.double(),))
