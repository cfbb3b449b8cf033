"""GPU: the tower conv with GroupNorm + ReLU applied inside the conv kernel (ptb_conv3x3_c256_f16_gn, ops.conv3x3_c256_f16_gn).

The fused launch must give the bits of the two kernels it replaces:
  * y bit for bit what ops.conv3x3_c256_f16 computes on the same operands (the K loop and epilogue are unchanged);
  * the fp16 (h, l) pair bit for bit what ops.gn_relu_apply_f16 computes on the fused launch's own y and statistics, and the fp32
    output what ops.gn_relu_apply(split=False) computes (the statistics are sums of fp64 atomics whose order varies from launch to
    launch, so each side is checked against the apply of its own statistics);
  * the statistics those of the unfused launch to fp64 rounding.
Every first-layer operand form (fp32 split, fp16 as is with lo == 0, bf16 split) and both output forms run at the headline map, at
maps whose bottom and right strips have every height and width class, at 1 to 16 images, with fewer items than SMs and with a
number of items per image that is not a multiple of the grid.  The towers (inference, both `want` forms, and the training forward)
must equal the explicit unfused op sequence bit for bit."""
import pytest
import torch

from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

EPS = 1e-5


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _assert_bit_equal(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    n = int((_bits(a) != _bits(b)).sum())
    assert n == 0, f'{what}: {n} / {a.numel()} elements differ in their bits'


def _operands(ops, x, form):
    """first-layer operands (h, l, device 1/scale) of a tower input x (B,H,W,Cin) fp32, in the given input form."""
    if form == 'fp32-split':
        return ops.split_f16(x, auto_scale=True)
    if form == 'fp16-direct':
        return x.half(), None, None
    return ops.split_f16_from_bf16(x.to(torch.bfloat16))


def _case(B, H, W, Cin, seed, gamma_scale=1.0):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).to(dev)
    w = (torch.randn(256, Cin, 3, 3, generator=g) * (1.4 / (Cin * 9) ** 0.5)).to(dev)
    gamma = ((1.0 + 0.3 * torch.randn(256, generator=g)) * gamma_scale).to(dev)
    beta = (0.2 * torch.randn(256, generator=g)).to(dev)
    return x, w, gamma, beta


def _check(ops, x, w, gamma, beta, form, out):
    h, l, inv = _operands(ops, x, form)
    wh, wl, inv_w = ops.conv3x3_pack_weight_f16(w)
    flag = torch.zeros(1, dtype=torch.int32, device=x.device)
    a, b, y, st = ops.conv3x3_c256_f16_gn(h, l, wh, wl, inv_w, inv, gamma, beta, EPS, flag, out=out)
    y0, st0 = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, inv)
    _assert_bit_equal(y, y0, 'conv output y')
    assert_close(st, st0, 1e-12, 'GroupNorm statistics')
    flag0 = torch.zeros(1, dtype=torch.int32, device=x.device)
    if out == 'f16pair':
        h0, l0 = ops.gn_relu_apply_f16(y, st, gamma, beta, 32, EPS, True, flag0)
        _assert_bit_equal(a, h0, 'h')
        _assert_bit_equal(b, l0, 'l')
        assert int(flag) == int(flag0), (int(flag), int(flag0))
    else:
        assert b is None
        o0 = ops.gn_relu_apply(y, st, gamma, beta, 32, EPS, True, split=False)
        _assert_bit_equal(a, o0, 'fp32 output')
    return flag


FORMS = ['fp32-split', 'fp16-direct', 'bf16-split']
OUTS = ['f16pair', 'fp32']
# bottom strip (H % 8 in 1..4), no strip (H % 8 in 5..7 or 0), right strip (W % 16 in 1..8), none (9..15, 0)
EDGE_SHAPES = [(3, h, w) for h in (1, 2, 3, 5, 9) for w in (8, 17, 40, 168)]
SHAPES = EDGE_SHAPES + [
    (1, 9, 17),        # 4 items on a grid of one CTA per SM: fewer items than SMs
    (16, 40, 40),      # 26 items per image, 416 items: not a multiple of the grid
    (3, 64, 96),       # 96 items per image
    (16, 5, 8),        # 16 images of 2 items
    (8, 100, 168),     # the headline map
]


@pytest.mark.parametrize('out', OUTS)
@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('B,H,W', SHAPES)
def test_fused_conv_gn_is_bit_equal_to_conv_then_apply(ops, B, H, W, form, out):
    x, w, gamma, beta = _case(B, H, W, 256, B * 100003 + H * 1009 + W * 13 + FORMS.index(form))
    _check(ops, x, w, gamma, beta, form, out)


@pytest.mark.parametrize('form', FORMS)
def test_fused_conv_gn_narrow_input(ops, form):
    x, w, gamma, beta = _case(2, 17, 40, 32, 77 + FORMS.index(form))
    for out in OUTS:
        _check(ops, x, w, gamma, beta, form, out)


@pytest.mark.parametrize('form', FORMS)
def test_fused_conv_gn_clamp_raises_the_overflow_flag(ops, form):
    x, w, gamma, beta = _case(2, 9, 40, 256, 5 + FORMS.index(form), gamma_scale=3.0e5)
    flag = _check(ops, x, w, gamma, beta, form, 'f16pair')
    assert int(flag) == 1, 'a GroupNorm output beyond 60000 must be clamped and flagged'


def _tower_modules(n, dev, seed):
    from pointtinybenchmark_b200.layers import ConvModule
    torch.manual_seed(seed)
    convs = torch.nn.ModuleList([ConvModule(256, 256, norm_cfg=dict(type='GN', num_groups=32)) for _ in range(n)]).to(dev)
    with torch.no_grad():
        for m in convs:
            m.conv.weight.normal_(0.0, 0.03)
            m.gn.weight.uniform_(0.5, 1.5)
            m.gn.bias.uniform_(-0.3, 0.3)
    return convs


def _unfused_tower(ops, convs, xm, want):
    """the explicit op sequence the tower ran before the fused launch: conv + statistics, then the apply kernel."""
    from pointtinybenchmark_b200.layers import _first_operands, _packed_weight_f16
    h, l, inv = _first_operands(xm)
    for i, m in enumerate(convs):
        wh, wl, inv_w = _packed_weight_f16(m)
        y, st = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, inv if i == 0 else None)
        ga, be = m.gn.weight.detach(), m.gn.bias.detach()
        if i == len(convs) - 1 and want == 'fp32':
            return ops.gn_relu_apply(y, st, ga, be, 32, m.gn.eps, True, split=False)
        h, l = ops.gn_relu_apply_f16(y, st, ga, be, 32, m.gn.eps, True, None)
    return h, l


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('want', ['f16pair', 'fp32'])
def test_tower_equals_the_unfused_sequence(ops, want, dtype):
    """layer by layer (each fused layer against conv + apply on its own y and statistics), then the whole tower against the explicit
    unfused sequence.  The statistics are fp64 atomic sums in a launch-dependent order; their float mean and rstd agree unless a
    last-bit difference crosses a float rounding boundary, which these inputs do not hit."""
    from pointtinybenchmark_b200.layers import _first_operands, _packed_weight_f16, tower
    dev = torch.device('cuda:0')
    convs = _tower_modules(4, dev, 3)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 256, 24, 40, generator=g).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    info = {}
    with torch.no_grad():
        res = tower(convs, x, info, want=want)
        assert info['backend'] == 'wgmma-f16x2'
        xm = ops.to_nhwc(x).contiguous()
        h, l, inv = _first_operands(xm)
        for i, m in enumerate(convs):
            wh, wl, inv_w = _packed_weight_f16(m)
            last = i == len(convs) - 1 and want == 'fp32'
            a, b, y, st = ops.conv3x3_c256_f16_gn(h, l, wh, wl, inv_w, inv if i == 0 else None, m.gn.weight.detach(),
                                                  m.gn.bias.detach(), m.gn.eps, None, out='fp32' if last else 'f16pair')
            y0, st0 = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, inv if i == 0 else None)
            _assert_bit_equal(y, y0, f'layer {i} y')
            if last:
                _assert_bit_equal(a, ops.gn_relu_apply(y, st, m.gn.weight.detach(), m.gn.bias.detach(), 32, m.gn.eps, True), 'tower output')
            else:
                h0, l0 = ops.gn_relu_apply_f16(y, st, m.gn.weight.detach(), m.gn.bias.detach(), 32, m.gn.eps, True, None)
                _assert_bit_equal(a, h0, f'layer {i} h')
                _assert_bit_equal(b, l0, f'layer {i} l')
            h, l = a, b
        # the tower itself against the explicit unfused sequence
        ref = _unfused_tower(ops, convs, xm, want)
        if want == 'fp32':
            _assert_bit_equal(res.permute(0, 2, 3, 1).contiguous(), ref, 'tower output vs unfused')
        else:
            _assert_bit_equal(res[0], ref[0], 'tower h vs unfused')
            _assert_bit_equal(res[1], ref[1], 'tower l vs unfused')


def test_training_forward_equals_the_unfused_sequence(ops):
    from pointtinybenchmark_b200.layers import tower
    dev = torch.device('cuda:0')
    convs = _tower_modules(4, dev, 4)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(2, 256, 17, 40, generator=g).to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    info = {}
    out = tower(convs, x, info, want='fp32')
    assert info['backend'] == 'wgmma-f16x2-train'
    with torch.no_grad():
        ref = _unfused_tower(ops, convs, ops.to_nhwc(x.detach()).contiguous(), 'fp32')
    _assert_bit_equal(out.detach().permute(0, 2, 3, 1).contiguous(), ref, 'training forward vs unfused')
    out.float().square().sum().backward()
    assert x.grad is not None and bool(torch.isfinite(x.grad).all())
    assert all(m.conv.weight.grad is not None and bool(torch.isfinite(m.conv.weight.grad).all()) for m in convs)
