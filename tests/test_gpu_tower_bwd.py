"""GPU: the tower's training path on the tensor cores — GroupNorm/ReLU backward, dgrad, wgmma wgrad (MN-major operands) and the
autograd function that chains them — against fp64 autograd on the same device and against the CPU oracle (oracle.cpr.tower_forward,
= the reference's ConvModule stack, cpr_head.py:983-995, 1033-1043)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import cpr as ocpr, synth
from tests.helpers import assert_close, oracle_cfg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def _stats(y, groups):
    B, H, W, C = y.shape
    yg = y.double().reshape(B, H * W, groups, C // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1).contiguous()      # (B, groups, 2)


@pytest.mark.parametrize('B,H,W', [(2, 9, 21), (1, 16, 16), (3, 5, 7)])
def test_gn_relu_bwd_matches_fp64_autograd(ops, B, H, W):
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cpu').manual_seed(B * 100 + H)
    C, groups = 256, 32
    y = (torch.randn(B, H, W, C, generator=g) * 2 + 0.3).to(dev)
    da = torch.randn(B, H, W, C, generator=g).to(dev)
    gamma = (torch.rand(C, generator=g) + 0.5).to(dev)
    beta = (torch.randn(C, generator=g) * 0.3).to(dev)
    dy, dg, db, amax = ops.gn_relu_bwd(da, y, _stats(y, groups), gamma, beta, groups, 1e-5, True)
    yd = y.double().permute(0, 3, 1, 2).requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = F.relu(F.group_norm(yd, groups, gd, bd, 1e-5))
    out.backward(da.double().permute(0, 3, 1, 2))
    assert_close(dy, yd.grad.permute(0, 2, 3, 1), 2e-5, 'dy')
    assert_close(dg, gd.grad, 2e-5, 'dgamma')
    assert_close(db, bd.grad, 2e-5, 'dbeta')
    assert float(torch.tensor([int(amax)], dtype=torch.int32).view(torch.float32)) == float(dy.abs().max())
    h, l, inv = ops.split_f16_amax(dy, amax)
    assert_close((h.float() + l.float()) * inv, dy, 1e-6, 'fp16 pair of dy')
    assert 2048 <= float(h.float().abs().max()) <= 4096


@pytest.mark.parametrize('B,H,W', [(2, 19, 37), (1, 8, 16), (8, 100, 168)])
def test_tc_wgrad_and_dgrad_match_fp64(ops, B, H, W):
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cpu').manual_seed(H)
    C = 256
    x = torch.randn(B, H, W, C, generator=g).to(dev) * 3
    dy = (torch.randn(B, H, W, C, generator=g) * 1e-3).to(dev)                # gradients are small: the device scale must cope
    w = (torch.randn(C, C, 3, 3, generator=g) * 0.02).to(dev)
    xh, xl, inv_x = ops.split_f16(x, auto_scale=True)
    amax = dy.abs().max().reshape(1).view(torch.int32)
    dh, dl, inv_dy = ops.split_f16_amax(dy, amax)
    dw = ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 9, 1.0, inv_dy, inv_x)
    wt = w.flip(2, 3).transpose(0, 1).reshape(C, C, 9).contiguous()
    dx = ops.conv_tc_f16(dh, dl, ops.conv_tc_pack_weight_f16(wt, 9), 9, C, dev_out_scale=inv_dy)
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wd = w.double().requires_grad_(True)
    F.conv2d(xd, wd, None, 1, 1).backward(dy.double().permute(0, 3, 1, 2))
    ref_dw, ref_dx = wd.grad, xd.grad.permute(0, 2, 3, 1)
    from tests.helpers import scale_rel_err
    print(f'[{B}x{H}x{W}] wgrad err {scale_rel_err(dw, ref_dw):.2e}, dgrad err {scale_rel_err(dx, ref_dx):.2e} (vs fp64)')
    if B * H * W > 4096:        # what the library's fp32 path achieves on the same sums, for scale
        xf = x.permute(0, 3, 1, 2).requires_grad_(True)
        wf = w.clone().requires_grad_(True)
        F.conv2d(xf, wf, None, 1, 1).backward(dy.permute(0, 3, 1, 2))
        print(f'    cuDNN fp32: wgrad err {scale_rel_err(wf.grad, ref_dw):.2e}, dgrad err {scale_rel_err(xf.grad.permute(0, 2, 3, 1), ref_dx):.2e}')
    e1 = assert_close(dw, ref_dw, 5e-5, 'dW (wgmma wgrad, MN-major operands)')
    e2 = assert_close(dx, ref_dx, 2e-5, 'dX (forward kernel on W^T flipped)')
    dw2 = ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 9, 1.0, inv_dy, inv_x, out=dw.clone(), accumulate=True)
    assert_close(dw2, 2 * ref_dw, 5e-5, 'accumulate')
    assert torch.equal(ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 9, 1.0, inv_dy, inv_x), dw), 'deterministic'


def _tower_modules(weights, dev, dtype):
    from pointtinybenchmark_b200.layers import ConvModule
    convs = torch.nn.ModuleList([ConvModule(256, 256, 3, 1, 1, norm_cfg=dict(type='GN', num_groups=32)) for _ in range(4)]).to(dev)
    sd = {k[len('cls_convs.'):]: v for k, v in weights.items() if k.startswith('cls_convs.')}
    convs.load_state_dict(sd, strict=True)
    return convs.to(dtype)


def _frac_outliers(a, b, tol):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    scale = torch.clamp(b.abs(), min=float(b.pow(2).mean().sqrt()))
    return float(((a - b).abs() > tol * scale).double().mean())


def test_tower_training_path_vs_fp64_and_oracle(ops):
    """The whole autograd function.  ReLU'(0) is discontinuous: two implementations whose pre-activations differ by 1e-6 flip the
    mask of the few elements with |z| < 1e-6, and each flip is an O(1) change of that element's gradient (any two fp32 conv
    implementations differ like this, cuDNN vs the CPU included).  So (1) the strict max-norm comparison is done against an fp64
    network whose ReLU masks are FIXED to the ones our own forward kernels produce, and (2) against the true-ReLU fp64 network and
    the CPU oracle (= the reference's arithmetic) the statement is: all but a vanishing fraction of elements agree to 2e-4."""
    from pointtinybenchmark_b200.layers import tower
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 99, with_towers=True)
    cfg = oracle_cfg(inp['cfgd'])
    w = inp['weights']
    x0 = inp['cls_feat']
    g = torch.Generator().manual_seed(3)
    dout = torch.randn(x0.shape[0], 256, x0.shape[2], x0.shape[3], generator=g)
    # ours
    convs = _tower_modules(w, dev, torch.float32)
    x = x0.to(dev).requires_grad_(True)
    info = {}
    out = tower(convs, x, info)
    assert info['backend'] == 'wgmma-f16x2-train', info
    out.backward(dout.to(dev))
    # ReLU masks of our forward kernels (inference entry points, same arithmetic)
    masks = []
    with torch.no_grad():
        h, l, dinv = ops.split_f16(ops.to_nhwc(x0.to(dev)).contiguous(), auto_scale=True)
        for i, m in enumerate(convs):
            wh, wl, inv_w = ops.conv3x3_pack_weight_f16(m.conv.weight)
            y, st = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, dinv if i == 0 else None)
            masks.append(ops.gn_relu_apply(y, st, m.gn.weight, m.gn.bias, 32, m.gn.eps, True, split=False).permute(0, 3, 1, 2) > 0)
            h, l = ops.gn_relu_apply_f16(y, st, m.gn.weight, m.gn.bias, 32, m.gn.eps, True, None)
    # fp64 on the device: (a) masks fixed to ours, (b) true ReLU
    refs = {}
    for kind in ('fixed-mask', 'relu'):
        c64 = _tower_modules(w, dev, torch.float64)
        x64 = x0.to(dev).double().requires_grad_(True)
        o = x64
        for i, m in enumerate(c64):
            z = m.gn(m.conv(o))
            o = z * masks[i].double() if kind == 'fixed-mask' else F.relu(z)
        o.backward(dout.to(dev).double())
        refs[kind] = (o, x64, c64)
    o64, x64, c64 = refs['fixed-mask']
    assert_close(out, o64, 5e-5, 'tower output vs fp64')
    e = assert_close(x.grad, x64.grad, 1e-4, 'dX vs fp64 (fixed masks)')
    errs = []
    for i, (m, m64) in enumerate(zip(convs, c64)):
        errs.append(assert_close(m.conv.weight.grad, m64.conv.weight.grad, 1e-4, f'dW[{i}] vs fp64 (fixed masks)'))
        assert_close(m.gn.weight.grad, m64.gn.weight.grad, 1e-4, f'dgamma[{i}] vs fp64 (fixed masks)')
        assert_close(m.gn.bias.grad, m64.gn.bias.grad, 1e-4, f'dbeta[{i}] vs fp64 (fixed masks)')
    print(f'tower training path (fixed masks): dX err {e:.1e}, dW errs {[f"{v:.1e}" for v in errs]}')
    # true ReLU: fp64 on the device and the CPU oracle
    _, x64r, c64r = refs['relu']
    xo = x0.clone().requires_grad_(True)
    wo = {k: v.clone().requires_grad_(True) for k, v in w.items() if k.startswith('cls_convs.')}
    oo = ocpr.tower_forward(xo, wo, cfg)
    oo.backward(dout)
    assert_close(out, oo, 1e-4, 'tower output vs oracle')
    # Our forward is exact to ~1e-5 (two-term fp16 operands), the CPU's to ~1e-7: a handful of |z| < 1e-5 elements per layer get the
    # other ReLU branch, and GroupNorm's backward spreads each flip over its whole (image, group) at relative size 1/n.  The
    # gradients therefore agree with the true-ReLU references in the L2 sense (a perturbed-network statement), not element-wise.
    def l2(a, b):
        a, b = a.detach().double().cpu(), b.detach().double().cpu()
        return float((a - b).norm() / b.norm())
    rows = [('dX', x.grad, x64r.grad, xo.grad)]
    for i, m in enumerate(convs):
        rows.append((f'dW[{i}]', m.conv.weight.grad, c64r[i].conv.weight.grad, wo[f'cls_convs.{i}.conv.weight'].grad))
        rows.append((f'dgamma[{i}]', m.gn.weight.grad, c64r[i].gn.weight.grad, wo[f'cls_convs.{i}.gn.weight'].grad))
    worst = 0.0
    for name, mine, r64, ror in rows:
        e64, eor = l2(mine, r64), l2(mine, ror)
        worst = max(worst, e64, eor)
        print(f'true ReLU {name}: rel-L2 vs fp64 {e64:.1e}, vs CPU oracle {eor:.1e}; outliers(>2e-4) {_frac_outliers(mine, r64, 2e-4):.1e}')
    print(f'CPU fp32 oracle vs fp64, dX rel-L2: {l2(xo.grad, x64r.grad):.1e}')
    assert worst < 1e-2, worst


@pytest.mark.parametrize('B,H,W,Cout', [(2, 13, 21, 160), (1, 100, 168, 160), (1, 9, 16, 80)])
def test_one_tap_wgrad_and_col_sum_match_fp64(ops, B, H, W, Cout):
    """dW / db of the logit-map Linear (cls_out | ins_out stacked, cpr_head.py:1045-1078 under autograd) on the tensor cores:
    ptb_conv_tc_wgrad_f16x2_ld with taps = 1 (K = pixels) and ptb_col_sum against float64, plus run-to-run bit equality."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 100 + Cout)
    x = torch.relu(torch.randn(B, H, W, 256, generator=g)).to(dev)
    dy = (torch.randn(B, H, W, Cout, generator=g) * 1e-4).to(dev)
    xh, xl, xinv = ops.split_f16(x, auto_scale=True)
    dh, dl, dinv = ops.split_f16(dy, auto_scale=True)
    dw = ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 1, 1.0, dinv, xinv)
    ref = dy.double().reshape(-1, Cout).t() @ x.double().reshape(-1, 256)
    e = assert_close(dw, ref, 1e-4, '1-tap wgrad vs fp64')
    db = ops.col_sum(dy.reshape(-1, Cout))
    assert_close(db, dy.double().reshape(-1, Cout).sum(0), 1e-5, 'col_sum vs fp64')
    dw2 = ops.conv_tc_wgrad_f16(dh, dl, xh, xl, 1, 1.0, dinv, xinv)
    assert torch.equal(dw, dw2) and torch.equal(db, ops.col_sum(dy.reshape(-1, Cout))), 'deterministic'
    print(f'[1-tap wgrad {B}x{H}x{W}x{Cout}] err vs fp64 {e:.1e}')
