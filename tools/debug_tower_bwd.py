"""scratch: per-layer comparison of the tensor-core tower backward against fp64 autograd."""
import os, sys
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointtinybenchmark_b200 import ops
from tests.helpers import scale_rel_err as err

dev = torch.device('cuda:0')
torch.manual_seed(0)
B, H, W, C, G = 1, 32, 32, 256, 32
x = torch.randn(B, H, W, C, device=dev)
ws = [torch.randn(C, C, 3, 3, device=dev) * 0.02 for _ in range(4)]
gs = [torch.rand(C, device=dev) + 0.5 for _ in range(4)]
bs = [torch.randn(C, device=dev) * 0.1 for _ in range(4)]
dout = torch.randn(B, H, W, C, device=dev)
# fp64 reference with intermediates
xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
acts, ys = [xd], []
a = xd
for i in range(4):
    y = F.conv2d(a, ws[i].double(), None, 1, 1); y.retain_grad(); ys.append(y)
    a = F.relu(F.group_norm(y, G, gs[i].double(), bs[i].double(), 1e-5)); a.retain_grad(); acts.append(a)
a.backward(dout.double().permute(0, 3, 1, 2))
nhwc = lambda t: t.permute(0, 2, 3, 1)
# ours, step by step
h, l, dinv = ops.split_f16(x, auto_scale=True)
saved = []
for i in range(4):
    wh, wl, inv_w = ops.conv3x3_pack_weight_f16(ws[i])
    y, st = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, dinv if i == 0 else None)
    print(i, 'fwd y err', err(y, nhwc(ys[i])))
    saved.append((h, l, y, st))
    clones = globals().setdefault('clones', [])
    clones.append((y.clone(), st.clone(), h.clone(), l.clone()))
    if i < 3:
        h, l = ops.gn_relu_apply_f16(y, st, gs[i], bs[i], G, 1e-5, True, None)
    else:
        out = ops.gn_relu_apply(y, st, gs[i], bs[i], G, 1e-5, True, split=False)
print('out err', err(out, nhwc(acts[4])))
da = dout.contiguous()
def check(tag):
    torch.cuda.synchronize()
    for j in range(4):
        hh, ll, yy, ss = saved[j]
        cy, cs, ch, cl = clones[j]
        bad = [n for n, a, b in (('y', yy, cy), ('stats', ss, cs), ('h', hh, ch), ('l', ll, cl)) if not torch.equal(a, b)]
        if bad:
            print(f'   !! after {tag}: layer {j} saved tensors changed: {bad}', 'stats' in bad and (ss - cs).abs().max().item())
check('forward')
for i in reversed(range(4)):
    h, l, y, st = saved[i]
    dy, dg, db, amax = ops.gn_relu_bwd(da, y, st, gs[i], bs[i], G, 1e-5, True)
    check(f'gn_bwd[{i}]')
    print(i, 'dy err', err(dy, nhwc(ys[i].grad)), 'with ref da:', err(ops.gn_relu_bwd(nhwc(acts[i + 1].grad).float().contiguous(), y, st, gs[i], bs[i], G, 1e-5, True)[0], nhwc(ys[i].grad)))
    dyh, dyl, inv_dy = ops.split_f16_amax(dy, amax)
    check(f'split[{i}]')
    print('   pair err', err((dyh.float() + dyl.float()) * inv_dy, dy), 'amax', float(amax.view(torch.float32)), float(dy.abs().max()))
    wt = ws[i].flip(2, 3).transpose(0, 1).reshape(C, C, 9).contiguous()
    da = ops.conv_tc_f16(dyh, dyl, ops.conv_tc_pack_weight_f16(wt, 9), 9, C, dev_out_scale=inv_dy)
    check(f'dgrad[{i}]')
    print('   da err', err(da, nhwc(acts[i].grad)))
    dw = ops.conv_tc_wgrad_f16(dyh, dyl, h, l, 9, 1.0, inv_dy, dinv if i == 0 else None)
    check(f'wgrad[{i}]')
