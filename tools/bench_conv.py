"""timing of the wgmma 3xTF32 conv3x3 + GN + ReLU layer vs cuDNN fp32 / TF32 at the headline shape (scratch tool)."""
import os, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointtinybenchmark_b200 import ops

dev = torch.device('cuda:0')
torch.manual_seed(0)
B, H, W, C = 8, 100, 168, 256
x = torch.randn(B, C, H, W, device=dev).contiguous(memory_format=torch.channels_last)
conv = torch.nn.Conv2d(C, C, 3, padding=1, bias=False).to(dev).to(memory_format=torch.channels_last)
gn = torch.nn.GroupNorm(32, C).to(dev)
xh, xl = ops.split_tf32(ops.to_nhwc(x).contiguous())
wh, wl = ops.conv3x3_pack_weight(conv.weight)


def t(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for _ in range(n):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n


res = {}
flops = 2 * 9 * C * C * B * H * W
ms = t(lambda: ops.conv3x3_c256(xh, xl, wh, wl))
res['tc_conv_3xtf32'] = dict(ms=ms, eff_tflops=flops / ms / 1e9, tf32_tflops=3 * flops / ms / 1e9)
y, st = ops.conv3x3_c256(xh, xl, wh, wl)
res['gn_relu_apply_split'] = dict(ms=t(lambda: ops.gn_relu_apply(y, st, gn.weight.detach(), gn.bias.detach(), split=True)))
res['split_tf32'] = dict(ms=t(lambda: ops.split_tf32(ops.to_nhwc(x).contiguous())))
h16, l16, dinv = ops.split_f16(ops.to_nhwc(x).contiguous(), auto_scale=True)
wh16, wl16, invw = ops.conv3x3_pack_weight_f16(conv.weight)
ms = t(lambda: ops.conv3x3_c256_f16(h16, l16, wh16, wl16, invw, dinv))
res['tc_conv_f16x2'] = dict(ms=ms, eff_tflops=flops / ms / 1e9, f16_mma_tflops=3 * flops / ms / 1e9)
y16, st16 = ops.conv3x3_c256_f16(h16, l16, wh16, wl16, invw, dinv)
res['gn_relu_apply_f16'] = dict(ms=t(lambda: ops.gn_relu_apply_f16(y16, st16, gn.weight.detach(), gn.bias.detach())))
res['split_f16_autoscale'] = dict(ms=t(lambda: ops.split_f16(ops.to_nhwc(x).contiguous(), auto_scale=True)))
# training tower backward of one layer
da = torch.randn_like(y16)
res['gn_relu_bwd'] = dict(ms=t(lambda: ops.gn_relu_bwd(da, y16, st16, gn.weight.detach(), gn.bias.detach())))
dy, _, _, amax = ops.gn_relu_bwd(da, y16, st16, gn.weight.detach(), gn.bias.detach())
res['split_f16_amax'] = dict(ms=t(lambda: ops.split_f16_amax(dy, amax)))
dyh, dyl, inv_dy = ops.split_f16_amax(dy, amax)
ms = t(lambda: ops.conv_tc_wgrad_f16(dyh, dyl, h16, l16, 9, 1.0, inv_dy, dinv))
res['tc_wgrad_f16x2'] = dict(ms=ms, eff_tflops=flops / ms / 1e9, f16_mma_tflops=3 * flops / ms / 1e9)
wt = conv.weight.detach().flip(2, 3).transpose(0, 1).reshape(C, C, 9).contiguous()
pk = ops.conv_tc_pack_weight_f16(wt, 9)
ms = t(lambda: ops.conv_tc_f16(dyh, dyl, pk, 9, C, dev_out_scale=inv_dy))
res['tc_dgrad_f16x2'] = dict(ms=ms, eff_tflops=flops / ms / 1e9)
xg = x.clone().requires_grad_(True)
torch.backends.cudnn.allow_tf32 = False
def cudnn_bwd():
    conv.zero_grad(set_to_none=True)
    o = conv(xg)
    o.backward(da.permute(0, 3, 1, 2))
res['cudnn_fp32_conv_fwd_plus_bwd'] = dict(ms=t(cudnn_bwd, n=3))
torch.backends.cudnn.benchmark = True
for tf32 in (False, True):
    torch.backends.cudnn.allow_tf32 = tf32
    with torch.no_grad():
        ms = t(lambda: conv(x))
        res[f'cudnn_conv_tf32={tf32}'] = dict(ms=ms, tflops=flops / ms / 1e9)
        res[f'cudnn_conv_gn_relu_tf32={tf32}'] = dict(ms=t(lambda: torch.relu(gn(conv(x)))))
with torch.no_grad():
    torch.backends.cudnn.allow_tf32 = False
    ref = conv(x)
err = float((y.permute(0, 3, 1, 2) - ref).abs().max() / ref.abs().max())
res['max_rel_err_vs_cudnn_fp32'] = err
res['max_rel_err_f16x2_vs_cudnn_fp32'] = float((y16.permute(0, 3, 1, 2) - ref).abs().max() / ref.abs().max())
print(json.dumps(res, indent=1))
