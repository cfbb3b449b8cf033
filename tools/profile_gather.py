"""runs the neighbor-gather (C=256), the fused refine, the wgmma conv / GroupNorm kernels and one layer of the training tower's
backward (GroupNorm backward, split, wgrad, dgrad) a few times at the headline config: target for `ncu --set full`."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointtinybenchmark_b200 import ops

dev = torch.device('cuda:0')
torch.manual_seed(0)
B, H, W, C, n, r, s, ncls = 8, 100, 168, 256, 500, 8, 8, 80
feat = torch.relu(torch.randn(B, H, W, C, device=dev))
centers = (torch.rand(B * n, 2, device=dev) * torch.tensor([1344., 800.], device=dev)).contiguous()
bag_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(n).contiguous()
labels = torch.randint(0, ncls, (B * n,), device=dev, dtype=torch.int32)
pad_hw = torch.tensor([[800, 1344]] * B, dtype=torch.int32, device=dev)
img_hw = torch.tensor([[800, 1333]] * B, dtype=torch.int32, device=dev)
off = ops.circle_offsets(r, s).to(dev)
lmap = torch.randn(B, H, W, ncls, device=dev)
groups = ops.label_groups(bag_img, labels, ncls)
rc = ops._refine_cfg(0.1, 0.5, 0.1, True, True, False)
wc = torch.randn(ncls, C, device=dev) * 0.05
h16, l16, dinv = ops.split_f16(feat, auto_scale=True)
convw = torch.randn(256, C, 3, 3, device=dev) * 0.02
wh, wl, invw = ops.conv3x3_pack_weight_f16(convw)
bc = torch.zeros(ncls, device=dev)
y16, st16 = ops.conv3x3_c256_f16(h16, l16, wh, wl, invw, dinv)
gamma, beta = torch.rand(256, device=dev) + 0.5, torch.randn(256, device=dev) * 0.1
da = torch.randn_like(y16)
wt = convw.flip(2, 3).transpose(0, 1).reshape(256, 256, 9).contiguous()
packed_t = ops.conv_tc_pack_weight_f16(wt, 9)
for _ in range(int(sys.argv[1]) if len(sys.argv) > 1 else 3):
    ops.bag_gather(feat, centers, bag_img, off, s, pad_hw)
    ops.refine_fused(lmap, ncls, centers, labels, bag_img, off, s, pad_hw, img_hw, groups, rc)
    ops.linear_rows(feat.reshape(-1, C), wc, bc)
    ops.conv3x3_c256_f16(h16, l16, wh, wl, invw, dinv)
    ops.gn_relu_apply_f16(y16, st16, gamma, beta)
    # training tower backward of one layer
    dy, dg, db, amax = ops.gn_relu_bwd(da, y16, st16, gamma, beta)
    dyh, dyl, inv_dy = ops.split_f16_amax(dy, amax)
    ops.conv_tc_wgrad_f16(dyh, dyl, h16, l16, 9, 1.0, inv_dy, dinv)
    ops.conv_tc_f16(dyh, dyl, packed_t, 9, 256, dev_out_scale=inv_dy)
torch.cuda.synchronize()
