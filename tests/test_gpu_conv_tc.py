"""GPU parity of the wgmma 3xTF32 conv3x3 + GroupNorm + ReLU tower against fp32 references (oracle.tower_forward on the CPU
and cuDNN fp32 on the GPU); tolerance 1e-4 scale-relative like every other float output of the head."""
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


@pytest.mark.parametrize('B,H,W,Cin', [(1, 8, 16, 32), (1, 16, 32, 256), (2, 13, 21, 256), (1, 100, 168, 256), (3, 7, 5, 64)])
def test_conv3x3_tf32x3_matches_fp32(ops, B, H, W, Cin):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 100 + H)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(256, Cin, 3, 3, generator=g) * (1.4 / (Cin * 9) ** 0.5)
    ref = F.conv2d(x.double(), w.double(), None, 1, 1).float()            # fp64 truth
    xh, xl = ops.split_tf32(ops.to_nhwc(x.to(dev)).contiguous())
    assert torch.equal(xh + xl, ops.to_nhwc(x.to(dev)))                  # the split is exact
    wh, wl = ops.conv3x3_pack_weight(w.to(dev))
    y, stats = ops.conv3x3_c256(xh, xl, wh, wl)
    got = y.permute(0, 3, 1, 2)
    e = assert_close(got, ref, 5e-5, f'conv3x3 3xTF32 ({B},{H},{W},{Cin})')
    e32 = float((F.conv2d(x, w, None, 1, 1) - ref).abs().max() / ref.abs().max())
    print(f'[{B}x{H}x{W}x{Cin}] 3xTF32 err {e:.2e} (plain fp32 CPU conv err {e32:.2e})')
    # GroupNorm statistics accumulated by the epilogue
    yr = ref.double().reshape(B, 32, 8, H * W)
    assert_close(stats[..., 0], yr.sum((2, 3)), 1e-4, 'GN sum')
    assert_close(stats[..., 1], (yr * yr).sum((2, 3)), 1e-4, 'GN sum of squares')
    gamma = 1 + 0.1 * torch.randn(256, generator=g)
    beta = 0.1 * torch.randn(256, generator=g)
    out = ops.gn_relu_apply(y, stats, gamma.to(dev), beta.to(dev))
    refo = F.relu(F.group_norm(ref, 32, gamma, beta))
    assert_close(out.permute(0, 3, 1, 2), refo, 1e-4, 'GN + ReLU')
    oh, ol = ops.gn_relu_apply(y, stats, gamma.to(dev), beta.to(dev), split=True)
    assert torch.equal(oh + ol, out)
    assert int((oh.view(torch.int32) & 0x1FFF).abs().max()) == 0          # hi is an exact TF32 value


def test_tower_matches_oracle_and_golden(ops, golden_dir):
    import os
    import numpy as np
    from pointtinybenchmark_b200 import cpr_head  # noqa
    from pointtinybenchmark_b200.registry import build_head
    from tests.test_gpu_cpr_head import head_cfg
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 99, with_towers=True)
    cfg = oracle_cfg(inp['cfgd'])
    head = build_head(head_cfg(inp['cfgd'])).to(dev).eval()
    sd = head.state_dict(); sd.update(inp['weights']); head.load_state_dict(sd)
    with torch.no_grad():
        out = head([inp['cls_feat'].to(dev)])[0][0]
        ref = ocpr.tower_forward(inp['cls_feat'], inp['weights'], cfg)
    assert head.last_tower_backend in ('wgmma-3xtf32', 'wgmma-f16x2')
    assert_close(out, ref, 1e-4, 'tower (wgmma 3xTF32) vs oracle')
    gold = np.load(os.path.join(golden_dir, 'cpr_lite_tower.npz'))
    sub = out.cpu().contiguous().flatten()[::97].numpy()
    assert np.abs(sub - gold['tower_sub']).max() <= 1e-4 * np.abs(gold['tower_sub']).max()
    # the autograd (training) path: tensor-core autograd function for the shipped geometry; must agree with the inference path, and
    # so must the explicit library path (PTB_TOWER_TRAIN=cudnn: cuDNN fp32 with TF32 switched off locally)
    x = inp['cls_feat'].to(dev).requires_grad_(True)
    out_train = head([x])[0][0]
    assert head.last_tower_backend == 'wgmma-f16x2-train'
    assert out_train.requires_grad
    assert_close(out_train, out, 1e-5, 'tensor-core training path vs inference path')
    old = os.environ.get('PTB_TOWER_TRAIN')
    os.environ['PTB_TOWER_TRAIN'] = 'cudnn'
    try:
        out_lib = head([x])[0][0]
        assert head.last_tower_backend == 'cudnn'
    finally:
        if old is None:
            del os.environ['PTB_TOWER_TRAIN']
        else:
            os.environ['PTB_TOWER_TRAIN'] = old
    assert_close(out_lib, out, 1e-4, 'cuDNN training path vs wgmma inference path')


def test_conv_is_bit_identical_across_processes():
    """two processes running the same 3xTF32 conv3x3 give the same bits (the MMA accumulation order is fixed)."""
    import os, subprocess, sys
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    code = (
        "import torch, sys; sys.path.insert(0, %r)\n"
        "from pointtinybenchmark_b200 import ops\n"
        "g = torch.Generator().manual_seed(3)\n"
        "x = torch.randn(2, 21, 37, 64, generator=g).cuda(); w = (torch.randn(256, 64, 3, 3, generator=g) * 0.05).cuda()\n"
        "xh, xl = ops.split_tf32(x); wh, wl = ops.conv3x3_pack_weight(w)\n"
        "y, st = ops.conv3x3_c256(xh, xl, wh, wl); print(float(y.double().sum()), float(y.abs().double().sum()), round(float(st.sum()), 3))\n"
    ).replace('%r', repr(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    outs = []
    for _ in range(2):
        r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-1500:]
        outs.append(r.stdout.strip().splitlines()[-1])
    assert outs[0] == outs[1], outs


@pytest.mark.parametrize('B,H,W,Cin,xs', [(1, 8, 16, 32, 1.0), (2, 13, 21, 256, 1.0), (1, 100, 168, 256, 1.0), (1, 16, 32, 64, 3000.0),
                                          (1, 16, 32, 64, 1e-3)])
def test_conv3x3_f16x2_matches_fp32(ops, B, H, W, Cin, xs):
    """two-term fp16 split: same fp32-level accuracy as 3xTF32, also for inputs far outside fp16's comfortable range (xs)."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(B * 100 + H + Cin)
    x = torch.randn(B, Cin, H, W, generator=g) * xs
    w = torch.randn(256, Cin, 3, 3, generator=g) * (1.4 / (Cin * 9) ** 0.5)
    ref = F.conv2d(x.double(), w.double(), None, 1, 1).float()
    h, l, dev_inv = ops.split_f16(ops.to_nhwc(x.to(dev)).contiguous(), auto_scale=True)
    wh, wl, inv_w = ops.conv3x3_pack_weight_f16(w.to(dev))
    y, stats = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, dev_inv)
    e = assert_close(y.permute(0, 3, 1, 2), ref, 5e-5, f'conv3x3 fp16x2 ({B},{H},{W},{Cin}, x*{xs})')
    print(f'[{B}x{H}x{W}x{Cin} x{xs}] fp16x2 err {e:.2e}')
    yr = ref.double().reshape(B, 32, 8, H * W)
    assert_close(stats[..., 0], yr.sum((2, 3)), 1e-4, 'GN sum')
    gamma = 1 + 0.1 * torch.randn(256, generator=g)
    beta = 0.1 * torch.randn(256, generator=g)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    oh, ol = ops.gn_relu_apply_f16(y, stats, gamma.to(dev), beta.to(dev), overflow_flag=flag)
    refo = F.relu(F.group_norm(ref, 32, gamma, beta))
    assert_close((oh.float() + ol.float()).permute(0, 3, 1, 2), refo, 1e-4, 'GN + ReLU as fp16 pair')
    assert int(flag) == 0


def test_general_tc_conv_linear_and_biased_conv(ops):
    """ptb_conv_tc_f16x2: 1 tap (per-cell Linear, N=80 / 160) and 9 taps with bias and small N (P2P cls_out / reg_out)."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(17)
    B, H, W, C = 2, 19, 27, 256
    x = torch.relu(torch.randn(B, C, H, W, generator=g))
    h, l, dinv = ops.split_f16(ops.to_nhwc(x.to(dev)).contiguous(), auto_scale=True)
    for n_out in (80, 160, 1, 20):
        w = torch.randn(n_out, C, generator=g) * 0.05
        b = torch.randn(n_out, generator=g)
        ref = F.linear(x.permute(0, 2, 3, 1).double(), w.double(), b.double()).float()
        y = ops.conv_tc_f16(h, l, ops.conv_tc_pack_weight_f16(w.to(dev), 1), 1, n_out, bias=b.to(dev), dev_out_scale=dinv)
        assert_close(y[..., :n_out], ref, 2e-5, f'tc linear N={n_out}')
    for n_out in (80, 2, 8):
        w = torch.randn(n_out, C, 3, 3, generator=g) * 0.02
        b = torch.randn(n_out, generator=g)
        ref = F.conv2d(x.double(), w.double(), b.double(), 1, 1).float()
        packed = ops.conv_tc_pack_weight_f16(w.reshape(n_out, C, 9).to(dev), 9)
        y = ops.conv_tc_f16(h, l, packed, 9, n_out, bias=b.to(dev), dev_out_scale=dinv)
        assert_close(y[..., :n_out].permute(0, 3, 1, 2), ref, 2e-5, f'tc conv3x3+bias N={n_out}')


def test_heads_fast_paths_match_oracle(ops, golden_dir):
    """CPRHead.simple_test (towers -> fp16 pair -> tensor-core logit map -> fused refine) and P2PHead.forward (towers + output
    convs on wgmma) against the CPU oracle."""
    from oracle import p2p as op2p
    from pointtinybenchmark_b200 import cpr_head, p2p_head  # noqa
    from pointtinybenchmark_b200.registry import build_head
    from tests.test_gpu_cpr_head import head_cfg
    from tests.test_gpu_p2p import head_cfg as p2p_cfg
    dev = torch.device('cuda:0')
    inp = synth.cpr_inputs('lite', 99, with_towers=True)
    cfg = oracle_cfg(inp['cfgd'])
    head = build_head(head_cfg(inp['cfgd'])).to(dev).eval()
    sd = head.state_dict(); sd.update(inp['weights']); head.load_state_dict(sd)
    gtb = [b.to(dev) for b in inp['gt_bboxes']]; gtl = [l.to(dev) for l in inp['gt_labels']]; aid = [a.to(dev) for a in inp['gt_anns_id']]
    with torch.no_grad():
        res = head.simple_test((inp['cls_feat'].to(dev),), inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
        slow = head.get_bboxes(*head.forward((inp['cls_feat'].to(dev),)), inp['img_metas'], gt_bboxes=gtb, gt_labels=gtl, gt_anns_id=aid)
        feat = ocpr.tower_forward(inp['cls_feat'], inp['weights'], cfg)
    ora = ocpr.cpr_get_bboxes(feat, inp['weights'], inp['gt_bboxes'], inp['gt_labels'], inp['gt_anns_id'], inp['img_metas'], cfg)
    assert_close(res[0][0][:, :5], ora[0][0][:, :5], 1e-4, 'simple_test fast path vs oracle')
    assert_close(res[0][0][:, :5], slow[0][0][:, :5], 1e-4, 'fast path vs forward+get_bboxes')
    # ---- P2P forward
    g = torch.Generator().manual_seed(8)
    d = dict(num_classes=80, C=256, stride=8)
    ph = build_head(p2p_cfg(d)).to(dev).eval()
    with torch.no_grad():
        for m in ph.modules():
            if isinstance(m, torch.nn.Conv2d):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.2 / (m.weight[0].numel()) ** 0.5))
    w = {k: v.detach().cpu() for k, v in ph.state_dict().items()}
    x = torch.randn(2, 256, 24, 40, generator=g)
    pc = op2p.default_cfg(num_classes=80, stride=8)
    with torch.no_grad():
        co, po = ph.forward((x.to(dev),))
        rco, rpo = op2p.head_forward(x, w, pc)
    assert ph.last_tower_backend == 'wgmma-f16x2'
    assert_close(co[0], rco, 1e-4, 'P2P cls_out (wgmma) vs oracle')
    assert_close(po[0], rpo, 1e-4, 'P2P pts_out (wgmma) vs oracle')


def test_stale_packed_weights_are_dropped_by_eval_and_invalidate(ops):
    """ADVICE r1: a `.data` write does not bump Tensor._version; eval() / train() / load_state_dict / invalidate_packed() drop the cached
    tensor-core packings, so the next forward sees the new weights."""
    from pointtinybenchmark_b200 import cpr_head  # noqa: F401
    from pointtinybenchmark_b200.registry import build_head
    from tests.test_gpu_cpr_head import head_cfg
    d = dict(num_classes=80, C=256, stride=8, radius=5)
    head = build_head(head_cfg(d)).cuda().eval()
    x = torch.randn(1, 256, 16, 24, generator=torch.Generator().manual_seed(1)).cuda()
    with torch.no_grad():
        y0 = head((x,))[0][0].clone()
        w = head.cls_convs[0].conv.weight
        v0 = w._version
        w.data.mul_(-1.0)                               # EMA-swap style write: the version does not move
        assert w._version == v0
        y_stale = head((x,))[0][0].clone()
        head.eval()                                     # drops the packs
        y1 = head((x,))[0][0].clone()
        w.data.mul_(-1.0)
        head.invalidate_packed()
        y2 = head((x,))[0][0].clone()
    assert head.last_tower_backend == 'wgmma-f16x2'
    assert torch.equal(y_stale, y0), 'documented hazard: without invalidation the stale pack is used'
    assert not torch.equal(y1, y0), 'eval() must make the new weights visible'
    assert torch.equal(y2, y0), 'invalidate_packed() after restoring the weights gives the original output back'
    # FCOS: conv_centerness runs in the same launch as conv_cls, from one packing of both
    from pointtinybenchmark_b200.fcos_head import FCOSHead
    fcos = FCOSHead(num_classes=4, in_channels=256, strides=(8,), regress_ranges=((-1, 1e8),)).cuda().eval()
    with torch.no_grad():
        c0 = fcos((x,))[2][0].clone()
        fcos.conv_centerness.weight.data.mul_(-1.0)
        c_stale = fcos((x,))[2][0].clone()
        fcos.eval()
        c1 = fcos((x,))[2][0].clone()
        fcos.conv_centerness.weight.data.mul_(-1.0)
        fcos.invalidate_packed()
        c2 = fcos((x,))[2][0].clone()
    assert fcos.last_tower_backend == 'wgmma-f16x2'
    assert torch.equal(c_stale, c0), 'documented hazard: without invalidation the stale pack is used'
    assert not torch.equal(c1, c0), 'eval() must make the new centerness weights visible'
    assert torch.equal(c2, c0), 'invalidate_packed() after restoring the weights gives the original output back'
