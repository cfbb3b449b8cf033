"""GPU parity of the wgmma conv at the map shapes where its activation box (tile h + 2 rows: one box serves the three vertical taps of a
column offset) reaches past the image: maps shorter than the box, a one-row bottom strip, a one-column right strip, an odd tile count.
Same float64 references and tolerances as tests/test_gpu_conv_tc.py."""
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

# (B, H, W, Cin): H = 1, 2, 3 (shorter than every box; bottom-strip tiles only), H = 5 (one 8 x 16 tile row, box 10 rows), a one-row
# bottom strip (H % 8 == 1) next to a right strip, a one-column right strip (W % 16 == 1), odd tile counts (3 x 3 and 3 x 1 tiles)
EDGE_SHAPES = [(1, 1, 40, 64), (2, 2, 16, 32), (1, 3, 33, 256), (1, 5, 23, 64), (1, 17, 40, 64), (2, 9, 16, 256), (1, 16, 33, 64),
               (1, 24, 17, 32), (1, 24, 48, 64), (3, 8, 16, 32)]


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def _inputs(B, H, W, Cin, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(256, Cin, 3, 3, generator=g) * (1.4 / (Cin * 9) ** 0.5)
    return x, w, F.conv2d(x.double(), w.double(), None, 1, 1)


def _check_stats(stats, ref, B, H, W):
    yr = ref.reshape(B, 32, 8, H * W)
    assert_close(stats[..., 0], yr.sum((2, 3)), 1e-4, 'GN sum')
    assert_close(stats[..., 1], (yr * yr).sum((2, 3)), 1e-4, 'GN sum of squares')


@pytest.mark.parametrize('B,H,W,Cin', EDGE_SHAPES)
def test_conv3x3_f16x2_box_edges(ops, B, H, W, Cin):
    dev = torch.device('cuda:0')
    x, w, ref = _inputs(B, H, W, Cin, 1000 + B * 100 + H * 7 + W)
    h, l, dev_inv = ops.split_f16(ops.to_nhwc(x.to(dev)).contiguous(), auto_scale=True)
    wh, wl, inv_w = ops.conv3x3_pack_weight_f16(w.to(dev))
    y, stats = ops.conv3x3_c256_f16(h, l, wh, wl, inv_w, dev_inv)
    assert_close(y.permute(0, 3, 1, 2), ref.float(), 5e-5, f'conv3x3 fp16x2 ({B},{H},{W},{Cin})')
    _check_stats(stats, ref, B, H, W)


@pytest.mark.parametrize('B,H,W,Cin', EDGE_SHAPES)
def test_conv3x3_tf32x3_box_edges(ops, B, H, W, Cin):
    dev = torch.device('cuda:0')
    x, w, ref = _inputs(B, H, W, Cin, 2000 + B * 100 + H * 7 + W)
    xh, xl = ops.split_tf32(ops.to_nhwc(x.to(dev)).contiguous())
    wh, wl = ops.conv3x3_pack_weight(w.to(dev))
    y, stats = ops.conv3x3_c256(xh, xl, wh, wl)
    assert_close(y.permute(0, 3, 1, 2), ref.float(), 5e-5, f'conv3x3 3xTF32 ({B},{H},{W},{Cin})')
    _check_stats(stats, ref, B, H, W)


@pytest.mark.parametrize('B,H,W', [(1, 1, 40), (1, 17, 40), (1, 16, 33), (3, 8, 16)])
@pytest.mark.parametrize('taps,n_out', [(9, 320), (9, 20), (1, 80)])
def test_general_tc_conv_box_edges(ops, B, H, W, taps, n_out):
    """ptb_conv_tc_f16x2 at the same edges: 9 taps over several channel slices (320 = P2P cls_out) and one narrow slice, and the
    1-tap Linear, whose box is the tile itself."""
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(3000 + B * 100 + H * 7 + W + taps + n_out)
    C = 256
    x = torch.relu(torch.randn(B, C, H, W, generator=g))
    h, l, dinv = ops.split_f16(ops.to_nhwc(x.to(dev)).contiguous(), auto_scale=True)
    b = torch.randn(n_out, generator=g)
    if taps == 9:
        w = torch.randn(n_out, C, 3, 3, generator=g) * 0.02
        ref = F.conv2d(x.double(), w.double(), b.double(), 1, 1).permute(0, 2, 3, 1)
        packed = ops.conv_tc_pack_weight_f16(w.reshape(n_out, C, 9).to(dev), 9)
    else:
        w = torch.randn(n_out, C, generator=g) * 0.05
        ref = F.linear(x.permute(0, 2, 3, 1).double(), w.double(), b.double())
        packed = ops.conv_tc_pack_weight_f16(w.to(dev), 1)
    y = ops.conv_tc_f16(h, l, packed, taps, n_out, bias=b.to(dev), dev_out_scale=dinv)
    assert_close(y[..., :n_out], ref.float(), 2e-5, f'tc conv taps={taps} N={n_out} ({B},{H},{W})')
