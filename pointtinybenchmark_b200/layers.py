"""Host-side layer containers with the reference's parameter names (checkpoint compatibility, SURVEY.md §5).

Conv towers (SURVEY.md §8f rank 1): at inference they run on the hand-written wgmma implicit-GEMM kernel of csrc/conv_tc.cu
(fp16 two-term split by default, 3xTF32 with PTB_CONV_MODE=tf32x3; both fp32-accurate); under autograd (training) the shipped
256 -> 256 geometry runs `_TowerTCFn`: the same forward kernel plus hand-written GroupNorm/ReLU backward, dgrad (the forward
kernel on transposed, flipped weights) and a wgmma wgrad with MN-major operands.  Other geometries (or PTB_TOWER_TRAIN=cudnn)
use cuDNN fp32 through torch with TF32 switched off locally (library path).

Input dtype: fp32, or the fp16 / bf16 feature map of a backbone under torch.autocast, taken as it is (`input_plan`): an fp16 tensor is
the first conv's hi operand itself, a bf16 tensor is split from its 2-byte storage, and the input gradient comes back in that dtype.
Everything after the first conv, parameters and outputs stay fp32.
"""
import contextlib
import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F


class ConvModule(nn.Module):
    """conv3x3 (bias iff no norm) -> GN/BN -> ReLU with mmcv.cnn.ConvModule's submodule names (`conv`, `gn`|`bn`)."""

    def __init__(self, cin, cout, k=3, stride=1, padding=1, norm_cfg=None, bias='auto', act=True):
        super().__init__()
        with_norm = norm_cfg is not None
        if bias == 'auto':
            bias = not with_norm
        self.conv = nn.Conv2d(cin, cout, k, stride, padding, bias=bias)
        self.norm_name = None
        if with_norm:
            t = norm_cfg['type']
            if t == 'GN':
                self.norm_name = 'gn'
                self.add_module('gn', nn.GroupNorm(norm_cfg['num_groups'], cout))
            elif t in ('BN', 'SyncBN'):
                self.norm_name = 'bn'
                self.add_module('bn', nn.BatchNorm2d(cout))
            else:
                raise NotImplementedError(f'norm type {t}')
        self.with_act = act

    def forward(self, x):
        x = self.conv(x)
        if self.norm_name is not None:
            x = getattr(self, self.norm_name)(x)
        return F.relu(x) if self.with_act else x


def normal_init_(module, std=0.01, bias=0.0):
    nn.init.normal_(module.weight, 0.0, std)
    if getattr(module, 'bias', None) is not None:
        nn.init.constant_(module.bias, bias)


def bias_init_with_prob(p):
    return float(-math.log((1 - p) / p))


_PACK_ATTRS = ('_ptb_packs',)      # the one attribute cached_pack keeps a module's packings in


def invalidate_packed(module):
    """drop every cached tensor-core packing of `module`'s weights (`cached_pack`).  The caches are keyed on (data_ptr, Tensor._version,
    device); in-place writes through `.data` (mmcv's EMAHook swap, manual weight surgery) do NOT bump `_version`, so the heads call this
    from train() / eval() and after load_state_dict, and anything else that writes `.data` must call it explicitly (`.data` writes are
    otherwise unsupported: the packed copy would go stale).  Costs nothing when there is no cache."""
    for m in module.modules():
        for a in _PACK_ATTRS:
            if hasattr(m, a):
                delattr(m, a)


def cached_pack(module, name, tensors, make):
    """make(), kept in `module`'s one dict of packings under `name` until a tensor of `tensors` is replaced (data_ptr), written in
    place (Tensor._version) or moved to another device.  Every packing of a head's weights goes through here, so that
    invalidate_packed drops them all."""
    key = tuple((t.data_ptr(), t._version) for t in tensors) + (str(tensors[0].device),)
    packs = getattr(module, _PACK_ATTRS[0], None)
    if packs is None:
        packs = {}
        setattr(module, _PACK_ATTRS[0], packs)
    hit = packs.get(name)
    if hit is None or hit[0] != key:
        hit = packs[name] = (key, make())
    return hit[1]


class PackedWeightsMixin:
    """nn.Module mixin of the heads: packed-weight caches are invalidated on train() / eval() and after load_state_dict."""

    def _init_packed_hooks(self):
        self.register_load_state_dict_post_hook(lambda mod, incompatible_keys: invalidate_packed(mod))

    def train(self, mode=True):
        invalidate_packed(self)
        return super().train(mode)

    def invalidate_packed(self):
        invalidate_packed(self)

    def _record_tower(self, info):
        """what the last tower() call ran (its `info`): backend, input path and, on wgmma-f16x2, the fp16-overflow flag"""
        self.last_tower_backend, self.last_input_path, self.last_overflow_flag = \
            info.get('backend'), info.get('input_path'), info.get('overflow_flag')


@contextlib.contextmanager
def no_tf32():
    """cuDNN convolutions and cuBLAS matmuls in full fp32 inside the block, whatever the global TF32 flags say (the heads' float
    outputs must match the fp32 reference to 1e-4); the other cuDNN flags stay as they are."""
    matmul_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=torch.backends.cudnn.benchmark,
                                        deterministic=torch.backends.cudnn.deterministic, allow_tf32=False):
            yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = matmul_tf32


HALF_INPUT_DTYPES = (torch.float16, torch.bfloat16)
_INPUT_DTYPES = (torch.float32,) + HALF_INPUT_DTYPES


def input_plan(dtype, conv_mode='f16x2'):
    """How a tower takes an input of `dtype` with PTB_CONV_MODE = conv_mode: (input_path, first conv, dtype of the input gradient), a
    pure function decided on the host (no device flag is read).  None for a dtype the tensor-core towers do not take.
      fp32  'fp32-split'   the (hi, lo) pair from ptb_split_f16 (or the TF32 pair)    conv 'f16x2' | 'tf32x3'
      fp16  'fp16-direct'  hi is the tensor's own storage, lo == 0, scale 1           conv 'f16x1a' (no lo MMA, no lo loads)
      bf16  'bf16-split'   the pair from ptb_split_f16_from_bf16 (2 B / element)      conv 'f16x2'
    Only the first conv of a tower differs: later layers consume fp32 GroupNorm outputs."""
    if dtype == torch.float32:
        return 'fp32-split', 'f16x2' if conv_mode == 'f16x2' else 'tf32x3', torch.float32
    if dtype in HALF_INPUT_DTYPES:
        if conv_mode != 'f16x2':
            raise NotImplementedError(f'PTB_CONV_MODE={conv_mode}: {dtype} feature maps are taken by the fp16-split mode only '
                                      '(PTB_CONV_MODE=f16x2, the default); convert the input to fp32 for this mode')
        return ('fp16-direct', 'f16x1a', dtype) if dtype == torch.float16 else ('bf16-split', 'f16x2', dtype)
    return None


def _first_operands(xm):
    """fp16 operand pair of a channels-last tower input: (hi, lo, device 1/scale); lo and the scale are None for an fp16 input
    (hi is xm itself, lo == 0, scale 1)."""
    from . import ops
    if xm.dtype == torch.float16:
        return xm, None, None
    if xm.dtype == torch.bfloat16:
        return ops.split_f16_from_bf16(xm)
    return ops.split_f16(xm, auto_scale=True)


def _packed_weight_f16(m):
    """fp16 (h, l, device 1/scale) packing of a tower conv's weight for ops.conv3x3_c256_f16*"""
    from . import ops
    w = m.conv.weight
    return cached_pack(m, 'f16', (w,), lambda: ops.conv3x3_pack_weight_f16(w))


def _packed_weight_f16_t(m):
    """dgrad operand: W^T with the taps reversed ([ci][co][8 - tap]), packed like a forward weight"""
    from . import ops
    w = m.conv.weight
    return cached_pack(m, 'f16t', (w,), lambda: ops.conv_tc_pack_weight_f16(
        w.detach().flip(2, 3).transpose(0, 1).reshape(w.shape[1], w.shape[0], 9).contiguous(), 9))


def _packed_weight(m):
    """TF32 hi/lo packing of a tower conv's weight for ops.conv3x3_c256"""
    from . import ops
    w = m.conv.weight
    return cached_pack(m, 'tf32', (w,), lambda: ops.conv3x3_pack_weight(w))


def _packed_tc(module, taps):
    """fp16 (h, l) column-slice packing (ops.conv_tc_pack_weight_f16) of a Linear (taps 1) / Conv2d (taps 9) weight for
    ops.conv_tc_f16"""
    from . import ops
    w = module.weight

    def make():
        w2 = w.detach().reshape(w.shape[0], w.shape[1], -1) if w.dim() == 4 else w.detach()
        return ops.conv_tc_pack_weight_f16(w2.contiguous(), taps)
    return cached_pack(module, ('tc', taps), (w,), make)


def _packed_tc_stacked(convs):
    """(packing, bias) of 3x3 Conv2d layers that read one input, their output channels stacked in order, so that one ops.conv_tc_f16
    launch computes them all; kept on convs[0]"""
    from . import ops

    def make():
        w = torch.cat([c.weight.detach() for c in convs])
        return (ops.conv_tc_pack_weight_f16(w.reshape(w.shape[0], w.shape[1], 9).contiguous(), 9),
                torch.cat([c.bias.detach() for c in convs]).contiguous())
    return cached_pack(convs[0], 'tc_stacked', [t for c in convs for t in (c.weight, c.bias)], make)


INT32_MAX = 2 ** 31 - 1
TMA_STRIDE_LIMIT = 2 ** 40         # bytes: cuTensorMapEncodeTiled's bound on a global stride


def wide_out_conv_plan(B, H, W, n_out, k=1, backward=False):
    """Row stride ldy of the (B,H,W,ldy) fp32 map that a conv3x3 output layer wider than one wgmma launch (n_out > 512) writes, and the
    refusal of shapes the kernels on that path cannot index.  A pure function of the shape (no device is touched).

    ldy = ceil4(n_out) for a forward alone: the (B,H,W,n_out) view of the map is the whole map when n_out % 4 == 0, so the per-anchor
    reshape downstream needs no copy.  ldy = ceil32(n_out) when a backward follows: the input gradient is one conv with Cin = ldy, and the
    conv kernel takes Cin % 32 == 0 (the padded weight rows are zero).
    Every kernel of the path indexes elements with 64-bit offsets (conv epilogue, ptb_split_f16*, ptb_col_sum, the loss and cost
    kernels); what stays 32-bit is the proposal index of the decode and top-k (H * W * k per image, int32 indices), and the tensor maps
    of the conv and wgrad operands (the fp16 pair of the (B,H,W,ldy) gradient) take per-image strides below 2^40 bytes.  Above either bound this raises ValueError."""
    if min(B, H, W, n_out, k) <= 0:
        raise ValueError(f'wide output conv: empty shape B={B} H={H} W={W} n_out={n_out} k={k}')
    ldy = (n_out + 31) // 32 * 32 if backward else (n_out + 3) // 4 * 4
    if H * W * k > INT32_MAX:
        raise ValueError(f'wide output conv: {H} x {W} cells x {k} anchors = {H * W * k} proposals per image; the decode indexes them '
                         f'in 32 bits (at most {INT32_MAX})')
    if H * W * ldy * 2 >= TMA_STRIDE_LIMIT:
        raise ValueError(f'wide output conv: an fp16 {H} x {W} x {ldy} gradient is {H * W * ldy * 2} bytes per image; the tensor maps '
                         f'of the conv and wgrad operands take per-image strides below 2^40 bytes')
    return ldy


class _WideOutConvFn(torch.autograd.Function):
    """conv3x3 (pad 1, bias) from 256 channels to n_out > 512 on the tensor cores, with a deterministic hand-written backward:
    forward  ptb_split_f16 of the input, then one ptb_conv_tc_f16x2 launch per column slice of <= 512 into one (B,H,W,ldy) map
             (ops.conv_tc_f16; the columns from n_out to ldy are not written)
    backward the (B,H,W,ldy) gradient split once (columns past n_out are zero: the caller takes the [..., :n_out] view), then
             dW: one ptb_conv_tc_wgrad_f16x2_ld per 256-column slice, read in place; db: ptb_col_sum; dX: ONE 9-tap conv with
             Cin = ldy on the transposed, flipped weights, zero-padded to ldy rows (ldy % 32 == 0, wide_out_conv_plan).
    Every sum is formed in a fixed order: two backward passes give the same bits."""

    @staticmethod
    def forward(ctx, xm, weight, bias, ldy):
        from . import ops
        n_out = weight.shape[0]
        h, l, inv = ops.split_f16(xm, auto_scale=True)
        packs = ops.conv_tc_pack_weight_f16(weight.detach().reshape(n_out, weight.shape[1], 9).contiguous(), 9)
        y = ops.conv_tc_f16(h, l, packs, 9, n_out, bias=bias.detach(), dev_out_scale=inv, ldy=ldy)
        ctx.save_for_backward(h, l, inv, weight.detach())
        return y

    @staticmethod
    def backward(ctx, g):
        from . import ops
        h, l, inv, weight = ctx.saved_tensors
        n_out, C = weight.shape[:2]
        g = g.contiguous()
        ldy = g.shape[-1]
        gh, gl, ginv = ops.split_f16(g, auto_scale=True)
        dw = db = dx = None
        if ctx.needs_input_grad[1]:
            dw = ops.conv_tc_wgrad_f16(gh, gl, h, l, 9, 1.0, ginv, inv)[:n_out]
        if ctx.needs_input_grad[2]:
            db = ops.col_sum(g.view(-1, ldy))[:n_out]
        if ctx.needs_input_grad[0]:
            wt = weight.new_zeros((C, ldy, 3, 3))
            wt[:, :n_out] = weight.flip(2, 3).transpose(0, 1)
            dx = ops.conv_tc_f16(gh, gl, ops.conv_tc_pack_weight_f16(wt.reshape(C, ldy, 9), 9), 9, C, dev_out_scale=ginv, ldy=C)
        return dx, dw, db, None


def wide_out_conv(conv, x, k=1):
    """conv(x) for an nn.Conv2d(256, n_out > 512, 3, padding=1) output layer on the tensor cores (_WideOutConvFn), differentiable in x,
    weight and bias.  x: fp32 CUDA (B,256,H,W); returns a (B,n_out,H,W) view of the (B,H,W,ldy) map."""
    from . import ops
    if not x.is_cuda or x.dtype != torch.float32:
        raise RuntimeError(f'wide output conv ({conv.out_channels} channels): expected an fp32 CUDA input, got {x.dtype} on {x.device}')
    B, _, H, W = x.shape
    backward = torch.is_grad_enabled() and (x.requires_grad or conv.weight.requires_grad or conv.bias.requires_grad)
    ldy = wide_out_conv_plan(B, H, W, conv.out_channels, k, backward)
    y = _WideOutConvFn.apply(ops.to_nhwc(x).contiguous(), conv.weight, conv.bias, ldy)
    return y[..., :conv.out_channels].permute(0, 3, 1, 2)


def _tc_geometry(convs, train):
    """the shipped head geometry of the tensor-core towers: conv3x3 s1 p1 without bias -> 256 channels, GroupNorm(32), ReLU; at
    inference Cin % 32 == 0, in training 256 -> 256 with an affine GroupNorm"""
    return len(convs) > 0 and all(
        m.conv.kernel_size == (3, 3) and m.conv.stride == (1, 1) and m.conv.padding == (1, 1) and m.conv.dilation == (1, 1)
        and m.conv.groups == 1 and m.conv.bias is None and m.conv.out_channels == 256 and m.norm_name == 'gn' and m.with_act
        and m.gn.num_groups == 32 and ((m.conv.in_channels == 256 and m.gn.affine) if train else m.conv.in_channels % 32 == 0)
        for m in convs)


def tower_path(convs, x, also=()):
    """The backend a tower of `convs` runs on for the input `x`, decided on the host from PTB_CONV_MODE, PTB_TOWER_TRAIN, the grad
    mode and, of x, only is_cuda, dtype and requires_grad:
      'wgmma-f16x2'        inference (grad disabled, or nothing of x, convs and `also` requires grad), a CUDA fp32 / fp16 / bf16
                           input and the inference geometry (_tc_geometry), with PTB_CONV_MODE=f16x2 (the default)
      'wgmma-3xtf32'       the same with any other PTB_CONV_MODE
      'wgmma-f16x2-train'  otherwise under grad, whatever requires it: PTB_CONV_MODE=f16x2, PTB_TOWER_TRAIN=tc (the default), a CUDA
                           fp32 / fp16 / bf16 input and the training geometry
      'cudnn'              everything else: torch's convs
    `also`: modules whose parameters count only toward "is this inference?" (a head's output convs, which run after the tower).
    A half-precision input raises here on the CPU (RuntimeError), and under a PTB_CONV_MODE other than f16x2 (input_plan)."""
    mode = os.environ.get('PTB_CONV_MODE', 'f16x2')
    if x.dtype in HALF_INPUT_DTYPES and not x.is_cuda:
        raise RuntimeError(f'tower: expected a CUDA tensor for a {x.dtype} input (pointtinybenchmark_b200 has no CPU path)')
    input_plan(x.dtype, mode)
    tc_input = x.is_cuda and x.dtype in _INPUT_DTYPES
    grad = torch.is_grad_enabled()
    inference = not (grad and (x.requires_grad or any(p.requires_grad for m in (*convs, *also) for p in m.parameters())))
    if tc_input and inference and _tc_geometry(convs, train=False):
        return 'wgmma-f16x2' if mode == 'f16x2' else 'wgmma-3xtf32'
    if tc_input and grad and mode == 'f16x2' and os.environ.get('PTB_TOWER_TRAIN', 'tc') == 'tc' and _tc_geometry(convs, train=True):
        return 'wgmma-f16x2-train'
    return 'cudnn'


class _TowerTCFn(torch.autograd.Function):
    """[conv3x3 -> GroupNorm -> ReLU] x n on the tensor cores with a hand-written backward:
    forward  ptb_conv3x3_c256_f16_gn: the conv with GroupNorm statistics and the GroupNorm + ReLU apply in one launch
             (the next layer's fp16 pair, fp32 after the last layer)                         (csrc/conv_tc.cu)
    backward ptb_gn_relu_bwd -> ptb_split_f16_amax -> ptb_conv_tc_wgrad_f16x2_ld (dW) and ptb_conv_tc_f16x2 with the transposed,
             flipped weights (dX)                                                          (csrc/tower_bwd.cu, wgrad_tc.cu)
    Saved per layer: the fp16 operand pair of its input (re-used as the wgrad operand), the conv output y and the statistics.
    A half-precision input is saved itself instead of a pair (backward derives the pair again as forward did), and its gradient is
    written in its dtype by the first layer's dgrad epilogue."""

    @staticmethod
    def forward(ctx, xm, convs, *params):
        from . import ops
        n_layers = len(convs)
        groups, eps = [m.gn.num_groups for m in convs], [float(m.gn.eps) for m in convs]
        h, l, dev_inv = _first_operands(xm)
        half_in = xm.dtype != torch.float32
        flag = torch.zeros(1, dtype=torch.int32, device=xm.device)
        saved, out = [], None
        for i in range(n_layers):
            gamma, beta = params[3 * i + 1], params[3 * i + 2]
            wh, wl, inv_w = _packed_weight_f16(convs[i])          # cached per parameter version (no host sync per step)
            inv_x = dev_inv if i == 0 else None
            last = i == n_layers - 1
            a, b, y, stats = ops.conv3x3_c256_f16_gn(h, l, wh, wl, inv_w, inv_x, gamma.detach(), beta.detach(), eps[i], flag,
                                                     out='fp32' if last else 'f16pair')
            saved += [xm, None, y, stats] if i == 0 and half_in else [h, l, y, stats]
            if last:
                out = a
            else:
                h, l = a, b
        ctx.n_layers, ctx.groups, ctx.eps, ctx.convs = n_layers, groups, eps, convs
        ctx.dev_inv, ctx.in_dtype = dev_inv, xm.dtype
        ctx.save_for_backward(*saved, *[p.detach() for p in params])
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import ops
        n = ctx.n_layers
        saved = ctx.saved_tensors
        acts, params = saved[:4 * n], saved[4 * n:]
        da = dout.contiguous()
        grads = [None] * (3 * n)
        for i in reversed(range(n)):
            h, l, y, stats = acts[4 * i:4 * i + 4]
            inv_x = ctx.dev_inv if i == 0 else None
            if i == 0 and ctx.in_dtype != torch.float32:
                h, l, inv_x = _first_operands(h)
                if l is None:                                     # the wgrad kernel reads a materialised lo
                    l = torch.zeros_like(h)
            w, gamma, beta = params[3 * i], params[3 * i + 1], params[3 * i + 2]
            dy, dg, db, amax = ops.gn_relu_bwd(da, y, stats, gamma, beta, ctx.groups[i], ctx.eps[i], True)
            dyh, dyl, inv_dy = ops.split_f16_amax(dy, amax)
            grads[3 * i + 1], grads[3 * i + 2] = dg, db
            if ctx.needs_input_grad[2 + 3 * i]:
                grads[3 * i] = ops.conv_tc_wgrad_f16(dyh, dyl, h, l, 9, 1.0, inv_dy, inv_x)
            if i > 0 or ctx.needs_input_grad[0]:
                # dgrad = the forward kernel with W^T and reversed taps
                da = ops.conv_tc_f16(dyh, dyl, _packed_weight_f16_t(ctx.convs[i]), 9, w.shape[1], dev_out_scale=inv_dy,
                                     out_dtype=ctx.in_dtype if i == 0 else torch.float32)
            else:
                da = None
        return (da, None, *grads)


def tower(convs, x, info=None, want='fp32'):
    """4 x [conv3x3 + GN + ReLU] on the backend tower_path names.  Inference: hand-written wgmma implicit GEMM (fp16 two-term split or
    3xTF32) with GroupNorm statistics in the epilogue (csrc/conv_tc.cu).  Training (autograd): _TowerTCFn for the shipped 256 -> 256
    geometry (same forward kernel + hand-written backward), else cuDNN fp32 through torch.
    x: fp32, or an fp16 / bf16 CUDA feature map on the tensor-core paths (`input_plan`; the output is fp32 either way).
    want='f16pair' returns the (B,H,W,C) fp16 operand pair of the output instead, on the wgmma-f16x2 path only (ValueError elsewhere:
    ask tower_path first).  info (optional dict) receives 'backend' and, on the tensor-core paths, 'input_path'; on wgmma-f16x2 also
    'overflow_flag'."""
    from . import ops
    path = tower_path(convs, x)
    if want == 'f16pair' and path != 'wgmma-f16x2':
        raise ValueError(f"tower: want='f16pair' needs the wgmma-f16x2 path; this tower and input take {path}")
    if path == 'cudnn':
        if x.dtype in HALF_INPUT_DTYPES:
            raise NotImplementedError(f'tower: a {x.dtype} input needs the tensor-core geometry (conv3x3 s1 p1 without bias -> 256 '
                                      'channels, GroupNorm(32), ReLU, Cin % 32 == 0; 256 -> 256 under autograd); convert it to fp32 for '
                                      'the cuDNN path')
        if info is not None:
            info['backend'] = 'cudnn'
        x = x.contiguous(memory_format=torch.channels_last)
        with no_tf32():
            for m in convs:
                x = m(x)
        return x
    xm = ops.to_nhwc(x).contiguous()
    if info is not None:
        info['backend'] = path
        info['input_path'] = input_plan(x.dtype)[0]
    if path == 'wgmma-f16x2':
        # two-term fp16 split (22 significant bits), kind::f16: half the tensor-pipe time of 3xTF32.  The first layer's input
        # is scaled by a power of two chosen on the device from max|x| (no host sync); later layers consume GroupNorm outputs.
        h, l, dev_inv = _first_operands(xm)
        flag = torch.zeros(1, dtype=torch.int32, device=x.device)
        if info is not None:
            info['overflow_flag'] = flag
        for i, m in enumerate(convs):
            wh, wl, inv_w = _packed_weight_f16(m)
            # conv + GroupNorm + ReLU in one launch: the apply runs inside the conv kernel (ptb_conv3x3_c256_f16_gn)
            fp32_out = i == len(convs) - 1 and want == 'fp32'
            a, b, _, _ = ops.conv3x3_c256_f16_gn(h, l, wh, wl, inv_w, dev_inv if i == 0 else None, m.gn.weight.detach(),
                                                 m.gn.bias.detach(), m.gn.eps, flag, out='fp32' if fp32_out else 'f16pair')
            if fp32_out:
                out = a
            else:
                h, l = a, b
        if want == 'f16pair':
            return h, l              # feeds ptb_conv_tc_f16x2 directly
    elif path == 'wgmma-3xtf32':
        hi, lo = ops.split_tf32(xm)
        for i, m in enumerate(convs):
            wh, wl = _packed_weight(m)
            y, stats = ops.conv3x3_c256(hi, lo, wh, wl)
            last = i == len(convs) - 1
            res = ops.gn_relu_apply(y, stats, m.gn.weight.detach(), m.gn.bias.detach(), m.gn.num_groups, m.gn.eps, True,
                                    split=not last)
            if last:
                out = res
            else:
                hi, lo = res
    else:
        params = []
        for m in convs:
            params += [m.conv.weight, m.gn.weight, m.gn.bias]
        out = _TowerTCFn.apply(xm, convs, *params)
    return out.permute(0, 3, 1, 2)          # (B,C,H,W) view with channels_last strides
