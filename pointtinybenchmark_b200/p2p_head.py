"""P2PHead — host-side mirror of the reference's P2PNet-style head over the sm_90a kernels.

reference: TOV_mmdetection/mmdet/models/point/dense_heads/p2p_head.py:18-572 (P2PHead), HungarianAssignerV2
(core/bbox/assigners/hungarian_assigner.py:149-270) with lists of FocalLossCost, ClassificationCostV2, ZeroCost and DisCostV2
(core/bbox/match_costs/match_cost.py; parsed by assigners.match_cost_terms),
multiclass_nms (core/post_processing/bbox_nms.py).  Same ctor kwargs / outputs / state_dict keys
(cls_convs.*, reg_convs.*, cls_out (conv3x3), reg_out (conv3x3)).

What runs where: towers and the two output convs = wgmma implicit GEMMs of libptb_b200.so at inference; under autograd the
towers use the tensor-core autograd function of layers.py (dgrad / wgrad / GroupNorm backward kernels), the two output convs cuDNN fp32
up to 512 channels and a cls_out wider than that (257 to 1280 classes: Objects365, LVIS) the tensor-core autograd function
layers._WideOutConvFn (column-sliced forward, deterministic wgrad / dgrad); decode, top-k, NMS / soft-NMS, cost matrix, the Hungarian matching (scipy's shortest-augmenting-path algorithm
restated as a one-CTA-per-image kernel, bit-identical assignments incl. ties: csrc/lsap_core.cuh; SURVEY.md §8f rank 2) and the
losses = libptb_b200.so: FocalLoss or the reference's default CrossEntropyLoss(use_sigmoid=True) for classification, the latter
also with class_weight (= pos_weight) or in softmax mode (use_sigmoid=False: C+1 outputs per anchor, background last, softmax decode
and cross-entropy kernels), SmoothL1Loss or the default MSELoss for the points.  Nothing of the training step returns to the host
except one (B,) status read.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .assigners import cost_matrix, match_cost_terms
from .post_processing import check_split_thr, parse_nms_cfg, run_multiclass_nms
from .layers import ConvModule, PackedWeightsMixin, bias_init_with_prob, normal_init_, no_tf32, tower, tower_path, wide_out_conv, \
    wide_out_conv_plan, _packed_tc
from .registry import CfgNode, register_head


class _LossSumFn(torch.autograd.Function):
    """op(x, *args)[0] for a fused loss of ops (sigmoid_focal, sigmoid_bce, softmax_ce, ghmc, smooth_l1, mse, l1_rows, balanced_l1_rows,
    ghmr), differentiable in x: the backward is op's gradient launch, op(x, *args, scale=g, want_grad=True), with the tensors the
    forward saw (GHM: the bin weights of the forward step, not ones recomputed from an updated acc_sum)."""

    @staticmethod
    def forward(ctx, op, x, *args):
        is_tensor = [isinstance(a, torch.Tensor) for a in args]
        ctx.save_for_backward(x, *(a if t else None for a, t in zip(args, is_tensor)))
        ctx.op, ctx.args = op, [None if t else a for a, t in zip(args, is_tensor)]
        return op(x, *args)[0]

    @staticmethod
    def backward(ctx, g):
        x, *tensors = ctx.saved_tensors
        args = [a if t is None else t for a, t in zip(ctx.args, tensors)]
        scale = g.reshape(1).float().contiguous()
        return (None, ctx.op(x, *args, scale=scale, want_grad=True)) + (None,) * len(args)


MAX_OUT_CHANNELS = 512     # widest output of one wgmma conv launch (ptb_conv_tc_f16x2): cls_out beyond it runs in column slices
MAX_CLASSES = 1280         # CPRHead's limit (cpr_head.MAX_CLASSES): the second stage takes every dataset the first one refines
WIDE_MIN_CLASSES = 257     # the many-class path (cls_out in column slices) starts above 256 classes, where CPRHead's sliced logit map does;
                           # up to 256 classes cls_out must fit one launch, as it always had to
MAX_LEVELS = 8             # levels of one multi-level decode launch (ptb_p2p_decode_topk_levels)
LOSS_CLS_TYPES = ('FocalLoss', 'CrossEntropyLoss', 'GHMC')
LOSS_REG_TYPES = ('SmoothL1Loss', 'MSELoss', 'GHMR', 'L1Loss', 'BalancedL1Loss')
# the mmdet defaults of the losses added after the first four (ghm_loss.py, smooth_l1_loss.py, balanced_l1_loss.py); a config of one
# of them takes these, not the defaults the head fills in for the others
LOSS_DEFAULTS = {'GHMC': dict(bins=10, momentum=0, use_sigmoid=True, loss_weight=1.0),
                 'GHMR': dict(mu=0.02, bins=10, momentum=0, loss_weight=1.0),
                 'L1Loss': dict(reduction='mean', loss_weight=1.0),
                 'BalancedL1Loss': dict(alpha=0.5, gamma=1.5, beta=1.0, reduction='mean', loss_weight=1.0)}
# losses of the reference tree that cannot run on P2PHead's (labels, label_weights) / (points, point_weights) targets
UNSUPPORTED_LOSSES = {
    'VarifocalLoss': 'it takes soft IoU-aware score targets of the logits\' shape; P2PHead\'s targets are integer labels '
                     '(the reference fails its pred.size() == target.size() assertion)',
    'QualityFocalLoss': 'it takes a (labels, quality scores) target pair; P2PHead passes labels only (the reference fails its '
                        'len(target) == 2 assertion)',
    'SeesawLoss': 'it needs num_classes + 2 softmax columns (an objectness pair); P2PHead has num_classes or num_classes + 1',
    **{t: 'it compares boxes; P2PHead regresses points' for t in ('IoULoss', 'BoundedIoULoss', 'GIoULoss', 'DIoULoss', 'CIoULoss')}}


class GHMBuffers(nn.Module):
    """The state of GHMC / GHMR (ghm_loss.py:35-48, 113-124): the bin `edges` buffer and, with momentum > 0, `acc_sum`, under the
    reference's names (loss_cls.edges, loss_cls.acc_sum, loss_reg.*), so its checkpoints load with strict=True.  The loss reads
    `edges` from the buffer; a loaded set must be nondecreasing (the kernels' bins are disjoint)."""

    def __init__(self, bins, momentum, last_edge):
        super().__init__()
        if not 1 <= int(bins) <= ops.GHM_MAX_BINS:
            raise NotImplementedError(f'P2PHead: GHM bins={bins}; the CUDA histogram takes 1 to {ops.GHM_MAX_BINS} bins')
        self.bins, self.momentum = int(bins), float(momentum)
        edges = torch.arange(self.bins + 1).float() / self.bins
        if last_edge is None:
            edges[-1] += 1e-6           # GHMC
        else:
            edges[-1] = last_edge       # GHMR: 1e3
        self.register_buffer('edges', edges)
        if self.momentum > 0:
            self.register_buffer('acc_sum', torch.zeros(self.bins))
        else:
            self.acc_sum = None

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        e = state_dict.get(prefix + 'edges')
        if e is not None and e.numel() > 1 and bool((e[1:] < e[:-1]).any()):
            raise ValueError(f'{prefix}edges must be nondecreasing, got {e.tolist()}')
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


@register_head
class P2PHead(PackedWeightsMixin, nn.Module):
    def __init__(self, num_classes, in_channels,
                 point_anchor=((-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)),
                 assign_before_pred=False, pts_gamma=100. / 8, reg_norm=1. / 8,
                 loss_cls=None, loss_reg=None, init_cfg=None,
                 feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64),
                 conv_cfg=None, norm_cfg=None, conv_bias='auto', dcn_on_last_conv=False, loss_bbox=None,
                 train_cfg=None, test_cfg=None, **kwargs):
        super().__init__()
        if kwargs:
            raise TypeError(f'P2PHead: unexpected kwargs {sorted(kwargs)}')
        self.num_classes, self.in_channels, self.feat_channels = num_classes, in_channels, feat_channels
        self.stacked_convs, self.strides = stacked_convs, list(strides)
        self.point_anchor = torch.tensor(point_anchor, dtype=torch.float32).reshape(-1, 2)
        self.num_points = self.point_anchor.shape[0]
        self.assign_before_pred, self.pts_gamma, self.reg_norm = assign_before_pred, pts_gamma, reg_norm
        self.loss_cls_cfg = dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0)
        self.loss_cls_cfg.update(loss_cls or {})
        self.loss_reg_cfg = dict(type='MSELoss', loss_weight=2e-4)
        self.loss_reg_cfg.update(loss_reg or {})
        if self.loss_cls_cfg['type'] in LOSS_DEFAULTS:
            self.loss_cls_cfg = dict(LOSS_DEFAULTS[self.loss_cls_cfg['type']], **loss_cls)
        if self.loss_reg_cfg['type'] in LOSS_DEFAULTS:
            self.loss_reg_cfg = dict(LOSS_DEFAULTS[self.loss_reg_cfg['type']], **loss_reg)
        for c in (self.loss_cls_cfg, self.loss_reg_cfg):
            if c['type'] in ('L1Loss', 'BalancedL1Loss') and c['reduction'] != 'mean':
                raise NotImplementedError(f"P2PHead: {c['type']}(reduction={c['reduction']!r}); the head averages the point loss over "
                                          f"the positives, which mmdet does for reduction='mean' only")
        rc = self.loss_reg_cfg
        if rc['type'] == 'BalancedL1Loss':
            # balanced_l1_loss.py divides by b = e^(gamma / alpha) - 1 and by beta
            a, g, be = float(rc['alpha']), float(rc['gamma']), float(rc['beta'])
            if not (a > 0 and be > 0 and g == g and g != 0):
                raise ValueError(f'P2PHead: BalancedL1Loss(alpha={a}, gamma={g}, beta={be}); alpha and beta must be positive and gamma '
                                 f'non-zero (b = e^(gamma / alpha) - 1 divides the loss; mmdet raises ZeroDivisionError at gamma=0)')
        self.train_cfg = CfgNode(train_cfg) if train_cfg is not None else None
        self.test_cfg = CfgNode(test_cfg) if test_cfg is not None else None
        if not 1 <= len(self.strides) <= MAX_LEVELS:
            raise NotImplementedError(f'P2PHead: {len(self.strides)} FPN levels; the CUDA head takes 1 to {MAX_LEVELS} (strides)')
        # p2p_head.py:63-67: sigmoid scores C classes, softmax C + 1 with the background column last
        self.use_sigmoid_cls = bool(self.loss_cls_cfg.get('use_sigmoid', False))
        if self.loss_cls_cfg['type'] == 'GHMC':
            if not self.loss_cls_cfg['use_sigmoid']:
                raise NotImplementedError('P2PHead: GHMC supports use_sigmoid=True only (ghm_loss.py raises NotImplementedError '
                                          'for the softmax form)')
            # p2p_head.py:63 reads use_sigmoid from the config as written (default False): a GHMC config without it makes a
            # softmax head of num_classes + 1 columns, whose background label then fills the last column of GHMC's one-hot
            self.use_sigmoid_cls = bool(loss_cls.get('use_sigmoid', False))
        if not self.use_sigmoid_cls and self.loss_cls_cfg['type'] == 'FocalLoss':
            raise NotImplementedError('P2PHead: FocalLoss supports sigmoid classification only (use_sigmoid=True)')
        self.num_cls_out = num_classes if self.use_sigmoid_cls else num_classes + 1
        cw = self.loss_cls_cfg.get('class_weight') if self.loss_cls_cfg['type'] == 'CrossEntropyLoss' else None
        if cw is not None and len(cw) != self.num_cls_out:
            raise ValueError(f'P2PHead: CrossEntropyLoss.class_weight has {len(cw)} entries; '
                             f'{"sigmoid" if self.use_sigmoid_cls else "softmax"} classification needs {self.num_cls_out}')
        self.class_weight = None if cw is None else torch.tensor([float(v) for v in cw], dtype=torch.float32)
        if num_classes > MAX_CLASSES:
            raise NotImplementedError(f'P2PHead: num_classes={num_classes} exceeds the {MAX_CLASSES} classes the CUDA head supports')
        if self.num_cls_out * self.num_points > MAX_OUT_CHANNELS and num_classes < WIDE_MIN_CLASSES:
            raise NotImplementedError(
                f'P2PHead: cls_out would have {self.num_cls_out} classes x {self.num_points} anchors = '
                f'{self.num_cls_out * self.num_points} output channels; up to {WIDE_MIN_CLASSES - 1} classes the output conv kernel '
                f'supports at most {MAX_OUT_CHANNELS} (heads of {WIDE_MIN_CLASSES} to {MAX_CLASSES} classes run it in column slices)')
        if 2 * self.num_points > MAX_OUT_CHANNELS:
            raise NotImplementedError(f'P2PHead: reg_out would have 2 x {self.num_points} anchors = {2 * self.num_points} output '
                                      f'channels; the output conv kernel supports at most {MAX_OUT_CHANNELS}')
        if self.num_cls_out * self.num_points > MAX_OUT_CHANNELS and feat_channels != 256:
            raise NotImplementedError(f'P2PHead: a cls_out of {self.num_cls_out * self.num_points} output channels (> {MAX_OUT_CHANNELS}) '
                                      f'runs on the tensor-core wide conv, which takes feat_channels=256 (got {feat_channels})')
        self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList()
        for i in range(stacked_convs):
            chn = in_channels if i == 0 else feat_channels
            self.cls_convs.append(ConvModule(chn, feat_channels, 3, 1, 1, norm_cfg=norm_cfg, bias=conv_bias))
            self.reg_convs.append(ConvModule(chn, feat_channels, 3, 1, 1, norm_cfg=norm_cfg, bias=conv_bias))
        self.cls_out = nn.Conv2d(feat_channels, self.num_cls_out * self.num_points, 3, padding=1)
        self.reg_out = nn.Conv2d(feat_channels, self.num_points * 2, 3, padding=1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                normal_init_(m, 0.01, 0.0)
        nn.init.constant_(self.cls_out.bias, bias_init_with_prob(0.01))
        if self.train_cfg is not None:
            a = dict(self.train_cfg.assigner)
            if a.get('type') != 'HungarianAssignerV2':
                raise NotImplementedError(f"assigner {a.get('type')}")
            self.assign = dict(terms=match_cost_terms(a.get('cls_costs'), a.get('reg_costs')), topk_k=a.get('topk_k', 1))
        if self.loss_cls_cfg['type'] == 'GHMC':
            self.loss_cls = GHMBuffers(self.loss_cls_cfg['bins'], self.loss_cls_cfg['momentum'], None)
        if self.loss_reg_cfg['type'] == 'GHMR':
            self.loss_reg = GHMBuffers(self.loss_reg_cfg['bins'], self.loss_reg_cfg['momentum'], 1e3)
        self._init_packed_hooks()
        self.check_assign_status = True      # read the (B,) status of the matching kernel each step (scipy's ValueErrors)

    # ------------------------------------------------------------------------------------------------
    def forward(self, feats):
        """p2p_head.py:104-123.  Inference: towers AND the two conv3x3 output layers run on the wgmma kernel (fp16 two-term
        split, fp32-level accuracy; a cls_out of up to 512 channels, e.g. 320 at the reference's default 4 anchors x 80 classes, in one
        launch, a wider one as column slices of <= 512 into one map, layers.wide_out_conv_plan's ldy); with autograd recording the
        towers use the tensor-core autograd function of layers.py and the two output convs cuDNN fp32 up to 512 channels, a wider
        cls_out layers._WideOutConvFn (also inside a caller's autocast region).
        feats[i]: fp32, or the fp16 / bf16 map of a backbone under torch.autocast, taken as it is (layers.input_plan; no .float() in
        front of the head).  The outputs are fp32; `last_input_path` names the path the towers took."""
        cls_outs, pts_outs = [], []
        for x in feats:
            info = {}
            if tower_path([*self.cls_convs, *self.reg_convs], x, also=(self.cls_out, self.reg_out)) == 'wgmma-f16x2':
                pc = tower(self.cls_convs, x, info, want='f16pair')
                pr = tower(self.reg_convs, x, info, want='f16pair')
                self._record_tower(info)
                nc, nr = self.cls_out.out_channels, self.reg_out.out_channels
                ldy = None
                if nc > MAX_OUT_CHANNELS:      # ldy = ceil4(nc): [..., :nc] is the whole map if 4 | nc
                    B_, H_, W_ = pc[0].shape[:3]
                    ldy = wide_out_conv_plan(B_, H_, W_, nc, self.num_points)
                yc = ops.conv_tc_f16(pc[0], pc[1], _packed_tc(self.cls_out, 9), 9, nc, bias=self.cls_out.bias.detach(), ldy=ldy)
                yr = ops.conv_tc_f16(pr[0], pr[1], _packed_tc(self.reg_out, 9), 9, nr, bias=self.reg_out.bias.detach())
                cls_outs.append(yc[..., :nc].permute(0, 3, 1, 2))
                pts_outs.append(yr[..., :nr].permute(0, 3, 1, 2))
                continue
            # autograd path: the towers run layers._TowerTCFn (tensor-core forward + dgrad + wgrad + GroupNorm backward) for the
            # shipped geometry; output convs of up to 512 channels stay cuDNN fp32, never TF32 (1e-4 logits); a wider cls_out runs
            # layers._WideOutConvFn on the tensor cores (selected from the width alone)
            fc, fr = tower(self.cls_convs, x, info), tower(self.reg_convs, x, info)
            self._record_tower(info)
            with no_tf32(), torch.autocast('cuda', enabled=False):
                if self.cls_out.out_channels > MAX_OUT_CHANNELS:
                    cls_outs.append(wide_out_conv(self.cls_out, fc, self.num_points))
                else:
                    cls_outs.append(self.cls_out(fc))
                pts_outs.append(self.reg_out(fr))
        return cls_outs, pts_outs

    def forward_train(self, x, img_metas, gt_bboxes, gt_labels=None, gt_bboxes_ignore=None, proposal_cfg=None, **kwargs):
        outs = self(x)
        return self.loss(*outs, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=gt_bboxes_ignore)

    def simple_test(self, feats, img_metas, rescale=False, **kwargs):
        outs = self.forward(feats)
        return self.get_bboxes(*outs, img_metas, rescale=rescale)

    # ------------------------------------------------------------------------------------------------
    def _grid(self, H, W, device, s=None):
        s = float(self.strides[0]) if s is None else s
        xx = (torch.arange(0., W, device=device) * s).repeat(H)
        yy = (torch.arange(0., H, device=device) * s).view(-1, 1).repeat(1, W).view(-1)
        return xx, yy

    @torch.autocast('cuda', enabled=False)
    def get_pred_points(self, cls_out, pts_out, img_metas):
        """p2p_head.py:125-170 (single level): differentiable torch elementwise ops on channels-last views."""
        B, _, H, W = cls_out.shape
        k, C, s = self.num_points, self.num_cls_out, float(self.strides[0])
        dev = cls_out.device
        cls = ops.to_nhwc(cls_out).reshape(B, H * W * k, C)
        reg = ops.to_nhwc(pts_out).reshape(B, H * W, k, 2)
        xx, yy = self._grid(H, W, dev)
        anchor = torch.stack([xx, yy], -1)[None, :, None, :] + (self.point_anchor.to(dev) * s)[None, None]
        anchor = anchor.expand(B, H * W, k, 2)
        pred = anchor + reg * self.pts_gamma * s
        vflag = []
        for m in img_metas:
            ph, pw = m['pad_shape'][:2]
            vh, vw = min(int(np.ceil(ph / s)), H), min(int(np.ceil(pw / s)), W)
            v = torch.zeros(H, W, dtype=torch.bool)
            v[:vh, :vw] = True
            vflag.append(v.reshape(-1))
        self._valid_host = vflag                       # host copy: the assignment sizes its launches without a device sync
        valid = torch.stack(vflag).to(dev)[:, :, None].expand(B, H * W, k).reshape(B, -1)
        return anchor.reshape(B, -1, 2), pred.reshape(B, -1, 2), valid, cls

    @torch.autocast('cuda', enabled=False)
    def get_pred_points_levels(self, cls_outs, pts_outs, img_metas):
        """p2p_head.py:125-170 over L >= 2 levels: each level as get_pred_points with its own stride, the rows concatenated
        level-major (cell-major, anchor-minor inside a level), as the reference's torch.cat of the flattened maps orders them."""
        B = cls_outs[0].shape[0]
        k, C = self.num_points, self.num_cls_out
        dev = cls_outs[0].device
        if len(cls_outs) != len(self.strides) or len(pts_outs) != len(self.strides):
            raise ValueError(f'P2PHead has {len(self.strides)} strides but got {len(cls_outs)} cls maps and {len(pts_outs)} pts maps')
        anchors, preds, clss, vflag = [], [], [], [[] for _ in img_metas]
        for cls_out, pts_out, s in zip(cls_outs, pts_outs, self.strides):
            s = float(s)
            _, _, H, W = cls_out.shape
            clss.append(ops.to_nhwc(cls_out).reshape(B, H * W * k, C))
            reg = ops.to_nhwc(pts_out).reshape(B, H * W, k, 2)
            xx, yy = self._grid(H, W, dev, s)
            anchor = torch.stack([xx, yy], -1)[None, :, None, :] + (self.point_anchor.to(dev) * s)[None, None]
            anchor = anchor.expand(B, H * W, k, 2)
            preds.append((anchor + reg * self.pts_gamma * s).reshape(B, -1, 2))
            anchors.append(anchor.reshape(B, -1, 2))
            for b, m in enumerate(img_metas):
                ph, pw = m['pad_shape'][:2]
                vh, vw = min(int(np.ceil(ph / s)), H), min(int(np.ceil(pw / s)), W)
                v = torch.zeros(H, W, dtype=torch.bool)
                v[:vh, :vw] = True
                vflag[b].append(v.reshape(-1))
        self._valid_host = [torch.cat(v) for v in vflag]
        valid = torch.stack(self._valid_host).to(dev)[:, :, None].expand(B, -1, k).reshape(B, -1)
        return torch.cat(anchors, 1), torch.cat(preds, 1), valid, torch.cat(clss, 1)

    def row_inv_norm(self, featmap_sizes, device):
        """(Q,) fp32 1 / (stride_q * reg_norm) of every proposal row of get_pred_points_levels (p2p_head.py:234-240 divides each row
        by its own stride, column 2 of pred_pts).  Depends on the map sizes only: built once per size set and device."""
        key = (tuple(tuple(int(v) for v in hw) for hw in featmap_sizes), str(device))
        if getattr(self, '_row_inv_cache', (None,))[0] != key:
            inv = torch.cat([torch.full((int(h) * int(w) * self.num_points,), 1.0 / (float(s) * self.reg_norm))
                             for (h, w), s in zip(featmap_sizes, self.strides)])
            self._row_inv_cache = (key, inv.to(device))
        return self._row_inv_cache[1]

    def loss(self, cls_outs, pts_outs, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=None):
        """p2p_head.py:172-248 -> dict(loss_cls=[B], loss_pts=[B])."""
        cls_type, reg_type = self.loss_cls_cfg['type'], self.loss_reg_cfg['type']
        for t in (cls_type, reg_type):
            if t in UNSUPPORTED_LOSSES:
                raise NotImplementedError(f'P2PHead cannot train with {t}: {UNSUPPORTED_LOSSES[t]}')
        if cls_type not in LOSS_CLS_TYPES or reg_type not in LOSS_REG_TYPES:
            raise NotImplementedError(f'P2PHead: loss_cls must be one of {LOSS_CLS_TYPES} and loss_reg one of {LOSS_REG_TYPES}')
        cls_out, pts_out = cls_outs[0], pts_outs[0]
        if not cls_out.is_cuda:
            raise RuntimeError('P2PHead runs on CUDA tensors only; there is no CPU fallback')
        for gb in gt_bboxes:                       # p2p_head.py:183-184: the reference refuses images without a GT point
            assert len(gb) > 0, gt_bboxes
        dev = cls_out.device
        multi = len(self.strides) > 1
        if multi:
            anchor, pred, valid, cls = self.get_pred_points_levels(cls_outs, pts_outs, img_metas)
        else:
            anchor, pred, valid, cls = self.get_pred_points(cls_out, pts_out, img_metas)
        B, Q, C = cls.shape
        s = float(self.strides[0])
        prop = (anchor if self.assign_before_pred else pred).detach().contiguous()
        a = self.assign
        # ---- cost matrices and the Hungarian matching on the GPU: no cost.cpu(), no scipy (hungarian_assigner.py:229-270)
        key = (tuple(tuple(c.shape[-2:]) for c in cls_outs), tuple(tuple(m['pad_shape'][:2]) for m in img_metas), str(dev))
        if getattr(self, '_ridx_cache', (None,))[0] != key:           # valid-row lists depend on the map size and pad shapes only
            valid_host = torch.stack(self._valid_host)[:, :, None].expand(B, valid.shape[1] // self.num_points, self.num_points).reshape(B, -1)
            ridx_l = [torch.nonzero(valid_host[b]).squeeze(1).int() for b in range(B)]
            n_valid = [int(r.shape[0]) for r in ridx_l]
            r_off = np.concatenate([[0], np.cumsum(n_valid)]).astype(np.int64)
            r_flat = torch.cat(ridx_l).to(dev) if r_off[-1] > 0 else torch.zeros(1, dtype=torch.int32, device=dev)
            self._ridx_cache = (key, n_valid, r_off, r_flat)
        _, n_valid, ridx_off, ridx_flat = self._ridx_cache
        shapes = [(n_valid[b], int(gt_labels[b].shape[0])) for b in range(B)]
        cost_off = np.concatenate([[0], np.cumsum([sh[0] * sh[1] for sh in shapes])]).astype(np.int64)
        cost_flat = torch.empty(max(int(cost_off[-1]), 1), dtype=torch.float32, device=dev)
        gpts_l = []
        for b in range(B):
            gpts = ((gt_bboxes[b][:, :2] + gt_bboxes[b][:, 2:]) / 2).to(dev).float().contiguous()
            gpts_l.append(gpts)
            if shapes[b][0] == 0 or shapes[b][1] == 0:
                continue
            cost_matrix(cls[b].detach().contiguous(), prop[b], ridx_flat[ridx_off[b]:ridx_off[b + 1]], gpts,
                        gt_labels[b].to(dev).int().contiguous(), a['terms'], img_metas[b]['img_shape'],
                        out=cost_flat[cost_off[b]:cost_off[b + 1]])
        gi_all = torch.zeros((B, Q), dtype=torch.int64, device=dev)
        status = ops.hungarian_v2_batch(cost_flat, shapes, a['topk_k'], gi_all, [b * Q for b in range(B)], ridx_flat, ridx_off[:-1])
        if self.check_assign_status:                          # one (B,) int32 read per batch: scipy's two ValueErrors
            st = status.cpu()
            if int(st.max()) != 0:
                bad = int(torch.nonzero(st)[0])
                raise ValueError({1: 'cost matrix is infeasible', 2: 'matrix contains invalid numeric entries'}.get(
                    int(st[bad]), f'hungarian kernel status {int(st[bad])}') + f' (image {bad})')
        self._last_assign = dict(gt_inds=gi_all, status=status)
        labels_l, lw_l, gp_l, pw_l = [], [], [], []
        neg_w = self.train_cfg.get('neg_weight', 1.0)
        pos_w = self.train_cfg.get('pos_weight', 1.0)
        for b in range(B):
            gi = gi_all[b]
            vb = valid[b]
            pos = gi > 0
            gl = gt_labels[b].to(dev)
            gpts = gpts_l[b]
            if gl.shape[0] == 0:                                 # no GT: everything background (hungarian_assigner.py:214-219)
                gl = torch.zeros(1, dtype=torch.long, device=dev)
                gpts = torch.zeros(1, 2, device=dev)
            labels = torch.where(pos, gl[(gi - 1).clamp(min=0)], torch.full_like(gi, self.num_classes))
            labels = torch.where(vb, labels, torch.zeros_like(labels))               # unmap(fill=0)
            lw = torch.where(pos, torch.full((Q,), float(pos_w), device=dev),
                             torch.full((Q,), 1.0 if neg_w <= 0 else float(neg_w), device=dev)) * vb.float()
            gp = torch.where(pos[:, None], gpts[(gi - 1).clamp(min=0)], torch.zeros(Q, 2, device=dev))
            pw = pos.float()[:, None].expand(Q, 2).contiguous()
            labels_l.append(labels); lw_l.append(lw.contiguous()); gp_l.append(gp.contiguous()); pw_l.append(pw)
        num_total_pos = sum([(p[:, 0] > 0).sum() for p in pw_l]).float()
        # loss_single (p2p_head.py:220-231): CrossEntropyLoss averages over every proposal of the batch, FocalLoss over the positives
        cls_avg = float(B * Q) if cls_type == 'CrossEntropyLoss' else num_total_pos
        inv_norm = 1.0 / (s * self.reg_norm)
        cw = self.class_weight.to(dev) if self.class_weight is not None else None
        if cls_type == 'FocalLoss':
            cls_op, cls_args = ops.sigmoid_focal, (self.loss_cls_cfg.get('gamma', 2.0), self.loss_cls_cfg.get('alpha', 0.25))
        else:
            cls_op, cls_args = (ops.sigmoid_bce if self.use_sigmoid_cls else ops.softmax_ce), (cw,)
        # p2p_head.py:234-240: every row divided by its own level's stride (the losses added with GHM take the per-row form at
        # any level count)
        if multi or reg_type in ('GHMR', 'L1Loss', 'BalancedL1Loss'):
            row_inv = self.row_inv_norm([c.shape[-2:] for c in cls_outs], dev)
        rc = self.loss_reg_cfg
        if reg_type == 'MSELoss':
            reg_op, reg_args = (ops.mse_rows, (row_inv,)) if multi else (ops.mse, (inv_norm,))
        elif reg_type == 'L1Loss':
            reg_op, reg_args = ops.l1_rows, (row_inv,)
        elif reg_type == 'BalancedL1Loss':
            reg_op, reg_args = ops.balanced_l1_rows, (row_inv, rc['alpha'], rc['gamma'], rc['beta'])
        else:
            beta = rc.get('beta', 1.0)
            reg_op, reg_args = (ops.smooth_l1_rows, (row_inv, beta)) if multi else (ops.smooth_l1, (inv_norm, beta))
        self._last_ghm = {}
        # GHMC / GHMR (ghm_loss.py:50-94, 127-172), called per image by loss_single: the batch's histograms and bin weights in one
        # step (momentum: acc_sum updated image by image, in the forward pass), then each image's sum over its tot with the bin
        # weights that step made, which _LossSumFn keeps for the backward.  avg_factor is not used.
        if cls_type == 'GHMC':
            x_all, m = cls.contiguous(), self.loss_cls
            counts, cls_bw, cls_tot = ops.ghmc_bin_weights(x_all.detach(), torch.stack(labels_l), torch.stack(lw_l), m.edges,
                                                           m.momentum, m.acc_sum)
            self._last_ghm['cls_counts'] = counts
        if reg_type == 'GHMR':
            p_all, m = pred.contiguous(), self.loss_reg
            counts, reg_bw, reg_tot = ops.ghmr_bin_weights(p_all.detach(), torch.stack(gp_l), torch.stack(pw_l), row_inv, rc['mu'],
                                                           m.edges, m.momentum, m.acc_sum)
            self._last_ghm['reg_counts'] = counts
        loss_cls, loss_pts = [], []
        for b in range(B):
            if cls_type == 'GHMC':
                lc = _LossSumFn.apply(ops.ghmc, x_all[b], labels_l[b], lw_l[b], self.loss_cls.edges, cls_bw[b])
                loss_cls.append(lc / cls_tot[b] * self.loss_cls_cfg['loss_weight'])
            else:
                lc = _LossSumFn.apply(cls_op, cls[b].contiguous(), labels_l[b], lw_l[b], *cls_args)
                loss_cls.append(self.loss_cls_cfg.get('loss_weight', 1.0) * lc / cls_avg)
            if reg_type == 'GHMR':
                lp = _LossSumFn.apply(ops.ghmr, p_all[b], gp_l[b], pw_l[b], row_inv, rc['mu'], self.loss_reg.edges, reg_bw[b])
                loss_pts.append(lp / reg_tot[b] * rc['loss_weight'])
            else:
                lp = _LossSumFn.apply(reg_op, pred[b].contiguous(), gp_l[b], pw_l[b], *reg_args)
                loss_pts.append(rc.get('loss_weight', 1.0) * lp / num_total_pos)
        self._last_targets = dict(labels=labels_l, label_weights=lw_l, gt_pts=gp_l, pts_weights=pw_l)
        return dict(loss_cls=loss_cls, loss_pts=loss_pts)

    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def get_bboxes(self, cls_outs, pts_outs, img_metas, cfg=None, rescale=False, with_nms=True, return_all=False):
        """p2p_head.py:330-423: per image (pseudo boxes (m,5), labels (m,))."""
        cfg = CfgNode(cfg) if cfg is not None else self.test_cfg
        cls_out, pts_out = cls_outs[0], pts_outs[0]
        if not cls_out.is_cuda:
            raise RuntimeError('P2PHead runs on CUDA tensors only; there is no CPU fallback')
        if not with_nms:
            raise NotImplementedError('with_nms=False')
        dev = cls_out.device
        B = cls_out.shape[0]
        img_hw = torch.tensor(np.array([m['img_shape'][:2] for m in img_metas], dtype=np.int32), device=dev)
        scale_xy = None
        if rescale:
            scale_xy = torch.tensor(np.array([m['scale_factor'][:2] for m in img_metas], dtype=np.float32), device=dev)
        multi = len(self.strides) > 1
        if multi:
            plan = ops.p2p_chunk_plan([c.shape[-2:] for c in cls_outs], self.num_points, cfg.get('nms_pre', -1))
            if plan['L'] * plan['P'] > ops.NMS_WIDE_MAX_POINTS:
                raise RuntimeError(
                    f"P2PHead over {plan['L']} levels: nms_pre={cfg.get('nms_pre', -1)} keeps {plan['P']} of the {plan['chunk']} rows of "
                    f"each of the {plan['L']} chunks, {plan['L'] * plan['P']} NMS points per image; the NMS takes at most "
                    f"{ops.NMS_WIDE_MAX_POINTS}: set test_cfg.nms_pre to at most {ops.NMS_WIDE_MAX_POINTS // plan['L']}")
            # p2p_head.py:355-381: the level-major rows cut into len(strides) equal chunks, top nms_pre per chunk (ops.p2p_chunk_plan);
            # up to 8192 candidates go to NMS
            idx, pts, scores = ops.p2p_decode_topk_levels(
                [ops.to_nhwc(c).contiguous() for c in cls_outs], [ops.to_nhwc(p).contiguous() for p in pts_outs], self.strides,
                self.num_classes, self.num_points, self.point_anchor.to(dev), self.pts_gamma, img_hw, cfg.get('nms_pre', -1),
                scale_xy, softmax=not self.use_sigmoid_cls)
        else:
            cmap, rmap = ops.to_nhwc(cls_out).contiguous(), ops.to_nhwc(pts_out).contiguous()
            # p2p_head.py:363-372: sigmoid scores, or the softmax over C+1 columns of which NMS sees the C foreground ones
            decode = ops.p2p_decode_topk if self.use_sigmoid_cls else ops.p2p_decode_topk_softmax
            idx, pts, scores = decode(cmap, rmap, self.num_classes, self.num_points, self.point_anchor.to(dev), self.strides[0],
                                      self.pts_gamma, img_hw, cfg.get('nms_pre', -1), scale_xy)
        wh = cfg.get('pseudo_wh', (16, 16))
        check_split_thr(cfg.get('nms'))
        nms = parse_nms_cfg(cfg.get('nms'))
        if nms.class_agnostic:
            raise NotImplementedError('P2PHead: class_agnostic NMS is not implemented')
        cnt, det, lab, keep, cc = run_multiclass_nms(pts, scores, cfg.get('score_thr'), nms, cfg.get('max_per_img'), wh, wide=multi)
        cnt_h = cnt.cpu().tolist()
        res = []
        for b in range(B):
            m = cnt_h[b]
            d = det[b, :m]
            cxcy = torch.stack([(d[:, 0] + d[:, 2]) / 2, (d[:, 1] + d[:, 3]) / 2], -1)      # bbox_xyxy_to_cxcywh
            half = cxcy.new_tensor(wh) / 2
            res.append((torch.cat([cxcy - half, cxcy + half, d[:, 4:5]], -1), lab[b, :m].long()))
        if return_all:
            return res, dict(topk_idx=idx, pts=pts, scores=scores, keep=keep, count=cnt, cand_count=cc)
        return res

    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def bbox_mapping_back(bboxes, img_shape, scale_factor, flip, flip_direction, tile_offset=None):
        """core/bbox/transforms.py:62-85 (incl. the reference's tile_offset extension)."""
        b = bboxes
        if flip:
            f = b.clone()
            if flip_direction in ('horizontal', 'diagonal'):
                f[..., 0::4] = img_shape[1] - b[..., 2::4]
                f[..., 2::4] = img_shape[1] - b[..., 0::4]
            if flip_direction in ('vertical', 'diagonal'):
                f[..., 1::4] = img_shape[0] - b[..., 3::4]
                f[..., 3::4] = img_shape[0] - b[..., 1::4]
            b = f
        b = b.view(-1, 4) / b.new_tensor(scale_factor)
        if tile_offset is not None:
            dx, dy = tile_offset
            b[:, [0, 2]] += dx
            b[:, [1, 3]] += dy
        return b.view(bboxes.shape)

    @torch.no_grad()
    def aug_test_bboxes(self, feats, img_metas, rescale=False):
        """test-time-aug / cropped-tile merge (p2p_head.py:487-572, dense_test_mixins.py:173-204): per aug run get_bboxes
        (with NMS), map the kept boxes back, then a SECOND multiclass NMS over the union (ptb_multiclass_nms_boxes)."""
        aug_bboxes, aug_scores = [], []
        for x, img_meta in zip(feats, img_metas):
            outs = self.forward(x)
            boxes5, labels = self.get_bboxes(*outs, img_meta, cfg=self.test_cfg, rescale=False, with_nms=True)[0]
            sc = boxes5.new_zeros((boxes5.shape[0], self.num_classes))
            sc[torch.arange(boxes5.shape[0], device=boxes5.device), labels] = boxes5[:, 4]
            m = img_meta[0]
            aug_bboxes.append(self.bbox_mapping_back(boxes5[:, :4], m['img_shape'], m['scale_factor'], m.get('flip', False),
                                                     m.get('flip_direction', 'horizontal'), m.get('tile_offset', None)))
            aug_scores.append(sc)
        boxes = torch.cat(aug_bboxes).contiguous()
        scores = torch.cat(aug_scores).contiguous()
        if not self.use_sigmoid_cls:
            # p2p_head.py:549-556: the reference pads a background column only in sigmoid mode, so in softmax mode
            # multiclass_nms takes the last real class (C-1) for the background and drops it from the merged detections
            scores = scores[:, :-1].contiguous()
        cfg = self.test_cfg
        if boxes.shape[0] == 0 or scores.shape[1] == 0:
            return [(boxes.new_zeros((0, 5)), boxes.new_zeros((0,), dtype=torch.long))]
        check_split_thr(cfg.get('nms'))
        nms = parse_nms_cfg(cfg.get('nms'))
        if nms.class_agnostic:
            raise NotImplementedError('P2PHead: class_agnostic NMS is not implemented')
        cnt, det, lab, _, _ = run_multiclass_nms(boxes[None], scores[None], cfg.get('score_thr'), nms, cfg.get('max_per_img'))
        n = int(cnt[0])
        d = det[0, :n].clone()
        if not rescale:
            d[:, :4] *= d.new_tensor(img_metas[0][0]['scale_factor'])
        return [(d, lab[0, :n].long())]
