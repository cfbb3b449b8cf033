"""FCOSHead — the reference's anchor-free FCOS head (mmdet/models/dense_heads/fcos_head.py, anchor_free_head.py) over the sm_90a kernels.

Same constructor keywords, state_dict keys (cls_convs.i.conv / .gn, reg_convs.i.*, conv_cls, conv_reg, conv_centerness, scales.i.scale)
and method outputs as the reference.  What runs where:
  towers        layers.tower per level: the wgmma conv with fused GroupNorm at inference, the tensor-core training tower under autograd
  output convs  inference: the wgmma conv (ops.conv_tc_f16), conv_centerness in the same launch as the conv sharing its input
                (conv_cls, or conv_reg with centerness_on_reg); training: cuDNN fp32 under autograd, TF32 off
  loss          ptb_fcos_targets (every image and point, GTs in CSR layout), the positive count and centerness sum on the device,
                FocalLoss (ptb_sigmoid_focal_fwd_bwd), the centerness-weighted IoU / GIoU loss and the centerness BCE on the fixed-order
                sum kernels.  No host synchronisation and no compaction of the positives: negative rows weigh 0.
  decode        ptb_fcos_decode (per-level top nms_pre keys, gather, distance2bbox with clipping), then one multiclass NMS over the
                batch: the batched multiclass kernels up to 4096 candidates per image, ptb_batched_nms above.
CUDA tensors only; there is no CPU path.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .dist import reduce_mean_
from .layers import ConvModule, PackedWeightsMixin, bias_init_with_prob, normal_init_, no_tf32, tower, tower_path, _packed_tc, \
    _packed_tc_stacked
from .p2p_head import _LossSumFn
from .post_processing import check_split_thr, parse_nms_cfg, run_multiclass_nms
from .registry import CfgNode

INF = 1e8
MAX_CLS_CTR_CHANNELS = 512        # widest output of one wgmma conv launch: conv_cls and conv_centerness share it
MULTICLASS_NMS_MAX = 4096         # candidates per image of the batched multiclass NMS kernels
FLT_LOWEST = -3.4028234663852886e38


class Scale(nn.Module):
    """mmcv.cnn.Scale: a learnable scalar `scale`, forward x * scale."""

    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))

    def forward(self, x):
        return x * self.scale


class LevelPoints(list):
    """get_points' per-level (H*W, 2) points, carrying the feature map sizes they were made for (get_targets needs them)."""

    def __init__(self, points, featmap_sizes):
        super().__init__(points)
        self.featmap_sizes = [tuple(int(v) for v in s) for s in featmap_sizes]


def _pinned(rows, dtype, device):
    """a small host table on the device without a synchronising copy"""
    return torch.tensor(rows, dtype=dtype).pin_memory().to(device, non_blocking=True)


class FCOSHead(PackedWeightsMixin, nn.Module):
    def __init__(self, num_classes, in_channels, regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)),
                 center_sampling=False, center_sample_radius=1.5, norm_on_bbox=False, centerness_on_reg=False,
                 loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                 loss_bbox=dict(type='IoULoss', loss_weight=1.0),
                 loss_centerness=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True),
                 init_cfg=dict(type='Normal', layer='Conv2d', std=0.01,
                               override=dict(type='Normal', name='conv_cls', std=0.01, bias_prob=0.01)),
                 feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64), dcn_on_last_conv=False, conv_bias='auto',
                 conv_cfg=None, train_cfg=None, test_cfg=None):
        super().__init__()
        if norm_cfg is None:
            raise NotImplementedError('FCOSHead(norm_cfg=None): bias + ReLU towers (the fcos_standard configs) are not implemented; '
                                      'the towers run conv + GroupNorm(32) + ReLU')
        if dict(norm_cfg).get('type') != 'GN' or dict(norm_cfg).get('num_groups') != 32:
            raise NotImplementedError(f'FCOSHead norm_cfg={norm_cfg}: the tensor-core towers take GroupNorm with 32 groups')
        if dcn_on_last_conv:
            raise NotImplementedError('FCOSHead(dcn_on_last_conv=True): deformable convolution is not implemented')
        if conv_bias is True:
            raise NotImplementedError('FCOSHead(conv_bias=True) with GroupNorm: the tensor-core towers take convs without bias')
        if conv_cfg is not None:
            raise NotImplementedError(f'FCOSHead conv_cfg={conv_cfg}: plain Conv2d towers are implemented')
        if feat_channels != 256:
            raise NotImplementedError(f'FCOSHead(feat_channels={feat_channels}): the tensor-core towers take 256 channels')
        if num_classes + 1 > MAX_CLS_CTR_CHANNELS:
            raise NotImplementedError(f'FCOSHead(num_classes={num_classes}): conv_cls and conv_centerness share one conv launch of at most '
                                      f'{MAX_CLS_CTR_CHANNELS} channels, so at most {MAX_CLS_CTR_CHANNELS - 1} classes')
        if len(strides) != len(regress_ranges) or not 1 <= len(strides) <= ops.FCOS_MAX_LEVELS:
            raise ValueError(f'FCOSHead: {len(strides)} strides and {len(regress_ranges)} regress ranges; one range per level, '
                             f'1 to {ops.FCOS_MAX_LEVELS} levels')
        lc, lb, lk = dict(loss_cls), dict(loss_bbox), dict(loss_centerness)
        if lc.get('type') != 'FocalLoss' or not lc.get('use_sigmoid', True):
            raise NotImplementedError(f"FCOSHead loss_cls {lc.get('type')}: FocalLoss (use_sigmoid=True) is implemented")
        if lb.get('type') not in ('IoULoss', 'GIoULoss'):
            raise NotImplementedError(f"FCOSHead loss_bbox {lb.get('type')}: IoULoss and GIoULoss are implemented")
        if lk.get('type') != 'CrossEntropyLoss' or not lk.get('use_sigmoid', False) or lk.get('class_weight') is not None:
            raise NotImplementedError(f"FCOSHead loss_centerness {lk}: CrossEntropyLoss(use_sigmoid=True) without class_weight is "
                                      f"implemented")
        for c in (lc, lb, lk):
            if c.get('reduction', 'mean') != 'mean':
                raise NotImplementedError(f"FCOSHead {c['type']}(reduction={c['reduction']!r}): 'mean' is implemented")
        self.num_classes = self.cls_out_channels = num_classes
        self.in_channels, self.feat_channels, self.stacked_convs = in_channels, feat_channels, stacked_convs
        self.strides, self.regress_ranges = list(strides), regress_ranges
        self.center_sampling, self.center_sample_radius = center_sampling, center_sample_radius
        self.norm_on_bbox, self.centerness_on_reg = norm_on_bbox, centerness_on_reg
        self.dcn_on_last_conv, self.conv_bias, self.conv_cfg, self.norm_cfg = dcn_on_last_conv, conv_bias, conv_cfg, norm_cfg
        self.focal = (float(lc.get('gamma', 2.0)), float(lc.get('alpha', 0.25)))
        self.w_cls, self.w_bbox, self.w_ctr = (float(c.get('loss_weight', 1.0)) for c in (lc, lb, lk))
        if lb['type'] == 'IoULoss':
            # iou_loss: bbox_overlaps at its default eps 1e-6, then clamp(min=IoULoss.eps); GIoU: bbox_overlaps(eps=GIoULoss.eps)
            self.box_mode = ops.FCOS_BOX_LOSS_MODES['IoULoss_linear' if lb.get('linear', False) else 'IoULoss']
        else:
            self.box_mode = ops.FCOS_BOX_LOSS_MODES['GIoULoss']
        self.box_eps = float(lb.get('eps', 1e-6))
        self.train_cfg = CfgNode(train_cfg) if train_cfg is not None else None     # its assigner is not used, as in the reference
        self.test_cfg = CfgNode(test_cfg) if test_cfg is not None else None
        self.init_cfg = init_cfg
        self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList()
        for i in range(stacked_convs):
            chn = in_channels if i == 0 else feat_channels
            self.cls_convs.append(ConvModule(chn, feat_channels, 3, 1, 1, norm_cfg=norm_cfg, bias=conv_bias))
            self.reg_convs.append(ConvModule(chn, feat_channels, 3, 1, 1, norm_cfg=norm_cfg, bias=conv_bias))
        self.conv_cls = nn.Conv2d(feat_channels, num_classes, 3, padding=1)
        self.conv_reg = nn.Conv2d(feat_channels, 4, 3, padding=1)
        self.conv_centerness = nn.Conv2d(feat_channels, 1, 3, padding=1)
        self.scales = nn.ModuleList([Scale(1.0) for _ in self.strides])
        self.init_weights()
        self._init_packed_hooks()
        self._dev_tables = {}

    def init_weights(self):
        """init_cfg: Normal(std=0.01) on every Conv2d with bias 0, conv_cls' bias from bias_prob=0.01"""
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                normal_init_(m, 0.01, 0.0)
        nn.init.constant_(self.conv_cls.bias, bias_init_with_prob(0.01))

    # ------------------------------------------------------------------------------------------------
    def _out_tc(self, pc, pr):
        """inference output convs on the wgmma conv: two launches, the centerness channel appended to the conv sharing its input"""
        C = self.num_classes
        if self.centerness_on_reg:
            packs, bias = _packed_tc_stacked((self.conv_reg, self.conv_centerness))
            yr = ops.conv_tc_f16(pr[0], pr[1], packs, 9, 5, bias=bias)
            yc = ops.conv_tc_f16(pc[0], pc[1], _packed_tc(self.conv_cls, 9), 9, C, bias=self.conv_cls.bias.detach())
            return yc[..., :C], yr[..., :4], yr[..., 4:5]
        packs, bias = _packed_tc_stacked((self.conv_cls, self.conv_centerness))
        yc = ops.conv_tc_f16(pc[0], pc[1], packs, 9, C + 1, bias=bias)
        yr = ops.conv_tc_f16(pr[0], pr[1], _packed_tc(self.conv_reg, 9), 9, 4, bias=self.conv_reg.bias.detach())
        return yc[..., :C], yr[..., :4], yc[..., C:C + 1]

    def forward_single(self, x, scale, stride):
        """fcos_head.py:131-160: (cls_score, bbox_pred, centerness) of one level.  x: fp32, or an fp16 / bf16 map taken as it is."""
        info = {}
        if tower_path([*self.cls_convs, *self.reg_convs], x,
                      also=(self.conv_cls, self.conv_reg, self.conv_centerness, scale)) == 'wgmma-f16x2':
            pc = tower(self.cls_convs, x, info, want='f16pair')
            pr = tower(self.reg_convs, x, info, want='f16pair')
            self._record_tower(info)
            out = [t.permute(0, 3, 1, 2) for t in self._out_tc(pc, pr)]
        else:
            fc, fr = tower(self.cls_convs, x, info), tower(self.reg_convs, x, info)
            self._record_tower(info)
            with no_tf32(), torch.autocast('cuda', enabled=False):
                out = [self.conv_cls(fc), self.conv_reg(fr), self.conv_centerness(fr if self.centerness_on_reg else fc)]
        cls_score, bbox_pred, centerness = out
        bbox_pred = scale(bbox_pred).float()
        if self.norm_on_bbox:
            bbox_pred = F.relu(bbox_pred)
            if not self.training:
                bbox_pred = bbox_pred * stride
        else:
            bbox_pred = bbox_pred.exp()
        return cls_score, bbox_pred, centerness

    def forward(self, feats):
        outs = [self.forward_single(x, s, st) for x, s, st in zip(feats, self.scales, self.strides)]
        return tuple(list(t) for t in zip(*outs))

    def forward_train(self, x, img_metas, gt_bboxes, gt_labels=None, gt_bboxes_ignore=None, proposal_cfg=None, **kwargs):
        """base_dense_head.py:22-59"""
        outs = self(x)
        losses = self.loss(*outs, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=gt_bboxes_ignore)
        if proposal_cfg is None:
            return losses
        return losses, self.get_bboxes(*outs, img_metas, cfg=proposal_cfg)

    # ------------------------------------------------------------------------------------------------
    def get_points(self, featmap_sizes, dtype, device, flatten=False):
        """fcos_head.py:472-482: per level (H*W, 2) points x * stride + stride // 2, y likewise"""
        pts = []
        for (h, w), s in zip(featmap_sizes, self.strides):
            x = torch.arange(int(w), device=device).to(dtype)
            y = torch.arange(int(h), device=device).to(dtype)
            yy, xx = torch.meshgrid(y, x, indexing='ij')
            pts.append(torch.stack((xx.reshape(-1) * s, yy.reshape(-1) * s), dim=-1) + s // 2)
        return LevelPoints(pts, featmap_sizes)

    def _tables(self, device):
        key = str(device)
        if key not in self._dev_tables:
            ranges = _pinned([[float(v) for v in r] for r in self.regress_ranges], torch.float32, device)
            radius = _pinned([float(np.float32(s * self.center_sample_radius)) for s in self.strides], torch.float32, device) \
                if self.center_sampling else None
            self._dev_tables[key] = (ranges, radius)
        return self._dev_tables[key]

    def _flat_targets(self, featmap_sizes, gt_bboxes, gt_labels, device):
        """(labels (N,), bbox_targets (N, 4)) of the whole batch in the flattened rows' order (level, image, y, x)"""
        B = len(gt_bboxes)
        n = [int(g.numel()) // int(g.shape[-1]) if g.numel() else 0 for g in gt_bboxes]
        gt = torch.cat([g.reshape(k, -1)[:, :4].to(device).float() for g, k in zip(gt_bboxes, n) if k]).contiguous() if sum(n) else None
        gl = torch.cat([l.reshape(-1).to(device).long() for l, k in zip(gt_labels, n) if k]).contiguous() if sum(n) else None
        off = _pinned(np.concatenate([[0], np.cumsum(n)]).astype(np.int32).tolist(), torch.int32, device)
        ranges, radius = self._tables(device)
        return ops.fcos_targets(featmap_sizes, self.strides, B, gt, gl, off, ranges, radius, self.norm_on_bbox, self.num_classes)

    def get_targets(self, points, gt_bboxes_list, gt_labels_list):
        """fcos_head.py:484-550: per level the labels (B*H*W,) and bbox_targets (B*H*W, 4) of all images, image after image.
        `points` as get_points returns them."""
        sizes = getattr(points, 'featmap_sizes', None)
        if sizes is None:
            raise ValueError('FCOSHead.get_targets takes the points of FCOSHead.get_points (they carry the feature map sizes)')
        labels, targets = self._flat_targets(sizes, gt_bboxes_list, gt_labels_list, points[0].device)
        rows = [len(gt_bboxes_list) * h * w for h, w in sizes]
        return list(labels.split(rows)), list(targets.split(rows))

    def loss(self, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=None):
        """fcos_head.py:163-260 -> dict(loss_cls, loss_bbox, loss_centerness)"""
        assert len(cls_scores) == len(bbox_preds) == len(centernesses) == len(self.strides)
        if not cls_scores[0].is_cuda:
            raise RuntimeError('FCOSHead runs on CUDA tensors only; there is no CPU fallback')
        dev = cls_scores[0].device
        B, C = cls_scores[0].shape[0], self.cls_out_channels
        featmap_sizes = [tuple(int(v) for v in c.shape[-2:]) for c in cls_scores]
        with torch.autocast('cuda', enabled=False):
            labels, targets = self._flat_targets(featmap_sizes, gt_bboxes, gt_labels, dev)
            flat_cls = torch.cat([c.float().permute(0, 2, 3, 1).reshape(-1, C) for c in cls_scores]).contiguous()
            flat_reg = torch.cat([r.float().permute(0, 2, 3, 1).reshape(-1, 4) for r in bbox_preds]).contiguous()
            flat_ctr = torch.cat([k.float().permute(0, 2, 3, 1).reshape(-1) for k in centernesses]).contiguous()
            sums = reduce_mean_(ops.fcos_norm_sums(labels, targets, self.num_classes))
            num_pos, ctr_denorm = sums[0].clamp(min=1.0), sums[1].clamp(min=1e-6)
            loss_cls = _LossSumFn.apply(ops.sigmoid_focal, flat_cls, labels, None, *self.focal) / num_pos * self.w_cls
            loss_bbox = _LossSumFn.apply(ops.fcos_bbox_loss, flat_reg, targets, labels, featmap_sizes, self.strides, B, self.num_classes,
                                         self.box_mode, 1e-6, self.box_eps) / ctr_denorm * self.w_bbox
            loss_ctr = _LossSumFn.apply(ops.fcos_centerness_loss, flat_ctr, targets, labels, self.num_classes) / num_pos * self.w_ctr
        self._last_targets = dict(labels=labels, bbox_targets=targets, norm_sums=sums)
        return dict(loss_cls=loss_cls, loss_bbox=loss_bbox, loss_centerness=loss_ctr)

    # ------------------------------------------------------------------------------------------------
    def _decode(self, cls_scores, bbox_preds, centernesses, img_metas, cfg, rescale):
        """ptb_fcos_decode of the batch: idx (B,R), boxes (B,R,4), scores (B,R,C), centerness (B,R)"""
        if not cls_scores[0].is_cuda:
            raise RuntimeError('FCOSHead runs on CUDA tensors only; there is no CPU fallback')
        dev = cls_scores[0].device
        nhwc = lambda ts: [ops.to_nhwc(t.detach().float()).contiguous() for t in ts]
        img_hw = _pinned([[float(m['img_shape'][0]), float(m['img_shape'][1])] for m in img_metas], torch.float32, dev)
        sf = None
        if rescale:
            sf = _pinned([(np.asarray(m['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32)).tolist() for m in img_metas],
                         torch.float32, dev)
        return ops.fcos_decode(nhwc(cls_scores), nhwc(bbox_preds), nhwc(centernesses), self.strides, self.num_classes, img_hw,
                               int(cfg.get('nms_pre', -1)), sf)

    def _nms(self, boxes, scores, factors, cfg):
        """multiclass_nms (bbox_nms.py:7-94) with score_factors of every image of the batch in one launch: the raw scores pass
        score_thr, the products rank.  -> count (B,), det (B, K, 5), labels (B, K) int32"""
        check_split_thr(cfg.get('nms'))
        nms = parse_nms_cfg(cfg.get('nms'))
        if nms.kind != 'nms':
            raise NotImplementedError(f"FCOSHead test_cfg.nms type {nms.kind}: 'nms' is implemented")
        if nms.class_agnostic:
            raise NotImplementedError('FCOSHead: class_agnostic NMS is not implemented')
        max_num = int(cfg.get('max_per_img', -1))
        if not 0 < max_num <= 1024:
            raise NotImplementedError(f'FCOSHead test_cfg.max_per_img={max_num}: 1 to 1024 is implemented')
        thr = float(cfg.get('score_thr'))
        B, P, C = scores.shape
        valid = scores > thr
        prod = scores * factors[..., None]
        if P <= MULTICLASS_NMS_MAX:
            s = torch.where(valid, prod, prod.new_full((), float('-inf'))).contiguous()
            return run_multiclass_nms(boxes.contiguous(), s, FLT_LOWEST, nms, max_num)[:3]
        # mmcv batched_nms over the candidates in (row, class) order, compacted on the device: candidate i of image b goes to row
        # b * N + (its rank among the image's candidates), the rest to one spare row past the batch
        flat = valid.reshape(B, P * C)
        count = flat.sum(1, dtype=torch.int32)
        N = P * C
        if N > ops.BATCHED_NMS_MAX_ROWS:
            N = int(count.max())                     # the one host read of this route: the row bound of the NMS launch
            if N > ops.BATCHED_NMS_MAX_ROWS:
                raise NotImplementedError(f'FCOSHead: {N} candidates of one image pass score_thr={thr} ({P} boxes x {C} classes); '
                                          f'the NMS takes at most {ops.BATCHED_NMS_MAX_ROWS}')
            N = max(N, 1)
        base = torch.arange(B, device=boxes.device)[:, None] * N
        dst = torch.where(flat, base + flat.cumsum(1) - 1, torch.full_like(base, B * N)).reshape(-1)
        out_b = boxes.new_zeros((B * N + 1, 4))
        out_s = boxes.new_zeros((B * N + 1,))
        out_l = torch.zeros((B * N + 1,), dtype=torch.int32, device=boxes.device)
        out_b.index_copy_(0, dst, boxes[:, :, None, :].expand(B, P, C, 4).reshape(-1, 4))
        out_s.index_copy_(0, dst, prod.reshape(-1))
        out_l.index_copy_(0, dst, torch.arange(C, dtype=torch.int32, device=boxes.device).repeat(B * P))
        cnt, det, lab, _ = ops.batched_nms(out_b[:B * N].view(B, N, 4), out_s[:B * N].view(B, N), out_l[:B * N].view(B, N), count, nms.iou,
                                           10000, max_num)
        return cnt, det[:, :max_num], lab[:, :max_num]

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, centernesses, img_metas, cfg=None, rescale=False, with_nms=True):
        """fcos_head.py:263-470: per image (det_bboxes (n, 5), det_labels (n,)), or with_nms=False (bboxes, scores with the background
        column, centerness)"""
        cfg = CfgNode(cfg) if cfg is not None else self.test_cfg
        _, boxes, scores, ctr = self._decode(cls_scores, bbox_preds, centernesses, img_metas, cfg, rescale)
        B = boxes.shape[0]
        if not with_nms:
            padded = torch.cat([scores, scores.new_zeros(scores.shape[:2] + (1,))], -1)
            return [(boxes[b], padded[b], ctr[b]) for b in range(B)]
        cnt, det, lab = self._nms(boxes, scores, ctr, cfg)
        cnt = cnt.cpu().tolist()
        return [(det[b, :cnt[b]], lab[b, :cnt[b]].long()) for b in range(B)]

    def simple_test(self, feats, img_metas, rescale=False):
        """base_dense_head.simple_test -> simple_test_bboxes: per image (det_bboxes, det_labels)"""
        return self.get_bboxes(*self.forward(feats), img_metas, rescale=rescale)

    def aug_test(self, feats, img_metas, rescale=False):
        """anchor_free_head.py:324-340"""
        return self.aug_test_bboxes(feats, img_metas, rescale=rescale)

    @torch.no_grad()
    def aug_test_bboxes(self, feats, img_metas, rescale=False):
        """dense_test_mixins.py:38-108 on the device: augs whose feature maps agree in shape run as one batch through the towers and the
        decode (get_bboxes(with_nms=False)); ptb_proposal_map_back maps every aug's boxes back (flip, / scale_factor, + tile_offset) and
        concatenates them in aug order (merge_aug_bboxes); one multiclass NMS with the concatenated centerness as score_factors."""
        cfg = self.test_cfg
        A = len(feats)
        groups = {}
        for a, x in enumerate(feats):
            assert len(img_metas[a]) == 1, 'aug_test takes one image per aug'
            groups.setdefault(tuple(tuple(t.shape) for t in x), []).append(a)
        per_aug = [None] * A
        for augs in groups.values():
            batch = [torch.cat([feats[a][l] for a in augs]) for l in range(len(feats[augs[0]]))]
            _, boxes, scores, ctr = self._decode(*self.forward(batch), [img_metas[a][0] for a in augs], cfg, False)
            for i, a in enumerate(augs):
                per_aug[a] = (boxes[i], scores[i], ctr[i])
        rows = [int(p[0].shape[0]) for p in per_aug]
        N = max(rows)
        dev = per_aug[0][0].device
        det = torch.zeros((A, N, 5), dtype=torch.float32, device=dev)
        for a, (bx, _, _) in enumerate(per_aug):
            det[a, :rows[a], :4] = bx
        meta = ops.aug_meta([m[0] for m in img_metas], [0] * A, [0] * A, dev)
        mapped, _ = ops.proposal_map_back(det, _pinned(rows, torch.int32, dev), meta, A)
        total = sum(rows)
        boxes = mapped[0, :total, :4]
        scores = torch.cat([p[1] for p in per_aug])
        ctr = torch.cat([p[2] for p in per_aug])
        cnt, det, lab = self._nms(boxes[None], scores[None], ctr[None], cfg)
        n = int(cnt[0])
        d = det[0, :n].clone()
        if not rescale:
            d[:, :4] *= d.new_tensor(img_metas[0][0]['scale_factor'])
        return [(d, lab[0, :n].long())]
