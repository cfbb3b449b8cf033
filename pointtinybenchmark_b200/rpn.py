"""Dense-anchor proposal path (SURVEY.md §8f rank 4, BASELINE.json configs[3]) — host-side mirror of the reference pieces around
ptb_rpn_proposals:

  AnchorGenerator   mmdet/core/anchor/anchor_generator.py:9-330 (base anchors, grid anchors, valid flags; same ctor kwargs).  The base
                    anchors are input-independent (a few floats per level): computed once with torch CPU ops in the reference's
                    order, so they are bit-identical; the H*W*A grid anchors are NOT materialised on the proposal path — the decode
                    kernel forms `base[a] + shift(x, y)` on the fly — `grid_anchors` exists for callers that want the tensor
                    (e.g. to feed MaxIoUAssigner).
  RPNProposals      the `get_bboxes` of RPNHead (AnchorHead.get_bboxes, anchor_head.py:551-590 -> RPNHead._get_bboxes,
                    rpn_head.py:78-186): same arguments (cls_scores, bbox_preds, img_metas, cfg, rescale, with_nms), same result
                    (list of (n, 5) tensors), one library call for the whole batch instead of the per-level / per-image Python loop.
There is no CPU path: CUDA tensors only.
"""
import numpy as np
import torch

from . import ops
from .registry import CfgNode


def _as_wh(stride):
    """a stride given as one number means the same step along x and y"""
    if isinstance(stride, (tuple, list)):
        if len(stride) != 2:
            raise ValueError(f'a stride is one number or an (x, y) pair, got {stride!r}')
        return int(stride[0]), int(stride[1])
    return int(stride), int(stride)


class AnchorGenerator:
    """Same constructor keywords, attributes and method names as the reference generator (anchor_generator.py:9-330), organised around
    one table per pyramid level: `strides[l]` = (step_x, step_y), `base_sizes[l]`, `base_anchors[l]` = (A, 4) fp32 boxes around the
    level's anchor centre.  Only the base-anchor arithmetic has to follow the reference operation by operation (it is the one place where
    fp32 rounding enters: sqrt of the ratios, two products per side); grid anchors are `base + (x * step_x, y * step_y)` — one exact
    integer-valued shift and one fp32 add per coordinate however the shift grid is laid out — and the valid flags are index comparisons."""

    def __init__(self, strides, ratios, scales=None, base_sizes=None, scale_major=True, octave_base_scale=None, scales_per_octave=None,
                 centers=None, center_offset=0.):
        self.strides = [_as_wh(st) for st in strides]
        n_lvl = len(self.strides)
        if not 0 <= center_offset <= 1:
            raise ValueError(f'center_offset must lie in [0, 1] (fraction of the base size), got {center_offset}')
        if centers is not None and center_offset != 0:
            raise AssertionError(f'explicit centers ({centers}) and a non-zero center_offset exclude each other')
        if centers is not None and len(centers) != n_lvl:
            raise AssertionError(f'{len(centers)} centers for {n_lvl} levels')
        self.base_sizes = [min(st) for st in self.strides] if base_sizes is None else list(base_sizes)
        if len(self.base_sizes) != n_lvl:
            raise AssertionError(f'{len(self.base_sizes)} base sizes for {n_lvl} strides')
        octave = octave_base_scale is not None and scales_per_octave is not None
        if octave == (scales is not None):
            raise AssertionError('give either `scales` or (`octave_base_scale`, `scales_per_octave`), not both and not neither')
        if octave:
            steps = np.array([2 ** (k / scales_per_octave) for k in range(scales_per_octave)])
            self.scales = torch.Tensor(steps * octave_base_scale)
        else:
            self.scales = torch.Tensor(scales)
        self.ratios = torch.Tensor(ratios)
        self.octave_base_scale, self.scales_per_octave = octave_base_scale, scales_per_octave
        self.scale_major, self.centers, self.center_offset = scale_major, centers, center_offset
        self.base_anchors = self.gen_base_anchors()

    num_levels = property(lambda self: len(self.strides))
    num_base_anchors = property(lambda self: [int(t.shape[0]) for t in self.base_anchors])

    def gen_base_anchors(self):
        return [self.gen_single_level_base_anchors(size, self.scales, self.ratios, self.centers[lvl] if self.centers is not None else None)
                for lvl, size in enumerate(self.base_sizes)]

    def gen_single_level_base_anchors(self, base_size, scales, ratios, center=None):
        """(A, 4) boxes of side base_size * scale, aspect h / w = ratio, around the level's centre — the reference's fp32 operation order
        (anchor_generator.py:112-151): sqrt(ratio) and its reciprocal, then (size * ratio_term) * scale, or scale first when not scale_major."""
        cx, cy = center if center is not None else (self.center_offset * base_size, self.center_offset * base_size)
        tall = torch.sqrt(ratios)
        wide = 1 / tall
        if self.scale_major:
            half_w = 0.5 * (base_size * wide[:, None] * scales[None, :]).view(-1)
            half_h = 0.5 * (base_size * tall[:, None] * scales[None, :]).view(-1)
        else:
            half_w = 0.5 * (base_size * scales[:, None] * wide[None, :]).view(-1)
            half_h = 0.5 * (base_size * scales[:, None] * tall[None, :]).view(-1)
        return torch.stack([cx - half_w, cy - half_h, cx + half_w, cy + half_h], dim=-1)

    def single_level_grid_anchors(self, base_anchors, featmap_size, stride=(16, 16), device='cuda'):
        """(H*W*A, 4): cell (y, x) major, base anchor minor — the order of the head's permute(0, 2, 3, 1) logits."""
        rows, cols = featmap_size
        step_x, step_y = stride
        xs = (torch.arange(cols, device=device) * step_x).to(base_anchors.dtype)
        ys = (torch.arange(rows, device=device) * step_y).to(base_anchors.dtype)
        shift = torch.stack([xs[None, :].expand(rows, cols), ys[:, None].expand(rows, cols)], dim=-1).repeat(1, 1, 2)      # (H, W, 4) = x, y, x, y
        return (shift[:, :, None, :] + base_anchors[None, None, :, :]).reshape(-1, 4)

    def grid_anchors(self, featmap_sizes, device='cuda'):
        if len(featmap_sizes) != self.num_levels:
            raise AssertionError(f'{len(featmap_sizes)} feature maps for {self.num_levels} levels')
        return [self.single_level_grid_anchors(self.base_anchors[lvl].to(device), size, self.strides[lvl], device=device)
                for lvl, size in enumerate(featmap_sizes)]

    def valid_flags(self, featmap_sizes, pad_shape, device='cuda'):
        """per level a bool (H*W*A,): the anchors of the cells whose index is below ceil(padded image extent / stride)
        (anchor_generator.py:272-330)"""
        if len(featmap_sizes) != self.num_levels:
            raise AssertionError(f'{len(featmap_sizes)} feature maps for {self.num_levels} levels')
        img_h, img_w = pad_shape[:2]
        flags = []
        for lvl, (rows, cols) in enumerate(featmap_sizes):
            step_x, step_y = self.strides[lvl]
            ok_cols = min(-(-int(img_w) // step_x) if float(img_w).is_integer() else int(np.ceil(img_w / step_x)), cols)
            ok_rows = min(-(-int(img_h) // step_y) if float(img_h).is_integer() else int(np.ceil(img_h / step_y)), rows)
            cell_ok = (torch.arange(rows, device=device) < ok_rows)[:, None] & (torch.arange(cols, device=device) < ok_cols)[None, :]
            flags.append(cell_ok.reshape(-1, 1).expand(rows * cols, self.num_base_anchors[lvl]).reshape(-1))
        return flags


class RPNProposals:
    """get_bboxes of the reference RPNHead (sigmoid classification, DeltaXYWHBBoxCoder) over ptb_rpn_proposals."""

    def __init__(self, anchor_generator, bbox_coder=None, test_cfg=None, use_sigmoid_cls=True):
        ag = dict(anchor_generator)
        if ag.pop('type', 'AnchorGenerator') != 'AnchorGenerator':
            raise NotImplementedError('only AnchorGenerator is implemented')
        self.anchor_generator = AnchorGenerator(**ag)
        bc = dict(bbox_coder or dict(type='DeltaXYWHBBoxCoder'))
        if bc.pop('type', 'DeltaXYWHBBoxCoder') != 'DeltaXYWHBBoxCoder':
            raise NotImplementedError('only DeltaXYWHBBoxCoder is implemented')
        if bc.get('add_ctr_clamp', False) or not bc.get('clip_border', True):
            raise NotImplementedError('DeltaXYWHBBoxCoder(add_ctr_clamp=True / clip_border=False)')
        self.means, self.stds = tuple(bc.get('target_means', (0., 0., 0., 0.))), tuple(bc.get('target_stds', (1., 1., 1., 1.)))
        self.wh_ratio_clip = 16 / 1000                       # DeltaXYWHBBoxCoder.decode default (delta_xywh_bbox_coder.py:88)
        if not use_sigmoid_cls:
            raise NotImplementedError('RPN softmax classification (loss_cls.use_sigmoid=False)')
        if len(set(self.anchor_generator.num_base_anchors)) != 1:
            raise NotImplementedError('levels with different numbers of base anchors')
        self.test_cfg = CfgNode(test_cfg) if test_cfg is not None else None
        self._base_dev = {}

    def _base(self, device):
        if device not in self._base_dev:
            self._base_dev[device] = torch.stack(self.anchor_generator.base_anchors).to(device).contiguous()
        return self._base_dev[device]

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, img_metas, cfg=None, rescale=False, with_nms=True, return_levels=False):
        assert len(cls_scores) == len(bbox_preds) == self.anchor_generator.num_levels
        if not with_nms:
            raise NotImplementedError('with_nms=False')
        if not cls_scores[0].is_cuda:
            raise RuntimeError('RPNProposals runs on CUDA tensors only; there is no CPU fallback')
        cfg = CfgNode(cfg) if cfg is not None else self.test_cfg
        nms = dict(cfg.get('nms', dict(type='nms', iou_threshold=cfg.get('nms_thr', 0.7))))
        if nms.get('type', 'nms') != 'nms':
            raise NotImplementedError(f"rpn nms type {nms.get('type')}")
        max_per_img = cfg.get('max_per_img', cfg.get('max_num', cfg.get('nms_post', 1000)))   # older configs spell it max_num / nms_post
        dev = cls_scores[0].device
        img_hw = torch.tensor([[int(m['img_shape'][0]), int(m['img_shape'][1])] for m in img_metas], dtype=torch.int32).to(dev)
        cnt, det, lvl = ops.rpn_proposals([c.detach().float().contiguous() for c in cls_scores], [r.detach().float().contiguous() for r in bbox_preds],
                                          self._base(dev), self.anchor_generator.strides, img_hw, self.means, self.stds, self.wh_ratio_clip,
                                          cfg.get('nms_pre', -1), cfg.get('min_bbox_size', 0), nms.get('iou_threshold', 0.7), max_per_img)
        cnt = cnt.cpu().tolist()                      # ragged result lists, like the reference's per-image dets
        out = [det[b, :cnt[b]] for b in range(len(cnt))]
        if return_levels:
            return out, [lvl[b, :cnt[b]] for b in range(len(cnt))]
        return out
