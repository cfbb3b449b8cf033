"""Tile testing of the two-stage detector: TwoStageDetector.tile_aug_test (detectors/two_stage.py:195-258) after extract_feats, the
path the TinyPerson Faster R-CNN config evaluates with (CroppedTilesFlipAug hands every tile of a test image to the detector as an
aug with a `tile_offset`; test_cfg.rcnn.do_tile_as_aug=False).  For one image:
  * the RPN forward and one ptb_rpn_proposals launch per FPN shape over all tiles x augs, then merge_aug_proposals of every tile
    (ptb_proposal_map_back and one ptb_batched_nms launch: plain NMS, sort, cut to the RPN's max_per_img);
  * StandardRoIHead's aug test of every tile at once (ptb_box_map, one RoIAlign per FPN shape, one FC pass, ptb_roi_decode,
    ptb_aug_merge, one multiclass NMS launch over the tiles);
  * each tile's detections scaled by its first aug's scale_factor (rescale=False) and shifted by its offset, concatenated in
    bbox2result's class-major order (ptb_tile_concat), then one class-aware batched_nms over the image (ptb_batched_nms) and the
    max_per_img cut; one device-to-host copy at the end.
There is no CPU path: CUDA tensors only."""
import numpy as np
import torch

from . import ops
from .post_processing import HARD_NMS_KEYS, check_kept, parse_nms_cfg
from .registry import CfgNode
from .results import bbox2result


def _rpn_merge_cfg(cfg):
    """merge_aug_proposals' reading of the RPN test cfg: (IoU threshold, max_per_img), max_num being the older max_per_img"""
    cfg = CfgNode(cfg)
    nms = parse_nms_cfg(cfg.get('nms') or dict(iou_threshold=cfg.get('nms_thr')))
    if nms.kind != 'nms':
        raise NotImplementedError(f'merge_aug_proposals nms type {nms.kind}')
    max_per_img = cfg.get('max_per_img', cfg.get('max_num'))
    if 'max_num' in cfg and max_per_img != cfg.max_num:
        raise AssertionError(f'You set max_num and max_per_img at the same time, but get {cfg.max_num} and {max_per_img} respectively')
    return nms.iou, int(max_per_img)


def _merge_nms_cfg(rcnn_test_cfg):
    nms_cfg = CfgNode(rcnn_test_cfg).get('nms') or {}
    nms = parse_nms_cfg(nms_cfg, default_iou=0.5)
    if nms.kind != 'nms':
        raise NotImplementedError('tile_aug_test: soft-NMS at the cross-tile merge is not implemented (nms type must be nms)')
    if nms.class_agnostic:
        raise NotImplementedError('tile_aug_test: class_agnostic NMS at the cross-tile merge')
    if set(nms_cfg) - HARD_NMS_KEYS:
        raise NotImplementedError(f'tile_aug_test: nms options {sorted(set(nms_cfg) - HARD_NMS_KEYS)} at the cross-tile merge')
    return nms.iou, int(nms.split_thr)


def group_tiles(img_metas):
    """pops every aug's tile_offset (as the reference does) and groups the augs by it in order of first appearance: [(offset, [i])]"""
    tiles = {}
    for i, m in enumerate(img_metas):
        if len(m) != 1:
            raise ValueError('tile_aug_test: one image per call (each aug meta a list of one dict)')
        tiles.setdefault(m[0].pop('tile_offset'), []).append(i)
    return list(tiles.items())


@torch.no_grad()
def tile_aug_test(rpn_head, roi_head, feats, img_metas, rcnn_test_cfg, rescale=False):
    """TwoStageDetector.tile_aug_test after extract_feats: feats per aug (the FPN levels of one image each), img_metas per aug [meta]
    with a `tile_offset` each.  returns [bbox_results] (one (k, 5) array per class)."""
    if len(feats) != len(img_metas):
        raise AssertionError('tile_aug_test: one feature list per aug meta')
    tiles = group_tiles(img_metas)
    A = len(tiles[0][1])
    if any(len(ix) != A for _, ix in tiles):
        raise NotImplementedError('tile_aug_test: every tile must have the same number of augs')
    T = len(tiles)
    order = [i for _, ix in tiles for i in ix]
    fts = [feats[i] for i in order]
    metas = [img_metas[i][0] for i in order]
    G = T * A
    dev = fts[0][0].device
    if not fts[0][0].is_cuda:
        raise RuntimeError('tile_aug_test runs on CUDA tensors only; there is no CPU fallback')
    C = roi_head.bbox_head.num_classes
    iou_rpn, max_prop = _rpn_merge_cfg(rpn_head.test_cfg)
    iou, split_thr = _merge_nms_cfg(rcnn_test_cfg)
    roi_cfg = CfgNode(rcnn_test_cfg)
    # RPN: one forward and one proposal launch per FPN shape
    batch = roi_head.shape_batches(fts)
    groups = {}
    for g, b in enumerate(batch):
        groups.setdefault(tuple(tuple(m.shape[-2:]) for m in fts[g]), []).append(g)
    counts, dets = [None] * len(groups), [None] * len(groups)
    for k, gs in enumerate(groups.values()):
        x = [torch.cat([fts[g][l] for g in gs]) for l in range(len(fts[gs[0]]))]
        cnt, det, _ = rpn_head.proposals.get_bboxes_padded(*rpn_head(x), [metas[g] for g in gs])
        counts[k], dets[k] = cnt, det
    if len(groups) == 1:
        cnt, det = counts[0], dets[0]
    else:
        inv = torch.empty(G, dtype=torch.int64)
        inv[torch.tensor([g for gs in groups.values() for g in gs])] = torch.arange(G)
        inv = inv.to(dev)
        cnt, det = torch.cat(counts)[inv].contiguous(), torch.cat(dets)[inv].contiguous()
    meta_back = ops.aug_meta(metas, [g // A for g in range(G)], batch, dev)
    props, pcnt = ops.proposal_map_back(det, cnt, meta_back, A)
    pcnt, props, _, _ = ops.batched_nms(props, props[..., 4], None, pcnt, iou_rpn, max_num=max_prop)
    Np = min(props.shape[1], max_prop)
    props = props[:, :Np].contiguous()
    # the RoI head's aug test of every tile
    rois = ops.box_map(props, pcnt, meta_back)
    boxes, scores = roi_head.aug_forward_merge(fts, metas, meta_back, rois, pcnt, A)
    tcnt, tdet, tlab, kmax, unlimited = roi_head._multiclass_nms(boxes, scores, roi_cfg)
    first = [metas[t * A] for t in range(T)]
    host = np.array([[float(o[0]), float(o[1])] for o, _ in tiles], np.float32)
    if not rescale:
        sf = np.stack([np.asarray(m['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32) for m in first])
        host = np.concatenate([host, sf], 1)
    host = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
    off, sf = host[:, :2].contiguous(), (host[:, 2:].contiguous() if not rescale else None)
    rows, rlab, rcnt = ops.tile_concat(tdet, tlab, tcnt, off, sf)
    if rows.shape[0] > ops.BATCHED_NMS_MAX_ROWS:
        raise NotImplementedError(f'tile_aug_test: {T} tiles x {kmax} detections exceed the cross-tile NMS limit of '
                                  f'{ops.BATCHED_NMS_MAX_ROWS} rows (PTB_BATCHED_NMS_MAX_ROWS)')
    fcnt, fdet, flab, _ = ops.batched_nms(rows[None], rows[None, :, 4], rlab[None], rcnt, iou, split_thr,
                                          -1 if unlimited else kmax)
    n = fdet.shape[1]
    out = torch.cat([fcnt.float(), tcnt.float(), fdet[0].reshape(-1), flab[0].float()]).cpu()   # the one device-to-host copy
    k = int(out[0])
    check_kept(int(out[1:1 + T].max()), kmax, unlimited)
    d = out[1 + T:1 + T + 5 * n].view(n, 5)[:k]
    lab = out[1 + T + 5 * n:].long()[:k]
    return [bbox2result(d, lab, C)]
