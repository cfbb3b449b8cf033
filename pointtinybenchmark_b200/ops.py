"""Thin torch-tensor wrappers over the C ABI (include/ptb_b200.h).  Device memory, streams and autograd plumbing
only — all math happens in libptb_b200.so.  Every op raises if the library is missing or a tensor is not on CUDA.
"""
import ctypes
import math

import numpy as np

import torch

from . import _lib
from ._lib import RefineCfg, check


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    """lib.<name>(*args, stream) on the current stream, a tensor passed as its data_ptr() and None as NULL (ctypes arrays, structs and
    scalars as they are); raises with the entry point's name and message when it returns non-zero."""
    check(getattr(_lib.load(), name)(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args], _stream()), name)


def _chk(t, dtype, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f'{name}: expected a CUDA tensor (pointtinybenchmark_b200 has no CPU path)')
    if t.dtype != dtype:
        raise TypeError(f'{name}: expected {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise ValueError(f'{name}: must be contiguous')
    return t


def to_nhwc(x):
    """(B,C,H,W) tensor -> contiguous (B,H,W,C) view (no copy when x is already channels_last)."""
    if x.dim() != 4:
        raise ValueError('expected (B,C,H,W)')
    return x.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)


def circle_offsets(radius, stride, start_angle=0, base_num_point=8, same_num_all_radius=False, append_center=True):
    """Bag offset table, computed once on the host with the reference's exact torch-CPU op sequence
    (cpr_head.py:484-497) so the sample coordinates are bit-identical.  (K,2) fp32 CPU tensor, centre LAST."""
    out = []
    for i in range(radius):
        r = (i + 1) * stride
        m = base_num_point if same_num_all_radius else base_num_point * (i + 1)
        ang = torch.arange(m).float() / m * 360 + start_angle
        ang = ang / 360 * math.pi * 2
        out.append(torch.stack([r * torch.cos(ang), r * torch.sin(ang)], dim=-1))
    off = torch.cat(out) if out else torch.zeros(0, 2)
    if append_center:
        off = torch.cat([off, torch.zeros(1, 2)])
    return off.float().contiguous()


# ----------------------------------------------------------------------------------------------------------------------
def bag_gather(map_nhwc, centers, bag_img, offsets, stride, pad_hw, feats=True, pts=True, valid=True, C=None, reach_px=None):
    """ptb_cpr_bag_gather. map_nhwc (B,H,W,ld) fp32; centers (G,2); bag_img (G,) int32; offsets (K,2); pad_hw (B,2) int32;
    reach_px: max |offset| (offsets_reach(offsets) when None).
    returns (feats (G,K,C) | None, pts (G,K,3) | None, valid (G,K) bool | None)."""
    _chk(map_nhwc, torch.float32, 'map'); _chk(centers, torch.float32, 'centers'); _chk(bag_img, torch.int32, 'bag_img')
    _chk(offsets, torch.float32, 'offsets'); _chk(pad_hw, torch.int32, 'pad_hw')
    B, H, W, ld = map_nhwc.shape
    C = ld if C is None else C
    G, K = centers.shape[0], offsets.shape[0]
    dev = map_nhwc.device
    o_f = torch.empty((G, K, C), dtype=torch.float32, device=dev) if feats else None
    o_p = torch.empty((G, K, 3), dtype=torch.float32, device=dev) if pts else None
    o_v = torch.empty((G, K), dtype=torch.uint8, device=dev) if valid else None
    _call('ptb_cpr_bag_gather', map_nhwc, B, H, W, C, ld, centers, bag_img, G, offsets, K, float(stride),
          (float(offsets_reach(offsets) if reach_px is None else reach_px)) if feats else 0.0, pad_hw, o_f, o_p, o_v)
    return o_f, o_p, (o_v.bool() if o_v is not None else None)


def bag_gather_bwd(grad_out, map_shape, centers, bag_img, offsets, stride):
    _chk(grad_out, torch.float32, 'grad_out')
    B, H, W, ld = map_shape
    G, K, C = grad_out.shape
    gm = torch.zeros(map_shape, dtype=torch.float32, device=grad_out.device)
    _call('ptb_cpr_bag_gather_bwd', grad_out, B, H, W, C, ld, centers, bag_img, G, offsets, K, float(stride), gm)
    return gm


def grid_circles_max_pos_num(radius, max_pos_num=-1):
    """GridCirclesPtFeatGenerator.get_max_pos_num (cpr_head.py:440-444)."""
    return 2 * (2 * radius) ** 2 if max_pos_num <= 0 else max_pos_num


def grid_bag(map_nhwc, centers, bag_img, stride, radius, max_pos_num=-1, feats=True, pts=True, valid=True, cell=True, C=None,
             check_overflow=True):
    """ptb_cpr_grid_bag: grid-cell bags of GridCirclesPtFeatGenerator (cpr_head.py:296-350, 418-444).
    returns (feats (G,Kt,C) | None, pts (G,Kt,3) | None, valid (G,Kt) bool | None, cell (G,Kt) int32 | None), Kt = max_pos_num + 2."""
    _chk(map_nhwc, torch.float32, 'map'); _chk(centers, torch.float32, 'centers'); _chk(bag_img, torch.int32, 'bag_img')
    mp = grid_circles_max_pos_num(radius, max_pos_num)
    if not isinstance(mp, int):
        # the reference passes this straight to torch.zeros(n, max_pos_num + R, ...) which rejects floats
        raise TypeError(f'max_pos_num must be an int, got {mp!r} (use an int radius or set max_pos_num)')
    B, H, W, ld = map_nhwc.shape
    C = ld if C is None else C
    G = centers.shape[0]
    Kt = mp + 2
    dev = map_nhwc.device
    o_f = torch.empty((G, Kt, C), dtype=torch.float32, device=dev) if feats else None
    o_p = torch.empty((G, Kt, 3), dtype=torch.float32, device=dev) if pts else None
    o_v = torch.empty((G, Kt), dtype=torch.uint8, device=dev) if valid else None
    o_c = torch.empty((G, Kt), dtype=torch.int32, device=dev) if cell else None
    ovf = torch.zeros(1, dtype=torch.int32, device=dev)
    radius_px = float(torch.tensor(radius * stride, dtype=torch.float32))      # the comparison scalar is cast to fp32
    _call('ptb_cpr_grid_bag', map_nhwc, B, H, W, C, ld, centers, bag_img, G, float(stride), radius_px, mp, o_f, o_p, o_v, o_c, ovf)
    if check_overflow and int(ovf.item()):
        raise RuntimeError(f'GridCirclesPtFeatGenerator: a GT has more than max_pos_num + num_refine = {mp + 1} cells within '
                           f'radius {radius}*{stride}; the reference fails here too (cpr_head.py:334)')
    return o_f, o_p, (o_v.bool() if valid else None), o_c


def grid_bag_bwd(grad_out, map_shape, centers, bag_img, cell, stride):
    _chk(grad_out, torch.float32, 'grad_out'); _chk(cell, torch.int32, 'cell')
    B, H, W, ld = map_shape
    G, Kt, C = grad_out.shape
    gm = torch.zeros(map_shape, dtype=torch.float32, device=grad_out.device)
    _call('ptb_cpr_grid_bag_bwd', grad_out, B, H, W, C, ld, centers, bag_img, cell, G, Kt, float(stride), gm)
    return gm


def linear_rows(x2d, weight, bias=None, out=None):
    """y = x2d @ weight.T + bias with the library's fp32 FFMA GEMM. x2d (M,Cin) view with row stride ldx."""
    if x2d.dim() != 2 or x2d.stride(1) != 1:
        raise ValueError('x2d must be 2-D with unit inner stride')
    if x2d.dtype != torch.float32 or not x2d.is_cuda:
        raise RuntimeError('x2d: expected a CUDA fp32 tensor')
    _chk(weight, torch.float32, 'weight')
    M, Cin = x2d.shape
    N = weight.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x2d.device)
    ldx = x2d.stride(0) if M > 1 else Cin
    _call('ptb_linear_rows', x2d, M, Cin, ldx, weight, bias, N, out, out.stride(0))
    return out


def linear_rows_bwd_x(dy, weight, accumulate_into=None):
    _chk(dy, torch.float32, 'dy'); _chk(weight, torch.float32, 'weight')
    M, N = dy.shape
    Cin = weight.shape[1]
    dx = accumulate_into if accumulate_into is not None else torch.empty((M, Cin), dtype=torch.float32, device=dy.device)
    _call('ptb_linear_rows_bwd_x', dy, M, N, dy.stride(0), weight, Cin, dx, dx.stride(0), 1 if accumulate_into is not None else 0)
    return dx


def linear_rows_bwd_w(dy, x2d):
    _chk(dy, torch.float32, 'dy')
    M, N = dy.shape
    Cin = x2d.shape[1]
    ldx = x2d.stride(0) if M > 1 else Cin
    nbytes = _lib.load().ptb_linear_rows_bwd_w_workspace(M, N, Cin)
    ws = torch.empty(nbytes // 4, dtype=torch.float32, device=dy.device)
    dw = torch.empty((N, Cin), dtype=torch.float32, device=dy.device)
    db = torch.empty((N,), dtype=torch.float32, device=dy.device)
    _call('ptb_linear_rows_bwd_w', dy, M, N, dy.stride(0), x2d, Cin, ldx, dw, db, ws, nbytes)
    return dw, db


def neg_mask(B, H, W, stride, pad_hw, centers, labels, img_ptr, thresh, num_classes, class_wise=True, as_bool=True):
    """ptb_cpr_neg_mask -> bool (or uint8 0/1) (B,H,W,num_classes)."""
    _chk(pad_hw, torch.int32, 'pad_hw'); _chk(centers, torch.float32, 'centers'); _chk(labels, torch.int32, 'labels')
    _chk(img_ptr, torch.int32, 'img_ptr')
    out = torch.empty((B, H, W, num_classes), dtype=torch.uint8, device=centers.device)
    _call('ptb_cpr_neg_mask', B, H, W, float(stride), pad_hw, centers, labels, img_ptr, centers.shape[0], float(thresh), num_classes,
          1 if class_wise else 0, out)
    return out.bool() if as_bool else out


def label_groups(bag_img, labels, num_classes):
    """CSR of same-(image,label) GT groups, built on the device without a host sync (replaces group_by_label,
    cpr_head.py:64-70, which forces labels.cpu()).  returns grp_of (G,), grp_ptr (G+1,), grp_idx (G,) int32."""
    G = labels.shape[0]
    key = bag_img.long() * num_classes + labels.long()
    order = torch.argsort(key, stable=True)
    ks = key[order]
    change = torch.ones(G, dtype=torch.long, device=key.device)
    if G > 1:
        change[1:] = (ks[1:] != ks[:-1]).long()
    gid = torch.cumsum(change, 0) - 1
    pos = torch.arange(G, device=key.device)
    grp_ptr = torch.full((G + 1,), G, dtype=torch.long, device=key.device)
    grp_ptr.scatter_reduce_(0, gid, pos, reduce='amin', include_self=True)
    grp_of = torch.empty(G, dtype=torch.long, device=key.device)
    grp_of[order] = gid
    return grp_of.int().contiguous(), grp_ptr.int().contiguous(), order.int().contiguous()


def label_groups_csr(labels, img_ptr, num_classes, max_per_image):
    """ptb_label_groups: same result as label_groups() (tested against it) in one ~10 us launch instead of a torch sort + scans."""
    _chk(labels, torch.int32, 'labels'); _chk(img_ptr, torch.int32, 'img_ptr')
    G = labels.shape[0]
    dev = labels.device
    grp_of = torch.empty(G, dtype=torch.int32, device=dev)
    grp_ptr = torch.empty(G + 1, dtype=torch.int32, device=dev)
    grp_idx = torch.empty(G, dtype=torch.int32, device=dev)
    _call('ptb_label_groups', labels, img_ptr, img_ptr.shape[0] - 1, G, int(num_classes), int(max_per_image), grp_of, grp_ptr, grp_idx)
    return grp_of, grp_ptr, grp_idx


def _refine_cfg(merge_th, gt_alpha, refine_th, nearest_filter, classify_filter, score_max):
    return RefineCfg(float(merge_th), float(gt_alpha), float(refine_th),
                     (1 if nearest_filter else 0) | (2 if classify_filter else 0) | (4 if score_max else 0))


def refine(bag_prob, bag_pts, bag_valid, K, labels, bag_img, img_hw, groups, cfg, not_refine=None, want_masks=True):
    """ptb_cpr_refine (stage form).  bag_prob (G,Kt,C), bag_pts (G,Kt,3), bag_valid (G,Kt) bool/uint8."""
    _chk(bag_prob, torch.float32, 'bag_prob'); _chk(bag_pts, torch.float32, 'bag_pts')
    bv = bag_valid.to(torch.uint8).contiguous()
    G, Kt, C = bag_prob.shape
    dev = bag_prob.device
    grp_of, grp_ptr, grp_idx = groups
    o_pts = torch.empty((G, 2), dtype=torch.float32, device=dev)
    o_sc = torch.empty((G,), dtype=torch.float32, device=dev)
    o_nr = torch.empty((G,), dtype=torch.uint8, device=dev)
    o_ch = torch.empty((G, Kt), dtype=torch.uint8, device=dev) if want_masks else None
    o_mv = torch.empty((G, Kt), dtype=torch.uint8, device=dev) if want_masks else None
    nr_in = not_refine.to(torch.uint8).contiguous() if not_refine is not None else None
    _call('ptb_cpr_refine', bag_prob, bag_pts, bv, G, Kt, K, C, labels, bag_img, img_hw, grp_of, grp_ptr, grp_idx, nr_in, cfg, o_pts, o_sc,
          o_nr, o_ch, o_mv)
    return o_pts, o_sc, o_nr.bool(), (o_ch.bool() if want_masks else None), (o_mv.bool() if want_masks else None)


def with_reach(offsets, reach):
    """attach the reach of a bag offset table to the tensor object (see offsets_reach); returns `offsets`.  Inference tensors have no
    version counter, so nothing is attached to them (an in-place change could not be detected)."""
    if not offsets.is_inference():
        offsets._ptb_reach = (offsets._version, float(reach))
    return offsets


def offsets_reach(offsets):
    """max |offset| of a bag offset table in pixels (= radius * stride for ring bags): sizes the shared-memory windows the gather, the
    fused refine and the deterministic loss backward stage per GT.  Cached on the tensor object itself (valid while the tensor is not
    modified in place), never by address: the caching allocator hands a freed table's address to the next allocation of that size.
    A device table without a cached reach is read back (a host sync): once per table, or on every call for an inference tensor.
    CPRHead keeps the reach of its host table beside the device table and passes it explicitly instead."""
    if not offsets.is_inference():
        cached = getattr(offsets, '_ptb_reach', None)
        if cached is not None and cached[0] == offsets._version:
            return cached[1]
    r = float(offsets.detach().abs().max()) if offsets.numel() else 0.0
    with_reach(offsets, r)
    return r


def refine_fused(logit_map, num_classes, centers, labels, bag_img, offsets, stride, pad_hw, img_hw, groups, cfg,
                 not_refine=None, want_chosen=False, reach_px=None):
    """ptb_cpr_refine_fused.  logit_map (B,H,W,ld) fp32 class logits (channels-last)."""
    if reach_px is None:
        reach_px = offsets_reach(offsets)
    _chk(logit_map, torch.float32, 'logit_map'); _chk(centers, torch.float32, 'centers')
    _chk(labels, torch.int32, 'labels'); _chk(bag_img, torch.int32, 'bag_img'); _chk(offsets, torch.float32, 'offsets')
    B, H, W, ld = logit_map.shape
    G, K = centers.shape[0], offsets.shape[0]
    dev = logit_map.device
    grp_of, grp_ptr, grp_idx = groups
    o_pts = torch.empty((G, 2), dtype=torch.float32, device=dev)
    o_sc = torch.empty((G,), dtype=torch.float32, device=dev)
    o_nr = torch.empty((G,), dtype=torch.uint8, device=dev)
    o_ch = torch.empty((G, K), dtype=torch.uint8, device=dev) if want_chosen else None
    nr_in = not_refine.to(torch.uint8).contiguous() if not_refine is not None else None
    _call('ptb_cpr_refine_fused', logit_map, B, H, W, num_classes, ld, centers, labels, bag_img, G, offsets, K, float(stride),
          float(reach_px), pad_hw, img_hw, grp_of, grp_ptr, grp_idx, nr_in, cfg, o_pts, o_sc, o_nr, o_ch)
    return o_pts, o_sc, o_nr.bool(), (o_ch.bool() if want_chosen else None)


def launch_count():
    return int(_lib.load().ptb_launch_count())


# ----------------------------------------------------------------------------------------------------------------------
# losses
# ----------------------------------------------------------------------------------------------------------------------
LOSS_KINDS = {'gfocal_loss': _lib.DEFINES['PTB_LOSS_GFOCAL'],      # the reference's `loss_type` names
              'binary_cross_entropy': _lib.DEFINES['PTB_LOSS_BCE']}


def mil_loss_fwd(logits, num_classes, ins_off, weight, labels, eps, want_aux=False, loss_kind=0):
    """ptb_mil_loss_fwd.  logits (G,Kt,ld) [cls | ins]; weight (G,Kt) fp32; labels (G,) int32.
    returns bag_prob (G,C), loss_sum (1,), stats (2,) = [#bags with weight, #top-1 hits]."""
    _chk(logits, torch.float32, 'logits'); _chk(weight, torch.float32, 'weight'); _chk(labels, torch.int32, 'labels')
    G, Kt, ld = logits.shape
    buf = torch.empty(G * num_classes + 3 * G, dtype=torch.float32, device=logits.device)
    loss = torch.zeros(1, dtype=torch.float32, device=logits.device)
    stats = torch.zeros(2, dtype=torch.float32, device=logits.device)
    mt = torch.empty((G, num_classes, 2), dtype=torch.float32, device=logits.device) if want_aux else None
    _call('ptb_mil_loss_fwd', logits, G, Kt, num_classes, ld, ins_off, weight, labels, float(eps), int(loss_kind), buf, loss, stats, mt)
    bag_prob = buf[:G * num_classes].view(G, num_classes)
    if want_aux:         # (max ins, 1/T) per (bag, class) and the per-bag label weight: inputs of ptb_cpr_loss_bwd_map
        return bag_prob, loss, stats, mt, buf[G * num_classes + G:G * num_classes + 2 * G]
    return bag_prob, loss, stats


def bag_mil_fwd(lmap, num_classes, ins_off, centers, bag_img, offsets, stride, pad_hw, labels, eps, loss_kind=0):
    """ptb_cpr_bag_mil_fwd: fused ring-bag gather of the [cls | ins] logit map + MIL forward.
    returns bag_logits (G,K,ld), weight (G,K) fp32 0/1, bag_prob (G,N), loss_sum (1,), stats (2,), mt (G,N,2), label_weight (G,)."""
    _chk(lmap, torch.float32, 'lmap'); _chk(centers, torch.float32, 'centers'); _chk(labels, torch.int32, 'labels')
    B, H, W, ld = lmap.shape
    G, K = centers.shape[0], offsets.shape[0]
    dev = lmap.device
    bl = torch.empty((G, K, ld), dtype=torch.float32, device=dev)
    if ld > ins_off + (num_classes + 3) // 4 * 4 or ins_off > (num_classes + 3) // 4 * 4:
        bl.zero_()                               # pad columns the kernel does not write
    weight = torch.empty((G, K), dtype=torch.float32, device=dev)
    buf = torch.empty(G * num_classes + 3 * G, dtype=torch.float32, device=dev)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    stats = torch.zeros(2, dtype=torch.float32, device=dev)
    mt = torch.empty((G, num_classes, 2), dtype=torch.float32, device=dev)
    _call('ptb_cpr_bag_mil_fwd', lmap, B, H, W, ld, num_classes, ins_off, centers, bag_img, G, offsets, K, float(stride), pad_hw, labels,
          float(eps), int(loss_kind), bl, weight, buf, loss, stats, mt)
    return (bl, weight, buf[:G * num_classes].view(G, num_classes), loss, stats, mt, buf[G * num_classes + G:G * num_classes + 2 * G])


def mil_loss_bwd(logits, num_classes, ins_off, weight, labels, eps, bag_prob, scale, grad_out=None, loss_kind=0):
    G, Kt, ld = logits.shape
    grad = grad_out if grad_out is not None else torch.zeros_like(logits)
    _chk(scale, torch.float32, 'scale')
    bp = bag_prob.contiguous()
    _call('ptb_mil_loss_bwd', logits, G, Kt, num_classes, ld, ins_off, weight, labels, float(eps), int(loss_kind), bp, scale, grad)
    return grad


def allpos_fwd(bag_logits, num_classes, weight, labels, eps, loss_kind):
    """ptb_cpr_allpos_fwd (AllPosLoss).  bag_logits (G,K,ld) with the cls logits in columns 0..num_classes; weight (G,K) fp32.
    returns loss_sum (1,), stats (2,) = [#samples with weight > 0, #samples whose top-1 class is the label]."""
    _chk(bag_logits, torch.float32, 'bag_logits'); _chk(weight, torch.float32, 'weight'); _chk(labels, torch.int32, 'labels')
    G, K, ld = bag_logits.shape
    dev = bag_logits.device
    aux = torch.empty(3 * max(G, 1), dtype=torch.float32, device=dev)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    stats = torch.zeros(2, dtype=torch.float32, device=dev)
    _call('ptb_cpr_allpos_fwd', bag_logits, G, K, num_classes, ld, weight, labels, float(eps), int(loss_kind), aux, loss, stats)
    return loss, stats


def cpr_loss_bwd_map(bag_logits, weight, mil_mt, bag_prob, label_weight, labels, centers, img_ptr, offsets, map_shape, num_classes, ins_off,
                     stride, reach_px, eps, scale_mil=None, scale_gt=None, valid_center=None, logit_map=None, neg_mask=None, scale_neg=None,
                     loss_kind=0, scale_pos=None):
    """ptb_cpr_loss_bwd_map: d loss / d logit map (B,H,W,ld), deterministic, every element written.  mil_mt None drops the MIL term,
    scale_pos adds the per-sample positive term of AllPosLoss."""
    _chk(bag_logits, torch.float32, 'bag_logits'); _chk(weight, torch.float32, 'weight'); _chk(centers, torch.float32, 'centers')
    B, H, W, ld = map_shape
    G, K, _ = bag_logits.shape
    out = torch.empty((B, H, W, ld), dtype=torch.float32, device=bag_logits.device)
    ws = torch.empty(int(_lib.load().ptb_cpr_loss_bwd_map_workspace(G, num_classes)) // 4, dtype=torch.float32, device=bag_logits.device)
    _call('ptb_cpr_loss_bwd_map', bag_logits, weight, mil_mt, bag_prob, label_weight, labels, centers, img_ptr, offsets, B, H, W, G, K,
          num_classes, ins_off, ld, float(stride), float(reach_px), float(eps), scale_mil, scale_gt, valid_center, logit_map, neg_mask,
          scale_neg, int(loss_kind), scale_pos, ws, out)
    return out


def cpr_loss_bwd_scatter(bag_logits, weight, mil_mt, bag_prob, label_weight, labels, centers, bag_img, offsets, grad_map, num_classes, ins_off,
                         stride, eps, scale_mil=None, scale_gt=None, valid_center=None, loss_kind=0, scale_pos=None):
    """ptb_cpr_loss_bwd_scatter: adds the MIL + gt part of d loss / d logit map into grad_map (B,H,W,ld) with fp32 vector atomics."""
    _chk(bag_logits, torch.float32, 'bag_logits'); _chk(weight, torch.float32, 'weight'); _chk(grad_map, torch.float32, 'grad_map')
    B, H, W, ld = grad_map.shape
    G, K, _ = bag_logits.shape
    ws = torch.empty(int(_lib.load().ptb_cpr_loss_bwd_map_workspace(G, num_classes)) // 4, dtype=torch.float32, device=bag_logits.device)
    _call('ptb_cpr_loss_bwd_scatter', bag_logits, weight, mil_mt, bag_prob, label_weight, labels, centers, bag_img, offsets, B, H, W, G, K,
          num_classes, ins_off, ld, float(stride), float(eps), scale_mil, scale_gt, valid_center, int(loss_kind), scale_pos, ws, grad_map)
    return grad_map


def gfocal_fwd(logits, M, num_classes, row_stride, target_label, weight, eps, loss_sum=None):
    """sum of gfocal(sigmoid(logits[m, :C]), onehot(target_label[m]) or 0) * weight.  weight: uint8 (M,C) | float (M,) | None."""
    if loss_sum is None:
        loss_sum = torch.zeros(1, dtype=torch.float32, device=logits.device)
    wmode = 0 if (weight is not None and weight.dtype == torch.uint8) else 1
    _call('ptb_gfocal_sigmoid_fwd', logits, M, num_classes, row_stride, target_label, weight, wmode, float(eps), loss_sum)
    return loss_sum


def gfocal_bwd(logits, M, num_classes, row_stride, target_label, weight, eps, scale, grad, grad_row_stride, accumulate, loss_kind=0):
    """ptb_sigmoid_loss_bwd: grad (+)= scale * weight * d term(sigmoid(logits), target) / d logits; term = gfocal or, with loss_kind 1,
    binary cross-entropy."""
    wmode = 0 if (weight is not None and weight.dtype == torch.uint8) else 1
    _call('ptb_sigmoid_loss_bwd', logits, M, num_classes, row_stride, target_label, weight, wmode, float(eps), int(loss_kind), scale, grad,
          grad_row_stride, 1 if accumulate else 0)
    return grad


# ----------------------------------------------------------------------------------------------------------------------
# P2P
# ----------------------------------------------------------------------------------------------------------------------
def p2p_decode_topk(cls_map, reg_map, num_classes, k, point_anchor, stride, pts_gamma, img_hw, nms_pre, scale_xy=None):
    """ptb_p2p_decode_topk. cls_map (B,H,W,k*C), reg_map (B,H,W,2k) channels-last logits.
    returns topk_idx (B,P) int32, pts (B,P,2), scores (B,P,C)."""
    _chk(cls_map, torch.float32, 'cls_map'); _chk(reg_map, torch.float32, 'reg_map'); _chk(point_anchor, torch.float32, 'anchor')
    _chk(img_hw, torch.int32, 'img_hw')
    B, H, W, _ = cls_map.shape
    Q = H * W * k
    P = nms_pre if 0 < nms_pre < Q else Q
    dev = cls_map.device
    idx = torch.empty((B, P), dtype=torch.int32, device=dev)
    pts = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
    sc = torch.empty((B, P, num_classes), dtype=torch.float32, device=dev)
    nbytes = _lib.load().ptb_p2p_decode_topk_workspace(B, H, W, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _call('ptb_p2p_decode_topk', cls_map, reg_map, B, H, W, num_classes, k, point_anchor, float(stride), float(pts_gamma), img_hw, scale_xy,
          int(nms_pre), idx, pts, sc, ws, nbytes)
    return idx, pts, sc


def p2p_decode_topk_softmax(cls_map, reg_map, num_classes, k, point_anchor, stride, pts_gamma, img_hw, nms_pre, scale_xy=None):
    """ptb_p2p_decode_topk_softmax. cls_map (B,H,W,k*(C+1)) logits with the background column last, reg_map (B,H,W,2k).
    returns topk_idx (B,P) int32, pts (B,P,2), scores (B,P,C) = the foreground softmax probabilities."""
    _chk(cls_map, torch.float32, 'cls_map'); _chk(reg_map, torch.float32, 'reg_map'); _chk(point_anchor, torch.float32, 'anchor')
    _chk(img_hw, torch.int32, 'img_hw')
    B, H, W, ch = cls_map.shape
    if ch != k * (num_classes + 1):
        raise ValueError(f'cls_map has {ch} channels; softmax scores need k * (num_classes + 1) = {k * (num_classes + 1)}')
    Q = H * W * k
    P = nms_pre if 0 < nms_pre < Q else Q
    dev = cls_map.device
    idx = torch.empty((B, P), dtype=torch.int32, device=dev)
    pts = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
    sc = torch.empty((B, P, num_classes), dtype=torch.float32, device=dev)
    nbytes = _lib.load().ptb_p2p_decode_topk_workspace(B, H, W, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _call('ptb_p2p_decode_topk_softmax', cls_map, reg_map, B, H, W, num_classes, k, point_anchor, float(stride), float(pts_gamma), img_hw,
          scale_xy, int(nms_pre), idx, pts, sc, ws, nbytes)
    return idx, pts, sc


def p2p_chunk_plan(featmap_sizes, k, nms_pre):
    """Host plan of the multi-level decode (P2PHead._get_bboxes_single, p2p_head.py:355-373).  featmap_sizes [(H_l, W_l)], k anchors.
    An image's T = sum_l H_l W_l k rows (level-major) are reshaped into L = len(featmap_sizes) equal chunks of T / L rows, so chunk
    boundaries need not fall on level boundaries; each chunk keeps its top nms_pre rows, or all of them when nms_pre <= 0 or
    nms_pre >= T / L.  Returns dict(T, L, chunk = T / L, P = rows kept per chunk, level_row0 = [first row of each level] + [T]).
    Raises RuntimeError when L does not divide T: the reference's reshape raises there (training is unaffected)."""
    L = len(featmap_sizes)
    row0 = [0]
    for h, w in featmap_sizes:
        row0.append(row0[-1] + int(h) * int(w) * int(k))
    T = row0[-1]
    if L < 1 or T % L:
        raise RuntimeError(f'P2PHead inference over {L} levels: {T} proposals per image (sum of H*W*{k} over the levels) do not '
                           f'split into {L} equal chunks, which the reference\'s _get_bboxes_single reshapes them into (it raises '
                           f'there too); pick feature map sizes whose proposal count is a multiple of {L}')
    chunk = T // L
    return dict(T=T, L=L, chunk=chunk, P=nms_pre if 0 < nms_pre < chunk else chunk, level_row0=row0)


def p2p_decode_topk_levels(cls_maps, reg_maps, strides, num_classes, k, point_anchor, pts_gamma, img_hw, nms_pre, scale_xy=None,
                           softmax=False):
    """ptb_p2p_decode_topk_levels(_softmax): decode + per-chunk top-k over L FPN levels.  cls_maps[l] (B,H_l,W_l,k*C1) and
    reg_maps[l] (B,H_l,W_l,2k) channels-last logits (C1 = C, or C+1 with softmax).  The T = sum_l H_l W_l k rows of an image are cut
    into L equal chunks (p2p_chunk_plan); each keeps its top nms_pre rows (or all when nms_pre <= 0 or >= T / L).
    returns topk_idx (B,L*P) int32 chunk-local row indices, pts (B,L*P,2), scores (B,L*P,C), chunk-major."""
    L = len(cls_maps)
    if len(reg_maps) != L or len(strides) != L:
        raise ValueError(f'{L} cls maps, {len(reg_maps)} reg maps and {len(strides)} strides')
    _chk(point_anchor, torch.float32, 'anchor'); _chk(img_hw, torch.int32, 'img_hw')
    B = cls_maps[0].shape[0]
    n_cls = k * (num_classes + 1 if softmax else num_classes)
    if point_anchor.shape != (k, 2):
        raise ValueError(f'point_anchor must have shape ({k}, 2), got {tuple(point_anchor.shape)}')
    if img_hw.shape != (B, 2) or (scale_xy is not None and tuple(scale_xy.shape) != (B, 2)):
        raise ValueError(f'img_hw (and scale_xy) must have shape ({B}, 2)')
    if scale_xy is not None:
        _chk(scale_xy, torch.float32, 'scale_xy')
    for l, (c, r) in enumerate(zip(cls_maps, reg_maps)):
        _chk(c, torch.float32, f'cls_maps[{l}]'); _chk(r, torch.float32, f'reg_maps[{l}]')
        if c.dim() != 4 or tuple(c.shape) != (B, c.shape[1], c.shape[2], n_cls):
            raise ValueError(f'cls_maps[{l}] must be (B={B}, H, W, {n_cls}) channels-last, got {tuple(c.shape)}')
        if tuple(r.shape) != (B, c.shape[1], c.shape[2], 2 * k):
            raise ValueError(f'reg_maps[{l}] must be {(B, c.shape[1], c.shape[2], 2 * k)} like cls_maps[{l}], got {tuple(r.shape)}')
    hw = [(int(c.shape[1]), int(c.shape[2])) for c in cls_maps]
    P = p2p_chunk_plan(hw, k, nms_pre)['P']
    dev = cls_maps[0].device
    idx = torch.empty((B, L * P), dtype=torch.int32, device=dev)
    pts = torch.empty((B, L * P, 2), dtype=torch.float32, device=dev)
    sc = torch.empty((B, L * P, num_classes), dtype=torch.float32, device=dev)
    hw_arr = (ctypes.c_int32 * (2 * L))(*[v for p in hw for v in p])
    st_arr = (ctypes.c_float * L)(*[float(s) for s in strides])
    cls_arr = (ctypes.c_void_p * L)(*[c.data_ptr() for c in cls_maps])
    reg_arr = (ctypes.c_void_p * L)(*[r.data_ptr() for r in reg_maps])
    nbytes = _lib.load().ptb_p2p_decode_topk_levels_workspace(B, L, hw_arr, k)
    ws = torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device=dev)
    _call('ptb_p2p_decode_topk_levels_softmax' if softmax else 'ptb_p2p_decode_topk_levels', cls_arr, reg_arr, L, hw_arr, st_arr, B,
          num_classes, k, point_anchor, float(pts_gamma), img_hw, scale_xy, int(nms_pre), idx, pts, sc, ws, nbytes)
    return idx, pts, sc


NMS_WIDE_MAX_POINTS = 8192    # points per image of ptb_multiclass_nms_wide / ptb_multiclass_soft_nms_wide


def _nms_outputs(B, max_per_img, device):
    """the outputs of the multiclass NMS entry points: count (B,), det (B,max,5), label (B,max), keep (B,max), cand_count (B,)"""
    return (torch.empty((B,), dtype=torch.int32, device=device), torch.zeros((B, max_per_img, 5), dtype=torch.float32, device=device),
            torch.zeros((B, max_per_img), dtype=torch.int32, device=device), torch.zeros((B, max_per_img), dtype=torch.int32, device=device),
            torch.empty((B,), dtype=torch.int32, device=device))


def multiclass_nms(pts, scores, pseudo_wh, score_thr, iou_thr, max_per_img, wide=False):
    """ptb_multiclass_nms. pts (B,P,2), scores (B,P,C) -> count (B,), det (B,max,5), label (B,max), keep (B,max), cand_count (B,)
    P <= 4096; wide=True: ptb_multiclass_nms_wide, P <= 8192 (the multi-level P2P head's candidates)."""
    _chk(pts, torch.float32, 'pts'); _chk(scores, torch.float32, 'scores')
    B, P, C = scores.shape
    dev = pts.device
    cnt, det, lab, keep, cc = _nms_outputs(B, max_per_img, dev)
    nbytes = _lib.load().ptb_multiclass_nms_workspace(B, P, C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _call('ptb_multiclass_nms_wide' if wide else 'ptb_multiclass_nms', pts, scores, B, P, C, float(pseudo_wh[0]), float(pseudo_wh[1]),
          float(score_thr), float(iou_thr), int(max_per_img), cnt, det, lab, keep, cc, ws, nbytes)
    return cnt, det, lab, keep, cc


def _cls_boxes(boxes, scores):
    """True for class-specific boxes (B,P,C,4), False for boxes shared by the classes (B,P,4)."""
    if boxes.dim() == 3:
        return False
    if tuple(boxes.shape) != tuple(scores.shape) + (4,):
        raise ValueError(f'class-specific boxes must be (B, P, C, 4) = {tuple(scores.shape) + (4,)}, got {tuple(boxes.shape)}')
    return True


def multiclass_nms_boxes(boxes, scores, score_thr, iou_thr, max_per_img):
    """ptb_multiclass_nms_boxes: boxes (B,P,4) xyxy shared by the classes, or ptb_multiclass_nms_cls_boxes: class-specific boxes
    (B,P,C,4), candidate (p, c) using boxes[b, p, c];  scores (B,P,C) -> count, det (B,max,5), label, keep, cand_count."""
    _chk(boxes, torch.float32, 'boxes'); _chk(scores, torch.float32, 'scores')
    B, P, C = scores.shape
    name = 'ptb_multiclass_nms_cls_boxes' if _cls_boxes(boxes, scores) else 'ptb_multiclass_nms_boxes'
    dev = boxes.device
    cnt, det, lab, keep, cc = _nms_outputs(B, max_per_img, dev)
    nbytes = _lib.load().ptb_multiclass_nms_workspace(B, P, C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _call(name, boxes, scores, B, P, C, float(score_thr), float(iou_thr), int(max_per_img), cnt, det, lab, keep, cc, ws, nbytes)
    return cnt, det, lab, keep, cc


SOFT_NMS_METHODS = {'naive': 0, 'linear': 1, 'gaussian': 2}


def multiclass_soft_nms(pts_or_boxes, scores, pseudo_wh, score_thr, iou_thr, max_per_img, sigma=0.5, min_score=1e-3, method='linear',
                        wide=False):
    """ptb_multiclass_soft_nms.  pts_or_boxes: (B,P,2) points (pseudo boxes of pseudo_wh) or (B,P,4) boxes; scores (B,P,C).
    Class-specific boxes (B,P,C,4) go to ptb_multiclass_soft_nms_cls_boxes.  P <= 4096; wide=True (points or shared boxes):
    ptb_multiclass_soft_nms_wide, P <= 8192.
    returns count (B,), det (B,max,5) with DECAYED scores, label, keep, cand_count."""
    _chk(pts_or_boxes, torch.float32, 'pts_or_boxes'); _chk(scores, torch.float32, 'scores')
    if method not in SOFT_NMS_METHODS:
        raise KeyError(method)
    B, P, C = scores.shape
    dev = scores.device
    cls_boxes = pts_or_boxes.dim() == 4 and _cls_boxes(pts_or_boxes, scores)
    is_boxes = pts_or_boxes.shape[-1] == 4
    cnt, det, lab, keep, cc = _nms_outputs(B, max_per_img, dev)
    nbytes = _lib.load().ptb_multiclass_soft_nms_workspace(B, P, C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    outs = (SOFT_NMS_METHODS[method], int(max_per_img), cnt, det, lab, keep, cc, ws, nbytes)
    if cls_boxes and wide:
        raise ValueError('multiclass_soft_nms: wide=True takes points or shared boxes, not class-specific boxes')
    if cls_boxes:
        name = 'ptb_multiclass_soft_nms_cls_boxes'
        _call(name, pts_or_boxes, scores, B, P, C, float(score_thr), float(iou_thr), float(sigma), float(min_score), *outs)
    else:
        name = 'ptb_multiclass_soft_nms_wide' if wide else 'ptb_multiclass_soft_nms'
        wh = pseudo_wh if pseudo_wh is not None else (0.0, 0.0)
        _call(name, None if is_boxes else pts_or_boxes, pts_or_boxes if is_boxes else None, scores, B, P, C, float(wh[0]), float(wh[1]),
              float(score_thr), float(iou_thr), float(sigma), float(min_score), *outs)
    if method == 'gaussian':              # refused images (count -1): one device read, gaussian only
        bad = torch.nonzero(cnt < 0).flatten().tolist()
        if bad:
            raise RuntimeError(f'{name}: gaussian soft-NMS refused image(s) {bad}: two candidate boxes of zero area '
                               '(or one of negative area) give IoU 0/0 = NaN weights')
    return cnt, det, lab, keep, cc


def p2p_cost_matrix(cls_logits, pts, row_idx, gts, gt_labels, w_cls, alpha, gamma, eps, w_dis, fx=1.0, fy=1.0, out=None):
    """ptb_p2p_cost_matrix -> (n_rows, n_gt) fp32 (written into `out`, a contiguous fp32 buffer of n_rows*n_gt elements, if given)."""
    _chk(cls_logits, torch.float32, 'cls_logits'); _chk(gts, torch.float32, 'gts'); _chk(gt_labels, torch.int32, 'gt_labels')
    if pts.stride(-1) != 1 or pts.dtype != torch.float32:
        raise ValueError('pts must be fp32 with unit inner stride')
    n_rows = row_idx.shape[0] if row_idx is not None else cls_logits.shape[0]
    n_gt = gts.shape[0]
    if out is None:
        cost = torch.empty((n_rows, n_gt), dtype=torch.float32, device=cls_logits.device)
    else:
        _chk(out, torch.float32, 'out')
        if out.numel() != n_rows * n_gt:
            raise ValueError('out must hold n_rows*n_gt elements')
        cost = out.view(n_rows, n_gt)
    _call('ptb_p2p_cost_matrix', cls_logits, pts, pts.stride(0), row_idx, n_rows, cls_logits.shape[1], gts, gt_labels, n_gt, float(w_cls),
          float(alpha), float(gamma), float(eps), float(w_dis), float(fx), float(fy), cost)
    return cost


MATCH_COST_KINDS = {'FocalLossCost': _lib.DEFINES['PTB_MATCH_COST_FOCAL'],            # ptb_match_cost.kind
                    'ClassificationCostV2_sigmoid': _lib.DEFINES['PTB_MATCH_COST_CLS_SIGMOID'],
                    'ClassificationCostV2_softmax': _lib.DEFINES['PTB_MATCH_COST_CLS_SOFTMAX'],
                    'ZeroCost': _lib.DEFINES['PTB_MATCH_COST_ZERO'], 'DisCostV2': _lib.DEFINES['PTB_MATCH_COST_DIS']}


def p2p_cost_matrix_terms(cls_logits, pts, row_idx, gts, gt_labels, terms, fx=1.0, fy=1.0, out=None):
    """ptb_p2p_cost_matrix_terms -> (n_rows, n_gt) fp32: sum(classification terms) + sum(DisCostV2 terms), each in list order.
    terms: dicts with 'kind' (a MATCH_COST_KINDS key) and 'weight', plus 'alpha', 'gamma', 'eps' (FocalLossCost) or 'p',
    'norm_with_img_wh' (DisCostV2), as assigners.match_cost_terms makes them.  cls_logits (Q, num_cols): the softmax term normalises
    over all num_cols columns.  fx, fy: the image width and height DisCostV2 divides by when norm_with_img_wh is set."""
    _chk(cls_logits, torch.float32, 'cls_logits'); _chk(gts, torch.float32, 'gts'); _chk(gt_labels, torch.int32, 'gt_labels')
    if pts.stride(-1) != 1 or pts.dtype != torch.float32:
        raise ValueError('pts must be fp32 with unit inner stride')
    if row_idx is not None:
        _chk(row_idx, torch.int32, 'row_idx')
    n_rows = row_idx.shape[0] if row_idx is not None else cls_logits.shape[0]
    n_gt = gts.shape[0]
    if out is None:
        cost = torch.empty((n_rows, n_gt), dtype=torch.float32, device=cls_logits.device)
    else:
        _chk(out, torch.float32, 'out')
        if out.numel() != n_rows * n_gt:
            raise ValueError('out must hold n_rows*n_gt elements')
        cost = out.view(n_rows, n_gt)
    arr = (_lib.MatchCost * max(len(terms), 1))(*[
        _lib.MatchCost(MATCH_COST_KINDS[t['kind']], float(t['weight']), float(t.get('alpha', 0.0)), float(t.get('gamma', 0.0)),
                       float(t.get('eps', 0.0)), int(t.get('p', 0)), int(bool(t.get('norm_with_img_wh', False)))) for t in terms])
    ws = None
    if any(t['kind'] == 'ClassificationCostV2_softmax' for t in terms):
        ws = torch.empty(max(int(_lib.load().ptb_p2p_cost_matrix_terms_workspace(n_rows)), 8), dtype=torch.uint8, device=cls_logits.device)
    _call('ptb_p2p_cost_matrix_terms', cls_logits, pts, pts.stride(0), row_idx, n_rows, cls_logits.shape[1], gts, gt_labels, n_gt, arr,
          len(terms), float(fx), float(fy), cost, ws, ws.numel() if ws is not None else 0)
    return cost


def rpn_proposals(cls_scores, bbox_preds, base_anchors, strides_wh, img_hw, means, stds, wh_ratio_clip, nms_pre, min_bbox_size, iou_thr,
                  max_per_img, want_candidates=False):
    """ptb_rpn_proposals.  cls_scores[l] (B,A,H,W) / bbox_preds[l] (B,4A,H,W) contiguous NCHW fp32 CUDA tensors, base_anchors (L,A,4),
    img_hw (B,2) int32 (h, w).  returns count (B,), det (B,max,5), level (B,max) [, dict(pos, cand_box, cand_score, cand_idx)]."""
    L = len(cls_scores)
    if L == 0 or len(bbox_preds) != L:
        raise ValueError('cls_scores / bbox_preds: one tensor per level')
    for c, r in zip(cls_scores, bbox_preds):
        _chk(c, torch.float32, 'cls_score'); _chk(r, torch.float32, 'bbox_pred')
        if c.dim() != 4 or r.dim() != 4 or r.shape[1] != 4 * c.shape[1] or r.shape[-2:] != c.shape[-2:] or r.shape[0] != c.shape[0]:
            raise ValueError(f'level shapes {tuple(c.shape)} / {tuple(r.shape)}')
    _chk(base_anchors, torch.float32, 'base_anchors'); _chk(img_hw, torch.int32, 'img_hw')
    B, A = cls_scores[0].shape[:2]
    if tuple(base_anchors.shape) != (L, A, 4) or tuple(img_hw.shape) != (B, 2):
        raise ValueError('base_anchors must be (L, A, 4) and img_hw (B, 2)')
    dev = cls_scores[0].device
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for c in cls_scores for v in c.shape[-2:]])
    st = (ctypes.c_int32 * (2 * L))(*[int(v) for s in strides_wh for v in s])
    cp = (ctypes.c_void_p * L)(*[c.data_ptr() for c in cls_scores])
    bp = (ctypes.c_void_p * L)(*[r.data_ptr() for r in bbox_preds])
    mean = (ctypes.c_float * 4)(*[float(v) for v in means])
    std = (ctypes.c_float * 4)(*[float(v) for v in stds])
    Ptot = sum(min(nms_pre, c.shape[1] * c.shape[2] * c.shape[3]) if nms_pre > 0 else c.shape[1] * c.shape[2] * c.shape[3] for c in cls_scores)
    cnt = torch.empty((B,), dtype=torch.int32, device=dev)
    det = torch.zeros((B, max_per_img, 5), dtype=torch.float32, device=dev)
    lvl = torch.zeros((B, max_per_img), dtype=torch.int32, device=dev)
    extra = None
    if want_candidates:
        extra = dict(pos=torch.zeros((B, max_per_img), dtype=torch.int32, device=dev), cand_box=torch.empty((B, Ptot, 4), device=dev),
                     cand_score=torch.empty((B, Ptot), device=dev), cand_idx=torch.empty((B, Ptot), dtype=torch.int32, device=dev))
    nbytes = int(_lib.load().ptb_rpn_proposals_workspace(hw, L, B, A, int(nms_pre), int(max_per_img)))
    if nbytes == 0:
        raise ValueError('ptb_rpn_proposals_workspace: unsupported shape')
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    e = extra or {}
    _call('ptb_rpn_proposals', cp, bp, hw, st, base_anchors, L, B, A, img_hw, mean, std, float(wh_ratio_clip), int(nms_pre),
          float(min_bbox_size), float(iou_thr), int(max_per_img), cnt, det, lvl, e.get('pos'), e.get('cand_box'), e.get('cand_score'),
          e.get('cand_idx'), ws, nbytes)
    return (cnt, det, lvl, extra) if want_candidates else (cnt, det, lvl)


def hungarian_v2_batch(cost_flat, shapes, topk_k, out, out_offsets, row_idx=None, row_idx_offsets=None):
    """ptb_hungarian_v2_batch: HungarianAssignerV2's matching for a batch of images, on the device.
    cost_flat      : fp32 CUDA buffer, image b = (N_b, n_b) row-major at element offset sum_{a<b} N_a*n_a
    shapes         : [(N_b, n_b)] host ints
    out            : int64 CUDA buffer, pre-zeroed; image b's assigned_gt_inds slice starts at out_offsets[b]
    row_idx        : optional int32 CUDA buffer (concatenated per image, offsets row_idx_offsets[b]): cost row -> slot in the slice
    returns status : int32 CUDA tensor (B,): 0 ok, 1 infeasible, 2 invalid entries (scipy raises ValueError for both), 3 internal."""
    _chk(cost_flat, torch.float32, 'cost'); _chk(out, torch.int64, 'out')
    if row_idx is not None:
        _chk(row_idx, torch.int32, 'row_idx')
    dev = cost_flat.device
    B = len(shapes)
    status = torch.zeros((max(B, 1),), dtype=torch.int32, device=dev)
    if B == 0:
        return status[:0]
    desc, co, wo = [], 0, 0
    for b, (N, n) in enumerate(shapes):
        desc.append([co, wo, int(out_offsets[b]), int(row_idx_offsets[b]) if row_idx is not None else -1, int(N), int(n)])
        co += int(N) * int(n)
        wo += (int(_lib.load().ptb_hungarian_v2_workspace(int(N), int(n))) + 7) // 8 * 8
    if co > cost_flat.numel():
        raise ValueError('cost buffer smaller than the shapes imply')
    max_N, max_n = max(s[0] for s in shapes), max(s[1] for s in shapes)
    d = torch.tensor(desc, dtype=torch.int64).pin_memory().to(dev, non_blocking=True)
    ws = torch.empty(max(wo, 64), dtype=torch.uint8, device=dev)
    _call('ptb_hungarian_v2_batch', cost_flat, d, B, int(max_N), int(max_n), int(topk_k), row_idx, out, ws, status)
    return status


def bbox_overlaps(boxes1, boxes2, mode='iou'):
    """ptb_bbox_overlaps: (m,4),(n,4) -> (m,n) IoU ('iou') or IoF w.r.t. boxes1 ('iof')  (BboxOverlaps2D, is_aligned=False)."""
    _chk(boxes1, torch.float32, 'boxes1'); _chk(boxes2, torch.float32, 'boxes2')
    if mode not in ('iou', 'iof'):
        raise NotImplementedError(f'bbox_overlaps mode {mode}')
    m, n = boxes1.shape[0], boxes2.shape[0]
    out = torch.empty((m, n), dtype=torch.float32, device=boxes1.device)
    _call('ptb_bbox_overlaps', boxes1, m, boxes2, n, 1 if mode == 'iof' else 0, out)
    return out


def max_iou_assign(bboxes, gt_bboxes, gt_labels=None, gt_bboxes_ignore=None, pos_iou_thr=0.5, neg_iou_thr=0.5, min_pos_iou=0.0,
                   gt_max_assign_all=True, ignore_iof_thr=-1, ignore_wrt_candidates=True, match_low_quality=True, out=None):
    """ptb_max_iou_assign.  returns gt_inds (N,) int64, max_overlaps (N,), labels (N,) int64 | None.  out: optional contiguous
    (gt_inds, max_overlaps) tensors of N elements to write into, e.g. one image's rows of a batch buffer."""
    _chk(bboxes, torch.float32, 'bboxes'); _chk(gt_bboxes, torch.float32, 'gt_bboxes')
    N, n = bboxes.shape[0], gt_bboxes.shape[0]
    dev = bboxes.device
    lo, hi = (0.0, float(neg_iou_thr)) if isinstance(neg_iou_thr, float) else (float(neg_iou_thr[0]), float(neg_iou_thr[1]))
    if out is not None:
        gt_inds, max_ov = out
        _chk(gt_inds, torch.int64, 'out gt_inds'); _chk(max_ov, torch.float32, 'out max_overlaps')
        if gt_inds.numel() != N or max_ov.numel() != N:
            raise ValueError(f'out tensors must have {N} elements')
    else:
        gt_inds = torch.empty((N,), dtype=torch.int64, device=dev)
        max_ov = torch.empty((N,), dtype=torch.float32, device=dev)
    labels = torch.empty((N,), dtype=torch.int64, device=dev) if gt_labels is not None else None
    gl = gt_labels.to(torch.int32).contiguous() if gt_labels is not None else None
    ign = gt_bboxes_ignore if (gt_bboxes_ignore is not None and gt_bboxes_ignore.numel() > 0) else None
    if ign is not None:
        _chk(ign, torch.float32, 'gt_bboxes_ignore')
    nbytes = int(_lib.load().ptb_max_iou_assign_workspace(N, n))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _call('ptb_max_iou_assign', bboxes, N, gt_bboxes, n, gl, ign, 0 if ign is None else ign.shape[0], float(pos_iou_thr), lo, hi,
          float(min_pos_iou), 1 if gt_max_assign_all else 0, 1 if match_low_quality else 0, float(ignore_iof_thr),
          1 if ignore_wrt_candidates else 0, gt_inds, max_ov, labels, ws, ws.numel())
    return gt_inds, max_ov, labels


def point_assigner(points, gt_bboxes, scale=4, pos_num=3):
    _chk(points, torch.float32, 'points'); _chk(gt_bboxes, torch.float32, 'gt_bboxes')
    N, n = points.shape[0], gt_bboxes.shape[0]
    out = torch.zeros((N,), dtype=torch.int64, device=points.device)
    nbytes = _lib.load().ptb_point_assigner_workspace(N, n)
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=points.device)
    _call('ptb_point_assigner', points, N, gt_bboxes, n, float(scale), int(pos_num), out, ws, nbytes)
    return out


def _loss_sum(name, x, args, scale, want_grad):
    """name(x, *args, loss_sum, scale, grad, stream), the calling convention of the fused loss entry points.  Returns the (1,) loss
    sum or, with want_grad, the gradient scale * d/dx instead (the sum is then not computed)."""
    loss = torch.zeros(1, dtype=torch.float32, device=x.device)
    grad = torch.empty_like(x) if want_grad else None
    _call(name, x, *args, loss if not want_grad else None, scale, grad)
    return grad if want_grad else loss


def sigmoid_focal(logits, labels, weight, gamma, alpha, scale=None, want_grad=False):
    """sum_m,c focal(logits, labels) * weight[m]; optional grad = scale * d/dlogits."""
    _chk(logits, torch.float32, 'logits'); _chk(labels, torch.int64, 'labels')
    M, C = logits.shape
    return _loss_sum('ptb_sigmoid_focal_fwd_bwd', logits, (labels, weight, M, C, float(gamma), float(alpha)), scale, want_grad)


def smooth_l1(pred, target, weight, inv_norm, beta, scale=None, want_grad=False):
    _chk(pred, torch.float32, 'pred'); _chk(target, torch.float32, 'target')
    return _loss_sum('ptb_smooth_l1_fwd_bwd', pred, (target, weight, pred.shape[0], float(inv_norm), float(beta)), scale, want_grad)


def smooth_l1_rows(pred, target, weight, row_inv_norm, beta, scale=None, want_grad=False):
    """smooth_l1 with one normalisation per row of pred (M, 2): row_inv_norm (M,) = 1 / (stride_m * reg_norm)."""
    _chk(pred, torch.float32, 'pred'); _chk(target, torch.float32, 'target'); _chk(row_inv_norm, torch.float32, 'row_inv_norm')
    if row_inv_norm.shape != (pred.shape[0],):
        raise ValueError(f'row_inv_norm must have shape ({pred.shape[0]},), got {tuple(row_inv_norm.shape)}')
    return _loss_sum('ptb_smooth_l1_rows_fwd_bwd', pred, (target, weight, pred.shape[0], row_inv_norm, float(beta)), scale, want_grad)


def sigmoid_bce(logits, labels, weight, pos_weight=None, scale=None, want_grad=False):
    """sum_m,c binary_cross_entropy_with_logits(logits, onehot(labels), pos_weight) * weight[m] (labels == C: background row);
    optional grad = scale * d/dlogits.  pos_weight (C,) = CrossEntropyLoss.class_weight in sigmoid mode."""
    _chk(logits, torch.float32, 'logits'); _chk(labels, torch.int64, 'labels')
    M, C = logits.shape
    if pos_weight is not None:
        _chk(pos_weight, torch.float32, 'pos_weight')
        if pos_weight.shape != (C,):
            raise ValueError(f'pos_weight must have shape ({C},), got {tuple(pos_weight.shape)}')
    return _loss_sum('ptb_sigmoid_bce_cw_fwd_bwd', logits, (labels, weight, pos_weight, M, C), scale, want_grad)


def softmax_ce(logits, labels, weight, class_weight=None, scale=None, want_grad=False):
    """sum_m cross_entropy(logits[m], labels[m], weight=class_weight) * weight[m] over rows of C+1 logits (label C: background);
    optional grad = scale * d/dlogits."""
    _chk(logits, torch.float32, 'logits'); _chk(labels, torch.int64, 'labels')
    M, C1 = logits.shape
    if class_weight is not None:
        _chk(class_weight, torch.float32, 'class_weight')
        if class_weight.shape != (C1,):
            raise ValueError(f'class_weight must have shape ({C1},), got {tuple(class_weight.shape)}')
    return _loss_sum('ptb_softmax_ce_fwd_bwd', logits, (labels, weight, class_weight, M, C1), scale, want_grad)


def mse(pred, target, weight, inv_norm, scale=None, want_grad=False):
    """sum ((pred - target) * inv_norm)^2 * weight over (M, 2) points; optional grad = scale * d/dpred."""
    _chk(pred, torch.float32, 'pred'); _chk(target, torch.float32, 'target')
    return _loss_sum('ptb_mse_fwd_bwd', pred, (target, weight, pred.shape[0], float(inv_norm)), scale, want_grad)


def mse_rows(pred, target, weight, row_inv_norm, scale=None, want_grad=False):
    """mse with one normalisation per row of pred (M, 2): row_inv_norm (M,) = 1 / (stride_m * reg_norm)."""
    _chk(pred, torch.float32, 'pred'); _chk(target, torch.float32, 'target'); _chk(row_inv_norm, torch.float32, 'row_inv_norm')
    if row_inv_norm.shape != (pred.shape[0],):
        raise ValueError(f'row_inv_norm must have shape ({pred.shape[0]},), got {tuple(row_inv_norm.shape)}')
    return _loss_sum('ptb_mse_rows_fwd_bwd', pred, (target, weight, pred.shape[0], row_inv_norm), scale, want_grad)


def _chk_shape(t, dtype, name, shape):
    """_chk and an exact shape: the kernels index these tensors by the sizes of the others"""
    _chk(t, dtype, name)
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f'{name} must have shape {tuple(shape)}, got {tuple(t.shape)}')
    return t


def _check_rows(pred, target, row_inv_norm, ndim=None):
    _chk(pred, torch.float32, 'pred'); _chk(target, torch.float32, 'target'); _chk(row_inv_norm, torch.float32, 'row_inv_norm')
    if ndim is not None and pred.dim() != ndim:
        raise ValueError(f'pred must have {ndim} dimensions, got shape {tuple(pred.shape)}')
    if pred.shape[-1] != 2 or target.shape != pred.shape:
        raise ValueError(f'pred and target must be (..., Q, 2) of one shape, got {tuple(pred.shape)} and {tuple(target.shape)}')
    if row_inv_norm.shape != (pred.shape[-2],):
        raise ValueError(f'row_inv_norm must have shape ({pred.shape[-2]},), got {tuple(row_inv_norm.shape)}')


def _check_point_weight(weight, pred):
    if weight is not None:
        _chk_shape(weight, torch.float32, 'weight', pred.shape)


def l1_rows(pred, target, weight, row_inv_norm, scale=None, want_grad=False):
    """sum |(pred - target) * row_inv_norm[m]| * weight over (M, 2) points (L1Loss); optional grad = scale * d/dpred."""
    _check_rows(pred, target, row_inv_norm, 2); _check_point_weight(weight, pred)
    return _loss_sum('ptb_l1_rows_fwd_bwd', pred, (target, weight, pred.shape[0], row_inv_norm), scale, want_grad)


def balanced_l1_rows(pred, target, weight, row_inv_norm, alpha, gamma, beta, scale=None, want_grad=False):
    """BalancedL1Loss(alpha, gamma, beta) summed over (M, 2) normalised points times weight; optional grad = scale * d/dpred."""
    _check_rows(pred, target, row_inv_norm, 2); _check_point_weight(weight, pred)
    return _loss_sum('ptb_balanced_l1_rows_fwd_bwd', pred, (target, weight, pred.shape[0], row_inv_norm,
                                                            float(alpha), float(gamma), float(beta)), scale, want_grad)


def _check_edges(edges, acc_sum, momentum):
    _chk(edges, torch.float32, 'edges')
    bins = edges.numel() - 1
    if not 1 <= bins <= GHM_MAX_BINS:
        raise ValueError(f'GHM takes 1 to {GHM_MAX_BINS} bins (PTB_GHM_MAX_BINS), got {bins}')
    if momentum > 0:
        _chk(acc_sum, torch.float32, 'acc_sum')
        if acc_sum.shape != (bins,):
            raise ValueError(f'acc_sum must have shape ({bins},), got {tuple(acc_sum.shape)}')
    return bins


def _ghm_outputs(B, bins, dev):
    return (torch.empty((B, bins + 1), dtype=torch.int32, device=dev), torch.empty((B, bins), dtype=torch.float32, device=dev),
            torch.empty((B,), dtype=torch.float32, device=dev))


GHM_MAX_BINS = _lib.DEFINES['PTB_GHM_MAX_BINS']        # the edges and counts of a bin histogram live in shared memory


def ghmc_bin_weights(logits, labels, label_weight, edges, momentum=0.0, acc_sum=None):
    """GHMC's histogram and weight step over a batch (B, Q, C) of logits, labels (B, Q) (== C: background) and label_weight (B, Q).
    Returns counts (B, bins + 1) int32 (the last column: valid elements), bin_weight (B, bins) and tot (B,), all on the device; with
    momentum > 0 acc_sum (bins,) is updated in place, image by image."""
    _chk(logits, torch.float32, 'logits'); _chk(labels, torch.int64, 'labels'); _chk(label_weight, torch.float32, 'label_weight')
    if logits.dim() != 3:
        raise ValueError(f'logits must be (B, Q, C), got shape {tuple(logits.shape)}')
    B, Q, C = logits.shape
    if labels.shape != (B, Q) or label_weight.shape != (B, Q):
        raise ValueError(f'labels and label_weight must be ({B}, {Q})')
    bins = _check_edges(edges, acc_sum, momentum)
    counts, bw, tot = _ghm_outputs(B, bins, logits.device)
    _call('ptb_ghmc_bin_weights', logits, labels, label_weight, B, Q, C, edges, bins, float(momentum), acc_sum if momentum > 0 else None,
          counts, bw, tot)
    return counts, bw, tot


def ghmc(logits, labels, label_weight, edges, bin_weight, scale=None, want_grad=False):
    """one image's GHMC sum: sum_q,c BCE-with-logits(logits, onehot(labels)) * bin_weight[bin(q, c)] over valid elements (not yet
    divided by tot); optional grad = scale * d/dlogits.  bin_weight (bins,) is ghmc_bin_weights' row for this image."""
    _chk(logits, torch.float32, 'logits')
    if logits.dim() != 2:
        raise ValueError(f'logits must be (Q, C), got shape {tuple(logits.shape)}')
    Q, C = logits.shape
    bins = _check_edges(edges, None, 0)
    _chk_shape(labels, torch.int64, 'labels', (Q,)); _chk_shape(label_weight, torch.float32, 'label_weight', (Q,))
    _chk_shape(bin_weight, torch.float32, 'bin_weight', (bins,))
    return _loss_sum('ptb_ghmc_fwd_bwd', logits, (labels, label_weight, Q, C, edges, bins, bin_weight), scale, want_grad)


def ghmr_bin_weights(pred, target, weight, row_inv_norm, mu, edges, momentum=0.0, acc_sum=None):
    """GHMR's histogram and weight step over a batch of (B, Q, 2) points (d = (pred - target) * row_inv_norm[q]) and weights; returns
    and updates as ghmc_bin_weights."""
    _check_rows(pred, target, row_inv_norm, 3); _chk(weight, torch.float32, 'weight')
    B, Q, _ = pred.shape
    if weight.shape != pred.shape:
        raise ValueError(f'weight must have shape {tuple(pred.shape)}, got {tuple(weight.shape)}')
    bins = _check_edges(edges, acc_sum, momentum)
    counts, bw, tot = _ghm_outputs(B, bins, pred.device)
    _call('ptb_ghmr_bin_weights', pred, target, weight, row_inv_norm, float(mu), B, Q, edges, bins, float(momentum),
          acc_sum if momentum > 0 else None, counts, bw, tot)
    return counts, bw, tot


def ghmr(pred, target, weight, row_inv_norm, mu, edges, bin_weight, scale=None, want_grad=False):
    """one image's GHMR sum: sum (sqrt(d^2 + mu^2) - mu) * bin_weight[bin] over valid (Q, 2) elements; optional grad = scale * d/dpred."""
    _check_rows(pred, target, row_inv_norm, 2); _chk_shape(weight, torch.float32, 'weight', pred.shape)
    bins = _check_edges(edges, None, 0)
    _chk_shape(bin_weight, torch.float32, 'bin_weight', (bins,))
    return _loss_sum('ptb_ghmr_fwd_bwd', pred, (target, weight, pred.shape[0], row_inv_norm, float(mu), edges,
                                                bins, bin_weight), scale, want_grad)


# ----------------------------------------------------------------------------------------------------------------------
# conv towers on the tensor cores (3xTF32 implicit GEMM + GroupNorm + ReLU)
# ----------------------------------------------------------------------------------------------------------------------
def split_tf32(x):
    _chk(x, torch.float32, 'x')
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    _call('ptb_split_tf32', x, x.numel(), hi, lo)
    return hi, lo


def conv3x3_pack_weight(w):
    """nn.Conv2d weight (Cout,Cin,3,3) -> packed (Cout, 9*Cin) hi / lo."""
    w = _chk(w.detach().contiguous(), torch.float32, 'w')
    Cout, Cin = w.shape[:2]
    hi = torch.empty((Cout, 9 * Cin), dtype=torch.float32, device=w.device)
    lo = torch.empty_like(hi)
    _call('ptb_conv3x3_pack_weight', w, Cout, Cin, hi, lo)
    return hi, lo


def conv3x3_c256(x_hi, x_lo, w_hi, w_lo, want_stats=True):
    """x_* (B,H,W,Cin) channels-last hi/lo; w_* packed (256, 9*Cin) -> y (B,H,W,256), stats (B,32,2) fp64 | None."""
    _chk(x_hi, torch.float32, 'x_hi'); _chk(x_lo, torch.float32, 'x_lo'); _chk(w_hi, torch.float32, 'w_hi'); _chk(w_lo, torch.float32, 'w_lo')
    B, H, W, Cin = x_hi.shape
    if w_hi.shape != (256, 9 * Cin):
        raise ValueError('packed weight must be (256, 9*Cin)')
    y = torch.empty((B, H, W, 256), dtype=torch.float32, device=x_hi.device)
    stats = torch.zeros((B, 32, 2), dtype=torch.float64, device=x_hi.device) if want_stats else None
    _call('ptb_conv3x3_c256_tf32x3', x_hi, x_lo, w_hi, w_lo, B, H, W, Cin, y, stats)
    return y, stats


def gn_relu_apply(y, stats, gamma, beta, groups=32, eps=1e-5, relu=True, split=False):
    """GroupNorm(+ReLU) from the conv epilogue's statistics; split=True returns the (hi, lo) pair for the next conv."""
    _chk(y, torch.float32, 'y'); _chk(stats, torch.float64, 'stats'); _chk(gamma, torch.float32, 'gamma'); _chk(beta, torch.float32, 'beta')
    B, H, W, C = y.shape
    out_hi = torch.empty_like(y)
    out_lo = torch.empty_like(y) if split else None
    _call('ptb_gn_relu_apply', y, stats, gamma, beta, B, H * W, C, groups, float(eps), 1 if relu else 0, out_hi, out_lo)
    return (out_hi, out_lo) if split else out_hi


# ---- fp16 two-term variant (half the tensor-pipe time of 3xTF32) ----
def split_f16(x, auto_scale=False):
    """x fp32 -> (h, l) fp16 with x*scale = h + l; returns (h, l, dev_inv_scale | None)."""
    _chk(x, torch.float32, 'x')
    h = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    l = torch.empty_like(h)
    inv = torch.empty(1, dtype=torch.float32, device=x.device) if auto_scale else None
    ws = torch.empty(1, dtype=torch.int32, device=x.device) if auto_scale else None
    _call('ptb_split_f16', x, x.numel(), 1 if auto_scale else 0, h, l, inv, ws)
    return h, l, inv


def split_f16_from_bf16(x):
    """ptb_split_f16_from_bf16: x bf16 -> (h, l, dev_inv_scale), bit for bit split_f16(x.float(), auto_scale=True) without the fp32 copy."""
    _chk(x, torch.bfloat16, 'x')
    h = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    l = torch.empty_like(h)
    inv = torch.empty(1, dtype=torch.float32, device=x.device)
    ws = torch.empty(1, dtype=torch.int32, device=x.device)
    _call('ptb_split_f16_from_bf16', x, x.numel(), h, l, inv, ws)
    return h, l, inv


def conv3x3_pack_weight_f16(w):
    """(Cout,Cin,3,3) -> packed fp16 (h, l) of w*scale and 1/scale; scale = power of two with max|w|*scale in [2^9, 2^10)."""
    w = _chk(w.detach().contiguous(), torch.float32, 'w')
    Cout, Cin = w.shape[:2]
    amax = float(w.abs().max())
    scale = 1.0
    if amax > 0 and math.isfinite(amax):
        scale = 2.0 ** (10 - math.frexp(amax)[1])
    h = torch.empty((Cout, 9 * Cin), dtype=torch.float16, device=w.device)
    l = torch.empty_like(h)
    _call('ptb_conv3x3_pack_weight_f16', w, Cout, Cin, float(scale), h, l)
    return h, l, 1.0 / scale


def conv3x3_c256_f16(x_h, x_l, w_h, w_l, out_scale, dev_out_scale=None, want_stats=True):
    """tower conv3x3 -> 256 channels with GroupNorm statistics.  x_l None: x_h is an fp16 tensor used as is (lo == 0, ptb_conv_tc_f16x1a)."""
    _chk(x_h, torch.float16, 'x_h'); _chk(w_h, torch.float16, 'w_h'); _chk(w_l, torch.float16, 'w_l')
    B, H, W, Cin = x_h.shape
    if w_h.shape != (256, 9 * Cin):
        raise ValueError('packed weight must be (256, 9*Cin)')
    y = torch.empty((B, H, W, 256), dtype=torch.float32, device=x_h.device)
    stats = torch.zeros((B, 32, 2), dtype=torch.float64, device=x_h.device) if want_stats else None
    if x_l is None:
        _call('ptb_conv_tc_f16x1a', x_h, w_h, w_l, B, H, W, Cin, 9, 256, 256, float(out_scale), dev_out_scale, None, y, 256, stats)
        return y, stats
    _chk(x_l, torch.float16, 'x_l')
    _call('ptb_conv3x3_c256_f16x2', x_h, x_l, w_h, w_l, B, H, W, Cin, float(out_scale), dev_out_scale, y, stats)
    return y, stats


def conv3x3_c256_f16_gn(x_h, x_l, w_h, w_l, out_scale, dev_out_scale, gamma, beta, eps=1e-5, overflow_flag=None, out='f16pair'):
    """ptb_conv3x3_c256_f16_gn: conv3x3_c256_f16 and GroupNorm(32) + ReLU in one launch.  out='f16pair' -> (h, l, y, stats), what
    gn_relu_apply_f16 gives on y and stats; out='fp32' -> (relu(GN(y)), None, y, stats), what gn_relu_apply(split=False) gives.
    x_l None: x_h is an fp16 tensor used as is (lo == 0)."""
    _chk(x_h, torch.float16, 'x_h'); _chk(w_h, torch.float16, 'w_h'); _chk(w_l, torch.float16, 'w_l')
    _chk(gamma, torch.float32, 'gamma'); _chk(beta, torch.float32, 'beta')
    if x_l is not None:
        _chk(x_l, torch.float16, 'x_l')
    if out not in ('f16pair', 'fp32'):
        raise ValueError(f"out must be 'f16pair' or 'fp32', got {out!r}")
    B, H, W, Cin = x_h.shape
    if w_h.shape != (256, 9 * Cin) or gamma.shape != (256,) or beta.shape != (256,):
        raise ValueError('packed weight must be (256, 9*Cin), gamma and beta (256,)')
    dev = x_h.device
    y = torch.empty((B, H, W, 256), dtype=torch.float32, device=dev)
    ws = torch.zeros(B * 64 + (B + 1) // 2, dtype=torch.float64, device=dev)     # statistics [B][32][2], then B int32 counters
    stats = ws[:B * 64].view(B, 32, 2)
    if out == 'f16pair':
        a = torch.empty((B, H, W, 256), dtype=torch.float16, device=dev)
        b = torch.empty_like(a)
    else:
        a, b = torch.empty_like(y), None
    _call('ptb_conv3x3_c256_f16_gn', x_h, x_l, w_h, w_l, B, H, W, Cin, float(out_scale), dev_out_scale, y, ws, gamma, beta, float(eps), a,
          b, overflow_flag)
    return a, b, y, stats


def gn_relu_apply_f16(y, stats, gamma, beta, groups=32, eps=1e-5, relu=True, overflow_flag=None):
    _chk(y, torch.float32, 'y'); _chk(stats, torch.float64, 'stats')
    B, H, W, C = y.shape
    h = torch.empty(y.shape, dtype=torch.float16, device=y.device)
    l = torch.empty_like(h)
    _call('ptb_gn_relu_apply_f16', y, stats, gamma, beta, B, H * W, C, groups, float(eps), 1 if relu else 0, h, l, overflow_flag)
    return h, l


def gn_relu_bwd(da, y, stats, gamma, beta, groups=32, eps=1e-5, relu=True, want_amax=True):
    """ptb_gn_relu_bwd: backward of GroupNorm(+ReLU) on channels-last (B,H,W,C) tensors.
    returns dy (B,H,W,C) fp32, dgamma (C,), dbeta (C,), amax_bits (1,) int32 device (float bits of max|dy|) | None."""
    _chk(da, torch.float32, 'da'); _chk(y, torch.float32, 'y'); _chk(stats, torch.float64, 'stats')
    B, H, W, C = y.shape
    dev = y.device
    nbytes = int(_lib.load().ptb_gn_relu_bwd_workspace(B, H * W, C, groups))
    if nbytes == 0:
        raise ValueError(f'ptb_gn_relu_bwd: unsupported shape C={C}, groups={groups}')
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dy = torch.empty_like(y)
    dg = torch.empty(C, dtype=torch.float32, device=dev)
    db = torch.empty(C, dtype=torch.float32, device=dev)
    amax = torch.zeros(1, dtype=torch.int32, device=dev) if want_amax else None
    _call('ptb_gn_relu_bwd', da, y, stats, gamma, beta, B, H * W, C, groups, float(eps), 1 if relu else 0, ws, dy, dg, db, amax)
    return dy, dg, db, amax


def split_f16_amax(x, amax_bits):
    """x fp32 -> (h, l, dev_inv_scale) with the power-of-two scale chosen on the device from amax_bits (float bits of max|x|)."""
    _chk(x, torch.float32, 'x')
    h = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    l = torch.empty_like(h)
    inv = torch.empty(1, dtype=torch.float32, device=x.device)
    _call('ptb_split_f16_amax', x, x.numel(), amax_bits, h, l, inv)
    return h, l, inv


def conv_tc_wgrad_f16(dy_h, dy_l, x_h, x_l, taps, scale=1.0, dev_scale_dy=None, dev_scale_x=None, out=None, accumulate=False):
    """dW (Cout, 256, 3, 3) of a conv3x3 (taps 9) or (Cout, 256) of a per-cell Linear (taps 1) (+)= scale * s_dy * s_x *
    sum_pixels dy (x) x_shifted from fp16 operand pairs dy (B,H,W,Cout) and x (B,H,W,256); tensor cores with K = pixels, deterministic.
    One ptb_conv_tc_wgrad_f16x2_ld launch per column slice of <= 256 (the wgrad's widest output) of dy, read in place (row stride
    Cout), writing rows [c0, c0 + n) of dW.  Cout a multiple of 8.  accumulate: add into out."""
    _chk(dy_h, torch.float16, 'dy_h'); _chk(dy_l, torch.float16, 'dy_l'); _chk(x_h, torch.float16, 'x_h'); _chk(x_l, torch.float16, 'x_l')
    B, H, W, Cout = dy_h.shape
    Cin = x_h.shape[3]
    ws = torch.empty(int(_lib.load().ptb_conv_tc_wgrad_workspace(B, H, W, taps)), dtype=torch.uint8, device=dy_h.device)
    dw = out if out is not None else torch.empty((Cout, Cin, 3, 3) if taps == 9 else (Cout, Cin), dtype=torch.float32, device=dy_h.device)
    for c0 in range(0, Cout, CONV_TC_WGRAD_N_MAX):
        n = min(CONV_TC_WGRAD_N_MAX, Cout - c0)
        _call('ptb_conv_tc_wgrad_f16x2_ld', dy_h[..., c0:], dy_l[..., c0:], Cout, x_h, x_l, B, H, W, n, Cin, taps, float(scale),
              dev_scale_dy, dev_scale_x, ws, dw[c0:], 1 if accumulate else 0)
    return dw


def col_sum(y2d):
    """ptb_col_sum: out[n] = sum_m y[m][n] of a contiguous fp32 (M, N) matrix, fixed order."""
    _chk(y2d, torch.float32, 'y2d')
    M, N = y2d.shape
    ws = torch.empty(int(_lib.load().ptb_col_sum_workspace(M, N)) // 4, dtype=torch.float32, device=y2d.device)
    out = torch.empty(N, dtype=torch.float32, device=y2d.device)
    _call('ptb_col_sum', y2d, M, N, N, ws, out)
    return out


CONV_TC_N_MAX = 512         # widest output of one ptb_conv_tc_f16x2 launch
CONV_TC_WGRAD_N_MAX = 256   # widest output of one ptb_conv_tc_wgrad_f16x2_ld launch


def _pack_slice_f16(w, taps):
    w = _chk(w.detach().contiguous(), torch.float32, 'w')
    n_out, Cin = w.shape[0], w.shape[1]
    n_mma = (n_out + 15) // 16 * 16
    amax = float(w.abs().max())
    scale = 2.0 ** (10 - math.frexp(amax)[1]) if (amax > 0 and math.isfinite(amax)) else 1.0
    h = torch.empty((n_mma, taps * Cin), dtype=torch.float16, device=w.device)
    l = torch.empty_like(h)
    _call('ptb_conv_tc_pack_weight_f16', w, n_out, n_mma, Cin, taps, float(scale), h, l)
    return h, l, 1.0 / scale, n_mma


def conv_tc_pack_weight_f16(w, taps):
    """weights of a conv3x3 (n_out,Cin,3,3) or Linear / conv1x1 (n_out,Cin) -> column slices of <= CONV_TC_N_MAX output rows for
    conv_tc_f16, each packed as fp16 (h, l) with its own power-of-two scale: [(c0, n, (h, l, 1/scale, n_mma)), ...]."""
    return [(c0, min(CONV_TC_N_MAX, w.shape[0] - c0), _pack_slice_f16(w[c0:c0 + CONV_TC_N_MAX], taps))
            for c0 in range(0, w.shape[0], CONV_TC_N_MAX)]


HALF_DTYPES = {torch.float16: _lib.DEFINES['PTB_DTYPE_F16'], torch.bfloat16: _lib.DEFINES['PTB_DTYPE_BF16']}


def conv_tc_f16(x_h, x_l, packs, taps, n_out, bias=None, dev_out_scale=None, ldy=None, out_dtype=torch.float32):
    """general wgmma conv (taps 1|9) on fp16 operand pairs -> (B,H,W,ldy) fp32 (+bias), at any n_out: one launch per column slice
    of conv_tc_pack_weight_f16, each writing columns [c0, c0 + n) of the one map.  x_l None: x_h is an fp16 tensor used as is
    (lo == 0: ptb_conv_tc_f16x1a).  out_dtype fp16 / bf16: the fp32 result rounded to nearest even in the epilogue
    (ptb_conv_tc_f16x2_half_out), the input gradient of a half-precision feature map."""
    _chk(x_h, torch.float16, 'x_h')
    if x_l is None:
        if out_dtype != torch.float32:
            raise NotImplementedError('conv_tc_f16: a half-precision output of the lo == 0 variant')
    else:
        _chk(x_l, torch.float16, 'x_l')
    if out_dtype != torch.float32 and out_dtype not in HALF_DTYPES:
        raise TypeError(f'conv_tc_f16: out_dtype must be float32, float16 or bfloat16, got {out_dtype}')
    if packs[-1][0] + packs[-1][1] != n_out:
        raise ValueError(f'conv_tc_f16: the packed slices cover {packs[-1][0] + packs[-1][1]} columns, not n_out = {n_out}')
    B, H, W, Cin = x_h.shape
    ldy = ldy or (n_out + 3) // 4 * 4
    y = torch.empty((B, H, W, ldy), dtype=out_dtype, device=x_h.device)
    for c0, n, (w_h, w_l, inv_w, n_mma) in packs:
        yc, bc = y[..., c0:], (bias[c0:c0 + n] if bias is not None else None)
        if x_l is None:
            _call('ptb_conv_tc_f16x1a', x_h, w_h, w_l, B, H, W, Cin, taps, n, n_mma, float(inv_w), dev_out_scale, bc, yc, ldy, None)
        elif out_dtype == torch.float32:
            _call('ptb_conv_tc_f16x2', x_h, x_l, w_h, w_l, B, H, W, Cin, taps, n, n_mma, float(inv_w), dev_out_scale, bc, yc, ldy)
        else:
            _call('ptb_conv_tc_f16x2_half_out', x_h, x_l, w_h, w_l, B, H, W, Cin, taps, n, n_mma, float(inv_w), dev_out_scale, bc, yc,
                  HALF_DTYPES[out_dtype], ldy)
    return y


# ---- RPN training (ptb_rpn_*): targets, sampling plan and losses of AnchorHead.loss with RandomSampler
RPN_MAX_LEVELS = _lib.DEFINES['PTB_RPN_MAX_LEVELS']
RPN_LOSS_L1, RPN_LOSS_SMOOTH_L1 = _lib.DEFINES['PTB_RPN_LOSS_L1'], _lib.DEFINES['PTB_RPN_LOSS_SMOOTH_L1']


def _level_arrays(featmap_sizes, strides_wh):
    L = len(featmap_sizes)
    if not 1 <= L <= RPN_MAX_LEVELS:
        raise ValueError(f'1 to {RPN_MAX_LEVELS} levels, got {L}')
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for s in featmap_sizes for v in s])
    st = (ctypes.c_int32 * (2 * L))(*[int(v) for s in strides_wh for v in s])
    return L, hw, st


def rpn_inside_anchors(base_anchors, featmap_sizes, strides_wh, inside_box):
    """ptb_rpn_inside_anchors.  base_anchors (L, A, 4) fp32, inside_box (B, L, A, 4) int32 (x0, x1, y0, y1).
    returns inside_anchors (B, N, 4) (image b's first n_inside[b] rows), inside_idx (B, N) int32, n_inside (B,) int32."""
    _chk(base_anchors, torch.float32, 'base_anchors'); _chk(inside_box, torch.int32, 'inside_box')
    L, hw, st = _level_arrays(featmap_sizes, strides_wh)
    A = base_anchors.shape[1]
    B = inside_box.shape[0]
    if tuple(base_anchors.shape) != (L, A, 4) or tuple(inside_box.shape) != (B, L, A, 4):
        raise ValueError('base_anchors must be (L, A, 4) and inside_box (B, L, A, 4)')
    N = sum(int(h) * int(w) * A for h, w in featmap_sizes)
    dev = base_anchors.device
    anchors = torch.empty((B, N, 4), dtype=torch.float32, device=dev)
    idx = torch.empty((B, N), dtype=torch.int32, device=dev)
    n_inside = torch.empty((B,), dtype=torch.int32, device=dev)
    _call('ptb_rpn_inside_anchors', base_anchors, hw, st, L, A, B, inside_box, anchors, idx, n_inside)
    return anchors, idx, n_inside


def rpn_candidate_ranks(gt_inds, n_inside):
    """ptb_rpn_candidate_ranks.  gt_inds (B, N) int64, n_inside (B,) int32 -> rank (B, N) int32, counts (B, 2) int32 (pos, neg)."""
    _chk(gt_inds, torch.int64, 'gt_inds'); _chk(n_inside, torch.int32, 'n_inside')
    B, N = gt_inds.shape
    if tuple(n_inside.shape) != (B,):
        raise ValueError(f'n_inside must have shape ({B},)')
    rank = torch.empty((B, N), dtype=torch.int32, device=gt_inds.device)
    counts = torch.empty((B, 2), dtype=torch.int32, device=gt_inds.device)
    _call('ptb_rpn_candidate_ranks', gt_inds, n_inside, B, N, rank, counts)
    return rank, counts


def rpn_anchor_targets(featmap_sizes, strides_wh, A, inside_idx, inside_anchors, gt_inds, rank, plan, gt_bboxes, gt_off, means, stds,
                       pos_weight):
    """ptb_rpn_anchor_targets.  returns labels (int64), label_weights like the concatenated cls_score maps (B*A*H*W per level, level
    after level) and bbox_targets, bbox_weights like the concatenated bbox_pred maps (B*4A*H*W per level)."""
    L, hw, st = _level_arrays(featmap_sizes, strides_wh)
    B, N = inside_idx.shape
    for t, dt, name in ((inside_idx, torch.int32, 'inside_idx'), (inside_anchors, torch.float32, 'inside_anchors'),
                        (gt_inds, torch.int64, 'gt_inds'), (rank, torch.int32, 'rank'), (plan, torch.int32, 'plan'),
                        (gt_bboxes, torch.float32, 'gt_bboxes'), (gt_off, torch.int32, 'gt_off')):
        _chk(t, dt, name)
    if N != sum(int(h) * int(w) * A for h, w in featmap_sizes) or tuple(inside_anchors.shape) != (B, N, 4) or \
            tuple(gt_inds.shape) != (B, N) or tuple(rank.shape) != (B, N) or tuple(gt_off.shape) != (B + 1,) or \
            gt_bboxes.dim() != 2 or gt_bboxes.shape[1] != 4 or plan.numel() < 4 * B:
        raise ValueError('rpn_anchor_targets: inconsistent shapes')
    dev = inside_idx.device
    labels = torch.empty((B * N,), dtype=torch.int64, device=dev)
    lw = torch.empty((B * N,), dtype=torch.float32, device=dev)
    bt = torch.empty((B * N * 4,), dtype=torch.float32, device=dev)
    bw = torch.empty((B * N * 4,), dtype=torch.float32, device=dev)
    mean = (ctypes.c_float * 4)(*[float(v) for v in means])
    std = (ctypes.c_float * 4)(*[float(v) for v in stds])
    _call('ptb_rpn_anchor_targets', hw, st, L, A, B, inside_idx, inside_anchors, gt_inds, rank, plan, gt_bboxes, gt_off, mean, std,
          float(pos_weight), labels, lw, bt, bw)
    return labels, lw, bt, bw


def rpn_sampled_indices(gt_inds, rank, plan, n_pos, n_neg):
    """ptb_rpn_sampled_indices for one image: the sampled positive and negative rows (int64, ascending)."""
    _chk(gt_inds, torch.int64, 'gt_inds'); _chk(rank, torch.int32, 'rank'); _chk(plan, torch.int32, 'plan')
    n = gt_inds.numel()
    if rank.numel() != n or plan.numel() < 4:
        raise ValueError('rpn_sampled_indices: inconsistent shapes')
    pos = torch.empty((n_pos,), dtype=torch.int64, device=gt_inds.device)
    neg = torch.empty((n_neg,), dtype=torch.int64, device=gt_inds.device)
    _call('ptb_rpn_sampled_indices', gt_inds, rank, n, plan, pos, neg)
    return pos, neg


def rpn_level_loss(cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, bbox_loss, beta, scale=None, want_grad=False):
    """ptb_rpn_level_loss on one level's maps cls_score (B, A, H, W) / bbox_pred (B, 4A, H, W) and its target slices.  Returns the
    (2,) un-normalised sums (cls, bbox) or, with want_grad, (scale[0] d/dcls_score, scale[1] d/dbbox_pred)."""
    _chk(cls_score, torch.float32, 'cls_score'); _chk(bbox_pred, torch.float32, 'bbox_pred')
    M = cls_score.numel()
    if bbox_pred.numel() != 4 * M or labels.numel() != M or label_weights.numel() != M or bbox_targets.numel() != 4 * M or \
            bbox_weights.numel() != 4 * M:
        raise ValueError('rpn_level_loss: inconsistent sizes')
    _chk(labels, torch.int64, 'labels'); _chk(label_weights, torch.float32, 'label_weights')
    _chk(bbox_targets, torch.float32, 'bbox_targets'); _chk(bbox_weights, torch.float32, 'bbox_weights')
    if want_grad:
        _chk(scale, torch.float32, 'scale')
        gc, gb = torch.empty_like(cls_score), torch.empty_like(bbox_pred)
        _call('ptb_rpn_level_loss', cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, M, int(bbox_loss), float(beta),
              None, scale, gc, gb)
        return gc, gb
    loss = torch.zeros(2, dtype=torch.float32, device=cls_score.device)
    _call('ptb_rpn_level_loss', cls_score, bbox_pred, labels, label_weights, bbox_targets, bbox_weights, M, int(bbox_loss), float(beta),
          loss, None, None, None)
    return loss


# ---- RoI head (ptb_roi_*): multi-level RoIAlign, RoI targets, box loss, accuracy and test decode of StandardRoIHead's bbox branch
ROI_MAX_LEVELS = _lib.DEFINES['PTB_ROI_MAX_LEVELS']


def _roi_level_arrays(maps_nhwc, strides):
    L = len(maps_nhwc)
    if not 1 <= L <= ROI_MAX_LEVELS or len(strides) != L:
        raise ValueError(f'1 to {ROI_MAX_LEVELS} levels with one stride each, got {L} maps and {len(strides)} strides')
    B, C = maps_nhwc[0].shape[0], maps_nhwc[0].shape[3]
    for m in maps_nhwc:
        _chk(m, torch.float32, 'feature map')
        if m.dim() != 4 or m.shape[0] != B or m.shape[3] != C:
            raise ValueError('feature maps must be channels-last (B, H, W, C) with the same B and C')
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for m in maps_nhwc for v in m.shape[1:3]])
    st = (ctypes.c_float * L)(*[float(s) for s in strides])
    ptrs = (ctypes.c_void_p * L)(*[m.data_ptr() for m in maps_nhwc])
    return L, B, C, hw, st, ptrs


def roi_align_fwd(maps_nhwc, strides, rois, out_size, sampling_ratio, finest_scale):
    """ptb_roi_align_fwd.  maps_nhwc: per level (B, H, W, C) fp32 contiguous; rois (R, 5).
    returns features (R, C, out, out) and levels (R,) int32."""
    _chk(rois, torch.float32, 'rois')
    L, B, C, hw, st, ptrs = _roi_level_arrays(maps_nhwc, strides)
    R = rois.shape[0]
    y = torch.empty((R, C, out_size, out_size), dtype=torch.float32, device=rois.device)
    lv = torch.empty((R,), dtype=torch.int32, device=rois.device)
    _call('ptb_roi_align_fwd', ptrs, hw, st, L, B, C, rois, R, int(out_size), int(sampling_ratio), float(finest_scale), y, lv)
    return y, lv


def roi_align_bwd(grad_y, map_shapes, strides, rois, levels, sampling_ratio):
    """ptb_roi_align_bwd: the gradients (B, H, W, C) of the channels-last maps of shapes map_shapes (zero where no RoI reads)."""
    _chk(grad_y, torch.float32, 'grad_y'); _chk(rois, torch.float32, 'rois'); _chk(levels, torch.int32, 'levels')
    grads = [torch.zeros(s, dtype=torch.float32, device=grad_y.device) for s in map_shapes]
    L, B, C, hw, st, ptrs = _roi_level_arrays(grads, strides)
    R, out = grad_y.shape[0], grad_y.shape[-1]
    if tuple(grad_y.shape) != (R, C, out, out) or rois.shape[0] != R or levels.shape != (R,):
        raise ValueError('roi_align_bwd: inconsistent shapes')
    _call('ptb_roi_align_bwd', ptrs, hw, st, L, B, C, rois, levels, R, int(out), int(sampling_ratio), grad_y)
    return grads


def roi_targets(cand, gt_inds, rank, plan, row_off, gt_bboxes, gt_off, gt_labels, num_classes, means, stds, pos_weight, R):
    """ptb_roi_targets.  returns rois (R, 5), labels (R,) int64, label_weights (R,), bbox_targets (R, 4), bbox_weights (R, 4)."""
    B, N = gt_inds.shape
    for t, dt, name in ((cand, torch.float32, 'cand'), (gt_inds, torch.int64, 'gt_inds'), (rank, torch.int32, 'rank'),
                        (plan, torch.int32, 'plan'), (row_off, torch.int32, 'row_off'), (gt_bboxes, torch.float32, 'gt_bboxes'),
                        (gt_off, torch.int32, 'gt_off'), (gt_labels, torch.int64, 'gt_labels')):
        _chk(t, dt, name)
    if tuple(cand.shape) != (B, N, 4) or tuple(rank.shape) != (B, N) or row_off.numel() != 2 * B or tuple(gt_off.shape) != (B + 1,) or \
            plan.numel() < 4 * B or gt_bboxes.shape[-1] != 4 or gt_labels.shape[0] != gt_bboxes.shape[0]:
        raise ValueError('roi_targets: inconsistent shapes')
    dev = cand.device
    rois = torch.empty((R, 5), dtype=torch.float32, device=dev)
    labels = torch.empty((R,), dtype=torch.int64, device=dev)
    lw = torch.empty((R,), dtype=torch.float32, device=dev)
    bt = torch.empty((R, 4), dtype=torch.float32, device=dev)
    bw = torch.empty((R, 4), dtype=torch.float32, device=dev)
    mean = (ctypes.c_float * 4)(*[float(v) for v in means])
    std = (ctypes.c_float * 4)(*[float(v) for v in stds])
    _call('ptb_roi_targets', B, N, cand, gt_inds, rank, plan, row_off, gt_bboxes, gt_off, gt_labels, int(num_classes), mean, std,
          float(pos_weight), rois, labels, lw, bt, bw)
    return rois, labels, lw, bt, bw


def roi_bbox_loss(bbox_pred, labels, bbox_targets, bbox_weights, num_classes, class_agnostic, bbox_loss, beta, scale=None,
                  want_grad=False):
    """ptb_roi_bbox_loss: the (1,) un-normalised box-loss sum over the positive rows, or with want_grad the gradient
    scale * d/dbbox_pred (zero outside the positive rows' class columns)."""
    _chk(bbox_pred, torch.float32, 'bbox_pred'); _chk(labels, torch.int64, 'labels')
    _chk(bbox_targets, torch.float32, 'bbox_targets'); _chk(bbox_weights, torch.float32, 'bbox_weights')
    R, ld = bbox_pred.shape
    if labels.shape != (R,) or tuple(bbox_targets.shape) != (R, 4) or tuple(bbox_weights.shape) != (R, 4):
        raise ValueError('roi_bbox_loss: inconsistent shapes')
    if want_grad:
        _chk(scale, torch.float32, 'scale')
        g = torch.zeros_like(bbox_pred)
        _call('ptb_roi_bbox_loss', bbox_pred, ld, labels, bbox_targets, bbox_weights, R, int(num_classes), int(bool(class_agnostic)),
              int(bbox_loss), float(beta), None, scale, g)
        return g
    loss = torch.zeros(1, dtype=torch.float32, device=bbox_pred.device)
    _call('ptb_roi_bbox_loss', bbox_pred, ld, labels, bbox_targets, bbox_weights, R, int(num_classes), int(bool(class_agnostic)),
          int(bbox_loss), float(beta), loss, None, None)
    return loss


def roi_accuracy(cls_score, labels):
    """ptb_roi_accuracy: top-1 accuracy in percent (losses/accuracy.py), (1,) fp32."""
    _chk(cls_score, torch.float32, 'cls_score'); _chk(labels, torch.int64, 'labels')
    R, C1 = cls_score.shape
    out = torch.empty((1,), dtype=torch.float32, device=cls_score.device)
    _call('ptb_roi_accuracy', cls_score, labels, R, C1, float(100.0 / R), out)
    return out


def roi_decode(rois, cls_score, bbox_pred, B, num_classes, class_agnostic, means, stds, max_ratio, img_hw, scale_factor=None):
    """ptb_roi_decode over B images of N padded RoI rows.  returns boxes (B, N, C, 4) and foreground scores (B, N, C)."""
    for t, name in ((rois, 'rois'), (cls_score, 'cls_score'), (bbox_pred, 'bbox_pred'), (img_hw, 'img_hw')):
        _chk(t, torch.float32, name)
    M = rois.shape[0]
    N = M // B
    C = int(num_classes)
    if M != B * N or tuple(cls_score.shape) != (M, C + 1) or tuple(bbox_pred.shape) != (M, 4 if class_agnostic else 4 * C) or \
            tuple(img_hw.shape) != (B, 2):
        raise ValueError('roi_decode: inconsistent shapes')
    if scale_factor is not None:
        _chk(scale_factor, torch.float32, 'scale_factor')
    boxes = torch.empty((B, N, C, 4), dtype=torch.float32, device=rois.device)
    scores = torch.empty((B, N, C), dtype=torch.float32, device=rois.device)
    mean = (ctypes.c_float * 4)(*[float(v) for v in means])
    std = (ctypes.c_float * 4)(*[float(v) for v in stds])
    _call('ptb_roi_decode', rois, cls_score, bbox_pred, B, N, C, int(bool(class_agnostic)), mean, std, float(max_ratio), img_hw,
          scale_factor, boxes, scores)
    return boxes, scores


# ---- test-time augmentation and tile testing (ptb_box_map / ptb_aug_merge / ptb_batched_nms / ptb_tile_concat)
BATCHED_NMS_MAX_ROWS = _lib.DEFINES['PTB_BATCHED_NMS_MAX_ROWS']
FLIP_DIRECTIONS = {'horizontal': 1, 'vertical': 2, 'diagonal': 3}


def aug_meta(img_metas, segments, roi_batch, device):
    """the (G, 12) meta rows of ptb_box_map / ptb_aug_merge: segment, RoI batch index, scale_factor[4], flip, img_h, img_w, has_offset,
    dx, dy of each aug's meta dict (uploaded in one copy)"""
    rows = []
    for m, s, r in zip(img_metas, segments, roi_batch):
        sf = np.asarray(m['scale_factor'], np.float32).reshape(-1) * np.ones(4, np.float32)
        flip = FLIP_DIRECTIONS[m.get('flip_direction') or 'horizontal'] if m.get('flip', False) else 0
        off = m.get('tile_offset', None)
        rows.append([s, r, *sf.tolist(), flip, float(m['img_shape'][0]), float(m['img_shape'][1]), float(off is not None),
                     *(np.float32(v) for v in (off if off is not None else (0, 0)))])
    return torch.tensor(np.array(rows, np.float32)).pin_memory().to(device, non_blocking=True)


def box_map(boxes, counts, meta, want_keep=False):
    """ptb_box_map: boxes (S, N, ld >= 4) fp32, counts (S,) int32 or None, meta (G, 12) -> rois (G, N, 5) [, keep (G, N) bool]"""
    _chk(boxes, torch.float32, 'boxes'); _chk(meta, torch.float32, 'meta')
    if counts is not None:
        _chk(counts, torch.int32, 'counts')
    S, N, ld = boxes.shape
    G = meta.shape[0]
    rois = torch.empty((G, N, 5), dtype=torch.float32, device=boxes.device)
    keep = torch.empty((G, N), dtype=torch.bool, device=boxes.device) if want_keep else None
    _call('ptb_box_map', boxes, ld, counts, N, G, meta, rois, keep)
    return (rois, keep) if want_keep else rois


def proposal_map_back(det, counts, meta, A):
    """ptb_proposal_map_back: det (T*A, N, 5) proposals and counts (T*A,) int32 of every aug -> (T, A*N, 5) recovered and concatenated
    per tile, count (T,)"""
    _chk(det, torch.float32, 'det'); _chk(counts, torch.int32, 'counts'); _chk(meta, torch.float32, 'meta')
    G, N = det.shape[:2]
    if G % A or det.shape[2] != 5 or meta.shape[0] != G:
        raise ValueError('proposal_map_back: inconsistent shapes')
    T = G // A
    out = torch.empty((T, A * N, 5), dtype=torch.float32, device=det.device)
    cnt = torch.empty((T,), dtype=torch.int32, device=det.device)
    _call('ptb_proposal_map_back', det, counts, N, T, A, meta, out, cnt)
    return out, cnt


def aug_merge(boxes, scores, counts, meta, A, box_cols):
    """ptb_aug_merge: boxes (T*A, N, C, 4) and scores (T*A, N, C) of ptb_roi_decode -> merged (T, N, C, 4), (T, N, C)"""
    _chk(boxes, torch.float32, 'boxes'); _chk(scores, torch.float32, 'scores'); _chk(meta, torch.float32, 'meta')
    if counts is not None:
        _chk(counts, torch.int32, 'counts')
    G, N, C = scores.shape
    if G % A or tuple(boxes.shape) != (G, N, C, 4) or meta.shape[0] != G:
        raise ValueError('aug_merge: inconsistent shapes')
    if not 1 <= A <= 63:
        raise NotImplementedError(f'{A} augs per tile: 1 to 63 are implemented')
    T = G // A
    ob = torch.empty((T, N, C, 4), dtype=torch.float32, device=boxes.device)
    os_ = torch.empty((T, N, C), dtype=torch.float32, device=boxes.device)
    _call('ptb_aug_merge', boxes, scores, N, C, int(box_cols), counts, T, A, meta, ob, os_)
    return ob, os_


def batched_nms(boxes, scores, labels, counts, iou_thr, split_thr=10000, max_num=-1):
    """ptb_batched_nms: mmcv batched_nms (labels (S, N) int32) or nms (labels None) of S segments.  boxes (S, N, ld >= 4) and scores
    (S, N) or (S, N, lds) views of contiguous rows (scores may be boxes[..., 4]), counts (S,) int32 or None.
    returns count (S,), det (S, N, 5), label (S, N) or None, keep (S, N) int32 in output order."""
    if boxes.dim() != 3 or not boxes.is_cuda or boxes.dtype != torch.float32 or boxes.stride(2) != 1 or boxes.stride(0) != boxes.shape[1] * boxes.stride(1):
        raise ValueError('batched_nms: boxes must be (S, N, ld) fp32 CUDA rows with unit column stride')
    S, N = boxes.shape[:2]
    if N > BATCHED_NMS_MAX_ROWS:
        raise NotImplementedError(f'batched_nms over {N} rows: at most {BATCHED_NMS_MAX_ROWS} (PTB_BATCHED_NMS_MAX_ROWS) are implemented')
    if not scores.is_cuda or scores.dtype != torch.float32 or scores.shape[:2] != (S, N) or scores.stride(0) != N * scores.stride(1):
        raise ValueError('batched_nms: scores must be (S, N) fp32 CUDA with row-major segments')
    if labels is not None:
        _chk(labels, torch.int32, 'labels')
    if counts is not None:
        _chk(counts, torch.int32, 'counts')
    dev = boxes.device
    cnt = torch.empty((S,), dtype=torch.int32, device=dev)
    det = torch.empty((S, N, 5), dtype=torch.float32, device=dev)
    lab = torch.empty((S, N), dtype=torch.int32, device=dev) if labels is not None else None
    keep = torch.empty((S, N), dtype=torch.int32, device=dev)
    nbytes = int(_lib.load().ptb_batched_nms_workspace(S, N))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _call('ptb_batched_nms', boxes, boxes.stride(1), scores, scores.stride(1), labels, counts, S, N, float(iou_thr), int(split_thr),
          int(max_num), cnt, det, lab, keep, ws, nbytes)
    return cnt, det, lab, keep


def tile_concat(det, labels, counts, offsets, scale_factor=None):
    """ptb_tile_concat: det (T, K, 5), labels (T, K) int32, counts (T,) int32, offsets (T, 2), scale_factor (T, 4) or None
    -> rows (T*K, 5), labels (T*K,), count (1,)"""
    _chk(det, torch.float32, 'det'); _chk(labels, torch.int32, 'labels'); _chk(counts, torch.int32, 'counts')
    _chk(offsets, torch.float32, 'offsets')
    if scale_factor is not None:
        _chk(scale_factor, torch.float32, 'scale_factor')
    T, K = labels.shape
    out = torch.empty((T * K, 5), dtype=torch.float32, device=det.device)
    lab = torch.empty((T * K,), dtype=torch.int32, device=det.device)
    cnt = torch.empty((1,), dtype=torch.int32, device=det.device)
    _call('ptb_tile_concat', det, labels, counts, T, K, scale_factor, offsets, out, lab, cnt)
    return out, lab, cnt


# ---- FCOS head (ptb_fcos_*): targets, loss normalisers, box and centerness losses, decode
FCOS_MAX_LEVELS = 8                    # levels of one ptb_fcos_* launch
FCOS_BOX_LOSS_MODES = {'IoULoss': 0, 'IoULoss_linear': 1, 'GIoULoss': 2}


def _fcos_levels(featmap_sizes, strides):
    L = len(featmap_sizes)
    if not 1 <= L <= FCOS_MAX_LEVELS or len(strides) != L:
        raise ValueError(f'{L} feature maps and {len(strides)} strides: 1 to {FCOS_MAX_LEVELS} levels, one stride each')
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for s in featmap_sizes for v in s])
    st = (ctypes.c_float * L)(*[float(s) for s in strides])
    return L, hw, st


def fcos_targets(featmap_sizes, strides, B, gt_bboxes, gt_labels, gt_off, ranges, radius_px, norm_on_bbox, num_classes):
    """ptb_fcos_targets: gt_bboxes (G, 4) fp32, gt_labels (G,) int64, gt_off (B+1,) int32 CSR offsets of the batch's GTs, ranges (L, 2)
    fp32 on the device, radius_px (L,) fp32 or None -> labels (N,) int64, bbox_targets (N, 4) fp32 in level / image / y / x row order."""
    L, hw, st = _fcos_levels(featmap_sizes, strides)
    _chk(gt_off, torch.int32, 'gt_off'); _chk(ranges, torch.float32, 'ranges')
    if gt_off.shape != (B + 1,) or ranges.shape != (L, 2):
        raise ValueError(f'gt_off must be ({B + 1},) and ranges ({L}, 2)')
    if gt_bboxes is not None:
        _chk(gt_bboxes, torch.float32, 'gt_bboxes'); _chk(gt_labels, torch.int64, 'gt_labels')
    if radius_px is not None:
        _chk(radius_px, torch.float32, 'radius_px')
    N = B * sum(int(h) * int(w) for h, w in featmap_sizes)
    dev = gt_off.device
    labels = torch.empty((N,), dtype=torch.int64, device=dev)
    targets = torch.empty((N, 4), dtype=torch.float32, device=dev)
    _call('ptb_fcos_targets', gt_bboxes, gt_labels, gt_off, B, L, hw, st, ranges, radius_px, int(bool(norm_on_bbox)), int(num_classes),
          labels, targets)
    return labels, targets


def fcos_norm_sums(labels, targets, num_classes):
    """ptb_fcos_norm_sums: (2,) fp32 [number of positive rows, sum of their centerness targets], on the device"""
    _chk(labels, torch.int64, 'labels'); _chk(targets, torch.float32, 'targets')
    out = torch.zeros(2, dtype=torch.float32, device=labels.device)
    _call('ptb_fcos_norm_sums', labels, targets, labels.shape[0], int(num_classes), out)
    return out


def fcos_bbox_loss(pred, targets, labels, featmap_sizes, strides, B, num_classes, mode, overlap_eps, eps, scale=None, want_grad=False):
    """ptb_fcos_bbox_loss: the (1,) sum of the centerness-weighted IoU / GIoU loss over the positive rows of pred (N, 4), or with
    want_grad the gradient scale * d/dpred (zero rows for negatives)."""
    _chk(pred, torch.float32, 'pred'); _chk(targets, torch.float32, 'targets'); _chk(labels, torch.int64, 'labels')
    L, hw, st = _fcos_levels(featmap_sizes, strides)
    return _loss_sum('ptb_fcos_bbox_loss', pred, (targets, labels, B, L, hw, st, int(num_classes), int(mode),
                                                  float(overlap_eps), float(eps)), scale, want_grad)


def fcos_centerness_loss(logits, targets, labels, num_classes, scale=None, want_grad=False):
    """ptb_fcos_centerness_loss: the (1,) sum of the soft-target centerness BCE over the positive rows of logits (N,), or its gradient"""
    _chk(logits, torch.float32, 'logits'); _chk(targets, torch.float32, 'targets'); _chk(labels, torch.int64, 'labels')
    return _loss_sum('ptb_fcos_centerness_loss', logits, (targets, labels, logits.shape[0], int(num_classes)), scale, want_grad)


def fcos_decode_rows(featmap_sizes, nms_pre):
    """rows per image each level keeps: nms_pre when 0 < nms_pre < H*W (get_k_for_topk), else H*W"""
    return [nms_pre if 0 < nms_pre < h * w else h * w for h, w in featmap_sizes]


def fcos_decode(cls_maps, reg_maps, ctr_maps, strides, num_classes, img_hw, nms_pre, scale_factor=None):
    """ptb_fcos_decode: channels-last maps cls (B,H,W,C), reg (B,H,W,4), ctr (B,H,W,1) per level, img_hw (B, 2) fp32, scale_factor (B, 4)
    fp32 or None -> idx (B,R) int32 cells, boxes (B,R,4), scores (B,R,C), centerness (B,R), the levels' rows in level order."""
    hw_list = [(int(c.shape[1]), int(c.shape[2])) for c in cls_maps]
    L, hw, st = _fcos_levels(hw_list, strides)
    B = cls_maps[0].shape[0]
    if nms_pre > 4096 and any(nms_pre < h * w for h, w in hw_list):
        raise NotImplementedError(f'test_cfg.nms_pre={nms_pre}: the top-k select takes at most 4096 rows per level')
    _chk(img_hw, torch.float32, 'img_hw')
    if img_hw.shape != (B, 2) or (scale_factor is not None and tuple(scale_factor.shape) != (B, 4)):
        raise ValueError(f'img_hw must be ({B}, 2) and scale_factor ({B}, 4)')
    if scale_factor is not None:
        _chk(scale_factor, torch.float32, 'scale_factor')
    for l, (c, r, k) in enumerate(zip(cls_maps, reg_maps, ctr_maps)):
        _chk(c, torch.float32, f'cls_maps[{l}]'); _chk(r, torch.float32, f'reg_maps[{l}]'); _chk(k, torch.float32, f'ctr_maps[{l}]')
        if tuple(c.shape) != (B,) + hw_list[l] + (num_classes,) or tuple(r.shape) != (B,) + hw_list[l] + (4,) \
                or tuple(k.shape) != (B,) + hw_list[l] + (1,):
            raise ValueError(f'level {l}: maps must be channels-last (B, H, W, {num_classes} | 4 | 1)')
    R = sum(fcos_decode_rows(hw_list, nms_pre))
    dev = cls_maps[0].device
    idx = torch.empty((B, R), dtype=torch.int32, device=dev)
    boxes = torch.empty((B, R, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((B, R, num_classes), dtype=torch.float32, device=dev)
    ctr = torch.empty((B, R), dtype=torch.float32, device=dev)
    nbytes = int(_lib.load().ptb_fcos_decode_workspace(B, L, hw))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
    arr = lambda ts: (ctypes.c_void_p * L)(*[t.data_ptr() for t in ts])
    _call('ptb_fcos_decode', arr(cls_maps), arr(reg_maps), arr(ctr_maps), L, hw, st, B, int(num_classes), img_hw, scale_factor,
          int(nms_pre), idx, boxes, scores, ctr, ws, nbytes)
    return idx, boxes, scores, ctr
