"""Host restatement of the bag gather, ptb_cpr_bag_gather and ptb_cpr_bag_gather_bwd (csrc/gather.cu), for its tests.  Plain torch
arithmetic on CPU or GPU tensors; no library needed.

Forward.  Every form of the kernel computes, for sample k of bag g and channel c, in fp32 with round-to-nearest at every step:
    p = offsets[k] + centers[g]
    ix = sample_coord(p.x): u = p / s, t = 2u + 1, g = t / W - 1, ix = fma(g + 1, W / 2, -0.5), clamped to [0, W - 1]  (iy alike)
    taps x0 = floor(ix), x1 = min(x0 + 1, W - 1) (y alike), ex = (x0 + 1) - ix, wx = ix - x0,
    weights w00 = ex * ey, w01 = wx * ey, w10 = ex * wy, w11 = wx * wy
    out = fma(q11, w11, fma(q10, w10, fma(q01, w01, q00 * w00)))
(ptb_common.cuh sample_coord / make_taps_at / bilerp1).  That is ATen's CPU grid_sample with bilinear interpolation, border padding
and align_corners=False.  gather_f32 reproduces it bit for bit in float64 arithmetic: a +, -, * or / of two fp32 values rounded to
float64 and then to fp32 is the correctly rounded fp32 result, a product of two fp32 values is exact in float64, and the sum of each
fma is rounded to odd in float64 so that its one rounding to fp32 is that of a true fma.  gather_f64 blends the same fp32 taps with
the same fp32 weights in float64.

Backward.  scatter_f64 adds grad_out * w from the same fp32 weights into the map gradient in float64.  The kernel adds fp32 products
with fp32 atomics in an arbitrary order, so it also returns, per map element, the sum of |w * g| and the number of terms, which bound
the error of any fp32 order.

Dispatch.  window_staged says which bags the TMA-staged kernel stages in shared memory (the others read global memory), and
expected_path which kernel the host launches.
"""
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from tests.cpr_loss_ref import point_valid, sample_coord, sample_points  # noqa: F401  (fp32 sample coordinates, validity)

TAP_BYTES = 32                 # sizeof(GtTap): four int offsets and four fp32 weights per sample
TMA_SMEM_LIMIT = 112 * 1024    # the host's cap on the staged kernel's dynamic shared memory


def _f32(x):
    return x.float().double()


def taps(pts, stride, H, W):
    """fp32 image points (..., 2) -> cell index y * W + x (..., 4) int64 and fp32 weight (..., 4) of the taps nw, ne, sw, se."""
    ix = sample_coord(pts[..., 0], stride, W)
    iy = sample_coord(pts[..., 1], stride, H)
    x0, y0 = ix.floor(), iy.floor()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)          # a clamped east / south tap has weight 0
    ex, wx = _f32((x0 + 1) - ix), _f32(ix - x0)
    ey, wy = _f32((y0 + 1) - iy), _f32(iy - y0)
    idx = torch.stack([y0 * W + x0, y0 * W + x1, y1 * W + x0, y1 * W + x1], dim=-1).long()
    w = torch.stack([ex * ey, wx * ey, ex * wy, wx * wy], dim=-1).float()
    return idx, w


def bag_taps(centers, bag_img, offsets, stride, H, W):
    """rows (into the B*H*W cells of the map) and fp32 weights of the four taps of every sample: (G,K,4) int64, (G,K,4) fp32, CPU."""
    idx, w = taps(sample_points(centers.cpu(), offsets.cpu()), stride, H, W)
    return idx + bag_img.cpu().long()[:, None, None] * (H * W), w


def fma_f32(a, b, c):
    """fp32 fma(a, b, c) with one rounding, for fp32 tensors (broadcasting)."""
    p = a.double() * b.double()                        # exact: two 24-bit significands
    c = c.double()
    s = p + c
    bp = s - p
    e = (p - (s - bp)) + (c - bp)                      # s + e == p + c exactly (two-sum)
    # round to odd: where s is inexact and its last bit even, take the float64 neighbour on the side of p + c.  The rounding to fp32
    # then sees a float64 tie only where p + c is one, and 53 >= 24 + 2 bits makes it the correctly rounded fp32 result.
    even = (s.view(torch.int64) & 1) == 0
    away = torch.nextafter(s, torch.where(e > 0, torch.full_like(s, math.inf), torch.full_like(s, -math.inf)))
    return torch.where((e != 0) & even & torch.isfinite(s), away, s).float()


def _chunks(n_rows, C):
    step = max(1, (1 << 22) // max(C, 1))
    return [slice(i, min(i + step, n_rows)) for i in range(0, n_rows, step)]


def gather_f32(map_nhwc, centers, bag_img, offsets, stride, C=None):
    """(G,K,C) fp32 bag samples of the kernel, bit for bit, on map_nhwc's device.  map_nhwc (B,H,W,ld) fp32; columns >= C unread."""
    B, H, W, ld = map_nhwc.shape
    C = ld if C is None else C
    G, K = centers.shape[0], offsets.shape[0]
    dev = map_nhwc.device
    idx, w = bag_taps(centers, bag_img, offsets, stride, H, W)
    idx, w = idx.reshape(-1, 4).to(dev), w.reshape(-1, 4).to(dev)
    rows = map_nhwc.reshape(B * H * W, ld)[:, :C]
    out = torch.empty((G * K, C), dtype=torch.float32, device=dev)
    for j in _chunks(G * K, C):
        q = [rows[idx[j, t]] for t in range(4)]
        wt = [w[j, t, None] for t in range(4)]
        r = (q[0].double() * wt[0].double()).float()
        for t in (1, 2, 3):
            r = fma_f32(q[t], wt[t], r)
        out[j] = r
    return out.reshape(G, K, C)


def gather_f64(map_nhwc, centers, bag_img, offsets, stride, C=None):
    """(G,K,C) float64: the kernel's fp32 taps and weights, blended without rounding."""
    B, H, W, ld = map_nhwc.shape
    C = ld if C is None else C
    dev = map_nhwc.device
    idx, w = bag_taps(centers, bag_img, offsets, stride, H, W)
    rows = map_nhwc.reshape(B * H * W, ld)[:, :C].double()
    idx, w = idx.to(dev), w.to(dev).double()
    return sum(rows[idx[..., t]] * w[..., t, None] for t in range(4))


def scatter_f64(grad_out, map_shape, centers, bag_img, offsets, stride):
    """float64 map gradient (B,H,W,ld) of grad_out (G,K,C) through the kernel's fp32 weights, on the CPU.  Also returns per element
    the sum of |w * g| over its terms (B,H,W,ld) and the number of terms per cell (B,H,W,1); padding columns >= C are 0 in all three.
    A tap of weight 0 is not a term: the kernel skips it."""
    B, H, W, ld = map_shape
    G, K, C = grad_out.shape
    idx, w = bag_taps(centers, bag_img, offsets, stride, H, W)
    go = grad_out.detach().cpu().double().reshape(G * K, C)
    grad = torch.zeros((B * H * W, ld), dtype=torch.float64)
    absum = torch.zeros((B * H * W, ld), dtype=torch.float64)
    count = torch.zeros((B * H * W, 1), dtype=torch.int64)
    for t in range(4):
        wt = w[..., t].reshape(-1).double()
        it = idx[..., t].reshape(-1)
        nz = wt != 0
        term = go[nz] * wt[nz, None]
        grad[:, :C].index_add_(0, it[nz], term)
        absum[:, :C].index_add_(0, it[nz], term.abs())
        count.index_add_(0, it[nz], torch.ones((int(nz.sum()), 1), dtype=torch.int64))
    return grad.reshape(B, H, W, ld), absum.reshape(B, H, W, ld), count.reshape(B, H, W, 1)


def window_size(reach_px, stride):
    """WS, the side in cells of the staged window: 2 ceil(reach / stride) + 2, the division in fp32."""
    return 2 * math.ceil(float(np.float32(reach_px) / np.float32(stride))) + 2


def window_staged(centers, reach_px, stride, H, W):
    """(G,) bool: the TMA-staged kernel stages the bag's window (gather.cu bag_gather_tma_kernel).  The window spans the taps of
    the fp32 sample coordinates of centre -/+ reach; a bag whose span is wider than WS reads its taps from global memory."""
    ws = window_size(reach_px, stride)
    c = centers.cpu().float()
    r = float(np.float32(reach_px))

    def span(p, size):
        lo = sample_coord(p - r, stride, size).floor()
        hi = (sample_coord(p + r, stride, size).floor() + 1).clamp(max=size - 1)
        return hi - lo + 1

    return (span(c[:, 0], W) <= ws) & (span(c[:, 1], H) <= ws)


class Path(NamedTuple):
    kernel: Optional[str]      # 'tma<64>', 'tma<32>', 'ldg<64>', 'ldg<40>', 'ldg<20>', 'ldg<0>'; None when nothing is launched (G = 0)
    fallback: Optional[str]    # why a TMA request ends on an LDG kernel: 'window' (too large), 'reach0' (no reach or no features)


def expected_path(C, ld, K, reach_px, stride, env, G=1, feats=True):
    """the kernel ptb_cpr_bag_gather launches for these arguments (gather.cu host dispatch); env holds PTB_GATHER_TMA / PTB_GATHER_CC.
    Assumes the tensor map encodes, as it does for every layout the host accepts (ld % 4 == 0)."""
    if G == 0:
        return Path(None, None)
    e_tma, e_cc = env.get('PTB_GATHER_TMA'), env.get('PTB_GATHER_CC')
    cc = 64 if C % 64 == 0 else (32 if C % 32 == 0 else 0)
    if e_cc is not None and e_cc[:1] == '3' and C % 32 == 0:
        cc = 32
    if e_cc is None and C % 32 == 0 and C < 256:
        cc = 32
    want_tma = (e_tma[:1] != '0') if e_tma is not None else C <= 192
    reach = float(np.float32(reach_px)) if feats else 0.0        # ops.bag_gather passes no reach without features
    fallback = None
    if want_tma and cc and G * (C // cc) < (1 << 31):
        if reach > 0:
            ws = window_size(reach, stride)
            smem = ws * ws * cc * 4 + 128 + K * TAP_BYTES
            if ws <= 256 and smem <= TMA_SMEM_LIMIT:
                return Path(f'tma<{cc}>', None)
            fallback = 'window'
        else:
            fallback = 'reach0'
    cg = C // 4
    return Path(f'ldg<{cg if cg in (64, 40, 20) else 0}>', fallback)
