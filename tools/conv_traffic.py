"""Per-launch operand traffic and time of the wgmma conv (conv_tc_kernel) at the bench shape (batch 8, 100 x 168 x 256).

For each launch the head makes, prints one JSON line with
  * the TMA bytes (L2 -> shared memory) and shared-memory bytes (TMA writes + wgmma operand reads) computed from the tile plan, for the
    old feed (one activation box per tap and K-block) and the current one (one box of tile h + 2 rows per column offset, read by the
    three vertical taps),
  * the CUDA-event time per launch,
and one line with the GPU name, its power limit and the SM clock, read while the timed launches run.
    python tools/conv_traffic.py [--iters N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {0: (8, 16), 1: (4, 32), 2: (16, 8)}      # tile shape id -> (tile h, tile w); 128 pixels each


def tile_counts(H, W):
    """tiles of one image per tile shape: the host tile plan of conv_tc.cu (8 x 16 main region, 4 x 32 bottom strip, 16 x 8 right strip)."""
    rh, rw = H % 8, W % 16
    bottom = 1 <= rh <= 4
    tiles_h = H // 8 if bottom else (H + 7) // 8
    n_bottom = (W + 31) // 32 if bottom else 0
    right = 1 <= rw <= 8 and tiles_h > 0
    tiles_w = W // 16 if right else (W + 15) // 16
    right_h = min(tiles_h * 8, H)
    n_right = (right_h + 15) // 16 if right else 0
    return {0: tiles_h * tiles_w, 1: n_bottom, 2: n_right}


def traffic(B, H, W, Cin, taps, n_mma, f16=True):
    """(TMA bytes, shared-memory bytes) of one launch, old feed and current feed."""
    kbc = 32 if f16 else 16                                        # channels per 64 B K-block
    nt = 128 if (not f16 or n_mma > 64) else 64 if n_mma > 32 else 32 if n_mma > 16 else 16
    slices = (n_mma + nt - 1) // nt
    kpt = Cin // kbc
    w_box = nt * 64                                                # one weight box (hi or lo)
    # wgmma operand reads per K-block: 2 warpgroups x 2 k-steps x 3 MMAs x (A: 64 rows x 32 B, B: nt rows x 32 B)
    mma_read = 2 * 2 * 3 * (64 * 32 + nt * 32)
    out = dict(tma_old=0, tma_new=0, smem_old=0, smem_new=0)
    for shape, n in tile_counts(H, W).items():
        th, tw = SHAPES[shape]
        items = B * n * slices
        kb = taps * kpt
        old = kb * (2 * 128 * 64 + 2 * w_box)
        n_kh = 3 if taps == 9 else 1
        halo = 2 if taps == 9 else 0
        new = (taps // n_kh) * kpt * (2 * (th + halo) * tw * 64 + n_kh * 2 * w_box)
        out['tma_old'] += items * old
        out['tma_new'] += items * new
        out['smem_old'] += items * (old + kb * mma_read)
        out['smem_new'] += items * (new + kb * mma_read)
    return out


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=60)
    first = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ''
    vals = [v.strip() for v in first.split(',')] if first else []
    return dict(zip(q.split(','), vals)) if len(vals) == 4 else dict(nvidia_smi=r.stdout.strip() or r.stderr.strip())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('conv_traffic.py times kernels on a CUDA device; none is visible')
    from pointtinybenchmark_b200 import ops
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    B, H, W, C = 8, 100, 168, 256
    x = torch.randn(B, H, W, C, generator=g).to(dev)
    w = (torch.randn(C, C, 3, 3, generator=g) * (1.4 / (C * 9) ** 0.5)).to(dev)
    h16, l16, dinv = ops.split_f16(x, auto_scale=True)
    wh16, wl16, invw = ops.conv3x3_pack_weight_f16(w)
    xh, xl = ops.split_tf32(x)
    wh, wl = ops.conv3x3_pack_weight(w)
    pk_dgrad = ops.conv_tc_pack_weight_f16(w.flip(2, 3).transpose(0, 1).reshape(C, C, 9).contiguous(), 9)
    pk_p2p = ops.conv_tc_pack_weight_f16((torch.randn(320, C, 3, 3, generator=g) * 0.02).reshape(320, C, 9).to(dev), 9)
    pk_lin = ops.conv_tc_pack_weight_f16((torch.randn(80, C, generator=g) * 0.05).to(dev), 1)
    bias = torch.zeros(320, device=dev)
    gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    launches = [
        ('tower conv3x3 256->256 fp16x2 (+GN stats)', lambda: ops.conv3x3_c256_f16(h16, l16, wh16, wl16, invw, dinv), 9, 256, True),
        # the launch the towers make: the same conv with GroupNorm + ReLU applied in the kernel, written as the next layer's fp16 pair
        ('tower conv3x3 256->256 fp16x2 + GN apply in the kernel (fp16 pair out)',
         lambda: ops.conv3x3_c256_f16_gn(h16, l16, wh16, wl16, invw, dinv, gamma, beta), 9, 256, True),
        ('tower conv3x3 256->256 3xTF32 (+GN stats)', lambda: ops.conv3x3_c256(xh, xl, wh, wl), 9, 256, False),
        ('tower dgrad conv3x3 256->256 fp16x2', lambda: ops.conv_tc_f16(h16, l16, pk_dgrad, 9, C, dev_out_scale=dinv), 9, 256, True),
        ('P2P cls_out conv3x3 256->320 fp16x2', lambda: ops.conv_tc_f16(h16, l16, pk_p2p, 9, 320, bias=bias, dev_out_scale=dinv), 9, 320, True),
        ('logit map 1-tap 256->80 fp16x2', lambda: ops.conv_tc_f16(h16, l16, pk_lin, 1, 80, bias=bias[:80], dev_out_scale=dinv), 1, 80, True),
    ]
    info = None
    for name, fn, taps, n_out, f16 in launches:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        s.record()
        for _ in range(args.iters):
            fn()
        e.record()
        if info is None:
            info = gpu_info()                                      # queried while the launches above are still running
        e.synchronize()
        ms = s.elapsed_time(e) / args.iters
        tr = traffic(B, H, W, C, taps, (n_out + 15) // 16 * 16, f16)
        print(json.dumps(dict(launch=name, shape=[B, H, W, C], ms_per_launch=round(ms, 4),
                              tma_gb_old=round(tr['tma_old'] / 1e9, 3), tma_gb_new=round(tr['tma_new'] / 1e9, 3),
                              smem_gb_old=round(tr['smem_old'] / 1e9, 3), smem_gb_new=round(tr['smem_new'] / 1e9, 3),
                              tma_tb_per_s=round(tr['tma_new'] / (ms * 1e-3) / 1e12, 2))))
    print(json.dumps(dict(gpu=info, iters=args.iters, timing='CUDA events over back-to-back launches (L2 warm)')))


if __name__ == '__main__':
    main()
