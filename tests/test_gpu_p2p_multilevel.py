"""GPU: P2PHead over several FPN levels against the REAL reference's vectors (tests/golden/p2p_multilevel_*.npz): assignments, top-k
indices and NMS keep bit-exact, losses and parameter gradients within 1e-4, detections within 1e-4; aug_test_bboxes at two scales;
the refusal of maps whose proposal count does not split into equal chunks, and of more NMS points than the NMS takes.  The multi-level
decode kernels (sigmoid and softmax) against a host restatement with chunk boundaries inside a level and on a level boundary and an
exact key tie inside one chunk; the 8192-point NMS entry points against tests/nms_ref.py
at P = 4096, 4097, 5000 and 8192; and a bit-identical repeat of the training step in deterministic mode."""
import os

import numpy as np
import pytest
import torch

from oracle import p2p_multilevel as oml
from oracle.make_golden_p2p_multilevel import GRAD_STEP
from tests import nms_ref as ref
from tests.test_gpu_p2p_defaults import TEST_CFG, TRAIN_CFG
from tests.test_p2p_multilevel_golden import head_kwargs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return ops


def _close(a, ref_, tol, what):
    a, ref_ = np.asarray(a, np.float64), np.asarray(ref_, np.float64)
    assert a.shape == ref_.shape, (what, a.shape, ref_.shape)
    d = np.abs(a - ref_).max() if a.size else 0.0
    assert d <= tol * max(1.0, np.abs(ref_).max()), f'{what}: max |diff| {d:.3e}'


def build(cfg, weights):
    from pointtinybenchmark_b200.p2p_head import P2PHead
    head = P2PHead(**head_kwargs(cfg), train_cfg=TRAIN_CFG, test_cfg=dict(TEST_CFG, nms_pre=cfg['nms_pre']))
    head.load_state_dict(weights, strict=True)
    return head.cuda()


def train_step(head, inp):
    dev = torch.device('cuda:0')
    head.train()
    head.zero_grad(set_to_none=True)
    xs = [x.to(dev) for x in inp['xs']]
    losses = head.forward_train(xs, inp['img_metas'], [b.to(dev) for b in inp['gt_bboxes']], [l.to(dev) for l in inp['gt_labels']])
    (sum(losses['loss_cls']) + sum(losses['loss_pts'])).backward()
    return losses


@pytest.mark.parametrize('name', sorted(oml.CASES))
def test_training_matches_reference(ops, golden_dir, name):
    gold = np.load(os.path.join(golden_dir, f'p2p_multilevel_{name}.npz'))
    inp, cfg = oml.case_inputs(name)
    head = build(cfg, inp['weights'])
    losses = train_step(head, inp)
    assert np.array_equal(head._last_assign['gt_inds'].cpu().numpy().astype(np.int32), gold['gt_inds'])
    assert np.array_equal(torch.stack(head._last_targets['labels']).cpu().numpy(), gold['labels'])
    for k in ('loss_cls', 'loss_pts'):
        _close(torch.stack([v.detach() for v in losses[k]]).cpu().numpy(), gold[k], 1e-4, f'{name} {k}')
    for k, p in head.named_parameters():
        step = GRAD_STEP if p.dim() == 4 else 1
        g, ref_ = p.grad.flatten()[::step].double().cpu().numpy(), gold[f'grad/{k}'].astype(np.float64)
        if k.startswith(('cls_out', 'reg_out')):
            _close(g, ref_, 1e-4, f'{name} d/d{k}')
        else:
            # The tower gradients are compared by norm: this problem is that sensitive to rounding.  On the host, multiplying the
            # oracle's (= the reference's) input maps by 1 + 1e-5 * N(0, 1) keeps every assignment and moves the reg tower's weight
            # gradients by up to 1.9e-2 (norm-relative; a_focal_sl1, whose reg gradients are ~1e-3 of the cls tower's; b 6.1e-3,
            # c 1.8e-3) and the cls tower's by up to 1.6e-3 (c_softmax_cw): pre-activations within rounding of zero pass the
            # eight GroupNorm + ReLU layers gated differently.  Measured on the GPU (fp16-pair tensor-core towers against the fp32 CPU
            # reference): reg towers up to 2.0e-2, cls towers up to 2.4e-3.
            rel = float(np.linalg.norm(g - ref_) / np.linalg.norm(ref_))
            print(f'[{name}] d/d{k}: norm-relative error {rel:.2e}')
            tol = 3e-2 if k.startswith('reg_convs') else 5e-3
            assert rel <= tol, f'{name} d/d{k}: norm-relative error {rel:.3e}'


@pytest.mark.parametrize('name', sorted(oml.CASES))
def test_inference_matches_reference(ops, golden_dir, name):
    """get_bboxes on the reference's own logit maps (the oracle's forward, which oracle/make_golden_p2p_multilevel.py asserts
    bit-equal to the reference's): per-chunk top-k and NMS keep bit-exact, labels exact, detections within 1e-4 of the vectors."""
    gold = np.load(os.path.join(golden_dir, f'p2p_multilevel_{name}.npz'))
    inp, cfg = oml.case_inputs(name)
    head = build(cfg, inp['weights']).eval()
    oc, op_ = oml.head_forward(inp['xs'], inp['weights'], cfg)
    maps = ([c.cuda() for c in oc], [p.cuda() for p in op_])
    if 'ref_error' in gold.files:
        with pytest.raises(RuntimeError, match='equal chunks'):
            head.get_bboxes(*maps, inp['img_metas'])
        return
    res, aux = head.get_bboxes(*maps, inp['img_metas'], return_all=True)
    B, L = len(res), len(cfg['strides'])
    assert np.array_equal(aux['topk_idx'].reshape(B, L, -1).cpu().numpy(), gold['topk'])
    assert np.array_equal(aux['count'].cpu().numpy(), gold['det_len'])
    keep = torch.cat([aux['keep'][b, :int(aux['count'][b])] for b in range(B)]).cpu().numpy()
    assert np.array_equal(keep, gold['keep'])
    assert np.array_equal(torch.cat([r[1] for r in res]).cpu().numpy(), gold['det_labels'])
    _close(torch.cat([r[0] for r in res]).cpu().numpy(), gold['det'], 1e-4, f'{name} det')


@pytest.mark.parametrize('name', sorted(n for n in oml.CASES if n != 'd_uneven'))
def test_inference_on_own_maps(ops, name):
    """simple_test from the feature maps: the head's own logits differ from the reference's by ~1e-6, so its top-k is checked by
    the tie-group rule on its own keys (selection exact outside the boundary group, order exact outside any group; 1e-4 relative
    groups for softmax, whose decode is within a few ulps of ATen's, exact ties for sigmoid), and in sigmoid mode, where the decode
    is bit-identical to ATen's, keep / labels / detections against the oracle run on those same maps when the top-k agree."""
    from tests.test_gpu_p2p_softmax import check_topk_tie_groups
    inp, cfg = oml.case_inputs(name)
    head = build(cfg, inp['weights']).eval()
    xs = [x.cuda() for x in inp['xs']]
    with torch.no_grad():
        outs = head(xs)
        st = head.simple_test(xs, inp['img_metas'])
    res, aux = head.get_bboxes(*outs, inp['img_metas'], return_all=True)
    assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(st, res))
    B, L = len(res), len(cfg['strides'])
    sig = cfg.get('use_sigmoid', True)
    topk = aux['topk_idx'].reshape(B, L, -1).cpu().numpy()
    n_out = outs[0][0].shape[1] // len(cfg['point_anchor'])
    for b in range(B):
        rows = torch.cat([c[b:b + 1].cpu().permute(0, 2, 3, 1).reshape(-1, n_out) for c in outs[0]]).reshape(L, -1, n_out)
        for ch in range(L):
            keys = rows[ch].sigmoid().max(1)[0] if sig else rows[ch].double().softmax(-1)[:, :-1].max(1)[0]
            check_topk_tie_groups(topk[b, ch], keys.double().numpy(), topk.shape[-1], f'{name} head top-k [{b}, {ch}]',
                                  rel=0.0 if sig else 1e-4)
    if sig:
        ores, oaux = oml.p2p_get_bboxes([c.cpu() for c in outs[0]], [p.cpu() for p in outs[1]], inp['img_metas'], cfg, return_all=True)
        if np.array_equal(topk, torch.stack([torch.stack(a['topk_inds']) for a in oaux]).numpy()):
            keep = torch.cat([aux['keep'][b, :int(aux['count'][b])] for b in range(B)]).cpu().numpy()
            assert np.array_equal(keep, torch.cat([a['keep'] for a in oaux]).numpy())
            assert np.array_equal(torch.cat([r[1] for r in res]).cpu().numpy(), torch.cat([r[1] for r in ores]).numpy())
            _close(torch.cat([r[0] for r in res]).cpu().numpy(), torch.cat([r[0] for r in ores]).numpy(), 1e-4, f'{name} det vs oracle')


def test_nms_point_limit_is_named_by_the_head(ops):
    """nms_pre <= 0 keeps every row of every chunk: beyond 8192 NMS points the head names nms_pre, the level count and the limit."""
    inp, cfg = oml.case_inputs('b_defaults')
    head = build(cfg, inp['weights']).eval()
    head.test_cfg['nms_pre'] = -1
    maps = ([torch.zeros(1, 320, 64, 64, device='cuda'), torch.zeros(1, 320, 32, 32, device='cuda')],
            [torch.zeros(1, 8, 64, 64, device='cuda'), torch.zeros(1, 8, 32, 32, device='cuda')])
    with pytest.raises(RuntimeError, match=r'nms_pre=-1 .* 2 chunks, 20480 NMS points .* at most 8192: set test_cfg.nms_pre to at most 4096'):
        head.get_bboxes(*maps, inp['img_metas'][:1])


def test_aug_test_matches_reference(ops, golden_dir):
    gold = np.load(os.path.join(golden_dir, 'p2p_multilevel_aug.npz'))
    feats, metas, w, cfg = oml.aug_inputs()
    head = build(cfg, w).eval()
    res = head.aug_test_bboxes([[x.cuda() for x in f] for f in feats], metas)
    assert np.array_equal(res[0][1].cpu().numpy(), gold['det_labels'])
    _close(res[0][0].cpu().numpy(), gold['det'], 1e-4, 'aug det')


def level_rows(maps, k):
    """(level, i, j, anchor) of every row of an image, level-major as the decode orders them."""
    return [(l, c // w, c % w, a) for l, (h, w) in enumerate(maps) for c in range(h * w) for a in range(k)]


def host_decode(cls_maps, reg_maps, strides, C, k, anchors, gamma, img_hw, nms_pre, softmax):
    """host restatement of ptb_p2p_decode_topk_levels(_softmax): level-major rows, L equal chunks, per chunk the rows ordered by
    (key desc, row asc) - a stable sort - and the first nms_pre kept (every row in row order when nms_pre <= 0 or >= the chunk), then
    the decode with the row's stride and the clamp.  Sigmoid keys and scores are ATen's fp32, softmax ones float64; the kernel's are
    within a few ulps of both.
    Returns per image and chunk the selected chunk-local rows, the float64 keys of the chunk, points and scores."""
    B = cls_maps[0].shape[0]
    C1 = C + 1 if softmax else C
    rows_c, rows_p = [], []
    for c, r, s in zip(cls_maps, reg_maps, strides):
        _, H, W, _ = c.shape
        rows_c.append(c.reshape(B, H * W * k, C1))
        reg = r.reshape(B, H * W, k, 2)
        jj = torch.arange(W, dtype=torch.float32).repeat(H)
        ii = torch.arange(H, dtype=torch.float32).repeat_interleave(W)
        ax = (jj * s)[:, None] + anchors[None, :, 0] * s
        ay = (ii * s)[:, None] + anchors[None, :, 1] * s
        px = ax[None] + reg[..., 0] * gamma * s
        py = ay[None] + reg[..., 1] * gamma * s
        rows_p.append(torch.stack([px, py], -1).reshape(B, -1, 2))
    cls, pts = torch.cat(rows_c, 1), torch.cat(rows_p, 1)
    L = len(cls_maps)
    chunk = cls.shape[1] // L
    out = []
    for b in range(B):
        per = []
        for ch in range(L):
            x = cls[b, ch * chunk:(ch + 1) * chunk]
            sc = x.double().softmax(-1)[:, :-1] if softmax else x.sigmoid()
            keys = sc.max(1)[0].double()
            ti = torch.sort(keys, descending=True, stable=True)[1]
            ti = ti[:nms_pre] if 0 < nms_pre < chunk else torch.arange(chunk)
            p = pts[b, ch * chunk:(ch + 1) * chunk][ti]
            p = torch.stack([p[:, 0].clamp(0, img_hw[b][1]), p[:, 1].clamp(0, img_hw[b][0])], -1)
            per.append((ti, keys.numpy(), p, sc[ti]))
        out.append(per)
    return out


@pytest.mark.parametrize('maps,nms_pre', [
    ([(6, 6), (3, 3), (3, 3)], 7),       # T = 54k, chunks of 18k: boundaries inside level 0 / on its end; the last chunk straddles
    ([(4, 4), (2, 2)], 3),               # T = 20k, the chunk boundary 10k inside level 0, the last chunk straddles the level boundary
    ([(4, 4), (4, 4)], 5),               # T = 32k, the chunk boundary is the level boundary
    ([(4, 4), (4, 4)], 16),              # nms_pre == chunk length (k = 1): every row kept
    ([(6, 6), (3, 3), (3, 3)], 1000),    # nms_pre > chunk length
    ([(6, 6), (3, 3), (3, 3)], -1),
])
@pytest.mark.parametrize('k', [1, 4])
@pytest.mark.parametrize('softmax', [False, True])
def test_decode_levels_against_host_restatement(ops, maps, nms_pre, k, softmax):
    from tests.test_gpu_p2p_softmax import check_topk_tie_groups
    gen = torch.Generator().manual_seed(17 + len(maps) + k + 10 * softmax)
    B, C, strides = 2, 7, [8, 16, 32][:len(maps)]
    C1 = C + 1 if softmax else C
    cls_maps = [torch.randn(B, h, w, k * C1, generator=gen) * 3 for h, w in maps]
    # an exact key tie inside one chunk: the first and the last row of the last chunk (two levels where that chunk straddles a level
    # boundary) get the same, highest logits; the kernel keeps the lower row first
    rows = level_rows(maps, k)
    T, L = len(rows), len(maps)
    r1, r2 = T - T // L, T - 1
    tied = torch.full((C1,), -4.0)
    tied[2] = 9.0
    for r in (r1, r2):
        l, i, j, a = rows[r]
        cls_maps[l][0, i, j, a * C1:(a + 1) * C1] = tied
    reg_maps = [torch.randn(B, h, w, 2 * k, generator=gen) for h, w in maps]
    anchors = torch.tensor([(-0.25, -0.25), (0.25, -0.25), (0.25, 0.25), (-0.25, 0.25)][:k] if k == 4 else [(0., 0.)])
    img_hw = [(maps[0][0] * 8 - 3, maps[0][1] * 8 - 5), (maps[0][0] * 8, maps[0][1] * 8)]
    dev = torch.device('cuda:0')
    idx, pts, sc = ops.p2p_decode_topk_levels([c.to(dev) for c in cls_maps], [r.to(dev) for r in reg_maps], strides, C, k,
                                              anchors.to(dev), 2.0, torch.tensor(img_hw, dtype=torch.int32, device=dev), nms_pre,
                                              softmax=softmax)
    host = host_decode(cls_maps, reg_maps, strides, C, k, anchors, 2.0, img_hw, nms_pre, softmax)
    host_all = host_decode(cls_maps, reg_maps, strides, C, k, anchors, 2.0, img_hw, -1, softmax)
    P = idx.shape[1] // L
    idx, pts, sc = idx.cpu().long().reshape(B, L, P), pts.cpu().reshape(B, L, P, 2), sc.cpu().reshape(B, L, P, C)
    for b in range(B):
        for ch in range(L):
            ti, keys = host[b][ch][:2]
            if not 0 < nms_pre < T // L:      # every row of the chunk, in row order
                assert torch.equal(idx[b, ch], torch.arange(T // L)), (b, ch)
            elif softmax:   # float64 keys: the selection and order by the tie-group rule at 1e-6
                check_topk_tie_groups(idx[b, ch].numpy(), keys, P, f'softmax top-k [{b}, {ch}]', rel=1e-6)
            else:
                assert torch.equal(idx[b, ch], ti), (b, ch)
            got = idx[b, ch]      # points and scores on the kernel's own selection
            x = torch.cat([c.reshape(B, -1, C1) for c in cls_maps], 1)[b, ch * (T // L):(ch + 1) * (T // L)][got]
            want = x.double().softmax(-1)[:, :-1] if softmax else x.sigmoid()
            _close(sc[b, ch].numpy(), want.numpy(), 1e-6, 'scores')
            if b == 0 and ch == L - 1:
                local = idx[b, ch].tolist()
                assert local.index(r1 - ch * (T // L)) < local.index(r2 - ch * (T // L)), 'tied rows: lower row first'
            hp_all = host_all[b][ch][2]
            _close(pts[b, ch].numpy(), hp_all[got].numpy(), 1e-6, 'points')


@pytest.mark.parametrize('P', [4096, 4097, 5000, 8192])
@pytest.mark.parametrize('soft', [False, True])
def test_wide_nms_against_host_restatement(ops, P, soft):
    gen = torch.Generator().manual_seed(P + soft)
    C = 4
    pts = torch.rand(1, P, 2, generator=gen) * torch.tensor([1333., 800.])
    sc = (torch.rand(1, P, C, generator=gen) ** 3)
    dev = torch.device('cuda:0')
    wh, thr, iou, mk = (32, 32), 0.05, 0.5, 100
    if soft:
        cnt, det, lab, keep, cc = ops.multiclass_soft_nms(pts.to(dev), sc.to(dev), wh, thr, iou, mk, method='linear', wide=True)
        r = ref.image(pts[0].numpy(), sc[0].numpy(), thr, iou, mk, wh, dict(sigma=0.5, min_score=1e-3, method='linear'))
    else:
        cnt, det, lab, keep, cc = ops.multiclass_nms(pts.to(dev), sc.to(dev), wh, thr, iou, mk, wide=True)
        r = ref.image(pts[0].numpy(), sc[0].numpy(), thr, iou, mk, wh)
    n = int(cnt[0])
    assert int(cc[0]) == r['cand_count'] and n == r['count']
    assert np.array_equal(keep[0, :n].cpu().numpy(), r['keep'])
    assert np.array_equal(lab[0, :n].cpu().numpy(), r['labels'])
    assert np.array_equal(det[0, :n].cpu().numpy(), r['det'])
    if P > 4096:            # the existing entry points keep their limit
        with pytest.raises(RuntimeError, match='4096'):
            ops.multiclass_nms(pts.to(dev), sc.to(dev), wh, thr, iou, mk)
    if P == 8192:
        p2 = torch.cat([pts, pts[:, :1]], 1).to(dev)
        with pytest.raises(RuntimeError, match='8192'):
            ops.multiclass_nms(p2, torch.cat([sc, sc[:, :1]], 1).to(dev), wh, thr, iou, mk, wide=True)


def test_deterministic_training_repeats_bit_for_bit(ops):
    inp, cfg = oml.case_inputs('b_defaults')
    head = build(cfg, inp['weights'])
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            losses = train_step(head, inp)
            runs.append(([v.detach().clone() for v in losses['loss_cls'] + losses['loss_pts']],
                         [p.grad.clone() for p in head.parameters()]))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
