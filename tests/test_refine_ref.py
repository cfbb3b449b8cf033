"""CPU: the refine restatement of tests/refine_ref.py against the oracle's refine_single (oracle/cpr.py), and its dispatch mirror."""
import numpy as np
import pytest
import torch

from oracle import cpr as ocpr
from pointtinybenchmark_b200 import ops
from tests import refine_ref as ref

FLAG_SETS = [(a, b, c) for a in (True, False) for b in (True, False) for c in (True, False)]


def lattice_offsets():
    """integer offsets: on a 16 px lattice of centres, a sample halfway between two centres is exactly equidistant in both formulas"""
    return torch.tensor([[8.0, 0.0], [-8.0, 0.0], [0.0, 8.0], [0.0, -8.0], [8.0, 8.0], [0.0, 0.0]])


def make_case(seed, B, n, C, R, off, scale=3.0, lattice=False, pool=None):
    """a batch for refine_single: probabilities with planted ties, R refine bags per GT"""
    g = torch.Generator().manual_seed(seed)
    K = off.shape[0]
    G = B * n
    bag_img = torch.arange(B, dtype=torch.int32).repeat_interleave(n)
    if lattice:
        c0 = torch.stack([torch.randint(2, 40, (G,), generator=g), torch.randint(2, 30, (G,), generator=g)], 1).float() * 16
    else:
        c0 = torch.rand(G, 2, generator=g) * torch.tensor([400.0, 300.0]) - 10
    cr = c0[:, None].repeat(1, R, 1)                  # the reference model centres every refine bag of a GT on its point
    pts = off[None, None] + cr[:, :, None]                                          # (G,R,K,2)
    pool = pool if pool is not None else sorted({0, C - 1, min(1, C - 1), min(2, C - 1), C // 2})
    labels = torch.tensor(pool)[torch.randint(0, len(pool), (G,), generator=g)].int()
    prob = torch.sigmoid(torch.randn(G, R, K, C, generator=g) * scale)
    if C >= 4:
        prob[..., C - 3] = prob[..., 0]                 # ties: one lower and one higher class of the same probability
        prob[..., 2] = prob[..., 1]                     # inside one float4
    if C >= 2:
        hot = torch.rand(G, R, K, generator=g) < 0.3
        prob[..., 1] = torch.where(hot, torch.ones(()), prob[..., 1])       # saturated 1.0 ties with class C - 1 below / above
        prob[..., C - 1] = torch.where(hot, torch.ones(()), prob[..., C - 1])
    pad_hw = torch.tensor([[300 - 11 * b, 400 - 7 * b] for b in range(B)], dtype=torch.int32)
    img_hw = torch.tensor([[280 - 13 * b, 390 - 17 * b] for b in range(B)], dtype=torch.int32)
    ph, pw = pad_hw[bag_img.long(), 0].float(), pad_hw[bag_img.long(), 1].float()
    valid = ocpr.point_valid(pts, ph[:, None, None], pw[:, None, None])
    nr_in = torch.rand(G, generator=g) < 0.1
    return dict(prob=prob, pts=pts, valid=valid, centres=cr, labels=labels, bag_img=bag_img, img_hw=img_hw, K=K, R=R, nr_in=nr_in)


def oracle(case, cfg, with_nr_in):
    outs = []
    B = int(case['bag_img'].max()) + 1
    for b in range(B):
        sel = case['bag_img'] == b
        n = int(sel.sum())
        pts3 = torch.cat([case['pts'][sel], torch.full(case['pts'][sel].shape[:-1] + (1,), 8.0)], -1)
        img_shape = tuple(case['img_hw'][b].tolist())
        outs.append(ocpr.refine_single(case['prob'][sel], pts3, case['valid'][sel][..., None], case['centres'][sel],
                                       case['labels'][sel].long(), img_shape,
                                       ocpr.default_cfg(merge_th=cfg.merge_th, gt_alpha=cfg.gt_alpha, refine_th=cfg.refine_th,
                                                        nearest_filter=cfg.nearest, classify_filter=cfg.classify,
                                                        return_score_type='max' if cfg.score_max else 'mean'),
                                       case['nr_in'][sel] if with_nr_in else None))
        assert n == outs[-1]['refine_pts'].shape[0]
    return {k: torch.cat([o[k] for o in outs]) for k in outs[0] if isinstance(outs[0][k], torch.Tensor)}


CASES = [dict(seed=1, B=2, n=40, C=80, R=1, r=3), dict(seed=2, B=3, n=30, C=5, R=1, r=1), dict(seed=3, B=2, n=25, C=20, R=2, r=2),
         dict(seed=4, B=1, n=40, C=1, R=1, r=1), dict(seed=5, B=2, n=60, C=33, R=1, r=0), dict(seed=6, B=1, n=35, C=8, R=1, r=2, pool=[3]),
         dict(seed=7, B=2, n=80, C=6, R=1, r=None, lattice=True), dict(seed=8, B=2, n=40, C=80, R=1, r=3, scale=14.0)]


@pytest.mark.parametrize('spec', CASES, ids=lambda d: f"C{d['C']}_R{d['R']}_r{d['r']}_s{d['seed']}")
def test_reference_matches_the_oracle(spec):
    spec = dict(spec)
    r = spec.pop('r')
    off = lattice_offsets() if r is None else ops.circle_offsets(r, 8.0)
    case = make_case(spec.pop('seed'), off=off, **spec)
    G, R, K, C = case['prob'].shape
    prob = case['prob'].reshape(G, R * K, C)
    pts = case['pts'].reshape(G, R * K, 2)
    comp = ref.components(prob, pts, case['valid'].reshape(G, R * K), K, case['labels'], case['bag_img'], case['img_hw'])
    n_sqrt = 0
    for flags in FLAG_SETS:
        for th in (0.1, 0.3):
            cfg = ref.Cfg(0.1, 0.5, th, *flags)
            for with_nr in (False, True):
                o = oracle(case, cfg, with_nr)
                want = ref.combine(comp, cfg, case['nr_in'] if with_nr else None)
                if flags[0]:
                    diff = o['mask_nearest'] != comp.nearest
                    if diff.any():
                        # MKL's sqrt inside torch.cdist is not correctly rounded: it may only decide where two candidates are 1 ulp apart
                        do, da = comp.d_own[diff], comp.d_alt[diff]
                        ulp = torch.from_numpy(np.spacing(np.maximum(do, da).numpy().astype(np.float32)).astype(np.float64))
                        assert bool(((do - da).abs() <= ulp).all()), 'nearest mask differs where the distances are not 1 ulp apart'
                        n_sqrt += int(diff.sum())
                    mv = o['merge_valid'] & ~diff
                    assert torch.equal(mv, want.merge_valid & ~diff)
                    if diff.any():
                        continue
                if flags[1]:
                    assert torch.equal(o['mask_classify'], comp.classify)
                assert torch.equal(o['mask_inside'], comp.inside)
                assert torch.equal(o['merge_valid'], want.merge_valid), (flags, th, with_nr)
                assert torch.equal(o['chosen'], want.chosen)
                bad, worst, und = ref.check(want, o['refine_pts'], o['refine_scores'], o['not_refine'])
                assert not bad, (flags, th, with_nr, bad)
                assert worst <= 1.0
    assert int(comp.classify.sum()) > 0
    print(f'[oracle] samples whose nearest GT the cdist sqrt decides: {n_sqrt}')


def test_planted_ties_resolve_to_the_first_index():
    """on the lattice, samples halfway between two same-label centres keep only the lower GT; a class tied with a lower class is
    never chosen, with a higher class always"""
    case = make_case(7, 2, 80, 6, 1, lattice_offsets(), lattice=True)
    G, R, K, C = case['prob'].shape
    pts = case['pts'].reshape(G, K, 2)
    comp = ref.components(case['prob'].reshape(G, K, C), pts, case['valid'].reshape(G, K), K, case['labels'], case['bag_img'],
                          case['img_hw'])
    ties = (comp.d_own == comp.d_alt)
    assert int(ties.sum()) > 10
    # a tie keeps the sample only when its own GT comes first in the group
    first_own = torch.zeros_like(ties)
    for members in ref.groups(case['bag_img'], case['labels']):
        if len(members) > 1:
            f, _ = ref.nearest_choice(pts, members, 1, K, ref.use_mm(len(members), 1, K))
            first_own[members] = f == torch.arange(len(members))[:, None]
    assert torch.equal(comp.nearest[ties], first_own[ties])
    assert bool(comp.nearest[ties].any()) and bool((~comp.nearest[ties]).any())
    lab = case['labels'].long()[:, None].expand(G, K)
    top = case['prob'].reshape(G, K, C).max(2)[0]
    is_max = comp.pl == top
    assert not bool(comp.classify[(lab == C - 3) & is_max & (case['prob'].reshape(G, K, C)[..., 0] == top)].any())
    assert bool(comp.classify[(lab == 1) & is_max].all()) and bool(comp.classify[(lab == 1) & is_max].any())


def test_distance_restatements_match_torch_cdist_before_the_sqrt():
    """cdist_direct is the plain formula; cdist_mm's pre-sqrt value is torch.cdist's above 25 rows (squared values compared through
    the correctly rounded square of the fp32 result would lose bits, so the check is on the distances themselves within 1 ulp)"""
    g = torch.Generator().manual_seed(3)
    p = (torch.rand(300, 2, generator=g) * 1300).float()
    c = (torch.rand(30, 2, generator=g) * 1300).float()
    mm = ref.cdist_mm(p.double()[:, 0:1], p.double()[:, 1:2], c.double()[None, :, 0], c.double()[None, :, 1]).float()
    want = torch.cdist(p, c)
    assert float(((mm - want).abs() / torch.from_numpy(np.spacing(want.numpy()))).max()) <= 1.0
    d = ref.cdist_direct(p.double()[:10, 0:1], p.double()[:10, 1:2], c.double()[None, :5, 0], c.double()[None, :5, 1]).float()
    dw = torch.cdist(p[:10], c[:5])
    assert float(((d - dw).abs() / torch.from_numpy(np.spacing(dw.numpy()))).max()) <= 1.0


def test_expected_plan_mirrors_the_host_dispatch():
    P = ref.expected_plan
    assert P(80, 80, 289, 64.0, 8, {}) == ('fast<3>', True, None, 18, 320, 1)
    assert P(80, 80, 289, 64.0, 8, {'PTB_REFINE_TMA': '0'}) == ('fast<3>', False, 'env', 0, 320, 1)
    assert P(20, 24, 289, 64.0, 8, {}).phase == 'fast<1>'
    assert P(4, 4, 9, 8.0, 8, {}) == ('fast<1>', True, None, 4, 64, 1)
    assert P(32, 32, 33, 64.0, 8, {}).phase == 'fast<1>'
    assert P(36, 36, 289, 64.0, 8, {}).phase == 'fast<2>' and P(64, 64, 289, 64.0, 8, {}).phase == 'fast<2>'
    assert P(68, 68, 289, 64.0, 8, {}).phase == 'fast<3>' and P(96, 96, 289, 64.0, 8, {}).phase == 'fast<3>'
    assert P(100, 100, 289, 64.0, 8, {}) == ('fast<4>', False, 'window', 18, 320, 1)        # 18 x 18 x 100 x 4 B > 112 KB
    assert P(84, 84, 289, 64.0, 8, {}).use_tma and not P(88, 88, 289, 64.0, 8, {}).use_tma
    assert P(128, 128, 9, 8.0, 8, {}) == ('fast<4>', True, None, 4, 64, 1)
    for c in (1, 3, 5, 33, 127, 132, 256):
        assert P(c, (c + 3) // 4 * 4, 9, 8.0, 8, {}).phase == 'loop', c
    assert P(260, 264, 9, 8.0, 8, {}) == ('loop', False, 'ld', 0, 64, 1)
    assert P(256, 256, 9, 8.0, 8, {}).use_tma
    assert P(80, 80, 1, 0.0, 8, {}) == ('fast<3>', False, 'reach0', 0, 64, 1)
    assert P(80, 80, 320, 64.0, 8, {}).passes == 1 and P(80, 80, 321, 64.0, 8, {}) == ('fast<3>', True, None, 18, 320, 2)
    assert P(80, 80, 441, 80.0, 8, {}) == ('fast<3>', False, 'window', 22, 320, 2)
    assert P(20, 20, 441, 80.0, 8, {}) == ('fast<1>', True, None, 22, 320, 2)
    assert P(20, 20, 2891, 300.0, 8, {}).passes == 10
    with pytest.raises(ValueError):
        P(20, 20, 2892, 300.0, 8, {})
    assert ref.tail_bytes(2891) == 48 * 1024
