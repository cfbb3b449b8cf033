"""GPU: the point refinement, ptb_cpr_refine_fused and ptb_cpr_refine (csrc/refine.cu), against the host restatement of
tests/refine_ref.py on every path the fused kernel dispatches on:

  class phase  rf_class_phase<NT> for ncls % 4 == 0 and NT = ceil(ceil(ncls / 4) / 8) <= 4 (fast<1> 4..32 classes, fast<2> 36..64,
               fast<3> 68..96, fast<4> 100..128); rf_class_phase_loop for every other class count
  staging      the bag's window of logits staged by one TMA box, or global memory: PTB_REFINE_TMA=0, ld > 256, no reach (K = 1),
               a window beyond 112 KB, or a bag whose taps straddle its window
  passes       ceil(K / 32) warps clamped to [2, 10]: K > 320 takes several passes per warp
  groups       the nearest filter on cdist_direct or cdist_mm (torch.cdist's rule), members beyond 256 read from global memory

Every case runs the default environment and PTB_REFINE_TMA=0: the chosen masks and not_refine equal the reference's decisions bit for
bit (not_refine wherever the score is further than its error bound from refine_th), points and scores lie within the bound of their
float64 sums, the two environments give torch.equal outputs, two runs give the same outputs, and every call is one launch."""
import collections
import math
from typing import NamedTuple

import pytest
import torch

from pointtinybenchmark_b200.ops import circle_offsets
from tests import refine_ref as ref
from tests.gather_ref import window_staged

pytestmark = pytest.mark.gpu

ENVS = {'default': {}, 'tma0': {'PTB_REFINE_TMA': '0'}}
FLAG_SETS = [(a, b, c) for a in (True, False) for b in (True, False) for c in (True, False)]
THRESHOLDS = [(0.1, 0.5, 0.1), (0.05, 0.8, 0.3), (0.3, 0.25, 0.5)]

_runs = collections.Counter()
_worst = {'fused': 0.0, 'stage': 0.0}
_undecided = collections.Counter()


class Spec(NamedTuple):
    name: str
    ncls: int
    ld: int
    off: str                # 'r<n>' ring radius n, 'k<n>' the first n - 1 ring offsets + centre, 'rand<n>' n random off-grid offsets
                            # with the centre last, 'lattice', 'split' (small random offsets of the formula-split cases)
    G: int
    B: int = 2
    H: int = 20
    W: int = 28
    s: float = 8.0
    centres: str = 'mixed'  # 'mixed', 'near' (a few ulps from cell positions), 'lattice', 'split<t>' (formula-split cluster)
    labels: str = 'pool'    # 'pool' (the labels of every trip and remainder), 'one' (a single label), 'random'
    scale: float = 3.0
    plant: bool = True
    all_flags: bool = False
    seed: int = 0


def _specs():
    out = []
    for ncls, ld in ((4, 4), (20, 24), (32, 32), (36, 36), (64, 64), (68, 68), (80, 80), (96, 96), (100, 100), (128, 128),
                     (1, 4), (3, 4), (5, 8), (33, 36), (127, 128), (132, 132), (256, 256), (260, 264)):
        out.append(Spec(f'ncls{ncls}_ld{ld}_r3', ncls, ld, 'r3', 80, all_flags=ncls in (20, 80, 127, 260), seed=ncls))
    for ncls, ld in ((20, 24), (100, 100), (127, 128), (80, 80)):
        out.append(Spec(f'ncls{ncls}_ld{ld}_r8', ncls, ld, 'r8', 60, seed=ncls + 1))
    # the seven cases of the former fused-versus-staged comparison (3 images of 20 x 28, n GTs per image)
    for ncls, ld, r, n, scale in ((5, 8, 1, 40, 3.0), (80, 80, 8, 60, 3.0), (33, 36, 3, 50, 3.0), (1, 4, 2, 9, 3.0),
                                  (131, 132, 5, 30, 3.0), (80, 80, 4, 60, 14.0), (6, 8, 2, 40, 40.0)):
        out.append(Spec(f'staged_pair_ncls{ncls}_r{r}_x{int(scale)}', ncls, ld, f'r{r}', 3 * n, B=3, scale=scale, plant=False,
                        labels='random', seed=1000 * ncls + r))
    # bag sizes and passes
    for K in (1, 9, 32, 33, 289, 320, 321, 441):
        out.append(Spec(f'K{K}_ncls80', 80, 80, f'k{K}', 40, H=40, W=56, seed=K))
        out.append(Spec(f'K{K}_ncls20', 20, 20, f'k{K}', 40, H=40, W=56, seed=K + 1))
    out += [Spec('rand441_ncls36', 36, 36, 'rand441', 30, H=40, W=56, seed=5),
            Spec('rand2891_ncls20', 20, 24, 'rand2891', 12, H=40, W=56, seed=6),          # the tail's 48 KB limit exactly
            Spec('rand2891_ncls131', 131, 132, 'rand2891', 8, H=40, W=56, seed=7)]
    # staging edges
    out += [Spec('straddle_ncls80_r8', 80, 80, 'r8', 200, H=40, W=56, centres='near', seed=8),
            Spec('straddle_ncls20_r3', 20, 24, 'r3', 200, H=40, W=56, centres='near', seed=9),
            Spec('straddle_ncls127_r3', 127, 128, 'r3', 200, H=40, W=56, centres='near', seed=10)]
    for H, W in ((1, 1), (1, 5), (5, 1), (2, 5), (5, 5)):
        out.append(Spec(f'map{H}x{W}_ncls20', 20, 24, 'r8', 30, H=H, W=W, seed=H * 10 + W))
        out.append(Spec(f'map{H}x{W}_ncls33', 33, 36, 'r3', 30, H=H, W=W, seed=H * 10 + W + 1))
    # groups
    out += [Spec('unique_labels', 128, 128, 'r3', 64, B=1, labels='unique', seed=11),
            Spec('lattice_ties', 8, 8, 'lattice', 120, H=40, W=56, centres='lattice', all_flags=True, seed=12),
            Spec('lattice_ties_mm', 8, 8, 'lattice', 300, H=40, W=56, centres='lattice', labels='one', seed=13),
            Spec('group30', 80, 80, 'r2', 60, B=2, labels='one', all_flags=True, seed=14),
            Spec('group300_K9', 20, 20, 'r1', 300, B=1, H=40, W=56, labels='one', all_flags=True, seed=15),
            Spec('group300_K33', 36, 36, 'k33', 300, B=1, H=40, W=56, labels='one', all_flags=True, seed=16),
            Spec('direct_t2_K9', 20, 20, 'r1', 40, B=2, labels='pool', seed=17)]
    for t, K in ((5, 5), (13, 2), (2, 13), (25, 1), (26, 1)):
        out.append(Spec(f'split_t{t}_K{K}', 80, 80, f'split{K}', t, B=1, H=100, W=168, centres=f'split{t}', labels='one',
                        all_flags=True, seed=t * 100 + K))
    out.append(Spec('headline', 80, 80, 'r8', 4000, B=8, H=100, W=168, labels='random', plant=False, seed=20))
    return out


SPECS = _specs()


def offsets(spec):
    s = spec.s
    if spec.off == 'lattice':
        return torch.tensor([[16.0, 0.0], [-16.0, 0.0], [0.0, 16.0], [0.0, -16.0], [8.0, 0.0], [0.0, 0.0]])
    kind = spec.off.rstrip('0123456789')
    n = int(spec.off[len(kind):])
    if kind == 'r':
        return circle_offsets(n, s)
    if kind == 'k':
        return torch.cat([circle_offsets(10, s)[:n - 1], torch.zeros(1, 2)]).contiguous()
    g = torch.Generator().manual_seed(spec.seed + 5)
    reach = 1.5 if kind == 'split' else (60.0 if n < 1000 else 300.0)
    return torch.cat([(torch.rand(n - 1, 2, generator=g) * 2 - 1) * reach, torch.zeros(1, 2)]).contiguous()


def label_pool(ncls):
    """0, ncls - 1, every remainder mod 4, both sides of the 32-class trip, the last (partial) trip"""
    cand = {0, 1, 2, 3, 30, 31, 32, 33, ncls // 2, ncls - 4, ncls - 3, ncls - 2, ncls - 1, 32 * ((ncls - 1) // 32)}
    return sorted(c for c in cand if 0 <= c < ncls)


def _ulps(x, n):
    for i in (1, 2, 3):
        x = torch.where(n >= i, torch.nextafter(x, torch.full_like(x, math.inf)), x)
        x = torch.where(n <= -i, torch.nextafter(x, torch.full_like(x, -math.inf)), x)
    return x


class Case(NamedTuple):
    spec: Spec
    map: torch.Tensor
    centers: torch.Tensor
    labels: torch.Tensor
    bag_img: torch.Tensor
    off: torch.Tensor
    pad_hw: torch.Tensor
    img_hw: torch.Tensor
    nr_in: torch.Tensor
    reach: float


def _split_centres(spec, off, t):
    """a cluster of t same-label GTs where cdist_mm and cdist_direct choose different nearest GTs for some sample"""
    K = off.shape[0]
    for seed in range(400):
        g = torch.Generator().manual_seed(spec.seed * 1000 + seed)
        base = torch.tensor([[1000.37, 600.61]])
        if K == 1:          # near-identical centres a few ulps apart: cdist_mm's rounding noise decides between them
            c = _ulps(base.expand(t, 2).clone(), torch.randint(-3, 4, (t, 2), generator=g))
        else:
            c = base + torch.rand(t, 2, generator=g) * 2.0
        c = c.float()
        pts = c[:, None, :] + off[None]
        members = torch.arange(t)
        own = torch.arange(t)[:, None]
        a, _ = ref.nearest_choice(pts, members, 1, K, True)
        b, _ = ref.nearest_choice(pts, members, 1, K, False)
        if bool(((a == own) != (b == own)).any()):
            return c.contiguous()
    raise AssertionError(f'{spec.name}: no formula split found')


def build(spec, dev=None, with_map=True):
    g = torch.Generator().manual_seed(2000 + spec.seed)
    off = offsets(spec)
    K = off.shape[0]
    reach = float(off.abs().max())
    B, H, W, s, G = spec.B, spec.H, spec.W, spec.s, spec.G
    ext = torch.tensor([W * s, H * s])
    if spec.centres.startswith('split'):
        c = _split_centres(spec, off, G)
    elif spec.centres == 'lattice':
        c = torch.stack([torch.randint(2, int(W * s) // 16 - 1, (G,), generator=g),
                         torch.randint(2, int(H * s) // 16 - 1, (G,), generator=g)], 1).float() * 16
    else:
        cells = torch.stack([torch.randint(0, W, (G,), generator=g), torch.randint(0, H, (G,), generator=g)], 1).float() * s
        near = _ulps(cells, torch.randint(-2, 3, (G, 2), generator=g))
        if spec.centres == 'near':
            c = near
        else:
            c = torch.rand(G, 2, generator=g) * ext * 1.2 - 0.1 * ext
            pick = torch.randint(0, 4, (G,), generator=g)[:, None]
            c = torch.where(pick == 0, near, c)
            # clusters of a few GTs within a bag's reach, so that groups compete
            if G > 4:
                n_cl = G // 4
                src = torch.randint(0, G, (n_cl,), generator=g)
                dst = torch.randint(0, G, (n_cl,), generator=g)
                c[dst] = c[src] + (torch.rand(n_cl, 2, generator=g) - 0.5) * max(reach, s)
            # outside the pad (and so the image) on every side
            far = [(-reach - 5, 7.0), (W * s + 3, 9.0), (11.0, -2.0), (13.0, H * s + 1)]
            n_far = min(len(far), G // 8)
            if n_far:
                c[torch.randperm(G, generator=g)[:n_far]] = torch.tensor(far[:n_far])
        c = c.float().contiguous()
    bag_img = torch.randint(0, B, (G,), generator=g).int()
    if spec.labels == 'one':
        labels = torch.full((G,), min(2, spec.ncls - 1), dtype=torch.int32)
    elif spec.labels == 'unique':
        labels = torch.randperm(spec.ncls, generator=g)[:G].int()
    elif spec.labels == 'random':
        labels = torch.randint(0, spec.ncls, (G,), generator=g).int()
    else:
        pool = torch.tensor(label_pool(spec.ncls))
        labels = pool[torch.randint(0, len(pool), (G,), generator=g)].int()
    pad_hw = torch.tensor([[max(1, int(H * s) - 7 * b), max(1, int(W * s) - 5 * b)] for b in range(B)], dtype=torch.int32)
    img_hw = torch.tensor([[max(1, int(H * s) - 7 * b - 3 - 4 * b), max(1, int(W * s) - 5 * b - 9 - 2 * b)] for b in range(B)],
                          dtype=torch.int32)
    nr_in = torch.rand(G, generator=g) < 0.15
    m = None
    if with_map:
        C, ld = spec.ncls, spec.ld
        m = torch.randn(B, H, W, ld, generator=g) * spec.scale
        if spec.plant and C >= 2:
            # two channels equal across a band of the map: their sampled logits tie bit for bit.  Band 0: a tie below the label
            # C - 1 (rejects it); band 1: above the label 0 (accepts it); band 2: inside the float4 of labels 1 and 2; band 3: the
            # labels 0 and C - 1 both saturate to probability 1.0 (the lower class wins)
            base = torch.randn(B, H, W, generator=g) + 4.0
            band = torch.arange(W)[None, None, :].expand(B, H, W) * 4 // W
            lo = max(0, C - 5)
            for col in (C - 1, lo):
                m[..., col] = torch.where(band == 0, base, m[..., col])
            for col in (0, min(C - 1, 5)):
                m[..., col] = torch.where(band == 1, base, m[..., col])
            if C >= 3:
                for col in (1, 2):
                    m[..., col] = torch.where(band == 2, base, m[..., col])
            for col in (0, C - 1):
                m[..., col] = torch.where(band == 3, 20.0 + 10.0 * torch.rand(B, H, W, generator=g), m[..., col])
        m[..., C:] = float('nan')
    to = (lambda t: t.to(dev)) if dev is not None else (lambda t: t)
    return Case(spec, None if m is None else to(m), to(c), to(labels), to(bag_img), to(off), to(pad_hw), to(img_hw), to(nr_in), reach)


def plan_of(spec, reach, env_name):
    return ref.expected_plan(spec.ncls, spec.ld, offsets(spec).shape[0], reach, spec.s, ENVS[env_name])


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from pointtinybenchmark_b200 import ops
    return ops


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    for k in sorted(_runs, key=str):
        print(f'[refine calls] {k}: {_runs[k]}')
    for k, v in _worst.items():
        print(f'[refine] {k}: worst float error / bound {v:.3e}')
    for k, v in _undecided.items():
        print(f'[refine] {k}: GTs whose score lies within its bound of refine_th: {v}')


@pytest.fixture
def env(monkeypatch):
    def use(name):
        monkeypatch.delenv('PTB_REFINE_TMA', raising=False)
        for k, v in ENVS[name].items():
            monkeypatch.setenv(k, v)
    use('default')
    return use


def configs(spec):
    flag_sets = FLAG_SETS if spec.all_flags else [(True, True, False), (True, True, True), (False, False, False)]
    out = [(f, THRESHOLDS[0], False) for f in flag_sets]
    out += [((True, True, i == 1), th, True) for i, th in enumerate(THRESHOLDS[1:])]
    return out


def _fail(what, bad, worst, kind):
    _worst[kind] = max(_worst[kind], worst)
    assert not bad, f'{what}: {bad}'


@pytest.mark.parametrize('spec', SPECS, ids=lambda s: s.name)
def test_fused_refine_against_the_reference(ops, env, spec):
    dev = torch.device('cuda:0')
    d = build(spec, dev)
    comp = ref.fused_components(d.map, spec.ncls, d.centers, d.labels, d.bag_img, d.off, spec.s, d.pad_hw, d.img_hw)
    groups = ops.label_groups(d.bag_img, d.labels, spec.ncls)
    plans = {name: plan_of(spec, d.reach, name) for name in ENVS}
    if spec.centres == 'near':
        staged = window_staged(d.centers, d.reach, spec.s, spec.H, spec.W)
        assert plans['default'].use_tma and bool(staged.any()) and bool((~staged).any()), 'straddling and staged bags'
    for flags, (mth, alpha, rth), with_nr in configs(spec):
        cfg = ref.Cfg(mth, alpha, rth, *flags)
        rc = ops._refine_cfg(*cfg)
        want = ref.combine(comp, cfg, d.nr_in if with_nr else None)
        outs = {}
        for name in ENVS:
            env(name)
            n0 = ops.launch_count()
            o = ops.refine_fused(d.map, spec.ncls, d.centers, d.labels, d.bag_img, d.off, spec.s, d.pad_hw, d.img_hw, groups, rc,
                                 not_refine=d.nr_in if with_nr else None, want_chosen=True)
            assert ops.launch_count() == n0 + 1
            bad, worst, und = ref.check(want, o[0], o[1], o[2], chosen=o[3])
            _fail(f'{name} {plans[name]} {cfg} not_refine_in={with_nr}', bad, worst, 'fused')
            outs[name] = o
            _runs[plans[name].phase + (' tma' if plans[name].use_tma else ' global: ' + plans[name].fallback)] += 1
        _undecided['fused'] += und
        again = ops.refine_fused(d.map, spec.ncls, d.centers, d.labels, d.bag_img, d.off, spec.s, d.pad_hw, d.img_hw, groups, rc,
                                 not_refine=d.nr_in if with_nr else None, want_chosen=True)
        for a, b, c in zip(outs['default'], outs['tma0'], again):
            assert torch.equal(a, b), 'the staged and the global-memory path must agree bit for bit'
            assert torch.equal(a, c), 'two runs must agree bit for bit'
    # the padding columns are never read: other padding values change no bit
    env('default')
    m2 = d.map.clone()
    m2[..., spec.ncls:] = 1e30
    rc = ops._refine_cfg(0.1, 0.5, 0.1, True, True, False)
    a = ops.refine_fused(d.map, spec.ncls, d.centers, d.labels, d.bag_img, d.off, spec.s, d.pad_hw, d.img_hw, groups, rc, want_chosen=True)
    b = ops.refine_fused(m2, spec.ncls, d.centers, d.labels, d.bag_img, d.off, spec.s, d.pad_hw, d.img_hw, groups, rc, want_chosen=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    if spec.name == 'headline':
        assert int(a[3].sum()) > 0 and not bool(a[2].all())


def test_no_gts_launches_nothing(ops):
    dev = torch.device('cuda:0')
    m = torch.randn(1, 5, 6, 8, device=dev)
    z2 = torch.zeros(0, 2, device=dev)
    zi = torch.zeros(0, dtype=torch.int32, device=dev)
    hw = torch.tensor([[40, 48]], dtype=torch.int32, device=dev)
    groups = (zi, torch.zeros(1, dtype=torch.int32, device=dev), zi)
    n0 = ops.launch_count()
    o = ops.refine_fused(m, 5, z2, zi, zi, circle_offsets(1, 8.0).to(dev), 8.0, hw, hw, groups, ops._refine_cfg(0.1, 0.5, 0.1, True, True, False),
                         want_chosen=True)
    assert ops.launch_count() == n0
    assert o[0].shape == (0, 2) and o[3].shape == (0, 9)


# ----------------------------------------------------------------------------------------------------------------------------------
# stage kernel: probabilities given
# ----------------------------------------------------------------------------------------------------------------------------------
class StageSpec(NamedTuple):
    name: str
    ncls: int
    K: int
    R: int
    G: int
    labels: str = 'pool'


STAGE = [StageSpec('ncls20_K289', 20, 289, 1, 60), StageSpec('ncls32_K289', 32, 289, 1, 60), StageSpec('ncls33_K9', 33, 9, 1, 80),
         StageSpec('ncls80_K289', 80, 289, 1, 60), StageSpec('ncls131_K33', 131, 33, 1, 60), StageSpec('ncls5_Kt4096', 5, 4096, 1, 12),
         StageSpec('ncls80_group30', 80, 9, 1, 30, 'one'), StageSpec('ncls20_R2_K121', 20, 121, 2, 40),
         StageSpec('ncls6_R2_K5_direct', 6, 5, 2, 6, 'one')]


@pytest.mark.parametrize('spec', STAGE, ids=lambda s: s.name)
def test_stage_refine_against_the_reference(ops, spec):
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(spec.ncls * 7 + spec.K)
    C, K, R, G = spec.ncls, spec.K, spec.R, spec.G
    if K <= 441:
        off = torch.cat([circle_offsets(10, 8.0)[:K - 1], torch.zeros(1, 2)])
    else:
        off = torch.cat([(torch.rand(K - 1, 2, generator=g) * 2 - 1) * 200, torch.zeros(1, 2)])
    B = 2
    c0 = torch.rand(G, 2, generator=g) * torch.tensor([300.0, 200.0]) - 10
    c0[G // 2:] = c0[:G - G // 2][:G // 2] + torch.randn(G // 2, 2, generator=g) * 6        # neighbours that compete
    cr = torch.stack([c0] + [c0 + torch.randn(G, 2, generator=g) * 4 for _ in range(R - 1)], 1)   # (G,R,2)
    pts = (off[None, None] + cr[:, :, None]).reshape(G, R * K, 2).float()
    bag_img = torch.randint(0, B, (G,), generator=g).int()
    pad_hw = torch.tensor([[220, 300], [200, 290]], dtype=torch.int32)
    img_hw = torch.tensor([[210, 280], [190, 270]], dtype=torch.int32)
    ph, pw = pad_hw[bag_img.long(), 0].float()[:, None], pad_hw[bag_img.long(), 1].float()[:, None]
    valid = (pts[..., 0] >= 0) & (pts[..., 0] < pw) & (pts[..., 1] >= 0) & (pts[..., 1] < ph)
    prob = torch.sigmoid(torch.randn(G, R * K, C, generator=g) * 3)
    if C >= 4:
        prob[..., C - 3] = prob[..., 0]
        prob[..., 2] = prob[..., 1]
        hot = torch.rand(G, R * K, generator=g) < 0.2
        prob[..., 1] = torch.where(hot, torch.ones(()), prob[..., 1])
        prob[..., C - 1] = torch.where(hot, torch.ones(()), prob[..., C - 1])
    pool = torch.tensor(label_pool(C))
    labels = (torch.full((G,), min(2, C - 1)) if spec.labels == 'one' else pool[torch.randint(0, len(pool), (G,), generator=g)]).int()
    nr_in = torch.rand(G, generator=g) < 0.15
    comp = ref.components(prob, pts, valid, K, labels, bag_img, img_hw)
    t = comp.t
    if spec.labels == 'one':
        assert int(t.max()) > 2
    pts3 = torch.cat([pts, torch.full((G, R * K, 1), 8.0)], -1).to(dev)
    args = [x.to(dev) for x in (prob, valid, labels, bag_img, img_hw)]
    groups = ops.label_groups(args[3], args[2], C)
    for flags in FLAG_SETS:
        for th, with_nr in ((THRESHOLDS[0], False), (THRESHOLDS[1], True)):
            cfg = ref.Cfg(*th, *flags)
            want = ref.combine(comp, cfg, nr_in if with_nr else None)
            n0 = ops.launch_count()
            o = ops.refine(args[0], pts3, args[1], K, args[2], args[3], args[4], groups, ops._refine_cfg(*cfg),
                           not_refine=nr_in.to(dev) if with_nr else None)
            assert ops.launch_count() == n0 + 1
            bad, worst, und = ref.check(want, o[0], o[1], o[2], chosen=o[3], merge_valid=o[4])
            _fail(f'{cfg} not_refine_in={with_nr}', bad, worst, 'stage')
            _undecided['stage'] += und
            o2 = ops.refine(args[0], pts3, args[1], K, args[2], args[3], args[4], groups, ops._refine_cfg(*cfg),
                            not_refine=nr_in.to(dev) if with_nr else None)
            assert all(torch.equal(a, b) for a, b in zip(o, o2))


# ----------------------------------------------------------------------------------------------------------------------------------
# coverage of the dispatch table
# ----------------------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_row_of_the_dispatch_table():
    """from the case table alone, so that it holds whatever subset ran"""
    rows = collections.Counter()
    for spec in SPECS:
        d = build(spec, with_map=False)
        K = d.off.shape[0]
        for name in ENVS:
            p = plan_of(spec, d.reach, name)
            rows[p.phase] += 1
            rows['tma' if p.use_tma else 'global: ' + p.fallback] += 1
            rows[f'{p.phase} {"tma" if p.use_tma else "global"}'] += 1
            if p.passes >= 2:
                rows['passes >= 2'] += 1
            if p.use_tma:
                rows['straddling bags'] += int((~window_staged(d.centers, d.reach, spec.s, spec.H, spec.W)).sum())
        for members in ref.groups(d.bag_img, d.labels):
            t = len(members)
            if t > 1:
                rows['cdist_mm' if ref.use_mm(t, 1, K) else 'cdist_direct'] += 1
            if t > ref.GCAP:
                rows['t > 256'] += 1
            if t > 25:
                rows['t > 25'] += 1
    for k in sorted(rows):
        print(f'[coverage] {k}: {rows[k]}')
    for ph in ('fast<1>', 'fast<2>', 'fast<3>', 'fast<4>', 'loop'):
        for where in ('tma', 'global'):
            assert rows[f'{ph} {where}'] > 0, (ph, where)
    for row in ('global: env', 'global: ld', 'global: reach0', 'global: window', 'straddling bags', 'passes >= 2', 't > 256', 't > 25',
                'cdist_mm', 'cdist_direct'):
        assert rows[row] > 0, row
