"""GPU: the bag gather, ptb_cpr_bag_gather and ptb_cpr_bag_gather_bwd, against the host restatement of tests/gather_ref.py on every
kernel the host dispatches to (csrc/gather.cu):

  tma<32>, tma<64>   bag_gather_tma_kernel: one (bag, 32- or 64-channel chunk) per CTA, the bag's WS x WS window of the chunk staged in
                     shared memory by one TMA box; a bag whose window rounds one cell wider than WS reads global memory instead
  ldg<64>            bag_gather_kernel, 256 channels: whole samples per step
  ldg<40>, <20>, <0> bag_gather_kernel over the flattened (sample, 4-channel group) space, <0> with the width known at run time only
  TMA requested, but the window needs more than 112 KB of shared memory or the table has no reach -> the LDG kernel
  bwd                bag_gather_bwd_kernel: fp32 vector atomics, grid-stride over 32-sample groups

Forward: under the default environment and every forced path (PTB_GATHER_TMA, PTB_GATHER_CC, read by the host on every call), the
features are torch.equal to gather_f32, which is ATen's CPU grid_sample bit for bit; the points equal centre + offset in fp32 and the
validity the pad_hw test.  Backward: every element is within gamma(n + 2) * sum |w g| of the float64 scatter, the error bound of n fp32
terms added in any order; cells no sample touches and padding columns are exactly 0.  The LDG kernel takes its work items from a ticket
counter in the stream's scratch block, which resets itself at the end of every launch: tests interleave sizes, streams and the
fixed-order loss sums that share the block.  The last test checks that the cases cover every row of the dispatch table."""
import collections
import math
import re
from typing import NamedTuple, Optional

import pytest
import torch

from pointtinybenchmark_b200.ops import circle_offsets
from tests import gather_ref as ref

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ENVS = {'default': {}, 'tma0': {'PTB_GATHER_TMA': '0'}, 'tma1': {'PTB_GATHER_TMA': '1'}, 'cc32': {'PTB_GATHER_CC': '32'},
        'cc64': {'PTB_GATHER_CC': '64'}, 'tma1_cc32': {'PTB_GATHER_TMA': '1', 'PTB_GATHER_CC': '32'}}
SAMPLES_PER_BWD_TRIP = 132 * 8 * 256          # H100: sm_count * 8 blocks of 8 warps, 32 samples per warp per trip


class Spec(NamedTuple):
    name: str
    B: int
    H: int
    W: int
    C: int
    ld: int
    r: Optional[int]        # ring radius of ops.circle_offsets (0: the centre alone); None: the first K - 1 ring offsets of r = 8
    K: Optional[int]
    s: float
    G: int
    centres: str            # 'mixed', 'near' (a few ulps either side of cell positions), 'random', 'same'
    seed: int = 0


def _fwd_specs():
    out = []
    for C in (4, 16, 48, 80, 128, 160, 192, 256, 272):
        for pad in (0, 4, 32):
            out.append(Spec(f'width{C}_ld{C + pad}', 3, 13, 21, C, C + pad, 3, None, 8.0, 60, 'mixed', C + pad))
    for r in (1, 3, 8, 10, 16):
        out.append(Spec(f'radius{r}', 2, 40, 56, 128, 128, r, None, 8.0, 40, 'mixed', r))
    for s in (4.0, 16.0):
        for r in (3, 8):
            out.append(Spec(f'stride{int(s)}_r{r}', 2, 40, 56, 128, 128, r, None, s, 40, 'mixed', r))
    out += [Spec('centre_only_C128', 2, 13, 21, 128, 128, 0, None, 8.0, 50, 'mixed'),
            Spec('centre_only_C160', 2, 13, 21, 160, 164, 0, None, 8.0, 50, 'mixed')]
    for H, W in ((1, 1), (1, 5), (2, 1), (5, 2), (2, 5), (5, 5)):
        out.append(Spec(f'map{H}x{W}_C64', 2, H, W, 64, 64, 8, None, 8.0, 30, 'mixed', H * 10 + W))
    for H, W in ((1, 5), (5, 2)):
        out.append(Spec(f'map{H}x{W}_C160', 2, H, W, 160, 160, 8, None, 8.0, 30, 'mixed', H * 10 + W))
    out += [Spec('straddle_C160_r8', 2, 40, 56, 160, 160, 8, None, 8.0, 300, 'near'),
            Spec('straddle_C256_r8', 2, 40, 56, 256, 256, 8, None, 8.0, 300, 'near'),
            Spec('straddle_C128_r3', 2, 40, 56, 128, 128, 3, None, 8.0, 300, 'near')]
    for S, K in ((31, 31), (32, 16), (33, 11), (255, 15), (256, 16), (257, 257)):
        for C in (16, 80, 256):
            out.append(Spec(f'S{S}_K{K}_C{C}', 2, 13, 21, C, C, None, K, 8.0, S // K, 'mixed', S))
    out += [Spec('G1_C160', 1, 13, 21, 160, 160, 8, None, 8.0, 1, 'random'),
            Spec('headline_C160', 8, 100, 168, 160, 160, 8, None, 8.0, 4000, 'mixed'),
            Spec('headline_C256', 8, 100, 168, 256, 256, 8, None, 8.0, 4000, 'mixed')]
    return out


FWD = _fwd_specs()
BWD = ([Spec(f'bwd_width{C}_ld{ld}', 3, 13, 21, C, ld, 3, None, 8.0, 60, 'mixed', C) for C in (4, 16, 80, 160, 256, 272)
        for ld in (C, C + 4 if C < 100 else C + 32)]
       + [Spec('bwd_map1x5', 2, 1, 5, 16, 16, 8, None, 8.0, 40, 'mixed'),
          Spec('bwd_map5x2', 2, 5, 2, 80, 84, 8, None, 8.0, 40, 'mixed'),
          Spec('bwd_same_centre', 2, 13, 21, 16, 20, 8, None, 8.0, 2000, 'same'),
          Spec('bwd_headline_C4', 8, 100, 168, 4, 4, 8, None, 8.0, 4000, 'mixed'),
          Spec('bwd_headline_C16', 8, 100, 168, 16, 20, 8, None, 8.0, 4000, 'mixed')])
FLAGS = [Spec(f'flags_C{C}', 3, 13, 21, C, C, 3, None, 8.0, 60, 'mixed', 7) for C in (16, 160, 256)]
FLAG_SETS = [(a, b, c) for a in (True, False) for b in (True, False) for c in (True, False)]

_runs = collections.Counter()        # (kernel, fallback) of every forward call made
_stage = collections.Counter()       # staged / unstaged bags of the TMA calls
_worst = {}


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
        print(f'[gather calls] {k[0]}{" (TMA requested, fallback: " + k[1] + ")" if k[1] else ""}: {_runs[k]}')
    print(f'[gather calls] TMA bags staged: {_stage["staged"]}, read from global memory: {_stage["unstaged"]}')
    for k in sorted(_worst):
        print(f'[backward] worst error / bound {k}: {_worst[k]:.3e}')


@pytest.fixture
def env(monkeypatch):
    """sets one of ENVS for the calls that follow"""
    def use(name):
        for k in ('PTB_GATHER_TMA', 'PTB_GATHER_CC'):
            monkeypatch.delenv(k, raising=False)
        for k, v in ENVS[name].items():
            monkeypatch.setenv(k, v)
    use('default')
    return use


# ----------------------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------------------
def offsets(spec):
    if spec.K is None:
        return circle_offsets(spec.r, spec.s)
    return torch.cat([circle_offsets(8, spec.s)[:spec.K - 1], torch.zeros(1, 2)]).contiguous()


def _ulps(x, n):
    """x moved n (|n| <= 2) fp32 ulps, elementwise"""
    for i in (1, 2):
        x = torch.where(n >= i, torch.nextafter(x, torch.full_like(x, math.inf)), x)
        x = torch.where(n <= -i, torch.nextafter(x, torch.full_like(x, -math.inf)), x)
    return x


def centres(spec, g, reach):
    H, W, s, G = spec.H, spec.W, spec.s, spec.G
    ext = torch.tensor([W * s, H * s])
    cells = torch.stack([torch.randint(0, W, (G,), generator=g), torch.randint(0, H, (G,), generator=g)], 1).float() * s
    near = _ulps(cells, torch.randint(-2, 3, (G, 2), generator=g))
    if spec.centres == 'near':
        return near.contiguous()
    if spec.centres == 'random':
        return (torch.rand(G, 2, generator=g) * ext).contiguous()
    if spec.centres == 'same':              # one interior point and one beyond a corner, where the rings' taps clamp to the border
        two = torch.tensor([[W * s * 0.5 + 1.3, H * s * 0.5 - 2.1], [-2.5 * s, H * s + 1.5 * s]])
        return two[torch.arange(G) % 2].contiguous()
    c = torch.rand(G, 2, generator=g) * ext * 1.3 - 0.15 * ext
    pick = torch.randint(0, 3, (G,), generator=g)[:, None]
    c = torch.where(pick == 0, near, torch.where(pick == 1, cells, c))
    # outside each side and corner: partly (half the reach) and wholly (beyond the reach) off the map
    edges = []
    for d in (0.5 * reach + 1.25, reach + 2 * s + 0.5):
        mx, my = W * s * 0.5 + 0.75, H * s * 0.5 - 0.25
        edges += [(-d, my), (W * s + d, my), (mx, -d), (mx, H * s + d), (-d, -d), (W * s + d, H * s + d)]
    n_e = min(len(edges), G // 3)
    if n_e:
        c[torch.randperm(G, generator=g)[:n_e]] = torch.tensor(edges[:n_e])
    return c.float().contiguous()


class Case(NamedTuple):
    spec: Spec
    map: Optional[torch.Tensor]      # (B,H,W,ld) fp32 on the device, NaN in the padding columns
    centers: torch.Tensor
    bag_img: torch.Tensor
    off: torch.Tensor
    pad_hw: torch.Tensor
    reach: float


def build(spec, dev=None, with_map=True):
    """the case's tensors (on dev, CPU when None); the map only when with_map"""
    g = torch.Generator().manual_seed(1000 + spec.seed)
    off = offsets(spec)
    reach = float(off.abs().max())
    c = centres(spec, g, reach)
    bag_img = torch.randint(0, spec.B, (spec.G,), generator=g).int()            # images in no particular order
    pad_hw = torch.tensor([[max(1, int(spec.H * spec.s) - 7 * b), max(1, int(spec.W * spec.s) - 5 * b)] for b in range(spec.B)],
                          dtype=torch.int32)
    m = None
    if with_map:
        m = torch.randn(spec.B, spec.H, spec.W, spec.ld, generator=g)
        m[..., spec.C:] = float('nan')
    to = (lambda t: t.to(dev)) if dev is not None else (lambda t: t)
    return Case(spec, None if m is None else to(m), to(c), to(bag_img), to(off), to(pad_hw), reach)


def path_of(spec, reach, env_name, feats=True):
    return ref.expected_path(spec.C, spec.ld, offsets(spec).shape[0], reach, spec.s, ENVS[env_name], spec.G, feats)


def _ndiff(a, b):
    return int((a.view(torch.int32) != b.view(torch.int32)).sum()) if a.shape == b.shape else -1


# ----------------------------------------------------------------------------------------------------------------------------------
# forward
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('spec', FWD, ids=lambda s: s.name)
def test_forward_is_bit_exact_on_every_path(ops, env, spec):
    dev = torch.device('cuda:0')
    d = build(spec, dev)
    want = ref.gather_f32(d.map, d.centers, d.bag_img, d.off, spec.s, spec.C)
    assert not torch.isnan(want).any()
    pts_want = ref.sample_points(d.centers.cpu(), d.off.cpu()).to(dev)
    valid_want = ref.point_valid(d.centers.cpu(), d.bag_img.cpu(), d.off.cpu(), d.pad_hw.cpu()).to(dev)
    staged = ref.window_staged(d.centers, d.reach, spec.s, spec.H, spec.W)
    if spec.centres == 'near':
        assert bool(staged.any()) and bool((~staged).any()), 'the case must hold both staged and straddling bags'
    for name in ENVS:
        env(name)
        p = path_of(spec, d.reach, name)
        f, pts, valid = ops.bag_gather(d.map, d.centers, d.bag_img, d.off, spec.s, d.pad_hw, C=spec.C)
        assert torch.equal(f, want), f'{name} -> {p.kernel}: {_ndiff(f, want)} / {want.numel()} values differ from gather_f32'
        assert torch.equal(pts[..., :2], pts_want) and bool((pts[..., 2] == spec.s).all()), f'{name} -> {p.kernel}: points'
        assert torch.equal(valid, valid_want), f'{name} -> {p.kernel}: validity'
        _runs[p] += 1
        if p.kernel.startswith('tma'):
            _stage['staged'] += int(staged.sum())
            _stage['unstaged'] += int((~staged).sum())


@pytest.mark.parametrize('spec', FLAGS, ids=lambda s: s.name)
def test_each_output_switches_off_alone(ops, env, spec):
    """feats, pts and valid in all eight combinations: what is written equals the full call.  Without features the host passes no
    reach and takes the LDG kernel; with them at 160 channels the TMA kernel, which writes points and validity once per bag"""
    dev = torch.device('cuda:0')
    d = build(spec, dev)
    for name in ('default', 'tma0'):
        env(name)
        full = ops.bag_gather(d.map, d.centers, d.bag_img, d.off, spec.s, d.pad_hw)
        for flags in FLAG_SETS:
            got = ops.bag_gather(d.map, d.centers, d.bag_img, d.off, spec.s, d.pad_hw, feats=flags[0], pts=flags[1], valid=flags[2])
            for on, x, y, what in zip(flags, got, full, ('feats', 'pts', 'valid')):
                assert (x is not None) == on, (name, flags, what)
                if on:
                    assert torch.equal(x, y), (name, flags, what)
            _runs[path_of(spec, d.reach, name, feats=flags[0])] += 1


def test_no_bags_launches_nothing(ops, env):
    dev = torch.device('cuda:0')
    m = torch.randn(2, 13, 21, 16, device=dev)
    off = circle_offsets(3, 8.0).to(dev)
    c, b = torch.zeros(0, 2, device=dev), torch.zeros(0, dtype=torch.int32, device=dev)
    pad = torch.tensor([[104, 168]] * 2, dtype=torch.int32, device=dev)
    n0 = ops.launch_count()
    f, p, v = ops.bag_gather(m, c, b, off, 8.0, pad, reach_px=24.0)
    assert f.shape == (0, off.shape[0], 16) and p.shape == (0, off.shape[0], 3) and v.shape == (0, off.shape[0])
    gm = ops.bag_gather_bwd(torch.zeros(0, off.shape[0], 16, device=dev), (2, 13, 21, 16), c, b, off, 8.0)
    assert ops.launch_count() == n0
    assert gm.shape == (2, 13, 21, 16) and not bool(gm.any())


def _sched_jobs(dev):
    """cases of different sizes for the LDG kernel (many, one and a partial 256-sample work item)"""
    specs = [Spec('sched_a', 3, 13, 21, 16, 16, 3, None, 8.0, 700, 'mixed', 1),
             Spec('sched_b', 3, 13, 21, 16, 16, None, 15, 8.0, 17, 'mixed', 2),
             Spec('sched_c', 3, 13, 21, 256, 256, 8, None, 8.0, 90, 'mixed', 3),
             Spec('sched_d', 3, 13, 21, 80, 80, 0, None, 8.0, 1, 'mixed', 4),
             Spec('sched_e', 8, 100, 168, 80, 80, 8, None, 8.0, 2000, 'mixed', 5)]
    out = []
    for spec in specs:
        d = build(spec, dev)
        out.append((d, ref.gather_f32(d.map, d.centers, d.bag_img, d.off, spec.s, spec.C)))
    return out


def _call(ops, d):
    return ops.bag_gather(d.map, d.centers, d.bag_img, d.off, d.spec.s, d.pad_hw, reach_px=d.reach)[0]


def test_back_to_back_calls_on_one_stream(ops, env):
    dev = torch.device('cuda:0')
    env('tma0')
    jobs = _sched_jobs(dev)
    order = [0, 1, 2, 3, 4, 3, 1, 0, 4, 2, 2, 1, 1, 0, 3, 4]
    runs = []
    for _ in range(2):
        runs.append([_call(ops, jobs[i][0]) for i in order])          # no synchronisation in between
    torch.cuda.synchronize()
    for k, i in enumerate(order):
        assert torch.equal(runs[0][k], jobs[i][1]), f'call {k} ({jobs[i][0].spec.name}): {_ndiff(runs[0][k], jobs[i][1])} values differ'
        assert torch.equal(runs[1][k], runs[0][k])


def test_concurrent_calls_on_two_streams(ops, env):
    dev = torch.device('cuda:0')
    env('tma0')
    jobs = _sched_jobs(dev)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    main = torch.cuda.current_stream()
    a, b = [4, 0, 4, 1, 4, 2], [0, 4, 3, 4, 1, 4]
    ra, rb = [], []
    torch.cuda.synchronize()
    for _ in range(3):
        torch.cuda._sleep(50_000_000)          # holds both streams back until all their launches are queued, so that they overlap
        s1.wait_stream(main)
        s2.wait_stream(main)
        for i, j in zip(a, b):
            with torch.cuda.stream(s1):
                ra.append((i, _call(ops, jobs[i][0])))
            with torch.cuda.stream(s2):
                rb.append((j, _call(ops, jobs[j][0])))
    torch.cuda.synchronize()
    for i, r in ra + rb:
        assert torch.equal(r, jobs[i][1]), f'{jobs[i][0].spec.name} on two streams: {_ndiff(r, jobs[i][1])} values differ'


def test_gather_after_a_fixed_order_sum_on_the_same_stream(ops, env):
    """the fixed-order loss sums use the same per-stream scratch block as the gather's ticket counter"""
    dev = torch.device('cuda:0')
    env('tma0')
    jobs = _sched_jobs(dev)
    g = torch.Generator().manual_seed(8)
    pred, tgt = torch.randn(100_000, 2, generator=g).to(dev), torch.randn(100_000, 2, generator=g).to(dev)
    solo = ops.mse(pred, tgt, None, 0.125)
    got = []
    for i in (0, 4, 1, 2, 3):
        s1 = ops.mse(pred, tgt, None, 0.125)
        got.append((i, _call(ops, jobs[i][0]), s1, ops.mse(pred, tgt, None, 0.125)))
    torch.cuda.synchronize()
    for i, f, s1, s2 in got:
        assert torch.equal(f, jobs[i][1]), f'{jobs[i][0].spec.name} after a loss sum: {_ndiff(f, jobs[i][1])} values differ'
        assert torch.equal(s1, solo) and torch.equal(s2, solo)


_KERNEL = re.compile(r'bag_gather_(tma_)?kernel<(\d+)>')


def test_expected_path_names_the_kernel_that_runs(ops, env):
    """expected_path, which the coverage count relies on, against the kernel names torch.profiler records"""
    dev = torch.device('cuda:0')
    by_name = {s.name: s for s in FWD}
    calls = [('width160_ld160', 'default', True), ('radius8', 'cc64', True), ('width256_ld256', 'tma1', True),
             ('width256_ld288', 'tma1_cc32', True), ('width256_ld256', 'default', True), ('width160_ld164', 'tma0', True),
             ('width80_ld80', 'default', True), ('width16_ld16', 'default', True), ('radius16', 'default', True),
             ('radius10', 'default', True), ('radius10', 'cc64', True), ('centre_only_C160', 'default', True),
             ('width160_ld160', 'default', False), ('map1x5_C64', 'default', True), ('map5x2_C160', 'tma1', True)]
    for name, env_name, feats in calls:
        spec = by_name[name]
        d = build(spec, dev)
        env(env_name)
        want = path_of(spec, d.reach, env_name, feats)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ops.bag_gather(d.map, d.centers, d.bag_img, d.off, spec.s, d.pad_hw, C=spec.C, feats=feats)
            torch.cuda.synchronize()
        got = []
        for e in prof.events():
            m = _KERNEL.search(e.name)
            if m:
                got.append(f'{"tma" if m.group(1) else "ldg"}<{m.group(2)}>')
        assert got == [want.kernel], (name, env_name, feats, got, want)


# ----------------------------------------------------------------------------------------------------------------------------------
# backward
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('spec', BWD, ids=lambda s: s.name)
def test_backward_within_the_any_order_bound_of_float64(ops, spec):
    dev = torch.device('cuda:0')
    d = build(spec, dev, with_map=False)
    K = d.off.shape[0]
    g = torch.Generator().manual_seed(spec.seed + 77)
    go = torch.randn(spec.G, K, spec.C, generator=g)
    gm = ops.bag_gather_bwd(go.to(dev), (spec.B, spec.H, spec.W, spec.ld), d.centers, d.bag_img, d.off, spec.s).cpu()
    want, absum, count = ref.scatter_f64(go, (spec.B, spec.H, spec.W, spec.ld), d.centers, d.bag_img, d.off, spec.s)
    n = count.double()
    # n fp32 products and their sum in any order: |error| <= gamma(n + 2) * sum |w g|; fp32 atomics flush subnormals (< 2^-126 each)
    bound = (n + 2) * U / (1 - (n + 2) * U) * absum + n * 2.0 ** -126
    err = (gm.double() - want).abs()
    ratio = float((err / bound)[bound > 0].max())
    _worst[spec.name] = ratio
    nbad = int((err > bound).sum())
    assert nbad == 0, f'{nbad} elements outside the bound (worst error / bound {ratio:.3e}, most terms in a cell {int(count.max())})'
    assert bool((gm[..., spec.C:] == 0).all()), 'padding columns must stay 0'
    assert bool((gm[(count == 0).expand_as(gm)] == 0).all()), 'cells no sample touches must stay 0'
    if spec.centres == 'same':
        assert int(count.max()) >= 1000
    if spec.name.startswith('bwd_headline'):
        assert spec.G * K > 4 * SAMPLES_PER_BWD_TRIP


# ----------------------------------------------------------------------------------------------------------------------------------
# coverage of the dispatch table
# ----------------------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_row_of_the_dispatch_table():
    """from the case table alone (expected_path is checked against the profiler above), so that it holds whatever subset ran"""
    per_kernel = collections.Counter()
    rows = collections.Counter()
    stage = collections.Counter()
    for spec in FWD:
        d = build(spec, with_map=False)
        staged = None
        for name in ENVS:
            p = path_of(spec, d.reach, name)
            per_kernel[p.kernel] += 1
            if p.fallback:
                rows['TMA requested -> ldg: ' + p.fallback] += 1
            if spec.ld > spec.C:
                rows[('tma' if p.kernel.startswith('tma') else 'ldg') + ' with ld > C'] += 1
            if p.kernel.startswith('tma'):
                if staged is None:
                    staged = ref.window_staged(d.centers, d.reach, spec.s, spec.H, spec.W)
                stage[p.kernel + ' staged'] += int(staged.sum())
                stage[p.kernel + ' unstaged'] += int((~staged).sum())
    for spec in FLAGS:
        reach = float(offsets(spec).abs().max())
        for name in ('default', 'tma0'):
            for flags in FLAG_SETS:
                p = path_of(spec, reach, name, feats=flags[0])
                per_kernel[p.kernel] += 1
                if p.fallback:
                    rows['TMA requested -> ldg: ' + p.fallback] += 1
    for spec in BWD:
        K = offsets(spec).shape[0]
        rows['bwd'] += 1
        if spec.ld > spec.C:
            rows['bwd with ld > C'] += 1
        if spec.G * K > SAMPLES_PER_BWD_TRIP:
            rows['bwd over several grid-stride trips'] += 1
    for k in sorted(per_kernel):
        print(f'[coverage] {k}: {per_kernel[k]} forward calls')
    for k in sorted(rows):
        print(f'[coverage] {k}: {rows[k]}')
    for k in sorted(stage):
        print(f'[coverage] bags {k}: {stage[k]}')
    assert set(per_kernel) == {'tma<32>', 'tma<64>', 'ldg<64>', 'ldg<40>', 'ldg<20>', 'ldg<0>'}
    for row in ('TMA requested -> ldg: window', 'TMA requested -> ldg: reach0', 'tma with ld > C', 'ldg with ld > C',
                'bwd with ld > C', 'bwd over several grid-stride trips'):
        assert rows[row] > 0, row
    for k in ('tma<32>', 'tma<64>'):
        assert stage[k + ' staged'] > 0 and stage[k + ' unstaged'] > 0, k
