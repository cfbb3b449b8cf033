"""CPU: layers.tower_path, the one decision of which backend a tower runs on, over PTB_CONV_MODE x PTB_TOWER_TRAIN x input dtype x
device x grad state x geometry, and tower()'s refusals that come before any device work.  The decision reads of its input only
is_cuda, dtype and requires_grad, so a stand-in drives it here for CUDA inputs too.  The expectations were written from the
predicates that made this decision before it was one function."""
import contextlib
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn

from pointtinybenchmark_b200 import layers

GN = dict(type='GN', num_groups=32)
DT = dict(fp32=torch.float32, fp16=torch.float16, bf16=torch.bfloat16, fp64=torch.float64)
INPUTS = [(dev, dt) for dev in ('cpu', 'cuda') for dt in DT]
MODES = [(mode, train) for mode in ('f16x2', 'tf32x3') for train in ('tc', 'cudnn')]
CODE = {'f16': 'wgmma-f16x2', 'tf32': 'wgmma-3xtf32', 'train': 'wgmma-f16x2-train', 'cudnn': 'cudnn'}
RAISES = {'cpu!': (RuntimeError, 'no CPU'), 'plan!': (NotImplementedError, 'PTB_CONV_MODE=tf32x3')}


def _module(cin=256, cout=256, k=3, stride=1, padding=1, norm_cfg=GN, bias=False, act=True, **conv):
    m = layers.ConvModule(cin, cout, k, stride, padding, norm_cfg=norm_cfg, bias=bias, act=act)
    if conv:
        m.conv = nn.Conv2d(cin, cout, k, stride, padding, bias=bias, **conv)
    return m


def _non_affine():
    m = _module()
    m.gn = nn.GroupNorm(32, 256, affine=False)
    return m


# one tower per row; every row but the first two changes one field of the shipped 256 -> 256 layer
GEOMETRY = {
    'shipped': lambda: [_module(), _module()],
    'cin64': lambda: [_module(cin=64), _module()],
    'kernel': lambda: [_module(k=1, padding=0)],
    'stride': lambda: [_module(stride=2)],
    'padding': lambda: [_module(padding=0)],
    'dilation': lambda: [_module(dilation=2)],
    'groups': lambda: [_module(groups=2)],
    'bias': lambda: [_module(bias=True)],
    'out128': lambda: [_module(cout=128)],
    'cin48': lambda: [_module(cin=48)],
    'bn': lambda: [_module(norm_cfg=dict(type='BN'))],
    'gn16': lambda: [_module(norm_cfg=dict(type='GN', num_groups=16))],
    'gn_non_affine': lambda: [_non_affine()],
    'no_act': lambda: [_module(act=False)],
    'empty': lambda: [],
    'second_layer_bias': lambda: [_module(), _module(bias=True)],
}

# grad states: off = under no_grad; on = grad enabled, nothing requires grad; x = the input requires grad; w = the tower's
# parameters require grad; also-tower / also-head = frozen tower, an output conv that requires grad, asked without / with `also`
GRAD_STATES = ('off', 'on', 'x', 'w', 'also-tower', 'also-head')


def make_state(convs, state, dev, dtype):
    """(convs, stand-in x, also, grad context) for one grad state"""
    out = nn.Conv2d(256, 8, 3, padding=1)
    for m in convs:
        m.requires_grad_(state in ('off', 'w'))
    x = SimpleNamespace(is_cuda=dev == 'cuda', dtype=dtype, requires_grad=state == 'x')
    ctx = torch.no_grad() if state == 'off' else contextlib.nullcontext()
    return convs, x, ((out,) if state == 'also-head' else ()), ctx


TABLE = {
    # (PTB_CONV_MODE, PTB_TOWER_TRAIN, grad state): the shipped tower for an input in
    # CPU fp32, fp16, bf16, fp64, then CUDA fp32, fp16, bf16, fp64
    ('f16x2', 'tc', 'off'):              'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'tc', 'on'):               'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'tc', 'x'):                'cudnn cpu!  cpu!  cudnn train train train cudnn',
    ('f16x2', 'tc', 'w'):                'cudnn cpu!  cpu!  cudnn train train train cudnn',
    ('f16x2', 'tc', 'also-tower'):       'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'tc', 'also-head'):        'cudnn cpu!  cpu!  cudnn train train train cudnn',
    ('f16x2', 'cudnn', 'off'):           'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'cudnn', 'on'):            'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'cudnn', 'x'):             'cudnn cpu!  cpu!  cudnn cudnn cudnn cudnn cudnn',
    ('f16x2', 'cudnn', 'w'):             'cudnn cpu!  cpu!  cudnn cudnn cudnn cudnn cudnn',
    ('f16x2', 'cudnn', 'also-tower'):    'cudnn cpu!  cpu!  cudnn f16   f16   f16   cudnn',
    ('f16x2', 'cudnn', 'also-head'):     'cudnn cpu!  cpu!  cudnn cudnn cudnn cudnn cudnn',
    ('tf32x3', 'tc', 'off'):             'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'tc', 'on'):              'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'tc', 'x'):               'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
    ('tf32x3', 'tc', 'w'):               'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
    ('tf32x3', 'tc', 'also-tower'):      'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'tc', 'also-head'):       'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'off'):          'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'on'):           'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'x'):            'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'w'):            'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'also-tower'):   'cudnn cpu!  cpu!  cudnn tf32  plan! plan! cudnn',
    ('tf32x3', 'cudnn', 'also-head'):    'cudnn cpu!  cpu!  cudnn cudnn plan! plan! cudnn',
}

GEOMETRY_TABLE = {
    # a CUDA fp32 input at f16x2 inference, tf32x3 inference, f16x2 training (grad, weights require grad)
    'shipped':           'f16   tf32  train',
    'cin64':             'f16   tf32  cudnn',
    'kernel':            'cudnn cudnn cudnn',
    'stride':            'cudnn cudnn cudnn',
    'padding':           'cudnn cudnn cudnn',
    'dilation':          'cudnn cudnn cudnn',
    'groups':            'cudnn cudnn cudnn',
    'bias':              'cudnn cudnn cudnn',
    'out128':            'cudnn cudnn cudnn',
    'cin48':             'cudnn cudnn cudnn',
    'bn':                'cudnn cudnn cudnn',
    'gn16':              'cudnn cudnn cudnn',
    'gn_non_affine':     'f16   tf32  cudnn',
    'no_act':            'cudnn cudnn cudnn',
    'empty':             'cudnn cudnn cudnn',
    'second_layer_bias': 'cudnn cudnn cudnn',
}


def _expect(code, convs, x, also=()):
    if code in RAISES:
        exc, match = RAISES[code]
        with pytest.raises(exc, match=match):
            layers.tower_path(convs, x, also)
    else:
        assert layers.tower_path(convs, x, also) == CODE[code]


@pytest.mark.parametrize('mode,train,state', list(TABLE))
def test_tower_path_over_mode_dtype_device_and_grad_state(monkeypatch, mode, train, state):
    monkeypatch.setenv('PTB_CONV_MODE', mode)
    monkeypatch.setenv('PTB_TOWER_TRAIN', train)
    codes = TABLE[mode, train, state].split()
    assert len(codes) == len(INPUTS)
    tower = GEOMETRY['shipped']()
    for (dev, dt), code in zip(INPUTS, codes):
        convs, x, also, ctx = make_state(tower, state, dev, DT[dt])
        with ctx:
            _expect(code, convs, x, also)


@pytest.mark.parametrize('name', list(GEOMETRY_TABLE))
def test_tower_path_over_geometry(monkeypatch, name):
    assert set(GEOMETRY) == set(GEOMETRY_TABLE)
    monkeypatch.setenv('PTB_TOWER_TRAIN', 'tc')
    tower = GEOMETRY[name]()
    for (mode, state), code in zip((('f16x2', 'off'), ('tf32x3', 'off'), ('f16x2', 'w')), GEOMETRY_TABLE[name].split()):
        monkeypatch.setenv('PTB_CONV_MODE', mode)
        convs, x, also, ctx = make_state(tower, state, 'cuda', torch.float32)
        with ctx:
            _expect(code, convs, x, also)


def test_tower_path_defaults_and_other_modes(monkeypatch):
    """unset variables mean PTB_CONV_MODE=f16x2 and PTB_TOWER_TRAIN=tc; any mode other than f16x2 is the 3xTF32 mode"""
    monkeypatch.delenv('PTB_CONV_MODE', raising=False)
    monkeypatch.delenv('PTB_TOWER_TRAIN', raising=False)
    tower = GEOMETRY['shipped']()
    for state, code in (('off', 'f16'), ('w', 'train')):
        convs, x, also, ctx = make_state(tower, state, 'cuda', torch.float32)
        with ctx:
            _expect(code, convs, x, also)
    monkeypatch.setenv('PTB_CONV_MODE', 'fp32')
    convs, x, also, ctx = make_state(tower, 'off', 'cuda', torch.float32)
    with ctx:
        _expect('tf32', convs, x, also)
    x.dtype = torch.float16
    with ctx, pytest.raises(NotImplementedError, match='PTB_CONV_MODE=fp32'):
        layers.tower_path(convs, x)


def test_tower_refusals_come_before_any_device_work(monkeypatch):
    """tower(): want='f16pair' off the wgmma-f16x2 path is a ValueError, and a CUDA half input bound for cuDNN is refused"""
    monkeypatch.setenv('PTB_TOWER_TRAIN', 'tc')
    shipped = GEOMETRY['shipped']()
    for mode, state, dev in (('tf32x3', 'off', 'cuda'), ('f16x2', 'w', 'cuda'), ('f16x2', 'off', 'cpu')):
        monkeypatch.setenv('PTB_CONV_MODE', mode)
        convs, x, _, ctx = make_state(shipped, state, dev, torch.float32)
        with ctx, pytest.raises(ValueError, match='f16pair'):
            layers.tower(convs, x, {}, want='f16pair')
    monkeypatch.setenv('PTB_CONV_MODE', 'f16x2')
    for dt in (torch.float16, torch.bfloat16):
        for name, state in (('bias', 'off'), ('cin64', 'w')):
            convs, x, _, ctx = make_state(GEOMETRY[name](), state, 'cuda', dt)
            with ctx, pytest.raises(NotImplementedError, match='needs the tensor-core geometry'):
                layers.tower(convs, x)
