"""CPU: host side of the half-precision input paths of the towers (layers.input_plan), the number-level statement behind them
(an fp16 value is its own hi operand; a bf16 value fits one fp16 hi after the per-tensor power-of-two scale) restated in numpy over
every bit pattern, and the 'no CPU path' rule for half inputs."""
import numpy as np
import pytest
import torch

from pointtinybenchmark_b200 import cpr_head, layers, p2p_head  # noqa: F401  (the head modules register their classes)
from pointtinybenchmark_b200.registry import build_head
from tests.test_gpu_cpr_head import head_cfg as cpr_cfg
from tests.test_gpu_p2p import head_cfg as p2p_cfg

D = dict(num_classes=80, C=256, stride=8, radius=8)


def test_input_plan_is_a_pure_function_of_dtype_and_conv_mode():
    plan = layers.input_plan
    # fp32: exactly the choice made without half-precision support
    assert plan(torch.float32, 'f16x2') == ('fp32-split', 'f16x2', torch.float32)
    assert plan(torch.float32, 'tf32x3') == ('fp32-split', 'tf32x3', torch.float32)
    assert plan(torch.float32) == plan(torch.float32, 'f16x2')
    assert plan(torch.float16, 'f16x2') == ('fp16-direct', 'f16x1a', torch.float16)
    assert plan(torch.bfloat16, 'f16x2') == ('bf16-split', 'f16x2', torch.bfloat16)
    for dt in (torch.float16, torch.bfloat16):
        with pytest.raises(NotImplementedError, match='PTB_CONV_MODE=tf32x3'):
            plan(dt, 'tf32x3')
    for dt in (torch.float64, torch.int32, torch.uint8, torch.bool):
        assert plan(dt, 'f16x2') is None and plan(dt, 'tf32x3') is None


def _pow2_scale_for(amax):
    """pow2_scale_for of csrc/conv_tc.cu: the power of two that brings amax into [2^11, 2^12); 1 for 0 / inf / nan."""
    if not (amax > 0) or not np.isfinite(amax):
        return np.float32(1.0)
    _, e = np.frexp(np.float32(amax))
    return np.ldexp(np.float32(1.0), 12 - int(e))


def _split(v):
    """split_h2 of csrc/tc_ptx.cuh on fp32 values: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


F16_MIN_SUBNORMAL, F16_MIN_NORMAL = 2.0 ** -24, 2.0 ** -14


@pytest.mark.parametrize('amax_bits', [0x7F7F, 0x4780, 0x3F80, 0x3C00, 0x0800])
def test_bf16_to_operand_pair_rule_over_every_bit_pattern(amax_bits):
    """every finite bf16 value not above a tensor maximum `amax` (from bf16's largest finite value down to 2^-111; the
    power-of-two scale of a maximum below 2^-116 is not an fp32 number, for fp32 inputs alike),
    with s = pow2_scale_for(amax) and v = x * s as the kernel forms it in fp32:
      * v is the exact product wherever it reaches fp16's smallest subnormal 2^-24 (a power-of-two scale);
      * |v| a normal fp16 number: hi == v and lo == 0 (8 significand bits fit fp16's 11);
      * 2^-24 <= |v| < 2^-14: hi + lo == v whenever v is a multiple of 2^-24 (every |v| >= 2^-17), and within 2^-25 otherwise,
        which is 2^-36 of the tensor's maximum (amax * s >= 2^11): lo cannot hold a residual below half of fp16's smallest step."""
    bits = np.arange(65536, dtype=np.uint32)
    x = (bits << 16).view(np.float32)
    amax = (np.array([amax_bits], dtype=np.uint32) << 16).view(np.float32)[0]
    x = x[np.isfinite(x) & (np.abs(x) <= amax)]
    s = _pow2_scale_for(amax)
    with np.errstate(under='ignore', invalid='ignore'):
        v = x * s
    assert 2048 <= float(amax) * float(s) < 4096
    exact = x.astype(np.float64) * float(s)
    big = np.abs(exact) >= F16_MIN_SUBNORMAL
    v64 = v.astype(np.float64)
    assert np.array_equal(v64[big], exact[big])
    hi, lo = _split(v)
    assert np.all(np.isfinite(hi.astype(np.float32))), 'the scale keeps every value of the tensor inside the fp16 range'
    pair = hi.astype(np.float64) + lo.astype(np.float64)
    normal = np.abs(exact) >= F16_MIN_NORMAL
    assert normal.sum() > 0 and np.array_equal(pair[normal], exact[normal]) and np.all(lo[normal] == 0)
    sub = big & ~normal
    on_grid = sub & (np.abs(exact) >= 2.0 ** -17)
    assert np.array_equal(pair[on_grid], exact[on_grid])
    assert np.all(np.abs(pair[sub] - exact[sub]) <= 2.0 ** -25)


def test_every_finite_fp16_value_is_its_own_hi_operand():
    h = np.arange(65536, dtype=np.uint16).view(np.float16)
    h = h[np.isfinite(h)]
    hi, lo = _split(h.astype(np.float32))           # scale 1
    assert np.array_equal(hi.view(np.uint16), h.view(np.uint16))
    assert np.all(lo == 0) and not np.any(np.signbit(lo))


def test_heads_keep_their_constructor_surface_and_tower_path_refuses_cpu_half_inputs():
    cpr, p2p = build_head(cpr_cfg(D)), build_head(p2p_cfg(dict(D, stride=4)))
    assert all(p.dtype == torch.float32 for h in (cpr, p2p) for p in h.parameters()), 'parameters stay fp32'
    for dt in (torch.float16, torch.bfloat16):
        x = torch.zeros(1, 256, 8, 8, dtype=dt)
        with pytest.raises(RuntimeError, match='no CPU'):
            cpr.forward((x,))
        with pytest.raises(RuntimeError, match='no CPU'):
            p2p.forward((x,))
        with pytest.raises(RuntimeError, match='no CPU'):
            layers.tower(cpr.cls_convs, x)
        with pytest.raises(RuntimeError, match='no CPU'):
            layers.tower_path(cpr.cls_convs, x)
