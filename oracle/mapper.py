"""Oracle: iw3/mapper.py get_mapper(name) for every name, blend and chain (TEST INFRASTRUCTURE).

A torch-CPU fp32 restatement.  ``none`` and ``div_*`` are oracle.iw3.mapper itself (the bench's reference arm uses
that one); the other functions are restated here:
  mapper.py:7-11   softplus01_legacy (softplus, softplus2)
  mapper.py:14-19  softplus01 (mul_*)
  mapper.py:22-26  inv_softplus01 (inv_mul_*; its min/max are fp32 tensor values)
  mapper.py:39-61  shift_relative_depth (shift_*)
  mapper.py:129-151 the chain "s1:s2" and the blend "a+b=w", where every blend of a chain takes the LAST blend's
                   functions and weight (the reference's lambdas are late-bound).
oracle/gen_golden_mapper.py pins it to the real reference (tests/golden/mapper.npz).
"""
import math
import torch

from . import iw3 as _iw3

_MUL = {"mul_1": (0.343, 12), "mul_2": (0.515, 12), "mul_3": (0.687, 12)}
_INV_MUL = {"inv_mul_1": (-0.002102, 7.8788), "inv_mul_2": (-0.0003, 6.2626), "inv_mul_3": (-0.0001, 3.4343)}
_SHIFT = {"shift_30": 3.0, "shift_20": 2.0, "shift_14": 1.4, "shift_08": 0.8, "shift_06": 0.6, "shift_045": 0.45}


def _softplus_legacy(x):
    lo = math.log(1 + math.exp(-6.0)) / 6
    hi = math.log(1 + math.exp(6.0)) / 6
    return (torch.log(1. + torch.exp(x * 12.0 - 6)) / 6 - lo) / (hi - lo)


def _softplus01(x, bias, scale):
    lo = math.log(1 + math.exp(-bias * scale))
    hi = math.log(1 + math.exp((1 - bias) * scale))
    return (torch.log(1. + torch.exp((x - bias) * scale)) - lo) / (hi - lo)


def _inv_softplus01(x, bias, scale):
    def f(v):
        return ((v - bias) * scale).expm1().clamp(min=1e-6).log()
    lo, hi = f(torch.zeros(1, dtype=x.dtype)), f(torch.ones(1, dtype=x.dtype))
    return (f(x) - lo) / (hi - lo)


def _shift(x, d, far=16):
    near_far = d + far
    distance = 1 / (1.0 / near_far + (1.0 / d - 1.0 / near_far) * x)
    disparity = 1.0 / ((1.0 - d) + distance)
    return (disparity - 1.0 / (far + 1)) / (1.0 - 1.0 / (far + 1))


def function(name):
    """One function of resolve_mapper_function (mapper.py:64-120)."""
    if name == "none" or name in _iw3._DIV_C:
        return lambda x: _iw3.mapper(x, name)
    if name == "pow2":
        return lambda x: x ** 2
    if name == "softplus":
        return _softplus_legacy
    if name == "softplus2":
        return lambda x: _softplus_legacy(x) ** 2
    if name in _MUL:
        return lambda x: _softplus01(x, *_MUL[name])
    if name in _INV_MUL:
        return lambda x: _inv_softplus01(x, *_INV_MUL[name])
    if name in _SHIFT:
        return lambda x: _shift(x, _SHIFT[name])
    raise NotImplementedError(f"mapper={name}")


def mapper(x, name):
    """get_mapper(name)(x) for any name: a chain of functions and blends, blends late-bound to the last one."""
    stages, blend = [], None
    for part in name.split(":"):
        if "+" in part:
            pair, w = part.split("=")
            w = float(w) if w else 0.5
            assert 0.0 <= w <= 1.0
            a, b = pair.split("+")
            blend = (function(a), function(b), w)
            stages.append(None)
        else:
            stages.append(function(part))
    for f in stages:
        if f is None:
            fa, fb, w = blend
            x = fa(x) * (1 - w) + fb(x) * w
        else:
            x = f(x)
    return x
