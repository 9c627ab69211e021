"""Mirror of iw3/mapper.py: the disparity mappers under the reference's names.

``get_mapper(name)`` parses the name once on the host into an ``nb200_mapper`` descriptor (include/nunif_b200.h) and
returns a callable that evaluates it on the device (csrc/mapper.cuh).  The parse keeps the reference's behaviour:
an unknown name (and ``auto``) raises ``NotImplementedError``, ``a+b`` without ``=`` a ``ValueError``, a weight outside
[0, 1] an ``AssertionError``, an empty weight means 0.5, and every blend stage of a chain uses the functions and
weight of the chain's LAST blend (the reference builds its blend lambdas in a loop, so they all see the loop
variables' final values).  Constants the reference computes from Python floats are computed in double and rounded
to fp32 once; ``inv_softplus01``'s min/max are fp32 tensor values there and are computed the same way here."""
import ctypes
import functools
import math

import numpy as np
import torch

from .. import _lib
from ._common import prep

METRIC_DIV_MAPPER = ["none", "div_25", "div_10", "div_6", "div_4", "div_2", "div_1"]
RELATIVE_MUL_MAPPER = ["inv_mul_3", "inv_mul_2", "inv_mul_1", "none", "mul_1", "mul_2", "mul_3"]
RELATIVE_SHIFT_MAPPER = ["shift_045", "shift_06", "shift_08", "none", "shift_14", "shift_20", "shift_30"]
LEGACY_MAPPER = ["pow2", "softplus", "softplus2"]
MAPPER_ALL = ["auto"] + list(dict.fromkeys(LEGACY_MAPPER + RELATIVE_MUL_MAPPER + METRIC_DIV_MAPPER + RELATIVE_SHIFT_MAPPER))

# function kinds of csrc/mapper.cuh
_NONE, _POW2, _SOFTPLUS, _SOFTPLUS2, _SOFTPLUS01, _INV_SOFTPLUS01, _DIV, _SHIFT = range(8)

# parameters of resolve_mapper_function (iw3/mapper.py:64-120)
_MUL = {"mul_1": (0.343, 12), "mul_2": (0.515, 12), "mul_3": (0.687, 12)}                                   # (bias, scale)
_INV_MUL = {"inv_mul_1": (-0.002102, 7.8788), "inv_mul_2": (-0.0003, 6.2626), "inv_mul_3": (-0.0001, 3.4343)}  # (bias, scale)
_SHIFT_D = {"shift_30": 3.0, "shift_20": 2.0, "shift_14": 1.4, "shift_08": 0.8, "shift_06": 0.6, "shift_045": 0.45}  # min_distance
_DIV_C = {"div_25": 2.5, "div_10": 1, "div_6": 0.6, "div_4": 0.4, "div_2": 0.2, "div_1": 0.1}


def _f32(v):
    return float(np.float32(v))


def _function(name):
    """(kind, constants) of one mapper function; resolve_mapper_function's NotImplementedError for other names."""
    if name == "none":
        return _NONE, ()
    if name == "pow2":
        return _POW2, ()
    if name in ("softplus", "softplus2"):
        # softplus01_legacy, c = 6: the values of log(1 + exp(x * 12 - 6)) / 6 at x = 0 and 1, in double
        lo = math.log(1 + math.exp(-6.0)) / 6
        hi = math.log(1 + math.exp(6.0)) / 6
        return (_SOFTPLUS if name == "softplus" else _SOFTPLUS2), (_f32(lo), _f32(hi - lo))
    if name in _MUL:
        bias, scale = _MUL[name]
        lo = math.log(1 + math.exp((0 - bias) * scale))
        hi = math.log(1 + math.exp((1 - bias) * scale))
        return _SOFTPLUS01, (_f32(bias), _f32(scale), _f32(lo), _f32(hi - lo))
    if name in _INV_MUL:
        bias, scale = _INV_MUL[name]
        ends = ((torch.tensor([0.0, 1.0], dtype=torch.float32) - bias) * scale).expm1().clamp(min=1e-6).log()
        lo, hi = ends[0:1], ends[1:2]
        return _INV_SOFTPLUS01, (_f32(bias), _f32(scale), float(lo), float(hi - lo))
    if name in _DIV_C:
        c = _DIV_C[name]
        c1 = 1.0 + c
        min_v = c / c1
        return _DIV, (_f32(c), _f32(c1), _f32(min_v), _f32(1.0 - min_v))
    if name in _SHIFT_D:
        d = _SHIFT_D[name]
        far = d + 16
        return _SHIFT, (_f32(1.0 / far), _f32(1.0 / d - 1.0 / far), _f32(1.0 - d), _f32(1.0 / 17), _f32(1.0 - 1.0 / 17))
    raise NotImplementedError(f"mapper={name}")


def _parse(name):
    """get_mapper's parse (iw3/mapper.py:129-151): a list of (fn_a, fn_b or None, weight) stages, late-bound blends."""
    stages, last_blend = [], None
    for part in name.split(":"):
        if "+" not in part:
            stages.append((_function(part), None, None))
            continue
        pair, weight = part.split("=")                     # ValueError without (or with more than one) "="
        if weight:
            weight = float(weight)
            if not 0.0 <= weight <= 1.0:
                raise AssertionError(f"mapper={name}: blend weight {weight} is outside [0, 1]")
        else:
            weight = 0.5
        a, b = pair.split("+")                             # ValueError for a+b+c
        last_blend = (_function(a), _function(b), weight)
        stages.append(None)
    return [last_blend if s is None else s for s in stages]


def _fill(fn, spec):
    fn.kind = spec[0]
    for i, v in enumerate(spec[1]):
        fn.k[i] = v


@functools.lru_cache(maxsize=256)
def descriptor(name):
    """The nb200_mapper descriptor of get_mapper(name); identity stages are dropped ("none" is 0 stages)."""
    stages = _parse(name)
    if len(stages) > _lib.MAPPER_MAX_STAGES:
        raise NotImplementedError(f"mapper={name}: a chain of {len(stages)} stages; the engine evaluates at most "
                                  f"{_lib.MAPPER_MAX_STAGES}")
    m = _lib.Mapper()
    n = 0
    for a, b, weight in stages:
        if b is None and a[0] == _NONE:
            continue
        st = m.stage[n]
        _fill(st.a, a)
        if b is not None:
            _fill(st.b, b)
            st.blend, st.one_minus_w, st.w = 1, _f32(1 - weight), _f32(weight)
        n += 1
    m.n_stages = n
    return m


def apply_mapper(x, desc):
    """Evaluate a descriptor on a CUDA tensor; the 0-stage descriptor returns ``x`` itself, like the reference's
    identity."""
    if desc.n_stages == 0:
        return x
    d = prep(x, "depth")
    out = torch.empty_like(d)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().nb200_mapper_apply(_lib.ptr(d), d.numel(), ctypes.byref(desc), _lib.ptr(out), _lib.stream_ptr(d.device)))
    return out


def get_mapper(name):
    """iw3/mapper.py:129-151: a callable x -> mapped x running on the engine (parse errors raise here, as there)."""
    desc = descriptor(name)
    return lambda x: apply_mapper(x, desc)


def get_mapper_levels(metric_depth, mapper_type=None):
    """iw3/mapper.py:174-192: the 7-level ladder for a metric or relative depth model."""
    if metric_depth:
        if mapper_type is None or mapper_type == "div":
            return METRIC_DIV_MAPPER
        raise ValueError(f"{mapper_type} is not metric depth mapper")
    if mapper_type is None or mapper_type == "mul":
        return RELATIVE_MUL_MAPPER
    if mapper_type == "shift":
        return RELATIVE_SHIFT_MAPPER
    raise ValueError(f"{mapper_type} is not relative depth mapper")


def resolve_mapper_name(mapper, foreground_scale, metric_depth, mapper_type=None):
    """iw3/mapper.py:195-232: --mapper / --foreground-scale / --mapper-type -> a mapper name.  An integer scale picks a
    ladder level; a fractional one blends the two levels around it as "a+b=w" with w formatted by round(w, 2)."""
    if mapper is not None:
        if mapper == "auto":
            return "div_6" if metric_depth else "none"
        return mapper
    if float(foreground_scale).is_integer():
        return get_mapper_levels(metric_depth=metric_depth, mapper_type=mapper_type)[int(foreground_scale) + 3]
    sign = 1 if foreground_scale > 0 else -1
    magnitude = foreground_scale if sign > 0 else -foreground_scale
    lo, hi = math.floor(magnitude), math.ceil(magnitude)
    weight = magnitude - lo
    levels = get_mapper_levels(metric_depth=metric_depth, mapper_type=mapper_type)
    return f"{levels[sign * lo + 3]}+{levels[sign * hi + 3]}={round(weight, 2)}"
