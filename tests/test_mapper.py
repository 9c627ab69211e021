"""CPU: the host side of the disparity mappers (nunif_b200/iw3/mapper.py) against tests/golden/mapper.npz, which the
real iw3/mapper.py generated (oracle/gen_golden_mapper.py): resolve_mapper_name string for string, the exception type
of every invalid name, the descriptor's constants, and the torch oracle (oracle/mapper.py) on every name and case."""
import ctypes

import numpy as np
import pytest
import torch

from tests.util import load_golden, t

EXC = {"ValueError": ValueError, "AssertionError": AssertionError, "NotImplementedError": NotImplementedError}


@pytest.fixture(scope="module")
def g():
    return load_golden("mapper")


def _opt(s):
    return None if s == "None" else s


def test_name_lists():
    from nunif_b200.iw3 import mapper as m
    assert m.MAPPER_ALL[0] == "auto" and len(m.MAPPER_ALL) == len(set(m.MAPPER_ALL)) == 23
    assert m.get_mapper_levels(True) is m.METRIC_DIV_MAPPER and m.get_mapper_levels(False) is m.RELATIVE_MUL_MAPPER
    assert m.get_mapper_levels(False, "shift") is m.RELATIVE_SHIFT_MAPPER
    assert m.METRIC_DIV_MAPPER[0] == m.RELATIVE_MUL_MAPPER[3] == m.RELATIVE_SHIFT_MAPPER[3] == "none"
    assert all(len(levels) == 7 for levels in (m.METRIC_DIV_MAPPER, m.RELATIVE_MUL_MAPPER, m.RELATIVE_SHIFT_MAPPER))


def test_names_match_golden(g):
    from nunif_b200.iw3 import MAPPER_ALL
    assert list(g["names"]) == [n for n in MAPPER_ALL if n != "auto"]


def test_resolve_mapper_name_table(g):
    from nunif_b200.iw3 import resolve_mapper_name
    n = 0
    for mapper, scale, metric, mtype, want in zip(g["table_mapper"], g["table_scale"], g["table_metric"], g["table_type"],
                                                  g["table_name"]):
        got = resolve_mapper_name(_opt(str(mapper)), float(scale), bool(metric), _opt(str(mtype)))
        assert got == str(want), (mapper, scale, metric, mtype, got, want)
        n += 1
    assert n > 600
    # round(2.675 - 2, 2): the weight is 0.67499999999999982 in binary, so the name says 0.67
    assert resolve_mapper_name(None, 2.675, False) == "mul_2+mul_3=0.67"


def test_resolve_mapper_name_errors(g):
    from nunif_b200.iw3 import resolve_mapper_name
    for args, want in zip(g["resolve_err_args"], g["resolve_err"]):
        mapper, scale, metric, mtype = (str(a) for a in args)
        scale = float(scale) if "." in scale else int(scale)
        with pytest.raises(EXC[str(want)]):
            resolve_mapper_name(_opt(mapper), scale, metric == "True", _opt(mtype))


def test_get_mapper_parse_errors(g):
    from nunif_b200.iw3 import get_mapper
    for name, want in zip(g["mapper_err_names"], g["mapper_err"]):
        with pytest.raises(EXC[str(want)]) as e:
            get_mapper(str(name))
        assert type(e.value) is EXC[str(want)], (name, type(e.value), want)


def test_chain_stage_limit():
    from nunif_b200.iw3 import get_mapper
    from nunif_b200.iw3.mapper import descriptor
    assert descriptor(":".join(["mul_1"] * 8)).n_stages == 8
    with pytest.raises(NotImplementedError, match="at most 8"):
        get_mapper(":".join(["mul_1"] * 9))


def test_descriptor_layout_and_identity():
    from nunif_b200 import _lib
    from nunif_b200.iw3.mapper import descriptor
    assert ctypes.sizeof(_lib.Mapper) == 528 and ctypes.sizeof(_lib.MapperStage) == 64
    for name in ("none", "none:none", "none:none:none"):
        assert descriptor(name).n_stages == 0
    d = descriptor("mul_1+mul_2=0.5:div_6+div_1=0.25")
    # late binding: both blends are div_6 + div_1 at w = 0.25
    assert d.n_stages == 2
    for s in d.stage[:2]:
        assert s.blend == 1 and s.a.kind == s.b.kind == 6 and s.w == 0.25 and s.one_minus_w == 0.75
        assert s.a.k[0] == np.float32(0.6) and s.b.k[0] == np.float32(0.1)
    assert descriptor("div_2+div_1=").stage[0].w == 0.5


def test_div_constants_match_mapper_c_entries():
    """The descriptor's div_* constants (double from the Python float) are the ones the float mapper_c entries derive
    (double from the fp32 c), so both entry points compute the same bits."""
    from nunif_b200.iw3.mapper import descriptor, _DIV_C
    f32 = np.float32
    for name, c in _DIV_C.items():
        cd = float(f32(c))
        want = [f32(cd), f32(1.0 + cd), f32(cd / (1.0 + cd)), f32(1.0 - cd / (1.0 + cd))]
        k = descriptor(name).stage[0].a.k
        assert [f32(v) for v in k[:4]] == want, name


def _close(got, want, tol):
    d = float((got.double() - t(want).double()).abs().max())
    assert d <= tol, d
    return d


def test_oracle_every_name_and_case(g):
    from oracle.mapper import mapper
    from oracle.iw3 import minmax_normalize
    pts, conv, raw = t(g["pts"]), t(g["conv"]), t(g["raw"])
    for n in g["names"]:
        n = str(n)
        _close(mapper(pts, n), g["pts/" + n], 1e-7)
        _close(mapper(conv, n), g["conv/" + n], 1e-7)
        _close(mapper(minmax_normalize(raw), n), g["mm/" + n], 1e-7)
    for c in g["cases"]:
        _close(mapper(pts, str(c)), g["pts/" + str(c)], 1e-7)
    for i, n in enumerate(g["ladder_names"]):
        _close(mapper(pts[::16], str(n)), g["ladder"][i], 1e-7)


def test_oracle_none_and_div_are_oracle_iw3():
    from oracle import iw3 as oiw
    from oracle.mapper import mapper
    x = torch.rand(2, 1, 9, 13, generator=torch.Generator().manual_seed(4))
    for n in ("none", "div_25", "div_10", "div_6", "div_4", "div_2", "div_1"):
        assert torch.equal(mapper(x, n), oiw.mapper(x, n))
