"""GPU: replay every launch of the forward stereo warp (csrc/warp_forward.cu: nb200_forward_warp, and _conv for a per-frame
convergence), the warp of `forward`, `forward_fill` and `forward_inpaint`, against the oracle and a float64 resize.

The discipline of tests/test_gpu_kernel_replay_warp.py, with the helpers of tests/replay.py: a module fixture turns on bit 4
of the launch recorder and records the production flows of FWARP_FLOWS, and each unique configuration, plus a synthetic list
for the edges production does not reach, is replayed through the C entry point on fresh seeded data.  A configuration with a
resized depth runs with a workspace (the column-table resize when both axes go up) and without one (the generic taps), and
every configuration also with the colour, depth and output pointers one float off 16-byte alignment.  Outputs sit between
guard blocks whose NaN sentinel must survive, the inputs must keep their bits, and the recorder confirms the resize path of
each call.

Debug tap 300 makes the production row kernel write its padded depth row, so the two halves of the warp are checked apart:
  the resize: the tapped interior against F.interpolate(depth, (H, W), bilinear, align_corners=True, antialias=True) in
    float64, within tests/replay.py's aa_resize_reference bound (the same bound as nb200_depth_resize_aa's replay); the
    resize-free path returns the input's bits, and the pads repeat the border cells bit for bit;
  the warp: oracle.iw3.forward_warp on the CPU, given the tapped interior as a full-resolution depth.  The splat's floor()
    and z-order decisions are defined by iw3's fp32 ops, so the oracle, which is pinned to the reference's goldens
    (tests/test_oracle_golden.py), is the specification here, and eyes, masks and SBS halves must equal it bit for bit.
Rows are independent in the warp (each index the reference touches stays inside its row), so a tall configuration compares
the warp on a seeded sample of rows, always with the first two and the last two; the resize and the pads are compared on
every row.
"""
import math
import random

import pytest
import torch

from tests.util import log_metric
from tests.replay import (DEV, GUARD, SENTINEL32, FWARP_FLOWS, Tally, aa_resize_reference, configurations, guarded32,
                          record_networks, recorded, replay)
from nunif_b200 import _lib, synth
from nunif_b200._lib import ptr

pytestmark = pytest.mark.gpu
REC_WARP = 16                  # nb200_record_launches bit of the fwarp kind
TAP_DEPTH = 300                # nb200_debug_tap id of the warp's padded depth rows
TINY = 1e-300                  # bound floor: an exact element has err / bound 0
SECOND_ORDER = 1 + 2.0 ** -20  # the first-order resize bound leaves out products of two roundings
SMEM = 227 * 1024              # the row kernel's shared memory: 7 fp32 rows of Wp cells
ROWS = 64                      # a configuration taller than this compares the warp on this many sampled rows per frame
VIEWS = ("both", "left", "right")

# the launches of each flow of FWARP_FLOWS
EXPECTED = {
    "stereo_sbs_1080p": 1,
    "stereo_anaglyph": 1,
    "forward_views": 18,       # 3 frames x 2 methods x 3 views
    "forward_conv_tensor": 1,
    "forward_inpaint": 1,
    "forward_inpaint_max_width": 1,
    "null_depth": 1,
}


@pytest.fixture(scope="module")
def production():
    """name -> every record (kind, config) of each flow of FWARP_FLOWS (configurations() deduplicates)."""
    return record_networks(REC_WARP, FWARP_FLOWS, unique=False)


def test_every_flow_records_its_launches(production):
    for name, _ in FWARP_FLOWS:
        kinds = [k for k, _ in production[name]]
        log_metric("replay_fwarp_launches", model=name, fwarp=kinds.count("fwarp"))
        assert kinds == ["fwarp"] * EXPECTED[name], (name, kinds)
    recs = lambda name: [r for _, r in production[name]]
    f = lambda name, *fields: [tuple(r[x] for x in fields) for r in recs(name)]
    shape = ("B", "H", "W", "h", "w")
    assert f("stereo_sbs_1080p", *shape, "compose", "fill", "view", "path") == [(4, 1080, 1920, 392, 686, 1, 1, 0, 1)]
    assert f("stereo_sbs_1080p", "P", "Wp", "shift") == [(40, 2000, 19.2000008)]
    assert f("stereo_anaglyph", "compose", "fill", "lmask", "rmask", "path") == [(0, 0, 0, 0, 1)]
    got = sorted(f("forward_views", "H", "W", "view", "fill", "path"))
    want = sorted((H, W, v, fill, path) for H, W, path in ((1080, 1920, 1), (1920, 1080, 1), (240, 320, 2))
                  for v in (0, 1, 2) for fill in (0, 1))
    assert got == want
    assert f("forward_conv_tensor", "B", "conv", "conv_term") == [(4, 1, 0.0)]
    assert f("forward_inpaint", "W", "lmask", "rmask", "fill", "path") == [(1920, 1, 1, 0, 1)]
    assert f("forward_inpaint_max_width", "H", "W", "h", "w", "path") == [(360, 640, 392, 686, 2)]
    assert f("null_depth", "H", "W", "h", "w", "path") == [(512, 512, 512, 512, 0)]


# ------------------------------------------------------------------------------------------------------------ helpers
def f32(v):
    """v rounded to fp32 (a recorded value prints 9 significant digits: this recovers the value the kernel got)."""
    return float(torch.tensor(float(v), dtype=torch.float32))


def buf32(n, off):
    """A guarded fp32 buffer whose body of n elements starts `off` elements after the front guard -> (buffer, body)."""
    b = guarded32(n + off)
    return b, b[GUARD + off:GUARD + off + n]


def untouched(b):
    return bool((b.view(torch.int32) == SENTINEL32).all())


def guards(tally, what, b, n, off):
    """Everything outside the body of buf32(n, off) still holds the sentinel."""
    bits = b.view(torch.int32)
    if not (bool((bits[:GUARD + off] == SENTINEL32).all()) and bool((bits[GUARD + off + n:] == SENTINEL32).all())):
        tally.bad.append(f"{what}: guard changed")


def same_bits(tally, what, got, want):
    tally.exact(what, got.contiguous().view(torch.int32), want.contiguous().view(torch.int32))


def host_args(r):
    """(divergence, convergence) that make the host code, with width_base = 1 (base = W), compute the recorded P and the
    fp32 shift and conv_term: the double arithmetic of forward_warp() and of oracle.iw3.forward_warp, searched a few ulps
    around the quotients."""
    k = 1 if r["view"] == 0 else 2
    W = r["W"]
    host = lambda div: (int(W * (div * k) * 0.01 + 2), (div * k) * 0.01 * W * 0.5)
    div = f32(r["shift"]) / (0.01 * W * 0.5) / k
    for _ in range(8):
        P, s = host(div)
        if (P, f32(s)) == (r["P"], f32(r["shift"])):
            break
        div = math.nextafter(div, math.inf if (P, f32(s)) < (r["P"], f32(r["shift"])) else -math.inf)
    else:
        raise AssertionError(f"no divergence reproduces P={r['P']} shift={r['shift']}")
    if r["conv"]:
        return div, 0.0
    s = host(div)[1]
    cv = f32(r["conv_term"]) / s if s else 0.0
    for _ in range(8):
        if f32(s * cv) == f32(r["conv_term"]):
            break
        cv = math.nextafter(cv, math.inf if (f32(s * cv) < f32(r["conv_term"])) == (s > 0) else -math.inf)
    else:
        raise AssertionError(f"no convergence reproduces conv_term={r['conv_term']}")
    return div, cv


def expected_path(r, ws):
    """The resize path the host code takes: 0 none, 1 the column table (a workspace and both fp32 scales below 1), 2 the
    generic taps."""
    B, H, W, h, w = (r[f] for f in ("B", "H", "W", "h", "w"))
    if (h, w) == (H, W):
        return 0
    sy = f32(f32(h - 1) / f32(H - 1)) if H > 1 else 0.0
    sx = f32(f32(w - 1) / f32(W - 1)) if W > 1 else 0.0
    return 1 if ws and sy < 1 and sx < 1 else 2


def sample_rows(H, seed):
    if H <= ROWS:
        return list(range(H))
    rng = random.Random(seed)
    return sorted({0, 1, H - 2, H - 1} | set(rng.sample(range(2, H - 2), ROWS - 4)))


# ------------------------------------------------------------------------------------------------------------ data
def crafted_depth(craft, B, H, W, g):
    """The full-resolution depth of a crafted configuration (shift 128 and conv_term 0, so depth k / 128 moves a pixel by
    exactly k cells)."""
    d = torch.zeros(B, 1, H, W)
    if craft == "holes":
        # a near object 150 wide moved by 100 (row 0) and 101 cells (row 1): in each eye the hole behind it is 100 or 101
        # cells long, either side of shift_fill's 100-cell cap
        for y, k in enumerate((100, 101)):
            d[:, :, y, 60:210] = k / 128
    elif craft == "layered":
        # one near pixel moved by 120 (row 0), 100 and 101 cells (row 1): the cells it jumps over have a larger index than
        # it has after the move, so fix_layered_holes marks those within 100 cells to its left: the cell whose only smaller
        # index is exactly 100 cells to the right is marked, the one 101 cells away is not
        d[:, :, 0, 40] = d[:, :, 0, 250] = 120 / 128
        d[:, :, 1, 30] = 100 / 128
        d[:, :, 1, 160] = 101 / 128
    elif craft == "integer":
        # integer shifts (floor = ceil: the ceil weight is clamped to 1e-5) mixed with fractional ones
        k = torch.randint(-20, 140, (B, 1, H, W), generator=g).float() / 128
        d = torch.where(torch.rand(B, 1, H, W, generator=g) < 0.5, k, torch.rand(B, 1, H, W, generator=g) * 1.2 - 0.1)
    elif craft == "plateau":
        # runs of 1 to 40 equal depths
        for b in range(B):
            for y in range(H):
                x = 0
                while x < W:
                    n = int(torch.randint(1, 41, (1,), generator=g))
                    d[b, 0, y, x:x + n] = float(torch.rand(1, generator=g)) * 1.5 - 0.25
                    x += n
    elif craft == "signed":
        # both zeros and negative depth: in the even rows the zeros are the deepest values, so with P = 0 they win the
        # clamped end cells, where the sort ties -0.0 with +0.0
        for y, vals in enumerate([torch.tensor([-0.0, 0.0, -0.0, 0.0, -0.3]), torch.tensor([-0.0, 0.0, -0.3, 0.7, 1.0 / 3])] * (H // 2 + 1)):
            if y < H:
                d[:, :, y] = vals[torch.randint(0, len(vals), (B, 1, W), generator=g)]
    else:
        raise ValueError(craft)
    return d


def fwarp_data(r, seed):
    """Seeded inputs: colour in [-0.1, 1.1] (both sides of the clamps), depth in about [-0.25, 1.25] (a smooth map with
    boxes plus noise, or a crafted row), per-frame convergence in [-0.5, 1.5]."""
    B, H, W, h, w = (r[f] for f in ("B", "H", "W", "h", "w"))
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(B, 3, H, W, generator=g) * 1.2 - 0.1
    if r.get("craft"):
        depth = crafted_depth(r["craft"], B, h, w, g)
    else:
        smooth = synth.synth_depth(seed % 100003, B, h, w).nan_to_num(0.5)      # a 1 x 1 map normalises 0 / 0
        depth = (0.8 * smooth + 0.2 * torch.rand(B, 1, h, w, generator=g)) * 1.5 - 0.25
    conv = torch.rand(B, generator=g) * 2 - 0.5
    return dict(c=c, depth=depth, conv=conv, oracle={})


_cache = {}


def cached(seed, make):
    """The inputs and oracle results of one configuration, shared by its variants (replay() runs them one after another)."""
    if seed not in _cache:
        _cache.clear()
        _cache[seed] = make()
    return _cache[seed]


WORST = {}   # resize path -> worst err / bound of the tapped depth


def fwarp_check(r, seed, variant):
    """nb200_forward_warp (or _conv) with `variant` = 10 ws + offset: ws passes a workspace (the column table when both
    axes upsample), offset puts the colour, depth and output pointers one float off 16-byte alignment."""
    from oracle import iw3 as oiw
    B, H, W, h, w, P, Wp = (r[f] for f in ("B", "H", "W", "h", "w", "P", "Wp"))
    view, compose, fill = r["view"], r["compose"], r["fill"]
    ws, off = variant // 10, variant % 10
    data = cached(seed, lambda: fwarp_data(r, seed))
    lib = _lib.lib()
    tally = Tally()
    n, npx = B * 3 * H * W, B * H * W
    cb, c = buf32(n, off)
    c.copy_(data["c"].flatten())
    db, d = buf32(B * h * w, off)
    d.copy_(data["depth"].flatten())
    vb, v = buf32(B, 0)
    v.copy_(data["conv"])
    snap = [cb.clone(), db.clone(), vb.clone()]
    no = 2 * n if compose == 1 else n
    lb, left = buf32(no, off)
    rb, right = buf32(n, off) if compose == 0 else (None, None)
    lmb, lm = buf32(npx, off) if r["lmask"] else (None, None)
    rmb, rm = buf32(npx, off) if r["rmask"] else (None, None)
    tb, tap = buf32(B * H * Wp, 0)
    ws_bytes = lib.nb200_forward_warp_workspace(B, H, W, h, w) if ws else 0
    wb, work = buf32(ws_bytes // 4, 0) if ws_bytes else (None, None)
    divergence, convergence = host_args(r)
    path = expected_path(r, ws)
    want = {f: r[f] for f in ("B", "H", "W", "h", "w", "P", "Wp", "conv", "fill", "view", "compose", "lmask", "rmask")}
    want.update(shift=f32(r["shift"]), conv_term=f32(r["conv_term"]), path=path)

    def call():
        args = (B, H, W, h, w, divergence, ptr(v) if r["conv"] else convergence, fill, view, 1, compose, ptr(left),
                ptr(right) if right is not None else None, ptr(lm) if lm is not None else None,
                ptr(rm) if rm is not None else None, ptr(work) if work is not None else None, _lib.stream_ptr())
        fn = lib.nb200_forward_warp_conv if r["conv"] else lib.nb200_forward_warp
        return fn(ptr(c), ptr(d), *args)

    _lib.check(lib.nb200_debug_tap(TAP_DEPTH, ptr(tap), tap.numel() * 4))
    try:
        if Wp * 7 * 4 > SMEM:
            # refused before any CUDA call: nothing recorded, nothing written
            recs = recorded(REC_WARP, lambda: tally.bad.append("not refused") if call() == 0 else None)
            if b"does not fit shared memory" not in lib.nb200_last_error() or recs:
                tally.bad.append(f"refusal: {lib.nb200_last_error()} {recs}")
            for what, b in (("left", lb), ("right", rb), ("left mask", lmb), ("right mask", rmb), ("tap", tb), ("workspace", wb)):
                if b is None:
                    continue
                if not untouched(b):
                    tally.bad.append(f"{what} written by a refused call")
            return tally.result()
        recs = recorded(REC_WARP, lambda: _lib.check(call()))
    finally:
        lib.nb200_debug_tap(-1, None, 0)
    if len(recs) != 1 or recs[0][0] != "fwarp":
        tally.bad.append(f"recorded {recs}, expected one fwarp")
    else:
        got = recs[0][1]
        for f, x in want.items():
            if (f32(got[f]) != x) if isinstance(x, float) else got[f] != x:
                tally.bad.append(f"fwarp recorded {f}={got[f]}, expected {x}")
    for what, b, s in (("c", cb, snap[0]), ("depth", db, snap[1]), ("convergence", vb, snap[2])):
        tally.exact(what, b.view(torch.int32), s.view(torch.int32))
    for what, b, m, o in (("left", lb, no, off), ("right", rb, n, off), ("left mask", lmb, npx, off),
                          ("right mask", rmb, npx, off), ("tap", tb, B * H * Wp, 0), ("workspace", wb, ws_bytes // 4, 0)):
        if b is not None:
            guards(tally, what, b, m, o)
    tally.no_nan("tap", tap)
    if tally.bad:
        return tally.result()

    # ---- the resize, every row
    tap = tap.view(B, 1, H, Wp)
    dep = tap[..., P:P + W]
    same_bits(tally, "left pad", tap[..., :P], dep[..., :1].expand(B, 1, H, P))
    same_bits(tally, "right pad", tap[..., P + W:], dep[..., W - 1:].expand(B, 1, H, P))
    if path == 0:
        same_bits(tally, "resize-free depth", dep, d.view(B, 1, H, W))
    else:
        ref, bound = aa_resize_reference(d.view(B, 1, h, w).double(), H, W)
        before = tally.worst
        tally.worst = 0.0
        tally.add(dep, ref, SECOND_ORDER * bound + TINY)
        WORST[path] = max(WORST.get(path, 0.0), tally.worst)
        tally.worst = max(tally.worst, before)

    # ---- the warp on the sampled rows, against the oracle on the tapped depth
    rows = sample_rows(H, seed)
    ri = torch.tensor(rows, device=DEV)
    dep_rows = dep[:, :, ri].cpu()
    key = dep_rows.numpy().tobytes()
    if key not in data["oracle"]:
        cv = data["conv"].view(B, 1, 1, 1) if r["conv"] else convergence
        data["oracle"][key] = oiw.forward_warp(data["c"][:, :, rows].contiguous(), dep_rows, divergence, cv, fill=bool(fill),
                                               synthetic_view=VIEWS[view], return_mask=True, width_base=True)
    ol, orr, olm, orm = (t.to(DEV) if t is not None else None for t in data["oracle"][key])
    src = data["c"].to(DEV)
    if compose == 1:
        sbs = left.view(B, 3, H, 2 * W)
        tally.no_nan("SBS", sbs)
        same_bits(tally, "SBS", sbs[:, :, ri], torch.clamp(torch.cat([ol, orr], 3), 0, 1))
        if view != 0:
            half = sbs[..., W:] if view == 1 else sbs[..., :W]
            same_bits(tally, "SBS source half", half, torch.clamp(src, 0, 1))
    else:
        for what, got, ref, synthesised in (("left", left, ol, view != 2), ("right", right, orr, view != 1)):
            got = got.view(B, 3, H, W)
            tally.no_nan(what, got)
            if synthesised:
                same_bits(tally, what, got[:, :, ri], ref)
            else:
                same_bits(tally, f"{what} (the source)", got, src)
    for what, got, ref, synthesised in (("left mask", lm, olm, view != 2), ("right mask", rm, orm, view != 1)):
        if got is None:
            continue
        if not synthesised:
            if not untouched(got):
                tally.bad.append(f"{what} written for the source eye")
            continue
        got = got.view(B, 1, H, W)
        tally.no_nan(what, got)
        same_bits(tally, what, got[:, :, ri], ref)
    return tally.result()


# ------------------------------------------------------------------------------------------------------------ synthetic
def _fwarp(B, H, W, h, w, div=10.0, convergence=0.5, view=0, fill=1, compose=0, conv=0, lmask=None, rmask=None, craft=None):
    """A synthetic configuration with the host's fields for width_base = 1 (base = W); the masks default to production's
    choice (one per synthesised eye, none in an SBS frame)."""
    k = 1 if view == 0 else 2
    P = int(W * (div * k) * 0.01 + 2)
    s = (div * k) * 0.01 * W * 0.5
    r = dict(B=B, H=H, W=W, h=h, w=w, P=P, Wp=W + 2 * P, shift=f32(s), conv_term=0.0 if conv else f32(s * convergence),
             conv=conv, fill=fill, view=view, compose=compose,
             lmask=int(compose == 0 and view != 2) if lmask is None else lmask,
             rmask=int(compose == 0 and view != 1) if rmask is None else rmask)
    if craft:
        r["craft"] = craft
    return r


def _fwarp_synthetic():
    out = []
    for W in (1, 2, 3, 36, 37, 38, 63, 64, 65, 99, 100, 101, 257):
        out += [_fwarp(1, 1, W, 1, W), _fwarp(1, 1, W, 1, 7), _fwarp(1, 1, W, 5, 1, fill=0)]
    out += [_fwarp(1, 9, 50, 9, 20),                 # h = H, w != W: the generic taps even with a workspace
            _fwarp(1, 20, 40, 30, 15),               # rows down, columns up
            _fwarp(1, 30, 15, 20, 40),               # rows up, columns down
            _fwarp(1, 6, 13, 64, 200),               # downsampling by a large factor
            _fwarp(2, 17, 60, 2, 25),                # upsampling from 2 rows
            _fwarp(1, 9, 11, 23, 31, view=1)]        # depth larger than the frame
    # either side of 227 KB at 28 B per padded cell: Wp = 8301 runs, 8302 is refused; both axes upsample, so with a
    # workspace the column table is the path, and the refusal must come before its launch
    out += [_fwarp(1, 3, 8001, 2, 3000, div=1.85), _fwarp(1, 3, 8002, 2, 3000, div=1.85)]
    # P = 0 (the clamped end cells are visible) and P = 1
    out += [_fwarp(1, 6, 100, 6, 100, div=-1.5, convergence=-20.0), _fwarp(1, 6, 100, 4, 37, div=-1.5, convergence=30.0),
            _fwarp(1, 6, 100, 6, 100, div=-0.5, convergence=-80.0)]
    # negative and > 1 convergence, also per frame; views and SBS
    out += [_fwarp(1, 12, 50, 7, 19, convergence=-0.5), _fwarp(1, 12, 50, 7, 19, convergence=1.5),
            _fwarp(3, 12, 50, 7, 19, conv=1), _fwarp(3, 10, 24, 6, 13, view=2, conv=1, fill=0)]
    out += [_fwarp(2, 10, 24, 6, 13, view=v, compose=cm, lmask=1, rmask=1) for v in (1, 2) for cm in (0, 1)]
    out += [_fwarp(2, 10, 24, 6, 13, compose=1, fill=0)]
    return out


def _fwarp_crafted():
    # shift 128 (div 85.33 at W = 300) and convergence 0: depth k / 128 moves a pixel by exactly k cells
    div = 128 / (0.01 * 300 * 0.5)
    out = [_fwarp(1, 2, 300, 2, 300, div=div, convergence=0.0, fill=f, craft="holes") for f in (1, 0)]
    out += [_fwarp(1, 2, 300, 2, 300, div=div, convergence=0.0, craft="layered")]
    out += [_fwarp(2, 4, 257, 4, 257, div=div, convergence=0.0, craft="integer")]
    out += [_fwarp(1, 4, 300, 4, 300, div=5.0, craft="plateau"), _fwarp(1, 4, 300, 4, 300, div=-0.5, convergence=-20.0, craft="plateau")]
    # both zeros: with P = 0 many equal keys clamp into the visible end cells, where the largest source index wins
    out += [_fwarp(1, 6, 100, 6, 100, div=-1.5, convergence=c, craft="signed") for c in (-60.0, 60.0)]
    out += [_fwarp(1, 6, 100, 6, 100, div=-0.5, convergence=60.0, craft="signed"), _fwarp(1, 6, 100, 6, 100, craft="signed")]
    out += [_fwarp(1, 6, 100, 6, 100, div=-1.5, convergence=c, craft="plateau") for c in (-60.0, 60.0)]
    return out


VARIANTS = (0, 1, 10, 11)


def _report(kind):
    for path, worst in sorted(WORST.items()):
        print(f"{kind}: resize path {path} worst err/bound {worst:.3g}")
        log_metric(f"replay_{kind}_resize", path=path, worst=worst)
    WORST.clear()
    _cache.clear()


def test_forward_warp_replay(production):
    cases = configurations(production, "fwarp", _fwarp_synthetic())
    assert any(r["P"] == 0 for _, r in cases) and any(r["P"] == 1 for _, r in cases)
    assert {r["Wp"] for _, r in cases} >= {8301, 8302}
    replay("fwarp", cases, fwarp_check, variant=("ws_offset", VARIANTS))
    _report("fwarp")


def test_forward_warp_crafted_rows_replay():
    cases = configurations({}, "fwarp", _fwarp_crafted())
    replay("fwarp_crafted", cases, fwarp_check, variant=("ws_offset", (0, 1)))
    _report("fwarp_crafted")
