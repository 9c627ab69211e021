"""GPU: replay every launch that the engine's networks make of the wgmma implicit GEMM (gemm_conv_kernel), the ViT flash
attention (flash_attention_kernel) and the fused Swin block (swin_attn_fused_kernel, swin_mlp_fused_kernel), at their production
shapes, against float64 references.

A module fixture turns the library's launch recorder on (nb200_record_launches) and runs one forward of each network of
MODELS.  Each unique recorded configuration is then replayed through a low-level entry point on fresh seeded data:
  * guards: input elements outside the view the launch describes are fp16 NaN, output elements outside the view it writes
    hold a sentinel bit pattern (also a NaN), and a guard block sits before and after every buffer.  A replay passes only
    if its output holds no NaN and every guard element is bit-identical after the call;
  * the reference is float64, written from the semantics of gemm.h / gemm_wgmma.cuh / the kernels' comments (per-tap shifted
    slices, not the kernels' tensor-map views), and each element is checked against an error bound derived from the
    kernel's arithmetic (see the bound helpers).
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from tests.replay import (DEV, GUARD, MODELS, Tally, bits, body, configurations, extent, gelu64, guarded, mlp_reference, record_networks,
                          recorded, replay, swin_attn_check, ulp16, view)
from nunif_b200 import _lib

pytestmark = pytest.mark.gpu
LOG2E = math.log2(math.e)
CHUNK_BYTES = 2 << 30        # float64 working set of one reference chunk
REC_GEMMS = 1                # nb200_record_launches bit of the kinds replayed here
KINDS = ("gemm", "attn", "swin_attn", "swin_mlp")
DESC_FIELDS = [f for f, _ in _lib.GemmDesc._fields_]
# every instantiation gemm.cu launch_bn can select: (BLOCK_N, BK, A2)
INSTANTIATIONS = {(bn, bk, 0) for bn in (16, 32, 48, 64, 96, 128) for bk in (32, 64)} | {(bn, bk, 1) for bn in (64, 96) for bk in (32, 64)}


@pytest.fixture(scope="module")
def production():
    """name -> unique records (kind, config) of one forward of each network of MODELS."""
    return record_networks(REC_GEMMS, MODELS)


def test_every_network_records_its_launches(production):
    lines = []
    for name, _ in MODELS:
        recs = production[name]
        counts = {k: sum(1 for kk, _ in recs if kk == k) for k in KINDS}
        inst = sorted({(r["block_n"], r["bk"], r["has_a2"]) for k, r in recs if k == "gemm"})
        lines.append(f"{name:22s} unique: gemm {counts['gemm']:3d} attn {counts['attn']:2d} swin_attn {counts['swin_attn']:2d} "
                     f"swin_mlp {counts['swin_mlp']:2d}   (BLOCK_N, BK, A2): {inst}")
        log_metric("replay_configs", model=name, **counts)
        assert counts["gemm"] > 0, f"{name}: no implicit-GEMM launch was recorded"
    print("\n" + "\n".join(lines))
    for name in ("depth_anything_v2_s", "depth_anything_v2_l", "zoed_n", "zoed_any_n"):
        assert any(k == "attn" for k, _ in production[name]), name
    for name in ("swin_unet_4x", "swin_unet_2x", "swin_unet_1x"):
        assert any(k == "swin_attn" for k, _ in production[name]) and any(k == "swin_mlp" and r["cs"] > 0 for k, r in production[name]), name


# ------------------------------------------------------------------------------------------------------------ helpers
def fill_normal(v, g, std=1.0):
    v.copy_((torch.randn(v.shape, generator=g, device=DEV) * std).to(v.dtype))


ACT = {0: lambda v: v, 1: lambda v: torch.where(v > 0, v, 0.1 * v), 2: gelu64, 3: lambda v: v.clamp_min(0.0)}


# ------------------------------------------------------------------------------------------------------------ GEMM replay
def _gemm_cfg(**kw):
    """A launch's ConvGemm fields (nb200_gemm_desc) and its recorded flags; what is not given is 0 (dil, a_planes 1, a bias)."""
    r = dict.fromkeys(DESC_FIELDS, 0)
    r.update(dil=1, a_planes=1, has_bias=1, has_res=0, has_a2=0, out_is_res=0, out_is_a=0)
    r.update(kw)
    return r


def _synthetic_gemm():
    """Small launches that, with the production ones, reach every instantiation launch_bn can select, plus the ConvGemm
    paths a production shape exercises only at one size."""
    big = 148 * 128   # enough 128-row tiles that the small-M narrowing keeps the widest BLOCK_N
    out = []
    for N in (16, 32, 48, 64, 96, 128):
        for Cin in (32, 64):
            out.append(_gemm_cfg(kind=0, B=1, Hi=1, Wi=big + 77, Ci=Cin + 8, Cin=Cin, N=N, ldo=N + 16, act=1))
    for cout, Cin, Cin2 in ((64, 64, 64), (64, 96, 32), (96, 128, 64), (96, 64, 96)):
        out.append(_gemm_cfg(kind=1, B=2, Hi=21, Wi=19, Ci=Cin, Cin=Cin, N=4 * cout, ldo=cout, out_mode=1, cout=cout, act=1,
                             has_a2=1, Cin2=Cin2, ld2=Cin2 + 32))
    # TCONV3 with a dilation that spans most of a short window, a channel slice and ldo > N
    out.append(_gemm_cfg(kind=5, dil=3, B=2, Hi=7, Wi=45, Ci=96, Cin=32, N=64, ldo=128, act=3))
    # residual before the activation, cropped residual, cropped A view
    out.append(_gemm_cfg(kind=2, pad=0, B=2, Hi=19, Wi=37, Ci=64, Cin=64, a_row_stride=41 * 64, a_img_stride=23 * 41 * 64, N=64,
                         ldo=64, act=2, has_res=1, ldr=72, res_H=21, res_W=39, res_cy=2, res_cx=3, res_before_act=1))
    out.append(_gemm_cfg(kind=2, pad=1, B=3, Hi=13, Wi=29, Ci=32, Cin=32, N=48, ldo=48, act=1, has_res=1, ldr=48, res_H=13,
                         res_W=29, res_before_act=0))
    out.append(_gemm_cfg(kind=0, B=1, Hi=1, Wi=3001, Ci=64, Cin=64, N=192, ldo=64, out_mode=2, cout=64, split_stride=3001 * 64 + 8))
    out.append(_gemm_cfg(kind=0, B=1, Hi=1, Wi=2000, Ci=64, Cin=64, a_planes=3, a_plane_stride=2000 * 64 + 24, N=96, ldo=96))
    return out


class GemmCase:
    """Buffers of one replayed launch, laid out from its record with the same strides and aliasing."""

    def __init__(self, r, seed):
        self.r = r
        g = torch.Generator(device=DEV).manual_seed(seed)
        kind = r["kind"]
        B, Hi, Wi, Ci, Cin = r["B"], r["Hi"], r["Wi"], r["Ci"], r["Cin"]
        if kind == 0:
            self.B, self.Ho, self.Wo = 1, 1, B * Hi * Wi
            self.taps, ktap = r["a_planes"], Cin
            M = self.Wo
            ps = r["a_plane_stride"] if r["a_planes"] > 1 else M * Ci
            self.a_shape, self.a_strides = (r["a_planes"], M, Cin), (ps, Ci, 1)
        else:
            rs = r["a_row_stride"] or Wi * Ci
            ims = r["a_img_stride"] or Hi * rs
            self.a_shape, self.a_strides = (B, Hi, Wi, Cin), (ims, rs, Ci, 1)
            self.B = B
            if kind == 1:
                self.Ho, self.Wo, self.taps, ktap = Hi, Wi, 1, Cin
            elif kind == 2:
                p = r["pad"]
                self.Ho, self.Wo, self.taps, ktap = Hi - 2 + 2 * p, Wi - 2 + 2 * p, 9, Cin
            elif kind == 5:
                self.Ho, self.Wo, self.taps, ktap = Hi, Wi, 3, Cin
            elif kind == 3:
                self.Ho, self.Wo, self.taps, ktap = Hi // 2, Wi // 2, 2, 2 * Cin
            else:
                raise AssertionError(f"unknown kind {kind}")
        N, ldo, mode, cout = r["N"], r["ldo"], r["out_mode"], r["cout"]
        Bo, Ho, Wo = self.B, self.Ho, self.Wo
        self.K = self.taps * ktap + r["Cin2"]
        # output view (B, Ho, Wo, g1, g2, cg): n = (g1 * g2dim + g2) * cg + c
        if mode == 0:
            self.o_shape, self.o_strides = (Bo, Ho, Wo, 1, 1, N), (Ho * Wo * ldo, Wo * ldo, ldo, 1, 1, 1)
        elif mode == 2:
            self.o_shape = (Bo, Ho, Wo, N // cout, 1, cout)
            self.o_strides = (Ho * Wo * ldo, Wo * ldo, ldo, r["split_stride"], 1, 1)
        else:
            self.o_shape, self.o_strides = (Bo, Ho, Wo, 2, 2, cout), (4 * Ho * Wo * ldo, 4 * Wo * ldo, 2 * ldo, 2 * Wo * ldo, ldo, 1)
        o_ext = extent(self.o_shape, self.o_strides)
        if mode == 1:
            o_ext = max(o_ext, Bo * 4 * Ho * Wo * ldo)
        # residual view, read at (y + res_cy, x + res_cx) of [B][res_H][res_W][ldr] (the whole M row for kind 0)
        self.res = None
        if r["has_res"]:
            rH, rW, cy, cx, ldr = r["res_H"], r["res_W"], r["res_cy"], r["res_cx"], r["ldr"]
            if kind == 0:
                rH, rW, cy, cx = 1, Wo, 0, 0
            if mode == 1:
                shp, st = (Bo, Ho, Wo, 2, 2, cout), (rH * rW * ldr, 2 * rW * ldr, 2 * ldr, rW * ldr, ldr, 1)
                assert cy + 1 + 2 * (Ho - 1) < rH and cx + 1 + 2 * (Wo - 1) < rW, r
            else:
                shp, st = (Bo, Ho, Wo, 1, 1, N), (rH * rW * ldr, rW * ldr, ldr, 1, 1, 1)
                assert cy + Ho <= rH and cx + Wo <= rW, f"residual view outside the residual tensor: {r}"
            self.r_shape, self.r_strides, self.r_off = shp, st, (cy * rW + cx) * ldr
            r_ext = max(Bo * rH * rW * ldr, extent(shp, st, self.r_off))
        a_ext = extent(self.a_shape, self.a_strides)
        # buffers: aliasing as recorded
        if r["out_is_a"]:
            self.out = guarded(max(o_ext, a_ext))
            self.a = self.out
        else:
            self.out = guarded(o_ext)
            self.a = guarded(a_ext)
        fill_normal(view(self.a, self.a_shape, self.a_strides), g)
        self.a_ref = view(self.a, self.a_shape, self.a_strides).clone()
        if r["has_res"]:
            self.res = self.out if r["out_is_res"] else guarded(r_ext)
            if r["out_is_res"]:
                assert self.r_off == 0 and self.r_strides == self.o_strides, f"in-place residual with a different view: {r}"
            fill_normal(view(self.res, self.r_shape, self.r_strides, self.r_off), g)
            self.res_ref = view(self.res, self.r_shape, self.r_strides, self.r_off).clone()
        self.a2 = None
        if r["has_a2"]:
            ld2, C2 = r["ld2"], r["Cin2"]
            self.a2_shape = (Bo, Ho, Wo, 2, 2, C2)
            self.a2_strides = (4 * Ho * Wo * ld2, 4 * Wo * ld2, 2 * ld2, 2 * Wo * ld2, ld2, 1)
            self.a2 = guarded(Bo * 4 * Ho * Wo * ld2)
            fill_normal(view(self.a2, self.a2_shape, self.a2_strides), g)
        self.W = (torch.randn(N, self.K, generator=g, device=DEV) / math.sqrt(self.K)).half()
        self.bias = 0.5 * torch.randn(N, generator=g, device=DEV) if r["has_bias"] else None
        self.snap = {id(t): t.clone() for t in {id(x): x for x in (self.a, self.out, self.res, self.a2) if x is not None}.values()}

    def launch(self):
        r = self.r
        d = _lib.GemmDesc(**{f: r[f] for f in DESC_FIELDS})
        p = lambda t: _lib.ptr(t) if t is None else ctypes.c_void_p(t.data_ptr() + 2 * GUARD)
        _lib.check(_lib.lib().nb200_conv_gemm_ex_f16(ctypes.byref(d), p(self.a), _lib.ptr(self.W), _lib.ptr(self.bias), p(self.out),
                                                     p(self.res), p(self.a2), _lib.stream_ptr()))
        torch.cuda.synchronize()

    def check_guards(self, tally):
        """Problems: NaN in the output view, guard / unviewed elements changed."""
        written = torch.zeros(self.out.numel(), dtype=torch.bool, device=DEV)
        view(written, self.o_shape, self.o_strides).fill_(True)
        for buf in {id(x): x for x in (self.a, self.out, self.res, self.a2) if x is not None}.values():
            keep = ~written if buf is self.out else torch.ones_like(written[:1]).expand(buf.numel())
            changed = (bits(buf) != bits(self.snap[id(buf)])) & keep
            if bool(changed.any()):
                i = int(changed.nonzero()[0]) - GUARD
                tally.bad.append(f"element {i} outside the written view changed (buffer of {buf.numel() - 2 * GUARD})")
        tally.no_nan("the output", view(self.out, self.o_shape, self.o_strides))

    def _tap_slices(self, a16, y0, y1):
        """(float64 [rows, Cin] slice, first K column) per tap for output rows [y0, y1) of the images in a16."""
        r, kind, Cin = self.r, self.r["kind"], self.r["Cin"]
        Wo = self.Wo
        if kind == 1:
            yield a16[:, y0:y1], 0
        elif kind == 2:
            for t in range(9):
                ky, kx = divmod(t, 3)
                yield a16[:, y0 + ky:y1 + ky, kx:kx + Wo], t * Cin
        elif kind == 5:
            d = r["dil"]
            for t in range(3):
                yield a16[:, y0 + t * d:y1 + t * d], t * Cin
        elif kind == 3:
            for t in range(4):
                dy, dx = divmod(t, 2)
                yield a16[:, 2 * y0 + dy:2 * y1:2, dx::2], t * Cin

    def reference_chunks(self):
        """-> iterator of (index into the [B, Ho, Wo, N] output, float64 pre-epilogue accumulator, float64 sum |a w|)."""
        r, kind, N = self.r, self.r["kind"], self.r["N"]
        W = self.W.double()
        Wa = W.abs()
        if kind == 0:
            A = self.a_ref
            M = A.shape[1]
            rows = max(1, CHUNK_BYTES // (8 * 4 * (N + A.shape[2])))
            for m0 in range(0, M, rows):
                m1 = min(M, m0 + rows)
                acc = torch.zeros(m1 - m0, N, dtype=torch.float64, device=DEV)
                sab = torch.zeros_like(acc)
                for p in range(A.shape[0]):
                    x = A[p, m0:m1].double()
                    w = W[:, p * r["Cin"]:(p + 1) * r["Cin"]]
                    acc += x @ w.t()
                    sab += x.abs() @ Wa[:, p * r["Cin"]:(p + 1) * r["Cin"]].t()
                yield (0, 0, slice(m0, m1)), acc.view(1, 1, m1 - m0, N), sab.view(1, 1, m1 - m0, N)
            return
        Cin = r["Cin"]
        per_row = self.Wo * 8 * 4 * (N + 2 * Cin + r["Cin2"])
        rows = max(1, CHUNK_BYTES // per_row)
        for b in range(self.B):
            a16 = self.a_ref[b:b + 1]
            if kind == 2 and r["pad"]:
                a16 = F.pad(a16, (0, 0, 1, 1, 1, 1))
            elif kind == 5:
                d = r["dil"]
                a16 = F.pad(a16, (0, 0, 0, 0, d, d))
            for y0 in range(0, self.Ho, rows):
                y1 = min(self.Ho, y0 + rows)
                acc = torch.zeros((y1 - y0) * self.Wo, N, dtype=torch.float64, device=DEV)
                sab = torch.zeros_like(acc)
                for x, k0 in self._tap_slices(a16, y0, y1):
                    kw = x.shape[-1]
                    x = x.double().reshape(-1, kw)
                    acc += x @ W[:, k0:k0 + kw].t()
                    sab += x.abs() @ Wa[:, k0:k0 + kw].t()
                if self.a2 is not None:
                    C2, cout, k2 = r["Cin2"], r["cout"], self.K - r["Cin2"]
                    a2 = view(self.a2, self.a2_shape, self.a2_strides)[b:b + 1, y0:y1]
                    for q in range(4):
                        x = a2[:, :, :, q // 2, q % 2].double().reshape(-1, C2)
                        cols = slice(q * cout, (q + 1) * cout)
                        acc[:, cols] += x @ W[cols, k2:].t()
                        sab[:, cols] += x.abs() @ Wa[cols, k2:].t()
                shp = (1, y1 - y0, self.Wo, N)
                yield (slice(b, b + 1), slice(y0, y1), slice(None)), acc.view(shp), sab.view(shp)

    def check(self, tally):
        """Every output element against the float64 reference."""
        r = self.r
        act = r["act"]
        L = 1.13 if act == 2 else 1.0
        got_all = view(self.out, self.o_shape, self.o_strides)
        res_all = self.res_ref if self.res is not None else None
        for idx, acc, sab in self.reference_chunks():
            v = acc + (self.bias.double() if self.bias is not None else 0.0)
            if res_all is not None:
                rv = res_all[idx].double().reshape(v.shape)
                v = ACT[act](v + rv) if r["res_before_act"] else ACT[act](v) + rv
            else:
                v = ACT[act](v)
            tally.add(got_all[idx].reshape(v.shape), v, ulp16(v) + 2.0 ** -20 * L * sab + (1e-6 if act == 2 else 0.0))


def gemm_check(r, seed):
    case = GemmCase(r, seed)
    case.launch()
    tally = Tally()
    case.check_guards(tally)
    case.check(tally)
    return tally.result()


def test_gemm_instantiation_coverage(production):
    """Every (BLOCK_N, BK, A2) instantiation gemm.cu can select is reached by a recorded launch or a synthetic one."""
    have = {(r["block_n"], r["bk"], r["has_a2"]) for recs in production.values() for k, r in recs if k == "gemm"}
    rows = []
    for r in _synthetic_gemm():
        case = GemmCase(r, 1)
        recs = recorded(REC_GEMMS, case.launch)
        rows.append((recs[0][1]["block_n"], recs[0][1]["bk"], recs[0][1]["has_a2"]))
    table = {i: ("recorded" if i in have else ("synthetic" if i in rows else "MISSING")) for i in sorted(INSTANTIATIONS)}
    print("\n" + "\n".join(f"BLOCK_N {bn:3d} BK {bk} A2 {a2}: {src}" for (bn, bk, a2), src in table.items()))
    assert (have | set(rows)) >= INSTANTIATIONS, [i for i, s in table.items() if s == "MISSING"]
    assert (have | set(rows)) <= INSTANTIATIONS


def test_gemm_replay(production):
    replay("gemm", configurations(production, "gemm", _synthetic_gemm()), gemm_check)


# ------------------------------------------------------------------------------------------------------------ flash attention
SYNTH_ATTN = [dict(B=B, N=N, heads=h, has_bias=bias, ldb=(-(-N // 64) * 64 + (64 if bias and N % 2 else 0)) if bias else 0)
              for N in (1, 2, 63, 64, 65, 127, 128, 129) for h in (6, 16) for B in (1, 3) for bias in (0, 1)]


def _needle_targets(N):
    tail0 = (N - 1) // 64 * 64
    return sorted({t for t in (0, 63, 64, tail0, N - 1) if 0 <= t < N})


def attention_case(r, needle, seed):
    """-> (qkv fp16 [B][N][3][heads][64], bias fp32 [heads][N][ldb] or None, chosen key per row or None)."""
    g = torch.Generator().manual_seed(seed)
    B, N, H, ldb = r["B"], r["N"], r["heads"], r["ldb"]
    qkv = torch.randn(B, N, 3, H, 64, generator=g)
    bias = None
    targets = None
    if not needle:
        qkv[:, :, :2] *= 3 ** 0.5                       # q.k / 8 has a standard deviation of 3
        if r["has_bias"]:
            bias = torch.randn(H, N, ldb, generator=g) * LOG2E
    else:
        tk = _needle_targets(N)
        targets = torch.tensor([tk[i % len(tk)] for i in range(N)])
        if r["has_bias"]:
            # the bias makes the needle, at a column other than the row (a transposed index moves the output by O(1))
            for i in range(N):
                if targets[i] == i and len(tk) > 1:
                    targets[i] = tk[(i + 1) % len(tk)]
            qkv[:, :, :2] *= 0.7                        # scores of standard deviation 0.5 around the needle
            bias = torch.randn(H, N, ldb, generator=g) * 0.5
            bias[:, torch.arange(N), targets] = 14.0
            bias *= LOG2E
        else:
            # key t_j points along dimension j; each query points at its key
            qkv[:, :, :2] *= 0.3
            for j, t in enumerate(tk):
                qkv[:, t, 1, :, :] = 0.0
                qkv[:, t, 1, :, j] = 16.0
            for i in range(N):
                qkv[:, i, 0, :, tk.index(int(targets[i]))] += 8.0
    if bias is not None:
        bias[:, :, N:] = 1e4 * LOG2E                    # an unmasked tail column would take the whole softmax
        bias = bias.float().to(DEV)
    return qkv.half().to(DEV), bias, targets


def attention_check(r, seed, needle):
    """Bound per element: 2^-9 sum_j p_j |v_j| covers the fp16 rounding of P before PV (2^-11 relative), its mismatch with
    the fp32 row sum and ex2.approx.  Where P is below 2^-14 its fp16 value is subnormal and the rounding is absolute, up to
    2^-25 of the running maximum (which is 1 before the row sum l >= 1 divides): 2^-25 sum_j |v_j| / l = 2^-25 max_j p_j
    sum_j |v_j|.  A needle row puts its tiny P on every other key, so this term matters there."""
    B, N, H, ldb = r["B"], r["N"], r["heads"], r["ldb"]
    qkv, bias, targets = attention_case(r, needle, seed)
    dim = H * 64
    out = guarded(B * N * dim + 64 * dim)
    _lib.check(_lib.lib().nb200_flash_attention_f16(_lib.ptr(qkv), ctypes.c_void_p(out.data_ptr() + 2 * GUARD), B, N, H,
                                                    _lib.ptr(bias), ldb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = view(out, (B, N, H, 64), (N * dim, dim, 64, 1))
    tally.no_nan("the output", got)
    tally.guards("output", out, B * N * dim)
    for b in range(B):
        q, k, v = (qkv[b, :, i].double().permute(1, 0, 2) for i in range(3))   # [H][N][64]
        s = q @ k.transpose(1, 2) / 8.0
        if bias is not None:
            s = s + bias[:, :, :N].double() / LOG2E
        p = torch.softmax(s, dim=-1)
        if targets is not None:
            mass = p[:, torch.arange(N, device=DEV), targets.to(DEV)]
            assert float(mass.min()) >= 0.9, float(mass.min())
        ref = p @ v
        bound = 2.0 ** -9 * (p @ v.abs()) + 2.0 ** -25 * p.amax(-1, keepdim=True) * v.abs().sum(1, keepdim=True) + ulp16(ref)
        tally.add(got[b].permute(1, 0, 2), ref, bound)
    return tally.result()


def test_flash_attention_replay(production):
    replay("attn", configurations(production, "attn", SYNTH_ATTN), attention_check, variant=("needle", (False, True)))


# ------------------------------------------------------------------------------------------------------------ Swin head
SYNTH_SWIN_ATTN = [dict(B=1, H=6, W=6, C=192, shift=3), dict(B=3, H=18, W=30, C=96, shift=3), dict(B=2, H=24, W=12, C=192, shift=3),
                   dict(B=5, H=12, W=12, C=192, shift=0)]


def test_swin_attn_replay(production):
    replay("swin_attn", configurations(production, "swin_attn", SYNTH_SWIN_ATTN), swin_attn_check)


# ------------------------------------------------------------------------------------------------------------ Swin tail
SYNTH_SWIN_MLP = [dict(T=16 * 240 * 240, C=192, proj=1, cs=48),      # the 4x model's last block at tile 256, batch 16
                  dict(T=148 * 128 * 3 + 55, C=192, proj=1, cs=48), dict(T=148 * 128 * 2 + 1, C=96, proj=1, cs=16),
                  dict(T=148 * 128 + 127, C=192, proj=1, cs=0), dict(T=777, C=96, proj=0, cs=0)]


def swin_mlp_check(r, seed):
    T, C, proj, cs = r["T"], r["C"], r["proj"], r["cs"]
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=DEV)
    xb = guarded(T * C)
    x = xb[GUARD:GUARD + T * C].view(T, C)
    x.copy_(rn(T, C).half())
    att = rn(T, C).half() if proj else None
    wp = (rn(C, C) / C ** 0.5).half()
    bp = 0.1 * rn(C)
    w1 = (rn(2 * C, C) / C ** 0.5).half()
    b1 = 0.1 * rn(2 * C)
    w2 = (rn(C, 2 * C) / (2 * C) ** 0.5).half()
    b2 = 0.1 * rn(C)
    wy = (rn(cs, C) / C ** 0.5).half() if cs else None
    by = rn(cs) if cs else None          # O(1), so a lost bias is an O(1) error
    x0 = xb.clone()
    lib = _lib.lib()
    xp = ctypes.c_void_p(xb.data_ptr() + 2 * GUARD)
    if cs:
        yb = guarded(T * cs)
        _lib.check(lib.nb200_swin_mlp_fused_y_f16(xp, _lib.ptr(att), T, C, _lib.ptr(wp), _lib.ptr(bp), _lib.ptr(w1), _lib.ptr(b1),
                                                  _lib.ptr(w2), _lib.ptr(b2), ctypes.c_void_p(yb.data_ptr() + 2 * GUARD), cs,
                                                  _lib.ptr(wy), _lib.ptr(by), _lib.stream_ptr()))
        outb, width, x_in = yb, cs, x0[GUARD:GUARD + T * C].view(T, C)
    else:
        _lib.check(lib.nb200_swin_mlp_fused_f16(xp, _lib.ptr(att), T, C, _lib.ptr(wp), _lib.ptr(bp), _lib.ptr(w1), _lib.ptr(b1),
                                                _lib.ptr(w2), _lib.ptr(b2), _lib.stream_ptr()))
        outb, width, x_in = xb, C, x0[GUARD:GUARD + T * C].view(T, C)
    torch.cuda.synchronize()
    tally = Tally()
    got = body(outb, T * width).view(T, width)
    tally.no_nan("the output", got)
    tally.guards("output", outb, T * width)
    if cs:
        tally.exact("x although y was requested", bits(xb), bits(x0))
    rows = 1 << 16
    for t0 in range(0, T, rows):
        t1 = min(T, t0 + rows)
        ref, bound = mlp_reference(x_in[t0:t1], att[t0:t1] if proj else None, wp, bp, w1, b1, w2, b2, wy, by)
        tally.add(got[t0:t1], ref, bound)
    return tally.result()


def test_swin_mlp_replay(production):
    replay("swin_mlp", configurations(production, "swin_mlp", SYNTH_SWIN_MLP), swin_mlp_check)
