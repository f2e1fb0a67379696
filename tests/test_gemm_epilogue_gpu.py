"""The fused GEMM epilogue of gemm_tc.cu (1x1 convs, nn.Linear, the implicit-GEMM 3x3 conv, the 2x2 transposed conv), the
narrow pointwise pw_small.cu and the CUDA-core gemm_simt.cu, element by element against fp64.  Sections (a) to (g) are covering
designs over the epilogue's options and the tile geometries; section (i) adds one row for each route key (tests/routes.py: tile,
pipeline depth, epilogue options) that a model path reaches and those sections do not run.  covered_keys() lists the keys of all.

Operands are bf16-representable (A, W and bf16 residuals are rounded first), so the fp64 statement
y = act(s * (A W^T) + b) (+ r), in the order the call asks for, is what the kernel would compute with exact arithmetic.  Every
output element must lie within its own bound

    |got - ref| <= L_act * (gamma_K * |s| * (|A| |W|^T) + 4u (|s acc| + |b| [+ |r| when act follows the residual]) + eps_act(x))
                   + 4u |ref|        (+ 2^-8 |ref| for a bf16 output, the half-step of its rounding)

with u = 2^-24, gamma_K = GAMMA * K * u (fp32 accumulation of K products), L_act the Lipschitz constant of the activation
(1.5 hswish, 1.13 GELU, 0.25 sigmoid) and eps_act(x) the activation's own approximation error at its input x (the
Abramowitz-Stegun erf of common.cuh's es3_gelu_fast, the MUFU exp of sigmoid).  A bound per element, rather than a fraction of
the tensor's maximum, is what catches a wrong residual row or a missing scale on one 32-column chunk where the values are small.

Output buffers are prefilled with NaN: every cell inside the output region must be written (a NaN fails the bound), and every cell
outside it -- the rest of a wider buffer, or a tail past the end -- must keep its sentinel bits.  Strided operands are slices of
NaN-padded buffers, so a read outside the slice also shows.

GAMMA = 2 and the eps_act of tests/bounds.py were set from one run on an H100 80GB HBM3 (700 W power limit).  Measured maximum err/bound per
section, fp32 outputs: (a) epilogue matrix 0.18, (c) act/residual order 0.021, (d) RoPE 0.0037, (e) conv3x3 0.019,
(f) convt2x2 0.025, (g) gemm_simt 0.054, (i) model routes 0.0082, so the fp32 accumulation stays well inside 2 K u.  bf16 outputs:
0.87 ... 0.996 in every section (pw_small 0.995, (i) 0.99 and its pw_small rows 0.995), because the half-step of the output
rounding dominates their bound and is reached.
(b) reaches 1.0 of its half-step tolerance by construction: the residual sits at a bf16 midpoint.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from bounds import (L_ACT, U, _INT, _act64, _assert_untouched, _bf, _check, _eps_act, _flat_out, _gen, _matrix_out, _p, _padded,
                    _pairwise, _st, report_worst, WORST)
from routes import conv3x3_key, convt2x2_key, gemm_key

pytestmark = pytest.mark.gpu

GAMMA = 2.0                    # gamma_K = GAMMA * K * u
_report_worst = report_worst("gemm epilogue")


def _expect(acc, absprod, K, act=None, scale=None, bias=None, res=None, after=False, out_bf16=False):
    """fp64 reference and per-element bound (module docstring).  acc, absprod: fp64 A W^T and |A| |W|^T; scale / bias [N]
    broadcast over the last dim; res in the output's layout."""
    s = scale.double() if scale is not None else 1.0
    sacc = acc * s
    inner = GAMMA * K * U * absprod * (s.abs() if scale is not None else 1.0) + 4 * U * sacc.abs()
    pre = sacc
    if bias is not None:
        pre = pre + bias.double()
        inner = inner + 4 * U * bias.double().abs()
    if res is None:
        x = pre
        ref = _act64(x, act)
    elif after:
        x = pre + res.double()
        inner = inner + 4 * U * res.double().abs()
        ref = _act64(x, act)
    else:
        x = pre
        ref = _act64(x, act) + res.double()
    bound = L_ACT[act] * (inner + _eps_act(x, act)) + 4 * U * ref.abs() + 2.0 ** -126
    if out_bf16:
        bound = bound * (1 + 2.0 ** -8) + 2.0 ** -8 * ref.abs()
    return ref, bound


# ---------------------------------------------------------------------------------------------- (a) es3_gemm_bf16_ex epilogue
GEMM_FACTORS = dict(
    M=[1, 77, 127, 129, 231, 5184],
    N=[8, 24, 48, 80, 96, 1024, 4736],
    K=[8, 200, 1024],                  # one k-block / the TMA K tail / 16 k-blocks: both BN-128 stage counts
    act=[None, "relu", "hswish", "gelu"],
    after=[False, True],
    scale=[False, True],
    bias=[False, True],
    res=[None, "bf16", "f32"],
    out=["bf16", "f32"],
    bn=[0, 32, 64, 128],
    strided=[False, True],
)
GEMM_DESIGN = _pairwise(GEMM_FACTORS, seed=1)


def _gemm_id(c):
    M, N, K, act, after, sc, bi, res, out, bn, strided = c
    return (f"M{M}-N{N}-K{K}-{act}-{'after' if after else 'before'}-{'s' if sc else ''}{'b' if bi else ''}-r{res}-{out}-bn{bn}"
            f"{'-strided' if strided else ''}")


def _gemm_case(cuda, M, N, K, act, after, has_s, has_b, res, out, bn, strided, seed=(), c_entry=False):
    """One GEMM through ops.gemm, or with c_entry through es3_gemm_bf16's C entry (bf16 residual only, act before it)."""
    from efficientsam3_b200 import _lib, ops
    g = _gen(cuda, M, N, K, act, after, has_s, has_b, res, out, bn, strided, *seed)
    a = _padded(_bf(torch.randn(M, K, device=cuda, generator=g)), strided)
    w = _bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    scale = (torch.rand(N, device=cuda, generator=g) + 0.5) * torch.randn(N, device=cuda, generator=g).sign() if has_s else None
    bias = torch.randn(N, device=cuda, generator=g) if has_b else None
    r = None
    if res is not None:
        r = 2 * torch.randn(M, N, device=cuda, generator=g)
        r = _padded(_bf(r) if res == "bf16" else r, strided)
    dt = torch.float32 if out == "f32" else torch.bfloat16
    buf, o, inside = _matrix_out(M, N, dt, strided, cuda)
    if c_entry:
        assert res != "f32" and not after
        _lib.init(cuda.index or 0)
        rc = _lib.call_rc("es3_gemm_bf16", a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), o.data_ptr(), o.stride(0),
                          int(out == "f32"), M, N, K, _p(scale), _p(bias), ops.ACT[act], _p(r), 0 if r is None else r.stride(0),
                          bn, _st())
        assert rc == 0
    else:
        got = ops.gemm(a, w, scale=scale, bias=bias, act=act, residual=r, out=o, bn_hint=bn, act_after_res=after)
        assert got.data_ptr() == o.data_ptr()
    acc = a.double() @ w.double().t()
    absprod = a.double().abs() @ w.double().abs().t()
    ref, bound = _expect(acc, absprod, K, act, scale, bias, r, after, out_bf16=out == "bf16")
    return buf, o, inside, ref, bound


@pytest.mark.parametrize("M,N,K,act,after,has_s,has_b,res,out,bn,strided", GEMM_DESIGN, ids=[_gemm_id(c) for c in GEMM_DESIGN])
def test_gemm_epilogue(cuda, monkeypatch, M, N, K, act, after, has_s, has_b, res, out, bn, strided):
    """Pairwise cover of act x act-after-residual x scale x bias x residual dtype x out dtype x tile width x M x N (ragged 32-column
    chunks at 8, 24, 48, 80) x K, contiguous and strided; always on the wgmma kernel."""
    from efficientsam3_b200 import ops
    monkeypatch.setattr(ops, "PW_SMALL", False)
    buf, o, inside, ref, bound = _gemm_case(cuda, M, N, K, act, after, has_s, has_b, res, out, bn, strided)
    what = _gemm_id((M, N, K, act, after, has_s, has_b, res, out, bn, strided))
    _check(f"a/{out}", o, ref, bound, what)
    _assert_untouched(buf, inside, what)


PW_SMALL_ROWS = [(4099, 16, 16, "bf16", True), (231, 64, 32, None, False), (1, 32, 64, "bf16", False), (129, 16, 64, None, True),
                 (5184, 32, 16, "bf16", False)]


@pytest.mark.parametrize("pw_small", [True, False])
@pytest.mark.parametrize("M,N,K,res,strided", PW_SMALL_ROWS)
def test_gemm_pw_small_route(cuda, monkeypatch, M, N, K, res, strided, pw_small):
    """Plain narrow GEMMs (K, N <= 64, no scale / bias / act, bf16 out) on es3_pw_small_bf16 and, with the switch off, on wgmma."""
    from efficientsam3_b200 import ops
    monkeypatch.setattr(ops, "PW_SMALL", pw_small)
    buf, o, inside, ref, bound = _gemm_case(cuda, M, N, K, None, False, False, False, res, "bf16", 0, strided)
    what = f"pw_small={pw_small} {M}x{N}x{K} res={res} strided={strided}"
    _check("pw_small", o, ref, bound, what)
    _assert_untouched(buf, inside, what)


# ---------------------------------------------------------------------------------------------- (b) the fp32 residual's precision
FP32_RES_ROWS = [(bn, N, out) for bn in (32, 64, 128) for N in (96, 80) for out in ("f32", "bf16")]


@pytest.mark.parametrize("bn,N,out", FP32_RES_ROWS)
def test_fp32_residual_keeps_precision(cuda, bn, N, out):
    """|A W^T| ~ 1 on a residual near 4096, where bf16's step is 32.  fp32 out: the residual's fraction survives (|err| <= 1e-3).
    bf16 out: the residual sits within 1 of 4112, the midpoint between two bf16 values, so a sum rounded once at the store is
    within half a step (16) of the fp64 result, while a residual rounded to bf16 first lands on the far side.  N = 80 ends in a
    ragged 16-column chunk."""
    from efficientsam3_b200 import ops
    M, K = 300, 256
    g = _gen(cuda, "b", bn, N, out)
    a = _bf(torch.randn(M, K, device=cuda, generator=g))
    w = _bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    u01 = torch.rand(M, N, device=cuda, generator=g)
    r = 4096 + u01 if out == "f32" else 4112 + (2 * u01 - 1)
    dt = torch.float32 if out == "f32" else torch.bfloat16
    buf, o, inside = _matrix_out(M, N, dt, False, cuda)
    ops.gemm(a, w, residual=r, out=o, bn_hint=bn)
    ref = a.double() @ w.double().t() + r.double()
    tol = 1e-3 if out == "f32" else 16 + 1e-3
    err = (o.double() - ref).abs()
    assert not torch.isnan(o).any(), "unwritten output cells"
    assert err.max().item() <= tol, f"bn={bn} N={N} {out}: max |err| {err.max().item():.4g} > {tol}"
    WORST["b"] = max(WORST.get("b", 0.0), err.max().item() / tol)
    _assert_untouched(buf, inside, f"fp32 residual bn={bn} N={N}")


# ---------------------------------------------------------------------------------------------- (c) activation vs residual order
ORDER_ROWS = [(N, after, res) for N in (96, 40) for after in (False, True) for res in ("bf16", "f32")]


@pytest.mark.parametrize("N,after,res", ORDER_ROWS)
def test_act_residual_order(cuda, N, after, res):
    """relu on a negative pre-activation (about -2) with a positive residual (3 .. 4): relu(x) + r = r, relu(x + r) = x + r, two
    answers about 2 apart.  N = 96 runs the vectorised chunks only, N = 40 a full chunk and a ragged 8-column one."""
    from efficientsam3_b200 import ops
    M, K = 200, 64
    g = _gen(cuda, "c", N, after, res)
    a = _bf(torch.randn(M, K, device=cuda, generator=g))
    w = _bf(torch.randn(N, K, device=cuda, generator=g) / (4 * math.sqrt(K)))
    bias = torch.full((N,), -2.0, device=cuda)
    r = 3 + torch.rand(M, N, device=cuda, generator=g)
    r = _bf(r) if res == "bf16" else r
    buf, o, inside = _matrix_out(M, N, torch.float32, False, cuda)
    ops.gemm(a, w, bias=bias, act="relu", residual=r, out=o, act_after_res=after)
    acc = a.double() @ w.double().t()
    absprod = a.double().abs() @ w.double().abs().t()
    ref, bound = _expect(acc, absprod, K, "relu", None, bias, r, after)
    other, _ = _expect(acc, absprod, K, "relu", None, bias, r, not after)
    assert ((ref - other).abs() > 1).double().mean().item() > 0.99        # the two orders are far apart on this data
    _check("c", o, ref, bound, f"act/residual order N={N} after={after} res={res}")
    _assert_untouched(buf, inside, "act/residual order")


# ---------------------------------------------------------------------------------------------- (d) RoPE epilogue
ROPE_ROWS = [(24, "bf16", 128), (24, "f32", 64), (0, "bf16", 64), (0, "f32", 128)]


@pytest.mark.parametrize("win,out,bn", ROPE_ROWS)
def test_rope_epilogue_teacher_geometry(cuda, win, out, bn):
    """The SAM3 ViT's QKV projection: 72 x 72 tokens, B = 2, C = 1024, bias; windows of 24 (576 table positions) or global (5184).
    q | k (columns < 2C) rotated per 64-dim head; v (columns >= 2C) bit-identical to the same GEMM without RoPE."""
    _rope_case(cuda, 2, 72, 72, 1024, win, out, bn)


def _rope_case(cuda, B, H, W, C, win, out, bn, seed=(), section="d"):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.vitdet import compute_axial_cis
    M, N, K = B * H * W, 3 * C, C
    g = _gen(cuda, "d", win, out, bn, *seed)
    a = _bf(torch.randn(M, K, device=cuda, generator=g))
    w = _bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    bias = torch.randn(N, device=cuda, generator=g)
    cis = compute_axial_cis(64, win, win) if win else compute_axial_cis(64, H, W, scale_pos=24 / H)
    tab = torch.view_as_real(cis).float().contiguous().to(cuda)                 # [positions, 32, 2] (cos, sin)
    assert tab.shape[0] == (win * win if win else H * W)
    dt = torch.float32 if out == "f32" else torch.bfloat16
    buf, o, inside = _matrix_out(M, N, dt, False, cuda)
    ops.gemm(a, w, bias=bias, rope=(tab, 2 * C, H, W, win), out=o, bn_hint=bn)
    plain = ops.gemm(a, w, bias=bias, out_dtype=dt, bn_hint=bn)
    assert torch.equal(o[:, 2 * C:].view(_INT[dt]), plain[:, 2 * C:].view(_INT[dt])), "v columns differ from the GEMM without RoPE"

    acc = a.double() @ w.double().t()
    absprod = a.double().abs() @ w.double().abs().t()
    x, xb = _expect(acc, absprod, K, bias=bias)                                  # pre-rotation value and its bound
    t = torch.arange(M, device=cuda) % (H * W)
    hh, ww = t // W, t % W
    pidx = (hh % win) * win + (ww % win) if win else t
    cs = tab.double()[pidx]                                                      # [M, 32, 2]
    c, s = cs[..., 0].repeat(1, 2 * C // 64), cs[..., 1].repeat(1, 2 * C // 64)  # per (q | k) column pair
    x0, x1 = x[:, 0:2 * C:2], x[:, 1:2 * C:2]
    b0, b1 = xb[:, 0:2 * C:2], xb[:, 1:2 * C:2]
    ref, bound = x.clone(), xb.clone()
    ref[:, 0:2 * C:2], ref[:, 1:2 * C:2] = x0 * c - x1 * s, x0 * s + x1 * c
    rot = c.abs() * b0 + s.abs() * b1 + 4 * U * (x0.abs() * c.abs() + x1.abs() * s.abs())
    bound[:, 0:2 * C:2], bound[:, 1:2 * C:2] = rot, c.abs() * b1 + s.abs() * b0 + 4 * U * (x0.abs() * s.abs() + x1.abs() * c.abs())
    bound[:, :2 * C] += 4 * U * ref[:, :2 * C].abs()
    if out == "bf16":
        bound = bound * (1 + 2.0 ** -8) + 2.0 ** -8 * ref.abs()
    _check(f"{section}/{out}", o, ref, bound, f"rope {B}x{H}x{W} C{C} win={win} {out} bn={bn}")
    _assert_untouched(buf, inside, "rope")


# ---------------------------------------------------------------------------------------------- (e) es3_conv3x3_bf16
def _conv3x3(cuda, x, w, epi, bn=0, seed=0, section="e"):
    """Run the implicit-GEMM conv through its C entry into a NaN-prefilled buffer; check it against fp64 F.conv2d."""
    from efficientsam3_b200 import _lib, ops
    B, H, W, C = x.shape
    N = w.shape[0]
    g = _gen(cuda, "e", B, H, W, C, N, epi, seed)
    bias = torch.randn(N, device=cuda, generator=g) if epi != "nobias" else None
    scale = (torch.rand(N, device=cuda, generator=g) + 0.5) if epi.startswith("scale") else None
    act = {"scale_hswish": "hswish", "scale_gelu": "gelu"}.get(epi)
    res = _bf(torch.randn(B, H, W, N, device=cuda, generator=g)) if epi == "bias_res" else None
    dt = torch.float32 if epi == "bias_f32" else torch.bfloat16
    w9 = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    buf, inside = _flat_out(B * H * W * N, dt, cuda)
    _lib.init(cuda.index or 0)
    rc = _lib.call_rc("es3_conv3x3_bf16", x.data_ptr(), w9.data_ptr(), buf.data_ptr(), int(dt == torch.float32), B, H, W, C, N,
                      _p(scale), _p(bias), ops.ACT[act], _p(res), bn, _st())
    assert rc == 0
    xn, wd = x.double().permute(0, 3, 1, 2), w.double()
    acc = F.conv2d(xn, wd, padding=1).permute(0, 2, 3, 1)
    absprod = F.conv2d(xn.abs(), wd.abs(), padding=1).permute(0, 2, 3, 1)
    ref, bound = _expect(acc, absprod, 9 * C, act, scale, bias, res, False, out_bf16=dt == torch.bfloat16)
    what = f"conv3x3 B{B} {H}x{W} C{C}->N{N} {epi} bn{bn}"
    _check(f"{section}/{'f32' if dt == torch.float32 else 'bf16'}", buf[:B * H * W * N].view(B, H, W, N), ref, bound, what)
    _assert_untouched(buf, inside, what)


CONV_FACTORS = dict(
    W=[64, 48, 144, 36, 23],           # tile width 32, 16, 16, 8, 8 (W % 32, W % 16)
    H=[13, 7, 18],                     # never a multiple of the tile height (4, 8, 16): partial row tiles
    C=[8, 32, 96, 256, 1024],          # C % 64 != 0: a tap's last k-block runs into the next tap's weights
    N=[32, 64, 256, 1024],
    epi=["bias", "nobias", "scale_hswish", "scale_gelu", "bias_f32", "bias_res"],
)
CONV_DESIGN = _pairwise(CONV_FACTORS, seed=2)


@pytest.mark.parametrize("W,H,C,N,epi", CONV_DESIGN, ids=[f"W{c[0]}-H{c[1]}-C{c[2]}-N{c[3]}-{c[4]}" for c in CONV_DESIGN])
def test_conv3x3_geometry(cuda, W, H, C, N, epi):
    g = _gen(cuda, "conv", W, H, C, N, epi)
    x = _bf(torch.randn(3, H, W, C, device=cuda, generator=g))
    w = _bf(torch.randn(N, C, 3, 3, device=cuda, generator=g) / math.sqrt(9 * C))
    _conv3x3(cuda, x, w, epi)


CONV_PROD_ROWS = [(1, 144, 144, 256, 256, "bias_f32"), (2, 144, 144, 256, 256, "bias"), (2, 36, 36, 256, 256, "bias"),
                  (2, 64, 64, 1024, 1024, "bias"), (1, 64, 64, 1024, 1024, "nobias")]


@pytest.mark.parametrize("B,H,W,C,N,epi", CONV_PROD_ROWS)
def test_conv3x3_production_shapes(cuda, B, H, W, C, N, epi):
    """The FPN neck's 3x3 conv at the 2x (144^2, fp32 levels too) and 0.5x (36^2) levels; the student head at 64^2 and its input
    gradient (no bias)."""
    g = _gen(cuda, "prod", B, H, W, C, N, epi)
    x = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    w = _bf(torch.randn(N, C, 3, 3, device=cuda, generator=g) / math.sqrt(9 * C))
    _conv3x3(cuda, x, w, epi)


HALO_W = [64, 48, 23]


@pytest.mark.parametrize("W", HALO_W)
def test_conv3x3_halo(cuda, W):
    """Large values (8) in the last column and last row of every image, small ones (< 1/16) elsewhere: column 0 reading its left
    neighbour from the previous row's last column, or an image's last row reading the next image's first row (or the reverse),
    would be far outside the bound."""
    B, H, C, N = 3, 13, 64, 64
    g = _gen(cuda, "halo", W)
    x = (torch.rand(B, H, W, C, device=cuda, generator=g) - 0.5) / 8
    sgn = torch.randn(B, H, W, C, device=cuda, generator=g).sign()
    x[:, :, -1] = 8 * sgn[:, :, -1]
    x[:, -1] = 8 * sgn[:, -1]
    w = _bf(torch.randn(N, C, 3, 3, device=cuda, generator=g) / math.sqrt(9 * C))
    _conv3x3(cuda, _bf(x), w, "bias")


# ---------------------------------------------------------------------------------------------- (f) es3_convt2x2_bf16
def _convt2x2(cuda, B, H, W, Cin, Cout, mode, res, out, seed=0):
    from efficientsam3_b200 import _lib, ops
    g = _gen(cuda, "f", B, H, W, Cin, Cout, mode, res, out, seed)
    x = _bf(torch.randn(B, H, W, Cin, device=cuda, generator=g))
    w = _bf(torch.randn(Cin, Cout, 2, 2, device=cuda, generator=g) / math.sqrt(Cin))      # nn.ConvTranspose2d layout
    bias = torch.randn(Cout, device=cuda, generator=g)
    act = None if mode == "none" else "gelu"
    after = mode == "gelu_after"
    r = None
    if res is not None:
        r = torch.randn(B, 2 * H, 2 * W, Cout, device=cuda, generator=g)
        r = _bf(r) if res == "bf16" else r
    dt = torch.float32 if out == "f32" else torch.bfloat16
    wt = ops.convt2x2_weight(w)
    bias4 = bias.repeat(4).contiguous()
    n = B * 4 * H * W * Cout
    buf, inside = _flat_out(n, dt, cuda)
    _lib.init(cuda.index or 0)
    rc = _lib.call_rc("es3_convt2x2_bf16", x.data_ptr(), wt.data_ptr(), buf.data_ptr(), int(dt == torch.float32), B, H, W, Cin,
                      Cout, bias4.data_ptr(), ops.ACT[act], _p(r), int(res == "f32"), int(after), _st())
    assert rc == 0
    xn = x.double().permute(0, 3, 1, 2)
    acc = F.conv_transpose2d(xn, w.double(), stride=2).permute(0, 2, 3, 1)
    absprod = F.conv_transpose2d(xn.abs(), w.double().abs(), stride=2).permute(0, 2, 3, 1)
    ref, bound = _expect(acc, absprod, Cin, act, None, bias, r, after, out_bf16=out == "bf16")
    what = f"convt2x2 B{B} {H}x{W} {Cin}->{Cout} {mode} res={res} {out}"
    _check(f"f/{out}", buf[:n].view(B, 2 * H, 2 * W, Cout), ref, bound, what)
    _assert_untouched(buf, inside, what)


CONVT_FACTORS = dict(
    Cout=[32, 64, 256, 512],
    Cin=[64, 256, 1024],
    mode=["none", "gelu_before", "gelu_after"],
    res=[None, "bf16", "f32"],
    out=["bf16", "f32"],
    HW=[(5, 7), (9, 3), (7, 11)],
)
CONVT_DESIGN = _pairwise(CONVT_FACTORS, seed=3)


@pytest.mark.parametrize("Cout,Cin,mode,res,out,HW", CONVT_DESIGN,
                         ids=[f"{c[1]}to{c[0]}-{c[2]}-r{c[3]}-{c[4]}-{c[5][0]}x{c[5][1]}" for c in CONVT_DESIGN])
def test_convt2x2_scatter(cuda, Cout, Cin, mode, res, out, HW):
    """Depth-to-space scatter: every output pixel written, each with the value of its own (dy, dx) weight slice."""
    _convt2x2(cuda, 3, HW[0], HW[1], Cin, Cout, mode, res, out)


CONVT_PROD_ROWS = [(1, 72, 72, 1024, 512, "gelu_before", None, "bf16"), (1, 144, 144, 512, 256, "none", None, "bf16"),
                   (2, 72, 72, 256, 64, "none", "f32", "f32"), (2, 144, 144, 64, 32, "gelu_after", "f32", "f32")]


@pytest.mark.parametrize("B,H,W,Cin,Cout,mode,res,out", CONVT_PROD_ROWS)
def test_convt2x2_production_shapes(cuda, B, H, W, Cin, Cout, mode, res, out):
    """The FPN neck's 4x level (1024 -> 512 with GELU, 512 -> 256) and the mask decoder's upscaling (256 -> 64 on an fp32 residual,
    64 -> 32 with GELU after the residual)."""
    _convt2x2(cuda, B, H, W, Cin, Cout, mode, res, out)


# ---------------------------------------------------------------------------------------------- (g) es3_gemm_simt
SIMT_FACTORS = dict(
    dtypes=[("bf16", "bf16"), ("f32", "f32"), ("f32", "bf16"), ("bf16", "f32")],
    res=[None, "bf16", "f32"],
    out=["bf16", "f32"],
    M=[1, 3, 17],
    K=[20, 100],
    N=[7, 40],
    act=["relu", "sigmoid"],
    scale=[False, True],
)
SIMT_DESIGN = _pairwise(SIMT_FACTORS, seed=4)


@pytest.mark.parametrize("dtypes,res,out,M,K,N,act,has_s", SIMT_DESIGN,
                         ids=[f"a{c[0][0]}-w{c[0][1]}-r{c[1]}-{c[2]}-M{c[3]}-K{c[4]}-N{c[5]}-{c[6]}{'-s' if c[7] else ''}"
                              for c in SIMT_DESIGN])
def test_gemm_simt(cuda, dtypes, res, out, M, K, N, act, has_s):
    """The CUDA-core GEMM (SE MLPs and their backward in fp32, the decoder's token MLPs) with every operand dtype pair."""
    _simt_case(cuda, dtypes, res, out, M, K, N, act, has_s)


def _simt_case(cuda, dtypes, res, out, M, K, N, act, has_s, has_b=True, section="g"):
    from efficientsam3_b200 import ops
    g = _gen(cuda, "g", dtypes, res, out, M, K, N, act, has_s, *(() if has_b else ("no bias",)))
    a = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K)
    a = _bf(a) if dtypes[0] == "bf16" else a
    w = _bf(w) if dtypes[1] == "bf16" else w
    scale = (torch.rand(N, device=cuda, generator=g) + 0.5) if has_s else None
    bias = torch.randn(N, device=cuda, generator=g) if has_b else None
    r = None
    if res is not None:
        r = torch.randn(M, N, device=cuda, generator=g)
        r = _bf(r) if res == "bf16" else r
    dt = torch.float32 if out == "f32" else torch.bfloat16
    buf, o, inside = _matrix_out(M, N, dt, True, cuda)
    ops.gemm_simt(a, w, scale=scale, bias=bias, act=act, residual=r, out=o)
    acc = a.double() @ w.double().t()
    absprod = a.double().abs() @ w.double().abs().t()
    ref, bound = _expect(acc, absprod, K, act, scale, bias, r, False, out_bf16=out == "bf16")
    what = f"gemm_simt {dtypes} res={res} {out} {M}x{N}x{K} {act}{'' if has_b else ' no bias'}"
    _check(f"{section}/{out}", o, ref, bound, what)
    _assert_untouched(buf, inside, what)


# ---------------------------------------------------------------------------------------------- (i) the routes the models reach
# One row per route key (tests/routes.py) that a recorded model path (tests/test_route_closure_gpu.py) reaches and no row above runs,
# each at a shape that selects it; keys do not depend on M, so M stays small.  The comments name the paths that reach the key.
#   ("ex" | "c", M, N, K, act, act after the residual, scale, bias, residual, out): es3_gemm_bf16_ex through ops.gemm (pw_small
#       off), or es3_gemm_bf16 through its C entry; no tile hint
#   ("rope", B, H, W, C, win, out): the QKV projection of _rope_case, no tile hint
#   ("pw", M, N, K, residual): es3_pw_small_bf16 through ops.gemm
#   ("simt", M, N, K, act, scale, bias, residual, out): es3_gemm_simt on fp32 A and W
#   ("conv3x3", B, H, W, C, N, epi): es3_conv3x3_bf16 as _conv3x3 runs it
MODEL_ROWS = [
    # image students' eval forward: folded BN + hswish / GELU, project + bias + residual
    ("ex", 200, 384, 96, "hswish", False, False, True, None, "bf16"),          # EfficientViT-B2 (two k-blocks: 2 stages)
    ("ex", 231, 1024, 256, "hswish", False, False, True, None, "bf16"),        # EfficientViT-B1, B2; the EV-B1 point segmenter
    ("ex", 257, 32, 16, "hswish", False, False, True, None, "bf16"),           # EfficientViT-B0
    ("ex", 200, 96, 24, "hswish", False, False, True, None, "bf16"),           # EfficientViT-B0, B2
    ("ex", 257, 24, 96, None, False, False, True, "bf16", "bf16"),             # EfficientViT-B0, B2, RepViT-M0.9 (ragged)
    ("ex", 257, 8, 16, None, False, False, True, None, "bf16"),                # EfficientViT-B0, B2 (ragged)
    ("ex", 129, 64, 256, None, False, False, True, "bf16", "bf16"),            # every image student
    ("ex", 129, 256, 1024, None, False, False, True, "bf16", "bf16"),          # EfficientViT-B1, B2, RepViT, TinyViT
    ("ex", 160, 80, 160, None, False, False, True, "bf16", "bf16"),            # RepViT-M2.3 (80 channels: ragged on 64-wide tiles)
    ("ex", 196, 256, 64, "gelu", False, True, True, None, "bf16"),             # TinyViT
    ("ex", 196, 64, 256, "gelu", True, True, True, "bf16", "bf16"),            # TinyViT (GELU after the residual)
    ("ex", 196, 128, 64, None, False, True, True, None, "bf16"),               # TinyViT
    ("ex", 150, 448, 256, None, False, True, True, None, "bf16"),              # TinyViT-11M, 21M
    ("ex", 77, 384, 128, None, False, False, True, None, "bf16"),              # TinyViT-5M, 11M, eval and training
    ("ex", 144, 1184, 256, "gelu", False, False, True, None, "bf16"),          # every image student; the ViT backbones
    ("simt", 2, 40, 448, None, False, True, None, "bf16"),                     # TinyViT
    # image students' training steps: raw 1x1 convs (no epilogue) and input gradients on the skip gradient
    ("ex", 131, 512, 128, None, False, False, False, None, "bf16"),            # EfficientViT, TinyViT; EfficientViT-B0, B1 eval
    ("ex", 300, 32, 8, None, False, False, False, None, "bf16"),               # EfficientViT-B0, B1, RepViT-M0.9 (K = 8)
    ("ex", 129, 256, 1024, None, False, False, False, "bf16", "bf16"),         # EfficientViT, RepViT
    ("ex", 129, 64, 256, None, False, False, False, "bf16", "bf16"),           # every image student
    ("ex", 129, 128, 256, None, False, False, False, None, "f32"),             # every image student
    ("ex", 160, 80, 160, None, False, False, False, "bf16", "bf16"),           # RepViT-M2.3
    ("ex", 160, 80, 320, None, False, False, False, None, "bf16"),             # RepViT-M2.3
    ("pw", 129, 64, 16, None),                                                 # EfficientViT-B0, B1
    ("pw", 257, 32, 16, None),                                                 # EfficientViT-B0
    ("pw", 200, 16, 32, None),                                                 # EfficientViT-B0
    ("pw", 300, 16, 16, None),                                                 # EfficientViT-B1
    ("pw", 131, 16, 64, "bf16"),                                               # EfficientViT-B0
    ("pw", 77, 32, 64, None),                                                  # EfficientViT-B0, B1, RepViT-M1.1, TinyViT
    ("simt", 2, 16, 64, None, False, False, None, "f32"),                      # RepViT (SqueezeExcite gradients)
    # text encoders, the SAM3 ViT and the SAM heads
    ("ex", 77, 1536, 512, None, False, False, True, None, "bf16"),             # text encoders, SAM heads, most image students
    ("ex", 77, 512, 512, None, False, False, True, None, "f32"),               # text students, SAM3 text teacher
    ("ex", 77, 512, 2048, None, False, False, False, None, "bf16"),            # text and image students' training steps
    ("ex", 77, 4096, 1024, "gelu", False, False, True, None, "bf16"),          # SAM3 text teacher, SAM3 ViT, RepViT, TinyViT-21M
    ("ex", 196, 1024, 592, None, False, False, False, None, "f32"),            # ViT patch embedding (also the FP8 teacher's), text
    ("rope", 2, 12, 12, 1024, 0, "bf16"),                                      # global-RoPE QKV: teacher, ViT backbones
    ("ex", 100, 1024, 4736, None, False, False, True, "f32", "f32"),           # ViT proj / fc2 on the fp32 residual stream, text
    ("ex", 64, 32, 256, None, False, False, True, None, "f32"),                # SAM heads' high-resolution features
    ("ex", 64, 64, 256, None, False, False, True, None, "f32"),                # SAM heads' high-resolution features
    ("conv3x3", 1, 5, 36, 256, 256, "bias_f32"),                               # the ViT point segmenter's neck (W % 16 != 0)
    ("simt", 6, 4, 256, "sigmoid", False, True, None, "f32"),                  # mask decoder heads, RepViT SqueezeExcite
    ("simt", 7, 256, 256, None, False, True, "f32", "f32"),                    # mask decoder
    ("simt", 5, 32, 256, None, False, True, None, "f32"),                      # mask decoder
    # es3_gemm_bf16: a header entry point no Python path calls
    ("c", 150, 96, 64, "hswish", False, True, True, "bf16", "bf16"),
]


def _model_row_key(row):
    kind, *c = row
    if kind in ("ex", "c"):
        M, N, K, act, after, sc, bi, res, out = c
        return gemm_key("es3_gemm_bf16_ex" if kind == "ex" else "es3_gemm_bf16", N, K, act, sc, bi, res, after, out, None, 0)
    if kind == "rope":
        B, H, W, C, win, out = c
        return gemm_key("es3_gemm_bf16_ex", 3 * C, C, None, False, True, None, False, out, "window" if win else "global", 0)
    if kind == "pw":
        M, N, K, res = c
        return ("es3_pw_small_bf16", K, N, res is not None)
    if kind == "simt":
        M, N, K, act, sc, bi, res, out = c
        return ("es3_gemm_simt", "f32", "f32", act, sc, bi, res, out)
    B, H, W, C, N, epi = c
    return conv3x3_key(N, W, *_CONV_EPI[epi], 0)


@pytest.mark.parametrize("row", MODEL_ROWS, ids=["-".join(map(str, r)) for r in MODEL_ROWS])
def test_model_route(cuda, monkeypatch, row):
    """Each row against fp64 with the bound and NaN sentinels of its section above; the calls it makes are recorded and the row's
    route key must be among theirs, so the row runs the key covered_keys() claims for it."""
    from efficientsam3_b200 import ops
    from es3_recorder import record_calls
    from routes import KEYS
    kind, *c = row
    what = "model route " + "-".join(map(str, row))

    def run():
        if kind in ("ex", "c"):
            M, N, K, act, after, sc, bi, res, out = c
            monkeypatch.setattr(ops, "PW_SMALL", False)
            buf, o, inside, ref, bound = _gemm_case(cuda, M, N, K, act, after, sc, bi, res, out, 0, False, seed=("i",),
                                                    c_entry=kind == "c")
            _check(f"i/{out}", o, ref, bound, what)
            _assert_untouched(buf, inside, what)
        elif kind == "rope":
            B, H, W, C, win, out = c
            _rope_case(cuda, B, H, W, C, win, out, 0, seed=("i",), section="i")
        elif kind == "pw":
            M, N, K, res = c
            monkeypatch.setattr(ops, "PW_SMALL", True)
            buf, o, inside, ref, bound = _gemm_case(cuda, M, N, K, None, False, False, False, res, "bf16", 0, False, seed=("i",))
            _check("i/pw_small", o, ref, bound, what)
            _assert_untouched(buf, inside, what)
        elif kind == "simt":
            M, N, K, act, sc, bi, res, out = c
            _simt_case(cuda, ("f32", "f32"), res, out, M, K, N, act, sc, bi, section="i")
        else:
            B, H, W, C, N, epi = c
            g = _gen(cuda, "i", B, H, W, C, N, epi)
            x = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
            w = _bf(torch.randn(N, C, 3, 3, device=cuda, generator=g) / math.sqrt(9 * C))
            _conv3x3(cuda, x, w, epi, section="i")
    keys = {KEYS[n](a) for n, a in record_calls(monkeypatch, run)}
    assert _model_row_key(row) in keys, f"{what}: runs {sorted(keys, key=repr)}, not {_model_row_key(row)}"


# ---------------------------------------------------------------------------------------------- (h) what the wrappers refuse
@pytest.mark.parametrize("act", ["sigmoid", "relu6", "gelu_tanh"])
def test_tc_activation_not_instantiated(cuda, act):
    """The wgmma kernel instantiates none / relu / hswish / gelu only; any other code is an error, not a silent identity."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200._lib import Es3Error
    x = torch.zeros(1, 8, 8, 64, device=cuda, dtype=torch.bfloat16)
    with pytest.raises(Es3Error):
        ops.gemm(x.view(64, 64), torch.zeros(64, 64, device=cuda, dtype=torch.bfloat16), act=act)
    with pytest.raises(Es3Error):
        ops.conv3x3(x, torch.zeros(64, 9 * 64, device=cuda, dtype=torch.bfloat16), act=act)
    with pytest.raises(Es3Error):
        ops.convt2x2(x, torch.zeros(4 * 32, 64, device=cuda, dtype=torch.bfloat16), act=act)


def _refusals(cuda):
    from efficientsam3_b200 import ops
    bf, f32, f16 = torch.bfloat16, torch.float32, torch.float16
    a, w = torch.zeros(64, 64, device=cuda, dtype=bf), torch.zeros(32, 64, device=cuda, dtype=bf)
    x = torch.zeros(2, 8, 8, 64, device=cuda, dtype=bf)
    w9, wt = torch.zeros(32, 9 * 64, device=cuda, dtype=bf), torch.zeros(4 * 32, 64, device=cuda, dtype=bf)
    return {
        "gemm fp16 out": lambda: ops.gemm(a, w, out=torch.zeros(64, 32, device=cuda, dtype=f16)),
        "gemm fp16 residual": lambda: ops.gemm(a, w, residual=torch.zeros(64, 32, device=cuda, dtype=f16)),
        "gemm fp16 bias": lambda: ops.gemm(a, w, bias=torch.zeros(32, device=cuda, dtype=f16)),
        "gemm_simt fp16 a": lambda: ops.gemm_simt(a.half(), w),
        "gemm_simt fp16 w": lambda: ops.gemm_simt(a, w.half()),
        "gemm_simt fp64 a": lambda: ops.gemm_simt(a.double(), w),
        "gemm_simt fp16 residual": lambda: ops.gemm_simt(a, w, residual=torch.zeros(64, 32, device=cuda, dtype=f16)),
        "gemm_simt fp16 out": lambda: ops.gemm_simt(a, w, out_dtype=f16),
        "gemm_simt fp16 scale": lambda: ops.gemm_simt(a, w, scale=torch.ones(32, device=cuda, dtype=f16)),
        "conv3x3 fp32 residual": lambda: ops.conv3x3(x, w9, residual=torch.zeros(2, 8, 8, 32, device=cuda, dtype=f32)),
        "conv3x3 strided residual": lambda: ops.conv3x3(x, w9, residual=torch.zeros(2, 8, 8, 64, device=cuda, dtype=bf)[..., :32]),
        "conv3x3 residual shape": lambda: ops.conv3x3(x, w9, residual=torch.zeros(2, 8, 4, 64, device=cuda, dtype=bf)),
        "conv3x3 fp16 out": lambda: ops.conv3x3(x, w9, out_dtype=f16),
        "conv3x3 fp16 bias": lambda: ops.conv3x3(x, w9, bias=torch.zeros(32, device=cuda, dtype=f16)),
        "convt2x2 fp16 residual": lambda: ops.convt2x2(x, wt, residual=torch.zeros(2, 16, 16, 32, device=cuda, dtype=f16)),
        "convt2x2 fp16 out": lambda: ops.convt2x2(x, wt, out_dtype=f16),
        "convt2x2 fp64 bias4": lambda: ops.convt2x2(x, wt, bias4=torch.zeros(128, device=cuda, dtype=torch.float64)),
    }


REFUSALS = ["gemm fp16 out", "gemm fp16 residual", "gemm fp16 bias", "gemm_simt fp16 a", "gemm_simt fp16 w", "gemm_simt fp64 a",
            "gemm_simt fp16 residual", "gemm_simt fp16 out", "gemm_simt fp16 scale", "conv3x3 fp32 residual",
            "conv3x3 strided residual", "conv3x3 residual shape", "conv3x3 fp16 out", "conv3x3 fp16 bias",
            "convt2x2 fp16 residual", "convt2x2 fp16 out", "convt2x2 fp64 bias4"]


@pytest.mark.parametrize("case", REFUSALS)
def test_wrapper_rejects_dtype_the_kernel_would_misread(cuda, case):
    """Operand, residual and output dtypes other than the ones each kernel reads raise instead of being reinterpreted."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200._lib import Es3Error
    n0 = ops.launch_count
    with pytest.raises(Es3Error):
        _refusals(cuda)[case]()
    assert ops.launch_count == n0


# ---------------------------------------------------------------------------------------------- route keys
_CONV_EPI = {  # epi -> act, scale, bias, residual, out (as _conv3x3 reads it)
    "bias": (None, False, True, None, "bf16"), "nobias": (None, False, False, None, "bf16"),
    "scale_hswish": ("hswish", True, True, None, "bf16"), "scale_gelu": ("gelu", True, True, None, "bf16"),
    "bias_f32": (None, False, True, None, "f32"), "bias_res": (None, False, True, "bf16", "bf16")}


def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    return table_keys() | {_model_row_key(r) for r in MODEL_ROWS}


def table_keys():
    """The route keys of the tables of sections (a) to (g)."""
    ex = "es3_gemm_bf16_ex"
    keys = {gemm_key(ex, N, K, act, sc, bi, res, after, out, None, bn)
            for _, N, K, act, after, sc, bi, res, out, bn, _ in GEMM_DESIGN}
    keys |= {("es3_pw_small_bf16", K, N, res is not None) for M, N, K, res, _ in PW_SMALL_ROWS}
    keys |= {gemm_key(ex, N, K, None, False, False, res, False, "bf16", None, 0) for M, N, K, res, _ in PW_SMALL_ROWS}
    keys |= {gemm_key(ex, N, 256, None, False, False, "f32", False, out, None, bn) for bn, N, out in FP32_RES_ROWS}
    keys |= {gemm_key(ex, N, 64, "relu", False, True, res, after, "f32", None, 0) for N, after, res in ORDER_ROWS}
    keys |= {gemm_key(ex, 3072, 1024, None, False, True, None, False, out, "window" if win else "global", bn)
             for win, out, bn in ROPE_ROWS}
    convs = [(W, C, N, epi) for W, H, C, N, epi in CONV_DESIGN] + [(W, C, N, epi) for B, H, W, C, N, epi in CONV_PROD_ROWS]
    convs += [(W, 64, 64, "bias") for W in HALO_W]
    keys |= {conv3x3_key(N, W, *_CONV_EPI[epi], 0) for W, C, N, epi in convs}
    convts = [(Cin, Cout, mode, res, out) for Cout, Cin, mode, res, out, _ in CONVT_DESIGN]
    convts += [(Cin, Cout, mode, res, out) for B, H, W, Cin, Cout, mode, res, out in CONVT_PROD_ROWS]
    keys |= {convt2x2_key(Cin, Cout, None if mode == "none" else "gelu", res, mode == "gelu_after", out)
             for Cin, Cout, mode, res, out in convts}
    keys |= {("es3_gemm_simt", *dt, act, sc, True, res, out) for dt, res, out, M, K, N, act, sc in SIMT_DESIGN}
    return keys
