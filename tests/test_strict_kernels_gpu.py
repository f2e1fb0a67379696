"""The strict mode's student kernels (csrc/strict_f32.cu: es3_dwconv_f32, es3_litemla_attn_f32, es3_bilinear_nhwc_f32_to_nchw,
es3_bias_act_res_f32 and es3_scale_channels_f32), element by element against the fp64 statements of tests/ref_strict.py, each
output element within its own bound; the layout change and the channel gate bit for bit.

Outputs and the LiteMLA workspace are NaN-prefilled and the entry points called through _lib.call with the pixel strides the ops
wrappers do not expose: every cell inside the output region must be written and lie within its bound, every cell past it (a flat
TAIL, or the channels around a strided output) keeps its sentinel bits.  Every case runs twice and must be bit-identical; the last
image (or the last rows) run alone must be bit-identical to the same image inside the batch; the ops wrappers are bit-identical to
the direct call.  covered_keys() names the route keys (tests/routes.py) the tables run, for the route closure of
tests/test_route_closure_gpu.py (the nine students' strict eval forwards).

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power
limit), all fp32 outputs: dwconv_f32 0.213 (ks 3), 0.129 (ks 5), 0.197 (ks 7); litemla_attn_f32 0.028 (dim 16) and 0.027 (dim 32) in
one chunk, 0.00059 and 0.00040 over several (the kv chains of 2048 terms are far from their worst case); bilinear 0.378;
bias_act_res_f32 0.295.  The file (99 tests) took under 20 s there.
"""
import pytest
import torch

import ref_strict as R
from bounds import (TAIL, _assert_untouched, _bits_equal, _check, _flat_out, _gen, _lib, _p, _pairwise, _st, _twice, report_worst)

pytestmark = pytest.mark.gpu
_report_worst = report_worst("strict student kernels")
ACT = {None: 0, "relu": 1, "hswish": 2, "gelu": 3, "sigmoid": 6}


def _ops():
    from efficientsam3_b200 import ops
    return ops


def _nhwc_out(B, H, W, C, ld, cuda):
    """A NaN buffer of B H W ld + TAIL floats; returns (buffer, [B, H, W, C] view at channel 2 of pixels ld wide (channel 0 when ld
    = C), inside-mask)."""
    off = 2 if ld > C else 0
    buf = torch.full((B * H * W * ld + TAIL,), float("nan"), device=cuda)
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=cuda)
    inside[:B * H * W * ld].view(B, H, W, ld)[..., off:off + C] = True
    return buf, (lambda b: b[:B * H * W * ld].view(B, H, W, ld)[..., off:off + C]), inside


def _channel_slice(x, ld):
    """x [..., C] as channels [3, 3 + C) of a NaN-padded [..., ld] map (ld = C: x itself)."""
    if ld == x.shape[-1]:
        return x.contiguous()
    big = torch.full(x.shape[:-1] + (ld,), float("nan"), device=x.device)
    big[..., 3:3 + x.shape[-1]] = x
    return big[..., 3:3 + x.shape[-1]]


# ----------------------------------------------------------------------------------------------------------- (1) depthwise
DW = _pairwise(dict(ks=[3, 5, 7], stride=[1, 2], HW=[(9, 11), (16, 10), (2, 3), (7, 7), (1, 5)], C=[1, 3, 13, 16, 48, 160],
                    act=[None, "relu", "hswish", "gelu"], scale=[False, True], bias=[False, True], ldx=["dense", "wide"],
                    ldy=["dense", "wide"]), seed=31)
DW = [(2, *hw, C, ks, s, act, sc, bi, lx, ly) for ks, s, hw, C, act, sc, bi, lx, ly in DW]
DW += [  # the students' strict forwards at 1024^2, batch 2
    (2, 128, 128, 128, 3, 1, "hswish", True, True, "dense", "dense"),   # EfficientViT MBConv depthwise, stride 1
    (2, 256, 256, 128, 3, 2, "hswish", True, True, "dense", "dense"),   # ... stride 2
    (2, 128, 128, 256, 3, 2, "hswish", False, True, "dense", "dense"),  # EfficientViT stride-2 MBConv without its norm
    (2, 32, 32, 1024, 3, 1, "hswish", False, True, "dense", "dense"),   # EfficientViT-B2 stage 4
    (2, 64, 64, 384, 5, 1, None, False, False, "wide", "dense"),        # LiteMLA's 5 x 5 aggregation on ms[..., :c3]
    (2, 64, 64, 320, 3, 1, None, False, True, "dense", "dense"),        # RepViT RepVGG depthwise (BatchNorms folded into w, b)
    (2, 64, 64, 320, 3, 2, None, True, True, "dense", "dense"),         # RepViT stride-2 token mixer
    (2, 64, 64, 160, 3, 1, None, True, True, "dense", "dense"),         # TinyViT local conv
    (2, 256, 256, 256, 3, 1, "gelu", True, True, "dense", "dense"),     # TinyViT MBConv depthwise
    (2, 64, 64, 448, 3, 2, "gelu", True, True, "dense", "dense"),       # TinyViT patch merging
]


@pytest.mark.parametrize("B,H,W,C,ks,stride,act,scale,bias,ldx,ldy", DW)
def test_dwconv_f32(cuda, B, H, W, C, ks, stride, act, scale, bias, ldx, ldy):
    """Kernels 3, 5 and 7 at stride 1 and 2 on odd, even and smaller-than-kernel maps, ragged C, every activation, scale and bias
    each present or absent, a channel-slice input and a strided output; the last image alone; ops.dwconv_f32 bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "dw", B, H, W, C, ks, stride, act, scale, bias, ldx, ldy)
    x = _channel_slice(torch.randn(B, H, W, C, device=cuda, generator=g), C + 7 if ldx == "wide" else C)
    w = torch.randn(ks * ks, C, device=cuda, generator=g) / ks
    sc = torch.rand(C, device=cuda, generator=g) + 0.5 if scale else None
    bi = torch.randn(C, device=cuda, generator=g) if bias else None
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    ly = C + 5 if ldy == "wide" else C
    buf, view, ins = _nhwc_out(B, Ho, Wo, C, ly, cuda)

    def run(b, xx=x, nb=B):
        lib.call("es3_dwconv_f32", xx.data_ptr(), xx.stride(2), w.data_ptr(), _p(sc), _p(bi), view(b).data_ptr(), ly, nb, H, W, C, ks,
                 stride, ACT[act], _st())
    got = _twice(run, buf)
    d = lambda t: None if t is None else t.double()
    ref, bound = R.dwconv(x.double(), w.double(), d(sc), d(bi), ks, stride, act)
    what = f"dwconv_f32 B{B} {H}x{W} C{C} ks{ks} s{stride} act {act} scale={scale} bias={bias} ldx {ldx} ldy {ldy}"
    _check(f"1 dwconv_f32 ks{ks}", view(got), ref, bound, what)
    _assert_untouched(got, ins, what)
    one = buf.clone()
    run(one, x[-1:], 1)
    _bits_equal(view(one)[:1], view(got)[-1:], what + ": last image alone")
    out = view(torch.full_like(buf, float("nan")))
    _bits_equal(_ops().dwconv_f32(x, w, sc, bi, ks, stride, act, out=out), view(got), what + ": ops.dwconv_f32 vs direct")


# ----------------------------------------------------------------------------------------------------------- (2) LiteMLA
MLA = _pairwise(dict(dim=[16, 32], HW=[1, 31, 2048, 2049, 4096, 6145], heads=[1, 3], B=[1, 2], wide=[False, True]), seed=32)
MLA += [(16, 4096, 16, 2, False),             # EfficientViT-B1 stage 3 at 1024^2: two 2048-pixel chunks
        (32, 4096, 12, 2, False),             # EfficientViT-B2 stage 3
        (32, 1024, 24, 2, False)]             # EfficientViT-B2 stage 4: one chunk


def _mla_run(lib, ms, ld, ws, o, ldo, B, HW, heads, dim):
    lib.call("es3_litemla_attn_f32", ms.data_ptr(), ld, ws.data_ptr(), o.data_ptr(), ldo, B, HW, heads, dim, 1e-15, _st())


@pytest.mark.parametrize("dim,HW,heads,B,wide", MLA)
def test_litemla_attn_f32(cuda, dim, HW, heads, B, wide):
    """HW on both sides of every chunk boundary (one chunk up to 2048 pixels, then equal chunks), rows of ms and out wider than the
    heads, several images and heads; pixels whose q is all negative give exactly 0; the workspace is exactly the size
    es3_litemla_attn_f32_ws_floats reports and fully written; the last image alone; ops.litemla_attn_f32 bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "mla", dim, HW, heads, B, wide)
    C3 = 3 * dim * heads
    ld, ldo = (C3 + 12, dim * heads + 8) if wide else (C3, dim * heads)
    ms = torch.full((B * HW, ld), float("nan"), device=cuda)
    ms[:, :C3] = torch.randn(B * HW, C3, device=cuda, generator=g)
    dead = torch.arange(B * HW, device=cuda) % 7 == 3                          # pixels whose q is negative in every head
    for h in range(heads):
        ms[dead, 3 * dim * h:3 * dim * h + dim] = -ms[dead, 3 * dim * h:3 * dim * h + dim].abs() - 0.1
    n_ws = lib.size("es3_litemla_attn_f32_ws_floats", B, HW, heads, dim)
    chunk, nch = R.litemla_chunks(HW)
    assert n_ws == B * heads * nch * (dim + 1) * dim
    ws, ws_in = _flat_out(n_ws, torch.float32, cuda)
    buf, ins = _flat_out(B * HW * ldo, torch.float32, cuda)
    ins.view(-1)[:B * HW * ldo].view(B * HW, ldo)[:, dim * heads:] = False
    view = lambda b: b[:B * HW * ldo].view(B * HW, ldo)[:, :dim * heads]
    got = _twice(lambda b: _mla_run(lib, ms, ld, ws, b, ldo, B, HW, heads, dim), buf)
    what = f"litemla_attn_f32 dim{dim} HW{HW} heads{heads} B{B} wide={wide}"
    _assert_untouched(ws, ws_in, what + ": workspace past its reported size")
    assert not torch.isnan(ws[:n_ws]).any(), what + ": workspace not fully written"
    ref, bound = R.litemla_attn(ms[:, :C3].double(), B, HW, heads, dim, 1e-15)
    _check(f"2 litemla_attn_f32 dim{dim}" + (" multi-chunk" if nch > 1 else ""), view(got), ref, bound, what)
    assert (view(got)[dead] == 0).all(), what + ": a pixel with all-negative q is not exactly 0"
    _assert_untouched(got, ins, what)
    if B > 1:
        one = buf.clone()
        _mla_run(lib, ms[-HW:], ld, ws, one, ldo, 1, HW, heads, dim)
        _bits_equal(view(one)[:HW], view(got)[-HW:], what + ": last image alone")
    if not wide:
        H = next(h for h in range(int(HW ** 0.5), 0, -1) if HW % h == 0)
        _bits_equal(_ops().litemla_attn_f32(ms.view(B, H, HW // H, ld), heads, dim, 1e-15).view(B * HW, -1), view(got),
                    what + ": ops.litemla_attn_f32 vs direct")


# ----------------------------------------------------------------------------------------------------------- (3) bilinear
BIL = [  # B, Hi, Wi, C, Ho, Wo
    (2, 5, 7, 24, 5, 7), (3, 1, 1, 5, 1, 1), (1, 64, 64, 3, 64, 64),   # equal sizes: the layout change
    (2, 10, 10, 24, 12, 12), (1, 7, 13, 5, 20, 5), (2, 23, 23, 24, 9, 9), (3, 1, 1, 3, 6, 4), (2, 9, 1, 7, 1, 1),
    (2, 1, 9, 4, 4, 1), (1, 17, 3, 2, 1, 1), (2, 3, 17, 9, 31, 2),
    (2, 32, 32, 1024, 64, 64),                # the student head at 1024^2: the 32 x 32 feature map to embed_size 64
]


@pytest.mark.parametrize("B,Hi,Wi,C,Ho,Wo", BIL)
def test_bilinear_nhwc_f32_to_nchw(cuda, B, Hi, Wi, C, Ho, Wo):
    """Equal sizes bit-exact; up, down, non-square, 1 x 1 to n and n to 1 x 1 within 4u sum |w||v| plus the coordinate's ulp; the
    last image alone; ops.bilinear_nhwc_f32_to_nchw bit-identical."""
    lib = _lib(cuda)
    x = torch.randn(B, Hi, Wi, C, device=cuda, generator=_gen(cuda, "bil", B, Hi, Wi, C, Ho, Wo))
    n = B * C * Ho * Wo
    run = lambda b, xx=x, nb=B: lib.call("es3_bilinear_nhwc_f32_to_nchw", xx.data_ptr(), b.data_ptr(), nb, Hi, Wi, C, Ho, Wo, _st())
    buf, ins = _flat_out(n, torch.float32, cuda)
    got = _twice(run, buf)
    y = got[:n].view(B, C, Ho, Wo)
    what = f"bilinear_nhwc_f32_to_nchw B{B} {Hi}x{Wi} C{C} -> {Ho}x{Wo}"
    if (Hi, Wi) == (Ho, Wo):
        _bits_equal(y, x.permute(0, 3, 1, 2), what)
    else:
        ref, bound = R.bilinear(x.double(), Ho, Wo)
        _check("3 bilinear_nhwc_f32_to_nchw", y, ref, bound, what)
    _assert_untouched(got, ins, what)
    one = torch.full((C * Ho * Wo,), float("nan"), device=cuda)
    run(one, x[-1:], 1)
    _bits_equal(one.view(1, C, Ho, Wo), y[-1:], what + ": last image alone")
    _bits_equal(_ops().bilinear_nhwc_f32_to_nchw(x, Ho, Wo), y, what + ": ops.bilinear_nhwc_f32_to_nchw vs direct")


# ----------------------------------------------------------------------------------------------------------- (4) bias, act, residual
BAR = _pairwise(dict(act=[None, "relu", "hswish", "gelu", "sigmoid"], bias=[False, True], res=[False, True], after=[False, True],
                     shape=[(1003, 7), (4099, 64), (333, 1000), (70001, 160)]), seed=33)
BAR += [(None, False, False, False, (1024, 512)),      # strict.squeeze_excite's call with no argument: the pooled [B, C] copy
        ("gelu", True, False, False, (2 * 64 * 64 * 32, 32)),    # the SAM heads' strict output upscaling: ConvTranspose + bias + GELU
        ("gelu", True, True, True, (2 * 32 * 32 * 64, 64)),      # ... GELU after the high-res feature residual
        (None, True, False, False, (2 * 32 * 32 * 64, 64)),      # ConvTranspose + bias
        (None, True, True, False, (2 * 64 * 64 * 32, 32))]       # ... + residual


@pytest.mark.parametrize("act,bias,res,after,shape", BAR)
def test_bias_act_res_f32(cuda, act, bias, res, after, shape):
    """Every activation, bias and residual each present or absent, the activation before or after the residual; totals that are
    multiples of neither C nor 256; the copy it is without arguments bit for bit; the last rows alone; ops.bias_act_res_f32
    bit-identical."""
    lib = _lib(cuda)
    total, C = shape
    g = _gen(cuda, "bar", act, bias, res, after, shape)
    x = torch.randn(total, device=cuda, generator=g) * 3
    bi = torch.randn(C, device=cuda, generator=g) if bias else None
    r = torch.randn(total, device=cuda, generator=g) * 2 if res else None

    def run(b, lo=0):
        lib.call("es3_bias_act_res_f32", x[lo:].data_ptr(), _p(bi), 0 if r is None else r[lo:].data_ptr(), b.data_ptr(), total - lo, C,
                 ACT[act], int(after), _st())
    buf, ins = _flat_out(total, torch.float32, cuda)
    got = _twice(run, buf)
    what = f"bias_act_res_f32 total {total} C{C} act {act} bias={bias} res={res} after={after}"
    if act is None and not bias and not res:
        _bits_equal(got[:total], x, what + ": the copy")
    d = lambda t: None if t is None else t.double()
    ref, bound = R.bias_act_res(x.double(), d(bi), act, d(r), after)
    _check("4 bias_act_res_f32", got[:total], ref, bound, what)
    _assert_untouched(got, ins, what)
    lo = (total // C) * C                                                        # the partial last row of channels, on its own
    if 0 < lo < total:
        part = torch.full((total - lo + TAIL,), float("nan"), device=cuda)
        run(part, lo)
        _bits_equal(part[:total - lo], got[lo:total], what + ": the last rows alone")
    wx = x.view(-1, C) if total % C == 0 else x.view(1, -1)
    if total % C == 0 or not bias:
        _bits_equal(_ops().bias_act_res_f32(wx, bi, act, None if r is None else r.view(wx.shape), after).view(-1), got[:total],
                    what + ": ops.bias_act_res_f32 vs direct")


# ----------------------------------------------------------------------------------------------------------- (5) channel gate
SCH = [(2, 35, 13), (3, 1, 1), (1, 4096, 320), (2, 16384, 128), (3, 7, 161), (2, 1, 1024)]


@pytest.mark.parametrize("B,HW,C", SCH)
def test_scale_channels_f32(cuda, B, HW, C):
    """Bit-exact against torch's fp32 x * gate at ragged C and B > 1; the last image alone; ops.scale_channels_f32 bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "sch", B, HW, C)
    x, gate = torch.randn(B, HW, C, device=cuda, generator=g), torch.rand(B, C, device=cuda, generator=g)
    n = B * HW * C
    run = lambda b, xx=x, gg=gate, nb=B: lib.call("es3_scale_channels_f32", xx.data_ptr(), gg.data_ptr(), b.data_ptr(), nb, HW, C, _st())
    buf, ins = _flat_out(n, torch.float32, cuda)
    got = _twice(run, buf)
    what = f"scale_channels_f32 B{B} HW{HW} C{C}"
    _bits_equal(got[:n].view(B, HW, C), x * gate[:, None, :], what)
    _assert_untouched(got, ins, what)
    one = torch.full((HW * C,), float("nan"), device=cuda)
    run(one, x[-1:].contiguous(), gate[-1:].contiguous(), 1)
    _bits_equal(one, got[(B - 1) * HW * C:n], what + ": last image alone")
    _bits_equal(_ops().scale_channels_f32(x.view(B, 1, HW, C), gate).view(B, HW, C), got[:n].view(B, HW, C), what + ": ops vs direct")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    keys = {("es3_dwconv_f32", c[4], c[5], c[6], c[7], c[8]) for c in DW}
    keys |= {("es3_litemla_attn_f32", c[0], c[1] > 2048) for c in MLA}
    keys |= {("es3_bilinear_nhwc_f32_to_nchw", "same" if c[1:3] == c[4:6] else "resize") for c in BIL}
    keys |= {("es3_bias_act_res_f32", c[0], c[1], c[2], c[3]) for c in BAR}
    keys |= {("es3_scale_channels_f32",) for _ in SCH}
    return keys
