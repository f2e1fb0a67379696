"""The image students' forward kernels (mbconv_tc.cu, mbconv_tc_s2.cu, dwproj_tc.cu, dw_tc.cu, dw_tiled.cu, the
forward kernels of conv.cu, stem_fused.cu, litemla_tc.cu, litemla.cu, repvit_ops.cu, tinyvit_ops.cu), element by element against
the fp64 statements of tests/ref_fwd.py, each output element within its own bound.

Outputs are NaN-prefilled and called through _lib.call: every cell inside the output region must be written and lie within its
bound, every cell outside it (a flat TAIL, the channels past C of an ldo > C row, the channels of ms past 2 C3) keeps its
sentinel bits.  Workspaces (the LiteMLA KV partials, channel_mean's partials) are NaN-filled.  Strided operands are channel
slices of NaN-padded buffers.  Where an ops wrapper adds routing it is called too and must be bit-identical to the direct call.
Every persistent or tiled kernel runs twice and must be bit-identical, image i of a batch must be bit-identical to image i run
alone, and a shape an entry point declines (returns -1) writes nothing.  covered_keys() names the route keys (tests/routes.py)
the tables run, for the route closure of tests/test_route_closure_gpu.py.

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power
limit): fp32 outputs -- LiteMLA KV partials 0.0081 (generic) and 0.0015 (tensor core), channel_mean 0.0044, bilinear 0.0041;
bf16 outputs -- 0.95 ... 0.996 in every other section (depthwise, MBConv, dwproj, stems, aggreg, LiteMLA, LayerNorm, window
attention, scale_channels; LiteMLA tc 0.88), where the output's own rounding half-step dominates the bound and is reached.  The
whole file (319 tests, the route-closure forwards and training steps included, since moved to tests/test_route_closure_gpu.py) took
34 s there.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import ref_fwd as R
from bounds import (TAIL, _assert_untouched, _bf, _bits_equal, _check, _flat_out, _gen, _lib, _p, _pairwise, _st, _twice,
                    report_worst)
from routes import dw_tc_key, ln_key

pytestmark = pytest.mark.gpu
_report_worst = report_worst("fwd kernels")
ACT = {None: 0, "relu": 1, "hswish": 2, "gelu": 3}
ACTS = [None, "relu", "hswish", "gelu"]


def _out4(B, H, W, C, ld, dtype, cuda):
    """A NaN buffer of B H W ld + TAIL cells; returns (buffer, [B, H, W, C] view at channel 0 with pixel stride ld, inside-mask)."""
    buf = torch.full((B * H * W * ld + TAIL,), float("nan"), dtype=dtype, device=cuda)
    view = buf[:B * H * W * ld].view(B, H, W, ld)[..., :C]
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=cuda)
    inside[:B * H * W * ld].view(B, H, W, ld)[..., :C] = True
    return buf, view, inside


def _slice(x, extra):
    """x [..., C] as channels [8, 8 + C) of a NaN-padded [..., C + extra] buffer (extra = 0: x itself)."""
    if extra == 0:
        return x.contiguous()
    big = torch.full(x.shape[:-1] + (x.shape[-1] + extra,), float("nan"), dtype=x.dtype, device=x.device)
    big[..., 8:8 + x.shape[-1]] = x
    return big[..., 8:8 + x.shape[-1]]


def _taps(lib, w):
    out = torch.full_like(w, float("nan"))
    lib.call("es3_round_taps_sum_bf16", w.data_ptr(), out.data_ptr(), w.shape[0], w.shape[1], _st())
    return out


# ----------------------------------------------------------------------------------------------------------- (1) round_taps
@pytest.mark.parametrize("KK,C", [(9, 64), (9, 160), (25, 96), (25, 1000), (9, 1)])
def test_round_taps_bit_exact(cuda, KK, C):
    """es3_round_taps_sum_bf16 against its host emulation, bit for bit, plus the three properties the depthwise kernels rely on."""
    g = _gen(cuda, "taps", KK, C)
    w = torch.randn(KK, C, device=cuda, generator=g) / KK
    got = _taps(_lib(cuda), w)
    emu = R.round_taps_sum_emu(w)
    _bits_equal(got.cpu(), emu, "round_taps vs its emulation")
    near = w.to(torch.bfloat16).float()
    assert torch.equal(got, got.to(torch.bfloat16).float())
    assert ((got - near).abs() <= 1.01 * near.abs() * 2.0 ** -7).all()
    assert ((got.double().sum(0) - w.double().sum(0)).abs() <= (near.double().sum(0) - w.double().sum(0)).abs() + 1e-7).all()


# ----------------------------------------------------------------------------------------------------------- (2) depthwise
def _dw_case(cuda, fn, ks, stride, C, act, bias, sliced, B, H, W, tag, taps=False):
    lib = _lib(cuda)
    g = _gen(cuda, tag, ks, stride, C, act, bias, sliced, B, H, W)
    x = _slice(_bf(torch.randn(B, H, W, C, device=cuda, generator=g)), 16 if sliced else 0)
    w = torch.randn(ks * ks, C, device=cuda, generator=g) / ks
    b = torch.randn(C, device=cuda, generator=g) if bias else None
    wk = _taps(lib, w) if taps else w
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    ldo = C + 24 if sliced else C
    buf, view, inside = _out4(B, Ho, Wo, C, ldo, torch.bfloat16, cuda)
    if fn == "es3_dwconv_tc_bf16":
        args = lambda o: (x.data_ptr(), x.stride(2), wk.data_ptr(), _p(b), o.data_ptr(), ldo, B, H, W, C, ks, ACT[act], _st())
    else:
        args = lambda o: (x.data_ptr(), x.stride(2), wk.data_ptr(), _p(b), o.data_ptr(), ldo, B, H, W, C, ks, stride, ACT[act], _st())
    got = _twice(lambda o: lib.call(fn, *args(o)), buf)
    ref, bound = R.dwconv(x.double(), wk.double(), None if b is None else b.double(), ks, stride, act)
    what = f"{fn} ks{ks} s{stride} C{C} {act} bias={bias} sliced={sliced} B{B} {H}x{W}"
    v = got[:B * Ho * Wo * ldo].view(B, Ho, Wo, ldo)[..., :C]
    _check(f"2 {fn}", v, ref, bound, what)
    _assert_untouched(got, inside, what)
    return x, w, b, v


DWTC_FACTORS = dict(kc=[(3, 128), (3, 96), (3, 160), (5, 64), (5, 96)], act=ACTS, bias=[True, False], sliced=[False, True],
                    geo=[(2, 8, 32), (1, 9, 33), (3, 1, 1), (2, 17, 5), (1, 64, 64), (5, 7, 31)])
DWTC = _pairwise(DWTC_FACTORS, seed=1)


@pytest.mark.parametrize("kc,act,bias,sliced,geo", DWTC)
def test_dwconv_tc(cuda, kc, act, bias, sliced, geo):
    """ks 3 with CG 64 (C % 64 == 0) and CG 32 (96, 160), ks 5; four activations; bias present and absent; channel slices for x and
    out; 8 x 32 tiles ragged; the taps es3_round_taps_sum_bf16 makes.  ops.dwconv (which prepares the same taps) is bit-identical."""
    ks, C = kc
    x, w, b, v = _dw_case(cuda, "es3_dwconv_tc_bf16", ks, 1, C, act, bias, sliced, *geo, "dwtc", taps=True)
    from efficientsam3_b200 import ops
    _bits_equal(ops.dwconv(x, w.clone(), b, ks, 1, act), v, "ops.dwconv vs the direct call")


DWT = _pairwise(dict(C=[32, 96], act=ACTS, bias=[True, False], sliced=[False, True],
                     geo=[(2, 9, 67), (1, 8, 64), (3, 3, 1), (1, 17, 130), (2, 2, 2)]), seed=2)


@pytest.mark.parametrize("C,act,bias,sliced,geo", DWT)
def test_dwconv_tiled(cuda, C, act, bias, sliced, geo):
    """ks 3 stride 2, Wo ragged against TW = 32 and Ho against TH = 4; ops.dwconv routes here and is bit-identical."""
    x, w, b, v = _dw_case(cuda, "es3_dwconv_tiled_bf16", 3, 2, C, act, bias, sliced, *geo, "dwt")
    from efficientsam3_b200 import ops
    _bits_equal(ops.dwconv(x, w, b, 3, 2, act), v, "ops.dwconv vs the direct call")


DWG = _pairwise(dict(kst=[(3, 1), (3, 2), (5, 1)], act=ACTS, C=[8, 24, 40, 48], sliced=[False, True],
                     geo=[(2, 9, 7), (1, 1, 1), (3, 16, 5)]), seed=3)


@pytest.mark.parametrize("kst,act,C,sliced,geo", DWG)
def test_dwconv_generic(cuda, kst, act, C, sliced, geo):
    """One thread per 8 output channels: (3, 1), (3, 2), (5, 1) x activations, C not a multiple of 32."""
    _dw_case(cuda, "es3_dwconv_bf16", kst[0], kst[1], C, act, True, sliced, *geo, "dwg")


# ----------------------------------------------------------------------------------------------------------- (3) MBConv
def _mb_weights(cuda, cin, mid, cout, g):
    w1 = _bf(torch.randn(mid, cin, device=cuda, generator=g) / math.sqrt(cin))
    s1, b1 = torch.rand(mid, device=cuda, generator=g) + 0.5, torch.randn(mid, device=cuda, generator=g) * 0.2
    wdw, b2 = torch.randn(9, mid, device=cuda, generator=g) / 3, torch.randn(mid, device=cuda, generator=g) * 0.2
    w3 = _bf(torch.randn(cout, mid, device=cuda, generator=g) / math.sqrt(mid))
    s3, b3 = torch.rand(cout, device=cuda, generator=g) + 0.5, torch.randn(cout, device=cuda, generator=g) * 0.2
    return w1, s1, b1, wdw, b2, w3, s3, b3


def _mb_call(lib, x, y, wt, taps, cin, mid, cout, stride, res, act="hswish"):
    w1, s1, b1, _, b2, w3, s3, b3 = wt
    B, H, W = x.shape[:3]
    return lib.call_rc("es3_mbconv_bf16", x.data_ptr(), y.data_ptr(), w1.data_ptr(), s1.data_ptr(), b1.data_ptr(), taps.data_ptr(),
                       b2.data_ptr(), w3.data_ptr(), s3.data_ptr(), b3.data_ptr(), B, H, W, cin, mid, cout, stride, int(res), ACT[act],
                       _st())


def _mb_case(cuda, cin, mid, cout, stride, B, H, W):
    lib = _lib(cuda)
    g = _gen(cuda, "mb", cin, mid, cout, stride, B, H, W)
    x = _bf(torch.randn(B, H, W, cin, device=cuda, generator=g))
    wt = _mb_weights(cuda, cin, mid, cout, g)
    taps = _taps(lib, wt[3])
    res = stride == 1
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    buf, inside = _flat_out(B * Ho * Wo * cout, torch.bfloat16, cuda)

    def run(o):
        assert _mb_call(lib, x, o, wt, taps, cin, mid, cout, stride, res) == 0
    got = _twice(run, buf)
    y = got[:B * Ho * Wo * cout].view(B, Ho, Wo, cout)
    w1, s1, b1, _, b2, w3, s3, b3 = (t.double() for t in wt)
    ref, bound, _, _ = R.mbconv(x.double(), w1, s1, b1, taps.double(), b2, w3, s3, b3, stride, res)
    what = f"es3_mbconv_bf16 ({cin},{mid},{cout},s{stride}) B{B} {H}x{W}"
    _check(f"3 es3_mbconv_bf16 s{stride}", y, ref, bound, what)
    _assert_untouched(got, inside, what)
    from efficientsam3_b200 import ops
    _bits_equal(ops.mbconv_fused(x, *wt[:3], wt[3].clone(), *wt[4:], stride, res, "hswish"), y, "ops.mbconv_fused vs direct")
    return x, wt, taps, y


GEO = {1: [(2, 3, 5), (2, 1, 37), (2, 1, 1), (2, 17, 33), (2, 9, 17), (2, 7, 15), (1, 8, 16), (24, 37, 37)],
       2: [(2, 3, 5), (2, 1, 37), (2, 1, 1), (2, 17, 33), (2, 18, 34), (2, 7, 31), (1, 8, 32), (40, 37, 37)]}
# Cin 128 (input tile held as two 64-channel slabs): 1 x 1, below one tile, one tile (stride 1: 8 x 16 output, stride 2: 8 x 32
# input) and one pixel past it, the ragged 63 x 63 that 1008-px inputs give, and the EV-M shape of bench.py (64 x 64 at batch 32)
GEO_CIN128 = {1: [(2, 1, 1), (2, 3, 5), (2, 1, 37), (1, 8, 16), (2, 7, 15), (2, 9, 17), (2, 63, 63), (32, 64, 64)],
              2: [(2, 1, 1), (2, 3, 5), (2, 1, 37), (1, 8, 32), (2, 7, 31), (2, 10, 34), (2, 63, 63), (32, 64, 64)]}
MB_TC = [(32, 128, 32, 1), (64, 256, 64, 1), (128, 512, 128, 1)]
MB_S2 = [(16, 64, 32, 2), (32, 128, 64, 2), (64, 256, 128, 2), (128, 512, 256, 2)]


def _mb_rows(blocks):
    return [blk + geo for blk in blocks for geo in (GEO_CIN128 if blk[0] == 128 else GEO)[blk[3]]]


@pytest.mark.parametrize("cin,mid,cout,stride,B,H,W", _mb_rows(MB_TC))
def test_mbconv_tc(cuda, cin, mid, cout, stride, B, H, W):
    """The wgmma stride-1 residual kernel, 8 x 16 tiles: one-pixel edge tiles, images below one tile, and batches large enough that
    every persistent CTA runs tiles of several images (the rows of the former tile-geometry test, under per-element bounds)."""
    _mb_case(cuda, cin, mid, cout, stride, B, H, W)


@pytest.mark.parametrize("cin,mid,cout,stride,B,H,W", _mb_rows(MB_S2))
def test_mbconv_tc_s2(cuda, cin, mid, cout, stride, B, H, W):
    """The wgmma stride-2 kernel, 4 x 16 tiles over 9 x 33 input tiles: the expand rows past S2_PIN of the last 64-row block go to
    the scratch slot; W = 33 / 34 / 37 put real pixels in the last input column of a tile."""
    _mb_case(cuda, cin, mid, cout, stride, B, H, W)


@pytest.mark.parametrize("blk", MB_TC + MB_S2)
def test_mbconv_batch_invariant(cuda, blk):
    """Image i of a batch is bit-identical to image i run alone (state leaking between the tiles of a persistent CTA would not be)."""
    B = 24 if blk[3] == 1 else 40
    x, wt, taps, y = _mb_case(cuda, *blk, B, 37, 37)
    lib = _lib(cuda)
    for i in (0, B // 2, B - 1):
        one = torch.full_like(y[i:i + 1], float("nan"))
        assert _mb_call(lib, x[i:i + 1].contiguous(), one, wt, taps, *blk, blk[3] == 1) == 0
        _bits_equal(one[0], y[i], f"es3_mbconv_bf16 {blk} image {i} of {B} vs alone")


# Shapes es3_mbconv_bf16 declines: uninstantiated blocks, instantiated blocks at the other stride or residual setting, and every
# instantiated block with an activation other than hardswish
MB_DECLINED = [((48, 192, 48, 1), True, "hswish"), ((32, 128, 32, 2), False, "hswish"), ((64, 256, 64, 2), False, "hswish"),
               ((256, 1024, 256, 1), True, "hswish"), ((128, 256, 128, 1), True, "hswish"), ((128, 512, 128, 2), False, "hswish"),
               ((128, 512, 256, 1), True, "hswish"), ((32, 128, 32, 1), False, "hswish"), ((128, 512, 128, 1), False, "hswish"),
               ((128, 512, 256, 2), True, "hswish")]
MB_DECLINED += [(blk, blk[3] == 1, (None, "relu", "gelu")[i % 3]) for i, blk in enumerate(MB_TC + MB_S2)]


@pytest.mark.parametrize("blk,res,act", MB_DECLINED)
def test_mbconv_declined_shapes_write_nothing(cuda, blk, res, act):
    lib = _lib(cuda)
    cin, mid, cout, stride = blk
    g = _gen(cuda, "decl", blk, res, act)
    x = _bf(torch.randn(1, 9, 9, cin, device=cuda, generator=g))
    wt = _mb_weights(cuda, cin, mid, cout, g)
    buf, inside = _flat_out(81 * cout, torch.bfloat16, cuda)
    assert _mb_call(lib, x, buf, wt, wt[3], cin, mid, cout, stride, res, act) == -1
    torch.cuda.synchronize()
    _assert_untouched(buf, torch.zeros_like(inside), f"es3_mbconv_bf16 declined {blk} residual={res} act={act}")


DWP = [(mid, cout, res, geo) for mid, cout in ((512, 128), (1024, 256)) for res in (True, False)
       for geo in ((1, 64, 64), (2, 32, 32), (2, 9, 17), (1, 1, 1), (3, 13, 7))]


@pytest.mark.parametrize("mid,cout,res,geo", DWP)
def test_dwproj_tc(cuda, mid, cout, res, geo):
    """Depthwise + projection on wgmma, both instantiations, with and without residual, EfficientViT-B1's 1024^2 stage-3 / stage-4
    maps (64^2, 32^2) and ragged maps against the 8 x 16 tile; ops.dwproj is bit-identical."""
    lib = _lib(cuda)
    B, H, W = geo
    g = _gen(cuda, "dwp", mid, cout, res, geo)
    m = _bf(torch.randn(B, H, W, mid, device=cuda, generator=g))
    wdw, b2 = torch.randn(9, mid, device=cuda, generator=g) / 3, torch.randn(mid, device=cuda, generator=g) * 0.2
    w3 = _bf(torch.randn(cout, mid, device=cuda, generator=g) / math.sqrt(mid))
    s3, b3 = torch.rand(cout, device=cuda, generator=g) + 0.5, torch.randn(cout, device=cuda, generator=g) * 0.2
    r = _bf(torch.randn(B, H, W, cout, device=cuda, generator=g)) if res else None
    taps = _taps(lib, wdw)
    buf, inside = _flat_out(B * H * W * cout, torch.bfloat16, cuda)

    def run(o):
        assert lib.call_rc("es3_dwproj_tc_bf16", m.data_ptr(), taps.data_ptr(), b2.data_ptr(), w3.data_ptr(), s3.data_ptr(), b3.data_ptr(),
                           _p(r), o.data_ptr(), B, H, W, mid, cout, ACT["hswish"], _st()) == 0
    got = _twice(run, buf)
    y = got[:B * H * W * cout].view(B, H, W, cout)
    ref, bound = R.dwproj(m.double(), taps.double(), b2.double(), w3.double(), s3.double(), b3.double(), None if r is None else r.double())
    what = f"dwproj ({mid},{cout}) res={res} B{B} {H}x{W}"
    _check("3 dwproj_tc", y, ref, bound, what)
    _assert_untouched(got, inside, what)
    from efficientsam3_b200 import ops
    _bits_equal(ops.dwproj(m, wdw.clone(), b2, w3, s3, b3, r), y, "ops.dwproj vs direct")
    if B > 1:
        one = torch.full_like(y[-1:], float("nan"))
        lib.call_rc("es3_dwproj_tc_bf16", m[-1:].data_ptr(), taps.data_ptr(), b2.data_ptr(), w3.data_ptr(), s3.data_ptr(), b3.data_ptr(),
                    _p(None if r is None else r[-1:]), one.data_ptr(), 1, H, W, mid, cout, ACT["hswish"], _st())
        _bits_equal(one[0], y[-1], "dwproj last image vs alone")


def test_dwproj_declined_shape_writes_nothing(cuda):
    lib = _lib(cuda)
    m = torch.zeros(1, 8, 8, 256, device=cuda, dtype=torch.bfloat16)
    z = torch.zeros(9 * 256, device=cuda)
    w3 = torch.zeros(64, 256, device=cuda, dtype=torch.bfloat16)
    buf, inside = _flat_out(64 * 64, torch.bfloat16, cuda)
    assert lib.call_rc("es3_dwproj_tc_bf16", m.data_ptr(), z.data_ptr(), z.data_ptr(), w3.data_ptr(), z.data_ptr(), z.data_ptr(), 0,
                       buf.data_ptr(), 1, 8, 8, 256, 64, ACT["hswish"], _st()) == -1
    torch.cuda.synchronize()
    _assert_untouched(buf, torch.zeros_like(inside), "dwproj declined (256, 64)")


# ----------------------------------------------------------------------------------------------------------- (4) stems
STEM = _pairwise(dict(Cout=[8, 16, 24, 32, 48], act=ACTS, geo=[(2, 13, 9), (1, 1, 1), (3, 32, 31), (1, 65, 64)]), seed=4)


@pytest.mark.parametrize("Cout,act,geo", STEM)
def test_stem_conv3x3_s2(cuda, Cout, act, geo):
    lib = _lib(cuda)
    B, H, W = geo
    g = _gen(cuda, "stem", Cout, act, geo)
    img = torch.randn(B, 3, H, W, device=cuda, generator=g)
    w27, bias = torch.randn(27, Cout, device=cuda, generator=g) / 5, torch.randn(Cout, device=cuda, generator=g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    buf, inside = _flat_out(B * Ho * Wo * Cout, torch.bfloat16, cuda)
    lib.call("es3_stem_conv3x3_s2", img.data_ptr(), w27.data_ptr(), bias.data_ptr(), buf.data_ptr(), B, H, W, Cout, ACT[act], _st())
    ref, bound = R.stem_conv(img.double(), w27.double(), bias.double(), act)
    what = f"stem Cout{Cout} {act} B{B} {H}x{W}"
    _check("4 stem_conv3x3_s2", buf[:B * Ho * Wo * Cout].view(B, Ho, Wo, Cout), ref, bound, what)
    _assert_untouched(buf, inside, what)


DSC = _pairwise(dict(C=[8, 16, 24, 32], act=ACTS, bias=[True, False], geo=[(2, 7, 5), (1, 1, 1), (2, 33, 17)]), seed=5)


@pytest.mark.parametrize("C,act,bias,geo", DSC)
def test_dsconv_res(cuda, C, act, bias, geo):
    lib = _lib(cuda)
    B, H, W = geo
    g = _gen(cuda, "dsc", C, act, bias, geo)
    x = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    wd, wp = torch.randn(9, C, device=cuda, generator=g) / 3, torch.randn(C, C, device=cuda, generator=g) / 4
    bd = torch.randn(C, device=cuda, generator=g) if bias else None
    bp = torch.randn(C, device=cuda, generator=g) if bias else None
    buf, inside = _flat_out(B * H * W * C, torch.bfloat16, cuda)
    lib.call("es3_dsconv_res_bf16", x.data_ptr(), wd.data_ptr(), _p(bd), wp.data_ptr(), _p(bp), buf.data_ptr(), B, H, W, C, ACT[act], _st())
    ref, bound = R.dsconv_res(x.double(), wd.double(), None if bd is None else bd.double(), wp.double(),
                              None if bp is None else bp.double(), act)
    what = f"dsconv_res C{C} {act} bias={bias} B{B} {H}x{W}"
    _check("4 dsconv_res", buf[:B * H * W * C].view(B, H, W, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


@pytest.mark.parametrize("B,H,W", [(2, 30, 66), (1, 16, 64), (2, 17, 65), (1, 2, 2), (3, 1, 1), (1, 1024, 1024)])
def test_stem_fused_c16(cuda, B, H, W):
    """x1 = bf16(hswish(s0 conv3x3_s2(bf16(img); w0) + b0)), y = x1 + spw pw(bf16(hswish(dw3x3(x1) + bdw)); wpw) + bpw, over the
    8 x 32 output tiles (edges at Ho, Wo = 8 / 32 +- 1, odd sizes, 1024^2).  The kernel's MMA takes the image as bf16."""
    lib = _lib(cuda)
    g = _gen(cuda, "sf", B, H, W)
    img = torch.randn(B, 3, H, W, device=cuda, generator=g)
    w0 = torch.zeros(16, 32, device=cuda)
    w0[:, :27] = torch.randn(16, 27, device=cuda, generator=g) / 5
    w0 = _bf(w0)
    s0, b0 = torch.rand(16, device=cuda, generator=g) + 0.5, torch.randn(16, device=cuda, generator=g) * 0.2
    wdw, bdw = torch.randn(9, 16, device=cuda, generator=g) / 3, torch.randn(16, device=cuda, generator=g) * 0.2
    wpw = _bf(torch.randn(16, 16, device=cuda, generator=g) / 4)
    spw, bpw = torch.rand(16, device=cuda, generator=g) + 0.5, torch.randn(16, device=cuda, generator=g) * 0.2
    taps = _taps(lib, wdw)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    buf, inside = _flat_out(B * Ho * Wo * 16, torch.bfloat16, cuda)
    got = _twice(lambda o: lib.call("es3_stem_fused_c16", img.data_ptr(), w0.data_ptr(), s0.data_ptr(), b0.data_ptr(), taps.data_ptr(),
                                    bdw.data_ptr(), wpw.data_ptr(), spw.data_ptr(), bpw.data_ptr(), o.data_ptr(), B, H, W, _st()), buf)
    ref, bound = R.stem_fused(img.to(torch.bfloat16).double(), w0.double(), s0.double(), b0.double(), taps.double(), bdw.double(),
                              wpw.double(), spw.double(), bpw.double())
    what = f"stem_fused B{B} {H}x{W}"
    _check("4 stem_fused_c16", got[:B * Ho * Wo * 16].view(B, Ho, Wo, 16), ref, bound, what)
    _assert_untouched(got, inside, what)


NARROW = [(cin, cout, act, geo) for (cin, cout) in ((32, 32), (32, 48), (32, 64), (48, 80), (48, 96)) for act in (None, "gelu")
          for geo in ((2, 33, 50), (1, 1, 1))] + [(32, 64, None, (1, 64, 64)), (48, 96, "gelu", (3, 63, 41))]


@pytest.mark.parametrize("cin,cout,act,geo", NARROW)
def test_conv3x3_s2_narrow(cuda, cin, cout, act, geo):
    lib = _lib(cuda)
    B, H, W = geo
    g = _gen(cuda, "narrow", cin, cout, act, geo)
    x = _bf(torch.randn(B, H, W, cin, device=cuda, generator=g))
    w9 = _bf(torch.randn(9, cout, cin, device=cuda, generator=g) / 17)
    sc, bi = torch.rand(cout, device=cuda, generator=g) + 0.5, torch.randn(cout, device=cuda, generator=g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    buf, inside = _flat_out(B * Ho * Wo * cout, torch.bfloat16, cuda)
    got = _twice(lambda o: lib.call("es3_conv3x3_s2_narrow_bf16", x.data_ptr(), w9.data_ptr(), sc.data_ptr(), bi.data_ptr(), o.data_ptr(),
                                    B, H, W, cin, cout, ACT[act], _st()), buf)
    ref, bound = R.conv3x3_s2_narrow(x.double(), w9.double(), sc.double(), bi.double(), act)
    what = f"conv3x3_s2_narrow ({cin},{cout}) {act} B{B} {H}x{W}"
    _check("4 conv3x3_s2_narrow", got[:B * Ho * Wo * cout].view(B, Ho, Wo, cout), ref, bound, what)
    _assert_untouched(got, inside, what)


# ----------------------------------------------------------------------------------------------------------- (5) LiteMLA
@pytest.mark.parametrize("C3,H,W,extra", [(48, 16, 32, 0), (96, 17, 33, 16), (192, 1, 1, 0), (48, 15, 31, 8), (96, 40, 70, 24),
                                          (384, 32, 32, 0)])
def test_litemla_aggreg_dwpw(cuda, C3, H, W, extra):
    """dw5x5 on diagonal MMAs (bf16 taps of litemla_dwpw_weights), its bf16 result into the grouped 16 x 16 pointwise; writes channels
    [C3, 2 C3) of ms only: channels [0, C3) and past 2 C3 keep their bits."""
    lib = _lib(cuda)
    from efficientsam3_b200 import ops
    B = 2
    ld = 2 * C3 + extra
    g = _gen(cuda, "agg", C3, H, W, extra)
    ms = torch.full((B * H * W * ld + TAIL,), float("nan"), dtype=torch.bfloat16, device=cuda)
    msv = ms[:B * H * W * ld].view(B, H, W, ld)
    msv[..., :C3] = _bf(torch.randn(B, H, W, C3, device=cuda, generator=g))
    wdw, wpw = torch.randn(25, C3, device=cuda, generator=g) / 5, torch.randn(C3, 16, device=cuda, generator=g) / 4
    wd, wp = ops.litemla_dwpw_weights(wdw, wpw)
    before = ms.clone()
    lib.call("es3_litemla_aggreg_dwpw", ms.data_ptr(), ld, wd.data_ptr(), wp.data_ptr(), B, H, W, C3, _st())
    again = before.clone()
    lib.call("es3_litemla_aggreg_dwpw", again.data_ptr(), ld, wd.data_ptr(), wp.data_ptr(), B, H, W, C3, _st())
    _bits_equal(ms, again, "aggreg twice")
    taps = wd.double().permute(1, 0, 2).reshape(25, C3)
    ref, bound = R.litemla_aggreg(msv.double(), taps, wp.double(), C3)
    what = f"aggreg C3 {C3} {H}x{W} ld {ld}"
    _check("5 litemla_aggreg", msv[..., C3:2 * C3], ref, bound, what)
    inside = torch.zeros(ms.shape, dtype=torch.bool, device=cuda)
    inside[:B * H * W * ld].view(B, H, W, ld)[..., C3:2 * C3] = True
    changed = (ms.view(torch.int16) != before.view(torch.int16)) & ~inside
    assert int(changed.sum()) == 0, f"{what}: cells outside channels [C3, 2 C3) were written"


def _litemla_case(cuda, fn, dim, heads2, B, HW, extra, chunk, split):
    lib = _lib(cuda)
    g = _gen(cuda, fn, dim, heads2, B, HW, extra)
    ld = 3 * dim * heads2 + extra
    ms = torch.full((B, HW, ld), float("nan"), dtype=torch.bfloat16, device=cuda)
    ms[..., :3 * dim * heads2] = _bf(torch.randn(B, HW, 3 * dim * heads2, device=cuda, generator=g))
    nch = (HW + chunk - 1) // chunk
    ws_n = lib.size("es3_litemla_ws_floats", B, HW, heads2) if fn == "es3_litemla_attn_tc" else \
        lib.size("es3_litemla_generic_ws_floats", B, HW, heads2, dim)
    assert ws_n == B * heads2 * nch * (dim + 1) * dim
    ldo = dim * heads2 + (8 if extra else 0)
    buf, view, inside = _out4(B, HW, 1, dim * heads2, ldo, torch.bfloat16, cuda)
    wss = []

    def run(o):
        ws = torch.full((ws_n,), float("nan"), device=cuda)
        args = (ms.data_ptr(), ld, ws.data_ptr(), o.data_ptr(), ldo, B, HW, heads2) + ((dim,) if fn != "es3_litemla_attn_tc" else ())
        lib.call(fn, *args, 1e-15, _st())
        wss.append(ws)
    got = _twice(run, buf)
    _bits_equal(wss[0], wss[1], "KV partials twice")
    (y, yb), (part, pb) = R.litemla_attn(ms.double(), heads2, dim, 1e-15, chunk, split)
    what = f"{fn} dim{dim} heads2 {heads2} B{B} HW{HW} ld+{extra}"
    _check(f"5 {fn}", got[:B * HW * ldo].view(B, HW, ldo)[..., :dim * heads2], y, yb, what)
    _assert_untouched(got, inside, what)
    _check(f"5 {fn} KV partials", wss[0].view(B, heads2, nch, dim + 1, dim), part, pb, what + " partials")


@pytest.mark.parametrize("HW,heads2,B,extra", [(1, 2, 1, 0), (511, 4, 2, 16), (512, 2, 1, 0), (513, 2, 3, 8), (1025, 4, 1, 0),
                                               (4096, 8, 2, 0), (4096, 32, 1, 48)])
def test_litemla_attn_tc(cuda, HW, heads2, B, extra):
    """KV over 512-pixel chunks (HW around the chunk), the hi + lo apply; the KV partials the backward consumes against their fp64
    sums.  (4096, 32): efficientvit_b1's stage-4 LiteMLA at 1024^2 (heads2 = 2 x 16)."""
    _litemla_case(cuda, "es3_litemla_attn_tc", 16, heads2, B, HW, extra, 512, True)


@pytest.mark.parametrize("dim,HW,heads2,B,extra", [(16, 1, 2, 1, 0), (16, 127, 2, 2, 8), (16, 128, 3, 1, 0), (32, 129, 2, 2, 16),
                                                   (32, 300, 4, 1, 0), (32, 1024, 8, 2, 8)])
def test_litemla_attn_generic(cuda, dim, HW, heads2, B, extra):
    """The CUDA-core form for head dim 16 | 32, HW around the 128-pixel chunk."""
    _litemla_case(cuda, "es3_litemla_attn_generic", dim, heads2, B, HW, extra, 128, False)


# ----------------------------------------------------------------------------------------------------------- (6) SE, LayerNorm, windows
@pytest.mark.parametrize("B,HW,C", [(1, 1, 16), (2, 127, 40), (3, 128, 96), (2, 129, 2560), (1, 1000, 320), (2, 4096, 48)])
def test_channel_mean_scale_channels(cuda, B, HW, C):
    lib = _lib(cuda)
    g = _gen(cuda, "se", B, HW, C)
    x = _bf(torch.randn(B, HW, C, device=cuda, generator=g) + 0.5)
    nch = (HW + 127) // 128
    mean, mins = _flat_out(B * C, torch.float32, cuda)

    def run(o):
        ws = torch.full((B * nch * C,), float("nan"), device=cuda)
        lib.call("es3_channel_mean", x.data_ptr(), ws.data_ptr(), o.data_ptr(), B, HW, C, _st())
    got = _twice(run, mean)
    ref, bound = R.channel_mean(x.double())
    _check("6 channel_mean", got[:B * C].view(B, C), ref, bound, f"channel_mean B{B} HW{HW} C{C}")
    _assert_untouched(got, mins, "channel_mean")
    gate = torch.rand(B, C, device=cuda, generator=g) * 2
    y, yins = _flat_out(B * HW * C, torch.bfloat16, cuda)
    lib.call("es3_scale_channels", x.data_ptr(), gate.data_ptr(), y.data_ptr(), B, HW, C, _st())
    ref, bound = R.scale_channels(x.double(), gate.double())
    _check("6 scale_channels", y[:B * HW * C].view(B, HW, C), ref, bound, f"scale_channels B{B} HW{HW} C{C}")
    _assert_untouched(y, yins, "scale_channels")
    from efficientsam3_b200 import ops
    _bits_equal(ops.channel_mean(x.view(B, HW, 1, C)), got[:B * C].view(B, C), "ops.channel_mean vs direct")


LN = _pairwise(dict(C=[8, 64, 72, 128, 136, 448, 1024], M=[1, 33, 257, 1000], shift=[0.0, 30.0]), seed=6)


@pytest.mark.parametrize("C,M,shift", LN)
def test_layernorm_bf16(cuda, C, M, shift):
    """All three lane-group templates (C / 8 <= 8, <= 16, <= 128: 448 and 1024 included), M not a multiple of the rows per block,
    mean-shifted rows (|mean| >> std)."""
    lib = _lib(cuda)
    g = _gen(cuda, "ln", C, M, shift)
    x = _bf(torch.randn(M, C, device=cuda, generator=g) + shift)
    gm, bt = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    buf, inside = _flat_out(M * C, torch.bfloat16, cuda)
    lib.call("es3_layernorm_bf16", x.data_ptr(), gm.data_ptr(), bt.data_ptr(), 1e-5, buf.data_ptr(), M, C, _st())
    ref, bound = R.layernorm(x.double(), gm.double(), bt.double(), 1e-5)
    what = f"layernorm C{C} M{M} shift {shift}"
    _check("6 layernorm_bf16", buf[:M * C].view(M, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


WIN = [(1, 14, 14, 2, 7), (2, 9, 16, 4, 7), (3, 21, 7, 1, 7), (1, 14, 14, 2, 14), (2, 20, 15, 3, 14), (1, 28, 28, 10, 14),
       (2, 64, 64, 5, 14), (1, 1, 1, 2, 14)]


@pytest.mark.parametrize("B,H,W,heads,ws", WIN)
def test_win_attn_bias(cuda, B, H, W, heads, ws):
    """ws 7 (NT16 = 4, fp32 bias from global memory) and ws 14 (persistent, the head's bias table in shared memory as fp16 -- the
    reference takes the same fp16 values); padded windows; |bias| up to ~8; B nWin below the per-head CTA count.  Run twice."""
    lib = _lib(cuda)
    g = _gen(cuda, "win", B, H, W, heads, ws)
    C = 32 * heads
    qkv = _bf(torch.randn(B * H * W, 3 * C, device=cuda, generator=g))
    pad = _bf(torch.randn(3 * C, device=cuda, generator=g))
    bias = (torch.rand(heads, ws * ws, ws * ws, device=cuda, generator=g) * 2 - 1) * 8
    buf, inside = _flat_out(B * H * W * C, torch.bfloat16, cuda)
    got = _twice(lambda o: lib.call("es3_win_attn_bias_bf16", qkv.data_ptr(), pad.data_ptr(), bias.data_ptr(), o.data_ptr(), B, H, W, C,
                                    heads, ws, 32 ** -0.5, _st()), buf)
    used = bias.half().double() if ws == 14 else bias.double()
    ref, bound = R.win_attn_bias(qkv.double(), pad.double(), used, B, H, W, C, heads, ws, 32 ** -0.5)
    what = f"win_attn_bias B{B} {H}x{W} heads{heads} ws{ws}"
    _check(f"6 win_attn_bias ws{ws}", got[:B * H * W * C].view(B * H * W, C), ref, bound, what)
    _assert_untouched(got, inside, what)
    if B > 1:
        one = torch.full((H * W * C,), float("nan"), dtype=torch.bfloat16, device=cuda)
        lib.call("es3_win_attn_bias_bf16", qkv[-H * W:].data_ptr(), pad.data_ptr(), bias.data_ptr(), one.data_ptr(), 1, H, W, C, heads, ws,
                 32 ** -0.5, _st())
        _bits_equal(one, got[(B - 1) * H * W * C:B * H * W * C], "last image vs alone")


# ----------------------------------------------------------------------------------------------------------- (7) exact operations
@pytest.mark.parametrize("B,Hi,Wi,C,Ho,Wo", [(2, 16, 16, 32, 16, 16), (1, 16, 24, 16, 64, 64), (2, 40, 40, 48, 17, 9), (1, 1, 1, 16, 5, 3),
                                             (1, 32, 32, 16, 256, 256)])
def test_bilinear_nhwc_to_nchw(cuda, B, Hi, Wi, C, Ho, Wo):
    """Scaling up and down, within the bound of the fp32 interpolation weights; bit-exact at equal sizes (a layout change)."""
    lib = _lib(cuda)
    g = _gen(cuda, "bil", B, Hi, Wi, C, Ho, Wo)
    x = _bf(torch.randn(B, Hi, Wi, C, device=cuda, generator=g))
    buf, inside = _flat_out(B * C * Ho * Wo, torch.float32, cuda)
    lib.call("es3_bilinear_nhwc_to_nchw", x.data_ptr(), buf.data_ptr(), B, Hi, Wi, C, Ho, Wo, _st())
    got = buf[:B * C * Ho * Wo].view(B, C, Ho, Wo)
    ref, bound = R.bilinear(x.double(), Ho, Wo)
    _check("7 bilinear", got, ref, bound, f"bilinear {Hi}x{Wi} -> {Ho}x{Wo}")
    _assert_untouched(buf, inside, "bilinear")
    if (Hi, Wi) == (Ho, Wo):
        _bits_equal(got, x.float().permute(0, 3, 1, 2), "bilinear at equal sizes")


@pytest.mark.parametrize("B,H,W,C", [(2, 8, 8, 16), (1, 17, 33, 40), (3, 2, 2, 8), (1, 256, 256, 64)])
def test_maxpool_and_layouts_bit_exact(cuda, B, H, W, C):
    lib = _lib(cuda)
    g = _gen(cuda, "pool", B, H, W, C)
    x = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    n = B * (H // 2) * (W // 2) * C
    buf, inside = _flat_out(n, torch.bfloat16, cuda)
    lib.call("es3_maxpool2x2_bf16", x.data_ptr(), buf.data_ptr(), B, H, W, C, _st())
    _bits_equal(buf[:n].view(B, H // 2, W // 2, C), F.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1), "maxpool2x2")
    _assert_untouched(buf, inside, "maxpool2x2")
    o32, ins32 = _flat_out(B * H * W * C, torch.float32, cuda)
    lib.call("es3_nhwc_to_nchw_f32", x.data_ptr(), o32.data_ptr(), B, H * W, C, _st())
    _bits_equal(o32[:B * H * W * C].view(B, C, H, W), x.float().permute(0, 3, 1, 2), "nhwc_to_nchw_f32")
    _assert_untouched(o32, ins32, "nhwc_to_nchw_f32")
    f = torch.randn(B, C, H, W, device=cuda, generator=g)
    ob, insb = _flat_out(B * H * W * C, torch.bfloat16, cuda)
    lib.call("es3_nchw_f32_to_nhwc", f.data_ptr(), ob.data_ptr(), B, H * W, C, _st())
    _bits_equal(ob[:B * H * W * C].view(B, H, W, C), f.permute(0, 2, 3, 1).to(torch.bfloat16), "nchw_f32_to_nhwc")
    _assert_untouched(ob, insb, "nchw_f32_to_nhwc")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    keys = {dw_tc_key(c[0][0], c[0][1], c[1]) for c in DWTC}
    keys |= {("es3_dwconv_tiled_bf16", 3, 2, c[1]) for c in DWT}
    keys |= {("es3_dwconv_bf16", c[0][0], c[0][1], c[1]) for c in DWG}
    keys |= {("es3_mbconv_bf16",) + blk for blk in MB_TC + MB_S2}
    keys |= {("es3_dwproj_tc_bf16", c[0], c[1]) for c in DWP}
    keys |= {("es3_stem_conv3x3_s2", c[0], c[1]) for c in STEM} | {("es3_dsconv_res_bf16", c[0], c[1]) for c in DSC}
    keys |= {("es3_conv3x3_s2_narrow_bf16", c[0], c[1], c[2]) for c in NARROW}
    keys |= {("es3_litemla_attn_generic", 16), ("es3_litemla_attn_generic", 32)}
    keys |= {("es3_win_attn_bias_bf16", c[4]) for c in WIN} | {ln_key(c[0]) for c in LN}
    keys |= {(k,) for k in ("es3_stem_fused_c16", "es3_litemla_aggreg_dwpw", "es3_litemla_attn_tc", "es3_channel_mean",
                            "es3_scale_channels", "es3_round_taps_sum_bf16", "es3_bilinear_nhwc_to_nchw", "es3_maxpool2x2_bf16",
                            "es3_nhwc_to_nchw_f32", "es3_nchw_f32_to_nhwc")}
    return keys
