"""Kernel-level numerics: every C-ABI op against a plain PyTorch fp32 statement of the same op.

Inputs are rounded to bf16 first so the comparison isolates the kernel's arithmetic (fp32 accumulation,
bf16 output rounding) from input quantisation.  Tolerances: outputs are bf16 (rel. step 2^-8), so
atol/rtol = 1e-2 relative to the tensor's scale; fp32 outputs use 2e-3 (fp32 accumulation-order noise
on bf16 products).
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _close(got, ref, tol, what=""):
    got = got.float()
    scale = ref.abs().max().item() + 1e-12
    err = (got - ref).abs().max().item() / scale
    assert err <= tol, f"{what}: max err / scale = {err:.3e} > {tol}"


def _act(x, act):
    if act is None:
        return x
    return {"relu": F.relu, "hswish": F.hardswish, "gelu": F.gelu, "gelu_tanh": lambda v: F.gelu(v, approximate="tanh"),
            "relu6": F.relu6, "sigmoid": torch.sigmoid}[act](x)


GEMM_CASES = [
    # M, N, K, act, residual, out_f32, bn_hint
    (128, 32, 64, None, False, False, 0),
    (256, 64, 16, "hswish", False, False, 0),
    (300, 128, 128, "gelu", True, False, 0),
    (1000, 256, 256, None, True, False, 0),
    (127, 1024, 256, "gelu", False, False, 0),
    (5184, 1024, 1024, None, True, True, 256),
    (640, 3072, 1024, None, False, False, 256),
    (513, 4736, 1024, "gelu", False, False, 128),
    (384, 1024, 4736, None, True, False, 0),
    (3969, 384, 128, None, False, False, 0),
    (2048, 512, 128, "hswish", False, False, 64),
    (2048, 128, 512, None, True, False, 32),
    # N % 32 != 0 (ragged last 32-column chunk: channel widths 8/16/24/48/80 of efficientvit b0/b2, repvit m0_9/m2_3), small K
    (1000, 48, 96, "hswish", True, False, 0),
    (777, 80, 160, "gelu", True, False, 0),
    (513, 16, 64, None, True, False, 0),
    (300, 8, 32, "relu", False, True, 0),
    (640, 24, 8, None, False, False, 0),
    (2048, 160, 24, "hswish", True, True, 0),
]


@pytest.mark.parametrize("M,N,K,act,res,out_f32,bn", GEMM_CASES)
def test_gemm_tc(cuda, M, N, K, act, res, out_f32, bn):
    from efficientsam3_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = _bf(torch.randn(M, K, generator=g)).to(cuda)
    w = _bf(torch.randn(N, K, generator=g) / math.sqrt(K)).to(cuda)
    scale = (torch.rand(N, generator=g) + 0.5).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    r = _bf(torch.randn(M, N, generator=g)).to(cuda) if res else None
    out = ops.gemm(a, w, scale=scale, bias=bias, act=act, residual=r,
                   out_dtype=torch.float32 if out_f32 else torch.bfloat16, bn_hint=bn)
    ref = _act((a.float() @ w.float().t()) * scale + bias, act)
    if res:
        ref = ref + r.float()
    _close(out, ref, 2e-3 if out_f32 else 1e-2, f"gemm {M}x{N}x{K}")
    # independent on-device cross-check with the CUDA-core kernel
    out2 = ops.gemm_simt(a, w, scale=scale, bias=bias, act=act, residual=r, out_dtype=torch.float32)
    _close(out2, ref, 2e-3, "gemm_simt")


@pytest.mark.parametrize("K,N", [(16, 16), (16, 32), (16, 64), (32, 16), (32, 32), (32, 64), (64, 16), (64, 32)])
@pytest.mark.parametrize("M,res", [(1, False), (4099, True), (70000, False)])
def test_pw_small(cuda, K, N, M, res):
    """Narrow pointwise GEMMs (K, N <= 64) on es3_pw_small_bf16: against fp32, and against the wgmma kernel on the same operands."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(M + 3 * K + N)
    big = _bf(torch.randn(M, K + 8, generator=g)).to(cuda)
    a = big[:, :K]                                                  # row-strided operand view
    w = _bf(torch.randn(N, K, generator=g) / math.sqrt(K)).to(cuda)
    r = _bf(torch.randn(M, N, generator=g)).to(cuda) if res else None
    n0 = ops.launch_count
    out = ops.gemm(a, w, residual=r)
    assert ops.launch_count == n0 + 1
    ref = a.float() @ w.float().t() + (r.float() if res else 0)
    _close(out, ref, 1e-2, f"pw_small {M}x{N}x{K}")
    ops.PW_SMALL = False
    try:
        tc = ops.gemm(a, w, residual=r)
    finally:
        ops.PW_SMALL = True
    assert (out.float() - tc.float()).abs().max().item() <= 2 ** -7 * ref.abs().max().item()      # same rounding points: <= 1 bf16 ulp apart


def test_gemm_strided_views(cuda):
    """A is a channel slice of a wider buffer; out is written into a slice (the LiteMLA qkv layout)."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(5)
    big = _bf(torch.randn(777, 256, generator=g)).to(cuda)
    a = big[:, 64:192]
    w = _bf(torch.randn(384, 128, generator=g) / 11).to(cuda)
    outbuf = torch.zeros(777, 768, device=cuda, dtype=torch.bfloat16)
    ops.gemm(a, w, out=outbuf[:, :384])
    ref = a.float() @ w.float().t()
    _close(outbuf[:, :384], ref, 1e-2, "strided gemm")
    assert outbuf[:, 384:].abs().max().item() == 0


@pytest.mark.parametrize("B,H,W,C,N", [(2, 32, 32, 1024, 1024), (1, 8, 8, 64, 32), (2, 17, 23, 128, 64), (1, 72, 72, 256, 256)])
def test_conv3x3(cuda, B, H, W, C, N):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(B + H + C)
    x = _bf(torch.randn(B, H, W, C, generator=g)).to(cuda)
    w = _bf(torch.randn(N, C, 3, 3, generator=g) / math.sqrt(9 * C)).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    w9 = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops.conv3x3(x, w9, bias=bias)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    _close(out, ref, 1e-2, "conv3x3")


@pytest.mark.parametrize("H,W,Cout", [(64, 64, 16), (63, 65, 32)])
def test_stem(cuda, H, W, Cout):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(H)
    x = torch.randn(2, 3, H, W, generator=g).to(cuda)
    w = (torch.randn(Cout, 3, 3, 3, generator=g) / 5).to(cuda)
    b = torch.randn(Cout, generator=g).to(cuda)
    w27 = w.reshape(Cout, 27).t().contiguous()
    out = ops.stem_conv3x3_s2(x, w27, b, "hswish")
    ref = F.hardswish(F.conv2d(x, w, b, stride=2, padding=1)).permute(0, 2, 3, 1)
    _close(out, ref, 1e-2, "stem")


@pytest.mark.parametrize("simple", [False, True])
@pytest.mark.parametrize("ks,stride,H,W,C", [(3, 1, 20, 20, 64), (3, 2, 21, 19, 32), (5, 1, 16, 16, 48), (3, 2, 63, 63, 512),
                                             (3, 1, 64, 64, 128), (5, 1, 33, 70, 96), (3, 2, 128, 128, 64), (3, 1, 7, 5, 32)])
def test_dwconv(cuda, ks, stride, H, W, C, simple):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(ks * 10 + stride)
    x = _bf(torch.randn(2, H, W, C, generator=g)).to(cuda)
    w = (torch.randn(C, 1, ks, ks, generator=g) / ks).to(cuda)
    b = torch.randn(C, generator=g).to(cuda)
    wt = w.reshape(C, ks * ks).t().contiguous()
    out = ops.dwconv(x, wt, b, ks, stride, "hswish", force_simple=simple)
    ref = F.hardswish(F.conv2d(x.float().permute(0, 3, 1, 2), w, b, stride=stride, padding=ks // 2, groups=C)).permute(0, 2, 3, 1)
    _close(out, ref, 1e-2, "dwconv")


@pytest.mark.parametrize("ks,H,W,C,act,sliced", [(3, 20, 20, 64, "hswish", False), (3, 64, 64, 128, None, False), (3, 7, 5, 32, "gelu", False),
                                                 (5, 33, 70, 96, None, True), (5, 16, 16, 32, "relu", False), (3, 40, 37, 96, None, True),
                                                 (3, 9, 100, 256, "hswish", False), (5, 64, 64, 384, None, True)])
def test_dwconv_tc(cuda, ks, H, W, C, act, sliced):
    """Tensor-core depthwise kernel (diagonal bf16 tap operands, two taps per m16n8k16, tap sums preserved by es3_round_taps_sum_bf16):
    against torch at exactly the taps it computes with and against torch with the fp32 taps; `sliced`: input and output are
    channel windows of wider NHWC buffers."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(ks * 100 + C + H)
    B = 2
    wide = _bf(torch.randn(B, H, W, 2 * C if sliced else C, generator=g)).to(cuda)
    x = wide[..., :C]
    w = (torch.randn(C, 1, ks, ks, generator=g) / ks).to(cuda)
    b = torch.randn(C, generator=g).to(cuda) if act != "relu" else None
    wt = w.reshape(C, ks * ks).t().contiguous()
    obuf = torch.zeros(B, H, W, 2 * C if sliced else C, device=cuda, dtype=torch.bfloat16)
    out = ops.dwconv(x, wt, b, ks, 1, act, out=obuf[..., C:] if sliced else obuf)
    fn = {None: lambda t: t, "hswish": F.hardswish, "gelu": F.gelu, "relu": F.relu}[act]
    taps = ops.round_taps_sum_bf16(wt)                                           # [ks*ks, C]: what the kernel multiplies with
    assert torch.equal(taps, taps.to(torch.bfloat16).float())                   # bf16-representable ...
    near = wt.to(torch.bfloat16).float()
    assert ((taps - near).abs() <= 1.01 * near.abs() * 2.0 ** -7).all()         # ... at most one bf16 step from nearest rounding ...
    assert ((taps.sum(0) - wt.sum(0)).abs() <= (near.sum(0) - wt.sum(0)).abs() + 1e-7).all()   # ... with a tap sum at least as good
    wr = taps.t().reshape(C, 1, ks, ks)
    ref_taps = fn(F.conv2d(x.float().permute(0, 3, 1, 2), wr, b, stride=1, padding=ks // 2, groups=C)).permute(0, 2, 3, 1)
    _close(out, ref_taps, 4e-3, "dwconv_tc vs torch at the kernel's taps")
    ref = fn(F.conv2d(x.float().permute(0, 3, 1, 2), w, b, stride=1, padding=ks // 2, groups=C)).permute(0, 2, 3, 1)
    _close(out, ref, 8e-3, "dwconv_tc vs torch (fp32 taps)")
    if sliced:
        assert torch.count_nonzero(obuf[..., :C]) == 0       # the neighbouring channel window is untouched


def test_dsconv_res(cuda):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(3)
    C = 16
    x = _bf(torch.randn(2, 30, 34, C, generator=g)).to(cuda)
    wdw = (torch.randn(C, 1, 3, 3, generator=g) / 3).to(cuda)
    bdw = torch.randn(C, generator=g).to(cuda)
    wpw = (torch.randn(C, C, generator=g) / 4).to(cuda)
    bpw = torch.randn(C, generator=g).to(cuda)
    out = ops.dsconv_res(x, wdw.reshape(C, 9).t().contiguous(), bdw, wpw.contiguous(), bpw, "hswish")
    xn = x.float().permute(0, 3, 1, 2)
    mid = F.hardswish(F.conv2d(xn, wdw, bdw, padding=1, groups=C)).to(torch.bfloat16).float()
    ref = (F.conv2d(mid, wpw[:, :, None, None], bpw) + xn).permute(0, 2, 3, 1)
    _close(out, ref, 1e-2, "dsconv_res")


@pytest.mark.parametrize("H,W", [(64, 64), (61, 75), (130, 34), (18, 7)])
def test_stem_fused(cuda, H, W):
    """One-launch stem (conv3x3 s2 + residual DSConv on mma.sync) vs the fp32 torch composition with the same bf16 roundings."""
    from efficientsam3_b200 import ops
    _r = lambda t: t.to(torch.bfloat16).float()
    g = torch.Generator().manual_seed(H * 7 + W)
    C = 16
    x = torch.randn(2, 3, H, W, generator=g).to(cuda)
    w0 = _r(torch.randn(C, 3, 3, 3, generator=g) / 5).to(cuda)
    s0 = (torch.rand(C, generator=g) + 0.5).to(cuda)
    b0 = torch.randn(C, generator=g).to(cuda)
    wdw = _r(torch.randn(C, 1, 3, 3, generator=g) / 3).to(cuda)
    bdw = torch.randn(C, generator=g).to(cuda)
    wpw = _r(torch.randn(C, C, generator=g) / 4).to(cuda)
    spw = (torch.rand(C, generator=g) + 0.5).to(cuda)
    bpw = torch.randn(C, generator=g).to(cuda)
    w0p = torch.zeros(C, 32, device=cuda)
    w0p[:, :27] = w0.reshape(C, 27)
    out = ops.stem_fused_c16(x, w0p.to(torch.bfloat16).contiguous(), s0, b0, wdw.reshape(C, 9).t().contiguous(), bdw,
                             wpw.to(torch.bfloat16).contiguous(), spw, bpw)
    x1 = F.hardswish(F.conv2d(_r(x), w0, None, stride=2, padding=1) * s0.view(1, -1, 1, 1) + b0.view(1, -1, 1, 1))
    x1 = _r(x1)
    mid = _r(F.hardswish(F.conv2d(x1, wdw, bdw, padding=1, groups=C)))
    ref = (F.conv2d(mid, wpw[:, :, None, None]) * spw.view(1, -1, 1, 1) + bpw.view(1, -1, 1, 1) + x1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    _close(out, ref, 1e-2, "stem_fused")


@pytest.mark.parametrize("Hi,Wi,Ho,Wo", [(32, 32, 72, 72), (32, 32, 64, 64), (8, 8, 18, 18), (16, 16, 16, 16)])
def test_bilinear(cuda, Hi, Wi, Ho, Wo):
    from efficientsam3_b200 import ops
    x = _bf(torch.randn(2, Hi, Wi, 128, generator=torch.Generator().manual_seed(1))).to(cuda)
    out = ops.bilinear_nhwc_to_nchw(x, Ho, Wo)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=False)
    _close(out, ref, 1e-5, "bilinear")


def test_layout_roundtrip(cuda):
    from efficientsam3_b200 import ops
    x = torch.randn(2, 48, 9, 11, device=cuda)
    y = ops.nchw_f32_to_nhwc(x)
    assert torch.equal(y, x.permute(0, 2, 3, 1).to(torch.bfloat16))
    z = ops.nhwc_to_nchw_f32(y)
    assert torch.equal(z, x.to(torch.bfloat16).float())


@pytest.mark.parametrize("H,W,heads,B", [(32, 32, 16, 2), (63, 63, 8, 1), (64, 64, 8, 2), (5, 7, 2, 3)])
def test_litemla(cuda, H, W, heads, B):
    """aggreg + ReLU linear attention (the tensor-core kernels) vs the textbook formulation (efficientvit/nn/ops.py:584-621)."""
    from efficientsam3_b200 import ops
    dim = 16
    td = heads * dim
    C3 = 3 * td
    g = torch.Generator().manual_seed(H)
    qkv = _bf(torch.randn(B, H, W, C3, generator=g)).to(cuda)
    wdw = (torch.randn(C3, 1, 5, 5, generator=g) / 5).to(cuda)
    wpw = (torch.randn(C3, 16, 1, 1, generator=g) / 4).to(cuda)
    ms = torch.zeros(B, H, W, 2 * C3, device=cuda, dtype=torch.bfloat16)
    ms[..., :C3] = qkv
    wdw_t, wpw_t = wdw.reshape(C3, 25).t().contiguous(), wpw.reshape(C3, 16).contiguous()
    ops.litemla_aggreg_dwpw(ms, *ops.litemla_dwpw_weights(wdw_t, wpw_t), C3)
    x = qkv.float().permute(0, 3, 1, 2)
    dw = F.conv2d(x, wdw, padding=2, groups=C3).to(torch.bfloat16).float()     # the kernel rounds the depthwise output to bf16
    agg = F.conv2d(dw, wpw, groups=3 * heads)
    _close(ms[..., C3:], agg.permute(0, 2, 3, 1), 1e-2, "aggreg")
    att = ops.litemla_attn(ms, 2 * heads)
    full = ms.float().permute(0, 3, 1, 2).reshape(B, -1, 3 * dim, H * W)
    q, k, v = F.relu(full[:, :, :dim]), F.relu(full[:, :, dim:2 * dim]), full[:, :, 2 * dim:]
    v = F.pad(v, (0, 0, 0, 1), value=1.0)
    out = (v @ k.transpose(-1, -2)) @ q
    out = out[:, :, :-1] / (out[:, :, -1:] + 1e-15)
    ref = out.reshape(B, -1, H, W).permute(0, 2, 3, 1)
    _close(att, ref, 1e-2, "litemla attn")


def test_cpu_tensor_is_an_error():
    from efficientsam3_b200 import _lib, ops
    with pytest.raises(_lib.Es3Error):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(32, 8, dtype=torch.bfloat16))


@pytest.mark.parametrize("cin,mid,cout,stride,res,H,W", [
    (16, 64, 32, 2, False, 64, 64), (32, 128, 32, 1, True, 40, 48), (32, 128, 64, 2, False, 33, 47),
    (64, 256, 64, 1, True, 31, 17), (64, 256, 128, 2, False, 64, 64), (16, 64, 32, 2, False, 63, 65),
    (64, 256, 64, 1, True, 128, 128), (32, 128, 32, 1, True, 8, 16), (64, 256, 128, 2, False, 37, 29), (32, 128, 64, 2, False, 130, 66)])
def test_mbconv_fused(cuda, cin, mid, cout, stride, res, H, W):
    """One-kernel MBConv vs the op-by-op fp32 statement (intermediates rounded to bf16 where the unfused native path would
    materialise them)."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(cin + mid + H)
    B = 2
    x = _bf(torch.randn(B, H, W, cin, generator=g)).to(cuda)
    w1 = _bf(torch.randn(mid, cin, generator=g) / math.sqrt(cin)).to(cuda)
    s1 = (torch.rand(mid, generator=g) + 0.5).to(cuda); b1 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    wdw = (torch.randn(mid, 1, 3, 3, generator=g) / 3).to(cuda); b2 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    w3 = _bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid)).to(cuda)
    s3 = (torch.rand(cout, generator=g) + 0.5).to(cuda); b3 = (torch.randn(cout, generator=g) * 0.2).to(cuda)
    y = ops.mbconv_fused(x, w1, s1, b1, wdw.reshape(mid, 9).t().contiguous(), b2, w3, s3, b3, stride, res, "hswish")
    assert y is not None
    xn = x.float().permute(0, 3, 1, 2)
    e = F.hardswish(F.conv2d(xn, w1.float()[:, :, None, None]) * s1.view(1, -1, 1, 1) + b1.view(1, -1, 1, 1))
    e = e.to(torch.bfloat16).float()
    d = F.hardswish(F.conv2d(e, wdw, b2, stride=stride, padding=1, groups=mid)).to(torch.bfloat16).float()
    ref = F.conv2d(d, w3.float()[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)
    if res:
        ref = ref + xn
    _close(y, ref.permute(0, 2, 3, 1), 1e-2, "mbconv_fused")


@pytest.mark.parametrize("mid,cout,H,W,res", [(512, 128, 64, 64, True), (512, 128, 19, 37, True), (512, 128, 8, 16, False),
                                              (1024, 256, 32, 32, True), (1024, 256, 9, 21, False)])
def test_dwproj_tc(cuda, mid, cout, H, W, res):
    """depthwise 3x3 + bias + hswish + projection + BN (+ residual) in one wgmma kernel vs the op-by-op statement."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(mid + H)
    B = 2
    m = _bf(torch.randn(B, H, W, mid, generator=g)).to(cuda)
    wdw = (torch.randn(mid, 1, 3, 3, generator=g) / 3).to(cuda); b2 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    w3 = _bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid)).to(cuda)
    s3 = (torch.rand(cout, generator=g) + 0.5).to(cuda); b3 = (torch.randn(cout, generator=g) * 0.2).to(cuda)
    x = _bf(torch.randn(B, H, W, cout, generator=g)).to(cuda) if res else None
    y = ops.dwproj(m, wdw.reshape(mid, 9).t().contiguous(), b2, w3, s3, b3, residual=x)
    assert y is not None
    wq = wdw.to(torch.bfloat16).float()      # the kernel multiplies bf16 depthwise weights
    d = F.hardswish(F.conv2d(m.float().permute(0, 3, 1, 2), wq, b2, padding=1, groups=mid)).to(torch.bfloat16).float()
    ref = F.conv2d(d, w3.float()[:, :, None, None]) * s3.view(1, -1, 1, 1) + b3.view(1, -1, 1, 1)
    if res:
        ref = ref + x.float().permute(0, 3, 1, 2)
    _close(y, ref.permute(0, 2, 3, 1), 1e-2, "dwproj_tc")
    assert ops.dwproj(m[..., :256].contiguous(), wdw.reshape(mid, 9).t()[:, :256].contiguous(), b2[:256], w3[:, :256].contiguous(),
                      s3, b3) is None      # shape not instantiated -> None, the caller falls back to dwconv + gemm



@pytest.mark.parametrize("kind,cin,mid,cout,stride,H,W", [
    ("dwproj", 0, 512, 128, 1, 64, 64), ("dwproj", 0, 1024, 256, 1, 32, 32), ("mbconv", 32, 128, 32, 1, 128, 128),
    ("mbconv", 64, 256, 64, 1, 64, 64), ("mbconv", 16, 64, 32, 2, 256, 256), ("mbconv", 64, 256, 128, 2, 128, 128)])
def test_fused_wgmma_kernels_are_bit_reproducible(cuda, kind, cin, mid, cout, stride, H, W):
    """The persistent fused kernels (several tiles per CTA, TMA rings shared by the depthwise and the wgmma warpgroups) give
    bit-identical outputs when run again on the same inputs."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(mid + H + stride)
    B = 16
    wdw = (torch.randn(mid, 1, 3, 3, generator=g) / 3).reshape(mid, 9).t().contiguous().to(cuda)
    b2 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
    w3 = _bf(torch.randn(cout, mid, generator=g) / math.sqrt(mid)).to(cuda)
    s3 = (torch.rand(cout, generator=g) + 0.5).to(cuda); b3 = (torch.randn(cout, generator=g) * 0.2).to(cuda)
    if kind == "dwproj":
        m = _bf(torch.randn(B, H, W, mid, generator=g)).to(cuda)
        x = _bf(torch.randn(B, H, W, cout, generator=g)).to(cuda)
        run = lambda: ops.dwproj(m, wdw, b2, w3, s3, b3, residual=x)
    else:
        x = _bf(torch.randn(B, H, W, cin, generator=g)).to(cuda)
        w1 = _bf(torch.randn(mid, cin, generator=g) / math.sqrt(cin)).to(cuda)
        s1 = (torch.rand(mid, generator=g) + 0.5).to(cuda); b1 = (torch.randn(mid, generator=g) * 0.2).to(cuda)
        run = lambda: ops.mbconv_fused(x, w1, s1, b1, wdw, b2, w3, s3, b3, stride, stride == 1, "hswish")
    first = run()
    assert first is not None
    first = first.clone()
    for i in range(8):
        assert torch.equal(run(), first), f"{kind} run {i + 1} differs from the first"

def test_mbconv_fused_uninstantiated_shape_returns_none(cuda):
    from efficientsam3_b200 import ops
    x = torch.zeros(1, 8, 8, 48, device=cuda, dtype=torch.bfloat16)
    z = lambda *s: torch.zeros(*s, device=cuda)
    y = ops.mbconv_fused(x, z(192, 48).bfloat16(), z(192), z(192), z(9, 192), z(192), z(48, 192).bfloat16(), z(48), z(48),
                         1, True, "hswish")
    assert y is None


@pytest.mark.parametrize("H,W,Cin,Cout", [(64, 64, 32, 64), (63, 41, 32, 64), (20, 36, 32, 32), (40, 40, 32, 48), (33, 50, 48, 80),
                                          (64, 30, 48, 96)])
def test_conv3x3_s2_narrow(cuda, H, W, Cin, Cout):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(H + Cout)
    x = _bf(torch.randn(2, H, W, Cin, generator=g)).to(cuda)
    w = _bf(torch.randn(Cout, Cin, 3, 3, generator=g) / 17).to(cuda)
    sc = (torch.rand(Cout, generator=g) + 0.5).to(cuda); bi = torch.randn(Cout, generator=g).to(cuda)
    out = ops.conv3x3_s2_narrow(x, w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous(), sc, bi, None)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=2, padding=1) * sc.view(1, -1, 1, 1) + bi.view(1, -1, 1, 1)
    _close(out, ref.permute(0, 2, 3, 1), 1e-2, "conv3x3_s2_narrow")


def test_squeeze_excite_pieces(cuda):
    from efficientsam3_b200 import ops
    x = _bf(torch.randn(3, 17, 19, 128, generator=torch.Generator().manual_seed(2))).to(cuda)
    m = ops.channel_mean(x)
    _close(m, x.float().mean((1, 2)), 1e-5, "channel_mean")
    gate = torch.rand(3, 128, device=cuda)
    y = ops.scale_channels(x, gate)
    _close(y, x.float() * gate.view(3, 1, 1, 128), 1e-2, "scale_channels")


@pytest.mark.parametrize("H,W,ws,heads", [(16, 16, 7, 4), (14, 14, 14, 2), (63, 63, 14, 8), (8, 10, 7, 14)])
def test_win_attn_bias(cuda, H, W, ws, heads):
    """Window attention with relative bias over zero-padded partitions vs the TinyViT formulation (tiny_vit.py:270-293,
    352-375) on a given qkv tensor (padded tokens take the supplied constant row)."""
    from efficientsam3_b200 import ops
    B, kd = 2, 32
    C, N = heads * kd, ws * ws
    g = torch.Generator().manual_seed(H * 3 + ws)
    qkv = _bf(torch.randn(B * H * W, 3 * C, generator=g)).to(cuda)
    pad_row = _bf(torch.randn(3 * C, generator=g)).to(cuda)
    bias = torch.randn(heads, N, N, generator=g).to(cuda)
    out = ops.win_attn_bias(qkv, pad_row, bias, B, H, W, C, heads, ws, kd ** -0.5)
    x = qkv.float().view(B, H, W, 3 * C)
    pb, pr = (ws - H % ws) % ws, (ws - W % ws) % ws
    xp = pad_row.float().view(1, 1, 1, -1).expand(B, H + pb, W + pr, -1).clone()
    xp[:, :H, :W] = x
    nH, nW = (H + pb) // ws, (W + pr) // ws
    t = xp.view(B, nH, ws, nW, ws, 3 * C).transpose(2, 3).reshape(B * nH * nW, N, heads, 3 * kd)
    q, k, v = t.split([kd, kd, kd], dim=3)
    q, k, v = q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)
    a = (q @ k.transpose(-2, -1)) * kd ** -0.5 + bias
    o = (a.softmax(-1) @ v).transpose(1, 2).reshape(B * nH * nW, N, C)
    ref = o.view(B, nH, nW, ws, ws, C).transpose(2, 3).reshape(B, H + pb, W + pr, C)[:, :H, :W].reshape(B * H * W, C)
    _close(out, ref, 1e-2, "win_attn_bias")


@pytest.mark.parametrize("M,C", [(300, 448), (1000, 128), (77, 256)])
def test_layernorm_bf16(cuda, M, C):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(C)
    x = _bf(torch.randn(M, C, generator=g) * 2 + 0.5).to(cuda)
    gam, bet = (torch.rand(C, generator=g) + 0.5).to(cuda), torch.randn(C, generator=g).to(cuda)
    y = ops.layernorm_bf16(x, gam, bet, 1e-5)
    _close(y, F.layer_norm(x.float(), (C,), gam, bet, 1e-5), 1e-2, "layernorm_bf16")
