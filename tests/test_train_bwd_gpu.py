"""The image students' backward kernels (train_bwd.cu, wgrad_tc.cu, tinyvit_bwd.cu, litemla_bwd_generic.cu), element by element
against fp64.

Operands are bf16-representable; fp32 inputs (the stem image, the bilinear dout, statistics, dW prefills) are used as given, so
each fp64 statement in tests/ref_train_bwd.py is what the kernel computes with exact arithmetic.  Every output element must lie
within its own bound

    |got - ref| <= GAMMA n u sum|terms|  (fp32 sum of n terms, n = the total term count)  + 4u |ref|   (+ 2^-8 |ref| for bf16 outputs)

u = 2^-24.  The composite operations propagate their intermediates' errors to first order, evaluated in fp64 on absolute values
(ref_train_bwd.py states each one): the batch-statistics BN backward (the coef of bn_bwd_finalize_kernel: dgamma = invstd (sum g z -
mean sum g), B = -scale invstd dgamma / M, C = -scale sum g / M - B mean), LayerNorm backward (mean, rstd, xhat, the two row means),
the LiteMLA backward (KV from the forward's partials, o, r = 1 / (o[dim] + eps), y, do, dKV) and the window-softmax backward (the
scores, the MUFU exp's (2 + 1.16 |x|) ulp, the row sum, D, dS).  Activation derivatives use the epilogue file's L_ACT / EPS_GELU
for the forward activations, and hswish' 1/3 and gelu'' 0.8 for the pre-activation's rounding.  Kinks (relu at 0, hswish at
+-3): inputs avoid them -- da is zeroed where the fp64 pre-activation lies within 4u of a kink, the band where the fp32 branch can
legitimately flip.

Outputs are NaN-prefilled (entry points called through _lib.call where the ops wrapper allocates the output itself): every cell
inside the output region must be written, every cell outside it (a tail, the other eight taps of an ldn / ldk write, columns
K .. ldn - 1, dS columns past heads N^2) keeps its sentinel bits.  Accumulating outputs (dW, dgamma, dbeta, dgate, colsum, bias
gradients) are prefilled with finite values and checked as +=.  Every split-reduction workspace is NaN-prefilled, so a partial that
is read but never written fails; strided operands are slices of NaN-padded buffers.  Entries with a split reduction run twice and
must be bit-identical.

GAMMA = 2 was set from one run on an H100 80GB HBM3 (700 W power limit).  Worst err/bound per section there, fp32 outputs:
(1) wgrad_pw 0.125, its 3x3 / phase taps 0.006; (2) wgrad_tc 0.015; (3) conv3x3_wgrad 0.008; (5) dwconv_wgrad direct 0.098, win
0.0055; (6) bn_stats 0.26, bn_act_bwd dgamma 0.12, dbeta 0.12; (7) se_dgate 0.028, stem_wgrad 0.070, the SE fc gradient 0.25;
(10) layernorm_bwd dgamma 0.089, dbeta 0.003, window dS 0.007, colsum 0.18.  bf16 outputs: 0.95 ... 0.996 in every section
(dw_bwd_data, affine_act, bn_act_bwd dz, se_apply, litemla_bwd, layernorm_bwd dx, window dqkv), because the half-step of the
output rounding dominates their bound and is reached; bilinear_bwd 0.66.  The whole file (359 tests, the route-closure training
steps included, since moved to tests/test_route_closure_gpu.py) took 22 s there.  covered_keys() names the route keys
(tests/routes.py) the tables run.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import ref_train_bwd as R
from bounds import _INT, TAIL, _assert_untouched, _bf, _check, _flat_out, _gen, _lib, _p, _pairwise, _sentinel, _st, report_worst
from routes import key_dw_bwd_data, key_wgrad_pw, key_wgrad_tc

pytestmark = pytest.mark.gpu
_report_worst = report_worst("train bwd")
ACT_CODE = {None: 0, "relu": 1, "hswish": 2, "gelu": 3}
BN_MODE = {"none": 0, "eval": 1, "batch": 2}


def _nan_ws(lib, name, *args, cuda):
    return torch.full((max(lib.size(name, *args), 1),), float("nan"), device=cuda)


@pytest.fixture
def nan_ws(monkeypatch):
    """ops' split-reduction workspaces come NaN-filled."""
    from efficientsam3_b200 import ops
    monkeypatch.setattr(ops, "_f32ws", lambda n, dev: torch.full((max(int(n), 1),), float("nan"), device=dev))


def _twice(run, *bufs):
    """Run `run(copies)` on two clones of the prefilled buffers; both results must be bit-identical.  Returns the first."""
    a = [b.clone() for b in bufs]
    c = [b.clone() for b in bufs]
    run(a)
    run(c)
    for x, y in zip(a, c):
        assert torch.equal(x.view(_INT[x.dtype]), y.view(_INT[y.dtype])), "two runs of a split reduction differ"
    return a


def _nanpad(t, extra=16):
    """The same values as a slice of a NaN-padded [rows, cols + extra] buffer (row stride != width), at column 8 when extra >= 16
    (NaN on both sides), else at column 0; extra = 0 returns t."""
    if extra == 0:
        return t.contiguous()
    off = 8 if extra >= 16 else 0
    big = torch.full((t.shape[0], t.shape[1] + extra), float("nan"), dtype=t.dtype, device=t.device)
    big[:, off:off + t.shape[1]] = t
    return big[:, off:off + t.shape[1]]


def _strided_out(rows, cols, ld, dtype, cuda, fill=None):
    """A NaN buffer of rows * ld + TAIL cells; cells (r, c < cols) form the output region (optionally prefilled)."""
    buf = torch.full((rows * ld + TAIL,), float("nan"), dtype=dtype, device=cuda)
    inside = torch.zeros_like(buf, dtype=torch.bool)
    idx = (torch.arange(rows, device=cuda)[:, None] * ld + torch.arange(cols, device=cuda)[None]).reshape(-1)
    inside[idx] = True
    if fill is not None:
        buf[idx] = fill.reshape(-1).to(dtype)
    return buf, inside, idx


# ----------------------------------------------------------------------------------------------------------- (1) es3_wgrad_pw
def _wgrad_pw_run(cuda, dz, x, M, N, K, ldn, ldk, shift, dW_fill_idx, buf):
    lib = _lib(cuda)
    H, W, dy, dx = shift if shift is not None else (0, 0, 0, 0)
    ws = _nan_ws(lib, "es3_wgrad_pw_ws_floats", M, N, K, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_wgrad_pw", dz.data_ptr(), dz.stride(0), x.data_ptr(), x.stride(0), M, N, K, H, W, dy, dx, ws.data_ptr(),
                 bufs[0].data_ptr(), ldn, ldk, _st())
    return _twice(run, buf)[0]


WGPW_FACTORS = dict(
    N=[8, 16, 24, 48, 96, 136],        # wg_pick 1, 1, 2, 4, 4, 4 (136: a ragged third 64-row tile)
    K=[8, 32, 24, 64, 96, 200],        # wg_pick 1, 2, 2, 4, 4, 4
    M=[1, 255, 257, 700, 4099, 20000],  # ragged against WG_ROWS = 256; M <= 257: splits == nchunks
    strided=[False, True],
    wide=[False, True],                # ldn = K or K + 8 (columns K .. ldn - 1 keep their sentinels)
)
WGPW_DESIGN = _pairwise(WGPW_FACTORS, seed=11)


@pytest.mark.parametrize("N,K,M,strided,wide", WGPW_DESIGN, ids=[f"N{c[0]}-K{c[1]}-M{c[2]}{'-strided' if c[3] else ''}"
                                                                 f"{'-wide' if c[4] else ''}" for c in WGPW_DESIGN])
def test_wgrad_pw(cuda, N, K, M, strided, wide):
    """All nine (MT, NP) = wg_pick(N) x wg_pick(K) instantiations, M ragged against the 256-row chunks, split counts from
    wgrad_splits (M = 1, 255, 257: one split per chunk), NaN-padded strided dz / x, ldn > K."""
    g = _gen(cuda, "wgpw", N, K, M, strided, wide)
    dz = _bf(torch.randn(M, N, device=cuda, generator=g))
    x = _bf(torch.randn(M, K, device=cuda, generator=g))
    if strided:
        dz, x = _nanpad(dz), _nanpad(x, 24)
    ldn = K + 8 if wide else K
    dW0 = torch.randn(N, K, device=cuda, generator=g)
    buf, inside, idx = _strided_out(N, K, ldn, torch.float32, cuda, dW0)
    got = _wgrad_pw_run(cuda, dz, x, M, N, K, ldn, 1, None, idx, buf)
    ref, bound = R.wgrad(dz.double(), x.double(), dW0.double())
    what = f"wgrad_pw M{M} N{N} K{K} strided={strided} ldn={ldn}"
    _check("1 wgrad_pw", got[idx].view(N, K), ref, bound, what)
    _assert_untouched(got, inside, what)


def _tap_case(cuda, dz2, xs, N, C, ky, kx, shift, ref_tap, bound_tap, what):
    """One tap written with ldn = 9 C, ldk = 9 into a [N][C][3][3] buffer whose other eight taps hold NaN sentinels."""
    t = ky * 3 + kx
    buf = torch.full((N * C * 9 + TAIL,), float("nan"), device=cuda)
    inside = torch.zeros_like(buf, dtype=torch.bool)
    idx = (torch.arange(N, device=cuda)[:, None] * 9 * C + torch.arange(C, device=cuda)[None] * 9 + t).reshape(-1)
    inside[idx] = True
    g = _gen(cuda, "tap0", N, C, t)
    dW0 = torch.randn(N, C, device=cuda, generator=g)
    buf[idx] = dW0.reshape(-1)
    lib = _lib(cuda)
    M = dz2.shape[0]
    ws = _nan_ws(lib, "es3_wgrad_pw_ws_floats", M, N, C, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_wgrad_pw", dz2.data_ptr(), dz2.stride(0), xs.data_ptr(), xs.stride(0), M, N, C, *shift, ws.data_ptr(),
                 bufs[0].data_ptr() + 4 * t, 9 * C, 9, _st())
    got = _twice(run, buf)[0]
    _check("1 wgrad_pw taps", got[idx].view(N, C), dW0.double() + ref_tap, bound_tap + 4 * R.U * dW0.double().abs(), what)
    _assert_untouched(got, inside, what)


@pytest.mark.parametrize("B,H,W,N,C", [(2, 9, 7, 32, 16), (1, 12, 12, 64, 128), (3, 5, 33, 24, 8), (2, 16, 16, 136, 48),
                                       (1, 128, 128, 48, 24)])
def test_wgrad_pw_conv3x3_taps(cuda, B, H, W, N, C):
    """shift = (H, W, dy, dx): each of the nine taps of a dense 3x3 conv's weight gradient against the fp64 conv weight gradient's
    tap; the other eight taps stay untouched."""
    g = _gen(cuda, "taps", B, H, W, N, C)
    dy = _bf(torch.randn(B, H, W, N, device=cuda, generator=g))
    a = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    full = torch.nn.grad.conv2d_weight(a.double().permute(0, 3, 1, 2), (N, C, 3, 3), dy.double().permute(0, 3, 1, 2), padding=1)
    absf = torch.nn.grad.conv2d_weight(a.double().abs().permute(0, 3, 1, 2), (N, C, 3, 3), dy.double().abs().permute(0, 3, 1, 2),
                                       padding=1)
    dz2, x2 = dy.view(-1, N), a.view(-1, C)
    for ky in range(3):
        for kx in range(3):
            bound = R._out(full[..., ky, kx], R.GAMMA * (dz2.shape[0] + 1) * R.U * absf[..., ky, kx], False)
            _tap_case(cuda, dz2, x2, N, C, ky, kx, (H, W, ky - 1, kx - 1), full[..., ky, kx], bound,
                      f"conv3x3 tap ({ky},{kx}) B{B} {H}x{W} N{N} C{C}")


_TAP = {0: (1, -1), 1: (0, 0), 2: (1, 0)}          # kernel row / column -> (phase, shift inside the phase image)


@pytest.mark.parametrize("B,H,W,N,C", [(2, 10, 14, 24, 8), (1, 32, 32, 48, 16), (1, 512, 512, 24, 8)])
def test_wgrad_pw_repvit_phase_taps(cuda, B, H, W, N, C):
    """The RepViT stride-2 patch-embed weight gradient (repvit_train.py): tap (ky, kx) reads phase image a0[py::2, px::2] at a
    stride-1 shift; each tap against the fp64 weight gradient of the stride-2 conv itself.  (1, 512, 512, 24, 8): stage-1's shape."""
    g = _gen(cuda, "phase", B, H, W, N, C)
    a0 = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    Ho, Wo = H // 2, W // 2
    dz = _bf(torch.randn(B, Ho, Wo, N, device=cuda, generator=g))
    an, dn = a0.double().permute(0, 3, 1, 2), dz.double().permute(0, 3, 1, 2)
    full = torch.nn.grad.conv2d_weight(an, (N, C, 3, 3), dn, stride=2, padding=1)
    absf = torch.nn.grad.conv2d_weight(an.abs(), (N, C, 3, 3), dn.abs(), stride=2, padding=1)
    phase = {(py, px): a0[:, py::2, px::2, :].contiguous().view(-1, C) for py in (0, 1) for px in (0, 1)}
    dz2 = dz.view(-1, N)
    for ky in range(3):
        py, sy = _TAP[ky]
        for kx in range(3):
            px, sx = _TAP[kx]
            bound = R._out(full[..., ky, kx], R.GAMMA * (dz2.shape[0] + 1) * R.U * absf[..., ky, kx], False)
            _tap_case(cuda, dz2, phase[(py, px)], N, C, ky, kx, (Ho, Wo, sy, sx), full[..., ky, kx], bound,
                      f"repvit phase tap ({ky},{kx}) B{B} {H}x{W} N{N} C{C}")


# ----------------------------------------------------------------------------------------------------------- (2) es3_wgrad_tc
WGTC_FACTORS = dict(
    K=[64, 128, 192, 512],             # KT 64 / 128; 192: a half-empty second 128-wide tile
    N=[64, 128, 192, 384],
    M=[64, 100, 1000, 4099, 70001],    # never a multiple of WG_PX = 64 except 64; nsplit from 1 to 132 / tiles
    strided=[False, True],             # NaN-padded slices: the TMA box runs past the slice
    wide=[False, True],
)
WGTC_DESIGN = _pairwise(WGTC_FACTORS, seed=12)


@pytest.mark.parametrize("K,N,M,strided,wide", WGTC_DESIGN, ids=[f"K{c[0]}-N{c[1]}-M{c[2]}{'-strided' if c[3] else ''}"
                                                                 f"{'-wide' if c[4] else ''}" for c in WGTC_DESIGN])
def test_wgrad_tc(cuda, monkeypatch, nan_ws, K, N, M, strided, wide):
    """The wgmma split-K weight gradient; the public ops.wgrad_pw route takes it and is bit-identical to the direct call."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "wgtc", K, N, M, strided, wide)
    dz = _bf(torch.randn(M, N, device=cuda, generator=g))
    x = _bf(torch.randn(M, K, device=cuda, generator=g))
    if strided:
        dz, x = _nanpad(dz, 72), _nanpad(x, 136)
    ldn = K + 8 if wide else K
    dW0 = torch.randn(N, K, device=cuda, generator=g)
    buf, inside, idx = _strided_out(N, K, ldn, torch.float32, cuda, dW0)
    ws = _nan_ws(lib, "es3_wgrad_tc_ws_floats", M, N, K, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        assert lib.call_rc("es3_wgrad_tc", dz.data_ptr(), dz.stride(0), x.data_ptr(), x.stride(0), M, N, K, ws.data_ptr(),
                           bufs[0].data_ptr(), ldn, _st()) == 0
    got = _twice(run, buf)[0]
    ref, bound = R.wgrad(dz.double(), x.double(), dW0.double())
    what = f"wgrad_tc M{M} N{N} K{K} strided={strided} ldn={ldn}"
    _check("2 wgrad_tc", got[idx].view(N, K), ref, bound, what)
    _assert_untouched(got, inside, what)
    pub = buf.clone()
    ops.wgrad_pw(dz, x, pub, ldn=ldn)
    assert torch.equal(pub.view(torch.int32), got.view(torch.int32)), "ops.wgrad_pw differs from the direct es3_wgrad_tc call"


def test_wgrad_tc_declines_63_rows(cuda, monkeypatch, nan_ws):
    """M = 63 < WG_PX: the direct call returns -1, and ops.wgrad_pw goes to es3_wgrad_pw alone (and is right)."""
    from efficientsam3_b200 import _lib as L, ops
    lib = _lib(cuda)
    M, N, K = 63, 64, 128
    g = _gen(cuda, "wgtc63")
    dz, x = _bf(torch.randn(M, N, device=cuda, generator=g)), _bf(torch.randn(M, K, device=cuda, generator=g))
    ws = _nan_ws(lib, "es3_wgrad_tc_ws_floats", M, N, K, cuda=cuda)
    dW = torch.zeros(N, K, device=cuda)
    assert lib.call_rc("es3_wgrad_tc", dz.data_ptr(), N, x.data_ptr(), K, M, N, K, ws.data_ptr(), dW.data_ptr(), K, _st()) == -1
    names = []
    real_call, real_rc = L.call, L.call_rc
    monkeypatch.setattr(L, "call", lambda n, *a: (names.append(n), real_call(n, *a))[1])
    monkeypatch.setattr(L, "call_rc", lambda n, *a: (names.append(n), real_rc(n, *a))[1])
    dW0 = torch.randn(N, K, device=cuda, generator=g)
    got = dW0.clone()
    ops.wgrad_pw(dz, x, got)
    assert names == ["es3_wgrad_pw"], names
    ref, bound = R.wgrad(dz.double(), x.double(), dW0.double())
    _check("2 wgrad_tc", got, ref, bound, "wgrad_pw M63 fallback")


# ----------------------------------------------------------------------------------------------------------- (3) conv3x3_wgrad
@pytest.mark.parametrize("W", [14, 13, 12, 11, 10, 9, 8, 7])        # Wp - W - 2 = 0 .. 7
def test_transpose_pad_bit_exact(cuda, W):
    from efficientsam3_b200 import ops
    B, H, C = 2, 5, 72                                              # C % 64 != 0: a partial 64-channel tile
    x = _bf(torch.randn(B, H, W, C, device=cuda, generator=_gen(cuda, "tp", W)))
    Wp = (W + 2 + 7) // 8 * 8
    for dx in (-1, 0, 1):
        got = ops.transpose_pad(x, Wp, dx)
        assert torch.equal(got.view(torch.int16), R.transpose_pad(x, Wp, dx).view(torch.int16)), (W, dx)


@pytest.mark.parametrize("B,H,W,N,C", [(2, 9, 14, 64, 64), (1, 7, 13, 128, 64), (2, 5, 12, 64, 192), (1, 6, 11, 256, 128),
                                       (3, 4, 10, 64, 64), (1, 8, 9, 64, 512), (2, 3, 8, 128, 64), (1, 10, 7, 64, 128),
                                       (1, 32, 32, 1024, 64), (2, 64, 64, 64, 1024)])
def test_conv3x3_wgrad(cuda, nan_ws, B, H, W, N, C):
    """transpose_pad + nine GEMMs + accumulate_strided against the fp64 weight gradient, W across Wp - W - 2 = 0 .. 7; the last two
    rows are the student head's 3x3 conv at 1024^2 (64^2 map, 1024 <-> 64 channels... 32^2 for the /32 trunks)."""
    from efficientsam3_b200 import ops
    g = _gen(cuda, "c3w", B, H, W, N, C)
    dy = _bf(torch.randn(B, H, W, N, device=cuda, generator=g))
    a = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    gw0 = torch.randn(N, C, 3, 3, device=cuda, generator=g)
    buf, inside = _flat_out(N * C * 9, torch.float32, cuda)
    buf[:N * C * 9] = gw0.reshape(-1)
    ops.conv3x3_wgrad(dy, a, buf[:N * C * 9].view(N, C, 3, 3))
    ref, bound = R.conv3x3_wgrad(dy.double(), a.double(), gw0.double())
    what = f"conv3x3_wgrad B{B} {H}x{W} N{N} C{C}"
    _check("3 conv3x3_wgrad", buf[:N * C * 9].view(N, C, 3, 3), ref, bound, what)
    _assert_untouched(buf, inside, what)


# ----------------------------------------------------------------------------------------------------------- (4) es3_dwconv_bwd_data
def _dw_bwd_data(cuda, dz, w, H, W, ks, stride, what):
    lib = _lib(cuda)
    B, Ho, Wo, C = dz.shape
    buf, inside = _flat_out(B * H * W * C, torch.bfloat16, cuda)
    lib.call("es3_dwconv_bwd_data", dz.data_ptr(), w.data_ptr(), buf.data_ptr(), B, H, W, C, ks, stride, _st())
    ref, bound = R.dwconv_bwd_data(dz.double(), w.double(), H, W, ks, stride)
    _check("4 dw_bwd_data", buf[:B * H * W * C].view(B, H, W, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


DWBD_CASES = [(2, 17, 23, 64, 3, 2), (1, 16, 16, 8, 3, 2), (3, 9, 10, 24, 3, 2), (1, 10, 9, 40, 3, 2), (2, 1, 1, 16, 3, 2),
              (2, 21, 20, 128, 5, 2), (1, 8, 9, 40, 5, 2), (2, 13, 19, 64, 3, 1), (1, 7, 5, 24, 5, 1),
              (1, 512, 512, 32, 3, 2), (1, 256, 256, 64, 3, 2), (1, 64, 64, 256, 5, 2)]


@pytest.mark.parametrize("B,H,W,C,ks,stride", DWBD_CASES, ids=[f"B{c[0]}-{c[1]}x{c[2]}-C{c[3]}-k{c[4]}s{c[5]}" for c in DWBD_CASES])
def test_dwconv_bwd_data(cuda, B, H, W, C, ks, stride):
    """s2k3 at odd and even H, W; the generic kernel (ks 5 stride 2, stride 1); stage-1's stride-2 stage openers at 1024^2."""
    g = _gen(cuda, "dwbd", B, H, W, C, ks, stride)
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    dz = _bf(torch.randn(B, Ho, Wo, C, device=cuda, generator=g))
    w = torch.randn(ks * ks, C, device=cuda, generator=g) / ks
    _dw_bwd_data(cuda, dz, w, H, W, ks, stride, f"dwconv_bwd_data B{B} {H}x{W} C{C} k{ks}s{stride}")


@pytest.mark.parametrize("ks,stride,C", [(3, 2, 16), (5, 2, 24), (3, 1, 24), (5, 1, 16)])
@pytest.mark.parametrize("H,W", [(13, 11), (12, 14)])
def test_dwconv_bwd_data_halo(cuda, ks, stride, C, H, W):
    """Large values (8) in the last row and column of every dz image, small ones (< 1/16) elsewhere: a pixel reading across an image
    edge (or into the next image) is far outside the bound."""
    B = 3
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    g = _gen(cuda, "dwhalo", ks, stride, C, H, W)
    dz = (torch.rand(B, Ho, Wo, C, device=cuda, generator=g) - 0.5) / 8
    sgn = torch.randn(B, Ho, Wo, C, device=cuda, generator=g).sign()
    dz[:, :, -1] = 8 * sgn[:, :, -1]
    dz[:, -1] = 8 * sgn[:, -1]
    w = _bf(torch.randn(ks * ks, C, device=cuda, generator=g)).float()
    _dw_bwd_data(cuda, _bf(dz), w, H, W, ks, stride, f"dwconv_bwd_data halo k{ks}s{stride} {H}x{W}")


@pytest.mark.parametrize("B,H,W,C,ks", [(2, 13, 19, 64, 3), (1, 9, 11, 96, 5), (2, 16, 16, 16, 3), (1, 7, 5, 24, 5), (2, 64, 64, 256, 3),
                                        (1, 128, 128, 128, 3), (1, 64, 64, 384, 5)])
def test_dwconv_bwd_data_stride1_flipped_taps(cuda, B, H, W, C, ks):
    """Stride 1 as the training graph runs it: the forward depthwise kernel on the 180-degree rotated taps (bf16 weights)."""
    from efficientsam3_b200 import ops
    g = _gen(cuda, "dwflip", B, H, W, C, ks)
    dz = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    w = _bf(torch.randn(ks * ks, C, device=cuda, generator=g) / ks).float()
    buf, inside = _flat_out(B * H * W * C, torch.bfloat16, cuda)
    ops.dwconv(dz, w.flip(0).contiguous(), None, ks, 1, None, out=buf[:B * H * W * C].view(B, H, W, C))
    ref, bound = R.dwconv_bwd_data(dz.double(), w.double(), H, W, ks, 1)
    what = f"dwconv flipped taps B{B} {H}x{W} C{C} k{ks}"
    _check("4 dw_bwd_data flipped", buf[:B * H * W * C].view(B, H, W, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


# ----------------------------------------------------------------------------------------------------------- (5) dwconv weight gradient
def _dw_wgrad(cuda, name, B, H, W, C, ks, stride, sliced, seed=()):
    lib = _lib(cuda)
    g = _gen(cuda, "dww", name, B, H, W, C, ks, stride, sliced, *seed)
    pad = ks // 2
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    dz = _bf(torch.randn(B, Ho, Wo, C, device=cuda, generator=g))
    if sliced:                                     # x = the first C channels of a [B, H, W, 2C] buffer whose other half is NaN
        big = torch.full((B, H, W, 2 * C), float("nan"), device=cuda, dtype=torch.bfloat16)
        big[..., :C] = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
        x = big[..., :C]
    else:
        x = _bf(torch.randn(B, H, W, C, device=cuda, generator=g))
    dW0 = torch.randn(C, 1, ks, ks, device=cuda, generator=g)
    buf, inside = _flat_out(C * ks * ks, torch.float32, cuda)
    buf[:C * ks * ks] = dW0.reshape(-1)
    wsname = "es3_dwconv_wgrad_win_ws_floats" if name.endswith("win") else "es3_dwconv_wgrad_ws_floats"
    ws = _nan_ws(lib, wsname, B, H, W, C, ks, stride, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call(name, dz.data_ptr(), x.data_ptr(), x.stride(2), B, H, W, C, ks, stride, ws.data_ptr(), bufs[0].data_ptr(), _st())
    got = _twice(run, buf)[0]
    ref, bound = R.dwconv_wgrad(dz.double(), x.double(), dW0.double(), ks, stride)
    what = f"{name} B{B} {H}x{W} C{C} k{ks}s{stride} sliced={sliced}"
    _check("5 " + name[4:], got[:C * ks * ks].view(C, 1, ks, ks), ref, bound, what)
    _assert_untouched(got, inside, what)


DWD_FACTORS = dict(
    C=[8, 16, 24, 40, 48],             # C % 32 != 0: the direct kernels' route
    ks_stride=[(3, 1), (5, 1), (3, 2), (5, 2)],   # strip kernels (VEC 8 / 4) at stride 1, per-pixel kernels at stride 2
    HW=[(1, 1), (7, 5), (13, 19), (33, 40)],
    B=[1, 3],
    sliced=[False, True],
)
DWD_DESIGN = _pairwise(DWD_FACTORS, seed=13)


@pytest.mark.parametrize("C,ks_stride,HW,B,sliced", DWD_DESIGN, ids=[f"C{c[0]}-k{c[1][0]}s{c[1][1]}-{c[2][0]}x{c[2][1]}-B{c[3]}"
                                                                    f"{'-sliced' if c[4] else ''}" for c in DWD_DESIGN])
def test_dwconv_wgrad_direct(cuda, C, ks_stride, HW, B, sliced):
    _dw_wgrad(cuda, "es3_dwconv_wgrad", B, HW[0], HW[1], C, *ks_stride, sliced)


DWW_FACTORS = dict(
    C=[32, 64, 96],
    ks_stride=[(3, 1), (5, 1), (3, 2), (5, 2)],
    HW=[(8, 32), (9, 33), (17, 70), (5, 100), (40, 37)],     # ragged against the 8 x 32 output tile
    B=[1, 2],
    sliced=[False, True],
)
DWW_DESIGN = _pairwise(DWW_FACTORS, seed=14)


@pytest.mark.parametrize("C,ks_stride,HW,B,sliced", DWW_DESIGN, ids=[f"C{c[0]}-k{c[1][0]}s{c[1][1]}-{c[2][0]}x{c[2][1]}-B{c[3]}"
                                                                    f"{'-sliced' if c[4] else ''}" for c in DWW_DESIGN])
def test_dwconv_wgrad_win(cuda, C, ks_stride, HW, B, sliced):
    _dw_wgrad(cuda, "es3_dwconv_wgrad_win", B, HW[0], HW[1], C, *ks_stride, sliced)


def test_dwconv_wgrad_block_cap(cuda):
    """EfficientViT's stage-0 DSConv at stage-1's batch: C = 16, 3x3 stride 1, 512^2, B = 20 -- the strip kernel's 1184-block cap,
    so every block walks more than eight strips per lane (an nblk / upb split no smaller shape reaches)."""
    CG, lanes, P = 2, 128, 4
    strips = 20 * 512 * (512 // P)
    assert (strips + lanes * 8 - 1) // (lanes * 8) > 1184 and CG == 16 // 8
    _dw_wgrad(cuda, "es3_dwconv_wgrad", 20, 512, 512, 16, 3, 1, False)


@pytest.mark.parametrize("name,B,H,W,C,ks,stride", [("es3_dwconv_wgrad", 1, 512, 512, 16, 3, 1), ("es3_dwconv_wgrad", 2, 512, 512, 24, 3, 2),
                                                    ("es3_dwconv_wgrad_win", 1, 256, 256, 64, 3, 1), ("es3_dwconv_wgrad_win", 2, 128, 128, 128, 3, 2),
                                                    ("es3_dwconv_wgrad_win", 1, 64, 64, 384, 5, 1), ("es3_dwconv_wgrad_win", 1, 64, 64, 256, 5, 2)])
def test_dwconv_wgrad_production_shapes(cuda, name, B, H, W, C, ks, stride):
    """Stage-1's depthwise layers at 1024^2: the stage-0 DSConv, the stride-2 openers, the LiteMLA 5x5 aggregation."""
    _dw_wgrad(cuda, name, B, H, W, C, ks, stride, name.endswith("win"))


# ----------------------------------------------------------------------------------------------------------- (6) BatchNorm pieces
BNS_CASES = [(1, 8), (7, 24), (300, 40), (4099, 64), (20000, 128), (131, 2560), (65536, 16)]


@pytest.mark.parametrize("M,C", BNS_CASES)
def test_bn_stats(cuda, M, C):
    """Batch statistics (mean far from zero against the spread: the pivot-shifted sums), the folded scale / shift, the running
    buffers (momentum on the unbiased variance) and num_batches_tracked."""
    lib = _lib(cuda)
    g = _gen(cuda, "bns", M, C)
    z = _bf(torch.randn(M, C, device=cuda, generator=g) * (torch.rand(C, device=cuda, generator=g) + 0.2)
            + 8 * torch.randn(C, device=cuda, generator=g))
    gamma, beta = torch.rand(C, device=cuda, generator=g) + 0.5, torch.randn(C, device=cuda, generator=g)
    rm0, rv0 = torch.randn(C, device=cuda, generator=g), torch.rand(C, device=cuda, generator=g) + 0.5
    nbt = torch.tensor([7], device=cuda)
    outs = {k: _flat_out(C, torch.float32, cuda) for k in ("mean", "invstd", "scale", "shift")}
    run_bufs = {}
    for k, v0 in (("running_mean", rm0), ("running_var", rv0)):
        b, ins = _flat_out(C, torch.float32, cuda)
        b[:C] = v0
        run_bufs[k] = (b, ins)
    ws = _nan_ws(lib, "es3_col_reduce_ws_floats", M, C, cuda=cuda)
    lib.call("es3_bn_stats", z.data_ptr(), M, C, 1e-5, 0.1, gamma.data_ptr(), beta.data_ptr(), ws.data_ptr(),
             *(outs[k][0].data_ptr() for k in ("mean", "invstd", "scale", "shift")), run_bufs["running_mean"][0].data_ptr(),
             run_bufs["running_var"][0].data_ptr(), nbt.data_ptr(), _st())
    assert int(nbt) == 8
    ref = R.bn_stats(z.double(), gamma.double(), beta.double(), 1e-5, 0.1, rm0.double(), rv0.double())
    for k, (r, b) in ref.items():
        buf, inside = outs[k] if k in outs else run_bufs[k]
        _check("6 bn_stats", buf[:C], r, b, f"bn_stats {k} M{M} C{C}")
        _assert_untouched(buf, inside, f"bn_stats {k}")


AFF_FACTORS = dict(
    act=[None, "relu", "hswish", "gelu"],
    C=[8, 24, 40, 256, 2560],
    M=[1, 77, 513, 20000],
    scale=[True, False],               # False: bias-only (fewer_norm layers)
    res=[False, True],
)
AFF_DESIGN = _pairwise(AFF_FACTORS, seed=15)


# every (act, scale, residual) combination the training graphs pass, once each (the bias-less rows: TinyViT's GELU after the add)
AFF_ROUTES = [(a, 64, 300, s, r, sh) for a in (None, "relu", "hswish", "gelu") for s in (True, False) for r in (False, True)
              for sh in ((True, False) if not s else (True,))]
AFF_ROWS = [c + (True,) for c in AFF_DESIGN] + AFF_ROUTES


@pytest.mark.parametrize("act,C,M,has_scale,res,has_shift", AFF_ROWS, ids=[f"{c[0]}-C{c[1]}-M{c[2]}{'' if c[3] else '-noscale'}"
                                                                          f"{'-res' if c[4] else ''}{'' if c[5] else '-noshift'}"
                                                                          for c in AFF_ROWS])
def test_affine_act(cuda, act, C, M, has_scale, res, has_shift):
    lib = _lib(cuda)
    g = _gen(cuda, "aff", act, C, M, has_scale, res, has_shift)
    z = _bf(torch.randn(M, C, device=cuda, generator=g) * 3)
    scale = torch.rand(C, device=cuda, generator=g) + 0.5 if has_scale else None
    shift = torch.randn(C, device=cuda, generator=g) if has_shift else None
    r = _bf(torch.randn(M, C, device=cuda, generator=g)) if res else None
    buf, inside = _flat_out(M * C, torch.bfloat16, cuda)
    lib.call("es3_affine_act", z.data_ptr(), _p(scale), _p(shift), ACT_CODE[act], _p(r), buf.data_ptr(), M, C, _st())
    d = lambda t: None if t is None else t.double()
    ref, bound = R.affine_act(z.double(), d(scale), d(shift), act, d(r))
    what = f"affine_act {act} M{M} C{C} scale={has_scale} res={res} shift={has_shift}"
    _check("6 affine_act", buf[:M * C].view(M, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


BNB_FACTORS = dict(
    mode=["none", "eval", "batch"],
    act=[None, "relu", "hswish", "gelu"],
    C=[8, 24, 40, 64, 2560],           # C % 32 != 0; 2560: gy > 1
    M=[1, 7, 300, 4099, 20000],        # ragged against the rows per block of the ring reduction
    has_scale=[True, False],           # False: bias-only in mode none (scale 1 with given statistics otherwise)
)
BNB_DESIGN = _pairwise(BNB_FACTORS, seed=16)


def bn_bwd_case(cuda, mode, act, C, M, has_scale, seed=()):
    g = _gen(cuda, "bnb", mode, act, C, M, has_scale, *seed)
    z = _bf(torch.randn(M, C, device=cuda, generator=g) * (torch.rand(C, device=cuda, generator=g) + 0.3)
            + torch.randn(C, device=cuda, generator=g))
    da = torch.randn(M, C, device=cuda, generator=g)
    gamma = torch.rand(C, device=cuda, generator=g) + 0.5
    beta = torch.randn(C, device=cuda, generator=g) * 0.5
    mean = invstd = None
    if mode == "none":
        scale, shift = (gamma * 2 if has_scale else None), beta
    else:
        if mode == "eval":
            mean = torch.randn(C, device=cuda, generator=g) * 0.5
            invstd = torch.rsqrt(torch.rand(C, device=cuda, generator=g) + 0.5)
        else:
            zd = z.double()
            mean = zd.mean(0).float()
            invstd = torch.rsqrt(zd.var(0, unbiased=False) + 1e-5).float()
        scale = (gamma * invstd) if has_scale else None
        shift = beta - mean * (scale if scale is not None else 1.0)
    u = z.double() * (scale.double() if scale is not None else 1.0) + shift.double()
    da = _bf(torch.where(R.kink_band(u, act), 0.0, da))
    return z, da, scale, shift, mean, invstd


# every (act, mode, scale) combination, once each: the training graphs reach most of them (the pairwise design only covers pairs)
BNB_ROUTES = [(m, a, 40, 777, s) for m in ("none", "eval", "batch") for a in (None, "relu", "hswish", "gelu") for s in (True, False)]
BNB_ROWS = BNB_DESIGN + BNB_ROUTES


@pytest.mark.parametrize("mode,act,C,M,has_scale", BNB_ROWS, ids=[f"{c[0]}-{c[1]}-C{c[2]}-M{c[3]}{'' if c[4] else '-noscale'}"
                                                                  for c in BNB_ROWS])
def test_bn_act_bwd(cuda, mode, act, C, M, has_scale):
    """es3_bn_act_bwd_reduce (dbeta, dgamma accumulated, the coef of bn_bwd_finalize_kernel) and es3_bn_act_bwd_apply."""
    lib = _lib(cuda)
    z, da, scale, shift, mean, invstd = bn_bwd_case(cuda, mode, act, C, M, has_scale)
    dg0 = torch.full((C,), 0.25, device=cuda)
    db0 = torch.full((C,), -0.5, device=cuda)
    red = []
    for v0 in (dg0, db0):
        b, ins = _flat_out(C, torch.float32, cuda)
        b[:C] = v0
        red.append((b, ins))
    coef, cins = _flat_out(3 * C, torch.float32, cuda)
    ws = _nan_ws(lib, "es3_col_reduce_ws_floats", M, C, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_bn_act_bwd_reduce", da.data_ptr(), z.data_ptr(), _p(scale), _p(shift), ACT_CODE[act], BN_MODE[mode],
                 _p(mean), _p(invstd), M, C, ws.data_ptr(), bufs[0].data_ptr(), bufs[1].data_ptr() if mode != "none" else 0,
                 bufs[2].data_ptr(), _st())
    coef, dgb, dbb = _twice(run, coef, red[0][0], red[1][0])
    _assert_untouched(coef, cins, "coef")
    dz, dzins = _flat_out(M * C, torch.bfloat16, cuda)
    lib.call("es3_bn_act_bwd_apply", da.data_ptr(), z.data_ptr(), _p(scale), _p(shift), ACT_CODE[act], coef.data_ptr(),
             dz.data_ptr(), M, C, _st())
    d = lambda t: None if t is None else t.double()
    ref = R.bn_act_bwd(da.double(), z.double(), d(scale), d(shift), act, mode, d(mean), d(invstd), dg0.double(), db0.double())
    what = f"bn_act_bwd {mode} {act} M{M} C{C} scale={has_scale}"
    _check("6 bn_act_bwd dz", dz[:M * C].view(M, C), *ref["dz"], what + " dz")
    _assert_untouched(dz, dzins, what + " dz")
    _check("6 bn_act_bwd dbeta", dbb[:C], *ref["dbeta"], what + " dbeta")
    _assert_untouched(dbb, red[1][1], what + " dbeta")
    if mode != "none":
        _check("6 bn_act_bwd dgamma", dgb[:C], *ref["dgamma"], what + " dgamma")
        _assert_untouched(dgb, red[0][1], what + " dgamma")
    else:
        assert torch.equal(dgb[:C], dg0), "dgamma written in mode none"


# ----------------------------------------------------------------------------------------------------------- (7) element-wise pieces
@pytest.mark.parametrize("M,C,lda,ldb,ldo", [(999, 384, 768, 392, 400), (1, 8, 16, 24, 32), (4097, 24, 48, 32, 40),
                                             (65536, 64, 128, 72, 80)])
def test_add_bf16_bit_exact(cuda, M, C, lda, ldb, ldo):
    """All three row strides != C; bit-identical to torch's bf16 add; columns C .. ldo - 1 of the output keep their sentinels."""
    lib = _lib(cuda)
    g = _gen(cuda, "add", M, C)
    A = torch.full((M, lda), float("nan"), device=cuda, dtype=torch.bfloat16)
    Bm = torch.full((M, ldb), float("nan"), device=cuda, dtype=torch.bfloat16)
    A[:, lda - C:] = _bf(torch.randn(M, C, device=cuda, generator=g))
    Bm[:, :C] = _bf(torch.randn(M, C, device=cuda, generator=g))
    a, b = A[:, lda - C:], Bm[:, :C]
    buf, inside, idx = _strided_out(M, C, ldo, torch.bfloat16, cuda)
    lib.call("es3_add_bf16", a.data_ptr(), lda, b.data_ptr(), ldb, buf.data_ptr(), ldo, M, C, _st())
    assert torch.equal(buf[idx].view(M, C).view(torch.int16), (a + b).view(torch.int16))
    _assert_untouched(buf, inside, "add_bf16")


def _se_case(cuda, B, HW, C):
    lib = _lib(cuda)
    g = _gen(cuda, "se", B, HW, C)
    dy = _bf(torch.randn(B, HW, C, device=cuda, generator=g))
    x = _bf(torch.randn(B, HW, C, device=cuda, generator=g))
    dg0 = torch.randn(B, C, device=cuda, generator=g)
    buf, inside = _flat_out(B * C, torch.float32, cuda)
    buf[:B * C] = dg0.reshape(-1)
    ws = _nan_ws(lib, "es3_se_bwd_ws_floats", B, HW, C, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_se_bwd_dgate", dy.data_ptr(), x.data_ptr(), B, HW, C, ws.data_ptr(), bufs[0].data_ptr(), _st())
    got = _twice(run, buf)[0]
    ref, bound = R.se_dgate(dy.double(), x.double(), dg0.double())
    _check("7 se_dgate", got[:B * C].view(B, C), ref, bound, f"se_dgate B{B} HW{HW} C{C}")
    _assert_untouched(got, inside, "se_dgate")
    gate, add = torch.rand(B, C, device=cuda, generator=g), torch.randn(B, C, device=cuda, generator=g) * 0.1
    out, oins = _flat_out(B * HW * C, torch.bfloat16, cuda)
    lib.call("es3_se_bwd_apply", dy.data_ptr(), gate.data_ptr(), add.data_ptr(), out.data_ptr(), B, HW, C, _st())
    ref, bound = R.se_apply(dy.double(), gate.double(), add.double())
    _check("7 se_apply", out[:B * HW * C].view(B, HW, C), ref, bound, f"se_apply B{B} HW{HW} C{C}")
    _assert_untouched(out, oins, "se_apply")


# (16: 4096-pixel chunks; 512: 128-pixel chunks, 64-chunk cap above 8192 pixels; 2560: two passes over the channel vectors)
SE_CASES = [(3, 4097, 16), (2, 81, 16), (4, 8193, 512), (2, 9000, 512), (3, 256, 64), (2, 25, 2560), (1, 4096, 2560),
            (1, 16384, 48), (2, 1024, 96)]


@pytest.mark.parametrize("B,HW,C", SE_CASES)
def test_se_bwd(cuda, B, HW, C):
    """SqueezeExcite backward with several images: HW ragged against se_chunks, the 64-chunk cap, C = 2560; the last two rows are
    RepViT's SE layers at 1024^2."""
    _se_case(cuda, B, HW, C)


STEM_CASES = [(2, 3, 8, 37, 51), (1, 3, 16, 64, 64), (3, 3, 24, 33, 47), (1, 3, 32, 9, 7), (2, 3, 16, 511, 513),
              (1, 3, 24, 1024, 1024), (2, 3, 32, 1023, 1025)]


@pytest.mark.parametrize("B,ci,Cout,H,W", STEM_CASES)
def test_stem_wgrad(cuda, B, ci, Cout, H, W):
    """Cout 8 .. 32, odd H and W, chunk counts below and above the 592-block cap (1024^2: stage-1's stem, 2048 chunks)."""
    lib = _lib(cuda)
    g = _gen(cuda, "stem", B, Cout, H, W)
    img = torch.randn(B, 3, H, W, device=cuda, generator=g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dz = _bf(torch.randn(B, Ho, Wo, Cout, device=cuda, generator=g))
    dW0 = torch.randn(Cout, 3, 3, 3, device=cuda, generator=g)
    buf, inside = _flat_out(Cout * 27, torch.float32, cuda)
    buf[:Cout * 27] = dW0.reshape(-1)
    ws = _nan_ws(lib, "es3_stem_wgrad_ws_floats", B, H, W, Cout, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_stem_wgrad", img.data_ptr(), dz.data_ptr(), B, H, W, Cout, ws.data_ptr(), bufs[0].data_ptr(), _st())
    got = _twice(run, buf)[0]
    ref, bound = R.stem_wgrad(img.double(), dz.double(), dW0.double())
    what = f"stem_wgrad B{B} {H}x{W} Cout{Cout}"
    _check("7 stem_wgrad", got[:Cout * 27].view(Cout, 3, 3, 3), ref, bound, what)
    _assert_untouched(got, inside, what)


@pytest.mark.parametrize("C,rd", [(48, 8), (96, 24), (1024, 256)])
def test_se_weight_gradient_at_batch_one(cuda, C, rd):
    """The SqueezeExcite fc weight gradients of RepViT's training graph at batch 1: dpre^T h on es3_gemm_simt, whose operands
    x.t().contiguous() of [1, C] tensors are single columns with column stride C (they used to fail the wrapper's stride check)."""
    from efficientsam3_b200 import ops
    g = _gen(cuda, "se1", C, rd)
    dpre, h = torch.randn(1, C, device=cuda, generator=g), torch.randn(1, rd, device=cuda, generator=g).clamp_min(0)
    a, w = dpre.t().contiguous(), h.t().contiguous()
    assert a.shape == (C, 1) and a.stride(1) != 1
    got = ops.gemm_simt(a, w, out_dtype=torch.float32)
    ref = dpre.double().t() @ h.double()
    _check("7 se fc wgrad", got, ref, 4 * R.U * ref.abs() + R.TINY, f"SE fc weight gradient C{C} rd{rd}")


# ----------------------------------------------------------------------------------------------------------- (8) es3_bilinear_bwd
BIL_CASES = [(2, 64, 5, 5, 10, 10), (1, 40, 16, 16, 63, 63), (2, 96, 10, 7, 9, 20), (1, 32, 64, 48, 20, 17), (2, 8, 3, 4, 11, 15),
             (1, 1024, 32, 32, 64, 64), (2, 256, 32, 32, 64, 64)]


@pytest.mark.parametrize("B,C,Hi,Wi,Ho,Wo", BIL_CASES)
def test_bilinear_bwd(cuda, B, C, Hi, Wi, Ho, Wo):
    """Up by 2, by 3.94 (close to the 12-candidate limit), down-scaling, C % 32 != 0, and the EfficientViT students' 32^2 -> 64^2
    resize at 1024^2."""
    lib = _lib(cuda)
    dout = torch.randn(B, C, Ho, Wo, device=cuda, generator=_gen(cuda, "bil", B, C, Hi, Wi, Ho, Wo))
    buf, inside = _flat_out(B * Hi * Wi * C, torch.bfloat16, cuda)
    lib.call("es3_bilinear_bwd", dout.data_ptr(), buf.data_ptr(), B, Hi, Wi, C, Ho, Wo, _st())
    ref, bound = R.bilinear_bwd(dout.double(), Hi, Wi)
    what = f"bilinear_bwd B{B} C{C} {Hi}x{Wi} <- {Ho}x{Wo}"
    _check("8 bilinear_bwd", buf[:B * Hi * Wi * C].view(B, Hi, Wi, C), ref, bound, what)
    _assert_untouched(buf, inside, what)


# ----------------------------------------------------------------------------------------------------------- (9) LiteMLA backward
def _litemla(cuda, B, HW, heads2, dim, generic, pad, seed=()):
    """kv from the forward kernel, as in training; ms / dy / dms with row strides ld + pad (NaN-padded, sentinel columns)."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "lm", B, HW, heads2, dim, generic, pad, *seed)
    ld, ldy = 3 * dim * heads2, dim * heads2
    ms = _bf(torch.randn(B, 1, HW, ld, device=cuda, generator=g))
    dy = _bf(torch.randn(B * HW, ldy, device=cuda, generator=g))
    if generic:
        _, kv = ops.litemla_attn_generic(ms, heads2, dim, 1e-15, return_kv=True)
        nchunk_f = (HW + 127) // 128
    else:
        _, kv = ops.litemla_attn(ms, heads2, 1e-15, return_kv=True)
        nchunk_f = (HW + 511) // 512
    msp = _nanpad(ms.view(B * HW, ld), pad)
    dyp = _nanpad(dy, pad)
    buf, inside, idx = _strided_out(B * HW, ld, ld + pad, torch.bfloat16, cuda)
    if generic:
        ws = _nan_ws(lib, "es3_litemla_bwd_generic_ws_floats", B, HW, heads2, dim, cuda=cuda)
        args = ("es3_litemla_attn_bwd_generic", msp.data_ptr(), msp.stride(0), dyp.data_ptr(), dyp.stride(0), kv.data_ptr(),
                nchunk_f, ws.data_ptr(), buf.data_ptr(), ld + pad, B, HW, heads2, dim, 1e-15, _st())
    else:
        ws = _nan_ws(lib, "es3_litemla_bwd_ws_floats", B, HW, heads2, cuda=cuda)
        args = ("es3_litemla_attn_bwd", msp.data_ptr(), msp.stride(0), dyp.data_ptr(), dyp.stride(0), kv.data_ptr(), nchunk_f,
                ws.data_ptr(), buf.data_ptr(), ld + pad, B, HW, heads2, 1e-15, _st())

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call(args[0], *args[1:8], bufs[0].data_ptr(), *args[9:])
    got = _twice(run, buf)[0]
    kvp = kv.view(B, heads2, nchunk_f, dim + 1, dim).double()
    ref, bound = R.litemla_bwd(ms.view(B, HW, ld).double(), dy.view(B, HW, ldy).double(), kvp, heads2, dim, 1e-15)
    what = f"litemla_bwd{'_generic' if generic else ''} B{B} HW{HW} heads2={heads2} dim{dim} pad{pad}"
    _check("9 litemla_bwd" + ("_generic" if generic else ""), got[idx].view(B, HW, ld), ref, bound, what)
    _assert_untouched(got, inside, what)


@pytest.mark.parametrize("generic,dim", [(False, 16), (True, 16), (True, 32)])
def test_litemla_bwd_every_small_hw(cuda, generic, dim):
    """HW = 1 .. 129, every value: ragged against the 128-pixel chunks of the backward (and the 512-pixel forward chunks)."""
    for HW in range(1, 130):
        _litemla(cuda, 2, HW, 4, dim, generic, 8 * (HW % 3))


LM_CASES = [(False, 16, 2, 511, 8, 16), (False, 16, 1, 513, 4, 0), (False, 16, 2, 1025, 6, 8), (True, 16, 2, 257, 6, 16),
            (True, 32, 1, 383, 8, 8), (True, 32, 2, 640, 4, 0),
            (False, 16, 1, 4096, 16, 0), (False, 16, 2, 1024, 32, 0), (True, 32, 1, 4096, 16, 0), (True, 32, 2, 1024, 32, 0)]


@pytest.mark.parametrize("generic,dim,B,HW,heads2,pad", LM_CASES)
def test_litemla_bwd(cuda, generic, dim, B, HW, heads2, pad):
    """Forward chunks of 512 pixels ragged (511, 513, 1025), strided ld; the last four rows are the LiteMLA stages of EfficientViT
    b1 (dim 16) and b2 (dim 32) at 1024^2 (64^2 and 32^2 maps)."""
    _litemla(cuda, B, HW, heads2, dim, generic, pad)


# ----------------------------------------------------------------------------------------------------------- (10) TinyViT pieces
LN_FACTORS = dict(
    C=[8, 64, 160, 448, 576, 1024],
    M=[1, 63, 65, 4100, 40000],
    dres=[False, True],
)
LN_DESIGN = _pairwise(LN_FACTORS, seed=17)


@pytest.mark.parametrize("C,M,dres", LN_DESIGN + [(64, 65536, True), (128, 16384, False), (320, 4096, True)],
                         ids=[f"C{c[0]}-M{c[1]}{'-dres' if c[2] else ''}" for c in LN_DESIGN + [(64, 65536, True), (128, 16384, False),
                                                                                             (320, 4096, True)]])
def test_layernorm_bwd(cuda, C, M, dres):
    """LayerNorm backward up to C = 1024, with and without the residual gradient; the last three rows are TinyViT 5m's stage widths
    at 1024^2."""
    lib = _lib(cuda)
    g = _gen(cuda, "ln", C, M, dres)
    x = _bf(torch.randn(M, C, device=cuda, generator=g) * 2 + 0.5)
    dy = _bf(torch.randn(M, C, device=cuda, generator=g))
    r = _bf(torch.randn(M, C, device=cuda, generator=g)) if dres else None
    gamma = torch.rand(C, device=cuda, generator=g) + 0.5
    dx, dxins = _flat_out(M * C, torch.bfloat16, cuda)
    acc = []
    for v in (0.5, -1.0):
        b, ins = _flat_out(C, torch.float32, cuda)
        b[:C] = v
        acc.append((b, ins))
    ws = _nan_ws(lib, "es3_layernorm_bwd_ws_floats", M, C, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_layernorm_bwd", x.data_ptr(), dy.data_ptr(), gamma.data_ptr(), _p(r), 1e-5, bufs[0].data_ptr(), M, C,
                 ws.data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), _st())
    dx, dg, db = _twice(run, dx, acc[0][0], acc[1][0])
    ref = R.layernorm_bwd(x.double(), dy.double(), gamma.double(), 1e-5, torch.full((C,), 0.5, dtype=torch.float64, device=cuda),
                          torch.full((C,), -1.0, dtype=torch.float64, device=cuda), None if r is None else r.double())
    what = f"layernorm_bwd M{M} C{C} dres={dres}"
    _check("10 layernorm_bwd dx", dx[:M * C].view(M, C), *ref["dx"], what)
    _check("10 layernorm_bwd dgamma", dg[:C], *ref["dgamma"], what + " dgamma")
    _check("10 layernorm_bwd dbeta", db[:C], *ref["dbeta"], what + " dbeta")
    for b, (_, ins) in zip((dx, dg, db), ((None, dxins), *acc)):
        _assert_untouched(b, ins, what)


WIN_CASES = [(2, 14, 21, 4, 7, 0), (1, 14, 28, 8, 14, 64), (3, 7, 7, 5, 7, 8), (2, 28, 14, 2, 14, 0), (1, 64, 64, 4, 7, 8),
             (1, 70, 70, 5, 7, 0), (1, 28, 28, 16, 14, 0)]


@pytest.mark.parametrize("B,H,W,heads,ws,extra", WIN_CASES)
def test_win_attn_bias_bwd(cuda, B, H, W, heads, ws, extra):
    """Windows 7 and 14 over several windows and images; dS written through ldS = heads N^2 + extra (its columns past heads N^2 keep
    their sentinels).  The last three rows are TinyViT's stages at 1024^2 (64^2 -> 70^2 padded for the 7-windows, 32^2 -> 28^2...)."""
    lib = _lib(cuda)
    g = _gen(cuda, "win", B, H, W, heads, ws, extra)
    C, N = 32 * heads, ws * ws
    H, W = H // ws * ws, W // ws * ws
    qkv = _bf(torch.randn(B * H * W, 3 * C, device=cuda, generator=g))
    dout = _bf(torch.randn(B * H * W, C, device=cuda, generator=g))
    bias = torch.randn(heads, N, N, device=cuda, generator=g) * 0.5
    scale = 32 ** -0.5
    nwin = B * (H // ws) * (W // ws)
    row = heads * N * N
    ldS = row + extra
    dS, dSins, dSidx = _strided_out(nwin, row, ldS, torch.float32, cuda)
    dq, dqins = _flat_out(B * H * W * 3 * C, torch.bfloat16, cuda)
    lib.call("es3_win_attn_bias_bwd", qkv.data_ptr(), dout.data_ptr(), bias.data_ptr(), dq.data_ptr(), dS.data_ptr(), ldS, B, H, W,
             C, heads, ws, scale, _st())
    ref = R.win_attn_bias_bwd(qkv.double(), dout.double(), bias.double(), B, H, W, C, heads, ws, scale)
    what = f"win_attn_bias_bwd B{B} {H}x{W} heads{heads} ws{ws} ldS+{extra}"
    _check("10 win_attn_bias_bwd dqkv", dq[:B * H * W * 3 * C].view(B * H * W, 3 * C), *ref["dqkv"], what)
    _check("10 win_attn_bias_bwd dS", dS[dSidx].view(nwin, heads, N, N), *ref["dS"], what + " dS")
    _assert_untouched(dq, dqins, what)
    _assert_untouched(dS, dSins, what + " dS")


@pytest.mark.parametrize("M,L,ld", [(1, 5, 5), (37, 130, 136), (4000, 784, 800), (200000, 5, 16), (3, 38416, 38424), (1154, 9604, 9604)])
def test_colsum_f32(cuda, M, L, ld):
    """Column sums with ld > L (NaN in the columns past L) and very tall M; the last row is TinyViT's 7-window bias gradient at
    1024^2."""
    lib = _lib(cuda)
    g = _gen(cuda, "colsum", M, L, ld)
    src = torch.full((M, ld), float("nan"), device=cuda)
    src[:, :L] = torch.randn(M, L, device=cuda, generator=g)
    o0 = torch.randn(L, device=cuda, generator=g)
    buf, inside = _flat_out(L, torch.float32, cuda)
    buf[:L] = o0
    ws = _nan_ws(lib, "es3_colsum_f32_ws_floats", M, L, cuda=cuda)

    def run(bufs):
        ws.fill_(float("nan"))
        lib.call("es3_colsum_f32", src.data_ptr(), ld, M, L, ws.data_ptr(), bufs[0].data_ptr(), _st())
    got = _twice(run, buf)[0]
    ref, bound = R.colsum(src[:, :L].double(), o0.double())
    _check("10 colsum", got[:L], ref, bound, f"colsum M{M} L{L} ld{ld}")
    _assert_untouched(got, inside, "colsum")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above exercises."""
    keys = set()
    keys |= {key_wgrad_pw(c[0], c[1], False) for c in WGPW_DESIGN}
    keys |= {key_wgrad_pw(N, C, True) for _, _, _, N, C in [(2, 9, 7, 32, 16), (1, 12, 12, 64, 128), (3, 5, 33, 24, 8),
                                                             (2, 16, 16, 136, 48), (1, 128, 128, 48, 24)]}
    keys |= {key_wgrad_pw(N, C, True) for _, _, _, N, C in [(2, 10, 14, 24, 8), (1, 32, 32, 48, 16), (1, 512, 512, 24, 8)]}
    keys |= {key_wgrad_tc(c[0]) for c in WGTC_DESIGN}
    keys |= {key_dw_bwd_data(c[4], c[5]) for c in DWBD_CASES}
    keys |= {("es3_dwconv_wgrad",) + c[1] for c in DWD_DESIGN} | {("es3_dwconv_wgrad_win",) + c[1] for c in DWW_DESIGN}
    keys |= {("es3_bn_act_bwd_reduce", c[1], c[0], c[4]) for c in BNB_ROWS}
    keys |= {("es3_bn_act_bwd_apply", c[1], c[4]) for c in BNB_ROWS}
    keys |= {("es3_affine_act", c[0], c[3], c[4]) for c in AFF_ROWS}
    keys |= {("es3_stem_wgrad", c[2]) for c in STEM_CASES}
    keys |= {("es3_litemla_attn_bwd_generic", c[1]) for c in LM_CASES if c[0]}
    keys |= {("es3_layernorm_bwd", c[2]) for c in LN_DESIGN}
    keys |= {("es3_win_attn_bias_bwd", c[4]) for c in WIN_CASES}
    keys |= {(k,) for k in ("es3_bn_stats", "es3_add_bf16", "es3_se_bwd_dgate", "es3_se_bwd_apply", "es3_bilinear_bwd",
                            "es3_litemla_attn_bwd", "es3_colsum_f32", "es3_transpose_pad_bf16", "es3_accumulate_strided")}
    return keys
