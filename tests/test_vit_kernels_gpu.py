"""The SAM3 ViT trunk's kernels (attention_tc.cu's wgmma and attention.cu's mma.sync flash attention at the trunk's windowed and global
shapes, vit_ops.cu's patch im2col and token layout change, and the strict-mode sgemm_f32, rope_f32, attention_f32, ln_rows_f32 and
im2col_f32 of strict_f32.cu), element by element against the fp64 statements of tests/ref_vit.py, each output element within its
own bound; the exact operations bit for bit.

Outputs are NaN-prefilled and called through _lib.call: every cell inside the output region must be written and lie within its
bound, every cell past it (a flat TAIL, or the columns around a strided output) keeps its sentinel bits; rope_f32 works in place
and must keep the bits of the v block and of the row padding.  Every case runs twice and must be bit-identical; the last image run
alone must be bit-identical to the same image inside the batch; es3_attention_bf16 and the ops wrappers are bit-identical to the
direct entry point they pick; a shape or pointer an entry point declines writes nothing.  covered_keys() names the route keys
(tests/routes.py) the tables run, for the route closure of tests/test_route_closure_gpu.py (the 1008 px teacher, bf16 and strict,
the 336 and vit_small_112 trunks and Sam3PointPromptSegmenter.set_image).  The strict SGEMM table also holds the strict students'
GEMM routes: their folded-BatchNorm epilogues and RepViT's SqueezeExcite fc1 (ReLU) and fc2 (sigmoid gate) on the pooled rows.

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power
limit): bf16 attention -- wgmma BN 96 0.888 (windowed) and 0.612 (global), BN 128 0.931 (global) and 0.945 (windowed), mma.sync MT 1
0.938 (windowed) and 0.9 (global), MT 2 0.919 (windowed) and 0.618 (global), where the output's own rounding half-step dominates the
bound; fp32 outputs -- sgemm_f32 0.239, rope_f32 0.249, attention_f32 0.0086 (head_dim 32) and 0.0048 (head_dim 64), ln_rows_f32
0.022.  The whole file (128 tests, the route-closure forwards included, since moved to tests/test_route_closure_gpu.py) took 14 s
there.
"""
import functools

import pytest
import torch

import ref_vit as R
from bounds import (_assert_untouched, _bits_equal, _check, _declined, _flat_out, _gen, _lib, _matrix_out, _p, _padded, _pairwise,
                    _qkv, _st, _twice, report_worst)
from routes import attn_key

pytestmark = pytest.mark.gpu
_report_worst = report_worst("ViT kernels")
BF = torch.bfloat16


def _ops():
    from efficientsam3_b200 import ops
    return ops


def _last_image(B, n):
    return slice((B - 1) * n, B * n)


# ----------------------------------------------------------------------------------------------------------- (1) wgmma attention
TC = [  # B, H, W, heads, win, kind, scale
    (1, 72, 72, 16, 24, "normal", 0.125),      # the teacher's windowed blocks: L 576 on 96-key tiles, 16 heads, C 1024
    (2, 72, 72, 2, 24, "peaked", 0.125),
    (1, 72, 72, 2, 0, "normal", 0.125),        # the teacher's global blocks: L 5184, 54 key tiles of 96, 40.5 query tiles
    (2, 72, 72, 1, 0, "tied", 0.125),
    (1, 12, 16, 2, 0, "flat", 0.125),          # L 192: BN 96, two key tiles, 1.5 query tiles
    (2, 24, 24, 2, 0, "tied", 0.125),          # L 576 global
    (1, 16, 24, 2, 0, "peaked", 0.125),        # L 384: a multiple of 96 and of 128 -> BN 128
    (3, 10, 20, 2, 0, "normal", 0.3),          # L 200: BN 128, a partial key tile; scale 0.3
    (1, 20, 32, 1, 0, "flat", 0.125),          # L 640: BN 128, five key tiles
    (2, 36, 24, 2, 12, "normal", 0.125),       # win 12 (L 144: partial key and query tiles) on a 3 x 2 window grid
    (1, 32, 80, 2, 16, "tied", 0.2),           # win 16 (L 256) on a 2 x 5 grid
    (1, 48, 72, 4, 24, "peaked", 0.125),       # win 24 on a 2 x 3 grid
    (3, 6, 10, 2, 2, "normal", 0.125),         # L 4 on a 3 x 5 grid: one partial key tile, a query tile of 124 padded rows
    (2, 8, 8, 4, 4, "tied", 0.125),            # L 16
    (1, 24, 24, 2, 8, "peaked", 0.125),        # L 64
]


def _attn(lib, name, qkv, o, B, H, W, heads, win, scale):
    lib.call(name, qkv.data_ptr(), o.data_ptr(), B, H, W, 64 * heads, heads, win, scale, _st())


def _attn_case(cuda, name, kernel, B, H, W, heads, win, kind, scale):
    lib = _lib(cuda)
    g = _gen(cuda, name, B, H, W, heads, win, kind, scale)
    C, n = 64 * heads, B * H * W
    qkv = _qkv(cuda, 1, n, heads, kind, g)
    buf, ins = _flat_out(n * C, BF, cuda)
    got = _twice(lambda o: _attn(lib, name, qkv, o, B, H, W, heads, win, scale), buf)
    o = got[:n * C].view(n, C)
    ref, bound = R.attention_bf16(qkv.double(), B, H, W, heads, win, scale, kernel)
    key = attn_key(name, H, W, win)
    what = f"{name} B{B} {H}x{W} heads{heads} win{win} {kind} scale {scale}"
    _check(f"1 {key}", o, ref, bound, what)
    _assert_untouched(got, ins, what)
    if attn_key("es3_attention_bf16", H, W, win)[1:] == key[1:]:
        d = torch.full((n, C), float("nan"), dtype=BF, device=cuda)
        _attn(lib, "es3_attention_bf16", qkv, d, B, H, W, heads, win, scale)
        _bits_equal(d, o, what + ": es3_attention_bf16 vs the direct call")
        _bits_equal(_ops().attention(qkv, B, H, W, C, heads, win, scale), o, what + ": ops.attention vs the direct call")
    _bits_equal(_ops().attention(qkv, B, H, W, C, heads, win, scale, impl=kernel), o, what + f": ops.attention({kernel}) vs direct")
    if B > 1:
        sl = _last_image(B, H * W)
        one = torch.full((H * W, C), float("nan"), dtype=BF, device=cuda)
        _attn(lib, name, qkv[sl].contiguous(), one, 1, H, W, heads, win, scale)
        _bits_equal(one, o[sl], what + ": last image alone")


@pytest.mark.parametrize("B,H,W,heads,win,kind,scale", TC)
def test_attention_tc(cuda, B, H, W, heads, win, kind, scale):
    """attn_tc_kernel<96> and <128>, windowed (window gather on square and non-square grids) and global, one to 54 key tiles,
    partial key and query tiles, and windows of L < 128 (which es3_attention_bf16 sends to the mma.sync kernel, but ops.attention(impl
    = "tc") and the entry point accept)."""
    _attn_case(cuda, "es3_attention_tc_bf16", "tc", B, H, W, heads, win, kind, scale)


# ----------------------------------------------------------------------------------------------------------- (2) mma.sync attention
MMA = [  # B, H, W, heads, win, kind
    (2, 8, 8, 2, 4, "normal"),                 # L 16, MT 1 (the vit_small_112 windows)
    (1, 16, 40, 2, 8, "peaked"),               # L 64 on a 2 x 5 window grid (the 336 trunk's windows)
    (2, 18, 27, 1, 9, "tied"),                 # L 81: a partial key tile, 2 x 3 grid
    (2, 10, 10, 1, 0, "normal"),               # global L 100, MT 1
    (3, 24, 24, 2, 12, "flat"),                # L 144, MT 2: a partial key tile
    (1, 32, 48, 2, 16, "normal"),              # L 256, MT 2 on a 2 x 3 grid
    (2, 48, 48, 1, 24, "peaked"),              # L 576, MT 2
    (1, 24, 24, 2, 0, "tied"),                 # global L 576, MT 2
    (1, 36, 20, 2, 0, "peaked"),               # global L 720, MT 2: a partial key tile
    (1, 72, 72, 1, 0, "normal"),               # global L 5184, MT 2: 81 key tiles
]


@pytest.mark.parametrize("B,H,W,heads,win,kind", MMA)
def test_attention_mma(cuda, B, H, W, heads, win, kind):
    """attn_fwd_kernel (non-causal) at MT 1 and 2, windowed and global up to L 5184 (81 key tiles), L % 64 != 0."""
    _attn_case(cuda, "es3_attention_mma_bf16", "mma", B, H, W, heads, win, kind, 0.125)


def test_attention_declined_arguments_write_nothing(cuda):
    """A negative window, B, H or W = 0, qkv off 16 bytes, out off 16 bytes (mma.sync) or 4 bytes (wgmma): declined by each entry
    point and by the dispatcher, nothing written."""
    lib = _lib(cuda)
    heads, C = 2, 128
    z = torch.zeros(16 * 16 * 3 * C + 64, dtype=BF, device=cuda)
    out, _ = _flat_out(16 * 16 * C + 64, BF, cuda)
    q0, o0 = z.data_ptr(), out.data_ptr()
    for name in ("es3_attention_tc_bf16", "es3_attention_mma_bf16", "es3_attention_bf16"):
        cases = [((q0, o0, 1, 16, 16, C, heads, -8, 0.125), "win -8"), ((q0, o0, 0, 16, 16, C, heads, 8, 0.125), "B 0"),
                 ((q0, o0, 1, 0, 16, C, heads, 0, 0.125), "H 0"), ((q0, o0, 1, 16, 0, C, heads, 0, 0.125), "W 0"),
                 ((q0 + 8, o0, 1, 16, 16, C, heads, 8, 0.125), "qkv + 8 bytes"),
                 ((q0, o0 + 2, 1, 16, 16, C, heads, 8 if name != "es3_attention_tc_bf16" else 0, 0.125), "out + 2 bytes")]
        if name == "es3_attention_mma_bf16":
            cases.append(((q0, o0 + 4, 1, 16, 16, C, heads, 8, 0.125), "out + 4 bytes"))
        for args, what in cases:
            _declined(lib, name, args + (_st(),), [out], f"{name} {what}")


# ----------------------------------------------------------------------------------------------------------- (3) patch im2col
PATCH = [(1, 1008, 14, 592), (3, 336, 14, 592), (1, 112, 14, 592), (3, 112, 14, 600), (2, 336, 14, 640)]


@pytest.mark.parametrize("B,S,P,Kp", PATCH)
def test_im2col_patch(cuda, B, S, P, Kp):
    """Bit-exact against bf16(F.unfold); the pad columns 3 P^2 .. Kp are +0 exactly; ops.im2col_patch bit-identical."""
    lib = _lib(cuda)
    x = torch.randn(B, 3, S, S, device=cuda, generator=_gen(cuda, "patch", B, S, Kp))
    n = B * (S // P) ** 2
    buf, ins = _flat_out(n * Kp, BF, cuda)
    got = _twice(lambda o: lib.call("es3_im2col_patch", x.data_ptr(), o.data_ptr(), B, S, P, Kp, _st()), buf)
    cols = got[:n * Kp].view(n, Kp)
    what = f"im2col_patch B{B} S{S} Kp{Kp}"
    _bits_equal(cols, R.im2col_patch(x, P, Kp), what)
    assert int((cols[:, 3 * P * P:].view(torch.int16) != 0).sum()) == 0, what + ": pad columns are not +0"
    _assert_untouched(got, ins, what)
    _bits_equal(_ops().im2col_patch(x, P, Kp), cols, "ops.im2col_patch vs direct")
    if B > 1:
        one = torch.full((n // B, Kp), float("nan"), dtype=BF, device=cuda)
        lib.call("es3_im2col_patch", x[-1:].contiguous().data_ptr(), one.data_ptr(), 1, S, P, Kp, _st())
        _bits_equal(one, cols[_last_image(B, n // B)], what + ": last image alone")


def test_im2col_patch_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    x = torch.zeros(3 * 112 * 112, device=cuda)
    out, _ = _flat_out(64 * 600, BF, cuda)
    for B, S, P, Kp in ((0, 112, 14, 592), (1, 110, 14, 592), (1, 112, 14, 584), (1, 112, 14, 596)):
        _declined(lib, "es3_im2col_patch", (x.data_ptr(), out.data_ptr(), B, S, P, Kp, _st()), [out], f"im2col_patch B{B} S{S} Kp{Kp}")


# ----------------------------------------------------------------------------------------------------------- (4) tokens -> NCHW
T2N = [(1, 5184, 1024), (3, 35, 96), (2, 99, 33), (1, 1, 1), (3, 1000, 100), (2, 64, 31)]


@pytest.mark.parametrize("B,HW,C", T2N)
def test_tokens_to_nchw(cuda, B, HW, C):
    lib = _lib(cuda)
    x = torch.randn(B * HW, C, device=cuda, generator=_gen(cuda, "t2n", B, HW, C))
    buf, ins = _flat_out(B * HW * C, torch.float32, cuda)
    got = _twice(lambda o: lib.call("es3_tokens_f32_to_nchw", x.data_ptr(), o.data_ptr(), B, HW, C, _st()), buf)
    y = got[:B * HW * C].view(B, C, HW)
    what = f"tokens_f32_to_nchw B{B} HW{HW} C{C}"
    _bits_equal(y, R.tokens_to_nchw(x, B, HW, C), what)
    _assert_untouched(got, ins, what)
    _bits_equal(_ops().tokens_f32_to_nchw(x, B, 1, HW).view(B, C, HW), y, "ops.tokens_f32_to_nchw vs direct")


def test_tokens_to_nchw_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    x = torch.zeros(64, device=cuda)
    out, _ = _flat_out(64, torch.float32, cuda)
    for B, HW, C in ((0, 8, 8), (1, 0, 8), (1, 8, 0)):
        _declined(lib, "es3_tokens_f32_to_nchw", (x.data_ptr(), out.data_ptr(), B, HW, C, _st()), [out], f"tokens_to_nchw {B} {HW} {C}")


# ----------------------------------------------------------------------------------------------------------- (5) strict SGEMM
SG = _pairwise(dict(M=[1, 63, 64, 65, 300], N=[1, 17, 64, 100, 1024], K=[1, 15, 16, 17, 333, 4736], act=[None, "gelu", "hswish"],
                    after=[False, True], epi=["none", "scale", "bias", "bias_res", "scale_bias_res", "res"], strided=[False, True]),
                seed=21)
SG += [(63, 1024, 588, None, False, "none", False),            # the strict teacher's patch embedding (im2col of 14 x 14 x 3)
       (300, 1024, 1024, None, False, "bias", True),           # qkv
       (65, 1024, 4736, None, False, "bias_res", True),        # fc2 + residual
       (64, 4736, 1024, "gelu", False, "bias", False),         # fc1
       (257, 16, 27, "hswish", False, "scale_bias", False),    # the strict student encoder: BatchNorm folded into scale and bias
       (300, 128, 64, None, False, "scale_bias", True),
       (65, 96, 576, "gelu", False, "scale_bias", False),
       (2, 80, 320, "relu", False, "bias", False),             # the strict RepViT SqueezeExcite: fc1 on the pooled [B, C] rows
       (2, 320, 80, "sigmoid", False, "bias", False),          # fc2, the gate
       (3, 24, 96, "relu", False, "bias", True),
       (3, 96, 24, "sigmoid", False, "bias", True)]


@pytest.mark.parametrize("M,N,K,act,after,epi,strided", SG)
def test_sgemm_f32(cuda, M, N, K, act, after, epi, strided):
    """The 64 x 64 tile ragged in M and N, K % 16 != 0 up to the teacher's fc2, every epilogue flag, strided A, W, output and
    residual; the last row alone; ops.sgemm bit-identical."""
    ops = _ops()
    lib = _lib(cuda)
    g = _gen(cuda, "sgemm", M, N, K, act, after, epi, strided)
    a = _padded(torch.randn(M, K, device=cuda, generator=g), strided)
    w = _padded(torch.randn(N, K, device=cuda, generator=g) / K ** 0.5, strided)
    sc = torch.rand(N, device=cuda, generator=g) + 0.5 if "scale" in epi else None
    bi = torch.randn(N, device=cuda, generator=g) if "bias" in epi else None
    res = _padded(torch.randn(M, N, device=cuda, generator=g), strided) if "res" in epi else None
    buf, _, ins = _matrix_out(M, N, torch.float32, strided, cuda)
    view = (lambda b: b[:M, 8:8 + N]) if strided else (lambda b: b[:M * N].view(M, N))

    def run(b, rows=slice(None)):
        o = view(b)[rows]
        aa, rr = a[rows], None if res is None else res[rows]
        lib.call("es3_sgemm_f32", aa.data_ptr(), aa.stride(0), w.data_ptr(), w.stride(0), o.data_ptr(), o.stride(0), o.shape[0], N, K,
                 _p(sc), _p(bi), ops.ACT[act], _p(rr), 0 if rr is None else rr.stride(0), int(after), _st())
    got = _twice(run, buf)
    d = lambda t: None if t is None else t.double()
    ref, bound = R.sgemm(a.double(), w.double(), d(sc), d(bi), act, d(res), after)
    what = f"sgemm_f32 {M}x{N}x{K} act {act} after={after} {epi} strided={strided}"
    _check("5 sgemm_f32", view(got), ref, bound, what)
    _assert_untouched(got, ins, what)
    if M > 1:
        one = buf.clone()
        run(one, slice(M - 1, M))
        _bits_equal(view(one)[M - 1:], view(got)[M - 1:], what + ": last row alone")
    _bits_equal(ops.sgemm(a, w, scale=sc, bias=bi, act=act, residual=res, act_after_res=after), view(got), "ops.sgemm vs direct")


# ----------------------------------------------------------------------------------------------------------- (6) strict RoPE
@functools.lru_cache(None)
def _teacher_tables():
    """The RoPE tables of the teacher's windowed (24 x 24) and global (72 x 72) blocks, as the module builds them."""
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    vit = create_sam3_vit_backbone(depth=2, global_att_blocks=(1,))
    return {b.window_size: torch.view_as_real(b.attn.freqs_cis.to(torch.complex64)).float().contiguous() for b in vit.blocks}


def _table(win, H, cuda):
    if H == 72:
        return _teacher_tables()[win].to(cuda)
    from efficientsam3_b200.model.vitdet import compute_axial_cis
    return torch.view_as_real(compute_axial_cis(64, win or H, win or H)).float().contiguous().to(cuda)


ROPE = [(0, 72, 72, 16, 1), (24, 72, 72, 4, 2), (8, 16, 16, 3, 2), (0, 8, 8, 2, 3)]


@pytest.mark.parametrize("win,H,W,heads,B", ROPE)
def test_rope_f32(cuda, win, H, W, heads, B):
    """In place on rows 24 columns wider than 3C: the q | k columns within their bound, the v block and the padding columns bit for
    bit, the cells past the rows untouched; the last image alone; ops.rope_f32 bit-identical."""
    lib = _lib(cuda)
    C = 64 * heads
    M, ld = B * H * W, 3 * C + 24
    table = _table(win, H, cuda)
    x = torch.randn(M, ld, device=cuda, generator=_gen(cuda, "rope", win, H, heads, B))
    buf, ins = _flat_out(M * ld, torch.float32, cuda)
    buf[:M * ld] = x.reshape(-1)
    run = lambda b: lib.call("es3_rope_f32", b.data_ptr(), ld, M, table.data_ptr(), 2 * C, H, W, win, _st())
    got = _twice(run, buf)
    rows = got[:M * ld].view(M, ld)
    ref, bound = R.rope(x.double(), table.double(), 2 * C, H, W, win)
    what = f"rope_f32 win{win} {H}x{W} heads{heads} B{B}"
    _check("6 rope_f32", rows[:, :2 * C], ref, bound, what)
    _bits_equal(rows[:, 2 * C:], x[:, 2 * C:], what + ": v block and padding columns")
    _assert_untouched(got, ins, what)
    if B > 1:
        sl = _last_image(B, H * W)
        one = x[sl].clone()
        lib.call("es3_rope_f32", one.data_ptr(), ld, H * W, table.data_ptr(), 2 * C, H, W, win, _st())
        _bits_equal(one, rows[sl], what + ": last image alone")
    wx = x.clone()
    _bits_equal(_ops().rope_f32(wx[:, :3 * C], table, 2 * C, H, W, win), rows[:, :3 * C], "ops.rope_f32 vs direct")


# ----------------------------------------------------------------------------------------------------------- (7) strict attention
AF32 = [  # B, H, W, heads, hd, win, layout, bias, pad
    (2, 16, 16, 4, 64, 8, "blocks", False, False),
    (1, 72, 72, 2, 64, 24, "blocks", False, False),     # the teacher's windowed blocks
    (1, 72, 72, 1, 64, 0, "blocks", False, False),      # the teacher's global blocks: L 5184
    (2, 24, 24, 2, 64, 0, "blocks", False, False),
    (2, 14, 14, 3, 32, 7, "per_head", True, False),     # TinyViT: exact windows with the relative bias
    (2, 10, 10, 2, 32, 7, "per_head", True, True),      # overhanging windows take pad_row
    (1, 5, 5, 5, 32, 7, "per_head", True, True),        # one window larger than the grid
    (1, 9, 6, 2, 32, 0, "per_head", False, False),
]


def _offs(layout, C, hd):
    return (0, C, 2 * C, hd) if layout == "blocks" else (0, hd, 2 * hd, 3 * hd)


@pytest.mark.parametrize("B,H,W,heads,hd,win,layout,bias,pad", AF32)
def test_attention_f32(cuda, B, H, W, heads, hd, win, layout, bias, pad):
    lib = _lib(cuda)
    g = _gen(cuda, "af32", B, H, W, heads, hd, win, layout)
    C, n = heads * hd, B * H * W
    L = win * win if win else H * W
    scale = hd ** -0.5
    qkv = torch.randn(n, 3 * C, device=cuda, generator=g)
    bs = torch.randn(heads, L, L, device=cuda, generator=g) if bias else None
    pr = torch.randn(3 * C, device=cuda, generator=g) if pad else None

    def run(o, x=qkv, B_=B):
        lib.call("es3_attention_f32", x.data_ptr(), o.data_ptr(), _p(bs), _p(pr), B_, H, W, 3 * C, heads, hd, *_offs(layout, C, hd), win,
                 scale, _st())
    buf, ins = _flat_out(n * C, torch.float32, cuda)
    got = _twice(run, buf)
    o = got[:n * C].view(n, C)
    d = lambda t: None if t is None else t.double()
    ref, bound = R.attention_f32(qkv.double(), B, H, W, heads, hd, win, scale, layout, d(bs), d(pr))
    what = f"attention_f32 B{B} {H}x{W} heads{heads} hd{hd} win{win} {layout} bias={bias} pad={pad}"
    _check(f"7 attention_f32 hd{hd}", o, ref, bound, what)
    _assert_untouched(got, ins, what)
    if B > 1:
        sl = _last_image(B, H * W)
        one = torch.full((H * W, C), float("nan"), device=cuda)
        run(one, qkv[sl].contiguous(), 1)
        _bits_equal(one, o[sl], what + ": last image alone")
    _bits_equal(_ops().attention_f32(qkv, B, H, W, heads, hd, win, scale, layout=layout, bias=bs, pad_row=pr), o,
                "ops.attention_f32 vs direct")


def test_attention_f32_declined_arguments_write_nothing(cuda):
    """qkv or pad_row off 16 bytes, head_dim 48, windows overhanging the grid without pad_row."""
    lib = _lib(cuda)
    z = torch.zeros(2 * 10 * 10 * 288 + 64, device=cuda)             # every row below addresses at most B H W ld floats
    out, _ = _flat_out(10 * 10 * 64, torch.float32, cuda)
    q0, o0 = z.data_ptr(), out.data_ptr()
    base = (2, 10, 10, 192, 2, 32, 0, 32, 64, 96, 7, 0.2)
    for args, what in (((q0 + 4, o0, 0, q0) + base, "qkv + 4 bytes"), ((q0, o0, 0, q0 + 4) + base, "pad_row + 4 bytes"),
                       ((q0, o0, 0, q0, 2, 10, 10, 288, 2, 48, 0, 48, 96, 144, 7, 0.2), "head_dim 48"),
                       ((q0, o0, 0, 0) + base, "overhanging windows without pad_row")):
        _declined(lib, "es3_attention_f32", args + (_st(),), [out], f"attention_f32 {what}")


# ----------------------------------------------------------------------------------------------------------- (8) strict LayerNorm
LNR = _pairwise(dict(C=[64, 96, 100, 160, 576, 1000, 1024], M=[1, 77, 1000], shift=[0.0, 30.0]), seed=22)


@pytest.mark.parametrize("C,M,shift", LNR)
def test_ln_rows_f32(cuda, C, M, shift):
    """Widths from 64 to 1024, not all multiples of 32; mean-shifted rows; the last row alone; ops.ln_rows_f32 bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "lnr", C, M, shift)
    x = torch.randn(M, C, device=cuda, generator=g) * 3 + shift
    w, b = torch.rand(C, device=cuda, generator=g) + 0.5, torch.randn(C, device=cuda, generator=g)
    run = lambda o, x_=x, m=M: lib.call("es3_ln_rows_f32", x_.data_ptr(), w.data_ptr(), b.data_ptr(), 1e-5, o.data_ptr(), m, C, _st())
    buf, ins = _flat_out(M * C, torch.float32, cuda)
    got = _twice(run, buf)
    y = got[:M * C].view(M, C)
    ref, bound = R.ln_rows(x.double(), w.double(), b.double(), 1e-5)
    what = f"ln_rows_f32 C{C} M{M} shift {shift}"
    _check("8 ln_rows_f32", y, ref, bound, what)
    _assert_untouched(got, ins, what)
    one = torch.full((1, C), float("nan"), device=cuda)
    run(one, x[-1:].contiguous(), 1)
    _bits_equal(one, y[-1:], what + ": last row alone")
    _bits_equal(_ops().ln_rows_f32(x, w, b, 1e-5), y, "ops.ln_rows_f32 vs direct")


# ----------------------------------------------------------------------------------------------------------- (9) strict im2col
I2C = [(1, 1008, 1008, 3, 14, 14, 0, True), (2, 112, 112, 3, 14, 14, 0, True), (2, 9, 11, 16, 3, 1, 1, False),
       (2, 15, 13, 32, 3, 2, 1, False), (1, 20, 18, 24, 3, 2, 1, False),
       (2, 33, 31, 3, 3, 2, 1, True)]                   # the strict student's stem: 3 x 3 stride 2 on the NCHW image


@pytest.mark.parametrize("B,H,W,C,ks,stride,pad,nchw", I2C)
def test_im2col_f32(cuda, B, H, W, C, ks, stride, pad, nchw):
    """The NCHW patch form (ks 14, stride 14), the NCHW 3 x 3 stride-2 stem and the NHWC 3 x 3 forms at stride 1 and 2, bit-exact
    against F.unfold."""
    lib = _lib(cuda)
    shape = (B, C, H, W) if nchw else (B, H, W, C)
    x = torch.randn(*shape, device=cuda, generator=_gen(cuda, "i2c", B, H, W, C, ks, stride))
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    n = B * Ho * Wo * ks * ks * C
    run = lambda o, x_=x, b=B: lib.call("es3_im2col_f32", x_.data_ptr(), o.data_ptr(), b, H, W, C, ks, stride, pad, int(nchw), _st())
    buf, ins = _flat_out(n, torch.float32, cuda)
    got = _twice(run, buf)
    cols = got[:n].view(B * Ho * Wo, ks * ks * C)
    what = f"im2col_f32 B{B} {H}x{W} C{C} ks{ks} s{stride} nchw={nchw}"
    _bits_equal(cols, R.im2col_f32(x, ks, stride, pad, nchw), what)
    _assert_untouched(got, ins, what)
    if B > 1:
        one = torch.full((Ho * Wo, ks * ks * C), float("nan"), device=cuda)
        run(one, x[-1:].contiguous(), 1)
        _bits_equal(one, cols[_last_image(B, Ho * Wo)], what + ": last image alone")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs; es3_attention_bf16 where _attn_case calls it too."""
    keys = set()
    for name, rows in (("es3_attention_tc_bf16", TC), ("es3_attention_mma_bf16", MMA)):
        for c in rows:
            key, dispatched = attn_key(name, c[1], c[2], c[4]), attn_key("es3_attention_bf16", c[1], c[2], c[4])
            keys |= {key, dispatched} if dispatched[1:] == key[1:] else {key}
    keys |= {("es3_im2col_patch",) for _ in PATCH} | {("es3_tokens_f32_to_nchw",) for _ in T2N} | {("es3_ln_rows_f32",) for _ in LNR}
    from efficientsam3_b200.ops import ACT
    keys |= {("es3_sgemm_f32", ACT[c[3]], c[4], "scale" in c[5], "bias" in c[5], "res" in c[5]) for c in SG}
    keys |= {("es3_rope_f32", c[0] > 0) for c in ROPE}
    keys |= {("es3_attention_f32", c[4], c[7], c[8], c[5] > 0) for c in AF32}
    keys |= {("es3_im2col_f32", c[7], c[4], c[5]) for c in I2C}
    return keys
