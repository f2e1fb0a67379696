"""The text encoders' kernels (attention.cu, attention_tc.cu and text_bwd.cu's attention backward at text shapes, text.cu, the
fp32 LayerNorm of vit_ops.cu, text_bwd.cu's LayerNorm backward, embedding gradients and KD loss, the casts), element by element
against the fp64 statements of tests/ref_text.py, each output element within its own bound.

Outputs and workspaces are NaN-prefilled and called through _lib.call: every cell inside the output region must be written and lie
within its bound, every cell past it (a flat TAIL) keeps its sentinel bits.  Accumulating outputs (dgamma, dbeta, the embedding
and positional gradients, consistency's dp and loss) are prefilled with random values and checked as +=.  Every fixed-order
reduction runs twice and must be bit-identical; a sequence run alone must be bit-identical to the same sequence inside a batch; a
shape an entry point declines writes nothing; the ops wrappers are bit-identical to the direct calls.  covered_keys() names the
route keys (tests/routes.py) the tables run, for the route closure of tests/test_route_closure_gpu.py.

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power
limit): bf16 outputs -- attention 0.995 (mma.sync) and 0.934 (wgmma), attention backward 0.994, LayerNorm 0.995, RepMixer u 0.994,
RepMixer backward dy 0.996, where the output's own rounding half-step dominates the bound; fp32 outputs -- LayerNorm 0.134, LayerNorm backward 0.155 (dx),
0.065 (dgamma), 0.125 (dbeta), RepMixer x1 0.169, embedding gradient 0.186, positional gradient 0.099, positional resize 0.991
(its bound is its own two roundings), RepMixer backward 0.681 (tm dx), 0.197 (ffn e), <= 0.085 (the accumulated gradients), KD
partials 0.038, out3 0.017, dp 0.143, consistency 0.2 at most.  The whole file (226 tests, the route-closure training steps
included, since moved to tests/test_route_closure_gpu.py) took 29 s there.
"""
import zlib

import pytest
import torch

import ref_text as R
from bounds import (TAIL, _assert_untouched, _bf, _bits_equal, _check, _declined, _flat_out, _gen, _lib, _p, _pairwise,
                    _prefilled, _qkv, _st, _twice, report_worst)
from routes import attn_key, causal_attn_key

pytestmark = pytest.mark.gpu
_report_worst = report_worst("text kernels")


# ----------------------------------------------------------------------------------------------------------- (1) attention
ATTN = _pairwise(dict(L=[1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 77, 127, 128], heads=[1, 8, 12, 16], B=[1, 3, 64],
                      kind=["normal", "peaked", "flat", "tied"], causal=[True, False]), seed=11)
ATTN_SCALE = 64 ** -0.5


def _attn_fwd(lib, qkv, o, B, L, C, heads, causal):
    if causal:
        lib.call("es3_attention_causal_bf16", qkv.data_ptr(), o.data_ptr(), B, L, C, heads, ATTN_SCALE, _st())
    else:
        lib.call("es3_attention_bf16", qkv.data_ptr(), o.data_ptr(), B, 1, L, C, heads, 0, ATTN_SCALE, _st())


def _attn_bwd(lib, qkv, o, dout, dq, B, L, C, heads, causal):
    lib.call("es3_text_attn_bwd", qkv.data_ptr(), o.data_ptr(), dout.data_ptr(), dq.data_ptr(), B, L, C, heads, int(causal),
             ATTN_SCALE, _st())


@pytest.mark.parametrize("L,heads,B,kind,causal", ATTN)
def test_attention_fwd_bwd(cuda, L, heads, B, kind, causal):
    """Causal mma.sync (MT = 1 below L = 128, MT = 2 at 128), non-causal mma.sync (L < 128) and wgmma (L = 128) forwards, then
    es3_text_attn_bwd on the kernel's own O; the last sequence of a batch is bit-identical run alone, in both directions; the
    ops wrappers are bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "attn", L, heads, B, kind, causal)
    C = 64 * heads
    qkv = _qkv(cuda, B, L, heads, kind, g)
    dout = _bf(torch.randn(B * L, C, device=cuda, generator=g))
    buf, inside = _flat_out(B * L * C, torch.bfloat16, cuda)
    got = _twice(lambda o: _attn_fwd(lib, qkv, o, B, L, C, heads, causal), buf)
    o = got[:B * L * C].view(B * L, C)
    kernel = "mma" if causal else attn_key("es3_attention_bf16", 1, L, 0)[1]
    ref, bound = R.attention(qkv.double(), B, L, heads, ATTN_SCALE, causal, kernel)
    what = f"attention {kernel} causal={causal} L{L} heads{heads} B{B} {kind}"
    _check(f"1 attention {kernel} causal={causal}", o, ref, bound, what)
    _assert_untouched(got, inside, what)
    dbuf, dins = _flat_out(B * L * 3 * C, torch.bfloat16, cuda)
    dgot = _twice(lambda d: _attn_bwd(lib, qkv, o, dout, d, B, L, C, heads, causal), dbuf)
    dq = dgot[:B * L * 3 * C].view(B * L, 3 * C)
    ref, bound = R.attention_bwd(qkv.double(), o.double(), dout.double(), B, L, heads, ATTN_SCALE, causal)
    _check(f"1 text_attn_bwd causal={causal}", dq, ref, bound, "bwd " + what)
    _assert_untouched(dgot, dins, "bwd " + what)
    from efficientsam3_b200 import ops
    wo = ops.attention_causal(qkv, B, L, C, heads, ATTN_SCALE) if causal else ops.attention(qkv, B, 1, L, C, heads, 0, ATTN_SCALE)
    _bits_equal(wo, o, "ops attention vs the direct call")
    _bits_equal(ops.text_attn_bwd(qkv, o, dout, B, L, C, heads, ATTN_SCALE, causal), dq, "ops.text_attn_bwd vs the direct call")
    if B > 1:
        sl = slice((B - 1) * L, B * L)
        one = torch.full((L, C), float("nan"), dtype=torch.bfloat16, device=cuda)
        _attn_fwd(lib, qkv[sl].contiguous(), one, 1, L, C, heads, causal)
        _bits_equal(one, o[sl], "attention: last sequence vs alone")
        done = torch.full((L, 3 * C), float("nan"), dtype=torch.bfloat16, device=cuda)
        _attn_bwd(lib, qkv[sl].contiguous(), o[sl].contiguous(), dout[sl].contiguous(), done, 1, L, C, heads, causal)
        _bits_equal(done, dq[sl], "text_attn_bwd: last sequence vs alone")


def test_attention_declined_shapes_write_nothing(cuda):
    """L = 129 and head_dim != 64 for the backward; head_dim != 64 for both forwards."""
    lib = _lib(cuda)
    z = torch.zeros(129 * 3 * 512, dtype=torch.bfloat16, device=cuda)
    out, _ = _flat_out(129 * 3 * 512, torch.bfloat16, cuda)
    _declined(lib, "es3_text_attn_bwd", (z.data_ptr(), z.data_ptr(), z.data_ptr(), out.data_ptr(), 1, 129, 512, 8, 1, 0.125, _st()),
              [out], "text_attn_bwd L129")
    _declined(lib, "es3_text_attn_bwd", (z.data_ptr(), z.data_ptr(), z.data_ptr(), out.data_ptr(), 1, 16, 512, 16, 0, 0.125, _st()),
              [out], "text_attn_bwd head_dim 32")
    _declined(lib, "es3_attention_causal_bf16", (z.data_ptr(), out.data_ptr(), 1, 16, 512, 16, 0.125, _st()), [out],
              "attention_causal head_dim 32")
    _declined(lib, "es3_attention_bf16", (z.data_ptr(), out.data_ptr(), 1, 1, 16, 512, 16, 0, 0.125, _st()), [out],
              "attention head_dim 32")
    from efficientsam3_b200 import ops
    with pytest.raises(ValueError, match="1..128"):
        ops.text_attn_bwd(*(torch.zeros(1, 1, device=cuda, dtype=torch.bfloat16),) * 3, 1, 129, 512, 8, 0.125, False)


# ----------------------------------------------------------------------------------------------------------- (2) LayerNorm
LN_C = [128, 256, 384, 512, 640, 768, 896, 1024, 1280, 1536, 2048]          # every es3_layernorm_f32 instantiation
LNF = [(C, M, pos, shift, out, (3, 5, 4)) for (C, M, pos, shift, out) in
       _pairwise(dict(C=LN_C, M=[1, 7, 77 * 3, 1000], pos=[False, True], shift=[0.0, 30.0], out=["f32", "bf16", "both"]), seed=12)]
LNF += [(1024, 2 * 5184, True, 0.0, "f32", (24, 72, 72))]                     # the ViT teacher's ln_pre: 24 x 24 table over 72 x 72


def _lnf_id(c):
    return "-".join(map(str, c[:5])) + ("" if c[5] == (3, 5, 4) else "-ps{}-{}x{}".format(*c[5]))


@pytest.mark.parametrize("C,M,pos,shift,out,geom", LNF, ids=[_lnf_id(c) for c in LNF])
def test_layernorm_f32(cuda, C, M, pos, shift, out, geom):
    """All eleven lane-vector counts; the tiled positional add (ps = 3 over a 5 x 4 grid, and the teacher's ln_pre: ps = 24 over
    72 x 72 tokens of two images); mean-shifted rows; fp32 and / or bf16 stores (bf16 = bf16 of the same fp32 value bit for bit);
    ops.layernorm is bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "lnf", C, M, pos, shift, out) if geom == (3, 5, 4) else _gen(cuda, "lnf", C, M, pos, shift, out, geom)
    x = torch.randn(M, C, device=cuda, generator=g) + shift
    gm, bt = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    ps, H, W = geom
    pt = torch.randn(ps * ps, C, device=cuda, generator=g) if pos else None
    yf, fins = _flat_out(M * C, torch.float32, cuda)
    yb, bins = _flat_out(M * C, torch.bfloat16, cuda)
    want_f, want_b = out in ("f32", "both"), out in ("bf16", "both")
    lib.call("es3_layernorm_f32", x.data_ptr(), _p(pt), ps if pos else 0, H if pos else 0, W if pos else 0, gm.data_ptr(),
             bt.data_ptr(), 1e-5, yb.data_ptr() if want_b else 0, yf.data_ptr() if want_f else 0, M, C, _st())
    what = f"layernorm_f32 C{C} M{M} pos={pos} shift {shift} {out}"
    args = (x.double(), gm.double(), bt.double(), 1e-5, None if pt is None else pt.double(), ps, H, W)
    if want_f:
        ref, bound = R.layernorm_f32(*args)
        _check("2 layernorm_f32 fp32", yf[:M * C].view(M, C), ref, bound, what)
        _assert_untouched(yf, fins, what)
    else:
        _assert_untouched(yf, torch.zeros_like(fins), what + " (fp32 not requested)")
    if want_b:
        ref, bound = R.layernorm_f32(*args, bf16=True)
        _check("2 layernorm_f32 bf16", yb[:M * C].view(M, C), ref, bound, what)
        _assert_untouched(yb, bins, what)
        if want_f:
            _bits_equal(yb[:M * C], yf[:M * C].to(torch.bfloat16), what + ": bf16 store vs bf16(fp32 store)")
    else:
        _assert_untouched(yb, torch.zeros_like(bins), what + " (bf16 not requested)")
    from efficientsam3_b200 import ops
    wb, wf = ops.layernorm(x, gm, bt, 1e-5, pos=pt, pos_size=ps if pos else 0, H=H if pos else 0, W=W if pos else 0,
                           out_bf16=want_b, out_f32=want_f)
    if want_f:
        _bits_equal(wf, yf[:M * C].view(M, C), "ops.layernorm fp32 vs direct")
    if want_b:
        _bits_equal(wb, yb[:M * C].view(M, C), "ops.layernorm bf16 vs direct")


def test_layernorm_f32_declined_width_writes_nothing(cuda):
    lib = _lib(cuda)
    for C in (1152, 1000):
        x = torch.zeros(4 * C, device=cuda)
        yf, _ = _flat_out(4 * C, torch.float32, cuda)
        _declined(lib, "es3_layernorm_f32", (x.data_ptr(), 0, 0, 0, 0, x.data_ptr(), x.data_ptr(), 1e-5, 0, yf.data_ptr(), 4, C, _st()),
                  [yf], f"layernorm_f32 C{C}")


LNB = _pairwise(dict(C=[4, 132, 260, 516, 768], M=[1, 63, 64, 65, 5000, 37889, 40000], dres=[False, True], dxb=[False, True]),
                seed=13)


@pytest.mark.parametrize("C,M,dres,dxb", LNB)
def test_layernorm_bwd_f32(cuda, C, M, dres, dxb):
    """Lanes partially used (C = 4, 132, 260, 516) and full (768); M on both sides of the 64-row blocks and of the 592-block cap
    (M > 37 888: several rows per warp per block); dres and the bf16 copy each present and absent (the copy is bf16(dx32) bit for
    bit); dgamma / dbeta accumulated into random values; the NaN-filled workspace; twice bit-identical; the last row alone is
    bit-identical; ops.layernorm_bwd_f32 is bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "lnb", C, M, dres, dxb)
    x = torch.randn(M, C, device=cuda, generator=g) * 3 + 0.5
    dy = torch.randn(M, C, device=cuda, generator=g)
    gm = torch.randn(C, device=cuda, generator=g) + 1
    r = torch.randn(M, C, device=cuda, generator=g) if dres else None
    dg, dgi = _prefilled(C, cuda, g)
    db, dbi = _prefilled(C, cuda, g)
    ws_n = lib.size("es3_layernorm_bwd_f32_ws_floats", M, C)
    outs = []

    def run(dx):
        b = torch.full((M * C + TAIL,), float("nan"), dtype=torch.bfloat16, device=cuda) if dxb else None
        dga, dba = dg.clone(), db.clone()
        ws = torch.full((ws_n,), float("nan"), device=cuda)
        lib.call("es3_layernorm_bwd_f32", x.data_ptr(), dy.data_ptr(), gm.data_ptr(), _p(r), 1e-5, dx.data_ptr(), _p(b), M, C,
                 ws.data_ptr(), dga.data_ptr(), dba.data_ptr(), _st())
        outs.append((b, dga, dba))
    buf, ins = _flat_out(M * C, torch.float32, cuda)
    got = _twice(run, buf)
    for i in range(3 if dxb else 1, 3):
        _bits_equal(outs[0][i], outs[1][i], "layernorm_bwd_f32 gradients twice")
    if dxb:
        _bits_equal(outs[0][0], outs[1][0], "layernorm_bwd_f32 dxb twice")
    ref = R.layernorm_bwd_f32(x.double(), dy.double(), gm.double(), 1e-5, dg[:C].double(), db[:C].double(),
                              None if r is None else r.double())
    what = f"layernorm_bwd_f32 C{C} M{M} dres={dres} dxb={dxb}"
    _check("2 layernorm_bwd_f32 dx", got[:M * C].view(M, C), *ref["dx"], what)
    _assert_untouched(got, ins, what)
    _check("2 layernorm_bwd_f32 dgamma", outs[0][1][:C], *ref["dgamma"], what + " dgamma")
    _check("2 layernorm_bwd_f32 dbeta", outs[0][2][:C], *ref["dbeta"], what + " dbeta")
    _assert_untouched(outs[0][1], dgi, what + " dgamma")
    _assert_untouched(outs[0][2], dbi, what + " dbeta")
    if dxb:
        _bits_equal(outs[0][0][:M * C], got[:M * C].to(torch.bfloat16), what + ": dxb vs bf16(dx)")
        _assert_untouched(outs[0][0], ins, what + " dxb")
    one = torch.full((C,), float("nan"), device=cuda)
    ws = torch.full((lib.size("es3_layernorm_bwd_f32_ws_floats", 1, C),), float("nan"), device=cuda)
    lib.call("es3_layernorm_bwd_f32", x[-1:].data_ptr(), dy[-1:].data_ptr(), gm.data_ptr(), _p(None if r is None else r[-1:]), 1e-5,
             one.data_ptr(), 0, 1, C, ws.data_ptr(), 0, 0, _st())
    _bits_equal(one, got[(M - 1) * C:M * C], what + ": last row alone")
    from efficientsam3_b200 import ops
    dga, dba = dg[:C].clone(), db[:C].clone()
    wdx, wdxb = ops.layernorm_bwd_f32(x, dy, gm, 1e-5, dga, dba, dres=r, want_bf16=dxb)
    _bits_equal(wdx, got[:M * C].view(M, C), "ops.layernorm_bwd_f32 vs direct")
    _bits_equal(dga, outs[0][1][:C], "ops.layernorm_bwd_f32 dgamma vs direct")


def test_layernorm_bwd_f32_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    for C in (772, 130):
        x = torch.zeros(8 * C, device=cuda)
        dx, _ = _flat_out(8 * C, torch.float32, cuda)
        dg, _ = _flat_out(C, torch.float32, cuda)
        ws = torch.full((8 * 2 * C,), float("nan"), device=cuda)
        _declined(lib, "es3_layernorm_bwd_f32", (x.data_ptr(), x.data_ptr(), x.data_ptr(), 0, 1e-5, dx.data_ptr(), 0, 8, C, ws.data_ptr(),
                                                 dg.data_ptr(), dg.data_ptr(), _st()), [dx, dg, ws], f"layernorm_bwd_f32 C{C}")


# ----------------------------------------------------------------------------------------------------------- (3) RepMixer
REPMIXER = [(4, 1, 512), (4, 5, 512), (4, 11, 512), (4, 32, 512), (4, 77, 512), (1, 1, 32), (3, 128, 64), (64, 77, 512)]


@pytest.mark.parametrize("B,L,C", REPMIXER)
def test_repmixer(cuda, B, L, C):
    """The S0 shapes (C 512, L 1 ... 77), B L = 1, the 128-token maximum; x1 fp32 and u bf16; twice bit-identical; the last sequence
    alone; ops.repmixer bit-identical."""
    lib = _lib(cuda)
    g = _gen(cuda, "rm", B, L, C)
    x = torch.randn(B * L, C, device=cuda, generator=g)
    wm, wf = torch.randn(11, C, device=cuda, generator=g) * 0.3, torch.randn(11, C, device=cuda, generator=g) * 0.3
    bm, bf = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    us = []

    def run(x1):
        u = torch.full((B * L * C + TAIL,), float("nan"), dtype=torch.bfloat16, device=cuda)
        lib.call("es3_repmixer_bf16", x.data_ptr(), x1.data_ptr(), u.data_ptr(), wm.data_ptr(), bm.data_ptr(), wf.data_ptr(),
                 bf.data_ptr(), B, L, C, _st())
        us.append(u)
    buf, ins = _flat_out(B * L * C, torch.float32, cuda)
    x1 = _twice(run, buf)
    _bits_equal(us[0], us[1], "repmixer u twice")
    (r1, b1), (ru, bu) = R.repmixer(x.double(), wm.double(), bm.double(), wf.double(), bf.double(), B, L)
    what = f"repmixer B{B} L{L} C{C}"
    _check("3 repmixer x1", x1[:B * L * C].view(B * L, C), r1, b1, what)
    _check("3 repmixer u", us[0][:B * L * C].view(B * L, C), ru, bu, what)
    _assert_untouched(x1, ins, what)
    _assert_untouched(us[0], ins, what + " u")
    if B > 1:
        one1 = torch.full((L, C), float("nan"), device=cuda)
        oneu = torch.full((L, C), float("nan"), dtype=torch.bfloat16, device=cuda)
        lib.call("es3_repmixer_bf16", x[-L:].data_ptr(), one1.data_ptr(), oneu.data_ptr(), wm.data_ptr(), bm.data_ptr(), wf.data_ptr(),
                 bf.data_ptr(), 1, L, C, _st())
        _bits_equal(oneu, us[0][(B - 1) * L * C:B * L * C].view(L, C), "repmixer last sequence alone")
    from efficientsam3_b200 import ops
    w1, wu = ops.repmixer(x, B, L, wm, bm, wf, bf)
    _bits_equal(w1, x1[:B * L * C].view(B * L, C), "ops.repmixer x1 vs direct")
    _bits_equal(wu, us[0][:B * L * C].view(B * L, C), "ops.repmixer u vs direct")


def test_repmixer_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    for L, C in ((129, 64), (8, 48)):
        x = torch.zeros(L * C, device=cuda)
        w = torch.zeros(11 * C, device=cuda)
        x1, _ = _flat_out(L * C, torch.float32, cuda)
        u, _ = _flat_out(L * C, torch.bfloat16, cuda)
        _declined(lib, "es3_repmixer_bf16", (x.data_ptr(), x1.data_ptr(), u.data_ptr(), w.data_ptr(), w.data_ptr(), w.data_ptr(),
                                             w.data_ptr(), 1, L, C, _st()), [x1, u], f"repmixer L{L} C{C}")
    from efficientsam3_b200 import ops
    z = torch.zeros(11, 64, device=cuda)
    with pytest.raises(ValueError, match="1..128"):
        ops.repmixer(torch.zeros(129, 64, device=cuda), 1, 129, z, z[0], z, z[0])


RMB = _pairwise(dict(B=[1, 3, 64], L=[1, 4, 11, 16, 32, 77, 128], C=[32, 512]), seed=15)


def _rmb_ws(lib, B, C, cuda):
    return torch.full((lib.size("es3_repmixer_bwd_ws_floats", B, C),), float("nan"), device=cuda)


@pytest.mark.parametrize("B,L,C", RMB)
def test_repmixer_bwd(cuda, B, L, C):
    """es3_repmixer_ls_bwd, _ffn_bwd and _tm_bwd (frozen BN) on taps and packed (s, b, rm, invstd) rows: every output and workspace
    NaN-prefilled, every gradient prefilled with random values and checked as +=, the bf16 dy and dxb bit-identical to bf16 of the
    fp32 values, each call twice bit-identical, the last sequence alone bit-identical, the ops wrappers bit-identical."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "rmb", B, L, C)
    n = B * L * C
    rows = lambda: torch.randn(B * L, C, device=cuda, generator=g)
    x, x1, gg, du, y, e = (rows() for _ in range(6))
    ls, wf, wmc = torch.randn(C, device=cuda, generator=g), torch.randn(11, C, device=cuda, generator=g) * 0.3, \
        torch.randn(11, C, device=cuda, generator=g) * 0.3

    def pack():
        inv = torch.rand(C, device=cuda, generator=g) + 0.5
        s_ = torch.randn(C, device=cuda, generator=g)
        return [s_, torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g), inv]
    bnf = torch.stack(pack())
    bnp = torch.stack(pack() + pack() + pack() + [torch.randn(C, device=cuda, generator=g)])
    what = f"repmixer_bwd B{B} L{L} C{C}"
    d64 = lambda t: t.double()

    # layer scale
    acc = {k: _prefilled(C, cuda, g) for k in ("dls", "dbias")}
    got = {}

    def run_ls(dy):
        a = {k: v[0].clone() for k, v in acc.items()}
        lib.call("es3_repmixer_ls_bwd", gg.data_ptr(), y.data_ptr(), ls.data_ptr(), dy.data_ptr(), _rmb_ws(lib, B, C, cuda).data_ptr(),
                 a["dls"].data_ptr(), a["dbias"].data_ptr(), B, L, C, _st())
        got.setdefault("ls", []).append(a)
    dyb, dyi = _flat_out(n, torch.bfloat16, cuda)
    dy = _twice(run_ls, dyb)
    ref = R.repmixer_ls_bwd(d64(gg), d64(y), d64(ls), B, L, d64(acc["dls"][0][:C]), d64(acc["dbias"][0][:C]))
    _check("3 repmixer_ls_bwd dy", dy[:n].view(B * L, C), *ref["dy"], what + " dy")
    _bits_equal(dy[:n], (ls * gg).reshape(-1).to(torch.bfloat16), what + ": dy vs bf16(ls g)")
    _assert_untouched(dy, dyi, what + " dy")
    for k in ("dls", "dbias"):
        _bits_equal(got["ls"][0][k], got["ls"][1][k], what + f" {k} twice")
        _check(f"3 repmixer_ls_bwd {k}", got["ls"][0][k][:C], *ref[k], what + " " + k)
        _assert_untouched(got["ls"][0][k], acc[k][1], what + " " + k)

    # ConvFFN.conv + BN_f
    acc = {"dwf": _prefilled(11 * C, cuda, g), "dgamma": _prefilled(C, cuda, g), "dbeta": _prefilled(C, cuda, g)}

    def run_ffn(eo):
        a = {k: v[0].clone() for k, v in acc.items()}
        lib.call("es3_repmixer_ffn_bwd", x1.data_ptr(), du.data_ptr(), gg.data_ptr(), wf.data_ptr(), bnf.data_ptr(), eo.data_ptr(),
                 _rmb_ws(lib, B, C, cuda).data_ptr(), a["dwf"].data_ptr(), a["dgamma"].data_ptr(), a["dbeta"].data_ptr(), B, L, C, _st())
        got.setdefault("ffn", []).append(a)
    eb, ei = _flat_out(n, torch.float32, cuda)
    eo = _twice(run_ffn, eb)
    ref = R.repmixer_ffn_bwd(d64(x1), d64(du), d64(gg), d64(wf), d64(bnf), B, L, d64(acc["dwf"][0][:11 * C]).view(C, 11),
                             d64(acc["dgamma"][0][:C]), d64(acc["dbeta"][0][:C]))
    _check("3 repmixer_ffn_bwd e", eo[:n].view(B * L, C), *ref["e"], what + " e")
    _assert_untouched(eo, ei, what + " e")
    for k, m in (("dwf", 11 * C), ("dgamma", C), ("dbeta", C)):
        _bits_equal(got["ffn"][0][k], got["ffn"][1][k], what + f" {k} twice")
        v = got["ffn"][0][k][:m]
        _check(f"3 repmixer_ffn_bwd {k}", v.view(C, 11) if k == "dwf" else v, *ref[k], what + " " + k)
        _assert_untouched(got["ffn"][0][k], acc[k][1], what + " " + k)

    # token mixer
    names = ["dwmc", "dls", "dg_ms", "db_ms", "dg_mc", "db_mc", "dg_ns", "db_ns"]
    acc = {k: _prefilled(11 * C if k == "dwmc" else C, cuda, g) for k in names}

    def run_tm(dx):
        a = {k: v[0].clone() for k, v in acc.items()}
        a["dxb"] = torch.full((n + TAIL,), float("nan"), dtype=torch.bfloat16, device=cuda)
        lib.call("es3_repmixer_tm_bwd", x.data_ptr(), e.data_ptr(), wmc.data_ptr(), bnp.data_ptr(), dx.data_ptr(), a["dxb"].data_ptr(),
                 _rmb_ws(lib, B, C, cuda).data_ptr(), *[a[k].data_ptr() for k in names], B, L, C, _st())
        got.setdefault("tm", []).append(a)
    dxb_, dxi = _flat_out(n, torch.float32, cuda)
    dx = _twice(run_tm, dxb_)
    ref = R.repmixer_tm_bwd(d64(x), d64(e), d64(wmc), d64(bnp), B, L, d64(acc["dwmc"][0][:11 * C]).view(C, 11),
                            d64(acc["dls"][0][:C]), [d64(acc[k][0][:C]) for k in names[2:]])
    _check("3 repmixer_tm_bwd dx", dx[:n].view(B * L, C), *ref["dx"], what + " dx")
    _assert_untouched(dx, dxi, what + " dx")
    _bits_equal(got["tm"][0]["dxb"][:n], dx[:n].to(torch.bfloat16), what + ": dxb vs bf16(dx)")
    _assert_untouched(got["tm"][0]["dxb"], dxi, what + " dxb")
    for k in names:
        _bits_equal(got["tm"][0][k], got["tm"][1][k], what + f" {k} twice")
        m = 11 * C if k == "dwmc" else C
        v = got["tm"][0][k][:m]
        _check(f"3 repmixer_tm_bwd {k}", v.view(C, 11) if k == "dwmc" else v, *ref[k], what + " " + k)
        _assert_untouched(got["tm"][0][k], acc[k][1], what + " " + k)

    if B > 1:                                  # the last sequence alone: its per-row outputs bit-identical
        sl = slice((B - 1) * L, B * L)
        one = torch.full((L, C), float("nan"), device=cuda)
        lib.call("es3_repmixer_tm_bwd", x[sl].contiguous().data_ptr(), e[sl].contiguous().data_ptr(), wmc.data_ptr(), bnp.data_ptr(),
                 one.data_ptr(), 0, _rmb_ws(lib, 1, C, cuda).data_ptr(), *([0] * 8), 1, L, C, _st())
        _bits_equal(one, dx[:n].view(B * L, C)[sl], what + ": tm dx of the last sequence alone")
        one = torch.full((L, C), float("nan"), device=cuda)
        lib.call("es3_repmixer_ffn_bwd", x1[sl].contiguous().data_ptr(), du[sl].contiguous().data_ptr(), gg[sl].contiguous().data_ptr(),
                 wf.data_ptr(), bnf.data_ptr(), one.data_ptr(), _rmb_ws(lib, 1, C, cuda).data_ptr(), 0, 0, 0, 1, L, C, _st())
        _bits_equal(one, eo[:n].view(B * L, C)[sl], what + ": ffn e of the last sequence alone")

    a = {k: acc[k][0][:11 * C if k == "dwmc" else C].clone() for k in names}
    wdx, wdxb = ops.repmixer_tm_bwd(x, e, wmc, bnp, B, L, dtaps=a["dwmc"], dls=a["dls"], dbn=[a[k] for k in names[2:]], want_bf16=True)
    _bits_equal(wdx, dx[:n].view(B * L, C), "ops.repmixer_tm_bwd vs direct")
    _bits_equal(a["db_ns"], got["tm"][0]["db_ns"][:C], "ops.repmixer_tm_bwd db_ns vs direct")
    _bits_equal(ops.repmixer_ffn_bwd(x1, du, gg, wf, bnf, B, L), eo[:n].view(B * L, C), "ops.repmixer_ffn_bwd vs direct")
    _bits_equal(ops.repmixer_ls_bwd(gg, y, ls, B, L), dy[:n].view(B * L, C), "ops.repmixer_ls_bwd vs direct")


def test_repmixer_bwd_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    for L, C in ((129, 64), (8, 48)):
        z = torch.zeros(L * C * 13, device=cuda)
        out, _ = _flat_out(L * C, torch.float32, cuda)
        acc, _ = _flat_out(11 * C, torch.float32, cuda)
        ws = torch.full((13 * C * 2,), float("nan"), device=cuda)
        _declined(lib, "es3_repmixer_tm_bwd", (z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), out.data_ptr(), 0, ws.data_ptr(),
                                               acc.data_ptr(), *([0] * 7), 1, L, C, _st()), [out, acc, ws], f"repmixer_tm_bwd L{L} C{C}")
        _declined(lib, "es3_repmixer_ffn_bwd", (z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), out.data_ptr(),
                                                ws.data_ptr(), acc.data_ptr(), 0, 0, 1, L, C, _st()), [out, acc, ws],
                  f"repmixer_ffn_bwd L{L} C{C}")
        _declined(lib, "es3_repmixer_ls_bwd", (z.data_ptr(), z.data_ptr(), z.data_ptr(), out.data_ptr(), ws.data_ptr(), acc.data_ptr(),
                                               0, 1, L, C, _st()), [out, acc, ws], f"repmixer_ls_bwd L{L} C{C}")


# ----------------------------------------------------------------------------------------------------------- (4) embedding gradients
V_TEXT = 49408


def _ids(kind, cuda):
    """[B, L] int64 ids (CPU) with the structure `kind` names."""
    g = torch.Generator().manual_seed(zlib.crc32(kind.encode()))
    if kind == "chunk_edges":                  # ids with exactly 31, 32, 33, 64, 65 tokens, and some singletons
        ids = torch.cat([torch.full((n,), i + 1) for i, n in enumerate((31, 32, 33, 64, 65))] + [torch.arange(100, 125)])
        ids = ids[torch.randperm(ids.numel(), generator=g)]
        return ids.view(5, -1)
    if kind == "one_id":
        return torch.full((8, 77), 0)
    if kind == "distinct":
        return torch.randperm(V_TEXT, generator=g)[:4 * 77].view(4, 77)
    if kind == "single":
        return torch.tensor([[V_TEXT - 1]])
    if kind == "high":                         # ids near V - 1, with repeats and padding
        ids = V_TEXT - 1 - torch.randint(0, 40, (6, 32), generator=g)
        ids[:, 20:] = 0
        return ids
    raise ValueError(kind)


EMBED_GRAD = ["chunk_edges", "one_id", "distinct", "single", "high"]


@pytest.mark.parametrize("kind", EMBED_GRAD)
def test_embed_grad(cuda, kind):
    """es3_text_embed_grad over embed_grad_plan's chunks: the 32-token chunk edges, one id holding every token, all ids distinct,
    one token, ids at V - 1; the table prefilled with random values: used rows +=, every other row keeps its bits exactly."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    ids = _ids(kind, cuda)
    B, L = ids.shape
    C = 512
    g = _gen(cuda, "eg", kind)
    dx = torch.randn(B * L, C, device=cuda, generator=g)
    grad, ins = _prefilled(V_TEXT * C, cuda, g)
    plan = ops.embed_grad_plan(ids, cuda)
    wss = []

    def run(out):
        ws = torch.full((plan["nchunk"] * C,), float("nan"), device=cuda)
        lib.call("es3_text_embed_grad", dx.data_ptr(), plan["perm"].data_ptr(), plan["chunk_start"].data_ptr(), plan["nchunk"],
                 plan["seg"].data_ptr(), plan["uid"].data_ptr(), plan["uid"].numel(), C, ws.data_ptr(), out.data_ptr(), _st())
        wss.append(ws)
    got = _twice(run, grad)
    _bits_equal(wss[0], wss[1], "embed_grad chunk partials twice")
    ref, bound = R.embed_grad(dx.double(), ids.to(cuda), grad[:V_TEXT * C].view(V_TEXT, C).double())
    used = torch.zeros(V_TEXT, dtype=torch.bool, device=cuda)
    used[ids.reshape(-1).to(cuda)] = True
    gv = got[:V_TEXT * C].view(V_TEXT, C)
    _check("4 embed_grad", gv[used], ref[used], bound[used], f"embed_grad {kind}")
    _bits_equal(gv[~used], grad[:V_TEXT * C].view(V_TEXT, C)[~used], f"embed_grad {kind}: rows of absent ids")
    _assert_untouched(got, ins, f"embed_grad {kind}")
    w = grad[:V_TEXT * C].view(V_TEXT, C).clone()
    ops.text_embed_grad(dx, plan, w)
    _bits_equal(w, gv, "ops.text_embed_grad vs direct")


POS = [(77, 77, 4), (77, 32, 6), (16, 32, 3), (1, 9, 2), (9, 1, 5), (32, 77, 1), (1, 1, 64)]


@pytest.mark.parametrize("N,L,B", POS)
def test_pos_grad_and_resize(cuda, N, L, B):
    """es3_text_pos_grad (N = L, the 77-entry table at 32 tokens, 16 -> 32, N = 1, L = 1) into a random table, and
    es3_text_pos_resize (N != L) on the weights of the kernel's fp32 expression order."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    C = 512
    g = _gen(cuda, "pos", N, L, B)
    dx = torch.randn(B * L, C, device=cuda, generator=g)
    grad, ins = _prefilled(N * C, cuda, g)
    got = _twice(lambda o: lib.call("es3_text_pos_grad", dx.data_ptr(), B, L, N, C, o.data_ptr(), _st()), grad)
    ref, bound = R.pos_grad(dx.double().view(B, L, C), N, grad[:N * C].view(N, C).double())
    what = f"pos_grad N{N} L{L} B{B}"
    _check("4 pos_grad", got[:N * C].view(N, C), ref, bound, what)
    _assert_untouched(got, ins, what)
    w = grad[:N * C].view(N, C).clone()
    ops.text_pos_grad(dx, B, L, w)
    _bits_equal(w, got[:N * C].view(N, C), "ops.text_pos_grad vs direct")
    if N != L:
        tab = torch.randn(N, C, device=cuda, generator=g)
        out, oins = _flat_out(L * C, torch.float32, cuda)
        lib.call("es3_text_pos_resize", tab.data_ptr(), N, L, C, out.data_ptr(), _st())
        ref, bound = R.pos_resize(tab.double(), L)
        _check("4 pos_resize", out[:L * C].view(L, C), ref, bound, f"pos_resize N{N} L{L}")
        _assert_untouched(out, oins, f"pos_resize N{N} L{L}")
        _bits_equal(ops.text_pos_resize(tab, L), out[:L * C].view(L, C), "ops.text_pos_resize vs direct")


# ----------------------------------------------------------------------------------------------------------- (5) KD loss
KD = _pairwise(dict(D=[1, 33, 256, 1024], L=[1, 7, 8, 9, 32, 77], masked=[False, True], sd=[False, True], go=[False, True]),
               seed=14)


def _kd_inputs(cuda, B, L, D, g):
    p = torch.randn(B, L, D, device=cuda, generator=g)
    t = torch.randn(B, L, D, device=cuda, generator=g)
    p[0, 0] = 0.0                                                  # p = 0
    if L > 1:
        p[0, 1] = p[0, 1] / p[0, 1].norm() * 1e-9                  # |p| below the 1e-8 clamp
        t[1, 1] = 0.0                                              # t = 0
    pad = torch.zeros(B, L, dtype=torch.bool, device=cuda)
    for b in range(B):
        pad[b, (b % L) + 1:] = True
    pad[-1] = True                                                 # a sample without a valid token
    return p, t, pad


@pytest.mark.parametrize("D,L,masked,sd,go", KD)
def test_text_kd_loss(cuda, D, L, masked, sd, go):
    """ws [B, 3] and out3 of es3_text_kd_loss_fwd, then dp of es3_text_kd_loss_bwd (fp64 autograd of F.cosine_similarity + MSE) with
    scale_dev and gout each null or not; tokens with p = 0, |p| = 1e-9 and t = 0, a sample without a valid token; sample i's
    partials are bit-identical when it runs alone; ops wrappers bit-identical."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    B, w, gs = 5, 0.7, 0.5
    g = _gen(cuda, "kd", D, L, masked, sd, go)
    p, t, pad = _kd_inputs(cuda, B, L, D, g)
    padp = pad.view(torch.uint8) if masked else None
    ws_buf, wins = _flat_out(B * 3, torch.float32, cuda)
    outs = []

    def run(ws):
        o3 = torch.full((3 + TAIL,), float("nan"), device=cuda)
        lib.call("es3_text_kd_loss_fwd", p.data_ptr(), t.data_ptr(), _p(padp), B, L, D, w, ws.data_ptr(), o3.data_ptr(), _st())
        outs.append(o3)
    ws = _twice(run, ws_buf)
    _bits_equal(outs[0], outs[1], "kd out3 twice")
    (rws, bws), _ = R.kd_partials(p.double(), t.double(), pad if masked else None)
    what = f"kd_loss D{D} L{L} masked={masked}"
    _check("5 kd ws", ws[:B * 3].view(B, 3), rws, bws, what)
    _assert_untouched(ws, wins, what + " ws")
    r3, b3 = R.kd_out3(ws[:B * 3].view(B, 3).double(), bws, L, D, masked, w)
    _check("5 kd out3", outs[0][:3], r3, b3, what + " out3")
    _assert_untouched(outs[0], torch.arange(3 + TAIL, device=cuda) < 3, what + " out3")
    one = torch.full((3,), float("nan"), device=cuda)
    o3 = torch.full((3,), float("nan"), device=cuda)
    lib.call("es3_text_kd_loss_fwd", p[2:3].data_ptr(), t[2:3].data_ptr(), _p(None if padp is None else padp[2:3]), 1, L, D, w,
             one.data_ptr(), o3.data_ptr(), _st())
    _bits_equal(one, ws[6:9], what + ": sample 2 alone")
    sdv = torch.tensor([1.25], device=cuda) if sd else None
    gov = torch.tensor([3.0], device=cuda) if go else None
    gtot = gs * (1.25 if sd else 1.0) * (3.0 if go else 1.0)
    dbuf, dins = _flat_out(B * L * D, torch.float32, cuda)
    dp = _twice(lambda o: lib.call("es3_text_kd_loss_bwd", p.data_ptr(), t.data_ptr(), _p(padp), ws.data_ptr(), B, L, D, w, gs, _p(sdv),
                                   _p(gov), o.data_ptr(), _st()), dbuf)
    ref, bound = R.kd_bwd(p.double(), t.double(), pad if masked else None, ws[:B * 3].view(B, 3)[:, 2].double(), w, gtot)
    _check("5 kd dp", dp[:B * L * D].view(B, L, D), ref, bound, what + f" bwd sd={sd} gout={go}")
    _assert_untouched(dp, dins, what + " dp")
    wo, wws = ops.text_kd_loss_fwd(p, t, pad if masked else None, w)
    _bits_equal(wws, ws[:B * 3].view(B, 3), "ops.text_kd_loss_fwd ws vs direct")
    _bits_equal(wo, outs[0][:3], "ops.text_kd_loss_fwd out3 vs direct")
    wdp = ops.text_kd_loss_bwd(p, t, padp, wws, w, gs, sdv, gov)
    _bits_equal(wdp, dp[:B * L * D].view(B, L, D), "ops.text_kd_loss_bwd vs direct")


CON = [(1, 1, 1, False, False), (5, 7, 33, True, False), (3, 32, 256, False, True), (16, 77, 1024, True, True), (2, 9, 1, True, True)]


@pytest.mark.parametrize("B,L,D,sd,go", CON)
def test_text_consistency(cuda, B, L, D, sd, go):
    """mdiff [B, D], ws [B], value and loss += of es3_text_consistency_fwd; dp += and dq of es3_text_consistency_bwd on the mdiff
    it is given, with scale_dev and gout each null or not."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "con", B, L, D, sd, go)
    p, q = torch.randn(B, L, D, device=cuda, generator=g), torch.randn(B, L, D, device=cuda, generator=g)
    weight, gs = 0.3, 0.5
    md, mins = _flat_out(B * D, torch.float32, cuda)
    loss, lins = _prefilled(1, cuda, g)
    extra = []

    def run(m):
        ws = torch.full((B + TAIL,), float("nan"), device=cuda)
        val = torch.full((1 + TAIL,), float("nan"), device=cuda)
        ls = loss.clone()
        lib.call("es3_text_consistency_fwd", p.data_ptr(), q.data_ptr(), B, L, D, weight, m.data_ptr(), ws.data_ptr(), ls.data_ptr(),
                 val.data_ptr(), _st())
        extra.append((ws, val, ls))
    got = _twice(run, md)
    for i in range(3):
        _bits_equal(extra[0][i], extra[1][i], "consistency twice")
    r = R.consistency_fwd(p.double(), q.double(), weight, loss[:1].double()[0])
    what = f"consistency B{B} L{L} D{D}"
    _check("5 consistency mdiff", got[:B * D].view(B, D), *r["mdiff"], what)
    _assert_untouched(got, mins, what)
    ws, val, ls = extra[0]
    _check("5 consistency ws", ws[:B], *r["ws"], what + " ws")
    _check("5 consistency value", val[:1], *r["value"], what + " value")
    _check("5 consistency loss", ls[:1], *r["loss"], what + " loss +=")
    for t_, n in ((ws, B), (val, 1), (ls, 1)):
        _assert_untouched(t_, torch.arange(t_.numel(), device=cuda) < n, what)
    sdv = torch.tensor([1.25], device=cuda) if sd else None
    gov = torch.tensor([3.0], device=cuda) if go else None
    gtot = gs * (1.25 if sd else 1.0) * (3.0 if go else 1.0)
    dp0, dpins = _prefilled(B * L * D, cuda, g)
    dqs = []

    def runb(dp):
        dq = torch.full((B * L * D + TAIL,), float("nan"), device=cuda)
        lib.call("es3_text_consistency_bwd", got.data_ptr(), B, L, D, weight, gs, _p(sdv), _p(gov), dp.data_ptr(), dq.data_ptr(), _st())
        dqs.append(dq)
    dp = _twice(runb, dp0)
    rb = R.consistency_bwd(got[:B * D].view(B, D).double(), L, weight, gtot, dp0[:B * L * D].view(B, L, D).double())
    _check("5 consistency dp", dp[:B * L * D].view(B, L, D), *rb["dp"], what + " dp +=")
    _check("5 consistency dq", dqs[0][:B * L * D].view(B, L, D), *rb["dq"], what + " dq")
    _assert_untouched(dp, dpins, what + " dp")
    _assert_untouched(dqs[0], dpins, what + " dq")
    wv, wm = ops.text_consistency_fwd(p, q)
    _bits_equal(wm, got[:B * D].view(B, D), "ops.text_consistency_fwd vs direct")
    wdp = dp0[:B * L * D].view(B, L, D).clone()
    wdq = ops.text_consistency_bwd(wm, L, weight, wdp, gs, sdv, gov)
    _bits_equal(wdq, dqs[0][:B * L * D].view(B, L, D), "ops.text_consistency_bwd vs direct")


# ----------------------------------------------------------------------------------------------------------- (6) exact operations
EMB = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.parametrize("pos,emb", EMB)
def test_text_embed_exact(cuda, pos, emb):
    """x = table[id] (+ pos[l]) in fp32 (one rounding: torch's fp32 add), emb = the plain rows; ids outside [0, V) give zero rows."""
    from efficientsam3_b200 import ops
    lib = _lib(cuda)
    g = _gen(cuda, "emb", pos, emb)
    V, C, B, L = 1000, 512, 5, 20
    table = torch.randn(V, C, device=cuda, generator=g)
    pt = torch.randn(L, C, device=cuda, generator=g) if pos else None
    ids = torch.randint(0, V, (B, L), device=cuda, generator=g)
    ids[1, 3], ids[2, 0], ids[4, L - 1] = -1, V, V - 1
    x, xins = _flat_out(B * L * C, torch.float32, cuda)
    e, eins = _flat_out(B * L * C, torch.float32, cuda)
    lib.call("es3_text_embed", ids.data_ptr(), table.data_ptr(), V, _p(pt), x.data_ptr(), e.data_ptr() if emb else 0, B, L, C, _st())
    rows = torch.where(((ids >= 0) & (ids < V))[..., None], table[ids.clamp(0, V - 1)], torch.zeros(()).to(cuda))
    want = rows + pt if pos else rows
    _bits_equal(x[:B * L * C].view(B, L, C), want, "text_embed x")
    _assert_untouched(x, xins, "text_embed x")
    if emb:
        _bits_equal(e[:B * L * C].view(B, L, C), rows, "text_embed emb")
        _assert_untouched(e, eins, "text_embed emb")
    else:
        _assert_untouched(e, torch.zeros_like(eins), "text_embed emb (not requested)")
    wx, we = ops.text_embed(ids, table, pt, emb="plain")
    _bits_equal(wx, x[:B * L * C].view(B * L, C), "ops.text_embed x vs direct")
    _bits_equal(we, e[:B * L * C].view(B * L, C) if emb else rows.view(B * L, C), "ops.text_embed emb vs direct")
    px, pe = ops.text_embed(ids, table, pt, emb="pos")
    assert pe is px, "ops.text_embed(emb='pos') returns x itself"
    _bits_equal(px, wx, "ops.text_embed(emb='pos') x")


def _cast_inputs(n, cuda, g):
    x = torch.randn(n, device=cuda, generator=g) * torch.exp(torch.randn(n, device=cuda, generator=g) * 6)
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-40, 2.0 ** -149, 65504.0, 65520.0,
                             65519.99, 1e6, -1e6, 6e-8, 3e-8, 1.00390625, 1.01171875, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8,
                             1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 3.4e38, -3.4e38, 1.1754944e-38], device=cuda)
    x[:specials.numel()] = specials
    bf = x.to(torch.bfloat16).float()                       # exact ties of bf16 and of f16 steps
    x[100:1100] = bf[100:1100] + torch.ldexp(torch.ones(1000, device=cuda), torch.frexp(bf[100:1100])[1] - 9)
    hf = x[2000:3000].half().float()
    x[2000:3000] = hf + torch.ldexp(torch.ones(1000, device=cuda), torch.frexp(hf)[1] - 12)
    return x


CASTS = [4, 4096, 132 * 16 * 256 * 4 + 44]


@pytest.mark.parametrize("n", CASTS)
def test_casts_bit_exact(cuda, n):
    """es3_cast_f32_to_bf16 and es3_cast_f32_to_f16 against torch's .to(): ties, +-0, subnormals, +-inf, NaN, f16 overflow, at n past
    one grid stride (132 x 16 blocks of 256 threads x 4)."""
    lib = _lib(cuda)
    g = _gen(cuda, "cast", n)
    x = _cast_inputs(max(n, 4096), cuda, g)[:n].contiguous()
    yb, bins = _flat_out(n, torch.bfloat16, cuda)
    lib.call("es3_cast_f32_to_bf16", x.data_ptr(), yb.data_ptr(), n, _st())
    want = x.to(torch.bfloat16)
    nan = torch.isnan(want)
    _bits_equal(yb[:n][~nan], want[~nan], "cast_f32_to_bf16")
    assert torch.isnan(yb[:n][nan]).all()
    _assert_untouched(yb, bins, "cast_f32_to_bf16")
    yh = torch.full((n + TAIL,), float("nan"), dtype=torch.float16, device=cuda)
    lib.call("es3_cast_f32_to_f16", x.data_ptr(), yh.data_ptr(), n, _st())
    wh = x.to(torch.float16)
    nan = torch.isnan(wh)
    assert torch.equal(yh[:n][~nan].view(torch.int16), wh[~nan].view(torch.int16)), "cast_f32_to_f16"
    assert torch.isnan(yh[:n][nan]).all()
    assert torch.isnan(yh[n:]).all() and int((yh[n:].view(torch.int16) != yh[n:n + 1].view(torch.int16)).sum()) == 0


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    keys = {causal_attn_key(c[0]) if c[4] else attn_key("es3_attention_bf16", 1, c[0], 0) for c in ATTN}
    keys |= {("es3_text_attn_bwd", c[4]) for c in ATTN}
    keys |= {("es3_layernorm_f32", c[0] // 128) for c in LNF}
    keys |= {("es3_layernorm_bwd_f32", c[2], c[3], c[1] > 37888) for c in LNB}
    keys |= {("es3_repmixer_bf16",) for _ in REPMIXER}
    keys |= {(k,) for _ in RMB for k in ("es3_repmixer_ls_bwd", "es3_repmixer_ffn_bwd", "es3_repmixer_tm_bwd")}
    keys |= {("es3_text_pos_resize",) for N, L, _ in POS if N != L} | {("es3_text_pos_grad", N == L) for N, L, _ in POS}
    keys |= {("es3_text_embed_grad",) for _ in EMBED_GRAD}
    keys |= {("es3_text_kd_loss_fwd", c[2]) for c in KD} | {("es3_text_kd_loss_bwd", c[2], c[3], c[4]) for c in KD}
    keys |= {("es3_text_consistency_fwd",) for _ in CON} | {("es3_text_consistency_bwd", c[3], c[4]) for c in CON}
    keys |= {("es3_text_embed",) for _ in EMB} | {k for _ in CASTS for k in (("es3_cast_f32_to_bf16",), ("es3_cast_f32_to_f16",))}
    return keys
