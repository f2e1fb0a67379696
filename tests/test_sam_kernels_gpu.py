"""The SAM heads' kernels (decoder.cu's prompt encoder, two-way transformer and mask decoder kernels and the strict-mode twins in
strict_f32.cu), element by element against the fp64 statements of tests/ref_sam.py, each output element within its own bound.

Outputs are NaN-prefilled and called through _lib.call: every cell inside the output region must be written and lie within its bound,
every cell past it (a flat TAIL) keeps its sentinel bits.  Every kernel runs twice and must be bit-identical; the last prompt or image
of a batch is bit-identical to the same one run alone; a shape an entry point declines writes nothing; the ops wrappers are
bit-identical to the direct calls.  The copies (es3_nchw_f32_to_tokens, es3_add_rows' stores, the gated masks, the same-size resize)
are bit-exact.  covered_keys() names the route keys (tests/routes.py) the tables run, for the route closure of
tests/test_route_closure_gpu.py (the interactive predictor and the point segmenter on the ViT and an EV-B1 student, every prompt
kind, >= 10 points, both output modes, the object-gated batch path, the module API, strict mode).

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power
limit): bf16 outputs, where the output's own rounding half-step dominates the bound -- attn_few_keys 0.987, ln_rows_gelu 0.991,
mask_downscale's bf16 store 0.977; fp32 outputs -- dense_pe 0.412, point_embed 0.376, add_rows 0.25, attn_few_keys_f32 0.059,
attn_few_queries 0.014 (head_dim 16) and 0.048 (head_dim 32), ln_rows_gelu_f32 0.071, bilinear 0.432, hyper_masks 0.062,
mask_downscale 0.0052.  The whole file (137 tests, the route-closure predictor runs included, since moved to tests/test_route_closure_gpu.py) took 15 s
there.
"""
import pytest
import torch

import ref_sam as R
from bounds import (TAIL, _assert_untouched, _bf, _bits_equal, _check, _declined, _flat_out, _gen, _lib, _p, _pairwise, _st, _twice,
                    report_worst)

pytestmark = pytest.mark.gpu
_report_worst = report_worst("SAM-head kernels")


# ----------------------------------------------------------------------------------------------------------- (1) positional encodings
DENSE = [(72, 72), (28, 28), (5, 7), (1, 1)]


@pytest.mark.parametrize("h,w", DENSE)
def test_dense_pe(cuda, h, w):
    lib = _lib(cuda)
    gauss = torch.randn(2, 128, device=cuda, generator=_gen(cuda, "dpe", h, w)) * 3
    buf, ins = _flat_out(h * w * 256, torch.float32, cuda)
    got = _twice(lambda o: lib.call("es3_dense_pe", gauss.data_ptr(), 128, h, w, o.data_ptr(), _st()), buf)
    ref, bound = R.dense_pe(gauss.double(), h, w)
    _check("1 dense_pe", got[:h * w * 256].view(h * w, 256), ref, bound, f"dense_pe {h}x{w}")
    _assert_untouched(got, ins, f"dense_pe {h}x{w}")
    from efficientsam3_b200 import ops
    _bits_equal(ops.dense_pe(gauss, h, w), got[:h * w * 256].view(h * w, 256), "ops.dense_pe vs direct")


def _prompt(kind, B, P, S, cuda, g):
    coords = torch.rand(B, P, 2, device=cuda, generator=g) * (S - 1)
    labels = torch.randint(0, 4, (B, P), device=cuda, generator=g, dtype=torch.int32)
    if kind == "labels":                 # -1 .. 3 and the out-of-range 4, -2, 7 in turn
        labels = torch.tensor([-1, 0, 1, 2, 3, 4, -2, 7], dtype=torch.int32, device=cuda).repeat(B * P)[:B * P].view(B, P).contiguous()
    if kind == "edges" and P:
        edge = torch.tensor([[0.0, 0.0], [S - 1.0, S - 1.0], [-3.0, 5.0], [S + 40.0, 2.0 * S], [0.0, S - 1.0]], device=cuda)
        coords.view(-1, 2)[:min(5, B * P)] = edge[:min(5, B * P)]
    return coords, labels


POINTS = [(1, 1, True, "labels"), (4, 5, True, "edges"), (3, 12, True, "labels"), (2, 2, False, "edges"), (1, 0, True, "labels"),
          (2, 40, True, "random"), (1, 20, False, "labels")]


@pytest.mark.parametrize("B,P,pad,kind", POINTS)
def test_point_embed(cuda, B, P, pad, kind):
    """Labels -1..3, 4, -2 and 7; pad on and off; P = 0 (a box's corners come in with labels 2 / 3 and pad off, the pad point alone
    with pad on); coordinates at 0, S - 1, negative and past S; label -1 and the pad point are not_a_point exactly."""
    lib = _lib(cuda)
    S = 1008.0
    g = _gen(cuda, "pt", B, P, pad, kind)
    coords, labels = _prompt(kind, B, P, S, cuda, g)
    gauss = torch.randn(2, 128, device=cuda, generator=g)
    nap, table = torch.randn(256, device=cuda, generator=g), torch.randn(4, 256, device=cuda, generator=g)
    n = B * (P + int(pad)) * 256
    buf, ins = _flat_out(n, torch.float32, cuda)
    run = lambda o: lib.call("es3_point_embed", coords.data_ptr(), labels.data_ptr(), gauss.data_ptr(), nap.data_ptr(), table.data_ptr(),
                             128, B, P, int(pad), S, S, o.data_ptr(), _st())
    got = _twice(run, buf)
    ref, bound, exact = R.point_embed(coords.double(), labels, gauss.double(), nap.double(), table.double(), S, S, pad)
    out = got[:n].view(B, P + int(pad), 256)
    what = f"point_embed B{B} P{P} pad={pad} {kind}"
    _check("1 point_embed", out, ref, bound, what)
    _bits_equal(out[exact], ref[exact].float(), what + ": not_a_point rows")
    _assert_untouched(got, ins, what)
    from efficientsam3_b200 import ops
    _bits_equal(ops.point_embed(coords, labels, gauss, nap, table, S, S, pad=pad), out, "ops.point_embed vs direct")
    if B > 1:
        one = torch.full((P + int(pad), 256), float("nan"), device=cuda)
        lib.call("es3_point_embed", coords[-1:].contiguous().data_ptr(), labels[-1:].contiguous().data_ptr(), gauss.data_ptr(), nap.data_ptr(),
                 table.data_ptr(), 128, 1, P, int(pad), S, S, one.data_ptr(), _st())
        _bits_equal(one, out[-1], what + ": last prompt alone")


# ----------------------------------------------------------------------------------------------------------- (2) copies and adds
ADD = [(add, out) for add in ("none", "R1", "RHW") for out in ("f32", "bf16", "both")]


@pytest.mark.parametrize("add,out", ADD)
def test_add_rows(cuda, add, out):
    """x + add[m % R] with R = 1 (queries + a pe row), R = HW with M = P HW (keys + the image pe over P prompts), add = null (the trunk's
    bf16 cast): the fp32 store is torch's fp32 sum bit for bit, the bf16 store its round-to-nearest."""
    lib = _lib(cuda)
    g = _gen(cuda, "add", add, out)
    P, HW, C = 3, 5184 + 4, 256
    M = P * HW
    x = torch.randn(M, C, device=cuda, generator=g) * 4
    R_ = {"none": 0, "R1": 1, "RHW": HW}[add]
    a = torch.randn(max(R_, 1), C, device=cuda, generator=g) if R_ else None
    yf, fins = _flat_out(M * C, torch.float32, cuda)
    yb, bins = _flat_out(M * C, torch.bfloat16, cuda)
    want_f, want_b = out in ("f32", "both"), out in ("bf16", "both")
    bb = []

    def run(o):
        b = yb.clone()
        lib.call("es3_add_rows", x.data_ptr(), _p(a), M, C, R_, b.data_ptr() if want_b else 0, o.data_ptr() if want_f else 0, _st())
        bb.append(b)
    got = _twice(run, yf)
    _bits_equal(bb[0], bb[1], "add_rows bf16 twice")
    want = x if a is None else x + a.repeat(M // a.shape[0], 1)
    what = f"add_rows {add} {out}"
    if want_f:
        _bits_equal(got[:M * C].view(M, C), want, what + ": fp32 vs torch")
        ref = x.double() if a is None else x.double() + a.double().repeat(M // a.shape[0], 1)
        _check("2 add_rows", got[:M * C].view(M, C), ref, 4 * R.U * ref.abs() + 1e-30, what)
        _assert_untouched(got, fins, what)
    else:
        _assert_untouched(got, torch.zeros_like(fins), what + " (fp32 not requested)")
    if want_b:
        _bits_equal(bb[0][:M * C].view(M, C), want.to(torch.bfloat16), what + ": bf16 vs RN(fp32)")
        _assert_untouched(bb[0], bins, what)
    else:
        _assert_untouched(bb[0], torch.zeros_like(bins), what + " (bf16 not requested)")
    from efficientsam3_b200 import ops
    wb, wf = ops.add_rows(x, a, out_bf16=want_b, out_f32=want_f)
    if want_f:
        _bits_equal(wf, got[:M * C].view(M, C), "ops.add_rows vs direct")
    if want_b:
        _bits_equal(wb, bb[0][:M * C].view(M, C), "ops.add_rows bf16 vs direct")


NCHW = [(1, 256, 5184, "both"), (2, 256, 784, "f32"), (3, 32, 37, "bf16"), (1, 64, 1, "both"), (2, 40, 33, "f32")]


@pytest.mark.parametrize("B,C,HW,out", NCHW)
def test_nchw_to_tokens_bit_exact(cuda, B, C, HW, out):
    lib = _lib(cuda)
    x = torch.randn(B, C, HW, device=cuda, generator=_gen(cuda, "nchw", B, C, HW)) * 1e3
    n = B * HW * C
    yf, fins = _flat_out(n, torch.float32, cuda)
    yb, bins = _flat_out(n, torch.bfloat16, cuda)
    want_f, want_b = out in ("f32", "both"), out in ("bf16", "both")
    lib.call("es3_nchw_f32_to_tokens", x.data_ptr(), yf.data_ptr() if want_f else 0, yb.data_ptr() if want_b else 0, B, HW, C, _st())
    t = x.permute(0, 2, 1).reshape(B * HW, C)
    what = f"nchw_to_tokens B{B} C{C} HW{HW} {out}"
    _assert_untouched(yf, fins if want_f else torch.zeros_like(fins), what)
    _assert_untouched(yb, bins if want_b else torch.zeros_like(bins), what)
    if want_f:
        _bits_equal(yf[:n].view(B * HW, C), t, what)
    if want_b:
        _bits_equal(yb[:n].view(B * HW, C), t.to(torch.bfloat16), what + " bf16")
    from efficientsam3_b200 import ops
    wf, wb = ops.nchw_to_tokens(x.view(B, C, HW, 1), out_bf16=want_b, out_f32=want_f)
    if want_f:
        _bits_equal(wf, t, "ops.nchw_to_tokens")


# ----------------------------------------------------------------------------------------------------------- (3) attention
def _scores(q, k, kind):
    if kind == "peaked":
        return q * 6, k * 6
    if kind == "flat":
        return q * 0, k
    if kind == "tied":
        return q, k[:, torch.arange(k.shape[1], device=k.device) % 3]
    return q, k


FQ = _pairwise(dict(Tq=[6, 7, 8, 17, 27, 40], Tk=[256, 784, 5184, 0], hk=[(16, False), (16, True), (32, True)], B=[1, 3],
                    kind=["random", "peaked", "flat", "tied"]), seed=31)


@pytest.mark.parametrize("Tq,Tk,hk,B,kind", FQ)
def test_attn_few_queries(cuda, Tq, Tk, hk, B, kind):
    """Token-to-image (head_dim 16, bf16 or fp32 K/V) at the 256, 784 and 5184 image tokens of the ViT override, the 448-px student
    and 1008 px, and self-attention (head_dim 32, fp32 K/V, Tk = Tq: < 32 keys leaves lanes empty); Tq up to 40 (long prompts)."""
    lib = _lib(cuda)
    hd, kv32 = hk
    Tk = Tk or Tq
    H = 8
    Dm = H * hd
    g = _gen(cuda, "fq", Tq, Tk, hk, B, kind)
    q, k = _scores(torch.randn(B, Tq, Dm, device=cuda, generator=g), torch.randn(B, Tk, Dm, device=cuda, generator=g), kind)
    v = torch.randn(B, Tk, Dm, device=cuda, generator=g)
    if not kv32:
        k, v = _bf(k), _bf(v)
    scale = hd ** -0.5
    run = lambda qq, kk, vv, o, b: lib.call("es3_attn_few_queries", qq.data_ptr(), Dm, kk.data_ptr(), vv.data_ptr(), Dm, int(kv32),
                                            o.data_ptr(), Dm, b, H, hd, Tq, Tk, scale, _st())
    buf, ins = _flat_out(B * Tq * Dm, torch.float32, cuda)
    got = _twice(lambda o: run(q, k, v, o, B), buf)
    out = got[:B * Tq * Dm].view(B, Tq, Dm)
    ref, bound = R.attn_few_queries(q.double(), k.double(), v.double(), H, scale)
    what = f"attn_few_queries Tq{Tq} Tk{Tk} hd{hd} kv32={kv32} B{B} {kind}"
    _check(f"3 attn_few_queries hd{hd}", out, ref, bound, what)
    _assert_untouched(got, ins, what)
    from efficientsam3_b200 import ops
    _bits_equal(ops.attn_few_queries(q, k, v, H, scale), out, "ops.attn_few_queries vs direct")
    if B > 1:
        one = torch.full((Tq, Dm), float("nan"), device=cuda)
        run(q[-1:].contiguous(), k[-1:].contiguous(), v[-1:].contiguous(), one, 1)
        _bits_equal(one, out[-1], what + ": last image alone")


FK = _pairwise(dict(Tk=[6, 7, 16, 17, 31, 32, 33, 64], Nq=[1, 37, 784, 5184], B=[1, 2], kind=["random", "peaked", "flat", "tied"],
                    strict=[False, True]), seed=32)


@pytest.mark.parametrize("Tk,Nq,B,kind,strict", FK)
def test_attn_few_keys(cuda, Tk, Nq, B, kind, strict):
    """Image-to-token attention over one and several 16-key tiles (Tk up to 64), Nq H ragged against the 256-thread block (37 and 784
    queries x 8 heads), bf16 mode and the strict fp32 twin."""
    lib = _lib(cuda)
    H, hd = 8, 16
    Dm = H * hd
    g = _gen(cuda, "fk", Tk, Nq, B, kind, strict)
    q, k = _scores(torch.randn(B, Nq, Dm, device=cuda, generator=g), torch.randn(B, Tk, Dm, device=cuda, generator=g), kind)
    v = torch.randn(B, Tk, Dm, device=cuda, generator=g)
    dt = torch.float32 if strict else torch.bfloat16
    q = q.to(dt)
    name = "es3_attn_few_keys_f32" if strict else "es3_attn_few_keys"
    run = lambda qq, kk, vv, o, b: lib.call(name, qq.data_ptr(), Dm, kk.data_ptr(), vv.data_ptr(), Dm, o.data_ptr(), Dm, b, H, hd, Nq, Tk,
                                            0.25, _st())
    buf, ins = _flat_out(B * Nq * Dm, dt, cuda)
    got = _twice(lambda o: run(q, k, v, o, B), buf)
    out = got[:B * Nq * Dm].view(B, Nq, Dm)
    ref, bound = R.attn_few_keys(q.double(), k.double(), v.double(), H, 0.25, strict)
    what = f"attn_few_keys Tk{Tk} Nq{Nq} B{B} {kind} strict={strict}"
    _check(f"3 attn_few_keys{'_f32' if strict else ''}", out, ref, bound, what)
    _assert_untouched(got, ins, what)
    from efficientsam3_b200 import ops
    w = (ops.attn_few_keys_f32 if strict else ops.attn_few_keys)(q.view(B * Nq, Dm), k, v, B, H, 0.25)
    _bits_equal(w, out.view(B * Nq, Dm), "ops.attn_few_keys vs direct")
    if B > 1:
        one = torch.full((Nq, Dm), float("nan"), dtype=dt, device=cuda)
        run(q[-1:].contiguous(), k[-1:].contiguous(), v[-1:].contiguous(), one, 1)
        _bits_equal(one, out[-1], what + ": last image alone")


def test_attention_declined_shapes_write_nothing(cuda):
    """es3_attn_few_queries with head_dim 32 and bf16 K/V (no model reaches it) or head_dim 64; es3_attn_few_keys with head_dim 32
    or no key."""
    lib = _lib(cuda)
    z = torch.zeros(64 * 512, device=cuda)
    out, _ = _flat_out(8 * 512, torch.float32, cuda)
    for hd, kv32 in ((32, 0), (64, 1), (8, 1)):
        _declined(lib, "es3_attn_few_queries", (z.data_ptr(), 8 * hd, z.data_ptr(), z.data_ptr(), 8 * hd, kv32, out.data_ptr(), 8 * hd, 1, 8,
                                                hd, 4, 16, 0.1, _st()), [out], f"attn_few_queries hd{hd} kv32={kv32}")
    for name in ("es3_attn_few_keys", "es3_attn_few_keys_f32"):
        for hd, Tk in ((32, 8), (16, 0)):
            _declined(lib, name, (z.data_ptr(), 8 * hd, z.data_ptr(), z.data_ptr(), 8 * hd, out.data_ptr(), 8 * hd, 1, 8, hd, 4, Tk, 0.1, _st()),
                      [out], f"{name} hd{hd} Tk{Tk}")


# ----------------------------------------------------------------------------------------------------------- (4) LayerNorm + GELU
LNG = _pairwise(dict(C=[64, 32, 96, 128], M=[1, 13, 2051, 20736], kind=["random", "constant", "shifted"], strict=[False, True]), seed=33)


@pytest.mark.parametrize("C,M,kind,strict", LNG)
def test_ln_rows_gelu(cuda, C, M, kind, strict):
    """C = 64 (the upscaling's 256 / 4) and the other accepted widths; M ragged against 8 rows per block; constant rows (rstd = 1000
    at eps 1e-6) and rows whose mean is 1000 x their spread; bf16 (es3_gelu_fast) and the strict fp32 twin (erf)."""
    lib = _lib(cuda)
    g = _gen(cuda, "lng", C, M, kind, strict)
    x = torch.randn(M, C, device=cuda, generator=g)
    if kind == "constant":
        x = x[:, :1].expand(M, C).contiguous()
    elif kind == "shifted":
        x = x * 1e-2 + 10.0
    w, b = torch.randn(C, device=cuda, generator=g) + 1, torch.randn(C, device=cuda, generator=g)
    dt = torch.float32 if strict else torch.bfloat16
    name = "es3_ln_rows_gelu_f32" if strict else "es3_ln_rows_gelu"
    run = lambda xx, o, m: lib.call(name, xx.data_ptr(), w.data_ptr(), b.data_ptr(), 1e-6, o.data_ptr(), m, C, _st())
    buf, ins = _flat_out(M * C, dt, cuda)
    got = _twice(lambda o: run(x, o, M), buf)
    out = got[:M * C].view(M, C)
    ref, bound = R.ln_rows_gelu(x.double(), w.double(), b.double(), 1e-6, strict)
    what = f"ln_rows_gelu C{C} M{M} {kind} strict={strict}"
    _check(f"4 ln_rows_gelu{'_f32' if strict else ''}", out, ref, bound, what)
    _assert_untouched(got, ins, what)
    from efficientsam3_b200 import ops
    _bits_equal((ops.ln_rows_gelu_f32 if strict else ops.ln_rows_gelu)(x, w, b, 1e-6), out, "ops.ln_rows_gelu vs direct")
    one = torch.full((1, C), float("nan"), dtype=dt, device=cuda)
    run(x[-1:].contiguous(), one, 1)
    _bits_equal(one, out[-1:], what + ": last row alone")


def test_ln_rows_gelu_declined_widths_write_nothing(cuda):
    lib = _lib(cuda)
    for name, dt in (("es3_ln_rows_gelu", torch.bfloat16), ("es3_ln_rows_gelu_f32", torch.float32)):
        for C in (48, 160):
            x = torch.zeros(4 * C, device=cuda)
            y, _ = _flat_out(4 * C, dt, cuda)
            _declined(lib, name, (x.data_ptr(), x.data_ptr(), x.data_ptr(), 1e-6, y.data_ptr(), 4, C, _st()), [y], f"{name} C{C}")


# ----------------------------------------------------------------------------------------------------------- (5) mask tail
HM = _pairwise(dict(KO=[(3, 1), (1, 0), (4, 0)], HW=[20736, 1000, 300], B=[1, 2, 4], gate=[False, True]), seed=34)


@pytest.mark.parametrize("KO,HW,B,gate", HM)
def test_hyper_masks(cuda, KO, HW, B, gate):
    """The multimask (3 masks from token 1) and single (token 0) selections, HW ragged against 256 (1000, 300), B up to 4; the object
    gate with logits > 0, 0, -0, NaN and < 0: gated images are exactly -1024."""
    lib = _lib(cuda)
    K, off = KO
    g = _gen(cuda, "hm", KO, HW, B, gate)
    up, hyper = torch.randn(B, HW, 32, device=cuda, generator=g), torch.randn(B, 4, 32, device=cuda, generator=g)
    obj = torch.tensor([1.5, 0.0, -0.0, float("nan"), -2.0][:B] if B < 4 else [1.5, 0.0, float("nan"), -2.0], device=cuda) if gate else None
    run = lambda u, hh, ob, o, b: lib.call("es3_hyper_masks", u.data_ptr(), hh.data_ptr(), _p(ob), -1024.0, o.data_ptr(), b, HW, 32, 4, K,
                                           off, _st())
    buf, ins = _flat_out(B * K * HW, torch.float32, cuda)
    got = _twice(lambda o: run(up, hyper, obj, o, B), buf)
    out = got[:B * K * HW].view(B, K, HW)
    ref, bound, gated = R.hyper_masks(up.double(), hyper.double(), None if obj is None else obj.double(), -1024.0, K, off)
    what = f"hyper_masks K{K} off{off} HW{HW} B{B} gate={gate}"
    g_ = gated.reshape(-1)
    assert (out[g_] == -1024.0).all(), what + ": gated masks"
    if (~g_).any():
        _check("5 hyper_masks", out[~g_], ref[~g_], bound[~g_], what)
    _assert_untouched(got, ins, what)
    from efficientsam3_b200 import ops
    _bits_equal(ops.hyper_masks(up, hyper, obj, -1024.0, K, off), out, "ops.hyper_masks vs direct")
    if B > 1:
        one = torch.full((K, HW), float("nan"), device=cuda)
        run(up[-1:].contiguous(), hyper[-1:].contiguous(), None if obj is None else obj[-1:].contiguous(), one, 1)
        _bits_equal(one, out[-1], what + ": last image alone")


def test_hyper_masks_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    z = torch.zeros(300 * 32 * 9, device=cuda)
    out, _ = _flat_out(9 * 300, torch.float32, cuda)
    for K, CU in ((9, 32), (1, 16)):
        _declined(lib, "es3_hyper_masks", (z.data_ptr(), z.data_ptr(), 0, -1024.0, out.data_ptr(), 1, 300, CU, 9, K, 0, _st()), [out],
                  f"hyper_masks K{K} CU{CU}")


BIL = [(288, 288, 1008, 1008, "bin"), (288, 288, 1008, 1008, "float"), (288, 288, 300, 420, "both"), (288, 288, 100, 70, "bin"),
       (288, 288, 100, 70, "float"), (288, 288, 288, 288, "both"), (72, 72, 64, 64, "float"), (7, 5, 20, 33, "both")]


@pytest.mark.parametrize("Hi,Wi,Ho,Wo,mode", BIL)
def test_bilinear_nchw(cuda, Hi, Wi, Ho, Wo, mode):
    """The predictor's 288 -> 1008 high-res masks, the resizes to an original size of non-square aspect (300 x 420 up, 100 x 70 down),
    the identity (bit-exact), the stage-1 student's 72 -> 64 feature resize; float output, `bin` output, both: bin is out > thr of the
    same kernel bit for bit (== goes to 0) and agrees with the fp64 reference wherever |ref - thr| exceeds the bound."""
    lib = _lib(cuda)
    planes = 3
    g = _gen(cuda, "bil", Hi, Wi, Ho, Wo, mode)
    x = torch.randn(planes, Hi, Wi, device=cuda, generator=g) * 8
    x[0, :2, :2] = 0.0                                   # exact zeros at the threshold
    n = planes * Ho * Wo
    fo, fins = _flat_out(n, torch.float32, cuda)
    bo = torch.full((n + TAIL,), 0xA5, dtype=torch.uint8, device=cuda)
    want_f, want_b = mode in ("float", "both"), mode in ("bin", "both")
    bins = []

    def run(o):
        b = bo.clone()
        lib.call("es3_bilinear_nchw_f32", x.data_ptr(), o.data_ptr() if want_f else 0, b.data_ptr() if want_b else 0, 0.0, planes, Hi, Wi,
                 Ho, Wo, _st())
        bins.append(b)
    got = _twice(run, fo)
    assert torch.equal(bins[0], bins[1]), "bilinear bin twice"
    what = f"bilinear {Hi}x{Wi} -> {Ho}x{Wo} {mode}"
    ref, bound = R.bilinear(x.double(), Ho, Wo)
    full = torch.full((n,), float("nan"), device=cuda)
    lib.call("es3_bilinear_nchw_f32", x.data_ptr(), full.data_ptr(), 0, 0.0, planes, Hi, Wi, Ho, Wo, _st())
    val = full.view(planes, Ho, Wo)
    if want_f:
        _bits_equal(got[:n], full, what + ": float vs a float-only run")
        _check("5 bilinear", got[:n].view(planes, Ho, Wo), ref, bound, what)
        _assert_untouched(got, fins, what)
    else:
        _assert_untouched(got, torch.zeros_like(fins), what + " (float not requested)")
        _check("5 bilinear", val, ref, bound, what)
    if (Hi, Wi) == (Ho, Wo):
        _bits_equal(val, x, what + ": identity")
    if want_b:
        b = bins[0][:n].view(planes, Ho, Wo)
        assert torch.equal(b, (val > 0).to(torch.uint8)), what + ": bin vs out > thr"
        safe = (ref - 0.0).abs() > bound
        assert torch.equal(b.bool()[safe], (ref > 0)[safe]), what + ": bin vs the fp64 reference"
        assert (bins[0][n:] == 0xA5).all(), what + ": bin tail"
    else:
        assert (bins[0] == 0xA5).all(), what + " (bin not requested)"
    from efficientsam3_b200 import ops
    wf, wb = ops.bilinear_nchw(x.view(1, planes, Hi, Wi), Ho, Wo, binarize_thr=0.0 if want_b else None, want_float=want_f)
    if want_f:
        _bits_equal(wf.view(planes, Ho, Wo), val, "ops.bilinear_nchw vs direct")
    if want_b:
        assert torch.equal(wb.view(planes, Ho, Wo), bins[0][:n].view(planes, Ho, Wo))
    one = torch.full((Ho * Wo,), float("nan"), device=cuda)
    lib.call("es3_bilinear_nchw_f32", x[-1:].contiguous().data_ptr(), one.data_ptr(), 0, 0.0, 1, Hi, Wi, Ho, Wo, _st())
    _bits_equal(one.view(Ho, Wo), val[-1], what + ": last plane alone")


# ----------------------------------------------------------------------------------------------------------- (6) mask prompt
def _mask_wts(cuda, g, flat):
    w = [torch.randn(4, 4, device=cuda, generator=g) * 0.5, torch.randn(4, device=cuda, generator=g),
         torch.randn(4, device=cuda, generator=g) + 1, torch.randn(4, device=cuda, generator=g) * 0.1,
         torch.randn(16, 16, device=cuda, generator=g) * 0.3, torch.randn(16, device=cuda, generator=g),
         torch.randn(16, device=cuda, generator=g) + 1, torch.randn(16, device=cuda, generator=g) * 0.1,
         torch.randn(256, 16, device=cuda, generator=g) * 0.25, torch.randn(256, device=cuda, generator=g)]
    if flat:                                   # the first LayerNorm's variance comparable to eps
        w[0] = w[0] * 1e-3
        w[1] = 0.5 + 1e-3 * torch.randn(4, device=cuda, generator=g)
    return [t.contiguous() for t in w]


MD = _pairwise(dict(hw=[(72, 72), (28, 28), (5, 5), (7, 9)], B=[1, 2, 3], base=[False, True], out=["f32", "bf16", "both"],
                    kind=["random", "saturated", "flat"]), seed=35)


@pytest.mark.parametrize("hw,B,base,out,kind", MD)
def test_mask_downscale(cuda, hw, B, base, out, kind):
    """B h w ragged against the 16-pixel block; base null and base_rows = h w; fp32 and / or bf16 stores (bf16 = RN of the fp32 value
    bit for bit); mask logits random, saturated at +-1024 (a gated previous mask fed back), and constant with the first LayerNorm's
    variance near eps."""
    lib = _lib(cuda)
    h, w = hw
    C = 256
    g = _gen(cuda, "md", hw, B, base, out, kind)
    m = torch.randn(B, 1, 4 * h, 4 * w, device=cuda, generator=g) * 3
    if kind == "saturated":
        m = torch.where(m > 0, 1024.0, -1024.0)
    elif kind == "flat":
        m = torch.full_like(m, 0.25)
    wts = _mask_wts(cuda, g, kind == "flat")
    bt = torch.randn(h * w, C, device=cuda, generator=g) if base else None
    rows = B * h * w
    want_f, want_b = out in ("f32", "both"), out in ("bf16", "both")
    yb, bins = _flat_out(rows * C, torch.bfloat16, cuda)
    bbs = []

    def run(o):
        b = yb.clone()
        lib.call("es3_mask_downscale_tokens", m.data_ptr(), *[t.data_ptr() for t in wts], _p(bt), h * w if base else 0,
                 o.data_ptr() if want_f else 0, b.data_ptr() if want_b else 0, B, h, w, C, 1e-6, _st())
        bbs.append(b)
    buf, fins = _flat_out(rows * C, torch.float32, cuda)
    got = _twice(run, buf)
    _bits_equal(bbs[0], bbs[1], "mask_downscale bf16 twice")
    ref, bound = R.mask_downscale(m.double(), [t.double() for t in wts], 1e-6, None if bt is None else bt.double())
    what = f"mask_downscale {h}x{w} B{B} base={base} {out} {kind}"
    if want_f:
        _check("6 mask_downscale", got[:rows * C].view(rows, C), ref, bound, what)
        _assert_untouched(got, fins, what)
    else:
        _assert_untouched(got, torch.zeros_like(fins), what + " (fp32 not requested)")
    if want_b:
        _check("6 mask_downscale bf16", bbs[0][:rows * C].view(rows, C), ref, R._out(ref, bound, True), what + " bf16")
        _assert_untouched(bbs[0], bins, what + " bf16")
        if want_f:
            _bits_equal(bbs[0][:rows * C], got[:rows * C].to(torch.bfloat16), what + ": bf16 vs RN(fp32)")
    else:
        _assert_untouched(bbs[0], torch.zeros_like(bins), what + " (bf16 not requested)")
    from efficientsam3_b200 import ops
    wb, wf = ops.mask_downscale_tokens(m, wts, bt, 1e-6, out_bf16=want_b, out_f32=want_f)
    if want_f:
        _bits_equal(wf, got[:rows * C].view(rows, C), "ops.mask_downscale_tokens vs direct")
    if B > 1:
        one = torch.full((h * w, C), float("nan"), device=cuda)
        lib.call("es3_mask_downscale_tokens", m[-1:].contiguous().data_ptr(), *[t.data_ptr() for t in wts], _p(bt), h * w if base else 0,
                 one.data_ptr(), 0, 1, h, w, C, 1e-6, _st())
        ref_last = ops.mask_downscale_tokens(m, wts, bt, 1e-6, out_bf16=False)[1][-h * w:]
        _bits_equal(one, ref_last, what + ": last image alone")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    keys = {("es3_dense_pe",)} | {("es3_point_embed", pad) for _, _, pad, _ in POINTS}
    keys |= {("es3_add_rows", add != "none", out != "f32", out != "bf16") for add, out in ADD}
    keys |= {("es3_nchw_f32_to_tokens", out != "bf16", out != "f32") for *_, out in NCHW}
    keys |= {("es3_attn_few_queries", hk[0], hk[1]) for _, _, hk, _, _ in FQ}
    keys |= {("es3_attn_few_keys_f32" if s else "es3_attn_few_keys", tk > 16) for tk, _, _, _, s in FK}
    keys |= {("es3_ln_rows_gelu_f32" if s else "es3_ln_rows_gelu", C) for C, _, _, s in LNG}
    keys |= {("es3_hyper_masks", gate, K, off) for (K, off), _, _, gate in HM}
    keys |= {("es3_bilinear_nchw_f32", mode != "bin", mode != "float") for *_, mode in BIL}
    keys |= {("es3_mask_downscale_tokens", base, out != "bf16", out != "f32") for _, _, base, out, _ in MD}
    return keys
