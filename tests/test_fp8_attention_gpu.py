"""The FP8 attention of the SAM3 ViT teacher (csrc/attention_fp8.cu, ViT.enable_fp8(attention=True)).

The kernel is checked element by element against fp64 attention on the host-dequantised Q, K and V (tests/emu_fp8_attention.py
reproduces its codes bit for bit), with NaN-prefilled outputs that must be written everywhere.  Per output element (row i, channel
d), with O the fp64 result, pi the fp64 softmax, u_j = exp(t_ij - max_j t_ij) (so max u = 1) and U = sum_j u_j:

  P rounding   e4m3(p 2^8) is p (1 + e) with |e| <= 2^-4 for codes in the normal range, and within 2^-10 (2^-18 in units of p)
               below it, so the kernel's weights are u_j + dw_j with dw_j <= max(2^-4 u_j, min(u_j, 2^-18)).  The output is the
               ratio of weighted sums, so   |dO| <= sum_j dw_j |v_jd - O_id| / (U (1 - 2^-4) - L 2^-18).  The running maxima
               of the online softmax only make the kernel's weights larger than u_j, which shrinks the subnormal term.
  S            the logits come out of the tensor core with an error of at most EPS_INNER sum_d |q_id| |k_jd| (times the softmax
               scale), plus fp32 rounding of the scales (2^-22 |t|); a logit error dt moves the output by at most
               (e^(2 dt) - 1) sum_j pi_j |v_jd - O_id|.
  PV, l        the per-tile partial products and the row sum (the 1.0 row of V^T) carry the tensor core's inner accumulation:
               EPS_INNER (sum_j pi_j |v_jd| + |O_id|) for each of the two, 2 EPS_INNER in all.
  fp32         the promotion of each key tile and the final division: (3 tiles + 8) 2^-24 (sum_j pi_j |v_jd| + |O_id|);
               the bf16 output adds half an ulp, 2^-8 of the result.
EPS_INNER = 2^-11 is the FP8 GEMM's measured constant for the tensor core's undocumented accumulation of e4m3 products
(test_fp8_gpu.py); the attention's own products are at most 128 long (64 for S).  The worst err / bound is printed; measured
on an H100 80GB HBM3 (700 W): 0.583.
"""
import math
import zlib

import pytest
import torch

from emu_fp8_attention import HEAD, dequantized, key_tile, merge_out, split_qkv
from helpers import cosine, rel_l2
from routes import fp8_attn_key

pytestmark = pytest.mark.gpu

EPS_INNER = 2.0 ** -11
U24 = 2.0 ** -24
_WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k in sorted(_WORST):
        print(f"\nfp8 attention {k}: {_WORST[k]:.3g}", end="")


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _run(cuda, qkv, B, H, W, C, heads, win, scale):
    """es3_attention_fp8 into a NaN-prefilled output; every element must be written."""
    from efficientsam3_b200 import _lib
    out = torch.full((B * H * W, C), float("nan"), device=cuda, dtype=torch.bfloat16)
    qd = qkv.to(cuda).contiguous()
    _lib.init(cuda.index or 0)
    ws = torch.full((_lib.size("es3_attention_fp8_ws_floats", B, H, W, heads, win),), float("nan"), device=cuda)
    _lib.call("es3_attention_fp8", qd.data_ptr(), out.data_ptr(), ws.data_ptr(), B, H, W, C, heads, win, float(scale),
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = out.float().cpu()
    assert not torch.isnan(got).any(), f"{int(torch.isnan(got).sum())} output elements were not written"
    return got


def _reference(q, k, v, scale, rows=1024):
    """fp64 attention and the per-element bound (module docstring) for one (image, window, head): q, k, v [L, 64] fp64."""
    L = k.shape[0]
    nt = (L + key_tile(L) - 1) // key_tile(L)
    av = v.abs()
    outs, bounds = [], []
    for r0 in range(0, q.shape[0], rows):
        t = (q[r0:r0 + rows] @ k.t()) * scale
        u = torch.exp(t - t.amax(1, keepdim=True))
        Usum = u.sum(1, keepdim=True)
        pi = u / Usum
        o = pi @ v
        ao = o.abs()
        absv = pi @ av
        dw = torch.maximum(u * 2.0 ** -4, torch.clamp(u, max=2.0 ** -18))
        term_p = (dw @ av + ao * dw.sum(1, keepdim=True)) / (Usum * (1 - 2.0 ** -4) - L * 2.0 ** -18)
        dt = scale * EPS_INNER * (q[r0:r0 + rows].abs() @ k.abs().t()).amax(1, keepdim=True) + 2.0 ** -22 * t.abs().amax(1, keepdim=True)
        term_s = torch.expm1(2 * dt) * (absv + ao)
        term_acc = (2 * EPS_INNER + (3 * nt + 8) * U24) * (absv + ao)
        b = term_p + term_s + term_acc
        outs.append(o)
        bounds.append(b + 2.0 ** -8 * (ao + b))
    return torch.cat(outs), torch.cat(bounds)


def _check(cuda, qkv, B, H, W, C, heads, win, what):
    scale = HEAD ** -0.5
    got = _run(cuda, qkv, B, H, W, C, heads, win, scale)
    qd, kd, vd = dequantized(qkv, B, H, W, C, win)
    ref = torch.zeros(qd.shape, dtype=torch.float64)
    bound = torch.zeros_like(ref)
    for b in range(qd.shape[0]):
        for w in range(qd.shape[1]):
            for h in range(qd.shape[2]):
                ref[b, w, h], bound[b, w, h] = _reference(qd[b, w, h], kd[b, w, h], vd[b, w, h], scale)
    ref, bound = merge_out(ref, B, H, W, C, win), merge_out(bound, B, H, W, C, win)
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if int(bad.sum()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} outside the bound; first at {idx}: got {got[idx].item():.6g}, "
                             f"ref {ref[idx].item():.6g}, bound {bound[idx].item():.3g}")
    _WORST["err/bound"] = max(_WORST.get("err/bound", 0.0), (err / bound).max().item())
    return got, ref


def _qkv(B, H, W, C, kind, g):
    n = B * H * W
    x = torch.randn(n, 3 * C, generator=g)
    if kind == "spread":          # per-token amax spread over 2^-8 .. 2^8, independently for q, k and v
        x = x * torch.exp2(torch.randint(-8, 9, (n, 3), generator=g).float()).repeat_interleave(C, 1)
    elif kind == "sharp":         # logits of several hundred: near one-hot P
        x[:, :2 * C] *= 6.0
    elif kind == "uniform":       # logits within +-0.05: near-uniform P
        x[:, :2 * C] *= 0.03
    if kind in ("normal", "spread"):
        x[min(3, n - 1), :HEAD] = 0.0                      # an all-zero q head of one token
        x[min(5, n - 1), C + HEAD:C + 2 * HEAD] = 0.0      # ... and of a k head
        x[min(7, n - 1), 2 * C:2 * C + HEAD] = 0.0         # ... and of a v head
    return x.to(torch.bfloat16)


CASES = [
    # B, H, W, heads, win, kind
    (2, 24, 24, 4, 24, "normal"),        # L = 576, one 24-window per image
    (1, 72, 72, 4, 24, "spread"),        # L = 576, nine windows on the teacher's 72 x 72 grid
    (1, 72, 72, 4, 24, "sharp"),
    (1, 72, 72, 4, 0, "normal"),         # L = 5184 global
    (1, 72, 72, 4, 0, "uniform"),
    (3, 40, 40, 4, 0, "spread"),         # L = 1600: a partial last key tile
    (2, 8, 8, 16, 0, "normal"),          # L = 64 < one key tile
    (1, 24, 24, 16, 12, "sharp"),        # L = 144: 128 + 16
]


@pytest.mark.parametrize("B,H,W,heads,win,kind", CASES)
def test_attention_fp8_vs_fp64(cuda, B, H, W, heads, win, kind):
    C = heads * HEAD
    qkv = _qkv(B, H, W, C, kind, _gen("attn", B, H, W, heads, win, kind))
    _check(cuda, qkv, B, H, W, C, heads, win, f"B{B} {H}x{W} heads{heads} win{win} {kind}")


def covered_keys():
    """Every route key (tests/routes.py) some row of CASES runs: both key tiles, windowed and global."""
    return {fp8_attn_key(H, W, win) for B, H, W, heads, win, kind in CASES}


def test_attention_fp8_vs_unquantised_inputs(cuda):
    """Against fp64 attention of the bf16 inputs themselves (no e4m3 round trip): whole-output rel-L2 <= 6e-2, on N(0, 1) inputs
    at the teacher's two shapes (24-windows and global on 72 x 72).  The FP8 GEMM route's rel-L2 per linear layer is of the same
    order (e4m3's 2^-4 relative rounding).  Measured on an H100 80GB HBM3 (700 W): 5.30e-2 windowed, 5.42e-2 global."""
    for win in (24, 0):
        B, H, W, heads = 1, 72, 72, 4
        C = heads * HEAD
        qkv = _qkv(B, H, W, C, "normal", _gen("raw", win))
        got = _run(cuda, qkv, B, H, W, C, heads, win, HEAD ** -0.5)
        q, k, v = (x.double() for x in split_qkv(qkv.float(), B, H, W, C, win))
        ref = torch.softmax((q @ k.transpose(-1, -2)) * HEAD ** -0.5, -1) @ v
        r = rel_l2(got, merge_out(ref, B, H, W, C, win))
        _WORST[f"rel-L2 vs bf16 inputs win={win}"] = r
        assert r <= 6e-2, r


def test_constant_v_returns_its_dequantised_value(cuda):
    """V the same for every key: every output row is V's dequantised e4m3 value, whatever P is.  When V's code is a power of two
    every PV product is an exact shift of its P code, so the PV product and the row sum (the 1.0 row of V^T) round alike in the
    tensor core and the output is exact (within 1e-6 relative).  For any other code the products carry bits below the P codes' and
    the two inner accumulations may round apart; that case is held to 2^-6 (a quarter of e4m3's own rounding).  Measured on an
    H100 80GB HBM3 (700 W): 0 for power-of-two codes, at most 6.9e-3 for the others."""
    B, H, W, heads, win = 1, 72, 72, 4, 24
    C = heads * HEAD
    g = _gen("constv")
    base = _qkv(B, H, W, C, "spread", g).float()
    sign = torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    for pow2 in (True, False):
        e = torch.randint(-6, 7, (C,), generator=g).float()
        vrow = sign * torch.exp2(e) if pow2 else torch.randn(C, generator=g) * torch.exp2(e)
        qkv = base.clone()
        qkv[:, 2 * C:] = vrow
        qkv = qkv.to(torch.bfloat16)
        for w in (win, 0):
            got = _run(cuda, qkv, B, H, W, C, heads, w, HEAD ** -0.5)
            _, _, vd = dequantized(qkv, B, H, W, C, w)
            want = merge_out(vd[..., :1, :].expand(*vd.shape[:-2], vd.shape[-2], HEAD), B, H, W, C, w)
            rel = ((got.double() - want).abs() / want.abs()).max().item()
            _WORST[f"constant V rel err pow2={pow2} win={w}"] = rel
            assert rel <= (1e-6 if pow2 else 2.0 ** -6), (pow2, w, rel)


def test_windows_are_independent_and_runs_repeat(cuda):
    B, H, W, heads, win = 2, 72, 72, 4, 24
    C = heads * HEAD
    g = _gen("indep")
    qkv = _qkv(B, H, W, C, "normal", g)
    a = _run(cuda, qkv, B, H, W, C, heads, win, 0.125)
    assert torch.equal(_run(cuda, qkv, B, H, W, C, heads, win, 0.125), a), "two runs differ"
    moved = qkv.clone().reshape(B, H, W, 3 * C)
    moved[1, 24:48, 48:72] = (torch.randn(24, 24, 3 * C, generator=g) * 3).to(torch.bfloat16)    # window (1, 2) of image 1
    b = _run(cuda, moved.reshape(-1, 3 * C), B, H, W, C, heads, win, 0.125).reshape(B, H, W, C)
    a = a.reshape(B, H, W, C)
    inside = torch.zeros(B, H, W, dtype=torch.bool)
    inside[1, 24:48, 48:72] = True
    assert torch.equal(a[~inside], b[~inside]), "a change inside one window moved another window's output"
    assert not torch.equal(a[inside], b[inside])


# ---------------------------------------------------------------------------------------------- the teacher
def _teacher(over, seed, cuda):
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    from oracle.weights import fill_state_dict
    t = SAM3ImageTeacherEncoder(embed_size=72, vit_overrides=over)
    vit = t.sam3.backbone.vision_backbone.trunk
    sd = {k: v for k, v in fill_state_dict(vit.state_dict(), seed).items() if not v.is_complex()}
    vit.load_state_dict(sd, strict=False)
    return t.to(cuda), sd


def test_fp8_attention_teacher_vs_oracle(cuda):
    """The full-width teacher geometry of test_fp8_teacher_geometry_vs_oracle (1008 px, 72 x 72 tokens, 24-windows + one global
    block, dim 1024, 16 heads, depth 3) with FP8 linears and FP8 attention, against the fp32 CPU oracle: minimum per-token cosine
    >= 0.99 and rel-L2 <= 7.5e-2.  The figures of FP8 linears alone on the same input are printed beside them."""
    from efficientsam3_b200.model.vitdet import SAM3_VIT_KWARGS
    from oracle import vitdet as O
    over = dict(depth=3, global_att_blocks=(2,))
    t, sd = _teacher(over, 35, cuda)
    x = torch.randn(1, 3, 1008, 1008, generator=_gen("teacher"))
    with torch.no_grad():
        ref = O.vit_trunk(sd, "", x, dict(SAM3_VIT_KWARGS, **over))
    lin = t.enable_fp8()(x.to(cuda)).cpu()
    out = t.enable_fp8(attention=True)(x.to(cuda)).cpu()
    tok = lambda y: y.double().flatten(2).transpose(1, 2).reshape(-1, y.shape[1])

    def stats(y):
        a, b = tok(y), tok(ref)
        cos = (a * b).sum(1) / (a.norm(dim=1) * b.norm(dim=1))
        return cos.mean().item(), cos.min().item(), rel_l2(y, ref)
    c8, cl = stats(out), stats(lin)
    print(f"\nteacher depth 3 vs oracle: fp8 attention cos mean {c8[0]:.6f} min {c8[1]:.6f} rel-L2 {c8[2]:.3e}; "
          f"fp8 linears only cos mean {cl[0]:.6f} min {cl[1]:.6f} rel-L2 {cl[2]:.3e}")
    assert out.shape == ref.shape and torch.isfinite(out).all()
    assert c8[1] >= 0.99 and c8[2] <= 7.5e-2, c8


SMALL = dict(img_size=336, depth=2, global_att_blocks=(1,))      # 24 x 24 tokens: one window and one global block


def test_switch_changes_only_attention_and_switches_back(cuda):
    from efficientsam3_b200 import ops
    t, _ = _teacher(SMALL, 7, cuda)
    t.embed_size = 24
    x = torch.randn(2, 3, 336, 336, generator=_gen("sw")).to(cuda)
    lin = t.enable_fp8()(x)
    n0 = ops.launch_count
    prof = ops.Profiler()
    ops.set_profiler(prof)
    try:
        att = t.enable_fp8(attention=True)(x)
    finally:
        ops.set_profiler(None)
    names = set(prof.summary())
    assert {"attention_fp8[L=576]"} <= names and not any(n.startswith("attention[") for n in names), names
    assert ops.launch_count > n0
    assert not torch.equal(att, lin) and cosine(att.cpu(), lin.cpu()) > 0.99
    assert torch.equal(t.enable_fp8()(x), lin), "switching FP8 attention off must reproduce enable_fp8() bit for bit"
    assert torch.equal(t.enable_fp8(attention=True)(x), att)
    with ops.strict_precision():
        a = t.enable_fp8(False)(x)
        b = t.enable_fp8(attention=True)(x)
    assert torch.equal(a, b), "the strict precision mode ignores the switch"


def test_online_kd_step_with_fp8_attention(cuda):
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.losses import kd_train_step_online
    from efficientsam3_b200.stage1.model import build_image_student_model
    from efficientsam3_b200.stage1.optim import FlatAdamW
    t, _ = _teacher(dict(depth=2, global_att_blocks=(1,)), 11, cuda)
    t.enable_fp8(attention=True)
    cfg = NS(MODEL=NS(BACKBONE="efficientvit_b1"), DATA=NS(IMG_SIZE=1008), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=72))
    m = build_image_student_model(cfg).to(cuda).train()
    opt = FlatAdamW(m, lr=1e-4, weight_decay=0.01)
    x = torch.randn(2, 3, 1008, 1008, generator=_gen("kd")).to(cuda)
    emb = t(x)
    assert emb.shape == (2, 1024, 72, 72) and emb.dtype == torch.float32 and torch.isfinite(emb).all()
    sizes = [(3, 1008, 756), (3, 672, 1008)]
    losses = [float(kd_train_step_online(m, t, opt, x, sizes, 1.0, 5.0).item()) for _ in range(2)]
    assert all(math.isfinite(v) for v in losses), losses
