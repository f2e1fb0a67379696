"""fp64 statements of the SAM heads' kernels (decoder.cu: the prompt encoder's positional encodings and mask downscaling, the two-way
transformer's few-query and few-key attention, the upscaling LayerNorm + GELU, the hypernetwork masks, the bilinear resize; and the
strict-mode twins of strict_f32.cu) and, next to each, the per-element bound its fp32 arithmetic keeps to.

The bound form is ref_fwd.py's and ref_text.py's: an fp32 sum of n terms is held to GAMMA n u sum |terms|, an fp32 result adds 4u |ref|
and a bf16 result 2^-8 |ref| for its own rounding (_out).  Operands are the ones the kernel reads (the fp32 coordinates and Gaussian
matrix, bf16 or fp32 keys and values).  Every function takes and returns float64 tensors (CPU or CUDA).  tests/test_sam_kernels_cpu.py
ties each statement to textbook float64 torch and to oracle/sam_heads.py.
"""
import math

import torch
import torch.nn.functional as F

from bounds import U
from ref_fwd import _act_err, layernorm
from ref_text import EXPF_REL
from ref_train_bwd import GAMMA, _out

SINCOS_REL = 4 * U             # sincosf (no fast math): 2 ulp of each result (CUDA C++ Programming Guide, single-precision functions)
LN_EPS = 1e-6                  # LayerNorm2d of the SAM heads (sam/common.py)


def expf_fast_rel(arg):
    """Relative error of __expf(a) for a fp32 argument a: (2 + 1.16 |a|) ulp (ex2.approx of a log2 e; see ref_fwd.EX2_REL)."""
    return 2 * U * (2 + 1.16 * arg.abs())


# ------------------------------------------------------------------------------------------------ positional encodings
def pe(gauss, x01, y01, e01=None):
    """PositionEmbeddingRandom: c = 2 (x01, y01) - 1, a = 2 pi (cx g0 + cy g1), [sin a | cos a].  gauss [2, F]; x01, y01 [...].
    The kernel's x01 = fl(fl(x + 0.5) / W) is within e01 (default 2u |x01|) of exact; c = fl(2 x01 - 1) adds u |c|, the two-term
    dot product 2u sum |terms|, fl(2 pi) and the product u |a| each; sin and cos are 1-Lipschitz and sincosf adds 2 ulp.
    Returns (ref [..., 2F], inner bound [..., 2F] without the output's own rounding)."""
    if e01 is None:
        e01 = (2 * U * x01.abs(), 2 * U * y01.abs())
    cx, cy = 2 * x01 - 1, 2 * y01 - 1
    ecx, ecy = 2 * e01[0] + U * cx.abs(), 2 * e01[1] + U * cy.abs()
    g0, g1 = gauss[0], gauss[1]
    dot = cx[..., None] * g0 + cy[..., None] * g1
    e_dot = ecx[..., None] * g0.abs() + ecy[..., None] * g1.abs() + GAMMA * 2 * U * (cx[..., None].abs() * g0.abs() + cy[..., None].abs() * g1.abs())
    a = 2 * math.pi * dot
    e_a = 2 * math.pi * e_dot + 3 * U * a.abs()
    s, c = torch.sin(a), torch.cos(a)
    ref = torch.cat([s, c], -1)
    return ref, torch.cat([e_a, e_a], -1) + SINCOS_REL * ref.abs()


def dense_pe(gauss, h, w):
    """es3_dense_pe: [h w, 2F] token-major, pixel centres (x + 0.5) / w, (y + 0.5) / h.  fp32 store."""
    ys = (torch.arange(h, dtype=gauss.dtype, device=gauss.device) + 0.5) / h
    xs = (torch.arange(w, dtype=gauss.dtype, device=gauss.device) + 0.5) / w
    ref, e = pe(gauss, xs[None, :].expand(h, w).reshape(-1), ys[:, None].expand(h, w).reshape(-1))
    return ref, _out(ref, e, False)


def point_embed(coords, labels, gauss, not_a_point, point_emb, img_w, img_h, pad):
    """es3_point_embed on coords [B, P, 2] (x, y pixels, fp32 values), labels [B, P]: pe of ((x + 0.5) / W, (y + 0.5) / H); label -1
    takes not_a_point exactly, labels 0..3 add their row of point_emb [4, 2F] (one fp32 rounding), any other label leaves the pe as
    it is; pad appends a label -1 point.  Returns (ref, bound, exact) [B, P + pad, 2F]: exact marks the cells that are a copy."""
    B, P = labels.shape
    x01, y01 = (coords[..., 0] + 0.5) / img_w, (coords[..., 1] + 0.5) / img_h
    # fl(x + 0.5) and the division: 2u |x01| (x + 0.5 may round where |x| >= 2^23; the coordinates here are far below)
    ref, e = pe(gauss, x01, y01)
    lab = labels.to(torch.long)
    add = torch.zeros_like(ref)
    known = (lab >= 0) & (lab < 4)
    add[known] = point_emb[lab[known]]
    ref = ref + add
    e = e + known[..., None] * U * ref.abs()
    nap = (lab == -1)[..., None]
    ref = torch.where(nap, not_a_point.expand_as(ref), ref)
    e = torch.where(nap, torch.zeros_like(e), e)
    exact = nap.expand_as(ref)
    if pad:
        row = not_a_point.expand(B, 1, -1)
        ref = torch.cat([ref, row], 1)
        e = torch.cat([e, torch.zeros_like(row)], 1)
        exact = torch.cat([exact, torch.ones_like(row, dtype=torch.bool)], 1)
    return ref, _out(ref, e, False), exact


# ------------------------------------------------------------------------------------------------ attention
def _softmax_weighted(s, e_s, v, exp_rel, n_resc, resc_rel, n_sum, n_out):
    """y = softmax(s) v from fp32 scores within e_s of s [..., N, Tk], v [..., Tk, d].  exp_rel(arg): the relative error of one
    exponential; each weight is further multiplied by up to n_resc rescale factors, each within resc_rel (its exponential, its
    argument and the product); l is a sum of Tk terms held to GAMMA n_sum u, each output a sum held to GAMMA n_out u.  The division
    rounds the reciprocal and the product (2u).  Returns (y, bound on |y32 - y| before the output's own rounding)."""
    mx = s.amax(-1, keepdim=True)
    arg = s - mx
    p = torch.exp(arg)
    delta = e_s + e_s.amax(-1, keepdim=True) + U * arg.abs() + exp_rel(arg) + n_resc * resc_rel
    l = p.sum(-1, keepdim=True)
    rel_l = (p * delta).sum(-1, keepdim=True) / l + GAMMA * n_sum * U
    o = p @ v
    e_o = (p * delta) @ v.abs() + GAMMA * n_out * U * (p @ v.abs())
    y = o / l
    return y, e_o / l + y.abs() * (rel_l + 2 * U) + U * y.abs()


def _resc_rel(s):
    """Relative error of one online-softmax rescale factor __expf(m_old - m_new) and its product: |m_old - m_new| <= the row's
    score range A."""
    A = (s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True))
    return expf_fast_rel(A) + U * A + 2 * U


def attn_few_queries(q, k, v, heads, scale):
    """es3_attn_few_queries: q [B, Tq, D] fp32, k, v [B, Tk, D] (the values the kernel reads, bf16 or fp32) -> [B, Tq, D] fp32.
    One warp per query: qs = fl(q scale), lane j takes keys j, j + 32, ... with its own online softmax (__expf, up to ceil(Tk/32)
    terms and rescales), then the 32 states merge by butterfly: each lane's state is scaled once more by __expf(m - m_w), and l and
    P V are 32-way tree sums (5 levels)."""
    B, Tq, D = q.shape
    Tk, hd = k.shape[1], D // heads
    qh = q.reshape(B, Tq, heads, hd).transpose(1, 2)
    kh, vh = (t.reshape(B, Tk, heads, hd).transpose(1, 2) for t in (k, v))
    s = scale * qh @ kh.transpose(-1, -2)
    e_s = abs(scale) * (GAMMA * (hd + 1) * U) * (qh.abs() @ kh.abs().transpose(-1, -2))
    nl = -(-Tk // 32)
    y, e = _softmax_weighted(s, e_s, vh, expf_fast_rel, nl, _resc_rel(s), nl + 6, nl + 6)
    y, e = (t.transpose(1, 2).reshape(B, Tq, D) for t in (y, e))
    return y, _out(y, e, False)


def attn_few_keys(q, k, v, heads, scale, strict):
    """es3_attn_few_keys (strict = False): q [B, Nq, D] bf16 values, k, v [B, Tk, D] fp32 -> bf16: one thread per (query, head),
    qs = fl(q scale), a sequential online softmax over the Tk keys (__expf, one rescale per key).
    es3_attn_few_keys_f32 (strict = True): fp32 q; s = fl(fl(q . k) scale), the two-pass softmax with libm expf, w = fl(p fl(1 / l)),
    o = an fmaf chain of Tk terms of w v.  fp32 store."""
    B, Nq, D = q.shape
    Tk, hd = k.shape[1], D // heads
    qh = q.reshape(B, Nq, heads, hd).transpose(1, 2)
    kh, vh = (t.reshape(B, Tk, heads, hd).transpose(1, 2) for t in (k, v))
    s = scale * qh @ kh.transpose(-1, -2)
    e_s = abs(scale) * (GAMMA * (hd + 1) * U) * (qh.abs() @ kh.abs().transpose(-1, -2))
    if strict:
        y, e = _softmax_weighted(s, e_s, vh, lambda a: EXPF_REL + 0 * a, 1, 2 * U, Tk, Tk + 1)
    else:
        y, e = _softmax_weighted(s, e_s, vh, expf_fast_rel, Tk, _resc_rel(s), Tk + 1, Tk + 1)
    y, e = (t.transpose(1, 2).reshape(B, Nq, D) for t in (y, e))
    return y, _out(y, e, not strict)


def _sdpa(q, k, v, heads, scale):
    """Textbook multi-head softmax attention (for the CPU tests)."""
    B, N, D = q.shape
    Tk, hd = k.shape[1], D // heads
    qh = q.reshape(B, N, heads, hd).transpose(1, 2)
    kh, vh = (t.reshape(B, Tk, heads, hd).transpose(1, 2) for t in (k, v))
    return F.scaled_dot_product_attention(qh, kh, vh, scale=scale).transpose(1, 2).reshape(B, N, D)


# ------------------------------------------------------------------------------------------------ LayerNorm + GELU
def ln_rows_gelu(x, w, b, eps, strict):
    """es3_ln_rows_gelu (bf16 store, es3_gelu_fast) / es3_ln_rows_gelu_f32 (fp32 store, erf GELU) over rows x [M, C]: ref_fwd.layernorm
    (mean = fl(sum) / C, rstd within 4u -- rsqrtf, or 1 / sqrtf with two correct roundings -- and fmaf(xh, w, b)), then GELU with
    the EPS_GELU charge, which covers es3_gelu_fast's A&S erf and MUFU and erff's 2 ulp alike."""
    pre, e_pre = layernorm(x, w, b, eps, bf16=False)
    ref, e = _act_err(pre, e_pre, "gelu")
    return ref, _out(ref, e, not strict)


# ------------------------------------------------------------------------------------------------ mask tail
def hyper_masks(up, hyper, obj, no_obj, K, k_off):
    """es3_hyper_masks: masks[b, k, p] = sum_c hyper[b, k_off + k, c] up[b, p, c], a 32-term fmaf chain; where obj is given and
    !(obj[b] > 0) (0, -0 and NaN included) the image's masks are exactly no_obj.  Returns (ref, bound, gated [B, 1, 1])."""
    h = hyper[:, k_off:k_off + K]
    ref = h @ up.transpose(1, 2)
    e = GAMMA * 32 * U * (h.abs() @ up.abs().transpose(1, 2))
    gated = torch.zeros(up.shape[0], 1, 1, dtype=torch.bool, device=up.device)
    if obj is not None:
        gated = ~(obj > 0).reshape(-1, 1, 1)
    ref = torch.where(gated, torch.full_like(ref, no_obj), ref)
    return ref, torch.where(gated, torch.zeros_like(e), _out(ref, e, False)), gated


def _src_coord(n_out, n_in, dtype, device):
    """(exact source coordinate, clamped at 0; its floor index; the bound on the kernel's fp32 coordinate error):
    f = fl(fl(o + 0.5) sy) - 0.5, sy = fl(n_in / n_out): sy and the product are each within u, the subtraction u |f|."""
    o = torch.arange(n_out, dtype=dtype, device=device) + 0.5
    f = (o * (n_in / n_out) - 0.5).clamp_min(0)
    e = 3 * U * o * (n_in / n_out) + U * f
    return f, f.floor().long().clamp_max(n_in - 1), e


def bilinear(x, Ho, Wo):
    """es3_bilinear_nchw_f32: F.interpolate(x [P, Hi, Wi], (Ho, Wo), bilinear, align_corners=False).  The kernel's source
    coordinates are within e_f of exact; bilinear interpolation is continuous and piecewise linear, so a coordinate error moves the
    value by at most e_f times the largest slope next to the sample (the adjacent-pixel differences over a 3 x 3 window, which
    covers a floor that flips), and the lerp weights (1 - l rounds) and the two-level lerp add GAMMA 8 u of the largest tap."""
    P, Hi, Wi = x.shape
    ref = F.interpolate(x[:, None], size=(Ho, Wo), mode="bilinear", align_corners=False)[:, 0]
    fy, y0, ey = _src_coord(Ho, Hi, x.dtype, x.device)
    fx, x0, ex = _src_coord(Wo, Wi, x.dtype, x.device)
    y1, x1 = (y0 + 1).clamp_max(Hi - 1), (x0 + 1).clamp_max(Wi - 1)
    mp = lambda t: F.max_pool2d(t[:, None], 3, 1, 1)[:, 0]
    dy = mp(F.pad((x[:, 1:] - x[:, :-1]).abs(), (0, 0, 0, 1)))
    dx = mp(F.pad((x[:, :, 1:] - x[:, :, :-1]).abs(), (0, 1)))
    ax = mp(x.abs())
    g = lambda t, yy, xx: t[:, yy][:, :, xx]
    sy = torch.maximum(g(dy, y0, x0), g(dy, y0, x1))
    sx = torch.maximum(g(dx, y0, x0), g(dx, y1, x0))
    amax = torch.maximum(g(ax, y0, x0), g(ax, y1, x1))
    e = ey[:, None] * sy + ex[None, :] * sx + GAMMA * 8 * U * amax
    return ref, _out(ref, e, False)


# ------------------------------------------------------------------------------------------------ mask prompt
def _ln_gelu_ch(t, e_t, g, b, eps):
    """LayerNorm over the channel axis 1 of t [N, C, ...] (mu = fl(sum) / C, rsqrtf), then erf GELU; t known to within e_t.
    ref_fwd.layernorm's charges scale with gamma rstd, so a flat patch (rstd up to 1 / sqrt(eps)) carries them amplified."""
    C = t.shape[1]
    tm = t.movedim(1, -1).reshape(-1, C)
    pre, e_pre = layernorm(tm, g, b, eps, bf16=False, e_x=e_t.movedim(1, -1).reshape(-1, C))
    ref, e = _act_err(pre, e_pre, "gelu")
    shape = t.movedim(1, -1).shape
    return ref.reshape(shape).movedim(-1, 1), e.reshape(shape).movedim(-1, 1)


def mask_downscale(mask, wts, eps, base=None):
    """es3_mask_downscale_tokens: conv2x2 s2 (1 -> 4, an fmaf chain of 4 from the bias) -> LN(4) -> erf GELU -> conv2x2 s2 (4 -> 16,
    16 terms from the bias) -> LN(16) -> erf GELU -> 1x1 conv (16 -> C, 16 terms from the bias) [+ base[row % base_rows], one
    rounding], token-major [B h w, C].  mask [B, 1, 4h, 4w]; wts = (w0, b0, g1, be1, w1, b1, g2, be2, w2, b2) as the kernel reads
    them.  Each stage's error goes on through the absolute weights of the next.  Returns (ref, bound) of the fp32 store."""
    w0, b0, g1, be1, w1, b1, g2, be2, w2, b2 = wts
    t = F.conv2d(mask, w0.reshape(4, 1, 2, 2), b0, stride=2)
    e_t = GAMMA * 5 * U * (F.conv2d(mask.abs(), w0.abs().reshape(4, 1, 2, 2), b0.abs(), stride=2))
    a, e_a = _ln_gelu_ch(t, e_t, g1, be1, eps)
    W1 = w1.reshape(16, 4, 2, 2)
    u = F.conv2d(a, W1, b1, stride=2)
    e_u = GAMMA * 17 * U * F.conv2d(a.abs(), W1.abs(), b1.abs(), stride=2) + F.conv2d(e_a, W1.abs(), stride=2)
    s, e_s = _ln_gelu_ch(u, e_u, g2, be2, eps)
    B, _, h, w = s.shape
    s, e_s = (z.permute(0, 2, 3, 1).reshape(B * h * w, 16) for z in (s, e_s))
    W2 = w2.reshape(-1, 16)
    ref = s @ W2.t() + b2
    e = GAMMA * 17 * U * (s.abs() @ W2.abs().t() + b2.abs()) + e_s @ W2.abs().t()
    if base is not None:
        ref = ref + base[torch.arange(ref.shape[0], device=ref.device) % base.shape[0]]
        e = e + U * ref.abs()
    return ref, _out(ref, e, False)
