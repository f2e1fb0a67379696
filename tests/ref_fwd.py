"""fp64 statements of the image students' forward kernels and, next to each, the per-element bound its fp32 arithmetic keeps to.

Operands are the ones the kernel receives: bf16-representable activations, bf16 pointwise weights, the bf16 depthwise taps of
es3_round_taps_sum_bf16 where the kernel multiplies bf16 taps, fp32 scales and biases.  The bound form is ref_train_bwd.py's: an
fp32 sum of n terms is held to GAMMA n u sum |terms|, an fp32 result adds 4u |ref| and a bf16 result 2^-8 |ref| for its own
rounding; activations add L_ACT (u |pre| + EPS_GELU |pre|) and 2u |act| (the hswish form x sat(x / 6 + 1/2) rounds twice).

Intermediates the fused kernels round to bf16 (MBConv's expand output e and depthwise output d, dsconv_res's mid, window
attention's P) are rounded here at the same point, and charged only where that rounding is ambiguous (band()): the kernel's fp32
value v32 lies within its own bound delta of the fp64 value v, so rn(v32) can differ from rn(v) only where v lies within delta of
a bf16 rounding midpoint, and then by one bf16 step.  Those elements carry the step to the output to first order, through the
absolute values of the downstream weights; everywhere else the output bound stays at the level of the output rounding.

Every function takes and returns float64 tensors (CPU or CUDA) in NHWC unless stated.  tests/test_fwd_kernels_cpu.py ties each
statement to F.conv2d / F.hardswish / textbook attention in float64.
"""
import torch
import torch.nn.functional as F

from bounds import L_ACT, U, _act64, _eps_act
from ref_train_bwd import GAMMA, _out

KV_SPLIT = 2.0 ** -16          # litemla_apply_tc: KV = hi + lo + r, hi = bf16(KV), lo = bf16(KV - hi); |KV - hi| <= 2^-8 |KV| and
#                                the rounding of lo is within 2^-8 |KV - hi|, so |r| <= 2^-16 |KV| (the subtraction is exact)


# ------------------------------------------------------------------------------------------------ bf16 rounding
def rn_bf16(v):
    """Round-to-nearest-even of fp64 values to bf16, directly (no double rounding through fp32); normal range."""
    m, e = torch.frexp(v)                              # v = m 2^e, |m| in [0.5, 1): a bf16 step at v is 2^(e - 8)
    step = torch.ldexp(torch.ones_like(v), (e - 8).clamp_min(-133))
    return torch.where(v == 0, v, torch.round(v / step) * step)


def band(v, delta):
    """(rn(v), dev): the bf16 value the reference takes, and the most the kernel's bf16 value rn(v32), |v32 - v| <= delta, can
    differ from it -- rn is monotone, so the extremes are rn(v -+ delta); dev is one step where v lies within delta of a
    rounding midpoint and exactly 0 elsewhere."""
    r = rn_bf16(v)
    return r, torch.maximum((rn_bf16(v - delta) - r).abs(), (rn_bf16(v + delta) - r).abs())


def _act_err(pre, e_pre, act):
    """(act(pre), bound on |act(pre32) - act(pre)|) for a pre-activation known to within e_pre (which includes its own rounding)."""
    ref = _act64(pre, act)
    return ref, L_ACT[act] * (e_pre + _eps_act(pre, act)) + 2 * U * ref.abs()


# ------------------------------------------------------------------------------------------------ convolutions
def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def dw(x, w, ks, stride):
    """Depthwise ks x ks, pad ks // 2: x [B, H, W, C], w [ks*ks, C] tap-major -> [B, Ho, Wo, C] (no bias)."""
    C = x.shape[3]
    return _nhwc(F.conv2d(_nchw(x), w.t().reshape(C, 1, ks, ks), stride=stride, padding=ks // 2, groups=C))


def dwconv(x, w, bias, ks, stride, act):
    """act(dw(x; w) + bias), bf16 store: es3_dwconv_bf16 / _tiled_bf16 (fp32 FMA chain from the bias) and es3_dwconv_tc_bf16 (MMA,
    then + bias); w as the kernel multiplies it (fp32, or the bf16 taps of round_taps_sum for the tensor-core kernel)."""
    b = bias if bias is not None else torch.zeros_like(w[0])
    pre = dw(x, w, ks, stride) + b
    e_pre = GAMMA * (ks * ks + 1) * U * (dw(x.abs(), w.abs(), ks, stride) + b.abs()) + U * pre.abs()
    ref, e = _act_err(pre, e_pre, act)
    return ref, _out(ref, e, True)


def pw(a, w):
    """(a w^T, |a| |w|^T) over the channel axis: a [..., K], w [N, K]."""
    return a @ w.t(), a.abs() @ w.abs().t()


def mbconv(x, w1, s1, b1, wdw, b2, w3, s3, b3, stride, residual, act="hswish"):
    """The fused MBConv block y = [x +] s3 pw(d; w3) + b3, d = bf16(act(dw3x3_s(e; wdw) + b2)), e = bf16(act(s1 pw(x; w1) + b1)),
    e zero outside the image (the depthwise's padding).  wdw: the bf16 taps.  Returns (ref, bound, dev_e, dev_d) -- the last two
    are the band() charges of the rounded intermediates (for the tie-band tests)."""
    K = x.shape[3]
    a1, t1 = pw(x, w1)
    pre1 = s1 * a1 + b1
    e64, de = _act_err(pre1, s1.abs() * GAMMA * K * U * t1 + U * pre1.abs(), act)
    e, dev_e = band(e64, de)
    ref, bound, dev_d = dwproj(e, wdw, b2, w3, s3, b3, x if residual else None, act, dev_in=dev_e, stride=stride, full=True)
    return ref, bound, dev_e, dev_d


def dwproj(mid, wdw, b2, w3, s3, b3, residual=None, act="hswish", dev_in=None, stride=1, full=False):
    """es3_dwproj_tc_bf16: y = s3 pw(d; w3) + b3 [+ residual], d = bf16(act(dw3x3(mid; wdw) + b2)); wdw the bf16 taps.  dev_in: the
    band charge of mid when it is itself a rounded intermediate (mbconv)."""
    pre2 = dw(mid, wdw, 3, stride) + b2
    e_pre2 = GAMMA * 9 * U * dw(mid.abs(), wdw.abs(), 3, stride) + U * pre2.abs()
    if dev_in is not None:
        e_pre2 = e_pre2 + dw(dev_in, wdw.abs(), 3, stride)
    d64, dd = _act_err(pre2, e_pre2, act)
    d, dev_d = band(d64, dd)
    a3, t3 = pw(d, w3)
    ref = s3 * a3 + b3
    e = s3.abs() * (GAMMA * w3.shape[1] * U * t3 + dev_d @ w3.abs().t()) + U * ref.abs()
    if residual is not None:
        ref = ref + residual
        e = e + U * ref.abs()
    out = (ref, _out(ref, e, True))
    return out + (dev_d,) if full else out


def stem_conv(img, w27, bias, act):
    """es3_stem_conv3x3_s2: act(conv3x3_s2_p1(img) + bias), img [B, 3, H, W] fp32 NCHW, w27 [27, Cout] (ci*9 + ky*3 + kx), bf16
    NHWC store; an fp32 FMA chain of 27 terms from the bias."""
    Cout = w27.shape[1]
    wt = w27.t().reshape(Cout, 3, 3, 3)
    b = bias if bias is not None else torch.zeros(Cout, dtype=img.dtype, device=img.device)
    pre = _nhwc(F.conv2d(img, wt, stride=2, padding=1)) + b
    terms = _nhwc(F.conv2d(img.abs(), wt.abs(), stride=2, padding=1)) + b.abs()
    ref, e = _act_err(pre, GAMMA * 28 * U * terms + U * pre.abs(), act)
    return ref, _out(ref, e, True)


def dsconv_res(x, wdw, bdw, wpw, bpw, act):
    """es3_dsconv_res_bf16: y = x + pw(mid; wpw) + bpw, mid = bf16(act(dw3x3(x; wdw) + bdw)); wdw, wpw fp32 ([9, C], [C, C])."""
    C = x.shape[3]
    bd = bdw if bdw is not None else torch.zeros(C, dtype=x.dtype, device=x.device)
    bp = bpw if bpw is not None else torch.zeros(C, dtype=x.dtype, device=x.device)
    pre = dw(x, wdw, 3, 1) + bd
    m64, dm = _act_err(pre, GAMMA * 10 * U * (dw(x.abs(), wdw.abs(), 3, 1) + bd.abs()) + U * pre.abs(), act)
    mid, dev = band(m64, dm)
    a, t = pw(mid, wpw)
    ref = a + bp + x
    e = GAMMA * (C + 1) * U * (t + bp.abs()) + dev @ wpw.abs().t() + U * ref.abs()
    return ref, _out(ref, e, True)


def stem_fused(img, w0, s0, b0, wdw, bdw, wpw, spw, bpw):
    """es3_stem_fused_c16 on the bf16-rounded image (its MMA operand): x1 = bf16(hswish(s0 conv3x3_s2(img; w0[:, :27]) + b0)),
    y = x1 + spw pw(d; wpw) + bpw, d = bf16(hswish(dw3x3(x1; wdw) + bdw)); wdw the bf16 taps.  x1 enters both the depthwise and
    the residual, so its band charge is carried by both."""
    wt = w0[:, :27].reshape(16, 3, 3, 3)
    acc = _nhwc(F.conv2d(img, wt, stride=2, padding=1))
    terms = _nhwc(F.conv2d(img.abs(), wt.abs(), stride=2, padding=1))
    pre = s0 * acc + b0
    x64, dx = _act_err(pre, s0.abs() * GAMMA * 32 * U * terms + U * pre.abs(), "hswish")
    x1, dev = band(x64, dx)
    ref, bound = dwproj(x1, wdw, bdw, wpw, spw, bpw, x1, "hswish", dev_in=dev)
    return ref, bound + dev * (1 + 2.0 ** -8)


def conv3x3_s2_narrow(x, w9, scale, bias, act):
    """es3_conv3x3_s2_narrow_bf16: act(scale conv3x3_s2_p1(x) + bias), w9 [9, Cout, Cin] (tap = ky*3 + kx), bf16 store."""
    Cout, Cin = w9.shape[1], w9.shape[2]
    wt = w9.permute(1, 2, 0).reshape(Cout, Cin, 3, 3)
    acc = _nhwc(F.conv2d(_nchw(x), wt, stride=2, padding=1))
    terms = _nhwc(F.conv2d(_nchw(x.abs()), wt.abs(), stride=2, padding=1))
    pre = scale * acc + bias
    ref, e = _act_err(pre, scale.abs() * GAMMA * 9 * Cin * U * terms + U * pre.abs(), act)
    return ref, _out(ref, e, True)


# ------------------------------------------------------------------------------------------------ LiteMLA
def litemla_attn(ms, heads2, dim, eps, chunk, split):
    """ReLU linear attention over ms [B, HW, >= heads2 3 dim] (head h = q | k | v at [3 dim h, 3 dim (h + 1))):
    KV[d][j] = sum_p v[p, d] relu(k[p, j]) (row dim: sum_p relu(k[p, j])), summed per chunk of `chunk` pixels into the partials
    [B, heads2, nchunk, dim + 1, dim], then over the chunks; o = KV relu(q), y = o[:dim] / (o[dim] + eps), bf16 store.
    split: the tensor-core apply's hi + lo bf16 KV (KV_SPLIT, two MMAs of dim terms).
    Returns ((y, bound) [B, HW, heads2 dim], (partials, bound))."""
    B, HW = ms.shape[:2]
    t = ms[..., :heads2 * 3 * dim].reshape(B, HW, heads2, 3, dim)
    qr, kr, v = t[:, :, :, 0].clamp_min(0), t[:, :, :, 1].clamp_min(0), t[:, :, :, 2]
    vp = torch.cat([v, torch.ones_like(v[..., :1])], -1)                       # [B, HW, h, dim + 1]
    nch = (HW + chunk - 1) // chunk
    pad = nch * chunk - HW
    vc = F.pad(vp, (0, 0, 0, 0, 0, pad)).reshape(B, nch, chunk, heads2, dim + 1)
    kc = F.pad(kr, (0, 0, 0, 0, 0, pad)).reshape(B, nch, chunk, heads2, dim)
    part = torch.einsum("bcphi,bcphj->bhcij", vc, kc)
    e_part = GAMMA * chunk * U * torch.einsum("bcphi,bcphj->bhcij", vc.abs(), kc) + 4 * U * part.abs()
    KV = part.sum(2)
    aKV = torch.einsum("bcphi,bcphj->bhij", vc.abs(), kc)
    e_KV = GAMMA * (HW + nch) * U * aKV
    n_apply = dim
    if split:
        e_KV = e_KV + KV_SPLIT * KV.abs()
        n_apply = 2 * dim
    o = torch.einsum("bhij,bphj->bphi", KV, qr)                                # [B, HW, h, dim + 1]
    e_o = torch.einsum("bhij,bphj->bphi", e_KV + GAMMA * n_apply * U * KV.abs(), qr)
    den = o[..., dim] + eps
    e_den = e_o[..., dim] + U * den.abs()
    r = 1.0 / den
    e_r = r * r * e_den + U * r.abs()
    y = o[..., :dim] * r[..., None]
    e_y = o[..., :dim].abs() * e_r[..., None] + r.abs()[..., None] * e_o[..., :dim] + U * y.abs()
    y, e_y = y.reshape(B, HW, heads2 * dim), e_y.reshape(B, HW, heads2 * dim)
    return (y, _out(y, e_y, True)), (part, _out(part, e_part, False))


def litemla_aggreg(ms, wdw, wpw, C3):
    """es3_litemla_aggreg_dwpw: a = bf16(dw5x5(ms[..., :C3]; wdw)), then per group of 16 channels out[c] = sum_j wpw[c, j]
    a[16 (c // 16) + j], bf16 store into channels [C3, 2 C3).  wdw [25, C3] (bf16 taps), wpw [C3, 16] bf16.  Returns (ref, bound)."""
    x = ms[..., :C3]
    a64 = dw(x, wdw, 5, 1)
    a, dev = band(a64, GAMMA * 25 * U * dw(x.abs(), wdw.abs(), 5, 1) + U * a64.abs())
    B, H, W, _ = x.shape
    G = C3 // 16
    ag, dg = a.reshape(B, H, W, G, 16), dev.reshape(B, H, W, G, 16)
    wg = wpw.reshape(G, 16, 16)                                                 # [group, out j, in i]
    ref = torch.einsum("bhwgi,goi->bhwgo", ag, wg).reshape(B, H, W, C3)
    e = (GAMMA * 16 * U * torch.einsum("bhwgi,goi->bhwgo", ag.abs(), wg.abs()) + torch.einsum("bhwgi,goi->bhwgo", dg, wg.abs())
         ).reshape(B, H, W, C3) + U * ref.abs()
    return ref, _out(ref, e, True)


# ------------------------------------------------------------------------------------------------ RepViT / TinyViT pieces
def channel_mean(x, chunk=128):
    """es3_channel_mean: x [B, HW, C] -> [B, C] fp32, partial sums per chunk of 128 pixels, then over the chunks, times fl(1 / HW)."""
    HW = x.shape[1]
    ref = x.mean(1)
    nch = (HW + chunk - 1) // chunk
    e = GAMMA * (HW + nch) * U * x.abs().sum(1) / HW + 2 * U * ref.abs()
    return ref, _out(ref, e, False)


def scale_channels(x, gate):
    """es3_scale_channels: y[b, p, c] = x[b, p, c] gate[b, c], one fp32 product, bf16 store."""
    ref = x * gate[:, None, :]
    return ref, _out(ref, U * ref.abs(), True)


def layernorm(x, gamma, beta, eps, bf16=True, e_x=None):
    """es3_layernorm_bf16 over rows x [M, C]: mean = fl(sum) / C, q = sum (x - mean)^2, rstd = rsqrtf(q / C + eps) (2 ulp),
    y = fmaf((x - mean) rstd, gamma, beta), bf16 store; bf16 = False: the fp32 store of es3_layernorm_f32 (which multiplies by
    fl(1 / C): one more rounding of the mean).  e_x: a per-element error already in the kernel's x (the rounding of its pos add)."""
    C = x.shape[1]
    mu = x.mean(1, keepdim=True)
    e_mu = GAMMA * C * U * x.abs().mean(1, keepdim=True) + (U if bf16 else 2 * U) * mu.abs()
    if e_x is not None:
        e_mu = e_mu + e_x.mean(1, keepdim=True)
    d = x - mu
    e_d = e_mu + U * d.abs() + (0.0 if e_x is None else e_x)
    q = (d * d).sum(1, keepdim=True)
    e_q = (2 * d.abs() * e_d).sum(1, keepdim=True) + GAMMA * (C + 1) * U * q
    var = q / C + eps
    e_var = e_q / C + 2 * U * var
    rstd = var.rsqrt()
    e_rstd = 0.5 * rstd ** 3 * e_var + 4 * U * rstd
    xh = d * rstd
    e_xh = d.abs() * e_rstd + rstd * e_d + U * xh.abs()
    ref = xh * gamma + beta
    return ref, _out(ref, gamma.abs() * e_xh + U * ref.abs(), bf16)


def win_tokens(B, H, W, ws):
    """Window-raster token index [B nWin, ws^2] of the zero-padded map (-1: a padded position)."""
    nH, nW = -(-H // ws), -(-W // ws)
    yy = torch.arange(nH * ws)[:, None].expand(-1, nW * ws)
    xx = torch.arange(nW * ws)[None, :].expand(nH * ws, -1)
    idx = torch.where((yy < H) & (xx < W), yy * W + xx, torch.full_like(yy, -1))
    idx = idx.reshape(nH, ws, nW, ws).permute(0, 2, 1, 3).reshape(nH * nW, ws * ws)
    off = torch.arange(B)[:, None, None] * (H * W)
    return torch.where(idx[None] >= 0, idx[None] + off, torch.full_like(idx[None], -1)).reshape(B * nH * nW, ws * ws)


EX2_REL = 4 * U                 # ex2.approx.ftz.f32: 2 ulp of the result (CUDA C++ Programming Guide, intrinsic functions: exp2f's
#                                ex2.approx path; __expf = ex2.approx(x log2 e) is listed at 2 + floor(1.173 |x|) ulp, the |x| part
#                                being the product's rounding); an ulp is 2^-23 relative, i.e. 2u


def softmax_attn(q, k, v, scale, bias=None, causal=False, ex2=False, kv_tile=None):
    """Flash-style softmax attention over q [..., N, d], k, v [..., Nk, d] (heads in the leading axes): s = scale q k^T (+ bias)
    (+ -inf above the diagonal when causal), p = exp(s - rowmax) in fp32, P = bf16(p) into PV, l = sum of the fp32 p,
    y = (P v) / l.  Returns (y, bound on |y32 - y| before the output's own rounding).

    ex2 = False: p = __expf(fl(scale s32) + bias - m) (the window-attention kernels).  ex2 = True: the exponent is ex2.approx of an
    fp32 argument in log2 units -- fl(fl(s32 c) - m) with c = fl(scale log2 e) (attn_fwd_kernel, mma.sync) or fmaf(s32, c, -m),
    m = fl(rowmax s32 c) (attn_tc_kernel, wgmma): each of s32 c and m is within scale e_raw + 2u |s| of its exact value, the
    subtraction or fma rounds once (u |arg|), ex2 adds EX2_REL.
    kv_tile: the kernel's KV tile (online softmax): the running max, the corr = exp(m_old - m_new) rescale of l and of the P v
    accumulator, and the bf16 rounding of P against the running max of its tile.  Each rescale adds one rounding (corr's ex2 and
    its argument, then the product: 8u per tile to l and to P v); a tile after which the running max may still rise has its P
    rounded against that tile's max, not the row's, so its elements are charged a full bf16 rounding (2^-8 p) rather than band()."""
    d = q.shape[-1]
    raw = q @ k.transpose(-1, -2)
    s = scale * raw
    e_raw = abs(scale) * GAMMA * d * U * (q.abs() @ k.abs().transpose(-1, -2))
    if bias is not None:
        s = s + bias
    e_s = e_raw + U * s.abs() if not ex2 else e_raw + 2 * U * s.abs()
    masked = None
    if causal:
        N, Nk = s.shape[-2:]
        masked = torch.ones(N, Nk, dtype=torch.bool, device=s.device).triu(1)
        s = s.masked_fill(masked, float("-inf"))
        e_s = e_s.masked_fill(masked, 0.0)
    mx = s.amax(-1, keepdim=True)
    arg = s - mx
    p = torch.exp(arg)
    if ex2:
        delta = e_s + e_s.amax(-1, keepdim=True) + U * arg.abs() + EX2_REL
    else:
        delta = e_s + 2 * e_s.amax(-1, keepdim=True) + U * arg.abs() + 2 * U * (2 + 1.16 * arg.abs())   # relative error of each p
    if masked is not None:
        delta = delta.masked_fill(masked, 0.0)
    Nk = s.shape[-1]
    nt = 1 if kv_tile is None else -(-Nk // kv_tile)
    rescale = 8 * U * (nt - 1)
    l = p.sum(-1, keepdim=True)
    rel_l = (p * delta).sum(-1, keepdim=True) / l + GAMMA * Nk * U + rescale
    P, dev = band(p, p * delta)
    if nt > 1:
        err = (delta.amax(-1, keepdim=True) + U * mx.abs()).expand_as(s)
        tile = torch.arange(Nk, device=s.device) // kv_tile
        for t in range(nt - 1):
            cols = tile == t
            m_t = s[..., :kv_tile * (t + 1)].amax(-1, keepdim=True)
            later = s[..., kv_tile * (t + 1):].amax(-1, keepdim=True)
            rises = (later >= m_t - 2 * err[..., :1]) & cols
            dev = torch.where(rises, torch.maximum(dev, 2.0 ** -8 * p), dev)
    o = P @ v
    e_o = dev @ v.abs() + (GAMMA * Nk * U + rescale) * (P @ v.abs())
    y = o / l
    e_y = e_o / l + y.abs() * (rel_l + 2 * U) + U * y.abs()
    return y, e_y


def win_attn_bias(qkv, qkv_pad, bias, B, H, W, C, heads, ws, scale):
    """es3_win_attn_bias_bf16, head dim 32: per window (padded positions take qkv_pad), softmax_attn with the per-head bias and
    __expf, bf16 store.  `bias` is what the kernel reads: pass fp16(bias) for ws = 14 (its shared-memory table).
    Returns (ref, bound) of out [B H W, C]; padded queries are not outputs."""
    tok = win_tokens(B, H, W, ws).to(qkv.device)
    nwin, N = tok.shape
    rows = torch.cat([qkv, qkv_pad[None]], 0)[torch.where(tok >= 0, tok, torch.full_like(tok, qkv.shape[0]))]
    t = rows.reshape(nwin, N, heads, 3, 32).permute(3, 0, 2, 1, 4)              # [3, nwin, heads, N, 32]
    y, e_y = softmax_attn(t[0], t[1], t[2], scale, bias)
    y, e_y = y.permute(0, 2, 1, 3).reshape(nwin * N, C), e_y.permute(0, 2, 1, 3).reshape(nwin * N, C)
    keep = tok.reshape(-1) >= 0
    out = torch.empty(B * H * W, C, dtype=y.dtype, device=y.device)
    err = torch.empty_like(out)
    out[tok.reshape(-1)[keep]] = y[keep]
    err[tok.reshape(-1)[keep]] = e_y[keep]
    return out, _out(out, err, True)


# ------------------------------------------------------------------------------------------------ exact operations
def bilinear(x, Ho, Wo):
    """es3_bilinear_nhwc_to_nchw: F.interpolate(bilinear, align_corners=False) of x [B, Hi, Wi, C] -> NCHW fp32.  The kernel's
    fp32 source coordinates and weights are each within 4u (Hi + Wi + Ho + Wo) of exact; four taps of |x| <= max |x|."""
    Hi, Wi = x.shape[1:3]
    ref = F.interpolate(_nchw(x), size=(Ho, Wo), mode="bilinear", align_corners=False)
    amax = x.abs().amax((1, 2))[:, :, None, None]
    e = (8 * 4 * U * (Hi + Wi + Ho + Wo) + GAMMA * 8 * U) * amax
    return ref, _out(ref, e, False)


def round_taps_sum_emu(w):
    """Host emulation of es3_round_taps_sum_bf16's fixed fp32 algorithm, w [KK, C] fp32 -> [KK, C] fp32: nearest bf16 per tap, then
    up to four one-step moves of the tap with the largest same-sign rounding error (first index on ties), each kept only if it
    brings the fp32 running sum strictly closer to the fp32 tap sum (sums accumulated tap by tap in fp32)."""
    t = w.float().cpu()
    KK, C = t.shape
    r = t.to(torch.bfloat16).float()
    sw = torch.zeros(C)
    sr = torch.zeros(C)
    for i in range(KK):
        sw = sw + t[i]
        sr = sr + r[i]
    live = torch.ones(C, dtype=torch.bool)
    cols = torch.arange(C)
    for _ in range(4):
        res = sw - sr
        live &= res != 0
        sgn = torch.where(res > 0, 1.0, -1.0)
        best = torch.argmax((t - r) * sgn, 0)                       # first maximum, like the kernel's strict '>' scan
        rb = r[best, cols]
        ulp = (rb.view(torch.int32) & 0x7F800000).view(torch.float32) * 0.0078125
        live &= ulp != 0
        cand = (rb + sgn * ulp).to(torch.bfloat16).float()
        new = (sr - rb) + cand
        live &= (sw - new).abs() < res.abs()
        r[best[live], cols[live]] = cand[live]
        sr = torch.where(live, new, sr)
    return r
