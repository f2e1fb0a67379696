"""fp64 statements of the image students' backward kernels and, next to each, the per-element bound its fp32 arithmetic keeps
to (running error analysis: every intermediate's error is propagated to first order, evaluated in fp64 on absolute values).

Operands are bf16-representable or used as given (fp32 images, weights, statistics), so each statement is what the kernel
computes with exact arithmetic.  Notation: u = 2^-24; an fp32 sum of n terms is held to GAMMA n u sum |terms| (n = the total term
count, conservative for split and tree sums); an fp32 result adds 4u |ref| and a bf16 result 2^-8 |ref| for its own rounding.
Every function takes and returns float64 tensors (CPU or CUDA).  tests/test_train_bwd_cpu.py ties each statement to
torch.autograd of the forward operation in float64.
"""
import torch
import torch.nn.functional as F

from bounds import L_ACT, U, _act64, _eps_act

GAMMA = 2.0
BF16_HALF = 2.0 ** -8          # bound on the relative rounding of a bf16 store, with margin (the half-step is 2^-9)
TINY = 1e-30                   # keeps bound > 0 where the reference and every term are exactly zero
EPS_GELU_GRAD = 1e-6           # erff (2 ulp) and __expf ((2 + 1.16 |x|) ulp) in gelu'(x), per unit of |da|
KINKS = {"relu": (0.0,), "hswish": (-3.0, 3.0)}


def _out(ref, inner, bf16):
    b = inner + 4 * U * ref.abs() + TINY
    return b * (1 + BF16_HALF) + BF16_HALF * ref.abs() if bf16 else b


# ------------------------------------------------------------------------------------------------ pointwise weight gradient
def shift_rows(x, H, W, dy, dx):
    """Row (b, y, x) of the result is row (b, y + dy, x + dx) of x [B*H*W, K], zero outside the H x W map."""
    K = x.shape[1]
    x4 = F.pad(x.reshape(-1, H, W, K), (0, 0, 1, 1, 1, 1))
    return x4[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W].reshape(-1, K)


def wgrad(dz, x, dW0):
    """dW0 + dz^T x: dz [M, N], x [M, K], dW0 [N, K]."""
    ref = dW0 + dz.t() @ x
    terms = dW0.abs() + dz.abs().t() @ x.abs()
    return ref, _out(ref, GAMMA * (dz.shape[0] + 1) * U * terms, False)


# ------------------------------------------------------------------------------------------------ depthwise conv gradients
def dw_weight(w):
    """[ks*ks, C] tap-major weights -> [C, 1, ks, ks]."""
    kk, C = w.shape
    ks = int(round(kk ** 0.5))
    return w.t().reshape(C, 1, ks, ks)


def dwconv_bwd_data(dz, w, H, W, ks, stride):
    """Input gradient of the depthwise conv (pad ks // 2): dz [B, Ho, Wo, C], w [ks*ks, C] -> [B, H, W, C] (bf16 store)."""
    wt = dw_weight(w)
    C = dz.shape[3]
    op = (H + 2 * (ks // 2) - ks) % stride, (W + 2 * (ks // 2) - ks) % stride

    def adj(d, ww):
        return F.conv_transpose2d(d.permute(0, 3, 1, 2), ww, stride=stride, padding=ks // 2, output_padding=op,
                                  groups=C).permute(0, 2, 3, 1)
    ref = adj(dz, wt)
    terms = adj(dz.abs(), wt.abs())
    return ref, _out(ref, GAMMA * ks * ks * U * terms, True)


def dwconv_wgrad(dz, x, dW0, ks, stride):
    """dW0 [C, 1, ks, ks] + the depthwise weight gradient: dz [B, Ho, Wo, C], x [B, H, W, C]."""
    C = x.shape[3]

    def corr(d, xx):       # sum_p d[p][c] x[src(p, tap)][c] per (c, tap)
        xn = F.pad(xx.permute(0, 3, 1, 2), (ks // 2,) * 4)
        dn = d.permute(0, 3, 1, 2)
        out = torch.empty(C, ks, ks, dtype=d.dtype, device=d.device)
        Ho, Wo = dn.shape[2], dn.shape[3]
        for ky in range(ks):
            for kx in range(ks):
                win = xn[:, :, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
                out[:, ky, kx] = (win * dn).sum((0, 2, 3))
        return out.reshape(C, 1, ks, ks)
    ref = dW0 + corr(dz, x)
    terms = dW0.abs() + corr(dz.abs(), x.abs())
    n = dz.shape[0] * dz.shape[1] * dz.shape[2] + 1
    return ref, _out(ref, GAMMA * n * U * terms, False)


def stem_wgrad(img, dz, dW0):
    """dW0 [Cout, 3, 3, 3] + weight gradient of the 3x3 stride-2 pad-1 conv: img [B, 3, H, W], dz [B, Ho, Wo, Cout]."""
    def g(i, d):
        return torch.nn.grad.conv2d_weight(i, dW0.shape, d.permute(0, 3, 1, 2), stride=2, padding=1)
    ref = dW0 + g(img, dz)
    terms = dW0.abs() + g(img.abs(), dz.abs())
    n = dz.shape[0] * dz.shape[1] * dz.shape[2] + 1
    return ref, _out(ref, GAMMA * n * U * terms, False)


def conv3x3_wgrad(dy, a, gw0):
    """gw0 [N, C, 3, 3] + the weight gradient of a dense 3x3 pad-1 conv: dy [B, H, W, N], a [B, H, W, C]."""
    def g(aa, d):
        return torch.nn.grad.conv2d_weight(aa.permute(0, 3, 1, 2), gw0.shape, d.permute(0, 3, 1, 2), padding=1)
    ref = gw0 + g(a, dy)
    terms = gw0.abs() + g(a.abs(), dy.abs())
    n = dy.shape[0] * (dy.shape[1] + 2) * (dy.shape[2] + 8) + 1          # the GEMM runs over the zero-framed pixel index
    return ref, _out(ref, GAMMA * n * U * terms, False)


def transpose_pad(x, Wp, dx):
    """x [B, H, W, C] -> [C, B*(H+2)*Wp]: out[c][(b (H+2) + y + 1) Wp + x + 1 - dx] = x[b, y, x, c], zero elsewhere."""
    B, H, W, C = x.shape
    out = torch.zeros(C, B, H + 2, Wp, dtype=x.dtype, device=x.device)
    out[:, :, 1:H + 1, 1 - dx:1 - dx + W] = x.permute(3, 0, 1, 2)
    return out.reshape(C, -1)


# ------------------------------------------------------------------------------------------------ BatchNorm pieces
def bn_stats(z, gamma, beta, eps, momentum, rm, rv):
    """Batch statistics of z [M, C] and the running-buffer update.  The kernel sums d = z - z[0] (exact in fp32) and d^2 over the
    rows in fp32, then finalises in fp64.  Returns dict name -> (ref, bound)."""
    M = z.shape[0]
    d = z - z[:1]
    s0, s1 = d.sum(0), (d * d).sum(0)
    e0, e1 = GAMMA * M * U * d.abs().sum(0), GAMMA * (M + 1) * U * (d * d).sum(0)
    dm = s0 / M
    mu = z[0] + dm
    var = s1 / M - dm * dm
    e_dm = e0 / M
    e_var = e1 / M + 2 * dm.abs() * e_dm
    e_mu = e_dm + U * mu.abs()
    istd = 1.0 / torch.sqrt(var + eps)
    e_is = 0.5 * istd ** 3 * e_var + U * istd
    g = gamma if gamma is not None else torch.ones_like(mu)
    b = beta if beta is not None else torch.zeros_like(mu)
    sc = g * istd
    e_sc = g.abs() * e_is + U * sc.abs()
    sh = b - mu * sc
    e_sh = mu.abs() * e_sc + sc.abs() * e_mu + 2 * U * ((mu * sc).abs() + sh.abs())
    out = {"mean": (mu, _out(mu, e_mu, False)), "invstd": (istd, _out(istd, e_is, False)), "scale": (sc, _out(sc, e_sc, False)),
           "shift": (sh, _out(sh, e_sh, False))}
    if rm is not None:
        r = (1 - momentum) * rm + momentum * mu
        out["running_mean"] = (r, _out(r, momentum * e_mu + 4 * U * ((1 - momentum) * rm.abs() + momentum * mu.abs()), False))
    if rv is not None:
        f = M / (M - 1) if M > 1 else 1.0
        r = (1 - momentum) * rv + momentum * var * f
        out["running_var"] = (r, _out(r, momentum * f * e_var + 4 * U * ((1 - momentum) * rv.abs() + momentum * f * var.abs()), False))
    return out


def act_grad(x, act):
    """act'(x) in fp64 (aten's hardswish_backward convention at +-3)."""
    if act is None:
        return torch.ones_like(x)
    if act == "relu":
        return (x > 0).double()
    if act == "hswish":
        return torch.where(x < -3, 0.0, torch.where(x <= 3, x / 3 + 0.5, 1.0))
    if act == "gelu":
        return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
    raise ValueError(act)


def act_grad_err(x, act):
    """Bound on |act'(x32) - act'(x)| for the kernel's pre-activation x32 = fl(scale z + shift) (|x32 - x| <= u |x|), away from the
    kinks (KINKS: the inputs keep da = 0 within kink_band of them)."""
    dxa = U * x.abs()
    if act == "hswish":
        return 2 * dxa / 3 + 2 * U             # the pre-activation's rounding and fl(1/3) in fmaf(x, 1/3, 0.5)
    if act == "gelu":
        return 0.8 * dxa + EPS_GELU_GRAD
    return torch.zeros_like(x)


def kink_band(x, act):
    """Pre-activations within the fp32-error band of a derivative discontinuity of `act` (where the branch may flip)."""
    band = torch.zeros_like(x, dtype=torch.bool)
    for k in KINKS.get(act, ()):
        band |= (x - k).abs() <= 4 * U * x.abs() + 1e-30
    return band


def affine_act(z, scale, shift, act, res=None):
    """act(scale z + shift) (+ res), bf16 store."""
    pre = z * (scale if scale is not None else 1.0) + (shift if shift is not None else 0.0)
    ref = _act64(pre, act)
    inner = L_ACT[act] * (U * pre.abs() + _eps_act(pre, act)) + 2 * U * ref.abs()
    if res is not None:
        ref = ref + res
        inner = inner + U * ref.abs()
    return ref, _out(ref, inner, True)


def bn_act_bwd(da, z, scale, shift, act, mode, mean, invstd, dg0, db0):
    """Backward through act(scale z + shift) of the norm `mode` ("none": bias only, "eval": frozen BN, "batch": batch-statistics
    BN with the statistics mean / invstd): g = da act'(u); dbeta += sum g; dgamma += invstd (sum g z - mean sum g);
    dz = A g + B z + C (A = scale; batch mode: B = -scale invstd dgamma / M, C = -scale sum g / M - B mean).
    Returns dict name -> (ref, bound) for dz (bf16 store), dgamma, dbeta."""
    M, C = z.shape
    sc = scale if scale is not None else torch.ones(C, dtype=z.dtype, device=z.device)
    sh = shift if shift is not None else torch.zeros(C, dtype=z.dtype, device=z.device)
    u = sc * z + sh
    ag = act_grad(u, act)
    g = da * ag
    e_g = da.abs() * act_grad_err(u, act) + U * g.abs()
    sg, sgz = g.sum(0), (g * z).sum(0)
    e_sg = GAMMA * M * U * g.abs().sum(0) + e_g.sum(0)
    e_sgz = GAMMA * M * U * (g * z).abs().sum(0) + (e_g * z.abs()).sum(0)
    out = {}
    db = db0 + sg
    out["dbeta"] = (db, _out(db, e_sg + 4 * U * db0.abs(), False))
    Bc = torch.zeros_like(sg)
    Cc = torch.zeros_like(sg)
    e_B = torch.zeros_like(sg)
    e_C = torch.zeros_like(sg)
    if mode != "none":
        dgam = invstd * (sgz - mean * sg)
        e_dgam = invstd.abs() * (e_sgz + mean.abs() * e_sg) + U * dgam.abs()
        dg = dg0 + dgam
        out["dgamma"] = (dg, _out(dg, e_dgam + 4 * U * dg0.abs(), False))
        if mode == "batch":
            Bc = -sc * invstd * dgam / M
            Cc = -sc * sg / M - Bc * mean
            e_B = (sc * invstd).abs() * e_dgam / M + U * Bc.abs()
            e_C = sc.abs() * e_sg / M + (sc * invstd * mean).abs() * e_dgam / M + U * (Cc.abs() + (Bc * mean).abs())
    dz = sc * g + Bc * z + Cc
    e_dz = sc.abs() * e_g + e_B * z.abs() + e_C + 2 * U * ((sc * g).abs() + (Bc * z).abs() + Cc.abs())
    out["dz"] = (dz, _out(dz, e_dz, True))
    return out


# ------------------------------------------------------------------------------------------------ element-wise pieces
def se_dgate(dy, x, dgate0):
    """dgate0 [B, C] + sum over the pixels of dy x (dy, x: [B, HW, C])."""
    ref = dgate0 + (dy * x).sum(1)
    terms = dgate0.abs() + (dy * x).abs().sum(1)
    return ref, _out(ref, GAMMA * (dy.shape[1] + 1) * U * terms, False)


def se_apply(dy, gate, add):
    """dy gate[b, c] + add[b, c], bf16 store (dy [B, HW, C])."""
    ref = dy * gate[:, None] + add[:, None]
    return ref, _out(ref, U * ((dy * gate[:, None]).abs() + ref.abs()), True)


def bilinear_bwd(dout, Hi, Wi):
    """Adjoint of the align_corners=False bilinear resize [B, C, Hi, Wi] -> dout's [Ho, Wo]; result NHWC, bf16 store.  The kernel's
    interpolation weights come from fp32 source coordinates, each within 4u (Hi + Wi + Ho + Wo) of its exact value; at most
    12 x 12 candidate outputs feed an input pixel."""
    def adj(d):
        x = torch.zeros(d.shape[0], d.shape[1], Hi, Wi, dtype=d.dtype, device=d.device, requires_grad=True)
        with torch.enable_grad():
            y = F.interpolate(x, size=d.shape[2:], mode="bilinear", align_corners=False)
            (gx,) = torch.autograd.grad(y, x, d)
        return gx.permute(0, 2, 3, 1)
    Ho, Wo = dout.shape[2:]
    ref = adj(dout)
    terms = adj(dout.abs())
    e_w = 4 * U * (Hi + Wi + Ho + Wo)
    local = dout.abs().amax((2, 3))[:, None, None, :]           # per image and channel
    return ref, _out(ref, GAMMA * 144 * U * terms + 2 * e_w * 144 * local, True)


def colsum(src, out0):
    """out0 [L] + the column sums of src [M, L]."""
    ref = out0 + src.sum(0)
    return ref, _out(ref, GAMMA * (src.shape[0] + 1) * U * (out0.abs() + src.abs().sum(0)), False)


# ------------------------------------------------------------------------------------------------ LiteMLA backward
def litemla_bwd(ms, dy, kv_part, heads2, dim, eps):
    """Backward of the ReLU linear attention given the forward's partial KV sums.
    ms [B, HW, heads2 * 3 dim] (q | k | v per head), dy [B, HW, heads2 dim], kv_part [B, heads2, nchunk, dim + 1, dim].
    q' = relu(q), k' = relu(k), vpad = [v, 1]; KV = sum of the partials (fp32 sum in the kernel);
    o = KV q', r = 1 / (o[dim] + eps), y = o[:dim] r;  do[j] = dy[j] r, do[dim] = -r sum_j dy[j] y[j];
    dKV = sum_n do q'^T;  dq = [q > 0] KV^T do,  dk = [k > 0] dKV^T vpad,  dv = dKV[:dim] k'.
    Returns (ref, bound) of dms [B, HW, heads2 * 3 dim] (bf16 store)."""
    B, HW, _ = ms.shape
    d = dim
    t = ms.reshape(B, HW, heads2, 3 * d)
    q, k, v = t[..., :d], t[..., d:2 * d], t[..., 2 * d:]
    qr, kr = q.clamp_min(0), k.clamp_min(0)
    vpad = torch.cat([v, torch.ones_like(v[..., :1])], -1)                   # [B, HW, h, d+1]
    dyh = dy.reshape(B, HW, heads2, d)
    KV = kv_part.sum(2)                                                    # [B, h, d+1, d]
    e_KV = GAMMA * kv_part.shape[2] * U * kv_part.abs().sum(2)
    aKV = KV.abs()
    o = torch.einsum("bhji,bnhi->bnhj", KV, qr)                            # [B, HW, h, d+1]
    e_o = torch.einsum("bhji,bnhi->bnhj", e_KV + GAMMA * d * U * aKV, qr)
    den = o[..., d] + eps
    e_den = e_o[..., d] + U * den.abs()
    r = 1.0 / den
    e_r = r * r * e_den + U * r.abs()
    y = o[..., :d] * r[..., None]
    e_y = o[..., :d].abs() * e_r[..., None] + r.abs()[..., None] * e_o[..., :d] + U * y.abs()
    dot = (dyh * y).sum(-1)
    e_dot = (dyh.abs() * e_y).sum(-1) + GAMMA * d * U * (dyh * y).abs().sum(-1)
    do = torch.cat([dyh * r[..., None], (-r * dot)[..., None]], -1)          # [B, HW, h, d+1]
    e_do = torch.cat([dyh.abs() * e_r[..., None] + U * (dyh * r[..., None]).abs(),
                      (r.abs() * e_dot + dot.abs() * e_r + U * (r * dot).abs())[..., None]], -1)
    dKV = torch.einsum("bnhj,bnhi->bhji", do, qr)
    nchunk = (HW + 127) // 128
    e_dKV = torch.einsum("bnhj,bnhi->bhji", e_do, qr) + GAMMA * (HW + nchunk) * U * torch.einsum("bnhj,bnhi->bhji", do.abs(), qr)
    adKV = dKV.abs()
    dq = torch.einsum("bhji,bnhj->bnhi", KV, do) * (q > 0)
    e_dq = (torch.einsum("bhji,bnhj->bnhi", e_KV, do.abs()) + torch.einsum("bhji,bnhj->bnhi", aKV, e_do)
            + GAMMA * (d + 1) * U * torch.einsum("bhji,bnhj->bnhi", aKV, do.abs()))
    dk = torch.einsum("bhji,bnhj->bnhi", dKV, vpad) * (k > 0)
    e_dk = torch.einsum("bhji,bnhj->bnhi", e_dKV + GAMMA * (d + 1) * U * adKV, vpad.abs())
    dv = torch.einsum("bhji,bnhi->bnhj", dKV[:, :, :d], kr)
    e_dv = torch.einsum("bhji,bnhi->bnhj", e_dKV[:, :, :d] + GAMMA * d * U * adKV[:, :, :d], kr)
    ref = torch.cat([dq, dk, dv], -1).reshape(B, HW, heads2 * 3 * d)
    err = torch.cat([e_dq, e_dk, e_dv], -1).reshape(B, HW, heads2 * 3 * d)
    return ref, _out(ref, err, True)


# ------------------------------------------------------------------------------------------------ TinyViT pieces
def layernorm_bwd(x, dy, gamma, eps, dg0, db0, dres, bf16=True):
    """nn.LayerNorm backward over rows of x, dy [M, C]: dx = rstd (g - mean(g) - xh mean(g xh)) (+ dres), g = dy gamma;
    dgamma += sum dy xh, dbeta += sum dy.  Returns dict name -> (ref, bound); dx is a bf16 store (bf16 = False: fp32)."""
    M, C = x.shape
    mu = x.mean(1, keepdim=True)
    e_mu = GAMMA * C * U * x.abs().mean(1, keepdim=True) + U * mu.abs()
    dd = x - mu
    e_d = e_mu + U * dd.abs()
    q = (dd * dd).sum(1, keepdim=True)
    e_q = (2 * dd.abs() * e_d).sum(1, keepdim=True) + GAMMA * (C + 1) * U * q
    var = q / C + eps
    e_var = e_q / C + 2 * U * var
    rstd = var.rsqrt()
    e_rstd = 0.5 * rstd ** 3 * e_var + 4 * U * rstd
    xh = dd * rstd
    e_xh = dd.abs() * e_rstd + rstd * e_d + U * xh.abs()
    g = dy * gamma
    e_g = U * g.abs()
    c1 = g.mean(1, keepdim=True)
    e_c1 = (GAMMA * C * U * g.abs().sum(1, keepdim=True) + e_g.sum(1, keepdim=True)) / C + U * c1.abs()
    c2 = (g * xh).mean(1, keepdim=True)
    e_c2 = ((g.abs() * e_xh + xh.abs() * e_g).sum(1, keepdim=True) + GAMMA * C * U * (g * xh).abs().sum(1, keepdim=True)) / C \
        + U * c2.abs()
    tt = g - c1 - xh * c2
    e_t = e_g + e_c1 + xh.abs() * e_c2 + c2.abs() * e_xh + 3 * U * (g.abs() + c1.abs() + (xh * c2).abs())
    dx = rstd * tt
    e_dx = tt.abs() * e_rstd + rstd * e_t + U * dx.abs()
    if dres is not None:
        dx = dx + dres
        e_dx = e_dx + U * dx.abs()
    dg = dg0 + (dy * xh).sum(0)
    e_dg = (dy.abs() * e_xh).sum(0) + GAMMA * (M + 1) * U * (dg0.abs() + (dy * xh).abs().sum(0))
    db = db0 + dy.sum(0)
    e_db = GAMMA * (M + 1) * U * (db0.abs() + dy.abs().sum(0))
    return {"dx": (dx, _out(dx, e_dx, bf16)), "dgamma": (dg, _out(dg, e_dg, False)), "dbeta": (db, _out(db, e_db, False))}


def win_attn_tokens(B, H, W, ws):
    """Token index [B * nWin, ws*ws] of every window's tokens in window-raster order."""
    nH, nW = H // ws, W // ws
    t = torch.arange(B * H * W).reshape(B, nH, ws, nW, ws).permute(0, 1, 3, 2, 4)
    return t.reshape(B * nH * nW, ws * ws)


def softmax_attn_bwd(q, k, v, do, scale, bias=None, causal=False, o=None, exp_rel=None):
    """Backward of softmax attention over q, k, v, do [..., N, d]: s = scale q k^T (+ bias) (+ -inf above the diagonal when causal),
    P = softmax(s), o = P v.  dP = do v^T, D = rowsum(do o), dS = P (dP - D); dq = scale dS k, dk = scale dS^T q, dv = P^T do.
    o: the forward output the kernel is given (D is then taken over it, as es3_text_attn_bwd's contract states); None: the exact
    P v (D = rowsum(P dP)).  exp_rel(arg): the relative error of the kernel's exp (default __expf: (2 + 1.16 |arg|) ulp).
    Returns dict name -> (ref, inner bound) for dq, dk, dv and dS."""
    d = q.shape[-1]
    N = k.shape[-2]
    s = scale * q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    e_s = abs(scale) * GAMMA * d * U * (q.abs() @ k.abs().transpose(-1, -2)) + U * s.abs()
    masked = None
    if causal:
        masked = torch.ones(s.shape[-2], N, dtype=torch.bool, device=s.device).triu(1)
        s = s.masked_fill(masked, float("-inf"))
        e_s = e_s.masked_fill(masked, 0.0)
    P = torch.softmax(s, -1)
    mx = s.amax(-1, keepdim=True)
    arg = s - mx
    e_exp = 2 * U * (2 + 1.16 * arg.abs()) if exp_rel is None else exp_rel(arg)
    delta = e_s + 2 * e_s.amax(-1, keepdim=True) + U * arg.abs() + e_exp        # relative error of each exp
    if masked is not None:
        delta = delta.masked_fill(masked, 0.0)
    rel_l = (P * delta).sum(-1, keepdim=True) + GAMMA * N * U
    e_P = P * (delta + rel_l + 2 * U)
    dP = do @ v.transpose(-1, -2)
    e_dP = GAMMA * d * U * (do.abs() @ v.abs().transpose(-1, -2))
    if o is None:
        D = (P * dP).sum(-1, keepdim=True)
        e_D = (e_P * dP.abs() + P * e_dP).sum(-1, keepdim=True) + GAMMA * N * U * (P * dP.abs()).sum(-1, keepdim=True) + U * D.abs()
    else:
        D = (do * o).sum(-1, keepdim=True)
        e_D = GAMMA * d * U * (do * o).abs().sum(-1, keepdim=True) + U * D.abs()
    dS = P * (dP - D)
    e_dS = e_P * (dP - D).abs() + P * (e_dP + e_D + U * (dP - D).abs()) + U * dS.abs()
    if masked is not None:
        dS = dS.masked_fill(masked, 0.0)
        e_dS = e_dS.masked_fill(masked, 0.0)
    dq = scale * dS @ k
    e_dq = abs(scale) * (e_dS @ k.abs() + GAMMA * N * U * (dS.abs() @ k.abs())) + U * dq.abs()
    dk = scale * dS.transpose(-1, -2) @ q
    e_dk = abs(scale) * (e_dS.transpose(-1, -2) @ q.abs() + GAMMA * N * U * (dS.abs().transpose(-1, -2) @ q.abs())) + U * dk.abs()
    dv = P.transpose(-1, -2) @ do
    e_dv = e_P.transpose(-1, -2) @ do.abs() + GAMMA * N * U * (P.transpose(-1, -2) @ do.abs())
    return {"dq": (dq, e_dq), "dk": (dk, e_dk), "dv": (dv, e_dv), "dS": (dS, e_dS)}


def win_attn_bias_bwd(qkv, dout, bias, B, H, W, C, heads, ws, scale):
    """Backward of windowed attention with a per-head bias, head dim 32 (softmax_attn_bwd per window, D = rowsum(P dP)).
    Returns dict: "dqkv" (ref, bound) [B*H*W, 3C] bf16 store, "dS" (ref, bound) [nwin, heads, N, N] fp32."""
    tok = win_attn_tokens(B, H, W, ws).to(qkv.device)
    nwin, N = tok.shape
    t = qkv[tok].reshape(nwin, N, heads, 3, 32).permute(3, 0, 2, 1, 4)        # [3, nwin, heads, N, 32]
    do = dout[tok].reshape(nwin, N, heads, 32).permute(0, 2, 1, 3)
    r = softmax_attn_bwd(t[0], t[1], t[2], do, scale, bias)
    (dq, e_dq), (dk, e_dk), (dv, e_dv), (dS, e_dS) = r["dq"], r["dk"], r["dv"], r["dS"]

    def scatter(a, b, c):
        g = torch.stack([a, b, c], 3).permute(0, 2, 1, 3, 4).reshape(nwin * N, heads * 96)   # [nwin, N, heads, 3, 32]
        out = torch.empty(B * H * W, 3 * C, dtype=a.dtype, device=a.device)
        out[tok.reshape(-1)] = g
        return out
    ref = scatter(dq, dk, dv)
    return {"dqkv": (ref, _out(ref, scatter(e_dq, e_dk, e_dv), True)), "dS": (dS, _out(dS, e_dS, False))}
