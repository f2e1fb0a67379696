"""fp64 statements of the text encoders' kernels (attention.cu, attention_tc.cu, text.cu, text_bwd.cu, the LayerNorm of vit_ops.cu)
and, next to each, the per-element bound its fp32 arithmetic keeps to.

The bound form is ref_train_bwd.py's and ref_fwd.py's: an fp32 sum of n terms is held to GAMMA n u sum |terms|, an fp32 result adds
4u |ref| and a bf16 result 2^-8 |ref| for its own rounding (_out), bf16 intermediates are charged through band().  Operands are the
ones the kernel receives (bf16 qkv, the forward output O that the attention backward is given, the fp32 per-sample partials the KD
backward reads).  Every function takes and returns float64 tensors (CPU or CUDA).  tests/test_text_kernels_cpu.py ties each
statement to textbook float64 torch (autograd for the backward ones).
"""
import torch
import torch.nn.functional as F

from bounds import U
from ref_fwd import layernorm, softmax_attn
from ref_train_bwd import GAMMA, _out, layernorm_bwd, softmax_attn_bwd

COS_EPS = float(torch.tensor(1e-8, dtype=torch.float32))   # TXT_COS_EPS: the fp32 value of 1e-8 the kernels clamp the norms to
EXPF_REL = 4 * U               # expf (no fast math): 2 ulp (CUDA C++ Programming Guide, single-precision functions); an ulp is 2u


def _heads(t, B, L, parts, heads):
    """[B L, parts heads 64] -> parts x [B, heads, L, 64]."""
    return t.reshape(B, L, parts, heads, 64).permute(2, 0, 3, 1, 4)


def _tokens(t):
    """[B, heads, L, 64] -> [B L, heads 64]."""
    B, h, L, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * L, h * d)


# ------------------------------------------------------------------------------------------------ attention
def attention(qkv, B, L, heads, scale, causal, kernel):
    """es3_attention_causal_bf16 / es3_attention_bf16 (H = 1, W = L, win = 0) on qkv [B L, 3C]: softmax_attn with the ex2 exponent;
    kernel "mma" (attn_fwd_kernel, 64-key tiles) or "tc" (attn_tc_kernel, one 128-key tile at L <= 128).  bf16 store."""
    q, k, v = _heads(qkv, B, L, 3, heads)
    y, e = softmax_attn(q, k, v, scale, causal=causal, ex2=True, kv_tile=64 if kernel == "mma" else 128)
    y, e = _tokens(y), _tokens(e)
    return y, _out(y, e, True)


def attention_bwd(qkv, o, dout, B, L, heads, scale, causal):
    """es3_text_attn_bwd: softmax_attn_bwd with D_i = sum_c dO O over the O it is given and P recomputed with expf; dqkv in qkv's
    layout, bf16 store."""
    q, k, v = _heads(qkv, B, L, 3, heads)
    (oo,), (do,) = _heads(o, B, L, 1, heads), _heads(dout, B, L, 1, heads)
    r = softmax_attn_bwd(q, k, v, do, scale, causal=causal, o=oo, exp_rel=lambda a: EXPF_REL * torch.ones_like(a))
    ref = torch.cat([_tokens(r[n][0]).reshape(B * L, heads, 64) for n in ("dq", "dk", "dv")], 1).reshape(B * L, 3 * heads * 64)
    err = torch.cat([_tokens(r[n][1]).reshape(B * L, heads, 64) for n in ("dq", "dk", "dv")], 1).reshape(B * L, 3 * heads * 64)
    return ref, _out(ref, err, True)


# ------------------------------------------------------------------------------------------------ LayerNorm
def layernorm_f32(x, gamma, beta, eps, pos=None, ps=0, H=0, W=0, bf16=False):
    """es3_layernorm_f32 over rows x [M, C] fp32, with the optional tiled positional add first: row r takes pos[(h % ps) ps +
    (w % ps)], t = r % (H W), h = t // W, w = t % W, and the sum rounds once in fp32 (u |x + pos|).  bf16 or fp32 store."""
    e_x = None
    if pos is not None:
        t = torch.arange(x.shape[0], device=x.device) % (H * W)
        x = x + pos[(t // W % ps) * ps + t % W % ps]
        e_x = U * x.abs()
    return layernorm(x, gamma, beta, eps, bf16=bf16, e_x=e_x)


def layernorm_bwd_f32(x, dy, gamma, eps, dg0, db0, dres):
    """es3_layernorm_bwd_f32: ref_train_bwd.layernorm_bwd with the fp32 dx store (the bf16 copy is bf16(dx32) exactly)."""
    return layernorm_bwd(x, dy, gamma, eps, dg0, db0, dres, bf16=False)


# ------------------------------------------------------------------------------------------------ RepMixer
def _dw11(x, w, B, L):
    """Depthwise 1 x 11 along each sequence, zero padding 5: x [B L, C], w [11, C]."""
    C = x.shape[1]
    xs = x.reshape(B, L, C).permute(0, 2, 1)
    return F.conv1d(xs, w.t().unsqueeze(1), padding=5, groups=C).permute(0, 2, 1).reshape(B * L, C)


def repmixer(x, wm, bm, wf, bf, B, L):
    """es3_repmixer_bf16: x1 = bm + sum_k wm[k] x[l + k - 5] (an 11-term fp32 FMA chain from bm, fp32 store), u = bf16(bf + sum_k
    wf[k] x1[l + k - 5]) on the kernel's fp32 x1, whose error is carried through |wf|.  Returns ((x1, bound), (u, bound))."""
    x1 = _dw11(x, wm, B, L) + bm
    e1 = GAMMA * 12 * U * (_dw11(x.abs(), wm.abs(), B, L) + bm.abs())
    u = _dw11(x1, wf, B, L) + bf
    e_u = GAMMA * 12 * U * (_dw11(x1.abs(), wf.abs(), B, L) + bf.abs()) + _dw11(_out(x1, e1, False), wf.abs(), B, L)
    return (x1, _out(x1, e1, False)), (u, _out(u, e_u, True))


# ------------------------------------------------------------------------------------------------ embedding gradients
def embed_grad(dx, ids, grad0):
    """es3_text_embed_grad: grad0 [V, C] + the segmented sums of dx [B L, C] rows by id (chunk partials, then their sum)."""
    ids = ids.reshape(-1)
    ref = grad0.index_add(0, ids, dx)
    cnt = torch.bincount(ids, minlength=grad0.shape[0]).to(dx.dtype)[:, None]
    terms = grad0.abs().index_add(0, ids, dx.abs())
    return ref, _out(ref, GAMMA * (cnt + 1) * U * terms, False)


def resize_weights(N, L):
    """(i0, i1, l0, l1) of resize_src for rows l = 0 .. L-1, in the kernel's fp32 order: q = fl(N / L), src = fmaf(l + 0.5, q, -0.5)
    (one rounding: the product is exact in fp64), clamped at 0; i0 = trunc(src), i1 = i0 + (i0 < N - 1), l1 = src - i0 (exact),
    l0 = fl(1 - l1).  Weights as float64 values of the fp32 numbers."""
    f32 = torch.float32
    q = (torch.tensor(float(N), dtype=f32) / torch.tensor(float(L), dtype=f32)).double()
    t = torch.arange(L, dtype=torch.float64) + 0.5
    src = (t * q - 0.5).to(f32).clamp_min(0.0)
    i0 = src.to(torch.int64)
    i1 = i0 + (i0 < N - 1).to(torch.int64)
    l1 = src - i0.to(f32)
    l0 = 1.0 - l1
    return i0, i1, l0.double(), l1.double()


def pos_resize(table, L):
    """es3_text_pos_resize: out[l] = fmaf(l0, table[i0], l1 table[i1]) -- the product rounds, then the fma (in _out's 4u)."""
    N = table.shape[0]
    i0, i1, l0, l1 = (t.to(table.device) for t in resize_weights(N, L))
    b = l1[:, None] * table[i1]
    ref = l0[:, None] * table[i0] + b
    return ref, _out(ref, U * b.abs(), False)


def pos_weights(N, L):
    """[L, N] float64 values of the kernel's fp32 weights w(l, n) of text_pos_grad_kernel: the identity at N == L, else
    (i0 == n ? l0 : 0) + (i1 == n ? l1 : 0), the sum rounded in fp32 where i0 == i1."""
    if N == L:
        return torch.eye(L, dtype=torch.float64)
    i0, i1, l0, l1 = resize_weights(N, L)
    w = torch.zeros(L, N, dtype=torch.float32)
    ar = torch.arange(L)
    w[ar, i0] = l0.float()
    w[ar, i1] = w[ar, i1] + l1.float()
    return w.double()


def pos_grad(dx, N, grad0):
    """es3_text_pos_grad: grad0 [N, C] + sum_l w(l, n) sum_b dx[b, l] (dx [B, L, C]; b summed first, then an FMA chain over l)."""
    B, L, _ = dx.shape
    w = pos_weights(N, L).to(dx.device)
    ref = grad0 + w.t() @ dx.sum(0)
    terms = grad0.abs() + w.abs().t() @ dx.abs().sum(0)
    return ref, _out(ref, GAMMA * (B + L + 1) * U * terms, False)


# ------------------------------------------------------------------------------------------------ text KD loss
def _token_stats(p, t):
    """Per token: d2, dot, |p|, |t| and their bounds (fp32 FMA chains over D, the difference rounded before it is squared)."""
    D = p.shape[-1]
    d2 = ((p - t) ** 2).sum(-1)
    dot = (p * t).sum(-1)
    e_dot = GAMMA * D * U * (p * t).abs().sum(-1)
    np_, nt = p.norm(dim=-1), t.norm(dim=-1)
    return d2, (GAMMA * D + 2) * U * d2, dot, e_dot, np_, nt, GAMMA * D * U / 2 + U


def _valid(pad, shape, device):
    return torch.ones(shape, dtype=torch.float64, device=device) if pad is None else (~pad).double()


def kd_partials(p, t, pad):
    """es3_text_kd_loss_fwd's ws [B, 3] = (sum valid d2, sum valid (1 - cos), sum valid) per sample; cos = dot / (max(|p|, eps)
    max(|t|, eps)).  Returns ((ws, bound), cl) -- cl [B, L] = 1 - cos per token (for the tests)."""
    L = p.shape[1]
    d2, e_d2, dot, e_dot, np_, nt, rel_n = _token_stats(p, t)
    den = np_.clamp_min(COS_EPS) * nt.clamp_min(COS_EPS)
    cos = dot / den
    e_cos = e_dot / den + cos.abs() * (2 * rel_n + 2 * U)
    cl = 1 - cos
    e_cl = e_cos + U * cl.abs()
    v = _valid(pad, p.shape[:2], p.device)
    sq = (v * d2).sum(1)
    e_sq = (v * e_d2).sum(1) + GAMMA * (L + 8) * U * sq
    cls = (v * cl).sum(1)
    e_cls = (v * e_cl).sum(1) + GAMMA * (L + 8) * U * (v * cl.abs()).sum(1)
    n = v.sum(1)
    ws = torch.stack([sq, cls, n], 1)
    e_ws = torch.stack([e_sq, e_cls, torch.zeros_like(n)], 1)
    return (ws, _out(ws, e_ws, False)), cl


def kd_out3(ws, e_ws, L, D, masked, w):
    """out3 = (loss, mse, cos) from the per-sample partials (ws, e_ws) the final kernel reads, summed over the samples in order."""
    B = ws.shape[0]
    sq, cls, n = ws[:, 0], ws[:, 1], ws[:, 2]
    if masked:
        den = n.clamp_min(1.0)
        a, ea = sq / (den * D), e_ws[:, 0] / (den * D)
        c, ec = cls / den, e_ws[:, 1] / den
        mse, cos = a.mean(), c.mean()
        e_mse = (ea.sum() + GAMMA * (B + 3) * U * a.abs().sum()) / B
        e_cos = (ec.sum() + GAMMA * (B + 3) * U * c.abs().sum()) / B
    else:
        mse, cos = sq.sum() / (B * L * D), cls.sum() / (B * L)
        e_mse = (e_ws[:, 0].sum() + GAMMA * (B + 3) * U * sq.abs().sum()) / (B * L * D)
        e_cos = (e_ws[:, 1].sum() + GAMMA * (B + 3) * U * cls.abs().sum()) / (B * L)
    loss = mse + w * cos
    e_loss = e_mse + abs(w) * e_cos + 2 * U * (mse.abs() + abs(w) * cos.abs())
    ref = torch.stack([loss, mse, cos])
    return ref, _out(ref, torch.stack([e_loss, e_mse, e_cos]), False)


def kd_loss64(p, t, pad, w):
    """The text KD loss in float64 torch: masked_text_mse + w masked_text_cosine_loss (pad given), else text_mse + w
    text_cosine_loss, with F.cosine_similarity (eps = the kernels' fp32 1e-8)."""
    B, L, D = p.shape
    cl = 1 - F.cosine_similarity(p, t, dim=-1, eps=COS_EPS)
    d2 = ((p - t) ** 2).sum(-1)
    if pad is None:
        return d2.sum() / (B * L * D) + w * cl.mean()
    v = (~pad).to(p.dtype)
    den = v.sum(1).clamp_min(1.0)
    return ((v * d2).sum(1) / (den * D)).mean() + w * ((v * cl).sum(1) / den).mean()


def kd_bwd(p, t, pad, n_valid, w, g):
    """es3_text_kd_loss_bwd: dp = g d kd_loss64 / dp by float64 autograd (the padding tokens of a masked loss get exactly 0);
    n_valid [B]: the valid-token counts of the ws the kernel reads.  The bound follows the kernel's explicit form
    dp = g (a_mse (p - t) - a_cos (t ct - p cp)), ct = 1 / (np' nt'), cp = dot / (np'^2 nt' |p|) (0 at p = 0), np' = max(|p|, eps)."""
    B, L, D = p.shape
    pr = p.clone().requires_grad_(True)
    with torch.enable_grad():
        (ref,) = torch.autograd.grad(kd_loss64(pr, t, pad, w), pr)
    ref = g * ref
    _, _, dot, e_dot, np_, nt, rel_n = _token_stats(p, t)
    npc, ntc = np_.clamp_min(COS_EPS), nt.clamp_min(COS_EPS)
    ct = 1 / (npc * ntc)
    e_ct = ct * (2 * rel_n + 3 * U)
    cp = torch.where(np_ > 0, dot / (npc * npc * ntc * np_.clamp_min(1e-300)), torch.zeros_like(dot))
    e_cp = torch.where(np_ > 0, (e_dot + dot.abs() * (4 * rel_n + 6 * U)) / (npc * npc * ntc * np_.clamp_min(1e-300)),
                       torch.zeros_like(dot))
    dcos = t * ct[..., None] - p * cp[..., None]
    e_dcos = t.abs() * e_ct[..., None] + p.abs() * e_cp[..., None] + U * ((t * ct[..., None]).abs() + (p * cp[..., None]).abs()) \
        + U * dcos.abs()
    if pad is None:
        a_mse, a_cos = 2.0 / (B * L * D), w / (B * L)
    else:
        den = n_valid.clamp_min(1.0)[:, None, None]
        a_mse, a_cos = 2.0 / (den * D * B), w / (den * B)
    inner = a_mse * (p - t) - a_cos * dcos
    e_in = abs(a_mse) * 6 * U * (p - t).abs() if pad is None else a_mse.abs() * 6 * U * (p - t).abs()
    e_in = e_in + abs(a_cos) * (e_dcos + 6 * U * dcos.abs()) if pad is None else e_in + a_cos.abs() * (e_dcos + 6 * U * dcos.abs())
    e = abs(g) * (e_in + U * inner.abs()) + 3 * U * ref.abs()
    if pad is not None:
        e = e * (~pad)[..., None]
    return ref, _out(ref, e, False)


def consistency_fwd(p, q, weight, loss0):
    """es3_text_consistency_fwd: mdiff = fl(sum_l p / L) - fl(sum_l q / L) per (b, c), ws[b] = sum_c mdiff^2 (of the kernel's fp32
    mdiff), value = sum_b ws / (B D), loss = loss0 + weight value.  Returns dict name -> (ref, bound)."""
    B, L, D = p.shape
    mp, mq = p.mean(1), q.mean(1)
    md = mp - mq
    e_md = GAMMA * L * U * (p.abs().sum(1) + q.abs().sum(1)) / L + U * (mp.abs() + mq.abs() + md.abs())
    part = (md * md).sum(1)
    e_part = (2 * md.abs() * e_md + e_md * e_md).sum(1) + GAMMA * (D + 14) * U * part
    value = part.sum() / (B * D)
    e_value = (e_part.sum() + GAMMA * (B + 1) * U * part.sum()) / (B * D) + U * value
    loss = loss0 + weight * value
    e_loss = abs(weight) * e_value + 2 * U * (abs(weight) * value + loss.abs())
    return {"mdiff": (md, _out(md, e_md, False)), "ws": (part, _out(part, e_part, False)),
            "value": (value.reshape(1), _out(value.reshape(1), e_value.reshape(1), False)),
            "loss": (loss.reshape(1), _out(loss.reshape(1), e_loss.reshape(1), False))}


def consistency_bwd(mdiff, L, weight, g, dp0):
    """es3_text_consistency_bwd on the mdiff [B, D] it is given: v = 2 weight g mdiff / (B D L) per (b, l, c); dp = dp0 + v (+=),
    dq = -v.  k = fl(2 weight g / (B D L)) rounds up to five times (g's two products, 2 weight g, the division), then v and dp."""
    B, D = mdiff.shape
    v = (2 * weight * g / (B * D * L) * mdiff)[:, None, :].expand(B, L, D)
    dp = dp0 + v
    return {"dp": (dp, _out(dp, 6 * U * v.abs() + U * dp.abs(), False)), "dq": (-v, _out(-v, 6 * U * v.abs(), False))}


# ------------------------------------------------------------------------------------------------ RepMixerBlock backward (frozen BN)
def _shift(x, j, B, L):
    """Row (b, l) of the result is row (b, l + j) of x [B L, C], zero outside the sequence."""
    C = x.shape[1]
    xs = F.pad(x.reshape(B, L, C), (0, 0, 5, 5))
    return xs[:, 5 + j:5 + j + L].reshape(B * L, C)


def _acc_out(ref0, s, terms, extra, n):
    """ref0 + s with |terms| the absolute terms of the fixed-order sum s (n roundings deep) and `extra` the error already in them."""
    ref = ref0 + s
    return ref, _out(ref, extra + GAMMA * n * U * (ref0.abs() + terms), False)


def repmixer_ls_bwd(g, y, ls, B, L, dls0, db0):
    """es3_repmixer_ls_bwd: dy = bf16(fl(ls g)); dls += sum g y, dbias += sum fl(ls g) over the B L rows (per-CTA row groups,
    then the sequences in order: L + B + 10 roundings deep at most)."""
    n = L + B + 10
    d = ls * g
    return {"dy": (d, _out(d, U * d.abs(), True)),
            "dls": _acc_out(dls0, (g * y).sum(0), (g * y).abs().sum(0), 0.0, n),
            "dbias": _acc_out(db0, d.sum(0), d.abs().sum(0), U * d.abs().sum(0), n)}


def repmixer_ffn_bwd(x1, du, g, wf, bnf, B, L, dwf0, dg0, db0):
    """es3_repmixer_ffn_bwd on the packed bnf [4, C] = (s, b, rm, invstd) and the raw taps wf [11, C]: f = dw(x1; wf) (11-term FMA
    chain), e = fmaf(s, dw^T(du; wf), g); dwf[c, k] += s sum_l du[l] x1[l + k - 5] (s applied to each CTA's partial);
    dgamma += sum du (f - rm) invstd, dbeta += sum du.  dwf0 [C, 11] (the [C, 1, 1, 11] gradient's layout)."""
    n = L + B + 10
    s, rm, inv = bnf[0], bnf[2], bnf[3]
    xs = [_shift(x1, k - 5, B, L) for k in range(11)]
    f = sum(wf[k] * xs[k] for k in range(11))
    e_f = GAMMA * 11 * U * sum(wf[k].abs() * xs[k].abs() for k in range(11))
    ds = [_shift(du, 5 - k, B, L) for k in range(11)]
    t = sum(wf[k] * ds[k] for k in range(11))
    e_t = GAMMA * 11 * U * sum(wf[k].abs() * ds[k].abs() for k in range(11))
    e = g + s * t
    out = {"e": (e, _out(e, s.abs() * e_t + U * e.abs(), False))}
    tap = torch.stack([(du * xs[k]).sum(0) for k in range(11)], 1)              # [C, 11]
    tap_t = torch.stack([(du * xs[k]).abs().sum(0) for k in range(11)], 1)
    sc = s[:, None]
    out["dwf"] = _acc_out(dwf0, sc * tap, sc.abs() * tap_t, 2 * U * sc.abs() * tap_t, n + 1)
    fh = (f - rm) * inv
    e_fh = inv.abs() * (e_f + U * (f - rm).abs()) + U * fh.abs()
    out["dgamma"] = _acc_out(dg0, (du * fh).sum(0), (du * fh).abs().sum(0), (du.abs() * e_fh).sum(0), n)
    out["dbeta"] = _acc_out(db0, du.sum(0), du.abs().sum(0), 0.0, n)
    return out


def repmixer_tm_bwd(x, e, wmc, bnp, B, L, dwmc0, dls0, dbn0):
    """es3_repmixer_tm_bwd on the packed bnp [13, C] = (s, b, rm, invstd) of BN_ms, BN_mc, BN_ns, then ls_tm, and the raw taps wmc:
    c = dw(x; wmc), r = (s_ms - s_ns) x + s_mc c + (b_ms + b_mc - b_ns) (the kernel's fp32 sd and br, two fmas), e' = fl(ls e),
    dc = fl(s_mc e'); dx = fmaf(sd, fl(ls e), e) + dw^T(dc; wmc), fp32 (its bf16 copy is bf16(dx32) exactly);
    dwmc[c, k] += sum dc[l] x[l + k - 5], dls += sum e r, dgamma_ms += sum e' xhat_ms, dgamma_ns -= sum e' xhat_ns,
    dgamma_mc += sum e' chat, dbeta_ms += sum e', dbeta_mc += sum e', dbeta_ns -= sum e'.  dbn0 = (dg_ms, db_ms, dg_mc, db_mc,
    dg_ns, db_ns).  Returns dict name -> (ref, bound)."""
    n = L + B + 10
    s_ms, b_ms, rm_ms, inv_ms, s_mc, b_mc, rm_mc, inv_mc, s_ns, b_ns, rm_ns, inv_ns, ls = bnp
    sd, br = s_ms - s_ns, b_ms + b_mc - b_ns
    e_sd, e_br = U * sd.abs(), 2 * U * (b_ms.abs() + b_mc.abs() + b_ns.abs())
    xs = [_shift(x, k - 5, B, L) for k in range(11)]
    cv = sum(wmc[k] * xs[k] for k in range(11))
    e_cv = GAMMA * 11 * U * sum(wmc[k].abs() * xs[k].abs() for k in range(11))
    inner = s_mc * cv + br
    r = sd * x + inner
    e_r = e_sd * x.abs() + s_mc.abs() * e_cv + e_br + U * (inner.abs() + r.abs())
    ep = ls * e
    e_ep = U * ep.abs()
    dc = s_mc * ep
    e_dc = 2 * U * dc.abs()
    dcs = [_shift(dc, 5 - k, B, L) for k in range(11)]
    edcs = [_shift(e_dc, 5 - k, B, L) for k in range(11)]
    t = sum(wmc[k] * dcs[k] for k in range(11))
    e_t = sum(wmc[k].abs() * (edcs[k] + GAMMA * 11 * U * dcs[k].abs()) for k in range(11))
    dx = e + sd * ep + t
    e_dx = (e_sd + U * sd.abs()) * ep.abs() + U * (e + sd * ep).abs() + e_t + U * dx.abs()
    out = {"dx": (dx, _out(dx, e_dx, False))}
    tap = torch.stack([(dc * xs[k]).sum(0) for k in range(11)], 1)
    tap_t = torch.stack([(dc * xs[k]).abs().sum(0) for k in range(11)], 1)
    tap_e = torch.stack([(e_dc * xs[k].abs()).sum(0) for k in range(11)], 1)
    out["dwmc"] = _acc_out(dwmc0, tap, tap_t, tap_e, n)
    out["dls"] = _acc_out(dls0, (e * r).sum(0), (e * r).abs().sum(0), (e.abs() * e_r).sum(0), n)

    def hat(v, e_v, rm, inv):
        h = (v - rm) * inv
        return h, inv.abs() * (e_v + U * (v - rm).abs()) + U * h.abs()
    h_ms, eh_ms = hat(x, 0.0, rm_ms, inv_ms)
    h_ns, eh_ns = hat(x, 0.0, rm_ns, inv_ns)
    h_mc, eh_mc = hat(cv, e_cv, rm_mc, inv_mc)
    dg_ms0, db_ms0, dg_mc0, db_mc0, dg_ns0, db_ns0 = dbn0

    def gsum(h, eh, sign, ref0):
        return _acc_out(ref0, sign * (ep * h).sum(0), (ep * h).abs().sum(0), (e_ep * h.abs() + ep.abs() * eh).sum(0), n)
    out["dg_ms"] = gsum(h_ms, eh_ms, 1, dg_ms0)
    out["dg_mc"] = gsum(h_mc, eh_mc, 1, dg_mc0)
    out["dg_ns"] = gsum(h_ns, eh_ns, -1, dg_ns0)
    for name, sign, ref0 in (("db_ms", 1, db_ms0), ("db_mc", 1, db_mc0), ("db_ns", -1, db_ns0)):
        out[name] = _acc_out(ref0, sign * ep.sum(0), ep.abs().sum(0), e_ep.sum(0), n)
    return out
