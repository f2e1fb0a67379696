"""fp64 statements of the stage-1 KD step's loss and optimiser kernels (kd_loss.cu: es3_kd_loss_fwd; train_ops.cu: es3_kd_loss_bwd,
es3_grad_norm, es3_adamw_flat with its scaler update) and, next to each, the per-element bound its fp32 arithmetic keeps to.

The bound form is ref_train_bwd.py's and ref_text.py's: an fp32 sum of n terms is held to GAMMA n u sum |terms| (n = the number of
roundings a term goes through on its way to the result: its FMA chain, then the warp tree, the warps of a block, the blocks), an fp32
result adds 4u |ref| for its own rounding (_out), every other intermediate is propagated to first order and named where it is
charged.  Operands are the ones the kernels receive: fp32 tensors, and the scalars of the C ABI rounded to fp32.  Every function
takes and returns float64 tensors (CPU or CUDA) unless it says otherwise.  tests/test_stage1_kernels_cpu.py ties each statement to
the oracle's loss (oracle/kd_loss.py), torch autograd, torch.optim.AdamW and torch.amp.GradScaler in float64.

The valid mask is exact: the bilinear weights of an integer-sized resize are rationals with denominator 2E, so the statement uses
integer arithmetic and the kernels' fp32 mask must equal it bit for bit.
"""
import numpy as np
import torch
import torch.nn.functional as F

from bounds import U
from ref_train_bwd import GAMMA, _out

COS_EPS = float(torch.tensor(1e-8, dtype=torch.float32))   # the fp32 value of 1e-8 both kernels clamp the norms to
WARP_TREE, BLOCK_WARPS = 5, 8       # kd_loss_partial_kernel / grad_sumsq_partial_kernel: a 32-lane xor tree, then 8 warps in order
KD_PIX = 256                        # pixels per kd_loss_partial_kernel block
GN_ELEMS, GN_MAX_BLOCKS = 256 * 4 * 16, 4096   # es3_grad_norm_ws_floats: elements per block before the grid cap, and the cap
POWF_ULP = 4                        # powf: 4 ulp (CUDA C++ Programming Guide, single-precision functions); an ulp is <= 2u |result|
RSQRTF_ULP = 2                      # rsqrtf: 2 ulp (same table)


# ------------------------------------------------------------------------------------------------ valid mask (build_valid_mask)
def _axis_weights(img, E, extent):
    """Along one axis: 2E x the bilinear weight that the [i < extent] indicator resized img -> E (align_corners=False) gives each
    output index, as integers.  The source coordinate of output o is f = ((2o + 1) img - E) / (2E), clamped at 0; i0 = floor(f),
    i1 = min(i0 + 1, img - 1), lambda = f - i0 (the index clamps of kd_valid_mask_at and of torch's upsample_bilinear2d)."""
    o = np.arange(E, dtype=np.int64)
    num = np.maximum((2 * o + 1) * img - E, 0)                 # 2E f
    i0 = np.minimum(num // (2 * E), img - 1)
    i1 = np.minimum(i0 + 1, img - 1)
    lam = num - 2 * E * i0                                     # 2E lambda
    return (2 * E - lam) * (i0 < extent) + lam * (i1 < extent)


def valid_mask(img, E, h, w):
    """build_valid_mask of one image h x w before padding: [E, E] bool.  The indicator is separable, so the resized value at (y, x)
    is wy wx / (2E)^2 and the mask is 2 wy wx > (2E)^2, decided exactly (a tie at 1/2 is not valid, as `> 0.5`)."""
    wy, wx = _axis_weights(img, E, h), _axis_weights(img, E, w)
    return torch.from_numpy(2 * wy[:, None] * wx[None, :] > (2 * E) ** 2)


def valid_masks(img, E, sizes_hw):
    """[B, E, E] bool for int (h, w) rows."""
    return torch.stack([valid_mask(img, E, int(h), int(w)) for h, w in sizes_hw])


# ------------------------------------------------------------------------------------------------ forward
def _pixel_stats(p, t):
    """Per pixel of [B, C, E, E]: d2, dot, |p|, |t| (fp32 FMA chains over C; the difference rounded before it is squared) and the
    bounds of d2 and dot, and rel_n, the relative bound of |p| and |t| (half the chain's, plus sqrtf's rounding)."""
    C = p.shape[1]
    d2 = ((p - t) ** 2).sum(1)
    dot = (p * t).sum(1)
    e_dot = GAMMA * C * U * (p * t).abs().sum(1)
    return d2, (GAMMA * C + 2) * U * d2, dot, e_dot, p.norm(dim=1), t.norm(dim=1), GAMMA * C * U / 2 + U


def cos_terms(p, t):
    """Per pixel: (1 - cos, its bound), cos = dot / (max(|p|, eps) max(|t|, eps)) as F.cosine_similarity; the product of the clamped
    norms and the division each round once."""
    _, _, dot, e_dot, np_, nt, rel_n = _pixel_stats(p, t)
    den = np_.clamp_min(COS_EPS) * nt.clamp_min(COS_EPS)
    cos = dot / den
    cl = 1 - cos
    return cl, e_dot / den + cos.abs() * (2 * rel_n + 2 * U) + U * cl.abs()


def _nblk(E):
    return -(-E * E // KD_PIX)


def kd_fwd(p, t, mask, w):
    """es3_kd_loss_fwd on [B, C, E, E] operands and the [B, E, E] valid mask.  Returns dict name -> (ref, bound):
    "ws" [B, nblk, 3] block partials (sum valid d2, sum valid (1 - cos), valid count) -- a warp tree and 8 warps in order;
    "per_sample" [B, 3] = (mse_b, cos_b, count_b), the sums over the blocks in order divided by max(count, 1) -- counts exact;
    "out3" [3] = (loss, mse, cos), the samples in order divided by B, loss = mse + w cos."""
    B, C, E, _ = p.shape
    nb = _nblk(E)
    d2, e_d2, _, _, _, _, _ = _pixel_stats(p, t)
    cl, e_cl = cos_terms(p, t)
    v = mask.to(p.dtype)

    def blocks(x):                                             # [B, E, E] -> [B, nblk] per-block sums in fp64
        flat = torch.zeros(B, nb * KD_PIX, dtype=x.dtype, device=x.device)
        flat[:, :E * E] = x.reshape(B, -1)
        return flat.view(B, nb, KD_PIX).sum(-1)
    sq, cls, cnt = blocks(v * d2), blocks(v * cl), blocks(v)
    blk_depth = WARP_TREE + BLOCK_WARPS
    e_sq = blocks(v * e_d2) + GAMMA * blk_depth * U * sq
    e_cls = blocks(v * e_cl) + GAMMA * blk_depth * U * blocks(v * cl.abs())
    ws = torch.stack([sq, cls, cnt], -1)
    out = {"ws": (ws, _out(ws, torch.stack([e_sq, e_cls, torch.zeros_like(cnt)], -1), False))}
    depth = blk_depth + nb                                     # then nblk blocks in order
    S, Cl, N = sq.sum(1), cls.sum(1), cnt.sum(1)
    eS = e_sq.sum(1) + GAMMA * depth * U * S
    eC = e_cls.sum(1) + GAMMA * depth * U * blocks(v * cl.abs()).sum(1)
    den = N.clamp_min(1.0)
    mse_b, cos_b = S / den, Cl / den
    e_mse_b, e_cos_b = eS / den + U * mse_b.abs(), eC / den + U * cos_b.abs()      # the division rounds once
    per = torch.stack([mse_b, cos_b, N], 1)
    out["per_sample"] = (per, _out(per, torch.stack([e_mse_b, e_cos_b, torch.zeros_like(N)], 1), False))
    mse, cos = mse_b.mean(), cos_b.mean()
    e_mse = (e_mse_b.sum() + GAMMA * (B + 1) * U * mse_b.abs().sum()) / B          # B in order, then / B
    e_cos = (e_cos_b.sum() + GAMMA * (B + 1) * U * cos_b.abs().sum()) / B
    loss = mse + w * cos
    e_loss = e_mse + abs(w) * e_cos + 2 * U * (mse.abs() + abs(w) * cos.abs())     # w cos and the sum each round once
    o3 = torch.stack([loss, mse, cos])
    out["out3"] = (o3, _out(o3, torch.stack([e_loss, e_mse, e_cos]), False))
    return out


def kd_loss64(p, t, mask, w):
    """The stage-1 KD loss in float64 torch (masked_mse + w masked_cosine_loss of train_image_encoder_stage1.py, the oracle's
    kd_loss on a given mask), F.cosine_similarity with the kernels' fp32 eps."""
    v = mask.to(p.dtype)[:, None]
    den = v.sum((1, 2, 3)).clamp_min(1.0)
    mse = (((p - t) * v) ** 2).sum((1, 2, 3)) / den
    cos = ((1 - F.cosine_similarity(p, t, dim=1, eps=COS_EPS)) * v[:, 0]).sum((1, 2)) / den
    return mse.mean() + w * cos.mean()


# ------------------------------------------------------------------------------------------------ backward
def kd_bwd(p, t, mask, w, g):
    """es3_kd_loss_bwd: d kd_loss64 / dp by float64 autograd times g = grad_scale scale_dev[0] (masked pixels get exactly 0).  The
    bound follows the kernel's explicit form dp = k_mse (p - t) + k_t t + k_a p with
        up = g / (B max(count, 1)),  k_mse = 2 up,  k_t = -w up / (np' nt'),  k_a = w up dot / (np'^2 nt' |p|)  (0 at p = 0),
    np' = max(|p|, eps): up rounds three times (g's product, B count, the division), k_t three more, k_a six more (w up, its product
    with dot, np' np', |p|, nt', the division); each of the three products with p - t (itself rounded), t and p rounds once and the
    two additions round once each."""
    B, C, E, _ = p.shape
    pr = p.clone().requires_grad_(True)
    with torch.enable_grad():
        (ref,) = torch.autograd.grad(kd_loss64(pr, t, mask, w), pr)
    ref = g * ref
    _, _, dot, e_dot, np_, nt, rel_n = _pixel_stats(p, t)
    npc, ntc = np_.clamp_min(COS_EPS), nt.clamp_min(COS_EPS)
    den = mask.to(p.dtype).sum((1, 2)).clamp_min(1.0)[:, None, None]
    up = abs(g) / (B * den)
    r_up = 3 * U
    k_t = abs(w) * up / (npc * ntc)
    r_kt = r_up + 3 * U + 2 * rel_n
    pos = np_ > 0
    k_a = torch.where(pos, abs(w) * up * dot.abs() / (npc * npc * ntc * np_.clamp_min(1e-300)), torch.zeros_like(dot))
    e_ka = torch.where(pos, k_a * (r_up + 6 * U + 4 * rel_n) + abs(w) * up * e_dot / (npc * npc * ntc * np_.clamp_min(1e-300)),
                       torch.zeros_like(dot))
    T1 = 2 * up[:, None] * (p - t).abs()
    T2 = (k_t[:, None] * t).abs()
    T3 = (k_a[:, None] * p).abs()
    e = T1 * (r_up + 4 * U) + T2 * (r_kt + 3 * U) + T3 * 3 * U + e_ka[:, None] * p.abs() + U * ref.abs()
    e = e * mask[:, None].to(p.dtype)
    return ref, _out(ref, e, False)


# ------------------------------------------------------------------------------------------------ gradient norm
def gn_blocks(n):
    """es3_grad_norm's grid: min(4096, ceil(n / 16384)) blocks of 256 threads, each thread reads float4s at a stride of the grid."""
    return min(GN_MAX_BLOCKS, max(1, -(-n // GN_ELEMS)))


def grad_norm(g):
    """es3_grad_norm on a flat fp32 arena: (sum g^2 in fp64, its bound, non-finite flag).  A thread's FMA chain is 4 terms per float4
    it reads, ceil(n / (4 blocks 256)) float4s at most; then the warp tree and 8 warps; the block partials are summed in double
    (2^-53 per term, charged as u) and the total rounds to fp32 once."""
    g = g.double()
    n = g.numel()
    finite = bool(torch.isfinite(g).all())
    g = torch.where(torch.isfinite(g), g, torch.zeros_like(g))
    s = float((g * g).sum())
    chain = 4 * -(-n // (4 * gn_blocks(n) * 256))
    depth = chain + WARP_TREE + BLOCK_WARPS + 1
    return s, GAMMA * depth * U * s + 4 * U * s + 1e-30, 0.0 if finite else 1.0


# ------------------------------------------------------------------------------------------------ AdamW + GradScaler
def f32(x):
    """A Python scalar as the C ABI delivers it: rounded to fp32 (returned as a Python float)."""
    return float(np.float32(x))


def adamw(p, g, m, v, n_decay, lr, betas, eps, wd, max_norm, inv_world, sumsq, scale, step):
    """es3_adamw_flat's update of one unskipped step in fp64 from the fp32 operands and ABI scalars (pass them through f32 for the
    kernel; as doubles, this is torch.optim.AdamW after GradScaler.unscale_ and clip_grad_norm_):
        inv_scale = inv_world / scale, total = sqrt(sumsq) inv_scale, coef = min(max_norm / (total + 1e-6), 1) (max_norm > 0),
        g' = g inv_scale coef, t = step + 1, p *= 1 - lr wd (the first n_decay elements), m = b1 m + (1 - b1) g',
        v = b2 v + (1 - b2) g'^2, p -= lr / (1 - b1^t) m / (sqrt(v) / sqrt(1 - b2^t) + eps).
    sumsq: the fp32 norm_ws[0] the kernel reads; scale, step: state[0] and state[2].  Returns dict name -> (ref, bound) for p, m and v.  1 - b is exact in fp32 for b in [1/2, 1] (Sterbenz), so it costs nothing.
    The bias corrections carry powf's error: POWF_ULP ulp of b^t, divided by 1 - b^t -- the cancellation makes it ~1e-4 relative
    at t = 1 with b2 = 0.999."""
    b1, b2 = betas
    inv_scale = inv_world / scale
    total = sumsq ** 0.5 * inv_scale
    r_tot = 4 * U                                              # inv_scale, sqrtf, the product, + 1e-6
    coef, r_coef = 1.0, 0.0
    if max_norm > 0:
        c = max_norm / (total + 1e-6)
        coef = min(c, 1.0)
        if c * (1 - r_tot - U) < 1.0:                          # fminf(c, 1) with c off by (r_tot + u) c: within that of the clamp
            r_coef = c * (r_tot + U) / coef
    gm = inv_scale * coef
    r_g = U + r_coef + U + U                                   # inv_scale, coef, gmul, g * gmul
    t = step + 1.0
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    r_bc1 = (POWF_ULP * 2 * U * b1 ** t + U * bc1) / bc1
    r_bc2 = (POWF_ULP * 2 * U * b2 ** t + U * bc2) / bc2
    gp = g * gm
    m1 = b1 * m + (1 - b1) * gp
    e_m = 2 * U * (b1 * m).abs() + ((1 - b1) * gp).abs() * (r_g + 2 * U) + U * m1.abs()
    v1 = b2 * v + (1 - b2) * gp * gp
    e_v = 2 * U * (b2 * v).abs() + ((1 - b2) * gp * gp) * (2 * r_g + 3 * U) + U * v1.abs()
    sq = v1.sqrt()
    isb = bc2 ** -0.5
    denom = sq * isb + eps
    e_sq = torch.minimum(e_v / (2 * sq.clamp_min(1e-300)), e_v.sqrt()) + U * sq      # |sqrt a - sqrt b| <= sqrt |a - b| as well
    e_den = e_sq * isb + sq * isb * (r_bc2 / 2 + RSQRTF_ULP * 2 * U + U) + U * denom
    dec = torch.zeros_like(p, dtype=torch.bool)
    dec[:n_decay] = True
    fac = 1 - lr * wd
    pd = torch.where(dec, p * fac, p)
    e_pd = torch.where(dec, p.abs() * (U * lr * wd + 2 * U * abs(fac)), torch.zeros_like(p))     # lr wd, 1 - lr wd, the product
    ss = lr / bc1
    q = m1 / denom
    e_q = e_m / denom + q.abs() * (e_den / denom + U)
    upd = ss * q
    e_upd = abs(ss) * e_q + upd.abs() * (r_bc1 + 2 * U)
    p1 = pd - upd
    e_p = e_pd + e_upd + U * p1.abs()
    return {"p": (p1, _out(p1, e_p, False)), "m": (m1, _out(m1, e_m, False)), "v": (v1, _out(v1, e_v, False))}


def scaler_state(state, sumsq32, bad, inv_world32, dynamic, growth_interval, growth=2.0, backoff=0.5):
    """scaler_update_kernel on [scale, growth tracker, step count, last norm] (fp32 numpy array), exactly: GradScaler.update moves
    the scale by powers of two and counts in integers; the last norm is sqrtf(sumsq) inv_world / scale in fp32 (inf when skipped)."""
    s = np.array(state, dtype=np.float32)
    f = np.float32
    s[3] = np.inf if bad else f(f(np.sqrt(f(sumsq32))) * f(inv_world32)) / s[0]
    if not bad:
        s[2] += f(1)
    if dynamic:
        if bad:
            s[0] *= f(backoff)
            s[1] = 0
        else:
            s[1] += f(1)
            if int(s[1]) >= growth_interval:
                s[0] *= f(growth)
                s[1] = 0
    return s
