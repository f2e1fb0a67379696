"""fp64 statements of the SAM3 ViT trunk's kernels (attention.cu and attention_tc.cu at the trunk's windowed and global shapes,
vit_ops.cu's patch im2col and token layout change, and the strict-mode twins of strict_f32.cu: sgemm_f32, im2col_f32, ln_rows_f32,
rope_f32, attention_f32) and, next to each, the per-element bound its fp32 arithmetic keeps to.

The bound form is ref_fwd.py's, ref_text.py's and ref_sam.py's: an fp32 sum of n terms is held to GAMMA n u sum |terms|, an fp32 result
adds 4u |ref| and a bf16 result 2^-8 |ref| for its own rounding (_out).  Operands are the ones the kernel reads (bf16 qkv, fp32 rows
and tables).  Every function takes and returns float64 tensors (CPU or CUDA); the attention statements work one head at a time so
that the [L, L] temporaries of a 72 x 72 global block (L = 5184, 215 MB each in fp64) stay a few of them.
tests/test_vit_kernels_cpu.py ties each statement to textbook float64 torch, oracle/vitdet.py's window partition and
tests/emu_strict.py.
"""
import torch
import torch.nn.functional as F

from bounds import L_ACT, U, _act64, _eps_act
from ref_fwd import layernorm, softmax_attn, win_tokens
from ref_sam import _softmax_weighted
from ref_text import EXPF_REL
from ref_train_bwd import GAMMA, _out

CELLS = 1 << 26                # [windows, L, L] fp64 cells per statement chunk (512 MB)


# ------------------------------------------------------------------------------------------------ token maps
def tokens(B, H, W, win):
    """[B nwin, L] token rows of each (image, window) in the kernel's order: windows raster over the win x win grid, then the
    window's tokens raster inside it (-1: a padded position of an overhanging window); win = 0: one window of H W tokens."""
    if win == 0:
        return torch.arange(B * H * W).view(B, H * W)
    return win_tokens(B, H, W, win)


def bn_tile(L):
    """attn_tc_kernel's key tile: 96 for multiples of 96 that are not multiples of 128 (the 24 x 24 windows), else 128."""
    return 96 if L % 96 == 0 and L % 128 != 0 else 128


def _scatter(y, e, tok, n_rows):
    """Rows of y, e [nwin, L, C] back to token order (padded positions dropped)."""
    C = y.shape[-1]
    flat = tok.reshape(-1).to(y.device)
    keep = flat >= 0
    out = torch.full((n_rows, C), float("nan"), dtype=y.dtype, device=y.device)
    err = torch.full_like(out, float("nan"))
    out[flat[keep]] = y.reshape(-1, C)[keep]
    err[flat[keep]] = e.reshape(-1, C)[keep]
    return out, err


def _chunks(nwin, L):
    step = max(1, CELLS // (L * L))
    return [(i, min(nwin, i + step)) for i in range(0, nwin, step)]


# ------------------------------------------------------------------------------------------------ bf16 attention
def attention_bf16(qkv, B, H, W, heads, win, scale, kernel):
    """es3_attention_tc_bf16 (kernel "tc": attn_tc_kernel, key tiles of bn_tile(L)) / es3_attention_mma_bf16 ("mma": attn_fwd_kernel,
    key tiles of 64) on qkv [B H W, 3C] bf16 values, head_dim 64: per (image, window, head) ref_fwd.softmax_attn with the ex2 exponent
    and the kernel's online-softmax tiles, bf16 store in token order.  Returns (ref, bound) [B H W, C]."""
    C = heads * 64
    tok = tokens(B, H, W, win).to(qkv.device)
    nwin, L = tok.shape
    kv_tile = 64 if kernel == "mma" else bn_tile(L)
    y = torch.empty(nwin, L, C, dtype=qkv.dtype, device=qkv.device)
    e = torch.empty_like(y)
    for a, b in _chunks(nwin, L):
        rows = qkv[tok[a:b]]                                              # [n, L, 3C]
        for h in range(heads):
            q, k, v = (rows[..., i * C + 64 * h:i * C + 64 * (h + 1)] for i in range(3))
            y[a:b, :, 64 * h:64 * (h + 1)], e[a:b, :, 64 * h:64 * (h + 1)] = softmax_attn(q, k, v, scale, ex2=True, kv_tile=kv_tile)
    out, err = _scatter(y, e, tok, B * H * W)
    return out, _out(out, err, True)


# ------------------------------------------------------------------------------------------------ exact operations
def im2col_patch(x, P, Kp):
    """es3_im2col_patch: x [B, 3, S, S] fp32 -> [B (S/P)^2, Kp] bf16 values, column c P^2 + ky P + kx, zero columns from 3 P^2."""
    cols = F.unfold(x, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)
    return F.pad(cols.to(torch.bfloat16), (0, Kp - 3 * P * P))


def im2col_f32(x, ks, stride, pad, nchw):
    """es3_im2col_f32: x NCHW (nchw) or NHWC -> [B Ho Wo, ks^2 C], column (ky ks + kx) C + c, zero outside the image."""
    xn = x if nchw else x.permute(0, 3, 1, 2)
    B, C = xn.shape[:2]
    cols = F.unfold(xn, ks, padding=pad, stride=stride)                  # [B, C ks^2, Ho Wo], row c ks^2 + tap
    return cols.view(B, C, ks * ks, -1).permute(0, 3, 2, 1).reshape(-1, ks * ks * C)


def tokens_to_nchw(x, B, HW, C):
    """es3_tokens_f32_to_nchw: [B HW, C] -> [B, C, HW]."""
    return x.view(B, HW, C).permute(0, 2, 1)


# ------------------------------------------------------------------------------------------------ strict mode
def sgemm(a, w, scale=None, bias=None, act=None, residual=None, after=False):
    """es3_sgemm_f32: out = act(scale fl(a w^T) + bias) (+ residual), or act(... + residual) when `after`.  The accumulator is an fmaf
    chain of K terms from 0 on fp32 operands (no operand rounding): GAMMA K u |a| |w|^T; the scale, bias and residual each round
    once (4u of their operands, as tests/test_gemm_epilogue_gpu.py states it), the activation carries the error through L_ACT and
    adds its own."""
    K = a.shape[1]
    acc, absprod = a @ w.t(), a.abs() @ w.abs().t()
    s = scale if scale is not None else 1.0
    pre = acc * s
    inner = GAMMA * K * U * absprod * (scale.abs() if scale is not None else 1.0) + 4 * U * pre.abs()
    if bias is not None:
        pre = pre + bias
        inner = inner + 4 * U * bias.abs()
    if residual is not None and after:
        pre = pre + residual
        inner = inner + 4 * U * residual.abs()
    ref = _act64(pre, act)
    if residual is not None and not after:
        ref = ref + residual
    bound = L_ACT[act] * (inner + _eps_act(pre, act)) + 4 * U * ref.abs() + 2.0 ** -126
    return ref, bound


def rope(qkv, table, rope_cols, H, W, win):
    """es3_rope_f32 on qkv [M, >= rope_cols]: pair (2i, 2i + 1) of every 64-column head in [0, rope_cols) becomes
    (x0 c - x1 s, x0 s + x1 c), (c, s) = table[pos, i]; pos = the token's index (win = 0) or its index inside its window.  Two
    products and one sum per element: GAMMA 2 u (|x0 c| + |x1 s|).  Returns (ref, bound) of columns [0, rope_cols)."""
    M = qkv.shape[0]
    t = torch.arange(M, device=qkv.device) % (H * W)
    h, w = t // W, t % W
    pos = (h % win) * win + (w % win) if win else t
    cs = table[pos]                                                       # [M, 32, 2]
    x = qkv[:, :rope_cols].reshape(M, rope_cols // 64, 32, 2)
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    x0, x1 = x[..., 0], x[..., 1]
    ref = torch.stack([x0 * c - x1 * s, x0 * s + x1 * c], -1).reshape(M, rope_cols)
    terms = torch.stack([(x0 * c).abs() + (x1 * s).abs(), (x0 * s).abs() + (x1 * c).abs()], -1).reshape(M, rope_cols)
    return ref, _out(ref, GAMMA * 2 * U * terms, False)


def ln_rows(x, w, b, eps):
    """es3_ln_rows_f32 over rows x [M, C] of any width: lane-strided sums then a warp tree (GAMMA C u), mean = fl(sum / C), the
    centred variance as an fmaf chain of fl(x - mean)^2, rstd = 1 / sqrtf(fl(q / C) + eps) (four correct roundings); y =
    fl(fl(x - mean) rstd) w + b with the product by w rounded before the add (the u |xh w| term) -- ref_fwd.layernorm's fp32 form
    otherwise, as ref_text.layernorm_f32 uses it."""
    ref, bound = layernorm(x, w, b, eps, bf16=False)
    mu = x.mean(1, keepdim=True)
    xh = (x - mu) * ((x - mu).pow(2).mean(1, keepdim=True) + eps).rsqrt()
    return ref, bound + U * (xh * w).abs()


def rises(s, err):
    """Per row of s [..., N, L]: how many keys j >= 1 may raise attn_f32_kernel's running maximum -- s_j above the maximum of the
    keys before it, less twice the row's score error (the fp32 scores may tie or swap where fp64 ones differ by less)."""
    prev = torch.cummax(s, -1).values[..., :-1]
    return (s[..., 1:] > prev - 2 * err).sum(-1, keepdim=True).to(s.dtype)


def attention_f32(qkv, B, H, W, heads, hd, win, scale, layout="blocks", bias=None, pad_row=None):
    """es3_attention_f32: one thread per query; qs = fl(q scale), each score an fmaf chain of hd terms of qs k (+ bias, one
    rounding), then one sequential online softmax over the keys in order with libm expf: p = expf(fl(s - m)), l += p, o = fmaf(p,
    v, o); where a score beats the running maximum, l and o are multiplied by expf(fl(m_old - s)) (its argument, its expf and the
    product: EXPF_REL + u A + 2u, A the row's score range), which happens rises() times per row.  The end divides by l (2u).
    layout "blocks": q | k | v column blocks of heads hd; "per_head": (q, k, v) triples per head.  Windows that overhang the grid
    take pad_row for the missing tokens, whose outputs are not stored.  Returns (ref, bound) [B H W, heads hd]."""
    C = heads * hd
    tok = tokens(B, H, W, win).to(qkv.device)
    nwin, L = tok.shape
    src = torch.cat([qkv, (pad_row if pad_row is not None else torch.zeros_like(qkv[0]))[None]], 0)
    idx = torch.where(tok >= 0, tok, torch.full_like(tok, qkv.shape[0]))
    y = torch.empty(nwin, L, C, dtype=qkv.dtype, device=qkv.device)
    e = torch.empty_like(y)
    for a, b in _chunks(nwin, L):
        rows = src[idx[a:b]]
        for h in range(heads):
            if layout == "blocks":
                q, k, v = (rows[..., i * C + hd * h:i * C + hd * (h + 1)] for i in range(3))
            else:
                q, k, v = (rows[..., 3 * hd * h + i * hd:3 * hd * h + (i + 1) * hd] for i in range(3))
            s = scale * q @ k.transpose(-1, -2)
            e_s = abs(scale) * (GAMMA * hd + 1) * U * (q.abs() @ k.abs().transpose(-1, -2))
            if bias is not None:
                s = s + bias[h]
                e_s = e_s + U * s.abs()
            err = e_s.amax(-1, keepdim=True)
            A = s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True)
            n = rises(s, err)
            yy, ee = _softmax_weighted(s, e_s, v, lambda arg: EXPF_REL + 0 * arg, n, EXPF_REL + U * A + 2 * U, L, L)
            y[a:b, :, hd * h:hd * (h + 1)], e[a:b, :, hd * h:hd * (h + 1)] = yy, ee
    out, err = _scatter(y, e, tok, B * H * W)
    return out, _out(out, err, False)
