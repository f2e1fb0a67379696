"""Host emulation of the FP8 attention's quantisation (csrc/attention_fp8.cu), on CPU tensors, and the fp64 attention the kernel is
held to.

    s = 2^k,  k = ceil(log2(amax / 448)) clamped to >= -126  (s = 1 for an all-zero block),   q = e4m3_rn_satfinite(x * 2^-k)

Blocks: Q and K one (token, head) of 64 values; V one (key tile, head, channel) over the tile's BN keys (BN = 96 when L is a multiple
of 96 but not of 128, else 128).  Multiplying by a power of two is exact, so these are the kernel's codes bit for bit."""
import torch

from emu_fp8 import E4M3, e4m3_rn_satfinite

HEAD = 64


def pow2_exponent(amax):
    """k with 2^k the smallest power of two for which amax / 2^k <= 448 (0 for amax == 0; at least -126)."""
    amax = amax.float()
    m, e = torch.frexp(amax)                           # amax = m 2^e, m in [0.5, 1); 448 = 0.875 2^9
    k = e.to(torch.int32) - 9 + (m > 0.875).to(torch.int32)
    k = torch.clamp(k, min=-126)
    return torch.where(amax == 0, torch.zeros_like(k), k)


def pow2_scale(amax):
    return torch.ldexp(torch.ones_like(amax, dtype=torch.float32), pow2_exponent(amax))


def quantize_blocks(x, dim):
    """Quantise x (fp32, or bf16 widened exactly) with one scale per slice along `dim` -> (e4m3 codes, fp32 scales with `dim`
    kept as size 1)."""
    x = x.float()
    k = pow2_exponent(x.abs().amax(dim=dim, keepdim=True))
    q = e4m3_rn_satfinite(torch.ldexp(x, -k))
    return q, torch.ldexp(torch.ones_like(k, dtype=torch.float32), k)


def key_tile(L):
    return 96 if L % 96 == 0 and L % 128 != 0 else 128


def split_qkv(qkv, B, H, W, C, win):
    """qkv [B*H*W, 3C] -> q, k, v [B, nwin, heads, L, 64] in the kernel's token order (windows row-major, tokens row-major
    inside a window), and the inverse map back to rows of the [B*H*W, C] output."""
    heads = C // HEAD
    x = qkv.reshape(B, H, W, 3, heads, HEAD)
    if win:
        x = x.reshape(B, H // win, win, W // win, win, 3, heads, HEAD).permute(0, 1, 3, 2, 4, 5, 6, 7)
        x = x.reshape(B, (H // win) * (W // win), win * win, 3, heads, HEAD)
    else:
        x = x.reshape(B, 1, H * W, 3, heads, HEAD)
    x = x.permute(3, 0, 1, 4, 2, 5)                    # [3, B, nwin, heads, L, 64]
    return x[0], x[1], x[2]


def merge_out(o, B, H, W, C, win):
    """[B, nwin, heads, L, 64] -> [B*H*W, C]."""
    heads = C // HEAD
    x = o.permute(0, 1, 3, 2, 4)                       # [B, nwin, L, heads, 64]
    if win:
        x = x.reshape(B, H // win, W // win, win, win, heads, HEAD).permute(0, 1, 3, 2, 4, 5, 6)
    return x.reshape(B * H * W, C)


def dequantized(qkv, B, H, W, C, win):
    """The values the kernel computes with: Q, K, V after the e4m3 round trip, fp64 [B, nwin, heads, L, 64]."""
    q, k, v = split_qkv(qkv.float(), B, H, W, C, win)
    L = q.shape[-2]
    qq, sq = quantize_blocks(q, -1)
    kq, sk = quantize_blocks(k, -1)
    bn = key_tile(L)
    nt = (L + bn - 1) // bn
    vp = torch.zeros(*v.shape[:-2], nt * bn, HEAD)
    vp[..., :L, :] = v
    vt = vp.reshape(*v.shape[:-2], nt, bn, HEAD)
    vq, sv = quantize_blocks(vt, -2)
    vd = (vq.double() * sv.double()).reshape(*v.shape[:-2], nt * bn, HEAD)[..., :L, :]
    return qq.double() * sq.double(), kq.double() * sk.double(), vd
