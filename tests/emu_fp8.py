"""Host emulation of the block-scaled e4m3 format of the FP8 teacher linears (csrc/fp8.cuh), on CPU fp32 tensors.

    s = amax / 448 (fp32; s = 1 for an all-zero block),   q = e4m3_rn_satfinite(x / s)

torch's CPU float8_e4m3fn cast rounds to nearest even but turns values above 448 into NaN instead of saturating, so the emulation
clamps to +-448 first, then casts."""
import torch

E4M3 = torch.float8_e4m3fn
BLOCK = 128


def e4m3_rn_satfinite(x):
    return x.clamp(-448.0, 448.0).to(E4M3)


def block_scale(amax):
    amax = amax.float()
    return torch.where(amax == 0, torch.ones_like(amax), amax / torch.tensor(448.0))


def quantize_rows(x):
    """fp32 [M, C], C % 128 == 0 -> (e4m3 [M, C], fp32 [M, C / 128]): activation blocks (one row, 128 columns)."""
    x = x.float()
    M, C = x.shape
    xb = x.reshape(M, C // BLOCK, BLOCK)
    s = block_scale(xb.abs().amax(-1))
    return e4m3_rn_satfinite(xb / s[..., None]).reshape(M, C), s


def quantize_weight(w):
    """fp32 [N, K], K % 128 == 0 -> (e4m3 [N, K], fp32 [ceil(N / 128), K / 128]): 128 x 128 blocks, the last row block ragged."""
    w = w.float()
    N, K = w.shape
    nb = (N + BLOCK - 1) // BLOCK
    pad = torch.zeros(nb * BLOCK, K)
    pad[:N] = w
    wb = pad.reshape(nb, BLOCK, K // BLOCK, BLOCK)
    s = block_scale(wb.abs().amax(dim=(1, 3)))
    q = e4m3_rn_satfinite(wb / s[:, None, :, None]).reshape(nb * BLOCK, K)[:N]
    return q, s


def dequant_rows(q, s):
    M, C = q.shape
    return (q.float().reshape(M, C // BLOCK, BLOCK) * s.float()[..., None]).reshape(M, C)


def dequant_weight(q, s):
    N, K = q.shape
    rs = s.float().repeat_interleave(BLOCK, 0)[:N].repeat_interleave(BLOCK, 1)
    return q.float() * rs
