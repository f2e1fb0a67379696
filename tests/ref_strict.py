"""fp64 statements of the strict mode's student kernels (csrc/strict_f32.cu: es3_dwconv_f32, es3_litemla_attn_f32,
es3_bilinear_nhwc_f32_to_nchw, es3_bias_act_res_f32) and, next to each, the per-element bound its fp32 arithmetic keeps to;
es3_scale_channels_f32 is one rounded product and is compared bit for bit with torch.

The bound form is the epilogue bound of tests/test_gemm_epilogue_gpu.py: an fmaf chain of n terms from 0 is held to GAMMA n u
sum |terms|, the scale, bias and residual each round once (4u of their operands), the activation carries the error through L_ACT
and adds its own, and the fp32 result adds 4u |ref|.  The strict kernels evaluate GELU with libm erff (es3_act), not es3_gelu_fast:
EPS_GELU_ERF charges erff's documented 2 ulp (4u of erf), the rounding of x / sqrt(2) and its constant (2u relative in the
argument, at most 1.13 * 2u * max z exp(-z^2) < u of erf) and the add of 1 (2u): 7u of (1 + erf), times 0.5 |x|.
Every function takes and returns float64 tensors (CPU or CUDA) holding the fp32 values the kernel reads.
tests/test_strict_kernels_cpu.py ties each statement to textbook float64 torch and shows that float32 restatements of the kernels
lie inside the bounds while restatements with a known fault do not.
"""
import numpy as np
import torch
import torch.nn.functional as F

from bounds import L_ACT, U, _act64, _eps_act
from ref_fwd import dw
from ref_train_bwd import GAMMA, TINY

EPS_GELU_ERF = 3.5 * U         # 0.5 |x| * 7u: see the module docstring
F32 = np.float32


def eps_act(x, act):
    """The activation's own error in es3_act (the strict kernels' activation), per element of its fp32 input x."""
    if act == "gelu":
        return EPS_GELU_ERF * x.abs()
    return _eps_act(x, act)


def epilogue(acc, absprod, n, act=None, scale=None, bias=None, res=None, after=False):
    """(ref, bound) of act(scale acc + bias) (+ res), or act(scale acc + bias + res) when `after`, where acc is an fmaf chain of n
    terms (n a number or a tensor broadcast against acc) whose |terms| sum to absprod; n = 0 with absprod = 0 is the elementwise
    form (acc = the kernel's input)."""
    s = scale if scale is not None else 1.0
    sacc = acc * s
    inner = GAMMA * n * U * absprod * (scale.abs() if scale is not None else 1.0) + 4 * U * sacc.abs()
    pre = sacc
    if bias is not None:
        pre = pre + bias
        inner = inner + 4 * U * bias.abs()
    if res is None:
        x = pre
        ref = _act64(x, act)
    elif after:
        x = pre + res
        inner = inner + 4 * U * res.abs()
        ref = _act64(x, act)
    else:
        x = pre
        ref = _act64(x, act) + res
    bound = L_ACT[act] * (inner + eps_act(x, act)) + 4 * U * ref.abs() + 2.0 ** -126
    return ref, bound


# ------------------------------------------------------------------------------------------------ depthwise
def valid_taps(B, H, W, ks, stride, like):
    """[B, Ho, Wo, 1]: how many of the ks x ks taps of each output pixel fall inside the H x W map (the kernel skips the others)."""
    ones = torch.ones(B, H, W, 1, dtype=like.dtype, device=like.device)
    return dw(ones, torch.ones(ks * ks, 1, dtype=like.dtype, device=like.device), ks, stride)


def dwconv(x, w, scale, bias, ks, stride, act):
    """es3_dwconv_f32: y = act(scale[c] dw(x; w) + bias[c]), x [B, H, W, C], w [ks^2, C] tap-major, same padding.  One thread per
    output element: an fmaf chain over the valid taps in (ky, kx) order from 0, then the epilogue."""
    B, H, W, _ = x.shape
    n = valid_taps(B, H, W, ks, stride, x)
    return epilogue(dw(x, w, ks, stride), dw(x.abs(), w.abs(), ks, stride), n, act, scale, bias)


# ------------------------------------------------------------------------------------------------ LiteMLA
def litemla_chunks(HW):
    """litemla_f32_chunks: (pixels per chunk, chunks) -- one chunk up to 2048 pixels, else equal chunks rounded up to 32."""
    n = max(-(-HW // 2048), 1)
    chunk = -(-(-(-HW // n)) // 32) * 32
    return chunk, -(-HW // chunk)


def litemla_attn(ms, B, HW, heads, dim, eps):
    """es3_litemla_attn_f32 on ms [B HW, >= 3 dim heads] (head h: q | k | v at columns 3 dim h ...) -> (ref, bound) [B HW, dim heads].

    kv[i][j] = sum_p v1[p][i] relu(k[p][j]), v1 = (v, 1): per chunk an fmaf chain over its pixels, then the chunks summed in order,
    so each entry is a chain of at most min(chunk, HW) + nchunk - 1 terms.  num[i] = sum_j kv[i][j] relu(q[j]) and den = sum_j
    kv[dim][j] relu(q[j]) are fmaf chains of dim terms over the fp32 kv: GAMMA dim u sum (|kv| + e_kv) q plus the kv error
    carried, sum e_kv q.  out = num * (1 / (den + eps)): to first order (e_num + |out| e_den) / (den + eps - e_den), plus 3u |out| for
    the add of eps, the reciprocal and the product.  A pixel whose q is all negative has num = den = 0 and out exactly 0."""
    chunk, nch = litemla_chunks(HW)
    nkv = min(chunk, HW) + nch - 1
    eps = float(np.float32(eps))
    t = ms.reshape(B, HW, -1)
    ref = torch.empty(B, HW, heads * dim, dtype=ms.dtype, device=ms.device)
    bound = torch.empty_like(ref)
    for h in range(heads):
        c = 3 * dim * h
        q, k, v = F.relu(t[..., c:c + dim]), F.relu(t[..., c + dim:c + 2 * dim]), t[..., c + 2 * dim:c + 3 * dim]
        v1 = torch.cat([v, torch.ones_like(v[..., :1])], -1)                    # [B, HW, dim + 1]
        kv = v1.transpose(1, 2) @ k                                               # [B, dim + 1, dim]
        e_kv = GAMMA * nkv * U * (v1.abs().transpose(1, 2) @ k)
        nd = q @ kv.transpose(1, 2)                                               # [B, HW, dim + 1]
        e_nd = GAMMA * dim * U * (q @ (kv.abs() + e_kv).transpose(1, 2)) + q @ e_kv.transpose(1, 2)
        num, den, e_num, e_den = nd[..., :dim], nd[..., dim:], e_nd[..., :dim], e_nd[..., dim:]
        o = num / (den + eps)
        ref[..., dim * h:dim * (h + 1)] = o
        bound[..., dim * h:dim * (h + 1)] = (e_num + o.abs() * e_den) / (den + eps - e_den) + 3 * U * o.abs() + TINY
    return ref.view(B * HW, -1), bound.view(B * HW, -1)


# ------------------------------------------------------------------------------------------------ bilinear
def source_coords(n_in, n_out):
    """The kernel's fp32 source coordinate of each output row / column (align_corners=False), restated in numpy float32 without
    FMA contraction: (i0, i1, l, h, ulp) -- the two source indices, the fp32 weights l = f - i0 and h = 1 - l, and ulp, the
    largest shift FMA contraction of ((i + 0.5) * s - 0.5) can cause (one ulp of the product, or of 0.5 where that is larger)."""
    s = F32(n_in) / F32(n_out)
    i0, i1, lo, hi, ulp = [], [], [], [], []
    for i in range(n_out):
        p = F32(F32(i) + F32(0.5)) * s
        f = max(F32(p - F32(0.5)), F32(0))
        a = min(int(f), n_in - 1)
        l = F32(f - F32(a))
        i0.append(a)
        i1.append(min(a + 1, n_in - 1))
        lo.append(float(l))
        hi.append(float(F32(1) - l))
        ulp.append(float(np.spacing(max(p, F32(0.5)))))
    return [torch.tensor(v) for v in (i0, i1, lo, hi, ulp)]


def bilinear(x, Ho, Wo):
    """es3_bilinear_nhwc_f32_to_nchw: x [B, Hi, Wi, C] -> (ref, bound) [B, C, Ho, Wo]; ref = hy (hx v00 + lx v01) + ly (hx v10 +
    lx v11) in fp64 at the kernel's fp32 weights.  Bound: 4u sum |w| |v| for the four products and three adds (contracted or not),
    plus the coordinate's ulp times the largest neighbour difference along that axis (the cell on either side of i0, so a shift
    across a source pixel centre is covered too).  Equal sizes give weights 1 / 0 and no coordinate term: the layout change is exact."""
    B, Hi, Wi, C = x.shape
    dev = x.device
    y0, y1, ly, hy, uy = (t.to(dev) for t in source_coords(Hi, Ho))
    x0, x1, lx, hx, ux = (t.to(dev) for t in source_coords(Wi, Wo))
    ly, hy, uy, lx, hx, ux = (t.to(x.dtype) for t in (ly, hy, uy, lx, hx, ux))

    def at(yi, xi):
        return x[:, yi][:, :, xi]                                                # [B, Ho, Wo, C]
    v00, v01, v10, v11 = at(y0, x0), at(y0, x1), at(y1, x0), at(y1, x1)
    Y, X = (lambda t: t.view(1, -1, 1, 1)), (lambda t: t.view(1, 1, -1, 1))
    ref = Y(hy) * (X(hx) * v00 + X(lx) * v01) + Y(ly) * (X(hx) * v10 + X(lx) * v11)
    terms = Y(hy) * (X(hx) * v00.abs() + X(lx) * v01.abs()) + Y(ly) * (X(hx) * v10.abs() + X(lx) * v11.abs())
    ym, xm = (y0 - 1).clamp_min(0), (x0 - 1).clamp_min(0)
    dy = torch.stack([(at(y1, xi) - at(y0, xi)).abs() for xi in (x0, x1)] + [(at(y0, xi) - at(ym, xi)).abs() for xi in (x0, x1)]).amax(0)
    dx = torch.stack([(at(yi, x1) - at(yi, x0)).abs() for yi in (y0, y1)] + [(at(yi, x0) - at(yi, xm)).abs() for yi in (y0, y1)]).amax(0)
    slope = Y(uy) * dy + X(ux) * dx
    if (Hi, Wi) == (Ho, Wo):
        slope = torch.zeros_like(slope)                                          # the source index is exactly the pixel
    bound = 4 * U * terms + slope + TINY
    return ref.permute(0, 3, 1, 2), bound.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ elementwise
def bias_act_res(x, bias, act, res, after):
    """es3_bias_act_res_f32 on x [total] with bias [C] taken at channel i % C: act(x + bias) (+ res), or act(x + bias + res) when
    `after` -- the epilogue bound with n = 0 and x as the accumulator (no argument at all is a copy, which the caller checks bit for
    bit)."""
    b = None if bias is None else bias[torch.arange(x.numel(), device=x.device) % bias.numel()]
    return epilogue(x, torch.zeros_like(x), 0, act, None, b, res, after)
