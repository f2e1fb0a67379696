"""TEST INFRASTRUCTURE ONLY: a torch-CPU statement of what each libes3 op on the TRAINING path computes (same argument
lists, same layouts, outputs rounded to the dtype the kernel writes).  Two uses:

  * CPU (`-m "not gpu"`): `install(monkeypatch)` swaps these in for `efficientsam3_b200.ops.*`, so the host-side training
    graph (what is saved, in which order gradients are chained, every layout / stride / weight re-packing) is checked
    end to end against autograd of the oracle without a GPU;
  * GPU (`-m gpu`): each new kernel is compared with its function here on the same inputs (tests/test_train_gpu.py).

Backward ops are written through torch.autograd of the forward formula on purpose -- not by repeating the kernels' algebra.
The product package never imports this file.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

BF = torch.bfloat16     # activation storage dtype of the emulation
CD = torch.float32      # arithmetic dtype.  Tests set BF = CD = float64 for the exact-arithmetic mode (logic check)


def _act(x, act):
    if act in (None, "none"):
        return x
    return {"relu": F.relu, "hswish": F.hardswish, "gelu": F.gelu, "relu6": F.relu6, "sigmoid": torch.sigmoid}[act](x)


def _nchw(x):
    return x.to(CD).permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------ forward ops used in training
def gemm(a, w, *, scale=None, bias=None, act=None, residual=None, out=None, out_dtype=None, bn_hint=0, rope=None,
         act_after_res=False):
    assert rope is None and not act_after_res
    v = a.to(CD) @ w.to(CD).t()
    if scale is not None:
        v = v * scale
    if bias is not None:
        v = v + bias
    v = _act(v, act)
    if residual is not None:
        v = v + residual.to(CD)
    if out is None:
        return v.to(BF if out_dtype in (None, torch.bfloat16) else out_dtype)
    out.copy_(v.to(out.dtype))
    return out


def conv3x3(x, w9, *, scale=None, bias=None, act=None, residual=None, out_dtype=None, bn_hint=0):
    B, H, W, C = x.shape
    N = w9.shape[0]
    w = w9.to(CD).reshape(N, 3, 3, C).permute(0, 3, 1, 2)
    v = F.conv2d(_nchw(x), w, None, padding=1)
    if scale is not None:
        v = v * scale.view(1, -1, 1, 1)
    if bias is not None:
        v = v + bias.view(1, -1, 1, 1)
    v = _act(v, act)
    v = _nhwc(v)
    if residual is not None:
        v = v + residual.to(CD)
    return v.to(BF if out_dtype in (None, torch.bfloat16) else out_dtype)


def stem_conv3x3_s2(x, w27, bias, act):
    cout = w27.shape[1]
    w = w27.t().reshape(cout, 3, 3, 3).to(CD)
    v = F.conv2d(x.to(CD), w, bias.to(CD) if bias is not None else None, stride=2, padding=1)
    return _nhwc(_act(v, act)).to(BF)


def _dw(x4, w, ks, stride):
    C = x4.shape[1]
    return F.conv2d(x4, w.t().reshape(C, 1, ks, ks), None, stride=stride, padding=ks // 2, groups=C)


def dwconv(x, w, bias, ks, stride, act, out=None, force_simple=False):
    v = _dw(_nchw(x), w.to(CD), ks, stride)
    if bias is not None:
        v = v + bias.view(1, -1, 1, 1)
    v = _nhwc(_act(v, act)).to(BF)
    if out is not None:
        out.copy_(v)
        return out
    return v


def litemla_dwpw_weights(wdw, wpw):
    C3 = wpw.shape[0]
    d = wdw.reshape(25, C3 // 16, 16).permute(1, 0, 2)
    return d.to(torch.bfloat16).contiguous(), wpw.to(torch.bfloat16).contiguous()   # weights: always bf16


def litemla_aggreg_dwpw(ms, wd, wp, C3):
    G = C3 // 16
    wdw = wd.to(CD).permute(1, 0, 2).reshape(25, C3)                 # back to [25, C3]
    t = _dw(_nchw(ms[..., :C3]), wdw, 5, 1).to(BF).to(CD)            # depthwise result rounded to bf16 (as the kernel does)
    y = F.conv2d(t, wp.to(CD).reshape(C3, 16, 1, 1), None, groups=G)
    ms[..., C3:] = _nhwc(y).to(BF)
    return ms


def _lite_attn(ms, heads2, eps, dim=16):
    """ms [B,HW,heads2*3*dim] float -> (att [B,HW,heads2*dim], KV [B,heads2,dim+1,dim])."""
    B, HW, _ = ms.shape
    t = ms.reshape(B, HW, heads2, 3 * dim)
    q, k, v = F.relu(t[..., :dim]), F.relu(t[..., dim:2 * dim]), t[..., 2 * dim:]
    vpad = torch.cat([v, torch.ones_like(v[..., :1])], dim=-1)        # [B,HW,h,17]
    kv = torch.einsum("bnhj,bnhi->bhji", vpad, k)                     # [B,h,17,16]
    o = torch.einsum("bhji,bnhi->bnhj", kv, q)                        # [B,HW,h,17]
    y = o[..., :dim] / (o[..., dim:] + eps)
    return y.reshape(B, HW, heads2 * dim), kv


def litemla_attn(ms, heads2, eps=1e-15, return_kv=False):
    B, H, W, ld = ms.shape
    y, kv = _lite_attn(ms.to(CD).reshape(B, H * W, ld), heads2, eps)
    att = y.reshape(B, H, W, heads2 * 16).to(BF)
    if not return_kv:
        return att
    nchunk = (H * W + 511) // 512
    ws = torch.zeros(B, heads2, nchunk, 17, 16, dtype=CD)
    ws[:, :, 0] = kv                                                  # same layout as the kernel's partial sums
    return att, ws.reshape(-1)


def litemla_attn_generic(ms, heads2, dim, eps=1e-15, return_kv=False):
    B, H, W, ld = ms.shape
    y, kv = _lite_attn(ms.to(CD).reshape(B, H * W, ld), heads2, eps, dim)
    att = y.reshape(B, H, W, heads2 * dim).to(BF)
    if not return_kv:
        return att
    ws = torch.zeros(B, heads2, (H * W + 127) // 128, dim + 1, dim, dtype=CD)
    ws[:, :, 0] = kv
    return att, ws.reshape(-1)


def litemla_attn_bwd_generic(ms, datt, kv, heads2, dim, eps=1e-15):
    B, H, W, ld = ms.shape
    msf = ms.to(CD).reshape(B, H * W, ld).requires_grad_(True)
    with torch.enable_grad():
        y, _ = _lite_attn(msf, heads2, eps, dim)
        (g,) = torch.autograd.grad(y, msf, datt.to(CD).reshape(B, H * W, heads2 * dim))
    return g.reshape(ms.shape).to(BF)


def bilinear_nhwc_to_nchw(x, Ho, Wo):
    return F.interpolate(_nchw(x), size=(Ho, Wo), mode="bilinear", align_corners=False).contiguous()


def nhwc_to_nchw_f32(x):
    return _nchw(x).contiguous()


def nchw_f32_to_nhwc(x):
    return _nhwc(x).to(BF)


def gemm_simt(a, w, *, scale=None, bias=None, act=None, residual=None, out=None, out_dtype=None):
    return gemm(a, w, scale=scale, bias=bias, act=act, residual=residual, out=out, out_dtype=out_dtype)


def channel_mean(x):
    return x.to(CD).mean((1, 2))


def scale_channels(x, gate):
    return (x.to(CD) * gate.to(CD)[:, None, None, :]).to(BF)


def conv3x3_s2_narrow(x, w9, scale, bias, act=None):
    cout, cin = w9.shape[1], w9.shape[2]
    w = w9.to(CD).reshape(3, 3, cout, cin).permute(2, 3, 0, 1)
    v = F.conv2d(_nchw(x), w, None, stride=2, padding=1) * scale.to(CD).view(1, -1, 1, 1) + bias.to(CD).view(1, -1, 1, 1)
    return _nhwc(_act(v, act)).to(BF)


def layernorm_bf16(x, gamma, beta, eps=1e-5):
    return F.layer_norm(x.to(CD), (x.shape[-1],), gamma.to(CD), beta.to(CD), eps).to(BF)


def layernorm_bwd(x, dy, gamma, eps, dgamma=None, dbeta=None, dres=None):
    C = x.shape[-1]
    xf = x.to(CD).requires_grad_(True)
    g = gamma.to(CD).clone().requires_grad_(True)
    b = torch.zeros(C, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = F.layer_norm(xf, (C,), g, b, eps)
        gx, gg, gb = torch.autograd.grad(y, (xf, g, b), dy.to(CD))
    if dgamma is not None:
        dgamma += gg
    if dbeta is not None:
        dbeta += gb
    if dres is not None:
        gx = gx + dres.to(CD)
    return gx.to(BF)


def _win_attn(qkv, bias, B, H, W, C, heads, ws, scale):
    """qkv [B*H*W, 3C] (head h at columns [96h, 96h+96) = q|k|v), H, W multiples of ws -> out [B*H*W, C]."""
    nH, nW, N = H // ws, W // ws, ws * ws
    t = qkv.reshape(B, nH, ws, nW, ws, heads, 3, 32).permute(0, 1, 3, 5, 6, 2, 4, 7).reshape(B, nH, nW, heads, 3, N, 32)
    q, k, v = t[:, :, :, :, 0], t[:, :, :, :, 1], t[:, :, :, :, 2]
    a = (q @ k.transpose(-1, -2)) * scale + bias
    o = a.softmax(-1) @ v                                                   # [B,nH,nW,heads,N,32]
    o = o.reshape(B, nH, nW, heads, ws, ws, 32).permute(0, 1, 4, 2, 5, 3, 6)   # B,nH,ws,nW,ws,heads,32
    return o.reshape(B * H * W, C)


def win_attn_bias(qkv, qkv_pad, bias, B, H, W, C, heads, ws, scale):
    assert H % ws == 0 and W % ws == 0, "the emulation covers window-multiple maps (the training graph pads the map itself)"
    return _win_attn(qkv.to(CD), bias.to(CD), B, H, W, C, heads, ws, scale).to(BF)


def win_attn_bias_bwd(qkv, dout, bias, B, H, W, C, heads, ws, scale):
    q = qkv.to(CD).requires_grad_(True)
    b = bias.to(CD).clone().requires_grad_(True)
    with torch.enable_grad():
        o = _win_attn(q, b, B, H, W, C, heads, ws, scale)
        gq, gb = torch.autograd.grad(o, (q, b), dout.to(CD))
    return gq.to(BF), gb.float()


# ------------------------------------------------------------------------------------------ train_bwd.cu ops
def bn_stats(z, gamma, beta, eps, momentum, running_mean=None, running_var=None, num_batches_tracked=None):
    C = z.shape[-1]
    zf = z.to(CD).reshape(-1, C)
    M = zf.shape[0]
    mean = zf.mean(0)
    var = zf.var(0, unbiased=False)
    invstd = torch.rsqrt(var + eps)
    scale = (gamma.to(CD) if gamma is not None else 1.0) * invstd
    shift = (beta.to(CD) if beta is not None else 0.0) - mean * scale
    if running_mean is not None:
        running_mean.mul_(1 - momentum).add_(momentum * mean)
    if running_var is not None:
        running_var.mul_(1 - momentum).add_(momentum * var * (M / max(M - 1, 1)))
    if num_batches_tracked is not None:
        num_batches_tracked += 1
    return mean, invstd, scale, shift


def affine_act(z, scale, shift, act, residual=None, out=None):
    u = z.to(CD)
    if scale is not None:
        u = u * scale
    if shift is not None:
        u = u + shift
    v = _act(u, act)
    if residual is not None:
        v = v + residual.to(CD)
    if out is not None:
        out.copy_(v.to(out.dtype))
        return out
    return v.to(BF)


def bn_act_bwd(da, z, scale, shift, act, mode, mean=None, invstd=None, dgamma=None, dbeta=None, apply=True):
    """autograd through a = act(norm(z)), with norm = identity+bias (none), frozen BN (eval) or batch-stat BN (batch).
    gamma / beta are recovered from (scale, shift, mean, invstd)."""
    C = z.shape[-1]
    zf = z.to(CD).reshape(-1, C).requires_grad_(True)
    if mode != "none":      # the kernels read a NULL scale / shift as 1 / 0
        scale = torch.ones(C, dtype=CD) if scale is None else scale
        shift = torch.zeros(C, dtype=CD) if shift is None else shift
    with torch.enable_grad():
        if mode == "none":
            s = (scale if scale is not None else torch.ones(C, dtype=CD)).clone().requires_grad_(True)
            b = (shift if shift is not None else torch.zeros(C, dtype=CD)).clone().requires_grad_(True)
            u = zf * s.detach() + b
            params = (b,)
        else:
            gamma = (scale / invstd).clone().requires_grad_(True)
            beta = (shift + mean * scale).clone().requires_grad_(True)
            if mode == "eval":
                u = (zf - mean) * invstd * gamma + beta
            else:
                mu = zf.mean(0)
                var = zf.var(0, unbiased=False)
                eps_eff = 1.0 / invstd ** 2 - var.detach()          # the eps the forward used
                u = (zf - mu) * torch.rsqrt(var + eps_eff) * gamma + beta
            params = (gamma, beta)
        a = _act(u, act)
        outs = torch.autograd.grad(a, (zf,) + params, da.to(CD).reshape(-1, C))
    if mode == "none":
        if dbeta is not None:
            dbeta += outs[1]
    else:
        if dgamma is not None:
            dgamma += outs[1]
        if dbeta is not None:
            dbeta += outs[2]
    return outs[0].reshape(z.shape).to(BF) if apply else None


def add_bf16(a, b):
    return (a.to(CD) + b.to(CD)).to(BF)


def wgrad_pw(dz, x, dW, ldn=None, ldk=1, shift=None):
    M, N = dz.shape
    K = x.shape[1]
    xf = x.to(CD)
    if shift is not None:
        H, W, dy, dx = shift
        x4 = xf.reshape(-1, H, W, K)
        x4 = F.pad(x4, (0, 0, 1, 1, 1, 1))[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
        xf = x4.reshape(M, K)
    full = dz.to(CD).t() @ xf                                        # [N, K]
    ldn = K if ldn is None else ldn
    idx = (torch.arange(N).view(-1, 1) * ldn + torch.arange(K).view(1, -1) * ldk).reshape(-1)
    flat = dW.view(-1) if dW.dim() != 1 else dW
    flat[idx] += full.reshape(-1)
    return dW


def conv3x3_wgrad(dy, a, gw):
    N, C = dy.shape[3], a.shape[3]
    w = torch.zeros(N, C, 3, 3, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = F.conv2d(_nchw(a), w, padding=1)
        (g,) = torch.autograd.grad(y, w, _nchw(dy))
    gw += g
    return gw


def transpose_pad(x, Wp, dx):
    B, H, W, C = x.shape
    out = torch.zeros(C, B, H + 2, Wp, dtype=x.dtype)
    out[:, :, 1:H + 1, 1 - dx:1 - dx + W] = x.permute(3, 0, 1, 2)
    return out.reshape(C, -1)


def accumulate_strided(src, dst, inner, ld_outer, ld_inner):
    i = torch.arange(src.numel())
    dst.view(-1)[(i // inner) * ld_outer + (i % inner) * ld_inner] += src.reshape(-1)
    return dst


def se_bwd_dgate(dy, x):
    return (dy.to(CD) * x.to(CD)).sum((1, 2)).float()


def se_bwd_apply(dy, gate, add):
    return (dy.to(CD) * gate.to(CD)[:, None, None, :] + add.to(CD)[:, None, None, :]).to(BF)


def dwconv_bwd_data(dz, w, H, W, ks, stride):
    B, Ho, Wo, C = dz.shape
    x = torch.zeros(B, C, H, W, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = _dw(x, w.to(CD), ks, stride)
        (gx,) = torch.autograd.grad(y, x, _nchw(dz))
    return _nhwc(gx).to(BF)


def dwconv_wgrad(dz, x, dW, ks, stride, impl=None):
    C = x.shape[3]
    w = torch.zeros(ks * ks, C, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = _dw(_nchw(x), w, ks, stride)
        (gw,) = torch.autograd.grad(y, w, _nchw(dz))
    dW += gw.t().reshape(dW.shape)                                     # [k*k, C] -> [C,1,k,k]
    return dW


def stem_wgrad(img, dz, dW):
    cout = dz.shape[3]
    w = torch.zeros(cout, 3, 3, 3, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = F.conv2d(img.to(CD), w, None, stride=2, padding=1)
        (gw,) = torch.autograd.grad(y, w, _nchw(dz))
    dW += gw.reshape(dW.shape)
    return dW


def bilinear_bwd(dout, Hi, Wi):
    B, C, Ho, Wo = dout.shape
    x = torch.zeros(B, C, Hi, Wi, dtype=CD, requires_grad=True)
    with torch.enable_grad():
        y = F.interpolate(x, size=(Ho, Wo), mode="bilinear", align_corners=False)
        (gx,) = torch.autograd.grad(y, x, dout.to(CD))
    return _nhwc(gx).to(BF)


def litemla_attn_bwd(ms, datt, kv, heads2, eps=1e-15):
    B, H, W, ld = ms.shape
    msf = ms.to(CD).reshape(B, H * W, ld).requires_grad_(True)
    with torch.enable_grad():
        y, _ = _lite_attn(msf, heads2, eps)
        (g,) = torch.autograd.grad(y, msf, datt.to(CD).reshape(B, H * W, heads2 * 16))
    return g.reshape(ms.shape).to(BF)


PATCHED = ["layernorm_bf16", "layernorm_bwd", "win_attn_bias", "win_attn_bias_bwd", "gemm", "gemm_simt", "channel_mean", "scale_channels", "conv3x3_s2_narrow", "conv3x3", "stem_conv3x3_s2", "dwconv", "litemla_dwpw_weights", "litemla_aggreg_dwpw", "litemla_attn", "litemla_attn_generic", "litemla_attn_bwd_generic",
           "bilinear_nhwc_to_nchw", "nhwc_to_nchw_f32", "nchw_f32_to_nhwc", "bn_stats", "affine_act", "bn_act_bwd", "add_bf16",
           "wgrad_pw", "se_bwd_dgate", "se_bwd_apply", "transpose_pad", "accumulate_strided", "dwconv_bwd_data", "dwconv_wgrad", "stem_wgrad", "bilinear_bwd", "litemla_attn_bwd"]


def install(monkeypatch):
    """Route the training path's ops through the functions above (CPU tests only)."""
    import sys
    from efficientsam3_b200 import ops
    me = sys.modules[__name__]
    for name in PATCHED:
        monkeypatch.setattr(ops, name, getattr(me, name))
