"""Train-mode forward + backward of the EfficientViT student on libes3.so (SURVEY.md §8 A19/A20: the
`preds = model(samples)` / `loss.backward()` pair of train_one_epoch, stage1/train_image_encoder_stage1.py:154-268).

The inference plan (efficientvit.py) fuses whole blocks and keeps nothing; training needs the layer inputs and the
pre-normalisation conv outputs, and BatchNorm2d has to use batch statistics (ConvLayer.norm in .train(),
efficientvit/nn/ops.py:39-80) unless the caller froze it (`set_bn_state`, TRAIN.EVAL_BN_WHEN_TRAINING,
train_image_encoder_stage1.py:310-314: BN modules in eval() inside a training model).  So the training graph is a
list of *units* (one per ConvLayer / MBConv / LiteMLA / head), each with

    forward(x)   raw conv (es3_gemm_bf16 / es3_dwconv / es3_stem_conv3x3_s2 / es3_conv3x3_bf16, no epilogue)
                 -> es3_bn_stats -> es3_affine_act; keeps x, z and the folded (scale, shift)
    backward(d)  es3_bn_act_bwd_{reduce,apply} -> weight gradient (es3_wgrad_pw / es3_dwconv_wgrad / es3_stem_wgrad)
                 -> input gradient (es3_gemm_bf16 on W^T with the skip gradient as the residual operand, es3_dwconv on the
                 flipped taps / es3_dwconv_bwd_data, es3_conv3x3_bf16 on the flipped-transposed kernel)

Activation gradients are bf16 NHWC, parameter gradients fp32 in the parameter's own shape.  `StudentTrainFunction`
(stage1/model.py) wraps the whole graph in ONE torch.autograd.Function so that `loss.backward()`, DDP hooks and
`p.grad` behave as with the reference module.  Everything on the device goes through `ops` (no torch compute
beyond O(C) vector prep and weight re-layouts); a missing GPU raises inside the first op.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops, sync_bn
from ..nn_utils import cached_pack, dw_weight, dw_weight_rot, pw_weight, pw_weight_t
from .efficientvit import (ConvLayer, DSConv, EfficientViTBlock, LiteMLA, MBConv, ResidualBlock)

__all__ = ["EfficientViTTrainGraph", "HeadTrainUnit", "GradSink"]


class GradSink(dict):
    """parameter -> fp32 gradient accumulator of one backward pass.  `direct`: accumulate straight into `p.grad` when that is an fp32
    contiguous tensor -- with stage1.optim.FlatAdamW every `p.grad` is a view into the ONE flat gradient arena that is all-reduced, so
    the backward kernels write the communication buffer itself (no per-parameter temporaries, no autograd accumulate pass, and a
    finished range of the arena can be handed to NCCL while the rest of the backward is still running)."""
    direct = False


def _grad_of(grads: dict, p: torch.Tensor):
    """fp32 accumulator for parameter `p` (None when it does not require grad)."""
    if p is None or not p.requires_grad:
        return None
    if getattr(grads, "direct", False):
        g = p.grad
        if g is not None and g.dtype == torch.float32 and g.is_contiguous() and g.shape == p.shape:
            return g
    g = grads.get(p)
    if g is None:
        g = torch.zeros(p.shape, device=p.device, dtype=torch.float32)
        grads[p] = g
    return g


class ConvUnit:
    """conv [+ BatchNorm2d] [+ act] of one ConvLayer.  kind: "pw" (1x1), "dw" (depthwise k x k) or "stem" (3->C 3x3 s2 on
    the fp32 NCHW image)."""

    def __init__(self, conv: nn.Conv2d, norm: nn.BatchNorm2d | None, act: str | None, kind: str):
        if norm is not None and conv.bias is not None:
            raise NotImplementedError("conv bias followed by BatchNorm is not on the EfficientViT path")
        if norm is not None and (norm.momentum is None or not norm.track_running_stats or not norm.affine):
            raise NotImplementedError("BatchNorm2d variants other than affine / momentum / running stats")
        self.conv, self.norm, self.act, self.kind = conv, norm, act, kind
        self.plain = norm is None and conv.bias is None and act is None
        self.ks, self.stride = conv.kernel_size[0], conv.stride[0]
        self.saved = None

    # ---- forward ------------------------------------------------------------------------------------------------------
    def _raw(self, x):
        conv = self.conv
        if self.kind == "pw":
            B, H, W, C = x.shape
            self.w = pw_weight(conv)                                            # [N, K] bf16
            return ops.gemm(x.view(-1, C), self.w).view(B, H, W, -1)
        if self.kind == "dw":
            self.w = dw_weight(conv, None)                                      # [k*k, C] fp32
            return ops.dwconv(x, self.w, None, self.ks, self.stride, None)
        cout = conv.out_channels
        w27 = cached_pack(conv, "w27", conv.weight, lambda: conv.weight.detach().float().reshape(cout, 27).t().contiguous())   # [27, Cout]
        return ops.stem_conv3x3_s2(x, w27, None, None)

    def forward(self, x, residual=None):
        z = self._raw(x)
        if self.plain:
            assert residual is None
            self.saved = (x, None, None, None, None, None, "none", None)
            return z
        norm = self.norm
        sync = None
        if norm is None:
            scale, shift, mean, invstd, mode = None, self.conv.bias.detach().float().contiguous(), None, None, "none"
        elif norm.training:   # per-rank statistics, or synchronised over the process group of an nn.SyncBatchNorm (sync_bn.py)
            mean, invstd, scale, shift, sync = sync_bn.batch_stats(norm, z)
            mode = "batch"
        else:   # frozen BN inside a training model: O(C) vector prep on the running statistics
            mean = norm.running_mean.detach().float().contiguous()
            invstd = torch.rsqrt(norm.running_var.detach().float() + norm.eps).contiguous()
            scale = (norm.weight.detach().float() * invstd).contiguous()
            shift = (norm.bias.detach().float() - mean * scale).contiguous()
            mode = "eval"
        a = ops.affine_act(z, scale, shift, self.act, residual)
        self.saved = (x, z, scale, shift, mean, invstd, mode, sync)
        return a

    # ---- backward -----------------------------------------------------------------------------------------------------
    def backward(self, da, grads, need_dx=True, dx_residual=None):
        """da: gradient of the unit's output (bf16, NHWC).  dx_residual: gradient arriving at x over a skip connection,
        added to the returned dx.  Returns dx (None for the stem / need_dx=False)."""
        x, z, scale, shift, mean, invstd, mode, sync = self.saved
        self.saved = None
        conv, norm = self.conv, self.norm
        if self.plain:
            dz = da
        else:
            dgamma = _grad_of(grads, norm.weight) if norm is not None else None
            dbeta = _grad_of(grads, norm.bias) if norm is not None else _grad_of(grads, conv.bias)
            dz = sync_bn.bn_act_bwd(da.contiguous(), z, scale, shift, self.act, mode, mean, invstd, dgamma, dbeta, sync)
        gw = _grad_of(grads, conv.weight)
        if self.kind == "pw":
            B, H, W, K = x.shape
            N = dz.shape[-1]
            dz2, x2 = dz.reshape(-1, N), x.view(-1, K)
            if gw is not None:
                ops.wgrad_pw(dz2, x2, gw)
            if not need_dx:
                return None
            wt = pw_weight_t(conv)                                              # [K, N] bf16 (cached per optimiser step)
            res = dx_residual.reshape(-1, K) if dx_residual is not None else None
            return ops.gemm(dz2, wt, residual=res).view(B, H, W, K)
        if self.kind == "dw":
            B, H, W, C = x.shape
            if gw is not None:
                ops.dwconv_wgrad(dz, x, gw, self.ks, self.stride)
            if not need_dx:
                return None
            if self.stride == 1:   # correlation with the 180-degree rotated taps: the forward kernel itself
                dx = ops.dwconv(dz, dw_weight_rot(conv), None, self.ks, 1, None)
            else:
                dx = ops.dwconv_bwd_data(dz, self.w, H, W, self.ks, self.stride)
            if dx_residual is not None:
                dx = ops.add_bf16(dx.view(-1, C), dx_residual.reshape(-1, C)).view(B, H, W, C)
            return dx
        if gw is not None:       # stem: the image needs no gradient
            ops.stem_wgrad(x, dz, gw)
        return None


def _unit(layer: ConvLayer, kind: str) -> ConvUnit:
    return ConvUnit(layer.conv, layer.norm, layer.act, kind)


class DSConvUnit:
    """x + DSConv(x) of the input stem (backbone.py:58-67) or a bare DSConv."""

    def __init__(self, m: DSConv, residual: bool):
        self.dw, self.pt, self.residual = _unit(m.depth_conv, "dw"), _unit(m.point_conv, "pw"), residual

    def forward(self, x):
        return self.pt.forward(self.dw.forward(x), residual=x if self.residual else None)

    def backward(self, dy, grads):
        d1 = self.pt.backward(dy, grads)
        return self.dw.backward(d1, grads, dx_residual=dy if self.residual else None)


class MBConvUnit:
    """[x +] MBConv(x): 1x1 expand -> depthwise 3x3 -> 1x1 project (ops.py:315-367, 740-770)."""

    def __init__(self, m: MBConv, residual: bool):
        self.inv, self.dw, self.pt = _unit(m.inverted_conv, "pw"), _unit(m.depth_conv, "dw"), _unit(m.point_conv, "pw")
        self.residual = residual
        if self.pt.plain and residual:
            raise NotImplementedError("residual MBConv whose projection has neither norm nor bias")

    def forward(self, x):
        a = self.dw.forward(self.inv.forward(x))
        return self.pt.forward(a, residual=x if self.residual else None)

    def backward(self, dy, grads):
        d = self.dw.backward(self.pt.backward(dy, grads), grads)
        return self.inv.backward(d, grads, dx_residual=dy if self.residual else None)


class LiteMLAUnit:
    """x + LiteMLA(x) (ops.py:521-671), head dim 16 (efficientvit b0 / b1), linear-attention branch."""

    def __init__(self, m: LiteMLA):
        if m.dim != 16:
            raise NotImplementedError("train-mode LiteMLA is built for head dim 16 (efficientvit_b0 / b1); "
                                      f"got dim {m.dim}")
        assert m.qkv.norm is None and m.qkv.conv.bias is None and m.qkv.act is None and m.aggreg[0][0].bias is None
        self.m = m
        self.proj = _unit(m.proj, "pw")
        self.saved = None

    def forward(self, x):
        m = self.m
        B, H, W, C = x.shape
        if H * W <= m.dim:
            raise NotImplementedError("LiteMLA quadratic branch (H*W <= dim, ops.py:623-654) is not built natively")
        qkv_w = pw_weight(m.qkv.conv)
        c3 = qkv_w.shape[0]
        dwc, pwc = m.aggreg[0][0], m.aggreg[0][1]
        agg_dw = dw_weight(dwc, None)                                            # [25, c3] fp32
        agg_pw = pwc.weight.detach().float().reshape(c3, 16).contiguous()        # [c3, 16] fp32: [g*16+n][i]
        wd, wp = ops.litemla_dwpw_weights(agg_dw, agg_pw)
        ms = torch.empty((B, H, W, 2 * c3), device=x.device, dtype=ops.ACT_DTYPE)
        ops.gemm(x.view(-1, C), qkv_w, out=ms.view(-1, 2 * c3)[:, :c3])
        ops.litemla_aggreg_dwpw(ms, wd, wp, c3)
        att, kv = ops.litemla_attn(ms, 2 * m.heads, m.eps, return_kv=True)
        y = self.proj.forward(att, residual=x)
        # the forward kernel consumed the bf16-rounded taps: the backward differentiates that same function
        agg_dw_r = wd.float().permute(1, 0, 2).reshape(25, c3).contiguous()
        self.saved = (x, ms, kv, qkv_w, agg_dw_r, wp)
        return y

    def backward(self, dy, grads):
        m = self.m
        x, ms, kv, qkv_w, agg_dw, wp = self.saved
        self.saved = None
        B, H, W, C = x.shape
        c3 = qkv_w.shape[0]
        G = c3 // 16
        dwc, pwc = m.aggreg[0][0], m.aggreg[0][1]
        datt = self.proj.backward(dy, grads)                                     # [B,H,W,2*heads*16]
        dms = ops.litemla_attn_bwd(ms, datt.contiguous(), kv, 2 * m.heads, m.eps)   # [B,H,W,2*c3]
        dms2 = dms.view(-1, 2 * c3)
        d_y2 = dms2[:, c3:]                                                      # gradient of the aggregated (scale-5) qkv
        # grouped 1x1 (aggreg[0][1]): y2[:, 16g+n] = sum_i t[:, 16g+i] wp[16g+n][i], t = dw5x5(qkv) (recomputed)
        t = ops.dwconv(ms[..., :c3], agg_dw, None, 5, 1, None)
        g_pw = _grad_of(grads, pwc.weight)
        if g_pw is not None:   # full [c3 x c3] product on the tensor cores, the block diagonal is the grouped gradient
            full = torch.zeros((c3, c3), device=x.device, dtype=torch.float32)
            ops.wgrad_pw(d_y2, t.view(-1, c3), full)
            idx = torch.arange(G, device=x.device)
            g_pw += full.view(G, 16, G, 16)[idx, :, idx, :].reshape(pwc.weight.shape)
        wbd_t = cached_pack(pwc, "wbd_t", pwc.weight, lambda: torch.block_diag(*wp.view(G, 16, 16).transpose(1, 2)).contiguous())   # [16g+i][16g+n] bf16
        d_t = ops.gemm(d_y2, wbd_t).view(B, H, W, c3)
        # depthwise 5x5 (aggreg[0][0]) on qkv
        g_dw = _grad_of(grads, dwc.weight)
        if g_dw is not None:
            ops.dwconv_wgrad(d_t, ms[..., :c3], g_dw, 5, 1)
        d_q1 = ops.dwconv(d_t, cached_pack(dwc, "agg_rot", dwc.weight, lambda: agg_dw.flip(0).contiguous()), None, 5, 1, None)
        d_qkv = ops.add_bf16(dms2[:, :c3], d_q1.view(-1, c3))
        # qkv 1x1
        g_qkv = _grad_of(grads, m.qkv.conv.weight)
        if g_qkv is not None:
            ops.wgrad_pw(d_qkv, x.view(-1, C), g_qkv)
        return ops.gemm(d_qkv, pw_weight_t(m.qkv.conv), residual=dy.reshape(-1, C)).view(B, H, W, C)


class LiteMLAGenericUnit:
    """x + LiteMLA(x) for head dims other than 16 (efficientvit_b2: 32), on the route the inference plan takes for them:
    depthwise 5x5 (es3_dwconv) + the grouped 1x1 as a block-diagonal wgmma GEMM + es3_litemla_attn_generic; backward through
    es3_litemla_attn_bwd_generic (litemla_bwd_generic.cu)."""

    def __init__(self, m: LiteMLA):
        if m.dim not in (16, 32):
            raise NotImplementedError(f"LiteMLA head dim {m.dim} is not instantiated (16, 32)")
        assert m.qkv.norm is None and m.qkv.conv.bias is None and m.qkv.act is None and m.aggreg[0][0].bias is None
        self.m = m
        self.proj = _unit(m.proj, "pw")
        self.saved = None

    def forward(self, x):
        m = self.m
        d = m.dim
        B, H, W, C = x.shape
        if H * W <= d:
            raise NotImplementedError("LiteMLA quadratic branch (H*W <= dim, ops.py:623-654) is not built natively")
        qkv_w = pw_weight(m.qkv.conv)
        c3 = qkv_w.shape[0]
        G = c3 // d
        dwc, pwc = m.aggreg[0][0], m.aggreg[0][1]
        agg_dw = dw_weight(dwc, None)                                            # [25, c3] fp32
        wg = pwc.weight.detach().reshape(G, d, d).to(torch.bfloat16)             # [group][out n][in i]
        w_bd = torch.block_diag(*wg).contiguous()                                # y2 = t . w_bd^T
        ms = torch.empty((B, H, W, 2 * c3), device=x.device, dtype=ops.ACT_DTYPE)
        ms2 = ms.view(-1, 2 * c3)
        ops.gemm(x.view(-1, C), qkv_w, out=ms2[:, :c3])
        t = ops.dwconv(ms[..., :c3], agg_dw, None, 5, 1, None)
        ops.gemm(t.view(-1, c3), w_bd, out=ms2[:, c3:])
        att, kv = ops.litemla_attn_generic(ms, 2 * m.heads, d, m.eps, return_kv=True)
        y = self.proj.forward(att, residual=x)
        self.saved = (x, ms, t, kv, qkv_w, agg_dw, wg)
        return y

    def backward(self, dy, grads):
        m = self.m
        d = m.dim
        x, ms, t, kv, qkv_w, agg_dw, wg = self.saved
        self.saved = None
        B, H, W, C = x.shape
        c3 = qkv_w.shape[0]
        G = c3 // d
        dwc, pwc = m.aggreg[0][0], m.aggreg[0][1]
        datt = self.proj.backward(dy, grads)
        dms = ops.litemla_attn_bwd_generic(ms, datt.contiguous(), kv, 2 * m.heads, d, m.eps)
        dms2 = dms.view(-1, 2 * c3)
        d_y2 = dms2[:, c3:]
        g_pw = _grad_of(grads, pwc.weight)
        if g_pw is not None:
            full = torch.zeros((c3, c3), device=x.device, dtype=torch.float32)
            ops.wgrad_pw(d_y2, t.view(-1, c3), full)
            idx = torch.arange(G, device=x.device)
            g_pw += full.view(G, d, G, d)[idx, :, idx, :].reshape(pwc.weight.shape)
        w_bd_t = torch.block_diag(*wg.transpose(1, 2)).contiguous()              # [d g + i][d g + n]
        d_t = ops.gemm(d_y2, w_bd_t).view(B, H, W, c3)
        g_dw = _grad_of(grads, dwc.weight)
        if g_dw is not None:
            ops.dwconv_wgrad(d_t, ms[..., :c3], g_dw, 5, 1)
        d_q1 = ops.dwconv(d_t, agg_dw.flip(0).contiguous(), None, 5, 1, None)
        d_qkv = ops.add_bf16(dms2[:, :c3], d_q1.view(-1, c3))
        g_qkv = _grad_of(grads, m.qkv.conv.weight)
        if g_qkv is not None:
            ops.wgrad_pw(d_qkv, x.view(-1, C), g_qkv)
        return ops.gemm(d_qkv, pw_weight_t(m.qkv.conv), residual=dy.reshape(-1, C)).view(B, H, W, C)


class EfficientViTTrainGraph:
    """Units of EfficientViTBackbone in execution order (backbone.py:32-156)."""

    def __init__(self, backbone):
        stem_ops = list(backbone.input_stem.op_list)
        self.stem = _unit(stem_ops[0], "stem")
        self.units = []
        for blk in stem_ops[1:]:
            assert isinstance(blk, ResidualBlock) and isinstance(blk.main, DSConv)
            self.units.append(DSConvUnit(blk.main, blk.shortcut is not None))
        for stage in backbone.stages:
            for op in stage.op_list:
                if isinstance(op, ResidualBlock):
                    main = op.main
                    self.units.append(MBConvUnit(main, op.shortcut is not None) if isinstance(main, MBConv)
                                      else DSConvUnit(main, op.shortcut is not None))
                elif isinstance(op, EfficientViTBlock):
                    mla = op.context_module.main
                    self.units.append(LiteMLAUnit(mla) if mla.dim == 16 else LiteMLAGenericUnit(mla))
                    self.units.append(MBConvUnit(op.local_module.main, True))
                else:
                    raise TypeError(type(op))

    def forward(self, x):
        x = self.stem.forward(x)
        for u in self.units:
            x = u.forward(x)
        return x

    def backward(self, d, grads):
        for u in reversed(self.units):
            d = u.backward(d, grads)
        self.stem.backward(d, grads, need_dx=False)


class HeadTrainUnit:
    """ImageStudentEncoder.head + resize (stage1/model.py:194-211): Conv1x1(no bias) -> BN -> GELU -> Conv3x3(bias) ->
    bilinear to embed_size -> NCHW fp32."""

    def __init__(self, head: nn.Sequential, embed_size: int):
        self.c0 = ConvUnit(head[0], head[1], "gelu", "pw")
        self.conv3 = head[3]
        self.embed = embed_size
        self.saved = None

    def forward(self, feats):
        a1 = self.c0.forward(feats)                                              # [B,h,w,1024] bf16
        w = self.conv3.weight.detach()
        n, c = w.shape[:2]
        w9 = cached_pack(self.conv3, "w9", self.conv3.weight, lambda: w.permute(0, 2, 3, 1).reshape(n, 9 * c).to(torch.bfloat16).contiguous())
        y = ops.conv3x3(a1, w9, bias=self.conv3.bias.detach().float().contiguous())
        B, h, wd, _ = y.shape
        self.saved = (a1, h, wd)
        if h != self.embed or wd != self.embed:
            return ops.bilinear_nhwc_to_nchw(y, self.embed, self.embed)
        return ops.nhwc_to_nchw_f32(y)

    def backward(self, dout, grads):
        a1, h, wd = self.saved
        self.saved = None
        conv3 = self.conv3
        n, c = conv3.weight.shape[:2]
        dout = dout.float().contiguous()
        dy = ops.bilinear_bwd(dout, h, wd) if (h != self.embed or wd != self.embed) else ops.nchw_f32_to_nhwc(dout)
        gb = _grad_of(grads, conv3.bias)
        if gb is not None:      # d bias = column sums of dy: the reduce half of the BN/act backward with act = none
            ops.bn_act_bwd(dy, dy, None, None, None, "none", dbeta=gb, apply=False)
        gw = _grad_of(grads, conv3.weight)
        if gw is not None:      # nine wgmma GEMMs over the zero-framed, transposed pixel index
            ops.conv3x3_wgrad(dy, a1, gw)
        # input gradient: 3x3 conv of dy with the rotated, in/out-transposed kernel
        wt9 = cached_pack(conv3, "wt9", conv3.weight,
                          lambda: conv3.weight.detach().flip(2, 3).permute(1, 2, 3, 0).reshape(c, 9 * n).to(torch.bfloat16).contiguous())
        da1 = ops.conv3x3(dy, wt9)
        return self.c0.backward(da1, grads)
