"""EfficientViT backbone, H100-native.  Mirrors the module tree (class names, constructor arguments,
state_dict keys) of the reference `sam3/sam3/backbones/efficientvit/{backbone.py, nn/ops.py}` so that
reference checkpoints load unchanged, but every forward runs on the hand-written kernels of libes3.so:

  input stem (conv 3x3 s2 + residual DSConv)         -> es3_stem_fused_c16 (b1; other widths: es3_stem_conv3x3_s2 + es3_dsconv_res_bf16)
  MBConv blocks of b0 / b1 up to Cin 128             -> es3_mbconv_bf16 (wgmma, whole block on the SM)
  other MBConv blocks of stages 3-4                  -> es3_gemm_bf16 (expand) + es3_dwproj_tc_bf16 (depthwise + project + residual)
  LiteMLA (ops.py:521-671)                           -> es3_gemm_bf16 (qkv, proj) + es3_litemla_aggreg_dwpw + es3_litemla_attn_tc
  anything not instantiated                          -> es3_gemm_bf16 / es3_dwconv_tiled_bf16 (all native)

Activations live in HBM as NHWC bf16; accumulation is fp32.  Eval-mode only (see NativePlanMixin).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..nn_utils import NativePlanMixin, bn_scale_bias, dw_weight, pw_weight, pw_weight_scaled

__all__ = ["EfficientViTBackbone", "efficientvit_backbone_b0", "efficientvit_backbone_b1", "efficientvit_backbone_b2"]


def _val2tuple(x, n):
    if isinstance(x, (list, tuple)):
        x = list(x)
        return tuple(x + [x[-1]] * (n - len(x)))
    return tuple([x] * n)


# --------------------------------------------------------------------------- parameter containers
class ConvLayer(nn.Module):
    """ops.py:39-80.  Holds conv (+ optional BatchNorm2d); `act` is a name or None."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, dilation=1, groups=1, use_bias=False,
                 dropout=0, norm="bn2d", act_func="relu"):
        super().__init__()
        assert dilation == 1 and dropout == 0
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding=kernel_size // 2, groups=groups,
                              bias=use_bias)
        self.norm = nn.BatchNorm2d(out_channels) if norm == "bn2d" else None
        if norm not in ("bn2d", None):
            raise NotImplementedError(f"norm {norm!r} is not on the hot path")
        self.act = act_func
        self.stride, self.groups, self.kernel_size = stride, groups, kernel_size


class DSConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, use_bias=False, norm=("bn2d", "bn2d"),
                 act_func=("relu6", None)):
        super().__init__()
        use_bias, norm, act_func = _val2tuple(use_bias, 2), _val2tuple(norm, 2), _val2tuple(act_func, 2)
        self.depth_conv = ConvLayer(in_channels, in_channels, kernel_size, stride, groups=in_channels, norm=norm[0],
                                    act_func=act_func[0], use_bias=use_bias[0])
        self.point_conv = ConvLayer(in_channels, out_channels, 1, norm=norm[1], act_func=act_func[1],
                                    use_bias=use_bias[1])


class MBConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, mid_channels=None, expand_ratio=6,
                 use_bias=False, norm=("bn2d", "bn2d", "bn2d"), act_func=("relu6", "relu6", None)):
        super().__init__()
        use_bias, norm, act_func = _val2tuple(use_bias, 3), _val2tuple(norm, 3), _val2tuple(act_func, 3)
        mid = round(in_channels * expand_ratio) if mid_channels is None else mid_channels
        self.inverted_conv = ConvLayer(in_channels, mid, 1, stride=1, norm=norm[0], act_func=act_func[0],
                                       use_bias=use_bias[0])
        self.depth_conv = ConvLayer(mid, mid, kernel_size, stride=stride, groups=mid, norm=norm[1],
                                    act_func=act_func[1], use_bias=use_bias[1])
        self.point_conv = ConvLayer(mid, out_channels, 1, norm=norm[2], act_func=act_func[2], use_bias=use_bias[2])


class LiteMLA(nn.Module):
    def __init__(self, in_channels, out_channels, heads=None, heads_ratio=1.0, dim=8, use_bias=False,
                 norm=(None, "bn2d"), act_func=(None, None), kernel_func="relu", scales=(5,), eps=1.0e-15):
        super().__init__()
        assert kernel_func == "relu" and tuple(scales) == (5,)
        self.eps = eps
        heads = int(in_channels // dim * heads_ratio) if heads is None else heads
        total_dim = heads * dim
        use_bias, norm, act_func = _val2tuple(use_bias, 2), _val2tuple(norm, 2), _val2tuple(act_func, 2)
        self.dim, self.heads = dim, heads
        self.qkv = ConvLayer(in_channels, 3 * total_dim, 1, use_bias=use_bias[0], norm=norm[0], act_func=act_func[0])
        self.aggreg = nn.ModuleList([
            nn.Sequential(
                nn.Conv2d(3 * total_dim, 3 * total_dim, s, padding=s // 2, groups=3 * total_dim, bias=use_bias[0]),
                nn.Conv2d(3 * total_dim, 3 * total_dim, 1, groups=3 * heads, bias=use_bias[0]),
            ) for s in scales])
        self.proj = ConvLayer(total_dim * (1 + len(scales)), out_channels, 1, use_bias=use_bias[1], norm=norm[1],
                              act_func=act_func[1])


class IdentityLayer(nn.Module):
    pass


class ResidualBlock(nn.Module):
    def __init__(self, main, shortcut, post_act=None, pre_norm=None):
        super().__init__()
        assert post_act is None and pre_norm is None
        self.pre_norm = None
        self.main = main
        self.shortcut = shortcut
        self.post_act = None


class EfficientViTBlock(nn.Module):
    def __init__(self, in_channels, heads_ratio=1.0, dim=32, expand_ratio=4, scales=(5,), norm="bn2d",
                 act_func="hswish", context_module="LiteMLA", local_module="MBConv"):
        super().__init__()
        assert context_module == "LiteMLA" and local_module == "MBConv"
        self.context_module = ResidualBlock(
            LiteMLA(in_channels, in_channels, heads_ratio=heads_ratio, dim=dim, norm=(None, norm), scales=scales),
            IdentityLayer())
        self.local_module = ResidualBlock(
            MBConv(in_channels, in_channels, expand_ratio=expand_ratio, use_bias=(True, True, False),
                   norm=(None, None, norm), act_func=(act_func, act_func, None)),
            IdentityLayer())


class OpSequential(nn.Module):
    def __init__(self, op_list):
        super().__init__()
        self.op_list = nn.ModuleList([op for op in op_list if op is not None])


# --------------------------------------------------------------------------- native execution
def _fold(layer: ConvLayer, device):
    return bn_scale_bias(layer.norm, layer.conv.bias, layer.conv.out_channels, device)


class _PW:
    """Packed pointwise conv: bf16 [N,K] weight + fp32 scale/bias + act."""

    def __init__(self, layer: ConvLayer, device):
        self.w = pw_weight(layer.conv)                        # unscaled: the fused MBConv kernels take (w, scale, bias) separately
        self.scale, self.bias = _fold(layer, device)
        self.wf = pw_weight_scaled(layer.conv, self.scale)    # BN scale folded before the bf16 rounding: bias-only GEMM epilogue
        self.act = layer.act

    def __call__(self, x2d, residual=None, out=None):
        return ops.gemm(x2d, self.wf, bias=self.bias, act=self.act, residual=residual, out=out)


class _DW:
    def __init__(self, layer: ConvLayer, device):
        s, b = _fold(layer, device)
        self.w = dw_weight(layer.conv, s)
        self.bias = b
        self.ks, self.stride, self.act = layer.kernel_size, layer.stride, layer.act

    def __call__(self, x4d):
        return ops.dwconv(x4d, self.w, self.bias, self.ks, self.stride, self.act)


def _ones(n, dev):
    return torch.ones(n, device=dev, dtype=torch.float32)


def _zeros(n, dev):
    return torch.zeros(n, device=dev, dtype=torch.float32)


class _MBConvPlan:
    """MBConv (+ identity shortcut).  Tries the single-kernel fused path (es3_mbconv_bf16) and falls
    back to gemm_tc -> dwconv -> gemm_tc (all native kernels) for shapes it is not instantiated for."""

    def __init__(self, m: MBConv, residual: bool, device):
        self.inv, self.dw, self.pt = _PW(m.inverted_conv, device), _DW(m.depth_conv, device), _PW(m.point_conv, device)
        self.residual = residual
        mid, cout = self.inv.w.shape[0], self.pt.w.shape[0]
        self.f = dict(
            w1=self.inv.w, s1=self.inv.scale if self.inv.scale is not None else _ones(mid, device),
            b1=self.inv.bias if self.inv.bias is not None else _zeros(mid, device),
            wdw=self.dw.w, b2=self.dw.bias if self.dw.bias is not None else _zeros(mid, device),
            w3=self.pt.w, s3=self.pt.scale if self.pt.scale is not None else _ones(cout, device),
            b3=self.pt.bias if self.pt.bias is not None else _zeros(cout, device))
        self.fusable = (self.dw.ks == 3 and self.inv.act == self.dw.act == "hswish" and self.pt.act is None)
        self.dwproj = self.dw.ks == 3 and self.dw.stride == 1 and self.dw.act == "hswish" and self.pt.act is None

    def __call__(self, x):  # x: [B,H,W,C] bf16
        if self.fusable:
            y = ops.mbconv_fused(x, stride=self.dw.stride, residual=self.residual, act="hswish", **self.f)
            if y is not None:
                return y
            self.fusable = False  # shape not instantiated: remember and use the unfused native path
        B, H, W, C = x.shape
        mid = self.inv(x.view(-1, C)).view(B, H, W, -1)
        if self.dwproj:      # depthwise + projection in one wgmma kernel (stage 3/4 blocks)
            y = ops.dwproj(mid, self.f["wdw"], self.f["b2"], self.f["w3"], self.f["s3"], self.f["b3"],
                           residual=x if self.residual else None)
            if y is not None:
                return y
            self.dwproj = False
        mid = self.dw(mid)
        B2, H2, W2, Cm = mid.shape
        out = self.pt(mid.view(-1, Cm), residual=x.view(-1, C) if self.residual else None)
        return out.view(B2, H2, W2, -1)


class _LiteMLAPlan:
    """x + LiteMLA(x).  dim 16 (b0 / b1): the mma.sync kernels of litemla_tc.cu.  Other dims (b2: 32): depthwise 5x5 +
    the grouped 1x1 as a block-diagonal wgmma GEMM + the generic CUDA-core attention kernels."""

    def __init__(self, m: LiteMLA, device):
        assert m.qkv.norm is None and m.qkv.conv.bias is None and m.aggreg[0][0].bias is None
        self.dim = m.dim
        self.qkv_w = pw_weight(m.qkv.conv)
        self.c3 = self.qkv_w.shape[0]
        dw, pw = m.aggreg[0][0], m.aggreg[0][1]
        self.agg_dw = dw_weight(dw, None)                                         # [25, C3] fp32
        if self.dim == 16:
            self.agg_pw = pw.weight.detach().float().reshape(self.c3, 16).contiguous()  # [C3, 16] fp32
            self.agg_wd, self.agg_wp = ops.litemla_dwpw_weights(self.agg_dw, self.agg_pw)  # [C3/16, 25, 16], [C3, 16] bf16
        else:
            d = self.dim
            wg = pw.weight.detach().float().reshape(self.c3 // d, d, d)               # [group][out][in]
            self.agg_pw_bd = torch.block_diag(*wg).to(torch.bfloat16).contiguous()    # [C3, C3], zero off the groups
        self.proj = _PW(m.proj, device)
        self.heads2 = 2 * m.heads
        self.eps = m.eps

    def __call__(self, x):  # returns x + LiteMLA(x)
        B, H, W, C = x.shape
        if H * W <= self.dim:
            raise NotImplementedError("LiteMLA quadratic branch (H*W <= dim, ops.py:623-654) is never reached at "
                                      "the hot path's resolutions and is not built natively")
        c3 = self.c3
        ms = torch.empty((B, H, W, 2 * c3), device=x.device, dtype=torch.bfloat16)
        ms2d = ms.view(-1, 2 * c3)
        ops.gemm(x.view(-1, C), self.qkv_w, out=ms2d[:, :c3])
        if self.dim == 16:
            ops.litemla_aggreg_dwpw(ms, self.agg_wd, self.agg_wp, c3)
            att = ops.litemla_attn(ms, self.heads2, self.eps)
        else:
            t = ops.dwconv(ms[..., :c3], self.agg_dw, None, 5, 1, None)
            ops.gemm(t.view(-1, c3), self.agg_pw_bd, out=ms2d[:, c3:])
            att = ops.litemla_attn_generic(ms, self.heads2, self.dim, self.eps)
        out = self.proj(att.view(-1, att.shape[-1]), residual=x.view(-1, C))
        return out.view(B, H, W, C)


class EfficientViTBackbone(nn.Module, NativePlanMixin):
    """backbone.py:32-156.  forward(x NCHW fp32) -> dict of NCHW fp32 stage outputs (reference contract);
    forward_nhwc(x) -> final stage as NHWC bf16 (the fast path used by ImageStudentEncoder)."""

    def __init__(self, width_list, depth_list, in_channels=3, dim=32, expand_ratio=4, norm="bn2d", act_func="hswish"):
        super().__init__()
        self.width_list = []
        stem = [ConvLayer(in_channels, width_list[0], stride=2, norm=norm, act_func=act_func)]
        for _ in range(depth_list[0]):
            blk = self.build_local_block(width_list[0], width_list[0], 1, 1, norm, act_func)
            stem.append(ResidualBlock(blk, IdentityLayer()))
        in_channels = width_list[0]
        self.input_stem = OpSequential(stem)
        self.width_list.append(in_channels)
        stages = []
        for w, d in zip(width_list[1:3], depth_list[1:3]):
            stage = []
            for i in range(d):
                stride = 2 if i == 0 else 1
                blk = self.build_local_block(in_channels, w, stride, expand_ratio, norm, act_func)
                stage.append(ResidualBlock(blk, IdentityLayer() if stride == 1 else None))
                in_channels = w
            stages.append(OpSequential(stage))
            self.width_list.append(in_channels)
        for w, d in zip(width_list[3:], depth_list[3:]):
            stage = [ResidualBlock(self.build_local_block(in_channels, w, 2, expand_ratio, norm, act_func,
                                                          fewer_norm=True), None)]
            in_channels = w
            for _ in range(d):
                stage.append(EfficientViTBlock(in_channels, dim=dim, expand_ratio=expand_ratio, norm=norm,
                                               act_func=act_func))
            stages.append(OpSequential(stage))
            self.width_list.append(in_channels)
        self.stages = nn.ModuleList(stages)

    @staticmethod
    def build_local_block(in_channels, out_channels, stride, expand_ratio, norm, act_func, fewer_norm=False):
        if expand_ratio == 1:
            return DSConv(in_channels, out_channels, stride=stride, use_bias=(True, False) if fewer_norm else False,
                          norm=(None, norm) if fewer_norm else norm, act_func=(act_func, None))
        return MBConv(in_channels, out_channels, stride=stride, expand_ratio=expand_ratio,
                      use_bias=(True, True, False) if fewer_norm else False,
                      norm=(None, None, norm) if fewer_norm else norm, act_func=(act_func, act_func, None))

    # ---- plan -----------------------------------------------------------------------------------
    @staticmethod
    def _fused_stem_plan(stem_ops, dev):
        """One-launch stem (es3_stem_fused_c16) when the stem is conv(3->16, hswish) + one residual DSConv(16, hswish)."""
        if len(stem_ops) != 2:
            return None
        stem0, blk = stem_ops
        ds = blk.main
        if not (isinstance(ds, DSConv) and blk.shortcut is not None and stem0.conv.out_channels == 16
                and stem0.conv.in_channels == 3 and stem0.act == "hswish" and ds.depth_conv.act == "hswish"
                and ds.point_conv.act is None):
            return None
        ones = torch.ones(16, device=dev, dtype=torch.float32)
        zeros = torch.zeros(16, device=dev, dtype=torch.float32)
        s0, b0 = _fold(stem0, dev)
        w0 = torch.zeros(16, 32, device=dev, dtype=torch.float32)
        w0[:, :27] = stem0.conv.weight.detach().float().reshape(16, 27)
        w0 = w0.to(torch.bfloat16).contiguous()
        s1, b1 = _fold(ds.depth_conv, dev)
        wdw = dw_weight(ds.depth_conv.conv, s1)
        s2, b2 = _fold(ds.point_conv, dev)
        wpw = ds.point_conv.conv.weight.detach().reshape(16, 16).to(torch.bfloat16).contiguous()
        args = (w0, ones if s0 is None else s0, zeros if b0 is None else b0, wdw, zeros if b1 is None else b1, wpw,
                ones if s2 is None else s2, zeros if b2 is None else b2)
        return lambda x: ops.stem_fused_c16(x, *args)

    def _build_plan(self):
        dev = next(self.parameters()).device
        steps = []  # list of (stage_name_after | None, callable)
        stem0 = self.input_stem.op_list[0]
        stem_ops = list(self.input_stem.op_list)
        fused = self._fused_stem_plan(stem_ops, dev)
        if fused is not None:
            steps.append(fused)
            stem_ops = []
        s, b = _fold(stem0, dev)
        w = stem0.conv.weight.detach().float()
        if s is not None:
            w = w * s.view(-1, 1, 1, 1)
        w27 = w.reshape(w.shape[0], 27).t().contiguous()
        act0 = stem0.act
        if stem_ops:
            steps.append(lambda x: ops.stem_conv3x3_s2(x, w27, b, act0))
        for blk in stem_ops[1:]:
            ds = blk.main
            assert isinstance(ds, DSConv) and blk.shortcut is not None
            s1, b1 = _fold(ds.depth_conv, dev)
            wdw = dw_weight(ds.depth_conv.conv, s1)
            s2, b2 = _fold(ds.point_conv, dev)
            wpw = ds.point_conv.conv.weight.detach().float().reshape(ds.point_conv.conv.out_channels, -1)
            if s2 is not None:
                wpw = wpw * s2.view(-1, 1)
            wpw = wpw.contiguous()
            act1 = ds.depth_conv.act
            steps.append(lambda x, wdw=wdw, b1=b1, wpw=wpw, b2=b2, act1=act1: ops.dsconv_res(x, wdw, b1, wpw, b2, act1))
        marks = {len(steps): "stage0"}
        for sid, stage in enumerate(self.stages, 1):
            for op in stage.op_list:
                if isinstance(op, ResidualBlock):
                    steps.append(_MBConvPlan(op.main, op.shortcut is not None, dev))
                elif isinstance(op, EfficientViTBlock):
                    steps.append(_LiteMLAPlan(op.context_module.main, dev))
                    steps.append(_MBConvPlan(op.local_module.main, True, dev))
                else:
                    raise TypeError(type(op))
            marks[len(steps)] = f"stage{sid}"
        return steps, marks

    def _check_input(self, x):
        self._require_eval("EfficientViTBackbone.forward")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError("expected a CUDA fp32 NCHW image batch [B,3,H,W]; the native path has no CPU fallback")

    @torch.no_grad()
    def forward_nhwc(self, x: torch.Tensor) -> torch.Tensor:
        self._check_input(x)
        steps, _ = self._plan()
        for f in steps:
            x = f(x)
        return x

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> dict:
        self._check_input(x)
        steps, marks = self._plan()
        out = {"input": x}
        for i, f in enumerate(steps, 1):
            x = f(x)
            if i in marks:
                out[marks[i]] = ops.nhwc_to_nchw_f32(x)
        out["stage_final"] = out[f"stage{len(self.stages)}"]
        return out


def efficientvit_backbone_b0(**kwargs):
    return EfficientViTBackbone(width_list=[8, 16, 32, 64, 128], depth_list=[1, 2, 2, 2, 2], dim=16, **kwargs)


def efficientvit_backbone_b1(**kwargs):
    return EfficientViTBackbone(width_list=[16, 32, 64, 128, 256], depth_list=[1, 2, 3, 3, 4], dim=16, **kwargs)


def efficientvit_backbone_b2(**kwargs):
    return EfficientViTBackbone(width_list=[24, 48, 96, 192, 384], depth_list=[1, 3, 4, 4, 6], dim=32, **kwargs)
