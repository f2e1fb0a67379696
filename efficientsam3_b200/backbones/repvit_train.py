"""Train-mode forward + backward of the RepViT student (repvit_m1_1 = "RV-M", config 4 of BASELINE.json: stage-1
distillation of the RepViT-M student under DDP) on libes3.so.  Same scheme as efficientvit_train.py -- a list of units with
forward(x) / backward(d, grads) wrapped into ONE autograd node by stage1.model.StudentTrainFunction -- and built ENTIRELY from
entry points that already have GPU parity tests (tests/test_ops_gpu.py, tests/test_zz_train_gpu.py); what is new here is host
composition only:

  RepVGGDW in .train() (repvit.py:84-96)   BN_out( BN1(dw3x3(x)) + dw1x1(x) + x ) cannot be re-parameterised while BN1 uses batch
                                           statistics: u = scale1 z1 + (w1 + 1) x + (shift1 + b1) as two es3_affine_act passes,
                                           the dw1x1 weight / bias gradients are the column sums  sum du x,  sum du
                                           (es3_bn_act_bwd_reduce with mean 0, invstd 1)
  SqueezeExcite (timm, repvit.py:23,136)   es3_channel_mean -> es3_gemm_simt x2 -> es3_scale_channels; backward: per-image
                                           es3_bn_act_bwd_reduce (d gate = sum_hw dy y) and es3_affine_act (dy gate + d mean / HW),
                                           the [B,C] MLP gradients through es3_gemm_simt
  patch-embed conv 2 (3x3, stride 2)       forward es3_conv3x3_s2_narrow_bf16; weight gradient = 9 es3_wgrad_pw launches on the four
                                           2x2 phases of the input (a stride-2 tap is a stride-1 shift of one phase); input gradient =
                                           9 es3_gemm_bf16 calls on shifted dz, accumulated per phase through the residual operand

The phase split / interleave and the shifted copies are torch strided copies (re-layouts, as the weight packing is).
Built for all three RepViT widths: patch-embed mid widths 32 (m1_1), 24 (m0_9: zero-padded to 32 in front of the second conv) and
40 (m2_3: the whole first conv + BN runs zero-padded to 48, PaddedStemUnit).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops, sync_bn
from ..nn_utils import dw_weight
from .efficientvit_train import ConvUnit, _grad_of
from .repvit import Conv2d_BN, RepViTBlock, SqueezeExcite

__all__ = ["RepViTTrainGraph"]


def _cu(cb: Conv2d_BN, act, kind) -> ConvUnit:
    return ConvUnit(cb.c, cb.bn, act, kind)


def _norm_params(norm: nn.BatchNorm2d, z):
    """(mean, invstd, scale, shift, mode, sync) of a BatchNorm2d over z: batch statistics (+ running-stat update) in .train(),
    synchronised over the process group of an nn.SyncBatchNorm (sync: see sync_bn.batch_stats, None otherwise); running
    statistics when the module was frozen with .eval() (set_bn_state)."""
    if norm.training:
        mean, invstd, scale, shift, sync = sync_bn.batch_stats(norm, z)
        return mean, invstd, scale, shift, "batch", sync
    mean = norm.running_mean.detach().float().contiguous()
    invstd = torch.rsqrt(norm.running_var.detach().float() + norm.eps).contiguous()
    scale = (norm.weight.detach().float() * invstd).contiguous()
    shift = (norm.bias.detach().float() - mean * scale).contiguous()
    return mean, invstd, scale, shift, "eval", None


def _colsum_grads(d, z, dprod, dsum):
    """dprod[c] += sum_rows d z,  dsum[c] += sum_rows d  (either may be None) on verified reduction kernels."""
    C = d.shape[-1]
    dev = d.device
    zeros = torch.zeros(C, device=dev, dtype=torch.float32)
    ones = torch.ones(C, device=dev, dtype=torch.float32)
    ops.bn_act_bwd(d, z, None, None, None, "eval", mean=zeros, invstd=ones, dgamma=dprod, dbeta=dsum, apply=False)


class ChannelMixerUnit:
    """x + BN(pw(GELU(BN(pw(x)))))  (Residual(channel_mixer), repvit.py:51-81, 139-160)."""

    def __init__(self, seq: nn.Sequential):
        self.c0, self.c2 = _cu(seq[0], "gelu", "pw"), _cu(seq[2], None, "pw")

    def forward(self, x):
        return self.c2.forward(self.c0.forward(x), residual=x)

    def backward(self, dy, grads):
        return self.c0.backward(self.c2.backward(dy, grads), grads, dx_residual=dy)


class SEUnit:
    """timm SqueezeExcite: x * sigmoid(fc2(relu(fc1(mean_hw(x)))))."""

    def __init__(self, se: SqueezeExcite):
        self.se = se
        self.saved = None

    def forward(self, x):
        se = self.se
        w1 = se.fc1.weight.detach().float().reshape(se.fc1.out_channels, -1).contiguous()      # [rd, C]
        w2 = se.fc2.weight.detach().float().reshape(se.fc2.out_channels, -1).contiguous()      # [C, rd]
        m = ops.channel_mean(x)                                                                # [B, C] fp32
        h = ops.gemm_simt(m, w1, bias=se.fc1.bias.detach().float().contiguous(), act="relu", out_dtype=torch.float32)
        g = ops.gemm_simt(h, w2, bias=se.fc2.bias.detach().float().contiguous(), act="sigmoid", out_dtype=torch.float32)
        self.saved = (x, m, h, g, w1, w2)
        return ops.scale_channels(x, g)

    def backward(self, dy, grads):
        se = self.se
        x, m, h, g, w1, w2 = self.saved
        self.saved = None
        HW = x.shape[1] * x.shape[2]
        dy = dy.contiguous()
        dgate = ops.se_bwd_dgate(dy, x)                                                         # d gate[b, c] = sum_hw dy x
        # the two 1x1 convs on the pooled [B, C] vectors (O(B C) element-wise prep in torch, contractions on es3_gemm_simt)
        dpre2 = (dgate * g * (1.0 - g)).contiguous()                                            # [B, C]
        f32 = dict(out_dtype=torch.float32)
        g_w2, g_b2 = _grad_of(grads, se.fc2.weight), _grad_of(grads, se.fc2.bias)
        if g_w2 is not None:
            g_w2 += ops.gemm_simt(dpre2.t().contiguous(), h.t().contiguous(), **f32).reshape(g_w2.shape)   # [C, rd]
        if g_b2 is not None:
            g_b2 += dpre2.sum(0)
        dh = ops.gemm_simt(dpre2, w2.t().contiguous(), **f32)                                   # [B, rd]
        dpre1 = (dh * (h > 0).to(dh.dtype)).contiguous()
        g_w1, g_b1 = _grad_of(grads, se.fc1.weight), _grad_of(grads, se.fc1.bias)
        if g_w1 is not None:
            g_w1 += ops.gemm_simt(dpre1.t().contiguous(), m.t().contiguous(), **f32).reshape(g_w1.shape)   # [rd, C]
        if g_b1 is not None:
            g_b1 += dpre1.sum(0)
        dm = (ops.gemm_simt(dpre1, w1.t().contiguous(), **f32) / HW).contiguous()                # [B, C]: d mean / HW
        return ops.se_bwd_apply(dy, g, dm)                                                     # dx = dy * gate + d mean / HW


class RepVGGDWUnit:
    """BN( Conv2d_BN(dw3x3)(x) + dw1x1(x) + x )  (RepVGGDW.forward, repvit.py:93-96), un-fused as .train() runs it."""

    def __init__(self, rv):
        self.rv = rv
        self.saved = None

    def forward(self, x):
        rv = self.rv
        C = x.shape[-1]
        w3 = dw_weight(rv.conv.c, None)                                          # [9, C] fp32
        z1 = ops.dwconv(x, w3, None, 3, 1, None)
        n1 = _norm_params(rv.conv.bn, z1)
        mean1, invstd1, scale1, shift1, mode1, sync1 = n1
        sb = (rv.conv1.weight.detach().float().reshape(C) + 1.0).contiguous()    # dw1x1 weight + the identity branch
        tb = (shift1 + rv.conv1.bias.detach().float()).contiguous()
        tmp = ops.affine_act(x, sb, tb, None)
        u = ops.affine_act(z1, scale1, None, None, residual=tmp)
        no = _norm_params(rv.bn, u)
        self.saved = (x, z1, u, w3, sb, n1, no)
        return ops.affine_act(u, no[2], no[3], None)

    def backward(self, dy, grads):
        rv = self.rv
        x, z1, u, w3, sb, n1, no = self.saved
        self.saved = None
        mean1, invstd1, scale1, shift1, mode1, sync1 = n1
        mean_o, invstd_o, scale_o, shift_o, mode_o, sync_o = no
        du = sync_bn.bn_act_bwd(dy.contiguous(), u, scale_o, shift_o, None, mode_o, mean_o, invstd_o,
                                _grad_of(grads, rv.bn.weight), _grad_of(grads, rv.bn.bias), sync_o)
        dz1 = sync_bn.bn_act_bwd(du, z1, scale1, shift1, None, mode1, mean1, invstd1,
                                 _grad_of(grads, rv.conv.bn.weight), _grad_of(grads, rv.conv.bn.bias), sync1)
        g_w1, g_b1 = _grad_of(grads, rv.conv1.weight), _grad_of(grads, rv.conv1.bias)
        if g_w1 is not None or g_b1 is not None:
            _colsum_grads(du, x, g_w1.view(-1) if g_w1 is not None else None, g_b1)
        g_w3 = _grad_of(grads, rv.conv.c.weight)
        if g_w3 is not None:
            ops.dwconv_wgrad(dz1, x, g_w3, 3, 1)
        dxa = ops.dwconv(dz1, w3.flip(0).contiguous(), None, 3, 1, None)
        return ops.affine_act(du, sb, None, None, residual=dxa)


class TokenMixerDownUnit:
    """stride-2 token mixer: Conv2d_BN(dw3x3, s2) -> [SE] -> Conv2d_BN(1x1)  (repvit.py:131-138)."""

    def __init__(self, tm: nn.Sequential, use_se: bool):
        self.dw = _cu(tm[0], None, "dw")
        self.se = SEUnit(tm[1]) if use_se else None
        self.pw = _cu(tm[2], None, "pw")

    def forward(self, x):
        x = self.dw.forward(x)
        if self.se is not None:
            x = self.se.forward(x)
        return self.pw.forward(x)

    def backward(self, dy, grads):
        d = self.pw.backward(dy, grads)
        if self.se is not None:
            d = self.se.backward(d, grads)
        return self.dw.backward(d, grads)


class TokenMixerUnit:
    def __init__(self, tm: nn.Sequential, use_se: bool):
        self.rv = RepVGGDWUnit(tm[0])
        self.se = SEUnit(tm[1]) if use_se else None

    def forward(self, x):
        x = self.rv.forward(x)
        return self.se.forward(x) if self.se is not None else x

    def backward(self, dy, grads):
        if self.se is not None:
            dy = self.se.backward(dy, grads)
        return self.rv.backward(dy, grads)


_STEM_WIDTHS = (8, 16, 24, 32, 48)      # es3_stem_conv3x3_s2 instantiations
_STEM_WGRAD_MAX = 32                    # es3_stem_wgrad: one (output channel, tap) weight per thread, <= 32 channels per launch


class PaddedStemUnit:
    """First patch-embed conv (3 -> C, 3x3, stride 2) + BN + GELU when C is not a width the stem kernels are instantiated for
    (repvit_m2_3: 40): the conv, its BatchNorm vectors and the running statistics are zero-/one-padded to the next instantiated
    width P, so the extra channels are exactly zero after the GELU; the weight gradient runs in chunks of <= 32 output channels.
    Returns / consumes [B,H,W,P] activations (the following conv is padded to P input channels as well)."""

    def __init__(self, cb: Conv2d_BN):
        self.conv, self.bn = cb.c, cb.bn
        c = cb.c.out_channels
        wider = [w for w in _STEM_WIDTHS if w >= c]
        if not wider:
            raise NotImplementedError(f"stem conv with {c} output channels exceeds the instantiated widths {_STEM_WIDTHS}")
        self.c, self.p = c, wider[0]
        self.saved = None

    def _pad(self, v, fill):
        out = torch.full((self.p,), fill, device=v.device, dtype=torch.float32)
        out[:self.c] = v.detach().float()
        return out

    def forward(self, x):
        conv, bn, c, p = self.conv, self.bn, self.c, self.p
        w27 = torch.zeros((27, p), device=x.device, dtype=torch.float32)
        w27[:, :c] = conv.weight.detach().float().reshape(c, 27).t()
        z = ops.stem_conv3x3_s2(x, w27, None, None)                              # [B,Ho,Wo,P], extra channels = 0
        gamma, beta = self._pad(bn.weight, 1.0), self._pad(bn.bias, 0.0)
        sync = None
        if bn.training:
            rm, rv = self._pad(bn.running_mean, 0.0), self._pad(bn.running_var, 1.0)
            mean, invstd, scale, shift, sync = sync_bn.batch_stats(bn, z, gamma, beta, rm, rv)
            bn.running_mean.copy_(rm[:c])
            bn.running_var.copy_(rv[:c])
            mode = "batch"
        else:
            mean = self._pad(bn.running_mean, 0.0)
            invstd = torch.rsqrt(self._pad(bn.running_var, 1.0) + bn.eps).contiguous()
            scale = (gamma * invstd).contiguous()
            shift = (beta - mean * scale).contiguous()
            mode = "eval"
        self.saved = (x, z, scale, shift, mean, invstd, mode, sync)
        return ops.affine_act(z, scale, shift, "gelu")

    def backward(self, da, grads):
        x, z, scale, shift, mean, invstd, mode, sync = self.saved
        self.saved = None
        conv, bn, c, p = self.conv, self.bn, self.c, self.p
        dev = z.device
        dg, db = torch.zeros(p, device=dev, dtype=torch.float32), torch.zeros(p, device=dev, dtype=torch.float32)
        dz = sync_bn.bn_act_bwd(da.contiguous(), z, scale, shift, "gelu", mode, mean, invstd, dg, db, sync)
        g_w, g_b = _grad_of(grads, bn.weight), _grad_of(grads, bn.bias)
        if g_w is not None:
            g_w += dg[:c]
        if g_b is not None:
            g_b += db[:c]
        gw = _grad_of(grads, conv.weight)
        if gw is not None:      # chunks of output channels in widths the weight-gradient kernel is instantiated for (40 = 32 + 8)
            c0 = 0
            while c0 < c:
                n = max(w for w in _STEM_WIDTHS if w <= min(_STEM_WGRAD_MAX, c - c0))
                tmp = torch.zeros((n, 3, 3, 3), device=dev, dtype=torch.float32)
                ops.stem_wgrad(x, dz[..., c0:c0 + n].contiguous(), tmp)
                gw[c0:c0 + n] += tmp
                c0 += n


# stride-2 3x3 taps on the 2x2 phase decomposition of the input: input row 2 oy + k - 1 = 2 (oy + shift) + phase
_TAP = {0: (1, -1), 1: (0, 0), 2: (1, 0)}          # k -> (phase, shift of the OUTPUT index inside that phase image)


class PatchEmbedUnit:
    """Conv2d_BN(3, C/2, 3, 2, 1) -> GELU -> Conv2d_BN(C/2, C, 3, 2, 1)  (repvit.py:219-223)."""

    def __init__(self, pe: nn.Sequential):
        self.cb1 = pe[2]
        cmid = pe[2].c.in_channels
        # es3_conv3x3_s2_narrow_bf16 is instantiated for 32 / 48 input channels: narrower first convs (repvit_m0_9: 24,
        # repvit_m2_3: 40) are zero-padded, exactly as the eval path's pack_patch_embed does
        if cmid > 48:
            raise NotImplementedError(f"train-mode patch embed is built for a first conv of <= 48 channels; got {cmid}")
        self.cp = 32 if cmid <= 32 else 48
        # a first conv whose width the stem kernels are not instantiated for (40) runs zero-padded end to end
        self.padded_stem = cmid not in _STEM_WIDTHS or cmid > _STEM_WGRAD_MAX
        self.c0 = PaddedStemUnit(pe[0]) if self.padded_stem else _cu(pe[0], "gelu", "stem")
        self.saved = None

    def forward(self, x):
        a0 = self.c0.forward(x)                                                  # [B, H/2, W/2, Cmid] bf16
        conv, bn = self.cb1.c, self.cb1.bn
        cout, cin = conv.out_channels, conv.in_channels
        B, H, W, _ = a0.shape
        if H % 2 or W % 2:
            raise NotImplementedError("train-mode RepViT patch embed needs an even feature map after the first conv")
        cp = self.cp
        if a0.shape[-1] != cp:                                                   # zero-padded channels meet zero weights
            a0p = torch.zeros((B, H, W, cp), device=a0.device, dtype=a0.dtype)
            a0p[..., :a0.shape[-1]] = a0
            a0 = a0p
        w9 = torch.zeros((9, cout, cp), device=a0.device, dtype=torch.bfloat16)
        w9[:, :, :cin] = conv.weight.detach().permute(2, 3, 0, 1).reshape(9, cout, cin).to(torch.bfloat16)
        ones = torch.ones(cout, device=a0.device, dtype=torch.float32)
        z = ops.conv3x3_s2_narrow(a0, w9, ones, torch.zeros_like(ones), None)    # raw conv
        mean, invstd, scale, shift, mode, sync = _norm_params(bn, z)
        self.saved = (a0, z, w9, (mean, invstd, scale, shift, mode, sync))
        return ops.affine_act(z, scale, shift, None)

    def backward(self, dy, grads):
        a0, z, w9, (mean, invstd, scale, shift, mode, sync) = self.saved
        self.saved = None
        conv, bn = self.cb1.c, self.cb1.bn
        cout, cin_true = conv.out_channels, conv.in_channels
        B, H, W, cin = a0.shape                                                  # cin = padded width of the staged input
        Ho, Wo = H // 2, W // 2
        dz = sync_bn.bn_act_bwd(dy.contiguous(), z, scale, shift, None, mode, mean, invstd, _grad_of(grads, bn.weight),
                                _grad_of(grads, bn.bias), sync)
        dz2 = dz.view(-1, cout)
        # weight gradient: tap (ky, kx) reads phase (py, px) of a0 at a stride-1 shift
        gw_true = _grad_of(grads, conv.weight)
        gw = gw_true if cin == cin_true else (torch.zeros((cout, cin, 3, 3), device=a0.device, dtype=torch.float32)
                                             if gw_true is not None else None)
        if gw is not None:
            flat = gw.view(-1)
            phase = {(py, px): a0[:, py::2, px::2, :].contiguous().view(-1, cin) for py in (0, 1) for px in (0, 1)}
            for ky in range(3):
                py, sy = _TAP[ky]
                for kx in range(3):
                    px, sx = _TAP[kx]
                    ops.wgrad_pw(dz2, phase[(py, px)], flat[ky * 3 + kx:], ldn=9 * cin, ldk=9, shift=(Ho, Wo, sy, sx))
            if gw is not gw_true:
                gw_true += gw[:, :cin_true]
        # input gradient, phase by phase: d a0[2y'+py, 2x'+px] = sum over the taps landing on that phase of dz[y'-sy, x'-sx] W_tap
        shifted = {}

        def dz_at(oy_off, ox_off):          # dz read at (y' + oy_off, x' + ox_off), zero outside, as a [M, cout] matrix
            key = (oy_off, ox_off)
            if key not in shifted:
                if key == (0, 0):
                    shifted[key] = dz2
                else:
                    t = torch.zeros_like(dz)
                    t[:, :Ho - oy_off, :Wo - ox_off] = dz[:, oy_off:, ox_off:]
                    shifted[key] = t.view(-1, cout)
            return shifted[key]

        da0 = torch.empty_like(a0)
        for py in (0, 1):
            for px in (0, 1):
                acc = None
                for ky in range(3):
                    if _TAP[ky][0] != py:
                        continue
                    for kx in range(3):
                        if _TAP[kx][0] != px:
                            continue
                        wt = w9[ky * 3 + kx].t().contiguous()                    # [cin, cout]: d a0 = dz . W_tap
                        acc = ops.gemm(dz_at(-_TAP[ky][1], -_TAP[kx][1]), wt, residual=acc)
                da0[:, py::2, px::2, :] = acc.view(B, Ho, Wo, cin)
        if self.padded_stem:
            self.c0.backward(da0[..., :self.c0.p].contiguous(), grads)
            return None
        if cin != cin_true:
            da0 = da0[..., :cin_true].contiguous()
        self.c0.backward(da0, grads, need_dx=False)
        return None


class RepViTTrainGraph:
    """Units of RepViT.features in execution order (repvit.py:219-246)."""

    def __init__(self, model):
        feats = list(model.features)
        self.patch = PatchEmbedUnit(feats[0])
        self.units = []
        for blk in feats[1:]:
            assert isinstance(blk, RepViTBlock)
            tm = blk.token_mixer
            self.units.append(TokenMixerDownUnit(tm, blk.use_se) if blk.stride == 2 else TokenMixerUnit(tm, blk.use_se))
            self.units.append(ChannelMixerUnit(blk.channel_mixer.m))

    def forward(self, x):
        x = self.patch.forward(x)
        for u in self.units:
            x = u.forward(x)
        return x

    def backward(self, d, grads):
        for u in reversed(self.units):
            d = u.backward(d, grads)
        self.patch.backward(d, grads)
