"""Host-side helpers shared by the module shells: BN folding, weight packing, plan caching.

The shells (`backbones/*.py`, `stage1/model.py`, ...) keep the reference's class names, constructor
signatures and state_dict keys; torch.nn.Conv2d / BatchNorm2d / Linear objects inside them are used
ONLY as parameter containers (their forward is never called) -- all device work goes through
`efficientsam3_b200.ops` -> libes3.so.
"""
from __future__ import annotations

import torch
import torch.nn as nn


def bn_scale_bias(norm: nn.BatchNorm2d | None, conv_bias: torch.Tensor | None, cout: int, device):
    """Eval-mode BatchNorm folded to per-channel (scale, bias) in fp32; conv bias merged.
    Returns (scale|None, bias|None)."""
    if norm is None:
        return None, (conv_bias.detach().float().contiguous() if conv_bias is not None else None)
    s = (norm.weight.detach().float() / torch.sqrt(norm.running_var.detach().float() + norm.eps))
    b = norm.bias.detach().float() - norm.running_mean.detach().float() * s
    if conv_bias is not None:
        b = b + conv_bias.detach().float() * s
    return s.contiguous(), b.contiguous()


# Packed / re-laid-out copies of a parameter are cached on the module that owns it and rebuilt when the parameter changes:
# (data_ptr, _version) catches torch-side writes, WEIGHTS_EPOCH the fused AdamW kernel, which moves the parameters through raw
# pointers (stage1.optim.FlatAdamW.step bumps it).  The training graphs re-derive ~150 such tensors per iteration (bf16 casts,
# transposes for the input-gradient GEMMs, rotated depthwise taps): with the cache they are built once per optimiser step.
WEIGHTS_EPOCH = 0


def bump_weights_epoch():
    global WEIGHTS_EPOCH
    WEIGHTS_EPOCH += 1


def cached_pack(owner: nn.Module, name: str, src: torch.Tensor, fn):
    key = (src.data_ptr(), src._version, src.device, WEIGHTS_EPOCH)
    cache = owner.__dict__.setdefault("_es3_pack_cache", {})
    ent = cache.get(name)
    if ent is None or ent[0] != key:
        with torch.no_grad():
            ent = (key, fn())
        cache[name] = ent
    return ent[1]


def _pw_weight(conv):
    w = conv.weight.detach()
    return w.reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()


def pw_weight(conv: nn.Conv2d) -> torch.Tensor:
    """1x1 conv weight [N,C,1,1] -> bf16 [N,C] (K-major GEMM B operand)."""
    return cached_pack(conv, "pw", conv.weight, lambda: _pw_weight(conv))


def pw_weight_scaled(conv: nn.Conv2d, scale: torch.Tensor | None) -> torch.Tensor:
    """1x1 conv weight with the folded BatchNorm scale multiplied in BEFORE the bf16 rounding: bf16 [N,C].  The GEMM epilogue of an
    eval-mode conv + BN is then bias (+ act) only: the per-channel scale cost 8 broadcast LDG.128 + 32 FMUL per 32-column chunk of
    every row."""
    w = conv.weight.detach().float().reshape(conv.out_channels, -1)
    if scale is not None:
        w = w * scale.view(-1, 1)
    return w.to(torch.bfloat16).contiguous()


def pw_weight_t(conv: nn.Conv2d) -> torch.Tensor:
    """bf16 [C,N]: the transposed 1x1 weight, B operand of the input-gradient GEMM dx = dz . W."""
    return cached_pack(conv, "pw_t", conv.weight, lambda: _pw_weight(conv).t().contiguous())


def _dw_weight(conv, scale):
    w = conv.weight.detach().float()
    c, _, k, _ = w.shape
    if scale is not None:
        w = w * scale.view(-1, 1, 1, 1)
    return w.reshape(c, k * k).t().contiguous()


def dw_weight(conv: nn.Conv2d, scale: torch.Tensor | None) -> torch.Tensor:
    """depthwise weight [C,1,k,k] (x folded BN scale) -> fp32 [k*k, C] tap-major."""
    if scale is not None:
        return _dw_weight(conv, scale)
    return cached_pack(conv, "dw", conv.weight, lambda: _dw_weight(conv, None))


def dw_weight_rot(conv: nn.Conv2d) -> torch.Tensor:
    """fp32 [k*k, C] with the taps rotated by 180 degrees: the stride-1 input gradient is the forward kernel on these."""
    return cached_pack(conv, "dw_rot", conv.weight, lambda: _dw_weight(conv, None).flip(0).contiguous())


def pack_patch_embed(w0: torch.Tensor, s0, b0, w1: torch.Tensor):
    """Two-conv patch embed (3 -> C/2 -> C, both 3x3 stride 2; repvit.py:219-223, tiny_vit.py:67-84) packed for
    es3_stem_conv3x3_s2 + es3_conv3x3_s2_narrow_bf16.  The intermediate width C/2 (24/32/40/48) is zero-padded to the
    kernel widths 32 / 48: padded channels carry weight 0 and bias 0, so they stay act(0) = 0 and meet zero weights again.
    Returns (w27 fp32 [27, Cp] with BN scale folded, bias [Cp], w9 bf16 [9, Cout, Cp])."""
    cmid, cout = w0.shape[0], w1.shape[0]
    cp = 32 if cmid <= 32 else 48
    if cmid > 48:
        raise NotImplementedError(f"patch embed with a {cmid}-channel first conv is not instantiated (<= 48)")
    w0 = w0.detach().float()
    if s0 is not None:
        w0 = w0 * s0.view(-1, 1, 1, 1)
    w27 = torch.zeros(27, cp, device=w0.device, dtype=torch.float32)
    w27[:, :cmid] = w0.reshape(cmid, 27).t()
    bias = torch.zeros(cp, device=w0.device, dtype=torch.float32)
    if b0 is not None:
        bias[:cmid] = b0
    w9 = torch.zeros(9, cout, cp, device=w0.device, dtype=torch.bfloat16)
    w9[:, :, :cmid] = w1.detach().permute(2, 3, 0, 1).reshape(9, cout, cmid).to(torch.bfloat16)
    return w27.contiguous(), bias, w9.contiguous()


def conv3x3_weight(conv: nn.Conv2d) -> torch.Tensor:
    """dense 3x3 weight [N,C,3,3] -> bf16 [N, 9*C] with k = (ky*3+kx)*C + c."""
    w = conv.weight.detach()
    n, c = w.shape[:2]
    return w.permute(0, 2, 3, 1).reshape(n, 9 * c).to(torch.bfloat16).contiguous()


def params_fingerprint(module: nn.Module):
    """Cheap change detector for cached packed weights: (data_ptr, _version) of every tensor."""
    fp = []
    for t in list(module.parameters()) + list(module.buffers()):
        fp.append((t.data_ptr(), t._version))
    return tuple(fp)


class NativePlanMixin:
    """Caches packed / folded weights; rebuilds when parameters, device or mode change."""

    def _plan(self):
        from . import ops
        key = (params_fingerprint(self), self.training, ops.precision())
        if getattr(self, "_plan_key", None) != key:
            self._plan_cache = self._build_plan()
            self._plan_key = key
        return self._plan_cache

    def _require_eval(self, what: str):
        if self.training:
            raise NotImplementedError(
                f"{what}: this module's native sm_90a path is eval-mode only (train-mode forward / backward exist for the "
                "stage-1 student encoders: ImageStudentEncoder; see DESIGN.md).  Call .eval() first.")


class StagedGraphMixin:
    """CUDA-graph replay of an eval forward whose inputs arrive from the host (the text encoders: token ids validated on the
    host, EOT row indices; the point-prompt predictor: prompt coordinates and labels scaled on the host).  One graph per key
    (shapes, input kind, device): its inputs are static device buffers, refilled before each replay -- host tensors of any
    dtype through one pinned staging buffer (one asynchronous copy), CUDA tensors device to device -- and its outputs are the
    graph's own buffers, overwritten by the next replay with the same key.

    A graph reads the packed weights of every NativePlanMixin below the modules it runs (the module itself unless `_graphed`
    names others) by address, so it is captured again when a parameter or buffer of those modules moves (params_fingerprint: optimiser steps through torch, load_state_dict, a replaced Parameter, a move
    to another device) or a plan was invalidated (FlatAdamW's step and the batch-statistics BatchNorm reset `_plan_key`).  The
    entry keeps the plans it was captured with alive, so a stale graph never reads freed memory.  At most `max_graphs` graphs are
    kept; the oldest capture is evicted first."""

    _graphs = None
    graph_launches_per_step = 0     # kernels of the graph replayed last (es3 launches, as ops.launch_count counts them)

    def enable_cuda_graphs(self, enabled: bool = True, max_graphs: int = 4):
        """Replay the eval forward from CUDA graphs (off by default).  Returns self."""
        if max_graphs < 1:
            raise ValueError(f"max_graphs must be >= 1, got {max_graphs}")
        self._graphs = {} if enabled else None
        self._graph_max = max_graphs
        return self

    def _graphed(self, key, host, dev_in, fn, modules=None):
        """fn(*static inputs) -> outputs, replayed from the graph of `key` (its last element is the device).  host: CPU tensors,
        dev_in: CUDA tensors; fn receives device buffers of the same shapes and dtypes, host ones first.  modules: the modules
        whose parameters and plans the graph reads (default: this module)."""
        dev = key[-1]
        modules = (self,) if modules is None else tuple(modules)
        fp = tuple(params_fingerprint(m) for m in modules)
        ent = self._graphs.get(key)
        with torch.cuda.device(dev):
            if ent is None or ent["fp"] != fp or any(getattr(m, "_plan_key", None) is not k for m, k, _ in ent["plans"]):
                del ent                             # release the stale graph's memory before capturing its successor
                self._graphs.pop(key, None)
                ent = self._capture(dev, host, dev_in, fn, fp, modules)
                while len(self._graphs) >= self._graph_max:
                    self._graphs.pop(next(iter(self._graphs)))
                self._graphs[key] = ent
            else:
                self._stage(ent, host, dev_in)
            ent["graph"].replay()
        self.graph_launches_per_step = ent["launches"]
        return ent["out"]

    @staticmethod
    def _host_offsets(host):
        """Byte offset of each host tensor in the staging buffer (16-byte aligned, so every dtype can be viewed in place)."""
        offs, o = [], 0
        for h in host:
            offs.append(o)
            o += (h.numel() * h.element_size() + 15) // 16 * 16
        return offs, o

    @staticmethod
    def _stage(ent, host, dev_in):
        if host:
            ent["copied"].synchronize()             # the previous replay's copy out of the pinned buffer has been read
            for h, o in zip(host, ent["offs"]):
                b = h.reshape(-1).view(torch.uint8)
                ent["pinned"][o:o + b.numel()].copy_(b)
            ent["flat"].copy_(ent["pinned"], non_blocking=True)
            ent["copied"].record()
        for s, t in zip(ent["dev_in"], dev_in):
            s.copy_(t)

    def _capture(self, dev, host, dev_in, fn, fp, modules):
        from . import ops
        offs, n = self._host_offsets(host)
        ent = dict(fp=fp, offs=offs, pinned=torch.empty(n, dtype=torch.uint8, pin_memory=True),
                   flat=torch.empty(n, dtype=torch.uint8, device=dev), copied=torch.cuda.Event(),
                   dev_in=[torch.empty(t.shape, dtype=t.dtype, device=t.device) for t in dev_in])
        static = [ent["flat"][o:o + h.numel() * h.element_size()].view(h.dtype).view(h.shape) for h, o in zip(host, offs)]
        static += ent["dev_in"]
        self._stage(ent, host, dev_in)
        fn(*static)                                 # un-captured pass: packs weights, builds positional tables, configures kernels
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count
        # thread_local: another thread may wait on CUDA events meanwhile (the embedding dump's writer thread does)
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            out = fn(*static)
        ent.update(graph=graph, out=out, launches=ops.launch_count - n0,
                   plans=[(m, getattr(m, "_plan_key", None), getattr(m, "_plan_cache", None)) for top in modules
                          for m in top.modules() if isinstance(m, NativePlanMixin)])
        return ent
