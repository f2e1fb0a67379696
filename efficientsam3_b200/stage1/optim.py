"""Optimiser side of the stage-1 KD step on flat arenas (SURVEY.md §8 A19/A20, multi-GPU row (e)).

Reference pieces replaced:
  build_optimizer / set_weight_decay   stage1/optimizer.py:6-45    AdamW; 1-D params, `.bias`, skip-list names -> no decay
  NativeScalerWithGradNormCount        stage1/utils.py:341-368     scale(loss).backward, unscale_, clip_grad_norm_, step, update
  DDP bucketed allreduce               train_image_encoder_stage1.py:96-101 (DistributedDataParallel)
  build_scheduler (cosine)             stage1/lr_scheduler.py:9-48 -> timm CosineLRScheduler(t_in_epochs=False, cycle_limit=1)
  linear LR scaling                    train_image_encoder_stage1.py:347-373  lr * batch * world / 512

Design: every trainable parameter is a view into ONE contiguous fp32 arena ([decay group | no-decay group]); grads,
exp_avg and exp_avg_sq are arenas of the same layout.  A step is: one NCCL all-reduce of the grad arena (sum), one
two-stage norm kernel, one fused AdamW kernel that reads the norm / non-finite flag / loss scale from device memory.
No host synchronisation, no per-tensor launches (the reference's foreach path launches per dtype/shape bucket and syncs on
found_inf).  What is NOT here: the student's backward (train-mode BN, conv / LiteMLA gradients) -- see DESIGN.md scope.
"""
from __future__ import annotations

import math

import torch

from .. import ops


def scaled_lr(base_lr: float, batch_size: int, world_size: int) -> float:
    """train_image_encoder_stage1.py:347-373: linear scaling by the global batch over 512."""
    return base_lr * batch_size * world_size / 512.0


def cosine_lr(t: int, base_lr: float, t_initial: int, lr_min: float, warmup_t: int, warmup_lr_init: float) -> float:
    """timm CosineLRScheduler._get_lr with t_in_epochs=False, cycle_limit=1, cycle_mul=1, warmup_prefix=False
    (pin timm>=1.0.17, not vendored: restated).  Called once per optimiser update (`step_update`)."""
    if t < warmup_t:
        return warmup_lr_init + t * (base_lr - warmup_lr_init) / warmup_t
    if t >= t_initial:           # past the single cycle
        return lr_min
    return lr_min + 0.5 * (base_lr - lr_min) * (1.0 + math.cos(math.pi * t / t_initial))


def split_decay(named_params, skip_list=(), skip_keywords=()):
    """stage1/optimizer.py:33-45 (set_weight_decay + check_keywords_in_name)."""
    decay, no_decay = [], []
    for name, p in named_params:
        if not p.requires_grad:
            continue
        if p.dim() == 1 or name.endswith(".bias") or name in skip_list or any(k in name for k in skip_keywords):
            no_decay.append((name, p))
        else:
            decay.append((name, p))
    return decay, no_decay


class FlatAdamW:
    """AdamW + GradScaler + grad clipping + data-parallel gradient exchange over flat arenas."""

    ALIGN = 4   # floats: every parameter starts 16-byte aligned inside the arena

    def __init__(self, model: torch.nn.Module, lr: float, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01,
                 loss_scale: float = 1.0, dynamic_loss_scale: bool = False, growth_interval: int = 2000,
                 direct_grads: bool = True, overlap_allreduce: bool = True, exclude=()):
        skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else ()
        skip_kw = model.no_weight_decay_keywords() if hasattr(model, "no_weight_decay_keywords") else ()
        # `exclude`: parameter names left out of the arenas entirely (never updated, never decayed, `.grad` untouched), e.g. the
        # text student's unused `encoder.projection_layer`, which torch AdamW skips in the reference because its grad stays None
        excluded = set(exclude)
        unknown = excluded - {n for n, _ in model.named_parameters()}
        if unknown:
            raise ValueError(f"FlatAdamW(exclude=...): no parameter named {sorted(unknown)}")
        decay, no_decay = split_decay(((n, p) for n, p in model.named_parameters() if n not in excluded), skip, skip_kw)
        self._model = model
        self._plan_holders = None
        self.lr, self.betas, self.eps, self.weight_decay = lr, tuple(betas), eps, weight_decay
        # the configured LR the schedule is built from (timm keeps it as param_group['initial_lr']); `self.lr` is the value of the
        # current update and moves with the schedule, `base_lr` never does
        self.base_lr = lr
        self.dynamic, self.growth_interval = dynamic_loss_scale, growth_interval
        self.names, self.params, self.offsets = [], [], []
        off = 0
        for group in (decay, no_decay):
            for name, p in group:
                self.names.append(name); self.params.append(p); self.offsets.append(off)
                off += -(-p.numel() // self.ALIGN) * self.ALIGN
            if group is decay:
                self.n_decay = off
        self.numel = off
        dev = self.params[0].device if self.params else torch.device("cpu")
        mk = lambda: torch.zeros(self.numel, device=dev, dtype=torch.float32)
        self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq = mk(), mk(), mk(), mk()
        for p, o in zip(self.params, self.offsets):
            if p.dtype != torch.float32:
                raise TypeError("FlatAdamW keeps fp32 master parameters; got " + str(p.dtype))
            view = self.flat_param[o:o + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
            p.grad = self.flat_grad[o:o + p.numel()].view_as(p)
        # device-resident scaler / step state: [loss scale, growth tracker, step count, last total norm]
        self.state = torch.tensor([loss_scale, 0.0, 0.0, 0.0], device=dev, dtype=torch.float32)
        self._norm_ws = torch.zeros(2, device=dev, dtype=torch.float32)
        self._part_ws = torch.zeros(8192, device=dev, dtype=torch.float32)
        # The native student's backward accumulates straight into the arena views (`p.grad`) instead of returning per-parameter
        # gradients to autograd.  Do NOT combine with torch DDP (its hooks would never see a gradient): this class owns the exchange.
        self._pending, self._exchange_on, self._group = [], False, None
        self.early_exchanges = 0
        self.overlap = bool(overlap_allreduce)
        head = [o for n, o in zip(self.names, self.offsets) if n.startswith("head.") and o < self.n_decay]
        self._head_lo = min(head) if head else self.n_decay        # [head_lo, n_decay): head.0.weight, head.3.weight (decay group tail)
        if direct_grads and (hasattr(model, "head") or getattr(model, "supports_direct_grads", False)):
            model._es3_grad_arena = self
        self.overlap_note = ("two buckets: the head's weight gradients [%d, %d) are all-reduced asynchronously as soon as the head's backward "
                             "has been enqueued (they overlap the backbone's backward), the rest after the backward returns"
                             % (self._head_lo, self.n_decay)) if self.overlap else "blocking, after the backward returns"

    # ---- step pieces ---------------------------------------------------------------------------------------------------
    def zero_grad(self):
        self.flat_grad.zero_()

    @property
    def loss_scale_tensor(self):
        """Device float the backward kernels multiply by (es3_kd_loss_bwd scale_dev)."""
        return self.state[0:1]

    def begin_backward(self, exchange: bool, group=None):
        """Called by kd_train_step before `loss.backward()`: `exchange` = this backward ends an accumulation window, so finished
        ranges of the arena may be handed to NCCL from inside the backward (head_grads_ready)."""
        self._exchange_on, self._group = bool(exchange), group

    def head_grads_ready(self):
        """Hook of the native student's backward (stage1/model.StudentTrainFunction): every gradient in [head_lo, n_decay) is final.
        Launch their all-reduce now; it runs on NCCL's stream behind the kernels enqueued so far and overlaps the backbone backward."""
        import torch.distributed as dist
        if not (self.overlap and self._exchange_on and self._head_lo < self.n_decay):
            return
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self._group) > 1:
            w = dist.all_reduce(self.flat_grad[self._head_lo:self.n_decay], op=dist.ReduceOp.SUM, group=self._group, async_op=True)
            self._pending.append(w)
            self.early_exchanges += 1

    def all_reduce_grads(self, group=None):
        """The collective of the data-parallel step (SURVEY.md §8e): sum over ranks of the whole grad arena; the mean (1 / world) is
        folded into the AdamW kernel's gradient multiplier.  One all-reduce of the arena, or -- when the backward already handed
        the head range to NCCL (head_grads_ready) -- the remaining two ranges, after which the early one is waited for."""
        import torch.distributed as dist
        self._exchange_on = False
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            if self._pending:
                if self._head_lo > 0:
                    dist.all_reduce(self.flat_grad[:self._head_lo], op=dist.ReduceOp.SUM, group=group)
                if self.n_decay < self.numel:
                    dist.all_reduce(self.flat_grad[self.n_decay:], op=dist.ReduceOp.SUM, group=group)
                for w in self._pending:
                    w.wait()
                self._pending = []
            else:
                dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=group)
            return dist.get_world_size(group)
        return 1

    def step(self, lr: float | None = None, max_norm: float = 5.0, world_size: int = 1):
        """unscale -> global-norm clip -> AdamW -> scaler update, all on the device.  `world_size`: number of ranks whose
        gradients were summed into the arena.  The total norm of the last step is state[3] (read it lazily)."""
        if not self.flat_param.is_cuda:
            raise RuntimeError("FlatAdamW.step runs es3_adamw_flat on the GPU; there is no CPU fallback")
        if lr is not None:
            self.lr = lr
        # the kernel moves the parameters through raw pointers: cached eval-mode packings are stale.  The holders are collected
        # once (a per-step walk over every module cost 0.2 ms of host time per update, VERDICT r1 weak #12)
        if self._plan_holders is None:
            self._plan_holders = [mod for mod in self._model.modules() if hasattr(mod, "_plan_key")]
        for mod in self._plan_holders:
            mod._plan_key = None
        from ..nn_utils import bump_weights_epoch
        bump_weights_epoch()                     # packed training-graph weights (nn_utils.cached_pack) are stale as well
        ops.grad_norm(self.flat_grad, self._part_ws, self._norm_ws)
        ops.adamw_flat(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, self.n_decay, self.lr, self.betas,
                       self.eps, self.weight_decay, max_norm, 1.0 / world_size, self._norm_ws, self.state,
                       dynamic_scale=self.dynamic, growth_interval=self.growth_interval)

    def last_grad_norm(self) -> float:
        return float(self.state[3].item())

    def step_count(self) -> int:
        return int(self.state[2].item())

    # ---- checkpoint interop with torch.optim.AdamW (stage1/utils.py:286-298 saves optimizer.state_dict()) -----------------
    def state_dict(self):
        step = float(self.state[2].item())
        state = {}
        for i, (p, o) in enumerate(zip(self.params, self.offsets)):
            sl = slice(o, o + p.numel())
            state[i] = dict(step=torch.tensor(step), exp_avg=self.exp_avg[sl].view_as(p).clone(),
                            exp_avg_sq=self.exp_avg_sq[sl].view_as(p).clone())
        n_dec = sum(1 for o in self.offsets if o < self.n_decay)
        common = dict(lr=self.lr, initial_lr=self.base_lr, betas=self.betas, eps=self.eps, amsgrad=False, maximize=False)
        groups = [dict(common, weight_decay=self.weight_decay, params=list(range(n_dec))),
                  dict(common, weight_decay=0.0, params=list(range(n_dec, len(self.params))))]
        return dict(state=state, param_groups=groups,
                    amp_scaler=dict(scale=float(self.state[0].item()), _growth_tracker=int(self.state[1].item())))

    def load_state_dict(self, sd):
        for i, (p, o) in enumerate(zip(self.params, self.offsets)):
            st = sd["state"].get(i)
            if st is None:
                continue
            sl = slice(o, o + p.numel())
            self.exp_avg[sl].copy_(st["exp_avg"].reshape(-1))
            self.exp_avg_sq[sl].copy_(st["exp_avg_sq"].reshape(-1))
            self.state[2] = float(st["step"])
        if sd.get("param_groups"):
            g0 = sd["param_groups"][0]
            self.lr = g0["lr"]
            # timm schedulers write `initial_lr` into every group; a checkpoint without it (plain torch AdamW that never met a
            # scheduler) leaves the configured base LR of this object untouched rather than adopting a mid-schedule value
            if "initial_lr" in g0:
                self.base_lr = g0["initial_lr"]
        sc = sd.get("amp_scaler")
        if sc:
            self.state[0] = float(sc["scale"])
            self.state[1] = float(sc.get("_growth_tracker", 0))


class KDLossFunction(torch.autograd.Function):
    """loss = masked MSE + w * masked cosine (kd_loss.cu) with the analytic backward kernel: lets the KD loss sit at the
    end of an autograd graph (`loss.backward()` reaches `preds.grad` through es3_kd_loss_bwd)."""

    @staticmethod
    def forward(ctx, preds, teacher, sizes_hw, img_size, cosine_weight):
        out, per = ops.kd_loss_fwd(preds.detach(), teacher, sizes_hw, img_size, cosine_weight)
        ctx.save_for_backward(preds.detach(), teacher, sizes_hw, per)
        ctx.meta = (img_size, cosine_weight)
        return out[0].clone()

    @staticmethod
    def backward(ctx, grad_out):
        preds, teacher, sizes_hw, per = ctx.saved_tensors
        img_size, w = ctx.meta
        g = ops.kd_loss_bwd(preds, teacher, sizes_hw, per, img_size, w, 1.0, grad_out.reshape(1).float().contiguous())
        return g, None, None, None, None
