"""CPU, gloo: synchronised BatchNorm (nn.SyncBatchNorm.convert_sync_batchnorm) on the native image-student training graphs.

The libes3 ops run as their fp64 torch statements (tests/emu_ops.py, plus the SyncBN ops below), so what is checked is the host
logic: which BatchNorms synchronise, what travels in the all-gathers, and the algebra of the split statistics / backward.  A
2-rank step of a converted student must reproduce the global-batch step of the unconverted one."""
import os
import socket
import sys
from types import SimpleNamespace as NS

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import emu_ops

_HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------ the SyncBN ops as torch statements
def bn_stats_partial(z):
    C = z.shape[-1]
    zf = z.to(torch.float64).reshape(-1, C)
    mean = zf.mean(0)
    return torch.stack([torch.full((C,), float(zf.shape[0]), dtype=torch.float64), mean, (zf - mean).pow(2).sum(0)])


def bn_stats_combine(parts, gamma, beta, eps, momentum, running_mean=None, running_var=None, num_batches_tracked=None):
    n = torch.zeros(parts.shape[2], dtype=torch.float64)
    mu, m2 = torch.zeros_like(n), torch.zeros_like(n)
    for p in parts:                                                   # Chan's combination in rank order, as the kernel
        nb, d = p[0], p[1] - mu
        nn_ = n + nb
        mu = mu + d * nb / nn_
        m2 = m2 + p[2] + d * d * n * nb / nn_
        n = nn_
    var = m2 / n
    invstd = torch.rsqrt(var + eps)
    scale = gamma.to(torch.float64) * invstd
    shift = beta.to(torch.float64) - mu * scale
    if running_mean is not None:
        running_mean.mul_(1 - momentum).add_(momentum * mu)
    if running_var is not None:
        running_var.mul_(1 - momentum).add_(momentum * var * n / (n - 1))
    if num_batches_tracked is not None:
        num_batches_tracked += 1
    return mu, invstd, scale, shift, n[:1].clone()


def _g(da, z, scale, shift, act):
    C = z.shape[-1]
    zf = z.to(torch.float64).reshape(-1, C)
    u = (zf * scale + shift).requires_grad_(True)
    with torch.enable_grad():
        (g,) = torch.autograd.grad(emu_ops._act(u, act), u, da.to(torch.float64).reshape(-1, C))
    return g, zf


def bn_act_bwd_partial(da, z, scale, shift, act, mean, invstd, dgamma=None, dbeta=None):
    g, zf = _g(da, z, scale, shift, act)
    sg, sgx = g.sum(0), (g * (zf - mean)).sum(0)
    if dgamma is not None:
        dgamma += invstd * sgx
    if dbeta is not None:
        dbeta += sg
    return torch.stack([sg, sgx])


def bn_bwd_coef(parts, total, scale, mean, invstd):
    sg, sgx = parts[:, 0].sum(0), parts[:, 1].sum(0)
    mg, mgx = sg / total, invstd * sgx / total
    return torch.stack([scale, -scale * invstd * mgx, -scale * mg + scale * invstd * mean * mgx])


def bn_act_bwd_apply(da, z, scale, shift, act, coef):
    g, zf = _g(da, z, scale, shift, act)
    return (coef[0] * g + coef[1] * zf + coef[2]).reshape(z.shape).to(emu_ops.BF)


SYNC_OPS = ["bn_stats_partial", "bn_stats_combine", "bn_act_bwd_partial", "bn_bwd_coef", "bn_act_bwd_apply"]


class _Patch:
    def setattr(self, obj, name, value):
        setattr(obj, name, value)


def _install_exact(patch):
    from efficientsam3_b200 import ops
    emu_ops.install(patch)
    me = sys.modules[__name__]
    for name in SYNC_OPS:
        patch.setattr(ops, name, getattr(me, name))
    patch.setattr(emu_ops, "BF", torch.float64)
    patch.setattr(emu_ops, "CD", torch.float64)
    patch.setattr(ops, "ACT_DTYPE", torch.float64)


def _student(name, img, embed):
    from efficientsam3_b200.stage1.model import build_image_student_model
    from oracle.weights import fill_state_dict
    m = build_image_student_model(NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed)))
    m.load_state_dict(fill_state_dict(m.state_dict(), 5))
    return m.train()


def _buffers(m):
    return {k: v.clone() for k, v in m.state_dict().items() if "running_" in k or "num_batches" in k}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(target, world, *args, timeout=600):
    """Spawn `world` ranks, collect one result each, join with timeouts and terminate whatever is left on failure."""
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=target, args=(r, world, port, q, *args)) for r in range(world)]
    try:
        for p in ps:
            p.start()
        res = sorted((q.get(timeout=timeout) for _ in range(world)), key=lambda r: r[0])
    finally:
        for p in ps:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    for r in res:
        if isinstance(r[1], str):
            raise AssertionError(f"rank {r[0]}: {r[1]}")
    return res


def _init(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(4)
    sys.path.insert(0, _HERE)
    dist.init_process_group("gloo", rank=rank, world_size=world)


# ------------------------------------------------------------------------------------------ 2-rank KD step vs the global batch
def _dp_worker(rank, world, port, q, name, img, embed, counts):
    import traceback
    try:
        _init(rank, world, port)
        _install_exact(_Patch())
        from efficientsam3_b200.stage1.optim import FlatAdamW
        from oracle.kd_loss import kd_loss
        n_all = sum(counts)
        g = torch.Generator().manual_seed(7)
        x_all = torch.randn(n_all, 3, img, img, generator=g)
        t_all = torch.randn(n_all, 1024, embed, embed, generator=g).double()
        sizes = [(3, img, img)] * n_all

        ref = _student(name, img, embed)                     # global batch, plain BatchNorm2d with batch statistics
        ropt = FlatAdamW(ref, lr=1e-3)
        ropt.zero_grad()
        ref_out = ref(x_all)
        rl, _, _ = kd_loss(ref_out, t_all, img, sizes, 1.0)
        rl.backward()

        m = _student(name, img, embed)
        opt = FlatAdamW(m, lr=1e-3)                          # converted after the optimiser took the parameters, as the reference
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
        assert any(isinstance(mod, torch.nn.SyncBatchNorm) for mod in m.modules())
        opt.zero_grad()
        lo = sum(counts[:rank])
        sl = slice(lo, lo + counts[rank])
        out = m(x_all[sl])
        loss, _, _ = kd_loss(out, t_all[sl], img, sizes[sl], 1.0)
        loss = loss * (world * counts[rank] / n_all)         # the global loss is the ranks' losses weighted by their batch share
        opt.begin_backward(True)
        loss.backward()
        n = opt.all_reduce_grads()
        out_err = ((out.detach() - ref_out.detach()[sl]).norm() / ref_out.detach()[sl].norm()).item()
        gerr = ((opt.flat_grad / n - ropt.flat_grad).norm() / ropt.flat_grad.norm()).item()
        rb, mb = _buffers(ref), _buffers(m)
        assert rb.keys() == mb.keys() and rb
        buf_err = max(((mb[k].double() - rb[k].double()).norm() / rb[k].double().norm().clamp_min(1e-30)).item()
                      for k in rb if "running_" in k)
        nbt_ok = all(torch.equal(mb[k], rb[k]) for k in rb if "num_batches" in k)
        # a list, not a tensor: a CPU tensor on the queue is passed as a file descriptor that the rank, exiting, may
        # close before the parent has taken it
        flat = torch.cat([v.double().reshape(-1) for v in mb.values()]).tolist()
        q.put((rank, out_err, gerr, buf_err, nbt_ok, flat))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


@pytest.mark.parametrize("name,img,embed", [("efficientvit_b0", 160, 12), ("repvit_m0_9", 128, 8), ("tiny_vit_5m", 160, 12)])
def test_two_rank_syncbn_step_matches_the_global_batch(name, img, embed):
    res = _run(_dp_worker, 2, name, img, embed, [1, 1])
    for _, out_err, gerr, buf_err, nbt_ok, _ in res:
        assert out_err < 1e-9, out_err                       # each rank's output is its slice of the global-batch output
        assert gerr < 1e-5, gerr                             # fp32 accumulators in the arena are the only rounding left
        assert buf_err < 1e-6, buf_err                       # fp32 running buffers
        assert nbt_ok
    assert res[0][5] == res[1][5]                            # running buffers identical on both ranks


def test_uneven_batches_give_the_global_statistics():
    res = _run(_dp_worker, 2, "efficientvit_b0", 160, 12, [1, 2])
    for _, out_err, gerr, buf_err, nbt_ok, _ in res:
        assert out_err < 1e-9 and gerr < 1e-5 and buf_err < 1e-6 and nbt_ok, (out_err, gerr, buf_err)
    assert res[0][5] == res[1][5]


# ------------------------------------------------------------------------------------------ no synchronisation: unchanged path
def _step(m, x, t, img, embed):
    from oracle.kd_loss import kd_loss
    out = m(x)
    loss, _, _ = kd_loss(out, t, img, [(3, img, img)] * x.shape[0], 1.0)
    loss.backward()
    return out.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}, _buffers(m)


def _same_as_batchnorm2d(img=160, embed=12):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, img, img, generator=g)
    t = torch.randn(2, 1024, embed, embed, generator=g).double()
    a = _step(_student("efficientvit_b0", img, embed), x, t, img, embed)
    b = _step(torch.nn.SyncBatchNorm.convert_sync_batchnorm(_student("efficientvit_b0", img, embed)), x, t, img, embed)
    return (torch.equal(a[0], b[0]) and a[1].keys() == b[1].keys() and all(torch.equal(a[1][k], b[1][k]) for k in a[1])
            and all(torch.equal(a[2][k], b[2][k]) for k in a[2]))


def test_uninitialised_group_is_batchnorm2d(monkeypatch):
    from efficientsam3_b200 import sync_bn
    _install_exact(monkeypatch)
    before = sync_bn.exchanges
    assert _same_as_batchnorm2d()
    assert sync_bn.exchanges == before


def _world1_worker(rank, world, port, q):
    import traceback
    try:
        _init(rank, world, port)
        _install_exact(_Patch())
        from efficientsam3_b200 import sync_bn
        same = _same_as_batchnorm2d()
        q.put((rank, bool(same), sync_bn.exchanges))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


def test_world_one_is_batchnorm2d():
    (res,) = _run(_world1_worker, 1)
    assert res[1] and res[2] == 0, res


def test_sync_group_rules():
    from efficientsam3_b200.sync_bn import sync_group
    bn, sbn = torch.nn.BatchNorm2d(8), torch.nn.SyncBatchNorm(8)
    assert sync_group(bn) is None and sync_group(sbn) is None        # no process group
    assert sync_group(sbn.eval()) is None


# ------------------------------------------------------------------------------------------ MobileCLIP-S0
def _s0_cpu():
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    cfg = text_student_cfg("MobileCLIP-S0")
    cfg.update(n_transformer_layers=1, context_length=16)
    return TextStudentEncoder(cfg=cfg, context_length=16, output_dim=256)


def _s0_rules(what="S0"):
    from efficientsam3_b200.backbones.mobile_clip import check_trainable
    msgs = []
    for setup in ("plain", "mixed", "momentum", "frozen"):
        mm = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_s0_cpu())
        mm.train()
        if setup != "plain":
            mm.enable_batch_stat_bn()
        if setup == "mixed":
            mm.encoder.transformer[-1].convffn.conv.bn.eval()
        if setup == "momentum":
            mm.encoder.transformer[0].token_mixer.norm.rbr_skip.momentum = None
        if setup == "frozen":
            for mod in mm.modules():
                if isinstance(mod, torch.nn.SyncBatchNorm):
                    mod.eval()
        try:
            check_trainable(mm, mm.encoder, what)
            msgs.append(None)
        except (NotImplementedError, RuntimeError) as e:
            msgs.append(str(e))
    return msgs


def test_converted_s0_follows_the_batchnorm2d_rules():
    """convert_sync_batchnorm makes S0's BNs SyncBatchNorm, which is not a BatchNorm2d: the opt-in, mixed-state and momentum
    rules still fire, and frozen SyncBatchNorms take the frozen path (only the CPU-module error is left)."""
    plain, mixed, momentum, frozen = _s0_rules()
    assert "enable_batch_stat_bn" in plain
    assert "mixed" in mixed
    assert "momentum=None" in momentum
    assert "CUDA" in frozen or "cuda" in frozen


def _s0_worker(rank, world, port, q):
    import traceback
    try:
        _init(rank, world, port)
        from efficientsam3_b200.backbones.mobile_clip import check_trainable
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_s0_cpu()).enable_batch_stat_bn().train()
        synced = m.encoder.batch_stat_synced()
        try:
            check_trainable(m, m.encoder, "S0")
            msg = ""
        except (NotImplementedError, RuntimeError) as e:
            msg = str(e)
        q.put((rank, [msg, synced]))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


def test_s0_syncbn_over_two_ranks_passes_the_rules():
    """Over two ranks a converted batch-statistics S0 synchronises (the GPU test runs it): the rules pass, and only the CPU-module
    error is left."""
    for _, (msg, synced) in _run(_s0_worker, 2):
        assert synced and "CUDA" in msg and "SyncBatchNorm" not in msg, msg
