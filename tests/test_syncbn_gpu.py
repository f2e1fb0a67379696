"""GPU: synchronised BatchNorm (bn_sync.cu) -- the split statistics / backward kernels against es3_bn_stats / es3_bn_act_bwd on the
concatenated rows, and a 2-rank SyncBatchNorm training step against the single-process global-batch step."""
import os

import pytest
import torch

from test_syncbn_cpu import _free_port, _run  # noqa: F401  (spawn / join / terminate helper)

pytestmark = pytest.mark.gpu


def _parts(M, k, g):
    """k contiguous row partitions of M rows, each non-empty, sizes drawn from g."""
    if k == 1:
        return [M]
    cuts = sorted(torch.randperm(M - 1, generator=g)[:k - 1].add(1).tolist())
    bounds = [0, *cuts, M]
    return [b - a for a, b in zip(bounds, bounds[1:])]


def _z(M, C, g, mean=0.0, std=1.0):
    return (torch.randn(M, C, generator=g) * std + mean).to(torch.bfloat16)


def _stats_split(ops, z, sizes, gamma, beta, rm, rv, nbt):
    parts = torch.stack([ops.bn_stats_partial(s.contiguous()) for s in torch.split(z, sizes)])
    return ops.bn_stats_combine(parts, gamma, beta, 1e-5, 0.1, rm, rv, nbt)


@pytest.mark.parametrize("M,C,mean", [(1000, 64, 0.0), (4096 + 37, 96, 0.0), (2048, 256, 100.0), (3, 8, 0.0), (70000, 32, -100.0)])
def test_stats_partial_combine_equals_bn_stats(cuda, M, C, mean):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(M + C)
    z = _z(M, C, g, mean=mean).to(cuda)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    rm0, rv0 = torch.randn(C, generator=g).to(cuda), torch.rand(C, generator=g).add(0.5).to(cuda)
    ref_rm, ref_rv, ref_nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device=cuda)
    ref = ops.bn_stats(z, gamma, beta, 1e-5, 0.1, ref_rm, ref_rv, ref_nbt)
    zd = z.double()
    exact_mean, exact_var = zd.mean(0), zd.var(0, unbiased=False)
    for k in range(1, 5):
        if k > M:
            continue
        sizes = _parts(M, k, g)
        rm, rv, nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device=cuda)
        got = _stats_split(ops, z, sizes, gamma, beta, rm, rv, nbt)
        for a, b, what in zip(got[:4], ref, ("mean", "invstd", "scale", "shift")):
            torch.testing.assert_close(a, b, rtol=2e-6, atol=2e-6 * max(1.0, abs(mean)), msg=f"{what} k={k}")
        torch.testing.assert_close(got[0].double(), exact_mean, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close((1.0 / got[1].double() ** 2 - 1e-5), exact_var, rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(rm, ref_rm, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(rv, ref_rv, rtol=1e-5, atol=1e-6)
        assert int(nbt) == 1 and float(got[4]) == M
        rm2, rv2, nbt2 = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device=cuda)
        again = _stats_split(ops, z, sizes, gamma, beta, rm2, rv2, nbt2)
        assert all(torch.equal(a, b) for a, b in zip(got, again)) and torch.equal(rm, rm2) and torch.equal(rv, rv2)


@pytest.mark.parametrize("M,C,act", [(1000, 64, "gelu"), (4096 + 37, 96, None), (2048, 256, "relu"), (20000, 32, "hswish")])
def test_bwd_partial_coef_apply_equals_bn_act_bwd(cuda, M, C, act):
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(7 * M + C)
    z = _z(M, C, g, mean=0.5).to(cuda)
    da = _z(M, C, g).to(cuda)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    mean, invstd, scale, shift = ops.bn_stats(z, gamma, beta, 1e-5, 0.1)
    dg_ref, db_ref = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
    dz_ref = ops.bn_act_bwd(da, z, scale, shift, act, "batch", mean, invstd, dg_ref, db_ref)
    total = torch.tensor([float(M)], dtype=torch.float64, device=cuda)
    for k in range(1, 5):
        sizes = _parts(M, k, g)
        dg, db = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
        zs, ds = torch.split(z, sizes), torch.split(da, sizes)
        parts = torch.stack([ops.bn_act_bwd_partial(d.contiguous(), s.contiguous(), scale, shift, act, mean, invstd, dg, db)
                             for s, d in zip(zs, ds)])
        coef = ops.bn_bwd_coef(parts, total, scale, mean, invstd)
        dz = torch.cat([ops.bn_act_bwd_apply(d.contiguous(), s.contiguous(), scale, shift, act, coef) for s, d in zip(zs, ds)])
        rel = ((dz.double() - dz_ref.double()).norm() / dz_ref.double().norm()).item()
        assert rel < 2e-3, (k, rel)                           # bf16 outputs of near-identical fp32 coefficients
        torch.testing.assert_close(dg, dg_ref, rtol=1e-4, atol=1e-3)
        torch.testing.assert_close(db, db_ref, rtol=1e-4, atol=1e-3)
        coef2 = ops.bn_bwd_coef(parts, total, scale, mean, invstd)
        parts2 = torch.stack([ops.bn_act_bwd_partial(d.contiguous(), s.contiguous(), scale, shift, act, mean, invstd)
                              for s, d in zip(zs, ds)])
        assert torch.equal(coef, coef2) and torch.equal(parts, parts2)


def test_host_rejects_bad_shapes(cuda):
    from efficientsam3_b200 import _lib, ops
    z = torch.zeros(16, 12, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(ValueError):
        ops.bn_stats_partial(z)                                # C % 8 != 0
    with pytest.raises(_lib.Es3Error):
        ops.bn_stats_partial(z.float())
    zc = torch.zeros(16, 16, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(ValueError):
        ops.bn_stats_partial(zc[:, :8])                        # not contiguous
    v = torch.ones(16, device=cuda)
    with pytest.raises(ValueError):
        ops.bn_stats_combine(torch.zeros(2, 2, 16, dtype=torch.float64, device=cuda), v, v, 1e-5, 0.1)
    with pytest.raises(_lib.Es3Error):
        ops.bn_stats_combine(torch.zeros(2, 3, 16, dtype=torch.float32, device=cuda), v, v, 1e-5, 0.1)
    with pytest.raises(ValueError):
        ops.bn_stats_combine(torch.zeros(2, 3, 16, dtype=torch.float64, device=cuda), torch.ones(8, device=cuda), v, 1e-5, 0.1)
    with pytest.raises(ValueError):
        ops.bn_act_bwd_partial(zc, zc[:8].contiguous(), v, v, None, v, v)
    with pytest.raises(ValueError):
        ops.bn_bwd_coef(torch.zeros(2, 3, 16, dtype=torch.float64, device=cuda), torch.ones(1, dtype=torch.float64, device=cuda),
                        v, v, v)
    with pytest.raises(ValueError):
        ops.bn_bwd_coef(torch.zeros(2, 2, 16, dtype=torch.float64, device=cuda), torch.ones(2, dtype=torch.float64, device=cuda),
                        v, v, v)


# ------------------------------------------------------------------------------------------ 2-rank training step
def _student(name, img, embed):
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.model import build_image_student_model
    from oracle.weights import fill_state_dict
    m = build_image_student_model(NS(MODEL=NS(BACKBONE=name), DATA=NS(IMG_SIZE=img), DISTILL=NS(EMBED_DIM=1024, EMBED_SIZE=embed)))
    m.load_state_dict(fill_state_dict(m.state_dict(), 3))
    return m


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _mean_grads(m, world):
    """The parameters' gradients averaged over the ranks (one all-reduce of the concatenation), as DDP / FlatAdamW average them."""
    import torch.distributed as dist
    ps = [p for p in m.parameters() if p.grad is not None]
    flat = torch.cat([p.grad.reshape(-1).double() for p in ps])
    dist.all_reduce(flat)
    return flat / world, ps


def _step_worker(rank, world, port, q, backend, name, img, embed, b):
    import traceback
    import torch.distributed as dist
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        dist.init_process_group(backend, rank=rank, world_size=world)      # first: the port is taken before any long set-up
        from efficientsam3_b200 import sync_bn
        from efficientsam3_b200.stage1.optim import FlatAdamW, KDLossFunction
        g = torch.Generator().manual_seed(11)
        n = world * b
        x = torch.randn(n, 3, img, img, generator=g).to(dev)
        t = torch.randn(n, 1024, embed, embed, generator=g).to(dev)
        sz = torch.tensor([[img, img]] * n, dtype=torch.int32, device=dev)
        sl = slice(rank * b, (rank + 1) * b)

        ref = _student(name, img, embed).to(dev).train()      # this process alone, the global batch, plain BatchNorm2d
        ropt = FlatAdamW(ref, lr=1e-3)
        ropt.zero_grad()
        ref_out = ref(x)
        KDLossFunction.apply(ref_out, t, sz, img, 1.0).backward()

        def ranked(convert):
            m = _student(name, img, embed).to(dev)            # the reference's order: .cuda(), convert, then the optimiser
            if convert:
                m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
            m.train()
            opt = FlatAdamW(m, lr=1e-3)
            opt.zero_grad()
            e0 = sync_bn.exchanges
            out = m(x[sl])
            loss = KDLossFunction.apply(out, t[sl], sz[sl], img, 1.0)
            opt.begin_backward(True)
            loss.backward()
            k = opt.all_reduce_grads()
            torch.cuda.synchronize()
            bufs = {kk: v for kk, v in m.state_dict().items() if "running_" in kk or "num_batches" in kk}
            rbufs = {kk: v for kk, v in ref.state_dict().items() if kk in bufs}
            rel_buf = max(_rel(bufs[kk], rbufs[kk]) for kk in bufs if "running_" in kk)
            # a list, not a tensor: a CPU tensor on the queue is passed as a file descriptor that the rank, exiting, may
            # close before the parent has taken it
            flat = torch.cat([v.double().reshape(-1) for v in bufs.values()]).cpu().tolist()
            return (_rel(out.detach(), ref_out.detach()[sl]), _rel(opt.flat_grad / k, ropt.flat_grad), rel_buf,
                    sync_bn.exchanges - e0, flat)

        synced = ranked(True)
        plain = ranked(False)                                 # control: the same two-rank step with per-rank statistics
        q.put((rank, *synced, plain[:3]))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


def _check_step(res, name):
    for rank, rel_out, rel_g, rel_buf, exch, _, plain in res:
        print(f"SyncBN {name} rank {rank}: output rel-L2 {rel_out:.3e}, averaged gradient rel-L2 {rel_g:.3e}, running buffers "
              f"rel-L2 {rel_buf:.3e}, {exch} exchanges; per-rank BatchNorm2d control: {plain[0]:.3e} / {plain[1]:.3e} / {plain[2]:.3e}")
        # the batch-statistics train-test tolerances: a different reduction order moves bf16 roundings, which this random-weight
        # fixture's batch statistics amplify (tests/test_zz_train_gpu.py); the running buffers follow the batch means
        assert rel_out < 0.15 and rel_g < 0.6, (rel_out, rel_g)
        assert rel_buf < 0.15, rel_buf
        assert exch > 0
        # ... and the synchronisation is what brings them there: per-rank statistics are clearly further from the global batch
        assert plain[0] > 2 * rel_out and plain[2] > 2 * rel_buf, (plain, rel_out, rel_buf)
    assert res[0][5] == res[1][5]                                 # running buffers bit-identical across ranks


def test_two_ranks_one_gpu_gloo_evm_step_matches_the_global_batch(cuda):
    _check_step(_run(_step_worker, 2, "gloo", "efficientvit_b1", 256, 16, 2, timeout=900), "EV-M gloo")


def test_two_ranks_nccl_evm_step_matches_the_global_batch(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one GPU per rank; fewer than 2 GPUs are visible")
    _check_step(_run(_step_worker, 2, "nccl", "efficientvit_b1", 256, 16, 2, timeout=900), "EV-M nccl")


# ------------------------------------------------------------------------------------------ MobileCLIP-S0, ctx 16
def _s0_worker(rank, world, port, q, backend):
    import traceback
    import torch.distributed as dist
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        dist.init_process_group(backend, rank=rank, world_size=world)
        from efficientsam3_b200 import sync_bn
        from efficientsam3_b200.stage1.losses import TextKDLossFunction
        from test_text_gpu import captions
        from test_text_train_gpu import _student as text_student
        caps = captions()
        b = len(caps) // world
        teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(3)).to(dev)
        sl = slice(rank * b, (rank + 1) * b)

        def step(convert, text, tch):
            m, _ = text_student("MobileCLIP-S0", dev, layers=1, ctx=16, seed=29)
            if convert:
                m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
            m.enable_batch_stat_bn().train()
            e0 = sync_bn.exchanges
            _, mem, _ = m(text)
            mem = mem.transpose(0, 1)
            loss, _, _, _ = TextKDLossFunction.apply(mem, tch, None, 1.0, 0.0)    # unmasked: the global loss is the ranks' mean
            loss.backward()
            torch.cuda.synchronize()
            return m, mem.detach(), sync_bn.exchanges - e0

        ref, ref_mem, _ = step(False, caps[:world * b], teacher[:world * b])     # one process, the global batch, BatchNorm2d
        ref_g = torch.cat([p.grad.reshape(-1).double() for p in ref.parameters() if p.grad is not None])

        def ranked(convert):
            m, mem, exch = step(convert, caps[sl], teacher[sl])
            mean_g, _ = _mean_grads(m, world)
            bufs = {k: v for k, v in m.state_dict().items() if "running_" in k or "num_batches" in k}
            rbufs = {k: v for k, v in ref.state_dict().items() if k in bufs}
            rel_buf = max(_rel(bufs[k], rbufs[k]) for k in bufs if "running_" in k)
            nbt = all(torch.equal(bufs[k], rbufs[k]) for k in bufs if "num_batches" in k)
            # a list, not a tensor: a CPU tensor on the queue is passed as a file descriptor that the rank, exiting, may
            # close before the parent has taken it
            flat = torch.cat([v.double().reshape(-1) for v in bufs.values()]).cpu().tolist()
            return _rel(mem, ref_mem[sl]), _rel(mean_g, ref_g), rel_buf, exch, flat, nbt

        synced = ranked(True)
        plain = ranked(False)
        q.put((rank, *synced[:5], plain[:3], synced[5]))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


def test_two_ranks_one_gpu_gloo_s0_step_matches_the_global_batch(cuda):
    """MobileCLIP-S0 (depth 1, ctx 16) with batch-statistics BatchNorm converted to SyncBatchNorm: two ranks of 3 captions on one
    GPU over gloo vs one process on the 6 captions with plain BatchNorm2d.  Two exchanges per BN group in the forward and two in
    the backward, per RepMixerBlock."""
    res = _run(_s0_worker, 2, "gloo", timeout=900)
    for rank, rel_out, rel_g, rel_buf, exch, _, plain, nbt in res:
        print(f"SyncBN S0 rank {rank}: memory rel-L2 {rel_out:.3e}, averaged gradient rel-L2 {rel_g:.3e}, running buffers rel-L2 "
              f"{rel_buf:.3e}, {exch} exchanges; per-rank BatchNorm2d control: {plain[0]:.3e} / {plain[1]:.3e} / {plain[2]:.3e}")
        assert rel_out < 2e-2 and rel_g < 5e-2 and rel_buf < 1e-3, (rel_out, rel_g, rel_buf)   # the S0 train-test tolerances
        assert exch == 8 and nbt                                  # 2 RepMixerBlocks x (2 forward + 2 backward)
        assert plain[0] > 2 * rel_out and plain[2] > 2 * rel_buf, (plain, rel_out, rel_buf)
    assert res[0][5] == res[1][5]
