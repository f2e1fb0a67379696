"""GPU: MobileCLIP-S0's synchronised-BatchNorm entry points (csrc/repmixer_bn_train.cu: es3_repmixer_bn_stats_partial,
_finalize_sync, _ffn_sums, _ffn_apply, _tm_sums, _tm_apply) with W ranks emulated in one process, composed in the order
mobile_clip.repmixer_bn_forward and RepMixerBatchStatUnit.backward call them (the all-gather is a torch.stack in rank order):
against fp64 autograd / F.batch_norm on the global batch, against the per-rank kernels on the concatenated batch, bit-identical
across the virtual ranks and across repeats.  The cases hold uneven and single-token ranks and ranks whose means lie tens of
standard deviations apart, and the four BatchNorms get distinct eps and momentum, so a swapped scalar or statistic shows.  Also:
the host rejections of the sync entry points, mean-shifted row partitions for the image kernels (bn_sync.cu), and a 2-rank gloo
S0 step with ranks of 1 and 5 captions."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import max_err_over_scale
from oracle import text as OT
from oracle.weights import fill_state_dict
from test_syncbn_cpu import _run  # spawn / join / terminate helper
from test_syncbn_gpu import _parts, _rel, _stats_split, _z
from test_text_train_s0_bn_gpu import BN, _stats64
from test_text_train_s0_gpu import _acc, _leaves, _rows, _t

pytestmark = pytest.mark.gpu

# BN_ms, BN_mc, BN_ns, BN_f (repmixer_bns order).  All distinct: BN_ms and BN_ns normalise the same x and differ only in eps.
EPS = (1e-5, 1e-3, 3e-2, 2e-4)
MOM = (0.1, 0.3, 0.05, 0.9)
BN_LEAF = [f"{n}.{w}" for n in BN[:3] for w in ("weight", "bias")]
GRADS = ("dwf", "dgf", "dbf", "dwm", "dls_tm", *BN_LEAF)
RUNNING = [f"{s}{i}" for i in range(4) for s in ("rm", "rv", "nbt")]


# ------------------------------------------------------------------------------------------------ set-up and fp64 statement
def _setup(B, L, C, sizes, shifts, dev):
    """A train-mode RepMixerBlock with the EPS / MOM BatchNorms and its inputs.  x has per-channel standard deviations from 0.03
    to 3 (variances on both sides of the largest eps, so invstd depends on which eps is used), and the rows of rank r are offset
    by shifts[r] standard deviations."""
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock, repmixer_bn_pack, repmixer_bns
    blk = RepMixerBlock(dim=C)
    sd0 = fill_state_dict(blk.state_dict(), 13 * L + C + B)
    blk.load_state_dict(sd0)
    blk = blk.to(dev).train()
    bns = repmixer_bns(blk)
    for bn, eps, mom in zip(bns, EPS, MOM):
        bn.eps, bn.momentum = eps, mom
    sd = {k: v.to(dev, torch.float64) for k, v in sd0.items() if not k.endswith("num_batches_tracked")}
    run0 = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in bns]
    gen = torch.Generator().manual_seed(B * 1000 + L * 10 + C + len(sizes))
    std = torch.logspace(-1.5, 0.5, C)[torch.randperm(C, generator=gen)]
    shift = torch.cat([torch.full((n * L, 1), float(s)) for n, s in zip(sizes, shifts)])
    x = ((torch.randn(B * L, C, generator=gen) + shift) * std).to(dev)
    g, du, et = (torch.randn(B * L, C, generator=gen).to(dev) for _ in range(3))
    return repmixer_bn_pack(blk), bns, sd, run0, x, g, du, et


def _bt(t, sd, i):
    """BatchNorm i (BN order) in train mode without running buffers, with its own eps (fp64 reference)."""
    return F.batch_norm(t, None, None, sd[BN[i] + ".weight"], sd[BN[i] + ".bias"], True, 0.0, EPS[i])


def _reference(x, x1, g, du, et, B, L, sd, run0):
    """The block on the global batch in fp64 (test_repmixer_bn_kernels' statement, each BN with its own eps and momentum).  f's
    statistics are those of dw(x1) on the x1 given (the kernels' own); the token mixer's incoming gradient is et."""
    tm, f = "token_mixer", "convffn"
    ref = {}
    t = _t(x, B, L).detach()
    c = OT._dw(t, sd[tm + ".mixer.rbr_conv.0.conv.weight"])
    t1 = _t(x1, B, L).detach()
    fv = OT._dw(t1, sd[f + ".conv.conv.weight"])
    vals = (t, c, t, fv)
    ref["mean"], ref["var"] = zip(*[_stats64(v) for v in vals])
    for i, v in enumerate(vals):
        rm, rv = run0[i][0].double().clone(), run0[i][1].double().clone()
        F.batch_norm(v, rm, rv, None, None, True, MOM[i], EPS[i])
        ref[f"rm{i}"], ref[f"rv{i}"] = rm, rv
    ls = sd[tm + ".layer_scale"]
    ref["x1"] = _rows(t + ls * (_bt(t, sd, 0) + _bt(c, sd, 1) - _bt(t, sd, 2)))
    ref["u"] = _rows(_bt(fv, sd, 3))
    # the fold (wm, bm, wf, bf), restated from the fp64 statistics
    s = [sd[BN[i] + ".weight"] / (ref["var"][i] + EPS[i]).sqrt() for i in range(4)]
    b = [sd[BN[i] + ".bias"] - ref["mean"][i] * s[i] for i in range(4)]
    ls = ls.reshape(-1)
    wm = sd[tm + ".mixer.rbr_conv.0.conv.weight"].reshape(-1, 11).t() * (ls * s[1])
    wm[5] += 1.0 + ls * (s[0] - s[2])
    wf = sd[f + ".conv.conv.weight"].reshape(-1, 11).t() * s[3]
    ref["fold"] = torch.cat([wm, (ls * (b[0] + b[1] - b[2]))[None], wf, b[3][None]])
    # ConvFFN.conv + BN_f: e = d/dx1 of (sum du * BN_f(dw(x1)) + sum g * x1)
    lv = _leaves(sd, [f + ".conv.conv.weight", BN[3] + ".weight", BN[3] + ".bias"])
    t1 = t1.clone().requires_grad_(True)
    uu = _bt(OT._dw(t1, lv[f + ".conv.conv.weight"]), {**sd, **lv}, 3)
    ((uu * _t(du, B, L).detach()).sum() + (t1 * _t(g, B, L).detach()).sum()).backward()
    ref["e"], ref["dwf"] = _rows(t1.grad), lv[f + ".conv.conv.weight"].grad
    ref["dgf"], ref["dbf"] = lv[BN[3] + ".weight"].grad, lv[BN[3] + ".bias"].grad
    # token mixer: dx = d/dx of sum et * (x + ls_tm (BN_ms(x) + BN_mc(dw(x)) - BN_ns(x)))
    lv = _leaves(sd, [tm + ".mixer.rbr_conv.0.conv.weight", tm + ".layer_scale", *BN_LEAF])
    s_ = {**sd, **lv}
    tx = _t(x, B, L)
    out = tx + s_[tm + ".layer_scale"] * (_bt(tx, s_, 0) + _bt(OT._dw(tx, s_[tm + ".mixer.rbr_conv.0.conv.weight"]), s_, 1)
                                          - _bt(tx, s_, 2))
    (out * _t(et, B, L).detach()).sum().backward()
    ref["dx"], ref["dwm"], ref["dls_tm"] = _rows(tx.grad), lv[tm + ".mixer.rbr_conv.0.conv.weight"].grad, lv[tm + ".layer_scale"].grad
    ref.update((n, lv[n].grad) for n in BN_LEAF)
    return ref


# ------------------------------------------------------------------------------------------------ the two paths
def _grad_dsts(C, dev):
    """Gradient destinations pre-filled with 0.25 (the kernels add into them)."""
    return {"dwf": _acc((C, 1, 1, 11), dev), "dgf": _acc((C,), dev), "dbf": _acc((C,), dev), "dwm": _acc((C, 1, 1, 11), dev),
            "dls_tm": _acc((C, 1, 1), dev), **{n: _acc((C,), dev) for n in BN_LEAF}}


def _sync_run(ops, p, run0, x, g, du, et, sizes, L):
    """The synchronised block on W = len(sizes) virtual ranks holding contiguous groups of sizes[r] sequences, each with its own
    copies of the running buffers: one dict of outputs per rank.  The calls and their order are repmixer_bn_forward's and the
    sync branch of RepMixerBatchStatUnit.backward's; the token-mixer half takes et, not the e the ConvFFN half returns, so each
    half has its own fp64 statement (as in test_repmixer_bn_kernels)."""
    C, dev, taps, aff = x.shape[1], x.device, p["taps"], p["aff"]
    rows = [n * L for n in sizes]
    xs, gs, dus, ets = (torch.split(t, rows) for t in (x, g, du, et))
    rk = [{"bns": [NS(running_mean=rm.clone(), running_var=rv.clone(), num_batches_tracked=nbt.clone(), eps=eps, momentum=mom)
                   for (rm, rv, nbt), eps, mom in zip(run0, EPS, MOM)],
           "fold": torch.empty(24, C, device=dev), "stats": torch.empty(8, C, device=dev), **_grad_dsts(C, dev)} for _ in sizes]
    ranks = list(zip(rk, sizes, xs, gs, dus, ets))
    # forward: statistics of x and c -> finalize on every rank -> statistics of f -> finalize -> x1, u on the fold
    parts = torch.stack([ops.repmixer_bn_stats_partial(xr, n, L, taps, o["fold"], 0) for o, n, xr, *_ in ranks])
    for o, *_ in ranks:
        o["total"] = ops.repmixer_bn_finalize_sync(parts, 0, taps, aff, o["bns"], o["fold"], o["stats"])
    parts = torch.stack([ops.repmixer_bn_stats_partial(xr, n, L, taps, o["fold"], 1) for o, n, xr, *_ in ranks])
    for o, *_ in ranks:
        ops.repmixer_bn_finalize_sync(parts, 1, taps, aff, o["bns"], o["fold"], o["stats"])
    for o, n, xr, *_ in ranks:
        fo = o["fold"]
        o["x1"], o["u"] = ops.repmixer(xr, n, L, fo[:11], fo[11], fo[12:23], fo[23])
    # backward: ConvFFN sums -> gather -> apply (e); token-mixer sums -> gather -> apply (dx and its bf16 copy)
    parts = torch.stack([ops.repmixer_bn_ffn_sums(o["x1"], dur, taps, o["stats"], n, L, aff, dgamma=o["dgf"], dbeta=o["dbf"])
                         for o, n, xr, gr, dur, _ in ranks])
    for o, n, xr, gr, dur, _ in ranks:
        o["e"] = ops.repmixer_bn_ffn_apply(o["x1"], dur, gr, taps, aff, o["stats"], parts, o["total"], n, L, dtaps=o["dwf"])
    parts = torch.stack([ops.repmixer_bn_tm_sums(xr, er, taps, aff, o["stats"], n, L, dbn=[o[k] for k in BN_LEAF])
                         for o, n, xr, gr, dur, er in ranks])
    for o, n, xr, gr, dur, er in ranks:
        o["dx"], o["dxb"] = ops.repmixer_bn_tm_apply(xr, er, taps, aff, o["stats"], parts, o["total"], n, L, dtaps=o["dwm"],
                                                     dls=o["dls_tm"], want_bf16=True)
    for o in rk:
        for i, bn in enumerate(o.pop("bns")):
            o[f"rm{i}"], o[f"rv{i}"], o[f"nbt{i}"] = bn.running_mean, bn.running_var, bn.num_batches_tracked
    return rk


def _global(rk):
    """The ranks' outputs as one batch: rows concatenated in rank order, gradients summed over the ranks less their fills."""
    o = {k: rk[0][k] for k in ("fold", "stats", *RUNNING)}
    o.update((k, torch.cat([r[k] for r in rk])) for k in ("x1", "u", "e", "dx", "dxb"))
    o.update((k, sum(r[k].double() - 0.25 for r in rk)) for k in GRADS)
    return o


def _per_rank_fwd(ops, p, bns, run0, x, B, L):
    for bn, (rm, rv, nbt) in zip(bns, run0):
        bn.running_mean.copy_(rm); bn.running_var.copy_(rv); bn.num_batches_tracked.copy_(nbt)
    o = dict(zip(("x1", "u", "fold", "stats"), ops.repmixer_bn_fwd(x, B, L, p["taps"], p["aff"], bns)))
    for i, bn in enumerate(bns):
        o[f"rm{i}"], o[f"rv{i}"], o[f"nbt{i}"] = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    return o


def _per_rank_bwd(ops, p, x, x1, stats, g, du, et, B, L):
    o = _grad_dsts(x.shape[1], x.device)
    o["e"] = ops.repmixer_bn_ffn_bwd(x1, du, g, p["taps"], p["aff"], stats, B, L, dtaps=o["dwf"], dgamma=o["dgf"], dbeta=o["dbf"])
    o["dx"], o["dxb"] = ops.repmixer_bn_tm_bwd(x, et, p["taps"], p["aff"], stats, B, L, dtaps=o["dwm"], dls=o["dls_tm"],
                                               dbn=[o[k] for k in BN_LEAF], want_bf16=True)
    return o


# ------------------------------------------------------------------------------------------------ checks
def _chk(log, cls, what, err, tol):
    log.append((cls, what, err, tol))
    assert err <= tol, (cls, what, err, tol)


def _close(log, what, a, b, rtol, atol):
    """|a - b| <= atol + rtol |b| elementwise, logged as the worst ratio to that bound."""
    a, b = a.double(), b.double()
    _chk(log, "per-rank kernels", what, ((a - b).abs() / (atol + rtol * b.abs())).max().item(), 1.0)


def _ulps(a, b):
    """Largest distance between same-signed fp32 tensors in units in the last place."""
    return (a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs().max().item()


def _check_fp64(log, got, ref, run0, tap_tol):
    """got (as _global returns it, or one per-rank run with its fills removed) against _reference."""
    cls = "fp64"
    st = got["stats"].double()
    for i in range(4):
        mean, var = ref["mean"][i], ref["var"][i]
        _chk(log, cls, f"{BN[i]} mean", ((st[2 * i] - mean).abs() / var.sqrt()).max().item(), 1e-4)
        _chk(log, cls, f"{BN[i]} invstd", (st[2 * i + 1] * (var + EPS[i]).sqrt() - 1).abs().max().item(), 1e-4)
        for k in ("rm", "rv"):
            _chk(log, cls, f"{BN[i]} {k}", max_err_over_scale(got[f"{k}{i}"].cpu(), ref[f"{k}{i}"].cpu()), 1e-5)
        assert int(got[f"nbt{i}"]) == int(run0[i][2]) + 1, BN[i]
    for what, sl in (("wm", slice(0, 11)), ("bm", slice(11, 12)), ("wf", slice(12, 23)), ("bf", slice(23, 24))):
        _chk(log, cls, what, max_err_over_scale(got["fold"][sl].cpu(), ref["fold"][sl].cpu()), 1e-4)
    for k, tol in (("x1", 1e-5), ("u", 1e-2), ("e", 2e-3), ("dx", 2e-3)):
        _chk(log, cls, k, max_err_over_scale(got[k].cpu(), ref[k].cpu()), tol)
    assert torch.equal(got["dxb"], got["dx"].to(torch.bfloat16))
    for k in GRADS:
        _chk(log, cls, k, max_err_over_scale(got[k].cpu(), ref[k].cpu()), tap_tol if k in ("dwf", "dwm") else 2e-3)


def _tap_tol(shifts):
    # the tap gradients sum d x with sum d = 0 under batch statistics: with every token offset by 100 std that sum cancels by
    # ~100, and fp32 keeps about two fewer digits of it (test_repmixer_bn_kernels' tolerance for the same case)
    return 2e-1 if min(abs(s) for s in shifts) >= 100 else 2e-3


def _report(label, log):
    for cls in dict.fromkeys(c for c, *_ in log):
        ratio, what, err, tol = max((e / t, w, e, t) for c, w, e, t in log if c == cls)
        print(f"  {label} {cls}: worst {what} {err:.3e} (threshold {tol:.0e}, {ratio:.2f} of it)")


CASES = [  # B, L, C, sequences per rank, rank offsets in standard deviations
    (6, 16, 512, (3, 3), (0, 0)),            # the gloo S0 test's shape, at kernel level
    (6, 16, 512, (6,), (0,)),                # W = 1 against the per-rank kernels
    (5, 77, 512, (1, 4), (0, 0)),            # uneven; the table-77 length
    (2, 1, 32, (1, 1), (0, 0)),              # every rank B*L = 1: group count 2, M / (M - 1) = 2
    (3, 1, 32, (1, 1, 1), (0, 0, 0)),        # three single-token ranks
    (4, 128, 64, (1, 1, 2), (0, 0, 0)),      # the longest sequence; C neither 32 nor 512
    (64, 32, 512, (16,) * 4, (0,) * 4),      # many sequences per rank
    (64, 32, 512, (1, 63), (0, 0)),          # extreme imbalance
    (7, 11, 32, (2, 5), (50, -50)),          # Chan's between-rank term dominates M2
    (3, 16, 32, (1, 2), (100, 100)),         # |mean| >> std
]


@pytest.mark.parametrize("B,L,C,sizes,shifts", CASES, ids=[f"B{c[0]}L{c[1]}C{c[2]}-{'+'.join(map(str, c[3]))}"
                                                            + (f"-shift{'/'.join(map(str, sorted(set(c[4]))))}" if any(c[4]) else "")
                                                            for c in CASES])
def test_repmixer_bn_sync_entry_points(cuda, B, L, C, sizes, shifts):
    from efficientsam3_b200 import ops
    assert sum(sizes) == B
    W = len(sizes)
    p, bns, sd, run0, x, g, du, et = _setup(B, L, C, sizes, shifts, cuda)
    rk = _sync_run(ops, p, run0, x, g, du, et, sizes, L)
    log = []
    # every virtual rank holds the same statistics, fold, running buffers and count; each BN counted once per forward
    for r in rk[1:]:
        for k in ("fold", "stats", "total", *RUNNING):
            assert torch.equal(r[k], rk[0][k]), k
    assert rk[0]["total"].dtype == torch.float64 and float(rk[0]["total"]) == B * L
    for r in rk:
        for i in range(4):
            assert int(r[f"nbt{i}"]) == int(run0[i][2]) + 1, BN[i]
    # the global batch in fp64
    got = _global(rk)
    _check_fp64(log, got, _reference(x, got["x1"], g, du, et, B, L, sd, run0), run0, _tap_tol(shifts))
    # the per-rank kernels on the concatenated batch (per-sequence partials are the same; only fp64 / fp32 sum orders differ)
    pr = _per_rank_fwd(ops, p, bns, run0, x, B, L)
    big = max(1.0, *(abs(s) for s in shifts))
    for k in ("stats", "fold", *(k for k in RUNNING if not k.startswith("nbt"))):
        _close(log, k, got[k], pr[k], 2e-6, 2e-6 * big)
    for i in range(4):
        assert torch.equal(got[f"nbt{i}"], pr[f"nbt{i}"])
    _chk(log, "per-rank kernels", "x1", max_err_over_scale(got["x1"].cpu(), pr["x1"].cpu()), 1e-6)
    prb = _per_rank_bwd(ops, p, x, pr["x1"], pr["stats"], g, du, et, B, L)
    for k in ("e", "dx"):
        _chk(log, "per-rank kernels", k, max_err_over_scale(got[k].cpu(), prb[k].cpu()), 1e-5)
    if W == 1:
        # backward on the same x1 and stats: the same sums and apply kernels on the same partials in the same order (the rank
        # sum over one part adds it to 0.f).  The count's reciprocal is (float)(1.0 / total) synchronised and 1.f / (float)(B L)
        # per rank; they can differ by double rounding, but not at this B L.
        assert np.float32(1.0 / np.float64(B * L)) == np.float32(1.0) / np.float32(B * L)
        same = _per_rank_bwd(ops, p, x, rk[0]["x1"], rk[0]["stats"], g, du, et, B, L)
        for k in same:
            assert torch.equal(rk[0][k], same[k]), k
        # forward: M2 goes through (var M) / M in fp64, so the statistics agree to one fp32 ulp, not bitwise
        _chk(log, "W = 1 (ulps)", "stats", _ulps(rk[0]["stats"], pr["stats"]), 1)
    again = _sync_run(ops, p, run0, x, g, du, et, sizes, L)   # fixed-order reductions: bit-identical
    for r, a in zip(rk, again):
        for k in r:
            assert torch.equal(r[k], a[k]), k
    _report(f"B={B} L={L} C={C} ranks {sizes} shifts {shifts}", log)


@pytest.mark.parametrize("B,L,C,shift", [(6, 16, 512, 0), (64, 32, 512, 0), (3, 16, 32, 100)])
def test_repmixer_bn_per_rank_kernels_with_distinct_bn_scalars(cuda, B, L, C, shift):
    """es3_repmixer_bn_fwd / _ffn_bwd / _tm_bwd with four different eps and momenta against fp64: a swapped scalar, or BN_ms's
    invstd used for BN_ns, shows (every other test builds the BatchNorms with the defaults)."""
    from efficientsam3_b200 import ops
    p, bns, sd, run0, x, g, du, et = _setup(B, L, C, (B,), (shift,), cuda)
    got = _per_rank_fwd(ops, p, bns, run0, x, B, L)
    got.update(_per_rank_bwd(ops, p, x, got["x1"], got["stats"], g, du, et, B, L))
    got.update((k, got[k].double() - 0.25) for k in GRADS)
    log = []
    _check_fp64(log, got, _reference(x, got["x1"], g, du, et, B, L, sd, run0), run0, _tap_tol((shift,)))
    _report(f"per-rank B={B} L={L} C={C} shift {shift}", log)


# ------------------------------------------------------------------------------------------------ host rejection
def test_repmixer_bn_sync_entry_points_reject_bad_input_and_write_nothing(cuda):
    from efficientsam3_b200 import _lib, ops
    from efficientsam3_b200.backbones.mobile_clip import RepMixerBlock, repmixer_bns
    B, L, C, W = 2, 4, 32, 2
    gen = torch.Generator().manual_seed(5)

    def block(C):
        bns = repmixer_bns(RepMixerBlock(dim=C).to(cuda).train())
        taps, aff, fold, stats = (torch.randn(*s, generator=gen).to(cuda) for s in ((2, 11, C), (9, C), (24, C), (8, C)))
        return bns, taps, aff, fold, stats

    bns, taps, aff, fold, stats = block(C)
    x = torch.randn(B * L, C, generator=gen).to(cuda)
    dsts = _grad_dsts(C, cuda)
    dbn = [dsts[k] for k in BN_LEAF]
    total = torch.tensor([float(W * B * L)], dtype=torch.float64, device=cuda)
    f64, f32 = dict(dtype=torch.float64, device=cuda), dict(dtype=torch.float32, device=cuda)
    p2, p3 = torch.zeros(W, 2, C, **f32), torch.zeros(W, 3, C, **f32)

    def watched(bns, *ts):
        return [t for bn in bns for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)] + list(ts)

    def rejects(fn, host=True, watch=None):
        """fn raises ValueError (ops) or Es3Error (the C ABI) and changes nothing; with host, before any launch."""
        watch = watch or watched(bns, fold, stats, *dsts.values())
        before = [t.clone() for t in watch]
        n0 = ops.launch_count
        with pytest.raises((ValueError, _lib.Es3Error)):
            fn()
        torch.cuda.synchronize()
        if host:
            assert ops.launch_count == n0
        for a, b in zip(watch, before):
            assert torch.equal(a, b)

    def fin(parts, mode=0):
        return lambda: ops.repmixer_bn_finalize_sync(parts, mode, taps, aff, bns, fold, stats)

    def ffn_apply(parts=p2, tot=total, rows=x, L=L):
        return lambda: ops.repmixer_bn_ffn_apply(rows, rows, rows, taps, aff, stats, parts, tot, B, L, dtaps=dsts["dwf"])

    def tm_apply(parts=p3, tot=total, rows=x, L=L):
        return lambda: ops.repmixer_bn_tm_apply(rows, rows, taps, aff, stats, parts, tot, B, L, dtaps=dsts["dwm"], dls=dsts["dls_tm"])

    # parts of the wrong dtype, the wrong shape (mode 0 with mode 1's, another C, another Q), not contiguous
    rejects(fin(torch.zeros(W, 2, 3, C, **f32)))
    rejects(ffn_apply(parts=torch.zeros(W, 2, C, **f64)))
    rejects(tm_apply(parts=torch.zeros(W, 3, C, **f64)))
    rejects(fin(torch.zeros(W, 1, 3, C, **f64)))
    rejects(fin(torch.zeros(W, 2, 3, C, **f64), mode=1))
    rejects(fin(torch.zeros(W, 2, 3, C + 32, **f64)))
    rejects(ffn_apply(parts=torch.zeros(W, 2, C + 32, **f32)))
    rejects(ffn_apply(parts=p3))
    rejects(tm_apply(parts=torch.zeros(W, 3, C + 32, **f32)))
    rejects(tm_apply(parts=p2))
    rejects(fin(torch.zeros(W, 2, 3, 2 * C, **f64)[..., :C]))
    rejects(ffn_apply(parts=torch.zeros(W, 2, 2 * C, **f32)[..., :C]))
    rejects(tm_apply(parts=torch.zeros(W, 3, 2 * C, **f32)[..., :C]))
    # the group's count: fp32, or two elements
    for tot in (total.float(), torch.tensor([1.0, 7.0], **f64)):
        rejects(ffn_apply(tot=tot))
        rejects(tm_apply(tot=tot))
    # mode 2: the C ABI rejects it before launching anything
    rejects(lambda: ops.repmixer_bn_stats_partial(x, B, L, taps, fold, 2), host=False)
    rejects(fin(torch.zeros(W, 1, 3, C, **f64), mode=2), host=False)
    # L = 129 (a sequence is kept in shared memory), C = 48 (not a multiple of 32)
    for rows, L_, what in ((torch.zeros(B * 129, C, device=cuda), 129, "1..128"), (torch.zeros(B * L, 48, device=cuda), L, "multiple")):
        rejects(lambda: ops.repmixer_bn_stats_partial(rows, B, L_, taps, fold, 0))
        rejects(lambda: ops.repmixer_bn_ffn_sums(rows, rows, taps, stats, B, L_, aff, dgamma=dsts["dgf"], dbeta=dsts["dbf"]))
        rejects(ffn_apply(rows=rows, L=L_))
        rejects(lambda: ops.repmixer_bn_tm_sums(rows, rows, taps, aff, stats, B, L_, dbn=dbn))
        rejects(tm_apply(rows=rows, L=L_))
        with pytest.raises(ValueError, match=what):
            ops.repmixer_bn_stats_partial(rows, B, L_, taps, fold, 0)
    bns48, taps48, aff48, fold48, stats48 = block(48)
    rejects(lambda: ops.repmixer_bn_finalize_sync(torch.zeros(W, 2, 3, 48, **f64), 0, taps48, aff48, bns48, fold48, stats48),
            host=False, watch=watched(bns48, fold48, stats48))


# ------------------------------------------------------------------------------------------------ image kernels (bn_sync.cu)
@pytest.mark.parametrize("M,C", [(1000, 64), (4096 + 37, 96), (70000, 32)])
def test_stats_partial_combine_mean_shifted_partitions(cuda, M, C):
    """k = 2..4 row partitions whose rows are drawn around (-1)^i 50 std, one of them a single row: Chan's between-partition term
    carries nearly all of M2 (test_stats_partial_combine_equals_bn_stats draws every partition from one distribution)."""
    from efficientsam3_b200 import ops
    g = torch.Generator().manual_seed(3 * M + C)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    rm0, rv0 = torch.randn(C, generator=g).to(cuda), torch.rand(C, generator=g).add(0.5).to(cuda)
    for k in range(2, 5):
        for single in (0, k - 1):
            sizes = _parts(M - 1, k - 1, g)
            sizes.insert(single, 1)
            z = torch.cat([_z(n, C, g, mean=(-1) ** i * 50.0) for i, n in enumerate(sizes)]).to(cuda)
            ref_rm, ref_rv, ref_nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device=cuda)
            ref = ops.bn_stats(z, gamma, beta, 1e-5, 0.1, ref_rm, ref_rv, ref_nbt)
            zd = z.double()
            exact_mean, exact_var = zd.mean(0), zd.var(0, unbiased=False)
            rm, rv, nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device=cuda)
            got = _stats_split(ops, z, sizes, gamma, beta, rm, rv, nbt)
            torch.testing.assert_close(got[0].double(), exact_mean, rtol=1e-6, atol=1e-6)
            # 1e-4 in test_stats_partial_combine_equals_bn_stats; the split path keeps 1.1e-7 here (measured, H100)
            torch.testing.assert_close((1.0 / got[1].double() ** 2 - 1e-5), exact_var, rtol=1e-6, atol=1e-6)
            assert int(nbt) == 1 and float(got[4]) == M
            # es3_bn_stats pivots on row 0.  With two partitions and the single row first, that row lies 100 std from every
            # other row and its fp32 sums of (z - z[0])^2 keep the variance to 5e-5 .. 9e-5 relative (measured on an H100 at
            # M = 1000 / 4133 / 70000; the split path, which pivots in each partition: 1e-7), which moves shift by up to 3e-3.
            # There the split path is held to fp64 alone.
            if k == 2 and single == 0:
                continue
            for a, b, what in zip(got[:4], ref, ("mean", "invstd", "scale", "shift")):
                torch.testing.assert_close(a, b, rtol=2e-6, atol=2e-6 * 50.0, msg=f"{what} sizes={sizes}")
            torch.testing.assert_close(rm, ref_rm, rtol=1e-6, atol=1e-6)
            torch.testing.assert_close(rv, ref_rv, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ uneven ranks, gloo
def _s0_uneven_worker(rank, world, port, q, counts):
    import traceback
    import torch.distributed as dist
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from efficientsam3_b200 import sync_bn
        from efficientsam3_b200.stage1.losses import TextKDLossFunction
        from test_text_gpu import captions
        from test_text_train_gpu import _student as text_student
        caps = captions()
        B = sum(counts)
        assert len(caps) == B
        teacher = torch.randn(B, 16, 256, generator=torch.Generator().manual_seed(3)).to(dev)
        lo = sum(counts[:rank])
        sl = slice(lo, lo + counts[rank])

        def step(convert, text, tch, weight):
            m, _ = text_student("MobileCLIP-S0", dev, layers=1, ctx=16, seed=29)
            if convert:
                m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
            m.enable_batch_stat_bn().train()
            e0 = sync_bn.exchanges
            _, mem, _ = m(text)
            mem = mem.transpose(0, 1)
            loss, _, _, _ = TextKDLossFunction.apply(mem, tch, None, 1.0, 0.0)    # unmasked: a mean over this batch's tokens
            (loss * weight).backward()
            torch.cuda.synchronize()
            return m, mem.detach(), sync_bn.exchanges - e0

        ref, ref_mem, _ = step(False, caps, teacher, 1.0)     # one process, the global batch, BatchNorm2d
        ref_g = torch.cat([p.grad.reshape(-1).double() for p in ref.parameters() if p.grad is not None])
        # The global loss is sum_r (B_r / B) loss_r.  The synchronised backward exchanges every rank's BN sums, so each rank's
        # gradient holds terms of the other ranks' losses: the weight goes on the loss, before the backward, and the ranks'
        # gradients are then summed (weighting them after the backward would give the other ranks' terms this rank's weight).
        m, mem, exch = step(True, caps[sl], teacher[sl], counts[rank] / B)
        flat_g = torch.cat([p.grad.reshape(-1).double() for p in m.parameters() if p.grad is not None])
        dist.all_reduce(flat_g)
        bufs = {k: v for k, v in m.state_dict().items() if "running_" in k or "num_batches" in k}
        rbufs = {k: v for k, v in ref.state_dict().items() if k in bufs}
        rel_buf = max(_rel(bufs[k], rbufs[k]) for k in bufs if "running_" in k)
        nbt = all(torch.equal(bufs[k], rbufs[k]) for k in bufs if "num_batches" in k)
        # a list, not a tensor: a CPU tensor on the queue is passed as a file descriptor that the rank, exiting, may
        # close before the parent has taken it
        flat = torch.cat([v.double().reshape(-1) for v in bufs.values()]).cpu().tolist()
        q.put((rank, _rel(mem, ref_mem[sl]), _rel(flat_g, ref_g), rel_buf, exch, flat, nbt))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, traceback.format_exc()))


def test_uneven_ranks_one_gpu_gloo_s0_step_matches_the_global_batch(cuda):
    """MobileCLIP-S0 (depth 1, ctx 16) with SyncBatchNorm on two ranks of 1 and 5 captions vs one process on the 6 captions with
    plain BatchNorm2d: with uneven ranks only the group's count, passed from the forward to the backward, normalises right."""
    res = _run(_s0_uneven_worker, 2, (1, 5), timeout=900)
    for rank, rel_out, rel_g, rel_buf, exch, _, nbt in res:
        print(f"SyncBN S0 uneven rank {rank}: memory rel-L2 {rel_out:.3e}, weighted gradient rel-L2 {rel_g:.3e}, running buffers "
              f"rel-L2 {rel_buf:.3e}, {exch} exchanges")
        assert rel_out < 2e-2 and rel_g < 5e-2 and rel_buf < 1e-3, (rel_out, rel_g, rel_buf)   # the S0 train-test tolerances
        assert exch == 8 and nbt                                  # 2 RepMixerBlocks x (2 forward + 2 backward)
    assert res[0][5] == res[1][5]                                 # running buffers bit-identical across ranks
