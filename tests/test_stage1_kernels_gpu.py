"""The stage-1 KD step's loss and optimiser kernels (kd_loss.cu: es3_kd_loss_fwd; train_ops.cu: es3_kd_loss_bwd, es3_grad_norm,
es3_adamw_flat with its GradScaler update), element by element against the fp64 statements of tests/ref_stage1.py, each output
element within its own bound; the valid mask, the counts, the non-finite flag and the scaler state bit for bit.

Outputs and workspaces are NaN-prefilled and called through _lib.call: every cell inside the output region must be written and lie
within its bound, every cell past it (a flat TAIL) keeps its sentinel bits.  Every case runs twice and must be bit-identical; a
sample run alone must give the same partials as inside its batch; a shape an entry point declines writes nothing; the ops wrappers
are bit-identical to the direct calls.  covered_keys() names the route keys (tests/routes.py) the tables run, for the route
closure of tests/test_route_closure_gpu.py (whole stage-1 image and text iterations).

Sections: (a) the valid mask of every image size along each axis, and of the (h, w) pairs whose edge pixels sit at lambda = 0, 1/2
and just past 1/2; (b) the forward and (c) the backward over batch, channels, embedding size, padding, cosine weight, the optional
operands and the value kinds where they go wrong (cos -> 1, cos = -1, |pred| around the 1e-8 clamp, zero teacher pixels, large
magnitudes); (d) the gradient norm over ragged and grid-capped arenas, with inf and nan at every place a float4 read can hold
them; (e) AdamW with clipping, unscaling, weight decay split inside a float4, bias corrections from t = 1 to 1e6, skipped steps,
and a 12-step sequence of the dynamic loss scale.

GAMMA = 2 (ref_train_bwd.GAMMA) holds without change.  The kernels' valid mask equals the exact one on every pixel of every case of
(a).  Worst err/bound per section in one run on an H100 80GB HBM3 (700 W power limit), all fp32 outputs: KD partials 0.060,
per_sample 0.022, out3 0.017, dpred 0.334; gradient norm 0.0088; AdamW 0.322 (p, m, v of the table), 0.283 (the sequence).  The
file (89 tests) took 12 s there.  With kd_loss_bwd_kernel's cosine term back at dot / (na^3 nt), the rows with 0 < |pred| < 1e-8
and a cosine weight above 0 (five of the seven "tiny" rows) fail in (c) and every other test passes.
"""
import numpy as np
import pytest
import torch

import ref_stage1 as R
from bounds import TAIL, _assert_untouched, _bits_equal, _check, _declined, _flat_out, _gen, _lib, _p, _pairwise, _st, _twice, report_worst
from routes import adamw_key, grad_norm_key

pytestmark = pytest.mark.gpu
_report_worst = report_worst("stage-1 kernels")


def _ops():
    from efficientsam3_b200 import ops
    return ops


def _nblk(E):
    return -(-E * E // 256)


def _fwd(lib, p, t, sz, img, w, ws, o3, per):
    B, C, E, _ = p.shape
    lib.call("es3_kd_loss_fwd", p.data_ptr(), t.data_ptr(), sz.data_ptr(), B, C, E, img, w, ws.data_ptr(), o3.data_ptr(), _p(per),
             _st())


def _bwd(lib, p, t, sz, per, sd, gs, img, w, out):
    B, C, E, _ = p.shape
    lib.call("es3_kd_loss_bwd", p.data_ptr(), t.data_ptr(), sz.data_ptr(), per.data_ptr(), _p(sd), gs, B, C, E, img, w, out.data_ptr(),
             _st())


# ----------------------------------------------------------------------------------------------------------- (a) valid mask
# (img, E): the stage-1 geometries (1008 / 72, 1024 / 64), sizes where img / E is not an fp32-exact ratio, and an upsampling one
MASK_GEOMS = [(1008, 72), (1024, 64), (100, 7), (252, 18), (1000, 63), (512, 37), (800, 50), (32, 64)]


def _edge_extents(img, E):
    """Extents whose last valid-or-not output pixel sits at each weight class: for every output index o, the extents that give it
    2E-weight exactly E (lambda = 1/2), just above E, and 0 or 2E (lambda = 0), the first of each class found."""
    found = {}
    for ext in range(1, img + 1):
        wt = R._axis_weights(img, E, ext)
        part = wt[(wt > 0) & (wt < 2 * E)]
        cls = "zero" if part.size == 0 else ("half" if (part == E).any() else ("past" if (part > E).any() else "below"))
        found.setdefault(cls, []).append(ext)
    return [v for c in ("zero", "half", "past", "below") for v in found.get(c, [])[:4]]


def _mask_sizes(img, E):
    """Every h at w = img, every w at h = img, the pairs of edge extents, and the 1 x 1 image."""
    full = [(h, img) for h in range(1, img + 1)] + [(img, w) for w in range(1, img)]
    ext = _edge_extents(img, E)
    return full + [(h, w) for h in ext for w in ext] + [(1, 1)]


@pytest.mark.parametrize("img,E", MASK_GEOMS)
def test_valid_mask_is_exact(cuda, img, E):
    """The kernels' valid mask equals the exact one (ref_stage1.valid_mask) on every pixel: the forward's count per sample, and the
    zero pattern of the backward with cosine weight 0 and pred != teacher everywhere (2 up (pred - teacher) != 0 on a valid pixel)."""
    lib = _lib(cuda)
    sizes = _mask_sizes(img, E)
    B = len(sizes)
    want = R.valid_masks(img, E, sizes).to(cuda)
    g = _gen(cuda, "mask", img, E)
    p = torch.randn(B, 1, E, E, device=cuda, generator=g)
    t = p + 0.5 + torch.rand(B, 1, E, E, device=cuda, generator=g)
    sz = torch.tensor(sizes, dtype=torch.int32, device=cuda)
    ws = torch.empty(B * _nblk(E) * 3, device=cuda)
    o3 = torch.empty(3, device=cuda)
    per = torch.full((B, 3), float("nan"), device=cuda)
    _fwd(lib, p, t, sz, img, 0.0, ws, o3, per)
    cnt = want.sum((1, 2)).to(torch.float32)
    bad = (per[:, 2] != cnt).nonzero().flatten().tolist()
    assert not bad, f"img {img} E {E}: mask counts differ for (h, w) {[sizes[i] for i in bad[:5]]}: got {per[bad[:5], 2].tolist()}, " \
                    f"exact {cnt[bad[:5]].tolist()}"
    if img > E:                                     # downsampled, the 1 x 1 image has no valid pixel: count 0, denominator 1
        assert float(per[-1, 2]) == 0.0 and float(per[-1, 0]) == 0.0 and float(per[-1, 1]) == 0.0
    dp = torch.full_like(p, float("nan"))
    _bwd(lib, p, t, sz, per, None, 1.0, img, 0.0, dp)
    got = dp[:, 0] != 0
    diff = (got != want).nonzero()
    assert diff.numel() == 0, f"img {img} E {E}: {diff.shape[0]} pixels differ, first (sample, y, x) {diff[0].tolist()} at " \
                              f"(h, w) {sizes[int(diff[0, 0])]}: kernel {bool(got[tuple(diff[0].tolist())])}"


# ----------------------------------------------------------------------------------------------------------- (b, c) KD loss
KINDS = ["normal", "fp16", "neg", "tiny", "zero_t", "big"]
TINY_NORMS = [0.0, 3e-9, 7e-9, 9.9e-9, 2e-8]     # |pred| of five pixels of sample 0: zero, below, at and above the 1e-8 clamp
IMG = {7: 100, 12: 192, 16: 256, 64: 1024, 72: 1008}
KD = _pairwise(dict(B=[1, 2, 3, 8], C=[1, 32, 256, 1024], E=[7, 12, 16, 64, 72], kind=KINDS, pad=["none", "right", "bottom", "mixed"],
                    w=[0.0, 0.5, 1.0], per=[True, False], sd=[True, False], gs=[1.0, 0.375]), seed=41)
KD += [(8, 1024, 72, "tiny", "mixed", 1.0, True, True, 0.375), (2, 1024, 64, "tiny", "right", 1.0, True, True, 1.0),
       (3, 256, 72, "fp16", "mixed", 1.0, True, True, 1.0)]          # the stage-1 geometries: the clamp, and stored fp16 targets


def _sizes(B, img, pad):
    """(h, w) rows: none (full images), right (w = 3/4), bottom (h = 2/3), or mixed (alternating, the last one full)."""
    rows = []
    for b in range(B):
        if pad == "none" or (pad == "mixed" and b == B - 1 and B > 1):
            rows.append((img, img))
        elif pad == "right" or (pad == "mixed" and b % 2 == 0):
            rows.append((img, img * 3 // 4))
        else:
            rows.append((img * 2 // 3, img))
    return rows


def _kd_inputs(cuda, B, C, E, kind, g):
    t = torch.randn(B, C, E, E, device=cuda, generator=g)
    p = torch.randn(B, C, E, E, device=cuda, generator=g)
    if kind == "fp16":                              # the stored targets: the teacher is the prediction rounded through fp16
        t = p.half().float()
    elif kind == "neg":
        p = -t
    elif kind == "tiny":                            # |pred| around the clamp, pointing mostly along the teacher (|cos| ~ 0.9)
        for j, r in enumerate(TINY_NORMS):
            d = t[0, :, 0, j] + 0.3 * torch.randn(C, device=cuda, generator=g)
            p[0, :, 0, j] = d / d.norm() * r if r > 0 else 0.0
    elif kind == "zero_t":                          # teacher pixels of norm 0, one with pred 0 too
        t[0, :, 0, :3] = 0.0
        p[0, :, 0, 2] = 0.0
        t[-1, :, E - 1, E - 1] = 0.0
    elif kind == "big":
        p, t = p * 1e3, t * 1e3
    return p.contiguous(), t.contiguous()


def _kd_id(c):
    return "B{}-C{}-E{}-{}-{}-w{}-per{}-sd{}-gs{}".format(*c)


@pytest.mark.parametrize("B,C,E,kind,pad,w,per_on,sd_on,gs", KD, ids=[_kd_id(c) for c in KD])
def test_kd_loss(cuda, B, C, E, kind, pad, w, per_on, sd_on, gs):
    """(b) ws [B, nblk, 3], per_sample [B, 3] and out3 of es3_kd_loss_fwd, (c) dpred of es3_kd_loss_bwd (fp64 autograd of the loss with
    F.cosine_similarity), with per_sample and scale_dev each present or not; the last sample alone gives its batch partials."""
    lib = _lib(cuda)
    ops = _ops()
    img = IMG[E]
    g = _gen(cuda, "kd", B, C, E, kind, pad, w)
    p, t = _kd_inputs(cuda, B, C, E, kind, g)
    sizes = _sizes(B, img, pad)
    sz = torch.tensor(sizes, dtype=torch.int32, device=cuda)
    mask = R.valid_masks(img, E, sizes).to(cuda)
    nb = _nblk(E)
    what = f"kd_loss B{B} C{C} E{E} {kind} {pad} w={w}"
    ws_buf, ws_in = _flat_out(B * nb * 3, torch.float32, cuda)
    outs = []

    def run(ws):
        o3, _ = _flat_out(3, torch.float32, cuda)
        per, _ = _flat_out(B * 3, torch.float32, cuda)
        _fwd(lib, p, t, sz, img, w, ws, o3, per if per_on else None)
        outs.append((o3, per))
    ws = _twice(run, ws_buf)
    _bits_equal(outs[0][0], outs[1][0], what + ": out3 twice")
    o3, per = outs[0]
    ref = R.kd_fwd(p.double(), t.double(), mask, w)
    _check("b kd ws", ws[:B * nb * 3].view(B, nb, 3), *ref["ws"], what + " ws")
    _assert_untouched(ws, ws_in, what + " ws")
    _check("b kd out3", o3[:3], *ref["out3"], what + " out3")
    _assert_untouched(o3, torch.arange(3 + TAIL, device=cuda) < 3, what + " out3")
    if per_on:
        _check("b kd per_sample", per[:B * 3].view(B, 3), *ref["per_sample"], what + " per_sample")
        _assert_untouched(per, torch.arange(B * 3 + TAIL, device=cuda) < B * 3, what + " per_sample")
    else:
        _assert_untouched(per, torch.zeros(B * 3 + TAIL, dtype=torch.bool, device=cuda), what + " per_sample absent")
    wo, wper = ops.kd_loss_fwd(p, t, sz, img, w)
    _bits_equal(wo, o3[:3], what + ": ops.kd_loss_fwd vs direct")
    if per_on:
        _bits_equal(wper, per[:B * 3].view(B, 3), what + ": ops.kd_loss_fwd per_sample vs direct")
    one_ws, one_o3, one_per = torch.empty(nb * 3, device=cuda), torch.empty(3, device=cuda), torch.empty(3, device=cuda)
    _fwd(lib, p[-1:], t[-1:], sz[-1:], img, w, one_ws, one_o3, one_per)
    _bits_equal(one_ws, ws[(B - 1) * nb * 3:B * nb * 3], what + ": the last sample alone (ws)")
    _bits_equal(one_per, wper[-1], what + ": the last sample alone (per_sample)")

    sdv = torch.tensor([1.25], device=cuda) if sd_on else None
    gtot = gs * (1.25 if sd_on else 1.0)
    dbuf, dins = _flat_out(B * C * E * E, torch.float32, cuda)
    dp = _twice(lambda o: _bwd(lib, p, t, sz, wper, sdv, gs, img, w, o), dbuf)
    rdp, bdp = R.kd_bwd(p.double(), t.double(), mask, w, gtot)
    got = dp[:B * C * E * E].view(B, C, E, E)
    _check("c kd dpred", got, rdp, bdp, what + f" bwd sd={sd_on} gs={gs}")
    assert not got.masked_select(~mask[:, None].expand_as(got)).any(), what + ": a padded pixel's gradient is not exactly 0"
    _assert_untouched(dp, dins, what + " dpred")
    _bits_equal(ops.kd_loss_bwd(p, t, sz, wper, img, w, gs, sdv), got, what + ": ops.kd_loss_bwd vs direct")


def test_kd_loss_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    p = torch.randn(1, 4, 7, 7, device=cuda)
    sz = torch.tensor([[100, 100]], dtype=torch.int32, device=cuda)
    ws, o3, per, dp = (torch.full((n,), float("nan"), device=cuda) for n in (3 + TAIL, 3 + TAIL, 3 + TAIL, 196 + TAIL))
    for B, C, E, img in [(0, 4, 7, 100), (1, 0, 7, 100), (1, 4, 0, 100), (1, 4, 7, 0)]:
        _declined(lib, "es3_kd_loss_fwd", (p.data_ptr(), p.data_ptr(), sz.data_ptr(), B, C, E, img, 1.0, ws.data_ptr(), o3.data_ptr(),
                                           per.data_ptr(), _st()), [ws, o3, per], f"kd fwd B{B} C{C} E{E} img{img}")
        _declined(lib, "es3_kd_loss_bwd", (p.data_ptr(), p.data_ptr(), sz.data_ptr(), per.data_ptr(), 0, 1.0, B, C, E, img, 1.0,
                                           dp.data_ptr(), _st()), [dp], f"kd bwd B{B} C{C} E{E} img{img}")


# ----------------------------------------------------------------------------------------------------------- (d) gradient norm
GN_CAP = 4096 * 16384
GN_N = [1, 3, 4, 5, 16383, 16384, 16385, 20_450_003, GN_CAP + 5]
GN_SCALE = 65536.0 * 8 * 1e-2        # a loss-scaled gradient summed over 8 ranks: loss scale 65536, unscaled RMS 1e-2


def _gn_call(lib, g, n, part, out):
    lib.call("es3_grad_norm", g.data_ptr(), n, part.data_ptr(), out.data_ptr(), _st())


def _nonfinite_places(n):
    """First and last element, each lane of a float4 (the middle one, and the first), and every element of a ragged tail."""
    q = (n // 4) // 2 * 4
    places = {0, n - 1} | {q + j for j in range(4) if q + j < n} | {j for j in range(4) if j < n}
    places |= set(range(n - n % 4, n))
    return sorted(places)


@pytest.mark.parametrize("n", GN_N)
def test_grad_norm(cuda, n):
    """norm_ws = (sum g^2, non-finite flag) against fp64 with the launch geometry's bound (ref_stage1.grad_norm); the flag for +inf,
    -inf and nan at every place of _nonfinite_places, the partial workspace and norm_ws written inside and nowhere past."""
    lib = _lib(cuda)
    g = torch.randn(n, device=cuda, generator=_gen(cuda, "gn", n)) * GN_SCALE
    nws = lib.size("es3_grad_norm_ws_floats", n)
    assert nws == 2 * R.gn_blocks(n)
    part_buf, part_in = _flat_out(nws, torch.float32, cuda)
    out_buf, out_in = _flat_out(2, torch.float32, cuda)
    parts = []

    def run(out):
        part = part_buf.clone()
        _gn_call(lib, g, n, part, out)
        parts.append(part)
    out = _twice(run, out_buf)
    _bits_equal(parts[0], parts[1], f"grad_norm n={n}: partials twice")
    _assert_untouched(parts[0], part_in, f"grad_norm n={n} partials")
    assert not torch.isnan(parts[0][:nws]).any(), f"grad_norm n={n}: a block partial was not written"
    _assert_untouched(out, out_in, f"grad_norm n={n} norm_ws")
    s, bound, flag = R.grad_norm(g)
    _check("d grad_norm", out[:1], torch.tensor([s], dtype=torch.float64, device=cuda), torch.tensor([bound], dtype=torch.float64, device=cuda),
           f"grad_norm n={n}")
    assert float(out[1]) == flag == 0.0
    ws2 = torch.zeros(8192, device=cuda)
    o2 = torch.zeros(2, device=cuda)
    _ops().grad_norm(g, ws2, o2)
    _bits_equal(o2, out[:2], f"grad_norm n={n}: ops.grad_norm vs direct")
    places = _nonfinite_places(n) if n < 1_000_000 else [0, n - 1, n // 2 // 4 * 4 + 1, n - 1 - (n % 4) // 2]
    for i in places:
        keep = g[i].clone()
        for bad in (float("inf"), float("-inf"), float("nan")):
            g[i] = bad
            o = torch.zeros(2, device=cuda)
            _gn_call(lib, g, n, part_buf.clone(), o)
            assert float(o[1]) == 1.0 and not torch.isfinite(o[0]), f"grad_norm n={n}: {bad} at {i} gives {o.tolist()}"
        g[i] = keep


def test_grad_norm_overflow_of_the_scaled_sum_sets_the_flag(cuda):
    """Two finite elements in different blocks whose squares are finite but whose sum is not: the block partials are finite, their
    double total rounds to fp32 inf, and the skip flag is set (the documented behaviour of a loss-scaled norm, kept as is)."""
    lib = _lib(cuda)
    n = 3 * 16384
    g = torch.zeros(n, device=cuda)
    g[0] = g[16384] = 1.5e19                                   # 2.25e38 each; FLT_MAX is 3.4e38
    part = torch.zeros(lib.size("es3_grad_norm_ws_floats", n), device=cuda)
    out = torch.zeros(2, device=cuda)
    _gn_call(lib, g, n, part, out)
    assert torch.isfinite(part).all() and float(out[0]) == float("inf") and float(out[1]) == 1.0


def test_grad_norm_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    g = torch.randn(64, device=cuda)
    part, out = torch.full((8 + TAIL,), float("nan"), device=cuda), torch.full((2 + TAIL,), float("nan"), device=cuda)
    _declined(lib, "es3_grad_norm", (g.data_ptr(), 0, part.data_ptr(), out.data_ptr(), _st()), [part, out], "grad_norm n = 0")
    _declined(lib, "es3_grad_norm", (g[1:].data_ptr(), 63, part.data_ptr(), out.data_ptr(), _st()), [part, out],
              "grad_norm misaligned")


# ----------------------------------------------------------------------------------------------------------- (e) AdamW + scaler
ADAMW = _pairwise(dict(n=[1, 3, 4, 5, 1021, 1_000_003], decay=["none", "all", "mult4", "inside"], step=[0, 1, 9, 10_000, 1_000_000],
                       betas=[(0.9, 0.999), (0.5, 0.9)], max_norm=[0.0, 1.0, 5.0], ratio=[0.5, 1.0, 2.0], inv_world=[1.0, 0.125],
                       scale=[1.0, 65536.0], wd=[0.0, 0.05], dynamic=[False, True], bad=[False, True]), seed=43)
ADAMW += [(1_000_003, "mult4", 0, (0.9, 0.999), 5.0, 2.0, 0.125, 65536.0, 0.05, True, False),     # FlatAdamW's stage-1 call
          (1021, "inside", 9, (0.9, 0.999), 5.0, 0.5, 1.0, 65536.0, 0.05, True, False)]


def _n_decay(n, kind):
    q = (n // 2) // 4 * 4
    return {"none": 0, "all": n, "mult4": q, "inside": min(q + 1, n)}[kind]


def _adamw_call(lib, p, g, m, v, n, nd, lr, betas, eps, wd, max_norm, inv_world, norm_ws, state, dynamic, interval):
    lib.call("es3_adamw_flat", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, nd, lr, betas[0], betas[1], eps, wd, max_norm,
             inv_world, norm_ws.data_ptr(), state.data_ptr(), int(dynamic), 2.0, 0.5, interval, _st())


def _arenas(cuda, n, step, g_key):
    gen = _gen(cuda, *g_key)
    p = torch.randn(n, device=cuda, generator=gen)
    if step == 0:                                              # a fresh optimiser
        m, v = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    else:
        m = torch.randn(n, device=cuda, generator=gen) * 1e-2
        v = torch.rand(n, device=cuda, generator=gen) * 1e-4
    return p, m, v, torch.randn(n, device=cuda, generator=gen)


def _adamw_check(section, got, ref, what):
    for k in ("p", "m", "v"):
        _check(section, got[k], *ref[k], f"{what} {k}")


def _adamw_id(c):
    return "n{}-{}-t{}-b{}-clip{}-x{}-iw{}-s{:g}-wd{}-dyn{}-bad{}".format(c[0], c[1], c[2], c[3][1], c[4], c[5], c[6], c[7], c[8], c[9],
                                                                          c[10])


@pytest.mark.parametrize("n,decay,step,betas,max_norm,ratio,inv_world,scale,wd,dynamic,bad", ADAMW, ids=[_adamw_id(c) for c in ADAMW])
def test_adamw_flat(cuda, n, decay, step, betas, max_norm, ratio, inv_world, scale, wd, dynamic, bad):
    """One es3_adamw_flat call: p, m, v against ref_stage1.adamw from the fp32 ABI scalars (clipping with the unscaled total norm at
    ratio x the limit), or bit for bit unchanged when the non-finite flag is set; the scaler state bit for bit; arenas past n keep
    their sentinels; the ops wrapper is bit-identical."""
    lib = _lib(cuda)
    nd = _n_decay(n, decay)
    lr, eps, interval = 2e-3, 1e-8, 3
    p, m, v, g = _arenas(cuda, n, step, ("adamw", n, decay, step, betas, max_norm, ratio))
    world_total = ratio * (max_norm if max_norm > 0 else 3.0)            # the unscaled, rank-averaged total norm
    g = g * (world_total / g.double().norm()).float() * (scale / inv_world)
    sumsq = float(np.float32((g.double() ** 2).sum().item()))
    norm_ws = torch.tensor([sumsq, 1.0 if bad else 0.0], device=cuda)
    state0 = torch.tensor([scale, 2.0, float(step), 0.0], device=cuda)
    bufs = []
    for x in (p, m, v):
        b, inside = _flat_out(n, torch.float32, cuda)
        b[:n] = x
        bufs.append(b)
    runs = []
    for _ in range(2):
        pb, mb, vb = (b.clone() for b in bufs)
        st = state0.clone()
        _adamw_call(lib, pb, g, mb, vb, n, nd, lr, betas, eps, wd, max_norm, inv_world, norm_ws, st, dynamic, interval)
        runs.append((pb, mb, vb, st))
    for a, b in zip(runs[0], runs[1]):
        _bits_equal(a, b, "adamw twice")
    pb, mb, vb, st = runs[0]
    what = f"adamw n{n} decay {decay} ({nd}) t{step} clip {max_norm} x{ratio}"
    for b, name in zip((pb, mb, vb), "pmv"):
        _assert_untouched(b, inside, f"{what} {name}")
    if bad:
        for b, x, name in zip((pb, mb, vb), (p, m, v), "pmv"):
            _bits_equal(b[:n], x, f"{what}: a skipped step changed {name}")
    else:
        ref = R.adamw(p.double(), g.double(), m.double(), v.double(), nd, R.f32(lr), tuple(map(R.f32, betas)), R.f32(eps), R.f32(wd),
                      R.f32(max_norm), R.f32(inv_world), sumsq, scale, float(step))
        _adamw_check("e adamw", {"p": pb[:n], "m": mb[:n], "v": vb[:n]}, ref, what)
    want = R.scaler_state(state0.cpu().numpy(), sumsq, bad, R.f32(inv_world), dynamic, interval)
    _bits_equal(st.cpu(), torch.from_numpy(want), f"{what}: scaler state {st.tolist()} != {want.tolist()}")
    pw, mw, vw, sw = p.clone(), m.clone(), v.clone(), state0.clone()
    _ops().adamw_flat(pw, g, mw, vw, nd, lr, betas, eps, wd, max_norm, inv_world, norm_ws, sw, dynamic_scale=dynamic,
                      growth_interval=interval)
    for a, b in zip((pw, mw, vw, sw), (pb[:n], mb[:n], vb[:n], st)):
        _bits_equal(a, b, what + ": ops.adamw_flat vs direct")


# 12 steps of the dynamic loss scale (growth interval 3): clean, inf and nan gradients mixed, the norm from es3_grad_norm
SEQUENCE = ["clean", "clean", "inf", "clean", "clean", "clean", "nan", "clean", "clean", "clean", "clean", "inf"]


def test_adamw_flat_sequence_of_the_dynamic_scale(cuda):
    """es3_grad_norm then es3_adamw_flat for 12 steps with growth interval 3: after every step the scaler state matches GradScaler
    bit for bit (backoff on inf / nan, growth after 3 clean steps in a row, the step count on clean steps only); a skipped step keeps
    p, m and v bit for bit, a clean one is within ref_stage1.adamw of the state before it."""
    lib = _lib(cuda)
    n, nd, lr, betas, eps, wd, interval = 1021, 512, 1e-3, (0.9, 0.999), 1e-8, 0.05, 3
    gen = _gen(cuda, "sequence")
    p, m, v = torch.randn(n, device=cuda, generator=gen), torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    state = torch.tensor([65536.0, 0.0, 0.0, 0.0], device=cuda)
    part, norm_ws = torch.zeros(lib.size("es3_grad_norm_ws_floats", n), device=cuda), torch.zeros(2, device=cuda)
    scales = []
    for i, kind in enumerate(SEQUENCE):
        g = torch.randn(n, device=cuda, generator=gen) * float(state[0]) * 0.3
        if kind != "clean":
            g[(37 * i) % n] = float(kind)
        _gn_call(lib, g, n, part, norm_ws)
        sumsq, bad = float(norm_ws[0]), float(norm_ws[1]) != 0.0
        assert bad == (kind != "clean")
        before = (p.clone(), m.clone(), v.clone(), state.clone())
        _adamw_call(lib, p, g, m, v, n, nd, lr, betas, eps, wd, 5.0, 1.0, norm_ws, state, True, interval)
        want = R.scaler_state(before[3].cpu().numpy(), sumsq, bad, 1.0, True, interval)
        _bits_equal(state.cpu(), torch.from_numpy(want), f"step {i} ({kind}): state {state.tolist()} != {want.tolist()}")
        if bad:
            for a, b, name in zip((p, m, v), before, "pmv"):
                _bits_equal(a, b, f"step {i}: a skipped step changed {name}")
        else:
            ref = R.adamw(*(x.double() for x in (before[0], g, before[1], before[2])), nd, R.f32(lr), tuple(map(R.f32, betas)),
                          R.f32(eps), R.f32(wd), 5.0, 1.0, sumsq, float(before[3][0]), float(before[3][2]))
            _adamw_check("e adamw sequence", {"p": p, "m": m, "v": v}, ref, f"sequence step {i}")
        scales.append(float(state[0]))
    assert scales == [65536.0, 65536.0, 32768.0, 32768.0, 32768.0, 65536.0, 32768.0, 32768.0, 32768.0, 65536.0, 65536.0, 32768.0]
    assert float(state[2]) == SEQUENCE.count("clean")


def test_adamw_flat_declined_shapes_write_nothing(cuda):
    lib = _lib(cuda)
    p, g, m, v = (torch.randn(64, device=cuda) for _ in range(4))
    norm_ws, state = torch.tensor([1.0, 0.0], device=cuda), torch.tensor([1.0, 0.0, 0.0, 0.0], device=cuda)
    for n, nd, off in [(0, 0, 0), (8, 9, 0), (8, -1, 0), (8, 4, 1)]:
        args = (p[off:].data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, nd, 1e-3, 0.9, 0.999, 1e-8, 0.05, 5.0, 1.0,
                norm_ws.data_ptr(), state.data_ptr(), 1, 2.0, 0.5, 3, _st())
        _declined(lib, "es3_adamw_flat", args, [p, m, v, state], f"adamw n={n} n_decay={nd} offset {off}")


# ----------------------------------------------------------------------------------------------------------- route closure
def covered_keys():
    """Every route key (tests/routes.py) some table row above runs."""
    keys = {("es3_kd_loss_fwd", c[6]) for c in KD} | {("es3_kd_loss_fwd", True) for _ in MASK_GEOMS}
    keys |= {("es3_kd_loss_bwd", c[7]) for c in KD} | {("es3_kd_loss_bwd", False) for _ in MASK_GEOMS}
    keys |= {grad_norm_key(n) for n in GN_N}
    keys |= {adamw_key(c[0], _n_decay(c[0], c[1]), c[4], c[9]) for c in ADAMW} | {adamw_key(1021, 512, 5.0, True)}
    return keys
