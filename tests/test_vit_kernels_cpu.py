"""The fp64 statements of tests/ref_vit.py against textbook float64 torch (F.scaled_dot_product_attention over oracle/vitdet.py's
window partition, F.conv2d, F.layer_norm) and tests/emu_strict.py, and the bound logic on constructed rows: a row whose maximum
arrives in the last of six 96-key tiles, tied maxima across a tile boundary, a strict row whose running maximum rises at every key.
No GPU."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import emu_strict as E
import ref_vit as R

D = torch.float64


def _g(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _bf(t):
    return t.to(torch.bfloat16).to(D)


def _within(ref, bound, other, what):
    err = (ref - other).abs()
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} elements outside the bound (max err {err.max():.3g})"
    assert (bound > 0).all()


def _close(a, b, what=""):
    assert torch.allclose(a, b, rtol=1e-10, atol=1e-12), (what, (a - b).abs().max().item())


def _partition(t, B, H, W, win):
    """[B H W, X] -> [B nwin, win^2, X] exactly as oracle/vitdet.py's block() partitions (win = 0: one window per image)."""
    X = t.shape[-1]
    if win == 0:
        return t.view(B, H * W, X)
    return t.view(B, H // win, win, W // win, win, X).permute(0, 1, 3, 2, 4, 5).reshape(-1, win * win, X)


def _unpartition(o, B, H, W, win):
    X = o.shape[-1]
    if win == 0:
        return o.reshape(B * H * W, X)
    return o.view(B, H // win, W // win, win, win, X).permute(0, 1, 3, 2, 4, 5).reshape(B * H * W, X)


def _textbook(qkv, B, H, W, heads, win, scale, round_p):
    """softmax attention per window over the oracle's partition: exact (F.scaled_dot_product_attention), or with the unnormalised
    probabilities rounded to bf16 (through fp32) before P V and the row sums taken before that rounding."""
    t = _partition(qkv, B, H, W, win)
    n, L, _ = t.shape
    q, k, v = t.view(n, L, 3, heads, 64).permute(2, 0, 3, 1, 4)
    if round_p:
        s = scale * q @ k.transpose(-1, -2)
        p = torch.exp(s - s.amax(-1, keepdim=True))
        o = (p.float().to(torch.bfloat16).to(D) @ v) / p.sum(-1, keepdim=True)
    else:
        o = F.scaled_dot_product_attention(q, k, v, scale=scale)
    return _unpartition(o.permute(0, 2, 1, 3).reshape(n, L, heads * 64), B, H, W, win)


# ----------------------------------------------------------------------------------------------------------- bf16 attention
@pytest.mark.parametrize("B,H,W,heads,win,kernel", [(2, 12, 8, 2, 4, "mma"), (1, 8, 12, 1, 4, "tc"), (2, 6, 10, 2, 0, "mma"),
                                                    (1, 12, 16, 1, 0, "tc"), (1, 24, 24, 1, 24, "tc"), (1, 24, 48, 1, 12, "mma")])
def test_attention_bf16_statement(B, H, W, heads, win, kernel):
    """Windowed (non-square window grids included) and global, both kernels' key tiles (64; 96 at L = 192 and 576, 128 at L = 16)."""
    g = _g("attn", B, H, W, win, kernel)
    qkv = _bf(torch.randn(B * H * W, 3 * 64 * heads, generator=g, dtype=D) * 1.5)
    ref, bound = R.attention_bf16(qkv, B, H, W, heads, win, 0.125, kernel)
    _within(ref, bound, _textbook(qkv, B, H, W, heads, win, 0.125, True), "attention vs rounded-P textbook")
    exact = _textbook(qkv, B, H, W, heads, win, 0.125, False)
    vabs = _textbook(torch.cat([qkv[:, :128 * heads], qkv[:, 128 * heads:].abs()], 1), B, H, W, heads, win, 0.125, False)
    assert ((ref - exact).abs() <= 2.0 ** -8 * vabs + 1e-12).all()


def test_bn_tile_rule():
    assert [R.bn_tile(L) for L in (192, 576, 5184, 384, 200, 640, 144, 256)] == [96, 96, 96, 128, 128, 128, 128, 128]


def _rows(L, dominant):
    """One head, q = 1, v = 1 (the output is exactly 1 and its bound is the charge alone), small random keys; keys `dominant` = 0.5."""
    qkv = torch.zeros(L, 3 * 64, dtype=D)
    qkv[:, :64] = 1.0
    qkv[:, 64:128] = _bf(torch.randn(L, 64, generator=_g("rows", L), dtype=D) * 0.1)
    qkv[:, 128:] = 1.0
    for j in dominant:
        qkv[j, 64:128] = 0.5
    return qkv


def test_charge_where_the_maximum_arrives_in_the_last_of_six_tiles():
    """L = 576 on 96-key tiles: a row whose maximum is key 575 has every earlier tile's P rounded against a smaller running max
    and carries the full bf16 rounding there; with the maximum at key 5 those elements carry band() only."""
    late, early = _rows(576, [575]), _rows(576, [5])
    _, b_late = R.attention_bf16(late, 1, 24, 24, 1, 24, 0.125, "tc")
    _, b_early = R.attention_bf16(early, 1, 24, 24, 1, 24, 0.125, "tc")
    assert (b_late > b_early).all()


def test_charge_for_tied_maxima_across_a_tile_boundary():
    """Keys 95 and 96 tie for the maximum: the second 96-key tile may raise the fp32 running max (the tie may break either way),
    so tile 0 is charged; a single maximum at key 95 leaves it uncharged."""
    tied, single = _rows(576, [95, 96]), _rows(576, [95])
    _, b_tied = R.attention_bf16(tied, 1, 24, 24, 1, 24, 0.125, "tc")
    _, b_single = R.attention_bf16(single, 1, 24, 24, 1, 24, 0.125, "tc")
    assert (b_tied > b_single).all()


# ----------------------------------------------------------------------------------------------------------- exact operations
def test_im2col_patch_statement():
    g = _g("im2col")
    B, S, P, Kp = 2, 28, 14, 600
    x = torch.randn(B, 3, S, S, generator=g, dtype=D)
    cols = R.im2col_patch(x, P, Kp)
    assert cols.dtype == torch.bfloat16 and cols.shape == (B * 4, Kp) and (cols[:, 588:] == 0).all()
    for b, py, px, c, ky, kx in ((0, 0, 0, 0, 0, 0), (1, 1, 0, 2, 13, 5), (0, 1, 1, 1, 7, 13)):
        assert cols[b * 4 + py * 2 + px, c * P * P + ky * P + kx] == x[b, c, py * P + ky, px * P + kx].to(torch.bfloat16)
    w = torch.randn(5, 3, P, P, generator=g, dtype=D)
    _close(cols[:, :588].to(D) @ w.reshape(5, -1).t(), F.conv2d(_bf(x), w, stride=P).permute(0, 2, 3, 1).reshape(-1, 5))


@pytest.mark.parametrize("nchw,ks,stride,pad", [(True, 14, 14, 0), (False, 3, 1, 1), (False, 3, 2, 1), (True, 3, 2, 1)])
def test_im2col_f32_statement(nchw, ks, stride, pad):
    """cols @ the (ky, kx, c)-ordered weight is the convolution (emu_strict.conv2d_f32)."""
    g = _g("im2col_f32", nchw, ks, stride)
    x = torch.randn(2, 5, 28, 28, generator=g, dtype=D) if nchw else torch.randn(2, 13, 11, 6, generator=g, dtype=D)
    C = x.shape[1] if nchw else x.shape[3]
    w = torch.randn(7, C, ks, ks, generator=g, dtype=D)
    got = R.im2col_f32(x, ks, stride, pad, nchw) @ w.permute(0, 2, 3, 1).reshape(7, -1).t()
    _close(got, E.conv2d_f32(x, w, stride, pad, nchw=nchw).reshape(-1, 7))


def test_tokens_to_nchw_statement():
    x = torch.randn(2 * 35, 9, generator=_g("t2n"), dtype=D)
    assert torch.equal(R.tokens_to_nchw(x, 2, 35, 9), x.view(2, 5, 7, 9).permute(0, 3, 1, 2).reshape(2, 9, 35))


# ----------------------------------------------------------------------------------------------------------- strict statements
@pytest.mark.parametrize("act,after,res", [(None, False, False), ("gelu", False, True), ("hswish", True, True), ("gelu", True, False)])
def test_sgemm_statement(act, after, res):
    """Against emu_strict.sgemm; an fp32 run of the same sum (torch's CPU SGEMM) stays inside the bound."""
    g = _g("sgemm", act, after, res)
    M, N, K = 33, 20, 300
    a, w = torch.randn(M, K, generator=g, dtype=D), torch.randn(N, K, generator=g, dtype=D) / K ** 0.5
    sc, bi, r = torch.rand(N, generator=g, dtype=D) + 0.5, torch.randn(N, generator=g, dtype=D), torch.randn(M, N, generator=g, dtype=D)
    kw = dict(scale=sc, bias=bi, act=act, residual=r if res else None)
    ref, bound = R.sgemm(a, w, **kw, after=after)
    _close(ref, E.sgemm(a, w, **kw, act_after_res=after))
    f32 = E.sgemm(a.float(), w.float(), **{k: v.float() if torch.is_tensor(v) else v for k, v in kw.items()}, act_after_res=after)
    _within(ref, bound, f32.double(), "fp32 sgemm")


@pytest.mark.parametrize("win", [0, 4])
def test_rope_statement(win):
    from efficientsam3_b200.model.vitdet import compute_axial_cis
    g = _g("rope", win)
    B, H, W, C = 2, 8, 8, 128
    qkv = torch.randn(B * H * W, 3 * C, generator=g, dtype=D)
    table = torch.view_as_real(compute_axial_cis(64, win or H, win or W)).to(D).contiguous()
    ref, bound = R.rope(qkv, table, 2 * C, H, W, win)
    _close(ref, E.rope_f32(qkv.clone(), table, 2 * C, H, W, win)[:, :2 * C])
    f32 = E.rope_f32(qkv.float().clone(), table.float(), 2 * C, H, W, win)
    _within(ref, bound, f32[:, :2 * C].double(), "fp32 rope")


@pytest.mark.parametrize("C,shift", [(64, 0.0), (100, 30.0), (1024, 0.0), (160, 30.0)])
def test_ln_rows_statement(C, shift):
    g = _g("ln", C, shift)
    x = torch.randn(50, C, generator=g, dtype=D) * 3 + shift
    w, b = torch.rand(C, generator=g, dtype=D) + 0.5, torch.randn(C, generator=g, dtype=D)
    ref, bound = R.ln_rows(x, w, b, 1e-5)
    _close(ref, F.layer_norm(x, (C,), w, b, 1e-5))
    xf, mean = x.float(), x.float().mean(1, keepdim=True)           # the kernel's two-pass form in fp32
    d = xf - mean
    y = d * (1.0 / torch.sqrt((d * d).sum(1, keepdim=True) / C + 1e-5)) * w.float() + b.float()
    _within(ref, bound, y.double(), "fp32 two-pass LayerNorm")


@pytest.mark.parametrize("B,H,W,heads,hd,win,layout,bias,pad", [(2, 8, 8, 2, 64, 4, "blocks", False, False),
                                                                 (1, 6, 10, 1, 64, 0, "blocks", False, False),
                                                                 (2, 10, 10, 2, 32, 7, "per_head", True, True),
                                                                 (1, 5, 5, 3, 32, 7, "per_head", True, True)])
def test_attention_f32_statement(B, H, W, heads, hd, win, layout, bias, pad):
    """Against emu_strict.attention_f32 (windows padded with pad_row, one window larger than the grid); an fp32 softmax of the
    same scores stays inside the bound."""
    g = _g("af32", B, H, W, win, layout)
    C = heads * hd
    L = win * win if win else H * W
    qkv = torch.randn(B * H * W, 3 * C, generator=g, dtype=D)
    bs = torch.randn(heads, L, L, generator=g, dtype=D) if bias else None
    pr = torch.randn(3 * C, generator=g, dtype=D) if pad else None
    ref, bound = R.attention_f32(qkv, B, H, W, heads, hd, win, hd ** -0.5, layout, bs, pr)
    kw = dict(layout=layout, bias=bs, pad_row=pr)
    _close(ref, E.attention_f32(qkv, B, H, W, heads, hd, win, hd ** -0.5, **kw))
    f32 = E.attention_f32(qkv.float(), B, H, W, heads, hd, win, hd ** -0.5, layout=layout, bias=None if bs is None else bs.float(),
                          pad_row=None if pr is None else pr.float())
    _within(ref, bound, f32.double(), "fp32 attention")


def test_rises_counts_every_key_of_a_rising_row():
    """A row whose scores increase at every key rescales L - 1 times; a falling row never; a tie within the score error counts."""
    s = torch.arange(10, dtype=D).view(1, 10)
    z = torch.zeros(1, 1, dtype=D)
    assert R.rises(s, z).item() == 9 and R.rises(s.flip(-1), z).item() == 0
    assert R.rises(torch.tensor([[1.0, 1.0, 0.0]], dtype=D), torch.full((1, 1), 1e-9, dtype=D)).item() == 1


def test_strict_charge_grows_with_the_rescales():
    """Keys whose scores rise along the row charge every output one rescale each; the same keys in falling order charge none."""
    L, hd = 64, 32
    qkv = torch.zeros(L, 3 * hd, dtype=D)
    qkv[:, :hd] = 1.0
    qkv[:, hd:2 * hd] = (torch.arange(L, dtype=D) / L)[:, None]         # score of key j rises with j for every query
    qkv[:, 2 * hd:] = 1.0
    _, b_rise = R.attention_f32(qkv, 1, 8, 8, 1, hd, 0, 0.2, "per_head")
    fall = qkv.clone()
    fall[:, hd:2 * hd] = fall[:, hd:2 * hd].flip(0)
    _, b_fall = R.attention_f32(fall, 1, 8, 8, 1, hd, 0, 0.2, "per_head")
    assert (b_rise > b_fall).all()
