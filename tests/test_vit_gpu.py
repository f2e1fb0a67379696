"""GPU parity of the native teacher encoder (module API -> C ABI) and of the QKV GEMM's RoPE epilogue.  The trunk's own kernels
(attention, patch im2col, LayerNorm, the token layout change) are held element by element to fp64 bounds in
tests/test_vit_kernels_gpu.py and tests/test_text_kernels_gpu.py.

Tolerances (stated): the RoPE epilogue 2e-3 of the tensor scale;
end-to-end trunk embedding (bf16 GEMM operands, fp32 residual stream, fp32 softmax/LN statistics):
relative L2 <= 2e-2, cosine >= 0.9995 against the fp32 reference / oracle.
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from helpers import cosine, load_golden, max_err_over_scale, rel_l2, sd_from_keys

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _close(got, ref, tol, what=""):
    err = max_err_over_scale(got.float().cpu(), ref.float().cpu())
    assert err <= tol, f"{what}: max err / scale = {err:.3e} > {tol}"


@pytest.mark.parametrize("H,W,win", [(8, 8, 4), (24, 24, 0)])
def test_qkv_rope_epilogue(cuda, H, W, win):
    """QKV projection with the RoPE epilogue vs Linear + apply_rotary_enc (vitdet.py:68-90)."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.model.vitdet import compute_axial_cis
    heads, C, B = 2, 128, 2
    g = torch.Generator().manual_seed(H + win)
    a = _bf(torch.randn(B * H * W, C, generator=g)).to(cuda)
    w = _bf(torch.randn(3 * C, C, generator=g) / math.sqrt(C)).to(cuda)
    bias = torch.randn(3 * C, generator=g).to(cuda)
    if win:
        cis = compute_axial_cis(64, win, win, scale_pos=1.0)
    else:
        cis = compute_axial_cis(64, H, W, scale_pos=8 / H)
    tab = torch.view_as_real(cis).float().contiguous().to(cuda)
    out = ops.gemm(a, w, bias=bias, rope=(tab, 2 * C, H, W, win), out_dtype=torch.float32)
    lin = (a.float() @ w.float().t() + bias).view(B, H, W, 3, heads, 32, 2)
    hh = torch.arange(H, device=cuda).view(H, 1).expand(H, W)
    ww = torch.arange(W, device=cuda).view(1, W).expand(H, W)
    idx = ((hh % win) * win + (ww % win)) if win else (hh * W + ww)
    c = torch.view_as_complex(tab)[idx]                       # [H, W, 32]
    qk = torch.view_as_complex(lin[:, :, :, :2].contiguous()) * c.view(1, H, W, 1, 1, 32)
    ref = lin.clone()
    ref[:, :, :, :2] = torch.view_as_real(qk)
    _close(out, ref.reshape(B * H * W, 3 * C), 2e-3, "rope epilogue")


def _check(got, ref, what, l2=2e-2, cs=0.9995):
    a, c = rel_l2(got, ref), cosine(got, ref)
    print(f"{what}: rel_l2={a:.3e} cos={c:.6f} max/scale={max_err_over_scale(got, ref):.3e}")
    assert a <= l2 and c >= cs, (what, a, c)


def test_vit_small_matches_reference_fixture(cuda):
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    g = load_golden("vit_small_112")
    cfg = eval(str(g["cfg"]))
    sd = sd_from_keys(g["keys"], int(g["seed_w"]))
    m = create_sam3_vit_backbone(**cfg)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.endswith("freqs_cis") for k in missing)
    assert [f"{k}" for k in m.state_dict().keys()] == [str(r).split("|")[0] for r in g["keys"]]
    m = m.to(cuda).eval()
    x = torch.randn(int(g["batch"]), 3, cfg["img_size"], cfg["img_size"], generator=torch.Generator().manual_seed(int(g["seed_x"])))
    out = m(x.to(cuda))[-1].cpu()
    assert out.shape == tuple(g["out"].shape)
    _check(out, g["out"], "vit_small vs reference fixture")


@pytest.mark.parametrize("cfg,batch", [
    (dict(img_size=336, pretrain_img_size=112, patch_size=14, embed_dim=256, depth=4, num_heads=4, mlp_ratio=4.625,
          window_size=8, global_att_blocks=(1, 3)), 2),
    # full-width teacher geometry (1008px, 72x72 tokens, 24-windows, dim 1024, 16 heads), reduced depth so the
    # CPU oracle finishes in seconds
    (dict(img_size=1008, pretrain_img_size=336, patch_size=14, embed_dim=1024, depth=3, num_heads=16, mlp_ratio=4.625,
          window_size=24, global_att_blocks=(2,)), 1),
])
def test_vit_matches_oracle(cuda, cfg, batch):
    from efficientsam3_b200.model.vitdet import create_sam3_vit_backbone
    from oracle import vitdet as O
    from oracle.weights import fill_state_dict
    m = create_sam3_vit_backbone(**cfg)
    sd = {k: v for k, v in fill_state_dict(m.state_dict(), 33).items() if not v.is_complex()}
    m.load_state_dict(sd, strict=False)
    x = torch.randn(batch, 3, cfg["img_size"], cfg["img_size"], generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        ref = O.vit_trunk(sd, "", x, cfg)
    out = m.to(cuda).eval()(x.to(cuda))[-1].cpu()
    _check(out, ref, f"vit {cfg['img_size']}/{cfg['embed_dim']} vs oracle")


def test_teacher_encoder_api(cuda):
    """SAM3ImageTeacherEncoder drop-in: key prefix, frozen/eval behaviour, output contract."""
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    t = SAM3ImageTeacherEncoder(embed_size=72, vit_overrides=dict(depth=2, global_att_blocks=(1,)))
    assert all(k.startswith("sam3.backbone.vision_backbone.trunk.") for k in t.state_dict())
    assert not any(p.requires_grad for p in t.parameters())
    t.train()
    assert not t.training
    out = t.to(cuda)(torch.randn(1, 3, 1008, 1008, device=cuda))
    assert out.shape == (1, 1024, 72, 72) and out.dtype == torch.float32 and torch.isfinite(out).all()
    with pytest.raises(AssertionError):
        t(torch.randn(1, 3, 1022, 1022, device=cuda))   # the reference asserts on any size but 1008 (SURVEY D2)


def test_teacher_resize_and_embedding_dump(cuda, tmp_path):
    """A21: teacher forward -> device fp16 cast -> double-buffered D2H -> store records; read back through the store reader
    and compare with `model(x).half()` record by record (bit-exact: same forward, same RN cast)."""
    import numpy as np
    import torch.nn.functional as F
    from efficientsam3_b200.stage1 import embeddings as E
    from efficientsam3_b200.stage1.model import SAM3ImageTeacherEncoder
    torch.manual_seed(0)
    t = SAM3ImageTeacherEncoder(embed_size=64, vit_overrides=dict(depth=1, global_att_blocks=())).to(cuda)
    xs = [torch.randn(2, 3, 1008, 1008) for _ in range(3)]
    # resize path == bilinear of the 72x72 map
    t72 = SAM3ImageTeacherEncoder(embed_size=72, vit_overrides=dict(depth=1, global_att_blocks=())).to(cuda)
    t72.load_state_dict(t.state_dict())
    ref = F.interpolate(t72(xs[0].to(cuda)), size=(64, 64), mode="bilinear", align_corners=False)
    got = t(xs[0].to(cuda))
    assert got.shape == (2, 1024, 64, 64)
    assert (got - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()

    keys = [[f"img_{b}_{i}" for i in range(2)] for b in range(3)]
    keys[2][1] = keys[0][0]                         # duplicate key: the first record must win
    seeds = [[10 * b + i for i in range(2)] for b in range(3)]
    loader = [((list(x), None), (keys[b], np.array(seeds[b], dtype=np.int32))) for b, x in enumerate(xs)]
    path = str(tmp_path / "emb")
    n = E.save_embeddings_one_epoch(t, loader, path, rank=0)
    assert n == 6
    rd = E.EmbeddingStoreReader(path, E.item_size(1024, 64 * 64), 0)
    for b, x in enumerate(xs):
        want = t(x.to(cuda)).half().cpu().numpy()
        for i in range(2):
            if b == 2 and i == 1:
                continue
            seed, emb = rd.read_embedding(keys[b][i], (1024, 64, 64))
            assert seed == seeds[b][i]
            assert np.array_equal(emb, want[i]), (b, i)
    seed, emb = rd.read_embedding(keys[0][0], (1024, 64, 64))
    assert seed == 0
    with open(os.path.join(path, "rank0-keys.txt")) as f:
        assert len(f.read().split()) == 5
