"""GPU: the native text encoders (MobileCLIP students, SAM3 text teacher) end to end from strings against the reference
fixtures and the CPU oracle, batch invariance, the text dump, the raise paths (the kernels element by element:
tests/test_text_kernels_gpu.py)."""
import numpy as np
import pytest
import torch

from helpers import cosine, load_golden, rel_l2
from oracle import text as OT
from oracle.weights import fill_state_dict
from test_text_cpu import BPE, STUDENT_FIXTURES, build_student, oracle_cfg

pytestmark = pytest.mark.gpu


def captions():
    return [str(s) for s in load_golden("text_tokens")["strings"][:6]]


def loaded_student(g, dev):
    m = build_student(g)
    m.load_state_dict(fill_state_dict(m.state_dict(), int(g["seed_w"])))
    return m.to(dev).eval()


def small_teacher(dev, ctx=32, layers=2, seed=106):
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
    t = SAM3TextTeacherEncoder(context_length=ctx, bpe_path=BPE, ve_overrides=dict(layers=layers))
    ve = t.sam3.backbone.language_backbone
    ve.load_state_dict(fill_state_dict(ve.state_dict(), seed))
    return t.to(dev)


def check_memory(got, ref):
    assert got.shape == ref.shape and got.dtype == torch.float32
    r, c = rel_l2(got.cpu(), ref), cosine(got.cpu(), ref)
    assert r <= 2e-2 and c >= 0.9995, (r, c)


# ------------------------------------------------------------------------------------------------ end to end vs fixtures
@pytest.mark.parametrize("name", STUDENT_FIXTURES)
def test_student_fixture_from_strings(cuda, name):
    g = load_golden(name)
    m = loaded_student(g, cuda)
    mask, mem, emb = m(captions(), device=cuda)
    assert mask.is_cuda and torch.equal(mask.cpu(), torch.from_numpy(g["mask"]))
    check_memory(mem, torch.from_numpy(g["memory"]))
    keep = g["embeds"].shape[1]
    np.testing.assert_allclose(emb[:, :keep].cpu().numpy(), g["embeds"], rtol=1e-6, atol=1e-7)
    pooled = m.encoder(torch.from_numpy(g["ids"]))
    assert rel_l2(pooled.cpu(), torch.from_numpy(g["pooled"])) <= 2e-2


def test_teacher_fixture_from_strings(cuda):
    g = load_golden("text_teacher")
    t = small_teacher(cuda, ctx=int(g["ctx"]), layers=int(g["layers"]), seed=int(g["seed_w"]))
    mask, mem, emb = t.sam3.backbone.language_backbone(captions(), device=cuda)
    assert torch.equal(mask.cpu(), torch.from_numpy(g["mask"]))
    check_memory(mem, torch.from_numpy(g["memory"]))
    np.testing.assert_allclose(emb[:, :g["embeds"].shape[1]].cpu().numpy(), g["embeds"], rtol=0, atol=0)
    check_memory(t(captions(), device=cuda), torch.from_numpy(g["memory"]))


def test_teacher_full_depth_vs_oracle(cuda):
    """The 24-layer, 1024-wide SAM3 text encoder as SAM3TextTeacherEncoder builds it, tokenised at 16 (the ctx-16 configs)."""
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
    t = SAM3TextTeacherEncoder(context_length=16, bpe_path=BPE)
    ve = t.sam3.backbone.language_backbone
    sd = fill_state_dict(ve.state_dict(), 7)
    ve.load_state_dict(sd)
    t = t.to(cuda)
    caps = captions()[:4]
    mem = t(caps, device=cuda)
    ids = ve.tokenizer(caps, context_length=16)
    with torch.no_grad():
        _, ref, _ = OT.ve_text_encoder(sd, ids, heads=16)
    check_memory(mem, ref)


@pytest.mark.parametrize("backbone", ["MobileCLIP-B", "MobileCLIP-S1"])
def test_student_full_depth_vs_oracle(cuda, backbone):
    from types import SimpleNamespace as NS
    from efficientsam3_b200.stage1.model import build_text_student_model
    m = build_text_student_model(NS(MODEL=NS(BACKBONE=backbone, BPE_PATH=BPE), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32)))
    sd = fill_state_dict(m.state_dict(), 8)
    m.load_state_dict(sd)
    m = m.to(cuda).eval()
    _, mem, _ = m(captions(), device=cuda)
    ids = m.tokenizer(captions(), context_length=32)
    with torch.no_grad():
        _, ref, _ = OT.text_student(sd, ids, oracle_cfg(m))
    check_memory(mem, ref)


def test_caption_alone_equals_caption_in_batch_of_64(cuda):
    g = load_golden("text_s0_ctx32")
    m = loaded_student(g, cuda)
    caps = captions()
    batch = [caps[i % len(caps)] + (f" number {i}" if i >= len(caps) else "") for i in range(64)]
    _, alone, _ = m([caps[1]], device=cuda)
    _, many, _ = m(batch, device=cuda)
    assert torch.equal(alone[:, 0], many[:, 1])
    t = small_teacher(cuda)
    assert torch.equal(t([caps[3]], device=cuda)[:, 0], t(batch, device=cuda)[:, 3])


# ------------------------------------------------------------------------------------------------ dump and raise paths
def test_text_dump_reads_back_fp16_teacher_output(cuda, tmp_path):
    from efficientsam3_b200.stage1.embeddings import EmbeddingStoreReader, item_size, save_text_embeddings_one_epoch
    t = small_teacher(cuda)
    caps = captions()
    keys = [f"cap_{i}" for i in range(len(caps))]
    loader = [[caps[:3], [keys[:3], [11, 12, 13]]], [(c, (k, 20 + i)) for i, (c, k) in enumerate(zip(caps[3:], keys[3:]))]]
    n = save_text_embeddings_one_epoch(t, loader, str(tmp_path / "store"), rank=0)
    assert n == len(caps)
    ref = t(caps, device=cuda).transpose(0, 1).half().cpu().numpy()
    rd = EmbeddingStoreReader(str(tmp_path / "store"), item_size(256, 32))
    for i, k in enumerate(keys):
        seed, emb = rd.read_embedding(k, (32, 256))
        assert seed == (11 + i if i < 3 else 20 + i - 3)
        assert np.array_equal(emb, ref[i])
    rd.close()


def test_raise_paths(cuda):
    from types import SimpleNamespace as NS
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import build_text_student_model
    cfg = NS(MODEL=NS(BACKBONE="MobileCLIP-S0", BPE_PATH=BPE), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32))
    m = build_text_student_model(cfg).eval()
    with pytest.raises(RuntimeError, match="CPU fallback"):
        m(["a cat"])
    m = m.to(cuda)
    with pytest.raises(ValueError, match="CUDA fp32"):
        m.encoder(torch.zeros(1, 32, 512), return_all_tokens=True, input_is_embeddings=True)
    with pytest.raises(NotImplementedError, match="eval"):
        m.train()(["a cat"])
    m.eval()
    with pytest.raises(NotImplementedError, match="strict"):
        with ops.strict_precision():
            m(["a cat"])
    with pytest.raises(NotImplementedError, match="key_padding_mask"):
        m.encoder(torch.zeros(1, 32, dtype=torch.long), key_padding_mask=torch.zeros(1, 32, dtype=torch.bool))
    bad = torch.zeros(2, 32, dtype=torch.long)
    bad[1, 3] = 49408
    n0 = ops.launch_count
    with pytest.raises(ValueError, match="out of range"):
        m(bad.to(cuda))
    with pytest.raises(ValueError, match="out of range"):
        m.encoder(-bad)
    assert ops.launch_count == n0                     # rejected on the host: nothing reached the device
    long = build_text_student_model(NS(MODEL=NS(BACKBONE="MobileCLIP-S0", BPE_PATH=BPE),
                                       DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=160))).to(cuda).eval()
    with pytest.raises(ValueError, match="1..128"):
        long(["a cat"])
    t = small_teacher(cuda)
    t.train()
    assert not t.training
    with pytest.raises(NotImplementedError, match="strict"):
        with ops.strict_precision():
            t(["a cat"], device=cuda)
