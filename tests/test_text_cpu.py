"""CPU: the text encoders' host side -- the oracle restatement against the reference fixtures, the tokenizer, state_dict keys,
the builders' variant table, checkpoint loading and the text-student checkpoint merge."""
import atexit
import gzip
import json
import os
import shutil
import tempfile
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from helpers import GOLD, load_golden
from oracle import text as OT
from oracle.weights import fill_state_dict


def _bpe_from_subset():
    """A full-length CLIP merge list rebuilt from tests/golden/text_bpe_subset.json: the recorded pairs at their ranks, every other
    rank a pair no text can contain (byte 0x00 is not in the byte alphabet), so token ids keep their positions and the tests'
    strings tokenise exactly as with the full 1.3 MB list (tests/golden/gen_golden_text.py)."""
    with open(os.path.join(GOLD, "text_bpe_subset.json"), encoding="utf-8") as f:
        rec = json.load(f)
    merges = rec["merges"]
    lines = ["#version: 0.2"] + [merges.get(str(r), f"\x00{r} \x00") for r in range(rec["n_merges"])]
    d = tempfile.mkdtemp(prefix="es3_bpe_")
    atexit.register(shutil.rmtree, d, True)
    path = os.path.join(d, "bpe_subset.txt.gz")
    with gzip.open(path, "wb") as f:
        f.write("\n".join(lines).encode("utf-8"))
    return path


BPE = _bpe_from_subset()
STUDENT_FIXTURES = ["text_s0_ctx32", "text_b_causal", "text_768", "text_s0_interp", "text_s0_resize16"]


def sig(sd):
    return [f"{k}|{','.join(map(str, v.shape))}|{str(v.dtype).replace('torch.', '')}" for k, v in sd.items()]


def build_student(g):
    """The native TextStudentEncoder the fixture's reference module was built as (tests/golden/gen_golden_text.py)."""
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import build_text_student_model, text_student_cfg
    backbone, ctx, table, resize = str(g["backbone"]), int(g["ctx"]), int(g["table"]), int(g["resize"])
    layers = eval(str(g["layers"]))
    if layers is None:
        cfg = NS(MODEL=NS(BACKBONE=backbone, BPE_PATH=BPE),
                 DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=77 if resize else ctx, POS_EMBED_TABLE_SIZE=table))
        m = build_text_student_model(cfg)
    else:
        cfg = text_student_cfg(backbone)
        cfg.update(layers, context_length=ctx)
        m = TextStudentEncoder(cfg=cfg, context_length=ctx, output_dim=256, bpe_path=BPE)
    if resize:
        m.set_context_length(resize)
    return m.eval()


def oracle_cfg(m):
    enc = m.encoder
    mct = type(enc.transformer[0]).__name__ == "RepMixerBlock"
    n = len(enc.transformer) - (2 if mct else 0)
    heads = enc.transformer[1 if mct else 0].pre_norm_mha[1].num_heads
    return dict(causal_masking=enc.causal_masking, n_transformer_layers=n, model_name="mct" if mct else "base",
                n_heads_per_layer=heads, dim=enc.model_dim, ffn_multiplier_per_layer=4.0)


@pytest.mark.parametrize("name", STUDENT_FIXTURES)
def test_student_keys_and_oracle_match_reference(name):
    g = load_golden(name)
    m = build_student(g)
    assert sig(m.state_dict()) == [str(k) for k in g["keys"]]
    sd = fill_state_dict(m.state_dict(), int(g["seed_w"]))
    ids = torch.from_numpy(g["ids"])
    assert torch.equal(m.tokenizer(OT_CAPTIONS(), context_length=m.context_length), ids)
    cfg = oracle_cfg(m)
    with torch.no_grad():
        mask, mem, emb = OT.text_student(sd, ids, cfg)
        pooled = OT.mobileclip_pooled(sd, ids, cfg)
    assert torch.equal(mask, torch.from_numpy(g["mask"]))
    keep = g["embeds"].shape[1]
    np.testing.assert_allclose(emb[:, :keep].numpy(), g["embeds"], rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(mem.numpy(), g["memory"], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(pooled.numpy(), g["pooled"], rtol=2e-5, atol=2e-5)


def OT_CAPTIONS():
    return [str(s) for s in load_golden("text_tokens")["strings"][:6]]


def test_teacher_keys_and_oracle_match_reference():
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
    g = load_golden("text_teacher")
    t = SAM3TextTeacherEncoder(context_length=int(g["ctx"]), bpe_path=BPE, ve_overrides=dict(layers=int(g["layers"])))
    pre = "sam3.backbone.language_backbone."
    assert sig(t.state_dict()) == [pre + str(k) for k in g["keys"]]
    ve = t.sam3.backbone.language_backbone
    sd = fill_state_dict(ve.state_dict(), int(g["seed_w"]))
    ids = torch.from_numpy(g["ids"])
    with torch.no_grad():
        mask, mem, emb = OT.ve_text_encoder(sd, ids, heads=16)
    assert torch.equal(mask, torch.from_numpy(g["mask"]))
    np.testing.assert_allclose(emb[:, :g["embeds"].shape[1]].numpy(), g["embeds"], rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(mem.numpy(), g["memory"], rtol=2e-5, atol=2e-5)
    t.train()
    assert not t.training and not ve.training


def test_tokenizer_ids_match_reference():
    from efficientsam3_b200.model.tokenizer_ve import SimpleTokenizer
    g = load_golden("text_tokens")
    tok = SimpleTokenizer(bpe_path=BPE)
    strings = [str(s) for s in g["strings"]]
    assert tok.vocab_size == 49408 and tok.sot_token_id == 49406 and tok.eot_token_id == 49407
    for n in (16, 32, 77):
        got = tok(strings, context_length=n)
        assert torch.equal(got, torch.from_numpy(g[f"ids_{n}"])), n
    assert tok("!", context_length=4).tolist() == [[49406, 256, 49407, 0]]     # a standalone "!" is never id 0
    assert tok("", context_length=4).tolist() == [[49406, 49407, 0, 0]]
    long = tok("x " * 100, context_length=16)[0]
    assert long[-1] == 49407 and (long != 0).all()                              # truncation keeps EOT last


def test_string_input_without_vocabulary_raises():
    from efficientsam3_b200.stage1.model import build_text_student_model
    m = build_text_student_model(NS(MODEL=NS(BACKBONE="MobileCLIP-S0"), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32))).eval()
    with pytest.raises(ValueError, match="tokenizer"):
        m.tokenize(["a cat"])


def test_variant_table_and_unknown_name_fallthrough():
    from efficientsam3_b200.stage1.model import build_text_student_model
    want = {"MobileCLIP-S0": (512, 6, "RepMixerBlock", False), "MobileCLIP-S1": (512, 12, "TransformerEncoder", False),
            "MobileCLIP2-S0": (512, 12, "TransformerEncoder", False), "MobileCLIP2-S2": (512, 12, "TransformerEncoder", False),
            "MobileCLIP-B": (512, 12, "TransformerEncoder", True), "MobileCLIP2-S3": (768, 12, "TransformerEncoder", False),
            "MobileCLIP2-S4": (768, 12, "TransformerEncoder", False), "MobileCLIP2-L": (768, 12, "TransformerEncoder", False),
            "no-such-backbone": (512, 12, "TransformerEncoder", False)}
    for name, (dim, n, first, causal) in want.items():
        m = build_text_student_model(NS(MODEL=NS(BACKBONE=name), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=16)))
        enc = m.encoder
        assert (enc.model_dim, len(enc.transformer), type(enc.transformer[0]).__name__, enc.causal_masking) == \
            (dim, n, first, causal), name
        assert enc.positional_embedding.pos_embed.pos_embed.shape == (1, 1, 16, dim)
        assert m.projector.out_features == 256
    m = build_text_student_model(NS(MODEL=NS(BACKBONE="MobileCLIP-S0"),
                                    DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32, POS_EMBED_TABLE_SIZE=77)))
    assert m.context_length == 32 and m.encoder.positional_embedding.pos_embed.num_embeddings == 77
    assert sum(1 for _ in m.state_dict()) == 111


def test_pretrained_full_mobileclip_checkpoint_is_renamed(tmp_path):
    from efficientsam3_b200.stage1.model import build_text_student_model
    cfg = NS(MODEL=NS(BACKBONE="MobileCLIP-S0"), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=32))
    src = build_text_student_model(cfg)
    sd = fill_state_dict(src.state_dict(), 7)
    full = {("text_encoder." + k[len("encoder."):]): v for k, v in sd.items() if k.startswith("encoder.")}
    full["image_encoder.stem.weight"] = torch.zeros(3)
    torch.save(full, tmp_path / "mobileclip.pt")
    cfg.MODEL.PRETRAINED = str(tmp_path / "mobileclip.pt")
    m = build_text_student_model(cfg)
    for k, v in m.state_dict().items():
        if k.startswith("encoder."):
            assert torch.equal(v, sd[k]), k
    cfg.MODEL.PRETRAINED = str(tmp_path / "missing.pt")          # a load error only warns (stage1/model.py:158-163)
    build_text_student_model(cfg)


def test_merge_text_student_into_sam3():
    from efficientsam3_b200.stage1.convert import merge_text_student_into_sam3
    student = {"module.encoder.embedding_layer.weight": 1, "detector.backbone.language_backbone.projector.weight": 2,
               "backbone.language_backbone.projector.bias": 3}
    sam3 = {"detector.backbone.language_backbone.encoder.token_embedding.weight": 10,
            "detector.backbone.language_backbone.resizer.weight": 11,
            "detector.backbone.vision_backbone.trunk.pos_embed": 12, "detector.transformer.x": 13, "tracker.y": 14}
    got = merge_text_student_into_sam3(student, sam3)
    assert got == {"detector.backbone.language_backbone.encoder.embedding_layer.weight": 1,
                   "detector.backbone.language_backbone.projector.weight": 2,
                   "detector.backbone.language_backbone.projector.bias": 3,
                   "detector.backbone.vision_backbone.trunk.pos_embed": 12, "detector.transformer.x": 13, "tracker.y": 14}
    got = merge_text_student_into_sam3(student, sam3, replace_prefix="detector.backbone.language_backbone.resizer",
                                       skip_teacher_prefixes=["tracker"])
    assert "detector.backbone.language_backbone.encoder.token_embedding.weight" in got
    assert "detector.backbone.language_backbone.resizer.weight" not in got and "tracker.y" not in got


def test_flops_from_shapes():
    from efficientsam3_b200.stage1.model import text_student_cfg
    s0 = OT.flops_mobileclip(text_student_cfg("MobileCLIP-S0"), 64, 32, 256)
    assert 60e9 < s0 < 80e9, s0                      # about 69 GFLOP per batch of 64 x 32
    assert 1.1e12 < OT.flops_ve(1024, 24, 64, 32) < 1.4e12
