"""Generate the text-encoder golden fixtures by running the UNMODIFIED reference modules (CPU fp32).

    python tests/golden/gen_golden_text.py

Needs /root/reference (absent on the GPU box -- fixtures are committed).  Weights come from oracle.weights.fill_state_dict(seed)
so they are reproducible without being stored.  Writes:

  text_tokens.npz        reference tokenizer ids of TEXT_TOKEN_STRINGS at context 16 / 32 / 77
  text_*.npz             students / teacher: keys, ids, mask, memory, the first captions' input_embeds, pooled output
  text_bpe_subset.json   the part of the CLIP merge list (bpe_simple_vocab_16e6.txt.gz, 1.3 MB, not committed) that the
                         tests' strings touch: every ranked pair that is ever adjacent while BPE runs on one of their words,
                         with its rank.  tests/test_text_cpu.py rebuilds a full-length merge list from it (unused ranks become
                         pairs no text can contain), on which the tokenizer gives exactly the full vocabulary's ids for
                         these strings: at every step the lowest-ranked adjacent pair is one of the recorded ones.
"""
from __future__ import annotations

import json
import os
import sys
from types import SimpleNamespace as NS

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))

import install  # noqa: E402  (oracle/ref_shim/install.py)

install.install()
from oracle.weights import fill_state_dict  # noqa: E402

torch.set_grad_enabled(False)

REF_BPE = "/root/reference/sam3/assets/bpe_simple_vocab_16e6.txt.gz"

TEXT_CAPTIONS = ["a photo of a cat", "a dog!", "",
                 "two red apples on 3 wooden tables next to 12 bananas and a very long list of other fruit that keeps going "
                 "well beyond the thirty two token context of the text encoders",
                 "Café crème, naïve résumé & co.", "  multiple   spaces\tand\nnewlines  "]
TEXT_TOKEN_STRINGS = TEXT_CAPTIONS + ["!", "!!", "hello world", "HELLO World", "it's what they'll do", "1234567 apples",
                                      "日本語のテキスト", "a \U0001f436 dog", "rock &amp; roll",
                                      "<start_of_text> hello", "x" * 40, "don't-stop_me now", "3.14159 is pi"]
# other strings the tests tokenise (tests/test_text_cpu.py, tests/test_text_gpu.py): only their merges are recorded
OTHER_TEST_STRINGS = ["a cat", "x " * 100, "number 0123456789"]
TEXT_EMBED_KEEP = 2      # captions whose input_embeds are stored (the gather is exact; two rows pin it, the rest is size)


def keyshapes(sd):
    return np.array([f"{k}|{','.join(map(str, v.shape))}|{str(v.dtype).replace('torch.', '')}" for k, v in sd.items()])


def _tokenizer():
    from sam3.model.tokenizer_ve import SimpleTokenizer
    return SimpleTokenizer(bpe_path=REF_BPE)


def _text_student(backbone, ctx, table=None, resize=None, layers=None):
    import model as stage1_model  # /root/reference/stage1/model.py
    cfg = NS(MODEL=NS(BACKBONE=backbone), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=ctx, POS_EMBED_TABLE_SIZE=table or 0))
    if layers is None:
        m = stage1_model.build_text_student_model(cfg)
    else:   # the variant's cfg at reduced depth (stage1/model.py:61-96 table, TextStudentEncoder built directly)
        from sam3.model.text_encoder_student import TextStudentEncoder
        base = dict(context_length=table or ctx, vocab_size=49408, dim=512, ffn_multiplier_per_layer=4.0, n_heads_per_layer=8,
                    n_transformer_layers=12, norm_layer="layer_norm_fp32", causal_masking=False, model_name="base",
                    embed_dropout=0.0, no_scale_embedding=False, no_pos_embedding=False)
        base.update(layers)
        m = TextStudentEncoder(cfg=base, context_length=ctx, output_dim=256)
    if resize is not None:
        m.set_context_length(resize)
    return m.eval()


def gen_text_student(tag, backbone, ctx, seed_w, table=None, resize=None, layers=None):
    m = _text_student(backbone, ctx, table, resize, layers)
    m.load_state_dict(fill_state_dict(m.state_dict(), seed_w))
    mask, memory, embeds = m(TEXT_CAPTIONS, device="cpu")
    ids = m.tokenizer(TEXT_CAPTIONS, context_length=m.context_length)
    pooled = m.encoder(ids)
    cfg = {k: v for k, v in m.encoder.__dict__.items() if k in ("causal_masking", "model_dim")}
    path = os.path.join(HERE, f"{tag}.npz")
    np.savez_compressed(path, keys=keyshapes(m.state_dict()), ids=ids.numpy(), mask=mask.numpy(), memory=memory.numpy(),
                        embeds=embeds[:, :TEXT_EMBED_KEEP].numpy(), pooled=pooled.numpy(), seed_w=seed_w, ctx=m.context_length,
                        backbone=backbone, table=table or 0, resize=resize or 0, layers=np.array(repr(layers)), cfg=np.array(repr(cfg)))
    print(tag, "memory", tuple(memory.shape), "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


def gen_text_teacher(tag, seed_w, layers=2, ctx=32):
    from sam3.model.text_encoder_ve import VETextEncoder
    tok = _tokenizer()
    m = VETextEncoder(d_model=256, tokenizer=tok, width=1024, heads=16, layers=layers, context_length=ctx).eval()
    m.load_state_dict(fill_state_dict(m.state_dict(), seed_w))
    mask, memory, embeds = m(TEXT_CAPTIONS, device="cpu")
    path = os.path.join(HERE, f"{tag}.npz")
    np.savez_compressed(path, keys=keyshapes(m.state_dict()), ids=tok(TEXT_CAPTIONS, context_length=ctx).numpy(), mask=mask.numpy(),
                        memory=memory.numpy(), embeds=embeds[:, :TEXT_EMBED_KEEP].numpy(), seed_w=seed_w, ctx=ctx, layers=layers)
    print(tag, "memory", tuple(memory.shape), "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


def gen_text_tokens(tag="text_tokens"):
    tok = _tokenizer()
    path = os.path.join(HERE, f"{tag}.npz")
    np.savez_compressed(path, strings=np.array(TEXT_TOKEN_STRINGS), **{f"ids_{n}": tok(TEXT_TOKEN_STRINGS, context_length=n).numpy()
                                                                      for n in (16, 32, 77)})
    print(tag, len(TEXT_TOKEN_STRINGS), "strings ->", path)


def gen_bpe_subset(tag="text_bpe_subset"):
    """Runs the reference tokenizer's own pre-tokenisation (clean_fn, pat, byte_encoder) and replays its BPE loop on every word,
    recording each ranked pair that is adjacent at any step."""
    import regex
    tok = _tokenizer()
    used = {}
    for text in TEXT_TOKEN_STRINGS + OTHER_TEST_STRINGS:
        for piece in regex.findall(tok.pat, tok.clean_fn(text)):
            if piece in ("<start_of_text>", "<end_of_text>"):
                continue
            mapped = "".join(tok.byte_encoder[b] for b in piece.encode("utf-8"))
            word = list(mapped)
            word[-1] += "</w>"
            while len(word) > 1:
                ranked = [(tok.bpe_ranks[p], p) for p in zip(word, word[1:]) if p in tok.bpe_ranks]
                used.update({r: " ".join(p) for r, p in ranked})
                if not ranked:
                    break
                a, b = min(ranked)[1]
                merged, i = [], 0
                while i < len(word):
                    if i + 1 < len(word) and word[i] == a and word[i + 1] == b:
                        merged.append(a + b)
                        i += 2
                    else:
                        merged.append(word[i])
                        i += 1
                word = merged
            assert " ".join(word) == tok.bpe(mapped)       # the replay is the reference's own result
    rec = dict(source="bpe_simple_vocab_16e6.txt.gz (CLIP), merge lines 1..48894", n_merges=49152 - 256 - 2,
               merges={str(r): used[r] for r in sorted(used)})
    path = os.path.join(HERE, f"{tag}.json")
    with open(path, "w", encoding="utf-8") as f:
        json.dump(rec, f, ensure_ascii=True, indent=0, sort_keys=False)
    print(tag, len(used), "ranked pairs ->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


def main():
    gen_bpe_subset()
    gen_text_tokens()
    gen_text_student("text_s0_ctx32", "MobileCLIP-S0", 32, seed_w=101)
    gen_text_student("text_b_causal", "MobileCLIP-B", 32, seed_w=102, layers=dict(n_transformer_layers=2, causal_masking=True))
    gen_text_student("text_768", "MobileCLIP2-S3", 32, seed_w=103, layers=dict(dim=768, n_transformer_layers=2, n_heads_per_layer=12))
    gen_text_student("text_s0_interp", "MobileCLIP-S0", 32, seed_w=104, table=77)
    gen_text_student("text_s0_resize16", "MobileCLIP-S0", 77, seed_w=105, resize=16)
    gen_text_teacher("text_teacher", seed_w=106)


if __name__ == "__main__":
    main()
