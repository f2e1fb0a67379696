"""GPU: training the MobileCLIP base text students natively -- the text KD loss's composition against torch fp32 autograd, whole
training graphs against the oracle's fp32 autograd (with the bf16-autocast oracle as the precision yardstick), the train-mode
forward against the eval fixtures, the optimiser interplay (arena, exclusion, accumulation, determinism) and the raise paths."""
import random

import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden, max_err_over_scale, rel_l2
from oracle import text as OT
from oracle.weights import fill_state_dict
from test_text_cpu import BPE, oracle_cfg
from test_text_gpu import captions, check_memory, loaded_student
from test_text_train_cpu import ref_text_loss

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernels vs torch fp32
@pytest.mark.parametrize("masked", [False, True])
def test_text_kd_loss_kernels(cuda, masked):
    from efficientsam3_b200.stage1.losses import TextKDLossFunction, text_kd_loss
    g = torch.Generator().manual_seed(11 + masked)
    B, L, D = 5, 32, 256
    p = torch.randn(B, L, D, generator=g).to(cuda)
    t = torch.randn(B, L, D, generator=g).to(cuda)
    t[1, 3] = 0.0                                               # all-zero teacher row: the eps branch of cosine_similarity
    pad = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        pad[b, 4 + 5 * b:] = True
    pad[4] = True                                               # a sample without a valid token: denominator clamp(., 1)
    pad = pad.to(cuda)
    qs = [torch.randn(B, L, D, generator=g).to(cuda) for _ in range(2)]
    w_cos, w_con = 0.7, 0.3
    loss, mse, cos = text_kd_loss(p, t, pad if masked else None, w_cos)
    pr = p.clone().requires_grad_(True)
    qr = [q.clone().requires_grad_(True) for q in qs]
    ref, ref_mse, ref_cos = ref_text_loss(pr, t, (~pad).float() if masked else None, w_cos)
    for a, b_ in ((loss, ref), (mse, ref_mse), (cos, ref_cos)):
        assert abs(a.item() - b_.item()) <= 1e-4 * abs(b_.item()), (a.item(), b_.item())
    total = ref + sum(w_con * F.mse_loss(pr.mean(1), q.mean(1)) for q in qr)
    total.backward(torch.tensor(3.0, device=cuda))
    pn = p.clone().requires_grad_(True)
    qn = [q.clone().requires_grad_(True) for q in qs]
    got, _, _, cons = TextKDLossFunction.apply(pn, t, pad if masked else None, w_cos, w_con, *qn)
    assert abs(got.item() - total.item()) <= 1e-4 * abs(total.item())
    for c, q in zip(cons, qs):
        r = F.mse_loss(p.mean(1), q.mean(1)).item()
        assert abs(c.item() - r) <= 1e-4 * r
    got.backward(torch.tensor(3.0, device=cuda))
    assert max_err_over_scale(pn.grad.cpu(), pr.grad.cpu()) <= 2e-3
    for a, b_ in zip(qn, qr):
        assert max_err_over_scale(a.grad.cpu(), b_.grad.cpu()) <= 2e-3


# ------------------------------------------------------------------------------------------------ whole graphs vs the oracle
def _student(backbone, dev, layers=None, ctx=32, table=None, seed=21):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    cfg = text_student_cfg(backbone)
    if layers is not None:
        cfg["n_transformer_layers"] = layers
    cfg["context_length"] = table or ctx
    m = TextStudentEncoder(cfg=cfg, context_length=ctx, output_dim=256, bpe_path=BPE)
    sd = fill_state_dict(m.state_dict(), seed)
    m.load_state_dict(sd)
    return m.to(dev), sd


def _permuted(caps, seed):
    from efficientsam3_b200.stage1.losses import permute_words
    random.seed(seed)
    return [[permute_words(s) for s in caps] for _ in range(2)]


def _oracle_grads(sd0, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev, autocast=None):
    import contextlib
    sd = {k: v.detach().clone().to(dev).requires_grad_(True) for k, v in sd0.items()}
    cfg = oracle_cfg(m)
    ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else contextlib.nullcontext()
    with ctx:
        preds = OT.text_student(sd, ids.to(dev), cfg)[1].transpose(0, 1)
        perms = [OT.text_student(sd, q.to(dev), cfg)[1].transpose(0, 1) for q in perm_ids]
    preds, perms = preds.float(), [q.float() for q in perms]
    loss, _, _ = ref_text_loss(preds, teacher, valid, w_cos)
    for q in perms:
        loss = loss + w_con * F.mse_loss(preds.mean(1), q.mean(1))
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in sd.items()}


def _native_grads(m, caps, perm_caps, teacher, masked, w_cos, w_con):
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    m.train()
    m.zero_grad(set_to_none=True)
    pad, mem, _ = m(caps)
    perms = [m(pc)[1].transpose(0, 1) for pc in perm_caps]
    loss, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if masked else None, w_cos, w_con, *perms)
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in m.named_parameters()}


def _all_grad_rel(got, ref, names):
    num = sum((got[n].double().cpu() - ref[n].double().cpu()).pow(2).sum().item() for n in names)
    den = sum(ref[n].double().cpu().pow(2).sum().item() for n in names)
    return (num / den) ** 0.5


def _compare_to_oracle(m, sd, caps, masked, w_con, dev, label):
    w_cos = 1.0
    ids = m.tokenizer(caps, context_length=m.context_length)
    perm_caps = _permuted(caps, 5) if w_con > 0 else []
    perm_ids = [m.tokenizer(pc, context_length=m.context_length) for pc in perm_caps]
    teacher = torch.randn(len(caps), m.context_length, 256, generator=torch.Generator().manual_seed(9)).to(dev)
    valid = (ids != 0).float().to(dev) if masked else None
    loss_n, got = _native_grads(m, caps, perm_caps, teacher, masked, w_cos, w_con)
    loss_r, ref = _oracle_grads(sd, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev)
    _, ref_bf = _oracle_grads(sd, m, ids, perm_ids, teacher, valid, w_cos, w_con, dev, autocast=torch.bfloat16)
    assert got["encoder.projection_layer"] is None and ref["encoder.projection_layer"] is None
    names = [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    rel = _all_grad_rel(got, ref, names)
    d_bf16 = _all_grad_rel(ref_bf, ref, names)
    print(f"  {label}: loss native {loss_n.item():.6f} oracle {loss_r.item():.6f}; all-gradient rel-L2 native {rel:.3e}, "
          f"torch.autocast(bf16) oracle {d_bf16:.3e}")
    assert abs(loss_n.item() - loss_r.item()) <= 2e-2 * abs(loss_r.item())
    assert rel <= 5e-2 and rel <= 3 * d_bf16, (rel, d_bf16)
    return got


def test_s1_shaped_depth2_masked_consistency(cuda):
    m, sd = _student("MobileCLIP-S1", cuda, layers=2, ctx=32)
    _compare_to_oracle(m, sd, captions(), masked=True, w_con=0.5, dev=cuda, label="S1-shaped depth 2, masked + consistency")


def test_b_causal_depth2_unmasked(cuda):
    m, sd = _student("MobileCLIP-B", cuda, layers=2, ctx=32, seed=22)
    _compare_to_oracle(m, sd, captions(), masked=False, w_con=0.0, dev=cuda, label="MobileCLIP-B depth 2, causal, unmasked")


def test_768_table77_at_32_positional_resize(cuda):
    m, sd = _student("MobileCLIP2-L", cuda, layers=2, ctx=32, table=77, seed=23)
    got = _compare_to_oracle(m, sd, captions(), masked=True, w_con=0.0, dev=cuda, label="768-wide depth 2, table 77 at 32")
    assert got["encoder.positional_embedding.pos_embed.pos_embed"].abs().sum().item() > 0


@pytest.mark.parametrize("backbone", ["MobileCLIP2-L", "MobileCLIP-B"])
def test_full_depth_vs_oracle(cuda, backbone):
    m, sd = _student(backbone, cuda, ctx=32, seed=24)
    _compare_to_oracle(m, sd, captions(), masked=True, w_con=0.0, dev=cuda, label=f"{backbone} 12 layers")


@pytest.mark.parametrize("name", ["text_b_causal", "text_768"])
def test_train_mode_memory_matches_eval_fixture(cuda, name):
    g = load_golden(name)
    m = loaded_student(g, cuda).train()
    mask, mem, emb = m(captions())
    assert mem.grad_fn is not None and not emb.requires_grad
    assert torch.equal(mask.cpu(), torch.from_numpy(g["mask"]))
    check_memory(mem.detach(), torch.from_numpy(g["memory"]))
    with torch.no_grad():                                       # train mode under no_grad: the eval path
        _, mem_ng, _ = m(captions())
    assert mem_ng.grad_fn is None
    check_memory(mem_ng, torch.from_numpy(g["memory"]))


# ------------------------------------------------------------------------------------------------ optimiser interplay
def _cfg_ns(backbone="MobileCLIP-S1", ctx=16):
    from types import SimpleNamespace as NS
    return NS(MODEL=NS(BACKBONE=backbone, BPE_PATH=BPE), DISTILL=NS(EMBED_DIM=256, CONTEXT_LENGTH=ctx))


def _steps(seed, n=3, dev="cuda"):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    m, _ = _student("MobileCLIP-S1", dev, layers=2, ctx=16, seed=seed)
    m.train()
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(seed)).to(dev)
    proj0 = m.encoder.projection_layer.detach().clone()
    random.seed(seed)
    losses = [text_kd_train_step(m, opt, caps, teacher, cosine_weight=1.0, mask_pad_tokens=True, consistency_weight=0.5,
                                 clip_grad=5.0, lr=1e-3).item() for _ in range(n)]
    return m, opt, losses, proj0


def test_seeded_steps_bit_identical_projection_untouched(cuda):
    m1, opt1, l1, proj0 = _steps(31)
    m2, _, l2, _ = _steps(31)
    print(f"  3 steps: losses {l1}")
    assert l1 == l2 and l1[-1] < l1[0]
    for (n, a), (_, b) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(a, b), n
    assert torch.equal(m1.encoder.projection_layer.detach(), proj0)
    assert m1.encoder.projection_layer.grad is None
    assert "encoder.projection_layer" not in opt1.names
    assert m1._es3_grad_arena is opt1


def test_direct_arena_grads_equal_autograd_grads_and_accumulation(cuda):
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    from efficientsam3_b200.stage1.optim import FlatAdamW
    caps = captions()
    teacher = torch.randn(len(caps), 16, 256, generator=torch.Generator().manual_seed(2)).to(cuda)

    def backward(m, text):
        pad, mem, _ = m(text)
        loss, _, _, _ = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad, 1.0, 0.0)
        loss.backward()

    m, _ = _student("MobileCLIP-S1", cuda, layers=2, ctx=16, seed=41)
    m.train()
    backward(m, caps)
    auto = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    backward(m, caps[::-1])
    auto2 = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    md, _ = _student("MobileCLIP-S1", cuda, layers=2, ctx=16, seed=41)
    md.train()
    opt = FlatAdamW(md, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    backward(md, caps)
    for n, p in md.named_parameters():
        if n in auto:
            assert torch.equal(p.grad, auto[n]), n
    backward(md, caps[::-1])                                    # a second micro-batch adds into the arena
    for n, p in md.named_parameters():
        if n in auto:
            r = rel_l2(p.grad.cpu(), (auto[n] + auto2[n]).cpu())
            assert r <= 1e-6, (n, r)
    assert md.encoder.projection_layer.grad is None and opt.flat_grad.numel() > 0


def test_raise_paths_train(cuda):
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.model import build_text_student_model
    s0 = build_text_student_model(_cfg_ns("MobileCLIP-S0", 32)).to(cuda).train()
    with pytest.raises(NotImplementedError, match=r"RepMixerBlocks.*Call \.eval\(\) first\."):
        s0(["a cat"])
    with torch.no_grad(), pytest.raises(NotImplementedError, match="RepMixerBlocks"):
        s0(["a cat"])
    m = build_text_student_model(_cfg_ns("MobileCLIP-S1", 32)).to(cuda).train()
    with pytest.raises(NotImplementedError, match="strict"):
        with ops.strict_precision():
            m(["a cat"])
    pad, mem, _ = m(["a cat", "a dog on a mat"])
    mem.sum().backward()
    with pytest.raises(RuntimeError, match="ONE backward"):
        mem.sum().backward()
    long = build_text_student_model(_cfg_ns("MobileCLIP-S1", 160)).to(cuda).train()
    n0 = ops.launch_count
    with pytest.raises(ValueError, match="1..128"):
        long(["a cat"])
    bad = torch.zeros(2, 32, dtype=torch.long)
    bad[1, 3] = 49408
    with pytest.raises(ValueError, match="out of range"):
        m(bad)
    assert ops.launch_count == n0
    with pytest.raises(ValueError, match="1..128"):
        ops.text_attn_bwd(*(torch.zeros(1, 1, device=cuda, dtype=torch.bfloat16),) * 3, 1, 129, 512, 8, 0.125, False)
    drop = build_text_student_model(_cfg_ns("MobileCLIP-S1", 32)).to(cuda).train()
    drop.encoder.transformer[0].pre_norm_ffn[3].p = 0.1
    with pytest.raises(NotImplementedError, match="dropout"):
        drop(["a cat"])


# ------------------------------------------------------------------------------------------------ reference training fixtures
@pytest.mark.parametrize("name", ["text_train_s1", "text_train_b_causal", "text_train_768"])
def test_train_fixture_end_to_end_from_strings(cuda, name):
    """The reference's own train-mode iteration (tests/golden/gen_golden_text_train.py) natively from strings: permuted captions
    drawn by permute_words after the fixture's seed, loss terms, and every parameter's gradient statistics (all-gradient rel-L2 of
    the recorded entries and norms)."""
    from efficientsam3_b200.stage1.losses import TextKDLossFunction
    from test_text_train_cpu import build_train_student, fixture_permutations, grad_stats
    g = load_golden(name)
    m, _ = build_train_student(g)
    m = m.to(cuda).train()
    caps, perms = fixture_permutations(g)
    assert [list(p) for p in perms] == [[str(s) for s in row] for row in g["perm_strings"]]
    teacher = torch.from_numpy(g["teacher"]).float().to(cuda)
    pad, mem, _ = m(caps)
    assert torch.equal(pad.cpu(), torch.from_numpy(g["pad"]))
    qs = [m(p)[1].transpose(0, 1) for p in perms]
    loss, mse, cos, cons = TextKDLossFunction.apply(mem.transpose(0, 1), teacher, pad if int(g["masked"]) else None,
                                                    float(g["cosine"]), float(g["consistency"]), *qs)
    loss.backward()
    got_terms = [loss.item(), mse.item(), cos.item(), *cons.tolist()] + [0.0] * (2 - cons.numel())
    for a, b in zip(got_terms[:3], g["loss"][:3]):
        assert abs(a - b) <= 1e-2 * abs(b), (got_terms, g["loss"].tolist())
    # a consistency term is mse(mean_L(p) - mean_L(q)): a small difference of two pooled vectors, so its error follows the pooled
    # vectors' scale s, not its own size: |d c| <= 2 sqrt(c) e + e^2 with e = 1e-2 s (the bf16 output tolerance on that scale)
    e = 1e-2 * mem.detach().transpose(0, 1).mean(1).pow(2).mean().sqrt().item()
    for a, b in zip(got_terms[3:], g["loss"][3:]):
        assert abs(a - b) <= 2 * abs(b) ** 0.5 * e + e * e, (got_terms, g["loss"].tolist(), e)
    params = dict(m.named_parameters())
    got = torch.stack([grad_stats(params[str(n)].grad.cpu()) for n in g["grad_names"]])
    ref = torch.from_numpy(g["grad_stats"])
    r = rel_l2(got, ref)
    print(f"  {name}: loss native {got_terms[0]:.6f} reference {g['loss'][0]:.6f}; gradient statistics rel-L2 {r:.3e}")
    assert r <= 5e-2, r
    assert params["encoder.projection_layer"].grad is None


def test_train_text_one_epoch_matches_the_steps_it_composes(cuda):
    """train_text_one_epoch over the reference's two batch structures (fp16 stored embeddings, accumulation 2, masked loss, COSINE,
    CONSISTENCY_LOSS, the cosine LR schedule per update) gives bit-identically the parameters of the same text_kd_train_step
    sequence called by hand with the upcast embeddings and lr_for_update."""
    import numpy as np
    from types import SimpleNamespace as NS
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.losses import text_kd_train_step
    from efficientsam3_b200.stage1.optim import FlatAdamW
    from efficientsam3_b200.stage1.train import default_lr_at, lr_for_update, train_text_one_epoch
    cfg = NS(TRAIN=NS(ACCUMULATION_STEPS=2, EPOCHS=3, WARMUP_EPOCHS=1, MIN_LR=1e-5, WARMUP_LR=1e-6, CLIP_GRAD=5.0),
             DISTILL=NS(NUM_EMBED=16, EMBED_DIM=256, MASK_PAD_TOKENS=True, COSINE=2.0, CONSISTENCY_LOSS=0.05))
    caps = captions()
    g = np.random.default_rng(0)
    embs = [[(g.standard_normal(16 * 256) * 0.5).astype(np.float16) for _ in caps] for _ in range(4)]
    loader = []
    for i, e in enumerate(embs):
        if i % 2 == 0:
            loader.append([list(caps), [e, list(range(len(caps)))]])                        # default-collated structure
        else:
            loader.append([(c, (x, k)) for k, (c, x) in enumerate(zip(caps, e))])          # list of (caption, (embedding, seed))
    m1, _ = _student("MobileCLIP-S1", cuda, layers=2, ctx=16, seed=51)
    m2, _ = _student("MobileCLIP-S1", cuda, layers=2, ctx=16, seed=51)
    o1 = FlatAdamW(m1, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    o2 = FlatAdamW(m2, lr=2e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    random.seed(7)
    losses = train_text_one_epoch(cfg, m1, loader, o1, epoch=1)
    m2.train()
    lr_at = default_lr_at(cfg, o2, len(loader))
    random.seed(7)
    want = []
    for idx, e in enumerate(embs):
        t = torch.from_numpy(np.stack(e)).float().view(len(caps), 16, 256).to(cuda)
        update = (idx + 1) % 2 == 0
        want.append(text_kd_train_step(m2, o2, caps, t, cosine_weight=2.0, mask_pad_tokens=True, consistency_weight=0.05,
                                       clip_grad=5.0, lr=lr_for_update(idx, 1, len(loader), 2, lr_at) if update else None,
                                       accumulation_steps=2, update=update))
    assert [x.item() for x in losses] == [x.item() for x in want]
    # updates at iterations 1 and 3 of epoch 1 run at lr_at(1) and lr_at(2) (the value the previous update's step_update left)
    assert o1.lr == o2.lr == lr_at(2) and o1.step_count() == 2
    for (n, a), (_, b) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(a, b), n
