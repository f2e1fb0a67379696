"""CPU: the pieces of native text-student training that need no GPU -- the text KD loss restated from the reference's formulas and
the analytic gradient the loss kernel implements (against torch autograd, including cosine_similarity's eps branch), the
reference's batch structures, the per-update LR timing, the word permutation and FlatAdamW's parameter exclusion."""
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_text_cpu import BPE


def ref_text_loss(preds, teacher, valid=None, cosine_weight=1.0):
    """train_text_encoder_stage1.py:230-242 with :336-370 restated: (loss, mse, cos) on [B, L, D]; valid [B, L] float or None."""
    sim = F.cosine_similarity(preds, teacher, dim=2)
    if valid is None:
        mse = F.mse_loss(preds, teacher)
        cos = (1.0 - sim).mean()
    else:
        n = valid.sum(dim=1).clamp(min=1.0)
        mse = (((preds - teacher) * valid.unsqueeze(-1)).square().sum(dim=(1, 2)) / (n * preds.size(2))).mean()
        cos = (((1.0 - sim) * valid).sum(dim=1) / n).mean()
    return mse + cosine_weight * cos, mse, cos


def kernel_formula_grad(p, t, valid, w):
    """The gradient es3_text_kd_loss_bwd evaluates (text_bwd.cu), in fp64 torch."""
    B, L, D = p.shape
    np_, nt = p.norm(dim=2, keepdim=True), t.norm(dim=2, keepdim=True)
    npc, ntc = np_.clamp_min(1e-8), nt.clamp_min(1e-8)
    dot = (p * t).sum(2, keepdim=True)
    dcos = t / (npc * ntc) - torch.where(np_ > 0, dot / (npc * npc * ntc * np_), torch.zeros_like(np_)) * p
    if valid is None:
        a_mse, a_cos, v = 2.0 / (B * L * D), w / (B * L), torch.ones(B, L, 1, dtype=p.dtype)
    else:
        n = valid.sum(1).clamp(min=1.0).view(B, 1, 1)
        a_mse, a_cos, v = 2.0 / (n * D * B), w / (n * B), valid.unsqueeze(-1)
    return v * (a_mse * (p - t) - a_cos * dcos)


@pytest.mark.parametrize("masked", [False, True])
def test_loss_gradient_formula_matches_autograd(masked):
    g = torch.Generator().manual_seed(1)
    p = torch.randn(3, 7, 16, generator=g, dtype=torch.float64)
    t = torch.randn(3, 7, 16, generator=g, dtype=torch.float64)
    t[0, 2] = 0.0                                         # all-zero teacher row: cos = 0, no gradient from the cosine term
    p[1, 4] *= 1e-10                                      # |p| below eps: the clamped-norm branch
    valid = torch.ones(3, 7, dtype=torch.float64)
    valid[1, 5:] = 0.0
    valid[2] = 0.0
    pr = p.clone().requires_grad_(True)
    loss, _, cos = ref_text_loss(pr, t, valid if masked else None, 0.6)
    loss.backward()
    got = kernel_formula_grad(p, t, valid if masked else None, 0.6)
    assert torch.allclose(got, pr.grad, rtol=1e-9, atol=1e-12 * pr.grad.abs().max().item())


def test_parse_text_batch_structures():
    from efficientsam3_b200.stage1.train import parse_text_batch
    e = [np.zeros((4, 2), np.float16), np.ones((4, 2), np.float16)]
    caps, emb, seeds = parse_text_batch([["a cat", "a dog"], [e, [1, 2]]])
    assert caps == ["a cat", "a dog"] and emb is e and list(seeds) == [1, 2]
    # three items: a list of exactly two (caption, ...) tuples matches the first structure, in the reference as here (:198)
    caps, emb, seeds = parse_text_batch([("a cat", (e[0], 1)), ("a dog", (e[1], 2)), ("a cow", (e[0], 3))])
    assert caps == ["a cat", "a dog", "a cow"] and emb[1] is e[1] and seeds == [1, 2, 3]
    for bad in ({"text": ["a"]}, [], [["a cat"]], (["a cat"], [e, [1]]), [[1, 2], [e, [1, 2]]]):
        with pytest.raises(ValueError, match="Unexpected batch structure"):
            parse_text_batch(bad)


def test_lr_per_update_follows_reference_scheduler_timing():
    from efficientsam3_b200.stage1.train import lr_for_update

    def lr_at(t):
        return 1.0 + t                                    # any injective schedule shows the timing

    for num_steps, accum in ((7, 1), (7, 2), (8, 3)):
        current = lr_at(0)                                # the scheduler's value before the first step_update
        for epoch in range(3):
            for idx in range(num_steps):
                if (idx + 1) % accum == 0:                # the reference: step with the current LR, then step_update
                    assert lr_for_update(idx, epoch, num_steps, accum, lr_at) == current, (num_steps, accum, epoch, idx)
                    current = lr_at((epoch * num_steps + idx) // accum)


def test_permute_words_draws_from_global_random():
    from efficientsam3_b200.stage1.losses import permute_words
    caps = ["a red car on the road", "cat", "two dogs playing"]
    random.seed(123)
    got = [permute_words(s) for s in caps]
    random.seed(123)
    want = []
    for s in caps:
        w = s.split()
        if len(w) > 1:
            random.shuffle(w)
        want.append(" ".join(w))
    assert got == want and got[1] == "cat"
    assert sorted(got[0].split()) == sorted(caps[0].split())


def test_flat_adamw_excludes_projection_layer():
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    from efficientsam3_b200.stage1.optim import FlatAdamW
    cfg = text_student_cfg("MobileCLIP-S1")
    cfg.update(n_transformer_layers=1, context_length=16)
    m = TextStudentEncoder(cfg=cfg, context_length=16, output_dim=256, bpe_path=BPE)
    proj = m.encoder.projection_layer.detach().clone()
    opt = FlatAdamW(m, lr=1e-3, exclude=TextStudentEncoder.UNUSED_PARAMETERS)
    assert "encoder.projection_layer" not in opt.names
    assert len(opt.names) == len(list(m.parameters())) - 1
    assert m.encoder.projection_layer.grad is None and torch.equal(m.encoder.projection_layer.detach(), proj)
    assert m._es3_grad_arena is opt                       # the native backward may write the arena directly
    assert all(p.grad is not None for n, p in m.named_parameters() if n != "encoder.projection_layer")
    assert sorted(n for n, _ in m.named_parameters() if n not in opt.names) == ["encoder.projection_layer"]
    trainable = {id(p) for p in m.trainable_parameters()}
    assert sorted(n for n, p in m.named_parameters() if id(p) in trainable) == sorted(opt.names)
    with pytest.raises(ValueError, match="no parameter named"):
        FlatAdamW(m, lr=1e-3, exclude=("encoder.nope",))
    plain = FlatAdamW(TextStudentEncoder(cfg=cfg, context_length=16, output_dim=256, bpe_path=BPE), lr=1e-3)
    assert "encoder.projection_layer" in plain.names     # the default leaves every parameter in (existing callers unchanged)


def test_train_text_one_epoch_rejects_unknown_batch_structure():
    from efficientsam3_b200.stage1.train import train_text_one_epoch

    class Opt:
        lr = base_lr = 1e-3

        def zero_grad(self):
            pass

    cfg = NS(TRAIN=NS(ACCUMULATION_STEPS=1, EPOCHS=1, WARMUP_EPOCHS=0, MIN_LR=0.0, WARMUP_LR=0.0, CLIP_GRAD=5.0),
             DISTILL=NS(NUM_EMBED=16, EMBED_DIM=256, COSINE=1.0))
    model = torch.nn.Linear(2, 2)
    with pytest.raises(ValueError, match="Unexpected batch structure"):
        train_text_one_epoch(cfg, model, [{"bad": 1}], Opt(), 0)


# ------------------------------------------------------------------------------------------------ reference training fixtures
TRAIN_FIXTURES = ["text_train_s1", "text_train_b_causal", "text_train_768"]


def build_train_student(g):
    """The native TextStudentEncoder of a text_train_* fixture (tests/golden/gen_golden_text_train.py), weights loaded."""
    from efficientsam3_b200.model.text_encoder_student import TextStudentEncoder
    from efficientsam3_b200.stage1.model import text_student_cfg
    from oracle.weights import fill_state_dict
    ctx, table = int(g["ctx"]), int(g["table"])
    cfg = text_student_cfg(str(g["backbone"]))
    cfg.update(eval(str(g["layers"])), context_length=table or ctx)
    m = TextStudentEncoder(cfg=cfg, context_length=ctx, output_dim=256, bpe_path=BPE)
    sd = fill_state_dict(m.state_dict(), int(g["seed_w"]))
    m.load_state_dict(sd)
    return m, sd


def fixture_permutations(g):
    """The permuted captions as the step draws them: random.seed(seed_p), then permute_words per caption, once per consistency block."""
    from efficientsam3_b200.stage1.losses import permute_words
    from test_text_cpu import OT_CAPTIONS
    caps = OT_CAPTIONS()
    random.seed(int(g["seed_p"]))
    return caps, [[permute_words(s) for s in caps] for _ in range(g["perm_ids"].shape[0])]


def oracle_train_grads(g, sd0, m, device="cpu", dtype=torch.float32):
    """The fixture's iteration on the oracle (oracle/text.py) with ref_text_loss: (loss terms, {name: grad})."""
    from oracle import text as OT
    from test_text_cpu import oracle_cfg
    sd = {k: v.detach().clone().to(device, dtype).requires_grad_(True) for k, v in sd0.items()}
    cfg = oracle_cfg(m)
    ids = torch.from_numpy(g["ids"]).to(device)
    teacher = torch.from_numpy(g["teacher"]).float().to(device, dtype)
    preds = OT.text_student(sd, ids, cfg)[1].transpose(0, 1)
    valid = (ids != 0).to(dtype) if int(g["masked"]) else None
    loss, mse, cos = ref_text_loss(preds, teacher, valid, float(g["cosine"]))
    cons = []
    for pid in g["perm_ids"]:
        q = OT.text_student(sd, torch.from_numpy(pid).to(device), cfg)[1].transpose(0, 1)
        c = F.mse_loss(preds.mean(1), q.mean(1))
        loss = loss + float(g["consistency"]) * c
        cons.append(c.item())
    loss.backward()
    terms = [loss.item(), mse.item(), cos.item(), *cons] + [0.0] * (2 - len(cons))
    return terms, {k: v.grad for k, v in sd.items()}


def grad_stats(gr):
    gr = gr.reshape(-1).double()
    first = torch.zeros(4, dtype=torch.float64)
    first[:min(4, gr.numel())] = gr[:4]
    return torch.cat([gr.norm().reshape(1), gr.sum().reshape(1), first])


@pytest.mark.parametrize("name", TRAIN_FIXTURES)
def test_train_fixture_ids_permutations_and_keys(name):
    from helpers import load_golden
    from test_text_cpu import sig
    g = load_golden(name)
    m, _ = build_train_student(g)
    assert sig(m.state_dict()) == [str(k) for k in g["keys"]]
    caps, perms = fixture_permutations(g)
    assert torch.equal(m.tokenizer(caps, context_length=m.context_length), torch.from_numpy(g["ids"]))
    assert torch.equal(torch.from_numpy(g["pad"]), torch.from_numpy(g["ids"]) == 0)
    assert [list(p) for p in perms] == [[str(s) for s in row] for row in g["perm_strings"]]
    for p, pid in zip(perms, g["perm_ids"]):
        assert torch.equal(m.tokenizer(p, context_length=m.context_length), torch.from_numpy(pid))


@pytest.mark.parametrize("name", TRAIN_FIXTURES)
def test_train_fixture_oracle_loss_and_gradients(name):
    """The oracle's autograd and the loss restatement against the reference's own train-mode iteration: loss terms rtol 1e-5;
    every gradient statistic within 1e-4 of that parameter's gradient norm."""
    from helpers import load_golden
    g = load_golden(name)
    m, sd = build_train_student(g)
    terms, grads = oracle_train_grads(g, sd, m)
    ref_terms = g["loss"]
    for a, b in zip(terms, ref_terms):
        assert abs(a - b) <= 1e-5 * max(abs(b), 1e-12), (terms, ref_terms.tolist())
    names = [str(n) for n in g["grad_names"]]
    assert names == [n for n, _ in m.named_parameters() if n != "encoder.projection_layer"]
    assert grads["encoder.projection_layer"] is None
    for n, ref in zip(names, g["grad_stats"]):
        got = grad_stats(grads[n]).numpy()
        err = np.abs(got - ref).max() / ref[0]
        assert err <= 1e-4, (n, err)
