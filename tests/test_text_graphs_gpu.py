"""GPU: CUDA-graph replay of the text encoders' eval forward (enable_cuda_graphs on TextStudentEncoder,
MobileCLIPTextTransformer, VETextEncoder and SAM3TextTeacherEncoder).  Replay is bit-identical to the host-launched kernel
sequence; graphs are keyed by shape and captured again when parameters, buffers or plans move; the paths that are never
replayed (training, batch-statistics BatchNorm, strict precision, host-side rejection) behave exactly as with graphs off; the
text dump writes the same bytes."""
import os

import pytest
import torch

from helpers import load_golden
from oracle.weights import fill_state_dict
from test_text_cpu import BPE, build_student

pytestmark = pytest.mark.gpu

GRAPH_FIXTURES = ["text_s0_ctx32", "text_s0_resize16", "text_b_causal", "text_768"]


def captions():
    return [str(s) for s in load_golden("text_tokens")["strings"][:6]]


@pytest.fixture
def student(cuda):
    """A loaded student of one fixture: student(name) -> eval-mode TextStudentEncoder on the GPU."""
    def make(name="text_s0_ctx32", seed=None):
        g = load_golden(name)
        m = build_student(g)
        m.load_state_dict(fill_state_dict(m.state_dict(), int(g["seed_w"]) if seed is None else seed))
        return m.to(cuda).eval()
    return make


@pytest.fixture
def teacher(cuda):
    """teacher(ctx, layers) -> SAM3TextTeacherEncoder on the GPU (layers=None: the full 24-layer encoder)."""
    def make(ctx=32, layers=2, seed=106):
        from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
        t = SAM3TextTeacherEncoder(context_length=ctx, bpe_path=BPE, ve_overrides=None if layers is None else dict(layers=layers))
        ve = t.sam3.backbone.language_backbone
        ve.load_state_dict(fill_state_dict(ve.state_dict(), seed))
        return t.to(cuda)
    return make


def snap(out):
    return tuple(t.clone() for t in out) if isinstance(out, tuple) else out.clone()


def same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ bit-identical replay
@pytest.mark.parametrize("name", GRAPH_FIXTURES)
def test_student_replay_is_bit_identical(cuda, student, name):
    m = student(name)
    caps = captions()
    ids = m.tokenizer(caps, context_length=m.context_length)
    ref_str, ref_ids = snap(m(caps, device=cuda)), snap(m(ids.to(cuda)))
    m.enable_cuda_graphs()
    for _ in range(3):
        got = m(caps, device=cuda)
        assert same(got, ref_str)                                   # mask, memory and input_embeds
        assert got[0].is_cuda and got[1].shape == ref_str[1].shape
        assert same(m(ids.to(cuda)), ref_ids)
        assert same(m(ids), ref_ids)                                # host ids
    assert len(m._graphs) == 1 and m.graph_launches_per_step > 0
    assert same(m.forward_uncaptured(caps, device=cuda), ref_str)


@pytest.mark.parametrize("name", GRAPH_FIXTURES)
def test_text_transformer_replay_is_bit_identical(cuda, student, name):
    """MobileCLIPTextTransformer: pooled projection and all tokens, from ids and from embeddings."""
    m = student(name)
    enc = m.encoder
    ids = m.tokenizer(captions(), context_length=m.context_length)
    emb = m(ids)[2].transpose(0, 1).contiguous()                    # input_embeds [B, L, dim]
    calls = [dict(text_tokens=ids), dict(text_tokens=ids, return_all_tokens=True),
             dict(text_tokens=emb, input_is_embeddings=True), dict(text_tokens=emb, input_is_embeddings=True, return_all_tokens=True)]
    refs = [enc(**kw).clone() for kw in calls]
    enc.enable_cuda_graphs()
    for _ in range(2):
        for kw, ref in zip(calls, refs):
            assert torch.equal(enc(**kw), ref), kw
    assert len(enc._graphs) == 4 and enc.graph_launches_per_step > 0
    other = (emb * 0.5).contiguous()                               # new contents: replay copies the input in, it does not keep it
    assert torch.equal(enc(other, input_is_embeddings=True), enc.forward_uncaptured(other, input_is_embeddings=True))


@pytest.mark.parametrize("ctx,layers", [(32, 2), (16, None)])
def test_teacher_replay_is_bit_identical(cuda, teacher, ctx, layers):
    """The 2-layer teacher of the text_teacher fixture and the full-depth 24-layer teacher at ctx 16."""
    if layers == 2:
        g = load_golden("text_teacher")
        t = teacher(ctx=int(g["ctx"]), layers=int(g["layers"]), seed=int(g["seed_w"]))
    else:
        t = teacher(ctx=ctx, layers=None, seed=7)
    ve = t.sam3.backbone.language_backbone
    caps = captions()
    ids = ve.tokenizer(caps, context_length=ve.context_length)
    ref_str, ref_ids, ref_t = snap(ve(caps, device=cuda)), snap(ve(ids)), t(caps, device=cuda).clone()
    t.enable_cuda_graphs()
    for _ in range(3):
        assert same(ve(caps, device=cuda), ref_str)
        assert same(ve(ids.to(cuda)), ref_ids)
        assert torch.equal(t(caps, device=cuda), ref_t)
    assert len(ve._graphs) == 1 and t.graph_launches_per_step > 0
    assert torch.equal(t.forward_uncaptured(caps, device=cuda), ref_t)


# ------------------------------------------------------------------------------------------------ shapes and eviction
def test_shapes_alternate_and_the_oldest_graph_is_evicted(cuda, student):
    m = student("text_s0_ctx32")
    ids = m.tokenizer(captions(), context_length=32)
    a, b, c = ids[:4], ids[:3, :16].contiguous(), ids[:5]
    refs = [snap(m(x)) for x in (a, b, c)]
    m.enable_cuda_graphs(max_graphs=2)
    for _ in range(3):
        assert same(m(a), refs[0])
        assert same(m(b), refs[1])
    assert set(m._graphs) == {(4, 32, "ids", True, cuda), (3, 16, "ids", True, cuda)} and m.graph_launches_per_step > 0
    assert same(m(c), refs[2])                                       # a third shape: the oldest (a) goes
    assert set(m._graphs) == {(3, 16, "ids", True, cuda), (5, 32, "ids", True, cuda)}
    assert same(m(a), refs[0])


# ------------------------------------------------------------------------------------------------ re-capture
def test_parameter_update_and_load_state_dict_recapture(cuda, student):
    m = student("text_b_causal")
    caps = captions()
    m.enable_cuda_graphs()
    stale = snap(m(caps, device=cuda))
    with torch.no_grad():
        m.projector.bias.add_(1.0)                                  # in place: the parameter's version moves
    got = snap(m(caps, device=cuda))
    assert same(got, m.forward_uncaptured(caps, device=cuda)) and not torch.equal(got[1], stale[1])
    m.load_state_dict(fill_state_dict(m.state_dict(), 1234))
    got2 = snap(m(caps, device=cuda))
    assert same(got2, m.forward_uncaptured(caps, device=cuda)) and not torch.equal(got2[1], got[1])
    assert not torch.equal(got2[2], got[2])                          # the token table moved too: new input_embeds


def test_set_context_length_recaptures(cuda, student):
    """A ctx-32 student fed 16-token ids interpolates its 32-entry positional table; after set_context_length(16) the table is a
    new, truncated Parameter and the same 16-token key is captured again."""
    m = student("text_s0_ctx32")
    assert m.encoder.positional_embedding.pos_embed.num_embeddings == 32
    ids = m.tokenizer(captions(), context_length=16)
    m.enable_cuda_graphs()
    stale = snap(m(ids))
    m.set_context_length(16)
    got = snap(m(ids))
    assert same(got, m.forward_uncaptured(ids)) and not torch.equal(got[1], stale[1])
    assert same(m(captions(), device=cuda), m.forward_uncaptured(captions(), device=cuda))


def test_plan_invalidation_recaptures(cuda, student):
    """FlatAdamW's step writes the parameters through their pointers (their versions stay) and drops the packed plans: the graph
    is captured again rather than replayed on the old packing."""
    m = student("text_s0_ctx32")
    ids = m.tokenizer(captions(), context_length=32)
    m.enable_cuda_graphs()
    stale = snap(m(ids))
    m.projector.bias.data.add_(1.0)                                  # .data: the parameter's version does not move
    for mod in m.modules():                                          # what FlatAdamW.step does after its kernel
        if hasattr(mod, "_plan_key"):
            mod._plan_key = None
    got = snap(m(ids))
    assert same(got, m.forward_uncaptured(ids)) and not torch.equal(got[1], stale[1])


# ------------------------------------------------------------------------------------------------ host rejection and unchanged paths
def test_out_of_range_ids_are_rejected_on_the_host(cuda, student, teacher):
    from efficientsam3_b200 import ops
    m = student("text_s0_ctx32").enable_cuda_graphs()
    m.encoder.enable_cuda_graphs()
    ve = teacher().sam3.backbone.language_backbone.enable_cuda_graphs()
    bad = torch.zeros(2, 32, dtype=torch.long)
    bad[1, 3] = 49408
    n0 = ops.launch_count
    for call in (lambda: m(bad.to(cuda)), lambda: m.encoder(-bad), lambda: m.encoder(bad, return_all_tokens=True),
                 lambda: ve(bad)):
        with pytest.raises(ValueError, match="out of range"):
            call()
    assert ops.launch_count == n0 and not m._graphs and not m.encoder._graphs and not ve._graphs


def test_train_mode_gradients_are_unchanged(cuda, student):
    ids = student("text_b_causal").tokenizer(captions(), context_length=32)
    grads = []
    for graphs in (False, True):
        m = student("text_b_causal").enable_cuda_graphs(graphs).train()
        _, mem, _ = m(ids)
        (mem.float() ** 2).mean().backward()
        grads.append([None if p.grad is None else p.grad.clone() for p in m.parameters()])
        if graphs:
            assert not m._graphs                                     # the training graph is never captured
    for a, b in zip(*grads):
        assert (a is None and b is None) or torch.equal(a, b)


def test_batch_stat_bn_updates_running_buffers_as_without_graphs(cuda, student):
    ids = student().tokenizer(captions(), context_length=32)
    bufs, outs = [], []
    for graphs in (False, True):
        m = student().enable_cuda_graphs(graphs).enable_batch_stat_bn()
        if graphs:
            before = snap(m(ids))                                    # eval: captured with the initial running statistics
            assert len(m._graphs) == 1
        m.train()
        with torch.no_grad():
            outs.append([snap(m(ids)) for _ in range(2)])
        bufs.append([b.clone() for b in m.buffers()])
        if graphs:
            assert len(m._graphs) == 1                               # every forward updated the running buffers: never replayed
            m.eval()                                                 # the moved running statistics are folded into a new capture
            after = snap(m(ids))
            assert same(after, m.forward_uncaptured(ids)) and not torch.equal(after[1], before[1])
    assert all(same(a, b) for a, b in zip(*outs))
    assert all(torch.equal(a, b) for a, b in zip(*bufs))


def test_strict_and_cpu_still_raise(cuda, student, teacher):
    from efficientsam3_b200 import ops
    m = student().enable_cuda_graphs()
    m.encoder.enable_cuda_graphs()
    t = teacher().enable_cuda_graphs()
    with ops.strict_precision():
        with pytest.raises(NotImplementedError, match="strict"):
            m(["a cat"])
        with pytest.raises(NotImplementedError, match="strict"):
            m.encoder(torch.zeros(1, 32, dtype=torch.long))
        with pytest.raises(NotImplementedError, match="strict"):
            t(["a cat"], device=cuda)
    assert not m._graphs and not m.encoder._graphs
    with pytest.raises(RuntimeError, match="CPU fallback"):
        student().cpu().enable_cuda_graphs()(["a cat"])


# ------------------------------------------------------------------------------------------------ dump and off switch
def test_dump_with_graphs_writes_the_same_bytes(cuda, teacher, tmp_path):
    from efficientsam3_b200.stage1.embeddings import save_text_embeddings_one_epoch
    caps = captions() + [c + " again" for c in captions()[:4]]                       # 10 captions: batches 4, 4 and a short 2
    keys = [f"cap_{i}" for i in range(len(caps))]
    loader = [[caps[i:i + 4], [keys[i:i + 4], list(range(100 + i, 100 + i + len(caps[i:i + 4])))]] for i in range(0, len(caps), 4)]
    t = teacher()
    for graphs in (False, True):
        t.enable_cuda_graphs(graphs)
        assert save_text_embeddings_one_epoch(t, loader, str(tmp_path / f"store_{graphs}"), rank=0) == len(caps)
    assert len(t.sam3.backbone.language_backbone._graphs) == 2                    # batch 4 and the short last batch
    for f in ("rank0-keys.txt", "rank0-values.bin"):
        with open(tmp_path / "store_False" / f, "rb") as a, open(tmp_path / "store_True" / f, "rb") as b:
            assert a.read() == b.read(), f
    assert os.path.getsize(tmp_path / "store_True" / "rank0-values.bin") == len(caps) * (4 + 32 * 256 * 2)


def test_off_switch_returns_to_host_launches(cuda, student):
    from efficientsam3_b200 import ops
    m = student("text_b_causal")
    caps = captions()
    m.enable_cuda_graphs()
    got = snap(m(caps, device=cuda))
    m.enable_cuda_graphs(False)
    assert m._graphs is None
    n0 = ops.launch_count
    assert same(m(caps, device=cuda), got)
    assert ops.launch_count - n0 == m.graph_launches_per_step        # launched kernel by kernel again: the graph's kernels
