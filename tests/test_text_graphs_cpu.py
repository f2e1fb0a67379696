"""CPU: the CUDA-graph switch of the text encoders (enable_cuda_graphs) is off by default, delegates from the SAM3 text teacher to
its VETextEncoder, and leaves the raise paths of CPU modules as they are (no CPU fallback, nothing captured)."""
import pytest
import torch

from helpers import load_golden
from test_text_cpu import BPE, build_student


def test_switch_is_off_by_default_and_returns_the_module():
    m = build_student(load_golden("text_s0_ctx32"))
    assert m._graphs is None and m.encoder._graphs is None and m.graph_launches_per_step == 0
    assert m.enable_cuda_graphs(max_graphs=3) is m and m._graphs == {} and m._graph_max == 3
    assert m.encoder._graphs is None                                 # each module has its own switch
    assert m.enable_cuda_graphs(False) is m and m._graphs is None
    with pytest.raises(ValueError, match="max_graphs"):
        m.enable_cuda_graphs(max_graphs=0)


def test_teacher_delegates_to_its_text_encoder():
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
    t = SAM3TextTeacherEncoder(context_length=16, bpe_path=BPE, ve_overrides=dict(layers=1))
    ve = t.sam3.backbone.language_backbone
    assert t.enable_cuda_graphs(max_graphs=2) is t and ve._graphs == {} and ve._graph_max == 2
    assert t.graph_launches_per_step == ve.graph_launches_per_step == 0
    t.enable_cuda_graphs(False)
    assert ve._graphs is None


def test_cpu_modules_still_raise_with_graphs_on():
    from efficientsam3_b200.stage1.model import SAM3TextTeacherEncoder
    m = build_student(load_golden("text_s0_ctx32")).enable_cuda_graphs()
    m.encoder.enable_cuda_graphs()
    t = SAM3TextTeacherEncoder(context_length=16, bpe_path=BPE, ve_overrides=dict(layers=1)).enable_cuda_graphs()
    for call in (lambda: m(["a cat"]), lambda: m.encoder(torch.zeros(1, 32, dtype=torch.long)), lambda: t(["a cat"])):
        with pytest.raises(RuntimeError, match="CPU fallback"):
            call()
    assert m._graphs == {} and m.encoder._graphs == {} and t.sam3.backbone.language_backbone._graphs == {}
