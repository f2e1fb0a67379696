"""es3_mbconv_tc_wide_bf16: the Cin-128 blocks of the fused wgmma MBConv kernels -- (128, 512, 128) stride 1 with residual in
mbconv_tc.cu and (128, 512, 256) stride 2 without in mbconv_tc_s2.cu, their input tile held as two 64-channel slabs -- element by
element against the fp64 statement of tests/ref_fwd.py, under the harness of tests/test_fwd_kernels_gpu.py: NaN-prefilled
outputs, two runs bit-identical, image i of a batch bit-identical to image i alone, nothing written outside the output region,
declined shapes write nothing, ops.mbconv_fused bit-identical to the direct call.  The route-closure test records every key of
this entry point the nine students reach in an eval forward and asserts that WIDE has a row for it.
"""
import pytest
import torch

from bounds import _assert_untouched, _bf, _flat_out, _gen, report_worst
from es3_recorder import STUDENTS, eval_forward_calls
from test_fwd_kernels_gpu import _bits_equal, _lib, _mb_call, _mb_case, _mb_weights

pytestmark = pytest.mark.gpu
_report_worst = report_worst("mbconv wide")
FN = "es3_mbconv_tc_wide_bf16"
WIDE = [(128, 512, 128, 1), (128, 512, 256, 2)]
# 1 x 1, below one tile, one tile (stride 1: 8 x 16 output, stride 2: 8 x 32 input) and one pixel past it, the ragged 63 x 63
# that 1008-px inputs give, and the EV-M shape of bench.py (64 x 64 at batch 32)
GEO = {1: [(2, 1, 1), (2, 3, 5), (2, 1, 37), (1, 8, 16), (2, 7, 15), (2, 9, 17), (2, 63, 63), (32, 64, 64)],
       2: [(2, 1, 1), (2, 3, 5), (2, 1, 37), (1, 8, 32), (2, 7, 31), (2, 10, 34), (2, 63, 63), (32, 64, 64)]}


@pytest.mark.parametrize("cin,mid,cout,stride,B,H,W", [blk + geo for blk in WIDE for geo in GEO[blk[3]]])
def test_mbconv_tc_wide(cuda, cin, mid, cout, stride, B, H, W):
    """Both instantiations; ops.mbconv_fused (default routing, as the models call it) must be bit-identical to the direct call."""
    _mb_case(cuda, FN, None, cin, mid, cout, stride, B, H, W)


@pytest.mark.parametrize("blk", WIDE)
def test_mbconv_tc_wide_batch_invariant(cuda, blk):
    """Image i of a batch is bit-identical to image i run alone (every persistent CTA runs tiles of several images)."""
    B = 24
    x, wt, taps, y = _mb_case(cuda, FN, None, *blk, B, 37, 37)
    lib = _lib(cuda)
    for i in (0, B // 2, B - 1):
        one = torch.full_like(y[i:i + 1], float("nan"))
        assert _mb_call(lib, FN, x[i:i + 1].contiguous(), one, wt, taps, *blk, blk[3] == 1) == 0
        _bits_equal(one[0], y[i], f"{FN} image {i} of {B} vs alone")


@pytest.mark.parametrize("blk,res", [((256, 1024, 256, 1), True), ((128, 512, 128, 2), False), ((128, 512, 256, 1), True),
                                     ((128, 512, 128, 1), False), ((128, 512, 256, 2), True), ((64, 256, 64, 1), True),
                                     ((128, 256, 128, 1), True)])
def test_mbconv_tc_wide_declined_shapes_write_nothing(cuda, blk, res):
    lib = _lib(cuda)
    cin, mid, cout, stride = blk
    g = _gen(cuda, "decl-wide", blk, res)
    x = _bf(torch.randn(1, 9, 9, cin, device=cuda, generator=g))
    wt = _mb_weights(cuda, cin, mid, cout, g)
    buf, inside = _flat_out(81 * cout, torch.bfloat16, cuda)
    assert _mb_call(lib, FN, x, buf, wt, wt[3], cin, mid, cout, stride, res) == -1
    torch.cuda.synchronize()
    _assert_untouched(buf, torch.zeros_like(inside), f"{FN} declined {blk} residual={res}")


@pytest.mark.parametrize("name", STUDENTS)
def test_mbconv_tc_wide_route_closure(cuda, monkeypatch, name):
    """Every (Cin, Mid, Cout, stride) `name` runs through es3_mbconv_tc_wide_bf16 in the eval forward at 1024^2 is a row of WIDE;
    efficientvit_b1 runs both (its stage-3 blocks and stage-4 opener), efficientvit_b0 the stride-1 one (its stage-4 blocks)."""
    reached = {tuple(a[13:17]) for n, a in eval_forward_calls(cuda, monkeypatch, name) if n == FN}
    print(f"\n{name}: {FN} keys reached: {sorted(reached)}", end="")
    assert reached <= set(WIDE), f"{name} reaches {FN} shapes no row runs: {sorted(reached - set(WIDE))}"
    expected = {"efficientvit_b1": set(WIDE), "efficientvit_b0": {WIDE[0]}}.get(name)
    if expected is not None:
        assert reached == expected, f"{name}: {FN} reached {sorted(reached)}, expected {sorted(expected)}"
