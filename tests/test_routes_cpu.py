"""tests/routes.py on the CPU: the route keys cover exactly the kernel entry points of include/es3.h, every entry point names the
test files whose tables run it, every covered key belongs to an entry point its file is listed for, and the route closure
rejects an unkeyed entry point and a key no table row runs; the GEMM tile rules routes.py restates from gemm_tc.cu, on the cases
their comments name."""
import ast
import importlib
import os

import pytest

import routes
from routes import COVERED, KEYS, assert_closed, conv3x3_num_kb, conv_tile_w, gemm_bn, gemm_stages, pick_bn
from test_boundary import _declared

HERE = os.path.dirname(os.path.abspath(__file__))
KERNEL_TEST_FILES = ["test_gemm_epilogue_gpu.py", "test_train_bwd_gpu.py", "test_fwd_kernels_gpu.py", "test_text_kernels_gpu.py",
                     "test_sam_kernels_gpu.py", "test_vit_kernels_gpu.py", "test_strict_kernels_gpu.py", "test_fp8_gpu.py",
                     "test_fp8_attention_gpu.py", "test_stage1_kernels_gpu.py"]
MBCONV_B1_STAGE3 = (0,) * 13 + (128, 512, 128, 1, 1, 2, 0)     # es3_mbconv_bf16 arguments: Cin 128, mid 512, Cout 128, stride 1
# es3_dwconv_f32 arguments of LiteMLA's strict 5 x 5 aggregation (EfficientViT-B1 stage 3 at 1024^2): no scale, no bias, no act
LITEMLA_AGGREG_F32 = (0, 768, 0, 0, 0, 0, 384, 2, 64, 64, 384, 5, 1, 0, 0)
# es3_gemm_bf16_ex arguments of the SAM3 ViT's global-attention QKV projection at 1008 px (72 x 72 tokens, B = 2): N = 3072, K = 1024,
# bias, bf16 out, RoPE on q | k with no window, no tile hint
GLOBAL_ROPE_QKV = (1, 1024, 2, 1024, 3, 3072, 0, 10368, 3072, 1024, 0, 4, 0, 0, 0, 0, 5, 2048, 72, 72, 0, 0, 0, 0)
GLOBAL_ROPE_QKV_KEY = ("es3_gemm_bf16_ex", 128, 4, None, False, True, None, False, "bf16", "global", False)
# es3_pw_small_bf16 arguments of an expand 16 -> 64 without residual (EfficientViT-B0 / B1 training forward at 1024^2)
PW_SMALL_16_64 = (1, 16, 2, 16, 3, 64, 0, 0, 2 * 256 * 256, 64, 16, 0)
# es3_adamw_flat arguments of a stage-1 update: a 9M-element arena whose decay group ends at 8M, clipped at 5, dynamic loss scale
ADAMW_STAGE1 = (1, 2, 3, 4, 9_000_000, 8_000_000, 1e-4, 0.9, 0.999, 1e-8, 0.05, 5.0, 1.0, 5, 6, 1, 2.0, 0.5, 2000, 0)


def test_keys_are_the_kernel_entry_points_of_the_header():
    assert set(KEYS) == {n for n in _declared() if routes.is_kernel(n)}


def test_every_entry_point_has_an_existing_covering_file():
    assert set(COVERED) == set(KEYS)
    for name, files in COVERED.items():
        assert files, name
        for f in files:
            assert os.path.isfile(os.path.join(HERE, f)), (name, f)


def test_covered_keys_belong_to_entry_points_listed_for_their_file():
    for f in sorted({f for files in COVERED.values() for f in files}):
        for key in routes.covered_keys(f):
            assert key[0] in KEYS, (f, key)
            assert f in COVERED[key[0]], (f, key)


def _top_level_defs(path):
    tree = ast.parse(open(path).read())
    names = {n.name for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef))}
    return names | {t.id for n in tree.body if isinstance(n, ast.Assign) for t in n.targets if isinstance(t, ast.Name)}


def test_no_test_file_defines_its_own_route_closure():
    for f in sorted(os.listdir(HERE)):
        if f.startswith("test_") and f.endswith(".py"):
            assert not _top_level_defs(os.path.join(HERE, f)) & {"route_key", "EXCLUDED", "_closure"}, f


@pytest.mark.parametrize("f", KERNEL_TEST_FILES)
def test_kernel_test_files_import_no_test_module(f):
    tree = ast.parse(open(os.path.join(HERE, f)).read())
    mods = {a.name for n in ast.walk(tree) if isinstance(n, ast.Import) for a in n.names}
    mods |= {n.module for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and n.module}
    assert not {m for m in mods if m.split(".")[0].startswith("test_")}, f


def test_closure_accepts_covered_calls_and_ignores_host_queries():
    reached = assert_closed([("es3_init", (0, 0, 0, 0)), ("es3_mbconv_bf16", MBCONV_B1_STAGE3)], "covered")
    assert reached == {("es3_mbconv_bf16", 128, 512, 128, 1)}


def test_closure_rejects_an_unkeyed_entry_point(monkeypatch):
    monkeypatch.delitem(KEYS, "es3_dense_pe")
    with pytest.raises(AssertionError, match="no route key"):
        assert_closed([("es3_dense_pe", (0,) * 6)], "unkeyed")


def test_closure_rejects_a_key_whose_table_row_is_gone(monkeypatch):
    fwd = importlib.import_module("test_fwd_kernels_gpu")
    monkeypatch.setattr(fwd, "MB_TC", [blk for blk in fwd.MB_TC if blk[0] != 128])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([("es3_mbconv_bf16", MBCONV_B1_STAGE3)], "row removed")


def test_closure_rejects_the_global_rope_qkv_once_its_row_is_gone(monkeypatch):
    call = ("es3_gemm_bf16_ex", GLOBAL_ROPE_QKV)
    assert assert_closed([call], "global rope qkv") == {GLOBAL_ROPE_QKV_KEY}
    gemm = importlib.import_module("test_gemm_epilogue_gpu")
    monkeypatch.setattr(gemm, "MODEL_ROWS", [r for r in gemm.MODEL_ROWS if r[0] != "rope"])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "global rope qkv row removed")


def test_closure_rejects_a_pw_small_16_to_64_once_its_row_is_gone(monkeypatch):
    call = ("es3_pw_small_bf16", PW_SMALL_16_64)
    assert assert_closed([call], "pw_small 16 -> 64") == {("es3_pw_small_bf16", 16, 64, False)}
    gemm = importlib.import_module("test_gemm_epilogue_gpu")
    monkeypatch.setattr(gemm, "MODEL_ROWS", [r for r in gemm.MODEL_ROWS if r[:1] + r[2:] != ("pw", 64, 16, None)])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "pw_small 16 -> 64 row removed")


def test_gemm_model_rows_add_keys_no_other_row_runs():
    """Each row of the GEMM file's model-route table selects its own key, one no table of sections (a) to (g) runs."""
    gemm = importlib.import_module("test_gemm_epilogue_gpu")
    keys = [gemm._model_row_key(r) for r in gemm.MODEL_ROWS]
    assert len(set(keys)) == len(keys)
    assert not set(keys) & gemm.table_keys()
    assert {k[0] for k in keys} == {"es3_gemm_bf16_ex", "es3_gemm_bf16", "es3_pw_small_bf16", "es3_gemm_simt", "es3_conv3x3_bf16"}


@pytest.mark.parametrize("N,bn_hint,K,act,bn", [
    (4096, 0, 256, "gelu", 64), (256, 0, 128, "gelu", 64),              # short K with GELU: 64 whatever N
    (384, 0, 256, None, 128), (1024, 0, 128, "hswish", 128),            # short K, N >= 384: 128
    (256, 0, 256, None, 64), (96, 0, 128, "relu", 64),                  # short K, 64 <= N < 384: 64
    (96, 256, 64, None, 128), (48, 256, 1024, "gelu", 128),             # hint 256: 128
    (256, 32, 1024, None, 32), (4736, 64, 1024, "gelu", 64),            # hints 32 / 64 / 128 are taken as given
    (1024, 0, 1024, None, 128), (1056, 0, 512, None, 128),              # long K: N % 128 == 0 or N > 1024
    (192, 0, 512, None, 64), (160, 0, 1024, None, 128), (96, 0, 512, None, 32), (48, 0, 64, None, 32)])
def test_pick_bn_restates_gemm_tc(N, bn_hint, K, act, bn):
    assert pick_bn(N, bn_hint, K, act) == bn


@pytest.mark.parametrize("N,K,bn_hint,bn", [(3072, 1024, 0, 128), (192, 1024, 0, 128), (128, 64, 0, 128), (96, 1024, 0, 32),
                                            (192, 1024, 64, 64)])
def test_rope_takes_128_wide_tiles_from_n_128(N, K, bn_hint, bn):
    """With RoPE, no hint and N >= 128 the tile is 128 wide, where pick_bn alone would give 64 (N = 192, or short K)."""
    assert gemm_bn(N, K, None, "global", bn_hint) == bn


def test_stage_rule_and_conv_geometry():
    assert [gemm_stages(128, kb) for kb in (1, 2, 3, 16)] == [2, 2, 4, 4]
    assert gemm_stages(64, 16) == 2 and gemm_stages(32, 1) == 4
    assert [conv_tile_w(W) for W in (64, 48, 144, 36, 23)] == [32, 16, 16, 8, 8]
    assert conv3x3_num_kb(8) == 9 and conv3x3_num_kb(96) == 18


def test_closure_rejects_a_strict_dwconv_whose_table_row_is_gone(monkeypatch):
    call = ("es3_dwconv_f32", LITEMLA_AGGREG_F32)
    assert assert_closed([call], "strict dwconv") == {("es3_dwconv_f32", 5, 1, None, False, False)}
    strict = importlib.import_module("test_strict_kernels_gpu")
    monkeypatch.setattr(strict, "DW", [c for c in strict.DW if (c[4], c[5], c[6], c[7], c[8]) != (5, 1, None, False, False)])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "strict dwconv row removed")


def test_closure_rejects_a_clipped_decay_split_adamw_once_its_row_is_gone(monkeypatch):
    call = ("es3_adamw_flat", ADAMW_STAGE1)
    key = ("es3_adamw_flat", True, True, False, True)
    assert assert_closed([call], "stage-1 adamw") == {key}
    stage1 = importlib.import_module("test_stage1_kernels_gpu")
    monkeypatch.setattr(stage1, "ADAMW", [c for c in stage1.ADAMW if routes.adamw_key(c[0], stage1._n_decay(c[0], c[1]), c[4], c[9]) != key])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "stage-1 adamw row removed")


def test_stage1_keys_follow_what_the_arguments_select():
    assert KEYS["es3_grad_norm"]((1, 16384 * 4096, 2, 3, 0)) == ("es3_grad_norm", False, False)
    assert KEYS["es3_grad_norm"]((1, 16384 * 4096 + 4, 2, 3, 0)) == ("es3_grad_norm", False, True)
    assert KEYS["es3_grad_norm"]((1, 1021, 2, 3, 0)) == ("es3_grad_norm", True, False)
    assert KEYS["es3_adamw_flat"](ADAMW_STAGE1[:4] + (8, 8) + ADAMW_STAGE1[6:11] + (0.0,) + ADAMW_STAGE1[12:15] + (0,) +
                                  ADAMW_STAGE1[16:]) == ("es3_adamw_flat", False, False, False, False)
    assert KEYS["es3_kd_loss_fwd"]((1, 2, 3, 2, 1024, 64, 1024, 1.0, 4, 5, 0, 0)) == ("es3_kd_loss_fwd", False)
    assert KEYS["es3_kd_loss_bwd"]((1, 2, 3, 4, 5, 1.0, 2, 1024, 64, 1024, 1.0, 6, 0)) == ("es3_kd_loss_bwd", True)
