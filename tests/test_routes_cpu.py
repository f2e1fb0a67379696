"""tests/routes.py on the CPU: the route keys cover exactly the kernel entry points of include/es3.h, every entry point names the
test files whose tables run it, every covered key belongs to an entry point its file is listed for, and the route closure
rejects an unkeyed entry point and a key no table row runs."""
import ast
import importlib
import os

import pytest

import routes
from routes import COVERED, KEYS, assert_closed
from test_boundary import _declared

HERE = os.path.dirname(os.path.abspath(__file__))
KERNEL_TEST_FILES = ["test_gemm_epilogue_gpu.py", "test_train_bwd_gpu.py", "test_fwd_kernels_gpu.py", "test_text_kernels_gpu.py",
                     "test_sam_kernels_gpu.py", "test_vit_kernels_gpu.py", "test_strict_kernels_gpu.py"]
MBCONV_B1_STAGE3 = (0,) * 13 + (128, 512, 128, 1, 1, 2, 0)     # es3_mbconv_bf16 arguments: Cin 128, mid 512, Cout 128, stride 1
# es3_dwconv_f32 arguments of LiteMLA's strict 5 x 5 aggregation (EfficientViT-B1 stage 3 at 1024^2): no scale, no bias, no act
LITEMLA_AGGREG_F32 = (0, 768, 0, 0, 0, 0, 384, 2, 64, 64, 384, 5, 1, 0, 0)


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


def test_closure_accepts_a_gemm_only_because_covered_lists_it(monkeypatch):
    call = ("es3_gemm_bf16_ex", (0,) * 24)
    assert assert_closed([call], "gemm") == {("es3_gemm_bf16_ex",)}
    monkeypatch.setitem(COVERED, "es3_gemm_bf16_ex", ["test_fwd_kernels_gpu.py"])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "gemm unlisted")


def test_closure_rejects_a_strict_dwconv_whose_table_row_is_gone(monkeypatch):
    call = ("es3_dwconv_f32", LITEMLA_AGGREG_F32)
    assert assert_closed([call], "strict dwconv") == {("es3_dwconv_f32", 5, 1, None, False, False)}
    strict = importlib.import_module("test_strict_kernels_gpu")
    monkeypatch.setattr(strict, "DW", [c for c in strict.DW if (c[4], c[5], c[6], c[7], c[8]) != (5, 1, None, False, False)])
    with pytest.raises(AssertionError, match="no table row runs"):
        assert_closed([call], "strict dwconv row removed")
