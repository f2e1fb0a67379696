"""Stage-1 image preparation from decoded uint8 (stage1/preprocess.py, csrc/preprocess.cu), host side: the resized shape, the oracle
against the reference's own transform (tests/golden/preprocess_small.npz), the packed layout, the host-side refusal of every
malformed input before anything is copied or launched, and the kernels' register budget."""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import preprocess as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from gen_golden_preprocess import CASES, case_image  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preprocess_small.npz")


def test_preprocess_shape_matches_fixture_and_formula():
    from efficientsam3_b200.stage1.preprocess import get_preprocess_shape
    g = np.load(GOLDEN)
    for (tag, h, w, S, _), size in zip(CASES, g["sizes"]):
        assert (3, *get_preprocess_shape(h, w, S)) == tuple(size), tag
    for S in (1, 96, 1008, 1024):
        for h in (1, 2, 3, 7, 37, 375, 1500, 2250, 4000):
            for w in (1, 5, 23, 640, 1001, 1500, 2250):
                assert get_preprocess_shape(h, w, S) == O.get_preprocess_shape(h, w, S), (h, w, S)


def test_kernel_shape_rule_matches_python():
    """es3_prepare_images_ws_floats sizes the workspace from the C restatement of get_preprocess_shape: h * w' * 3 per image."""
    from efficientsam3_b200 import ops
    from efficientsam3_b200.stage1.preprocess import get_preprocess_shape
    for S in (1, 96, 1008):
        for h, w in [(1, 1), (2250, 1500), (1500, 2250), (37, 23), (600, 800), (1, 2), (999, 1001)]:
            if min(get_preprocess_shape(h, w, S)) < 1:
                continue
            table = torch.tensor([[0, h, w]], dtype=torch.int64)
            assert ops.image_table_ws_floats(table, h * w * 3, S) == h * get_preprocess_shape(h, w, S)[1] * 3, (h, w, S)


def test_oracle_matches_reference_fixture():
    g = np.load(GOLDEN)
    for (tag, h, w, S, seed), size in zip(CASES, g["sizes"]):
        x, sz = O.prepare_image(case_image(h, w, seed), S)
        want = torch.from_numpy(g[f"out_{tag}"])
        assert sz == tuple(size) and x.shape == want.shape == (3, S, S), tag
        assert (x - want).abs().max().item() <= 1e-6, tag


def test_pack_images_layout():
    from efficientsam3_b200.stage1.preprocess import PackedImages, pack_images
    imgs = [case_image(h, w, s) for h, w, s in [(5, 7, 0), (1, 1, 1), (3, 2, 2)]]
    p = pack_images(imgs)
    assert isinstance(p, PackedImages) and len(p) == 3
    assert p.data.dtype == torch.uint8 and p.data.shape == (5 * 7 * 3 + 3 + 3 * 2 * 3,)
    assert p.sizes.dtype == torch.int64 and p.sizes.tolist() == [[5, 7], [1, 1], [3, 2]]
    assert p.table().tolist() == [[0, 5, 7], [105, 1, 1], [108, 3, 2]]
    for (off, h, w), img in zip(p.table().tolist(), imgs):
        assert torch.equal(p.data[off:off + h * w * 3].view(h, w, 3), img)


def _malformed():
    good = case_image(20, 30, 0)
    return {
        "float_image": ([good.float()], 64),
        "two_channels": ([good[:, :, :2].contiguous()], 64),
        "chw_layout": ([good.permute(2, 0, 1).contiguous()], 64),
        "zero_height": ([good[:0]], 64),
        "zero_width": ([good[:, :0]], 64),
        "not_contiguous": ([good[:, ::2]], 64),
        "no_images": ([], 64),
        "size_zero": ([good], 0),
        "thin_strip_rounds_to_zero": ([case_image(1, 300, 1)], 128),
    }


@pytest.mark.parametrize("case", sorted(_malformed()))
def test_malformed_inputs_raise_before_any_launch(case):
    from efficientsam3_b200 import _lib, ops
    from efficientsam3_b200.stage1.preprocess import prepare_images
    images, S = _malformed()[case]
    n0 = ops.launch_count
    with pytest.raises(_lib.Es3Error):
        prepare_images(images, S)
    assert ops.launch_count == n0


def test_packed_batch_outside_its_buffer_raises_before_any_launch():
    from efficientsam3_b200 import _lib, ops
    from efficientsam3_b200.stage1.preprocess import PackedImages, prepare_images
    data = case_image(10, 10, 0).reshape(-1)
    n0 = ops.launch_count
    for sizes in ([[10, 11]], [[10, 10], [1, 1]]):
        with pytest.raises(_lib.Es3Error, match="outside"):
            prepare_images(PackedImages(data, torch.tensor(sizes, dtype=torch.int64)), 32)
    with pytest.raises(_lib.Es3Error, match="outside"):
        ops.image_table_ws_floats(torch.tensor([[-3, 2, 2]], dtype=torch.int64), data.numel(), 32)
    assert ops.launch_count == n0


def test_uint8_batch_detection():
    from efficientsam3_b200.stage1.preprocess import is_uint8_batch, pack_images
    img = case_image(4, 4, 0)
    assert is_uint8_batch([img]) and is_uint8_batch((img,)) and is_uint8_batch(pack_images([img]))
    assert not is_uint8_batch([img.float()]) and not is_uint8_batch(torch.zeros(1, 3, 4, 4)) and not is_uint8_batch([])


def _nvcc():
    from efficientsam3_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None
    return nvcc if shutil.which(nvcc) else None


def test_preprocess_kernels_do_not_spill(tmp_path):
    """-Xptxas -v for sm_90a: neither pass spills or keeps a stack frame (the descriptor table is a __grid_constant__ parameter:
    indexing a by-value parameter array would otherwise copy it to local memory)."""
    from efficientsam3_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "preprocess.cu"), "-o", str(tmp_path / "preprocess.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rows, name = [], None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name is not None:
            rows.append((name, *map(int, m.groups())))
            name = None
    assert {n for n in (r[0] for r in rows) if "prep_" in n} and len(rows) == 2, rows
    assert all(r[1] == r[2] == r[3] == 0 for r in rows), rows
