"""Run bench.py against another build of libes3.so (same C ABI), so that two builds can be timed alternately without
rebuilding the tree in between:

    python scripts/ab_bench.py PATH/TO/libes3.so [bench.py arguments ...]
"""
from __future__ import annotations

import os
import runpy
import sys
from pathlib import Path

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from efficientsam3_b200 import _lib  # noqa: E402

_lib.LIB_PATH = Path(sys.argv[1]).resolve()
sys.argv = [os.path.join(ROOT, "bench.py"), *sys.argv[2:]]
runpy.run_path(sys.argv[0], run_name="__main__")
