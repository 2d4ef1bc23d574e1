#!/usr/bin/env python
"""Debug aid (GPU box): align a named case of tests/cases.py with the product and compare every DP row's band, arg-max and
planes with the scalar oracle after every read (tests/planes.py, the rule tests/test_gpu_planes.py asserts), printing
which kernel ran and the first mismatching cells.
usage: python tests/debug_planes.py <case-name>"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
from abpoa_b200.aligner import PoaConfig  # noqa: E402
from cases import CASES, case_reads  # noqa: E402
from planes import run_planes  # noqa: E402


def main():
    name = sys.argv[1]
    case = CASES[name]

    def show(i, info):
        print(f"read {i}: {info.name} kernel, lean={int(info.lean)} tma={int(info.tma)} ring {info.ring_rows}x{info.ring_cells}: all rows equal")
    try:
        run_planes(PoaConfig(**case["cfg"]), case_reads(case), tag=name, check=show)
    except AssertionError as e:
        print(e)
        sys.exit(1)


if __name__ == "__main__":
    main()
