"""Compile models/convex.xml (the convex narrow-phase test model, authored here) into tests/golden/convex.mjb with the
reference's own compiler and mj_saveModel (the product has no MJCF compiler).  Run where the oracle is built.

Usage: python tests/golden/make_convex_fixture.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_util import Oracle  # noqa: E402


def main():
    out = os.path.join(ROOT, "tests", "golden", "convex.mjb")
    Oracle(os.path.join(ROOT, "models", "convex.xml")).save_mjb(out)
    print("wrote tests/golden/convex.mjb")


if __name__ == "__main__":
    main()
