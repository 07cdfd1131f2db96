"""Compile models/ant_delay.xml (the ant with actuator and sensor history buffers, authored here) into
tests/golden/ant_delay.mjb with the reference's own compiler and mj_saveModel (the product has no MJCF compiler).
Run where the oracle is built.

Usage: python tests/golden/make_delay_fixture.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_util import Oracle  # noqa: E402


def main():
    Oracle(os.path.join(ROOT, "models", "ant_delay.xml")).save_mjb(os.path.join(ROOT, "tests", "golden", "ant_delay.mjb"))
    print("wrote tests/golden/ant_delay.mjb")


if __name__ == "__main__":
    main()
