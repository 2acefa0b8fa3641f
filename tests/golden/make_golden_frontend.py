"""Frozen outputs of the reference build (oracle/_ref) on the front-end frame families of tests/frontend_cases.py, so
that test_frontend_cases_cpu.py needs neither the reference tree nor oracle/_ref at run time.  Run where oracle/_ref has
been built (oracle/Makefile `ref`):

    python tests/golden/make_golden_frontend.py

writes tests/golden/frontend_digests.json: per case, oracle.digest of the sampled plane, of the angle and modulus planes
and of the bucket list (LSD), or of the blurred plane and of the edge-point records (contour)."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import pyoracle as po  # noqa: E402
import frontend_cases as fc  # noqa: E402


def main():
    assert po.have_ref("contour") and po.have_ref("lsd"), "build oracle/_ref first"
    with open(os.path.join(HERE, "frontend_digests.json"), "w") as f:
        json.dump(fc.all_digests(po, "ref"), f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
