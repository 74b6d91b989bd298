"""Generates tests/golden/initflow_digests.json from the REFERENCE build (oracle/_ref, the reference's own sources
compiled in place by oracle/Makefile): SHA-256 of the reference's float32 output bits for runs that start from the
init flow of tests/test_initflow.py's cases (inputs the tests regenerate from seeds).  Run where the reference
sources are (oracle/Makefile's REF):

    make -C oracle ref && python tests/golden/make_initflow_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_initflow  # noqa: E402


def main():
    out_dir = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(out_dir, "initflow_digests.json"), "w") as f:
        json.dump(test_initflow.make_digests(), f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
