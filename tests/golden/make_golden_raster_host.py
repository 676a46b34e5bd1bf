"""Writes tests/golden/raster_host_calls.json: the digest of each case's record of test_raster_host_cpu (the rasterizer
host layer's library calls and gradients, with the library replaced by stand-ins).  Run from the repository root
after building: python tests/golden/make_golden_raster_host.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import pytest  # noqa: E402

import test_raster_host_cpu as T  # noqa: E402


def main():
    out = {}
    for case in T.cases():
        with pytest.MonkeyPatch.context() as mp:
            out[case[0]] = T.digest(T.record(case, mp))
    with open(T.GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {T.GOLDEN}")


if __name__ == "__main__":
    main()
